// ControlNet edges: the conditioning embedding's few-channel 3x3 convolutions at image resolution
// (sfb_conv3x3_small; sfb_conv3x3_small_ex adds the input transform and ReLU of the tiny VAE's edge
// convolutions) and the gather of the 13 scaled residuals into the NCHW outputs
// (sfb_nhwc_to_nchw_scaled).  The reference leaves the whole ControlNetModel to eager PyTorch.
#include "common.cuh"
#include "host.h"

namespace sfb {

// ---------------------------------------------------------------------------------------
// 3x3 convolution, padding 1, stride 1 or 2, cin < 64, as an implicit GEMM on mma.sync m16n8k16:
// M = output pixels, N = cout, K = (tap, 16-channel group).  One CTA = 4 warps = an 8 x 16 output
// patch; warp w owns output rows 2w and 2w + 1 (one m16 tile = 16 consecutive pixels of a row).
// The input halo of the patch is staged in shared memory once, channels zero-padded to cin16 and the
// pixel pitch padded by 8 halves (fewer bank conflicts on the A-fragment loads); the weights
// ([cout][3][3][cin16], a few KB) are read straight from global memory and stay in L1.
// ---------------------------------------------------------------------------------------
constexpr int kSmallTH = 8, kSmallTW = 16;

struct ConvSmallArgs {
    const uint16_t* x;
    const uint16_t* w;
    const float* bias;
    uint16_t* y;
    int n, h, wd, cin, cin16, cout, stride, ldx, ldy, x_nchw, silu, ho, wo, tiles_w;
    int in_xform, relu;  // sfb_conv3x3_small_ex (NCHW input only)
};

// SFB_XFORM_* of an in-image input value, rounded back to 16 bits (the stored input of the conv)
template <int BF16>
__device__ __forceinline__ uint16_t xform16(uint16_t v, int xform) {
    float f = unpack2(v, BF16).x;
    f = xform == SFB_XFORM_TANH3 ? tanhf(f * (1.0f / 3.0f)) * 3.0f : (f + 1.0f) * 0.5f;
    return (uint16_t)(pack2(f, 0.f, BF16) & 0xffffu);
}

template <int BF16>
__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    if (BF16) {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                     "{%0,%1,%2,%3};"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    } else {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                     "{%0,%1,%2,%3};"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    }
}

template <int BF16>
__global__ void __launch_bounds__(128) conv3x3_small_kernel(const ConvSmallArgs a) {
    extern __shared__ __align__(16) uint16_t halo[];
    const int s = a.stride;
    const int hh = (kSmallTH - 1) * s + 3, hw = (kSmallTW - 1) * s + 3;
    const int ps = a.cin16 + 8;  // halves per staged pixel
    const int img = blockIdx.y;
    const int oy0 = (blockIdx.x / a.tiles_w) * kSmallTH, ox0 = (blockIdx.x % a.tiles_w) * kSmallTW;
    const int gy0 = oy0 * s - 1, gx0 = ox0 * s - 1;
    pdl_launch_dependents();
    pdl_wait();
    if (a.x_nchw) {
        // one 16-bit element per thread and step, w fastest: coalesced along image rows
        const int total = a.cin16 * hh * hw;
        for (int i = threadIdx.x; i < total; i += blockDim.x) {
            const int hx = i % hw, hy = (i / hw) % hh, c = i / (hw * hh);
            const int gy = gy0 + hy, gx = gx0 + hx;
            uint16_t v = 0;
            if (c < a.cin && gy >= 0 && gy < a.h && gx >= 0 && gx < a.wd)
                v = a.x[(((size_t)img * a.cin + c) * a.h + gy) * a.wd + gx];
            if (a.in_xform && c < a.cin && gy >= 0 && gy < a.h && gx >= 0 && gx < a.wd) v = xform16<BF16>(v, a.in_xform);
            halo[(hy * hw + hx) * ps + c] = v;
        }
    } else {
        // one 8-channel (16-byte) vector per thread and step
        const int nv = a.cin16 / 8;
        const int total = nv * hh * hw;
        for (int i = threadIdx.x; i < total; i += blockDim.x) {
            const int v = i % nv, px = i / nv;
            const int hx = px % hw, hy = px / hw;
            const int gy = gy0 + hy, gx = gx0 + hx;
            uint4 val = make_uint4(0u, 0u, 0u, 0u);
            if (v * 8 < a.cin && gy >= 0 && gy < a.h && gx >= 0 && gx < a.wd)
                val = *reinterpret_cast<const uint4*>(a.x + (((size_t)img * a.h + gy) * a.wd + gx) * a.ldx + v * 8);
            *reinterpret_cast<uint4*>(&halo[(hy * hw + hx) * ps + v * 8]) = val;
        }
    }
    __syncthreads();

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, q = lane & 3;  // fragment row group / column pair
    const int ck = a.cin16 / 16;
    const int nk = 9 * ck;
    for (int nc0 = 0; nc0 < a.cout; nc0 += 32) {
        float acc[2][4][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.f;
        for (int kc = 0; kc < nk; ++kc) {
            const int tap = kc / ck, cg = kc - tap * ck;
            const int ty = tap / 3, tx = tap - ty * 3;
            const int ch = cg * 16 + q * 2;
            uint32_t af[2][4];
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                const int hy = (2 * warp + mt) * s + ty;
                const uint16_t* r0 = &halo[(hy * hw + g * s + tx) * ps + ch];
                const uint16_t* r1 = &halo[(hy * hw + (g + 8) * s + tx) * ps + ch];
                af[mt][0] = *reinterpret_cast<const uint32_t*>(r0);
                af[mt][1] = *reinterpret_cast<const uint32_t*>(r1);
                af[mt][2] = *reinterpret_cast<const uint32_t*>(r0 + 8);
                af[mt][3] = *reinterpret_cast<const uint32_t*>(r1 + 8);
            }
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const int n = nc0 + nt * 8;
                if (n >= a.cout) break;  // warp-uniform
                const uint16_t* wr = a.w + ((size_t)(n + g) * 9 + tap) * a.cin16 + ch;
                const uint32_t b0 = __ldg(reinterpret_cast<const unsigned int*>(wr));
                const uint32_t b1 = __ldg(reinterpret_cast<const unsigned int*>(wr + 8));
                mma_16816<BF16>(acc[0][nt], af[0], b0, b1);
                mma_16816<BF16>(acc[1][nt], af[1], b0, b1);
            }
        }
        // epilogue: c0, c1 -> pixel g, channels 2q, 2q + 1; c2, c3 -> pixel g + 8
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            const int c = nc0 + nt * 8 + q * 2;
            if (c >= a.cout) break;
            const float b0 = a.bias ? a.bias[c] : 0.f, b1 = a.bias ? a.bias[c + 1] : 0.f;
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                const int oy = oy0 + 2 * warp + mt;
                if (oy >= a.ho) continue;
#pragma unroll
                for (int half = 0; half < 2; ++half) {
                    const int ox = ox0 + g + 8 * half;
                    if (ox >= a.wo) continue;
                    float v0 = acc[mt][nt][2 * half] + b0, v1 = acc[mt][nt][2 * half + 1] + b1;
                    if (a.silu) { v0 = silu_f(v0); v1 = silu_f(v1); }
                    if (a.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                    *reinterpret_cast<uint32_t*>(a.y + (((size_t)img * a.ho + oy) * a.wo + ox) * a.ldy + c) =
                        pack2(v0, v1, BF16);
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------
// dst[n, c, hw] (NCHW contiguous) = scale[item] * src[n, hw, c] (NHWC, channel pitch ld) for up to 16
// tensors in ONE launch: the ControlNet's 12 (SD-1.5) down-block residuals and its mid-block residual,
// times conditioning_scale.  32 x 32 (pixel, channel) tiles transposed through shared memory: reads
// coalesced along c, writes along hw.  The scale is read from device memory, so a captured graph
// serves every conditioning_scale / guess-mode setting.
// ---------------------------------------------------------------------------------------
struct NchwScaledArgs {
    int count, dtype;
    const float* scale;
    const uint16_t* src[16];
    uint16_t* dst[16];
    int n[16], c[16], hw[16], ld[16];
    int tile_end[16];  // exclusive prefix of 32x32 tiles per item
};

__global__ void __launch_bounds__(256) nhwc_to_nchw_scaled_kernel(const NchwScaledArgs a) {
    __shared__ float tile[32][33];
    pdl_launch_dependents();
    pdl_wait();
    int it = 0;
    while (it < a.count - 1 && (int)blockIdx.x >= a.tile_end[it]) ++it;
    const int t = blockIdx.x - (it ? a.tile_end[it - 1] : 0);
    const int c = a.c[it], hw = a.hw[it], ld = a.ld[it];
    const int tc = (c + 31) / 32, tp = (hw + 31) / 32;
    const int img = t / (tc * tp);
    const int rem = t - img * tc * tp;
    const int c0 = (rem / tp) * 32, p0 = (rem % tp) * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
    const uint16_t* src = a.src[it] + (size_t)img * hw * ld;
    uint16_t* dst = a.dst[it] + (size_t)img * c * hw;
    const float sc = a.scale[it];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int px = p0 + ty + 8 * j, ch = c0 + tx;
        tile[ty + 8 * j][tx] = (ch < c && px < hw) ? load1(src, (size_t)px * ld + ch, a.dtype) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int ch = c0 + ty + 8 * j, px = p0 + tx;
        if (ch < c && px < hw) store1(dst, (size_t)ch * hw + px, sc * tile[tx][ty + 8 * j], a.dtype);
    }
}

}  // namespace sfb

using namespace sfb;

static int conv3x3_small(const sfb_conv_small_params* p, int in_xform, int relu, sfb_stream_t stream) {
    if (!p || !p->x || !p->weight || !p->y || p->n <= 0 || p->h <= 0 || p->w <= 0)
        return fail(SFB_ERR_INVALID, "conv3x3_small: null pointer or empty image");
    if (p->stride != 1 && p->stride != 2) return fail(SFB_ERR_INVALID, "conv3x3_small: stride %d must be 1 or 2", p->stride);
    if (p->x_nchw ? (p->cin <= 0 || p->cin > 8) : (p->cin <= 0 || p->cin >= 64 || p->cin % 8 || p->ldx % 8 || p->ldx < p->cin))
        return fail(SFB_ERR_INVALID, "conv3x3_small: cin=%d ldx=%d (NCHW: cin <= 8; NHWC: cin < 64, cin and ldx multiples of 8)",
                    p->cin, p->ldx);
    if (p->cout <= 0 || p->cout % 8 || p->ldy % 8 || p->ldy < p->cout)
        return fail(SFB_ERR_INVALID, "conv3x3_small: cout=%d ldy=%d must be multiples of 8 with ldy >= cout", p->cout, p->ldy);
    if (p->dtype != SFB_F16 && p->dtype != SFB_BF16) return fail(SFB_ERR_INVALID, "conv3x3_small: dtype %d", p->dtype);
    ConvSmallArgs a{};
    a.x = reinterpret_cast<const uint16_t*>(p->x);
    a.w = reinterpret_cast<const uint16_t*>(p->weight);
    a.bias = p->bias;
    a.y = reinterpret_cast<uint16_t*>(p->y);
    a.n = p->n; a.h = p->h; a.wd = p->w; a.cin = p->cin; a.cin16 = (p->cin + 15) / 16 * 16;
    a.cout = p->cout; a.stride = p->stride; a.ldx = p->ldx; a.ldy = p->ldy;
    a.x_nchw = p->x_nchw ? 1 : 0; a.silu = p->silu ? 1 : 0;
    a.in_xform = in_xform; a.relu = relu ? 1 : 0;
    a.ho = (p->h - 1) / p->stride + 1;
    a.wo = (p->w - 1) / p->stride + 1;
    a.tiles_w = (a.wo + kSmallTW - 1) / kSmallTW;
    const int tiles = a.tiles_w * ((a.ho + kSmallTH - 1) / kSmallTH);
    if (p->n > 65535) return fail(SFB_ERR_INVALID, "conv3x3_small: batch %d > 65535", p->n);
    const size_t smem = (size_t)((kSmallTH - 1) * p->stride + 3) * ((kSmallTW - 1) * p->stride + 3) * (a.cin16 + 8) * 2;
    // stride 2 with cin16 = 64 stages 79 KB: past the default 48 KB, opted in once per device
    constexpr size_t kSmemOptin = 96 * 1024;
    if (smem > 48 * 1024) {
        static PerDeviceOnce attr_once;
        bool& attr_set = attr_once.flag();
        if (!attr_set) {
            for (cudaError_t err : {cudaFuncSetAttribute(conv3x3_small_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                         (int)kSmemOptin),
                                    cudaFuncSetAttribute(conv3x3_small_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                         (int)kSmemOptin)})
                if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "conv3x3_small: smem attribute: %s", cudaGetErrorString(err));
            attr_set = true;
        }
    }
    const dim3 grid(tiles, p->n);
    cudaError_t err = p->dtype == SFB_BF16
        ? launch_pdl(conv3x3_small_kernel<1>, grid, dim3(128), smem, static_cast<cudaStream_t>(stream), a)
        : launch_pdl(conv3x3_small_kernel<0>, grid, dim3(128), smem, static_cast<cudaStream_t>(stream), a);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "conv3x3_small: %s", cudaGetErrorString(err));
    return check_launch("sfb_conv3x3_small");
}

extern "C" int sfb_conv3x3_small(const sfb_conv_small_params* p, sfb_stream_t stream) {
    return conv3x3_small(p, SFB_XFORM_NONE, 0, stream);
}

extern "C" int sfb_conv3x3_small_ex(const sfb_conv_small_ex_params* p, sfb_stream_t stream) {
    if (!p) return fail(SFB_ERR_INVALID, "conv3x3_small_ex: null params");
    if (p->in_xform < SFB_XFORM_NONE || p->in_xform > SFB_XFORM_UNIT)
        return fail(SFB_ERR_INVALID, "conv3x3_small_ex: in_xform %d", p->in_xform);
    if (p->in_xform != SFB_XFORM_NONE && !p->base.x_nchw)
        return fail(SFB_ERR_INVALID, "conv3x3_small_ex: an input transform needs the NCHW input (x_nchw = 1)");
    if (p->relu && p->base.silu) return fail(SFB_ERR_INVALID, "conv3x3_small_ex: relu and silu are exclusive");
    return conv3x3_small(&p->base, p->in_xform, p->relu, stream);
}

extern "C" int sfb_nhwc_to_nchw_scaled(const sfb_nhwc_to_nchw_params* p, sfb_stream_t stream) {
    if (!p || p->count <= 0 || p->count > 16) return fail(SFB_ERR_INVALID, "nhwc_to_nchw_scaled: count must be 1..16");
    if (!p->scale) return fail(SFB_ERR_INVALID, "nhwc_to_nchw_scaled: scale is NULL");
    NchwScaledArgs a{};
    a.count = p->count; a.dtype = p->dtype; a.scale = p->scale;
    long long tiles = 0;
    for (int i = 0; i < p->count; ++i) {
        const sfb_nchw_scaled_item& it = p->items[i];
        if (!it.src || !it.dst || it.n <= 0 || it.c <= 0 || it.hw <= 0 || it.ld_src < it.c)
            return fail(SFB_ERR_INVALID, "nhwc_to_nchw_scaled: bad item %d", i);
        a.src[i] = reinterpret_cast<const uint16_t*>(it.src);
        a.dst[i] = reinterpret_cast<uint16_t*>(it.dst);
        a.n[i] = it.n; a.c[i] = it.c; a.hw[i] = it.hw; a.ld[i] = it.ld_src;
        tiles += (long long)it.n * ((it.c + 31) / 32) * ((it.hw + 31) / 32);
        if (tiles > 0x7fffffff) return fail(SFB_ERR_INVALID, "nhwc_to_nchw_scaled: too many tiles");
        a.tile_end[i] = (int)tiles;
    }
    cudaError_t err = launch_pdl(nhwc_to_nchw_scaled_kernel, dim3((unsigned)tiles), dim3(256), 0,
                                 static_cast<cudaStream_t>(stream), a);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "nhwc_to_nchw_scaled: %s", cudaGetErrorString(err));
    return check_launch("sfb_nhwc_to_nchw_scaled");
}
