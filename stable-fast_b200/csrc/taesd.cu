// AutoencoderTiny (TAESD / TAESDXL): every layer between the tiny VAE's two edge convolutions is a 3x3
// convolution with 64 input and 64 output channels (sfb_conv3x3_c64).  The wgmma GEMM's 128 x 160 tile
// would spend 60 % of its tensor-core work on padding at N = 64, so this kernel has an N of exactly 64.
#include "common.cuh"
#include "host.h"

namespace sfb {
namespace {

// ---------------------------------------------------------------------------------------
// Implicit GEMM on mma.sync m16n8k16: M = output pixels, N = 64 output channels, K = 9 taps x 64
// input channels.  A persistent CTA of 4 warps keeps the whole [64, 576] weight in shared memory
// (loaded once) and walks 8 x 16-pixel output tiles.  Per tile it stages the SOURCE pixels the tile
// reads (its halo, zero outside the image) with cp.async; all nine taps are shifted views of that
// halo, addressed row by row through ldmatrix, which is what lets one kernel serve three input
// modes:
//   mode 0: stride 1, pad 1                 halo (8 + 2) x (16 + 2)
//   mode 1: stride 2, pad 1 on every side   halo (2 * 8 + 1) x (2 * 16 + 1), columns stored even
//                                           ones first, so a stride-2 ldmatrix row walk stays
//                                           bank-conflict free
//   mode 2: nearest-2x upsample, then stride 1, pad 1, read from the low-resolution image: output
//           row r, tap ty reads upsampled row r + ty - 1, i.e. source row (r + ty - 1) >> 1
//           (-1 >> 1 = -1: the upsampled image's padding row is the source's zero row); halo
//           (8 / 2 + 2) x (16 / 2 + 2).
// Warp w owns output rows 4 (w & 1) .. + 3 (four m16 tiles = 16 consecutive pixels of a row each) and
// channels 32 (w >> 1) .. + 31 (four n8 tiles).  Epilogue: the fp32 accumulators go through shared
// memory (aliasing the halo) so that each thread finishes 8 consecutive channels of a pixel --
// bias, residual, ReLU -- with one 16-byte residual load and one 16-byte store.
// ---------------------------------------------------------------------------------------
constexpr int kC = 64;
constexpr int kK = 9 * kC;
constexpr int kWPitch = kK + 8;    // halves per weight row in smem (1168 B: ldmatrix rows hit distinct banks)
constexpr int kPixPitch = kC + 8;  // halves per staged source pixel (144 B)
constexpr int kTH = 8, kTW = 16;   // output tile
constexpr int kOutPitch = kC + 8;  // floats per staged output pixel
constexpr int kThreads = 128;
constexpr int kWBytes = kC * kWPitch * 2;
constexpr int kOutBytes = kTH * kTW * kOutPitch * 4;

template <int MODE>
struct Halo {
    static constexpr int H = MODE == 0 ? kTH + 2 : (MODE == 1 ? 2 * kTH + 1 : kTH / 2 + 2);
    static constexpr int W = MODE == 0 ? kTW + 2 : (MODE == 1 ? 2 * kTW + 1 : kTW / 2 + 2);
    static constexpr int bytes = H * W * kPixPitch * 2;
    static constexpr int region = bytes > kOutBytes ? bytes : kOutBytes;  // halo, then the output stage
    static constexpr int smem = kWBytes + region;
};

struct C64Args {
    const uint16_t* x;
    const uint16_t* w;
    const float* bias;
    const uint16_t* res;
    uint16_t* y;
    int h, wd, ho, wo, ldx, ldy, ldr, relu;
    int tiles_w, tiles_per_img, tiles;
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0)
                 : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
    asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
}

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(addr));
}

template <int BF16>
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
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

// halo row of output row r (0..kTH-1) and tap row ty
template <int MODE>
__device__ __forceinline__ int halo_row(int r, int ty) {
    return MODE == 0 ? r + ty : (MODE == 1 ? 2 * r + ty : (r + ty + 1) >> 1);
}
// stored halo column of output column c (0..kTW-1) and tap column tx
template <int MODE>
__device__ __forceinline__ int halo_col(int c, int tx) {
    if (MODE == 0) return c + tx;
    if (MODE == 2) return (c + tx + 1) >> 1;
    return tx == 1 ? kTW + 1 + c : c + (tx >> 1);  // even local columns 0..32 first, then the odd ones
}

template <int MODE, int BF16>
__global__ void __launch_bounds__(kThreads) conv3x3_c64_kernel(const C64Args a) {
    using HG = Halo<MODE>;
    extern __shared__ __align__(16) uint8_t smem[];
    uint16_t* wsm = reinterpret_cast<uint16_t*>(smem);
    uint16_t* halo = reinterpret_cast<uint16_t*>(smem + kWBytes);
    float* stage = reinterpret_cast<float*>(smem + kWBytes);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    pdl_launch_dependents();
    pdl_wait();
    // the weight: [64][576] global -> [64][kWPitch] smem, once per CTA (completes with the first halo)
    for (int i = tid; i < kC * (kK / 8); i += kThreads) {
        const int n = i / (kK / 8), v = i - n * (kK / 8);
        cp_async16(smem_u32(wsm + n * kWPitch + v * 8), a.w + (size_t)n * kK + v * 8, true);
    }
    const int wm = warp & 1, wn = warp >> 1;
    const int g = lane >> 2, q = lane & 3;
    const int lpix = lane & 15, lk = (lane >> 4) * 8;            // A: ldmatrix row = pixel, 8-channel half
    const int bn = ((lane >> 4) << 3) + (lane & 7), bk = ((lane >> 3) & 1) * 8;  // B: row = out channel
    const uint32_t w_lane = smem_u32(wsm + (wn * 32 + bn) * kWPitch + bk);
    const uint32_t halo_base = smem_u32(halo);

    for (int tile = blockIdx.x; tile < a.tiles; tile += gridDim.x) {
        const int img = tile / a.tiles_per_img, t = tile - img * a.tiles_per_img;
        const int oy0 = (t / a.tiles_w) * kTH, ox0 = (t % a.tiles_w) * kTW;
        const int sy0 = MODE == 0 ? oy0 - 1 : (MODE == 1 ? 2 * oy0 - 1 : (oy0 >> 1) - 1);
        const int sx0 = MODE == 0 ? ox0 - 1 : (MODE == 1 ? 2 * ox0 - 1 : (ox0 >> 1) - 1);
        const uint16_t* ximg = a.x + (size_t)img * a.h * a.wd * a.ldx;
        for (int i = tid; i < HG::H * HG::W * 8; i += kThreads) {
            const int v = i & 7, px = i >> 3;
            const int ly = px / HG::W, lx = px - ly * HG::W;
            const int sy = sy0 + ly, sx = sx0 + lx;
            const bool in = sy >= 0 && sy < a.h && sx >= 0 && sx < a.wd;
            const int sc = MODE == 1 ? ((lx & 1) ? kTW + 1 + (lx >> 1) : (lx >> 1)) : lx;
            cp_async16(smem_u32(halo + (ly * HG::W + sc) * kPixPitch + v * 8),
                       in ? ximg + ((size_t)sy * a.wd + sx) * a.ldx + v * 8 : a.x, in);
        }
        cp_async_wait_all();
        __syncthreads();

        float acc[4][4][4];
#pragma unroll
        for (int mt = 0; mt < 4; ++mt)
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.f;
#pragma unroll 1
        for (int tap = 0; tap < 9; ++tap) {
            const int ty = tap / 3, tx = tap - ty * 3;
            const int col = halo_col<MODE>(lpix, tx);
            uint32_t a_addr[4];
#pragma unroll
            for (int mt = 0; mt < 4; ++mt)
                a_addr[mt] = halo_base + ((halo_row<MODE>(wm * 4 + mt, ty) * HG::W + col) * kPixPitch + lk) * 2;
            const uint32_t w_tap = w_lane + tap * kC * 2;
#pragma unroll
            for (int kc = 0; kc < 4; ++kc) {
                uint32_t b[2][4];
                ldsm_x4(w_tap + kc * 32, b[0]);
                ldsm_x4(w_tap + 16 * kWPitch * 2 + kc * 32, b[1]);
#pragma unroll
                for (int mt = 0; mt < 4; ++mt) {
                    uint32_t af[4];
                    ldsm_x4(a_addr[mt] + kc * 32, af);
#pragma unroll
                    for (int nt = 0; nt < 4; ++nt)
                        mma16816<BF16>(acc[mt][nt], af, b[nt >> 1][(nt & 1) * 2], b[nt >> 1][(nt & 1) * 2 + 1]);
                }
            }
        }
        __syncthreads();  // every warp is done with the halo: the output stage aliases it
#pragma unroll
        for (int mt = 0; mt < 4; ++mt)
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                for (int hf = 0; hf < 2; ++hf) {
                    const int p = (wm * 4 + mt) * kTW + g + 8 * hf;
                    *reinterpret_cast<float2*>(&stage[p * kOutPitch + wn * 32 + nt * 8 + 2 * q]) =
                        make_float2(acc[mt][nt][2 * hf], acc[mt][nt][2 * hf + 1]);
                }
        __syncthreads();
#pragma unroll
        for (int it = 0; it < kTH * kTW * 8 / kThreads; ++it) {
            const int item = it * kThreads + tid;
            const int p = item >> 3, v = item & 7;
            const int oy = oy0 + p / kTW, ox = ox0 + p % kTW;
            if (oy >= a.ho || ox >= a.wo) continue;
            const float4 s0 = *reinterpret_cast<const float4*>(&stage[p * kOutPitch + v * 8]);
            const float4 s1 = *reinterpret_cast<const float4*>(&stage[p * kOutPitch + v * 8 + 4]);
            float o[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
            if (a.bias) {
                const float4 b0 = __ldg(reinterpret_cast<const float4*>(a.bias + v * 8));
                const float4 b1 = __ldg(reinterpret_cast<const float4*>(a.bias + v * 8 + 4));
                o[0] += b0.x; o[1] += b0.y; o[2] += b0.z; o[3] += b0.w;
                o[4] += b1.x; o[5] += b1.y; o[6] += b1.z; o[7] += b1.w;
            }
            const size_t pix = ((size_t)img * a.ho + oy) * a.wo + ox;
            if (a.res) {
                // (may alias y: this thread reads these 8 channels before it writes them)
                const uint4 r = *reinterpret_cast<const uint4*>(a.res + pix * a.ldr + v * 8);
                const uint32_t rw[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 f = unpack2(rw[j], BF16);
                    o[2 * j] += f.x;
                    o[2 * j + 1] += f.y;
                }
            }
            if (a.relu) {
#pragma unroll
                for (int j = 0; j < 8; ++j) o[j] = fmaxf(o[j], 0.f);
            }
            *reinterpret_cast<uint4*>(a.y + pix * a.ldy + v * 8) =
                make_uint4(pack2(o[0], o[1], BF16), pack2(o[2], o[3], BF16), pack2(o[4], o[5], BF16),
                           pack2(o[6], o[7], BF16));
        }
        __syncthreads();  // the next tile's halo overwrites the output stage
    }
}

template <int MODE>
int launch_c64(const C64Args& a, int bf16, cudaStream_t stream) {
    constexpr int smem = Halo<MODE>::smem;
    static PerDeviceOnce attr_once;
    bool& attr_set = attr_once.flag();
    if (!attr_set) {
        for (cudaError_t err : {cudaFuncSetAttribute(conv3x3_c64_kernel<MODE, 0>,
                                                     cudaFuncAttributeMaxDynamicSharedMemorySize, smem),
                                cudaFuncSetAttribute(conv3x3_c64_kernel<MODE, 1>,
                                                     cudaFuncAttributeMaxDynamicSharedMemorySize, smem)})
            if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "conv3x3_c64: smem attribute: %s", cudaGetErrorString(err));
        attr_set = true;
    }
    // persistent: as many CTAs as fit on the device at once (two per SM when the smem allows), at most one per tile
    const int per_sm = 2 * (smem + 1024) <= 228 * 1024 ? 2 : 1;
    const int grid = a.tiles < per_sm * sm_count() ? a.tiles : per_sm * sm_count();
    const cudaError_t err = bf16 ? launch_pdl(conv3x3_c64_kernel<MODE, 1>, dim3(grid), dim3(kThreads), smem, stream, a)
                                 : launch_pdl(conv3x3_c64_kernel<MODE, 0>, dim3(grid), dim3(kThreads), smem, stream, a);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "conv3x3_c64: %s", cudaGetErrorString(err));
    return check_launch("sfb_conv3x3_c64");
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace
}  // namespace sfb

using namespace sfb;

extern "C" int sfb_conv3x3_c64(const sfb_conv_c64_params* p, sfb_stream_t stream) {
    if (!p || !p->x || !p->weight || !p->y) return fail(SFB_ERR_INVALID, "conv3x3_c64: null pointer");
    if (p->n <= 0 || p->h <= 0 || p->w <= 0) return fail(SFB_ERR_INVALID, "conv3x3_c64: empty image");
    if (p->mode < SFB_C64_SAME || p->mode > SFB_C64_UP2X) return fail(SFB_ERR_INVALID, "conv3x3_c64: mode %d", p->mode);
    if (p->dtype != SFB_F16 && p->dtype != SFB_BF16) return fail(SFB_ERR_INVALID, "conv3x3_c64: dtype %d", p->dtype);
    if (p->ldx < kC || p->ldy < kC || p->ldx % 8 || p->ldy % 8 || (p->residual && (p->ldr < kC || p->ldr % 8)))
        return fail(SFB_ERR_INVALID, "conv3x3_c64: channel pitches ldx=%d ldy=%d ldr=%d must be multiples of 8, >= 64",
                    p->ldx, p->ldy, p->ldr);
    if (!aligned16(p->x) || !aligned16(p->weight) || !aligned16(p->y) || (p->bias && !aligned16(p->bias)) ||
        (p->residual && !aligned16(p->residual)))
        return fail(SFB_ERR_INVALID, "conv3x3_c64: x, weight, bias, residual and y must be 16-byte aligned");
    C64Args a{};
    a.x = reinterpret_cast<const uint16_t*>(p->x);
    a.w = reinterpret_cast<const uint16_t*>(p->weight);
    a.bias = p->bias;
    a.res = reinterpret_cast<const uint16_t*>(p->residual);
    a.y = reinterpret_cast<uint16_t*>(p->y);
    a.h = p->h; a.wd = p->w; a.ldx = p->ldx; a.ldy = p->ldy; a.ldr = p->ldr; a.relu = p->relu ? 1 : 0;
    if (p->mode == SFB_C64_STRIDE2) {
        a.ho = (p->h + 1) / 2; a.wo = (p->w + 1) / 2;
    } else if (p->mode == SFB_C64_UP2X) {
        a.ho = 2 * p->h; a.wo = 2 * p->w;
    } else {
        a.ho = p->h; a.wo = p->w;
    }
    if ((long long)a.ho * a.wo > INT32_MAX) return fail(SFB_ERR_INVALID, "conv3x3_c64: image too large");
    a.tiles_w = (a.wo + kTW - 1) / kTW;
    const long long per_img = (long long)a.tiles_w * ((a.ho + kTH - 1) / kTH);
    if (per_img * p->n > INT32_MAX) return fail(SFB_ERR_INVALID, "conv3x3_c64: more than 2^31 output tiles");
    a.tiles_per_img = (int)per_img;
    a.tiles = (int)(per_img * p->n);
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int bf16 = p->dtype == SFB_BF16;
    if (p->mode == SFB_C64_STRIDE2) return launch_c64<1>(a, bf16, s);
    if (p->mode == SFB_C64_UP2X) return launch_c64<2>(a, bf16, s);
    return launch_c64<0>(a, bf16, s);
}
