// T2I-Adapter edges: PixelUnshuffle of the NCHW conditioning image into the NHWC input of the adapter's
// conv_in (sfb_pixel_unshuffle), and the 2x2 average pool in front of a downsampling AdapterBlock
// (sfb_avg_pool2x2).  Every convolution of the adapter runs on the wgmma GEMM / conv.
#include "common.cuh"
#include "host.h"

namespace sfb {

// y[img, oy, ox, ch * r * r + i * r + j] = x[img, ch, oy * r + i, ox * r + j]: one output element per thread
// and step, output order, so the stores are coalesced along the channel and each run of r consecutive
// channels reads r consecutive pixels of one input row.  A pure permutation of 16-bit values.
__global__ void __launch_bounds__(256) pixel_unshuffle_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ y,
                                                              int c, int h, int w, int r, int cout, int ldy,
                                                              long long total) {
    pdl_launch_dependents();
    pdl_wait();
    const int ho = h / r, wo = w / r;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(idx % cout);
        long long p = idx / cout;
        const int ox = (int)(p % wo); p /= wo;
        const int oy = (int)(p % ho);
        const int img = (int)(p / ho);
        const int j = k % r, i = (k / r) % r, ch = k / (r * r);
        const uint16_t v = x[(((size_t)img * c + ch) * h + oy * r + i) * w + ox * r + j];
        y[(((size_t)img * ho + oy) * wo + ox) * ldy + k] = v;
    }
}

// y[img, oy, ox, :] = (x[2oy, 2ox] + x[2oy, 2ox+1] + x[2oy+1, 2ox] + x[2oy+1, 2ox+1]) / 4, NHWC, 8 channels
// (16 bytes) per thread and step, fp32 sum, one rounding.
template <int BF16>
__global__ void __launch_bounds__(256) avg_pool2x2_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ y,
                                                          int h, int w, int nvec, int ldx, int ldy, long long total) {
    pdl_launch_dependents();
    pdl_wait();
    const int ho = h / 2, wo = w / 2;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int vec = (int)(idx % nvec);
        long long p = idx / nvec;
        const int ox = (int)(p % wo); p /= wo;
        const int oy = (int)(p % ho);
        const int img = (int)(p / ho);
        float acc[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = 0.f;
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                const uint4 v = *reinterpret_cast<const uint4*>(
                    x + (((size_t)img * h + 2 * oy + dy) * w + 2 * ox + dx) * ldx + vec * 8);
                const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float2 f = unpack2(u[e], BF16);
                    acc[2 * e] += f.x;
                    acc[2 * e + 1] += f.y;
                }
            }
        uint4 o;
        o.x = pack2(acc[0] * 0.25f, acc[1] * 0.25f, BF16);
        o.y = pack2(acc[2] * 0.25f, acc[3] * 0.25f, BF16);
        o.z = pack2(acc[4] * 0.25f, acc[5] * 0.25f, BF16);
        o.w = pack2(acc[6] * 0.25f, acc[7] * 0.25f, BF16);
        *reinterpret_cast<uint4*>(y + (((size_t)img * ho + oy) * wo + ox) * ldy + vec * 8) = o;
    }
}

}  // namespace sfb

using namespace sfb;

static int grid_stride_blocks(long long total) {
    const long long blocks = (total + 255) / 256;
    return (int)(blocks < 132 * 16 ? blocks : 132 * 16);
}

extern "C" int sfb_pixel_unshuffle(const void* x, void* y, int32_t n, int32_t c, int32_t h, int32_t w, int32_t r,
                                   int32_t ldy, sfb_stream_t stream) {
    if (!x || !y) return fail(SFB_ERR_INVALID, "pixel_unshuffle: null pointer");
    if (n <= 0 || c <= 0 || h <= 0 || w <= 0) return fail(SFB_ERR_INVALID, "pixel_unshuffle: empty tensor n=%d c=%d h=%d w=%d", n, c, h, w);
    if (r <= 0 || h % r || w % r)
        return fail(SFB_ERR_INVALID, "pixel_unshuffle: factor r=%d must be positive and divide h=%d and w=%d", r, h, w);
    const long long cout = (long long)c * r * r;
    if (cout > 0x7fffffff || ldy < cout)
        return fail(SFB_ERR_INVALID, "pixel_unshuffle: ldy=%d must be at least c*r*r=%lld", ldy, cout);
    const long long total = (long long)n * (h / r) * (w / r) * cout;
    cudaError_t err = launch_pdl(pixel_unshuffle_kernel, dim3(grid_stride_blocks(total)), dim3(256), 0,
                                 static_cast<cudaStream_t>(stream), reinterpret_cast<const uint16_t*>(x),
                                 reinterpret_cast<uint16_t*>(y), c, h, w, r, (int)cout, ldy, total);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "pixel_unshuffle: %s", cudaGetErrorString(err));
    return check_launch("sfb_pixel_unshuffle");
}

extern "C" int sfb_avg_pool2x2(const void* x, void* y, int32_t n, int32_t h, int32_t w, int32_t c, int32_t ldx,
                               int32_t ldy, int32_t dtype, sfb_stream_t stream) {
    if (!x || !y) return fail(SFB_ERR_INVALID, "avg_pool2x2: null pointer");
    if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15)
        return fail(SFB_ERR_INVALID, "avg_pool2x2: x and y must be 16-byte aligned");
    if (n <= 0 || h <= 0 || w <= 0 || h % 2 || w % 2)
        return fail(SFB_ERR_INVALID, "avg_pool2x2: n=%d, h=%d and w=%d must be positive, h and w even", n, h, w);
    if (c <= 0 || c % 8 || ldx % 8 || ldy % 8 || ldx < c || ldy < c)
        return fail(SFB_ERR_INVALID, "avg_pool2x2: c=%d ldx=%d ldy=%d must be multiples of 8 with ldx, ldy >= c",
                    c, ldx, ldy);
    if (dtype != SFB_F16 && dtype != SFB_BF16) return fail(SFB_ERR_INVALID, "avg_pool2x2: dtype %d", dtype);
    const long long total = (long long)n * (h / 2) * (w / 2) * (c / 8);
    const dim3 grid(grid_stride_blocks(total));
    const auto* xs = reinterpret_cast<const uint16_t*>(x);
    auto* ys = reinterpret_cast<uint16_t*>(y);
    cudaError_t err = dtype == SFB_BF16
        ? launch_pdl(avg_pool2x2_kernel<1>, grid, dim3(256), 0, static_cast<cudaStream_t>(stream), xs, ys, h, w, c / 8,
                     ldx, ldy, total)
        : launch_pdl(avg_pool2x2_kernel<0>, grid, dim3(256), 0, static_cast<cudaStream_t>(stream), xs, ys, h, w, c / 8,
                     ldx, ldy, total);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "avg_pool2x2: %s", cudaGetErrorString(err));
    return check_launch("sfb_avg_pool2x2");
}
