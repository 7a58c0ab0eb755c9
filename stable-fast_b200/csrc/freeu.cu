// FreeU (Si et al., "FreeU: Free Lunch in Diffusion U-Net"; diffusers' apply_freeu) on one up-block resnet's NHWC
// concat buffer [hidden | skip]: the first c_hidden / 2 hidden channels times b, and the skip slice through
// diffusers' fourier_filter(threshold=1, scale=s), in place, in one launch (sfb_freeu).
//
// fourier_filter scales the 2x2 box around the centre of the fftshift-ed spectrum, i.e. exactly the frequencies
// P x Q with P = {0, H-1} ({0} when H = 1) and Q = {0, W-1} ({0} when W = 1).  Per (image, channel), with
// th = 2 pi h / H and ph = 2 pi w / W:
//     y = x + (s - 1) / (H W) * [S + Re(A e^-i th) + Re(B e^-i ph) + Re(D e^-i (th + ph))]
//     S = sum x,  A = sum x e^i th,  B = sum x e^i ph,  D = sum x e^i (th + ph)
// (A and D drop out when H = 1, B and D when W = 1): seven real sums per channel, no FFT.
#include "common.cuh"
#include "host.h"

namespace sfb {

constexpr int FREEU_THREADS = 256;
constexpr int FREEU_VEC = 8;                                // channels per thread: one 16-byte load
constexpr int FREEU_LANES = 2;                              // threads per pixel: 16 channels per filter CTA
constexpr int FREEU_CB = FREEU_VEC * FREEU_LANES;
constexpr int FREEU_PIX = FREEU_THREADS / FREEU_LANES;     // pixels per sweep step
constexpr int FREEU_UNROLL = 4;                             // loads in flight per thread
constexpr int FREEU_SUMS = 7;                               // S, Re A, Im A, Re B, Im B, Re D, Im D
constexpr int FREEU_ACC = FREEU_SUMS * FREEU_VEC;

struct Twiddle {
    float ct, st, cp, sp, cd, sd;  // cos / sin of th, ph and th + ph
};

__device__ __forceinline__ Twiddle twiddle(int p, int h, int w) {
    const int hh = p / w, ww = p - hh * w;
    Twiddle t;
    sincospif(static_cast<float>(2 * hh) / static_cast<float>(h), &t.st, &t.ct);
    sincospif(static_cast<float>(2 * ww) / static_cast<float>(w), &t.sp, &t.cp);
    t.cd = t.ct * t.cp - t.st * t.sp;
    t.sd = t.st * t.cp + t.ct * t.sp;
    return t;
}

__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[FREEU_VEC], int bf16) {
    const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float2 q = unpack2(u[e], bf16);
        f[2 * e] = q.x;
        f[2 * e + 1] = q.y;
    }
}

// grid: [filter_ctas = n * ceil(c_skip / 16) | scale CTAs].  A filter CTA owns 16 skip channels of one image and
// sweeps its pixels twice: the seven sums (fp32, reduced in a fixed order, so replays are bit-identical), then
// the update, one rounding per element.  Its slab (h * w * 32 bytes) is read back from L2.  The scale CTAs
// grid-stride over the first c_hidden / 2 channels, 4 per step: y = x * b, one fp32 multiply and one rounding.
template <int BF16>
__global__ void __launch_bounds__(FREEU_THREADS) freeu_kernel(uint16_t* __restrict__ x, const float* __restrict__ bs,
                                                              int h, int w, int c_hidden, int c_skip, int ld,
                                                              int filter_ctas, long long scale_total) {
    pdl_launch_dependents();
    pdl_wait();
    const int hw = h * w;
    if (static_cast<int>(blockIdx.x) >= filter_ctas) {
        const float b = bs[0];
        const int nv = c_hidden / 8;  // 4-channel vectors in c_hidden / 2
        for (long long idx = (long long)(blockIdx.x - filter_ctas) * FREEU_THREADS + threadIdx.x; idx < scale_total;
             idx += (long long)(gridDim.x - filter_ctas) * FREEU_THREADS) {
            uint2* p = reinterpret_cast<uint2*>(x + (size_t)(idx / nv) * ld + (idx % nv) * 4);
            uint2 v = *p;
            const float2 a = unpack2(v.x, BF16), c = unpack2(v.y, BF16);
            v.x = pack2(a.x * b, a.y * b, BF16);
            v.y = pack2(c.x * b, c.y * b, BF16);
            *p = v;
        }
        return;
    }
    __shared__ float red[FREEU_THREADS / 32][FREEU_LANES][FREEU_ACC];
    __shared__ float tot[FREEU_LANES][FREEU_ACC];
    const int cblocks = (c_skip + FREEU_CB - 1) / FREEU_CB;
    const int img = blockIdx.x / cblocks;
    const int lane_v = threadIdx.x % FREEU_LANES, pix0 = threadIdx.x / FREEU_LANES;
    const int ch = (blockIdx.x % cblocks) * FREEU_CB + lane_v * FREEU_VEC;
    const bool active = ch < c_skip;  // c_skip % 16 == 8: the last block's second lane has no channels
    uint16_t* base = x + (size_t)img * hw * ld + c_hidden + ch;

    float acc[FREEU_ACC];
#pragma unroll
    for (int i = 0; i < FREEU_ACC; ++i) acc[i] = 0.f;
    if (active) {
        for (int p0 = pix0; p0 < hw; p0 += FREEU_UNROLL * FREEU_PIX) {
            uint4 v[FREEU_UNROLL];
#pragma unroll
            for (int u = 0; u < FREEU_UNROLL; ++u) {
                const int p = p0 + u * FREEU_PIX;
                v[u] = p < hw ? *reinterpret_cast<const uint4*>(base + (size_t)p * ld) : make_uint4(0, 0, 0, 0);
            }
#pragma unroll
            for (int u = 0; u < FREEU_UNROLL; ++u) {
                const int p = p0 + u * FREEU_PIX;
                if (p >= hw) break;
                const Twiddle t = twiddle(p, h, w);
                float f[FREEU_VEC];
                unpack8(v[u], f, BF16);
#pragma unroll
                for (int e = 0; e < FREEU_VEC; ++e) {
                    float* a = acc + e * FREEU_SUMS;
                    a[0] += f[e];
                    a[1] = fmaf(f[e], t.ct, a[1]);
                    a[2] = fmaf(f[e], t.st, a[2]);
                    a[3] = fmaf(f[e], t.cp, a[3]);
                    a[4] = fmaf(f[e], t.sp, a[4]);
                    a[5] = fmaf(f[e], t.cd, a[5]);
                    a[6] = fmaf(f[e], t.sd, a[6]);
                }
            }
        }
    }
    // lanes of one channel vector are FREEU_LANES apart in the warp
#pragma unroll
    for (int i = 0; i < FREEU_ACC; ++i)
#pragma unroll
        for (int off = FREEU_LANES; off < 32; off *= 2) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], off);
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    if (lane < FREEU_LANES) {
#pragma unroll
        for (int i = 0; i < FREEU_ACC; ++i) red[warp][lane][i] = acc[i];
    }
    __syncthreads();
    if (threadIdx.x < FREEU_LANES * FREEU_ACC) {
        const int l = threadIdx.x / FREEU_ACC, i = threadIdx.x % FREEU_ACC;
        float s = 0.f;
#pragma unroll
        for (int wi = 0; wi < FREEU_THREADS / 32; ++wi) s += red[wi][l][i];
        tot[l][i] = s;
    }
    __syncthreads();
    if (!active) return;
    const float k = (bs[1] - 1.f) / static_cast<float>(hw);
    const float mh = h > 1 ? 1.f : 0.f, mw = w > 1 ? 1.f : 0.f, md = mh * mw;
#pragma unroll
    for (int e = 0; e < FREEU_VEC; ++e) {
        const float* t = tot[lane_v] + e * FREEU_SUMS;
        acc[e * FREEU_SUMS + 0] = t[0];
        acc[e * FREEU_SUMS + 1] = t[1] * mh;
        acc[e * FREEU_SUMS + 2] = t[2] * mh;
        acc[e * FREEU_SUMS + 3] = t[3] * mw;
        acc[e * FREEU_SUMS + 4] = t[4] * mw;
        acc[e * FREEU_SUMS + 5] = t[5] * md;
        acc[e * FREEU_SUMS + 6] = t[6] * md;
    }
    for (int p0 = pix0; p0 < hw; p0 += FREEU_UNROLL * FREEU_PIX) {
        uint4 v[FREEU_UNROLL];
#pragma unroll
        for (int u = 0; u < FREEU_UNROLL; ++u) {
            const int p = p0 + u * FREEU_PIX;
            v[u] = p < hw ? *reinterpret_cast<const uint4*>(base + (size_t)p * ld) : make_uint4(0, 0, 0, 0);
        }
#pragma unroll
        for (int u = 0; u < FREEU_UNROLL; ++u) {
            const int p = p0 + u * FREEU_PIX;
            if (p >= hw) break;
            const Twiddle t = twiddle(p, h, w);
            float f[FREEU_VEC];
            unpack8(v[u], f, BF16);
#pragma unroll
            for (int e = 0; e < FREEU_VEC; ++e) {
                const float* a = acc + e * FREEU_SUMS;
                float low = a[0];
                low = fmaf(a[1], t.ct, low);
                low = fmaf(a[2], t.st, low);
                low = fmaf(a[3], t.cp, low);
                low = fmaf(a[4], t.sp, low);
                low = fmaf(a[5], t.cd, low);
                low = fmaf(a[6], t.sd, low);
                f[e] = fmaf(k, low, f[e]);
            }
            uint4 o;
            o.x = pack2(f[0], f[1], BF16);
            o.y = pack2(f[2], f[3], BF16);
            o.z = pack2(f[4], f[5], BF16);
            o.w = pack2(f[6], f[7], BF16);
            *reinterpret_cast<uint4*>(base + (size_t)p * ld) = o;
        }
    }
}

}  // namespace sfb

using namespace sfb;

extern "C" int sfb_freeu(const sfb_freeu_params* p, sfb_stream_t stream) {
    if (!p || !p->x || !p->bs) return fail(SFB_ERR_INVALID, "freeu: null pointer");
    if (reinterpret_cast<uintptr_t>(p->x) & 15) return fail(SFB_ERR_INVALID, "freeu: x must be 16-byte aligned");
    if (p->n <= 0 || p->h <= 0 || p->w <= 0 || (long long)p->h * p->w > 0x7fffffff)
        return fail(SFB_ERR_INVALID, "freeu: n=%d h=%d w=%d must be positive with h*w < 2^31", p->n, p->h, p->w);
    if (p->c_hidden <= 0 || p->c_skip <= 0 || p->c_hidden % 8 || p->c_skip % 8 || p->ld % 8 ||
        (long long)p->ld < (long long)p->c_hidden + p->c_skip)
        return fail(SFB_ERR_INVALID,
                    "freeu: c_hidden=%d c_skip=%d ld=%d must be positive multiples of 8 with ld >= c_hidden + c_skip",
                    p->c_hidden, p->c_skip, p->ld);
    if (p->dtype != SFB_F16 && p->dtype != SFB_BF16) return fail(SFB_ERR_INVALID, "freeu: dtype %d", p->dtype);
    const long long filter_ctas = (long long)p->n * ((p->c_skip + FREEU_CB - 1) / FREEU_CB);
    const long long scale_total = (long long)p->n * p->h * p->w * (p->c_hidden / 8);
    const long long scale_blocks = (scale_total + FREEU_THREADS - 1) / FREEU_THREADS;
    const long long scale_ctas = scale_blocks < 2 * 132 ? scale_blocks : 2 * 132;
    if (filter_ctas + scale_ctas > 0x7fffffff) return fail(SFB_ERR_INVALID, "freeu: n=%d too large", p->n);
    const dim3 grid(static_cast<unsigned>(filter_ctas + scale_ctas));
    auto* x = reinterpret_cast<uint16_t*>(p->x);
    cudaError_t err = p->dtype == SFB_BF16
        ? launch_pdl(freeu_kernel<1>, grid, dim3(FREEU_THREADS), 0, static_cast<cudaStream_t>(stream), x, p->bs, p->h,
                     p->w, p->c_hidden, p->c_skip, p->ld, (int)filter_ctas, scale_total)
        : launch_pdl(freeu_kernel<0>, grid, dim3(FREEU_THREADS), 0, static_cast<cudaStream_t>(stream), x, p->bs, p->h,
                     p->w, p->c_hidden, p->c_skip, p->ld, (int)filter_ctas, scale_total);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "freeu: %s", cudaGetErrorString(err));
    return check_launch("sfb_freeu");
}
