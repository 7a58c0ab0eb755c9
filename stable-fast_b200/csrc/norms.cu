// GroupNorm (+SiLU) and LayerNorm for NHWC / token-major 16-bit activations (HBM-bound kernels).
//
// GroupNorm is two passes, like the reference's NHWC path (/root/reference/src/sfast/triton/ops/
// group_norm.py:126-165 stats, :272-320 apply) but with the statistics kept in fp32 end to end
// (the reference round-trips mean/rstd through the input dtype, group_norm.py:405-416) and with
// the stats grid sized to fill the SMs instead of groups*batch CTAs.
//
// Variance: the reference merges Welford partials (triton/ops/utils.py:5-15).  Here every
// (image, group) accumulates the SHIFTED moments  S1 = sum(x - K), S2 = sum((x - K)^2)  with
// K = the group's first stored value x[img, pixel 0, first channel of the group] (identical for
// every CTA of the image), and  mean = K + S1/n,  var = S2/n - (S1/n)^2.  With K inside the data
// range the subtraction no longer cancels the leading digits when |mean| >> sigma (outlier
// channels of real checkpoints), which the raw sum-of-squares form E[x^2] - mean^2 does.
// LayerNorm is one warp per row, row held in registers, two-pass mean/variance in fp32
// (reference: triton/ops/layer_norm.py:51-133).
#include "common.cuh"
#include "host.h"

#include <stdlib.h>

namespace sfb {

constexpr int kGnThreads = 512;

struct GnArgs {
    const uint16_t* x;
    uint16_t* y;
    const float* gamma;
    const float* beta;
    float* stats;
    int n, hw, c, ldx, ldy, groups, cpg, nvec, rows_per_block;
    float eps;
    int silu, dtype;
    // deferred split-K finish of the GEMM producing channels [0, part_c) (fused kernel only)
    const float* part_ws;
    int part_splits, part_c, part_ld;
    const float* part_bias;
    const float* part_rowbias;
    int part_ld_rowbias;
    const uint16_t* part_residual;
    int part_ldr;
};

// Finished 16-bit values of channels [tx*8, tx*8+8) of pixel `row` of image `img` from the
// producer GEMM's fp32 split-K partials: sum + bias + per-image row bias + residual (the STORE
// epilogue of gemm_tc.cu's reduction kernel), also written to x.
__device__ __forceinline__ uint4 gn_finish_partials(const GnArgs& a, int img, int row, int tx) {
    const int m = img * a.hw + row;
    const int col = tx * 8;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    constexpr int kU = 6;  // partial loads in flight per batch
    const size_t stride = (size_t)a.n * a.hw * a.part_ld;
    const float* p0 = a.part_ws + (size_t)m * a.part_ld + col;
    for (int s0 = 0; s0 < a.part_splits; s0 += kU) {
        float4 lo[kU], hi[kU];
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            if (s0 + u < a.part_splits) {
                const float* p = p0 + (size_t)(s0 + u) * stride;
                lo[u] = __ldcg(reinterpret_cast<const float4*>(p));
                hi[u] = __ldcg(reinterpret_cast<const float4*>(p + 4));
            }
        }
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            if (s0 + u < a.part_splits) {
                acc[0] += lo[u].x; acc[1] += lo[u].y; acc[2] += lo[u].z; acc[3] += lo[u].w;
                acc[4] += hi[u].x; acc[5] += hi[u].y; acc[6] += hi[u].z; acc[7] += hi[u].w;
            }
        }
    }
    auto add8 = [&](const float* b) {
        const float4 b0 = *reinterpret_cast<const float4*>(b);
        const float4 b1 = *reinterpret_cast<const float4*>(b + 4);
        acc[0] += b0.x; acc[1] += b0.y; acc[2] += b0.z; acc[3] += b0.w;
        acc[4] += b1.x; acc[5] += b1.y; acc[6] += b1.z; acc[7] += b1.w;
    };
    if (a.part_bias) add8(a.part_bias + col);
    if (a.part_rowbias) add8(a.part_rowbias + (size_t)img * a.part_ld_rowbias + col);
    if (a.part_residual) {
        const uint4 r = *reinterpret_cast<const uint4*>(a.part_residual + (size_t)m * a.part_ldr + col);
        const uint32_t w[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 f = unpack2(w[i], a.dtype);
            acc[2 * i] += f.x; acc[2 * i + 1] += f.y;
        }
    }
    uint4 v;
    v.x = pack2(acc[0], acc[1], a.dtype); v.y = pack2(acc[2], acc[3], a.dtype);
    v.z = pack2(acc[4], acc[5], a.dtype); v.w = pack2(acc[6], acc[7], a.dtype);
    *reinterpret_cast<uint4*>(const_cast<uint16_t*>(a.x) + (size_t)m * a.ldx + col) = v;
    return v;
}

// One finished 16-bit value (as float) of channel `ch` of pixel `row`: the same arithmetic, in the
// same order, as gn_finish_partials -- so every CTA derives the identical shift K from it.
__device__ __forceinline__ float gn_finish_partial1(const GnArgs& a, int img, int row, int ch) {
    const int m = img * a.hw + row;
    const size_t stride = (size_t)a.n * a.hw * a.part_ld;
    const float* p0 = a.part_ws + (size_t)m * a.part_ld + ch;
    float acc = 0.f;
    constexpr int kU = 6;
    for (int s0 = 0; s0 < a.part_splits; s0 += kU) {
        float v[kU];
#pragma unroll
        for (int u = 0; u < kU; ++u)
            if (s0 + u < a.part_splits) v[u] = __ldcg(p0 + (size_t)(s0 + u) * stride);
#pragma unroll
        for (int u = 0; u < kU; ++u)
            if (s0 + u < a.part_splits) acc += v[u];
    }
    if (a.part_bias) acc += a.part_bias[ch];
    if (a.part_rowbias) acc += a.part_rowbias[(size_t)img * a.part_ld_rowbias + ch];
    if (a.part_residual) acc += load1(a.part_residual, (size_t)m * a.part_ldr + ch, a.dtype);
    const uint32_t r = pack2(acc, 0.f, a.dtype);
    return unpack2(r, a.dtype).x;
}

// Shift K of every group of image `img` into shared memory: the first stored value of the group
// (pixel 0, first channel).  kPart: channels below part_c do not exist in x yet.
template <bool kPart>
__device__ __forceinline__ void gn_load_shifts(const GnArgs& a, int img, float* sK) {
    for (int g = threadIdx.x; g < a.groups; g += blockDim.x) {
        const int ch = g * a.cpg;
        float k;
        if (kPart && ch < a.part_c) k = gn_finish_partial1(a, img, 0, ch);
        else k = load1(a.x, (size_t)img * a.hw * a.ldx + ch, a.dtype);
        sK[g] = k;
    }
}

// (S1, S2) of the 8 channels of `v` about their groups' shifts
struct GnAcc8 {
    float s[8], ss[8];
    __device__ __forceinline__ void zero() {
#pragma unroll
        for (int i = 0; i < 8; ++i) s[i] = ss[i] = 0.f;
    }
    __device__ __forceinline__ void add(const uint4& v, const float (&k)[8], int dtype) {
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 f = unpack2(w[i], dtype);
            const float d0 = f.x - k[2 * i], d1 = f.y - k[2 * i + 1];
            s[2 * i] += d0; ss[2 * i] += d0 * d0;
            s[2 * i + 1] += d1; ss[2 * i + 1] += d1 * d1;
        }
    }
};

// Compile-time dtype form of GnAcc8::add for the streaming statistics kernel, which is INSTRUCTION-bound
// with the generic one (ncu: 85 warp instructions per 16-byte load, 41 % issue utilisation at 2 TB/s -- a
// uniform dtype branch per row, FMUL + FADD where an FFMA does, a 64-bit multiply per address).  fp16: the
// shift subtraction rides on the half -> float conversion (HADD2.F32 takes two half operands; K is a
// stored 16-bit value, so x - K is exact in fp32 either way).
template <int BF16>
__device__ __forceinline__ void gn_add8_t(GnAcc8& st, const uint4& v, const uint32_t (&kp)[4], const float (&k)[8]) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float d0, d1;
        if (BF16) {
            const float2 f = unpack2(w[i], 1);
            d0 = f.x - k[2 * i];
            d1 = f.y - k[2 * i + 1];
        } else {
            const __half2 x = *reinterpret_cast<const __half2*>(&w[i]);
            const __half2 kk = *reinterpret_cast<const __half2*>(&kp[i]);
            d0 = __half2float(__low2half(x)) - __half2float(__low2half(kk));
            d1 = __half2float(__high2half(x)) - __half2float(__high2half(kk));
        }
        st.s[2 * i] += d0;
        st.ss[2 * i] = fmaf(d0, d0, st.ss[2 * i]);
        st.s[2 * i + 1] += d1;
        st.ss[2 * i + 1] = fmaf(d1, d1, st.ss[2 * i + 1]);
    }
}

// ---- deterministic reductions (no floating-point atomics anywhere: replays are bit-identical) --------
// kGnThreads x 16 floats of scratch: per-thread moments, then per-channel totals, then slot partials
constexpr int kGnRedFloats = kGnThreads * 16;

// CTA level: the (S1, S2) of thread (tx, ty)'s 8 channels -> acc[2 * groups] in shared memory, every
// addition in a fixed order: (1) row slots ty = 0, 1, ... per channel, (2) channels in order per group.
// All threads of the CTA call it (it synchronises); `active` = the thread holds data.
__device__ __forceinline__ void gn_block_reduce(const GnAcc8& st, bool active, int tx, int ty, int by,
                                                const GnArgs& a, float* red, float* acc) {
    float4* red4 = reinterpret_cast<float4*>(red);
    if (active && ty > 0) {
        const int t = ty * a.nvec + tx;
        red4[0 * kGnThreads + t] = make_float4(st.s[0], st.s[1], st.s[2], st.s[3]);
        red4[1 * kGnThreads + t] = make_float4(st.s[4], st.s[5], st.s[6], st.s[7]);
        red4[2 * kGnThreads + t] = make_float4(st.ss[0], st.ss[1], st.ss[2], st.ss[3]);
        red4[3 * kGnThreads + t] = make_float4(st.ss[4], st.ss[5], st.ss[6], st.ss[7]);
    }
    __syncthreads();
    float s[8], ss[8];
    const bool owner = active && ty == 0;
    if (owner) {
#pragma unroll
        for (int i = 0; i < 8; ++i) { s[i] = st.s[i]; ss[i] = st.ss[i]; }
        for (int r = 1; r < by; ++r) {
            const int t = r * a.nvec + tx;
            const float4 a0 = red4[0 * kGnThreads + t], a1 = red4[1 * kGnThreads + t];
            const float4 b0 = red4[2 * kGnThreads + t], b1 = red4[3 * kGnThreads + t];
            s[0] += a0.x; s[1] += a0.y; s[2] += a0.z; s[3] += a0.w;
            s[4] += a1.x; s[5] += a1.y; s[6] += a1.z; s[7] += a1.w;
            ss[0] += b0.x; ss[1] += b0.y; ss[2] += b0.z; ss[3] += b0.w;
            ss[4] += b1.x; ss[5] += b1.y; ss[6] += b1.z; ss[7] += b1.w;
        }
    }
    __syncthreads();  // the per-thread partials are consumed: the scratch becomes [2][c] channel totals
    if (owner) {
        float4* ch = reinterpret_cast<float4*>(red + tx * 8);
        ch[0] = make_float4(s[0], s[1], s[2], s[3]);
        ch[1] = make_float4(s[4], s[5], s[6], s[7]);
        float4* ch2 = reinterpret_cast<float4*>(red + a.c + tx * 8);
        ch2[0] = make_float4(ss[0], ss[1], ss[2], ss[3]);
        ch2[1] = make_float4(ss[4], ss[5], ss[6], ss[7]);
    }
    __syncthreads();
    if ((int)threadIdx.x < a.groups) {
        const int c0 = threadIdx.x * a.cpg;
        float g1 = 0.f, g2 = 0.f;
        for (int c = c0; c < c0 + a.cpg; ++c) { g1 += red[c]; g2 += red[a.c + c]; }
        acc[2 * threadIdx.x] = g1;
        acc[2 * threadIdx.x + 1] = g2;
    }
    __syncthreads();
}

// this CTA's group moments -> its own slot of the statistics workspace [n][blocks_per_img][2 * groups]
__device__ __forceinline__ void gn_store_slot(const GnArgs& a, int img, const float* acc) {
    float* slot = a.stats + ((size_t)img * gridDim.x + blockIdx.x) * 2 * a.groups;
    for (int i = threadIdx.x; i < 2 * a.groups; i += kGnThreads) slot[i] = acc[i];
}

// grid level: the slots of image `img` summed in a fixed order (identical in every CTA and every replay):
// kGnThreads / (2 * groups) interleaved chains over the slots, then the chains in order.  -> acc (shared)
__device__ __forceinline__ void gn_sum_slots(const GnArgs& a, int img, float* red, float* acc) {
    const int pairs = 2 * a.groups;
    const int chains = kGnThreads / pairs;  // >= 4 (groups <= 64)
    const int pair = threadIdx.x % pairs, q = threadIdx.x / pairs;
    const int bpi = gridDim.x;
    if (q < chains) {
        const float* base = a.stats + (size_t)img * bpi * pairs + pair;
        float part = 0.f;
        constexpr int kU = 8;
        for (int b0 = q; b0 < bpi; b0 += chains * kU) {
            float v[kU];
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                const int b = b0 + u * chains;
                if (b < bpi) v[u] = __ldcg(base + (size_t)b * pairs);
            }
#pragma unroll
            for (int u = 0; u < kU; ++u)
                if (b0 + u * chains < bpi) part += v[u];
        }
        red[q * pairs + pair] = part;
    }
    __syncthreads();
    if ((int)threadIdx.x < pairs) {
        float t = 0.f;
        for (int c = 0; c < chains; ++c) t += red[c * pairs + threadIdx.x];
        acc[threadIdx.x] = t;
    }
    __syncthreads();
}

// per-channel scale / shift from the finished shifted moments
__device__ __forceinline__ void gn_scale_shift(const GnArgs& a, const float* acc, const float* sK, float inv_cnt,
                                               int ch, float gamma, float beta, float& sc, float& sh) {
    const int g = ch / a.cpg;
    const float s1 = acc[2 * g] * inv_cnt;
    const float s2 = acc[2 * g + 1] * inv_cnt;
    const float mean = sK[g] + s1;
    const float var = fmaxf(s2 - s1 * s1, 0.f);
    sc = rsqrtf(var + a.eps) * gamma;
    sh = beta - mean * sc;
}

// grid (blocks_per_img, n).  Thread (tx = vector column, ty = row slot) keeps per-channel
// partial sums for its 8 channels over rows ty, ty+BY, ...; one shared-memory atomic per
// (thread, group run) at the end, then one global atomic per (block, group, moment).
template <int BF16>
__global__ void __launch_bounds__(kGnThreads) gn_stats_kernel(const GnArgs a) {
    __shared__ float acc[2 * 64];
    __shared__ float sK[64];
    __shared__ __align__(16) float red[kGnRedFloats];
    pdl_launch_dependents();
    pdl_wait();
    const int img = blockIdx.y;
    const int by = kGnThreads / a.nvec;
    const int tx = threadIdx.x % a.nvec;
    const int ty = threadIdx.x / a.nvec;
    GnAcc8 st;
    st.zero();
    if (ty < by) {
        // every thread fetches the shifts of its own 8 channels itself (one 2-byte load per group run, of a
        // line the whole group shares): in flight together with the first batch of rows instead of a
        // load -> barrier -> load chain
        float k[8];
        {
            int g_prev = -1;
            float kv = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int g = (tx * 8 + i) / a.cpg;
                if (g != g_prev) {
                    kv = load1(a.x, (size_t)img * a.hw * a.ldx + g * a.cpg, a.dtype);
                    g_prev = g;
                    if (ty == 0 && g * a.cpg >= tx * 8) sK[g] = kv;  // the group's first channel is this thread's
                }
                k[i] = kv;
            }
        }
        uint32_t kp[4];  // the shifts again as packed 16-bit pairs (exact: they ARE stored values)
#pragma unroll
        for (int i = 0; i < 4; ++i) kp[i] = pack2(k[2 * i], k[2 * i + 1], BF16);
        const int row0 = blockIdx.x * a.rows_per_block;
        const int row1 = min(row0 + a.rows_per_block, a.hw);
        // one pointer walked down the rows (no 64-bit multiply per load)
        const uint16_t* ptr = a.x + ((size_t)img * a.hw + row0 + ty) * a.ldx + tx * 8;
        const size_t step = (size_t)by * a.ldx;
        constexpr int kU = 8;
        for (int rb = row0 + ty; rb < row1; rb += by * kU, ptr += kU * step) {
            uint4 v[kU];
#pragma unroll
            for (int u = 0; u < kU; ++u)
                if (rb + u * by < row1) v[u] = *reinterpret_cast<const uint4*>(ptr + u * step);
#pragma unroll
            for (int u = 0; u < kU; ++u)
                if (rb + u * by < row1) gn_add8_t<BF16>(st, v[u], kp, k);
        }
    }
    gn_block_reduce(st, ty < by, tx, ty, by, a, red, acc);
    gn_store_slot(a, img, acc);
}

// gn_stats_kernel + the finish: the last CTA of an image to arrive (integer ticket) sums the image's slots
// in the fixed order and writes the per-channel (scale, shift) pairs the halo convolution applies.
template <int BF16>
__global__ void __launch_bounds__(kGnThreads) gn_stats_ab_kernel(const GnArgs a, float* __restrict__ ab,
                                                                  unsigned* counters) {
    __shared__ float acc[2 * 64];
    __shared__ float sK[64];
    __shared__ __align__(16) float red[kGnRedFloats];
    __shared__ int s_last;
    pdl_launch_dependents();
    // the finishing CTA reads gamma / beta at the very end of a dependent chain: pull them into L2 now
    // (parameters: not produced by the predecessor kernel, so before the dependency wait)
    if (blockIdx.x == 0 && (int)threadIdx.x * 32 < a.c) {
        asm volatile("prefetch.global.L2 [%0];" ::"l"(a.gamma + threadIdx.x * 32));
        asm volatile("prefetch.global.L2 [%0];" ::"l"(a.beta + threadIdx.x * 32));
    }
    pdl_wait();
    const int img = blockIdx.y;
    const int by = kGnThreads / a.nvec;
    const int tx = threadIdx.x % a.nvec;
    const int ty = threadIdx.x / a.nvec;
    GnAcc8 st;
    st.zero();
    if (ty < by) {
        // every thread fetches the shifts of its own 8 channels itself (one 2-byte load per group run, of a
        // line the whole group shares): in flight together with the first batch of rows instead of a
        // load -> barrier -> load chain
        float k[8];
        {
            int g_prev = -1;
            float kv = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int g = (tx * 8 + i) / a.cpg;
                if (g != g_prev) {
                    kv = load1(a.x, (size_t)img * a.hw * a.ldx + g * a.cpg, a.dtype);
                    g_prev = g;
                    if (ty == 0 && g * a.cpg >= tx * 8) sK[g] = kv;  // the group's first channel is this thread's
                }
                k[i] = kv;
            }
        }
        uint32_t kp[4];  // the shifts again as packed 16-bit pairs (exact: they ARE stored values)
#pragma unroll
        for (int i = 0; i < 4; ++i) kp[i] = pack2(k[2 * i], k[2 * i + 1], BF16);
        const int row0 = blockIdx.x * a.rows_per_block;
        const int row1 = min(row0 + a.rows_per_block, a.hw);
        // one pointer walked down the rows (no 64-bit multiply per load)
        const uint16_t* ptr = a.x + ((size_t)img * a.hw + row0 + ty) * a.ldx + tx * 8;
        const size_t step = (size_t)by * a.ldx;
        constexpr int kU = 8;
        for (int rb = row0 + ty; rb < row1; rb += by * kU, ptr += kU * step) {
            uint4 v[kU];
#pragma unroll
            for (int u = 0; u < kU; ++u)
                if (rb + u * by < row1) v[u] = *reinterpret_cast<const uint4*>(ptr + u * step);
#pragma unroll
            for (int u = 0; u < kU; ++u)
                if (rb + u * by < row1) gn_add8_t<BF16>(st, v[u], kp, k);
        }
    }
    gn_block_reduce(st, ty < by, tx, ty, by, a, red, acc);
    gn_store_slot(a, img, acc);
    __threadfence();   // this CTA's slot is visible device-wide before its ticket is
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(&counters[img], 1u) == gridDim.x - 1) ? 1 : 0;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    gn_sum_slots(a, img, red, acc);
    const float inv_cnt = 1.0f / ((float)a.hw * (float)a.cpg);
    for (int ch = threadIdx.x; ch < a.c; ch += kGnThreads) {
        float sc, sh;
        gn_scale_shift(a, acc, sK, inv_cnt, ch, a.gamma[ch], a.beta[ch], sc, sh);
        *reinterpret_cast<float2*>(ab + ((size_t)img * a.c + ch) * 2) = make_float2(sc, sh);
    }
    if (threadIdx.x == 0) counters[img] = 0;  // every CTA of the image has arrived: ready for the next launch
}

// grid (blocks_per_img, n): per-channel scale/shift for this image staged in shared memory, then
// a streaming y = act(x * scale + shift) over the block's rows with 16-byte accesses.
__global__ void __launch_bounds__(kGnThreads) gn_apply_kernel(const GnArgs a) {
    extern __shared__ float sm[];
    __shared__ float sK[64];
    __shared__ float acc[2 * 64];
    __shared__ float red[kGnThreads];
    pdl_launch_dependents();
    pdl_wait();
    float* scale = sm;
    float* shift = sm + a.c;
    const int img = blockIdx.y;
    const float inv_cnt = 1.0f / ((float)a.hw * (float)a.cpg);
    gn_load_shifts<false>(a, img, sK);
    gn_sum_slots(a, img, red, acc);  // (the statistics kernel ran with the same grid: one slot per CTA of it)
    for (int ch = threadIdx.x; ch < a.c; ch += kGnThreads)
        gn_scale_shift(a, acc, sK, inv_cnt, ch, a.gamma[ch], a.beta[ch], scale[ch], shift[ch]);
    __syncthreads();
    const int row0 = blockIdx.x * a.rows_per_block;
    const int row1 = min(row0 + a.rows_per_block, a.hw);
    const int items = (row1 - row0) * a.nvec;
    const uint16_t* xb = a.x + ((size_t)img * a.hw + row0) * a.ldx;
    uint16_t* yb = a.y + ((size_t)img * a.hw + row0) * a.ldy;
    constexpr int kU = 4;
    for (int it0 = threadIdx.x; it0 < items; it0 += kGnThreads * kU) {
        uint4 v[kU];
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            const int it = it0 + u * kGnThreads;
            if (it < items) {
                const int row = it / a.nvec, vec = it - row * a.nvec;
                v[u] = *reinterpret_cast<const uint4*>(xb + (size_t)row * a.ldx + vec * 8);
            }
        }
#pragma unroll
        for (int u = 0; u < kU; ++u) {
            const int it = it0 + u * kGnThreads;
            if (it >= items) continue;
            const int row = it / a.nvec, vec = it - row * a.nvec;
            const uint32_t w[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
            uint32_t o[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 f = unpack2(w[i], a.dtype);
                const int ch = vec * 8 + 2 * i;
                float y0 = f.x * scale[ch] + shift[ch];
                float y1 = f.y * scale[ch + 1] + shift[ch + 1];
                if (a.silu) { y0 = silu_f(y0); y1 = silu_f(y1); }
                o[i] = pack2(y0, y1, a.dtype);
            }
            *reinterpret_cast<uint4*>(yb + (size_t)row * a.ldy + vec * 8) = make_uint4(o[0], o[1], o[2], o[3]);
        }
    }
}


// ---------------------------------------------------------------------------------------
// Fused GroupNorm for tensors that fit in the machine's shared memory (the B <= 2 regime the
// SD-1.5 bs=1 config lives in): ONE launch, x is read from HBM/L2 once.
//   phase 1  each CTA pulls its slab of rows into shared memory and accumulates group sums
//            (fp32, one global atomic per (CTA, group, moment));
//   barrier  grid-wide arrive/spin on a global counter (grid <= 148 CTAs, all co-resident);
//   phase 2  scale/shift from the finished statistics, y = act(x * scale + shift) from smem.
// ---------------------------------------------------------------------------------------
template <bool kPart>
__global__ void __launch_bounds__(kGnThreads) gn_fused_kernel(const GnArgs a, unsigned* sync_counter) {
    extern __shared__ __align__(16) uint8_t fsm[];
    __shared__ float acc[2 * 64];
    __shared__ float sK[64];
    __shared__ __align__(16) float red[kGnRedFloats];
    float* scale = reinterpret_cast<float*>(fsm);
    float* shift = scale + a.c;
    uint4* slab = reinterpret_cast<uint4*>(fsm + 2 * a.c * sizeof(float));
    pdl_launch_dependents();
    pdl_wait();
    const int img = blockIdx.y;
    const int by = kGnThreads / a.nvec;
    const int tx = threadIdx.x % a.nvec;
    const int ty = threadIdx.x / a.nvec;
    const int row0 = blockIdx.x * a.rows_per_block;
    const int row1 = min(row0 + a.rows_per_block, a.hw);
    const uint16_t* base = a.x + (size_t)img * a.hw * a.ldx + tx * 8;
    GnAcc8 st;
    st.zero();
    if constexpr (kPart) {
        // channels [0, part_c) come from the producer GEMM's split-K partials (a few rows per thread,
        // each with all its partial loads in flight); the shifts need a finished value -> shared memory
        gn_load_shifts<true>(a, img, sK);
        if (ty < by) {
            const bool from_partials = tx * 8 < a.part_c;
            for (int row = row0 + ty; row < row1; row += by)
                slab[(row - row0) * a.nvec + tx] = from_partials
                    ? gn_finish_partials(a, img, row, tx)
                    : *reinterpret_cast<const uint4*>(base + (size_t)row * a.ldx);
        }
        __syncthreads();  // shifts visible; each thread re-reads only its own slab rows
        if (ty < by) {
            float k[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) k[i] = sK[(tx * 8 + i) / a.cpg];
            for (int row = row0 + ty; row < row1; row += by) st.add(slab[(row - row0) * a.nvec + tx], k, a.dtype);
        }
    } else {
        if (ty < by) {
            // every thread fetches the shifts of its own 8 channels itself (a group's shift is one
            // 2-byte load of a line all threads of the group share): they are in flight together with
            // the slab loads, and the sums accumulate straight from the registers the loads land in
            float k[8];
            {
                int g_prev = -1;
                float kv = 0.f;
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int g = (tx * 8 + i) / a.cpg;
                    if (g != g_prev) {
                        kv = load1(a.x, (size_t)img * a.hw * a.ldx + g * a.cpg, a.dtype);
                        g_prev = g;
                        if (ty == 0 && g * a.cpg >= tx * 8) sK[g] = kv;  // the group's first channel is this thread's
                    }
                    k[i] = kv;
                }
            }
            // all of a thread's loads of one batch are in flight together: the slab is a handful of
            // rows per thread, so a load-use-load chain would be nothing but exposed L2 latency
            constexpr int kU = 8;
            for (int rb = row0 + ty; rb < row1; rb += by * kU) {
                uint4 v[kU];
#pragma unroll
                for (int u = 0; u < kU; ++u) {
                    const int row = rb + u * by;
                    if (row < row1) v[u] = *reinterpret_cast<const uint4*>(base + (size_t)row * a.ldx);
                }
#pragma unroll
                for (int u = 0; u < kU; ++u) {
                    const int row = rb + u * by;
                    if (row < row1) {
                        slab[(row - row0) * a.nvec + tx] = v[u];
                        st.add(v[u], k, a.dtype);
                    }
                }
            }
        }
    }
    gn_block_reduce(st, ty < by, tx, ty, by, a, red, acc);
    gn_store_slot(a, img, acc);
    // affine parameters do not depend on the statistics: fetch them (cold, from HBM) while the
    // grid barrier is pending
    for (int ch = threadIdx.x; ch < a.c; ch += kGnThreads) {
        scale[ch] = a.gamma[ch];
        shift[ch] = a.beta[ch];
    }
    // ---- grid barrier.  The launch is COOPERATIVE (cudaLaunchAttributeCooperative): the driver
    // only starts the grid when every CTA can be resident, so the arrive / spin below cannot
    // wait for an unscheduled CTA -- not with other streams' kernels on the GPU, not on a MIG or
    // green-context slice (the grid is sized from the occupancy query, see sfb_group_norm_fused).
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned total = gridDim.x * gridDim.y;
        atomicAdd(sync_counter, 1u);
        while (*reinterpret_cast<volatile unsigned*>(sync_counter) < total) {
        }
        __threadfence();
    }
    __syncthreads();
    // ---- phase 2: every CTA of the image sums the image's slots in the same fixed order
    gn_sum_slots(a, img, red, acc);
    const float inv_cnt = 1.0f / ((float)a.hw * (float)a.cpg);
    for (int ch = threadIdx.x; ch < a.c; ch += kGnThreads) {
        float sc, sh;
        gn_scale_shift(a, acc, sK, inv_cnt, ch, scale[ch], shift[ch], sc, sh);
        scale[ch] = sc;
        shift[ch] = sh;
    }
    __syncthreads();
    if (ty < by) {
        uint16_t* yb = a.y + (size_t)img * a.hw * a.ldy + tx * 8;
        float sc[8], sh[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) { sc[i] = scale[tx * 8 + i]; sh[i] = shift[tx * 8 + i]; }
        for (int row = row0 + ty; row < row1; row += by) {
            const uint4 v = slab[(row - row0) * a.nvec + tx];
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
            uint32_t o[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 f = unpack2(w[i], a.dtype);
                float y0 = f.x * sc[2 * i] + sh[2 * i];
                float y1 = f.y * sc[2 * i + 1] + sh[2 * i + 1];
                if (a.silu) { y0 = silu_f(y0); y1 = silu_f(y1); }
                o[i] = pack2(y0, y1, a.dtype);
            }
            *reinterpret_cast<uint4*>(yb + (size_t)row * a.ldy) = make_uint4(o[0], o[1], o[2], o[3]);
        }
    }
}

constexpr int kGnFusedMaxSmem = 190 * 1024;  // + 33 KB of static scratch for the ordered reductions

// grid geometry of the fused kernel; returns false if the tensor does not fit in shared memory
static bool gn_fused_geometry(const sfb_gn_params* p, int& blocks_per_img, int& rows_per_block,
                              size_t& smem) {
    const int sms = sm_count();
    if (p->n <= 0 || p->n > sms) return false;
    blocks_per_img = sms / p->n;
    if (blocks_per_img > p->hw) blocks_per_img = p->hw;
    if (blocks_per_img < 1) return false;
    rows_per_block = (p->hw + blocks_per_img - 1) / blocks_per_img;
    blocks_per_img = (p->hw + rows_per_block - 1) / rows_per_block;
    smem = (size_t)rows_per_block * p->c * 2 + 2 * (size_t)p->c * sizeof(float);
    return smem <= (size_t)kGnFusedMaxSmem;
}

struct LnArgs {
    const uint16_t* x;
    uint16_t* y;
    const float* gamma;
    const float* beta;
    int rows, c, ldx, ldy, nvec;
    float eps;
    int dtype;
};

constexpr int kLnMaxVec = 8;  // c <= 8 * 32 * 8 = 2048

__global__ void __launch_bounds__(256) layer_norm_kernel(const LnArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= a.rows) return;
    const uint16_t* xr = a.x + (size_t)warp * a.ldx;
    float v[kLnMaxVec][8];
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < kLnMaxVec; ++j) {
        const int vec = lane + j * 32;
        if (vec < a.nvec) {
            const uint4 u = *reinterpret_cast<const uint4*>(xr + vec * 8);
            const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 f = unpack2(w[i], a.dtype);
                v[j][2 * i] = f.x; v[j][2 * i + 1] = f.y;
                sum += f.x + f.y;
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / (float)a.c;
    float sq = 0.f;
#pragma unroll
    for (int j = 0; j < kLnMaxVec; ++j) {
        if (lane + j * 32 < a.nvec) {
#pragma unroll
            for (int i = 0; i < 8; ++i) { const float d = v[j][i] - mean; sq += d * d; }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    const float rstd = rsqrtf(sq / (float)a.c + a.eps);
    uint16_t* yr = a.y + (size_t)warp * a.ldy;
#pragma unroll
    for (int j = 0; j < kLnMaxVec; ++j) {
        const int vec = lane + j * 32;
        if (vec < a.nvec) {
            const float4 g0 = *reinterpret_cast<const float4*>(a.gamma + vec * 8);
            const float4 g1 = *reinterpret_cast<const float4*>(a.gamma + vec * 8 + 4);
            const float4 b0 = *reinterpret_cast<const float4*>(a.beta + vec * 8);
            const float4 b1 = *reinterpret_cast<const float4*>(a.beta + vec * 8 + 4);
            const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
            const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
            uint32_t o[4];
#pragma unroll
            for (int i = 0; i < 4; ++i)
                o[i] = pack2((v[j][2 * i] - mean) * rstd * g[2 * i] + b[2 * i],
                             (v[j][2 * i + 1] - mean) * rstd * g[2 * i + 1] + b[2 * i + 1], a.dtype);
            *reinterpret_cast<uint4*>(yr + vec * 8) = make_uint4(o[0], o[1], o[2], o[3]);
        }
    }
}

static int make_gn_args(const sfb_gn_params* p, GnArgs& a, int& blocks_per_img) {
    if (!p || !p->x || !p->stats) return fail(SFB_ERR_INVALID, "group_norm: null argument");
    // n and hw divide the grid sizing below (an empty tensor has nothing to normalise)
    if (p->n <= 0 || p->hw <= 0) return fail(SFB_ERR_INVALID, "group_norm: n=%d and hw=%d must be positive", p->n, p->hw);
    if (p->c <= 0 || p->c % 8 || p->ldx % 8 || p->groups <= 0 || p->groups > 64 || p->c % p->groups ||
        p->c / 8 > kGnThreads || p->c > 4096)
        return fail(SFB_ERR_INVALID, "group_norm: unsupported geometry c=%d groups=%d ldx=%d", p->c, p->groups, p->ldx);
    a.x = reinterpret_cast<const uint16_t*>(p->x);
    a.y = reinterpret_cast<uint16_t*>(p->y);
    a.gamma = p->gamma; a.beta = p->beta; a.stats = p->stats;
    a.n = p->n; a.hw = p->hw; a.c = p->c; a.ldx = p->ldx; a.ldy = p->ldy; a.groups = p->groups;
    a.cpg = p->c / p->groups; a.nvec = p->c / 8; a.eps = p->eps; a.silu = p->silu; a.dtype = p->dtype;
    const int by = kGnThreads / a.nvec;
    // aim for >= 2 waves of the SMs while giving each thread a few rows
    int want = (2 * sm_count() + p->n - 1) / p->n;
    int max_blocks = (p->hw + by - 1) / by;
    blocks_per_img = want < max_blocks ? want : max_blocks;
    if (blocks_per_img < 1) blocks_per_img = 1;
    a.rows_per_block = (p->hw + blocks_per_img - 1) / blocks_per_img;
    blocks_per_img = (p->hw + a.rows_per_block - 1) / a.rows_per_block;
    return SFB_OK;
}

}  // namespace sfb

using namespace sfb;

extern "C" int sfb_group_norm_stats(const sfb_gn_params* p, sfb_stream_t stream) {
    GnArgs a{};
    int bpi = 1;
    int rc = make_gn_args(p, a, bpi);
    if (rc) return rc;
    cudaError_t err = p->dtype == SFB_BF16
        ? launch_pdl(gn_stats_kernel<1>, dim3(bpi, p->n), dim3(kGnThreads), 0, static_cast<cudaStream_t>(stream), a)
        : launch_pdl(gn_stats_kernel<0>, dim3(bpi, p->n), dim3(kGnThreads), 0, static_cast<cudaStream_t>(stream), a);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "group_norm_stats: %s", cudaGetErrorString(err));
    return check_launch("sfb_group_norm_stats");
}

extern "C" int sfb_group_norm_scale_shift(const sfb_gn_params* p, float* scale_shift, sfb_stream_t stream) {
    GnArgs a{};
    int bpi = 1;
    int rc = make_gn_args(p, a, bpi);
    if (rc) return rc;
    if (!scale_shift || !p->gamma || !p->beta || !p->sync_counter)
        return fail(SFB_ERR_INVALID, "group_norm_scale_shift: null scale_shift / gamma / beta / sync_counter");
    cudaError_t err = p->dtype == SFB_BF16
        ? launch_pdl(gn_stats_ab_kernel<1>, dim3(bpi, p->n), dim3(kGnThreads), 0, static_cast<cudaStream_t>(stream), a,
                     scale_shift, p->sync_counter)
        : launch_pdl(gn_stats_ab_kernel<0>, dim3(bpi, p->n), dim3(kGnThreads), 0, static_cast<cudaStream_t>(stream), a,
                     scale_shift, p->sync_counter);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "group_norm_scale_shift: %s", cudaGetErrorString(err));
    return check_launch("sfb_group_norm_scale_shift");
}

extern "C" int sfb_group_norm_apply(const sfb_gn_params* p, sfb_stream_t stream) {
    GnArgs a{};
    int bpi = 1;
    int rc = make_gn_args(p, a, bpi);
    if (rc) return rc;
    if (!p->y || !p->gamma || !p->beta || p->ldy % 8) return fail(SFB_ERR_INVALID, "group_norm_apply: null/ldy");
    cudaError_t err = launch_pdl(gn_apply_kernel, dim3(bpi, p->n), dim3(kGnThreads),
                                 2 * p->c * sizeof(float), static_cast<cudaStream_t>(stream), a);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "group_norm_apply: %s", cudaGetErrorString(err));
    return check_launch("sfb_group_norm_apply");
}


extern "C" int sfb_group_norm_ws_floats(int32_t n, int32_t groups) {
    // two-pass grid: n * ceil(2 * SMs / n) <= 2 * SMs + n CTAs; fused grid: <= SMs CTAs
    return (2 * sm_count() + (n > 0 ? n : 1)) * 2 * (groups > 0 ? groups : 1);
}

extern "C" int sfb_group_norm_fused_fits(const sfb_gn_params* p) {
    int bpi, rpb;
    size_t smem;
    if (!p || p->c % 8 || p->c <= 0 || p->groups <= 0 || p->c % p->groups || p->c / 8 > kGnThreads) return 0;
    return gn_fused_geometry(p, bpi, rpb, smem) ? 1 : 0;
}

// Cooperative launch of the fused kernel (the grid barrier needs every CTA resident).  The
// programmatic-dependent-launch attribute is added when the driver accepts the combination
// (probed once per device on the first launch, outside any graph capture: the runtime's warm-up
// pass precedes capture).
template <bool kPart>
static cudaError_t launch_gn_fused(dim3 grid, size_t smem, cudaStream_t stream, const GnArgs& a, unsigned* sync) {
    static int pdl_ok[64];  // 0 unknown, 1 yes, -1 no
    const int dev = current_device();
    // measurement switch only: SFB_GN_COOP=0 launches the kernel WITHOUT the co-residency guarantee
    static const bool coop = [] { const char* v = getenv("SFB_GN_COOP"); return !(v && v[0] == '0'); }();
    if (!coop) return launch_pdl(gn_fused_kernel<kPart>, grid, dim3(kGnThreads), smem, stream, a, sync);
    for (int attempt = 0; attempt < 2; ++attempt) {
        const bool with_pdl = g_pdl && pdl_ok[dev] >= 0;
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = grid;
        cfg.blockDim = dim3(kGnThreads);
        cfg.dynamicSmemBytes = smem;
        cfg.stream = stream;
        cudaLaunchAttribute attr[2];
        int n = 0;
        attr[n].id = cudaLaunchAttributeCooperative;
        attr[n].val.cooperative = 1;
        ++n;
        if (with_pdl) {
            attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
            attr[n].val.programmaticStreamSerializationAllowed = 1;
            ++n;
        }
        cfg.attrs = attr;
        cfg.numAttrs = n;
        const cudaError_t err = cudaLaunchKernelEx(&cfg, gn_fused_kernel<kPart>, a, sync);
        if (err == cudaSuccess) {
            if (with_pdl) pdl_ok[dev] = 1;
            return err;
        }
        if (!with_pdl || pdl_ok[dev] == 1) return err;
        cudaGetLastError();
        pdl_ok[dev] = -1;  // cooperative + PDL refused: cooperative alone from now on
    }
    return cudaErrorUnknown;
}

extern "C" int sfb_group_norm_fused(const sfb_gn_params* p, sfb_stream_t stream) {
    GnArgs a{};
    int bpi = 1;
    int rc = make_gn_args(p, a, bpi);
    if (rc) return rc;
    if (!p->y || !p->gamma || !p->beta || p->ldy % 8 || !p->sync_counter)
        return fail(SFB_ERR_INVALID, "group_norm_fused: null/ldy/sync_counter");
    int rpb = 0;
    size_t smem;
    if (!gn_fused_geometry(p, bpi, rpb, smem))
        return fail(SFB_ERR_INVALID, "group_norm_fused: tensor does not fit in shared memory");
    a.rows_per_block = rpb;
    if (p->part_splits > 1) {
        if (!p->part_ws || p->part_c <= 0 || p->part_c % 8 || p->part_c > p->c || p->part_ld % 4 ||
            p->part_ld < p->part_c || (p->part_residual && p->part_ldr % 8))
            return fail(SFB_ERR_INVALID, "group_norm_fused: bad deferred split-K description");
        a.part_ws = p->part_ws; a.part_splits = p->part_splits; a.part_c = p->part_c; a.part_ld = p->part_ld;
        a.part_bias = p->part_bias; a.part_rowbias = p->part_rowbias; a.part_ld_rowbias = p->part_ld_rowbias;
        a.part_residual = reinterpret_cast<const uint16_t*>(p->part_residual); a.part_ldr = p->part_ldr;
    }
    static PerDeviceOnce attr_once;
    bool& attr_set = attr_once.flag();
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(gn_fused_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             kGnFusedMaxSmem);
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(gn_fused_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     kGnFusedMaxSmem);
        if (e != cudaSuccess) return fail(SFB_ERR_CUDA, "group_norm_fused: smem attribute: %s", cudaGetErrorString(e));
        attr_set = true;
    }
    // the whole grid must be co-resident: check against the occupancy of this kernel on this device
    int per_sm = 0;
    cudaError_t oe = a.part_splits > 1
        ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gn_fused_kernel<true>, kGnThreads, smem)
        : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gn_fused_kernel<false>, kGnThreads, smem);
    if (oe != cudaSuccess || (long long)per_sm * sm_count() < (long long)bpi * p->n)
        return fail(SFB_ERR_INVALID, "group_norm_fused: grid of %d CTAs cannot be co-resident (%d per SM x %d SMs)",
                    bpi * p->n, per_sm, sm_count());
    const dim3 grid(bpi, p->n);
    cudaError_t err = a.part_splits > 1
        ? launch_gn_fused<true>(grid, smem, static_cast<cudaStream_t>(stream), a, p->sync_counter)
        : launch_gn_fused<false>(grid, smem, static_cast<cudaStream_t>(stream), a, p->sync_counter);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "group_norm_fused: %s", cudaGetErrorString(err));
    return check_launch("sfb_group_norm_fused");
}

extern "C" int sfb_layer_norm(const sfb_ln_params* p, sfb_stream_t stream) {
    if (!p || !p->x || !p->y || !p->gamma || !p->beta) return fail(SFB_ERR_INVALID, "layer_norm: null argument");
    if (p->c <= 0 || p->c % 8 || p->c > kLnMaxVec * 256 || p->ldx % 8 || p->ldy % 8 || p->rows <= 0)
        return fail(SFB_ERR_INVALID, "layer_norm: unsupported geometry c=%d", p->c);
    LnArgs a{};
    a.x = reinterpret_cast<const uint16_t*>(p->x);
    a.y = reinterpret_cast<uint16_t*>(p->y);
    a.gamma = p->gamma; a.beta = p->beta; a.rows = p->rows; a.c = p->c; a.ldx = p->ldx; a.ldy = p->ldy;
    a.nvec = p->c / 8; a.eps = p->eps; a.dtype = p->dtype;
    const int blocks = (p->rows + 7) / 8;
    cudaError_t err = launch_pdl(layer_norm_kernel, dim3(blocks), dim3(256), 0,
                                 static_cast<cudaStream_t>(stream), a);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "layer_norm: %s", cudaGetErrorString(err));
    return check_launch("sfb_layer_norm");
}
