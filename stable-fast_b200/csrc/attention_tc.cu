// wgmma flash attention for sm_90a:  O = softmax(Q K^T * scale) V, one (batch, head, 128-query
// tile) per CTA, online softmax over 128- or 64-wide KV tiles.
//
// Warp roles (288 threads):
//   warps 0..7  two consumer warpgroups, each owning 64 query rows:
//                 S = Q K^T   wgmma.m64nKVk16, Q and K from shared memory, S in registers;
//                 softmax in registers: running max over the row's four threads, one FFMA
//                 (s*scale*log2e - max) + exp2 per element, P packed to 16 bits straight into the
//                 A-operand fragments of
//                 O += P V    wgmma.m64nDVk16 with A from registers, V^T from shared memory.
//               The softmax denominator costs nothing: row `head_dim` of V^T is all ones, so column
//               `head_dim` of O accumulates sum(P) on the tensor core, consistently with the rounded P
//               and the O rescales;
//   warp 8      TMA producer: Q once, then a ring of K tiles and a ring of V^T tiles.
// All three operands are K-major: Q/K as [rows, head_dim] and V pre-transposed as V^T
// [head_dim, seq] -- the QKV projection's epilogue (gemm_tc.cu, SFB_EPI_QKV) writes those
// layouts directly, so no permute/copy kernels exist between projection and attention.
//
// attention_ip_kernel (sfb_attention_ip) is the same body with IP-Adapter's image-prompt term added after the
// text tiles: O + s * softmax(Q K_ip^T * scale) V_ip, the image tokens being one more KV tile.
//
// Replaces xformers.ops.memory_efficient_attention as wrapped at
// /root/reference/src/sfast/libs/xformers/xformers_attention.py:26-63.
#include "common.cuh"
#include "host.h"

#include <stdlib.h>
#include <string.h>

namespace sfb {

constexpr int kAttnThreads = 288;  // two consumer warpgroups + one TMA producer warp
constexpr int kTileQ = 128;

struct AttnArgs {
    void* out;
    int batch, heads, head_dim;
    int seq_q, seq_kv;
    int q_rows, k_rows, vt_rows;
    int dtype;
    float scale_log2;  // scale * log2(e)
    int causal;        // v2 only: key j is visible to query i iff j <= i
};

__device__ __forceinline__ float fast_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// 2^x on the FMA / ALU pipes instead of the MUFU (special-function) pipe: Cody-Waite split
// x = n + f, f in [-0.5, 0.5], 2^f by a degree-3 minimax polynomial (max relative error 1.0e-4,
// below the half-ulp of the 16-bit probability it is rounded to), 2^n by an integer add into the
// exponent.  The softmax of these kernels is bound by MUFU.EX2 (16 lanes / clk / SM against 128 for
// FMA): one exponential per score with head_dim 40 / 64 means one MUFU op per 160 / 256 tensor FLOPs.
// Sending a fixed fraction of every row's exponentials through this routine (kPolyMask: which of each
// 8 consecutive scores) trades 8 extra issue slots per element for a free MUFU slot; the balance
// point of the two pipes was estimated at ~30 %, measured lower (below).  x <= ~8 here (lazy maximum).
__device__ __forceinline__ float poly_exp2(float x) {
    x = fmaxf(x, -125.0f);                       // 2^-125: a zero probability after rounding
    const float t = x + 12582912.0f;             // 1.5 * 2^23: round(x) lands in the low mantissa bits
    const float f = x - (t - 12582912.0f);       // [-0.5, 0.5]
    float p = fmaf(f, 0.05500893f, 0.24221096f);
    p = fmaf(p, f, 0.69328293f);
    p = fmaf(p, f, 1.0f);
    return __int_as_float(__float_as_int(p) + (__float_as_int(t) << 23));
}
// The split is per KV tile size: 1 of every 8 exponentials of the 128-key kernel, none in the 64-key
// kernel.  (The split was tuned on an earlier build of these kernels; it is not re-tuned for the H100.)
#ifndef SFB_EXP_POLY_MASK
#define SFB_EXP_POLY_MASK 0x08   // element 3 of every 8 scores: 12.5 % of the exponentials
#endif
constexpr unsigned kPolyMaskV1 = SFB_EXP_POLY_MASK;  // 128-key tiles
constexpr unsigned kPolyMaskV2 = 0x00;               // 64-key tiles
template <int I, unsigned MASK>
__device__ __forceinline__ float softmax_exp2(float x) {
    if constexpr ((MASK >> (I & 7)) & 1u) return poly_exp2(x);
    else return fast_exp2(x);
}

__device__ __forceinline__ float fmax3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }

// Shared memory: Q [DC chunks][128 rows][64 head dims], a ring of K tiles [DC][KV rows][64] and a ring
// of V^T tiles [KV / 64 chunks][DV rows][64 keys], all 128-byte-swizzled K-major (what TMA writes and
// wgmma reads).  P never leaves the registers: the accumulator fragment of S is the A operand of P V.
template <int DC, int DV, int KV, int KVS>
struct AttnSmem {
    static constexpr int kQBytes = DC * kTileQ * 128;
    static constexpr int kKStage = DC * KV * 128;
    static constexpr int kVChunk = DV * 128;  // [DV rows x 64 kv columns]
    static constexpr int kVStage = (KV / 64) * kVChunk;
    static constexpr int kOffK = kQBytes;
    static constexpr int kOffV = kOffK + KVS * kKStage;
    static constexpr int kOffBar = kOffV + KVS * kVStage;
    static constexpr int kTotal = kOffBar + 256 + 1024;
    static_assert(kVChunk % 1024 == 0, "V^T chunk must keep 1024-byte swizzle-atom alignment");
    static_assert(kTotal <= 227 * 1024, "shared memory per block");
};

// Image-prompt (IP-Adapter) term of sfb_attention_ip: one more key / value set of at most one KV tile,
// attended with its own softmax and added as `*scale` times its output.
struct IpArgs {
    int seq_ip, k_ip_rows;
    const float* scale;  // device memory: a captured graph serves every scale
};

// HD = head_dim (DK: HD rounded up to 16).  IP: the image-prompt pass after the text tiles (below).
template <int DC, int HD, int DK, int DV, int KV, int KVS, int BF16, bool IP>
__device__ __forceinline__ void attention_body(const CUtensorMap* tma_q, const CUtensorMap* tma_k,
                                               const CUtensorMap* tma_vt, const AttnArgs& a,
                                               const CUtensorMap* tma_k_ip, const CUtensorMap* tma_vt_ip,
                                               const IpArgs& ip) {
    using L = AttnSmem<DC, DV, KV, KVS>;
    constexpr unsigned kPolyMask = KV == 128 ? kPolyMaskV1 : kPolyMaskV2;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024 - (smem_u32(smem_raw) & 1023)) & 1023);
    uint8_t* sQ = smem;
    uint8_t* sK = smem + L::kOffK;
    uint8_t* sV = smem + L::kOffV;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::kOffBar);
    uint64_t* q_full = bars;
    uint64_t* k_full = bars + 1;
    uint64_t* k_empty = k_full + KVS;
    uint64_t* v_full = k_empty + KVS;
    uint64_t* v_empty = v_full + KVS;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int q_tile = blockIdx.x;
    const int bh = blockIdx.y;
    const int n_kv = (a.seq_kv + KV - 1) / KV;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(tma_q);
        tma_prefetch_desc(tma_k);
        tma_prefetch_desc(tma_vt);
        if constexpr (IP) {
            tma_prefetch_desc(tma_k_ip);
            tma_prefetch_desc(tma_vt_ip);
        }
        mbar_init(q_full, 1);
        for (int i = 0; i < KVS; ++i) {
            mbar_init(&k_full[i], 1);
            mbar_init(&k_empty[i], 2);  // one arrival per consumer warpgroup
            mbar_init(&v_full[i], 1);
            mbar_init(&v_empty[i], 2);
        }
        fence_barrier_init();
    }
    pdl_launch_dependents();
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            // only this thread reads the predecessor's output (Q/K/V via TMA); everything the other
            // warps do is ordered behind these loads
            pdl_wait();
            mbar_expect_tx(q_full, L::kQBytes);
#pragma unroll
            for (int c = 0; c < DC; ++c)
                tma_load_2d(sQ + c * (kTileQ * 128), tma_q, q_full, c * 64, bh * a.q_rows + q_tile * kTileQ);
            for (int j = 0; j < n_kv; ++j) {
                const int st = j % KVS;
                const uint32_t ph = (j / KVS) & 1;
                mbar_wait(&k_empty[st], ph ^ 1);
                mbar_expect_tx(&k_full[st], L::kKStage);
#pragma unroll
                for (int c = 0; c < DC; ++c)
                    tma_load_2d(sK + st * L::kKStage + c * (KV * 128), tma_k, &k_full[st], c * 64,
                                bh * a.k_rows + j * KV);
                mbar_wait(&v_empty[st], ph ^ 1);
                mbar_expect_tx(&v_full[st], L::kVStage);
#pragma unroll
                for (int c = 0; c < KV / 64; ++c)
                    tma_load_2d(sV + st * L::kVStage + c * L::kVChunk, tma_vt, &v_full[st], j * KV + c * 64,
                                bh * a.vt_rows);
            }
            // image-prompt keys / values: one more ring iteration (skipped, like the consumers' pass,
            // when the scale is 0)
            if constexpr (IP) {
                if (*ip.scale != 0.f) {
                    const int st = n_kv % KVS;
                    const uint32_t ph = (n_kv / KVS) & 1;
                    mbar_wait(&k_empty[st], ph ^ 1);
                    mbar_expect_tx(&k_full[st], L::kKStage);
#pragma unroll
                    for (int c = 0; c < DC; ++c)
                        tma_load_2d(sK + st * L::kKStage + c * (KV * 128), tma_k_ip, &k_full[st], c * 64,
                                    bh * ip.k_ip_rows);
                    mbar_wait(&v_empty[st], ph ^ 1);
                    mbar_expect_tx(&v_full[st], L::kVStage);
#pragma unroll
                    for (int c = 0; c < KV / 64; ++c)
                        tma_load_2d(sV + st * L::kVStage + c * L::kVChunk, tma_vt_ip, &v_full[st], c * 64,
                                    bh * a.vt_rows);
                }
            }
        }
    } else {
        // Consumer warpgroup wg owns query rows [64 wg, 64 wg + 64) of the tile.  Fragment ownership
        // (wgmma m64 accumulators): this thread holds rows g and g + 8 of its warp's 16 rows, g = lane / 4,
        // columns 8 jj + 2 (lane % 4) + {0, 1}: element 4 jj + e is row g + 8 (e >> 1), column
        // 8 jj + 2 (lane % 4) + (e & 1).
        const int wg = warp >> 2;
        const int row_g = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // tile row of elements e < 2
        const int qcol = 2 * (lane & 3);
        float o[DV / 2];
#pragma unroll
        for (int i = 0; i < DV / 2; ++i) o[i] = 0.f;
        float m_run[2] = {-INFINITY, -INFINITY};
        const float sl2 = a.scale_log2;
        mbar_wait(q_full, 0);
        for (int j = 0; j < n_kv; ++j) {
            const int st = j % KVS;
            const uint32_t ph = (j / KVS) & 1;
            // ---- S = Q K_j^T
            float s[KV / 2];
#pragma unroll
            for (int i = 0; i < KV / 2; ++i) s[i] = 0.f;
            mbar_wait(&k_full[st], ph);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < DK / 16; ++kk) {
                const int c = kk / 4, k4 = kk % 4;
                const uint64_t dq = wgmma_desc_k_sw128(smem_u32(sQ + c * (kTileQ * 128) + wg * 64 * 128));
                const uint64_t dk = wgmma_desc_k_sw128(smem_u32(sK + st * L::kKStage + c * (KV * 128)));
                wgmma_ss<BF16>(s, dq + (uint64_t)(k4 * 2), dk + (uint64_t)(k4 * 2));
            }
            wgmma_commit();
            wgmma_wait<0>(s);
            if ((threadIdx.x & 127) == 0) mbar_arrive(&k_empty[st]);

            // ragged tail: only the last KV tile can hold columns >= seq_kv.  causal (text encoders): a
            // row sees keys 0 .. its own position.  Key 0 is visible to every row, so tile 0 always moves
            // the running maximum off -inf; a later tile that is entirely masked for a row leaves
            // exp2(-inf) = 0 everywhere.
            int n_valid[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                n_valid[h] = a.seq_kv - j * KV;
                if (a.causal) n_valid[h] = min(n_valid[h], q_tile * kTileQ + row_g + 8 * h - j * KV + 1);
            }
            if (n_valid[0] < KV || n_valid[1] < KV) {
#pragma unroll
                for (int i = 0; i < KV / 2; ++i)
                    if ((i / 4) * 8 + qcol + (i & 1) >= n_valid[(i >> 1) & 1]) s[i] = -INFINITY;
            }
            // Lazy reference maximum: the softmax is invariant to the reference (O and the
            // denominator, which is column head_dim of O, carry the same factor), so the stale
            // reference is kept until a row's maximum exceeds it by more than 2^kLazyLog2 -- the
            // probabilities then stay <= 2^kLazyLog2 (exact in 16-bit floating point, fp32
            // accumulation) and O is rescaled only when some row's reference moved.
            constexpr float kLazyLog2 = 8.0f;
            float alpha[2], neg_m[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
                for (int jj = 0; jj < KV / 8; jj += 2) {
                    mx0 = fmax3(mx0, s[4 * jj + 2 * h], s[4 * jj + 2 * h + 1]);
                    mx1 = fmax3(mx1, s[4 * jj + 4 + 2 * h], s[4 * jj + 4 + 2 * h + 1]);
                }
                float mx = fmaxf(mx0, mx1);
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));  // the row's four threads
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                const float m_cand = mx * sl2;  // scale > 0
                const bool moved = m_cand > m_run[h] + kLazyLog2;  // always true on the first tile (-inf)
                const float m_new = moved ? m_cand : m_run[h];
                alpha[h] = moved ? fast_exp2(m_run[h] - m_new) : 1.0f;  // 0 on the first tile
                m_run[h] = m_new;
                neg_m[h] = -m_new;
            }
            // ---- P = exp2(S * scale * log2e - m), packed straight into the A fragments of P V
            uint32_t pa[KV / 16][4];
#pragma unroll
            for (int kc = 0; kc < KV / 16; ++kc) {
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    const int i = 8 * kc + 2 * r;  // elements i, i + 1: row half r & 1
                    const float nm = neg_m[r & 1];
                    pa[kc][r] = pack2(softmax_exp2<0, kPolyMask>(fmaf(s[i], sl2, nm)),
                                      softmax_exp2<1, kPolyMask>(fmaf(s[i + 1], sl2, nm)), BF16);
                }
            }
            if (alpha[0] != 1.0f || alpha[1] != 1.0f) {
#pragma unroll
                for (int i = 0; i < DV / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
            }
            // ---- O += P V_j
            mbar_wait(&v_full[st], ph);
            wgmma_fence();
#pragma unroll
            for (int kc = 0; kc < KV / 16; ++kc) {
                const int c = kc / 4, k4 = kc % 4;
                const uint64_t dv = wgmma_desc_k_sw128(smem_u32(sV + st * L::kVStage + c * L::kVChunk));
                wgmma_rs<BF16>(o, pa[kc], dv + (uint64_t)(k4 * 2));
            }
            wgmma_commit();
            wgmma_wait<0>(o);
            if ((threadIdx.x & 127) == 0) mbar_arrive(&v_empty[st]);
        }
        // final: O / l, with l = O[:, head_dim] (the ones row of V^T), held by lane (lane & ~3) + src
        constexpr int hd = HD;
        float l[2] = {1.f, 1.f};
#pragma unroll
        for (int jj = 0; jj < DV / 8; ++jj)
            if (jj == (hd >> 3)) {
                l[0] = (hd & 1) ? o[4 * jj + 1] : o[4 * jj];
                l[1] = (hd & 1) ? o[4 * jj + 3] : o[4 * jj + 2];
            }
        const int src = (lane & ~3) | ((hd & 7) >> 1);
        float inv_l[2];
#pragma unroll
        for (int rh = 0; rh < 2; ++rh) inv_l[rh] = 1.0f / __shfl_sync(0xffffffffu, l[rh], src);
        if constexpr (IP) {
            // O = O_text / l + s * softmax(Q K_ip^T * scale) V_ip.  The text output is normalised in fp32
            // first (the same product the plain store rounds), then the image term is added on the tensor
            // core with its probabilities pre-multiplied by s / l_ip: no second accumulator.  s == 0 skips
            // the pass, so the stored bits are exactly sfb_attention's.
            const float s_ip = *ip.scale;
            if (s_ip != 0.f) {
                const int st = n_kv % KVS;
                const uint32_t ph = (n_kv / KVS) & 1;
                float s[KV / 2];
#pragma unroll
                for (int i = 0; i < KV / 2; ++i) s[i] = 0.f;
                mbar_wait(&k_full[st], ph);
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < DK / 16; ++kk) {
                    const int c = kk / 4, k4 = kk % 4;
                    const uint64_t dq = wgmma_desc_k_sw128(smem_u32(sQ + c * (kTileQ * 128) + wg * 64 * 128));
                    const uint64_t dk = wgmma_desc_k_sw128(smem_u32(sK + st * L::kKStage + c * (KV * 128)));
                    wgmma_ss<BF16>(s, dq + (uint64_t)(k4 * 2), dk + (uint64_t)(k4 * 2));
                }
                wgmma_commit();
                wgmma_wait<0>(s);
                // columns >= seq_ip: the next (batch, head)'s rows or TMA zero fill
                if (ip.seq_ip < KV) {
#pragma unroll
                    for (int i = 0; i < KV / 2; ++i)
                        if ((i / 4) * 8 + qcol + (i & 1) >= ip.seq_ip) s[i] = -INFINITY;
                }
                float neg_m[2], l_ip[2] = {0.f, 0.f};
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float mx = -INFINITY;
#pragma unroll
                    for (int jj = 0; jj < KV / 8; ++jj) mx = fmax3(mx, s[4 * jj + 2 * h], s[4 * jj + 2 * h + 1]);
                    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                    neg_m[h] = -mx * sl2;  // column 0 is always valid: finite
                }
#pragma unroll
                for (int i = 0; i < KV / 2; ++i) {
                    s[i] = fast_exp2(fmaf(s[i], sl2, neg_m[(i >> 1) & 1]));
                    l_ip[(i >> 1) & 1] += s[i];
                }
                float f[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    l_ip[h] += __shfl_xor_sync(0xffffffffu, l_ip[h], 1);
                    l_ip[h] += __shfl_xor_sync(0xffffffffu, l_ip[h], 2);
                    f[h] = s_ip / l_ip[h];
                }
                uint32_t pa[KV / 16][4];
#pragma unroll
                for (int kc = 0; kc < KV / 16; ++kc)
#pragma unroll
                    for (int r = 0; r < 4; ++r) {
                        const int i = 8 * kc + 2 * r;
                        pa[kc][r] = pack2(s[i] * f[r & 1], s[i + 1] * f[r & 1], BF16);
                    }
#pragma unroll
                for (int i = 0; i < DV / 2; ++i) o[i] *= inv_l[(i >> 1) & 1];
                mbar_wait(&v_full[st], ph);
                wgmma_fence();
#pragma unroll
                for (int kc = 0; kc < KV / 16; ++kc) {
                    const int c = kc / 4, k4 = kc % 4;
                    const uint64_t dv = wgmma_desc_k_sw128(smem_u32(sV + st * L::kVStage + c * L::kVChunk));
                    wgmma_rs<BF16>(o, pa[kc], dv + (uint64_t)(k4 * 2));
                }
                wgmma_commit();
                wgmma_wait<0>(o);
                inv_l[0] = inv_l[1] = 1.f;
            }
        }
        const int b = bh / a.heads, h = bh % a.heads;
#pragma unroll
        for (int rh = 0; rh < 2; ++rh) {
            const int srow = q_tile * kTileQ + row_g + 8 * rh;
            if (srow < a.seq_q) {
                uint16_t* orow = reinterpret_cast<uint16_t*>(a.out) + ((size_t)b * a.seq_q + srow) * (a.heads * hd) +
                                 h * hd + qcol;
#pragma unroll
                for (int jj = 0; jj < DV / 8; ++jj)
                    if (jj * 8 < hd)
                        *reinterpret_cast<uint32_t*>(orow + jj * 8) =
                            pack2(o[4 * jj + 2 * rh] * inv_l[rh], o[4 * jj + 2 * rh + 1] * inv_l[rh], BF16);
            }
        }
    }
}

// 9 warps: three share an SM sub-partition's 64 KB register file, hence at most 168 registers
template <int DC, int HD, int DK, int DV, int KV, int KVS, int BF16>
__global__ void __maxnreg__(168)  // kAttnThreads threads, one CTA per SM
attention_tc_kernel(const __grid_constant__ CUtensorMap tma_q,
                    const __grid_constant__ CUtensorMap tma_k,
                    const __grid_constant__ CUtensorMap tma_vt, const AttnArgs a) {
    attention_body<DC, HD, DK, DV, KV, KVS, BF16, false>(&tma_q, &tma_k, &tma_vt, a, nullptr, nullptr, IpArgs{});
}

template <int DC, int HD, int DK, int DV, int KV, int KVS, int BF16>
__global__ void __maxnreg__(168)
attention_ip_kernel(const __grid_constant__ CUtensorMap tma_q,
                    const __grid_constant__ CUtensorMap tma_k,
                    const __grid_constant__ CUtensorMap tma_vt, const AttnArgs a,
                    const __grid_constant__ CUtensorMap tma_k_ip,
                    const __grid_constant__ CUtensorMap tma_vt_ip, const IpArgs ip) {
    attention_body<DC, HD, DK, DV, KV, KVS, BF16, true>(&tma_q, &tma_k, &tma_vt, a, &tma_k_ip, &tma_vt_ip, ip);
}

template <int DC, int HD, int DK, int DV, int KV, int KVS, int BF16, bool IP>
static int launch_attention_t(const sfb_attn_params* p, const sfb_attn_ip_params* ipp, const AttnArgs& a,
                              cudaStream_t stream) {
    using L = AttnSmem<DC, DV, KV, KVS>;
    const char* what = IP ? "sfb_attention_ip" : "sfb_attention";
    static PerDeviceOnce attr_once;
    bool& attr_set = attr_once.flag();
    if (!attr_set) {
        cudaError_t err = IP ? cudaFuncSetAttribute(attention_ip_kernel<DC, HD, DK, DV, KV, KVS, BF16>,
                                                    cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal)
                             : cudaFuncSetAttribute(attention_tc_kernel<DC, HD, DK, DV, KV, KVS, BF16>,
                                                    cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal);
        if (err != cudaSuccess)
            return fail(SFB_ERR_CUDA, "%s: smem attribute: %s", what, cudaGetErrorString(err));
        attr_set = true;
    }
    CUtensorMap tq, tk, tv;
    memcpy(&tq, p->tmap_q, sizeof(CUtensorMap));
    memcpy(&tk, p->tmap_k, sizeof(CUtensorMap));
    memcpy(&tv, p->tmap_vt, sizeof(CUtensorMap));
    dim3 grid((p->seq_q + kTileQ - 1) / kTileQ, p->batch * p->heads);
    cudaError_t err;
    if constexpr (IP) {
        CUtensorMap tk_ip, tv_ip;
        memcpy(&tk_ip, ipp->tmap_k_ip, sizeof(CUtensorMap));
        memcpy(&tv_ip, ipp->tmap_vt_ip, sizeof(CUtensorMap));
        const IpArgs ip{ipp->seq_ip, ipp->k_ip_rows, ipp->ip_scale};
        err = launch_pdl(attention_ip_kernel<DC, HD, DK, DV, KV, KVS, BF16>, grid, dim3(kAttnThreads), L::kTotal,
                         stream, tq, tk, tv, a, tk_ip, tv_ip, ip);
    } else {
        err = launch_pdl(attention_tc_kernel<DC, HD, DK, DV, KV, KVS, BF16>, grid, dim3(kAttnThreads), L::kTotal,
                         stream, tq, tk, tv, a);
    }
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "%s: launch: %s", what, cudaGetErrorString(err));
    return check_launch(what);
}

template <int DC, int HD, int DK, int DV, int KV, int KVS, bool IP>
static int launch_attention(const sfb_attn_params* p, const sfb_attn_ip_params* ipp, const AttnArgs& a,
                            cudaStream_t stream) {
    return a.dtype == SFB_BF16 ? launch_attention_t<DC, HD, DK, DV, KV, KVS, 1, IP>(p, ipp, a, stream)
                               : launch_attention_t<DC, HD, DK, DV, KV, KVS, 0, IP>(p, ipp, a, stream);
}

// Argument checks and the (head_dim, kv_tile) dispatch both entry points share; `ipp` is non-null for the
// image-prompt variant only (checked by the caller).
template <bool IP>
static int attention_dispatch(const sfb_attn_params* p, const sfb_attn_ip_params* ipp, cudaStream_t stream) {
    const char* what = IP ? "sfb_attention_ip" : "sfb_attention";
    if (!p || !p->tmap_q || !p->tmap_k || !p->tmap_vt || !p->out)
        return fail(SFB_ERR_INVALID, "%s: null argument", what);
    if (p->head_dim % 8 || p->head_dim <= 0 || p->seq_q <= 0 || p->seq_kv <= 0)
        return fail(SFB_ERR_INVALID, "%s: bad geometry head_dim=%d seq_q=%d seq_kv=%d", what, p->head_dim, p->seq_q,
                    p->seq_kv);
    // V^T carries one extra all-ones row at index head_dim (softmax denominator on the tensor
    // core), so its row count is (head_dim + 1) rounded up to 16
    const int dv = (p->head_dim + 1 + 15) / 16 * 16;
    if (p->vt_rows != dv)
        return fail(SFB_ERR_INVALID, "%s: vt_rows=%d must be (head_dim+1) rounded to 16 (%d)", what, p->vt_rows, dv);
    AttnArgs a{};
    a.out = p->out; a.batch = p->batch; a.heads = p->heads; a.head_dim = p->head_dim;
    a.seq_q = p->seq_q; a.seq_kv = p->seq_kv; a.q_rows = p->q_rows; a.k_rows = p->k_rows;
    a.vt_rows = p->vt_rows; a.dtype = p->dtype;
    a.scale_log2 = p->scale * 1.4426950408889634f;
    a.causal = p->causal ? 1 : 0;
    if (a.causal && (p->kv_tile != 64 || p->seq_q != p->seq_kv))
        return fail(SFB_ERR_INVALID, "%s: causal needs kv_tile 64 and seq_q == seq_kv", what);
    if (p->kv_tile == 64) {  // v2: the caller built tmap_k with a 64-row box
        switch (p->head_dim) {
            case 32: return launch_attention<1, 32, 32, 48, 64, 4, IP>(p, ipp, a, stream);
            case 40: return launch_attention<1, 40, 48, 48, 64, 4, IP>(p, ipp, a, stream);
            case 64: return launch_attention<1, 64, 64, 80, 64, 3, IP>(p, ipp, a, stream);
            case 160: return launch_attention<3, 160, 160, 176, 64, 2, IP>(p, ipp, a, stream);
            default:
                return fail(SFB_ERR_INVALID, "%s: kv_tile 64 supports head_dim 32 / 40 / 64 / 160, not %d", what,
                            p->head_dim);
        }
    }
    if (p->kv_tile != 0 && p->kv_tile != 128) return fail(SFB_ERR_INVALID, "%s: kv_tile must be 0, 64 or 128", what);
    switch (p->head_dim) {
        case 32: return launch_attention<1, 32, 32, 48, 128, 2, IP>(p, ipp, a, stream);
        case 40: return launch_attention<1, 40, 48, 48, 128, 2, IP>(p, ipp, a, stream);
        case 64: return launch_attention<1, 64, 64, 80, 128, 2, IP>(p, ipp, a, stream);
        case 80: return launch_attention<2, 80, 80, 96, 128, 2, IP>(p, ipp, a, stream);
        case 128: return launch_attention<2, 128, 128, 144, 128, 1, IP>(p, ipp, a, stream);
        case 160: return launch_attention<3, 160, 160, 176, 128, 1, IP>(p, ipp, a, stream);
        default:
            return fail(SFB_ERR_INVALID, "%s: unsupported head_dim %d", what, p->head_dim);
    }
}

}  // namespace sfb

using namespace sfb;

extern "C" int sfb_attention(const sfb_attn_params* p, sfb_stream_t stream) {
    return attention_dispatch<false>(p, nullptr, static_cast<cudaStream_t>(stream));
}

extern "C" int sfb_attention_ip(const sfb_attn_ip_params* p, sfb_stream_t stream) {
    if (!p || !p->tmap_k_ip || !p->tmap_vt_ip || !p->ip_scale)
        return fail(SFB_ERR_INVALID, "sfb_attention_ip: null argument (tmap_k_ip / tmap_vt_ip / ip_scale)");
    const int kv = p->base.kv_tile == 64 ? 64 : 128;
    if (p->seq_ip <= 0 || p->seq_ip > kv)
        return fail(SFB_ERR_INVALID, "sfb_attention_ip: seq_ip=%d must be in 1..kv_tile (%d): the image tokens are "
                    "one KV tile", p->seq_ip, kv);
    if (p->k_ip_rows < p->seq_ip)
        return fail(SFB_ERR_INVALID, "sfb_attention_ip: k_ip_rows=%d < seq_ip=%d", p->k_ip_rows, p->seq_ip);
    if (p->base.causal) return fail(SFB_ERR_INVALID, "sfb_attention_ip: causal is not supported");
    return attention_dispatch<true>(&p->base, p, static_cast<cudaStream_t>(stream));
}
