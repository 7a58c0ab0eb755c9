// Self-attention across frames on the tensor cores: the attention of AnimateDiff's motion modules
// (diffusers UNetMotionModel, AnimateDiffTransformer3D / TransformerTemporalModel).
//
// For every (video b, pixel p, head h) the F <= 32 frame tokens of head_dim D in {40, 80, 160} attend to
// each other.  The fused QKV projection is read in the spatial row order m = (b * F + f) * S + p -- the
// diffusers permute to [B * S, F, C] is only an index map here, as in sfb_temporal_attention.
//
//   * One warp owns one (pixel, head) sequence at a time.  It stages q, k and v of its F frames in shared
//     memory (16-byte loads; the fp32 frame bias -- the motion modules' sinusoidal position embedding
//     projected by W_q / W_k / W_v at pack time -- is added on the way and the sum rounded once), then
//     computes S = q k^T and O = P v with mma.sync m16n8k16 (fp32 accumulation): one or two m16 query
//     tiles hold all frames; the keys are n8 tiles of S and k16 steps of P v.
//   * head_dim 40 is zero-padded to 48 for the k16 steps of q k^T (the padding columns are zeroed once and
//     never written).  Rows past F are zero keys (masked to -inf) and zero values.
//   * The softmax is fp32 in registers: a row lives in the four lanes of one quad.  P is repacked to 16 bits
//     as the A operand of P v straight from the S accumulators (the C fragment of two n8 tiles is the A
//     fragment of one k16 step), normalised by the fp32 row sum at the end.
//   * A CTA of four warps owns a run of consecutive pixels of one video and every head of them, so the rows
//     it reads are contiguous and each is read in whole by neighbouring warps.  The work is a few MFLOP
//     per KB read: the kernel is bound by the bandwidth of the q / k / v reads and the output writes.
//
// wgmma is the wrong shape here: its m64 tile would be 2 to 4 times the sequence.
#include "common.cuh"
#include "host.h"

namespace sfb {

constexpr int kFaWarps = 4;
constexpr int kFaMaxF = 32;

struct FrameAttnArgs {
    const uint16_t* qkv;  // [B * F * S, ldq]: q | k | v, head h at columns h * D of each block
    const float* bias;    // [F, ldb] fp32 (q | k | v columns like qkv) or null
    uint16_t* out;        // [B * F * S, ldo]
    int frames, seq, heads, ldq, ldb, ldo;
    int tiles;            // pixel runs per video
    int ppc;              // pixels per CTA
    float scale_log2;     // scale * log2(e)
};

__device__ __forceinline__ void fa_ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(addr));
}
__device__ __forceinline__ void fa_ldsm_x4_t(uint32_t addr, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(addr));
}

template <int BF16>
__device__ __forceinline__ void fa_mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
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

// shared memory row pitch (halves) of one staged q / k / v row: K extent padded to 16, plus 8 halves so that
// the eight 16-byte rows of an ldmatrix land in distinct banks
template <int D>
struct FaGeom {
    static constexpr int Dp = (D + 15) / 16 * 16;
    static constexpr int P = Dp + 8;
};

template <int D, int FP>
constexpr int fa_smem_bytes() {
    return kFaWarps * 3 * FP * FaGeom<D>::P * 2;
}

template <int D, int FP, int BF16>
__global__ void __launch_bounds__(kFaWarps * 32) frame_attention_kernel(const FrameAttnArgs a) {
    constexpr int Dp = FaGeom<D>::Dp, P = FaGeom<D>::P;
    constexpr int kChunks = D / 8;       // 16-byte chunks per row and operand
    constexpr int KT = FP / 8;           // key n8 tiles of S
    constexpr int NP = (D / 8 + 1) / 2;  // pairs of n8 value tiles of O (D = 40: the sixth tile is padding)
    constexpr int kU = 4;                // staging loads in flight per lane
    extern __shared__ __align__(16) uint16_t fa_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint16_t* sQ = fa_smem + warp * 3 * FP * P;
    uint16_t* sK = sQ + FP * P;
    uint16_t* sV = sK + FP * P;
    // zero once: rows >= F and (D = 40) columns 40..47 are never written again
    for (int i = lane; i < 3 * FP * P / 8; i += 32) reinterpret_cast<uint4*>(sQ)[i] = make_uint4(0, 0, 0, 0);
    pdl_launch_dependents();
    pdl_wait();
    const int F = a.frames, C = a.heads * D;
    const int b = blockIdx.x / a.tiles, p0 = (blockIdx.x - b * a.tiles) * a.ppc;
    const int npix = min(a.ppc, a.seq - p0);
    const int g = lane >> 2, cq = lane & 3;
    const uint32_t q_base = static_cast<uint32_t>(__cvta_generic_to_shared(sQ));
    const uint32_t k_base = q_base + FP * P * 2, v_base = k_base + FP * P * 2;
    for (int item = warp; item < npix * a.heads; item += kFaWarps) {
        const int p = p0 + item / a.heads, h = item - (item / a.heads) * a.heads;
        const size_t row0 = (size_t)b * F * a.seq + p;  // row of frame 0; frames are S rows apart
        // ---- stage q, k, v (+ frame bias): i = (frame, operand, chunk)
        const int total = F * 3 * kChunks;
        for (int i0 = 0; i0 < total; i0 += 32 * kU) {
            uint4 v[kU];
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                const int i = i0 + u * 32 + lane;
                if (i < total) {
                    const int f = i / (3 * kChunks), r = i - f * 3 * kChunks;
                    const int op = r / kChunks, c = r - op * kChunks;
                    v[u] = __ldg(reinterpret_cast<const uint4*>(a.qkv + (row0 + (size_t)f * a.seq) * a.ldq +
                                                                op * C + h * D + c * 8));
                }
            }
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                const int i = i0 + u * 32 + lane;
                if (i < total) {
                    const int f = i / (3 * kChunks), r = i - f * 3 * kChunks;
                    const int op = r / kChunks, c = r - op * kChunks;
                    uint4 w = v[u];
                    if (a.bias) {
                        const float4* bp = reinterpret_cast<const float4*>(a.bias + (size_t)f * a.ldb + op * C +
                                                                           h * D + c * 8);
                        const float4 b0 = __ldg(bp), b1 = __ldg(bp + 1);
                        float2 x0 = unpack2(w.x, BF16), x1 = unpack2(w.y, BF16), x2 = unpack2(w.z, BF16),
                               x3 = unpack2(w.w, BF16);
                        w = make_uint4(pack2(x0.x + b0.x, x0.y + b0.y, BF16), pack2(x1.x + b0.z, x1.y + b0.w, BF16),
                                       pack2(x2.x + b1.x, x2.y + b1.y, BF16), pack2(x3.x + b1.z, x3.y + b1.w, BF16));
                    }
                    *reinterpret_cast<uint4*>(sQ + (op * FP + f) * P + c * 8) = w;
                }
            }
        }
        __syncwarp();
#pragma unroll
        for (int mt = 0; mt < FP / 16; ++mt) {
            // ---- S = q k^T for query rows mt*16 .. +15
            float s[KT][4];
#pragma unroll
            for (int j = 0; j < KT; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
            for (int ks = 0; ks < Dp / 16; ++ks) {
                uint32_t qa[4];
                fa_ldsm_x4(q_base + ((mt * 16 + (lane & 15)) * P + ks * 16 + (lane >> 4) * 8) * 2, qa);
#pragma unroll
                for (int j = 0; j < KT; j += 2) {
                    // two key tiles: matrices (j, k lo), (j, k hi), (j + 1, k lo), (j + 1, k hi)
                    const int mi = lane >> 3;
                    uint32_t kb[4];
                    fa_ldsm_x4(k_base + (((j + (mi >> 1)) * 8 + (lane & 7)) * P + ks * 16 + (mi & 1) * 8) * 2, kb);
                    fa_mma<BF16>(s[j], qa, kb[0], kb[1]);
                    fa_mma<BF16>(s[j + 1], qa, kb[2], kb[3]);
                }
            }
            // ---- softmax over the keys (rows g and g + 8 of the tile; a row is spread over one quad)
            float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
            for (int j = 0; j < KT; ++j) {
                const int key = j * 8 + 2 * cq;
                if (key >= F) s[j][0] = s[j][2] = -INFINITY;
                if (key + 1 >= F) s[j][1] = s[j][3] = -INFINITY;
                m0 = fmaxf(m0, fmaxf(s[j][0], s[j][1]));
                m1 = fmaxf(m1, fmaxf(s[j][2], s[j][3]));
            }
#pragma unroll
            for (int o = 1; o <= 2; o <<= 1) {
                m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, o));
                m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, o));
            }
            const float mo0 = m0 * a.scale_log2, mo1 = m1 * a.scale_log2;
            float l0 = 0.f, l1 = 0.f;
#pragma unroll
            for (int j = 0; j < KT; ++j) {
                s[j][0] = exp2f(fmaf(s[j][0], a.scale_log2, -mo0));
                s[j][1] = exp2f(fmaf(s[j][1], a.scale_log2, -mo0));
                s[j][2] = exp2f(fmaf(s[j][2], a.scale_log2, -mo1));
                s[j][3] = exp2f(fmaf(s[j][3], a.scale_log2, -mo1));
                l0 += s[j][0] + s[j][1];
                l1 += s[j][2] + s[j][3];
            }
#pragma unroll
            for (int o = 1; o <= 2; o <<= 1) {
                l0 += __shfl_xor_sync(0xffffffffu, l0, o);
                l1 += __shfl_xor_sync(0xffffffffu, l1, o);
            }
            // ---- O = P v: P (16 bits) from the S fragments, v^T fragments by transposing ldmatrix
            float o[2 * NP][4];
#pragma unroll
            for (int n = 0; n < 2 * NP; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
#pragma unroll
            for (int kk = 0; kk < FP / 16; ++kk) {
                const uint32_t pa[4] = {pack2(s[2 * kk][0], s[2 * kk][1], BF16), pack2(s[2 * kk][2], s[2 * kk][3], BF16),
                                        pack2(s[2 * kk + 1][0], s[2 * kk + 1][1], BF16),
                                        pack2(s[2 * kk + 1][2], s[2 * kk + 1][3], BF16)};
#pragma unroll
                for (int n = 0; n < NP; ++n) {
                    // matrices (keys lo, d tile 2n), (keys hi, 2n), (keys lo, 2n + 1), (keys hi, 2n + 1)
                    const int mi = lane >> 3;
                    uint32_t vb[4];
                    fa_ldsm_x4_t(v_base + ((kk * 16 + (mi & 1) * 8 + (lane & 7)) * P + (2 * n + (mi >> 1)) * 8) * 2,
                                 vb);
                    fa_mma<BF16>(o[2 * n], pa, vb[0], vb[1]);
                    fa_mma<BF16>(o[2 * n + 1], pa, vb[2], vb[3]);
                }
            }
            // ---- normalise; this tile's output rows replace its (consumed) q rows in shared memory
            __syncwarp();
            const float i0 = 1.0f / l0, i1 = 1.0f / l1;
            const int r0 = mt * 16 + g, r1 = r0 + 8;
#pragma unroll
            for (int n = 0; n < D / 8; ++n) {
                if (r0 < F)
                    *reinterpret_cast<uint32_t*>(sQ + r0 * P + n * 8 + 2 * cq) = pack2(o[n][0] * i0, o[n][1] * i0, BF16);
                if (r1 < F)
                    *reinterpret_cast<uint32_t*>(sQ + r1 * P + n * 8 + 2 * cq) = pack2(o[n][2] * i1, o[n][3] * i1, BF16);
            }
        }
        __syncwarp();
        // ---- write the F output rows of this head (16-byte stores)
        uint16_t* dst = a.out + row0 * a.ldo + h * D;
        for (int i = lane; i < F * kChunks; i += 32) {
            const int f = i / kChunks, c = i - f * kChunks;
            *reinterpret_cast<uint4*>(dst + (size_t)f * a.seq * a.ldo + c * 8) =
                *reinterpret_cast<const uint4*>(sQ + f * P + c * 8);
        }
        __syncwarp();  // the next item's staging overwrites sQ
    }
}

template <int D, int FP, int BF16>
static int launch_frame_attention(const FrameAttnArgs& a, int blocks, cudaStream_t stream) {
    constexpr int smem = fa_smem_bytes<D, FP>();
    static PerDeviceOnce attr_once;
    bool& attr_set = attr_once.flag();
    if (!attr_set) {
        const cudaError_t err = cudaFuncSetAttribute(frame_attention_kernel<D, FP, BF16>,
                                                     cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "frame_attention: smem attribute: %s", cudaGetErrorString(err));
        attr_set = true;
    }
    const cudaError_t err = launch_pdl(frame_attention_kernel<D, FP, BF16>, dim3((unsigned)blocks), dim3(kFaWarps * 32),
                                       smem, stream, a);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "frame_attention: %s", cudaGetErrorString(err));
    return check_launch("sfb_frame_attention");
}

template <int D, int BF16>
static int launch_frame_attention_d(const FrameAttnArgs& a, int blocks, cudaStream_t stream) {
    return a.frames <= 16 ? launch_frame_attention<D, 16, BF16>(a, blocks, stream)
                          : launch_frame_attention<D, 32, BF16>(a, blocks, stream);
}

}  // namespace sfb

using namespace sfb;

extern "C" int sfb_frame_attention(const sfb_frame_attn_params* p, sfb_stream_t stream) {
    if (!p || !p->qkv || !p->out) return fail(SFB_ERR_INVALID, "frame_attention: null argument");
    if ((reinterpret_cast<uintptr_t>(p->qkv) | reinterpret_cast<uintptr_t>(p->out) |
         reinterpret_cast<uintptr_t>(p->frame_bias)) & 15)
        return fail(SFB_ERR_INVALID, "frame_attention: qkv, out and frame_bias must be 16-byte aligned");
    if (p->frames <= 0 || p->frames > kFaMaxF)
        return fail(SFB_ERR_INVALID, "frame_attention: frames=%d (supported: 1 to 32)", p->frames);
    if (p->head_dim != 40 && p->head_dim != 80 && p->head_dim != 160)
        return fail(SFB_ERR_INVALID, "frame_attention: head_dim=%d (supported: 40, 80, 160)", p->head_dim);
    if (p->dtype != SFB_F16 && p->dtype != SFB_BF16)
        return fail(SFB_ERR_INVALID, "frame_attention: dtype %d (supported: fp16, bf16)", p->dtype);
    if (p->batch <= 0 || p->seq <= 0 || p->heads <= 0 || !(p->scale > 0.f))
        return fail(SFB_ERR_INVALID, "frame_attention: batch=%d seq=%d heads=%d scale=%g must be positive", p->batch,
                    p->seq, p->heads, (double)p->scale);
    const long long C = (long long)p->heads * p->head_dim;
    if (p->ld_qkv % 8 || p->ld_out % 8 || p->ld_qkv < 3 * C || p->ld_out < C)
        return fail(SFB_ERR_INVALID, "frame_attention: ld_qkv=%d ld_out=%d must be multiples of 8 with ld_qkv >= %lld "
                    "and ld_out >= %lld", p->ld_qkv, p->ld_out, 3 * C, C);
    if (p->frame_bias && (p->ld_bias % 4 || p->ld_bias < 3 * C))
        return fail(SFB_ERR_INVALID, "frame_attention: ld_bias=%d must be a multiple of 4 and >= %lld", p->ld_bias,
                    3 * C);
    if ((long long)p->batch * p->frames * p->seq > 0x7fffffffLL)
        return fail(SFB_ERR_INVALID, "frame_attention: batch * frames * seq must be < 2^31");
    // pixels per CTA: up to 4, fewer where that leaves the SMs short of CTAs
    const long long pixels = (long long)p->batch * p->seq;
    long long ppc = pixels / (2LL * sm_count());
    ppc = ppc < 1 ? 1 : (ppc > 4 ? 4 : ppc);
    const long long tiles = (p->seq + ppc - 1) / ppc;
    const long long blocks = (long long)p->batch * tiles;
    if (blocks > 0x7fffffffLL) return fail(SFB_ERR_INVALID, "frame_attention: too many pixels");
    FrameAttnArgs a{reinterpret_cast<const uint16_t*>(p->qkv), p->frame_bias, reinterpret_cast<uint16_t*>(p->out),
                    p->frames, p->seq, p->heads, p->ld_qkv, p->ld_bias, p->ld_out, (int)tiles, (int)ppc,
                    p->scale * 1.4426950408889634f};
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int bf = p->dtype == SFB_BF16;
    switch (p->head_dim) {
        case 40: return bf ? launch_frame_attention_d<40, 1>(a, (int)blocks, s) : launch_frame_attention_d<40, 0>(a, (int)blocks, s);
        case 80: return bf ? launch_frame_attention_d<80, 1>(a, (int)blocks, s) : launch_frame_attention_d<80, 0>(a, (int)blocks, s);
        default: return bf ? launch_frame_attention_d<160, 1>(a, (int)blocks, s) : launch_frame_attention_d<160, 0>(a, (int)blocks, s);
    }
}
