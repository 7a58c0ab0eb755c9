// wgmma GEMM / implicit-GEMM 3x3 convolution for sm_90a.
//
//   D[M, N] = A[M, K] * W[N, K]^T   (fp16/bf16 operands, fp32 accumulation in registers)
//
// gemm_tc_kernel: one 128 x 160 tile per CTA, used for every launch (split-K for the
// weight-bandwidth-bound low-resolution layers).  The cta_pair / persistent launch flags of the C ABI
// only describe the caller's weight tensor map (80-row box), which the kernel loads as two boxes.
//
// Warp roles (288 threads):
//   warps 0..7  two consumer warpgroups: wgmma.m64n160k16 on rows [64 g, 64 g + 64) of the tile, then
//               the epilogue: accumulator fragments -> fp32 staging tile in the idle stage buffers ->
//               fuse bias / time-embedding row bias / LayerNorm fold / residual / GEGLU / QKV head
//               scatter, 16-byte stores;
//   warp 8      TMA producer: A tile (128 rows x 64 K) + W tile per stage, 128-byte-swizzled K-major
//               shared memory.
// For the convolution the A tile of filter tap (kh, kw) is a *shifted NHWC box*: the tile's
// 128 output pixels are a [box_n, box_h, box_w] block, so one 4-D TMA box load at
// (c, w0+kw-1, h0*stride+kh-1, n0) is exactly the im2col slice, and TMA's out-of-bounds zero fill
// is the convolution's zero padding.  No im2col buffer, no index tables.
//
// SFB_A_CONV3X3_GN (template parameter HALO) folds the GroupNorm(+SiLU) in front of a 3x3 conv into this
// kernel's operand path: ONE raw halo tile per 64-channel block by TMA, normalised + activated once per
// element by the consumer warps into three column-shifted swizzled copies,
// nine taps = shifted views of those copies (see GemmSmem and DESIGN.md section 4.2).  It replaces the
// reference's separate sfast_triton::group_norm_silu launch (/root/reference/src/sfast/jit/passes/
// triton_passes.py:68-88, src/sfast/triton/ops/group_norm.py:272-320) in front of the conv.
//
// Replaces: cudnn_convolution_bias(_add) (/root/reference/src/sfast/csrc/operators/cudnn/
// cudnn_convolution_impl.cc:890-987), cublas_lowp_linear(_add) (csrc/operators/cublas/
// cublas_gemm.cpp:798-853,900-948) and cutlass_linear_geglu (csrc/operators/cutlass/
// cutlass_dual_linear_kernel.cu:442-525).
#include "common.cuh"
#include "host.h"

#include <stdlib.h>
#include <string.h>

namespace sfb {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int BN = 160;
// two consumer warpgroups (MMA + epilogue) and one TMA producer warp
constexpr int kConsumerWGs = 2;
constexpr int kEpiWarps = 4 * kConsumerWGs;
constexpr int kEpiThreads = kEpiWarps * 32;
constexpr int kColSplit = 2;  // epilogue phase A: two threads per tile row, half of the columns each
constexpr int kGemmThreads = kEpiThreads + 32;
constexpr int kGemmStages = 6;
__device__ __forceinline__ void epi_bar() {
    asm volatile("bar.sync 1, %0;" ::"n"(kEpiThreads) : "memory");
}

struct EpiArgs {
    int epi;
    int dtype;
    int M, N;
    void* out;
    int ldo;
    const float* bias;
    const float* rowbias;
    int rows_per_img;
    int ld_rowbias;
    const void* residual;
    int ldr;
    int geglu_n_out;
    void* q;
    void* k;
    void* vt;
    int heads, head_dim, which_base, seq, q_pitch, q_rows, k_rows, vt_rows, vt_pitch;
    // LayerNorm folded around the GEMM (see sfb200.h): producer side / consumer side
    float* rowstats_out;
    const float* ln_rowstats;
    const float* ln_colsum;
    float ln_eps;
    int ln_dim;
    int act;  // SFB_ACT_*: STORE epilogue only
    // Row statistics live in SLOTS: [M][slots] x (sum, sum of squares).  Every producer writes each of
    // its slots exactly once (GEMM epilogue: slot = its 160-column tile; split-K reduction: slot = warp
    // segment of the row), nothing is accumulated atomically, and the consumer adds the slots in index
    // order -- bit-identical from run to run.  Unwritten slots are zero (the caller clears the buffer).
    int rs_slots;  // slots per row of rowstats_out
    int ln_slots;  // slots per row of ln_rowstats
};

// quick_gelu (x * sigmoid(1.702 x)) / erf gelu of the CLIP text encoders' MLP; SiLU of the ControlNet's
// conditioning-embedding convs; ReLU of the T2I-Adapter's 3x3 convs
__device__ __forceinline__ float epi_act(float x, int act) {
    if (act == SFB_ACT_QUICK_GELU) return __fdividef(x, 1.0f + __expf(-1.702f * x));
    if (act == SFB_ACT_SILU) return silu_f(x);
    if (act == SFB_ACT_RELU) return fmaxf(x, 0.f);
    return gelu_erf_f(x);
}

// LayerNorm(x) W^T == rstd * (x W'^T - mean * colsum(W')) + (beta W^T + b), W' = W * gamma.
// (mean, rstd) of row m from the (sum, sum of squares) its producer GEMMs accumulated.
__device__ __forceinline__ float2 ln_row_params(const EpiArgs& e, int m) {
    const float2* sp = reinterpret_cast<const float2*>(e.ln_rowstats) + (size_t)m * e.ln_slots;
    float2 st = __ldcg(sp);
    for (int i = 1; i < e.ln_slots; ++i) {
        const float2 t = __ldcg(sp + i);
        st.x += t.x; st.y += t.y;
    }
    const float inv = 1.0f / (float)e.ln_dim;
    const float mean = st.x * inv;
    const float var = fmaxf(st.y * inv - mean * mean, 0.f);
    return make_float2(mean, rsqrtf(var + e.ln_eps));
}

struct GemmArgs {
    int a_mode;
    int nkb_total;  // K / 64
    int splits;
    float* ws;
    // conv geometry
    int img_n, img_h, img_w, cpb /* cin / 64 */, conv_stride, box_h, box_n, tiles_per_img;
    int box_w, tiles_per_row;  // M tile = [box_n, box_h, box_w] pixels; box_w < img_w: 2-D patches
    int up_tiles;   // SFB_A_UPCONV2X: M tiles per output phase
    int up_ntiles;  // ... and N tiles per phase in the phase-concatenated weight matrix
    int b_plain;    // B is a plain row-major [N, K] matrix (an activation), not a pre-tiled weight
    int b_half;     // tmap_b has the 80-row box (cta_pair / persistent callers): two loads per B tile
    int m_tile_base;  // M tile of blockIdx.y == 0: more M tiles than a grid's y extent run as several launches
    // SFB_A_CONV3X3_GN: per-(image, channel) GroupNorm (scale, shift) pairs [img_n][cin][2], SiLU flag
    const float* gn_ab;
    int gn_silu;
    EpiArgs e;
#ifdef SFB_TRACE
    unsigned long long* trace;  // [ctas][16] %globaltimer stamps (latency anatomy builds only)
#endif
};

// Latency-anatomy instrumentation: compiled only into the -DSFB_TRACE measurement build
// (tests/gemm_latency.py); the product library carries none of it.
#ifdef SFB_TRACE
__device__ __forceinline__ void trace_stamp(const GemmArgs& a, int slot) {
    if (a.trace) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        const int cta = blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z);
        a.trace[(size_t)cta * 16 + slot] = t;
    }
}
#define SFB_STAMP(slot) trace_stamp(args, slot)
#else
#define SFB_STAMP(slot) ((void)0)
#endif

// ---------------------------------------------------------------------------------------
// epilogue building blocks (shared by both GEMM kernels and the split-K reduction kernel)
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void add_bias8(const float* __restrict__ b, int n, float (&acc)[8]) {
    const float4 b0 = *reinterpret_cast<const float4*>(b + n);
    const float4 b1 = *reinterpret_cast<const float4*>(b + n + 4);
    acc[0] += b0.x; acc[1] += b0.y; acc[2] += b0.z; acc[3] += b0.w;
    acc[4] += b1.x; acc[5] += b1.y; acc[6] += b1.z; acc[7] += b1.w;
}

__device__ __forceinline__ uint4 pack8(const float (&acc)[8], int bf16) {
    uint4 o;
    o.x = pack2(acc[0], acc[1], bf16);
    o.y = pack2(acc[2], acc[3], bf16);
    o.z = pack2(acc[4], acc[5], bf16);
    o.w = pack2(acc[6], acc[7], bf16);
    return o;
}

__device__ __forceinline__ void add_res8(uint4 r, int dtype, float (&acc)[8]) {
    float2 f;
    f = unpack2(r.x, dtype); acc[0] += f.x; acc[1] += f.y;
    f = unpack2(r.y, dtype); acc[2] += f.x; acc[3] += f.y;
    f = unpack2(r.z, dtype); acc[4] += f.x; acc[5] += f.y;
    f = unpack2(r.w, dtype); acc[6] += f.x; acc[7] += f.y;
}

// (sum, sum of squares) of 8 values as they will be stored (rounded to the 16-bit type)
__device__ __forceinline__ void row_stats8(const float (&acc)[8], int dtype, float& s, float& ss) {
    const uint4 p = pack8(acc, dtype);
    const uint32_t w[4] = {p.x, p.y, p.z, p.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 f = unpack2(w[i], dtype);
        s += f.x + f.y;
        ss += f.x * f.x + f.y * f.y;
    }
}

// 8 consecutive output columns [n, n+8) of row m; `acc` already holds bias / row bias / residual.
template <int BF16>
__device__ __forceinline__ void epi_store8(const EpiArgs& e, int m, int n, const float (&acc)[8]) {
    if (e.epi == SFB_EPI_STORE) {
        *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(e.out) + (size_t)m * e.ldo + n) =
            pack8(acc, BF16);
    } else {  // SFB_EPI_QKV
        const int C = e.heads * e.head_dim;
        const int which = n / C + e.which_base;
        const int nn = n % C;
        const int h = nn / e.head_dim;
        const int d = nn % e.head_dim;
        const int b = m / e.seq;
        const int s = m % e.seq;
        const size_t bh = (size_t)b * e.heads + h;
        if (which == 0) {
            *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(e.q) +
                                      (bh * e.q_rows + s) * e.q_pitch + d) = pack8(acc, BF16);
        } else if (which == 1) {
            *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(e.k) +
                                      (bh * e.k_rows + s) * e.q_pitch + d) = pack8(acc, BF16);
        } else {
#pragma unroll
            for (int i = 0; i < 8; ++i)
                store1(e.vt, (bh * e.vt_rows + d + i) * e.vt_pitch + s, acc[i], BF16);
        }
    }
}

// GEGLU: value / gate (bias already added) of 8 output columns [nout, nout+8)
template <int BF16>
__device__ __forceinline__ void epi_geglu8(const EpiArgs& e, int m, int nout, const float (&v)[8],
                                           const float (&g)[8]) {
    float o[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = v[i] * gelu_erf_f(g[i]);
    *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(e.out) + (size_t)m * e.ldo + nout) =
        pack8(o, BF16);
}

// origin (image, row, column) of conv M-tile `tile` (already reduced to one up-conv phase)
__device__ __forceinline__ void conv_tile_origin(const GemmArgs& a, int tile, int& n0, int& h0, int& w0) {
    if (a.box_n == 1) {
        n0 = tile / a.tiles_per_img;
        const int rem = tile - n0 * a.tiles_per_img;
        const int trow = rem / a.tiles_per_row;
        h0 = trow * a.box_h;
        w0 = (rem - trow * a.tiles_per_row) * a.box_w;
    } else {
        n0 = tile * a.box_n;
        h0 = 0;
        w0 = 0;
    }
}

// tile-local row r (0..127) of M-tile `tile` -> global row m; false if the row is padding
__device__ __forceinline__ bool tile_row_to_m(const GemmArgs& a, int tile, int r, int& m) {
    if (a.a_mode == SFB_A_MATRIX) {
        m = tile * BM + r;
        return m < a.e.M;
    }
    int phase = 0;
    if (a.a_mode == SFB_A_UPCONV2X) {
        phase = tile / a.up_tiles;
        tile -= phase * a.up_tiles;
    }
    int n0, h0, w0;
    conv_tile_origin(a, tile, n0, h0, w0);
    const int w = w0 + r % a.box_w;
    const int t = r / a.box_w;
    const int dh = t % a.box_h;
    const int dn = t / a.box_h;
    const int n = n0 + dn, h = h0 + dh;
    if (a.a_mode == SFB_A_UPCONV2X)  // source pixel (h, w) -> output pixel (2h + py, 2w + px)
        m = (n * 2 * a.img_h + 2 * h + (phase >> 1)) * 2 * a.img_w + 2 * w + (phase & 1);
    else
        m = (n * a.img_h + h) * a.img_w + w;
    return (n < a.img_n) && (h < a.img_h);
}

// A-operand TMA coordinates of M-tile `m_tile`: conv tile origin, up-conv phase, weight row block
struct ATile {
    int n0, h0, w0, up_py, up_px, b_nbase;  // b_nbase: first 160-row weight tile of the phase
};
__device__ __forceinline__ ATile a_tile_coords(const GemmArgs& a, int m_tile) {
    ATile t{0, 0, 0, 0, 0, 0};
    if (a.a_mode != SFB_A_MATRIX) {
        int mt = m_tile;
        if (a.a_mode == SFB_A_UPCONV2X) {
            const int ph = m_tile / a.up_tiles;
            mt = m_tile - ph * a.up_tiles;
            t.up_py = ph >> 1; t.up_px = ph & 1;
            t.b_nbase = ph * a.up_ntiles;
        }
        conv_tile_origin(a, mt, t.n0, t.h0, t.w0);
    }
    return t;
}
// conv tap of K block -> (w, h) source offset of the A box
__device__ __forceinline__ void tap_offset(const GemmArgs& a, const ATile& t, int tap, int& dw, int& dh) {
    if (a.a_mode == SFB_A_UPCONV2X) {  // 2x2 taps of phase (py, px) sit at (py - 1 + ty, px - 1 + tx)
        const int ty = tap >> 1, tx = tap & 1;
        dw = t.up_px - 1 + tx;
        dh = t.up_py - 1 + ty;
    } else if (a.a_mode == SFB_A_CONV3X1) {  // temporal conv: taps along the frame (h) axis only
        dw = 0;
        dh = tap - 1;
    } else {
        // SFB_A_DOWNCONV3X3 pads only after the last row / column: its taps start at the pixel itself
        const int org = a.a_mode == SFB_A_DOWNCONV3X3 ? 0 : 1;
        const int kh = tap / 3, kw = tap - kh * 3;
        dw = kw - org;
        dh = kh - org;
    }
}

// ---------------------------------------------------------------------------------------
// split-K reduction + epilogue
// ---------------------------------------------------------------------------------------
// Sum the `splits` fp32 partials of 8 output columns of row m and run the fused epilogue on them.
// `n` is the output column (GEGLU: output column of the gated product).  Partials were written by
// other SMs: read them through L2 (ld.global.cg).
template <int BF16, typename Sum8>
__device__ __forceinline__ void reduce_epilogue8(Sum8&& sum8, const EpiArgs& e, int m, int n, float& rs, float& rss) {
    if (e.epi == SFB_EPI_GEGLU) {
        const int tile = n / (BN / 2);
        const int nv = tile * BN + (n - tile * (BN / 2));
        const int ng = nv + BN / 2;
        float v[8], g[8];
        sum8(nv, v);
        sum8(ng, g);
        if (e.ln_rowstats) {
            const float2 ln = ln_row_params(e, m);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                v[i] = ln.y * (v[i] - ln.x * e.ln_colsum[nv + i]);
                g[i] = ln.y * (g[i] - ln.x * e.ln_colsum[ng + i]);
            }
        }
        if (e.bias) {
            add_bias8(e.bias, nv, v);
            add_bias8(e.bias, ng, g);
        }
        epi_geglu8<BF16>(e, m, n, v, g);
    } else {
        float acc[8];
        sum8(n, acc);
        if (e.ln_rowstats) {
            const float2 ln = ln_row_params(e, m);
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[i] = ln.y * (acc[i] - ln.x * e.ln_colsum[n + i]);
        }
        if (e.bias) add_bias8(e.bias, n, acc);
        if (e.epi == SFB_EPI_STORE) {
            if (e.rowbias) add_bias8(e.rowbias + (size_t)(m / e.rows_per_img) * e.ld_rowbias, n, acc);
            if (e.residual)
                add_res8(*reinterpret_cast<const uint4*>(
                             reinterpret_cast<const uint16_t*>(e.residual) + (size_t)m * e.ldr + n),
                         BF16, acc);
        }
        if (e.rowstats_out) row_stats8(acc, BF16, rs, rss);
        epi_store8<BF16>(e, m, n, acc);
    }
}

// Stand-alone split-K reduction kernel.  One thread per (row, 8 columns); convs that feed a
// GroupNorm skip it (defer_finish) and let that kernel sum the partials.
template <int BF16>
__global__ void __launch_bounds__(256)
splitk_finish_kernel(const float* __restrict__ ws, int splits, const EpiArgs e) {
    pdl_launch_dependents();
    pdl_wait();
    const int ncols = (e.epi == SFB_EPI_GEGLU) ? e.geglu_n_out : e.N;
    const int groups = ncols / 8;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = idx < (long long)e.M * groups;
    if (!live && !e.rowstats_out) return;
    const int m = live ? (int)(idx / groups) : -1, n = live ? (int)(idx % groups) * 8 : 0;
    float rs = 0.f, rss = 0.f;  // (sum, sum of squares) of this thread's 8 stored values (rowstats_out)
    if (live) {
    auto sum8 = [&](int col, float (&acc)[8]) {
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = 0.f;
        // batches of 6 partials with every load in flight before the first add: this kernel is
        // one L2 round trip per batch, not per partial
        constexpr int kU = 6;
        const float* p0 = ws + (size_t)m * e.N + col;
        const size_t stride = (size_t)e.M * e.N;
        for (int s0 = 0; s0 < splits; s0 += kU) {
            float4 a[kU], b[kU];
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                if (s0 + u < splits) {
                    const float* p = p0 + (size_t)(s0 + u) * stride;
                    a[u] = __ldcg(reinterpret_cast<const float4*>(p));
                    b[u] = __ldcg(reinterpret_cast<const float4*>(p + 4));
                }
            }
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                if (s0 + u < splits) {
                    acc[0] += a[u].x; acc[1] += a[u].y; acc[2] += a[u].z; acc[3] += a[u].w;
                    acc[4] += b[u].x; acc[5] += b[u].y; acc[6] += b[u].z; acc[7] += b[u].w;
                }
            }
        }
    };
    reduce_epilogue8<BF16>(sum8, e, m, n, rs, rss);
    }
    if (e.rowstats_out) {
        // (the whole warp gets here: out-of-range threads carry m = -1)  Segmented sum over the lanes that
        // hold the same row, fixed shuffle tree; the segment's first lane writes slot = how many warp
        // boundaries lie between the row's first column group and this segment.
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const float o1 = __shfl_down_sync(0xffffffffu, rs, d), o2 = __shfl_down_sync(0xffffffffu, rss, d);
            const int om = __shfl_down_sync(0xffffffffu, m, d);
            if ((int)(threadIdx.x & 31) + d < 32 && om == m) { rs += o1; rss += o2; }
        }
        const int pm = __shfl_up_sync(0xffffffffu, m, 1);
        const bool head = live && ((threadIdx.x & 31) == 0 || pm != m);
        if (head) {
            const long long row_start = (long long)m * groups;
            const int seg = (int)((idx - row_start + 31) / 32);
            float* d = e.rowstats_out + ((size_t)m * e.rs_slots + seg) * 2;
            d[0] = rs; d[1] = rss;
        }
    }
}

// ---------------------------------------------------------------------------------------
// one-tile-per-CTA kernel
// ---------------------------------------------------------------------------------------
// One CTA per 128 x 160 tile.  Warps 0..7 are two consumer warpgroups: warpgroup g multiplies rows
// [64 g, 64 g + 64) of the tile with wgmma.m64n160k16 (accumulator in registers, 80 fp32 per thread) and
// then runs the epilogue together with the other warpgroup; warp 8 is the TMA producer.
// HALO = 1 (SFB_A_CONV3X3_GN): the A operand is not staged tap by tap.  Per 64-channel block ONE
// raw [18 x 10] pixel halo tile of the 16 x 8 pixel output patch lands by TMA; the consumer warps
// apply GroupNorm scale / shift + SiLU to every halo element ONCE and write it into three
// column-shifted copies (dx = 0, 1, 2), each [18 halo rows][8 columns] x 128 B in the
// 128-byte-swizzled K-major layout: one halo row = one 8-row swizzle atom (1024 B), so the A tile
// of tap (dy, dx) is simply copy dx advanced by dy atoms -- every wgmma descriptor stays 1024-byte
// aligned.  The nine taps of a channel block re-read that copy from shared memory instead of
// pulling nine shifted boxes through L2.
template <int STAGES, int HALO = 0>
struct GemmSmem {
    static constexpr int kABytes = HALO ? 0 : BM * BK * 2;
    static constexpr int kBBytes = BN * BK * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kHaloRows = 18, kHaloCols = 10;
    static constexpr int kHaloABuf = kHaloRows * 1024;                    // one shifted copy
    static constexpr int kHaloRawBytes = kHaloRows * kHaloCols * 128;     // the TMA box
    static constexpr int kHaloRawAlloc = (kHaloRawBytes + 1023) / 1024 * 1024;
    static constexpr int kHaloBytes = HALO ? 3 * kHaloABuf + kHaloRawAlloc : 0;
    static constexpr int kBarOffset = kHaloBytes + STAGES * kStageBytes;
    static constexpr int kBiasOffset = kBarOffset + 256;              // fp32 [kBiasSlots][BN]
    // images per conv M-tile whose row bias is staged
    static constexpr int kBiasSlots = HALO ? 2 : 4;
    static constexpr int kRowMOffset = kBiasOffset + kBiasSlots * BN * 4;  // int [128]: row -> m
    static constexpr int kTotal = kRowMOffset + BM * 4 + 1024;                // + alignment slack
    // fp32 staging tile of the epilogue, aliased onto the (by then idle) pipeline stages; the
    // +4 float pad makes the thread-per-row float4 accesses of phase A bank-conflict free
    static constexpr int kStagePitch = BN + 4;
    // QKV scatter tables (row -> (batch, position), column slice -> (q/k/v, offset)), also aliased
    // onto the idle stage buffers
    static constexpr int kQkvRowOffset = BM * kStagePitch * 4;
    static constexpr int kQkvColOffset = kQkvRowOffset + BM * 8;
    static_assert(kQkvColOffset + (BN / 8) * 16 <= kBarOffset,
                  "staging tile + QKV tables must fit in the stage buffers");
    static_assert(kTotal <= 227 * 1024, "shared memory per block");
};

// GroupNorm affine + SiLU of two conv-input elements -> one packed 16-bit pair.
// x * sigmoid(x) = h + h * tanh(h), h = x / 2: ONE MUFU per element (the exp + rcp form is two).
// fp16: the SiLU runs on the packed pair (HMUL2 / 2 x MUFU.TANH.F16 / HFMA2, error ~2^-11 like the
// storage type).  bf16: three more 8-bit roundings in front of the conv would show (SDXL 128^2:
// 4.1e-2 vs 3.7e-2 whole-UNet error), so the SiLU stays in fp32 and is rounded once.
template <int BF16>
__device__ __forceinline__ uint32_t gn_act_pair(float y0, float y1, int silu) {
    if (BF16) {
        if (silu) {
            float t0, t1;
            const float h0 = 0.5f * y0, h1 = 0.5f * y1;
            asm("tanh.approx.f32 %0, %1;" : "=f"(t0) : "f"(h0));
            asm("tanh.approx.f32 %0, %1;" : "=f"(t1) : "f"(h1));
            y0 = fmaf(h0, t0, h0);
            y1 = fmaf(h1, t1, h1);
        }
        return pack2(y0, y1, 1);
    }
    const uint32_t x = pack2(y0, y1, 0);
    if (!silu) return x;
    uint32_t h, t, o;
    asm("mul.f16x2 %0, %1, %2;" : "=r"(h) : "r"(x), "r"(0x38003800u));
    asm("tanh.approx.f16x2 %0, %1;" : "=r"(t) : "r"(h));
    asm("fma.rn.f16x2 %0, %1, %2, %1;" : "=r"(o) : "r"(h), "r"(t));
    return o;
}

template <int STAGES, int BF16, int HALO = 0>
// 9 warps: three share an SM sub-partition's 64 KB register file, hence at most 168 registers
__global__ void __maxnreg__(168)  // kGemmThreads threads, one CTA per SM
gemm_tc_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
               const GemmArgs args) {
    using L = GemmSmem<STAGES, HALO>;
    static_assert(!HALO || STAGES <= 4, "halo conv: shallow weight ring");
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024 - (smem_u32(smem_raw) & 1023)) & 1023);
    uint8_t* sA = smem;                                   // HALO: the three shifted copies
    uint8_t* sRaw = smem + 3 * L::kHaloABuf;              // HALO: raw halo tile (TMA destination)
    uint8_t* sB = smem + L::kHaloBytes + STAGES * L::kABytes;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::kBarOffset);
    uint64_t* empty_bar = full_bar + STAGES;
    // HALO: raw tile landed / consumed
    uint64_t* raw_full = empty_bar + STAGES;
    uint64_t* raw_empty = raw_full + 1;
    float* sBias = reinterpret_cast<float*>(smem + L::kBiasOffset);
    int* sRowM = reinterpret_cast<int*>(smem + L::kRowMOffset);
    float* sStage = reinterpret_cast<float*>(smem);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int n_tile = blockIdx.x;
    const int m_tile = args.m_tile_base + blockIdx.y;
    const int split = blockIdx.z;
    const int kb_begin = (int)(((long long)args.nkb_total * split) / args.splits);
    const int kb_end = (int)(((long long)args.nkb_total * (split + 1)) / args.splits);
    const int nkb = kb_end - kb_begin;

    if (threadIdx.x == 0) {
        SFB_STAMP(0);
        tma_prefetch_desc(&tma_a);
        tma_prefetch_desc(&tma_b);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], kConsumerWGs);  // one arrival per consumer warpgroup
        }
        if (HALO) {
            mbar_init(raw_full, 1);
            mbar_init(raw_empty, kEpiWarps);
        }
        fence_barrier_init();
    }
    // Everything up to each role's pdl_wait() overlaps the previous kernel's tail (programmatic
    // dependent launch); global memory produced by it is only touched after that wait.
    pdl_launch_dependents();
    __syncthreads();
    if (threadIdx.x == 0) SFB_STAMP(1);

    if (warp == kEpiWarps) {
        if (lane == 0) {
            const ATile at = a_tile_coords(args, m_tile);
            // one 160-row weight tile: a single box, or two 80-row boxes when the caller built tmap_b
            // with the half-height box (cta_pair)
            auto load_b_tile = [&](uint8_t* dB, uint64_t* bar, int b_col, int b_row) {
                tma_load_2d(dB, &tma_b, bar, b_col, b_row);
                if (args.b_half) tma_load_2d(dB + (BN / 2) * 128, &tma_b, bar, b_col, b_row + BN / 2);
            };
            if (HALO) {
                // ---- halo conv producer: per 64-channel block cb ONE raw halo tile, and the nine weight
                // tiles (tap, cb) of the block through the STAGES-deep ring
                const int ncb = args.cpb, total = ncb * 9;
                auto load_w = [&](int i) {
                    // taps run copy-major (dx, dy): the three taps of one shifted copy are consecutive
                    const int cb = i / 9, t = i - cb * 9;
                    const int dx = t / 3, dy = t - dx * 3;
                    const int kb = (dy * 3 + dx) * ncb + cb;  // weight K order is (kh, kw, cin)
                    const int stage = i % STAGES;
                    mbar_expect_tx(&full_bar[stage], L::kBBytes);
                    load_b_tile(sB + stage * L::kBBytes, &full_bar[stage], 0, (n_tile * args.nkb_total + kb) * BN);
                };
                auto load_raw = [&](int cb) {
                    mbar_expect_tx(raw_full, L::kHaloRawBytes);
                    // box [64 ch][10 w][18 h][1 n] at the patch origin minus the one-pixel border:
                    // out-of-image pixels arrive as zeros (and are re-zeroed after the transform)
                    tma_load_4d(sRaw, &tma_a, raw_full, cb * BK, at.w0 - 1, at.h0 - 1, at.n0);
                };
                const int npre = min(total, STAGES);
                for (int i = 0; i < npre; ++i) load_w(i);  // weights never depend on the predecessor
                pdl_wait();
                SFB_STAMP(2);
                load_raw(0);
                for (int i = 0; i < total; ++i) {
                    const int cb = i / 9, tap = i - cb * 9;
                    if (tap == 3 && cb + 1 < ncb) {
                        // the transform of block cb has read the raw tile (it ran before this block's
                        // first MMA): fetch the next one while the taps of this block are multiplied
                        mbar_wait(raw_empty, cb & 1);
                        load_raw(cb + 1);
                    }
                    if (i >= npre) {
                        mbar_wait(&empty_bar[i % STAGES], ((i / STAGES) & 1) ^ 1);
                        load_w(i);
                    }
                }
            } else {
                const int b_ntile = at.b_nbase + n_tile;
                auto load_b = [&](int i) {
                    const int stage = i % STAGES;
                    const int kb = kb_begin + i;
                    // weights are pre-tiled in HBM: tile (n_tile, kb) is one contiguous 160 x 64 block
                    int b_col = 0, b_row = (b_ntile * args.nkb_total + kb) * BN;
                    if (args.b_plain) { b_col = kb * BK; b_row = b_ntile * BN; }
                    mbar_expect_tx(&full_bar[stage], L::kStageBytes);
                    load_b_tile(sB + stage * L::kBBytes, &full_bar[stage], b_col, b_row);
                };
                // Pre-tiled weights never depend on the predecessor kernel: the first pipeline fill of
                // W tiles is in flight before the programmatic-dependent-launch wait releases the
                // activation loads.  (b_plain: B is an activation -> nothing is loaded early.)
                const int npre = args.b_plain ? 0 : min(nkb, STAGES);
                for (int i = 0; i < npre; ++i) load_b(i);
                pdl_wait();
                SFB_STAMP(2);
                for (int i = 0; i < nkb; ++i) {
                    const int stage = i % STAGES;
                    const uint32_t phase = (i / STAGES) & 1;
                    if (i >= npre) {
                        mbar_wait(&empty_bar[stage], phase ^ 1);
                        load_b(i);
                    }
                    const int kb = kb_begin + i;
                    uint8_t* dA = sA + stage * L::kABytes;
                    if (args.a_mode == SFB_A_MATRIX) {
                        tma_load_2d(dA, &tma_a, &full_bar[stage], kb * BK, m_tile * BM);
                    } else {
                        const int tap = kb / args.cpb;
                        int dw, dh;
                        tap_offset(args, at, tap, dw, dh);
                        tma_load_4d(dA, &tma_a, &full_bar[stage], (kb - tap * args.cpb) * BK,
                                    at.w0 * args.conv_stride + dw, at.h0 * args.conv_stride + dh, at.n0);
                    }
                }
            }
        }
    } else {
        pdl_wait();
        const int et = threadIdx.x;          // index among the consumer threads
        const int wg = et >> 7;              // consumer warpgroup: tile rows [64 wg, 64 wg + 64)
        const int r = et & (BM - 1);         // epilogue phase A: the tile row this thread finishes
        const int chalf = et >> 7;           // ... and which half of the tile's columns
        int m;
        const bool valid = tile_row_to_m(args, m_tile, r, m);
        sRowM[r] = valid ? m : -1;
        if (args.splits == 1) {
            // stage bias (+ per-image time-embedding row bias) for this tile's columns in smem;
            // only the consumer warps take part (named barrier 1), the TMA warp is already streaming
            const EpiArgs& e = args.e;
            int img0 = 0, nslots = 1;
            const bool rb_staged = e.rowbias && args.box_n <= L::kBiasSlots;
            if (rb_staged) {
                nslots = args.box_n;
                img0 = (args.box_n == 1) ? (m_tile / args.tiles_per_img) : m_tile * args.box_n;
            }
            for (int i = et; i < nslots * BN; i += kEpiThreads) {
                const int slot = i / BN, c = i - slot * BN;
                const int n = n_tile * BN + c;
                float v = 0.f;
                if (n < e.N) {
                    if (e.bias) v = e.bias[n];
                    if (rb_staged && img0 + slot < args.img_n)
                        v += e.rowbias[(size_t)(img0 + slot) * e.ld_rowbias + n];
                }
                sBias[i] = v;
            }
            if (e.ln_rowstats) {  // slot 1: column sums of the gamma-scaled weight
                for (int c = et; c < BN; c += kEpiThreads) {
                    const int n = n_tile * BN + c;
                    sBias[BN + c] = (n < e.N) ? e.ln_colsum[n] : 0.f;
                }
            }
        }

        // ---- main loop: this warpgroup's 64 x 160 accumulator in registers
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        // K block i: wait for its weight (and A) tile, issue 4 x K=16, and release the stage of K block
        // i - 1 once the group before this one has completed (one group stays in flight)
        auto mma_block = [&](int i, uint64_t da) {
            const int stage = i % STAGES;
            mbar_wait(&full_bar[stage], (i / STAGES) & 1);
            if (i == 0 && et == 0) SFB_STAMP(3);
            const uint64_t db = wgmma_desc_k_sw128(smem_u32(sB + stage * L::kBBytes));
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) wgmma_ss<BF16>(acc, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2));
            wgmma_commit();
            wgmma_wait<1>(acc);
            if (i > 0 && (et & 127) == 0) mbar_arrive(&empty_bar[(i - 1) % STAGES]);
        };
        if (HALO) {
            // ---- GroupNorm(+SiLU) transform of the conv's A operand.  Thread = (16-byte channel chunk c,
            // halo pixels p0 + 32 i): a warp reads / writes four consecutive 128-byte rows per
            // instruction -- conflict-free.
            const int c = et & 7;
            const int p0 = et >> 3;
            const ATile at = a_tile_coords(args, m_tile);
            const int cin = args.cpb * BK;
            constexpr int kPix = (L::kHaloRows * L::kHaloCols + 31) / 32;  // 6 halo pixels per thread
            uint32_t roff[kPix], dbase[kPix], meta[kPix];
#pragma unroll
            for (int i = 0; i < kPix; ++i) {
                const int p = p0 + 32 * i;
                const bool live = p < L::kHaloRows * L::kHaloCols;
                const int hy = p / L::kHaloCols, hx = p - hy * L::kHaloCols;
                const int gy = at.h0 - 1 + hy, gx = at.w0 - 1 + hx;
                const bool inside = live && gy >= 0 && gy < args.img_h && gx >= 0 && gx < args.img_w;
                roff[i] = (uint32_t)(p * 128 + ((c ^ (p & 7)) << 4));   // TMA's 128-byte swizzle
                dbase[i] = (uint32_t)(hy * 1024);
                meta[i] = (uint32_t)hx | (inside ? 16u : 0u) | (live ? 32u : 0u);
            }
            float sc[8], sh[8];
            auto load_ab = [&](int cb) {
                const float4* q = reinterpret_cast<const float4*>(
                    args.gn_ab + 2 * ((size_t)at.n0 * cin + cb * BK + c * 8));
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float4 t = q[j];
                    sc[2 * j] = t.x; sh[2 * j] = t.y; sc[2 * j + 1] = t.z; sh[2 * j + 1] = t.w;
                }
            };
            load_ab(0);
            int i = 0;
            for (int cb = 0; cb < args.cpb; ++cb) {
                mbar_wait(raw_full, cb & 1);
                uint4 v[kPix];
#pragma unroll
                for (int q = 0; q < kPix; ++q)
                    if (meta[q] & 32u) v[q] = *reinterpret_cast<const uint4*>(sRaw + roff[q]);
#pragma unroll
                for (int q = 0; q < kPix; ++q) {
                    uint32_t w[4] = {v[q].x, v[q].y, v[q].z, v[q].w};
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float2 f = unpack2(w[j], BF16);
                        w[j] = gn_act_pair<BF16>(fmaf(f.x, sc[2 * j], sh[2 * j]), fmaf(f.y, sc[2 * j + 1], sh[2 * j + 1]),
                                                 args.gn_silu);
                    }
                    // padding pixels must be zero AFTER the transform: silu(0 * scale + shift) != 0
                    v[q] = (meta[q] & 16u) ? make_uint4(w[0], w[1], w[2], w[3]) : make_uint4(0, 0, 0, 0);
                }
                // the raw tile is consumed (its values sit in registers): release it for the next block
                __syncwarp();
                if (lane == 0) mbar_arrive(raw_empty);
                // the copies of the previous block may be overwritten once both warpgroups' MMAs on them
                // have completed
                wgmma_wait<0>(acc);
                epi_bar();
#pragma unroll
                for (int dx = 0; dx < 3; ++dx) {
#pragma unroll
                    for (int q = 0; q < kPix; ++q) {
                        const int x = (int)(meta[q] & 15) - dx;  // column inside the shifted copy
                        if ((meta[q] & 32u) && x >= 0 && x < 8)
                            *reinterpret_cast<uint4*>(sA + dx * L::kHaloABuf + dbase[q] + x * 128 + ((c ^ x) << 4)) = v[q];
                    }
                }
                fence_proxy_async_smem();  // generic-proxy stores -> visible to the tensor core's reads
                epi_bar();
                // next block's (scale, shift): in flight during this block's MMAs
                if (cb + 1 < args.cpb) load_ab(cb + 1);
                for (int dx = 0; dx < 3; ++dx)
                    for (int dy = 0; dy < 3; ++dy, ++i)  // tap (dy, dx): copy dx advanced by dy halo rows
                        mma_block(i, wgmma_desc_k_sw128(smem_u32(sA + dx * L::kHaloABuf + (dy + 8 * wg) * 1024)));
            }
        } else {
            for (int i = 0; i < nkb; ++i)
                mma_block(i, wgmma_desc_k_sw128(smem_u32(sA + (i % STAGES) * L::kABytes + wg * 64 * 128)));
        }
        wgmma_wait<0>(acc);
        if (et == 0) SFB_STAMP(4);
        // every stage has been read by both warpgroups (and the producer has nothing in flight): the
        // stage buffers become the fp32 staging tile
        epi_bar();
        {
            // accumulator fragment: d[4 j + {0,1}] = (row lane / 4, columns 8 j + 2 (lane % 4) + {0,1}) of
            // the warp's 16 rows, d[4 j + {2,3}] = the same columns 8 rows further down
            const int row0 = wg * 64 + ((et >> 5) & 3) * 16 + (lane >> 2);
            float* s0 = sStage + row0 * L::kStagePitch + 2 * (lane & 3);
            float* s1 = s0 + 8 * L::kStagePitch;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                *reinterpret_cast<float2*>(s0 + 8 * j) = make_float2(acc[4 * j], acc[4 * j + 1]);
                *reinterpret_cast<float2*>(s1 + 8 * j) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
            }
        }
        epi_bar();

        // ---- epilogue.  Phase A: thread = tile row: staged accumulator -> (+bias / LayerNorm fold) ->
        // back to the fp32 staging tile.  Phase B: threads re-partition the tile so that every global
        // access (residual load, output store) is a coalesced 16-byte slice of a row segment
        // instead of 32 rows x 16 bytes per warp instruction.
        const EpiArgs& e = args.e;
        const int ncol0 = n_tile * BN;
        const bool partial = args.splits > 1;
        constexpr int kGroups = BN / 8;  // 16-byte output slices per row
        constexpr int kItems = BM * kGroups / kEpiThreads;  // slices per epilogue thread
        // Residual in the coalesced phase-B ownership (thread <-> 16-byte slice), software-pipelined
        // in batches of 5 slices; the first batch is issued before the accumulator is even ready.
        // (Loops here are deliberately ROLLED: the epilogue runs once per CTA, so straight-line
        // unrolled code is all instruction-cache misses -- an earlier build measured 5 us per tile.)
        const bool has_res = (e.residual != nullptr) && (e.epi == SFB_EPI_STORE) && !partial;
        constexpr int kBatch = 5;
        auto item_addr = [&](int it, int& row, int& grp, int& mm, int& n) {
            const int idx = et + it * kEpiThreads;
            row = idx / kGroups;
            grp = idx - row * kGroups;
            mm = sRowM[row];
            n = ncol0 + grp * 8;
        };
        auto load_res = [&](int it) -> uint4 {
            int row, grp, mm, n;
            item_addr(it, row, grp, mm, n);
            return (mm >= 0 && n < e.N)
                ? *reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(e.residual) + (size_t)mm * e.ldr + n)
                : make_uint4(0, 0, 0, 0);
        };
        // LEAN path (plain STORE, the common case): phase B gives every thread ONE 4-column slice
        // (fixed n, fixed output / residual column pointers) and walks it down the rows -- no
        // per-item divisions, conflict-free 16-byte staging reads, 8-byte global accesses that
        // still cover whole 32-byte sectors per warp.
        const bool rb_staged0 = e.rowbias && args.box_n <= L::kBiasSlots;
        const bool lean = (e.epi == SFB_EPI_STORE) && !partial && !e.rowstats_out && !(e.rowbias && !rb_staged0);
        constexpr int kLSlices = BN / 4;                       // 16-byte fp32 slices per tile row
        constexpr int kLRows = kEpiThreads / kLSlices;         // rows covered per pass (6)
        constexpr int kLItems = (BM + kLRows - 1) / kLRows;    // 22
        // residual slices in flight per thread: ALL of them (issued before the accumulator is
        // ready) where one CTA owns the SM's registers, batches of 8 under the 2-CTAs/SM cap
        constexpr int kLBatch = STAGES > 4 ? kLItems : 8;
        constexpr int kLSub = STAGES > 4 ? 6 : 4;              // staging rows fetched ahead per step
        constexpr int kLBatches = (kLItems + kLBatch - 1) / kLBatch;
        const int lgrp = et % kLSlices, lrow0 = et / kLSlices;
        const int ln_col = ncol0 + lgrp * 4;
        const bool lactive = lean && lrow0 < kLRows && ln_col < e.N;
        const uint16_t* lres = reinterpret_cast<const uint16_t*>(e.residual) + ln_col;
        uint2 lcur[kLBatch], lnxt[kLBatch];
        auto lean_load = [&](int b, uint2 (&dst)[kLBatch]) {
#pragma unroll
            for (int j = 0; j < kLBatch; ++j) {
                const int row = lrow0 + (b * kLBatch + j) * kLRows;
                const int mm = row < BM ? sRowM[row] : -1;
                dst[j] = mm >= 0 ? *reinterpret_cast<const uint2*>(lres + (size_t)mm * e.ldr) : make_uint2(0, 0);
            }
        };
        uint4 rcur[kBatch], rnxt[kBatch];
        if (has_res && !lean) {
#pragma unroll
            for (int j = 0; j < kBatch; ++j) rcur[j] = load_res(j);
        }
        if (has_res && lactive) lean_load(0, lcur);
        float2 ln = make_float2(0.f, 1.f);
        if (e.ln_rowstats && valid && !partial) ln = ln_row_params(e, m);
        const float* brow = sBias;
        const bool rb_staged = e.rowbias && args.box_n <= L::kBiasSlots;
        if (rb_staged) brow += (r / (args.box_h * args.img_w)) * BN;
        // many tiny images per tile (4x4 feature maps): row bias straight from global memory
        const float* rb_global = nullptr;
        if (e.rowbias && !rb_staged && !partial)
            rb_global = e.rowbias + (size_t)min(m_tile * args.box_n + r / (args.box_h * args.img_w), args.img_n - 1) * e.ld_rowbias;  // (padding rows of the last tile: clamped, never stored)

        if (et == 0) SFB_STAMP(5);
        // QKV scatter: the integer divisions of the address computation once per row / per column
        // slice (tables in the now idle stage buffers) instead of five per stored 16-byte slice
        int2* sQkvRow = reinterpret_cast<int2*>(smem + L::kQkvRowOffset);
        longlong2* sQkvCol = reinterpret_cast<longlong2*>(smem + L::kQkvColOffset);
        if (args.e.epi == SFB_EPI_QKV && !partial) {
            const EpiArgs& q = args.e;
            if (chalf == 0) sQkvRow[r] = valid ? make_int2(m / q.seq, m % q.seq) : make_int2(0, 0);
            if (et < BN / 8) {
                const int n = ncol0 + et * 8;
                const int C = q.heads * q.head_dim;
                const int which = n / C + q.which_base;
                const int nn = n % C;
                const int h = nn / q.head_dim, d = nn % q.head_dim;
                long long off;
                if (which == 0) off = (long long)h * q.q_rows * q.q_pitch + d;
                else if (which == 1) off = (long long)h * q.k_rows * q.q_pitch + d;
                else off = ((long long)h * q.vt_rows + d) * q.vt_pitch;
                sQkvCol[et] = make_longlong2(which, off);
            }
        }
        float* srow = sStage + r * L::kStagePitch;
        constexpr int kColsPer = BN / kColSplit;             // columns finished per thread
        const bool has_ln = e.ln_rowstats != nullptr;
#pragma unroll 1
        for (int cl = chalf * kColsPer; cl < (chalf + 1) * kColsPer; cl += 8) {
            float f[8];
            const float4 v0 = *reinterpret_cast<const float4*>(srow + cl);
            const float4 v1 = *reinterpret_cast<const float4*>(srow + cl + 4);
            f[0] = v0.x; f[1] = v0.y; f[2] = v0.z; f[3] = v0.w; f[4] = v1.x; f[5] = v1.y; f[6] = v1.z; f[7] = v1.w;
            if (!partial) {
                if (has_ln) {
                    const float4 s0 = *reinterpret_cast<const float4*>(sBias + BN + cl);
                    const float4 s1 = *reinterpret_cast<const float4*>(sBias + BN + cl + 4);
                    f[0] = ln.y * (f[0] - ln.x * s0.x); f[1] = ln.y * (f[1] - ln.x * s0.y);
                    f[2] = ln.y * (f[2] - ln.x * s0.z); f[3] = ln.y * (f[3] - ln.x * s0.w);
                    f[4] = ln.y * (f[4] - ln.x * s1.x); f[5] = ln.y * (f[5] - ln.x * s1.y);
                    f[6] = ln.y * (f[6] - ln.x * s1.z); f[7] = ln.y * (f[7] - ln.x * s1.w);
                }
                add_bias8(brow, cl, f);
            }
            if (rb_global && ncol0 + cl < e.N) add_bias8(rb_global, ncol0 + cl, f);
            *reinterpret_cast<float4*>(srow + cl) = make_float4(f[0], f[1], f[2], f[3]);
            *reinterpret_cast<float4*>(srow + cl + 4) = make_float4(f[4], f[5], f[6], f[7]);
        }
        if (e.act) {
            // activation (CLIP MLP): a ROLLED second pass over this thread's own staged values -- kept
            // out of the unrolled conversion above, whose straight-line code every launch pays for
            // in instruction fetch whether it has an activation or not
#pragma unroll 1
            for (int c = 0; c < kColsPer; c += 4) {
                float4 v = *reinterpret_cast<float4*>(srow + chalf * kColsPer + c);
                v.x = epi_act(v.x, e.act); v.y = epi_act(v.y, e.act);
                v.z = epi_act(v.z, e.act); v.w = epi_act(v.w, e.act);
                *reinterpret_cast<float4*>(srow + chalf * kColsPer + c) = v;
            }
        }
        epi_bar();
        if (et == 0) SFB_STAMP(6);

        // ---- phase B
        auto load8 = [&](int row, int col, float (&f)[8]) {
            const float4 a = *reinterpret_cast<const float4*>(sStage + row * L::kStagePitch + col);
            const float4 b = *reinterpret_cast<const float4*>(sStage + row * L::kStagePitch + col + 4);
            f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
        };
        if (lean) {
            if (lactive) {
                uint16_t* lout = reinterpret_cast<uint16_t*>(e.out) + ln_col;
                const float* lst = sStage + lgrp * 4;
#pragma unroll 1
                for (int b = 0; b < kLBatches; ++b) {
                    if (has_res && b + 1 < kLBatches) lean_load(b + 1, lnxt);
#pragma unroll
                    for (int j0 = 0; j0 < kLBatch; j0 += kLSub) {
                        // loads of kLSub rows first (row -> m, staged fp32 slice), then the math /
                        // stores: two epilogue warps per scheduler cannot hide a dependent
                        // LDS -> LDS -> STG chain per row
                        int mmv[kLSub];
                        float4 fv[kLSub];
#pragma unroll
                        for (int u = 0; u < kLSub; ++u) {
                            if (j0 + u < kLBatch) {
                                const int row = lrow0 + (b * kLBatch + j0 + u) * kLRows;
                                const int rr = min(row, BM - 1);
                                mmv[u] = row < BM ? sRowM[rr] : -1;
                                fv[u] = *reinterpret_cast<const float4*>(lst + rr * L::kStagePitch);
                            }
                        }
#pragma unroll
                        for (int u = 0; u < kLSub; ++u) {
                            if (j0 + u < kLBatch) {
                                if (mmv[u] >= 0) {
                                    float4 f = fv[u];
                                    if (has_res) {
                                        const float2 r0 = unpack2(lcur[j0 + u].x, BF16), r1 = unpack2(lcur[j0 + u].y, BF16);
                                        f.x += r0.x; f.y += r0.y; f.z += r1.x; f.w += r1.y;
                                    }
                                    *reinterpret_cast<uint2*>(lout + (size_t)mmv[u] * e.ldo) =
                                        make_uint2(pack2(f.x, f.y, BF16), pack2(f.z, f.w, BF16));
                                }
                            }
                        }
                    }
#pragma unroll
                    for (int j = 0; j < kLBatch; ++j) lcur[j] = lnxt[j];
                }
            }
        } else if (partial) {
#pragma unroll 1
            for (int it = 0; it < kItems; ++it) {
                const int idx = et + it * kEpiThreads;
                const int row = idx / kGroups, grp = idx - row * kGroups;
                const int mm = sRowM[row], n = ncol0 + grp * 8;
                if (mm >= 0 && n < e.N) {
                    float f[8];
                    load8(row, grp * 8, f);
                    float* dst = args.ws + ((size_t)split * e.M + mm) * e.N + n;
                    *reinterpret_cast<float4*>(dst) = make_float4(f[0], f[1], f[2], f[3]);
                    *reinterpret_cast<float4*>(dst + 4) = make_float4(f[4], f[5], f[6], f[7]);
                }
            }
        } else if (e.epi == SFB_EPI_STORE_F32) {
#pragma unroll 1
            for (int it = 0; it < kItems; ++it) {
                const int idx = et + it * kEpiThreads;
                const int row = idx / kGroups, grp = idx - row * kGroups;
                const int mm = sRowM[row], n = ncol0 + grp * 8;
                if (mm >= 0 && n < e.N) {
                    float f[8];
                    load8(row, grp * 8, f);
                    float* dst = reinterpret_cast<float*>(e.out) + (size_t)mm * e.ldo + n;
                    *reinterpret_cast<float4*>(dst) = make_float4(f[0], f[1], f[2], f[3]);
                    *reinterpret_cast<float4*>(dst + 4) = make_float4(f[4], f[5], f[6], f[7]);
                }
            }
        } else if (e.epi == SFB_EPI_GEGLU) {
#pragma unroll 1
            for (int it = 0; it < kItems / 2; ++it) {
                const int idx = et + it * kEpiThreads;
                const int row = idx / (kGroups / 2), og = idx - row * (kGroups / 2);
                const int mm = sRowM[row], nout = n_tile * (BN / 2) + og * 8;
                if (mm >= 0 && nout < e.geglu_n_out) {
                    float fv[8], fg[8];
                    load8(row, og * 8, fv);
                    load8(row, BN / 2 + og * 8, fg);
                    epi_geglu8<BF16>(e, mm, nout, fv, fg);
                }
            }
        } else {
            if (e.epi == SFB_EPI_STORE) {
#pragma unroll 1
                for (int b = 0; b < kItems / kBatch; ++b) {
                    if (has_res && b + 1 < kItems / kBatch) {
#pragma unroll
                        for (int j = 0; j < kBatch; ++j) rnxt[j] = load_res((b + 1) * kBatch + j);
                    }
#pragma unroll
                    for (int j = 0; j < kBatch; ++j) {
                        int row, grp, mm, n;
                        item_addr(b * kBatch + j, row, grp, mm, n);
                        if (mm >= 0 && n < e.N) {
                            float f[8];
                            load8(row, grp * 8, f);
                            if (has_res) add_res8(rcur[j], BF16, f);
                            if (e.rowstats_out) {  // final values back to the tile (row sums below)
                                float* d = sStage + row * L::kStagePitch + grp * 8;
                                *reinterpret_cast<float4*>(d) = make_float4(f[0], f[1], f[2], f[3]);
                                *reinterpret_cast<float4*>(d + 4) = make_float4(f[4], f[5], f[6], f[7]);
                            }
                            *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(e.out) + (size_t)mm * e.ldo + n) =
                                pack8(f, BF16);
                        }
                    }
#pragma unroll
                    for (int j = 0; j < kBatch; ++j) rcur[j] = rnxt[j];
                }
            } else {
                // QKV scatter.  V^T columns want consecutive lanes = consecutive rows (2-byte stores
                // along seq); Q / K want consecutive lanes = consecutive 16-byte slices of a row.
                const int C = e.heads * e.head_dim;
                const int n_last = min(ncol0 + BN, e.N) - 1;
                const bool row_fastest = (ncol0 / C + e.which_base == 2) && (n_last / C + e.which_base == 2);
#pragma unroll 1
                for (int it = 0; it < kItems; ++it) {
                    const int idx = et + it * kEpiThreads;
                    int row, grp;
                    if (row_fastest) { grp = idx >> 7; row = idx & 127; }
                    else { row = idx / kGroups; grp = idx - row * kGroups; }
                    const int mm = sRowM[row], n = ncol0 + grp * 8;
                    if (mm >= 0 && n < e.N) {
                        float f[8];
                        load8(row, grp * 8, f);
                        const int2 bs = sQkvRow[row];          // (batch, position)
                        const longlong2 ci = sQkvCol[grp];     // (q / k / v, column offset)
                        if (ci.x == 0) {
                            *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(e.q) +
                                ((size_t)bs.x * e.heads * e.q_rows + bs.y) * e.q_pitch + ci.y) = pack8(f, BF16);
                        } else if (ci.x == 1) {
                            *reinterpret_cast<uint4*>(reinterpret_cast<uint16_t*>(e.k) +
                                ((size_t)bs.x * e.heads * e.k_rows + bs.y) * e.q_pitch + ci.y) = pack8(f, BF16);
                        } else {
                            const size_t base = (size_t)bs.x * e.heads * e.vt_rows * e.vt_pitch + ci.y + bs.y;
#pragma unroll
                            for (int i = 0; i < 8; ++i) store1(e.vt, base + (size_t)i * e.vt_pitch, f[i], BF16);
                        }
                    }
                }
            }
            if (e.rowstats_out) {
                epi_bar();
                float2 rs_keep = make_float2(0.f, 0.f);
                if (valid) {
                    float rs_sum = 0.f, rs_sq = 0.f;
                    for (int g = chalf * (kGroups / kColSplit); g < (chalf + 1) * (kGroups / kColSplit); ++g) {
                        if (ncol0 + g * 8 < e.N) {
                            float f[8];
                            load8(r, g * 8, f);
                            row_stats8(f, BF16, rs_sum, rs_sq);
                        }
                    }
                    // the other column half of the same row sits in the partner warp: hand it over
                    // through shared memory (the bias slots are idle by now) and add in a fixed order
                    if (chalf == 1) *reinterpret_cast<float2*>(sBias + 2 * r) = make_float2(rs_sum, rs_sq);
                    rs_keep = make_float2(rs_sum, rs_sq);
                }
                epi_bar();
                if (valid && chalf == 0) {
                    float2 o = make_float2(0.f, 0.f);
                    if (kColSplit == 2) o = *reinterpret_cast<const float2*>(sBias + 2 * r);
                    float* d = e.rowstats_out + ((size_t)m * e.rs_slots + n_tile) * 2;
                    d[0] = rs_keep.x + o.x;
                    d[1] = rs_keep.y + o.y;
                }
            }
        }
    }

    if (threadIdx.x == 0) SFB_STAMP(7);
}

}  // namespace sfb

using namespace sfb;

template <int STAGES, int BF16, int HALO = 0>
static int launch_gemm_t(const CUtensorMap& ta, const CUtensorMap& tb, const GemmArgs& a, dim3 grid,
                         cudaStream_t stream) {
    using L = GemmSmem<STAGES, HALO>;
    static PerDeviceOnce attr_once;
    bool& attr_set = attr_once.flag();
    if (!attr_set) {
        cudaError_t err = cudaFuncSetAttribute(gemm_tc_kernel<STAGES, BF16, HALO>,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal);
        if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "sfb_gemm: smem attribute: %s", cudaGetErrorString(err));
        attr_set = true;
    }
    cudaError_t err = launch_pdl(gemm_tc_kernel<STAGES, BF16, HALO>, grid, dim3(kGemmThreads), L::kTotal, stream, ta, tb, a);
    if (err != cudaSuccess)
        return fail(SFB_ERR_CUDA, "sfb_gemm: launch: %s (%s) grid=(%u,%u,%u) smem=%d stages=%d",
                    cudaGetErrorString(err), cudaGetErrorName(err), grid.x, grid.y, grid.z, (int)L::kTotal, STAGES);
    return check_launch("sfb_gemm");
}

#ifdef SFB_TRACE
static thread_local unsigned long long* g_trace_next = nullptr;
// measurement build only: the NEXT sfb_gemm call writes its per-CTA stamps to `buf` ([ctas][16] u64)
extern "C" void sfb_trace_next_gemm(void* buf) { g_trace_next = static_cast<unsigned long long*>(buf); }
#endif

extern "C" int sfb_rowstats_slots(int32_t n_cols) {
    const int tiles = (n_cols + BN - 1) / BN;                 // one-tile kernel: a slot per 160-column tile
    const int segs = (n_cols / 8 - 1 + 31) / 32 + 1;          // split-K reduction: a slot per warp segment
    return tiles > segs ? tiles : segs;
}

extern "C" int sfb_gemm(const sfb_gemm_params* p, sfb_stream_t stream_) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    if (!p || !p->tmap_a || !p->tmap_b) return fail(SFB_ERR_INVALID, "sfb_gemm: null argument");
    if (p->K <= 0 || p->K % BK) return fail(SFB_ERR_INVALID, "sfb_gemm: K=%d must be a multiple of 64", p->K);
    if (p->N <= 0 || p->N % 8 || p->M <= 0) return fail(SFB_ERR_INVALID, "sfb_gemm: bad M=%d N=%d", p->M, p->N);
    if (p->dtype != SFB_F16 && p->dtype != SFB_BF16) return fail(SFB_ERR_INVALID, "sfb_gemm: dtype");
    GemmArgs a{};
    a.a_mode = p->a_mode;
    a.nkb_total = p->K / BK;
    a.splits = p->splits < 1 ? 1 : p->splits;
    if (a.splits > a.nkb_total) return fail(SFB_ERR_INVALID, "sfb_gemm: splits > K blocks");
    if (a.splits > 1 && !p->ws) return fail(SFB_ERR_INVALID, "sfb_gemm: split-K needs a workspace");
    a.ws = p->ws;
    a.b_plain = p->b_plain ? 1 : 0;
    if (a.b_plain && p->a_mode == SFB_A_UPCONV2X) return fail(SFB_ERR_INVALID, "sfb_gemm: b_plain with up-conv");
    int m_tiles;
    const bool upconv = p->a_mode == SFB_A_UPCONV2X;
    const bool tconv = p->a_mode == SFB_A_CONV3X1;
    const bool gnconv = p->a_mode == SFB_A_CONV3X3_GN;
    const bool downconv = p->a_mode == SFB_A_DOWNCONV3X3;
    if (downconv && (p->conv_stride != 2 || p->rowbias))
        return fail(SFB_ERR_INVALID, "sfb_gemm: SFB_A_DOWNCONV3X3 needs stride 2 and no rowbias (stride=%d)",
                    p->conv_stride);
    if (gnconv) {
        // 16 x 8 pixel patches, halo tile transformed in shared memory (tmap_a box = [64, 10, 18, 1])
        if (!p->gn_scale_shift) return fail(SFB_ERR_INVALID, "sfb_gemm: SFB_A_CONV3X3_GN needs gn_scale_shift");
        if (p->box_n != 1 || p->box_h != 16 || p->box_w != 8 || p->conv_stride != 1 ||
            a.splits != 1 || p->persistent || p->epi != SFB_EPI_STORE || p->b_plain)
            return fail(SFB_ERR_INVALID, "sfb_gemm: SFB_A_CONV3X3_GN needs the 1x16x8 box, stride 1, "
                                         "no split-K, the one-tile kernel and the STORE epilogue");
        a.gn_ab = p->gn_scale_shift;
        a.gn_silu = p->gn_silu ? 1 : 0;
    }
    if (p->a_mode == SFB_A_CONV3X3 || upconv || tconv || gnconv || downconv) {
        if (p->cin <= 0 || p->cin % BK || p->K != (upconv ? 4 : (tconv ? 3 : 9)) * p->cin)
            return fail(SFB_ERR_INVALID, "sfb_gemm: conv cin=%d K=%d", p->cin, p->K);
        const int box_w = p->box_w > 0 ? p->box_w : p->img_w;
        if (p->box_n * p->box_h * box_w != BM || box_w > p->img_w || p->img_w % box_w)
            return fail(SFB_ERR_INVALID, "sfb_gemm: conv M-tile box %dx%dx%d != 128 pixels / does not tile width %d",
                        p->box_n, p->box_h, box_w, p->img_w);
        if (p->box_n > 1 && (p->box_h != p->img_h || box_w != p->img_w))
            return fail(SFB_ERR_INVALID, "sfb_gemm: multi-image box needs box_h == img_h and box_w == img_w");
        if (p->M != (upconv ? 4 : 1) * p->img_n * p->img_h * p->img_w) return fail(SFB_ERR_INVALID, "sfb_gemm: conv M mismatch");
        if (upconv && (p->conv_stride != 1 || p->epi != SFB_EPI_STORE))
            return fail(SFB_ERR_INVALID, "sfb_gemm: up-conv needs stride 1 and the STORE epilogue");
        a.img_n = p->img_n; a.img_h = p->img_h; a.img_w = p->img_w;
        a.cpb = p->cin / BK;
        a.conv_stride = p->conv_stride;
        a.box_h = p->box_h; a.box_n = p->box_n; a.box_w = box_w;
        a.tiles_per_row = p->img_w / box_w;
        a.tiles_per_img = ((p->img_h + p->box_h - 1) / p->box_h) * a.tiles_per_row;
        m_tiles = (p->box_n == 1) ? p->img_n * a.tiles_per_img : (p->img_n + p->box_n - 1) / p->box_n;
        if (upconv) {  // 4 output phases, each its own set of M tiles and its own weight row block
            a.up_tiles = m_tiles;
            a.up_ntiles = (p->N + BN - 1) / BN;
            m_tiles *= 4;
        }
    } else if (p->a_mode == SFB_A_MATRIX) {
        m_tiles = (p->M + BM - 1) / BM;
    } else {
        return fail(SFB_ERR_INVALID, "sfb_gemm: a_mode");
    }
    if (p->rowbias && p->a_mode != SFB_A_CONV3X3 && !tconv && !gnconv)
        return fail(SFB_ERR_INVALID, "sfb_gemm: rowbias (time-embedding add) needs conv mode");
    // the epilogues read rows of 8 row-bias floats as two float4 loads (global memory when a tile spans more
    // images than the shared-memory bias slots hold, and in the split-K reduction)
    if (p->rowbias && ((reinterpret_cast<uintptr_t>(p->rowbias) & 15) || p->ld_rowbias % 4 || p->ld_rowbias < p->N))
        return fail(SFB_ERR_INVALID, "sfb_gemm: rowbias must be 16-byte aligned with ld_rowbias %% 4 == 0 and "
                                     ">= N (ld_rowbias=%d)", p->ld_rowbias);
    if (tconv && p->conv_stride != 1) return fail(SFB_ERR_INVALID, "sfb_gemm: temporal conv needs stride 1");
    EpiArgs& e = a.e;
    e.epi = p->epi; e.dtype = p->dtype; e.M = p->M; e.N = p->N;
    e.out = p->out; e.ldo = p->ldo; e.bias = p->bias; e.rowbias = p->rowbias;
    e.rows_per_img = p->rows_per_img > 0 ? p->rows_per_img : 1;
    e.ld_rowbias = p->ld_rowbias; e.residual = p->residual; e.ldr = p->ldr;
    e.q = p->q; e.k = p->k; e.vt = p->vt; e.heads = p->heads; e.head_dim = p->head_dim;
    e.which_base = p->which_base; e.seq = p->seq; e.q_pitch = p->q_pitch; e.q_rows = p->q_rows;
    e.k_rows = p->k_rows; e.vt_rows = p->vt_rows; e.vt_pitch = p->vt_pitch;
    e.rowstats_out = p->rowstats_out; e.ln_rowstats = p->ln_rowstats; e.ln_colsum = p->ln_colsum;
    e.ln_eps = p->ln_eps; e.ln_dim = p->ln_dim;
    e.act = p->act;
    e.rs_slots = p->rowstats_out_slots; e.ln_slots = p->ln_slots;
    if (p->rowstats_out) {
        // slots a producer may write: its 160-column tiles, or (split-K reduction kernel, one thread per 8
        // columns) the warp segments of a row
        int need = (p->N + BN - 1) / BN;
        if (p->splits > 1) need = (p->N / 8 - 1 + 31) / 32 + 1;
        if (p->rowstats_out_slots < need || p->persistent)
            return fail(SFB_ERR_INVALID, "sfb_gemm: rowstats_out needs rowstats_out_slots >= %d (got %d) and the one-tile kernel",
                        need, p->rowstats_out_slots);
    }
    if (p->ln_rowstats && p->ln_slots < 1) return fail(SFB_ERR_INVALID, "sfb_gemm: ln_rowstats needs ln_slots >= 1");
    if (p->act < SFB_ACT_NONE || p->act > SFB_ACT_RELU)
        return fail(SFB_ERR_INVALID, "sfb_gemm: unknown activation %d", p->act);
    if (p->act && (p->epi != SFB_EPI_STORE || p->splits > 1 || p->persistent || p->rowbias))
        return fail(SFB_ERR_INVALID, "sfb_gemm: act needs the STORE epilogue of the one-tile kernel without split-K / row bias");
    if (p->ln_rowstats && (!p->ln_colsum || p->ln_dim <= 0 || p->rowbias))
        return fail(SFB_ERR_INVALID, "sfb_gemm: LayerNorm fold needs ln_colsum / ln_dim and no rowbias");
    if (p->rowstats_out && p->epi != SFB_EPI_STORE)
        return fail(SFB_ERR_INVALID, "sfb_gemm: rowstats_out needs the STORE epilogue");
    if (p->epi == SFB_EPI_STORE) {
        if (!p->out || p->ldo % 8) return fail(SFB_ERR_INVALID, "sfb_gemm: out/ldo");
        if (p->residual && p->ldr % 8) return fail(SFB_ERR_INVALID, "sfb_gemm: ldr");
    } else if (p->epi == SFB_EPI_GEGLU) {
        if (!p->out || p->ldo % 8 || p->N % BN) return fail(SFB_ERR_INVALID, "sfb_gemm: geglu needs N %% 160 == 0");
        if (p->geglu_n_out <= 0 || p->geglu_n_out % 8 || p->geglu_n_out > p->N / 2)
            return fail(SFB_ERR_INVALID, "sfb_gemm: geglu_n_out");
        e.geglu_n_out = p->geglu_n_out;
    } else if (p->epi == SFB_EPI_QKV) {
        if (p->head_dim % 8 || p->heads <= 0 || p->seq <= 0 || p->N % (p->heads * p->head_dim))
            return fail(SFB_ERR_INVALID, "sfb_gemm: qkv geometry");
    } else if (p->epi == SFB_EPI_STORE_F32) {
        if (!p->out || p->ldo % 4 || p->residual || p->rowstats_out || p->ln_rowstats || a.splits != 1 || p->persistent)
            return fail(SFB_ERR_INVALID, "sfb_gemm: the fp32 store epilogue takes bias only, no split-K, one-tile kernel");
    } else {
        return fail(SFB_ERR_INVALID, "sfb_gemm: epilogue mode");
    }
#ifdef SFB_TRACE
    a.trace = g_trace_next;
    g_trace_next = nullptr;
#endif
    const int n_tiles = (p->N + BN - 1) / BN;
    CUtensorMap ta, tb;
    memcpy(&ta, p->tmap_a, sizeof(CUtensorMap));
    memcpy(&tb, p->tmap_b, sizeof(CUtensorMap));
    if (p->persistent && (!p->cta_pair || a.splits != 1 || m_tiles % 2 || (upconv && a.up_tiles % 2) || p->defer_finish))
        return fail(SFB_ERR_INVALID, "sfb_gemm: persistent needs cta_pair, no split-K and an even number of M tiles (per up-conv phase)");
    if (p->cta_pair && (m_tiles % 2 || (upconv && a.up_tiles % 2)))
        return fail(SFB_ERR_INVALID, "sfb_gemm: cta_pair needs an even number of M tiles (per up-conv phase)");
    // cta_pair / persistent describe the caller's tensor maps (tmap_b box = 80 rows); every launch is the
    // one-tile kernel, which loads such a 160-row weight tile as two boxes
    a.b_half = p->cta_pair ? 1 : 0;
    // gridDim.y is at most 65535: a larger M (e.g. 25 frames of 576 x 1024 = 115,200 tiles) runs as several
    // launches over consecutive M-tile ranges (an even count each, so CTA pairs stay whole)
    constexpr int kMaxGridY = 65534;
    if (m_tiles > kMaxGridY && a.splits != 1)
        return fail(SFB_ERR_INVALID, "sfb_gemm: %d M tiles with split-K (at most %d)", m_tiles, kMaxGridY);
    if (p->defer_finish && a.splits > 1 && (e.epi != SFB_EPI_STORE || e.rowstats_out || e.ln_rowstats))
        return fail(SFB_ERR_INVALID, "sfb_gemm: defer_finish needs a plain STORE epilogue");
    int rc = 0;
    for (int m0 = 0; m0 < m_tiles && rc == 0; m0 += kMaxGridY) {
        a.m_tile_base = m0;
        const dim3 grid(n_tiles, m_tiles - m0 < kMaxGridY ? m_tiles - m0 : kMaxGridY, a.splits);
        if (gnconv)
            rc = e.dtype == SFB_BF16 ? launch_gemm_t<3, 1, 1>(ta, tb, a, grid, stream)
                                     : launch_gemm_t<3, 0, 1>(ta, tb, a, grid, stream);
        else
            rc = e.dtype == SFB_BF16 ? launch_gemm_t<kGemmStages, 1>(ta, tb, a, grid, stream)
                                     : launch_gemm_t<kGemmStages, 0>(ta, tb, a, grid, stream);
    }
    if (rc) return rc;
    if (p->defer_finish && a.splits > 1) return rc;  // the consumer (sfb_group_norm_fused with part_ws) finishes the tensor
    if (a.splits > 1) {
        const int ncols = (e.epi == SFB_EPI_GEGLU) ? e.geglu_n_out : e.N;
        const long long items = (long long)e.M * (ncols / 8);
        const int blocks = (int)((items + 255) / 256);
        cudaError_t err = (e.dtype == SFB_BF16)
            ? launch_pdl(splitk_finish_kernel<1>, dim3(blocks), dim3(256), 0, stream, (const float*)a.ws, a.splits, e)
            : launch_pdl(splitk_finish_kernel<0>, dim3(blocks), dim3(256), 0, stream, (const float*)a.ws, a.splits, e);
        if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "sfb_gemm: finish launch: %s", cudaGetErrorString(err));
        rc = check_launch("sfb_gemm(split-K finish)");
    }
    return rc;
}
