// sfb_lora_merge: the effective weight of a LoRA-adapted layer, W + sum_i s_i * B_i A_i, rounded once to
// 16 bits.  Runs when a pipeline's adapter state changes (never inside a step): its output is fed to the
// same weight packers as a plain parameter, so the step's launch list does not change.
//
// One CTA owns a TN x TK tile of the output and walks every adapter's rank in chunks of RC: s_i * B_i[rows,
// chunk] and A_i[chunk, cols] are staged in shared memory as fp32, each thread accumulates a 4 x 4 block in
// fp32 registers (CUDA-core FMA: about r / 2 FLOP per byte of a 16-bit W, well under the FP32 roofline's
// balance point for the ranks adapters use).
#include "common.cuh"
#include "host.h"

namespace sfb {
namespace {

constexpr int TN = 32, TK = 128, RC = 32, THREADS = 256;
constexpr int RPT = TN / (THREADS / 32);  // output rows per thread (4)
constexpr int CPT = TK / 32;              // output columns per thread (4), strided by 32

__device__ __forceinline__ float load_any(const void* p, size_t i, int dt) {
    if (dt == SFB_F32) return reinterpret_cast<const float*>(p)[i];
    return load1(p, i, dt == SFB_BF16);
}

__global__ void __launch_bounds__(THREADS) lora_merge_kernel(const sfb_lora_merge_params p) {
    __shared__ float sB[TN][RC + 1];
    __shared__ float sA[RC][TK];
    pdl_launch_dependents();
    pdl_wait();
    const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
    const int n0 = blockIdx.y * TN, k0 = blockIdx.x * TK;
    float acc[RPT][CPT];
#pragma unroll
    for (int r = 0; r < RPT; ++r)
#pragma unroll
        for (int c = 0; c < CPT; ++c) acc[r][c] = 0.f;

    for (int i = 0; i < p.count; ++i) {
        const sfb_lora_adapter& ad = p.adapters[i];
        for (int j0 = 0; j0 < ad.rank; j0 += RC) {
            for (int e = tid; e < TN * RC; e += THREADS) {
                const int r = e / RC, j = e % RC, n = n0 + r, jj = j0 + j;
                sB[r][j] = (n < p.n && jj < ad.rank)
                    ? ad.scale * load_any(ad.b, (size_t)n * ad.ldb + jj, ad.b_dtype) : 0.f;
            }
            for (int e = tid; e < RC * TK; e += THREADS) {
                const int j = e / TK, c = e % TK, k = k0 + c, jj = j0 + j;
                sA[j][c] = (k < p.k && jj < ad.rank) ? load_any(ad.a, (size_t)jj * ad.lda + k, ad.a_dtype) : 0.f;
            }
            __syncthreads();
#pragma unroll 8
            for (int j = 0; j < RC; ++j) {
                float a[CPT], b[RPT];
#pragma unroll
                for (int c = 0; c < CPT; ++c) a[c] = sA[j][tx + 32 * c];
#pragma unroll
                for (int r = 0; r < RPT; ++r) b[r] = sB[ty * RPT + r][j];
#pragma unroll
                for (int r = 0; r < RPT; ++r)
#pragma unroll
                    for (int c = 0; c < CPT; ++c) acc[r][c] = fmaf(b[r], a[c], acc[r][c]);
            }
            __syncthreads();
        }
    }
#pragma unroll
    for (int r = 0; r < RPT; ++r) {
        const int n = n0 + ty * RPT + r;
        if (n >= p.n) continue;
#pragma unroll
        for (int c = 0; c < CPT; ++c) {
            const int k = k0 + tx + 32 * c;
            if (k < p.k)
                store1(p.out, (size_t)n * p.ldo + k, load_any(p.w, (size_t)n * p.ldw + k, p.w_dtype) + acc[r][c],
                       p.out_dtype == SFB_BF16);
        }
    }
}

}  // namespace
}  // namespace sfb

using namespace sfb;

extern "C" int sfb_lora_merge(const sfb_lora_merge_params* p, sfb_stream_t stream) {
    if (!p) return fail(SFB_ERR_INVALID, "lora_merge: null parameters");
    if (!p->w || !p->out || p->n <= 0 || p->k <= 0 || p->ldw < p->k || p->ldo < p->k)
        return fail(SFB_ERR_INVALID, "lora_merge: bad W / out geometry (n=%d k=%d ldw=%d ldo=%d)", p->n, p->k,
                    p->ldw, p->ldo);
    if (p->w_dtype < SFB_F16 || p->w_dtype > SFB_F32 || (p->out_dtype != SFB_F16 && p->out_dtype != SFB_BF16))
        return fail(SFB_ERR_INVALID, "lora_merge: W must be fp16 / bf16 / fp32 and out fp16 / bf16");
    if (p->count < 1 || p->count > SFB_LORA_MAX_ADAPTERS)
        return fail(SFB_ERR_INVALID, "lora_merge: %d adapters (1..%d)", p->count, SFB_LORA_MAX_ADAPTERS);
    for (int i = 0; i < p->count; ++i) {
        const sfb_lora_adapter& a = p->adapters[i];
        if (!a.a || !a.b || a.rank < 1 || a.rank > SFB_LORA_MAX_RANK || a.lda < p->k || a.ldb < a.rank ||
            a.a_dtype < SFB_F16 || a.a_dtype > SFB_F32 || a.b_dtype < SFB_F16 || a.b_dtype > SFB_F32)
            return fail(SFB_ERR_INVALID, "lora_merge: bad adapter %d (rank %d, lda %d, ldb %d)", i, a.rank, a.lda,
                        a.ldb);
    }
    if ((p->n + TN - 1) / TN > 65535) return fail(SFB_ERR_INVALID, "lora_merge: n=%d too large", p->n);
    const dim3 grid((p->k + TK - 1) / TK, (p->n + TN - 1) / TN);
    cudaError_t err = launch_pdl(lora_merge_kernel, grid, dim3(THREADS), 0, static_cast<cudaStream_t>(stream), *p);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "lora_merge: %s", cudaGetErrorString(err));
    return check_launch("sfb_lora_merge");
}
