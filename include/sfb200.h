/*
 * sfb200.h -- C ABI of the H100-native diffusion-UNet hot path (libsfb200.so).
 *
 * Drop-in boundary.  The reference binds its native code as a pybind11/TORCH_LIBRARY module
 * (`sfast._C`, /root/reference/src/sfast/csrc/main.cpp:13-24) whose operators take at::Tensor,
 * allocate their outputs and launch on at::cuda::getCurrentCUDAStream().  This library is the
 * replacement for the operators on the UNet hot path, re-cut as a plain C ABI:
 *
 *   - plain pointers and sizes only (no torch / ATen types);
 *   - the CALLER owns every buffer (activations, packed weights, workspaces, tensor maps);
 *   - the library never allocates device memory, never synchronises and only launches on the
 *     stream it is given, so every entry point is CUDA-graph capturable;
 *   - every entry point returns 0 on success or a negative sfb_status; sfb_last_error() gives a
 *     thread-local message.  There is NO CPU / library fallback: a missing GPU path is an error.
 *
 * Reference operator each entry point replaces (file:line under /root/reference/src/sfast):
 *   sfb_gemm            csrc/operators/cudnn/cudnn_convolution_impl.cc:890-987,1413-1433
 *                       (cudnn_convolution_bias / _bias_add), csrc/operators/cublas/
 *                       cublas_gemm.cpp:798-853,900-948 (cublas_lowp_linear / _linear_add),
 *                       csrc/operators/cutlass/cutlass_dual_linear_kernel.cu:442-539
 *                       (cutlass_linear_geglu_unified)
 *   sfb_attention       libs/xformers/xformers_attention.py:26-63 (memory_efficient_attention)
 *   sfb_attention_ip    the same attention plus the IP-Adapter image-prompt term (the reference traces
 *                       diffusers' IPAdapterAttnProcessor2_0 into two aten attention calls)
 *   sfb_group_norm_*    triton/ops/group_norm.py:126-165,272-320 (group_norm / group_norm_silu)
 *   sfb_layer_norm      triton/ops/layer_norm.py:51-133
 *   sfb_small_linear    csrc/operators/cublas/cublas_gemm.cpp:798-853 at M = batch rows
 *   sfb_timestep_embed, sfb_conv_in, sfb_conv_out, sfb_upsample2x: aten ops the reference
 *                       leaves untouched in the traced graph (SURVEY.md section 8a, row a11)
 */
#ifndef SFB200_H_
#define SFB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SFB_ABI_VERSION 4

typedef void* sfb_stream_t; /* cudaStream_t */

enum sfb_status {
    SFB_OK = 0,
    SFB_ERR_INVALID = -1,   /* bad argument / unsupported shape */
    SFB_ERR_CUDA = -2,      /* CUDA runtime / driver error */
    SFB_ERR_NO_DRIVER = -3, /* driver entry point unavailable */
};

enum sfb_dtype { SFB_F16 = 0, SFB_BF16 = 1, SFB_F32 = 2 /* sfb_lora_merge inputs only */ };

int sfb_abi_version(void);
const char* sfb_last_error(void);
/* Number of kernel launches issued through this library since load (host-side counter). */
uint64_t sfb_launch_count(void);
/* Programmatic dependent launch (default on): kernels are launched with the programmatic stream
 * serialization attribute and gate their first dependent global access on griddepcontrol.wait, so
 * a kernel's prologue overlaps its predecessor's tail (also inside captured CUDA graphs). */
void sfb_set_pdl(int enable);
/* Streaming multiprocessors of the current CUDA device (grid sizing of persistent / cooperative
 * kernels; 132 on an H100 SXM). */
int sfb_sm_count(void);

/* ---- TMA tensor maps (host side; `out128` receives a 128-byte, 64-byte-aligned CUtensorMap) */

/* Row-major 2-D matrix [rows, cols] of 16-bit elements, row pitch `pitch_elems`;
 * box = [box_rows, 64 cols], 128-byte swizzle. */
int sfb_tmap_2d(void* out128, const void* base, uint64_t rows, uint64_t cols,
                uint64_t pitch_elems, uint32_t box_rows);

/* NHWC activation [n, h, w, c] of 16-bit elements with channel pitch `pitch_elems`
 * (>= c; lets a tensor live inside a wider concat buffer).  box = [box_n, box_h, box_w, 64 ch];
 * `stride` (1 or 2) is the traversal stride along h and w (stride-2 convolution). */
int sfb_tmap_nhwc(void* out128, const void* base, uint32_t n, uint32_t h, uint32_t w, uint32_t c,
                  uint64_t pitch_elems, uint32_t box_n, uint32_t box_h, uint32_t box_w,
                  uint32_t stride);

/* ---- wgmma GEMM / implicit-GEMM convolution -------------------------------------------- */

enum sfb_gemm_a_mode {
    SFB_A_MATRIX = 0,  /* A is [M, K] row-major (linear layers, 1x1 convolutions) */
    SFB_A_CONV3X3 = 1, /* A is an NHWC image; K = 9 * cin, padding 1, stride 1 or 2 */
    /* (SFB_A_DOWNCONV3X3 = 5, below: the stride-2 variant with padding after the image only) */
    /* nearest-2x upsample followed by a 3x3 convolution, computed on the LOW-resolution image
     * without materialising the upsampled tensor: output pixel (2y+py, 2x+px) only sees a 2x2
     * neighbourhood of the source, so each of the 4 output phases (py, px) is a 2x2 convolution
     * with pre-summed weights -- K = 4 * cin instead of 9 * cin (2.25x fewer FLOPs).  img_* are
     * the SOURCE dims, M = 4 * img_n * img_h * img_w output pixels; the weight matrix holds the
     * 4 phases back to back, each padded to a multiple of 160 rows ([4 * Np, 4 * cin],
     * K order (ty, tx, c)); M tiles of phase p are tiles [p * T, (p + 1) * T) of the grid. */
    SFB_A_UPCONV2X = 2,
    /* Conv3d with a (3, 1, 1) kernel, padding (1, 0, 0), over the FRAME axis of a video tensor (SVD
     * TemporalResnetBlock): the activation is viewed as NHWC [n = videos, h = frames, w = pixels
     * per frame, c]; K = 3 * cin in (kt, c) order; tap kt reads frame f - 1 + kt (TMA zero fill =
     * the temporal padding).  img_* / box_* describe that view. */
    SFB_A_CONV3X1 = 3,
    /* GroupNorm(+SiLU) FOLDED INTO the 3x3 convolution's A-operand path (stride 1, padding 1): A is the
     * RAW (un-normalised) NHWC activation and gn_scale_shift holds, per (image, channel), the pair
     * (scale, shift) = (rstd * gamma, beta - mean * rstd * gamma) written by sfb_group_norm_scale_shift.
     * The M tile is a 16 x 8 pixel patch (box_n = 1, box_h = 16, box_w = 8; img_w % 8 == 0; rows past
     * the image are masked).  Per 64-channel block the kernel pulls ONE [18 x 10]-pixel halo tile of
     * the patch through TMA (tmap_a: sfb_tmap_nhwc with box_n = 1, box_h = 18, box_w = 10), applies
     * y = act(x * scale + shift) to each halo element once, in shared memory (padding pixels forced back
     * to zero), and all nine filter taps multiply shifted views of that tile: the normalised activation
     * never exists in HBM and the conv reads its input through L2 once instead of nine times.  Needs
     * splits == 1, no persistent, the STORE epilogue (bias / rowbias / residual as for SFB_A_CONV3X3).
     * Replaces the separate group_norm_silu launch of the reference
     * (/root/reference/src/sfast/jit/passes/triton_passes.py:68-88,
     *  src/sfast/triton/ops/group_norm.py:272-320) in front of cudnn_convolution_bias(_add). */
    SFB_A_CONV3X3_GN = 4,
    /* 3x3 convolution, stride 2, zero padding of ONE row and ONE column AFTER the image and none before
     * (diffusers' Downsample2D with padding=0, the VAE encoder's downsampler: F.pad(x, (0, 1, 0, 1))
     * then a pad-0 stride-2 conv): output pixel (i, j) reads input rows 2i..2i+2 and columns 2j..2j+2.
     * A is the INPUT image through sfb_tmap_nhwc with stride 2 over [n, 2 * img_h, 2 * img_w, cin];
     * the last tap lands on row / column 2 * img_h / 2 * img_w, past the image, which TMA zero-fills.
     * img_* are the OUTPUT dims; K = 9 * cin (cin % 64 == 0), conv_stride must be 2, no rowbias;
     * box, split-K and epilogue rules as for SFB_A_CONV3X3. */
    SFB_A_DOWNCONV3X3 = 5,
};

enum sfb_epilogue {
    SFB_EPI_STORE = 0, /* out[m, n] = acc + bias[n] + rowbias[img(m), n] + residual[m, n] */
    SFB_EPI_GEGLU = 1, /* out[m, j] = (acc_v + b_v) * gelu(acc_g + b_g); weights tile-interleaved */
    SFB_EPI_QKV = 2,   /* scatter columns into per-head Q / K ([bh, s, dp]) and V^T ([bh, d, sp]) */
    /* out is fp32 [M, ldo floats]: acc + bias, unrounded (attention scores of the VAE's single-head
     * attention: 16-bit scores lose ~2 % on the probabilities).  One-tile kernel only, no split-K. */
    SFB_EPI_STORE_F32 = 3,
};

enum { SFB_ACT_NONE = 0, SFB_ACT_QUICK_GELU = 1 /* x * sigmoid(1.702 x) */, SFB_ACT_GELU = 2 /* erf form */,
       SFB_ACT_SILU = 3 /* x * sigmoid(x) */, SFB_ACT_RELU = 4 /* max(x, 0) */ };

typedef struct sfb_gemm_params {
    const void* tmap_a; /* host pointer to a 128-byte tensor map */
    const void* tmap_b; /* weights, TILED: block (n_tile, k_block) = contiguous [160, 64]; 2-D map
                         * over [n_tiles * K/64 * 160, 64], box rows = 160 (80 with cta_pair).  With
                         * b_plain: a plain row-major [N, K] matrix (sfb_tmap_2d, same box rows) */
    int32_t a_mode;
    int32_t M, N, K;
    int32_t dtype;
    /* SFB_A_CONV3X3 geometry: OUTPUT image dims and the M-tile box: 128 pixels =
     * [box_n images, box_h rows, box_w columns].  box_w = 0 means img_w (full-width rows; the only
     * form that allows box_n > 1); box_w < img_w (must divide img_w) tiles the image with 2-D
     * patches, which is how widths that do not divide 128 (96, 104, ...) are handled. */
    int32_t img_n, img_h, img_w, cin, conv_stride, box_h, box_n, box_w;
    /* split-K: >1 writes fp32 partials to `ws` ([splits, M, N]); a second kernel sums them and runs
     * the fused epilogue (or, with defer_finish, the consuming GroupNorm does). */
    int32_t splits;
    float* ws;
    /* 1 (with splits > 1 and the STORE epilogue): only write the partials; the consumer
     * (sfb_group_norm_fused with part_ws) finishes the tensor */
    int32_t defer_finish;
    /* epilogue */
    int32_t epi;
    void* out;
    int32_t ldo;
    const float* bias;    /* [N] fp32 or NULL */
    const float* rowbias; /* [M / rows_per_img, ld_rowbias] fp32 or NULL (time-embedding add) */
    int32_t rows_per_img;
    int32_t ld_rowbias;
    const void* residual; /* [M, ldr] 16-bit or NULL */
    int32_t ldr;
    /* SFB_EPI_GEGLU: logical output width; weight rows are tile-interleaved: physical columns
     * [160 j, 160 j + 80) are the value half and [160 j + 80, 160 j + 160) the gate half of
     * output columns [80 j, 80 j + 80); N is the padded physical width (multiple of 160). */
    int32_t geglu_n_out;
    /* SFB_EPI_QKV */
    void* q;
    void* k;
    void* vt;
    int32_t heads, head_dim; /* column n -> which = n / (heads*head_dim) + which_base */
    int32_t which_base;      /* 0: q,k,v   1: k,v (cross-attention K/V projection) */
    int32_t seq;             /* tokens per batch item: row m -> (b, s) = (m / seq, m % seq) */
    int32_t q_pitch;         /* element pitch of a Q/K row (64 / 128 / 192) */
    int32_t q_rows;          /* rows allocated per (b, head) in the Q buffer */
    int32_t k_rows;          /* rows allocated per (b, head) in the K buffer */
    int32_t vt_rows;         /* rows per (b, head) in V^T: (head_dim + 1) rounded up to 16; row
                              * `head_dim` must be pre-filled with ones (softmax denominator) */
    int32_t vt_pitch;        /* element pitch of a V^T row */
    /* 1: tmap_b was built with the 80-row box (half a 160-row weight tile; the kernel loads a tile as
     * two boxes); needs an even number of M tiles (per up-conv phase). */
    int32_t cta_pair;
    /* 1: accepted for ABI compatibility with the same requirements as before (cta_pair, splits == 1,
     * even number of M tiles, no defer_finish / rowstats_out / act / fp32 store); the launch is the
     * one-tile kernel like every other. */
    int32_t persistent;
    /* 1: the B operand is a plain row-major [N, K] 16-bit matrix -- an ACTIVATION (activation x
     * activation products: Q K^T and P V of the VAE's single-head attention), not a pre-tiled weight */
    int32_t b_plain;
    /* LayerNorm folded around the GEMM (replaces sfast_triton::layer_norm,
     * /root/reference/src/sfast/triton/ops/layer_norm.py:51-133, as a separate pass):
     *   producer (SFB_EPI_STORE): rowstats_out[m][slot] = (sum, sum of squares) over the columns that slot
     *     covers of the stored row -- slot = the 160-column tile (one-tile kernel) or the warp segment of the
     *     row (split-K reduction); every slot is WRITTEN once, nothing is accumulated atomically;
     *   consumer: A is the RAW activation, the weight is pre-scaled by gamma (W' = W * gamma),
     *     out = rstd_m * (acc - mean_m * ln_colsum[n]) + bias[n],  bias = beta W^T + b,
     *     (mean_m, rstd_m) from the ln_slots slots of ln_rowstats[m] added in index order, over ln_dim columns.
     *   Slots no producer wrote must be zero: the caller clears the buffer (once per step).  Results are
     *   bit-identical from run to run.  sfb_rowstats_slots(N) = slots a producer of N columns may write. */
    float* rowstats_out;       /* [M, rowstats_out_slots, 2] fp32 or NULL */
    const float* ln_rowstats;  /* [M, ln_slots, 2] fp32 or NULL */
    const float* ln_colsum;    /* [N] fp32: sum_k W'[n, k] */
    float ln_eps;
    int32_t ln_dim;
    /* element-wise activation of the SFB_EPI_STORE epilogue, applied after bias / LayerNorm fold and
     * before the residual add (the CLIP text encoders' MLP: fc1 + quick_gelu / gelu, encoders traced by
     * /root/reference/src/sfast/compilers/diffusion_pipeline_compiler.py:93-103; ReLU: the T2I-Adapter's
     * 3x3 convs).  Needs splits == 1. */
    int32_t act; /* SFB_ACT_* */
    int32_t rowstats_out_slots; /* slots per row of rowstats_out (>= sfb_rowstats_slots(N)) */
    int32_t ln_slots;           /* slots per row of ln_rowstats */
    /* SFB_A_CONV3X3_GN */
    const float* gn_scale_shift; /* [img_n, cin, 2] fp32: (scale, shift) per image and input channel */
    int32_t gn_silu;             /* 1: SiLU after the affine */
} sfb_gemm_params;

/* slots per row a rowstats_out producer with N output columns needs (any split-K factor) */
int sfb_rowstats_slots(int32_t n_cols);

int sfb_gemm(const sfb_gemm_params* p, sfb_stream_t stream);

/* ---- wgmma flash attention: O = softmax(Q K^T * scale) V ------------------------------- */

typedef struct sfb_attn_params {
    const void* tmap_q;  /* 2-D map over Q  [bh * q_rows,  q_pitch], box 128 rows */
    const void* tmap_k;  /* 2-D map over K  [bh * k_rows,  q_pitch], box 128 rows (kv_tile 64: 64) */
    const void* tmap_vt; /* 2-D map over V^T [bh * vt_rows, vt_pitch], box vt_rows rows */
    void* out;           /* [batch, seq_q, heads * head_dim] 16-bit */
    int32_t batch, heads, head_dim;
    int32_t seq_q, seq_kv;
    int32_t q_rows, k_rows, vt_rows;
    int32_t dtype;
    float scale; /* 1 / sqrt(head_dim) */
    /* 0 / 128: 128-key score tiles.  64 (head_dim 32 / 40 / 64 / 160): 64-key score tiles (fewer
     * accumulator registers per thread). */
    int32_t kv_tile;
    /* 1: causal mask (key j attends to query i only if j <= i; seq_q == seq_kv, kv_tile 64): the text
     * encoders' self-attention */
    int32_t causal;
} sfb_attn_params;

int sfb_attention(const sfb_attn_params* p, sfb_stream_t stream);

/* Attention with an image prompt (diffusers' IPAdapterAttnProcessor2_0 of one IP-Adapter):
 *   O = softmax(Q K^T * scale) V + s * softmax(Q K_ip^T * scale) V_ip,   s = *ip_scale
 * `base` describes the text attention exactly as for sfb_attention.  K_ip / V_ip^T are laid out like K /
 * V^T (the QKV-scatter epilogue writes them): K_ip [bh * k_ip_rows, q_pitch] through tmap_k_ip (box kv_tile
 * rows), V_ip^T [bh * vt_rows, pitch >= kv_tile] through tmap_vt_ip (box vt_rows rows; the ones row of V^T
 * is not needed).  Limits: 1 <= seq_ip <= kv_tile (the image tokens are one KV tile: n_img * 4 tokens up to
 * 64 fit every head_dim), k_ip_rows >= seq_ip, no causal mask; every head_dim / kv_tile pair of
 * sfb_attention, fp16 and bf16.  `ip_scale` is ONE fp32 value in DEVICE memory, so a captured graph serves
 * every scale.  When it is 0 the image pass is skipped and the output is bit-identical to sfb_attention's
 * on `base`. */
typedef struct sfb_attn_ip_params {
    sfb_attn_params base;
    const void* tmap_k_ip;
    const void* tmap_vt_ip;
    int32_t seq_ip, k_ip_rows;
    const float* ip_scale;
} sfb_attn_ip_params;

int sfb_attention_ip(const sfb_attn_ip_params* p, sfb_stream_t stream);

/* ---- normalisation ----------------------------------------------------------------------- */

typedef struct sfb_gn_params {
    const void* x;   /* NHWC [n, hw, c] 16-bit, channel pitch ldx */
    void* y;         /* [n, hw, c] 16-bit, channel pitch ldy */
    const float* gamma;
    const float* beta;
    float* stats;    /* statistics WORKSPACE, sfb_group_norm_ws_floats(n, groups) floats, no initialisation
                      * needed: one slot of [groups][2] SHIFTED moments (sum(x - K), sum((x - K)^2) about the
                      * group's first stored value K = x[img, 0, g * c/groups]) per CTA of the statistics
                      * pass, summed by the apply pass in a fixed order -- no floating-point atomics, so
                      * results are bit-identical from run to run.  stats -> apply must use the same params. */
    int32_t n, hw, c, ldx, ldy, groups;
    float eps;
    int32_t silu;    /* 1: y = silu(gn(x)) */
    int32_t dtype;
    uint32_t* sync_counter; /* sfb_group_norm_fused only: grid-barrier counter, zeroed by caller */
    /* sfb_group_norm_fused only.  part_splits > 1: channels [0, part_c) of x do not exist yet --
     * they are the fp32 split-K partials `part_ws` ([part_splits, n*hw, part_ld]) of a sfb_gemm
     * launched with defer_finish.  The kernel sums them, applies that GEMM's STORE epilogue
     * (part_bias [part_c], part_rowbias [n, part_ld_rowbias] per image, part_residual with pitch
     * part_ldr; each may be NULL), writes the finished 16-bit values into x and normalises them
     * in the same pass: the split-K reduction kernel disappears. */
    const float* part_ws;
    int32_t part_splits, part_c, part_ld;
    const float* part_bias;
    const float* part_rowbias;
    int32_t part_ld_rowbias;
    const void* part_residual;
    int32_t part_ldr;
} sfb_gn_params;

/* two-pass path (any size) */
int sfb_group_norm_stats(const sfb_gn_params* p, sfb_stream_t stream);
int sfb_group_norm_apply(const sfb_gn_params* p, sfb_stream_t stream);
/* Statistics pass that ends in the per-(image, channel) affine a consumer applies itself -- the conv with
 * SFB_A_CONV3X3_GN: scale_shift[img][ch] = (rstd * gamma[ch], beta[ch] - mean * rstd * gamma[ch]), fp32
 * [n, c, 2].  One launch: every CTA writes its slot of `stats`, the LAST CTA of an image to finish (an
 * integer ticket in p->sync_counter[img]; n counters, zero before the first launch, reset by the kernel)
 * adds the image's slots in the fixed order of the other paths and writes the pairs -- bit-identical from
 * run to run.  p->y / ldy / silu are unused. */
int sfb_group_norm_scale_shift(const sfb_gn_params* p, float* scale_shift, sfb_stream_t stream);
/* single-launch path for tensors that fit in the GPU's shared memory: a COOPERATIVE launch of at
 * most one CTA per SM of the current device with a grid-wide barrier; x is read once.  `stats` and
 * `sync_counter` must be zero on entry.  sfb_group_norm_fused_fits() returns 1 when the geometry
 * qualifies on the current device. */
/* floats the `stats` workspace of one GroupNorm over n images must hold on this device */
int sfb_group_norm_ws_floats(int32_t n, int32_t groups);
int sfb_group_norm_fused_fits(const sfb_gn_params* p);
int sfb_group_norm_fused(const sfb_gn_params* p, sfb_stream_t stream);

typedef struct sfb_ln_params {
    const void* x; /* [rows, c] 16-bit, pitch ldx */
    void* y;       /* [rows, c] 16-bit, pitch ldy */
    const float* gamma;
    const float* beta;
    int32_t rows, c, ldx, ldy;
    float eps;
    int32_t dtype;
} sfb_ln_params;

int sfb_layer_norm(const sfb_ln_params* p, sfb_stream_t stream);

/* ---- small / glue kernels ---------------------------------------------------------------- */

/* out[b, :] = [cos(t_b f_i) | sin(t_b f_i)] (flip_sin_to_cos) or [sin | cos], 16-bit output */
int sfb_timestep_embed(const float* t, int32_t batch, int32_t dim, int32_t flip_sin_to_cos,
                       float freq_shift, void* out, int32_t ldo, int32_t dtype,
                       sfb_stream_t stream);

/* y[b, n] = act_out(sum_k act_in(x[b, k]) W[n, k] + bias[n] (+ add[b, n]));
 * act: 0 none, 1 SiLU.  x 16-bit [batch, k]; W 16-bit [n, k]; y 16-bit (y16) or fp32 (y32). */
typedef struct sfb_small_linear_params {
    const void* x;
    const void* w;
    const float* bias;
    const void* add16; /* optional 16-bit [batch, n] added before act_out */
    void* y16;
    float* y32;
    int32_t batch, n, k, ldx, ldy;
    int32_t act_in, act_out;
    int32_t dtype;
} sfb_small_linear_params;

int sfb_small_linear(const sfb_small_linear_params* p, sfb_stream_t stream);

/* 3x3 pad-1 convolution with tiny channel counts at the two ends of the UNet.
 * conv_in:  x NCHW [n, cin<=8, h, w] 16-bit  -> y NHWC [n, h, w, cout] (channel pitch ldy)
 * conv_out: x NHWC [n, h, w, cin] (pitch ldx) -> y NCHW [n, cout<=8, h, w] 16-bit
 * conv_in  w: 16-bit [3, 3, cin, cout] (tap-major, cout contiguous);
 * conv_out w: 16-bit [cout, 3, 3, cin]; bias fp32.  Both stage the whole weight in shared memory:
 * conv_in up to 48 KB, conv_out up to 227 KB (e.g. the VAE encoder's 512 -> 8 conv_out, 72 KB). */
/* im2col of the first convolution: x NCHW [n, cin<=7, h, w] 16-bit -> a [n*h*w, 64] 16-bit with
 * a[p, (kh*3+kw)*cin + c] and zero padding up to 64; feeds sfb_gemm (K = 64). */
int sfb_im2col_in(const void* x, void* a, int32_t n, int32_t h, int32_t wd, int32_t cin,
                  sfb_stream_t stream);
/* The same for a wide first convolution (e.g. the inpainting UNets' 9 input channels): x NCHW
 * [n, 9 <= cin <= 14, h, w] 16-bit -> a [n*h*w, 128] 16-bit with a[p, (kh*3+kw)*cin + c] and zero
 * padding up to 128; feeds sfb_gemm (K = 128).  n, h, w positive, n*h*w < 2^31. */
int sfb_im2col_in_wide(const void* x, void* a, int32_t n, int32_t h, int32_t wd, int32_t cin,
                       sfb_stream_t stream);
int sfb_conv_in(const void* x, const void* w, const float* bias, void* y, int32_t n, int32_t h,
                int32_t wd, int32_t cin, int32_t cout, int32_t ldy, int32_t dtype,
                sfb_stream_t stream);
int sfb_conv_out(const void* x, const void* w, const float* bias, void* y, int32_t n, int32_t h,
                 int32_t wd, int32_t cin, int32_t cout, int32_t ldx, int32_t dtype,
                 sfb_stream_t stream);
/* The tail of SVD's temporal VAE decoder: conv_out then time_conv_out.  The n images of x are
 * n / frames videos of `frames` consecutive frames (n % frames == 0).
 *   c[i]    = round16(conv3x3(x[i], w) + bias)           (sfb_conv_out's conv, same x / w / bias layout)
 *   y[v, f] = bt + sum_k wt[:, k, :] . c[v, f + k - 1]   (k = 0..2; frames -1 and `frames` are zero)
 * wt: 16-bit [cout, 3, cout] (output channel, frame tap, input channel) -- Conv3d weight
 * [cout, cout, 3, 1, 1] permuted; bt fp32 (may be NULL).  y NCHW [n, cout<=8, h, w] 16-bit.  c never
 * reaches memory.  Needs (n / frames) * h * w < 2^31. */
int sfb_conv_out_temporal(const void* x, const void* w, const float* bias, const void* wt, const float* bt,
                          void* y, int32_t n, int32_t h, int32_t wd, int32_t cin, int32_t cout, int32_t ldx,
                          int32_t frames, int32_t dtype, sfb_stream_t stream);

/* nearest-neighbour 2x upsample, NHWC, 16-bit */
int sfb_upsample2x(const void* x, void* y, int32_t n, int32_t h, int32_t w, int32_t c,
                   int32_t ldx, int32_t ldy, sfb_stream_t stream);

/* ---- SVD temporal path (UNetSpatioTemporalConditionModel; the reference traces the diffusers
 * module and leaves these to aten, compilers/diffusion_pipeline_compiler.py:101-103) ---------- */

/* Self-attention across frames: for every (video b, pixel p, head h) a sequence of `frames` <= 32
 * tokens of head_dim 64.  qkv is the fused projection [batch * frames * seq, ld_qkv] = q | k | v in
 * the SPATIAL row order m = (b * frames + f) * seq + p (no transposed copy of the activations);
 * out has the same row order. */
typedef struct sfb_temporal_attn_params {
    const void* qkv;
    void* out;
    int32_t batch, frames, seq, heads, head_dim;
    int32_t ld_qkv, ld_out, dtype;
    float scale;
} sfb_temporal_attn_params;

int sfb_temporal_attention(const sfb_temporal_attn_params* p, sfb_stream_t stream);

/* ---- AnimateDiff motion modules (diffusers UNetMotionModel; the reference traces the module) ---------- */

/* Self-attention across frames on the tensor cores: for every (video b, pixel p, head h) a sequence of `frames`
 * tokens, softmax(scale * q k^T) v with fp32 accumulation and an fp32 softmax.
 *   qkv:        [batch * frames * seq, ld_qkv] 16-bit = q | k | v column blocks of heads * head_dim each, in the
 *               SPATIAL row order m = (b * frames + f) * seq + p; out [same rows, ld_out] receives heads * head_dim
 *               columns in the same order;
 *   frame_bias: fp32 [frames, ld_bias] (q | k | v columns like qkv) or NULL: row f is added to the q / k / v of
 *               frame f as they are loaded (the sum is rounded to 16 bits once) -- a position embedding added
 *               in front of the projections, (x + pe_f) W^T = x W^T + pe_f W^T.
 * 1 <= frames <= 32, head_dim 40, 80 or 160, scale > 0; ld_qkv >= 3 * heads * head_dim and ld_out >= heads *
 * head_dim are multiples of 8; ld_bias >= 3 * heads * head_dim is a multiple of 4; pointers are 16-byte
 * aligned; out must not overlap qkv. */
typedef struct sfb_frame_attn_params {
    const void* qkv;
    const float* frame_bias;
    void* out;
    int32_t batch, frames, seq, heads, head_dim;
    int32_t ld_qkv, ld_bias, ld_out, dtype;
    float scale;
} sfb_frame_attn_params;

int sfb_frame_attention(const sfb_frame_attn_params* p, sfb_stream_t stream);

enum sfb_row_index_mode {
    SFB_ROW_IDX_DIV_MOD = 0,      /* vec row = (m / div) % mod */
    SFB_ROW_IDX_TEMPORAL_CTX = 1, /* vec row = ((b * seq + p) % batch) * frames, m = (b*frames + f)*seq + p:
                                   * diffusers' [H*W, B]-interleaved temporal cross-attention context */
};

/* Row-wise ops on token matrices [rows, c] of 16-bit elements, one warp per row:
 *   sfb_row_broadcast_add: y[m, :] = x[m, :] + vec[idx(m), :]   (frame position embedding; cross-
 *                          attention over ONE context token, where softmax over a single key is 1)
 *   sfb_alpha_blend:       y[m, :] = alpha * x[m, :] + (1 - alpha) * x2[m, :], alpha = sigmoid(*mix_factor)
 * rowstats_out (optional): [rows, rowstats_slots, 2] fp32; slot 0 receives (sum, sum of squares) of the STORED
 * row (written, not accumulated; the other slots stay as the caller cleared them) -- the statistics a
 * following folded LayerNorm consumes (sfb_gemm ln_rowstats / ln_slots). */
typedef struct sfb_row_op_params {
    const void* x;
    const void* x2;
    const void* vec;
    void* y;
    float* rowstats_out;
    const float* mix_factor;
    int32_t rows, c, ldx, ldx2, ldv, ldy, dtype;
    int32_t mode, div, mod, frames, seq, batch;
    int32_t rowstats_slots; /* slots per row of rowstats_out (0 = 1) */
} sfb_row_op_params;

int sfb_row_broadcast_add(const sfb_row_op_params* p, sfb_stream_t stream);
int sfb_alpha_blend(const sfb_row_op_params* p, sfb_stream_t stream);

/* ControlNet residuals (reference: compile() leaves the ControlNet eager and the traced UNet takes
 * `down_block_additional_residuals` / `mid_block_additional_residual` as extra inputs,
 * /root/reference/src/sfast/compilers/diffusion_pipeline_compiler.py:89-90):
 * dst[n, hw, c] (NHWC slice, channel pitch ld_dst) += src[n, c, hw] (NCHW contiguous), up to 16
 * tensors per launch. */
typedef struct sfb_add_nchw_item {
    const void* src;
    void* dst;
    int32_t n, c, hw, ld_dst;
} sfb_add_nchw_item;

typedef struct sfb_add_nchw_params {
    int32_t count;
    int32_t dtype;
    sfb_add_nchw_item items[16];
} sfb_add_nchw_params;

int sfb_add_nchw_residuals(const sfb_add_nchw_params* p, sfb_stream_t stream);

/* ---- ControlNet (diffusers ControlNetModel: a second UNet encoder plus the conditioning-image
 * embedding; the reference leaves the module itself to eager PyTorch) ------------------------- */

/* 3x3 convolution, zero padding 1 on every side, stride 1 or 2, for inputs with few channels (the
 * conditioning embedding's layers at image resolution): y = act(conv(x) + bias), fp32 accumulation
 * on mma.sync tensor cores, 16-bit storage.
 *   x:      NCHW [n, cin, h, w] contiguous (x_nchw = 1, cin <= 8), or NHWC [n, h, w] with channel
 *           pitch ldx (x_nchw = 0, cin < 64; cin and ldx multiples of 8);
 *   weight: 16-bit [cout, 3, 3, cin16], cin16 = cin rounded up to 16, channels past cin zero;
 *   bias:   fp32 [cout] or NULL;  silu: 1 applies SiLU after the bias;
 *   y:      NHWC [n, ho, wo] with channel pitch ldy (ho = (h - 1) / stride + 1, likewise wo);
 *           cout and ldy multiples of 8; only channels [0, cout) are written. */
typedef struct sfb_conv_small_params {
    const void* x;
    const void* weight;
    const float* bias;
    void* y;
    int32_t n, h, w, cin, cout, stride;
    int32_t ldx, ldy;
    int32_t x_nchw, silu, dtype;
} sfb_conv_small_params;

int sfb_conv3x3_small(const sfb_conv_small_params* p, sfb_stream_t stream);

/* sfb_conv3x3_small with an element-wise transform of the input and a ReLU option (the edge convolutions of
 * diffusers' AutoencoderTiny).  in_xform is applied to in-image input values only, so the zero padding stays
 * zero (which is why it cannot be folded into the weights); it needs the NCHW input (base.x_nchw = 1).
 * relu: 1 applies ReLU after the bias (base.silu must then be 0). */
enum sfb_conv_xform {
    SFB_XFORM_NONE = 0,
    SFB_XFORM_TANH3 = 1, /* tanh(x / 3) * 3   (DecoderTiny's latent clamp) */
    SFB_XFORM_UNIT = 2,  /* (x + 1) / 2       (EncoderTiny's [-1, 1] -> [0, 1]) */
};

typedef struct sfb_conv_small_ex_params {
    sfb_conv_small_params base;
    int32_t in_xform; /* enum sfb_conv_xform */
    int32_t relu;
} sfb_conv_small_ex_params;

int sfb_conv3x3_small_ex(const sfb_conv_small_ex_params* p, sfb_stream_t stream);

/* ---- AutoencoderTiny (TAESD / TAESDXL; the reference compiles it through the same auto-trace hooks as
 * any VAE, compilers/diffusion_pipeline_compiler.py:154-190) ------------------------------------------ */

enum sfb_c64_mode {
    SFB_C64_SAME = 0,    /* stride 1, zero padding 1: output h x w */
    SFB_C64_STRIDE2 = 1, /* stride 2, zero padding 1 on EVERY side (nn.Conv2d(stride=2, padding=1)): output
                          * ceil(h / 2) x ceil(w / 2); output row i reads input rows 2i - 1 .. 2i + 1 */
    SFB_C64_UP2X = 2,    /* nearest-2x upsample of x, then stride 1, padding 1: output 2h x 2w, computed from the
                          * h x w input (the upsampled tensor never exists) */
};

/* 3x3 convolution with cin = cout = 64, fp32 accumulation on tensor cores, 16-bit storage:
 *   y = relu?(conv(x) + bias (+ residual))
 *   x:        NHWC [n, h, w, 64], channel pitch ldx (input dims; `mode` gives the output dims ho x wo);
 *   weight:   16-bit [64, 3, 3, 64] (cout, kh, kw, cin), contiguous -- [64, 576] K-major;
 *   bias:     fp32 [64] or NULL;
 *   residual: NHWC [n, ho, wo, 64] 16-bit, channel pitch ldr, or NULL; may be y itself (in place);
 *   y:        NHWC [n, ho, wo, 64], channel pitch ldy;
 *   relu:     1 applies ReLU last (after the residual add).
 * Pitches are multiples of 8 and at least 64; every pointer is 16-byte aligned; x must not overlap y. */
typedef struct sfb_conv_c64_params {
    const void* x;
    const void* weight;
    const float* bias;
    const void* residual;
    void* y;
    int32_t n, h, w;
    int32_t ldx, ldy, ldr;
    int32_t mode; /* enum sfb_c64_mode */
    int32_t relu;
    int32_t dtype;
} sfb_conv_c64_params;

int sfb_conv3x3_c64(const sfb_conv_c64_params* p, sfb_stream_t stream);

/* dst[n, c, hw] (NCHW contiguous) = scale[i] * src[n, hw, c] (NHWC, channel pitch ld_src) for item i,
 * fp32 arithmetic, up to 16 tensors per launch (the ControlNet's down / mid residuals times
 * conditioning_scale).  `scale` is a DEVICE fp32 array [count]: a captured graph serves every scale. */
typedef struct sfb_nchw_scaled_item {
    const void* src;
    void* dst;
    int32_t n, c, hw, ld_src;
} sfb_nchw_scaled_item;

typedef struct sfb_nhwc_to_nchw_params {
    int32_t count;
    int32_t dtype;
    const float* scale;
    sfb_nchw_scaled_item items[16];
} sfb_nhwc_to_nchw_params;

int sfb_nhwc_to_nchw_scaled(const sfb_nhwc_to_nchw_params* p, sfb_stream_t stream);

/* ---- T2I-Adapter (diffusers T2IAdapter: PixelUnshuffle, convolutions and 2x2 average pools; the
 * reference traces the UNet with the adapter residuals as inputs and leaves the adapter eager) ---------- */

/* PixelUnshuffle(r) of a 16-bit NCHW tensor into NHWC:
 *   y[img, oy, ox, ch * r * r + i * r + j] = x[img, ch, oy * r + i, ox * r + j]
 * x: NCHW [n, c, h, w] contiguous; y: NHWC [n, h / r, w / r] with channel pitch ldy >= c * r * r (channels
 * past c * r * r are not written).  r >= 1 divides h and w.  Bit-exact (a permutation). */
int sfb_pixel_unshuffle(const void* x, void* y, int32_t n, int32_t c, int32_t h, int32_t w, int32_t r,
                        int32_t ldy, sfb_stream_t stream);

/* nn.AvgPool2d(2, 2) of a 16-bit NHWC tensor: y[img, oy, ox, :] = mean of the 2x2 window at (2oy, 2ox), summed
 * in fp32 and rounded once.  x: [n, h, w, c] with channel pitch ldx; y: [n, h / 2, w / 2, c] with pitch ldy.
 * h and w even (where ceil_mode=True pools the same windows); c, ldx, ldy multiples of 8; x and y 16-byte
 * aligned. */
int sfb_avg_pool2x2(const void* x, void* y, int32_t n, int32_t h, int32_t w, int32_t c, int32_t ldx,
                    int32_t ldy, int32_t dtype, sfb_stream_t stream);

/* ---- FreeU (diffusers UNet2DConditionModel.enable_freeu: up blocks 0 and 1 rescale the backbone features and
 * filter the skip features in front of every resnet; the reference traces the forward, torch.fft included) --- */

/* FreeU on one up-block resnet's NHWC concat buffer x [n, h, w] (channel pitch ld) = hidden [0, c_hidden) |
 * skip [c_hidden, c_hidden + c_skip), in place, 16-bit:
 *   hidden channels [0, c_hidden / 2):  y = x * b       (one fp32 multiply, one rounding: torch's x * b)
 *   skip channels:                      y = diffusers' fourier_filter(x, threshold=1, scale=s) per (image,
 *                                       channel), computed in closed form in fp32 with one rounding;
 *   every other channel and the pitch gap are not touched.
 * bs: DEVICE fp32 [2] = (b, s): a captured graph serves every value.  c_hidden, c_skip and ld are positive
 * multiples of 8, ld >= c_hidden + c_skip, x 16-byte aligned. */
typedef struct sfb_freeu_params {
    void* x;
    const float* bs;
    int32_t n, h, w, c_hidden, c_skip, ld, dtype;
} sfb_freeu_params;

int sfb_freeu(const sfb_freeu_params* p, sfb_stream_t stream);

/* dst[r, 0:cols] = src[r, 0:cols], 16-bit elements, row pitches in elements */
int sfb_copy2d(const void* src, void* dst, int32_t rows, int32_t cols, int32_t ld_src,
               int32_t ld_dst, sfb_stream_t stream);

/* Softmax over the rows of x [rows, cols] (fp32 when x_is_f32, else 16-bit; row pitch ldx elements of
 * its type) -> y 16-bit [rows, cols] (row pitch ldy elements), fp32 arithmetic.  y may alias x (each
 * row is read completely before it is written): the softmax of an attention computed as GEMMs (VAE
 * decoder, head_dim 512). */
int sfb_row_softmax(const void* x, void* y, int32_t rows, int32_t cols, int32_t ldx, int32_t ldy,
                    int32_t x_is_f32, int32_t dtype, sfb_stream_t stream);

/* 1x1 convolution with tiny channel counts on NCHW tensors (the VAE's post_quant_conv, 4 -> 4):
 * y[n, co, p] = bias[co] + sum_ci w[co, ci] x[n, ci, p]; cin, cout <= 8; w 16-bit [cout, cin]. */
int sfb_pointwise_nchw(const void* x, const void* w, const float* bias, void* y, int32_t n, int32_t hw,
                       int32_t cin, int32_t cout, int32_t dtype, sfb_stream_t stream);

/* cudaMemsetAsync wrapper (graph capturable) */
int sfb_memset(void* p, int32_t value, size_t bytes, sfb_stream_t stream);

/* ---- CLIP text encoder edges (reference: text_encoder / text_encoder_2 traced + graphed by
 * /root/reference/src/sfast/compilers/diffusion_pipeline_compiler.py:93-112) ---------------- */

/* out[b * seq + s, :] = tok_emb[ids[b, s], :] + pos_emb[s, :]   (16-bit tables and output, row pitch ld_out);
 * rowstats (optional, [rows, rowstats_slots, 2] fp32): slot 0 = (sum, sum of squares) of each stored row, WRITTEN
 * (not accumulated) -- the statistics the first folded LayerNorm consumes.  ids: int64 [batch, seq]; ids outside [0, vocab) are an
 * error the kernel reports by writing zeros for that row. */
int sfb_embed_tokens(const int64_t* ids, const void* tok_emb, const void* pos_emb, void* out, float* rowstats,
                     int32_t rowstats_slots, int32_t batch, int32_t seq, int32_t dim, int32_t vocab, int32_t ld_out,
                     int32_t dtype, sfb_stream_t stream);

/* pooled[b, :] = x[b * seq + p_b, :], p_b = first position whose id equals eos_id, or (eos_id == 2, the
 * legacy CLIP config) the position of the largest id -- transformers' CLIPTextTransformer pooling rule. */
int sfb_clip_pool(const int64_t* ids, const void* x, void* pooled, int32_t batch, int32_t seq, int32_t dim,
                  int32_t ld_x, int32_t eos_id, sfb_stream_t stream);

/* CLIP vision tower (SVD image_encoder, reference :100-103): non-overlapping patch x patch blocks of an NCHW
 * 16-bit image as rows of a GEMM A operand: a[(b, py, px), (c, i, j)] = x[b, c, py*patch + i, px*patch + j],
 * row pitch kpad (a multiple of 64 for the GEMM), columns beyond chans * patch^2 zeroed. */
int sfb_patchify(const void* x, void* a, int32_t batch, int32_t chans, int32_t h, int32_t w, int32_t patch,
                 int32_t kpad, sfb_stream_t stream);

/* ---- LoRA adapters (PEFT LoraLayer, merged into the weights when the adapter state changes; the
 * reference's recipe is fuse_lora() on the module before compiling) ------------------------------ */

#define SFB_LORA_MAX_ADAPTERS 8
#define SFB_LORA_MAX_RANK 256

/* One adapter: A [rank, k] (row pitch lda), B [n, rank] (row pitch ldb), each SFB_F16 / SFB_BF16 /
 * SFB_F32 independently of W; `scale` is PEFT's scaling[adapter] times any call-time factor. */
typedef struct sfb_lora_adapter {
    const void* a;
    const void* b;
    int32_t rank, lda, ldb, a_dtype, b_dtype;
    float scale;
} sfb_lora_adapter;

/* out[n, k] = round(W[n, k] + sum_i scale_i * sum_j B_i[n, j] A_i[j, k]), fp32 arithmetic and ONE rounding
 * to out_dtype (SFB_F16 / SFB_BF16) at the end.  W [n, k] (row pitch ldw) is SFB_F16 / SFB_BF16 / SFB_F32;
 * out (row pitch ldo) is caller-owned and must not alias W, A or B.  A conv weight [cout, cin, kh, kw] is
 * W [cout, cin*kh*kw] with A the lora_A conv weight [rank, cin*kh*kw] (OIHW order) and B the 1x1 lora_B
 * weight [cout, rank].  1 <= count <= SFB_LORA_MAX_ADAPTERS, 1 <= rank <= SFB_LORA_MAX_RANK. */
typedef struct sfb_lora_merge_params {
    const void* w;
    void* out;
    int32_t n, k, ldw, ldo, w_dtype, out_dtype;
    int32_t count;
    sfb_lora_adapter adapters[SFB_LORA_MAX_ADAPTERS];
} sfb_lora_merge_params;

int sfb_lora_merge(const sfb_lora_merge_params* p, sfb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* SFB200_H_ */
