// Small kernels at the edges of the UNet: sinusoidal timestep embedding, batch-row linears
// (time-embedding MLP and all per-resnet time projections: weight-bandwidth-bound GEMV-like work,
// one warp per output column), the 4-channel conv_in / conv_out, nearest-neighbour upsampling.
// These are the ops the reference leaves as plain aten kernels in its traced graph
// (SURVEY.md section 8a, rows a6 (M = batch linears) and a11).
#include "common.cuh"
#include "host.h"

namespace sfb {

// ---------------------------------------------------------------------------------------
// timestep embedding (diffusers get_timestep_embedding; fp32 math, 16-bit output)
// ---------------------------------------------------------------------------------------
__global__ void timestep_embed_kernel(const float* __restrict__ t, int batch, int half, int flip,
                                      float freq_shift, void* out, int ldo, int dtype) {
    pdl_launch_dependents();
    pdl_wait();
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= batch * half) return;
    const int b = idx / half, i = idx - b * half;
    const float freq = expf(-9.210340371976184f * (float)i / ((float)half - freq_shift));
    const float arg = t[b] * freq;
    const float s = sinf(arg), c = cosf(arg);
    const size_t row = (size_t)b * ldo;
    if (flip) {
        store1(out, row + i, c, dtype);
        store1(out, row + half + i, s, dtype);
    } else {
        store1(out, row + i, s, dtype);
        store1(out, row + half + i, c, dtype);
    }
}

// ---------------------------------------------------------------------------------------
// batch-row linear: one warp per output column, up to 8 batch rows per pass
// ---------------------------------------------------------------------------------------
struct SmallLinearArgs {
    const uint16_t* x;
    const uint16_t* w;
    const float* bias;
    const uint16_t* add16;
    uint16_t* y16;
    float* y32;
    int batch, n, k, ldx, ldy, act_in, act_out, dtype;
};

__global__ void __launch_bounds__(256) small_linear_kernel(const SmallLinearArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    const int col = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    const int b0 = blockIdx.y * 8;
    if (col >= a.n) return;
    const int nb = min(8, a.batch - b0);
    float acc[8];
#pragma unroll
    for (int b = 0; b < 8; ++b) acc[b] = 0.f;
    const uint16_t* wr = a.w + (size_t)col * a.k;
    for (int kv = lane; kv < a.k / 8; kv += 32) {
        const uint4 wv = *reinterpret_cast<const uint4*>(wr + kv * 8);
        const uint32_t ww[4] = {wv.x, wv.y, wv.z, wv.w};
        float wf[8];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 f = unpack2(ww[i], a.dtype);
            wf[2 * i] = f.x; wf[2 * i + 1] = f.y;
        }
#pragma unroll
        for (int b = 0; b < 8; ++b) {
            if (b < nb) {
                const uint4 xv = *reinterpret_cast<const uint4*>(a.x + (size_t)(b0 + b) * a.ldx + kv * 8);
                const uint32_t xw[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    float2 f = unpack2(xw[i], a.dtype);
                    if (a.act_in) { f.x = silu_f(f.x); f.y = silu_f(f.y); }
                    acc[b] += f.x * wf[2 * i] + f.y * wf[2 * i + 1];
                }
            }
        }
    }
#pragma unroll
    for (int b = 0; b < 8; ++b) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[b] += __shfl_xor_sync(0xffffffffu, acc[b], o);
    }
    if (lane == 0) {
        for (int b = 0; b < nb; ++b) {
            float v = acc[b] + (a.bias ? a.bias[col] : 0.f);
            const size_t o = (size_t)(b0 + b) * a.ldy + col;
            // add16 is a contiguous [batch, n] tensor (sfb200.h), not laid out at the output pitch
            if (a.add16) v += load1(a.add16, (size_t)(b0 + b) * a.n + col, a.dtype);
            if (a.act_out) v = silu_f(v);
            if (a.y32) a.y32[o] = v;
            if (a.y16) store1(a.y16, o, v, a.dtype);
        }
    }
}

// ---------------------------------------------------------------------------------------
// conv_in: NCHW (cin <= 8) -> NHWC, 3x3 pad 1.  Weights arrive pre-transposed as
// [9*cin][cout] (tap-major, cout contiguous) and are staged in smem with 16-byte copies.
// thread = (pixel slot, group of 8 output channels)
// ---------------------------------------------------------------------------------------
struct ConvEdgeArgs {
    const uint16_t* x;
    const uint16_t* w;
    const float* bias;
    uint16_t* y;
    int n, h, wd, cin, cout, ld, dtype;
};

constexpr int kConvInPixelsPerBlock = 24;

__global__ void __launch_bounds__(256) conv_in_kernel(const ConvEdgeArgs a) {
    extern __shared__ uint16_t wsm[];  // [9*cin][cout]
    pdl_launch_dependents();
    pdl_wait();
    const int kk = 9 * a.cin;
    for (int i = threadIdx.x; i < (kk * a.cout) / 8; i += blockDim.x)
        reinterpret_cast<uint4*>(wsm)[i] = reinterpret_cast<const uint4*>(a.w)[i];
    __syncthreads();
    const int ngroups = a.cout / 8;
    const int slots = blockDim.x / ngroups;
    const int g = threadIdx.x % ngroups;
    const int slot = threadIdx.x / ngroups;
    if (slot >= slots) return;
    const int total = a.n * a.h * a.wd;
    const int p0 = blockIdx.x * kConvInPixelsPerBlock;
    for (int p = p0 + slot; p < min(p0 + kConvInPixelsPerBlock, total); p += slots) {
        const int xw = p % a.wd;
        const int yh = (p / a.wd) % a.h;
        const int img = p / (a.wd * a.h);
        float acc[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = a.bias ? a.bias[g * 8 + i] : 0.f;
        // gather the 9 * cin inputs first (independent loads), then do the FMAs
        float xin[9 * 8];
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const int iy = yh + tap / 3 - 1, ix = xw + tap % 3 - 1;
            const bool ok = iy >= 0 && iy < a.h && ix >= 0 && ix < a.wd;
#pragma unroll
            for (int ci = 0; ci < 8; ++ci)
                xin[tap * 8 + ci] = (ok && ci < a.cin)
                    ? load1(a.x, (((size_t)img * a.cin + ci) * a.h + iy) * a.wd + ix, a.dtype) : 0.f;
        }
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
#pragma unroll
            for (int ci = 0; ci < 8; ++ci) {
                if (ci < a.cin) {
                    const int j = tap * a.cin + ci;
                    const uint4 wv = *reinterpret_cast<const uint4*>(&wsm[j * a.cout + g * 8]);
                    const uint32_t ww[4] = {wv.x, wv.y, wv.z, wv.w};
                    const float xv = xin[tap * 8 + ci];
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const float2 f = unpack2(ww[i], a.dtype);
                        acc[2 * i] += xv * f.x;
                        acc[2 * i + 1] += xv * f.y;
                    }
                }
            }
        }
        uint4 o;
        o.x = pack2(acc[0], acc[1], a.dtype); o.y = pack2(acc[2], acc[3], a.dtype);
        o.z = pack2(acc[4], acc[5], a.dtype); o.w = pack2(acc[6], acc[7], a.dtype);
        *reinterpret_cast<uint4*>(a.y + (size_t)p * a.ld + g * 8) = o;
    }
}


// ---------------------------------------------------------------------------------------
// im2col for the UNet's first convolution (cin <= 7: K = 9*cin <= 63): NCHW input ->
// A[pixels, 64] (K zero-padded to one 64-wide K block), so conv_in runs on the wgmma GEMM with
// its fused bias epilogue writing NHWC straight into the first skip-concat slice.
// One thread per output pixel; loads are coalesced along w, each thread writes one 128-byte row.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) im2col_in_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ a,
                                                        int n, int h, int w, int cin) {
    pdl_launch_dependents();
    pdl_wait();
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n * h * w) return;
    const int xw = p % w;
    const int yh = (p / w) % h;
    const int img = p / (w * h);
    uint16_t row[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) row[i] = 0;
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
        const int iy = yh + tap / 3 - 1, ix = xw + tap % 3 - 1;
        const bool ok = iy >= 0 && iy < h && ix >= 0 && ix < w;
#pragma unroll
        for (int ci = 0; ci < 7; ++ci) {
            if (ci < cin && ok) row[tap * cin + ci] = x[(((size_t)img * cin + ci) * h + iy) * w + ix];
        }
    }
    uint4* dst = reinterpret_cast<uint4*>(a + (size_t)p * 64);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        uint4 v;
        v.x = row[i * 8 + 0] | ((uint32_t)row[i * 8 + 1] << 16);
        v.y = row[i * 8 + 2] | ((uint32_t)row[i * 8 + 3] << 16);
        v.z = row[i * 8 + 4] | ((uint32_t)row[i * 8 + 5] << 16);
        v.w = row[i * 8 + 6] | ((uint32_t)row[i * 8 + 7] << 16);
        dst[i] = v;
    }
}

// ---------------------------------------------------------------------------------------
// im2col for a wide first convolution (9 <= cin <= 14: K = 9*cin <= 126, e.g. the inpainting
// UNets' 9 channels): NCHW input -> A[pixels, 128] (K zero-padded to two 64-wide K blocks).
// One thread per output pixel.  Each output column's (tap, ci) is carried along the unrolled
// column loop, so every register index is a compile-time constant (no local-memory row array).
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) im2col_in_wide_kernel(const uint16_t* __restrict__ x,
                                                             uint16_t* __restrict__ a, int n, int h, int w,
                                                             int cin) {
    pdl_launch_dependents();
    pdl_wait();
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n * h * w) return;
    const int xw = p % w;
    const int yh = (p / w) % h;
    const int img = p / (w * h);
    const size_t plane = (size_t)h * w;
    const uint16_t* xi = x + (size_t)img * cin * plane;
    uint4* dst = reinterpret_cast<uint4*>(a + (size_t)p * 128);
    int tap = 0, ci = 0;
#pragma unroll
    for (int v = 0; v < 16; ++v) {
        uint32_t word[4];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            uint32_t val = 0;
            if (tap < 9) {
                const int iy = yh + tap / 3 - 1, ix = xw + tap % 3 - 1;
                if (iy >= 0 && iy < h && ix >= 0 && ix < w) val = xi[ci * plane + (size_t)iy * w + ix];
            }
            if (e & 1) word[e >> 1] |= val << 16;
            else word[e >> 1] = val;
            if (++ci == cin) { ci = 0; ++tap; }
        }
        dst[v] = make_uint4(word[0], word[1], word[2], word[3]);
    }
}

// ---------------------------------------------------------------------------------------
// conv_out: NHWC (pitch ld) -> NCHW (cout <= 8), 3x3 pad 1.  One warp per output pixel; lanes
// split the 9 * cin/8 (tap, 8-channel vector) items; weights [cout][9][cin] staged in smem.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void conv_out_stage_weights(const ConvEdgeArgs& a, uint16_t* wsm) {
    for (int i = threadIdx.x; i < (9 * a.cin * a.cout) / 8; i += blockDim.x)
        reinterpret_cast<uint4*>(wsm)[i] = reinterpret_cast<const uint4*>(a.w)[i];
}

// The conv of pixel (yh, xw) of image img without bias, summed over the warp: every lane holds all
// cout sums (a butterfly reduction gives every lane the same bits).
__device__ __forceinline__ void conv_out_pixel(const ConvEdgeArgs& a, const uint16_t* wsm, int img, int yh, int xw,
                                               int lane, float (&acc)[8]) {
    const int kk = 9 * a.cin;
    const int nvec = a.cin / 8;
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    for (int it = lane; it < 9 * nvec; it += 32) {
        const int tap = it / nvec, vec = it - tap * nvec;
        const int iy = yh + tap / 3 - 1, ix = xw + tap % 3 - 1;
        if (iy < 0 || iy >= a.h || ix < 0 || ix >= a.wd) continue;
        const uint4 xv = *reinterpret_cast<const uint4*>(
            a.x + (((size_t)img * a.h + iy) * a.wd + ix) * a.ld + vec * 8);
        const uint32_t xw4[4] = {xv.x, xv.y, xv.z, xv.w};
        float xf[8];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 f = unpack2(xw4[i], a.dtype);
            xf[2 * i] = f.x; xf[2 * i + 1] = f.y;
        }
#pragma unroll
        for (int co = 0; co < 8; ++co) {
            if (co < a.cout) {
                const uint4 wv = *reinterpret_cast<const uint4*>(&wsm[co * kk + tap * a.cin + vec * 8]);
                const uint32_t ww[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float2 f = unpack2(ww[i], a.dtype);
                    acc[co] += xf[2 * i] * f.x + xf[2 * i + 1] * f.y;
                }
            }
        }
    }
#pragma unroll
    for (int co = 0; co < 8; ++co) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[co] += __shfl_xor_sync(0xffffffffu, acc[co], o);
    }
}

__global__ void __launch_bounds__(256) conv_out_kernel(const ConvEdgeArgs a) {
    extern __shared__ uint16_t wsm[];  // [cout][9*cin]
    pdl_launch_dependents();
    pdl_wait();
    conv_out_stage_weights(a, wsm);
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int total = a.n * a.h * a.wd;
    for (int p = blockIdx.x * 8 + (threadIdx.x >> 5); p < total; p += gridDim.x * 8) {
        const int xw = p % a.wd;
        const int yh = (p / a.wd) % a.h;
        const int img = p / (a.wd * a.h);
        float acc[8];
        conv_out_pixel(a, wsm, img, yh, xw, lane, acc);
        if (lane < a.cout) {
            float v = 0.f;
#pragma unroll
            for (int co = 0; co < 8; ++co) if (lane == co) v = acc[co];
            v += a.bias ? a.bias[lane] : 0.f;
            store1(a.y, (((size_t)img * a.cout + lane) * a.h + yh) * a.wd + xw, v, a.dtype);
        }
    }
}

// ---------------------------------------------------------------------------------------
// conv_out + time_conv_out of SVD's temporal VAE decoder: the 3x3 conv above, rounded to 16 bits,
// then a Conv3d (3,1,1) with zero padding over the frames of each video.  One warp per output
// pixel of a video walks its frames with a three-frame window (previous, current, next conv_out
// values, all lanes holding all channels), so every conv_out value is computed once and never
// leaves registers.  The images of a.n are videos of `frames` consecutive frames.
// ---------------------------------------------------------------------------------------
struct ConvOutTemporalArgs {
    ConvEdgeArgs e;
    const uint16_t* wt;  // [cout][3][cout] 16-bit: output channel, frame tap, input channel
    const float* bt;
    int frames;
};

__device__ __forceinline__ void conv_out_frame(const ConvEdgeArgs& a, const uint16_t* wsm, int img, int yh, int xw,
                                               int lane, float (&c)[8]) {
    conv_out_pixel(a, wsm, img, yh, xw, lane, c);
#pragma unroll
    for (int co = 0; co < 8; ++co) {
        // rounded to the storage type, as diffusers stores conv_out's output before time_conv_out
        const float v = c[co] + (co < a.cout && a.bias ? a.bias[co] : 0.f);
        c[co] = unpack2(pack2(v, 0.f, a.dtype), a.dtype).x;
    }
}

__global__ void __launch_bounds__(256) conv_out_temporal_kernel(const ConvOutTemporalArgs t) {
    extern __shared__ uint16_t wsm[];  // [cout][9*cin]
    __shared__ float wts[8 * 3 * 8];   // [cout][3][cout]
    const ConvEdgeArgs& a = t.e;
    pdl_launch_dependents();
    pdl_wait();
    conv_out_stage_weights(a, wsm);
    for (int i = threadIdx.x; i < a.cout * 3 * a.cout; i += blockDim.x) wts[i] = load1(t.wt, i, a.dtype);
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const int hw = a.h * a.wd;
    const int total = (a.n / t.frames) * hw;  // (video, pixel) pairs
    for (int q = blockIdx.x * 8 + (threadIdx.x >> 5); q < total; q += gridDim.x * 8) {
        const int vid = q / hw, pix = q - vid * hw;
        const int yh = pix / a.wd, xw = pix - yh * a.wd;
        const int img0 = vid * t.frames;
        float prev[8], cur[8], next[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) prev[i] = 0.f;  // frame -1: zero padding
        conv_out_frame(a, wsm, img0, yh, xw, lane, cur);
        for (int f = 0; f < t.frames; ++f) {
            if (f + 1 < t.frames) {
                conv_out_frame(a, wsm, img0 + f + 1, yh, xw, lane, next);
            } else {
#pragma unroll
                for (int i = 0; i < 8; ++i) next[i] = 0.f;  // frame F: zero padding
            }
            if (lane < a.cout) {
                const float* wr = wts + lane * 3 * a.cout;
                float v = t.bt ? t.bt[lane] : 0.f;
#pragma unroll
                for (int ci = 0; ci < 8; ++ci) {
                    if (ci < a.cout)
                        v += wr[ci] * prev[ci] + wr[a.cout + ci] * cur[ci] + wr[2 * a.cout + ci] * next[ci];
                }
                store1(a.y, ((size_t)(img0 + f) * a.cout + lane) * hw + pix, v, a.dtype);
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) { prev[i] = cur[i]; cur[i] = next[i]; }
        }
    }
}

// ---------------------------------------------------------------------------------------
// nearest-neighbour 2x upsample, NHWC, 16-byte vectors
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) upsample2x_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ y,
                                                         int n, int h, int w, int nvec, int ldx, int ldy) {
    pdl_launch_dependents();
    pdl_wait();
    const long long total = (long long)n * 2 * h * 2 * w * nvec;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int vec = (int)(idx % nvec);
        long long p = idx / nvec;
        const int ox = (int)(p % (2 * w)); p /= (2 * w);
        const int oy = (int)(p % (2 * h));
        const int img = (int)(p / (2 * h));
        const uint4 v = *reinterpret_cast<const uint4*>(
            x + (((size_t)img * h + oy / 2) * w + ox / 2) * ldx + vec * 8);
        *reinterpret_cast<uint4*>(y + (((size_t)img * 2 * h + oy) * 2 * w + ox) * ldy + vec * 8) = v;
    }
}


// ---------------------------------------------------------------------------------------
// ControlNet residuals: dst[n, hw, c] (NHWC slice, channel pitch ld) += src[n, c, hw] (NCHW) for
// up to 16 tensors in ONE launch (diffusers adds `down_block_additional_residuals` to the 12 skip
// tensors and `mid_block_additional_residual` to the mid-block output).  32 x 32 (pixel, channel)
// tiles transposed through shared memory: reads coalesced along hw, writes along c.
// ---------------------------------------------------------------------------------------
struct AddNchwArgs {
    int count, dtype;
    const uint16_t* src[16];
    uint16_t* dst[16];
    int n[16], c[16], hw[16], ld[16];
    int tile_end[16];  // exclusive prefix of 32x32 tiles per item
};

__global__ void __launch_bounds__(256) add_nchw_kernel(const AddNchwArgs a) {
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
    const uint16_t* src = a.src[it] + (size_t)img * c * hw;
    uint16_t* dst = a.dst[it] + (size_t)img * hw * ld;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int ch = c0 + ty + 8 * j, px = p0 + tx;
        tile[ty + 8 * j][tx] = (ch < c && px < hw) ? load1(src, (size_t)ch * hw + px, a.dtype) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int px = p0 + ty + 8 * j, ch = c0 + tx;
        if (ch < c && px < hw) {
            const size_t o = (size_t)px * ld + ch;
            store1(dst, o, load1(dst, o, a.dtype) + tile[tx][ty + 8 * j], a.dtype);
        }
    }
}

// dst[r, 0:cols] = src[r, 0:cols] (16-bit, arbitrary pitches): the one strided copy a plan needs
// (SDXL: time-id sinusoids behind text_embeds in the add-embedding input row)
__global__ void copy2d_kernel(const uint16_t* __restrict__ src, uint16_t* __restrict__ dst, int rows,
                              int cols, int lds, int ldd) {
    pdl_launch_dependents();
    pdl_wait();
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx < rows * cols) {
        const int r = idx / cols, c = idx - r * cols;
        dst[(size_t)r * ldd + c] = src[(size_t)r * lds + c];
    }
}

// row softmax: one CTA per row, the row (<= 16384 columns) held in registers; y may alias x
template <bool kF32>
__global__ void __launch_bounds__(256) row_softmax_kernel(const void* x, uint16_t* y, int rows, int cols, int ldx,
                                                          int ldy, int dtype) {
    __shared__ float red[8];
    pdl_launch_dependents();
    pdl_wait();
    const int nvec = cols / 8;
    constexpr int kMaxVec = 8;  // 8 vectors x 8 values x 256 threads = 16384 columns
    float v[kMaxVec][8];
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < kMaxVec; ++j) {
        const int vec = threadIdx.x + j * 256;
        if (vec < nvec) {
            if (kF32) {
                const float* xr = reinterpret_cast<const float*>(x) + (size_t)blockIdx.x * ldx + vec * 8;
                const float4 a = *reinterpret_cast<const float4*>(xr), b = *reinterpret_cast<const float4*>(xr + 4);
                v[j][0] = a.x; v[j][1] = a.y; v[j][2] = a.z; v[j][3] = a.w;
                v[j][4] = b.x; v[j][5] = b.y; v[j][6] = b.z; v[j][7] = b.w;
            } else {
                const uint16_t* xr = reinterpret_cast<const uint16_t*>(x) + (size_t)blockIdx.x * ldx + vec * 8;
                const uint4 u = *reinterpret_cast<const uint4*>(xr);
                const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float2 f = unpack2(w[i], dtype);
                    v[j][2 * i] = f.x; v[j][2 * i + 1] = f.y;
                }
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) mx = fmaxf(mx, v[j][i]);
        }
    }
    auto block_reduce = [&](float val, bool is_max) -> float {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float other = __shfl_xor_sync(0xffffffffu, val, o);
            val = is_max ? fmaxf(val, other) : val + other;
        }
        __syncthreads();
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = val;
        __syncthreads();
        float r = red[0];
#pragma unroll
        for (int i = 1; i < 8; ++i) r = is_max ? fmaxf(r, red[i]) : r + red[i];
        return r;
    };
    mx = block_reduce(mx, true);  // (its barriers also order every read of the row before any write)
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < kMaxVec; ++j) {
        if (threadIdx.x + j * 256 < nvec) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                v[j][i] = __expf(v[j][i] - mx);
                sum += v[j][i];
            }
        }
    }
    const float inv = 1.0f / block_reduce(sum, false);
    uint16_t* yr = y + (size_t)blockIdx.x * ldy;
#pragma unroll
    for (int j = 0; j < kMaxVec; ++j) {
        const int vec = threadIdx.x + j * 256;
        if (vec < nvec) {
            uint4 o;
            o.x = pack2(v[j][0] * inv, v[j][1] * inv, dtype);
            o.y = pack2(v[j][2] * inv, v[j][3] * inv, dtype);
            o.z = pack2(v[j][4] * inv, v[j][5] * inv, dtype);
            o.w = pack2(v[j][6] * inv, v[j][7] * inv, dtype);
            *reinterpret_cast<uint4*>(yr + vec * 8) = o;
        }
    }
}

__global__ void pointwise_nchw_kernel(const uint16_t* __restrict__ x, const uint16_t* __restrict__ w,
                                      const float* __restrict__ bias, uint16_t* __restrict__ y, int n, int hw,
                                      int cin, int cout, int dtype) {
    pdl_launch_dependents();
    pdl_wait();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)n * hw) return;
    const int img = (int)(idx / hw), p = (int)(idx % hw);
    float xin[8];
    for (int ci = 0; ci < cin; ++ci) xin[ci] = load1(x, ((size_t)img * cin + ci) * hw + p, dtype);
    for (int co = 0; co < cout; ++co) {
        float acc = bias ? bias[co] : 0.f;
        for (int ci = 0; ci < cin; ++ci) acc += load1(w, (size_t)co * cin + ci, dtype) * xin[ci];
        store1(y, ((size_t)img * cout + co) * hw + p, acc, dtype);
    }
}

}  // namespace sfb

using namespace sfb;

extern "C" int sfb_row_softmax(const void* x, void* y, int32_t rows, int32_t cols, int32_t ldx, int32_t ldy,
                               int32_t x_is_f32, int32_t dtype, sfb_stream_t stream) {
    if (!x || !y || rows <= 0 || cols <= 0 || cols % 8 || ldx % 8 || ldy % 8 || cols > 16384 || ldx < cols || ldy < cols)
        return fail(SFB_ERR_INVALID, "row_softmax: cols=%d must be a multiple of 8 and <= 16384", cols);
    cudaError_t err = x_is_f32
        ? launch_pdl(row_softmax_kernel<true>, dim3(rows), dim3(256), 0, static_cast<cudaStream_t>(stream), x,
                     reinterpret_cast<uint16_t*>(y), rows, cols, ldx, ldy, dtype)
        : launch_pdl(row_softmax_kernel<false>, dim3(rows), dim3(256), 0, static_cast<cudaStream_t>(stream), x,
                     reinterpret_cast<uint16_t*>(y), rows, cols, ldx, ldy, dtype);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "row_softmax: %s", cudaGetErrorString(err));
    return check_launch("sfb_row_softmax");
}

extern "C" int sfb_pointwise_nchw(const void* x, const void* w, const float* bias, void* y, int32_t n, int32_t hw,
                                  int32_t cin, int32_t cout, int32_t dtype, sfb_stream_t stream) {
    if (!x || !w || !y || n <= 0 || hw <= 0 || cin <= 0 || cin > 8 || cout <= 0 || cout > 8)
        return fail(SFB_ERR_INVALID, "pointwise_nchw: cin / cout must be 1..8");
    const long long total = (long long)n * hw;
    cudaError_t err = launch_pdl(pointwise_nchw_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0,
                                 static_cast<cudaStream_t>(stream), reinterpret_cast<const uint16_t*>(x),
                                 reinterpret_cast<const uint16_t*>(w), bias, reinterpret_cast<uint16_t*>(y), n, hw,
                                 cin, cout, dtype);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "pointwise_nchw: %s", cudaGetErrorString(err));
    return check_launch("sfb_pointwise_nchw");
}

extern "C" int sfb_add_nchw_residuals(const sfb_add_nchw_params* p, sfb_stream_t stream) {
    if (!p || p->count <= 0 || p->count > 16) return fail(SFB_ERR_INVALID, "add_nchw_residuals: count must be 1..16");
    AddNchwArgs a{};
    a.count = p->count; a.dtype = p->dtype;
    int tiles = 0;
    for (int i = 0; i < p->count; ++i) {
        const sfb_add_nchw_item& it = p->items[i];
        if (!it.src || !it.dst || it.n <= 0 || it.c <= 0 || it.hw <= 0 || it.ld_dst < it.c)
            return fail(SFB_ERR_INVALID, "add_nchw_residuals: bad item %d", i);
        a.src[i] = reinterpret_cast<const uint16_t*>(it.src);
        a.dst[i] = reinterpret_cast<uint16_t*>(it.dst);
        a.n[i] = it.n; a.c[i] = it.c; a.hw[i] = it.hw; a.ld[i] = it.ld_dst;
        tiles += it.n * ((it.c + 31) / 32) * ((it.hw + 31) / 32);
        a.tile_end[i] = tiles;
    }
    cudaError_t err = launch_pdl(add_nchw_kernel, dim3(tiles), dim3(256), 0, static_cast<cudaStream_t>(stream), a);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "add_nchw_residuals: %s", cudaGetErrorString(err));
    return check_launch("sfb_add_nchw_residuals");
}

extern "C" int sfb_copy2d(const void* src, void* dst, int32_t rows, int32_t cols, int32_t ld_src,
                          int32_t ld_dst, sfb_stream_t stream) {
    if (!src || !dst || rows <= 0 || cols <= 0 || ld_src < cols || ld_dst < cols)
        return fail(SFB_ERR_INVALID, "copy2d: bad argument");
    const int total = rows * cols;
    cudaError_t err = launch_pdl(copy2d_kernel, dim3((total + 255) / 256), dim3(256), 0,
                                 static_cast<cudaStream_t>(stream), reinterpret_cast<const uint16_t*>(src),
                                 reinterpret_cast<uint16_t*>(dst), rows, cols, ld_src, ld_dst);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "copy2d: %s", cudaGetErrorString(err));
    return check_launch("sfb_copy2d");
}

extern "C" int sfb_timestep_embed(const float* t, int32_t batch, int32_t dim, int32_t flip,
                                  float freq_shift, void* out, int32_t ldo, int32_t dtype,
                                  sfb_stream_t stream) {
    if (!t || !out) return fail(SFB_ERR_INVALID, "timestep_embed: null argument");
    if (dim <= 0 || dim % 2 || batch <= 0 || ldo < dim)
        return fail(SFB_ERR_INVALID, "timestep_embed: dim=%d must be even and positive, batch=%d positive, ldo=%d >= dim",
                    dim, batch, ldo);
    const int half = dim / 2;
    const int total = batch * half;
    cudaError_t err = launch_pdl(timestep_embed_kernel, dim3((total + 127) / 128), dim3(128), 0,
                                 static_cast<cudaStream_t>(stream), t, batch, half, flip, freq_shift,
                                 out, ldo, dtype);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "timestep_embed: %s", cudaGetErrorString(err));
    return check_launch("sfb_timestep_embed");
}

extern "C" int sfb_small_linear(const sfb_small_linear_params* p, sfb_stream_t stream) {
    if (!p || !p->x || !p->w || (!p->y16 && !p->y32)) return fail(SFB_ERR_INVALID, "small_linear: null argument");
    if (p->k % 8 || p->ldx % 8 || p->batch <= 0 || p->n <= 0)
        return fail(SFB_ERR_INVALID, "small_linear: k=%d and ldx=%d must be multiples of 8 (batch=%d n=%d)", p->k,
                    p->ldx, p->batch, p->n);
    SmallLinearArgs a{};
    a.x = reinterpret_cast<const uint16_t*>(p->x);
    a.w = reinterpret_cast<const uint16_t*>(p->w);
    a.bias = p->bias; a.add16 = reinterpret_cast<const uint16_t*>(p->add16);
    a.y16 = reinterpret_cast<uint16_t*>(p->y16); a.y32 = p->y32;
    a.batch = p->batch; a.n = p->n; a.k = p->k; a.ldx = p->ldx; a.ldy = p->ldy;
    a.act_in = p->act_in; a.act_out = p->act_out; a.dtype = p->dtype;
    dim3 grid((p->n + 7) / 8, (p->batch + 7) / 8);
    cudaError_t err = launch_pdl(small_linear_kernel, grid, dim3(256), 0,
                                 static_cast<cudaStream_t>(stream), a);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "small_linear: %s", cudaGetErrorString(err));
    return check_launch("sfb_small_linear");
}

extern "C" int sfb_conv_in(const void* x, const void* w, const float* bias, void* y, int32_t n,
                           int32_t h, int32_t wd, int32_t cin, int32_t cout, int32_t ldy,
                           int32_t dtype, sfb_stream_t stream) {
    if (!x || !w || !y || cin <= 0 || cin > 8 || cout % 8 || cout / 8 > 256 || ldy % 8)
        return fail(SFB_ERR_INVALID, "conv_in: unsupported geometry cin=%d cout=%d", cin, cout);
    const size_t smem = (size_t)9 * cin * cout * 2;
    if (smem > 48 * 1024) return fail(SFB_ERR_INVALID, "conv_in: weights exceed 48 KB of shared memory");
    ConvEdgeArgs a{reinterpret_cast<const uint16_t*>(x), reinterpret_cast<const uint16_t*>(w), bias,
                   reinterpret_cast<uint16_t*>(y), n, h, wd, cin, cout, ldy, dtype};
    const int total = n * h * wd;
    cudaError_t err = launch_pdl(conv_in_kernel,
                                 dim3((total + kConvInPixelsPerBlock - 1) / kConvInPixelsPerBlock),
                                 dim3(256), smem, static_cast<cudaStream_t>(stream), a);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "conv_in: %s", cudaGetErrorString(err));
    return check_launch("sfb_conv_in");
}

extern "C" int sfb_im2col_in(const void* x, void* a, int32_t n, int32_t h, int32_t wd, int32_t cin,
                             sfb_stream_t stream) {
    if (!x || !a || cin <= 0 || cin > 7) return fail(SFB_ERR_INVALID, "im2col_in: cin=%d must be 1..7", cin);
    const int total = n * h * wd;
    cudaError_t err = launch_pdl(im2col_in_kernel, dim3((total + 127) / 128), dim3(128), 0,
                                 static_cast<cudaStream_t>(stream), reinterpret_cast<const uint16_t*>(x),
                                 reinterpret_cast<uint16_t*>(a), n, h, wd, cin);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "im2col_in: %s", cudaGetErrorString(err));
    return check_launch("sfb_im2col_in");
}

extern "C" int sfb_im2col_in_wide(const void* x, void* a, int32_t n, int32_t h, int32_t wd, int32_t cin,
                                  sfb_stream_t stream) {
    if (!x || !a) return fail(SFB_ERR_INVALID, "im2col_in_wide: null argument");
    if (reinterpret_cast<uintptr_t>(a) & 15) return fail(SFB_ERR_INVALID, "im2col_in_wide: a must be 16-byte aligned");
    if (n <= 0 || h <= 0 || wd <= 0) return fail(SFB_ERR_INVALID, "im2col_in_wide: n=%d h=%d w=%d must be positive",
                                                 n, h, wd);
    if ((int64_t)n * h * wd > INT32_MAX)
        return fail(SFB_ERR_INVALID, "im2col_in_wide: n*h*w=%lld must be below 2^31", (long long)n * h * wd);
    if (cin < 9 || cin > 14) return fail(SFB_ERR_INVALID, "im2col_in_wide: cin=%d must be 9..14", cin);
    const int total = n * h * wd;
    cudaError_t err = launch_pdl(im2col_in_wide_kernel, dim3((total + 127) / 128), dim3(128), 0,
                                 static_cast<cudaStream_t>(stream), reinterpret_cast<const uint16_t*>(x),
                                 reinterpret_cast<uint16_t*>(a), n, h, wd, cin);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "im2col_in_wide: %s", cudaGetErrorString(err));
    return check_launch("sfb_im2col_in_wide");
}

extern "C" int sfb_conv_out(const void* x, const void* w, const float* bias, void* y, int32_t n,
                            int32_t h, int32_t wd, int32_t cin, int32_t cout, int32_t ldx,
                            int32_t dtype, sfb_stream_t stream) {
    if (!x || !w || !y || cout <= 0 || cout > 8 || cin % 8 || ldx % 8)
        return fail(SFB_ERR_INVALID, "conv_out: unsupported geometry cin=%d cout=%d", cin, cout);
    const size_t smem = (size_t)9 * cin * cout * 2;
    // sm_90's per-block opt-in limit: the VAE encoder's conv_out (512 -> 8, 72 KB) needs more than the
    // default 48 KB; launches within 48 KB (the decoder's 128 -> 3) never touch the attribute
    constexpr size_t kSmemOptin = 227 * 1024;
    if (smem > kSmemOptin) return fail(SFB_ERR_INVALID, "conv_out: weights exceed 227 KB of shared memory");
    if (smem > 48 * 1024) {
        static PerDeviceOnce attr_once;
        bool& attr_set = attr_once.flag();
        if (!attr_set) {
            cudaError_t err = cudaFuncSetAttribute(conv_out_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                   (int)kSmemOptin);
            if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "conv_out: smem attribute: %s", cudaGetErrorString(err));
            attr_set = true;
        }
    }
    ConvEdgeArgs a{reinterpret_cast<const uint16_t*>(x), reinterpret_cast<const uint16_t*>(w), bias,
                   reinterpret_cast<uint16_t*>(y), n, h, wd, cin, cout, ldx, dtype};
    const int total = n * h * wd;
    int blocks = (total + 7) / 8;
    if (blocks > 132 * 8) blocks = 132 * 8;
    cudaError_t err = launch_pdl(conv_out_kernel, dim3(blocks), dim3(256), smem,
                                 static_cast<cudaStream_t>(stream), a);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "conv_out: %s", cudaGetErrorString(err));
    return check_launch("sfb_conv_out");
}

extern "C" int sfb_conv_out_temporal(const void* x, const void* w, const float* bias, const void* wt,
                                     const float* bt, void* y, int32_t n, int32_t h, int32_t wd, int32_t cin,
                                     int32_t cout, int32_t ldx, int32_t frames, int32_t dtype,
                                     sfb_stream_t stream) {
    if (!x || !w || !wt || !y || cout <= 0 || cout > 8 || cin <= 0 || cin % 8 || ldx < cin || ldx % 8)
        return fail(SFB_ERR_INVALID, "conv_out_temporal: unsupported geometry cin=%d cout=%d ldx=%d", cin, cout, ldx);
    if (n <= 0 || h <= 0 || wd <= 0 || frames <= 0 || n % frames)
        return fail(SFB_ERR_INVALID, "conv_out_temporal: %d images are not whole videos of %d frames", n, frames);
    if ((long long)(n / frames) * h * wd > INT32_MAX)
        return fail(SFB_ERR_INVALID, "conv_out_temporal: more than 2^31 (video, pixel) pairs");
    const size_t smem = (size_t)9 * cin * cout * 2;
    constexpr size_t kSmemOptin = 227 * 1024 - 8 * 3 * 8 * sizeof(float);
    if (smem > kSmemOptin)
        return fail(SFB_ERR_INVALID, "conv_out_temporal: weights exceed the shared memory limit (227 KB)");
    if (smem > 48 * 1024 - 8 * 3 * 8 * sizeof(float)) {
        static PerDeviceOnce attr_once;
        bool& attr_set = attr_once.flag();
        if (!attr_set) {
            cudaError_t err = cudaFuncSetAttribute(conv_out_temporal_kernel,
                                                   cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemOptin);
            if (err != cudaSuccess)
                return fail(SFB_ERR_CUDA, "conv_out_temporal: smem attribute: %s", cudaGetErrorString(err));
            attr_set = true;
        }
    }
    ConvOutTemporalArgs t{};
    t.e = ConvEdgeArgs{reinterpret_cast<const uint16_t*>(x), reinterpret_cast<const uint16_t*>(w), bias,
                       reinterpret_cast<uint16_t*>(y), n, h, wd, cin, cout, ldx, dtype};
    t.wt = reinterpret_cast<const uint16_t*>(wt);
    t.bt = bt;
    t.frames = frames;
    const long long total = (long long)(n / frames) * h * wd;
    int blocks = (int)((total + 7) / 8);
    if (blocks > 132 * 8) blocks = 132 * 8;
    cudaError_t err = launch_pdl(conv_out_temporal_kernel, dim3(blocks), dim3(256), smem,
                                 static_cast<cudaStream_t>(stream), t);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "conv_out_temporal: %s", cudaGetErrorString(err));
    return check_launch("sfb_conv_out_temporal");
}

extern "C" int sfb_upsample2x(const void* x, void* y, int32_t n, int32_t h, int32_t w, int32_t c,
                              int32_t ldx, int32_t ldy, sfb_stream_t stream) {
    if (!x || !y || c % 8 || ldx % 8 || ldy % 8) return fail(SFB_ERR_INVALID, "upsample2x: bad argument");
    const long long total = (long long)n * 4 * h * w * (c / 8);
    int blocks = (int)((total + 255) / 256);
    if (blocks > 132 * 16) blocks = 132 * 16;
    cudaError_t err = launch_pdl(upsample2x_kernel, dim3(blocks), dim3(256), 0,
                                 static_cast<cudaStream_t>(stream), reinterpret_cast<const uint16_t*>(x),
                                 reinterpret_cast<uint16_t*>(y), n, h, w, c / 8, ldx, ldy);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "upsample2x: %s", cudaGetErrorString(err));
    return check_launch("sfb_upsample2x");
}

// ---------------------------------------------------------------------------------------
// CLIP text encoder edges: token + position embedding gather (with the row statistics of the first
// folded LayerNorm), end-of-text pooling
// ---------------------------------------------------------------------------------------
namespace sfb {

// one warp per token row
__global__ void __launch_bounds__(256) embed_tokens_kernel(const long long* __restrict__ ids,
                                                           const uint16_t* __restrict__ tok,
                                                           const uint16_t* __restrict__ pos, uint16_t* __restrict__ out,
                                                           float* __restrict__ rowstats, int rs_slots, int rows, int seq,
                                                           int nvec, int vocab, int ld_out, int dtype) {
    pdl_launch_dependents();
    pdl_wait();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int row = blockIdx.x * 8 + warp;
    if (row >= rows) return;
    const long long id = ids[row];
    const bool ok = id >= 0 && id < vocab;
    const int s = row % seq;
    const uint4* t = reinterpret_cast<const uint4*>(tok + (size_t)(ok ? id : 0) * nvec * 8);
    const uint4* p = reinterpret_cast<const uint4*>(pos + (size_t)s * nvec * 8);
    float sum = 0.f, sq = 0.f;
    for (int v = lane; v < nvec; v += 32) {
        const uint4 a = t[v], b = p[v];
        const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
        uint32_t o[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 fa = unpack2(aw[i], dtype), fb = unpack2(bw[i], dtype);
            o[i] = ok ? pack2(fa.x + fb.x, fa.y + fb.y, dtype) : 0u;
            const float2 r = unpack2(o[i], dtype);  // statistics of the values as stored
            sum += r.x + r.y;
            sq += r.x * r.x + r.y * r.y;
        }
        *reinterpret_cast<uint4*>(out + (size_t)row * ld_out + v * 8) = make_uint4(o[0], o[1], o[2], o[3]);
    }
    if (rowstats) {
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            sum += __shfl_xor_sync(0xffffffffu, sum, d);
            sq += __shfl_xor_sync(0xffffffffu, sq, d);
        }
        if (lane == 0) {
            rowstats[2 * (size_t)row * rs_slots] = sum;
            rowstats[2 * (size_t)row * rs_slots + 1] = sq;
        }
    }
}

// one warp per batch row: position of the first end-of-text token (or of the first maximal id), then
// the row copy
__global__ void __launch_bounds__(32) clip_pool_kernel(const long long* __restrict__ ids,
                                                       const uint16_t* __restrict__ x, uint16_t* __restrict__ pooled,
                                                       int seq, int nvec, int ld_x, int eos_id) {
    pdl_launch_dependents();
    pdl_wait();
    const int b = blockIdx.x, lane = threadIdx.x;
    long long best = -1;
    int best_pos = 0x7fffffff;
    for (int s = lane; s < seq; s += 32) {
        const long long id = ids[(size_t)b * seq + s];
        const long long key = (eos_id == 2) ? id : (long long)(id == eos_id);
        if (key > best) { best = key; best_pos = s; }  // ascending s: the first maximum of this lane
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        const long long ob = __shfl_xor_sync(0xffffffffu, best, d);
        const int op = __shfl_xor_sync(0xffffffffu, best_pos, d);
        if (ob > best || (ob == best && op < best_pos)) { best = ob; best_pos = op; }
    }
    const uint4* src = reinterpret_cast<const uint4*>(x + ((size_t)b * seq + best_pos) * ld_x);
    uint4* dst = reinterpret_cast<uint4*>(pooled + (size_t)b * nvec * 8);
    for (int v = lane; v < nvec; v += 32) dst[v] = src[v];
}

}  // namespace sfb

extern "C" int sfb_embed_tokens(const int64_t* ids, const void* tok_emb, const void* pos_emb, void* out,
                                float* rowstats, int32_t rowstats_slots, int32_t batch, int32_t seq, int32_t dim,
                                int32_t vocab, int32_t ld_out, int32_t dtype, sfb_stream_t stream) {
    if (!ids || !tok_emb || !pos_emb || !out || batch <= 0 || seq <= 0 || dim <= 0 || dim % 8 || ld_out % 8 ||
        ld_out < dim || vocab <= 0)
        return fail(SFB_ERR_INVALID, "embed_tokens: bad argument (dim=%d ld_out=%d)", dim, ld_out);
    const int rows = batch * seq;
    cudaError_t err = launch_pdl(sfb::embed_tokens_kernel, dim3((rows + 7) / 8), dim3(256), 0,
                                 static_cast<cudaStream_t>(stream), reinterpret_cast<const long long*>(ids),
                                 reinterpret_cast<const uint16_t*>(tok_emb), reinterpret_cast<const uint16_t*>(pos_emb),
                                 reinterpret_cast<uint16_t*>(out), rowstats, rowstats_slots > 0 ? rowstats_slots : 1, rows,
                                 seq, dim / 8, vocab, ld_out, dtype);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "embed_tokens: %s", cudaGetErrorString(err));
    return check_launch("sfb_embed_tokens");
}

extern "C" int sfb_clip_pool(const int64_t* ids, const void* x, void* pooled, int32_t batch, int32_t seq, int32_t dim,
                             int32_t ld_x, int32_t eos_id, sfb_stream_t stream) {
    if (!ids || !x || !pooled || batch <= 0 || seq <= 0 || dim <= 0 || dim % 8 || ld_x % 8 || ld_x < dim)
        return fail(SFB_ERR_INVALID, "clip_pool: bad argument (dim=%d ld_x=%d)", dim, ld_x);
    cudaError_t err = launch_pdl(sfb::clip_pool_kernel, dim3(batch), dim3(32), 0, static_cast<cudaStream_t>(stream),
                                 reinterpret_cast<const long long*>(ids), reinterpret_cast<const uint16_t*>(x),
                                 reinterpret_cast<uint16_t*>(pooled), seq, dim / 8, ld_x, eos_id);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "clip_pool: %s", cudaGetErrorString(err));
    return check_launch("sfb_clip_pool");
}

// ---------------------------------------------------------------------------------------
// CLIP vision tower edge: non-overlapping P x P patches of an NCHW image as GEMM rows
// ---------------------------------------------------------------------------------------
namespace sfb {

// a[(b, py, px), (c, i, j)] = x[b, c, py*P + i, px*P + j]; columns [C*P*P, kpad) are zero.  One thread
// per 8 output columns (one 16-byte store).
__global__ void __launch_bounds__(256) patchify_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ a,
                                                       int batch, int chans, int h, int w, int patch, int kpad) {
    pdl_launch_dependents();
    pdl_wait();
    const int gw = w / patch, gh = h / patch, kv = kpad / 8, k_real = chans * patch * patch;
    const long long total = (long long)batch * gh * gw * kv;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const int v = (int)(idx % kv);
        const long long row = idx / kv;
        const int px = (int)(row % gw), py = (int)((row / gw) % gh), b = (int)(row / ((long long)gw * gh));
        uint16_t o[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const int k = v * 8 + e;
            uint16_t val = 0;
            if (k < k_real) {
                const int c = k / (patch * patch), ij = k - c * patch * patch, i = ij / patch, j = ij - i * patch;
                val = x[(((size_t)b * chans + c) * h + py * patch + i) * w + px * patch + j];
            }
            o[e] = val;
        }
        *reinterpret_cast<uint4*>(a + (size_t)row * kpad + v * 8) = *reinterpret_cast<const uint4*>(o);
    }
}

}  // namespace sfb

extern "C" int sfb_patchify(const void* x, void* a, int32_t batch, int32_t chans, int32_t h, int32_t w, int32_t patch,
                            int32_t kpad, sfb_stream_t stream) {
    if (!x || !a || batch <= 0 || chans <= 0 || patch <= 0 || h % patch || w % patch || kpad % 8 ||
        kpad < chans * patch * patch)
        return fail(SFB_ERR_INVALID, "patchify: bad geometry (h=%d w=%d patch=%d kpad=%d)", h, w, patch, kpad);
    const long long total = (long long)batch * (h / patch) * (w / patch) * (kpad / 8);
    int blocks = (int)((total + 255) / 256);
    if (blocks > 132 * 8) blocks = 132 * 8;
    cudaError_t err = launch_pdl(sfb::patchify_kernel, dim3(blocks), dim3(256), 0, static_cast<cudaStream_t>(stream),
                                 reinterpret_cast<const uint16_t*>(x), reinterpret_cast<uint16_t*>(a), batch, chans, h,
                                 w, patch, kpad);
    if (err != cudaSuccess) return fail(SFB_ERR_CUDA, "patchify: %s", cudaGetErrorString(err));
    return check_launch("sfb_patchify");
}
