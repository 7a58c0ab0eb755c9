"""Launch schedule of the SVD denoiser, diffusers ``UNetSpatioTemporalConditionModel``
(BASELINE.json configs[3]; the reference compiles it generically by tracing,
/root/reference/src/sfast/compilers/diffusion_pipeline_compiler.py:101-103).

The B x F frames are a batch of B*F images for everything spatial (the SD-style resnets, spatial
self-attention, convs: the UNetPlan emitters are reused as they are), and every temporal operator
is expressed on the SAME token-major [B*F*H*W, C] tensors without a single transpose:

  * TemporalResnetBlock: GroupNorm over (F, H, W) per video = the GroupNorm kernels with n = B
    "images" of F*H*W pixels; Conv3d (3,1,1) = the implicit-GEMM conv with three taps along the frame
    axis of the [B, F, H*W, C] view (SFB_A_CONV3X1; TMA zero fill = the temporal padding); the
    AlphaBlender after it is folded into conv2's weights: x_s + (1 - alpha) * conv2(..).
  * TemporalBasicTransformerBlock: its LayerNorm / GEGLU / projections are row-local, so they run on
    the spatial row order with the LayerNorms folded into the GEMMs like everywhere else; only the
    self-attention over the F frames of one (video, pixel) needs the other order, and
    sfb_temporal_attention reads its Q/K/V rows with a stride of H*W rows.
  * cross-attention over ONE context token (SVD conditions on a single image embedding): softmax over
    one key is 1, so attn2(x) = to_out(to_v(ctx)) for every query -- two M = B*F row linears on the
    side stream and a broadcast add (sfb_row_broadcast_add), which also leaves the row statistics of
    the next LayerNorm.  norm2 / to_q / to_k never run.
"""
import ctypes as C

import torch

from . import _lib, ops
from .ops import Act, Op, _ptr
from .plan import UNetPlan, VideoPlanMixin, _JoinOp


class SVDPlan(VideoPlanMixin, UNetPlan):
    def __init__(self, weights, videos, height, width):
        self.nvid = videos
        self.F = weights.spec.num_frames
        self._ctx_vecs = {}
        self._pos_embs = {}
        super().__init__(weights, videos * self.F, height, width, ctx_len=1)

    # --------------------------------------------------------------------------- bookkeeping
    @staticmethod
    def _ln_arena_floats(spec, batch, height, width):
        # spatial + temporal blocks: <= 6 row-statistic slots per depth
        return 2 * UNetPlan._ln_arena_floats(spec, batch, height, width)

    def _alloc_extra_inputs(self):
        spec = self.spec
        self.time_ids_in = self._alloc((self.B * 3,), torch.float32)   # added_time_ids, one row per frame
        self.frame_idx = self._alloc((self.F,), torch.float32)
        if not self.dry:
            self.frame_idx.copy_(torch.arange(self.F, dtype=torch.float32))

    # --------------------------------------------------------------------------- time embedding
    def time_embedding(self):
        """emb = time_embedding(sin(t)) + add_embedding(sin(added_time_ids)); SiLU applied once for
        all consumers; every time_emb_proj (spatial and temporal halves) in one launch."""
        spec, B, lib = self.spec, self.B, self.lib_or_dry()
        self._alloc_extra_inputs()
        c0 = spec.block_out_channels[0]
        t_emb = self.buf("t_emb", (B, c0))
        self._emit(Op("time_proj", lib.sfb_timestep_embed,
                      (_ptr(self.t_in), B, c0, 1, 0.0, _ptr(t_emb), c0, ops.dtype_code(self.dt)),
                      (self.t_in, t_emb)))
        h = self.buf("temb_h", (B, spec.temb_dim))
        self._emit(ops.small_linear_op("time_embedding.linear_1", lib, x=t_emb,
                                       w=self.w.small("time_embedding.linear_1.weight"),
                                       bias=self.w.f32("time_embedding.linear_1.bias"), batch=B,
                                       n=spec.temb_dim, k=c0, dt=self.dt, y16=h, act_out=1))
        emb_t = self.buf("temb_t", (B, spec.temb_dim))
        self._emit(ops.small_linear_op("time_embedding.linear_2", lib, x=h,
                                       w=self.w.small("time_embedding.linear_2.weight"),
                                       bias=self.w.f32("time_embedding.linear_2.bias"), batch=B,
                                       n=spec.temb_dim, k=spec.temb_dim, dt=self.dt, y16=emb_t))
        ad = spec.addition_time_embed_dim
        tid = self.buf("add_tid", (B * 3, ad))  # == [B, 3 * ad] rows: the add_embedding input
        self._emit(Op("add_time_proj", lib.sfb_timestep_embed,
                      (_ptr(self.time_ids_in), B * 3, ad, 1, 0.0, _ptr(tid), ad, ops.dtype_code(self.dt)),
                      (self.time_ids_in, tid)))
        h2 = self.buf("add_h", (B, spec.temb_dim))
        self._emit(ops.small_linear_op("add_embedding.linear_1", lib, x=tid,
                                       w=self.w.small("add_embedding.linear_1.weight"),
                                       bias=self.w.f32("add_embedding.linear_1.bias"), batch=B,
                                       n=spec.temb_dim, k=spec.add_in_dim, dt=self.dt, y16=h2, act_out=1))
        temb_act = self.buf("temb_act", (B, spec.temb_dim))
        self._emit(ops.small_linear_op("add_embedding.linear_2", lib, x=h2,
                                       w=self.w.small("add_embedding.linear_2.weight"),
                                       bias=self.w.f32("add_embedding.linear_2.bias"), batch=B,
                                       n=spec.temb_dim, k=spec.temb_dim, dt=self.dt,
                                       y16=temb_act, add16=emb_t, act_out=1))
        self.temb_proj = self.buf("temb_proj", (B, self.w.tproj_total), torch.float32)
        self._emit(ops.small_linear_op("time_emb_proj(all)", lib, x=temb_act, w=self.w.tproj_w,
                                       bias=self.w.tproj_b, batch=B, n=self.w.tproj_total,
                                       k=spec.temb_dim, dt=self.dt, y32=self.temb_proj))

    # --------------------------------------------------------------------------- resnets
    def resnet(self, r, x: Act, dst: Act):
        if not r.temporal_prefix:
            return super().resnet(r, x, dst)
        xs = self.act("st_spatial", x.n, x.h, x.w, r.cout)
        super().resnet(r, x, xs)
        self.temporal_resnet(r, xs, dst)

    def temporal_resnet(self, r, xs: Act, dst: Act):
        tp, eps = r.temporal_prefix, (r.eps if r.eps is not None else self.spec.eps)
        a1 = self._frame_view(self.group_norm(tp + ".norm1", self._video_view(xs), tp + ".norm1", True, eps), xs)
        h1 = self.act("tres_h1", xs.n, xs.h, xs.w, r.cout)
        # temb is identical for the F frames of a video: row b * F of the [B*F, sum(cout)] projection
        rb_ptr = _ptr(self.temb_proj) + 4 * self.w.tproj_off[tp]
        self.conv3x1_t(tp + ".conv1", a1, self.w.conv3x1_t(tp + ".conv1.weight"), self.w.f32(tp + ".conv1.bias"),
                       h1, rowbias=(rb_ptr, self.F * self.w.tproj_total))
        a2 = self._frame_view(self.group_norm(tp + ".norm2", self._video_view(h1), tp + ".norm2", True, eps), xs)
        # AlphaBlender folded in: dst = xs + (1 - alpha) * (conv2(a2) + b)
        mix = (r.mixer, False)
        self.conv3x1_t(tp + ".conv2", a2, self.w.conv3x1_t(tp + ".conv2.weight", mix),
                       self.w.f32_scaled(tp + ".conv2.bias", mix), dst, residual=xs)

    # --------------------------------------------------------------------------- transformers
    def _row_op(self, name, fn, *, x: Act, y: Act, vec=None, ldv=0, x2: Act = None, mix=None, stats=None,
                mode=0, div=1, mod=1, flops=0):
        p = _lib.RowOpParams()
        p.x, p.y = x.ptr, y.ptr
        p.x2 = x2.ptr if x2 is not None else None
        p.vec, p.ldv = _ptr(vec), ldv
        p.rowstats_out = _ptr(stats)
        p.rowstats_slots = getattr(stats, "slots", 1)
        p.mix_factor = _ptr(mix)
        p.rows, p.c, p.ldx, p.ldy = x.rows, x.c, x.ld, y.ld
        p.ldx2 = x2.ld if x2 is not None else 0
        p.dtype = ops.dtype_code(self.dt)
        p.mode, p.div, p.mod = mode, div, mod
        p.frames, p.seq, p.batch = self.F, x.h * x.w, self.nvid
        nb = (3 if x2 is not None else 2) * x.rows * x.c * 2
        return Op(name, fn, (C.byref(p),), (p, x.buf, y.buf, vec, x2.buf if x2 is not None else None, mix, stats),
                  0, nb)

    def ctx_vector(self, a):
        """[B*F, C] rows of to_out(to_v(encoder_hidden_states)): cross-attention over one token."""
        if a not in self._ctx_vecs:
            lib, B = self.lib_or_dry(), self.B
            ctx_dim = self.spec.cross_attention_dim
            wv = self.w.small(a + ".to_v.weight")
            C_ = wv.shape[0]
            v = self.buf("ctx_v_" + a, (B, C_))
            vec = self.buf("ctx_vec_" + a, (B, C_))
            self.side_ops.append(ops.small_linear_op(a + ".to_v(ctx)", lib, x=self.ehs_in, w=wv, bias=None,
                                                     batch=B, n=C_, k=ctx_dim, dt=self.dt, y16=v))
            self.side_ops.append(ops.small_linear_op(a + ".to_out(ctx)", lib, x=v,
                                                     w=self.w.small(a + ".to_out.0.weight"),
                                                     bias=self.w.f32(a + ".to_out.0.bias"), batch=B, n=C_, k=C_,
                                                     dt=self.dt, y16=vec))
            self._ctx_vecs[a] = vec
        return self._ctx_vecs[a]

    def frame_pos_embedding(self, t):
        """time_pos_embed(sinusoid(frame index)): [F, C]; depends on the weights only."""
        if t.prefix not in self._pos_embs:
            lib, F_, dim = self.lib_or_dry(), self.F, t.dim
            sin = self.buf("pos_sin_" + t.prefix, (F_, dim))
            self.side_ops.append(Op(t.prefix + ".time_proj", lib.sfb_timestep_embed,
                                    (_ptr(self.frame_idx), F_, dim, 1, 0.0, _ptr(sin), dim, ops.dtype_code(self.dt)),
                                    (self.frame_idx, sin)))
            h = self.buf("pos_h_" + t.prefix, (F_, 4 * dim))
            self.side_ops.append(ops.small_linear_op(t.prefix + ".time_pos_embed.linear_1", lib, x=sin,
                                                     w=self.w.small(t.prefix + ".time_pos_embed.linear_1.weight"),
                                                     bias=self.w.f32(t.prefix + ".time_pos_embed.linear_1.bias"),
                                                     batch=F_, n=4 * dim, k=dim, dt=self.dt, y16=h, act_out=1))
            emb = self.buf("pos_emb_" + t.prefix, (F_, dim))
            self.side_ops.append(ops.small_linear_op(t.prefix + ".time_pos_embed.linear_2", lib, x=h,
                                                     w=self.w.small(t.prefix + ".time_pos_embed.linear_2.weight"),
                                                     bias=self.w.f32(t.prefix + ".time_pos_embed.linear_2.bias"),
                                                     batch=F_, n=dim, k=4 * dim, dt=self.dt, y16=emb))
            self._pos_embs[t.prefix] = emb
        return self._pos_embs[t.prefix]

    def _join_side(self):
        if not self._joined:
            self._joined = True
            self._emit(_JoinOp("all"))

    def transformer(self, t, x: Act, dst: Act):
        if not t.temporal:
            return super().transformer(t, x, dst)
        lib, p, dim = self.lib_or_dry(), t.prefix, t.dim
        S = x.h * x.w
        a1 = self.group_norm(p + ".norm", x, p + ".norm", False, 1e-6)
        hs = self.act("tf_hidden", x.n, x.h, x.w, dim)
        hm = self.act("tf_mix", x.n, x.h, x.w, dim)
        st = self.ln_slot(hs.rows, dim)
        self.linear(p + ".proj_in", a1, self.w.matrix(p + ".proj_in.weight"), self.w.f32(p + ".proj_in.bias"),
                    hs, rowstats_out=st)
        pos = self.frame_pos_embedding(t)
        for d in range(t.depth):
            b = f"{p}.transformer_blocks.{d}"
            tb = f"{p}.temporal_transformer_blocks.{d}"
            vec_s, vec_t = self.ctx_vector(b + ".attn2"), self.ctx_vector(tb + ".attn2")
            # ---- spatial block: self-attention per frame; cross-attention over one token = add
            self.attention(b + ".attn1", hs, b + ".norm1", st, b, t, cross=False, stats_next=None)
            self._join_side()
            st3 = self.ln_slot(hs.rows, dim)
            self._emit(self._row_op(b + ".attn2(ctx add)", lib.sfb_row_broadcast_add, x=hs, y=hs, vec=vec_s,
                                    ldv=dim, stats=st3, mode=_lib.ROW_IDX_DIV_MOD, div=S, mod=self.B))
            self._ff(b, "ff", b + ".norm3", hs, st3, None, dim)
            # ---- temporal block on hm = hs + frame position embedding
            st_in = self.ln_slot(hs.rows, dim)
            self._emit(self._row_op(tb + ".pos add", lib.sfb_row_broadcast_add, x=hs, y=hm, vec=pos, ldv=dim,
                                    stats=st_in, mode=_lib.ROW_IDX_DIV_MOD, div=S, mod=self.F))
            st1 = self.ln_slot(hs.rows, dim)
            self._ff(tb, "ff_in", tb + ".norm_in", hm, st_in, st1, dim)
            # self-attention across frames
            wm, bias, colsum = self.w.ln_matrix([f"{tb}.attn1.to_q.weight", f"{tb}.attn1.to_k.weight",
                                                 f"{tb}.attn1.to_v.weight"], tb + ".norm1")
            qkv = self.act("t_qkv", x.n, x.h, x.w, 3 * dim)
            self._emit(self._gemm(tb + ".attn1.qkv", a=self._a_matrix(hm), b=wm, M=hm.rows, N=3 * dim, K=dim,
                                  dt=self.dt, out=qkv.ptr, ldo=3 * dim, bias=bias,
                                  ln=dict(rowstats=st1, colsum=colsum, eps=1e-5, dim=dim),
                                  keep=(hm.buf, qkv.buf, wm, colsum)))
            ao = self.act("attn_out", x.n, x.h, x.w, dim)
            tp_ = _lib.TemporalAttnParams()
            tp_.qkv, tp_.out = qkv.ptr, ao.ptr
            tp_.batch, tp_.frames, tp_.seq, tp_.heads, tp_.head_dim = self.nvid, self.F, S, t.heads, t.head_dim
            tp_.ld_qkv, tp_.ld_out, tp_.dtype, tp_.scale = 3 * dim, dim, ops.dtype_code(self.dt), t.head_dim ** -0.5
            self._emit(Op(tb + ".attn1.core", lib.sfb_temporal_attention, (C.byref(tp_),), (tp_, qkv.buf, ao.buf),
                          4 * self.nvid * S * t.heads * self.F * self.F * t.head_dim,
                          4 * hm.rows * dim * 2))
            self.linear(tb + ".attn1.to_out", ao, self.w.matrix(f"{tb}.attn1.to_out.0.weight"),
                        self.w.f32(f"{tb}.attn1.to_out.0.bias"), hm, residual=hm)
            st3t = self.ln_slot(hs.rows, dim)
            self._emit(self._row_op(tb + ".attn2(ctx add)", lib.sfb_row_broadcast_add, x=hm, y=hm, vec=vec_t,
                                    ldv=dim, stats=st3t, mode=_lib.ROW_IDX_TEMPORAL_CTX))
            self._ff(tb, "ff", tb + ".norm3", hm, st3t, None, dim)
            # ---- AlphaBlender
            st = self.ln_slot(hs.rows, dim) if d + 1 < t.depth else None
            self._emit(self._row_op(p + ".time_mixer", lib.sfb_alpha_blend, x=hs, y=hs, x2=hm,
                                    mix=self.w.f32(p + ".time_mixer.mix_factor"), stats=st))
        self.linear(p + ".proj_out", hs, self.w.matrix(p + ".proj_out.weight"),
                    self.w.f32(p + ".proj_out.bias"), dst, residual=x)
