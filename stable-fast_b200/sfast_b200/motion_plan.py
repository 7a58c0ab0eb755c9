"""Launch schedule of the AnimateDiff denoiser, diffusers ``UNetMotionModel``: an SD-1.5 / SDXL UNet with a motion
module after every (resnet, transformer) layer of its down and up blocks and, optionally, one in the mid block.

The B videos x F frames are a batch of B*F images for everything spatial -- the UNetPlan emitters run unchanged,
with one time-embedding row and one copy of the prompt per frame, as diffusers repeats them -- and a motion module
works on the same token-major [B*F*H*W, C] tensors (AnimateDiffTransformer3D / TransformerTemporalModel):

  * norm: GroupNorm over (C / G, F, H, W) per video = the GroupNorm kernels on the [B, F*H, W, C] view;
  * proj_in, then per transformer block: LayerNorm (folded into the QKV GEMM) + the sinusoidal position embedding
    pe_f, self-attention across the F frames of each (video, pixel), to_out + residual -- twice (attn1 and attn2
    are both self-attention) -- then the GEGLU FeedForward; proj_out with the module input as residual, written
    straight into the layer's output (a skip slice or the next layer's input).
  * pe_f enters after the LayerNorm's affine, in front of W_q / W_k / W_v; it is packed as the fp32 table
    pe W^T (PackedWeights.frame_bias_table) that sfb_frame_attention adds to the q / k / v of frame f as it
    loads them.  The attention reads the QKV rows in the spatial order: no tensor is ever transposed.
"""
import ctypes as C

from . import _lib, ops
from .ops import Act, Op, _ptr
from .plan import UNetPlan, VideoPlanMixin


class MotionUNetPlan(VideoPlanMixin, UNetPlan):
    _motion = True

    def __init__(self, weights, videos, frames, height, width, ctx_len=77, controlnet=False):
        spec = weights.spec
        if not spec.motion:
            raise ValueError("MotionUNetPlan needs a UNetMotionModel spec (spec.motion)")
        max_seq = min(m.max_seq_len for m in spec.motion)
        if not 1 <= frames <= max_seq:
            raise NotImplementedError(f"sfast (H100 build): {frames} frames; the motion modules take 1 to "
                                      f"motion_max_seq_length = {max_seq}")
        self.nvid, self.F = videos, frames
        self._motion_after = {m.after: m for m in spec.motion}
        super().__init__(weights, videos * frames, height, width, ctx_len, controlnet=controlnet)

    @staticmethod
    def _ln_arena_floats(spec, batch, height, width):
        """UNetPlan's, plus 3 * depth LayerNorms per motion module at its resolution."""
        tot = UNetPlan._ln_arena_floats(spec, batch, height, width)
        h, w, rows = height, width, {}
        for blk in spec.down:
            rows[blk.prefix] = batch * h * w
            if blk.sampler:
                h, w = h // 2, w // 2
        rows[spec.mid.prefix] = batch * h * w
        for blk in spec.up:
            rows[blk.prefix] = batch * h * w
            if blk.sampler:
                h, w = h * 2, w * 2
        for m in spec.motion:
            r = rows[m.prefix.rsplit(".motion_modules.", 1)[0]]
            tot += 3 * m.depth * r * 2 * ops.rowstats_slots(m.dim)
        return tot

    # --------------------------------------------------------------------------- layer hooks
    def resnet(self, r, x: Act, dst: Act):
        m = self._motion_after.get(r.prefix)
        if m is None:
            return super().resnet(r, x, dst)
        h = self.act("motion_in", x.n, x.h, x.w, r.cout)
        super().resnet(r, x, h)
        self.motion_module(m, h, dst)

    def transformer(self, t, x: Act, dst: Act):
        m = self._motion_after.get(t.prefix)
        if m is None:
            return super().transformer(t, x, dst)
        h = self.act("motion_in", x.n, x.h, x.w, t.dim)
        super().transformer(t, x, h)
        self.motion_module(m, h, dst)

    # --------------------------------------------------------------------------- motion module
    def frame_attention(self, name, qkv: Act, table, out: Act, m):
        """softmax(q k^T / sqrt(D)) v across the F frames of every (video, pixel, head), with the frame bias
        `table` [max_seq, 3C] added to q | k | v."""
        S, D = qkv.h * qkv.w, m.head_dim
        p = _lib.FrameAttnParams()
        p.qkv, p.frame_bias, p.out = qkv.ptr, _ptr(table), out.ptr
        p.batch, p.frames, p.seq, p.heads, p.head_dim = self.nvid, self.F, S, m.heads, D
        p.ld_qkv, p.ld_bias, p.ld_out = qkv.ld, table.shape[1], out.ld
        p.dtype, p.scale = ops.dtype_code(self.dt), D ** -0.5
        self._emit(Op(name, self.lib_or_dry().sfb_frame_attention, (C.byref(p),), (p, qkv.buf, table, out.buf),
                      4 * self.nvid * S * m.heads * self.F * self.F * D, qkv.rows * (3 + 1) * m.dim * 2))

    def motion_module(self, m, x: Act, dst: Act):
        """dst = x + motion_module(x) (AnimateDiffTransformer3D with double self-attention blocks)."""
        p, dim = m.prefix, m.dim
        a1 = self._frame_view(self.group_norm(p + ".norm", self._video_view(x), p + ".norm", False, 1e-6), x)
        hs = self.act("motion_hidden", x.n, x.h, x.w, dim)
        st = self.ln_slot(hs.rows, dim)
        self.linear(p + ".proj_in", a1, self.w.matrix(p + ".proj_in.weight"), self.w.f32(p + ".proj_in.bias"),
                    hs, rowstats_out=st)
        qkv = self.act("motion_qkv", x.n, x.h, x.w, 3 * dim)
        ao = self.act("attn_out", x.n, x.h, x.w, dim)
        for d in range(m.depth):
            b = f"{p}.transformer_blocks.{d}"
            for a, ln in (("attn1", "norm1"), ("attn2", "norm2")):
                names = [f"{b}.{a}.to_{n}.weight" for n in ("q", "k", "v")]
                wm, bias, colsum = self.w.ln_matrix(names, f"{b}.{ln}")
                self._emit(self._gemm(f"{b}.{a}.qkv", a=self._a_matrix(hs), b=wm, M=hs.rows, N=3 * dim, K=dim,
                                      dt=self.dt, out=qkv.ptr, ldo=qkv.ld, bias=bias,
                                      ln=dict(rowstats=st, colsum=colsum, eps=1e-5, dim=dim),
                                      keep=(hs.buf, qkv.buf, wm, colsum)))
                self.frame_attention(f"{b}.{a}.core", qkv,
                                     self.w.frame_bias_table(names, b + ".pos_embed.pe", m.max_seq_len), ao, m)
                st = self.ln_slot(hs.rows, dim)
                self.linear(f"{b}.{a}.to_out", ao, self.w.matrix(f"{b}.{a}.to_out.0.weight"),
                            self.w.f32(f"{b}.{a}.to_out.0.bias"), hs, residual=hs, rowstats_out=st)
            st_next = self.ln_slot(hs.rows, dim) if d + 1 < m.depth else None
            self._ff(b, "ff", b + ".norm3", hs, st, st_next, dim)
            st = st_next
        self.linear(p + ".proj_out", hs, self.w.matrix(p + ".proj_out.weight"), self.w.f32(p + ".proj_out.bias"),
                    dst, residual=x)
