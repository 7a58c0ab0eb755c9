"""Launch schedule of diffusers' ``ControlNetModel``: the UNet's encoder half (time embedding, conv_in, down
blocks, mid block, built by UNetPlan's emitters) plus the conditioning-image embedding, the 1x1 zero convs
and the scaled NCHW outputs.

  * conditioning embedding: layers with fewer than 64 input channels run on sfb_conv3x3_small (the first
    reads the NCHW image); the others on the wgmma conv, whose K blocks are 64 channels wide, so an
    activation with c >= 64 channels lives in a buffer of round_up(c, 64) channels whose tail its
    producer writes as zeros (zero weight rows, zero bias, SiLU(0) = 0).  conv_out adds conv_in(sample)
    in its epilogue.  A BGR conditioning image is handled by reversing the first conv's input channels.
  * every down-block output keeps its own buffer (no up path reads them); the zero convs are 1x1 GEMMs,
    and one sfb_nhwc_to_nchw_scaled launch writes all residuals into the static NCHW outputs times the
    per-residual factors in `scale_in` (device memory: a captured graph serves every conditioning_scale
    and guess mode).
"""
import torch

from . import _lib, ops
from .ops import Act
from .plan import UNetPlan, _JoinOp, _round_up


def stored_channels(c):
    """Channel pitch of a conditioning-embedding activation with c channels: the few-channel kernel reads
    it as is, the wgmma conv (c >= 64) in whole 64-channel K blocks."""
    return c if c < 64 else _round_up(c, 64)


def residual_scales(n_down, conditioning_scale, guess_mode):
    """fp32 factor of each of the n_down down residuals and (last) of the mid residual, as diffusers'
    ControlNetModel computes them: conditioning_scale, or in guess mode
    logspace(-1, 0, n_down + 1) * conditioning_scale."""
    if guess_mode:
        return torch.logspace(-1, 0, n_down + 1) * conditioning_scale
    return torch.full((n_down + 1,), float(conditioning_scale))


class ControlNetPlan(UNetPlan):
    """One static launch schedule of a ControlNet for a fixed (batch, latent height, latent width).  Static
    inputs: sample_in, t_in, ehs_in, cond_in (NCHW image, cond_factor times the latent size), scale_in
    (fp32 factor per residual), and for SDXL add_in / time_ids_in.  Outputs: down_out (NCHW list),
    mid_out."""

    @property
    def cond_factor(self):
        return 1 << (len(self.spec.cond_embed_channels) - 1)

    def cond_embedding(self, residual: Act, dst: Act):
        """dst = conv_out(embedding(cond_in)) + residual."""
        spec, B, lib = self.spec, self.B, self.lib_or_dry()
        emb, e = spec.cond_embed_channels, "controlnet_cond_embedding"
        f = self.cond_factor
        h, w = f * self.H, f * self.W
        layers = [(e + ".conv_in", spec.cond_channels, emb[0], 1)]
        for i in range(len(emb) - 1):
            layers += [(f"{e}.blocks.{2 * i}", emb[i], emb[i], 1), (f"{e}.blocks.{2 * i + 1}", emb[i], emb[i + 1], 2)]
        x = None  # NHWC input of the next layer (None: the NCHW image)
        for k, (name, cin, cout, stride) in enumerate(layers):
            ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
            cst = stored_channels(cout)
            y = self.act(f"cn_emb_{k}", B, ho, wo, cst)
            bias = self.w.f32_padded(name + ".bias", cst)
            if x is None or cin < 64:
                wt = self.w.conv3x3_small(name + ".weight", cst, flip_cin=x is None and spec.cond_bgr)
                self._emit(ops.conv_small_op(
                    name, lib, x=self.cond_in if x is None else x.buf, weight=wt, bias=bias, y=y, n=B, h=h, w=w,
                    cin=cin, cout=cst, stride=stride, dt=self.dt, ldx=0 if x is None else x.ld,
                    x_nchw=x is None, silu=True))
                self.ops[-1].flops = 2 * B * ho * wo * cout * 9 * cin  # algorithmic, not padded
            else:
                wm = self.w.conv3x3_padded(name + ".weight", x.c, cst)
                self.conv3x3(name, x, name, y, stride=stride, weights=(wm, bias), act=_lib.ACT_SILU)
            x, h, w = y, ho, wo
        wm = self.w.conv3x3_padded(e + ".conv_out.weight", x.c, dst.c)
        self.conv3x3(e + ".conv_out", x, e + ".conv_out", dst, residual=residual,
                     weights=(wm, self.w.f32(e + ".conv_out.bias")))

    def _build(self):
        spec, B, H, W = self.spec, self.B, self.H, self.W
        f = self.cond_factor
        self.cond_in = self._alloc((B, spec.cond_channels, f * H, f * W), self.dt)
        chans = spec.residual_channels()
        self.scale_in = self._alloc((len(chans) + 1,), torch.float32)
        # time embedding on the forked stream (as in the UNet), joined before the first resnet
        n_main = len(self.ops)
        self.time_embedding()
        self.side_ops.extend(self.ops[n_main:])
        del self.ops[n_main:]
        self._temb_last = self.side_ops[-1]

        c0 = spec.block_out_channels[0]
        xs = self.act("cn_conv_in", B, H, W, c0)
        self._sample_conv_in(xs)
        res = [self.act("cn_res_0", B, H, W, c0)]
        self.cond_embedding(xs, res[0])
        self._emit(_JoinOp("temb"))
        # ---- down path: every resnet (+ transformer) and downsampler output is a residual
        x, h, w = res[0], H, W
        for blk in spec.down:
            for r, t in zip(blk.resnets, blk.attentions):
                dst = self.act(f"cn_res_{len(res)}", B, h, w, r.cout)
                if t is None:
                    self.resnet(r, x, dst)
                else:
                    mid = self.act("res_out", B, h, w, r.cout)
                    self.resnet(r, x, mid)
                    self.transformer(t, mid, dst)
                res.append(dst)
                x = dst
            if blk.sampler:
                h, w = h // 2, w // 2
                dst = self.act(f"cn_res_{len(res)}", B, h, w, blk.cout)
                self.conv3x3(blk.sampler, x, blk.sampler, dst, stride=2)
                res.append(dst)
                x = dst
        assert [a.c for a in res] == chans
        # ---- mid
        m = spec.mid
        a = self.act("res_out", B, h, w, m.cout)
        self.resnet(m.resnets[0], x, a)
        b = self.act("mid_tf_out", B, h, w, m.cout)
        self.transformer(m.attentions[0], a, b)
        mid = self.act("cn_mid", B, h, w, m.cout)
        self.resnet(m.resnets[1], b, mid)
        # ---- zero convs, then all residuals times their factors into the NCHW outputs in one launch
        zc = []
        for i, r in enumerate(res + [mid]):
            name = f"controlnet_down_blocks.{i}" if i < len(res) else "controlnet_mid_block"
            z = self.act(f"cn_zc_{i}", r.n, r.h, r.w, r.c)
            self.linear(name, r, self.w.matrix(name + ".weight"), self.w.f32(name + ".bias"), z)
            zc.append(z)
        outs = [self._alloc((B, z.c, z.h, z.w), self.dt) for z in zc]
        self.down_out, self.mid_out = outs[:-1], outs[-1]
        self._emit(ops.nhwc_to_nchw_scaled_op("controlnet.outputs", self.lib_or_dry(), srcs=zc, dsts=outs,
                                              scale=self.scale_in, dt=self.dt))
        self._finish()
