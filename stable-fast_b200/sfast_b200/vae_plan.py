"""Launch schedules of the VAE decoder and encoder (diffusers ``AutoencoderKL.decode`` / ``encode``), the
module the reference's `compile_vae` wraps (/root/reference/src/sfast/compilers/diffusion_pipeline_compiler.py:
154-190).  The encoder mirrors the decoder: GroupNorm-folded resnets, the same single-head attention, and
stride-2 down-convs with diffusers' one-sided padding (SFB_A_DOWNCONV3X3) where the decoder has up-convs.

Same kernel families as the UNet at larger spatial sizes: GroupNorm(+SiLU) -> implicit-GEMM 3x3
convolutions with fused bias / residual, nearest-2x upsample folded into four 2x2 phase convolutions,
and ONE single-head attention over the 64 x 64 latent tokens with head_dim 512.  That head does not fit
the flash kernel's TMEM budget (O would need 528 columns), and it is one layer of ~34 GFLOP, so it runs
as five tcgen05 GEMMs around a row-softmax kernel: Q (scale folded into W_q), K, V^T (= W_v X^T: the
weight is the A operand, the activation the B operand), S = Q K^T (activation x activation: plain
row-major B operand), P = softmax(S), O = P V^T^T + b_v (rows of P sum to 1, so V's bias is added after
the product), out-projection + residual.
"""
import ctypes as C
from dataclasses import dataclass
from typing import Tuple

import torch

from . import _lib, ops
from .ops import Act, Op, _ptr
from .plan import Plan, VideoPlanMixin
from .unet_spec import cfg_get


@dataclass
class VAESpec:
    latent_channels: int
    out_channels: int
    block_out_channels: Tuple[int, ...]
    layers_per_block: int
    groups: int
    eps: float = 1e-6
    num_frames: int = 0
    in_channels: int = 3

    @property
    def temporal(self):
        return False

    def all_resnets(self):
        return []


def vae_spec_from_config(cfg) -> VAESpec:
    boc = tuple(cfg_get(cfg, "block_out_channels"))
    for key, allowed in (("act_fn", ("silu", "swish")), ("mid_block_add_attention", (True,)),
                         ("use_quant_conv", (True,)), ("use_post_quant_conv", (True,))):
        v = cfg_get(cfg, key, allowed[0])
        if v not in allowed:
            raise NotImplementedError(f"VAE config {key}={v!r} is not supported by the H100 path")
    for t in cfg_get(cfg, "up_block_types", ("UpDecoderBlock2D",) * len(boc)):
        if t != "UpDecoderBlock2D":
            raise NotImplementedError(f"VAE up block type {t}")
    if boc[-1] % 64 or any(c % 64 for c in boc):
        raise NotImplementedError("VAE channel counts must be multiples of 64")
    return VAESpec(latent_channels=cfg_get(cfg, "latent_channels", 4), out_channels=cfg_get(cfg, "out_channels", 3),
                   block_out_channels=boc, layers_per_block=cfg_get(cfg, "layers_per_block", 2),
                   groups=cfg_get(cfg, "norm_num_groups", 32), in_channels=cfg_get(cfg, "in_channels", 3))


def vae_encoder_spec_from_config(cfg) -> VAESpec:
    """vae_spec_from_config plus what the native encoder needs of `AutoencoderKL.encode`."""
    spec = vae_spec_from_config(cfg)
    for t in cfg_get(cfg, "down_block_types", ("DownEncoderBlock2D",) * len(spec.block_out_channels)):
        if t != "DownEncoderBlock2D":
            raise NotImplementedError(f"VAE down block type {t}")
    if not cfg_get(cfg, "double_z", True):
        raise NotImplementedError("VAE config double_z=False is not supported by the H100 path")
    if spec.in_channels > 8 or 2 * spec.latent_channels > 8:
        # sfb_conv_in / sfb_conv_out take at most 8 image channels / moments
        raise NotImplementedError(f"VAE encoder with {spec.in_channels} image channels and "
                                  f"{2 * spec.latent_channels} moments (at most 8 each)")
    return spec


def vae_decoder_param_shapes(spec: VAESpec):
    """{diffusers parameter name: shape} of post_quant_conv + decoder."""
    out = {}

    def conv(p, cout, cin, k):
        out[p + ".weight"] = (cout, cin, k, k)
        out[p + ".bias"] = (cout,)

    def norm(p, c):
        out[p + ".weight"] = (c,)
        out[p + ".bias"] = (c,)

    def lin(p, n, k):
        out[p + ".weight"] = (n, k)
        out[p + ".bias"] = (n,)

    def resnet(p, cin, cout):
        norm(p + ".norm1", cin)
        conv(p + ".conv1", cout, cin, 3)
        norm(p + ".norm2", cout)
        conv(p + ".conv2", cout, cout, 3)
        if cin != cout:
            conv(p + ".conv_shortcut", cout, cin, 1)

    lc, boc = spec.latent_channels, spec.block_out_channels
    conv("post_quant_conv", lc, lc, 1)
    c = boc[-1]
    conv("decoder.conv_in", c, lc, 3)
    resnet("decoder.mid_block.resnets.0", c, c)
    a = "decoder.mid_block.attentions.0"
    norm(a + ".group_norm", c)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        lin(f"{a}.{n}", c, c)
    resnet("decoder.mid_block.resnets.1", c, c)
    cout = c
    for i, ch in enumerate(reversed(boc)):
        cin, cout = cout, ch
        for j in range(spec.layers_per_block + 1):
            resnet(f"decoder.up_blocks.{i}.resnets.{j}", cin if j == 0 else cout, cout)
        if i != len(boc) - 1:
            conv(f"decoder.up_blocks.{i}.upsamplers.0.conv", cout, cout, 3)
    norm("decoder.conv_norm_out", boc[0])
    conv("decoder.conv_out", spec.out_channels, boc[0], 3)
    return out


def decoder_resnets(spec: VAESpec):
    """(module prefix, cin, cout) of every resnet of the decoder, in schedule order."""
    c = spec.block_out_channels[-1]
    out = [(f"decoder.mid_block.resnets.{j}", c, c) for j in (0, 1)]
    cout = c
    for i, ch in enumerate(reversed(spec.block_out_channels)):
        cin, cout = cout, ch
        out += [(f"decoder.up_blocks.{i}.resnets.{j}", cin if j == 0 else cout, cout)
                for j in range(spec.layers_per_block + 1)]
    return out


def vae_temporal_decoder_param_shapes(spec: VAESpec):
    """{diffusers parameter name: shape} of the decoder of `AutoencoderKLTemporalDecoder` (SVD's VAE): the 2-D
    decoder without post_quant_conv, every resnet a SpatioTemporalResBlock (the 2-D resnet as its
    `spatial_res_block`, a `temporal_res_block` of two (3,1,1) Conv3d and a learned `time_mixer`), and a
    (3,1,1) `time_conv_out` after conv_out."""
    out = {}
    for k, v in vae_decoder_param_shapes(spec).items():
        if k.startswith("post_quant_conv."):
            continue
        p, sep, rest = k.partition(".resnets.")
        if sep:
            j, leaf = rest.split(".", 1)
            k = f"{p}.resnets.{j}.spatial_res_block.{leaf}"
        out[k] = v
    for p, _, c in decoder_resnets(spec):
        t = p + ".temporal_res_block"
        for n in ("norm1", "norm2"):
            out[f"{t}.{n}.weight"] = out[f"{t}.{n}.bias"] = (c,)
        for n in ("conv1", "conv2"):
            out[f"{t}.{n}.weight"], out[f"{t}.{n}.bias"] = (c, c, 3, 1, 1), (c,)
        out[p + ".time_mixer.mix_factor"] = (1,)
    oc = spec.out_channels
    out["decoder.time_conv_out.weight"], out["decoder.time_conv_out.bias"] = (oc, oc, 3, 1, 1), (oc,)
    return out


def vae_encoder_param_shapes(spec: VAESpec):
    """{diffusers parameter name: shape} of encoder + quant_conv."""
    out = {}

    def conv(p, cout, cin, k):
        out[p + ".weight"] = (cout, cin, k, k)
        out[p + ".bias"] = (cout,)

    def norm(p, c):
        out[p + ".weight"] = (c,)
        out[p + ".bias"] = (c,)

    def resnet(p, cin, cout):
        norm(p + ".norm1", cin)
        conv(p + ".conv1", cout, cin, 3)
        norm(p + ".norm2", cout)
        conv(p + ".conv2", cout, cout, 3)
        if cin != cout:
            conv(p + ".conv_shortcut", cout, cin, 1)

    boc, m = spec.block_out_channels, 2 * spec.latent_channels
    conv("encoder.conv_in", boc[0], spec.in_channels, 3)
    cout = boc[0]
    for i, ch in enumerate(boc):
        cin, cout = cout, ch
        for j in range(spec.layers_per_block):
            resnet(f"encoder.down_blocks.{i}.resnets.{j}", cin if j == 0 else cout, cout)
        if i != len(boc) - 1:
            conv(f"encoder.down_blocks.{i}.downsamplers.0.conv", cout, cout, 3)
    c = boc[-1]
    resnet("encoder.mid_block.resnets.0", c, c)
    a = "encoder.mid_block.attentions.0"
    norm(a + ".group_norm", c)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        out[f"{a}.{n}.weight"] = (c, c)
        out[f"{a}.{n}.bias"] = (c,)
    resnet("encoder.mid_block.resnets.1", c, c)
    norm("encoder.conv_norm_out", c)
    conv("encoder.conv_out", m, c, 3)
    conv("quant_conv", m, m, 1)
    return out


class _VAEPlan(Plan):
    """What the VAE's decoder and encoder schedules share: the GroupNorm-folded resnet and single-head
    attention sub-graphs (no time embedding, no folded LayerNorms)."""

    def vae_resnet(self, p, x: Act, dst: Act, cin, cout):
        eps = self.spec.eps
        a1, gn1 = self.norm_for_conv(p + ".norm1", x, p + ".norm1", eps, cout)
        h1 = self.act("res_h1", x.n, x.h, x.w, cout)
        self.conv3x3(p + ".conv1", a1, p + ".conv1", h1, gn=gn1)
        a2, gn2 = self.norm_for_conv(p + ".norm2", h1, p + ".norm2", eps, cout)
        res = x
        if cin != cout:
            res = self.act("res_sc", x.n, x.h, x.w, cout)
            self.linear(p + ".conv_shortcut", x, self.w.matrix(p + ".conv_shortcut.weight"),
                        self.w.f32(p + ".conv_shortcut.bias"), res)
        self.conv3x3(p + ".conv2", a2, p + ".conv2", dst, residual=res, gn=gn2)

    def vae_attention(self, p, x: Act, dst: Act):
        """dst = x + to_out(softmax(q k^T / sqrt(c)) v) over the h*w tokens of each image, one head."""
        lib, c, S, B = self.lib_or_dry(), x.c, x.h * x.w, x.n
        hn = self.group_norm(p + ".group_norm", x, p + ".group_norm", False, self.spec.eps)
        q = self.act("vae_q", x.n, x.h, x.w, c)
        k = self.act("vae_k", x.n, x.h, x.w, c)
        wq, bq = self.w.scaled_linear(p + ".to_q", c ** -0.5)
        self.linear(p + ".to_q", hn, wq, bq, q)
        self.linear(p + ".to_k", hn, self.w.matrix(p + ".to_k.weight"), self.w.f32(p + ".to_k.bias"), k)
        vt = self.buf("vae_vt", (B, c, S))        # V^T per image: [c, S]
        # fp32 scores, one image at a time (stream order makes reuse safe); the softmax writes the 16-bit
        # probabilities over the first half of each row (16-bit scores cost ~2 % on the probabilities)
        sc = self.buf("vae_scores", (S, S), torch.float32)
        o = self.act("vae_o", x.n, x.h, x.w, c)
        wv_plain = self.w.small(p + ".to_v.weight")  # [c, c] row-major: the A operand of V^T = W_v X^T
        es = 2
        for b in range(B):
            hn_b = _ptr(hn.buf) + b * S * hn.ld * es
            # V^T[c, S] = W_v [c, c] . hn_b[S, c]^T   (bias added after P V: softmax rows sum to 1)
            self._emit(self._gemm(f"{p}.to_v^T[{b}]", a=ops.a_matrix(_ptr(wv_plain), c, c, c),
                                  b=ops.PlainB(hn_b, S, c, hn.ld, self.dry), M=c, N=S, K=c, dt=self.dt,
                                  out=_ptr(vt) + b * c * S * es, ldo=S, splits=1, keep=(wv_plain, hn.buf, vt)))
            # S = q_b k_b^T
            self._emit(self._gemm(f"{p}.qk^T[{b}]", a=ops.a_matrix(_ptr(q.buf) + b * S * c * es, S, c, c),
                                  b=ops.PlainB(_ptr(k.buf) + b * S * c * es, S, c, c, self.dry), M=S, N=S, K=c,
                                  dt=self.dt, out=_ptr(sc), ldo=S, splits=1, epi=_lib.EPI_STORE_F32,
                                  keep=(q.buf, k.buf, sc)))
            self._emit(Op(f"{p}.softmax[{b}]", lib.sfb_row_softmax,
                          (_ptr(sc), _ptr(sc), S, S, S, 2 * S, 1, ops.dtype_code(self.dt)), (sc,), 0, 6 * S * S))
            # O = P V + b_v   (P: 16-bit rows at a pitch of 2 * S elements inside the fp32 buffer)
            self._emit(self._gemm(f"{p}.pv[{b}]", a=ops.a_matrix(_ptr(sc), S, S, 2 * S),
                                  b=ops.PlainB(_ptr(vt) + b * c * S * es, c, S, S, self.dry), M=S, N=c, K=S,
                                  dt=self.dt, out=_ptr(o.buf) + b * S * c * es, ldo=c,
                                  bias=self.w.f32(p + ".to_v.bias"), splits=1, keep=(sc, vt, o.buf)))
        self.linear(p + ".to_out", o, self.w.matrix(p + ".to_out.0.weight"), self.w.f32(p + ".to_out.0.bias"),
                    dst, residual=x)


class VAEDecodePlan(_VAEPlan):
    """Static launch schedule of `AutoencoderKL.decode` for a fixed (batch, latent height, width)."""

    def __init__(self, weights, batch, height, width):
        spec = weights.spec
        super().__init__(weights, batch, height, width,
                         n_gn=2 * (2 + len(spec.block_out_channels) * (spec.layers_per_block + 1)) + 2)
        self.z_in = self._alloc((batch, spec.latent_channels, height, width), self.dt)
        up = 1 << (len(spec.block_out_channels) - 1)
        self.out = self._alloc((batch, spec.out_channels, height * up, width * up), self.dt)
        self._build()

    def _build(self):
        spec, B, H, W, lib = self.spec, self.B, self.H, self.W, self.lib_or_dry()
        lc, boc = spec.latent_channels, spec.block_out_channels
        c = boc[-1]
        # post_quant_conv (1x1, NCHW -> NCHW) then conv_in (NCHW -> NHWC)
        zq = self.buf("pq_out", (B, lc, H, W))
        wpq = self.w.small("post_quant_conv.weight")
        self._emit(Op("post_quant_conv", lib.sfb_pointwise_nchw,
                      (_ptr(self.z_in), _ptr(wpq), _ptr(self.w.f32("post_quant_conv.bias")), _ptr(zq), B, H * W,
                       lc, lc, ops.dtype_code(self.dt)), (self.z_in, wpq, zq)))
        x = self.act("vae_x0", B, H, W, c)
        self.conv_in("decoder.conv_in", zq, x)
        m = "decoder.mid_block"
        a = self.act("vae_x1", B, H, W, c)
        self.vae_resnet(m + ".resnets.0", x, a, c, c)
        self.vae_attention(m + ".attentions.0", a, x)
        self.vae_resnet(m + ".resnets.1", x, a, c, c)
        x, cout, h, w = a, c, H, W
        for i, ch in enumerate(reversed(boc)):
            cin, cout = cout, ch
            for j in range(spec.layers_per_block + 1):
                dst = self.act(f"vae_up{i}_{j % 2}", B, h, w, cout)
                self.vae_resnet(f"decoder.up_blocks.{i}.resnets.{j}", x, dst, cin if j == 0 else cout, cout)
                x = dst
            if i != len(boc) - 1:
                dst = self.act(f"vae_ups{i}", B, 2 * h, 2 * w, cout)
                self.upconv3x3(f"decoder.up_blocks.{i}.upsamplers.0.conv", x,
                               f"decoder.up_blocks.{i}.upsamplers.0.conv", dst)
                x, h, w = dst, 2 * h, 2 * w
        y = self.group_norm("decoder.conv_norm_out", x, "decoder.conv_norm_out", True, spec.eps)
        self.conv_out("decoder.conv_out", y, self.w.conv3x3_plain("decoder.conv_out.weight"),
                      self.w.f32("decoder.conv_out.bias"), self.out)
        self._finish()


class TemporalDecodePlan(VideoPlanMixin, _VAEPlan):
    """Static launch schedule of `AutoencoderKLTemporalDecoder.decode(z, num_frames)` (SVD's VAE) for a fixed
    (frames, num_frames, latent height, width): NCHW latents [frames, latent_channels, h, w], `frames` / num_frames
    videos of num_frames consecutive frames -> NCHW frames [frames, out_channels, 8 h, 8 w].

    The 2-D decoder's schedule with every resnet a SpatioTemporalResBlock: the 2-D resnet (vae_resnet) writes
    x_s, then the temporal resnet -- GroupNorm over (frames, height, width) per video, Conv3d (3,1,1),
    GroupNorm, Conv3d -- adds its output to x_s IN PLACE (the second conv's residual epilogue), with the
    learned AlphaBlender folded into that conv: x_s + sigmoid(mix_factor) * conv2(..) (the decoder's blenders
    switch spatial and temporal, the SVD UNet's do not).  The temporal half reuses the spatial half's
    GroupNorm output and conv1 buffers; its only new buffers are GroupNorm outputs at the resolutions where
    the spatial convs apply their GroupNorm themselves (about 6 % over the 2-D decoder's total).  conv_out and
    time_conv_out run as one kernel (sfb_conv_out_temporal)."""

    def __init__(self, weights, frames, num_frames, height, width):
        spec = weights.spec
        if num_frames <= 0 or frames <= 0 or frames % num_frames:
            raise ValueError(f"sfast (H100 build): {frames} latents are not whole videos of num_frames={num_frames}")
        if height * width % 64:
            # the mid-block attention runs P V with the token count as its K
            raise NotImplementedError(f"sfast (H100 build): temporal VAE decode of a {height}x{width} latent: the "
                                      "mid-block attention needs a latent of a multiple of 64 pixels")
        self.nvid, self.F = frames // num_frames, num_frames
        n_resnets = 2 + len(spec.block_out_channels) * (spec.layers_per_block + 1)
        # 2 GroupNorms per spatial and 2 per temporal resnet, the attention's and conv_norm_out
        super().__init__(weights, frames, height, width, n_gn=4 * n_resnets + 2)
        self.z_in = self._alloc((frames, spec.latent_channels, height, width), self.dt)
        up = 1 << (len(spec.block_out_channels) - 1)
        self.out = self._alloc((frames, spec.out_channels, height * up, width * up), self.dt)
        self._build()

    def st_resnet(self, p, x: Act, dst: Act, cin, cout):
        """SpatioTemporalResBlock: x_s = spatial_res_block(x) into dst, then in place
        dst = x_s + sigmoid(mix_factor) * conv2(silu(norm2(conv1(silu(norm1(x_s))))))."""
        self.vae_resnet(p + ".spatial_res_block", x, dst, cin, cout)
        t, eps = p + ".temporal_res_block", 1e-5
        g = self.act("gn_out", dst.n, dst.h, dst.w, cout)
        self.group_norm(t + ".norm1", self._video_view(dst), t + ".norm1", True, eps, dst=self._video_view(g))
        h1 = self.act("res_h1", dst.n, dst.h, dst.w, cout)
        self.conv3x1_t(t + ".conv1", g, self.w.conv3x1_t(t + ".conv1.weight"), self.w.f32(t + ".conv1.bias"), h1)
        self.group_norm(t + ".norm2", self._video_view(h1), t + ".norm2", True, eps, dst=self._video_view(g))
        mix = (p + ".time_mixer.mix_factor", True)
        self.conv3x1_t(t + ".conv2", g, self.w.conv3x1_t(t + ".conv2.weight", mix),
                       self.w.f32_scaled(t + ".conv2.bias", mix), dst, residual=dst)

    def _build(self):
        spec, B, H, W = self.spec, self.B, self.H, self.W
        boc = spec.block_out_channels
        c = boc[-1]
        x = self.act("vae_x0", B, H, W, c)
        self.conv_in("decoder.conv_in", self.z_in, x)
        m = "decoder.mid_block"
        a = self.act("vae_x1", B, H, W, c)
        self.st_resnet(m + ".resnets.0", x, a, c, c)
        self.vae_attention(m + ".attentions.0", a, x)
        self.st_resnet(m + ".resnets.1", x, a, c, c)
        x, cout, h, w = a, c, H, W
        for i, ch in enumerate(reversed(boc)):
            cin, cout = cout, ch
            for j in range(spec.layers_per_block + 1):
                dst = self.act(f"vae_up{i}_{j % 2}", B, h, w, cout)
                self.st_resnet(f"decoder.up_blocks.{i}.resnets.{j}", x, dst, cin if j == 0 else cout, cout)
                x = dst
            if i != len(boc) - 1:
                dst = self.act(f"vae_ups{i}", B, 2 * h, 2 * w, cout)
                self.upconv3x3(f"decoder.up_blocks.{i}.upsamplers.0.conv", x,
                               f"decoder.up_blocks.{i}.upsamplers.0.conv", dst)
                x, h, w = dst, 2 * h, 2 * w
        y = self.group_norm("decoder.conv_norm_out", x, "decoder.conv_norm_out", True, spec.eps)
        self._emit(ops.conv_out_temporal_op(
            "decoder.conv_out+time_conv_out", self.lib_or_dry(), x=y,
            w=self.w.conv3x3_plain("decoder.conv_out.weight"), bias=self.w.f32("decoder.conv_out.bias"),
            wt=self.w.time_conv_out("decoder.time_conv_out.weight"), bt=self.w.f32("decoder.time_conv_out.bias"),
            out=self.out, frames=self.F, dt=self.dt))
        self._finish()


class VAEEncodePlan(_VAEPlan):
    """Static launch schedule of `AutoencoderKL.encode` for a fixed (batch, image height, width): NCHW image
    [B, in_channels, H, W] -> NCHW moments [B, 2 * latent_channels, H / 8, W / 8] (mean | logvar) of the
    latent distribution.  quant_conv is folded into conv_out at pack time."""

    def __init__(self, weights, batch, height, width):
        spec = weights.spec
        div = 1 << (len(spec.block_out_channels) - 1)
        if height % div or width % div or (height // div) * (width // div) % 64:
            # the mid-block attention runs P V with the token count as its K: a multiple of 64 (as in decode)
            raise NotImplementedError(
                f"sfast (H100 build): VAE encode of a {height}x{width} image: the size must be a multiple of "
                f"{div} with a latent of a multiple of 64 pixels")
        super().__init__(weights, batch, height, width,
                         n_gn=2 * (2 + len(spec.block_out_channels) * spec.layers_per_block) + 2)
        self.x_in = self._alloc((batch, spec.in_channels, height, width), self.dt)
        self.out = self._alloc((batch, 2 * spec.latent_channels, height // div, width // div), self.dt)
        self._build()

    def _build(self):
        spec, B, H, W = self.spec, self.B, self.H, self.W
        boc, m = spec.block_out_channels, 2 * spec.latent_channels
        x = self.act("enc_x0", B, H, W, boc[0])
        self.conv_in("encoder.conv_in", self.x_in, x)
        cout, h, w = boc[0], H, W
        for i, ch in enumerate(boc):
            cin, cout = cout, ch
            for j in range(spec.layers_per_block):
                dst = self.act(f"enc_down{i}_{j % 2}", B, h, w, cout)
                self.vae_resnet(f"encoder.down_blocks.{i}.resnets.{j}", x, dst, cin if j == 0 else cout, cout)
                x = dst
            if i != len(boc) - 1:
                dst = self.act(f"enc_ds{i}", B, h // 2, w // 2, cout)
                name = f"encoder.down_blocks.{i}.downsamplers.0.conv"
                self.conv3x3(name, x, name, dst, down=True)
                x, h, w = dst, h // 2, w // 2
        mid = "encoder.mid_block"
        a = self.act("enc_mid0", B, h, w, cout)
        b = self.act("enc_mid1", B, h, w, cout)
        self.vae_resnet(mid + ".resnets.0", x, a, cout, cout)
        self.vae_attention(mid + ".attentions.0", a, b)
        self.vae_resnet(mid + ".resnets.1", b, a, cout, cout)
        y = self.group_norm("encoder.conv_norm_out", a, "encoder.conv_norm_out", True, spec.eps)
        # conv_out then quant_conv (1x1) as ONE 3x3 conv with the folded weight (NHWC -> NCHW)
        w_out, b_out = self.w.conv3x3_pointwise("encoder.conv_out", "quant_conv")
        self.conv_out("encoder.conv_out+quant_conv", y, w_out, b_out, self.out, flops=2 * B * h * w * m * (9 * cout + m))
        self._finish()
