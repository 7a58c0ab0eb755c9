"""Launch schedules of diffusers' ``AutoencoderTiny`` (TAESD / TAESDXL, ``madebyollin/taesd``): its decode and
encode, the VAE the few-step (LCM, Turbo) pipelines pair with, where the decoder's share of an image is large.

Every layer between the two edge convolutions is a 3x3 conv with 64 input and 64 output channels, run by
sfb_conv3x3_c64 (an N of exactly 64; the wgmma GEMM's 160-wide tile would be 60 % padding):
  * a block ``relu(conv4(relu(conv2(relu(conv0(x))))) + x)`` is three launches: conv0 and conv2 with bias +
    ReLU into a ping-pong pair of buffers, conv4 with bias + residual + ReLU written IN PLACE over the block
    input x (each output pixel reads its residual right before writing it), so one block-input buffer per
    resolution plus one ping-pong pair is all the activation memory;
  * the decoder's ``Upsample(2, nearest)`` + bias-free conv is one launch in the kernel's upsample mode (the
    upsampled tensor never exists); the encoder's stride-2 conv (symmetric padding 1) one launch in its
    stride-2 mode;
  * conv_in (few channels, NCHW input) runs on sfb_conv3x3_small_ex with the model's input transform applied to
    in-image values -- ``tanh(x / 3) * 3`` for the decoder, ``(x + 1) / 2`` for the encoder -- which the zero
    padding keeps out of the weights; conv_out on sfb_conv_out (NHWC -> NCHW), the decoder's
    ``.mul(2).sub(1)`` folded into its weight and bias at pack time (w' = 2 w, b' = 2 b - 1).
No GroupNorm or LayerNorm anywhere, so no statistics arenas.
"""
from dataclasses import dataclass
from typing import Tuple

from . import _lib, ops
from .ops import Act
from .plan import Plan
from .unet_spec import cfg_get

C = 64  # the only block width the kernel computes


@dataclass
class TAESDSpec:
    in_channels: int = 3
    out_channels: int = 3
    latent_channels: int = 4
    num_encoder_blocks: Tuple[int, ...] = (1, 3, 3, 3)
    num_decoder_blocks: Tuple[int, ...] = (3, 3, 3, 1)

    @property
    def temporal(self):
        return False

    def all_resnets(self):
        return []

    @property
    def up(self):
        """Decoder upsampling factor (2 per stage but the last)."""
        return 1 << (len(self.num_decoder_blocks) - 1)


def taesd_spec_from_config(cfg) -> TAESDSpec:
    """The spec of an AutoencoderTiny config; NotImplementedError naming the key for what the native path does
    not compute."""
    for key, want in (("act_fn", "relu"), ("upsample_fn", "nearest"), ("upsampling_scaling_factor", 2)):
        v = cfg_get(cfg, key, want)
        if v != want:
            raise NotImplementedError(f"AutoencoderTiny config {key}={v!r} is not supported by the H100 path "
                                      f"(only {want!r})")
    stages = {}
    for side in ("encoder", "decoder"):
        boc = tuple(cfg_get(cfg, f"{side}_block_out_channels", (C,) * 4))
        nb = tuple(int(n) for n in cfg_get(cfg, f"num_{side}_blocks", (1, 3, 3, 3) if side == "encoder" else (3, 3, 3, 1)))
        if any(c != C for c in boc):
            raise NotImplementedError(f"AutoencoderTiny config {side}_block_out_channels={boc}: only {C}-channel "
                                      "blocks are supported by the H100 path")
        if len(nb) != len(boc) or not nb or any(n < 0 for n in nb):
            raise NotImplementedError(f"AutoencoderTiny config num_{side}_blocks={nb} does not match "
                                      f"{side}_block_out_channels={boc}")
        stages[side] = nb
    chans = {k: int(cfg_get(cfg, k, d)) for k, d in (("latent_channels", 4), ("in_channels", 3), ("out_channels", 3))}
    for k, v in chans.items():
        if not 1 <= v <= 8:
            # sfb_conv3x3_small_ex reads at most 8 NCHW channels, sfb_conv_out writes at most 8 (rules out the
            # 16-channel latents of TAESD3 / TAEF1)
            raise NotImplementedError(f"AutoencoderTiny config {k}={v}: the H100 path takes 1 to 8 channels")
    return TAESDSpec(num_encoder_blocks=stages["encoder"], num_decoder_blocks=stages["decoder"], **chans)


def decoder_layers(spec: TAESDSpec):
    """(index in DecoderTiny.layers, kind) in diffusers' construction order; kind is 'conv_in', 'relu', 'block',
    'upsample', 'conv' (64 -> 64, no bias) or 'conv_out'."""
    out, i = [(0, "conv_in"), (1, "relu")], 2
    for s, nb in enumerate(spec.num_decoder_blocks):
        final = s == len(spec.num_decoder_blocks) - 1
        kinds = ["block"] * nb + ([] if final else ["upsample"]) + ["conv_out" if final else "conv"]
        for k in kinds:
            out.append((i, k))
            i += 1
    return out


def encoder_layers(spec: TAESDSpec):
    """(index in EncoderTiny.layers, kind): 'conv_in', 'down' (64 -> 64, stride 2, no bias), 'block', 'conv_out'."""
    out, i = [], 0
    for s, nb in enumerate(spec.num_encoder_blocks):
        for k in ["conv_in" if s == 0 else "down"] + ["block"] * nb:
            out.append((i, k))
            i += 1
    out.append((i, "conv_out"))
    return out


def _shapes(prefix, layers, cin, cout):
    out = {}
    for i, kind in layers:
        p = f"{prefix}.layers.{i}"
        if kind == "block":
            for j in (0, 2, 4):
                out[f"{p}.conv.{j}.weight"], out[f"{p}.conv.{j}.bias"] = (C, C, 3, 3), (C,)
        elif kind in ("conv", "down"):
            out[p + ".weight"] = (C, C, 3, 3)
        elif kind == "conv_in":
            out[p + ".weight"], out[p + ".bias"] = (C, cin, 3, 3), (C,)
        elif kind == "conv_out":
            out[p + ".weight"], out[p + ".bias"] = (cout, C, 3, 3), (cout,)
    return out


def taesd_decoder_param_shapes(spec: TAESDSpec):
    """{diffusers parameter name: shape} of AutoencoderTiny's decoder."""
    return _shapes("decoder", decoder_layers(spec), spec.latent_channels, spec.out_channels)


def taesd_encoder_param_shapes(spec: TAESDSpec):
    """{diffusers parameter name: shape} of AutoencoderTiny's encoder."""
    return _shapes("encoder", encoder_layers(spec), spec.in_channels, spec.latent_channels)


class _TAESDPlan(Plan):
    def c64(self, name, x: Act, y: Act, mode=_lib.C64_SAME, bias=None, relu=False, residual=None):
        self._emit(ops.conv_c64_op(name, self.lib_or_dry(), x=x, weight=self.w.conv3x3_plain(name + ".weight"),
                                   bias=bias, y=y, mode=mode, dt=self.dt, relu=relu, residual=residual))

    def block(self, p, x: Act):
        """AutoencoderTinyBlock(64, 64) over x, in place: x = relu(conv4(relu(conv2(relu(conv0(x))))) + x)."""
        t0 = self.act("taesd_t0", x.n, x.h, x.w, C)
        t1 = self.act("taesd_t1", x.n, x.h, x.w, C)
        self.c64(p + ".conv.0", x, t0, bias=self.w.f32(p + ".conv.0.bias"), relu=True)
        self.c64(p + ".conv.2", t0, t1, bias=self.w.f32(p + ".conv.2.bias"), relu=True)
        self.c64(p + ".conv.4", t1, x, bias=self.w.f32(p + ".conv.4.bias"), relu=True, residual=x)


class TAESDDecodePlan(_TAESDPlan):
    """Static launch schedule of `AutoencoderTiny.decode` for a fixed (batch, latent height, width): NCHW latents
    z_in [B, latent_channels, h, w] -> NCHW images out [B, out_channels, up * h, up * w]."""

    def __init__(self, weights, batch, height, width):
        super().__init__(weights, batch, height, width)
        spec = self.spec
        self.z_in = self._alloc((batch, spec.latent_channels, height, width), self.dt)
        self.out = self._alloc((batch, spec.out_channels, spec.up * height, spec.up * width), self.dt)
        self._build()

    def _build(self):
        spec, B, h, w = self.spec, self.B, self.H, self.W
        stage = 0
        x = self.act("taesd_x0", B, h, w, C)
        for i, kind in decoder_layers(spec):
            p = f"decoder.layers.{i}"
            if kind == "conv_in":
                self._emit(ops.conv_small_ex_op(
                    p, self.lib_or_dry(), x=self.z_in, weight=self.w.conv3x3_small(p + ".weight", C),
                    bias=self.w.f32(p + ".bias"), y=x, n=B, h=h, w=w, cin=spec.latent_channels, cout=C, dt=self.dt,
                    in_xform=_lib.XFORM_TANH3, relu=True))  # (the ReLU is layers.1)
            elif kind == "block":
                self.block(p, x)
            elif kind == "conv":  # after layers[i - 1], the nearest-2x Upsample
                stage += 1
                y = self.act(f"taesd_x{stage}", B, 2 * x.h, 2 * x.w, C)
                self.c64(p, x, y, mode=_lib.C64_UP2X)
                x = y
            elif kind == "conv_out":
                wt, b = self.w.conv3x3_affine(p, 2.0, -1.0)  # DecoderTiny's .mul(2).sub(1)
                self.conv_out(p, x, wt, b, self.out)
        self._finish()


class TAESDEncodePlan(_TAESDPlan):
    """Static launch schedule of `AutoencoderTiny.encode` for a fixed (batch, image height, width): NCHW images
    x_in [B, in_channels, H, W] in [-1, 1] -> NCHW latents out [B, latent_channels, h, w], each stride-2 stage
    taking a size s to ceil(s / 2)."""

    def __init__(self, weights, batch, height, width):
        super().__init__(weights, batch, height, width)
        spec = self.spec
        h, w = height, width
        for _ in range(len(spec.num_encoder_blocks) - 1):
            h, w = (h + 1) // 2, (w + 1) // 2
        self.x_in = self._alloc((batch, spec.in_channels, height, width), self.dt)
        self.out = self._alloc((batch, spec.latent_channels, h, w), self.dt)
        self._build()

    def _build(self):
        spec, B = self.spec, self.B
        stage = 0
        x = self.act("taesd_x0", B, self.H, self.W, C)
        for i, kind in encoder_layers(spec):
            p = f"encoder.layers.{i}"
            if kind == "conv_in":
                self._emit(ops.conv_small_ex_op(
                    p, self.lib_or_dry(), x=self.x_in, weight=self.w.conv3x3_small(p + ".weight", C),
                    bias=self.w.f32(p + ".bias"), y=x, n=B, h=self.H, w=self.W, cin=spec.in_channels, cout=C,
                    dt=self.dt, in_xform=_lib.XFORM_UNIT))
            elif kind == "down":
                stage += 1
                y = self.act(f"taesd_x{stage}", B, (x.h + 1) // 2, (x.w + 1) // 2, C)
                self.c64(p, x, y, mode=_lib.C64_STRIDE2)
                x = y
            elif kind == "block":
                self.block(p, x)
            elif kind == "conv_out":
                self.conv_out(p, x, self.w.conv3x3_plain(p + ".weight"), self.w.f32(p + ".bias"), self.out)
        self._finish()
