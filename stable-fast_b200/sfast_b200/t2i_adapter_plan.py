"""Launch schedule of diffusers' ``T2IAdapter`` (``adapter_type`` "full_adapter" for SD-1.5, "full_adapter_xl" for
SDXL; TencentARC's canny / sketch / depth / lineart / openpose adapters): the conditioning image to the list of
features the adapter pipelines pass to the UNet as ``down_intrablock_additional_residuals``.

  * PixelUnshuffle(r) (sfb_pixel_unshuffle) writes the NCHW image as the NHWC input of conv_in, whose
    in_channels * r^2 channels are whole 64-channel K blocks of the wgmma conv;
  * conv_in and every resnet's 3x3 block1 run on the wgmma conv, block1 with the ReLU in its epilogue; the 1x1
    in_conv and block2 on the wgmma GEMM, block2 adding the resnet input in its epilogue (``x + block2(h)``);
  * a downsampling block starts with sfb_avg_pool2x2 (AvgPool2d(2, 2, ceil_mode=True) of an even-sized input);
  * the first resnet of block i writes the block's own feature buffer and the later ones update it in place, so
    every feature survives the blocks after it; one sfb_nhwc_to_nchw_scaled launch (factor 1) writes all of them
    into the static NCHW outputs.
No GroupNorm or LayerNorm, so no statistics arenas.
"""
from dataclasses import dataclass
from typing import Tuple

import torch

from . import _lib, ops
from .ops import Act, Op, _ptr
from .plan import Plan
from .unet_spec import cfg_get

ADAPTER_TYPES = ("full_adapter", "full_adapter_xl")


@dataclass
class T2IAdapterSpec:
    in_channels: int = 3
    channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    num_res_blocks: int = 2
    downscale_factor: int = 8
    adapter_type: str = "full_adapter"

    @property
    def temporal(self):
        return False

    def all_resnets(self):
        return []

    def blocks(self):
        """(pools, cin, cout) of each AdapterBlock in diffusers' order: `pools` is its AvgPool2d, cin != cout
        its 1x1 in_conv."""
        ch = self.channels
        if self.adapter_type == "full_adapter":
            return [(False, ch[0], ch[0])] + [(True, ch[i - 1], ch[i]) for i in range(1, len(ch))]
        # FullAdapterXL: block 1 changes channels without pooling, block 2 pools, the others keep their width
        return [(i == 2, ch[i - 1] if i in (1, 2) else ch[i], ch[i]) for i in range(len(ch))]

    @property
    def total_downscale_factor(self):
        return self.downscale_factor * 2 ** sum(p for p, _, _ in self.blocks())


def t2i_adapter_spec_from_config(cfg) -> T2IAdapterSpec:
    """The spec of a T2IAdapter config; NotImplementedError naming the key for what the native path does not
    compute."""
    kind = cfg_get(cfg, "adapter_type", "full_adapter")
    if kind not in ADAPTER_TYPES:
        # light_adapter's 80 / 160-channel middle widths are not whole 64-channel K blocks of the wgmma conv
        raise NotImplementedError(f"T2IAdapter config adapter_type={kind!r} is not supported by the H100 path "
                                  f"(only {', '.join(ADAPTER_TYPES)})")
    channels = tuple(int(c) for c in cfg_get(cfg, "channels", (320, 640, 1280, 1280)))
    if not channels or any(c <= 0 or c % 64 for c in channels):
        raise NotImplementedError(f"T2IAdapter config channels={channels}: the H100 path needs multiples of 64")
    nrb = int(cfg_get(cfg, "num_res_blocks", 2))
    if nrb < 1:
        raise NotImplementedError(f"T2IAdapter config num_res_blocks={nrb}: the H100 path needs at least 1")
    cin = int(cfg_get(cfg, "in_channels", 3))
    r = int(cfg_get(cfg, "downscale_factor", 8))
    if cin <= 0 or r <= 0 or cin * r * r % 64:
        raise NotImplementedError(f"T2IAdapter config in_channels={cin}, downscale_factor={r}: the H100 path needs "
                                  "in_channels * downscale_factor ** 2 to be a multiple of 64")
    return T2IAdapterSpec(in_channels=cin, channels=channels, num_res_blocks=nrb, downscale_factor=r,
                          adapter_type=kind)


def t2i_adapter_param_shapes(spec: T2IAdapterSpec):
    """{diffusers parameter name: shape} of a T2IAdapter."""
    r = spec.downscale_factor
    out = {"adapter.conv_in.weight": (spec.channels[0], spec.in_channels * r * r, 3, 3),
           "adapter.conv_in.bias": (spec.channels[0],)}
    for i, (_, cin, cout) in enumerate(spec.blocks()):
        p = f"adapter.body.{i}"
        if cin != cout:
            out[p + ".in_conv.weight"], out[p + ".in_conv.bias"] = (cout, cin, 1, 1), (cout,)
        for j in range(spec.num_res_blocks):
            q = f"{p}.resnets.{j}"
            out[q + ".block1.weight"], out[q + ".block1.bias"] = (cout, cout, 3, 3), (cout,)
            out[q + ".block2.weight"], out[q + ".block2.bias"] = (cout, cout, 1, 1), (cout,)
    return out


class AdapterPlan(Plan):
    """Static launch schedule of `T2IAdapter.forward` for a fixed (batch, image height, width): the NCHW image
    x_in [B, in_channels, H, W] -> features_out, one NCHW tensor per AdapterBlock."""

    def __init__(self, weights, batch, height, width):
        spec = weights.spec
        f = spec.total_downscale_factor
        if height % f or width % f:
            raise NotImplementedError(f"sfast (H100 build): T2I-Adapter image size {height}x{width} must be a "
                                      f"multiple of its total_downscale_factor {f}")
        super().__init__(weights, batch, height, width)
        self.x_in = self._alloc((batch, spec.in_channels, height, width), self.dt)
        self._build()

    def avg_pool(self, name, x: Act, y: Act):
        self._emit(Op(name, self.lib_or_dry().sfb_avg_pool2x2,
                      (x.ptr, y.ptr, x.n, x.h, x.w, x.c, x.ld, y.ld, ops.dtype_code(self.dt)),
                      (x.buf, y.buf), 3 * y.rows * y.c, 2 * (x.rows + y.rows) * x.c))

    def _build(self):
        spec, B, lib = self.spec, self.B, self.lib_or_dry()
        r = spec.downscale_factor
        h, w = self.H // r, self.W // r
        u = self.act("t2i_unshuffled", B, h, w, spec.in_channels * r * r)
        self._emit(Op("adapter.unshuffle", lib.sfb_pixel_unshuffle,
                      (_ptr(self.x_in), u.ptr, B, spec.in_channels, self.H, self.W, r, u.ld),
                      (self.x_in, u.buf), 0, 4 * self.x_in.numel()))
        x = self.act("t2i_conv_in", B, h, w, spec.channels[0])
        self.conv3x3("adapter.conv_in", u, "adapter.conv_in", x)
        feats = []
        for i, (pools, cin, cout) in enumerate(spec.blocks()):
            p = f"adapter.body.{i}"
            if pools:
                y = self.act(f"t2i_pool_{i}", B, x.h // 2, x.w // 2, cin)
                self.avg_pool(p + ".downsample", x, y)
                x = y
            if cin != cout:
                y = self.act(f"t2i_in_conv_{i}", B, x.h, x.w, cout)
                self.linear(p + ".in_conv", x, self.w.matrix(p + ".in_conv.weight"), self.w.f32(p + ".in_conv.bias"), y)
                x = y
            feat = self.act(f"t2i_feature_{i}", B, x.h, x.w, cout)
            hid = self.act("t2i_hidden", B, x.h, x.w, cout)
            for j in range(spec.num_res_blocks):
                q = f"{p}.resnets.{j}"
                self.conv3x3(q + ".block1", x, q + ".block1", hid, act=_lib.ACT_RELU)
                self.linear(q + ".block2", hid, self.w.matrix(q + ".block2.weight"), self.w.f32(q + ".block2.bias"),
                            feat, residual=x)
                x = feat
            feats.append(feat)
        self.features_out = [self._alloc((B, a.c, a.h, a.w), self.dt) for a in feats]
        self.scale_in = self._alloc((len(feats),), torch.float32)
        if not self.dry:
            self.scale_in.fill_(1.0)
        self._emit(ops.nhwc_to_nchw_scaled_op("adapter.features", lib, srcs=feats, dsts=self.features_out,
                                              scale=self.scale_in, dt=self.dt))
        self._finish()
