"""ORACLE (test infrastructure, NOT product code).

PyTorch restatement of diffusers' ``T2IAdapter`` with ``adapter_type="full_adapter"`` (``FullAdapter``, SD-1.5) and
``"full_adapter_xl"`` (``FullAdapterXL``, SDXL), its ``AdapterBlock`` / ``AdapterResnetBlock``, and ``MultiAdapter``'s
weighted sum.  PARITY STATUS: **unpinned** -- written from diffusers' structure, not run against it.  Module tree and
parameter names follow diffusers (``adapter.conv_in``, ``adapter.body.{i}.in_conv``,
``adapter.body.{i}.resnets.{j}.block1`` / ``block2``).  Structural check: 77,369,280 parameters for the 3-channel SD
adapter, 77,000,640 for the 1-channel one, 79,028,160 for the 3-channel XL adapter (tests/test_t2i_adapter_cpu.py).

`unet_forward` is the UNet side: ``UNet2DConditionModel.forward`` of ``oracle/unet_oracle.py``, restated over that
module's own sub-modules, with diffusers' ``down_intrablock_additional_residuals`` (and its deprecated form).

Only ``tests/`` may import this.
"""
from dataclasses import dataclass
from typing import Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle.unet_oracle import UNetOutput, timestep_embedding


@dataclass
class T2IAdapterConfig:
    in_channels: int = 3
    channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    num_res_blocks: int = 2
    downscale_factor: int = 8
    adapter_type: str = "full_adapter"


def sd_config(**kw):
    """TencentARC's SD-1.5 adapters (canny / sketch: in_channels 1; depth / openpose: 3)."""
    return T2IAdapterConfig(**kw)


def sdxl_config(**kw):
    """TencentARC's SDXL adapters (t2i-adapter-*-sdxl-1.0)."""
    return T2IAdapterConfig(**dict(dict(downscale_factor=16, adapter_type="full_adapter_xl"), **kw))


class AdapterResnetBlock(nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.block1 = nn.Conv2d(channels, channels, 3, padding=1)
        self.act = nn.ReLU()
        self.block2 = nn.Conv2d(channels, channels, 1)

    def forward(self, x):
        return self.block2(self.act(self.block1(x))) + x


class AdapterBlock(nn.Module):
    def __init__(self, cin, cout, num_res_blocks, down=False):
        super().__init__()
        self.downsample = nn.AvgPool2d(2, 2, ceil_mode=True) if down else None
        self.in_conv = nn.Conv2d(cin, cout, 1) if cin != cout else None
        self.resnets = nn.Sequential(*[AdapterResnetBlock(cout) for _ in range(num_res_blocks)])

    def forward(self, x):
        if self.downsample is not None:
            x = self.downsample(x)
        if self.in_conv is not None:
            x = self.in_conv(x)
        return self.resnets(x)


class FullAdapter(nn.Module):
    def __init__(self, in_channels, channels, num_res_blocks, downscale_factor):
        super().__init__()
        self.unshuffle = nn.PixelUnshuffle(downscale_factor)
        self.conv_in = nn.Conv2d(in_channels * downscale_factor ** 2, channels[0], 3, padding=1)
        self.body = nn.ModuleList(
            [AdapterBlock(channels[0], channels[0], num_res_blocks)]
            + [AdapterBlock(channels[i - 1], channels[i], num_res_blocks, down=True) for i in range(1, len(channels))])
        self.total_downscale_factor = downscale_factor * 2 ** (len(channels) - 1)

    def forward(self, x):
        x = self.conv_in(self.unshuffle(x))
        features = []
        for block in self.body:
            x = block(x)
            features.append(x)
        return features


class FullAdapterXL(FullAdapter):
    def __init__(self, in_channels, channels, num_res_blocks, downscale_factor):
        nn.Module.__init__(self)
        self.unshuffle = nn.PixelUnshuffle(downscale_factor)
        self.conv_in = nn.Conv2d(in_channels * downscale_factor ** 2, channels[0], 3, padding=1)
        body = []
        for i in range(len(channels)):
            if i == 1:
                body.append(AdapterBlock(channels[i - 1], channels[i], num_res_blocks))
            elif i == 2:
                body.append(AdapterBlock(channels[i - 1], channels[i], num_res_blocks, down=True))
            else:
                body.append(AdapterBlock(channels[i], channels[i], num_res_blocks))
        self.body = nn.ModuleList(body)
        self.total_downscale_factor = downscale_factor * 2  # one downsampling block


class T2IAdapter(nn.Module):
    def __init__(self, cfg: T2IAdapterConfig):
        super().__init__()
        self.config = cfg
        args = (cfg.in_channels, list(cfg.channels), cfg.num_res_blocks, cfg.downscale_factor)
        if cfg.adapter_type == "full_adapter":
            self.adapter = FullAdapter(*args)
        elif cfg.adapter_type == "full_adapter_xl":
            self.adapter = FullAdapterXL(*args)
        else:
            raise ValueError(f"adapter_type {cfg.adapter_type!r} is not restated here")

    def forward(self, x):
        return self.adapter(x)

    @property
    def total_downscale_factor(self):
        return self.adapter.total_downscale_factor

    @property
    def downscale_factor(self):
        return self.adapter.unshuffle.downscale_factor


class MultiAdapter(nn.Module):
    def __init__(self, adapters):
        super().__init__()
        self.num_adapter = len(adapters)
        self.adapters = nn.ModuleList(adapters)

    def forward(self, xs, adapter_weights=None):
        if adapter_weights is None:
            adapter_weights = torch.tensor([1 / self.num_adapter] * self.num_adapter)
        else:
            adapter_weights = torch.tensor(adapter_weights)
        acc = None
        for x, w, adapter in zip(xs, adapter_weights, self.adapters):
            features = adapter(x)
            if acc is None:
                acc = [w * f for f in features]
            else:
                for i in range(len(features)):
                    acc[i] += w * features[i]
        return acc


def build_adapter(cfg: T2IAdapterConfig, seed: int = 0, dtype=torch.float32, device="cpu"):
    """Seeded default-PyTorch-init adapter (no checkpoints exist offline)."""
    g = torch.random.get_rng_state()
    torch.manual_seed(seed)
    m = T2IAdapter(cfg)
    torch.random.set_rng_state(g)
    return m.to(device=device, dtype=dtype).eval()


def _down_block(blk, x, temb, ctx, residual):
    """oracle DownBlock.forward plus a T2I-Adapter residual: diffusers' CrossAttnDownBlock2D adds it to the output of
    its last (resnet, transformer) pair, before the downsampler; for a plain DownBlock2D, UNet2DConditionModel.forward
    adds it in place to the block's output, which is also its last skip tensor."""
    outs = []
    for i, r in enumerate(blk.resnets):
        x = r(x, temb)
        if blk.attentions is not None:
            x = blk.attentions[i](x, ctx)
            if residual is not None and i == len(blk.resnets) - 1:
                x = x + residual
        outs.append(x)
    if blk.downsamplers is not None:
        x = blk.downsamplers[0](x)
        outs.append(x)
    if blk.attentions is None and residual is not None:
        x = x + residual
        outs[-1] = x
    return x, outs


def unet_forward(unet, sample, timestep, encoder_hidden_states, added_cond_kwargs=None,
                 down_block_additional_residuals=None, mid_block_additional_residual=None,
                 down_intrablock_additional_residuals=None):
    """diffusers ``UNet2DConditionModel.forward`` of an ``oracle.unet_oracle`` UNet with T2I-Adapter residuals: they
    are taken in order, one per down block, then one after the mid block when the next one has the mid output's
    shape (T2I-Adapter-XL); leftovers are ignored.  ``down_block_additional_residuals`` without
    ``mid_block_additional_residual`` is diffusers' deprecated T2I-Adapter form.  ControlNet residuals are added
    after, on top of them.  The caller's list is not consumed (diffusers pops from it).  Returns UNetOutput."""
    cfg = unet.config
    if (down_intrablock_additional_residuals is None and mid_block_additional_residual is None
            and down_block_additional_residuals is not None):
        down_intrablock_additional_residuals, down_block_additional_residuals = down_block_additional_residuals, None
    adapter = None if down_intrablock_additional_residuals is None else list(down_intrablock_additional_residuals)
    b = sample.shape[0]
    if not torch.is_tensor(timestep):
        timestep = torch.tensor([timestep], device=sample.device)
    t = timestep.reshape(-1).to(sample.device)
    t = t.expand(b) if t.numel() == 1 else t
    emb = unet.time_embedding(timestep_embedding(t, cfg.block_out_channels[0], cfg.flip_sin_to_cos,
                                                 cfg.freq_shift).to(sample.dtype))
    if cfg.addition_embed_type == "text_time":
        tid = timestep_embedding(added_cond_kwargs["time_ids"].flatten(), cfg.addition_time_embed_dim,
                                 cfg.flip_sin_to_cos, cfg.freq_shift).reshape(b, -1).to(sample.dtype)
        emb = emb + unet.add_embedding(torch.cat([added_cond_kwargs["text_embeds"], tid], dim=-1))
    ctx = encoder_hidden_states
    x = unet.conv_in(sample)
    skips = [x]
    for blk in unet.down_blocks:
        x, outs = _down_block(blk, x, emb, ctx, adapter.pop(0) if adapter else None)
        skips.extend(outs)
    if down_block_additional_residuals is not None:
        skips = [s + r for s, r in zip(skips, down_block_additional_residuals)]
    x = unet.mid_block(x, emb, ctx)
    if adapter and adapter[0].shape == x.shape:
        x = x + adapter.pop(0)
    if mid_block_additional_residual is not None:
        x = x + mid_block_additional_residual
    for blk in unet.up_blocks:
        x = blk(x, skips, emb, ctx)
    return UNetOutput(sample=unet.conv_out(F.silu(unet.conv_norm_out(x))))
