"""ORACLE (test infrastructure, NOT product code).

PyTorch restatement of diffusers' ``AutoencoderTiny`` (TAESD / TAESDXL): ``EncoderTiny``, ``DecoderTiny``,
``AutoencoderTinyBlock``, ``encode`` / ``decode`` with the ``use_slicing`` and ``use_tiling`` options (the
blended ``_tiled_encode`` / ``_tiled_decode``).  PARITY STATUS: **unpinned** -- written from diffusers'
structure, not run against it.  Module tree and parameter names follow diffusers (``encoder.layers.{i}``,
``decoder.layers.{i}``, a block's ``conv.0`` / ``conv.2`` / ``conv.4``), with the ``layers`` indices counted by
the loop diffusers uses.  Structural check: 1,222,531 decoder + 1,222,532 encoder = 2,445,063 parameters at the
published config (tests/test_taesd_cpu.py).

`build_taesd` initialises every conv He-style (std sqrt(2 / fan_in)) from a seed, so activations keep their
scale through the ~30 ReLU layers instead of decaying toward the biases.

Only ``tests/`` may import this.
"""
import math
from dataclasses import dataclass, field
from typing import Tuple

import torch
import torch.nn as nn


@dataclass
class TAESDConfig:
    in_channels: int = 3
    out_channels: int = 3
    encoder_block_out_channels: Tuple[int, ...] = (64, 64, 64, 64)
    decoder_block_out_channels: Tuple[int, ...] = (64, 64, 64, 64)
    act_fn: str = "relu"
    upsample_fn: str = "nearest"
    latent_channels: int = 4
    upsampling_scaling_factor: int = 2
    num_encoder_blocks: Tuple[int, ...] = (1, 3, 3, 3)
    num_decoder_blocks: Tuple[int, ...] = (3, 3, 3, 1)
    latent_magnitude: int = 3
    latent_shift: float = 0.5
    force_upcast: bool = False
    scaling_factor: float = 1.0
    shift_factor: float = 0.0
    block_out_channels: Tuple[int, ...] = field(default=(64, 64, 64, 64))


def tiny_config(**kw):
    return TAESDConfig(**kw)


class AutoencoderTinyBlock(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.conv = nn.Sequential(nn.Conv2d(cin, cout, 3, padding=1), nn.ReLU(),
                                  nn.Conv2d(cout, cout, 3, padding=1), nn.ReLU(),
                                  nn.Conv2d(cout, cout, 3, padding=1))
        self.skip = nn.Conv2d(cin, cout, 1, bias=False) if cin != cout else nn.Identity()
        self.fuse = nn.ReLU()

    def forward(self, x):
        return self.fuse(self.conv(x) + self.skip(x))


class EncoderTiny(nn.Module):
    def __init__(self, cfg: TAESDConfig):
        super().__init__()
        layers = []
        for i, nb in enumerate(cfg.num_encoder_blocks):
            c = cfg.encoder_block_out_channels[i]
            if i == 0:
                layers.append(nn.Conv2d(cfg.in_channels, c, 3, padding=1))
            else:
                layers.append(nn.Conv2d(c, c, 3, padding=1, stride=2, bias=False))
            for _ in range(nb):
                layers.append(AutoencoderTinyBlock(c, c))
        layers.append(nn.Conv2d(cfg.encoder_block_out_channels[-1], cfg.latent_channels, 3, padding=1))
        self.layers = nn.Sequential(*layers)

    def forward(self, x):
        return self.layers(x.add(1).div(2))


class DecoderTiny(nn.Module):
    def __init__(self, cfg: TAESDConfig):
        super().__init__()
        boc = cfg.decoder_block_out_channels
        layers = [nn.Conv2d(cfg.latent_channels, boc[0], 3, padding=1), nn.ReLU()]
        for i, nb in enumerate(cfg.num_decoder_blocks):
            final = i == len(cfg.num_decoder_blocks) - 1
            c = boc[i]
            for _ in range(nb):
                layers.append(AutoencoderTinyBlock(c, c))
            if not final:
                layers.append(nn.Upsample(scale_factor=cfg.upsampling_scaling_factor, mode=cfg.upsample_fn))
            layers.append(nn.Conv2d(c, c if not final else cfg.out_channels, 3, padding=1, bias=final))
        self.layers = nn.Sequential(*layers)

    def forward(self, x):
        x = torch.tanh(x / 3) * 3
        return self.layers(x).mul(2).sub(1)


class DecoderOutput(dict):
    def __init__(self, sample):
        super().__init__(sample=sample)
        self.sample = sample


class AutoencoderTinyOutput(dict):
    def __init__(self, latents):
        super().__init__(latents=latents)
        self.latents = latents


class AutoencoderTiny(nn.Module):
    def __init__(self, cfg: TAESDConfig):
        super().__init__()
        self.config = cfg
        self.encoder = EncoderTiny(cfg)
        self.decoder = DecoderTiny(cfg)
        self.spatial_scale_factor = cfg.upsampling_scaling_factor ** (len(cfg.num_decoder_blocks) - 1)
        self.tile_overlap_factor = 0.125
        self.tile_sample_min_size = 512
        self.tile_latent_min_size = self.tile_sample_min_size // self.spatial_scale_factor
        self.use_slicing = False
        self.use_tiling = False

    @property
    def device(self):
        return next(self.parameters()).device

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    def _tiled(self, x, fn, sf_in, sf_out, tile_size, out_channels):
        """diffusers' _tiled_encode / _tiled_decode: tiles of tile_size input pixels overlapping by
        tile_overlap_factor, each output tile blended over what earlier tiles wrote with a linear ramp."""
        blend_size = int(tile_size * self.tile_overlap_factor)
        traverse = tile_size - blend_size
        ti, tj = range(0, x.shape[-2], traverse), range(0, x.shape[-1], traverse)
        n_out = tile_size * sf_out // sf_in
        b_out = blend_size * sf_out // sf_in
        ramp = (torch.arange(n_out) / (b_out - 1)).clamp(0, 1)
        masks = torch.stack(torch.meshgrid([ramp, ramp], indexing="ij")).to(x.device)
        out = torch.zeros(x.shape[0], out_channels, x.shape[-2] * sf_out // sf_in, x.shape[-1] * sf_out // sf_in,
                          device=x.device, dtype=x.dtype)
        for i in ti:
            for j in tj:
                tile_in = x[..., i:i + tile_size, j:j + tile_size]
                o = out[..., i * sf_out // sf_in:(i + tile_size) * sf_out // sf_in,
                        j * sf_out // sf_in:(j + tile_size) * sf_out // sf_in]
                tile = fn(tile_in)
                h, w = tile.shape[-2], tile.shape[-1]
                mi = torch.ones_like(masks[0]) if i == 0 else masks[0]
                mj = torch.ones_like(masks[1]) if j == 0 else masks[1]
                m = (mi * mj)[:h, :w]
                o.copy_(m * tile[..., :h, :w] + (1 - m) * o)
        return out

    def _tiled_encode(self, x):
        return self._tiled(x, self.encoder, self.spatial_scale_factor, 1, self.tile_sample_min_size,
                           self.config.latent_channels)

    def _tiled_decode(self, x):
        return self._tiled(x, self.decoder, 1, self.spatial_scale_factor, self.tile_latent_min_size,
                           self.config.out_channels)

    def encode(self, x, return_dict=True):
        if self.use_slicing and x.shape[0] > 1:
            out = torch.cat([self._tiled_encode(s) if self.use_tiling else self.encoder(s) for s in x.split(1)])
        else:
            out = self._tiled_encode(x) if self.use_tiling else self.encoder(x)
        if not return_dict:
            return (out,)
        return AutoencoderTinyOutput(latents=out)

    def decode(self, x, generator=None, return_dict=True):
        if self.use_slicing and x.shape[0] > 1:
            out = torch.cat([self._tiled_decode(s) if self.use_tiling else self.decoder(s) for s in x.split(1)])
        else:
            out = self._tiled_decode(x) if self.use_tiling else self.decoder(x)
        if not return_dict:
            return (out,)
        return DecoderOutput(sample=out)


def he_init_(m: nn.Module, seed=0):
    """Seeded He-scaled conv weights (std sqrt(2 / fan_in)) and small biases."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in sorted(m.named_parameters()):
            if p.dim() == 4:
                fan_in = p.shape[1] * p.shape[2] * p.shape[3]
                p.copy_(torch.randn(p.shape, generator=g) * math.sqrt(2.0 / fan_in))
            else:
                p.copy_(torch.randn(p.shape, generator=g) * 0.05)
    return m


def build_taesd(cfg=None, seed=0, dtype=torch.float32, device="cpu"):
    m = he_init_(AutoencoderTiny(cfg or tiny_config()), seed)
    return m.to(device=device, dtype=dtype).eval()
