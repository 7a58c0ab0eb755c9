"""ORACLE (test infrastructure, NOT product code).

PyTorch restatement of the encoder half of diffusers ``AutoencoderKL`` (the SD-1.5 / SDXL VAE) and of the
whole module (`encode` + `decode`), the module `compile_vae` wraps in the reference
(/root/reference/src/sfast/compilers/diffusion_pipeline_compiler.py:154-190).  PARITY STATUS:
**unpinned**, as for oracle/vae_oracle.py, whose decoder, resnet, attention and config this file reuses.
Module tree and parameter names follow diffusers (`encoder.conv_in`, `encoder.down_blocks.N.{resnets,
downsamplers}`, `encoder.mid_block`, `encoder.conv_norm_out`, `encoder.conv_out`, `quant_conv`).
diffusers' Downsample2D with padding=0 pads one zero row / column AFTER the image before a pad-0
stride-2 conv.  Structural check: encoder + quant_conv of the SD VAE is 34,163,664 parameters, the whole
module diffusers' 83,653,863 (tests/test_vae_encode_cpu.py).

Only ``tests/`` may import this.
"""
from dataclasses import dataclass

import torch
import torch.nn as nn
import torch.nn.functional as F

from .vae_oracle import Decoder, DecoderOutput, VAEConfig, VaeMidBlock, VaeResnet


class VaeDownsample(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, stride=2, padding=0)

    def forward(self, x):
        return self.conv(F.pad(x, (0, 1, 0, 1), mode="constant", value=0))


class VaeDownBlock(nn.Module):
    def __init__(self, cin, cout, n, groups, add_down):
        super().__init__()
        self.resnets = nn.ModuleList([VaeResnet(cin if i == 0 else cout, cout, groups) for i in range(n)])
        self.downsamplers = nn.ModuleList([VaeDownsample(cout)]) if add_down else None

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0](x)
        return x


class Encoder(nn.Module):
    def __init__(self, cfg: VAEConfig):
        super().__init__()
        boc, g = cfg.block_out_channels, cfg.norm_num_groups
        self.conv_in = nn.Conv2d(cfg.in_channels, boc[0], 3, padding=1)
        self.down_blocks = nn.ModuleList()
        cout = boc[0]
        for i, c in enumerate(boc):
            cin, cout = cout, c
            self.down_blocks.append(VaeDownBlock(cin, cout, cfg.layers_per_block, g, i != len(boc) - 1))
        self.mid_block = VaeMidBlock(boc[-1], g)
        self.conv_norm_out = nn.GroupNorm(g, boc[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(boc[-1], 2 * cfg.latent_channels, 3, padding=1)  # double_z

    def forward(self, x):
        x = self.conv_in(x)
        for blk in self.down_blocks:
            x = blk(x)
        x = self.mid_block(x)
        return self.conv_out(F.silu(self.conv_norm_out(x)))


class DiagonalGaussianDistribution:
    """diffusers' latent distribution over the moments [B, 2 * C, h, w] (mean | log-variance)."""

    def __init__(self, parameters):
        self.parameters = parameters
        self.mean, logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)

    def sample(self, generator=None):
        eps = torch.randn(self.mean.shape, generator=generator, device=self.parameters.device,
                          dtype=self.parameters.dtype)
        return self.mean + self.std * eps

    def mode(self):
        return self.mean


@dataclass
class AutoencoderKLOutput:
    latent_dist: DiagonalGaussianDistribution


class AutoencoderKL(nn.Module):
    """The whole `AutoencoderKL`: encoder + quant_conv (`encode`), post_quant_conv + decoder (`decode`)."""

    def __init__(self, cfg: VAEConfig):
        super().__init__()
        self.config = cfg
        self.encoder = Encoder(cfg)
        self.quant_conv = nn.Conv2d(2 * cfg.latent_channels, 2 * cfg.latent_channels, 1)
        self.post_quant_conv = nn.Conv2d(cfg.latent_channels, cfg.latent_channels, 1)
        self.decoder = Decoder(cfg)

    @property
    def dtype(self):
        return self.post_quant_conv.weight.dtype

    @property
    def device(self):
        return self.post_quant_conv.weight.device

    def encode(self, x, return_dict=True):
        dist = DiagonalGaussianDistribution(self.quant_conv(self.encoder(x)))
        if not return_dict:
            return (dist,)
        return AutoencoderKLOutput(latent_dist=dist)

    def decode(self, z, return_dict=True):
        x = self.decoder(self.post_quant_conv(z))
        if not return_dict:
            return (x,)
        return DecoderOutput(sample=x)


def build_autoencoder_kl(cfg: VAEConfig, seed: int = 0, dtype=torch.float32, device="cpu"):
    """`AutoencoderKL` with seeded default-init weights and random GroupNorm affines (as `build_vae`)."""
    g = torch.random.get_rng_state()
    torch.manual_seed(seed)
    m = AutoencoderKL(cfg)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, nn.GroupNorm):
                mod.weight.copy_(1.0 + 0.3 * torch.randn_like(mod.weight))
                mod.bias.copy_(0.3 * torch.randn_like(mod.bias))
    torch.random.set_rng_state(g)
    return m.to(device=device, dtype=dtype).eval()
