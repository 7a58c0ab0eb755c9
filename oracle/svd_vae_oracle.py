"""ORACLE (test infrastructure, NOT product code).

PyTorch restatement of diffusers ``AutoencoderKLTemporalDecoder``, the VAE of Stable Video Diffusion: the
2-D VAE's encoder (oracle/vae_encoder_oracle.py) and quant_conv, no post_quant_conv, and a
``TemporalDecoder``.  PARITY STATUS: **unpinned** -- the arithmetic lives in the un-vendored dependency
``diffusers`` (absent here), as for the other VAE oracles.

``decode(z, num_frames)`` treats the N = batch x num_frames latents as videos of num_frames consecutive
frames.  Module tree and parameter names follow diffusers:

  * ``decoder.conv_in``; ``decoder.mid_block`` = resnets.0, attentions.0 (the 2-D VAE's single-head
    attention), resnets.1; ``decoder.up_blocks.N`` = layers_per_block + 1 resnets and, except on the last
    block, ``upsamplers.0.conv`` (nearest 2x, then a 3x3 conv);
  * every resnet is a SpatioTemporalResBlock: ``spatial_res_block`` (the 2-D resnet, eps 1e-6),
    ``temporal_res_block`` (x + conv2(silu(norm2(conv1(silu(norm1(x)))))), Conv3d (3,1,1) with padding
    (1,0,0), GroupNorm eps 1e-5 over (frames, height, width)) and ``time_mixer``, an AlphaBlender with
    merge_strategy="learned" and switch_spatial_to_temporal_mix=True:
    out = sigmoid(m) * x_temporal + (1 - sigmoid(m)) * x_spatial;
  * ``decoder.conv_norm_out`` (eps 1e-6), SiLU, ``decoder.conv_out``, whose output is stored in the module's
    dtype, then ``decoder.time_conv_out``, a Conv3d 3 -> 3 with kernel (3,1,1) and zero padding (1,0,0) over
    each video's frames.

`build_svd_vae` randomises the GroupNorm affines (as `build_vae`) and every mix_factor (diffusers initialises
them to 0, where sigmoid and 1 - sigmoid agree and a swapped blend would go unnoticed).

Only ``tests/`` may import this.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .vae_encoder_oracle import AutoencoderKLOutput, DiagonalGaussianDistribution, Encoder
from .vae_oracle import DecoderOutput, VAEConfig, VaeAttention, VaeResnet


def svd_vae_config() -> VAEConfig:
    """SVD / SVD-XT's VAE: the SD VAE's widths (128, 256, 512, 512), 2 layers per block, 4 latent channels."""
    return VAEConfig(sample_size=768)


def tiny_svd_vae_config() -> VAEConfig:
    return VAEConfig(block_out_channels=(64, 64, 128, 128), sample_size=64)


def _videos(x, num_frames):
    """[B*F, C, H, W] -> [B, C, F, H, W]"""
    bf, c, h, w = x.shape
    return x.reshape(bf // num_frames, num_frames, c, h, w).permute(0, 2, 1, 3, 4)


def _frames(x):
    """[B, C, F, H, W] -> [B*F, C, H, W]"""
    b, c, f, h, w = x.shape
    return x.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w)


class TemporalResnetBlock(nn.Module):
    def __init__(self, c, groups, eps=1e-5):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, c, eps=eps)
        self.conv1 = nn.Conv3d(c, c, (3, 1, 1), padding=(1, 0, 0))
        self.norm2 = nn.GroupNorm(groups, c, eps=eps)
        self.conv2 = nn.Conv3d(c, c, (3, 1, 1), padding=(1, 0, 0))

    def forward(self, x):  # [B, C, F, H, W]
        h = self.conv1(F.silu(self.norm1(x)))
        return x + self.conv2(F.silu(self.norm2(h)))


class AlphaBlender(nn.Module):
    """merge_strategy="learned", switch_spatial_to_temporal_mix=True."""

    def __init__(self):
        super().__init__()
        self.mix_factor = nn.Parameter(torch.zeros(1))

    def forward(self, x_spatial, x_temporal):
        alpha = (1.0 - torch.sigmoid(self.mix_factor)).to(x_spatial.dtype)   # the switched blend
        return alpha * x_spatial + (1.0 - alpha) * x_temporal


class SpatioTemporalResBlock(nn.Module):
    def __init__(self, cin, cout, groups):
        super().__init__()
        self.spatial_res_block = VaeResnet(cin, cout, groups)
        self.temporal_res_block = TemporalResnetBlock(cout, groups)
        self.time_mixer = AlphaBlender()

    def forward(self, x, num_frames):
        xs = _videos(self.spatial_res_block(x), num_frames)
        return _frames(self.time_mixer(xs, self.temporal_res_block(xs)))


class MidBlockTemporalDecoder(nn.Module):
    def __init__(self, c, groups):
        super().__init__()
        self.resnets = nn.ModuleList([SpatioTemporalResBlock(c, c, groups), SpatioTemporalResBlock(c, c, groups)])
        self.attentions = nn.ModuleList([VaeAttention(c, groups)])

    def forward(self, x, num_frames):
        x = self.resnets[0](x, num_frames)
        return self.resnets[1](self.attentions[0](x), num_frames)


class Upsample(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, padding=1)

    def forward(self, x):
        return self.conv(F.interpolate(x, scale_factor=2.0, mode="nearest"))


class UpBlockTemporalDecoder(nn.Module):
    def __init__(self, cin, cout, n, groups, add_up):
        super().__init__()
        self.resnets = nn.ModuleList([SpatioTemporalResBlock(cin if i == 0 else cout, cout, groups)
                                      for i in range(n)])
        self.upsamplers = nn.ModuleList([Upsample(cout)]) if add_up else None

    def forward(self, x, num_frames):
        for r in self.resnets:
            x = r(x, num_frames)
        if self.upsamplers is not None:
            x = self.upsamplers[0](x)
        return x


class TemporalDecoder(nn.Module):
    def __init__(self, cfg: VAEConfig):
        super().__init__()
        boc, g = cfg.block_out_channels, cfg.norm_num_groups
        self.conv_in = nn.Conv2d(cfg.latent_channels, boc[-1], 3, padding=1)
        self.mid_block = MidBlockTemporalDecoder(boc[-1], g)
        self.up_blocks = nn.ModuleList()
        cout = boc[-1]
        for i, c in enumerate(reversed(boc)):
            cin, cout = cout, c
            self.up_blocks.append(UpBlockTemporalDecoder(cin, cout, cfg.layers_per_block + 1, g, i != len(boc) - 1))
        self.conv_norm_out = nn.GroupNorm(g, boc[0], eps=1e-6)
        self.conv_out = nn.Conv2d(boc[0], cfg.out_channels, 3, padding=1)
        self.time_conv_out = nn.Conv3d(cfg.out_channels, cfg.out_channels, (3, 1, 1), padding=(1, 0, 0))

    def forward(self, z, num_frames):
        x = self.mid_block(self.conv_in(z), num_frames)
        for blk in self.up_blocks:
            x = blk(x, num_frames)
        x = self.conv_out(F.silu(self.conv_norm_out(x)))    # stored in the module's dtype
        return _frames(self.time_conv_out(_videos(x, num_frames)))


class AutoencoderKLTemporalDecoder(nn.Module):
    def __init__(self, cfg: VAEConfig):
        super().__init__()
        self.config = cfg
        self.encoder = Encoder(cfg)
        self.quant_conv = nn.Conv2d(2 * cfg.latent_channels, 2 * cfg.latent_channels, 1)
        self.decoder = TemporalDecoder(cfg)

    @property
    def dtype(self):
        return self.quant_conv.weight.dtype

    @property
    def device(self):
        return self.quant_conv.weight.device

    def encode(self, x, return_dict=True):
        dist = DiagonalGaussianDistribution(self.quant_conv(self.encoder(x)))
        if not return_dict:
            return (dist,)
        return AutoencoderKLOutput(latent_dist=dist)

    def decode(self, z, num_frames, return_dict=True):
        x = self.decoder(z, num_frames)
        if not return_dict:
            return (x,)
        return DecoderOutput(sample=x)


def build_svd_vae(cfg: VAEConfig, seed: int = 0, dtype=torch.float32, device="cpu"):
    """`AutoencoderKLTemporalDecoder` with seeded default-init weights, random GroupNorm affines and random
    mix_factors."""
    g = torch.random.get_rng_state()
    torch.manual_seed(seed)
    m = AutoencoderKLTemporalDecoder(cfg)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, nn.GroupNorm):
                mod.weight.copy_(1.0 + 0.3 * torch.randn_like(mod.weight))
                mod.bias.copy_(0.3 * torch.randn_like(mod.bias))
            elif isinstance(mod, AlphaBlender):
                mod.mix_factor.copy_(1.5 * torch.randn_like(mod.mix_factor))
    torch.random.set_rng_state(g)
    return m.to(device=device, dtype=dtype).eval()
