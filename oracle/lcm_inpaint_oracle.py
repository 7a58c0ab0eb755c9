"""ORACLE (test infrastructure, NOT product code).

The inpainting and LCM UNets of diffusers' ``UNet2DConditionModel``, on top of ``oracle.unet_oracle``:

  * inpainting: ``in_channels: 9`` (latents 4 | mask 1 | masked-image latents 4); unet_oracle's conv_in already
    follows ``cfg.in_channels``, so only the configs are new;
  * LCM: ``time_cond_proj_dim`` adds diffusers' ``TimestepEmbedding.cond_proj`` (a Linear without bias, created
    after linear_1), and the forward takes ``timestep_cond``: ``emb = linear_2(silu(linear_1(t_emb +
    cond_proj(timestep_cond))))``; without ``timestep_cond`` the add is skipped;
  * ``upcast_attention`` (SD-2.1 768-v) is a config field only: diffusers' legacy AttnProcessor reads it (fp32
    QK^T), SDPA -- the oracle's attention -- ignores it.

Parameter totals (diffusers' module definitions): SD-1.5 inpainting 859,535,364, SDXL inpainting 2,567,478,084,
LCM SD-1.5 859,602,884, LCM SDXL 2,567,545,604 (``tests/test_lcm_inpaint_cpu.py``)."""
from dataclasses import dataclass
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import unet_oracle as uo


@dataclass
class UNetConfig(uo.UNetConfig):
    """unet_oracle's config plus the two keys of the LCM and SD-2.1 checkpoints."""
    time_cond_proj_dim: Optional[int] = None
    upcast_attention: bool = False


def config_with(base: uo.UNetConfig, **kw) -> UNetConfig:
    return UNetConfig(**dict(vars(base), **kw))


def sd15_inpaint_config() -> UNetConfig:
    return config_with(uo.sd15_config(), in_channels=9)


def sdxl_inpaint_config() -> UNetConfig:
    return config_with(uo.sdxl_config(), in_channels=9)


def lcm_sd15_config() -> UNetConfig:
    """An LCM-distilled SD-1.5 UNet (LCM-Dreamshaper): a 256-wide guidance embedding."""
    return config_with(uo.sd15_config(), time_cond_proj_dim=256)


def lcm_sdxl_config() -> UNetConfig:
    return config_with(uo.sdxl_config(), time_cond_proj_dim=256)


def tiny_config(**kw) -> UNetConfig:
    """unet_oracle's tiny topology with any of the keys above."""
    return config_with(uo.tiny_config(), **kw)


class TimestepEmbedding(nn.Module):
    """diffusers' TimestepEmbedding with cond_proj_dim: linear_1, cond_proj (no bias), linear_2, in that order."""

    def __init__(self, base: uo.TimestepEmbedding, cond_proj_dim):
        super().__init__()
        self.linear_1 = base.linear_1
        self.cond_proj = nn.Linear(cond_proj_dim, base.linear_1.in_features, bias=False)
        self.linear_2 = base.linear_2

    def forward(self, x, condition=None):
        if condition is not None:
            x = x + self.cond_proj(condition)
        return self.linear_2(F.silu(self.linear_1(x)))


def add_cond_proj(unet: uo.UNet2DConditionModel, cond_proj_dim):
    """Give `unet` diffusers' cond_proj (PyTorch's default Linear init from the current RNG); the other
    parameters are untouched and keep their place in the state dict."""
    te = unet.time_embedding
    new = TimestepEmbedding(te, cond_proj_dim).to(device=te.linear_1.weight.device, dtype=te.linear_1.weight.dtype)
    unet.time_embedding = new
    return unet


def build_unet(cfg: UNetConfig, seed: int = 0, dtype=torch.float32, device="cpu"):
    """unet_oracle.build_unet (the same weights for the same seed), plus cond_proj when cfg.time_cond_proj_dim is
    set, seeded from `seed` as well."""
    m = uo.build_unet(cfg, seed=seed, dtype=torch.float32, device="cpu")
    if getattr(cfg, "time_cond_proj_dim", None):
        g = torch.random.get_rng_state()
        torch.manual_seed(seed + 1)
        add_cond_proj(m, cfg.time_cond_proj_dim)
        torch.random.set_rng_state(g)
    return m.to(device=device, dtype=dtype).eval()


def unet_forward(unet, sample, timestep, encoder_hidden_states, timestep_cond=None, **kw):
    """diffusers' ``UNet2DConditionModel.forward(..., timestep_cond=...)`` of an oracle UNet: unet_oracle's forward,
    with `timestep_cond` handed to the time embedding as its condition.  Every other keyword (added_cond_kwargs,
    ControlNet residuals) goes to unet_oracle's forward.  Returns UNetOutput."""
    if timestep_cond is None:
        return unet(sample, timestep, encoder_hidden_states, **kw)
    hook = unet.time_embedding.register_forward_pre_hook(lambda mod, args: (args[0], timestep_cond))
    try:
        return unet(sample, timestep, encoder_hidden_states, **kw)
    finally:
        hook.remove()

