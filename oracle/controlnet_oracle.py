"""ORACLE (test infrastructure, NOT product code).

CPU/fp32-capable PyTorch restatement of diffusers' ``ControlNetModel`` (module tree and parameter names
follow diffusers), built from the UNet blocks of ``oracle/unet_oracle.py``.  A ControlNet is the UNet's
encoder half (time embedding, conv_in, down blocks, mid block) plus

  * ``controlnet_cond_embedding``: conv_in -> SiLU -> (block -> SiLU) x 2(len(channels) - 1) -> conv_out,
    the blocks alternating a stride-1 conv and a stride-2 conv (padding 1 on every side), no activation
    after conv_out; its output is added to ``conv_in(sample)``;
  * one 1x1 "zero conv" per down-block residual (``controlnet_down_blocks.{i}``) and one for the mid
    output (``controlnet_mid_block``);
  * the residuals times ``conditioning_scale`` -- in guess mode times
    ``logspace(-1, 0, n_down + 1) * conditioning_scale``, the last factor for the mid residual;
  * ``controlnet_conditioning_channel_order="bgr"``: the conditioning image's channels are flipped.

Pinned structurally by the parameter totals in ``tests/test_controlnet_cpu.py``.
"""
from dataclasses import dataclass
from typing import Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import unet_oracle as uo


@dataclass
class ControlNetConfig(uo.UNetConfig):
    """Subset of diffusers ``ControlNetModel.config`` the hot path reads (up_block_types / out_channels of
    the base class are not used)."""
    conditioning_channels: int = 3
    conditioning_embedding_out_channels: Tuple[int, ...] = (16, 32, 96, 256)
    controlnet_conditioning_channel_order: str = "rgb"
    global_pool_conditions: bool = False


def _from_unet(cfg: uo.UNetConfig, **kw) -> ControlNetConfig:
    return ControlNetConfig(**dict(vars(cfg), **kw))


def sd15_config(**kw) -> ControlNetConfig:
    return _from_unet(uo.sd15_config(), **kw)


def sdxl_config(**kw) -> ControlNetConfig:
    return _from_unet(uo.sdxl_config(), **kw)


def tiny_config(**kw) -> ControlNetConfig:
    """The tiny UNet's encoder with diffusers' default conditioning embedding -- seconds-scale parity tests."""
    return _from_unet(uo.tiny_config(), **kw)


class ControlNetConditioningEmbedding(nn.Module):
    def __init__(self, out_channels, cond_channels, channels):
        super().__init__()
        self.conv_in = nn.Conv2d(cond_channels, channels[0], 3, padding=1)
        blocks = []
        for i in range(len(channels) - 1):
            blocks.append(nn.Conv2d(channels[i], channels[i], 3, padding=1))
            blocks.append(nn.Conv2d(channels[i], channels[i + 1], 3, padding=1, stride=2))
        self.blocks = nn.ModuleList(blocks)
        self.conv_out = nn.Conv2d(channels[-1], out_channels, 3, padding=1)

    def forward(self, x):
        x = F.silu(self.conv_in(x))
        for b in self.blocks:
            x = F.silu(b(x))
        return self.conv_out(x)


@dataclass
class ControlNetOutput:
    down_block_res_samples: Tuple[torch.Tensor, ...]
    mid_block_res_sample: torch.Tensor


class ControlNetModel(nn.Module):
    """Restatement of diffusers ``ControlNetModel`` (state_dict keys match diffusers')."""

    def __init__(self, cfg: ControlNetConfig):
        super().__init__()
        self.config = cfg
        boc = cfg.block_out_channels
        temb_dim = boc[0] * 4
        self.conv_in = nn.Conv2d(cfg.in_channels, boc[0], 3, padding=1)
        self.time_embedding = uo.TimestepEmbedding(boc[0], temb_dim)
        if cfg.addition_embed_type == "text_time":
            self.add_embedding = uo.TimestepEmbedding(cfg.projection_class_embeddings_input_dim, temb_dim)
        self.controlnet_cond_embedding = ControlNetConditioningEmbedding(
            boc[0], cfg.conditioning_channels, cfg.conditioning_embedding_out_channels)
        nb = len(boc)
        self.down_blocks = nn.ModuleList()
        zero = [nn.Conv2d(boc[0], boc[0], 1)]
        cout = boc[0]
        for i, t in enumerate(cfg.down_block_types):
            cin, cout = cout, boc[i]
            self.down_blocks.append(uo.DownBlock(
                cfg, cin, cout, temb_dim, t.startswith("CrossAttn"), cfg.attention_head_dim[i],
                cfg.transformer_layers_per_block[i], i != nb - 1))
            zero += [nn.Conv2d(cout, cout, 1) for _ in range(cfg.layers_per_block + (i != nb - 1))]
        self.controlnet_down_blocks = nn.ModuleList(zero)
        self.mid_block = uo.MidBlock(cfg, boc[-1], temb_dim, cfg.attention_head_dim[-1],
                                     cfg.transformer_layers_per_block[-1])
        self.controlnet_mid_block = nn.Conv2d(boc[-1], boc[-1], 1)

    @property
    def dtype(self):
        return self.conv_in.weight.dtype

    @property
    def device(self):
        return self.conv_in.weight.device

    def forward(self, sample, timestep, encoder_hidden_states, controlnet_cond, conditioning_scale=1.0,
                added_cond_kwargs=None, guess_mode=False, return_dict=True, **unused):
        cfg = self.config
        b = sample.shape[0]
        if cfg.controlnet_conditioning_channel_order == "bgr":
            controlnet_cond = torch.flip(controlnet_cond, dims=[1])
        if not torch.is_tensor(timestep):
            timestep = torch.tensor([timestep], device=sample.device)
        t = timestep.reshape(-1).to(sample.device)
        t = t.expand(b) if t.numel() == 1 else t
        t_emb = uo.timestep_embedding(t, cfg.block_out_channels[0], cfg.flip_sin_to_cos,
                                      cfg.freq_shift).to(sample.dtype)
        emb = self.time_embedding(t_emb)
        if cfg.addition_embed_type == "text_time":
            tid = uo.timestep_embedding(added_cond_kwargs["time_ids"].flatten(), cfg.addition_time_embed_dim,
                                        cfg.flip_sin_to_cos, cfg.freq_shift)
            tid = tid.reshape(b, -1).to(sample.dtype)
            emb = emb + self.add_embedding(torch.cat([added_cond_kwargs["text_embeds"], tid], dim=-1))
        x = self.conv_in(sample) + self.controlnet_cond_embedding(controlnet_cond)
        res = [x]
        for blk in self.down_blocks:
            x, outs = blk(x, emb, encoder_hidden_states)
            res.extend(outs)
        x = self.mid_block(x, emb, encoder_hidden_states)
        down = [zc(r) for zc, r in zip(self.controlnet_down_blocks, res)]
        mid = self.controlnet_mid_block(x)
        scales = guess_mode_scales(len(down), conditioning_scale, guess_mode, device=sample.device)
        down = tuple(d * s for d, s in zip(down, scales[:-1]))
        mid = mid * scales[-1]
        if not return_dict:
            return down, mid
        return ControlNetOutput(down, mid)


def guess_mode_scales(n_down, conditioning_scale, guess_mode, device="cpu"):
    """Factor of each of the n_down down residuals and (last) of the mid residual, as diffusers computes
    them: `conditioning_scale` everywhere, or in guess mode logspace(-1, 0, n_down + 1) times it."""
    if guess_mode:
        return torch.logspace(-1, 0, n_down + 1, device=device) * conditioning_scale
    return torch.full((n_down + 1,), float(conditioning_scale), device=device)


def build_controlnet(cfg: ControlNetConfig, seed: int = 0, dtype=torch.float32, device="cpu"):
    """Seeded ControlNet with NO zero-initialised layer: diffusers zeroes the zero convs and the
    embedding's conv_out, which would make a parity check vacuous, so they keep PyTorch's default init
    here; every GroupNorm / LayerNorm affine is random (gamma ~ 1 + 0.3 N(0, 1), beta ~ 0.3 N(0, 1))."""
    g = torch.random.get_rng_state()
    torch.manual_seed(seed)
    m = ControlNetModel(cfg)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, (nn.GroupNorm, nn.LayerNorm)):
                mod.weight.copy_(1.0 + 0.3 * torch.randn_like(mod.weight))
                mod.bias.copy_(0.3 * torch.randn_like(mod.bias))
    torch.random.set_rng_state(g)
    return m.to(device=device, dtype=dtype).eval()
