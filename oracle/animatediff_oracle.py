"""ORACLE (test infrastructure, NOT product code).

diffusers' ``UNetMotionModel`` (AnimateDiff), restated on top of ``oracle.unet_oracle``'s pieces with diffusers'
parameter names.

PARITY STATUS: **unpinned.**  The module lives in diffusers (>= 0.25, ``models/unets/unet_motion_model.py``; the
motion module class is ``AnimateDiffTransformer3D`` since 0.30, ``TransformerTemporalModel`` before, with the same
parameters and forward), which is absent from this image; no AnimateDiff checkpoint is available either.  This file
restates the published algorithm:

  * ``forward(sample [B, C, F, H, W], timestep, encoder_hidden_states [B, L, ctx], ...)``: the time embedding (plus
    SDXL's text_time embedding, plus an LCM's cond_proj) is computed per sample and repeated per frame, as is the
    prompt; the frames run through the 2-D UNet as B*F images; the output is reshaped back to [B, C, F, H, W];
  * the Motion blocks run resnet -> transformer (cross-attention blocks only) -> ``motion_modules.j`` per layer, and
    the down-block skip is the output of the motion module; ``UNetMidBlockCrossAttnMotion`` runs resnets.0,
    attentions.0, motion_modules.0 (``use_motion_mid_block``), resnets.1;
  * a motion module on x [B*F, C, H, W]: GroupNorm(32, C, eps 1e-6) over the 5-D video view, tokens regrouped to
    sequences of F frames per (video, pixel), proj_in, ``BasicTransformerBlock``s with double self-attention, GEGLU,
    LayerNorm eps 1e-5 and the sinusoidal position embedding ``pos_embed.pe`` [1, max_seq, C] added after norm1 and
    after norm2, proj_out, and the residual x.

Its structure is pinned by parameter totals derived from that architecture: 22 C^2 + 21 C per motion module with one
transformer block, 453,209,280 motion parameters for the SD-1.5 v1-5-2 geometry (21 modules) and 417,137,600 without
the mid-block module (``tests/test_video_motion_unet_cpu.py``).  These have not been checked against a checkpoint.
"""
import math
from dataclasses import dataclass
from typing import Optional, Tuple, Union

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import unet_oracle as uo

_TO_2D = {"CrossAttnDownBlockMotion": "CrossAttnDownBlock2D", "DownBlockMotion": "DownBlock2D",
          "CrossAttnUpBlockMotion": "CrossAttnUpBlock2D", "UpBlockMotion": "UpBlock2D"}


@dataclass
class MotionConfig(uo.UNetConfig):
    """The keys of diffusers' ``UNetMotionModel.config`` the hot path reads (on top of the 2-D UNet's)."""
    down_block_types: Tuple[str, ...] = ("CrossAttnDownBlockMotion", "CrossAttnDownBlockMotion",
                                         "CrossAttnDownBlockMotion", "DownBlockMotion")
    up_block_types: Tuple[str, ...] = ("UpBlockMotion", "CrossAttnUpBlockMotion", "CrossAttnUpBlockMotion",
                                       "CrossAttnUpBlockMotion")
    motion_num_attention_heads: Union[int, Tuple[int, ...]] = 8
    motion_max_seq_length: int = 32
    temporal_transformer_layers_per_block: Union[int, Tuple[int, ...]] = 1
    use_motion_mid_block: bool = True
    time_cond_proj_dim: Optional[int] = None

    def per_block(self, key):
        v = getattr(self, key)
        return tuple(v) if isinstance(v, (list, tuple)) else (v,) * len(self.block_out_channels)


def v152_config() -> MotionConfig:
    """SD-1.5 with the motion adapter geometry of AnimateDiff v1-5-2 (motion modules in the mid block too)."""
    return MotionConfig()


def no_mid_config() -> MotionConfig:
    """SD-1.5 with a motion adapter without the mid-block module (AnimateDiff v1-5 / v1-5-3 geometry)."""
    return MotionConfig(use_motion_mid_block=False)


def tiny_config() -> MotionConfig:
    """Three blocks of 320 / 640 / 640 channels and one layer each: motion head sizes 40, 80 and 160 (the three the
    frame attention compiles) in seconds-scale parity tests."""
    return MotionConfig(block_out_channels=(320, 640, 640),
                        down_block_types=("CrossAttnDownBlockMotion", "CrossAttnDownBlockMotion", "DownBlockMotion"),
                        up_block_types=("UpBlockMotion", "CrossAttnUpBlockMotion", "CrossAttnUpBlockMotion"),
                        layers_per_block=1, attention_head_dim=(8, 8, 4), transformer_layers_per_block=(1, 1, 1),
                        cross_attention_dim=128, motion_num_attention_heads=(8, 8, 4), sample_size=32)


def tiny_sdxl_config() -> MotionConfig:
    """SDXL-shaped (text_time add embedding, linear projections, no attention in the first block, two transformer
    blocks in the last, two motion blocks in the middle one) at tiny width."""
    return MotionConfig(block_out_channels=(320, 640, 640),
                        down_block_types=("DownBlockMotion", "CrossAttnDownBlockMotion", "CrossAttnDownBlockMotion"),
                        up_block_types=("CrossAttnUpBlockMotion", "CrossAttnUpBlockMotion", "UpBlockMotion"),
                        layers_per_block=1, attention_head_dim=(4, 8, 4), transformer_layers_per_block=(1, 1, 2),
                        cross_attention_dim=128, use_linear_projection=True, addition_embed_type="text_time",
                        addition_time_embed_dim=16, projection_class_embeddings_input_dim=128 + 6 * 16,
                        motion_num_attention_heads=(8, 8, 4), temporal_transformer_layers_per_block=(1, 2, 1),
                        sample_size=32)


def config_2d(cfg: MotionConfig) -> uo.UNetConfig:
    """The 2-D UNet config the motion UNet extends."""
    keep = {k: v for k, v in vars(cfg).items() if k in uo.UNetConfig.__dataclass_fields__}
    keep["down_block_types"] = tuple(_TO_2D[t] for t in cfg.down_block_types)
    keep["up_block_types"] = tuple(_TO_2D[t] for t in cfg.up_block_types)
    return uo.UNetConfig(**keep)


class SinusoidalPositionalEmbedding(nn.Module):
    """diffusers' ``SinusoidalPositionalEmbedding``: x + pe[:, :seq], pe a persistent buffer."""

    def __init__(self, dim, max_seq_length):
        super().__init__()
        pos = torch.arange(max_seq_length).unsqueeze(1)
        div = torch.exp(torch.arange(0, dim, 2) * (-math.log(10000.0) / dim))
        pe = torch.zeros(1, max_seq_length, dim)
        pe[0, :, 0::2] = torch.sin(pos * div)
        pe[0, :, 1::2] = torch.cos(pos * div)
        self.register_buffer("pe", pe)

    def forward(self, x):
        return x + self.pe[:, :x.shape[1]].to(x.dtype)


class MotionTransformerBlock(nn.Module):
    """``BasicTransformerBlock(double_self_attention=True, cross_attention_dim=None, activation_fn="geglu",
    positional_embeddings="sinusoidal")`` on [B*S, F, C] frame sequences."""

    def __init__(self, dim, heads, max_seq_length):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim)
        self.attn1 = uo.Attention(dim, heads)
        self.norm2 = nn.LayerNorm(dim)
        self.attn2 = uo.Attention(dim, heads)
        self.norm3 = nn.LayerNorm(dim)
        self.ff = uo.FeedForward(dim)
        self.pos_embed = SinusoidalPositionalEmbedding(dim, max_seq_length)

    def forward(self, x):
        x = self.attn1(self.pos_embed(self.norm1(x))) + x
        x = self.attn2(self.pos_embed(self.norm2(x))) + x
        return self.ff(self.norm3(x)) + x


class MotionModule(nn.Module):
    """``AnimateDiffTransformer3D`` (``TransformerTemporalModel``)."""

    def __init__(self, dim, heads, depth, max_seq_length, groups=32):
        super().__init__()
        self.norm = nn.GroupNorm(groups, dim, eps=1e-6, affine=True)
        self.proj_in = nn.Linear(dim, dim)
        self.transformer_blocks = nn.ModuleList([MotionTransformerBlock(dim, heads, max_seq_length)
                                                 for _ in range(depth)])
        self.proj_out = nn.Linear(dim, dim)

    def forward(self, x, num_frames):
        bf, c, h, w = x.shape
        b = bf // num_frames
        hs = x.reshape(b, num_frames, c, h, w).permute(0, 2, 1, 3, 4)
        hs = self.norm(hs)
        hs = hs.permute(0, 3, 4, 2, 1).reshape(b * h * w, num_frames, c)
        hs = self.proj_in(hs)
        for blk in self.transformer_blocks:
            hs = blk(hs)
        hs = self.proj_out(hs)
        hs = hs.reshape(b, h, w, num_frames, c).permute(0, 3, 4, 1, 2).reshape(bf, c, h, w)
        return hs + x


class UNetMotionModel(uo.UNet2DConditionModel):
    """Restatement of diffusers ``UNetMotionModel`` (state_dict keys match diffusers')."""

    def __init__(self, cfg: MotionConfig):
        super().__init__(config_2d(cfg))
        self.config = cfg
        boc = cfg.block_out_channels
        heads = cfg.per_block("motion_num_attention_heads")
        depth = cfg.per_block("temporal_transformer_layers_per_block")
        ms = cfg.motion_max_seq_length
        for i, blk in enumerate(self.down_blocks):
            blk.motion_modules = nn.ModuleList([MotionModule(boc[i], heads[i], depth[i], ms, cfg.norm_num_groups)
                                                for _ in blk.resnets])
        if cfg.use_motion_mid_block:
            self.mid_block.motion_modules = nn.ModuleList([MotionModule(boc[-1], heads[-1], 1, ms,
                                                                        cfg.norm_num_groups)])
        rboc, rheads, rdepth = list(reversed(boc)), list(reversed(heads)), list(reversed(depth))
        for i, blk in enumerate(self.up_blocks):
            blk.motion_modules = nn.ModuleList([MotionModule(rboc[i], rheads[i], rdepth[i], ms, cfg.norm_num_groups)
                                                for _ in blk.resnets])
        if cfg.time_cond_proj_dim:  # diffusers' TimestepEmbedding(cond_proj_dim=...): no bias
            self.time_embedding.cond_proj = nn.Linear(cfg.time_cond_proj_dim, boc[0], bias=False)

    def forward(self, sample, timestep, encoder_hidden_states, timestep_cond=None, added_cond_kwargs=None,
                down_block_additional_residuals=None, mid_block_additional_residual=None, return_dict=True,
                **unused):
        cfg = self.config
        b, _, nf, hh, ww = sample.shape
        if not torch.is_tensor(timestep):
            timestep = torch.tensor([timestep], device=sample.device)
        t = timestep.reshape(-1).to(sample.device)
        t = t.expand(b) if t.numel() == 1 else t
        t_emb = uo.timestep_embedding(t, cfg.block_out_channels[0], cfg.flip_sin_to_cos,
                                      cfg.freq_shift).to(sample.dtype)
        if timestep_cond is not None:
            t_emb = t_emb + self.time_embedding.cond_proj(timestep_cond)
        emb = self.time_embedding(t_emb)
        if cfg.addition_embed_type == "text_time":
            tid = uo.timestep_embedding(added_cond_kwargs["time_ids"].flatten(), cfg.addition_time_embed_dim,
                                        cfg.flip_sin_to_cos, cfg.freq_shift).reshape(b, -1).to(sample.dtype)
            emb = emb + self.add_embedding(torch.cat([added_cond_kwargs["text_embeds"], tid], dim=-1))
        emb = emb.repeat_interleave(nf, dim=0)
        ctx = encoder_hidden_states.repeat_interleave(nf, dim=0)
        x = sample.permute(0, 2, 1, 3, 4).reshape(b * nf, -1, hh, ww)
        x = self.conv_in(x)
        skips = [x]
        for blk in self.down_blocks:
            for j, r in enumerate(blk.resnets):
                x = r(x, emb)
                if blk.attentions is not None:
                    x = blk.attentions[j](x, ctx)
                x = blk.motion_modules[j](x, nf)
                skips.append(x)
            if blk.downsamplers is not None:
                x = blk.downsamplers[0](x)
                skips.append(x)
        if down_block_additional_residuals is not None:
            skips = [s + r for s, r in zip(skips, down_block_additional_residuals)]
        mid = self.mid_block
        x = mid.resnets[0](x, emb)
        x = mid.attentions[0](x, ctx)
        if cfg.use_motion_mid_block:
            x = mid.motion_modules[0](x, nf)
        x = mid.resnets[1](x, emb)
        if mid_block_additional_residual is not None:
            x = x + mid_block_additional_residual
        for blk in self.up_blocks:
            for j, r in enumerate(blk.resnets):
                x = r(torch.cat([x, skips.pop()], dim=1), emb)
                if blk.attentions is not None:
                    x = blk.attentions[j](x, ctx)
                x = blk.motion_modules[j](x, nf)
            if blk.upsamplers is not None:
                x = blk.upsamplers[0](x)
        x = self.conv_out(F.silu(self.conv_norm_out(x)))
        x = x.reshape(b, nf, -1, hh, ww).permute(0, 2, 1, 3, 4)
        if not return_dict:
            return (x,)
        return uo.UNetOutput(sample=x)


def motion_parameter_count(m: nn.Module):
    """Parameters of the motion modules (``pos_embed.pe`` is a buffer, not counted)."""
    return sum(p.numel() for n, p in m.named_parameters() if ".motion_modules." in n)


def build_unet(cfg: MotionConfig, seed: int = 0, dtype=torch.float32, device="cpu", randomize_affine=True,
               randomize_pe=False):
    """Seeded default-PyTorch-init motion UNet.  `randomize_affine`: every GroupNorm / LayerNorm gets gamma ~ 1 +
    0.3 N(0, 1) and beta ~ 0.3 N(0, 1) (the Linear biases are PyTorch's nonzero default); `randomize_pe`: the
    position embeddings get 0.5 N(0, 1) instead of the sinusoid, so a frame index mixed up anywhere shows."""
    g = torch.random.get_rng_state()
    torch.manual_seed(seed)
    m = UNetMotionModel(cfg)
    with torch.no_grad():
        for mod in m.modules():
            if randomize_affine and isinstance(mod, (nn.GroupNorm, nn.LayerNorm)):
                mod.weight.copy_(1.0 + 0.3 * torch.randn_like(mod.weight))
                mod.bias.copy_(0.3 * torch.randn_like(mod.bias))
            if randomize_pe and isinstance(mod, SinusoidalPositionalEmbedding):
                mod.pe.copy_(0.5 * torch.randn_like(mod.pe))
    torch.random.set_rng_state(g)
    return m.to(device=device, dtype=dtype).eval()


def sdxl_config() -> MotionConfig:
    """SDXL-base with a motion adapter of 8 motion heads per block (AnimateDiff SDXL geometry; parameter total not
    pinned)."""
    keep = dict(vars(uo.sdxl_config()))
    keep["down_block_types"] = ("DownBlockMotion", "CrossAttnDownBlockMotion", "CrossAttnDownBlockMotion")
    keep["up_block_types"] = ("CrossAttnUpBlockMotion", "CrossAttnUpBlockMotion", "UpBlockMotion")
    return MotionConfig(**keep)
