"""ORACLE (test infrastructure, NOT product code).

PyTorch restatement of IP-Adapter Plus as diffusers' ``load_ip_adapter`` attaches it to a ``UNet2DConditionModel``
(``ip-adapter-plus_sd15``, ``ip-adapter-plus-face_sd15``, ``ip-adapter-plus_sdxl_vit-h``), on top of the oracle UNet
of ``oracle/unet_oracle.py`` and the plain adapter's pieces in ``oracle/ip_adapter_oracle.py`` (neither modified).

``unet.encoder_hid_proj.image_projection_layers[0]`` is diffusers' ``IPAdapterPlusImageProjection``, a small
perceiver ("Resampler") over the image encoder's penultimate hidden states [B, n_img, S_img, D_img]: Q learned
latents, proj_in, `depth` blocks of (cross-attention of the latents over cat(ln0(x), ln1(latents)), FeedForward
with the erf GELU, both residual), proj_out and norm_out.  The Q tokens per image go to the same
``IPAdapterAttnProcessor2_0`` as the plain adapter's (num_tokens=(Q,)).  Parameter names follow diffusers
(``encoder_hid_proj.image_projection_layers.0.latents``, ``...layers.0.attn.to_q.weight``, ...); the totals are
pinned in tests/test_ip_adapter_plus_cpu.py.
"""
import copy
import types

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle.ip_adapter_oracle import (AttnProcessor2_0, IPAdapterAttnProcessor2_0, MultiIPAdapterImageProjection,
                                      _attn2_forward, _unet_forward, cross_attentions)


class ResamplerAttention(nn.Module):
    """diffusers ``Attention(query_dim=dim, dim_head=64, heads=heads, out_bias=False)`` with its default
    processor: to_q / to_k / to_v / to_out.0 without bias, SDPA with scale 1 / sqrt(dim_head)."""

    def __init__(self, dim, heads, dim_head=64):
        super().__init__()
        inner = heads * dim_head
        self.heads, self.scale = heads, dim_head ** -0.5
        self.rescale_output_factor, self.residual_connection = 1.0, False
        self.to_q = nn.Linear(dim, inner, bias=False)
        self.to_k = nn.Linear(dim, inner, bias=False)
        self.to_v = nn.Linear(dim, inner, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(inner, dim, bias=False), nn.Dropout(0.0)])
        self.processor = AttnProcessor2_0()

    def forward(self, x, ctx):
        b, h = x.shape[0], self.heads

        def split(t):
            return t.view(b, -1, h, t.shape[-1] // h).transpose(1, 2)
        o = F.scaled_dot_product_attention(split(self.to_q(x)), split(self.to_k(ctx)), split(self.to_v(ctx)),
                                           scale=self.scale)
        return self.to_out[0](o.transpose(1, 2).reshape(b, -1, o.shape[1] * o.shape[3]))


class GELU(nn.Module):
    def __init__(self, dim_in, dim_out, approximate="none", bias=True):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out, bias=bias)
        self.approximate = approximate

    def forward(self, x):
        return F.gelu(self.proj(x), approximate=self.approximate)


class FeedForward(nn.Module):
    """diffusers ``FeedForward(dim, dim_out, mult, activation_fn="gelu", bias)``: net = [GELU, Dropout, Linear]."""

    def __init__(self, dim, dim_out, mult=4, bias=True):
        super().__init__()
        self.net = nn.ModuleList([GELU(dim, dim * mult, bias=bias), nn.Dropout(0.0),
                                  nn.Linear(dim * mult, dim_out, bias=bias)])

    def forward(self, x):
        for m in self.net:
            x = m(x)
        return x


class IPAdapterPlusImageProjectionBlock(nn.Module):
    def __init__(self, embed_dims=768, dim_head=64, heads=16, ffn_ratio=4):
        super().__init__()
        self.ln0 = nn.LayerNorm(embed_dims)
        self.ln1 = nn.LayerNorm(embed_dims)
        self.attn = ResamplerAttention(embed_dims, heads, dim_head)
        self.ff = nn.Sequential(nn.LayerNorm(embed_dims), FeedForward(embed_dims, embed_dims, ffn_ratio, bias=False))

    def forward(self, x, latents, residual):
        encoder_hidden_states = self.ln0(x)
        latents = self.ln1(latents)
        encoder_hidden_states = torch.cat([encoder_hidden_states, latents], dim=-2)
        latents = self.attn(latents, encoder_hidden_states) + residual
        return self.ff(latents) + latents


class IPAdapterPlusImageProjection(nn.Module):
    def __init__(self, embed_dims=768, output_dims=1024, hidden_dims=1280, depth=4, dim_head=64, heads=16,
                 num_queries=8, ffn_ratio=4):
        super().__init__()
        self.latents = nn.Parameter(torch.randn(1, num_queries, hidden_dims) / hidden_dims ** 0.5)
        self.proj_in = nn.Linear(embed_dims, hidden_dims)
        self.proj_out = nn.Linear(hidden_dims, output_dims)
        self.norm_out = nn.LayerNorm(output_dims)
        self.layers = nn.ModuleList([IPAdapterPlusImageProjectionBlock(hidden_dims, dim_head, heads, ffn_ratio)
                                     for _ in range(depth)])

    def forward(self, x):
        latents = self.latents.repeat(x.size(0), 1, 1)
        x = self.proj_in(x)
        for block in self.layers:
            residual = latents
            latents = block(x, latents, residual)
        return self.norm_out(self.proj_out(latents))


def load_ip_adapter_plus(unet, image_embed_dim=1280, hidden_dims=None, num_queries=16, depth=4, seed=0,
                         scale=1.0, gain=1.0):
    """Attach a randomly initialised IP-Adapter Plus to an oracle UNet in place and return the UNet:
    ``IPAdapterPlusImageProjection(embed_dims=image_embed_dim, output_dims=ctx, hidden_dims, heads =
    hidden_dims / 64, num_queries)`` (hidden_dims defaults to the UNet's cross_attention_dim, as for
    ip-adapter-plus_sd15) with random LayerNorm affines, and ``IPAdapterAttnProcessor2_0(num_tokens=(Q,))`` on
    every cross-attention.  `gain` multiplies the image K / V weights, as in ip_adapter_oracle.load_ip_adapter."""
    cfg = unet.config = copy.copy(unet.config)
    ctx = cfg.cross_attention_dim
    hidden_dims = hidden_dims or ctx
    p0 = next(unet.parameters())
    g = torch.random.get_rng_state()
    torch.manual_seed(seed)
    proj = IPAdapterPlusImageProjection(image_embed_dim, ctx, hidden_dims, depth, 64, hidden_dims // 64, num_queries)
    with torch.no_grad():
        for m in proj.modules():
            if isinstance(m, nn.LayerNorm):
                m.weight.copy_(1.0 + 0.3 * torch.randn_like(m.weight))
                m.bias.copy_(0.3 * torch.randn_like(m.bias))
    unet.encoder_hid_proj = MultiIPAdapterImageProjection([proj]).to(device=p0.device, dtype=p0.dtype)
    for name, attn in cross_attentions(unet):
        proc = IPAdapterAttnProcessor2_0(attn.to_q.out_features, ctx, (num_queries,), scale)
        with torch.no_grad():
            for lin in (proc.to_k_ip[0], proc.to_v_ip[0]):
                lin.weight.mul_(gain)
        attn.processor = proc.to(device=p0.device, dtype=p0.dtype)
        attn.forward = types.MethodType(_attn2_forward, attn)
    for name, m in unet.named_modules():
        if name.endswith(".attn1"):
            m.processor = AttnProcessor2_0()
    torch.random.set_rng_state(g)
    cfg.encoder_hid_dim_type = "ip_image_proj"
    unet.forward = types.MethodType(_unet_forward, unet)
    return unet
