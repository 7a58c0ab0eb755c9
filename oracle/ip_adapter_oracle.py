"""ORACLE (test infrastructure, NOT product code).

PyTorch restatement of a plain IP-Adapter as diffusers' ``load_ip_adapter`` attaches it to a
``UNet2DConditionModel`` (``ip-adapter_sd15``, ``ip-adapter_sdxl_vit-h``, ``ip-adapter_sdxl``), on top of the
oracle UNet of ``oracle/unet_oracle.py`` (not modified: the adapter is attached to a built model).

  * ``unet.encoder_hid_proj`` is a ``MultiIPAdapterImageProjection`` whose ``image_projection_layers[0]`` is an
    ``ImageProjection``: Linear(D_img, T * ctx) then LayerNorm(ctx), eps 1e-5, over [B, n_img, D_img];
  * every ``attn2`` gets an ``IPAdapterAttnProcessor2_0`` submodule ``processor`` (``to_k_ip[0]``,
    ``to_v_ip[0]``: Linear(ctx, C, bias=False), ``scale``: one float per adapter), and its forward takes the
    ``(text, [ip_tokens])`` tuple the UNet passes down:
        to_out(attn(q, k_txt, v_txt) + scale * attn(q, to_k_ip(ip), to_v_ip(ip)))
    with the n_img * T image tokens as one key sequence and the image term skipped when scale == 0;
  * ``unet.config.encoder_hid_dim_type = "ip_image_proj"``; a missing ``image_embeds`` is a ValueError and a
    bare [B, D_img] tensor is read as one image per sample.

Parameter names follow diffusers (``encoder_hid_proj.image_projection_layers.0.image_embeds.weight``,
``<block>.attn2.processor.to_k_ip.0.weight``, ...); the totals are pinned in tests/test_ip_adapter_cpu.py.
"""
import copy
import types

import torch
import torch.nn as nn
import torch.nn.functional as F


class ImageProjection(nn.Module):
    def __init__(self, image_embed_dim=1024, cross_attention_dim=768, num_image_text_embeds=4):
        super().__init__()
        self.num_image_text_embeds = num_image_text_embeds
        self.cross_attention_dim = cross_attention_dim
        self.image_embeds = nn.Linear(image_embed_dim, num_image_text_embeds * cross_attention_dim)
        self.norm = nn.LayerNorm(cross_attention_dim)

    def forward(self, image_embeds):
        b = image_embeds.shape[0]
        x = self.image_embeds(image_embeds.to(self.image_embeds.weight.dtype))
        x = x.reshape(b, self.num_image_text_embeds, -1)
        return self.norm(x)


class MultiIPAdapterImageProjection(nn.Module):
    def __init__(self, layers):
        super().__init__()
        self.image_projection_layers = nn.ModuleList(layers)

    def forward(self, image_embeds):
        out = []
        for emb, layer in zip(image_embeds, self.image_projection_layers):
            b, n = emb.shape[:2]
            x = layer(emb.flatten(0, 1))
            out.append(x.reshape(b, n, *x.shape[1:]))
        return out


class AttnProcessor2_0:
    """The parameter-free processor self-attention keeps."""


class IPAdapterAttnProcessor2_0(nn.Module):
    def __init__(self, hidden_size, cross_attention_dim, num_tokens=(4,), scale=1.0):
        super().__init__()
        self.hidden_size, self.cross_attention_dim = hidden_size, cross_attention_dim
        self.num_tokens = list(num_tokens)
        self.scale = [scale] * len(self.num_tokens)
        self.to_k_ip = nn.ModuleList([nn.Linear(cross_attention_dim, hidden_size, bias=False)
                                      for _ in self.num_tokens])
        self.to_v_ip = nn.ModuleList([nn.Linear(cross_attention_dim, hidden_size, bias=False)
                                      for _ in self.num_tokens])

    def __call__(self, attn, x, ctx):
        text, ip_list = ctx
        b, s, c = x.shape
        h = attn.heads

        def heads(t):
            return t.view(b, -1, h, c // h).transpose(1, 2)
        q = heads(attn.to_q(x))
        o = F.scaled_dot_product_attention(q, heads(attn.to_k(text)), heads(attn.to_v(text)))
        for ip, scale, to_k, to_v in zip(ip_list, self.scale, self.to_k_ip, self.to_v_ip):
            if scale == 0:
                continue
            ip = ip.reshape(b, -1, ip.shape[-1])  # the n_img * T tokens as one sequence
            o = o + scale * F.scaled_dot_product_attention(q, heads(to_k(ip)), heads(to_v(ip)))
        return attn.to_out[0](o.transpose(1, 2).reshape(b, s, c))


def _attn2_forward(self, x, ctx=None):
    if isinstance(ctx, tuple):
        return self.processor(self, x, ctx)
    return type(self).forward(self, x, ctx)


def _unet_forward(self, sample, timestep, encoder_hidden_states, added_cond_kwargs=None, **kw):
    if self.encoder_hid_proj is not None and self.config.encoder_hid_dim_type == "ip_image_proj":
        if not added_cond_kwargs or "image_embeds" not in added_cond_kwargs:
            raise ValueError(f"{type(self).__name__} has the config param `encoder_hid_dim_type` set to "
                             "'ip_image_proj' which requires the keyword argument `image_embeds` to be passed in "
                             "`added_cond_kwargs`")
        emb = added_cond_kwargs["image_embeds"]
        if torch.is_tensor(emb):
            emb = [emb.unsqueeze(1)]  # diffusers' deprecated bare [B, D_img] form
        encoder_hidden_states = (encoder_hidden_states, self.encoder_hid_proj(emb))
    return type(self).forward(self, sample, timestep, encoder_hidden_states, added_cond_kwargs=added_cond_kwargs,
                              **kw)


def cross_attentions(unet):
    """(name, module) of every attn2, in module order."""
    return [(n, m) for n, m in unet.named_modules() if n.endswith(".attn2")]


def load_ip_adapter(unet, image_embed_dim=1024, num_tokens=4, seed=0, scale=1.0, gain=1.0):
    """Attach a randomly initialised plain IP-Adapter to an oracle UNet in place (what diffusers'
    ``load_ip_adapter`` does with a checkpoint) and return the UNet.  `gain` multiplies the image K / V
    weights (random weights at PyTorch's default scale give a small image term)."""
    cfg = unet.config = copy.copy(unet.config)  # the config object may be shared with other models
    ctx = cfg.cross_attention_dim
    p0 = next(unet.parameters())
    g = torch.random.get_rng_state()
    torch.manual_seed(seed)
    proj = ImageProjection(image_embed_dim, ctx, num_tokens)
    with torch.no_grad():
        proj.norm.weight.copy_(1.0 + 0.3 * torch.randn_like(proj.norm.weight))
        proj.norm.bias.copy_(0.3 * torch.randn_like(proj.norm.bias))
    unet.encoder_hid_proj = MultiIPAdapterImageProjection([proj]).to(device=p0.device, dtype=p0.dtype)
    for name, attn in cross_attentions(unet):
        c = attn.to_q.out_features
        proc = IPAdapterAttnProcessor2_0(c, ctx, (num_tokens,), scale)
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


def set_ip_adapter_scale(unet, scale):
    """diffusers' ``set_ip_adapter_scale``: a float for every layer, or an InstantStyle dict {block prefix:
    float} (other layers 0)."""
    for name, attn in cross_attentions(unet):
        if isinstance(scale, dict):
            s = next((v for k, v in scale.items() if name.startswith(k)), 0.0)
        else:
            s = scale
        attn.processor.scale = [float(s)]


def ip_adapter_param_count(unet):
    return sum(p.numel() for n, p in unet.named_parameters()
               if n.startswith("encoder_hid_proj.") or ".processor." in n)
