"""Architecture description of a diffusers ``UNet2DConditionModel`` derived from its config.

The plan builder never touches ``nn.Module`` classes: it consumes ``unet.config`` (any object or
dict with the diffusers field names) and ``unet.state_dict()`` (diffusers parameter names).  This
module turns the config into the ordered block structure both the weight packer and the plan
builder walk, and can synthesise a random state dict of that architecture for benchmarks (there
are no checkpoints offline).
"""
import math
from dataclasses import dataclass, field
from typing import List, Optional

import torch


def cfg_get(cfg, key, default=None):
    if isinstance(cfg, dict):
        return cfg.get(key, default)
    return getattr(cfg, key, default)


def _tuple(v, n):
    if isinstance(v, (list, tuple)):
        assert len(v) == n
        return tuple(v)
    return (v,) * n


@dataclass
class ResnetSpec:
    prefix: str
    cin: int
    cout: int
    eps: Optional[float] = None          # GroupNorm eps (None: the UNet's norm_eps)
    # SVD SpatioTemporalResBlock: `prefix` is the spatial ResnetBlock2D; the temporal
    # TemporalResnetBlock ((3,1,1) convolutions over the frame axis) and the AlphaBlender follow
    temporal_prefix: Optional[str] = None
    mixer: Optional[str] = None          # name of the AlphaBlender's mix_factor parameter

    @property
    def has_shortcut(self):
        return self.cin != self.cout


@dataclass
class TransformerSpec:
    prefix: str
    dim: int
    heads: int
    depth: int
    ctx_dim: int
    linear_proj: bool
    temporal: bool = False  # SVD TransformerSpatioTemporalModel (temporal blocks + time_pos_embed + mixer)

    @property
    def head_dim(self):
        return self.dim // self.heads


@dataclass
class BlockSpec:
    prefix: str
    resnets: List[ResnetSpec]
    attentions: List[Optional[TransformerSpec]]
    sampler: Optional[str] = None  # prefix of the down/up-sampler conv
    cout: int = 0


@dataclass
class ResamplerSpec:
    """Geometry of IP-Adapter Plus's image projection (diffusers ``IPAdapterPlusImageProjection``, the
    "Resampler"): `dim` = hidden width Dh, `heads` attention heads of 64 dims, `depth` blocks with a FeedForward
    of `ff_dim`, and the eps of each block's LayerNorms as ((ln0, ln1, ff.0), ...).  The learned latents are
    the IPAdapterSpec's `tokens` queries; norm_out's eps is the IPAdapterSpec's `norm_eps`."""
    dim: int
    heads: int
    depth: int
    ff_dim: int
    block_eps: tuple

    @property
    def inner(self):
        return self.heads * RESAMPLER_HEAD_DIM


RESAMPLER_HEAD_DIM = 64


@dataclass
class IPAdapterSpec:
    """Geometry of one IP-Adapter (diffusers ``ImageProjection`` or ``IPAdapterPlusImageProjection`` +
    ``IPAdapterAttnProcessor2_0``): image embeddings of `image_embed_dim` are projected to `tokens` context
    tokens of `ctx_dim` each (plain: linear, then LayerNorm with `norm_eps`; Plus: the `resampler` over the
    image's feature tokens, `tokens` learned queries); every cross-attention in `layers` (attn2 prefixes, in
    schedule order) attends to them with its own K / V projections and a scale read per call."""
    image_embed_dim: int
    tokens: int
    ctx_dim: int
    layers: tuple
    norm_eps: float = 1e-5
    resampler: Optional[ResamplerSpec] = None  # IP-Adapter Plus


@dataclass
class MotionSpec:
    """One AnimateDiff motion module (diffusers ``AnimateDiffTransformer3D``, formerly
    ``TransformerTemporalModel``) at `prefix`: a video GroupNorm of `groups` groups, proj_in, `depth`
    BasicTransformerBlocks whose two self-attentions run across the frames with the sinusoidal position
    embedding of `max_seq_len` positions, proj_out, and the residual.  `after`: the module that produces its
    input (the layer's resnet or transformer prefix)."""
    prefix: str
    dim: int
    heads: int
    depth: int
    max_seq_len: int
    groups: int
    after: str = ""

    @property
    def head_dim(self):
        return self.dim // self.heads


# head sizes sfb_frame_attention compiles
MOTION_HEAD_DIMS = (40, 80, 160)
MOTION_MAX_FRAMES = 32


@dataclass
class UNetSpec:
    in_channels: int
    out_channels: int
    block_out_channels: tuple
    temb_dim: int
    groups: int
    eps: float
    flip_sin_to_cos: bool
    freq_shift: float
    cross_attention_dim: int
    addition_embed_type: Optional[str]
    addition_time_embed_dim: Optional[int]
    add_in_dim: Optional[int]
    down: List[BlockSpec] = field(default_factory=list)
    mid: Optional[BlockSpec] = None
    up: List[BlockSpec] = field(default_factory=list)
    num_frames: int = 0     # > 0: UNetSpatioTemporalConditionModel (SVD)
    # ControlNetModel (cond_channels > 0): conditioning image channels, the embedding's channel counts,
    # and whether the image arrives in BGR order (controlnet_conditioning_channel_order)
    cond_channels: int = 0
    cond_embed_channels: tuple = ()
    cond_bgr: bool = False
    ip: Optional[IPAdapterSpec] = None  # an IP-Adapter is loaded (UNet only)
    # LCM (diffusers time_cond_proj_dim, UNet only): width of the guidance embedding `timestep_cond` that
    # time_embedding.cond_proj (no bias) projects and adds to the sinusoidal timestep embedding; 0: none
    time_cond_dim: int = 0
    # AnimateDiff (diffusers UNetMotionModel): the motion modules in schedule order; [] for every other UNet
    motion: List[MotionSpec] = field(default_factory=list)

    @property
    def temporal(self):
        return self.num_frames > 0

    def all_resnets(self):
        """Every block that owns a `time_emb_proj` (SVD: spatial and temporal halves)."""
        out = []
        for b in self.down + [self.mid] + self.up:
            for r in b.resnets:
                out.append(r)
                if r.temporal_prefix:
                    out.append(ResnetSpec(r.temporal_prefix, r.cout, r.cout, r.eps))
        return out

    def cross_attention_layers(self):
        """(attn2 prefix, TransformerSpec) of every cross-attention, in the order the plan runs them."""
        return [(f"{t.prefix}.transformer_blocks.{d}.attn2", t)
                for b in self.down + [self.mid] + self.up for t in b.attentions if t is not None
                for d in range(t.depth)]

    def residual_channels(self):
        """Channels of the ControlNet's down-block residuals, in diffusers' order: conv_in's output, then
        every resnet (+ transformer) output and every downsampler output of the down path."""
        out = [self.block_out_channels[0]]
        for b in self.down:
            out += [b.cout] * len(b.resnets) + ([b.cout] if b.sampler else [])
        return out


_SUPPORTED_DOWN = ("CrossAttnDownBlock2D", "DownBlock2D")
_SUPPORTED_UP = ("CrossAttnUpBlock2D", "UpBlock2D")


def spec_from_config(cfg) -> UNetSpec:
    if is_svd_config(cfg):
        return svd_spec_from_config(cfg)
    if is_motion_config(cfg):
        return motion_spec_from_config(cfg)
    # an IP-Adapter sets encoder_hid_dim_type = "ip_image_proj"; its geometry is read from the module
    # (ip_adapter_spec), not the config.  A ControlNet never receives image embeddings: it keeps refusing it.
    spec, tf, layers = _encoder_spec(cfg, out_channels=cfg_get(cfg, "out_channels", 4), accept_ip=True,
                                     accept_time_cond=True)
    up_types = tuple(cfg_get(cfg, "up_block_types"))
    for t in up_types:
        if t not in _SUPPORTED_UP:
            raise NotImplementedError(f"up block type {t} is not supported by the H100 path")
    boc = spec.block_out_channels
    nb = len(boc)
    rboc = list(reversed(boc))
    cout = rboc[0]
    for i, t in enumerate(up_types):
        cprev, cout = cout, rboc[i]
        cin = rboc[min(i + 1, nb - 1)]
        p = f"up_blocks.{i}"
        res = []
        for j in range(layers + 1):
            skip = cin if j == layers else cout
            rin = cprev if j == 0 else cout
            res.append(ResnetSpec(f"{p}.resnets.{j}", rin + skip, cout))
        att = [tf(f"{p}.attentions.{j}", cout, nb - 1 - i) if t.startswith("CrossAttn") else None
               for j in range(layers + 1)]
        spec.up.append(BlockSpec(p, res, att, f"{p}.upsamplers.0.conv" if i != nb - 1 else None,
                                 cout))
    return spec


def _encoder_spec(cfg, out_channels, accept_ip=False, accept_time_cond=False):
    """The part of the architecture a UNet and a ControlNet share (time embedding, conv_in, down blocks,
    mid block), with every check of the config keys both carry.  Returns (spec without up blocks, the
    transformer-spec factory, layers per block).  `accept_ip`: encoder_hid_dim_type="ip_image_proj" (an
    IP-Adapter) passes; the caller reads the adapter from the module.  `accept_time_cond`: time_cond_proj_dim
    (an LCM's guidance embedding) passes."""
    boc = tuple(cfg_get(cfg, "block_out_channels"))
    nb = len(boc)
    down_types = tuple(cfg_get(cfg, "down_block_types"))
    for t in down_types:
        if t not in _SUPPORTED_DOWN:
            raise NotImplementedError(f"down block type {t} is not supported by the H100 path")
    # upcast_attention (SD-2.1 768-v) only makes diffusers' legacy AttnProcessor compute QK^T in fp32; the fused
    # attention always accumulates QK^T and runs the softmax in fp32, so both values compute the same
    for key in ("class_embed_type", "encoder_hid_dim_type", "time_cond_proj_dim",
                "resnet_time_scale_shift", "dual_cross_attention", "only_cross_attention",
                "time_embedding_act_fn", "attention_type"):
        v = cfg_get(cfg, key)
        if accept_ip and key == "encoder_hid_dim_type" and v == "ip_image_proj":
            continue
        if accept_time_cond and key == "time_cond_proj_dim" and v is not None:
            continue
        if v not in (None, False, "default", "positional"):
            raise NotImplementedError(f"UNet config {key}={v!r} is not supported by the H100 path")
    # fields whose only supported value is the SD-1.5 / SDXL one: anything else would compile and
    # return wrong numerics, so it is refused by name
    required = {
        "act_fn": ("silu", "swish"), "time_embedding_type": ("positional",),
        "conv_in_kernel": (3,), "conv_out_kernel": (3,), "downsample_padding": (1,),
        "mid_block_scale_factor": (1, 1.0), "resnet_out_scale_factor": (1, 1.0),
        "resnet_skip_time_act": (False,), "mid_block_only_cross_attention": (None, False),
        "cross_attention_norm": (None,), "attention_bias": (False,), "num_class_embeds": (None,),
        "addition_embed_type_num_heads": (64,), "timestep_post_act": (None,),
        "time_embedding_dim": (None,), "class_embeddings_concat": (False,),
        "reverse_transformer_layers_per_block": (None,), "dropout": (0, 0.0),
        "center_input_sample": (False,), "encoder_hid_dim": (None,), "upcast_attention": (None, False, True),
    }
    for key, allowed in required.items():
        v = cfg_get(cfg, key, allowed[0])
        if v not in allowed:
            raise NotImplementedError(f"UNet config {key}={v!r} is not supported by the H100 path "
                                      f"(supported: {allowed})")
    mid_type = cfg_get(cfg, "mid_block_type", "UNetMidBlock2DCrossAttn")
    if mid_type not in (None, "UNetMidBlock2DCrossAttn"):
        raise NotImplementedError(f"mid block type {mid_type}")
    layers = cfg_get(cfg, "layers_per_block", 2)
    if isinstance(layers, (list, tuple)):
        if len(set(layers)) != 1:
            raise NotImplementedError("per-block layers_per_block")
        layers = layers[0]
    # `num_attention_heads` if given, else diffusers' historical alias `attention_head_dim`
    heads_cfg = cfg_get(cfg, "num_attention_heads") or cfg_get(cfg, "attention_head_dim")
    heads = _tuple(heads_cfg, nb)
    depth = _tuple(cfg_get(cfg, "transformer_layers_per_block", 1), nb)
    ctx = cfg_get(cfg, "cross_attention_dim")
    if isinstance(ctx, (list, tuple)):
        if len(set(ctx)) != 1:
            raise NotImplementedError("per-block cross_attention_dim")
        ctx = ctx[0]
    linear = bool(cfg_get(cfg, "use_linear_projection", False))
    add_type = cfg_get(cfg, "addition_embed_type")
    if add_type not in (None, "text_time"):
        raise NotImplementedError(f"addition_embed_type={add_type}")
    cin = cfg_get(cfg, "in_channels", 4)
    if cin > 14:
        # conv_in's im2col rows hold 9 * in_channels columns in at most two 64-wide K blocks
        raise NotImplementedError(f"UNet config in_channels={cin} is not supported by the H100 path "
                                  "(supported: 1 to 14)")
    time_cond = cfg_get(cfg, "time_cond_proj_dim") if accept_time_cond else None
    if time_cond is not None and (int(time_cond) <= 0 or int(time_cond) % 8):
        # cond_proj runs on sfb_small_linear, whose K is read in 8-element vectors
        raise NotImplementedError(f"UNet config time_cond_proj_dim={time_cond!r} is not supported by the H100 "
                                  "path (supported: a positive multiple of 8)")
    spec = UNetSpec(
        in_channels=cin, out_channels=out_channels,
        block_out_channels=boc, temb_dim=boc[0] * 4, groups=cfg_get(cfg, "norm_num_groups", 32),
        eps=cfg_get(cfg, "norm_eps", 1e-5), flip_sin_to_cos=cfg_get(cfg, "flip_sin_to_cos", True),
        freq_shift=float(cfg_get(cfg, "freq_shift", 0)), cross_attention_dim=ctx,
        addition_embed_type=add_type,
        addition_time_embed_dim=cfg_get(cfg, "addition_time_embed_dim"),
        add_in_dim=cfg_get(cfg, "projection_class_embeddings_input_dim"), time_cond_dim=int(time_cond or 0))

    def tf(prefix, dim, i):
        return TransformerSpec(prefix, dim, heads[i], depth[i], ctx, linear)

    cout = boc[0]
    for i, t in enumerate(down_types):
        cin, cout = cout, boc[i]
        p = f"down_blocks.{i}"
        res = [ResnetSpec(f"{p}.resnets.{j}", cin if j == 0 else cout, cout) for j in range(layers)]
        att = [tf(f"{p}.attentions.{j}", cout, i) if t.startswith("CrossAttn") else None
               for j in range(layers)]
        spec.down.append(BlockSpec(p, res, att, f"{p}.downsamplers.0.conv" if i != nb - 1 else None,
                                   cout))
    c = boc[-1]
    spec.mid = BlockSpec("mid_block",
                         [ResnetSpec("mid_block.resnets.0", c, c),
                          ResnetSpec("mid_block.resnets.1", c, c)],
                         [tf("mid_block.attentions.0", c, nb - 1)], None, c)
    return spec, tf, layers


def controlnet_spec_from_config(cfg) -> UNetSpec:
    """diffusers ``ControlNetModel``: the UNet's encoder half (``up = []``) plus the conditioning fields.
    Every channel count of the conditioning embedding must be a multiple of 8 (the few-channel conv kernel
    reads 8-channel vectors) and the conditioning image may have 1 to 8 channels."""
    if cfg_get(cfg, "global_pool_conditions", False):
        raise NotImplementedError("ControlNet config global_pool_conditions=True (shuffle models) is not "
                                  "supported by the H100 path")
    order = cfg_get(cfg, "controlnet_conditioning_channel_order", "rgb")
    if order not in ("rgb", "bgr"):
        raise NotImplementedError(f"ControlNet config controlnet_conditioning_channel_order={order!r} is not "
                                  "supported by the H100 path (supported: 'rgb', 'bgr')")
    cc = cfg_get(cfg, "conditioning_channels", 3)
    if not 1 <= cc <= 8:
        raise NotImplementedError(f"ControlNet config conditioning_channels={cc} is not supported by the H100 "
                                  "path (supported: 1 to 8)")
    emb = tuple(cfg_get(cfg, "conditioning_embedding_out_channels", (16, 32, 96, 256)))
    if not emb or any(c <= 0 or c % 8 for c in emb) or emb[-1] < 64:
        raise NotImplementedError(f"ControlNet config conditioning_embedding_out_channels={emb} is not supported "
                                  "by the H100 path (every count a multiple of 8, the last one at least 64)")
    spec, _, _ = _encoder_spec(cfg, out_channels=0)
    spec.cond_channels, spec.cond_embed_channels, spec.cond_bgr = cc, emb, order == "bgr"
    return spec


def ip_adapter_geometry(spec: UNetSpec, image_embed_dim, tokens=4, norm_eps=1e-5) -> IPAdapterSpec:
    """The IPAdapterSpec of a plain IP-Adapter on `spec`'s UNet (every cross-attention carries it)."""
    return IPAdapterSpec(int(image_embed_dim), int(tokens), spec.cross_attention_dim,
                         tuple(p for p, _ in spec.cross_attention_layers()), float(norm_eps))


def ip_adapter_plus_geometry(spec: UNetSpec, image_embed_dim, dim, tokens=16, depth=4, ff_mult=4,
                             eps=1e-5) -> IPAdapterSpec:
    """The IPAdapterSpec of an IP-Adapter Plus on `spec`'s UNet: a Resampler of hidden width `dim` (dim / 64
    heads) with `tokens` learned queries and `depth` blocks, every LayerNorm with `eps`."""
    ip = ip_adapter_geometry(spec, image_embed_dim, tokens, eps)
    ip.resampler = ResamplerSpec(int(dim), int(dim) // RESAMPLER_HEAD_DIM, int(depth), int(dim) * ff_mult,
                                 ((float(eps),) * 3,) * depth)
    return ip


_FACEID_PROJECTIONS = ("IPAdapterFaceIDImageProjection", "IPAdapterFaceIDPlusImageProjection")


def ip_adapter_spec(unet, spec: UNetSpec) -> IPAdapterSpec:
    """Read the IP-Adapter loaded on a diffusers UNet (``pipe.load_ip_adapter``): exactly one
    ``ImageProjection`` or ``IPAdapterPlusImageProjection`` in ``unet.encoder_hid_proj`` and, on every
    cross-attention, an ``IPAdapterAttnProcessor2_0``-like ``processor`` with ``to_k_ip[0]`` / ``to_v_ip[0]``
    and a one-float ``scale``.  Anything else is refused by name: it would otherwise compute something
    different."""
    def refuse(what):
        raise NotImplementedError(f"sfast (H100 build): {what} is not supported by the H100 path (one "
                                  "IP-Adapter with an ImageProjection or an IPAdapterPlusImageProjection is)")
    if spec.temporal:
        refuse("an IP-Adapter on the SVD UNet (UNetSpatioTemporalConditionModel)")
    if getattr(unet, "text_encoder_hid_proj", None) is not None:
        refuse("text_encoder_hid_proj (a text projection next to the IP-Adapter)")
    proj = getattr(unet, "encoder_hid_proj", None)
    if proj is None:
        refuse("encoder_hid_dim_type='ip_image_proj' without an encoder_hid_proj")
    layers = getattr(proj, "image_projection_layers", None)
    if layers is None:
        refuse(f"encoder_hid_proj of type {type(proj).__name__}")
    layers = list(layers)
    if len(layers) != 1:
        refuse(f"more than one IP-Adapter at once ({len(layers)} image projections)")
    lay = layers[0]
    kind = type(lay).__name__
    if kind in _FACEID_PROJECTIONS:
        refuse(f"{kind} (IP-Adapter FaceID)")
    if kind == "IPAdapterPlusImageProjection":
        ip = _resampler_ip_spec(lay, spec, refuse)
        ctx = ip.ctx_dim
    elif kind != "ImageProjection":
        refuse(f"image projection {kind}")
    else:
        lin, norm = lay.image_embeds, lay.norm
        tokens = int(getattr(lay, "num_image_text_embeds", 0) or 0)
        ctx = int(getattr(lay, "cross_attention_dim", norm.normalized_shape[0]))
        if ctx != spec.cross_attention_dim or tuple(norm.normalized_shape) != (ctx,) or \
                tokens <= 0 or lin.out_features != tokens * ctx:
            refuse(f"ImageProjection geometry (tokens {tokens}, context {ctx}, linear {lin.out_features}, UNet "
                   f"cross_attention_dim {spec.cross_attention_dim})")
        ip = ip_adapter_geometry(spec, lin.in_features, tokens, norm.eps)
    dims = dict(spec.cross_attention_layers())
    for prefix in ip.layers:
        proc = getattr(unet.get_submodule(prefix), "processor", None)
        k, v = getattr(proc, "to_k_ip", None), getattr(proc, "to_v_ip", None)
        if k is None or v is None:
            refuse(f"{prefix}.processor of type {type(proc).__name__} (no to_k_ip / to_v_ip)")
        if len(k) != 1 or len(v) != 1:
            refuse(f"more than one IP-Adapter at once ({prefix}.processor has {len(k)} image K projections)")
        C = dims[prefix].dim
        for lin_ in (k[0], v[0]):
            if tuple(lin_.weight.shape) != (C, ctx) or getattr(lin_, "bias", None) is not None:
                refuse(f"{prefix}.processor image K/V projection of shape {tuple(lin_.weight.shape)}")
        ip_scale_of(proc, prefix)
    return ip


_DEFAULT_ATTN_PROCESSORS = ("AttnProcessor2_0", "AttnProcessor")


def _resampler_ip_spec(lay, spec: UNetSpec, refuse) -> IPAdapterSpec:
    """The IPAdapterSpec of an ``IPAdapterPlusImageProjection``, read from the module; everything the plan would
    compute differently (another head size, a bias diffusers' layers do not have, a non-default attention
    processor, a tanh GELU, a missing sub-module) is refused by name."""
    kind = "IPAdapterPlusImageProjection"
    parts = {n: getattr(lay, n, None) for n in ("latents", "proj_in", "layers", "proj_out", "norm_out")}
    missing = [n for n, v in parts.items() if v is None]
    if missing:
        refuse(f"{kind} without {' / '.join(missing)} (not diffusers' IP-Adapter Plus layout)")
    lat, proj_in, blocks, proj_out, norm_out = parts.values()
    if lat.dim() != 3 or lat.shape[0] != 1:
        refuse(f"{kind}.latents of shape {tuple(lat.shape)} (expected [1, num_queries, hidden_dims])")
    tokens, dh = int(lat.shape[1]), int(lat.shape[2])
    ctx = spec.cross_attention_dim
    if dh % RESAMPLER_HEAD_DIM:
        refuse(f"{kind} hidden_dims {dh} (not a multiple of {RESAMPLER_HEAD_DIM})")
    if proj_in.out_features != dh or proj_in.bias is None or proj_out.in_features != dh or \
            proj_out.out_features != ctx or proj_out.bias is None:
        refuse(f"{kind} proj_in / proj_out geometry (hidden_dims {dh}, proj_in {tuple(proj_in.weight.shape)}, "
               f"proj_out {tuple(proj_out.weight.shape)}, UNet cross_attention_dim {ctx})")

    def layer_norm(m, what, c):
        if m is None or tuple(getattr(m, "normalized_shape", ())) != (c,) or getattr(m, "weight", None) is None \
                or getattr(m, "bias", None) is None:
            refuse(f"{kind} {what} (expected an affine LayerNorm over {c})")
        return float(m.eps)

    def no_bias_linear(m, what, shape):
        if m is None or tuple(m.weight.shape) != shape:
            refuse(f"{kind} {what} of shape {None if m is None else tuple(m.weight.shape)} (expected {shape})")
        if getattr(m, "bias", None) is not None:
            refuse(f"{kind} {what} with a bias (diffusers' layer has none)")

    norm_eps = layer_norm(norm_out, "norm_out", ctx)
    blocks = list(blocks)
    if not blocks:
        refuse(f"{kind} with no blocks")
    heads = ff_dim = None
    block_eps = []
    for i, blk in enumerate(blocks):
        b = f"layers.{i}"
        attn, ff = getattr(blk, "attn", None), getattr(blk, "ff", None)
        if attn is None or ff is None or not hasattr(attn, "to_q"):
            refuse(f"{kind} {b} without attn / ff")
        h = int(getattr(attn, "heads", 0) or 0)
        inner = attn.to_q.out_features
        if h <= 0 or inner != h * RESAMPLER_HEAD_DIM:
            refuse(f"{kind} {b}.attn with dim_head {inner / max(h, 1):g} (heads {h}; dim_head "
                   f"{RESAMPLER_HEAD_DIM} is)")
        if heads is not None and h != heads:
            refuse(f"{kind} with a different head count per block")
        heads = h
        proc = getattr(attn, "processor", None)
        if type(proc).__name__ not in _DEFAULT_ATTN_PROCESSORS:
            refuse(f"{kind} {b}.attn.processor of type {type(proc).__name__} (diffusers' default "
                   "AttnProcessor2_0 is)")
        if abs(float(getattr(attn, "scale", RESAMPLER_HEAD_DIM ** -0.5)) - RESAMPLER_HEAD_DIM ** -0.5) > 1e-12 or \
                float(getattr(attn, "rescale_output_factor", 1.0)) != 1.0 or \
                getattr(attn, "residual_connection", False):
            refuse(f"{kind} {b}.attn with a non-default scale / rescale_output_factor / residual_connection")
        for n in ("to_q", "to_k", "to_v"):
            no_bias_linear(getattr(attn, n, None), f"{b}.attn.{n}", (inner, dh))
        to_out = getattr(attn, "to_out", None)
        no_bias_linear(to_out[0] if to_out is not None else None, f"{b}.attn.to_out.0", (dh, inner))
        net = getattr(ff[1], "net", None) if len(ff) == 2 else None
        if net is None or len(net) != 3 or not hasattr(net[0], "proj"):
            refuse(f"{kind} {b}.ff (expected Sequential(LayerNorm, FeedForward))")
        if getattr(net[0], "approximate", "none") != "none" or type(net[0]).__name__ != "GELU":
            refuse(f"{kind} {b}.ff activation {type(net[0]).__name__}"
                   f"(approximate={getattr(net[0], 'approximate', None)!r}); the erf GELU is")
        f = net[0].proj.out_features
        if ff_dim is not None and f != ff_dim:
            refuse(f"{kind} with a different FeedForward width per block")
        ff_dim = f
        no_bias_linear(net[0].proj, f"{b}.ff.1.net.0.proj", (f, dh))
        no_bias_linear(net[2], f"{b}.ff.1.net.2", (dh, f))
        block_eps.append((layer_norm(getattr(blk, "ln0", None), f"{b}.ln0", dh),
                          layer_norm(getattr(blk, "ln1", None), f"{b}.ln1", dh),
                          layer_norm(ff[0], f"{b}.ff.0", dh)))
    ip = ip_adapter_geometry(spec, proj_in.in_features, tokens, norm_eps)
    ip.resampler = ResamplerSpec(dh, heads, len(blocks), ff_dim, tuple(block_eps))
    return ip


def ip_scale_of(proc, prefix):
    """The one float an IPAdapterAttnProcessor2_0's `scale` holds (set_ip_adapter_scale writes it in place)."""
    scale = getattr(proc, "scale", None)
    if not isinstance(scale, (list, tuple)) or len(scale) != 1:
        raise NotImplementedError(f"sfast (H100 build): {prefix}.processor.scale={scale!r} is not supported by "
                                  "the H100 path (one float per layer)")
    s = scale[0]
    if isinstance(s, (list, tuple)) or (torch.is_tensor(s) and s.numel() != 1):
        raise NotImplementedError(f"sfast (H100 build): per-image IP-Adapter scale lists ({prefix}.processor."
                                  f"scale={scale!r}) are not supported by the H100 path")
    return float(s)


_MOTION_TYPES = {"CrossAttnDownBlockMotion": "CrossAttnDownBlock2D", "DownBlockMotion": "DownBlock2D",
                 "CrossAttnUpBlockMotion": "CrossAttnUpBlock2D", "UpBlockMotion": "UpBlock2D"}


def is_motion_config(cfg):
    return any(str(t).endswith("Motion") for t in (cfg_get(cfg, "down_block_types") or ()))


class _Config2D:
    """A UNetMotionModel config read as the 2-D UNet config it extends: the Motion block types become their
    2-D counterparts, every other key is the config's own."""

    def __init__(self, cfg):
        self._cfg = cfg
        self._over = {k: tuple(_MOTION_TYPES.get(t, t) for t in cfg_get(cfg, k))
                      for k in ("down_block_types", "up_block_types")}

    def __getattr__(self, key):
        if key.startswith("_"):
            raise AttributeError(key)
        if key in self._over:
            return self._over[key]
        v = cfg_get(self._cfg, key, _MISSING)
        if v is _MISSING:
            raise AttributeError(key)
        return v


_MISSING = object()


def motion_spec_from_config(cfg) -> UNetSpec:
    """diffusers ``UNetMotionModel`` (AnimateDiff): the SD-1.5 / SDXL UNet it extends, built from the same
    config with the Motion block types read as their 2-D counterparts, plus one MotionSpec per motion module in
    schedule order -- after every (resnet, transformer) layer of the down and up blocks and, with
    use_motion_mid_block, between the mid block's transformer and its second resnet.  What the plan would compute
    differently is refused by name."""
    def refuse(what, supported):
        raise NotImplementedError(f"UNetMotionModel config {what} is not supported by the H100 path "
                                  f"(supported: {supported})")
    for t in tuple(cfg_get(cfg, "down_block_types")) + tuple(cfg_get(cfg, "up_block_types")):
        if t not in _MOTION_TYPES:
            raise NotImplementedError(f"block type {t} is not supported by the H100 path in a UNetMotionModel")
    spec = spec_from_config(_Config2D(cfg))
    boc = spec.block_out_channels
    nb = len(boc)
    mid_layers = cfg_get(cfg, "mid_block_layers", 1)
    if mid_layers != 1:
        refuse(f"mid_block_layers={mid_layers!r}", "1")
    mid_depth = cfg_get(cfg, "transformer_layers_per_mid_block")
    if mid_depth is not None:
        spec.mid.attentions[0].depth = int(mid_depth)
    heads = _tuple(cfg_get(cfg, "motion_num_attention_heads", 8), nb)
    depth = _tuple(cfg_get(cfg, "temporal_transformer_layers_per_block", 1), nb)
    for key, fwd in (("reverse_motion_num_attention_heads", heads),
                     ("reverse_temporal_transformer_layers_per_block", depth)):
        v = cfg_get(cfg, key)
        if v is not None and _tuple(v, nb) != tuple(reversed(fwd)):
            refuse(f"{key}={v!r}", f"None or the reversed forward values {tuple(reversed(fwd))}")
    max_seq = int(cfg_get(cfg, "motion_max_seq_length", 32))
    if not 1 <= max_seq <= MOTION_MAX_FRAMES:
        refuse(f"motion_max_seq_length={max_seq}", f"1 to {MOTION_MAX_FRAMES}")
    groups = int(cfg_get(cfg, "motion_norm_num_groups", 32))
    if groups != spec.groups:
        refuse(f"motion_norm_num_groups={groups}", f"norm_num_groups = {spec.groups}")

    def motion(prefix, dim, h, d, after):
        if dim % h or dim // h not in MOTION_HEAD_DIMS:
            refuse(f"motion head_dim {dim}/{h} at {prefix}", f"one of {MOTION_HEAD_DIMS}")
        return MotionSpec(prefix, dim, h, int(d), max_seq, groups, after)

    for i, blk in enumerate(spec.down):
        for j, (r, t) in enumerate(zip(blk.resnets, blk.attentions)):
            spec.motion.append(motion(f"{blk.prefix}.motion_modules.{j}", blk.cout, heads[i], depth[i],
                                      (t or r).prefix))
    if cfg_get(cfg, "use_motion_mid_block", True):
        mdepth = cfg_get(cfg, "temporal_transformer_layers_per_mid_block", 1)
        if isinstance(mdepth, (list, tuple)):
            if len(mdepth) != 1:
                refuse(f"temporal_transformer_layers_per_mid_block={mdepth!r}", "one value (mid_block_layers = 1)")
            mdepth = mdepth[0]
        spec.motion.append(motion("mid_block.motion_modules.0", boc[-1], heads[-1], mdepth,
                                  spec.mid.attentions[0].prefix))
    rheads, rdepth = tuple(reversed(heads)), tuple(reversed(depth))
    for i, blk in enumerate(spec.up):
        for j, (r, t) in enumerate(zip(blk.resnets, blk.attentions)):
            spec.motion.append(motion(f"{blk.prefix}.motion_modules.{j}", blk.cout, rheads[i], rdepth[i],
                                      (t or r).prefix))
    return spec


def motion_pe(max_seq_len, dim):
    """diffusers ``SinusoidalPositionalEmbedding.pe`` [1, max_seq_len, dim]: sin on the even columns, cos on the odd
    ones, frequencies exp(-2i ln(10000) / dim)."""
    pos = torch.arange(max_seq_len, dtype=torch.float32).unsqueeze(1)
    div = torch.exp(torch.arange(0, dim, 2, dtype=torch.float32) * (-math.log(10000.0) / dim))
    pe = torch.zeros(1, max_seq_len, dim)
    pe[0, :, 0::2] = torch.sin(pos * div)
    pe[0, :, 1::2] = torch.cos(pos * div)
    return pe


_SVD_DOWN = ("CrossAttnDownBlockSpatioTemporal", "DownBlockSpatioTemporal")
_SVD_UP = ("CrossAttnUpBlockSpatioTemporal", "UpBlockSpatioTemporal")


def is_svd_config(cfg):
    return any("SpatioTemporal" in t for t in (cfg_get(cfg, "down_block_types") or ()))


def svd_spec_from_config(cfg) -> UNetSpec:
    """diffusers UNetSpatioTemporalConditionModel (Stable Video Diffusion)."""
    boc = tuple(cfg_get(cfg, "block_out_channels"))
    nb = len(boc)
    down_types, up_types = tuple(cfg_get(cfg, "down_block_types")), tuple(cfg_get(cfg, "up_block_types"))
    for t in down_types:
        if t not in _SVD_DOWN:
            raise NotImplementedError(f"down block type {t} is not supported by the H100 path")
    for t in up_types:
        if t not in _SVD_UP:
            raise NotImplementedError(f"up block type {t} is not supported by the H100 path")
    layers = cfg_get(cfg, "layers_per_block", 2)
    if isinstance(layers, (list, tuple)):
        if len(set(layers)) != 1:
            raise NotImplementedError("per-block layers_per_block")
        layers = layers[0]
    heads = _tuple(cfg_get(cfg, "num_attention_heads"), nb)
    depth = _tuple(cfg_get(cfg, "transformer_layers_per_block", 1), nb)
    ctx = cfg_get(cfg, "cross_attention_dim")
    if isinstance(ctx, (list, tuple)):
        ctx = ctx[0]
    frames = int(cfg_get(cfg, "num_frames", 25))
    if frames > 32:
        raise NotImplementedError("temporal attention kernel handles at most 32 frames")
    for i in range(nb):
        if boc[i] % heads[i] or boc[i] // heads[i] != 64:
            raise NotImplementedError("SVD path needs attention head_dim 64")
    spec = UNetSpec(
        in_channels=cfg_get(cfg, "in_channels", 8), out_channels=cfg_get(cfg, "out_channels", 4),
        block_out_channels=boc, temb_dim=boc[0] * 4, groups=cfg_get(cfg, "norm_num_groups", 32) or 32,
        eps=1e-5, flip_sin_to_cos=True, freq_shift=0.0, cross_attention_dim=ctx,
        addition_embed_type="time_ids",
        addition_time_embed_dim=cfg_get(cfg, "addition_time_embed_dim", 256),
        add_in_dim=cfg_get(cfg, "projection_class_embeddings_input_dim", 768), num_frames=frames)

    def res(p, cin, cout, eps):
        return ResnetSpec(p + ".spatial_res_block", cin, cout, eps, p + ".temporal_res_block",
                          p + ".time_mixer.mix_factor")

    def tf(prefix, dim, i):
        return TransformerSpec(prefix, dim, heads[i], depth[i], ctx, True, temporal=True)

    cout = boc[0]
    for i, t in enumerate(down_types):
        cin, cout = cout, boc[i]
        p = f"down_blocks.{i}"
        attn = t.startswith("CrossAttn")
        eps = 1e-6 if attn else 1e-5
        rs = [res(f"{p}.resnets.{j}", cin if j == 0 else cout, cout, eps) for j in range(layers)]
        att = [tf(f"{p}.attentions.{j}", cout, i) if attn else None for j in range(layers)]
        spec.down.append(BlockSpec(p, rs, att, f"{p}.downsamplers.0.conv" if i != nb - 1 else None, cout))
    c = boc[-1]
    spec.mid = BlockSpec("mid_block", [res("mid_block.resnets.0", c, c, 1e-5), res("mid_block.resnets.1", c, c, 1e-5)],
                         [tf("mid_block.attentions.0", c, nb - 1)], None, c)
    rboc = list(reversed(boc))
    cout = rboc[0]
    for i, t in enumerate(up_types):
        cprev, cout = cout, rboc[i]
        cin = rboc[min(i + 1, nb - 1)]
        p = f"up_blocks.{i}"
        rs = []
        for j in range(layers + 1):
            skip = cin if j == layers else cout
            rin = cprev if j == 0 else cout
            rs.append(res(f"{p}.resnets.{j}", rin + skip, cout, 1e-6))
        att = [tf(f"{p}.attentions.{j}", cout, nb - 1 - i) if t.startswith("CrossAttn") else None
               for j in range(layers + 1)]
        spec.up.append(BlockSpec(p, rs, att, f"{p}.upsamplers.0.conv" if i != nb - 1 else None, cout))
    return spec


def param_shapes(spec: UNetSpec):
    """Ordered {diffusers parameter name: shape} of the architecture."""
    out = {}

    def conv(p, cout, cin, k):
        out[p + ".weight"] = (cout, cin, k, k)
        out[p + ".bias"] = (cout,)

    def lin(p, n, k, bias=True):
        out[p + ".weight"] = (n, k)
        if bias:
            out[p + ".bias"] = (n,)

    def norm(p, c):
        out[p + ".weight"] = (c,)
        out[p + ".bias"] = (c,)

    def resnet(r):
        norm(r.prefix + ".norm1", r.cin)
        conv(r.prefix + ".conv1", r.cout, r.cin, 3)
        lin(r.prefix + ".time_emb_proj", r.cout, spec.temb_dim)
        norm(r.prefix + ".norm2", r.cout)
        conv(r.prefix + ".conv2", r.cout, r.cout, 3)
        if r.has_shortcut:
            conv(r.prefix + ".conv_shortcut", r.cout, r.cin, 1)
        if r.temporal_prefix:
            t = r.temporal_prefix
            norm(t + ".norm1", r.cout)
            out[t + ".conv1.weight"] = (r.cout, r.cout, 3, 1, 1)
            out[t + ".conv1.bias"] = (r.cout,)
            lin(t + ".time_emb_proj", r.cout, spec.temb_dim)
            norm(t + ".norm2", r.cout)
            out[t + ".conv2.weight"] = (r.cout, r.cout, 3, 1, 1)
            out[t + ".conv2.bias"] = (r.cout,)
            out[r.mixer] = (1,)

    def tblock(b, dim, ctx_dim, temporal):
        if temporal:
            norm(b + ".norm_in", dim)
            lin(b + ".ff_in.net.0.proj", dim * 8, dim)
            lin(b + ".ff_in.net.2", dim, dim * 4)
        norm(b + ".norm1", dim)
        for a, kd in (("attn1", dim), ("attn2", ctx_dim)):
            lin(f"{b}.{a}.to_q", dim, dim, False)
            lin(f"{b}.{a}.to_k", dim, kd, False)
            lin(f"{b}.{a}.to_v", dim, kd, False)
            lin(f"{b}.{a}.to_out.0", dim, dim)
            if a == "attn1":
                norm(b + ".norm2", dim)
        norm(b + ".norm3", dim)
        lin(b + ".ff.net.0.proj", dim * 8, dim)
        lin(b + ".ff.net.2", dim, dim * 4)

    def transformer(t):
        if t.temporal:
            norm(t.prefix + ".norm", t.dim)
            lin(t.prefix + ".proj_in", t.dim, t.dim)
            for d in range(t.depth):
                tblock(f"{t.prefix}.transformer_blocks.{d}", t.dim, t.ctx_dim, False)
            for d in range(t.depth):
                tblock(f"{t.prefix}.temporal_transformer_blocks.{d}", t.dim, t.ctx_dim, True)
            lin(t.prefix + ".time_pos_embed.linear_1", t.dim * 4, t.dim)
            lin(t.prefix + ".time_pos_embed.linear_2", t.dim, t.dim * 4)
            out[t.prefix + ".time_mixer.mix_factor"] = (1,)
            lin(t.prefix + ".proj_out", t.dim, t.dim)
            return
        norm(t.prefix + ".norm", t.dim)
        if t.linear_proj:
            lin(t.prefix + ".proj_in", t.dim, t.dim)
        else:
            conv(t.prefix + ".proj_in", t.dim, t.dim, 1)
        for d in range(t.depth):
            b = f"{t.prefix}.transformer_blocks.{d}"
            norm(b + ".norm1", t.dim)
            for a, kd in (("attn1", t.dim), ("attn2", t.ctx_dim)):
                lin(f"{b}.{a}.to_q", t.dim, t.dim, False)
                lin(f"{b}.{a}.to_k", t.dim, kd, False)
                lin(f"{b}.{a}.to_v", t.dim, kd, False)
                lin(f"{b}.{a}.to_out.0", t.dim, t.dim)
                if a == "attn1":
                    norm(b + ".norm2", t.dim)
            norm(b + ".norm3", t.dim)
            lin(b + ".ff.net.0.proj", t.dim * 8, t.dim)
            lin(b + ".ff.net.2", t.dim, t.dim * 4)
        if t.linear_proj:
            lin(t.prefix + ".proj_out", t.dim, t.dim)
        else:
            conv(t.prefix + ".proj_out", t.dim, t.dim, 1)

    conv("conv_in", spec.block_out_channels[0], spec.in_channels, 3)
    lin("time_embedding.linear_1", spec.temb_dim, spec.block_out_channels[0])
    if spec.time_cond_dim:  # diffusers' TimestepEmbedding(cond_proj_dim=...): no bias
        lin("time_embedding.cond_proj", spec.block_out_channels[0], spec.time_cond_dim, False)
    lin("time_embedding.linear_2", spec.temb_dim, spec.temb_dim)
    if spec.addition_embed_type in ("text_time", "time_ids"):
        lin("add_embedding.linear_1", spec.temb_dim, spec.add_in_dim)
        lin("add_embedding.linear_2", spec.temb_dim, spec.temb_dim)
    for blk in spec.down + [spec.mid] + spec.up:
        if blk is spec.mid:
            resnet(blk.resnets[0])
            transformer(blk.attentions[0])
            resnet(blk.resnets[1])
            continue
        for r, t in zip(blk.resnets, blk.attentions):
            resnet(r)
            if t is not None:
                transformer(t)
        if blk.sampler:
            conv(blk.sampler, blk.cout, blk.cout, 3)
    if spec.cond_channels:
        emb, e = spec.cond_embed_channels, "controlnet_cond_embedding"
        conv(e + ".conv_in", emb[0], spec.cond_channels, 3)
        for i in range(len(emb) - 1):
            conv(f"{e}.blocks.{2 * i}", emb[i], emb[i], 3)
            conv(f"{e}.blocks.{2 * i + 1}", emb[i + 1], emb[i], 3)
        conv(e + ".conv_out", spec.block_out_channels[0], emb[-1], 3)
        for i, c in enumerate(spec.residual_channels()):
            conv(f"controlnet_down_blocks.{i}", c, c, 1)
        conv("controlnet_mid_block", spec.mid.cout, spec.mid.cout, 1)
        return out
    for m in spec.motion:
        norm(m.prefix + ".norm", m.dim)
        lin(m.prefix + ".proj_in", m.dim, m.dim)
        for d in range(m.depth):
            b = f"{m.prefix}.transformer_blocks.{d}"
            for a, n in (("attn1", "norm1"), ("attn2", "norm2")):
                norm(f"{b}.{n}", m.dim)
                for x in ("to_q", "to_k", "to_v"):
                    lin(f"{b}.{a}.{x}", m.dim, m.dim, False)
                lin(f"{b}.{a}.to_out.0", m.dim, m.dim)
            norm(b + ".norm3", m.dim)
            lin(b + ".ff.net.0.proj", m.dim * 8, m.dim)
            lin(b + ".ff.net.2", m.dim, m.dim * 4)
            out[b + ".pos_embed.pe"] = (1, m.max_seq_len, m.dim)  # a persistent buffer, not a parameter
        lin(m.prefix + ".proj_out", m.dim, m.dim)
    norm("conv_norm_out", spec.block_out_channels[0])
    conv("conv_out", spec.out_channels, spec.block_out_channels[0], 3)
    if spec.ip is not None:
        # diffusers' names after load_ip_adapter
        ip, pp = spec.ip, "encoder_hid_proj.image_projection_layers.0"
        rs = ip.resampler
        if rs is None:
            lin(pp + ".image_embeds", ip.tokens * ip.ctx_dim, ip.image_embed_dim)
            norm(pp + ".norm", ip.ctx_dim)
        else:
            out[pp + ".latents"] = (1, ip.tokens, rs.dim)
            lin(pp + ".proj_in", rs.dim, ip.image_embed_dim)
            for i in range(rs.depth):
                b = f"{pp}.layers.{i}"
                norm(b + ".ln0", rs.dim)
                norm(b + ".ln1", rs.dim)
                for n in ("to_q", "to_k", "to_v"):
                    lin(f"{b}.attn.{n}", rs.inner, rs.dim, False)
                lin(b + ".attn.to_out.0", rs.dim, rs.inner, False)
                norm(b + ".ff.0", rs.dim)
                lin(b + ".ff.1.net.0.proj", rs.ff_dim, rs.dim, False)
                lin(b + ".ff.1.net.2", rs.dim, rs.ff_dim, False)
            lin(pp + ".proj_out", ip.ctx_dim, rs.dim)
            norm(pp + ".norm_out", ip.ctx_dim)
        dims = dict(spec.cross_attention_layers())
        for prefix in ip.layers:
            lin(prefix + ".processor.to_k_ip.0", dims[prefix].dim, ip.ctx_dim, False)
            lin(prefix + ".processor.to_v_ip.0", dims[prefix].dim, ip.ctx_dim, False)
    return out


def random_state_dict(spec: UNetSpec, seed=0, dtype=torch.float16, device="cpu"):
    """Random weights of the architecture (PyTorch-default-like uniform(-1/sqrt(fan_in), ..);
    norm layers: gamma ~ 1 + 0.3 N(0, 1), beta ~ 0.3 N(0, 1))."""
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    sd = {}
    for name, shape in param_shapes(spec).items():
        is_norm = ".norm" in name or name.startswith("conv_norm_out")
        if name.endswith(".pos_embed.pe"):  # AnimateDiff's sinusoid buffer
            t = motion_pe(shape[1], shape[2])
        elif name.endswith("mix_factor"):
            t = torch.randn(shape, generator=g) * 1.5
        elif name.endswith(".latents"):  # IP-Adapter Plus queries, initialised as diffusers does
            t = torch.randn(shape, generator=g) / math.sqrt(shape[-1])
        elif is_norm:
            # random affine (not PyTorch's 1 / 0): a benchmark must not hide a dropped beta
            t = torch.randn(shape, generator=g) * 0.3 + (1.0 if name.endswith("weight") else 0.0)
        else:
            wshape = shape if name.endswith("weight") else None
            if wshape is None:
                # bias: fan-in of the matching weight
                wshape = param_shapes_cache_fan_in(spec, name)
            fan_in = int(math.prod(wshape[1:])) if len(wshape) > 1 else int(wshape[0])
            bound = 1.0 / math.sqrt(max(fan_in, 1))
            t = (torch.rand(shape, generator=g) * 2 - 1) * bound
        sd[name] = t.to(dtype=dtype, device=device)
    return sd


_FAN_CACHE = {}


def param_shapes_cache_fan_in(spec, bias_name):
    key = id(spec)
    if key not in _FAN_CACHE:
        _FAN_CACHE.clear()
        _FAN_CACHE[key] = param_shapes(spec)
    return _FAN_CACHE[key][bias_name[:-4] + "weight"]
