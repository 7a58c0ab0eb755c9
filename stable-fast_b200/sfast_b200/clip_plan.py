"""Launch schedule of the CLIP text encoders (transformers ``CLIPTextModel`` /
``CLIPTextModelWithProjection``), the modules the reference traces and graphs around the UNet
(/root/reference/src/sfast/compilers/diffusion_pipeline_compiler.py:93-112: ``text_encoder`` of SD-1.5,
``text_encoder`` + ``text_encoder_2`` of SDXL).

Same kernel families as the UNet's transformer blocks, on 77-token rows:

  ids -> token + position embedding (one gather kernel, which also writes the row statistics of the
         first LayerNorm)
  per layer:  LayerNorm1 folded into the fused QKV projection (tcgen05 GEMM, QKV-scatter epilogue)
              -> causal flash attention (64-key tiles) -> out_proj + residual (+ row statistics)
              -> LayerNorm2 folded into fc1 + quick_gelu / gelu (GEMM epilogue activation)
              -> fc2 + residual (+ row statistics)
  final LayerNorm (stand-alone kernel), end-of-text pooling (gather kernel), text projection.

Every layer's output lives in its own buffer: ``output_hidden_states=True`` (SDXL reads the penultimate
layer, clip_skip reads others) returns views of them at no extra cost.
"""
from dataclasses import dataclass

import torch

from . import _lib, ops
from .ops import Act, EPI_QKV, Op, _ptr
from .plan import Plan, _round_up
from .unet_spec import cfg_get

_ACTS = {"quick_gelu": _lib.ACT_QUICK_GELU, "gelu": _lib.ACT_GELU}


@dataclass
class ClipTextSpec:
    vocab_size: int
    hidden: int
    intermediate: int
    layers: int
    heads: int
    max_positions: int
    act: str
    eps: float
    eos_token_id: int
    projection_dim: int = 0  # > 0: CLIPTextModelWithProjection (text_projection, no bias)

    @property
    def temporal(self):
        return False

    @property
    def head_dim(self):
        return self.hidden // self.heads

    def all_resnets(self):
        return []


def clip_text_spec_from_config(cfg, with_projection=False) -> ClipTextSpec:
    act = cfg_get(cfg, "hidden_act", "quick_gelu")
    if act not in _ACTS:
        raise NotImplementedError(f"CLIP text encoder hidden_act={act!r} is not supported by the H100 path")
    hidden, heads = cfg_get(cfg, "hidden_size"), cfg_get(cfg, "num_attention_heads")
    if hidden % heads or hidden // heads not in (32, 64):
        raise NotImplementedError(f"CLIP text encoder head_dim {hidden / heads} (causal attention kernel: 32 / 64)")
    if hidden % 64 or cfg_get(cfg, "intermediate_size") % 64:
        raise NotImplementedError("CLIP text encoder widths must be multiples of 64")
    return ClipTextSpec(vocab_size=cfg_get(cfg, "vocab_size"), hidden=hidden,
                        intermediate=cfg_get(cfg, "intermediate_size"), layers=cfg_get(cfg, "num_hidden_layers"),
                        heads=heads, max_positions=cfg_get(cfg, "max_position_embeddings", 77), act=act,
                        eps=float(cfg_get(cfg, "layer_norm_eps", 1e-5)), eos_token_id=cfg_get(cfg, "eos_token_id", 2),
                        projection_dim=cfg_get(cfg, "projection_dim", 0) if with_projection else 0)


def clip_text_param_shapes(spec: ClipTextSpec):
    """{transformers parameter name: shape} of CLIPTextModel(WithProjection)."""
    out, c, i = {}, spec.hidden, spec.intermediate
    out["text_model.embeddings.token_embedding.weight"] = (spec.vocab_size, c)
    out["text_model.embeddings.position_embedding.weight"] = (spec.max_positions, c)
    for l in range(spec.layers):
        p = f"text_model.encoder.layers.{l}"
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            out[f"{p}.self_attn.{n}.weight"], out[f"{p}.self_attn.{n}.bias"] = (c, c), (c,)
        for n in ("layer_norm1", "layer_norm2"):
            out[f"{p}.{n}.weight"], out[f"{p}.{n}.bias"] = (c,), (c,)
        out[f"{p}.mlp.fc1.weight"], out[f"{p}.mlp.fc1.bias"] = (i, c), (i,)
        out[f"{p}.mlp.fc2.weight"], out[f"{p}.mlp.fc2.bias"] = (c, i), (c,)
    out["text_model.final_layer_norm.weight"] = out["text_model.final_layer_norm.bias"] = (c,)
    if spec.projection_dim:
        out["text_projection.weight"] = (spec.projection_dim, c)
    return out


def random_clip_state_dict(spec: ClipTextSpec, dtype, device, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    sd = {}
    for name, shape in clip_text_param_shapes(spec).items():
        if "layer_norm" in name:
            v = (1.0 + 0.2 * torch.randn(shape, generator=g)) if name.endswith(".weight") else 0.2 * torch.randn(shape, generator=g)
        elif name.endswith(".bias"):
            v = 0.05 * torch.randn(shape, generator=g)
        elif "embedding" in name:
            v = 0.05 * torch.randn(shape, generator=g)
        else:
            v = torch.randn(shape, generator=g) / (shape[-1] ** 0.5)
        sd[name] = v.to(device=device, dtype=dtype)
    return sd


class _ClipPlan(Plan):
    """What the text and vision towers share: [B, S] token rows, the encoder layers, and every layer's output
    in its own buffer (hidden_states())."""

    def __init__(self, weights, batch, seq, ln_floats):
        super().__init__(weights, batch, 1, seq, ln_floats=ln_floats)
        self.S = seq
        self.hidden = []       # [layers + 1] activations: embedding output, then every layer's output
        self.last_hidden_state = None
        self.pooled = None

    def encoder(self, prefix, hs: Act, st, **attn):
        """The encoder layers of `prefix` ("text_model" / "vision_model") on hs; returns the last layer's output.
        Per layer: LayerNorm1 folded into the fused QKV projection -> attention (`attn`: attention_op options)
        -> out_proj + residual -> LayerNorm2 folded into fc1 + activation -> fc2 + residual.  `st`: hs's row
        statistics; None where no GEMM epilogue produced them (the vision tower's pre-LayerNorm output), and
        then layer 0's LayerNorm1 is the stand-alone kernel."""
        spec, B, S = self.spec, self.B, self.S
        C, I, rows = spec.hidden, spec.intermediate, B * S
        qkv = self.attention_operands(B, spec.heads, S, S, spec.head_dim)
        qkv_epi = dict(qkv, which_base=0, seq=S)
        for l in range(spec.layers):
            p = f"{prefix}.encoder.layers.{l}"
            a = p + ".self_attn"
            wn = [f"{a}.{n}_proj.weight" for n in "qkv"]
            bn = [f"{a}.{n}_proj.bias" for n in "qkv"]
            if st is None:
                x1 = self.layer_norm(p + ".layer_norm1", hs, p + ".layer_norm1", spec.eps)
                wm = self.w.cat_matrix(wn)
                self._emit(self._gemm(a + ".qkv", a=self._a_matrix(x1), b=wm, M=rows, N=wm.n, K=C, dt=self.dt,
                                      epi=EPI_QKV, bias=self.w.f32_cat(bn), qkv=qkv_epi, splits=1, keep=(x1.buf, wm)))
            else:
                wm, bias, colsum = self.w.ln_matrix(wn, p + ".layer_norm1", bias_names=bn)
                self._emit(self._gemm(a + ".qkv", a=self._a_matrix(hs), b=wm, M=rows, N=wm.n, K=C, dt=self.dt,
                                      epi=EPI_QKV, bias=bias, qkv=qkv_epi, splits=1,
                                      ln=dict(rowstats=st, colsum=colsum, eps=spec.eps, dim=C),
                                      keep=(hs.buf, wm, colsum)))
            ao = self.act("clip_attn_out", B, 1, S, C)
            self.attention_core(a + ".core", qkv, ao, **attn)
            mid = self.act("clip_mid", B, 1, S, C)
            st2 = self.ln_slot(rows, C)
            self.linear(a + ".out_proj", ao, self.w.matrix(f"{a}.out_proj.weight"), self.w.f32(f"{a}.out_proj.bias"),
                        mid, residual=hs, rowstats_out=st2, splits=1)
            w1, b1, cs1 = self.w.ln_matrix([p + ".mlp.fc1.weight"], p + ".layer_norm2",
                                           bias_names=[p + ".mlp.fc1.bias"])
            ff = self.act("clip_ff", B, 1, S, I)
            self._emit(self._gemm(p + ".mlp.fc1", a=self._a_matrix(mid), b=w1, M=rows, N=I, K=C, dt=self.dt,
                                  out=ff.ptr, ldo=ff.ld, bias=b1, splits=1, act=_ACTS[spec.act],
                                  ln=dict(rowstats=st2, colsum=cs1, eps=spec.eps, dim=C),
                                  keep=(mid.buf, ff.buf, w1, cs1)))
            nxt = self.act(f"clip_h{l + 1}", B, 1, S, C)
            st = self.ln_slot(rows, C) if l + 1 < spec.layers else None
            self.linear(p + ".mlp.fc2", ff, self.w.matrix(p + ".mlp.fc2.weight"), self.w.f32(p + ".mlp.fc2.bias"),
                        nxt, residual=mid, rowstats_out=st, splits=1)
            hs = nxt
            self.hidden.append(hs)
        return hs

    def hidden_states(self):
        """Tuple of [B, S, C] views: embedding output, then each encoder layer's output."""
        return tuple(h.buf.view(self.B, self.S, self.spec.hidden) for h in self.hidden)


class ClipTextPlan(_ClipPlan):
    """Static launch schedule of one text-encoder forward for a fixed (batch, sequence length)."""

    def __init__(self, weights, batch, seq):
        spec = weights.spec
        if seq > spec.max_positions:
            raise ValueError(f"sequence length {seq} exceeds max_position_embeddings {spec.max_positions}")
        # row statistics of every folded LayerNorm: 2 per layer + the embedding's
        super().__init__(weights, batch, seq,
                         (2 * spec.layers + 1) * batch * seq * 2 * ops.rowstats_slots(spec.hidden))
        self.ids_in = self._alloc((batch, seq), torch.int64)
        self.text_embeds = None
        self._build()

    def _build(self):
        spec, B, S, lib = self.spec, self.B, self.S, self.lib_or_dry()
        C, rows = spec.hidden, B * S
        hs = self.act("clip_h0", B, 1, S, C)
        st = self.ln_slot(rows, C)
        tok = self.w.small("text_model.embeddings.token_embedding.weight")
        pos = self.w.small("text_model.embeddings.position_embedding.weight")
        self._emit(Op("embeddings", lib.sfb_embed_tokens,
                      (_ptr(self.ids_in), _ptr(tok), _ptr(pos), hs.ptr, _ptr(st), st.slots, B, S, C, spec.vocab_size, hs.ld,
                       ops.dtype_code(self.dt)), (self.ids_in, tok, pos, hs.buf, st), 0, 4 * rows * C))
        self.hidden.append(hs)
        hs = self.encoder("text_model", hs, st, kv_tile=64, causal=True)
        out = self.layer_norm("final_layer_norm", hs, "text_model.final_layer_norm", spec.eps)
        self.last_hidden_state = out.buf.view(B, S, C) if not self.dry else out.buf
        self.pooled = self.buf("clip_pooled", (B, C))
        self._emit(Op("pool(eos)", lib.sfb_clip_pool,
                      (_ptr(self.ids_in), out.ptr, _ptr(self.pooled), B, S, C, out.ld, spec.eos_token_id),
                      (self.ids_in, out.buf, self.pooled)))
        if spec.projection_dim:
            self.text_embeds = self.buf("clip_text_embeds", (B, spec.projection_dim))
            self._emit(ops.small_linear_op("text_projection", lib, x=self.pooled,
                                           w=self.w.small("text_projection.weight"), bias=None, batch=B,
                                           n=spec.projection_dim, k=C, dt=self.dt, y16=self.text_embeds))
        self._finish()


# =================================================================================================
# CLIP vision tower (transformers CLIPVisionModel / CLIPVisionModelWithProjection): the SVD pipeline's
# image_encoder (reference :100-103).  Same encoder layers without the causal mask; the patch embedding is
# a patchify gather + one GEMM per image whose epilogue adds the position embedding.
# =================================================================================================
@dataclass
class ClipVisionSpec:
    hidden: int
    intermediate: int
    layers: int
    heads: int
    image_size: int
    patch_size: int
    channels: int
    act: str
    eps: float
    projection_dim: int = 0  # > 0: CLIPVisionModelWithProjection (visual_projection, no bias)

    @property
    def temporal(self):
        return False

    @property
    def head_dim(self):
        return self.hidden // self.heads

    @property
    def grid(self):
        return self.image_size // self.patch_size

    @property
    def tokens(self):
        return self.grid * self.grid + 1

    def all_resnets(self):
        return []


def clip_vision_spec_from_config(cfg, with_projection=False) -> ClipVisionSpec:
    act = cfg_get(cfg, "hidden_act", "quick_gelu")
    if act not in _ACTS:
        raise NotImplementedError(f"CLIP vision encoder hidden_act={act!r} is not supported by the H100 path")
    hidden, heads = cfg_get(cfg, "hidden_size"), cfg_get(cfg, "num_attention_heads")
    if hidden % heads or hidden // heads not in (32, 40, 64, 80, 128, 160):
        raise NotImplementedError(f"CLIP vision encoder head_dim {hidden / heads} has no attention kernel")
    if hidden % 64 or cfg_get(cfg, "intermediate_size") % 64:
        raise NotImplementedError("CLIP vision encoder widths must be multiples of 64")
    size, patch = cfg_get(cfg, "image_size", 224), cfg_get(cfg, "patch_size", 14)
    if size % patch:
        raise NotImplementedError("CLIP vision encoder: image_size must be a multiple of patch_size")
    return ClipVisionSpec(hidden=hidden, intermediate=cfg_get(cfg, "intermediate_size"),
                          layers=cfg_get(cfg, "num_hidden_layers"), heads=heads, image_size=size, patch_size=patch,
                          channels=cfg_get(cfg, "num_channels", 3), act=act,
                          eps=float(cfg_get(cfg, "layer_norm_eps", 1e-5)),
                          projection_dim=cfg_get(cfg, "projection_dim", 0) if with_projection else 0)


def clip_vision_param_shapes(spec: ClipVisionSpec):
    out, c, i = {}, spec.hidden, spec.intermediate
    e = "vision_model.embeddings"
    out[e + ".class_embedding"] = (c,)
    out[e + ".patch_embedding.weight"] = (c, spec.channels, spec.patch_size, spec.patch_size)
    out[e + ".position_embedding.weight"] = (spec.tokens, c)
    out["vision_model.pre_layrnorm.weight"] = out["vision_model.pre_layrnorm.bias"] = (c,)
    for l in range(spec.layers):
        p = f"vision_model.encoder.layers.{l}"
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            out[f"{p}.self_attn.{n}.weight"], out[f"{p}.self_attn.{n}.bias"] = (c, c), (c,)
        for n in ("layer_norm1", "layer_norm2"):
            out[f"{p}.{n}.weight"], out[f"{p}.{n}.bias"] = (c,), (c,)
        out[f"{p}.mlp.fc1.weight"], out[f"{p}.mlp.fc1.bias"] = (i, c), (i,)
        out[f"{p}.mlp.fc2.weight"], out[f"{p}.mlp.fc2.bias"] = (c, i), (c,)
    out["vision_model.post_layernorm.weight"] = out["vision_model.post_layernorm.bias"] = (c,)
    if spec.projection_dim:
        out["visual_projection.weight"] = (spec.projection_dim, c)
    return out


class ClipVisionPlan(_ClipPlan):
    """Static launch schedule of one vision-tower forward for a fixed batch of image_size^2 images."""

    def __init__(self, weights, batch):
        spec = weights.spec
        super().__init__(weights, batch, spec.tokens,
                         2 * spec.layers * batch * spec.tokens * 2 * ops.rowstats_slots(spec.hidden))
        self.pixels_in = self._alloc((batch, spec.channels, spec.image_size, spec.image_size), self.dt)
        self.image_embeds = None
        self._build()

    def _build(self):
        spec, B, S, lib = self.spec, self.B, self.S, self.lib_or_dry()
        C, rows, np_ = spec.hidden, B * S, spec.grid * spec.grid
        es = 2
        # ---- embeddings: patchify -> GEMM (+ position embedding as the residual) per image; class rows copied
        kreal = spec.channels * spec.patch_size ** 2
        kpad = _round_up(kreal, 64)
        patches = self.buf("clipv_patches", (B * np_, kpad))
        self._emit(Op("patchify", lib.sfb_patchify,
                      (_ptr(self.pixels_in), _ptr(patches), B, spec.channels, spec.image_size, spec.image_size,
                       spec.patch_size, kpad), (self.pixels_in, patches), 0, 4 * B * np_ * kpad))
        emb = self.act("clipv_emb", B, 1, S, C)
        e = "vision_model.embeddings"
        wm = self.w.patch_matrix(e + ".patch_embedding.weight", kpad)
        pos = self.w.rows_from_1(e + ".position_embedding.weight")
        cls = self.w.class_row(e + ".class_embedding", e + ".position_embedding.weight")
        for b in range(B):
            dst = emb.ptr + (b * S + 1) * C * es
            self._emit(self._gemm(f"patch_embedding[{b}]", a=ops.a_matrix(_ptr(patches) + b * np_ * kpad * es, np_, kpad, kpad),
                                  b=wm, M=np_, N=C, K=kpad, dt=self.dt, out=dst, ldo=C, residual=_ptr(pos), ldr=C,
                                  splits=1, keep=(patches, emb.buf, wm, pos)))
            self._emit(Op(f"class_embedding[{b}]", lib.sfb_copy2d, (_ptr(cls), emb.ptr + b * S * C * es, 1, C, C, C),
                          (cls, emb.buf)))
        hs = self.act("clip_h0", B, 1, S, C)
        self._emit(ops.ln_op("pre_layrnorm", lib, x=emb.buf, y=hs.buf, rows=rows, c=C,
                             gamma=self.w.f32("vision_model.pre_layrnorm.weight"),
                             beta=self.w.f32("vision_model.pre_layrnorm.bias"), eps=spec.eps, dt=self.dt))
        self.hidden.append(hs)
        hs = self.encoder("vision_model", hs, None)
        self.last_hidden_state = hs.buf.view(B, S, C) if not self.dry else hs.buf
        # pooled = post_layernorm(class-token rows); image_embeds = visual_projection(pooled)
        cls_rows = self.buf("clipv_cls", (B, C))
        self._emit(Op("gather(class rows)", lib.sfb_copy2d, (hs.ptr, _ptr(cls_rows), B, C, S * C, C),
                      (hs.buf, cls_rows)))
        self.pooled = self.buf("clipv_pooled", (B, C))
        self._emit(ops.ln_op("post_layernorm", lib, x=cls_rows, y=self.pooled, rows=B, c=C,
                             gamma=self.w.f32("vision_model.post_layernorm.weight"),
                             beta=self.w.f32("vision_model.post_layernorm.bias"), eps=spec.eps, dt=self.dt))
        if spec.projection_dim:
            self.image_embeds = self.buf("clipv_image_embeds", (B, spec.projection_dim))
            self._emit(ops.small_linear_op("visual_projection", lib, x=self.pooled,
                                           w=self.w.small("visual_projection.weight"), bias=None, batch=B,
                                           n=spec.projection_dim, k=C, dt=self.dt, y16=self.image_embeds))
        self._finish()
