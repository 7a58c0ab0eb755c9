"""Host-side checks of the native IP-Adapter Plus (the Resampler image projection): the oracle's parameter names
and totals, an independent float64 restatement of the Resampler in the original IP-Adapter form, the spec read
from the module and every refusal by name, host validation of the dry Plus plans, the schedules of plain-adapter
and adapter-free plans pinned to their launch-for-launch fingerprints, and the sensitivity of the UNet output to
the mistakes a Resampler implementation is likely to make."""
import ctypes
import hashlib
import math
import types

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import controlnet_oracle as co
from oracle import ip_adapter_oracle as ipo
from oracle import ip_adapter_plus_oracle as ipp
from oracle import svd_oracle as so
from oracle import unet_oracle as uo
from sfast_b200 import _lib, ops
from sfast_b200.plan import PackedWeights, UNetPlan
from sfast_b200.runtime import CompiledUNet
from sfast_b200.unet_spec import (controlnet_spec_from_config, ip_adapter_geometry, ip_adapter_plus_geometry,
                                  ip_adapter_spec, param_shapes, spec_from_config)
from test_host_logic import _validate_plan_on_cpu

_NO_GPU = pytest.mark.skipif(torch.cuda.is_available(), reason="needs a box without a GPU: launches must fail")
CFGS = {"tiny": uo.tiny_config, "sd15": uo.sd15_config, "sdxl": uo.sdxl_config}
PP = "encoder_hid_proj.image_projection_layers.0"
# (D_img, Dh) of the published adapters (ViT-H/14 image features) and of the tiny test adapter
GEOMETRY = {"tiny": (128, 128), "sd15": (1280, 768), "sdxl": (1280, 1280)}
S_IMG = 257  # ViT-H/14 tokens at 224^2
GPU_TOL = 1e-2  # MODEL_TOL[fp16] of the GPU tests


def _meta_plus(cfg):
    with torch.device("meta"):
        m = uo.UNet2DConditionModel(CFGS[cfg]())
    d_img, dh = GEOMETRY[cfg]
    return ipp.load_ip_adapter_plus(m, d_img, dh)


def _tiny_plus(seed=0):
    return ipp.load_ip_adapter_plus(uo.build_unet(uo.tiny_config(), seed=seed), 128, seed=seed + 1)


# ---------------------------------------------------------------------------------------------------
# the oracle against the published layout
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg,total,resampler", [("sd15", 49_087_488, 29_918_208), ("sdxl", 423_748_864, 82_961_664)])
def test_parameter_totals_are_pinned_and_the_oracle_matches_the_spec(cfg, total, resampler):
    m = _meta_plus(cfg)
    assert ipo.ip_adapter_param_count(m) == total
    assert sum(p.numel() for n, p in m.named_parameters() if n.startswith("encoder_hid_proj.")) == resampler
    spec = spec_from_config(m.config)
    spec.ip = ip_adapter_spec(m, spec)
    d_img, dh = GEOMETRY[cfg]
    rs = spec.ip.resampler
    assert (spec.ip.image_embed_dim, spec.ip.tokens, rs.dim, rs.heads, rs.depth, rs.ff_dim) == \
        (d_img, 16, dh, dh // 64, 4, 4 * dh)
    assert spec.ip == ip_adapter_plus_geometry(spec, d_img, dh)
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert got == {k: tuple(v) for k, v in param_shapes(spec).items()}
    ctx = m.config.cross_attention_dim
    layout = {"latents": (1, 16, dh), "proj_in.weight": (dh, d_img), "proj_in.bias": (dh,),
              "layers.3.ln0.weight": (dh,), "layers.3.ln1.bias": (dh,), "layers.0.attn.to_q.weight": (dh, dh),
              "layers.0.attn.to_k.weight": (dh, dh), "layers.0.attn.to_v.weight": (dh, dh),
              "layers.0.attn.to_out.0.weight": (dh, dh), "layers.2.ff.0.weight": (dh,),
              "layers.2.ff.1.net.0.proj.weight": (4 * dh, dh), "layers.2.ff.1.net.2.weight": (dh, 4 * dh),
              "proj_out.weight": (ctx, dh), "proj_out.bias": (ctx,), "norm_out.weight": (ctx,),
              "norm_out.bias": (ctx,)}
    for k, shape in layout.items():
        assert got[f"{PP}.{k}"] == shape, k
    for n in ("attn.to_q.bias", "attn.to_out.0.bias", "ff.1.net.0.proj.bias", "ff.1.net.2.bias", "layers.4.ln0"):
        assert not any(k.startswith(f"{PP}.") and k.endswith(n) for k in got), n


def resampler_original_form(sd, x, heads, eps=1e-5):
    """The Resampler as the original IP-Adapter code writes it, in float64: PerceiverAttention with one fused
    to_kv projection split into halves, the key sequence cat(x, latents), and q and k each scaled by
    dim_head^-1/4 before the product; FeedForward = LayerNorm, Linear, GELU, Linear.  `sd` holds the
    diffusers-named parameters of one IPAdapterPlusImageProjection."""
    def ln(t, p):
        return F.layer_norm(t, t.shape[-1:], sd[p + ".weight"], sd[p + ".bias"], eps)
    n = x.shape[0]
    lat = sd["latents"].repeat(n, 1, 1)
    x = x @ sd["proj_in.weight"].T + sd["proj_in.bias"]
    depth = 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("layers."))
    for i in range(depth):
        b = f"layers.{i}"
        xn, latn = ln(x, b + ".ln0"), ln(lat, b + ".ln1")
        q = latn @ sd[b + ".attn.to_q.weight"].T
        to_kv = torch.cat([sd[b + ".attn.to_k.weight"], sd[b + ".attn.to_v.weight"]], 0)
        k, v = (torch.cat((xn, latn), dim=-2) @ to_kv.T).chunk(2, dim=-1)

        def heads_(t):
            return t.reshape(n, t.shape[1], heads, -1).transpose(1, 2)
        q, k, v = heads_(q), heads_(k), heads_(v)
        scale = 1 / math.sqrt(math.sqrt(q.shape[-1]))
        w = torch.softmax((q * scale) @ (k * scale).transpose(-2, -1), dim=-1)
        out = (w @ v).transpose(1, 2).reshape(n, lat.shape[1], -1)
        lat = out @ sd[b + ".attn.to_out.0.weight"].T + lat
        h = ln(lat, b + ".ff.0") @ sd[b + ".ff.1.net.0.proj.weight"].T
        lat = F.gelu(h) @ sd[b + ".ff.1.net.2.weight"].T + lat
    return ln(lat @ sd["proj_out.weight"].T + sd["proj_out.bias"], "norm_out")


def test_the_oracle_resampler_matches_the_original_form_in_float64():
    torch.manual_seed(0)
    proj = ipp.IPAdapterPlusImageProjection(96, 128, 192, depth=3, heads=3, num_queries=8).double()
    with torch.no_grad():
        for mod in proj.modules():
            if isinstance(mod, nn.LayerNorm):
                mod.weight.copy_(1 + 0.3 * torch.randn_like(mod.weight))
                mod.bias.copy_(0.3 * torch.randn_like(mod.bias))
        x = torch.randn(3, 37, 96, dtype=torch.float64)
        got = proj(x)
        ref = resampler_original_form({k: v for k, v in proj.state_dict().items()}, x, 3)
    assert got.shape == (3, 8, 128)
    assert torch.allclose(got, ref, rtol=0, atol=1e-12), (got - ref).abs().max()


# ---------------------------------------------------------------------------------------------------
# the spec and the refusals
# ---------------------------------------------------------------------------------------------------
def test_a_plus_adapter_is_read_from_the_module():
    m = _tiny_plus()
    spec = spec_from_config(m.config)
    ip = ip_adapter_spec(m, spec)
    assert ip == ip_adapter_plus_geometry(spec, 128, 128) and len(ip.layers) == 16
    # eps values come from the modules
    proj = m.encoder_hid_proj.image_projection_layers[0]
    proj.layers[1].ln0.eps, proj.layers[2].ff[0].eps, proj.norm_out.eps = 1e-6, 2e-6, 3e-6
    ip = ip_adapter_spec(m, spec)
    assert ip.resampler.block_eps[1][0] == 1e-6 and ip.resampler.block_eps[2][2] == 2e-6 and ip.norm_eps == 3e-6
    # a plain adapter's spec is unchanged
    plain = ipo.load_ip_adapter(uo.build_unet(uo.tiny_config(), seed=0), 64)
    assert ip_adapter_spec(plain, spec) == ip_adapter_geometry(spec, 64)
    assert ip_adapter_geometry(spec, 64).resampler is None


def _renamed(obj, name):
    obj.__class__ = type(name, (type(obj),), {})
    return obj


def _proj(m):
    return m.encoder_hid_proj.image_projection_layers[0]


def _set_ff_act(m, approximate):
    _proj(m).layers[0].ff[1].net[0].approximate = approximate


@pytest.mark.parametrize("mutate,match", [
    (lambda m: setattr(_proj(m).layers[1], "attn", ipp.ResamplerAttention(128, 4, 32)), "dim_head"),
    (lambda m: setattr(_proj(m).layers[0].attn, "processor", type("XFormersAttnProcessor", (), {})()),
     "XFormersAttnProcessor"),
    (lambda m: setattr(_proj(m).layers[2].attn, "to_q", nn.Linear(128, 128)), "with a bias"),
    (lambda m: setattr(_proj(m).layers[3].ff[1].net, "2", nn.Linear(512, 128)), "with a bias"),
    (lambda m: delattr(_proj(m), "layers"), "IPAdapterPlusImageProjection without layers"),
    (lambda m: delattr(_proj(m), "latents"), "IPAdapterPlusImageProjection without latents"),
    (lambda m: setattr(_proj(m).layers[0], "ff", nn.Sequential(nn.LayerNorm(128))), "ff"),
    (lambda m: _set_ff_act(m, "tanh"), "erf GELU"),
    (lambda m: setattr(_proj(m).layers[1].attn, "scale", 1 / math.sqrt(128)), "non-default scale"),
    (lambda m: _renamed(_proj(m), "IPAdapterFaceIDPlusImageProjection"), "FaceID"),
    (lambda m: m.encoder_hid_proj.image_projection_layers.append(_proj(m)), "more than one IP-Adapter"),
    (lambda m: m.mid_block.attentions[0].transformer_blocks[0].attn2.processor.to_v_ip.append(nn.Linear(128, 256)),
     "more than one IP-Adapter"),
])
def test_unsupported_plus_adapters_are_refused_by_name(mutate, match):
    m = _tiny_plus()
    mutate(m)
    with pytest.raises(NotImplementedError, match=match):
        ip_adapter_spec(m, spec_from_config(m.config))
    with pytest.raises(NotImplementedError, match=match):
        CompiledUNet(m.config, m.state_dict, module=m)


def test_a_renamed_image_projection_is_refused_as_plus():
    m = ipo.load_ip_adapter(uo.build_unet(uo.tiny_config(), seed=0), 64)
    _renamed(_proj(m), "IPAdapterPlusImageProjection")
    with pytest.raises(NotImplementedError, match="IPAdapterPlusImageProjection without latents / proj_in / layers"):
        ip_adapter_spec(m, spec_from_config(m.config))


def test_hidden_dims_not_a_multiple_of_64_are_refused():
    m = _tiny_plus()
    m.encoder_hid_proj.image_projection_layers[0] = ipp.IPAdapterPlusImageProjection(128, 128, 96, 1, 64, 1, 16)
    with pytest.raises(NotImplementedError, match="hidden_dims 96"):
        ip_adapter_spec(m, spec_from_config(m.config))


def test_plus_on_the_svd_unet_and_the_controlnet_is_refused():
    m = _tiny_plus()
    with pytest.raises(NotImplementedError, match="SVD UNet"):
        ip_adapter_spec(m, spec_from_config(so.svd_tiny_config()))
    cfg = dict(vars(co.sd15_config()), encoder_hid_dim_type="ip_image_proj")
    with pytest.raises(NotImplementedError, match="encoder_hid_dim_type"):
        controlnet_spec_from_config(cfg)


def test_call_time_refusals_and_shape_checks():
    m = _tiny_plus()
    c = CompiledUNet(m.config, m.state_dict, module=m)
    x, t, e = torch.randn(1, 4, 32, 32).half(), torch.tensor(1), torch.randn(1, 77, 128).half()
    feats = [torch.randn(1, 1, S_IMG, 128).half()]
    with pytest.raises(ValueError, match="image_embeds"):
        c(x, t, e)
    with pytest.raises(NotImplementedError, match="ip_adapter_masks"):
        c(x, t, e, added_cond_kwargs=dict(image_embeds=feats), cross_attention_kwargs=dict(ip_adapter_masks=[None]))
    with pytest.raises(NotImplementedError, match="one adapter"):
        c(x, t, e, added_cond_kwargs=dict(image_embeds=feats * 2))
    for bad in ([torch.randn(1, 1, 128).half()], [torch.randn(1, 1, S_IMG, 64).half()],
                [torch.randn(2, 1, S_IMG, 128).half()], torch.randn(1, 128).half()):
        with pytest.raises(ValueError, match=r"expected \[1, n_images, S_img, 128\]"):
            c(x, t, e, added_cond_kwargs=dict(image_embeds=bad))
    # what the runtime hands to the plan: ip_len = n_img * Q, ip_seq = S_img, [B * n_img * S_img, D_img]
    for emb, n_img in (([torch.randn(1, 3, S_IMG, 128)], 3), (torch.randn(1, S_IMG, 128), 1)):
        ip_len, ip_seq, rows, _ = c._ip_inputs(dict(image_embeds=emb), None, 1)
        assert (ip_len, ip_seq, tuple(rows.shape)) == (16 * n_img, S_IMG, (n_img * S_IMG, 128))
    m.encoder_hid_proj = None  # unload_ip_adapter
    with pytest.raises(NotImplementedError, match="compile"):
        c(x, t, e, added_cond_kwargs=dict(image_embeds=feats))


# ---------------------------------------------------------------------------------------------------
# dry plans
# ---------------------------------------------------------------------------------------------------
def _dry_plus(cfg, b, h, w, n_img, dt=torch.float16, s_img=S_IMG):
    spec = spec_from_config(CFGS[cfg]())
    spec.ip = ip_adapter_plus_geometry(spec, *GEOMETRY[cfg])
    sd = {k: torch.empty(v, dtype=dt, device="meta") for k, v in param_shapes(spec).items()}
    return UNetPlan(PackedWeights(spec, sd, dt, "meta", dry=True), b, h, w, ip_len=16 * n_img, ip_seq=s_img)


def _names(plan):
    return [(op.name, op.fn.name if op.fn is not None else None) for op in plan.all_ops()]


@pytest.mark.parametrize("cfg,h", [("tiny", 32), ("sd15", 64), ("sdxl", 64)])
def test_plus_plans_run_the_resampler_on_the_side_stream(cfg, h):
    base = _dry_plus(cfg, 2, h, h, 1)
    n_cross = len(base.spec.ip.layers)
    side = [(op.name, op.fn.name) for op in base.side_ops if op.name.startswith(PP)]
    # latents broadcast, proj_in, 9 launches per block, proj_out, norm_out
    assert len(side) == 1 + 1 + 9 * 4 + 2
    fns = [f for _, f in side]
    assert fns.count("sfb_attention") == 4 and fns.count("sfb_layer_norm") == 3 * 4 + 1
    assert fns.count("sfb_row_broadcast_add") == 1 and fns.count("sfb_gemm") == 1 + 5 * 4 + 1
    assert sum(n.endswith(".ip_kv") for n, _ in _names(base)) == n_cross
    assert tuple(base.image_embeds_in.shape) == (2 * S_IMG, GEOMETRY[cfg][0])
    for op in base.side_ops:
        if op.fn.name == "sfb_gemm":
            assert op.keep[0].splits == 1, op.name  # the split-K workspace belongs to the main stream
    att = [op for op in base.side_ops if op.name.endswith(".attn.core")]
    assert all((op.keep[0].seq_q, op.keep[0].seq_kv, op.keep[0].head_dim) == (16, 16 + S_IMG, 64) for op in att)
    assert all(abs(op.keep[0].scale - 0.125) < 1e-9 for op in att)
    # the image-feature keys start Q = 16 rows into K and 16 columns into V^T
    img = next(op.keep[0] for op in base.side_ops if op.name.endswith("layers.0.attn.kv_image"))
    lat = next(op.keep[0] for op in base.side_ops if op.name.endswith("layers.0.attn.qkv"))
    assert ((img.k or 0) - (lat.k or 0), (img.vt or 0) - (lat.vt or 0)) == (16 * 64 * 2, 16 * 2)  # dry: offsets
    assert (img.seq, img.k_rows, lat.seq, lat.k_rows, img.which_base, lat.which_base) == \
        (S_IMG, 16 + S_IMG, 16, 16 + S_IMG, 1, 0)
    four = _dry_plus(cfg, 2, h, h, 4)
    assert _names(four) == _names(base) and tuple(four.image_embeds_in.shape) == (8 * S_IMG, GEOMETRY[cfg][0])


@_NO_GPU
@pytest.mark.parametrize("cfg,h,dt", [("tiny", 32, torch.float16), ("sd15", 64, torch.float16),
                                      ("sdxl", 64, torch.bfloat16)])
@pytest.mark.parametrize("n_img", [1, 4])
def test_dry_plus_plans_pass_host_validation(cfg, h, dt, n_img):
    plan = _dry_plus(cfg, 2, h, h, n_img, dt)
    n = _validate_plan_on_cpu(plan)
    assert n["sfb_gemm"] > 0 and n["sfb_attention"] > 0 and n["sfb_row_broadcast_add"] == 1


def test_too_many_images_are_refused():
    with pytest.raises(NotImplementedError, match="one KV tile"):
        _dry_plus("sd15", 1, 64, 64, 5)
    with pytest.raises(ValueError, match="ip_seq"):
        _dry_plus("tiny", 1, 32, 32, 1, s_img=0)


def plan_fingerprint(plan):
    """sha1 over every launch of a dry plan in schedule order: op name, entry point, the bytes of its parameter
    struct (dry pointers are buffer offsets, dry tensor maps are 0) or its plain arguments, and the geometry of
    every tensor map."""
    h = hashlib.sha1()
    for op in plan.all_ops():
        if op.fn is None:
            continue
        p = op.keep[0] if op.keep else None
        if isinstance(p, ctypes.Structure):
            body = ctypes.string_at(ctypes.addressof(p), ctypes.sizeof(p)).hex()
        else:
            body = repr(tuple(a if isinstance(a, (int, float)) or a is None else type(a).__name__ for a in op.args))
        maps = tuple(m.geom for m in op.keep if isinstance(m, ops.DryMap))
        h.update(repr((op.name, op.fn.name, body, maps)).encode())
    return h.hexdigest()


def _dry_plain(cfg, b, h, w, ip_len, d_img, dt=torch.float16):
    spec = spec_from_config(CFGS[cfg]())
    if ip_len:
        spec.ip = ip_adapter_geometry(spec, d_img)
    sd = {k: torch.empty(v, dtype=dt, device="meta") for k, v in param_shapes(spec).items()}
    return UNetPlan(PackedWeights(spec, sd, dt, "meta", dry=True), b, h, w, ip_len=ip_len)


# fingerprints of the schedules the commit before IP-Adapter Plus built (same function, same arguments)
PARENT_FINGERPRINTS = {
    ("tiny", 2, 32, 32, 4, 64): "816f5cd8e75a500be2e6a123d08d0e49e2691215",
    ("sd15", 2, 64, 64, 16, 1024): "96554e2d81629501738c271424178ce094d78f1b",
    ("sdxl", 1, 64, 64, 8, 1280): "7423ba621697257df291e3895da51caa1c8841d0",
    ("sd15", 2, 64, 64, 0, 0): "62ada28a6a0c1c9bf8c859462c07d236857a8a49",
    ("sdxl", 2, 128, 128, 0, 0): "b2c1bc4d1c5d2fa90012576eca9a12867fad1f37",
}


@pytest.mark.parametrize("key", list(PARENT_FINGERPRINTS))
def test_plain_and_adapter_free_schedules_are_unchanged(key, monkeypatch):
    monkeypatch.setattr(ops, "num_sms", lambda: 132)  # the split-K choices of an H100 SXM
    assert plan_fingerprint(_dry_plain(*key)) == PARENT_FINGERPRINTS[key]


# ---------------------------------------------------------------------------------------------------
# sensitivity: the mistakes the GPU tolerance must be able to see
# ---------------------------------------------------------------------------------------------------
def _rel(got, ref):
    got, ref = got.float(), ref.float()
    d = (got - ref).abs()
    rms = ref.pow(2).mean().sqrt()
    return max((d.max() / ref.abs().max()).item(), (d / (ref.abs() + rms)).max().item())


def _no_latent_keys(self, x, latents, residual):
    latents = self.attn(self.ln1(latents), self.ln0(x)) + residual
    return self.ff(latents) + latents


def _ln_swapped(self, x, latents, residual):
    ehs = self.ln1(x)
    latents = self.ln0(latents)
    latents = self.attn(latents, torch.cat([ehs, latents], dim=-2)) + residual
    return self.ff(latents) + latents


def _scale_of_hidden_dims(self, x, latents, residual):
    self.attn.scale = 1 / math.sqrt(self.attn.to_q.in_features)
    try:
        return ipp.IPAdapterPlusImageProjectionBlock.forward(self, x, latents, residual)
    finally:
        self.attn.scale = 1 / 8


@pytest.mark.parametrize("mistake", [_no_latent_keys, _ln_swapped, _scale_of_hidden_dims])
def test_resampler_mistakes_move_the_unet_output_past_ten_times_the_gpu_tolerance(mistake):
    # the tiny UNet and adapter of the GPU parity test (weights seed 3, adapter seed 4, gain 4)
    m = ipp.load_ip_adapter_plus(uo.build_unet(uo.tiny_config(), seed=3), 128, seed=4, gain=4.0)
    g = torch.Generator().manual_seed(0)
    sample, ehs = torch.randn(2, 4, 32, 32, generator=g), torch.randn(2, 77, 128, generator=g)
    kw = dict(image_embeds=[torch.randn(2, 1, S_IMG, 128, generator=g)])
    with torch.no_grad():
        ref = m(sample, torch.tensor(437), ehs, added_cond_kwargs=kw).sample
        for blk in _proj(m).layers:
            blk.forward = types.MethodType(mistake, blk)
        bad = m(sample, torch.tensor(437), ehs, added_cond_kwargs=kw).sample
    err = _rel(bad, ref)
    print(f"{mistake.__name__}: {err:.3f}")
    assert err > 10 * GPU_TOL, err
