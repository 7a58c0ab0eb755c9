"""IP-Adapter Plus on the GPU: every distinct launch of the Plus plans replayed against float64, the Resampler's
output alone and whole-UNet parity with the oracle adapter (oracle/ip_adapter_plus_oracle.py), and
the behaviour of the compiled UNet (one graph for every scale, bitwise replays, in-place weight updates,
refusals, compile() with a CLIP vision encoder)."""
import dataclasses
import types

import pytest
import torch

import plan_launches as pl
from oracle import ip_adapter_oracle as ipo
from oracle import ip_adapter_plus_oracle as ipp
from oracle import unet_oracle as uo
from sfast_b200 import _lib
from sfast_b200.plan import PackedWeights, UNetPlan
from sfast_b200.unet_spec import ip_adapter_plus_geometry, param_shapes, spec_from_config
from test_ip_adapter_gpu import MODEL_TOL, _f32, _ip_key, _rel, _replay_attention_ip

pytestmark = pytest.mark.gpu

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

DEV = "cuda"
PP = "encoder_hid_proj.image_projection_layers.0"
S_IMG = 257  # ViT-H/14 at 224^2
# published geometries: (UNet config, D_img, Dh)
SD15_PLUS = (uo.sd15_config, 1280, 768)
SDXL_PLUS = (uo.sdxl_config, 1280, 1280)


# ---------------------------------------------------------------------------------------------------
# every distinct launch of the Plus plans
# ---------------------------------------------------------------------------------------------------
def _dry_plus_plan(cfg_name, b, h, w, dt, d_img, dh, n_img):
    spec = spec_from_config(getattr(uo, cfg_name)())
    spec.ip = ip_adapter_plus_geometry(spec, d_img, dh)
    sd = {k: torch.empty(v, dtype=dt, device="meta") for k, v in param_shapes(spec).items()}
    with pl.recording_map_offsets():
        return UNetPlan(PackedWeights(spec, sd, dt, "meta", dry=True), b, h, w, ip_len=16 * n_img, ip_seq=S_IMG)


PLUS_PLANS = [
    ("tiny_plus1_2x32x32", lambda: _dry_plus_plan("tiny_config", 2, 32, 32, torch.float16, 128, 128, 1)),
    ("tiny_plus4_1x32x32", lambda: _dry_plus_plan("tiny_config", 1, 32, 32, torch.float16, 128, 128, 4)),
    ("sd15_plus1_2x64x64", lambda: _dry_plus_plan("sd15_config", 2, 64, 64, torch.float16, 1280, 768, 1)),
    ("sd15_plus4_1x64x64", lambda: _dry_plus_plan("sd15_config", 1, 64, 64, torch.float16, 1280, 768, 4)),
    ("sdxl_bf16_plus1_2x128x128", lambda: _dry_plus_plan("sdxl_config", 2, 128, 128, torch.bfloat16, 1280, 1280, 1)),
]


def test_every_ip_adapter_plus_plan_launch_matches_float64():
    entries = {}
    for pname, build in PLUS_PLANS:
        plan = build()
        for op in plan.all_ops():
            if op.fn is None or op.fn.name in pl.SKIP:
                continue
            if op.fn.name == "sfb_attention_ip":
                entries.setdefault(_ip_key(op), (pname, op))
            elif ".ip_kv" in op.name or op.name.startswith("encoder_hid_proj"):
                entries.setdefault(pl.launch_key(op), (pname, op))
    names = {op.fn.name for _, op in entries.values()}
    assert {"sfb_attention_ip", "sfb_gemm", "sfb_attention", "sfb_layer_norm", "sfb_row_broadcast_add"} <= names, names
    failures = []
    for key, (pname, op) in entries.items():
        torch.manual_seed(int(pl.key_id(key), 16) % (1 << 31))
        if op.fn.name == "sfb_attention_ip":
            ok, err = _replay_attention_ip(op)
        else:
            recs = list(pl.run_keys({key: dict(op=op, plans=[pname], family="unet", name=op.fn.name)}, [key]))
            ok, err = all(r["ok"] for r in recs), max(r["err"] for r in recs)
        torch.cuda.empty_cache()
        if not ok:
            failures.append(f"{pname}: {op.name}: err {err}")
    print(f"{len(entries)} distinct IP-Adapter Plus plan launches replayed")
    assert not failures, "\n".join(failures)


# ---------------------------------------------------------------------------------------------------
# whole model
# ---------------------------------------------------------------------------------------------------
def _plus_pair(cfg, seed, dt, d_img, dh=None, graph=True, gain=4.0):
    """(compiled fast UNet with a random Plus adapter, fp32 oracle with the same weights)."""
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_unet
    fast = ipp.load_ip_adapter_plus(uo.build_unet(cfg, seed=seed, dtype=dt, device=DEV), d_img, dh, seed=seed + 1,
                                    gain=gain)
    oracle = ipp.load_ip_adapter_plus(uo.build_unet(cfg, seed=seed, dtype=torch.float32, device=DEV), d_img, dh,
                                      seed=seed + 1, gain=gain)
    oracle.load_state_dict({k: v.float() for k, v in fast.state_dict().items()})
    cc = CompilationConfig.Default()
    cc.enable_cuda_graph = graph
    return compile_unet(fast, cc), oracle


def _inputs(cfg, b, h, w, dt, d_img, n_img=1, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    sample = torch.randn(b, 4, h, w, device=DEV, generator=g).to(dt)
    ehs = torch.randn(b, 77, cfg.cross_attention_dim, device=DEV, generator=g).to(dt)
    feats = torch.randn(b, n_img, S_IMG, d_img, device=DEV, generator=g).to(dt)
    kw = dict(image_embeds=[feats])
    if cfg.addition_embed_type == "text_time":
        kw.update(text_embeds=torch.randn(b, 1280, device=DEV, generator=g).to(dt),
                  time_ids=torch.tensor([[h * 8, w * 8, 0, 0, h * 8, w * 8]] * b, device=DEV, dtype=torch.float32))
    return sample, torch.tensor(437, device=DEV), ehs, kw


def _check(fast, oracle, sample, t, ehs, kw, dt, tol=None):
    got = fast(sample, t, ehs, added_cond_kwargs=kw).sample
    with torch.no_grad():
        ref = oracle(sample.float(), t, ehs.float(), added_cond_kwargs=_f32(kw)).sample
    err = _rel(got, ref)
    assert err <= (tol or MODEL_TOL[dt]), err
    return got, err


def _plan(fast):
    (gp,) = fast.forward._cached.values()
    return gp.plan


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("geom", [SD15_PLUS, SDXL_PLUS], ids=["sd15_plus", "sdxl_plus_vit_h"])
def test_resampler_output_matches_the_oracle(geom, dt):
    """The Resampler alone at a published geometry (D_img, Dh, 16 queries, ctx), on a tiny UNet with that
    cross_attention_dim: the image tokens the plan hands to the cross-attentions vs the fp32 oracle projection."""
    cfg_f, d_img, dh = geom
    cfg = dataclasses.replace(uo.tiny_config(), cross_attention_dim=cfg_f().cross_attention_dim)
    fast, oracle = _plus_pair(cfg, 5, dt, d_img, dh)
    sample, t, ehs, kw = _inputs(cfg, 2, 32, 32, dt, d_img, n_img=2)
    fast(sample, t, ehs, added_cond_kwargs=kw)
    got = _plan(fast)._ip_tokens.view(2 * 2, 16, -1)
    with torch.no_grad():
        ref = oracle.encoder_hid_proj.image_projection_layers[0](kw["image_embeds"][0].float().flatten(0, 1))
    err = _rel(got, ref)
    print(f"Resampler D_img {d_img} Dh {dh} ctx {cfg.cross_attention_dim} {dt}: {err:.2e}")
    assert err <= MODEL_TOL[dt], err


@pytest.mark.parametrize("graph", [True, False])
def test_tiny_unet_with_ip_adapter_plus_matches_the_oracle(graph):
    cfg = uo.tiny_config()
    fast, oracle = _plus_pair(cfg, 3, torch.float16, 128, graph=graph)
    for b in (1, 2):
        for n_img in (1, 4):
            _, err = _check(fast, oracle, *_inputs(cfg, b, 32, 32, torch.float16, 128, n_img), torch.float16)
            print(f"tiny Plus B={b} n_img={n_img} graph={graph}: {err:.2e}")
    # the deprecated bare [B, S_img, D_img] form
    s, t, e, kw = _inputs(cfg, 2, 32, 32, torch.float16, 128)
    kw["image_embeds"] = kw["image_embeds"][0][:, 0]
    _check(fast, oracle, s, t, e, kw, torch.float16)
    # five images are more than one KV tile of image tokens
    s, t, e, kw = _inputs(cfg, 1, 32, 32, torch.float16, 128, 5)
    with pytest.raises(NotImplementedError, match="one KV tile"):
        fast(s, t, e, added_cond_kwargs=kw)


def test_sd15_unet_with_ip_adapter_plus_matches_the_oracle():
    cfg_f, d_img, dh = SD15_PLUS
    cfg = cfg_f()
    fast, oracle = _plus_pair(cfg, 1, torch.float16, d_img, dh)
    _, err = _check(fast, oracle, *_inputs(cfg, 2, 64, 64, torch.float16, d_img), torch.float16)
    print(f"SD-1.5 + ip-adapter-plus_sd15 shape, 64x64, B=2: {err:.2e}")


def test_sdxl_unet_with_ip_adapter_plus_vit_h_matches_the_oracle_bf16():
    cfg_f, d_img, dh = SDXL_PLUS
    cfg = cfg_f()
    fast, oracle = _plus_pair(cfg, 2, torch.bfloat16, d_img, dh)
    _, err = _check(fast, oracle, *_inputs(cfg, 2, 64, 64, torch.bfloat16, d_img), torch.bfloat16)
    print(f"SDXL + ip-adapter-plus_sdxl_vit-h shape, 64x64, B=2, bf16: {err:.2e}")


def test_scale_changes_share_one_graph_and_replays_are_bitwise_identical():
    cfg = uo.tiny_config()
    fast, oracle = _plus_pair(cfg, 6, torch.float16, 128)
    args = _inputs(cfg, 2, 32, 32, torch.float16, 128)
    first, _ = _check(fast, oracle, *args, torch.float16)
    n = len(fast.forward._cached)
    again = fast(*args[:3], added_cond_kwargs=args[3]).sample
    assert torch.equal(first, again)
    for scale in (0.6, {"down_blocks.1": 1.0, "up_blocks.2": 0.3}, -0.5):
        ipo.set_ip_adapter_scale(fast, scale)
        ipo.set_ip_adapter_scale(oracle, scale)
        _check(fast, oracle, *args, torch.float16)
    assert len(fast.forward._cached) == n


def test_all_scales_zero_equal_the_unet_without_the_adapter():
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_unet
    cfg = uo.tiny_config()
    fast, _ = _plus_pair(cfg, 7, torch.float16, 128)
    plain = uo.build_unet(cfg, seed=7, dtype=torch.float16, device=DEV)
    plain.load_state_dict({k: v for k, v in fast.state_dict().items() if k in plain.state_dict()})
    plain = compile_unet(plain, CompilationConfig.Default())
    ipo.set_ip_adapter_scale(fast, 0.0)
    s, t, e, kw = _inputs(cfg, 2, 32, 32, torch.float16, 128)
    assert torch.equal(fast(s, t, e, added_cond_kwargs=kw).sample, plain(s, t, e).sample)


@pytest.mark.parametrize("name", [f"{PP}.layers.1.attn.to_k.weight", f"{PP}.latents"])
def test_in_place_update_of_the_resampler_is_seen(name):
    cfg = uo.tiny_config()
    fast, oracle = _plus_pair(cfg, 8, torch.float16, 128)
    args = _inputs(cfg, 2, 32, 32, torch.float16, 128)
    before, _ = _check(fast, oracle, *args, torch.float16)
    n = len(fast.forward._cached)
    with torch.no_grad():
        w = dict(fast.named_parameters())[name]
        w.mul_(-2.0)
        dict(oracle.named_parameters())[name].copy_(w.float())
    after, _ = _check(fast, oracle, *args, torch.float16)
    assert not torch.equal(before, after) and len(fast.forward._cached) == n


def test_refusals_after_compile():
    cfg = uo.tiny_config()
    fast, _ = _plus_pair(cfg, 9, torch.float16, 128)
    s, t, e, kw = _inputs(cfg, 1, 32, 32, torch.float16, 128)
    with pytest.raises(ValueError, match="image_embeds"):
        fast(s, t, e)
    with pytest.raises(ValueError, match=r"\[1, n_images, S_img, 128\]"):
        fast(s, t, e, added_cond_kwargs=dict(image_embeds=[kw["image_embeds"][0][:, :, 0]]))
    with pytest.raises(NotImplementedError, match="ip_adapter_masks"):
        fast(s, t, e, added_cond_kwargs=kw, cross_attention_kwargs={"ip_adapter_masks": [None]})
    fast.encoder_hid_proj = ipo.MultiIPAdapterImageProjection([ipo.ImageProjection(128, 128)]).to(DEV)  # replaced
    with pytest.raises(NotImplementedError, match="compile"):
        fast(s, t, e, added_cond_kwargs=kw)
    fast.encoder_hid_proj = None  # unload_ip_adapter
    with pytest.raises(NotImplementedError, match="compile"):
        fast(s, t, e, added_cond_kwargs=kw)


def test_compile_runs_the_vision_tower_hidden_states_into_a_plus_unet_natively():
    transformers = pytest.importorskip("transformers")
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile
    vcfg = transformers.CLIPVisionConfig(hidden_size=128, intermediate_size=256, num_hidden_layers=3,
                                         num_attention_heads=2, image_size=224, patch_size=14, projection_dim=64,
                                         hidden_act="gelu")
    torch.manual_seed(0)
    enc = transformers.CLIPVisionModelWithProjection(vcfg).to(DEV, torch.float16).eval()
    cfg = uo.tiny_config()
    unet = ipp.load_ip_adapter_plus(uo.build_unet(cfg, seed=11, dtype=torch.float16, device=DEV), 128, seed=12,
                                    gain=4.0)
    oracle = ipp.load_ip_adapter_plus(uo.build_unet(cfg, seed=11, dtype=torch.float32, device=DEV), 128, seed=12,
                                      gain=4.0)
    oracle.load_state_dict({k: v.float() for k, v in unet.state_dict().items()})
    pipe = types.SimpleNamespace(unet=unet, image_encoder=enc, vae=None, text_encoder=None, controlnet=None)
    pipe = compile(pipe, CompilationConfig.Default())
    lib = _lib.lib()
    pix = torch.randn(2, 3, 224, 224, device=DEV).half()
    n0 = lib.sfb_launch_count()
    feats = pipe.image_encoder(pix, output_hidden_states=True).hidden_states[-2]
    assert lib.sfb_launch_count() > n0 and hasattr(pipe.image_encoder.forward, "_compiled")
    assert tuple(feats.shape) == (2, S_IMG, 128)
    s, t, e, _ = _inputs(cfg, 2, 32, 32, torch.float16, 128)
    n0 = lib.sfb_launch_count()
    got = pipe.unet(s, t, e, added_cond_kwargs={"image_embeds": [feats[:, None]]}).sample
    assert lib.sfb_launch_count() > n0 and hasattr(pipe.unet.forward, "_compiled")
    with torch.no_grad():
        ref = oracle(s.float(), t, e.float(), added_cond_kwargs={"image_embeds": [feats[:, None].float()]}).sample
    err = _rel(got, ref)
    print(f"compile(pipe): CLIP hidden_states[-2] -> tiny Plus UNet: {err:.2e}")
    assert err <= MODEL_TOL[torch.float16]
