"""IP-Adapter on the GPU: sfb_attention_ip against float64, every distinct launch of the IP-Adapter plans
replayed, and whole-UNet parity with the oracle adapter (oracle/ip_adapter_oracle.py)."""
import ctypes as C
import math
import types

import pytest
import torch

import plan_launches as pl
from kernel_checks import rel_err
from oracle import controlnet_oracle as co
from oracle import ip_adapter_oracle as ipo
from oracle import unet_oracle as uo
from sfast_b200 import _lib, ops
from sfast_b200._lib import TensorMap
from sfast_b200.plan import PackedWeights, UNetPlan
from sfast_b200.unet_spec import ip_adapter_geometry, param_shapes, spec_from_config

pytestmark = pytest.mark.gpu

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

DEV = "cuda"
MODEL_TOL = {torch.float16: 1e-2, torch.bfloat16: 4e-2}
DTS = {_lib.SFB_F16: torch.float16, _lib.SFB_BF16: torch.bfloat16}


def _rel(got, ref):
    """max(global max-norm error, elementwise |d| / (|ref| + rms(ref))), as in test_unet_gpu.py"""
    got, ref = got.float(), ref.float()
    d = (got - ref).abs()
    rms = ref.pow(2).mean().sqrt()
    return max((d.max() / ref.abs().max()).item(), (d / (ref.abs() + rms)).max().item())


# ---------------------------------------------------------------------------------------------------
# kernel
# ---------------------------------------------------------------------------------------------------
def _ip_operands(B, H, D, sq, skv, seq_ip, kv, dt, peaked, k_ip_rows=None):
    """Random q / k / v^T and image k / v^T laid out as the plan lays them out, fp64 copies of the logical
    tensors, and the tensor maps."""
    bh = B * H
    qp, dv = ops.tk_cols(D), (D + 1 + 15) // 16 * 16
    vtp = (skv + 63) // 64 * 64
    k_ip_rows = k_ip_rows or seq_ip
    q = torch.zeros(bh, sq, qp, device=DEV, dtype=dt)
    k = torch.zeros(bh, skv, qp, device=DEV, dtype=dt)
    vt = torch.zeros(bh, dv, vtp, device=DEV, dtype=dt)
    ki = torch.zeros(bh, k_ip_rows, qp, device=DEV, dtype=dt)
    vti = torch.zeros(bh, dv, kv, device=DEV, dtype=dt)
    q[..., :D] = pl._randn(bh * sq * D, dt, 8.0 if peaked else 1.0).view(bh, sq, D)
    k[..., :D] = pl._randn(bh * skv * D, dt).view(bh, skv, D)
    vt[:, :D, :skv] = pl._randn(bh * D * skv, dt).view(bh, D, skv)
    vt[:, D, :] = 1.0
    ki[:, :seq_ip, :D] = pl._randn(bh * seq_ip * D, dt).view(bh, seq_ip, D)
    vti[:, :D, :seq_ip] = pl._randn(bh * D * seq_ip, dt).view(bh, D, seq_ip)
    maps = [TensorMap.matrix(q.data_ptr(), bh * sq, qp, qp, 128),
            TensorMap.matrix(k.data_ptr(), bh * skv, qp, qp, kv),
            TensorMap.matrix(vt.data_ptr(), bh * dv, vtp, vtp, dv),
            TensorMap.matrix(ki.data_ptr(), bh * k_ip_rows, qp, qp, kv),
            TensorMap.matrix(vti.data_ptr(), bh * dv, kv, kv, dv)]
    t = dict(q=q[..., :D].double(), k=k[..., :D].double(), v=vt[:, :D, :skv].double().transpose(1, 2),
             ki=ki[:, :seq_ip, :D].double(), vi=vti[:, :D, :seq_ip].double().transpose(1, 2))
    return (q, k, vt, ki, vti), t, maps


def _ip_params(maps, B, H, D, sq, skv, seq_ip, kv, dt, k_ip_rows, scale_t, out_ptr):
    p = _lib.AttnIpParams()
    b = p.base
    b.tmap_q, b.tmap_k, b.tmap_vt = maps[0].ptr, maps[1].ptr, maps[2].ptr
    b.out = out_ptr
    b.batch, b.heads, b.head_dim, b.seq_q, b.seq_kv = B, H, D, sq, skv
    b.q_rows, b.k_rows, b.vt_rows = sq, skv, (D + 1 + 15) // 16 * 16
    b.dtype, b.scale, b.kv_tile, b.causal = ops.dtype_code(dt), 1.0 / math.sqrt(D), kv, 0
    p.tmap_k_ip, p.tmap_vt_ip = maps[3].ptr, maps[4].ptr
    p.seq_ip, p.k_ip_rows = seq_ip, k_ip_rows
    p.ip_scale = scale_t.data_ptr()
    return p


def run_attention_ip(B, H, D, sq, skv, seq_ip, kv, dt, scales, peaked=True):
    """sfb_attention_ip at each scale (one operand set) and sfb_attention on the text operands: {scale: (rel
    err vs float64, outside-output intact, bits equal to sfb_attention's)}."""
    bufs, t, maps = _ip_operands(B, H, D, sq, skv, seq_ip, kv, dt, peaked)
    sc = 1.0 / math.sqrt(D)
    text = pl.ref_attention(t["q"], t["k"], t["v"], sc, False)
    img = pl.ref_attention(t["q"], t["ki"], t["vi"], sc, False)
    base = pl.Canvas(dt, 0, B * sq, H * D)
    p = _ip_params(maps, B, H, D, sq, skv, seq_ip, kv, dt, seq_ip, torch.zeros(1, device=DEV), base.ptr)
    base.arm()
    _lib.check(_lib.lib().sfb_attention(C.byref(p.base), pl._stream()), "sfb_attention")
    torch.cuda.synchronize()
    plain = base.take(base.region(B * sq, H * D))
    out = {}
    for s in scales:
        scale_t = torch.tensor([s], device=DEV, dtype=torch.float32)
        cv = pl.Canvas(dt, 0, B * sq, H * D)
        p = _ip_params(maps, B, H, D, sq, skv, seq_ip, kv, dt, seq_ip, scale_t, cv.ptr)
        cv.arm()
        _lib.check(_lib.lib().sfb_attention_ip(C.byref(p), pl._stream()), "sfb_attention_ip")
        torch.cuda.synchronize()
        got = cv.take(cv.region(B * sq, H * D))
        ref = (text + s * img).view(B, H, sq, D).permute(0, 2, 1, 3).reshape(B * sq, H * D)
        out[s] = (rel_err(got, ref), cv.intact(), torch.equal(got.view(torch.int16), plain.view(torch.int16)))
    del bufs
    return out


PAIRS = [(40, 128), (40, 64), (64, 128), (64, 64), (80, 128), (160, 128), (160, 64)]


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("D,kv", PAIRS)
def test_attention_ip_matches_float64(D, kv, dt):
    torch.manual_seed(D * 7 + kv)
    tl = pl.tol("attention", dt)
    for seq_ip in (4, 16):
        res = run_attention_ip(2, 3, D, 200, 77, seq_ip, kv, dt, (0.0, 0.6, 1.0, -0.5))
        for s, (err, intact, same) in res.items():
            print(f"D={D} kv={kv} {dt} seq_ip={seq_ip} scale={s}: err {err:.2e}")
            assert intact, (seq_ip, s)
            assert err <= tl, (seq_ip, s, err)
            if s == 0.0:
                assert same, "scale 0 must give sfb_attention's bits"


def test_attention_ip_full_kv_tile():
    """seq_ip = kv_tile (the limit), unpeaked scores."""
    torch.manual_seed(3)
    for D, kv in ((40, 128), (64, 64)):
        res = run_attention_ip(1, 2, D, 130, 77, kv, kv, torch.float16, (0.6,), peaked=False)
        err, intact, _ = res[0.6]
        assert intact and err <= pl.tol("attention", torch.float16), (D, kv, err)


# ---------------------------------------------------------------------------------------------------
# every distinct launch of the IP-Adapter plans
# ---------------------------------------------------------------------------------------------------
def _dry_ip_plan(cfg_name, b, h, w, dt, d_img, ip_len):
    spec = spec_from_config(getattr(uo, cfg_name)())
    spec.ip = ip_adapter_geometry(spec, d_img)
    sd = {k: torch.empty(v, dtype=dt, device="meta") for k, v in param_shapes(spec).items()}
    with pl.recording_map_offsets():
        return UNetPlan(PackedWeights(spec, sd, dt, "meta", dry=True), b, h, w, ip_len=ip_len)


IP_PLANS = [
    ("tiny_ip4_2x32x32", lambda: _dry_ip_plan("tiny_config", 2, 32, 32, torch.float16, 64, 4)),
    ("sd15_ip4_2x64x64", lambda: _dry_ip_plan("sd15_config", 2, 64, 64, torch.float16, 1024, 4)),
    ("sd15_ip16_1x64x96", lambda: _dry_ip_plan("sd15_config", 1, 64, 96, torch.float16, 1024, 16)),
    ("sdxl_bf16_ip4_2x128x128", lambda: _dry_ip_plan("sdxl_config", 2, 128, 128, torch.bfloat16, 1024, 4)),
    ("sdxl_ip8_1x64x64", lambda: _dry_ip_plan("sdxl_config", 1, 64, 64, torch.float16, 1280, 8)),
]


def _ip_key(op):
    """Launch key of an sfb_attention_ip op: plan_launches' key of its text launch plus the image fields."""
    p, tki, tvi = op.keep[:3]
    text = types.SimpleNamespace(fn=types.SimpleNamespace(name="sfb_attention"), keep=(p.base,) + tuple(op.keep[6:9]))
    return ("sfb_attention_ip", pl.launch_key(text), p.seq_ip, p.k_ip_rows, tki.geom, tvi.geom)


def _replay_attention_ip(op):
    p0 = op.keep[0]
    b, tki, tvi = p0.base, op.keep[1], op.keep[2]
    dt = DTS[b.dtype]
    assert tki.geom[1] == b.batch * b.heads * p0.k_ip_rows and tvi.geom[2] == b.kv_tile
    res = run_attention_ip(b.batch, b.heads, b.head_dim, b.seq_q, b.seq_kv, p0.seq_ip, b.kv_tile, dt, (0.0, 0.75))
    ok = all(intact and err <= pl.tol("attention", dt) for err, intact, _ in res.values()) and res[0.0][2]
    return ok, max(e for e, _, _ in res.values())


def test_every_ip_adapter_plan_launch_matches_float64():
    entries = {}
    for pname, build in IP_PLANS:
        plan = build()
        for op in plan.all_ops():
            if op.fn is None or op.fn.name in pl.SKIP:
                continue
            name = op.fn.name
            if name == "sfb_attention_ip":
                entries.setdefault(_ip_key(op), (pname, op))
            elif ".ip_kv" in op.name or op.name.startswith("encoder_hid_proj"):
                entries.setdefault(pl.launch_key(op), (pname, op))
    names = {op.fn.name for _, op in entries.values()}
    assert {"sfb_attention_ip", "sfb_gemm", "sfb_small_linear", "sfb_layer_norm"} <= names, names
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
    print(f"{len(entries)} distinct IP-Adapter plan launches replayed")
    assert not failures, "\n".join(failures)


# ---------------------------------------------------------------------------------------------------
# whole model
# ---------------------------------------------------------------------------------------------------
def _ip_pair(cfg, seed, dt, d_img, graph=True, gain=4.0):
    """(compiled fast UNet with a random adapter, fp32 oracle with the same weights, adapter-free copy of the
    fast UNet's weights compiled separately)."""
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_unet
    fast = ipo.load_ip_adapter(uo.build_unet(cfg, seed=seed, dtype=dt, device=DEV), d_img, seed=seed + 1, gain=gain)
    oracle = ipo.load_ip_adapter(uo.build_unet(cfg, seed=seed, dtype=torch.float32, device=DEV), d_img,
                                 seed=seed + 1, gain=gain)
    oracle.load_state_dict({k: v.float() for k, v in fast.state_dict().items()})
    cc = CompilationConfig.Default()
    cc.enable_cuda_graph = graph
    return compile_unet(fast, cc), oracle


def _inputs(cfg, b, h, w, dt, d_img, n_img=1, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    sample = torch.randn(b, 4, h, w, device=DEV, generator=g).to(dt)
    ehs = torch.randn(b, 77, cfg.cross_attention_dim, device=DEV, generator=g).to(dt)
    emb = torch.randn(b, n_img, d_img, device=DEV, generator=g).to(dt)
    kw = dict(image_embeds=[emb])
    if cfg.addition_embed_type == "text_time":
        kw.update(text_embeds=torch.randn(b, 1280, device=DEV, generator=g).to(dt),
                  time_ids=torch.tensor([[h * 8, w * 8, 0, 0, h * 8, w * 8]] * b, device=DEV, dtype=torch.float32))
    return sample, torch.tensor(437, device=DEV), ehs, kw


def _f32(kw):
    return {k: ([x.float() for x in v] if isinstance(v, list) else v.float()) for k, v in kw.items()}


def _check(fast, oracle, sample, t, ehs, kw, dt, tol=None, **call):
    got = fast(sample, t, ehs, added_cond_kwargs=kw, **call).sample
    with torch.no_grad():
        ref = oracle(sample.float(), t, ehs.float(), added_cond_kwargs=_f32(kw), **call).sample
    err = _rel(got, ref)
    assert err <= (tol or MODEL_TOL[dt]), err
    return got, err


@pytest.mark.parametrize("graph", [True, False])
def test_tiny_unet_with_ip_adapter_matches_the_oracle(graph):
    cfg = uo.tiny_config()
    fast, oracle = _ip_pair(cfg, 3, torch.float16, 64, graph)
    for b in (1, 2):
        for n_img in (1, 4):
            _, err = _check(fast, oracle, *_inputs(cfg, b, 32, 32, torch.float16, 64, n_img), torch.float16)
            print(f"tiny B={b} n_img={n_img} graph={graph}: {err:.2e}")
    # the deprecated bare [B, D_img] form
    s, t, e, kw = _inputs(cfg, 2, 32, 32, torch.float16, 64)
    kw["image_embeds"] = kw["image_embeds"][0][:, 0]
    _check(fast, oracle, s, t, e, kw, torch.float16)


def test_sd15_unet_with_ip_adapter_matches_the_oracle():
    cfg = uo.sd15_config()
    fast, oracle = _ip_pair(cfg, 1, torch.float16, 1024)
    _, err = _check(fast, oracle, *_inputs(cfg, 2, 64, 64, torch.float16, 1024), torch.float16)
    print(f"SD-1.5 + ip-adapter_sd15 shape, 64x64, B=2: {err:.2e}")


def test_sdxl_unet_with_vit_h_ip_adapter_matches_the_oracle_bf16():
    cfg = uo.sdxl_config()
    fast, oracle = _ip_pair(cfg, 2, torch.bfloat16, 1024)
    _, err = _check(fast, oracle, *_inputs(cfg, 2, 64, 64, torch.bfloat16, 1024), torch.bfloat16)
    print(f"SDXL + ViT-H adapter, 64x64, B=2, bf16: {err:.2e}")


def test_controlnet_and_ip_adapter_together_at_the_community_example_shape():
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_controlnet
    ucfg, ccfg = uo.sd15_config(), co.sd15_config()
    fast, oracle = _ip_pair(ucfg, 4, torch.float16, 1024)
    cn = co.build_controlnet(ccfg, seed=5, dtype=torch.float16, device=DEV)
    cn_ref = co.build_controlnet(ccfg, seed=5, dtype=torch.float32, device=DEV)
    cn_ref.load_state_dict({k: v.float() for k, v in cn.state_dict().items()})
    cn = compile_controlnet(cn, CompilationConfig.Default())
    sample, t, ehs, kw = _inputs(ucfg, 2, 64, 96, torch.float16, 1024)
    cond = torch.rand(2, 3, 512, 768, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1)).half()
    down, mid = cn(sample, t, ehs, cond, return_dict=False)
    got = fast(sample, t, ehs, added_cond_kwargs=kw, down_block_additional_residuals=down,
               mid_block_additional_residual=mid).sample
    with torch.no_grad():
        rd, rm = cn_ref(sample.float(), t, ehs.float(), cond.float(), return_dict=False)
        ref = oracle(sample.float(), t, ehs.float(), added_cond_kwargs=_f32(kw),
                     down_block_additional_residuals=rd, mid_block_additional_residual=rm).sample
    err = _rel(got, ref)
    print(f"ControlNet + IP-Adapter (SD-1.5, B=2, 64x96): {err:.2e}")
    assert err <= MODEL_TOL[torch.float16], err


def test_scale_changes_share_one_graph_and_replays_are_bitwise_identical():
    cfg = uo.tiny_config()
    fast, oracle = _ip_pair(cfg, 6, torch.float16, 64)
    args = _inputs(cfg, 2, 32, 32, torch.float16, 64)
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
    fast, _ = _ip_pair(cfg, 7, torch.float16, 64)
    plain = uo.build_unet(cfg, seed=7, dtype=torch.float16, device=DEV)
    plain.load_state_dict({k: v for k, v in fast.state_dict().items() if k in plain.state_dict()})
    plain = compile_unet(plain, CompilationConfig.Default())
    ipo.set_ip_adapter_scale(fast, 0.0)
    s, t, e, kw = _inputs(cfg, 2, 32, 32, torch.float16, 64)
    assert torch.equal(fast(s, t, e, added_cond_kwargs=kw).sample, plain(s, t, e).sample)


def test_in_place_update_of_the_image_projection_is_seen():
    cfg = uo.tiny_config()
    fast, oracle = _ip_pair(cfg, 8, torch.float16, 64)
    args = _inputs(cfg, 2, 32, 32, torch.float16, 64)
    before, _ = _check(fast, oracle, *args, torch.float16)
    name = "down_blocks.1.attentions.0.transformer_blocks.0.attn2.processor.to_k_ip.0.weight"
    with torch.no_grad():
        w = dict(fast.named_parameters())[name]
        w.mul_(3.0)
        dict(oracle.named_parameters())[name].copy_(w.float())
    after, _ = _check(fast, oracle, *args, torch.float16)
    assert not torch.equal(before, after)


def test_refusals_after_compile():
    cfg = uo.tiny_config()
    fast, _ = _ip_pair(cfg, 9, torch.float16, 64)
    s, t, e, kw = _inputs(cfg, 1, 32, 32, torch.float16, 64)
    with pytest.raises(ValueError, match="image_embeds"):
        fast(s, t, e)
    with pytest.raises(NotImplementedError, match="ip_adapter_masks"):
        fast(s, t, e, added_cond_kwargs=kw, cross_attention_kwargs={"ip_adapter_masks": [None]})
    fast.encoder_hid_proj = None  # unload_ip_adapter
    with pytest.raises(NotImplementedError, match="compile"):
        fast(s, t, e, added_cond_kwargs=kw)
    # an adapter loaded after compile() is not dropped silently
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_unet
    plain = compile_unet(uo.build_unet(cfg, seed=9, dtype=torch.float16, device=DEV), CompilationConfig.Default())
    plain(s, t, e)
    compiled_forward = plain.forward
    ipo.load_ip_adapter(plain, 64)
    plain.forward = compiled_forward  # diffusers' load_ip_adapter leaves forward alone
    with pytest.raises(NotImplementedError, match="compile"):
        plain(s, t, e, added_cond_kwargs=kw)


def test_compile_runs_image_encoder_and_ip_adapter_unet_natively():
    transformers = pytest.importorskip("transformers")
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile
    vcfg = transformers.CLIPVisionConfig(hidden_size=128, intermediate_size=256, num_hidden_layers=2,
                                         num_attention_heads=2, image_size=224, patch_size=14, projection_dim=64,
                                         hidden_act="gelu")
    torch.manual_seed(0)
    enc = transformers.CLIPVisionModelWithProjection(vcfg).to(DEV, torch.float16).eval()
    cfg = uo.tiny_config()
    unet = ipo.load_ip_adapter(uo.build_unet(cfg, seed=11, dtype=torch.float16, device=DEV), 64, seed=12, gain=4.0)
    oracle = ipo.load_ip_adapter(uo.build_unet(cfg, seed=11, dtype=torch.float32, device=DEV), 64, seed=12, gain=4.0)
    oracle.load_state_dict({k: v.float() for k, v in unet.state_dict().items()})
    pipe = types.SimpleNamespace(unet=unet, image_encoder=enc, vae=None, text_encoder=None, controlnet=None)
    pipe = compile(pipe, CompilationConfig.Default())
    lib = _lib.lib()
    pix = torch.randn(2, 3, 224, 224, device=DEV).half()
    n0 = lib.sfb_launch_count()
    emb = pipe.image_encoder(pix).image_embeds
    assert lib.sfb_launch_count() > n0 and hasattr(pipe.image_encoder.forward, "_compiled")
    s, t, e, _ = _inputs(cfg, 2, 32, 32, torch.float16, 64)
    n0 = lib.sfb_launch_count()
    got = pipe.unet(s, t, e, added_cond_kwargs={"image_embeds": [emb[:, None]]}).sample
    assert lib.sfb_launch_count() > n0 and hasattr(pipe.unet.forward, "_compiled")
    with torch.no_grad():
        ref = oracle(s.float(), t, e.float(), added_cond_kwargs={"image_embeds": [emb[:, None].float()]}).sample
    assert _rel(got, ref) <= MODEL_TOL[torch.float16]
