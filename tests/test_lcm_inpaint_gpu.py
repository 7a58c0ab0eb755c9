"""Inpainting and LCM UNets on the GPU (pytest -m gpu): sfb_im2col_in_wide bit-exact against F.unfold, the K = 128
conv_in GEMM against a float64 conv, a float64 replay of every launch the new plans add (with the access-model
check), the whole UNet against the fp32 oracle with and without the CUDA graph, the guidance input, and the
combinations with ControlNet residuals and PEFT LoRA adapters."""
import copy
import types

import pytest
import torch
import torch.nn.functional as F

import lcm_inpaint_checks as lc
import plan_launches as pl
from kernel_checks import rel_err
from oracle import lcm_inpaint_oracle as lio
from oracle import lora_oracle as lo
from oracle import unet_oracle as uo
from sfast_b200 import _lib, ops
from sfast_b200.plan import PackedWeights, UNetPlan
from sfast_b200.unet_spec import param_shapes, spec_from_config
from test_freeu_gpu import _controlnet_residuals

pytestmark = pytest.mark.gpu
F16, BF16 = torch.float16, torch.bfloat16
TOL = {F16: 1e-2, BF16: 4e-2}
DEV = "cuda"


def _rel(got, ref):
    got, ref = got.float(), ref.float()
    d = (got - ref).abs()
    rms = ref.pow(2).mean().sqrt()
    return max((d.max() / ref.abs().max()).item(), (d / (ref.abs() + rms)).max().item())


def tiny_inpaint_config():
    return lio.tiny_config(in_channels=9)


def tiny_lcm_config():
    return lio.tiny_config(time_cond_proj_dim=32)


def tiny_sd2_config():
    """SD-2.1 768-v's topology at the tiny width: linear projections, head_dim 32, upcast_attention."""
    return lio.tiny_config(use_linear_projection=True, attention_head_dim=(2, 4, 8, 8), upcast_attention=True)


# ---- the kernel on its own
IM2COL_CASES = [(n, h, w, cin) for cin in range(9, 15) for n, h, w in ((1, 1, 1), (2, 3, 5), (3, 7, 13))] + [
    (2, 64, 64, 9), (2, 128, 128, 9), (1, 17, 33, 14), (4, 40, 72, 11)]


@pytest.mark.parametrize("case", IM2COL_CASES, ids=[f"{n}x{h}x{w}_c{c}" for n, h, w, c in IM2COL_CASES])
def test_wide_im2col_is_bit_exact(case):
    n, h, w, cin = case
    torch.manual_seed(n * 1000 + h * 10 + cin)
    res = lc.replay_im2col_wide(types.SimpleNamespace(args=(0, 0, n, h, w, cin)))
    assert res.ok, res.parts


@pytest.mark.parametrize("dt", [F16, BF16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("n,h,w,cin,cout", [(2, 64, 64, 9, 320), (1, 24, 40, 14, 64), (3, 8, 16, 9, 64)])
def test_conv_in_gemm_with_k128_matches_a_float64_conv(n, h, w, cin, cout, dt):
    lib, s = _lib.lib(), torch.cuda.current_stream().cuda_stream
    g = torch.Generator(device=DEV).manual_seed(cin)
    x = torch.randn(n, cin, h, w, device=DEV, generator=g).to(dt)
    wt = (0.2 * torch.randn(cout, cin, 3, 3, device=DEV, generator=g)).to(dt)
    b = torch.randn(cout, device=DEV, generator=g)
    wp = torch.zeros(cout, 128, device=DEV, dtype=dt)
    wp[:, :9 * cin] = ops.pack_conv3x3(wt, dt)
    M = n * h * w
    a = torch.zeros(M, 128, device=DEV, dtype=dt)
    y = torch.zeros(M, cout, device=DEV, dtype=dt)
    _lib.check(lib.sfb_im2col_in_wide(x.data_ptr(), a.data_ptr(), n, h, w, cin, s))
    ops.gemm_op("conv_in", lib, a=ops.a_matrix(a.data_ptr(), M, 128, 128), b=ops.Mat(wp), M=M, N=cout, K=128,
                dt=dt, out=y, ldo=cout, bias=b).launch(s)
    torch.cuda.synchronize()
    ref = F.conv2d(x.double(), wt.double(), b.double(), padding=1).permute(0, 2, 3, 1).reshape(M, cout)
    assert rel_err(y, ref) < pl.tol("pointwise", dt) * 4


def _dry_plan(cfg, b, h, w, dt):
    spec = spec_from_config(cfg)
    sd = {k: torch.empty(tuple(v), dtype=dt, device="meta") for k, v in param_shapes(spec).items()}
    return UNetPlan(PackedWeights(spec, sd, dt, "meta", dry=True), b, h, w)


def _new_entries():
    """Every launch key of the inpainting / LCM plans that the plain plans of the same sizes do not have."""
    pairs = [(lio.sd15_inpaint_config, uo.sd15_config, 2, 64, 64, F16),
             (lio.sdxl_inpaint_config, uo.sdxl_config, 2, 128, 128, BF16),
             (lio.sd15_inpaint_config, uo.sd15_config, 1, 40, 72, F16),
             (lio.lcm_sd15_config, uo.sd15_config, 4, 64, 64, F16),
             (lio.lcm_sdxl_config, uo.sdxl_config, 1, 128, 128, BF16)]
    out = {}
    for new, old, b, h, w, dt in pairs:
        with pl.recording_map_offsets():  # (the GEMM replay reads each map's offset in its buffer)
            plain, plan = _dry_plan(old(), b, h, w, dt), _dry_plan(new(), b, h, w, dt)
        have = {k for _, k, _ in pl.launches(plain)}
        for name, key, op in pl.launches(plan):
            if key not in have:
                out.setdefault(key, dict(op=op, name=name, plans=[new.__name__]))
    return out


def test_every_new_launch_matches_float64_and_the_access_model():
    entries = _new_entries()
    names = sorted({e["name"] for e in entries.values()})
    assert names == ["sfb_gemm", "sfb_im2col_in_wide", "sfb_small_linear"], names
    for key, ent in entries.items():
        res = pl.replay(key, ent, soundness="rw")
        print(pl.describe(key), [(w, f"{e:.2e}") for w, e, _ in res.parts])
        assert res.ok, (pl.describe(key), res.parts, getattr(res, "model", None))


# ---- the whole UNet against the oracle
def _pair(cfg, seed, dt):
    oracle = lio.build_unet(cfg, seed=seed, dtype=torch.float32, device=DEV)
    fast = copy.deepcopy(oracle).to(dt)
    oracle.load_state_dict({k: v.float() for k, v in fast.state_dict().items()})
    return oracle, fast


def _compile(m, graph=True):
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_unet
    c = CompilationConfig.Default()
    c.enable_cuda_graph = graph
    return compile_unet(m, c)


def _inputs(cfg, b, h, w, dt, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    s = torch.randn(b, cfg.in_channels, h, w, device=DEV, generator=g).to(dt)
    e = torch.randn(b, 77, cfg.cross_attention_dim, device=DEV, generator=g).to(dt)
    kw = {}
    if cfg.addition_embed_type == "text_time":
        kw["added_cond_kwargs"] = {"text_embeds": torch.randn(b, 1280, device=DEV, generator=g).to(dt),
                                   "time_ids": torch.tensor([[8. * h, 8 * w, 0, 0, 8 * h, 8 * w]] * b, device=DEV).to(dt)}
    return s, e, kw


def _f32(v):
    if isinstance(v, dict):
        return {k: _f32(x) for k, x in v.items()}
    if isinstance(v, (list, tuple)):
        return [_f32(x) for x in v]
    return v.float() if torch.is_tensor(v) and v.is_floating_point() else v


def _ref(oracle, s, t, e, **kw):
    with torch.no_grad():
        return lio.unet_forward(oracle, s.float(), t, e.float(), **_f32(kw)).sample


def _guidance(b, dim, w, dt):
    """The LCM pipeline's guidance-scale embedding of (w - 1) (diffusers get_guidance_scale_embedding), [b, dim]."""
    w = torch.as_tensor(w, dtype=torch.float32, device=DEV).reshape(-1).expand(b) * 1000.0 - 1000.0
    half = dim // 2
    f = torch.exp(torch.arange(half, device=DEV) * -(torch.log(torch.tensor(10000.0)) / (half - 1)))
    a = w[:, None] * f[None, :]
    return torch.cat([torch.sin(a), torch.cos(a)], 1).to(dt)


UNET_CASES = [  # name, config, batch, h, w, dtype, guidance scales (LCM)
    ("tiny_inpaint_b1", tiny_inpaint_config, 1, 32, 32, F16, None),
    ("tiny_inpaint_b2", tiny_inpaint_config, 2, 24, 40, F16, None),
    ("tiny_inpaint_b3", tiny_inpaint_config, 3, 16, 16, F16, None),
    ("sd15_inpaint_64", lio.sd15_inpaint_config, 2, 64, 64, F16, None),
    ("sdxl_inpaint_128_bf16", lio.sdxl_inpaint_config, 2, 128, 128, BF16, None),
    ("sdxl_inpaint_128_fp16", lio.sdxl_inpaint_config, 2, 128, 128, F16, None),
    ("tiny_lcm", tiny_lcm_config, 2, 32, 32, F16, (8.0,)),
    ("sd15_lcm_b1", lio.lcm_sd15_config, 1, 64, 64, F16, (8.0,)),
    ("sd15_lcm_b4_two_guidance", lio.lcm_sd15_config, 4, 64, 64, F16, (8.0, 8.0, 2.5, 2.5)),
    ("sdxl_lcm_128", lio.lcm_sdxl_config, 1, 128, 128, BF16, (6.0,)),
    ("tiny_sd2_upcast", tiny_sd2_config, 2, 32, 32, F16, None),
]


@pytest.mark.parametrize("name,cfgf,b,h,w,dt,gs", UNET_CASES, ids=[c[0] for c in UNET_CASES])
def test_unet_matches_the_oracle(name, cfgf, b, h, w, dt, gs):
    cfg = cfgf()
    oracle, fast = _pair(cfg, 21, dt)
    s, e, kw = _inputs(cfg, b, h, w, dt)
    t = torch.tensor(500, device=DEV)
    if gs is not None:
        kw["timestep_cond"] = _guidance(b, cfg.time_cond_proj_dim, torch.tensor(gs), dt)
    ref = _ref(oracle, s, t, e, **kw)
    del oracle
    for graph in (False, True):
        got = _compile(fast, graph)(s, t, e, **kw).sample
        err = _rel(got, ref)
        print(f"{name} graph={graph}: rel err {err:.3e}")
        assert err < TOL[dt]


# ---- the guidance input
def test_timestep_cond_none_is_the_unet_without_cond_proj():
    cfg = tiny_lcm_config()
    _, lcm = _pair(cfg, 5, F16)
    plain = uo.build_unet(uo.tiny_config(), seed=5, dtype=F16, device=DEV)
    plain.load_state_dict({k: v for k, v in lcm.state_dict().items() if "cond_proj" not in k})
    s, e, _ = _inputs(cfg, 2, 32, 32, F16)
    t = torch.tensor(300, device=DEV)
    a = _compile(lcm)(s, t, e).sample
    assert torch.equal(a, _compile(plain)(s, t, e).sample)


def test_a_new_guidance_value_reuses_the_graph_and_moves_the_output():
    cfg = tiny_lcm_config()
    oracle, fast = _pair(cfg, 7, F16)
    unet = _compile(fast)
    s, e, _ = _inputs(cfg, 2, 32, 32, F16)
    t = torch.tensor(400, device=DEV)
    outs = []
    for gs in (8.0, 2.0, 8.0):
        tc = _guidance(2, 32, torch.tensor(gs), F16)
        outs.append(unet(s, t, e, timestep_cond=tc).sample)
        assert _rel(outs[-1], _ref(oracle, s, t, e, timestep_cond=tc)) < TOL[F16]
    assert len(unet.forward._cached) == 1
    assert torch.equal(outs[0], outs[2]) and _rel(outs[1], outs[0]) > 5 * TOL[F16]
    one = unet(s, t, e, timestep_cond=_guidance(1, 32, torch.tensor(2.0), F16)).sample   # [1, dim] broadcast
    assert torch.equal(one, outs[1]) and len(unet.forward._cached) == 1


# ---- combinations
@pytest.mark.parametrize("cfgf", [tiny_inpaint_config, tiny_lcm_config], ids=["inpaint", "lcm"])
def test_controlnet_residuals_in_one_call(cfgf):
    cfg = cfgf()
    oracle, fast = _pair(cfg, 13, F16)
    unet = _compile(fast)
    s, e, kw = _inputs(cfg, 2, 32, 32, F16)
    if cfg.time_cond_proj_dim:
        kw["timestep_cond"] = _guidance(2, 32, torch.tensor(4.0), F16)
    down, mid = _controlnet_residuals(cfg, 2, 32, F16)
    t = torch.tensor(600, device=DEV)
    plain_ref = _ref(oracle, s, t, e, **kw)
    kw.update(down_block_additional_residuals=down, mid_block_additional_residual=mid)
    got = unet(s, t, e, **kw).sample
    assert _rel(got, _ref(oracle, s, t, e, **kw)) < TOL[F16] and _rel(got, plain_ref) > 5 * TOL[F16]


def test_lora_on_the_wide_conv_in_and_cond_proj_merges_and_switches():
    cfg = lio.tiny_config(in_channels=9, time_cond_proj_dim=32)
    oracle, fast = _pair(cfg, 3, F16)
    targets = ["conv_in", "time_embedding.cond_proj"]
    for m in (fast, oracle):
        lo.inject_adapter(m, "a", targets, r=8, lora_alpha=16, seed=3)
        lo.inject_adapter(m, "b", targets, r=4, lora_alpha=8, seed=9)
    assert len(lo.lora_layers(fast)) == 2
    unet = _compile(fast)
    s, e, kw = _inputs(cfg, 2, 32, 32, F16)
    kw["timestep_cond"] = _guidance(2, 32, torch.tensor(8.0), F16)
    t = torch.tensor(500, device=DEV)
    lo.disable_lora(oracle)
    free = _ref(oracle, s, t, e, **kw)
    lo.enable_lora(oracle)
    outs = []
    for names in ("a", "b", "a"):
        for m in (fast, oracle):
            lo.set_adapters(m, names)
        outs.append(unet(s, t, e, **kw).sample)
        ref = _ref(oracle, s, t, e, **kw)
        assert _rel(outs[-1], ref) < TOL[F16] and _rel(ref, free) > 5 * TOL[F16], names
    assert torch.equal(outs[0], outs[2]) and len(unet.forward._cached) == 1
