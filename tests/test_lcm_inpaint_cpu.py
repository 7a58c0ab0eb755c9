"""Inpainting and LCM UNets without a GPU: the config keys the spec now accepts (time_cond_proj_dim on the UNet only,
in_channels up to 14, upcast_attention) and what it refuses by name, the oracle's parameter totals, the plans (plain
plans unchanged; an inpainting plan's conv_in as one wide im2col + a K = 128 GEMM; an LCM plan's one cond_proj launch
on the time-embedding branch), free of races and stale reads, the host validation of sfb_im2col_in_wide, and the
runtime's handling of `timestep_cond`."""
import contextlib
import hashlib
import math

import pytest
import torch

import lcm_inpaint_checks  # noqa: F401  (registers sfb_im2col_in_wide and timestep_cond_in)
import plan_hazards as ph
import plan_launches as pl
from oracle import controlnet_oracle as co
from oracle import lcm_inpaint_oracle as lio
from oracle import unet_oracle as uo
from sfast_b200 import _lib, runtime
from sfast_b200.plan import PackedWeights, UNetPlan
from sfast_b200.unet_spec import controlnet_spec_from_config, param_shapes, random_state_dict, spec_from_config
from test_freeu_cpu import PARENT, _keys
from test_host_logic import _DUMMY_PTR

_NO_GPU = pytest.mark.skipif(torch.cuda.is_available(), reason="needs a box without a GPU: launches must fail")
F16, BF16 = torch.float16, torch.bfloat16


def tiny_inpaint_config():
    return lio.tiny_config(in_channels=9)


def tiny_lcm_config():
    return lio.tiny_config(time_cond_proj_dim=32)


CFGS = {"tiny": uo.tiny_config, "sd15": uo.sd15_config, "sdxl": uo.sdxl_config,
        "tiny_inpaint": tiny_inpaint_config, "tiny_lcm": tiny_lcm_config,
        "sd15_inpaint": lio.sd15_inpaint_config, "sdxl_inpaint": lio.sdxl_inpaint_config,
        "sd15_lcm": lio.lcm_sd15_config, "sdxl_lcm": lio.lcm_sdxl_config}


# ---- the spec
def test_time_cond_proj_dim_is_accepted_on_the_unet():
    spec = spec_from_config(lio.lcm_sd15_config())
    assert spec.time_cond_dim == 256
    assert param_shapes(spec)["time_embedding.cond_proj.weight"] == (320, 256)
    assert "time_embedding.cond_proj.bias" not in param_shapes(spec)
    assert spec_from_config(uo.sd15_config()).time_cond_dim == 0
    assert spec_from_config(lio.lcm_sdxl_config()).time_cond_dim == 256


def test_controlnet_keeps_refusing_time_cond_proj_dim():
    with pytest.raises(NotImplementedError, match="time_cond_proj_dim"):
        controlnet_spec_from_config(dict(vars(co.sd15_config()), time_cond_proj_dim=256))


@pytest.mark.parametrize("dim", [100, 4, 0, -8])
def test_a_guidance_width_that_is_not_a_positive_multiple_of_8_is_refused_by_name(dim):
    with pytest.raises(NotImplementedError, match="time_cond_proj_dim"):
        spec_from_config(lio.config_with(uo.sd15_config(), time_cond_proj_dim=dim))


@pytest.mark.parametrize("cin", [9, 12, 14])
def test_in_channels_up_to_14_are_accepted(cin):
    spec = spec_from_config(lio.config_with(uo.sd15_config(), in_channels=cin))
    assert spec.in_channels == cin and param_shapes(spec)["conv_in.weight"] == (320, cin, 3, 3)


@pytest.mark.parametrize("cin", [15, 16, 32])
def test_in_channels_above_14_are_refused_by_name(cin):
    with pytest.raises(NotImplementedError, match="in_channels"):
        spec_from_config(lio.config_with(uo.sd15_config(), in_channels=cin))


@pytest.mark.parametrize("value", [True, False, None])
def test_upcast_attention_is_accepted_on_unet_and_controlnet(value):
    sd2 = dict(use_linear_projection=True, attention_head_dim=(5, 10, 20, 20), cross_attention_dim=1024,
               upcast_attention=value)
    a = spec_from_config(lio.config_with(uo.sd15_config(), **sd2))
    b = spec_from_config(lio.config_with(uo.sd15_config(), **dict(sd2, upcast_attention=False)))
    assert a == b
    controlnet_spec_from_config(dict(vars(co.sd15_config()), **sd2))


def test_random_state_dict_of_an_lcm_spec_holds_cond_proj():
    spec = spec_from_config(tiny_lcm_config())
    sd = random_state_dict(spec, seed=1)
    w = sd["time_embedding.cond_proj.weight"]
    assert tuple(w.shape) == (64, 32) and w.abs().max() <= 1 / math.sqrt(32)
    # the plain spec draws the same weights as before: cond_proj only exists in a time-cond spec
    plain = random_state_dict(spec_from_config(uo.tiny_config()), seed=1)
    assert torch.equal(plain["time_embedding.linear_1.weight"], sd["time_embedding.linear_1.weight"])


# ---- the oracle
TOTALS = {"sd15_inpaint_config": 859_535_364, "sdxl_inpaint_config": 2_567_478_084,
          "lcm_sd15_config": 859_602_884, "lcm_sdxl_config": 2_567_545_604}


@pytest.mark.parametrize("name", list(TOTALS))
def test_oracle_parameter_totals(name):
    cfg = getattr(lio, name)()
    with torch.device("meta"):
        m = uo.UNet2DConditionModel(cfg)
        if cfg.time_cond_proj_dim:
            lio.add_cond_proj(m, cfg.time_cond_proj_dim)
    assert sum(p.numel() for p in m.parameters()) == TOTALS[name]
    shapes = param_shapes(spec_from_config(cfg))
    assert sum(math.prod(s) for s in shapes.values()) == TOTALS[name]
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {k: tuple(v) for k, v in shapes.items()}


def test_oracle_without_timestep_cond_is_the_plain_time_embedding():
    m = lio.build_unet(tiny_lcm_config(), seed=3)
    plain = uo.build_unet(uo.tiny_config(), seed=3)
    plain.load_state_dict({k: v for k, v in m.state_dict().items() if "cond_proj" not in k})
    g = torch.Generator().manual_seed(0)
    x, ehs = torch.randn(1, 4, 16, 16, generator=g), torch.randn(1, 77, 128, generator=g)
    with torch.no_grad():
        ref = plain(x, 500, ehs).sample
        assert torch.equal(lio.unet_forward(m, x, 500, ehs).sample, ref)
        assert torch.equal(lio.unet_forward(m, x, 500, ehs, timestep_cond=torch.zeros(1, 32)).sample, ref)
        moved = lio.unet_forward(m, x, 500, ehs, timestep_cond=torch.randn(1, 32, generator=g)).sample
        # the condition applies to that call only
        assert torch.equal(lio.unet_forward(m, x, 500, ehs).sample, ref)
    assert (moved - ref).abs().max() > 1e-3 * ref.abs().max()


# ---- plans
def _sd(shapes, dt):
    return {k: torch.empty(tuple(v), dtype=dt, device="meta") for k, v in shapes.items()}


def _unet(cfg, b, h, w, dt=F16, **kw):
    spec = spec_from_config(CFGS[cfg]())
    return UNetPlan(PackedWeights(spec, _sd(param_shapes(spec), dt), dt, "meta", dry=True), b, h, w, **kw)


@pytest.mark.parametrize("key", list(PARENT), ids=[k[0] for k in PARENT])
def test_plain_plans_are_the_parent_plans(key):
    cfg, b, h, w = key
    plan = _unet(cfg, b, h, w, BF16 if cfg == "sdxl" else F16)
    assert hashlib.sha1(repr(_keys(plan)).encode()).hexdigest() == PARENT[key]
    assert not hasattr(plan, "timestep_cond_in")


def _names(plan):
    return [o.fn.name for o in plan.all_ops() if o.fn is not None]


@pytest.mark.parametrize("cfg,b,h,w,dt", [("tiny_inpaint", 2, 32, 32, F16), ("sd15_inpaint", 2, 64, 64, F16),
                                          ("sdxl_inpaint", 2, 128, 128, BF16), ("sd15_inpaint", 1, 40, 72, F16)])
def test_inpainting_conv_in_is_one_wide_im2col_and_a_k128_gemm(cfg, b, h, w, dt):
    plan = _unet(cfg, b, h, w, dt)
    names = _names(plan)
    assert names.count("sfb_im2col_in_wide") == 1
    assert "sfb_im2col_in" not in names and "sfb_conv_in" not in names
    ops_ = plan.all_ops()
    i = next(k for k, o in enumerate(ops_) if o.name == "conv_in.im2col")
    im2col, gemm = ops_[i], ops_[i + 1]
    assert im2col.fn.name == "sfb_im2col_in_wide" and im2col.args[2:] == (b, h, w, 9)
    assert gemm.name == "conv_in" and gemm.fn.name == "sfb_gemm"
    p = gemm.keep[0]
    assert (p.M, p.N, p.K) == (b * h * w, plan.spec.block_out_channels[0], 128)
    assert gemm.flops == 2 * b * h * w * plan.spec.block_out_channels[0] * 81
    # everything else is the plain plan's launch list
    base = spec_from_config(CFGS[cfg.replace("_inpaint", "") if cfg != "tiny_inpaint" else "tiny"]())
    plain = UNetPlan(PackedWeights(base, _sd(param_shapes(base), dt), dt, "meta", dry=True), b, h, w)
    pn = _names(plain)
    assert [n for n in names if n != "sfb_im2col_in_wide"] == [n for n in pn if n != "sfb_im2col_in"]


def test_inpainting_weight_is_padded_to_two_k_blocks():
    spec = spec_from_config(tiny_inpaint_config())
    sd = random_state_dict(spec, seed=2, dtype=torch.float32)
    pw = PackedWeights(spec, sd, torch.float32, "cpu", dry=True)
    mat = pw.conv_in_matrix("conv_in.weight")
    assert mat.k == 128 and mat.n == 64
    # (kh, kw, cin) columns, zero from 81 on
    wt = sd["conv_in.weight"]
    dense = torch.zeros(64, 128)
    dense[:, :81] = wt.permute(0, 2, 3, 1).reshape(64, 81)
    assert torch.equal(pw._padded_mat(dense, 128).data, mat.data)


@pytest.mark.parametrize("cfg,b,h,w,dt", [("tiny_lcm", 2, 32, 32, F16), ("sd15_lcm", 4, 64, 64, F16),
                                          ("sdxl_lcm", 1, 128, 128, BF16)])
def test_lcm_adds_one_cond_proj_on_the_time_embedding_branch(cfg, b, h, w, dt):
    plan = _unet(cfg, b, h, w, dt)
    plain = _unet(cfg.replace("_lcm", ""), b, h, w, dt)
    dim = plan.spec.time_cond_dim
    assert tuple(plan.timestep_cond_in.shape) == (b, dim) and plan.timestep_cond_in.dtype == dt
    side = [o.name for o in plan.side_ops]
    assert [n for n in side if n != "time_embedding.cond_proj"] == [o.name for o in plain.side_ops]
    assert side.count("time_embedding.cond_proj") == 1
    k = side.index("time_embedding.cond_proj")
    assert side[k - 1] == "time_proj" and side[k + 1] == "time_embedding.linear_1"
    assert "time_embedding.cond_proj" not in [o.name for o in plan.ops]
    main = lambda p: [(o.name, type(o).__name__ if o.fn is None else pl.launch_key(o)) for o in p.ops]  # noqa: E731
    assert main(plan) == main(plain)
    cp, lin1 = plan.side_ops[k], plan.side_ops[k + 1]
    x, wt, bias, add16, y16, y32 = cp.keep[1:]
    assert cp.fn.name == "sfb_small_linear" and x is plan.timestep_cond_in and bias is None and y32 is None
    assert add16 is plan.side_ops[k - 1].keep[1]          # t_emb, written by time_proj
    assert lin1.keep[1] is y16 and y16 is not add16       # linear_1 reads the sum, from its own buffer
    p = cp.keep[0]
    assert (p.batch, p.n, p.k, p.act_in, p.act_out) == (b, plan.spec.block_out_channels[0], dim, 0, 0)


HAZARD_PLANS = {
    "sd15_inpaint": lambda: _unet("sd15_inpaint", 2, 64, 64),
    "sd15_lcm": lambda: _unet("sd15_lcm", 2, 64, 64),
    "sd15_inpaint_controlnet": lambda: _unet("sd15_inpaint", 2, 64, 64, controlnet=True),
    "sd15_lcm_controlnet_freeu": lambda: _unet("sd15_lcm", 1, 64, 64, controlnet=True, freeu=(True, True)),
    "sdxl_inpaint": lambda: _unet("sdxl_inpaint", 2, 128, 128, BF16),
    "sdxl_lcm": lambda: _unet("sdxl_lcm", 1, 128, 128, BF16),
    "sdxl_inpaint_controlnet": lambda: _unet("sdxl_inpaint", 2, 128, 128, BF16, controlnet=True),
}


@pytest.mark.parametrize("name", list(HAZARD_PLANS))
def test_plans_are_free_of_races_and_stale_reads(name):
    plan, rep = ph.check_plan(HAZARD_PLANS[name])
    assert not rep.findings, "\n".join(map(str, rep.findings))
    assert rep.pairs
    n_ss = sum(1 for op in plan.all_ops() if op.fn is not None and op.fn.name == "sfb_group_norm_scale_shift")
    assert len(rep.declared) == n_ss


def test_new_launches_have_keys_and_a_replay():
    plan = _unet("sd15_inpaint", 2, 64, 64)
    keys = {k for n, k, _ in pl.launches(plan) if n == "sfb_im2col_in_wide"}
    assert keys == {("sfb_im2col_in_wide", 0, 0, 2, 64, 64, 9)}
    assert pl.describe(next(iter(keys))) == "sfb_im2col_in_wide(n=2, h=64, wd=64, cin=9)"
    assert "sfb_im2col_in_wide" in pl.REPLAY and "sfb_im2col_in_wide" in ph.MODELLED


# ---- host validation of sfb_im2col_in_wide
def _wide(x=_DUMMY_PTR, a=_DUMMY_PTR, n=1, h=1, w=1, cin=9):
    return _lib.lib().sfb_im2col_in_wide(x, a, n, h, w, cin, None)


ACCEPTED = [("cin 9", dict(cin=9)), ("cin 14", dict(cin=14)), ("1x1", dict()),
            ("n*h*w = 2^31 - 1", dict(h=65537, w=32767))]
OUTSIDE = [("cin 8", dict(cin=8), "cin=8"), ("cin 15", dict(cin=15), "cin=15"), ("null x", dict(x=None), "null"),
           ("null a", dict(a=None), "null"), ("unaligned a", dict(a=_DUMMY_PTR + 8), "aligned"),
           ("n = 0", dict(n=0), "n=0"), ("h = 0", dict(h=0), "h=0"), ("w = 0", dict(w=0), "w=0"),
           ("h = -1", dict(h=-1), "h=-1"), ("n*h*w = 2^31", dict(h=65536, w=32768), "n*h*w")]


@_NO_GPU
@pytest.mark.parametrize("what,kw", ACCEPTED, ids=[a for a, _ in ACCEPTED])
def test_boundary_is_accepted(what, kw):
    rc = _wide(**kw)
    assert rc == -2, f"{what}: {_lib.lib().sfb_last_error().decode()}"


@_NO_GPU
@pytest.mark.parametrize("what,kw,word", OUTSIDE, ids=[a for a, _, _ in OUTSIDE])
def test_one_step_outside_is_refused_by_name(what, kw, word):
    rc = _wide(**kw)
    err = _lib.lib().sfb_last_error().decode()
    assert rc == -1, f"{what}: not refused (rc {rc}: {err})"
    assert word in err, f"{what}: the error does not name {word!r}: {err}"


def test_the_existing_im2col_keeps_its_range():
    # cin 8 belongs to sfb_conv_in, 9..14 to the wide im2col: sfb_im2col_in still refuses them
    for cin in (8, 9):
        assert _lib.lib().sfb_im2col_in(_DUMMY_PTR, _DUMMY_PTR, 1, 1, 1, cin, None) == -1


# ---- the runtime's handling of timestep_cond
class _FakePlan:
    built = []

    def __init__(self, weights, B, H, W, ctx_len, controlnet=False, ip_len=0, ip_seq=0, intrablock=0,
                 freeu=(False, False)):
        _FakePlan.built.append((B, H, W))
        self.intrablock_in = []
        self.sample_in, self.out = torch.zeros(B, 4, H, W), torch.zeros(B, 4, H, W)
        self.ehs_in, self.t_in = torch.zeros(B, ctx_len, 128), torch.zeros(B)
        self.timestep_cond_in = torch.full((B, 32), float("nan"), dtype=torch.float16)


class _FakeGraphed:
    def __init__(self, plan, use_graph):
        self.plan, self.steps = plan, []

    def step(self):
        self.steps.append(self.plan.timestep_cond_in.clone())


@pytest.fixture
def compiled(monkeypatch):
    monkeypatch.setattr(runtime, "require_sm90", lambda device: None)
    monkeypatch.setattr(runtime, "UNetPlan", _FakePlan)
    monkeypatch.setattr(runtime, "_GraphedPlan", _FakeGraphed)
    monkeypatch.setattr(runtime.torch.cuda, "device", lambda d: contextlib.nullcontext())
    _FakePlan.built = []
    m = lio.build_unet(tiny_lcm_config(), seed=0)
    c = runtime.CompiledUNet(m.config, m.state_dict, module=m)
    c._weights_for = lambda *a, **k: None
    c.first_call_s = 0.0

    def call(b, **kw):
        c(torch.zeros(b, 4, 16, 16, dtype=F16), 10, torch.zeros(b, 77, 128, dtype=F16), **kw)
        return c._cached
    return c, call


def test_timestep_cond_is_copied_in_and_reuses_the_plan(compiled):
    c, call = compiled
    g = torch.Generator().manual_seed(0)
    w1, w2 = torch.randn(3, 32, generator=g).half(), torch.randn(3, 32, generator=g).half()
    cache = call(3, timestep_cond=w1)
    gp = next(iter(cache.values()))
    assert torch.equal(gp.steps[-1], w1)
    cache = call(3, timestep_cond=w2)
    assert len(cache) == 1 and len(_FakePlan.built) == 1 and torch.equal(gp.steps[-1], w2)
    call(3, timestep_cond=w1[:1])                              # [1, dim]: broadcast over the batch
    assert len(cache) == 1 and torch.equal(gp.steps[-1], w1[:1].expand(3, 32))
    call(3)                                                    # None: zeros
    assert len(cache) == 1 and torch.equal(gp.steps[-1], torch.zeros(3, 32, dtype=F16))


@pytest.mark.parametrize("shape", [(2, 32), (3, 16), (3, 33), (3, 1, 32), (32,), (1, 3, 32)])
def test_a_wrong_timestep_cond_shape_is_refused(compiled, shape):
    c, call = compiled
    with pytest.raises(ValueError, match="timestep_cond"):
        call(3, timestep_cond=torch.zeros(shape, dtype=F16))
    assert not _FakePlan.built


def test_a_unet_without_cond_proj_keeps_refusing_timestep_cond():
    m = uo.build_unet(uo.tiny_config(), seed=0)
    c = runtime.CompiledUNet(m.config, m.state_dict, module=m)
    assert c._timestep_cond_input(None, 2) is None
    with pytest.raises(NotImplementedError, match="timestep_cond"):
        c(torch.zeros(1, 4, 16, 16, dtype=F16), 10, torch.zeros(1, 77, 128, dtype=F16),
          timestep_cond=torch.zeros(1, 256, dtype=F16))
