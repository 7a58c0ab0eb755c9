"""Host-side checks of the native T2I-Adapter: the oracle's parameter layout against the spec, the refusals, the
dry adapter plans and the C ABI's validation of every launch, the boundaries of the two new entry points and of
the GEMM's ReLU epilogue, where the UNet adds the adapter residuals, and compile()'s routing."""
import ctypes
import logging

import pytest
import torch

import abi_sweep as sw
from oracle import t2i_adapter_oracle as to
from oracle import unet_oracle as uo
from sfast_b200 import _lib, ops
from sfast_b200.plan import PackedWeights, UNetPlan, _ForkOp, _JoinOp, intrablock_shapes
from sfast_b200.t2i_adapter_plan import AdapterPlan, t2i_adapter_param_shapes, t2i_adapter_spec_from_config
from sfast_b200.unet_spec import param_shapes, spec_from_config
from test_abi_sweep_cpu import _call
from test_host_logic import _DUMMY_PTR, _clone, _validate_plan_on_cpu

_NO_GPU = pytest.mark.skipif(torch.cuda.is_available(), reason="needs a box without a GPU: launches must fail")
F16 = _lib.SFB_F16


def _dry_adapter(cfg, b, h, w, dt=torch.float16):
    spec = t2i_adapter_spec_from_config(cfg)
    sd = {k: torch.empty(v, dtype=dt, device="meta") for k, v in t2i_adapter_param_shapes(spec).items()}
    return AdapterPlan(PackedWeights(spec, sd, dt, "meta", dry=True), b, h, w)


def _dry_unet(cfgf, b, h, w, **kw):
    spec = spec_from_config(cfgf())
    sd = {k: torch.empty(v, dtype=torch.float16, device="meta") for k, v in param_shapes(spec).items()}
    return UNetPlan(PackedWeights(spec, sd, torch.float16, "meta", dry=True), b, h, w, **kw)


@pytest.mark.parametrize("cfg,total", [(to.sd_config(), 77_369_280), (to.sd_config(in_channels=1), 77_000_640),
                                       (to.sdxl_config(), 79_028_160)], ids=["sd_3ch", "sd_1ch", "xl_3ch"])
def test_oracle_parameters_match_the_spec_and_totals_are_pinned(cfg, total):
    with torch.device("meta"):
        m = to.T2IAdapter(cfg)
    spec = t2i_adapter_spec_from_config(cfg)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == t2i_adapter_param_shapes(spec)
    assert sum(v.numel() for v in m.state_dict().values()) == total
    assert spec.total_downscale_factor == m.total_downscale_factor == (64 if cfg.adapter_type == "full_adapter" else 32)


@pytest.mark.parametrize("cfg,key", [
    (to.sd_config(adapter_type="light_adapter", channels=(320, 640, 1280)), "adapter_type"),
    (to.sd_config(channels=(320, 640, 1280, 1248)), "channels"),
    (to.sd_config(in_channels=1, downscale_factor=4), "in_channels"),
    (to.sd_config(num_res_blocks=0), "num_res_blocks"),
], ids=["light_adapter", "channels", "in_channels", "num_res_blocks"])
def test_unsupported_configs_are_refused_by_name(cfg, key):
    with pytest.raises(NotImplementedError, match=key):
        t2i_adapter_spec_from_config(cfg)


def test_image_size_and_dtype_are_refused_by_name():
    with pytest.raises(NotImplementedError, match="total_downscale_factor 64"):
        _dry_adapter(to.sd_config(), 1, 512, 544)
    with pytest.raises(NotImplementedError, match="total_downscale_factor 32"):
        _dry_adapter(to.sdxl_config(), 1, 1040, 1024)
    from sfast_b200.runtime import CompiledT2IAdapter
    c = CompiledT2IAdapter(to.sd_config(), lambda: {})
    with pytest.raises(NotImplementedError, match="dtype torch.float32"):
        c(torch.zeros(1, 3, 512, 512))
    with pytest.raises(NotImplementedError, match="total_downscale_factor"):
        c(torch.zeros(1, 3, 512, 520, dtype=torch.float16))
    with pytest.raises(ValueError, match=r"\[B, 3, H, W\]"):
        c(torch.zeros(1, 1, 512, 512, dtype=torch.float16))


def _validate_adapter_plan(plan):
    """_validate_plan_on_cpu for the GEMMs, plus the adapter's own entry points with dummy pointers."""
    n = _validate_plan_on_cpu(plan)
    lib = _lib.lib()
    for op in plan.all_ops():
        name = op.fn.name
        if name in ("sfb_pixel_unshuffle", "sfb_avg_pool2x2"):
            rc = getattr(lib, name)(_DUMMY_PTR, _DUMMY_PTR, *op.args[2:], None)
        elif name == "sfb_nhwc_to_nchw_scaled":
            prm = _clone(op.keep[0])
            prm.scale = _DUMMY_PTR
            for it in prm.items[:prm.count]:
                it.src, it.dst = _DUMMY_PTR, _DUMMY_PTR
            rc = lib.sfb_nhwc_to_nchw_scaled(ctypes.byref(prm), None)
        else:
            continue
        assert rc == -2, f"{op.name}: {lib.sfb_last_error().decode()}"
        n[name] += 1
    return n


@_NO_GPU
@pytest.mark.parametrize("xl,b,h,w", [(False, 1, 512, 512), (False, 2, 512, 512), (False, 1, 768, 768),
                                      (False, 2, 512, 768), (True, 1, 1024, 1024), (True, 2, 1024, 1024)])
def test_dry_adapter_plans_pass_host_validation(xl, b, h, w):
    cfg = to.sdxl_config() if xl else to.sd_config()
    plan = _dry_adapter(cfg, b, h, w)
    n = _validate_adapter_plan(plan)
    blocks = t2i_adapter_spec_from_config(cfg).blocks()
    # conv_in + per block: (in_conv) + 2 x (block1, block2)
    assert n["sfb_gemm"] == 1 + sum(cin != cout for _, cin, cout in blocks) + 4 * len(blocks)
    assert n["sfb_pixel_unshuffle"] == 1 and n["sfb_nhwc_to_nchw_scaled"] == 1
    assert n["sfb_avg_pool2x2"] == sum(p for p, _, _ in blocks)
    relu = [op for op in plan.all_ops() if op.fn.name == "sfb_gemm" and op.keep[0].act]
    assert len(relu) == 2 * len(blocks) and all(op.keep[0].act == _lib.ACT_RELU and op.keep[0].splits == 1
                                                 for op in relu)
    r = 16 if xl else 8
    want = [(b, 320, h // r, w // r), (b, 640, h // (r * (1 if xl else 2)), w // (r * (1 if xl else 2))),
            (b, 1280, h // (2 * r) if xl else h // (4 * r), w // (2 * r) if xl else w // (4 * r))]
    want.append((b, 1280) + (want[2][2:] if xl else (h // (8 * r), w // (8 * r))))
    assert [tuple(f.shape) for f in plan.features_out] == want


# ---- boundaries of the new entry points and of act = SFB_ACT_RELU, in the style of tests/abi_sweep.py
def _unshuffle(n=1, c=3, h=16, w=16, r=8, ldy=None):
    return _lib.lib().sfb_pixel_unshuffle(_DUMMY_PTR, _DUMMY_PTR, n, c, h, w, r, c * r * r if ldy is None else ldy,
                                          None)


def _pool(n=1, h=2, w=2, c=8, ldx=None, ldy=None, dtype=F16, x=_DUMMY_PTR):
    return _lib.lib().sfb_avg_pool2x2(x, _DUMMY_PTR, n, h, w, c, c if ldx is None else ldx, c if ldy is None else ldy,
                                      dtype, None)


ACCEPTED = [
    ("unshuffle r=1 1x1", lambda: _unshuffle(c=1, h=1, w=1, r=1)),
    ("unshuffle r=16 one output pixel", lambda: _unshuffle(c=3, h=16, w=16, r=16)),
    ("unshuffle ldy = c*r*r + 1", lambda: _unshuffle(ldy=3 * 64 + 1)),
    ("unshuffle 1x2 output pixels", lambda: _unshuffle(h=8, w=16)),
    ("pool 2x2 -> 1x1, c=8", lambda: _pool()),
    ("pool ldx = ldy = c + 8", lambda: _pool(c=8, ldx=16, ldy=16, n=3, h=4, w=6)),
    ("pool bf16", lambda: _pool(dtype=_lib.SFB_BF16, h=2, w=64, c=1280)),
]
for _m, _n in ((1, 8), (127, 152), (128, 160), (129, 168)):
    ACCEPTED.append((f"gemm relu M={_m} N={_n}", lambda m=_m, n=_n: _call(sw.gemm_op(m, n, 64, sw.F16, act=4))[0]))
ACCEPTED.append(("gemm relu residual ldo", lambda: _call(sw.gemm_op(129, 168, 320, sw.BF16, act=4, residual=True,
                                                                    ldr=176, ldo=176))[0]))

OUTSIDE = [
    ("unshuffle r=0", lambda: _unshuffle(r=0), "r=0"),
    ("unshuffle h not a multiple of r", lambda: _unshuffle(h=12), "h=12"),
    ("unshuffle w not a multiple of r", lambda: _unshuffle(w=20), "w=20"),
    ("unshuffle ldy = c*r*r - 1", lambda: _unshuffle(ldy=3 * 64 - 1), "ldy"),
    ("unshuffle c=0", lambda: _unshuffle(c=0), "c=0"),
    ("pool odd h", lambda: _pool(h=3), "h=3"),
    ("pool odd w", lambda: _pool(w=1), "w=1"),
    ("pool c not a multiple of 8", lambda: _pool(c=12), "c=12"),
    ("pool ldx < c", lambda: _pool(c=16, ldx=8), "ldx=8"),
    ("pool ldy not a multiple of 8", lambda: _pool(ldy=12), "ldy=12"),
    ("pool dtype fp32", lambda: _pool(dtype=_lib.SFB_F32), "dtype"),
    ("pool unaligned x", lambda: _pool(x=_DUMMY_PTR + 2), "aligned"),
]


@_NO_GPU
@pytest.mark.parametrize("what,fn", ACCEPTED, ids=[a for a, _ in ACCEPTED])
def test_boundary_is_accepted(what, fn):
    rc = fn()
    assert rc == -2, f"{what}: {_lib.lib().sfb_last_error().decode()}"


@_NO_GPU
@pytest.mark.parametrize("what,fn,word", OUTSIDE, ids=[a for a, _, _ in OUTSIDE])
def test_one_step_outside_is_refused_by_name(what, fn, word):
    rc = fn()
    err = _lib.lib().sfb_last_error().decode()
    assert rc == -1, f"{what}: not refused (rc {rc}: {err})"
    assert word in err, f"{what}: the error does not name {word!r}: {err}"


@_NO_GPU
@pytest.mark.parametrize("what,build,word", [
    ("relu + 1", lambda: sw.gemm_op(128, 160, 64, sw.F16, act=5), "activation 5"),
    ("relu with split-K", lambda: sw.gemm_op(129, 168, 128, sw.F16, act=4, splits=2), "act"),
], ids=["act5", "relu_splitk"])
def test_gemm_relu_one_step_outside_is_refused(what, build, word):
    rc, err = _call(build())
    assert rc == -1 and word in err, (what, rc, err)


# ---- the UNet side
@pytest.mark.parametrize("cfgf,b,h,w,n_ops", [(uo.sd15_config, 2, 64, 64, 326), (uo.sdxl_config, 2, 128, 128, 773)],
                         ids=["sd15", "sdxl"])
def test_unet_plan_without_residuals_is_unchanged(cfgf, b, h, w, n_ops):
    import plan_launches as pl
    base, zero = _dry_unet(cfgf, b, h, w), _dry_unet(cfgf, b, h, w, intrablock=0)

    def keys(p):
        return [(o.name, type(o).__name__ if o.fn is None else pl.launch_key(o)) for o in p.ops + p.side_ops]
    assert keys(base) == keys(zero) and len(base.ops) + len(base.side_ops) == n_ops
    assert base.intrablock_in == [] and not any(o.name.startswith("t2i_adapter") for o in base.all_ops())


def _gemm_out_buf(op):
    return op.keep[9][1] if op.fn is not None and op.fn.name == "sfb_gemm" else None


@pytest.mark.parametrize("cfgf,h,n,readers", [
    (uo.sd15_config, 64, 5, ["down_blocks.0.downsamplers.0.conv", "down_blocks.1.downsamplers.0.conv",
                             "down_blocks.2.downsamplers.0.conv", "mid_block.resnets.0.norm1",
                             "controlnet.residuals"]),
    (uo.sdxl_config, 128, 4, ["down_blocks.1.resnets.0.norm1", "down_blocks.1.downsamplers.0.conv",
                              "mid_block.resnets.0.norm1", "controlnet.residuals"]),
], ids=["sd15", "sdxl"])
def test_each_residual_add_sits_between_its_producer_and_the_first_reader(cfgf, h, n, readers):
    plan = _dry_unet(cfgf, 2, h, h, intrablock=n, controlnet=True)
    main = [o for o in plan.ops if not isinstance(o, (_ForkOp, _JoinOp))]
    adds = [i for i, o in enumerate(main) if o.name.startswith("t2i_adapter.residual.")]
    assert [main[i].name for i in adds] == [f"t2i_adapter.residual.{k}" for k in range(n)]
    shapes = intrablock_shapes(plan.spec, 2, h, h)
    for k, i in enumerate(adds):
        p = main[i].keep[0]
        assert p.count == 1 and (p.items[0].n, p.items[0].c, p.items[0].hw) == (
            shapes[k][0], shapes[k][1], shapes[k][2] * shapes[k][3])
        assert tuple(plan.intrablock_in[k].shape) == shapes[k]
        prod = main[i - 1]
        # the producer wrote the tensor and finished its own split-K reduction (no GroupNorm finishes it later)
        assert _gemm_out_buf(prod) is main[i].keep[2][0] and prod.keep[0].defer_finish == 0
        assert main[i + 1].name.startswith(readers[k])
    # the mid residual is added before the ControlNet residuals, and without them the up path reads it next
    plain = [o for o in _dry_unet(cfgf, 2, h, h, intrablock=n).ops if not isinstance(o, (_ForkOp, _JoinOp))]
    i = [o.name for o in plain].index(f"t2i_adapter.residual.{n - 1}")
    assert plain[i + 1].name.startswith("up_blocks.0.resnets.0.norm1")


def test_insertion_points_match_the_adapter_features():
    sd = _dry_adapter(to.sd_config(), 2, 512, 512)
    assert intrablock_shapes(spec_from_config(uo.sd15_config()), 2, 64, 64)[:4] == \
        [tuple(f.shape) for f in sd.features_out]
    xl = _dry_adapter(to.sdxl_config(), 2, 1024, 1024)
    pts = intrablock_shapes(spec_from_config(uo.sdxl_config()), 2, 128, 128)
    assert pts == [tuple(f.shape) for f in xl.features_out]  # the 4th feature is the mid-block residual


# ---- compile() routing on stand-in pipelines
class T2IAdapter:
    """The attributes compile_adapter reads of a diffusers T2IAdapter."""

    def __init__(self, cfg):
        self.config = cfg
        self.device = torch.device("cuda")

    def state_dict(self):
        return {}

    def forward(self, *a, **k):
        return "eager"

    @property
    def total_downscale_factor(self):
        return 64


class MultiAdapter:
    def __init__(self, adapters):
        self.adapters = adapters


class LightAdapter(T2IAdapter):
    pass


class _Pipe:
    def __init__(self, adapter):
        self.unet = "unet"
        self.adapter = adapter


@pytest.fixture
def routing(monkeypatch):
    from sfast.compilers import diffusion_pipeline_compiler as dpc
    from sfast_b200 import runtime
    monkeypatch.setattr(runtime, "require_sm90", lambda device: None)
    monkeypatch.setattr(dpc, "compile_unet", lambda m, config: m)
    return dpc, dpc.CompilationConfig.Default()


def test_compile_replaces_forward_of_a_single_adapter(routing):
    dpc, cfg = routing
    a = T2IAdapter(to.sdxl_config())
    pipe = dpc.compile(_Pipe(a), cfg)
    assert pipe.adapter is a and a.forward._compiled.spec.adapter_type == "full_adapter_xl"
    assert a.forward._cached == {} and a.total_downscale_factor == 64
    assert dpc.compile_adapter is not None


def test_compile_replaces_forward_of_every_adapter_of_a_multi_adapter(routing, caplog):
    dpc, cfg = routing
    nets = [T2IAdapter(to.sd_config()), T2IAdapter(to.sd_config(in_channels=1)),
            T2IAdapter(to.sd_config(adapter_type="light_adapter")), LightAdapter(to.sd_config())]
    multi = MultiAdapter(nets)
    with caplog.at_level(logging.WARNING):
        assert dpc.compile(_Pipe(multi), cfg).adapter is multi
    assert nets[0].forward._compiled is not None and nets[1].forward._compiled.spec.in_channels == 1
    assert nets[2].forward() == "eager" and nets[3].forward() == "eager"
    assert "adapter_type='light_adapter'" in caplog.text and "LightAdapter is not a T2IAdapter" in caplog.text


def test_compile_leaves_an_unsupported_adapter_eager_with_one_warning(routing, caplog):
    dpc, cfg = routing
    a = T2IAdapter(to.sd_config(channels=(320, 640, 1280, 1300)))
    with caplog.at_level(logging.WARNING):
        dpc.compile(_Pipe(a), cfg)
    assert a.forward() == "eager"
    assert [r.getMessage() for r in caplog.records if "T2I-Adapter" in r.getMessage()] == [
        "sfast (H100 build): T2I-Adapter left on its eager path (T2IAdapter config channels=(320, 640, 1280, 1300): "
        "the H100 path needs multiples of 64)"]


def test_compile_without_an_adapter(routing):
    dpc, cfg = routing
    assert dpc.compile(_Pipe(None), cfg).adapter is None


def test_oracle_unet_forward_legacy_form_agrees_and_matches_the_oracle_unet_without_residuals():
    cfg = uo.tiny_config()
    m = uo.build_unet(cfg, seed=3)
    g = torch.Generator().manual_seed(0)
    s, e, t = torch.randn(1, 4, 32, 32, generator=g), torch.randn(1, 77, cfg.cross_attention_dim, generator=g), 10
    res = [torch.randn(s_, generator=g) for s_ in intrablock_shapes(spec_from_config(cfg), 1, 32, 32)]
    keep = list(res)
    with torch.no_grad():
        a = to.unet_forward(m, s, t, e, down_intrablock_additional_residuals=res).sample
        b = to.unet_forward(m, s, t, e, down_block_additional_residuals=res).sample
        plain = to.unet_forward(m, s, t, e).sample
        ref = m(s, t, e).sample
        zero = to.unet_forward(m, s, t, e, down_intrablock_additional_residuals=[torch.zeros_like(r) for r in res]).sample
    assert res == keep and torch.equal(a, b) and not torch.equal(a, plain)
    # without residuals (or with zero ones) the restatement computes what the oracle UNet computes
    assert torch.equal(plain, ref) and torch.equal(zero, ref)
