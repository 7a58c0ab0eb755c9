"""FreeU without a GPU: the closed form the kernel computes against the oracle's FFT restatement of diffusers'
fourier_filter, the UNet plans with FreeU off (unchanged) and on (one sfb_freeu per resnet of up blocks 0 and 1,
after every writer of its concat buffer and before its resnet, free of races and stale reads), the host
validation of sfb_freeu, and the runtime's reading of diffusers' FreeU attributes."""
import contextlib
import ctypes
import hashlib
import types

import pytest
import torch

import freeu_checks as fc
import plan_hazards as ph
import plan_launches as pl
from oracle import freeu_oracle as fo
from oracle import unet_oracle as uo
from sfast_b200 import _lib, runtime
from sfast_b200.plan import PackedWeights, UNetPlan, _ForkOp, _JoinOp
from sfast_b200.unet_spec import ip_adapter_geometry, param_shapes, spec_from_config
from test_host_logic import _DUMMY_PTR

_NO_GPU = pytest.mark.skipif(torch.cuda.is_available(), reason="needs a box without a GPU: launches must fail")
CFGS = {"tiny": uo.tiny_config, "sd15": uo.sd15_config, "sdxl": uo.sdxl_config}
SIZES = (1, 2, 3, 4, 5, 6, 7, 8, 12, 16, 32)
SIZES_W = (1, 2, 3, 4, 5, 8, 12, 24)


# ---- the closed form
@pytest.mark.parametrize("h", SIZES)
def test_closed_form_matches_the_fft_filter_in_float64(h):
    g = torch.Generator().manual_seed(h)
    for w in SIZES_W:
        x = torch.randn(2, 3, h, w, generator=g, dtype=torch.float64) + 0.7
        # fourier_filter's mask is fp32 (as in diffusers), so s is the fp32 value the kernel reads too
        for s in (float(torch.tensor(v, dtype=torch.float32)) for v in (0.2, 0.9, 1.6)):
            ref = fo.fourier_filter(x, threshold=1, scale=s)
            got = fc.ref_fourier_filter(x, s)
            # diffusers' filter runs the FFT of a size that is not a power of two in fp32, even for fp64 inputs
            pow2 = not (h & (h - 1) or w & (w - 1))
            assert ref.dtype == torch.float64
            assert (got - ref).abs().max().item() < (1e-12 if pow2 else 2e-6 * x.abs().max().item()), (h, w, s)


@pytest.mark.parametrize("h,w", [(3, 5), (8, 12), (16, 16), (7, 24), (1, 8), (12, 1)])
def test_closed_form_matches_the_fft_filter_for_fp32_inputs(h, w):
    x = torch.randn(2, 5, h, w, generator=torch.Generator().manual_seed(h * 100 + w)) + 0.5
    ref = fo.fourier_filter(x, threshold=1, scale=0.4)
    assert ref.dtype == torch.float32
    got = fc.ref_fourier_filter(x, 0.4)
    assert (got - ref.double()).abs().max().item() < 1e-5 * x.abs().max().item()


def test_fourier_filter_of_2x2_is_a_plain_scale_and_s_1_is_the_identity():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1, 4, 2, 2, dtype=torch.float64, generator=g)
    assert torch.allclose(fo.fourier_filter(x, 1, 0.25), 0.25 * x, atol=1e-14)
    x = torch.randn(1, 4, 8, 4, dtype=torch.float64, generator=g)
    assert torch.allclose(fo.fourier_filter(x, 1, 1.0), x, atol=1e-14)


# ---- the oracle
def test_oracle_freeu_off_is_bit_identical_and_on_changes_blocks_0_and_1_only():
    m = uo.build_unet(uo.tiny_config(), seed=3)
    g = torch.Generator().manual_seed(0)
    x, ehs = torch.randn(1, 4, 16, 16, generator=g), torch.randn(1, 77, 128, generator=g)
    with torch.no_grad():
        ref = m(x, 500, ehs).sample
        fo.enable_freeu(m, 0.9, 0.2, 1.2, 1.4)
        assert [blk.resolution_idx for blk in m.up_blocks] == [0, 1, 2, 3]
        on = m(x, 500, ehs).sample
        fo.disable_freeu(m)
        assert all(getattr(blk, k) is None for blk in m.up_blocks for k in ("s1", "s2", "b1", "b2"))
        off = m(x, 500, ehs).sample
        # blocks >= 2 never apply it: switching those on alone changes nothing
        for blk in m.up_blocks[2:]:
            blk.s1, blk.s2, blk.b1, blk.b2 = 0.9, 0.2, 1.2, 1.4
        late = m(x, 500, ehs).sample
    assert torch.equal(off, ref) and torch.equal(late, ref)
    assert (on - ref).abs().max() > 1e-3 * ref.abs().max()


def test_oracle_freeu_leaves_the_parameters_alone():
    m = uo.build_unet(uo.tiny_config(), seed=0)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    fo.enable_freeu(m, 0.9, 0.2, 1.2, 1.4)
    after = m.state_dict()
    assert list(after) == list(sd) and all(torch.equal(after[k], v) for k, v in sd.items())


# ---- dry plans
def _sd(shapes, dt):
    return {k: torch.empty(tuple(v), dtype=dt, device="meta") for k, v in shapes.items()}


def _unet(cfg, b, h, w, dt=torch.float16, ip=False, **kw):
    spec = spec_from_config(CFGS[cfg]())
    if ip:
        spec.ip = ip_adapter_geometry(spec, 64 if cfg == "tiny" else 1024)
    return UNetPlan(PackedWeights(spec, _sd(param_shapes(spec), dt), dt, "meta", dry=True), b, h, w, **kw)


def _keys(plan):
    return [(o.name, type(o).__name__ if o.fn is None else pl.launch_key(o)) for o in plan.ops + plan.side_ops]


# sha1 of the (op name, launch key) list of these plans at the commit before FreeU (whose UNetPlan had no flag)
PARENT = {
    ("tiny", 2, 32, 32): "f8a188fb61d2fc5426308a59790bd4fcc44a4707",
    ("sd15", 2, 64, 64): "f01c18fca41f7bb96b2d7c4f1c446778c496d264",
    ("sdxl", 2, 128, 128): "92681a1e9f73a2f9ef9d5697663711c7c6798941",
}


@pytest.mark.parametrize("key", list(PARENT), ids=[k[0] for k in PARENT])
def test_plan_with_freeu_off_is_the_parent_plan(key):
    cfg, b, h, w = key
    dt = torch.bfloat16 if cfg == "sdxl" else torch.float16
    base, off = _unet(cfg, b, h, w, dt), _unet(cfg, b, h, w, dt, freeu=(False, False))
    assert _keys(base) == _keys(off)
    assert hashlib.sha1(repr(_keys(off)).encode()).hexdigest() == PARENT[key]
    assert not hasattr(off, "freeu_in") and not any(o.name.endswith(".freeu") for o in off.all_ops())


FREEU_PLANS = {
    "tiny": lambda f: _unet("tiny", 2, 32, 32, freeu=f),
    "tiny_8x8": lambda f: _unet("tiny", 1, 8, 8, freeu=f),
    "sd15": lambda f: _unet("sd15", 2, 64, 64, freeu=f),
    "sd15_64x96": lambda f: _unet("sd15", 2, 64, 96, freeu=f),
    "sdxl": lambda f: _unet("sdxl", 2, 128, 128, torch.bfloat16, freeu=f),
    "sd15_controlnet_t2i_ip": lambda f: _unet("sd15", 2, 64, 64, ip=True, ip_len=4, controlnet=True, intrablock=4,
                                               freeu=f),
}


def _linear(plan):
    """Main-stream launches in issue order, forked branches where they are issued."""
    out = []
    for op in plan.ops:
        if isinstance(op, _ForkOp):
            out.extend(op.branch)
        elif not isinstance(op, _JoinOp):
            out.append(op)
    return out


@pytest.mark.parametrize("name", list(FREEU_PLANS))
@pytest.mark.parametrize("flags", [(True, True), (True, False), (False, True)], ids=["both", "block0", "block1"])
def test_each_freeu_sits_between_the_last_writer_and_the_resnet(name, flags):
    plan, space = ph.build(lambda: FREEU_PLANS[name](flags))
    spec = plan.spec
    want = [r.prefix + ".freeu" for i in (0, 1) if flags[i] for r in spec.up[i].resnets]
    with ph.virtual_addresses_of(space):
        ops = _linear(plan)
        fu = [k for k, o in enumerate(ops) if o.fn is not None and o.fn.name == "sfb_freeu"]
        assert [ops[k].name for k in fu] == want
        for k in fu:
            p = ops[k].keep[0]
            i = int(ops[k].name.split(".")[1])
            regions = [a for a in ph.accesses(ops[k]) if a.field.startswith("x.")]
            touch = [(j, a) for j, o in enumerate(ops) if j != k and o.fn is not None
                     for a in ph.accesses(o) if any(ph.overlap(a, r) for r in regions)]
            last_w = max(j for j, a in touch if a.writes)
            first_r = min(j for j, a in touch if a.reads and j > last_w)
            assert last_w < k < first_r, (ops[k].name, ops[last_w].name, ops[first_r].name)
            assert ops[first_r].name.startswith(ops[k].name[:-len("freeu")] + "norm1"), ops[first_r].name
            prod = ops[last_w]
            if prod.fn.name == "sfb_gemm":  # the producer finished its own split-K reduction
                assert prod.keep[0].defer_finish == 0
            assert p.c_hidden + p.c_skip == p.ld == spec.up[i].resnets[int(ops[k].name.split(".")[3])].cin
            assert all(j < k for j, a in touch if a.writes)
    assert len(fu) == (6 if flags == (True, True) else 3)


@pytest.mark.parametrize("name", list(FREEU_PLANS))
def test_freeu_plans_are_free_of_races_and_stale_reads(name):
    plan, rep = ph.check_plan(lambda: FREEU_PLANS[name]((True, True)))
    assert not rep.findings, "\n".join(map(str, rep.findings))
    n_ss = sum(1 for op in plan.all_ops() if op.fn is not None and op.fn.name == "sfb_group_norm_scale_shift")
    assert len(rep.declared) == n_ss


def test_freeu_values_are_one_static_input_per_block():
    plan = _unet("sd15", 2, 64, 64, freeu=(True, True))
    assert tuple(plan.freeu_in.shape) == (4,) and plan.freeu_in.dtype == torch.float32
    fu = [o for o in plan.all_ops() if o.fn is not None and o.fn.name == "sfb_freeu"]
    # block 0 reads (b1, s1) at byte 0 of freeu_in, block 1 (b2, s2) at byte 8 (dry buffers sit at address 0)
    assert [ph._p(o.keep[0].bs) for o in fu] == [0] * 3 + [8] * 3


def test_freeu_flags_are_validated():
    with pytest.raises(ValueError, match="one flag"):
        _unet("tiny", 1, 32, 32, freeu=(True,))


# ---- host validation of sfb_freeu
def _freeu(**kw):
    p = _lib.FreeUParams()
    p.x, p.bs = _DUMMY_PTR, _DUMMY_PTR
    p.n, p.h, p.w, p.c_hidden, p.c_skip, p.ld, p.dtype = 1, 1, 1, 8, 8, 16, _lib.SFB_F16
    for k, v in kw.items():
        setattr(p, k, v)
    return _lib.lib().sfb_freeu(ctypes.byref(p), None)


ACCEPTED = [
    ("smallest", dict()),
    ("ld = c_hidden + c_skip", dict(c_hidden=1280, c_skip=640, ld=1920)),
    ("pitch gap", dict(c_hidden=8, c_skip=16, ld=32)),
    ("bf16", dict(dtype=_lib.SFB_BF16)),
    ("h*w = 2^31 - 1", dict(h=65537, w=32767)),
]
OUTSIDE = [
    ("null x", dict(x=None), "null"),
    ("null bs", dict(bs=None), "null"),
    ("unaligned x", dict(x=_DUMMY_PTR + 8), "aligned"),
    ("n = 0", dict(n=0), "n=0"),
    ("h = 0", dict(h=0), "h=0"),
    ("w = 0", dict(w=0), "w=0"),
    ("h*w = 2^31", dict(h=65536, w=32768), "h*w"),
    ("c_hidden = 0", dict(c_hidden=0), "c_hidden=0"),
    ("c_hidden not a multiple of 8", dict(c_hidden=12, ld=24), "c_hidden=12"),
    ("c_skip = 0", dict(c_skip=0), "c_skip=0"),
    ("c_skip not a multiple of 8", dict(c_skip=4, ld=16), "c_skip=4"),
    ("ld not a multiple of 8", dict(ld=20), "ld=20"),
    ("ld = c_hidden + c_skip - 8", dict(c_hidden=16, c_skip=16, ld=24), "ld=24"),
    ("dtype fp32", dict(dtype=_lib.SFB_F32), "dtype"),
]


@_NO_GPU
@pytest.mark.parametrize("what,kw", ACCEPTED, ids=[a for a, _ in ACCEPTED])
def test_boundary_is_accepted(what, kw):
    rc = _freeu(**kw)
    assert rc == -2, f"{what}: {_lib.lib().sfb_last_error().decode()}"


@_NO_GPU
@pytest.mark.parametrize("what,kw,word", OUTSIDE, ids=[a for a, _, _ in OUTSIDE])
def test_one_step_outside_is_refused_by_name(what, kw, word):
    rc = _freeu(**kw)
    err = _lib.lib().sfb_last_error().decode()
    assert rc == -1, f"{what}: not refused (rc {rc}: {err})"
    assert word in err, f"{what}: the error does not name {word!r}: {err}"


# ---- the runtime's reading of diffusers' FreeU state
class _FakePlan:
    built = []

    def __init__(self, weights, B, H, W, ctx_len, controlnet=False, ip_len=0, ip_seq=0, intrablock=0,
                 freeu=(False, False)):
        _FakePlan.built.append(freeu)
        self.freeu = freeu
        self.intrablock_in = []
        self.sample_in, self.out = torch.zeros(B, 4, H, W), torch.zeros(B, 4, H, W)
        self.ehs_in, self.t_in = torch.zeros(B, ctx_len, 128), torch.zeros(B)
        if any(freeu):
            self.freeu_in = torch.zeros(4)


class _FakeGraphed:
    def __init__(self, plan, use_graph):
        self.plan, self.steps = plan, []

    def step(self):
        self.steps.append(self.plan.freeu_in.tolist() if hasattr(self.plan, "freeu_in") else None)


@pytest.fixture
def compiled(monkeypatch):
    monkeypatch.setattr(runtime, "require_sm90", lambda device: None)
    monkeypatch.setattr(runtime, "UNetPlan", _FakePlan)
    monkeypatch.setattr(runtime, "_GraphedPlan", _FakeGraphed)
    monkeypatch.setattr(runtime.torch.cuda, "device", lambda d: contextlib.nullcontext())
    _FakePlan.built = []
    m = uo.build_unet(uo.tiny_config(), seed=0)
    c = runtime.CompiledUNet(m.config, m.state_dict, module=m)
    c._weights_for = lambda *a, **k: None
    c.first_call_s = 0.0  # no first-call timing (it synchronises the device)

    def call():
        c(torch.zeros(1, 4, 16, 16, dtype=torch.float16), 10, torch.zeros(1, 77, 128, dtype=torch.float16))
        return c._cached
    return m, c, call


def _last(cache):
    return next(reversed(cache.values())).steps[-1]


def test_runtime_follows_the_truthiness_rule_per_block(compiled):
    m, c, call = compiled
    assert c._freeu_state() == ((False, False), None)
    fo.enable_freeu(m, 0.9, 0.2, 1.2, 1.4)
    assert c._freeu_state() == ((True, True), [1.2, 0.9, 1.4, 0.2])
    m.up_blocks[0].s2 = 0.0  # a zero switches that block off, whichever value it is
    assert c._freeu_state() == ((False, True), [0.0, 0.0, 1.4, 0.2])
    m.up_blocks[1].b1 = None
    assert c._freeu_state() == ((False, False), None)
    fo.disable_freeu(m)
    for blk in m.up_blocks[2:]:  # later blocks do nothing
        blk.s1, blk.s2, blk.b1, blk.b2 = 0.9, 0.2, 1.2, 1.4
    assert c._freeu_state() == ((False, False), None)
    # each block uses its own values: block 0 its b1 / s1, block 1 its b2 / s2
    m.up_blocks[0].s1, m.up_blocks[0].s2, m.up_blocks[0].b1, m.up_blocks[0].b2 = 0.5, 7.0, 1.5, 9.0
    m.up_blocks[1].s1, m.up_blocks[1].s2, m.up_blocks[1].b1, m.up_blocks[1].b2 = 8.0, 0.25, 6.0, 1.25
    assert c._freeu_state() == ((True, True), [1.5, 0.5, 1.25, 0.25])


def test_value_changes_reuse_the_plan_and_toggling_adds_one_key(compiled):
    m, c, call = compiled
    cache = call()
    assert len(cache) == 1 and _FakePlan.built == [(False, False)]
    fo.enable_freeu(m, 0.9, 0.2, 1.2, 1.4)
    cache = call()
    assert len(cache) == 2 and _FakePlan.built[-1] == (True, True)
    assert _last(cache) == pytest.approx([1.2, 0.9, 1.4, 0.2])
    fo.enable_freeu(m, 0.6, 0.4, 1.1, 1.2)
    cache = call()
    assert len(cache) == 2 and len(_FakePlan.built) == 2
    assert _last(cache) == pytest.approx([1.1, 0.6, 1.2, 0.4])
    fo.disable_freeu(m)
    cache = call()
    assert len(cache) == 2 and len(_FakePlan.built) == 2
    m.up_blocks[1].b2 = 0  # block 0 only
    fo.enable_freeu(m, 0.9, 0.2, 1.2, 1.4)
    m.up_blocks[1].b2 = 0
    cache = call()
    assert len(cache) == 3 and _FakePlan.built[-1] == (True, False)
    assert _last(cache) == pytest.approx([1.2, 0.9, 0.0, 0.0])


def test_preserve_parameters_off_still_reads_freeu_on_every_call(compiled, monkeypatch):
    m, c, call = compiled
    c.preserve_parameters = False
    fo.enable_freeu(m, 0.9, 0.2, 1.2, 1.4)
    call()
    fo.enable_freeu(m, 0.6, 0.4, 1.1, 1.2)
    assert _last(call()) == pytest.approx([1.1, 0.6, 1.2, 0.4])


def test_config_only_and_svd_unets_ignore_the_attributes():
    m = uo.build_unet(uo.tiny_config(), seed=0)
    fo.enable_freeu(m, 0.9, 0.2, 1.2, 1.4)
    c = runtime.CompiledUNet(m.config, m.state_dict)
    assert c._freeu_state() == ((False, False), None)
    from oracle import svd_oracle as so
    svd = types.SimpleNamespace(config=so.svd_tiny_config())
    cs = runtime.CompiledUNet(svd.config, lambda: {})
    assert cs.spec.temporal
    calls = []
    cs._freeu_state = lambda: calls.append(1)
    cs._call_svd = lambda *a, **k: "svd"
    assert cs(None, 1, None) == "svd" and not calls
