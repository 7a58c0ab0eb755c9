"""Host-side checks of the native ControlNet: the oracle's parameter layout against the spec, the dry launch
schedules and the C ABI's validation of their launches, the guess-mode factors, float64 references of the two
new kernels against independent forms, the new parameter structs' layout, and compile()'s routing."""
import ctypes
import logging
import os
import subprocess

import pytest
import torch
import torch.nn.functional as F

from oracle import controlnet_oracle as co
from sfast_b200 import _lib, ops
from sfast_b200.controlnet_plan import ControlNetPlan, residual_scales, stored_channels
from sfast_b200.plan import PackedWeights
from sfast_b200.unet_spec import controlnet_spec_from_config, param_shapes, random_state_dict
from test_host_logic import _DUMMY_PTR, _clone, _nonnull, _validate_plan_on_cpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_NO_GPU = pytest.mark.skipif(torch.cuda.is_available(), reason="needs a box without a GPU: launches must fail")


def _dry(cfg, b, h, w, dt=torch.float16):
    spec = controlnet_spec_from_config(cfg)
    sd = {k: torch.empty(v, dtype=dt, device="meta") for k, v in param_shapes(spec).items()}
    return ControlNetPlan(PackedWeights(spec, sd, dt, "meta", dry=True), b, h, w)


def _names(plan):
    return [op.fn.name for op in plan.all_ops() if op.fn is not None]


@pytest.mark.parametrize("cfgf,total", [(co.sd15_config, 361_279_120), (co.sdxl_config, 1_251_014_160),
                                        (co.tiny_config, 14_879_632)])
def test_oracle_parameters_match_the_spec_and_totals_are_pinned(cfgf, total):
    cfg = cfgf()
    with torch.device("meta"):
        m = co.ControlNetModel(cfg)
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    spec = controlnet_spec_from_config(cfg)
    assert got == {k: tuple(v) for k, v in param_shapes(spec).items()}
    assert sum(v.numel() for v in m.state_dict().values()) == total
    assert spec.up == [] and len(spec.residual_channels()) == (12 if cfgf is not co.sdxl_config else 9)


def test_random_state_dict_loads_into_the_oracle():
    spec = controlnet_spec_from_config(co.tiny_config())
    m = co.ControlNetModel(co.tiny_config())
    m.load_state_dict({k: v.float() for k, v in random_state_dict(spec, seed=1).items()})


@pytest.mark.parametrize("cfgf,b,h,w", [(co.sd15_config, 2, 64, 64), (co.sdxl_config, 2, 128, 128),
                                        (co.tiny_config, 2, 32, 32), (co.sd15_config, 1, 64, 96)])
def test_dry_plans_pass_host_validation(cfgf, b, h, w):
    plan = _dry(cfgf(), b, h, w)
    names = _names(plan)
    spec = plan.spec
    n_res = len(spec.residual_channels())
    assert names.count("sfb_nhwc_to_nchw_scaled") == 1 and names.count("sfb_conv3x3_small") == 5
    assert len(plan.down_out) == n_res and tuple(plan.cond_in.shape) == (b, 3, 8 * h, 8 * w)
    zc = [op for op in plan.all_ops() if op.name.startswith(("controlnet_down_blocks.", "controlnet_mid_block"))]
    assert len(zc) == n_res + 1 and all(op.fn.name == "sfb_gemm" and op.keep[0].a_mode == _lib.A_MATRIX for op in zc)
    silu = [op.keep[0] for op in plan.all_ops() if op.fn is not None and op.fn.name == "sfb_gemm"
            and op.keep[0].act == _lib.ACT_SILU]
    # 96 -> 96 and 96 -> 256 / s2 on the wgmma conv, 96 channels stored as 128
    assert [(g.cin, g.N, g.conv_stride) for g in silu] == [(128, 128, 1), (128, 256, 2)]
    assert all(g.splits == 1 for g in silu)
    if (cfgf, b, h, w) == (co.sd15_config, 2, 64, 64):
        # 13 zero-conv GEMMs and one gather
        assert len(zc) == 13 and names.count("sfb_nhwc_to_nchw_scaled") == 1
        print("SD-1.5 ControlNet 2x64x64: %.3f TFLOP, %d launches" % (plan.flops() / 1e12, len(names)))
    if torch.cuda.is_available():
        return
    n = _validate_plan_on_cpu(plan)
    assert n["sfb_gemm"] == names.count("sfb_gemm")
    lib = _lib.lib()
    for op in plan.all_ops():
        if op.fn is None or op.fn.name not in ("sfb_conv3x3_small", "sfb_nhwc_to_nchw_scaled"):
            continue
        p = _clone(op.keep[0])
        if op.fn.name == "sfb_conv3x3_small":
            _nonnull(p, ["x", "weight", "bias", "y"])
            rc = lib.sfb_conv3x3_small(ctypes.byref(p), None)
        else:
            _nonnull(p, ["scale"])
            for it in p.items[:p.count]:
                _nonnull(it, ["src", "dst"])
            rc = lib.sfb_nhwc_to_nchw_scaled(ctypes.byref(p), None)
        assert rc == -2, f"{op.name}: {lib.sfb_last_error().decode()}"


def test_unet_emitters_are_shared_not_copied():
    """The ControlNet's time embedding, conv_in and down / mid blocks are the UNet's launches: the same
    GEMM geometry as the UNet plan's down path at the same size."""
    from oracle import unet_oracle as uo
    from sfast_b200.plan import UNetPlan
    from sfast_b200.unet_spec import spec_from_config
    spec = spec_from_config(uo.tiny_config())
    sd = {k: torch.empty(v, dtype=torch.float16, device="meta") for k, v in param_shapes(spec).items()}
    unet = UNetPlan(PackedWeights(spec, sd, torch.float16, "meta", dry=True), 2, 32, 32)
    cn = _dry(co.tiny_config(), 2, 32, 32)

    def geo(plan, prefix):
        return [(o.name, o.keep[0].M, o.keep[0].N, o.keep[0].K) for o in plan.all_ops()
                if o.fn is not None and o.fn.name == "sfb_gemm" and o.name.startswith(prefix)]
    for prefix in ("down_blocks.", "mid_block.", "conv_in"):
        assert geo(cn, prefix) == geo(unet, prefix), prefix


@pytest.mark.parametrize("n_down,scale", [(12, 1.0), (12, 0.55), (9, 2.0)])
def test_guess_mode_factors_equal_diffusers_logspace(n_down, scale):
    got = residual_scales(n_down, scale, guess_mode=True)
    assert got.dtype == torch.float32 and torch.equal(got, torch.logspace(-1, 0, n_down + 1) * scale)
    assert torch.equal(got, co.guess_mode_scales(n_down, scale, True))
    assert torch.equal(residual_scales(n_down, scale, False), torch.full((n_down + 1,), scale))


def conv_small_reference(x, w, b, stride, silu, nchw, ldx=None):
    """float64 reference of sfb_conv3x3_small from the header: packed weight [cout, 3, 3, cin16] read back, NHWC
    output [n, ho, wo, cout]."""
    if not nchw:
        x = x[..., :x.shape[-1] if ldx is None else ldx].permute(0, 3, 1, 2)
    cout = w.shape[0]
    wl = w.view(cout, 3, 3, -1).permute(0, 3, 1, 2)[:, :x.shape[1]]
    y = F.conv2d(x.double(), wl.double(), None if b is None else b.double(), stride=stride, padding=1)
    return (F.silu(y) if silu else y).permute(0, 2, 3, 1)


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("n,cin,h,w,cout", [(2, 3, 11, 9, 16), (1, 16, 8, 13, 24), (3, 32, 7, 7, 8)])
def test_conv_small_reference_equals_im2col_matmul(n, cin, h, w, cout, stride):
    g = torch.Generator().manual_seed(cin * 31 + h)
    x = torch.randn(n, cin, h, w, dtype=torch.float64, generator=g)
    w4 = torch.randn(cout, cin, 3, 3, dtype=torch.float64, generator=g)
    b = torch.randn(cout, dtype=torch.float64, generator=g)
    cin16 = (cin + 15) // 16 * 16
    packed = ops.pack_conv3x3(F.pad(w4, (0, 0, 0, 0, 0, cin16 - cin)), torch.float64)
    ref = conv_small_reference(x, packed, b, stride, True, True)
    cols = F.unfold(x, 3, padding=1, stride=stride)                    # [n, cin*9, L] in (c, kh, kw) order
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    mm = (w4.reshape(cout, -1) @ cols + b[:, None]).view(n, cout, ho, wo)
    torch.testing.assert_close(ref, F.silu(mm).permute(0, 2, 3, 1), rtol=1e-12, atol=1e-12)
    # the NHWC form with a channel pitch reads the same values
    xh = F.pad(x.permute(0, 2, 3, 1), (0, 8))
    torch.testing.assert_close(conv_small_reference(xh, packed, b, stride, True, False, ldx=cin), ref)


def test_gather_reference_equals_an_explicit_permute():
    g = torch.Generator().manual_seed(2)
    n, hw, c, ld = 2, 15, 24, 40
    src = torch.randn(n, hw, ld, dtype=torch.float64, generator=g)
    s = -0.7
    ref = s * src[..., :c].permute(0, 2, 1)                             # what the GPU test compares against
    explicit = torch.empty(n, c, hw, dtype=torch.float64)
    for i in range(n):
        for ch in range(c):
            for p in range(hw):
                explicit[i, ch, p] = s * src[i, p, ch]
    assert torch.equal(ref, explicit)


def test_new_struct_layouts_match_the_header(tmp_path):
    structs = {"sfb_conv_small_params": _lib.ConvSmallParams, "sfb_nhwc_to_nchw_params": _lib.NhwcToNchwParams,
               "sfb_nchw_scaled_item": _lib.NchwScaledItem}
    lines = []
    for cname, cls in structs.items():
        lines.append(f'printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            lines.append(f'printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "sfb200.h"\nint main(void) {\n'
                   + "\n".join(lines) + "\nreturn 0; }\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    got = dict(line.split() for line in out.strip().splitlines())
    for cname, cls in structs.items():
        assert int(got[cname]) == ctypes.sizeof(cls), cname
        for fname, _ in cls._fields_:
            assert int(got[f"{cname}.{fname}"]) == getattr(cls, fname).offset, f"{cname}.{fname}"


@_NO_GPU
def test_new_entry_points_reject_bad_arguments():
    lib = _lib.lib()

    def conv(**kw):
        p = _lib.ConvSmallParams(x=_DUMMY_PTR, weight=_DUMMY_PTR, y=_DUMMY_PTR, n=1, h=8, w=8, cin=16, cout=16,
                                 stride=1, ldx=16, ldy=16)
        for k, v in kw.items():
            setattr(p, k, v)
        return lib.sfb_conv3x3_small(ctypes.byref(p), None)
    assert conv() == -2 and conv(x_nchw=1, cin=3, ldx=0) == -2 and conv(cin=56, ldx=64, stride=2) == -2
    for bad in (dict(cin=64, ldx=64), dict(cin=12, ldx=16), dict(ldx=8), dict(stride=3), dict(cout=20, ldy=24),
                dict(ldy=8), dict(x_nchw=1, cin=9), dict(x=None), dict(dtype=2)):
        assert conv(**bad) == -1, bad

    def gather(count=1, **kw):
        p = _lib.NhwcToNchwParams(count=count, scale=_DUMMY_PTR)
        for it in p.items[:max(count, 0)]:
            it.src, it.dst, it.n, it.c, it.hw, it.ld_src = _DUMMY_PTR, _DUMMY_PTR, 1, 8, 4, 8
        for k, v in kw.items():
            setattr(p.items[0], k, v)
        return lib.sfb_nhwc_to_nchw_scaled(ctypes.byref(p), None)
    assert gather() == -2 and gather(16) == -2
    assert gather(0) == -1 and gather(17) == -1 and gather(ld_src=4) == -1 and gather(src=None) == -1
    p = _lib.NhwcToNchwParams(count=1)
    assert lib.sfb_nhwc_to_nchw_scaled(ctypes.byref(p), None) == -1 and b"scale" in lib.sfb_last_error()


def test_gemm_accepts_the_silu_epilogue_by_its_enum_value():
    header = open(os.path.join(ROOT, "include", "sfb200.h")).read()
    assert "SFB_ACT_SILU = 3" in header and _lib.ACT_SILU == 3


@pytest.mark.parametrize("key,value,match", [
    ("global_pool_conditions", True, "global_pool_conditions"),
    ("controlnet_conditioning_channel_order", "rgba", "controlnet_conditioning_channel_order"),
    ("conditioning_channels", 9, "conditioning_channels"),
    ("conditioning_embedding_out_channels", (16, 36, 96, 256), "conditioning_embedding_out_channels"),
    ("conditioning_embedding_out_channels", (16, 32), "conditioning_embedding_out_channels"),
    ("act_fn", "gelu", "act_fn"),
    ("down_block_types", ("SimpleCrossAttnDownBlock2D",) * 4, "down block type"),
])
def test_unsupported_controlnet_configs_are_rejected_by_name(key, value, match):
    with pytest.raises(NotImplementedError, match=match):
        controlnet_spec_from_config(dict(vars(co.sd15_config()), **{key: value}))


def test_stored_channels_pad_only_what_the_wgmma_conv_reads():
    assert [stored_channels(c) for c in (16, 32, 56, 64, 96, 256, 320)] == [16, 32, 56, 64, 128, 256, 320]


# ---------------------------------------------------------------------------------------------------
# compile() routing on stand-in pipelines
# ---------------------------------------------------------------------------------------------------
class ControlNetModel:
    """The attributes compile_controlnet reads of a diffusers ControlNetModel."""

    def __init__(self, cfg):
        self.config = cfg
        self.device = torch.device("cuda")

    def state_dict(self):
        return {}

    def forward(self, *a, **k):
        return "eager"


class MultiControlNetModel:
    def __init__(self, nets):
        self.nets = nets


class OtherAdapter(ControlNetModel):
    pass


class _Pipe:
    def __init__(self, controlnet):
        self.unet = "unet"
        self.controlnet = controlnet


@pytest.fixture
def routing(monkeypatch):
    from sfast.compilers import diffusion_pipeline_compiler as dpc
    from sfast_b200 import runtime
    monkeypatch.setattr(runtime, "require_sm90", lambda device: None)
    monkeypatch.setattr(dpc, "compile_unet", lambda m, config: m)
    cfg = dpc.CompilationConfig.Default()
    return dpc, cfg


def test_compile_replaces_forward_of_a_single_controlnet(routing):
    dpc, cfg = routing
    net = ControlNetModel(co.sd15_config())
    pipe = dpc.compile(_Pipe(net), cfg)
    assert pipe.controlnet is net and net.forward._compiled is not None
    assert net.forward._compiled.spec.cond_channels == 3 and net.forward._cached == {}


def test_compile_replaces_forward_of_every_net_of_a_multi_controlnet(routing, caplog):
    dpc, cfg = routing
    nets = [ControlNetModel(co.sd15_config()), ControlNetModel(co.sd15_config(global_pool_conditions=True)),
            OtherAdapter(co.sd15_config())]
    multi = MultiControlNetModel(nets)
    with caplog.at_level(logging.WARNING):
        assert dpc.compile(_Pipe(multi), cfg).controlnet is multi
    assert nets[0].forward._compiled is not None
    assert nets[1].forward() == "eager" and nets[2].forward() == "eager"
    assert "global_pool_conditions" in caplog.text and "OtherAdapter is not a ControlNetModel" in caplog.text


def test_compile_leaves_an_unsupported_class_eager_with_a_warning(routing, caplog):
    dpc, cfg = routing
    other = OtherAdapter(co.sd15_config())
    with caplog.at_level(logging.WARNING):
        dpc.compile(_Pipe(other), cfg)
    assert other.forward() == "eager" and "left on its eager path" in caplog.text


def test_compile_without_a_controlnet(routing):
    dpc, cfg = routing
    pipe = _Pipe(None)
    assert dpc.compile(pipe, cfg).controlnet is None
