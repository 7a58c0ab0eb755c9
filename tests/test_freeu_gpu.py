"""FreeU on the GPU (pytest -m gpu): sfb_freeu against float64 (the backbone scale bit-exact, the Fourier skip filter
within the pointwise tolerance of its closed form, pitch gaps and guard bands untouched), every distinct sfb_freeu
launch of the FreeU plans replayed with the access-model check, the whole UNet with FreeU on against the fp32
oracle (diffusers' FFT form), together with ControlNet and T2I-Adapter residuals, and the enable / change /
disable lifecycle of a compiled UNet."""
import ctypes
import types

import pytest
import torch

import freeu_checks as fc
import plan_hazards as ph
import plan_launches as pl
from oracle import t2i_adapter_oracle as to
from oracle import freeu_oracle as fo
from oracle import unet_oracle as uo
from sfast_b200 import _lib
from sfast_b200.plan import UNetPlan, intrablock_shapes
from sfast_b200.unet_spec import spec_from_config
from test_plan_hazards_gpu import _copy_in, _inputs
from test_plan_hazards_gpu import _unet as _gpu_plan

pytestmark = pytest.mark.gpu
F16, BF16 = torch.float16, torch.bfloat16
TOL = {F16: 1e-2, BF16: 4e-2}
SD15_FREEU, SDXL_FREEU = (0.9, 0.2, 1.2, 1.4), (0.6, 0.4, 1.1, 1.2)   # (s1, s2, b1, b2)


def _rel(got, ref):
    got, ref = got.float(), ref.float()
    d = (got - ref).abs()
    rms = ref.pow(2).mean().sqrt()
    return max((d.max() / ref.abs().max()).item(), (d / (ref.abs() + rms)).max().item())


# ---- the kernel on its own
KERNEL_CASES = [  # n, h, w, c_hidden, c_skip, ld, leading offset (elements)
    (1, 1, 1, 8, 8, 16, 0),
    (2, 2, 2, 16, 24, 48, 8),
    (3, 3, 5, 64, 40, 112, 0),
    (8, 8, 12, 320, 320, 640, 0),
    (2, 16, 16, 1280, 1280, 2560, 0),
    (4, 16, 16, 8, 1280, 1296, 16),
    (2, 64, 64, 640, 320, 968, 0),
    (1, 128, 128, 64, 72, 144, 8),
    (1, 128, 128, 1280, 640, 1920, 0),
]


@pytest.mark.parametrize("dt", [F16, BF16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("case", KERNEL_CASES, ids=[f"{c[0]}x{c[1]}x{c[2]}_{c[3]}+{c[4]}_ld{c[5]}" for c in KERNEL_CASES])
def test_kernel_matches_float64(case, dt):
    n, h, w, ch, cs, ld, off = case
    p = _lib.FreeUParams()
    p.x, p.n, p.h, p.w, p.c_hidden, p.c_skip, p.ld = off * 2 or None, n, h, w, ch, cs, ld
    p.dtype = _lib.SFB_BF16 if dt == BF16 else _lib.SFB_F16
    torch.manual_seed(n * 1000 + h * 10 + w)
    res = fc.replay_freeu(types.SimpleNamespace(keep=(p,)))
    print(f"{case} {dt}: {res.parts}")
    assert res.ok, res.parts


def test_kernel_is_deterministic_and_reads_its_values_from_device_memory():
    n, h, w, ch, cs = 2, 64, 64, 640, 640
    x0 = torch.randn(n, h, w, ch + cs, device="cuda").half() + 0.3
    bs = torch.tensor([1.2, 0.5], device="cuda")
    outs = []
    for vals in ((1.2, 0.5), (1.2, 0.5), (1.0, 1.0)):
        x = x0.clone()
        bs.copy_(torch.tensor(vals))
        p = _lib.FreeUParams()
        p.x, p.bs, p.n, p.h, p.w, p.c_hidden, p.c_skip, p.ld, p.dtype = (
            x.data_ptr(), bs.data_ptr(), n, h, w, ch, cs, ch + cs, _lib.SFB_F16)
        _lib.check(_lib.lib().sfb_freeu(ctypes.byref(p), torch.cuda.current_stream().cuda_stream), "sfb_freeu")
        outs.append(x)
    assert torch.equal(outs[0], outs[1]) and not torch.equal(outs[0], x0)
    # b = s = 1 is the identity up to the filter's fp32 rounding
    assert torch.equal(outs[2][..., :ch], x0[..., :ch]) and _rel(outs[2], x0) < 1e-3


# ---- every distinct launch of the FreeU plans, with the access-model check
def _freeu_entries():
    plans = [pl._unet("tiny_config", 2, 32, 32, freeu=(True, True)),
             pl._unet("tiny_config", 1, 8, 8, freeu=(True, True)),
             pl._unet("sd15_config", 2, 64, 64, freeu=(True, True)),
             pl._unet("sd15_config", 1, 64, 96, freeu=(True, True)),
             pl._unet("sdxl_config", 2, 128, 128, dt=BF16, freeu=(True, True))]
    out = {}
    for plan in plans:
        for name, key, op in pl.launches(plan):
            if name == "sfb_freeu":
                out.setdefault(key, dict(op=op, name=name, plans=[]))
    return out


def test_every_distinct_freeu_launch_matches_float64_and_the_access_model():
    entries = _freeu_entries()
    assert len(entries) >= 10
    for key, ent in entries.items():
        res = pl.replay(key, ent, soundness="rw")
        print(pl.describe(key), [(w, f"{e:.2e}") for w, e, _ in res.parts])
        assert res.ok, (pl.describe(key), res.parts, getattr(res, "model", None))


def test_access_model_holds_on_every_launch_of_a_freeu_plan():
    make = _gpu_plan(uo.tiny_config, 2, 32, 32, controlnet=True, intrablock=4, freeu=(True, True))
    with ph.recording_tensor_maps():
        plan = make()
    _copy_in(_inputs(plan, 3))
    plan.freeu_in.copy_(torch.tensor([1.2, 0.9, 1.4, 0.2]))
    sound = ph.Soundness(read_check=True)
    s = torch.cuda.current_stream().cuda_stream
    for op in plan.all_ops():
        assert ph.checked_call(sound, ph._fn_name(op), op.fn, tuple(op.args) + (s,)) == 0, op.name
    torch.cuda.synchronize()
    assert sound.writes == sound.reads == len(plan.all_ops())
    assert not sound.violations, "\n".join(sound.violations)


# ---- the whole UNet against the oracle
def _pair(cfg, seed, dt):
    oracle = uo.build_unet(cfg, seed=seed, dtype=torch.float32, device="cuda")
    fast = uo.build_unet(cfg, seed=seed, dtype=dt, device="cuda")
    oracle.load_state_dict({k: v.float() for k, v in fast.state_dict().items()})
    return oracle, fast


def _compile(m, graph=True):
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_unet
    c = CompilationConfig.Default()
    c.enable_cuda_graph = graph
    return compile_unet(m, c)


def _inputs_for(cfg, b, h, w, dt, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    s = torch.randn(b, 4, h, w, device="cuda", generator=g).to(dt)
    e = torch.randn(b, 77, cfg.cross_attention_dim, device="cuda", generator=g).to(dt)
    added = None
    if cfg.addition_embed_type == "text_time":
        added = {"text_embeds": torch.randn(b, 1280, device="cuda", generator=g).to(dt),
                 "time_ids": torch.tensor([[1024., 1024, 0, 0, 1024, 1024]] * b, device="cuda").to(dt)}
    return s, e, added


def _oracle(m, s, t, e, added, dtype=torch.float32, **res):
    f = {k: (None if v is None else (v.to(dtype) if torch.is_tensor(v) else [r.to(dtype) for r in v]))
         for k, v in res.items()}
    with torch.no_grad():
        return to.unet_forward(m, s.to(dtype), t, e.to(dtype), added_cond_kwargs=None if added is None else
                               {k: v.to(dtype) for k, v in added.items()}, **f).sample


UNET_CASES = [  # name, config, batch, h, w, dtype, FreeU values
    ("tiny_32x32", uo.tiny_config, 2, 32, 32, F16, SD15_FREEU),
    ("tiny_24x40", uo.tiny_config, 1, 24, 40, F16, SD15_FREEU),
    ("tiny_8x8", uo.tiny_config, 2, 8, 8, F16, SD15_FREEU),
    ("sd15_64x64", uo.sd15_config, 2, 64, 64, F16, SD15_FREEU),
    ("sd15_64x96", uo.sd15_config, 2, 64, 96, F16, SD15_FREEU),
    ("sdxl_128x128_bf16", uo.sdxl_config, 2, 128, 128, BF16, SDXL_FREEU),
]


@pytest.mark.parametrize("name,cfgf,b,h,w,dt,vals", UNET_CASES, ids=[c[0] for c in UNET_CASES])
def test_unet_with_freeu_matches_the_oracle(name, cfgf, b, h, w, dt, vals):
    cfg = cfgf()
    oracle, fast = _pair(cfg, 21, dt)
    s, e, added = _inputs_for(cfg, b, h, w, dt)
    t = torch.tensor(500, device="cuda")
    plain_ref = _oracle(oracle, s, t, e, added)
    fo.enable_freeu(oracle, *vals)
    ref = _oracle(oracle, s, t, e, added)
    fo.enable_freeu(fast, *vals)
    pow2 = dt == F16 and not (h & (h - 1) or w & (w - 1))
    if pow2:
        # the eager fp16 module runs the FFT in half precision at power-of-two sizes: the native step must be no
        # further from the float64 oracle than it is
        o64 = uo.build_unet(cfg, seed=21, dtype=torch.float64, device="cuda")
        o64.load_state_dict({k: v.double() for k, v in fast.state_dict().items()})
        fo.enable_freeu(o64, *vals)
        ref64 = _oracle(o64, s, t, e, added, torch.float64)
        del o64
        eager = _oracle(fast, s, t, e, added, dt)
        eager_err = _rel(eager, ref64)
    for graph in (False, True):
        unet = _compile(fast, graph)
        got = unet(s, t, e, added_cond_kwargs=added).sample
        err = _rel(got, ref)
        print(f"{name} graph={graph}: rel err {err:.3e}, vs FreeU off {_rel(got, plain_ref):.3e}")
        assert err < TOL[dt] and _rel(got, plain_ref) > 5 * TOL[dt]
        if pow2:
            print(f"  vs float64: native {_rel(got, ref64):.3e}, eager fp16 {eager_err:.3e}")
            if eager_err == eager_err:  # (an eager fp16 run that overflowed bounds nothing)
                assert _rel(got, ref64) <= eager_err
        assert [k[-2] for k in unet.forward._cached] == [(True, True)]


def _controlnet_residuals(cfg, b, h, dt, seed=4):
    g = torch.Generator(device="cuda").manual_seed(seed)
    boc, shapes = cfg.block_out_channels, [(cfg.block_out_channels[0], h)]
    for i, c in enumerate(boc):
        shapes += [(c, h)] * cfg.layers_per_block
        if i != len(boc) - 1:
            h //= 2
            shapes.append((c, h))
    down = [(0.5 * torch.randn(b, c, hh, hh, device="cuda", generator=g)).to(dt) for c, hh in shapes]
    mid = (0.5 * torch.randn(b, boc[-1], h, h, device="cuda", generator=g)).to(dt)
    return down, mid


def test_controlnet_adapter_residuals_and_freeu_in_one_call():
    cfg = uo.tiny_config()
    oracle, fast = _pair(cfg, 13, F16)
    unet = _compile(fast, True)
    s, e, _ = _inputs_for(cfg, 2, 32, 32, F16)
    g = torch.Generator(device="cuda").manual_seed(3)
    res = [(0.5 * torch.randn(sh, device="cuda", generator=g)).half()
           for sh in intrablock_shapes(spec_from_config(cfg), 2, 32, 32)[:-1]]
    down, mid = _controlnet_residuals(cfg, 2, 32, F16)
    t = torch.tensor(600, device="cuda")
    kw = dict(down_block_additional_residuals=down, mid_block_additional_residual=mid,
              down_intrablock_additional_residuals=res)
    plain_ref = _oracle(oracle, s, t, e, None, **kw)
    fo.enable_freeu(fast, *SD15_FREEU)
    fo.enable_freeu(oracle, *SD15_FREEU)
    got = unet(s, t, e, **kw).sample
    ref = _oracle(oracle, s, t, e, None, **kw)
    assert _rel(got, ref) < TOL[F16] and _rel(got, plain_ref) > 5 * TOL[F16]


def test_enable_change_disable_reenable():
    cfg = uo.tiny_config()
    oracle, fast = _pair(cfg, 17, F16)
    unet = _compile(fast, True)
    s, e, _ = _inputs_for(cfg, 2, 32, 32, F16)
    t = torch.tensor(700, device="cuda")
    before = unet(s, t, e).sample
    n_plans = lambda: len(unet.forward._cached)  # noqa: E731
    fo.enable_freeu(fast, *SD15_FREEU)
    a1 = unet(s, t, e).sample
    a2 = unet(s, t, e).sample
    assert torch.equal(a1, a2) and n_plans() == 2
    fo.enable_freeu(fast, *SDXL_FREEU)
    b1 = unet(s, t, e).sample
    assert n_plans() == 2 and not torch.equal(a1, b1)
    fo.enable_freeu(oracle, *SDXL_FREEU)
    assert _rel(b1, _oracle(oracle, s, t, e, None)) < TOL[F16]
    fo.disable_freeu(fast)
    off = unet(s, t, e).sample
    assert torch.equal(off, before) and n_plans() == 2
    fo.enable_freeu(fast, *SD15_FREEU)
    assert torch.equal(unet(s, t, e).sample, a1) and n_plans() == 2
    fast.up_blocks[1].s2 = 0.0  # block 1 off: a plan of its own
    fo.enable_freeu(oracle, *SD15_FREEU)
    oracle.up_blocks[1].s2 = 0.0
    c1 = unet(s, t, e).sample
    assert n_plans() == 3 and _rel(c1, _oracle(oracle, s, t, e, None)) < TOL[F16]
    assert isinstance(next(iter(unet.forward._cached.values())).plan, UNetPlan)
