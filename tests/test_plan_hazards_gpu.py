"""Schedule independence of every plan with side-stream work: two consecutive steps on different seeded inputs give
bit-identical outputs under five schedules of the same launches --
  A  the captured CUDA graph, as the runtime replays it;
  B  Plan.run() without a graph (two streams);
  C  one stream, side work as early as possible (side_ops first, fork branches in place);
  D  one stream, side work as late as possible (each side op right before the first join that covers it, each fork
     branch right before its join);
  E  schedule C with programmatic dependent launch off --
and to a fresh plan's first step on the second inputs.  C and D order every side launch at the opposite ends of
what the joins allow, so a dependency the joins miss makes them disagree on every run, whatever the timing."""
import math
import os
import time

import pytest
import torch

import plan_hazards as ph

from oracle import controlnet_oracle as co
from oracle import svd_oracle as so
from oracle import unet_oracle as uo
from sfast_b200 import _lib
from sfast_b200.plan import PackedWeights, UNetPlan, _ForkOp, _JoinOp
from sfast_b200.unet_spec import (controlnet_spec_from_config, ip_adapter_geometry, ip_adapter_plus_geometry,
                                  param_shapes, spec_from_config)

pytestmark = pytest.mark.gpu

INPUTS = ("sample_in", "ehs_in", "t_in", "add_in", "time_ids_in", "image_embeds_in", "ip_scale_in", "cond_in",
          "scale_in")
LISTS = ("ctrl_in", "intrablock_in")


def _weights(spec, shapes, dt, seed):
    """Seeded weights scaled by fan-in (finite activations through every layer)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    sd = {}
    for k, s in sorted(shapes.items()):
        s = tuple(s)
        if len(s) == 1:
            v = (1.0 if k.endswith("weight") else 0.0) + 0.1 * torch.randn(s, device="cuda", generator=g)
        else:
            v = torch.randn(s, device="cuda", generator=g) / math.sqrt(max(1, math.prod(s[1:])))
        sd[k] = v.to(dt)
    return PackedWeights(spec, sd, dt, "cuda")


def _unet(cfg, b, h, w, dt=torch.float16, ip=None, **kw):
    spec = spec_from_config(cfg())
    if ip == "plain":
        spec.ip = ip_adapter_geometry(spec, 64)
    elif ip == "plus":
        spec.ip = ip_adapter_plus_geometry(spec, 128, 128)
    wts = _weights(spec, param_shapes(spec), dt, 0)
    return lambda: UNetPlan(wts, b, h, w, **kw)


def _controlnet():
    from sfast_b200.controlnet_plan import ControlNetPlan
    spec = controlnet_spec_from_config(co.tiny_config())
    wts = _weights(spec, param_shapes(spec), torch.float16, 1)
    return lambda: ControlNetPlan(wts, 2, 32, 32)


def _svd():
    from sfast_b200.svd_plan import SVDPlan
    spec = spec_from_config(so.svd_tiny_config())
    wts = _weights(spec, param_shapes(spec), torch.float16, 2)
    return lambda: SVDPlan(wts, 2, 16, 16)


PLANS = {
    "tiny": lambda: _unet(uo.tiny_config, 2, 32, 32),
    "tiny_controlnet_ip_t2i": lambda: _unet(uo.tiny_config, 2, 32, 32, controlnet=True, intrablock=5, ip="plain",
                                            ip_len=4),
    "tiny_ip_plus": lambda: _unet(uo.tiny_config, 2, 32, 32, ip="plus", ip_len=16, ip_seq=257),
    "tiny_t2i": lambda: _unet(uo.tiny_config, 2, 32, 32, intrablock=4),
    "controlnet_tiny": _controlnet,
    "svd_tiny": _svd,
    "sd15_2x64x64_fp16": lambda: _unet(uo.sd15_config, 2, 64, 64),
    "sdxl_2x128x128_bf16": lambda: _unet(uo.sdxl_config, 2, 128, 128, dt=torch.bfloat16),
}


def _inputs(plan, seed):
    """{input tensor: value} of one step."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for n in INPUTS:
        t = getattr(plan, n, None)
        if t is not None:
            out.append((n, t))
    for n in LISTS:
        out += [(f"{n}[{i}]", t) for i, t in enumerate(getattr(plan, n, []) or [])]
    vals = {}
    for n, t in out:
        if n == "t_in":
            v = torch.rand(t.shape, device="cuda", generator=g) * 999.0
        elif n == "time_ids_in":
            v = torch.randint(0, 1024, t.shape, device="cuda", generator=g).float()
        elif n in ("ip_scale_in", "scale_in"):
            v = 0.5 + torch.rand(t.shape, device="cuda", generator=g)
        else:
            v = torch.randn(t.shape, device="cuda", generator=g)
        vals[n] = (t, v.to(t.dtype))
    return vals


def _outputs(plan):
    outs = {"out": plan.out}
    if getattr(plan, "down_out", None):
        outs.update({f"down_out[{i}]": t for i, t in enumerate(plan.down_out)})
        outs["mid_out"] = plan.mid_out
    return {k: t for k, t in outs.items() if t.numel()}   # (a ControlNet plan's UNet output is empty)


def _copy_in(vals):
    for t, v in vals.values():
        t.copy_(v)


def _serial(plan, late):
    """One step on the current stream: side work as early (late=False) or as late (late=True) as the joins allow."""
    s = torch.cuda.current_stream().cuda_stream
    pending = list(plan.side_ops)
    temb = getattr(plan, "_temb_last", None)
    if not late:
        for op in pending:
            op.launch(s)
        pending = []
    for op in plan.ops:
        if isinstance(op, _JoinOp):
            if op.kind == "temb" and late:
                n = pending.index(temb) + 1 if temb in pending else 0
                for o in pending[:n]:
                    o.launch(s)
                pending = pending[n:]
            elif op.kind == "all" and late:
                for o in pending:
                    o.launch(s)
                pending = []
            elif op.kind not in ("temb", "all") and late:
                for o in op.kind.branch:
                    o.launch(s)
        elif isinstance(op, _ForkOp):
            if not late:
                for o in op.branch:
                    o.launch(s)
        else:
            op.launch(s)
    for o in pending:
        o.launch(s)


def _two_steps(plan, step, in1, in2):
    _copy_in(in1)
    step()
    _copy_in(in2)
    step()
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in _outputs(plan).items()}


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


@pytest.mark.parametrize("name", list(PLANS))
def test_outputs_do_not_depend_on_the_schedule(name):
    from sfast_b200.runtime import _GraphedPlan
    make = PLANS[name]()
    plan = make()
    assert plan.side_ops or any(isinstance(op, _ForkOp) for op in plan.ops)
    in1, in2 = _inputs(plan, 1), _inputs(plan, 2)
    lib = _lib.lib()
    got = {}
    gp = _GraphedPlan(plan, True)
    got["A graph"] = _two_steps(plan, gp.step, in1, in2)
    got["B run"] = _two_steps(plan, plan.run, in1, in2)
    got["C early"] = _two_steps(plan, lambda: _serial(plan, False), in1, in2)
    got["D late"] = _two_steps(plan, lambda: _serial(plan, True), in1, in2)
    pdl = int(os.environ.get("SFB_PDL", "1") or 0) != 0   # the library's setting (it reads SFB_PDL at load)
    try:
        lib.sfb_set_pdl(0)
        got["E early, no PDL"] = _two_steps(plan, lambda: _serial(plan, False), in1, in2)
    finally:
        lib.sfb_set_pdl(int(pdl))
    fresh = make()
    _copy_in({k: (getattr(fresh, k) if "[" not in k else getattr(fresh, k.split("[")[0])[int(k[:-1].split("[")[1])],
                  v) for k, (_, v) in in2.items()})
    fresh.run()
    torch.cuda.synchronize()
    got["fresh plan, first step"] = {k: v.clone() for k, v in _outputs(fresh).items()}
    ref = got["A graph"]
    for k, v in ref.items():
        assert bool(torch.isfinite(v.float()).all()), f"{name}: {k} is not finite"
        assert v.float().abs().max() > 0, f"{name}: {k} is all zero"
    bad = [f"{sched}: {k}" for sched, outs in got.items() for k, v in outs.items()
           if not torch.equal(_bits(v), _bits(ref[k]))]
    print(f"\n{name}: {len(ref)} outputs, {len(got)} schedules")
    assert not bad, f"{name}: outputs differ from the captured graph's: {bad}"


# ---------------------------------------------------------------------------------------------------------------------
# the access model of tests/plan_hazards.py against the kernels, on the launches of real feature plans (their entry
# points -- IP-Adapter attention, the few-channel and 64-channel convs, PixelUnshuffle, pooling, the scaled NCHW
# outputs, the temporal conv_out -- have no float64 replay in plan_launches.py; the core ones are checked there)
# ---------------------------------------------------------------------------------------------------------------------
def _adapter():
    from oracle import t2i_adapter_oracle as tio
    from sfast_b200.t2i_adapter_plan import AdapterPlan, t2i_adapter_param_shapes, t2i_adapter_spec_from_config
    spec = t2i_adapter_spec_from_config(tio.sd_config())
    wts = _weights(spec, t2i_adapter_param_shapes(spec), torch.float16, 3)
    return lambda: AdapterPlan(wts, 1, 256, 256)


def _taesd(kind):
    from oracle import taesd_oracle as tao
    from sfast_b200 import taesd_plan as tp
    spec = tp.taesd_spec_from_config(tao.tiny_config())
    wts = _weights(spec, {**tp.taesd_decoder_param_shapes(spec), **tp.taesd_encoder_param_shapes(spec)},
                   torch.float16, 4)
    return lambda: (tp.TAESDDecodePlan(wts, 1, 32, 32) if kind == "decode" else tp.TAESDEncodePlan(wts, 1, 256, 256))


def _temporal_decode():
    from oracle import svd_vae_oracle as svo
    from sfast_b200.vae_plan import TemporalDecodePlan, vae_spec_from_config, vae_temporal_decoder_param_shapes
    spec = vae_spec_from_config(svo.svd_vae_config())
    wts = _weights(spec, vae_temporal_decoder_param_shapes(spec), torch.float16, 5)
    return lambda: TemporalDecodePlan(wts, 4, 2, 16, 16)


MODEL_PLANS = {
    "tiny_controlnet_ip_t2i": PLANS["tiny_controlnet_ip_t2i"],
    "tiny_ip_plus": PLANS["tiny_ip_plus"],
    "controlnet_tiny": _controlnet,
    "svd_tiny": _svd,
    "adapter_sd_1x256x256": _adapter,
    "taesd_decode_1x32x32": lambda: _taesd("decode"),
    "taesd_encode_1x256x256": lambda: _taesd("encode"),
    "temporal_decode_4f2_16x16": _temporal_decode,
}


@pytest.mark.parametrize("name", list(MODEL_PLANS))
def test_access_model_holds_on_every_launch_of_the_feature_plans(name):
    """One step, serially, every launch checked: bytes written outside the modelled write regions, or outputs that
    depend on bytes outside the modelled read regions, fail."""
    t0 = time.time()
    make = MODEL_PLANS[name]()
    with ph.recording_tensor_maps():
        plan = make()
    _copy_in(_inputs(plan, 7))
    for n in ("z_in", "x_in"):
        if getattr(plan, n, None) is not None:
            getattr(plan, n).copy_(torch.randn(getattr(plan, n).shape, device="cuda").to(plan.dt))
    sound = ph.Soundness(read_check=True)
    s = torch.cuda.current_stream().cuda_stream
    names = set()
    for op in plan.all_ops():
        name_ = ph._fn_name(op)
        names.add(name_)
        assert ph.checked_call(sound, name_, op.fn, tuple(op.args) + (s,)) == 0, op.name
    torch.cuda.synchronize()
    print(f"\n{name}: {sound.writes} launches, writes and reads checked ({', '.join(sorted(names))}), "
          f"{time.time() - t0:.1f} s")
    assert sound.writes == sound.reads == len(plan.all_ops())
    assert not sound.violations, "\n".join(sound.violations)
