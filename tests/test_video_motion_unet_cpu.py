"""AnimateDiff (UNetMotionModel) without a GPU: the spec read from motion configs and every refusal, the parameter
totals against the oracle module, the dry-built MotionUNetPlan (one motion module per layer in schedule order, each
module's launch sequence, the skip slices proj_out writes, no races or stale reads), the existing plans' launch lists
unchanged, host validation of sfb_frame_attention, and the runtime's call-time refusals."""
import ctypes
import hashlib
import math

import pytest
import torch

import animatediff_checks  # noqa: F401  (registers sfb_frame_attention with the plan checks)
import lcm_inpaint_checks  # noqa: F401  (registers the static input timestep_cond_in)
import plan_hazards as ph
import plan_launches as pl
from oracle import animatediff_oracle as ao
from oracle import unet_oracle as uo
from sfast_b200 import _lib, runtime
from sfast_b200.motion_plan import MotionUNetPlan
from sfast_b200.plan import PackedWeights, UNetPlan, _ForkOp, _JoinOp
from sfast_b200.unet_spec import motion_pe, param_shapes, random_state_dict, spec_from_config
from test_host_logic import _DUMMY_PTR

_NO_GPU = pytest.mark.skipif(torch.cuda.is_available(), reason="needs a box without a GPU: launches must fail")


def _cfg(base, **kw):
    d = dict(vars(base))
    d.update(kw)
    return d


# ---- spec
def test_v152_spec_has_21_motion_modules_in_schedule_order():
    spec = spec_from_config(ao.v152_config())
    names = [m.prefix for m in spec.motion]
    want = [f"down_blocks.{i}.motion_modules.{j}" for i in range(4) for j in range(2)] + \
        ["mid_block.motion_modules.0"] + [f"up_blocks.{i}.motion_modules.{j}" for i in range(4) for j in range(3)]
    assert names == want
    assert [m.head_dim for m in spec.motion] == [40] * 2 + [80] * 2 + [160] * 5 + [160] * 6 + [80] * 3 + [40] * 3
    assert all((m.depth, m.max_seq_len, m.groups, m.heads) == (1, 32, 32, 8) for m in spec.motion)
    after = {m.prefix: m.after for m in spec.motion}
    assert after["down_blocks.0.motion_modules.1"] == "down_blocks.0.attentions.1"
    assert after["down_blocks.3.motion_modules.0"] == "down_blocks.3.resnets.0"
    assert after["mid_block.motion_modules.0"] == "mid_block.attentions.0"
    assert after["up_blocks.0.motion_modules.2"] == "up_blocks.0.resnets.2"
    assert after["up_blocks.3.motion_modules.2"] == "up_blocks.3.attentions.2"
    # the 2-D part is the SD-1.5 UNet's, and the motion spec is not an SVD spec
    sd15 = spec_from_config(uo.sd15_config())
    assert param_shapes(sd15).items() <= param_shapes(spec).items()
    assert not spec.temporal and spec.num_frames == 0


def test_no_mid_tiny_and_sdxl_specs():
    assert len(spec_from_config(ao.no_mid_config()).motion) == 20
    assert "mid_block.motion_modules.0" not in [m.prefix for m in spec_from_config(ao.no_mid_config()).motion]
    tiny = spec_from_config(ao.tiny_config())
    assert [m.head_dim for m in tiny.motion] == [40, 80, 160, 160, 160, 160, 80, 80, 40, 40]
    xl = spec_from_config(ao.tiny_sdxl_config())
    assert xl.addition_embed_type == "text_time" and xl.down[0].attentions == [None]
    assert [m.depth for m in xl.motion] == [1, 2, 1, 1, 1, 1, 2, 2, 1, 1]


def test_per_block_tuples_and_matching_reverse_values_are_accepted():
    cfg = _cfg(ao.v152_config(), motion_num_attention_heads=(8, 8, 8, 8),
               reverse_motion_num_attention_heads=(8, 8, 8, 8), temporal_transformer_layers_per_block=(1, 1, 2, 2),
               reverse_temporal_transformer_layers_per_block=(2, 2, 1, 1), mid_block_layers=1)
    spec = spec_from_config(cfg)
    assert [m.depth for m in spec.motion if m.prefix.startswith("up_blocks.0")] == [2, 2, 2]


REFUSALS = [
    (dict(reverse_motion_num_attention_heads=(4, 8, 8, 8)), "reverse_motion_num_attention_heads"),
    (dict(reverse_temporal_transformer_layers_per_block=(1, 1, 1, 2)), "reverse_temporal_transformer_layers_per_block"),
    (dict(mid_block_layers=2), "mid_block_layers=2"),
    (dict(motion_num_attention_heads=5), "motion head_dim 320/5"),
    (dict(motion_num_attention_heads=(8, 8, 8, 4)), "motion head_dim 1280/4"),
    (dict(motion_max_seq_length=33), "motion_max_seq_length=33"),
    (dict(motion_norm_num_groups=16), "motion_norm_num_groups=16"),
    (dict(down_block_types=("CrossAttnDownBlockMotion",) * 3 + ("DownBlock3D",)), "block type DownBlock3D"),
    (dict(temporal_transformer_layers_per_mid_block=(1, 1)), "temporal_transformer_layers_per_mid_block"),
]


@pytest.mark.parametrize("kw,msg", REFUSALS, ids=[m.split("=")[0].split(" ")[0] for _, m in REFUSALS])
def test_spec_refusals_name_the_key(kw, msg):
    with pytest.raises(NotImplementedError, match=msg.replace("(", r"\(").replace(")", r"\)")):
        spec_from_config(_cfg(ao.v152_config(), **kw))


# ---- parameter totals
@pytest.mark.parametrize("name", ["v152_config", "no_mid_config", "tiny_config", "tiny_sdxl_config"])
def test_param_shapes_equal_the_oracle_module(name):
    cfg = getattr(ao, name)()
    spec = spec_from_config(cfg)
    shapes = param_shapes(spec)
    with torch.device("meta"):
        m = ao.UNetMotionModel(cfg)
    sd = m.state_dict()
    assert set(sd) == set(shapes)
    assert all(tuple(sd[k].shape) == tuple(v) for k, v in shapes.items())
    params = sum(math.prod(v) for k, v in shapes.items() if not k.endswith(".pos_embed.pe"))
    assert params == sum(p.numel() for p in m.parameters())
    per = sum(22 * mm.dim ** 2 + 21 * mm.dim for mm in spec.motion if mm.depth == 1)
    if all(mm.depth == 1 for mm in spec.motion):
        assert ao.motion_parameter_count(m) == per


def test_v152_motion_totals():
    with torch.device("meta"):
        assert ao.motion_parameter_count(ao.UNetMotionModel(ao.v152_config())) == 453_209_280
        assert ao.motion_parameter_count(ao.UNetMotionModel(ao.no_mid_config())) == 417_137_600


def test_random_state_dict_fills_pe_with_the_sinusoid():
    spec = spec_from_config(ao.tiny_config())
    sd = random_state_dict(spec, dtype=torch.float32)
    pe = sd["down_blocks.0.motion_modules.0.transformer_blocks.0.pos_embed.pe"]
    ref = ao.SinusoidalPositionalEmbedding(320, 32).pe
    assert torch.equal(pe, ref) and torch.equal(motion_pe(32, 320), ref)


# ---- dry plans
def _sd(shapes, dt):
    return {k: torch.empty(tuple(v), dtype=dt, device="meta") for k, v in shapes.items()}


def _weights(cfg, dt=torch.float16):
    spec = spec_from_config(cfg)
    return PackedWeights(spec, _sd(param_shapes(spec), dt), dt, "meta", dry=True)


def _motion(cfg, videos, frames, h, w, dt=torch.float16, **kw):
    return MotionUNetPlan(_weights(cfg, dt), videos, frames, h, w, **kw)


def _linear(plan):
    out = []
    for op in plan.ops:
        if isinstance(op, _ForkOp):
            out.extend(op.branch)
        elif not isinstance(op, _JoinOp):
            out.append(op)
    return out


def _module_sequence(m, ops):
    """The module's launches: its GroupNorm (one fused launch, or statistics + apply), proj_in, per block the two
    (QKV, frame attention, to_out) triples and the FeedForward, proj_out."""
    seq = [o for o in ops if o in (m.prefix + ".norm.fused", m.prefix + ".norm.stats", m.prefix + ".norm.apply")]
    assert seq in ([m.prefix + ".norm.fused"], [m.prefix + ".norm.stats", m.prefix + ".norm.apply"]), seq
    seq = seq + [m.prefix + ".proj_in"]
    for d in range(m.depth):
        b = f"{m.prefix}.transformer_blocks.{d}"
        for a in ("attn1", "attn2"):
            seq += [f"{b}.{a}.qkv", f"{b}.{a}.core", f"{b}.{a}.to_out"]
        seq += [b + ".ff.geglu", b + ".ff.out"]
    return seq + [m.prefix + ".proj_out"]


MOTION_PLANS = {
    "tiny_2x8_16x24": lambda: _motion(ao.tiny_config(), 2, 8, 16, 24),
    "tiny_1x16_32x32": lambda: _motion(ao.tiny_config(), 1, 16, 32, 32),
    "tiny_sdxl_bf16": lambda: _motion(ao.tiny_sdxl_config(), 1, 8, 16, 16, torch.bfloat16),
    "v152_2x16_64x64": lambda: _motion(ao.v152_config(), 2, 16, 64, 64),
    "no_mid_1x24_64x64": lambda: _motion(ao.no_mid_config(), 1, 24, 64, 64),
    "v152_controlnet": lambda: _motion(ao.v152_config(), 2, 16, 64, 64, controlnet=True),
}


@pytest.mark.parametrize("name", list(MOTION_PLANS))
def test_one_motion_module_per_layer_in_schedule_order_with_its_launch_sequence(name):
    plan = MOTION_PLANS[name]()
    spec = plan.spec
    ops = [o.name for o in _linear(plan)]
    pos = []
    for m in spec.motion:
        seq = _module_sequence(m, ops)
        k = ops.index(seq[0])
        assert ops[k:k + len(seq)] == seq, m.prefix
        pos.append(k)
        # the module follows its layer's last producer: the resnet's conv2 or the transformer's proj_out
        assert ops[k - 1] == m.after + (".proj_out" if ".attentions." in m.after else ".conv2"), (m.prefix, ops[k - 1])
    assert pos == sorted(pos)
    fa = [o for o in plan.all_ops() if o.fn is not None and o.fn.name == "sfb_frame_attention"]
    assert len(fa) == 2 * sum(m.depth for m in spec.motion)
    for o in fa:
        p = o.keep[0]
        assert (p.batch, p.frames) == (plan.nvid, plan.F) and p.ld_qkv == 3 * p.heads * p.head_dim
        assert tuple(o.keep[2].shape) == (32, 3 * p.heads * p.head_dim) and o.keep[2].dtype == torch.float32


def test_proj_out_writes_the_skip_slices_and_the_next_inputs():
    """A down-block module's proj_out writes its skip slice inside an up-block concat buffer (pitch = that resnet's
    cin, at the skip's channel offset), and that slice is next read by the up path; no other launch writes it."""
    plan, space = ph.build(MOTION_PLANS["v152_2x16_64x64"])
    spec = plan.spec
    up_cin = {r.cin for blk in spec.up for r in blk.resnets}
    with ph.virtual_addresses_of(space):
        ops = _linear(plan)
        idx = {o.name: k for k, o in enumerate(ops)}
        for m in spec.motion:
            k = idx[m.prefix + ".proj_out"]
            out = ops[k]
            gp = out.keep[0]
            if not m.prefix.startswith("down_blocks"):
                continue
            assert gp.ldo in up_cin and gp.ldo > m.dim, (m.prefix, gp.ldo)
            w = [a for a in ph.accesses(out) if a.writes]
            writers = [o.name for j, o in enumerate(ops) if j != k and o.fn is not None and
                       o.fn.name != "sfb_add_nchw_residuals" and
                       any(ph.overlap(a, r) for a in ph.accesses(o) if a.writes for r in w)]
            assert writers == [], (m.prefix, writers)


def test_the_per_frame_inputs():
    plan = _motion(ao.v152_config(), 2, 16, 64, 64)
    assert tuple(plan.sample_in.shape) == (32, 4, 64, 64) and tuple(plan.t_in.shape) == (32,)
    assert tuple(plan.ehs_in.shape) == (32, 77, 768) and tuple(plan.out.shape) == (32, 4, 64, 64)
    fa = [o for o in plan.all_ops() if o.fn is not None and o.fn.name == "sfb_frame_attention"]
    assert fa[0].bytes == 335_544_320 and fa[0].flops == 2_684_354_560  # 64^2 level, C = 320


@pytest.mark.parametrize("name", list(MOTION_PLANS))
def test_motion_plans_are_free_of_races_and_stale_reads(name):
    plan, rep = ph.check_plan(MOTION_PLANS[name])
    assert not rep.findings, "\n".join(map(str, rep.findings))


def test_the_motion_spec_is_refused_by_the_2d_plan_and_frames_are_bounded():
    w = _weights(ao.tiny_config())
    with pytest.raises(ValueError, match="MotionUNetPlan"):
        UNetPlan(w, 2, 16, 16)
    with pytest.raises(NotImplementedError, match="33 frames"):
        MotionUNetPlan(w, 1, 33, 16, 16)
    with pytest.raises(ValueError, match="UNetMotionModel spec"):
        MotionUNetPlan(PackedWeights(spec_from_config(uo.tiny_config()),
                                     _sd(param_shapes(spec_from_config(uo.tiny_config())), torch.float16),
                                     torch.float16, "meta", dry=True), 1, 8, 16, 16)


# ---- the existing plans
def _keys(plan):
    return [(o.name, type(o).__name__ if o.fn is None else pl.launch_key(o)) for o in plan.ops + plan.side_ops]


# sha1 of the (op name, launch key) list of these plans at the commit before the motion UNet
PARENT = {
    "tiny": "f8a188fb61d2fc5426308a59790bd4fcc44a4707",
    "sd15": "f01c18fca41f7bb96b2d7c4f1c446778c496d264",
    "sd15_controlnet": "d1e24c65ef2ca6c61ceb406338fdb2016c5cbec6",
    "sdxl": "92681a1e9f73a2f9ef9d5697663711c7c6798941",
    "svd_xt": "0f190e4a1ce70d25275ba5da4baeb9ff9eb4652c",
}


def _existing(name):
    from oracle import svd_oracle as so
    from sfast_b200.svd_plan import SVDPlan
    if name == "svd_xt":
        spec = spec_from_config(so.svd_xt_config())
        return SVDPlan(PackedWeights(spec, _sd(param_shapes(spec), torch.float16), torch.float16, "meta", dry=True),
                       1, 72, 128)
    cfg, b, h, w, dt, kw = {"tiny": (uo.tiny_config(), 2, 32, 32, torch.float16, {}),
                            "sd15": (uo.sd15_config(), 2, 64, 64, torch.float16, {}),
                            "sd15_controlnet": (uo.sd15_config(), 2, 64, 64, torch.float16, dict(controlnet=True)),
                            "sdxl": (uo.sdxl_config(), 2, 128, 128, torch.bfloat16, {})}[name]
    spec = spec_from_config(cfg)
    return UNetPlan(PackedWeights(spec, _sd(param_shapes(spec), dt), dt, "meta", dry=True), b, h, w, **kw)


@pytest.mark.parametrize("name", list(PARENT))
def test_existing_plans_are_the_parent_plans(name):
    assert hashlib.sha1(repr(_keys(_existing(name))).encode()).hexdigest() == PARENT[name]


# ---- host validation of sfb_frame_attention
def _fa(**kw):
    p = _lib.FrameAttnParams()
    p.qkv, p.out, p.frame_bias = _DUMMY_PTR, _DUMMY_PTR, None
    p.batch, p.frames, p.seq, p.heads, p.head_dim = 1, 16, 1, 8, 40
    p.ld_qkv, p.ld_bias, p.ld_out, p.dtype, p.scale = 960, 960, 320, _lib.SFB_F16, 40 ** -0.5
    for k, v in kw.items():
        setattr(p, k, v)
    return _lib.lib().sfb_frame_attention(ctypes.byref(p), None)


@pytest.mark.parametrize("kw", [dict(frames=0), dict(frames=33), dict(head_dim=48), dict(head_dim=64),
                                dict(head_dim=0), dict(ld_qkv=956), dict(ld_qkv=952), dict(ld_out=316),
                                dict(ld_out=312), dict(qkv=None), dict(out=None), dict(qkv=_DUMMY_PTR + 8),
                                dict(frame_bias=_DUMMY_PTR + 4), dict(frame_bias=_DUMMY_PTR, ld_bias=956),
                                dict(frame_bias=_DUMMY_PTR, ld_bias=962), dict(dtype=_lib.SFB_F32), dict(batch=0),
                                dict(seq=0), dict(heads=0), dict(scale=0.0), dict(scale=-1.0),
                                dict(batch=1 << 20, seq=1 << 7, frames=32)],
                         ids=lambda kw: ",".join(f"{k}={v}" for k, v in kw.items()))
def test_frame_attention_host_validation_rejects(kw):
    rc = _fa(**kw)
    assert rc == -1 and "frame_attention:" in _lib.lib().sfb_last_error().decode()


@_NO_GPU
@pytest.mark.parametrize("kw", [dict(), dict(frames=1, head_dim=80, heads=4), dict(frames=32, head_dim=160, heads=2),
                                dict(frame_bias=_DUMMY_PTR)])
def test_frame_attention_accepted_geometry_reaches_the_launch(kw):
    rc = _fa(**kw)
    assert rc == -2, _lib.lib().sfb_last_error().decode()


# ---- runtime refusals
class _FakeMotionUNet(torch.nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.config = cfg
        self.up_blocks = torch.nn.ModuleList([torch.nn.Module() for _ in cfg.up_block_types])


def _compiled(cfg=None):
    cfg = cfg or ao.tiny_config()
    m = _FakeMotionUNet(cfg)
    return runtime.CompiledUNet(cfg, lambda: {}, module=m), m


def _call(c, **kw):
    x = torch.zeros(1, 4, 8, 16, 16)
    return c(x, 10, torch.zeros(1, 77, 128), **kw)


def test_runtime_refuses_by_name_on_every_call():
    c, m = _compiled()
    with pytest.raises(NotImplementedError, match="attention_mask"):
        _call(c, attention_mask=torch.ones(1, 77))
    with pytest.raises(NotImplementedError, match="down_intrablock_additional_residuals"):
        _call(c, down_intrablock_additional_residuals=[torch.zeros(1)])
    m.up_blocks[0].s1 = 0.9
    with pytest.raises(NotImplementedError, match="FreeU"):
        _call(c)
    m.up_blocks[0].s1 = None
    m.encoder_hid_proj = torch.nn.Identity()
    with pytest.raises(NotImplementedError, match="IP-Adapter"):
        _call(c)
    del m.encoder_hid_proj
    with pytest.raises(NotImplementedError, match="40 frames"):
        c(torch.zeros(1, 4, 40, 16, 16), 10, torch.zeros(1, 77, 128))


def test_runtime_refuses_free_noise_blocks():
    cfg = ao.tiny_config()
    m = _FakeMotionUNet(cfg)
    c = runtime.CompiledUNet(cfg, lambda: {}, module=m)
    FreeNoiseTransformerBlock = type("FreeNoiseTransformerBlock", (torch.nn.Module,), {})
    mods = {}
    for mm in c.spec.motion:
        mod = torch.nn.Module()
        mod.transformer_blocks = torch.nn.ModuleList([FreeNoiseTransformerBlock()])
        mods[mm.prefix] = mod
    m.get_submodule = lambda name: mods[name]
    with pytest.raises(NotImplementedError, match="FreeNoise"):
        _call(c)


def test_runtime_needs_the_5d_sample_and_a_gpu():
    c, _ = _compiled()
    with pytest.raises(ValueError, match=r"\[B, C, F, H, W\]"):
        c(torch.zeros(1, 4, 16, 16), 10, torch.zeros(1, 77, 128))
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="sm_90"):
            _call(c)
