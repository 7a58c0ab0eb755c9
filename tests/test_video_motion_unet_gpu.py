"""AnimateDiff (UNetMotionModel) on the GPU (pytest -m gpu): sfb_frame_attention against float64 over its accepted
domain (frames, head sizes, pixels, videos, heads, pitches, frame bias, dtypes), bit-identical replays and boundary
rejections that write nothing; a float64 replay of every distinct launch the motion plans add, with the access-model
check; the whole motion UNet against the fp32 oracle; and the combinations with ControlNet residuals, PEFT LoRA
adapters on spatial and motion layers, in-place weight updates, timestep_cond and compile(pipe)."""
import copy
import ctypes as C
import gc
import types

import pytest
import torch

import animatediff_checks as ac
import plan_launches as pl
from kernel_checks import rel_err
from oracle import animatediff_oracle as ao
from oracle import lora_oracle as lo
from sfast_b200 import _lib
from sfast_b200.motion_plan import MotionUNetPlan
from sfast_b200.plan import PackedWeights
from sfast_b200.unet_spec import param_shapes, spec_from_config

pytestmark = pytest.mark.gpu
F16, BF16 = torch.float16, torch.bfloat16
TOL = {F16: 1e-2, BF16: 4e-2}
DEV = "cuda"


@pytest.fixture(autouse=True)
def _release_gpu_memory():
    """A compiled module and its replaced forward reference each other, so the packed weights, plans and CUDA graphs
    of a test (tens of GB for the full-width v1-5-2 step) live until the cycle collector runs.  Collecting when each
    test ends frees them, and also frees whatever earlier GPU test files left to the collector, so these full-width
    tests do not depend on when it last ran."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


# ---- the kernel on its own
def _frame_attention(qkv, bias, out, videos, frames, seq, heads, head_dim, dt, scale=None):
    p = _lib.FrameAttnParams()
    p.qkv, p.out = qkv.data_ptr(), out.data_ptr()
    p.frame_bias = None if bias is None else bias.data_ptr()
    p.batch, p.frames, p.seq, p.heads, p.head_dim = videos, frames, seq, heads, head_dim
    p.ld_qkv, p.ld_out = qkv.shape[1], out.shape[1]
    p.ld_bias = 0 if bias is None else bias.shape[1]
    p.dtype = _lib.SFB_F16 if dt == F16 else _lib.SFB_BF16
    p.scale = head_dim ** -0.5 if scale is None else scale
    return _lib.lib().sfb_frame_attention(C.byref(p), torch.cuda.current_stream().cuda_stream)


# (videos, pixels, heads, extra q|k|v pitch, extra out pitch, extra bias pitch, bias)
GEOMETRIES = [(1, 1, 8, 0, 0, 0, True), (2, 7, 5, 8, 16, 4, True), (3, 33, 8, 24, 8, 0, False),
              (1, 130, 5, 0, 0, 12, True), (2, 64, 8, 64, 0, 0, False)]


@pytest.mark.parametrize("dt", [F16, BF16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("head_dim", [40, 80, 160])
@pytest.mark.parametrize("frames", [1, 2, 7, 16, 24, 32])
def test_frame_attention_matches_float64(frames, head_dim, dt):
    g = torch.Generator(device=DEV).manual_seed(frames * 1000 + head_dim)
    for videos, seq, heads, xq, xo, xb, with_bias in GEOMETRIES:
        Cm = heads * head_dim
        rows = videos * frames * seq
        qkv = (torch.randn(rows, 3 * Cm + xq, device=DEV, generator=g) * 1.5).to(dt)
        bias = torch.randn(frames, 3 * Cm + xb, device=DEV, generator=g) if with_bias else None
        outs = []
        for _ in range(2):
            out = torch.full((rows, Cm + xo), 7.0, device=DEV, dtype=dt)
            _lib.check(_frame_attention(qkv, bias, out, videos, frames, seq, heads, head_dim, dt),
                       "sfb_frame_attention")
            outs.append(out)
        torch.cuda.synchronize()
        ref = ac.ref_frame_attention(qkv, bias, videos, frames, seq, heads, head_dim, head_dim ** -0.5)
        err = rel_err(outs[0][:, :Cm], ref)
        what = (videos, seq, heads, xq, xo, xb, with_bias)
        assert err < pl.tol("temporal", dt), (what, err)
        assert torch.equal(outs[0], outs[1]), what                       # bit-identical replay
        assert bool((outs[0][:, Cm:] == 7.0).all()), what                # the pitch gap is untouched


def test_frame_bias_is_the_position_embedding_in_front_of_the_projection():
    """(x + pe_f) W^T through the kernel's frame bias equals the attention of the biased projections."""
    g = torch.Generator(device=DEV).manual_seed(3)
    videos, frames, seq, heads, D = 2, 16, 9, 8, 40
    Cm = heads * D
    x = torch.randn(videos * frames * seq, Cm, device=DEV, generator=g)
    w = torch.randn(3 * Cm, Cm, device=DEV, generator=g) / Cm ** 0.5
    pe = ao.SinusoidalPositionalEmbedding(Cm, 32).pe.to(DEV)[0, :frames]
    qkv = (x @ w.t()).half()
    out = torch.empty(x.shape[0], Cm, device=DEV, dtype=F16)
    _lib.check(_frame_attention(qkv, (pe @ w.t()).contiguous(), out, videos, frames, seq, heads, D, F16))
    xp = x.view(videos, frames, seq, Cm) + pe[None, :, None, :]
    ref = ac.ref_frame_attention((xp.reshape(-1, Cm) @ w.t()).double(), None, videos, frames, seq, heads, D,
                                 D ** -0.5)
    assert rel_err(out, ref) < 1e-2  # q / k / v rounded twice (the projection, then the biased sum)


BOUNDARY = [dict(frames=0), dict(frames=33), dict(head_dim=48), dict(head_dim=64), dict(misaligned_pitch=True),
            dict(null_qkv=True), dict(null_out=True)]


@pytest.mark.parametrize("kw", BOUNDARY, ids=lambda kw: ",".join(f"{k}={v}" for k, v in kw.items()))
def test_rejected_launches_write_nothing(kw):
    frames, D, heads, seq = kw.get("frames", 16), kw.get("head_dim", 40), 8, 5
    Cm = heads * D
    rows = max(frames, 1) * seq
    qkv = torch.randn(rows, 3 * Cm + 8, device=DEV).half()
    out = torch.full((rows, Cm), 3.0, device=DEV, dtype=F16)
    p = _lib.FrameAttnParams()
    p.qkv = None if kw.get("null_qkv") else qkv.data_ptr()
    p.out = None if kw.get("null_out") else out.data_ptr()
    p.batch, p.frames, p.seq, p.heads, p.head_dim = 1, frames, seq, heads, D
    p.ld_qkv = 3 * Cm + (4 if kw.get("misaligned_pitch") else 0)
    p.ld_out, p.dtype, p.scale = Cm, _lib.SFB_F16, 0.1
    before = _lib.lib().sfb_launch_count()
    rc = _lib.lib().sfb_frame_attention(C.byref(p), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert rc == -1 and "frame_attention:" in _lib.lib().sfb_last_error().decode()
    assert _lib.lib().sfb_launch_count() == before and bool((out == 3.0).all())


# ---- every launch the motion plans add, against float64
def _dry(cfg, videos, frames, h, w, dt, **kw):
    spec = spec_from_config(cfg)
    sd = {k: torch.empty(tuple(v), dtype=dt, device="meta") for k, v in param_shapes(spec).items()}
    return MotionUNetPlan(PackedWeights(spec, sd, dt, "meta", dry=True), videos, frames, h, w, **kw)


def _motion_entries():
    """Every distinct launch key of the motion modules of the v1-5-2 (fp16, 2 x 16 frames, 64^2 and 1 x 24 frames,
    40 x 72), no-mid and SDXL-shaped (bf16) plans."""
    out = {}
    for cfg, v, f, h, w, dt in [(ao.v152_config(), 2, 16, 64, 64, F16), (ao.v152_config(), 1, 24, 40, 72, F16),
                                (ao.no_mid_config(), 1, 7, 32, 32, F16), (ao.tiny_sdxl_config(), 2, 8, 16, 24, BF16)]:
        with pl.recording_map_offsets():
            plan = _dry(cfg, v, f, h, w, dt)
        for name, key, op in pl.launches(plan):
            if ".motion_modules." in op.name and name not in pl.SKIP:
                out.setdefault(key, dict(op=op, name=name, plans=[cfg.__class__.__name__]))
    return out


def test_every_motion_launch_matches_float64_and_the_access_model():
    entries = _motion_entries()
    names = sorted({e["name"] for e in entries.values()})
    assert "sfb_frame_attention" in names and "sfb_gemm" in names, names
    for key, ent in entries.items():
        res = pl.replay(key, ent, soundness="rw")
        print(pl.describe(key), [(w, f"{e:.2e}") for w, e, _ in res.parts])
        assert res.ok, (pl.describe(key), res.parts, getattr(res, "model", None))


# ---- the whole UNet against the oracle
def _rel(got, ref):
    got, ref = got.float(), ref.float()
    d = (got - ref).abs()
    rms = ref.pow(2).mean().sqrt()
    return max((d.max() / ref.abs().max()).item(), (d / (ref.abs() + rms)).max().item())


def _pair(cfg, seed, dt):
    oracle = ao.build_unet(cfg, seed=seed, dtype=torch.float32, device=DEV, randomize_pe=True)
    fast = copy.deepcopy(oracle).to(dt)
    oracle.load_state_dict({k: v.float() for k, v in fast.state_dict().items()})
    return oracle, fast


def _compile(m, graph=True):
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_unet
    c = CompilationConfig.Default()
    c.enable_cuda_graph = graph
    return compile_unet(m, c)


def _inputs(cfg, b, f, h, w, dt, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    s = torch.randn(b, cfg.in_channels, f, h, w, device=DEV, generator=g).to(dt)
    e = torch.randn(b, 77, cfg.cross_attention_dim, device=DEV, generator=g).to(dt)
    kw = {}
    if cfg.addition_embed_type == "text_time":
        n_text = cfg.projection_class_embeddings_input_dim - 6 * cfg.addition_time_embed_dim
        kw["added_cond_kwargs"] = {"text_embeds": torch.randn(b, n_text, device=DEV, generator=g).to(dt),
                                   "time_ids": torch.tensor([[8. * h, 8 * w, 0, 0, 8 * h, 8 * w]] * b,
                                                            device=DEV).to(dt)}
    return s, e, kw


def _f32(v):
    if isinstance(v, dict):
        return {k: _f32(x) for k, x in v.items()}
    if isinstance(v, (list, tuple)):
        return [_f32(x) for x in v]
    return v.float() if torch.is_tensor(v) and v.is_floating_point() else v


def _ref(oracle, s, t, e, **kw):
    with torch.no_grad():
        return oracle(s.float(), t, e.float(), **_f32(kw)).sample


UNET_CASES = [  # name, config, videos, frames, h, w, dtype, graph modes
    ("tiny_1x8", ao.tiny_config, 1, 8, 16, 16, F16, (False, True)),
    ("tiny_2x16_rect", ao.tiny_config, 2, 16, 16, 24, F16, (False, True)),
    ("tiny_2x8_rect", ao.tiny_config, 2, 8, 24, 16, F16, (True,)),
    ("tiny_1x16", ao.tiny_config, 1, 16, 32, 32, F16, (True,)),
    ("tiny_sdxl_bf16", ao.tiny_sdxl_config, 2, 8, 16, 24, BF16, (False, True)),
    ("v152_2x16_64", ao.v152_config, 2, 16, 64, 64, F16, (True,)),
]


@pytest.mark.parametrize("name,cfgf,b,f,h,w,dt,graphs", UNET_CASES, ids=[c[0] for c in UNET_CASES])
def test_motion_unet_matches_the_oracle(name, cfgf, b, f, h, w, dt, graphs):
    cfg = cfgf()
    oracle, fast = _pair(cfg, 21, dt)
    s, e, kw = _inputs(cfg, b, f, h, w, dt)
    t = torch.tensor(500, device=DEV)
    ref = _ref(oracle, s, t, e, **kw)
    del oracle
    torch.cuda.empty_cache()
    for graph in graphs:
        got = _compile(fast, graph)(s, t, e, **kw).sample
        assert got.shape == (b, cfg.out_channels, f, h, w)
        err = _rel(got, ref)
        print(f"{name} graph={graph}: rel err {err:.3e}")
        assert err < TOL[dt]
        again = fast(s, t, e, **kw).sample
        assert torch.equal(again, got)  # bit-identical replay


# ---- combinations
def _controlnet_residuals(cfg, b, f, h, w, dt, seed=1):
    spec = spec_from_config(cfg)
    g = torch.Generator(device=DEV).manual_seed(seed)
    shapes, hh, ww = [(spec.block_out_channels[0], h, w)], h, w
    for blk in spec.down:
        shapes += [(blk.cout, hh, ww)] * len(blk.resnets)
        if blk.sampler:
            hh, ww = hh // 2, ww // 2
            shapes.append((blk.cout, hh, ww))
    down = [0.3 * torch.randn(b * f, *s_, device=DEV, generator=g).to(dt) for s_ in shapes]
    mid = 0.3 * torch.randn(b * f, spec.mid.cout, hh, ww, device=DEV, generator=g).to(dt)
    return down, mid


def test_controlnet_residuals_and_timestep_cond():
    cfg = ao.tiny_config()
    cfg.time_cond_proj_dim = 32
    oracle, fast = _pair(cfg, 13, F16)
    unet = _compile(fast)
    s, e, kw = _inputs(cfg, 2, 8, 16, 16, F16)
    t = torch.tensor(600, device=DEV)
    kw["timestep_cond"] = torch.randn(2, 32, device=DEV).half()
    plain_ref = _ref(oracle, s, t, e, **kw)
    got = unet(s, t, e, **kw).sample
    assert _rel(got, plain_ref) < TOL[F16]
    no_cond = unet(s, t, e).sample
    assert _rel(no_cond, _ref(oracle, s, t, e)) < TOL[F16] and _rel(no_cond, got) > 5 * TOL[F16]
    down, mid = _controlnet_residuals(cfg, 2, 8, 16, 16, F16)
    kw.update(down_block_additional_residuals=down, mid_block_additional_residual=mid)
    got = unet(s, t, e, **kw).sample
    ref = _ref(oracle, s, t, e, **kw)
    assert _rel(got, ref) < TOL[F16] and _rel(ref, plain_ref) > 5 * TOL[F16]
    assert len(unet.forward._cached) == 2


def test_lora_on_spatial_and_motion_layers_merges_and_switches_off():
    cfg = ao.tiny_config()
    oracle, fast = _pair(cfg, 3, F16)
    targets = ["down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_q",
               "down_blocks.0.motion_modules.0.transformer_blocks.0.attn1.to_q",
               "down_blocks.0.motion_modules.0.transformer_blocks.0.attn2.to_v",
               "up_blocks.2.motion_modules.1.transformer_blocks.0.attn1.to_out.0"]
    for m in (fast, oracle):
        lo.inject_adapter(m, "motion", targets, r=8, lora_alpha=16, seed=3)
    unet = _compile(fast)
    s, e, kw = _inputs(cfg, 1, 8, 16, 16, F16)
    t = torch.tensor(500, device=DEV)
    got = unet(s, t, e).sample
    ref = _ref(oracle, s, t, e)
    lo.disable_lora(oracle)
    free = _ref(oracle, s, t, e)
    assert _rel(got, ref) < TOL[F16] and _rel(ref, free) > 5 * TOL[F16]
    lo.disable_lora(fast)
    off = unet(s, t, e).sample
    assert _rel(off, free) < TOL[F16] and len(unet.forward._cached) == 1


def test_in_place_weight_update_is_picked_up_on_the_same_graph():
    cfg = ao.tiny_config()
    oracle, fast = _pair(cfg, 5, F16)
    unet = _compile(fast)
    s, e, _ = _inputs(cfg, 1, 8, 16, 16, F16)
    t = torch.tensor(300, device=DEV)
    before = unet(s, t, e).sample
    names = ["down_blocks.1.motion_modules.0.transformer_blocks.0.attn1.to_k.weight",
             "up_blocks.0.motion_modules.0.transformer_blocks.0.pos_embed.pe",
             "mid_block.motion_modules.0.proj_out.weight"]
    with torch.no_grad():
        for n in names:
            for m in (fast, oracle):
                sdm = dict(m.named_parameters())
                sdm.update(dict(m.named_buffers()))
                sdm[n].mul_(1.5)
    after = unet(s, t, e).sample
    assert len(unet.forward._cached) == 1
    assert _rel(after, _ref(oracle, s, t, e)) < TOL[F16] and _rel(after, before) > 5 * TOL[F16]


def test_compile_pipe_replaces_the_motion_unet_forward():
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile
    cfg = ao.tiny_config()
    oracle, fast = _pair(cfg, 9, F16)
    pipe = types.SimpleNamespace(unet=fast, vae=None, text_encoder=None)
    c = CompilationConfig.Default()
    c.enable_cuda_graph = True
    compile(pipe, c)
    assert hasattr(pipe.unet.forward, "_compiled")
    s, e, _ = _inputs(cfg, 2, 16, 16, 16, F16)
    out = pipe.unet(s, torch.tensor(700, device=DEV), e)
    assert out.sample.shape == (2, 4, 16, 16, 16) and torch.equal(out[0], out.sample)
    assert _rel(out.sample, _ref(oracle, s, torch.tensor(700, device=DEV), e)) < TOL[F16]
    assert pipe.unet(s, 700, e, return_dict=False)[0].shape == (2, 4, 16, 16, 16)
