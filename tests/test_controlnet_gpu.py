"""Native ControlNet on the GPU: the two new kernels against float64 references (outputs sentinel-filled), every
distinct launch of the dry ControlNet plans replayed, whole-model parity against the fp32 oracle, and the runtime's
caching / refresh / refusal behaviour.

Every oracle net here has random zero convs, a random embedding conv_out and random norm affines
(controlnet_oracle.build_controlnet): diffusers' zero init would make the parity checks vacuous."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

import plan_launches as pl
from kernel_checks import rel_err
from oracle import controlnet_oracle as co
from oracle import unet_oracle as uo
from sfast_b200 import _lib, ops
from sfast_b200.controlnet_plan import ControlNetPlan
from sfast_b200.plan import PackedWeights
from sfast_b200.unet_spec import controlnet_spec_from_config, param_shapes

pytestmark = pytest.mark.gpu

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

DEV = "cuda"
TOL = {torch.float16: 2e-3, torch.bfloat16: 1e-2}
MODEL_TOL = {torch.float16: 1e-2, torch.bfloat16: 4e-2}
DTS = {_lib.SFB_F16: torch.float16, _lib.SFB_BF16: torch.bfloat16}


def _rel(got, ref):
    """max(global max-norm error, elementwise |d| / (|ref| + rms(ref))), as in test_unet_gpu.py"""
    got, ref = got.float(), ref.float()
    d = (got - ref).abs()
    rms = ref.pow(2).mean().sqrt()
    return max((d.max() / ref.abs().max()).item(), (d / (ref.abs() + rms)).max().item())


# ---------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------
def run_conv_small(n, cin, h, w, cout, stride, dt, nchw, ldx=None, ldy=None, silu=True, with_bias=True):
    """One sfb_conv3x3_small launch on seeded data: (rel err vs float64, outside-output bytes intact)."""
    ldx = ldx or cin
    ldy = ldy or cout
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    if nchw:
        x = torch.randn(n, cin, h, w, device=DEV).to(dt)
        xl = x.double()
    else:
        xb = torch.randn(n, h, w, ldx, device=DEV).to(dt)
        x = xb
        xl = xb[..., :cin].permute(0, 3, 1, 2).double()
    wt = (torch.randn(cout, cin, 3, 3, device=DEV) / math.sqrt(9 * cin)).to(dt)
    cin16 = (cin + 15) // 16 * 16
    wp = ops.pack_conv3x3(F.pad(wt, (0, 0, 0, 0, 0, cin16 - cin)), dt)
    bias = torch.randn(cout, device=DEV) if with_bias else None
    y = pl.Canvas(dt, 0, n * ho * wo, ldy)
    p = _lib.ConvSmallParams()
    p.x, p.weight, p.bias, p.y = x.data_ptr(), wp.data_ptr(), bias.data_ptr() if with_bias else None, y.ptr
    p.n, p.h, p.w, p.cin, p.cout, p.stride, p.ldx, p.ldy = n, h, w, cin, cout, stride, 0 if nchw else ldx, ldy
    p.x_nchw, p.silu, p.dtype = int(nchw), int(silu), ops.dtype_code(dt)
    y.arm()
    _lib.check(_lib.lib().sfb_conv3x3_small(C.byref(p), torch.cuda.current_stream().cuda_stream), "conv3x3_small")
    torch.cuda.synchronize()
    ref = F.conv2d(xl, wt.double(), bias.double() if with_bias else None, stride=stride, padding=1)
    if silu:
        ref = F.silu(ref)
    got = y.take(y.region(n * ho * wo, cout))
    return rel_err(got, ref.permute(0, 2, 3, 1).reshape(-1, cout)), y.intact()


def run_gather(items, dt, scales):
    """One sfb_nhwc_to_nchw_scaled launch; items = [(n, c, hw, ld_src)]: (max rel err, all canvases intact)."""
    p = _lib.NhwcToNchwParams()
    p.count, p.dtype = len(items), ops.dtype_code(dt)
    scale = torch.tensor(scales, dtype=torch.float32, device=DEV)
    p.scale = scale.data_ptr()
    keep, errs, canv = [], [], []
    for i, (n, c, hw, ld) in enumerate(items):
        src = torch.randn(n, hw, ld, device=DEV).to(dt)
        dst = pl.Canvas(dt, 0, n * c, hw)
        dst.arm()
        it = p.items[i]
        it.src, it.dst, it.n, it.c, it.hw, it.ld_src = src.data_ptr(), dst.ptr, n, c, hw, ld
        keep.append((src, dst, n, c, hw))
    _lib.check(_lib.lib().sfb_nhwc_to_nchw_scaled(C.byref(p), torch.cuda.current_stream().cuda_stream), "gather")
    torch.cuda.synchronize()
    for i, (src, dst, n, c, hw) in enumerate(keep):
        ref = scales[i] * src[..., :c].double().permute(0, 2, 1).reshape(n * c, hw)
        errs.append(rel_err(dst.take(dst.region(n * c, hw)), ref))
        canv.append(dst)
    return max(errs), all(d.intact() for d in canv)


# (n, cin, h, w, cout, stride, nchw, ldx, ldy): the SD-1.5 embedding's layers 0-4 at B=2, 512^2 (layer 4's 96
# outputs padded to 128), then odd sizes, stride 2 on odd sizes, channel pitches wider than cin / cout
CONV_CASES = [
    (2, 3, 512, 512, 16, 1, True, None, None),
    (2, 16, 512, 512, 16, 1, False, None, None),
    (2, 16, 512, 512, 32, 2, False, None, None),
    (2, 32, 256, 256, 32, 1, False, None, None),
    (2, 32, 256, 256, 128, 2, False, None, None),
    (1, 3, 37, 53, 16, 1, True, None, 24),
    (3, 1, 19, 7, 8, 2, True, None, 16),
    (1, 24, 37, 53, 40, 2, False, 32, 48),
    (2, 56, 21, 33, 64, 2, False, 64, 72),
    (1, 8, 9, 130, 24, 1, False, 16, 32),
]


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("case", CONV_CASES)
def test_conv3x3_small_matches_float64(case, dt):
    torch.manual_seed(hash(case) % 1000)
    n, cin, h, w, cout, stride, nchw, ldx, ldy = case
    err, intact = run_conv_small(n, cin, h, w, cout, stride, dt, nchw, ldx=ldx, ldy=ldy)
    assert intact, "wrote outside its output"
    assert err <= TOL[dt], err


# the 13 SD-1.5 residuals at B=2, 64^2, some read through a channel pitch wider than c
GATHER_ITEMS = ([(2, 320, 4096, 320)] * 3 + [(2, 320, 1024, 384)] + [(2, 640, 1024, 640)] * 2 +
                [(2, 640, 256, 640)] + [(2, 1280, 256, 1280)] * 2 + [(2, 1280, 64, 1344)] + [(2, 1280, 64, 1280)] * 2 +
                [(2, 1280, 64, 1280)])


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_nhwc_to_nchw_scaled_matches_float64(dt):
    torch.manual_seed(5)
    scales = [0.1 * (i + 1) - 0.35 for i in range(len(GATHER_ITEMS))]
    err, intact = run_gather(GATHER_ITEMS, dt, scales)
    assert intact and err <= TOL[dt], err
    err, intact = run_gather([(3, 24, 37, 40), (1, 8, 5, 8)], dt, [1.5, -2.0])
    assert intact and err <= TOL[dt], err


# ---------------------------------------------------------------------------------------------------
# every distinct launch of the dry ControlNet plans
# ---------------------------------------------------------------------------------------------------
def _dry(cfg, b, h, w, dt=torch.float16):
    spec = controlnet_spec_from_config(cfg)
    sd = {k: torch.empty(v, dtype=dt, device="meta") for k, v in param_shapes(spec).items()}
    with pl.recording_map_offsets():
        return ControlNetPlan(PackedWeights(spec, sd, dt, "meta", dry=True), b, h, w)


PLANS = [("sd15_2x64x64", lambda: _dry(co.sd15_config(), 2, 64, 64)),
         ("sd15_1x64x96", lambda: _dry(co.sd15_config(), 1, 64, 96)),
         ("sdxl_bf16_2x128x128", lambda: _dry(co.sdxl_config(), 2, 128, 128, torch.bfloat16)),
         ("tiny_2x32x32", lambda: _dry(co.tiny_config(), 2, 32, 32))]


def _key(op):
    p = op.keep[0]
    if op.fn.name == "sfb_nhwc_to_nchw_scaled":
        return (op.fn.name, p.count, p.dtype, tuple((it.n, it.c, it.hw, it.ld_src) for it in p.items[:p.count]))
    return pl.launch_key(op)


def _replay_conv_small(op):
    p = op.keep[0]
    err, intact = run_conv_small(p.n, p.cin, p.h, p.w, p.cout, p.stride, DTS[p.dtype], bool(p.x_nchw),
                                 ldx=p.ldx or None, ldy=p.ldy, silu=bool(p.silu), with_bias=bool(p.bias))
    return err, TOL[DTS[p.dtype]], intact


def _replay_gather(op):
    p = op.keep[0]
    items = [(it.n, it.c, it.hw, it.ld_src) for it in p.items[:p.count]]
    scales = [0.1 + 0.07 * i for i in range(p.count)]
    err, intact = run_gather(items, DTS[p.dtype], scales)
    return err, TOL[DTS[p.dtype]], intact


def _replay_conv_silu(op):
    """An SFB_A_CONV3X3 launch with the SiLU epilogue (the embedding layers on the wgmma conv): fresh input laid
    out by the plan's tensor-map geometry, random weights through the project's packer, float64 reference."""
    p = pl._clone(op.keep[0])
    a_geom, b_geom = op.keep[1].geom, op.keep[2].geom
    _, n, h, w, c, pitch, box_n, box_h, box_w, stride = a_geom
    dt = DTS[p.dtype]
    assert p.a_mode == _lib.A_CONV3X3 and p.cin == c and not p.residual and p.splits == 1
    x = torch.randn(n, h, w, pitch, device=DEV).to(dt)
    wt = (torch.randn(p.N, c, 3, 3, device=DEV) / math.sqrt(9 * c)).to(dt)
    mat = ops.Mat(ops.pack_conv3x3(wt, dt))
    ta = _lib.TensorMap.nhwc(x.data_ptr(), n, h, w, c, pitch, box_n, box_h, box_w, stride)
    tb = _lib.TensorMap.matrix(mat.data.data_ptr(), *b_geom[1:])
    bias = torch.randn(p.N, device=DEV)
    out = pl.Canvas(dt, 0, p.M, p.ldo)
    p.tmap_a, p.tmap_b, p.out, p.bias = ta.ptr, tb.ptr, out.ptr, bias.data_ptr()
    out.arm()
    _lib.check(_lib.lib().sfb_gemm(C.byref(p), torch.cuda.current_stream().cuda_stream), "sfb_gemm")
    torch.cuda.synchronize()
    ref = F.silu(F.conv2d(x[..., :c].permute(0, 3, 1, 2).double(), wt.double(), bias.double(), stride=stride,
                          padding=1))
    got = out.take(out.region(p.M, p.N))
    return rel_err(got, ref.permute(0, 2, 3, 1).reshape(-1, p.N)), 1e-2 if dt == torch.bfloat16 else 2e-3, out.intact()


def test_every_controlnet_plan_launch_matches_float64():
    entries = {}
    for pname, build in PLANS:
        for op in build().all_ops():
            if op.fn is None or op.fn.name in pl.SKIP:
                continue
            entries.setdefault(_key(op), (pname, op))
    names = {op.fn.name for _, op in entries.values()}
    assert {"sfb_conv3x3_small", "sfb_nhwc_to_nchw_scaled", "sfb_gemm"} <= names
    failures, n_silu = [], 0
    for key, (pname, op) in entries.items():
        torch.manual_seed(int(pl.key_id(key), 16) % (1 << 31))
        name = op.fn.name
        if name == "sfb_conv3x3_small":
            err, tl, intact = _replay_conv_small(op)
            ok = intact and err <= tl
        elif name == "sfb_nhwc_to_nchw_scaled":
            err, tl, intact = _replay_gather(op)
            ok = intact and err <= tl
        elif name == "sfb_gemm" and op.keep[0].act == _lib.ACT_SILU:
            n_silu += 1
            err, tl, intact = _replay_conv_silu(op)
            ok = intact and err <= tl
        else:
            recs = list(pl.run_keys({key: dict(op=op, plans=[pname], family="controlnet", name=name)}, [key]))
            ok = all(r["ok"] for r in recs)
            err = max(r["err"] for r in recs)
        torch.cuda.empty_cache()
        if not ok:
            failures.append(f"{pname}: {pl.describe(key) if name != 'sfb_nhwc_to_nchw_scaled' else key}: err {err}")
    print(f"{len(entries)} distinct ControlNet plan launches replayed ({n_silu} SiLU convs)")
    assert n_silu >= 2
    assert not failures, "\n".join(failures)


# ---------------------------------------------------------------------------------------------------
# whole model
# ---------------------------------------------------------------------------------------------------
def _compiled_pair(cfg, seed, dt, graph=True):
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_controlnet
    fast = co.build_controlnet(cfg, seed=seed, dtype=dt, device=DEV)
    oracle = co.build_controlnet(cfg, seed=seed, dtype=torch.float32, device=DEV)
    oracle.load_state_dict({k: v.float() for k, v in fast.state_dict().items()})
    cc = CompilationConfig.Default()
    cc.enable_cuda_graph = graph
    return compile_controlnet(fast, cc), oracle


def _inputs(cfg, b, h, w, dt, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    sample = torch.randn(b, 4, h, w, device=DEV, generator=g).to(dt)
    cond = torch.rand(b, cfg.conditioning_channels, 8 * h, 8 * w, device=DEV, generator=g).to(dt)
    ehs = torch.randn(b, 77, cfg.cross_attention_dim, device=DEV, generator=g).to(dt)
    t = torch.tensor(437, device=DEV)
    kw = {}
    if cfg.addition_embed_type == "text_time":
        kw["added_cond_kwargs"] = dict(
            text_embeds=torch.randn(b, 1280, device=DEV, generator=g).to(dt),
            time_ids=torch.tensor([[h * 8, w * 8, 0, 0, h * 8, w * 8]] * b, device=DEV, dtype=torch.float32))
    return sample, t, ehs, cond, kw


def _check(fast, oracle, args, kw, dt, tol=None, **call):
    got = fast(*args, **kw, **call)
    with torch.no_grad():
        fkw = {k: ({kk: vv.float() for kk, vv in v.items()} if isinstance(v, dict) else v) for k, v in kw.items()}
        ref = oracle(*[a.float() if a.is_floating_point() else a for a in args], **fkw, **call)
    errs = [_rel(g, r) for g, r in zip(got.down_block_res_samples, ref.down_block_res_samples)]
    errs.append(_rel(got.mid_block_res_sample, ref.mid_block_res_sample))
    assert len(got.down_block_res_samples) == len(ref.down_block_res_samples)
    assert max(errs) <= (tol or MODEL_TOL[dt]), errs
    return got, max(errs)


@pytest.mark.parametrize("graph", [True, False])
def test_tiny_controlnet_matches_the_oracle(graph):
    cfg = co.tiny_config()
    fast, oracle = _compiled_pair(cfg, 3, torch.float16, graph)
    for b in (1, 2, 3):
        _, err = _check(fast, oracle, _inputs(cfg, b, 32, 32, torch.float16, b)[:4], {}, torch.float16)
        print(f"tiny B={b} graph={graph}: {err:.2e}")


def test_bgr_channel_order():
    cfg = co.tiny_config(controlnet_conditioning_channel_order="bgr")
    fast, oracle = _compiled_pair(cfg, 4, torch.float16)
    _check(fast, oracle, _inputs(cfg, 2, 32, 32, torch.float16)[:4], {}, torch.float16)


@pytest.mark.parametrize("b,h,w", [(2, 64, 64), (1, 64, 96)])
def test_sd15_controlnet_matches_the_oracle(b, h, w):
    cfg = co.sd15_config()
    fast, oracle = _compiled_pair(cfg, 1, torch.float16)
    *args, kw = _inputs(cfg, b, h, w, torch.float16)
    _, err = _check(fast, oracle, args, kw, torch.float16)
    print(f"SD-1.5 ControlNet {b}x{h}x{w}: {err:.2e}")


# SDXL's deep residuals (10-deep transformers) in bf16: every residual's error is ~8x its fp16 error (3 fewer
# mantissa bits; measured on an H100: fp16 <= 6.8e-3, bf16 <= 4.8e-2 under _rel), so the bf16 bound is the fp16
# one scaled by that ratio, capped below it; the fp16 run of the same plan holds the 1e-2 of the UNet tests.
SDXL_TOL = {torch.float16: 1e-2, torch.bfloat16: 6e-2}


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_sdxl_controlnet_matches_the_oracle(dt):
    cfg = co.sdxl_config()
    fast, oracle = _compiled_pair(cfg, 2, dt)
    *args, kw = _inputs(cfg, 2, 128, 128, dt)
    _, err = _check(fast, oracle, args, kw, dt, tol=SDXL_TOL[dt])
    print(f"SDXL ControlNet {dt} 2x128x128: {err:.2e}")


# ---------------------------------------------------------------------------------------------------
# behaviour
# ---------------------------------------------------------------------------------------------------
def test_scales_and_guess_mode_share_one_graph_and_replays_are_identical():
    cfg = co.tiny_config()
    fast, oracle = _compiled_pair(cfg, 5, torch.float16)
    args = _inputs(cfg, 2, 32, 32, torch.float16)[:4]
    first, _ = _check(fast, oracle, args, {}, torch.float16)
    again = fast(*args)
    assert all(torch.equal(a, b) for a, b in zip(first.down_block_res_samples + (first.mid_block_res_sample,),
                                                 again.down_block_res_samples + (again.mid_block_res_sample,)))
    _check(fast, oracle, args, {}, torch.float16, conditioning_scale=0.35)
    _check(fast, oracle, args, {}, torch.float16, conditioning_scale=0.8, guess_mode=True)
    assert len(fast.forward._cached) == 1
    down, mid = fast(*args, return_dict=False)
    assert isinstance(down, tuple) and len(down) == 12 and torch.is_tensor(mid)


def test_in_place_parameter_update_is_seen_by_the_next_call():
    cfg = co.tiny_config()
    fast, oracle = _compiled_pair(cfg, 6, torch.float16)
    args = _inputs(cfg, 2, 32, 32, torch.float16)[:4]
    _check(fast, oracle, args, {}, torch.float16)
    with torch.no_grad():
        for m in (fast, oracle):
            m.controlnet_cond_embedding.blocks[3].weight.mul_(1.5)
            m.controlnet_mid_block.bias.add_(0.25)
    _check(fast, oracle, args, {}, torch.float16)


def test_controlnet_into_unet_matches_oracle_into_oracle():
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_unet
    cfg = co.tiny_config()
    cn, cn_ref = _compiled_pair(cfg, 7, torch.float16)
    unet = uo.build_unet(uo.tiny_config(), seed=8, dtype=torch.float16, device=DEV)
    unet_ref = uo.build_unet(uo.tiny_config(), seed=8, dtype=torch.float32, device=DEV)
    unet_ref.load_state_dict({k: v.float() for k, v in unet.state_dict().items()})
    cc = CompilationConfig.Default()
    cc.enable_cuda_graph = True
    unet = compile_unet(unet, cc)
    sample, t, ehs, cond, _ = _inputs(cfg, 2, 32, 32, torch.float16)
    down, mid = cn(sample, t, ehs, cond, conditioning_scale=0.7, return_dict=False)
    got = unet(sample, t, ehs, down_block_additional_residuals=down, mid_block_additional_residual=mid).sample
    with torch.no_grad():
        rd, rm = cn_ref(sample.float(), t, ehs.float(), cond.float(), conditioning_scale=0.7, return_dict=False)
        ref = unet_ref(sample.float(), t, ehs.float(), down_block_additional_residuals=rd,
                       mid_block_additional_residual=rm).sample
    err = _rel(got, ref)
    print(f"ControlNet -> UNet (tiny): {err:.2e}")
    assert err <= MODEL_TOL[torch.float16], err


def test_refusals_name_the_argument():
    cfg = co.tiny_config()
    fast, _ = _compiled_pair(cfg, 9, torch.float16)
    sample, t, ehs, cond, _ = _inputs(cfg, 1, 32, 32, torch.float16)
    with pytest.raises(NotImplementedError, match="class_labels"):
        fast(sample, t, ehs, cond, class_labels=torch.zeros(1, device=DEV))
    with pytest.raises(NotImplementedError, match="timestep_cond"):
        fast(sample, t, ehs, cond, timestep_cond=torch.zeros(1, 4, device=DEV))
    with pytest.raises(NotImplementedError, match="attention_mask"):
        fast(sample, t, ehs, cond, attention_mask=torch.ones(1, 77, device=DEV))
    with pytest.raises(NotImplementedError, match="cross_attention_kwargs"):
        fast(sample, t, ehs, cond, cross_attention_kwargs={"scale": 0.5})
    with pytest.raises(NotImplementedError, match="dtype"):
        fast(sample.float(), t, ehs.float(), cond.float())
    with pytest.raises(ValueError, match="8x the latent size"):
        fast(sample, t, ehs, cond[:, :, :128, :128])
