"""GPU checks of the native T2I-Adapter (pytest -m gpu -k t2i): the two new kernels and the GEMM's ReLU epilogue
against float64 on sentinel-filled canvases, a replay of every distinct launch of the adapter plans, the whole
adapter (and a MultiAdapter) against the oracle, the UNet with adapter residuals against the oracle, and the
adapter -> UNet chain of the adapter pipelines."""
import math

import pytest
import torch
import torch.nn.functional as F

import plan_launches as pl
from kernel_checks import rel_err
from oracle import t2i_adapter_oracle as to
from oracle import unet_oracle as uo
from sfast_b200 import _lib, ops
from sfast_b200._lib import TensorMap
from sfast_b200.plan import PackedWeights, intrablock_shapes
from sfast_b200.t2i_adapter_plan import AdapterPlan, t2i_adapter_param_shapes, t2i_adapter_spec_from_config
from sfast_b200.unet_spec import spec_from_config

pytestmark = pytest.mark.gpu
DT = {"fp16": torch.float16, "bf16": torch.bfloat16}
TOL = {torch.float16: 1e-2, torch.bfloat16: 4e-2}


def _rel(got, ref):
    """max(global max-norm error, elementwise |d| / (|ref| + rms(ref))), as tests/test_unet_gpu.py"""
    got, ref = got.float(), ref.float()
    d = (got - ref).abs()
    rms = ref.pow(2).mean().sqrt()
    return max((d.max() / ref.abs().max()).item(), (d / (ref.abs() + rms)).max().item())


def _config(graph=True):
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig
    c = CompilationConfig.Default()
    c.enable_cuda_graph = graph
    return c


# ---------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------
def _unshuffle(x, r, ldy, dt):
    n, c, h, w = x.shape
    out = pl.Canvas(dt, 8, n * (h // r) * (w // r), ldy)
    out.arm()
    _lib.check(_lib.lib().sfb_pixel_unshuffle(x.data_ptr(), out.ptr, n, c, h, w, r, ldy, pl._stream()),
               "sfb_pixel_unshuffle")
    torch.cuda.synchronize()
    got = out.take(out.region(n * (h // r) * (w // r), c * r * r))
    assert out.intact()
    return got


@pytest.mark.parametrize("dt", ["fp16", "bf16"])
@pytest.mark.parametrize("n,c,h,w,r,pad", [(2, 3, 512, 768, 8, 0), (1, 1, 1024, 1024, 16, 0), (1, 1, 1, 1, 1, 8),
                                           (3, 3, 16, 32, 16, 8), (1, 2, 24, 8, 8, 64)])
def test_pixel_unshuffle_is_bit_exact(n, c, h, w, r, pad, dt):
    dt = DT[dt]
    x = torch.randn(n, c, h, w, device="cuda").to(dt)
    got = _unshuffle(x, r, c * r * r + pad, dt)
    ref = F.pixel_unshuffle(x, r).permute(0, 2, 3, 1).reshape(-1, c * r * r)
    assert torch.equal(pl._bits(got), pl._bits(ref.contiguous()))


@pytest.mark.parametrize("dt", ["fp16", "bf16"])
@pytest.mark.parametrize("n,h,w,c,ldx,ldy", [(2, 64, 64, 320, 320, 320), (1, 2, 2, 8, 16, 16), (3, 4, 6, 1280, 1280, 1288),
                                             (1, 32, 64, 640, 648, 640)])
def test_avg_pool2x2_matches_float64(n, h, w, c, ldx, ldy, dt):
    dt = DT[dt]
    xb = pl._randn(n * h * w * ldx + 8, dt)
    x = pl._nhwc_view(xb, 8, n, h, w, c, ldx)
    y = pl.Canvas(dt, 16, n * (h // 2) * (w // 2), ldy)
    y.arm()
    _lib.check(_lib.lib().sfb_avg_pool2x2(xb.data_ptr() + 16, y.ptr, n, h, w, c, ldx, ldy, ops.dtype_code(dt),
                                          pl._stream()), "sfb_avg_pool2x2")
    torch.cuda.synchronize()
    got = y.take(y.region(n * (h // 2) * (w // 2), c))
    ref = F.avg_pool2d(x.double().permute(0, 3, 1, 2), 2, 2, ceil_mode=True).permute(0, 2, 3, 1).reshape(-1, c)
    assert rel_err(got, ref) <= pl.tol("conv_edge", dt) and y.intact()


# ---------------------------------------------------------------------------------------------------
# replay of every distinct launch of the adapter plans
# ---------------------------------------------------------------------------------------------------
def _dry_adapter(cfg, b, h, w, dt):
    spec = t2i_adapter_spec_from_config(cfg)
    sd = {k: torch.empty(v, dtype=dt, device="meta") for k, v in t2i_adapter_param_shapes(spec).items()}
    with pl.recording_map_offsets():
        return AdapterPlan(PackedWeights(spec, sd, dt, "meta", dry=True), b, h, w)


def replay_relu_conv(op):
    """sfb_gemm with SFB_ACT_RELU (the adapter's 3x3 block1): y = relu(conv3x3(x) + bias)."""
    p0, am = op.keep[0], op.keep[1]
    p, dt, res = pl._clone(p0), pl.DTYPES[p0.dtype], pl.Result()
    assert p.a_mode == _lib.A_CONV3X3 and p.splits == 1 and not p.residual and p.act == _lib.ACT_RELU
    n, h, w, c, pitch, bn, bh, bw, stride = am.geom[1:]
    offa = am.base // 2
    abuf = pl._randn(offa + n * h * w * pitch, dt)
    A = pl._nhwc_view(abuf, offa, n, h, w, c, pitch)
    amap = TensorMap.nhwc(abuf.data_ptr() + offa * 2, n, h, w, c, pitch, bn, bh, bw, stride)
    w3 = pl._randn(p.N * c * 9, dt, 1 / math.sqrt(9 * c)).view(p.N, c, 3, 3)
    mat = ops.Mat(ops.pack_conv3x3(w3, dt))
    bmap = mat.map_for(ops.BN // op.keep[2].geom[4])
    bias = torch.randn(p.N, device="cuda")
    out = pl.Canvas(dt, pl._off(p0.out, 2), p.M, p.ldo)
    p.tmap_a, p.tmap_b, p.bias, p.out = amap.ptr, bmap.ptr, bias.data_ptr(), out.ptr
    out.arm()
    _lib.check(_lib.lib().sfb_gemm(pl.C.byref(p), pl._stream()), "sfb_gemm")
    torch.cuda.synchronize()
    ref = (pl.ref_conv3x3(A.double(), w3.double(), stride).reshape(p.M, p.N) + bias.double()).clamp_min(0)
    res.add("out", rel_err(out.take(out.region(p.M, p.N)), ref), pl.tol("conv", dt))
    res.canary(out)
    return res


def replay_unshuffle(op):
    _, _, n, c, h, w, r, ldy = op.args
    dt = op.keep[0].dtype  # the plan's static input: the entry point itself only moves 16-bit values
    x = torch.randn(n, c, h, w, device="cuda").to(dt)
    res = pl.Result()
    got = _unshuffle(x, r, ldy, dt)
    ref = F.pixel_unshuffle(x, r).permute(0, 2, 3, 1).reshape(-1, c * r * r)
    res.add("y", 0.0 if torch.equal(pl._bits(got), pl._bits(ref.contiguous())) else float("inf"), 0.0)
    return res


def replay_pool(op):
    _, _, n, h, w, c, ldx, ldy, code = op.args
    dt = pl.DTYPES[code]
    xb = pl._randn(n * h * w * ldx, dt)
    x = pl._nhwc_view(xb, 0, n, h, w, c, ldx)
    y = pl.Canvas(dt, 0, n * (h // 2) * (w // 2), ldy)
    y.arm()
    _lib.check(_lib.lib().sfb_avg_pool2x2(xb.data_ptr(), y.ptr, n, h, w, c, ldx, ldy, code, pl._stream()), "pool")
    torch.cuda.synchronize()
    ref = F.avg_pool2d(x.double().permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1).reshape(-1, c)
    res = pl.Result()
    res.add("y", rel_err(y.take(y.region(n * (h // 2) * (w // 2), c)), ref), pl.tol("conv_edge", dt))
    res.canary(y)
    return res


def replay_to_nchw(op):
    p = pl._clone(op.keep[0])
    dt = pl.DTYPES[p.dtype]
    scale = torch.rand(p.count, device="cuda") + 0.5
    p.scale = scale.data_ptr()
    items, res = [], pl.Result()
    for i in range(p.count):
        it = p.items[i]
        src = pl._randn(it.n * it.hw * it.ld_src, dt)
        dst = pl.Canvas(dt, 0, it.n * it.c, it.hw)
        it.src, it.dst = src.data_ptr(), dst.ptr
        dst.arm()
        ref = src.view(it.n, it.hw, it.ld_src)[:, :, :it.c].double().permute(0, 2, 1).reshape(-1, it.hw) * scale[i]
        items.append((dst, ref, it.n * it.c, it.hw, src))
    _lib.check(_lib.lib().sfb_nhwc_to_nchw_scaled(pl.C.byref(p), pl._stream()), "sfb_nhwc_to_nchw_scaled")
    torch.cuda.synchronize()
    for i, (dst, ref, rows, cols, _) in enumerate(items):
        res.add(f"dst{i}", rel_err(dst.take(dst.region(rows, cols)), ref), pl.tol("pointwise", dt))
    res.canary(*[it[0] for it in items])
    return res


def _key(op):
    """Distinct-launch key: the GEMMs' as plan_launches keys them; the other launches by their geometry."""
    name = op.fn.name
    if name == "sfb_gemm":
        return pl.launch_key(op)
    if name == "sfb_nhwc_to_nchw_scaled":
        p = op.keep[0]
        return (name, p.dtype, tuple((it.n, it.c, it.hw, it.ld_src) for it in p.items[:p.count]))
    return (name,) + tuple(op.args[2:]) + ((str(op.keep[0].dtype),) if name == "sfb_pixel_unshuffle" else ())


def _replay(op):
    name = op.fn.name
    if name == "sfb_gemm":
        return replay_relu_conv(op) if op.keep[0].act else pl.replay_gemm(op)
    return {"sfb_pixel_unshuffle": replay_unshuffle, "sfb_avg_pool2x2": replay_pool,
            "sfb_nhwc_to_nchw_scaled": replay_to_nchw}[name](op)


def test_every_distinct_launch_of_the_adapter_plans_matches_float64():
    plans = [(to.sd_config(), 1, 512, 512, torch.float16), (to.sd_config(), 2, 512, 768, torch.float16),
             (to.sd_config(in_channels=1), 1, 512, 512, torch.bfloat16),
             (to.sdxl_config(), 1, 1024, 1024, torch.float16), (to.sdxl_config(), 2, 1024, 1024, torch.bfloat16)]
    seen, bad = {}, []
    for cfg, b, h, w, dt in plans:
        plan = _dry_adapter(cfg, b, h, w, dt)
        for op in plan.all_ops():
            seen.setdefault(_key(op), op)
    names = {op.fn.name for op in seen.values()}
    assert names == {"sfb_gemm", "sfb_pixel_unshuffle", "sfb_avg_pool2x2", "sfb_nhwc_to_nchw_scaled"}
    for key, op in seen.items():
        torch.manual_seed(len(bad) + 17)
        r = _replay(op)
        if not r.ok:
            bad.append((op.name, pl.describe(key) if op.fn.name == "sfb_gemm" else key, r.parts))
    print(f"adapter plans: {len(seen)} distinct launches replayed")
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------
# the whole adapter against the oracle
# ---------------------------------------------------------------------------------------------------
def _adapter_pair(cfg, seed, dtype):
    oracle = to.build_adapter(cfg, seed=seed, device="cuda")
    fast = to.build_adapter(cfg, seed=seed, dtype=dtype, device="cuda")
    oracle.load_state_dict({k: v.float() for k, v in fast.state_dict().items()})
    return oracle, fast


def _image(b, c, h, w, dtype, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(b, c, h, w, device="cuda", generator=g).to(dtype)


@pytest.mark.parametrize("cfg,b,size,dt", [
    (to.sd_config(), 1, 512, "fp16"), (to.sd_config(), 2, 512, "fp16"),
    (to.sd_config(in_channels=1), 1, 512, "fp16"), (to.sd_config(in_channels=1), 2, 512, "fp16"),
    (to.sdxl_config(), 1, 1024, "fp16"), (to.sdxl_config(), 1, 1024, "bf16"),
], ids=["sd3_b1", "sd3_b2", "sd1_b1", "sd1_b2", "xl_fp16", "xl_bf16"])
def test_adapter_matches_oracle(cfg, b, size, dt):
    from sfast.compilers.diffusion_pipeline_compiler import compile_adapter
    dt = DT[dt]
    oracle, fast = _adapter_pair(cfg, seed=4, dtype=dt)
    r = fast.total_downscale_factor
    fast = compile_adapter(fast, _config())
    assert fast.total_downscale_factor == r and fast.downscale_factor == cfg.downscale_factor
    x = _image(b, cfg.in_channels, size, size, dt)
    got = fast(x)
    again = fast(x)
    with torch.no_grad():
        ref = oracle(x.float())
    assert len(got) == len(ref) == 4
    for i, (g_, r_) in enumerate(zip(got, ref)):
        assert g_.shape == r_.shape and g_.dtype == dt and g_.is_contiguous()
        err = _rel(g_, r_)
        print(f"adapter {cfg.adapter_type} {cfg.in_channels}ch B={b} {dt} feature {i}: rel err {err:.3e}")
        assert err < TOL[dt], (i, err)
        assert torch.equal(g_, again[i]) and g_.data_ptr() != again[i].data_ptr()
    assert len(fast.forward._cached) == 1


def test_multi_adapter_weighted_sum_matches_oracle():
    from sfast.compilers.diffusion_pipeline_compiler import compile_adapter
    pairs = [_adapter_pair(to.sd_config(), 5, torch.float16), _adapter_pair(to.sd_config(in_channels=1), 6, torch.float16)]
    multi_ref = to.MultiAdapter([p[0] for p in pairs])
    multi = compile_adapter(to.MultiAdapter([p[1] for p in pairs]), _config())
    assert all(a.forward._compiled is not None for a in multi.adapters)
    xs = [_image(2, 3, 512, 512, torch.float16, 1), _image(2, 1, 512, 512, torch.float16, 2)]
    got = multi(xs, [0.7, 0.3])
    with torch.no_grad():
        ref = multi_ref([x.float() for x in xs], [0.7, 0.3])
    for g_, r_ in zip(got, ref):
        assert _rel(g_, r_) < TOL[torch.float16]


# ---------------------------------------------------------------------------------------------------
# the UNet with T2I-Adapter residuals
# ---------------------------------------------------------------------------------------------------
def _unet_pair(cfg, seed, dtype):
    oracle = uo.build_unet(cfg, seed=seed, dtype=torch.float32, device="cuda")
    fast = uo.build_unet(cfg, seed=seed, dtype=dtype, device="cuda")
    oracle.load_state_dict({k: v.float() for k, v in fast.state_dict().items()})
    return oracle, fast


def _compile_unet(m, graph):
    from sfast.compilers.diffusion_pipeline_compiler import compile_unet
    return compile_unet(m, _config(graph))


def _residuals(cfg, b, h, w, dtype, n=None, seed=3):
    g = torch.Generator(device="cuda").manual_seed(seed)
    shapes = intrablock_shapes(spec_from_config(cfg), b, h, w)
    return [(0.5 * torch.randn(s, device="cuda", generator=g)).to(dtype) for s in shapes[:n or len(shapes) - 1]]


def _unet_inputs(cfg, b, h, w, dtype, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    s = torch.randn(b, 4, h, w, device="cuda", generator=g).to(dtype)
    e = torch.randn(b, 77, cfg.cross_attention_dim, device="cuda", generator=g).to(dtype)
    added = None
    if cfg.addition_embed_type == "text_time":
        added = {"text_embeds": torch.randn(b, 1280, device="cuda", generator=g).to(dtype),
                 "time_ids": torch.tensor([[1024., 1024, 0, 0, 1024, 1024]] * b, device="cuda").to(dtype)}
    return s, e, added


def _oracle_call(oracle, s, t, e, added, **res):
    f = {k: (None if v is None else (v.float() if torch.is_tensor(v) else [r.float() for r in v])) for k, v in res.items()}
    with torch.no_grad():
        return to.unet_forward(oracle, s.float(), t, e.float(), added_cond_kwargs=None if added is None else
                      {k: v.float() for k, v in added.items()}, **f).sample


@pytest.mark.parametrize("name,cfgf,size,dt,n", [("tiny", uo.tiny_config, 32, "fp16", None),
                                                 ("sd15", uo.sd15_config, 64, "fp16", None),
                                                 ("sdxl", uo.sdxl_config, 128, "bf16", 4)])
def test_unet_with_adapter_residuals_matches_oracle(name, cfgf, size, dt, n):
    """SDXL: 4 residuals against 3 down blocks, the 4th added after the mid block."""
    cfg, dt = cfgf(), DT[dt]
    oracle, fast = _unet_pair(cfg, seed=9, dtype=dt)
    s, e, added = _unet_inputs(cfg, 2, size, size, dt)
    res = _residuals(cfg, 2, size, size, dt, n)
    keep = list(res)
    t = torch.tensor(400, device="cuda")
    ref = _oracle_call(oracle, s, t, e, added, down_intrablock_additional_residuals=res)
    plain_ref = _oracle_call(oracle, s, t, e, added)
    for graph in (False, True):
        unet = _compile_unet(fast, graph)
        got = unet(s, t, e, added_cond_kwargs=added, down_intrablock_additional_residuals=res).sample
        err = _rel(got, ref)
        print(f"{name} graph={graph}: rel err {err:.3e}")
        assert err < TOL[dt] and _rel(got, plain_ref) > 5 * TOL[dt]
        assert res == keep  # the caller's list is not consumed
        used = len(res)
        assert [k[-1] for k in unet.forward._cached] == [used]


def test_legacy_form_equals_intrablock_form_and_calls_switch_plans():
    cfg = uo.tiny_config()
    oracle, fast = _unet_pair(cfg, seed=12, dtype=torch.float16)
    unet = _compile_unet(fast, True)
    s, e, _ = _unet_inputs(cfg, 2, 32, 32, torch.float16)
    res = _residuals(cfg, 2, 32, 32, torch.float16)
    t = torch.tensor(300, device="cuda")
    a = unet(s, t, e, down_intrablock_additional_residuals=res).sample
    plain = unet(s, t, e).sample
    b = unet(s, t, e, down_block_additional_residuals=res).sample
    assert torch.equal(a, b) and len(unet.forward._cached) == 2
    assert _rel(a, _oracle_call(oracle, s, t, e, None, down_intrablock_additional_residuals=res)) < TOL[torch.float16]
    assert _rel(plain, _oracle_call(oracle, s, t, e, None)) < TOL[torch.float16]
    # leftover residuals are ignored; a mid-shaped one is used only where the mid output has its shape
    extra = res + [torch.zeros(2, 7, 4, 4, device="cuda", dtype=torch.float16)]
    assert torch.equal(unet(s, t, e, down_intrablock_additional_residuals=extra).sample, a)
    with pytest.raises(ValueError, match=r"down_intrablock_additional_residuals\[1\]"):
        unet(s, t, e, down_intrablock_additional_residuals=[res[0], res[0]])
    with pytest.raises(ValueError, match=r"down_block_additional_residuals\[2\]"):
        unet(s, t, e, down_block_additional_residuals=[res[0], res[1], res[1]])


def test_controlnet_and_adapter_residuals_in_one_call():
    cfg = uo.tiny_config()
    oracle, fast = _unet_pair(cfg, seed=13, dtype=torch.float16)
    unet = _compile_unet(fast, True)
    s, e, _ = _unet_inputs(cfg, 2, 32, 32, torch.float16)
    res = _residuals(cfg, 2, 32, 32, torch.float16)
    spec = spec_from_config(cfg)
    g = torch.Generator(device="cuda").manual_seed(4)
    boc, shapes, h = cfg.block_out_channels, [], 32
    shapes.append((boc[0], h))
    for i, c in enumerate(boc):
        shapes += [(c, h)] * cfg.layers_per_block
        if i != len(boc) - 1:
            h //= 2
            shapes.append((c, h))
    down = [(0.5 * torch.randn(2, c, hh, hh, device="cuda", generator=g)).half() for c, hh in shapes]
    mid = (0.5 * torch.randn(2, spec.mid.cout, h, h, device="cuda", generator=g)).half()
    t = torch.tensor(600, device="cuda")
    got = unet(s, t, e, down_block_additional_residuals=down, mid_block_additional_residual=mid,
               down_intrablock_additional_residuals=res).sample
    ref = _oracle_call(oracle, s, t, e, None, down_block_additional_residuals=down, mid_block_additional_residual=mid,
                       down_intrablock_additional_residuals=res)
    assert _rel(got, ref) < TOL[torch.float16]


def test_switching_calls_keep_two_plans_and_replay_bit_identically():
    """The SDXL pipeline's adapter_conditioning_factor drops the residuals for the later steps."""
    cfg = uo.tiny_config()
    oracle, fast = _unet_pair(cfg, seed=14, dtype=torch.float16)
    unet = _compile_unet(fast, True)
    s, e, _ = _unet_inputs(cfg, 2, 32, 32, torch.float16)
    res = _residuals(cfg, 2, 32, 32, torch.float16)
    t = torch.tensor(800, device="cuda")
    first = unet(s, t, e, down_intrablock_additional_residuals=res).sample
    without = unet(s, t, e).sample
    second = unet(s, t, e, down_intrablock_additional_residuals=res).sample
    assert len(unet.forward._cached) == 2 and torch.equal(first, second)
    assert _rel(first, _oracle_call(oracle, s, t, e, None, down_intrablock_additional_residuals=res)) < 1e-2
    assert _rel(without, _oracle_call(oracle, s, t, e, None)) < 1e-2


def test_adapter_pipeline_chain_matches_oracle_chain():
    """StableDiffusionAdapterPipeline's step: features = adapter(image) * adapter_conditioning_scale, repeated for
    classifier-free guidance, then UNet(latents, t, text, down_intrablock_additional_residuals=features)."""
    from sfast.compilers.diffusion_pipeline_compiler import compile_adapter
    a_ref, a_fast = _adapter_pair(to.sd_config(), 21, torch.float16)
    u_ref, u_fast = _unet_pair(uo.sd15_config(), 22, torch.float16)
    a_fast, u_fast = compile_adapter(a_fast, _config()), _compile_unet(u_fast, True)
    cfg = uo.sd15_config()
    img = _image(1, 3, 512, 512, torch.float16, 5)
    s, e, _ = _unet_inputs(cfg, 2, 64, 64, torch.float16)
    t = torch.tensor(500, device="cuda")
    feats = [torch.cat([f * 0.8] * 2) for f in a_fast(img)]
    got = u_fast(s, t, e, down_intrablock_additional_residuals=feats).sample
    with torch.no_grad():
        rfeats = [torch.cat([f * 0.8] * 2) for f in a_ref(img.float())]
    ref = _oracle_call(u_ref, s, t, e, None, down_intrablock_additional_residuals=rfeats)
    err = _rel(got, ref)
    print(f"adapter -> UNet chain (SD-1.5, 512x512, CFG batch 2): rel err {err:.3e}")
    assert err < TOL[torch.float16] and _rel(got, _oracle_call(u_ref, s, t, e, None)) > 5 * TOL[torch.float16]
