"""GPU checks of the native AutoencoderTiny (TAESD) path: sfb_conv3x3_c64 and the edge convs against float64,
every distinct launch of small decode / encode plans replayed against float64, the whole model against the fp32
oracle (oracle/taesd_oracle.py) with the two-sided bar of tests/test_vae_gpu.py, and the compiled module's
behaviour (call forms, graph cache, bit-identical replays, in-place updates, eager routes, use_slicing).

Tolerance of the whole model: against the fp32 oracle the native path must be no worse than 1.25 x the error of
the same oracle module run eagerly in the same 16-bit type (cuDNN, 16-bit storage between layers), in the
elementwise and the rms metric, and its rms error stays below 5e-3 (fp16) / 4e-2 (bf16) absolutely."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from oracle import taesd_oracle as to
from sfast_b200 import _lib, ops

pytestmark = pytest.mark.gpu
DT = [torch.float16, torch.bfloat16]
SENT = -7.0


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _kernel_tol(dt):
    return 4e-3 if dt == torch.float16 else 2.4e-2


def _close(got, ref, dt, what):
    got = got.double()
    scale = ref.abs().max().item() + 1e-6
    err = ((got - ref).abs() / (ref.abs() + 0.05 * scale)).max().item()
    assert err < _kernel_tol(dt), (what, err)


# ----------------------------------------------------------------------------------------------------------
# kernel level
# ----------------------------------------------------------------------------------------------------------
def _padded(n, h, w, ld, dt, fill=None, g=None):
    """NHWC [n, h, w, 64] view with channel pitch ld inside a sentinel-filled buffer with a guard band of two
    rows past the last one; (view, buffer)."""
    buf = torch.full((n * h * w + 2 * w + 8, ld), SENT, dtype=dt, device="cuda")
    v = buf[:n * h * w].view(n, h, w, ld)[..., :64]
    if fill is not None:
        v.copy_(fill)
    elif g is not None:
        v.copy_(torch.randn(n, h, w, 64, generator=g, device="cuda").to(dt))
    return v, buf


def _c64_ref(x, w, b, mode, res, relu):
    xc = x.double().permute(0, 3, 1, 2)
    if mode == _lib.C64_UP2X:
        xc = F.interpolate(xc, scale_factor=2, mode="nearest")
    y = F.conv2d(xc, w.double(), None if b is None else b.double(), stride=2 if mode == _lib.C64_STRIDE2 else 1,
                 padding=1).permute(0, 2, 3, 1)
    if res is not None:
        y = y + res.double()
    return y.relu() if relu else y


def run_c64(x, xbuf, w_oihw, bias, y, ybuf, mode, dt, res=None, rbuf=None, relu=False):
    p = _lib.ConvC64Params()
    p.x, p.weight, p.y = x.data_ptr(), None, y.data_ptr()
    wp = ops.pack_conv3x3(w_oihw, dt)
    p.weight = wp.data_ptr()
    p.bias = bias.data_ptr() if bias is not None else None
    p.residual = res.data_ptr() if res is not None else None
    p.n, p.h, p.w = x.shape[:3]
    p.ldx, p.ldy = xbuf.shape[1], ybuf.shape[1]
    p.ldr = rbuf.shape[1] if rbuf is not None else 0
    p.mode, p.relu, p.dtype = mode, int(relu), ops.dtype_code(dt)
    _lib.check(_lib.lib().sfb_conv3x3_c64(ctypes.byref(p), _stream()), "sfb_conv3x3_c64")


@pytest.mark.parametrize("dt", DT)
@pytest.mark.parametrize("mode", [_lib.C64_SAME, _lib.C64_STRIDE2, _lib.C64_UP2X])
@pytest.mark.parametrize("h,w", [(1, 1), (7, 13), (64, 64), (9, 37)])
def test_conv3x3_c64_against_float64(dt, mode, h, w):
    g = torch.Generator(device="cuda").manual_seed(h * 131 + w * 7 + mode)
    for combo in range(8):
        has_bias, relu, has_res = combo & 1, combo >> 1 & 1, combo >> 2 & 1
        n = 1 + combo % 4
        x, xbuf = _padded(n, h, w, 72, dt, g=g)
        wt = (torch.randn(64, 64, 3, 3, generator=g, device="cuda") / 24).to(dt)
        bias = torch.randn(64, generator=g, device="cuda") if has_bias else None
        ho, wo = ops.c64_out_hw(mode, h, w)
        y, ybuf = _padded(n, ho, wo, 80, dt)
        res = rbuf = None
        if has_res:
            res, rbuf = _padded(n, ho, wo, 96, dt, g=g)
        run_c64(x, xbuf, wt, bias, y, ybuf, mode, dt, res, rbuf, bool(relu))
        torch.cuda.synchronize()
        ref = _c64_ref(x, wt, bias, mode, res, relu)
        _close(y, ref, dt, (mode, h, w, combo))
        # pitch gaps and guard band untouched
        assert bool((ybuf[:, 64:] == SENT).all()) and bool((ybuf[n * ho * wo:] == SENT).all()), combo


def test_conv3x3_c64_in_place_residual():
    g = torch.Generator(device="cuda").manual_seed(5)
    dt = torch.float16
    x, xbuf = _padded(2, 33, 20, 64, dt, g=g)
    r, rbuf = _padded(2, 33, 20, 64, dt, g=g)
    r0 = r.clone()
    wt = (torch.randn(64, 64, 3, 3, generator=g, device="cuda") / 24).to(dt)
    b = torch.randn(64, generator=g, device="cuda")
    run_c64(x, xbuf, wt, b, r, rbuf, _lib.C64_SAME, dt, r, rbuf, True)
    torch.cuda.synchronize()
    _close(r, _c64_ref(x, wt, b, _lib.C64_SAME, r0, True), dt, "in place")


@pytest.mark.parametrize("dt", DT)
@pytest.mark.parametrize("xform,relu,cin", [(_lib.XFORM_TANH3, True, 4), (_lib.XFORM_UNIT, False, 3),
                                            (_lib.XFORM_NONE, True, 8)])
@pytest.mark.parametrize("h,w", [(1, 1), (7, 13), (64, 64), (9, 37)])
def test_edge_conv_against_float64(dt, xform, relu, cin, h, w):
    g = torch.Generator(device="cuda").manual_seed(h + w + cin)
    n = 1 + (h + w) % 4
    x = (torch.randn(n, cin, h, w, generator=g, device="cuda") * 4).to(dt)
    wt = (torch.randn(64, cin, 3, 3, generator=g, device="cuda") / 4).to(dt)
    b = torch.randn(64, generator=g, device="cuda")
    y, ybuf = _padded(n, h, w, 72, dt)
    wp = ops.pack_conv3x3(F.pad(wt, (0, 0, 0, 0, 0, 16 - cin)), dt)
    p = _lib.ConvSmallExParams()
    p.base.x, p.base.weight, p.base.bias, p.base.y = x.data_ptr(), wp.data_ptr(), b.data_ptr(), y.data_ptr()
    p.base.n, p.base.h, p.base.w, p.base.cin, p.base.cout, p.base.stride = n, h, w, cin, 64, 1
    p.base.ldx, p.base.ldy, p.base.x_nchw, p.base.dtype = 0, 72, 1, ops.dtype_code(dt)
    p.in_xform, p.relu = xform, int(relu)
    _lib.check(_lib.lib().sfb_conv3x3_small_ex(ctypes.byref(p), _stream()), "sfb_conv3x3_small_ex")
    torch.cuda.synchronize()
    xd = x.double()
    xd = torch.tanh(xd / 3) * 3 if xform == _lib.XFORM_TANH3 else ((xd + 1) / 2 if xform == _lib.XFORM_UNIT else xd)
    ref = F.conv2d(xd, wt.double(), b.double(), padding=1).permute(0, 2, 3, 1)
    _close(y, ref.relu() if relu else ref, dt, (xform, h, w))
    assert bool((ybuf[:, 64:] == SENT).all()) and bool((ybuf[n * h * w:] == SENT).all())


# ----------------------------------------------------------------------------------------------------------
# plan replay: every distinct launch of a small decode and encode plan against float64
# ----------------------------------------------------------------------------------------------------------
def _weights(dt, seed=3):
    from sfast_b200.plan import PackedWeights
    from sfast_b200.taesd_plan import taesd_spec_from_config
    m = to.build_taesd(seed=seed, dtype=dt, device="cuda")
    return m, PackedWeights(taesd_spec_from_config(m.config), m.state_dict(), dt, torch.device("cuda"))


def _replay(op, dt, g):
    lib = _lib.lib()
    if op.fn is lib.sfb_conv3x3_c64:
        p, xb, w, b, rb, yb = op.keep
        x = xb.view(p.n, p.h, p.w, 64)
        ho, wo = ops.c64_out_hw(p.mode, p.h, p.w)
        x.copy_(torch.randn(x.shape, generator=g, device="cuda").to(dt))
        res = None
        if rb is not None:
            rb.view(-1).copy_(torch.randn(rb.numel(), generator=g, device="cuda").to(dt))
            res = rb.view(p.n, ho, wo, 64).clone()
        op.launch(_stream())
        torch.cuda.synchronize()
        ref = _c64_ref(x, w.view(64, 3, 3, 64).permute(0, 3, 1, 2), b, p.mode, res, p.relu)
        _close(yb.view(p.n, ho, wo, 64), ref, dt, op.name)
    elif op.fn is lib.sfb_conv3x3_small_ex:
        p, x, w, b, yb = op.keep
        x.copy_(torch.randn(x.shape, generator=g, device="cuda").mul(4).to(dt))
        op.launch(_stream())
        torch.cuda.synchronize()
        cin = p.base.cin
        xd = x.double()
        xd = torch.tanh(xd / 3) * 3 if p.in_xform == _lib.XFORM_TANH3 else (xd + 1) / 2
        wt = w.view(64, 3, 3, -1)[..., :cin].permute(0, 3, 1, 2).double()
        ref = F.conv2d(xd, wt, b.double(), padding=1).permute(0, 2, 3, 1)
        _close(yb.view(p.base.n, p.base.h, p.base.w, 64), ref.relu() if p.relu else ref, dt, op.name)
    else:
        assert op.fn is lib.sfb_conv_out
        xb, w, b, out = op.keep
        n, h, wd, c, cout = op.args[4:9]
        x = xb.view(n, h, wd, c)
        x.copy_(torch.randn(x.shape, generator=g, device="cuda").to(dt))
        op.launch(_stream())
        torch.cuda.synchronize()
        ref = F.conv2d(x.double().permute(0, 3, 1, 2), w.view(cout, 3, 3, c).permute(0, 3, 1, 2).double(),
                       b.double(), padding=1)
        _close(out, ref, dt, op.name)


def _launch_key(op):
    lib = _lib.lib()
    if op.fn is lib.sfb_conv3x3_c64:
        p = op.keep[0]
        return ("c64", p.n, p.h, p.w, p.mode, p.relu, p.bias is not None, p.residual is not None)
    if op.fn is lib.sfb_conv3x3_small_ex:
        p = op.keep[0]
        return ("edge", p.base.n, p.base.h, p.base.w, p.base.cin, p.in_xform, p.relu)
    return ("out",) + tuple(op.args[4:9])


@pytest.mark.parametrize("dt", DT)
def test_plan_replay_every_distinct_launch(dt):
    from sfast_b200.taesd_plan import TAESDDecodePlan, TAESDEncodePlan
    _, wts = _weights(dt)
    g = torch.Generator(device="cuda").manual_seed(11)
    seen = set()
    for plan in (TAESDDecodePlan(wts, 2, 6, 10), TAESDEncodePlan(wts, 2, 37, 52)):
        for op in plan.all_ops():
            k = _launch_key(op)
            if k not in seen:
                seen.add(k)
                _replay(op, dt, g)
    assert len(seen) >= 15, seen


# ----------------------------------------------------------------------------------------------------------
# whole model
# ----------------------------------------------------------------------------------------------------------
def _rel(got, ref):
    got, ref = got.float(), ref.float()
    d = (got - ref).abs()
    rms = ref.pow(2).mean().sqrt()
    return max((d.max() / ref.abs().max()).item(), (d / (ref.abs() + rms)).max().item())


def _rms(got, ref):
    got, ref = got.float(), ref.float()
    return ((got - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()


def _compile(m, graph=True):
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_vae
    c = CompilationConfig.Default()
    c.enable_cuda_graph = graph
    return compile_vae(m, c)


def _oracle_of(m16):
    """The fp32 oracle holding exactly the 16-bit module's weights."""
    oracle = to.build_taesd(dtype=torch.float32, device="cuda")
    oracle.load_state_dict({k: v.float() for k, v in m16.state_dict().items()})
    return oracle


def _trio(dt, seed=1, graph=True):
    eager = to.build_taesd(seed=seed, dtype=dt, device="cuda")
    fast = _compile(to.build_taesd(seed=seed, dtype=dt, device="cuda"), graph)
    return _oracle_of(eager), eager, fast


def _bar(got, ref, lib, dt, what):
    e_ours, e_lib, r_ours, r_lib = _rel(got, ref), _rel(lib, ref), _rms(got, ref), _rms(lib, ref)
    print(f"{what}: native {e_ours:.3e} (rms {r_ours:.3e}) | eager 16-bit {e_lib:.3e} (rms {r_lib:.3e})")
    assert got.shape == ref.shape and got.dtype == dt
    assert e_ours < max(1e-2, 1.25 * e_lib), (what, e_ours, e_lib)
    assert r_ours < max(1e-3, 1.25 * r_lib) and r_ours < (5e-3 if dt == torch.float16 else 4e-2), (what, r_ours, r_lib)


@pytest.mark.parametrize("dt", DT)
@pytest.mark.parametrize("h,w,batch,graph,scale", [(64, 64, 1, True, 1.0), (64, 64, 3, False, 1.0),
                                                   (128, 128, 1, True, 1.0), (104, 152, 3, True, 1.0),
                                                   (64, 64, 1, True, 6.0)])
def test_decode_matches_oracle(dt, h, w, batch, graph, scale):
    oracle, eager, fast = _trio(dt, graph=graph)
    g = torch.Generator(device="cuda").manual_seed(h + batch)
    z = (torch.randn(batch, 4, h, w, generator=g, device="cuda") * scale).to(dt)
    with torch.no_grad():
        ref = oracle.decode(z.float()).sample
        lib = eager.decode(z).sample
        got = fast.decode(z).sample
    if scale > 1:
        assert (z.float().abs() > 6).float().mean() > 0.1  # the tanh clamp is active on many latents
    _bar(got, ref, lib, dt, f"decode {batch}x{h}x{w} x{scale} {dt}")


@pytest.mark.parametrize("dt", DT)
@pytest.mark.parametrize("h,w,batch", [(512, 512, 1), (1024, 1024, 1), (517, 300, 2)])
def test_encode_matches_oracle(dt, h, w, batch):
    oracle, eager, fast = _trio(dt)
    g = torch.Generator(device="cuda").manual_seed(h + w)
    x = (torch.rand(batch, 3, h, w, generator=g, device="cuda") * 2 - 1).to(dt)
    with torch.no_grad():
        ref = oracle.encode(x.float()).latents
        lib = eager.encode(x).latents
        got = fast.encode(x).latents
    _bar(got, ref, lib, dt, f"encode {batch}x{h}x{w} {dt}")


# ----------------------------------------------------------------------------------------------------------
# behaviour
# ----------------------------------------------------------------------------------------------------------
def test_call_forms_cache_and_bitwise_replays():
    from sfast_b200.runtime import CompiledTinyVAE
    dt = torch.float16
    m = _compile(to.build_taesd(seed=2, dtype=dt, device="cuda"))
    assert isinstance(m.decode._compiled, CompiledTinyVAE)
    g = torch.Generator(device="cuda").manual_seed(0)
    z = torch.randn(2, 4, 32, 48, generator=g, device="cuda").to(dt)
    a = m.decode(z / m.config.scaling_factor, return_dict=False, generator=g)[0]
    b = m.decode(z).sample
    c = m.decode(z)[0]
    assert torch.equal(a, b) and torch.equal(b, c)
    x = torch.rand(2, 3, 256, 384, generator=g, device="cuda").to(dt) * 2 - 1
    l1 = m.encode(x).latents
    l2 = m.encode(x, return_dict=False)[0]
    assert torch.equal(l1, l2) and tuple(l1.shape) == (2, 4, 32, 48)
    m.decode(z[:1])
    assert len(m.decode._cached) == 3  # decode at batch 2 and 1, encode at batch 2
    assert m.decode._cached is m.encode._cached


def test_in_place_weight_update_is_seen():
    dt = torch.float16
    m = _compile(to.build_taesd(seed=4, dtype=dt, device="cuda"))
    oracle = _oracle_of(m)
    z = torch.randn(1, 4, 24, 24, device="cuda").to(dt)
    before = m.decode(z).sample
    with torch.no_grad():
        for mod in (m, oracle):
            mod.decoder.layers[3].conv[2].weight.mul_(-1.0)
            mod.encoder.layers[0].bias.add_(0.25)
    after = m.decode(z).sample
    assert not torch.equal(before, after)
    with torch.no_grad():
        ref = oracle.decode(z.float()).sample
    assert _rms(after, ref) < 5e-3
    x = torch.rand(1, 3, 64, 64, device="cuda").to(dt) * 2 - 1
    with torch.no_grad():
        assert _rms(m.encode(x).latents, oracle.encode(x.float()).latents) < 5e-3


def test_fp32_and_tiling_go_to_the_modules_own_methods():
    m = _compile(to.build_taesd(seed=6, dtype=torch.float32, device="cuda"))
    z = torch.randn(1, 4, 80, 72, device="cuda")
    x = torch.rand(1, 3, 640, 576, device="cuda") * 2 - 1
    with torch.no_grad():
        assert torch.equal(m.decode(z).sample, to.AutoencoderTiny.decode(m, z).sample)
        assert torch.equal(m.encode(x).latents, to.AutoencoderTiny.encode(m, x).latents)
        m.half()
        m.use_tiling = True
        zh, xh = z.half(), x.half()
        assert torch.equal(m.decode(zh).sample, to.AutoencoderTiny.decode(m, zh).sample)
        assert torch.equal(m.encode(xh).latents, to.AutoencoderTiny.encode(m, xh).latents)
    assert len(m.decode._cached) == 0


def test_use_slicing_equals_batched():
    dt = torch.bfloat16
    m = _compile(to.build_taesd(seed=8, dtype=dt, device="cuda"))
    z = torch.randn(3, 4, 40, 24, device="cuda").to(dt)
    x = torch.rand(3, 3, 96, 160, device="cuda").to(dt) * 2 - 1
    batched, enc = m.decode(z).sample, m.encode(x).latents
    m.use_slicing = True
    assert torch.equal(m.decode(z).sample, batched)
    assert torch.equal(m.encode(x).latents, enc)
    # per image, the batched result is the single-image one
    assert torch.equal(m.decode(z[1:2]).sample, batched[1:2])
