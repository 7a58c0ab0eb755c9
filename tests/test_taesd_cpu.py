"""Host-side checks of the native AutoencoderTiny (TAESD) decode and encode: parameter names against the oracle,
the config refusals, dry launch schedules and their buffers, an fp64 restatement of sfb_conv3x3_c64's three
input modes and two epilogues, and the routing of `compile_vae_module`."""
import logging

import pytest
import torch
import torch.nn.functional as F

from oracle import taesd_oracle as to
from sfast_b200 import _lib, ops
from sfast_b200.plan import PackedWeights
from sfast_b200.taesd_plan import (TAESDDecodePlan, TAESDEncodePlan, taesd_decoder_param_shapes,
                                   taesd_encoder_param_shapes, taesd_spec_from_config)


def _dry(cfg=None, dt=torch.float16):
    spec = taesd_spec_from_config(cfg or to.tiny_config())
    shapes = {**taesd_decoder_param_shapes(spec), **taesd_encoder_param_shapes(spec)}
    sd = {k: torch.empty(v, dtype=dt, device="meta") for k, v in shapes.items()}
    return PackedWeights(spec, sd, dt, "meta", dry=True)


def test_param_names_and_shapes_match_the_oracle():
    m = to.AutoencoderTiny(to.tiny_config())
    spec = taesd_spec_from_config(m.config)
    want = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    got = {**taesd_decoder_param_shapes(spec), **taesd_encoder_param_shapes(spec)}
    assert got == want
    dec = sum(v.numel() for k, v in m.state_dict().items() if k.startswith("decoder."))
    enc = sum(v.numel() for k, v in m.state_dict().items() if k.startswith("encoder."))
    assert (dec, enc, dec + enc) == (1_222_531, 1_222_532, 2_445_063)


def test_stage_lengths_are_free():
    cfg = to.tiny_config(num_encoder_blocks=(2, 1, 0), num_decoder_blocks=(0, 2, 1),
                         encoder_block_out_channels=(64,) * 3, decoder_block_out_channels=(64,) * 3)
    m = to.AutoencoderTiny(cfg)
    spec = taesd_spec_from_config(cfg)
    got = {**taesd_decoder_param_shapes(spec), **taesd_encoder_param_shapes(spec)}
    assert got == {k: tuple(v.shape) for k, v in m.state_dict().items()}


@pytest.mark.parametrize("key,value", [
    ("act_fn", "silu"), ("upsample_fn", "bilinear"), ("upsampling_scaling_factor", 4),
    ("decoder_block_out_channels", (64, 64, 128, 64)), ("encoder_block_out_channels", (32, 64, 64, 64)),
    ("latent_channels", 16), ("in_channels", 9), ("out_channels", 12)])
def test_refusals_name_the_key(key, value):
    with pytest.raises(NotImplementedError, match=key):
        taesd_spec_from_config(to.tiny_config(**{key: value}))


def _bytes(plan, io):
    seen, tot = set(), 0
    for t in list(plan._bufs.values()) + io:
        if id(t) not in seen:
            seen.add(id(t))
            tot += t.numel() * t.element_size()
    return tot


@pytest.mark.parametrize("h,w", [(64, 64), (128, 128), (104, 152), (13, 21)])
@pytest.mark.parametrize("batch", [1, 4])
def test_dry_decode_plan(h, w, batch):
    wts = _dry()
    plan = TAESDDecodePlan(wts, batch, h, w)
    names = [op.fn.name for op in plan.all_ops()]
    # conv_in, 3 convs per block (10 blocks), 3 upsampling convs, conv_out
    assert names == ["sfb_conv3x3_small_ex"] + ["sfb_conv3x3_c64"] * 33 + ["sfb_conv_out"]
    assert tuple(plan.out.shape) == (batch, 3, 8 * h, 8 * w)
    # per resolution: block input + ping-pong pair, 64 channels of 16 bits
    act = sum(3 * batch * (h << s) * (w << s) * 64 * 2 for s in range(4))
    assert _bytes(plan, [plan.z_in, plan.out]) == act + 2 * batch * (4 * h * w + 3 * 64 * h * w)
    c64 = 2 * 64 * 576
    want = (2 * batch * h * w * 64 * 9 * 4 + sum(c64 * batch * (h << s) * (w << s) * n
                                                  for s, n in enumerate((9, 10, 10, 4)))
            + 2 * batch * 64 * h * w * 64 * 9 * 3)
    assert plan.flops() == want


@pytest.mark.parametrize("h,w", [(512, 512), (1024, 1024), (832, 1216), (104, 168), (13, 21)])
@pytest.mark.parametrize("batch", [1, 4])
def test_dry_encode_plan(h, w, batch):
    plan = TAESDEncodePlan(_dry(), batch, h, w)
    names = [op.fn.name for op in plan.all_ops()]
    assert names == ["sfb_conv3x3_small_ex"] + ["sfb_conv3x3_c64"] * 33 + ["sfb_conv_out"]
    sizes = [(h, w)]
    for _ in range(3):
        sizes.append(((sizes[-1][0] + 1) // 2, (sizes[-1][1] + 1) // 2))
    assert tuple(plan.out.shape) == (batch, 4) + sizes[-1]
    x_bytes = sum(batch * a * b * 64 * 2 for a, b in sizes)
    pp = sum(2 * batch * a * b * 64 * 2 for (a, b), n in zip(sizes, (1, 3, 3, 3)) if n)
    io = 2 * batch * (3 * h * w + 4 * sizes[-1][0] * sizes[-1][1])
    assert _bytes(plan, [plan.x_in, plan.out]) == x_bytes + pp + io


def test_c64_op_checks_the_output_geometry():
    plan = TAESDDecodePlan(_dry(), 1, 8, 8)
    x = plan.act("t", 1, 8, 8, 64)
    with pytest.raises(ValueError, match="does not match"):
        ops.conv_c64_op("bad", plan.lib_or_dry(), x=x, weight=None, bias=None, y=plan.act("u", 1, 8, 8, 64),
                        mode=_lib.C64_UP2X, dt=torch.float16)


def test_c_abi_validation_without_a_gpu():
    lib = _lib.lib()
    import ctypes
    p = _lib.ConvC64Params()
    assert lib.sfb_conv3x3_c64(ctypes.byref(p), None) < 0
    p.x = p.weight = p.y = 1 << 20
    p.n, p.h, p.w, p.ldx, p.ldy, p.mode, p.dtype = 1, 8, 8, 64, 64, 3, 0
    assert lib.sfb_conv3x3_c64(ctypes.byref(p), None) < 0 and b"mode" in lib.sfb_last_error()
    p.mode, p.ldx = 0, 60
    assert lib.sfb_conv3x3_c64(ctypes.byref(p), None) < 0 and b"pitch" in lib.sfb_last_error()
    q = _lib.ConvSmallExParams()
    q.base.x = q.base.weight = q.base.y = 1 << 20
    q.base.n, q.base.h, q.base.w, q.base.cin, q.base.cout, q.base.stride, q.base.ldx, q.base.ldy = 1, 8, 8, 8, 64, 1, 8, 64
    q.in_xform = _lib.XFORM_TANH3
    assert lib.sfb_conv3x3_small_ex(ctypes.byref(q), None) < 0 and b"NCHW" in lib.sfb_last_error()


# ---------------------------------------------------------------------------------------------------------
# fp64 restatement of sfb_conv3x3_c64, written from include/sfb200.h: the source pixel each (output pixel,
# tap) reads, then the epilogue -- compared with F.conv2d / F.interpolate
# ---------------------------------------------------------------------------------------------------------
def c64_restated(x, w, bias, mode, residual=None, relu=False):
    """x [n, h, w, 64] NHWC, w [64, 3, 3, 64] (cout, kh, kw, cin) -> y NHWC, element by element over taps."""
    n, h, wd, _ = x.shape
    ho, wo = ops.c64_out_hw(mode, h, wd)
    y = torch.zeros(n, ho, wo, 64, dtype=torch.float64)
    oy = torch.arange(ho).view(-1, 1).expand(ho, wo)
    ox = torch.arange(wo).view(1, -1).expand(ho, wo)
    for ty in range(3):
        for tx in range(3):
            if mode == _lib.C64_STRIDE2:
                sy, sx = 2 * oy + ty - 1, 2 * ox + tx - 1
                valid = (sy >= 0) & (sy < h) & (sx >= 0) & (sx < wd)
            elif mode == _lib.C64_UP2X:
                uy, ux = oy + ty - 1, ox + tx - 1   # in the upsampled image
                valid = (uy >= 0) & (uy < 2 * h) & (ux >= 0) & (ux < 2 * wd)
                sy, sx = torch.div(uy, 2, rounding_mode="floor"), torch.div(ux, 2, rounding_mode="floor")
            else:
                sy, sx = oy + ty - 1, ox + tx - 1
                valid = (sy >= 0) & (sy < h) & (sx >= 0) & (sx < wd)
            src = x[:, sy.clamp(0, h - 1), sx.clamp(0, wd - 1), :] * valid[None, :, :, None]
            y += src @ w[:, ty, tx, :].T
    if bias is not None:
        y += bias
    if residual is not None:
        y += residual
    return y.clamp_min(0) if relu else y


@pytest.mark.parametrize("mode", [_lib.C64_SAME, _lib.C64_STRIDE2, _lib.C64_UP2X])
@pytest.mark.parametrize("h,w", [(1, 1), (7, 13), (10, 9)])
def test_c64_restatement_matches_torch(mode, h, w):
    g = torch.Generator().manual_seed(h * 100 + w + mode)
    x = torch.randn(2, 64, h, w, generator=g, dtype=torch.float64)
    wt = torch.randn(64, 64, 3, 3, generator=g, dtype=torch.float64) / 24
    b = torch.randn(64, generator=g, dtype=torch.float64)
    xn, wk = x.permute(0, 2, 3, 1), wt.permute(0, 2, 3, 1)
    if mode == _lib.C64_STRIDE2:
        ref = F.conv2d(x, wt, b, stride=2, padding=1)
    elif mode == _lib.C64_UP2X:
        ref = F.conv2d(F.interpolate(x, scale_factor=2, mode="nearest"), wt, b, padding=1)
    else:
        ref = F.conv2d(x, wt, b, padding=1)
    ref = ref.permute(0, 2, 3, 1)
    torch.testing.assert_close(c64_restated(xn, wk, b, mode), ref, rtol=1e-12, atol=1e-12)
    r = torch.randn(ref.shape, generator=g, dtype=torch.float64)
    torch.testing.assert_close(c64_restated(xn, wk, b, mode, residual=r, relu=True), (ref + r).relu(),
                               rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(c64_restated(xn, wk, None, mode, relu=True), (ref - b).relu(), rtol=1e-12, atol=1e-12)


# ---------------------------------------------------------------------------------------------------------
# compile_vae_module routing (stand-in modules; no GPU needed to install)
# ---------------------------------------------------------------------------------------------------------
def test_compile_installs_native_decode_and_encode_for_a_tiny_vae(caplog):
    from sfast_b200.runtime import CompiledTinyVAE, compile_vae_module
    m = to.AutoencoderTiny(to.tiny_config())
    with caplog.at_level(logging.WARNING):
        out = compile_vae_module(m)
    assert out is m
    assert isinstance(m.decode._compiled, CompiledTinyVAE) and m.encode._compiled is m.decode._compiled
    assert "eager path" not in caplog.text
    # fp32 calls go to the module's own methods (CPU: no GPU needed), with one warning
    z = torch.randn(1, 4, 3, 5)
    with caplog.at_level(logging.WARNING):
        a = m.decode(z, return_dict=False)[0]
        m.decode(z)
    assert torch.equal(a, to.AutoencoderTiny.decode(m, z).sample)
    assert caplog.text.count("tiny VAE decode left on the module's eager path") == 1
    lat = m.encode(torch.rand(1, 3, 16, 16) * 2 - 1).latents
    assert tuple(lat.shape) == (1, 4, 2, 2)


def test_compile_leaves_a_16_channel_tiny_vae_eager(caplog):
    from sfast_b200.runtime import compile_vae_module
    m = to.AutoencoderTiny(to.tiny_config(latent_channels=16))
    own_decode, own_encode = m.decode, m.encode
    with caplog.at_level(logging.WARNING):
        compile_vae_module(m)
    assert m.decode == own_decode and m.encode == own_encode
    assert "latent_channels=16" in caplog.text
    assert "decode is left on the module's eager path" in caplog.text


def test_autoencoder_kl_and_temporal_routing_is_unchanged():
    from oracle import svd_vae_oracle as svo
    from oracle import vae_encoder_oracle as veo
    from oracle import vae_oracle as vo
    from sfast_b200.runtime import CompiledTinyVAE, CompiledVAE, compile_vae_module, is_tiny_vae
    from test_svd_vae_decode_cpu import _StandInSVDVAE, _svd_sd
    m = veo.build_autoencoder_kl(vo.tiny_vae_config())
    assert not is_tiny_vae(m)
    compile_vae_module(m)
    assert type(m.decode._compiled) is CompiledVAE and m.encode._compiled is m.decode._compiled
    t = _StandInSVDVAE(_svd_sd(svo.tiny_svd_vae_config()))
    assert not is_tiny_vae(t)
    compile_vae_module(t)
    assert type(t.decode._compiled) is CompiledVAE and not isinstance(t.decode._compiled, CompiledTinyVAE)
