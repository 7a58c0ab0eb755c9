"""Host-side checks of the native temporal VAE decode (SVD's `AutoencoderKLTemporalDecoder.decode(z, num_frames)`):
parameter layout against the oracle, the switched AlphaBlender fold, the dry launch schedule and its buffer
total, the C ABI's validation of sfb_conv_out_temporal, an independent restatement of that kernel's
arithmetic, and the routing of `compile_vae_module`."""
import ctypes
import logging

import pytest
import torch
import torch.nn.functional as F

from oracle import svd_vae_oracle as svo
from sfast_b200 import _lib, ops
from sfast_b200.plan import PackedWeights
from sfast_b200.vae_plan import (TemporalDecodePlan, VAEDecodePlan, decoder_resnets, vae_decoder_param_shapes,
                                 vae_encoder_param_shapes, vae_spec_from_config, vae_temporal_decoder_param_shapes)
from test_host_logic import _DUMMY_PTR, _clone, _nonnull, _validate_plan_on_cpu

_NO_GPU = pytest.mark.skipif(torch.cuda.is_available(), reason="needs a box without a GPU: launches must fail")


def _meta_sd(shapes, dt=torch.float16):
    return {k: torch.empty(v, dtype=dt, device="meta") for k, v in shapes.items()}


def _dry_weights(cfg, shapes_fn):
    spec = vae_spec_from_config(cfg)
    return PackedWeights(spec, _meta_sd(shapes_fn(spec)), torch.float16, "meta", dry=True)


def _plan_bytes(plan):
    """Every device buffer a plan allocates: named buffers, statistics arenas, split-K workspace, I/O."""
    seen, tot = set(), 0
    tensors = list(plan._bufs.values()) + [plan.z_in, plan.out, plan.ln_arena]
    tensors += [getattr(plan, n) for n in ("gn_stats", "gn_sync", "gn_tickets") if hasattr(plan, n)]
    ws = getattr(plan._ws_token, "buf", None)
    if torch.is_tensor(ws):
        tensors.append(ws)
    for t in tensors:
        if id(t) not in seen:
            seen.add(id(t))
            tot += t.numel() * t.element_size()
    return tot


@pytest.mark.parametrize("cfgf", [svo.svd_vae_config, svo.tiny_svd_vae_config])
def test_oracle_parameter_names_and_shapes_match_the_spec(cfgf):
    cfg = cfgf()
    with torch.device("meta"):
        m = svo.AutoencoderKLTemporalDecoder(cfg)
    sd = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    spec = vae_spec_from_config(cfg)
    want = vae_temporal_decoder_param_shapes(spec)
    assert {k: v for k, v in sd.items() if k.startswith("decoder.")} == {k: tuple(v) for k, v in want.items()}
    # encoder + quant_conv are the 2-D VAE's: the native encode reads the same names
    assert {k: v for k, v in sd.items() if not k.startswith("decoder.")} == {
        k: tuple(v) for k, v in vae_encoder_param_shapes(spec).items()}
    assert "post_quant_conv.weight" not in sd
    n_dec = sum(torch.Size(v).numel() for v in want.values())
    n_2d = sum(torch.Size(v).numel() for k, v in vae_decoder_param_shapes(spec).items()
               if not k.startswith("post_quant_conv"))
    # each temporal resnet: 2 (3,1,1) convs + 2 GroupNorms + mix_factor; time_conv_out 3 x 3 x 3 + 3
    n_t = sum(2 * (3 * c * c + c) + 4 * c + 1 for _, _, c in decoder_resnets(spec)) + 30
    assert n_dec == n_2d + n_t
    print(f"{cfgf.__name__}: temporal decoder {n_dec:,} parameters ({n_t:,} temporal)")


def _blend_case(switched, seed=0):
    g = torch.Generator().manual_seed(seed)
    c, bf, f = 64, 6, 3
    conv = torch.nn.Conv3d(c, c, (3, 1, 1), padding=(1, 0, 0)).double()
    mix = torch.randn(1, generator=g, dtype=torch.float64) * 2
    sd = {"t.conv.weight": conv.weight.detach(), "t.conv.bias": conv.bias.detach(), "mix": mix}
    xs = torch.randn(bf // f, c, f, 4, 5, generator=g, dtype=torch.float64)
    a = torch.randn(bf // f, c, f, 4, 5, generator=g, dtype=torch.float64)
    # dry: Mat keeps the packed values but builds no TMA map
    pw = PackedWeights(vae_spec_from_config(svo.tiny_svd_vae_config()), sd, torch.float64, "cpu", dry=True)
    wm = pw.conv3x1_t("t.conv.weight", ("mix", switched))
    b = pw.f32_scaled("t.conv.bias", ("mix", switched))
    # the packed weight is K-major [cout, (kt, cin)] tiled into a Mat: undo the tiling through its logical rows
    nt, nkb = -(-c // ops.BN), wm.k // ops.BK
    w = wm.data.view(nt, nkb, ops.BN, ops.BK).permute(0, 2, 1, 3).reshape(nt * ops.BN, wm.k)[:c]
    w5 = w.view(c, 3, c).permute(0, 2, 1)[..., None, None]
    folded = xs + F.conv3d(a, w5, b.double(), padding=(1, 0, 0))
    return folded, xs, a, conv, mix


def test_sigma_fold_equals_the_switched_alpha_blender_and_fails_flipped():
    for seed in range(3):
        folded, xs, a, conv, mix = _blend_case(True, seed)
        blender = svo.AlphaBlender().double()
        with torch.no_grad():
            blender.mix_factor.copy_(mix)
            ref = blender(xs, xs + conv(a))
        torch.testing.assert_close(folded, ref, rtol=1e-6, atol=1e-6)   # (fp32 bias)
        flipped, *_ = _blend_case(False, seed)
        assert (flipped - ref).abs().max() > 1e-2


def test_svd_unet_fold_is_unchanged():
    """The SVD UNet's blend (not switched) still packs w * (1 - sigmoid(mix)), bit for bit."""
    g = torch.Generator().manual_seed(4)
    w = torch.randn(64, 64, 3, 1, 1, generator=g)
    bias, mix = torch.randn(64, generator=g), torch.randn(1, generator=g)
    sd = {"c.weight": w, "c.bias": bias, "mix": mix}
    pw = PackedWeights(vae_spec_from_config(svo.tiny_svd_vae_config()), sd, torch.float16, "cpu", dry=True)
    old = (w[:, :, :, 0, 0].permute(0, 2, 1).reshape(64, -1) * (1.0 - torch.sigmoid(mix))).half()
    assert torch.equal(pw.conv3x1_t("c.weight", ("mix", False)).data, ops.Mat(old.contiguous(), dry=True).data)
    assert torch.equal(pw.f32_scaled("c.bias", ("mix", False)), bias * (1.0 - torch.sigmoid(mix)))


@pytest.mark.parametrize("frames,num_frames", [(25, 25), (14, 14), (8, 8), (1, 1), (6, 3)])
def test_dry_plans_build_and_stay_within_the_2d_buffer_budget(frames, num_frames):
    h, w = 72, 128
    plan = TemporalDecodePlan(_dry_weights(svo.svd_vae_config(), vae_temporal_decoder_param_shapes),
                              frames, num_frames, h, w)
    names = [op.fn.name for op in plan.all_ops() if op.fn is not None]
    spec = plan.spec
    n_res = 2 + len(spec.block_out_channels) * (spec.layers_per_block + 1)
    temporal = [op.keep[0] for op in plan.all_ops() if op.fn is not None and op.fn.name == "sfb_gemm"
                and op.keep[0].a_mode == _lib.A_CONV3X1]
    assert len(temporal) == 2 * n_res
    assert all((g.img_n, g.img_h) == (frames // num_frames, num_frames) and g.splits == 1 for g in temporal)
    assert names.count("sfb_conv_out_temporal") == 1 and "sfb_conv_out" not in names
    assert names.count("sfb_row_softmax") == frames and names.count("sfb_conv_in") == 1
    assert "sfb_pointwise_nchw" not in names                       # no post_quant_conv
    assert tuple(plan.out.shape) == (frames, 3, 8 * h, 8 * w)
    op = next(op for op in plan.all_ops() if op.fn is not None and op.fn.name == "sfb_conv_out_temporal")
    assert op.args[6:13] == (frames, 8 * h, 8 * w, 128, 3, 128, num_frames)
    ref = VAEDecodePlan(_dry_weights(svo.svd_vae_config(), vae_decoder_param_shapes), frames, h, w)
    got, base = _plan_bytes(plan), _plan_bytes(ref)
    print(f"temporal decode {frames} frames (videos of {num_frames}) at {h}x{w}: {got / 1e9:.2f} GB of buffers, "
          f"2-D decode of {frames} latents {base / 1e9:.2f} GB ({got / base:.3f}x); {plan.flops() / 1e12:.2f} TFLOP, "
          f"{len(names)} launches")
    assert got <= 1.2 * base
    largest = max(t.numel() for t in plan._bufs.values())
    assert largest == frames * 8 * h * 8 * w * 256     # vae_ups2: 256 channels at the output size
    if not torch.cuda.is_available():
        n = _validate_plan_on_cpu(plan)
        assert n["sfb_gemm"] == names.count("sfb_gemm")
        lib = _lib.lib()
        rc = lib.sfb_conv_out_temporal(*[_DUMMY_PTR] * 6, *op.args[6:], None)
        assert rc == -2, lib.sfb_last_error().decode()


def test_tiny_plan_and_other_latent_sizes_build():
    wts = _dry_weights(svo.tiny_svd_vae_config(), vae_temporal_decoder_param_shapes)
    for frames, nf, h, w in ((2, 1, 8, 8), (6, 3, 8, 16), (16, 8, 16, 16), (3, 3, 40, 64)):
        plan = TemporalDecodePlan(wts, frames, nf, h, w)
        assert tuple(plan.out.shape) == (frames, 3, 8 * h, 8 * w)


@pytest.mark.parametrize("h,w", [(9, 7), (10, 10), (6, 6)])
def test_latents_the_attention_cannot_take_are_refused_by_name(h, w):
    wts = _dry_weights(svo.tiny_svd_vae_config(), vae_temporal_decoder_param_shapes)
    with pytest.raises(NotImplementedError, match="multiple of 64"):
        TemporalDecodePlan(wts, 2, 2, h, w)


@pytest.mark.parametrize("frames,nf", [(7, 3), (4, 0), (2, 4)])
def test_frames_that_are_not_whole_videos_are_refused(frames, nf):
    wts = _dry_weights(svo.tiny_svd_vae_config(), vae_temporal_decoder_param_shapes)
    with pytest.raises(ValueError, match=f"{frames} latents .*num_frames={nf}"):
        TemporalDecodePlan(wts, frames, nf, 8, 8)


@_NO_GPU
def test_sfb_conv_out_temporal_host_validation():
    lib = _lib.lib()
    P = [_DUMMY_PTR] * 6

    def call(n=6, h=8, w=8, cin=128, cout=3, ldx=128, frames=3, ptrs=P):
        return lib.sfb_conv_out_temporal(*ptrs, n, h, w, cin, cout, ldx, frames, 0, None)

    assert call() == -2                                   # valid: fails only at the launch
    assert call(cout=8, cin=64, ldx=72, frames=6) == -2
    assert call(n=7) == -1 and b"whole videos" in lib.sfb_last_error()
    assert call(frames=0) == -1
    assert call(cout=9) == -1 and call(cout=0) == -1
    assert call(cin=100) == -1 and call(ldx=120) == -1 and call(ldx=132) == -1
    assert call(cin=2048, cout=8, ldx=2048) == -1 and b"227 KB" in lib.sfb_last_error()
    assert call(ptrs=[_DUMMY_PTR] * 3 + [None] + [_DUMMY_PTR] * 2) == -1     # wt is required
    assert call(ptrs=[_DUMMY_PTR] * 4 + [None, _DUMMY_PTR]) == -2            # bt may be NULL
    assert call(n=25, h=65536, w=65536, frames=1) == -1 and b"2^31" in lib.sfb_last_error()


@_NO_GPU
def test_gemms_past_the_grid_limit_are_accepted_without_split_k():
    """25 frames at 576 x 1024: 115,200 M tiles, more than a grid's y extent; sfb_gemm runs such a GEMM as
    several launches, which it cannot do with split-K."""
    plan = TemporalDecodePlan(_dry_weights(svo.svd_vae_config(), vae_temporal_decoder_param_shapes), 25, 25, 72, 128)
    big = [op.keep[0] for op in plan.all_ops() if op.fn is not None and op.fn.name == "sfb_gemm"
           and op.keep[0].M > 65534 * 128]
    modes = {g.a_mode for g in big}
    assert {_lib.A_UPCONV2X, _lib.A_CONV3X1, _lib.A_MATRIX} <= modes and all(g.splits == 1 for g in big)
    lib = _lib.lib()
    for g in [g for g in big if g.a_mode != _lib.A_CONV3X3_GN][:4]:   # (that mode never takes split-K)
        p = _clone(g)
        _nonnull(p, ["tmap_a", "tmap_b", "out", "ws", "gn_scale_shift"])
        assert lib.sfb_gemm(ctypes.byref(p), None) == -2, lib.sfb_last_error().decode()
        p.splits = 2
        assert lib.sfb_gemm(ctypes.byref(p), None) == -1 and b"M tiles with split-K" in lib.sfb_last_error()


def _round16(t, dt):
    return t.to(dt).double()


def _kernel_restatement(x, w, b, wt, bt, frames, dt):
    """The kernel's arithmetic in fp64, written as it walks: per (video, pixel) a window of three conv_out
    values rounded to 16 bits; frames -1 and F contribute nothing."""
    n, cin, h, wd = x.shape
    cout = w.shape[0]
    xp = F.pad(x, (1, 1, 1, 1))
    # conv_out of every frame as an explicit sum over the 9 taps
    c = torch.zeros(n, cout, h, wd, dtype=torch.float64)
    for ky in range(3):
        for kx in range(3):
            c += torch.einsum("nchw,oc->nohw", xp[:, :, ky:ky + h, kx:kx + wd], w[:, :, ky, kx])
    c = _round16(c + b[None, :, None, None], dt)
    y = torch.empty_like(c)
    for v in range(n // frames):
        prev = torch.zeros(cout, h, wd, dtype=torch.float64)
        for f in range(frames):
            cur = c[v * frames + f]
            nxt = c[v * frames + f + 1] if f + 1 < frames else torch.zeros_like(cur)
            y[v * frames + f] = bt[:, None, None] + sum(
                torch.einsum("oc,chw->ohw", wt[:, :, k], win) for k, win in enumerate((prev, cur, nxt)))
            prev = cur
    return y


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("n,frames,cout", [(6, 3, 3), (2, 1, 1), (5, 5, 8), (4, 2, 3)])
def test_kernel_restatement_equals_conv3d_of_conv2d(dt, n, frames, cout):
    g = torch.Generator().manual_seed(n * 10 + frames)
    cin, h, wd = 16, 5, 7
    x = _round16(torch.randn(n, cin, h, wd, generator=g, dtype=torch.float64), dt)
    w = _round16(torch.randn(cout, cin, 3, 3, generator=g, dtype=torch.float64) / 12, dt)
    b = torch.randn(cout, generator=g, dtype=torch.float64)
    wt = _round16(torch.randn(cout, cout, 3, 1, 1, generator=g, dtype=torch.float64) / 3, dt)
    bt = torch.randn(cout, generator=g, dtype=torch.float64)
    ref = svo._frames(F.conv3d(svo._videos(_round16(F.conv2d(x, w, b, padding=1), dt), frames), wt, bt,
                               padding=(1, 0, 0)))
    got = _kernel_restatement(x, w, b, wt[:, :, :, 0, 0], bt, frames, dt)
    torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)
    # what the plan packs for time_conv_out: [cout, 3, cin] in the compute type
    pw = PackedWeights(vae_spec_from_config(svo.tiny_svd_vae_config()), {"t.weight": wt}, dt, "cpu")
    assert torch.equal(pw.time_conv_out("t.weight").double(), wt[:, :, :, 0, 0].permute(0, 2, 1))


class _StandInSVDVAE:
    """The attributes compile_vae_module reads of diffusers' AutoencoderKLTemporalDecoder."""

    def __init__(self, state_dict):
        self.config = vars(svo.tiny_svd_vae_config())
        self._sd = state_dict
        self.encode = lambda x, return_dict=True: "eager encode"
        self.calls = []

    def state_dict(self):
        return self._sd

    def decode(self, z, num_frames, return_dict=True):
        self.calls.append((z.dtype, num_frames))
        return "eager decode"


def _svd_sd(cfg, dt=torch.float16, device="meta"):
    spec = vae_spec_from_config(cfg)
    shapes = dict(vae_encoder_param_shapes(spec), **vae_temporal_decoder_param_shapes(spec))
    return {k: torch.empty(v, dtype=dt, device=device) for k, v in shapes.items()}


def test_compile_installs_the_native_temporal_decode_only_for_a_complete_decoder(caplog):
    from sfast_b200.runtime import compile_vae_module, temporal_decoder
    sd = _svd_sd(svo.tiny_svd_vae_config())
    assert temporal_decoder(sd)
    m = _StandInSVDVAE(sd)
    own = m.decode
    compile_vae_module(m)
    assert m.decode != own and m.decode._compiled is m.encode._compiled and m.decode._cached is m.encode._cached
    assert m.decode._compiled._eager == own
    # one missing or mis-shaped parameter: the module keeps its own decode
    for change in ("drop", "shape"):
        sd2 = dict(sd)
        k = "decoder.up_blocks.1.resnets.2.time_mixer.mix_factor"
        if change == "drop":
            del sd2[k]
        else:
            sd2[k] = torch.empty(2, device="meta")
        m = _StandInSVDVAE(sd2)
        own = m.decode
        with caplog.at_level(logging.WARNING):
            compile_vae_module(m)
        assert m.decode == own and m.encode._compiled is not None
        assert "decode is left on the module's eager path" in caplog.text


def test_decode_refusals_and_routing_without_a_gpu(caplog):
    from sfast_b200.runtime import compile_vae_module
    m = _StandInSVDVAE(_svd_sd(svo.tiny_svd_vae_config()))
    compile_vae_module(m)
    # fp32 latents go to the module's own decode, with one warning
    z32 = torch.zeros(4, 4, 8, 8)
    with caplog.at_level(logging.WARNING):
        assert m.decode(z32, num_frames=2) == "eager decode"
        assert m.decode(z32, 4) == "eager decode"
    assert m.calls == [(torch.float32, 2), (torch.float32, 4)]
    assert caplog.text.count("VAE decode in torch.float32") == 1
    # frames that are not whole videos: ValueError naming both numbers
    z = torch.zeros(7, 4, 8, 8, dtype=torch.float16)
    with pytest.raises(ValueError, match="7 latent frames with num_frames=3"):
        m.decode(z, num_frames=3)
    with pytest.raises(ValueError, match="num_frames=0"):
        m.decode(z, 0)
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="sm_90"):           # no eager fall-back for 16-bit latents
            m.decode(torch.zeros(6, 4, 8, 8, dtype=torch.float16), num_frames=3)
