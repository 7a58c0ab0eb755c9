"""Host-side checks of the native VAE encode (`compile_vae` -> AutoencoderKL.encode): parameter layout,
the conv_out . quant_conv fold, the dry launch schedule and the C ABI's validation of the down-conv
mode (SFB_A_DOWNCONV3X3), the output types and the routing of VAEs whose decoder stays eager."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from oracle import vae_encoder_oracle as veo
from oracle import vae_oracle as vo
from sfast_b200 import _lib, ops
from sfast_b200.plan import PackedWeights
from sfast_b200.vae_plan import VAEEncodePlan, vae_encoder_param_shapes, vae_encoder_spec_from_config
from test_host_logic import _DUMMY_PTR, _clone, _nonnull, _validate_plan_on_cpu

_NO_GPU = pytest.mark.skipif(torch.cuda.is_available(), reason="needs a box without a GPU: launches must fail")


def _dry_encode_plan(cfg, batch, h, w):
    spec = vae_encoder_spec_from_config(cfg)
    sd = {k: torch.empty(v, dtype=torch.float16, device="meta") for k, v in vae_encoder_param_shapes(spec).items()}
    return VAEEncodePlan(PackedWeights(spec, sd, torch.float16, "meta", dry=True), batch, h, w)


def _gemms(plan):
    return [op.keep[0] for op in plan.all_ops() if op.fn is not None and op.fn.name == "sfb_gemm"]


def test_encoder_parameter_total_and_names_match_the_oracle():
    spec = vae_encoder_spec_from_config(vo.sd_vae_config())
    shapes = vae_encoder_param_shapes(spec)
    # diffusers' SD VAE (83,653,863) minus decoder + post_quant_conv (49,490,199)
    assert sum(torch.Size(s).numel() for s in shapes.values()) == 34_163_664
    with torch.device("meta"):
        m = veo.AutoencoderKL(vo.sd_vae_config())
    got = {k: tuple(v.shape) for k, v in m.state_dict().items() if k.startswith(("encoder.", "quant_conv."))}
    assert got == {k: tuple(v) for k, v in shapes.items()}
    assert sum(v.numel() for v in m.state_dict().values()) == 83_653_863


def test_conv_out_quant_conv_fold_equals_the_two_step_oracle_in_fp64():
    cfg = vo.tiny_vae_config()
    m = veo.build_autoencoder_kl(cfg, seed=5, dtype=torch.float64)
    x = torch.randn(2, cfg.block_out_channels[-1], 6, 10, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
    ref = m.quant_conv(m.encoder.conv_out(x))
    sd = m.state_dict()
    w, b = ops.fold_pointwise_into_conv(sd["encoder.conv_out.weight"], sd["encoder.conv_out.bias"],
                                        sd["quant_conv.weight"], sd["quant_conv.bias"])
    torch.testing.assert_close(F.conv2d(x, w, b, padding=1), ref, rtol=1e-12, atol=1e-12)
    # what the plan packs: that fold, weight in the compute type ([cout, (kh, kw, cin)]), bias in fp32
    pw = PackedWeights(vae_encoder_spec_from_config(cfg), sd, torch.float64, "cpu")
    wp, bp = pw.conv3x3_pointwise("encoder.conv_out", "quant_conv")
    assert torch.equal(wp, ops.pack_conv3x3(w, torch.float64)) and torch.equal(bp, b.float())
    # refresh() re-forms the fold in place after an in-place update of quant_conv
    ptr = wp.data_ptr()
    sd2 = {k: v.clone() for k, v in sd.items()}
    sd2["quant_conv.weight"] = sd2["quant_conv.weight"] * 2
    sd2["quant_conv.bias"] = sd2["quant_conv.bias"] * 2
    pw.refresh(sd2)
    assert wp.data_ptr() == ptr
    got2 = F.conv2d(x, wp.view(wp.shape[0], 3, 3, -1).permute(0, 3, 1, 2), bp.double(), padding=1)
    torch.testing.assert_close(got2, 2 * ref, rtol=1e-6, atol=1e-6)    # (fp32 bias)


@pytest.mark.parametrize("cfgf,batch,h,w", [
    (vo.sd_vae_config, 1, 512, 512), (vo.sd_vae_config, 2, 512, 768), (vo.sd_vae_config, 1, 576, 1024),
    (vo.tiny_vae_config, 2, 128, 192), (vo.tiny_vae_config, 1, 64, 64),
])
def test_encode_plan_schedule_and_host_validation(cfgf, batch, h, w):
    plan = _dry_encode_plan(cfgf(), batch, h, w)
    names = [op.fn.name for op in plan.all_ops() if op.fn is not None]
    assert names.count("sfb_row_softmax") == batch and names.count("sfb_conv_in") == 1
    assert names.count("sfb_conv_out") == 1
    down = [g for g in _gemms(plan) if g.a_mode == _lib.A_DOWNCONV3X3]
    assert len(down) == 3 and all(g.conv_stride == 2 and not g.rowbias for g in down)
    assert [(g.img_h, g.img_w) for g in down] == [(h // 2, w // 2), (h // 4, w // 4), (h // 8, w // 8)]
    assert not any(g.a_mode == _lib.A_CONV3X3 and g.conv_stride == 2 for g in _gemms(plan))
    assert tuple(plan.out.shape) == (batch, 8, h // 8, w // 8)
    if (cfgf, batch, h, w) == (vo.sd_vae_config, 1, 512, 512):
        assert 1.0e12 < plan.flops() < 1.2e12      # ~1.1 TFLOP by a hand count
        print("VAE encode 1x3x512x512: %.3f TFLOP, %d launches" % (plan.flops() / 1e12, len(names)))
    if not torch.cuda.is_available():
        n = _validate_plan_on_cpu(plan)
        assert n["sfb_gemm"] == len(_gemms(plan))
        lib = _lib.lib()
        op = next(op for op in plan.all_ops() if op.fn is not None and op.fn.name == "sfb_conv_out")
        y, wt, b, out, *geom = op.args
        assert (geom[3], geom[4]) == (cfgf().block_out_channels[-1], 8)
        # 512 -> 8 needs 72 KB of weights in shared memory: past validation, only the launch fails here
        rc = lib.sfb_conv_out(_DUMMY_PTR, _DUMMY_PTR, _DUMMY_PTR, _DUMMY_PTR, *geom, None)
        assert rc == -2, lib.sfb_last_error().decode()


@_NO_GPU
def test_sfb_conv_out_rejects_weights_past_the_shared_memory_limit():
    lib = _lib.lib()
    # 9 * 2048 * 8 * 2 B = 288 KB > 227 KB
    rc = lib.sfb_conv_out(_DUMMY_PTR, _DUMMY_PTR, _DUMMY_PTR, _DUMMY_PTR, 1, 8, 8, 2048, 8, 2048, 0, None)
    assert rc == -1 and b"227 KB" in lib.sfb_last_error()


@_NO_GPU
def test_sfb_gemm_rejects_bad_down_conv_arguments():
    lib = _lib.lib()
    g = next(g for g in _gemms(_dry_encode_plan(vo.sd_vae_config(), 1, 512, 512)) if g.a_mode == _lib.A_DOWNCONV3X3)

    def call(**changes):
        p = _clone(g)
        _nonnull(p, ["tmap_a", "tmap_b", "out", "ws"])
        for k, v in changes.items():
            setattr(p, k, v)
        return lib.sfb_gemm(ctypes.byref(p), None)

    assert call() == -2                                    # valid: fails only at the launch
    assert call(splits=4) == -2                            # split-K is allowed
    assert call(conv_stride=1) == -1
    assert call(K=9 * g.cin + 64) == -1
    assert call(K=4 * g.cin) == -1
    assert call(rowbias=_DUMMY_PTR, rows_per_img=g.img_h * g.img_w, ld_rowbias=g.N) == -1


@pytest.mark.parametrize("key,value,match", [
    ("down_block_types", ("DownEncoderBlock2D",) * 3 + ("DownBlock2D",), "down block type"),
    ("block_out_channels", (128, 256, 480, 512), "multiples of 64"),
    ("double_z", False, "double_z"),
    ("latent_channels", 16, "moments"),
])
def test_unsupported_encoder_configs_are_rejected_by_name(key, value, match):
    cfg = dict(vars(vo.sd_vae_config()), **{key: value})
    with pytest.raises(NotImplementedError, match=match):
        vae_encoder_spec_from_config(cfg)


@pytest.mark.parametrize("h,w", [(500, 512), (512, 508), (72, 64)])
def test_unsupported_image_sizes_raise(h, w):
    with pytest.raises(NotImplementedError):
        _dry_encode_plan(vo.sd_vae_config(), 1, h, w)


def test_latent_dist_stand_in_samples_like_diffusers():
    from sfast_b200.runtime import AutoencoderKLOutput, DiagonalGaussianDistribution
    moments = torch.randn(2, 8, 4, 6, dtype=torch.float64)
    moments[:, 4:5] = 40.0                                  # logvar clamped to 20
    d = DiagonalGaussianDistribution(moments)
    mean, logvar = moments[:, :4], moments[:, 4:].clamp(-30, 20)
    assert torch.equal(d.mode(), mean) and torch.equal(d.logvar, logvar)
    torch.testing.assert_close(d.std, torch.exp(0.5 * logvar))
    torch.testing.assert_close(d.var, torch.exp(logvar))
    s = d.sample(torch.Generator().manual_seed(3))
    eps = torch.randn(mean.shape, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    assert torch.equal(s, mean + d.std * eps)
    gens = [torch.Generator().manual_seed(i) for i in (4, 5)]
    s = d.sample([torch.Generator().manual_seed(i) for i in (4, 5)])
    eps = torch.cat([torch.randn((1, 4, 4, 6), generator=g, dtype=torch.float64) for g in gens])
    assert torch.equal(s, mean + d.std * eps)
    out = AutoencoderKLOutput(latent_dist=d)
    assert out.latent_dist is d and out["latent_dist"] is d and out[0] is d


class _StandInVAE:
    """The attributes compile_vae_module reads of a diffusers VAE."""

    def __init__(self, state_dict, with_encode=True):
        self.config = vars(vo.tiny_vae_config())
        self._sd = state_dict
        if with_encode:
            self.encode = lambda x, return_dict=True: "eager encode"

    def state_dict(self):
        return self._sd

    def decode(self, z, return_dict=True, num_frames=None):
        return "eager decode"


def test_temporal_decoder_keeps_its_own_decode_and_gets_a_native_encode():
    from sfast_b200.runtime import compile_vae_module, temporal_decoder
    spec = vae_encoder_spec_from_config(vo.tiny_vae_config())
    enc = {k: torch.empty(v, device="meta") for k, v in vae_encoder_param_shapes(spec).items()}
    svd = dict(enc, **{"decoder.conv_in.weight": torch.empty(512, 4, 3, 3, device="meta"),
                       "decoder.time_mix_conv.weight": torch.empty(3, 3, 3, 3, 3, device="meta")})
    kl = dict(enc, **{"post_quant_conv.weight": torch.empty(4, 4, 1, 1, device="meta")})
    assert temporal_decoder(svd) and not temporal_decoder(kl)

    m = _StandInVAE(svd)
    own_decode = m.decode
    compile_vae_module(m)
    assert m.decode == own_decode and m.decode(None, num_frames=14) == "eager decode"
    assert m.encode._compiled is not None

    m = _StandInVAE(kl)
    compile_vae_module(m)
    assert m.encode._compiled is m.decode._compiled and m.encode._cached is m.decode._cached

    m = _StandInVAE(kl, with_encode=False)               # decoder only (SyntheticVAE): no encode appears
    compile_vae_module(m)
    assert not hasattr(m, "encode") and m.decode._compiled is not None
