"""GPU checks of the native VAE encode: the down-conv kernel mode (SFB_A_DOWNCONV3X3) against
F.conv2d(F.pad(x, (0, 1, 0, 1)), w, stride=2) in fp32, sfb_conv_out at the encoder's 512 -> 8, and
`compile_vae(...).encode` against oracle/vae_encoder_oracle.py's AutoencoderKL with the two-sided bar of
tests/test_vae_gpu.py (no worse than 1.25 x the eager 16-bit oracle's error against fp32, plus an
absolute rms cap)."""
import math

import pytest
import torch
import torch.nn.functional as F

import kernel_checks as kc
from oracle import vae_encoder_oracle as veo
from oracle import vae_oracle as vo
from sfast_b200 import _lib, ops
from sfast_b200.ops import Act
from test_vae_gpu import TOL, _rel, _rms

pytestmark = pytest.mark.gpu


def check_downconv(n, h, w, cin, cout, dt=torch.float16, splits=None, pitch_extra=0, seed=61):
    """diffusers' Downsample2D(padding=0): pad one zero row / column after the image, 3x3 stride-2 conv."""
    lib = _lib.lib()
    torch.manual_seed(seed)
    ld = cin + pitch_extra
    x = Act(kc._rand(n, h, w, ld, dt=dt), n, h, w, cin, ld=ld)
    wt = kc._rand(cout, cin, 3, 3, dt=dt, scale=1 / math.sqrt(9 * cin))
    b = torch.randn(cout, device="cuda")
    ho, wo = h // 2, w // 2
    M = n * ho * wo
    out = torch.zeros(M, cout, device="cuda", dtype=dt)
    box_n, box_h, box_w = ops.conv_tile_box(ho, wo)
    ws = torch.empty(splits * M * cout, device="cuda", dtype=torch.float32) if splits else None
    op = ops.gemm_op("downconv", lib, a=ops.a_conv(x.ptr, n, h, w, cin, ld, box_n, box_h, box_w, 2),
                     b=ops.Mat(ops.pack_conv3x3(wt, dt)), M=M, N=cout, K=9 * cin, dt=dt, out=out, ldo=cout, bias=b,
                     ws=ws, splits=splits,
                     conv=dict(n=n, h=ho, w=wo, cin=cin, stride=2, box_n=box_n, box_h=box_h, box_w=box_w, down=True))
    p = op.keep[0]
    assert p.a_mode == _lib.A_DOWNCONV3X3 and p.splits == (splits or 1)
    op.launch(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    xin = x.tensor().permute(0, 3, 1, 2).float()
    ref = F.conv2d(F.pad(xin, (0, 1, 0, 1)), wt.float(), b, stride=2)
    return kc.rel_err(out, ref.permute(0, 2, 3, 1).reshape(M, cout)), (p.box_n, p.box_h, p.box_w)


@pytest.mark.parametrize("n,h,w,c,dt,splits,pitch_extra,tol", [
    (1, 512, 512, 128, torch.float16, None, 0, 2e-3),     # SD VAE level 0 -> 1
    (1, 256, 256, 256, torch.float16, None, 0, 2e-3),     # level 1 -> 2
    (1, 128, 128, 512, torch.float16, None, 0, 2e-3),     # level 2 -> 3
    (1, 576, 1024, 128, torch.float16, None, 0, 2e-3),    # SVD 576 x 1024 -> 288 x 512
    (2, 48, 40, 128, torch.float16, None, 0, 2e-3),       # output width 20: 2-D patches
    (2, 64, 64, 128, torch.float16, None, 64, 2e-3),      # input inside a wider concat buffer
    (1, 32, 32, 512, torch.float16, 4, 0, 2e-3),          # split-K
    (1, 128, 128, 256, torch.bfloat16, None, 0, 2e-2),
], ids=["sd_l0", "sd_l1", "sd_l2", "svd_576x1024", "patch_48x40", "concat_pitch", "splitk", "bf16"])
def test_down_conv_kernel(n, h, w, c, dt, splits, pitch_extra, tol):
    err, box = check_downconv(n, h, w, c, c, dt=dt, splits=splits, pitch_extra=pitch_extra)
    if (h, w) == (48, 40):
        assert box[2] < w // 2, box  # really tiled with 2-D patches
    assert err == err and err <= tol, f"rel err {err:.3e} > {tol}"


def test_symmetric_stride2_conv_is_unchanged():
    fn, tol = kc.CHECKS["conv_stride2"]
    err = fn()
    assert err == err and err <= tol, f"rel err {err:.3e} > {tol}"


def test_conv_out_512_to_8():
    err = kc.check_conv_out(n=2, h=64, w=64, cin=512, cout=8)
    assert err == err and err <= 2e-3, err


# ---------------------------------------------------------------------------------------------------
# whole encoder
# ---------------------------------------------------------------------------------------------------
def _compile(m, graph=True):
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_vae
    c = CompilationConfig.Default()
    c.enable_cuda_graph = graph
    return compile_vae(m, c)


def _triple(cfg, seed, dtype=torch.float16):
    oracle = veo.build_autoencoder_kl(cfg, seed=seed, dtype=torch.float32, device="cuda")
    fast = veo.build_autoencoder_kl(cfg, seed=seed, dtype=dtype, device="cuda")
    eager = veo.build_autoencoder_kl(cfg, seed=seed, dtype=dtype, device="cuda")
    oracle.load_state_dict({k: v.float() for k, v in fast.state_dict().items()})
    return oracle, fast, eager


def _image(b, h, w, seed, dtype):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.rand(b, 3, h, w, device="cuda", generator=g) * 2 - 1).to(dtype)


def _check(dist, oracle32, eager16, x, rms_cap, what):
    with torch.no_grad():
        ref = oracle32.encode(x.float()).latent_dist
        lib = eager16.encode(x).latent_dist
    for name, got, r, l in (("moments", dist.parameters, ref.parameters, lib.parameters),
                            ("mode", dist.mode(), ref.mode(), lib.mode())):
        e_ours, e_lib = _rel(got, r), _rel(l, r)
        r_ours, r_lib = _rms(got, r), _rms(l, r)
        print(f"{what} {name}: native {e_ours:.3e} (rms {r_ours:.3e}) | eager 16-bit {e_lib:.3e} (rms {r_lib:.3e})")
        assert got.shape == r.shape and got.dtype == x.dtype
        assert e_ours < max(TOL, 1.25 * e_lib), (what, name, e_ours, e_lib)
        assert r_ours < max(2e-3, 1.25 * r_lib) and r_ours < rms_cap, (what, name, r_ours, r_lib)


@pytest.mark.parametrize("graph", [False, True])
def test_tiny_vae_encode_vs_oracle(graph):
    cfg = vo.tiny_vae_config()
    oracle, fast, eager = _triple(cfg, seed=6)
    fast = _compile(fast, graph)
    for b, h, w in ((1, 64, 64), (2, 128, 192), (1, 64, 128)):
        x = _image(b, h, w, seed=b * 100 + h, dtype=torch.float16)
        dist = fast.encode(x).latent_dist
        assert dist.parameters.shape == (b, 8, h // 8, w // 8)
        _check(dist, oracle, eager, x, 1e-2, f"tiny VAE encode {b}x{h}x{w} graph={graph}")
    assert len(fast.encode._cached) == 3


@pytest.mark.parametrize("dtype,rms_cap", [(torch.float16, 1e-2), (torch.bfloat16, 6e-2)])
def test_sd_vae_encode_512(dtype, rms_cap):
    """The SD-1.5 VAE encoder at its pipeline shape: 3 x 512 x 512 image -> 8 x 64 x 64 moments."""
    oracle, fast, eager = _triple(vo.sd_vae_config(), seed=2, dtype=dtype)
    fast = _compile(fast, True)
    x = _image(1, 512, 512, seed=11, dtype=dtype)
    (dist,) = fast.encode(x, return_dict=False)
    _check(dist, oracle, eager, x, rms_cap, f"SD VAE encode 512x512 {dtype}")


def test_sd_vae_encode_576x1024():
    oracle, fast, eager = _triple(vo.sd_vae_config(), seed=3)
    fast = _compile(fast, True)
    x = _image(1, 576, 1024, seed=12, dtype=torch.float16)
    _check(fast.encode(x).latent_dist, oracle, eager, x, 1e-2, "SD VAE encode 576x1024 fp16")


def test_sample_replay_inplace_updates_and_decode_on_one_module():
    cfg = vo.tiny_vae_config()
    oracle, fast, eager = _triple(cfg, seed=8)
    fast = _compile(fast, True)
    x = _image(2, 64, 128, seed=5, dtype=torch.float16)
    d1 = fast.encode(x).latent_dist
    d2 = fast.encode(x).latent_dist
    assert torch.equal(d1.parameters, d2.parameters)           # graph replays are bitwise equal
    assert d1.parameters.data_ptr() != d2.parameters.data_ptr()  # fresh tensors, not the static buffer

    # sample(): mean + std * randn drawn like diffusers' randn_tensor (generator's device, moments' dtype)
    s = d1.sample(generator=torch.Generator(device="cuda").manual_seed(7))
    eps = torch.randn(d1.mean.shape, generator=torch.Generator(device="cuda").manual_seed(7), device="cuda",
                      dtype=torch.float16)
    assert torch.equal(s, d1.mean + d1.std * eps)

    # in-place updates of an encoder weight and of quant_conv reach the next encode, same graph
    n_graphs = len(fast.encode._cached)
    gp = next(iter(fast.encode._cached.values()))
    for mod in (fast, eager):
        with torch.no_grad():
            mod.encoder.down_blocks[1].resnets[0].conv1.weight.mul_(1.5)
            mod.quant_conv.weight.mul_(-0.5)
    oracle.load_state_dict({k: v.float() for k, v in fast.state_dict().items()})
    d3 = fast.encode(x).latent_dist
    assert len(fast.encode._cached) == n_graphs and next(iter(fast.encode._cached.values())) is gp
    assert not torch.equal(d3.parameters, d1.parameters)
    _check(d3, oracle, eager, x, 1e-2, "tiny VAE encode after in-place update")

    # decode on the same compiled module (shared weights and cache)
    z = d3.mode()
    got = fast.decode(z).sample
    with torch.no_grad():
        ref = oracle.decode(z.float()).sample
        lib = eager.decode(z).sample
    e_ours, e_lib = _rel(got, ref), _rel(lib, ref)
    print(f"decode after encode: native {e_ours:.3e} | eager 16-bit {e_lib:.3e}")
    assert e_ours < max(TOL, 1.25 * e_lib)
    assert fast.decode._compiled is fast.encode._compiled and len(fast.decode._cached) == n_graphs + 1


def test_fp32_encode_is_the_modules_eager_result():
    m = veo.build_autoencoder_kl(vo.tiny_vae_config(), seed=9, dtype=torch.float32, device="cuda")
    x = _image(1, 64, 64, seed=3, dtype=torch.float32)
    with torch.no_grad():
        want = m.encode(x).latent_dist.parameters
    m = _compile(m, True)
    with torch.no_grad():
        got = m.encode(x).latent_dist.parameters
    assert torch.equal(got, want) and len(m.encode._cached) == 0
