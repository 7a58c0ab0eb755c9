"""GPU checks of the native temporal VAE decode (SVD's `AutoencoderKLTemporalDecoder.decode(z, num_frames)`):
sfb_conv_out_temporal against float64, every distinct launch of a moderate plan replayed against float64, the
whole decoder against oracle/svd_vae_oracle.py with the rule of tests/test_vae_gpu.py (no worse than 1.25 x
the same module run eagerly in the same 16-bit type, rms below 1e-2 in fp16 / 6e-2 in bf16), the default
25-frame chunk (tensors past 2^31 elements) against the eager module, and the runtime's behaviour."""
import pytest
import torch
import torch.nn.functional as F

import plan_launches as pl
from oracle import svd_vae_oracle as svo
from sfast_b200 import _lib, ops
from sfast_b200.plan import PackedWeights
from sfast_b200.vae_plan import TemporalDecodePlan, vae_spec_from_config, vae_temporal_decoder_param_shapes
from test_vae_gpu import TOL, _rel, _rms

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENT = 0x7E11


# ---------------------------------------------------------------------------------------- the kernel
def _ref_tail(x, w, b, wt, bt, frames, dt):
    """float64: time_conv_out(round16(conv_out(x))) over videos of `frames` frames; x NHWC [n, h, w, cin]."""
    c = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), b.double(), padding=1).to(dt).double()
    v = svo._videos(c, frames)
    return svo._frames(F.conv3d(v, wt.double()[..., None, None], bt.double(), padding=(1, 0, 0)))


def run_conv_out_temporal(n, frames, h, w, cin, cout, ldx, dt, seed=0):
    """One sfb_conv_out_temporal launch on fresh inputs (x at channel pitch ldx, output between guard bands):
    (relative error against float64, guard bands intact)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    xb = torch.randn(n * h * w, ldx, device=DEV, generator=g).to(dt)
    x = xb[:, :cin].view(n, h, w, cin)
    wc = (torch.randn(cout, cin, 3, 3, device=DEV, generator=g) / (3 * cin ** 0.5)).to(dt)
    bc = torch.randn(cout, device=DEV, generator=g)
    wt = (torch.randn(cout, cout, 3, device=DEV, generator=g) / (3 * cout) ** 0.5).to(dt)
    bt = torch.randn(cout, device=DEV, generator=g)
    guard = 4096
    yb = torch.empty(n * cout * h * w + 2 * guard, dtype=torch.int16, device=DEV).fill_(SENT)
    y = yb[guard:guard + n * cout * h * w].view(dt).view(n, cout, h, w)
    wp = ops.pack_conv3x3(wc, dt)
    wtp = wt.permute(0, 2, 1).contiguous()
    lib = _lib.lib()
    _lib.check(lib.sfb_conv_out_temporal(xb.data_ptr(), wp.data_ptr(), bc.data_ptr(), wtp.data_ptr(), bt.data_ptr(),
                                         y.data_ptr(), n, h, w, cin, cout, ldx, frames, ops.dtype_code(dt),
                                         torch.cuda.current_stream().cuda_stream), "sfb_conv_out_temporal")
    torch.cuda.synchronize()
    ref = _ref_tail(x, wc, bc, wt, bt, frames, dt)
    err = ((y.double() - ref).abs().max() / ref.abs().max()).item()
    intact = bool((yb[:guard] == SENT).all() and (yb[-guard:] == SENT).all())
    return err, intact


def _tol(dt):
    # one 16-bit rounding of the output, and at most one of the intermediate (fp32 vs fp64 sums)
    return 2e-3 if dt == torch.float16 else 1.6e-2


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("frames,videos", [(1, 3), (2, 2), (8, 2), (25, 1), (25, 2)])
@pytest.mark.parametrize("cin,cout,ldx", [(64, 1, 64), (128, 3, 136), (256, 8, 256), (128, 3, 128)])
def test_conv_out_temporal_matches_float64(dt, frames, videos, cin, cout, ldx):
    err, intact = run_conv_out_temporal(frames * videos, frames, 12, 20, cin, cout, ldx, dt,
                                        seed=frames * 7 + cin + cout)
    print(f"conv_out_temporal F={frames} videos={videos} {cin}->{cout} ldx={ldx} {dt}: {err:.2e}")
    assert err < _tol(dt) and intact


# ---------------------------------------------------------------------------------------- distinct launches
def test_every_distinct_launch_of_a_temporal_plan_matches_float64():
    """SVD-XT widths, 3 frames at a 40 x 64 latent (two videos): every distinct launch replayed on fresh inputs."""
    spec = vae_spec_from_config(svo.svd_vae_config())
    shapes = vae_temporal_decoder_param_shapes(spec)
    sd = {k: torch.empty(v, dtype=torch.float16, device="meta") for k, v in shapes.items()}
    with pl.recording_map_offsets():
        plan = TemporalDecodePlan(PackedWeights(spec, sd, torch.float16, "meta", dry=True), 6, 3, 40, 64)
    # pl.launches() keys the entry points plan_launches.py knows; the new tail kernel is replayed here
    tail = [op for op in plan.all_ops() if op.fn is not None and op.fn.name == "sfb_conv_out_temporal"]
    entries, names = {}, set()
    for op in plan.all_ops():
        if op.fn is None or op in tail:
            continue
        names.add(op.fn.name)
        if op.fn.name not in pl.SKIP:
            entries.setdefault(pl.launch_key(op), dict(op=op, name=op.fn.name, plans=["svd_vae_decode"]))
    assert not pl.check_coverage(names) and len(tail) == 1
    failures, n = [], 0
    a = tail[0].args   # (x, w, bias, wt, bt, y, n, h, wd, cin, cout, ldx, frames, dtype)
    err, intact = run_conv_out_temporal(a[6], a[12], a[7], a[8], a[9], a[10], a[11], torch.float16)
    if not (err < _tol(torch.float16) and intact):
        failures.append(f"conv_out_temporal: {err}, guard intact {intact}")
    for rec in pl.run_keys(entries, list(entries)):
        n += 1
        if not rec["ok"]:
            failures.append(f"{rec['desc']} peaked={rec['peaked']}: {rec.get('error') or rec['parts']}")
    print(f"temporal decode 6x3 at 40x64: {len(entries) + 1} distinct launches, {n + 1} replays")
    assert not failures, "\n".join(failures)


# ---------------------------------------------------------------------------------------- whole decoder
def _compile(m, graph=True):
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_vae
    c = CompilationConfig.Default()
    c.enable_cuda_graph = graph
    return compile_vae(m, c)


def _models(cfg, seed, dtype, oracle=True):
    fast = svo.build_svd_vae(cfg, seed=seed, dtype=dtype, device=DEV)
    eager = svo.build_svd_vae(cfg, seed=seed, dtype=dtype, device=DEV)
    ref = None
    if oracle:
        ref = svo.build_svd_vae(cfg, seed=seed, dtype=torch.float32, device=DEV)
        ref.load_state_dict({k: v.float() for k, v in fast.state_dict().items()})
    return ref, fast, eager


def _refs(oracle32, eager16, z, nf):
    with torch.no_grad():
        return oracle32.decode(z.float(), nf).sample, eager16.decode(z, nf).sample


def _check(got, ref, lib, rms_cap, what):
    e_ours, e_lib = _rel(got, ref), _rel(lib, ref)
    r_ours, r_lib = _rms(got, ref), _rms(lib, ref)
    print(f"{what}: native {e_ours:.3e} (rms {r_ours:.3e}) | eager 16-bit {e_lib:.3e} (rms {r_lib:.3e})")
    assert got.shape == ref.shape
    assert e_ours < max(TOL, 1.25 * e_lib), (what, e_ours, e_lib)
    assert r_ours < max(2e-3, 1.25 * r_lib) and r_ours < rms_cap, (what, r_ours, r_lib)


@pytest.mark.parametrize("graph", [False, True])
def test_tiny_temporal_decode_vs_oracle(graph):
    oracle, fast, eager = _models(svo.tiny_svd_vae_config(), 3, torch.float16)
    fast = _compile(fast, graph)
    for nf, h, w in ((1, 16, 16), (3, 8, 16), (8, 16, 24)):
        g = torch.Generator(device=DEV).manual_seed(nf * 100 + h)
        z = torch.randn(2 * nf, 4, h, w, device=DEV, generator=g).half()      # two videos
        ref, lib = _refs(oracle, eager, z, nf)
        got = fast.decode(z, num_frames=nf).sample
        assert got.shape == (2 * nf, 3, 8 * h, 8 * w)
        _check(got, ref, lib, 1e-2, f"tiny temporal decode 2 x {nf} frames {h}x{w} graph={graph}")


@pytest.mark.parametrize("dtype,rms_cap", [(torch.float16, 1e-2), (torch.bfloat16, 6e-2)])
def test_tiny_temporal_decode_dtypes(dtype, rms_cap):
    oracle, fast, eager = _models(svo.tiny_svd_vae_config(), 5, dtype)
    fast = _compile(fast)
    z = torch.randn(6, 4, 16, 16, device=DEV, generator=torch.Generator(DEV).manual_seed(2)).to(dtype)
    ref, lib = _refs(oracle, eager, z, 3)
    _check(fast.decode(z, 3, return_dict=False)[0], ref, lib, rms_cap, f"tiny temporal decode {dtype}")


def test_svd_xt_decode_8_frames_576x1024():
    """The pipeline's shape at decode_chunk_size=8: 8 latent frames of 72 x 128 -> 8 x 3 x 576 x 1024."""
    oracle, fast, eager = _models(svo.svd_vae_config(), 1, torch.float16)
    z = (torch.randn(8, 4, 72, 128, device=DEV, generator=torch.Generator(DEV).manual_seed(9)) / 0.18215 * 0.2).half()
    ref, lib = _refs(oracle, eager, z, 8)
    ref, lib = ref.cpu(), lib.cpu()
    del oracle, eager
    torch.cuda.empty_cache()
    fast = _compile(fast)
    got = fast.decode(z, num_frames=8).sample.cpu()
    _check(got, ref, lib, 1e-2, "SVD-XT VAE decode 8 frames 576x1024 fp16")


def test_svd_xt_decode_25_frames_past_2_31_elements():
    """The default chunk (25 frames of 576 x 1024): vae_ups2 holds 3.77e9 elements, so every launch past the
    last up-sampler addresses tensors beyond 2^31 elements.  Checked against the eager 16-bit module (the
    fp32 oracle does not fit next to it), overall and on the last frames alone."""
    _, fast, eager = _models(svo.svd_vae_config(), 2, torch.float16, oracle=False)
    z = (torch.randn(25, 4, 72, 128, device=DEV, generator=torch.Generator(DEV).manual_seed(4)) / 0.18215 * 0.2).half()
    with torch.no_grad():
        lib = eager.decode(z, 25).sample.cpu()
    del eager
    torch.cuda.empty_cache()
    fast = _compile(fast)
    got = fast.decode(z, num_frames=25).sample.cpu()
    r_all, r_last = _rms(got, lib), _rms(got[-3:], lib[-3:])
    e_last = _rel(got[-1:], lib[-1:])
    print(f"SVD-XT decode 25 frames vs eager fp16: rms {r_all:.3e}, last 3 frames rms {r_last:.3e}, "
          f"last frame max-rel {e_last:.3e}")
    assert r_all < 1e-2 and r_last < 1e-2 and e_last < 5e-2


# ---------------------------------------------------------------------------------------- runtime behaviour
def test_pipeline_chunks_dtype_round_trip_replays_and_in_place_updates():
    cfg = svo.tiny_svd_vae_config()
    oracle, fast, eager = _models(cfg, 7, torch.float16)
    fast = _compile(fast)
    assert fast.decode._compiled is fast.encode._compiled
    z = torch.randn(25, 4, 16, 16, device=DEV, generator=torch.Generator(DEV).manual_seed(1)).half()
    # StableVideoDiffusionPipeline.decode_latents with decode_chunk_size=8: chunks of 8, 8, 8 and 1 frames
    outs = []
    for i in range(0, 25, 8):
        zc = z[i:i + 8]
        got = fast.decode(zc, num_frames=zc.shape[0]).sample
        ref, lib = _refs(oracle, eager, zc, zc.shape[0])
        _check(got, ref, lib, 1e-2, f"chunk {i // 8} ({zc.shape[0]} frames)")
        outs.append(got)
    assert len(fast.decode._cached) == 2
    assert all(k[0] == "decode_t" for k in fast.decode._cached)
    # replays are bit-identical
    assert torch.equal(fast.decode(z[:8], 8).sample, outs[0])
    # in-place updates of a temporal conv weight and of a mix_factor reach the next call
    t = "decoder.up_blocks.3.resnets.1"
    prev = outs[0]
    for name, update in ((f"{t}.temporal_res_block.conv2.weight", lambda p: p.mul_(-1.5)),
                         (f"{t}.time_mixer.mix_factor", lambda p: p.add_(2.0))):
        with torch.no_grad():
            p = dict(fast.named_parameters())[name]
            update(p)
            dict(oracle.named_parameters())[name].copy_(p.float())
            dict(eager.named_parameters())[name].copy_(p)
        got = fast.decode(z[:8], 8).sample
        assert not torch.equal(got, prev)
        ref, lib = _refs(oracle, eager, z[:8], 8)
        _check(got, ref, lib, 1e-2, f"after an in-place update of {name}")
        prev = got
    # the pipeline upcasts the VAE around its encode and casts it back: still native, same result
    fast.to(torch.float32)
    fast.to(torch.float16)
    n_cached = len(fast.decode._cached)
    assert torch.equal(fast.decode(z[:8], 8).sample, prev)
    assert fast.decode._compiled is fast.encode._compiled and len(fast.decode._cached) == n_cached
