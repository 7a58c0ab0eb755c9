"""PEFT LoRA on an H100: sfb_lora_merge against float64, whole-model parity of merged adapters against the
unfused fp32 oracle, the adapter lifecycle on one compiled UNet (same graph throughout), the CLIP text encoder,
and compile() on a pipeline."""
import copy
import types

import pytest
import torch

from oracle import lora_oracle as lo
from oracle import unet_oracle as uo
from sfast_b200 import _lib, ops
from test_ip_adapter_gpu import MODEL_TOL, _rel
from test_lora_cpu import merge_reference

pytestmark = pytest.mark.gpu
torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False
DEV = "cuda:0"
DTS = (torch.float16, torch.bfloat16, torch.float32)


def _ulp(x, dt):
    """One unit in the last place of the 16-bit values x (as fp64)."""
    mant, emin = (10, -14) if dt == torch.float16 else (7, -126)
    e = torch.floor(torch.log2(x.double().abs().clamp_min(2.0 ** emin))).clamp_min(emin)
    return torch.exp2(e - mant)


def _merge_case(n, k, ranks, w_dt, a_dt, b_dt, out_dt, pitch_gap=0, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    wbuf = torch.randn(n, k + pitch_gap, device=DEV, generator=g).to(w_dt)
    w = wbuf[:, :k]
    ads = []
    for i, r in enumerate(ranks):
        a = torch.randn(r, k + pitch_gap, device=DEV, generator=g).to(a_dt)[:, :k] / r ** 0.5
        b = torch.randn(n, r + pitch_gap, device=DEV, generator=g).to(b_dt)[:, :r] / 4
        ads.append((a, b, 0.5 + 0.75 * i - (i == 2)))
    guard = 7
    obuf = torch.full((n + 1, k + pitch_gap + guard), 1234.0, device=DEV, dtype=out_dt)
    out = obuf[:n, :k]
    p = ops.lora_merge_params(w, ads, out)
    _lib.check(_lib.lib().sfb_lora_merge(ctypes_byref(p), torch.cuda.current_stream().cuda_stream), "merge")
    torch.cuda.synchronize()
    ref64 = w.double() + sum(s * (b.double() @ a.double()) for a, b, s in ads)
    ref = ref64.to(out_dt)
    # one ulp of the output, plus the worst-case error of the fp32 sums (R + 1 terms, R = total rank) where they
    # cancel to below what fp32 resolves: |fl(sum) - sum| <= (R + 1) * 2^-24 * sum of |terms|
    mag = w.double().abs() + sum(abs(s) * (b.double().abs() @ a.double().abs()) for a, b, s in ads)
    bound = _ulp(ref, out_dt) + (sum(ranks) + 1) * 2.0 ** -24 * mag
    err = (out.double() - ref64).abs() - (ref.double() - ref64).abs()
    assert (err <= bound).all(), (n, k, ranks, w_dt, a_dt, b_dt, out_dt)
    # guard bands: nothing outside out[:n, :k] is written
    mask = torch.ones_like(obuf, dtype=torch.bool)
    mask[:n, :k] = False
    assert (obuf[mask] == 1234.0).all()
    assert torch.equal(merge_reference(w, ads, out_dt), ref)


def ctypes_byref(p):
    import ctypes
    return ctypes.byref(p)


@pytest.mark.parametrize("rank", [1, 4, 64, 128, 256])
@pytest.mark.parametrize("out_dt", [torch.float16, torch.bfloat16])
def test_lora_merge_matches_float64_within_one_ulp(rank, out_dt):
    i = 0
    for w_dt in DTS:
        for a_dt in DTS:
            for b_dt in DTS:
                n, k = [(320, 36), (77, 200), (1280, 2880)][i % 3]
                _merge_case(n, k, [rank] * (1 + i % 4), w_dt, a_dt, b_dt, out_dt, pitch_gap=8 * (i % 2), seed=i)
                i += 1


# ---------------------------------------------------------------------------------------------------
# whole model
# ---------------------------------------------------------------------------------------------------
def _compile(m, graph=True, preserve=True):
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_unet
    cc = CompilationConfig.Default()
    cc.enable_cuda_graph, cc.preserve_parameters = graph, preserve
    return compile_unet(m, cc)


def _inputs(cfg, b, h, dt, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    s = torch.randn(b, 4, h, h, device=DEV, generator=g).to(dt)
    e = torch.randn(b, 77, cfg.cross_attention_dim, device=DEV, generator=g).to(dt)
    kw = {}
    if cfg.addition_embed_type == "text_time":
        kw = dict(added_cond_kwargs=dict(
            text_embeds=torch.randn(b, 1280, device=DEV, generator=g).to(dt),
            time_ids=torch.tensor([[h * 8, h * 8, 0, 0, h * 8, h * 8]] * b, device=DEV, dtype=dt)))
    return s, torch.tensor(500, device=DEV), e, kw


def _pair(cfg, dt, r=8, alpha=16, seed=3, targets="all"):
    fast = lo.inject_adapter(uo.build_unet(cfg, seed=seed, dtype=dt, device=DEV), "a", targets, r=r,
                             lora_alpha=alpha, seed=seed)
    oracle = lo.inject_adapter(uo.build_unet(cfg, seed=seed, dtype=torch.float32, device=DEV), "a", targets, r=r,
                               lora_alpha=alpha, seed=seed)
    return fast, oracle


def _ref(oracle, s, t, e, kw, **call):
    f32 = {k: {kk: vv.float() for kk, vv in v.items()} for k, v in kw.items()}
    scale = (call.get("cross_attention_kwargs") or {}).get("scale", 1.0)
    with torch.no_grad():
        lo.scale_lora_layers(oracle, scale)
        out = oracle(s.float(), t, e.float(), **f32).sample
        lo.unscale_lora_layers(oracle, scale)
    return out


def _adapter_free(oracle, s, t, e, kw):
    lo.disable_lora(oracle)
    out = _ref(oracle, s, t, e, kw)
    lo.enable_lora(oracle)
    return out


@pytest.mark.parametrize("graph", [True, False])
def test_tiny_unet_parity_and_the_adapter_moves_the_output(graph):
    cfg, dt = uo.tiny_config(), torch.float16
    fast, oracle = _pair(cfg, dt)
    fast = _compile(fast, graph)
    s, t, e, kw = _inputs(cfg, 2, 32, dt)
    ref = _ref(oracle, s, t, e, kw)
    got = fast(s, t, e).sample
    assert _rel(got, ref) <= MODEL_TOL[dt]
    assert _rel(_adapter_free(oracle, s, t, e, kw), ref) > 10 * MODEL_TOL[dt]
    got = fast(s, t, e, cross_attention_kwargs={"scale": 0.5}).sample
    assert _rel(got, _ref(oracle, s, t, e, kw, cross_attention_kwargs={"scale": 0.5})) <= MODEL_TOL[dt]


def test_two_adapters_and_per_block_weights():
    cfg, dt = uo.tiny_config(), torch.float16
    fast, oracle = _pair(cfg, dt)
    for m in (fast, oracle):
        lo.inject_adapter(m, "b", ["to_q", "to_k", "to_v", "to_out.0", "conv1", "conv2", "proj_out"], r=16,
                          lora_alpha=8, seed=11)
    fast = _compile(fast)
    s, t, e, kw = _inputs(cfg, 2, 32, dt)
    for weights in ([0.7, 0.3], [{"down_blocks.1": 0.0, "up_blocks.2": 2.0, "mid_block": -1.0}, 0.4]):
        for m in (fast, oracle):
            lo.set_adapters(m, ["a", "b"], weights)
        assert _rel(fast(s, t, e).sample, _ref(oracle, s, t, e, kw)) <= MODEL_TOL[dt], weights


@pytest.mark.parametrize("name,h,dt,layers", [("sd15", 64, torch.float16, 282), ("sdxl", 16, torch.bfloat16, 794)])
def test_published_unets_with_a_rank_64_adapter_on_every_weight(name, h, dt, layers):
    cfg = uo.sd15_config() if name == "sd15" else uo.sdxl_config()
    fast, oracle = _pair(cfg, dt, r=64, alpha=64)
    assert len(lo.lora_layers(fast)) == layers
    fast = _compile(fast)
    s, t, e, kw = _inputs(cfg, 2, h, dt)
    ref = _ref(oracle, s, t, e, kw)
    err = _rel(fast(s, t, e, **kw).sample, ref)
    print(f"{name}: rel err {err:.3e}")
    assert err <= MODEL_TOL[dt]
    assert _rel(_adapter_free(oracle, s, t, e, kw), ref) > 10 * MODEL_TOL[dt]


def test_lifecycle_on_one_compiled_unet_keeps_its_graph():
    cfg, dt = uo.tiny_config(), torch.float16
    fast = _compile(uo.build_unet(cfg, seed=3, dtype=dt, device=DEV))
    oracle = uo.build_unet(cfg, seed=3, dtype=torch.float32, device=DEV)
    s, t, e, kw = _inputs(cfg, 2, 32, dt)
    free = fast(s, t, e).sample
    compiled = fast.forward._compiled
    graph = next(iter(fast.forward._cached.values())).graph
    tol = MODEL_TOL[dt]

    def check(**call):
        got = fast(s, t, e, **call).sample
        assert _rel(got, _ref(oracle, s, t, e, kw, **call)) <= tol
        assert next(iter(fast.forward._cached.values())).graph is graph and len(fast.forward._cached) == 1
        return got

    for m in (fast, oracle):                          # loaded after compile()
        lo.inject_adapter(m, "a", "all", r=8, lora_alpha=16, seed=5)
    y = check()
    assert _rel(y, free) > 10 * tol
    n = compiled._lora.merges
    assert torch.equal(fast(s, t, e).sample, y) and compiled._lora.merges == n     # steady: no merge, bitwise
    for m in (fast, oracle):
        lo.set_adapters(m, "a", 0.4)
    check()
    check(cross_attention_kwargs={"scale": 0.5})
    assert torch.equal(fast(s, t, e, cross_attention_kwargs={"scale": 0.0}).sample, free)
    check()
    lo.disable_lora(fast)
    assert torch.equal(fast(s, t, e).sample, free)
    lo.enable_lora(fast)
    check()
    with torch.no_grad():                              # in-place edit of one lora_B
        for m in (fast, oracle):
            lo.lora_layers(m)[5][1].lora_B["a"].weight.mul_(-3.0)
    check()
    lo.delete_adapters(fast, "a")
    assert torch.equal(fast(s, t, e).sample, free)
    lo.inject_adapter(fast, "b", ["to_k"], r=4, seed=9)
    lo.unload_lora_weights(fast)
    assert torch.equal(fast(s, t, e).sample, free)
    oracle = uo.build_unet(cfg, seed=3, dtype=torch.float32, device=DEV)
    for m in (fast, oracle):                          # fuse_lora writes weight.data: no version counter moves
        lo.inject_adapter(m, "c", "all", r=4, lora_alpha=8, seed=13)
        lo.fuse_lora(m, lora_scale=0.8)
    check()
    for m in (fast, oracle):
        lo.unfuse_lora(m)
    check()


def test_preserve_parameters_false_freezes_the_adapter_state_until_rebind():
    cfg, dt = uo.tiny_config(), torch.float16
    fast, oracle = _pair(cfg, dt)
    fast = _compile(fast, preserve=False)
    s, t, e, kw = _inputs(cfg, 2, 32, dt)
    y = fast(s, t, e).sample
    with pytest.raises(NotImplementedError, match="rebind"):
        fast(s, t, e, cross_attention_kwargs={"scale": 0.5})
    lo.set_adapters(fast, "a", 0.2)
    assert torch.equal(fast(s, t, e).sample, y)
    fast.forward._compiled.rebind()
    lo.set_adapters(oracle, "a", 0.2)
    assert _rel(fast(s, t, e, cross_attention_kwargs={"scale": 0.5}).sample,
                _ref(oracle, s, t, e, kw, cross_attention_kwargs={"scale": 0.5})) <= MODEL_TOL[dt]


def test_reference_lcm_lora_recipe_fused_then_compiled():
    cfg, dt = uo.tiny_config(), torch.float16
    fast, oracle = _pair(cfg, dt)
    for m in (fast, oracle):
        lo.fuse_lora(m)
    fast = _compile(fast)
    s, t, e, kw = _inputs(cfg, 2, 32, dt)
    assert _rel(fast(s, t, e).sample, _ref(oracle, s, t, e, kw)) <= MODEL_TOL[dt]


def test_real_peft_injection_matches():
    peft = pytest.importorskip("peft")
    cfg, dt = uo.tiny_config(), torch.float16
    conf = peft.LoraConfig(r=8, lora_alpha=16, target_modules=["to_q", "to_k", "to_v", "to_out.0", "conv1"],
                           init_lora_weights=False)
    fast = peft.inject_adapter_in_model(conf, uo.build_unet(cfg, seed=3, dtype=torch.float32, device=DEV))
    oracle = copy.deepcopy(fast)
    fast = _compile(fast.to(dt))
    s, t, e, kw = _inputs(cfg, 2, 32, dt)
    with torch.no_grad():
        ref = oracle(s.float(), t, e.float()).sample
    assert _rel(fast(s, t, e).sample, ref) <= MODEL_TOL[dt]


# ---------------------------------------------------------------------------------------------------
# text encoder and the pipeline surface
# ---------------------------------------------------------------------------------------------------
def _clip(layers=12, hidden=768, inter=3072, heads=12, proj=False, seed=0):
    transformers = pytest.importorskip("transformers")
    cfg = transformers.CLIPTextConfig(hidden_size=hidden, intermediate_size=inter, num_hidden_layers=layers,
                                      num_attention_heads=heads, projection_dim=hidden)
    torch.manual_seed(seed)
    cls = transformers.CLIPTextModelWithProjection if proj else transformers.CLIPTextModel
    m = cls(cfg).eval()
    return lo.inject_adapter(m, "a", ["q_proj", "k_proj", "v_proj", "out_proj", "fc1", "fc2"], r=16,
                             lora_alpha=32, seed=seed)


def test_text_encoder_with_an_adapter_and_encode_prompts_scale():
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile_text_encoder
    eager = _clip().to(DEV)
    fast = compile_text_encoder(copy.deepcopy(eager).half(), CompilationConfig.Default())
    ids = torch.randint(0, 49000, (2, 77), device=DEV)
    for scale in (1.0, 0.6):
        lo.scale_lora_layers(fast, scale)
        lo.scale_lora_layers(eager, scale)
        got = fast(ids).last_hidden_state
        with torch.no_grad():
            ref = eager(ids).last_hidden_state
        lo.unscale_lora_layers(fast, scale)
        lo.unscale_lora_layers(eager, scale)
        assert _rel(got, ref) <= MODEL_TOL[torch.float16], scale
    fast(ids)                                          # the state of the unscaled encoder is merged once
    n = fast.forward._compiled._lora.merges
    fast(ids)
    assert fast.forward._compiled._lora.merges == n


def test_compile_pipeline_with_adapters_on_the_unet_and_both_text_encoders():
    from sfast.compilers.diffusion_pipeline_compiler import CompilationConfig, compile
    cfg, dt = uo.tiny_config(), torch.float16
    unet, oracle = _pair(cfg, dt)
    te1 = _clip(layers=2, hidden=128, inter=256, heads=2).to(DEV)
    te2 = _clip(layers=2, hidden=128, inter=256, heads=2, proj=True, seed=1).to(DEV)
    e1, e2 = copy.deepcopy(te1), copy.deepcopy(te2)
    pipe = types.SimpleNamespace(unet=unet, text_encoder=te1.half(), text_encoder_2=te2.half())
    pipe = compile(pipe, CompilationConfig.Default())
    ids = torch.randint(0, 49000, (2, 77), device=DEV)
    with torch.no_grad():
        assert _rel(pipe.text_encoder(ids).last_hidden_state, e1(ids).last_hidden_state) <= 1e-2
        assert _rel(pipe.text_encoder_2(ids).text_embeds, e2(ids).text_embeds) <= 1e-2
    s, t, e, kw = _inputs(cfg, 2, 32, dt)
    assert _rel(pipe.unet(s, t, e).sample, _ref(oracle, s, t, e, kw)) <= MODEL_TOL[dt]
