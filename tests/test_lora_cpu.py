"""PEFT LoRA on the native path, without a GPU: name resolution on wrapped modules, the effective-scale table
against the oracle's PEFT forward in every lifecycle state, refusals, change detection (the scale round trip
merges nothing), dependency tracking of the packed weights, sfb_lora_merge's host validation and its fp64
restatement, dry launch lists that do not change with an adapter on every layer, and two likely mistakes."""
import ctypes
import math

import pytest
import torch

from oracle import lora_oracle as lo
from oracle import unet_oracle as uo
from sfast_b200 import _lib, lora, ops
from sfast_b200.plan import PackedWeights, UNetPlan
from sfast_b200.unet_spec import param_shapes, spec_from_config
from test_host_logic import _DUMMY_PTR
from test_ip_adapter_plus_cpu import PARENT_FINGERPRINTS, plan_fingerprint

CFGS = {"tiny": uo.tiny_config, "sd15": uo.sd15_config, "sdxl": uo.sdxl_config}


def _wrapped_tiny(seed=0, **kw):
    m = uo.build_unet(uo.tiny_config(), seed=seed, dtype=torch.float64)
    return lo.inject_adapter(m, "a", r=kw.pop("r", 4), lora_alpha=kw.pop("lora_alpha", 8), seed=seed + 1, **kw)


def merge_reference(w, adapters, out_dtype):
    """fp64 restatement of sfb_lora_merge: round(W + sum_i s_i B_i A_i) to out_dtype, once."""
    acc = w.double()
    for a, b, s in adapters:
        acc = acc + s * (b.double() @ a.double())
    return acc.to(out_dtype)


def _effective_sd(m, mult=1.0):
    """fp64 state dict under diffusers' names with every LoRA layer's effective weight (lora.effective_scales)."""
    sd = {k: v.double() for k, v in lora.plain_state_dict(m.state_dict()).items()}
    for p, layer in lora.scan(m).items():
        sc = lora.effective_scales(layer, mult, p)
        w = layer.base_layer.weight.detach().double()
        ad = [(layer.lora_A[a].weight.detach().reshape(layer.lora_A[a].weight.shape[0], -1),
               layer.lora_B[a].weight.detach().reshape(w.shape[0], -1), s) for a, s in sc]
        sd[p + ".weight"] = merge_reference(w.reshape(w.shape[0], -1), ad, torch.float64).reshape(w.shape) if ad else w
    return sd


def _inputs(b=1, h=16, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(b, 4, h, h, generator=g, dtype=torch.float64), torch.tensor([321.0], dtype=torch.float64),
            torch.randn(b, 7, 128, generator=g, dtype=torch.float64))


def _merged_equals_peft_forward(m, mult=1.0):
    """The plain oracle UNet with the effective weights computes what the wrapped one does (fp64)."""
    plain = uo.build_unet(uo.tiny_config(), dtype=torch.float64)
    plain.load_state_dict(_effective_sd(m, mult))
    s, t, e = _inputs()
    with torch.no_grad():
        if mult != 1.0:
            lo.scale_lora_layers(m, mult)
        want = m(s, t, e).sample
        if mult != 1.0:
            lo.unscale_lora_layers(m, mult)
        got = plain(s, t, e).sample
    torch.testing.assert_close(got, want, rtol=1e-9, atol=1e-9)
    return want


# ---------------------------------------------------------------------------------------------------
# names
# ---------------------------------------------------------------------------------------------------
def test_every_param_shapes_name_resolves_on_a_wrapped_unet():
    m = _wrapped_tiny()
    spec = spec_from_config(uo.tiny_config())
    layers = lora.scan(m)
    assert len(layers) == sum(isinstance(x, (torch.nn.Linear, torch.nn.Conv2d))
                              for x in uo.build_unet(uo.tiny_config()).modules())
    assert {"conv_in", "up_blocks.1.attentions.0.transformer_blocks.0.attn1.to_out.0",
            "down_blocks.0.attentions.0.transformer_blocks.0.ff.net.0.proj"} <= set(layers)
    sd = lora.plain_state_dict(m.state_dict())
    assert set(sd) == set(param_shapes(spec))
    assert all(tuple(sd[k].shape) == tuple(v) for k, v in param_shapes(spec).items())


def test_every_param_shapes_name_resolves_on_a_wrapped_clip_text_model():
    transformers = pytest.importorskip("transformers")
    from sfast_b200.clip_plan import clip_text_param_shapes, clip_text_spec_from_config
    cfg = transformers.CLIPTextConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2,
                                      num_attention_heads=2, vocab_size=100, max_position_embeddings=16)
    m = transformers.CLIPTextModel(cfg)
    lo.inject_adapter(m, "a", ["q_proj", "k_proj", "v_proj", "out_proj", "fc1", "fc2"], r=4)
    assert len(lora.scan(m, "text encoder")) == 2 * 6
    sd = lora.plain_state_dict(m.state_dict())
    shapes = clip_text_param_shapes(clip_text_spec_from_config(cfg))
    assert set(shapes) <= set(sd) and all(tuple(sd[k].shape) == tuple(v) for k, v in shapes.items())


# ---------------------------------------------------------------------------------------------------
# semantics: the effective-scale table against the oracle's PEFT forward
# ---------------------------------------------------------------------------------------------------
def test_effective_scales_match_the_peft_forward_in_every_lifecycle_state():
    m = _wrapped_tiny(r=4, lora_alpha=8)
    with torch.no_grad():
        base = uo.build_unet(uo.tiny_config(), seed=0, dtype=torch.float64)(*_inputs()).sample
    y1 = _merged_equals_peft_forward(m)
    assert (y1 - base).abs().max() > 1e-2
    _merged_equals_peft_forward(m, mult=0.5)                              # cross_attention_kwargs scale
    lo.inject_adapter(m, "b", ["to_q", "to_v", "proj_in", "conv1"], r=8, lora_alpha=4, seed=5,
                      rank_pattern={"conv1": 2})
    _merged_equals_peft_forward(m)                                        # only b active now
    lo.set_adapters(m, ["a", "b"], [0.7, 0.3])
    _merged_equals_peft_forward(m)
    lo.set_adapters(m, ["a", "b"], [{"down_blocks.1": 0.0, "up_blocks": 2.0}, 0.5])   # per-layer weights
    _merged_equals_peft_forward(m)
    lo.fuse_lora(m, adapter_names=["a"])                                  # merged + active unmerged: base only
    assert all(lora.effective_scales(layer) == () for layer in lora.scan(m).values())
    _merged_equals_peft_forward(m)
    lo.unfuse_lora(m)
    _merged_equals_peft_forward(m)
    lo.disable_lora(m)
    assert all(lora.effective_scales(layer) == () for layer in lora.scan(m).values())
    lo.enable_lora(m)
    lo.delete_adapters(m, "a")
    _merged_equals_peft_forward(m)
    lo.set_adapters(m, "b", 0.0)
    assert all(lora.effective_scales(layer) == () for layer in lora.scan(m).values())


def test_rslora_scaling_is_read_from_the_layer():
    m = lo.inject_adapter(uo.build_unet(uo.tiny_config(), dtype=torch.float64), "a", ["to_k"], r=16,
                          lora_alpha=8, use_rslora=True)
    layer = next(iter(lora.scan(m).values()))
    assert lora.effective_scales(layer) == (("a", 8 / 4.0),)
    _merged_equals_peft_forward(m)


# ---------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------
def _dry_view(m, mult=1.0):
    t = lora.LoraTracker(m)
    _, states = t.poll(mult)
    return t, t.view(m.state_dict(), states, torch.float16, "meta", dry=True)


def _first(m, suffix):
    return next((p, layer) for p, layer in lora.scan(m).items() if p.endswith(suffix))


def test_dora_lora_bias_and_conv_geometry_are_refused_by_name():
    for mutate, match in (
            (lambda layer: layer.use_dora.__setitem__("a", True), "DoRA"),
            (lambda layer: layer.lora_bias.__setitem__("a", True), "lora_bias")):
        m = _wrapped_tiny()
        p, layer = _first(m, "attn2.to_k")
        mutate(layer)
        with pytest.raises(NotImplementedError, match=f"{p}.*{match}"):
            _dry_view(m)
    m = _wrapped_tiny()
    p, layer = _first(m, "resnets.0.conv1")
    layer.lora_A["a"] = torch.nn.Conv2d(layer.base_layer.in_channels, 4, 1, bias=False).double()
    with pytest.raises(NotImplementedError, match=f"{p}.*kernel size"):
        _dry_view(m)
    m = _wrapped_tiny()
    p, layer = _first(m, "resnets.0.conv2")
    layer.lora_B["a"] = torch.nn.Conv2d(4, layer.base_layer.out_channels, 3, padding=1, bias=False).double()
    with pytest.raises(NotImplementedError, match="1x1"):
        _dry_view(m)


def test_other_peft_wrappers_legacy_lora_layers_and_disabled_merged_adapters_are_refused():
    class LoHa(torch.nn.Module):
        def __init__(self, base):
            super().__init__()
            self.base_layer = base
            self.hada_w1_a = torch.nn.ParameterDict({"a": torch.nn.Parameter(torch.zeros(2, 2))})

    m = uo.build_unet(uo.tiny_config())
    m.conv_in = LoHa(m.conv_in)
    with pytest.raises(NotImplementedError, match="'conv_in'.*not LoRA"):
        lora.scan(m)
    m = uo.build_unet(uo.tiny_config())
    m.conv_out.lora_layer = torch.nn.Linear(2, 2)
    with pytest.raises(NotImplementedError, match="'conv_out'.*legacy"):
        lora.scan(m)
    m = _wrapped_tiny()
    lo.fuse_lora(m)
    lo.disable_lora(m)
    with pytest.raises(NotImplementedError, match="unfuse_lora"):
        lora.LoraTracker(m).poll()


def test_adapters_on_modules_without_lora_support_are_refused_by_name():
    m = lo.inject_adapter(uo.build_unet(uo.tiny_config()), "a", ["to_q"])
    with pytest.raises(NotImplementedError, match="ControlNet layer 'down_blocks.0.attentions.0.*to_q'"):
        lora.refuse_adapters(m.state_dict(), "ControlNet")
    lora.refuse_adapters(uo.build_unet(uo.tiny_config()).state_dict(), "VAE")   # nothing to refuse


# ---------------------------------------------------------------------------------------------------
# change detection
# ---------------------------------------------------------------------------------------------------
def test_change_detection_and_the_scale_round_trip():
    plain = uo.build_unet(uo.tiny_config())
    t = lora.LoraTracker(plain)
    assert t.quiet() and t.poll() == (set(), {}) and t.records == []
    m = _wrapped_tiny()
    t = lora.LoraTracker(m)
    changed, states = t.poll()
    assert changed == set(t.layers)
    t.applied = states
    assert t.poll()[0] == set()
    for w in (0.6, 0.3, 1.7, 1e-3):  # encode_prompt's scale_lora_layers / unscale_lora_layers round trip
        lo.scale_lora_layers(m, w)
        assert t.poll()[0] == set(t.layers)
        lo.unscale_lora_layers(m, w)
        assert t.poll()[0] == set(), w
    assert t.poll(0.5)[0] == set(t.layers)
    p, layer = _first(m, "attn1.to_v")
    layer.scaling["a"] *= 2
    assert t.poll()[0] == {p}
    layer.scaling["a"] /= 2
    lo.unload_lora_weights(m)                      # children swapped back: every old layer changes
    changed, states = t.poll()
    assert changed == set(states) | set(t.applied) and states == {} and t.layers == {}
    t.applied = states
    assert t.quiet() and t.poll() == (set(), {})
    lo.inject_adapter(m, "b", ["to_k"])            # loaded after compile
    changed, _ = t.poll()
    assert changed == set(t.layers) and len(changed) == 32 and all(p.endswith(".to_k") for p in changed)


def test_a_relaunched_adapter_with_the_same_name_and_scale_is_a_change():
    m = _wrapped_tiny()
    t = lora.LoraTracker(m)
    t.applied = t.poll()[1]
    lo.delete_adapters(m, "a")
    lo.inject_adapter(m, "a", "all", r=4, lora_alpha=8, seed=9)
    assert t.poll()[0] == set(t.layers)


# ---------------------------------------------------------------------------------------------------
# dependency tracking and dry launch lists
# ---------------------------------------------------------------------------------------------------
def _meta_wrapped(cfg, dt=torch.float16):
    with torch.device("meta"):
        m = uo.UNet2DConditionModel(CFGS[cfg]()).to(dt)
    return lo.inject_adapter(m, "a", "all", r=64)


def _dry_plan(cfg, b, h, w, dt=torch.float16, wrapped=True):
    spec = spec_from_config(CFGS[cfg]())
    if wrapped:
        m = _meta_wrapped(cfg, dt)
        t = lora.LoraTracker(m)
        sd = t.view(m.state_dict(), t.poll()[1], dt, "meta", dry=True)
    else:
        sd = {k: torch.empty(v, dtype=dt, device="meta") for k, v in param_shapes(spec).items()}
    pw = PackedWeights(spec, sd, dt, "meta", dry=True)
    return UNetPlan(pw, b, h, w), pw, sd


@pytest.mark.parametrize("cfg,b,h,n_layers", [("sd15", 2, 64, 282), ("sdxl", 2, 128, 794)])
def test_dry_schedules_with_an_adapter_on_every_weight_match_the_parent(cfg, b, h, n_layers):
    plan, _, sd = _dry_plan(cfg, b, h, h)
    assert len(sd.tracker.layers) == n_layers
    assert plan_fingerprint(plan) == PARENT_FINGERPRINTS[(cfg, b, h, h, 0, 0)]


def test_a_changed_layer_re_runs_only_the_builders_that_read_it():
    plan, pw, sd = _dry_plan("tiny", 2, 32, 32)
    total = len(pw._builders)
    assert pw.refresh(sd) == total
    blk = "down_blocks.0.attentions.0.transformer_blocks.0"
    cases = {f"{blk}.attn1.to_q": 1,                     # the LayerNorm-folded QKV matrix
             f"{blk}.ff.net.0.proj": 1,                  # the GEGLU interleave
             "down_blocks.0.resnets.0.time_emb_proj": 1,  # the one concatenated time-embedding matrix
             "up_blocks.0.upsamplers.0.conv": 1,         # the four-phase upconv
             "conv_in": 1}
    for p, n in cases.items():
        assert pw.refresh(sd, {p + ".weight"}) == n, p
    assert pw.refresh(sd, {"down_blocks.0.resnets.0.time_emb_proj.weight", "conv_in.weight"}) == 2
    assert pw.refresh(sd, set()) == 0


# ---------------------------------------------------------------------------------------------------
# sfb_lora_merge: host validation and the fp64 restatement
# ---------------------------------------------------------------------------------------------------
def test_lora_merge_struct_layout_matches_the_header(tmp_path):
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lines = ['printf("size %zu\\n", sizeof(sfb_lora_merge_params));',
             'printf("asize %zu\\n", sizeof(sfb_lora_adapter));']
    lines += [f'printf("{f} %zu\\n", offsetof(sfb_lora_merge_params, {f}));' for f, _ in _lib.LoraMergeParams._fields_]
    lines += [f'printf("a.{f} %zu\\n", offsetof(sfb_lora_adapter, {f}));' for f, _ in _lib.LoraAdapter._fields_]
    src = tmp_path / "l.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "sfb200.h"\nint main(void) {\n'
                   + "\n".join(lines) + "\nreturn 0; }\n")
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), str(src), "-o", str(tmp_path / "l")], check=True)
    got = dict(x.split() for x in subprocess.run([str(tmp_path / "l")], capture_output=True, text=True,
                                                  check=True).stdout.split("\n") if x)
    assert int(got["size"]) == ctypes.sizeof(_lib.LoraMergeParams)
    assert int(got["asize"]) == ctypes.sizeof(_lib.LoraAdapter)
    for f, _ in _lib.LoraMergeParams._fields_:
        assert int(got[f]) == getattr(_lib.LoraMergeParams, f).offset, f
    for f, _ in _lib.LoraAdapter._fields_:
        assert int(got["a." + f]) == getattr(_lib.LoraAdapter, f).offset, f


_NO_GPU = pytest.mark.skipif(torch.cuda.is_available(), reason="needs a box without a GPU: launches must fail")


def test_lora_merge_host_validation():
    n, k, r = 40, 36, 4
    w, out = torch.zeros(n, k, dtype=torch.float16), torch.zeros(n, k, dtype=torch.bfloat16)
    a, b = torch.zeros(r, k), torch.zeros(n, r, dtype=torch.bfloat16)
    p = ops.lora_merge_params(w, [(a, b, 0.5)], out)
    assert (p.n, p.k, p.ldw, p.ldo, p.w_dtype, p.out_dtype, p.count) == (n, k, k, k, 0, 1, 1)
    assert (p.adapters[0].rank, p.adapters[0].a_dtype, p.adapters[0].b_dtype, p.adapters[0].scale) == (r, 2, 1, 0.5)
    wide = torch.zeros(n, 64, dtype=torch.float32)[:, :k]             # pitched W
    assert ops.lora_merge_params(wide, [(a, b, 1.0)] * 8, out).ldw == 64
    bad = [(dict(w=w.t()), "same 2-D shape"), (dict(out=out.float()), "fp16 / bf16"),
           (dict(ad=[(a, b, 1.0)] * 9), "1..8"), (dict(ad=[]), "1..8"),
           (dict(ad=[(a[:, :8], b, 1.0)]), "do not fit"), (dict(ad=[(a, b[:, :2], 1.0)]), "do not fit"),
           (dict(ad=[(torch.zeros(257, k), torch.zeros(n, 257), 1.0)]), "rank 257"),
           (dict(ad=[(a.double(), b, 1.0)]), "fp16 / bf16 / fp32"),
           (dict(ad=[(a.t().contiguous().t(), b, 1.0)]), "unit column stride"),
           (dict(out=w.view(torch.bfloat16)), "shares memory")]
    for kw, match in bad:
        with pytest.raises(ValueError, match=match):
            ops.lora_merge_params(kw.get("w", w), kw.get("ad", [(a, b, 1.0)]), kw.get("out", out))


@_NO_GPU
def test_lora_merge_library_validation():
    n, k, r = 40, 36, 4
    p = ops.lora_merge_params(torch.zeros(n, k, dtype=torch.float16), [(torch.zeros(r, k), torch.zeros(n, r), 0.5)],
                              torch.zeros(n, k, dtype=torch.float16))
    lib = _lib.lib()
    q = _lib.LoraMergeParams()
    ctypes.memmove(ctypes.byref(q), ctypes.byref(p), ctypes.sizeof(p))
    q.w = q.out = q.adapters[0].a = q.adapters[0].b = _DUMMY_PTR
    assert lib.sfb_lora_merge(ctypes.byref(q), None) == -2   # past validation: fails at the launch (no GPU)
    for field, val in (("count", 0), ("count", 9), ("ldo", k - 1), ("w_dtype", 3), ("out_dtype", 2)):
        c = _lib.LoraMergeParams()
        ctypes.memmove(ctypes.byref(c), ctypes.byref(q), ctypes.sizeof(q))
        setattr(c, field, val)
        assert lib.sfb_lora_merge(ctypes.byref(c), None) == -1, field
    c = _lib.LoraMergeParams()
    ctypes.memmove(ctypes.byref(c), ctypes.byref(q), ctypes.sizeof(q))
    c.adapters[0].rank = 257
    assert lib.sfb_lora_merge(ctypes.byref(c), None) == -1


@pytest.mark.parametrize("kh", [1, 3])
def test_restatement_with_oihw_flattening_equals_peft_conv_delta(kh):
    torch.manual_seed(0)
    base = torch.nn.Conv2d(6, 5, kh, padding=kh // 2).double()
    layer = lo.Conv2d(base, "a")
    layer.update_layer("a", 3, 6, generator=torch.Generator().manual_seed(1))
    w = base.weight.detach()
    a = layer.lora_A["a"].weight.detach().reshape(3, -1)
    b = layer.lora_B["a"].weight.detach().reshape(5, -1)
    got = merge_reference(w.reshape(5, -1), [(a, b, layer.scaling["a"])], torch.float64).reshape(w.shape)
    torch.testing.assert_close(got, w + layer.get_delta_weight("a"), rtol=1e-12, atol=1e-12)


def _rel(got, ref):
    d = (got - ref).abs()
    rms = ref.pow(2).mean().sqrt()
    return max((d.max() / ref.abs().max()).item(), (d / (ref.abs() + rms)).max().item())


def test_likely_mistakes_move_the_tiny_unet_by_more_than_ten_times_the_gpu_tolerance():
    """Flattening conv A in the packed K-major order (kh, kw, cin) instead of OIHW's (cin, kh, kw), or dropping
    alpha / r, each move the output by more than 10x the fp16 tolerance (1e-2)."""
    m = _wrapped_tiny(r=4, lora_alpha=16)
    s, t, e = _inputs()
    plain = uo.build_unet(uo.tiny_config(), dtype=torch.float64)
    with torch.no_grad():
        want = m(s, t, e).sample
    for mistake in ("khwc", "no_alpha"):
        sd = _effective_sd(m)
        for p, layer in lora.scan(m).items():
            w = layer.base_layer.weight.detach()
            A, B = layer.lora_A["a"].weight.detach(), layer.lora_B["a"].weight.detach()
            if mistake == "khwc":
                if w.dim() != 4 or w.shape[2] == 1:
                    continue
                A = A.permute(0, 2, 3, 1)
                s_ = layer.scaling["a"]
            else:
                s_ = 1.0
            sd[p + ".weight"] = (w.reshape(w.shape[0], -1) + s_ * B.reshape(w.shape[0], -1)
                                 @ A.reshape(A.shape[0], -1)).reshape(w.shape)
        plain.load_state_dict(sd)
        with torch.no_grad():
            got = plain(s, t, e).sample
        assert _rel(got, want) > 10 * 1e-2, mistake
    assert not math.isclose(lora.scan(m)["conv_in"].scaling["a"], 1.0)


# ---------------------------------------------------------------------------------------------------
# a refusal or a failure during a re-pack is never followed by a silent, half-merged call
# ---------------------------------------------------------------------------------------------------
class _ReadingWeights:
    """PackedWeights stand-in that reads every name it is asked to re-pack (which merges adapted weights)."""

    def __init__(self, spec, state_dict, dtype, device, dry=False):
        self.dtype, self.device = dtype, torch.device(device)
        self.calls = []
        self._read(state_dict, None)

    def _read(self, sd, names):
        for n in sorted(sd if names is None else names):
            sd[n]
        self.calls.append(names)

    def refresh(self, state_dict, names=None):
        self._read(state_dict, names)


@pytest.fixture
def reading(monkeypatch):
    import contextlib
    from types import SimpleNamespace
    from sfast_b200 import runtime
    monkeypatch.setattr(runtime, "PackedWeights", _ReadingWeights)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: SimpleNamespace(synchronize=lambda: None))
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    merges = []

    def fake_merge(layer, scales, out_dtype, device, name="?"):
        merges.append(name)
        if getattr(layer, "fail_merge", False):
            raise RuntimeError("out of memory")
        return layer.base_layer.weight.detach()
    monkeypatch.setattr(lora, "merged_weight", fake_merge)
    return runtime, merges


def _weights(c):
    with c._lock:
        return c._weights_for(torch.float16, torch.device("cpu"))


def test_a_refused_adapter_loaded_after_the_first_call_is_refused_on_every_call(reading):
    runtime, merges = reading
    m = uo.build_unet(uo.tiny_config())
    c = runtime.CompiledUNet(m.config, m.state_dict, module=m)
    w = _weights(c)
    lo.inject_adapter(m, "a", "all", r=4)
    p, layer = _first(m, "attn2.to_k")
    layer.use_dora["a"] = True
    for _ in range(3):
        with pytest.raises(NotImplementedError, match=f"{p}.*DoRA"):
            _weights(c)
    assert merges == [] and w.calls == [None]        # refused before anything was re-packed
    layer.use_dora["a"] = False
    _weights(c)
    assert len(merges) == len(lora.scan(m)) and len(w.calls) == 2


def test_a_re_pack_that_fails_part_way_is_redone_in_full(reading):
    runtime, merges = reading
    m = uo.build_unet(uo.tiny_config())
    c = runtime.CompiledUNet(m.config, m.state_dict, module=m)
    w = _weights(c)
    lo.inject_adapter(m, "a", "all", r=4)
    p, layer = _first(m, "up_blocks.3.resnets.2.conv2")
    layer.fail_merge = True
    with pytest.raises(RuntimeError, match="out of memory"):
        _weights(c)
    assert 0 < len(merges) < len(lora.scan(m))       # part of the layers were merged when it failed
    with pytest.raises(RuntimeError, match="out of memory"):
        _weights(c)                                  # not marked applied: the next call tries again
    layer.fail_merge = False
    merges.clear()
    _weights(c)
    assert w.calls[-1] is None and len(merges) == len(lora.scan(m))   # everything re-packed
    merges.clear()
    _weights(c)
    assert merges == [] and len(w.calls) == 2        # steady: the first pack and the full re-pack


def test_peft_adapters_loaded_after_the_first_call_on_a_module_without_lora_support_are_refused(reading):
    runtime, _ = reading
    m = uo.build_unet(uo.tiny_config())
    c = runtime.CompiledControlNet.__new__(runtime.CompiledControlNet)
    runtime._CompiledModule.__init__(c, spec_from_config(uo.tiny_config()), m.state_dict)
    _weights(c)
    lo.inject_adapter(m, "a", ["to_q"])
    with pytest.raises(NotImplementedError, match="ControlNet layer 'down_blocks.0.*to_q'"):
        _weights(c)


def test_the_steady_check_does_not_recompute_states_and_sees_in_place_state_edits():
    m = _wrapped_tiny()
    t = lora.LoraTracker(m)
    t.applied = t.poll()[1]
    changed, states = t.poll()
    assert changed == set() and states is t.applied
    p, layer = _first(m, "attn1.to_q")
    layer.merged_adapters.append("a")                # a list edited in place
    assert t.poll()[0] == {p}
    layer.merged_adapters.clear()
    assert t.poll()[0] == set()
    layer.lora_B["a"] = torch.nn.Linear(4, layer.base_layer.out_features, bias=False).double()
    assert t.poll()[0] == {p}
