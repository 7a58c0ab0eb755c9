"""Host-side checks of the weight lifecycle every compiled module shares (UNet, VAE, CLIP text and vision
towers): pack on first use, refresh in place when a parameter's version counter moves, re-pack and drop the
cached plans on a dtype or device change, and the replaced methods that carry `_compiled` / `_cached`.
PackedWeights is replaced by a recording stand-in, so no packing, plan or device is involved."""
import contextlib
from types import SimpleNamespace

import pytest
import torch

from oracle import unet_oracle as uo
from oracle import vae_oracle as vo
from sfast_b200 import runtime

_TEXT = dict(vocab_size=1000, hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=2,
             max_position_embeddings=77, hidden_act="quick_gelu", eos_token_id=2)
_VISION = dict(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=2, image_size=28,
               patch_size=14, hidden_act="quick_gelu")


class _RecordingWeights:
    def __init__(self, spec, state_dict, dtype, device, dry=False):
        self.spec, self.dtype, self.device = spec, dtype, torch.device(device)
        self.refreshes = 0

    def refresh(self, state_dict):
        self.refreshes += 1


@pytest.fixture
def packs(monkeypatch):
    """Every PackedWeights the runtime creates, in order; CUDA stream / device calls become no-ops."""
    made = []

    def pack(*args, **kwargs):
        made.append(_RecordingWeights(*args, **kwargs))
        return made[-1]
    monkeypatch.setattr(runtime, "PackedWeights", pack)
    monkeypatch.setattr(runtime, "_GraphedPlan", lambda plan, use_graph: SimpleNamespace(plan=plan))
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: SimpleNamespace(synchronize=lambda: None))
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    return made


class _StandIn:
    """The attributes the compile_*_module functions read of a diffusers / transformers module."""

    def __init__(self, config):
        self.config = config
        self.params = {"a.weight": torch.zeros(4), "b.weight": torch.zeros(2, 2)}
        self.forward = self.decode = self.encode = lambda *a, **k: "eager"

    def state_dict(self):
        return dict(self.params)


def _compiled(kind, **kw):
    if kind == "unet":
        m = _StandIn(uo.tiny_config())
        return m, runtime.CompiledUNet(m.config, m.state_dict, **kw)
    if kind == "vae":
        m = _StandIn(vars(vo.tiny_vae_config()))
        return m, runtime.CompiledVAE(m, m.decode, m.encode)
    m = _StandIn(_TEXT if kind == "text" else _VISION)
    cls = runtime.CompiledTextEncoder if kind == "text" else runtime.CompiledVisionEncoder
    return m, cls(m.config, m.state_dict, m.forward, with_projection=False)


def _weights(c, dtype=torch.float16, device="cpu"):
    with c._lock:
        return c._weights_for(dtype, torch.device(device))


@pytest.mark.parametrize("kind", ["unet", "vae", "text", "vision"])
def test_pack_refresh_and_repack(packs, kind):
    m, c = _compiled(kind)
    w = _weights(c)
    assert len(packs) == 1 and packs[0] is w and w.dtype == torch.float16
    c._graphed("key", lambda: "plan")
    assert _weights(c) is w and len(packs) == 1 and w.refreshes == 0       # unchanged: neither pack nor refresh

    m.params["b.weight"].add_(1.0)                                           # in-place update (LoRA fuse)
    assert _weights(c) is w and w.refreshes == 1 and "key" in c._cached
    assert _weights(c) is w and w.refreshes == 1                             # counted once

    w16 = _weights(c, dtype=torch.bfloat16)                                  # dtype change: re-pack
    assert w16 is not w and len(packs) == 2 and not c._cached
    c._graphed("key", lambda: "plan")
    wm = _weights(c, dtype=torch.bfloat16, device="meta")                    # device change: re-pack
    assert wm is not w16 and len(packs) == 3 and wm.device.type == "meta" and not c._cached


def test_preserve_parameters_off_refreshes_only_on_rebind(packs):
    m, c = _compiled("unet", preserve_parameters=False)
    w = _weights(c)
    m.params["a.weight"].add_(1.0)
    assert _weights(c) is w and w.refreshes == 0
    c.rebind()
    assert w.refreshes == 1 and len(packs) == 1
    assert _weights(c) is w and w.refreshes == 1


def test_graphed_builds_each_key_once(packs):
    _, c = _compiled("unet")
    built = []
    for key in ("a", "b", "a"):
        c._graphed(key, lambda: built.append(key) or key)
    assert built == ["a", "b"] and c._cached["a"].plan == "a"


@pytest.mark.parametrize("kind", ["unet", "vae", "text", "vision"])
def test_replaced_methods_carry_the_compiled_object(kind):
    m = _StandIn(uo.tiny_config() if kind == "unet" else vars(vo.tiny_vae_config()) if kind == "vae"
                 else _TEXT if kind == "text" else _VISION)
    if kind == "vae":
        m.params = {"post_quant_conv.weight": torch.zeros(1)}
        runtime.compile_vae_module(m)
        names = ("decode", "encode")
    else:
        {"unet": runtime.compile_unet_module, "text": runtime.compile_text_encoder_module,
         "vision": runtime.compile_image_encoder_module}[kind](m)
        names = ("forward",)
    compiled = getattr(m, names[0])._compiled
    assert compiled is not None
    for n in names:
        fn = getattr(m, n)
        assert fn._compiled is compiled and fn._cached is compiled._cached and fn.__self__ is m
