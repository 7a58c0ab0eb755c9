"""ORACLE (test infrastructure, NOT product code).

A restatement of PEFT's LoRA layers and of the diffusers LoRA lifecycle, for modules without `peft` or
`diffusers` installed.  The semantics restated are those of PEFT 0.13 (`peft/tuners/lora/layer.py`: `LoraLayer`,
`Linear`, `Conv2d`; `peft/tuners/tuners_utils.py`: `BaseTunerLayer`) and of diffusers 0.31 (`utils/peft_utils.py`:
`scale_lora_layers`, `unscale_lora_layers`, `set_weights_and_activate_adapters`, `get_module_weight`;
`loaders/lora_base.py`: `fuse_lora`, `unfuse_lora`, `unload_lora_weights`, `delete_adapters`,
`enable_lora`, `disable_lora`).  They were restated from that source and not run against it.

Deliberate difference: PEFT initialises `lora_B` to zero, so a freshly injected adapter is a no-op.  Here
`lora_B` is random (seeded, about a tenth of `lora_A`'s scale, so that a delta is a fraction of the
base weight as in trained adapters): an adapter that is dropped, mis-scaled or mis-shaped moves the output.

Only `tests/` may import this module.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F


class LoraLayer(nn.Module):
    """PEFT's LoRA wrapper: `base_layer` plus one (lora_A, lora_B) pair per adapter, same attribute names."""

    def __init__(self, base_layer, adapter_name):
        super().__init__()
        self.base_layer = base_layer
        self.r, self.lora_alpha, self.scaling = {}, {}, {}
        self.lora_dropout = nn.ModuleDict()
        self.lora_A, self.lora_B = nn.ModuleDict(), nn.ModuleDict()
        self.use_dora, self.lora_bias = {}, {}
        self.merged_adapters = []
        self._disable_adapters = False
        self._active_adapter = adapter_name

    # -- BaseTunerLayer properties ------------------------------------------------------------------
    @property
    def weight(self):
        return self.base_layer.weight

    @property
    def bias(self):
        return self.base_layer.bias

    @property
    def disable_adapters(self):
        return self._disable_adapters

    @property
    def merged(self):
        return bool(self.merged_adapters)

    @property
    def active_adapter(self):
        return self._active_adapter

    @property
    def active_adapters(self):
        return [self._active_adapter] if isinstance(self._active_adapter, str) else list(self._active_adapter)

    # -- adapters -----------------------------------------------------------------------------------
    def _make_ab(self, r):
        raise NotImplementedError

    def update_layer(self, adapter_name, r, lora_alpha, use_rslora=False, generator=None):
        a, b = self._make_ab(r)
        dev, dt = self.base_layer.weight.device, self.base_layer.weight.dtype
        if dev.type != "meta":  # (a meta model only has shapes: dry plans)
            with torch.no_grad():
                a.weight.copy_(torch.randn(a.weight.shape, generator=generator) / math.sqrt(a.weight[0].numel()))
                b.weight.copy_(torch.randn(b.weight.shape, generator=generator) * (0.1 / math.sqrt(r)))
        self.lora_A[adapter_name], self.lora_B[adapter_name] = a.to(dev, dt), b.to(dev, dt)
        self.lora_dropout[adapter_name] = nn.Identity()
        self.r[adapter_name], self.lora_alpha[adapter_name] = r, lora_alpha
        self.scaling[adapter_name] = lora_alpha / (math.sqrt(r) if use_rslora else r)
        self.use_dora[adapter_name], self.lora_bias[adapter_name] = False, False

    def set_adapter(self, adapter_names):
        self._active_adapter = adapter_names

    def set_scale(self, adapter, scale):
        if adapter not in self.scaling:
            return
        self.scaling[adapter] = scale * self.lora_alpha[adapter] / self.r[adapter]

    def scale_layer(self, scale):
        if scale == 1:
            return
        for a in self.active_adapters:
            if a in self.lora_A:
                self.scaling[a] *= scale

    def unscale_layer(self, scale=None):
        for a in self.active_adapters:
            if a in self.lora_A:
                if scale is None:
                    self.scaling[a] = self.lora_alpha[a] / self.r[a]
                else:
                    self.scaling[a] /= scale

    def enable_adapters(self, enabled):
        self._disable_adapters = not enabled

    def delete_adapter(self, adapter_name):
        for d in (self.lora_A, self.lora_B, self.lora_dropout):
            if adapter_name in d:
                del d[adapter_name]
        for d in (self.r, self.lora_alpha, self.scaling, self.use_dora, self.lora_bias):
            d.pop(adapter_name, None)
        if adapter_name in self.active_adapters:
            rest = [a for a in self.active_adapters if a != adapter_name]
            if rest:
                self.set_adapter(rest)
            else:
                left = list(self.lora_A.keys())
                self.set_adapter(left[0] if left else [])

    def get_delta_weight(self, adapter):
        raise NotImplementedError

    def merge(self, adapter_names=None):
        for a in adapter_names or self.active_adapters:
            if a in self.lora_A:
                self.base_layer.weight.data += self.get_delta_weight(a)
                self.merged_adapters.append(a)

    def unmerge(self):
        while self.merged_adapters:
            a = self.merged_adapters.pop()
            if a in self.lora_A:
                self.base_layer.weight.data -= self.get_delta_weight(a)

    # -- PEFT Linear / Conv2d forward -----------------------------------------------------------------
    def forward(self, x, *args, **kwargs):
        if self.disable_adapters:
            if self.merged:
                self.unmerge()
            return self.base_layer(x, *args, **kwargs)
        if self.merged:
            return self.base_layer(x, *args, **kwargs)
        result = self.base_layer(x, *args, **kwargs)
        dt = result.dtype
        for a in self.active_adapters:
            if a not in self.lora_A:
                continue
            la, lb = self.lora_A[a], self.lora_B[a]
            xa = x.to(la.weight.dtype)
            result = result + lb(la(self.lora_dropout[a](xa))) * self.scaling[a]
        return result.to(dt)


class Linear(LoraLayer):
    def _make_ab(self, r):
        base = self.base_layer
        return nn.Linear(base.in_features, r, bias=False), nn.Linear(r, base.out_features, bias=False)

    def get_delta_weight(self, adapter):
        w = self.base_layer.weight
        ct = torch.promote_types(w.dtype, torch.float32)  # PEFT upcasts 16-bit weights for the product
        a, b = self.lora_A[adapter].weight.to(ct), self.lora_B[adapter].weight.to(ct)
        return ((b @ a) * self.scaling[adapter]).to(w.dtype)


class Conv2d(LoraLayer):
    def _make_ab(self, r):
        base = self.base_layer
        return (nn.Conv2d(base.in_channels, r, base.kernel_size, base.stride, base.padding, bias=False),
                nn.Conv2d(r, base.out_channels, (1, 1), (1, 1), bias=False))

    def get_delta_weight(self, adapter):
        w = self.base_layer.weight
        ct = torch.promote_types(w.dtype, torch.float32)  # PEFT upcasts 16-bit weights for the product
        a, b = self.lora_A[adapter].weight.to(ct), self.lora_B[adapter].weight.to(ct)
        if tuple(w.shape[2:4]) == (1, 1):
            d = (b.squeeze(3).squeeze(2) @ a.squeeze(3).squeeze(2)).unsqueeze(2).unsqueeze(3)
        else:
            d = F.conv2d(a.permute(1, 0, 2, 3), b).permute(1, 0, 2, 3)
        return (d * self.scaling[adapter]).to(w.dtype)


def lora_layers(model):
    return [(n, m) for n, m in model.named_modules() if isinstance(m, LoraLayer)]


def _targets(model, target_modules):
    """Names of the Linear / Conv2d modules PEFT's `target_modules` matches (exact name or '.'-suffix)."""
    out = []
    for name, m in model.named_modules():
        if isinstance(m, LoraLayer) or ".base_layer" in name or ".lora_" in name:
            continue
        if isinstance(m, (nn.Linear, nn.Conv2d)) and (
                target_modules == "all" or any(name == t or name.endswith("." + t) for t in target_modules)):
            out.append(name)
    out += [n for n, m in model.named_modules() if isinstance(m, LoraLayer)
            and (target_modules == "all" or any(n == t or n.endswith("." + t) for t in target_modules))]
    return out


def inject_adapter(model, adapter_name, target_modules="all", r=4, lora_alpha=None, rank_pattern=None,
                   use_rslora=False, seed=0):
    """PEFT's inject_adapter_in_model: wrap (or extend) every targeted layer with adapter `adapter_name`, record
    `model.peft_config`, and make `adapter_name` the active adapter of every LoRA layer (as PEFT's tuner does
    after an injection).  `rank_pattern`: {name suffix: rank}; alpha follows the rank (alpha = r) unless
    `lora_alpha` is given."""
    g = torch.Generator().manual_seed(seed)
    for name in _targets(model, target_modules):
        parent_name, _, key = name.rpartition(".")
        parent = model.get_submodule(parent_name) if parent_name else model
        m = parent._modules[key]
        rank = next((v for k, v in (rank_pattern or {}).items() if name == k or name.endswith("." + k)), r)
        if not isinstance(m, LoraLayer):
            m = (Conv2d if isinstance(m, nn.Conv2d) else Linear)(m, adapter_name)
            parent._modules[key] = m
        m.update_layer(adapter_name, rank, rank if lora_alpha is None else lora_alpha, use_rslora, g)
    cfg = getattr(model, "peft_config", None)
    if cfg is None:
        model.peft_config = cfg = {}
    cfg[adapter_name] = dict(target_modules=target_modules, r=r, lora_alpha=lora_alpha)
    for _, m in lora_layers(model):
        m.set_adapter(adapter_name)
    return model


def get_module_weight(weight, module_name):
    """diffusers' get_module_weight: a number, or {name fragment: weight} (first fragment in the name wins)."""
    if not isinstance(weight, dict):
        return weight
    for k, v in weight.items():
        if k in module_name:
            return v
    return 1.0


def set_adapters(model, adapter_names, weights=None):
    """diffusers' set_adapters -> set_weights_and_activate_adapters."""
    names = [adapter_names] if isinstance(adapter_names, str) else list(adapter_names)
    weights = [1.0] * len(names) if weights is None else (weights if isinstance(weights, list) else [weights])
    for mname, m in lora_layers(model):
        m.set_adapter(names)
        for a, w in zip(names, weights):
            m.set_scale(a, get_module_weight(w, mname))


def scale_lora_layers(model, weight):
    if weight == 1.0:
        return
    for _, m in lora_layers(model):
        m.scale_layer(weight)


def unscale_lora_layers(model, weight=None):
    if weight is None or weight == 1.0:
        return
    for _, m in lora_layers(model):
        m.unscale_layer(weight)


def fuse_lora(model, lora_scale=1.0, adapter_names=None):
    """diffusers' fuse_lora: scale the active adapters, then PEFT's merge through `weight.data`."""
    for _, m in lora_layers(model):
        if lora_scale != 1.0:
            m.scale_layer(lora_scale)
        m.merge(adapter_names)


def unfuse_lora(model):
    for _, m in lora_layers(model):
        m.unmerge()


def enable_lora(model):
    for _, m in lora_layers(model):
        m.enable_adapters(True)


def disable_lora(model):
    for _, m in lora_layers(model):
        m.enable_adapters(False)


def delete_adapters(model, adapter_names):
    names = [adapter_names] if isinstance(adapter_names, str) else list(adapter_names)
    for a in names:
        for _, m in lora_layers(model):
            m.delete_adapter(a)
        getattr(model, "peft_config", {}).pop(a, None)
    if not getattr(model, "peft_config", None) and hasattr(model, "peft_config"):
        del model.peft_config


def unload_lora_weights(model):
    """diffusers' unload_lora_weights: every LoRA layer replaced by its base layer (a fused delta stays in it)."""
    for name, m in lora_layers(model):
        parent_name, _, key = name.rpartition(".")
        parent = model.get_submodule(parent_name) if parent_name else model
        parent._modules[key] = m.base_layer
    if hasattr(model, "peft_config"):
        del model.peft_config
