"""PEFT LoRA adapters on the native path: the active adapters are MERGED into the packed weights.

diffusers loads every LoRA through PEFT, which replaces each targeted ``nn.Linear`` / ``nn.Conv2d`` by a
wrapper holding the original module as ``base_layer`` and one ``lora_A`` / ``lora_B`` pair per adapter.  PEFT
computes an unfused adapter as a branch, ``y = base(x) + sum_i s_i * B_i(A_i(x))``.  Here the effective weight
``W + sum_i s_i * B_i A_i`` is formed on the GPU (``sfb_lora_merge``, one rounding to the packed dtype) whenever
the adapter state changes, and handed to the same packers as a plain parameter: a step runs the launch list
of the adapter-free model, and a switch re-packs only the tensors that read the changed layers, into the same
device storage (plans and captured graphs stay valid).

Per layer, the semantics are PEFT's ``Linear`` / ``Conv2d`` forward: adapters disabled or any adapter merged
-> the base weight alone (it already holds a merged delta); otherwise every active adapter present in
``lora_A`` with ``s = scaling[adapter]`` (which carries lora_alpha / r, rsLoRA, rank / alpha patterns and
diffusers' ``set_adapters`` weights), times the call's ``cross_attention_kwargs["scale"]`` on the UNet.
``peft`` is not a dependency: layers are recognised by their attributes.
"""
import math

import torch

from . import ops

_LORA_ATTRS = ("base_layer", "lora_A", "lora_B", "scaling", "r", "merged_adapters", "active_adapters",
               "disable_adapters")
SCALE_RTOL = 1e-6  # scale_lora_layers / unscale_lora_layers round trips may move the last bit


def is_lora_layer(m):
    return all(hasattr(m, a) for a in _LORA_ATTRS)


def plain_name(name):
    """diffusers' name of a (possibly PEFT-wrapped) module or parameter: '.base_layer' segments dropped."""
    return name.replace(".base_layer", "")


def _is_adapter_key(key):
    """A state-dict key that belongs to an adapter, not to the model (lora_A / lora_B / DoRA / LoHa / LoKr ...)."""
    return any(part.startswith(("lora_", "hada_", "lokr_")) for part in key.split("."))


def plain_state_dict(sd):
    """{diffusers name: tensor} of a module's state dict with any PEFT wrapping removed."""
    return {plain_name(k): v for k, v in sd.items() if not _is_adapter_key(k)}


def refuse_adapters(sd, what):
    """NotImplementedError naming the first PEFT-wrapped or legacy-LoRA layer in a state dict: for the modules
    whose adapters the native path does not compute (ControlNet, SVD UNet, VAE, vision tower)."""
    for k in sd:
        if ".base_layer." in k or ".lora_layer." in k or _is_adapter_key(k):
            layer = k.split(".base_layer.")[0].split(".lora_layer.")[0]
            raise NotImplementedError(
                f"sfast (H100 build): {what} layer {plain_name(layer)!r} carries an adapter (PEFT / LoRA); adapters "
                f"on the {what} are not supported by the H100 path: fuse_lora() and unload_lora_weights() first")


def scan(module, what="UNet"):
    """{diffusers prefix: PEFT LoRA layer} of `module`.  Refuses by name what the merge does not compute: a
    PEFT wrapper that is not LoRA, a base that is not Linear / Conv2d, diffusers' legacy `lora_layer`."""
    layers = {}
    for name, m in module.named_modules():
        if getattr(m, "lora_layer", None) is not None:
            raise NotImplementedError(
                f"sfast (H100 build): {what} layer {plain_name(name)!r} has a legacy diffusers `lora_layer`; load the "
                "LoRA through PEFT (current diffusers) or fuse it into the weights")
        if not hasattr(m, "base_layer"):
            continue
        if not is_lora_layer(m):
            kinds = sorted({n.split("_")[0] for n, _ in m.named_parameters() if n.startswith(("hada_", "lokr_"))})
            raise NotImplementedError(
                f"sfast (H100 build): {what} layer {plain_name(name)!r} is a PEFT {type(m).__name__} wrapper "
                f"{'(' + ', '.join(kinds) + ') ' if kinds else ''}that is not LoRA; only LoRA adapters are supported")
        if not isinstance(m.base_layer, (torch.nn.Linear, torch.nn.Conv2d)):
            raise NotImplementedError(f"sfast (H100 build): {what} LoRA layer {plain_name(name)!r} wraps a "
                                      f"{type(m.base_layer).__name__}; only Linear and Conv2d are supported")
        layers[plain_name(name)] = m
    return layers


def _active(layer):
    act = layer.active_adapters
    return [act] if isinstance(act, str) else list(act)


def effective_scales(layer, mult=1.0, name="?"):
    """((adapter, s), ...) that PEFT's forward adds to the base output of `layer`, s != 0; () = base only."""
    if layer.disable_adapters:
        if layer.merged_adapters:
            raise NotImplementedError(
                f"sfast (H100 build): LoRA layer {name!r} has adapters disabled while {list(layer.merged_adapters)} "
                "are merged (PEFT would unmerge them in its forward); call unfuse_lora() first")
        return ()
    if layer.merged_adapters:
        return ()
    out = []
    for a in _active(layer):
        if a in layer.lora_A:
            s = float(layer.scaling[a]) * mult
            if s != 0.0:
                out.append((a, s))
    return tuple(out)


def _layer_state(layer, mult, name):
    """What the merged weight of `layer` depends on besides tensor contents: (adapter, lora_A, lora_B, s) per
    adapter."""
    return tuple((a, layer.lora_A[a], layer.lora_B[a], s) for a, s in effective_scales(layer, mult, name))


def _same_state(x, y):
    if x is None or y is None or len(x) != len(y):
        return False
    return all(n0 == n1 and a0 is a1 and b0 is b1 and math.isclose(s0, s1, rel_tol=SCALE_RTOL, abs_tol=0.0)
               for (n0, a0, b0, s0), (n1, a1, b1, s1) in zip(x, y))


def check_layer(layer, state, name):
    """Refuse, by name, a layer whose merge sfb_lora_merge does not compute: more than 8 active adapters, or an
    adapter whose delta is not B A (DoRA, lora_bias, conv geometry) or whose rank exceeds 256."""
    if len(state) > ops._lib.LORA_MAX_ADAPTERS:
        raise NotImplementedError(f"sfast (H100 build): LoRA layer {name!r} has {len(state)} active adapters; "
                                  f"at most {ops._lib.LORA_MAX_ADAPTERS} are merged")
    for a, _, _, _ in state:
        _check_adapter(layer, a, name)


def _check_adapter(layer, a, name):
    if (getattr(layer, "use_dora", None) or {}).get(a, False):
        raise NotImplementedError(f"sfast (H100 build): LoRA layer {name!r} adapter {a!r} uses DoRA (use_dora); "
                                  "DoRA is not supported by the H100 path")
    if (getattr(layer, "lora_bias", None) or {}).get(a, False):
        raise NotImplementedError(f"sfast (H100 build): LoRA layer {name!r} adapter {a!r} has lora_bias; "
                                  "not supported by the H100 path")
    base, la, lb = layer.base_layer, layer.lora_A[a], layer.lora_B[a]
    if isinstance(base, torch.nn.Conv2d):
        ok = (isinstance(la, torch.nn.Conv2d) and isinstance(lb, torch.nn.Conv2d)
              and tuple(la.kernel_size) == tuple(base.kernel_size) and tuple(la.stride) == tuple(base.stride)
              and tuple(la.padding) == tuple(base.padding) and tuple(la.dilation) == tuple(base.dilation)
              and la.groups == base.groups == 1 and tuple(lb.kernel_size) == (1, 1) and tuple(lb.stride) == (1, 1))
        if not ok:
            raise NotImplementedError(
                f"sfast (H100 build): LoRA conv layer {name!r} adapter {a!r}: lora_A must share the base conv's "
                "kernel size, stride, padding and dilation and lora_B must be 1x1; not supported otherwise")
    if la.weight.shape[0] > ops._lib.LORA_MAX_RANK:
        raise NotImplementedError(f"sfast (H100 build): LoRA layer {name!r} adapter {a!r} has rank "
                                  f"{la.weight.shape[0]}; at most {ops._lib.LORA_MAX_RANK} is merged")


def merged_weight(layer, scales, out_dtype, device, name="?"):
    """W + sum_i s_i B_i A_i of `layer`, rounded once to out_dtype (sfb_lora_merge).  Conv weights: A is
    [r, cin*kh*kw] in OIHW order, B [cout, r]."""
    w = layer.base_layer.weight.detach().to(device)
    w2 = w.reshape(w.shape[0], -1)
    adapters = []
    for a, s in scales:
        A = layer.lora_A[a].weight.detach().to(device)
        B = layer.lora_B[a].weight.detach().to(device)
        adapters.append((A.reshape(A.shape[0], -1), B.reshape(B.shape[0], -1), s))
    return ops.lora_merge(w2.contiguous() if w2.stride(1) != 1 else w2, adapters, out_dtype).reshape(w.shape)


def _records(module):
    """(parent._modules, key, child) of every child that owns parameters or is a LoRA layer; the inside of a LoRA
    layer is covered by its state (poll) instead."""
    out, stack = [], [module]
    while stack:
        parent = stack.pop()
        for key, child in parent._modules.items():
            if child is None:
                continue
            wrapped = is_lora_layer(child)
            if wrapped or child._parameters:
                out.append((parent._modules, key, child))
            if not wrapped:
                stack.append(child)
    return out


def _snapshot(layer):
    """What a layer's state is computed from, copied: equal snapshots mean an equal state."""
    return (layer, layer._modules, dict(layer.scaling), list(layer.merged_adapters), list(layer.active_adapters),
            layer.disable_adapters, dict(layer.lora_A._modules), dict(layer.lora_B._modules))


class LoraTracker:
    """The LoRA layers of one compiled module and the adapter state last merged into its packed weights.

    Change detection needs no walk of the module tree per call: the (parent._modules, key, child) records of
    every module that owns parameters are compared by identity (loading or unloading an adapter swaps children),
    then every LoRA layer's scaling, merged / active / disabled state and adapter modules against a snapshot
    (C-level dict and list comparisons); only when one differs are the effective scales recomputed and compared
    with a tolerance.  A module with no LoRA layer and no ``peft_config`` (which PEFT sets on the model it
    injects into) costs one attribute lookup.  The caller sets `applied` to the polled states once they are
    packed."""

    def __init__(self, module, what="UNet"):
        self.module, self.what = module, what
        self.layers, self.records = {}, []
        self.applied = {}   # prefix -> state merged into the packed weights
        self.merges = 0     # sfb_lora_merge launches (tests: a steady state merges nothing)
        self._snap, self._snap_mult, self._states = [], None, {}
        self.rescan()

    def rescan(self):
        self.layers = scan(self.module, self.what)
        self._snap_mult = None
        if not self.layers and getattr(self.module, "peft_config", None) is None:
            self.records = []
            return
        self.records = _records(self.module)

    def quiet(self):
        return not self.layers and getattr(self.module, "peft_config", None) is None

    def poll(self, mult=1.0):
        """(changed prefixes, current states).  Changed: layers whose merged weight differs from the applied one
        (a re-scan after a child swap marks every layer of before and after).  Refuses, by name, a changed layer
        the merge does not compute, before anything is packed."""
        if self.quiet() and not self.applied:
            return set(), {}
        changed = set()
        if not self.records or any(d.get(k) is not c for d, k, c in self.records):
            changed |= set(self.layers)
            self.rescan()
            changed |= set(self.layers)
        elif mult == self._snap_mult and all(
                lay.scaling == sc and lay.merged_adapters == mg and lay.disable_adapters == dis
                and lay.active_adapters == ac and mods["lora_A"]._modules == am and mods["lora_B"]._modules == bm
                for lay, mods, sc, mg, ac, dis, am, bm in self._snap):
            if self._states is self.applied:
                return changed, self._states
        else:
            self._states = None
        if self._states is None or self._snap_mult is None:
            self._states = {p: _layer_state(lay, mult, p) for p, lay in self.layers.items()}
            self._snap = [_snapshot(lay) for lay in self.layers.values()]
            self._snap_mult = mult
        states = self._states
        changed |= {p for p, st in states.items() if not _same_state(st, self.applied.get(p, ()))}
        changed |= set(self.applied) - set(states)
        for p in changed & set(states):
            check_layer(self.layers[p], states[p], p)
        if not changed:  # equal within the tolerance: keep what was packed
            self._states = self.applied
        return changed, self._states

    def view(self, raw_sd, states, dtype, device, dry):
        return EffectiveStateDict(self, plain_state_dict(raw_sd), states, dtype, device, dry)


class EffectiveStateDict(dict):
    """{diffusers name: tensor} whose adapted weights are merged on first read (not kept: the packers copy)."""

    def __init__(self, tracker, plain, states, dtype, device, dry):
        super().__init__(plain)
        self.tracker, self.states, self.dtype, self.device, self.dry = tracker, states, dtype, device, dry

    def __getitem__(self, name):
        prefix, _, leaf = name.rpartition(".")
        st = self.states.get(prefix)
        if leaf != "weight" or not st or self.dry:
            return super().__getitem__(name)
        self.tracker.merges += 1
        return merged_weight(self.tracker.layers[prefix], [(a, s) for a, _, _, s in st], self.dtype, self.device,
                             prefix)
