"""Runtime that replaces ``unet.forward``: per-(batch, H, W, dtype) plan cache + CUDA-graph replay.

Reference counterparts: the lazy-trace wrapper (/root/reference/src/sfast/jit/trace_helper.py:
33-72) and the dynamic CUDA-graph cache (/root/reference/src/sfast/cuda/graphs.py:16-51,
147-157).  Same contract: inputs are copied into static buffers, the graph is replayed, the
output is returned as a fresh clone, all under a per-object lock; unlike the reference the
timestep is always read from device memory inside the graph (never keyed by value,
graphs.py:229-231).
"""
import functools
import logging
import math
import threading
import time

import torch

from . import lora
from .motion_plan import MotionUNetPlan
from .plan import PackedWeights, UNetPlan, intrablock_shapes
from .svd_plan import SVDPlan
from .unet_spec import cfg_get, ip_adapter_spec, ip_scale_of, spec_from_config

logger = logging.getLogger(__name__)

try:  # diffusers is not a dependency; use its output type when present
    from diffusers.models.unets.unet_2d_condition import UNet2DConditionOutput  # type: ignore
except Exception:  # noqa: BLE001
    class UNet2DConditionOutput(dict):
        """Minimal stand-in for diffusers' BaseOutput: attribute, key and index access."""

        def __init__(self, sample):
            super().__init__(sample=sample)
            self.sample = sample

        def __getitem__(self, k):
            if isinstance(k, int):
                return tuple(self.values())[k]
            return super().__getitem__(k)

        def to_tuple(self):
            return tuple(self.values())


try:  # the AnimateDiff UNet's output class (diffusers >= 0.28); the 2-D one has the same fields
    from diffusers.models.unets.unet_motion_model import UNetMotionOutput  # type: ignore
except Exception:  # noqa: BLE001
    UNetMotionOutput = UNet2DConditionOutput


_UNSUPPORTED_KWARGS = ("class_labels", "attention_mask", "encoder_attention_mask")


class LegacyResidualShapeError(ValueError, NotImplementedError):
    """A residual of diffusers' deprecated T2I-Adapter form (``down_block_additional_residuals`` without
    ``mid_block_additional_residual``) whose shape fits no insertion point.  Such a list is most likely a
    ControlNet's down residuals passed without their mid residual, which the UNet refuses: the error is also
    the NotImplementedError it raised for that call before the T2I-Adapter form was supported."""


def require_sm90(device):
    if device.type != "cuda" or not torch.cuda.is_available():
        raise RuntimeError("sfast (H100 build): the UNet hot path needs a CUDA sm_90 device; "
                           "there is no CPU / eager fallback")
    major, minor = torch.cuda.get_device_capability(device)
    if (major, minor) != (9, 0):  # the cubin is sm_90a (wgmma): it loads on no other architecture
        raise RuntimeError(f"sfast (H100 build): kernels are sm_90a only, device is sm_{major}{minor}")


class _GraphedPlan:
    def __init__(self, plan: UNetPlan, use_graph: bool):
        self.plan = plan
        self.graph = None
        stream = torch.cuda.current_stream()
        # warm-up (also sets kernel attributes, which must not happen during capture)
        side = torch.cuda.Stream()
        side.wait_stream(stream)
        with torch.cuda.stream(side):
            plan.run()
        stream.wait_stream(side)
        torch.cuda.synchronize()
        if use_graph:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                plan.run()
            self.graph = g

    def step(self):
        if self.graph is not None:
            self.graph.replay()
        else:
            self.plan.run()


class _CompiledModule:
    """What every compiled module shares: one packed copy of the weights and a cache of plans + CUDA graphs,
    used under one lock.

    Reference contract (preserve_parameters=True): an in-place parameter update is seen by the next call.
    The packed weights are copies, so the parameters' version counters are compared on every call and the
    copies refreshed in place when they moved.

    `lora_module`: the torch module whose PEFT LoRA layers are merged into the packed weights
    (lora.LoraTracker); without it, a module carrying adapters is refused by name when its weights are packed."""

    _what = "module"  # for log messages

    def __init__(self, spec, state_dict_fn, enable_cuda_graph=True, preserve_parameters=True, lora_module=None):
        self.spec = spec
        self._state_dict_fn = state_dict_fn
        self.enable_cuda_graph = enable_cuda_graph
        self.preserve_parameters = preserve_parameters
        self._weights = None
        self._param_refs = None
        self._param_versions = None
        self._cached = {}
        self._lock = threading.Lock()
        self._warned = set()
        self._lora = lora.LoraTracker(lora_module, self._what) if isinstance(lora_module, torch.nn.Module) else None
        self._lora_scale = 1.0      # call-time LoRA scale merged into the packed weights
        self._lora_states = None    # adapter state of the next (re-)pack
        self._lora_frozen = False   # preserve_parameters=False: adapter state frozen until rebind()
        self._repack_all = False    # a re-pack failed part-way: the next one re-runs every packer
        # a module whose adapters are not merged: PEFT's peft_config appearing on it is refused at the next call
        self._unmerged_module = None if self._lora is not None else getattr(state_dict_fn, "__self__", None)

    def _warn_once(self, what, msg, *args):
        if what not in self._warned:
            logger.warning(msg, *args)
            self._warned.add(what)

    def _track(self, sd):
        self._param_refs = [t for t in sd.values() if torch.is_tensor(t)]
        self._param_versions = [t._version for t in self._param_refs]

    def _weights_for(self, dtype, device, lora_scale=1.0):
        """The packed weights for (dtype, device): packed on first use and re-packed when either changes (the
        plans of the old copy are dropped); refreshed in place when the parameters' version counters moved, and
        the layers whose LoRA adapter state changed (at `lora_scale`, the call's LoRA scale) re-merged and
        re-packed.  The caller holds the lock and `device` is current."""
        w, lo = self._weights, self._lora
        if w is None or w.dtype != dtype or w.device != device:
            logger.info("Packing %s weights for the H100 path (%s, %s)", self._what, dtype, device)
            self._poll_lora(lora_scale)
            sd = self._state_dict_fn()
            self._weights = PackedWeights(self.spec, self._packed_state_dict(sd, dtype, device), dtype, device)
            self._applied()
            self._track(sd)
            self._cached.clear()
        elif self.preserve_parameters or (lo is not None and not self._lora_frozen):
            if lo is None and getattr(self._unmerged_module, "peft_config", None) is not None:
                lora.refuse_adapters(self._state_dict_fn(), self._what)
            changed = self._poll_lora(lora_scale)
            if self._repack_all or (self.preserve_parameters
                                    and [t._version for t in self._param_refs] != self._param_versions):
                logger.info("%s parameters changed in place: refreshing the packed weights", self._what)
                self._refresh_locked()
            elif changed:
                logger.info("%s LoRA adapter state changed: re-merging %d layers", self._what, len(changed))
                self._refresh_locked({p + ".weight" for p in changed})
        elif lo is not None and not math.isclose(lora_scale, self._lora_scale, rel_tol=lora.SCALE_RTOL):
            raise NotImplementedError(
                f"sfast (H100 build): LoRA scale {lora_scale} differs from the scale {self._lora_scale} frozen into the "
                f"packed {self._what} weights (preserve_parameters=False); call rebind() to re-merge")
        if lora_scale != 1.0 and (lo is None or not lo.layers):
            raise NotImplementedError("sfast (H100 build): cross_attention_kwargs (LoRA scale) "
                                      "is not supported; fuse the LoRA weights into the parameters")
        self._lora_frozen = not self.preserve_parameters
        return self._weights

    def _poll_lora(self, lora_scale):
        """Prefixes of the LoRA layers whose adapter state changed; keeps their state for the next re-pack."""
        if self._lora is None:
            return set()
        changed, self._lora_states = self._lora.poll(lora_scale)
        self._lora_scale = lora_scale
        return changed

    def _packed_state_dict(self, sd, dtype, device):
        """What PackedWeights reads: the state dict itself, or, with LoRA layers, their merged weights under
        diffusers' names (the polled adapter state)."""
        if self._lora is None:
            lora.refuse_adapters(sd, self._what)
            return sd
        return self._lora.view(sd, self._lora_states, dtype, device, dry=False)

    def _applied(self):
        """The polled adapter state is now in the packed weights."""
        if self._lora is not None:
            self._lora.applied = self._lora_states

    def _refresh_locked(self, names=None):
        sd = self._state_dict_fn()
        torch.cuda.current_stream().synchronize()  # no replay may be reading the old values
        w = self._weights
        sd_packed = self._packed_state_dict(sd, w.dtype, w.device)
        try:
            w.refresh(sd_packed) if names is None else w.refresh(sd_packed, names)
        except BaseException:
            # some packers may hold the new state and others the old one: nothing is marked applied, and the
            # next call re-packs everything (or raises again)
            self._repack_all = True
            raise
        self._repack_all = False
        self._applied()
        self._track(sd)

    def rebind(self):
        """Re-pack the weights now (same device storage: plans and CUDA graphs stay valid).
        Only needed with preserve_parameters=False or after replacing parameter objects in a way
        the version counters cannot see.  With preserve_parameters=False it also releases the frozen LoRA
        adapter state: the next call merges the adapters and LoRA scale current at that call."""
        with self._lock:
            if self._weights is not None:
                with torch.cuda.device(self._weights.device):
                    self._poll_lora(self._lora_scale)
                    self._refresh_locked()
                    self._lora_frozen = False

    def _graphed(self, key, make_plan):
        """The plan + graph cached under `key`, built by make_plan() on first use (caller holds the lock)."""
        gp = self._cached.get(key)
        if gp is None:
            logger.info("Building %s launch plan for %s", self._what, key)
            gp = _GraphedPlan(make_plan(), self.enable_cuda_graph)
            self._cached[key] = gp
        return gp


def _install(m, name, compiled, fn):
    """Replace m.<name> by fn, which carries the compiled object and its plan cache."""
    fn.__self__ = m
    fn._cached = compiled._cached
    fn._compiled = compiled
    setattr(m, name, fn)
    return m


class CompiledUNet(_CompiledModule):
    """Callable with the signature of diffusers ``UNet2DConditionModel.forward``."""

    _what = "UNet"

    def __init__(self, config, state_dict_fn, enable_cuda_graph=True, preserve_parameters=True, module=None):
        """`module`: the UNet itself.  It is where a loaded IP-Adapter lives (``encoder_hid_proj`` and the
        cross-attention processors, whose ``scale`` is read on every call); without it no adapter can be
        compiled."""
        spec = spec_from_config(config)
        # PEFT LoRA layers are merged into the 2-D UNet's weights; the SVD UNet refuses them by name
        super().__init__(spec, state_dict_fn, enable_cuda_graph, preserve_parameters,
                         lora_module=None if spec.temporal else module)
        self.first_call_s = None  # wall time of the first call (packing + plan + capture)
        self._module = module
        self._ip_proj = getattr(module, "encoder_hid_proj", None)
        self._ip_procs = None
        if spec.motion:
            pass  # an IP-Adapter on the motion UNet is refused by name on every call (_motion_refusals)
        elif cfg_get(config, "encoder_hid_dim_type") == "ip_image_proj" or self._ip_proj is not None:
            if module is None:
                raise NotImplementedError("sfast (H100 build): an IP-Adapter UNet is compiled from the module "
                                          "(compile_unet_module), not from its config alone")
            self.spec.ip = ip_adapter_spec(module, self.spec)
            self._ip_procs = [module.get_submodule(p).processor for p in self.spec.ip.layers]

    def _ip_inputs(self, added_cond_kwargs, cross_attention_kwargs, B):
        """(ip_len, ip_seq, image embeddings, per-layer scales) of this call; (0, 0, None, None) without an
        adapter.  The embeddings are [B * n_img, D_img] for a plain adapter (ip_seq 0) and the image features
        [B * n_img * ip_seq, D_img] for IP-Adapter Plus.  Refuses, by name, what the fused attention does not
        compute."""
        if cross_attention_kwargs and "ip_adapter_masks" in cross_attention_kwargs:
            raise NotImplementedError("sfast (H100 build): cross_attention_kwargs['ip_adapter_masks'] (IP-Adapter "
                                      "masks) is not supported by the H100 path")
        if self._module is not None and getattr(self._module, "encoder_hid_proj", None) is not self._ip_proj:
            raise NotImplementedError("sfast (H100 build): the UNet's IP-Adapter was loaded, unloaded or replaced "
                                      "after compile(); call compile() again")
        ip = self.spec.ip
        if ip is None:
            return 0, 0, None, None
        if not added_cond_kwargs or "image_embeds" not in added_cond_kwargs:
            raise ValueError(f"{type(self._module).__name__} has the config param `encoder_hid_dim_type` set to "
                             "'ip_image_proj' which requires the keyword argument `image_embeds` to be passed in "
                             "`added_cond_kwargs`")
        emb = added_cond_kwargs["image_embeds"]
        bare = not isinstance(emb, (list, tuple))
        if not bare:
            if len(emb) != 1:
                raise NotImplementedError(f"sfast (H100 build): {len(emb)} image_embeds entries (one per "
                                          "IP-Adapter); one adapter is supported")
            emb = emb[0]
        if ip.resampler is not None:
            # IP-Adapter Plus: image features (the vision tower's hidden_states[-2]) [B, n_img, S_img, D_img]; the
            # deprecated bare [B, S_img, D_img] form is one image per sample
            if bare and emb.dim() == 3:
                emb = emb.unsqueeze(1)
            if emb.dim() != 4 or emb.shape[0] != B or emb.shape[3] != ip.image_embed_dim or emb.shape[2] < 1:
                raise ValueError(f"image_embeds of shape {tuple(emb.shape)}: expected [{B}, n_images, S_img, "
                                 f"{ip.image_embed_dim}] (IP-Adapter Plus image features)")
            ip_seq = emb.shape[2]
        else:
            if emb.dim() == 2:  # diffusers' deprecated bare [B, D_img] form: one image per sample
                emb = emb.unsqueeze(1)
            if emb.dim() != 3 or emb.shape[0] != B or emb.shape[2] != ip.image_embed_dim:
                raise ValueError(f"image_embeds of shape {tuple(emb.shape)}: expected [{B}, n_images, "
                                 f"{ip.image_embed_dim}]")
            ip_seq = 0
        scales = [ip_scale_of(p, n) for p, n in zip(self._ip_procs, ip.layers)]
        return emb.shape[1] * ip.tokens, ip_seq, emb.reshape(-1, ip.image_embed_dim), scales

    def _intrablock_inputs(self, residuals, B, H, W, legacy):
        """The T2I-Adapter residuals this call adds, in order: one per down block, then the mid-block one when
        the next residual has the mid output's shape (diffusers' rule for T2I-Adapter-XL); any further ones are
        ignored, as diffusers ignores them.  The caller's list is not modified (diffusers pops from it).  Raises
        ValueError naming the index of a down-block residual whose shape does not fit."""
        points = intrablock_shapes(self.spec, B, H, W)
        n_down = len(points) - 1
        res = list(residuals)
        arg = "down_block_additional_residuals" if legacy else "down_intrablock_additional_residuals"
        for i, r in enumerate(res[:n_down]):
            if tuple(r.shape) != points[i]:
                msg = (f"{arg}[{i}] has shape {tuple(r.shape)}; down block {i} adds a T2I-Adapter residual of "
                       f"shape {points[i]}")
                if legacy:
                    raise LegacyResidualShapeError(
                        msg + " (without mid_block_additional_residual this is diffusers' deprecated T2I-Adapter "
                        "form; ControlNet residuals need both down_block_additional_residuals and "
                        "mid_block_additional_residual)")
                raise ValueError(msg)
        n = min(len(res), n_down)
        if len(res) > n_down and tuple(res[n_down].shape) == points[n_down]:
            n += 1
        return res[:n]

    def _freeu_state(self):
        """((on0, on1), [b1, s1, b2, s2]) of this call: the FreeU attributes diffusers' ``enable_freeu`` sets on
        ``up_blocks[0]`` and ``[1]``.  Like diffusers' up blocks, a block applies FreeU only when all four of its
        own s1, s2, b1, b2 are truthy (so a zero switches it off, and ``disable_freeu`` sets them to None); block 0
        uses its b1 / s1, block 1 its b2 / s2.  Later up blocks do nothing in diffusers either.  Without the
        module (compiled from its config alone) FreeU is off."""
        blocks = getattr(self._module, "up_blocks", None)
        if blocks is None or len(blocks) < 2:
            return (False, False), None
        on = tuple(all(getattr(blk, k, None) for k in ("s1", "s2", "b1", "b2")) for blk in blocks[:2])
        if not any(on):
            return on, None
        vals = [0.0] * 4
        for i, (b, s) in enumerate((("b1", "s1"), ("b2", "s2"))):
            if on[i]:
                vals[2 * i], vals[2 * i + 1] = float(getattr(blocks[i], b)), float(getattr(blocks[i], s))
        return on, vals

    def _timestep_cond_input(self, timestep_cond, B):
        """The [B, time_cond_proj_dim] guidance embedding this call copies into the plan's `timestep_cond_in`, or
        None for a UNet without time_embedding.cond_proj (which refuses the argument by name).  [1, dim] is
        broadcast over the batch, as diffusers' add broadcasts it; None is zeros: diffusers then skips the add, and
        adding an exact zero to the timestep embedding gives the same bits."""
        dim = self.spec.time_cond_dim
        if not dim:
            if timestep_cond is not None:
                raise NotImplementedError("sfast (H100 build): UNet argument `timestep_cond` is not supported (the "
                                          "UNet has no time_cond_proj_dim)")
            return None
        if timestep_cond is None:
            return torch.zeros(B, dim)
        shape = tuple(timestep_cond.shape)
        if shape not in ((B, dim), (1, dim)):
            raise ValueError(f"timestep_cond of shape {shape}: expected [{B}, {dim}] or [1, {dim}]")
        return timestep_cond.expand(B, dim)

    # -- forward -------------------------------------------------------------------------
    def _call_svd(self, sample, timestep, encoder_hidden_states, added_time_ids, return_dict=True):
        """diffusers UNetSpatioTemporalConditionModel.forward(sample [B, F, C, H, W], timestep,
        encoder_hidden_states [B, 1, ctx], added_time_ids [B, 3])."""
        require_sm90(sample.device)
        dtype = sample.dtype
        if dtype not in (torch.float16, torch.bfloat16):
            raise NotImplementedError(f"sfast (H100 build): UNet dtype {dtype}; use fp16 or bf16")
        B, F_, _, H, W = sample.shape
        if F_ != self.spec.num_frames:
            raise NotImplementedError(f"sfast (H100 build): {F_} frames, the UNet was configured for "
                                      f"{self.spec.num_frames}")
        if encoder_hidden_states.shape[1] != 1:
            raise NotImplementedError("sfast (H100 build): SVD path needs a single-token encoder_hidden_states")
        with self._lock, torch.cuda.device(sample.device):
            t_first = time.perf_counter() if self.first_call_s is None else None
            weights = self._weights_for(dtype, sample.device)
            gp = self._graphed(("svd", B, H, W, dtype, sample.device.index), lambda: SVDPlan(weights, B, H, W))
            plan = gp.plan
            plan.sample_in.copy_(sample.reshape(B * F_, -1, H, W), non_blocking=True)
            plan.ehs_in.copy_(encoder_hidden_states.repeat_interleave(F_, dim=0), non_blocking=True)
            t = timestep if torch.is_tensor(timestep) else torch.tensor(float(timestep))
            t = t.reshape(-1).to(device=sample.device, dtype=torch.float32, non_blocking=True)
            plan.t_in.copy_((t.expand(B) if t.numel() == 1 else t).repeat_interleave(F_))
            plan.time_ids_in.copy_(added_time_ids.to(device=sample.device, dtype=torch.float32)
                                   .repeat_interleave(F_, dim=0).reshape(-1))
            gp.step()
            out = plan.out.clone().reshape(B, F_, -1, H, W)
            if t_first is not None:
                torch.cuda.current_stream().synchronize()
                self.first_call_s = time.perf_counter() - t_first
        if not return_dict:
            return (out,)
        return UNet2DConditionOutput(sample=out)

    def _motion_refusals(self, attention_mask, down_intrablock_additional_residuals):
        """NotImplementedError naming what the motion UNet's plan does not compute.  Everything here can change
        after compile() (an adapter loaded, FreeU or FreeNoise switched on), so it is checked on every call."""
        def refuse(what):
            raise NotImplementedError(f"sfast (H100 build): {what} is not supported by the H100 path on the "
                                      "AnimateDiff UNet (UNetMotionModel)")
        if attention_mask is not None:
            refuse("UNet argument `attention_mask`")
        if down_intrablock_additional_residuals is not None:
            refuse("`down_intrablock_additional_residuals` (T2I-Adapter)")
        m = self._module
        if cfg_get(getattr(m, "config", None), "encoder_hid_dim_type") == "ip_image_proj" or \
                getattr(m, "encoder_hid_proj", None) is not None:
            refuse("an IP-Adapter")
        if m is None:
            return
        if any(getattr(blk, k, None) for blk in getattr(m, "up_blocks", ()) for k in ("s1", "s2", "b1", "b2")):
            refuse("FreeU (enable_freeu)")
        for mm in self.spec.motion:
            try:
                mod = m.get_submodule(mm.prefix)
            except AttributeError:
                continue
            for blk in getattr(mod, "transformer_blocks", ()):
                if type(blk).__name__ == "FreeNoiseTransformerBlock":
                    refuse(f"FreeNoise (enable_free_noise: {mm.prefix} runs FreeNoiseTransformerBlock)")

    def _call_motion(self, sample, timestep, encoder_hidden_states, timestep_cond=None, attention_mask=None,
                     cross_attention_kwargs=None, added_cond_kwargs=None, down_block_additional_residuals=None,
                     mid_block_additional_residual=None, down_intrablock_additional_residuals=None, return_dict=True):
        """diffusers UNetMotionModel.forward(sample [B, C, F, H, W], timestep, encoder_hidden_states [B, L, ctx],
        ...): the F frames of each video are a batch of B*F images, and the time embedding (with an LCM's
        timestep_cond and SDXL's added_cond_kwargs) and the prompt are repeated per frame, as diffusers repeats
        them.  ControlNet residuals are [B*F, C, h, w].  Returns [B, C_out, F, H, W]."""
        self._motion_refusals(attention_mask, down_intrablock_additional_residuals)
        if sample.dim() != 5:
            raise ValueError(f"sample of shape {tuple(sample.shape)}: the motion UNet takes [B, C, F, H, W]")
        B, _, F_, H, W = sample.shape
        max_seq = min(m.max_seq_len for m in self.spec.motion)
        if F_ > max_seq:
            raise NotImplementedError(f"sfast (H100 build): {F_} frames; the motion modules take at most "
                                      f"motion_max_seq_length = {max_seq} (FreeNoise's sliding windows are not "
                                      "supported)")
        t_cond = self._timestep_cond_input(timestep_cond, B)
        lora_scale = 1.0
        if cross_attention_kwargs:
            lora_scale = float(cross_attention_kwargs.get("scale", 1.0))
            if set(cross_attention_kwargs) - {"scale"} or (lora_scale != 1.0 and (self._lora is None or self._lora.quiet())):
                raise NotImplementedError("sfast (H100 build): cross_attention_kwargs (LoRA scale) "
                                          "is not supported; fuse the LoRA weights into the parameters")
        require_sm90(sample.device)
        dtype = sample.dtype
        if dtype not in (torch.float16, torch.bfloat16):
            raise NotImplementedError(f"sfast (H100 build): UNet dtype {dtype}; use fp16 or bf16")
        controlnet = down_block_additional_residuals is not None or mid_block_additional_residual is not None
        if controlnet and (down_block_additional_residuals is None or mid_block_additional_residual is None):
            raise NotImplementedError("sfast (H100 build): ControlNet residuals need both "
                                      "down_block_additional_residuals and mid_block_additional_residual")
        ctx_len = encoder_hidden_states.shape[1]
        with self._lock, torch.cuda.device(sample.device):
            t_first = time.perf_counter() if self.first_call_s is None else None
            weights = self._weights_for(dtype, sample.device, lora_scale)
            gp = self._graphed(("motion", B, F_, H, W, dtype, ctx_len, sample.device.index, controlnet),
                               lambda: MotionUNetPlan(weights, B, F_, H, W, ctx_len, controlnet=controlnet))
            plan = gp.plan
            # [B, C, F, H, W] -> the static [B*F, C, H, W] input, permuted by the copy itself
            plan.sample_in.view(B, F_, -1, H, W).copy_(sample.permute(0, 2, 1, 3, 4), non_blocking=True)
            plan.ehs_in.view(B, F_, ctx_len, -1).copy_(encoder_hidden_states.unsqueeze(1), non_blocking=True)
            t = timestep if torch.is_tensor(timestep) else torch.tensor(float(timestep))
            t = t.reshape(-1).to(device=sample.device, dtype=torch.float32, non_blocking=True)
            plan.t_in.copy_((t.expand(B) if t.numel() == 1 else t).repeat_interleave(F_))
            if t_cond is not None:
                plan.timestep_cond_in.copy_(t_cond.repeat_interleave(F_, dim=0))
            if self.spec.addition_embed_type == "text_time":
                if not added_cond_kwargs or "text_embeds" not in added_cond_kwargs:
                    raise ValueError("added_cond_kwargs with text_embeds / time_ids is required")
                te = added_cond_kwargs["text_embeds"]
                plan.add_in[:, :te.shape[1]].copy_(te.repeat_interleave(F_, dim=0))
                plan.time_ids_in.copy_(added_cond_kwargs["time_ids"].reshape(B, -1).float()
                                       .repeat_interleave(F_, dim=0).reshape(-1))
            if controlnet:
                res = list(down_block_additional_residuals) + [mid_block_additional_residual]
                if len(res) != len(plan.ctrl_in):
                    raise ValueError(f"expected {len(plan.ctrl_in) - 1} down-block residuals, got {len(res) - 1}")
                for dst, src in zip(plan.ctrl_in, res):
                    if tuple(src.shape) != tuple(dst.shape):
                        raise ValueError(f"ControlNet residual shape {tuple(src.shape)} != {tuple(dst.shape)} "
                                         "(the motion UNet takes [B * frames, C, h, w])")
                    dst.copy_(src, non_blocking=True)
            gp.step()
            out = plan.out.view(B, F_, -1, H, W).permute(0, 2, 1, 3, 4).contiguous()
            if t_first is not None:
                torch.cuda.current_stream().synchronize()
                self.first_call_s = time.perf_counter() - t_first
        if not return_dict:
            return (out,)
        return UNetMotionOutput(sample=out)

    def __call__(self, sample, timestep, encoder_hidden_states, *args, **kwargs):
        if self.spec.temporal:
            return self._call_svd(sample, timestep, encoder_hidden_states, *args, **kwargs)
        if self.spec.motion:
            return self._call_motion(sample, timestep, encoder_hidden_states, *args, **kwargs)
        return self._call_2d(sample, timestep, encoder_hidden_states, *args, **kwargs)

    def _call_2d(self, sample, timestep, encoder_hidden_states, class_labels=None,
                 timestep_cond=None, attention_mask=None, cross_attention_kwargs=None,
                 added_cond_kwargs=None, down_block_additional_residuals=None,
                 mid_block_additional_residual=None, down_intrablock_additional_residuals=None,
                 encoder_attention_mask=None, return_dict=True):
        given = dict(class_labels=class_labels, attention_mask=attention_mask,
                     encoder_attention_mask=encoder_attention_mask)
        for k in _UNSUPPORTED_KWARGS:
            if given[k] is not None:
                raise NotImplementedError(f"sfast (H100 build): UNet argument `{k}` is not supported")
        B, _, H, W = sample.shape
        t_cond = self._timestep_cond_input(timestep_cond, B)
        ip_len, ip_seq, image_embeds, ip_scales = self._ip_inputs(added_cond_kwargs, cross_attention_kwargs, B)
        lora_scale = 1.0
        if cross_attention_kwargs:
            lora_scale = float(cross_attention_kwargs.get("scale", 1.0))
            if set(cross_attention_kwargs) - {"scale"} or (lora_scale != 1.0 and (self._lora is None or self._lora.quiet())):
                raise NotImplementedError("sfast (H100 build): cross_attention_kwargs (LoRA scale) "
                                          "is not supported; fuse the LoRA weights into the parameters")
        require_sm90(sample.device)
        dtype = sample.dtype
        if dtype not in (torch.float16, torch.bfloat16):
            raise NotImplementedError(f"sfast (H100 build): UNet dtype {dtype}; use fp16 or bf16")
        ctx_len = encoder_hidden_states.shape[1]
        legacy = (down_intrablock_additional_residuals is None and mid_block_additional_residual is None
                  and down_block_additional_residuals is not None)
        if legacy:  # diffusers' deprecated T2I-Adapter form: the down residuals are the adapter's
            down_intrablock_additional_residuals, down_block_additional_residuals = down_block_additional_residuals, None
        controlnet = down_block_additional_residuals is not None or mid_block_additional_residual is not None
        if controlnet and (down_block_additional_residuals is None or mid_block_additional_residual is None):
            raise NotImplementedError("sfast (H100 build): ControlNet residuals need both "
                                      "down_block_additional_residuals and mid_block_additional_residual")
        intrablock = []
        if down_intrablock_additional_residuals is not None:
            intrablock = self._intrablock_inputs(down_intrablock_additional_residuals, B, H, W, legacy)
        freeu, freeu_vals = self._freeu_state()
        # everything below (allocation, TMA maps, launches, capture) targets sample's device
        with self._lock, torch.cuda.device(sample.device):
            t_first = time.perf_counter() if self.first_call_s is None else None
            weights = self._weights_for(dtype, sample.device, lora_scale)
            gp = self._graphed((B, H, W, dtype, ctx_len, sample.device.index, controlnet, ip_len, ip_seq, freeu,
                                len(intrablock)),
                               lambda: UNetPlan(weights, B, H, W, ctx_len, controlnet=controlnet, ip_len=ip_len,
                                                ip_seq=ip_seq, intrablock=len(intrablock), freeu=freeu))
            plan = gp.plan
            for dst, src in zip(plan.intrablock_in, intrablock):
                dst.copy_(src, non_blocking=True)
            if freeu_vals is not None:
                plan.freeu_in.copy_(torch.tensor(freeu_vals, dtype=torch.float32))
            if ip_len:
                plan.image_embeds_in.copy_(image_embeds, non_blocking=True)
                plan.ip_scale_in.copy_(torch.tensor(ip_scales, dtype=torch.float32))
            plan.sample_in.copy_(sample, non_blocking=True)
            plan.ehs_in.copy_(encoder_hidden_states, non_blocking=True)
            t = timestep if torch.is_tensor(timestep) else torch.tensor(float(timestep))
            t = t.reshape(-1).to(device=sample.device, dtype=torch.float32, non_blocking=True)
            plan.t_in.copy_(t.expand(B) if t.numel() == 1 else t)
            if t_cond is not None:
                plan.timestep_cond_in.copy_(t_cond)
            if self.spec.addition_embed_type == "text_time":
                if not added_cond_kwargs or "text_embeds" not in added_cond_kwargs:
                    raise ValueError("added_cond_kwargs with text_embeds / time_ids is required")
                te = added_cond_kwargs["text_embeds"]
                plan.add_in[:, :te.shape[1]].copy_(te)
                plan.time_ids_in.copy_(added_cond_kwargs["time_ids"].reshape(-1).float())
            if controlnet:
                res = list(down_block_additional_residuals) + [mid_block_additional_residual]
                if len(res) != len(plan.ctrl_in):
                    raise ValueError(f"expected {len(plan.ctrl_in) - 1} down-block residuals, got {len(res) - 1}")
                for dst, src in zip(plan.ctrl_in, res):
                    if tuple(src.shape) != tuple(dst.shape):
                        raise ValueError(f"ControlNet residual shape {tuple(src.shape)} != {tuple(dst.shape)}")
                    dst.copy_(src, non_blocking=True)
            gp.step()
            out = plan.out.clone()
            if t_first is not None:
                torch.cuda.current_stream().synchronize()
                self.first_call_s = time.perf_counter() - t_first
        if not return_dict:
            return (out,)
        return UNet2DConditionOutput(sample=out)


class DecoderOutput(dict):
    """Stand-in for diffusers' DecoderOutput (attribute, key and index access)."""

    def __init__(self, sample):
        super().__init__(sample=sample)
        self.sample = sample

    def __getitem__(self, k):
        return tuple(self.values())[k] if isinstance(k, int) else super().__getitem__(k)


class AutoencoderKLOutput(dict):
    """Stand-in for diffusers' AutoencoderKLOutput (attribute, key and index access)."""

    def __init__(self, latent_dist):
        super().__init__(latent_dist=latent_dist)
        self.latent_dist = latent_dist

    def __getitem__(self, k):
        return tuple(self.values())[k] if isinstance(k, int) else super().__getitem__(k)


class DiagonalGaussianDistribution:
    """Stand-in for diffusers' DiagonalGaussianDistribution over the encoder's moments [B, 2 * C, h, w]
    (mean | log-variance along dim 1)."""

    def __init__(self, parameters, deterministic=False):
        self.parameters = parameters
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.deterministic = deterministic
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)
        if deterministic:
            self.var = self.std = torch.zeros_like(self.mean)

    def sample(self, generator=None):
        # diffusers' randn_tensor: drawn in the moments' dtype on the generator's device when that is the
        # CPU, else on the moments' device; one [1, ...] draw per generator when given a list
        shape, dev, dt = tuple(self.mean.shape), self.parameters.device, self.parameters.dtype
        g0 = generator[0] if isinstance(generator, (list, tuple)) else generator
        rdev = torch.device("cpu") if g0 is not None and g0.device.type == "cpu" else dev
        if isinstance(generator, (list, tuple)):
            eps = torch.cat([torch.randn((1,) + shape[1:], generator=g, device=rdev, dtype=dt) for g in generator])
        else:
            eps = torch.randn(shape, generator=generator, device=rdev, dtype=dt)
        return self.mean + self.std * eps.to(dev)

    def mode(self):
        return self.mean


@functools.lru_cache(maxsize=None)
def _latent_dist_classes():
    """(AutoencoderKLOutput, DiagonalGaussianDistribution): diffusers' own where it imports."""
    try:
        from diffusers.models.autoencoders.vae import DiagonalGaussianDistribution as DGD  # type: ignore
        from diffusers.models.modeling_outputs import AutoencoderKLOutput as Out  # type: ignore
        return Out, DGD
    except Exception:  # noqa: BLE001
        return AutoencoderKLOutput, DiagonalGaussianDistribution


def temporal_decoder(state_dict):
    """True for a VAE whose decoder is not the 2-D `Decoder` the native path runs: SVD's
    AutoencoderKLTemporalDecoder has no post_quant_conv and takes decode(z, num_frames=...)."""
    return "post_quant_conv.weight" not in state_dict


class CompiledVAE(_CompiledModule):
    """`AutoencoderKL.decode(z, return_dict=True, generator=None)` and `encode(x, return_dict=True)` on the
    native path.  Both share one packed copy of the weights and one cache of plans + CUDA graphs keyed by
    (kind, B, H, W, dtype, device)."""

    _what = "VAE"

    def __init__(self, module, eager_decode, eager_encode, enable_cuda_graph=True):
        from .vae_plan import vae_spec_from_config
        super().__init__(vae_spec_from_config(module.config), module.state_dict, enable_cuda_graph)
        # eager_decode / eager_encode None: that entry is not compiled (it stays the module's own)
        self._module = module
        self._eager, self._eager_encode = eager_decode, eager_encode

    def _step(self, kind, plan_cls, input_name, x, extra=()):
        """Copy x into the static input `input_name` of the plan of `kind` for x's shape (and the plan
        arguments `extra`, which follow the batch), run it, return a copy of its output."""
        B, _, H, W = x.shape
        with self._lock, torch.cuda.device(x.device):
            weights = self._weights_for(x.dtype, x.device)
            gp = self._graphed((kind, B, *extra, H, W, x.dtype, x.device.index),
                               lambda: plan_cls(weights, B, *extra, H, W))
            getattr(gp.plan, input_name).copy_(x, non_blocking=True)
            gp.step()
            return gp.plan.out.clone()

    @staticmethod
    def _decoder_output(out, return_dict):
        if not return_dict:
            return (out,)
        try:
            from diffusers.models.autoencoders.vae import DecoderOutput as DO  # type: ignore
            return DO(sample=out)
        except Exception:  # noqa: BLE001
            return DecoderOutput(sample=out)

    def decode(self, z, return_dict=True, generator=None):
        from .vae_plan import VAEDecodePlan
        if z.dtype not in (torch.float16, torch.bfloat16):
            # e.g. SDXL's force_upcast fp32 VAE: the whole module stays on its own eager path
            self._warn_once("decode_dtype", "sfast (H100 build): VAE decode in %s is left on the module's eager "
                            "path (the native decoder computes in fp16 / bf16)", z.dtype)
            return self._eager(z, return_dict=return_dict, generator=generator)
        require_sm90(z.device)
        return self._decoder_output(self._step("decode", VAEDecodePlan, "z_in", z), return_dict)

    def decode_temporal(self, z, num_frames, return_dict=True):
        """`AutoencoderKLTemporalDecoder.decode(z, num_frames, return_dict=True)`: z holds z.shape[0] /
        num_frames videos of num_frames consecutive latent frames."""
        from .vae_plan import TemporalDecodePlan
        if z.dtype not in (torch.float16, torch.bfloat16):
            self._warn_once("decode_dtype", "sfast (H100 build): VAE decode in %s is left on the module's eager "
                            "path (the native decoder computes in fp16 / bf16)", z.dtype)
            return self._eager(z, num_frames=num_frames, return_dict=return_dict)
        num_frames = int(num_frames)
        if num_frames <= 0 or z.shape[0] % num_frames:
            raise ValueError(f"sfast (H100 build): temporal VAE decode of {z.shape[0]} latent frames with "
                             f"num_frames={num_frames}: the frames must be whole videos")
        require_sm90(z.device)
        out = self._step("decode_t", TemporalDecodePlan, "z_in", z, extra=(num_frames,))
        return self._decoder_output(out, return_dict)

    def encode(self, x, return_dict=True):
        from .vae_plan import VAEEncodePlan
        m = self._module
        if x.dtype not in (torch.float16, torch.bfloat16):
            self._warn_once("encode_dtype", "sfast (H100 build): VAE encode in %s is left on the module's eager "
                            "path (the native encoder computes in fp16 / bf16)", x.dtype)
            return self._eager_encode(x, return_dict=return_dict)
        tile = getattr(m, "tile_sample_min_size", None)
        if getattr(m, "use_tiling", False) and tile is not None and (x.shape[-1] > tile or x.shape[-2] > tile):
            # diffusers' tiled encode blends overlapping tiles: different numbers from a whole-image encode
            self._warn_once("encode_tiling", "sfast (H100 build): tiled VAE encode (use_tiling, image larger "
                            "than %s) is left on the module's eager path", tile)
            return self._eager_encode(x, return_dict=return_dict)
        require_sm90(x.device)
        moments = self._step("encode", VAEEncodePlan, "x_in", x)
        out_cls, dist_cls = _latent_dist_classes()
        dist = dist_cls(moments)
        if not return_dict:
            return (dist,)
        return out_cls(latent_dist=dist)


class AutoencoderTinyOutput(dict):
    """Stand-in for diffusers' AutoencoderTinyOutput (attribute, key and index access)."""

    def __init__(self, latents):
        super().__init__(latents=latents)
        self.latents = latents

    def __getitem__(self, k):
        return tuple(self.values())[k] if isinstance(k, int) else super().__getitem__(k)


def _tiny_output_class():
    try:
        from diffusers.models.autoencoders.autoencoder_tiny import AutoencoderTinyOutput as Out  # type: ignore
        return Out
    except Exception:  # noqa: BLE001
        return AutoencoderTinyOutput


def is_tiny_vae(m):
    """True for a diffusers AutoencoderTiny (TAESD), recognised by its config."""
    cfg = getattr(m, "config", None)
    return any(cfg_get(cfg, k) is not None for k in ("decoder_block_out_channels", "num_decoder_blocks"))


class CompiledTinyVAE(CompiledVAE):
    """`AutoencoderTiny.decode(x, generator=None, return_dict=True)` and `encode(x, return_dict=True)` on the
    native path, sharing one packed copy of the weights and one plan + CUDA-graph cache keyed by
    (kind, B, H, W, dtype, device).  fp32 calls and `use_tiling` (diffusers' blended tiles: different numbers
    from a whole-image pass) go to the module's own methods.  `use_slicing` runs the whole batch in one plan:
    the images are independent, so the result is the per-image one."""

    _what = "tiny VAE"

    def __init__(self, module, enable_cuda_graph=True):
        from .taesd_plan import taesd_spec_from_config
        _CompiledModule.__init__(self, taesd_spec_from_config(module.config), module.state_dict, enable_cuda_graph)
        self._module = module
        self._eager, self._eager_encode = module.decode, module.encode

    def _eager_reason(self, x):
        if x.dtype not in (torch.float16, torch.bfloat16):
            return f"{x.dtype} input: the native path computes in fp16 / bf16"
        if getattr(self._module, "use_tiling", False):
            return "use_tiling: diffusers' blended tiles"
        return None

    def _check(self, x, channels, what):
        if x.dim() != 4 or x.shape[1] != channels:
            raise ValueError(f"AutoencoderTiny.{what} of a {tuple(x.shape)} tensor: expected [B, {channels}, H, W]")
        require_sm90(x.device)

    def decode(self, x, generator=None, return_dict=True):
        from .taesd_plan import TAESDDecodePlan
        why = self._eager_reason(x)
        if why:
            self._warn_once("decode_eager", "sfast (H100 build): tiny VAE decode left on the module's eager path (%s)",
                            why)
            return self._eager(x, generator=generator, return_dict=return_dict)
        self._check(x, self.spec.latent_channels, "decode")
        return self._decoder_output(self._step("decode", TAESDDecodePlan, "z_in", x), return_dict)

    def encode(self, x, return_dict=True):
        from .taesd_plan import TAESDEncodePlan
        why = self._eager_reason(x)
        if why:
            self._warn_once("encode_eager", "sfast (H100 build): tiny VAE encode left on the module's eager path (%s)",
                            why)
            return self._eager_encode(x, return_dict=return_dict)
        self._check(x, self.spec.in_channels, "encode")
        out = self._step("encode", TAESDEncodePlan, "x_in", x)
        if not return_dict:
            return (out,)
        return _tiny_output_class()(latents=out)


def _compile_tiny_vae_module(m, enable_cuda_graph):
    """Install the native decode and encode of an AutoencoderTiny; None when its config is not supported."""
    from .taesd_plan import taesd_spec_from_config
    try:
        taesd_spec_from_config(m.config)
    except NotImplementedError as exc:
        logger.warning("sfast (H100 build): %s: %s", type(m).__name__, exc)
        return None
    compiled = CompiledTinyVAE(m, enable_cuda_graph)

    def decode(x, generator=None, return_dict=True):
        return compiled.decode(x, generator=generator, return_dict=return_dict)

    def encode(x, return_dict=True):
        return compiled.encode(x, return_dict=return_dict)
    _install(m, "decode", compiled, decode)
    return _install(m, "encode", compiled, encode)


def _has_temporal_decoder(m):
    """True when m's state dict holds every parameter of SVD's temporal decoder with its shape."""
    from .vae_plan import vae_spec_from_config, vae_temporal_decoder_param_shapes
    try:
        shapes = vae_temporal_decoder_param_shapes(vae_spec_from_config(m.config))
    except NotImplementedError:
        return False
    sd = m.state_dict()
    return all(k in sd and tuple(sd[k].shape) == tuple(s) for k, s in shapes.items())


def compile_vae_module(m, enable_cuda_graph=True):
    """Replace ``m.decode`` and ``m.encode`` of an AutoencoderKL (same module object).  `encode` is
    replaced only where the module has one and its encoder is supported.  A VAE whose decoder is not the
    2-D one gets the native `decode(z, num_frames, return_dict=True)` of SVD's temporal decoder when its
    state dict holds every parameter of that decoder; otherwise its decode is kept.  A tiny VAE
    (AutoencoderTiny, recognised by its config) gets the native `decode(x, generator=None, return_dict=True)`
    and `encode(x, return_dict=True)` when its config is supported; otherwise it takes the path below, which
    leaves both entries alone.  Either entry left alone is logged once."""
    from .vae_plan import vae_encoder_spec_from_config
    if is_tiny_vae(m) and hasattr(m, "encode"):
        tiny = _compile_tiny_vae_module(m, enable_cuda_graph)
        if tiny is not None:
            return tiny
    eager_decode, temporal = m.decode, False
    if temporal_decoder(m.state_dict()):
        temporal = _has_temporal_decoder(m)
        if not temporal:
            logger.warning("sfast (H100 build): %s has no post_quant_conv and is not SVD's temporal decoder: its "
                           "decode is left on the module's eager path", type(m).__name__)
            eager_decode = None
    eager_encode = getattr(m, "encode", None)
    if eager_encode is not None:
        try:
            vae_encoder_spec_from_config(m.config)
        except NotImplementedError as exc:
            logger.warning("sfast (H100 build): VAE encode is left on the module's eager path (%s)", exc)
            eager_encode = None
    if eager_decode is None and eager_encode is None:
        return m
    compiled = CompiledVAE(m, eager_decode, eager_encode, enable_cuda_graph)

    if temporal:
        def decode(z, num_frames, return_dict=True):
            return compiled.decode_temporal(z, num_frames, return_dict=return_dict)
        _install(m, "decode", compiled, decode)
    elif eager_decode is not None:
        def decode(z, return_dict=True, generator=None):
            return compiled.decode(z, return_dict=return_dict, generator=generator)
        _install(m, "decode", compiled, decode)
    if eager_encode is not None:
        def encode(x, return_dict=True):
            return compiled.encode(x, return_dict=return_dict)
        _install(m, "encode", compiled, encode)
    return m


class _CompiledClip(_CompiledModule):
    """A CLIP tower's forward on the native path: one plan + CUDA graph per input shape, outputs are fresh
    tensors.  Subclasses name the tower's first weight (its dtype is the one computed in), its static input
    and its projection output."""

    _weight0 = _input = _embeds = _proj_output = None

    def __init__(self, spec, config, state_dict_fn, eager_forward, with_projection, enable_cuda_graph=True,
                 lora_module=None):
        super().__init__(spec, state_dict_fn, enable_cuda_graph, lora_module=lora_module)
        self._eager = eager_forward
        self.with_projection = with_projection
        rd = cfg_get(config, "return_dict", None)
        self._return_dict_default = True if rd is None else bool(rd)

    def _route_eager(self, why, call):
        self._warn_once("eager", "sfast (H100 build): %s call left on the module's eager path (%s)", self._what, why)
        return self._eager(**call)

    def _run(self, x, key, make_plan, call, output_hidden_states, return_dict):
        if self._weights is None:
            dtype = lora.plain_state_dict(self._state_dict_fn())[self._weight0].dtype
            if dtype not in (torch.float16, torch.bfloat16):
                return self._route_eager(f"{dtype} weights: the native encoder computes in fp16 / bf16", call)
        else:
            dtype = self._weights.dtype
        require_sm90(x.device)
        with self._lock, torch.cuda.device(x.device):
            weights = self._weights_for(dtype, x.device)
            gp = self._graphed(key, lambda: make_plan(weights))
            plan = gp.plan
            getattr(plan, self._input).copy_(x, non_blocking=True)
            gp.step()
            last = plan.last_hidden_state.clone()
            pooled = plan.pooled.clone()
            embeds = getattr(plan, self._embeds).clone() if self.with_projection else None
            hidden = tuple(h.clone() for h in plan.hidden_states()) if output_hidden_states else None
        if return_dict is None:
            return_dict = self._return_dict_default
        if self.with_projection:
            if not return_dict:
                return tuple(v for v in (embeds, last, hidden) if v is not None)
            return _clip_output(self._proj_output, **{self._embeds: embeds}, last_hidden_state=last,
                                hidden_states=hidden)
        if not return_dict:
            return tuple(v for v in (last, pooled, hidden) if v is not None)
        return _clip_output("BaseModelOutputWithPooling", last_hidden_state=last, pooler_output=pooled,
                            hidden_states=hidden)


class CompiledTextEncoder(_CompiledClip):
    """transformers ``CLIPTextModel`` / ``CLIPTextModelWithProjection`` forward on the native path: the
    text encoders the reference traces and graphs
    (/root/reference/src/sfast/compilers/diffusion_pipeline_compiler.py:93-112).  One plan + CUDA graph
    per (batch, sequence length)."""

    _what = "text encoder"
    _weight0, _input = "text_model.embeddings.token_embedding.weight", "ids_in"
    _embeds, _proj_output = "text_embeds", "CLIPTextModelOutput"

    def __init__(self, config, state_dict_fn, eager_forward, with_projection, enable_cuda_graph=True, module=None):
        """`module`: the encoder itself, whose PEFT LoRA layers are merged into the packed weights (their scale
        is read on every call, so diffusers' scale_lora_layers around the call is honoured)."""
        from .clip_plan import clip_text_spec_from_config
        super().__init__(clip_text_spec_from_config(config, with_projection), config, state_dict_fn, eager_forward,
                         with_projection, enable_cuda_graph, lora_module=module)

    def __call__(self, input_ids=None, attention_mask=None, position_ids=None, output_attentions=None,
                 output_hidden_states=None, return_dict=None, **kwargs):
        from .clip_plan import ClipTextPlan
        call = dict(input_ids=input_ids, attention_mask=attention_mask, position_ids=position_ids,
                    output_attentions=output_attentions, output_hidden_states=output_hidden_states,
                    return_dict=return_dict, **kwargs)
        call = {k: v for k, v in call.items() if v is not None}
        if input_ids is None:
            raise ValueError("You have to specify input_ids")
        if attention_mask is not None or position_ids is not None or output_attentions or kwargs:
            return self._route_eager("attention_mask / position_ids / output_attentions / extra kwargs", call)
        ids = input_ids.view(-1, input_ids.shape[-1])
        B, S = ids.shape
        return self._run(ids, (B, S, ids.device.index), lambda w: ClipTextPlan(w, B, S), call,
                         output_hidden_states, return_dict)


class CompiledVisionEncoder(_CompiledClip):
    """transformers ``CLIPVisionModel`` / ``CLIPVisionModelWithProjection`` forward on the native path (the
    SVD pipeline's image_encoder, reference :100-103).  One plan + CUDA graph per batch size."""

    _what = "image encoder"
    _weight0, _input = "vision_model.embeddings.patch_embedding.weight", "pixels_in"
    _embeds, _proj_output = "image_embeds", "CLIPVisionModelOutput"

    def __init__(self, config, state_dict_fn, eager_forward, with_projection, enable_cuda_graph=True):
        from .clip_plan import clip_vision_spec_from_config
        super().__init__(clip_vision_spec_from_config(config, with_projection), config, state_dict_fn,
                         eager_forward, with_projection, enable_cuda_graph)

    def __call__(self, pixel_values=None, interpolate_pos_encoding=False, output_attentions=None,
                 output_hidden_states=None, return_dict=None, **kwargs):
        from .clip_plan import ClipVisionPlan
        call = dict(pixel_values=pixel_values, interpolate_pos_encoding=interpolate_pos_encoding,
                    output_attentions=output_attentions, output_hidden_states=output_hidden_states,
                    return_dict=return_dict, **kwargs)
        call = {k: v for k, v in call.items() if v is not None}
        if pixel_values is None:
            raise ValueError("You have to specify pixel_values")
        spec = self.spec
        if interpolate_pos_encoding or output_attentions or kwargs:
            return self._route_eager("interpolate_pos_encoding / output_attentions / extra kwargs", call)
        if tuple(pixel_values.shape[1:]) != (spec.channels, spec.image_size, spec.image_size):
            raise ValueError(f"Input image size {tuple(pixel_values.shape[2:])} doesn't match model "
                             f"({spec.image_size}*{spec.image_size}).")
        # (the copy into the static input casts to the module's dtype, as the module does)
        B = pixel_values.shape[0]
        return self._run(pixel_values, (B, pixel_values.device.index), lambda w: ClipVisionPlan(w, B), call,
                         output_hidden_states, return_dict)


def compile_image_encoder_module(m, enable_cuda_graph=True):
    """Replace ``m.forward`` of a CLIPVisionModel / CLIPVisionModelWithProjection (same module object)."""
    compiled = CompiledVisionEncoder(m.config, m.state_dict, m.forward, hasattr(m, "visual_projection"),
                                     enable_cuda_graph)

    def forward(*args, **kwargs):
        if args:
            kwargs = dict(zip(("pixel_values",), args), **kwargs)
        return compiled(**kwargs)
    return _install(m, "forward", compiled, forward)


class _PlainOutput(dict):
    """Stand-in for transformers' ModelOutput when transformers is not importable: attribute, key and
    integer access over the non-None fields, like the real class."""

    def __init__(self, **kw):
        super().__init__({k: v for k, v in kw.items() if v is not None})
        self.__dict__.update(kw)

    def __getitem__(self, k):
        return tuple(self.values())[k] if isinstance(k, (int, slice)) else super().__getitem__(k)


def _clip_output(kind, **fields):
    try:
        if kind == "CLIPTextModelOutput":
            from transformers.models.clip.modeling_clip import CLIPTextModelOutput as cls
        elif kind == "CLIPVisionModelOutput":
            from transformers.models.clip.modeling_clip import CLIPVisionModelOutput as cls
        else:
            from transformers.modeling_outputs import BaseModelOutputWithPooling as cls
        return cls(**fields)
    except Exception:  # noqa: BLE001
        return _PlainOutput(**fields)


def compile_text_encoder_module(m, enable_cuda_graph=True):
    """Replace ``m.forward`` of a CLIPTextModel / CLIPTextModelWithProjection (same module object)."""
    compiled = CompiledTextEncoder(m.config, m.state_dict, m.forward, hasattr(m, "text_projection"),
                                   enable_cuda_graph, module=m)

    def forward(*args, **kwargs):
        if args:
            kwargs = dict(zip(("input_ids", "attention_mask", "position_ids"), args), **kwargs)
        return compiled(**kwargs)
    return _install(m, "forward", compiled, forward)


@functools.lru_cache(maxsize=None)
def _controlnet_output_class():
    """diffusers' ControlNetOutput where it imports, else a stand-in with attribute, key and index access."""
    for mod in ("diffusers.models.controlnets.controlnet", "diffusers.models.controlnet"):
        try:
            return __import__(mod, fromlist=["ControlNetOutput"]).ControlNetOutput
        except Exception:  # noqa: BLE001
            pass
    return ControlNetOutput


class ControlNetOutput(dict):
    """Stand-in for diffusers' ControlNetOutput (attribute, key and index access)."""

    def __init__(self, down_block_res_samples, mid_block_res_sample):
        super().__init__(down_block_res_samples=down_block_res_samples, mid_block_res_sample=mid_block_res_sample)
        self.down_block_res_samples = down_block_res_samples
        self.mid_block_res_sample = mid_block_res_sample

    def __getitem__(self, k):
        return tuple(self.values())[k] if isinstance(k, int) else super().__getitem__(k)

    def to_tuple(self):
        return tuple(self.values())


class CompiledControlNet(_CompiledModule):
    """Callable with the signature of diffusers ``ControlNetModel.forward``.  One plan + CUDA graph per
    (batch, latent height, latent width, dtype, text length, device); conditioning_scale and guess mode are
    inputs of the graph, not part of the key."""

    _what = "ControlNet"

    def __init__(self, config, state_dict_fn, enable_cuda_graph=True, preserve_parameters=True):
        from .unet_spec import controlnet_spec_from_config
        super().__init__(controlnet_spec_from_config(config), state_dict_fn, enable_cuda_graph, preserve_parameters)

    def __call__(self, sample, timestep, encoder_hidden_states, controlnet_cond, conditioning_scale=1.0,
                 class_labels=None, timestep_cond=None, attention_mask=None, added_cond_kwargs=None,
                 cross_attention_kwargs=None, guess_mode=False, return_dict=True):
        from .controlnet_plan import ControlNetPlan, residual_scales
        given = dict(class_labels=class_labels, timestep_cond=timestep_cond, attention_mask=attention_mask)
        for k, v in given.items():
            if v is not None:
                raise NotImplementedError(f"sfast (H100 build): ControlNet argument `{k}` is not supported")
        if cross_attention_kwargs:
            scale = cross_attention_kwargs.get("scale", 1.0)
            if set(cross_attention_kwargs) - {"scale"} or scale != 1.0:
                raise NotImplementedError("sfast (H100 build): cross_attention_kwargs (LoRA scale) "
                                          "is not supported; fuse the LoRA weights into the parameters")
        require_sm90(sample.device)
        dtype = sample.dtype
        if dtype not in (torch.float16, torch.bfloat16):
            raise NotImplementedError(f"sfast (H100 build): ControlNet dtype {dtype}; use fp16 or bf16")
        spec = self.spec
        B, _, H, W = sample.shape
        f = 1 << (len(spec.cond_embed_channels) - 1)
        if tuple(controlnet_cond.shape) != (B, spec.cond_channels, f * H, f * W):
            raise ValueError(f"controlnet_cond {tuple(controlnet_cond.shape)} must be {f}x the latent size: "
                             f"expected {(B, spec.cond_channels, f * H, f * W)}")
        ctx_len = encoder_hidden_states.shape[1]
        with self._lock, torch.cuda.device(sample.device):
            weights = self._weights_for(dtype, sample.device)
            gp = self._graphed((B, H, W, dtype, ctx_len, sample.device.index),
                               lambda: ControlNetPlan(weights, B, H, W, ctx_len))
            plan = gp.plan
            plan.sample_in.copy_(sample, non_blocking=True)
            plan.ehs_in.copy_(encoder_hidden_states, non_blocking=True)
            plan.cond_in.copy_(controlnet_cond, non_blocking=True)
            plan.scale_in.copy_(residual_scales(len(plan.down_out), conditioning_scale, guess_mode))
            t = timestep if torch.is_tensor(timestep) else torch.tensor(float(timestep))
            t = t.reshape(-1).to(device=sample.device, dtype=torch.float32, non_blocking=True)
            plan.t_in.copy_(t.expand(B) if t.numel() == 1 else t)
            if spec.addition_embed_type == "text_time":
                if not added_cond_kwargs or "text_embeds" not in added_cond_kwargs:
                    raise ValueError("added_cond_kwargs with text_embeds / time_ids is required")
                te = added_cond_kwargs["text_embeds"]
                plan.add_in[:, :te.shape[1]].copy_(te)
                plan.time_ids_in.copy_(added_cond_kwargs["time_ids"].reshape(-1).float())
            gp.step()
            down = tuple(o.clone() for o in plan.down_out)
            mid = plan.mid_out.clone()
        if not return_dict:
            return down, mid
        return _controlnet_output_class()(down_block_res_samples=down, mid_block_res_sample=mid)


def compile_controlnet_module(m, enable_cuda_graph=True, preserve_parameters=True):
    """Replace ``m.forward`` of a diffusers ControlNetModel (same module object)."""
    compiled = CompiledControlNet(m.config, m.state_dict, enable_cuda_graph, preserve_parameters)

    def forward(*args, **kwargs):
        return compiled(*args, **kwargs)
    return _install(m, "forward", compiled, forward)


class CompiledT2IAdapter(_CompiledModule):
    """Callable with the signature of diffusers ``T2IAdapter.forward(x)``: the list of NCHW features, fresh
    tensors.  One plan + CUDA graph per (batch, image height, width, dtype, device)."""

    _what = "T2I-Adapter"

    def __init__(self, config, state_dict_fn, enable_cuda_graph=True, preserve_parameters=True):
        from .t2i_adapter_plan import t2i_adapter_spec_from_config
        super().__init__(t2i_adapter_spec_from_config(config), state_dict_fn, enable_cuda_graph, preserve_parameters)

    def __call__(self, x):
        from .t2i_adapter_plan import AdapterPlan
        spec = self.spec
        if x.dim() != 4 or x.shape[1] != spec.in_channels:
            raise ValueError(f"T2IAdapter input of shape {tuple(x.shape)}: expected [B, {spec.in_channels}, H, W]")
        if x.dtype not in (torch.float16, torch.bfloat16):
            raise NotImplementedError(f"sfast (H100 build): T2I-Adapter dtype {x.dtype}; use fp16 or bf16")
        B, _, H, W = x.shape
        f = spec.total_downscale_factor
        if H % f or W % f:
            raise NotImplementedError(f"sfast (H100 build): T2I-Adapter image size {H}x{W} must be a multiple of its "
                                      f"total_downscale_factor {f}")
        require_sm90(x.device)
        with self._lock, torch.cuda.device(x.device):
            weights = self._weights_for(x.dtype, x.device)
            gp = self._graphed((B, H, W, x.dtype, x.device.index), lambda: AdapterPlan(weights, B, H, W))
            gp.plan.x_in.copy_(x, non_blocking=True)
            gp.step()
            return [o.clone() for o in gp.plan.features_out]


def compile_adapter_module(m, enable_cuda_graph=True, preserve_parameters=True):
    """Replace ``m.forward`` of a diffusers T2IAdapter (same module object: ``downscale_factor`` and
    ``total_downscale_factor`` keep working)."""
    compiled = CompiledT2IAdapter(m.config, m.state_dict, enable_cuda_graph, preserve_parameters)

    def forward(x):
        return compiled(x)
    return _install(m, "forward", compiled, forward)


def compile_unet_module(m, enable_cuda_graph=True, preserve_parameters=True):
    """Replace ``m.forward`` (same module object, as the reference does at
    /root/reference/src/sfast/compilers/diffusion_pipeline_compiler.py:146-149)."""
    compiled = CompiledUNet(m.config, m.state_dict, enable_cuda_graph, preserve_parameters, module=m)

    def forward(*args, **kwargs):
        return compiled(*args, **kwargs)
    return _install(m, "forward", compiled, forward)
