"""Schedule builder: turns (UNet config, state dict, batch, height, width) into a flat, static
list of C-ABI kernel launches over pre-allocated buffers -- the replacement for the reference's
TorchScript trace + graph passes (/root/reference/src/sfast/jit/trace_helper.py:33-72,
/root/reference/src/sfast/jit/passes/__init__.py) on the UNet hot path.

Design points (see DESIGN.md):
  * NHWC / token-major activations end to end: [B, H, W, C] is also [B*H*W, C], so the
    resnet -> transformer hand-off needs no layout kernels.
  * zero-copy skip concatenation: every skip tensor is produced directly into the channel slice
    of the buffer its up-block consumer reads (`torch.cat` never runs).
  * every residual / bias / time-embedding add / GEGLU / head split lives in a GEMM epilogue.
  * weights are repacked once (conv OIHW -> K-major [cout, 9*cin], fused QKV, tile-interleaved
    GEGLU, one concatenated matrix for all 22 time-embedding projections, LayerNorm folded into
    the consuming projection, upsampler convs as four pre-summed 2x2 phases).
  * work that is off the critical path runs on a forked stream = parallel branches of the captured
    graph: time-embedding chain, cross-attention K/V projections, resnet shortcut GEMMs.
  * a split-K conv followed by a GroupNorm leaves its reduction to that GroupNorm kernel.
"""
import ctypes as C
import math
import os

import torch

from . import _lib, ops
from .ops import Act, EPI_GEGLU, EPI_QKV, Op, _ptr
from .unet_spec import RESAMPLER_HEAD_DIM, UNetSpec, spec_from_config


def _round_up(a, b):
    return (a + b - 1) // b * b


def intrablock_shapes(spec, batch, height, width):
    """NCHW shapes of the T2I-Adapter residuals (``down_intrablock_additional_residuals``) a 2-D UNet adds, in
    the order it takes them: one per down block, then one for the mid-block output.  A down block with
    cross-attention adds its residual to the output of its last (resnet, transformer) pair, in front of its
    downsampler; a plain down block to its own output, after the downsampler."""
    out, h, w = [], height, width
    for blk in spec.down:
        cross = any(t is not None for t in blk.attentions)
        if cross:
            out.append((batch, blk.cout, h, w))
        if blk.sampler:
            h, w = h // 2, w // 2
        if not cross:
            out.append((batch, blk.cout, h, w))
    out.append((batch, spec.mid.cout, h, w))
    return out


class PackedWeights:
    """Device-resident, kernel-ready copy of a UNet state dict (shape independent).

    The packed tensors are COPIES of the module's parameters.  The reference keeps pointer
    aliasing with the live parameters (`preserve_parameters=True`,
    /root/reference/src/sfast/compilers/diffusion_pipeline_compiler.py:35-39,70) so that an
    in-place update (LoRA switch, /root/reference/README.md:228-265) is seen by the next call;
    here `refresh()` re-packs every tensor INTO THE SAME device storage, so launch plans, TMA maps
    and captured CUDA graphs stay valid, and the runtime calls it when the parameters' version
    counters move.
    """

    def __init__(self, spec: UNetSpec, state_dict, dtype, device, dry=False):
        self.spec, self.dtype, self.device, self.dry = spec, dtype, torch.device(device), dry
        self.sd = state_dict
        self._cache = {}
        self._builders = {}
        self._deps = {}        # builder key -> the state-dict names its build read
        self._reading = None
        # all per-resnet time projections as ONE [sum(cout), temb_dim] matrix
        self.tproj_off = {}
        off = 0
        for r in spec.all_resnets():
            self.tproj_off[r.prefix] = off
            off += r.cout
        self.tproj_total = off
        if off:  # (the VAE decoder has no time embedding)
            self.tproj_w, self.tproj_b = self._get(("tproj",), self._build_tproj)

    def _build_tproj(self):
        ws = [self._raw(r.prefix + ".time_emb_proj.weight") for r in self.spec.all_resnets()]
        bs = [self._raw(r.prefix + ".time_emb_proj.bias") for r in self.spec.all_resnets()]
        return (torch.cat(ws, 0).to(device=self.device, dtype=self.dtype).contiguous(),
                torch.cat(bs, 0).to(device=self.device, dtype=torch.float32).contiguous())

    def _raw(self, name):
        """The state-dict tensor `name`, read once per build (an adapted weight is merged on each read)."""
        if self._reading is not None and name in self._reading:
            return self._reading[name]
        if name not in self.sd:
            raise KeyError(f"UNet state dict has no parameter {name!r}")
        t = self.sd[name].detach()
        if self._reading is not None:
            self._reading[name] = t
        return t

    def _build(self, key, builder):
        outer, self._reading = self._reading, {}
        try:
            out = builder()
            self._deps[key] = frozenset(self._reading)
        finally:
            inner, self._reading = self._reading, outer
            if outer is not None:
                outer.update(inner)
        return out

    def _get(self, key, builder):
        if key not in self._cache:
            self._cache[key] = self._build(key, builder)
            self._builders[key] = builder
        return self._cache[key]

    def refresh(self, state_dict, names=None):
        """Re-pack from `state_dict` into the existing device tensors (addresses unchanged).  `names`: re-run only
        the builders that read one of these state-dict names (an adapter change); returns how many ran."""
        self.sd = state_dict

        def copy_into(old, new):
            if isinstance(old, ops.Mat):
                old.data.copy_(new.data)
            elif torch.is_tensor(old):
                old.copy_(new)
            elif isinstance(old, (tuple, list)):
                for o, n in zip(old, new):
                    copy_into(o, n)
            elif old != new:
                raise RuntimeError("UNet architecture changed under a compiled module")

        ran = 0
        for key, builder in self._builders.items():
            if names is None or not self._deps[key].isdisjoint(names):
                copy_into(self._cache[key], self._build(key, builder))
                ran += 1
        return ran

    def f32(self, name):
        return self._get(("f32", name), lambda: self._raw(name).to(
            device=self.device, dtype=torch.float32, memory_format=torch.contiguous_format, copy=True))

    def _mat(self, w):
        return ops.Mat(w, self.dry)

    def matrix(self, name):
        """[n, k] weight (linear or 1x1 conv) as a tiled GEMM operand."""
        def build():
            w = self._raw(name)
            return self._mat(w.reshape(w.shape[0], -1).to(device=self.device, dtype=self.dtype).contiguous())
        return self._get(("mat", name), build)

    def conv3x3(self, name):
        return self._get(("c3", name), lambda: self._mat(
            ops.pack_conv3x3(self._raw(name).to(self.device), self.dtype)))

    def upconv(self, name):
        """Upsampler conv as the 4-phase 2x2 formulation (ops.pack_upconv): (Mat, cout)."""
        def build():
            w = self._raw(name)
            return (self._mat(ops.pack_upconv(w.to(self.device), self.dtype)), w.shape[0])
        return self._get(("up", name), build)

    def conv3x3_plain(self, name):
        return self._get(("c3p", name), lambda: ops.pack_conv3x3(self._raw(name).to(self.device),
                                                                self.dtype))

    def conv3x3_pointwise(self, conv, pointwise):
        """3x3 conv `conv` followed by the 1x1 conv `pointwise` (module prefixes) as one 3x3 conv
        (ops.fold_pointwise_into_conv): (weight packed like conv3x3_plain, fp32 bias)."""
        def build():
            w, b = ops.fold_pointwise_into_conv(*(self._raw(f"{p}.{t}").to(self.device)
                                                  for p in (conv, pointwise) for t in ("weight", "bias")))
            return ops.pack_conv3x3(w, self.dtype), b.float().contiguous()
        return self._get(("c3pw", conv, pointwise), build)

    def conv3x3_affine(self, conv, scale, shift):
        """3x3 conv `conv` (module prefix) followed by y * scale + shift, as one conv: (weight packed like
        conv3x3_plain of scale * W, fp32 scale * b + shift), formed in fp32 before the weight is rounded."""
        def build():
            w = self._raw(conv + ".weight").to(self.device).float() * scale
            b = self._raw(conv + ".bias").to(self.device).float() * scale + shift
            return ops.pack_conv3x3(w, self.dtype), b.contiguous()
        return self._get(("c3aff", conv, scale, shift), build)

    def _padded_mat(self, w, kpad):
        """[n, k] weight zero-padded along K to kpad columns, as a GEMM operand."""
        if w.device.type == "meta":
            wp = torch.empty(w.shape[0], kpad, dtype=self.dtype, device="meta")
        else:
            wp = torch.zeros(w.shape[0], kpad, dtype=self.dtype, device=w.device)
            wp[:, :w.shape[1]] = w.to(self.dtype)
        return self._mat(wp)

    def conv_in_matrix(self, name):
        """First conv as a GEMM operand: [cout, (kh, kw, cin)] zero-padded along K to the next multiple of 64
        (64 for cin <= 7, 128 for 9 <= cin <= 14)."""
        def build():
            w = ops.pack_conv3x3(self._raw(name).to(self.device), self.dtype)
            return self._padded_mat(w, _round_up(w.shape[1], 64))
        return self._get(("cin_mat", name), build)

    def patch_matrix(self, name, kpad):
        """Patch-embedding conv [cout, cin, p, p] as a GEMM operand over patchified rows: [cout, (cin, p, p)]
        zero-padded along K to kpad."""
        def build():
            w = self._raw(name).to(self.device)
            return self._padded_mat(w.reshape(w.shape[0], -1), kpad)
        return self._get(("patch_mat", name, kpad), build)

    def class_row(self, class_name, pos_name):
        """[1, c] class embedding plus the first position embedding: the class token's input row."""
        def build():
            v = self._raw(class_name).to(self.device).float() + self._raw(pos_name).to(self.device)[0].float()
            return v.to(self.dtype).reshape(1, -1).contiguous()
        return self._get(("cls_row", class_name, pos_name), build)

    def rows_from_1(self, name):
        """Rows 1.. of a [n, c] table (the patch tokens' position embeddings)."""
        return self._get(("rows1", name), lambda: self._raw(name).to(
            device=self.device, dtype=self.dtype)[1:].contiguous())

    def f32_cat(self, names):
        return self._get(("f32cat",) + tuple(names), lambda: torch.cat(
            [self._raw(n).to(device=self.device, dtype=torch.float32) for n in names]).contiguous())

    def conv_in_weight(self, name):
        return self._get(("cin", name), lambda: ops.pack_conv_in(self._raw(name).to(self.device),
                                                                self.dtype))

    def cat_matrix(self, names):
        def build():
            w = torch.cat([self._raw(n) for n in names], 0)
            return self._mat(w.to(device=self.device, dtype=self.dtype).contiguous())
        return self._get(("cat",) + tuple(names), build)

    def ln_matrix(self, names, ln_prefix, bias_names=None, row_scale=None):
        """cat(names) with LayerNorm `ln_prefix` folded in: (Mat, bias', colsum).  `bias_names`: the
        linear layers' own biases (CLIP projections have them, the UNet's attention projections do
        not); `row_scale`: per-matrix constants folded into weight and bias (CLIP scales q by
        head_dim ** -0.5 before the scores)."""
        def build():
            ws = [self._raw(n).to(self.device).float() for n in names]
            bs = None if bias_names is None else [self._raw(n).to(self.device).float() for n in bias_names]
            if row_scale is not None:
                ws = [w * s for w, s in zip(ws, row_scale)]
                if bs is not None:
                    bs = [b * s for b, s in zip(bs, row_scale)]
            wp, bias, colsum = ops.fold_layer_norm(
                torch.cat(ws, 0), None if bs is None else torch.cat(bs, 0),
                self._raw(ln_prefix + ".weight").to(self.device),
                self._raw(ln_prefix + ".bias").to(self.device), self.dtype)
            return (self._mat(wp.contiguous()), bias, colsum)
        return self._get(("lnmat", ln_prefix, tuple(bias_names or ()), tuple(row_scale or ())) + tuple(names), build)

    def ln_geglu(self, prefix, ln_prefix):
        def build():
            wp, bias, colsum = ops.fold_layer_norm(
                self._raw(prefix + ".weight").to(self.device), self._raw(prefix + ".bias").to(self.device),
                self._raw(ln_prefix + ".weight").to(self.device),
                self._raw(ln_prefix + ".bias").to(self.device), self.dtype)
            wt, bp, inner, cs = ops.pack_geglu(wp, bias, self.dtype, extra=colsum)
            return (self._mat(wt), bp, inner, cs)
        return self._get(("lngeglu", prefix, ln_prefix), build)

    def frame_bias_table(self, names, pe_name, max_seq):
        """fp32 pe[0, :max_seq] cat(names)^T -> [max_seq, sum of the rows of names]: a position embedding added
        after a LayerNorm's affine and in front of the projections `names` (AnimateDiff's motion attentions), as
        the per-frame bias sfb_frame_attention adds to q | k | v.  The LayerNorm stays folded into the QKV GEMM,
        which cannot also take a row bias: (LN(x) + pe_f) W^T = LN(x) W^T + pe_f W^T.  Built from the same
        state-dict names as the QKV matrix, so a parameter update or a LoRA merge re-packs both."""
        def build():
            w = torch.cat([self._raw(n).to(self.device).float() for n in names], 0)
            pe = self._raw(pe_name).to(self.device).float()[0, :max_seq]
            return (pe @ w.t()).contiguous()
        return self._get(("frame_bias", pe_name, max_seq) + tuple(names), build)

    def geglu(self, prefix):
        def build():
            wp, bp, inner = ops.pack_geglu(self._raw(prefix + ".weight").to(self.device),
                                           self._raw(prefix + ".bias").to(self.device), self.dtype)
            return (self._mat(wp), bp, inner)
        return self._get(("geglu", prefix), build)

    def _blend_scaled(self, v, mix):
        """v times the temporal share of an AlphaBlender: `mix` = (mix_factor name, switched).  The blend of
        the spatial x_s and the temporal x_s + t is  x_s + s * t,  with s = 1 - sigmoid(mix_factor) (the SVD
        UNet) or, with switch_spatial_to_temporal_mix (SVD's temporal VAE decoder), s = sigmoid(mix_factor)."""
        if mix is None:
            return v
        name, switched = mix
        alpha = torch.sigmoid(self._raw(name).to(self.device).float())
        return v * (alpha if switched else 1.0 - alpha)

    def conv3x1_t(self, name, mix=None):
        """Temporal conv weight [cout, cin, 3, 1, 1] -> K-major [cout, (kt, cin)] as a GEMM operand;
        `mix`: (AlphaBlender mix_factor name, switched) -- the weight is pre-scaled by the blend's temporal
        share (_blend_scaled), so that the blend is a plain residual epilogue."""
        def build():
            w = self._raw(name).to(self.device).float()
            w = w[:, :, :, 0, 0].permute(0, 2, 1).reshape(w.shape[0], -1)
            return self._mat(self._blend_scaled(w, mix).to(self.dtype).contiguous())
        return self._get(("c3t", name, mix), build)

    def f32_scaled(self, name, mix):
        """fp32 vector scaled like conv3x1_t(.., mix) (the temporal conv's bias)."""
        return self._get(("f32s", name, mix), lambda: self._blend_scaled(
            self._raw(name).to(device=self.device, dtype=torch.float32), mix).contiguous())

    def time_conv_out(self, name):
        """Conv3d (3,1,1) weight [cout, cin, 3, 1, 1] as sfb_conv_out_temporal takes it: 16-bit [cout, 3, cin]."""
        return self._get(("c3tout", name), lambda: self._raw(name).to(self.device)[:, :, :, 0, 0].permute(
            0, 2, 1).to(self.dtype).contiguous())

    def scaled_linear(self, prefix, scale):
        """(Mat of scale * W, fp32 scale * b): a linear layer with a constant folded in."""
        def build():
            w = (self._raw(prefix + ".weight").to(self.device).float() * scale).to(self.dtype).contiguous()
            b = (self._raw(prefix + ".bias").to(self.device).float() * scale).contiguous()
            return (self._mat(w), b)
        return self._get(("slin", prefix, scale), build)

    def _padded_conv(self, name, cin_pad, cout_pad, flip_cin=False):
        """[cout, cin, 3, 3] weight zero-padded to [cout_pad, cin_pad, 3, 3] (`flip_cin`: input channels in
        reverse order -- a BGR conditioning image read as RGB)."""
        w = self._raw(name).to(self.device)
        if flip_cin:
            w = w.flip(1)
        return torch.nn.functional.pad(w, (0, 0, 0, 0, 0, cin_pad - w.shape[1], 0, cout_pad - w.shape[0]))

    def conv3x3_small(self, name, cout_pad, flip_cin=False):
        """3x3 conv weight for sfb_conv3x3_small: 16-bit [cout_pad, 3, 3, cin16], zero rows past cout and
        zero input channels past cin."""
        def build():
            w = self._raw(name)
            return ops.pack_conv3x3(self._padded_conv(name, _round_up(w.shape[1], 16), cout_pad, flip_cin),
                                    self.dtype)
        return self._get(("c3small", name, cout_pad, flip_cin), build)

    def conv3x3_padded(self, name, cin_pad, cout_pad):
        """3x3 conv weight zero-padded to cin_pad inputs and cout_pad outputs, as a GEMM operand."""
        return self._get(("c3pad", name, cin_pad, cout_pad), lambda: self._mat(
            ops.pack_conv3x3(self._padded_conv(name, cin_pad, cout_pad), self.dtype)))

    def f32_padded(self, name, n):
        """fp32 vector zero-padded to n entries."""
        return self._get(("f32pad", name, n), lambda: torch.nn.functional.pad(
            self._raw(name).to(device=self.device, dtype=torch.float32), (0, n - self._raw(name).shape[0])))

    def small(self, name):
        # (copy=True: a packed tensor never aliases the parameter; refresh() writes into it)
        return self._get(("small", name), lambda: self._raw(name).to(
            device=self.device, dtype=self.dtype, memory_format=torch.contiguous_format, copy=True))


class Plan:
    """One static launch schedule over pre-allocated buffers, for a fixed (batch, height, width): the state and
    the emitters every model's schedule shares.  `n_gn`: GroupNorms the schedule runs (their statistics arenas
    are allocated only when > 0); `ln_floats`: fp32 row statistics of its folded LayerNorms.  Both arenas
    are zeroed at the start of every step; `_finish()` closes the schedule."""

    def __init__(self, weights: PackedWeights, batch, height, width, *, n_gn=0, ln_floats=0):
        self.w = weights
        self.spec = weights.spec
        self.dt, self.dev, self.dry = weights.dtype, weights.device, weights.dry
        self.lib = None if self.dry else _lib.lib()
        self.B, self.H, self.W = batch, height, width
        self.ops = []
        # Ops that depend only on the step's inputs (e.g. the UNet's cross-attention K/V projections of the
        # text embedding): issued on a forked stream so they run concurrently with the start of the main
        # chain (a parallel branch of the captured CUDA graph).
        self.side_ops = []
        self._side_stream = None
        self._pending = None      # conv GEMM whose split-K finish the next GroupNorm may absorb
        self._gn_ws_patches = []  # GnParams that read the split-K workspace (pointer known late)
        self._joined = False
        self._bufs = {}
        self._gn_count = 0
        self._n_gn = n_gn
        lib = self.lib_or_dry()
        if n_gn:
            # per-GroupNorm statistics workspace (one [groups][2] slot per CTA of the statistics pass, summed in
            # a fixed order by the apply pass: no initialisation needed) and the fused kernel's grid-barrier
            # counters (zeroed once per step)
            self.gn_stats = self._alloc((n_gn, ops.gn_ws_floats(batch, self.spec.groups)), torch.float32)
            self.gn_sync = self._alloc((n_gn, 4), torch.int32)
            # GroupNorm folded into the conv: per-image tickets of the statistics kernel (self-resetting)
            self.gn_tickets = self._alloc((n_gn, max(batch, 4)), torch.int32)
            self._emit(Op("gn_sync.zero", lib.sfb_memset, (_ptr(self.gn_sync), 0, self.gn_sync.numel() * 4),
                          (self.gn_sync,)))
        # folded-LayerNorm row statistics: [rows, slots, 2] fp32 per LayerNorm (ln_slot)
        self._ln_used = 0
        self.ln_arena = self._alloc((max(ln_floats, 2),), torch.float32)
        if ln_floats:
            self._emit(Op("ln_stats.zero", lib.sfb_memset, (_ptr(self.ln_arena), 0, self.ln_arena.numel() * 4),
                          (self.ln_arena,)))
        # split-K workspace: one shared fp32 buffer, sized by _finish() once all ops are known
        self._ws_token = _WsToken()

    def _finish(self):
        """Close the schedule: a deferred split-K finish nothing consumed is done by its own GEMM; check the
        GroupNorm and LayerNorm budgets; allocate the split-K workspace and patch the ops."""
        if self._pending is not None:
            self._pending["p"].defer_finish = 0
            self._pending = None
        assert self._gn_count == self._n_gn, (self._gn_count, self._n_gn)
        assert self._ln_used <= self.ln_arena.numel(), (self._ln_used, self.ln_arena.numel())
        self._ws_token.finalize(self)

    # ------------------------------------------------------------------ buffers
    def _alloc(self, shape, dtype):
        if self.dry:
            return torch.empty(shape, dtype=dtype, device="meta")
        return torch.zeros(shape, dtype=dtype, device=self.dev)

    def buf(self, name, shape, dtype=None):
        key = (name, tuple(shape), dtype or self.dt)
        if key not in self._bufs:
            self._bufs[key] = self._alloc(shape, dtype or self.dt)
        return self._bufs[key]

    def act(self, name, n, h, w, c):
        return Act(self.buf(name, (n, h, w, c)), n, h, w, c)

    def ln_slot(self, rows, dim):
        """[rows, slots, 2] fp32 (sum, sum of squares) statistics of one folded LayerNorm over `dim`
        columns: every producer writes its own slots, the consumer adds them in order."""
        slots = ops.rowstats_slots(dim)
        off = self._ln_used
        self._ln_used += rows * slots * 2
        return ops.RowStats(self.ln_arena[off:off + rows * slots * 2], slots)

    # ------------------------------------------------------------------ op emitters
    def _emit(self, op):
        # a split-K conv whose finish was tentatively left to the next GroupNorm: anything else
        # being emitted first means that GroupNorm is not the next consumer -> finish it normally
        if self._pending is not None:
            self._pending["p"].defer_finish = 0
            self._pending = None
        if isinstance(op, (list, tuple)):
            self.ops.extend(op)
        else:
            self.ops.append(op)

    def _gemm(self, name, **kw):
        kw.setdefault("ws", self._ws_token)
        return ops.gemm_op(name, self.lib_or_dry(), dry=self.dry, **kw)

    def lib_or_dry(self):
        return self.lib if self.lib is not None else _DryLib

    def _a_matrix(self, x: Act):
        return ops.a_matrix(x.ptr, x.rows, x.c, x.ld)

    def group_norm(self, name, x: Act, prefix, silu, eps, dst: Act = None):
        """GroupNorm(+SiLU) of x into `dst` (by default the plan's "gn_out" buffer of x's shape)."""
        y = dst if dst is not None else self.act("gn_out", x.n, x.h, x.w, x.c)
        slot, sync = self.gn_stats[self._gn_count], self.gn_sync[self._gn_count]
        self._gn_count += 1
        partial, pend = None, self._pending
        if pend is not None:
            d = pend["dst"]
            if (d.buf is x.buf and d.off == x.off and d.c <= x.c and
                    (d.n, d.h, d.w) == (x.n, x.h, x.w) and
                    ops.gn_fused_ok(self.lib_or_dry(), x, self.spec.groups, self.dt, self.dry)):
                partial = pend["info"]
                self._pending = None  # absorbed: the GEMM keeps defer_finish = 1
        gn = ops.gn_ops(name, self.lib_or_dry(), x=x, y=y, gamma=self.w.f32(prefix + ".weight"),
                        beta=self.w.f32(prefix + ".bias"), stats=slot, sync=sync,
                        groups=self.spec.groups, eps=eps, silu=silu, dt=self.dt,
                        dry=self.dry, partial=partial)
        if partial is not None:
            self._gn_ws_patches.append(gn[0].keep[0])
        self._emit(gn)
        return y

    def _conv_gn_ok(self, x: Act, cout):
        """Whether GroupNorm+SiLU over `x` is folded into the 3x3 conv that consumes it (halo conv,
        SFB_A_CONV3X3_GN) instead of running as its own kernel.  SFB_CONV_GN = 0: never; 1: wherever the
        geometry allows; auto: where, additionally, the conv is a full launch (no split-K -- the
        weight-bandwidth-bound low-resolution layers keep the fused GroupNorm that also finishes
        their producer's split-K partials)."""
        mode = ops.CONV_GN
        if mode == "0" or x.c % ops.BK:
            return False
        tiles = ops.conv_gn_tiles(x.n, x.h, x.w)
        if not tiles:
            return False
        if mode == "1":
            return True
        if self._pending is not None:
            return False
        if x.c < 640 and x.rows < 16384:
            # few channel blocks in a single-wave launch: the halo kernel's longer pipeline fill costs
            # more than the GroupNorm write + read it saves (measured: 2 x 64^2 x 320 -> +2 us per pair)
            return False
        return ops.choose_splits(tiles, -(-cout // ops.BN), 9 * x.c // ops.BK, x.rows, cout) == 1

    def norm_for_conv(self, name, x: Act, prefix, eps, cout):
        """GroupNorm + SiLU in front of a 3x3 conv with `cout` outputs.  Returns (conv input, gn):
        gn is None when the normalised activation was materialised by a GroupNorm kernel, else the
        descriptor the conv needs to normalise its raw input itself."""
        if not self._conv_gn_ok(x, cout):
            return self.group_norm(name, x, prefix, True, eps), None
        idx = self._gn_count
        self._gn_count += 1
        assert x.n <= self.gn_tickets.shape[1], "one ticket per image of the GroupNorm"
        ab = self.buf(f"gn_scale_shift.{idx}", (x.n, x.c, 2), torch.float32)
        self._emit(ops.gn_scale_shift_op(name, self.lib_or_dry(), x=x, gamma=self.w.f32(prefix + ".weight"),
                                         beta=self.w.f32(prefix + ".bias"), stats=self.gn_stats[idx],
                                         counters=self.gn_tickets[idx], scale_shift=ab,
                                         groups=self.spec.groups, eps=eps, dt=self.dt))
        return x, dict(scale_shift=ab, silu=True)

    def conv3x3(self, name, x: Act, wname, dst: Act, stride=1, rowbias=None, residual: Act = None, gn=None,
                down=False, weights=None, act=0):
        """`down`: diffusers' Downsample2D with padding=0 (the VAE encoder's) -- stride 2, one zero row and
        column AFTER the image, none before (SFB_A_DOWNCONV3X3).  `weights`: a packed (Mat, fp32 bias) pair
        used instead of the parameters `wname`; `act`: SFB_ACT_* of the epilogue (no split-K then)."""
        if down:
            stride = 2
        wm = self.w.conv3x3(wname + ".weight") if weights is None else weights[0]
        cout = wm.n
        ho, wo = x.h // stride, x.w // stride
        if gn is not None:  # raw input, GroupNorm applied on the conv's operand path
            assert stride == 1
            box_n, box_h, box_w = 1, ops.HALO_BOX_H, ops.HALO_BOX_W
            adesc = ops.a_conv_halo(x.ptr, x.n, x.h, x.w, x.c, x.ld)
        else:
            box_n, box_h, box_w = ops.conv_tile_box(ho, wo)
            adesc = ops.a_conv(x.ptr, x.n, x.h, x.w, x.c, x.ld, box_n, box_h, box_w, stride)
        M = x.n * ho * wo
        kw = dict(a=adesc, b=wm, M=M, N=cout, K=9 * x.c, dt=self.dt,
                  out=dst.ptr, ldo=dst.ld, bias=self.w.f32(wname + ".bias") if weights is None else weights[1],
                  conv=dict(n=x.n, h=ho, w=wo, cin=x.c, stride=stride, box_n=box_n, box_h=box_h,
                            box_w=box_w, down=down),
                  keep=(x.buf, dst.buf, wm))
        if act:
            kw.update(act=act, splits=1)
        if rowbias is not None:
            kw.update(rowbias=rowbias[0], rows_per_img=ho * wo, ld_rowbias=rowbias[1])
        if residual is not None:
            kw.update(residual=residual.ptr, ldr=residual.ld)
        if gn is not None:
            kw.update(gn=gn)
        op = self._gemm(name, **kw)
        self._emit(op)
        self._maybe_defer_finish(op.keep[0], dst, cout, kw["bias"], rowbias, residual)

    def _maybe_defer_finish(self, gp, dst, cout, bias, rowbias=None, residual=None):
        """Tentatively leave a conv's split-K reduction to the GroupNorm that consumes dst next."""
        if gp.splits > 1 and os.environ.get("SFB_GN_FINISH", "1") != "0":
            gp.defer_finish = 1
            info = dict(splits=gp.splits, c=cout, ld=cout, bias=bias)
            if rowbias is not None:
                info.update(rowbias=rowbias[0], ld_rowbias=rowbias[1])
            if residual is not None:
                info.update(residual=residual.ptr, ldr=residual.ld, res_buf=residual.buf)
            self._pending = dict(p=gp, dst=dst, info=info)

    def upconv3x3(self, name, x: Act, wname, dst: Act):
        """nearest-2x upsample + conv3x3 of `x` -> dst ([n, 2h, 2w, cout]) without materialising
        the upsampled tensor: four 2x2 convolutions on x (one per output phase), 4/9 of the MACs."""
        wm, cout = self.w.upconv(wname + ".weight")
        box_n, box_h, box_w = ops.conv_tile_box(x.h, x.w)
        adesc = ops.a_conv(x.ptr, x.n, x.h, x.w, x.c, x.ld, box_n, box_h, box_w, 1)
        M = 4 * x.n * x.h * x.w
        bias = self.w.f32(wname + ".bias")
        op = self._gemm(name, a=adesc, b=wm, M=M, N=cout, K=4 * x.c, dt=self.dt, out=dst.ptr,
                        ldo=dst.ld, bias=bias, keep=(x.buf, dst.buf, wm),
                        conv=dict(n=x.n, h=x.h, w=x.w, cin=x.c, stride=1, box_n=box_n, box_h=box_h,
                                  box_w=box_w, up=True))
        op.flops = 2 * M * cout * 9 * x.c  # algorithmic count of the reference formulation
        self._emit(op)
        self._maybe_defer_finish(op.keep[0], dst, cout, bias)

    def linear(self, name, x: Act, wm, bias, dst: Act, residual: Act = None, rowstats_out=None,
               splits=None):
        kw = dict(a=self._a_matrix(x), b=wm, M=x.rows, N=wm.n, K=x.c, dt=self.dt,
                  out=dst.ptr, ldo=dst.ld, bias=bias, keep=(x.buf, dst.buf, wm),
                  rowstats_out=rowstats_out, splits=splits)
        if residual is not None:
            kw.update(residual=residual.ptr, ldr=residual.ld)
        op = self._gemm(name, **kw)
        self._emit(op)

    def layer_norm(self, name, x: Act, prefix, eps=1e-5):
        y = self.act("ln_out", x.n, x.h, x.w, x.c)
        self._emit(ops.ln_op(name, self.lib_or_dry(), x=x.buf, y=y.buf, rows=x.rows, c=x.c,
                             gamma=self.w.f32(prefix + ".weight"), beta=self.w.f32(prefix + ".bias"),
                             eps=eps, dt=self.dt))
        return y

    def attention_operands(self, B, H, S, skv, D, kv_tag="", q_tag=""):
        """q [B*H*S, q_pitch], k [B*H*skv, q_pitch] and v^T [B*H*dv, vt_pitch] buffers of one flash-attention
        launch, as the QKV-scatter epilogue and the attention kernel address them.  v^T carries an all-ones
        row after the D value rows: P times it is the softmax denominator, computed on the tensor core.
        `kv_tag` keeps k / v^T apart from other launches of the same shape (the UNet's hoisted cross K/V);
        `q_tag` does the same for q (operands written on the side stream)."""
        dv = _round_up(D + 1, 16)
        q_pitch, vt_pitch = _round_up(D, 64), _round_up(skv, 64)
        tag = f"{B}x{H}x{S}x{skv}x{D}"
        q = self.buf("attn_q_" + tag + q_tag, (B * H * S, q_pitch))
        k = self.buf("attn_k_" + tag + kv_tag, (B * H * skv, q_pitch))
        new_vt = ("attn_vt_" + tag + kv_tag, (B * H * dv, vt_pitch), self.dt) not in self._bufs
        vt = self.buf("attn_vt_" + tag + kv_tag, (B * H * dv, vt_pitch))
        if new_vt and not self.dry:
            vt.view(B * H, dv, vt_pitch)[:, D, :] = 1.0
        return dict(q=q, k=k, vt=vt, heads=H, head_dim=D, q_pitch=q_pitch, q_rows=S, k_rows=skv,
                    vt_rows=dv, vt_pitch=vt_pitch)

    def attention_core(self, name, qkv, out: Act, **kw):
        """softmax(q k^T / sqrt(D)) v over the attention_operands `qkv` -> out ([B, S, heads * D] rows)."""
        self._emit(ops.attention_op(name, self.lib_or_dry(), out=out.buf, batch=out.n, seq_q=qkv["q_rows"],
                                    seq_kv=qkv["k_rows"], dt=self.dt, dry=self.dry, **qkv, **kw))

    def conv_in(self, prefix, x, dst: Act):
        """3x3 conv of the NCHW model input x (few channels, sfb_conv_in) -> NHWC dst."""
        B, cin, H, W = x.shape
        w = self.w.conv_in_weight(prefix + ".weight")
        self._emit(Op(prefix, self.lib_or_dry().sfb_conv_in,
                      (_ptr(x), _ptr(w), _ptr(self.w.f32(prefix + ".bias")), dst.ptr, B, H, W, cin, dst.c, dst.ld,
                       ops.dtype_code(self.dt)), (x, w, dst.buf), 2 * B * H * W * dst.c * 9 * cin))

    def conv_out(self, name, y: Act, w, bias, out, flops=None):
        """3x3 conv of NHWC y to the few-channel NCHW model output `out` (sfb_conv_out); `w` packed like
        PackedWeights.conv3x3_plain."""
        cout = out.shape[1]
        self._emit(Op(name, self.lib_or_dry().sfb_conv_out,
                      (y.ptr, _ptr(w), _ptr(bias), _ptr(out), y.n, y.h, y.w, y.c, cout, y.ld, ops.dtype_code(self.dt)),
                      (y.buf, w, bias, out), flops or 2 * y.rows * y.c * 9 * cout))

    # ------------------------------------------------------------------ execution
    def run(self, stream=None):
        """Launch one step on torch's current stream (plus the forked side stream)."""
        main = torch.cuda.current_stream()
        mptr = main.cuda_stream
        if self.side_ops:
            if self._side_stream is None:
                self._side_stream = torch.cuda.Stream()
                self._temb_event = torch.cuda.Event()
            side = self._side_stream
            side.wait_stream(main)  # inputs were copied on the main stream
            sptr = side.cuda_stream
            for op in self.side_ops:
                op.launch(sptr)
                if op is self._temb_last:
                    self._temb_event.record(side)
        for op in self.ops:
            if isinstance(op, _JoinOp):
                if op.kind == "temb":
                    main.wait_event(self._temb_event)
                elif op.kind == "all":
                    main.wait_stream(self._side_stream)
                else:  # join of one forked branch
                    main.wait_event(op.kind.ev_done)
            elif isinstance(op, _ForkOp):
                if op.ev_fork is None:
                    op.ev_fork, op.ev_done = torch.cuda.Event(), torch.cuda.Event()
                op.ev_fork.record(main)
                side.wait_event(op.ev_fork)
                for o in op.branch:
                    o.launch(sptr)
                op.ev_done.record(side)
            else:
                op.launch(mptr)

    def all_ops(self):
        """Every kernel-launching op of one step (markers removed, forked branches expanded)."""
        out = list(self.side_ops)
        for op in self.ops:
            if isinstance(op, _ForkOp):
                out.extend(op.branch)
            elif not isinstance(op, _JoinOp):
                out.append(op)
        return out

    def flops(self):
        return sum(op.flops for op in self.all_ops())


class VideoPlanMixin:
    """Emitters of a plan whose batch is `nvid` videos of `F` consecutive frames (both set by the plan) --
    the SVD UNet, SVD's temporal VAE decoder and the AnimateDiff UNet.  Frames are a batch of images for everything
    spatial; a temporal operator works on the same token-major [B*F*H*W, C] tensors viewed as [B, F, H*W, C]."""

    def _video_view(self, x: Act):
        """[B*F, h, w, c] -> [B, F*h, w, c]: GroupNorm statistics over (frames, height, width)."""
        return Act(x.buf, self.nvid, self.F * x.h, x.w, x.c, ld=x.ld, off=x.off)

    def _frame_view(self, y: Act, like: Act):
        return Act(y.buf, like.n, like.h, like.w, y.c, ld=y.ld, off=y.off)

    def _ff(self, b, ffname, ln_prefix, hs: Act, st, stats_next, dim):
        """hs += ff(LayerNorm(hs)): GEGLU projection (LayerNorm folded) + output projection."""
        gm, bp, inner, colsum = self.w.ln_geglu(f"{b}.{ffname}.net.0.proj", ln_prefix)
        ff = self.act("ff_act", hs.n, hs.h, hs.w, inner)
        self._emit(self._gemm(f"{b}.{ffname}.geglu", a=self._a_matrix(hs), b=gm, M=hs.rows, N=gm.n, K=dim,
                              dt=self.dt, out=ff.ptr, ldo=inner, bias=bp, epi=EPI_GEGLU, geglu_n_out=inner,
                              ln=dict(rowstats=st, colsum=colsum, eps=1e-5, dim=dim),
                              keep=(hs.buf, ff.buf, gm, colsum)))
        self.linear(f"{b}.{ffname}.out", ff, self.w.matrix(f"{b}.{ffname}.net.2.weight"),
                    self.w.f32(f"{b}.{ffname}.net.2.bias"), hs, residual=hs, rowstats_out=stats_next)

    def conv3x1_t(self, name, x: Act, wm, bias, dst: Act, rowbias=None, residual: Act = None):
        """Conv3d (3,1,1), padding (1,0,0) over the frame axis of x viewed as [B, F, H*W, C]."""
        S = x.h * x.w
        box_n, box_h, box_w = ops.conv_tile_box(self.F, S)
        adesc = ops.a_conv(x.ptr, self.nvid, self.F, S, x.c, x.ld, box_n, box_h, box_w, 1)
        M = x.rows
        kw = dict(a=adesc, b=wm, M=M, N=wm.n, K=3 * x.c, dt=self.dt, out=dst.ptr, ldo=dst.ld, bias=bias,
                  conv=dict(n=self.nvid, h=self.F, w=S, cin=x.c, stride=1, box_n=box_n, box_h=box_h,
                            box_w=box_w, temporal=True),
                  keep=(x.buf, dst.buf, wm), splits=1)
        if rowbias is not None:
            kw.update(rowbias=rowbias[0], rows_per_img=self.F * S, ld_rowbias=rowbias[1])
        if residual is not None:
            kw.update(residual=residual.ptr, ldr=residual.ld)
        self._emit(self._gemm(name, **kw))


class UNetPlan(Plan):
    """One static launch schedule of the UNet for a fixed (batch, height, width)."""

    _motion = False  # MotionUNetPlan: emits the motion modules of spec.motion

    def __init__(self, weights: PackedWeights, batch, height, width, ctx_len=77, controlnet=False, ip_len=0,
                 ip_seq=0, intrablock=0, freeu=(False, False)):
        """`ip_len` > 0: an IP-Adapter (spec.ip) adds ip_len image tokens per sample (n_img images x its
        tokens per image) to every cross-attention; 0 builds exactly the schedule without one.  `ip_seq`:
        feature tokens per image of an IP-Adapter Plus (spec.ip.resampler), the input of its Resampler.
        `intrablock`: how many T2I-Adapter residuals the step adds (the first `intrablock` insertion points of
        intrablock_shapes, static NCHW inputs `intrablock_in`); 0 builds exactly the schedule without them.
        `freeu`: (up block 0, up block 1) flags; a block that is on runs FreeU (sfb_freeu) in front of each of
        its resnets with the values of the static input `freeu_in` = (b1, s1, b2, s2); (False, False) builds
        exactly the schedule without it."""
        spec = weights.spec
        if spec.motion and not self._motion:
            raise ValueError("a UNetMotionModel spec (spec.motion) is built by motion_plan.MotionUNetPlan")
        div = 1 << (len(spec.block_out_channels) - 1)
        if height % div or width % div:
            # diffusers switches to explicit upsample sizes there (forward_upsample_size); not built
            raise NotImplementedError(
                f"sfast (H100 build): latent size {height}x{width} must be a multiple of {div}")
        # (+1: conv_norm_out, the head of the up path; a ControlNet has none)
        n_gn = sum(2 for _ in spec.all_resnets()) + (1 if spec.up else 0) + sum(
            1 for blk in spec.down + [spec.mid] + spec.up for t in blk.attentions if t is not None) + len(spec.motion)
        super().__init__(weights, batch, height, width, n_gn=n_gn,
                         ln_floats=self._ln_arena_floats(spec, batch, height, width))
        self.ctx_len = ctx_len
        self.controlnet = controlnet
        self.ctrl_in = []  # static NCHW inputs: 12 (SD-1.5) down-block residuals + the mid-block one
        points = intrablock_shapes(spec, batch, height, width)
        if not 0 <= intrablock <= len(points):
            raise ValueError(f"intrablock={intrablock}: the UNet has {len(points)} T2I-Adapter insertion points")
        self.intrablock_in = [self._alloc(s, self.dt) for s in points[:intrablock]]
        self.freeu = tuple(bool(f) for f in freeu)
        if len(self.freeu) != 2:
            raise ValueError(f"freeu={freeu!r}: one flag for each of up blocks 0 and 1")
        if any(self.freeu):
            if len(spec.up) < 2:
                raise ValueError(f"freeu={freeu!r}: the UNet has {len(spec.up)} up blocks")
            # device memory: a captured graph serves every value
            self.freeu_in = self._alloc((4,), torch.float32)
        # ---- static inputs / output
        self.sample_in = self._alloc((batch, spec.in_channels, height, width), self.dt)
        self.t_in = self._alloc((batch,), torch.float32)
        self.ehs_in = self._alloc((batch, ctx_len, spec.cross_attention_dim), self.dt)
        self.out = self._alloc((batch, spec.out_channels, height, width), self.dt)
        if spec.time_cond_dim:  # LCM: the guidance embedding timestep_cond
            self.timestep_cond_in = self._alloc((batch, spec.time_cond_dim), self.dt)
        if spec.addition_embed_type == "text_time":
            self.add_in = self._alloc((batch, spec.add_in_dim), self.dt)
            self.time_ids_in = self._alloc((batch * 6,), torch.float32)
        self.ip_len = ip_len
        if ip_len:
            ip = spec.ip
            if ip is None or ip_len % ip.tokens:
                raise ValueError(f"ip_len={ip_len} needs an IP-Adapter spec with a multiple of its tokens per image")
            kv = min(ops.attention_kv_tile(t.head_dim) for _, t in spec.cross_attention_layers())
            if ip_len > kv:
                raise NotImplementedError(f"sfast (H100 build): {ip_len} IP-Adapter image tokens per sample; the "
                                          f"fused attention takes at most {kv} (one KV tile)")
            # static inputs: the image embeddings [B * n_img, D_img] (Plus: the image features [B * n_img *
            # ip_seq, D_img]) and one scale per cross-attention (device memory: a captured graph serves every
            # scale, per-block scales included)
            rows = batch * (ip_len // ip.tokens)
            self.ip_seq = 0
            if ip.resampler is not None:
                if ip_seq <= 0:
                    raise ValueError("an IP-Adapter Plus plan needs ip_seq > 0 (image feature tokens per image)")
                self.ip_seq = ip_seq
                rows *= ip_seq
            self.image_embeds_in = self._alloc((rows, ip.image_embed_dim), self.dt)
            self.ip_scale_in = self._alloc((len(ip.layers),), torch.float32)
            self._ip_slot = {p: i for i, p in enumerate(ip.layers)}
            self._ip_tokens = None
        self._build()

    @staticmethod
    def _ln_arena_floats(spec, batch, height, width):
        """3 * depth LayerNorms per transformer, each [B*h*w, slots(dim), 2] floats at its resolution."""
        tot, h, w = 0, height, width

        def need(blk):
            return sum(3 * t.depth * batch * h * w * 2 * ops.rowstats_slots(t.dim)
                       for t in blk.attentions if t is not None)
        for blk in spec.down:
            tot += need(blk)
            if blk.sampler:
                h, w = h // 2, w // 2
        tot += need(spec.mid)
        for blk in spec.up:
            tot += need(blk)
            if blk.sampler:
                h, w = h * 2, w * 2
        return tot

    # ------------------------------------------------------------------ sub-graphs
    def resnet(self, r, x: Act, dst: Act):
        p = r.prefix
        fork = None
        # norm1 first: it may be the kernel that finishes x (deferred split-K reduction of the
        # conv that produced it), so every other reader of x is ordered after it
        eps = r.eps if r.eps is not None else self.spec.eps
        a1, gn1 = self.norm_for_conv(p + ".norm1", x, p + ".norm1", eps, r.cout)
        if r.has_shortcut and os.environ.get("SFB_SIDE_SHORTCUT", "1") != "0":
            # the 1x1 shortcut only needs the block input: parallel graph branch next to
            # norm1 / conv1 / norm2 (most of these launches leave SMs idle at small batch)
            sc = self.act("res_sc", x.n, x.h, x.w, r.cout)
            n0 = len(self.ops)
            self.linear(p + ".conv_shortcut", x, self.w.matrix(p + ".conv_shortcut.weight"),
                        self.w.f32(p + ".conv_shortcut.bias"), sc, splits=1)
            fork = _ForkOp(self.ops[n0:])
            del self.ops[n0:]
            self._emit(fork)
        h1 = self.act("res_h1", x.n, x.h, x.w, r.cout)
        rb_ptr = _ptr(self.temb_proj) + 4 * self.w.tproj_off[p]
        self.conv3x3(p + ".conv1", a1, p + ".conv1", h1, rowbias=(rb_ptr, self.w.tproj_total), gn=gn1)
        a2, gn2 = self.norm_for_conv(p + ".norm2", h1, p + ".norm2", eps, r.cout)
        if fork is not None:
            self._emit(_JoinOp(fork))
            res = sc
        elif r.has_shortcut:
            sc = self.act("res_sc", x.n, x.h, x.w, r.cout)
            self.linear(p + ".conv_shortcut", x, self.w.matrix(p + ".conv_shortcut.weight"),
                        self.w.f32(p + ".conv_shortcut.bias"), sc)
            res = sc
        else:
            res = x
        self.conv3x3(p + ".conv2", a2, p + ".conv2", dst, residual=res, gn=gn2)

    def attention(self, name, hs: Act, ln_prefix, ln_stats, blk, t, cross, stats_next):
        """attn(LayerNorm(hs)) + hs -> hs (in place).  The LayerNorm is folded into the Q(KV)
        projection (gamma-scaled weights + epilogue mean/rstd correction from `ln_stats`, the row
        sums the previous GEMM accumulated); `stats_next` receives the row sums of the new hs.
        Self-attention: fused QKV projection; cross: Q from the tokens, K/V from the text."""
        B, S, C = hs.n, hs.h * hs.w, t.dim
        a = f"{blk}.attn2" if cross else f"{blk}.attn1"
        # hoisted cross K/V: one buffer pair per layer
        qkv = self.attention_operands(B, t.heads, S, self.ctx_len if cross else S, t.head_dim,
                                      kv_tag="@" + a if cross else "")
        names = [f"{a}.to_q.weight"] if cross else [f"{a}.to_q.weight", f"{a}.to_k.weight",
                                                    f"{a}.to_v.weight"]
        wm, bias, colsum = self.w.ln_matrix(names, ln_prefix)
        self._emit(self._gemm(a + (".q" if cross else ".qkv"), a=self._a_matrix(hs), b=wm,
                              M=hs.rows, N=wm.n, K=C, dt=self.dt, epi=EPI_QKV, bias=bias,
                              qkv=dict(qkv, which_base=0, seq=S),
                              ln=dict(rowstats=ln_stats, colsum=colsum, eps=1e-5, dim=C),
                              keep=(hs.buf, wm, colsum)))
        if cross:
            wkv = self.w.cat_matrix([f"{a}.to_k.weight", f"{a}.to_v.weight"])
            ehs = Act(self.ehs_in, B, 1, self.ctx_len, self.spec.cross_attention_dim)
            self.side_ops.append(self._gemm(a + ".kv", a=self._a_matrix(ehs), b=wkv, M=ehs.rows,
                                            N=2 * C, K=ehs.c, dt=self.dt, epi=EPI_QKV,
                                            qkv=dict(qkv, which_base=1, seq=self.ctx_len),
                                            splits=1, keep=(self.ehs_in, wkv)))
            if not self._joined:
                self._joined = True
                self._emit(_JoinOp("all"))
        ao = self.act("attn_out", hs.n, hs.h, hs.w, C)
        if cross and self.ip_len:
            self.attention_core(a + ".core", qkv, ao, ip=self._ip_kv(a, B, t))
            return self.linear(a + ".to_out", ao, self.w.matrix(f"{a}.to_out.0.weight"),
                               self.w.f32(f"{a}.to_out.0.bias"), hs, residual=hs, rowstats_out=stats_next)
        self.attention_core(a + ".core", qkv, ao)
        self.linear(a + ".to_out", ao, self.w.matrix(f"{a}.to_out.0.weight"),
                    self.w.f32(f"{a}.to_out.0.bias"), hs, residual=hs, rowstats_out=stats_next)

    def _ip_kv(self, a, B, t):
        """IP-Adapter operands of cross-attention `a` (side stream, before the join of the first one): the
        image tokens LayerNorm(image_embeds W^T + b) (IP-Adapter Plus: the Resampler, _resampler) once per
        step, then this layer's K / V^T of them through the QKV-scatter epilogue into its own buffers.  Returns
        the `ip` argument of ops.attention_op."""
        ip, lib = self.spec.ip, self.lib_or_dry()
        if self._ip_tokens is None and ip.resampler is not None:
            self._ip_tokens = self._resampler(lib)
        if self._ip_tokens is None:
            pp = "encoder_hid_proj.image_projection_layers.0"
            rows = self.image_embeds_in.shape[0]
            proj = self.buf("ip_proj", (rows, ip.tokens * ip.ctx_dim))
            self.side_ops.append(ops.small_linear_op(
                pp + ".image_embeds", lib, x=self.image_embeds_in, w=self.w.small(pp + ".image_embeds.weight"),
                bias=self.w.f32(pp + ".image_embeds.bias"), batch=rows, n=ip.tokens * ip.ctx_dim,
                k=ip.image_embed_dim, dt=self.dt, y16=proj))
            self._ip_tokens = self.buf("ip_tokens", (rows * ip.tokens, ip.ctx_dim))
            self.side_ops.append(ops.ln_op(pp + ".norm", lib, x=proj, y=self._ip_tokens, rows=rows * ip.tokens,
                                           c=ip.ctx_dim, gamma=self.w.f32(pp + ".norm.weight"),
                                           beta=self.w.f32(pp + ".norm.bias"), eps=ip.norm_eps, dt=self.dt))
        H, D, C = t.heads, t.head_dim, t.dim
        kv_tile = ops.attention_kv_tile(D)
        # k [B*H*ip_len, q_pitch] like the text K; v^T [B*H*dv, kv_tile]: one whole KV tile of columns, so the
        # kernel's V^T loads stay inside the buffer (columns >= ip_len stay zero); no ones row is needed
        dv, q_pitch = _round_up(D + 1, 16), _round_up(D, 64)
        k = self.buf("attn_k_ip@" + a, (B * H * self.ip_len, q_pitch))
        vt = self.buf("attn_vt_ip@" + a, (B * H * dv, kv_tile))
        wkv = self.w.cat_matrix([f"{a}.processor.to_k_ip.0.weight", f"{a}.processor.to_v_ip.0.weight"])
        tok = Act(self._ip_tokens, B, 1, self.ip_len, ip.ctx_dim)
        self.side_ops.append(self._gemm(
            a + ".ip_kv", a=self._a_matrix(tok), b=wkv, M=tok.rows, N=2 * C, K=ip.ctx_dim, dt=self.dt, epi=EPI_QKV,
            qkv=dict(k=k, vt=vt, heads=H, head_dim=D, which_base=1, seq=self.ip_len, q_pitch=q_pitch,
                     q_rows=self.ip_len, k_rows=self.ip_len, vt_rows=dv, vt_pitch=kv_tile),
            splits=1, keep=(self._ip_tokens, wkv)))
        i = self._ip_slot[a]
        return dict(k=k, vt=vt, seq=self.ip_len, k_rows=self.ip_len, vt_pitch=kv_tile,
                    scale=self.ip_scale_in[i:i + 1])

    def _resampler(self, lib):
        """IP-Adapter Plus's image projection (diffusers ``IPAdapterPlusImageProjection``), on the side stream:
        the image tokens [N * Q, ctx] of the image features image_embeds_in [N * S, D_img], N = B * n_img,
        Q learned queries (latents), S = ip_seq.  Per block:
            kv = cat(ln1(latents), ln0(x))                     x = proj_in(image features)
            latents += to_out(attention(to_q(ln1(latents)), to_k(kv), to_v(kv)))   dim_head 64, scale 1/8
            latents += ff.2(gelu(ff.1(ff.0(latents))))
        then LayerNorm(proj_out(latents)).  diffusers concatenates (ln0(x), ln1(latents)); softmax . V is a
        sum over keys, so the order is free: the Q latent keys come first and the S feature keys start at a
        Q-row offset of K and a Q-column offset of V^T (16-byte aligned for Q % 8 == 0).  The two segments
        are two QKV-scatter GEMMs into one K / V^T pair.  The latents are broadcast to N rows as
        0 + latents[m % Q] (sfb_row_broadcast_add).  Every GEMM here is split-K free: the split-K workspace
        is shared with the main stream."""
        ip, rs, dt = self.spec.ip, self.spec.ip.resampler, self.dt
        pp = "encoder_hid_proj.image_projection_layers.0"
        Q, S, Dh, H, D = ip.tokens, self.ip_seq, rs.dim, rs.heads, RESAMPLER_HEAD_DIM
        N = self.image_embeds_in.shape[0] // S
        side = self.side_ops

        def gemm(name, x: Act, wm, dst: Act = None, **kw):
            keep = (x.buf, wm) + ((dst.buf,) if dst is not None else ())
            if dst is not None:
                kw.update(out=dst.ptr, ldo=dst.ld)
            side.append(self._gemm(name, a=self._a_matrix(x), b=wm, M=x.rows, N=wm.n, K=x.c, dt=dt, splits=1,
                                   keep=keep, **kw))

        def layer_norm(name, x: Act, y: Act, eps):
            side.append(ops.ln_op(name, lib, x=x.buf, y=y.buf, rows=x.rows, c=x.c, gamma=self.w.f32(name + ".weight"),
                                  beta=self.w.f32(name + ".bias"), eps=eps, dt=dt))

        lat = Act(self.buf("rs_latents", (N * Q, Dh)), N, 1, Q, Dh)
        zero = Act(self.buf("rs_zero", (N * Q, Dh)), N, 1, Q, Dh)  # never written
        latents = self.w.small(pp + ".latents")
        p = _lib.RowOpParams()
        p.x, p.y, p.vec, p.ldv = zero.ptr, lat.ptr, _ptr(latents), Dh
        p.rows, p.c, p.ldx, p.ldy, p.dtype = lat.rows, Dh, Dh, Dh, ops.dtype_code(dt)
        p.mode, p.div, p.mod = _lib.ROW_IDX_DIV_MOD, 1, Q
        side.append(Op(pp + ".latents", lib.sfb_row_broadcast_add, (C.byref(p),),
                       (p, zero.buf, lat.buf, latents, None, None, None), 0, 3 * lat.rows * Dh * 2))
        x = Act(self.buf("rs_x", (N * S, Dh)), N, 1, S, Dh)
        gemm(pp + ".proj_in", Act(self.image_embeds_in, N, 1, S, ip.image_embed_dim),
             self.w.matrix(pp + ".proj_in.weight"), x, bias=self.w.f32(pp + ".proj_in.bias"))
        skv = Q + S
        qkv = self.attention_operands(N, H, Q, skv, D, kv_tag="@resampler", q_tag="@resampler")
        esz = qkv["q"].element_size()
        img_kv = dict(qkv, k=_ptr(qkv["k"]) + Q * qkv["q_pitch"] * esz, vt=_ptr(qkv["vt"]) + Q * esz, which_base=1,
                      seq=S)
        xn = Act(self.buf("rs_ln0", (N * S, Dh)), N, 1, S, Dh)
        ln = Act(self.buf("rs_ln1", (N * Q, Dh)), N, 1, Q, Dh)
        ao = Act(self.buf("rs_attn", (N * Q, rs.inner)), N, 1, Q, rs.inner)
        hid = Act(self.buf("rs_ff", (N * Q, rs.ff_dim)), N, 1, Q, rs.ff_dim)
        for i in range(rs.depth):
            b = f"{pp}.layers.{i}"
            e0, e1, e2 = rs.block_eps[i]
            layer_norm(b + ".ln0", x, xn, e0)
            layer_norm(b + ".ln1", lat, ln, e1)
            wq, wk, wv = (f"{b}.attn.{n}.weight" for n in ("to_q", "to_k", "to_v"))
            gemm(b + ".attn.qkv", ln, self.w.cat_matrix([wq, wk, wv]), epi=EPI_QKV,
                 qkv=dict(qkv, which_base=0, seq=Q))
            gemm(b + ".attn.kv_image", xn, self.w.cat_matrix([wk, wv]), epi=EPI_QKV, qkv=img_kv)
            side.append(ops.attention_op(b + ".attn.core", lib, out=ao.buf, batch=N, seq_q=Q, seq_kv=skv, dt=dt,
                                         dry=self.dry, **qkv))
            gemm(b + ".attn.to_out", ao, self.w.matrix(b + ".attn.to_out.0.weight"), lat,
                 residual=lat.ptr, ldr=lat.ld)
            layer_norm(b + ".ff.0", lat, ln, e2)
            gemm(b + ".ff.1.net.0.proj", ln, self.w.matrix(b + ".ff.1.net.0.proj.weight"), hid, act=_lib.ACT_GELU)
            gemm(b + ".ff.1.net.2", hid, self.w.matrix(b + ".ff.1.net.2.weight"), lat, residual=lat.ptr,
                 ldr=lat.ld)
        proj = Act(self.buf("ip_proj", (N * Q, ip.ctx_dim)), N, 1, Q, ip.ctx_dim)
        gemm(pp + ".proj_out", lat, self.w.matrix(pp + ".proj_out.weight"), proj,
             bias=self.w.f32(pp + ".proj_out.bias"))
        tokens = Act(self.buf("ip_tokens", (N * Q, ip.ctx_dim)), N, 1, Q, ip.ctx_dim)
        layer_norm(pp + ".norm_out", proj, tokens, ip.norm_eps)
        return tokens.buf

    def transformer(self, t, x: Act, dst: Act):
        p = t.prefix
        a1 = self.group_norm(p + ".norm", x, p + ".norm", False, 1e-6)
        hs = self.act("tf_hidden", x.n, x.h, x.w, t.dim)
        st = self.ln_slot(hs.rows, t.dim)
        self.linear(p + ".proj_in", a1, self.w.matrix(p + ".proj_in.weight"),
                    self.w.f32(p + ".proj_in.bias"), hs, rowstats_out=st)
        for d in range(t.depth):
            b = f"{p}.transformer_blocks.{d}"
            st2 = self.ln_slot(hs.rows, t.dim)
            self.attention(b + ".attn1", hs, b + ".norm1", st, b, t, cross=False, stats_next=st2)
            st3 = self.ln_slot(hs.rows, t.dim)
            self.attention(b + ".attn2", hs, b + ".norm2", st2, b, t, cross=True, stats_next=st3)
            gm, bp, inner, colsum = self.w.ln_geglu(b + ".ff.net.0.proj", b + ".norm3")
            ff = self.act("ff_act", x.n, x.h, x.w, inner)
            self._emit(self._gemm(b + ".ff.geglu", a=self._a_matrix(hs), b=gm, M=hs.rows,
                                  N=gm.n, K=t.dim, dt=self.dt, out=ff.ptr, ldo=inner,
                                  bias=bp, epi=EPI_GEGLU, geglu_n_out=inner,
                                  ln=dict(rowstats=st3, colsum=colsum, eps=1e-5, dim=t.dim),
                                  keep=(hs.buf, ff.buf, gm, colsum)))
            st = self.ln_slot(hs.rows, t.dim) if d + 1 < t.depth else None
            self.linear(b + ".ff.out", ff, self.w.matrix(b + ".ff.net.2.weight"),
                        self.w.f32(b + ".ff.net.2.bias"), hs, residual=hs, rowstats_out=st)
        self.linear(p + ".proj_out", hs, self.w.matrix(p + ".proj_out.weight"),
                    self.w.f32(p + ".proj_out.bias"), dst, residual=x)

    def time_embedding(self):
        spec, B, lib = self.spec, self.B, self.lib_or_dry()
        c0 = spec.block_out_channels[0]
        t_emb = self.buf("t_emb", (B, c0))
        self._emit(Op("time_proj", lib.sfb_timestep_embed,
                      (_ptr(self.t_in), B, c0,
                       int(spec.flip_sin_to_cos), float(spec.freq_shift),
                       _ptr(t_emb), c0, ops.dtype_code(self.dt)),
                      (self.t_in, t_emb)))
        if spec.time_cond_dim:
            # LCM: diffusers' t_emb + cond_proj(timestep_cond), one fp32 sum rounded once
            t_cond = self.buf("t_emb_cond", (B, c0))
            self._emit(ops.small_linear_op("time_embedding.cond_proj", lib, x=self.timestep_cond_in,
                                           w=self.w.small("time_embedding.cond_proj.weight"), bias=None, batch=B,
                                           n=c0, k=spec.time_cond_dim, dt=self.dt, y16=t_cond, add16=t_emb))
            t_emb = t_cond
        h = self.buf("temb_h", (B, spec.temb_dim))
        self._emit(ops.small_linear_op("time_embedding.linear_1", lib, x=t_emb,
                                       w=self.w.small("time_embedding.linear_1.weight"),
                                       bias=self.w.f32("time_embedding.linear_1.bias"), batch=B,
                                       n=spec.temb_dim, k=c0, dt=self.dt, y16=h, act_out=1))
        temb_act = self.buf("temb_act", (B, spec.temb_dim))  # silu(emb): all consumers apply SiLU
        if spec.addition_embed_type == "text_time":
            emb_t = self.buf("temb_t", (B, spec.temb_dim))
            self._emit(ops.small_linear_op("time_embedding.linear_2", lib, x=h,
                                           w=self.w.small("time_embedding.linear_2.weight"),
                                           bias=self.w.f32("time_embedding.linear_2.bias"), batch=B,
                                           n=spec.temb_dim, k=spec.temb_dim, dt=self.dt, y16=emb_t))
            ad = spec.addition_time_embed_dim
            # time_ids -> sinusoid written straight into the tail of the [text_embeds | time] row
            n_text = spec.add_in_dim - 6 * ad
            tid = self.buf("add_tid", (B * 6, ad))
            self._emit(Op("add_time_proj", lib.sfb_timestep_embed,
                          (_ptr(self.time_ids_in), B * 6, ad,
                           int(spec.flip_sin_to_cos), float(spec.freq_shift),
                           _ptr(tid), ad, ops.dtype_code(self.dt)),
                          (self.time_ids_in, tid)))
            h2 = self.buf("add_h", (B, spec.temb_dim))
            self._emit(Op("add_embedding.concat", lib.sfb_copy2d,
                          (_ptr(tid), _ptr(self.add_in) + 2 * n_text, B, 6 * ad, 6 * ad, spec.add_in_dim),
                          (tid, self.add_in)))
            self._emit(ops.small_linear_op("add_embedding.linear_1", lib, x=self.add_in,
                                           w=self.w.small("add_embedding.linear_1.weight"),
                                           bias=self.w.f32("add_embedding.linear_1.bias"), batch=B,
                                           n=spec.temb_dim, k=spec.add_in_dim, dt=self.dt, y16=h2,
                                           act_out=1))
            self._emit(ops.small_linear_op("add_embedding.linear_2", lib, x=h2,
                                           w=self.w.small("add_embedding.linear_2.weight"),
                                           bias=self.w.f32("add_embedding.linear_2.bias"), batch=B,
                                           n=spec.temb_dim, k=spec.temb_dim, dt=self.dt,
                                           y16=temb_act, add16=emb_t, act_out=1))
        else:
            self._emit(ops.small_linear_op("time_embedding.linear_2", lib, x=h,
                                           w=self.w.small("time_embedding.linear_2.weight"),
                                           bias=self.w.f32("time_embedding.linear_2.bias"), batch=B,
                                           n=spec.temb_dim, k=spec.temb_dim, dt=self.dt,
                                           y16=temb_act, act_out=1))
        # all resnets' time projections in one launch: [B, sum(cout)] fp32 row biases
        self.temb_proj = self.buf("temb_proj", (B, self.w.tproj_total), torch.float32)
        self._emit(ops.small_linear_op("time_emb_proj(all)", lib, x=temb_act, w=self.w.tproj_w,
                                       bias=self.w.tproj_b, batch=B, n=self.w.tproj_total,
                                       k=spec.temb_dim, dt=self.dt, y32=self.temb_proj))

    def _sample_conv_in(self, x: Act):
        """conv_in of the static NCHW input sample_in -> x (NHWC)."""
        spec, B, H, W, lib = self.spec, self.B, self.H, self.W, self.lib_or_dry()
        if spec.in_channels <= 7:
            # im2col (K = 9*cin padded to one 64-wide K block) + the tcgen05 GEMM with fused bias
            a_col = self.buf("conv_in_im2col", (B * H * W, 64))
            self._emit(Op("conv_in.im2col", lib.sfb_im2col_in,
                          (_ptr(self.sample_in), _ptr(a_col), B, H, W, spec.in_channels),
                          (self.sample_in, a_col), 0, B * H * W * 128))
            self.linear("conv_in", Act(a_col, B, H, W, 64), self.w.conv_in_matrix("conv_in.weight"),
                        self.w.f32("conv_in.bias"), x)
            self.ops[-1].flops = 2 * B * H * W * x.c * 9 * spec.in_channels  # algorithmic, not padded
        elif spec.in_channels >= 9:
            # inpainting (9 channels): K = 9*cin padded to two 64-wide K blocks, the same GEMM
            a_col = self.buf("conv_in_im2col", (B * H * W, 128))
            self._emit(Op("conv_in.im2col", lib.sfb_im2col_in_wide,
                          (_ptr(self.sample_in), _ptr(a_col), B, H, W, spec.in_channels),
                          (self.sample_in, a_col), 0, B * H * W * (2 * spec.in_channels + 256)))
            self.linear("conv_in", Act(a_col, B, H, W, 128), self.w.conv_in_matrix("conv_in.weight"),
                        self.w.f32("conv_in.bias"), x)
            self.ops[-1].flops = 2 * B * H * W * x.c * 9 * spec.in_channels  # algorithmic, not padded
        else:
            self.conv_in("conv_in", self.sample_in, x)

    def _add_nchw(self, name, srcs, dsts):
        """dsts[i] (NHWC slices) += srcs[i] (static NCHW inputs) in one sfb_add_nchw_residuals launch."""
        prm = _lib.AddNchwParams()
        prm.count, prm.dtype = len(dsts), ops.dtype_code(self.dt)
        for i, (src, d) in enumerate(zip(srcs, dsts)):
            it = prm.items[i]
            it.src, it.dst, it.n, it.c, it.hw, it.ld_dst = _ptr(src), d.ptr, d.n, d.c, d.h * d.w, d.ld
        self._emit(Op(name, self.lib_or_dry().sfb_add_nchw_residuals, (C.byref(prm),),
                      (prm, srcs, [d.buf for d in dsts]), 0, sum(3 * t.numel() * 2 for t in srcs)))

    def _intrablock_add(self, i, x: Act):
        """x += T2I-Adapter residual i, in place, when the step takes one there: right after x's producer, so
        every later reader (the downsampler, the next block, the up-path skip) sees the sum, as in diffusers."""
        if i < len(self.intrablock_in):
            self._add_nchw(f"t2i_adapter.residual.{i}", [self.intrablock_in[i]], [x])

    def _freeu(self, i, name, cat: Act, c_hidden):
        """FreeU of up block i (0 or 1) on one resnet's concat buffer `cat` = hidden [0, c_hidden) | skip, in
        place: after every writer of the buffer and before its resnet, the only reader of both slices."""
        p = _lib.FreeUParams()
        p.x, p.bs = cat.ptr, _ptr(self.freeu_in) + 8 * i
        p.n, p.h, p.w, p.c_hidden, p.c_skip, p.ld = cat.n, cat.h, cat.w, c_hidden, cat.c - c_hidden, cat.ld
        p.dtype = ops.dtype_code(self.dt)
        rows = cat.n * cat.h * cat.w
        self._emit(Op(name, self.lib_or_dry().sfb_freeu, (C.byref(p),), (p, cat.buf, self.freeu_in), 0,
                      rows * (c_hidden + 3 * p.c_skip) * 2))

    # ------------------------------------------------------------------ whole UNet
    def _build(self):
        spec, B, H, W, lib = self.spec, self.B, self.H, self.W, self.lib_or_dry()
        # the time-embedding chain only depends on the timestep: forked stream, joined before the
        # first resnet (its conv1 epilogue adds the projected embedding)
        n_main = len(self.ops)
        self.time_embedding()
        self.side_ops.extend(self.ops[n_main:])
        del self.ops[n_main:]
        self._temb_last = self.side_ops[-1]

        # ---- shape pass: where does every skip tensor live (inside its consumer's concat buffer)
        skip_shapes = [(spec.block_out_channels[0], H, W)]
        h, w = H, W
        for blk in spec.down:
            for _ in blk.resnets:
                skip_shapes.append((blk.cout, h, w))
            if blk.sampler:
                h, w = h // 2, w // 2
                skip_shapes.append((blk.cout, h, w))
        pending = list(range(len(skip_shapes)))
        skip_dst = {}
        up_in = {}
        for i, blk in enumerate(spec.up):
            for j, r in enumerate(blk.resnets):
                idx = pending.pop()
                sc, sh, sw = skip_shapes[idx]
                xc = r.cin - sc
                cat = self.buf(f"cat_{i}_{j}", (B, sh, sw, r.cin))
                skip_dst[idx] = Act(cat, B, sh, sw, sc, ld=r.cin, off=xc)
                up_in[(i, j)] = (Act(cat, B, sh, sw, r.cin), Act(cat, B, sh, sw, xc, ld=r.cin))
        assert not pending

        # ---- conv_in
        x = skip_dst[0]
        self._sample_conv_in(x)
        self._emit(_JoinOp("temb"))
        # ---- down path
        k = 1
        for bi, blk in enumerate(spec.down):
            cross = any(t is not None for t in blk.attentions)
            for r, t in zip(blk.resnets, blk.attentions):
                dst = skip_dst[k]
                k += 1
                if t is None:
                    self.resnet(r, x, dst)
                else:
                    mid = self.act("res_out", x.n, x.h, x.w, r.cout)
                    self.resnet(r, x, mid)
                    self.transformer(t, mid, dst)
                x = dst
            if cross:
                self._intrablock_add(bi, x)
            if blk.sampler:
                dst = skip_dst[k]
                k += 1
                self.conv3x3(blk.sampler, x, blk.sampler, dst, stride=2)
                x = dst
            if not cross:
                self._intrablock_add(bi, x)
        # ---- mid
        m = spec.mid
        a = self.act("res_out", x.n, x.h, x.w, m.cout)
        self.resnet(m.resnets[0], x, a)
        b = self.act("mid_tf_out", x.n, x.h, x.w, m.cout)
        self.transformer(m.attentions[0], a, b)
        self.resnet(m.resnets[1], b, up_in[(0, 0)][1])
        self._intrablock_add(len(spec.down), up_in[(0, 0)][1])
        if self.controlnet:
            # ControlNet: skip tensor i += down_block_additional_residuals[i], mid output +=
            # mid_block_additional_residual (diffusers adds them after the down / mid blocks; the
            # reference passes them through its traced UNet as plain inputs,
            # /root/reference/src/sfast/compilers/diffusion_pipeline_compiler.py:89-90).  Every
            # down-path reader of a skip slice has run by now and no up-path reader has: one
            # multi-tensor launch adds all of them in place (on top of any T2I-Adapter residual).
            dsts = [skip_dst[i] for i in range(len(skip_shapes))] + [up_in[(0, 0)][1]]
            self.ctrl_in = [self._alloc((B, d.c, d.h, d.w), self.dt) for d in dsts]
            self._add_nchw("controlnet.residuals", self.ctrl_in, dsts)
        # ---- up path
        for i, blk in enumerate(spec.up):
            n_res = len(blk.resnets)
            for j, (r, t) in enumerate(zip(blk.resnets, blk.attentions)):
                xin = up_in[(i, j)][0]
                if i < 2 and self.freeu[i]:
                    self._freeu(i, r.prefix + ".freeu", xin, up_in[(i, j)][1].c)
                last = j == n_res - 1
                if not last:
                    dst = up_in[(i, j + 1)][1]
                elif blk.sampler:
                    dst = self.act("up_block_out", xin.n, xin.h, xin.w, r.cout)
                else:
                    dst = self.act("final_hidden", xin.n, xin.h, xin.w, r.cout)
                if t is None:
                    self.resnet(r, xin, dst)
                else:
                    mid = self.act("res_out", xin.n, xin.h, xin.w, r.cout)
                    self.resnet(r, xin, mid)
                    self.transformer(t, mid, dst)
                x = dst
            if blk.sampler and os.environ.get("SFB_UPCONV", "1") != "0":
                self.upconv3x3(blk.sampler, x, blk.sampler, up_in[(i + 1, 0)][1])
            elif blk.sampler:
                up = self.act("upsampled", x.n, 2 * x.h, 2 * x.w, x.c)
                self._emit(Op(blk.sampler + ".nearest2x", lib.sfb_upsample2x,
                              (x.ptr, up.ptr, x.n,
                               x.h, x.w, x.c, x.ld, up.ld), (x.buf, up.buf), 0,
                              5 * x.rows * x.c * 2))
                self.conv3x3(blk.sampler, up, blk.sampler, up_in[(i + 1, 0)][1])
        # ---- head
        y = self.group_norm("conv_norm_out", x, "conv_norm_out", True, spec.eps)
        self.conv_out("conv_out", y, self.w.conv3x3_plain("conv_out.weight"), self.w.f32("conv_out.bias"), self.out)
        self._finish()


class _WsToken:
    """Deferred split-K workspace: ops are created before the shared buffer size is known."""

    def numel(self):
        return 1 << 62

    def data_ptr(self):
        return 0

    def finalize(self, plan):
        need = 0
        gemm = plan.lib_or_dry().sfb_gemm
        main_ops = [op for op in plan.ops if not isinstance(op, (_ForkOp, _JoinOp))]
        for op in main_ops:
            if op.fn is gemm and op.keep[0].splits > 1:
                need = max(need, op.keep[0].splits * op.keep[0].M * op.keep[0].N)
        plan.ws = plan._alloc((max(need, 1),), torch.float32)
        for op in main_ops:
            if op.fn is gemm and op.keep[0].splits > 1:
                op.keep[0].ws = _ptr(plan.ws)
        # side-stream GEMMs run concurrently with the main chain: they must not share the
        # split-K workspace, so they are never split
        for gp in plan._gn_ws_patches:
            gp.part_ws = _ptr(plan.ws)
        forked = [o for op in plan.ops if isinstance(op, _ForkOp) for o in op.branch]
        for op in plan.side_ops + forked:
            if op.fn is gemm and op.keep[0].splits > 1:
                raise AssertionError("side-stream GEMM must not use split-K")


class _JoinOp(Op):
    """Main stream waits for the side stream here: "all" (everything issued so far), "temb" (the
    time-embedding chain) or a _ForkOp (that branch only)."""

    def __init__(self, kind="all"):
        super().__init__("join(side stream)", None, (), ())
        self.kind = kind

    def launch(self, stream):
        raise RuntimeError("join marker is handled by Plan.run")


class _ForkOp(Op):
    """`branch` runs on the side stream, ordered after everything already on the main stream."""

    def __init__(self, branch):
        super().__init__("fork(side stream)", None, (), ())
        self.branch = list(branch)
        self.ev_fork = self.ev_done = None

    def launch(self, stream):
        raise RuntimeError("fork marker is handled by Plan.run")


class _DryFn:
    def __init__(self, name):
        self.name = name

    def __call__(self, *a):
        raise RuntimeError("dry plan cannot be launched")


class _DryLibT:
    def __getattr__(self, name):
        fn = _DryFn(name)
        setattr(self, name, fn)
        return fn


_DryLib = _DryLibT()
