"""Ordering checks between the launches of a plan: an access model of every entry point the plans launch and a
happens-before model of `Plan.run` (two streams, PDL-free stream order) around the runtime's copy-ins and
clone-outs, unrolled over two consecutive steps.

  * `accesses(op)`: the byte regions (field, address, rows, row_bytes, pitch, mode) one launch reads ("r"),
    writes ("w") or reads then writes ("rw"), from the semantics in include/sfb200.h, computed from the op's
    parameter struct / plain arguments and its TMA map geometry.  Inside one launch the model may
    over-approximate (a TMA map's whole tensor is read, a QKV scatter writes whole q / k rows); the model is
    checked against the kernels on the GPU (checked_call: plan_launches.py's replay and real feature plans);
    across columns it is exact, so column-disjoint accesses to one pitched buffer never overlap.
  * `virtual_addresses()`: while a dry plan is built, every meta storage gets its own 1 MiB-aligned virtual
    base, so that the pointers baked into the plan's launches tell buffers apart.
  * `analyse(plan)`: findings, each naming both ops, the buffer and the byte range:
      race        two overlapping accesses, at least one a write, neither ordered before the other;
      stale read  a read of bytes the step writes, with no writer of those bytes ordered before it (the op
                  would see the previous step's value), including a read-modify-write of state nothing reset;
      prefetched weight written  a write into the pre-tiled B operand of a GEMM, which loads it before its
                  programmatic-dependent-launch wait;
    and the declared cross-step state of ALLOWED_CROSS_STEP, which is reported separately and not a finding.

    python tests/plan_hazards.py [--plans NAME ...]
"""
import argparse
import bisect
import collections
import contextlib
import ctypes as C
import importlib
import sys
import time

import numpy as np
import torch

import plan_launches as pl
from sfast_b200 import _lib, ops
from sfast_b200.plan import _ForkOp, _JoinOp

PLAN_MODULES = ("sfast_b200.plan", "sfast_b200.controlnet_plan", "sfast_b200.svd_plan", "sfast_b200.vae_plan",
                "sfast_b200.taesd_plan", "sfast_b200.t2i_adapter_plan", "sfast_b200.clip_plan")
ESZ = 2            # every activation and weight the kernels touch is 16-bit (fp32 vectors are sized below)
VBASE_ALIGN = 1 << 20

# Cross-step state a step reads before it writes it, on purpose: (entry point, field) -> reason.
ALLOWED_CROSS_STEP = {
    ("sfb_group_norm_scale_shift", "sync_counter"):
        "per-image tickets of the statistics kernel: the last CTA of an image resets its ticket to zero, so every "
        "launch finds them zero (they are zero-initialised once, at allocation)",
}

# static inputs the runtime copies in before a step, and outputs it clones after it (runtime.py)
INPUTS = ("sample_in", "ehs_in", "t_in", "add_in", "time_ids_in", "ctrl_in", "intrablock_in", "image_embeds_in",
          "ip_scale_in", "cond_in", "scale_in", "z_in", "x_in", "ids_in", "pixels_in")
OUTPUTS = ("out", "down_out", "mid_out", "features_out", "last_hidden_state", "pooled", "text_embeds",
           "image_embeds")


class Access:
    """`rows` rows of `row_bytes` bytes, `pitch` bytes apart, from byte address `addr`."""
    __slots__ = ("field", "addr", "rows", "row_bytes", "pitch", "mode")

    def __init__(self, field, addr, rows, row_bytes, pitch, mode):
        rows, row_bytes, pitch = int(rows), int(row_bytes), int(pitch)
        if rows > 1 and row_bytes >= pitch:
            assert row_bytes == pitch, (field, rows, row_bytes, pitch)
            row_bytes, rows = rows * pitch, 1
        if rows == 1:
            pitch = row_bytes
        self.field, self.addr, self.rows, self.row_bytes, self.pitch, self.mode = \
            field, int(addr), rows, row_bytes, pitch, mode

    @property
    def lo(self):
        return self.addr

    @property
    def hi(self):
        return self.addr + (self.rows - 1) * self.pitch + self.row_bytes

    @property
    def reads(self):
        return "r" in self.mode

    @property
    def writes(self):
        return "w" in self.mode

    def __repr__(self):
        return f"Access({self.field}, {self.addr:#x}, {self.rows}x{self.row_bytes}/{self.pitch}, {self.mode})"


# =====================================================================================================
# byte-set arithmetic on strided regions
# =====================================================================================================
def _intervals(a, lo=None, hi=None):
    """Sorted disjoint [start, end) byte intervals of `a`, clipped to [lo, hi)."""
    lo = a.lo if lo is None else max(lo, a.lo)
    hi = a.hi if hi is None else min(hi, a.hi)
    if hi <= lo:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    r0 = max(0, (lo - a.addr - a.row_bytes) // a.pitch + 1)
    r1 = min(a.rows, (hi - a.addr - 1) // a.pitch + 1)
    s = a.addr + np.arange(r0, max(r0, r1), dtype=np.int64) * a.pitch
    e = s + a.row_bytes
    return np.maximum(s, lo), np.minimum(e, hi)


def _union(parts):
    s = np.concatenate([p[0] for p in parts]) if parts else np.zeros(0, np.int64)
    e = np.concatenate([p[1] for p in parts]) if parts else np.zeros(0, np.int64)
    keep = e > s
    s, e = s[keep], e[keep]
    if not len(s):
        return s, e
    o = np.argsort(s, kind="stable")
    s, e = s[o], e[o]
    em = np.maximum.accumulate(e)
    new = np.ones(len(s), bool)
    new[1:] = s[1:] > em[:-1]
    idx = np.flatnonzero(new)
    ends = np.append(idx[1:], len(s)) - 1
    return s[idx], em[ends]


def _covered(iv, x):
    s, e = iv
    if not len(s):
        return np.zeros(len(x), bool)
    i = np.searchsorted(s, x, side="right") - 1
    ok = i >= 0
    return ok & (e[np.maximum(i, 0)] > x)


def _segments(*ivs):
    pts = np.unique(np.concatenate([np.concatenate(iv) for iv in ivs]))
    if len(pts) < 2:
        return pts, []
    mids = pts[:-1]
    return pts, [_covered(iv, mids) for iv in ivs]


def overlap(a, b):
    """First overlapping byte range (lo, hi) of two regions, or None.  Exact for any pair of pitches."""
    lo, hi = max(a.lo, b.lo), min(a.hi, b.hi)
    if hi <= lo:
        return None
    if a.rows == 1 and b.rows == 1:
        return lo, hi
    ia, ib = _intervals(a, lo, hi), _intervals(b, lo, hi)
    pts, (ina, inb) = _segments(ia, ib)
    both = np.flatnonzero(ina & inb) if len(pts) >= 2 else []
    if not len(both):
        return None
    return int(pts[both[0]]), int(pts[both[0] + 1])


def contains(w, r):
    """Whether region `w` covers every byte of region `r` (cheap forms first)."""
    if r.lo < w.lo or r.hi > w.hi:
        return False
    if w.rows == 1:
        return True
    if r.rows == 1 or r.pitch == w.pitch:
        return (r.addr - w.addr) % w.pitch + r.row_bytes <= w.row_bytes
    return uncovered(r, [], [w]) is None


def uncovered(r, writers, cover):
    """First byte range of r that some region of `writers` writes and no region of `cover` covers (an empty
    `writers` list stands for all of r), or None."""
    ir = _intervals(r)
    iw = _union([_intervals(w, r.lo, r.hi) for w in writers]) if writers else ir
    ic = _union([_intervals(c, r.lo, r.hi) for c in cover])
    pts, (inr, inw, inc) = _segments(ir, iw, ic)
    if len(pts) < 2:
        return None
    bad = np.flatnonzero(inr & inw & ~inc)
    if not len(bad):
        return None
    return int(pts[bad[0]]), int(pts[bad[0] + 1])


# =====================================================================================================
# distinct addresses for dry plans
# =====================================================================================================
class AddressSpace:
    """Virtual bases of the meta storages seen while a plan was built (keeps the tensors alive, so a storage's
    identity is never reused)."""

    def __init__(self):
        self.next = VBASE_ALIGN
        self.base = {}          # storage key -> base
        self.spans = []         # sorted (base, nbytes, tensor)
        self.names = {}         # base -> name

    def ptr(self, t):
        st = t.untyped_storage()
        key = st._cdata
        b = self.base.get(key)
        if b is None:
            b = self.next
            n = max(st.nbytes(), 1)
            self.next += (n + 2 * VBASE_ALIGN - 1) // VBASE_ALIGN * VBASE_ALIGN
            self.base[key] = b
            self.spans.append((b, n, t))
        return b + t.storage_offset() * t.element_size()

    def find(self, addr):
        i = bisect.bisect_right(self.spans, addr, key=lambda s: s[0]) - 1
        if i >= 0 and addr < self.spans[i][0] + self.spans[i][1]:
            return self.spans[i][0]
        return None

    def name(self, base):
        return self.names.get(base, f"weight@{base:#x}")

    def name_plan_buffers(self, plan):
        """Plan names of the buffers: `name[shape]` for Plan.buf buffers, the attribute name for the others."""
        def put(t, name):
            if torch.is_tensor(t) and t.device.type == "meta":
                b = self.find(self.ptr(t))
                if b is not None:
                    self.names.setdefault(b, name)
        for (name, shape, _), t in plan._bufs.items():
            put(t, f"{name}[{'x'.join(str(s) for s in shape)}]")
        def unwrap(v):
            return v.buf if isinstance(v, ops.Act) else v.t if isinstance(v, ops.RowStats) else v
        for attr, v in vars(plan).items():
            if isinstance(v, (list, tuple)):
                for i, t in enumerate(v):
                    put(unwrap(t), f"{attr}[{i}]")
            else:
                put(unwrap(v), attr)


_MAPS = {}   # host address of a TensorMap built under recording_tensor_maps() -> the map


@contextlib.contextmanager
def recording_tensor_maps():
    """While plans are built or launches replayed on the GPU: every _lib.TensorMap records its geometry and base
    address the way a DryMap does (`geom`, `base`), so that accesses() reads a real op like a dry one, and the map
    is found by its host address (raw_keep)."""
    TM = _lib.TensorMap
    mm, nm = TM.__dict__["matrix"], TM.__dict__["nhwc"]

    def matrix(cls, base_ptr, rows, cols, pitch, box_rows):
        t = mm.__func__(cls, base_ptr, rows, cols, pitch, box_rows)
        t.geom, t.base = ("2d", rows, cols, pitch, box_rows), int(base_ptr or 0)
        _MAPS[t.ptr] = t
        return t

    def nhwc(cls, base_ptr, n, h, w, c, pitch, box_n, box_h, box_w, stride=1):
        t = nm.__func__(cls, base_ptr, n, h, w, c, pitch, box_n, box_h, box_w, stride)
        t.geom, t.base = ("nhwc", n, h, w, c, pitch, box_n, box_h, box_w, stride), int(base_ptr or 0)
        _MAPS[t.ptr] = t
        return t

    TM.matrix, TM.nhwc = classmethod(matrix), classmethod(nhwc)
    try:
        yield
    finally:
        TM.matrix, TM.nhwc = mm, nm


@contextlib.contextmanager
def virtual_addresses():
    """While a dry plan is built: every meta storage (t.untyped_storage()._cdata) gets its own 1 MiB-aligned
    virtual base and a view's address is that base plus storage_offset * itemsize.  Hooks ops._ptr and every
    module that imported it by name (RowStats and Mat pointers go through it), and records every DryMap's base
    address (plan_launches.recording_map_offsets).  Yields the AddressSpace."""
    for m in PLAN_MODULES:  # imported first: a module imported under the hook would keep it
        importlib.import_module(m)
    space = AddressSpace()
    orig = ops._ptr

    def _ptr(t):
        if isinstance(t, ops.RowStats):
            t = t.t
        if torch.is_tensor(t) and t.device.type == "meta":
            return space.ptr(t)
        return orig(t)

    mods = [m for n, m in list(sys.modules.items()) if n.startswith("sfast_b200") and getattr(m, "_ptr", None) is orig]
    for m in mods:
        m._ptr = _ptr
    try:
        with pl.recording_map_offsets():
            yield space
    finally:
        for m in mods:
            m._ptr = orig


# =====================================================================================================
# access model
# =====================================================================================================
def _fn_name(op):
    return getattr(op.fn, "name", None) or getattr(op.fn, "__name__", None)


def _p(v):
    return int(v or 0)


def _map_region(field, m, mode="r"):
    g = m.geom
    if g[0] == "2d":
        rows, cols, pitch = g[1], g[2], g[3]
        return Access(field, m.base, rows, cols * ESZ, pitch * ESZ, mode)
    n, h, w, c, pitch = g[1:6]
    return Access(field, m.base, n * h * w, c * ESZ, pitch * ESZ, mode)


def _gemm(p, keep):
    out = [_map_region("tmap_a", keep[1]), _map_region("tmap_b", keep[2])]
    M, N = p.M, p.N
    if p.splits > 1:
        out.append(Access("ws", p.ws, 1, p.splits * M * N * 4, 0, "w"))
    if not (p.splits > 1 and p.defer_finish):
        if p.epi == _lib.EPI_QKV:
            bh = M // p.seq * p.heads
            for which in range(p.which_base, p.which_base + N // (p.heads * p.head_dim)):
                if which == 0:
                    out.append(Access("q", p.q, bh, p.seq * p.q_pitch * ESZ, p.q_rows * p.q_pitch * ESZ, "w"))
                elif which == 1:
                    out.append(Access("k", p.k, bh, p.seq * p.q_pitch * ESZ, p.k_rows * p.q_pitch * ESZ, "w"))
                else:   # rows [0, head_dim) of every (batch, head) block: not the ones row, not the padding
                    out += [Access("vt", _p(p.vt) + d * p.vt_pitch * ESZ, bh, p.seq * ESZ,
                                   p.vt_rows * p.vt_pitch * ESZ, "w") for d in range(p.head_dim)]
        else:
            oesz = 4 if p.epi == _lib.EPI_STORE_F32 else ESZ
            width = p.geglu_n_out if p.epi == _lib.EPI_GEGLU else N
            out.append(Access("out", p.out, M, width * oesz, p.ldo * oesz, "w"))
            if p.rowstats_out:
                out.append(Access("rowstats_out", p.rowstats_out, M, ops.rowstats_slots(N) * 8,
                                  p.rowstats_out_slots * 8, "w"))
    if p.bias:
        out.append(Access("bias", p.bias, 1, N * 4, 0, "r"))
    if p.rowbias:
        out.append(Access("rowbias", p.rowbias, M // p.rows_per_img, N * 4, p.ld_rowbias * 4, "r"))
    if p.residual:
        out.append(Access("residual", p.residual, M, N * ESZ, p.ldr * ESZ, "r"))
    if p.ln_rowstats:
        out.append(Access("ln_rowstats", p.ln_rowstats, M, p.ln_slots * 8, p.ln_slots * 8, "r"))
        out.append(Access("ln_colsum", p.ln_colsum, 1, N * 4, 0, "r"))
    if p.gn_scale_shift:
        out.append(Access("gn_scale_shift", p.gn_scale_shift, 1, p.img_n * p.cin * 8, 0, "r"))
    return out


def _attn_out(p):
    return Access("out", p.out, p.batch * p.seq_q, p.heads * p.head_dim * ESZ, p.heads * p.head_dim * ESZ, "w")


def _gn(name, p, args):
    rows, c = p.n * p.hw, p.c
    out = []
    if name != "sfb_group_norm_apply":
        out.append(Access("stats", p.stats, 1, ops.gn_ws_floats(p.n, p.groups) * 4, 0, "w"))
    else:
        out.append(Access("stats", p.stats, 1, ops.gn_ws_floats(p.n, p.groups) * 4, 0, "r"))
    part_c = p.part_c if (name == "sfb_group_norm_fused" and p.part_ws) else 0
    if part_c:
        out.append(Access("x", p.x, rows, part_c * ESZ, p.ldx * ESZ, "w"))
        out.append(Access("part_ws", p.part_ws, 1, p.part_splits * rows * p.part_ld * 4, 0, "r"))
        if p.part_bias:
            out.append(Access("part_bias", p.part_bias, 1, part_c * 4, 0, "r"))
        if p.part_rowbias:
            out.append(Access("part_rowbias", p.part_rowbias, p.n, part_c * 4, p.part_ld_rowbias * 4, "r"))
        if p.part_residual:
            out.append(Access("part_residual", p.part_residual, rows, part_c * ESZ, p.part_ldr * ESZ, "r"))
    if part_c < c:
        out.append(Access("x", _p(p.x) + part_c * ESZ, rows, (c - part_c) * ESZ, p.ldx * ESZ, "r"))
    if name == "sfb_group_norm_stats":
        return out
    out += [Access("gamma", p.gamma, 1, c * 4, 0, "r"), Access("beta", p.beta, 1, c * 4, 0, "r")]
    if name == "sfb_group_norm_scale_shift":
        out.append(Access("sync_counter", p.sync_counter, 1, p.n * 4, 0, "rw"))
        out.append(Access("scale_shift", args[1], 1, p.n * c * 8, 0, "w"))
        return out
    out.append(Access("y", p.y, rows, c * ESZ, p.ldy * ESZ, "w"))
    if name == "sfb_group_norm_fused":
        out.append(Access("sync_counter", p.sync_counter, 1, 4, 0, "rw"))
    return out


def _conv_small(p):
    cin16 = (p.cin + 15) // 16 * 16
    ho, wo = (p.h - 1) // p.stride + 1, (p.w - 1) // p.stride + 1
    if p.x_nchw:
        x = Access("x", p.x, 1, p.n * p.cin * p.h * p.w * ESZ, 0, "r")
    else:
        x = Access("x", p.x, p.n * p.h * p.w, p.cin * ESZ, p.ldx * ESZ, "r")
    out = [x, Access("weight", p.weight, 1, p.cout * 9 * cin16 * ESZ, 0, "r"),
           Access("y", p.y, p.n * ho * wo, p.cout * ESZ, p.ldy * ESZ, "w")]
    if p.bias:
        out.append(Access("bias", p.bias, 1, p.cout * 4, 0, "r"))
    return out


def _row_op(name, p):
    rows, c = p.rows, p.c
    out = [Access("x", p.x, rows, c * ESZ, p.ldx * ESZ, "r"), Access("y", p.y, rows, c * ESZ, p.ldy * ESZ, "w")]
    if name == "sfb_row_broadcast_add":
        nvec = p.mod if p.mode == _lib.ROW_IDX_DIV_MOD else p.batch * p.frames
        out.append(Access("vec", p.vec, nvec, c * ESZ, p.ldv * ESZ, "r"))
    else:
        out.append(Access("x2", p.x2, rows, c * ESZ, p.ldx2 * ESZ, "r"))
        out.append(Access("mix_factor", p.mix_factor, 1, 4, 0, "r"))
    if p.rowstats_out:
        slots = p.rowstats_slots or 1
        out.append(Access("rowstats_out", p.rowstats_out, rows, 8, slots * 8, "w"))
    return out


def _plain(name, a):
    A = Access
    if name == "sfb_memset":
        return [A("p", a[0], 1, a[2], 0, "w")]
    if name == "sfb_row_softmax":
        x, y, rows, cols, ldx, ldy, f32 = a[:7]
        xs = 4 if f32 else ESZ
        return [A("x", x, rows, cols * xs, ldx * xs, "r"), A("y", y, rows, cols * ESZ, ldy * ESZ, "w")]
    if name == "sfb_conv_in":
        x, w, b, y, n, h, wd, cin, cout, ldy = a[:10]
        return [A("x", x, 1, n * cin * h * wd * ESZ, 0, "r"), A("w", w, 1, 9 * cin * cout * ESZ, 0, "r"),
                A("bias", b, 1, cout * 4, 0, "r"), A("y", y, n * h * wd, cout * ESZ, ldy * ESZ, "w")]
    if name == "sfb_conv_out":
        x, w, b, y, n, h, wd, cin, cout, ldx = a[:10]
        return [A("x", x, n * h * wd, cin * ESZ, ldx * ESZ, "r"), A("w", w, 1, cout * 9 * cin * ESZ, 0, "r"),
                A("bias", b, 1, cout * 4, 0, "r"), A("y", y, 1, n * cout * h * wd * ESZ, 0, "w")]
    if name == "sfb_conv_out_temporal":
        x, w, b, wt, bt, y, n, h, wd, cin, cout, ldx = a[:12]
        out = [A("x", x, n * h * wd, cin * ESZ, ldx * ESZ, "r"), A("w", w, 1, cout * 9 * cin * ESZ, 0, "r"),
               A("bias", b, 1, cout * 4, 0, "r"), A("wt", wt, 1, cout * 3 * cout * ESZ, 0, "r"),
               A("y", y, 1, n * cout * h * wd * ESZ, 0, "w")]
        if bt:
            out.append(A("bt", bt, 1, cout * 4, 0, "r"))
        return out
    if name == "sfb_im2col_in":
        x, y, n, h, wd, cin = a[:6]
        return [A("x", x, 1, n * cin * h * wd * ESZ, 0, "r"), A("a", y, 1, n * h * wd * 64 * ESZ, 0, "w")]
    if name == "sfb_upsample2x":
        x, y, n, h, w, c, ldx, ldy = a[:8]
        return [A("x", x, n * h * w, c * ESZ, ldx * ESZ, "r"), A("y", y, 4 * n * h * w, c * ESZ, ldy * ESZ, "w")]
    if name == "sfb_timestep_embed":
        t, batch, dim, _, _, out, ldo = a[:7]
        return [A("t", t, 1, batch * 4, 0, "r"), A("out", out, batch, dim * ESZ, ldo * ESZ, "w")]
    if name == "sfb_pointwise_nchw":
        x, w, b, y, n, hw, cin, cout = a[:8]
        return [A("x", x, 1, n * cin * hw * ESZ, 0, "r"), A("w", w, 1, cout * cin * ESZ, 0, "r"),
                A("bias", b, 1, cout * 4, 0, "r"), A("y", y, 1, n * cout * hw * ESZ, 0, "w")]
    if name == "sfb_embed_tokens":
        ids, tok, pos, out, rs, slots, batch, seq, dim, vocab, ld = a[:11]
        acc = [A("ids", ids, 1, batch * seq * 8, 0, "r"), A("tok_emb", tok, 1, vocab * dim * ESZ, 0, "r"),
               A("pos_emb", pos, 1, seq * dim * ESZ, 0, "r"), A("out", out, batch * seq, dim * ESZ, ld * ESZ, "w")]
        if rs:
            acc.append(A("rowstats", rs, batch * seq, 8, slots * 8, "w"))
        return acc
    if name == "sfb_clip_pool":
        ids, x, pooled, batch, seq, dim, ldx = a[:7]
        return [A("ids", ids, 1, batch * seq * 8, 0, "r"), A("x", x, batch * seq, dim * ESZ, ldx * ESZ, "r"),
                A("pooled", pooled, 1, batch * dim * ESZ, 0, "w")]
    if name == "sfb_patchify":
        x, y, batch, chans, h, w, patch, kpad = a[:8]
        rows = batch * (h // patch) * (w // patch)
        return [A("x", x, 1, batch * chans * h * w * ESZ, 0, "r"), A("a", y, 1, rows * kpad * ESZ, 0, "w")]
    if name == "sfb_copy2d":
        src, dst, rows, cols, lds, ldd = a[:6]
        return [A("src", src, rows, cols * ESZ, lds * ESZ, "r"), A("dst", dst, rows, cols * ESZ, ldd * ESZ, "w")]
    if name == "sfb_pixel_unshuffle":
        x, y, n, c, h, w, r, ldy = a[:8]
        return [A("x", x, 1, n * c * h * w * ESZ, 0, "r"),
                A("y", y, n * (h // r) * (w // r), c * r * r * ESZ, ldy * ESZ, "w")]
    if name == "sfb_avg_pool2x2":
        x, y, n, h, w, c, ldx, ldy = a[:8]
        return [A("x", x, n * h * w, c * ESZ, ldx * ESZ, "r"),
                A("y", y, n * (h // 2) * (w // 2), c * ESZ, ldy * ESZ, "w")]
    raise KeyError(name)


PLAIN_MODELLED = ("sfb_memset", "sfb_row_softmax", "sfb_conv_in", "sfb_conv_out", "sfb_conv_out_temporal",
                  "sfb_im2col_in", "sfb_upsample2x", "sfb_timestep_embed", "sfb_pointwise_nchw", "sfb_embed_tokens",
                  "sfb_clip_pool", "sfb_patchify", "sfb_copy2d", "sfb_pixel_unshuffle", "sfb_avg_pool2x2")
STRUCT_MODELLED = ("sfb_gemm", "sfb_attention", "sfb_attention_ip", "sfb_group_norm_fused", "sfb_group_norm_stats",
                   "sfb_group_norm_apply", "sfb_group_norm_scale_shift", "sfb_layer_norm", "sfb_small_linear",
                   "sfb_temporal_attention", "sfb_row_broadcast_add", "sfb_alpha_blend", "sfb_add_nchw_residuals",
                   "sfb_conv3x3_small", "sfb_conv3x3_small_ex", "sfb_conv3x3_c64", "sfb_nhwc_to_nchw_scaled")
MODELLED = frozenset(PLAIN_MODELLED + STRUCT_MODELLED)


def accesses(op):
    """[Access] of one launch, a dry op or one of a plan built on the GPU (its TMA maps were built under
    recording_tensor_maps()).  Raises KeyError for an entry point the model does not know."""
    return launch_accesses(_fn_name(op), op.args, op.keep)


def _struct(a):
    return getattr(a, "_obj", a)


def raw_keep(name, args):
    """The `keep` tuple accesses() reads, rebuilt from a launch's raw arguments: the parameter struct and the TMA
    maps its pointers name (looked up in the maps recording_tensor_maps() saw being built)."""
    p = _struct(args[0])
    m = lambda ptr: _MAPS[int(ptr)]  # noqa: E731
    if name == "sfb_gemm":
        return (p, m(p.tmap_a), m(p.tmap_b))
    if name == "sfb_attention":
        return (p, m(p.tmap_q), m(p.tmap_k), m(p.tmap_vt))
    if name == "sfb_attention_ip":
        b = p.base
        return (p, m(p.tmap_k_ip), m(p.tmap_vt_ip), None, None, None, m(b.tmap_q), m(b.tmap_k), m(b.tmap_vt))
    return (p,)


def launch_accesses(name, args, keep=None):
    """[Access] of one launch of entry point `name` with arguments `args` (without the stream); `keep`: the op's
    keep tuple (None: rebuilt from the arguments, raw_keep)."""
    if name in PLAIN_MODELLED:
        return [a for a in _plain(name, args) if a.addr and a.row_bytes]
    if name not in STRUCT_MODELLED:
        raise KeyError(name)
    if keep is None:
        keep = raw_keep(name, args)
    p = _struct(keep[0])
    if name == "sfb_gemm":
        out = _gemm(p, keep)
    elif name == "sfb_attention":
        out = [_map_region("tmap_q", keep[1]), _map_region("tmap_k", keep[2]), _map_region("tmap_vt", keep[3]),
               _attn_out(p)]
    elif name == "sfb_attention_ip":
        out = [_map_region("tmap_q", keep[6]), _map_region("tmap_k", keep[7]), _map_region("tmap_vt", keep[8]),
               _map_region("tmap_k_ip", keep[1]), _map_region("tmap_vt_ip", keep[2]),
               Access("ip_scale", p.ip_scale, 1, 4, 0, "r"), _attn_out(p.base)]
    elif name.startswith("sfb_group_norm"):
        out = _gn(name, p, args)
    elif name == "sfb_layer_norm":
        out = [Access("x", p.x, p.rows, p.c * ESZ, p.ldx * ESZ, "r"), Access("y", p.y, p.rows, p.c * ESZ, p.ldy * ESZ, "w"),
               Access("gamma", p.gamma, 1, p.c * 4, 0, "r"), Access("beta", p.beta, 1, p.c * 4, 0, "r")]
    elif name == "sfb_small_linear":
        out = [Access("x", p.x, p.batch, p.k * ESZ, p.ldx * ESZ, "r"), Access("w", p.w, 1, p.n * p.k * ESZ, 0, "r")]
        if p.bias:
            out.append(Access("bias", p.bias, 1, p.n * 4, 0, "r"))
        if p.add16:
            out.append(Access("add16", p.add16, 1, p.batch * p.n * ESZ, 0, "r"))
        if p.y16:
            out.append(Access("y16", p.y16, p.batch, p.n * ESZ, p.ldy * ESZ, "w"))
        if p.y32:
            out.append(Access("y32", p.y32, p.batch, p.n * 4, p.ldy * 4, "w"))
    elif name == "sfb_temporal_attention":
        rows, cm = p.batch * p.frames * p.seq, p.heads * p.head_dim
        out = [Access("qkv", p.qkv, rows, 3 * cm * ESZ, p.ld_qkv * ESZ, "r"),
               Access("out", p.out, rows, cm * ESZ, p.ld_out * ESZ, "w")]
    elif name in ("sfb_row_broadcast_add", "sfb_alpha_blend"):
        out = _row_op(name, p)
    elif name == "sfb_add_nchw_residuals":
        out = []
        for i in range(p.count):
            it = p.items[i]
            out.append(Access(f"items[{i}].src", it.src, 1, it.n * it.c * it.hw * ESZ, 0, "r"))
            out.append(Access(f"items[{i}].dst", it.dst, it.n * it.hw, it.c * ESZ, it.ld_dst * ESZ, "rw"))
    elif name == "sfb_nhwc_to_nchw_scaled":
        out = [Access("scale", p.scale, 1, p.count * 4, 0, "r")]
        for i in range(p.count):
            it = p.items[i]
            out.append(Access(f"items[{i}].src", it.src, it.n * it.hw, it.c * ESZ, it.ld_src * ESZ, "r"))
            out.append(Access(f"items[{i}].dst", it.dst, 1, it.n * it.c * it.hw * ESZ, 0, "w"))
    elif name == "sfb_conv3x3_small":
        out = _conv_small(p)
    elif name == "sfb_conv3x3_small_ex":
        out = _conv_small(p.base)
    elif name == "sfb_conv3x3_c64":
        ho, wo = ops.c64_out_hw(p.mode, p.h, p.w)
        out = [Access("x", p.x, p.n * p.h * p.w, 64 * ESZ, p.ldx * ESZ, "r"),
               Access("weight", p.weight, 1, 64 * 576 * ESZ, 0, "r"),
               Access("y", p.y, p.n * ho * wo, 64 * ESZ, p.ldy * ESZ, "w")]
        if p.bias:
            out.append(Access("bias", p.bias, 1, 64 * 4, 0, "r"))
        if p.residual:
            out.append(Access("residual", p.residual, p.n * ho * wo, 64 * ESZ, p.ldr * ESZ, "r"))
    return [a for a in out if a.addr and a.row_bytes]


# =====================================================================================================
# soundness of the model, on the GPU
# =====================================================================================================
class _Cai:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 3,
                                         "strides": None}


def _device_bytes(ptr, n):
    return torch.as_tensor(_Cai(ptr, n), device="cuda")


def _allocations():
    """Sorted (address, bytes) of every live block of torch's caching allocator."""
    out = []
    for seg in torch.cuda.memory_snapshot():
        a = seg["address"]
        for b in seg["blocks"]:
            if b["state"] == "active_allocated":
                out.append((b.get("address", a), b["size"]))
            a += b["size"]
    return sorted(out)


def _pointers(obj):
    """Device pointers of a parameter struct (nested structs and item arrays included; tensor-map fields are host
    addresses and left out)."""
    out = []
    for f, t in obj._fields_:
        v = getattr(obj, f)
        if t is C.c_void_p:
            if v and not f.startswith("tmap"):
                out.append(int(v))
        elif isinstance(v, C.Structure):
            out += _pointers(v)
        elif isinstance(v, C.Array) and len(v) and isinstance(v[0], C.Structure):
            for it in v:
                out += _pointers(it)
    return out


def _mask(acc, base, n, modes):
    """Bool mask over the n bytes at `base` of the accesses whose mode is in `modes`."""
    m = torch.zeros(n, dtype=torch.bool, device="cuda")
    for a in acc:
        if a.mode not in modes or a.hi <= base or a.lo >= base + n:
            continue
        r0 = max(0, -(-(base - a.addr) // a.pitch))
        r1 = min(a.rows, (base + n - a.addr - a.row_bytes) // a.pitch + 1)
        if r1 > r0:
            m.as_strided((r1 - r0, a.row_bytes), (a.pitch, 1), a.addr + r0 * a.pitch - base).fill_(True)
        for r in {r0 - 1, max(r0, r1)}:   # rows that cross the block's ends
            if 0 <= r < a.rows:
                s, e = max(a.addr + r * a.pitch, base), min(a.addr + r * a.pitch + a.row_bytes, base + n)
                if e > s:
                    m[s - base:e - base] = True
    return m


class Soundness:
    """Findings of checked launches: `violations` (messages), `writes` / `reads`: launches whose write / read
    model was checked."""

    def __init__(self, read_check):
        self.read_check, self.violations, self.writes, self.reads = read_check, [], 0, 0


P_FIRST, P_SECOND = 0xA5, 0x3C   # fill bytes outside the modelled read regions (never a plausible value pair)


def checked_call(sound, name, fn, args):
    """Launch `fn(*args)` (stream last) after checking the access model of this launch against the kernel, on every
    device buffer a pointer of the launch points into:
      writes: every byte outside the modelled read regions is set to P_FIRST, the launch runs, and every byte that
              changed must lie in a modelled write region;
      reads (sound.read_check): it runs again with those bytes set to P_SECOND instead; every byte it writes in
              either run must come out bit-identical.
    Then every buffer is restored and the launch runs as the caller meant it."""
    acc = launch_accesses(name, args[:-1])
    ptrs = [a.addr for a in acc]
    if name in STRUCT_MODELLED:
        ptrs += _pointers(_struct(args[0]))
    allocs = _allocations()
    starts = [a for a, _ in allocs]
    blocks = {}
    for p in ptrs:
        i = bisect.bisect_right(starts, p) - 1
        if i >= 0 and p < allocs[i][0] + allocs[i][1]:
            blocks[allocs[i][0]] = allocs[i][1]
    torch.cuda.synchronize()
    bufs = []
    for base, n in sorted(blocks.items()):
        t = _device_bytes(base, n)
        bufs.append((base, n, t, t.clone(), _mask(acc, base, n, ("r", "rw")), _mask(acc, base, n, ("w", "rw"))))

    def run(fill):
        for _, _, t, orig, rm, _ in bufs:
            t.copy_(torch.where(rm, orig, torch.full_like(orig, fill)))
        before = [t.clone() for _, _, t, _, _, _ in bufs]
        rc = fn(*args)
        torch.cuda.synchronize()
        return rc, before, [t.clone() for _, _, t, _, _, _ in bufs]

    try:
        rc, before, after = run(P_FIRST)
        if rc == 0:
            sound.writes += 1
            for (base, n, _, _, _, wm), b, a in zip(bufs, before, after):
                bad = ((a != b) & ~wm).nonzero()
                if len(bad):
                    sound.violations.append(
                        f"{name}: {len(bad)} bytes written outside the modelled write regions, first at +{int(bad[0])} "
                        f"of a {n}-byte buffer (pointers into it: "
                        f"{sorted({p - base for p in ptrs if base <= p < base + n})})")
            if sound.read_check:
                rc2, before2, after2 = run(P_SECOND)
                sound.reads += 1
                for (base, n, _, _, _, wm), b1, a1, b2, a2 in zip(bufs, before, after, before2, after2):
                    # the bytes the launch wrote in either run (a write region may over-approximate)
                    wrote = wm & ((a1 != b1) | (a2 != b2))
                    bad = ((a1 != a2) & wrote).nonzero()
                    if rc2 != 0 or len(bad):
                        sound.violations.append(
                            f"{name}: output depends on bytes outside the modelled read regions ({len(bad)} output "
                            f"bytes differ, first at +{int(bad[0]) if len(bad) else -1} of a {n}-byte buffer)")
    finally:
        for _, _, t, orig, _, _ in bufs:
            t.copy_(orig)
        torch.cuda.synchronize()
    return fn(*args)


@contextlib.contextmanager
def checking_launches(read_check):
    """Every modelled entry point called through _lib.lib() goes through checked_call; TMA maps are recorded.  Yields
    the Soundness."""
    sound = Soundness(read_check)
    real, orig = _lib.lib(), _lib.lib

    class Proxy:
        def __getattr__(self, n):
            f = getattr(real, n)
            if n not in MODELLED:
                return f
            return lambda *args: checked_call(sound, n, f, args)

    proxy = Proxy()
    _lib.lib = lambda: proxy
    try:
        with recording_tensor_maps():
            yield sound
    finally:
        _lib.lib = orig


# =====================================================================================================
# happens-before model of Plan.run and the runtime around it
# =====================================================================================================
MAIN, SIDE = 0, 1


class Event:
    __slots__ = ("step", "stream", "clock", "op", "label", "acc", "idx")

    def __init__(self, step, stream, clock, op, label, acc):
        self.step, self.stream, self.clock, self.op, self.label, self.acc = step, stream, tuple(clock), op, label, acc

    def __repr__(self):
        return self.label


def hb(a, b):
    """a happens before b (a is not b)."""
    return a is not b and a.clock[a.stream] <= b.clock[a.stream]


def _tensor_access(field, t, mode, cols=None):
    """Whole tensor (or its first `cols` columns of the last dimension) as one region."""
    addr = ops._ptr(t)
    if cols is None:
        return Access(field, addr, 1, t.numel() * t.element_size(), 0, mode)
    rows = t.numel() // t.shape[-1]
    return Access(field, addr, rows, cols * t.element_size(), t.shape[-1] * t.element_size(), mode)


def _io_tensors(plan, names):
    for n in names:
        v = getattr(plan, n, None)
        if v is None:
            continue
        if isinstance(v, (list, tuple)):
            for i, t in enumerate(v):
                yield f"{n}[{i}]", getattr(t, "buf", t)
        else:
            yield n, v
    if "out" in names and hasattr(plan, "hidden") and hasattr(plan, "hidden_states"):
        for i, h in enumerate(plan.hidden):
            yield f"hidden_states[{i}]", h.buf


def io_accesses(plan):
    """(copy-ins, clone-outs): [(label, Access)] of the runtime's host copies into the static inputs before a step
    and its clones of the outputs after it.  SDXL's add_in gets its text-embedding columns from the host; the
    step writes the time-id columns itself."""
    ins = []
    for n, t in _io_tensors(plan, INPUTS):
        cols = None
        if n == "add_in":
            spec = plan.spec
            cols = spec.add_in_dim - 6 * spec.addition_time_embed_dim
        ins.append((f"copy-in {n}", _tensor_access(n, t, "w", cols)))
    outs = [(f"clone-out {n}", _tensor_access(n, t, "r")) for n, t in _io_tensors(plan, OUTPUTS)]
    return ins, outs


def schedule(plan, steps=2):
    """Events (copy-ins, launches, clone-outs) of `steps` consecutive steps in the order Plan.run and the runtime
    enqueue them, with their vector clocks over (main, side)."""
    ins, outs = io_accesses(plan)
    clk = [[0, 0], [0, 0]]
    events = []

    def tick(step, s, op, label, acc):
        clk[s][s] += 1
        e = Event(step, s, clk[s], op, label, acc)
        e.idx = len(events)
        events.append(e)
        return e

    def join(dst, src):
        clk[dst] = [max(a, b) for a, b in zip(clk[dst], src)]

    def launch_label(step, s, i, op):
        return f"step{step}:{'side' if s else 'main'}#{i} {op.name} ({_fn_name(op)})"

    temb_last = getattr(plan, "_temb_last", None)
    for step in range(1, steps + 1):
        for label, a in ins:
            tick(step, MAIN, None, f"step{step}:{label}", [a])
        temb = None
        if plan.side_ops:
            join(SIDE, clk[MAIN])
            for i, op in enumerate(plan.side_ops):
                tick(step, SIDE, op, launch_label(step, SIDE, i, op), accesses(op))
                if op is temb_last:
                    temb = list(clk[SIDE])
        done = {}
        for i, op in enumerate(plan.ops):
            if isinstance(op, _JoinOp):
                if op.kind == "temb":
                    join(MAIN, temb)
                elif op.kind == "all":
                    join(MAIN, clk[SIDE])
                else:
                    join(MAIN, done[id(op.kind)])
            elif isinstance(op, _ForkOp):
                join(SIDE, clk[MAIN])
                for j, o in enumerate(op.branch):
                    tick(step, SIDE, o, launch_label(step, SIDE, f"{i}.{j}", o), accesses(o))
                done[id(op)] = list(clk[SIDE])
            else:
                tick(step, MAIN, op, launch_label(step, MAIN, i, op), accesses(op))
        for label, a in outs:
            tick(step, MAIN, None, f"step{step}:{label}", [a])
    return events


class Finding:
    __slots__ = ("kind", "a", "b", "buffer", "lo", "hi", "fields")

    def __init__(self, kind, a, b, buffer, lo, hi, fields):
        self.kind, self.a, self.b, self.buffer, self.lo, self.hi, self.fields = kind, a, b, buffer, lo, hi, fields

    def __str__(self):
        return (f"{self.kind}: {self.a} [{self.fields[0]}] / {self.b} [{self.fields[1]}] on {self.buffer} "
                f"bytes [{self.lo}, {self.hi})")

    __repr__ = __str__


class Report:
    def __init__(self, findings, declared, pairs, events):
        self.findings, self.declared, self.pairs, self.events = findings, declared, pairs, events

    def __str__(self):
        return "\n".join(str(f) for f in self.findings) or "no findings"


def analyse(plan, space, steps=2):
    """Report(findings, declared cross-step state, examined unordered (side, main) pairs, events) of a plan built
    under `space` = virtual_addresses()."""
    space.name_plan_buffers(plan)
    events = schedule(plan, steps)
    buf_of = {}

    def buffer(addr):
        b = buf_of.get(addr)
        if b is None:
            b = buf_of[addr] = space.find(addr)
            if b is None:
                raise AssertionError(f"address {addr:#x} is in no buffer of the plan")
        return b

    def rng(b, lo, hi):
        return space.name(b), lo - b, hi - b

    findings, seen = [], set()

    def add(kind, e1, a1, e2, a2, lo, hi):
        b = buffer(a1.addr)
        key = (kind, e1.op if e1.op is not None else e1.label, e2.op if e2.op is not None else e2.label, b,
               e1.step == e2.step)
        if key in seen:
            return
        seen.add(key)
        name, l, h = rng(b, lo, hi)
        findings.append(Finding(kind, e1.label, e2.label, name, l, h, (a1.field, a2.field)))

    # ---- races: every side event against the main events unordered with it (a contiguous range of main)
    mains = [e for e in events if e.stream == MAIN]
    main_side = [e.clock[SIDE] for e in mains]
    by_buf = collections.defaultdict(list)     # per main event index: accesses grouped by buffer
    for e in mains:
        g = collections.defaultdict(list)
        for a in e.acc:
            g[buffer(a.addr)].append(a)
        by_buf[e.idx] = g
    pairs = 0
    for s in events:
        if s.stream != SIDE:
            continue
        lo = s.clock[MAIN]                                   # mains[:lo] happen before s
        hi = bisect.bisect_left(main_side, s.clock[SIDE])    # mains[hi:] happen after s
        pairs += max(0, hi - lo)
        for m in mains[lo:hi]:
            g = by_buf[m.idx]
            for a in s.acc:
                for b in g.get(buffer(a.addr), ()):
                    if not (a.writes or b.writes):
                        continue
                    ov = overlap(a, b)
                    if ov is not None:
                        add("race", s, a, m, b, *ov)
    # ---- stale reads, over the first step
    step1 = [e for e in events if e.step == 1]
    writers = collections.defaultdict(list)
    for e in step1:
        for a in e.acc:
            if a.writes:
                writers[buffer(a.addr)].append((e, a))
    declared = []
    for e in step1:
        for r in e.acc:
            if not r.reads:
                continue
            ws = [(w, a) for w, a in writers.get(buffer(r.addr), ()) if a.hi > r.lo and a.lo < r.hi]
            # writers ordered after the read, and the op's own writes (a read-modify-write); a writer concurrent
            # with the read is a race, reported above
            later = [(w, a) for w, a in ws if (w is e or hb(e, w)) and overlap(a, r) is not None]
            if not later:
                continue
            cover = [a for w, a in ws if hb(w, e)]
            if any(contains(c, r) for c in cover):
                continue
            bad = uncovered(r, [a for _, a in later], cover)
            if bad is None:
                continue
            hit = [(w, a) for w, a in later if overlap(a, Access("", bad[0], 1, bad[1] - bad[0], 0, "r"))]
            w, a = next(((w, a) for w, a in hit if w is not e), hit[0])
            if e.op is not None and (_fn_name(e.op), r.field) in ALLOWED_CROSS_STEP:
                b = buffer(r.addr)
                declared.append((e.label, r.field, space.name(b)))
                continue
            add("stale read", e, r, w, a, *bad)
    # ---- programmatic dependent launch: a GEMM with a pre-tiled B operand loads its first weight tiles before it
    # waits for its predecessor, so nothing in a step may write bytes such a GEMM reads through tmap_b
    tiled_b = collections.defaultdict(list)
    for e in step1:
        if e.op is not None and _fn_name(e.op) == "sfb_gemm" and not e.op.keep[0].b_plain:
            tiled_b[buffer(e.acc[1].addr)].append((e, e.acc[1]))
    for e in step1:
        for a in e.acc:
            for g, b in tiled_b.get(buffer(a.addr), ()) if a.writes else ():
                ov = overlap(a, b)
                if ov is not None:
                    add("prefetched weight written", e, a, g, b, *ov)
    return Report(findings, declared, pairs, events)


def build(builder):
    """(plan, AddressSpace) of a dry plan built under virtual addresses."""
    with virtual_addresses() as space:
        plan = builder()
    return plan, space


def check_plan(builder):
    plan, space = build(builder)
    with virtual_addresses_of(space):
        return plan, analyse(plan, space)


@contextlib.contextmanager
def virtual_addresses_of(space):
    """Re-enter an AddressSpace (the io regions of a built plan are resolved through ops._ptr)."""
    orig = ops._ptr

    def _ptr(t):
        if torch.is_tensor(t) and t.device.type == "meta":
            return space.ptr(t)
        return orig(t)
    ops._ptr = _ptr
    try:
        yield space
    finally:
        ops._ptr = orig


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--plans", nargs="*", help="plan names of plan_launches.PLANS (default: all)")
    args = ap.parse_args(argv)
    bad = 0
    for name, _, builder in pl.PLANS:
        if args.plans and name not in args.plans:
            continue
        t0 = time.time()
        _, rep = check_plan(builder)
        print(f"{name}: {len(rep.findings)} findings, {rep.pairs} unordered pairs, {len(rep.events)} events, "
              f"{time.time() - t0:.1f} s")
        for f in rep.findings:
            print("  " + str(f))
        bad += len(rep.findings)
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
