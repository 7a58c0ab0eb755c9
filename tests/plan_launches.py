"""Replay every distinct kernel launch of the shipped launch plans against a float64 reference.

The kernel checks in ``kernel_checks.py`` run each kernel at shapes picked by hand; the plans launch
other mixes of geometry, pitch, split-K factor, tile box, epilogue and optional operands.  This module
builds the plans dry (no GPU needed), collapses their launches to distinct keys and, on a GPU, runs
each key once on fresh seeded inputs:

  * every pointer is re-pointed at a fresh tensor laid out like the plan's buffer (full pitch, the
    same leading offset), every TMA map is rebuilt from the plan's map geometry;
  * weights are random logical weights packed by the project's own packers (Mat tiling,
    pack_conv3x3 / pack_upconv / pack_geglu, the LayerNorm-gamma fold); the reference uses the
    logical weights, or the packed values where packing itself rounds (up-conv phase sums,
    gamma-folded weights and their column sums);
  * the reference is float64, written from the semantics in include/sfb200.h;
  * every output buffer is filled with a sentinel bit pattern first: pitch gaps, leading offsets and
    a guard band of GUARD_ROWS rows past the last row must come back bit-for-bit unchanged;
  * optionally (`soundness`), every launch also checks the access model of plan_hazards.py: bytes written
    outside its write regions, and outputs that depend on bytes outside its read regions, fail the key.

    python tests/plan_launches.py [--plans NAME ...] [--all] [--json out.json] [--list] [--soundness]

prints one JSON line per key (key id, entry point, plans that emit it, error, tolerance, pass) and a
summary of the largest error per entry point.  Without --all only the default subset
(`select_subset`) is replayed.
"""
import argparse
import collections
import contextlib
import ctypes as C
import hashlib
import json
import math
import os
import sys
import time

import torch
import torch.nn.functional as F

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
for _p in (_HERE, _ROOT, os.path.join(_ROOT, "stable-fast_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

# fp32 conv / matmul references must not silently run in TF32
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

from kernel_checks import rel_err  # noqa: E402
from sfast_b200 import _lib, ops  # noqa: E402
from sfast_b200._lib import TensorMap  # noqa: E402

DEV = "cuda"
GUARD_ROWS = 128          # one M tile of guard band past the last row of every output
SENT16, SENT32 = 0x7E11, 0x7FC0DEAD
STATS_SENT = -1.0e4       # rowstats sentinel: a sum of squares is never negative
DTYPES = {_lib.SFB_F16: torch.float16, _lib.SFB_BF16: torch.bfloat16}

# entry points called with plain arguments: argument names, "*" marks a pointer
PLAIN = {
    "sfb_row_softmax": ("x*", "y*", "rows", "cols", "ldx", "ldy", "x_is_f32", "dtype"),
    "sfb_conv_in": ("x*", "w*", "bias*", "y*", "n", "h", "wd", "cin", "cout", "ldy", "dtype"),
    "sfb_conv_out": ("x*", "w*", "bias*", "y*", "n", "h", "wd", "cin", "cout", "ldx", "dtype"),
    "sfb_im2col_in": ("x*", "a*", "n", "h", "wd", "cin"),
    "sfb_upsample2x": ("x*", "y*", "n", "h", "w", "c", "ldx", "ldy"),
    "sfb_timestep_embed": ("t*", "batch", "dim", "flip", "shift", "out*", "ldo", "dtype"),
    "sfb_pointwise_nchw": ("x*", "w*", "bias*", "y*", "n", "hw", "cin", "cout", "dtype"),
    "sfb_embed_tokens": ("ids*", "tok*", "pos*", "out*", "rowstats*", "slots", "batch", "seq", "dim", "vocab",
                         "ld_out", "dtype"),
    "sfb_clip_pool": ("ids*", "x*", "pooled*", "batch", "seq", "dim", "ld_x", "eos_id"),
    "sfb_patchify": ("x*", "a*", "batch", "chans", "h", "w", "patch", "kpad"),
    "sfb_copy2d": ("src*", "dst*", "rows", "cols", "ld_src", "ld_dst"),
}
STRUCT = ("sfb_gemm", "sfb_attention", "sfb_group_norm_fused", "sfb_group_norm_stats", "sfb_group_norm_apply",
          "sfb_group_norm_scale_shift", "sfb_layer_norm", "sfb_small_linear", "sfb_temporal_attention",
          "sfb_row_broadcast_add", "sfb_alpha_blend", "sfb_add_nchw_residuals")
SKIP = {"sfb_memset": "zeroes the plans' statistics arenas: a cudaMemsetAsync wrapper with no kernel of its own"}


# =====================================================================================================
# plan inventory
# =====================================================================================================
def _sd(shapes, dt):
    return {k: torch.empty(tuple(v), dtype=dt, device="meta") for k, v in shapes.items()}


def _unet(cfg_name, batch, h, w, dt=torch.float16, **kw):
    from oracle import unet_oracle as uo
    from sfast_b200.plan import PackedWeights, UNetPlan
    from sfast_b200.unet_spec import param_shapes, spec_from_config
    spec = spec_from_config(getattr(uo, cfg_name)())
    return UNetPlan(PackedWeights(spec, _sd(param_shapes(spec), dt), dt, "meta", dry=True), batch, h, w, **kw)


def _svd(tiny, videos, h, w):
    from oracle import svd_oracle as so
    from sfast_b200.plan import PackedWeights
    from sfast_b200.svd_plan import SVDPlan
    from sfast_b200.unet_spec import param_shapes, spec_from_config
    spec = spec_from_config(so.svd_tiny_config() if tiny else so.svd_xt_config())
    return SVDPlan(PackedWeights(spec, _sd(param_shapes(spec), torch.float16), torch.float16, "meta", dry=True),
                   videos, h, w)


def _vae_decode(batch, h, w, dt=torch.float16):
    from oracle import vae_oracle as vo
    from sfast_b200.plan import PackedWeights
    from sfast_b200.vae_plan import VAEDecodePlan, vae_decoder_param_shapes, vae_spec_from_config
    spec = vae_spec_from_config(vo.sd_vae_config())
    return VAEDecodePlan(PackedWeights(spec, _sd(vae_decoder_param_shapes(spec), dt), dt, "meta", dry=True),
                         batch, h, w)


def _vae_encode(batch, h, w):
    from oracle import vae_oracle as vo
    from sfast_b200.plan import PackedWeights
    from sfast_b200.vae_plan import VAEEncodePlan, vae_encoder_param_shapes, vae_encoder_spec_from_config
    spec = vae_encoder_spec_from_config(vo.sd_vae_config())
    dt = torch.float16
    return VAEEncodePlan(PackedWeights(spec, _sd(vae_encoder_param_shapes(spec), dt), dt, "meta", dry=True),
                         batch, h, w)


_CLIP_L = dict(vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12,
               num_attention_heads=12, max_position_embeddings=77, hidden_act="quick_gelu", eos_token_id=2,
               projection_dim=768, layer_norm_eps=1e-5)
_CLIP_BIGG = dict(_CLIP_L, hidden_size=1280, intermediate_size=5120, num_hidden_layers=32, num_attention_heads=20,
                  hidden_act="gelu", projection_dim=1280, eos_token_id=49407)
_VIT_H = dict(hidden_size=1280, intermediate_size=5120, num_hidden_layers=32, num_attention_heads=16,
              image_size=224, patch_size=14, hidden_act="gelu", projection_dim=1024)


def _clip_text(cfg, batch, with_projection=False):
    from sfast_b200 import clip_plan as cp
    from sfast_b200.plan import PackedWeights
    spec = cp.clip_text_spec_from_config(cfg, with_projection=with_projection)
    pw = PackedWeights(spec, _sd(cp.clip_text_param_shapes(spec), torch.float16), torch.float16, "meta", dry=True)
    return cp.ClipTextPlan(pw, batch, 77)


def _clip_vision(batch):
    from sfast_b200 import clip_plan as cp
    from sfast_b200.plan import PackedWeights
    spec = cp.clip_vision_spec_from_config(_VIT_H, with_projection=True)
    pw = PackedWeights(spec, _sd(cp.clip_vision_param_shapes(spec), torch.float16), torch.float16, "meta", dry=True)
    return cp.ClipVisionPlan(pw, batch)


# (plan name, family, builder); families in the order the GPU tests replay them
PLANS = [
    *[(f"sd15_{b}x64x64", "unet", (lambda b=b: _unet("sd15_config", b, 64, 64))) for b in (1, 2, 8, 16)],
    ("sd15_1x96x96", "unet", lambda: _unet("sd15_config", 1, 96, 96)),
    ("sd15_1x64x96", "unet", lambda: _unet("sd15_config", 1, 64, 96)),
    *[(f"sd15_{b}x128x128", "unet", (lambda b=b: _unet("sd15_config", b, 128, 128))) for b in (1, 8)],
    ("sd15_controlnet_2x64x64", "unet", lambda: _unet("sd15_config", 2, 64, 64, controlnet=True)),
    ("sdxl_2x128x128", "unet", lambda: _unet("sdxl_config", 2, 128, 128)),
    ("sdxl_1x104x152", "unet", lambda: _unet("sdxl_config", 1, 104, 152)),
    ("sdxl_8x128x128", "unet", lambda: _unet("sdxl_config", 8, 128, 128)),
    ("sdxl_bf16_2x128x128", "unet", lambda: _unet("sdxl_config", 2, 128, 128, dt=torch.bfloat16)),
    ("tiny_2x32x32", "unet", lambda: _unet("tiny_config", 2, 32, 32)),
    ("tiny_1x24x40", "unet", lambda: _unet("tiny_config", 1, 24, 40)),
    ("svd_tiny_2x16x16", "svd", lambda: _svd(True, 2, 16, 16)),
    ("svd_tiny_3x24x40", "svd", lambda: _svd(True, 3, 24, 40)),
    ("svd_xt_2x72x128", "svd", lambda: _svd(False, 2, 72, 128)),
    ("svd_xt_1x40x64", "svd", lambda: _svd(False, 1, 40, 64)),
    *[(f"vae_decode_{h}x{w}", "vae_decode", (lambda h=h, w=w: _vae_decode(1, h, w)))
      for h, w in ((64, 64), (96, 96), (128, 128), (72, 128))],
    ("vae_decode_bf16_128x128", "vae_decode", lambda: _vae_decode(1, 128, 128, dt=torch.bfloat16)),
    *[(f"vae_encode_{h}x{w}", "vae_encode", (lambda h=h, w=w: _vae_encode(1, h, w)))
      for h, w in ((512, 512), (768, 768), (1024, 1024), (576, 1024))],
    *[(f"clip_text_l_{b}", "clip", (lambda b=b: _clip_text(_CLIP_L, b))) for b in (1, 2)],
    *[(f"clip_text_bigg_{b}", "clip", (lambda b=b: _clip_text(_CLIP_BIGG, b, True))) for b in (1, 2)],
    ("clip_vision_h14_1", "clip", lambda: _clip_vision(1)),
]
FAMILIES = ("unet", "svd", "vae_decode", "vae_encode", "clip")


@contextlib.contextmanager
def recording_map_offsets():
    """While building dry plans: every DryMap also records the byte offset of its base pointer inside its
    buffer (dry buffers are meta tensors at address 0, so the pointer IS the offset)."""
    mm, nm = ops.matrix_map, ops.nhwc_map

    def matrix_map(ptr, rows, cols, pitch, box_rows, dry=False):
        m = mm(ptr, rows, cols, pitch, box_rows, dry)
        if dry:
            m.base = int(ptr or 0)
        return m

    def nhwc_map(ptr, n, h, w, c, pitch, box_n, box_h, box_w, stride=1, dry=False):
        m = nm(ptr, n, h, w, c, pitch, box_n, box_h, box_w, stride, dry)
        if dry:
            m.base = int(ptr or 0)
        return m

    ops.matrix_map, ops.nhwc_map = matrix_map, nhwc_map
    try:
        yield
    finally:
        ops.matrix_map, ops.nhwc_map = mm, nm


def build_plan(name):
    builder = dict((n, b) for n, _, b in PLANS)[name]
    with recording_map_offsets():
        return builder()


# =====================================================================================================
# launch keys
# =====================================================================================================
def _nonnull(op):
    """{pointer field: 1 / 0} of a struct launch.  A dry buffer sits at address 0, so a pointer's value
    cannot tell NULL from "offset 0 of a buffer": the op's `keep` tuple says what was passed."""
    name, k = op.fn.name, op.keep
    p = k[0]
    if name == "sfb_gemm":
        _, _, _, out, bias, rowbias, residual, _, qkv, _, rs, ln = k
        q = qkv or {}
        return dict(tmap_a=1, tmap_b=1, out=int(out is not None), bias=int(bias is not None),
                    rowbias=int(rowbias is not None), residual=int(residual is not None), ws=int(p.splits > 1),
                    q=int(q.get("q") is not None), k=int(q.get("k") is not None), vt=int(q.get("vt") is not None),
                    rowstats_out=int(rs is not None), ln_rowstats=int(ln is not None), ln_colsum=int(ln is not None),
                    gn_scale_shift=int(p.a_mode == _lib.A_CONV3X3_GN))
    if name == "sfb_group_norm_scale_shift":
        return dict(x=1, y=0, gamma=1, beta=1, stats=1, sync_counter=1, part_ws=0, part_bias=0, part_rowbias=0,
                    part_residual=0)
    if name.startswith("sfb_group_norm"):
        part = k[7] if len(k) > 7 else None
        return dict(x=1, y=1, gamma=1, beta=1, stats=1, sync_counter=int(k[6] is not None),
                    part_ws=int(part is not None), part_bias=int(bool(part) and part.get("bias") is not None),
                    part_rowbias=int(bool(part) and "rowbias" in part),
                    part_residual=int(bool(part) and "residual" in part))
    if name == "sfb_small_linear":
        return dict(x=1, w=1, bias=int(k[3] is not None), add16=int(k[4] is not None), y16=int(k[5] is not None),
                    y32=int(k[6] is not None))
    if name in ("sfb_row_broadcast_add", "sfb_alpha_blend"):
        return dict(x=1, y=1, vec=int(k[3] is not None), x2=int(k[4] is not None), mix_factor=int(k[5] is not None),
                    rowstats_out=int(k[6] is not None))
    # attention, temporal attention, layer norm: every pointer is an operand
    return {f: 1 for f, t in p._fields_ if t is C.c_void_p}


def _plain(v):
    return None if v is None else (round(v, 9) if isinstance(v, float) else int(v))


def launch_key(op):
    """Hashable key of one launch: entry point, every non-pointer field, one null bit and the byte offset
    inside its buffer per pointer, and the geometry (plus base offset) of every TMA map."""
    name = op.fn.name
    if name in PLAIN or name in SKIP:
        return (name,) + tuple(_plain(a) for a in op.args)
    p = op.keep[0]
    if name == "sfb_add_nchw_residuals":
        return (name, p.count, p.dtype,
                tuple((it.n, it.c, it.hw, it.ld_dst, int(it.dst or 0)) for it in p.items[:p.count]))
    nn = _nonnull(op)
    fields = []
    for f, t in p._fields_:
        v = getattr(p, f)
        if t is C.c_void_p:
            fields.append((f, nn[f], int(v or 0) if nn[f] else 0))
        else:
            fields.append((f, _plain(v)))
    maps = tuple((m.geom, getattr(m, "base", 0)) for m in op.keep if isinstance(m, ops.DryMap))
    extra = ()
    if name == "sfb_group_norm_scale_shift":
        extra = (("scale_shift", int(op.args[1] or 0)),)
    return (name, tuple(fields), maps) + extra


def key_id(key):
    return hashlib.sha1(repr(key).encode()).hexdigest()[:12]


def launches(plan):
    """(entry point, key, op) of every launch of a plan, in schedule order."""
    for op in plan.all_ops():
        if op.fn is None:
            continue
        yield op.fn.name, launch_key(op), op


def check_coverage(names):
    """Entry points that appear in a plan but have no replay and no SKIP entry."""
    return sorted(n for n in set(names) if n not in SKIP and n not in PLAIN and n not in STRUCT)


def collect(plan_names=None):
    """{key: dict(op=first op with that key, plans=[plan names], family=first family)} over the plans, and
    the set of entry-point names seen."""
    out, names = collections.OrderedDict(), set()
    fam_of = {n: f for n, f, _ in PLANS}
    for pname in plan_names or [n for n, _, _ in PLANS]:
        plan = build_plan(pname)
        for name, key, op in launches(plan):
            names.add(name)
            if name in SKIP:
                continue
            ent = out.get(key)
            if ent is None:
                out[key] = dict(op=op, plans=[pname], family=fam_of[pname], name=name)
            elif pname not in ent["plans"]:
                ent["plans"].append(pname)
    return out, names


def launch_class(key):
    """The (entry point, A mode, epilogue, flag set, null pattern, dtype) class of a key: what the default
    subset must cover."""
    name = key[0]
    if name == "sfb_gemm":
        g = {kv[0]: kv for kv in key[1]}
        flags = tuple(int(bool(g[f][-1])) for f in ("defer_finish", "b_plain", "cta_pair", "persistent"))
        flags += (min(g["splits"][-1], 2), g["act"][-1], int(g["ldo"][-1] > g["N"][-1]),
                  int(g["conv_stride"][-1] == 2), g["gn_silu"][-1])
        nulls = tuple(v[1] for v in key[1] if len(v) == 3)
        return (name, g["a_mode"][-1], g["epi"][-1], flags, nulls, g["dtype"][-1])
    if name in PLAIN:
        return (name, len(key))
    if name == "sfb_add_nchw_residuals":
        return (name,)
    g = {kv[0]: kv for kv in key[1]}
    flags = tuple((f, v[-1]) for f, v in g.items() if f in ("causal", "kv_tile", "silu", "part_splits", "mode",
                                                               "act_in", "act_out", "dtype"))
    nulls = tuple(v[1] for v in key[1] if len(v) == 3)
    return (name, flags, nulls)


def launch_work(key, op):
    return max(int(op.flops or 0), int(op.bytes or 0), 1)


def select_subset(entries):
    """Default subset: for every launch class, its largest and its smallest key; plus every key of the
    largest shape of each family (by its plan's total work)."""
    by_class = collections.defaultdict(list)
    for key, ent in entries.items():
        by_class[launch_class(key)].append(key)
    keep = set()
    for keys in by_class.values():
        keys.sort(key=lambda k: launch_work(k, entries[k]["op"]))
        keep.add(keys[0])
        keep.add(keys[-1])
    return [k for k in entries if k in keep]


# =====================================================================================================
# replay helpers
# =====================================================================================================
def _clone(struct):
    c = type(struct)()
    C.memmove(C.byref(c), C.byref(struct), C.sizeof(struct))
    return c


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _randn(n, dt, scale=1.0):
    return (torch.randn(n, device=DEV, dtype=torch.float32) * scale).to(dt)


def sentinel_fill(t):
    if t.element_size() == 2:
        t.view(torch.int16).fill_(SENT16)
    elif t.element_size() == 4:
        t.view(torch.int32).fill_(SENT32)
    else:
        raise TypeError(t.dtype)


def _bits(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


class Canvas:
    """An output buffer: `off` elements of leading offset, `rows` declared rows of pitch `ld`, GUARD_ROWS guard
    rows, all filled with the sentinel.  `arm()` snapshots it before the launch; `take(view)` returns the
    declared output region and restores it from the snapshot, and `intact()` then says whether anything
    outside the declared outputs changed."""

    def __init__(self, dt, off, rows, ld, guard=GUARD_ROWS, device=DEV):
        self.t = torch.empty(off + (rows + guard) * ld, dtype=dt, device=device)
        sentinel_fill(self.t)
        self.off, self.ld, self.before = off, ld, None

    @property
    def ptr(self):
        return self.t.data_ptr() + self.off * self.t.element_size()

    def region(self, rows, cols, off=0, ld=None, dt=None):
        """[rows, cols] view at pitch `ld` (default: the canvas pitch) starting `off` elements past the
        canvas offset; `dt`: the view's element type (16-bit data written into an fp32 buffer)."""
        t = self.t if dt is None else self.t.view(dt)
        ratio = self.t.element_size() // t.element_size()
        return t.as_strided((rows, cols), (ld or self.ld * ratio, 1), self.off * ratio + off)

    def arm(self):
        self.before = self.t.clone()

    def take(self, view):
        got = view.clone()
        src = self.before if view.dtype == self.t.dtype else self.before.view(view.dtype)
        view.copy_(src.as_strided(view.size(), view.stride(), view.storage_offset()))
        return got

    def intact(self):
        return torch.equal(_bits(self.t), _bits(self.before))


def _off(ptr, esz):
    """Element offset of a dry pointer (a byte offset from address 0; ctypes reads a zero pointer as None)."""
    return int(ptr or 0) // esz


def _nhwc_view(flat, off, n, h, w, c, pitch):
    return flat.as_strided((n, h, w, c), (h * w * pitch, w * pitch, pitch, 1), off)


def _mat_view(flat, off, rows, cols, pitch):
    return flat.as_strided((rows, cols), (pitch, 1), off)


class Result:
    """Components (name, err, tol) of one replay; passes when every err <= tol."""

    def __init__(self):
        self.parts = []

    def add(self, what, err, tol):
        err = float(err)
        if err != err:
            err = float("inf")
        self.parts.append((what, err, tol))

    def canary(self, *canvases):
        ok = all(c.intact() for c in canvases)
        self.parts.append(("canary", 0.0 if ok else float("inf"), 0.0))

    @property
    def ok(self):
        return all(e <= t for _, e, t in self.parts)

    def main(self):
        """(err, tol) of the first numerical component (what the summary reports)."""
        for w, e, t in self.parts:
            if w != "canary":
                return e, t
        return 0.0, 0.0


# ---- tolerances: one table, keyed by (kernel class, dtype); fp16 from kernel_checks.CHECKS, bf16 likewise
TOL = {
    "gemm": (2e-3, 1e-2), "conv": (2e-3, 1e-2), "upconv": (3e-3, 2e-2), "conv_gn": (4e-3, 3e-2),
    "ln_fold": (5e-3, 2e-2), "geglu": (2e-2, 2e-2), "gemm_f32": (1e-5, 1e-5), "rowstats": (2e-3, 1e-2),
    "attention": (5e-3, 2e-2), "temporal": (5e-3, 2e-2), "group_norm": (1e-2, 4e-2), "layer_norm": (1e-2, 4e-2),
    "softmax": (2e-3, 1e-2), "small_linear": (2e-3, 1e-2), "timestep": (2e-3, 1e-2), "conv_edge": (2e-3, 1e-2),
    "pointwise": (2e-3, 1e-2), "row_ops": (2e-3, 1e-2), "add_nchw": (2e-3, 1e-2), "exact": (0.0, 0.0),
}


def tol(kind, dt):
    return TOL[kind][0 if dt == torch.float16 else 1]


def gemm_kind(p):
    """Tolerance class of an sfb_gemm launch (A mode, epilogue, LayerNorm fold)."""
    if p.epi == _lib.EPI_GEGLU:
        return "geglu"
    if p.epi == _lib.EPI_STORE_F32:
        return "gemm_f32"
    if p.a_mode == _lib.A_UPCONV2X:
        return "upconv"
    if p.a_mode == _lib.A_CONV3X3_GN:
        return "conv_gn"
    if p.ln_dim > 0:
        return "ln_fold"
    if p.a_mode in (_lib.A_CONV3X3, _lib.A_DOWNCONV3X3, _lib.A_CONV3X1):
        return "conv"
    return "gemm"


# =====================================================================================================
# float64 references (semantics of include/sfb200.h; none calls the code under test)
# =====================================================================================================
def ref_conv3x3(x, w, stride=1):
    """x NHWC [n, h, w, cin] fp64, w [cout, cin, 3, 3] -> NHWC, zero padding 1."""
    return F.conv2d(x.permute(0, 3, 1, 2), w, stride=stride, padding=1).permute(0, 2, 3, 1)


def ref_downconv3x3(x, w):
    """diffusers Downsample2D(padding=0): one zero row / column AFTER the image, 3x3 stride-2 conv."""
    return F.conv2d(F.pad(x.permute(0, 3, 1, 2), (0, 1, 0, 1)), w, stride=2).permute(0, 2, 3, 1)


def ref_upconv_phases(x, packed, cout):
    """Nearest-2x upsample + 3x3 conv from the PACKED 4-phase weights ([4 * Np, 4 * cin], K order (ty, tx, c)):
    output pixel (2y + py, 2x + px) = sum over taps (ty, tx) of W[phase][ty, tx] . x[y + py - 1 + ty, x + px - 1 + tx]."""
    n, h, w, cin = x.shape
    npad = packed.shape[0] // 4
    xp = F.pad(x.permute(0, 3, 1, 2), (1, 1, 1, 1))
    out = x.new_zeros(n, cout, 2 * h, 2 * w)
    for py in range(2):
        for px in range(2):
            ph = 2 * py + px
            wk = packed[ph * npad:ph * npad + cout].reshape(cout, 2, 2, cin).permute(0, 3, 1, 2)
            out[:, :, py::2, px::2] = F.conv2d(xp[:, :, py:py + h + 1, px:px + w + 1], wk)
    return out.permute(0, 2, 3, 1)


def ref_conv3x1(x, w):
    """x [videos, frames, pixels, cin], w [cout, cin, 3]: Conv3d (3, 1, 1), padding (1, 0, 0) over frames."""
    y = F.conv3d(x.permute(0, 3, 1, 2).unsqueeze(-1), w[..., None, None], padding=(1, 0, 0))
    return y.squeeze(-1).permute(0, 2, 3, 1)


def ref_conv3x3_gn(x, w, scale_shift, silu):
    """conv2d(act(x * scale + shift)) with the zero padding applied AFTER the affine."""
    y = x * scale_shift[:, None, None, :, 0] + scale_shift[:, None, None, :, 1]
    if silu:
        y = F.silu(y)
    return ref_conv3x3(y, w)


def ref_layer_norm_rows(a, eps):
    mean = a.mean(-1, keepdim=True)
    var = a.var(-1, unbiased=False, keepdim=True)
    return (a - mean) / torch.sqrt(var + eps)


def ref_geglu(y, n_out):
    """Tile-interleaved GEGLU: physical columns [160 j, 160 j + 80) value, [160 j + 80, 160 j + 160) gate of
    output columns [80 j, 80 j + 80)."""
    M, Np = y.shape
    t = y.view(M, Np // ops.BN, 2, ops.BN // 2)
    return (t[:, :, 0] * F.gelu(t[:, :, 1])).reshape(M, Np // 2)[:, :n_out]


def ref_qkv_scatter(y, batch, seq, heads, head_dim, which_base):
    """[M, n_which * heads * head_dim] -> {which: tensor} with Q / K as [batch * heads, seq, head_dim] and V^T as
    [batch * heads, head_dim, seq] (column n -> which = n / (heads * head_dim) + which_base)."""
    t = y.view(batch, seq, -1, heads, head_dim)
    out = {}
    for i in range(t.shape[2]):
        which = i + which_base
        part = t[:, :, i].permute(0, 2, 1, 3).reshape(batch * heads, seq, head_dim)
        out[which] = part.transpose(1, 2) if which == 2 else part
    return out


def ref_attention(q, k, v, scale, causal, chunk_bytes=1 << 31):
    """q [bh, sq, d], k / v [bh, skv, d] fp64 -> [bh, sq, d]: softmax(q k^T * scale) v, chunked over queries."""
    bh, sq, _ = q.shape
    skv = k.shape[1]
    out = torch.empty_like(q)
    rows = max(1, min(sq, chunk_bytes // max(1, bh * skv * 8)))
    for b0 in range(0, bh, max(1, bh if rows < sq else bh)):
        for r0 in range(0, sq, rows):
            s = torch.matmul(q[:, r0:r0 + rows], k.transpose(1, 2)) * scale
            if causal:
                qi = torch.arange(r0, min(sq, r0 + rows), device=q.device)[:, None]
                s = s.masked_fill(torch.arange(skv, device=q.device)[None] > qi, float("-inf"))
            out[:, r0:r0 + rows] = torch.matmul(torch.softmax(s, -1), v)
            del s
    return out


def ref_group_norm(x, groups, gamma, beta, eps, silu):
    """x [n, hw, c] fp64 -> group_norm over (hw, c / groups) per image."""
    n, hw, c = x.shape
    g = x.view(n, hw, groups, c // groups)
    mean = g.mean(dim=(1, 3), keepdim=True)
    var = g.var(dim=(1, 3), unbiased=False, keepdim=True)
    y = ((g - mean) / torch.sqrt(var + eps)).view(n, hw, c) * gamma + beta
    return F.silu(y) if silu else y


def ref_group_stats(x, groups, eps):
    n, hw, c = x.shape
    g = x.view(n, hw, groups, c // groups)
    mean = g.mean(dim=(1, 3))
    var = g.var(dim=(1, 3), unbiased=False)
    return mean, 1.0 / torch.sqrt(var + eps)


def ref_timestep_embed(t, dim, flip, shift):
    half = dim // 2
    ex = -math.log(10000.0) * torch.arange(half, device=t.device, dtype=torch.float64) / (half - shift)
    e = t[:, None] * torch.exp(ex)[None]
    s, c = torch.sin(e), torch.cos(e)
    return torch.cat([c, s] if flip else [s, c], -1)


def split_slots(sums, slots):
    """[M, 2] row statistics split at random across `slots` slots (the first k of them; the rest zero): a
    consumer must add every slot."""
    M = sums.shape[0]
    out = torch.zeros(M, slots, 2, dtype=torch.float64, device=sums.device)
    if slots == 1:
        out[:, 0] = sums
        return out
    k = torch.randint(1, slots + 1, (M,), device=sums.device)
    w = torch.rand(M, slots, device=sums.device, dtype=torch.float64)
    w = w * (torch.arange(slots, device=sums.device)[None] < k[:, None])
    w = w / w.sum(1, keepdim=True)
    return out + w[:, :, None] * sums[:, None, :]


def check_rowstats(res, what, stats, stored, n_cols, dt):
    """`stats` [M, slots, 2] after a producer wrote it over the STATS_SENT fill: slots at or past
    rowstats_slots(n_cols) untouched, and the written ones (sum, sum of squares) adding up to the stored
    rows' statistics."""
    owned = ops.rowstats_slots(n_cols)
    beyond = stats[:, owned:]
    res.add(what + ".unowned_slots", 0.0 if bool((beyond == STATS_SENT).all()) else float("inf"), 0.0)
    s = stats[:, :owned].double()
    written = s[..., 1] != STATS_SENT
    res.add(what + ".rows_written", 0.0 if bool(written.any(1).all()) else float("inf"), 0.0)
    tot = (s * written[..., None]).sum(1)
    o = stored.double()
    res.add(what + ".sum", rel_err(tot[:, 0], o.sum(1)), tol("rowstats", dt))
    res.add(what + ".sumsq", rel_err(tot[:, 1], (o * o).sum(1)), tol("rowstats", dt))


# =====================================================================================================
# replays
# =====================================================================================================
def _gemm_weights(p, dt, ln):
    """Logical weights of a GEMM launch, packed by the project's packers.  Returns (packed [rows, K] for Mat,
    reference weight, bias fp32 or None, ln colsum or None)."""
    N, K = p.N, p.K
    s = 1.0 / math.sqrt(K)
    bias = torch.randn(N, device=DEV)
    if p.a_mode == _lib.A_UPCONV2X:
        cin = p.cin
        w3 = _randn(N * cin * 9, dt, 1 / math.sqrt(9 * cin)).view(N, cin, 3, 3)
        packed = ops.pack_upconv(w3, dt)
        return packed, packed.double(), bias, None
    if p.a_mode in (_lib.A_CONV3X3, _lib.A_DOWNCONV3X3, _lib.A_CONV3X3_GN):
        cin = p.cin
        w3 = _randn(N * cin * 9, dt, 1 / math.sqrt(9 * cin)).view(N, cin, 3, 3)
        return ops.pack_conv3x3(w3, dt), w3.double(), bias, None
    if p.a_mode == _lib.A_CONV3X1:
        cin = p.cin
        wt = _randn(N * cin * 3, dt, 1 / math.sqrt(3 * cin)).view(N, cin, 3)
        return wt.permute(0, 2, 1).reshape(N, 3 * cin).contiguous(), wt.double(), bias, None
    if p.epi == _lib.EPI_GEGLU:
        inner = p.geglu_n_out
        w = _randn(2 * inner * K, dt, s).view(2 * inner, K)
        b = torch.randn(2 * inner, device=DEV) * 0.1
        if ln:
            gamma, beta = 1.0 + 0.5 * torch.randn(K, device=DEV), 0.3 * torch.randn(K, device=DEV)
            wp, bias2, colsum = ops.fold_layer_norm(w, b, gamma, beta, dt)
            wt, bp, _, cs = ops.pack_geglu(wp, bias2, dt, extra=colsum)
            return wt, wt.double(), bp, cs
        wt, bp, _ = ops.pack_geglu(w, b, dt)
        return wt, wt.double(), bp, None
    w = _randn(N * K, dt, s).view(N, K)
    if ln:
        gamma, beta = 1.0 + 0.5 * torch.randn(K, device=DEV), 0.3 * torch.randn(K, device=DEV)
        wp, bias2, colsum = ops.fold_layer_norm(w, bias * 0.1, gamma, beta, dt)
        return wp.contiguous(), wp.double(), bias2, colsum
    return w, w.double(), bias, None


def replay_gemm(op, peaked=False):
    p0 = op.keep[0]
    p = _clone(p0)
    nn = _nonnull(op)
    am, bm = op.keep[1], op.keep[2]
    dt = DTYPES[p.dtype]
    esz = 2
    M, N, K = p.M, p.N, p.K
    res = Result()
    hold = []
    # ---- A operand
    ga, offa = am.geom, am.base // esz
    if ga[0] == "2d":
        rows, cols, pitch, box = ga[1:]
        abuf = _randn(offa + rows * pitch, dt)
        A = _mat_view(abuf, offa, rows, cols, pitch)
        amap = TensorMap.matrix(abuf.data_ptr() + offa * esz, rows, cols, pitch, box)
    else:
        n, h, w, c, pitch, bn, bh, bw, stride = ga[1:]
        abuf = _randn(offa + n * h * w * pitch, dt)
        A = _nhwc_view(abuf, offa, n, h, w, c, pitch)
        amap = TensorMap.nhwc(abuf.data_ptr() + offa * esz, n, h, w, c, pitch, bn, bh, bw, stride)
    p.tmap_a = amap.ptr
    hold += [abuf, amap]
    ln = bool(nn["ln_rowstats"])
    # ---- B operand
    gb = bm.geom
    if p.b_plain:
        rows, cols, pitch, box = gb[1:]
        offb = bm.base // esz
        bbuf = _randn(offb + rows * pitch, dt, 1 / math.sqrt(K))
        Wref = _mat_view(bbuf, offb, rows, cols, pitch).double()
        bmap = TensorMap.matrix(bbuf.data_ptr() + offb * esz, rows, cols, pitch, box)
        bias, colsum = torch.randn(N, device=DEV), None
        hold += [bbuf, bmap]
    else:
        packed, Wref, bias, colsum = _gemm_weights(p, dt, ln)
        mat = ops.Mat(packed)
        if (mat._rows, ops.BK) != (gb[1], gb[2]):
            raise AssertionError(f"packed weight rows {mat._rows} != plan map rows {gb[1]}")
        bmap = mat.map_for(ops.BN // gb[4])
        hold += [mat, bmap]
    p.tmap_b = bmap.ptr
    if nn["bias"]:
        bias = bias.contiguous()
        p.bias = bias.data_ptr()
    else:
        bias = None
        p.bias = None
    # ---- core product, fp64
    A64 = A.double()
    if p.a_mode == _lib.A_MATRIX:
        a2 = A64
        if ln:
            a2 = ref_layer_norm_rows(A64, p.ln_eps)
        acc = a2 @ Wref.t()
    elif p.a_mode == _lib.A_CONV3X3:
        acc = ref_conv3x3(A64, Wref, p.conv_stride).reshape(M, N)
    elif p.a_mode == _lib.A_DOWNCONV3X3:
        acc = ref_downconv3x3(A64, Wref).reshape(M, N)
    elif p.a_mode == _lib.A_UPCONV2X:
        acc = ref_upconv_phases(A64, Wref, N).reshape(M, N)
    elif p.a_mode == _lib.A_CONV3X1:
        acc = ref_conv3x1(A64, Wref).reshape(M, N)
    elif p.a_mode == _lib.A_CONV3X3_GN:
        ss = torch.stack([1.0 + 0.5 * torch.randn(p.img_n, p.cin, device=DEV),
                          0.5 + torch.randn(p.img_n, p.cin, device=DEV)], -1).contiguous()
        p.gn_scale_shift = ss.data_ptr()
        hold.append(ss)
        acc = ref_conv3x3_gn(A64, Wref, ss.double(), bool(p.gn_silu)).reshape(M, N)
    else:
        raise NotImplementedError(f"A mode {p.a_mode}")
    del A64
    # ---- LayerNorm fold: row statistics of the raw A, split across the slots
    if ln:
        a = A.double()
        sums = torch.stack([a.sum(1), (a * a).sum(1)], -1)
        st = split_slots(sums, p.ln_slots).float().contiguous()
        cs = colsum.float().contiguous()
        p.ln_rowstats, p.ln_colsum = st.data_ptr(), cs.data_ptr()
        hold += [st, cs]
        del a
    # ---- split-K workspace
    ws = None
    if p.splits > 1:
        ws = torch.full((p.splits * M * N,), float("nan"), device=DEV)
        p.ws = ws.data_ptr()
    # ---- epilogue operands
    if bias is not None:
        acc = acc + bias.double()
    rb = None
    if nn["rowbias"]:
        offr = _off(p0.rowbias, 4)
        n_img = M // p.rows_per_img
        rbuf = torch.randn(offr + n_img * p.ld_rowbias, device=DEV)
        p.rowbias = rbuf.data_ptr() + offr * 4
        rb = _mat_view(rbuf, offr, n_img, N, p.ld_rowbias).double()
        hold.append(rbuf)
    resid = None
    if nn["residual"]:
        offq = _off(p0.residual, esz)
        qbuf = _randn(offq + M * p.ldr, dt)
        p.residual = qbuf.data_ptr() + offq * esz
        resid = _mat_view(qbuf, offq, M, N, p.ldr).double()
        hold.append(qbuf)
    kind = gemm_kind(p)
    tl = tol(kind, dt)
    canvases = []
    # ---- outputs
    out = None
    if nn["out"]:
        oesz = 4 if p.epi == _lib.EPI_STORE_F32 else esz
        out = Canvas(torch.float32 if oesz == 4 else dt, _off(p0.out, oesz), M, p.ldo)
        p.out = out.ptr
        canvases.append(out)
    qkvc = {}
    if p.epi == _lib.EPI_QKV:
        bq = M // p.seq
        bh = bq * p.heads
        for f, rws, pitch in (("q", p.q_rows, p.q_pitch), ("k", p.k_rows, p.q_pitch), ("vt", p.vt_rows, p.vt_pitch)):
            cv = Canvas(dt, 0, bh * rws, pitch)
            setattr(p, f, cv.ptr)
            qkvc[f] = cv
            canvases.append(cv)
        qkvc["vt"].region(bh * p.vt_rows, p.vt_pitch).view(bh, p.vt_rows, p.vt_pitch)[:, p.head_dim].fill_(1.0)
    rso = None
    if nn["rowstats_out"]:
        rso = torch.full((M + GUARD_ROWS, p.rowstats_out_slots, 2), STATS_SENT, device=DEV)
        p.rowstats_out = rso.data_ptr()
    for cv in canvases:
        cv.arm()
    # ---- launch
    _lib.check(_lib.lib().sfb_gemm(C.byref(p), _stream()), "sfb_gemm")
    torch.cuda.synchronize()
    # ---- compare
    if p.defer_finish:
        part = ws.view(p.splits, M, N).double().sum(0)
        res.add("partials", rel_err(part, acc - (bias.double() if bias is not None else 0)), tl)
        res.canary(*canvases)
        return res
    if p.epi == _lib.EPI_STORE or p.epi == _lib.EPI_STORE_F32:
        y = acc
        if rb is not None:
            y = y + rb.repeat_interleave(p.rows_per_img, 0)
        if p.act == _lib.ACT_QUICK_GELU:
            y = y * torch.sigmoid(1.702 * y)
        elif p.act == _lib.ACT_GELU:
            y = F.gelu(y)
        if resid is not None:
            y = y + resid
        got = out.take(out.region(M, N))
        res.add("out", rel_err(got, y), tl)
        if rso is not None:
            check_rowstats(res, "rowstats_out", rso[:M], got, N, dt)
            res.add("rowstats_guard", 0.0 if bool((rso[M:] == STATS_SENT).all()) else float("inf"), 0.0)
    elif p.epi == _lib.EPI_GEGLU:
        y = ref_geglu(acc, p.geglu_n_out)
        got = out.take(out.region(M, p.geglu_n_out))
        res.add("out", rel_err(got, y), tl)
    elif p.epi == _lib.EPI_QKV:
        bq = M // p.seq
        bh = bq * p.heads
        D, S = p.head_dim, p.seq
        parts = ref_qkv_scatter(acc, bq, S, p.heads, D, p.which_base)
        for which, f in ((0, "q"), (1, "k"), (2, "vt")):
            if which not in parts:
                continue
            cv = qkvc[f]
            if f == "vt":
                full = cv.region(bh * p.vt_rows, p.vt_pitch).view(bh, p.vt_rows, p.vt_pitch)[:, :D, :S]
            else:
                rws = p.q_rows if f == "q" else p.k_rows
                full = cv.region(bh * rws, p.q_pitch).view(bh, rws, p.q_pitch)[:, :S, :D]
            got = cv.take(full)
            res.add(f, rel_err(got, parts[which]), tl)
    res.canary(*canvases)
    return res


def replay_attention(op, peaked=False):
    p = _clone(op.keep[0])
    dt = DTYPES[p.dtype]
    tq, tk, tv = op.keep[1], op.keep[2], op.keep[3]
    B, H, D = p.batch, p.heads, p.head_dim
    bh = B * H
    sq, skv = p.seq_q, p.seq_kv
    q_pitch, vt_pitch = tq.geom[2], tv.geom[2]
    res = Result()
    qf = torch.zeros(bh, p.q_rows, q_pitch, device=DEV, dtype=dt)
    kf = torch.zeros(bh, p.k_rows, q_pitch, device=DEV, dtype=dt)
    vf = torch.zeros(bh, p.vt_rows, vt_pitch, device=DEV, dtype=dt)
    qf[:, :sq, :D] = _randn(bh * sq * D, dt, 8.0 if peaked else 1.0).view(bh, sq, D)
    kf[:, :skv, :D] = _randn(bh * skv * D, dt).view(bh, skv, D)
    vf[:, :D, :skv] = _randn(bh * D * skv, dt).view(bh, D, skv)
    vf[:, D, :] = 1.0
    maps = [TensorMap.matrix(t.data_ptr(), *g.geom[1:]) for t, g in ((qf, tq), (kf, tk), (vf, tv))]
    p.tmap_q, p.tmap_k, p.tmap_vt = (m.ptr for m in maps)
    out = Canvas(dt, _off(p.out, 2), B * sq, H * D)
    p.out = out.ptr
    out.arm()
    _lib.check(_lib.lib().sfb_attention(C.byref(p), _stream()), "sfb_attention")
    torch.cuda.synchronize()
    got = out.take(out.region(B * sq, H * D))
    ref = ref_attention(qf[:, :sq, :D].double(), kf[:, :skv, :D].double(), vf[:, :D, :skv].double().transpose(1, 2),
                        float(p.scale), bool(p.causal))
    ref = ref.view(B, H, sq, D).permute(0, 2, 1, 3).reshape(B * sq, H * D)
    res.add("out", rel_err(got, ref), tol("attention", dt))
    res.canary(out)
    return res


def _gn_input(n, hw, c, ldx, off, dt):
    x = Canvas(dt, off, n * hw, ldx)
    v = x.region(n * hw, c)
    v.copy_((torch.randn(n * hw, c, device=DEV) + 0.5 * torch.randn(c, device=DEV)).to(dt))
    return x


def replay_group_norm(op, peaked=False):
    name = op.fn.name
    p0 = op.keep[0]
    p = _clone(p0)
    nn = _nonnull(op)
    dt = DTYPES[p.dtype]
    n, hw, c, G = p.n, p.hw, p.c, p.groups
    res = Result()
    lib = _lib.lib()
    x = _gn_input(n, hw, c, p.ldx, _off(p0.x, 2), dt)
    p.x = x.ptr
    gamma, beta = torch.randn(c, device=DEV), torch.randn(c, device=DEV)
    p.gamma, p.beta = gamma.data_ptr(), beta.data_ptr()
    stats = torch.full((ops.gn_ws_floats(n, G),), float("nan"), device=DEV)
    p.stats = stats.data_ptr()
    sync = torch.zeros(max(n, 4), device=DEV, dtype=torch.int32)
    p.sync_counter = sync.data_ptr() if nn["sync_counter"] else None
    canv = [x]
    if name == "sfb_group_norm_scale_shift":
        ab = Canvas(torch.float32, 0, n * c, 2)
        x.arm()
        ab.arm()
        _lib.check(lib.sfb_group_norm_scale_shift(C.byref(p), ab.ptr, _stream()), name)
        torch.cuda.synchronize()
        xin = x.region(n * hw, c).double().view(n, hw, c)
        mean, rstd = ref_group_stats(xin, G, p.eps)
        sc = gamma.double().view(1, G, -1) * rstd[:, :, None]
        sh = beta.double()[None] - (mean[:, :, None] * sc).reshape(n, c)
        got = ab.take(ab.region(n * c, 2)).view(n, c, 2)
        res.add("scale", rel_err(got[..., 0], sc.reshape(n, c)), tol("group_norm", dt))
        res.add("shift", rel_err(got[..., 1], sh), tol("group_norm", dt))
        res.add("tickets_reset", 0.0 if int(sync.abs().sum()) == 0 else float("inf"), 0.0)
        res.canary(x, ab)
        return res
    y = Canvas(dt, _off(p0.y, 2), n * hw, p.ldy)
    p.y = y.ptr
    canv.append(y)
    finished = None
    if nn["part_ws"]:
        S_, pc, pld = p.part_splits, p.part_c, p.part_ld
        ws = torch.randn(S_ * n * hw * pld, device=DEV) / math.sqrt(S_)
        p.part_ws = ws.data_ptr()
        fin = ws.view(S_, n * hw, pld)[:, :, :pc].double().sum(0)
        keep = [ws]
        if nn["part_bias"]:
            pb = torch.randn(pc, device=DEV)
            p.part_bias = pb.data_ptr()
            fin = fin + pb.double()
            keep.append(pb)
        if nn["part_rowbias"]:
            offr = _off(p0.part_rowbias, 4)
            rbuf = torch.randn(offr + n * p.part_ld_rowbias, device=DEV)
            p.part_rowbias = rbuf.data_ptr() + offr * 4
            fin = fin + _mat_view(rbuf, offr, n, pc, p.part_ld_rowbias).double().repeat_interleave(hw, 0)
            keep.append(rbuf)
        if nn["part_residual"]:
            offq = _off(p0.part_residual, 2)
            qbuf = _randn(offq + n * hw * p.part_ldr, dt)
            p.part_residual = qbuf.data_ptr() + offq * 2
            fin = fin + _mat_view(qbuf, offq, n * hw, pc, p.part_ldr).double()
            keep.append(qbuf)
        finished = fin
        sentinel_fill(x.region(n * hw, pc))   # these channels do not exist yet: the kernel writes them
    for cv in canv:
        cv.arm()
    if name == "sfb_group_norm_fused":
        _lib.check(lib.sfb_group_norm_fused(C.byref(p), _stream()), name)
    else:  # the stats -> apply pair the plan emits, over the same parameters
        _lib.check(lib.sfb_group_norm_stats(C.byref(p), _stream()), "sfb_group_norm_stats")
        _lib.check(lib.sfb_group_norm_apply(C.byref(p), _stream()), "sfb_group_norm_apply")
    torch.cuda.synchronize()
    xin = x.region(n * hw, c).double()
    if finished is not None:
        got_x = x.take(x.region(n * hw, p.part_c))
        res.add("finished_x", rel_err(got_x, finished), tol("gemm", dt))
        xin = torch.cat([got_x.double(), xin[:, p.part_c:]], 1)
    ref = ref_group_norm(xin.view(n, hw, c), G, gamma.double(), beta.double(), p.eps, bool(p.silu))
    got = y.take(y.region(n * hw, c))
    res.add("y", rel_err(got, ref.view(n * hw, c)), tol("group_norm", dt))
    res.canary(*canv)
    return res


def replay_layer_norm(op, peaked=False):
    p = _clone(op.keep[0])
    dt = DTYPES[p.dtype]
    res = Result()
    x = torch.randn(p.rows, p.ldx, device=DEV).to(dt)
    x[:, :p.c] += (0.5 * torch.randn(p.c, device=DEV)).to(dt)
    y = Canvas(dt, 0, p.rows, p.ldy)
    gamma, beta = torch.randn(p.c, device=DEV), torch.randn(p.c, device=DEV)
    p.x, p.y, p.gamma, p.beta = x.data_ptr(), y.ptr, gamma.data_ptr(), beta.data_ptr()
    y.arm()
    _lib.check(_lib.lib().sfb_layer_norm(C.byref(p), _stream()), "sfb_layer_norm")
    torch.cuda.synchronize()
    ref = ref_layer_norm_rows(x[:, :p.c].double(), p.eps) * gamma.double() + beta.double()
    res.add("y", rel_err(y.take(y.region(p.rows, p.c)), ref), tol("layer_norm", dt))
    res.canary(y)
    return res


def replay_small_linear(op, peaked=False):
    p = _clone(op.keep[0])
    nn = _nonnull(op)
    dt = DTYPES[p.dtype]
    res = Result()
    x = _randn(p.batch * p.ldx, dt).view(p.batch, p.ldx)
    w = _randn(p.n * p.k, dt, 1 / math.sqrt(p.k)).view(p.n, p.k)
    p.x, p.w = x.data_ptr(), w.data_ptr()
    xin = x[:, :p.k].double()
    if p.act_in:
        xin = F.silu(xin)
    ref = xin @ w.double().t()
    keep = []
    if nn["bias"]:
        b = torch.randn(p.n, device=DEV)
        p.bias = b.data_ptr()
        ref = ref + b.double()
        keep.append(b)
    if nn["add16"]:
        a16 = _randn(p.batch * p.n, dt).view(p.batch, p.n)
        p.add16 = a16.data_ptr()
        ref = ref + a16.double()
        keep.append(a16)
    if p.act_out:
        ref = F.silu(ref)
    outs = []
    if nn["y16"]:
        y16 = Canvas(dt, 0, p.batch, p.ldy)
        p.y16 = y16.ptr
        outs.append(("y16", y16))
    if nn["y32"]:
        y32 = Canvas(torch.float32, 0, p.batch, p.ldy)
        p.y32 = y32.ptr
        outs.append(("y32", y32))
    for _, cv in outs:
        cv.arm()
    _lib.check(_lib.lib().sfb_small_linear(C.byref(p), _stream()), "sfb_small_linear")
    torch.cuda.synchronize()
    for f, cv in outs:
        res.add(f, rel_err(cv.take(cv.region(p.batch, p.n)), ref), tol("small_linear", dt))
    res.canary(*[cv for _, cv in outs])
    return res


def replay_temporal(op, peaked=False):
    p = _clone(op.keep[0])
    dt = DTYPES[p.dtype]
    res = Result()
    B, Fr, S, H, D = p.batch, p.frames, p.seq, p.heads, p.head_dim
    rows, Cm = B * Fr * S, H * D
    qkv = _randn(rows * p.ld_qkv, dt).view(rows, p.ld_qkv)
    out = Canvas(dt, 0, rows, p.ld_out)
    p.qkv, p.out = qkv.data_ptr(), out.ptr
    out.arm()
    _lib.check(_lib.lib().sfb_temporal_attention(C.byref(p), _stream()), "sfb_temporal_attention")
    torch.cuda.synchronize()
    x = qkv[:, :3 * Cm].double().view(B, Fr, S, 3, H, D).permute(3, 0, 2, 4, 1, 5).reshape(3, B * S * H, Fr, D)
    ref = ref_attention(x[0], x[1], x[2], float(p.scale), False)
    ref = ref.view(B, S, H, Fr, D).permute(0, 3, 1, 2, 4).reshape(rows, Cm)
    res.add("out", rel_err(out.take(out.region(rows, Cm)), ref), tol("temporal", dt))
    res.canary(out)
    return res


def replay_row_op(op, peaked=False):
    name = op.fn.name
    p0 = op.keep[0]
    p = _clone(p0)
    nn = _nonnull(op)
    dt = DTYPES[p.dtype]
    res = Result()
    rows, c = p.rows, p.c
    x = _randn(_off(p0.x, 2) + rows * p.ldx, dt)
    X = _mat_view(x, _off(p0.x, 2), rows, c, p.ldx).double()
    p.x = x.data_ptr() + _off(p0.x, 2) * 2
    y = Canvas(dt, _off(p0.y, 2), rows, p.ldy)
    p.y = y.ptr
    m = torch.arange(rows, device=DEV)
    keep = []
    if name == "sfb_row_broadcast_add":
        if p.mode == _lib.ROW_IDX_DIV_MOD:
            idx = (m // p.div) % p.mod
            nvec = p.mod
        else:
            b_, px = m // (p.frames * p.seq), m % p.seq
            idx = ((b_ * p.seq + px) % p.batch) * p.frames
            nvec = p.batch * p.frames
        vec = _randn(nvec * p.ldv, dt).view(nvec, p.ldv)
        p.vec = vec.data_ptr()
        ref = X + vec[:, :c].double()[idx]
        keep.append(vec)
    else:
        x2 = _randn(_off(p0.x2, 2) + rows * p.ldx2, dt)
        p.x2 = x2.data_ptr() + _off(p0.x2, 2) * 2
        mix = torch.randn(1, device=DEV)
        p.mix_factor = mix.data_ptr()
        al = torch.sigmoid(mix.double())
        ref = al * X + (1 - al) * _mat_view(x2, _off(p0.x2, 2), rows, c, p.ldx2).double()
        keep += [x2, mix]
    rso = None
    slots = p.rowstats_slots or 1
    if nn["rowstats_out"]:
        rso = torch.full((rows + GUARD_ROWS, slots, 2), STATS_SENT, device=DEV)
        p.rowstats_out = rso.data_ptr()
    y.arm()
    _lib.check(getattr(_lib.lib(), name)(C.byref(p), _stream()), name)
    torch.cuda.synchronize()
    got = y.take(y.region(rows, c))
    res.add("y", rel_err(got, ref), tol("row_ops", dt))
    if rso is not None:
        check_rowstats(res, "rowstats_out", rso[:rows], got, 8, dt)   # slot 0 only
        res.add("rowstats_other_slots", 0.0 if bool((rso[:rows, 1:] == STATS_SENT).all()) else float("inf"), 0.0)
        res.add("rowstats_guard", 0.0 if bool((rso[rows:] == STATS_SENT).all()) else float("inf"), 0.0)
    res.canary(y)
    return res


def replay_add_nchw(op, peaked=False):
    p0 = op.keep[0]
    p = _clone(p0)
    dt = DTYPES[p.dtype]
    res = Result()
    items = []
    for i in range(p.count):
        it = p.items[i]
        off = int(p0.items[i].dst or 0) // 2
        dst = Canvas(dt, off, it.n * it.hw, it.ld_dst)
        region = dst.region(it.n * it.hw, it.c)
        region.copy_(_randn(it.n * it.hw * it.c, dt).view(-1, it.c))
        src = _randn(it.n * it.c * it.hw, dt).view(it.n, it.c, it.hw)
        ref = region.double() + src.double().permute(0, 2, 1).reshape(-1, it.c)
        it.src, it.dst = src.data_ptr(), dst.ptr
        dst.arm()
        items.append((dst, src, ref, it))
    _lib.check(_lib.lib().sfb_add_nchw_residuals(C.byref(p), _stream()), "sfb_add_nchw_residuals")
    torch.cuda.synchronize()
    for i, (dst, _, ref, it) in enumerate(items):
        res.add(f"dst{i}", rel_err(dst.take(dst.region(it.n * it.hw, it.c)), ref), tol("add_nchw", dt))
    res.canary(*[d for d, _, _, _ in items])
    return res


def replay_plain(op, peaked=False):
    name = op.fn.name
    a = dict(zip(PLAIN[name], op.args))
    lib = _lib.lib()
    res = Result()
    s = _stream()
    if name == "sfb_row_softmax":
        rows, cols, ldx, ldy = a["rows"], a["cols"], a["ldx"], a["ldy"]
        dt = DTYPES[a["dtype"]]
        xdt = torch.float32 if a["x_is_f32"] else dt
        scale = 8.0 if peaked else 1.0
        alias = a["x*"] == a["y*"]
        xb = Canvas(xdt, int(a["x*"] or 0) // xdt.itemsize, rows, ldx)
        xb.region(rows, cols).copy_((torch.randn(rows, cols, device=DEV) * scale).to(xdt))
        X = xb.region(rows, cols).double()
        yb = xb if alias else Canvas(dt, int(a["y*"] or 0) // 2, rows, ldy)
        xb.arm()
        if not alias:
            yb.arm()
        _lib.check(lib.sfb_row_softmax(xb.ptr, yb.ptr, rows, cols, ldx, ldy, a["x_is_f32"], a["dtype"], s), name)
        torch.cuda.synchronize()
        yv = yb.region(rows, cols, ld=ldy, dt=dt) if alias else yb.region(rows, cols)
        res.add("y", rel_err(yb.take(yv), torch.softmax(X, -1)), tol("softmax", dt))
        res.canary(xb, yb)
        return res
    if name == "sfb_conv_in":
        n, h, w, cin, cout, ldy, dt = a["n"], a["h"], a["wd"], a["cin"], a["cout"], a["ldy"], DTYPES[a["dtype"]]
        x = _randn(n * cin * h * w, dt).view(n, cin, h, w)
        w3 = _randn(cout * cin * 9, dt, 1 / math.sqrt(9 * cin)).view(cout, cin, 3, 3)
        wp, b = ops.pack_conv_in(w3, dt), torch.randn(cout, device=DEV)
        y = Canvas(dt, int(a["y*"] or 0) // 2, n * h * w, ldy)
        y.arm()
        _lib.check(lib.sfb_conv_in(x.data_ptr(), wp.data_ptr(), b.data_ptr(), y.ptr, n, h, w, cin, cout, ldy,
                                   a["dtype"], s), name)
        torch.cuda.synchronize()
        ref = F.conv2d(x.double(), w3.double(), b.double(), padding=1).permute(0, 2, 3, 1).reshape(-1, cout)
        res.add("y", rel_err(y.take(y.region(n * h * w, cout)), ref), tol("conv_edge", dt))
        res.canary(y)
        return res
    if name == "sfb_conv_out":
        n, h, w, cin, cout, ldx, dt = a["n"], a["h"], a["wd"], a["cin"], a["cout"], a["ldx"], DTYPES[a["dtype"]]
        offx = int(a["x*"] or 0) // 2
        xb = _randn(offx + n * h * w * ldx, dt)
        X = _nhwc_view(xb, offx, n, h, w, cin, ldx)
        w3 = _randn(cout * cin * 9, dt, 1 / math.sqrt(9 * cin)).view(cout, cin, 3, 3)
        wp, b = ops.pack_conv3x3(w3, dt), torch.randn(cout, device=DEV)
        y = Canvas(dt, 0, n * cout, h * w)
        y.arm()
        _lib.check(lib.sfb_conv_out(xb.data_ptr() + offx * 2, wp.data_ptr(), b.data_ptr(), y.ptr, n, h, w, cin, cout,
                                    ldx, a["dtype"], s), name)
        torch.cuda.synchronize()
        ref = F.conv2d(X.double().permute(0, 3, 1, 2), w3.double(), b.double(), padding=1).reshape(n * cout, h * w)
        res.add("y", rel_err(y.take(y.region(n * cout, h * w)), ref), tol("conv_edge", dt))
        res.canary(y)
        return res
    if name == "sfb_im2col_in":
        n, h, w, cin = a["n"], a["h"], a["wd"], a["cin"]
        dt = torch.float16
        x = _randn(n * cin * h * w, dt).view(n, cin, h, w)
        A = Canvas(dt, 0, n * h * w, 64)
        A.arm()
        _lib.check(lib.sfb_im2col_in(x.data_ptr(), A.ptr, n, h, w, cin, s), name)
        torch.cuda.synchronize()
        cols = F.unfold(x.double(), 3, padding=1).view(n, cin, 9, h * w).permute(0, 3, 2, 1).reshape(n * h * w, 9 * cin)
        ref = torch.zeros(n * h * w, 64, dtype=torch.float64, device=DEV)
        ref[:, :9 * cin] = cols
        res.add("a", rel_err(A.take(A.region(n * h * w, 64)), ref), tol("exact", dt))
        res.canary(A)
        return res
    if name == "sfb_upsample2x":
        n, h, w, c, ldx, ldy = a["n"], a["h"], a["w"], a["c"], a["ldx"], a["ldy"]
        dt = torch.float16
        offx = int(a["x*"] or 0) // 2
        xb = _randn(offx + n * h * w * ldx, dt)
        X = _nhwc_view(xb, offx, n, h, w, c, ldx)
        y = Canvas(dt, int(a["y*"] or 0) // 2, 4 * n * h * w, ldy)
        y.arm()
        _lib.check(lib.sfb_upsample2x(xb.data_ptr() + offx * 2, y.ptr, n, h, w, c, ldx, ldy, s), name)
        torch.cuda.synchronize()
        ref = X.double().repeat_interleave(2, 1).repeat_interleave(2, 2).reshape(-1, c)
        res.add("y", rel_err(y.take(y.region(4 * n * h * w, c)), ref), tol("exact", dt))
        res.canary(y)
        return res
    if name == "sfb_timestep_embed":
        B, dim, ldo, dt = a["batch"], a["dim"], a["ldo"], DTYPES[a["dtype"]]
        t = torch.rand(B, device=DEV) * 1000.0
        out = Canvas(dt, int(a["out*"] or 0) // 2, B, ldo)
        out.arm()
        _lib.check(lib.sfb_timestep_embed(t.data_ptr(), B, dim, a["flip"], a["shift"], out.ptr, ldo, a["dtype"], s),
                   name)
        torch.cuda.synchronize()
        ref = ref_timestep_embed(t.double(), dim, a["flip"], a["shift"])
        res.add("out", rel_err(out.take(out.region(B, dim)), ref), tol("timestep", dt))
        res.canary(out)
        return res
    if name == "sfb_pointwise_nchw":
        n, hw, cin, cout, dt = a["n"], a["hw"], a["cin"], a["cout"], DTYPES[a["dtype"]]
        x = _randn(n * cin * hw, dt).view(n, cin, hw)
        w = _randn(cout * cin, dt, 1 / math.sqrt(cin)).view(cout, cin)
        b = torch.randn(cout, device=DEV)
        y = Canvas(dt, 0, n * cout, hw)
        y.arm()
        _lib.check(lib.sfb_pointwise_nchw(x.data_ptr(), w.data_ptr(), b.data_ptr(), y.ptr, n, hw, cin, cout,
                                          a["dtype"], s), name)
        torch.cuda.synchronize()
        ref = (torch.einsum("oc,ncp->nop", w.double(), x.double()) + b.double()[None, :, None]).reshape(n * cout, hw)
        res.add("y", rel_err(y.take(y.region(n * cout, hw)), ref), tol("pointwise", dt))
        res.canary(y)
        return res
    if name == "sfb_embed_tokens":
        B, S, dim, V, ld, dt = a["batch"], a["seq"], a["dim"], a["vocab"], a["ld_out"], DTYPES[a["dtype"]]
        tok, pos = _randn(V * dim, dt).view(V, dim), _randn(S * dim, dt).view(S, dim)
        ids = torch.randint(0, V, (B, S), device=DEV)
        out = Canvas(dt, int(a["out*"] or 0) // 2, B * S, ld)
        slots = a["slots"]
        rso = None
        if a["rowstats*"] is not None:
            rso = torch.full((B * S + GUARD_ROWS, slots, 2), STATS_SENT, device=DEV)
        out.arm()
        _lib.check(lib.sfb_embed_tokens(ids.data_ptr(), tok.data_ptr(), pos.data_ptr(), out.ptr,
                                        rso.data_ptr() if rso is not None else None, slots, B, S, dim, V, ld,
                                        a["dtype"], s), name)
        torch.cuda.synchronize()
        ref = (tok[ids].double() + pos[None].double()).reshape(B * S, dim).to(dt)
        got = out.take(out.region(B * S, dim))
        res.add("out", rel_err(got, ref), tol("exact", dt))
        if rso is not None:
            check_rowstats(res, "rowstats", rso[:B * S], got, 8, dt)
            res.add("rowstats_other_slots", 0.0 if bool((rso[:B * S, 1:] == STATS_SENT).all()) else float("inf"), 0.0)
            res.add("rowstats_guard", 0.0 if bool((rso[B * S:] == STATS_SENT).all()) else float("inf"), 0.0)
        res.canary(out)
        return res
    if name == "sfb_clip_pool":
        B, S, dim, ld, eos = a["batch"], a["seq"], a["dim"], a["ld_x"], a["eos_id"]
        dt = torch.float16
        offx = int(a["x*"] or 0) // 2
        xb = _randn(offx + B * S * ld, dt)
        X = _mat_view(xb, offx, B * S, dim, ld)
        ids = torch.randint(3, 1000, (B, S), device=DEV)
        eos_tok = 49407 if eos == 2 else eos
        for b in range(B):
            ids[b, (5 + 13 * b) % S:] = eos_tok
        pooled = Canvas(dt, 0, B, dim)
        pooled.arm()
        _lib.check(lib.sfb_clip_pool(ids.data_ptr(), xb.data_ptr() + offx * 2, pooled.ptr, B, S, dim, ld, eos, s),
                   name)
        torch.cuda.synchronize()
        pos = ids.argmax(-1) if eos == 2 else (ids == eos).int().argmax(-1)
        ref = X.view(B, S, dim)[torch.arange(B, device=DEV), pos].double()
        res.add("pooled", rel_err(pooled.take(pooled.region(B, dim)), ref), tol("exact", dt))
        res.canary(pooled)
        return res
    if name == "sfb_patchify":
        B, Cc, h, w, P, kpad = a["batch"], a["chans"], a["h"], a["w"], a["patch"], a["kpad"]
        dt = torch.float16
        x = _randn(B * Cc * h * w, dt).view(B, Cc, h, w)
        rows = B * (h // P) * (w // P)
        A = Canvas(dt, 0, rows, kpad)
        A.arm()
        _lib.check(lib.sfb_patchify(x.data_ptr(), A.ptr, B, Cc, h, w, P, kpad, s), name)
        torch.cuda.synchronize()
        ref = torch.zeros(rows, kpad, dtype=torch.float64, device=DEV)
        ref[:, :Cc * P * P] = F.unfold(x.double(), P, stride=P).transpose(1, 2).reshape(rows, Cc * P * P)
        res.add("a", rel_err(A.take(A.region(rows, kpad)), ref), tol("exact", dt))
        res.canary(A)
        return res
    if name == "sfb_copy2d":
        rows, cols, lds, ldd = a["rows"], a["cols"], a["ld_src"], a["ld_dst"]
        dt = torch.float16
        offs = int(a["src*"] or 0) // 2
        src = _randn(offs + rows * lds, dt)
        dst = Canvas(dt, int(a["dst*"] or 0) // 2, rows, ldd)
        dst.arm()
        _lib.check(lib.sfb_copy2d(src.data_ptr() + offs * 2, dst.ptr, rows, cols, lds, ldd, s), name)
        torch.cuda.synchronize()
        res.add("dst", rel_err(dst.take(dst.region(rows, cols)), _mat_view(src, offs, rows, cols, lds).double()),
                tol("exact", dt))
        res.canary(dst)
        return res
    raise NotImplementedError(name)


REPLAY = {"sfb_gemm": replay_gemm, "sfb_attention": replay_attention,
          "sfb_group_norm_fused": replay_group_norm, "sfb_group_norm_stats": replay_group_norm,
          "sfb_group_norm_apply": replay_group_norm, "sfb_group_norm_scale_shift": replay_group_norm,
          "sfb_layer_norm": replay_layer_norm, "sfb_small_linear": replay_small_linear,
          "sfb_temporal_attention": replay_temporal, "sfb_row_broadcast_add": replay_row_op,
          "sfb_alpha_blend": replay_row_op, "sfb_add_nchw_residuals": replay_add_nchw,
          **{n: replay_plain for n in PLAIN}}
PEAKED = ("sfb_attention", "sfb_row_softmax")   # replayed a second time with score std ~8


def describe(key):
    """Short human-readable summary of a key."""
    name = key[0]
    if name in PLAIN:
        return f"{name}({', '.join(f'{n}={v}' for n, v in zip(PLAIN[name], key[1:]) if not n.endswith('*'))})"
    if name == "sfb_add_nchw_residuals":
        return f"{name}(count={key[1]})"
    g = {kv[0]: kv[-1] for kv in key[1]}
    if name == "sfb_gemm":
        return (f"sfb_gemm(a_mode={g['a_mode']} epi={g['epi']} M={g['M']} N={g['N']} K={g['K']} ldo={g['ldo']} "
                f"splits={g['splits']} defer={g['defer_finish']} act={g['act']} b_plain={g['b_plain']} "
                f"ln_slots={g['ln_slots']} img={g['img_n']}x{g['img_h']}x{g['img_w']} box={g['box_n']}x{g['box_h']}"
                f"x{g['box_w']} dtype={g['dtype']})")
    show = ", ".join(f"{k}={v}" for k, v in g.items() if not isinstance(v, float) or k in ("eps", "scale"))
    return f"{name}({show})"


def replay(key, ent, peaked=False, soundness=None):
    """Replay one key on the GPU: a Result.  `soundness` "w" / "rw": also check the access model of
    plan_hazards.py against every launch of the replay -- its writes ("w"), and its writes and reads ("rw")."""
    seed = int(hashlib.sha1(repr(key).encode()).hexdigest()[:8], 16) + int(peaked)
    torch.manual_seed(seed)
    try:
        if not soundness:
            return REPLAY[ent["name"]](ent["op"], peaked=peaked)
        import plan_hazards  # (imports this module)
        with plan_hazards.checking_launches(read_check="r" in soundness) as sound:
            res = REPLAY[ent["name"]](ent["op"], peaked=peaked)
        assert sound.writes and (sound.reads or "r" not in soundness), "no launch of the replay was checked"
        res.add("access_model", float("inf") if sound.violations else 0.0, 0.0)
        res.model = sound.violations
        return res
    finally:
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def run_keys(entries, keys, log=None, soundness=None):
    """Replay `keys`; yields one record per replay (peaked entry points twice).  `soundness`: {key: "w" / "rw"},
    the access-model check of each key's first replay (replay())."""
    for key in keys:
        ent = entries[key]
        for peaked in ((False, True) if ent["name"] in PEAKED else (False,)):
            t0 = time.time()
            sound = None if peaked or not soundness else soundness.get(key)
            try:
                r = replay(key, ent, peaked, sound)
                err, tl = r.main()
                rec = dict(key=key_id(key), entry=ent["name"], peaked=peaked, desc=describe(key), plans=ent["plans"],
                           err=err, tol=tl, parts=[(w, e, t) for w, e, t in r.parts], ok=r.ok)
                if sound:
                    rec.update(soundness=sound, model=getattr(r, "model", []))
            except Exception as e:  # noqa: BLE001  -- a launch the library refuses is a failing key
                rec = dict(key=key_id(key), entry=ent["name"], peaked=peaked, desc=describe(key), plans=ent["plans"],
                           err=float("inf"), tol=0.0, error=repr(e)[:400], ok=False)
            rec["seconds"] = round(time.time() - t0, 3)
            if log is not None:
                log(rec)
            yield rec


def summarize(records):
    """{entry point: (largest error, its tolerance, keys replayed, failures)}"""
    out = {}
    for r in records:
        e = out.setdefault(r["entry"], [0.0, 0.0, 0, 0])
        if r["err"] >= e[0]:
            e[0], e[1] = r["err"], r["tol"]
        e[2] += 1
        e[3] += 0 if r["ok"] else 1
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--plans", nargs="*", help="plan names (default: all); see --list")
    ap.add_argument("--all", action="store_true", help="replay every distinct key, not the default subset")
    ap.add_argument("--json", help="also write the records (and the summary) to this JSON file")
    ap.add_argument("--list", action="store_true", help="list plans and distinct keys per entry point, no GPU")
    ap.add_argument("--soundness", action="store_true",
                    help="also check plan_hazards.py's access model: writes on every key, reads on the default subset")
    args = ap.parse_args(argv)
    t0 = time.time()
    entries, names = collect(args.plans)
    missing = check_coverage(names)
    if missing:
        print(json.dumps({"uncovered_entry_points": missing}))
        return 2
    keys = list(entries) if args.all else select_subset(entries)
    per = collections.Counter(e["name"] for e in entries.values())
    print(json.dumps({"plans": args.plans or [n for n, _, _ in PLANS], "distinct_keys": len(entries),
                      "replaying": len(keys), "keys_per_entry_point": dict(per),
                      "build_seconds": round(time.time() - t0, 1)}), flush=True)
    if args.list:
        return 0
    torch.cuda.reset_peak_memory_stats()
    t1 = time.time()
    sound = None
    if args.soundness:
        sub = set(select_subset(entries))
        sound = {k: "rw" if k in sub else "w" for k in keys}
    records = list(run_keys(entries, keys, log=lambda r: print(json.dumps(r), flush=True), soundness=sound))
    summ = summarize(records)
    tail = {"summary": {k: dict(max_err=v[0], tol=v[1], replays=v[2], failures=v[3]) for k, v in sorted(summ.items())},
            "replay_seconds": round(time.time() - t1, 1),
            "peak_max_memory_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
            "device": torch.cuda.get_device_name()}
    print(json.dumps(tail), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(records=records, **tail), f, indent=0)
    return 0 if all(r["ok"] for r in records) else 1


if __name__ == "__main__":
    sys.exit(main())
