"""Launch descriptors for the C-ABI kernels.

Each builder returns an :class:`Op`: a bound C entry point plus its argument block, created ONCE
at plan-build time (pointers, tensor maps, geometry are all static), so that running or
CUDA-graph-capturing a UNet step is a flat loop of ``op.launch(stream)`` calls.
"""
import ctypes as C
import math
import os

import torch

from . import _lib
from ._lib import (A_CONV3X1, A_CONV3X3, A_CONV3X3_GN, A_DOWNCONV3X3, A_MATRIX, A_UPCONV2X, EPI_GEGLU, EPI_QKV, EPI_STORE, AttnParams, GemmParams,
                   GnParams, LnParams, SmallLinearParams, TensorMap, check)

BM, BN, BK = 128, 160, 64
_NUM_SMS = None


def num_sms():
    """SMs of the current CUDA device (the C library's count: 132 on an H100 SXM, fewer under MIG
    or a green context); 132 when planning without a GPU (dry plans in CPU tests)."""
    global _NUM_SMS
    if _NUM_SMS is None:
        if torch.cuda.is_available():
            _NUM_SMS = int(_lib.lib().sfb_sm_count())
        else:
            return 132
    return _NUM_SMS


def dtype_code(dt):
    if dt == torch.float16:
        return _lib.SFB_F16
    if dt == torch.bfloat16:
        return _lib.SFB_BF16
    raise NotImplementedError(f"sfast_b200 computes in fp16/bf16 storage; got {dt}")


def _ptr(t):
    """Device address of a tensor / raw address; 0 for None-like dry-run (meta) tensors."""
    if t is None:
        return None
    if isinstance(t, int):
        return t
    if t.device.type == "meta":
        return 0
    return t.data_ptr()


class Act:
    """A [n, h, w, c] (or [rows, c] with h = w = 1) activation view with channel pitch ``ld``
    inside a (possibly wider) buffer, e.g. one half of a skip-concat buffer."""
    __slots__ = ("buf", "off", "n", "h", "w", "c", "ld")

    def __init__(self, buf, n, h, w, c, ld=None, off=0):
        self.buf, self.n, self.h, self.w, self.c = buf, n, h, w, c
        self.ld = c if ld is None else ld
        self.off = off

    @property
    def ptr(self):
        return _ptr(self.buf) + self.off * self.buf.element_size()

    @property
    def rows(self):
        return self.n * self.h * self.w

    def tensor(self):
        """torch view [n, h, w, c] (for tests / debugging)."""
        flat = self.buf.view(-1)[self.off:]
        return flat.as_strided((self.n, self.h, self.w, self.c),
                               (self.h * self.w * self.ld, self.w * self.ld, self.ld, 1))


class Op:
    __slots__ = ("name", "fn", "args", "keep", "flops", "bytes")

    def __init__(self, name, fn, args, keep, flops=0, nbytes=0):
        self.name, self.fn, self.args, self.keep = name, fn, args, keep
        self.flops, self.bytes = flops, nbytes

    def launch(self, stream):
        rc = self.fn(*self.args, stream)
        if rc != 0:
            check(rc, self.name)


class DryMap:
    """Stand-in for a TMA tensor map when a plan is built without a GPU (host-logic tests)."""
    ptr = 0

    def __init__(self, *geom):
        self.geom = geom


def matrix_map(ptr, rows, cols, pitch, box_rows, dry=False):
    if dry:
        return DryMap("2d", rows, cols, pitch, box_rows)
    return TensorMap.matrix(ptr, rows, cols, pitch, box_rows)


def nhwc_map(ptr, n, h, w, c, pitch, box_n, box_h, box_w, stride=1, dry=False):
    if dry:
        return DryMap("nhwc", n, h, w, c, pitch, box_n, box_h, box_w, stride)
    return TensorMap.nhwc(ptr, n, h, w, c, pitch, box_n, box_h, box_w, stride)


def conv_tile_box(ho, wo):
    """[box_n, box_h, box_w] of the 128-pixel M tile for an output image of ho x wo.
    Widths that divide 128: full-width rows (several images per tile when the image is smaller than
    128 pixels).  Any other width: 2-D patches of box_w = gcd(wo, 128) columns x 128 / box_w rows
    (rows past the image are zero-filled by TMA on load and masked in the epilogue)."""
    if wo <= BM and BM % wo == 0:
        rows = BM // wo
        if rows <= ho:
            return 1, rows, wo
        if rows % ho == 0:
            return rows // ho, ho, wo
    box_w = math.gcd(wo, BM)
    return 1, BM // box_w, box_w


# split-K cost model (microseconds): a single-wave GEMM launch costs a fixed prologue + epilogue +
# drain plus a per-64-wide-K-block time of its longest CTA; the stand-alone reduction kernel ~10 us
# plus its fp32 partial traffic at ~3 TB/s (a conv followed by a GroupNorm leaves the reduction to
# that kernel).  The constants were fitted on an earlier build of the GEMM and are not re-fitted for
# the H100 kernel; they only choose the split factor, never the result.
_T_FIXED, _T_KB = 4.5, 0.34


def choose_splits(m_tiles, n_tiles, nkb, M=None, N=None):
    """Split-K factor minimising the modelled launch time.  Only grids of at most half a wave are
    split (the weight-bandwidth-bound low-resolution layers); all split CTAs fit in one wave."""
    tiles = m_tiles * n_tiles
    sms = num_sms()
    if tiles * 2 > sms:
        return 1
    M = M if M is not None else m_tiles * BM
    N = N if N is not None else n_tiles * BN
    best, best_t = 1, _T_FIXED + _T_KB * nkb
    for s in range(2, min(sms // tiles, nkb) + 1):
        t = _T_FIXED + _T_KB * -(-nkb // s) + 10.0 + s * M * N * 4 / 3e6
        if t < best_t - 0.5:
            best, best_t = s, t
    return best


# cta_pair / persistent only select the weight tensor map's box height in the C ABI (80 rows instead
# of 160, loaded as two boxes per tile); every launch runs the one-tile wgmma kernel.  Off by default:
# one 160-row box per weight tile is one TMA instruction instead of two.
ENABLE_CTA_PAIR = os.environ.get("SFB_CTA_PAIR", "0") != "0"
# "auto" = request `persistent` for grids of at least SFB_PERSIST_MIN_CTAS CTAs (needs cta_pair).
PERSIST = os.environ.get("SFB_PERSIST", "0")
PERSIST_MIN_CTAS = int(os.environ.get("SFB_PERSIST_MIN_CTAS", "200"))


def a_matrix(x_ptr, rows, cols, pitch):
    return dict(kind="matrix", ptr=x_ptr, rows=rows, cols=cols, pitch=pitch)


def a_conv(x_ptr, n, h, w, c, pitch, box_n, box_h, box_w, stride):
    """NHWC conv input [n, h, w, c]; the M tile covers [box_n, box_h, box_w] OUTPUT pixels."""
    return dict(kind="conv", ptr=x_ptr, n=n, h=h, w=w, c=c, pitch=pitch, box_n=box_n, box_h=box_h,
                wo=box_w, stride=stride)


# GroupNorm folded into the conv (SFB_A_CONV3X3_GN): 16 x 8 pixel output patches, [18 x 10] halo tiles
HALO_BOX_H, HALO_BOX_W = 16, 8
CONV_GN = os.environ.get("SFB_CONV_GN", "auto")


def a_conv_halo(x_ptr, n, h, w, c, pitch):
    """RAW NHWC conv input whose GroupNorm(+SiLU) the conv applies itself: TMA box = the halo tile of
    a 16 x 8 output patch."""
    return dict(kind="conv_halo", ptr=x_ptr, n=n, h=h, w=w, c=c, pitch=pitch)


def conv_gn_tiles(n, h, w):
    """M tiles of the halo conv over n images of h x w pixels, or 0 if the geometry is not eligible
    (width a multiple of 8, an even number of tiles for the CTA pairs)."""
    if w % HALO_BOX_W or h < 1:
        return 0
    tiles = n * ((h + HALO_BOX_H - 1) // HALO_BOX_H) * (w // HALO_BOX_W)
    return tiles if tiles % 2 == 0 else 0


def _a_map(a, dry):
    """A-operand TMA map with a box of one 128-row tile."""
    if a["kind"] == "matrix":
        return matrix_map(a["ptr"], a["rows"], a["cols"], a["pitch"], BM, dry)
    if a["kind"] == "conv_halo":
        return nhwc_map(a["ptr"], a["n"], a["h"], a["w"], a["c"], a["pitch"], 1, HALO_BOX_H + 2,
                        HALO_BOX_W + 2, 1, dry)
    return nhwc_map(a["ptr"], a["n"], a["h"], a["w"], a["c"], a["pitch"], a["box_n"], a["box_h"],
                    a["wo"], a["stride"], dry)


def gemm_op(name, lib, *, M, N, K, dt, a_map=None, b_map=None, a=None, b=None, out=None, ldo=0,
            bias=None, rowbias=None, rows_per_img=1, ld_rowbias=0, residual=None, ldr=0,
            epi=EPI_STORE, geglu_n_out=0, conv=None, qkv=None, ws=None, splits=None, keep=(),
            rowstats_out=None, ln=None, dry=False, cta_pair=None, persistent=None, act=0, gn=None):
    """Either pass ready-made maps (`a_map`, `b_map`) or operand descriptors (`a` from
    a_matrix()/a_conv(), `b` a Mat), in which case the weight map gets the 160-row box, or the 80-row
    box of the cta_pair flag (ENABLE_CTA_PAIR / `cta_pair=True`, even number of M tiles only)."""
    p = GemmParams()
    up = bool(conv and conv.get("up"))
    if gn is not None:
        # GroupNorm folded into the conv: `gn` = dict(scale_shift=[n, cin, 2] fp32 tensor, silu=bool)
        assert conv and a is not None and a["kind"] == "conv_halo" and not up
        assert (conv["box_n"], conv["box_h"], conv["box_w"]) == (1, HALO_BOX_H, HALO_BOX_W)
        splits, persistent = 1, False
        p.gn_scale_shift, p.gn_silu = _ptr(gn["scale_shift"]), int(bool(gn.get("silu", True)))
        keep = tuple(keep) + (gn["scale_shift"],)
    if conv:
        if conv["box_n"] == 1:
            m_tiles = conv["n"] * ((conv["h"] + conv["box_h"] - 1) // conv["box_h"]) * \
                (conv["w"] // conv.get("box_w", conv["w"]))
        else:
            m_tiles = (conv["n"] + conv["box_n"] - 1) // conv["box_n"]
        phase_tiles = m_tiles
        if up:
            m_tiles *= 4  # one set of M tiles per output phase
    else:
        m_tiles = phase_tiles = (M + BM - 1) // BM
    n_tiles = (N + BN - 1) // BN
    nkb = K // BK
    if a is not None:
        # `persistent` is defined on the 80-row weight box: asking for it asks for cta_pair
        if cta_pair is None:
            cta_pair = ENABLE_CTA_PAIR or bool(persistent)
        pair = cta_pair and phase_tiles % 2 == 0
        a_map = _a_map(a, dry)
        b_map = b.map_for(2 if pair else 1)
        p.cta_pair = 1 if pair else 0
        p.b_plain = 1 if isinstance(b, PlainB) else 0
        keep = tuple(keep) + (b,)
    p.tmap_a, p.tmap_b = a_map.ptr, b_map.ptr
    p.a_mode = (A_UPCONV2X if up else (A_CONV3X1 if conv.get("temporal") else A_CONV3X3)) if conv else A_MATRIX
    if gn is not None:
        p.a_mode = A_CONV3X3_GN
    if conv and conv.get("down"):
        # the tensor map covers the input image, which the C side cannot see: output = input / 2 here
        if a is not None and (a["h"], a["w"]) != (2 * conv["h"], 2 * conv["w"]):
            raise ValueError(f"{name}: down-conv output {conv['h']}x{conv['w']} is not half of the input "
                             f"{a['h']}x{a['w']}")
        p.a_mode = A_DOWNCONV3X3
    p.M, p.N, p.K, p.dtype = M, N, K, dtype_code(dt)
    if conv:
        p.img_n, p.img_h, p.img_w = conv["n"], conv["h"], conv["w"]
        p.cin, p.conv_stride = conv["cin"], conv["stride"]
        p.box_n, p.box_h = conv["box_n"], conv["box_h"]
        p.box_w = conv.get("box_w", conv["w"])
    if splits is None:
        splits = choose_splits(m_tiles, n_tiles, nkb, M, N)
    if ws is None:
        splits = 1
    p.splits = splits
    if splits > 1:
        need = splits * M * N
        if ws.numel() < need:
            raise ValueError(f"{name}: split-K workspace too small ({ws.numel()} < {need})")
        p.ws = _ptr(ws) if not hasattr(ws, "finalize") else 0
    if persistent is None:
        persistent = PERSIST == "1" or (PERSIST == "auto" and m_tiles * n_tiles >= PERSIST_MIN_CTAS)
    p.persistent = 1 if (persistent and p.cta_pair and splits == 1 and epi != _lib.EPI_STORE_F32 and not act
                         and rowstats_out is None) else 0
    p.act = act
    p.epi = epi
    p.out = _ptr(out)
    p.ldo = ldo
    p.bias = _ptr(bias)
    p.rowbias = _ptr(rowbias)
    p.rows_per_img, p.ld_rowbias = rows_per_img, ld_rowbias
    p.residual = _ptr(residual)
    p.ldr = ldr
    p.geglu_n_out = geglu_n_out
    if qkv:
        p.q, p.k, p.vt = _ptr(qkv.get("q")), _ptr(qkv.get("k")), _ptr(qkv.get("vt"))
        for f in ("heads", "head_dim", "which_base", "seq", "q_pitch", "q_rows", "k_rows",
                  "vt_rows", "vt_pitch"):
            setattr(p, f, qkv[f])
    p.rowstats_out = _ptr(rowstats_out)
    p.rowstats_out_slots = getattr(rowstats_out, "slots", rowstats_slots(N)) if rowstats_out is not None else 0
    if ln is not None:
        p.ln_rowstats, p.ln_colsum = _ptr(ln["rowstats"]), _ptr(ln["colsum"])
        p.ln_eps, p.ln_dim = ln["eps"], ln["dim"]
        p.ln_slots = getattr(ln["rowstats"], "slots", 1)
    esz = 2
    flops = 2 * M * N * K
    nbytes = (M * K + N * K) * esz + M * (geglu_n_out if epi == EPI_GEGLU else N) * esz
    op = Op(name, lib.sfb_gemm, (C.byref(p),), (p, a_map, b_map, out, bias, rowbias, residual, ws,
                                               qkv, keep, rowstats_out, ln), flops, nbytes)
    return op


# Attention KV tile: 64 or 128 keys per wgmma score tile.  The 64-key kernel exists for head_dim
# 32 / 40 / 64 / 160; "auto" takes it for head_dim 64 and for head_dim 160, where the 128-key score tile
# next to the 176-column O accumulator would not fit the 168 registers a thread may use.
# "0": always 128; "1": 64 wherever it exists.
ATTN_V2 = os.environ.get("SFB_ATTN_V2", "auto")


def attention_kv_tile(head_dim):
    if ATTN_V2 == "0" or head_dim not in (32, 40, 64, 160):
        return 128
    if ATTN_V2 == "auto":
        return 64 if head_dim in (64, 160) else 128
    return 64  # "1" / "all": wherever the kernel exists


def attention_op(name, lib, *, q, k, vt, out, batch, heads, head_dim, seq_q, seq_kv, q_rows, k_rows,
                 vt_rows, q_pitch, vt_pitch, dt, dry=False, kv_tile=None, causal=False, ip=None):
    """sfb_attention; with `ip` (dict: k, vt, seq, k_rows, vt_pitch, scale -- a one-float device tensor)
    sfb_attention_ip, which adds scale * softmax(q k_ip^T / sqrt(D)) v_ip."""
    if ip is not None:
        return _attention_ip_op(name, lib, ip, attention_op(
            name, lib, q=q, k=k, vt=vt, out=out, batch=batch, heads=heads, head_dim=head_dim, seq_q=seq_q,
            seq_kv=seq_kv, q_rows=q_rows, k_rows=k_rows, vt_rows=vt_rows, q_pitch=q_pitch, vt_pitch=vt_pitch,
            dt=dt, dry=dry, kv_tile=kv_tile), dry)
    bh = batch * heads
    # v2 kernel (64-key tiles, double-buffered score / probability tiles) for head_dim <= 64
    if kv_tile is None:
        kv_tile = attention_kv_tile(head_dim)
    tq = matrix_map(_ptr(q), bh * q_rows, q_pitch, q_pitch, 128, dry)
    tk = matrix_map(_ptr(k), bh * k_rows, q_pitch, q_pitch, kv_tile, dry)
    tv = matrix_map(_ptr(vt), bh * vt_rows, vt_pitch, vt_pitch, vt_rows, dry)
    p = AttnParams()
    p.tmap_q, p.tmap_k, p.tmap_vt = tq.ptr, tk.ptr, tv.ptr
    p.out = _ptr(out)
    p.batch, p.heads, p.head_dim = batch, heads, head_dim
    p.seq_q, p.seq_kv = seq_q, seq_kv
    p.q_rows, p.k_rows, p.vt_rows = q_rows, k_rows, vt_rows
    p.dtype = dtype_code(dt)
    p.scale = 1.0 / math.sqrt(head_dim)
    p.kv_tile = kv_tile
    p.causal = 1 if causal else 0
    flops = 4 * batch * heads * seq_q * seq_kv * head_dim
    nbytes = 2 * bh * (2 * seq_q + 2 * seq_kv) * head_dim
    return Op(name, lib.sfb_attention, (C.byref(p),), (p, tq, tk, tv, q, k, vt, out), flops, nbytes)


def _attention_ip_op(name, lib, ip, text, dry):
    """The sfb_attention_ip launch around the text attention op `text` (its params become `base`)."""
    p0, tq, tk, tv = text.keep[:4]
    bh = p0.batch * p0.heads
    tki = matrix_map(_ptr(ip["k"]), bh * ip["k_rows"], tk_cols(p0.head_dim), tk_cols(p0.head_dim), p0.kv_tile, dry)
    tvi = matrix_map(_ptr(ip["vt"]), bh * p0.vt_rows, ip["vt_pitch"], ip["vt_pitch"], p0.vt_rows, dry)
    p = _lib.AttnIpParams()
    p.base = p0
    p.tmap_k_ip, p.tmap_vt_ip = tki.ptr, tvi.ptr
    p.seq_ip, p.k_ip_rows = ip["seq"], ip["k_rows"]
    p.ip_scale = _ptr(ip["scale"])
    flops = text.flops + 4 * bh * p0.seq_q * ip["seq"] * p0.head_dim
    nbytes = text.bytes + 2 * bh * 2 * ip["seq"] * p0.head_dim
    return Op(name, lib.sfb_attention_ip, (C.byref(p),),
              (p, tki, tvi, ip["k"], ip["vt"], ip["scale"]) + tuple(text.keep[1:]), flops, nbytes)


def tk_cols(head_dim):
    """Element pitch of a Q / K row: head_dim rounded up to 64 (one 128-byte swizzle row per 64 dims)."""
    return (head_dim + 63) // 64 * 64


def gn_fused_fits(n, hw, c, groups):
    """Python mirror of sfb_group_norm_fused_fits (used for dry plans; the C predicate is the
    authority on a GPU box)."""
    if n <= 0 or c % 8 or c % groups or c // 8 > 512:
        return False
    if n > num_sms():
        return False
    bpi = max(1, min(num_sms() // n, hw))
    rpb = (hw + bpi - 1) // bpi
    return rpb * c * 2 + 2 * c * 4 <= 190 * 1024


def rowstats_slots(n_cols):
    """Slots per row of a folded LayerNorm's statistics buffer whose producer has n_cols output columns
    (mirror of sfb_rowstats_slots): one per 160-column GEMM tile, or per warp segment of the split-K
    reduction kernel, whichever is more."""
    return max((n_cols + BN - 1) // BN, (n_cols // 8 - 1 + 31) // 32 + 1)


class RowStats:
    """[rows, slots, 2] fp32 view of a statistics arena; quacks like a tensor for _ptr()."""
    __slots__ = ("t", "slots")

    def __init__(self, t, slots):
        self.t, self.slots = t, slots

    @property
    def device(self):
        return self.t.device

    def data_ptr(self):
        return self.t.data_ptr()


def gn_ws_floats(n, groups):
    """Floats of the statistics workspace of one GroupNorm over n images (mirror of
    sfb_group_norm_ws_floats): one [groups][2] slot per CTA of the statistics pass."""
    return (2 * num_sms() + max(n, 1)) * 2 * groups


def gn_fused_ok(lib, x: Act, groups, dt, dry):
    """Whether GroupNorm over `x` takes the single-launch fused kernel."""
    if dry:
        return gn_fused_fits(x.n, x.h * x.w, x.c, groups)
    p = GnParams()
    p.n, p.hw, p.c, p.ldx, p.groups, p.dtype = x.n, x.h * x.w, x.c, x.ld, groups, dtype_code(dt)
    return bool(lib.sfb_group_norm_fused_fits(C.byref(p)))


def gn_ops(name, lib, *, x: Act, y: Act, gamma, beta, stats, groups, eps, silu, dt, sync=None,
           dry=False, partial=None):
    """GroupNorm(+SiLU): one fused launch when the tensor fits in shared memory (stats + apply
    with a grid barrier, x read once), else the two-pass stats / apply kernels.
    `partial`: channels [0, c) of x are still the fp32 split-K partials of their producer GEMM
    (launched with defer_finish); the fused kernel finishes them (dict: splits, c, ld, bias,
    rowbias, ld_rowbias, residual, ldr; the workspace pointer is patched in by the plan)."""
    p = GnParams()
    p.x, p.y = x.ptr, y.ptr
    p.gamma, p.beta, p.stats = _ptr(gamma), _ptr(beta), _ptr(stats)
    p.n, p.hw, p.c, p.ldx, p.ldy, p.groups = x.n, x.h * x.w, x.c, x.ld, y.ld, groups
    p.eps, p.silu, p.dtype = eps, int(silu), dtype_code(dt)
    p.sync_counter = _ptr(sync)
    keep = (p, x.buf, y.buf, gamma, beta, stats, sync)
    nb = x.rows * x.c * 2
    if sync is not None:
        fits = gn_fused_fits(p.n, p.hw, p.c, groups) if dry else bool(
            lib.sfb_group_norm_fused_fits(C.byref(p)))
        if fits:
            if partial is not None:
                p.part_splits, p.part_c, p.part_ld = partial["splits"], partial["c"], partial["ld"]
                p.part_bias, p.part_rowbias = _ptr(partial.get("bias")), partial.get("rowbias") or 0
                p.part_ld_rowbias = partial.get("ld_rowbias", 0)
                p.part_residual, p.part_ldr = partial.get("residual") or 0, partial.get("ldr", 0)
                p.part_ws = _ptr(partial.get("ws"))
                keep = keep + (partial,)
            return [Op(name + ".fused", lib.sfb_group_norm_fused, (C.byref(p),), keep, 0, 2 * nb)]
    if partial is not None:
        raise ValueError(f"{name}: deferred split-K finish needs the fused GroupNorm kernel")
    return [Op(name + ".stats", lib.sfb_group_norm_stats, (C.byref(p),), keep, 0, nb),
            Op(name + ".apply", lib.sfb_group_norm_apply, (C.byref(p),), keep, 0, 2 * nb)]


def gn_scale_shift_op(name, lib, *, x: Act, gamma, beta, stats, counters, scale_shift, groups, eps, dt):
    """GroupNorm statistics of x ending in per-(image, channel) (scale, shift) pairs -- the producer side of
    the halo conv (`gemm_op(..., gn=...)`).  `counters`: x.n int32 tickets, zero before the first launch."""
    p = GnParams()
    p.x = x.ptr
    p.gamma, p.beta, p.stats = _ptr(gamma), _ptr(beta), _ptr(stats)
    p.n, p.hw, p.c, p.ldx, p.ldy, p.groups = x.n, x.h * x.w, x.c, x.ld, x.ld, groups
    p.eps, p.silu, p.dtype = eps, 0, dtype_code(dt)
    p.sync_counter = _ptr(counters)
    return Op(name + ".scale_shift", lib.sfb_group_norm_scale_shift, (C.byref(p), _ptr(scale_shift)),
              (p, x.buf, gamma, beta, stats, counters, scale_shift), 0, x.rows * x.c * 2)


def ln_op(name, lib, *, x, y, rows, c, gamma, beta, eps, dt, ldx=None, ldy=None):
    p = LnParams()
    p.x, p.y = _ptr(x), _ptr(y)
    p.gamma, p.beta = _ptr(gamma), _ptr(beta)
    p.rows, p.c, p.ldx, p.ldy = rows, c, ldx or c, ldy or c
    p.eps, p.dtype = eps, dtype_code(dt)
    return Op(name, lib.sfb_layer_norm, (C.byref(p),), (p, x, y, gamma, beta), 0, 4 * rows * c)


def small_linear_op(name, lib, *, x, w, bias, batch, n, k, dt, y16=None, y32=None, add16=None,
                    act_in=0, act_out=0, ldx=None, ldy=None):
    p = SmallLinearParams()
    p.x, p.w = _ptr(x), _ptr(w)
    p.bias, p.add16, p.y16, p.y32 = _ptr(bias), _ptr(add16), _ptr(y16), _ptr(y32)
    p.batch, p.n, p.k, p.ldx, p.ldy = batch, n, k, ldx or k, ldy or n
    p.act_in, p.act_out, p.dtype = act_in, act_out, dtype_code(dt)
    return Op(name, lib.sfb_small_linear, (C.byref(p),), (p, x, w, bias, add16, y16, y32),
              2 * batch * n * k, 2 * n * k)


def conv_small_op(name, lib, *, x, weight, bias, y: Act, n, h, w, cin, cout, stride, dt, ldx=0, x_nchw=False,
                  silu=False):
    """sfb_conv3x3_small: 3x3 pad-1 conv of a few-channel input (NCHW tensor `x` when x_nchw, else an NHWC
    buffer with channel pitch ldx) into the NHWC activation y; `weight` packed by
    PackedWeights.conv3x3_small ([cout, 3, 3, cin16])."""
    p = _lib.ConvSmallParams()
    p.x, p.weight, p.bias, p.y = _ptr(x), _ptr(weight), _ptr(bias), y.ptr
    p.n, p.h, p.w, p.cin, p.cout, p.stride = n, h, w, cin, cout, stride
    p.ldx, p.ldy = ldx, y.ld
    p.x_nchw, p.silu, p.dtype = int(bool(x_nchw)), int(bool(silu)), dtype_code(dt)
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    return Op(name, lib.sfb_conv3x3_small, (C.byref(p),), (p, x, weight, bias, y.buf),
              2 * n * ho * wo * cout * 9 * cin, 2 * (n * h * w * cin + n * ho * wo * cout))


def conv_small_ex_op(name, lib, *, x, weight, bias, y: Act, n, h, w, cin, cout, dt, in_xform=0, relu=False):
    """sfb_conv3x3_small_ex: stride-1 3x3 pad-1 conv of the NCHW few-channel tensor `x` with the input transform
    `in_xform` (_lib.XFORM_*) on in-image values and an optional ReLU, into the NHWC activation y; `weight` packed
    by PackedWeights.conv3x3_small."""
    p = _lib.ConvSmallExParams()
    b = p.base
    b.x, b.weight, b.bias, b.y = _ptr(x), _ptr(weight), _ptr(bias), y.ptr
    b.n, b.h, b.w, b.cin, b.cout, b.stride = n, h, w, cin, cout, 1
    b.ldx, b.ldy, b.x_nchw, b.silu, b.dtype = 0, y.ld, 1, 0, dtype_code(dt)
    p.in_xform, p.relu = in_xform, int(bool(relu))
    return Op(name, lib.sfb_conv3x3_small_ex, (C.byref(p),), (p, x, weight, bias, y.buf),
              2 * n * h * w * cout * 9 * cin, 2 * (n * h * w * cin + n * h * w * cout))


def c64_out_hw(mode, h, w):
    """Output size of sfb_conv3x3_c64 in `mode` (_lib.C64_*) for an h x w input."""
    if mode == _lib.C64_STRIDE2:
        return (h + 1) // 2, (w + 1) // 2
    if mode == _lib.C64_UP2X:
        return 2 * h, 2 * w
    return h, w


def conv_c64_op(name, lib, *, x: Act, weight, bias, y: Act, mode, dt, relu=False, residual: Act = None):
    """sfb_conv3x3_c64: y = relu?(conv3x3(x) + bias (+ residual)) with 64 input and output channels; `mode`
    (_lib.C64_*) picks stride 1, stride 2 or nearest-2x upsample first; `weight` packed like
    PackedWeights.conv3x3_plain ([64, 576]); `bias` fp32 [64] or None."""
    assert x.c == y.c == 64 and (residual is None or residual.c == 64), (x.c, y.c)
    if (y.n, y.h, y.w) != (x.n,) + c64_out_hw(mode, x.h, x.w):
        raise ValueError(f"{name}: output {y.n}x{y.h}x{y.w} does not match mode {mode} of a {x.n}x{x.h}x{x.w} input")
    p = _lib.ConvC64Params()
    p.x, p.weight, p.bias, p.y = x.ptr, _ptr(weight), _ptr(bias), y.ptr
    p.residual = residual.ptr if residual is not None else None
    p.n, p.h, p.w = x.n, x.h, x.w
    p.ldx, p.ldy, p.ldr = x.ld, y.ld, residual.ld if residual is not None else 0
    p.mode, p.relu, p.dtype = mode, int(bool(relu)), dtype_code(dt)
    nbytes = 2 * 64 * (x.rows + y.rows * (2 if residual is not None else 1))
    return Op(name, lib.sfb_conv3x3_c64, (C.byref(p),),
              (p, x.buf, weight, bias, residual.buf if residual is not None else None, y.buf),
              2 * y.rows * 64 * 9 * 64, nbytes)


def conv_out_temporal_op(name, lib, *, x: Act, w, bias, wt, bt, out, frames, dt):
    """sfb_conv_out_temporal: NCHW out [n, cout, H, W] = time_conv_out(conv_out(x)) over videos of `frames`
    frames; `w` packed like PackedWeights.conv3x3_plain, `wt` like PackedWeights.time_conv_out."""
    cout = out.shape[1]
    return Op(name, lib.sfb_conv_out_temporal,
              (x.ptr, _ptr(w), _ptr(bias), _ptr(wt), _ptr(bt), _ptr(out), x.n, x.h, x.w, x.c, cout, x.ld, frames,
               dtype_code(dt)),
              (x.buf, w, bias, wt, bt, out), 2 * x.rows * cout * (9 * x.c + 3 * cout),
              2 * (x.rows * x.c + out.numel()))


def nhwc_to_nchw_scaled_op(name, lib, *, srcs, dsts, scale, dt):
    """sfb_nhwc_to_nchw_scaled: dsts[i] (NCHW tensors) = scale[i] * srcs[i] (NHWC Acts), one launch."""
    assert 0 < len(srcs) == len(dsts) <= 16
    p = _lib.NhwcToNchwParams()
    p.count, p.dtype, p.scale = len(srcs), dtype_code(dt), _ptr(scale)
    for i, (s, d) in enumerate(zip(srcs, dsts)):
        it = p.items[i]
        it.src, it.dst, it.n, it.c, it.hw, it.ld_src = s.ptr, _ptr(d), s.n, s.c, s.h * s.w, s.ld
    return Op(name, lib.sfb_nhwc_to_nchw_scaled, (C.byref(p),), (p, scale, [s.buf for s in srcs], list(dsts)),
              0, sum(4 * d.numel() for d in dsts))


# ---------------------------------------------------------------------------------------------
# weight packing (done once at plan-build time)
# ---------------------------------------------------------------------------------------------
class Mat:
    """A GEMM B operand: logical [n, k] weight stored TILED in HBM -- tile (n_tile, k_block) is one
    contiguous 160 x 64 block (20 KB), so each TMA box is a single contiguous DRAM stream instead
    of 160 rows strided by k -- plus its TMA map (2-D view [tiles*160, 64], box 160 rows)."""
    __slots__ = ("data", "map", "n", "k", "_dry", "_rows", "_maps")

    def __init__(self, w, dry=False):
        n, k = w.shape
        assert k % BK == 0, f"weight K={k} must be a multiple of {BK}"
        nt, nkb = (n + BN - 1) // BN, k // BK
        self.n, self.k = n, k
        if w.device.type == "meta":
            self.data = torch.empty(nt * nkb * BN, BK, dtype=w.dtype, device="meta")
        else:
            wp = torch.zeros(nt * BN, k, dtype=w.dtype, device=w.device)
            wp[:n] = w
            self.data = wp.view(nt, BN, nkb, BK).permute(0, 2, 1, 3).contiguous().view(-1, BK)
        self._dry = dry
        self._rows = nt * nkb * BN
        self._maps = {}
        self.map = self.map_for(1)

    def map_for(self, cluster_m):
        """TMA map whose box is 1/cluster_m of a weight tile (each CTA of a cluster along M loads
        its slice and multicasts it to the others)."""
        if cluster_m not in self._maps:
            m = matrix_map(_ptr(self.data), self._rows, BK, BK, BN // cluster_m, self._dry)
            m.keep = self.data  # the map alone keeps the tiled copy alive
            self._maps[cluster_m] = m
        return self._maps[cluster_m]



class PlainB:
    """A GEMM B operand that is a plain row-major [n, k] 16-bit matrix in device memory (an
    activation: Q K^T, P V), addressed by a 2-D TMA map instead of the tiled weight layout."""
    __slots__ = ("ptr", "n", "k", "pitch", "_dry", "_maps")

    def __init__(self, ptr, n, k, pitch, dry=False):
        assert k % BK == 0, f"K={k} must be a multiple of {BK}"
        self.ptr, self.n, self.k, self.pitch, self._dry, self._maps = ptr, n, k, pitch, dry, {}

    def map_for(self, cluster_m):
        if cluster_m not in self._maps:
            self._maps[cluster_m] = matrix_map(self.ptr, self.n, self.k, self.pitch, BN // cluster_m, self._dry)
        return self._maps[cluster_m]


def pack_conv3x3(w, dt):
    """[cout, cin, 3, 3] -> K-major [cout, (kh, kw, cin)]"""
    return w.detach().permute(0, 2, 3, 1).reshape(w.shape[0], -1).to(dt).contiguous()


# 3x3 taps of the upsampled image that read the same source pixel: S[(phase, tap)]
_UP_TAPS = {(0, 0): (0,), (0, 1): (1, 2), (1, 0): (0, 1), (1, 1): (2,)}


def pack_upconv(w, dt):
    """Nearest-2x upsample + conv3x3 as four 2x2 convolutions on the source image (one per output
    phase (py, px)): [cout, cin, 3, 3] -> [4 * Np, 4 * cin], Np = cout rounded up to 160, phase p =
    2*py + px in rows [p*Np, p*Np + cout), K order (ty, tx, cin).  Tap (ty, tx) of phase (py, px)
    reads source offset (py-1+ty, px-1+tx) and carries the SUM (in fp32) of the 3x3 weights whose
    upsampled-image taps fall on that source pixel."""
    cout, cin = w.shape[0], w.shape[1]
    npad = (cout + BN - 1) // BN * BN
    if w.device.type == "meta":
        return torch.empty(4 * npad, 4 * cin, dtype=dt, device="meta")
    wf = w.detach().float()
    out = torch.zeros(4 * npad, 4 * cin, dtype=torch.float32, device=w.device)
    for py in range(2):
        for px in range(2):
            r0 = (2 * py + px) * npad
            for ty in range(2):
                for tx in range(2):
                    acc = sum(wf[:, :, kh, kw] for kh in _UP_TAPS[(py, ty)] for kw in _UP_TAPS[(px, tx)])
                    c0 = (2 * ty + tx) * cin
                    out[r0:r0 + cout, c0:c0 + cin] = acc
    return out.to(dt).contiguous()


def fold_pointwise_into_conv(w, b, w_pw, b_pw):
    """A conv (w [c1, cin, kh, kw], b [c1]) followed by a 1x1 conv (w_pw [c2, c1, 1, 1], b_pw [c2]) as ONE
    conv: W = W_pw . W, b = W_pw . b + b_pw, formed in fp32 (fp64 stays fp64) before any rounding."""
    dt = torch.promote_types(w.dtype, torch.float32)
    wq = w_pw.detach().to(dt).reshape(w_pw.shape[0], -1)
    wf = torch.einsum("qo,ochw->qchw", wq, w.detach().to(dt))
    bf = wq @ b.detach().to(dt) + b_pw.detach().to(dt)
    return wf, bf


def pack_conv_in(w, dt):
    """[cout, cin, 3, 3] -> [(kh, kw, cin), cout] (tap-major, cout contiguous) for sfb_conv_in"""
    return w.detach().permute(2, 3, 1, 0).reshape(-1, w.shape[0]).to(dt).contiguous()


def pack_geglu(w, b, dt, extra=None):
    """GEGLU projection [2*inner, k] (value rows first, gate rows second; reference chunk order
    /root/reference/src/sfast/jit/passes/__init__.py:643-648) -> tile-interleaved
    [ceil(inner/80)*160, k]: per 160-row tile, 80 value rows then the matching 80 gate rows.
    `extra`: optional per-row fp32 vector permuted the same way (LayerNorm-fold column sums).
    One gather per tensor (no per-tile loop: packing is on the first-call latency path)."""
    inner = w.shape[0] // 2
    half = BN // 2
    tiles = (inner + half - 1) // half
    # source row of every packed row; rows past `inner` inside the last tile point at a zero row
    j = torch.arange(tiles * BN, device=w.device)
    t, r = j // BN, j % BN
    col = t * half + (r % half)                      # output column of the packed row
    src = torch.where(r < half, col, col + inner)   # value row | gate row of that column
    valid = col < inner
    src = torch.where(valid, src, torch.full_like(src, 2 * inner))  # -> appended zero row

    def gather(v, dtype):
        pad = torch.zeros((1,) + tuple(v.shape[1:]), dtype=dtype, device=w.device)
        return torch.cat([v.detach().to(dtype), pad], 0).index_select(0, src).contiguous()

    wp = gather(w, dt)
    bp = gather(b, torch.float32) if b is not None else torch.zeros(tiles * BN, dtype=torch.float32,
                                                                     device=w.device)
    if extra is not None:
        return wp, bp, inner, gather(extra, torch.float32)
    return wp, bp, inner


_ANY_DTYPE = {torch.float16: _lib.SFB_F16, torch.bfloat16: _lib.SFB_BF16, torch.float32: _lib.SFB_F32}


def lora_merge_params(w, adapters, out):
    """Validated sfb_lora_merge argument block for out = round(w + sum_i s_i * B_i A_i).  w: [n, k] (fp16 / bf16 /
    fp32, unit column stride); adapters: 1..8 tuples (A [r, k], B [n, r], s) with 1 <= r <= 256, A and B each fp16
    / bf16 / fp32; out: fp16 / bf16 [n, k], unit column stride, sharing no memory with the inputs.  Row pitches
    are taken from the tensors' strides.  Raises ValueError naming what is wrong."""
    if w.dim() != 2 or out.dim() != 2 or tuple(out.shape) != tuple(w.shape):
        raise ValueError(f"lora_merge: W {tuple(w.shape)} and out {tuple(out.shape)} must be the same 2-D shape")
    n, k = w.shape
    if w.dtype not in _ANY_DTYPE or out.dtype not in (torch.float16, torch.bfloat16):
        raise ValueError(f"lora_merge: W {w.dtype} must be fp16 / bf16 / fp32 and out {out.dtype} fp16 / bf16")
    if not 1 <= len(adapters) <= _lib.LORA_MAX_ADAPTERS:
        raise ValueError(f"lora_merge: {len(adapters)} adapters; 1..{_lib.LORA_MAX_ADAPTERS} per launch")
    mats = [w, out]
    p = _lib.LoraMergeParams()
    for i, (a, b, s) in enumerate(adapters):
        if a.dim() != 2 or b.dim() != 2:
            raise ValueError(f"lora_merge: adapter {i}: A and B must be 2-D")
        r = a.shape[0]
        if tuple(a.shape) != (r, k) or tuple(b.shape) != (n, r):
            raise ValueError(f"lora_merge: adapter {i}: A {tuple(a.shape)} / B {tuple(b.shape)} do not fit W "
                             f"{(n, k)}: expected A [r, {k}] and B [{n}, r]")
        if not 1 <= r <= _lib.LORA_MAX_RANK:
            raise ValueError(f"lora_merge: adapter {i}: rank {r}; 1..{_lib.LORA_MAX_RANK}")
        if a.dtype not in _ANY_DTYPE or b.dtype not in _ANY_DTYPE:
            raise ValueError(f"lora_merge: adapter {i}: A {a.dtype} / B {b.dtype} must be fp16 / bf16 / fp32")
        ad = p.adapters[i]
        ad.a, ad.b, ad.rank, ad.lda, ad.ldb = _ptr(a), _ptr(b), r, a.stride(0), b.stride(0)
        ad.a_dtype, ad.b_dtype, ad.scale = _ANY_DTYPE[a.dtype], _ANY_DTYPE[b.dtype], float(s)
        mats += [a, b]
    for t in mats:
        if t.stride(1) != 1 and t.shape[1] > 1:
            raise ValueError("lora_merge: every operand needs unit column stride (rows may be pitched)")
        if t.device != w.device:
            raise ValueError(f"lora_merge: operands on {t.device} and {w.device}")
    if any(out.untyped_storage().data_ptr() == t.untyped_storage().data_ptr() for t in mats[:1] + mats[2:]):
        raise ValueError("lora_merge: out shares memory with W, A or B")
    p.w, p.out, p.n, p.k, p.ldw, p.ldo = _ptr(w), _ptr(out), n, k, w.stride(0), out.stride(0)
    p.w_dtype, p.out_dtype, p.count = _ANY_DTYPE[w.dtype], dtype_code(out.dtype), len(adapters)
    return p


def lora_merge(w, adapters, out_dtype):
    """sfb_lora_merge on the current stream into a new [n, k] tensor of out_dtype (see lora_merge_params)."""
    out = torch.empty(w.shape, dtype=out_dtype, device=w.device)
    p = lora_merge_params(w, adapters, out)
    check(_lib.lib().sfb_lora_merge(C.byref(p), torch.cuda.current_stream(w.device).cuda_stream), "sfb_lora_merge")
    return out


def fold_layer_norm(w, b, gamma, beta, dt):
    """Fold LayerNorm(gamma, beta) into the following linear layer y = LN(x) W^T + b:
    returns (W' = W * gamma in the 16-bit type, bias' = beta W^T + b, colsum = sum_k W'[n, k]
    taken from the ROUNDED W' so that the epilogue's mean correction matches the MMA exactly)."""
    wf = w.detach().float()
    wp = (wf * gamma.detach().float()[None, :]).to(dt)
    colsum = wp.float().sum(dim=1)
    bias = wf @ beta.detach().float()
    if b is not None:
        bias = bias + b.detach().float()
    return wp, bias.contiguous(), colsum.contiguous()
