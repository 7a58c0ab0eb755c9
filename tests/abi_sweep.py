"""Boundary sweep of the geometry the C ABI accepts, against a float64 reference.

``kernel_checks.py`` runs hand-picked shapes and ``plan_launches.py`` replays what the shipped plans emit.
Neither reaches the edges of what each entry point's host validation *accepts*: a head_dim the dispatch
compiles that no plan uses, a K loop one block longer than the GEMM's 6-stage ring, a last KV tile that
holds one key, a 1 x 1 image in a multi-image conv box.  This module holds a frozen list of such cases,
each built as a dry launch descriptor by the project's own op builders (`sfast_b200.ops`), and runs them
with the replays, float64 references, sentinel canvases and tolerance table of ``plan_launches.py``:

  * every output goes into a sentinel-filled buffer with a leading offset, a pitch gap where the entry
    point takes a pitch, and guard rows; a case passes only if all of that comes back bit-for-bit;
  * attention inputs carry large finite garbage (not zeros) in the padding rows of Q / K / K_ip and the
    padding columns of V^T, so a mask that lets one padding key through fails;
  * ``ONE_STEP_OUTSIDE`` lists, per boundary, a launch one step past what the kernels compute; the CPU
    test checks that each is refused with SFB_ERR_INVALID and an error naming the field.

    python tests/abi_sweep.py [--family NAME ...] [--json out.json] [--list]

prints one JSON line per case (id, entry point, parameters, error, tolerance, pass) and a summary of the
largest error per entry point.
"""
import argparse
import contextlib
import ctypes as C
import hashlib
import json
import math
import os
import sys
import time

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
if _HERE not in sys.path:
    sys.path.insert(0, _HERE)

import plan_launches as pl  # noqa: E402  (also puts the package on sys.path)
from plan_launches import DEV, Canvas, Result, TensorMap, rel_err, tol  # noqa: E402
from sfast_b200 import _lib, ops  # noqa: E402
from sfast_b200.plan import _DryLib  # noqa: E402

F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32
BOTH = (F16, BF16)
GARBAGE = 300.0   # magnitude of the padding garbage in the attention operands (finite: 0 * garbage = 0)
IP_SCALE = 0.75


def _meta(*shape, dt=F16):
    return torch.empty(shape, dtype=dt, device="meta")


def _rup(x, m):
    return (x + m - 1) // m * m


def _dn(dt):
    return "bf16" if dt == BF16 else "fp16"


class Case:
    """One sweep launch: `build()` returns a dry ops.Op (pointers are byte offsets inside their buffers);
    `run` is the replay (default: plan_launches.REPLAY of the entry point); `peaked` also runs it with
    score std ~8."""
    __slots__ = ("cid", "family", "params", "build", "run", "peaked")

    def __init__(self, family, params, build, run=None, peaked=False):
        self.family, self.params, self.build, self.run, self.peaked = family, params, build, run, peaked
        self.cid = family + ":" + ",".join(f"{k}={v}" for k, v in params.items())

    def op(self):
        with pl.recording_map_offsets():
            return self.build()


# =====================================================================================================
# op builders (dry: meta tensors sit at address 0, so a pointer is its byte offset)
# =====================================================================================================
def attn_op(hd, kv, sq, skv, dt, *, q_rows=None, k_rows=None, scale=None, causal=False, ip=None, batch=2,
            heads=2, out_off=0):
    """sfb_attention (or, with ip = (seq_ip, k_ip_rows), sfb_attention_ip) over Q [bh, q_rows, pitch], K
    [bh, k_rows, pitch] and V^T [bh, vt_rows, round64(seq_kv)]."""
    q_pitch, vt_rows, vt_pitch = ops.tk_cols(hd), _rup(hd + 1, 16), _rup(skv, 64)
    ipd = None
    if ip is not None:
        ipd = dict(k=_meta(1), vt=_meta(1), seq=ip[0], k_rows=ip[1], vt_pitch=kv, scale=_meta(1, dt=F32))
    op = ops.attention_op("sweep", _DryLib, q=_meta(1), k=_meta(1), vt=_meta(1), out=out_off, batch=batch,
                          heads=heads, head_dim=hd, seq_q=sq, seq_kv=skv, q_rows=q_rows or sq,
                          k_rows=k_rows or skv, vt_rows=vt_rows, q_pitch=q_pitch, vt_pitch=vt_pitch, dt=dt,
                          dry=True, kv_tile=kv, causal=causal, ip=ipd)
    if scale is not None:
        (op.keep[0].base if ip is not None else op.keep[0]).scale = scale
    return op


def gemm_op(M, N, K, dt, *, splits=1, ldo=None, out_off=0, bias=True, residual=False, ldr=None, act=0,
            rowstats=False, epi=_lib.EPI_STORE, geglu_n_out=0, qkv=None, a_pitch=None, defer=False):
    """sfb_gemm with SFB_A_MATRIX: A [M, K] (pitch a_pitch), the tiled weight of an [N, K] matrix."""
    ws = _meta(splits * M * N, dt=F32) if splits > 1 else None
    op = ops.gemm_op("sweep", _DryLib, M=M, N=N, K=K, dt=dt, a=ops.a_matrix(0, M, K, a_pitch or K),
                     b=ops.Mat(_meta(N, K, dt=dt), dry=True), out=None if epi == _lib.EPI_QKV else out_off,
                     ldo=ldo or N, bias=_meta(N, dt=F32) if bias else None, residual=0 if residual else None,
                     ldr=ldr or 0, act=act, epi=epi, geglu_n_out=geglu_n_out, qkv=qkv, ws=ws, splits=splits,
                     rowstats_out=_meta(M, ops.rowstats_slots(N), 2, dt=F32) if rowstats else None, dry=True,
                     cta_pair=False, persistent=False)
    op.keep[0].defer_finish = int(defer)
    return op


def qkv_op(heads, hd, batch, seq, dt, which_base=0, K=128):
    n_which = 3 - which_base
    qkv = dict(q=_meta(1), k=_meta(1), vt=_meta(1), heads=heads, head_dim=hd, which_base=which_base, seq=seq,
               q_pitch=ops.tk_cols(hd), q_rows=seq, k_rows=seq, vt_rows=_rup(hd + 1, 16), vt_pitch=_rup(seq, 64))
    return gemm_op(batch * seq, n_which * heads * hd, K, dt, epi=_lib.EPI_QKV, qkv=qkv)


def conv_op(mode, n, h, w, cin, N, dt, *, stride=1, rowbias=False, residual=False, ldo=None, silu=True,
            out_off=0, ld_in=None, rowbias_off=16):
    """A convolution A mode on n images.  (h, w): the INPUT of "conv3x3" (stride 1 or 2), the OUTPUT of
    "down" (input 2h x 2w), the SOURCE of "up" (output 2h x 2w), (frames, pixels) of "temporal" (n videos),
    the input = output of "halo" (GroupNorm folded into the conv)."""
    ld_in = ld_in or cin
    conv, kw = None, {}
    if mode == "halo":
        a = ops.a_conv_halo(0, n, h, w, cin, ld_in)
        conv = dict(n=n, h=h, w=w, cin=cin, stride=1, box_n=1, box_h=ops.HALO_BOX_H, box_w=ops.HALO_BOX_W)
        kw["gn"] = dict(scale_shift=_meta(n, cin, 2, dt=F32), silu=silu)
        M, K, wrows = n * h * w, 9 * cin, N
    elif mode == "up":
        bn, bh, bw = ops.conv_tile_box(h, w)
        a = ops.a_conv(0, n, h, w, cin, ld_in, bn, bh, bw, 1)
        conv = dict(n=n, h=h, w=w, cin=cin, stride=1, box_n=bn, box_h=bh, box_w=bw, up=True)
        M, K, wrows = 4 * n * h * w, 4 * cin, 4 * _rup(N, ops.BN)
    elif mode == "temporal":
        bn, bh, bw = ops.conv_tile_box(h, w)
        a = ops.a_conv(0, n, h, w, cin, ld_in, bn, bh, bw, 1)
        conv = dict(n=n, h=h, w=w, cin=cin, stride=1, box_n=bn, box_h=bh, box_w=bw, temporal=True)
        M, K, wrows = n * h * w, 3 * cin, N
    elif mode == "down":
        bn, bh, bw = ops.conv_tile_box(h, w)
        a = ops.a_conv(0, n, 2 * h, 2 * w, cin, ld_in, bn, bh, bw, 2)
        conv = dict(n=n, h=h, w=w, cin=cin, stride=2, box_n=bn, box_h=bh, box_w=bw, down=True)
        M, K, wrows = n * h * w, 9 * cin, N
    else:
        ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
        bn, bh, bw = ops.conv_tile_box(ho, wo)
        a = ops.a_conv(0, n, h, w, cin, ld_in, bn, bh, bw, stride)
        conv = dict(n=n, h=ho, w=wo, cin=cin, stride=stride, box_n=bn, box_h=bh, box_w=bw)
        M, K, wrows = n * ho * wo, 9 * cin, N
    if rowbias:
        kw.update(rowbias=rowbias_off, rows_per_img=M // n, ld_rowbias=N + 8)
    return ops.gemm_op("sweep", _DryLib, M=M, N=N, K=K, dt=dt, a=a, b=ops.Mat(_meta(wrows, K, dt=dt), dry=True),
                       out=out_off, ldo=ldo or N, bias=_meta(N, dt=F32), residual=0 if residual else None,
                       ldr=(N + 16) if residual else 0, conv=conv, splits=1, dry=True, cta_pair=False,
                       persistent=False, **kw)


def gn_op(kind, n, hw, c, groups, dt, *, silu=False, eps=1e-5):
    """GroupNorm over x [n, hw, c] (channel pitch c + 8, 8 elements of leading offset) into y (pitch c + 16):
    kind "two_pass" (stats -> apply), "fused" (single cooperative launch) or "scale_shift"."""
    x = ops.Act(_meta(1), n, hw, 1, c, ld=c + 8, off=8)
    y = ops.Act(_meta(1), n, hw, 1, c, ld=c + 16, off=24)
    common = dict(x=x, gamma=_meta(c, dt=F32), beta=_meta(c, dt=F32), stats=_meta(1, dt=F32), groups=groups,
                  eps=eps, dt=dt)
    if kind == "scale_shift":
        return ops.gn_scale_shift_op("sweep", _DryLib, counters=_meta(n, dt=torch.int32),
                                     scale_shift=_meta(n, c, 2, dt=F32), **common)
    sync = _meta(n, dt=torch.int32) if kind == "fused" else None
    got = ops.gn_ops("sweep", _DryLib, y=y, silu=silu, sync=sync, dry=True, **common)[0]
    if kind == "fused" and got.fn.name != "sfb_group_norm_fused":
        raise AssertionError(f"GroupNorm n={n} hw={hw} c={c} does not take the fused kernel")
    return got


def gn_params(n, hw, c, groups, ldx=None):
    p = _lib.GnParams()
    p.n, p.hw, p.c, p.ldx, p.ldy, p.groups, p.dtype = n, hw, c, ldx or c, ldx or c, groups, _lib.SFB_F16
    return p


def fused_hw_limit(n, c, groups):
    """Largest hw sfb_group_norm_fused_fits accepts for n images of c channels (on this device)."""
    lib = _lib.lib()
    lo, hi = 1, 1 << 20
    if not lib.sfb_group_norm_fused_fits(C.byref(gn_params(n, lo, c, groups))):
        raise AssertionError("not even hw = 1 fits")
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if lib.sfb_group_norm_fused_fits(C.byref(gn_params(n, mid, c, groups))):
            lo = mid
        else:
            hi = mid
    return lo


def ln_op(rows, c, dt):
    return ops.ln_op("sweep", _DryLib, x=_meta(1), y=_meta(1), rows=rows, c=c, gamma=_meta(c, dt=F32),
                     beta=_meta(c, dt=F32), eps=1e-5, dt=dt, ldx=c + 8, ldy=c + 24)


def temporal_op(frames, seq, dt, heads=2, batch=2, hd=64):
    p = _lib.TemporalAttnParams()
    p.batch, p.frames, p.seq, p.heads, p.head_dim = batch, frames, seq, heads, hd
    p.ld_qkv, p.ld_out, p.dtype, p.scale = 3 * heads * hd + 8, heads * hd + 16, ops.dtype_code(dt), 1 / math.sqrt(hd)
    return ops.Op("sweep", _DryLib.sfb_temporal_attention, (C.byref(p),), (p,))


def small_linear_op(batch, n, k, dt, *, act=0, y32=False):
    return ops.small_linear_op("sweep", _DryLib, x=_meta(1), w=_meta(1), bias=_meta(n, dt=F32), batch=batch, n=n,
                               k=k, dt=dt, y16=None if y32 else _meta(1), y32=_meta(1, dt=F32) if y32 else None,
                               add16=_meta(1), act_in=act, act_out=act, ldx=k + 8, ldy=n + 8)


def row_op(name, rows, c, dt, *, rowstats=False):
    p = _lib.RowOpParams()
    p.x, p.y = 16, 32
    p.rows, p.c, p.ldx, p.ldx2, p.ldv, p.ldy, p.dtype = rows, c, c + 8, c + 16, c, c + 24, ops.dtype_code(dt)
    p.mode, p.div, p.mod = _lib.ROW_IDX_DIV_MOD, 2, 3
    p.rowstats_slots = 2 if rowstats else 0
    blend = name == "sfb_alpha_blend"
    vec, x2, mix = (None, 0, _meta(1, dt=F32)) if blend else (_meta(1), None, None)
    rs = _meta(1, dt=F32) if rowstats else None
    return ops.Op("sweep", getattr(_DryLib, name), (C.byref(p),), (p, None, None, vec, x2, mix, rs))


def plain_op(name, **kw):
    """A plain-argument launch; `kw` by plan_launches.PLAIN argument name (pointers: byte offsets)."""
    return ops.Op("sweep", getattr(_DryLib, name), tuple(kw[a] for a in pl.PLAIN[name]), ())


# =====================================================================================================
# replays this sweep needs beyond plan_launches.REPLAY
# =====================================================================================================
def _garbage(*shape, dt):
    """Large finite values: what a padding row holds after some other kernel used the buffer."""
    return (torch.randn(*shape, device=DEV) * GARBAGE).to(dt)


def run_attention(op, peaked=False):
    """sfb_attention / sfb_attention_ip with garbage in every padding row of Q / K / K_ip, every V^T column past
    the sequence and every V^T row past the ones row (columns past head_dim are zero, as the QKV-scatter
    epilogue leaves them in the plans' zeroed buffers)."""
    ip = op.fn.name == "sfb_attention_ip"
    P = pl._clone(op.keep[0])
    p = P.base if ip else P
    tq, tk, tv = op.keep[6:9] if ip else op.keep[1:4]
    dt = pl.DTYPES[p.dtype]
    B, H, D = p.batch, p.heads, p.head_dim
    bh, sq, skv = B * H, p.seq_q, p.seq_kv
    q_pitch, vt_pitch = tq.geom[2], tv.geom[2]

    def operand(rows, valid, pitch, scale=1.0):
        t = _garbage(bh, rows, pitch, dt=dt)
        t[..., D:] = 0
        t[:, :valid, :D] = pl._randn(bh * valid * D, dt, scale).view(bh, valid, D)
        return t

    qf = operand(p.q_rows, sq, q_pitch, 8.0 if peaked else 1.0)
    kf = operand(p.k_rows, skv, q_pitch)
    vf = _garbage(bh, p.vt_rows, vt_pitch, dt=dt)
    vf[:, :D, :skv] = pl._randn(bh * D * skv, dt).view(bh, D, skv)
    vf[:, D, :] = 1.0
    maps = [TensorMap.matrix(t.data_ptr(), *g.geom[1:]) for t, g in ((qf, tq), (kf, tk), (vf, tv))]
    p.tmap_q, p.tmap_k, p.tmap_vt = (m.ptr for m in maps)
    q, k, v = qf[:, :sq, :D].double(), kf[:, :skv, :D].double(), vf[:, :D, :skv].double().transpose(1, 2)
    ref = pl.ref_attention(q, k, v, float(p.scale), bool(p.causal))
    if ip:
        tki, tvi = op.keep[1], op.keep[2]
        sip = P.seq_ip
        kif = operand(P.k_ip_rows, sip, tki.geom[2])
        vif = _garbage(bh, p.vt_rows, tvi.geom[2], dt=dt)
        vif[:, :D, :sip] = pl._randn(bh * D * sip, dt).view(bh, D, sip)
        maps += [TensorMap.matrix(kif.data_ptr(), *tki.geom[1:]), TensorMap.matrix(vif.data_ptr(), *tvi.geom[1:])]
        P.tmap_k_ip, P.tmap_vt_ip = maps[3].ptr, maps[4].ptr
        s_ip = torch.full((1,), IP_SCALE, device=DEV)
        P.ip_scale = s_ip.data_ptr()
        ref = ref + IP_SCALE * pl.ref_attention(q, kif[:, :sip, :D].double(),
                                                vif[:, :D, :sip].double().transpose(1, 2), float(p.scale), False)
    out = Canvas(dt, pl._off(p.out, 2), B * sq, H * D)
    p.out = out.ptr
    out.arm()
    fn = _lib.lib().sfb_attention_ip if ip else _lib.lib().sfb_attention
    _lib.check(fn(C.byref(P), pl._stream()), op.fn.name)
    torch.cuda.synchronize()
    res = Result()
    ref = ref.view(B, H, sq, D).permute(0, 2, 1, 3).reshape(B * sq, H * D)
    res.add("out", rel_err(out.take(out.region(B * sq, H * D)), ref), tol("attention", dt))
    res.canary(out)
    return res


TIMESTEPS = (999.0, 0.5, 0.0, 1.0, 617.375)


def run_timestep(op, peaked=False):
    """sfb_timestep_embed at fixed timesteps: the last training step, fractional ones and zero."""
    a = dict(zip(pl.PLAIN["sfb_timestep_embed"], op.args))
    B, dim, ldo, dt = a["batch"], a["dim"], a["ldo"], pl.DTYPES[a["dtype"]]
    t = torch.tensor(TIMESTEPS[:B], device=DEV)
    out = Canvas(dt, int(a["out*"] or 0) // 2, B, ldo)
    out.arm()
    _lib.check(_lib.lib().sfb_timestep_embed(t.data_ptr(), B, dim, a["flip"], a["shift"], out.ptr, ldo, a["dtype"],
                                             pl._stream()), "sfb_timestep_embed")
    torch.cuda.synchronize()
    res = Result()
    ref = pl.ref_timestep_embed(t.double(), dim, a["flip"], a["shift"])
    res.add("out", rel_err(out.take(out.region(B, dim)), ref), tol("timestep", dt))
    res.canary(out)
    return res


# =====================================================================================================
# the cases
# =====================================================================================================
# every (head_dim, kv_tile) pair attention_dispatch compiles
ATTN_PAIRS = ((32, 64), (40, 64), (64, 64), (160, 64), (32, 128), (40, 128), (64, 128), (160, 128), (80, 128),
              (128, 128))
SEQ_Q = (1, 63, 64, 65, 129)
SEQ_KV = (1, 63, 64, 65, 127, 128, 129)
CAUSAL_S = (1, 63, 64, 65, 128, 129)
GEMM_M = (1, 127, 128, 129)
GEMM_N = (8, 152, 160, 168)
K_BLOCKS_PER_SPLIT = (1, 5, 6, 7, 13)   # against the 6-stage ring (kGemmStages)
CONV_IMAGES = ((1, 1), (1, 2), (2, 1), (3, 3))


def _multi_n(h, w, fallback=2):
    """Images enough that a multi-image M-tile box ends ragged (one image in the last tile)."""
    bn = ops.conv_tile_box(h, w)[0]
    return 2 * bn + 1 if bn > 1 else fallback


def attention_cases():
    out = []
    for hd, kv in ATTN_PAIRS:
        for i, skv in enumerate(SEQ_KV):
            sq = SEQ_Q[i % len(SEQ_Q)]
            q_pad, k_pad = (0, 5, 64)[i % 3], (0, 9)[i % 2]
            scale = 0.3 if i == 3 else None
            for dt in BOTH:
                prm = dict(head_dim=hd, kv_tile=kv, seq_q=sq, seq_kv=skv, q_rows=sq + q_pad, k_rows=skv + k_pad,
                           scale=scale or "1/sqrt(D)", dtype=_dn(dt))
                out.append(Case("attention", prm, lambda hd=hd, kv=kv, sq=sq, skv=skv, qp=q_pad, kp=k_pad, s=scale,
                                dt=dt: attn_op(hd, kv, sq, skv, dt, q_rows=sq + qp, k_rows=skv + kp, scale=s,
                                               out_off=8 * (kp + 1)),
                                run_attention, peaked=i in (2, 5)))
    for s in CAUSAL_S:
        for dt in BOTH:
            out.append(Case("attention", dict(head_dim=64, kv_tile=64, causal=1, seq=s, dtype=_dn(dt)),
                            lambda s=s, dt=dt: attn_op(64, 64, s, s, dt, causal=True), run_attention, peaked=s == 65))
    for hd, kv in ((128, 128), (64, 64)):
        for sip in (1, kv):
            for dt in BOTH:
                out.append(Case("attention", dict(entry="ip", head_dim=hd, kv_tile=kv, seq_ip=sip, k_ip_rows=sip + 3,
                                                  dtype=_dn(dt)),
                                lambda hd=hd, kv=kv, sip=sip, dt=dt: attn_op(hd, kv, 65, 77, dt, k_rows=80,
                                                                             ip=(sip, sip + 3)),
                                run_attention))
    return out


def gemm_cases():
    specs = []
    for M in GEMM_M:
        for N in GEMM_N:
            specs.append(dict(M=M, N=N, K=384))
    for b in K_BLOCKS_PER_SPLIT:
        specs.append(dict(M=129, N=168, K=64 * b, a_pitch=64 * b + 64))
        specs.append(dict(M=127, N=152, K=128 * b, splits=2))
    for nkb, s in ((7, 6), (13, 12), (2, 1), (6, 6), (2, 2), (13, 13)):   # ragged, and one K block per split
        specs.append(dict(M=128, N=160, K=64 * nkb, splits=s))
        specs.append(dict(M=1, N=8, K=64 * nkb, splits=s))
    specs += [dict(M=129, N=168, K=384, ldo=200, residual=1, ldr=176, out_off=8),
              dict(M=129, N=168, K=448, splits=3, ldo=184, residual=1, ldr=256),
              dict(M=129, N=168, K=320, act=_lib.ACT_GELU, ldo=176),
              dict(M=127, N=168, K=320, act=_lib.ACT_QUICK_GELU, residual=1, ldr=168),
              dict(M=129, N=168, K=320, rowstats=1),
              dict(M=129, N=168, K=448, splits=3, rowstats=1),
              dict(M=1, N=328, K=128, rowstats=1, splits=2),
              dict(M=129, N=160, K=320, epi=_lib.EPI_GEGLU, geglu_n_out=80),
              dict(M=129, N=160, K=320, epi=_lib.EPI_GEGLU, geglu_n_out=72, ldo=88),
              dict(M=127, N=480, K=384, epi=_lib.EPI_GEGLU, geglu_n_out=232),
              dict(M=129, N=480, K=448, epi=_lib.EPI_GEGLU, geglu_n_out=232, splits=2),
              dict(M=129, N=168, K=320, epi=_lib.EPI_STORE_F32, ldo=172),
              dict(M=1, N=8, K=64, epi=_lib.EPI_STORE_F32)]
    out = []
    for s in specs:
        for dt in BOTH:
            prm = dict(s, dtype=_dn(dt))
            out.append(Case("gemm", prm, lambda s=s, dt=dt: gemm_op(s["M"], s["N"], s["K"], dt,
                                                                    **{k: v for k, v in s.items() if k not in "MNK"})))
    for hd, seq, wb in ((128, 77, 0), (128, 77, 1), (128, 1, 0), (40, 65, 0)):
        for dt in BOTH:
            out.append(Case("gemm", dict(epi="qkv", head_dim=hd, heads=2, batch=2, seq=seq, which_base=wb,
                                         dtype=_dn(dt)),
                            lambda hd=hd, seq=seq, wb=wb, dt=dt: qkv_op(2, hd, 2, seq, dt, wb)))
    return out


def conv_cases():
    specs = []
    for h, w in CONV_IMAGES:
        n = _multi_n(h, w)
        specs.append(dict(mode="conv3x3", n=n, h=h, w=w, cin=64, N=168))
        specs.append(dict(mode="down", n=_multi_n(h, w), h=h, w=w, cin=64, N=152))
        specs.append(dict(mode="up", n=n, h=h, w=w, cin=64, N=168))
        specs.append(dict(mode="temporal", n=n, h=h, w=w, cin=64, N=160))
    specs += [dict(mode="conv3x3", n=3, h=3, w=3, cin=64, N=168, stride=2),
              dict(mode="conv3x3", n=2, h=1, w=1, cin=128, N=8, stride=2),
              dict(mode="conv3x3", n=3, h=3, w=3, cin=64, N=168, rowbias=1, residual=1, ldo=184, out_off=8),
              dict(mode="temporal", n=3, h=2, w=1, cin=64, N=168, rowbias=1, residual=1),
              dict(mode="conv3x3", n=257, h=1, w=1, cin=64, N=8, ld_in=72)]
    for (n, h, w) in ((1, 1, 8), (2, 17, 8), (3, 16, 16)):
        specs.append(dict(mode="halo", n=n, h=h, w=w, cin=64, N=168, silu=int(h != 16)))
    specs.append(dict(mode="halo", n=2, h=3, w=8, cin=128, N=64, residual=1, rowbias=1, silu=1))
    out = []
    for s in specs:
        for dt in BOTH:
            out.append(Case("conv", dict(s, dtype=_dn(dt)), lambda s=s, dt=dt: conv_op(
                s["mode"], s["n"], s["h"], s["w"], s["cin"], s["N"], dt,
                **{k: v for k, v in s.items() if k not in ("mode", "n", "h", "w", "cin", "N")})))
    return out


GN_GEOMS = ((1, 1, 8, 1), (2, 7, 8, 8), (2, 7, 320, 64), (1, 7, 4096, 64), (2, 1, 4096, 1), (3, 7, 4096, 32),
            (2, 1, 64, 8), (2, 5, 64, 64))
GN_FUSED_LIMIT = (1, 4096, 32)   # (n, c, groups) of the largest-tensor case of the fused kernel


def group_norm_cases():
    out = []
    for i, (n, hw, c, g) in enumerate(GN_GEOMS):
        for kind in ("two_pass", "fused", "scale_shift"):
            for dt in BOTH:
                out.append(Case("group_norm", dict(kind=kind, n=n, hw=hw, c=c, groups=g, silu=i % 2, dtype=_dn(dt)),
                                lambda kind=kind, n=n, hw=hw, c=c, g=g, s=i % 2, dt=dt: gn_op(kind, n, hw, c, g, dt,
                                                                                             silu=bool(s))))
    n, c, g = GN_FUSED_LIMIT
    for dt in BOTH:
        out.append(Case("group_norm", dict(kind="fused", n=n, hw="fused_hw_limit", c=c, groups=g, dtype=_dn(dt)),
                        lambda dt=dt: gn_op("fused", n, fused_hw_limit(n, c, g), c, g, dt, silu=True)))
    return out


def layer_norm_cases():
    return [Case("layer_norm", dict(rows=r, c=c, dtype=_dn(dt)), lambda r=r, c=c, dt=dt: ln_op(r, c, dt))
            for c in (8, 2040, 2048) for r in (1, 37) for dt in BOTH]


def temporal_cases():
    return [Case("temporal", dict(frames=f, seq=s, dtype=_dn(dt)), lambda f=f, s=s, dt=dt: temporal_op(f, s, dt))
            for f in (1, 2, 31, 32) for s in (1, 5) for dt in BOTH]


def softmax_cases():
    out = []
    for cols in (8, 16384):
        for rows in (1, 3):
            for f32 in (0, 1):
                for dt in BOTH:
                    alias = rows == 3 and f32 == 1
                    out.append(Case("softmax", dict(rows=rows, cols=cols, x_is_f32=f32, alias=int(alias), dtype=_dn(dt)),
                                    lambda rows=rows, cols=cols, f32=f32, dt=dt, alias=alias: plain_op(
                                        "sfb_row_softmax", **{"x*": 0, "y*": 0 if alias else 16, "rows": rows,
                                                              "cols": cols, "ldx": cols + 8,
                                                              "ldy": 2 * (cols + 8) if alias else cols + 16,
                                                              "x_is_f32": f32, "dtype": ops.dtype_code(dt)}),
                                    peaked=True))
    return out


def edge_cases():
    out = []
    for dt in BOTH:
        d = _dn(dt)
        code = ops.dtype_code(dt)
        for act, y32 in ((0, False), (1, False), (0, True)):
            out.append(Case("edge", dict(entry="small_linear", batch=1, n=1, k=8, act=act, y32=int(y32), dtype=d),
                            lambda act=act, y32=y32, dt=dt: small_linear_op(1, 1, 8, dt, act=act, y32=y32)))
        out.append(Case("edge", dict(entry="small_linear", batch=9, n=17, k=8, dtype=d),
                        lambda dt=dt: small_linear_op(9, 17, 8, dt)))
        for dim, shift in ((2, 0.0), (320, 1.0)):
            for flip in (0, 1):
                out.append(Case("edge", dict(entry="timestep_embed", dim=dim, shift=shift, flip=flip, dtype=d),
                                lambda dim=dim, shift=shift, flip=flip, code=code: plain_op(
                                    "sfb_timestep_embed", **{"t*": 0, "batch": len(TIMESTEPS), "dim": dim,
                                                             "flip": flip, "shift": shift, "out*": 16,
                                                             "ldo": dim + 6, "dtype": code}),
                                run_timestep))
        for name in ("sfb_row_broadcast_add", "sfb_alpha_blend"):
            for rows, rs in ((1, False), (7, True)):
                out.append(Case("edge", dict(entry=name[4:], rows=rows, c=8, rowstats=int(rs), dtype=d),
                                lambda name=name, rows=rows, rs=rs, dt=dt: row_op(name, rows, 8, dt, rowstats=rs)))
        for ci in (1, 8):
            for co in (1, 8):
                out.append(Case("edge", dict(entry="pointwise_nchw", cin=ci, cout=co, n=2, hw=7, dtype=d),
                                lambda ci=ci, co=co, code=code: plain_op(
                                    "sfb_pointwise_nchw", **{"x*": 0, "w*": 0, "bias*": 0, "y*": 0, "n": 2, "hw": 7,
                                                             "cin": ci, "cout": co, "dtype": code})))
    # 16-bit moves: dtype-agnostic kernels
    for (n, h, w, c, ldx, ldy) in ((1, 1, 1, 8, 8, 8), (2, 1, 1, 8, 16, 24), (1, 3, 1, 16, 24, 40)):
        out.append(Case("edge", dict(entry="upsample2x", n=n, h=h, w=w, c=c, ldx=ldx, ldy=ldy),
                        lambda n=n, h=h, w=w, c=c, ldx=ldx, ldy=ldy: plain_op(
                            "sfb_upsample2x", **{"x*": 16, "y*": 32, "n": n, "h": h, "w": w, "c": c, "ldx": ldx,
                                                 "ldy": ldy})))
    for (rows, cols, lds, ldd) in ((1, 1, 1, 1), (1, 8, 16, 24), (3, 5, 7, 9)):
        out.append(Case("edge", dict(entry="copy2d", rows=rows, cols=cols, ld_src=lds, ld_dst=ldd),
                        lambda rows=rows, cols=cols, lds=lds, ldd=ldd: plain_op(
                            "sfb_copy2d", **{"src*": 2, "dst*": 6, "rows": rows, "cols": cols, "ld_src": lds,
                                             "ld_dst": ldd})))
    return out


FAMILIES = {"attention": attention_cases, "gemm": gemm_cases, "conv": conv_cases, "group_norm": group_norm_cases,
            "layer_norm": layer_norm_cases, "temporal": temporal_cases, "softmax": softmax_cases, "edge": edge_cases}


def cases(families=None):
    out = []
    for f in families or FAMILIES:
        out += FAMILIES[f]()
    ids = [c.cid for c in out]
    if len(set(ids)) != len(ids):
        raise AssertionError("duplicate sweep case ids")
    return out


# =====================================================================================================
# one step outside: launches each boundary must refuse, and a word the error must contain
# =====================================================================================================
def _with(op, **fields):
    """`op` with fields of its parameter block overwritten."""
    for k, v in fields.items():
        setattr(op.keep[0], k, v)
    return op


def gn_fused_n_limit():
    return int(_lib.lib().sfb_sm_count())


ONE_STEP_OUTSIDE = [
    # (id, builder, word the error names)
    ("attention head_dim 48", lambda: attn_op(48, 128, 65, 65, F16), "head_dim 48"),
    ("attention kv_tile 64 with head_dim 80", lambda: attn_op(80, 64, 65, 65, F16), "kv_tile 64"),
    ("attention kv_tile 64 with head_dim 128", lambda: attn_op(128, 64, 65, 65, F16), "kv_tile 64"),
    ("attention kv_tile 96", lambda: attn_op(64, 96, 65, 65, F16), "kv_tile"),
    ("attention causal seq_q != seq_kv", lambda: attn_op(64, 64, 65, 64, F16, causal=True), "causal"),
    ("attention causal kv_tile 128", lambda: attn_op(64, 128, 65, 65, F16, causal=True), "causal"),
    ("attention vt_rows", lambda: _with(attn_op(128, 128, 65, 65, F16), vt_rows=128), "vt_rows"),
    ("attention seq_kv 0", lambda: attn_op(64, 64, 65, 0, F16), "seq_kv=0"),
    ("attention_ip seq_ip kv_tile + 1", lambda: attn_op(64, 64, 65, 77, F16, ip=(65, 65)), "seq_ip"),
    ("attention_ip seq_ip 129 at kv_tile 128", lambda: attn_op(128, 128, 65, 77, F16, ip=(129, 129)), "seq_ip"),
    ("attention_ip k_ip_rows < seq_ip", lambda: attn_op(128, 128, 65, 77, F16, ip=(5, 4)), "k_ip_rows"),
    ("gemm K 96", lambda: _with(gemm_op(129, 168, 128, F16), K=96), "K=96"),
    ("gemm N 12", lambda: gemm_op(129, 12, 64, F16), "N=12"),
    ("gemm M 0", lambda: gemm_op(0, 168, 64, F16), "M=0"),
    ("gemm splits > K blocks", lambda: gemm_op(128, 160, 64 * 6, F16, splits=7), "splits"),
    ("gemm geglu N 168", lambda: gemm_op(129, 168, 64, F16, epi=_lib.EPI_GEGLU, geglu_n_out=80), "geglu"),
    ("gemm geglu_n_out > N / 2", lambda: gemm_op(129, 160, 64, F16, epi=_lib.EPI_GEGLU, geglu_n_out=88),
     "geglu_n_out"),
    ("gemm act with split-K", lambda: gemm_op(129, 168, 128, F16, act=_lib.ACT_GELU, splits=2), "act"),
    ("gemm fp32 store with split-K", lambda: gemm_op(129, 168, 128, F16, epi=_lib.EPI_STORE_F32, splits=2), "fp32"),
    ("gemm rowstats_out_slots short", lambda: _with(gemm_op(129, 168, 448, F16, splits=3, rowstats=True),
                                                   rowstats_out_slots=1), "rowstats_out_slots"),
    ("gemm defer_finish with GEGLU", lambda: gemm_op(129, 160, 128, F16, epi=_lib.EPI_GEGLU, geglu_n_out=80,
                                                     splits=2, defer=True), "defer_finish"),
    ("up-conv cin 32", lambda: _with(conv_op("up", 2, 3, 3, 64, 168, F16), cin=32, K=128), "cin=32"),
    ("conv K != 9 cin", lambda: _with(conv_op("conv3x3", 2, 3, 3, 64, 168, F16), K=512), "K=512"),
    ("conv box of 64 pixels", lambda: _with(conv_op("conv3x3", 257, 1, 1, 64, 8, F16), box_n=64), "box"),
    ("conv box wider than the image", lambda: _with(conv_op("conv3x3", 3, 3, 3, 64, 168, F16), box_w=4, box_h=32),
     "box"),
    ("conv M mismatch", lambda: _with(conv_op("conv3x3", 3, 3, 3, 64, 168, F16), M=28), "M mismatch"),
    ("halo conv width 12", lambda: conv_op("halo", 1, 16, 12, 64, 168, F16), "tile width 12"),
    ("halo conv with split-K", lambda: _with(conv_op("halo", 1, 16, 8, 64, 168, F16), splits=2, ws=1), "split-K"),
    ("conv rowbias 8-byte aligned", lambda: conv_op("temporal", 3, 2, 1, 64, 168, F16, rowbias=True, rowbias_off=8),
     "16-byte aligned"),
    ("conv ld_rowbias % 4", lambda: _with(conv_op("temporal", 3, 2, 1, 64, 168, F16, rowbias=True), ld_rowbias=174),
     "ld_rowbias=174"),
    ("down-conv stride 1", lambda: _with(conv_op("down", 3, 3, 3, 64, 168, F16), conv_stride=1), "stride"),
    ("group_norm groups 65", lambda: gn_op("two_pass", 1, 7, 520, 65, F16), "groups=65"),
    ("group_norm c 4104", lambda: gn_op("two_pass", 1, 7, 4104, 8, F16), "c=4104"),
    ("group_norm c % groups", lambda: gn_op("two_pass", 1, 7, 320, 64 - 1, F16), "groups=63"),
    ("group_norm n 0", lambda: _with(gn_op("two_pass", 1, 7, 320, 32, F16), n=0), "n=0"),
    ("group_norm hw 0", lambda: _with(gn_op("two_pass", 1, 7, 320, 32, F16), hw=0), "hw=0"),
    ("group_norm scale_shift n 0", lambda: _with(gn_op("scale_shift", 1, 7, 320, 32, F16), n=0), "n=0"),
    ("group_norm fused hw past the limit",
     lambda: _with(gn_op("fused", 1, 7, 4096, 32, F16), hw=fused_hw_limit(*GN_FUSED_LIMIT) + 1), "does not fit"),
    ("group_norm fused n past the SM count",
     lambda: _with(gn_op("fused", 1, 1, 64, 8, F16), n=gn_fused_n_limit() + 1), "does not fit"),
    ("layer_norm c 2056", lambda: ln_op(1, 2056, F16), "c=2056"),
    ("layer_norm c 0", lambda: ln_op(1, 0, F16), "c=0"),
    ("temporal frames 33", lambda: temporal_op(33, 1, F16), "frames=33"),
    ("temporal head_dim 80", lambda: temporal_op(8, 1, F16, hd=80), "head_dim=80"),
    ("row_softmax cols 16392", lambda: plain_op("sfb_row_softmax", **{"x*": 0, "y*": 16, "rows": 1, "cols": 16392,
                                                                      "ldx": 16392, "ldy": 16392, "x_is_f32": 0,
                                                                      "dtype": 0}), "cols=16392"),
    ("pointwise_nchw cin 9", lambda: plain_op("sfb_pointwise_nchw", **{"x*": 0, "w*": 0, "bias*": 0, "y*": 0, "n": 1,
                                                                       "hw": 7, "cin": 9, "cout": 1, "dtype": 0}),
     "cin"),
    ("small_linear k 12", lambda: small_linear_op(1, 1, 12, F16), "k=12"),
    ("timestep_embed dim 3", lambda: plain_op("sfb_timestep_embed", **{"t*": 0, "batch": 1, "dim": 3, "flip": 0,
                                                                       "shift": 0.0, "out*": 0, "ldo": 8, "dtype": 0}),
     "dim=3"),
]


# =====================================================================================================
# runner
# =====================================================================================================
@contextlib.contextmanager
def capturing_outputs():
    """While active, every output region a replay takes off its canvas is also appended to the yielded
    list (what the PDL on / off comparison compares bit for bit)."""
    got, take = [], Canvas.take

    def recording(self, view):
        t = take(self, view)
        got.append(t)
        return t

    Canvas.take = recording
    try:
        yield got
    finally:
        Canvas.take = take


def run_case(case, peaked=False):
    """Run one case on the GPU: a Result."""
    torch.manual_seed(int(hashlib.sha1(case.cid.encode()).hexdigest()[:8], 16) + int(peaked))
    op = case.op()
    try:
        return (case.run or pl.REPLAY[op.fn.name])(op, peaked=peaked)
    finally:
        torch.cuda.synchronize()


def run_cases(cs, log=None):
    """Run `cs`; yields one record per run (peaked cases twice)."""
    for case in cs:
        for peaked in ((False, True) if case.peaked else (False,)):
            t0 = time.time()
            rec = dict(id=case.cid, family=case.family, params=case.params, peaked=peaked)
            try:
                r = run_case(case, peaked)
                rec["entry"] = case.op().fn.name
                err, tl = r.main()
                rec.update(err=err, tol=tl, parts=r.parts, ok=r.ok)
            except Exception as e:  # noqa: BLE001  -- a refused or failing launch is a failing case
                if "CUDA error" in str(e):
                    raise   # a device fault poisons the context: every later case would fail with it
                rec.update(entry=rec.get("entry", "?"), err=float("inf"), tol=0.0, error=repr(e)[:400], ok=False)
            rec["seconds"] = round(time.time() - t0, 3)
            if log is not None:
                log(rec)
            yield rec


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--family", nargs="*", choices=sorted(FAMILIES), help="case families (default: all)")
    ap.add_argument("--json", help="also write the records (and the summary) to this JSON file")
    ap.add_argument("--list", action="store_true", help="list the cases, no GPU")
    args = ap.parse_args(argv)
    cs = cases(args.family)
    if args.list:
        for c in cs:
            print(json.dumps(dict(id=c.cid, family=c.family, params=c.params, peaked=c.peaked)))
        print(json.dumps({"cases": len(cs)}))
        return 0
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    records = list(run_cases(cs, log=lambda r: print(json.dumps(r), flush=True)))
    summ = pl.summarize(records)
    tail = {"summary": {k: dict(max_err=v[0], tol=v[1], runs=v[2], failures=v[3]) for k, v in sorted(summ.items())},
            "cases": len(cs), "runs": len(records), "seconds": round(time.time() - t0, 1),
            "peak_max_memory_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
            "device": torch.cuda.get_device_name()}
    print(json.dumps(tail), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(records=records, **tail), f, indent=0)
    return 0 if all(r["ok"] for r in records) else 1


if __name__ == "__main__":
    sys.exit(main())
