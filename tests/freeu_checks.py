"""sfb_freeu in the launch-level checks: its float64 reference (the closed form of diffusers' fourier_filter), its
access rule for plan_hazards.py and its float64 replay for plan_launches.py.

Importing this module registers sfb_freeu with both (register()): plan_hazards gains the access rule and the
static input `freeu_in`, plan_launches the replay.  Neither changes anything for a plan without FreeU."""
import ctypes as C
import math

import torch

import plan_hazards as ph
import plan_launches as pl
from kernel_checks import rel_err
from sfast_b200 import _lib

ESZ = ph.ESZ


def ref_fourier_filter(x, s):
    """diffusers' fourier_filter(x, threshold=1, scale=s) of x [n, c, h, w] in closed form, float64: the scaled
    box is exactly the frequencies {0, h-1} x {0, w-1} (as sets), so
    y = x + (s - 1) / (h w) * sum_{p, q} Re(X[p, q] e^{+2 pi i (p y / h + q x / w)}) with X the 2-D DFT."""
    x = x.double()
    n, c, h, w = x.shape
    hh = torch.arange(h, dtype=torch.float64, device=x.device)
    ww = torch.arange(w, dtype=torch.float64, device=x.device)
    corr = torch.zeros_like(x)
    for p in sorted({0, h - 1}):
        for q in sorted({0, w - 1}):
            e = torch.polar(torch.ones(h, w, dtype=torch.float64, device=x.device),
                            2 * math.pi * (p * hh[:, None] / h + q * ww[None, :] / w))
            X = (x.to(torch.complex128) * e.conj()).sum((-2, -1))
            corr += (X[..., None, None] * e).real
    return x + (s - 1) / (h * w) * corr


def freeu_accesses(p):
    """[Access] of one sfb_freeu launch: (b, s) read; the first c_hidden / 2 hidden channels and the skip slice of
    every pixel read and written in place (the rest of the row, and the pitch gap, untouched)."""
    rows, ld = p.n * p.h * p.w, p.ld * ESZ
    return [ph.Access("bs", p.bs, 1, 8, 0, "r"),
            ph.Access("x.hidden", p.x, rows, p.c_hidden // 2 * ESZ, ld, "rw"),
            ph.Access("x.skip", ph._p(p.x) + p.c_hidden * ESZ, rows, p.c_skip * ESZ, ld, "rw")]


def replay_freeu(op, peaked=False):
    """sfb_freeu on a concat buffer with a low-frequency component in every channel, so the filter moves the
    output: the hidden half bit-exact against torch's x * b, the skip slice against ref_fourier_filter, and every
    other byte of the buffer (untouched channels, pitch gap, leading offset, guard band) unchanged."""
    p0 = op.keep[0]
    p = pl._clone(p0)
    dt, rows, ch, cs = pl.DTYPES[p.dtype], p.n * p.h * p.w, p.c_hidden, p.c_skip
    half = ch // 2
    cat = pl.Canvas(dt, pl._off(p0.x, 2), rows, p.ld)
    hh = torch.arange(p.h, device=pl.DEV)[:, None] / p.h
    ww = torch.arange(p.w, device=pl.DEV)[None, :] / p.w
    low = torch.cos(2 * math.pi * (hh + ww) + torch.rand(p.n, ch + cs, 1, 1, device=pl.DEV) * 6.3)
    x = torch.randn(p.n, ch + cs, p.h, p.w, device=pl.DEV) + 2 * torch.rand(p.n, ch + cs, 1, 1, device=pl.DEV) * low + 0.5
    cat.region(rows, ch + cs).copy_(x.permute(0, 2, 3, 1).reshape(rows, ch + cs).to(dt))
    X = cat.region(rows, ch + cs).clone()
    bs = torch.tensor([1.4, 0.2], device=pl.DEV)
    p.x, p.bs = cat.ptr, bs.data_ptr()
    cat.arm()
    _lib.check(_lib.lib().sfb_freeu(C.byref(p), pl._stream()), "sfb_freeu")
    torch.cuda.synchronize()
    res = pl.Result()
    res.add("hidden", rel_err(cat.take(cat.region(rows, half)), (X[:, :half].float() * bs[0]).to(dt).double()),
            pl.tol("exact", dt))
    skip = X[:, ch:].double().view(p.n, p.h, p.w, cs).permute(0, 3, 1, 2)
    ref = ref_fourier_filter(skip, float(bs[1])).permute(0, 2, 3, 1).reshape(rows, cs)
    res.add("skip", rel_err(cat.take(cat.region(rows, cs, off=ch)), ref), pl.tol("pointwise", dt))
    res.canary(cat)
    return res


def register():
    """Teach plan_hazards (access rule, the static input freeu_in) and plan_launches (replay) about sfb_freeu.
    Idempotent."""
    if "sfb_freeu" in ph.MODELLED:
        return
    base = ph.launch_accesses

    def launch_accesses(name, args, keep=None):
        if name == "sfb_freeu":
            return freeu_accesses(ph._struct(keep[0] if keep is not None else args[0]))
        return base(name, args, keep)

    ph.launch_accesses = launch_accesses
    ph.STRUCT_MODELLED = ph.STRUCT_MODELLED + ("sfb_freeu",)
    ph.MODELLED = frozenset(ph.PLAIN_MODELLED + ph.STRUCT_MODELLED)
    ph.INPUTS = ph.INPUTS + ("freeu_in",)
    pl.STRUCT = pl.STRUCT + ("sfb_freeu",)
    pl.REPLAY["sfb_freeu"] = replay_freeu


register()
