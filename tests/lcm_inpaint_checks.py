"""sfb_im2col_in_wide and the LCM guidance input in the launch-level checks: the access rule of sfb_im2col_in_wide for
plan_hazards.py, its float64 replay for plan_launches.py, and the static input `timestep_cond_in`.

Importing this module registers them (register()).  Neither changes anything for a plan without a wide conv_in or
a guidance embedding."""
import torch
import torch.nn.functional as F

import plan_hazards as ph
import plan_launches as pl
from kernel_checks import rel_err
from sfast_b200 import _lib

ESZ = ph.ESZ
WIDE_K = 128   # two 64-wide K blocks
# argument names of sfb_im2col_in_wide ("*": a pointer), as plan_launches.PLAIN lists them for the plain entry points;
# kept out of PLAIN, whose every entry the shipped plans must launch
ARGS = ("x*", "a*", "n", "h", "wd", "cin")


def ref_im2col_wide(x):
    """The rows sfb_im2col_in_wide writes for x [n, cin, h, w], float64: a[p, (kh*3+kw)*cin + c], zero up to 128."""
    n, cin, h, w = x.shape
    cols = F.unfold(x.double(), 3, padding=1).view(n, cin, 9, h * w).permute(0, 3, 2, 1).reshape(n * h * w, 9 * cin)
    ref = torch.zeros(n * h * w, WIDE_K, dtype=torch.float64, device=x.device)
    ref[:, :9 * cin] = cols
    return ref


def im2col_wide_accesses(args):
    """[Access] of one sfb_im2col_in_wide launch: the whole NCHW input read, every 128-wide row written."""
    x, a, n, h, wd, cin = args[:6]
    return [ph.Access("x", x, 1, n * cin * h * wd * ESZ, 0, "r"),
            ph.Access("a", a, 1, n * h * wd * WIDE_K * ESZ, 0, "w")]


def replay_im2col_wide(op, peaked=False):
    """sfb_im2col_in_wide at the launch's geometry on a fresh input: bit-exact against F.unfold, and the guard band
    after the last row unchanged."""
    a = dict(zip(ARGS, op.args))
    n, h, w, cin = a["n"], a["h"], a["wd"], a["cin"]
    dt = torch.float16
    x = pl._randn(n * cin * h * w, dt).view(n, cin, h, w)
    A = pl.Canvas(dt, 0, n * h * w, WIDE_K)
    A.arm()
    _lib.check(_lib.lib().sfb_im2col_in_wide(x.data_ptr(), A.ptr, n, h, w, cin, pl._stream()), "sfb_im2col_in_wide")
    torch.cuda.synchronize()
    res = pl.Result()
    res.add("a", rel_err(A.take(A.region(n * h * w, WIDE_K)), ref_im2col_wide(x)), pl.tol("exact", dt))
    res.canary(A)
    return res


def register():
    """Teach plan_hazards (access rule, the static input timestep_cond_in) and plan_launches (replay) about the
    wide conv_in and the LCM guidance input.  Idempotent."""
    if "sfb_im2col_in_wide" in ph.MODELLED:
        return
    base = ph.launch_accesses

    def launch_accesses(name, args, keep=None):
        if name == "sfb_im2col_in_wide":
            return [acc for acc in im2col_wide_accesses(args) if acc.addr and acc.row_bytes]
        return base(name, args, keep)

    ph.launch_accesses = launch_accesses
    ph.PLAIN_MODELLED = ph.PLAIN_MODELLED + ("sfb_im2col_in_wide",)
    ph.MODELLED = frozenset(ph.PLAIN_MODELLED + ph.STRUCT_MODELLED)
    ph.INPUTS = ph.INPUTS + ("timestep_cond_in",)
    key, describe = pl.launch_key, pl.describe

    def launch_key(op):
        if op.fn.name == "sfb_im2col_in_wide":
            return (op.fn.name,) + tuple(pl._plain(a) for a in op.args)
        return key(op)

    def describe_(k):
        if k[0] == "sfb_im2col_in_wide":
            return f"{k[0]}({', '.join(f'{n}={v}' for n, v in zip(ARGS, k[1:]) if not n.endswith('*'))})"
        return describe(k)

    pl.launch_key, pl.describe = launch_key, describe_
    pl.REPLAY["sfb_im2col_in_wide"] = replay_im2col_wide


register()
