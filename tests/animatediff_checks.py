"""sfb_frame_attention in the launch-level checks: its float64 reference, its access rule for plan_hazards.py and its
float64 replay for plan_launches.py.

Importing this module registers sfb_frame_attention with both (register()).  Nothing changes for a plan without
motion modules."""
import ctypes as C

import torch

import plan_hazards as ph
import plan_launches as pl
from kernel_checks import rel_err
from sfast_b200 import _lib

ESZ = ph.ESZ


def ref_frame_attention(qkv, bias, batch, frames, seq, heads, head_dim, scale):
    """float64 softmax(scale q k^T) v across the frames of every (video, pixel, head) of the fused QKV rows
    [batch * frames * seq, >= 3C] (spatial row order), with the fp32 frame bias [frames, >= 3C] added to q | k | v
    and the sum rounded to qkv's 16-bit type, as the kernel stores it; returns [rows, C]."""
    Cm = heads * head_dim
    x = qkv[:, :3 * Cm].double()
    if bias is not None:
        b = bias[:, :3 * Cm].float().repeat_interleave(seq, 0).repeat(batch, 1)
        x = (qkv[:, :3 * Cm].float() + b).to(qkv.dtype).double()
    x = x.view(batch, frames, seq, 3, heads, head_dim).permute(3, 0, 2, 4, 1, 5)
    q, k, v = x[0], x[1], x[2]  # [batch, seq, heads, frames, D]
    p = torch.softmax(scale * q @ k.transpose(-1, -2), -1)
    return (p @ v).permute(0, 3, 1, 2, 4).reshape(batch * frames * seq, Cm)


def frame_attention_accesses(p):
    """[Access] of one sfb_frame_attention launch: the q | k | v columns of every row and the frame-bias rows read,
    the heads * head_dim output columns of every row written."""
    rows, Cm = p.batch * p.frames * p.seq, p.heads * p.head_dim
    acc = [ph.Access("qkv", p.qkv, rows, 3 * Cm * ESZ, p.ld_qkv * ESZ, "r"),
           ph.Access("out", p.out, rows, Cm * ESZ, p.ld_out * ESZ, "w")]
    if p.frame_bias:
        acc.append(ph.Access("frame_bias", p.frame_bias, p.frames, 3 * Cm * 4, p.ld_bias * 4, "r"))
    return acc


def replay_frame_attention(op, peaked=False):
    """The launch's geometry on random q / k / v and frame bias against ref_frame_attention; the output canvas
    outside the declared columns (pitch gap, guard rows) must be unchanged."""
    p0 = op.keep[0]
    p = pl._clone(p0)
    dt = pl.DTYPES[p.dtype]
    rows, Cm = p.batch * p.frames * p.seq, p.heads * p.head_dim
    qkv = pl._randn(rows * p.ld_qkv, dt).view(rows, p.ld_qkv)
    bias = None
    if p0.frame_bias:
        bias = torch.randn(p.frames, p.ld_bias, device=pl.DEV) * 0.5
        p.frame_bias = bias.data_ptr()
    out = pl.Canvas(dt, pl._off(p0.out, 2), rows, p.ld_out)
    p.qkv, p.out = qkv.data_ptr(), out.ptr
    out.arm()
    _lib.check(_lib.lib().sfb_frame_attention(C.byref(p), pl._stream()), "sfb_frame_attention")
    torch.cuda.synchronize()
    ref = ref_frame_attention(qkv, bias, p.batch, p.frames, p.seq, p.heads, p.head_dim, float(p.scale))
    res = pl.Result()
    res.add("out", rel_err(out.take(out.region(rows, Cm)), ref), pl.tol("temporal", dt))
    res.canary(out)
    return res


def register():
    """Teach plan_hazards (access rule) and plan_launches (replay) about sfb_frame_attention.  Idempotent."""
    if "sfb_frame_attention" in ph.MODELLED:
        return
    base = ph.launch_accesses

    def launch_accesses(name, args, keep=None):
        if name == "sfb_frame_attention":
            return frame_attention_accesses(ph._struct(keep[0] if keep is not None else args[0]))
        return base(name, args, keep)

    ph.launch_accesses = launch_accesses
    ph.STRUCT_MODELLED = ph.STRUCT_MODELLED + ("sfb_frame_attention",)
    ph.MODELLED = frozenset(ph.PLAIN_MODELLED + ph.STRUCT_MODELLED)
    pl.STRUCT = pl.STRUCT + ("sfb_frame_attention",)
    pl.REPLAY["sfb_frame_attention"] = replay_frame_attention


register()
