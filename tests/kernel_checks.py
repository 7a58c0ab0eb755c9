"""Per-kernel parity checks of the CUDA path (through the C ABI) against plain PyTorch fp32
references of the same op on the same seeded inputs.  Imported by ``tests/test_kernels_gpu.py``
(pytest, ``-m gpu``) and runnable as a script so each check can be isolated in its own process:

    python tests/kernel_checks.py [name ...]      # prints one JSON line per check

Tolerances mirror the reference's own operator tests: conv 1e-3-class
(/root/reference/tests/operators/test_cudnn_convolution.py:65), GEGLU 2e-2
(tests/operators/test_cutlass_dual_linear.py:56), GroupNorm / LayerNorm 1e-2
(src/sfast/triton/ops/group_norm.py:485-523, layer_norm.py:435-438).
"""
import json
import math
import os
import sys

import torch
import torch.nn.functional as F

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(_ROOT, "stable-fast_b200"))
sys.path.insert(0, _ROOT)  # oracle/ (the checker)

from sfast_b200 import _lib, ops  # noqa: E402
from sfast_b200.ops import Act  # noqa: E402

# the fp32 F.conv2d / matmul references must not run in TF32 (cuDNN allows it by default): check_conv_gn's
# normalised fp32 activations would be rounded to 10 mantissa bits inside the reference
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False

DEV = "cuda"


def _stream():
    return torch.cuda.current_stream().cuda_stream


def rel_err(got, ref):
    """max of two normalised errors, both of which must be below the check's tolerance `tol`:
      * global max-norm:  max|d| / max|ref|
      * elementwise:      max(|d| / (|ref| + rms(ref)))   i.e. |d| <= tol * |ref| + tol * rms(ref),
        the assert_close(rtol, atol) form of the reference's own operator tests
        (/root/reference/tests/operators/test_cudnn_convolution.py:65) with atol scaled to the
        tensor; a small-magnitude output that is 100 % wrong fails this one."""
    got, ref = got.float(), ref.float()
    d = (got - ref).abs()
    rms = ref.pow(2).mean().sqrt().clamp_min(1e-6)
    return max((d.max() / ref.abs().max().clamp_min(1e-6)).item(), (d / (ref.abs() + rms)).max().item())


def _rand(*shape, dt=torch.float16, scale=1.0, seed=None):
    if seed is not None:
        torch.manual_seed(seed)
    return (torch.randn(*shape, device=DEV) * scale).to(dt)


# ------------------------------------------------------------------------------------------
def check_gemm(M=300, N=320, K=320, dt=torch.float16, splits=1, bias=True, residual=True, seed=0,
               pair=None, persistent=False, act=0):
    lib = _lib.lib()
    a = _rand(M, K, dt=dt, seed=seed)
    w = _rand(N, K, dt=dt, scale=1 / math.sqrt(K))
    b = torch.randn(N, device=DEV) if bias else None
    r = _rand(M, N, dt=dt) if residual else None
    out = torch.zeros(M, N, device=DEV, dtype=dt)
    ws = torch.empty(max(splits, 1) * M * N, device=DEV, dtype=torch.float32)
    op = ops.gemm_op("gemm", lib, a=ops.a_matrix(a.data_ptr(), M, K, K), b=ops.Mat(w), M=M, N=N, K=K,
                     dt=dt, out=out, ldo=N, bias=b, residual=r, ldr=N, ws=ws, splits=splits,
                     cta_pair=pair, persistent=persistent, act=act)
    assert op.keep[0].persistent == int(bool(persistent)), "persistent kernel was not selected"
    op.launch(_stream())
    torch.cuda.synchronize()
    ref = a.float() @ w.float().t()
    if bias:
        ref = ref + b
    if act == _lib.ACT_QUICK_GELU:   # CLIP: x * sigmoid(1.702 x), before the residual
        ref = ref * torch.sigmoid(1.702 * ref)
    elif act == _lib.ACT_GELU:
        ref = F.gelu(ref)
    if residual:
        ref = ref + r.float()
    return rel_err(out, ref)


def check_geglu(M=256, K=320, inner=1280, dt=torch.float16, splits=1, seed=1, persistent=False):
    lib = _lib.lib()
    x = _rand(M, K, dt=dt, seed=seed)
    w = _rand(2 * inner, K, dt=dt, scale=1 / math.sqrt(K))
    b = torch.randn(2 * inner, device=DEV) * 0.1
    wp, bp, _ = ops.pack_geglu(w, b, dt)
    Np = wp.shape[0]
    out = torch.zeros(M, inner, device=DEV, dtype=dt)
    ws = torch.empty(max(splits, 1) * M * Np, device=DEV, dtype=torch.float32)
    op = ops.gemm_op("geglu", lib, a=ops.a_matrix(x.data_ptr(), M, K, K), b=ops.Mat(wp), M=M, N=Np, K=K,
                     dt=dt,
                     out=out, ldo=inner, bias=bp, epi=ops.EPI_GEGLU, geglu_n_out=inner, ws=ws,
                     splits=splits, persistent=persistent)
    assert op.keep[0].persistent == int(bool(persistent))
    op.launch(_stream())
    torch.cuda.synchronize()
    # reference semantics: h * gelu(gate), hidden first (sfast passes/__init__.py:643-648)
    y = x.float() @ w.float().t() + b
    h, g = y.chunk(2, dim=-1)
    return rel_err(out, h * F.gelu(g))


def check_conv(n=2, h=64, w=64, cin=320, cout=320, stride=1, dt=torch.float16, splits=None,
               rowbias=True, residual=True, pitch_extra=0, seed=2, pair=None, persistent=False):
    lib = _lib.lib()
    torch.manual_seed(seed)
    ld = cin + pitch_extra
    xbuf = _rand(n, h, w, ld, dt=dt)
    x = Act(xbuf, n, h, w, cin, ld=ld)
    wt = _rand(cout, cin, 3, 3, dt=dt, scale=1 / math.sqrt(9 * cin))
    b = torch.randn(cout, device=DEV)
    ho, wo = h // stride, w // stride
    M = n * ho * wo
    rb = torch.randn(n, cout, device=DEV) if rowbias else None
    r = _rand(M, cout, dt=dt) if residual else None
    out = torch.zeros(M, cout, device=DEV, dtype=dt)
    wp = ops.pack_conv3x3(wt, dt)
    box_n, box_h, box_w = ops.conv_tile_box(ho, wo)
    adesc = ops.a_conv(x.ptr, n, h, w, cin, ld, box_n, box_h, box_w, stride)
    ws = torch.empty(64 * M * cout, device=DEV, dtype=torch.float32) if splits != 1 else None
    op = ops.gemm_op("conv", lib, a=adesc, b=ops.Mat(wp),
                     M=M, N=cout, K=9 * cin, dt=dt, out=out, ldo=cout, bias=b, rowbias=rb,
                     rows_per_img=ho * wo, ld_rowbias=cout, residual=r, ldr=cout, ws=ws,
                     splits=splits, cta_pair=pair, persistent=persistent,
                     conv=dict(n=n, h=ho, w=wo, cin=cin, stride=stride, box_n=box_n, box_h=box_h, box_w=box_w))
    assert op.keep[0].persistent == int(bool(persistent))
    op.launch(_stream())
    torch.cuda.synchronize()
    xin = x.tensor().permute(0, 3, 1, 2).float()
    ref = F.conv2d(xin, wt.float(), b, stride=stride, padding=1)
    if rowbias:
        ref = ref + rb[:, :, None, None]
    ref = ref.permute(0, 2, 3, 1).reshape(M, cout)
    if residual:
        ref = ref + r.float()
    return rel_err(out, ref)


def check_conv_gn(n=2, h=64, w=64, cin=320, cout=320, dt=torch.float16, groups=32, silu=True, rowbias=True,
                  residual=True, pitch_extra=0, out_extra=0, mean=0.0, seed=51, eps=1e-5, replay=False):
    """GroupNorm(+SiLU) folded into the 3x3 conv's A-operand path (SFB_A_CONV3X3_GN: statistics ->
    per-channel (scale, shift) -> halo tile transformed in shared memory) vs fp32
    conv2d(silu(group_norm(x))) + bias + per-image row bias + residual."""
    lib = _lib.lib()
    torch.manual_seed(seed)
    ld = cin + pitch_extra
    xbuf = (torch.randn(n, h, w, ld, device=DEV) * (1.0 + torch.rand(ld, device=DEV)) + mean
            + torch.randn(ld, device=DEV) * (0.5 if mean == 0.0 else 2.0)).to(dt)
    x = Act(xbuf, n, h, w, cin, ld=ld)
    gamma = 1.0 + 0.5 * torch.randn(cin, device=DEV)
    beta = 0.3 * torch.randn(cin, device=DEV)
    wt = _rand(cout, cin, 3, 3, dt=dt, scale=1 / math.sqrt(9 * cin))
    b = torch.randn(cout, device=DEV)
    M = n * h * w
    rb = torch.randn(n, cout, device=DEV) if rowbias else None
    r = _rand(M, cout, dt=dt) if residual else None
    ldo = cout + out_extra
    out = torch.zeros(M, ldo, device=DEV, dtype=dt)
    stats = torch.zeros(ops.gn_ws_floats(n, groups), device=DEV)
    counters = torch.zeros(max(n, 4), device=DEV, dtype=torch.int32)
    ab = torch.zeros(n, cin, 2, device=DEV)
    assert ops.conv_gn_tiles(n, h, w) > 0, "geometry not eligible for the halo conv"
    st = ops.gn_scale_shift_op("gn", lib, x=x, gamma=gamma, beta=beta, stats=stats, counters=counters,
                               scale_shift=ab, groups=groups, eps=eps, dt=dt)
    op = ops.gemm_op("conv_gn", lib, a=ops.a_conv_halo(x.ptr, n, h, w, cin, ld), b=ops.Mat(ops.pack_conv3x3(wt, dt)),
                     M=M, N=cout, K=9 * cin, dt=dt, out=out, ldo=ldo, bias=b, rowbias=rb, rows_per_img=h * w,
                     ld_rowbias=cout, residual=r, ldr=cout,
                     conv=dict(n=n, h=h, w=w, cin=cin, stride=1, box_n=1, box_h=ops.HALO_BOX_H, box_w=ops.HALO_BOX_W),
                     gn=dict(scale_shift=ab, silu=silu))
    assert op.keep[0].a_mode == _lib.A_CONV3X3_GN
    st.launch(_stream())
    op.launch(_stream())
    torch.cuda.synchronize()
    xin = x.tensor().permute(0, 3, 1, 2).float().contiguous()
    y = F.group_norm(xin, groups, gamma, beta, eps)
    # (scale, shift) against the fp32 statistics
    mean_ = xin.view(n, groups, -1).mean(-1)
    var_ = xin.view(n, groups, -1).var(-1, unbiased=False)
    sc_ref = (gamma.view(1, groups, -1) * torch.rsqrt(var_ + eps)[:, :, None]).reshape(n, cin)
    sh_ref = beta[None] - (mean_[:, :, None] * sc_ref.view(n, groups, -1)).reshape(n, cin)
    e_ab = max(rel_err(ab[..., 0], sc_ref), rel_err(ab[..., 1], sh_ref))
    if silu:
        y = F.silu(y)
    ref = F.conv2d(y, wt.float(), b, padding=1)
    if rowbias:
        ref = ref + rb[:, :, None, None]
    ref = ref.permute(0, 2, 3, 1).reshape(M, cout)
    if residual:
        ref = ref + r.float()
    err = max(rel_err(out[:, :cout], ref), e_ab)
    if out_extra and float(out[:, cout:].abs().max()) != 0.0:
        return float("inf")  # wrote outside its channel slice
    if replay:  # a second pass (self-resetting tickets, ordered reductions) must be bit-identical
        first, ab1 = out.clone(), ab.clone()
        out.zero_()
        st.launch(_stream())
        op.launch(_stream())
        torch.cuda.synchronize()
        if not (torch.equal(first, out) and torch.equal(ab1, ab)):
            return float("inf")
    return err


def check_upconv(n=2, h=16, w=16, cin=640, cout=640, dt=torch.float16, splits=None, pair=None,
                 out_extra=0, seed=23, persistent=False):
    """nearest-2x upsample + conv3x3 as the 4-phase 2x2 implicit GEMM on the low-res image vs
    F.conv2d(F.interpolate(x, 2, 'nearest')) in fp32 (weights as packed: sums rounded to 16 bit)."""
    lib = _lib.lib()
    torch.manual_seed(seed)
    xin = _rand(n, h, w, cin, dt=dt)
    wt = _rand(cout, cin, 3, 3, dt=dt, scale=1 / math.sqrt(9 * cin))
    b = torch.randn(cout, device=DEV)
    M = 4 * n * h * w
    ld = cout + out_extra
    out = torch.zeros(n, 2 * h, 2 * w, ld, device=DEV, dtype=dt)
    box_n, box_h, box_w = ops.conv_tile_box(h, w)
    adesc = ops.a_conv(xin.data_ptr(), n, h, w, cin, cin, box_n, box_h, box_w, 1)
    ws = torch.empty(32 * M * cout, device=DEV, dtype=torch.float32) if splits != 1 else None
    op = ops.gemm_op("upconv", lib, a=adesc, b=ops.Mat(ops.pack_upconv(wt, dt)), M=M, N=cout, K=4 * cin,
                     dt=dt, out=out.data_ptr(), ldo=ld, bias=b, ws=ws, splits=splits, cta_pair=pair,
                     persistent=persistent,
                     conv=dict(n=n, h=h, w=w, cin=cin, stride=1, box_n=box_n, box_h=box_h, box_w=box_w, up=True))
    op.launch(_stream())
    torch.cuda.synchronize()
    up = F.interpolate(xin.permute(0, 3, 1, 2).float(), scale_factor=2, mode="nearest")
    ref = F.conv2d(up, wt.float(), b, padding=1).permute(0, 2, 3, 1)
    if out_extra:
        assert float(out[..., cout:].abs().max()) == 0.0
    return rel_err(out[..., :cout], ref)


def _attn_buffers(B, H, S, Skv, D, dt):
    dv = (D + 1 + 15) // 16 * 16  # + the all-ones row (softmax denominator on the tensor core)
    q_pitch = (D + 63) // 64 * 64
    vt_pitch = (Skv + 63) // 64 * 64
    q = torch.zeros(B * H * S, q_pitch, device=DEV, dtype=dt)
    k = torch.zeros(B * H * Skv, q_pitch, device=DEV, dtype=dt)
    vt = torch.zeros(B * H * dv, vt_pitch, device=DEV, dtype=dt)
    vt.view(B * H, dv, vt_pitch)[:, D, :] = 1.0
    return q, k, vt, dv, q_pitch, vt_pitch


def check_attention(B=2, H=8, S=1024, Skv=None, D=40, dt=torch.float16, seed=3, kv_tile=None, causal=False):
    lib = _lib.lib()
    Skv = Skv or S
    torch.manual_seed(seed)
    qr = _rand(B, H, S, D, dt=dt)
    kr = _rand(B, H, Skv, D, dt=dt)
    vr = _rand(B, H, Skv, D, dt=dt)
    q, k, vt, dv, q_pitch, vt_pitch = _attn_buffers(B, H, S, Skv, D, dt)
    q.view(B * H, S, q_pitch)[:, :, :D] = qr.reshape(B * H, S, D)
    k.view(B * H, Skv, q_pitch)[:, :, :D] = kr.reshape(B * H, Skv, D)
    vt.view(B * H, dv, vt_pitch)[:, :D, :Skv] = vr.reshape(B * H, Skv, D).transpose(1, 2)
    out = torch.zeros(B, S, H * D, device=DEV, dtype=dt)
    op = ops.attention_op("attn", lib, q=q, k=k, vt=vt, out=out, batch=B, heads=H, head_dim=D,
                          seq_q=S, seq_kv=Skv, q_rows=S, k_rows=Skv, vt_rows=dv, q_pitch=q_pitch,
                          vt_pitch=vt_pitch, dt=dt, kv_tile=kv_tile, causal=causal)
    if kv_tile is not None:
        assert op.keep[0].kv_tile == kv_tile
    op.launch(_stream())
    torch.cuda.synchronize()
    ref = F.scaled_dot_product_attention(qr.float(), kr.float(), vr.float(), is_causal=causal)
    ref = ref.transpose(1, 2).reshape(B, S, H * D)
    return rel_err(out, ref)



def check_embed_tokens(B=3, S=77, C=768, V=1000, dt=torch.float16, seed=11):
    """Token + position embedding gather and the row statistics it hands to the first folded LayerNorm."""
    lib = _lib.lib()
    torch.manual_seed(seed)
    tok, pos = _rand(V, C, dt=dt), _rand(S, C, dt=dt)
    ids = torch.randint(0, V, (B, S), device=DEV)
    out = torch.zeros(B * S, C, device=DEV, dtype=dt)
    stats = torch.full((B * S, 2), 7.0, device=DEV)  # written, not accumulated
    _lib.check(lib.sfb_embed_tokens(ids.data_ptr(), tok.data_ptr(), pos.data_ptr(), out.data_ptr(), stats.data_ptr(),
                                    1, B, S, C, V, C, ops.dtype_code(dt), _stream()), "embed")
    torch.cuda.synchronize()
    ref = (tok[ids].float() + pos[None].float()).reshape(B * S, C)
    e = rel_err(out, ref)
    o = out.float()
    e_s = float((stats[:, 0] - o.sum(1)).abs().max() / o.sum(1).abs().max())
    e_q = float((stats[:, 1] - (o * o).sum(1)).abs().max() / (o * o).sum(1).abs().max())
    return max(e, e_s, e_q)


def check_clip_pool(eos_id, B=5, S=77, C=768, dt=torch.float16, seed=12):
    """End-of-text pooling: first eos position (or, eos_id == 2, the first maximal id) per row."""
    lib = _lib.lib()
    torch.manual_seed(seed)
    x = _rand(B * S, C, dt=dt)
    ids = torch.randint(3, 1000, (B, S), device=DEV)
    eos_tok = 49407 if eos_id == 2 else eos_id
    for b in range(B):   # eos somewhere, then padded with eos (SD pads with the eos token)
        p = 5 + 13 * b
        ids[b, p:] = eos_tok
    if eos_id != 2:
        ids[B - 1] = 7   # a row without any eos: transformers' argmax of all-False is position 0
    pooled = torch.zeros(B, C, device=DEV, dtype=dt)
    _lib.check(lib.sfb_clip_pool(ids.data_ptr(), x.data_ptr(), pooled.data_ptr(), B, S, C, C, eos_id, _stream()), "pool")
    torch.cuda.synchronize()
    if eos_id == 2:
        pos = ids.to(torch.int).argmax(dim=-1)
    else:
        pos = (ids.to(torch.int) == eos_id).int().argmax(dim=-1)
    ref = x.view(B, S, C)[torch.arange(B, device=DEV), pos]
    return float((pooled.float() - ref.float()).abs().max())



def check_patchify(B=2, C=3, H=56, P=14, kpad=640, dt=torch.float16, seed=13):
    """Non-overlapping patches as GEMM rows == unfold; padding columns zero."""
    lib = _lib.lib()
    x = _rand(B, C, H, H, dt=dt, seed=seed)
    g = H // P
    a = torch.full((B * g * g, kpad), 3.0, device=DEV, dtype=dt)
    _lib.check(lib.sfb_patchify(x.data_ptr(), a.data_ptr(), B, C, H, H, P, kpad, _stream()), "patchify")
    torch.cuda.synchronize()
    ref = F.unfold(x.float(), kernel_size=P, stride=P).transpose(1, 2).reshape(B * g * g, C * P * P)
    pad = float(a[:, C * P * P:].float().abs().max()) if kpad > C * P * P else 0.0
    return float((a[:, :C * P * P].float() - ref).abs().max()) + pad


def check_qkv_scatter(B=2, H=8, S=256, D=40, dt=torch.float16, cross_kv=0, seed=4, persistent=False):
    """QKV projection GEMM whose epilogue writes the attention layouts directly."""
    lib = _lib.lib()
    C = H * D
    torch.manual_seed(seed)
    if cross_kv:
        Kdim, seq, which_base, ncols = 768, cross_kv, 1, 2 * C
    else:
        Kdim, seq, which_base, ncols = C, S, 0, 3 * C
    x = _rand(B * seq, Kdim, dt=dt)
    w = _rand(ncols, Kdim, dt=dt, scale=1 / math.sqrt(Kdim))
    q, k, vt, dv, q_pitch, vt_pitch = _attn_buffers(B, H, S, seq, D, dt)
    M = B * seq
    op = ops.gemm_op("qkv", lib, a=ops.a_matrix(x.data_ptr(), M, Kdim, Kdim), b=ops.Mat(w), M=M, N=ncols,
                     K=Kdim, dt=dt, epi=ops.EPI_QKV,
                     qkv=dict(q=q, k=k, vt=vt, heads=H, head_dim=D, which_base=which_base,
                              seq=seq, q_pitch=q_pitch, q_rows=S, k_rows=seq, vt_rows=dv,
                              vt_pitch=vt_pitch), persistent=persistent)
    assert op.keep[0].persistent == int(bool(persistent))
    op.launch(_stream())
    torch.cuda.synchronize()
    y = (x.float() @ w.float().t()).view(B, seq, -1, H, D)  # [B, seq, which, H, D]
    errs = []
    idx = 0
    if not cross_kv:
        qref = y[:, :, 0].permute(0, 2, 1, 3).reshape(B * H, S, D)
        errs.append(rel_err(q.view(B * H, S, q_pitch)[:, :, :D], qref))
        idx = 1
    kref = y[:, :, idx].permute(0, 2, 1, 3).reshape(B * H, seq, D)
    vref = y[:, :, idx + 1].permute(0, 2, 3, 1).reshape(B * H, D, seq)
    errs.append(rel_err(k.view(B * H, seq, q_pitch)[:, :, :D], kref))
    errs.append(rel_err(vt.view(B * H, dv, vt_pitch)[:, :D, :seq], vref))
    # padding must stay zero
    pad = float(q.view(B * H, S, q_pitch)[:, :, D:].abs().max()) if not cross_kv else 0.0
    pad += float(vt.view(B * H, dv, vt_pitch)[:, :D, seq:].abs().max()) if vt_pitch > seq else 0.0
    return max(errs) + pad


def check_group_norm(n=2, c=320, h=32, w=32, silu=True, dt=torch.float16, pitch_extra=0, eps=1e-5,
                     seed=5, fused=True, adversarial=None):
    """`adversarial`: "mean50" (every value offset by 50: |mean| >> sigma, the case a raw
    sum-of-squares variance loses digits on), "outlier" (channel 7 scaled by 100, as real
    checkpoints have) -- compared against oracle/ops_oracle.py (two-pass fp32 statistics)."""
    lib = _lib.lib()
    torch.manual_seed(seed)
    ld = c + pitch_extra
    xb = torch.randn(n, h, w, ld, device=DEV)
    if adversarial == "mean50":
        xb = xb + 50.0
    elif adversarial == "outlier":
        xb[..., 7] *= 100.0
    xb = xb.to(dt)
    x = Act(xb, n, h, w, c, ld=ld)
    yb = torch.zeros(n, h, w, c, device=DEV, dtype=dt)
    y = Act(yb, n, h, w, c)
    gamma = torch.randn(c, device=DEV)
    beta = torch.randn(c, device=DEV)
    stats = torch.full((ops.gn_ws_floats(n, 32),), float("nan"), device=DEV)  # workspace: never needs zeroing
    sync = torch.zeros(4, device=DEV, dtype=torch.int32)
    gops = ops.gn_ops("gn", lib, x=x, y=y, gamma=gamma, beta=beta, stats=stats, groups=32, eps=eps,
                      silu=silu, dt=dt, sync=sync if fused else None)
    assert len(gops) == (1 if fused else 2), [o.name for o in gops]
    for op in gops:
        op.launch(_stream())
    torch.cuda.synchronize()
    if adversarial:
        from oracle import ops_oracle as oo
        ref = oo.group_norm(x.tensor().permute(0, 3, 1, 2).float(), 32, gamma, beta, eps, silu)
        return rel_err(yb, ref.permute(0, 2, 3, 1))
    ref = F.group_norm(x.tensor().permute(0, 3, 1, 2).float(), 32, gamma, beta, eps)
    if silu:
        ref = F.silu(ref)
    return rel_err(yb, ref.permute(0, 2, 3, 1))


def check_group_norm_bitwise_replay(n=2, c=960, h=64, w=64, fused=True, dt=torch.float16):
    """Two launches over the same input give bit-identical outputs (ordered reductions, no fp atomics)."""
    lib = _lib.lib()
    torch.manual_seed(5)
    xb = (torch.randn(n, h, w, c, device=DEV) * 3 + 1).to(dt)
    x = Act(xb, n, h, w, c)
    gamma, beta = torch.randn(c, device=DEV), torch.randn(c, device=DEV)
    outs = []
    for rep in range(3):
        yb = torch.zeros(n, h, w, c, device=DEV, dtype=dt)
        stats = torch.full((ops.gn_ws_floats(n, 32),), float(rep), device=DEV)  # stale garbage must not matter
        sync = torch.zeros(4, device=DEV, dtype=torch.int32)
        gops = ops.gn_ops("gn", lib, x=x, y=Act(yb, n, h, w, c), gamma=gamma, beta=beta, stats=stats, groups=32,
                          eps=1e-5, silu=True, dt=dt, sync=sync if fused else None)
        assert len(gops) == (1 if fused else 2)
        for op in gops:
            op.launch(_stream())
        torch.cuda.synchronize()
        outs.append(yb)
    return 0.0 if (torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])) else 1.0


def check_gn_finish(n=2, h=16, w=16, cin=1280, cout=1280, extra=0, splits=4, rowbias=True,
                    residual=True, silu=True, dt=torch.float16, seed=21):
    """Split-K conv launched with defer_finish + fused GroupNorm that sums the fp32 partials,
    applies the conv's bias / time-embedding row bias / residual, writes the finished activation
    and normalises it -- against conv -> (+adds) -> GroupNorm(+SiLU) in fp32.  `extra` channels of
    the GroupNorm input come from an ordinary tensor slice (the zero-copy skip concat)."""
    lib = _lib.lib()
    torch.manual_seed(seed)
    xin = _rand(n, h, w, cin, dt=dt)
    wt = _rand(cout, cin, 3, 3, dt=dt, scale=1 / math.sqrt(9 * cin))
    b = torch.randn(cout, device=DEV)
    M = n * h * w
    rb = torch.randn(n, cout, device=DEV) if rowbias else None
    r = _rand(M, cout, dt=dt) if residual else None
    C = cout + extra
    cat = _rand(n, h, w, C, dt=dt)          # [conv output slice | skip slice]
    skip_ref = cat[..., cout:].clone()
    cat[..., :cout] = 7.0                     # must be overwritten by the GroupNorm kernel
    box_n, box_h, box_w = ops.conv_tile_box(h, w)
    adesc = ops.a_conv(xin.data_ptr(), n, h, w, cin, cin, box_n, box_h, box_w, 1)
    ws = torch.empty(splits * M * cout, device=DEV, dtype=torch.float32)
    conv = ops.gemm_op("conv", lib, a=adesc, b=ops.Mat(ops.pack_conv3x3(wt, dt)), M=M, N=cout, K=9 * cin,
                       dt=dt, out=cat.data_ptr(), ldo=C, bias=b, rowbias=rb, rows_per_img=h * w,
                       ld_rowbias=cout, residual=r, ldr=cout, ws=ws, splits=splits, persistent=False,
                       conv=dict(n=n, h=h, w=w, cin=cin, stride=1, box_n=box_n, box_h=box_h, box_w=box_w))
    assert conv.keep[0].splits == splits
    conv.keep[0].defer_finish = 1
    x = Act(cat, n, h, w, C)
    yb = torch.zeros(n, h, w, C, device=DEV, dtype=dt)
    gamma, beta = torch.randn(C, device=DEV), torch.randn(C, device=DEV)
    stats = torch.full((ops.gn_ws_floats(n, 32),), float("nan"), device=DEV)
    sync = torch.zeros(4, device=DEV, dtype=torch.int32)
    part = dict(splits=splits, c=cout, ld=cout, bias=b, ws=ws)
    if rowbias:
        part.update(rowbias=rb.data_ptr(), ld_rowbias=cout)
    if residual:
        part.update(residual=r.data_ptr(), ldr=cout)
    gops = ops.gn_ops("gn", lib, x=x, y=Act(yb, n, h, w, C), gamma=gamma, beta=beta, stats=stats,
                      groups=32, eps=1e-5, silu=silu, dt=dt, sync=sync, partial=part)
    assert len(gops) == 1
    n0 = lib.sfb_launch_count()
    conv.launch(_stream())
    assert lib.sfb_launch_count() - n0 == 1, "deferred finish must not launch the reduction kernel"
    gops[0].launch(_stream())
    torch.cuda.synchronize()
    ref = F.conv2d(xin.permute(0, 3, 1, 2).float(), wt.float(), b, padding=1)
    if rowbias:
        ref = ref + rb[:, :, None, None]
    ref = ref.permute(0, 2, 3, 1)
    if residual:
        ref = ref + r.float().view(n, h, w, cout)
    e_x = rel_err(cat[..., :cout], ref)
    assert torch.equal(cat[..., cout:], skip_ref)
    full = torch.cat([cat[..., :cout].float(), skip_ref.float()], -1)  # what the kernel normalised
    gref = F.group_norm(full.permute(0, 3, 1, 2), 32, gamma, beta, 1e-5)
    if silu:
        gref = F.silu(gref)
    return max(e_x, rel_err(yb, gref.permute(0, 2, 3, 1)))


def check_layer_norm(rows=1151, c=1280, dt=torch.float16, seed=6):
    lib = _lib.lib()
    x = _rand(rows, c, dt=dt, seed=seed)
    y = torch.zeros_like(x)
    gamma = torch.randn(c, device=DEV)
    beta = torch.randn(c, device=DEV)
    ops.ln_op("ln", lib, x=x, y=y, rows=rows, c=c, gamma=gamma, beta=beta, eps=1e-5,
              dt=dt).launch(_stream())
    torch.cuda.synchronize()
    return rel_err(y, F.layer_norm(x.float(), (c,), gamma, beta, 1e-5))


def check_timestep_embed(batch=3, dim=320, dt=torch.float16):
    lib = _lib.lib()
    t = torch.tensor([999.0, 500.0, 1.0], device=DEV)[:batch]
    out = torch.zeros(batch, dim, device=DEV, dtype=dt)
    _lib.check(lib.sfb_timestep_embed(t.data_ptr(), batch, dim, 1, 0.0, out.data_ptr(), dim,
                                      ops.dtype_code(dt), _stream()))
    torch.cuda.synchronize()
    half = dim // 2
    ex = -math.log(10000) * torch.arange(half, device=DEV, dtype=torch.float32) / half
    emb = t[:, None] * torch.exp(ex)[None]
    ref = torch.cat([torch.cos(emb), torch.sin(emb)], dim=-1)
    return (out.float() - ref).abs().max().item()


def check_small_linear(batch=11, n=1280, k=320, act_out=1, dt=torch.float16, seed=7):
    lib = _lib.lib()
    x = _rand(batch, k, dt=dt, seed=seed)
    w = _rand(n, k, dt=dt, scale=1 / math.sqrt(k))
    b = torch.randn(n, device=DEV)
    add = _rand(batch, n, dt=dt)
    y16 = torch.zeros(batch, n, device=DEV, dtype=dt)
    y32 = torch.zeros(batch, n, device=DEV)
    ops.small_linear_op("sl", lib, x=x, w=w, bias=b, batch=batch, n=n, k=k, dt=dt, y16=y16,
                        y32=y32, add16=add, act_out=act_out).launch(_stream())
    torch.cuda.synchronize()
    ref = x.float() @ w.float().t() + b + add.float()
    if act_out:
        ref = F.silu(ref)
    return max(rel_err(y16, ref), rel_err(y32, ref))


def check_conv_in(n=2, h=64, w=64, cin=4, cout=320, dt=torch.float16, seed=8):
    lib = _lib.lib()
    x = _rand(n, cin, h, w, dt=dt, seed=seed)
    wt = _rand(cout, cin, 3, 3, dt=dt, scale=0.2)
    b = torch.randn(cout, device=DEV)
    wp = ops.pack_conv_in(wt, dt)
    y = torch.zeros(n, h, w, cout, device=DEV, dtype=dt)
    _lib.check(lib.sfb_conv_in(x.data_ptr(), wp.data_ptr(), b.data_ptr(), y.data_ptr(), n, h, w,
                               cin, cout, cout, ops.dtype_code(dt), _stream()))
    torch.cuda.synchronize()
    ref = F.conv2d(x.float(), wt.float(), b, padding=1).permute(0, 2, 3, 1)
    return rel_err(y, ref)


def check_conv_in_gemm(n=2, h=64, w=64, cin=4, cout=320, dt=torch.float16, seed=13):
    """First conv as im2col (K padded to 64) + the wgmma GEMM with fused bias."""
    lib = _lib.lib()
    x = _rand(n, cin, h, w, dt=dt, seed=seed)
    wt = _rand(cout, cin, 3, 3, dt=dt, scale=0.2)
    b = torch.randn(cout, device=DEV)
    wp = torch.zeros(cout, 64, device=DEV, dtype=dt)
    wp[:, :9 * cin] = ops.pack_conv3x3(wt, dt)
    M = n * h * w
    a = torch.zeros(M, 64, device=DEV, dtype=dt)
    y = torch.zeros(M, cout, device=DEV, dtype=dt)
    _lib.check(lib.sfb_im2col_in(x.data_ptr(), a.data_ptr(), n, h, w, cin, _stream()))
    ops.gemm_op("conv_in", lib, a=ops.a_matrix(a.data_ptr(), M, 64, 64), b=ops.Mat(wp), M=M, N=cout, K=64,
                dt=dt, out=y, ldo=cout, bias=b).launch(_stream())
    torch.cuda.synchronize()
    ref = F.conv2d(x.float(), wt.float(), b, padding=1).permute(0, 2, 3, 1).reshape(M, cout)
    return rel_err(y, ref)


def check_conv_out(n=2, h=64, w=64, cin=320, cout=4, dt=torch.float16, seed=9):
    lib = _lib.lib()
    x = _rand(n, h, w, cin, dt=dt, seed=seed)
    wt = _rand(cout, cin, 3, 3, dt=dt, scale=1 / math.sqrt(9 * cin))
    b = torch.randn(cout, device=DEV)
    wp = ops.pack_conv3x3(wt, dt)
    y = torch.zeros(n, cout, h, w, device=DEV, dtype=dt)
    _lib.check(lib.sfb_conv_out(x.data_ptr(), wp.data_ptr(), b.data_ptr(), y.data_ptr(), n, h, w,
                                cin, cout, cin, ops.dtype_code(dt), _stream()))
    torch.cuda.synchronize()
    ref = F.conv2d(x.permute(0, 3, 1, 2).float(), wt.float(), b, padding=1)
    return rel_err(y, ref)


def check_upsample(n=2, h=16, w=16, c=1280, dt=torch.float16):
    lib = _lib.lib()
    x = _rand(n, h, w, c, dt=dt, seed=10)
    y = torch.zeros(n, 2 * h, 2 * w, c, device=DEV, dtype=dt)
    _lib.check(lib.sfb_upsample2x(x.data_ptr(), y.data_ptr(), n, h, w, c, c, c, _stream()))
    torch.cuda.synchronize()
    ref = F.interpolate(x.permute(0, 3, 1, 2).float(), scale_factor=2.0, mode="nearest")
    return rel_err(y, ref.permute(0, 2, 3, 1))




def check_ln_fold(M=300, C=320, N=960, dt=torch.float16, mode="store", splits_p=1, splits_c=1, seed=12,
                  persistent=False, row_offset=0.5, outlier=False):
    """LayerNorm folded around two GEMMs: the producer accumulates per-row (sum, sum of squares)
    in its epilogue, the consumer runs on the RAW activation with gamma-scaled weights and
    corrects with mean / rstd in its epilogue.  Reference: F.layer_norm then the linear / GEGLU."""
    lib = _lib.lib()
    torch.manual_seed(seed)
    a = _rand(M, C, dt=dt)
    w0 = _rand(C, C, dt=dt, scale=1 / math.sqrt(C))
    res = torch.randn(M, C, device=DEV) * 2.0 + row_offset   # non-zero-mean rows (row_offset >> sigma: adversarial)
    if outlier:
        res[:, 5] *= 40.0                                      # one outlier channel, as real checkpoints have
    res = res.to(dt)
    x = torch.zeros(M, C, device=DEV, dtype=dt)
    slots = ops.rowstats_slots(C)
    stats = ops.RowStats(torch.zeros(M, slots, 2, device=DEV), slots)   # cleared by the caller, slots written once
    ws = torch.empty(16 * M * max(N, C) * 2, device=DEV, dtype=torch.float32)
    ops.gemm_op("producer", lib, a=ops.a_matrix(a.data_ptr(), M, C, C), b=ops.Mat(w0),
                M=M, N=C, K=C, dt=dt, out=x, ldo=C, residual=res, ldr=C, ws=ws, splits=splits_p,
                rowstats_out=stats, persistent=persistent).launch(_stream())
    gamma = torch.randn(C, device=DEV) * 0.5 + 1.0
    beta = torch.randn(C, device=DEV) * 0.3
    if mode == "geglu":
        inner = N
        w = _rand(2 * inner, C, dt=dt, scale=1 / math.sqrt(C))
        b = torch.randn(2 * inner, device=DEV) * 0.1
        wp, bias, colsum = ops.fold_layer_norm(w, b, gamma, beta, dt)
        wt, bp, _, cs = ops.pack_geglu(wp, bias, dt, extra=colsum)
        out = torch.zeros(M, inner, device=DEV, dtype=dt)
        ops.gemm_op("consumer", lib, a=ops.a_matrix(x.data_ptr(), M, C, C),
                    b=ops.Mat(wt), M=M, N=wt.shape[0], K=C, dt=dt, out=out, ldo=inner, bias=bp,
                    epi=ops.EPI_GEGLU, geglu_n_out=inner, ws=ws, splits=splits_c, persistent=persistent,
                    ln=dict(rowstats=stats, colsum=cs, eps=1e-5, dim=C)).launch(_stream())
    else:
        w = _rand(N, C, dt=dt, scale=1 / math.sqrt(C))
        b = torch.randn(N, device=DEV) * 0.1
        wp, bias, colsum = ops.fold_layer_norm(w, b, gamma, beta, dt)
        out = torch.zeros(M, N, device=DEV, dtype=dt)
        ops.gemm_op("consumer", lib, a=ops.a_matrix(x.data_ptr(), M, C, C),
                    b=ops.Mat(wp.contiguous()), M=M, N=N, K=C, dt=dt, out=out, ldo=N, bias=bias,
                    ws=ws, splits=splits_c, persistent=persistent,
                    ln=dict(rowstats=stats, colsum=colsum, eps=1e-5, dim=C)).launch(_stream())
    torch.cuda.synchronize()
    xr = (a.float() @ w0.float().t() + res.float())
    e0 = rel_err(x, xr)
    if row_offset != 0.5 or outlier:
        from oracle import ops_oracle as oo
        y = oo.layer_norm(x.float(), gamma, beta, 1e-5) @ w.float().t() + b
    else:
        y = F.layer_norm(x.float(), (C,), gamma, beta, 1e-5) @ w.float().t() + b
    if mode == "geglu":
        h, g = y.chunk(2, dim=-1)
        y = h * F.gelu(g)
    return max(e0, rel_err(out, y))




# ------------------------------------------------------------------------------------------
# SVD temporal path
def check_temporal_attention(B=2, F_=25, S=64, H=5, dt=torch.float16, seed=31):
    """Self-attention across frames on the fused QKV projection in the SPATIAL row order, against
    diffusers' formulation: reshape to [B*S, F, C], scaled_dot_product_attention, reshape back."""
    lib = _lib.lib()
    D, C_ = 64, H * 64
    torch.manual_seed(seed)
    rows = B * F_ * S
    qkv = _rand(rows, 3 * C_, dt=dt)
    out = torch.zeros(rows, C_, device=DEV, dtype=dt)
    p = _lib.TemporalAttnParams()
    p.qkv, p.out = qkv.data_ptr(), out.data_ptr()
    p.batch, p.frames, p.seq, p.heads, p.head_dim = B, F_, S, H, D
    p.ld_qkv, p.ld_out, p.dtype, p.scale = 3 * C_, C_, ops.dtype_code(dt), D ** -0.5
    import ctypes
    _lib.check(lib.sfb_temporal_attention(ctypes.byref(p), _stream()))
    torch.cuda.synchronize()
    x = qkv.float().view(B, F_, S, 3, H, D).permute(3, 0, 2, 4, 1, 5)  # [3, B, S, H, F, D]
    ref = F.scaled_dot_product_attention(x[0], x[1], x[2])             # [B, S, H, F, D]
    ref = ref.permute(0, 3, 1, 2, 4).reshape(rows, C_)
    return rel_err(out, ref)


def check_row_ops(B=2, F_=6, S=48, c=320, dt=torch.float16, seed=32):
    """sfb_row_broadcast_add (both index modes) and sfb_alpha_blend, with their row statistics."""
    import ctypes
    lib = _lib.lib()
    torch.manual_seed(seed)
    rows = B * F_ * S
    x = _rand(rows, c, dt=dt)
    errs = []

    def run(fn, **kw):
        p = _lib.RowOpParams()
        y = torch.zeros(rows, c, device=DEV, dtype=dt)
        st = torch.full((rows, 2), 7.0, device=DEV)
        p.x, p.y, p.rowstats_out = x.data_ptr(), y.data_ptr(), st.data_ptr()
        p.rows, p.c, p.ldx, p.ldy, p.dtype = rows, c, c, c, ops.dtype_code(dt)
        p.frames, p.seq, p.batch = F_, S, B
        for k, v in kw.items():
            setattr(p, k, v)
        _lib.check(fn(ctypes.byref(p), _stream()))
        torch.cuda.synchronize()
        return y, st

    m = torch.arange(rows, device=DEV)
    # frame position embedding: vec[(m / S) % F]
    vec = _rand(F_, c, dt=dt)
    y, st = run(lib.sfb_row_broadcast_add, vec=vec.data_ptr(), ldv=c, mode=_lib.ROW_IDX_DIV_MOD, div=S, mod=F_)
    ref = x.float() + vec.float()[(m // S) % F_]
    errs.append(rel_err(y, ref))
    errs.append(rel_err(st[:, 0], y.float().sum(-1)) + rel_err(st[:, 1], (y.float() ** 2).sum(-1)))
    # per image: vec[(m / S) % (B * F)]
    vec = _rand(B * F_, c, dt=dt)
    y, _ = run(lib.sfb_row_broadcast_add, vec=vec.data_ptr(), ldv=c, mode=_lib.ROW_IDX_DIV_MOD, div=S, mod=B * F_)
    errs.append(rel_err(y, x.float() + vec.float()[m // S]))
    # temporal context (diffusers layout quirk): sequence j = b * S + p reads video j % B, first frame
    y, _ = run(lib.sfb_row_broadcast_add, vec=vec.data_ptr(), ldv=c, mode=_lib.ROW_IDX_TEMPORAL_CTX)
    b_, p_ = m // (F_ * S), m % S
    errs.append(rel_err(y, x.float() + vec.float()[((b_ * S + p_) % B) * F_]))
    # AlphaBlender
    x2 = _rand(rows, c, dt=dt)
    mix = torch.tensor([0.37], device=DEV)
    y, st = run(lib.sfb_alpha_blend, x2=x2.data_ptr(), ldx2=c, mix_factor=mix.data_ptr())
    al = torch.sigmoid(mix)
    errs.append(rel_err(y, al * x.float() + (1 - al) * x2.float()))
    errs.append(rel_err(st[:, 0], y.float().sum(-1)))
    return max(errs)


def check_conv_t(B=2, F_=25, h=8, w=16, cin=320, cout=320, dt=torch.float16, rowbias=True, residual=True,
                 persistent=False, seed=33):
    """Conv3d (3,1,1) over the frame axis as the SFB_A_CONV3X1 implicit GEMM vs F.conv3d."""
    lib = _lib.lib()
    torch.manual_seed(seed)
    S = h * w
    x = _rand(B * F_, h, w, cin, dt=dt)
    wt = _rand(cout, cin, 3, 1, 1, dt=dt, scale=1 / math.sqrt(3 * cin))
    b = torch.randn(cout, device=DEV)
    M = B * F_ * S
    rb = torch.randn(B, cout, device=DEV) if rowbias else None
    r = _rand(M, cout, dt=dt) if residual else None
    out = torch.zeros(M, cout, device=DEV, dtype=dt)
    wp = wt[:, :, :, 0, 0].permute(0, 2, 1).reshape(cout, 3 * cin).contiguous()
    bn, bh, bw = ops.conv_tile_box(F_, S)
    op = ops.gemm_op("conv_t", lib, a=ops.a_conv(x.data_ptr(), B, F_, S, cin, cin, bn, bh, bw, 1), b=ops.Mat(wp),
                     M=M, N=cout, K=3 * cin, dt=dt, out=out, ldo=cout, bias=b, rowbias=rb, rows_per_img=F_ * S,
                     ld_rowbias=cout, residual=r, ldr=cout, splits=1, persistent=persistent,
                     conv=dict(n=B, h=F_, w=S, cin=cin, stride=1, box_n=bn, box_h=bh, box_w=bw, temporal=True))
    op.launch(_stream())
    torch.cuda.synchronize()
    xin = x.float().view(B, F_, h, w, cin).permute(0, 4, 1, 2, 3)  # [B, C, F, H, W]
    ref = F.conv3d(xin, wt.float(), b, padding=(1, 0, 0))
    if rowbias:
        ref = ref + rb[:, :, None, None, None]
    ref = ref.permute(0, 2, 3, 4, 1).reshape(M, cout)
    if residual:
        ref = ref + r.float()
    return rel_err(out, ref)



# ------------------------------------------------------------------------------------------
# VAE decoder pieces
def check_gemm_plain_b(M=512, N=4096, K=512, dt=torch.float16, bias=False, persistent=False, seed=41):
    """Activation x activation GEMM: B is a plain row-major [N, K] matrix (Q K^T, P V, V^T = W X^T)."""
    lib = _lib.lib()
    torch.manual_seed(seed)
    a = _rand(M, K, dt=dt)
    bm = _rand(N, K, dt=dt, scale=1 / math.sqrt(K))
    b = torch.randn(N, device=DEV) if bias else None
    out = torch.zeros(M, N, device=DEV, dtype=dt)
    op = ops.gemm_op("plain_b", lib, a=ops.a_matrix(a.data_ptr(), M, K, K), b=ops.PlainB(bm.data_ptr(), N, K, K),
                     M=M, N=N, K=K, dt=dt, out=out, ldo=N, bias=b, splits=1, persistent=persistent)
    assert op.keep[0].b_plain == 1
    op.launch(_stream())
    torch.cuda.synchronize()
    ref = a.float() @ bm.float().t()
    if bias:
        ref = ref + b
    return rel_err(out, ref)


def check_row_softmax(rows=300, cols=4096, dt=torch.float16, f32_in=False, seed=42):
    lib = _lib.lib()
    torch.manual_seed(seed)
    if f32_in:  # fp32 scores, 16-bit probabilities written over the first half of each row
        x = torch.randn(rows, cols, device=DEV) * 6.0
        ref = torch.softmax(x, dim=-1)
        _lib.check(lib.sfb_row_softmax(x.data_ptr(), x.data_ptr(), rows, cols, cols, 2 * cols, 1,
                                       ops.dtype_code(dt), _stream()))
        torch.cuda.synchronize()
        got = x.view(dt).view(rows, 2 * cols)[:, :cols]
        return rel_err(got, ref)
    x = _rand(rows, cols, dt=dt, scale=3.0)
    ref = torch.softmax(x.float(), dim=-1)
    _lib.check(lib.sfb_row_softmax(x.data_ptr(), x.data_ptr(), rows, cols, cols, cols, 0, ops.dtype_code(dt), _stream()))
    torch.cuda.synchronize()
    return rel_err(x, ref)


def check_gemm_f32_out(M=1024, N=1024, K=512, dt=torch.float16, seed=44):
    """fp32 store epilogue (attention scores) with a plain-B operand."""
    lib = _lib.lib()
    torch.manual_seed(seed)
    a = _rand(M, K, dt=dt)
    bm = _rand(N, K, dt=dt, scale=1 / math.sqrt(K))
    out = torch.zeros(M, N, device=DEV, dtype=torch.float32)
    op = ops.gemm_op("f32", lib, a=ops.a_matrix(a.data_ptr(), M, K, K), b=ops.PlainB(bm.data_ptr(), N, K, K),
                     M=M, N=N, K=K, dt=dt, out=out, ldo=N, splits=1, epi=_lib.EPI_STORE_F32)
    op.launch(_stream())
    torch.cuda.synchronize()
    return rel_err(out, a.float() @ bm.float().t())


def check_pointwise(n=2, hw=4096, cin=4, cout=4, dt=torch.float16, seed=43):
    lib = _lib.lib()
    torch.manual_seed(seed)
    x = _rand(n, cin, hw, dt=dt)
    w = _rand(cout, cin, dt=dt)
    b = torch.randn(cout, device=DEV)
    y = torch.zeros(n, cout, hw, device=DEV, dtype=dt)
    _lib.check(lib.sfb_pointwise_nchw(x.data_ptr(), w.data_ptr(), b.data_ptr(), y.data_ptr(), n, hw, cin, cout,
                                      ops.dtype_code(dt), _stream()))
    torch.cuda.synchronize()
    ref = torch.einsum("oc,ncp->nop", w.float(), x.float()) + b[None, :, None]
    return rel_err(y, ref)


CHECKS = {
    "gemm_small": (lambda: check_gemm(300, 320, 320), 2e-3),
    "gemm_k64": (lambda: check_gemm(128, 160, 64, bias=False, residual=False), 2e-3),
    "gemm_big": (lambda: check_gemm(8192, 1280, 1280), 2e-3),
    "gemm_splitk": (lambda: check_gemm(256, 1280, 5120, splits=8), 2e-3),
    "gemm_splitk_18": (lambda: check_gemm(128, 1280, 11520, splits=18), 2e-3),
    "group_norm_960_64_barrier_kernel": (lambda: check_group_norm(2, 960, 64, 64), 1e-2),
    "group_norm_320_64_b1": (lambda: check_group_norm(1, 320, 64, 64), 1e-2),
    "group_norm_1280_8_b16": (lambda: check_group_norm(16, 1280, 8, 8, silu=False, eps=1e-6), 1e-2),
    "group_norm_2560_16_pitch_bf16": (lambda: check_group_norm(2, 2560, 16, 16, dt=torch.bfloat16, pitch_extra=64), 4e-2),
    "upconv_32": (lambda: check_upconv(2, 32, 32, 640, 640, splits=1), 3e-3),
    "upconv_16": (lambda: check_upconv(2, 16, 16, 1280, 1280), 3e-3),
    "upconv_8_splitk": (lambda: check_upconv(2, 8, 8, 1280, 1280), 3e-3),
    "upconv_16_nopair_pitch": (lambda: check_upconv(1, 16, 16, 320, 320, pair=False, out_extra=320, splits=1), 3e-3),
    "upconv_64_bf16": (lambda: check_upconv(1, 64, 64, 320, 320, dt=torch.bfloat16, splits=1), 2e-2),
    "upconv_4_multi_image": (lambda: check_upconv(8, 4, 4, 256, 256, splits=1), 3e-3),
    "gn_finish_16": (lambda: check_gn_finish(2, 16, 16, 1280, 1280, splits=4), 3e-3),
    "gn_finish_8_s13": (lambda: check_gn_finish(2, 8, 8, 1280, 1280, splits=13), 3e-3),
    "gn_finish_concat": (lambda: check_gn_finish(2, 16, 16, 1280, 1280, extra=640, splits=4, rowbias=False), 3e-3),
    "gn_finish_32_s2": (lambda: check_gn_finish(2, 32, 32, 640, 640, extra=320, splits=2, residual=False), 3e-3),
    "gn_finish_plain": (lambda: check_gn_finish(1, 16, 16, 640, 1280, splits=3, rowbias=False, residual=False,
                                                silu=False), 3e-3),
    "gn_finish_bf16": (lambda: check_gn_finish(2, 16, 16, 1280, 1280, splits=4, dt=torch.bfloat16), 2e-2),
    "gemm_s2": (lambda: check_gemm(512, 1280, 1280, splits=2), 2e-3),
    "gemm_s4_pair": (lambda: check_gemm(256, 1280, 5120, splits=4, pair=True), 2e-3),
    "gemm_s4_nopair": (lambda: check_gemm(256, 1280, 5120, splits=4, pair=False), 2e-3),
    "gemm_s3_ragged": (lambda: check_gemm(300, 480, 2560, splits=3), 2e-3),
    "gemm_s2_bf16": (lambda: check_gemm(512, 640, 1280, splits=2, dt=torch.bfloat16), 1e-2),
    # persistent 256 x 320 pair kernel (forced, whatever the size policy would pick): more tiles than
    # SM pairs (several tiles per CTA: accumulator rotation, phase bits), ragged M / N, odd number of
    # 160-column tiles (single-half tiles), every epilogue and A mode
    "persist_gemm_big": (lambda: check_gemm(8192, 1280, 1280, persistent=True), 2e-3),
    "persist_gemm_many_tiles": (lambda: check_gemm(16384 + 256, 1920, 320, persistent=True), 2e-3),
    "persist_gemm_one_half": (lambda: check_gemm(4096, 160, 640, persistent=True), 2e-3),
    "persist_gemm_odd_halves": (lambda: check_gemm(2048, 480, 320, persistent=True), 2e-3),
    "persist_gemm_ragged": (lambda: check_gemm(400, 488, 320, persistent=True), 2e-3),
    "persist_gemm_k64_nobias": (lambda: check_gemm(8192, 320, 64, bias=False, residual=False, persistent=True), 2e-3),
    "persist_gemm_bf16": (lambda: check_gemm(4096, 640, 640, dt=torch.bfloat16, persistent=True), 1e-2),
    "persist_geglu": (lambda: check_geglu(8192, 320, 1280, persistent=True), 2e-2),
    "persist_geglu_ragged": (lambda: check_geglu(500, 64, 280, persistent=True), 2e-2),
    "persist_geglu_bf16": (lambda: check_geglu(2048, 640, 2560, dt=torch.bfloat16, persistent=True), 2e-2),
    "persist_conv_64": (lambda: check_conv(4, 64, 64, 320, 320, splits=1, persistent=True), 2e-3),
    "persist_conv_32_b8": (lambda: check_conv(8, 32, 32, 640, 640, splits=1, persistent=True), 2e-3),
    "persist_conv_8_multi_image": (lambda: check_conv(16, 8, 8, 1280, 1280, splits=1, persistent=True), 2e-3),
    "persist_conv_4_tiny": (lambda: check_conv(64, 4, 4, 256, 256, splits=1, persistent=True), 2e-3),
    "persist_conv_concat_pitch": (lambda: check_conv(2, 32, 32, 640, 320, pitch_extra=320, splits=1, persistent=True), 2e-3),
    "persist_conv_patch_96": (lambda: check_conv(2, 96, 96, 320, 320, splits=1, persistent=True), 2e-3),
    "persist_conv_stride2": (lambda: check_conv(2, 64, 64, 320, 320, stride=2, residual=False, rowbias=False,
                                                splits=1, persistent=True), 2e-3),
    "persist_upconv_32": (lambda: check_upconv(2, 32, 32, 640, 640, splits=1, persistent=True), 3e-3),
    "persist_upconv_16_pitch": (lambda: check_upconv(2, 16, 16, 320, 320, out_extra=320, splits=1, persistent=True), 3e-3),
    "persist_qkv_scatter": (lambda: check_qkv_scatter(2, 8, 1024, 40, persistent=True), 2e-3),
    "persist_qkv_scatter_d80": (lambda: check_qkv_scatter(2, 8, 512, 80, persistent=True), 2e-3),
    "persist_kv_scatter_cross": (lambda: check_qkv_scatter(6, 8, 256, 40, cross_kv=77, persistent=True), 2e-3),
    "persist_ln_fold": (lambda: check_ln_fold(2048, 320, 960, persistent=True), 5e-3),
    "persist_ln_fold_1280": (lambda: check_ln_fold(1024, 1280, 1280, persistent=True), 5e-3),
    "persist_ln_fold_geglu": (lambda: check_ln_fold(1024, 640, 2560, mode="geglu", persistent=True), 2e-2),
    # VAE decoder pieces
    "gemm_plain_b_vt": (lambda: check_gemm_plain_b(512, 4096, 512), 2e-3),
    "gemm_plain_b_scores": (lambda: check_gemm_plain_b(4096, 4096, 512), 2e-3),
    "gemm_plain_b_pv": (lambda: check_gemm_plain_b(4096, 512, 4096, bias=True), 2e-3),
    "gemm_plain_b_ragged": (lambda: check_gemm_plain_b(256, 1024, 128), 2e-3),
    "gemm_plain_b_bf16_persistent": (lambda: check_gemm_plain_b(4096, 4096, 512, dt=torch.bfloat16, persistent=True), 1e-2),
    "row_softmax": (lambda: check_row_softmax(), 2e-3),
    "row_softmax_f32_in_place": (lambda: check_row_softmax(257, 4096, f32_in=True), 2e-3),
    "row_softmax_f32_bf16": (lambda: check_row_softmax(64, 256, dt=torch.bfloat16, f32_in=True), 1e-2),
    "gemm_f32_out": (lambda: check_gemm_f32_out(), 1e-5),
    "gemm_f32_out_ragged_bf16": (lambda: check_gemm_f32_out(384, 384, 128, dt=torch.bfloat16), 1e-5),
    "row_softmax_1024_bf16": (lambda: check_row_softmax(64, 1024, dt=torch.bfloat16), 1e-2),
    "pointwise_nchw": (lambda: check_pointwise(), 2e-3),
    # SVD temporal path
    "temporal_attn_25": (lambda: check_temporal_attention(2, 25, 64, 5), 5e-3),
    "temporal_attn_6_d64x4": (lambda: check_temporal_attention(1, 6, 37, 4), 5e-3),
    "temporal_attn_32_bf16": (lambda: check_temporal_attention(2, 32, 16, 10, dt=torch.bfloat16), 2e-2),
    "row_ops": (lambda: check_row_ops(), 2e-3),
    "row_ops_1280_bf16": (lambda: check_row_ops(3, 5, 20, 1280, dt=torch.bfloat16), 1e-2),
    "conv_t_25": (lambda: check_conv_t(2, 25, 8, 16, 320, 320), 2e-3),
    "conv_t_small_frames": (lambda: check_conv_t(2, 6, 4, 4, 256, 256), 2e-3),
    "conv_t_patch_9x16": (lambda: check_conv_t(1, 25, 9, 16, 1280, 1280, rowbias=False), 2e-3),
    "conv_t_big": (lambda: check_conv_t(2, 25, 36, 64, 640, 640), 2e-3),
    "conv_t_persistent": (lambda: check_conv_t(2, 25, 16, 32, 320, 320, persistent=True), 2e-3),
    "gemm_pair": (lambda: check_gemm(512, 320, 640, pair=True), 2e-3),
    "gemm_pair_big": (lambda: check_gemm(8192, 1280, 1280, pair=True), 2e-3),
    "gemm_pair_ragged": (lambda: check_gemm(300, 480, 320, pair=True), 2e-3),
    "gemm_pair_splitk": (lambda: check_gemm(256, 1280, 5120, splits=8, pair=True), 2e-3),
    "gemm_pair_bf16": (lambda: check_gemm(512, 320, 320, dt=torch.bfloat16, pair=True), 1e-2),
    "conv_pair_64": (lambda: check_conv(2, 64, 64, 320, 320, splits=1, pair=True), 2e-3),
    "conv_pair_16_splitk": (lambda: check_conv(2, 16, 16, 1280, 1280, pair=True), 2e-3),
    "conv_pair_8": (lambda: check_conv(4, 8, 8, 1280, 1280, pair=True), 2e-3),
    "conv_pair_stride2": (lambda: check_conv(2, 64, 64, 320, 320, stride=2, residual=False, rowbias=False, pair=True), 2e-3),
    "gemm_1024_640": (lambda: check_gemm(1024, 640, 640), 2e-3),
    "gemm_500_480": (lambda: check_gemm(500, 480, 320), 2e-3),
    "gemm_256_640_splitk": (lambda: check_gemm(256, 640, 2560, splits=4), 2e-3),
    "gemm_bf16": (lambda: check_gemm(300, 320, 320, dt=torch.bfloat16), 1e-2),
    "geglu": (lambda: check_geglu(256, 320, 1280), 2e-2),
    "geglu_ragged": (lambda: check_geglu(100, 64, 256), 2e-2),
    "geglu_splitk": (lambda: check_geglu(128, 1280, 5120, splits=4), 2e-2),
    "ln_fold": (lambda: check_ln_fold(300, 320, 960), 5e-3),
    "ln_fold_1280": (lambda: check_ln_fold(512, 1280, 1280), 5e-3),
    "ln_fold_geglu": (lambda: check_ln_fold(300, 320, 1280, mode="geglu"), 2e-2),
    "ln_fold_splitk": (lambda: check_ln_fold(256, 1280, 1280, splits_p=2, splits_c=2), 5e-3),
    "ln_fold_geglu_splitk": (lambda: check_ln_fold(128, 1280, 5120, mode="geglu", splits_c=2), 2e-2),
    "conv_gn_64": (lambda: check_conv_gn(2, 64, 64, 320, 320, replay=True), 4e-3),
    "conv_gn_32_640": (lambda: check_conv_gn(2, 32, 32, 640, 640), 4e-3),
    "conv_gn_16_one_block": (lambda: check_conv_gn(2, 16, 16, 64, 160, groups=8, rowbias=False, residual=False), 4e-3),
    "conv_gn_concat_pitch": (lambda: check_conv_gn(2, 32, 32, 960, 320, pitch_extra=320, out_extra=160), 4e-3),
    "conv_gn_24_ragged_rows": (lambda: check_conv_gn(2, 24, 24, 640, 320), 4e-3),
    "conv_gn_40x24_ragged_n": (lambda: check_conv_gn(2, 40, 24, 320, 488), 4e-3),
    "conv_gn_mean50": (lambda: check_conv_gn(2, 32, 32, 320, 320, mean=50.0), 1e-2),
    "conv_gn_nosilu": (lambda: check_conv_gn(2, 32, 32, 320, 320, silu=False), 4e-3),
    "conv_gn_b8": (lambda: check_conv_gn(8, 64, 64, 320, 320), 4e-3),
    "conv_gn_bf16": (lambda: check_conv_gn(2, 32, 32, 640, 640, dt=torch.bfloat16), 3e-2),
    "conv_64": (lambda: check_conv(2, 64, 64, 320, 320, splits=1), 2e-3),
    "conv_32": (lambda: check_conv(2, 32, 32, 640, 640, splits=1), 2e-3),
    "conv_16_splitk": (lambda: check_conv(2, 16, 16, 1280, 1280), 2e-3),
    "conv_8_multi_image": (lambda: check_conv(3, 8, 8, 1280, 1280), 2e-3),
    "conv_4_tiny": (lambda: check_conv(5, 4, 4, 256, 256), 2e-3),
    "conv_concat_pitch": (lambda: check_conv(2, 32, 32, 640, 320, pitch_extra=320, splits=1), 2e-3),
    "conv_patch_96": (lambda: check_conv(1, 96, 96, 320, 320, splits=1), 2e-3),
    "conv_patch_24_splitk": (lambda: check_conv(2, 24, 24, 640, 640), 2e-3),
    "conv_patch_12x20": (lambda: check_conv(2, 12, 20, 1280, 640), 2e-3),
    "conv_patch_13x19": (lambda: check_conv(1, 13, 19, 256, 320, splits=1), 2e-3),
    "conv_patch_stride2_96": (lambda: check_conv(1, 96, 96, 320, 320, stride=2, residual=False,
                                                 rowbias=False, splits=1), 2e-3),
    "conv_patch_nopair_40x24": (lambda: check_conv(1, 40, 24, 320, 320, pair=False, splits=1), 2e-3),
    "upconv_patch_48": (lambda: check_upconv(1, 48, 48, 320, 320, splits=1), 3e-3),
    "upconv_patch_12": (lambda: check_upconv(2, 12, 12, 1280, 1280), 3e-3),
    "conv_stride2": (lambda: check_conv(2, 64, 64, 320, 320, stride=2, residual=False,
                                        rowbias=False), 2e-3),
    "conv_stride2_16": (lambda: check_conv(2, 16, 16, 1280, 1280, stride=2, residual=False,
                                           rowbias=False), 2e-3),
    # both attention kernels for every head_dim they exist for, whatever the default policy picks
    "attn_v2_d40": (lambda: check_attention(2, 8, 1024, None, 40, kv_tile=64), 5e-3),
    "attn_v2_d32": (lambda: check_attention(1, 4, 320, None, 32, kv_tile=64), 5e-3),
    "attn_v2_d64_4096": (lambda: check_attention(1, 10, 4096, None, 64, kv_tile=64), 5e-3),
    "attn_v2_d64_bf16_ragged": (lambda: check_attention(2, 5, 200, 333, 64, dt=torch.bfloat16, kv_tile=64), 2e-2),
    "attn_v2_cross77": (lambda: check_attention(2, 8, 1024, 77, 40, kv_tile=64), 5e-3),
    "attn_v2_one_tile": (lambda: check_attention(2, 8, 256, 40, 64, kv_tile=64), 5e-3),
    # causal self-attention of the CLIP text encoders (77 tokens; and several query / key tiles)
    "attn_v2_causal_77": (lambda: check_attention(2, 12, 77, None, 64, kv_tile=64, causal=True), 5e-3),
    "attn_v2_causal_77_bf16": (lambda: check_attention(1, 20, 77, None, 64, dt=torch.bfloat16, kv_tile=64, causal=True), 2e-2),
    "attn_v2_causal_300": (lambda: check_attention(2, 4, 300, None, 64, kv_tile=64, causal=True), 5e-3),
    "attn_v2_causal_d32": (lambda: check_attention(2, 4, 200, None, 32, kv_tile=64, causal=True), 5e-3),
    "gemm_act_quick_gelu": (lambda: check_gemm(154, 3072, 768, residual=False, act=_lib.ACT_QUICK_GELU), 2e-3),
    "gemm_act_gelu_bf16": (lambda: check_gemm(77, 5120, 1280, dt=torch.bfloat16, residual=False, act=_lib.ACT_GELU), 1e-2),
    "gemm_act_gelu_pair_residual": (lambda: check_gemm(512, 640, 320, pair=True, act=_lib.ACT_GELU), 2e-3),
    "embed_tokens": (lambda: check_embed_tokens(), 2e-3),
    "embed_tokens_bf16": (lambda: check_embed_tokens(2, 50, 1280, 5000, dt=torch.bfloat16), 1e-2),
    "clip_pool_legacy_argmax": (lambda: check_clip_pool(2), 0.0),
    "clip_pool_eos": (lambda: check_clip_pool(49407), 0.0),
    "patchify_14": (lambda: check_patchify(), 0.0),
    "patchify_224_bf16": (lambda: check_patchify(1, 3, 224, 14, 640, dt=torch.bfloat16), 0.0),
    "patchify_16": (lambda: check_patchify(3, 3, 64, 16, 768), 0.0),
    "attn_v1_d64": (lambda: check_attention(2, 8, 512, None, 64, kv_tile=128), 5e-3),
    "attn_d40": (lambda: check_attention(2, 8, 1024, None, 40), 5e-3),
    "attn_d40_4096": (lambda: check_attention(1, 8, 4096, None, 40), 5e-3),
    "attn_d80": (lambda: check_attention(2, 8, 256, None, 80), 5e-3),
    "attn_d160": (lambda: check_attention(2, 8, 64, None, 160), 5e-3),
    "attn_v1_d160": (lambda: check_attention(2, 8, 300, None, 160, kv_tile=128), 5e-3),
    "attn_v2_d160_ragged": (lambda: check_attention(2, 4, 300, 333, 160, kv_tile=64), 5e-3),
    "attn_d64": (lambda: check_attention(1, 10, 384, None, 64), 5e-3),
    "attn_d32": (lambda: check_attention(1, 2, 1024, None, 32), 5e-3),
    "attn_cross77": (lambda: check_attention(2, 8, 1024, 77, 40), 5e-3),
    "attn_cross77_d160": (lambda: check_attention(2, 8, 64, 77, 160), 5e-3),
    "attn_ragged_q": (lambda: check_attention(1, 8, 200, 300, 80), 5e-3),
    "qkv_scatter": (lambda: check_qkv_scatter(2, 8, 256, 40), 2e-3),
    "qkv_scatter_d160": (lambda: check_qkv_scatter(2, 8, 64, 160), 2e-3),
    "kv_scatter_cross": (lambda: check_qkv_scatter(2, 8, 256, 40, cross_kv=77), 2e-3),
    # adversarial statistics (vs oracle/ops_oracle.py): |mean| >> sigma, one outlier channel
    "group_norm_mean50": (lambda: check_group_norm(2, 320, 32, 32, True, adversarial="mean50"), 1e-2),
    "group_norm_mean50_two_pass": (lambda: check_group_norm(4, 320, 64, 64, True, fused=False, adversarial="mean50"), 1e-2),
    "group_norm_outlier": (lambda: check_group_norm(2, 640, 16, 16, True, adversarial="outlier"), 1e-2),
    "group_norm_outlier_two_pass": (lambda: check_group_norm(2, 640, 16, 16, False, fused=False, adversarial="outlier"), 1e-2),
    "ln_fold_mean30": (lambda: check_ln_fold(300, 320, 960, row_offset=30.0), 1e-2),
    "ln_fold_mean30_1280": (lambda: check_ln_fold(256, 1280, 1280, row_offset=30.0), 1e-2),
    "ln_fold_outlier": (lambda: check_ln_fold(300, 640, 640, outlier=True), 1e-2),
    "ln_fold_geglu_mean30": (lambda: check_ln_fold(300, 320, 1280, mode="geglu", row_offset=30.0), 2e-2),
    "group_norm_bitwise_replay_fused": (lambda: check_group_norm_bitwise_replay(), 0.0),
    "group_norm_bitwise_replay_two_pass": (lambda: check_group_norm_bitwise_replay(16, 320, 64, 64, fused=False), 0.0),
    "group_norm_silu": (lambda: check_group_norm(2, 320, 32, 32, True), 1e-2),
    "group_norm": (lambda: check_group_norm(2, 320, 32, 32, False, eps=1e-6), 1e-2),
    "group_norm_1920_pitch": (lambda: check_group_norm(2, 1920, 16, 16, True, pitch_extra=640), 1e-2),
    "group_norm_2560": (lambda: check_group_norm(3, 2560, 8, 8, True), 1e-2),
    "group_norm_64": (lambda: check_group_norm(1, 64, 32, 32, True), 1e-2),
    "group_norm_two_pass": (lambda: check_group_norm(2, 320, 32, 32, True, fused=False), 1e-2),
    "group_norm_two_pass_big": (lambda: check_group_norm(16, 320, 64, 64, True, fused=False), 1e-2),
    "group_norm_fused_64x64": (lambda: check_group_norm(2, 960, 64, 64, True, pitch_extra=0), 1e-2),
    "layer_norm": (lambda: check_layer_norm(1151, 1280), 1e-2),
    "layer_norm_320": (lambda: check_layer_norm(8192, 320), 1e-2),
    "timestep_embed": (lambda: check_timestep_embed(), 2e-3),
    "small_linear": (lambda: check_small_linear(), 2e-3),
    "small_linear_noact": (lambda: check_small_linear(2, 960, 1280, act_out=0), 2e-3),
    "conv_in": (lambda: check_conv_in(), 2e-3),
    "conv_in_gemm": (lambda: check_conv_in_gemm(), 2e-3),
    "conv_in_gemm_ragged": (lambda: check_conv_in_gemm(3, 8, 16, 4, 64), 2e-3),
    "conv_out": (lambda: check_conv_out(), 2e-3),
    "upsample": (lambda: check_upsample(), 0.0),
}


def main(argv):
    names = argv or list(CHECKS)
    ok = True
    for name in names:
        fn, tol = CHECKS[name]
        try:
            err = fn()
            passed = bool(err <= tol) and err == err
            print(json.dumps({"check": name, "err": err, "tol": tol, "pass": passed}), flush=True)
        except Exception as e:  # noqa: BLE001
            passed = False
            print(json.dumps({"check": name, "error": repr(e)[:300], "pass": False}), flush=True)
        ok = ok and passed
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
