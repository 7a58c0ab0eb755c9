"""CPU side of the plan-launch replay (tests/plan_launches.py): every listed dry plan builds, every entry point
it launches has a replay, launch keys are stable, each float64 reference agrees with an independent form of the
same operation, and the comparison / canary checks reject small, realistic kernel mistakes."""
import collections

import pytest
import torch
import torch.nn.functional as F

import plan_launches as pl
from kernel_checks import rel_err
from oracle import vae_encoder_oracle as veo
from sfast_b200 import ops

D64 = torch.float64


@pytest.fixture(scope="module")
def entries():
    entries, names = pl.collect()
    return entries, names


def test_every_plan_builds_and_every_entry_point_is_replayed(entries):
    ents, names = entries
    assert pl.check_coverage(names) == []
    assert set(pl.SKIP) == {"sfb_memset"}
    replayed = {e["name"] for e in ents.values()}
    assert replayed == set(names) - set(pl.SKIP)
    for name in ("sfb_gemm", "sfb_attention", "sfb_group_norm_fused", "sfb_group_norm_stats", "sfb_group_norm_apply",
                 "sfb_group_norm_scale_shift", "sfb_small_linear", "sfb_temporal_attention", "sfb_row_broadcast_add",
                 "sfb_alpha_blend", "sfb_layer_norm", *pl.PLAIN, "sfb_add_nchw_residuals"):
        # the stand-alone nearest-2x upsample only runs when SFB_UPCONV=0 turns the folded up-conv off
        assert name in replayed or name == "sfb_upsample2x", name
    assert {e["family"] for e in ents.values()} == set(pl.FAMILIES)
    per = collections.Counter(e["name"] for e in ents.values())
    print(f"\n{len(ents)} distinct launches over {len(pl.PLANS)} plans; "
          f"default subset {len(pl.select_subset(ents))}")
    for name, n in per.most_common():
        print(f"  {name:32s} {n}")


def test_an_entry_point_without_a_replay_fails_the_coverage_check():
    class FakeFn:
        name = "sfb_new_kernel"

    fake = ops.Op("fake", FakeFn(), (), ())
    assert pl.check_coverage(["sfb_gemm", fake.fn.name, "sfb_memset"]) == ["sfb_new_kernel"]


def test_default_subset_covers_every_launch_class(entries):
    ents, _ = entries
    sub = set(pl.select_subset(ents))
    assert {pl.launch_class(k) for k in ents} == {pl.launch_class(k) for k in sub}
    # the largest launch of every entry point is in it
    for name in {e["name"] for e in ents.values()}:
        ks = [k for k in ents if ents[k]["name"] == name]
        top = max(pl.launch_work(k, ents[k]["op"]) for k in ks)
        assert any(pl.launch_work(k, ents[k]["op"]) == top for k in ks if k in sub), name


def test_keys_are_stable_and_shared_launches_collapse():
    a = [k for _, k, _ in pl.launches(pl.build_plan("tiny_2x32x32"))]
    b = [k for _, k, _ in pl.launches(pl.build_plan("tiny_2x32x32"))]
    assert a == b
    hash(tuple(a))
    ents, _ = pl.collect(["sd15_2x64x64", "sd15_controlnet_2x64x64"])
    shared = [e for e in ents.values() if e["plans"] == ["sd15_2x64x64", "sd15_controlnet_2x64x64"]]
    only = [e for e in ents.values() if e["plans"] == ["sd15_controlnet_2x64x64"]]
    # the residual add is new; it also keeps the mid block's last conv from deferring its split-K finish
    assert len(shared) > 100 and "sfb_add_nchw_residuals" in [e["name"] for e in only] and len(only) < 10


def test_keys_carry_the_buffer_offset_of_concat_slices():
    """Two launches that differ only in where their output sits inside a concat buffer are distinct keys."""
    plan = pl.build_plan("sd15_2x64x64")
    outs = collections.defaultdict(set)
    for name, key, op in pl.launches(plan):
        if name == "sfb_gemm":
            g = {kv[0]: kv for kv in key[1]}
            outs[(g["M"][-1], g["N"][-1], g["K"][-1], g["a_mode"][-1])].add(g["out"][-1])
    assert any(len(v) > 1 for v in outs.values())
    # the A operand's map records its base offset (a conv reading the skip half of a concat buffer)
    bases = {m.base for op in plan.all_ops() for m in op.keep if isinstance(m, ops.DryMap) and hasattr(m, "base")}
    assert len(bases) > 1


# ---------------------------------------------------------------------------------------------------------
# each reference against an independent form, tiny shapes, fp64 on the CPU
# ---------------------------------------------------------------------------------------------------------
def _im2col_conv(x, w, stride, pad):
    """x NHWC, w [cout, cin, 3, 3], pad = (top, bottom, left, right): explicit taps + one matmul."""
    n, h, wd, c = x.shape
    xp = F.pad(x, (0, 0, pad[2], pad[3], pad[0], pad[1]))
    ho, wo = (h + pad[0] + pad[1] - 3) // stride + 1, (wd + pad[2] + pad[3] - 3) // stride + 1
    cols = torch.stack([xp[:, kh:kh + stride * (ho - 1) + 1:stride, kw:kw + stride * (wo - 1) + 1:stride]
                        for kh in range(3) for kw in range(3)], 3)          # [n, ho, wo, 9, c]
    return cols.reshape(n * ho * wo, 9 * c) @ ops.pack_conv3x3(w, D64).t()


@pytest.mark.parametrize("stride", [1, 2])
def test_conv_reference_matches_im2col_matmul(stride):
    g = torch.Generator().manual_seed(0)
    x, w = torch.randn(2, 6, 10, 5, generator=g, dtype=D64), torch.randn(7, 5, 3, 3, generator=g, dtype=D64)
    got = pl.ref_conv3x3(x, w, stride).reshape(-1, 7)
    torch.testing.assert_close(got, _im2col_conv(x, w, stride, (1, 1, 1, 1)), rtol=1e-12, atol=1e-12)


def test_downconv_reference_matches_the_encoder_oracle_and_im2col():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 8, 12, 64, generator=g, dtype=D64)
    down = veo.VaeDownsample(64).double()
    ref = down(x.permute(0, 3, 1, 2)).permute(0, 2, 3, 1) - down.conv.bias.detach()
    got = pl.ref_downconv3x3(x, down.conv.weight.detach())
    torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(got.reshape(-1, 64), _im2col_conv(x, down.conv.weight.detach(), 2, (0, 1, 0, 1)),
                               rtol=1e-12, atol=1e-12)


def test_upconv_phase_reference_matches_upsample_then_conv():
    g = torch.Generator().manual_seed(2)
    x, w = torch.randn(2, 5, 7, 3, generator=g, dtype=D64), torch.randn(6, 3, 3, 3, generator=g, dtype=D64)
    packed = ops.pack_upconv(w, D64)          # phase sums formed in fp32, not rounded to 16 bits
    up = F.interpolate(x.permute(0, 3, 1, 2), scale_factor=2, mode="nearest")
    ref = F.conv2d(up, w, padding=1).permute(0, 2, 3, 1)
    torch.testing.assert_close(pl.ref_upconv_phases(x, packed, 6), ref, rtol=1e-5, atol=1e-5)


def test_conv3x1_and_conv_gn_references_match_explicit_forms():
    g = torch.Generator().manual_seed(3)
    x, w = torch.randn(2, 5, 6, 4, generator=g, dtype=D64), torch.randn(3, 4, 3, generator=g, dtype=D64)
    xp = F.pad(x, (0, 0, 0, 0, 1, 1))
    ref = sum(torch.einsum("nfpc,oc->nfpo", xp[:, t:t + 5], w[:, :, t]) for t in range(3))
    torch.testing.assert_close(pl.ref_conv3x1(x, w), ref, rtol=1e-12, atol=1e-12)
    xi, w3 = torch.randn(2, 5, 6, 4, generator=g, dtype=D64), torch.randn(3, 4, 3, 3, generator=g, dtype=D64)
    ss = torch.randn(2, 4, 2, generator=g, dtype=D64)
    y = F.silu(xi * ss[:, None, None, :, 0] + ss[:, None, None, :, 1])
    torch.testing.assert_close(pl.ref_conv3x3_gn(xi, w3, ss, True).reshape(-1, 3), _im2col_conv(y, w3, 1, (1, 1, 1, 1)),
                               rtol=1e-12, atol=1e-12)


def test_qkv_scatter_reference_follows_the_header_layout():
    g = torch.Generator().manual_seed(4)
    B, S, H, D = 2, 5, 3, 4
    for which_base, n_which in ((0, 3), (1, 2)):
        y = torch.randn(B * S, n_which * H * D, generator=g, dtype=D64)
        got = pl.ref_qkv_scatter(y, B, S, H, D, which_base)
        for m in range(B * S):
            b, s = divmod(m, S)
            for n in range(n_which * H * D):
                which = n // (H * D) + which_base
                h, d = divmod(n % (H * D), D)
                if which == 2:
                    assert got[2][b * H + h, d, s] == y[m, n]
                else:
                    assert got[which][b * H + h, s, d] == y[m, n]


def test_ln_fold_reference_equals_layer_norm_then_linear():
    g = torch.Generator().manual_seed(5)
    M, K, N = 7, 64, 9
    a = torch.randn(M, K, generator=g, dtype=D64) * 2 + 0.7
    w, b = torch.randn(N, K, generator=g, dtype=D64), torch.randn(N, generator=g, dtype=D64)
    gamma, beta = 1 + torch.randn(K, generator=g, dtype=D64), torch.randn(K, generator=g, dtype=D64)
    wp, bias, colsum = ops.fold_layer_norm(w, b, gamma, beta, D64)
    ref = F.layer_norm(a, (K,), gamma, beta, 1e-5) @ w.t() + b
    got = pl.ref_layer_norm_rows(a, 1e-5) @ wp.double().t() + bias.double()
    torch.testing.assert_close(got, ref, rtol=1e-5, atol=1e-5)        # bias / colsum come back in fp32
    # the epilogue form the kernel computes from (sum, sum of squares) agrees as well
    mean, var = a.mean(1, keepdim=True), a.var(1, unbiased=False, keepdim=True)
    epi = (a @ wp.double().t() - mean * colsum.double()) / torch.sqrt(var + 1e-5) + bias.double()
    torch.testing.assert_close(epi, ref, rtol=1e-5, atol=1e-5)


def test_split_slot_rowstats_add_up_to_the_unsplit_stats():
    torch.manual_seed(6)
    sums = torch.randn(50, 2, dtype=D64)
    for slots in (1, 2, 5, 9):
        st = pl.split_slots(sums, slots)
        assert st.shape == (50, slots, 2)
        torch.testing.assert_close(st.sum(1), sums, rtol=1e-12, atol=1e-12)
    st = pl.split_slots(sums, 9)
    assert bool((st[..., 0] == 0).any())                  # some rows leave trailing slots empty


def test_geglu_reference_matches_the_packing_round_trip():
    g = torch.Generator().manual_seed(7)
    inner, K, M = 200, 64, 5
    w, b = torch.randn(2 * inner, K, generator=g, dtype=D64), torch.randn(2 * inner, generator=g, dtype=D64)
    wt, bp, _ = ops.pack_geglu(w, b, D64)
    x = torch.randn(M, K, generator=g, dtype=D64)
    h, gate = (x @ w.t() + b).chunk(2, -1)
    torch.testing.assert_close(pl.ref_geglu(x @ wt.t() + bp.double(), inner), h * F.gelu(gate), rtol=1e-6, atol=1e-6)


# ---------------------------------------------------------------------------------------------------------
# sensitivity: small, realistic kernel mistakes on a tiny CPU output must be rejected
# ---------------------------------------------------------------------------------------------------------
def _fp16_out(M=300, N=480, seed=8):
    g = torch.Generator().manual_seed(seed)
    ref = torch.randn(M, N, generator=g, dtype=D64)
    return ref, ref.to(torch.float16)


def test_correctly_rounded_output_passes():
    ref, got = _fp16_out()
    assert rel_err(got, ref) <= pl.tol("gemm", torch.float16)


def test_one_tile_off_by_four_ulp_fails():
    ref, got = _fp16_out()
    bad = got.clone()
    t = bad[128:256, 160:320]
    for _ in range(4):
        t.copy_(torch.nextafter(t, torch.full_like(t, float("inf"))))
    assert rel_err(bad, ref) > pl.tol("gemm", torch.float16)


def test_zeroed_last_ragged_row_fails():
    ref, got = _fp16_out(M=300)
    bad = got.clone()
    bad[-1] = 0
    assert rel_err(bad, ref) > pl.tol("gemm", torch.float16)


def test_conv_gn_border_from_the_affine_of_zero_fails():
    """A halo conv that pads AFTER-the-affine border pixels with act(0 * scale + shift) instead of 0."""
    g = torch.Generator().manual_seed(9)
    x, w = torch.randn(2, 16, 8, 64, generator=g, dtype=D64), torch.randn(32, 64, 3, 3, generator=g, dtype=D64) / 24
    ss = torch.stack([1 + 0.5 * torch.randn(2, 64, generator=g, dtype=D64),
                      0.5 + torch.randn(2, 64, generator=g, dtype=D64)], -1)
    ref = pl.ref_conv3x3_gn(x, w, ss, True)
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))                             # border = raw zeros, then the affine
    yp = F.silu(xp * ss[:, None, None, :, 0] + ss[:, None, None, :, 1])
    wrong = F.conv2d(yp.permute(0, 3, 1, 2), w).permute(0, 2, 3, 1)
    assert rel_err(wrong.to(torch.float16), ref) > pl.tol("conv_gn", torch.float16)
    assert rel_err(ref.to(torch.float16), ref) <= pl.tol("conv_gn", torch.float16)


def test_a_value_in_the_pitch_gap_breaks_the_canary():
    cv = pl.Canvas(torch.float16, 64, 10, 96, device="cpu")
    cv.arm()
    out = cv.region(10, 80)
    out.fill_(1.5)                               # the declared output
    got = cv.take(out)
    assert cv.intact() and bool((got == 1.5).all())
    out.fill_(1.5)
    cv.t[64 + 3 * 96 + 80] = 0.0                 # one value in columns [N, ldo)
    cv.take(out)
    assert not cv.intact()
    cv.t.copy_(cv.before)
    cv.t[63] = 0.0                               # the leading offset
    assert not cv.intact()
    cv.t.copy_(cv.before)
    cv.t[64 + 10 * 96 + 5] = 0.0                 # the guard band past the last row
    assert not cv.intact()


def test_a_rowstats_slot_accumulated_instead_of_written_fails():
    g = torch.Generator().manual_seed(10)
    M, N = 40, 320
    stored = torch.randn(M, N, generator=g).to(torch.float16)
    slots = ops.rowstats_slots(N)
    good = torch.full((M, slots, 2), pl.STATS_SENT)
    o = stored.double()
    for s in range(2):                                   # two 160-column tiles write their slot
        seg = o[:, 160 * s:160 * (s + 1)]
        good[:, s, 0], good[:, s, 1] = seg.sum(1).float(), (seg * seg).sum(1).float()
    res = pl.Result()
    pl.check_rowstats(res, "rs", good, stored, N, torch.float16)
    assert res.ok, res.parts
    bad = good.clone()
    bad[:, 1] += pl.STATS_SENT                           # slot 1 accumulated onto what was there
    res = pl.Result()
    pl.check_rowstats(res, "rs", bad, stored, N, torch.float16)
    assert not res.ok
    bad = torch.cat([good, torch.full((M, 1, 2), pl.STATS_SENT)], 1)
    bad[:, slots] = 0.0                                  # a slot no producer of N columns owns
    res = pl.Result()
    pl.check_rowstats(res, "rs", bad, stored, N, torch.float16)
    assert not res.ok
