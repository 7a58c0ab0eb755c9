"""Ordering between the launches of the shipped plans (tests/plan_hazards.py), without a GPU: every plan's two-stream
schedule over two consecutive steps is free of races and stale reads, the analysis really examines the concurrent
launches, seeded ordering mistakes are each reported as the expected finding, and the strided-region overlap test
is exact at its edges."""
import time

import pytest
import torch

import plan_hazards as ph
import plan_launches as pl
from oracle import svd_vae_oracle as svo
from oracle import taesd_oracle as tao
from oracle import t2i_adapter_oracle as tio
from oracle import unet_oracle as uo
from sfast_b200.plan import PackedWeights, UNetPlan, _ForkOp, _JoinOp
from sfast_b200.unet_spec import (controlnet_spec_from_config, ip_adapter_geometry, ip_adapter_plus_geometry,
                                  param_shapes, spec_from_config)

CFGS = {"tiny": uo.tiny_config, "sd15": uo.sd15_config, "sdxl": uo.sdxl_config}
F16 = torch.float16


def _sd(shapes, dt=F16):
    return {k: torch.empty(tuple(v), dtype=dt, device="meta") for k, v in shapes.items()}


def _unet(cfg, b, h, w, dt=F16, ip=None, **kw):
    """Dry UNetPlan; ip = ("plain", d_img) for an IP-Adapter, ("plus", d_img, dim_head) for IP-Adapter Plus."""
    spec = spec_from_config(CFGS[cfg]())
    if ip is not None and ip[0] == "plain":
        spec.ip = ip_adapter_geometry(spec, ip[1])
    elif ip is not None:
        spec.ip = ip_adapter_plus_geometry(spec, ip[1], ip[2])
    return UNetPlan(PackedWeights(spec, _sd(param_shapes(spec), dt), dt, "meta", dry=True), b, h, w, **kw)


def _controlnet(cfg, b, h, w, dt=F16):
    from oracle import controlnet_oracle as co
    from sfast_b200.controlnet_plan import ControlNetPlan
    spec = controlnet_spec_from_config({"tiny": co.tiny_config, "sd15": co.sd15_config, "sdxl": co.sdxl_config}[cfg]())
    return ControlNetPlan(PackedWeights(spec, _sd(param_shapes(spec), dt), dt, "meta", dry=True), b, h, w)


def _adapter(cfg, b, h, w):
    from sfast_b200.t2i_adapter_plan import AdapterPlan, t2i_adapter_param_shapes, t2i_adapter_spec_from_config
    spec = t2i_adapter_spec_from_config(cfg)
    return AdapterPlan(PackedWeights(spec, _sd(t2i_adapter_param_shapes(spec)), F16, "meta", dry=True), b, h, w)


def _taesd(kind, b, h, w):
    from sfast_b200 import taesd_plan as tp
    spec = tp.taesd_spec_from_config(tao.tiny_config())
    shapes = {**tp.taesd_decoder_param_shapes(spec), **tp.taesd_encoder_param_shapes(spec)}
    wts = PackedWeights(spec, _sd(shapes), F16, "meta", dry=True)
    return (tp.TAESDDecodePlan if kind == "decode" else tp.TAESDEncodePlan)(wts, b, h, w)


def _temporal_decode(frames, nf, h, w):
    from sfast_b200.vae_plan import TemporalDecodePlan, vae_spec_from_config, vae_temporal_decoder_param_shapes
    spec = vae_spec_from_config(svo.svd_vae_config())
    return TemporalDecodePlan(PackedWeights(spec, _sd(vae_temporal_decoder_param_shapes(spec)), F16, "meta", dry=True),
                              frames, nf, h, w)


# every plan of plan_launches.PLANS, plus the feature plans those do not build
FEATURE_PLANS = [
    ("tiny_ip_2x32x32", lambda: _unet("tiny", 2, 32, 32, ip=("plain", 64), ip_len=4)),
    ("sd15_ip_2x64x64", lambda: _unet("sd15", 2, 64, 64, ip=("plain", 1024), ip_len=4)),
    ("sdxl_ip_vith_2x128x128", lambda: _unet("sdxl", 2, 128, 128, ip=("plain", 1280), ip_len=4)),
    ("tiny_ip_plus_1img_2x32x32", lambda: _unet("tiny", 2, 32, 32, ip=("plus", 128, 128), ip_len=16, ip_seq=257)),
    ("sd15_ip_plus_4img_1x64x64", lambda: _unet("sd15", 1, 64, 64, ip=("plus", 1280, 768), ip_len=64, ip_seq=257)),
    ("sdxl_ip_plus_1img_2x128x128", lambda: _unet("sdxl", 2, 128, 128, ip=("plus", 1280, 1280), ip_len=16,
                                                  ip_seq=257)),
    ("tiny_t2i_2x32x32", lambda: _unet("tiny", 2, 32, 32, intrablock=4)),
    ("sd15_t2i_2x64x64", lambda: _unet("sd15", 2, 64, 64, intrablock=4)),
    ("sdxl_t2i_mid_2x128x128", lambda: _unet("sdxl", 2, 128, 128, intrablock=4)),
    ("sd15_controlnet_t2i_2x64x64", lambda: _unet("sd15", 2, 64, 64, controlnet=True, intrablock=4)),
    ("tiny_controlnet_t2i_ip_2x32x32", lambda: _unet("tiny", 2, 32, 32, controlnet=True, intrablock=5,
                                                     ip=("plain", 64), ip_len=4)),
    ("controlnet_tiny_2x32x32", lambda: _controlnet("tiny", 2, 32, 32)),
    ("controlnet_sd15_2x64x64", lambda: _controlnet("sd15", 2, 64, 64)),
    ("controlnet_sdxl_2x128x128", lambda: _controlnet("sdxl", 2, 128, 128)),
    ("adapter_sd_2x512x512", lambda: _adapter(tio.sd_config(), 2, 512, 512)),
    ("adapter_sdxl_1x1024x1024", lambda: _adapter(tio.sdxl_config(), 1, 1024, 1024)),
    ("taesd_decode_1x64x64", lambda: _taesd("decode", 1, 64, 64)),
    ("taesd_encode_1x512x512", lambda: _taesd("encode", 1, 512, 512)),
    ("temporal_decode_6f3_40x64", lambda: _temporal_decode(6, 3, 40, 64)),
]
ALL_PLANS = [(n, b) for n, _, b in pl.PLANS] + FEATURE_PLANS


@pytest.mark.parametrize("name,builder", ALL_PLANS, ids=[n for n, _ in ALL_PLANS])
def test_every_shipped_plan_is_free_of_races_and_stale_reads(name, builder):
    t0 = time.time()
    plan, rep = ph.check_plan(builder)
    side = bool(plan.side_ops) or any(isinstance(op, _ForkOp) for op in plan.ops)
    print(f"\n{name}: {len(rep.events)} events over 2 steps, {rep.pairs} unordered (side, main) pairs examined, "
          f"{len(rep.declared)} declared cross-step reads, {time.time() - t0:.2f} s")
    assert not rep.findings, "\n".join(map(str, rep.findings))
    if side:
        assert rep.pairs > 0
    # the only cross-step reads: the tickets of each GroupNorm statistics launch that feeds a conv, read once
    n_ss = sum(1 for op in plan.all_ops() if op.fn is not None and op.fn.name == "sfb_group_norm_scale_shift")
    assert len(rep.declared) == n_ss, rep.declared
    assert all(ev.endswith("(sfb_group_norm_scale_shift)") and f == "sync_counter" and buf.startswith("gn_tickets")
               for ev, f, buf in rep.declared), rep.declared


def test_every_entry_point_the_plans_launch_is_modelled():
    names = set()
    for _, builder in ALL_PLANS:
        plan, space = ph.build(builder)
        with ph.virtual_addresses_of(space):
            for op in plan.all_ops() + [o for o in plan.ops if o.fn is not None]:
                names.add(ph._fn_name(op))
                ph.accesses(op)
    names.discard(None)
    assert names <= ph.MODELLED
    assert "sfb_memset" in names
    assert set(pl.check_coverage(names)) <= ph.MODELLED


# =====================================================================================================
# seeded mistakes: each is reported as exactly the expected finding
# =====================================================================================================
def _mutated(builder, mutate):
    plan, space = ph.build(builder)
    with ph.virtual_addresses_of(space):
        ctx = mutate(plan)
        return ph.analyse(plan, space), ctx


def _main_index(plan, pred, start=0):
    return next(i for i in range(start, len(plan.ops)) if pred(plan.ops[i]))


def _tiny():
    return _unet("tiny", 2, 32, 32)


def _forks(plan):
    return [i for i, op in enumerate(plan.ops) if isinstance(op, _ForkOp)]


def _join_of(plan, fork):
    return _main_index(plan, lambda o: isinstance(o, _JoinOp) and o.kind is fork)


def _only(rep, kind, buffer_prefix):
    assert rep.findings, "the mistake went unreported"
    for f in rep.findings:
        assert f.kind == kind and f.buffer.startswith(buffer_prefix), str(rep)


def test_a_missing_fork_join_is_a_race_on_the_shortcut_output():
    def mutate(plan):
        fork = plan.ops[_forks(plan)[0]]   # (a later fork's join still orders the branch before the next step)
        del plan.ops[_join_of(plan, fork)]
        return fork.branch[0].name
    rep, sc = _mutated(_tiny, mutate)
    conv2 = sc.replace(".conv_shortcut", ".conv2")
    assert any(f.kind == "race" and sc in f.a and conv2 in f.b and f.buffer.startswith("res_sc[")
               for f in rep.findings), str(rep)
    # and conv2 may read res_sc before anything wrote it this step: a later resnet of the same shape writes it
    for f in rep.findings:
        assert f.buffer.startswith("res_sc[") and (f.kind == "race" and sc in f.a or
                                                    f.kind == "stale read" and conv2 in f.a), str(rep)
    print("\n" + str(rep))


def test_a_late_first_join_is_a_race_on_the_hoisted_cross_attention_kv():
    def mutate(plan):
        j = _main_index(plan, lambda o: isinstance(o, _JoinOp) and o.kind == "all")
        join = plan.ops.pop(j)
        core = _main_index(plan, lambda o: o.name.endswith(".attn2.core"), j)
        plan.ops.insert(core + 1, join)
        return plan.ops[core].name
    rep, core = _mutated(_tiny, mutate)
    _only(rep, "race", "attn_")
    bufs = {f.buffer.split("[")[0] for f in rep.findings}
    assert {b.split("_")[1] for b in bufs} == {"k", "vt"}, bufs
    layer = core[:-len(".core")]
    assert all(f.buffer.endswith("@" + layer + "]") or ("@" + layer) in f.buffer for f in rep.findings), str(rep)
    assert all(layer + ".kv" in f.a and core in f.b for f in rep.findings), str(rep)
    print("\n" + str(rep))


def test_an_early_temb_event_is_a_race_on_the_time_embedding_projection():
    def mutate(plan):
        plan._temb_last = plan.side_ops[plan.side_ops.index(plan._temb_last) - 1]
    rep, _ = _mutated(_tiny, mutate)
    _only(rep, "race", "temb_proj[")
    assert all("time_emb_proj(all)" in f.a and ".conv1 " in f.b and f.fields[1] == "rowbias" for f in rep.findings)
    print("\n" + str(rep))


def test_a_shortcut_written_over_conv1_output_is_a_write_write_race():
    def mutate(plan):
        i = _forks(plan)[0]
        fork = plan.ops[i]
        conv1 = plan.ops[_main_index(plan, lambda o: o.name.endswith(".conv1"), i)]
        sc = fork.branch[0].keep[0]
        sc.out, sc.ldo = conv1.keep[0].out, conv1.keep[0].ldo
        return fork.branch[0].name, conv1.name
    rep, (sc, conv1) = _mutated(_tiny, mutate)
    assert any(f.kind == "race" and sc in f.a and conv1 in f.b and f.fields == ("out", "out") for f in rep.findings)
    # the rest follows from it: norm2 reads res_h1 while the shortcut may be writing it, and conv2 now reads a
    # res_sc that only a later resnet of the same shape writes
    conv2 = conv1.replace(".conv1", ".conv2")
    for f in rep.findings:
        assert (f.kind == "race" and f.buffer.startswith("res_h1[") and sc in f.a or
                f.kind == "stale read" and f.buffer.startswith("res_sc[") and conv2 in f.a), str(rep)
    print("\n" + str(rep))


def test_an_adapter_residual_added_before_its_producer_is_a_stale_read():
    def mutate(plan):
        i = _main_index(plan, lambda o: o.name == "t2i_adapter.residual.1")
        add = plan.ops[i]
        dst = [a for a in ph.accesses(add) if a.writes][0]
        prod = max(j for j in range(i) if not isinstance(plan.ops[j], (_ForkOp, _JoinOp))
                   and any(a.writes and ph.overlap(a, dst) for a in ph.accesses(plan.ops[j])))
        plan.ops.insert(prod, plan.ops.pop(i))
        return plan.ops[prod + 1].name
    rep, prod = _mutated(lambda: _unet("tiny", 2, 32, 32, intrablock=4), mutate)
    _only(rep, "stale read", "cat_")
    assert all("t2i_adapter.residual.1" in f.a and prod in f.b for f in rep.findings), str(rep)
    print("\n" + str(rep))


def test_a_missing_barrier_counter_reset_is_a_stale_read_modify_write():
    def mutate(plan):
        plan.ops.remove(next(o for o in plan.ops if o.name == "gn_sync.zero"))
    rep, _ = _mutated(_tiny, mutate)
    _only(rep, "stale read", "gn_sync")
    assert all("sfb_group_norm_fused" in f.a and f.fields == ("sync_counter", "sync_counter") for f in rep.findings)
    print("\n" + str(rep))


def test_a_side_op_left_unjoined_races_with_the_next_steps_copy_in():
    def mutate(plan):
        kv = next(o for o in plan.side_ops if o.name.endswith(".attn2.kv"))
        plan.ops.append(_ForkOp([kv]))   # re-issued after the last join, never joined
        return kv.name
    rep, kv = _mutated(_tiny, mutate)
    _only(rep, "race", "ehs_in")
    assert all(kv in f.a and f.a.startswith("step1:") and f.b == "step2:copy-in ehs_in" for f in rep.findings), str(rep)
    print("\n" + str(rep))


def test_a_write_into_a_prefetched_weight_is_reported():
    """Under programmatic dependent launch a GEMM reads its pre-tiled weights before waiting for its predecessor."""
    def mutate(plan):
        g = next(o for o in plan.ops if o.fn is not None and o.fn.name == "sfb_gemm" and not o.keep[0].b_plain)
        b = ph.accesses(g)[1]
        plan.ops.append(pl.ops.Op("poke", plan.lib_or_dry().sfb_memset, (b.addr, 0, 64), ()))
        return g.name
    rep, gemm = _mutated(_tiny, mutate)
    assert any(f.kind == "prefetched weight written" and "poke" in f.a and gemm in f.b for f in rep.findings), str(rep)
    assert all(f.a.split(" ")[1] == "poke" or f.b.split(" ")[1] == "poke" for f in rep.findings), str(rep)


# =====================================================================================================
# the overlap test at its edges
# =====================================================================================================
A = ph.Access


@pytest.mark.parametrize("a,b,want", [
    # equal pitch: the two column halves of one skip-concat buffer never meet
    (A("x", 0, 64, 64, 128, "w"), A("y", 64, 64, 64, 128, "w"), None),
    # touching column ranges (end of one row == start of the other's columns) do not overlap
    (A("x", 0, 64, 64, 128, "w"), A("y", 64, 1, 64, 0, "r"), None),
    # one byte of shared column overlaps
    (A("x", 0, 64, 65, 128, "w"), A("y", 64, 64, 64, 128, "r"), (64, 65)),
    # contiguous ranges that touch do not overlap; one byte more does
    (A("x", 0, 1, 100, 0, "w"), A("y", 100, 1, 10, 0, "r"), None),
    (A("x", 0, 1, 101, 0, "w"), A("y", 100, 1, 10, 0, "r"), (100, 101)),
    # rows past the other region's last row
    (A("x", 0, 4, 32, 128, "w"), A("y", 512, 4, 32, 128, "r"), None),
    (A("x", 0, 5, 32, 128, "w"), A("y", 512, 4, 32, 128, "r"), (512, 544)),
    # unequal pitches: x rows [0,32) of every 128 bytes, y rows [96, 160) of every 96 bytes
    (A("x", 0, 8, 32, 128, "w"), A("y", 96, 2, 24, 200, "r"), None),
    (A("x", 0, 8, 32, 128, "w"), A("y", 96, 3, 24, 200, "r"), (512, 520)),
    # a column slice at an offset inside a wider pitch (skip_dst written at a column offset)
    (A("x", 640, 1024, 640, 1280, "w"), A("y", 0, 1024, 640, 1280, "r"), None),
    (A("x", 638, 1024, 642, 1280, "w"), A("y", 0, 1024, 640, 1280, "r"), (638, 640)),
])
def test_overlap_is_exact_at_its_edges(a, b, want):
    assert ph.overlap(a, b) == want
    assert ph.overlap(b, a) == want


def test_coverage_of_a_read_by_several_writers():
    r = A("r", 0, 16, 64, 128, "r")
    halves = [A("w0", 0, 16, 32, 128, "w"), A("w1", 32, 16, 32, 128, "w")]
    assert ph.uncovered(r, [], halves) is None
    assert ph.uncovered(r, [], halves[:1]) == (32, 64)
    assert ph.contains(A("w", 0, 16, 64, 128, "w"), r)
    assert not ph.contains(A("w", 0, 15, 64, 128, "w"), r)
    assert not ph.contains(A("w", 0, 16, 64, 256, "w"), r)


def test_column_disjoint_concurrent_accesses_are_not_a_race():
    """Two launches on different streams, unordered, each writing one column half of the same buffer: no finding;
    the same launches writing overlapping columns: a race in the step and one into the next step."""
    t = torch.empty(2, 8, 8, 128, dtype=F16, device="meta")
    src = torch.empty(128, 128, dtype=F16, device="meta")

    class FakePlan:
        side_ops, ops, _bufs, _temb_last = [], [], {("cat_0_0", (2, 8, 8, 128), F16): t}, None

    def copy(name, col, cols):
        return pl.ops.Op(name, _Fn("sfb_copy2d"), (pl.ops._ptr(src), pl.ops._ptr(t) + 2 * col, 128, cols, 128, 128),
                         ())

    for col, want in ((64, 0), (63, 2)):
        with ph.virtual_addresses() as space:
            plan = FakePlan()
            plan.side_ops = [copy("left", 0, 64)]
            plan.ops = [copy("right", col, 64)]
            rep = ph.analyse(plan, space)
        assert len([f for f in rep.findings if f.kind == "race"]) == want, str(rep)
        assert rep.pairs == 3   # step 1 / step 1, step 1 / step 2 (never joined), step 2 / step 2


class _Fn:
    def __init__(self, name):
        self.name = name
