"""Host validation of the ABI boundary sweep (tests/abi_sweep.py), no GPU needed.

  * every sweep case gets past the real library's argument validation and fails only at the CUDA launch
    (SFB_ERR_CUDA on a box without a GPU), so the GPU sweep runs kernels, not refusals;
  * every "one step outside" twin of a boundary is refused with SFB_ERR_INVALID, and the error names the
    field that crossed it.
"""
import ctypes

import pytest
import torch

import abi_sweep as sw
import plan_launches as pl
from sfast_b200 import _lib
from test_host_logic import _DUMMY_PTR, _clone

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="needs a box without a GPU: launches must fail")

_CASES = sw.cases()


def _fill(struct, fields):
    for f in fields:
        if not getattr(struct, f):
            setattr(struct, f, _DUMMY_PTR)


def _call(op):
    """Call the real entry point of a dry sweep op with a dummy host pointer for every operand the op
    passes; returns (rc, last error)."""
    lib = _lib.lib()
    name = op.fn.name
    if name in pl.PLAIN:
        args = [(_DUMMY_PTR if a.endswith("*") else v) for a, v in zip(pl.PLAIN[name], op.args)]
        rc = getattr(lib, name)(*args, None)
    elif name == "sfb_attention_ip":
        p = _clone(op.keep[0])
        _fill(p.base, ["tmap_q", "tmap_k", "tmap_vt", "out"])
        _fill(p, ["tmap_k_ip", "tmap_vt_ip", "ip_scale"])
        rc = lib.sfb_attention_ip(ctypes.byref(p), None)
    else:
        p = _clone(op.keep[0])
        _fill(p, [f for f, on in pl._nonnull(op).items() if on])
        if name == "sfb_group_norm_scale_shift":
            rc = lib.sfb_group_norm_scale_shift(ctypes.byref(p), _DUMMY_PTR, None)
        else:
            rc = getattr(lib, name)(ctypes.byref(p), None)
    return rc, lib.sfb_last_error().decode()


def test_sweep_cases_are_distinct_and_cover_every_family():
    assert len({c.cid for c in _CASES}) == len(_CASES)
    assert {c.family for c in _CASES} == set(sw.FAMILIES)


def test_attention_sweep_covers_every_dispatched_pair_and_sequence_edge():
    seen = {}
    for c in _CASES:
        q = c.params
        if c.family == "attention" and "seq_kv" in q:
            s = seen.setdefault((q["head_dim"], q["kv_tile"]), [set(), set()])
            s[0].add(q["seq_q"])
            s[1].add(q["seq_kv"])
    assert set(seen) == set(sw.ATTN_PAIRS) and (128, 128) in seen
    for sq, skv in seen.values():
        assert sq == set(sw.SEQ_Q) and skv == set(sw.SEQ_KV)


@pytest.mark.parametrize("case", _CASES, ids=[c.cid for c in _CASES])
def test_sweep_case_passes_host_validation(case):
    rc, err = _call(case.op())
    assert rc != 0, "launched without a GPU?"
    assert rc == -2, f"host validation refused a sweep case: {err}"


@pytest.mark.parametrize("what,build,word", sw.ONE_STEP_OUTSIDE, ids=[t[0] for t in sw.ONE_STEP_OUTSIDE])
def test_one_step_outside_is_refused_by_name(what, build, word):
    with pl.recording_map_offsets():
        op = build()
    rc, err = _call(op)
    assert rc == -1, f"{what}: not refused (rc {rc}: {err})"
    assert word in err, f"{what}: the error does not name {word!r}: {err}"


def test_fused_group_norm_limit_matches_the_fits_predicate():
    """The largest-tensor fused case sits exactly on the boundary of sfb_group_norm_fused_fits, whose
    Python mirror (dry plans) agrees with it on both sides; the n limit is the SM count."""
    from sfast_b200 import ops
    lib = _lib.lib()
    n, c, g = sw.GN_FUSED_LIMIT
    hw = sw.fused_hw_limit(n, c, g)
    assert lib.sfb_group_norm_fused_fits(ctypes.byref(sw.gn_params(n, hw, c, g))) == 1
    assert lib.sfb_group_norm_fused_fits(ctypes.byref(sw.gn_params(n, hw + 1, c, g))) == 0
    assert ops.gn_fused_fits(n, hw, c, g) and not ops.gn_fused_fits(n, hw + 1, c, g)
    sms = lib.sfb_sm_count()
    assert lib.sfb_group_norm_fused_fits(ctypes.byref(sw.gn_params(sms, 1, 64, 8))) == 1
    assert lib.sfb_group_norm_fused_fits(ctypes.byref(sw.gn_params(sms + 1, 1, 64, 8))) == 0
    assert lib.sfb_group_norm_ws_floats(n, g) == ops.gn_ws_floats(n, g)


def test_rowstats_slots_export_matches_python_mirror():
    from sfast_b200 import ops
    lib = _lib.lib()
    for n_cols in (8, 152, 160, 168, 256, 320, 328, 1280, 5120):
        assert lib.sfb_rowstats_slots(n_cols) == ops.rowstats_slots(n_cols)
