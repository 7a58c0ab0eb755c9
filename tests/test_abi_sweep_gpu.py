"""The ABI boundary sweep (tests/abi_sweep.py) on the GPU: every case against its float64 reference with its
canvas intact, one test per case family; and the attention + GEMM families once more with programmatic
dependent launch off, which must not change a single output bit."""
import os

import pytest
import torch

import abi_sweep as sw
from sfast_b200 import _lib

pytestmark = pytest.mark.gpu


def _failures(records):
    return [f"{r['id']} peaked={r['peaked']}: {r.get('error') or [p for p in r['parts'] if p[1] > p[2]]}"
            for r in records if not r["ok"]]


@pytest.mark.parametrize("family", sorted(sw.FAMILIES))
def test_abi_sweep_matches_float64_reference(family):
    cs = sw.FAMILIES[family]()
    records = list(sw.run_cases(cs))
    bad = _failures(records)
    worst = max(records, key=lambda r: r["err"] / r["tol"] if r["tol"] else (0.0 if r["ok"] else float("inf")))
    print(f"{family}: {len(records)} runs, worst {worst['id']} err {worst['err']:.3g} tol {worst['tol']:.3g}, "
          f"peak {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    assert not bad, f"{len(bad)} failing sweep cases:\n" + "\n".join(bad)


def _outputs(cs):
    outs = []
    for case in cs:
        with sw.capturing_outputs() as got:
            assert sw.run_case(case).ok, case.cid
        outs.append([t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32) for t in got])
    return outs


def test_pdl_off_is_bit_identical_for_attention_and_gemm():
    cs = sw.attention_cases()[::3] + sw.gemm_cases()[::3]
    with_pdl = _outputs(cs)
    lib = _lib.lib()
    lib.sfb_set_pdl(0)
    try:
        without = _outputs(cs)
    finally:
        lib.sfb_set_pdl(int(int(os.environ.get("SFB_PDL", "1") or 0) != 0))   # the setting the library loaded with
    for case, a, b in zip(cs, with_pdl, without):
        assert len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b)), case.cid
