"""Every distinct kernel launch of the shipped launch plans, replayed once on fresh seeded inputs and compared
with a float64 reference (tests/plan_launches.py), one test per plan family.  A key two families emit is
replayed by the first of them (UNet, SVD, VAE decode, VAE encode, CLIP).

All ~2,600 keys of the 33 plans replay in under a minute (H100 80GB HBM3 at a 400 W power limit; peak ~29 GiB
allocated), so every key runs, as `python tests/plan_launches.py --all` does; tests/golden/plan_launches_h100.json
holds the errors of such a run.  Each key also checks the access model of tests/plan_hazards.py against its launches:
its writes on every key, its reads on the default subset (2,620 and 260 keys; with these checks the file took ~95 s
on an H100 80GB HBM3, peak ~40 GiB)."""
import pytest
import torch

import plan_launches as pl

pytestmark = pytest.mark.gpu

_STATE = {}


def _entries():
    if "entries" not in _STATE:
        entries, names = pl.collect()
        assert not pl.check_coverage(names)
        _STATE.update(entries=entries, keys=list(entries), done=set())
    return _STATE["entries"]


@pytest.mark.parametrize("family", pl.FAMILIES)
def test_plan_launches_match_float64_reference(family):
    entries = _entries()
    keys = [k for k in _STATE["keys"] if entries[k]["family"] == family and k not in _STATE["done"]]
    assert keys, f"no launches for family {family}"
    # the access model of tests/plan_hazards.py: its writes checked on every key, its reads on the default subset
    sub = set(_STATE.setdefault("subset", pl.select_subset(entries)))
    sound = {k: "rw" if k in sub else "w" for k in keys}
    failures = []
    for rec in pl.run_keys(entries, keys, soundness=sound):
        if not rec["ok"]:
            failures.append(f"{rec['desc']} [{','.join(rec['plans'][:3])}] peaked={rec['peaked']}: "
                            f"{rec.get('error') or [p for p in rec['parts'] if p[1] > p[2]]} {rec.get('model', '')}")
    _STATE["done"].update(keys)
    print(f"{family}: {len(keys)} keys ({len(keys)} with the access model's writes checked, "
          f"{sum(v == 'rw' for v in sound.values())} with its reads), "
          f"peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")
    assert not failures, f"{len(failures)} failing launches:\n" + "\n".join(failures)
