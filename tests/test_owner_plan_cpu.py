"""The owner plan every multi-GPU exchange uses (mhb_plan_count_owner_rounds), for the stages that histogram 256
leading bytes and pass no cap: seq2sdbg's items, iterate's edges and the count's SdBG items.  Each rank's 256 bins are
placed at buckets b << 8; the plan must then be one round whose owner ranges follow multigpu.plan_ranges (the rule of
owner_bounds) and whose blocks are, per owner, each rank's records in the owner's bytes, placed in rank order."""
import numpy as np
import pytest

from megahit_b200 import lib, multigpu


def byte_hists(kind, n_ranks, rng):
    h = np.zeros((n_ranks, 256), np.uint64)
    if kind == "random":
        h[:] = rng.integers(0, 5000, (n_ranks, 256))
    elif kind == "a_skewed":  # canonical (k+1)-mers: heavy towards A-prefixes, a poly-A byte, empty bytes
        w = np.exp(-np.arange(256) / 20.0) * (rng.random(256) < 0.7)
        w[0] *= 40
        for r in range(n_ranks):
            h[r] = rng.multinomial(100000 + 31 * r, w / w.sum())
    elif kind == "single_byte":
        h[:, int(rng.integers(0, 256))] = rng.integers(0, 10**6, n_ranks)
    return h


@pytest.mark.parametrize("kind", ["random", "a_skewed", "single_byte", "empty"])
@pytest.mark.parametrize("n_ranks", [1, 2, 3, 5, 8, 16])
def test_uncapped_byte_plan_is_one_round_of_the_owner_rule(kind, n_ranks):
    rng = np.random.default_rng(1000 * n_ranks + len(kind))
    h256 = byte_hists(kind, n_ranks, rng)
    h16 = np.zeros((n_ranks, 65536), np.uint64)
    h16[:, ::256] = h256
    plan = lib.plan_count_owner_rounds(h16)

    assert plan["rounds"] == 1
    bounds = multigpu.plan_ranges(h256.sum(axis=0), n_ranks)
    assert plan["owners"] == [(int(bounds[o]) << 8, (int(bounds[o + 1]) << 8) - 1) for o in range(n_ranks)]
    for o in range(n_ranks):
        assert (int(plan["lo"][0, o]), int(plan["hi"][0, o])) == plan["owners"][o]
        send = h256[:, bounds[o]:bounds[o + 1]].sum(axis=1).astype(np.uint64)  # what each rank sends to o
        assert (plan["n"][0, o] == send).all()
        assert (plan["off"][0, o] == np.concatenate([[0], np.cumsum(send)[:-1]]).astype(np.uint64)).all()
