"""CPU: the blocked fp64 oracle of `tests/blocked_oracle.py` against `rank_oracle` and `ec.expected_padded`.

Integer-valued catalogues (tests/exact_cases.py) make every score exact and tie tens of objects on one value, so ties
straddle every block edge; blocks of 7, 64 and 1000 objects cut the catalogue at many places, with filters (empty rows,
everything-viewed rows, ids beyond the catalogue) and a whitelist."""
import numpy as np
import pytest

from oracle.topk_oracle import rank_oracle
from tests import exact_cases as ec
from tests.blocked_oracle import blocked_oracle
from tests.score_interval import from_keys as _from_keys
from tests.score_interval import order_keys as _order_keys

N_OBJ, D, N_ROWS = 3000, 6, 40


@pytest.fixture(scope="module")
def case():
    rng = np.random.default_rng(12)
    objects = ec.pooled_matrix(rng, N_OBJ, D, 200)
    subjects = ec.int_matrix(rng, N_ROWS, D)
    subjects[3] = 0  # every score 0
    rows = [rng.integers(0, N_OBJ + 40, rng.integers(0, 200)) for _ in range(N_ROWS)]
    rows[0], rows[1] = np.empty(0, np.int64), np.arange(N_OBJ)
    filt = ec.csr_from_rows(rows, N_OBJ)
    wl = np.sort(rng.choice(N_OBJ, 1700, replace=False))
    return objects, subjects, filt, wl


def test_order_keys_round_trip():
    sc = np.array([3.0, -0.0, 0.0, -1.5, np.finfo(np.float32).max, -np.finfo(np.float32).max, 1e-45, -1e-45], np.float32)
    ids = np.arange(len(sc), dtype=np.int64)[::-1].copy()
    keys = _order_keys(sc, ids)
    i2, s2 = _from_keys(keys)
    np.testing.assert_array_equal(i2, ids)
    np.testing.assert_array_equal(s2.view(np.int32), sc.view(np.int32))
    order = np.argsort(keys)
    exp = np.lexsort((ids, -sc.astype(np.float64)))
    # (-0.0 sorts after +0.0 here; lexsort holds them equal and orders them by id: only their places may differ)
    zero = sc == 0
    np.testing.assert_array_equal(order[~zero[order]], exp[~zero[exp]])


@pytest.mark.parametrize("block", [7, 64, 1000, 1 << 20])
@pytest.mark.parametrize("distance", ["dot", "cosine"])
@pytest.mark.parametrize("k", [1, 10, 65, None])
@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("whitelisted", [False, True])
def test_blocked_oracle_matches_rank_oracle(case, block, distance, k, filtered, whitelisted):
    objects, subjects, filt, wl = case
    f = filt if filtered else None
    w = wl if whitelisted else None
    got = blocked_oracle(distance, subjects, objects, k, f, w, block=block, row_block=16)
    exp = ec.expected_padded(distance, subjects, objects, np.arange(N_ROWS), k, f, w)
    ids, sc, cnt = got
    np.testing.assert_array_equal(cnt, exp[2])
    np.testing.assert_array_equal(ids, exp[0])
    np.testing.assert_array_equal(sc, exp[1])
    # the flat form of the reference restatement (COSINE: its scores are divided by the subject norm too)
    _, oid, osc = rank_oracle(distance, subjects, objects, np.arange(N_ROWS), k, f, w, accum="f64")
    valid = np.arange(ids.shape[1])[None, :] < cnt[:, None]
    np.testing.assert_array_equal(ids[valid], oid)
    flat = sc[valid]
    if distance == "cosine":
        flat = flat / np.repeat(ec.calc_norms(subjects, "f64"), cnt)
    np.testing.assert_array_equal(flat, osc)
