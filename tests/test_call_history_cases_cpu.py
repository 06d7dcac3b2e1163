"""CPU: the call sequences of tests/call_history_cases.py -- every route the long-lived engines of
tests/test_gpu_call_history.py must take, each directly after a larger call -- pinned through the plan of
rectools_b200/csrc/plan.h (tests/plan_driver.cpp, built as tests/test_call_plan_cpu.py builds it)."""
import numpy as np
import pytest

from tests import call_history_cases as ch
from tests.test_call_plan_cpu import driver  # noqa: F401  (the plan driver fixture)

MODES = dict(enumerate(ch.PATH_MODES))
SELECTS = dict(enumerate(ch.SELECTS))
PLANNED = ("topk", "rows", "sparse")  # routes of b200_rank_topk (path 5 has its own entry points)

# the route / tensor-core mode / selection combinations every suite of sequences reaches after a larger call
REQUIRED = {
    (0, None, None),
    (1, "narrow", None), (1, "wide", None), (1, "wide_l", None), (1, "multi_pass", None),
    (2, None, "passes"), (2, None, "radix"),
    (3, None, "passes"), (3, None, "radix"),
    (4, None, "radix"),
    (5, "host", None), (5, "device", None),
}
K_EDGES = {1, 24, 25, 128, 129, 1024, 1025, ch.S + 1, None}


def _combo(rec):
    if rec["path"] == 5:
        return 5, "host" if rec["route"] == "cand_host" else "device", None
    return rec["path"], rec["mode"], rec["select"]


@pytest.fixture(scope="module")
def sequences():
    return {e: ch.sequence(e) for e in ch.ENGINES}


def test_every_record_plans_to_its_route(driver, sequences):  # noqa: F811
    for engine, seq in sequences.items():
        recs = [r for r in ch.calls(seq) if r["route"] in PLANNED]
        plans = driver([ch.call_shape(engine, r) for r in recs])
        for r, p in zip(recs, plans):
            tag = f"{engine} record {r['i']}: {r}"
            assert p["error"] == 0, (tag, p["message"])
            assert p["path"] == r["path"] and p["k_out"] == ch.k_out(engine, r), (tag, p)
            if r["path"] == 1:
                assert MODES[p["mode"]] == r["mode"], (tag, p)
            if r["path"] in (2, 3, 4):
                assert SELECTS[p["select"]] == r["select"], (tag, p)
            if "B200_CHUNK_ROWS" in r["env"]:  # the forced chunks split the call
                assert p["n_chunks"] > 1, (tag, p)
        for r in ch.calls(seq):
            if r["route"] not in PLANNED:
                assert r["path"] == 5, r


def test_every_route_follows_a_larger_call(sequences):
    seen = set()
    for engine, seq in sequences.items():
        cs = ch.calls(seq)
        for prev, cur in zip(cs, cs[1:]):
            if cur["role"] == "checked":
                assert prev["role"] == "decoy" and prev["route"] == cur["route"], (engine, prev, cur)
                assert ch.larger(engine, prev, cur), (engine, ch.extent(engine, prev), ch.extent(engine, cur), cur)
                seen.add(_combo(cur))
    assert REQUIRED <= seen, REQUIRED - seen


def test_the_sequences_hold_the_edges(sequences):
    """k edges, rows from 1 to thousands, hooks and whitelists that change between calls, resident subjects replaced with
    another row count, device inputs and outputs."""
    dot = ch.calls(sequences["dot"])
    assert K_EDGES <= {r["k"] for r in dot}
    rows = [r["n_rows"] for r in dot]
    assert min(rows) == 1 and max(rows) > 2000
    for hook in ("B200_TC_SPLITS", "B200_TC_CAROUSEL", "B200_CHUNK_ROWS", "B200_WIDE", "B200_SELECT"):
        assert any(hook in a["env"] and hook not in b["env"] for a, b in zip(dot, dot[1:])), hook
    sq = ch.calls(sequences["square"])
    assert any(a["env"].get("B200_CHUNK_ROWS") != b["env"].get("B200_CHUNK_ROWS") and "B200_CHUNK_ROWS" in a["env"] and
               "B200_CHUNK_ROWS" in b["env"] for a, b in zip(sq, sq[1:]))
    for engine, seq in sequences.items():
        cs = ch.calls(seq)
        # two consecutive calls with equal-length, different whitelists (on the tensor-core path where a route allows)
        pairs = [(a, b) for a, b in zip(cs, cs[1:]) if a["wl"] and b["wl"] and a["wl"][1] == b["wl"][1] and a["wl"][0] != b["wl"][0]]
        assert pairs, engine
        if engine != "square":
            assert any(b["path"] == 1 for _, b in pairs), engine
            assert any(r["filter"] == "viewed_all" for r in cs), engine
            assert any(r["in_dev"] and r["out_dev"] for r in cs), engine
    for engine in ("dot", "cosine", "bf16"):
        sizes = [r["n_rows"] for r in sequences[engine] if r["route"] == "set_resident"]
        assert len(set(sizes)) == len(sizes) >= 2, engine
        seq = sequences[engine]
        for i, r in enumerate(seq):
            if r.get("source") == "resident":
                assert any(s["route"] == "set_resident" for s in seq[:i]), (engine, r)


def test_sequences_are_deterministic(sequences):
    for engine, seq in sequences.items():
        again = ch.sequence(engine)
        assert ch.dumps(again) == ch.dumps(seq), engine
        assert ch.loads(ch.dumps(seq)) == seq
        assert ch.dumps(ch.sequence(engine, seed=1)) != ch.dumps(seq), engine
    # the arrays of a record are a function of the record
    rec = next(r for r in ch.calls(sequences["dot"]) if r["filter"] and r["wl"])
    a, b = ch.inputs("dot", rec), ch.inputs("dot", dict(rec))
    for key in ("whitelist", "subjects"):
        np.testing.assert_array_equal(a[key], b[key])
    assert (a["filter"] != b["filter"]).nnz == 0


def test_decoys_rank_the_hot_block_first(sequences):
    """The planted block: first for every decoy row, last (below every other object) for every checked row -- on a few
    rows of each route, in fp64."""
    for engine in ch.ENGINES:
        objects = ch.catalogue(engine).astype(np.float64)
        if ch.ENGINES[engine]["cosine"]:
            objects /= np.linalg.norm(objects, axis=1, keepdims=True)
        hot = ch.hot_ids(engine)
        cold = np.setdiff1d(np.arange(len(objects)), hot)
        resident = None
        for rec in sequences[engine]:
            if rec["route"] == "set_resident":
                resident = ch.resident(engine, rec)
                continue
            x = ch.inputs(engine, rec, 0 if resident is None else len(resident))
            if "object_rows" in x:
                sc = objects[x["object_rows"][:4]]
            elif "sparse" in x:
                sc = np.asarray(x["sparse"][1:5].astype(np.float64) @ objects.T)
            else:
                sub = x["subjects"] if "subjects" in x else resident[x["subject_ids"]]
                sc = sub[:4].astype(np.float64) @ objects.T
            if rec["role"] == "decoy":
                assert (sc[:, hot].min(axis=1) > sc[:, cold].max(axis=1)).all(), (engine, rec)
            else:
                assert (sc[:, hot].max(axis=1) < sc[:, cold].min(axis=1)).all(), (engine, rec)
