"""GPU: a ranking does not depend on what the engine ranked before.

Engines live across many calls in production (`integration.cached_engine`), their scratch is a set of grow-only device
buffers shared by paths 0-5, and rankers that share a cached engine take its resident subjects from each other.  Each
call must set up every piece of state it reads.  Here long-lived engines -- fp32 DOT, fp32 COSINE, bf16 kept at 16 bits,
a square EASE-shaped engine (paths 2 and 4) and a group [0, 0] -- run the seeded call sequences of
tests/call_history_cases.py, where each checked call follows a larger decoy call that ranks a planted block of hot objects
first.  For every call:
  (a) the padded arrays (ids, score bits, counts) and the plan's statistics equal those of the same call on a fresh engine
      over the same objects;
  (b) the result holds against the rounding-interval oracle (tests/score_interval.check_topk) on sampled rows;
  (c) `last_stats["path"]` (and the wide flag) is the route the record asks for.
Then the first calls of the sequence are replayed on the same engine and must give identical results.  Through
`install()`: u2i and i2i rankers that share one cached engine, called alternately, each frame equal to the same call made
alone on an empty engine cache.

A failing sequence is printed as JSON (`call_history_cases.dumps`): `call_history_cases.loads` replays it."""
import contextlib
import os
import time

import numpy as np
import pytest
from scipy import sparse

from oracle import stage_reference
from tests import call_history_cases as ch
from tests.score_interval import check_topk

pytestmark = pytest.mark.gpu

CHECK_ROWS = 12  # evenly spread rows checked against the oracle per call, next to the filter's edge rows
REPLAY = 8  # records replayed at the end of a sequence
STATS = ("path", "k_out", "k_cand", "n_splits", "n_chunks", "wide", "tc_dtype")


@pytest.fixture(scope="module")
def torch():
    import torch

    return torch


@pytest.fixture(scope="module")
def lib():
    from rectools_b200 import _lib

    return _lib


class Memory:
    """Device memory in use (all processes: `cudaMemGetInfo`), sampled after every call; the peak over the module."""

    def __init__(self, torch):
        self.torch = torch
        free, self.total = torch.cuda.mem_get_info()
        self.start = self.peak = self.total - free

    def sample(self):
        free, _ = self.torch.cuda.mem_get_info()
        self.peak = max(self.peak, self.total - free)


@pytest.fixture(scope="module")
def memory(torch):
    m = Memory(torch)
    t0 = time.time()
    yield m
    print(f"\ncall history: device memory in use {m.start / 2**30:.2f} GiB at the start, peak {m.peak / 2**30:.2f} GiB "
          f"(+{(m.peak - m.start) / 2**30:.2f} GiB), {time.time() - t0:.0f} s")


def _engine(torch, lib, engine, objects):
    """A new engine as the sequence's engine is built; returns (engine, device tensor it reads or None)."""
    from rectools_b200.ranker import Engine, EngineGroup

    spec = ch.ENGINES[engine]
    if spec["dtype"] == "bf16":
        t = torch.from_numpy(objects).to("cuda:0").to(torch.bfloat16).contiguous()
        torch.cuda.synchronize()
        return Engine(None, cosine=spec["cosine"], objects_device_ptr=t.data_ptr(), shape=objects.shape, objects_dtype=lib.DT_BF16,
                      keep_16bit=True), t
    if isinstance(spec["devices"], tuple):
        return EngineGroup(objects, cosine=spec["cosine"], devices=spec["devices"]), None
    return Engine(objects, cosine=spec["cosine"]), None


@contextlib.contextmanager
def _hooks(env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda:0")


def _raw_lists(cand, seed):
    """The device form of candidate lists: each row shuffled, every third row with a -1 hole and a repeated id."""
    rng = np.random.default_rng(seed)
    rows = []
    for r, c in enumerate(cand):
        c = rng.permutation(c)
        if r % 3 == 0 and len(c):
            c = np.r_[c, -1, c[0]]
        rows.append(c.astype(np.int32))
    indptr = np.r_[0, np.cumsum([len(c) for c in rows])].astype(np.int64)
    return indptr, (np.concatenate(rows) if rows else np.empty(0)).astype(np.int32)


def _call(torch, lib, eng, engine, rec, res):
    """Run one record on `eng` (resident subjects `res`); returns ((ids, scores, counts) as numpy, stats, inputs)."""
    x = ch.inputs(engine, rec, 0 if res is None else len(res))
    k, f, wl = x["k"], x["filter"], x["whitelist"]
    fp, fi = (None, None) if f is None else (f.indptr.astype(np.int64), f.indices.astype(np.int32))
    flags = {None: 0, "exact": lib.Q_FORCE_EXACT, "tc": lib.Q_FORCE_TC}[rec["force"]]
    with _hooks(rec["env"]):
        if rec["route"] == "cand_host":
            cand = x["cand"]
            indptr = np.r_[0, np.cumsum([len(c) for c in cand])].astype(np.int64)
            indices = np.concatenate(cand).astype(np.int32)
            got = eng.topk_candidates(k, indptr, indices, subjects=x.get("subjects"), subject_ids=x.get("subject_ids"), indptr=fp,
                                      indices=fi, flags=flags)
        elif rec["route"] == "cand_device":
            indptr, indices = _raw_lists(x["cand"], rec["seed"])
            k_out = min(k, eng.n_objects)
            n = rec["n_rows"]
            out = None if rec["out_dev"] else (np.full((n, k_out), 7, np.int32), np.full((n, k_out), 5, np.float32), np.full(n, -3, np.int32))
            got = eng.topk_candidates_device(k, _dev(torch, indptr), _dev(torch, indices), subjects=_dev(torch, x["subjects"]),
                                             indptr=None if f is None else _dev(torch, fp), indices=None if f is None else _dev(torch, fi),
                                             out=out)
        elif not (rec["in_dev"] or rec["out_dev"]):
            got = eng.topk(k, subjects=x.get("subjects"), subject_ids=x.get("subject_ids"), indptr=fp, indices=fi, whitelist=wl,
                           flags=flags, sparse_subjects=x.get("sparse"), object_rows=x.get("object_rows"))
        else:
            assert "sparse" not in x and "subject_ids" not in x, "device records rank dense subjects or stored rows"
            n = rec["n_rows"]
            k_out = min(k, len(wl) if wl is not None else eng.n_objects)
            if rec["out_dev"]:
                out = (torch.full((n, k_out), 7, dtype=torch.int32, device="cuda:0"), torch.full((n, k_out), 5.0, device="cuda:0"),
                       torch.full((n,), -3, dtype=torch.int32, device="cuda:0"))
            else:
                out = (np.full((n, k_out), 7, np.int32), np.full((n, k_out), 5, np.float32), np.full(n, -3, np.int32))
            src = (lambda a: _dev(torch, a)) if rec["in_dev"] else np.ascontiguousarray
            keep = {}
            kw = {}
            for name, a in (("subjects", x.get("subjects")), ("object_rows", x.get("object_rows")), ("whitelist", wl), ("indptr", fp),
                            ("indices", fi)):
                if a is not None:
                    keep[name] = src(a)
                    kw[name] = keep[name].data_ptr() if rec["in_dev"] else keep[name].ctypes.data
            if wl is not None:
                kw["n_whitelist"] = len(wl)
            fl = flags | (lib.Q_INPUTS_ON_DEVICE if rec["in_dev"] else 0) | (lib.Q_OUTPUTS_ON_DEVICE if rec["out_dev"] else 0)
            torch.cuda.synchronize()
            eng.topk_ptrs(n, k, *(a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data for a in out), fl, **kw)
            torch.cuda.synchronize()
            got = out
            del keep
    got = tuple(a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a) for a in got)
    return got, dict(eng.last_stats), x


def _bits(a):
    return np.where(a == 0, np.float32(0), a).astype(np.float32).view(np.int32)


def _same(got, exp, name):
    """Full padded arrays; scores bit for bit (zeros of either sign equal)."""
    for what, a, b in (("counts", got[2], exp[2]), ("ids", got[0], exp[0]), ("score bits", _bits(got[1]), _bits(exp[1]))):
        assert a.shape == b.shape, f"{name}: {what} shape {a.shape} vs {b.shape}"
        bad = np.argwhere(a != b)
        assert not len(bad), f"{name}: {what} differ at {len(bad)} entries, first {bad[:3].tolist()}: {a[tuple(bad[0])]} vs {b[tuple(bad[0])]}"


def _sample(n, filt):
    rows = set(np.linspace(0, n - 1, min(n, CHECK_ROWS)).astype(np.int64).tolist()) | {r for r in (0, 1, 2) if r < n}
    if filt is not None:  # the rows whose whole positions are viewed
        lens = np.diff(filt.indptr)
        rows |= set(np.argsort(-lens, kind="stable")[:3].tolist())
    return np.array(sorted(rows), np.int64)


def _oracle(engine, objects, rec, got, x, res):
    """check_topk on the sampled rows of one call."""
    spec = ch.ENGINES[engine]
    rows = _sample(rec["n_rows"], x["filter"])
    sub_got = tuple(a[rows] for a in got)
    filt = None if x["filter"] is None else x["filter"][rows]
    name = f"{engine} call {rec['i']} ({rec['route']}, {rec['role']}, {rec['n_rows']} rows, k={rec['k']})"
    if rec["route"] in ("cand_host", "cand_device"):
        n_obj = spec["n_objects"]
        banned = []
        for j, r in enumerate(rows):
            b = np.setdiff1d(np.arange(n_obj), x["cand"][r])
            if filt is not None:
                b = np.union1d(b, filt.indices[filt.indptr[j] : filt.indptr[j + 1]])
            banned.append(b)
        filt = sparse.csr_matrix((np.ones(sum(map(len, banned)), np.float32), np.concatenate(banned), np.r_[0, np.cumsum([len(b) for b in banned])]),
                                 shape=(len(rows), n_obj))
    if rec["route"] == "rows":
        subjects, objs = np.eye(spec["n_objects"], dtype=np.float32)[x["object_rows"][rows]], objects.T
    elif rec["route"] == "sparse":
        subjects, objs = x["sparse"][rows], objects
    else:
        subjects, objs = (x["subjects"] if "subjects" in x else res[x["subject_ids"]])[rows], objects
    check_topk(sub_got, subjects, objs, x["k"], cosine=spec["cosine"], filter_csr=filt, whitelist=x["whitelist"], name=name, verbose=False)


def _run_sequence(torch, lib, memory, engine, seq):
    objects = ch.catalogue(engine)
    eng, keep = _engine(torch, lib, engine, objects)
    res = None
    first = {}
    try:
        for rec in seq:
            if rec["route"] == "set_resident":
                res = ch.resident(engine, rec)
                eng.set_subjects(res)
                continue
            name = f"{engine} call {rec['i']} ({rec['route']}, {rec['role']})"
            got, st, x = _call(torch, lib, eng, engine, rec, res)
            memory.sample()
            assert st["path"] == rec["path"], (name, st)
            if rec["path"] == 1:
                assert st["wide"] == (rec["mode"] in ("wide", "wide_l")), (name, st)
            fresh, fkeep = _engine(torch, lib, engine, objects)
            try:
                if res is not None:
                    fresh.set_subjects(res)
                exp, fst, _ = _call(torch, lib, fresh, engine, rec, res)
                memory.sample()
            finally:
                fresh.close()
                del fkeep
            _same(got, exp, f"{name} against a fresh engine")
            assert {s: st[s] for s in STATS} == {s: fst[s] for s in STATS}, (name, st, fst)
            _oracle(engine, objects, rec, got, x, res)
            if rec["i"] < REPLAY:
                first[rec["i"]] = got
        # replay the first records on the same engine
        for rec in seq[:REPLAY]:
            if rec["route"] == "set_resident":
                res = ch.resident(engine, rec)
                eng.set_subjects(res)
                continue
            got, _, _ = _call(torch, lib, eng, engine, rec, res)
            _same(got, first[rec["i"]], f"{engine} call {rec['i']} replayed at the end")
    finally:
        eng.close()
        del keep


@pytest.mark.parametrize("engine", list(ch.ENGINES))
def test_long_lived_engine_matches_fresh_engines(torch, lib, memory, engine):
    seq = ch.sequence(engine)
    t0 = time.time()
    try:
        _run_sequence(torch, lib, memory, engine, seq)
    except AssertionError:
        print(f"the sequence of the {engine} engine:\n{ch.dumps(seq)}")
        raise
    print(f"{engine}: {len(ch.calls(seq))} calls in {time.time() - t0:.0f} s")


# ------------------------------------------------------------------------------------------------ through install()
@pytest.fixture
def ref():
    if not stage_reference.available():
        pytest.skip("reference package not staged (oracle/_ref)")
    added = stage_reference.add_to_path()
    yield
    import rectools_b200

    rectools_b200.uninstall()
    stage_reference.remove_from_path(added)


def _factors(n, d, seed):
    return (np.random.default_rng(seed).standard_normal((n, d), dtype=np.float32) / np.sqrt(d)).astype(np.float32)


def test_rankers_sharing_a_cached_engine(ref, lib):
    """One item matrix, one cached engine: ALS u2i (DOT) and ALS i2i over the same item factors (DOT here, so that the two
    share the engine and take its resident subject slot from each other), EASE u2i (sparse subjects) and EASE i2i (stored
    rows) on the weight's engine, and two rankers built before either ranks.  Every frame equals the same call made alone
    after `clear_engine_cache()`."""
    from rectools.models import EASEModel
    from rectools.models.rank import Distance

    import rectools_b200
    from rectools_b200 import integration
    from tests.ref_models import injected_als, synthetic_dataset

    n_users, n_items = 4000, 2500
    dataset = synthetic_dataset(n_users, n_items, 20, seed=7)
    items = _factors(n_items, 48, 2)
    als = injected_als(_factors(n_users, 48, 1), items)
    als.i2i_dist = Distance.DOT
    als_b = injected_als(_factors(n_users, 48, 3), items)  # other users, the same items: the same cached engine
    ease = EASEModel(regularization=100.0).fit(dataset)
    users = dataset.user_id_map.external_ids
    targets = dataset.item_id_map.external_ids[::5]
    wl = dataset.item_id_map.external_ids[::3]
    calls = [
        ("als u2i", lambda: als.recommend(users, dataset, k=10, filter_viewed=True)),
        ("als i2i", lambda: als.recommend_to_items(targets, dataset, k=10)),
        ("als_b u2i", lambda: als_b.recommend(users[:700], dataset, k=30, filter_viewed=True, items_to_recommend=wl)),
        ("als u2i small", lambda: als.recommend(users[:50], dataset, k=5, filter_viewed=False)),
        ("ease u2i", lambda: ease.recommend(users[:1500], dataset, k=20, filter_viewed=True)),
        ("als i2i small", lambda: als.recommend_to_items(targets[:30], dataset, k=40, filter_itself=False)),
        ("ease i2i", lambda: ease.recommend_to_items(targets, dataset, k=15)),
        ("als_b u2i small", lambda: als_b.recommend(users[:20], dataset, k=10, filter_viewed=False)),
    ]
    rectools_b200.install(device=0)
    expected = {}
    for name, fn in calls:
        integration.clear_engine_cache()
        expected[name] = fn()
    integration.clear_engine_cache()
    for rnd in range(2):
        for name, fn in calls:
            got = fn()
            assert got.equals(expected[name]), f"round {rnd}: {name}"
    # rankers built before the other one ranks: each construction makes its own subjects resident
    user_f, item_f = als.model.user_factors, als.model.item_factors
    sids = np.arange(0, n_users, 3)
    tids = np.arange(0, n_items, 7)
    integration.clear_engine_cache()
    alone_u = integration.B200ImplicitRanker("dot", user_f, item_f).rank(sids, k=12)
    integration.clear_engine_cache()
    alone_i = integration.B200ImplicitRanker("dot", item_f, item_f).rank(tids, k=12)
    integration.clear_engine_cache()
    r_u = integration.B200ImplicitRanker("dot", user_f, item_f)
    r_i = integration.B200ImplicitRanker("dot", item_f, item_f)
    assert r_u.engine is r_i.engine
    for _ in range(2):
        for got, exp in ((r_u.rank(sids, k=12), alone_u), (r_i.rank(tids, k=12), alone_i)):
            for a, b in zip(got, exp):
                np.testing.assert_array_equal(a, b)
    integration.clear_engine_cache()
