"""Seeded call sequences for long-lived engines (plain numpy, no GPU): every route of `b200_rank_topk`,
`b200_rank_topk_candidates` and `b200_rank_topk_candidates_device` with changing shapes, whitelists, filters, subject
sources and B200_* hooks, so that a kernel reading state an earlier call left in the engine's grow-only scratch shows up.

A sequence is a list of small JSON-serialisable records; `inputs()` rebuilds a record's arrays from its seed, so a failing
sequence printed by `dumps()` replays exactly.  Record fields:
  route     topk | cand_host | cand_device | rows (path 4, stored rows) | sparse (path 2, CSR subjects) |
            set_resident (not a call: replaces the engine's resident subjects by `n_rows` new rows)
  n_rows, k k = None: every position (topk / rows / sparse) or the longest candidate list (cand_*)
  wl        None or [seed, length]: a sorted whitelist of `length` object ids, the hot block always among them
  filter    None | "overlap" (random viewed ids, some outside the positions, row 0 empty) |
            "viewed_all" (as overlap, and up to three rows have every position viewed)
  role      decoy (subjects that rank the hot block first) | checked (subjects that rank it last)
  source    batch (dense subject rows) | resident (subject ids over the resident subjects)
  in_dev, out_dev   inputs / outputs in device memory
  force     None | exact (B200_Q_FORCE_EXACT) | tc (B200_Q_FORCE_TC)
  env       B200_* hooks set for this call only
  path, mode, select   the route the call must take (`b200_rank_stats::path`, the tensor-core mode, the selection)

Every engine's catalogue holds a planted block of hot objects.  Each checked call follows a decoy call of the same route
with more rows, no smaller k and no fewer positions (an equal number, with other ids, for the equal-length whitelist
pairs): a stale candidate list, threshold, exclusion list, gathered object copy or output row of the decoy that leaks into
the checked call returns a hot id, or a score the checked call's subjects do not give."""
from __future__ import annotations

import json
import typing as tp

import numpy as np
from scipy import sparse

S = 12288  # LK_SMEM_PAIRS (rectools_b200/csrc/sizes.h): the radix selection's shared-memory survivors
SM_COUNT = 132  # H100 SXM
HOT = 64  # hot objects per catalogue
HOT_VALUE = 4.0

# name: objects [n_objects, d], distance, storage, devices (an int: one engine; a tuple: an engine group)
ENGINES: tp.Dict[str, tp.Dict[str, tp.Any]] = {
    "dot": dict(n_objects=50_000, d=128, cosine=False, dtype="f32", devices=0),
    "cosine": dict(n_objects=30_000, d=65, cosine=True, dtype="f32", devices=0),
    "bf16": dict(n_objects=20_000, d=24, cosine=False, dtype="bf16", devices=0),
    "square": dict(n_objects=3_000, d=3_000, cosine=False, dtype="f32", devices=0),
    "group": dict(n_objects=40_000, d=64, cosine=False, dtype="f32", devices=(0, 0)),
}

FLAG_IN_DEV, FLAG_OUT_DEV, FLAG_FORCE_EXACT, FLAG_FORCE_TC = 1, 2, 4, 8  # B200_Q_*
TC_FP16, TC_BF16 = 1, 2
PATH_MODES = ("narrow", "wide", "wide_l", "multi_pass")  # = plan.h TcMode
SELECTS = ("passes", "radix")  # = plan.h Select


def hot_ids(engine: str) -> np.ndarray:
    n = ENGINES[engine]["n_objects"]
    return np.arange(n // 3, n // 3 + HOT, dtype=np.int64)


def square_decoy_rows(n: int) -> np.ndarray:
    """Rows of the square engine whose hot columns are large and positive (decoy score rows), and the columns whose hot
    rows are (decoy sparse subjects); negative elsewhere."""
    return np.arange(0, n, 4, dtype=np.int64)


def square_pool(n: int, decoy: bool) -> np.ndarray:
    """Stored rows / sparse subject columns a decoy (checked) call of the square engine draws from: outside the hot block."""
    rows = square_decoy_rows(n) if decoy else np.setdiff1d(np.arange(n), square_decoy_rows(n))
    return np.setdiff1d(rows, hot_ids("square"))


def _bf16_round(x: np.ndarray) -> np.ndarray:
    u = np.ascontiguousarray(x, np.float32).view(np.uint32)
    u = (u + np.uint32(0x7FFF) + ((u >> np.uint32(16)) & np.uint32(1))) & np.uint32(0xFFFF0000)
    return u.view(np.float32)


def catalogue(engine: str) -> np.ndarray:
    """The engine's objects (fp32; values exact in bf16 for the bf16 engine).  Dense engines: hot objects have a large
    first column.  The square engine (an EASE weight): hot columns are +HOT_VALUE in the decoy rows, -HOT_VALUE elsewhere."""
    spec = ENGINES[engine]
    n, d = spec["n_objects"], spec["d"]
    rng = np.random.default_rng(1000 + sum(map(ord, engine)))
    obj = (rng.standard_normal((n, d), dtype=np.float32) / np.float32(np.sqrt(d))).astype(np.float32)
    hot = hot_ids(engine)
    if engine == "square":  # hot columns (stored score rows, path 4) and hot rows (sparse subjects, path 2)
        dec = square_decoy_rows(n)
        obj[:, hot] = -HOT_VALUE
        obj[np.ix_(dec, hot)] = HOT_VALUE
        obj[hot, :] = -HOT_VALUE
        obj[np.ix_(hot, dec)] = HOT_VALUE
    else:
        obj[hot, 0] = HOT_VALUE
    if spec["dtype"] == "bf16":
        obj = _bf16_round(obj)
    return obj


# ------------------------------------------------------------------------------------------------ record arrays
def whitelist(engine: str, wl: tp.Optional[tp.Sequence[int]]) -> tp.Optional[np.ndarray]:
    if wl is None:
        return None
    seed, length = wl
    n, hot = ENGINES[engine]["n_objects"], hot_ids(engine)
    rng = np.random.default_rng(seed)
    rest = np.setdiff1d(np.arange(n), hot)
    return np.union1d(hot, rng.choice(rest, length - len(hot), replace=False)).astype(np.int32)


def _subject_rows(rng: np.random.Generator, n: int, d: int, decoy: bool) -> np.ndarray:
    x = (rng.standard_normal((n, d), dtype=np.float32) / np.float32(np.sqrt(d))).astype(np.float32)
    x[:, 0] = (np.abs(x[:, 0]) + 1.0) * (1.0 if decoy else -1.0)
    return x


def resident(engine: str, rec: tp.Dict[str, tp.Any]) -> np.ndarray:
    """The subjects of a set_resident record: the first half of the rows rank the hot block first (decoy ids are drawn
    there), the second half last."""
    rng = np.random.default_rng(rec["seed"])
    n, d = rec["n_rows"], ENGINES[engine]["d"]
    return np.concatenate([_subject_rows(rng, n // 2, d, True), _subject_rows(rng, n - n // 2, d, False)])


def _filter(rng: np.random.Generator, kind: tp.Optional[str], n_rows: int, positions: np.ndarray, n_obj: int) -> tp.Optional[sparse.csr_matrix]:
    if kind is None:
        return None
    rows = []
    for r in range(n_rows):
        if r == 0:
            rows.append(np.empty(0, np.int64))
            continue
        m = int(rng.integers(1, 60))
        rows.append(np.unique(np.r_[rng.choice(positions, min(m, len(positions)), replace=False), rng.integers(0, n_obj, 3)]))
    if kind == "viewed_all":
        for r in range(1, n_rows, 7)[:3]:
            rows[r] = np.asarray(positions, np.int64)
    indptr = np.zeros(n_rows + 1, np.int64)
    np.cumsum([len(x) for x in rows], out=indptr[1:])
    idx = np.concatenate(rows).astype(np.int32) if rows else np.empty(0, np.int32)
    return sparse.csr_matrix((np.ones(len(idx), np.float32), idx, indptr), shape=(n_rows, n_obj))


def _cand_lists(rng: np.random.Generator, rec: tp.Dict[str, tp.Any], n_obj: int, hot: np.ndarray) -> tp.List[np.ndarray]:
    """Ascending unique ids per row: lengths from 0 to `cand_len` (row 0 the longest, row 1 empty), the hot block in
    every other row."""
    n, m = rec["n_rows"], rec["cand_len"]
    lens = rng.integers(0, m + 1, n)
    lens[0] = m
    if n > 2:
        lens[1] = 0
    rest = np.setdiff1d(np.arange(n_obj), hot)
    out = []
    for r in range(n):
        ids = rng.choice(rest, int(lens[r]), replace=False)
        if r % 2 == 0:
            h = min(len(hot), len(ids))
            ids[:h] = hot[:h]
        out.append(np.sort(ids).astype(np.int32))
    return out


def inputs(engine: str, rec: tp.Dict[str, tp.Any], resident_rows: int = 0) -> tp.Dict[str, tp.Any]:
    """The arrays of one call record: `subjects` (dense [n_rows, d]) or `subject_ids` (over the `resident_rows` resident
    subjects) or `sparse` (CSR [n_rows, d]) or `object_rows`; `whitelist`; `filter` (CSR of object ids); `cand` (list of
    ascending id arrays, cand_* routes) and `k` (the int k handed to the engine)."""
    spec = ENGINES[engine]
    n_obj, d, n = spec["n_objects"], spec["d"], rec["n_rows"]
    rng = np.random.default_rng(rec["seed"])
    decoy = rec["role"] == "decoy"
    out: tp.Dict[str, tp.Any] = {"whitelist": whitelist(engine, rec["wl"])}
    positions = np.arange(n_obj) if out["whitelist"] is None else out["whitelist"]
    if rec["route"] == "rows":
        pool = square_pool(n_obj, decoy)
        out["object_rows"] = rng.choice(pool, n, replace=n > len(pool)).astype(np.int64)
    elif rec["route"] == "sparse":
        pool = square_pool(n_obj, decoy)
        nnz = rng.integers(1, 24, n)
        nnz[0] = 0  # an empty subject row
        indptr = np.r_[0, np.cumsum(nnz)].astype(np.int64)
        indices = np.concatenate([np.sort(rng.choice(pool, c, replace=False)) for c in nnz]).astype(np.int32)
        data = rng.uniform(0.5, 2.0, int(indptr[-1])).astype(np.float32)
        out["sparse"] = sparse.csr_matrix((data, indices, indptr), shape=(n, d))
    elif rec["source"] == "resident":
        half = resident_rows // 2
        out["subject_ids"] = (rng.integers(0, half, n) if decoy else rng.integers(half, resident_rows, n)).astype(np.int64)
    else:
        out["subjects"] = _subject_rows(rng, n, d, decoy)
    if rec["route"] in ("cand_host", "cand_device"):
        out["cand"] = _cand_lists(rng, rec, n_obj, hot_ids(engine))
        longest = max((len(c) for c in out["cand"]), default=0)
        out["k"] = longest if rec["k"] is None else rec["k"]
        out["filter"] = None
        if rec["filter"] is not None:  # viewed_all: every candidate of up to three rows viewed
            allc = np.unique(np.concatenate(out["cand"]))
            f = _filter(rng, "overlap", n, allc if len(allc) else np.arange(n_obj), n_obj)
            if rec["filter"] == "viewed_all":
                f = f.tolil()
                for r in range(2, n, 7)[:3]:
                    f.rows[r] = sorted(set(f.rows[r]) | set(out["cand"][r].tolist()))
                    f.data[r] = [1.0] * len(f.rows[r])
                f = f.tocsr()
            out["filter"] = f
    else:
        out["k"] = len(positions) if rec["k"] is None else rec["k"]
        out["filter"] = _filter(rng, rec["filter"], n, positions, n_obj)
    return out


# ------------------------------------------------------------------------------------------------ shapes and plans
def n_pos(engine: str, rec: tp.Dict[str, tp.Any]) -> int:
    """Positions of a call: the whitelist, else the catalogue; candidate calls: the longest allowed list."""
    if rec["route"] in ("cand_host", "cand_device"):
        return rec["cand_len"]
    return rec["wl"][1] if rec["wl"] is not None else ENGINES[engine]["n_objects"]


def k_out(engine: str, rec: tp.Dict[str, tp.Any]) -> int:
    if rec["route"] in ("cand_host", "cand_device"):
        return min(rec["k"] if rec["k"] is not None else rec["cand_len"], ENGINES[engine]["n_objects"])
    p = n_pos(engine, rec)
    return p if rec["k"] is None else min(rec["k"], p)


def extent(engine: str, rec: tp.Dict[str, tp.Any]) -> tp.Tuple[int, int, int]:
    return rec["n_rows"], k_out(engine, rec), n_pos(engine, rec)


def larger(engine: str, prev: tp.Dict[str, tp.Any], cur: tp.Dict[str, tp.Any]) -> bool:
    """`prev` ranks more rows than `cur`, with no smaller k_out and no fewer positions."""
    (pr, pk, pp), (cr, ck, cp) = extent(engine, prev), extent(engine, cur)
    return pr > cr and pk >= ck and pp >= cp


def call_shape(engine: str, rec: tp.Dict[str, tp.Any]) -> tp.Dict[str, int]:
    """The CallShape words of tests/plan_driver.cpp for a topk / rows / sparse record, with its hooks."""
    spec = ENGINES[engine]
    flags = {None: 0, "exact": FLAG_FORCE_EXACT, "tc": FLAG_FORCE_TC}[rec["force"]]
    flags |= (FLAG_IN_DEV if rec["in_dev"] else 0) | (FLAG_OUT_DEV if rec["out_dev"] else 0)
    shape = {"n_rows": rec["n_rows"], "n_pos": n_pos(engine, rec), "k": k_out(engine, rec), "d": spec["d"], "sm_count": SM_COUNT,
             "tc_dtype": TC_BF16 if spec["dtype"] == "bf16" else TC_FP16, "flags": flags, "sparse": int(rec["route"] == "sparse"),
             "rows": int(rec["route"] == "rows"), "n_objects": spec["n_objects"], "cosine": int(spec["cosine"])}
    shape.update({k: int(v) for k, v in rec["env"].items()})
    return shape


def calls(seq: tp.Sequence[tp.Dict[str, tp.Any]]) -> tp.List[tp.Dict[str, tp.Any]]:
    return [r for r in seq if r["route"] != "set_resident"]


def dumps(seq: tp.Sequence[tp.Dict[str, tp.Any]]) -> str:
    """A sequence as JSON, one record per line: what a failing test prints, and what `loads` replays."""
    return "[\n" + ",\n".join(json.dumps(r, sort_keys=True) for r in seq) + "\n]"


def loads(text: str) -> tp.List[tp.Dict[str, tp.Any]]:
    return json.loads(text)


# ------------------------------------------------------------------------------------------------ the sequences
def _rec(route: str, n_rows: int, k: tp.Optional[int], path: int, mode: tp.Optional[str] = None, select: tp.Optional[str] = None,
         wl: tp.Optional[tp.Sequence[int]] = None, filt: tp.Optional[str] = None, source: str = "batch", in_dev: bool = False,
         out_dev: bool = False, force: tp.Optional[str] = None, env: tp.Optional[tp.Dict[str, str]] = None, cand_len: int = 0,
         decoy: tp.Optional[tp.Dict[str, tp.Any]] = None) -> tp.Dict[str, tp.Any]:
    """A checked call; `decoy` overrides fields of the decoy call that precedes it (default: twice the rows plus 37, the
    largest k of the same mode, a longer whitelist, longer candidate lists, the default split / carousel / chunk hooks)."""
    r = dict(route=route, n_rows=n_rows, k=k, wl=None if wl is None else list(wl), filter=filt, role="checked", source=source,
             in_dev=in_dev, out_dev=out_dev, force=force, env=dict(env or {}), path=path, mode=mode, select=select, cand_len=cand_len)
    r["decoy"] = dict(decoy or {})
    return r


# the largest k of each tensor-core mode / selection: a decoy's k stays in its checked call's mode
_MODE_K = {"narrow": 24, "wide": 128, "wide_l": 1024}


def _decoy_for(engine: str, c: tp.Dict[str, tp.Any], rng: np.random.Generator) -> tp.Dict[str, tp.Any]:
    n_obj = ENGINES[engine]["n_objects"]
    d = dict(c)
    # the route's hooks stay; the split, carousel and chunk hooks are the defaults in a decoy, so that they change
    env = {h: v for h, v in c["env"].items() if h not in ("B200_TC_SPLITS", "B200_TC_CAROUSEL", "B200_CHUNK_ROWS")}
    d.update(role="decoy", n_rows=2 * c["n_rows"] + 37, filter="overlap", env=env)
    if c["k"] is not None and c["mode"] in _MODE_K:
        d["k"] = _MODE_K[c["mode"]]
    if c["wl"] is not None:
        d["wl"] = [int(rng.integers(1 << 30)), min(n_obj, c["wl"][1] + 3000)]
    if c["cand_len"]:
        d["cand_len"] = min(n_obj, c["cand_len"] + 500)
    over = c.pop("decoy")
    d.pop("decoy", None)
    d.update(over)
    return d


def _dense_calls(engine: str, full: bool) -> tp.List[tp.Dict[str, tp.Any]]:
    """The topk and candidate-set calls of a dense engine; `full`: every k edge and hook (the fp32 DOT engine)."""
    n = ENGINES[engine]["n_objects"]
    L = n // 2  # whitelist length of the equal-length pairs
    out = [
        _rec("topk", 1, 1, 0, force="exact", filt="overlap"),
        _rec("topk", 700, 128, 0, force="exact", wl=[11, n // 3]),
        _rec("topk", 300, 24, 1, "narrow", force="tc", wl=[12, L], env={"B200_TC_SPLITS": "3"}, decoy={"wl": [13, L]}),
        _rec("topk", 1, 1, 1, "narrow", force="tc", env={"B200_TC_CAROUSEL": "0"}),
        _rec("topk", 2000, 25, 1, "wide", filt="viewed_all", wl=[14, 5000], decoy={"wl": [15, 5000]}),
        _rec("topk", 900, 129, 1, "wide_l", force="tc"),
        _rec("topk", 300, 1024, 1, "wide_l", force="tc", in_dev=True, out_dev=True, wl=[16, L], decoy={"wl": [17, L]}),
        _rec("topk", 400, 100, 1, "multi_pass", force="tc", env={"B200_WIDE": "0"}, filt="overlap"),
        _rec("topk", 100, 1025, 3, select="radix", filt="overlap"),
        _rec("topk", 8, None, 3, select="radix", wl=[18, 4000]),
        _rec("cand_host", 1000, 10, 5, filt="overlap", cand_len=300, env={"B200_CHUNK_ROWS": "256"}),
        _rec("cand_device", 300, 1025, 5, cand_len=3000, in_dev=True, out_dev=True, filt="viewed_all"),
        _rec("cand_device", 1, 24, 5, cand_len=40, in_dev=True),
    ]
    if full:
        out += [
            _rec("topk", 700, 128, 1, "wide", force="tc", filt="overlap", env={"B200_CHUNK_ROWS": "256"}),
            _rec("topk", 600, 129, 3, select="passes", force="exact", env={"B200_SELECT": "0"}, filt="overlap"),
            _rec("topk", 100, 129, 3, select="radix", force="exact", env={"B200_SELECT": "2"}, wl=[19, 20_000]),
            _rec("topk", 20, S + 1, 3, select="radix", filt="viewed_all", in_dev=True),
            _rec("topk", 3, 1024, 3, select="passes", force="exact", env={"B200_SELECT": "0"}),
            _rec("cand_host", 5, S + 1, 5, cand_len=20_000, filt="overlap"),
            _rec("cand_host", 50, None, 5, cand_len=2000),
            _rec("cand_device", 40, S + 1, 5, cand_len=15_000, in_dev=True),
        ]
    return out


def _resident_calls(engine: str) -> tp.List[tp.Dict[str, tp.Any]]:
    """Resident subjects replaced between calls with another row count, each followed by calls that rank them."""
    out: tp.List[tp.Dict[str, tp.Any]] = []
    for seed, n_res, k, mode, route in ((41, 3000, 24, "narrow", "topk"), (42, 1200, 25, "wide", "topk"), (43, 5000, 10, None, "cand_host")):
        out.append(dict(route="set_resident", n_rows=n_res, seed=seed))
        path = 5 if route == "cand_host" else 1
        extra = {"cand_len": 200} if route == "cand_host" else {}
        out.append(_rec(route, 500, k, path, mode, force=None if route == "cand_host" else "tc", source="resident", filt="overlap", **extra))
    return out


def _square_calls() -> tp.List[tp.Dict[str, tp.Any]]:
    n = ENGINES["square"]["n_objects"]
    return [
        _rec("rows", 1, 1, 4, select="radix", filt="overlap"),
        _rec("rows", 700, 128, 4, select="radix", wl=[21, 1500], env={"B200_CHUNK_ROWS": "256"}, decoy={"wl": [22, 1500], "env": {"B200_CHUNK_ROWS": "300"}}),
        _rec("rows", 300, 1025, 4, select="radix", filt="viewed_all"),
        _rec("rows", 40, None, 4, select="radix", in_dev=True, out_dev=True),
        _rec("sparse", 1, 24, 2, select="passes"),
        _rec("sparse", 500, 129, 2, select="passes", filt="overlap", wl=[23, n // 2]),
        _rec("sparse", 300, 129, 2, select="radix", env={"B200_SELECT": "2"}, filt="viewed_all"),
        _rec("sparse", 200, 1025, 2, select="radix", filt="overlap"),
        _rec("sparse", 30, None, 2, select="radix", wl=[24, 2000]),
    ]


def _group_calls() -> tp.List[tp.Dict[str, tp.Any]]:
    """An engine group refuses B200_Q_FORCE_TC (a member's row slice may be a tiny problem): its tensor-core calls are
    large enough for every member's slice to take the tensor cores."""
    n = ENGINES["group"]["n_objects"]
    return [
        _rec("topk", 1, 1, 0, force="exact"),
        _rec("topk", 600, 24, 1, "narrow", filt="overlap", wl=[31, n // 2], decoy={"wl": [32, n // 2]}),
        _rec("topk", 800, 128, 1, "wide", env={"B200_TC_SPLITS": "2"}),
        _rec("topk", 500, 1024, 1, "wide_l", filt="viewed_all", in_dev=True, out_dev=True),
        _rec("topk", 300, 50, 1, "multi_pass", env={"B200_WIDE": "0"}),
        _rec("topk", 100, 1025, 3, select="radix", filt="overlap"),
    ]


def sequence(engine: str, seed: int = 0) -> tp.List[tp.Dict[str, tp.Any]]:
    """The call sequence of one engine: its checked calls in a seeded order, each after its decoy, with the resident-subject
    replacements of the single dense engines; every record has its own data seed and index."""
    rng = np.random.default_rng([seed, sum(map(ord, engine))])
    if engine == "square":
        checked = _square_calls()
    elif engine == "group":
        checked = _group_calls()
    else:
        checked = _dense_calls(engine, full=engine == "dot")
    checked = [checked[i] for i in rng.permutation(len(checked))]
    blocks = [[_decoy_for(engine, c, rng), c] for c in checked]
    if engine in ("dot", "cosine", "bf16"):
        res = _resident_calls(engine)
        for i in range(0, len(res), 2):
            setr, c = res[i], res[i + 1]
            blocks.insert(int(rng.integers(0, len(blocks) + 1)), [setr, _decoy_for(engine, c, rng), c])
    seq = [r for b in blocks for r in b]
    for i, r in enumerate(seq):
        r["i"] = i
        r["seed"] = int(rng.integers(1 << 31))
    return seq
