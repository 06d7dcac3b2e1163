"""GPU: the tensor-core candidate pass itself, not only the final top-k.

Every case ranks on the tensor-core path with B200_TC_SNAPSHOT set, checks the captured pass with tests/tc_reference.py
on every row and list (list contents I1, premise P1 = I2, premise P2 = I3, thresholds I4, the certificate's verdict I5,
and the exponents / constants the kernel used), and holds the final ids and scores to the rounding-interval checker of tests/score_interval.py on every row.
Each case prints its largest observed fractions of the I2 bounds and its fallback counts."""
import numpy as np
import pytest
from scipy import sparse

from tests.helpers import synth_factors, synth_viewed_csr
from tests.score_interval import check_topk
from tests.tc_reference import TILE_N, Catalogue, check_snapshot

pytestmark = pytest.mark.gpu

N_ROWS, N_OBJ, D, K = 768, 16_000, 64, 10


@pytest.fixture(scope="module")
def lib():
    from rectools_b200 import _lib

    return _lib


def _csr(cols_per_row, n_cols):
    indptr = np.zeros(len(cols_per_row) + 1, np.int64)
    indptr[1:] = np.cumsum([len(c) for c in cols_per_row])
    indices = np.concatenate([np.sort(np.asarray(c, np.int64)) for c in cols_per_row]).astype(np.int32) if len(cols_per_row) else np.empty(0, np.int32)
    return indptr, indices


def _run(eng, lib, monkeypatch, capsys, name, sub32, k, objects, cosine, indptr=None, indices=None, whitelist=None, id_off=0,
         snaps=(1,), bf16=False, flags=None, min_launches=1):
    """Rank, check every row with the score-interval checker, check the snapshot of each requested launch.  Returns the reports and stats."""
    sub32 = np.ascontiguousarray(sub32, np.float32)
    n_rows = len(sub32)
    cat = Catalogue(objects, cosine=cosine, bf16=bf16, whitelist=whitelist, id_off=id_off)
    if indptr is not None:
        viewed = cat.viewed_positions(indptr, indices, n_rows)
    else:
        viewed = sparse.csr_matrix((n_rows, cat.n_pos), dtype=np.float32)
    reports = []
    for n in snaps:
        monkeypatch.setenv("B200_TC_SNAPSHOT", str(n))
        ids, sc, cnt = eng.topk(k, subjects=sub32, indptr=indptr, indices=indices, whitelist=whitelist,
                                flags=lib.Q_FORCE_TC if flags is None else flags)
        st = dict(eng.last_stats)
        assert st["path"] == 1 and st["n_tc_launches"] >= min_launches, st
        check_topk((ids, sc, cnt), sub32, objects, k, cosine=cosine, filter_csr=None if indptr is None else (indptr, indices),
                   whitelist=whitelist, id_offset=id_off, name=f"{name} {st}")
        snap = eng.candidate_snapshot()
        if n > st["n_tc_launches"]:
            assert snap is None
            continue
        assert snap is not None and snap["launch"] == n, st
        rows = snap["rows"].astype(np.int64)
        excluded = prev = None
        k0 = snap["k0"]
        if k0 > 0:  # objects returned by earlier passes are excluded: the first k0 final entries of each row
            g = ids[rows, :k0].astype(np.int64) - id_off
            ok = (g >= 0) & (g < cat.n_obj)
            pos = np.where(ok, cat.pos_of_obj[np.clip(g, 0, cat.n_obj - 1)], -1)
            rr = np.repeat(np.arange(len(rows)), k0).reshape(pos.shape)
            m = pos >= 0
            excluded = sparse.csr_matrix((np.ones(int(m.sum()), np.float32), (rr[m], pos[m])), shape=(len(rows), cat.n_pos))
            prev = (sc[rows, k0 - 1], ids[rows, k0 - 1].astype(np.int64) - id_off, cnt[rows] >= k0)
        rep = check_snapshot(snap, cat, sub32[rows], viewed[rows], excluded, prev)
        with capsys.disabled():
            print(f"\n[{name} launch {n}/{st['n_tc_launches']}] nw={snap['nw']} splits={snap['n_splits']} k0={k0} kp={snap['kp']} "
                  f"K'={snap['k_cand']} wide={snap['wide']} {rep.summary()} | fallback_rows={st['n_fallback_rows']} "
                  f"exact_rows={st['n_exact_rows']}")
        assert rep.ok, f"{name} launch {n}: {rep.summary()}"
        reports.append((snap, rep, st))
    return cat, reports


def _base(n_rows=N_ROWS, n_obj=N_OBJ, d=D, seed=0, per_user=50):
    u, i = synth_factors(n_rows, n_obj, d, seed=seed)
    csr = synth_viewed_csr(n_rows, n_obj, per_user, seed=seed + 2) if per_user else None
    return u, i, csr


# ------------------------------------------------------------------------------------------------ geometry
@pytest.mark.parametrize(
    "name, env, shape",
    [
        ("nw8", {}, {}),
        ("kcand32", {"B200_TC_KCAND": "32"}, {}),  # lists at their full 32 slots
        ("splits1", {"B200_TC_SPLITS": "1"}, {}),
        ("splits3", {"B200_TC_SPLITS": "3"}, {}),
        ("splits_max", {"B200_TC_SPLITS": "16"}, {"n_obj": 80_000, "d": 32, "n_rows": 512}),
        ("rows1", {}, {"n_rows": 1}),
        ("rows255", {}, {"n_rows": 255}),
        ("rows256", {}, {"n_rows": 256}),
        ("rows257", {}, {"n_rows": 257}),
        ("npos_4kcand", {}, {"n_obj": 48, "n_rows": 300, "per_user": 5}),
        ("npos_256m_plus_1", {}, {"n_obj": 256 * 20 + 1}),
        ("npos_not_64", {}, {"n_obj": 5_037}),
        ("rows257_splits3", {"B200_TC_SPLITS": "3"}, {"n_rows": 257}),  # six lists per row on a partial row tile
    ],
)
def test_geometry(lib, monkeypatch, capsys, name, env, shape):
    from rectools_b200 import Engine

    for k_, v_ in env.items():
        monkeypatch.setenv(k_, v_)
    u, i, csr = _base(**shape)
    eng = Engine(i, cosine=False)
    _, reps = _run(eng, lib, monkeypatch, capsys, name, u, K, i, False, csr.indptr, csr.indices)
    snap = reps[0][0]
    assert snap["nw"] == 8
    if "B200_TC_SPLITS" in env:
        assert snap["n_splits"] == int(env["B200_TC_SPLITS"])
    if name == "kcand32":
        assert snap["k_cand"] == 32
    if name == "npos_4kcand":
        assert snap["n_pos"] == 4 * snap["k_cand"]
    eng.close()


@pytest.mark.parametrize("carousel", ["0", "1"])
def test_more_row_tiles_than_pairs_viewed_packed_at_the_wrap(lib, monkeypatch, capsys, carousel):
    """More work items than CTA pairs (later items start mid-stream under the carousel and wrap around to the split's first
    tile, where the CSR cursors are repositioned); each row's viewed ids are packed into the first two tiles of every split,
    the last tile of every split and the last tile of the stream."""
    from rectools_b200 import Engine

    monkeypatch.setenv("B200_TC_CAROUSEL", carousel)
    monkeypatch.setenv("B200_TC_SPLITS", "2")
    n_rows, n_obj, d = 17_500, 12_000, 24
    u, i, _ = _base(n_rows, n_obj, d, seed=4, per_user=0)
    n_tiles = (n_obj + TILE_N - 1) // TILE_N
    tps = (n_tiles + 1) // 2
    hot = []
    for s in range(2):
        t0, t1 = s * tps, min((s + 1) * tps, n_tiles)
        for t in (t0, t0 + 1, t1 - 1):
            hot.append(np.arange(t * TILE_N, min((t + 1) * TILE_N, n_obj)))
    hot = np.unique(np.concatenate(hot))
    rng = np.random.default_rng(1)
    cols = [np.union1d(hot[rng.random(len(hot)) < 0.5], rng.choice(n_obj, 10)) for _ in range(n_rows)]
    indptr, indices = _csr(cols, n_obj)
    eng = Engine(i, cosine=False)
    _, reps = _run(eng, lib, monkeypatch, capsys, f"carousel{carousel}", u, K, i, False, indptr, indices)
    assert reps[0][0]["rows_pad"] // 256 > 66 and reps[0][0]["n_splits"] == 2  # more row tiles than the 66 CTA pairs of an H100 SXM
    eng.close()


# ------------------------------------------------------------------------------------------------ d
@pytest.mark.parametrize("d", [24, 128, 150, 256, 301, 320])
def test_every_k_block_count(lib, monkeypatch, capsys, d):
    """1 to 5 k blocks of 64; d = 320 is the largest tensor-core d (5 blocks with a 3-stage object ring); 150 and 301 are
    not multiples of 4 (the re-score's scalar loop)."""
    from rectools_b200 import Engine

    n_obj = max(4_000, int(1.0e9 / (N_ROWS * d)))
    u, i, csr = _base(N_ROWS, n_obj, d, seed=d)
    eng = Engine(i, cosine=d == 150)
    assert eng.info()["d_pad"] == (d + 63) // 64 * 64
    _run(eng, lib, monkeypatch, capsys, f"d{d}", u, K, i, d == 150, csr.indptr, csr.indices)
    eng.close()


@pytest.mark.parametrize("d", [321, 384])
def test_d_beyond_the_tensor_core_path(lib, d):
    """d_pad = 384 leaves no room for an object ring: FORCE_TC is refused, the default path is the exhaustive kernel."""
    from rectools_b200 import Engine

    u, i, csr = _base(200, 3_000, d, seed=d)
    eng = Engine(i, cosine=False)
    with pytest.raises(NotImplementedError):
        eng.topk(K, subjects=u, indptr=csr.indptr, indices=csr.indices, flags=lib.Q_FORCE_TC)
    ids, sc, cnt = eng.topk(K, subjects=u, indptr=csr.indptr, indices=csr.indices)
    assert eng.last_stats["path"] == 0
    check_topk((ids, sc, cnt), u, i, K, filter_csr=csr, name=f"d={d} exhaustive")
    eng.close()


# ------------------------------------------------------------------------------------------------ precision, dynamic range
def _range_case(kind):
    rng = np.random.default_rng(sum(map(ord, kind)))
    u, i, csr = _base(N_ROWS, N_OBJ, D, seed=7)
    cosine = False
    if kind == "subjects_1e-30_to_1e30":
        u = (u * 10.0 ** rng.uniform(-30, 30, size=(len(u), 1))).astype(np.float32)
    elif kind == "one_nonzero":
        j = rng.integers(0, D, len(u))
        v = np.where(rng.random(len(u)) < 0.5, 2.0 ** rng.integers(-60, 60, len(u)), rng.standard_normal(len(u)) * 10.0 ** rng.uniform(-20, 20, len(u)))
        v = np.where(rng.random(len(u)) < 0.3, -v, v)  # negative powers of two too
        u = np.zeros_like(u)
        u[np.arange(len(u)), j] = v
    elif kind == "subnormal_subjects":
        u[::3] *= np.float32(1e-39)  # every element an fp32 subnormal
        u[1::3, ::2] *= np.float32(1e-40)  # normal rows with subnormal elements
    elif kind == "heavy_objects_1e4":
        i[rng.choice(len(i), 5, replace=False)] *= np.float32(1e4)
    elif kind == "heavy_objects_1e9":  # the rest of the catalogue sits at or below the fp16 subnormal range
        i[rng.choice(len(i), 5, replace=False)] *= np.float32(1e9)
    elif kind == "cosine_zero_objects":
        cosine = True
        i[rng.choice(len(i), 300, replace=False)] = 0.0
        i[:40] *= np.float32(1e6)
    return u.astype(np.float32), i.astype(np.float32), csr, cosine


@pytest.mark.parametrize(
    "kind", ["subjects_1e-30_to_1e30", "one_nonzero", "subnormal_subjects", "heavy_objects_1e4", "heavy_objects_1e9", "cosine_zero_objects"]
)
@pytest.mark.parametrize("tc_mode", ["auto", "bf16"])
def test_dynamic_range(lib, monkeypatch, capsys, kind, tc_mode):
    """Row and object exponents against the emulation (exactly), P1 on rows far from unit scale.  AUTO keeps fp16 for
    fp32 factors whatever their range: one global object exponent, small objects rounded to fp16 subnormals or zero."""
    from rectools_b200 import Engine

    u, i, csr, cosine = _range_case(kind)
    eng = Engine(i, cosine=cosine, tc_mode=tc_mode)
    assert eng.info()["tc_dtype"] == (lib.TC_BF16 if tc_mode == "bf16" else lib.TC_FP16)
    _run(eng, lib, monkeypatch, capsys, f"{kind}/{tc_mode}", u, K, i, cosine, csr.indptr, csr.indices, bf16=tc_mode == "bf16")
    eng.close()


def test_bf16_factors_choose_bf16(lib, monkeypatch, capsys):
    """AUTO with bf16 object factors (device tensors): the bf16 copy is exact, exponents are 0."""
    import torch

    from rectools_b200 import Engine

    u, i, csr = _base(512, 12_000, 64, seed=12)
    t = torch.from_numpy(i).to("cuda:0").to(torch.bfloat16).contiguous()
    i16 = t.float().cpu().numpy()
    torch.cuda.synchronize()
    eng = Engine(None, cosine=False, objects_device_ptr=t.data_ptr(), shape=tuple(t.shape), objects_dtype=lib.DT_BF16)
    assert eng.info()["tc_dtype"] == lib.TC_BF16
    _, reps = _run(eng, lib, monkeypatch, capsys, "bf16_factors", u, K, i16, False, csr.indptr, csr.indices, bf16=True)
    assert reps[0][0]["bf16"] == 1
    eng.close()
    del t


def test_bf16_pass_scales_subnormal_subjects(lib, monkeypatch, capsys):
    """Regression: the bf16 pass used to round subject rows unscaled (row exponent 0).  Rows of fp32 subnormals became a
    few bf16-subnormal steps, their approximate scores were off by far more than eps (relative to the row's own norm),
    and such rows were certified with wrong ids.  Both operand types are now power-of-two scaled."""
    from rectools_b200 import Engine

    u, i, csr = _base(512, 12_000, 64, seed=13)
    u[::2] *= np.float32(1e-39)
    eng = Engine(i, cosine=False, tc_mode="bf16")
    _, reps = _run(eng, lib, monkeypatch, capsys, "bf16_subnormal_rows", u, K, i, False, csr.indptr, csr.indices, bf16=True)
    assert (reps[0][0]["row_exp"][::2] > 100).all()
    eng.close()


# ------------------------------------------------------------------------------------------------ filter
def _true_top(u, i, m):
    s = u.astype(np.float64) @ i.astype(np.float64).T
    return np.argsort(-s, axis=1)[:, :m]


@pytest.mark.parametrize("kind", ["true_top200", "half_catalogue", "duplicates", "beyond_catalogue", "whitelist_outside", "id_offset"])
def test_filter(lib, monkeypatch, capsys, kind):
    """Viewed objects must never enter a list (I1) and never be counted as discarded (I3): a row's true top-200 viewed
    (any leak shows in the output), half the catalogue viewed (the CSR window's binary search), duplicated CSR entries,
    ids beyond the catalogue, a whitelist with viewed ids outside it, a shard with an id offset and global CSR ids."""
    from rectools_b200 import Engine

    rng = np.random.default_rng(len(kind))
    n_rows = 256 if kind == "half_catalogue" else N_ROWS
    u, i, _ = _base(n_rows, N_OBJ, D, seed=21, per_user=0)
    objects, whitelist, id_off, n_cols = i, None, 0, N_OBJ
    if kind == "true_top200":
        cols = list(_true_top(u, i, 200))
    elif kind == "half_catalogue":
        cols = [np.nonzero(rng.random(N_OBJ) < 0.5)[0] for _ in range(n_rows)]
    elif kind == "duplicates":
        cols = [np.repeat(np.union1d(t[:20], rng.choice(N_OBJ, 30)), 2) for t in _true_top(u, i, 20)]
    elif kind == "beyond_catalogue":
        cols = [np.concatenate([t[:15], rng.integers(N_OBJ, 2 * N_OBJ, 40)]) for t in _true_top(u, i, 15)]
    elif kind == "whitelist_outside":
        whitelist = np.sort(rng.choice(N_OBJ, N_OBJ // 3, replace=False)).astype(np.int32)
        cols = [np.union1d(t[:30], rng.choice(N_OBJ, 60)) for t in _true_top(u, i, 30)]
    else:  # id_offset: this engine holds objects [4000, 12000) of a 16000-object catalogue
        id_off = 4_000
        objects = i[id_off : id_off + 8_000]
        top = _true_top(u, objects, 25) + id_off
        cols = [np.union1d(t, rng.choice(N_OBJ, 80)) for t in top]
    indptr, indices = _csr(cols, n_cols)
    eng = Engine(objects, cosine=False, id_offset=id_off)
    _run(eng, lib, monkeypatch, capsys, kind, u, K, objects, False, indptr, indices, whitelist=whitelist, id_off=id_off)
    eng.close()


# ------------------------------------------------------------------------------------------------ passes after the main one
def test_second_chance_pass_with_near_ties(lib, monkeypatch, capsys):
    """Planted near-ties far below the fp16 resolution: the main pass cannot decide, the rows go to the 32-slot re-rank pass
    (launch 2), which is checked like the main pass."""
    from rectools_b200 import Engine

    rng = np.random.default_rng(9)
    n_rows, n_obj, d = 400, 12_000, 64
    u = (rng.standard_normal((n_rows, d)) / np.sqrt(d)).astype(np.float32)
    i = (0.2 * rng.standard_normal((n_obj, d)) / np.sqrt(d)).astype(np.float32)
    base = u.mean(axis=0) + 0.5 * rng.standard_normal(d).astype(np.float32) / np.sqrt(d)
    hot = rng.choice(n_obj, 200, replace=False)
    i[hot] = (3.0 * base[None, :] * (1.0 + 1e-6 * rng.standard_normal((200, 1)))).astype(np.float32)
    u = (u * 0.05 + base[None, :]).astype(np.float32)
    csr = synth_viewed_csr(n_rows, n_obj, 20)
    eng = Engine(i, cosine=False)
    _, reps = _run(eng, lib, monkeypatch, capsys, "near_ties", u, K, i, False, csr.indptr, csr.indices, snaps=(1, 2), min_launches=2)
    assert reps[0][1].n_fb > 0 and reps[1][0]["k_cand"] == 32
    eng.close()


def test_multipass_route_excludes_earlier_results(lib, monkeypatch, capsys):
    """B200_WIDE=0 at k = 60: certified passes of 20 with the earlier results excluded like viewed objects (I1)."""
    from rectools_b200 import Engine

    monkeypatch.setenv("B200_WIDE", "0")
    u, i, csr = _base(600, 12_000, 48, seed=60)
    eng = Engine(i, cosine=True)
    _, reps = _run(eng, lib, monkeypatch, capsys, "multipass_k60", u, 60, i, True, csr.indptr, csr.indices, snaps=tuple(range(1, 8)), min_launches=3)
    assert {r[0]["k0"] for r in reps} >= {0, 20, 40}
    eng.close()


# ------------------------------------------------------------------------------------------------ wide mode
@pytest.mark.parametrize("T", [None, "400", "40", "2000"])
def test_wide_mode_phase_switch(lib, monkeypatch, capsys, T):
    """24 < k <= 128 in one pass: adaptive lists for phase 1, then the frozen threshold and appended candidates.  T = 40
    makes phase 1 the whole stream; T = 2000 freezes a weak threshold after one tile, so lists overflow and their rows must
    be re-ranked."""
    from rectools_b200 import Engine

    if T:
        monkeypatch.setenv("B200_WIDE_T", T)
    u, i, csr = _base(700, 8_000, 32, seed=61)
    eng = Engine(i, cosine=False)
    _, reps = _run(eng, lib, monkeypatch, capsys, f"wide_T{T}", u, 60, i, False, csr.indptr, csr.indices)
    snap, rep, _ = reps[0]
    assert snap["wide"] == 1
    if T == "40":
        assert snap["phase1_tiles"] >= snap["tiles_per_split"]
    if T == "2000":
        assert rep.n_overflow > 0 and rep.n_fb >= rep.n_overflow
    eng.close()
