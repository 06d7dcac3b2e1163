"""GPU: threshold sharing between the shards of an item-sharded catalogue, on one GPU.

Several engines live in one process, one per shard, each attached (`Engine.peer_attach`) to the others' published
arrays or to a planted array of chosen words.  Shards run one after another with the same epoch, so a later shard reads
the final values of the earlier ones; nothing depends on two kernels running at the same time.  Every case ranks each
shard with `B200_TC_SNAPSHOT`, checks the pass with tests/tc_reference.py on every row and list (I1-I4, no verdict I5,
justified thresholds I6, the shard bound restated in fp64 I7, the published array I8), merges the shards' packed
results with `b200_rank_merge_certified`, re-ranks the rejected rows without sharing, merges again, and compares every
row with the fp64 oracle.  Each case prints its global rejection rate and the fraction of lists whose final threshold
is a peer's value: that fraction depends on when the helper warps poll, so only a loose lower bound is asserted."""
import ctypes as C

import numpy as np
import pytest

from oracle.topk_oracle import implicit_topk, neginf_score
from tests.helpers import synth_factors, synth_viewed_csr
from tests.tc_reference import Catalogue, SharedPass, check_snapshot, list_justification, peer_word, subject_operands

pytestmark = pytest.mark.gpu

SENTINEL = int(peer_word(0, np.float32(-1.0)))  # epoch 0 never belongs to a call
_EPOCH = [100]


def _next_epoch():
    _EPOCH[0] += 1
    return _EPOCH[0]


def shared_kcand(k, n_ranks, bf16=False):
    """K' of a threshold-sharing pass (plan.h `plan_call`; pinned by tests/test_call_plan_cpu.py): two lists per rank."""
    L = n_ranks * 2
    cL = 0.56 if L <= 2 else 1.03 if L <= 4 else 1.42 if L <= 8 else 1.77 if L <= 16 else 2.07 if L <= 32 else 2.33
    target = k + max(12.0, 0.6 * k) + (20.0 if bf16 else 0.0)
    kc = 4
    while kc < 32 and L * kc - cL * L * np.sqrt(kc) < target:
        kc += 1
    return kc


def _torch():
    import torch

    return torch


def _words(t):
    return t.cpu().numpy().view(np.uint64).copy()


class Shard:
    """One engine holding objects [lo, lo + n) of the catalogue, with its own published array."""

    def __init__(self, objects, lo, cosine, tc_mode, max_rows, whitelist=None):
        from rectools_b200 import Engine

        torch = _torch()
        self.lo, self.objects, self.whitelist = lo, objects, whitelist
        self.eng = Engine(objects, cosine=cosine, tc_mode=tc_mode, id_offset=lo)
        self.cat = Catalogue(objects, cosine=cosine, bf16=tc_mode == "bf16", whitelist=whitelist, id_off=lo)
        self.pub = torch.full((max_rows,), SENTINEL, dtype=torch.int64, device="cuda:0")
        self.peers = []

    def attach(self, peers):
        self.peers = list(peers)
        self.eng.peer_attach(self.pub, self.peers)


def _rank(sh, monkeypatch, sub, k, epoch, indptr, indices, device_inputs, snap_launch=1, shared=True):
    """One call of shard `sh`: (ids, scores, counts, bounds) numpy, stats, snapshot, peer words before the call, own
    published array before the call."""
    from rectools_b200 import _lib

    torch = _torch()
    n = len(sub)
    peer_before = np.stack([_words(p) for p in sh.peers]) if sh.peers else np.zeros((0, n), np.uint64)
    pub_before = _words(sh.pub)
    monkeypatch.setenv("B200_TC_SNAPSHOT", str(snap_launch))
    wl = sh.whitelist
    k_out = min(k, sh.cat.n_pos)
    flags = _lib.Q_FORCE_TC | (_lib.Q_SHARED_THRESHOLDS if shared else 0)
    if device_inputs:
        dev = torch.device("cuda:0")
        t = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (sub, indptr, indices)]
        t_wl = torch.from_numpy(np.ascontiguousarray(wl, np.int32)).to(dev) if wl is not None else None
        o_ids = torch.empty((n, k_out), dtype=torch.int32, device=dev)
        o_sc = torch.empty((n, k_out), dtype=torch.float32, device=dev)
        o_cnt = torch.empty((n,), dtype=torch.int32, device=dev)
        o_b = torch.empty((n,), dtype=torch.float32, device=dev)
        st = sh.eng.topk_ptrs(n, k, o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(),
                              flags | _lib.Q_INPUTS_ON_DEVICE | _lib.Q_OUTPUTS_ON_DEVICE, subjects=t[0].data_ptr(),
                              indptr=t[1].data_ptr(), indices=t[2].data_ptr(), whitelist=t_wl.data_ptr() if wl is not None else 0,
                              n_whitelist=len(wl) if wl is not None else 0, out_bounds=o_b.data_ptr() if shared else 0,
                              peer_epoch=epoch if shared else 0)
        torch.cuda.synchronize()
        out = tuple(x.cpu().numpy() for x in (o_ids, o_sc, o_cnt, o_b))
    else:
        keep = [np.ascontiguousarray(sub, np.float32), np.ascontiguousarray(indptr, np.int64), np.ascontiguousarray(indices, np.int32)]
        wl32 = np.ascontiguousarray(wl, np.int32) if wl is not None else None
        out = (np.empty((n, k_out), np.int32), np.empty((n, k_out), np.float32), np.zeros(n, np.int32), np.empty(n, np.float32))
        st = sh.eng.topk_ptrs(n, k, out[0].ctypes.data, out[1].ctypes.data, out[2].ctypes.data, flags, subjects=keep[0].ctypes.data,
                              indptr=keep[1].ctypes.data, indices=keep[2].ctypes.data,
                              whitelist=wl32.ctypes.data if wl is not None else 0, n_whitelist=len(wl) if wl is not None else 0,
                              out_bounds=out[3].ctypes.data if shared else 0, peer_epoch=epoch if shared else 0)
    snap = sh.eng.candidate_snapshot()
    monkeypatch.delenv("B200_TC_SNAPSHOT")
    return out, dict(st), snap, peer_before, pub_before


def _merge(parts, n, k):
    """b200_rank_merge_certified over per-shard (ids, scores, counts, bounds) in packed buffers: merged arrays and the
    rejected rows."""
    from rectools_b200 import _lib
    from rectools_b200.sharded import Packed

    torch = _torch()
    dev = torch.device("cuda:0")
    bufs = []
    for ids, sc, cnt, bnd in parts:
        pk = Packed(torch, n, k, dev)
        pk.ids.fill_(-1)
        pk.scores.fill_(-np.finfo(np.float32).max)
        pk.ids[:, : ids.shape[1]] = torch.from_numpy(ids).to(dev)
        pk.scores[:, : sc.shape[1]] = torch.from_numpy(sc).to(dev)
        pk.counts.copy_(torch.from_numpy(cnt).to(dev))
        pk.bounds.copy_(torch.from_numpy(bnd).to(dev))
        bufs.append(pk.buf)
    g = torch.cat(bufs)
    o_ids = torch.empty((n, k), dtype=torch.int32, device=dev)
    o_sc = torch.empty((n, k), dtype=torch.float32, device=dev)
    o_cnt = torch.empty((n,), dtype=torch.int32, device=dev)
    fail_rows = torch.empty((max(n, 1),), dtype=torch.int32, device=dev)
    fail_count = torch.zeros((1,), dtype=torch.int32, device=dev)
    b = g.data_ptr()
    _lib.check(_lib.load().b200_rank_merge_certified(0, None, len(parts), n, k, b, b + 4 * n * k, b + 8 * n * k, b + 8 * n * k + 4 * n,
                                                     n * (2 * k + 2), o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(),
                                                     fail_rows.data_ptr(), fail_count.data_ptr()))
    torch.cuda.synchronize()
    nf = int(fail_count.item())
    return o_ids.cpu().numpy(), o_sc.cpu().numpy(), o_cnt.cpu().numpy(), np.sort(fail_rows[:nf].cpu().numpy())


def _oracle(objects, sub, k, csr, whitelist, cosine):
    cat = Catalogue(objects, cosine=cosine, bf16=False)
    outside = None if whitelist is None else np.setdiff1d(np.arange(len(objects)), whitelist)
    ids, sc = implicit_topk(objects, sub, k, cat.norms if cosine else None, csr, outside, accum="f64")
    valid = sc > np.float32(neginf_score())
    return np.where(valid, ids, -1), sc, valid.sum(axis=1)


def run_case(monkeypatch, capsys, name, shards, order, sub, k, csr, objects_all, cosine, device_inputs=True, snap_launch=1,
             whitelist_all=None, bf16=False, n_ranks=None, min_adopt=0.0, epoch=None):
    """Rank every shard of `order` in turn (shared), check each pass, merge, re-rank the rejected rows, compare with the
    oracle.  `n_ranks`: ranks K' is planned for (planted peer arrays count).  Returns the reports, the rejected rows and
    the raw results of each shard."""
    n = len(sub)
    epoch = epoch or _next_epoch()
    indptr, indices = csr.indptr.astype(np.int64), csr.indices.astype(np.int32)
    n_ranks = n_ranks or len(shards)
    runs = {}
    for s in order:
        sh = shards[s]
        out, st, snap, peer_before, pub_before = _rank(sh, monkeypatch, sub, k, epoch, indptr, indices, device_inputs, snap_launch)
        assert st["path"] == 1 and st["n_fallback_rows"] == 0, st
        assert st["k_cand"] == shared_kcand(k, n_ranks, bf16), st
        assert snap is not None and snap["k_cand"] == st["k_cand"] and snap["launch"] == snap_launch
        runs[s] = (out, st, snap, peer_before, pub_before, _words(sh.pub))
    # each pass's rows, subjects and the lists' own justification (published units)
    rows = runs[order[0]][2]["rows"].astype(np.int64)
    vw = {s: shards[s].cat.viewed_positions(indptr, indices, n)[rows] for s in order}
    just = {s: list_justification(runs[s][2], shards[s].cat, sub[rows], vw[s]) for s in order}
    reports = {}
    for s in order:
        out, st, snap, peer_before, pub_before, pub_after = runs[s]
        assert (snap["rows"] == rows).all()
        others = [just[o] for o in order if o != s]
        justify = np.max(others, axis=0) if others else np.full(len(rows), -np.inf)
        sp = SharedPass(out[3][rows], epoch, peer_before[:, rows], justify, pub_before, pub_after, n)
        rep = check_snapshot(snap, shards[s].cat, sub[rows], vw[s], shared=sp)
        with capsys.disabled():
            print(f"\n[{name} shard {s}] nw={snap['nw']} splits={snap['n_splits']} K'={snap['k_cand']} obj_exp={snap['obj_exp']} "
                  f"rows {rows[0]}..{rows[-1]} {rep.summary()} adopted_frac={rep.n_adopted / max(1, rep.n_peer_lists):.3f}")
        assert rep.ok, f"{name} shard {s}: {rep.summary()}"
        assert rep.n_published > 0, f"{name} shard {s}: nothing published at the pass's rows"
        reports[s] = rep
    # the global certificate, the re-rank of its rejected rows without sharing, the merge again
    parts = [runs[s][0] for s in sorted(order)]
    ids, sc, cnt, fail = _merge(parts, n, k)
    if len(fail):
        re = []
        for s in sorted(order):
            sub_csr = csr[fail]
            out, st, _, _, _ = _rank(shards[s], monkeypatch, sub[fail], k, 0, sub_csr.indptr.astype(np.int64),
                                     sub_csr.indices.astype(np.int32), device_inputs, shared=False)
            re.append((out[0], out[1], out[2], np.full(len(fail), -np.inf, np.float32)))
        r_ids, r_sc, r_cnt, r_fail = _merge(re, len(fail), k)
        assert len(r_fail) == 0
        ids[fail], sc[fail], cnt[fail] = r_ids, r_sc, r_cnt
    oid, osc, ocnt = _oracle(objects_all, sub, k, csr, whitelist_all, cosine)
    np.testing.assert_array_equal(cnt, ocnt, err_msg=name)
    valid = np.arange(k)[None, :] < cnt[:, None]
    np.testing.assert_array_equal(np.where(valid, ids, -1), oid, err_msg=name)
    np.testing.assert_allclose(sc[valid], osc[valid], rtol=3e-7, atol=1.5e-45, err_msg=name)
    n_peer = sum(r.n_peer_lists for r in reports.values())
    n_adopt = sum(r.n_adopted for r in reports.values())
    with capsys.disabled():
        print(f"[{name}] rejected by the global certificate: {len(fail)}/{n} = {len(fail) / n:.4f}; lists that adopted a peer "
              f"value: {n_adopt}/{n_peer} = {n_adopt / max(1, n_peer):.3f}")
    assert n_adopt >= min_adopt * n_peer, f"{name}: {n_adopt} of {n_peer} lists adopted a peer value"
    return reports, fail, runs


def _shards(objects, n_shards, cosine=False, tc_mode="auto", max_rows=None, n_rows=0, whitelist=None):
    from rectools_b200.sharded import shard_bounds, split_whitelist

    out = []
    for lo, hi in shard_bounds(len(objects), n_shards):
        wl = split_whitelist(whitelist, lo, hi) if whitelist is not None else None
        out.append(Shard(objects[lo:hi], lo, cosine, tc_mode, max_rows or n_rows + 64, wl))
    for s, sh in enumerate(out):
        sh.attach([o.pub for t, o in enumerate(out) if t != s])
    return out


def _close(shards):
    for sh in shards:
        sh.eng.close()


# ------------------------------------------------------------------------------------------------ two real shards
def test_two_shards_b_adopts_a(monkeypatch, capsys):
    """DOT fp16, k = 10, a filter, device inputs: the PEERS kernel runs, B adopts A's final values, K' = 9."""
    n_rows, n_obj, d, k = 768, 60_000, 64, 10
    u, i = synth_factors(n_rows, n_obj, d, seed=31)
    csr = synth_viewed_csr(n_rows, n_obj, 40, seed=32)
    shards = _shards(i, 2, n_rows=n_rows)
    assert shared_kcand(k, 2) == 9
    reps, _, _ = run_case(monkeypatch, capsys, "two_shards", shards, [0, 1], u, k, csr, i, False, min_adopt=0.05)
    assert reps[0].n_peer_lists == 0  # A ran first: B's array held no value of this epoch
    _close(shards)


def test_scaled_shard_runs_first(monkeypatch, capsys):
    """Shard B's objects scaled by 2^6 (its object exponent is 6 lower) and B ranked first: A adopts B's thresholds
    through the exponent conversion."""
    n_rows, n_obj, d, k = 768, 60_000, 64, 10
    u, i = synth_factors(n_rows, n_obj, d, seed=41)
    i[n_obj // 2 :] *= np.float32(64.0)
    csr = synth_viewed_csr(n_rows, n_obj, 40, seed=42)
    shards = _shards(i, 2, n_rows=n_rows)
    assert shards[0].cat.obj_exp - shards[1].cat.obj_exp == 6
    reps, _, _ = run_case(monkeypatch, capsys, "scaled_b_first", shards, [1, 0], u, k, csr, i, False, min_adopt=0.05)
    assert reps[1].n_peer_lists == 0 and reps[0].n_adopted > 0
    _close(shards)


# ------------------------------------------------------------------------------------------------ a planted peer
def test_planted_peer_chunked_host_inputs(monkeypatch, capsys):
    """One engine attached to one planted array, host inputs in four row chunks, the third chunk's pass checked
    (`peer_row0` = 600).  Rows = 0 mod 3: a valid value of the call's epoch; = 1 mod 3: a value above every score, which
    lists adopt and the global certificate rejects; = 2 mod 3: huge values of epoch 0 or epoch + 1, or NaN words of the
    call's epoch, which no list may adopt.  Slots past the call's 1000 rows stay untouched."""
    torch = _torch()
    n_rows, n_obj, d, k = 1000, 40_000, 64, 10
    u, i = synth_factors(n_rows, n_obj, d, seed=51)
    csr = synth_viewed_csr(n_rows, n_obj, 30, seed=52)
    monkeypatch.setenv("B200_CHUNK_ROWS", "300")
    sh = Shard(i, 0, False, "auto", n_rows + 100)
    epoch = _next_epoch()
    row_exp = subject_operands(u, False)[0]
    top, kth = np.empty(n_rows), np.empty(n_rows)
    for r0 in range(0, n_rows, 250):
        s = u[r0 : r0 + 250].astype(np.float64) @ i.astype(np.float64).T
        top[r0 : r0 + 250] = s.max(axis=1)
        kth[r0 : r0 + 250] = -np.partition(-s, 29, axis=1)[:, 29]
    r = np.arange(n_rows)
    value = np.where(r % 3 == 0, kth, top + 0.05 * np.abs(top) + 1e-6)
    words = np.full(n_rows + 100, SENTINEL, np.uint64)
    words[:n_rows] = peer_word(epoch, np.ldexp(value, row_exp))
    huge = np.float32(1e30)
    words[:n_rows][r % 9 == 2] = peer_word(0, huge)
    words[:n_rows][r % 9 == 5] = peer_word(epoch + 1, huge)
    words[:n_rows][r % 9 == 8] = peer_word(epoch, np.float32(np.nan))
    fake = torch.from_numpy(words.view(np.int64)).to("cuda:0")
    sh.attach([fake])
    reps, fail, runs = run_case(monkeypatch, capsys, "planted_chunked", [sh], [0], u, k, csr, i, False, device_inputs=False,
                                snap_launch=3, n_ranks=2, epoch=epoch)
    assert runs[0][1]["n_chunks"] == 4
    snap, rep = runs[0][2], reps[0]
    rows = snap["rows"].astype(np.int64)
    assert rows[0] == 600 and len(rows) == 300
    assert (_words(fake) == words).all()  # a peer's array is only read
    # rows = 1 mod 3: adopted (timing: loosely), and every adopting row rejected by the global certificate
    ones = rows % 3 == 1
    adopted = np.zeros(len(rows), bool)
    adopted[rep.adopted_rows] = True
    with capsys.disabled():
        print(f"[planted_chunked] rows = 1 mod 3 of the third chunk that adopted the planted value: {int((adopted & ones).sum())}/{int(ones.sum())}")
    assert (adopted & ones).sum() >= 0.5 * ones.sum()
    assert set(rows[adopted & ones].tolist()) <= set(fail.tolist())
    # rows = 2 mod 3: nothing of a wrong epoch and no NaN was adopted (I6 too)
    thr = snap["cand_thr"][:, : len(rows)]
    assert not adopted[rows % 3 == 2].any()
    assert (thr[:, rows % 3 == 2] < np.ldexp(np.float64(huge), snap["obj_exp"])).all() and not np.isnan(thr).any()
    sh.eng.close()


# ------------------------------------------------------------------------------------------------ negative bounds
@pytest.mark.parametrize("cosine", [False, True], ids=["dot", "cosine"])
def test_negative_rows(monkeypatch, capsys, cosine):
    """Every score negative (negative subjects, non-negative objects): the shard bound is negative, and its slack must
    still move it up (I7).  The factor (1 + 2.4e-7) of the earlier formula put it 2-4 ulps below max tau + eps."""
    n_rows, n_obj, d, k = 512, 40_000, 64, 10
    u, i = synth_factors(n_rows, n_obj, d, seed=61)
    u, i = -np.abs(u), np.abs(i)
    csr = synth_viewed_csr(n_rows, n_obj, 30, seed=62)
    shards = _shards(i, 2, cosine=cosine, n_rows=n_rows)
    _, _, runs = run_case(monkeypatch, capsys, f"negative_{'cos' if cosine else 'dot'}", shards, [0, 1], u, k, csr, i, cosine)
    for s in (0, 1):
        assert (runs[s][0][3] < 0).all()
    _close(shards)


# ------------------------------------------------------------------------------------------------ the other instantiations
@pytest.mark.parametrize(
    "name, env, tc_mode, k, whitelist",
    [
        ("bf16_splits3", {"B200_TC_SPLITS": "3"}, "bf16", 10, False),
        ("bf16_k24", {}, "bf16", 24, False),
        ("nw8_bf16", {}, "bf16", 10, False),
        ("splits3", {"B200_TC_SPLITS": "3"}, "auto", 10, False),
        ("whitelist", {}, "auto", 10, True),
        ("k1", {}, "auto", 1, False),
        ("k24", {}, "auto", 24, False),
    ],
)
def test_instantiations_and_options(monkeypatch, capsys, name, env, tc_mode, k, whitelist):
    """bf16 operands (the other PEERS kernel), also with three splits and k = 24; three object splits of a row publishing
    to the same slot; a per-shard whitelist; k = 1 and k = 24."""
    for key, val in env.items():
        monkeypatch.setenv(key, val)
    n_rows, n_obj, d = 640, 60_000, 64
    u, i = synth_factors(n_rows, n_obj, d, seed=70 + len(name))
    csr = synth_viewed_csr(n_rows, n_obj, 40, seed=71)
    wl = np.sort(np.random.default_rng(72).choice(n_obj, n_obj * 3 // 5, replace=False)) if whitelist else None
    shards = _shards(i, 2, tc_mode=tc_mode, n_rows=n_rows, whitelist=wl)
    _, _, runs = run_case(monkeypatch, capsys, name, shards, [0, 1], u, k, csr, i, False, whitelist_all=wl,
                          bf16=tc_mode == "bf16", min_adopt=0.01)
    snap = runs[1][2]
    assert snap["nw"] == 8 and snap["bf16"] == (tc_mode == "bf16")
    if "B200_TC_SPLITS" in env:
        assert snap["n_splits"] == 3
    if whitelist:
        assert snap["n_pos"] == len(shards[1].whitelist)
    _close(shards)


def test_nine_shards(monkeypatch, capsys):
    """The widest exchange: nine shards, each attached to the other eight (MAX_PEERS), k = 10, K' = 7."""
    n_rows, n_obj, d, k = 512, 72_000, 64, 10
    u, i = synth_factors(n_rows, n_obj, d, seed=81)
    csr = synth_viewed_csr(n_rows, n_obj, 40, seed=82)
    shards = _shards(i, 9, n_rows=n_rows)
    assert shared_kcand(k, 9) == 7 and all(len(sh.peers) == 8 for sh in shards)
    run_case(monkeypatch, capsys, "nine_shards", shards, list(range(9)), u, k, csr, i, False, min_adopt=0.05)
    _close(shards)


# ------------------------------------------------------------------------------------------------ refusals
def test_attach_refusals():
    from rectools_b200 import Engine, _lib

    torch = _torch()
    u, i = synth_factors(300, 4_000, 32, seed=91)
    lib = _lib.load()
    arr = [torch.zeros(200, dtype=torch.int64, device="cuda:0") for _ in range(10)]
    eng = Engine(i, cosine=False)
    with pytest.raises(NotImplementedError):  # more than MAX_PEERS = 8
        eng.peer_attach(arr[0], arr[1:10])
    ptrs = (C.c_void_p * 2)(arr[1].data_ptr(), None)
    assert lib.b200_rank_peer_attach(eng._h, 200, None, 1, ptrs) == _lib.E_INVALID  # pylint: disable=protected-access
    assert lib.b200_rank_peer_attach(eng._h, 200, arr[0].data_ptr(), 2, ptrs) == _lib.E_INVALID  # pylint: disable=protected-access
    assert lib.b200_rank_peer_attach(eng._h, 200, arr[0].data_ptr(), 1, None) == _lib.E_INVALID  # pylint: disable=protected-access
    host = np.zeros(200, np.uint64)
    ptrs = (C.c_void_p * 1)(host.ctypes.data)
    assert lib.b200_rank_peer_attach(eng._h, 200, arr[0].data_ptr(), 1, ptrs) == _lib.E_INVALID  # pylint: disable=protected-access
    # refused calls changed nothing: a call with shared thresholds runs the plain kernel (no peers)
    eng.peer_attach(arr[0], arr[1:3])
    with pytest.raises(ValueError):  # attached once already
        eng.peer_attach(arr[0], arr[1:2])
    with pytest.raises(ValueError):  # the engine's arrays are caller-owned now
        eng.peer_export(200)
    # n_rows > max_rows
    out = (np.empty((300, 10), np.int32), np.empty((300, 10), np.float32), np.zeros(300, np.int32), np.empty(300, np.float32))
    with pytest.raises(ValueError):
        eng.topk_ptrs(300, 10, out[0].ctypes.data, out[1].ctypes.data, out[2].ctypes.data, _lib.Q_SHARED_THRESHOLDS | _lib.Q_FORCE_TC,
                      subjects=np.ascontiguousarray(u).ctypes.data, out_bounds=out[3].ctypes.data, peer_epoch=3)
    eng.close()
    # attach after export
    eng = Engine(i, cosine=False)
    eng.peer_export(200)
    with pytest.raises(ValueError):
        eng.peer_attach(arr[0], arr[1:2])
    eng.close()
    assert all(int(a.abs().sum()) == 0 for a in arr)  # never written: no call ranked with them
