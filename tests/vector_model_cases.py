"""The case table of the vector-model tests (test infrastructure only): the unmodified `LightFMWrapperModel` (through the
`lightfm` stand-in), `ImplicitBPRWrapperModel` and `DSSMModel` ranked through `install()`, every engine row held to the
rounding-interval oracle of `tests/score_interval.py` with no tolerance.

The ranker behind `install()` is `integration.B200ImplicitRanker`; the tests bind a recording subclass of it
(`recording_ranker`) that logs every padded answer (`_rank_padded`, which `rank()` and `rank_padded()` both go through).
On an H100 the base is the engine's own class; on a CPU it is `OracleImplicitRanker`, the same surface backed by
`tests/blocked_oracle.py` (fp64 dots rounded once to fp32), so that the cases, the stand-ins and the checks run without
a GPU.  `OracleImplicitRanker.mutation` makes that provider subtly wrong, to show that `check_case` bites.

For every call `check_case` recomputes what the ranker must have seen -- the model's own vectors
(`_get_u2i_vectors` / `_get_i2i_vectors`), `prepare_factors`, the viewed-items filter, the whitelist and k -- from the
model and the dataset, not from what the ranker received, and asserts:
  1. `check_topk` on every padded answer;
  2. the frame from `install()` equal to the flattening of those answers with the reference's post-scaling
     (`/ subject norm` for COSINE, `sqrt(max(dots - s, 0))` for EUCLIDEAN; rank_implicit.py:132-140), bit for bit, the
     subject norms and dots restated here from the vectors;
  3. the frame against the stock frame: names and dtypes equal, ids equal up to near-ties of the stock fp32 arithmetic;
  4. the frames with `fast_recommend=True` and `False` identical."""
from __future__ import annotations

import typing as tp

import numpy as np

from tests.blocked_oracle import blocked_oracle
from tests.helpers import assert_same_ranking
from tests.score_interval import check_topk, rn32

SIZES = {"cpu": dict(n_users=400, n_items=1200, per_user=20), "gpu": dict(n_users=2000, n_items=5000, per_user=30)}
TC_MAX_D_PAD = 320  # the widest object rows the tensor-core pass takes (plan_fused in engine.cu: two smem stages)
TC_MIN_PAIRS = 4.0e6  # below rows x positions the plan ranks on the exhaustive kernel (plan.h)


# ------------------------------------------------------------------------------------------------ the providers
class OracleImplicitRanker:
    """`B200ImplicitRanker`'s surface on the CPU: `prepare_factors` as the engine's ranker does, padded answers from
    `blocked_oracle` (the engine's scores before post-scaling), `B200Ranker.rank` / `rank_padded` on top.  `mutation`
    (test infrastructure for the mutation test): "swap_tied", "ulp", "next_filter" or "no_norm"; `applied` counts the
    answers it changed."""

    mutation: tp.Optional[str] = None
    applied = [0]  # (a list: the recording subclass counts into its base's)

    def __init__(self, distance, subjects_factors, objects_factors, num_threads=0, use_gpu=False):  # pylint: disable=unused-argument
        from rectools_b200.ranker import _as_distance, _dense_f32, prepare_factors

        self.distance = _as_distance(distance)
        sub, obj = _dense_f32(subjects_factors), _dense_f32(objects_factors)
        self.n_subjects, self.n_objects = sub.shape[0], obj.shape[0]
        self._sub, self._obj, self.subjects_norms, self.subjects_dots = prepare_factors(self.distance, sub, obj)
        if self.mutation == "no_norm" and self.subjects_norms is not None:
            self.subjects_norms = np.ones_like(self.subjects_norms)
            self.applied[0] += 1
        self._subjects_csr = self._identity = None
        self.last_stats: tp.Dict[str, tp.Any] = {}

    def _rank_padded(self, subject_ids, k=None, filter_pairs_csr=None, sorted_object_whitelist=None, flags=0):  # pylint: disable=unused-argument
        sids = np.asarray(subject_ids, dtype=np.int64).reshape(-1)
        wl = None if sorted_object_whitelist is None else np.asarray(sorted_object_whitelist, np.int64)
        filt = filter_pairs_csr
        if self.mutation == "next_filter" and filt is not None and filt.shape[0] > 1:
            filt = filt[np.roll(np.arange(filt.shape[0]), -1)]
            self.applied[0] += 1
        dist = "cosine" if self.distance.value == "cosine" else "dot"
        ids, scores, counts = blocked_oracle(dist, self._sub[sids], self._obj, k, filt, wl)
        if self.mutation == "ulp" and counts.size and counts[0] > 0:
            scores[0, 0] = np.nextafter(scores[0, 0], np.float32(np.inf))
            self.applied[0] += 1
        if self.mutation == "swap_tied":
            tied = np.argwhere((scores[:, 1:] == scores[:, :-1]) & (np.arange(1, scores.shape[1])[None, :] < counts[:, None]))
            if len(tied):
                r, c = tied[0]
                ids[r, c], ids[r, c + 1] = ids[r, c + 1], ids[r, c]
                self.applied[0] += 1
        return sids, ids, scores, counts, None

    def rank_padded(self, subject_ids, k=None, filter_pairs_csr=None, sorted_object_whitelist=None, flags=0):
        return self._rank_padded(subject_ids, k, filter_pairs_csr, sorted_object_whitelist, flags)[:4]

    def rank(self, subject_ids, k=None, filter_pairs_csr=None, sorted_object_whitelist=None):
        """`B200Ranker.rank`: the flattening and the post-scaling of `B200Ranker._final_scores`."""
        from rectools_b200.ranker import B200Ranker, flatten_padded

        flat = flatten_padded(*self._rank_padded(subject_ids, k, filter_pairs_csr, sorted_object_whitelist)[:4])
        return B200Ranker._final_scores(self, *flat)  # pylint: disable=protected-access


def recording_ranker(base: type, log: tp.List[tp.Dict[str, tp.Any]]) -> type:
    """A subclass of `base` that appends every padded answer to `log`, with the plan statistics of the call and the
    engine's `d_pad` when there is an engine."""

    class Recording(base):  # type: ignore[misc, valid-type]
        def _rank_padded(self, subject_ids, k=None, filter_pairs_csr=None, sorted_object_whitelist=None, flags=0):
            out = super()._rank_padded(subject_ids, k, filter_pairs_csr, sorted_object_whitelist, flags)
            sids, ids, scores, counts = out[:4]
            engine = getattr(self, "engine", None)
            log.append(dict(distance=self.distance.value, sids=np.array(sids), ids=np.array(ids), scores=np.array(scores),
                            counts=np.array(counts), stats=dict(self.last_stats),
                            d_pad=engine.info()["d_pad"] if engine is not None else None))
            return out

    return Recording


# ------------------------------------------------------------------------------------------------ the models
def _lightfm_arrays(rng, n_user_rows, n_item_rows, nc, bias):
    """Embeddings N(0, 1/nc), item rows scaled by a log-normal factor (heavy-tailed item norms).  `bias`: "small"
    (|b| ~ 0.1) or "dominant" (b_u uniform in 5 ... 50, everything item-dependent ~1e-3: many items round to the same
    fp32 score, exact ties across the k-th entry)."""
    ue = rng.standard_normal((n_user_rows, nc)) / np.sqrt(nc)
    ie = rng.standard_normal((n_item_rows, nc)) / np.sqrt(nc) * rng.lognormal(0.0, 0.5, (n_item_rows, 1))
    if bias == "small":
        ub, ib = 0.1 * rng.standard_normal(n_user_rows), 0.1 * rng.standard_normal(n_item_rows)
    else:
        ue, ie = 0.03 * ue, 0.03 * ie
        ub, ib = rng.uniform(5.0, 50.0, n_user_rows), 1e-3 * rng.standard_normal(n_item_rows)
    return ue, ie, ub, ib


LIGHTFM = {f"lightfm_{nc}_{bias}": (nc, bias) for nc in (30, 64, 318, 319) for bias in ("small", "dominant")}
MODELS = [*LIGHTFM, "lightfm_features", "bpr", "dssm"]


def build(name: str, size: str) -> tp.Tuple[tp.Any, tp.Any]:
    """(model, dataset) of a case."""
    from tests.ref_models import featured_dataset, injected_bpr, injected_lightfm, small_dssm, synthetic_dataset

    sz = SIZES[size]
    rng = np.random.default_rng(sum(map(ord, name)))
    if name in LIGHTFM:
        nc, bias = LIGHTFM[name]
        ds = synthetic_dataset(sz["n_users"], sz["n_items"], sz["per_user"], seed=1)
        return injected_lightfm(ds, *_lightfm_arrays(rng, sz["n_users"], sz["n_items"], nc, bias)), ds
    if name == "lightfm_features":
        ds = featured_dataset(sz["n_users"], sz["n_items"], sz["per_user"], seed=2, n_warm_users=40, n_warm_items=60)
        n_uf = ds.n_hot_users + ds.user_features.get_sparse().shape[1]
        n_if = ds.n_hot_items + ds.item_features.get_sparse().shape[1]
        return injected_lightfm(ds, *_lightfm_arrays(rng, n_uf, n_if, 64, "small")), ds
    if name == "bpr":
        ds = synthetic_dataset(sz["n_users"], sz["n_items"], sz["per_user"], seed=3)
        d = 64
        u = rng.standard_normal((sz["n_users"], d)) / np.sqrt(d)
        i = rng.standard_normal((sz["n_items"], d)) / np.sqrt(d)
        return injected_bpr(u, i, 0.3 * rng.standard_normal(sz["n_items"])), ds
    if name == "dssm":
        ds = featured_dataset(sz["n_users"], sz["n_items"], sz["per_user"], seed=4)
        return small_dssm(ds), ds
    raise KeyError(name)


def calls(name: str, ds: tp.Any) -> tp.List[tp.Tuple[str, tp.Dict[str, tp.Any]]]:
    """(kind, keyword arguments of `recommend` / `recommend_to_items`) of a case; the targets are under "targets"."""
    users = ds.user_id_map.external_ids[: ds.n_hot_users]
    n_items = ds.n_hot_items if hasattr(ds, "n_hot_items") else ds.item_id_map.size
    items = ds.item_id_map.external_ids[:n_items]
    sub = users[np.random.default_rng(0).permutation(len(users))[: len(users) * 4 // 5]]  # a subset, out of order
    wl = np.setdiff1d(items, items[::4])  # three quarters of the catalogue
    wl_small = items[::3]
    targets = items[np.random.default_rng(1).permutation(len(items))[: len(items) // 4]]
    if name == "lightfm_features":
        warm_u = ds.user_id_map.external_ids[ds.n_hot_users :]
        warm_i = ds.item_id_map.external_ids[n_items :]
        mixed_u = np.concatenate([sub[:200], warm_u[::2], [-1, -8], sub[200:300]])
        mixed_i = np.concatenate([targets[:100], warm_i[::2], [-3], targets[100:150]])
        return [("u2i", dict(targets=sub, k=10, filter_viewed=True)),
                ("u2i", dict(targets=mixed_u, k=10, filter_viewed=True, on_unsupported_targets="ignore")),
                ("u2i", dict(targets=mixed_u, k=25, filter_viewed=False, items_to_recommend=wl, on_unsupported_targets="ignore")),
                ("i2i", dict(targets=targets, k=10, filter_itself=True)),
                ("i2i", dict(targets=mixed_i, k=10, filter_itself=True, on_unsupported_targets="ignore")),
                ("i2i", dict(targets=mixed_i, k=12, filter_itself=False, items_to_recommend=wl, on_unsupported_targets="ignore"))]
    if name in ("bpr", "dssm"):
        return [("u2i", dict(targets=sub, k=10, filter_viewed=True)),
                ("u2i", dict(targets=sub, k=100, filter_viewed=True, items_to_recommend=wl)),
                ("i2i", dict(targets=targets, k=10, filter_itself=True)),
                ("i2i", dict(targets=targets, k=100, filter_itself=True, items_to_recommend=wl))]
    nc, _ = LIGHTFM[name]
    ks = (1, 10, 24, 25, 100, 129, 1025) if nc == 64 else (1, 10, 25, 129, 1025)
    out = []
    for j, k in enumerate(ks):
        if k > n_items:
            continue
        out.append(("u2i", dict(targets=sub, k=k, filter_viewed=j % 2 == 0, items_to_recommend=wl if j % 3 == 2 else None)))
    out += [("u2i", dict(targets=sub[:64], k=n_items + 7, filter_viewed=True)),
            ("u2i", dict(targets=sub, k=10, filter_viewed=True, items_to_recommend=wl_small)),
            ("i2i", dict(targets=targets, k=10, filter_itself=True)),
            ("i2i", dict(targets=targets, k=10, filter_itself=False)),
            ("i2i", dict(targets=targets, k=100, filter_itself=True, items_to_recommend=wl))]
    return out


def invoke(model, ds, kind, kw):
    kw = dict(kw)
    targets = kw.pop("targets")
    if kind == "u2i":
        return model.recommend(targets, ds, **kw)
    return model.recommend_to_items(targets, ds, **kw)


# ------------------------------------------------------------------------------------------------ the checks
def _expected_vectors(model, ds, kind):
    """What the ranker must see: the model's vectors, as fp32 (rank_implicit.py:70-71), through `prepare_factors`;
    with the fp32 subject vectors (for the post-scaling)."""
    from rectools_b200.ranker import _as_distance, _dense_f32, prepare_factors

    dist = _as_distance(model.u2i_dist if kind == "u2i" else model.i2i_dist)
    s, o = model._get_u2i_vectors(ds) if kind == "u2i" else model._get_i2i_vectors(ds)  # pylint: disable=protected-access
    s32, o32 = _dense_f32(s), _dense_f32(o)
    s_aug, o_aug, _, _ = prepare_factors(dist, s32, o32)
    return dist.value, s32, s_aug, o_aug


def _post_scale(dist, s32, sids, scores):
    """The reference's post-scaling of engine scores (rank_implicit.py:132-140), restated: COSINE divides by the subject
    norm -- fp32 of the fp64 norm, zero read as 1e-10 --, EUCLIDEAN takes sqrt(max(|s|^2 - score, 0)) with the fp32 sum of
    squares the reference computes (`_calc_dots`)."""
    if dist == "cosine":
        norms = rn32(np.sqrt(np.einsum("ij,ij->i", s32.astype(np.float64), s32.astype(np.float64))))
        norms[norms == 0] = np.float32(1e-10)
        return (scores / norms[sids]).astype(np.float32)
    if dist == "euclidean":
        dots = (s32**2).sum(axis=1)
        return np.sqrt(np.maximum(dots[sids] - scores, 0)).astype(np.float32)
    return scores


def _ties_across_cut(rec, s_aug, o_aug, viewed, wl):
    """Rows whose k-th returned score (before post-scaling) is also the fp32 score of an eligible object left out."""
    k_out = rec["ids"].shape[1]
    pos = np.arange(o_aug.shape[0]) if wl is None else wl
    sc = rn32(s_aug[rec["sids"]].astype(np.float64) @ o_aug[pos].astype(np.float64).T)
    n = 0
    for r in np.nonzero(rec["counts"] == k_out)[0]:
        elig = np.ones(len(pos), bool)
        if viewed is not None:
            elig &= ~np.isin(pos, viewed[r].indices)
        elig &= ~np.isin(pos, rec["ids"][r])
        n += bool((sc[r][elig] == rec["scores"][r, k_out - 1]).any())
    return n


def _flat_frame(rec, dist, s32, kind, kw):
    """(target, item, score) of the frame the recorded answer must give: the flattening with post-scaling; i2i with
    `filter_itself` drops the target itself and keeps the first k (base.py:745-753)."""
    valid = np.arange(rec["ids"].shape[1])[None, :] < rec["counts"][:, None]
    sub = np.repeat(rec["sids"], rec["counts"])
    ids = rec["ids"][valid].astype(np.int64)
    scores = _post_scale(dist, s32, sub, rec["scores"][valid])
    if kind == "i2i" and kw.get("filter_itself", True):
        keep = ids != sub
        rank = np.concatenate([np.cumsum(keep[sub == t]) for t in rec["sids"]]) if len(sub) else keep
        keep &= rank <= kw["k"]
        sub, ids, scores = sub[keep], ids[keep], scores[keep]
    return sub, ids, scores


def _same_reco(ref_df, got_df, target_col, euclidean_scale=None):
    """The comparison with the stock frame: the only tolerance of these tests (near-ties of the stock fp32 arithmetic).
    EUCLIDEAN distances come from `|s|^2 - score`, a difference the stock path forms in fp32: its error is a multiple of
    the squared norms (`euclidean_scale`), not of the distance, so squared distances are compared at that scale."""
    assert list(ref_df.columns) == list(got_df.columns)
    assert [str(t) for t in ref_df.dtypes] == [str(t) for t in got_df.dtypes]
    np.testing.assert_array_equal(ref_df[target_col].to_numpy(), got_df[target_col].to_numpy())
    if "rank" in ref_df:
        np.testing.assert_array_equal(ref_df["rank"].to_numpy(), got_df["rank"].to_numpy())
    got, exp = (np.asarray(df["score"].to_numpy(), np.float64) for df in (got_df, ref_df))
    atol, tie_tol = 3e-6, 3e-6
    if euclidean_scale is not None:
        got, exp = got**2, exp**2
        atol = 3e-6 * euclidean_scale
        tie_tol = atol / max(1e-30, float(np.abs(exp).max(initial=0.0)))
    return assert_same_ranking(got_df["item_id"].to_numpy(), got, ref_df["item_id"].to_numpy(), exp, rtol=3e-5, atol=atol,
                               tie_tol=tie_tol)


def expected_path(rec, n_pos, k_out):
    """The plan's route for a recorded call (plan.h): the tensor cores for d_pad <= 320 where the call is large enough,
    path 3 above k = 1024; off the tensor cores path 0 (k <= 128) or 3."""
    n_rows = len(rec["sids"])
    if rec["d_pad"] > TC_MAX_D_PAD:
        return (3,) if k_out > 128 else (0,)
    if k_out > 1024:
        return (3,)
    if n_rows * n_pos < TC_MIN_PAIRS:
        return (0, 3) if k_out > 128 else (0,)
    return (1,) if k_out <= 128 else (1, 3)


def check_case(model, ds, kind, kw, stock, frames, logs, label="", need_ties=False):
    """Asserts 1-4 of the module docstring for one call; `frames` / `logs`: {fast_recommend: frame / recorded answers}.
    Returns a summary line.  `need_ties`: some row must have an exact fp32 tie across its k-th entry."""
    dist, s32, s_aug, o_aug = _expected_vectors(model, ds, kind)
    target_col = "user_id" if kind == "u2i" else "target_item_id"
    k = kw["k"] + 1 if kind == "i2i" and kw.get("filter_itself", True) else kw["k"]
    wl = None
    if kw.get("items_to_recommend") is not None:
        wl = np.unique(ds.item_id_map.convert_to_internal(kw["items_to_recommend"], strict=False))
    n_pos = o_aug.shape[0] if wl is None else len(wl)
    viewed_all = ds.get_user_item_matrix(include_weights=False) if kind == "u2i" and kw["filter_viewed"] else None
    n_hot = ds.n_hot_users if kind == "u2i" else ds.n_hot_items
    lines, ties, mixed = [], 0, False
    for fast, log in logs.items():
        assert log, f"{label}: the ranker was not called (fast_recommend={fast})"
        parts = []
        for rec in log:
            warm = bool(len(rec["sids"]) and rec["sids"].max() >= n_hot)
            mixed |= warm or len(log) > 1
            # the warm rows rank without the filter (`_recommend_u2i_warm`, lightfm.py:304-311)
            viewed = viewed_all[rec["sids"]] if viewed_all is not None and not warm else None
            rep = check_topk((rec["ids"], rec["scores"], rec["counts"]), s_aug[rec["sids"]], o_aug, k,
                             cosine=dist == "cosine", filter_csr=viewed, whitelist=wl, name=f"{label} fast={fast}", verbose=False,
                             max_ambiguous=5e-4)  # (d ~ 320 and whole-catalogue k: ~1e-4 of the returned scores straddle a rounding boundary)
            st = rec["stats"]
            k_out = rec["ids"].shape[1]
            if rec["d_pad"] is not None:
                assert st["path"] in expected_path(rec, n_pos, k_out), (label, fast, st, rec["d_pad"])
                lines.append(f"path {st['path']} d_pad {rec['d_pad']} launches {st['n_tc_launches']} fallback "
                             f"{st['n_fallback_rows']} exact {st.get('n_exact_rows')} of {len(rec['sids'])} rows, "
                             f"ambiguous {rep.n_ambiguous}")
            else:
                lines.append(f"oracle, {len(rec['sids'])} rows, ambiguous {rep.n_ambiguous}")
            if need_ties and not fast:
                ties += _ties_across_cut(rec, s_aug, o_aug, viewed, wl)
            parts.append(_flat_frame(rec, dist, s32, kind, kw))
        got = frames[fast]
        if not mixed:
            sub, ids, scores = (np.concatenate(p) for p in zip(*parts))
            np.testing.assert_array_equal(got[target_col].to_numpy(), ds.user_id_map.external_ids[sub] if kind == "u2i"
                                          else ds.item_id_map.external_ids[sub], err_msg=f"{label} fast={fast}: targets")
            np.testing.assert_array_equal(got["item_id"].to_numpy(), ds.item_id_map.external_ids[ids], err_msg=f"{label}: items")
            fs = got["score"].to_numpy()
            assert fs.dtype in (np.float32, np.float64) and (fs.astype(np.float32) == fs).all()
            np.testing.assert_array_equal(fs.astype(np.float32).view(np.int32), scores.view(np.int32), err_msg=f"{label}: scores")
    assert frames[True].equals(frames[False]), f"{label}: fast_recommend True and False differ"
    scale = None
    if dist == "euclidean":
        scale = float((s32.astype(np.float64) ** 2).sum(axis=1).max() + o_aug[:, 0].max())
    n_amb = _same_reco(stock, frames[True], target_col, scale)
    if need_ties:
        assert ties > 0, f"{label}: no row has an exact fp32 tie across its k-th entry"
    return f"{label}: {'; '.join(dict.fromkeys(lines))}; {n_amb} near-tie swaps against stock" + (f"; {ties} rows tied at the cut" if need_ties else "")


def run_case(name, size, base, need_ties=None):
    """Builds the case, ranks every call stock and through `install()` (fast_recommend True and False) with a recording
    `base` ranker, and checks each call.  Returns the summary lines."""
    import rectools_b200
    from rectools_b200 import integration

    model, ds = build(name, size)
    out = []
    for kind, kw in calls(name, ds):
        stock = invoke(model, ds, kind, kw)
        frames, logs = {}, {}
        for fast in (True, False):
            log: tp.List[tp.Dict[str, tp.Any]] = []
            saved = integration.B200ImplicitRanker
            integration.B200ImplicitRanker = recording_ranker(base, log)  # what install() binds, and recommend.py ranks with
            try:
                rectools_b200.install(fast_recommend=fast)
                frames[fast] = invoke(model, ds, kind, kw)
            finally:
                rectools_b200.uninstall()
                integration.B200ImplicitRanker = saved
            logs[fast] = log
        ties = need_ties if need_ties is not None else (name.endswith("dominant") and kind == "u2i" and kw["k"] in (10, 100))
        label = f"{name} {kind} " + ", ".join(f"{a}={'wl' if a == 'items_to_recommend' else v}" for a, v in kw.items()
                                               if a != "targets" and v is not None)
        out.append(check_case(model, ds, kind, kw, stock, frames, logs, label, need_ties=ties))
    return out

