"""numpy definition of ItemKNN ranking (engine path 9, `b200_rank_topk_knn`, `rectools_b200.item_knn`) and the `fit` /
`recommend` of implicit's item-item recommenders that the tests give the repository's `implicit` stub.

The stub (oracle/implicit_stub/implicit/nearest_neighbours.py) carries attributes only; `stub_methods()` adds, for the
length of a `with` block, the two methods `ImplicitItemKNNWrapperModel` calls.  Like the restatement of
`implicit.cpu.topk` in SURVEY section 8c, they restate implicit from recollection, not from its source; the known answers
of the reference's own tests (tests/golden/item_knn_known_answers.json) pin them.

  * `fit(user_items)`: the item-item neighbour matrix S = X^T X of the weighted users x items matrix X (raw counts for
    `ItemItemRecommender`; `normalize(X)` rows for `CosineRecommender`; `normalize(tfidf_weight(X^T)).T` for
    `TFIDFRecommender`; `bm25_weight(X^T, K1, B).T` for `BM25Recommender`), each row cut to its K largest values,
    ties by item id DESCENDING (the reference's TFIDF known answers need it: row 11 of their matrix holds 13 and 17 at
    one value and keeps 17), self-similarity included, as a float64 CSR with ascending ids (`similarity`).  BM25 and
    cosine have no known answer to pin them.
  * `recommend(userid, user_items, N, filter_already_liked_items=True, ...)`: on the user's row of `user_items`, the
    scores s(i) of `knn_scores`, then the top N touched items by (s desc, id asc), as (ids, scores).

u2i (`knn_scores`): row entries (j_e, w_e) in CSR order; item i of the touched set T (the union of the S rows of the
entries) scores (((0 + p_1) + p_2) + ...) over the entries whose S row holds i, p = fl64(S[j_e, i] * float64(w_e)); numpy
rounds the product and then the sum, as the kernel does with __dmul_rn / __dadd_rn.  Zero and negative scores count.
"""
import contextlib

import numpy as np
from scipy import sparse


# ------------------------------------------------------------------------------------------------------------ weighting
def normalize(X):
    X = sparse.coo_matrix(X, dtype=np.float64)
    X.data = X.data / np.sqrt(np.bincount(X.row, X.data**2, minlength=X.shape[0]))[X.row]
    return X


def tfidf_weight(X):
    X = sparse.coo_matrix(X, dtype=np.float64)
    N = float(X.shape[0])
    idf = np.log(N) - np.log1p(np.bincount(X.col, minlength=X.shape[1]))
    X.data = np.sqrt(X.data) * idf[X.col]
    return X


def bm25_weight(X, K1=100, B=0.8):
    X = sparse.coo_matrix(X, dtype=np.float64)
    N = float(X.shape[0])
    idf = np.log(N) - np.log1p(np.bincount(X.col, minlength=X.shape[1]))
    row_sums = np.ravel(X.sum(axis=1))
    length_norm = (1.0 - B) + B * row_sums / row_sums.mean()
    X.data = X.data * (K1 + 1.0) / (K1 * length_norm[X.row] + X.data) * idf[X.col]
    return X


def all_pairs_knn(X, K: int):
    """Rows of S = X^T X (items x items) cut to their K largest values, ties by id descending; float64 CSR."""
    X = sparse.csr_matrix(X, dtype=np.float64)
    full = (X.T @ X).tocsr()
    full.sort_indices()
    indptr, indices, data = [0], [], []
    for i in range(full.shape[0]):
        cols = full.indices[full.indptr[i] : full.indptr[i + 1]]
        vals = full.data[full.indptr[i] : full.indptr[i + 1]]
        keep = np.lexsort((-cols.astype(np.int64), -vals))[:K]
        keep = np.sort(keep)
        indices.append(cols[keep])
        data.append(vals[keep])
        indptr.append(indptr[-1] + len(keep))
    n = full.shape[0]
    cat = lambda parts, dt: np.concatenate(parts).astype(dt) if parts else np.zeros(0, dt)  # noqa: E731
    return sparse.csr_matrix((cat(data, np.float64), cat(indices, np.int32), np.asarray(indptr, np.int64)), shape=(n, n))


def fit_similarity(model, user_items):
    """The `similarity` the stub's `fit` gives `model` for a users x items `user_items`."""
    from implicit.nearest_neighbours import BM25Recommender, CosineRecommender, TFIDFRecommender

    X = sparse.csr_matrix(user_items, dtype=np.float64)
    if isinstance(model, CosineRecommender):
        X = normalize(X.T).T
    elif isinstance(model, TFIDFRecommender):
        X = normalize(tfidf_weight(X.T)).T
    elif isinstance(model, BM25Recommender):
        X = bm25_weight(X.T, model.K1, model.B).T
    return all_pairs_knn(X, model.K)


# ---------------------------------------------------------------------------------------------------------------- u2i
def knn_scores(S, js, ws):
    """(touched ids ascending, their fp64 scores) of one row with entries js / ws (fp32 weights), in entry order."""
    S = sparse.csr_matrix(S)
    n = S.shape[0]
    acc = np.zeros(n, np.float64)
    touched = np.zeros(n, bool)
    for j, w in zip(np.asarray(js), np.asarray(ws, dtype=np.float32)):
        lo, hi = S.indptr[j], S.indptr[j + 1]
        cols = S.indices[lo:hi]
        prod = S.data[lo:hi].astype(np.float64) * np.float64(w)
        acc[cols] = acc[cols] + prod
        touched[cols] = True
    ids = np.flatnonzero(touched)
    return ids, acc[ids]


def top_by_score(ids, scores, n):
    """The first n of (ids, scores) by (score desc, id asc); -0 equals +0."""
    order = np.lexsort((ids, -(scores + 0.0)))[:n]
    return ids[order], scores[order]


def rank_knn_np(S, user_rows, k: int, filter_rows=None, whitelist=None):
    """What `b200_rank_topk_knn` writes: ids int32 [n, k] (-1 padded), scores float64 [n, k] (0 padded), counts int32 [n]."""
    S = sparse.csr_matrix(S)
    U = sparse.csr_matrix(user_rows)
    n = U.shape[0]
    ids_out = np.full((n, k), -1, np.int32)
    sc_out = np.zeros((n, k), np.float64)
    counts = np.zeros(n, np.int32)
    wl = None if whitelist is None else np.asarray(whitelist)
    for r in range(n):
        lo, hi = U.indptr[r], U.indptr[r + 1]
        ids, sc = knn_scores(S, U.indices[lo:hi], U.data[lo:hi])
        keep = np.ones(len(ids), bool)
        if filter_rows is not None:
            F = filter_rows
            keep &= ~np.isin(ids, F.indices[F.indptr[r] : F.indptr[r + 1]])
        if wl is not None:
            keep &= np.isin(ids, wl)
        ids, sc = top_by_score(ids[keep], sc[keep], k)
        counts[r] = len(ids)
        ids_out[r, : len(ids)] = ids
        sc_out[r, : len(ids)] = sc
    return ids_out, sc_out, counts


def recommend_u2i_np(S, user_items, user_ids, k: int, filter_viewed: bool, whitelist=None):
    """`_recommend_u2i`'s triplet under the definition: per user the top min(k, |C_u|) of its candidates."""
    rows = user_items[user_ids]
    f = rows.sorted_indices() if filter_viewed else None
    ids, sc, counts = rank_knn_np(S, rows, max(int(k), 1), f, whitelist)
    mask = np.arange(ids.shape[1])[None, :] < counts[:, None]
    return np.repeat(np.asarray(user_ids), counts), ids[mask].astype(np.int64), sc[mask]


# ---------------------------------------------------------------------------------------------------------------- i2i
def recommend_i2i_np(S, target_ids, k: int, whitelist=None):
    """`_recommend_i2i`'s triplet under the definition: S[target] on the whitelist columns, its top min(k, stored entries)
    by (value desc, id asc)."""
    S = sparse.csr_matrix(S)
    tids, rids, scs = [], [], []
    for t in target_ids:
        lo, hi = S.indptr[t], S.indptr[t + 1]
        cols, vals = S.indices[lo:hi], S.data[lo:hi]
        if whitelist is not None:
            m = np.isin(cols, whitelist)
            cols, vals = cols[m], vals[m]
        ids, sc = top_by_score(cols.astype(np.int64), vals, k)
        tids.append(np.full(len(ids), t))
        rids.append(ids)
        scs.append(sc)
    return np.concatenate(tids), np.concatenate(rids), np.concatenate(scs)


# ---------------------------------------------------------------------------------------------------------------- stub
def _stub_fit(self, user_items, show_progress=True):  # pylint: disable=unused-argument
    self.similarity = fit_similarity(self, user_items)
    return self


def _stub_recommend(self, userid, user_items, N=10, filter_already_liked_items=True, filter_items=None,  # pylint: disable=unused-argument
                    recalculate_user=False, items=None):
    row = sparse.csr_matrix(user_items)
    if row.shape[0] != 1:
        row = row[[userid]]
    ids, sc = knn_scores(self.similarity, row.indices, row.data.astype(np.float32))
    if filter_already_liked_items:
        keep = ~np.isin(ids, row.indices)
        ids, sc = ids[keep], sc[keep]
    if filter_items is not None:
        keep = ~np.isin(ids, filter_items)
        ids, sc = ids[keep], sc[keep]
    ids, sc = top_by_score(ids, sc, int(N))
    return ids.astype(np.int32), sc


@contextlib.contextmanager
def stub_methods():
    """The stub's `ItemItemRecommender` with `fit` and `recommend` for the length of the block."""
    from implicit.nearest_neighbours import ItemItemRecommender

    saved = {name: ItemItemRecommender.__dict__.get(name) for name in ("fit", "recommend")}
    ItemItemRecommender.fit = _stub_fit
    ItemItemRecommender.recommend = _stub_recommend
    try:
        yield
    finally:
        for name, orig in saved.items():
            if orig is None:
                delattr(ItemItemRecommender, name)
            else:
                setattr(ItemItemRecommender, name, orig)
