"""`B200Ranker`: the reference's `Ranker` protocol on top of libb200rank.so.

Mirrors `rectools.models.rank.ImplicitRanker` (rectools/models/rank/rank_implicit.py:34-280) -- same constructor
meaning `(distance, subjects_factors, objects_factors, ...)`, same `rank(subject_ids, k, filter_pairs_csr,
sorted_object_whitelist)` signature, return triplet and error behaviour -- with the native top-k call
(rank_implicit.py:264-272 / :175-182) and the per-user Python post-loop (:120-146) replaced by one C-ABI call plus
vectorised numpy.  There is no CPU fallback: construction fails if the CUDA library or an sm_90 device is missing.
"""
from __future__ import annotations

import ctypes as C
import typing as tp
import weakref
from enum import Enum

import numpy as np
from scipy import sparse

from . import _lib

InternalIds = tp.Sequence[int]
Scores = tp.Union[tp.Sequence[float], np.ndarray]


class Distance(str, Enum):
    """Same members / values as `rectools.models.rank.Distance` (rectools/models/rank/rank.py:25-30)."""

    DOT = "dot"
    COSINE = "cosine"
    EUCLIDEAN = "euclidean"


_TC_MODES = {"auto": _lib.TC_AUTO, "fp16": _lib.TC_FP16, "bf16": _lib.TC_BF16, "off": _lib.TC_OFF}


def _as_distance(distance: tp.Any) -> Distance:
    return Distance(str(getattr(distance, "value", distance)))


def _dense_f32(x: tp.Any) -> np.ndarray:
    """`factors.astype(np.float32)` of the reference (rank_implicit.py:70-71), C-contiguous, torch tensors accepted."""
    if sparse.issparse(x):
        raise TypeError("sparse factors are kept sparse (B200Ranker: CSR subjects), never densified as a whole")
    if hasattr(x, "detach") and hasattr(x, "cpu"):
        x = x.detach().cpu().numpy()
    x = np.asarray(x)
    if x.ndim != 2:
        raise ValueError("factor matrices must be 2-dimensional")
    return np.ascontiguousarray(x, dtype=np.float32)


def _is_cuda_tensor(x: tp.Any) -> bool:
    return hasattr(x, "is_cuda") and bool(getattr(x, "is_cuda")) and hasattr(x, "data_ptr")


def _norms_f32(x: np.ndarray) -> np.ndarray:
    """`_calc_norms(avoid_zeros=True)` (rank_implicit.py:98-105), accumulated in fp64 as the engine does."""
    n = np.sqrt(np.einsum("ij,ij->i", x, x, dtype=np.float64)).astype(np.float32)
    n[n == 0] = 1e-10
    return n


def _device_norms(x: tp.Any) -> np.ndarray:
    """`_norms_f32` of a CUDA tensor's rows (any float type, widened exactly to fp64), as a host fp32 array."""
    import torch

    norms = torch.linalg.vector_norm(x.double(), dim=1).float()
    norms[norms == 0] = 1e-10
    return norms.cpu().numpy()


def check_whitelist(whitelist: np.ndarray, n_objects: int) -> None:
    """`sorted_object_whitelist` (rank.py:39): object ids in range, strictly ascending -- the kernels merge a row's viewed ids
    against the whitelist positions in ascending order, so an unsorted whitelist would let viewed objects through."""
    if len(whitelist) == 0:
        return
    if whitelist[0] < 0 or whitelist[-1] >= n_objects or whitelist.min() < 0 or whitelist.max() >= n_objects:
        raise IndexError("whitelist id out of range")
    if len(whitelist) > 1 and not bool((np.diff(whitelist) > 0).all()):
        raise ValueError("`sorted_object_whitelist` must be sorted ascending without duplicates")


def object_storage_dtype(distance: tp.Any, dtype: tp.Any, keep_16bit: bool) -> int:
    """Element type (`_lib.DT_*`) the engine keeps the object factors in.  fp16 / bf16 factors stay at 16 bits with
    `keep_16bit` (B200_F_OBJECTS_16BIT: results are bit for bit those of the widened engine, at half the master copy's
    HBM), except for EUCLIDEAN: its augmented objects carry a squared-norm column that is no 16-bit value.  Everything
    else is an fp32 master copy.  `dtype`: a numpy or torch dtype, or its name."""
    if isinstance(dtype, str) or str(dtype).startswith("torch."):
        name = str(dtype).replace("torch.", "")
    else:
        name = np.dtype(dtype).name
    if not keep_16bit or _as_distance(distance) == Distance.EUCLIDEAN:
        return _lib.DT_F32
    return {"float16": _lib.DT_F16, "bfloat16": _lib.DT_BF16}.get(name, _lib.DT_F32)


def prepare_factors(
    distance: Distance, subjects: np.ndarray, objects: np.ndarray
) -> tp.Tuple[np.ndarray, np.ndarray, tp.Optional[np.ndarray], tp.Optional[np.ndarray]]:
    """Host prologue of `ImplicitRanker`: COSINE subject norms (rank_implicit.py:76-77) or the EUCLIDEAN -> DOT
    augmentation (rank_implicit.py:79-81, :242-246).  Returns (subjects', objects', subjects_norms, subjects_dots)."""
    norms = dots = None
    if distance == Distance.COSINE:
        norms = _norms_f32(subjects)
    elif distance == Distance.EUCLIDEAN:
        dots = (subjects**2).sum(axis=1)
        subjects = np.hstack((-np.ones((subjects.shape[0], 1)), 2 * subjects)).astype(np.float32)
        objects = np.hstack(((objects**2).sum(axis=1).reshape(-1, 1), objects)).astype(np.float32)
    return subjects, objects, norms, dots


def _host_objects(objects: np.ndarray, objects_dtype: int) -> np.ndarray:
    """A host object matrix as the engine reads it: C-contiguous fp32, or fp16 for `objects_dtype` DT_F16."""
    if objects_dtype == _lib.DT_BF16:
        raise TypeError("bf16 object factors must be a CUDA tensor (numpy has no bfloat16)")
    return np.ascontiguousarray(objects, dtype=np.float16 if objects_dtype == _lib.DT_F16 else np.float32)


def _create_flags(on_device: bool, keep_16bit: bool) -> int:
    return (_lib.F_OBJECTS_ON_DEVICE if on_device else 0) | (_lib.F_OBJECTS_16BIT if keep_16bit else 0)


class Engine:
    """Owner of one `b200_rank_engine*` (resident object factors on one GPU).  `keep_16bit`: fp16 / bf16 objects stay in
    their own type (B200_F_OBJECTS_16BIT, no fp32 master copy); a device matrix is then read in place and must stay alive
    and unchanged until `close()`.  Without it, 16-bit objects must be device pointers and are widened to fp32."""

    def __init__(
        self,
        objects: np.ndarray,
        cosine: bool,
        device: int = 0,
        tc_mode: str = "auto",
        id_offset: int = 0,
        objects_device_ptr: tp.Optional[int] = None,
        shape: tp.Optional[tp.Tuple[int, int]] = None,
        objects_dtype: int = _lib.DT_F32,
        keep_16bit: bool = False,
    ) -> None:
        self._lib = _lib.load()
        self._h = C.c_void_p()
        if objects_device_ptr is not None:
            assert shape is not None
            n, d = shape
            ptr, flags = objects_device_ptr, _create_flags(True, keep_16bit)
            self._keep = None
        else:
            objects = _host_objects(objects, objects_dtype)
            n, d = objects.shape
            ptr, flags = objects.ctypes.data, _create_flags(False, keep_16bit)
            self._keep = objects
        _lib.check(
            self._lib.b200_rank_create_ex(
                C.byref(self._h), ptr, objects_dtype, n, d, _lib.DIST_COSINE if cosine else _lib.DIST_DOT, device,
                _TC_MODES[tc_mode], flags,
            )
        )
        self._keep = None  # the engine copied the host matrix
        self.n_objects, self.d, self.device = int(n), int(d), int(device)
        if id_offset:
            _lib.check(self._lib.b200_rank_set_id_offset(self._h, int(id_offset)))
        self.id_offset = int(id_offset)
        self.last_stats: tp.Dict[str, tp.Any] = {}

    def close(self) -> None:
        if getattr(self, "_h", None) is not None and self._h.value:
            self._lib.b200_rank_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self) -> None:  # pragma: no cover
        try:
            self.close()
        except Exception:  # pylint: disable=broad-except
            pass

    def info(self) -> tp.Dict[str, tp.Any]:
        inf = _lib.Info()
        _lib.check(self._lib.b200_rank_get_info(self._h, C.byref(inf)))
        out = {name: getattr(inf, name) for name, _ in inf._fields_}  # pylint: disable=protected-access
        out["device_name"] = inf.device_name.decode()
        return out

    def set_subjects(self, subjects: np.ndarray, key: tp.Optional[tp.Hashable] = None, owner: tp.Any = None) -> None:
        """Upload the resident subject factors.  `key` (optional identity of the matrix): a repeated call with the key of the
        matrix that is already resident is a no-op -- `VectorModel` builds a new ranker per `recommend()` call (vector.py:66).
        `owner`: the ranker whose subjects are resident now (several rankers may share one cached engine)."""
        subjects = np.ascontiguousarray(subjects, dtype=np.float32)
        if subjects.shape[1] != self.d:
            raise ValueError("subject and object factors must have the same number of columns")
        self._subjects_owner = weakref.ref(owner) if owner is not None else None
        if key is not None and key == getattr(self, "_subjects_key", None):
            return
        self._set_subjects(subjects.ctypes.data, subjects.shape[0], 0)
        self._subjects_key = key

    @property
    def subjects_owner(self) -> tp.Any:
        """The ranker whose subject factors are resident (None: nobody's / collected).  A weak reference: a cached engine
        must not keep its last ranker and that ranker's matrices alive."""
        ref = getattr(self, "_subjects_owner", None)
        return ref() if ref is not None else None

    def set_subjects_device(self, ptr: int, n_subjects: int) -> None:
        self._set_subjects(ptr, n_subjects, 1)

    def _set_subjects(self, ptr: int, n_subjects: int, on_device: int) -> None:
        _lib.check(self._lib.b200_rank_set_subjects(self._h, ptr, n_subjects, on_device))
        self.n_resident_subjects = int(n_subjects)

    def peer_export(self, max_rows: int) -> bytes:
        """Allocate this engine's published-threshold array (threshold sharing between the ranks of an item-sharded
        catalogue) and return its 64-byte CUDA IPC handle."""
        buf = C.create_string_buffer(64)
        _lib.check(self._lib.b200_rank_peer_export(self._h, int(max_rows), buf))
        return buf.raw

    def peer_import(self, handles: tp.Sequence[bytes], self_index: int) -> None:
        """Open the published-threshold arrays of all ranks (`handles` in rank order, this engine's own included)."""
        blob = b"".join(handles)
        assert len(blob) == 64 * len(handles)
        _lib.check(self._lib.b200_rank_peer_import(self._h, len(handles), int(self_index), blob))

    def peer_attach(self, pub: tp.Any, peers: tp.Sequence[tp.Any]) -> None:
        """Test interface: share thresholds inside one process through caller-owned device arrays (torch int64 / uint64
        tensors of `max_rows` words on the engine's device): `pub` is published to, `peers` are read.  The caller keeps the
        tensors alive for as long as the engine ranks with B200_Q_SHARED_THRESHOLDS."""
        ptrs = (C.c_void_p * max(1, len(peers)))(*[t.data_ptr() for t in peers])
        _lib.check(self._lib.b200_rank_peer_attach(self._h, int(pub.numel()), pub.data_ptr(), len(peers), ptrs))

    def candidate_snapshot(self) -> tp.Optional[tp.Dict[str, tp.Any]]:
        """Test interface: the tensor-core pass the last call captured with B200_TC_SNAPSHOT=n set (None: nothing was
        captured).  The metadata of `b200_rank_snapshot` plus numpy arrays: `cand_scores` / `cand_ids`
        [n_lists, rows_pad, cand_stride], `cand_counts` / `cand_thr` [n_lists, rows_pad], `row_exp` [n_sel], `rows` [n_sel]
        (the call's row of each batch row of the pass), `fb_rows` [n_fb] (rows the pass's re-score sent to the fallback)."""
        meta = _lib.Snapshot()
        null = [None] * 7
        _lib.check(self._lib.b200_rank_get_snapshot(self._h, C.byref(meta), *null))
        if not meta.valid:
            return None
        n_lr = meta.n_lists * meta.rows_pad
        out: tp.Dict[str, tp.Any] = {name: getattr(meta, name) for name, _ in meta._fields_}  # pylint: disable=protected-access
        arrays = {
            "cand_scores": np.empty(n_lr * meta.cand_stride, np.float32),
            "cand_ids": np.empty(n_lr * meta.cand_stride, np.int32),
            "cand_counts": np.empty(n_lr, np.int32),
            "cand_thr": np.empty(n_lr, np.float32),
            "row_exp": np.empty(meta.rows_pad, np.int32),
            "rows": np.empty(meta.n_sel, np.int32),
            "fb_rows": np.empty(meta.n_fb, np.int32),
        }
        _lib.check(self._lib.b200_rank_get_snapshot(self._h, C.byref(meta), *[a.ctypes.data for a in arrays.values()]))
        lists = (meta.n_lists, meta.rows_pad)
        arrays["cand_scores"] = arrays["cand_scores"].reshape(*lists, meta.cand_stride)
        arrays["cand_ids"] = arrays["cand_ids"].reshape(*lists, meta.cand_stride)
        arrays["cand_counts"] = arrays["cand_counts"].reshape(lists)
        arrays["cand_thr"] = arrays["cand_thr"].reshape(lists)
        arrays["row_exp"] = arrays["row_exp"][: meta.n_sel]
        out.update(arrays)
        return out

    def topk_raw(self, q: _lib.Query) -> tp.Dict[str, tp.Any]:
        st = _lib.Stats()
        _lib.check(self._lib.b200_rank_topk(self._h, C.byref(q), C.byref(st)))
        self.last_stats = st.as_dict()
        return self.last_stats

    def topk_ptrs(
        self,
        n_rows: int,
        k: int,
        out_ids: int,
        out_scores: int,
        out_counts: int,
        flags: int,
        subjects: int = 0,
        subject_ids: int = 0,
        n_subjects_total: int = 0,
        indptr: int = 0,
        indices: int = 0,
        whitelist: int = 0,
        n_whitelist: int = 0,
        stream: int = 0,
        out_bounds: int = 0,
        peer_epoch: int = 0,
        subject_dtype: int = _lib.DT_F32,
        object_rows: int = 0,
    ) -> tp.Dict[str, tp.Any]:
        """Raw-pointer call (host or device addresses according to `flags`); returns the call statistics."""
        q = _lib.Query()
        q.object_rows = object_rows or None
        q.out_bounds, q.peer_epoch, q.subject_dtype = out_bounds or None, int(peer_epoch), int(subject_dtype)
        q.subjects, q.subject_ids, q.n_rows, q.n_subjects_total = subjects or None, subject_ids or None, n_rows, n_subjects_total
        q.csr_indptr, q.csr_indices = indptr or None, indices or None
        q.whitelist, q.n_whitelist = whitelist or None, n_whitelist
        q.k, q.flags = int(k), int(flags)
        q.out_ids, q.out_scores, q.out_counts = out_ids, out_scores, out_counts
        q.stream = stream or None
        return self.topk_raw(q)

    def topk(
        self,
        k: int,
        subjects: tp.Optional[np.ndarray] = None,
        subject_ids: tp.Optional[np.ndarray] = None,
        indptr: tp.Optional[np.ndarray] = None,
        indices: tp.Optional[np.ndarray] = None,
        whitelist: tp.Optional[np.ndarray] = None,
        flags: int = 0,
        out: tp.Optional[tp.Tuple[np.ndarray, np.ndarray, np.ndarray]] = None,
        sparse_subjects: tp.Optional[sparse.csr_matrix] = None,
        object_rows: tp.Optional[np.ndarray] = None,
    ) -> tp.Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """Host-buffer call: returns padded `(ids [n,k_out] int32, scores [n,k_out] fp32, counts [n] int32)`.
        `sparse_subjects`: the batch rows as a CSR matrix [n_rows, d] (EASE), instead of `subjects` / `subject_ids`.
        `object_rows`: batch row r is the engine's own stored object row object_rows[r], used as the score row (EASE
        item-to-item; needs d == n_objects), instead of any subjects."""
        q, keep, n_rows, n_pos = self._host_query(k, subjects, subject_ids, indptr, indices, whitelist, flags, sparse_subjects, object_rows)
        k_out = max(0, min(int(k), n_pos))
        ids, scores, counts = self._host_outputs(q, n_rows, k_out, out)
        self.topk_raw(q)
        del keep
        return ids, scores, counts

    def topk_candidates(
        self,
        k: int,
        cand_indptr: np.ndarray,
        cand_indices: np.ndarray,
        subjects: tp.Optional[np.ndarray] = None,
        subject_ids: tp.Optional[np.ndarray] = None,
        indptr: tp.Optional[np.ndarray] = None,
        indices: tp.Optional[np.ndarray] = None,
        flags: int = 0,
        out: tp.Optional[tp.Tuple[np.ndarray, np.ndarray, np.ndarray]] = None,
        whitelist: tp.Optional[np.ndarray] = None,
        sparse_subjects: tp.Optional[sparse.csr_matrix] = None,
        object_rows: tp.Optional[np.ndarray] = None,
    ) -> tp.Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """Host-buffer call of `b200_rank_topk_candidates` (path 5): row r is ranked against its own object ids
        `cand_indices[cand_indptr[r]:cand_indptr[r+1]]` (strictly ascending within a row), minus its filter row.  Returns padded
        `(ids [n,k_out] int32, scores [n,k_out] fp32, counts [n] int32)` with k_out = min(k, n_objects).  `whitelist`,
        `sparse_subjects` and `object_rows` are passed through for the engine to refuse."""
        q, keep, n_rows, _ = self._host_query(k, subjects, subject_ids, indptr, indices, whitelist, flags, sparse_subjects, object_rows)
        cand_indptr = np.ascontiguousarray(cand_indptr, dtype=np.int64).reshape(-1)
        cand_indices = np.ascontiguousarray(cand_indices, dtype=np.int32).reshape(-1)
        if len(cand_indptr) != n_rows + 1:
            raise ValueError("`cand_indptr` must have `n_rows + 1` entries")
        k_out = max(0, min(int(k), self.n_objects))
        ids, scores, counts = self._host_outputs(q, n_rows, k_out, out)
        st = _lib.Stats()
        _lib.check(self._lib.b200_rank_topk_candidates(self._h, C.byref(q), cand_indptr.ctypes.data, cand_indices.ctypes.data, C.byref(st)))
        self.last_stats = st.as_dict()
        del keep
        return ids, scores, counts

    def topk_candidates_device(
        self,
        k: int,
        cand_indptr: tp.Any,
        cand_indices: tp.Any,
        subjects: tp.Any = None,
        subject_ids: tp.Any = None,
        indptr: tp.Any = None,
        indices: tp.Any = None,
        out: tp.Optional[tp.Tuple[tp.Any, tp.Any, tp.Any]] = None,
        stream: tp.Any = None,
    ) -> tp.Tuple[tp.Any, tp.Any, tp.Any]:
        """Device-memory call of `b200_rank_topk_candidates_device` (path 5): row r is ranked against the distinct ids of
        `cand_indices[cand_indptr[r]:cand_indptr[r+1]]` that are objects of the engine (any order, repeats and out-of-range
        ids such as -1 holes allowed), minus its filter row.  Every input is a CUDA tensor on the engine's device:
        `cand_indptr` int64 [n + 1] (any base), `cand_indices` int32, `subjects` fp32 / fp16 / bf16 in batch order or fp32
        with `subject_ids` (int64), else `subject_ids` over the resident subjects, and the filter CSR `indptr` / `indices`.
        Returns `(ids [n,k_out] int32, scores [n,k_out] fp32, counts [n] int32)`, k_out = min(k, n_objects): new CUDA
        tensors, or `out` filled in place (CUDA tensors, or numpy arrays for host outputs).  The call is ordered after
        `stream` (default: the current torch stream of the device), which waits for device outputs."""
        import torch

        dev = torch.device("cuda", self.device)

        def device_tensor(name: str, t: tp.Any, dtypes: tp.Tuple[tp.Any, ...]) -> tp.Any:
            if not _is_cuda_tensor(t) or t.device != dev:
                raise TypeError(f"`{name}` must be a CUDA tensor on {dev}")
            if t.dtype not in dtypes:
                raise TypeError(f"`{name}` must be of dtype {' / '.join(str(d) for d in dtypes)}, not {t.dtype}")
            return t.contiguous()

        keep = []
        cand_indptr = device_tensor("cand_indptr", cand_indptr, (torch.int64,)).reshape(-1)
        cand_indices = device_tensor("cand_indices", cand_indices, (torch.int32,)).reshape(-1)
        n_rows = len(cand_indptr) - 1
        if n_rows < 0:
            raise ValueError("`cand_indptr` must have `n_rows + 1` entries")
        keep += [cand_indptr, cand_indices]
        q = _lib.Query()
        q.flags = _lib.Q_INPUTS_ON_DEVICE
        if subjects is not None:
            subjects = device_tensor("subjects", subjects, (torch.float32, torch.float16, torch.bfloat16))
            if subjects.ndim != 2 or subjects.shape[1] != self.d:
                raise ValueError("subject and object factors must have the same number of columns")
            q.subjects = subjects.data_ptr()
            q.subject_dtype = {torch.float32: _lib.DT_F32, torch.float16: _lib.DT_F16, torch.bfloat16: _lib.DT_BF16}[subjects.dtype]
            keep.append(subjects)
        if subject_ids is not None:
            subject_ids = device_tensor("subject_ids", subject_ids, (torch.int64,)).reshape(-1)
            if len(subject_ids) != n_rows:
                raise ValueError("`subject_ids` must have one entry per candidate row")
            q.subject_ids = subject_ids.data_ptr()
            q.n_subjects_total = 0 if subjects is None else subjects.shape[0]
            keep.append(subject_ids)
        elif subjects is None:
            raise ValueError("either subjects or subject_ids is required")
        elif subjects.shape[0] != n_rows:
            raise ValueError("`subjects` must have one row per candidate row")
        q.n_rows = n_rows
        if indptr is not None:
            indptr = device_tensor("indptr", indptr, (torch.int64,)).reshape(-1)
            if len(indptr) != n_rows + 1:
                raise ValueError("Number of rows in `filter_pairs_csr` must be equal to `len(sublect_ids)`")
            indices = device_tensor("indices", indices if indices is not None else torch.empty(0, dtype=torch.int32, device=dev),
                                    (torch.int32,)).reshape(-1)
            q.csr_indptr, q.csr_indices = indptr.data_ptr(), indices.data_ptr()
            keep += [indptr, indices]
        q.k = int(k)
        k_out = max(0, min(int(k), self.n_objects))
        if out is None:
            out = (
                torch.empty((n_rows, k_out), dtype=torch.int32, device=dev),
                torch.empty((n_rows, k_out), dtype=torch.float32, device=dev),
                torch.zeros(n_rows, dtype=torch.int32, device=dev),
            )
        if check_candidate_outputs(out, n_rows, k_out, dev):
            q.flags |= _lib.Q_OUTPUTS_ON_DEVICE
            q.out_ids, q.out_scores, q.out_counts = (a.data_ptr() for a in out)
        else:
            self._host_outputs(q, n_rows, k_out, out)
        # what the engine takes on trust from device arrays, checked here in one device -> host read: the lists and the
        # filter stay inside their index arrays, the subject ids inside their matrix
        if n_rows > 0:
            n_sub = subjects.shape[0] if subjects is not None else getattr(self, "n_resident_subjects", None)
            bad = [cand_indptr[-1] > len(cand_indices)]
            if subject_ids is not None and n_sub is not None:
                bad.append(((subject_ids < 0) | (subject_ids >= n_sub)).any())
            if indptr is not None:
                bad.append((indptr[0] < 0) | (indptr[1:] < indptr[:-1]).any() | (indptr[-1] > len(indices)))
            bad = torch.stack(bad).cpu().tolist()
            if bad[0]:
                raise ValueError("`cand_indptr[-1]` exceeds the length of `cand_indices`")
            if subject_ids is not None and n_sub is not None and bad[1]:
                raise IndexError("subject id out of range")
            if indptr is not None and bad[-1]:
                raise ValueError("the filter's `indptr` must be non-negative, monotone and within `indices`")
        q.stream = stream if isinstance(stream, int) else (stream or torch.cuda.current_stream(dev)).cuda_stream
        st = _lib.Stats()
        _lib.check(self._lib.b200_rank_topk_candidates_device(self._h, C.byref(q), cand_indptr.data_ptr(), cand_indices.data_ptr(), C.byref(st)))
        self.last_stats = st.as_dict()
        del keep
        return tuple(out)

    @staticmethod
    def _host_outputs(
        q: _lib.Query, n_rows: int, k_out: int, out: tp.Optional[tp.Tuple[np.ndarray, np.ndarray, np.ndarray]]
    ) -> tp.Tuple[np.ndarray, np.ndarray, np.ndarray]:
        if out is None:
            ids = np.empty((n_rows, k_out), dtype=np.int32)
            scores = np.empty((n_rows, k_out), dtype=np.float32)
            counts = np.zeros(n_rows, dtype=np.int32)
        else:
            ids, scores, counts = out
        q.out_ids, q.out_scores, q.out_counts = ids.ctypes.data, scores.ctypes.data, counts.ctypes.data
        return ids, scores, counts

    def _host_query(
        self,
        k: int,
        subjects: tp.Optional[np.ndarray],
        subject_ids: tp.Optional[np.ndarray],
        indptr: tp.Optional[np.ndarray],
        indices: tp.Optional[np.ndarray],
        whitelist: tp.Optional[np.ndarray],
        flags: int,
        sparse_subjects: tp.Optional[sparse.csr_matrix],
        object_rows: tp.Optional[np.ndarray],
    ) -> tp.Tuple[_lib.Query, tp.List[np.ndarray], int, int]:
        """The query of a host-buffer call without its outputs: `(query, arrays it points into, n_rows, n_pos)`."""
        q = _lib.Query()
        keep = []
        if object_rows is not None:
            if subjects is not None or subject_ids is not None or sparse_subjects is not None:
                raise ValueError("object_rows excludes subjects / subject_ids / sparse_subjects")
            object_rows = np.ascontiguousarray(object_rows, dtype=np.int64).reshape(-1)
            q.object_rows = object_rows.ctypes.data
            keep.append(object_rows)
        if sparse_subjects is not None:
            if subjects is not None or subject_ids is not None:
                raise ValueError("sparse_subjects excludes subjects / subject_ids")
            if sparse_subjects.shape[1] != self.d:
                raise ValueError("subject and object factors must have the same number of columns")
            sp_indptr = np.ascontiguousarray(sparse_subjects.indptr, dtype=np.int64)
            sp_indices = np.ascontiguousarray(sparse_subjects.indices, dtype=np.int32)
            sp_data = np.ascontiguousarray(sparse_subjects.data, dtype=np.float32)
            q.sub_indptr, q.sub_indices, q.sub_data = sp_indptr.ctypes.data, sp_indices.ctypes.data, sp_data.ctypes.data
            keep += [sp_indptr, sp_indices, sp_data]
        if subjects is not None:
            subjects = np.ascontiguousarray(subjects, dtype=np.float32)
            if subjects.ndim != 2 or subjects.shape[1] != self.d:
                raise ValueError("subject and object factors must have the same number of columns")
            q.subjects = subjects.ctypes.data
            keep.append(subjects)
        if subject_ids is not None:
            subject_ids = np.ascontiguousarray(subject_ids, dtype=np.int64)
            q.subject_ids = subject_ids.ctypes.data
            keep.append(subject_ids)
            n_rows = len(subject_ids)
            q.n_subjects_total = 0 if subjects is None else subjects.shape[0]
        elif sparse_subjects is not None:
            n_rows = sparse_subjects.shape[0]
        elif object_rows is not None:
            n_rows = len(object_rows)
        else:
            if subjects is None:
                raise ValueError("either subjects or subject_ids is required")
            n_rows = subjects.shape[0]
        q.n_rows = n_rows
        if indptr is not None:
            indptr = np.ascontiguousarray(indptr, dtype=np.int64)
            if len(indptr) != n_rows + 1:
                raise ValueError("Number of rows in `filter_pairs_csr` must be equal to `len(sublect_ids)`")
            indices = np.ascontiguousarray(indices if indices is not None else np.empty(0), dtype=np.int32)
            q.csr_indptr = indptr.ctypes.data
            q.csr_indices = indices.ctypes.data
            keep += [indptr, indices]
        n_pos = self.n_objects
        if whitelist is not None:
            whitelist = np.ascontiguousarray(whitelist, dtype=np.int32)
            q.whitelist = whitelist.ctypes.data
            q.n_whitelist = len(whitelist)
            n_pos = len(whitelist)
            keep.append(whitelist)
        q.k = int(k)
        q.flags = int(flags)
        return q, keep, n_rows, n_pos


class EngineGroup(Engine):
    """Owner of one `b200_rank_group*`: an engine per entry of `devices` (duplicates: several engines on one device), each
    holding the whole catalogue, that rank the row slices of every call.  Results are bit for bit those of one `Engine`.
    `devices[0]` is the home device: device pointers (objects, subjects, inputs and outputs of `topk_ptrs`) live there.
    `keep_16bit` goes to every member (members on other devices read a 16-bit peer copy).  Threshold sharing, snapshots
    and id offsets are engine-only."""

    def __init__(
        self,
        objects: tp.Optional[np.ndarray],
        cosine: bool,
        devices: tp.Sequence[int],
        tc_mode: str = "auto",
        objects_device_ptr: tp.Optional[int] = None,
        shape: tp.Optional[tp.Tuple[int, int]] = None,
        objects_dtype: int = _lib.DT_F32,
        keep_16bit: bool = False,
    ) -> None:
        self._lib = _lib.load()
        self._h = C.c_void_p()
        self.devices = tuple(int(d) for d in devices)
        if not self.devices:
            raise ValueError("an engine group needs at least one device")
        if objects_device_ptr is not None:
            assert shape is not None
            n, d = shape
            ptr, flags = objects_device_ptr, _create_flags(True, keep_16bit)
        else:
            objects = _host_objects(objects, objects_dtype)
            n, d = objects.shape
            ptr, flags = objects.ctypes.data, _create_flags(False, keep_16bit)
        devs = (C.c_int32 * len(self.devices))(*self.devices)
        _lib.check(
            self._lib.b200_rank_group_create_ex(
                C.byref(self._h), ptr, objects_dtype, n, d, _lib.DIST_COSINE if cosine else _lib.DIST_DOT, devs,
                len(self.devices), _TC_MODES[tc_mode], flags,
            )
        )
        self.n_objects, self.d, self.device = int(n), int(d), self.devices[0]
        self.id_offset = 0
        self.last_stats: tp.Dict[str, tp.Any] = {}
        self.last_member_stats: tp.List[tp.Dict[str, tp.Any]] = []

    def close(self) -> None:
        if getattr(self, "_h", None) is not None and self._h.value:
            self._lib.b200_rank_group_destroy(self._h)
            self._h = C.c_void_p()

    def info(self) -> tp.Dict[str, tp.Any]:
        """Member 0's engine info, `hbm_bytes` of the whole group, and `members`: every member's engine info."""
        infos = (_lib.Info * len(self.devices))()
        total = C.c_int64()
        _lib.check(self._lib.b200_rank_group_get_info(self._h, infos, C.byref(total)))
        members = []
        for inf in infos:
            m = {name: getattr(inf, name) for name, _ in inf._fields_}  # pylint: disable=protected-access
            m["device_name"] = inf.device_name.decode()
            members.append(m)
        return {**members[0], "hbm_bytes": int(total.value), "members": members}

    def _set_subjects(self, ptr: int, n_subjects: int, on_device: int) -> None:
        _lib.check(self._lib.b200_rank_group_set_subjects(self._h, ptr, n_subjects, on_device))

    def topk_raw(self, q: _lib.Query) -> tp.Dict[str, tp.Any]:
        """`last_stats`: the group's totals (counters summed, times the maximum over members); `last_member_stats`: each
        member's own."""
        st = _lib.Stats()
        per = (_lib.Stats * len(self.devices))()
        _lib.check(self._lib.b200_rank_group_topk(self._h, C.byref(q), C.byref(st), per))
        self.last_stats = st.as_dict()
        self.last_member_stats = [p.as_dict() for p in per]
        return self.last_stats

    def peer_export(self, max_rows: int) -> bytes:
        raise NotImplementedError("threshold sharing is for item-sharded engines (ShardedB200Ranker), not engine groups")

    def peer_import(self, handles: tp.Sequence[bytes], self_index: int) -> None:
        raise NotImplementedError("threshold sharing is for item-sharded engines (ShardedB200Ranker), not engine groups")

    def peer_attach(self, pub: tp.Any, peers: tp.Sequence[tp.Any]) -> None:
        raise NotImplementedError("threshold sharing is for item-sharded engines (ShardedB200Ranker), not engine groups")

    def candidate_snapshot(self) -> tp.Optional[tp.Dict[str, tp.Any]]:
        raise NotImplementedError("snapshots are taken by single engines")

    def topk_candidates(self, *args: tp.Any, **kwargs: tp.Any) -> tp.Tuple[np.ndarray, np.ndarray, np.ndarray]:
        raise NotImplementedError(
            "candidate sets are ranked by single engines: an engine group has no candidate-set export yet (use one device)"
        )

    def topk_candidates_device(self, *args: tp.Any, **kwargs: tp.Any) -> tp.Tuple[tp.Any, tp.Any, tp.Any]:
        raise NotImplementedError(
            "candidate sets are ranked by single engines: an engine group has no candidate-set export yet (use one device)"
        )


Devices = tp.Union[int, str, tp.Sequence[int]]


def parse_devices(device: tp.Any) -> tp.Union[int, tp.Tuple[int, ...]]:
    """`device` of `B200Ranker` / `install()`: an int is one engine on that device (returned unchanged); a sequence of
    ints is an engine group over those devices (duplicates allowed), returned as a tuple; "all" is every visible device."""
    if isinstance(device, (bool, np.bool_)):
        raise TypeError(f"device must be an int, a sequence of ints or 'all', not {device!r}")
    if isinstance(device, (int, np.integer)):
        if device < 0:
            raise ValueError(f"device {device} is negative")
        return int(device)
    if isinstance(device, str):
        if device != "all":
            raise ValueError(f"device must be an int, a sequence of ints or 'all', not {device!r}")
        import torch

        n = torch.cuda.device_count()
        if n == 0:
            raise _lib.B200RankError("device='all': no CUDA device available (the engine has no CPU fallback)")
        return tuple(range(n))
    try:
        devices = tuple(device)
    except TypeError:
        raise TypeError(f"device must be an int, a sequence of ints or 'all', not {device!r}") from None
    if not devices:
        raise ValueError("device: an empty sequence of devices")
    for d in devices:
        if isinstance(d, (bool, np.bool_)) or not isinstance(d, (int, np.integer)):
            raise TypeError(f"device: {d!r} is not a device ordinal")
        if d < 0:
            raise ValueError(f"device {d} is negative")
    return tuple(int(d) for d in devices)


def new_engine(
    objects: tp.Optional[np.ndarray], cosine: bool, device: tp.Any, tc_mode: str = "auto", keep_16bit: bool = False, **kw: tp.Any
) -> Engine:
    """An `Engine` for an int device, an `EngineGroup` for a sequence of devices or "all" (`parse_devices`).
    `keep_16bit`: fp16 / bf16 objects stay at 16 bits (B200_F_OBJECTS_16BIT); no effect on fp32 objects."""
    dev = parse_devices(device)
    if isinstance(dev, int):
        return Engine(objects, cosine=cosine, device=dev, tc_mode=tc_mode, keep_16bit=keep_16bit, **kw)
    return EngineGroup(objects, cosine=cosine, devices=dev, tc_mode=tc_mode, keep_16bit=keep_16bit, **kw)


def rank_object_rows_padded(
    engine: Engine,
    target_ids: InternalIds,
    k: tp.Optional[int] = None,
    filter_pairs_csr: tp.Optional[sparse.csr_matrix] = None,
    sorted_object_whitelist: tp.Optional[np.ndarray] = None,
) -> tp.Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """Rank the engine's stored object rows as score rows: target t scores object j with objects[t, j] (an EASE weight
    matrix held as the objects of its u2i engine; d == n_objects).  `(target_ids, ids [n,k], scores [n,k], counts [n])`
    as `B200Ranker.rank_padded` returns them; k = None ranks every position.  Scores are the stored fp32 values, ordered
    by (score desc, id asc); -inf and NaN are never returned, filtered objects neither."""
    target_ids = np.asarray(target_ids, dtype=np.int64).reshape(-1)
    if filter_pairs_csr is not None and filter_pairs_csr.shape[0] != len(target_ids):
        raise ValueError("Number of rows in `filter_pairs_csr` must be equal to `len(target_ids)`")
    if len(target_ids) and (target_ids.min() < 0 or target_ids.max() >= engine.n_objects):
        raise IndexError("target id out of range")
    whitelist = None
    n_pos = engine.n_objects
    if sorted_object_whitelist is not None:
        whitelist = np.asarray(sorted_object_whitelist, dtype=np.int64).reshape(-1)
        check_whitelist(whitelist, engine.n_objects)
        n_pos = len(whitelist)
    if k is None:
        k = n_pos
    if k <= 0:
        raise ValueError("`k` must be positive")
    indptr = indices = None
    if filter_pairs_csr is not None:
        csr = filter_pairs_csr if sparse.isspmatrix_csr(filter_pairs_csr) else sparse.csr_matrix(filter_pairs_csr)
        if not csr.has_sorted_indices:
            csr = csr.sorted_indices()
        indptr, indices = csr.indptr, csr.indices
    if n_pos == 0 or len(target_ids) == 0:
        z = np.empty((len(target_ids), 0))
        return target_ids, z.astype(np.int32), z.astype(np.float32), np.zeros(len(target_ids), np.int32)
    ids, scores, counts = engine.topk(k, object_rows=target_ids, indptr=indptr, indices=indices, whitelist=whitelist)
    return target_ids, ids, scores, counts


def check_candidate_outputs(out: tp.Sequence[tp.Any], n_rows: int, k_out: int, dev: tp.Any) -> bool:
    """The `out` triplet of `Engine.topk_candidates_device`: `(ids int32 [n_rows, k_out], scores fp32 [n_rows, k_out],
    counts int32 [n_rows])`, all numpy arrays (host outputs: False) or all contiguous CUDA tensors on `dev` (True).  A
    wrong type, dtype or shape raises before the engine could write past the caller's buffers."""
    if len(out) != 3:
        raise ValueError("`out` must be (ids, scores, counts)")
    shapes = ((n_rows, k_out), (n_rows, k_out), (n_rows,))
    for name, a, shape, dtype in zip(("ids", "scores", "counts"), out, shapes, ("int32", "float32", "int32")):
        if not (isinstance(a, np.ndarray) or hasattr(a, "data_ptr")):
            raise TypeError(f"`out` {name}: a numpy array or a CUDA tensor, not {type(a).__name__}")
        if str(a.dtype).replace("torch.", "") != dtype:
            raise TypeError(f"`out` {name} must be {dtype}, not {a.dtype}")
        if tuple(a.shape) != shape:
            raise ValueError(f"`out` {name} must have shape {shape}, not {tuple(a.shape)}")
    if all(isinstance(a, np.ndarray) for a in out):
        if not all(a.flags.c_contiguous for a in out):
            raise ValueError("`out` numpy arrays must be C-contiguous")
        return False
    if all(_is_cuda_tensor(a) and a.device == dev and a.is_contiguous() for a in out):
        return True
    raise TypeError(f"`out` must be three numpy arrays or three contiguous CUDA tensors on {dev}")


def normalize_candidates(
    candidates_csr: tp.Any, n_rows: int, n_objects: int, sorted_object_whitelist: tp.Optional[np.ndarray] = None
) -> tp.Tuple[np.ndarray, np.ndarray]:
    """Per-row allow-lists as the engine takes them: `(indptr int64 [n_rows + 1], indices int32)`, row r = the sorted,
    de-duplicated column ids of the STRUCTURE of `candidates_csr` row r (stored values, zeros included, are ignored, as for
    `filter_pairs_csr`), intersected with `sorted_object_whitelist` when it is given.  Works on copies: the caller's matrix
    is never changed."""
    if candidates_csr.shape[0] != n_rows:
        raise ValueError("Number of rows in `candidates_csr` must be equal to `len(subject_ids)`")
    csr = candidates_csr if sparse.isspmatrix_csr(candidates_csr) else sparse.csr_matrix(candidates_csr)
    indptr = np.asarray(csr.indptr, dtype=np.int64)
    indices = np.asarray(csr.indices, dtype=np.int64)[indptr[0] : indptr[-1]]
    indptr = indptr - indptr[0]
    if len(indices) and (indices.min() < 0 or indices.max() >= n_objects):
        raise ValueError(f"Candidate object ids in `candidates_csr` must be in [0, {n_objects}) (the objects of the ranker)")
    rows = np.repeat(np.arange(n_rows, dtype=np.int64), np.diff(indptr))
    key = np.unique(rows * n_objects + indices)  # sorted within a row, duplicates once (a new array)
    if sorted_object_whitelist is not None:
        key = key[np.isin(key % max(n_objects, 1), sorted_object_whitelist)]
    rows, cols = np.divmod(key, max(n_objects, 1))
    out_indptr = np.zeros(n_rows + 1, dtype=np.int64)
    np.cumsum(np.bincount(rows, minlength=n_rows), out=out_indptr[1:])
    return out_indptr, cols.astype(np.int32)


def flatten_padded(
    subject_ids: np.ndarray, ids: np.ndarray, scores: np.ndarray, counts: np.ndarray
) -> tp.Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Vectorised `_process_implicit_scores` (rank_implicit.py:120-146): padded rows -> flat ragged triplet."""
    k_out = ids.shape[1] if ids.ndim == 2 else 0
    if k_out == 0 or len(subject_ids) == 0:
        return np.empty(0, dtype=np.int64), np.empty(0, dtype=np.int64), np.empty(0, dtype=np.float32)
    if int(counts.min()) == k_out:
        return np.repeat(subject_ids, k_out), ids.reshape(-1).astype(np.int64), scores.reshape(-1)
    mask = np.arange(k_out, dtype=np.int32)[None, :] < counts[:, None]
    return np.repeat(subject_ids, counts), ids[mask].astype(np.int64), scores[mask]


_NEGINF_SCORE = np.uint32(np.float32(-np.finfo(np.float32).max).view(np.uint32) - 1).view(np.float32)


def strip_sentinel_tail(ids: np.ndarray, scores: np.ndarray, counts: np.ndarray) -> tp.Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """`_get_mask_for_correct_scores` (rank_implicit.py:107-118) on padded rows, in place: the trailing entries whose score
    is at most `_get_neginf_score()` (:83-92; -FLT_MAX and its neighbour) leave the row.  The engine drops only -inf, so a
    real score that low is returned by the kernels and stripped here, as the reference does; its slots become unfilled."""
    k_out = ids.shape[1] if ids.ndim == 2 else 0
    if k_out == 0 or len(counts) == 0:
        return ids, scores, counts
    rows = np.nonzero(counts > 0)[0]
    hit = rows[scores[rows, counts[rows] - 1] <= _NEGINF_SCORE]  # (best first: only rows whose last entry is that low)
    for r in hit:
        c = int(counts[r])
        while c > 0 and scores[r, c - 1] <= _NEGINF_SCORE:
            c -= 1
        ids[r, c : counts[r]] = -1
        scores[r, c : counts[r]] = -np.finfo(np.float32).max
        counts[r] = c
    return ids, scores, counts


class B200Ranker:
    """Ranker backed by the B200 engine.

    Parameters mirror `ImplicitRanker.__init__` (rank_implicit.py:58-65); `num_threads` / `use_gpu` are accepted and
    ignored so that the class can be bound in place of `ImplicitRanker` (rectools/models/vector.py:66-72).

    Parameters
    ----------
    distance : Distance | str
    subjects_factors : np.ndarray | scipy.sparse.csr_matrix | torch.Tensor, shape (n_subjects, n_factors)
    objects_factors : np.ndarray | torch.Tensor, shape (n_objects, n_factors)
    device : int, CUDA device ordinal; or a sequence of ordinals / "all": an engine group that splits every call's rows
        between one engine per entry (`EngineGroup`, same results)
    tc_mode : "auto" | "fp16" | "bf16" | "off" -- dtype of the tensor-core candidate pass ("off": fp64 kernel only)
    keep_16bit : fp16 / bf16 CUDA tensors and numpy fp16 object factors stay at 16 bits in the engine, with no fp32
        master copy (same results; `object_storage_dtype`).  A CUDA tensor is then read in place for the ranker's life.
        False: the engine widens them into an fp32 copy.

    One CUDA tensor passed as both factors (`subjects_factors is objects_factors`, item-to-item) ranks the catalogue's own
    rows: no copy of it is made, each `rank()` gathers its rows in their own type (`_rank_identity_padded`).
    """

    def __init__(
        self,
        distance: tp.Any,
        subjects_factors: tp.Any,
        objects_factors: tp.Any,
        num_threads: int = 0,  # pylint: disable=unused-argument
        use_gpu: bool = True,  # pylint: disable=unused-argument
        device: Devices = 0,
        tc_mode: str = "auto",
        engine: tp.Optional[Engine] = None,
        subjects_key: tp.Optional[tp.Hashable] = None,
        keep_16bit: bool = True,
    ) -> None:
        self.distance = _as_distance(distance)
        self._subjects_csr = None
        if sparse.issparse(subjects_factors) and self.distance != Distance.DOT:
            raise ValueError("To use `sparse.csr_matrix` distance must be `Distance.DOT`")  # rank_implicit.py:66-67
        if engine is None and self.distance != Distance.EUCLIDEAN and _is_cuda_tensor(objects_factors):
            # embeddings that already live on the GPU (transformer scorers keep `item_embs` on the device,
            # rectools/models/nn/transformers/lightning.py:391, :398): hand the device pointers over, no host round trip
            self._init_from_device_tensors(subjects_factors, objects_factors, tc_mode, device, keep_16bit)
            return
        objects_dtype = _lib.DT_F32
        if engine is None and isinstance(objects_factors, np.ndarray):
            objects_dtype = object_storage_dtype(self.distance, objects_factors.dtype, keep_16bit)
        if objects_dtype == _lib.DT_F16:  # numpy fp16 objects: uploaded as they are
            objects = _host_objects(objects_factors, _lib.DT_F16)
            if objects.ndim != 2:
                raise ValueError("factor matrices must be 2-dimensional")
        else:
            objects = _dense_f32(objects_factors)
        host_kw = {"objects_dtype": objects_dtype, "keep_16bit": objects_dtype == _lib.DT_F16}
        if sparse.issparse(subjects_factors):
            # EASE: the subjects are the user x item interaction CSR (rectools/models/ease.py:134-161).  The reference keeps the
            # matrix sparse and densifies only the requested rows (rank_implicit.py:236, :157-160); here the rows stay sparse
            # all the way into the SpMM scorer of the engine.
            csr = subjects_factors.tocsr()
            if csr.shape[1] != objects.shape[1]:
                raise ValueError("subject and object factors must have the same number of columns")
            self._subjects_csr = csr.astype(np.float32)
            self.n_subjects, self.n_objects = csr.shape[0], objects.shape[0]
            self.subjects_norms = self.subjects_dots = None
            self.engine = engine or new_engine(objects, cosine=False, device=device, tc_mode=tc_mode, **host_kw)
            self._subjects, self._subjects_key = None, None
            self.last_stats = {}
            return
        subjects = _dense_f32(subjects_factors)
        if subjects.shape[1] != objects.shape[1]:
            raise ValueError("subject and object factors must have the same number of columns")
        self.n_subjects, self.n_objects = subjects.shape[0], objects.shape[0]
        subjects, objects, self.subjects_norms, self.subjects_dots = prepare_factors(self.distance, subjects, objects)
        self.engine = engine or new_engine(objects, cosine=self.distance == Distance.COSINE, device=device, tc_mode=tc_mode, **host_kw)
        self._subjects, self._subjects_key = subjects, subjects_key
        self.engine.set_subjects(subjects, key=subjects_key, owner=self)
        self.last_stats: tp.Dict[str, tp.Any] = {}

    def _init_from_device_tensors(
        self, subjects_factors: tp.Any, objects_factors: tp.Any, tc_mode: str, device: Devices = 0, keep_16bit: bool = True
    ) -> None:
        import torch

        # fp16 / bf16 embeddings go to the engine as they are: kept at 16 bits and read in place (keep_16bit), or widened
        # exactly into an fp32 copy on the device (b200_rank_create_ex)
        dtypes = {torch.float32: _lib.DT_F32, torch.float16: _lib.DT_F16, torch.bfloat16: _lib.DT_BF16}
        objects = objects_factors.detach()
        if objects.dtype not in dtypes:
            objects = objects.to(torch.float32)
        objects = objects.contiguous()
        dev = objects.device
        # item-to-item passes one tensor as both factors (rectools/models/nn/transformers/lightning.py:440-442): the
        # subjects are the engine's own objects, so no copy of the catalogue is made; each call gathers its target rows
        # (`_rank_identity_padded`)
        self._identity = objects if subjects_factors is objects_factors else None
        self.subjects_norms = self.subjects_dots = None
        if self._identity is not None:
            self.n_subjects = self.n_objects = int(objects.shape[0])
            self._device_tensors = (objects,)  # the engine references this memory: keep it alive
        else:
            subjects = subjects_factors
            if sparse.issparse(subjects):
                raise ValueError("CSR subjects need host object factors")
            if not hasattr(subjects, "detach"):
                subjects = torch.from_numpy(_dense_f32(subjects))
            subjects = subjects.detach().to(device=dev, dtype=torch.float32).contiguous()
            if subjects.shape[1] != objects.shape[1]:
                raise ValueError("subject and object factors must have the same number of columns")
            self.n_subjects, self.n_objects = int(subjects.shape[0]), int(objects.shape[0])
            if self.distance == Distance.COSINE:
                self.subjects_norms = _device_norms(subjects)
            self._device_tensors = (subjects, objects)  # the engine references this memory: keep it alive
        torch.cuda.current_stream(dev).synchronize()
        home = dev.index or 0
        devices = parse_devices(device)
        if not isinstance(devices, int):  # a group whose home device is the tensors' device
            if home not in devices:
                raise ValueError(f"the factors live on cuda:{home}, which is not among the group's devices {devices}")
            rest = list(devices)
            rest.remove(home)
            devices = (home, *rest)
        self.engine = new_engine(
            None, cosine=self.distance == Distance.COSINE, device=home if isinstance(devices, int) else devices, tc_mode=tc_mode,
            objects_device_ptr=objects.data_ptr(), shape=(self.n_objects, int(objects.shape[1])), objects_dtype=dtypes[objects.dtype],
            keep_16bit=object_storage_dtype(self.distance, objects.dtype, keep_16bit) != _lib.DT_F32,
        )
        if self._identity is None:
            self.engine.set_subjects_device(self._device_tensors[0].data_ptr(), self.n_subjects)
        self._subjects = self._subjects_key = None
        self.last_stats = {}

    def _make_subjects_resident(self) -> None:
        """Leave the identity route: an fp32 copy of the catalogue becomes the resident subjects, as for two tensors (the
        candidate-set calls rank resident subjects by id)."""
        if getattr(self, "_identity", None) is None:
            return
        import torch

        objects = self._identity
        subjects = objects.to(torch.float32).contiguous()
        if self.distance == Distance.COSINE:
            self.subjects_norms = _device_norms(subjects)
        torch.cuda.current_stream(objects.device).synchronize()
        self._device_tensors = (subjects, objects)
        self.engine.set_subjects_device(subjects.data_ptr(), self.n_subjects)
        self._identity = None

    def _rank_identity_padded(
        self,
        subject_ids: np.ndarray,
        k: int,
        indptr: tp.Optional[np.ndarray],
        indices: tp.Optional[np.ndarray],
        whitelist: tp.Optional[np.ndarray],
        flags: int,
    ) -> tp.Tuple[np.ndarray, np.ndarray, np.ndarray, tp.Optional[np.ndarray]]:
        """The identity route of `rank_padded`: the target rows are gathered on the device in the catalogue's own type and
        handed to the engine as a batch of device subjects (16-bit rows are widened exactly by the engine).  Returns
        `(ids, scores, counts, norms)`; `norms` are the fp32 COSINE norms of these rows, computed as `_device_norms` computes
        them for resident subjects (None for DOT)."""
        import torch

        objects = self._identity
        dev = objects.device
        rows = objects.index_select(0, torch.from_numpy(subject_ids).to(dev))
        norms = _device_norms(rows) if self.distance == Distance.COSINE else None
        keep = [rows]
        q_kw = {}
        if whitelist is not None:
            wl = torch.from_numpy(np.ascontiguousarray(whitelist, dtype=np.int32)).to(dev)
            q_kw.update(whitelist=wl.data_ptr(), n_whitelist=len(wl))
            keep.append(wl)
        if indptr is not None:
            ip = torch.from_numpy(np.ascontiguousarray(indptr, dtype=np.int64)).to(dev)
            ix = torch.from_numpy(np.ascontiguousarray(indices, dtype=np.int32)).to(dev)
            q_kw.update(indptr=ip.data_ptr(), indices=ix.data_ptr() if len(ix) else 0)
            keep += [ip, ix]
        n_rows = len(subject_ids)
        k_out = min(int(k), len(whitelist) if whitelist is not None else self.n_objects)
        ids = np.empty((n_rows, k_out), dtype=np.int32)
        scores = np.empty((n_rows, k_out), dtype=np.float32)
        counts = np.zeros(n_rows, dtype=np.int32)
        dtypes = {torch.float32: _lib.DT_F32, torch.float16: _lib.DT_F16, torch.bfloat16: _lib.DT_BF16}
        self.engine.topk_ptrs(
            n_rows, k, ids.ctypes.data, scores.ctypes.data, counts.ctypes.data, flags | _lib.Q_INPUTS_ON_DEVICE,
            subjects=rows.data_ptr(), subject_dtype=dtypes[rows.dtype], stream=torch.cuda.current_stream(dev).cuda_stream, **q_kw,
        )
        del keep
        return ids, scores, counts, norms

    # ------------------------------------------------------------------------------------------------------------
    def rank_padded(
        self,
        subject_ids: InternalIds,
        k: tp.Optional[int] = None,
        filter_pairs_csr: tp.Optional[sparse.csr_matrix] = None,
        sorted_object_whitelist: tp.Optional[np.ndarray] = None,
        flags: int = 0,
    ) -> tp.Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
        """`rank` without the ragged flattening: `(subject_ids, ids [n,k], scores [n,k], counts [n])`."""
        return self._rank_padded(subject_ids, k, filter_pairs_csr, sorted_object_whitelist, flags)[:4]

    def _rank_padded(
        self,
        subject_ids: InternalIds,
        k: tp.Optional[int] = None,
        filter_pairs_csr: tp.Optional[sparse.csr_matrix] = None,
        sorted_object_whitelist: tp.Optional[np.ndarray] = None,
        flags: int = 0,
    ) -> tp.Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray, tp.Optional[np.ndarray]]:
        """`rank_padded` plus the COSINE norms of the rows when the identity route computed them for this call (else None:
        `subjects_norms` holds them)."""
        subject_ids = np.asarray(subject_ids, dtype=np.int64).reshape(-1)
        if filter_pairs_csr is not None and filter_pairs_csr.shape[0] != len(subject_ids):
            raise ValueError("Number of rows in `filter_pairs_csr` must be equal to `len(sublect_ids)`")
        if len(subject_ids) and (subject_ids.min() < 0 or subject_ids.max() >= self.n_subjects):
            raise IndexError("subject id out of range")
        whitelist = None
        n_pos = self.n_objects
        if sorted_object_whitelist is not None:
            whitelist = np.asarray(sorted_object_whitelist, dtype=np.int64).reshape(-1)
            check_whitelist(whitelist, self.n_objects)
            n_pos = len(whitelist)
        if k is None:
            k = n_pos  # rank_implicit.py:233-234
        if k <= 0:
            raise ValueError("`k` must be positive")
        indptr = indices = None
        if filter_pairs_csr is not None:
            csr = filter_pairs_csr if sparse.isspmatrix_csr(filter_pairs_csr) else sparse.csr_matrix(filter_pairs_csr)
            if not csr.has_sorted_indices:
                csr = csr.sorted_indices()
            indptr, indices = csr.indptr, csr.indices
        if n_pos == 0 or len(subject_ids) == 0:
            z = np.empty((len(subject_ids), 0))
            return subject_ids, z.astype(np.int32), z.astype(np.float32), np.zeros(len(subject_ids), np.int32), None
        if self._subjects_csr is not None:
            rows = self._subjects_csr[subject_ids]  # CSR row gather: cheap, stays sparse (rank_implicit.py:236)
            ids, scores, counts = self.engine.topk(
                k, sparse_subjects=rows, indptr=indptr, indices=indices, whitelist=whitelist, flags=flags & ~_lib.Q_FORCE_TC
            )
            self.last_stats = self.engine.last_stats
            return (subject_ids,) + strip_sentinel_tail(ids, scores, counts) + (None,)
        if getattr(self, "_identity", None) is not None:
            ids, scores, counts, norms = self._rank_identity_padded(subject_ids, k, indptr, indices, whitelist, flags)
            self.last_stats = self.engine.last_stats
            return (subject_ids,) + strip_sentinel_tail(ids, scores, counts) + (norms,)
        if getattr(self, "_subjects", None) is not None and self.engine.subjects_owner is not self:
            # another ranker sharing this (cached) engine made its own subject factors resident in the meantime
            self.engine.set_subjects(self._subjects, key=self._subjects_key, owner=self)
        ids, scores, counts = self.engine.topk(
            k, subject_ids=subject_ids, indptr=indptr, indices=indices, whitelist=whitelist, flags=flags
        )
        self.last_stats = self.engine.last_stats
        return (subject_ids,) + strip_sentinel_tail(ids, scores, counts) + (None,)

    def rank_object_rows_padded(
        self,
        target_ids: InternalIds,
        k: tp.Optional[int] = None,
        filter_pairs_csr: tp.Optional[sparse.csr_matrix] = None,
        sorted_object_whitelist: tp.Optional[np.ndarray] = None,
    ) -> tp.Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
        """`rank_object_rows` without the ragged flattening: `(target_ids, ids [n,k], scores [n,k], counts [n])`."""
        if self.distance != Distance.DOT:
            raise NotImplementedError("stored rows are score rows for Distance.DOT only")
        out = rank_object_rows_padded(self.engine, target_ids, k, filter_pairs_csr, sorted_object_whitelist)
        self.last_stats = self.engine.last_stats
        return out

    def rank_object_rows(
        self,
        target_ids: InternalIds,
        k: tp.Optional[int] = None,
        filter_pairs_csr: tp.Optional[sparse.csr_matrix] = None,
        sorted_object_whitelist: tp.Optional[np.ndarray] = None,
    ) -> tp.Tuple[InternalIds, InternalIds, Scores]:
        """Rank the object factors' own rows as score rows (square object factors, e.g. an EASE weight matrix): target t
        scores object j with `objects_factors[t, j]`, as `EASEModel._recommend_i2i` does (rectools/models/ease.py:163-188).
        Flat `(target ids repeated, object ids, scores)`, grouped by target in input order, best first."""
        target_ids, ids, scores, counts = self.rank_object_rows_padded(target_ids, k, filter_pairs_csr, sorted_object_whitelist)
        return flatten_padded(target_ids, ids, scores, counts)

    def rank_candidates_padded(
        self,
        subject_ids: InternalIds,
        candidates_csr: tp.Any,
        k: tp.Optional[int] = None,
        filter_pairs_csr: tp.Optional[sparse.csr_matrix] = None,
        sorted_object_whitelist: tp.Optional[np.ndarray] = None,
        flags: int = 0,
    ) -> tp.Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
        """`rank_candidates` without the ragged flattening: `(subject_ids, ids [n,k], scores [n,k], counts [n])`."""
        subject_ids = np.asarray(subject_ids, dtype=np.int64).reshape(-1)
        if filter_pairs_csr is not None and filter_pairs_csr.shape[0] != len(subject_ids):
            raise ValueError("Number of rows in `filter_pairs_csr` must be equal to `len(sublect_ids)`")
        if len(subject_ids) and (subject_ids.min() < 0 or subject_ids.max() >= self.n_subjects):
            raise IndexError("subject id out of range")
        if self._subjects_csr is not None:
            raise NotImplementedError("sparse (CSR) subjects are not ranked against candidate sets")
        if isinstance(self.engine, EngineGroup):
            raise NotImplementedError(
                "candidate sets are ranked by single engines: an engine group has no candidate-set export yet (use one device)"
            )
        self._make_subjects_resident()
        whitelist = None
        if sorted_object_whitelist is not None:
            whitelist = np.asarray(sorted_object_whitelist, dtype=np.int64).reshape(-1)
            check_whitelist(whitelist, self.n_objects)
        cand_indptr, cand_indices = normalize_candidates(candidates_csr, len(subject_ids), self.n_objects, whitelist)
        if k is None:
            k = int(np.diff(cand_indptr).max()) if len(subject_ids) else 0  # the longest list
            if k == 0:
                z = np.empty((len(subject_ids), 0))
                return subject_ids, z.astype(np.int32), z.astype(np.float32), np.zeros(len(subject_ids), np.int32)
        if k <= 0:
            raise ValueError("`k` must be positive")
        indptr = indices = None
        if filter_pairs_csr is not None:
            csr = filter_pairs_csr if sparse.isspmatrix_csr(filter_pairs_csr) else sparse.csr_matrix(filter_pairs_csr)
            if not csr.has_sorted_indices:
                csr = csr.sorted_indices()
            indptr, indices = csr.indptr, csr.indices
        if self.n_objects == 0 or len(subject_ids) == 0:
            z = np.empty((len(subject_ids), 0))
            return subject_ids, z.astype(np.int32), z.astype(np.float32), np.zeros(len(subject_ids), np.int32)
        if getattr(self, "_subjects", None) is not None and self.engine.subjects_owner is not self:
            self.engine.set_subjects(self._subjects, key=self._subjects_key, owner=self)
        ids, scores, counts = self.engine.topk_candidates(
            k, cand_indptr, cand_indices, subject_ids=subject_ids, indptr=indptr, indices=indices, flags=flags
        )
        self.last_stats = self.engine.last_stats
        return (subject_ids,) + strip_sentinel_tail(ids, scores, counts)

    def rank_candidates(
        self,
        subject_ids: InternalIds,
        candidates_csr: tp.Any,
        k: tp.Optional[int] = None,
        filter_pairs_csr: tp.Optional[sparse.csr_matrix] = None,
        sorted_object_whitelist: tp.Optional[np.ndarray] = None,
    ) -> tp.Tuple[InternalIds, InternalIds, Scores]:
        """Rank subject r against its own allow-list only: the structure of `candidates_csr` row r (column ids are object ids;
        unsorted rows and repeated ids are fine), minus its `filter_pairs_csr` row, intersected with
        `sorted_object_whitelist`.  `k = None`: the longest list.  Returns what `rank` returns -- flat `(subject ids repeated,
        object ids, scores)`, grouped by subject in input order, best first, with the same scores for the same pairs."""
        subject_ids, ids, scores, counts = self.rank_candidates_padded(
            subject_ids, candidates_csr, k, filter_pairs_csr, sorted_object_whitelist
        )
        return self._final_scores(*flatten_padded(subject_ids, ids, scores, counts))

    def rank_candidates_device(
        self,
        subject_ids: tp.Any,
        candidates: tp.Any,
        k: tp.Optional[int] = None,
        filter_pairs_csr: tp.Any = None,
        sorted_object_whitelist: tp.Optional[np.ndarray] = None,
    ) -> tp.Tuple[tp.Any, tp.Any, tp.Any]:
        """`rank_candidates` for candidates a GPU stage produced, with no host round trip: `candidates` is a CUDA int32 /
        int64 tensor [len(subject_ids), m] on the engine's device, row r = subject r's candidate ids in any order, repeats
        allowed, negative entries meaning "no candidate" (an entry >= n_objects raises ValueError).  `subject_ids`: numpy or
        CUDA.  `filter_pairs_csr`: a scipy CSR matrix or a CUDA `torch.sparse_csr_tensor` (column ids sorted within each
        row).  The whitelist is masked into the lists on the device.  `k = None`: m.
        Returns CUDA tensors `(ids [n, k_out] int32, scores [n, k_out], counts [n] int32)`, padded as
        `rank_candidates_padded` pads them and post-scaled as `rank_candidates` scales them: flattened (the first counts[r]
        entries of each row), they are bit for bit what `rank_candidates` returns for the same lists."""
        import torch

        if self._subjects_csr is not None:
            raise NotImplementedError("sparse (CSR) subjects are not ranked against candidate sets")
        if isinstance(self.engine, EngineGroup):
            raise NotImplementedError(
                "candidate sets are ranked by single engines: an engine group has no candidate-set export yet (use one device)"
            )
        self._make_subjects_resident()
        dev = torch.device("cuda", self.engine.device)
        if not _is_cuda_tensor(candidates) or candidates.device != dev or candidates.ndim != 2:
            raise TypeError(f"`candidates` must be a 2-dimensional CUDA tensor on {dev}")
        if candidates.dtype not in (torch.int32, torch.int64):
            raise TypeError(f"`candidates` must be int32 or int64, not {candidates.dtype}")
        n, m = int(candidates.shape[0]), int(candidates.shape[1])
        sids = subject_ids if _is_cuda_tensor(subject_ids) else torch.from_numpy(np.asarray(subject_ids, dtype=np.int64).reshape(-1))
        sids = sids.to(device=dev, dtype=torch.int64).reshape(-1).contiguous()
        if len(sids) != n:
            raise ValueError("Number of rows in `candidates` must be equal to `len(subject_ids)`")
        if n and bool(((sids < 0) | (sids >= self.n_subjects)).any()):
            raise IndexError("subject id out of range")
        if filter_pairs_csr is not None and filter_pairs_csr.shape[0] != n:
            raise ValueError("Number of rows in `filter_pairs_csr` must be equal to `len(sublect_ids)`")
        whitelist = None
        if sorted_object_whitelist is not None:
            whitelist = np.asarray(sorted_object_whitelist, dtype=np.int64).reshape(-1)
            check_whitelist(whitelist, self.n_objects)
        if k is None:
            k = m
        if k <= 0:
            if m == 0:
                z = torch.empty((n, 0), device=dev)
                return z.to(torch.int32), z, torch.zeros(n, dtype=torch.int32, device=dev)
            raise ValueError("`k` must be positive")
        if n and bool((candidates >= self.n_objects).any()):
            raise ValueError(f"Candidate object ids in `candidates` must be in [0, {self.n_objects}) (the objects of the ranker)")
        cand = torch.where(candidates < 0, -1, candidates).to(torch.int32)  # (no int64 negative wraps to an id)
        if whitelist is not None:
            cand = torch.where(torch.isin(cand, torch.from_numpy(whitelist.astype(np.int32)).to(dev)), cand, -1)
        cand_indptr = torch.arange(n + 1, dtype=torch.int64, device=dev) * m
        indptr = indices = None
        if filter_pairs_csr is not None:
            if _is_cuda_tensor(filter_pairs_csr):
                indptr = filter_pairs_csr.crow_indices().to(torch.int64)
                indices = filter_pairs_csr.col_indices().to(torch.int32)
            else:
                csr = filter_pairs_csr if sparse.isspmatrix_csr(filter_pairs_csr) else sparse.csr_matrix(filter_pairs_csr)
                if not csr.has_sorted_indices:
                    csr = csr.sorted_indices()
                indptr = torch.from_numpy(np.asarray(csr.indptr, dtype=np.int64)).to(dev)
                indices = torch.from_numpy(np.asarray(csr.indices, dtype=np.int32)).to(dev)
        if getattr(self, "_subjects", None) is not None and self.engine.subjects_owner is not self:
            self.engine.set_subjects(self._subjects, key=self._subjects_key, owner=self)
        ids, scores, counts = self.engine.topk_candidates_device(
            k, cand_indptr, cand.reshape(-1), subject_ids=sids, indptr=indptr, indices=indices
        )
        self.last_stats = self.engine.last_stats
        # the sentinel tail (strip_sentinel_tail): rows are best first, so the kept entries are those above it
        pos = torch.arange(ids.shape[1], device=dev)[None, :]
        kept = (pos < counts[:, None].long()) & (scores > float(_NEGINF_SCORE))
        counts = kept.sum(dim=1, dtype=torch.int32)
        ids = torch.where(kept, ids, -1)
        scores = torch.where(kept, scores, -float(np.finfo(np.float32).max))
        # the post-scaling of _final_scores, in the dtypes of its numpy arrays (uploaded once per ranker)
        if self.distance in (Distance.COSINE, Distance.EUCLIDEAN):
            post = getattr(self, "_post_device", None)
            if post is None or post.device != dev:
                host = self.subjects_norms if self.distance == Distance.COSINE else self.subjects_dots
                post = self._post_device = torch.from_numpy(np.ascontiguousarray(host)).to(dev)
            per_row = post[sids][:, None]
            if self.distance == Distance.COSINE:
                scaled = scores / per_row
            else:
                scaled = torch.sqrt(torch.clamp_min(per_row - scores, 0)).to(torch.float32)
            scores = torch.where(kept, scaled, scores.to(scaled.dtype))
        return ids, scores, counts

    def _final_scores(
        self, all_subjects: np.ndarray, all_ids: np.ndarray, all_scores: np.ndarray
    ) -> tp.Tuple[InternalIds, InternalIds, Scores]:
        """COSINE / EUCLIDEAN post-scaling of the flat triplet (rank_implicit.py:132-140)."""
        if self.distance == Distance.COSINE:
            all_scores = all_scores / self.subjects_norms[all_subjects]  # rank_implicit.py:132-134
        elif self.distance == Distance.EUCLIDEAN:
            d2 = self.subjects_dots[all_subjects] - all_scores  # rank_implicit.py:136-140
            all_scores = np.sqrt(np.maximum(d2, 0)).astype(np.float32)
        return all_subjects, all_ids, all_scores

    def rank(
        self,
        subject_ids: InternalIds,
        k: tp.Optional[int] = None,
        filter_pairs_csr: tp.Optional[sparse.csr_matrix] = None,
        sorted_object_whitelist: tp.Optional[np.ndarray] = None,
    ) -> tp.Tuple[InternalIds, InternalIds, Scores]:
        """Same contract as `ImplicitRanker.rank` (rank_implicit.py:187-280): flat `(subject ids repeated, object ids,
        scores)`, grouped by subject in input order, best first, filtered objects never returned."""
        subject_ids, ids, scores, counts, norms = self._rank_padded(subject_ids, k, filter_pairs_csr, sorted_object_whitelist)
        flat = flatten_padded(subject_ids, ids, scores, counts)
        if getattr(self, "_identity", None) is None:
            return self._final_scores(*flat)
        # identity route: COSINE divides by the norms of this call's rows, in fp32 as `_final_scores` does (no rows: None)
        return flat if norms is None else (flat[0], flat[1], flat[2] / np.repeat(norms, counts))
