"""ctypes binding of libb200rank.so (include/b200_rank.h).  No fallback: a missing library is an error."""
from __future__ import annotations

import ctypes as C
import os
import typing as tp

HERE = os.path.dirname(os.path.abspath(__file__))
# B200_RANK_LIB: measurement hook -- load a variant build (python -m rectools_b200.build --variant NAME -DX=..) instead
LIB_PATH = os.environ.get("B200_RANK_LIB") or os.path.join(HERE, "libb200rank.so")

# mirrors of the #defines in include/b200_rank.h
ABI_VERSION = 6
OK, E_INVALID, E_CUDA, E_NOMEM, E_UNSUPPORTED = 0, -1, -2, -3, -4
DIST_DOT, DIST_COSINE = 0, 1
TC_AUTO, TC_FP16, TC_BF16, TC_OFF = 0, 1, 2, 3
F_OBJECTS_ON_DEVICE, F_OBJECTS_16BIT = 1, 2
Q_INPUTS_ON_DEVICE, Q_OUTPUTS_ON_DEVICE, Q_FORCE_EXACT, Q_FORCE_TC, Q_SHARED_THRESHOLDS = 1, 2, 4, 8, 16
DT_F32, DT_F16, DT_BF16 = 0, 1, 2
PAIRS_F64, PAIRS_F32, PAIRS_I64, PAIRS_I32 = 0, 1, 2, 3
MIX_ROTATE, MIX_GROUP = 0, 1

EXPORTS = (
    "b200_rank_create",
    "b200_rank_create_ex",
    "b200_rank_destroy",
    "b200_rank_set_subjects",
    "b200_rank_set_id_offset",
    "b200_rank_topk",
    "b200_rank_topk_candidates",
    "b200_rank_topk_candidates_device",
    "b200_rank_get_info",
    "b200_rank_merge",
    "b200_rank_merge_certified",
    "b200_rank_topk_pairs",
    "b200_rank_topk_list",
    "b200_rank_topk_list_mix",
    "b200_rank_topk_knn",
    "b200_rank_peer_export",
    "b200_rank_peer_import",
    "b200_rank_get_snapshot",
    "b200_rank_peer_attach",
    "b200_rank_last_error",
    "b200_rank_abi_version",
    "b200_rank_group_create",
    "b200_rank_group_create_ex",
    "b200_rank_group_destroy",
    "b200_rank_group_get_info",
    "b200_rank_group_set_subjects",
    "b200_rank_group_topk",
)


class Query(C.Structure):
    _fields_ = [
        ("subjects", C.c_void_p),
        ("subject_ids", C.c_void_p),
        ("n_rows", C.c_int64),
        ("n_subjects_total", C.c_int64),
        ("csr_indptr", C.c_void_p),
        ("csr_indices", C.c_void_p),
        ("whitelist", C.c_void_p),
        ("n_whitelist", C.c_int64),
        ("k", C.c_int32),
        ("flags", C.c_int32),
        ("out_ids", C.c_void_p),
        ("out_scores", C.c_void_p),
        ("out_counts", C.c_void_p),
        ("stream", C.c_void_p),
        ("out_bounds", C.c_void_p),
        ("peer_epoch", C.c_uint32),
        ("subject_dtype", C.c_int32),
        ("sub_indptr", C.c_void_p),
        ("sub_indices", C.c_void_p),
        ("sub_data", C.c_void_p),
        ("object_rows", C.c_void_p),  # ABI 6: stored rows as score rows (path 4)
        ("reserved", C.c_int64 * 1),
    ]


class Stats(C.Structure):
    _fields_ = [
        ("path", C.c_int32),
        ("tc_dtype", C.c_int32),
        ("k_out", C.c_int32),
        ("k_cand", C.c_int32),
        ("n_splits", C.c_int32),
        ("n_launches", C.c_int32),
        ("n_fallback_rows", C.c_int64),
        ("n_exact_rows", C.c_int64),
        ("ms_main", C.c_float),
        ("ms_total", C.c_float),
        ("ms_h2d", C.c_float),
        ("ms_d2h", C.c_float),
        ("h2d_bytes", C.c_int64),
        ("d2h_bytes", C.c_int64),
        ("n_chunks", C.c_int32),
        ("n_tc_launches", C.c_int32),
        ("epi_warps", C.c_int32),  # always 8 (one fused-kernel geometry)
        ("wide", C.c_int32),
        ("ms_select", C.c_float),
        ("ms_main_pass", C.c_float),  # the main-pass launches of the fused kernel inside ms_main (path 1)
    ]

    def as_dict(self) -> tp.Dict[str, tp.Any]:
        return {name: getattr(self, name) for name, _ in self._fields_ if name != "reserved"}


class Info(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int32),
        ("device", C.c_int32),
        ("sm_count", C.c_int32),
        ("cc_major", C.c_int32),
        ("cc_minor", C.c_int32),
        ("tc_dtype", C.c_int32),
        ("n_objects", C.c_int64),
        ("d", C.c_int32),
        ("d_pad", C.c_int32),
        ("hbm_bytes", C.c_int64),
        ("device_name", C.c_char * 128),
    ]


class Snapshot(C.Structure):
    """`b200_rank_snapshot`: metadata of the tensor-core pass captured with B200_TC_SNAPSHOT (test interface)."""

    _fields_ = [
        ("valid", C.c_int32),
        ("launch", C.c_int32),
        ("nw", C.c_int32),  # always 8: two lists per row and object split
        ("n_lists", C.c_int32),
        ("n_splits", C.c_int32),
        ("tiles_per_split", C.c_int32),
        ("n_obj_tiles", C.c_int32),
        ("cand_stride", C.c_int32),
        ("n_pos", C.c_int64),
        ("rows_pad", C.c_int64),
        ("n_sel", C.c_int64),
        ("k_out", C.c_int32),
        ("k_cand", C.c_int32),
        ("k0", C.c_int32),
        ("kp", C.c_int32),
        ("wide", C.c_int32),
        ("phase1_tiles", C.c_int32),
        ("bf16", C.c_int32),
        ("obj_exp", C.c_int32),
        ("eps_rel", C.c_float),
        ("max_obj_norm", C.c_float),
        ("id_off", C.c_int32),
        ("n_fb", C.c_int32),
    ]


class B200RankError(RuntimeError):
    """CUDA / driver failure inside libb200rank.so."""


_LIB: tp.Optional[C.CDLL] = None


def load() -> C.CDLL:
    """Load the shared library (once).  Raises if it has not been built -- there is deliberately no CPU fallback."""
    global _LIB  # pylint: disable=global-statement
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise B200RankError(
            f"{LIB_PATH} is missing: build it with `python -m rectools_b200.build` "
            "(nvcc, sm_90a).  rectools_b200 has no CPU fallback."
        )
    lib = C.CDLL(LIB_PATH)
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    lib.b200_rank_create.restype = C.c_int
    lib.b200_rank_create.argtypes = [C.POINTER(vp), vp, i64, i32, i32, i32, i32, i32]
    lib.b200_rank_create_ex.restype = C.c_int
    lib.b200_rank_create_ex.argtypes = [C.POINTER(vp), vp, i32, i64, i32, i32, i32, i32, i32]
    lib.b200_rank_destroy.restype = C.c_int
    lib.b200_rank_destroy.argtypes = [vp]
    lib.b200_rank_set_subjects.restype = C.c_int
    lib.b200_rank_set_subjects.argtypes = [vp, vp, i64, i32]
    lib.b200_rank_set_id_offset.restype = C.c_int
    lib.b200_rank_set_id_offset.argtypes = [vp, i64]
    lib.b200_rank_topk.restype = C.c_int
    lib.b200_rank_topk.argtypes = [vp, C.POINTER(Query), C.POINTER(Stats)]
    lib.b200_rank_topk_candidates.restype = C.c_int
    lib.b200_rank_topk_candidates.argtypes = [vp, C.POINTER(Query), vp, vp, C.POINTER(Stats)]
    lib.b200_rank_topk_candidates_device.restype = C.c_int
    lib.b200_rank_topk_candidates_device.argtypes = [vp, C.POINTER(Query), vp, vp, C.POINTER(Stats)]
    lib.b200_rank_get_info.restype = C.c_int
    lib.b200_rank_get_info.argtypes = [vp, C.POINTER(Info)]
    lib.b200_rank_merge.restype = C.c_int
    lib.b200_rank_merge.argtypes = [i32, vp, i32, i64, i32, vp, vp, vp, vp, vp, vp]
    lib.b200_rank_merge_certified.restype = C.c_int
    lib.b200_rank_merge_certified.argtypes = [i32, vp, i32, i64, i32, vp, vp, vp, vp, i64, vp, vp, vp, vp, vp]
    lib.b200_rank_topk_pairs.restype = C.c_int
    lib.b200_rank_topk_pairs.argtypes = [i32, vp, i64, vp, vp, i32, i64, i32, i32, vp, vp, C.POINTER(Stats)]
    lib.b200_rank_topk_list.restype = C.c_int
    lib.b200_rank_topk_list.argtypes = [i32, i64, vp, i64, vp, vp, i32, vp, vp, C.POINTER(Stats)]
    lib.b200_rank_topk_list_mix.restype = C.c_int
    lib.b200_rank_topk_list_mix.argtypes = [i32, i32, vp, vp, vp, i32, i64, vp, vp, i32, vp, vp, C.POINTER(Stats)]
    lib.b200_rank_topk_knn.restype = C.c_int
    lib.b200_rank_topk_knn.argtypes = [i32, i64, vp, vp, vp, i64, vp, vp, vp, vp, vp, vp, i64, i32, vp, vp, vp, C.POINTER(Stats)]
    lib.b200_rank_peer_export.restype = C.c_int
    lib.b200_rank_peer_export.argtypes = [vp, i64, vp]
    lib.b200_rank_peer_import.restype = C.c_int
    lib.b200_rank_peer_import.argtypes = [vp, i32, i32, vp]
    lib.b200_rank_get_snapshot.restype = C.c_int
    lib.b200_rank_get_snapshot.argtypes = [vp, C.POINTER(Snapshot), vp, vp, vp, vp, vp, vp, vp]
    lib.b200_rank_peer_attach.restype = C.c_int
    lib.b200_rank_peer_attach.argtypes = [vp, i64, vp, i32, C.POINTER(vp)]
    lib.b200_rank_last_error.restype = C.c_char_p
    lib.b200_rank_last_error.argtypes = []
    lib.b200_rank_abi_version.restype = C.c_int
    lib.b200_rank_abi_version.argtypes = []
    lib.b200_rank_group_create.restype = C.c_int
    lib.b200_rank_group_create.argtypes = [C.POINTER(vp), vp, i64, i32, i32, vp, i32, i32, i32]
    lib.b200_rank_group_create_ex.restype = C.c_int
    lib.b200_rank_group_create_ex.argtypes = [C.POINTER(vp), vp, i32, i64, i32, i32, vp, i32, i32, i32]
    lib.b200_rank_group_destroy.restype = C.c_int
    lib.b200_rank_group_destroy.argtypes = [vp]
    lib.b200_rank_group_get_info.restype = C.c_int
    lib.b200_rank_group_get_info.argtypes = [vp, C.POINTER(Info), C.POINTER(i64)]
    lib.b200_rank_group_set_subjects.restype = C.c_int
    lib.b200_rank_group_set_subjects.argtypes = [vp, vp, i64, i32]
    lib.b200_rank_group_topk.restype = C.c_int
    lib.b200_rank_group_topk.argtypes = [vp, C.POINTER(Query), C.POINTER(Stats), C.POINTER(Stats)]
    if lib.b200_rank_abi_version() != ABI_VERSION:
        raise B200RankError("libb200rank.so ABI version mismatch: rebuild with `python -m rectools_b200.build --force`")
    _LIB = lib
    return lib


def check(rc: int) -> None:
    """Map the C error convention onto the reference's exceptions: ValueError for contract violations
    (rank_implicit.py:215-217), RuntimeError subclasses for device failures."""
    if rc == OK:
        return
    msg = (load().b200_rank_last_error() or b"").decode("utf-8", "replace")
    if rc == E_INVALID:
        raise ValueError(msg)
    if rc == E_UNSUPPORTED:
        raise NotImplementedError(msg)
    if rc == E_NOMEM:
        raise MemoryError(msg)
    raise B200RankError(msg)
