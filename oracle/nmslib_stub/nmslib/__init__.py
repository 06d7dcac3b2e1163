"""Exact brute-force stand-in for the part of nmslib that `rectools.tools.ann` calls (test infrastructure only).

nmslib cannot be installed here, and RecTools skips its own ANN tests on Python >= 3.13.  With this directory on
sys.path the unmodified `rectools.tools.ann` imports, and its classes answer every query exactly: `knnQueryBatch`
returns the k stored points of smallest distance, by (distance asc, id asc), distances computed in fp64 over the float32
data, as nmslib stores it.  Spaces: "cosinesimil" (1 - cos), "negdotprod" (-dot), "l2" (Euclidean distance).  The index
parameters are recorded and have no effect.
"""
from __future__ import annotations

import pickle
import typing as tp

import numpy as np

_SPACES = ("cosinesimil", "negdotprod", "l2")


class FloatIndex:
    def __init__(self, space: str = "cosinesimil", method: str = "hnsw") -> None:
        if space not in _SPACES:
            raise ValueError(f"space {space!r} is not implemented by the stub")
        self.space, self.method = space, method
        self.data = np.empty((0, 0), dtype=np.float32)
        self.query_time_params: tp.Dict[str, tp.Any] = {}
        self.index_params: tp.Dict[str, tp.Any] = {}

    def addDataPointBatch(self, data: tp.Any, ids: tp.Any = None) -> np.ndarray:  # noqa: N802  pylint: disable=invalid-name
        data = np.asarray(data, dtype=np.float32)
        start = len(self.data)
        self.data = data.copy() if start == 0 else np.vstack([self.data, data])
        return np.arange(start, len(self.data))

    def createIndex(self, index_params: tp.Any = None, print_progress: bool = False) -> None:  # noqa: N802  pylint: disable=invalid-name,unused-argument
        self.index_params = dict(index_params or {})

    def setQueryTimeParams(self, params: tp.Any = None) -> None:  # noqa: N802  pylint: disable=invalid-name
        self.query_time_params = dict(params or {})

    def _distances(self, queries: np.ndarray) -> np.ndarray:
        x = self.data.astype(np.float64)
        q = queries.astype(np.float64)
        if self.space == "negdotprod":
            return -(q @ x.T)
        if self.space == "l2":
            return np.sqrt(np.maximum(((q[:, None, :] - x[None, :, :]) ** 2).sum(axis=2), 0.0))
        qn = np.linalg.norm(q, axis=1)[:, None]
        xn = np.linalg.norm(x, axis=1)[None, :]
        with np.errstate(invalid="ignore", divide="ignore"):
            cos = (q @ x.T) / (qn * xn)
        return 1.0 - np.nan_to_num(cos, nan=0.0)

    def knnQueryBatch(self, queries: tp.Any, k: int = 10, num_threads: int = 0) -> tp.List[tp.Tuple[np.ndarray, np.ndarray]]:  # noqa: N802  pylint: disable=invalid-name,unused-argument
        queries = np.atleast_2d(np.asarray(queries, dtype=np.float32))
        dist = self._distances(queries)
        k = min(int(k), len(self.data))
        out = []
        ids = np.arange(len(self.data))
        for row in dist:
            order = np.lexsort((ids, row))[:k]  # distance asc, then id asc
            out.append((order.astype(np.int32), row[order].astype(np.float32)))
        return out

    def saveIndex(self, filename: str, save_data: bool = False) -> None:  # noqa: N802  pylint: disable=invalid-name,unused-argument
        with open(filename, "wb") as f:
            pickle.dump({"space": self.space, "method": self.method, "data": self.data, "index_params": self.index_params}, f)

    def loadIndex(self, filename: str, load_data: bool = False) -> None:  # noqa: N802  pylint: disable=invalid-name,unused-argument
        with open(filename, "rb") as f:
            state = pickle.load(f)
        self.space, self.method, self.data, self.index_params = state["space"], state["method"], state["data"], state["index_params"]


def init(method: str = "hnsw", space: str = "cosinesimil", data_type: tp.Any = None, dtype: tp.Any = None, **_: tp.Any) -> FloatIndex:  # pylint: disable=unused-argument
    return FloatIndex(space=space, method=method)


def setQueryTimeParams(index: FloatIndex, params: tp.Any = None) -> None:  # noqa: N802  pylint: disable=invalid-name
    index.setQueryTimeParams(params)
