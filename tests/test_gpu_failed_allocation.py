"""GPU: an allocation the device refuses is reported as B200_E_NOMEM, and the engine's next call on the same thread ranks
as if it had not happened (a refused cudaMalloc leaves the thread's last CUDA error set until something clears it)."""
import numpy as np
import pytest

from oracle.topk_oracle import rank_oracle
from tests.helpers import synth_factors, synth_viewed_csr

pytestmark = pytest.mark.gpu


def test_refused_allocation_does_not_fail_the_next_call():
    from rectools_b200 import _lib
    from rectools_b200.ranker import Engine

    n_users, n_items, d, k = 512, 20_000, 64, 10
    u, i = synth_factors(n_users, n_items, d, seed=5)
    csr = synth_viewed_csr(n_users, n_items, 50)
    eng = Engine(i, cosine=False)
    try:
        lib = _lib.load()
        # 2^32 rows of 64 fp32 columns: 1 TiB, which the driver refuses before anything is copied, so the small host
        # array is never read
        tiny = np.zeros((4, d), np.float32)
        rc = lib.b200_rank_set_subjects(eng._h, tiny.ctypes.data, 1 << 32, 0)  # pylint: disable=protected-access
        msg = lib.b200_rank_last_error().decode()
        assert rc == _lib.E_NOMEM, (rc, msg)
        assert msg.startswith("b200_rank_set_subjects: "), msg

        ids, scores, counts = eng.topk(k, subjects=u, indptr=csr.indptr.astype(np.int64), indices=csr.indices.astype(np.int32))
        _, oid, osc = rank_oracle("dot", u, i, np.arange(n_users), k, csr, accum="f64")
        assert (counts == k).all()
        np.testing.assert_array_equal(ids.reshape(-1), oid)
        np.testing.assert_allclose(scores.reshape(-1), osc, rtol=3e-7)
    finally:
        eng.close()
