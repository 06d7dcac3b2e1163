"""CPU (gloo): the sharded case table of tests/sharded_cases.py with the oracle standing in for the engines.

Proves without a GPU that the generators produce the edges they claim (each generator asserts them from its data and the
table is printed), that the expectations agree with the host merge on every row -- EUCLIDEAN, k > 32, empty shards and
empty local whitelists included, which tests/test_sharded_gloo.py does not reach -- and that the launcher kills the
remaining ranks when one fails."""
import time

import numpy as np
import pytest

from rectools_b200.sharded import EngineShard, ShardedB200Ranker, merge_padded_numpy, shard_bounds, split_whitelist
from tests import sharded_cases as sc


@pytest.mark.parametrize("config", list(sc.CONFIGS))
def test_case_table_with_the_oracle_provider(config, tmp_path, capsys):
    world, _ = sc.CONFIGS[config]
    cases = list(sc.CASES)
    text = sc.launch(world, ["--backend", "gloo", "--provider", "oracle", "--configs", config, "--cases", ",".join(cases)], str(tmp_path),
                     timeout=600)
    report = sc.check_results(str(tmp_path), config, cases, "oracle")
    with capsys.disabled():
        print("\n" + "\n".join(l for l in text.splitlines() if not l.startswith("  " + config)) + "\n" + report)
    assert "bit-identical" in report


def test_generators_show_their_edges():
    """The edges, once more from the outside: shard ranges, duplicates, whitelists, planted rows."""
    case = sc.edges_case(3, None, "oracle")
    b = shard_bounds(len(case.i), 3)
    assert [hi - lo for lo, hi in b] == [434, 434, 433]
    by_key = {c.key: c for c in case.calls}
    assert {c.ranker.distance for c in case.calls} == {"dot", "cosine", "euclidean"}
    assert {c.k for c in case.calls} >= {1, 10, 24, 25, 33, 100, 1025, None}
    assert {len(c.sids) for c in case.calls} >= {1, 2, 4, 37}
    wl = by_key["dot/share=0/wlA"].wl
    assert [len(split_whitelist(wl, lo, hi)) for lo, hi in b] == [217, 0, 0]
    same = np.nonzero((case.i == case.i[0]).all(axis=1))[0]
    assert len(same) == 18 and {0, 433, 434, 867, 868, 1300} <= set(same.tolist())
    tiny = sc.tiny_case(3, None, "oracle")
    assert shard_bounds(len(tiny.i), 3)[-1] == (4, 4)
    big = sc.certificate_case(2, None, "engine")
    assert (big.i[50_000:50_040] == big.i[50_000]).all() and len(sc.PLANTED) == 35
    assert {c.kind for c in big.calls} == {"rank", "device_cuda", "device_host"}
    assert [len(c.sub) for c in big.calls if c.key.startswith("device_cuda/") and c.key[12] in "123"] == [600, 300, 600]
    assert sc._group_rows(4, 2, 600) == [(0, 350), (350, 600)] and sc._group_rows(3, 1, 600) == [(0, 250), (250, 450), (450, 600)]  # pylint: disable=protected-access


def test_host_merge_breaks_ties_by_smaller_id_across_lists():
    """`merge_padded_numpy`, the expectation of every merge: equal scores in different lists come out by ascending id."""
    ids = np.array([[[7, 9, -1]], [[3, 8, -1]]], dtype=np.int32)
    scores = np.array([[[2.0, 1.0, 0.0]], [[2.0, 1.0, 0.0]]], dtype=np.float32)
    counts = np.array([[2], [2]], dtype=np.int32)
    o_ids, o_sc, o_cnt = merge_padded_numpy(ids, scores, counts, 3)
    assert o_ids.tolist() == [[3, 7, 8]] and o_sc.tolist() == [[2.0, 2.0, 1.0]] and o_cnt.tolist() == [3]


def test_launcher_kills_the_other_ranks_when_one_fails(tmp_path):
    t0 = time.monotonic()
    with pytest.raises(sc.LaunchFailed) as err:
        sc.launch(3, ["--backend", "gloo", "--provider", "oracle", "--cases", "tiny", "--die-on-rank", "1"], str(tmp_path), timeout=100)
    assert "rank 1 exited with 3" in err.value.reason
    assert time.monotonic() - t0 < 100
    codes = [p.poll() for p in err.value.procs]  # nobody outlives the launch: the ranks that would have waited were killed
    assert codes[1] == 3 and all(c is not None and c < 0 for c in (codes[0], codes[2])), codes


def test_more_than_nine_ranks_rank_unshared():
    """`enable_sharing` with more than nine ranks (a kernel polls at most eight peers) returns without exporting anything: the
    ranker then works unshared.  No engine is touched, so a bare shard shows it."""

    class TenRanks:
        @staticmethod
        def get_world_size(group):
            return 10

    shard = object.__new__(EngineShard)
    shard.sharing = False
    shard.enable_sharing(TenRanks, None, 100)  # (an export would need `shard.engine`: AttributeError)
    assert shard.sharing is False
    ranker = object.__new__(ShardedB200Ranker)
    ranker.host_provider, ranker.local, ranker.item_shards = False, shard, 10
    assert not ranker._shared_ok(5, 10)  # pylint: disable=protected-access
