"""The oracle's track-sharded LM over emulated ranks (tests/emulated_ranks.py: threads meeting at a barrier for every
all-reduce), on CPU.  test_dist_gloo.py checks the sharding algebra through gloo; here a rank that leaves the loop while
the others ask for another reduction fails at once instead of blocking in all_reduce until its timeout.

The parameter tolerance compares the (reduced) step norm with |x|, and |x| sums every free point: with the point part
taken over the rank's own points only, each rank has its own |x| and the ranks may stop at different iterations.  The
case puts the far points in rank 0's shard, so the local |x| of the two ranks (35.9 and 29.5 at the start) are both well
below the true one (46.3)."""
import time

import numpy as np
import pytest

from oracle import ba_oracle as bo
from tests.ba_harness import oracle_solve
from tests.emulated_ranks import RankGroup, RanksFailed, run_shards
from tests.helpers import far_points_first_case
from vggsfm_b200.dist import shard_range


def check_against_unsharded(res, ref):
    for r, x in enumerate(res):
        summ, summ0 = x["s"], ref["s"]
        assert summ["termination"] == summ0["termination"], (r, summ["termination"], summ0["termination"])
        assert summ["iterations"] == summ0["iterations"] and summ["successful"] == summ0["successful"], (r, summ)
        assert [t["outcome"] for t in x["trace"]] == [t["outcome"] for t in ref["trace"]]
        for t, t0 in zip(x["trace"], ref["trace"]):
            assert abs(t["x_norm"] - t0["x_norm"]) <= 1e-12 * t0["x_norm"], (r, t["x_norm"], t0["x_norm"])
            assert abs(t["candidate_cost"] - t0["candidate_cost"]) <= 1e-9 * t0["candidate_cost"]
        assert np.array_equal(x["poses"], res[0]["poses"]) and np.array_equal(x["intr"], res[0]["intr"])


@pytest.mark.parametrize("K,ptol", [(2, 0.0072), (2, 0.0054), (4, 0.0072)])
def test_parameter_tolerance_over_shards(K, ptol):
    """every rank stops where the unsharded solve stops; the tolerance lies strictly between two iterations of the
    unsharded trace (ratio step_norm / (ptol (|x| + ptol)) at least 1e-6 away from 1)"""
    c = far_points_first_case()
    opt = bo.LMOptions(max_num_iterations=20, function_tolerance=0.0, gradient_tolerance=0.0, parameter_tolerance=ptol)
    ref = oracle_solve(c, opt=opt)
    summ0 = ref["s"]
    assert summ0["termination"] == "CONVERGENCE_PARAMETER", summ0
    ratios = [t["step_norm"] / (ptol * (t["x_norm"] + ptol)) for t in ref["trace"] if t["outcome"] != 2]
    assert all(abs(q - 1.0) > 1e-6 for q in ratios), ratios
    assert ratios[-1] < 1.0 and all(q > 1.0 for q in ratios[:-1]), ratios
    res, group = run_shards(c["mask"].shape[1], K, lambda r, lo, hi, hook: oracle_solve(c, opt=opt, lo=lo, hi=hi,
                                                                                           allreduce=hook),
                            timeout=60.0)
    check_against_unsharded(res, ref)
    assert len(group.tags[0]) >= 2 * summ0["iterations"]
    for x in res:
        assert np.abs(x["poses"] - ref["poses"]).max() < 1e-9
        assert np.abs(x["points"] - ref["points"][x["lo"]:x["hi"]]).max() < 1e-9


def test_local_x_norm_is_not_the_global_one():
    """the premise of the case: each rank's own points give an |x| far below the true one"""
    c = far_points_first_case()
    S, N = c["mask"].shape
    dc, ns = bo.dims(c["model"], c["mode"])
    pc = bo.default_param_const(S, c["model"], c["mode"])
    full = bo._x_norm(c["poses"], c["intr"], c["points"], S, dc, ns, pc, np.zeros(N, bool))
    local = [bo._x_norm(c["poses"], c["intr"], c["points"][lo:hi], S, dc, ns, pc, np.zeros(hi - lo, bool))
             for lo, hi in (shard_range(N, r, 2) for r in range(2))]
    assert local[0] < 0.8 * full and local[1] < 0.7 * full, (local, full)
    cams, _ = bo._x_norm_parts(c["poses"], c["intr"], c["points"], S, dc, ns, pc, np.zeros(N, bool))
    parts = [bo._x_norm_parts(c["poses"], c["intr"], c["points"][lo:hi], S, dc, ns, pc, np.zeros(hi - lo, bool))[1]
             for lo, hi in (shard_range(N, r, 2) for r in range(2))]
    assert abs(np.sqrt(cams + sum(parts)) - full) <= 1e-14 * full


def test_diverged_rank_fails_fast():
    """the emulation itself: a rank that stops while the other asks for another reduction ends the run at once, with
    the tags both arrived with, not after the barrier timeout"""
    group = RankGroup(2, timeout=600.0)

    def rank(r):
        if r == 1:
            group.reduce(r, 1, 0, np.zeros(1), lambda acc: None)
        return r

    t0 = time.perf_counter()
    with pytest.raises(RanksFailed, match=r"diverged: arrived with \['exit', \(1, 0\)\]"):
        group.run(rank)
    assert time.perf_counter() - t0 < 60.0


def test_failing_rank_releases_the_others():
    """a rank that raises before its first reduction (as a solve that rejects its arguments does) breaks the barrier:
    the other ranks' reductions fail at once and the error names the rank"""
    group = RankGroup(3, timeout=600.0)

    def rank(r):
        if r == 2:
            raise ValueError("null problem array")
        group.reduce(r, 1, 0, np.zeros(1), lambda acc: None)
        return r

    t0 = time.perf_counter()
    with pytest.raises(RanksFailed, match="null problem array"):
        group.run(rank)
    assert time.perf_counter() - t0 < 60.0
