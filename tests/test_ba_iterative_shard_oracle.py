"""The sharded ITERATIVE_SCHUR restatement (tests/ba_pcg_shard_oracle.py) on K = 2 and 3 thread ranks
(tests/emulated_ranks.py OracleAllReduce) against the same restatement unsharded, and that against
oracle/ba_pcg_oracle.py.

The ranks sum their parts of the reduced system in another order than the unsharded solve adds them, so the CG runs on
a system that differs by rounding.  Decisions must match exactly: termination, LM iterations, the outcome of every
iteration, and per LM iteration the CG iteration count and termination.  They are clear of rounding where the unsharded
run places them away from their thresholds, which is asserted: every zeta of every CG iteration at least 1e-6 from eta,
rho and the function-tolerance test outside their bands (tests/ba_harness.py assert_clear).  Values: costs and model
changes within 1e-9 relative, poses and points within 1e-8, intrinsics within 1e-8 relative.  Every rank makes the
same sequence of reductions (RankGroup.run).

CG iterates are not forward stable: a rounding-level change of the system grows with the CG iteration count (at C1 the
candidate cost of the 4th LM step, after 25 CG iterations, moves by 5e-7 relative between one and two ranks, and the
decisions of the steps after it then see costs 1e-5 apart).  The cases therefore run the first few LM iterations, whose
CG stops within a dozen iterations, where the bars above hold with a wide margin."""
import numpy as np
import pytest

from oracle import ba_oracle as bo
from oracle import ba_pcg_oracle as po
from tests import ba_pcg_shard_oracle as so
from tests.ba_loss_oracle import robust, with_outliers
from tests.ba_harness import assert_clear
from tests.emulated_ranks import run_shards
from tests.helpers import ba_case
from vggsfm_b200.dist import shard_range


def _shard(c, lo, hi, ptc):
    """the rank's slice of the track axis; an empty one becomes 16 masked padding tracks, as lm_solve pads"""
    S = c["mask"].shape[0]
    if hi > lo:
        return c["uv"][:, lo:hi], c["mask"][:, lo:hi], c["points"][lo:hi].copy(), ptc[lo:hi]
    pts = np.zeros((16, 3))
    pts[:, 2] = 1.0
    return np.zeros((S, 16, 2)), np.zeros((S, 16), bool), pts, np.ones(16, bool)


def _run(c, o, lo=0, hi=None, pc=None, ptc=None, allreduce=None, max_cg=500):
    N = c["mask"].shape[1]
    hi = N if hi is None else hi
    ptc = np.zeros(N, bool) if ptc is None else ptc
    uv, mask, pts, pt_c = _shard(c, lo, hi, ptc)
    trace, cgs = [], []
    poses, intr, pts, summ = so.lm_solve(c["poses"].copy(), c["intr"].copy(), pts, uv, mask, c["model"], c["mode"],
                                         param_const=pc, point_const=pt_c, options=o, trace=trace,
                                         max_linear_solver_iterations=max_cg, cg_traces=cgs, allreduce=allreduce)
    return dict(poses=poses, intr=intr, points=pts[:hi - lo], s=summ, trace=trace, cg=cgs, lo=lo, hi=hi)


def _sharded(c, K, o, **kw):
    return run_shards(c["mask"].shape[1], K, lambda r, lo, hi, hook: _run(c, o, lo, hi, allreduce=hook, **kw))


def _cg_key(cgs):
    return [(cg["summary"]["iterations"], cg["summary"]["termination"]) for cg in cgs]


def _check(res, ref, label):
    s0 = ref["s"]
    for r, x in enumerate(res):
        s = x["s"]
        what = (label, "rank", r, x["lo"], x["hi"])
        assert s["termination"] == s0["termination"] and s["iterations"] == s0["iterations"], (what, s, s0)
        assert [t["outcome"] for t in x["trace"]] == [t["outcome"] for t in ref["trace"]], what
        assert _cg_key(x["cg"]) == _cg_key(ref["cg"]), (what, _cg_key(x["cg"]), _cg_key(ref["cg"]))
        assert np.isclose(s["final_cost"], s0["final_cost"], rtol=1e-9, atol=0), what
        for t, t0 in zip(x["trace"], ref["trace"]):
            for k in ("candidate_cost", "model_change"):
                if k in t0 and np.isfinite(t0[k]):
                    assert np.isclose(t[k], t0[k], rtol=1e-9, atol=0), (what, k, t[k], t0[k])
        assert np.nanmax(np.abs(x["poses"] - ref["poses"])) < 1e-8, what
        assert np.all(np.abs(x["intr"] - ref["intr"]) <= 1e-8 * np.maximum(1.0, np.abs(ref["intr"]))), what
        if x["hi"] > x["lo"]:
            assert np.nanmax(np.abs(x["points"] - ref["points"][x["lo"]:x["hi"]])) < 1e-8, what
        # one CG on every rank: the same summed system and the same code
        assert _cg_key(x["cg"]) == _cg_key(res[0]["cg"])
        assert np.array_equal(x["poses"], res[0]["poses"], equal_nan=True), what


def _case(name):
    if name == "C1":
        return ba_case(8, 256, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=0), bo.LMOptions(max_num_iterations=3)
    return ba_case(50, 2048, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=1), bo.LMOptions(max_num_iterations=3)


def test_unsharded_restatement_is_the_pcg_oracle():
    """allreduce None: the same decisions and values as oracle/ba_pcg_oracle.py's lm_solve"""
    c, o = _case("C1")
    ref = _run(c, o)
    trace, cgs = [], []
    p, i, x, s = po.lm_solve(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], c["mode"], options=o,
                             trace=trace, cg_traces=cgs)
    assert s["termination"] == ref["s"]["termination"] and s["iterations"] == ref["s"]["iterations"]
    assert [t["outcome"] for t in trace] == [t["outcome"] for t in ref["trace"]]
    assert _cg_key(cgs) == _cg_key(ref["cg"])
    assert np.isclose(s["final_cost"], ref["s"]["final_cost"], rtol=1e-12, atol=0)
    assert np.abs(p - ref["poses"]).max() < 1e-10 and np.abs(x - ref["points"]).max() < 1e-10


@pytest.mark.parametrize("K", [2, 3])
@pytest.mark.parametrize("name", ["C1", "C2"])
def test_shards_match_unsharded(name, K):
    c, o = _case(name)
    ref = _run(c, o)
    assert_clear(ref["trace"], o, cg=ref["cg"])
    res, _ = _sharded(c, K, o)
    _check(res, ref, f"{name} K={K}")


def test_empty_shard():
    """64 tracks over 3 ranks: 32 / 32 / 0; the empty rank solves 16 masked padding tracks"""
    c = ba_case(8, 64, "SIMPLE_RADIAL", bo.INTR_PER_FRAME, seed=13)
    o = bo.LMOptions(max_num_iterations=3)
    assert shard_range(64, 2, 3) == (64, 64)
    ref = _run(c, o)
    assert_clear(ref["trace"], o, cg=ref["cg"])
    res, group = _sharded(c, 3, o)
    _check(res, ref, "empty shard")
    assert len(group.tags[2]) == len(group.tags[0]) > 3 * ref["s"]["iterations"]


@pytest.mark.parametrize("K", [2, 3])
def test_constant_and_unobserved(K):
    """a constant pose, constant points, a frame that only the first shard sees and a frame nothing sees"""
    c = ba_case(10, 300, "SIMPLE_RADIAL", bo.INTR_SHARED, seed=5)
    mask = c["mask"].copy()
    mask[7] = False
    lo, hi = shard_range(300, 0, K)
    mask[4, hi:] = False
    c = dict(c, mask=mask)
    const_pose = np.zeros(10, bool)
    const_pose[2] = True
    pc = bo.default_param_const(10, c["model"], c["mode"], const_pose=const_pose)
    ptc = np.zeros(300, bool)
    ptc[::11] = True
    o = bo.LMOptions(max_num_iterations=3)
    ref = _run(c, o, pc=pc, ptc=ptc)
    assert_clear(ref["trace"], o, cg=ref["cg"])
    assert np.abs(ref["poses"][4] - c["poses"][4]).max() > 1e-6
    res, _ = _sharded(c, K, o, pc=pc, ptc=ptc)
    _check(res, ref, f"constant / unobserved K={K}")
    for x in res:
        assert np.array_equal(x["poses"][7], c["poses"][7]) and np.array_equal(x["poses"][2], c["poses"][2])


@pytest.mark.parametrize("K", [2, 3])
def test_cauchy(K):
    c = with_outliers(ba_case(8, 256, "SIMPLE_RADIAL", bo.INTR_PER_FRAME, seed=3), frac=0.1, seed=3)
    o = bo.LMOptions(max_num_iterations=3)
    with robust("CAUCHY", 1.0):
        ref = _run(c, o)
        assert_clear(ref["trace"], o, cg=ref["cg"])
        res, _ = _sharded(c, K, o)
    _check(res, ref, f"CAUCHY K={K}")
