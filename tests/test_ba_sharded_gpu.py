"""The track-sharded LM loop of vgg_ba_solve on one GPU: K ranks emulated by K host threads (tests/emulated_ranks.py),
each with its own stream, shard and workspace, reducing through the solver's all-reduce hook.  This is the path
`bench.py --gpus N` runs over NCCL; test_dist_gpu.py needs two GPUs and test_dist_gloo.py runs the oracle only.

The reference is the unsharded CUDA solve of the same problem (and the float64 oracle where a decision is placed). Every
rank must take the unsharded run's decisions: the same termination, iterations and per-iteration outcome (trace column
7).  Values use test_dist_gpu.py's bars: final cost within 1e-9 relative, candidate costs (trace column 2) within 1e-8
relative, poses and points within 1e-8, intrinsics within 1e-8 relative.  The sum over shards adds the same terms as the
unsharded solve in another order, which moves the reduced system by rounding only; these bars hold while no decision
lies within its rounding band, so every run stops by max_num_iterations or by a tolerance placed between two iterations,
and assert_clear checks on the unsharded trace that rho and the function-tolerance test are outside their bands
(tests/ba_harness.py).  Every rank must also make the same sequence of reductions (RankGroup.run), at least two per
iteration, and hold the same cameras: bit-identical where the bordered reduced system fits one 128-wide Cholesky panel
(D + 1 <= 128), since then every rank factors the same matrix with the same arithmetic.  Beyond one panel the trailing
updates of csrc/chol.cu accumulate with atomicAdd, so two factorisations of the same matrix may differ in the last bits;
there the cameras of the ranks agree within the same bars as against the unsharded run.

C3 (D = 2402, 10 iterations) widens the parameter bar by a derived term.  The shard sum evaluates the costs in another
order, so rho of each step carries the rounding band e_rho of tests/ba_harness.py, and an accepted step multiplies the
radius by a factor whose relative derivative in rho is at most 18: the radius of iteration k may differ by rad_k = sum
of 18 e_rho over the accepted steps before it.  The LM step d = -(H + D/radius)^-1 g moves by at most |d| times the
relative change of the radius, so the parameters may differ by 1e-8 + sum_k rad_k |d_k| (trace column 6).  Measured on
an H100 80GB HBM3: up to 7.9e-8 in a point at 8 ranks, varying between runs by a factor of about 5 (two unsharded runs
agree to 3e-11)."""
import numpy as np
import pytest

from oracle import ba_oracle as bo
from oracle import band_oracle
from tests.ba_harness import assert_clear, band_record, device_solve, options, radius_bar, trace_rows
from tests.emulated_ranks import run_shards
from tests.helpers import ba_case, banded_ba_case, far_points_first_case, to_dev
from vggsfm_b200.dist import shard_range

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("cuda_dev")]

DEV = "cuda:0"
C3 = (400, 4096, "SIMPLE_RADIAL", bo.INTR_SHARED)


def _sharded(c, K, o, band=False, **kw):
    """the solve on K emulated ranks: per rank device_solve's result (with the band hint it took)"""
    def body(r, lo, hi, hook):
        return dict(device_solve(c, DEV, lo, hi, options=o, allreduce=hook, **kw), band=band_record() if band else None)

    return run_shards(c["mask"].shape[1], K, body, device=DEV)


def _single_panel(c):
    dc, ns = bo.dims(c["model"], c["mode"])
    return c["mask"].shape[0] * dc + ns + 1 <= 128


def _check(res, ref, label="", bar=1e-8, exact_cameras=True):
    s0, tr0 = ref["s"], ref["trace"]
    for r, x in enumerate(res):
        s, tr = x["s"], x["trace"]
        what = (label, "rank", r, x["lo"], x["hi"])
        assert s.termination == s0.termination, (what, s.termination, s0.termination)
        assert s.iterations == s0.iterations and s.successful == s0.successful, (what, s.iterations, s0.iterations)
        assert np.array_equal(tr[:, 7], tr0[:, 7]), (what, tr[:, 7], tr0[:, 7])
        assert x["calls"] >= 2 * s.iterations, (what, x["calls"], s.iterations)
        assert np.isclose(s.final_cost, s0.final_cost, rtol=1e-9, atol=0, equal_nan=True), (what, s.final_cost,
                                                                                          s0.final_cost)
        assert np.allclose(tr[:, 2], tr0[:, 2], rtol=1e-8, atol=0, equal_nan=True), (what, tr[:, 2], tr0[:, 2])
        assert np.abs(x["poses"] - ref["poses"]).max() < bar, what
        assert np.all(np.abs(x["intr"] - ref["intr"]) <= bar * np.maximum(1.0, np.abs(ref["intr"]))), what
        assert x["points"].shape == (x["hi"] - x["lo"], 3), what
        if x["hi"] > x["lo"]:
            assert np.abs(x["points"] - ref["points"][x["lo"]:x["hi"]]).max() < bar, what
        if exact_cameras:
            assert np.array_equal(x["poses"], res[0]["poses"]) and np.array_equal(x["intr"], res[0]["intr"]), what
        else:
            assert np.abs(x["poses"] - res[0]["poses"]).max() < bar, what
            assert np.all(np.abs(x["intr"] - res[0]["intr"]) <= bar * np.maximum(1.0, np.abs(res[0]["intr"]))), what
    print(f"{label}: {s0.termination} after {s0.iterations} iterations on {len(res)} ranks "
          f"({[x['hi'] - x['lo'] for x in res]} tracks), {res[0]['calls']} reductions per rank")


def _run_case(c, K, o, param_const=None, point_const=None, label="", derived_bar=False):
    ref = device_solve(c, DEV, options=o, param_const=param_const, point_const=point_const)
    assert_clear(trace_rows(ref["trace"]), o)
    res, group = _sharded(c, K, o, param_const=param_const, point_const=point_const)
    bar = radius_bar(trace_rows(ref["trace"])) if derived_bar else 1e-8
    _check(res, ref, label, bar, _single_panel(c))
    if derived_bar:
        print(f"{label}: parameter bar {bar:.3g}")
    return ref, res


# ------------------------------------------------------------------------------------------------------------------

def test_one_rank_through_the_hook():
    """K = 1: the hook 'sums' one term, so the solve through it is the solve without it.  Bit-identical when two runs
    without the hook are (the Jacobian kernels accumulate with float atomics, whose order may vary between runs)."""
    c = ba_case(8, 256, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=11)
    o = options(max_num_iterations=8)[0]
    a, b = device_solve(c, DEV, options=o), device_solve(c, DEV, options=o)
    res, _ = _sharded(c, 1, o)
    x = dict(res[0])
    same = all(np.array_equal(a[k], b[k]) for k in ("poses", "intr", "points", "trace"))
    print("two runs without the hook bit-identical:", same)
    if same:
        for k in ("poses", "intr", "points", "trace"):
            assert np.array_equal(x[k], a[k]), k
        assert x["s"].final_cost == a["s"].final_cost and x["s"].iterations == a["s"].iterations
    assert_clear(trace_rows(a["trace"]), o)
    _check(res, a, "K=1")


@pytest.mark.parametrize("K", [2, 3, 4, 8])
def test_shards_match_unsharded(K):
    c = ba_case(12, 512, "SIMPLE_RADIAL", bo.INTR_SHARED, seed=3)
    _run_case(c, K, options(max_num_iterations=8)[0], label=f"12x512 K={K}")


@pytest.mark.parametrize("mode", [bo.INTR_CONST, bo.INTR_PER_FRAME, bo.INTR_SHARED])
@pytest.mark.parametrize("cam", ["SIMPLE_PINHOLE", "SIMPLE_RADIAL"])
def test_every_dims_layout(cam, mode):
    """every (dc, ns) layout of the reduced system and the small vector through the reductions"""
    c = ba_case(9, 300, cam, mode, seed=5)
    _run_case(c, 3, options(max_num_iterations=6)[0], label=f"9x300 {cam} mode={mode} K=3")


@pytest.mark.parametrize("N,K", [(100, 8), (64, 3)])
def test_ragged_and_empty_shards(N, K):
    """N = 100 over 8 ranks: six shards of 16, a tail of 4 and an empty one; N = 64 over 3: 32 / 32 / 0.  A rank
    without tracks takes part in every reduction and ends with the same cameras."""
    spans = [shard_range(N, r, K) for r in range(K)]
    assert spans[-1][0] == spans[-1][1] == N
    c = ba_case(8, N, "SIMPLE_RADIAL", bo.INTR_PER_FRAME, seed=13)
    _run_case(c, K, options(max_num_iterations=6)[0], label=f"8x{N} K={K}")


@pytest.mark.parametrize("mode", [bo.INTR_PER_FRAME, bo.INTR_SHARED])
def test_frame_seen_in_one_shard(mode):
    """frame 5 is observed by the first shard's tracks only: the other ranks see nothing of it and must still refine it
    (the frame-seen flags are summed over the ranks before the constant flags are set)"""
    c = ba_case(10, 256, "SIMPLE_RADIAL", mode, seed=7)
    K = 2
    lo, hi = shard_range(256, 0, K)
    mask = c["mask"].copy()
    mask[5, hi:] = False
    assert mask[5, lo:hi].sum() >= 20
    c = dict(c, mask=mask)
    ref, res = _run_case(c, K, options(max_num_iterations=6)[0], label=f"frame seen by one shard, mode={mode}")
    moved = np.abs(ref["poses"][5] - c["poses"][5]).max()
    assert moved > 1e-6, moved


def test_gradient_max_decides():
    """gradient_tolerance between the largest and the second largest point gradient of the 2nd iterate, cameras held
    constant (so the point gradients alone decide), and the largest point moved into the last shard: every other rank's
    own maximum is below the tolerance there, only the max reduction keeps them iterating"""
    c = ba_case(8, 256, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=11)
    S, N = c["mask"].shape
    dc, ns = bo.dims(c["model"], c["mode"])
    pc = np.ones(S * dc + ns, dtype=bool)
    probe = bo.LMOptions()
    probe.max_num_iterations, probe.gradient_tolerance, probe.function_tolerance = 6, 0.0, 0.0
    tr = []
    bo.lm_solve(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], c["mode"], param_const=pc,
                options=probe, trace=tr)
    assert [t["outcome"] for t in tr[:4]] == [1, 1, 1, 1], tr
    probe.max_num_iterations = 2
    p2, i2, x2, _ = bo.lm_solve(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], c["mode"],
                                param_const=pc, options=probe)
    g = np.abs(bo.build_blocks(p2, i2, x2, c["uv"], c["mask"], c["model"], c["mode"])["g_p"]).max(axis=1)
    top = np.argsort(g)
    gtol = float(np.sqrt(g[top[-1]] * g[top[-2]]))
    assert g[top[-1]] > 1.1 * gtol and g[top[-2]] < gtol / 1.1 and tr[2]["gmax"] < 1e-2 * gtol
    assert abs(tr[1]["gmax"] - g[top[-1]]) <= 1e-9 * g[top[-1]] and tr[0]["gmax"] > 10 * gtol
    order = np.concatenate([np.delete(np.arange(N), top[-1]), [top[-1]]])
    c = dict(c, points=c["points"][order].copy(), uv=c["uv"][:, order].copy(), mask=c["mask"][:, order].copy())
    o = options(gradient_tolerance=gtol, function_tolerance=0.0, max_num_iterations=10)[0]
    for K in (2, 4):
        ref, res = _run_case(c, K, o, param_const=pc, label=f"gradient K={K}")
        assert ref["s"].termination == "CONVERGENCE_GRADIENT" and ref["s"].iterations == 3, ref["s"]


@pytest.mark.parametrize("K,ptol", [(2, 0.0072), (2, 0.0054), (4, 0.0072)])
def test_parameter_tolerance_over_shards(K, ptol):
    """|x| summed over the shards: the far points sit in rank 0's shard, so a rank-local |x| would stop the ranks at
    different iterations.  The oracle places the stop (margin asserted as in test_dist_threads.py); the unsharded solve
    and every rank must stop there."""
    c = far_points_first_case()
    probe = bo.LMOptions()
    probe.max_num_iterations, probe.gradient_tolerance, probe.function_tolerance = 20, 0.0, 0.0
    probe.parameter_tolerance = ptol
    tr = []
    _, _, _, summ = bo.lm_solve(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], c["mode"],
                                options=probe, trace=tr)
    ratios = [t["step_norm"] / (ptol * (t["x_norm"] + ptol)) for t in tr if t["outcome"] != 2]
    assert summ["termination"] == "CONVERGENCE_PARAMETER" and ratios[-1] < 1.0 - 1e-6
    assert all(q > 1.0 + 1e-6 for q in ratios[:-1]), ratios
    o = options(parameter_tolerance=ptol, gradient_tolerance=0.0, function_tolerance=0.0, max_num_iterations=20)[0]
    ref, res = _run_case(c, K, o, label=f"parameter tolerance {ptol} K={K}")
    assert ref["s"].termination == "CONVERGENCE_PARAMETER" and ref["s"].iterations == summ["iterations"], ref["s"]
    assert [int(v) for v in ref["trace"][:, 7]] == [t["outcome"] for t in tr]


def test_nan_observation_in_one_shard():
    """a NaN observation under a valid mask in the last shard: the summed cost is NaN on every rank, every step is
    invalid, and all ranks end in FAILURE_INVALID_STEPS with the parameters they started from"""
    c = ba_case(8, 256, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=11)
    K = 3
    lo, hi = shard_range(256, K - 1, K)
    s, n = np.argwhere(c["mask"][:, lo:hi])[7]
    uv = c["uv"].copy()
    uv[s, lo + n, 1] = np.nan
    c = dict(c, uv=uv)
    o = options()[0]
    ref = device_solve(c, DEV, options=o)
    res, _ = _sharded(c, K, o)
    assert ref["s"].termination == "FAILURE_INVALID_STEPS"
    _check(res, ref, "NaN observation")
    for x in res:
        assert x["s"].iterations == o.max_num_consecutive_invalid_steps and np.all(x["trace"][:, 7] == 2)
        assert np.array_equal(x["poses"], c["poses"]) and np.array_equal(x["intr"], c["intr"])
        assert np.array_equal(x["points"], c["points"][x["lo"]:x["hi"]])


def test_banded_shards():
    """a banded (video-like) problem over 2 ranks: each rank's SYRK skips k-blocks by its own tracks' ranges while the
    factorisation stays dense (the reduced system is the sum over the ranks); the unsharded solve factors with the band
    Cholesky.  Both must agree."""
    c = banded_ba_case(128, 4096, "SIMPLE_RADIAL", bo.INTR_SHARED, life=20, seed=33)
    dc, ns = bo.dims(c["model"], c["mode"])
    o = options(max_num_iterations=5)[0]
    ref = device_solve(c, DEV, options=o)
    b = band_record()
    assert b["active"] and b["chol"] and b["tables"], b
    assert b["rb_range"].shape[0] >= 6 and (128 * dc) // 128 >= 4
    assert_clear(trace_rows(ref["trace"]), o)
    K = 2
    res, _ = _sharded(c, K, o, band=True)
    for x in res:
        b = x["band"]
        assert b["active"] == 1 and b["chol"] == 0 and b["tables"] == 0, (x["lo"], b)
        t = band_oracle.band_tables(c["mask"][:, x["lo"]:x["hi"]], dc, ns)
        assert np.array_equal(b["rb_range"], t["rb_range"]), (x["lo"], b["rb_range"], t["rb_range"])
    assert not np.array_equal(res[0]["band"]["rb_range"], res[1]["band"]["rb_range"])
    assert not _single_panel(c)
    _check(res, ref, "banded 128x4096 K=2", exact_cameras=False)


@pytest.mark.parametrize("K", [2, 8])
def test_c3(K):
    """400 x 4096 SIMPLE_RADIAL shared intrinsics over 2 and 8 ranks, 10 iterations: the configurations of the
    benchmark's multi-GPU runs"""
    S, N, cam, mode = C3
    c = ba_case(S, N, cam, mode, seed=0, invisible_frac=0.0)
    o = options(max_num_iterations=10)[0]
    ref, res = _run_case(c, K, o, label=f"C3 K={K}", derived_bar=True)
    again = device_solve(c, DEV, options=o)
    print(f"C3 K={K}: largest difference to the unsharded run: poses "
          f"{max(np.abs(x['poses'] - ref['poses']).max() for x in res):.3g}, points "
          f"{max(np.abs(x['points'] - ref['points'][x['lo']:x['hi']]).max() for x in res):.3g}; "
          f"two unsharded runs: poses {np.abs(again['poses'] - ref['poses']).max():.3g}, points "
          f"{np.abs(again['points'] - ref['points']).max():.3g}")


def _ba_sharded(c, K, o, mask):
    """bundle_adjustment() of every rank's track shard: per rank (points, extrinsics, K, extra, global valid index,
    iterations, termination, hook calls)"""
    return run_shards(mask.shape[1], K, lambda r, lo, hi, hook: _ba(c, lo, hi, mask, o, hook) + (hook.calls,),
                      device=DEV)[0]


def _ba(c, lo, hi, mask, o, hook=None):
    import torch
    from vggsfm_b200 import bundle_adjustment as ba
    dev = DEV
    extra = to_dev(c["extra"], dev) if c["extra"] is not None else None
    pts, extr, K, ex, vidx, summ = ba.bundle_adjustment(
        to_dev(c["points"][lo:hi], dev), to_dev(c["poses"], dev), to_dev(c["K"], dev), extra,
        to_dev(c["uv"][:, lo:hi], dev, torch.float32), to_dev(mask[:, lo:hi], dev), shared_camera=False,
        camera_type="SIMPLE_RADIAL", options=o, allreduce=hook)
    torch.cuda.current_stream().synchronize()
    return (pts.cpu().numpy(), extr.cpu().numpy(), K.cpu().numpy(), ex.cpu().numpy(), lo + vidx.cpu().numpy(),
            summ.iterations, summ.termination)


@pytest.mark.parametrize("S,N,K", [(12, 512, 2), (8, 100, 8)])
def test_bundle_adjustment_sharded(S, N, K):
    """bundle_adjustment() with a sharded all-reduce, outputs compared with the unsharded call by global track index.
    At 8 x 100 over 8 ranks the 4 tracks of rank 6 keep one observation each (no valid track) and rank 7 has none."""
    c = ba_case(S, N, "SIMPLE_RADIAL", bo.INTR_PER_FRAME, seed=17)
    mask = c["mask"].copy()
    if K == 8:
        lo, hi = shard_range(N, 6, K)
        assert (lo, hi) == (96, 100) and shard_range(N, 7, K) == (100, 100)
        mask[1:, lo:hi] = False
        mask[0, lo:hi] = True
    o = options(max_num_iterations=6)[0]
    ref = _ba(c, 0, N, mask, o)
    res = _ba_sharded(c, K, o, mask)
    pos = {int(g): j for j, g in enumerate(ref[4])}
    assert sorted(np.concatenate([x[4] for x in res]).tolist()) == sorted(pos)
    for r, x in enumerate(res):
        assert x[5] == ref[5] and x[6] == ref[6] and x[7] >= 2 * x[5], (r, x[5:], ref[5:])
        assert np.abs(x[1] - ref[1]).max() < 1e-8, r
        assert np.all(np.abs(x[2] - ref[2]) <= 1e-8 * np.maximum(1.0, np.abs(ref[2]))), r
        assert np.abs(x[3] - ref[3]).max() < 1e-8, r
        if len(x[4]):
            assert np.abs(x[0] - ref[0][[pos[int(g)] for g in x[4]]]).max() < 1e-8, r
        assert np.array_equal(x[1], res[0][1]) and np.array_equal(x[2], res[0][2])
    if K == 8:
        assert len(res[6][4]) == 0 and len(res[7][4]) == 0

