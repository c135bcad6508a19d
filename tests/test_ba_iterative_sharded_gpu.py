"""ITERATIVE_SCHUR over track shards (vgg_ba_solve_iterative_sharded) on one GPU: K ranks emulated by K host threads
(tests/emulated_ranks.py), each with its own stream, shard, iterative workspace and DeviceAllReduce, against the
unsharded iterative CUDA solve of the same problem.

Every rank must take the unsharded run's decisions: the same termination, LM iterations and per-iteration outcome (trace
column 7), and per LM iteration the same CG iteration count and CG termination (cg_trace columns 0 and 1).  The shard
sum adds the same terms as the unsharded solve in another order, so the reduced system, and with it every CG scalar,
moves by rounding only.  The decisions are clear of that rounding where the unsharded run places them away from their
thresholds: assert_clear (tests/ba_harness.py) checks rho and the function-tolerance test as test_ba_sharded_gpu.py
does, and every CG stop by SUCCESS has its last zeta at least 1e-6 below eta.  The zetas of the iterations before the
stop are not in the trace; that no one of them sat within rounding of eta is what the exact match of the CG iteration
counts checks.

Values are not held to test_ba_sharded_gpu.py's bars (1e-9 / 1e-8): CG iterates are not forward stable, and a
rounding-level change of the reduced system grows with the CG iteration count and then through the LM iterations that
follow.  tests/test_ba_iterative_shard_oracle.py shows it in float64 without any GPU: 5e-7 relative in a candidate cost
after 25 CG iterations at C1 between one and two ranks.  Measured on an H100 80GB HBM3 at 10 LM iterations: 4e-6
relative in the final cost at C3 between sharded and unsharded runs, 2e-5 between two unsharded runs.  The bars are
therefore costs within 1e-5 relative and parameters within 1e-4 (intrinsics relative); the decisions, the CG iteration
counts and the bit-identity across ranks are what the sharding must keep exactly.

The unsharded iterative solve is not bit-reproducible itself (its kernels add with float atomics): two unsharded C3 runs
end 2.3e-5 relative apart after 10 LM iterations, and a small ill-conditioned problem (9 x 300 SIMPLE_RADIAL with shared
intrinsics) can take a different CG iteration count from its second LM iteration on.  The cases therefore run the first
few LM iterations (3, C2 and the banded problem more), and the small layouts leave out that pair, which C3 covers.

Across the ranks the CG state is formed from summed data only, by fixed-order reductions, so cg_trace, the outcomes and
the cameras must be bit-identical.  Trace columns summed by camera-side atomics outside the CG (the step norm, column 6)
agree within rounding, as in the direct path.  Every rank makes the same sequence of reductions (RankGroup.run), and as
many as the chunk schedule says: three before the loop, and per LM iteration one for the assembly, eleven per queued
CG chunk (ten matvecs and the residual reset's) and two for the candidate."""
import ctypes

import numpy as np
import pytest

from oracle import ba_oracle as bo
from tests.ba_harness import assert_clear, device_solve, options, radius_bar, trace_rows
from tests.emulated_ranks import run_shards
from tests.helpers import ba_case, banded_ba_case, shuffled_twin, to_dev
from vggsfm_b200.dist import shard_range

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("cuda_dev")]

DEV = "cuda:0"
COST_BAR = 1e-5
PARAM_BAR = 1e-4
CHUNK = 10


def _solve(c, o, max_cg=500, **kw):
    return device_solve(c, DEV, options=o, linear_solver="ITERATIVE_SCHUR", max_linear_solver_iterations=max_cg, **kw)


def expected_calls(cg, max_cg):
    """hook calls of one rank: the frame flags and the initial cost and gradient maximum, then per LM iteration the
    assembly, 11 per queued chunk and the candidate's sum and maximum.  pcg_run queues the chunk after the one the CG
    stopped in before it reads the stop flag."""
    nchunks = (max(1, max_cg) + CHUNK - 1) // CHUNK
    calls = 3
    for n in cg[:, 0].astype(int):
        stop_chunk = max(0, (n - 1) // CHUNK)
        calls += 1 + 11 * min(stop_chunk + 2, nchunks) + 2
    return calls


def _check(res, ref, label="", bar=1e-4, max_cg=500):
    s0, tr0, cg0 = ref["s"], ref["trace"], ref["cg"]
    for r, x in enumerate(res):
        s, tr, cg = x["s"], x["trace"], x["cg"]
        what = (label, "rank", r, x["lo"], x["hi"])
        assert s.termination == s0.termination, (what, s.termination, s0.termination)
        assert s.iterations == s0.iterations and s.successful == s0.successful, (what, s.iterations, s0.iterations)
        assert np.array_equal(tr[:, 7], tr0[:, 7]), (what, tr[:, 7], tr0[:, 7])
        assert np.array_equal(cg[:, :2], cg0[:, :2]), (what, cg[:, :2], cg0[:, :2])
        assert x["calls"] == expected_calls(cg, max_cg), (what, x["calls"], expected_calls(cg, max_cg))
        assert np.isclose(s.final_cost, s0.final_cost, rtol=COST_BAR, atol=0, equal_nan=True), (what, s.final_cost,
                                                                                              s0.final_cost)
        assert np.allclose(tr[:, 2], tr0[:, 2], rtol=COST_BAR, atol=0, equal_nan=True), (what, tr[:, 2], tr0[:, 2])
        fin = np.isfinite(ref["poses"])
        assert np.abs(x["poses"] - ref["poses"])[fin].max() < bar, what
        assert np.array_equal(x["poses"][~fin], ref["poses"][~fin]), what
        assert np.all(np.abs(x["intr"] - ref["intr"]) <= bar * np.maximum(1.0, np.abs(ref["intr"]))), what
        assert x["points"].shape == (x["hi"] - x["lo"], 3), what
        if x["hi"] > x["lo"]:
            d = np.abs(x["points"] - ref["points"][x["lo"]:x["hi"]])
            assert np.nanmax(np.where(np.isfinite(ref["points"][x["lo"]:x["hi"]]), d, 0.0)) < bar, what
        # the fixed-order CG reductions: one CG state on every rank
        assert np.array_equal(cg, res[0]["cg"]), (what, "cg_trace differs between ranks")
        assert np.array_equal(tr[:, 7], res[0]["trace"][:, 7]) and np.array_equal(tr[:, 5], res[0]["trace"][:, 5]), what
        assert np.array_equal(x["poses"], res[0]["poses"]) and np.array_equal(x["intr"], res[0]["intr"]), \
            (what, "cameras differ between ranks")
        assert np.allclose(tr[:, 6], res[0]["trace"][:, 6], rtol=1e-12, atol=0, equal_nan=True), what
    dp = max(np.nanmax(np.abs(x["poses"] - ref["poses"])) for x in res)
    dc = max(abs(x["s"].final_cost - s0.final_cost) / s0.final_cost for x in res)
    print(f"{label}: largest difference to the unsharded run: poses {dp:.3g}, final cost {dc:.3g} relative")
    print(f"{label}: {s0.termination} after {s0.iterations} LM it, {int(cg0[:, 0].sum())} CG it on {len(res)} ranks "
          f"({[x['hi'] - x['lo'] for x in res]} tracks), {res[0]['calls']} reductions per rank")


def _run_case(c, K, o, label="", derived_bar=False, max_cg=500, **kw):
    ref = _solve(c, o, max_cg=max_cg, **kw)
    assert_clear(trace_rows(ref["trace"]), o, cg=ref["cg"])
    res, _ = run_shards(c["mask"].shape[1], K,
                        lambda r, lo, hi, hook: _solve(c, o, max_cg, lo=lo, hi=hi, allreduce=hook, **kw), device=DEV)
    bar = max(PARAM_BAR, radius_bar(trace_rows(ref["trace"]))) if derived_bar else PARAM_BAR
    _check(res, ref, label, bar, max_cg)
    return ref, res


# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("K", [2, 3, 8])
def test_c2(K):
    c = ba_case(50, 2048, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=1)
    _run_case(c, K, options(max_num_iterations=10)[0], label=f"C2 K={K}")


@pytest.mark.parametrize("K", [2, 3, 8])
def test_c3(K):
    """400 x 4096 SIMPLE_RADIAL shared intrinsics with prepare_ba_options and at most 200 CG iterations per step"""
    from vggsfm_b200 import bundle_adjustment as ba
    c = ba_case(400, 4096, "SIMPLE_RADIAL", bo.INTR_SHARED, seed=0, invisible_frac=0.0)
    o = ba.prepare_ba_options()
    o.max_num_iterations = 3
    _run_case(c, K, o, label=f"C3 K={K}", derived_bar=True, max_cg=200)


@pytest.mark.parametrize("shuffled", [False, True])
@pytest.mark.parametrize("K", [2, 3, 8])
def test_banded(K, shuffled):
    """banded 160 x 4003: each rank's kernels skip frame groups by its own tracks' ranges; the shuffled twin has no
    band to skip"""
    c = banded_ba_case(160, 4003, "SIMPLE_RADIAL", bo.INTR_SHARED, life=24, seed=31)
    if shuffled:
        c = shuffled_twin(c)
    _run_case(c, K, options(max_num_iterations=5)[0], label=f"banded shuffled={shuffled} K={K}")


PAIRS = [("SIMPLE_PINHOLE", bo.INTR_CONST), ("SIMPLE_PINHOLE", bo.INTR_PER_FRAME), ("SIMPLE_PINHOLE", bo.INTR_SHARED),
         ("SIMPLE_RADIAL", bo.INTR_CONST), ("SIMPLE_RADIAL", bo.INTR_PER_FRAME), ("SIMPLE_RADIAL", bo.INTR_SHARED)]


@pytest.mark.parametrize("cam,mode", PAIRS[:5])
@pytest.mark.parametrize("K", [2, 3, 8])
def test_every_dims_layout(K, cam, mode):
    """five (dc, ns) layouts at 9 x 300; the sixth, SIMPLE_RADIAL with shared intrinsics, is C3's (module docstring)"""
    c = ba_case(9, 300, cam, mode, seed=5)
    _run_case(c, K, options(max_num_iterations=3)[0], label=f"9x300 {cam} mode={mode} K={K}")


@pytest.mark.parametrize("K", [2, 3, 8])
def test_cauchy_with_outliers(K):
    """CAUCHY at 1 px with about 10 % of the observations moved by 20-60 px"""
    c = ba_case(12, 512, "SIMPLE_RADIAL", bo.INTR_PER_FRAME, seed=23)
    rng = np.random.default_rng(23)
    uv = c["uv"].copy()
    bad = c["mask"] & (rng.random(c["mask"].shape) < 0.1)
    uv[bad] += rng.uniform(20, 60, (int(bad.sum()), 2)) * rng.choice([-1.0, 1.0], (int(bad.sum()), 2))
    c = dict(c, uv=uv)
    _run_case(c, K, options(max_num_iterations=3)[0], label=f"CAUCHY K={K}", loss=("CAUCHY", 1.0))


@pytest.mark.parametrize("K", [2, 3, 8])
def test_constant_unobserved_and_hidden(K):
    """a constant pose, constant points, a frame and a point nothing sees, and NaN / inf hidden in the unseen frame's
    pose, the unseen point and masked uv"""
    c = ba_case(10, 400, "SIMPLE_RADIAL", bo.INTR_PER_FRAME, seed=29)
    mask = c["mask"].copy()
    mask[6] = False
    mask[:, 123] = False
    uv, poses, pts = c["uv"].copy(), c["poses"].copy(), c["points"].copy()
    uv[~mask] = np.nan
    poses[6] = np.inf
    pts[123] = np.nan
    c = dict(c, mask=mask, uv=uv, poses=poses, points=pts)
    const_pose = np.zeros(10, bool)
    const_pose[3] = True
    pc = bo.default_param_const(10, c["model"], c["mode"], const_pose=const_pose)
    ptc = np.zeros(400, bool)
    ptc[::7] = True
    ref, res = _run_case(c, K, options(max_num_iterations=3)[0], label=f"edges K={K}", param_const=pc,
                         point_const=ptc)
    for x in res:
        assert np.all(np.isinf(x["poses"][6])) and np.array_equal(x["poses"][3], c["poses"][3])
        held = ptc[x["lo"]:x["hi"]] | ~mask[:, x["lo"]:x["hi"]].any(axis=0)
        assert np.array_equal(x["points"][held], c["points"][x["lo"]:x["hi"]][held], equal_nan=True)


@pytest.mark.parametrize("N,K", [(100, 8), (64, 3)])
def test_empty_shard(N, K):
    """a rank without tracks solves 16 masked padding tracks and makes every reduction"""
    spans = [shard_range(N, r, K) for r in range(K)]
    assert spans[-1][0] == spans[-1][1] == N
    c = ba_case(8, N, "SIMPLE_RADIAL", bo.INTR_PER_FRAME, seed=13)
    _run_case(c, K, options(max_num_iterations=3)[0], label=f"8x{N} K={K}")


def _ba(c, lo, hi, mask, o, hook=None):
    import torch
    from vggsfm_b200 import bundle_adjustment as ba
    dev = DEV
    pts, extr, K, ex, vidx, summ = ba.bundle_adjustment(
        to_dev(c["points"][lo:hi], dev), to_dev(c["poses"], dev), to_dev(c["K"], dev), to_dev(c["extra"], dev),
        to_dev(c["uv"][:, lo:hi], dev, torch.float32), to_dev(mask[:, lo:hi], dev), shared_camera=False,
        camera_type="SIMPLE_RADIAL", options=o, allreduce=hook, linear_solver_type="ITERATIVE_SCHUR")
    torch.cuda.current_stream().synchronize()
    return (pts.cpu().numpy(), extr.cpu().numpy(), K.cpu().numpy(), ex.cpu().numpy(), lo + vidx.cpu().numpy(),
            summ.iterations, summ.termination, summ.cg_trace.numpy().copy())


@pytest.mark.parametrize("S,N,K", [(12, 512, 2), (8, 100, 8)])
def test_bundle_adjustment_sharded(S, N, K):
    """bundle_adjustment(..., ITERATIVE_SCHUR, allreduce=hook) on track shards against the unsharded call, by global
    track index; at 8 x 100 over 8 ranks rank 6 keeps no valid track and rank 7 has none"""
    c = ba_case(S, N, "SIMPLE_RADIAL", bo.INTR_PER_FRAME, seed=17)
    mask = c["mask"].copy()
    if K == 8:
        lo, hi = shard_range(N, 6, K)
        mask[1:, lo:hi] = False
        mask[0, lo:hi] = True
    o = options(max_num_iterations=3)[0]
    ref = _ba(c, 0, N, mask, o)
    res, _ = run_shards(N, K, lambda r, lo, hi, hook: _ba(c, lo, hi, mask, o, hook), device=DEV)
    pos = {int(g): j for j, g in enumerate(ref[4])}
    assert sorted(np.concatenate([x[4] for x in res]).tolist()) == sorted(pos)
    for r, x in enumerate(res):
        assert x[5] == ref[5] and x[6] == ref[6], (r, x[5:7], ref[5:7])
        assert np.array_equal(x[7][:, :2], ref[7][:, :2]) and np.array_equal(x[7], res[0][7]), r
        assert np.abs(x[1] - ref[1]).max() < PARAM_BAR, r
        assert np.all(np.abs(x[2] - ref[2]) <= PARAM_BAR * np.maximum(1.0, np.abs(ref[2]))), r
        assert np.abs(x[3] - ref[3]).max() < PARAM_BAR, r
        if len(x[4]):
            assert np.abs(x[0] - ref[0][[pos[int(g)] for g in x[4]]]).max() < PARAM_BAR, r
        assert np.array_equal(x[1], res[0][1]) and np.array_equal(x[2], res[0][2])


def test_fabric_hook_and_bad_arguments_are_refused(cuda_dev):
    import torch
    from vggsfm_b200 import _lib
    from vggsfm_b200 import bundle_adjustment as ba

    class FabricHook:
        fabric = object()

        def bind(self, ws):
            raise AssertionError("bound before the refusal")

    c = ba_case(8, 256, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=0)
    args = (to_dev(c["uv"], cuda_dev, torch.float32), to_dev(c["mask"], cuda_dev, torch.uint8),
            to_dev(c["poses"], cuda_dev), to_dev(c["intr"], cuda_dev), to_dev(c["points"], cuda_dev), c["model"],
            c["mode"])
    with pytest.raises(ValueError, match="AllReduceHook"):
        ba.lm_solve(*args, allreduce=FabricHook(), linear_solver_type="ITERATIVE_SCHUR")
    with pytest.raises(ValueError):
        ba.lm_solve(*args, allreduce=object(), linear_solver_type="ITERATIVE_SCHUR")
    with pytest.raises(ValueError, match="AllReduceHook"):
        ba.bundle_adjustment(to_dev(c["points"], cuda_dev), to_dev(c["poses"], cuda_dev), to_dev(c["K"], cuda_dev),
                             None, args[0], to_dev(c["mask"], cuda_dev), allreduce=FabricHook(),
                             linear_solver_type="ITERATIVE_SCHUR")
    L = _lib.lib()
    summ = _lib.BASummary()
    calls = []
    cb = _lib.ALLREDUCE_FN(lambda *a: calls.append(a) or 0)
    for lin in (ba.linear_solver("DENSE_SCHUR"), ba.linear_solver("ITERATIVE_SCHUR", 3, 2),
                ba.linear_solver("ITERATIVE_SCHUR", eta=0.0), ba.linear_solver("ITERATIVE_SCHUR", eta=float("inf"))):
        rc = L.vgg_ba_solve_iterative_sharded(None, None, ctypes.byref(lin), None, 0, cb, None, ctypes.byref(summ),
                                              None, None, None)
        assert rc == -1
    assert not calls


def test_joint_ba_2500_frames_two_ranks():
    """The final joint BA of the 2500-frame sequence (tools/video_c5.py) over 2 emulated ranks, 2 LM iterations with at
    most 50 CG iterations each: every rank takes the unsharded run's decisions"""
    import torch
    from tools.video_c5 import final_problem_arrays
    from vggsfm_b200 import bundle_adjustment as ba
    dev = torch.device("cuda:0")
    tracks, masks, xyz, extr, Kmat = final_problem_arrays(2500, 2048, dev=dev)
    S, P = masks.shape
    o = ba.default_options()
    o.max_num_iterations = 2

    def run(lo, hi, hook=None):
        *_, summ = ba.bundle_adjustment(xyz[lo:hi], extr, Kmat.expand(S, -1, -1), None, tracks[:, lo:hi],
                                        masks[:, lo:hi], shared_camera=True, options=o, filter_reconstruction=False,
                                        linear_solver_type="ITERATIVE_SCHUR", max_linear_solver_iterations=50,
                                        allreduce=hook, want_trace=True)
        torch.cuda.current_stream().synchronize()
        return summ

    ref = run(0, P)
    init = ref.initial_cost
    unsharded = (ref.iterations, ref.termination, ref.trace[:, 7].numpy().copy(), ref.cg_trace.numpy().copy(),
               ref.final_cost)
    del ref
    torch.cuda.empty_cache()
    res, _ = run_shards(P, 2, lambda r, lo, hi, hook: run(lo, hi, hook), device=dev)
    print(f"2500 x {P}: {unsharded[0]} LM it, CG {unsharded[3][:, 0].tolist()}, cost {init:.6g} -> "
          f"{unsharded[4]:.6g}")
    for s in res:
        assert (s.iterations, s.termination) == unsharded[:2]
        assert np.array_equal(s.trace[:, 7].numpy(), unsharded[2])
        assert np.array_equal(s.cg_trace.numpy()[:, :2], unsharded[3][:, :2])
        assert np.array_equal(s.cg_trace.numpy(), res[0].cg_trace.numpy())
        assert abs(s.final_cost - unsharded[4]) <= COST_BAR * unsharded[4]


def _nccl_worker(rank, world, port, q):
    import os
    import torch
    import torch.distributed as dist
    from vggsfm_b200 import bundle_adjustment as ba
    from vggsfm_b200.dist import AllReduceHook
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    c = ba_case(12, 512, "SIMPLE_RADIAL", bo.INTR_SHARED, seed=3)
    lo, hi = shard_range(512, rank, world)
    t = lambda a, dt=None: to_dev(a, dev, dt)
    poses, intr, pts = t(c["poses"]), t(c["intr"]), t(c["points"][lo:hi])
    hook = AllReduceHook()
    s = ba.lm_solve(t(c["uv"][:, lo:hi], torch.float32), t(c["mask"][:, lo:hi].astype(np.uint8)), poses, intr, pts,
                    c["model"], c["mode"], options=options(max_num_iterations=8)[0], allreduce=hook, want_trace=True,
                    linear_solver_type="ITERATIVE_SCHUR")
    q.put((rank, poses.cpu().numpy(), intr.cpu().numpy(), pts.cpu().numpy(), s.iterations, s.final_cost,
           s.cg_trace.numpy().copy(), hook.calls))
    dist.barrier()
    dist.destroy_process_group()


def test_two_gpu_nccl():
    """two processes over NCCL (skipped below two GPUs): both ranks reproduce the single-GPU run with identical
    cameras and CG traces"""
    import socket
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    s_ = socket.socket()
    s_.bind(("127.0.0.1", 0))
    port = s_.getsockname()[1]
    s_.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_nccl_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=300) for _ in range(2)], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    c = ba_case(12, 512, "SIMPLE_RADIAL", bo.INTR_SHARED, seed=3)
    ref = _solve(c, options(max_num_iterations=8)[0])
    for rank, poses, intr, pts, its, cost, cg, calls in res:
        lo, hi = shard_range(512, rank, 2)
        assert its == ref["s"].iterations and np.array_equal(cg[:, :2], ref["cg"][:, :2])
        assert np.array_equal(cg, res[0][6]) and np.array_equal(poses, res[0][1]) and np.array_equal(intr, res[0][2])
        assert abs(cost - ref["s"].final_cost) <= COST_BAR * ref["s"].final_cost
        assert np.abs(poses - ref["poses"]).max() < PARAM_BAR and np.abs(pts - ref["points"][lo:hi]).max() < PARAM_BAR
        assert calls == expected_calls(cg, 500)
