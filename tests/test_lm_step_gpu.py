"""One LM iteration of vgg_ba_solve against the oracle's damped system at the start point.

The whole-solve tests (test_ba_gpu.py, test_video_c5_gpu.py) compare costs, and Levenberg-Marquardt corrects itself: a
wrong Schur complement, camera step or point step still reaches the same minimum, only in more iterations.  Here the
solver runs ONE iteration from a perturbed start and the step it took is read back from the parameters it updated in
place.  That step is checked in the FULL damped system (cameras and points, Jacobi-scaled variables, constant parameters
and points removed, built by oracle/ba_oracle.py from the same blocks the oracle's own LM uses), by its normwise
backward error

    eta = |H d + g|_inf / (|H|_inf (|d|_inf + |u|_inf) + |g|_inf)  <=  1e-12,

u being the rounding of the parameter update it was recovered from (2^-52 max(|old|, |new|) per entry).  A dropped
coupling block or observation gives eta of 1e-4 or more; rounding gives about 1e-15.  Also checked: the initial cost,
the model change and the step norm the solver reported (trace columns 3 and 6) at the recovered step, and the candidate
cost (column 2) against the oracle's cost at the returned parameters.

Banded (video-like) problems run with the band hint on (points in creation order) and off (the same problem with its
points in random order, which leaves the detection nothing to skip); each run is checked against the oracle on its
own, and the hint the solver computed is read back through a development probe and compared with
oracle/band_oracle.py table by table."""
import numpy as np
import pytest

from oracle import ba_oracle as bo
from oracle import band_oracle
from tests.ba_harness import band_record, check_one_step, device_solve, options
from tests.helpers import ba_case, banded_ba_case, shuffled_twin

pytestmark = pytest.mark.gpu


def _oracle_step(ref):
    """the oracle's own scaled step (Schur complement + Cholesky) and the 2-norm condition number of the reduced matrix"""
    A, B, V, fc = ref["A"], ref["B"], ref["V"], ref["fc"]
    N = V.shape[0]
    Vi = np.linalg.inv(V)
    T = np.einsum("dnk,nkj->dnj", B.reshape(-1, N, 3), Vi).reshape(B.shape)
    Sred = (A - T @ B.T)[np.ix_(fc, fc)]
    b = (-ref["gcs"] + T @ ref["gps"].reshape(-1))[fc]
    Lc = np.linalg.cholesky(Sred)
    dcs = np.zeros(A.shape[0])
    dcs[fc] = np.linalg.solve(Lc.T, np.linalg.solve(Lc, b))
    dps = np.einsum("nij,nj->ni", Vi, -ref["gps"] - (B.T @ dcs).reshape(N, 3))
    ev = np.linalg.eigvalsh(Sred)
    return dcs, dps, ev[-1] / ev[0]


def _check_band(c, band):
    """banded problem: the hint the solver took equals band_oracle.band_tables; band None or "shuffled" = dense expected"""
    rec = band_record()
    if band in (None, "shuffled"):
        assert not (rec["active"] or rec["chol"] or rec["tables"]), rec
        return
    dc, ns = bo.dims(c["model"], c["mode"])
    t = band_oracle.band_tables(c["mask"], dc, ns)
    assert rec["active"] and rec["chol"] and rec["tables"], rec
    assert np.array_equal(rec["rb_range"], t["rb_range"])
    assert np.array_equal(rec["end_blk"], t["end_blk"]) and rec["arrow_blk"] == t["arrow_blk"]
    assert np.array_equal(rec["kb_rows"], t["kb_rows"])
    assert np.array_equal(rec["fg_tracks"], t["fg_tracks"])


def _one_step(c, dev, param_const=None, point_const=None, label=""):
    """run one LM iteration on the GPU and check it against the oracle's system (tests/ba_harness.py
    check_one_step); prints the forward error against the oracle's own step"""
    S, N = c["mask"].shape
    if param_const is None:
        param_const = bo.default_param_const(S, c["model"], c["mode"])
    if point_const is None:
        point_const = np.zeros(N, dtype=bool)
    o, _ = options(max_num_iterations=1, function_tolerance=0.0, gradient_tolerance=0.0, parameter_tolerance=0.0)
    got = device_solve(c, dev, param_const=param_const, point_const=point_const, options=o)
    step = check_one_step(c, got, param_const, point_const, label=label)
    dcs, dps = step["dcs"], step["dps"]
    ref_dcs, ref_dps, kappa = _oracle_step(step["ref"])
    fwd = max(np.abs(dcs - ref_dcs).max(), np.abs(dps - ref_dps).max()) / max(np.abs(ref_dcs).max(), np.abs(ref_dps).max())
    print(f"lm step {label}: forward error vs oracle step = {fwd:.2e}  kappa2(reduced) = {kappa:.2e}")
    return step["eta"]


def _dense_case(name):
    if name == "8x256":          # D = 56: one trsv block, factorisation order 57
        return ba_case(8, 256, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=21), None, None
    if name == "64x1000":        # D = 448 = 7 x 64: the last trsv block is full
        return ba_case(64, 1000, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=22), None, None
    if name == "45x700":         # frame group 1 has nf = 13 frames of dc = 7: W goes out with plain stores
        c = ba_case(45, 700, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=23)
        const_pose = np.zeros(45, dtype=bool)
        const_pose[40] = True
        pc = bo.default_param_const(45, c["model"], c["mode"], const_pose=const_pose)
        ptc = np.zeros(700, dtype=bool)
        ptc[::7] = True
        return c, pc, ptc
    if name == "C3":             # the benchmark configuration
        return ba_case(400, 4096, "SIMPLE_RADIAL", bo.INTR_SHARED, seed=0, invisible_frac=0.0), None, None
    raise KeyError(name)


def _banded_case(name, mask_seed=0):
    if name == "160x4003":
        # partial last k block (3 N % 64 != 0) and partial last 32-track z_build tile; frame 77 sees nothing, point 1234
        # is seen by no frame, and point 5 is also seen by the last 3 frames (one long track widens the ranges)
        c = banded_ba_case(160, 4003, "SIMPLE_RADIAL", bo.INTR_SHARED, life=24, seed=31, mask_seed=mask_seed)
        c["mask"][77] = False
        c["mask"][:, 1234] = False
        c["mask"][-3:, 5] = True
        return c
    if name == "130x2500":       # dc = 7: frames straddle the 128-row blocks; no shared columns
        return banded_ba_case(130, 2500, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, life=20, seed=32, mask_seed=mask_seed)
    if name == "128x2048":       # S dc = 768: the arrow starts exactly at a block boundary, ns = 0
        return banded_ba_case(128, 2048, "SIMPLE_RADIAL", bo.INTR_CONST, life=20, seed=33, mask_seed=mask_seed)
    raise KeyError(name)


@pytest.mark.parametrize("name", ["8x256", "64x1000", "45x700", "C3"])
def test_dense_step_matches_oracle(cuda_dev, name):
    c, pc, ptc = _dense_case(name)
    _one_step(c, cuda_dev, pc, ptc, label=name)
    _check_band(c, None)


@pytest.mark.parametrize("band", ["shuffled", "1"])
@pytest.mark.parametrize("name", ["160x4003", "130x2500", "128x2048"])
def test_banded_step_matches_oracle(cuda_dev, name, band):
    """band "1": points in creation order (hint on); "shuffled": the shuffled twin (hint off)"""
    c = _banded_case(name)
    if band == "shuffled":
        c = shuffled_twin(c)
    _one_step(c, cuda_dev, label=f"{name} band hint {'on' if band == '1' else 'off (shuffled)'}")
    _check_band(c, band)


def test_back_to_back_band_dense_band(cuda_dev):
    """One process, one workspace: banded, then dense, then banded with another mask (a new hint): the workspace cache,
    the SYRK work-list cache and the thread-local band tables must follow."""
    c = _banded_case("160x4003", mask_seed=0)
    _one_step(c, cuda_dev, label="160x4003 first")
    _check_band(c, "1")
    c, pc, ptc = _dense_case("45x700")
    _one_step(c, cuda_dev, pc, ptc, label="45x700 between")
    _check_band(c, None)
    c = _banded_case("160x4003", mask_seed=7)
    _one_step(c, cuda_dev, label="160x4003 second mask")
    _check_band(c, "1")
