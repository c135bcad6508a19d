"""The ITERATIVE_SCHUR oracle (oracle/ba_pcg_oracle.py) against LAPACK, its own formulas and the direct oracle (no GPU)."""
import numpy as np
import pytest

from oracle import ba_oracle as bo
from oracle import ba_pcg_oracle as po
from tests.helpers import ba_case


def _spd(n, cond, seed):
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
    return (Q * np.geomspace(1.0, cond, n)) @ Q.T, rng.standard_normal(n)


def test_cg_n_iterations_equals_lapack():
    A, b = _spd(12, 50.0, 0)
    x, s = po.cg(A, b, eta=1e-300, max_iterations=12)
    ref = np.linalg.solve(A, b)
    assert np.max(np.abs(x - ref)) <= 1e-10 * np.max(np.abs(ref))
    assert s["termination"] in (po.SUCCESS, po.NO_CONVERGENCE) and s["iterations"] <= 12


def test_zeta_termination_at_formula_iteration():
    A, b = _spd(60, 1e3, 1)
    free = []
    po.cg(A, b, eta=-1.0, max_iterations=60, trace=free)          # never stops on zeta: the plain CG sequence
    Q = [0.0] + [t["Q"] for t in free]
    for eta, mn in ((0.1, 0), (0.1, 27), (0.05, 0)):
        expect = next(i for i in range(1, 61) if i * (Q[i] - Q[i - 1]) / Q[i] < eta and i >= mn)
        zetas = [i * (Q[i] - Q[i - 1]) / Q[i] for i in range(1, 61)]
        assert min(abs(z - eta) for z in zetas) > 1e-6        # no decision sits near its threshold
        _, s = po.cg(A, b, eta=eta, min_iterations=mn, max_iterations=60)
        assert s["iterations"] == expect and s["termination"] == po.SUCCESS


def test_residual_reset_every_ten_iterations():
    A, b = _spd(80, 1e6, 2)
    differs = False
    for n in range(1, 23):
        x, s = po.cg(A, b, eta=-1.0, max_iterations=n)
        true_r = np.linalg.norm(b - A @ x) / np.linalg.norm(b)
        if n % 10 == 0:
            assert s["rrel"] == true_r              # r = b - A x recomputed, bit for bit
        else:
            differs = differs or s["rrel"] != true_r
    assert differs                                  # the recurrence drifts between resets


@pytest.mark.parametrize("cam,mode", [("SIMPLE_PINHOLE", bo.INTR_PER_FRAME), ("SIMPLE_RADIAL", bo.INTR_SHARED),
                                      ("SIMPLE_RADIAL", bo.INTR_CONST), ("SIMPLE_RADIAL", bo.INTR_PER_FRAME)])
def test_schur_jacobi_blocks_are_the_block_diagonal(cam, mode):
    c = ba_case(8, 256, cam, mode, seed=5)
    S, N = c["mask"].shape
    dc, ns = bo.dims(c["model"], mode)
    A, b, M, *_ = _system(c)
    P, ok, store = po.schur_jacobi(A, S, dc, ns)
    assert ok
    blocks = po.parameter_blocks(S, dc, ns)
    assert len(blocks) == 3 * S + (1 if ns else 0)
    covered = np.zeros(S * dc + ns, dtype=int)
    for k, (r0, nb) in enumerate(blocks):
        covered[r0:r0 + nb] += 1
        if nb:
            blk = A[r0:r0 + nb, r0:r0 + nb]
            assert np.allclose(store[k][:nb, :nb] @ blk, np.eye(nb), atol=1e-10)
    assert (covered == 1).all()
    # P is block diagonal: nothing outside the blocks
    mask = np.zeros_like(P, dtype=bool)
    for r0, nb in blocks:
        mask[r0:r0 + nb, r0:r0 + nb] = True
    assert not P[~mask].any()


def _system(c, radius=1e4):
    S, N = c["mask"].shape
    dc, ns = bo.dims(c["model"], c["mode"])
    mask = c["mask"].astype(bool)
    pc = bo.default_param_const(S, c["model"], c["mode"])
    ptc = ~mask.any(axis=0)
    blk = bo.build_blocks(c["poses"], c["intr"], c["points"], c["uv"], mask, c["model"], c["mode"], ptc)
    Hc, gc = bo._assemble_camera_system(blk, S, dc, ns)
    hd = np.diag(Hc).copy()
    sc_c = 1.0 / (1.0 + np.sqrt(hd))
    sc_p = 1.0 / (1.0 + np.sqrt(np.einsum("nii->ni", blk["H_pp"])))
    return po.reduced_system(blk, Hc, gc, sc_c, sc_p, hd, pc, ptc, radius, S, dc, ns)


def test_zero_rho_and_indefinite_fail():
    A, b = _spd(6, 10.0, 3)
    _, s = po.cg(A, b, P=np.zeros((6, 6)))
    assert s["termination"] == po.FAILURE and s["iterations"] == 1
    _, s = po.cg(np.diag([1.0, -1.0]), np.array([0.0, 1.0]))
    assert s["termination"] == po.FAILURE
    _, s = po.cg(A, np.zeros(6))
    assert s["termination"] == po.SUCCESS and s["iterations"] == 0


def test_failed_cg_makes_the_lm_step_invalid(monkeypatch):
    c = ba_case(8, 256, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=0)
    real = po.cg
    calls = []

    def first_fails(A, b, P=None, *a, **k):
        calls.append(1)
        return real(A, b, np.zeros_like(A) if len(calls) == 1 else P, *a, **k)

    monkeypatch.setattr(po, "cg", first_fails)
    trace, cgs = [], []
    po.lm_solve(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], c["mode"],
                options=bo.LMOptions(max_num_iterations=2), trace=trace, cg_traces=cgs)
    assert cgs[0]["summary"]["termination"] == po.FAILURE and trace[0]["outcome"] == 2
    assert trace[1]["radius"] == trace[0]["radius"] * 0.5 and trace[1]["outcome"] != 2


def test_one_cg_iteration_is_used_with_the_jd_model_change():
    c = ba_case(8, 256, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=0)
    trace, cgs = [], []
    po.lm_solve(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], c["mode"],
                options=bo.LMOptions(max_num_iterations=1), trace=trace, cg_traces=cgs, max_linear_solver_iterations=1)
    assert cgs[0]["summary"]["termination"] == po.NO_CONVERGENCE and cgs[0]["summary"]["iterations"] == 1
    assert trace[0]["outcome"] == 1 and trace[0]["model_change"] > 0
    # the exact-solve identity would give another number for this inexact step
    tr_d = []
    po.lm_solve(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], c["mode"],
                options=bo.LMOptions(max_num_iterations=1), trace=tr_d, linear_solver="dense_schur")
    assert abs(trace[0]["model_change"] - tr_d[0]["model_change"]) > 1e-6 * tr_d[0]["model_change"]


def test_jd_model_change_equals_exact_identity_for_an_exact_step():
    """for the exact solve, -(J d)^T (f + J d / 2) = 0.5 (d^T D d - d^T g) (what the direct path uses)"""
    c = ba_case(8, 256, "SIMPLE_RADIAL", bo.INTR_SHARED, seed=4)
    tr_d, tr_i = [], []
    args = (c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], c["mode"])
    po.lm_solve(*args, options=bo.LMOptions(max_num_iterations=1), trace=tr_d, linear_solver="dense_schur")
    po.lm_solve(*args, options=bo.LMOptions(max_num_iterations=1), trace=tr_i, eta=1e-300,
                max_linear_solver_iterations=400)
    assert abs(tr_i[0]["model_change"] - tr_d[0]["model_change"]) <= 1e-9 * tr_d[0]["model_change"]


@pytest.mark.parametrize("mode", [bo.INTR_PER_FRAME, bo.INTR_SHARED])
def test_c1_iterative_reaches_the_direct_minimum(mode):
    c = ba_case(8, 256, "SIMPLE_PINHOLE", mode, seed=0)
    args = (c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], c["mode"])
    opt = bo.LMOptions(function_tolerance=1e-12, gradient_tolerance=1e-12, max_num_iterations=100)
    *_, sd = bo.lm_solve(*args, options=opt)
    *_, si = po.lm_solve(*args, options=opt)
    *_, sdd = po.lm_solve(*args, options=opt, linear_solver="dense_schur")
    assert abs(si["final_cost"] - sd["final_cost"]) <= 1e-9 * sd["final_cost"]
    assert abs(sdd["final_cost"] - sd["final_cost"]) <= 1e-12 * sd["final_cost"]


def test_iterative_workspace_has_no_grid_or_quadratic_term():
    """vgg_ba_workspace_bytes_iterative is linear in S and in N: its second differences stay within the 256-byte
    alignment of its ~30 buffers (plus one frame's bytes, S = 1 standing in for 0), and at S = 4000 it is a small
    fraction of the direct workspace."""
    from vggsfm_b200 import bundle_adjustment as ba
    S, N = 4000, 512000
    for model, mode in ((0, 0), (0, 1), (0, 2), (1, 0), (1, 1), (1, 2)):
        w = lambda s, n: ba.workspace_bytes(s, n, model, mode, iterative=True)
        assert abs(w(S, N) - 2 * w(S // 2, N) + w(1, N)) <= 64 * 256 + 2048
        assert abs(w(S, 2 * N) - 2 * w(S, N) + w(S, 16)) <= 64 * 256 + 2048
        assert w(S, N) < 300 * (8 * S + 3 * N)
        assert 100 * w(S, N) < ba.workspace_bytes(S, N, model, mode)
