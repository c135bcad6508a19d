"""Float64 restatement of the ITERATIVE_SCHUR linear solver of the LM loop (csrc/ba_pcg.cu) and of the loop around it.

Ceres' IterativeSchurSolver with the SCHUR_JACOBI preconditioner, and its ConjugateGradientsSolver as
LevenbergMarquardtStrategy calls it (Ceres 2.x, [3P-memory]):

* x0 = 0, r = b, Q0 = 0; the r-tolerance is disabled (r_tolerance = -1) and q_tolerance = eta.
* iteration i: z = P r; rho = r.z (zero or infinite: FAILURE); p = z (i = 1) or z + beta p with beta = rho / rho_prev
  (zero or infinite: FAILURE); q = A p; p.q <= 0 or infinite: FAILURE (Ceres 2.2 reports NO_CONVERGENCE there; this
  project fails the step, so that an indefinite system never moves the parameters); alpha = rho / p.q (zero or infinite:
  FAILURE); x += alpha p; r = b - A x when i % 10 == 0, else r -= alpha q; Q1 = -x.(b + r);
  zeta = i (Q1 - Q0) / Q1 < eta with i >= min_iterations: SUCCESS; Q0 = Q1; i >= max_iterations: NO_CONVERGENCE.
* |b| = 0: SUCCESS with x = 0 and no iteration.

SCHUR_JACOBI takes the diagonal block of the (scaled, damped) Schur complement of each camera parameter block.  COLMAP
3.10's blocks [3P-memory]: the rotation (3 tangent parameters), the translation (3) and the camera's intrinsics --
per frame in INTR_PER_FRAME, one block shared by all frames in INTR_SHARED, none in INTR_CONST.  A constant parameter is
a pinned row: identity in A and in its block.  A block that is not positive definite fails the solve.

The LM loop is ba_oracle.lm_solve's on one GPU, with the model change of an inexact step taken as Ceres computes it,
-(J d)^T (f + J d / 2), instead of the exact-solve identity; the explicit Schur complement is fine at oracle sizes."""
from __future__ import annotations

import numpy as np

from . import ba_oracle as bo

SUCCESS, NO_CONVERGENCE, FAILURE = 0, 1, 2
RESET_PERIOD = 10


def _zero_or_inf(v):
    return v == 0.0 or np.isinf(v)


def parameter_blocks(S, dc, ns):
    """[(first row, size)] of the Schur-Jacobi blocks in the order csrc/ba_pcg.cu stores them: per frame rotation,
    translation, intrinsics (size 0 unless INTR_PER_FRAME), then the shared-intrinsics block (only if ns > 0)."""
    out = []
    for s in range(S):
        out += [(s * dc, 3), (s * dc + 3, 3), (s * dc + 6, dc - 6)]
    if ns:
        out.append((S * dc, ns))
    return out


def schur_jacobi(A, S, dc, ns):
    """(P, ok, blocks): P = the block-diagonal inverse of A over parameter_blocks (inverted through each block's
    Cholesky factor), ok = every block positive definite, blocks = [9]-padded inverses as the kernel stores them."""
    D = A.shape[0]
    P = np.zeros((D, D))
    ok = True
    store = []
    for r0, nb in parameter_blocks(S, dc, ns):
        B3 = np.eye(3)
        if nb:
            blk = A[r0:r0 + nb, r0:r0 + nb]
            try:
                L = np.linalg.cholesky(blk)
                Li = np.linalg.inv(L)
                inv = Li.T @ Li
            except np.linalg.LinAlgError:
                ok = False
                inv = np.zeros((nb, nb))
            P[r0:r0 + nb, r0:r0 + nb] = inv
            B3[:nb, :nb] = inv
            if not ok:
                B3[:] = 0.0
        store.append(B3)
    return P, ok, np.array(store)


def cg(A, b, P=None, eta=0.1, min_iterations=0, max_iterations=500, trace=None, precond_ok=True):
    """Ceres' ConjugateGradientsSolver as above.  Returns (x, summary) with summary = {iterations, termination, zeta,
    rrel}; `trace` (a list) receives one dict per iteration: rho, beta, pq, alpha, Q, zeta, rnorm."""
    D = len(b)
    P = np.eye(D) if P is None else P
    x = np.zeros(D)
    summ = {"iterations": 0, "termination": NO_CONVERGENCE, "zeta": 0.0, "rrel": 1.0}
    if not precond_ok:
        summ.update(termination=FAILURE, rrel=1.0 if np.dot(b, b) > 0 else 0.0)
        return x, summ
    bnorm = float(np.linalg.norm(b))
    if bnorm == 0.0:
        summ.update(termination=SUCCESS, rrel=0.0)
        return x, summ
    r = b.copy()
    p = np.zeros(D)
    rho = 1.0
    Q0 = 0.0
    i = 1
    while True:
        z = P @ r
        last_rho = rho
        rho = float(r @ z)
        rec = {"i": i, "rho": rho}
        if trace is not None:
            trace.append(rec)
        if _zero_or_inf(rho):
            summ.update(iterations=i, termination=FAILURE)
            break
        if i == 1:
            p = z.copy()
        else:
            beta = rho / last_rho
            rec["beta"] = beta
            if _zero_or_inf(beta):
                summ.update(iterations=i, termination=FAILURE)
                break
            p = z + beta * p
        q = A @ p
        pq = float(p @ q)
        alpha = rho / pq if pq != 0.0 else np.inf
        rec.update(pq=pq, alpha=alpha)
        if pq <= 0.0 or np.isinf(pq) or _zero_or_inf(alpha):
            summ.update(iterations=i, termination=FAILURE)
            break
        x = x + alpha * p
        if i % RESET_PERIOD == 0:
            r = b - A @ x
        else:
            r = r - alpha * q
        Q1 = float(-(x @ (b + r)))
        zeta = i * (Q1 - Q0) / Q1
        rec.update(Q=Q1, zeta=zeta, rnorm=float(np.linalg.norm(r)), eta_margin=zeta - eta)
        summ.update(iterations=i, zeta=zeta, rrel=float(np.linalg.norm(r)) / bnorm)
        if zeta < eta and i >= min_iterations:
            summ["termination"] = SUCCESS
            break
        Q0 = Q1
        if i >= max_iterations:
            summ["termination"] = NO_CONVERGENCE
            break
        i += 1
    return x, summ


def reduced_system(blk, Hc, gc, sc_c, sc_p, Hc_diag, param_const, point_const, radius, S, dc, ns,
                   min_diag=1e-6, max_diag=1e32):
    """The scaled, damped, pinned reduced camera system (A, b) of one LM step and the point-side pieces (M, dpp, dcc) the
    back-substitution needs -- the same algebra as ba_oracle.lm_solve."""
    N = blk["g_p"].shape[0]
    Hpp_s = blk["H_pp"] * sc_p[:, :, None] * sc_p[:, None, :]
    dpp = np.clip(np.einsum("nii->ni", Hpp_s), min_diag, max_diag)
    V = Hpp_s + np.einsum("ni,ij->nij", dpp / radius, np.eye(3))
    V[point_const] = np.eye(3)
    L = np.linalg.cholesky(V)
    M = sc_p[:, :, None] * np.transpose(np.linalg.inv(L), (0, 2, 1))
    M[point_const] = 0.0
    q = np.einsum("nji,nj->ni", M, blk["g_p"])
    W = bo._full_W(blk, S, dc, ns)
    Z = (W[:, :, 0:1] * M[None, :, 0, :] + W[:, :, 1:2] * M[None, :, 1, :] + W[:, :, 2:3] * M[None, :, 2, :]).reshape(-1, N * 3)
    S_raw = Hc - Z @ Z.T
    rhs_raw = -(gc - Z @ q.reshape(-1))
    dcc = np.clip(Hc_diag * sc_c * sc_c, min_diag, max_diag)
    A = S_raw * sc_c[:, None] * sc_c[None, :] + np.diag(dcc / radius)
    b = rhs_raw * sc_c
    A[param_const, :] = 0.0
    A[:, param_const] = 0.0
    A[param_const, param_const] = 1.0
    b[param_const] = 0.0
    return A, b, M, dpp, dcc, W


def jd_model_change(poses, intr, points, uv, mask, model, mode, d_c, d_p, point_const):
    """Ceres' model change -(J d)^T (f + J d / 2) over the observations (unscaled step d_c [D], d_p [N,3])."""
    S, N = mask.shape
    dc, ns = bo.dims(model, mode)
    res, Jc8, Jp = bo.residuals_and_jacobians(poses, intr, points, uv, mask, model)
    Jp = np.where(np.asarray(point_const, dtype=bool)[None, :, None, None], 0.0, Jp)
    dcam = d_c[:S * dc].reshape(S, dc)
    jd = np.einsum("snri,si->snr", Jc8[..., :dc], dcam) + np.einsum("snrk,nk->snr", Jp, d_p)
    if ns:
        jd = jd + np.einsum("snri,i->snr", Jc8[..., 6:6 + ns], d_c[S * dc:])
    jd = np.where(mask[..., None], jd, 0.0)
    return float(-np.sum(jd * (res + 0.5 * jd)))


def lm_solve(poses, intr, points, uv, mask, model, mode, param_const=None, point_const=None,
             options: bo.LMOptions | None = None, trace: list | None = None, linear_solver="iterative_schur",
             min_linear_solver_iterations=0, max_linear_solver_iterations=500, eta=0.1, cg_traces: list | None = None):
    """ba_oracle.lm_solve on one GPU with the linear solver chosen: "dense_schur" (Cholesky of the reduced system, the
    model change 0.5 * quad) or "iterative_schur" (the CG above, Ceres' J d model change).  `cg_traces` receives, per LM
    iteration, {"summary": CG summary, "trace": per-CG-iteration list}.  Returns (poses, intr, points, summary)."""
    assert linear_solver in ("dense_schur", "iterative_schur")
    iterative = linear_solver == "iterative_schur"
    opt = options or bo.LMOptions()
    S, N = mask.shape
    dc, ns = bo.dims(model, mode)
    D = S * dc + ns
    if param_const is None:
        param_const = bo.default_param_const(S, model, mode)
    if point_const is None:
        point_const = np.zeros(N, dtype=bool)
    mask = np.asarray(mask, dtype=bool)
    point_const = np.asarray(point_const, dtype=bool) | ~mask.any(axis=0)
    param_const = np.asarray(param_const, dtype=bool).copy()
    param_const[:S * dc] |= np.repeat(~mask.any(axis=1), dc)
    free_c = ~param_const

    def evaluate(poses, intr, points):
        blk = bo.build_blocks(poses, intr, points, uv, mask, model, mode, point_const)
        Hc, gc = bo._assemble_camera_system(blk, S, dc, ns)
        return blk, Hc, gc

    blk, Hc, gc = evaluate(poses, intr, points)
    cost = blk["cost"]
    Hc_diag = np.diag(Hc).copy()
    if opt.jacobi_scaling:
        sc_c = 1.0 / (1.0 + np.sqrt(Hc_diag))
        sc_p = 1.0 / (1.0 + np.sqrt(np.einsum("nii->ni", blk["H_pp"])))
    else:
        sc_c = np.ones(D)
        sc_p = np.ones((N, 3))

    def grad_max_norm(gc, gp):
        a = np.max(np.abs(gc[free_c])) if free_c.any() else 0.0
        b = np.max(np.abs(gp[~point_const])) if (~point_const).any() else 0.0
        return float(np.max([a, b]))

    radius = opt.initial_trust_region_radius
    decrease_factor = 2.0
    summary = {"iterations": 0, "successful": 0, "initial_cost": cost, "termination": "NO_CONVERGENCE"}
    if grad_max_norm(gc, blk["g_p"]) <= opt.gradient_tolerance:
        summary.update(termination="CONVERGENCE_GRADIENT", final_cost=cost)
        return poses, intr, points, summary
    invalid_steps = 0
    it = 0
    while True:
        if it >= opt.max_num_iterations:
            break
        if radius < opt.min_trust_region_radius:
            summary["termination"] = "MIN_TRUST_REGION_RADIUS"
            break
        it += 1
        A, b, M, dpp, dcc, W = reduced_system(blk, Hc, gc, sc_c, sc_p, Hc_diag, param_const, point_const, radius, S, dc,
                                              ns, opt.min_lm_diagonal, opt.max_lm_diagonal)
        ok = True
        if iterative:
            P, pok, _ = schur_jacobi(A, S, dc, ns)
            cgt = []
            dcs, cs = cg(A, b, P, eta, min_linear_solver_iterations, max_linear_solver_iterations, cgt, pok)
            if cg_traces is not None:
                cg_traces.append({"summary": cs, "trace": cgt})
            ok = cs["termination"] != FAILURE
        else:
            try:
                dcs = np.linalg.solve(np.linalg.cholesky(A).T, np.linalg.solve(np.linalg.cholesky(A), b))
            except np.linalg.LinAlgError:
                ok = False
        if ok and not np.all(np.isfinite(dcs)):
            ok = False
        model_change = np.nan
        if ok:
            d_c = dcs * sc_c
            w = np.tensordot(d_c, W, axes=(0, 0))
            d_p = np.einsum("nij,nj->ni", M, np.einsum("nji,nj->ni", M, -(blk["g_p"] + w)))
            d_p[point_const] = 0.0
            if iterative:
                model_change = jd_model_change(poses, intr, points, uv, mask, model, mode, d_c, d_p, point_const)
            else:
                dps = d_p / np.where(sc_p == 0, 1.0, sc_p)
                quad = (np.sum(dcs * dcs * dcc / radius * free_c) - np.sum(d_c * gc) +
                        np.sum(np.where(point_const[:, None], 0.0, dps * dps * dpp / radius)) - np.sum(d_p * blk["g_p"]))
                model_change = 0.5 * quad
        if not ok or not (model_change > 0):
            invalid_steps += 1
            if trace is not None:
                trace.append({"it": it, "outcome": 2, "cost": cost, "radius": radius, "model_change": model_change})
            if invalid_steps >= opt.max_num_consecutive_invalid_steps:
                summary["termination"] = "FAILURE_INVALID_STEPS"
                break
            radius *= 0.5
            continue
        invalid_steps = 0
        c_poses, c_intr, c_points = bo.apply_step(poses, intr, points, d_c[:S * dc].reshape(S, dc), d_c[S * dc:], d_p,
                                                  model, mode)
        c_blk, c_Hc, c_gc = evaluate(c_poses, c_intr, c_points)
        c_cost = c_blk["cost"]
        step_norm = float(np.sqrt(np.sum(d_c * d_c) + np.sum(d_p * d_p)))
        cost_change = cost - c_cost
        rho = cost_change / model_change
        rec = {"it": it, "cost": cost, "candidate_cost": c_cost, "model_change": model_change, "rho": rho,
               "radius": radius, "step_norm": step_norm, "outcome": 0}
        if trace is not None:
            trace.append(rec)
        x_cams, x_pts = bo._x_norm_parts(poses, intr, points, S, dc, ns, param_const, point_const)
        if step_norm <= opt.parameter_tolerance * (np.sqrt(x_cams + x_pts) + opt.parameter_tolerance):
            summary["termination"] = "CONVERGENCE_PARAMETER"
            break
        if abs(cost_change) <= opt.function_tolerance * cost:
            summary["termination"] = "CONVERGENCE_FUNCTION"
            break
        if rho > opt.min_relative_decrease:
            rec["outcome"] = 1
            poses, intr, points, cost = c_poses, c_intr, c_points, c_cost
            blk, Hc, gc = c_blk, c_Hc, c_gc
            Hc_diag = np.diag(Hc).copy()
            summary["successful"] += 1
            radius = min(opt.max_trust_region_radius, radius / max(1.0 / 3.0, 1.0 - (2.0 * rho - 1.0) ** 3))
            decrease_factor = 2.0
            if grad_max_norm(gc, blk["g_p"]) <= opt.gradient_tolerance:
                summary["termination"] = "CONVERGENCE_GRADIENT"
                break
        else:
            radius = radius / decrease_factor
            decrease_factor *= 2.0
    summary.update(iterations=it, final_cost=cost, final_radius=radius)
    return poses, intr, points, summary
