"""Float64 restatement of ITERATIVE_SCHUR over track shards -- TEST INFRASTRUCTURE ONLY.

oracle/ba_pcg_oracle.py's lm_solve with the all-reduce of oracle/ba_oracle.py's lm_solve (``allreduce`` with ``.sum``
and ``.max``), in the order vgg_ba_solve_iterative_sharded reduces:

  * once per solve: the frames any rank sees (sum); the initial cost, camera gradient and diag(H_cc) (sum) and the
    gradient maximum (max);
  * once per LM iteration, one sum: the rank's H_cc, g_c, sum Z Z^T and sum Z q (the CUDA solve sums the preconditioner
    blocks and the right-hand side it builds from these, and multiplies by the Schur part of A per matvec instead of
    forming it: the same sums in another order);
  * per candidate: cost, the point part of |d|^2 and of |x|^2 and the J d model change (sum), the gradient maximum (max).

The CG then runs on the summed system exactly as the unsharded oracle's, the same code on every rank, so every rank
takes the same CG and LM decisions.  The files under oracle/ are not changed: this module reuses their pieces."""
from __future__ import annotations

import numpy as np

from oracle import ba_oracle as bo
from oracle import ba_pcg_oracle as po


def lm_solve(poses, intr, points, uv, mask, model, mode, param_const=None, point_const=None,
             options: bo.LMOptions | None = None, trace: list | None = None, min_linear_solver_iterations=0,
             max_linear_solver_iterations=500, eta=0.1, cg_traces: list | None = None, allreduce=None):
    """ba_pcg_oracle.lm_solve (iterative_schur) on this rank's tracks, reducing through `allreduce` (None: one rank,
    the unsharded solve).  Returns (poses, intr, points, summary); `trace` and `cg_traces` as ba_pcg_oracle's."""
    ar = allreduce.sum if allreduce is not None else (lambda a: np.asarray(a, dtype=np.float64))
    armax = allreduce.max if allreduce is not None else (lambda v: float(v))
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
    frame_seen = ar(mask.any(axis=1).astype(np.float64)) != 0.0
    param_const = np.asarray(param_const, dtype=bool).copy()
    param_const[:S * dc] |= np.repeat(~frame_seen, dc)
    free_c = ~param_const

    def evaluate(poses, intr, points):
        blk = bo.build_blocks(poses, intr, points, uv, mask, model, mode, point_const)
        Hc, gc = bo._assemble_camera_system(blk, S, dc, ns)
        return blk, Hc, gc

    def grad_max_norm(gc_glob, gp):
        a = np.max(np.abs(gc_glob[free_c])) if free_c.any() else 0.0
        b = np.max(np.abs(gp[~point_const])) if (~point_const).any() else 0.0
        return armax(np.max([a, b]))

    blk, Hc, gc = evaluate(poses, intr, points)
    first = ar(np.concatenate([[blk["cost"]], gc, np.diag(Hc)]))
    cost, gc_glob, Hc_diag = float(first[0]), first[1:1 + D], first[1 + D:]
    if opt.jacobi_scaling:
        sc_c = 1.0 / (1.0 + np.sqrt(Hc_diag))
        sc_p = 1.0 / (1.0 + np.sqrt(np.einsum("nii->ni", blk["H_pp"])))
    else:
        sc_c = np.ones(D)
        sc_p = np.ones((N, 3))
    radius = opt.initial_trust_region_radius
    decrease_factor = 2.0
    summary = {"iterations": 0, "successful": 0, "initial_cost": cost, "termination": "NO_CONVERGENCE"}
    if grad_max_norm(gc_glob, blk["g_p"]) <= opt.gradient_tolerance:
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
        # the rank's part of the reduced system: ba_pcg_oracle.reduced_system's algebra on this shard, then one sum
        Hpp_s = blk["H_pp"] * sc_p[:, :, None] * sc_p[:, None, :]
        dpp = np.clip(np.einsum("nii->ni", Hpp_s), opt.min_lm_diagonal, opt.max_lm_diagonal)
        V = Hpp_s + np.einsum("ni,ij->nij", dpp / radius, np.eye(3))
        V[point_const] = np.eye(3)
        M = sc_p[:, :, None] * np.transpose(np.linalg.inv(np.linalg.cholesky(V)), (0, 2, 1))
        M[point_const] = 0.0
        q = np.einsum("nji,nj->ni", M, blk["g_p"])
        W = bo._full_W(blk, S, dc, ns)
        Z = (W[:, :, 0:1] * M[None, :, 0, :] + W[:, :, 1:2] * M[None, :, 1, :] +
             W[:, :, 2:3] * M[None, :, 2, :]).reshape(D, N * 3)
        part = ar(np.concatenate([Hc.reshape(-1), gc, (Z @ Z.T).reshape(-1), Z @ q.reshape(-1)]))
        Hc_s = part[:D * D].reshape(D, D)
        gc_s = part[D * D:D * D + D]
        ZZ = part[D * D + D:2 * D * D + D].reshape(D, D)
        Zq = part[2 * D * D + D:]
        hd = np.diag(Hc_s).copy()
        dcc = np.clip(hd * sc_c * sc_c, opt.min_lm_diagonal, opt.max_lm_diagonal)
        A = (Hc_s - ZZ) * sc_c[:, None] * sc_c[None, :] + np.diag(dcc / radius)
        b = -(gc_s - Zq) * sc_c
        A[param_const, :] = 0.0
        A[:, param_const] = 0.0
        A[param_const, param_const] = 1.0
        b[param_const] = 0.0
        P, pok, _ = po.schur_jacobi(A, S, dc, ns)
        cgt = []
        dcs, cs = po.cg(A, b, P, eta, min_linear_solver_iterations, max_linear_solver_iterations, cgt, pok)
        if cg_traces is not None:
            cg_traces.append({"summary": cs, "trace": cgt})
        ok = cs["termination"] != po.FAILURE and bool(np.all(np.isfinite(dcs)))
        if ok:
            d_c = dcs * sc_c
            w = np.tensordot(d_c, W, axes=(0, 0))
            d_p = np.einsum("nij,nj->ni", M, np.einsum("nji,nj->ni", M, -(blk["g_p"] + w)))
            d_p[point_const] = 0.0
            c_poses, c_intr, c_points = bo.apply_step(poses, intr, points, d_c[:S * dc].reshape(S, dc), d_c[S * dc:],
                                                      d_p, model, mode)
            c_blk, c_Hc, c_gc = evaluate(c_poses, c_intr, c_points)
            x_cams, x_pts = bo._x_norm_parts(poses, intr, points, S, dc, ns, param_const, point_const)
            mc = po.jd_model_change(poses, intr, points, uv, mask, model, mode, d_c, d_p, point_const)
            cand = ar(np.concatenate([[c_blk["cost"], np.sum(d_p * d_p), x_pts, mc], c_gc]))
            c_cost, dp2, x_pts, model_change, c_gc_glob = float(cand[0]), cand[1], cand[2], float(cand[3]), cand[4:]
            c_gmax = grad_max_norm(c_gc_glob, c_blk["g_p"])
        else:
            model_change = np.nan
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
        step_norm = float(np.sqrt(np.sum(d_c * d_c) + dp2))
        cost_change = cost - c_cost
        rho = cost_change / model_change
        rec = {"it": it, "cost": cost, "candidate_cost": c_cost, "model_change": model_change, "rho": rho,
               "radius": radius, "step_norm": step_norm, "outcome": 0}
        if trace is not None:
            trace.append(rec)
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
            summary["successful"] += 1
            radius = min(opt.max_trust_region_radius, radius / max(1.0 / 3.0, 1.0 - (2.0 * rho - 1.0) ** 3))
            decrease_factor = 2.0
            if c_gmax <= opt.gradient_tolerance:
                summary["termination"] = "CONVERGENCE_GRADIENT"
                break
        else:
            radius = radius / decrease_factor
            decrease_factor *= 2.0
    summary.update(iterations=it, final_cost=cost, final_radius=radius)
    return poses, intr, points, summary
