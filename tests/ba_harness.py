"""What the bundle-adjustment tests share: running a case through the CUDA solve or the float64 oracle, and the bars
that hold one run to another.  Everything that compares takes host data (numpy arrays, the Summary, the oracle's trace
dicts), so each check runs without a GPU.

Rounding bands of the LM decisions.  Every decision of the loop reads cost_change = cost - c_cost.  Both costs are
float64 sums of M squared residuals (M = 2 x observations) that the kernel adds in another order than numpy, and c_cost
is evaluated at a step that carries the solve's forward error; test_lm_step_gpu.py measures one step at backward error
<= 1e-12 and its candidate cost within 1e-12.  Allowing the rounding of the two sums (sqrt(M) 2^-53 each, M < 2^24
here: < 5e-13) and that step error to grow over a few iterations, each cost is held to EPS_COST = 1e-10 of the larger
of the two costs, so that
    |d cost_change| <= 2 EPS_COST max(cost, c_cost) =: e_cc.
The model change is a sum of the same kind over the step (quadratic in it): EPS_MODEL = 1e-9 relative.  Then
    |d rho| <= (e_cc + |rho| EPS_MODEL |model_change|) / |model_change| =: e_rho,
and a successful step multiplies the radius by 1 / max(1/3, 1 - (2 rho - 1)^3), whose relative derivative in rho is at
most 6 (2 rho - 1)^2 / (1/3) <= 18: the radius bar is the running sum of 18 e_rho over the accepted steps before it
(a rejected or invalid step divides by a power of two, exactly).  The gradient and parameter tests compare quantities
computed to EPS_DECIDE = 1e-9 relative.  A CG step stops at the first iteration with zeta < eta: every zeta is held at
least 1e-6 away from eta.

These bars hold only while cost_change is well above the rounding of the cost.  Near the minimum (where the default
options' runs end, as in test_ba_gpu.py) the model change drops to 1e-10 and below: it cancels to a few digits, rho
and even "cost_change == 0" are then decided by rounding, and two solvers may legitimately differ.  So a run held to
these bars stops before that: by a tolerance placed between two iterations of a run without tolerances, or by
max_num_iterations; and no decision of the reference run may lie within its band (check_decisions' margins,
assert_clear).

Whole solves: rotations within 1e-6 degrees (geodesic), translations and points within 1e-7 (L2), intrinsics within
1e-6, the final cost within 1e-9 relative (check_same_solve)."""
import dataclasses

import numpy as np

from oracle import ba_oracle as bo
from oracle import ba_pcg_oracle as po
from tests import ba_loss_oracle as blo
from tests.helpers import backward_error, recovered_step, reference_system, rotation_angle_deg, to_dev

EPS_COST = 1e-10
EPS_MODEL = 1e-9
EPS_DECIDE = 1e-9
ETA = 0.1
ZETA_BAND = 1e-6
RADIUS = 1e4                 # initial_trust_region_radius of the default options
TRIVIAL = ("TRIVIAL", 1.0)

# C1-like shapes over both models and all three intrinsics modes
SHAPES = [
    (8, 256, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME),
    (10, 240, "SIMPLE_RADIAL", bo.INTR_SHARED),
    (12, 200, "SIMPLE_RADIAL", bo.INTR_PER_FRAME),
    (16, 300, "SIMPLE_PINHOLE", bo.INTR_SHARED),
    (9, 220, "SIMPLE_RADIAL", bo.INTR_CONST),
    (20, 300, "SIMPLE_PINHOLE", bo.INTR_CONST),
]


def relerr(a, b):
    return np.abs(a - b).max() / max(1e-300, np.abs(b).max())


def options(**kw):
    """(BAOptions, LMOptions) of one set of fields.  The BAOptions start from the library's vgg_ba_default_options, and
    each of its defaults must be the oracle's (COLMAP's)."""
    from vggsfm_b200 import bundle_adjustment as ba
    o, opt = ba.default_options(), bo.LMOptions(**kw)
    for f in dataclasses.fields(opt):
        assert getattr(o, f.name) == f.default, ("library default is not the oracle's", f.name, getattr(o, f.name))
        v = getattr(opt, f.name)
        setattr(o, f.name, int(v) if isinstance(v, bool) else v)
    return o, opt


# ------------------------------------------------------------------------------------------------------------------
# running a case
# ------------------------------------------------------------------------------------------------------------------

def device_args(c, dev, lo=0, hi=None, uv=None, mask=None):
    """(uv, mask, poses, intr, points, model, mode) of tracks [lo, hi) on the device, as lm_solve takes them"""
    import torch
    uv = c["uv"] if uv is None else uv
    mask = c["mask"] if mask is None else mask
    hi = mask.shape[1] if hi is None else hi
    return (to_dev(uv[:, lo:hi], dev, torch.float32), to_dev(mask[:, lo:hi].astype(np.uint8), dev),
            to_dev(c["poses"], dev), to_dev(c["intr"], dev), to_dev(c["points"][lo:hi], dev), c["model"], c["mode"])


def device_solve(c, dev, lo=0, hi=None, uv=None, mask=None, param_const=None, point_const=None, options=None,
                 allreduce=None, linear_solver=None, loss=None, **lin):
    """lm_solve of tracks [lo, hi) on the current thread and stream; host copies of the results.  point_const is
    given over all tracks; linear_solver and loss (type, scale) left None leave lm_solve's defaults; trace is (0, 8)
    and cg (0, 4) when no iteration ran; calls counts the hook's reductions."""
    import torch
    from vggsfm_b200 import bundle_adjustment as ba
    hi = c["mask"].shape[1] if hi is None else hi
    args = device_args(c, dev, lo, hi, uv, mask)
    if linear_solver is not None:
        lin["linear_solver_type"] = linear_solver
    if loss is not None:
        lin["loss_function_type"], lin["loss_function_scale"] = loss
    s = ba.lm_solve(*args, param_const=None if param_const is None else to_dev(param_const.astype(np.uint8), dev),
                    point_const=None if point_const is None else to_dev(point_const[lo:hi].astype(np.uint8), dev),
                    options=options, allreduce=allreduce, want_trace=True, **lin)
    torch.cuda.current_stream().synchronize()
    ran = s.iterations > 0
    return dict(poses=args[2].cpu().numpy(), intr=args[3].cpu().numpy(), points=args[4].cpu().numpy(), s=s,
                trace=s.trace.numpy().copy() if ran else np.zeros((0, 8)),
                cg=s.cg_trace.numpy().copy() if ran and s.cg_trace is not None else np.zeros((0, 4)),
                calls=allreduce.calls if allreduce is not None else 0, lo=lo, hi=hi)


def oracle_solve(c, uv=None, mask=None, param_const=None, point_const=None, opt=None, lo=0, hi=None, allreduce=None,
                 linear_solver="DENSE_SCHUR", loss=TRIVIAL, use_c=False, **cg):
    """tests/ba_loss_oracle.py lm_solve (dense or iterative, under the loss) of tracks [lo, hi): the state, the
    summary, the trace and (iterative) the CG traces"""
    uv = c["uv"] if uv is None else uv
    mask = c["mask"] if mask is None else mask
    hi = mask.shape[1] if hi is None else hi
    trace, cgs = [], []
    kw = dict(use_c=use_c, allreduce=allreduce) if linear_solver == "DENSE_SCHUR" else dict(cg_traces=cgs, **cg)
    p, i, x, summ = blo.lm_solve(c["poses"], c["intr"], c["points"][lo:hi], uv[:, lo:hi], mask[:, lo:hi], c["model"],
                                c["mode"], param_const=param_const,
                                point_const=None if point_const is None else point_const[lo:hi], options=opt,
                                trace=trace, linear_solver=linear_solver.lower(), loss_function_type=loss[0],
                                loss_function_scale=loss[1], **kw)
    return dict(poses=p, intr=i, points=x, s=summ, trace=trace, cg=cgs, lo=lo, hi=hi)


def band_record():
    """the band hint of the most recent solve on the calling thread (vgg_dev_last_band_hint), every table"""
    from vggsfm_b200 import _lib
    L = _lib.lib()
    meta = np.zeros(8, dtype=np.int32)
    _lib.check(L.vgg_dev_last_band_hint(meta.ctypes.data, None, None, None, None), "vgg_dev_last_band_hint")
    nb, KB, ng = int(meta[3]), int(meta[4]), int(meta[5])
    rec = dict(active=bool(meta[0]), chol=bool(meta[1]), tables=bool(meta[2]), arrow_blk=int(meta[6]),
               rb_range=np.zeros((nb, 2), np.int32), end_blk=np.zeros(nb, np.int32), kb_rows=np.zeros((KB, 2), np.int32),
               fg_tracks=np.zeros((ng, 2), np.int32))
    _lib.check(L.vgg_dev_last_band_hint(meta.ctypes.data, rec["rb_range"].ctypes.data, rec["end_blk"].ctypes.data,
                                        rec["kb_rows"].ctypes.data, rec["fg_tracks"].ctypes.data), "vgg_dev_last_band_hint")
    return rec


# ------------------------------------------------------------------------------------------------------------------
# LM decisions
# ------------------------------------------------------------------------------------------------------------------

def trace_rows(tr):
    """a GPU trace [iterations, 8] as the oracle's trace dicts"""
    return [dict(cost=r[1], candidate_cost=r[2], model_change=r[3], rho=r[4], radius=r[5], step_norm=r[6],
                 outcome=int(r[7])) for r in tr]


def cost_change_bar(r):
    """e_cc of one iteration (module docstring)"""
    return 2 * EPS_COST * max(r["cost"], r["candidate_cost"])


def rho_bar(r):
    """e_rho of one iteration (module docstring)"""
    mc = r["model_change"]
    return (cost_change_bar(r) + abs(r["rho"]) * EPS_MODEL * abs(mc)) / abs(mc)


def cg_zetas(cg):
    """the zetas a CG compared with eta: every CG iteration's of the oracle's cg_traces; of a GPU cg_trace, which keeps
    the last zeta only, the last one of each stop by SUCCESS"""
    if isinstance(cg, np.ndarray):
        return [float(r[2]) for r in cg if int(r[1]) == po.SUCCESS and r[0] > 0]
    return [t["zeta"] for x in cg for t in x["trace"] if "zeta" in t]


def assert_clear(trace, opt, cg=None, eta=ETA):
    """no decision of a reference run (oracle trace dicts, or trace_rows of a GPU trace) lies within its rounding
    band: rho against min_relative_decrease, the cost change against function_tolerance when that is > 0, and with
    a CG trace every zeta against eta"""
    for z in cg_zetas(cg) if cg is not None else ():
        assert abs(z - eta) > ZETA_BAND, ("zeta within its band of eta", z)
    for r in trace:
        if r["outcome"] == 2:
            continue
        assert abs(r["rho"] - opt.min_relative_decrease) > rho_bar(r), ("rho within its band", r, rho_bar(r))
        if opt.function_tolerance > 0:
            cost_change = r["cost"] - r["candidate_cost"]
            assert abs(abs(cost_change) - opt.function_tolerance * r["cost"]) > cost_change_bar(r), \
                ("cost change within its band", r)


def radius_bar(trace):
    """a parameter bar for runs whose rho carries its band: an accepted step's radius may move by the running sum of
    18 e_rho, and the step with it, so 1e-8 + sum over iterations of (radius bar) x (step norm)"""
    rad, bar = 0.0, 1e-8
    for r in trace:
        if r["outcome"] == 2:
            continue
        bar += rad * r["step_norm"]
        if r["outcome"] == 1:
            rad += 18 * rho_bar(r)
    return bar


def between(lo_, hi_):
    """a threshold strictly inside (lo_, hi_), as far from both as a ratio allows"""
    assert 0 < lo_ < hi_, (lo_, hi_)
    return float(np.sqrt(lo_ * hi_))


def first_drop(ratio, start):
    """the first index k >= start whose ratio is below every earlier one, and a threshold between them"""
    for k in range(start, len(ratio)):
        if ratio[k] < min(ratio[:k]):
            return k, between(ratio[k], min(ratio[:k]))
    raise AssertionError(("no decision to place", ratio))


def check_outcomes(got, ref, label=""):
    """device run against the oracle's: termination, counts, every iteration's outcome and the initial cost"""
    s, tr, summ, trace = got["s"], got["trace"], ref["s"], ref["trace"]
    assert s.termination == summ["termination"], (label, s.termination, summ["termination"])
    assert s.iterations == summ["iterations"] == len(trace), (label, s.iterations, summ["iterations"], len(trace))
    assert s.successful == summ["successful"], (label, s.successful, summ["successful"])
    assert [int(v) for v in tr[:, 7]] == [r["outcome"] for r in trace], (label, tr[:, 7], [r["outcome"] for r in trace])
    ic = summ["initial_cost"]
    if np.isfinite(ic):
        assert abs(s.initial_cost - ic) <= 1e-12 * ic, (label, s.initial_cost, ic)
    else:
        assert np.isnan(s.initial_cost) if np.isnan(ic) else s.initial_cost == ic, (label, s.initial_cost, ic)


def check_decisions(got, ref, opt, c, margins=True, label="", cost_bar=1e-9):
    """device run (device_solve) against the oracle's (oracle_solve) of case c under LMOptions opt, at the bars of the
    module docstring: check_outcomes; per iteration the cost, candidate cost, model change, rho and radius; with
    margins, no decision of the oracle's run within its band (the smallest margin / band is printed); the returned
    state (c's as given when no step was accepted, else check_same_solve at cost_bar); for CONVERGENCE_FUNCTION, that
    the state is the last accepted iterate"""
    check_outcomes(got, ref, label)
    s, tr, summ, trace = got["s"], got["trace"], ref["s"], ref["trace"]
    rad_bar = 0.0
    found = []
    for k, r in enumerate(trace):
        assert abs(tr[k, 5] - r["radius"]) <= rad_bar * r["radius"], (label, k, tr[k, 5], r["radius"], rad_bar)
        if r["outcome"] == 2:
            continue
        cc_bar, e_rho, mc = cost_change_bar(r), rho_bar(r), r["model_change"]
        assert abs(tr[k, 1] - r["cost"]) <= EPS_COST * r["cost"], (label, k, tr[k, 1], r["cost"])
        assert abs(tr[k, 2] - r["candidate_cost"]) <= EPS_COST * max(r["cost"], r["candidate_cost"]), \
            (label, k, tr[k, 2], r["candidate_cost"])
        assert abs(tr[k, 3] - mc) <= EPS_MODEL * abs(mc), (label, k, tr[k, 3], mc)
        assert abs(tr[k, 4] - r["rho"]) <= e_rho, (label, k, tr[k, 4], r["rho"], e_rho)
        if margins:
            found.append(abs(r["rho"] - opt.min_relative_decrease) / e_rho)
            found.append(abs(abs(r["cost_change"]) - opt.function_tolerance * r["cost"]) / cc_bar)
            if opt.parameter_tolerance > 0:
                thr = opt.parameter_tolerance * (r["x_norm"] + opt.parameter_tolerance)
                found.append(abs(r["step_norm"] - thr) / (EPS_DECIDE * thr))
            if "gmax" in r and opt.gradient_tolerance > 0:
                found.append(abs(r["gmax"] - opt.gradient_tolerance) / (EPS_DECIDE * opt.gradient_tolerance))
        if r["outcome"] == 1:
            rad_bar += 18 * e_rho
    if margins:
        g0 = summ["initial_gmax"]
        if opt.gradient_tolerance > 0 and np.isfinite(g0):
            found.append(abs(g0 - opt.gradient_tolerance) / (EPS_DECIDE * opt.gradient_tolerance))
        if summ["termination"] == "MIN_TRUST_REGION_RADIUS" or opt.min_trust_region_radius > 1e-32:
            last = summ.get("final_radius", opt.initial_trust_region_radius)
            found.append(abs(last - opt.min_trust_region_radius) / (max(rad_bar, 2.0 ** -52) * last))
        assert not found or min(found) > 1.0, (label, "a decision lies within its rounding band", min(found))
    mm = f"{min(found):.3g}" if found else "-"
    print(f"{label}: {s.termination} after {s.iterations} iterations ({s.successful} accepted), "
          f"smallest margin / band = {mm}")

    if summ["successful"] == 0:
        for k in ("poses", "intr", "points"):
            assert np.array_equal(got[k], c[k]), (label, k)
        assert s.final_cost == s.initial_cost or (np.isnan(s.final_cost) and np.isnan(s.initial_cost))
    else:
        check_same_solve(got, ref, label, cost_bar)
    if summ["termination"] == "CONVERGENCE_FUNCTION":
        assert s.final_cost == tr[-1, 1] and tr[-1, 2] != tr[-1, 1], (label, s.final_cost, tr[-1])
        assert summ["final_cost"] == trace[-1]["cost"] != trace[-1]["candidate_cost"]


def final_cost(x):
    """the final cost of a device_solve or oracle_solve result"""
    return x["s"]["final_cost"] if isinstance(x["s"], dict) else x["s"].final_cost


def check_trajectory(got, ref, traj_tol=1e-7):
    """a whole device solve (default tolerances, so its last decisions may be taken by rounding) against the oracle's:
    the same counts and termination, every valid iteration's candidate cost within traj_tol and radius within 1e-6"""
    s, tr, summ = got["s"], got["trace"], ref["s"]
    assert (s.iterations, s.successful, s.termination) == (summ["iterations"], summ["successful"], summ["termination"])
    for k, r in enumerate(ref["trace"]):
        if r.get("invalid"):
            continue
        assert abs(tr[k, 2] - r["candidate_cost"]) <= traj_tol * max(1.0, r["candidate_cost"]), (k, tr[k], r)
        assert abs(tr[k, 5] - r["radius"]) <= 1e-6 * r["radius"]


def check_same_solve(got, ref, label="", cost_bar=1e-9, frames=slice(None), points=slice(None), min_cost=0.0):
    """the whole-solve bars (module docstring) on the given frames and points: rotation geodesic <= 1e-6 degrees,
    translation and point L2 <= 1e-7, intrinsics <= 1e-6, final cost within cost_bar max(min_cost, cost)"""
    assert abs(final_cost(got) - final_cost(ref)) <= cost_bar * max(min_cost, final_cost(ref)), \
        (label, final_cost(got), final_cost(ref))
    gp, rp = got["poses"][frames], ref["poses"][frames]
    assert rotation_angle_deg(gp[:, :, :3], rp[:, :, :3]).max() <= 1e-6, label
    assert np.linalg.norm(gp[:, :, 3] - rp[:, :, 3], axis=1).max() <= 1e-7, label
    assert np.linalg.norm(got["points"][points] - ref["points"][points], axis=1).max(initial=0.0) <= 1e-7, label
    assert np.abs(got["intr"][frames] - ref["intr"][frames]).max() <= 1e-6, label


# ------------------------------------------------------------------------------------------------------------------
# one LM step
# ------------------------------------------------------------------------------------------------------------------

def check_one_step(c, got, param_const, point_const, loss=TRIVIAL, label=""):
    """one accepted LM iteration (device_solve with max_num_iterations = 1, tolerances 0) of case c in the oracle's full
    damped system at the start point (tests/helpers.py reference_system, under the loss): initial cost within 1e-12,
    the recovered step's backward error <= 1e-12 with constant parameters and points unmoved, the trace's model change
    and step norm within 1e-10 at that step, the candidate cost within 1e-12 of the oracle's at the returned state.
    Returns eta, the system and the scaled step for the caller's own checks."""
    S, N = c["mask"].shape
    model, mode = c["model"], c["mode"]
    dc, ns = bo.dims(model, mode)
    s, tr = got["s"], got["trace"]
    new = (got["poses"], got["intr"], got["points"])
    assert s.iterations == 1 and tr[0, 7] == 1 and tr[0, 5] == RADIUS, (label, tr)
    with blo.robust(*loss):
        ref = reference_system(c, param_const, point_const, RADIUS)
    assert abs(s.initial_cost - ref["cost"]) <= 1e-12 * ref["cost"], (label, s.initial_cost, ref["cost"])
    d_c, u_c, d_p, u_p = recovered_step((c["poses"], c["intr"], c["points"]), new, S, dc, ns, model, mode)
    assert not d_c[param_const].any() and not d_p[point_const].any(), label
    dcs, ucs, dps, ups = d_c / ref["sc_c"], u_c / ref["sc_c"], d_p / ref["sc_p"], u_p / ref["sc_p"]
    eta = backward_error(ref, dcs, ucs, dps, ups)
    # model change (oracle/ba_oracle.py lm_solve) and step norm at the recovered step
    model_change = 0.5 * (np.sum(dcs * dcs * ref["dcc"] / RADIUS * ref["fc"]) - np.sum(d_c * ref["gc"]) +
                          np.sum(dps * dps * ref["dpp"] / RADIUS * ref["fp"][:, None]) - np.sum(d_p * ref["gp"]))
    step_norm = np.sqrt(np.sum(d_c * d_c) + np.sum(d_p * d_p))
    c_cost = blo.cost_only(*new, c["uv"], c["mask"], model, *loss)
    print(f"lm step {label}: eta = {eta:.2e}  model change {abs(tr[0, 3] / model_change - 1):.1e}  "
          f"step norm {abs(tr[0, 6] / step_norm - 1):.1e}  candidate cost {abs(tr[0, 2] / c_cost - 1):.1e}")
    assert eta <= 1e-12, (label, eta)
    assert abs(tr[0, 3] - model_change) <= 1e-10 * abs(model_change), (label, tr[0, 3], model_change)
    assert abs(tr[0, 6] - step_norm) <= 1e-10 * step_norm, (label, tr[0, 6], step_norm)
    assert abs(tr[0, 2] - c_cost) <= 1e-12 * c_cost, (label, tr[0, 2], c_cost)
    return dict(eta=eta, ref=ref, dcs=dcs, dps=dps, d_p=d_p, u_p=u_p)
