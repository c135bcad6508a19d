"""Values the masks hide from the bundle adjustment, in the oracle (oracle/ba_oracle.py, oracle/ba_blocks_ref.c).

A hidden value is the uv of an observation whose mask is 0, the coordinates of a point that no valid observation sees,
or the pose / intrinsics of a frame that no valid observation sees.  None of them may reach anything the solve computes:
the reference for a problem is its clean twin, the same problem with uv = 0 in the masked slots, the unobserved points at
(0, 0, 1) and the unobserved frames at their original pose.  Both statements of the normal-equation blocks (numpy and C)
must equal the clean twin's, and lm_solve must take the clean twin's decisions and return hidden parameters as given."""
import numpy as np
import pytest

from oracle import ba_oracle as bo
from tests.helpers import hidden_case

FLT_MAX = float(np.finfo(np.float32).max)
UV_VALUES = [np.nan, np.inf, -np.inf, FLT_MAX, -FLT_MAX]
POINT_VALUES = [np.nan, np.inf, -np.inf, 1e308]
MODES = [(cam, mode) for cam in ("SIMPLE_PINHOLE", "SIMPLE_RADIAL")
         for mode in (bo.INTR_CONST, bo.INTR_PER_FRAME, bo.INTR_SHARED)]


def _blocks(fn, c, point_const=None):
    with np.errstate(all="ignore"):
        return fn(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], c["mode"], point_const)


def _close(a, b, tol, what):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert np.isfinite(a).all(), (what, "non-finite")
    scale = max(np.abs(b).max(initial=0.0), 1e-300)
    assert np.abs(a - b).max(initial=0.0) <= tol * scale, (what, np.abs(a - b).max() / scale)


KEYS = ("g_c", "H_cc", "g_p", "H_pp", "W")
SHARED_KEYS = ("g_s", "H_ss", "H_cs", "W_s")


@pytest.mark.parametrize("cam,mode", MODES)
@pytest.mark.parametrize("point_value", POINT_VALUES)
@pytest.mark.parametrize("uv_value", UV_VALUES)
def test_blocks_equal_clean_twin(cam, mode, point_value, uv_value):
    """numpy build_blocks and the C restatement agree within 1e-12 relative and both equal the clean twin; the hidden
    points' own rows are exact zeros"""
    dirty, clean, hidden = hidden_case(6, 40, cam, mode, 7, point_value, uv_value)
    ref = _blocks(bo.build_blocks, clean)
    outs = {"numpy": _blocks(bo.build_blocks, dirty)}
    if bo._load_c() is not None:
        outs["c"] = _blocks(bo.build_blocks_c, dirty)
    keys = KEYS + (SHARED_KEYS if mode == bo.INTR_SHARED else ())
    for name, out in outs.items():
        assert np.isfinite(out["cost"]) and abs(out["cost"] - ref["cost"]) <= 1e-12 * ref["cost"], name
        for k in keys:
            _close(out[k], ref[k], 1e-12, (name, k))
        assert not out["g_p"][hidden].any() and not out["H_pp"][hidden].any() and not out["W"][:, :, hidden].any()
    if "c" in outs:
        for k in keys:
            _close(outs["c"][k], outs["numpy"][k], 1e-12, ("c vs numpy", k))


@pytest.mark.parametrize("cam,mode", MODES)
def test_blocks_unobserved_frame(cam, mode):
    """a frame whose mask row is empty and whose pose is NaN contributes nothing, not even to the points it would see"""
    dirty, clean, _ = hidden_case(6, 40, cam, mode, 8, np.nan, np.nan, hidden_frame=3)
    ref = _blocks(bo.build_blocks, clean)
    for fn in (bo.build_blocks,) + ((bo.build_blocks_c,) if bo._load_c() is not None else ()):
        out = _blocks(fn, dirty)
        assert abs(out["cost"] - ref["cost"]) <= 1e-12 * ref["cost"]
        for k in KEYS + (SHARED_KEYS if mode == bo.INTR_SHARED else ()):
            _close(out[k], ref[k], 1e-12, k)
        assert not out["g_c"][3].any() and not out["H_cc"][3].any()


def test_cost_only_ignores_masked_uv():
    dirty, clean, _ = hidden_case(6, 40, "SIMPLE_RADIAL", bo.INTR_SHARED, 9, np.nan, np.nan)
    assert bo.cost_only(dirty["poses"], dirty["intr"], dirty["points"], dirty["uv"], dirty["mask"], dirty["model"]) == \
        bo.cost_only(clean["poses"], clean["intr"], clean["points"], clean["uv"], clean["mask"], clean["model"])


def _lm(c, **kw):
    trace = []
    opt = bo.LMOptions()
    opt.max_num_iterations = 8
    for k, v in kw.items():
        setattr(opt, k, v)
    with np.errstate(all="ignore"):
        out = bo.lm_solve(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], c["mode"], options=opt,
                          trace=trace)
    return out, trace


@pytest.mark.parametrize("cam,mode", [("SIMPLE_PINHOLE", bo.INTR_PER_FRAME), ("SIMPLE_RADIAL", bo.INTR_SHARED)])
@pytest.mark.parametrize("hidden_frame", [None, 2])
@pytest.mark.parametrize("parameter_tolerance", [0.0, 1e-12])
def test_lm_solve_takes_the_clean_twins_steps(cam, mode, hidden_frame, parameter_tolerance):
    """a hidden NaN point (not flagged constant) and a hidden NaN frame: the trace equals the clean twin's -- outcome,
    costs, step norm and |x| -- and the hidden parameters come back as given"""
    dirty, clean, hidden = hidden_case(8, 60, cam, mode, 10, np.nan, np.nan, hidden_frame=hidden_frame)
    (p_d, i_d, x_d, s_d), t_d = _lm(dirty, parameter_tolerance=parameter_tolerance)
    (p_c, i_c, x_c, s_c), t_c = _lm(clean, parameter_tolerance=parameter_tolerance)
    assert s_d["termination"] == s_c["termination"] and s_d["iterations"] == s_c["iterations"] >= 3
    assert [r["outcome"] for r in t_d] == [r["outcome"] for r in t_c]
    for rd, rc in zip(t_d, t_c):
        for k in ("cost", "candidate_cost", "model_change", "step_norm", "x_norm", "radius"):
            if k in rc:
                assert np.isfinite(rd[k]) and abs(rd[k] - rc[k]) <= 1e-12 * abs(rc[k]), (k, rd[k], rc[k])
    keep = np.setdiff1d(np.arange(dirty["mask"].shape[1]), hidden)
    assert np.array_equal(x_d[keep], x_c[keep])
    assert np.isnan(x_d[hidden]).all()
    frames = np.arange(dirty["mask"].shape[0]) != (hidden_frame if hidden_frame is not None else -1)
    assert np.array_equal(p_d[frames], p_c[frames]) and np.array_equal(i_d, i_c)
    if hidden_frame is not None:
        assert np.isnan(p_d[hidden_frame]).all()
        assert np.array_equal(p_c[hidden_frame], clean["poses"][hidden_frame])
