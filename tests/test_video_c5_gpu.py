"""The C5 driver (tools/video_c5.py) on a short sequence: the sequential pipeline (pose alignment, window triangulation,
window BA, scene tables, joint BA) must track the synthetic ground truth."""
import os
import sys

import pytest

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))


def test_sequential_run_tracks_ground_truth(cuda_dev):
    import video_c5
    out = video_c5.run(frames=128, new_per_window=96, joint_every=3, dev=cuda_dev)
    assert out["windows"] == 6 and out["joint_bas"] == 2
    assert out["final_joint_ba"]["frames"] == 128 and out["final_joint_ba"]["lm_iterations"] > 0
    assert out["store_points"] > 300
    # camera centres after a similarity alignment: a few millimetres on a 7.6-unit trajectory (0.3 px noise)
    assert out["camera_centre_rmse_vs_gt"] < 0.02 * out["trajectory_length"]


def _band_hint_meta():
    """{SYRK k-range hint, factorisation band, device tables} of the most recent solve (vgg_dev_last_band_hint)"""
    import numpy as np
    from vggsfm_b200 import _lib
    meta = np.zeros(8, dtype=np.int32)
    _lib.check(_lib.lib().vgg_dev_last_band_hint(meta.ctypes.data, None, None, None, None), "vgg_dev_last_band_hint")
    return [bool(v) for v in meta[:3]]


def test_band_hint_does_not_change_the_joint_ba(cuda_dev):
    """The band skipping (band hint from the visibility mask, csrc/ba_solve.cu: SYRK, Cholesky, ba_blocks, z_build and
    backsub) must leave the solve unchanged.  The same problem with its points in random order is the dense twin: every
    frame's [first, last] visible point then spans almost every track, so the detection must find nothing to skip.
    Both reach the same minimum (final cost to 1e-9 relative).  The iteration COUNT is not compared: the last
    iterations of these solves sit on the gradient / function tolerance and the count moves by a few from run to run
    in either mode (f64 RED order)."""
    import video_c5
    from vggsfm_b200 import video
    res = {}
    for shuffle in (False, True):
        out = video_c5.final_problem(frames=320, new_per_window=128, dev=cuda_dev, reps=1, shuffle=shuffle)
        res[shuffle] = (out["lm_iterations"][0], float(video.last_joint_summary.final_cost), _band_hint_meta())
    assert res[False][2] == [True, True, True], res[False]          # in order: banded
    assert res[True][2] == [False, False, False], res[True]         # shuffled: dense
    assert res[False][0] > 5 and res[True][0] > 5
    assert abs(res[False][1] - res[True][1]) <= 1e-9 * abs(res[True][1])
