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


def test_band_hint_does_not_change_the_joint_ba(cuda_dev):
    """The tile / k-range skipping of the tensor-core SYRK (band hint from the visibility mask, csrc/ba_solve.cu) must
    leave the solve unchanged: same minimum (final cost to 1e-9 relative).  The iteration COUNT is not compared: the
    last iterations of these solves sit on the gradient / function tolerance and the count moves by a few from run to
    run in either mode (f64 RED order; tools/band_parity_check.py shows it)."""
    import video_c5
    from vggsfm_b200 import video
    res = {}
    for band in ("0", "1"):               # dense / SYRK, Cholesky, ba_blocks, z_build and backsub skips
        os.environ["VGG_BAND"] = band
        try:
            out = video_c5.final_problem(frames=320, new_per_window=128, dev=cuda_dev, reps=1)
            res[band] = (out["lm_iterations"][0], float(video.last_joint_summary.final_cost))
        finally:
            os.environ.pop("VGG_BAND", None)
    assert res["0"][0] > 5 and res["1"][0] > 5
    assert abs(res["0"][1] - res["1"][1]) <= 1e-9 * abs(res["0"][1])


def test_band_detection_is_safe_for_unordered_points(cuda_dev):
    """Points in random order: every frame's [first, last] visible point spans almost everything, the hint must either
    stay off or change nothing."""
    import video_c5
    from vggsfm_b200 import video
    res = {}
    for band in ("0", "1"):
        os.environ["VGG_BAND"] = band
        try:
            video_c5.final_problem(frames=256, new_per_window=128, dev=cuda_dev, reps=1, shuffle=True)
            res[band] = float(video.last_joint_summary.final_cost)
        finally:
            os.environ.pop("VGG_BAND", None)
    assert abs(res["0"] - res["1"]) <= 1e-9 * abs(res["0"])
