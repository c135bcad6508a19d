"""estimate_preliminary_cameras_poselib -> Triangulator.forward on the CUDA path with no ground-truth shortcut: the
epipolar inlier mask the triangulator reads (models/triangulator.py:92) comes from the LO-MSAC two-view stage of the
default configuration (vggsfm_b200/two_view.py, csrc/twoview_msac.cu)."""
import numpy as np
import pytest

from tests.helpers import to_dev
from tests.test_pipeline_gpu import _Cameras, _umeyama

pytestmark = pytest.mark.gpu


def test_poselib_stage_feeds_the_triangulator(cuda_dev):
    import torch
    from vggsfm_b200 import triangulation as tri
    from vggsfm_b200 import two_view as tv
    from vggsfm_b200.synthetic import make_scene, perturb, project_np
    from vggsfm_b200.triangulator import Triangulator
    S, N = 12, 1024
    sc = make_scene(S, N, "SIMPLE_PINHOLE", seed=11, noise_px=0.2, invisible_frac=0.1, outlier_frac=0.02)
    dev = cuda_dev
    W = H = 1024
    tracks = to_dev(sc.tracks, dev)[None]
    vis = to_dev(sc.vis, dev)[None]
    score = to_dev(sc.score, dev)[None]
    cams0, prelim = tv.estimate_preliminary_cameras_poselib(tracks, vis, W, H, tracks_score=score, max_error=1.0)
    assert cams0 is None
    assert prelim["fmat"].shape == (1, S - 1, 3, 3) and prelim["fmat_inlier_mask"].shape == (1, S - 1, N)
    uv_gt, _ = project_np(sc.extrinsics, 1000.0, np.array([512.0, 512.0]), 0.0, sc.points3d)
    clean = np.linalg.norm(sc.tracks - uv_gt, axis=-1) < 3.0
    true_in = (clean[:1] & clean[1:]) & sc.mask[1:]
    planted = ~clean[1:] & sc.mask[1:]
    est = prelim["fmat_inlier_mask"][0].cpu().numpy()
    assert (est & true_in).sum() >= 0.95 * true_in.sum(), ((est & true_in).sum(), true_in.sum())
    assert (est & planted).sum() <= 0.01 * planted.sum() + 1, ((est & planted).sum(), planted.sum())
    extr0, K0, _, _ = perturb(sc, rot_deg=0.4, trans_frac=0.01, focal_frac=0.02, seed=12)
    cams = _Cameras(to_dev(np.stack([K0[:, 0, 0], K0[:, 1, 1]], -1) * 2.0 / min(W, H), dev, torch.float32),
                    to_dev(extr0[:, :, :3], dev, torch.float32), to_dev(extr0[:, :, 3], dev, torch.float32))
    images = torch.rand(1, S, 3, H, W, device=dev)
    torch.manual_seed(0)
    out = Triangulator()(cams, tracks, vis, images, prelim, pred_score=score, BA_iters=2, shared_camera=False,
                         robust_refine=2, camera_type="SIMPLE_PINHOLE")
    E, K, ex, pts, rgb, rec, vframe, v2d, vtracks = out
    P = int(vtracks.sum())
    assert P > 0.85 * N and bool(vframe.all())
    uvh = tri.project_3D_points(pts, E, K, ex)
    err = ((uvh - tracks[0][:, vtracks].double()) ** 2).sum(-1)
    rms = torch.sqrt(err[v2d[:, vtracks]].mean()).item()
    assert rms < 0.6, rms
    En = E.cpu().numpy()
    C_est = -np.einsum("sji,sj->si", En[:, :, :3], En[:, :, 3])
    C_gt = -np.einsum("sji,sj->si", sc.extrinsics[:, :, :3], sc.extrinsics[:, :, 3])
    s, R, t = _umeyama(C_est, C_gt)
    assert np.linalg.norm((s * (R @ C_est.T).T + t) - C_gt, axis=1).max() < 0.02
