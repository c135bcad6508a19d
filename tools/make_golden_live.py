"""Golden fixtures for the tests that used to compare against a live run of the reference (needs a reference checkout named by $VGGSFM_REFERENCE,
imported through oracle/reference_shim.py):

    python tools/make_golden_live.py

  tests/golden/tracker_score.npz    refine_track.compute_score_fn on the seeded inputs of tests/test_tracker_host.py
  tests/golden/reference_triangulate_10x40.npz   triangulation.triangulate_tracks on the 10 x 40 scene of tests/test_tri_oracle.py
  tests/golden/colmap_reader.npz    the COLMAP .bin files this project writes for marshal case c, and what the
                                    reference's reader (imc_helper.read_model) parses from them"""
import os
import sys
import tempfile
import types
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import reference_shim as rs  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def score():
    from tools.make_golden_tracker import create_meshgrid, spatial_expectation2d
    from vggsfm.models.track_modules import refine_track as rt
    rt.create_meshgrid = create_meshgrid
    rt.dsnt = types.SimpleNamespace(spatial_expectation2d=spatial_expectation2d)
    g = torch.Generator().manual_seed(0)
    out = {}
    for i, (B, N, S) in enumerate(((1, 5, 4), (2, 3, 3))):
        C, psize, sr = 8, 31, 2
        qf = torch.randn(B, N, C, generator=g)
        pf = torch.randn(B * N, S, C, psize, psize, generator=g)
        trk = torch.rand(B * N, S, 1, 2, generator=g) * 34 - 2
        out[f"score{i}"] = rt.compute_score_fn(qf, pf, trk, sr, psize, B, N, S, C).numpy()
    np.savez_compressed(os.path.join(GOLD, "tracker_score.npz"), **out)


def triangulation():
    from vggsfm.utils import triangulation as rt
    from vggsfm.utils import triangulation_helpers as rh
    from vggsfm_b200.synthetic import make_scene
    sc = make_scene(10, 40, "SIMPLE_RADIAL", seed=21, invisible_frac=0.2, outlier_frac=0.1)
    K, E, ex = torch.from_numpy(sc.intrinsics), torch.from_numpy(sc.extrinsics), torch.from_numpy(sc.extra_params)
    tn = rh.cam_from_img(torch.from_numpy(sc.tracks), K, ex)
    _sort = torch.sort

    def stable(*a, **k):
        k["stable"] = True
        return _sort(*a, **k)
    torch.manual_seed(3)
    torch.sort = stable
    try:
        p, n, m = rt.triangulate_tracks(E, rs.contiguous_tracks(tn), track_vis=torch.from_numpy(sc.vis),
                                        track_score=torch.from_numpy(sc.score))
    finally:
        torch.sort = _sort
    np.savez_compressed(os.path.join(GOLD, "reference_triangulate_10x40.npz"), tn=tn.numpy(), points=p.numpy(), num=n.numpy(),
                        mask=m.numpy())


def colmap_reader():
    sys.modules.setdefault("h5py", types.ModuleType("h5py"))
    from vggsfm.datasets import imc_helper as ih
    from tests.test_reconstruction import _build
    from tools.make_golden_marshal import cases
    rec = _build(cases()[2])
    rec.set_point_colors(np.linspace(0, 1, rec.num_points3D())[:, None].repeat(3, 1))
    out = {}
    with tempfile.TemporaryDirectory() as d:
        rec.write(d)
        for name in ("cameras", "images", "points3D"):
            out[f"bin_{name}"] = np.frombuffer(open(os.path.join(d, name + ".bin"), "rb").read(), dtype=np.uint8)
        cams, ims, pts = ih.read_model(d, ext=".bin")
    cids, iids, pids = sorted(cams), sorted(ims), sorted(pts)
    out["cam_ids"] = np.array(cids)
    out["cam_model"] = np.array([cams[c].model for c in cids])
    out["cam_wh"] = np.array([(cams[c].width, cams[c].height) for c in cids])
    out["cam_params"] = np.stack([cams[c].params for c in cids])
    out["img_ids"] = np.array(iids)
    out["img_name"] = np.array([ims[i].name for i in iids])
    out["img_camera_id"] = np.array([ims[i].camera_id for i in iids])
    out["img_rotmat"] = np.stack([ims[i].qvec2rotmat() for i in iids])
    out["img_tvec"] = np.stack([ims[i].tvec for i in iids])
    out["img_nxy"] = np.array([len(ims[i].xys) for i in iids])
    out["img_xys"] = np.concatenate([np.asarray(ims[i].xys).reshape(-1, 2) for i in iids])
    out["img_p3d"] = np.concatenate([np.asarray(ims[i].point3D_ids).reshape(-1) for i in iids])
    out["pt_ids"] = np.array(pids)
    out["pt_xyz"] = np.stack([pts[p].xyz for p in pids])
    out["pt_rgb"] = np.stack([pts[p].rgb for p in pids])
    out["pt_tracklen"] = np.array([len(pts[p].image_ids) for p in pids])
    out["pt_track"] = np.concatenate([np.stack([pts[p].image_ids, pts[p].point2D_idxs], 1).reshape(-1, 2) for p in pids])
    np.savez_compressed(os.path.join(GOLD, "colmap_reader.npz"), **out)


if __name__ == "__main__":
    warnings.filterwarnings("ignore")
    rs.install()
    score()
    triangulation()
    colmap_reader()
