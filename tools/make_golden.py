"""Generate tests/golden/*.npz by running the UNMODIFIED reference ($VGGSFM_REFERENCE, imported with stub
third-party modules) on seeded synthetic inputs.  Run in the build container only:

    python tools/make_golden.py

Pinned cases run the reference with torch.sort forced stable (its unstable descending sort leaves the
order of equal inlier counts implementation-defined, see oracle/tri_oracle.py); the `unpinned` case runs
it exactly as shipped.  The hypothesis frame pairs are recorded by replaying the CPU RNG draw of
vggsfm/utils/triangulation.py:811-813 from the same seed.
"""
import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
warnings.filterwarnings("ignore")

from oracle import reference_shim as rs          # noqa: E402
from oracle import tri_oracle as to              # noqa: E402
from vggsfm_b200.synthetic import make_scene     # noqa: E402

rs.install()
from vggsfm.utils import triangulation as rt               # noqa: E402
from vggsfm.utils import triangulation_helpers as rh       # noqa: E402

CASES = {
    # name: (S, N, camera, scene kwargs, max_ransac_iters, pinned)
    "tri_c1_8x256_pinhole": (8, 256, "SIMPLE_PINHOLE", dict(seed=0), 256, True),
    "tri_12x96_radial_outliers": (12, 96, "SIMPLE_RADIAL", dict(seed=1, invisible_frac=0.3, outlier_frac=0.1), 256, True),
    "tri_30x64_pinhole_256of435": (30, 64, "SIMPLE_PINHOLE", dict(seed=2, invisible_frac=0.2, outlier_frac=0.05), 256, True),
    "tri_40x48_radial_128hyp": (40, 48, "SIMPLE_RADIAL", dict(seed=3, invisible_frac=0.25, outlier_frac=0.08), 128, True),
    "tri_30x64_unpinned": (30, 64, "SIMPLE_PINHOLE", dict(seed=2, invisible_frac=0.2, outlier_frac=0.05), 256, False),
}

_sort = torch.sort


def _stable_sort(*a, **k):
    k["stable"] = True
    return _sort(*a, **k)


def main():
    out_dir = os.path.join(ROOT, "tests", "golden")
    os.makedirs(out_dir, exist_ok=True)
    for name, (S, N, cam, kw, iters, pinned) in CASES.items():
        sc = make_scene(S, N, cam, **kw)
        K = torch.from_numpy(sc.intrinsics)
        E = torch.from_numpy(sc.extrinsics)
        ex = torch.from_numpy(sc.extra_params) if sc.extra_params is not None else None
        tracks = torch.from_numpy(sc.tracks)
        tn = rh.cam_from_img(tracks, K, ex)
        seed = 1234 + S
        torch.manual_seed(seed)
        pairs = to.draw_pairs(S, iters)
        torch.manual_seed(seed)
        if pinned:
            torch.sort = _stable_sort
        try:
            p, n, m = rt.triangulate_tracks(E, rs.contiguous_tracks(tn), max_ransac_iters=iters,
                                            track_vis=torch.from_numpy(sc.vis), track_score=torch.from_numpy(sc.score))
        finally:
            torch.sort = _sort
        v, d = rh.filter_all_points3D(p, tracks.double(), E, K, ex, max_reproj_error=1.0, return_detail=True)
        v2, _ = rh.filter_all_points3D(p, tracks.double(), E, K, ex, max_reproj_error=4.0, check_triangle=False)
        p2d, pcam = rh.project_3D_points(p, E, K, ex, return_points_cam=True)
        bp, bche, bang = rt.triangulate_by_pair(E[None], tn[None])
        np.savez_compressed(
            os.path.join(out_dir, name + ".npz"),
            extrinsics=sc.extrinsics, intrinsics=sc.intrinsics,
            extra_params=sc.extra_params if sc.extra_params is not None else np.zeros((0, 1)),
            tracks=sc.tracks, vis=sc.vis, score=sc.score, pairs=pairs.astype(np.int32), max_ransac_iters=iters,
            pinned=pinned, tn=tn.numpy(), points=p.numpy(), inlier_num=n.numpy(), inlier_mask=m.numpy(),
            filt_valid=v.numpy(), filt_detail=d.numpy(), filt_valid_notri=v2.numpy(), proj2d=p2d.numpy(),
            projcam=pcam.numpy(), pair_points=bp.numpy(), pair_cheirality=bche.numpy(), pair_angle=bang.numpy())
        print(name, "inliers/track mean", n.float().mean().item(), "valid", int(v.sum()))
    edges(out_dir)


# Slow undistortion: (k, pixel coordinate c of four tracks at (c, c), (1024-c, c), ... near the image corners).  The
# reference's iteration (Jacobian ~ 2I + G, see oracle/tri_oracle.py) contracts at the rate 1/(2 + 3 k r^2) along the
# radius, so tracks whose undistorted radius lies just inside the turning point 3 k r^2 = -1 converge slowly but
# stably: 11 iterations at k = 0.05, 47 at -0.4, 80 at -0.55 (the second word of the kernel's non-convergence mask)
# and no convergence within max_iterations = 100 at -0.5.  Tracks past the turning point (no undistorted solution,
# e.g. the very corners at these k) make the iteration wander, and its stop then depends on rounding.
UNDIST_CASES = [(0.05, 0.5), (-0.4, 87.25), (-0.55, 145.921875), (-0.5, 127.328125)]


def corner_tracks(c):
    """four pixel tracks symmetric about the principal point (512, 512), exact in float32."""
    return np.array([[c, c], [1024 - c, c], [c, 1024 - c], [1024 - c, 1024 - c]])


def edges(out_dir):
    """tests/golden/edges_undistort_gate8.npz: the reference's cam_from_img on corner tracks at the slow-convergence
    k values (one call per k, and one call mixing the converging ones since the stop is global), with the iteration
    count at which it stopped; and one pinned triangulate_tracks with max_angular_error = 8 degrees (the kernel's
    acos branch)."""
    from vggsfm.utils import distortion as rd
    C = len(UNDIST_CASES)
    uv = np.stack([corner_tracks(d) for _, d in UNDIST_CASES]).astype(np.float32)        # [C,4,2] one frame per case
    ks = np.array([k for k, _ in UNDIST_CASES])[:, None]                                # [C,1]
    K = np.tile(np.array([[1000.0, 0, 512.0], [0, 1000.0, 512.0], [0, 0, 1.0]]), (C, 1, 1))

    def stop(k, tn):
        """the iteration the reference stopped at: the least max_iterations whose output equals the full run's."""
        full = rd.iterative_undistortion(k, tn)
        return next(m for m in range(1, 101) if torch.equal(rd.iterative_undistortion(k, tn, max_iterations=m), full))

    tn_each, it_each = [], []
    for c in range(C):
        t = torch.from_numpy(uv[c:c + 1]).double()
        tn_each.append(rh.cam_from_img(t, torch.from_numpy(K[c:c + 1]), torch.from_numpy(ks[c:c + 1])).numpy()[0])
        it_each.append(stop(torch.from_numpy(ks[c:c + 1]), (t - 512.0) / 1000.0))
    t = torch.from_numpy(uv[:-1]).double()                 # every case but the non-converging one
    tn_mixed = rh.cam_from_img(t, torch.from_numpy(K[:-1]), torch.from_numpy(ks[:-1])).numpy()
    it_mixed = stop(torch.from_numpy(ks[:-1]), (t - 512.0) / 1000.0)
    print("undistortion iterations", it_each, "mixed", it_mixed)

    S, N, iters = 12, 64, 256
    sc = make_scene(S, N, "SIMPLE_RADIAL", seed=11, invisible_frac=0.2, outlier_frac=0.15)
    E = torch.from_numpy(sc.extrinsics)
    tn = rh.cam_from_img(torch.from_numpy(sc.tracks), torch.from_numpy(sc.intrinsics), torch.from_numpy(sc.extra_params))
    seed = 4321
    torch.manual_seed(seed)
    pairs = to.draw_pairs(S, iters)
    torch.manual_seed(seed)
    torch.sort = _stable_sort
    try:
        p, n, m = rt.triangulate_tracks(E, rs.contiguous_tracks(tn), max_ransac_iters=iters, max_angular_error=8,
                                        track_vis=torch.from_numpy(sc.vis), track_score=torch.from_numpy(sc.score))
    finally:
        torch.sort = _sort
    np.savez_compressed(
        os.path.join(out_dir, "edges_undistort_gate8.npz"),
        und_k=ks, und_uv=uv, und_intrinsics=K, und_tn=np.stack(tn_each), und_iters=np.array(it_each),
        und_tn_mixed=tn_mixed, und_iters_mixed=it_mixed,
        extrinsics=sc.extrinsics, intrinsics=sc.intrinsics, extra_params=sc.extra_params, tracks=sc.tracks, vis=sc.vis,
        score=sc.score, pairs=pairs.astype(np.int32), tn=tn.numpy(), max_angular_error=8.0, points=p.numpy(),
        inlier_num=n.numpy(), inlier_mask=m.numpy())
    print("gate 8: inliers/track mean", n.float().mean().item())


if __name__ == "__main__":
    if sys.argv[1:] == ["edges"]:
        edges(os.path.join(ROOT, "tests", "golden"))
    else:
        main()
