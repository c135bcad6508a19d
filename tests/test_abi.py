"""The C-ABI library loads and exports every symbol include/vggsfm_b200.h declares (no GPU compute)."""
import os
import re

from vggsfm_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "vggsfm_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(vgg_[a-z0-9_]+)\s*\(", src)) - {"vgg_allreduce_fn"})


def test_library_exports_every_declared_symbol():
    L = _lib.lib()
    decl = declared_symbols()
    assert decl, "no declarations parsed"
    for name in decl:
        assert hasattr(L, name), f"libvggsfm_b200.so does not export {name}"
    assert sorted(_lib.EXPORTS) == decl
    assert L.vgg_version() >= 100


def test_host_only_entry_points():
    import ctypes
    L = _lib.lib()
    dc, ns = ctypes.c_int(), ctypes.c_int()
    assert L.vgg_ba_dims(1, 2, ctypes.byref(dc), ctypes.byref(ns)) == 0 and (dc.value, ns.value) == (6, 2)
    assert L.vgg_ba_dims(0, 1, ctypes.byref(dc), ctypes.byref(ns)) == 0 and (dc.value, ns.value) == (7, 0)
    assert L.vgg_ba_dims(7, 1, ctypes.byref(dc), ctypes.byref(ns)) != 0
    assert L.vgg_ba_camrec_len(1, 1) == 8 + 36
    o = _lib.BAOptions()
    L.vgg_ba_default_options(ctypes.byref(o))
    assert o.max_num_iterations == 100 and o.gradient_tolerance == 1e-4


def test_ba_workspace_bytes_is_host_only():
    """vgg_ba_workspace_bytes is a pure size computation: it succeeds without a GPU for the C1, C2 and C3 shapes and
    every camera model / intrinsics mode, and for 1001 frames (D = 7007 with per-frame SIMPLE_PINHOLE), and covers at least the Schur operand Zt [Kpad][Dpad] and the reduced system
    [D+3][Dpad] (matrix rows, right-hand side, diagonal, gradient) in float64."""
    import ctypes
    L = _lib.lib()
    for S, N in ((8, 256), (50, 2048), (400, 4096), (1001, 2048), (1001, 6000)):     # the last two: D > 7000
        for model in (0, 1):
            for mode in (0, 1, 2):
                dc, ns = ctypes.c_int(), ctypes.c_int()
                assert L.vgg_ba_dims(model, mode, ctypes.byref(dc), ctypes.byref(ns)) == 0
                D = S * dc.value + ns.value
                Dpad = (D + 2 + 127) // 128 * 128
                Kpad = (3 * N + 15) // 16 * 16
                red = ctypes.c_size_t()
                assert L.vgg_ba_reduced_system_doubles(S, model, mode, ctypes.byref(red)) == 0
                assert red.value == (D + 3) * Dpad
                n = ctypes.c_size_t()
                rc = L.vgg_ba_workspace_bytes(S, N, model, mode, ctypes.byref(n))
                assert rc == 0, (S, N, model, mode, rc, L.vgg_last_error())
                assert n.value >= 8 * (Kpad * Dpad + (D + 3) * Dpad), (S, N, model, mode, n.value)


def test_build_blocks_rejects_unaligned_tracks_per_warp():
    """vgg_ba_build_blocks: tracks_per_warp must be 0 (choose) or a positive multiple of 4, else a warp's vectorised
    observation loads would be misaligned.  The check comes before any CUDA call, so it needs no GPU: the buffers are
    host memory of the right sizes that nothing may touch."""
    import ctypes
    import numpy as np
    L = _lib.lib()
    S, N = 2, 5
    dc, ns = ctypes.c_int(), ctypes.c_int()
    assert L.vgg_ba_dims(0, 1, ctypes.byref(dc), ctypes.byref(ns)) == 0
    D = S * dc.value + ns.value
    arrays = dict(uv=np.zeros((S, N, 2), np.float32), mask=np.ones((S, N), np.uint8), poses=np.zeros((S, 12)),
                  intr=np.zeros((S, 4)), points=np.zeros((N, 3)))
    outs = [np.zeros(8), np.zeros(S * L.vgg_ba_camrec_len(0, 1)), np.zeros(N * 3), np.zeros(N * 6),
            np.zeros(N * (D + (D & 1)) * 3), np.zeros(8)]
    p = _lib.BAProblem()
    p.S, p.N, p.camera_model, p.intr_mode = S, N, 0, 1
    for k, a in arrays.items():
        setattr(p, k, a.ctypes.data)
    sentinel = [o.copy() for o in outs]
    for tpw in (-4, -1, 1, 2, 6, 30, 102):
        rc = L.vgg_ba_build_blocks(ctypes.byref(p), *[o.ctypes.data for o in outs], tpw, None)
        assert rc == -1, tpw                                         # VGG_EINVAL
        assert b"tracks_per_warp" in L.vgg_last_error()
    # W = NULL selects the LM solve's variant (no coupling blocks stored): it passes the pointer check and meets the
    # same tracks_per_warp check; any other null output is still refused
    no_w = [o.ctypes.data for o in outs]
    no_w[4] = None
    assert L.vgg_ba_build_blocks(ctypes.byref(p), *no_w, 6, None) == -1
    assert b"tracks_per_warp" in L.vgg_last_error()
    no_w[0] = None
    assert L.vgg_ba_build_blocks(ctypes.byref(p), *no_w, 0, None) == -1
    assert b"null pointer" in L.vgg_last_error()
    assert all(np.array_equal(a, b) for a, b in zip(outs, sentinel))


def test_fails_loudly_without_the_library_or_a_gpu(monkeypatch, tmp_path):
    """No fallback path: a missing .so raises NativeLibraryMissing, CPU tensors raise, on every public entry."""
    import pytest
    import torch
    from vggsfm_b200 import bundle_adjustment as ba
    from vggsfm_b200 import corr, pose_refinement as pr, triangulation as tri
    x = torch.zeros(2, 4, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        tri.cam_from_img(x, torch.eye(3).repeat(2, 1, 1))
    with pytest.raises(RuntimeError, match="CUDA"):
        tri.triangulate_tracks(torch.zeros(2, 3, 4), x, track_vis=torch.ones(2, 4))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ba.bundle_adjustment(torch.zeros(4, 3), torch.zeros(2, 3, 4), torch.eye(3).repeat(2, 1, 1), None, x, torch.ones(2, 4, dtype=torch.bool))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        pr.pose_refinement_batched(torch.zeros(2, 3, 4, dtype=torch.float64), torch.zeros(2, 4, dtype=torch.float64),
                                   torch.zeros(4, 3), x, torch.ones(2, 4, dtype=torch.bool), torch.ones(2, dtype=torch.uint8), 0)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        corr.sample_features4d(torch.zeros(1, 3, 8, 8), torch.zeros(1, 5, 2))
    # missing library
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "libvggsfm_b200.so"))
    with pytest.raises(_lib.NativeLibraryMissing, match="no CPU/PyTorch fallback"):
        _lib.lib()
    pcs = _lib.PoseOptions()
    assert pcs.min_inliers == 0                      # ctypes struct layout is importable without the library
