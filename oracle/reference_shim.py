"""Import the UNMODIFIED reference (a facebookresearch/vggsfm checkout named by $VGGSFM_REFERENCE) with stub
third-party modules -- GOLDEN GENERATION ONLY.

The tools/make_golden*.py scripts use it to run the reference and store what the tests compare against under
tests/golden/; no test, smoke() or bench.py calls this module.  Recipe: SURVEY.md Appendix C.
"""
import os
import sys
import types

REFERENCE_ROOT = os.environ.get("VGGSFM_REFERENCE", "")


def available() -> bool:
    return bool(REFERENCE_ROOT) and os.path.isdir(os.path.join(REFERENCE_ROOT, "vggsfm"))


class _Stub(types.ModuleType):
    def __getattr__(self, k):
        if k.startswith("__"):
            raise AttributeError(k)
        m = _Stub(self.__name__ + "." + k)
        setattr(self, k, m)
        return m

    def __call__(self, *a, **kw):
        raise RuntimeError("stub called: " + self.__name__)


_STUBS = ["hydra", "hydra.utils", "pycolmap", "pyceres", "kornia", "kornia.core", "kornia.core.check",
          "kornia.geometry", "kornia.geometry.conversions", "kornia.geometry.linalg", "kornia.geometry.solvers",
          "kornia.geometry.epipolar", "kornia.geometry.epipolar.fundamental", "kornia.geometry.homography",
          "kornia.geometry.calibration", "kornia.geometry.calibration.pnp", "kornia.geometry.subpix",
          "kornia.utils", "kornia.utils._compat", "kornia.utils.grid"]


def install():
    """Put the reference on sys.path with stubs for the absent third-party packages."""
    if not available():
        raise RuntimeError("set VGGSFM_REFERENCE to a facebookresearch/vggsfm checkout")
    import torch
    for name in _STUBS:
        sys.modules.setdefault(name, _Stub(name))
    sys.modules["kornia.core"].Tensor = torch.Tensor
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)


def contiguous_tracks(tn):
    """torch>=2.2 workaround for vggsfm/utils/triangulation.py:817-819 (caller side, no reference edit)."""
    return tn.transpose(0, 1).contiguous().transpose(0, 1)
