"""CPU oracle for the vggsfm_b200 hot path -- TEST INFRASTRUCTURE ONLY.

Nothing under ``oracle/`` is product code.  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs may import it, and only as the checker / the timed CPU baseline.  The product
package ``vggsfm_b200`` never imports this package and fails loudly when its CUDA
library is missing.

Modules
  ba_oracle    numpy float64 restatement of COLMAP 3.10's bundle adjustment
               (``ReprojErrorCostFunction`` + Ceres 2.x Levenberg-Marquardt with a
               direct Schur solve).  PARITY UNPINNED: pycolmap/pyceres are absent from
               this environment and from the reference, and the reference holds no golden
               vectors for this boundary (SURVEY.md section 8c).  Self-validated against
               scipy.optimize.least_squares and finite differences instead.
  tri_oracle   numpy float64 restatement of the reference's pure-torch triangulation
               side (vggsfm/utils/triangulation.py, triangulation_helpers.py,
               distortion.py, two_view_geo/utils.py:63-87).  PINNED: checked against the
               reference itself, imported in the build container with stub third-party
               modules (oracle/reference_shim.py), through the fixtures in tests/golden/.
  corr_oracle  torch-CPU float32 restatement of CorrBlock.corr + CorrBlock.sample
               (vggsfm/models/track_modules/blocks.py:338-416).  PINNED the same way.
"""
