// The arithmetic of one observation in the point filter (filter_all_points3D, triangulation_helpers.py:133-307), shared
// by the grid filter (filter_points_kernel) and the observation-list filter (filter_obs_list_kernel) in
// csrc/triangulate.cu, so that the same observation gives the same bit in both.
#pragma once
#include "common.cuh"

namespace vgg {

// squared reprojection error of X in frame s: P = cams[s] (3x4 row-major), K = Ks[s] (3x3 row-major), extra[s] the
// SIMPLE_RADIAL k (extra null: no distortion); the projection goes through nan_to_num (nan = 0, +-inf -> +-max) as the
// reference does, and a point at or behind the camera (depth <= 0) gets 1e6, so it is never an inlier
template <typename TUV>
__device__ __forceinline__ double filter_err2(const double* __restrict__ cams, const double* __restrict__ Ks,
                                              const double* __restrict__ extra, int s, double X0, double X1, double X2,
                                              TUV ou, TUV ov) {
  const double* Pm = cams + (size_t)s * 12;
  const double p0 = Pm[0] * X0 + Pm[1] * X1 + Pm[2] * X2 + Pm[3];
  const double p1 = Pm[4] * X0 + Pm[5] * X1 + Pm[6] * X2 + Pm[7];
  const double p2 = Pm[8] * X0 + Pm[9] * X1 + Pm[10] * X2 + Pm[11];
  double u = p0 / p2, v = p1 / p2;
  if (extra) {
    const double k = extra[s];
    const double rad = k * (u * u + v * v);
    const double du = u * rad, dv = v * rad;
    u = u + du; v = v + dv;
  }
  const double* Km = Ks + (size_t)s * 9;
  double x = Km[0] * u + Km[1] * v + Km[2];
  double y = Km[3] * u + Km[4] * v + Km[5];
  if (x != x) x = 0.0;                       // nan_to_num(nan=0); +-inf -> +-max
  if (y != y) y = 0.0;
  x = fmin(fmax(x, -1.7976931348623157e308), 1.7976931348623157e308);
  y = fmin(fmax(y, -1.7976931348623157e308), 1.7976931348623157e308);
  const double dx = x - (double)ou, dy = y - (double)ov;
  double e2 = dx * dx + dy * dy;
  if (p2 <= 0.0) e2 = 1e6;
  return e2;
}

// |cos| of the angle at X between two centres; returns 2 when the reference's guard gives angle 0
__device__ __forceinline__ double tri_cos_abs(const double* c1, const double* c2, double X0, double X1, double X2) {
  const double b0 = c1[0] - c2[0], b1 = c1[1] - c2[1], b2 = c1[2] - c2[2];
  const double base2 = b0 * b0 + b1 * b1 + b2 * b2;
  const double u0 = X0 - c1[0], u1 = X1 - c1[1], u2 = X2 - c1[2];
  const double w0 = X0 - c2[0], w1 = X1 - c2[1], w2 = X2 - c2[2];
  const double r1 = u0 * u0 + u1 * u1 + u2 * u2;
  const double r2 = w0 * w0 + w1 * w1 + w2 * w2;
  const double den = 2.0 * sqrt(r1 * r2);
  if (den <= 1e-12) return 2.0;
  return fabs((r1 + r2 - base2) / den);    // NaN propagates -> comparison false
}

}  // namespace vgg
