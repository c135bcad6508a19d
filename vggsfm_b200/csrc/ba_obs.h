// The Jacobian of one observation, shared by every bundle-adjustment kernel that needs one: ba_blocks (cost, camera
// records, point blocks), z_build (the Schur operand Zt = W M) and backsub (W^T d_c).  W = J_c^T J_p is never stored
// in the solve; the kernels that use it rebuild it from the observation with this one function, so every copy of a
// block is the same arithmetic.
#pragma once
#include <float.h>
#include <utility>
#include "common.cuh"

namespace vgg {

template <int MODEL, int MODE>
struct BlkCfg {
  static constexpr int NI = (MODEL == VGG_SIMPLE_PINHOLE) ? 1 : 2;
  static constexpr int DC = (MODE == VGG_INTR_PER_FRAME) ? 6 + NI : 6;
  static constexpr int NS = (MODE == VGG_INTR_SHARED) ? NI : 0;
  static constexpr int NPACK = DC * (DC + 1) / 2;
  static constexpr int KR = DC + NPACK + 6 * NS;   // per-frame camera record length
};

// Robust loss of a problem as the kernels take it (vgg_ba_problem.loss_function_type / _scale): SOFT_L1 or CAUCHY, b = a^2,
// c = 1 / b.  The kernels of the trivial loss are separate instantiations (ROBUST = false) that never read it.
struct BaLoss {
  int type;
  double b, c;
};
inline BaLoss ba_loss_of(const vgg_ba_problem* p) {
  const double a = p->loss_function_scale;
  return BaLoss{p->loss_function_type, a * a, 1.0 / (a * a)};
}

// One observation, branch-free: residual and Jacobian columns.  An invalid observation computes on a safe depth and its
// outputs are SELECTED to exact zeros, never multiplied by the mask: its uv, its point and its camera are then free to be
// anything, NaN and inf included (a point or a frame that no valid observation sees is not in the problem, and 0 * NaN
// would put it back).  jc: delta(3), t(3), f, k; jx: point(3).
// cam: R (row-major 3x4 with t), f, cx, cy, k at cam[0], cam[cs], ..., cam[15 cs]; pc: the point is held constant.
// cost: the observation's term of the cost, rho(s) / 2 with s = rx^2 + ry^2.  ROBUST: Ceres' Corrector for a loss with
// rho'' <= 0 (SOFT_L1 and CAUCHY everywhere), i.e. residual and Jacobian scaled by sqrt(rho'), so that every block and
// product built from them below is the robust one.  An invalid observation has s = 0, rho' = 1: still exact zeros.
template <int MODEL, bool ROBUST>
__device__ __forceinline__ void obs_math(const double* cam, int cs, double X0, double X1, double X2, bool pc, float ox,
                                         float oy, bool valid, double* jc0, double* jc1, double* jx0, double* jx1,
                                         double& rx, double& ry, const BaLoss& loss, double& cost) {
  const double R00 = cam[0 * cs], R01 = cam[1 * cs], R02 = cam[2 * cs], t0_ = cam[3 * cs];
  const double R10 = cam[4 * cs], R11 = cam[5 * cs], R12 = cam[6 * cs], t1_ = cam[7 * cs];
  const double R20 = cam[8 * cs], R21 = cam[9 * cs], R22 = cam[10 * cs], t2_ = cam[11 * cs];
  const double fo = cam[12 * cs], cx = cam[13 * cs], cy = cam[14 * cs];
  const double kk = (MODEL == VGG_SIMPLE_RADIAL) ? cam[15 * cs] : 0.0;
  const double a1 = R00 * X0 + R01 * X1 + R02 * X2;
  const double a2 = R10 * X0 + R11 * X1 + R12 * X2;
  const double a3 = R20 * X0 + R21 * X1 + R22 * X2;
  const double px = a1 + t0_, py = a2 + t1_;
  const double pz = valid ? (a3 + t2_) : 1.0;
  const double iz = 1.0 / pz;
  const double u = px * iz, w_ = py * iz;
  const double r2 = u * u + w_ * w_;
  const double d = 1.0 + kk * r2;
  rx = valid ? (fo * d * u + cx - (double)ox) : 0.0;
  ry = valid ? (fo * d * w_ + cy - (double)oy) : 0.0;
  double a00, a01, a11;
  if (MODEL == VGG_SIMPLE_RADIAL) {
    a00 = fo * (d + 2.0 * kk * u * u);
    a01 = fo * (2.0 * kk * u * w_);
    a11 = fo * (d + 2.0 * kk * w_ * w_);
  } else {
    a00 = fo; a01 = 0.0; a11 = fo;
  }
  // Jproj (2x3) = f*A * iz*[[1,0,-u],[0,1,-v]] and the rotated point, selected to zero for an invalid observation: the
  // products below are then exact zeros whatever the point and the camera hold
  const double j00 = valid ? a00 * iz : 0.0, j01 = valid ? a01 * iz : 0.0, j02 = valid ? -(a00 * u + a01 * w_) * iz : 0.0;
  const double j10 = valid ? a01 * iz : 0.0, j11 = valid ? a11 * iz : 0.0, j12 = valid ? -(a01 * u + a11 * w_) * iz : 0.0;
  const double b1 = valid ? 2.0 * a1 : 0.0, b2 = valid ? 2.0 * a2 : 0.0, b3 = valid ? 2.0 * a3 : 0.0;
  jc0[0] = b2 * j02 - b3 * j01;  jc1[0] = b2 * j12 - b3 * j11;
  jc0[1] = b3 * j00 - b1 * j02;  jc1[1] = b3 * j10 - b1 * j12;
  jc0[2] = b1 * j01 - b2 * j00;  jc1[2] = b1 * j11 - b2 * j10;
  jc0[3] = j00; jc0[4] = j01; jc0[5] = j02;
  jc1[3] = j10; jc1[4] = j11; jc1[5] = j12;
  jc0[6] = valid ? d * u : 0.0;            jc1[6] = valid ? d * w_ : 0.0;
  jc0[7] = valid ? fo * u * r2 : 0.0;      jc1[7] = valid ? fo * w_ * r2 : 0.0;
  const bool vp = valid && !pc;                                  // constant point: no point columns
  jx0[0] = vp ? j00 * R00 + j01 * R10 + j02 * R20 : 0.0;
  jx0[1] = vp ? j00 * R01 + j01 * R11 + j02 * R21 : 0.0;
  jx0[2] = vp ? j00 * R02 + j01 * R12 + j02 * R22 : 0.0;
  jx1[0] = vp ? j10 * R00 + j11 * R10 + j12 * R20 : 0.0;
  jx1[1] = vp ? j10 * R01 + j11 * R11 + j12 * R21 : 0.0;
  jx1[2] = vp ? j10 * R02 + j11 * R12 + j12 * R22 : 0.0;
  if constexpr (!ROBUST) {
    cost = 0.5 * (rx * rx + ry * ry);
  } else {
    // rho in forms without cancellation (the same functions as Ceres' b log(1 + s c) and 2 b (sqrt(1 + s c) - 1)), so
    // that a large scale reduces to the trivial loss to rounding; rho' = max(DBL_MIN, 1 / (1 + s c)) resp.
    // max(DBL_MIN, 1 / sqrt(1 + s c)).  One uniform branch per launch: the loss type is the same for every thread.
    const double s = rx * rx + ry * ry;
    const double x = s * loss.c;
    double rho, rho1;
    if (loss.type == VGG_LOSS_CAUCHY) {
      rho = loss.b * log1p(x);
      rho1 = fmax(DBL_MIN, 1.0 / (1.0 + x));
    } else {
      const double t = sqrt(1.0 + x);
      rho = t < 2.0 ? 2.0 * s / (1.0 + t) : 2.0 * loss.b * (t - 1.0);
      rho1 = fmax(DBL_MIN, 1.0 / t);
    }
    cost = 0.5 * rho;
    const double k = sqrt(rho1);
    rx *= k;
    ry *= k;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      jc0[i] *= k;
      jc1[i] *= k;
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      jx0[i] *= k;
      jx1[i] *= k;
    }
  }
}

// one entry of the coupling block W = J_c^T J_p: row i of the camera columns (6 + intrinsics), point column c
__device__ __forceinline__ double w_entry(const double* jc0, const double* jc1, const double* jx0, const double* jx1,
                                          int i, int c) {
  return jc0[i] * jx0[c] + jc1[i] * jx1[c];
}

// ---- compile-time layout of the per-frame camera record: g_c[DC] | H_cc upper-packed | H_cs[6][NS] ----
__host__ __device__ constexpr int pack_row(int dc, int p) {
  int i = 0;
  while (p >= dc - i) { p -= dc - i; ++i; }
  return i;
}
__host__ __device__ constexpr int pack_col(int dc, int p) {
  int i = 0;
  while (p >= dc - i) { p -= dc - i; ++i; }
  return i + p;
}

// one observation's terms of its frame's camera record (ba_blocks on the grid, ba_list on the observation list)
template <int DC, int NS, int K, int KR>
__device__ __forceinline__ void cam_accumulate_one(double (&acc)[KR], const double* jc0, const double* jc1, double rx,
                                                   double ry) {
  constexpr int NPACK = DC * (DC + 1) / 2;
  if constexpr (K < DC) {
    acc[K] = fma(jc0[K], rx, fma(jc1[K], ry, acc[K]));
  } else if constexpr (K < DC + NPACK) {
    constexpr int i = pack_row(DC, K - DC), j = pack_col(DC, K - DC);
    acc[K] = fma(jc0[i], jc0[j], fma(jc1[i], jc1[j], acc[K]));
  } else {
    constexpr int q = K - DC - NPACK;
    constexpr int i = q / (NS > 0 ? NS : 1), j = q % (NS > 0 ? NS : 1);
    acc[K] = fma(jc0[i], jc0[6 + j], fma(jc1[i], jc1[6 + j], acc[K]));
  }
}
template <int DC, int NS, int KR, int... K>
__device__ __forceinline__ void cam_accumulate(double (&acc)[KR], const double* jc0, const double* jc1, double rx,
                                               double ry, std::integer_sequence<int, K...>) {
  (cam_accumulate_one<DC, NS, K, KR>(acc, jc0, jc1, rx, ry), ...);
}

}  // namespace vgg

// the instantiation of a bundle-adjustment kernel template for the problem's camera model and intrinsics mode
#define VGG_PICK_BA_KERNEL(kern, tmpl, p)                                                          \
  decltype(&tmpl<0, 0, false>) kern = nullptr;                                                      \
  {                                                                                                 \
    const bool robust = (p)->loss_function_type != VGG_LOSS_TRIVIAL;                               \
    switch ((p)->camera_model * 3 + (p)->intr_mode) {                                               \
      case 0: kern = robust ? tmpl<0, 0, true> : tmpl<0, 0, false>; break;                           \
      case 1: kern = robust ? tmpl<0, 1, true> : tmpl<0, 1, false>; break;                           \
      case 2: kern = robust ? tmpl<0, 2, true> : tmpl<0, 2, false>; break;                           \
      case 3: kern = robust ? tmpl<1, 0, true> : tmpl<1, 0, false>; break;                           \
      case 4: kern = robust ? tmpl<1, 1, true> : tmpl<1, 1, false>; break;                           \
      case 5: kern = robust ? tmpl<1, 2, true> : tmpl<1, 2, false>; break;                           \
    }                                                                                               \
  }                                                                                                 \
  VGG_REQUIRE(kern, "bad camera_model/intr_mode")
