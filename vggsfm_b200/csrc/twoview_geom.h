// Device geometry shared by the two-view kernels (csrc/twoview.cu, csrc/twoview_msac.cu): the pinned 7-point solver
// of DESIGN.md section 3 and the small dense algebra around it.  Included once per translation unit.
#pragma once
#include <math.h>

namespace vgg {
namespace {

constexpr double TV_HOM = 1.0 / (1.0 + 1e-8);                 // kornia's homogeneous division at z = 1
constexpr double TV_SQRT2_F32 = 1.41421353816986083984375;    // torch.sqrt(torch.tensor(2.0)), float32

template <typename TP>
__device__ __forceinline__ double2 ldp(const TP* p, size_t i) {
  return make_double2((double)p[2 * i], (double)p[2 * i + 1]);
}

// -------------------------------------------------------------------------------------------------------------------
// small dense algebra on one thread
// -------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double det3(const double* m) {
  return m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
}

// tr(a adj(b)) = tr(a inv(b)) det(b)
__device__ __forceinline__ double tr_adj(const double* a, const double* b) {
  double adj[9];
  adj[0] = b[4] * b[8] - b[5] * b[7]; adj[1] = b[2] * b[7] - b[1] * b[8]; adj[2] = b[1] * b[5] - b[2] * b[4];
  adj[3] = b[5] * b[6] - b[3] * b[8]; adj[4] = b[0] * b[8] - b[2] * b[6]; adj[5] = b[2] * b[3] - b[0] * b[5];
  adj[6] = b[3] * b[7] - b[4] * b[6]; adj[7] = b[1] * b[6] - b[0] * b[7]; adj[8] = b[0] * b[4] - b[1] * b[3];
  double t = 0.0;
  for (int i = 0; i < 3; ++i)
    for (int k = 0; k < 3; ++k) t += a[i * 3 + k] * adj[k * 3 + i];
  return t;
}

// cyclic Jacobi on a symmetric n x n (row-major, destroyed): eigenvalues w, eigenvectors in the columns of V.
// Unrolled for the 3 x 3 / 4 x 4 cases (registers); the 9 x 9 case runs rolled on shared-memory A and V.
template <int n>
__device__ void jacobi_eig(double* A, double* V, double* w) {
#pragma unroll(n > 4 ? 1 : 16)
  for (int i = 0; i < n * n; ++i) V[i] = (i % (n + 1) == 0) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 50; ++sweep) {
    double off = 0.0;
#pragma unroll(n > 4 ? 1 : 16)
    for (int p = 0; p < n; ++p)
#pragma unroll(n > 4 ? 1 : 16)
      for (int q = p + 1; q < n; ++q) off += fabs(A[p * n + q]);
    if (off == 0.0) break;
#pragma unroll(n > 4 ? 1 : 16)
    for (int p = 0; p < n; ++p)
#pragma unroll(n > 4 ? 1 : 16)
      for (int q = p + 1; q < n; ++q) {
        const double apq = A[p * n + q];
        const double app = A[p * n + p], aqq = A[q * n + q];
        const double g = 100.0 * fabs(apq);
        if (sweep > 3 && fabs(app) + g == fabs(app) && fabs(aqq) + g == fabs(aqq)) {
          A[p * n + q] = A[q * n + p] = 0.0;
          continue;
        }
        if (apq == 0.0) continue;
        const double theta = (aqq - app) / (2.0 * apq);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll(n > 4 ? 1 : 16)
        for (int k = 0; k < n; ++k) {
          const double akp = A[k * n + p], akq = A[k * n + q];
          A[k * n + p] = c * akp - s * akq;
          A[k * n + q] = s * akp + c * akq;
        }
#pragma unroll(n > 4 ? 1 : 16)
        for (int k = 0; k < n; ++k) {
          const double apk = A[p * n + k], aqk = A[q * n + k];
          A[p * n + k] = c * apk - s * aqk;
          A[q * n + k] = s * apk + c * aqk;
        }
        A[p * n + q] = A[q * n + p] = 0.0;
#pragma unroll(n > 4 ? 1 : 16)
        for (int k = 0; k < n; ++k) {
          const double vkp = V[k * n + p], vkq = V[k * n + q];
          V[k * n + p] = c * vkp - s * vkq;
          V[k * n + q] = s * vkp + c * vkq;
        }
      }
  }
#pragma unroll(n > 4 ? 1 : 16)
  for (int i = 0; i < n; ++i) w[i] = A[i * n + i];
}

__device__ __forceinline__ void normalize_transformation(double* F) {
  const double n = F[8];
  if (fabs(n) > 1e-8) {
    const double d = n + 1e-8;
    for (int i = 0; i < 9; ++i) F[i] = F[i] / d;
  }
}

// F <- T2^T F T1 with T = [[s,0,-s mx],[0,s,-s my],[0,0,1]]
__device__ __forceinline__ void denormalize(double* F, const double* t1, const double* t2) {
  double T1[9] = {t1[0], 0.0, -t1[0] * t1[1], 0.0, t1[0], -t1[0] * t1[2], 0.0, 0.0, 1.0};
  double T2[9] = {t2[0], 0.0, -t2[0] * t2[1], 0.0, t2[0], -t2[0] * t2[2], 0.0, 0.0, 1.0};
  double G[9], H[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double s = 0.0;
      for (int k = 0; k < 3; ++k) s += F[i * 3 + k] * T1[k * 3 + j];
      G[i * 3 + j] = s;
    }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double s = 0.0;
      for (int k = 0; k < 3; ++k) s += T2[k * 3 + i] * G[k * 3 + j];
      H[i * 3 + j] = s;
    }
  for (int i = 0; i < 9; ++i) F[i] = H[i];
}

// kornia's solve_cubic (oracle/twoview_oracle.py:solve_cubic): real roots, other slots 0
// returns the number of leading slots that hold real roots (0 to 3)
__device__ int solve_cubic(double a, double b, double c, double d, double* x) {
  x[0] = x[1] = x[2] = 0.0;
  if (a == 0.0) {
    if (b == 0.0) {
      if (c != 0.0) x[0] = -d / c;
      return c != 0.0 ? 1 : 0;
    }
    const double delta = c * c - 4.0 * b * d, inv_2a = 0.5 / b;
    if (delta == 0.0) {
      x[0] = x[1] = -c * inv_2a;
    } else if (delta > 0.0) {
      const double sd = sqrt(delta);
      x[0] = (-c + sd) * inv_2a;
      x[1] = (-c - sd) * inv_2a;
    }
    return delta >= 0.0 ? 2 : 0;
  }
  const double inv_a = 1.0 / a;
  const double b_a = b * inv_a, b_a2 = b_a * b_a, c_a = c * inv_a, d_a = d * inv_a;
  const double Q = (3.0 * c_a - b_a2) / 9.0;
  const double R = (9.0 * b_a * c_a - 27.0 * d_a - 2.0 * b_a * b_a2) / 54.0;
  const double Q3 = Q * Q * Q, D = Q3 + R * R, b_a_3 = (1.0 / 3.0) * b_a;
  if (Q == 0.0) {
    if (R != 0.0) x[0] = cbrt(2.0 * R) - b_a_3;
    else x[0] = x[1] = x[2] = -b_a_3;
    return R != 0.0 ? 1 : 3;
  } else if (D <= 0.0) {
    const double th = acos(fmin(fmax(R / sqrt(-Q3), -1.0), 1.0));
    const double sq = 2.0 * sqrt(-Q);
    for (int k = 0; k < 3; ++k) x[k] = sq * cos((th + 2.0 * k * M_PI) / 3.0) - b_a_3;
    return 3;
  }
  const double AD = (R >= 0.0 ? 1.0 : -1.0) * cbrt(fabs(R) + sqrt(D));
  const double BD = AD == 0.0 ? 0.0 : -Q / AD;
  x[0] = AD + BD - b_a_3;
  return 1;
}

// kornia normalize_points over 7 points: returns (scale, mean x, mean y) and the normalised points
__device__ void normalize7(const double2* p, double2* pn, double* t) {
  double mx = 0.0, my = 0.0;
  for (int i = 0; i < 7; ++i) { mx += p[i].x; my += p[i].y; }
  mx /= 7.0;
  my /= 7.0;
  double sd = 0.0;
  for (int i = 0; i < 7; ++i) {
    const double dx = p[i].x - mx, dy = p[i].y - my;
    sd += sqrt(dx * dx + dy * dy);
  }
  const double s = TV_SQRT2_F32 / (sd / 7.0 + 1e-8);
  t[0] = s; t[1] = mx; t[2] = my;
  for (int i = 0; i < 7; ++i) pn[i] = make_double2((s * p[i].x + (-s * mx)) * TV_HOM, (s * p[i].y + (-s * my)) * TV_HOM);
}

// 7-point solve (fundamental.py:341-469) with the pinned null-space basis (oracle: null_basis); F [3][9], returns how
// many leading candidates come from real roots (the others are built from solve_cubic's zero-filled slots).
// Three kernels recompute the candidates of a trial (scoring, LO seeds, the winner); one out-of-line body gives them
// the same bits, whatever FMA contraction the compiler would choose in each inlining context.
__device__ __noinline__ int seven_point(const double2* a, const double2* b, double* F) {
  double2 an[7], bn[7];
  double t1[3], t2[3];
  normalize7(a, an, t1);
  normalize7(b, bn, t2);
  double A[7][9];
  for (int i = 0; i < 7; ++i) {
    const double x1 = an[i].x, y1 = an[i].y, x2 = bn[i].x, y2 = bn[i].y;
    A[i][0] = x2 * x1; A[i][1] = x2 * y1; A[i][2] = x2; A[i][3] = y2 * x1; A[i][4] = y2 * y1; A[i][5] = y2;
    A[i][6] = x1; A[i][7] = y1; A[i][8] = 1.0;
  }
  int pcol[7], rank = 0;
  bool is_piv[9];
  for (int c = 0; c < 9; ++c) {
    is_piv[c] = false;
    if (rank >= 7) continue;
    int p = rank;
    double mx = fabs(A[rank][c]);
    for (int r = rank + 1; r < 7; ++r)
      if (fabs(A[r][c]) > mx) { mx = fabs(A[r][c]); p = r; }
    if (!(mx > 0.0)) continue;
    if (p != rank)
      for (int j = 0; j < 9; ++j) { const double tt = A[rank][j]; A[rank][j] = A[p][j]; A[p][j] = tt; }
    const double piv = A[rank][c];
    for (int r = rank + 1; r < 7; ++r) {
      const double f = A[r][c] / piv;
      for (int j = c; j < 9; ++j) A[r][j] -= f * A[rank][j];
      A[r][c] = 0.0;
    }
    pcol[rank] = c;
    is_piv[c] = true;
    ++rank;
  }
  int fa = -1, fb = -1;
  for (int c = 0; c < 9; ++c)
    if (!is_piv[c]) { fa = fb; fb = c; }
  double f[2][9];
  for (int w = 0; w < 2; ++w) {
    double* x = f[w];
    for (int j = 0; j < 9; ++j) x[j] = 0.0;
    x[w == 0 ? fa : fb] = 1.0;
    for (int i = rank - 1; i >= 0; --i) {
      const int pc = pcol[i];
      double s = 0.0;
      for (int j = pc + 1; j < 9; ++j) s += A[i][j] * x[j];
      x[pc] = -s / A[i][pc];
    }
  }
  double* f1 = f[0];
  double* f2 = f[1];
  if (det3(f1) == 0.0)
    for (int i = 0; i < 9; ++i) f1[i] = (i % 4 == 0) ? 1.0 : 0.0;
  if (det3(f2) == 0.0)
    for (int i = 0; i < 9; ++i) f2[i] = (i % 4 == 0) ? 1.0 : 0.0;
  const double d1 = det3(f1), d2 = det3(f2);
  double roots[3];
  const int nreal = solve_cubic(d1, tr_adj(f2, f1), tr_adj(f1, f2), d2, roots);
  for (int k = 0; k < 3; ++k) {
    const double s = f1[8] * roots[k] + f2[8];
    const bool nz = !(fabs(s) <= 1e-8);
    const double mu = nz ? 1.0 / s : 1.0;
    const double lam = nz ? roots[k] * mu : roots[k];
    double* Fk = F + 9 * k;
    for (int i = 0; i < 9; ++i) Fk[i] = f1[i] * lam + f2[i] * mu;
    Fk[8] = nz ? 1.0 : 0.0;
    denormalize(Fk, t1, t2);
    normalize_transformation(Fk);
  }
  return nreal;
}

}  // namespace
}  // namespace vgg
