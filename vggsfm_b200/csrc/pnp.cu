// Batched absolute-pose estimation: P3P + LO-RANSAC over host-drawn minimal samples, with COLMAP's focal-length
// ladder -- the fall-back `pycolmap.absolute_pose_estimation` of refine_pose (vggsfm/utils/triangulation.py:404-433,
// estimate_focal_length=True, ransac.max_error=12) and of the video runner's PnP alignment
// (vggsfm/runners/video_runner.py:985-998).  The reference runs it frame after frame on the CPU; here one CTA owns one
// (frame, focal factor) pair -- up to S x 31 independent LO-RANSACs in ONE launch -- and a second small launch picks
// each frame's best factor and writes its inlier mask.  The arithmetic is the one restated in oracle/pnp_oracle.py
// (Grunert's P3P quartic, Ferrari + Newton polishing, support = inlier count then residual sum, local optimisation by
// 4 Gauss-Newton steps on the inliers, at most 10 rounds while the inlier count grows); the non-linear refinement that
// follows in COLMAP is the existing csrc/pose_refine.cu launch (vggsfm_b200/pose_refinement.py).
#include <math.h>
#include "common.cuh"

namespace vgg {

namespace {

constexpr int PNP_THREADS = 256;
constexpr int PNP_MAX_FACTORS = 31;
constexpr int PNP_GN_STEPS = 4;
constexpr int PNP_LOCAL_TRIALS = 10;

__device__ __forceinline__ double cbrt_signed(double x) { return cbrt(x); }

// COLMAP's focal-length ladder 0.2 + 4.8 (k / 30)^2, rounded step by step: a contracted FMA would move a factor by an
// ulp, and with it the focal length the frame reports
__device__ __forceinline__ double focal_factor(int k, int nfac) {
  if (nfac <= 1) return 1.0;
  const double i = (double)k / (double)(nfac - 1);
  return __dadd_rn(0.2, __dmul_rn(__dmul_rn(5.0 - 0.2, i), i));
}

// real roots of A4 x^4 + A3 x^3 + A2 x^2 + A1 x + A0 (same steps as oracle/pnp_oracle.py:solve_quartic_real)
__device__ int solve_quartic_real(double A4, double A3, double A2, double A1, double A0, double* roots) {
  if (!(isfinite(A4) && isfinite(A3) && isfinite(A2) && isfinite(A1) && isfinite(A0)) || fabs(A4) < 1e-300) return 0;
  const double b = A3 / A4, c = A2 / A4, d = A1 / A4, e = A0 / A4;
  const double p = c - 3.0 * b * b / 8.0;
  const double q = d - b * c / 2.0 + b * b * b / 8.0;
  const double r = e - b * d / 4.0 + b * b * c / 16.0 - 3.0 * (b * b) * (b * b) / 256.0;
  const double c2 = p, c1 = p * p / 4.0 - r, c0 = -q * q / 8.0;
  const double P = c1 - c2 * c2 / 3.0;
  const double Q = 2.0 * c2 * c2 * c2 / 27.0 - c2 * c1 / 3.0 + c0;
  const double disc = Q * Q / 4.0 + P * P * P / 27.0;
  double t;
  if (disc >= 0.0) {
    const double s = sqrt(disc);
    t = cbrt_signed(-Q / 2.0 + s) + cbrt_signed(-Q / 2.0 - s);
  } else {
    const double rr = 2.0 * sqrt(-P / 3.0);
    const double phi = acos(fmin(fmax(3.0 * Q / (P * rr), -1.0), 1.0));
    t = rr * cos(phi / 3.0);
  }
  double m = t - c2 / 3.0;
  for (int it = 0; it < 3; ++it) {
    const double fm = ((m + c2) * m + c1) * m + c0;
    const double dm = (3.0 * m + 2.0 * c2) * m + c1;
    if (dm != 0.0) m = m - fm / dm;
  }
  double ys[4];
  int ny = 0;
  if (m > 1e-14 * fmax(1.0, fabs(p))) {
    const double s2m = sqrt(2.0 * m);
    for (int k = 0; k < 2; ++k) {
      const double sg = k == 0 ? 1.0 : -1.0;
      const double bb = -sg * s2m, cc = p / 2.0 + m + sg * q / (2.0 * s2m);
      const double dd = bb * bb - 4.0 * cc;
      if (dd >= 0.0) {
        const double sd = sqrt(dd);
        ys[ny++] = (-bb + sd) / 2.0;
        ys[ny++] = (-bb - sd) / 2.0;
      }
    }
  } else {
    const double dd = p * p - 4.0 * r;
    if (dd >= 0.0) {
      const double z0 = (-p + sqrt(dd)) / 2.0, z1 = (-p - sqrt(dd)) / 2.0;
      if (z0 >= 0.0) { ys[ny++] = sqrt(z0); ys[ny++] = -sqrt(z0); }
      if (z1 >= 0.0) { ys[ny++] = sqrt(z1); ys[ny++] = -sqrt(z1); }
    }
  }
  int n = 0;
  for (int i = 0; i < ny; ++i) {
    double x = ys[i] - b / 4.0;
    for (int it = 0; it < 3; ++it) {
      const double f = (((A4 * x + A3) * x + A2) * x + A1) * x + A0;
      const double df = ((4.0 * A4 * x + 3.0 * A3) * x + 2.0 * A2) * x + A1;
      if (df != 0.0) x = x - f / df;
    }
    if (isfinite(x)) roots[n++] = x;
  }
  return n;
}

__device__ __forceinline__ void cross3(const double* a, const double* b, double* o) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}

// orthonormal frame with columns e1 | e2 | e3 from three points; E row-major [3][3]
__device__ void frame3(const double* p0, const double* p1, const double* p2, double* E) {
  double e1[3] = {p1[0] - p0[0], p1[1] - p0[1], p1[2] - p0[2]};
  const double n1 = sqrt(e1[0] * e1[0] + e1[1] * e1[1] + e1[2] * e1[2]);
  for (int i = 0; i < 3; ++i) e1[i] /= n1;
  const double d2[3] = {p2[0] - p0[0], p2[1] - p0[1], p2[2] - p0[2]};
  double e3[3], e2[3];
  cross3(e1, d2, e3);
  const double n3 = sqrt(e3[0] * e3[0] + e3[1] * e3[1] + e3[2] * e3[2]);
  for (int i = 0; i < 3; ++i) e3[i] /= n3;
  cross3(e3, e1, e2);
  for (int i = 0; i < 3; ++i) { E[i * 3 + 0] = e1[i]; E[i * 3 + 1] = e2[i]; E[i * 3 + 2] = e3[i]; }
}

// f [3][3] unit bearings (rows), X [3][3] world points (rows) -> up to 4 poses [12] (R|t row-major 3x4)
__device__ int p3p_solve(const double* f, const double* X, double* poses) {
  auto d2 = [&](int i, int j) {
    const double a = X[i * 3] - X[j * 3], b = X[i * 3 + 1] - X[j * 3 + 1], c = X[i * 3 + 2] - X[j * 3 + 2];
    return a * a + b * b + c * c;
  };
  auto dot = [&](int i, int j) { return f[i * 3] * f[j * 3] + f[i * 3 + 1] * f[j * 3 + 1] + f[i * 3 + 2] * f[j * 3 + 2]; };
  const double a2 = d2(1, 2), b2 = d2(0, 2), c2 = d2(0, 1);
  const double ca = dot(1, 2), cb = dot(0, 2), cg = dot(0, 1);
  const double A4 = a2 * a2 - 2 * a2 * b2 - 2 * a2 * c2 + b2 * b2 - 4 * b2 * c2 * ca * ca + 2 * b2 * c2 + c2 * c2;
  const double A3 = -4 * (a2 * a2 * cb - a2 * b2 * ca * cg - a2 * b2 * cb - 2 * a2 * c2 * cb + b2 * b2 * ca * cg -
                          2 * b2 * c2 * ca * ca * cb - b2 * c2 * ca * cg + b2 * c2 * cb + c2 * c2 * cb);
  const double A2 = 2 * (2 * a2 * a2 * cb * cb + a2 * a2 - 4 * a2 * b2 * ca * cb * cg - 2 * a2 * b2 * cg * cg -
                         4 * a2 * c2 * cb * cb - 2 * a2 * c2 + 2 * b2 * b2 * ca * ca + 2 * b2 * b2 * cg * cg - b2 * b2 -
                         2 * b2 * c2 * ca * ca - 4 * b2 * c2 * ca * cb * cg + 2 * c2 * c2 * cb * cb + c2 * c2);
  const double A1 = -4 * (a2 * a2 * cb - a2 * b2 * ca * cg - 2 * a2 * b2 * cb * cg * cg + a2 * b2 * cb - 2 * a2 * c2 * cb +
                          b2 * b2 * ca * cg - b2 * c2 * ca * cg - b2 * c2 * cb + c2 * c2 * cb);
  const double A0 = a2 * a2 - 4 * a2 * b2 * cg * cg + 2 * a2 * b2 - 2 * a2 * c2 + b2 * b2 - 2 * b2 * c2 + c2 * c2;
  double roots[4];
  const int nr = solve_quartic_real(A4, A3, A2, A1, A0, roots);
  int ns = 0;
  double Ex[9];
  frame3(X, X + 3, X + 6, Ex);
  for (int k = 0; k < nr; ++k) {
    const double v = roots[k];
    if (!(v > 0.0)) continue;
    const double den = 2.0 * b2 * (ca * v - cg);
    if (fabs(den) < 1e-300) continue;
    const double u = (2 * a2 * cb * v - a2 * v * v - a2 + b2 * v * v - b2 - 2 * c2 * cb * v + c2 * v * v + c2) / den;
    if (!(u > 0.0)) continue;
    const double w = 1.0 + v * v - 2.0 * v * cb;
    if (!(w > 0.0)) continue;
    const double s1 = sqrt(b2 / w);
    double Y[9];
    for (int i = 0; i < 3; ++i) {
      Y[i] = s1 * f[i];
      Y[3 + i] = u * s1 * f[3 + i];
      Y[6 + i] = v * s1 * f[6 + i];
    }
    double Ey[9];
    frame3(Y, Y + 3, Y + 6, Ey);
    double* P = poses + ns * 12;
    bool fin = true;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        const double rij = Ey[i * 3] * Ex[j * 3] + Ey[i * 3 + 1] * Ex[j * 3 + 1] + Ey[i * 3 + 2] * Ex[j * 3 + 2];
        P[i * 4 + j] = rij;
        fin = fin && isfinite(rij);
      }
    for (int i = 0; i < 3; ++i) {
      const double ti = Y[i] - (P[i * 4] * X[0] + P[i * 4 + 1] * X[1] + P[i * 4 + 2] * X[2]);
      P[i * 4 + 3] = ti;
      fin = fin && isfinite(ti);
    }
    if (fin) ++ns;
  }
  return ns;
}

__device__ __forceinline__ double residual_of(const double* P, const double* Xp, double xnx, double xny) {
  const double px = P[0] * Xp[0] + P[1] * Xp[1] + P[2] * Xp[2] + P[3];
  const double py = P[4] * Xp[0] + P[5] * Xp[1] + P[6] * Xp[2] + P[7];
  const double pz = P[8] * Xp[0] + P[9] * Xp[1] + P[10] * Xp[2] + P[11];
  if (!(pz > 0.0)) return INFINITY;
  const double du = px / pz - xnx, dv = py / pz - xny;
  return du * du + dv * dv;
}

// block-wide sums of NV doubles per thread; result valid in red[0..NV) for every thread after the call
template <int NV>
__device__ void block_sum(double (&v)[NV], double* red /*[8*NV + NV]*/, int tid) {
  const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = warp_sum(v[i]);
  __syncthreads();                         // previous readers of `red` are done
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i) red[NV + warp * NV + i] = v[i];
  }
  __syncthreads();
  if (tid < NV) {
    double s = 0.0;
    for (int w = 0; w < PNP_THREADS / 32; ++w) s += red[NV + w * NV + tid];
    red[tid] = s;
  }
  __syncthreads();
}

struct PnpShared {
  double poses[4 * 12];     // candidate poses of the current trial
  double best[12];
  double trial[12];         // local-optimisation iterate
  double red[9 * 27];
  double best_sum;
  int best_cnt;
  int nsol;
  int n_usable;
  int ok;
};

// Cholesky solve of the 6x6 system (H + eps tr(H) I) d = -g on one thread; returns false if not positive definite
__device__ bool solve6(const double* Hs /*21 upper packed row-major*/, const double* g, double* d) {
  double A[6][6];
  int k = 0;
  double tr = 0.0;
  for (int i = 0; i < 6; ++i)
    for (int j = i; j < 6; ++j) { A[i][j] = A[j][i] = Hs[k++]; }
  for (int i = 0; i < 6; ++i) tr += A[i][i];
  for (int i = 0; i < 6; ++i) A[i][i] += 1e-12 * tr;
  double L[6][6];
  for (int j = 0; j < 6; ++j) {
    double s = A[j][j];
    for (int q = 0; q < j; ++q) s -= L[j][q] * L[j][q];
    if (!(s > 0.0)) return false;
    L[j][j] = sqrt(s);
    for (int i = j + 1; i < 6; ++i) {
      double t = A[i][j];
      for (int q = 0; q < j; ++q) t -= L[i][q] * L[j][q];
      L[i][j] = t / L[j][j];
    }
  }
  double y[6];
  for (int i = 0; i < 6; ++i) {
    double t = -g[i];
    for (int q = 0; q < i; ++q) t -= L[i][q] * y[q];
    y[i] = t / L[i][i];
  }
  for (int i = 5; i >= 0; --i) {
    double t = y[i];
    for (int q = i + 1; q < 6; ++q) t -= L[q][i] * d[q];
    d[i] = t / L[i][i];
  }
  for (int i = 0; i < 6; ++i)
    if (!isfinite(d[i])) return false;
  return true;
}

__device__ void exp_so3_apply(const double* w, const double* P, double* out) {
  // out = [exp(w) R | t + dt] is assembled by the caller; here out[0..8] (3x3 row-major) = exp(w)
  const double th = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  double E[9];
  if (th < 1e-12) {
    E[0] = 1; E[1] = -w[2]; E[2] = w[1];
    E[3] = w[2]; E[4] = 1; E[5] = -w[0];
    E[6] = -w[1]; E[7] = w[0]; E[8] = 1;
  } else {
    const double a0 = w[0] / th, a1 = w[1] / th, a2 = w[2] / th;
    const double s = sin(th), c1 = 1.0 - cos(th);
    const double K[9] = {0, -a2, a1, a2, 0, -a0, -a1, a0, 0};
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        double kk = 0.0;
        for (int q = 0; q < 3; ++q) kk += K[i * 3 + q] * K[q * 3 + j];
        E[i * 3 + j] = (i == j ? 1.0 : 0.0) + s * K[i * 3 + j] + c1 * kk;
      }
  }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) out[i * 4 + j] = E[i * 3] * P[j] + E[i * 3 + 1] * P[4 + j] + E[i * 3 + 2] * P[8 + j];
}

// grid (S, nfac); one CTA = LO-RANSAC of one frame at one focal factor.  Results: res_pose [S][nfac][12],
// res_cnt [S][nfac], res_sum [S][nfac] (cnt = 0: nothing found / frame not selected).
__global__ void __launch_bounds__(PNP_THREADS) pnp_ransac_kernel(
    int S, int P, int model, int nfac, int T, double max_error, const float* __restrict__ uv,
    const uint8_t* __restrict__ mask, const uint8_t* __restrict__ frame_flags, const double* __restrict__ points,
    const double* __restrict__ intr, const double* __restrict__ u_samples, double* __restrict__ res_pose,
    int* __restrict__ res_cnt, double* __restrict__ res_sum) {
  extern __shared__ __align__(16) unsigned char pnp_smem[];
  double2* xn = reinterpret_cast<double2*>(pnp_smem);                 // [P] normalised coords of the usable points
  int* cidx = reinterpret_cast<int*>(xn + P);                         // [P] their indices
  uint8_t* inl = reinterpret_cast<uint8_t*>(cidx + P);                // [P] inlier flags of the current best
  __shared__ PnpShared sh;
  __shared__ int scan_warp[PNP_THREADS / 32];
  const int s = blockIdx.x, kf = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const size_t slot = (size_t)s * nfac + kf;
  if (tid == 0) {
    res_cnt[slot] = 0;
    res_sum[slot] = INFINITY;
  }
  if (!frame_flags[s]) return;
  const double f0 = intr[(size_t)s * 4], cx = intr[(size_t)s * 4 + 1], cy = intr[(size_t)s * 4 + 2];
  const double kdist = model == VGG_SIMPLE_RADIAL ? intr[(size_t)s * 4 + 3] : 0.0;
  const double f = f0 * focal_factor(kf, nfac);
  const double thr = max_error / f, thr2 = thr * thr;
  // ---- compaction of the usable points (order preserved) + normalised coordinates
  if (tid == 0) sh.n_usable = 0;
  __syncthreads();
  for (int base = 0; base < P; base += PNP_THREADS) {
    const int i = base + tid;
    const bool use = i < P && mask[(size_t)s * P + i] != 0;
    const unsigned bal = __ballot_sync(0xffffffffu, use);
    if (lane == 0) scan_warp[warp] = __popc(bal);
    __syncthreads();
    int off = sh.n_usable;
    for (int w = 0; w < warp; ++w) off += scan_warp[w];
    if (use) {
      const int pos = off + __popc(bal & ((1u << lane) - 1u));
      double x = ((double)uv[((size_t)s * P + i) * 2] - cx) / f, y = ((double)uv[((size_t)s * P + i) * 2 + 1] - cy) / f;
      if (model == VGG_SIMPLE_RADIAL) {
        const double rd = sqrt(x * x + y * y);
        double r = rd;
        for (int it = 0; it < 20; ++it) r = r - (r * (1.0 + kdist * r * r) - rd) / (1.0 + 3.0 * kdist * r * r);
        const double sc = rd > 0.0 ? r / rd : 1.0;
        x *= sc;
        y *= sc;
      }
      xn[pos] = make_double2(x, y);
      cidx[pos] = i;
    }
    __syncthreads();
    if (tid == 0) {
      int tot = 0;
      for (int w = 0; w < PNP_THREADS / 32; ++w) tot += scan_warp[w];
      sh.n_usable += tot;
    }
    __syncthreads();
  }
  const int n = sh.n_usable;
  if (tid == 0) {
    sh.best_cnt = 0;
    sh.best_sum = INFINITY;
  }
  __syncthreads();
  if (n < 3) return;

  // scores `np` poses at once: cnt/sum into sh.red[0..2np)
  auto score = [&](const double* poses, int np) {
    double acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.0;
    for (int i = tid; i < n; i += PNP_THREADS) {
      const double* Xp = points + (size_t)cidx[i] * 3;
      const double2 o = xn[i];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (q < np) {
          const double r = residual_of(poses + q * 12, Xp, o.x, o.y);
          if (r <= thr2) {
            acc[2 * q] += 1.0;
            acc[2 * q + 1] += r;
          }
        }
      }
    }
    block_sum<8>(acc, sh.red, tid);
  };
  auto mark_inliers = [&](const double* pose) {
    for (int i = tid; i < n; i += PNP_THREADS) {
      const double2 o = xn[i];
      inl[i] = residual_of(pose, points + (size_t)cidx[i] * 3, o.x, o.y) <= thr2 ? 1 : 0;
    }
    __syncthreads();
  };

  for (int t = 0; t < T; ++t) {
    if (tid == 0) {
      int id[3];
      for (int q = 0; q < 3; ++q) {
        const int v = (int)(u_samples[(size_t)t * 3 + q] * (double)n);
        id[q] = v < n - 1 ? v : n - 1;
      }
      int ns = 0;
      if (id[0] != id[1] && id[0] != id[2] && id[1] != id[2]) {
        double fb[9], X3[9];
        for (int q = 0; q < 3; ++q) {
          const double2 o = xn[id[q]];
          const double nr = sqrt(o.x * o.x + o.y * o.y + 1.0);
          fb[q * 3] = o.x / nr; fb[q * 3 + 1] = o.y / nr; fb[q * 3 + 2] = 1.0 / nr;
          for (int c = 0; c < 3; ++c) X3[q * 3 + c] = points[(size_t)cidx[id[q]] * 3 + c];
        }
        ns = p3p_solve(fb, X3, sh.poses);
      }
      sh.nsol = ns;
    }
    __syncthreads();
    const int ns = sh.nsol;
    __syncthreads();                            // thread 0 rewrites sh.nsol at the top of the next trial
    if (ns == 0) continue;
    score(sh.poses, ns);
    for (int q = 0; q < ns; ++q) {
      const int cnt = (int)(sh.red[2 * q] + 0.5);
      const double rs = sh.red[2 * q + 1];
      const bool better = cnt > sh.best_cnt || (cnt == sh.best_cnt && rs < sh.best_sum);
      __syncthreads();                          // everybody evaluated `better` on the same state
      if (!better) continue;
      if (tid < 12) sh.best[tid] = sh.poses[q * 12 + tid];
      if (tid == 0) { sh.best_cnt = cnt; sh.best_sum = rs; }
      __syncthreads();
      mark_inliers(sh.best);
      if (cnt < 4) continue;
      // ---- local optimisation: Gauss-Newton on the inliers of the best model, while the support grows
      double cand[8][2];                         // supports of the remaining candidates (the scratch is reused below)
      for (int qq = q + 1; qq < ns; ++qq) { cand[qq][0] = sh.red[2 * qq]; cand[qq][1] = sh.red[2 * qq + 1]; }
      for (int lt = 0; lt < PNP_LOCAL_TRIALS; ++lt) {
        const int prev = sh.best_cnt;
        if (tid < 12) sh.trial[tid] = sh.best[tid];
        __syncthreads();
        for (int step = 0; step < PNP_GN_STEPS; ++step) {
          double a27[27];
#pragma unroll
          for (int i = 0; i < 27; ++i) a27[i] = 0.0;
          const double* Pt = sh.trial;
          for (int i = tid; i < n; i += PNP_THREADS) {
            if (!inl[i]) continue;
            const double* Xp = points + (size_t)cidx[i] * 3;
            const double a0 = Pt[0] * Xp[0] + Pt[1] * Xp[1] + Pt[2] * Xp[2];
            const double a1 = Pt[4] * Xp[0] + Pt[5] * Xp[1] + Pt[6] * Xp[2];
            const double a2 = Pt[8] * Xp[0] + Pt[9] * Xp[1] + Pt[10] * Xp[2];
            const double pz = a2 + Pt[11];
            const double iz = 1.0 / pz;
            const double u = (a0 + Pt[3]) * iz, v = (a1 + Pt[7]) * iz;
            const double2 o = xn[i];
            const double rx = u - o.x, ry = v - o.y;
            // J rows: jp * [-[a]x | I], jp = [[iz,0,-u iz],[0,iz,-v iz]]
            double J0[6], J1[6];
            J0[3] = iz; J0[4] = 0.0; J0[5] = -u * iz;
            J1[3] = 0.0; J1[4] = iz; J1[5] = -v * iz;
            // -[a]x = [[0,a2,-a1],[-a2,0,a0],[a1,-a0,0]]
            J0[0] = J0[4] * (-a2) + J0[5] * a1;
            J0[1] = J0[3] * a2 + J0[5] * (-a0);
            J0[2] = J0[3] * (-a1) + J0[4] * a0;
            J1[0] = J1[4] * (-a2) + J1[5] * a1;
            J1[1] = J1[3] * a2 + J1[5] * (-a0);
            J1[2] = J1[3] * (-a1) + J1[4] * a0;
            int k = 0;
#pragma unroll
            for (int r = 0; r < 6; ++r)
#pragma unroll
              for (int c = r; c < 6; ++c) a27[k++] += J0[r] * J0[c] + J1[r] * J1[c];
#pragma unroll
            for (int r = 0; r < 6; ++r) a27[21 + r] += J0[r] * rx + J1[r] * ry;
          }
          block_sum<27>(a27, sh.red, tid);
          if (tid == 0) {
            double dstep[6];
            sh.ok = solve6(sh.red, sh.red + 21, dstep) ? 1 : 0;
            if (sh.ok) {
              double out[12];
              exp_so3_apply(dstep, sh.trial, out);
              out[3] = sh.trial[3] + dstep[3];
              out[7] = sh.trial[7] + dstep[4];
              out[11] = sh.trial[11] + dstep[5];
              for (int i = 0; i < 12; ++i) sh.trial[i] = out[i];
            }
          }
          __syncthreads();
          if (!sh.ok) break;
        }
        score(sh.trial, 1);
        const int c2 = (int)(sh.red[0] + 0.5);
        const double r2 = sh.red[1];
        const bool lbetter = c2 > sh.best_cnt || (c2 == sh.best_cnt && r2 < sh.best_sum);
        __syncthreads();
        if (lbetter) {
          if (tid < 12) sh.best[tid] = sh.trial[tid];
          if (tid == 0) { sh.best_cnt = c2; sh.best_sum = r2; }
          __syncthreads();
          mark_inliers(sh.best);
        }
        if (sh.best_cnt <= prev) break;
      }
      __syncthreads();
      for (int qq = q + 1; qq < ns; ++qq) {
        if (tid == 0) { sh.red[2 * qq] = cand[qq][0]; sh.red[2 * qq + 1] = cand[qq][1]; }
      }
      __syncthreads();
    }
  }
  if (tid < 12) res_pose[slot * 12 + tid] = sh.best[tid];
  if (tid == 0) {
    res_cnt[slot] = sh.best_cnt >= 3 ? sh.best_cnt : 0;
    res_sum[slot] = sh.best_sum;
  }
}

// one CTA per frame: best factor (largest inlier count, first wins ties), pose / focal / inlier mask out
__global__ void pnp_select_kernel(int S, int P, int model, int nfac, double max_error, const float* __restrict__ uv,
                                  const uint8_t* __restrict__ mask, const uint8_t* __restrict__ frame_flags,
                                  const double* __restrict__ points, const double* __restrict__ intr,
                                  const double* __restrict__ res_pose, const int* __restrict__ res_cnt,
                                  double* __restrict__ pose_out, double* __restrict__ focal_out,
                                  int* __restrict__ ninl_out, uint8_t* __restrict__ inl_out) {
  const int s = blockIdx.x, tid = threadIdx.x;
  __shared__ int best_k;
  if (tid == 0) {
    int bk = -1, bc = 0;
    if (frame_flags[s])
      for (int k = 0; k < nfac; ++k)
        if (res_cnt[(size_t)s * nfac + k] > bc) { bc = res_cnt[(size_t)s * nfac + k]; bk = k; }
    best_k = bk;
    ninl_out[s] = bc;
  }
  __syncthreads();
  const int bk = best_k;
  if (bk < 0) {
    for (int i = tid; i < P; i += blockDim.x) inl_out[(size_t)s * P + i] = 0;
    if (tid == 0) focal_out[s] = intr[(size_t)s * 4];
    return;
  }
  const double f0 = intr[(size_t)s * 4], cx = intr[(size_t)s * 4 + 1], cy = intr[(size_t)s * 4 + 2];
  const double kdist = model == VGG_SIMPLE_RADIAL ? intr[(size_t)s * 4 + 3] : 0.0;
  const double f = f0 * focal_factor(bk, nfac), thr = max_error / f, thr2 = thr * thr;
  const double* Pb = res_pose + ((size_t)s * nfac + bk) * 12;
  if (tid < 12) pose_out[(size_t)s * 12 + tid] = Pb[tid];
  if (tid == 0) focal_out[s] = f;
  for (int i = tid; i < P; i += blockDim.x) {
    uint8_t v = 0;
    if (mask[(size_t)s * P + i]) {
      double x = ((double)uv[((size_t)s * P + i) * 2] - cx) / f, y = ((double)uv[((size_t)s * P + i) * 2 + 1] - cy) / f;
      if (model == VGG_SIMPLE_RADIAL) {
        const double rd = sqrt(x * x + y * y);
        double r = rd;
        for (int it = 0; it < 20; ++it) r = r - (r * (1.0 + kdist * r * r) - rd) / (1.0 + 3.0 * kdist * r * r);
        const double sc = rd > 0.0 ? r / rd : 1.0;
        x *= sc;
        y *= sc;
      }
      v = residual_of(Pb, points + (size_t)i * 3, x, y) <= thr2 ? 1 : 0;
    }
    inl_out[(size_t)s * P + i] = v;
  }
}

}  // namespace

}  // namespace vgg

using namespace vgg;

extern "C" {

int vgg_pnp_workspace_bytes(int S, int estimate_focal_length, size_t* bytes) {
  VGG_REQUIRE(S >= 0 && bytes, "bad arguments");
  const size_t nfac = estimate_focal_length ? PNP_MAX_FACTORS : 1;
  *bytes = align_up((size_t)S * nfac * 12 * 8, 256) + align_up((size_t)S * nfac * 4, 256) + align_up((size_t)S * nfac * 8, 256);
  return VGG_OK;
}

int vgg_absolute_pose_estimation(int S, int P, int camera_model, const float* uv, const uint8_t* mask,
                                 const uint8_t* frame_flags, const double* points, const double* intr,
                                 const double* u_samples, int num_trials, int estimate_focal_length, double max_error,
                                 double* pose_out, double* focal_out, int* num_inliers_out, uint8_t* inlier_out,
                                 void* workspace, size_t ws_bytes, void* stream) {
  VGG_REQUIRE(camera_model == VGG_SIMPLE_PINHOLE || camera_model == VGG_SIMPLE_RADIAL, "bad camera_model");
  VGG_REQUIRE(S >= 0 && P >= 0 && num_trials >= 1, "bad sizes");
  g_launch_count = 0;
  if (S == 0) return VGG_OK;
  VGG_REQUIRE(uv && mask && frame_flags && points && intr && u_samples && pose_out && focal_out && num_inliers_out &&
                  inlier_out && workspace, "null pointer");
  const int nfac = estimate_focal_length ? PNP_MAX_FACTORS : 1;
  size_t need = 0;
  vgg_pnp_workspace_bytes(S, estimate_focal_length, &need);
  if (ws_bytes < need) {
    set_error("pnp workspace too small: need %zu bytes", need);
    return VGG_EWORKSPACE;
  }
  const size_t smem = (size_t)P * (sizeof(double2) + sizeof(int) + 1) + 16;
  VGG_REQUIRE(smem <= 200 * 1024, "absolute pose estimation: at most 9751 points per call (shared-memory resident)");
  cudaStream_t st = (cudaStream_t)stream;
  Carver c(workspace, ws_bytes);
  double* res_pose = c.take<double>((size_t)S * nfac * 12);
  int* res_cnt = c.take<int>((size_t)S * nfac);
  double* res_sum = c.take<double>((size_t)S * nfac);
  VGG_CUDA_CHECK(cudaFuncSetAttribute(pnp_ransac_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  pnp_ransac_kernel<<<dim3(S, nfac), PNP_THREADS, smem, st>>>(S, P, camera_model, nfac, num_trials, max_error, uv, mask,
                                                              frame_flags, points, intr, u_samples, res_pose, res_cnt, res_sum);
  VGG_LAUNCH_CHECK();
  pnp_select_kernel<<<S, 256, 0, st>>>(S, P, camera_model, nfac, max_error, uv, mask, frame_flags, points, intr, res_pose,
                                       res_cnt, pose_out, focal_out, num_inliers_out, inlier_out);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

}  // extern "C"
