// Fused LORANSAC multi-view triangulation (one CTA per track) and the reprojection / triangulation-
// angle filter.
//
// Replaces the reference's batched-PyTorch pipeline
//   triangulate_tracks_single_chunk        vggsfm/utils/triangulation.py:776-956
//   local_refine_and_compute_error         vggsfm/utils/triangulation.py:959-1017
//   local_refinement_tri / DLT / angular error / triangulation angle
//                                          vggsfm/utils/triangulation_helpers.py:27-131,431-587,648-725
//   calculate_residual_indicator           vggsfm/two_view_geo/utils.py:63-87
//   filter_all_points3D_single_chunk       vggsfm/utils/triangulation_helpers.py:215-307
//   triangulate_by_pair                    vggsfm/utils/triangulation.py:45-135
// which materialises [tracks x hypotheses x frames] tensors in HBM (1.7 GB f64 per 2048-track chunk at
// 400 frames) plus an [N, S^2] camera-pair angle table per refined hypothesis.  Here nothing of that
// leaves the SM: cameras (S x 96 B) are staged once per CTA into shared memory with TMA bulk copies,
// the 4x4 DLT eigenproblems are solved in registers with cyclic Jacobi, hypothesis scores live in
// shared memory as inlier bitmasks, and the "exists a camera pair with >= 1.5 deg" test is an
// early-exit search instead of a table.  Minimal HBM traffic: S*N*(16+2) B in, N*(24+8+S) B out.
// All arithmetic is float64 like the reference's real pipeline (triangulator.py:91).
#include "common.cuh"
#include "tri_obs.h"

namespace vgg {

constexpr double kPi = 3.14159265358979323846;
constexpr int TRI_THREADS = 256;

// ---- symmetric 4x4 eigen-solver (cyclic Jacobi), returns eigenvector of the smallest eigenvalue ----
// a: 00,01,02,03,11,12,13,22,23,33
__device__ __forceinline__ void smallest_eigvec4(const double* a_in, double* v_out) {
  double A[4][4], V[4][4];
  A[0][0] = a_in[0]; A[0][1] = A[1][0] = a_in[1]; A[0][2] = A[2][0] = a_in[2]; A[0][3] = A[3][0] = a_in[3];
  A[1][1] = a_in[4]; A[1][2] = A[2][1] = a_in[5]; A[1][3] = A[3][1] = a_in[6];
  A[2][2] = a_in[7]; A[2][3] = A[3][2] = a_in[8]; A[3][3] = a_in[9];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) V[i][j] = (i == j) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 12; ++sweep) {
    const double off = A[0][1] * A[0][1] + A[0][2] * A[0][2] + A[0][3] * A[0][3] + A[1][2] * A[1][2] +
                       A[1][3] * A[1][3] + A[2][3] * A[2][3];
    const double dg = A[0][0] * A[0][0] + A[1][1] * A[1][1] + A[2][2] * A[2][2] + A[3][3] * A[3][3];
    if (!(off > 1e-34 * dg)) break;        // also leaves on NaN
#pragma unroll
    for (int p = 0; p < 3; ++p) {
#pragma unroll
      for (int q = p + 1; q < 4; ++q) {
        const double apq = A[p][q];
        if (apq != 0.0) {
          const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
          const double t = copysign(1.0, theta) / (fabs(theta) + sqrt(theta * theta + 1.0));
          const double c = 1.0 / sqrt(t * t + 1.0);
          const double s = t * c;
          // A <- J^T A J
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const double akp = A[k][p], akq = A[k][q];
            A[k][p] = c * akp - s * akq;
            A[k][q] = s * akp + c * akq;
          }
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const double apk = A[p][k], aqk = A[q][k];
            A[p][k] = c * apk - s * aqk;
            A[q][k] = s * apk + c * aqk;
          }
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const double vkp = V[k][p], vkq = V[k][q];
            V[k][p] = c * vkp - s * vkq;
            V[k][q] = s * vkp + c * vkq;
          }
        }
      }
    }
  }
  int best = 0;
  double bv = A[0][0];
#pragma unroll
  for (int i = 1; i < 4; ++i)
    if (A[i][i] < bv) { bv = A[i][i]; best = i; }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    double r = V[k][0];
    if (best == 1) r = V[k][1];
    if (best == 2) r = V[k][2];
    if (best == 3) r = V[k][3];
    v_out[k] = r;
  }
}

// A += T^T T with T = P - x x^T P   (P row-major 3x4, x unit ray)
__device__ __forceinline__ void dlt_accumulate(double* a, const double* P, double x0, double x1, double x2) {
  double T[3][4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double y = x0 * P[k] + x1 * P[4 + k] + x2 * P[8 + k];
    T[0][k] = P[k] - x0 * y;
    T[1][k] = P[4 + k] - x1 * y;
    T[2][k] = P[8 + k] - x2 * y;
  }
  int idx = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = i; j < 4; ++j) a[idx++] += T[0][i] * T[0][j] + T[1][i] * T[1][j] + T[2][i] * T[2][j];
}

__device__ __forceinline__ double clamp_pm1(double x) {
  // torch.clamp propagates NaN
  return x != x ? x : fmin(fmax(x, -1.0), 1.0);
}

// angular error between the unit observation ray and R X + t (triangulation_helpers.py:431-472):
// acos(clamp(<r, p/max(|p|,1e-12)>)).  Only errors up to the inlier threshold are ever used (everything above is
// an outlier whose value is discarded), so the kernel evaluates the angle exactly where it matters and returns a
// sentinel (4.0 > pi) otherwise:
//   * one rsqrt instead of sqrt + three divides;
//   * for c within `cos_gate` of 1 and gates up to 0.1 rad:  acos(c) = 2 asin(sqrt((1-c)/2)) with the asin series
//     to x^9 (x <= 0.05: truncation < 3e-15 relative; 6e-20 at the reference's 2 degree gate); 1-c is exact for
//     c in [0.5, 1] (Sterbenz).  Wider gates fall back to acos().
// NaN inputs give a NaN cosine, fail the gate and come back as the sentinel (== "not an inlier", like NaN <= thr).
constexpr double kAngSentinel = 4.0;
__device__ __forceinline__ double ang_err(const double* P, double r0, double r1, double r2, double X0, double X1,
                                          double X2, double cos_gate) {
  const double p0 = P[0] * X0 + P[1] * X1 + P[2] * X2 + P[3];
  const double p1 = P[4] * X0 + P[5] * X1 + P[6] * X2 + P[7];
  const double p2 = P[8] * X0 + P[9] * X1 + P[10] * X2 + P[11];
  const double n2 = p0 * p0 + p1 * p1 + p2 * p2;
  const double dot = r0 * p0 + r1 * p1 + r2 * p2;
  double c = (n2 >= 1e-24) ? dot * rsqrt(n2) : dot * 1e12;       // max(|p|, 1e-12) in the denominator
  if (!(c >= cos_gate)) return kAngSentinel;
  if (cos_gate < 0.995) return acos(fmin(c, 1.0));                // wide gates (> 0.1 rad): plain acos
  const double om = fmax(1.0 - c, 0.0);                           // clamp(c, -1, 1)
  const double x2 = 0.5 * om;
  const double x = sqrt(x2);
  // asin(x) = x (1 + x^2/6 + 3x^4/40 + 5x^6/112 + 35x^8/1152)
  const double poly = fma(x2, fma(x2, fma(x2, fma(x2, 35.0 / 1152.0, 5.0 / 112.0), 3.0 / 40.0), 1.0 / 6.0), 1.0);
  return 2.0 * x * poly;
}

// triangulation angle in degrees (triangulation_helpers.py:547-587)
__device__ __forceinline__ double tri_angle_deg(const double* c1, const double* c2, double X0, double X1, double X2) {
  const double b0 = c1[0] - c2[0], b1 = c1[1] - c2[1], b2 = c1[2] - c2[2];
  const double base2 = b0 * b0 + b1 * b1 + b2 * b2;
  const double u0 = X0 - c1[0], u1 = X1 - c1[1], u2 = X2 - c1[2];
  const double w0 = X0 - c2[0], w1 = X1 - c2[1], w2 = X2 - c2[2];
  const double r1 = u0 * u0 + u1 * u1 + u2 * u2;
  const double r2 = w0 * w0 + w1 * w1 + w2 * w2;
  double den = 2.0 * sqrt(r1 * r2);
  double num = r1 + r2 - base2;
  if (den <= 1e-12) { num = 1.0; den = 1.0; }
  const double c = clamp_pm1(num / den);
  double t = fabs(acos(c));
  t = fmin(t, kPi - t);       // fmin drops NaN like torch.min? torch.min propagates NaN: handled by caller (>= false)
  if (c != c) t = c;
  return t * (180.0 / kPi);
}

struct TriParams {
  int S, N, H0, lo, lo2, W;           // W = ceil(S/32)
  double max_rad, min_tri_deg, cos_min_tri;
  double cos_gate;                    // cos(max_rad) minus a margin: below it an observation is certainly an outlier
};

// shared-memory carve-up (doubles first)
struct TriSmem {
  double* cams;      // [S][12]
  double* centers;   // [S][3]
  double* rays;      // [S][3] unit observation rays
  double* hypX;      // [HT][3]
  double* hypMean;   // [HT]
  double* Abuf;      // [lo][10]
  int* hypCnt;       // [HT]
  int* sel;          // [lo]
  uint32_t* bits;    // [HT][W]
  uint32_t* vbits;   // [W]   1 = observation usable (vis/score gate passed)
  uint8_t* hypInv;   // [HT]
  uint64_t* bar;
};

__device__ __forceinline__ TriSmem tri_carve(unsigned char* base, int S, int HT, int lo, int W) {
  TriSmem s;
  double* d = reinterpret_cast<double*>(base);
  s.cams = d; d += (size_t)S * 12;
  s.centers = d; d += (size_t)S * 3;
  s.rays = d; d += (size_t)S * 3;
  s.hypX = d; d += (size_t)HT * 3;
  s.hypMean = d; d += HT;
  s.Abuf = d; d += (size_t)lo * 10;
  s.bar = reinterpret_cast<uint64_t*>(d); d += 1;
  int* i = reinterpret_cast<int*>(d);
  s.hypCnt = i; i += HT;
  s.sel = i; i += lo;
  s.bits = reinterpret_cast<uint32_t*>(i); i += (size_t)HT * W;
  s.vbits = reinterpret_cast<uint32_t*>(i); i += W;
  s.hypInv = reinterpret_cast<uint8_t*>(i);
  return s;
}

static size_t tri_smem_bytes(int S, int HT, int lo, int W) {
  size_t b = sizeof(double) * ((size_t)S * 18 + (size_t)HT * 4 + (size_t)lo * 10 + 1);
  b += sizeof(int) * ((size_t)HT + lo + (size_t)HT * W + W);
  b += HT;
  return align_up(b, 16);
}

// score hypothesis X against all frames; one warp, lanes over frames; writes bits/cnt/mean for slot h
__device__ __forceinline__ void warp_score(const TriSmem& sm, const TriParams& p, int h, double X0, double X1,
                                           double X2, bool invalid, bool nan_to_num, int lane) {
  int cnt = 0;
  double sum = 0.0;
  for (int w = 0; w < p.W; ++w) {
    const int s = w * 32 + lane;
    bool inl = false;
    double e = 0.0;
    if (s < p.S && !invalid && ((sm.vbits[w] >> lane) & 1u)) {
      e = ang_err(sm.cams + (size_t)s * 12, sm.rays[s * 3], sm.rays[s * 3 + 1], sm.rays[s * 3 + 2], X0, X1, X2, p.cos_gate);
      inl = e <= p.max_rad;                     // (nan_to_num(100 pi) of the reference is also "not an inlier")
    }
    const uint32_t word = __ballot_sync(0xffffffffu, inl);
    if (lane == 0) sm.bits[(size_t)h * p.W + w] = word;
    cnt += __popc(word);
    sum += inl ? e : 0.0;
  }
  sum = warp_sum(sum);
  if (lane == 0) {
    sm.hypCnt[h] = cnt;
    sm.hypMean[h] = cnt > 0 ? sum / cnt : 2.0 * kPi;
  }
}

// exists a pair of cameras (a,b) with triangulation angle >= min at X ? (all S cameras) -- one warp
__device__ __forceinline__ bool warp_any_tri_pair(const TriSmem& sm, const TriParams& p, double X0, double X1,
                                                  double X2, int lane) {
  const int S = p.S;
  // visit separations d = S/2, S/2+1, ..., S-1, S/2-1, ..., 1: wide baselines first
  const int mid = S / 2 > 0 ? S / 2 : 1;
  for (int k = 0; k < S - 1; ++k) {
    const int d = (k < S - mid) ? (mid + k) : (S - 1 - k);
    bool found = false;
    for (int a = lane; a + d < S; a += 32) {
      const double c = tri_cos_abs(sm.centers + a * 3, sm.centers + (a + d) * 3, X0, X1, X2);
      if (c <= p.cos_min_tri) found = true;
    }
    if (__any_sync(0xffffffffu, found)) return true;
  }
  return false;
}

__global__ void __launch_bounds__(TRI_THREADS) tri_main_kernel(
    TriParams p, const double* __restrict__ cams_g, const double* __restrict__ centers_g,
    const double* __restrict__ tn, const uint8_t* __restrict__ usable, const int* __restrict__ pairs,
    double* __restrict__ outX, int* __restrict__ outCnt, double* __restrict__ outMean, uint8_t* __restrict__ outInv,
    unsigned long long* __restrict__ gmax_mean) {
  extern __shared__ __align__(16) unsigned char tri_smem[];
  const int HT = p.H0 + p.lo + p.lo2;
  TriSmem sm = tri_carve(tri_smem, p.S, HT, p.lo, p.W);
  const int n = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nwarps = TRI_THREADS / 32;
  const int S = p.S;

  // ---- stage cameras + centres with TMA bulk copies (chunks of <= 12 KB), rays/vis with plain loads
  if (tid == 0) {
    mbar_init(sm.bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (tid == 0) {
    const uint32_t cam_bytes = (uint32_t)S * 96u, cen_bytes = (uint32_t)S * 24u;
    const bool ok = (cen_bytes % 16u) == 0;     // S even; else centres go through plain loads below
    mbar_expect_tx(sm.bar, cam_bytes + (ok ? cen_bytes : 0u));
    for (uint32_t off = 0; off < cam_bytes; off += 12288u) {
      const uint32_t sz = min(12288u, cam_bytes - off);
      tma_load_1d(reinterpret_cast<unsigned char*>(sm.cams) + off, reinterpret_cast<const unsigned char*>(cams_g) + off, sz, sm.bar);
    }
    if (ok) {
      for (uint32_t off = 0; off < cen_bytes; off += 12288u) {
        const uint32_t sz = min(12288u, cen_bytes - off);
        tma_load_1d(reinterpret_cast<unsigned char*>(sm.centers) + off, reinterpret_cast<const unsigned char*>(centers_g) + off, sz, sm.bar);
      }
    }
  }
  if ((S * 24) % 16 != 0)
    for (int i = tid; i < S * 3; i += TRI_THREADS) sm.centers[i] = centers_g[i];
  for (int s = tid; s < S; s += TRI_THREADS) {
    const double u = tn[((size_t)s * p.N + n) * 2], v = tn[((size_t)s * p.N + n) * 2 + 1];
    const double nr = sqrt(u * u + v * v + 1.0);
    sm.rays[s * 3] = u / nr;
    sm.rays[s * 3 + 1] = v / nr;
    sm.rays[s * 3 + 2] = 1.0 / nr;
  }
  for (int w = warp; w < p.W; w += nwarps) {
    const int s = w * 32 + lane;
    const bool ok = s < S && usable[(size_t)s * p.N + n] != 0;
    const uint32_t word = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) sm.vbits[w] = word;
  }
  mbar_wait(sm.bar, 0);
  __syncthreads();

  // ---- phase 1: two-view hypotheses, thread per hypothesis
  for (int h = tid; h < p.H0; h += TRI_THREADS) {
    const int a = pairs[h * 2], b = pairs[h * 2 + 1];
    double A[10];
#pragma unroll
    for (int i = 0; i < 10; ++i) A[i] = 0.0;
    dlt_accumulate(A, sm.cams + (size_t)a * 12, sm.rays[a * 3], sm.rays[a * 3 + 1], sm.rays[a * 3 + 2]);
    dlt_accumulate(A, sm.cams + (size_t)b * 12, sm.rays[b * 3], sm.rays[b * 3 + 1], sm.rays[b * 3 + 2]);
    double v[4];
    smallest_eigvec4(A, v);
    const double X0 = v[0] / v[3], X1 = v[1] / v[3], X2 = v[2] / v[3];
    const double* Pa = sm.cams + (size_t)a * 12;
    const double* Pb = sm.cams + (size_t)b * 12;
    const double za = Pa[8] * X0 + Pa[9] * X1 + Pa[10] * X2 + Pa[11];
    const double zb = Pb[8] * X0 + Pb[9] * X1 + Pb[10] * X2 + Pb[11];
    const bool bad_che = (za <= 0.0) || (zb <= 0.0);
    const double ang = tri_angle_deg(sm.centers + a * 3, sm.centers + b * 3, X0, X1, X2);
    const bool bad_tri = !(ang >= p.min_tri_deg);
    const bool invalid = bad_che || bad_tri;
    sm.hypX[h * 3] = X0; sm.hypX[h * 3 + 1] = X1; sm.hypX[h * 3 + 2] = X2;
    sm.hypInv[h] = invalid ? 1 : 0;
    // score against every frame
    int cnt = 0;
    double sum = 0.0;
    for (int w = 0; w < p.W; ++w) {
      uint32_t word = 0;
      if (!invalid) {
        const uint32_t vb = sm.vbits[w];
        const int send = min(32, S - w * 32);
        for (int j = 0; j < send; ++j) {
          if ((vb >> j) & 1u) {
            const int s = w * 32 + j;
            const double e = ang_err(sm.cams + (size_t)s * 12, sm.rays[s * 3], sm.rays[s * 3 + 1], sm.rays[s * 3 + 2], X0, X1, X2, p.cos_gate);
            if (e <= p.max_rad) { word |= (1u << j); sum += e; ++cnt; }
          }
        }
      }
      sm.bits[(size_t)h * p.W + w] = word;
    }
    sm.hypCnt[h] = cnt;
    sm.hypMean[h] = cnt > 0 ? sum / cnt : 2.0 * kPi;
  }
  __syncthreads();

  // ---- two rounds of local refinement
  int src_base = 0, src_num = p.H0, dst_base = p.H0, num = p.lo;
  for (int round = 0; round < 2; ++round) {
    // rank source hypotheses by inlier count (stable, descending) and keep the top `num`
    for (int h = tid; h < src_num; h += TRI_THREADS) {
      const int c = sm.hypCnt[src_base + h];
      int rank = 0;
      for (int g = 0; g < src_num; ++g) {
        const int cg = sm.hypCnt[src_base + g];
        rank += (cg > c) || (cg == c && g < h);
      }
      if (rank < num) sm.sel[rank] = src_base + h;
    }
    __syncthreads();
    // masked multi-view DLT normal matrices: warp per hypothesis, lanes over frames
    for (int j = warp; j < num; j += nwarps) {
      const uint32_t* bw = sm.bits + (size_t)sm.sel[j] * p.W;
      double A[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) A[i] = 0.0;
      for (int w = 0; w < p.W; ++w) {
        const int s = w * 32 + lane;
        if (s < S && ((bw[w] >> lane) & 1u))
          dlt_accumulate(A, sm.cams + (size_t)s * 12, sm.rays[s * 3], sm.rays[s * 3 + 1], sm.rays[s * 3 + 2]);
      }
      const double r = warp_reduce_scatter<16>(A, lane);
      if (lane < 10) sm.Abuf[j * 10 + lane] = r;
    }
    __syncthreads();
    // eigen-solves: thread per hypothesis
    for (int j = tid; j < num; j += TRI_THREADS) {
      double v[4];
      smallest_eigvec4(sm.Abuf + j * 10, v);
      const int h = dst_base + j;
      sm.hypX[h * 3] = v[0] / v[3];
      sm.hypX[h * 3 + 1] = v[1] / v[3];
      sm.hypX[h * 3 + 2] = v[2] / v[3];
    }
    __syncthreads();
    // cheirality over ALL cameras, triangulation-angle existence over ALL camera pairs, re-score
    for (int j = warp; j < num; j += nwarps) {
      const int h = dst_base + j;
      const double X0 = sm.hypX[h * 3], X1 = sm.hypX[h * 3 + 1], X2 = sm.hypX[h * 3 + 2];
      bool bad = false;
      for (int s = lane; s < S; s += 32) {
        const double* P = sm.cams + (size_t)s * 12;
        const double z = P[8] * X0 + P[9] * X1 + P[10] * X2 + P[11];
        bad = bad || (z <= 0.0);
      }
      bool invalid = __any_sync(0xffffffffu, bad);
      if (!invalid) invalid = !warp_any_tri_pair(sm, p, X0, X1, X2, lane);
      if (lane == 0) sm.hypInv[h] = invalid ? 1 : 0;
      warp_score(sm, p, h, X0, X1, X2, invalid, true, lane);
    }
    __syncthreads();
    src_base = dst_base; src_num = num; dst_base += num; num = p.lo2;
  }

  // ---- write hypothesis summaries; the global threshold of calculate_residual_indicator needs a grid-wide max
  double mx = 0.0;
  for (int h = tid; h < HT; h += TRI_THREADS) {
    const size_t o = (size_t)n * HT + h;
    outX[o * 3] = sm.hypX[h * 3];
    outX[o * 3 + 1] = sm.hypX[h * 3 + 1];
    outX[o * 3 + 2] = sm.hypX[h * 3 + 2];
    outCnt[o] = sm.hypCnt[h];
    outMean[o] = sm.hypMean[h];
    outInv[o] = sm.hypInv[h];
    mx = fmax(mx, sm.hypMean[h]);
  }
  mx = warp_max(mx);
  if (lane == 0) atomicMax(gmax_mean, (unsigned long long)__double_as_longlong(mx));
}

// final selection: best = argmax_h cnt + (thres - mean)/thres; recompute the winner's inlier mask.
// One warp per track; cameras read through L1/L2 (S*96 B shared by all warps).
__global__ void __launch_bounds__(256) tri_select_kernel(TriParams p, const double* __restrict__ cams_g,
                                                         const double* __restrict__ tn,
                                                         const uint8_t* __restrict__ usable,
                                                         const double* __restrict__ hypX, const int* __restrict__ hypCnt,
                                                         const double* __restrict__ hypMean,
                                                         const uint8_t* __restrict__ hypInv,
                                                         const unsigned long long* __restrict__ gmax_mean,
                                                         double* __restrict__ points, long long* __restrict__ inl_num,
                                                         uint8_t* __restrict__ inl_mask) {
  const int HT = p.H0 + p.lo + p.lo2;
  const int lane = threadIdx.x & 31;
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= p.N) return;
  const double thres = __longlong_as_double((long long)*gmax_mean) + 1e-6;
  double best = -1.0;
  int bi = 0x7fffffff;
  for (int h = lane; h < HT; h += 32) {
    const size_t o = (size_t)n * HT + h;
    const double sc = (thres - hypMean[o]) / thres + (double)hypCnt[o];
    if (sc > best) { best = sc; bi = h; }
  }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const double ob = __shfl_xor_sync(0xffffffffu, best, off);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
    if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  const size_t o = (size_t)n * HT + bi;
  const double X0 = hypX[o * 3], X1 = hypX[o * 3 + 1], X2 = hypX[o * 3 + 2];
  const bool invalid = hypInv[o] != 0;
  const bool refined = bi >= p.H0;
  if (lane == 0) {
    points[(size_t)n * 3] = X0;
    points[(size_t)n * 3 + 1] = X1;
    points[(size_t)n * 3 + 2] = X2;
    inl_num[n] = hypCnt[o];
  }
  for (int s = lane; s < p.S; s += 32) {
    bool inl = false;
    if (!invalid && usable[(size_t)s * p.N + n] != 0) {
      const double u = tn[((size_t)s * p.N + n) * 2], v = tn[((size_t)s * p.N + n) * 2 + 1];
      const double nr = sqrt(u * u + v * v + 1.0);
      const double e = ang_err(cams_g + (size_t)s * 12, u / nr, v / nr, 1.0 / nr, X0, X1, X2, p.cos_gate);
      inl = e <= p.max_rad;
    }
    inl_mask[(size_t)n * p.S + s] = inl ? 1 : 0;
  }
}

__global__ void proj_centers_kernel(int S, const double* __restrict__ cams, double* __restrict__ centers) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S) return;
  const double* P = cams + (size_t)s * 12;
  centers[s * 3 + 0] = -(P[0] * P[3] + P[4] * P[7] + P[8] * P[11]);
  centers[s * 3 + 1] = -(P[1] * P[3] + P[5] * P[7] + P[9] * P[11]);
  centers[s * 3 + 2] = -(P[2] * P[3] + P[6] * P[7] + P[10] * P[11]);
}

// usable[s][n] = !(vis <= 0.05 || score <= 0.5)   (triangulation.py:867-872)
__global__ void usable_kernel(size_t total, const float* __restrict__ vis, const float* __restrict__ score,
                              uint8_t* __restrict__ usable) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  bool bad = vis[i] <= 0.05f;
  if (score) bad = bad || (score[i] <= 0.5f);
  usable[i] = bad ? 0 : 1;
}

// triangulate_by_pair (triangulation.py:45-135): pairs (0, s+1), thread per (pair, track)
__global__ void tri_by_pair_kernel(int S, int N, const double* __restrict__ cams, const double* __restrict__ centers,
                                   const double* __restrict__ tn, double* __restrict__ points,
                                   uint8_t* __restrict__ cheirality, double* __restrict__ angle) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)(S - 1) * N) return;
  const int s = (int)(i / N) + 1, n = (int)(i % N);
  double A[10];
#pragma unroll
  for (int k = 0; k < 10; ++k) A[k] = 0.0;
  {
    const double u = tn[(size_t)n * 2], v = tn[(size_t)n * 2 + 1];
    const double nr = sqrt(u * u + v * v + 1.0);
    dlt_accumulate(A, cams, u / nr, v / nr, 1.0 / nr);
  }
  {
    const double u = tn[((size_t)s * N + n) * 2], v = tn[((size_t)s * N + n) * 2 + 1];
    const double nr = sqrt(u * u + v * v + 1.0);
    dlt_accumulate(A, cams + (size_t)s * 12, u / nr, v / nr, 1.0 / nr);
  }
  double v4[4];
  smallest_eigvec4(A, v4);
  const double X0 = v4[0] / v4[3], X1 = v4[1] / v4[3], X2 = v4[2] / v4[3];
  const double* Pb = cams + (size_t)s * 12;
  const double za = cams[8] * X0 + cams[9] * X1 + cams[10] * X2 + cams[11];
  const double zb = Pb[8] * X0 + Pb[9] * X1 + Pb[10] * X2 + Pb[11];
  points[i * 3] = X0; points[i * 3 + 1] = X1; points[i * 3 + 2] = X2;
  cheirality[i] = ((za <= 0.0) || (zb <= 0.0)) ? 0 : 1;
  angle[i] = tri_angle_deg(centers, centers + s * 3, X0, X1, X2);
}

// ------------------------------------------------------------------------------------------------
// filter_all_points3D_single_chunk: warp per point
// ------------------------------------------------------------------------------------------------
template <typename TUV>
__global__ void __launch_bounds__(256) filter_points_kernel(
    int S, int P, const double* __restrict__ X, const TUV* __restrict__ uv, const double* __restrict__ cams,
    const double* __restrict__ centers, const double* __restrict__ K /*[S,9]*/, const double* __restrict__ extra,
    double max_err2, double cos_min_tri, int check_triangle, double hard_max, uint8_t* __restrict__ valid,
    uint8_t* __restrict__ detail /*[S,P] or null*/) {
  extern __shared__ uint32_t fbits[];           // [warps][W]
  const int W = (S + 31) / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int pidx = blockIdx.x * (blockDim.x >> 5) + warp;
  if (pidx >= P) return;
  uint32_t* bits = fbits + (size_t)warp * W;
  const double X0 = X[(size_t)pidx * 3], X1 = X[(size_t)pidx * 3 + 1], X2 = X[(size_t)pidx * 3 + 2];
  int cnt = 0;
  for (int w = 0; w < W; ++w) {
    const int s = w * 32 + lane;
    bool inl = false;
    if (s < S)
      inl = filter_err2(cams, K, extra, s, X0, X1, X2, uv[((size_t)s * P + pidx) * 2],
                        uv[((size_t)s * P + pidx) * 2 + 1]) <= max_err2;
    const uint32_t word = __ballot_sync(0xffffffffu, inl);
    if (lane == 0) bits[w] = word;
    cnt += __popc(word);
  }
  __syncwarp();
  bool ok = cnt >= 2;
  if (hard_max > 0.0) ok = ok && (fabs(X0) <= hard_max) && (fabs(X1) <= hard_max) && (fabs(X2) <= hard_max);
  bool tri_ok = true;
  if (check_triangle) {
    tri_ok = false;
    if (ok) {
      // exists inlier pair (a,b) with angle >= min: separations wide-first, early exit
      const int mid = S / 2 > 0 ? S / 2 : 1;
      for (int k = 0; k < S - 1 && !tri_ok; ++k) {
        const int d = (k < S - mid) ? (mid + k) : (S - 1 - k);
        bool found = false;
        for (int a = lane; a + d < S; a += 32) {
          const int b = a + d;
          if (((bits[a >> 5] >> (a & 31)) & 1u) && ((bits[b >> 5] >> (b & 31)) & 1u)) {
            const double c = tri_cos_abs(centers + a * 3, centers + b * 3, X0, X1, X2);
            if (c <= cos_min_tri) found = true;
          }
        }
        tri_ok = __any_sync(0xffffffffu, found);
      }
    }
  }
  if (lane == 0) valid[pidx] = (ok && tri_ok) ? 1 : 0;
  if (detail) {
    for (int s = lane; s < S; s += 32) {
      bool d = (bits[s >> 5] >> (s & 31)) & 1u;
      if (check_triangle) d = d && tri_ok;
      detail[(size_t)s * P + pidx] = d ? 1 : 0;
    }
  }
}

// The point filter on an observation list (vgg_filter_observations), warp per point over its track segment
// [track_start[n], track_start[n+1]): keep[m] = the observation reprojects within the bound at positive depth
// (filter_err2, the grid filter's arithmetic); valid[n] = at least two kept observations and one kept pair whose
// triangulation angle is at least the minimum (COLMAP's ObservationManager::FilterAllPoints3D, which considers the
// track's elements only; the grid filter also counts an unobserved cell that happens to reproject within the bound)
__global__ void __launch_bounds__(256) filter_obs_list_kernel(
    int S, int N, const float* __restrict__ uv, const int* __restrict__ frame, const int* __restrict__ track_start,
    const double* __restrict__ X, const double* __restrict__ cams, const double* __restrict__ centers,
    const double* __restrict__ K, const double* __restrict__ extra, double max_err2, double cos_min_tri,
    uint8_t* __restrict__ keep, uint8_t* __restrict__ valid) {
  const int lane = threadIdx.x & 31, n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= N) return;
  const double X0 = X[(size_t)n * 3], X1 = X[(size_t)n * 3 + 1], X2 = X[(size_t)n * 3 + 2];
  const int m0 = track_start[n], m1 = track_start[n + 1];
  int cnt = 0;
  for (int b = m0; b < m1; b += 32) {
    const int m = b + lane;
    const int s = m < m1 ? frame[m] : -1;
    const bool inl = s >= 0 && s < S &&
                     filter_err2(cams, K, extra, s, X0, X1, X2, uv[(size_t)m * 2], uv[(size_t)m * 2 + 1]) <= max_err2;
    if (m < m1) keep[m] = inl ? 1 : 0;
    cnt += __popc(__ballot_sync(0xffffffffu, inl));
  }
  __syncwarp();
  bool tri_ok = false;
  if (cnt >= 2)
    for (int a = m0; a < m1 && !tri_ok; ++a) {
      if (!keep[a]) continue;
      const double* ca = centers + (size_t)frame[a] * 3;
      bool found = false;
      for (int b = a + 1 + lane; b < m1; b += 32)
        if (keep[b] && tri_cos_abs(ca, centers + (size_t)frame[b] * 3, X0, X1, X2) <= cos_min_tri) found = true;
      tri_ok = __any_sync(0xffffffffu, found);
    }
  if (lane == 0) valid[n] = (cnt >= 2 && tri_ok) ? 1 : 0;
}

// project_3D_points (triangulation_helpers.py:311-395): out[S,P,2], cam[S,3,P]
__global__ void project_points_kernel(int S, int P, const double* __restrict__ X, const double* __restrict__ cams,
                                      const double* __restrict__ K /*[S,9]*/, const double* __restrict__ extra,
                                      double* __restrict__ out2d, double* __restrict__ outcam) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)S * P) return;
  const int s = (int)(i / P), pidx = (int)(i % P);
  const double* Pm = cams + (size_t)s * 12;
  const double X0 = X[(size_t)pidx * 3], X1 = X[(size_t)pidx * 3 + 1], X2 = X[(size_t)pidx * 3 + 2];
  const double p0 = Pm[0] * X0 + Pm[1] * X1 + Pm[2] * X2 + Pm[3];
  const double p1 = Pm[4] * X0 + Pm[5] * X1 + Pm[6] * X2 + Pm[7];
  const double p2 = Pm[8] * X0 + Pm[9] * X1 + Pm[10] * X2 + Pm[11];
  if (outcam) {
    outcam[((size_t)s * 3 + 0) * P + pidx] = p0;
    outcam[((size_t)s * 3 + 1) * P + pidx] = p1;
    outcam[((size_t)s * 3 + 2) * P + pidx] = p2;
  }
  if (!out2d) return;
  double u = p0 / p2, v = p1 / p2;
  if (extra) {
    const double k = extra[s];
    const double rad = k * (u * u + v * v);
    const double du = u * rad, dv = v * rad;
    u = u + du; v = v + dv;
  }
  const double* Km = K + (size_t)s * 9;
  double x = Km[0] * u + Km[1] * v + Km[2];
  double y = Km[3] * u + Km[4] * v + Km[5];
  if (x != x) x = 0.0;
  if (y != y) y = 0.0;
  x = fmin(fmax(x, -1.7976931348623157e308), 1.7976931348623157e308);
  y = fmin(fmax(y, -1.7976931348623157e308), 1.7976931348623157e308);
  out2d[i * 2] = x;
  out2d[i * 2 + 1] = y;
}

// cam_from_img without distortion: (uv - pp) / f in the input precision
template <typename T>
__global__ void normalize_tracks_kernel(int S, int N, const T* __restrict__ uv, const T* __restrict__ f2,
                                        const T* __restrict__ pp2, T* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)S * N * 2) return;
  const int s = (int)(i / ((size_t)N * 2)), c = (int)(i & 1);
  out[i] = (uv[i] - pp2[s * 2 + c]) / f2[s * 2 + c];
}

// iterative_undistortion (distortion.py:27-99), SIMPLE_RADIAL.  pass 0: find the global stop iteration
// (bit t of notconv set when some observation's step at iteration t is >= max_step_norm); pass 1: run
// exactly `iters` iterations.
__device__ __forceinline__ void distort1(double k, double u, double v, double& ou, double& ov) {
  const double r2 = u * u + v * v;
  const double radial = k * r2;
  const double du = u * radial, dv = v * radial;
  ou = u + du; ov = v + dv;
}
__global__ void undistort_kernel(int S, int N, const double* __restrict__ tn_in, const double* __restrict__ extra,
                                 int max_iters, double max_step_norm, double rel_step, int pass,
                                 unsigned long long* __restrict__ notconv /*[2]*/, int iters,
                                 double* __restrict__ tn_out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long nc0 = 0, nc1 = 0;
  if (i < (size_t)S * N) {
    const int s = (int)(i / N);
    const double k = extra[s];
    const double ou = tn_in[i * 2], ov = tn_in[i * 2 + 1];
    double u = ou, v = ov;
    const double eps = 2.220446049250313e-16;
    const int T = pass == 0 ? max_iters : iters;
    for (int t = 0; t < T; ++t) {
      double ud, vd;
      distort1(k, u, v, ud, vd);
      const double dx = ou - ud, dy = ov - vd;
      const double su = fmax(fabs(u) * rel_step, eps), sv = fmax(fabs(v) * rel_step, eps);
      double a0, a1, b0, b1, c0, c1, d0, d1;
      distort1(k, u + su, v, a0, a1);
      distort1(k, u - su, v, b0, b1);
      distort1(k, u, v + sv, c0, c1);
      distort1(k, u, v - sv, d0, d1);
      const double J00 = (a0 - b0) / (2 * su) + 1, J01 = (c0 - d0) / (2 * sv);
      const double J10 = (a1 - b1) / (2 * su), J11 = (c1 - d1) / (2 * sv) + 1;
      // 2x2 LU with partial pivoting like torch.linalg.solve
      double e0, e1;
      if (fabs(J00) >= fabs(J10)) {
        const double l = J10 / J00;
        const double u11 = J11 - l * J01;
        e1 = (dy - l * dx) / u11;
        e0 = (dx - J01 * e1) / J00;
      } else {
        const double l = J00 / J10;
        const double u11 = J01 - l * J11;
        e1 = (dx - l * dy) / u11;
        e0 = (dy - J11 * e1) / J10;
      }
      u += e0; v += e1;
      if (pass == 0) {
        const double st = e0 * e0 + e1 * e1;
        if (!(st < max_step_norm)) {
          if (t < 64) nc0 |= (1ull << t);
          else nc1 |= (1ull << (t - 64));
        }
        if (st < 1e-30) break;        // at the rounding floor; later steps stay below the threshold
      }
    }
    if (pass == 1) { tn_out[i * 2] = u; tn_out[i * 2 + 1] = v; }
  }
  if (pass == 0) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
      nc0 |= __shfl_xor_sync(0xffffffffu, nc0, off);
      nc1 |= __shfl_xor_sync(0xffffffffu, nc1, off);
    }
    if ((threadIdx.x & 31) == 0) {
      if (nc0) atomicOr(&notconv[0], nc0);
      if (nc1) atomicOr(&notconv[1], nc1);
    }
  }
}

}  // namespace vgg

using namespace vgg;

extern "C" {

int vgg_tri_workspace_bytes(int S, int N, int H0, int lo_num, size_t* bytes) {
  VGG_REQUIRE(S >= 2 && N > 0 && H0 > 0 && bytes, "bad sizes");
  const int lo = H0 >= lo_num ? lo_num : H0;
  const int lo2 = lo > 10 ? 10 : lo;
  const size_t HT = (size_t)H0 + lo + lo2;
  Carver c(nullptr, 0);
  c.take<double>((size_t)S * 3);          // centers
  c.take<uint8_t>((size_t)S * N);         // usable
  c.take<double>((size_t)N * HT * 3);     // hypX
  c.take<int>((size_t)N * HT);            // hypCnt
  c.take<double>((size_t)N * HT);         // hypMean
  c.take<uint8_t>((size_t)N * HT);        // hypInv
  c.take<unsigned long long>(4);
  *bytes = align_up(c.off, 256);
  return VGG_OK;
}

int vgg_triangulate_tracks(int S, int N, const double* extrinsics, const double* tracks_normalized,
                           const float* track_vis, const float* track_score, const int32_t* pairs, int H0,
                           int lo_num, double max_angular_error_deg, double min_tri_angle_deg, double* out_points,
                           int64_t* out_inlier_num, uint8_t* out_inlier_mask, void* workspace, size_t ws_bytes,
                           void* stream) {
  VGG_REQUIRE(extrinsics && tracks_normalized && track_vis && pairs && out_points && out_inlier_num && out_inlier_mask && workspace,
              "null pointer");
  VGG_REQUIRE(S >= 2 && N > 0 && H0 > 0, "bad sizes");
  cudaStream_t st = (cudaStream_t)stream;
  g_launch_count = 0;
  TriParams p;
  p.S = S; p.N = N; p.H0 = H0;
  p.lo = H0 >= lo_num ? lo_num : H0;
  p.lo2 = p.lo > 10 ? 10 : p.lo;
  p.W = (S + 31) / 32;
  p.max_rad = max_angular_error_deg * (kPi / 180.0);
  p.min_tri_deg = min_tri_angle_deg;
  p.cos_min_tri = cos(min_tri_angle_deg * (kPi / 180.0));
  p.cos_gate = cos(fmin(p.max_rad, 3.0)) - 1e-9;     // the series path is taken for gates <= 0.1 rad (cos >= 0.995)
  const size_t HT = (size_t)H0 + p.lo + p.lo2;
  size_t need = 0;
  vgg_tri_workspace_bytes(S, N, H0, lo_num, &need);
  if (ws_bytes < need) {
    set_error("triangulation workspace too small: need %zu, have %zu", need, ws_bytes);
    return VGG_EWORKSPACE;
  }
  Carver c(workspace, ws_bytes);
  double* centers = c.take<double>((size_t)S * 3);
  uint8_t* usable = c.take<uint8_t>((size_t)S * N);
  double* hypX = c.take<double>((size_t)N * HT * 3);
  int* hypCnt = c.take<int>((size_t)N * HT);
  double* hypMean = c.take<double>((size_t)N * HT);
  uint8_t* hypInv = c.take<uint8_t>((size_t)N * HT);
  unsigned long long* gmax = c.take<unsigned long long>(4);
  const size_t smem = tri_smem_bytes(S, (int)HT, p.lo, p.W);
  if (smem > 227 * 1024) {
    set_error("triangulate_tracks: S=%d frames need %zu B of shared memory (> 227 KB)", S, smem);
    return VGG_EINVAL;
  }
  VGG_CUDA_CHECK(cudaMemsetAsync(gmax, 0, 32, st));
  proj_centers_kernel<<<(S + 127) / 128, 128, 0, st>>>(S, extrinsics, centers);
  VGG_LAUNCH_CHECK();
  const size_t total = (size_t)S * N;
  usable_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(total, track_vis, track_score, usable);
  VGG_LAUNCH_CHECK();
  VGG_CUDA_CHECK(cudaFuncSetAttribute(tri_main_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  tri_main_kernel<<<N, TRI_THREADS, smem, st>>>(p, extrinsics, centers, tracks_normalized, usable, pairs, hypX, hypCnt,
                                                hypMean, hypInv, gmax);
  VGG_LAUNCH_CHECK();
  tri_select_kernel<<<(N + 7) / 8, 256, 0, st>>>(p, extrinsics, tracks_normalized, usable, hypX, hypCnt, hypMean, hypInv,
                                                 gmax, out_points, (long long*)out_inlier_num, out_inlier_mask);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

int vgg_triangulate_by_pair(int S, int N, const double* extrinsics, const double* tracks_normalized,
                            double* out_points, uint8_t* out_cheirality, double* out_angle_deg, void* workspace,
                            size_t ws_bytes, void* stream) {
  VGG_REQUIRE(extrinsics && tracks_normalized && out_points && out_cheirality && out_angle_deg && workspace, "null pointer");
  VGG_REQUIRE(S >= 2 && N > 0 && ws_bytes >= (size_t)S * 24, "bad sizes");
  cudaStream_t st = (cudaStream_t)stream;
  g_launch_count = 0;
  double* centers = reinterpret_cast<double*>(workspace);
  proj_centers_kernel<<<(S + 127) / 128, 128, 0, st>>>(S, extrinsics, centers);
  VGG_LAUNCH_CHECK();
  const size_t total = (size_t)(S - 1) * N;
  tri_by_pair_kernel<<<(unsigned)((total + 127) / 128), 128, 0, st>>>(S, N, extrinsics, centers, tracks_normalized,
                                                                      out_points, out_cheirality, out_angle_deg);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

int vgg_filter_points3d(int S, int P, const double* points3d, const void* points2d, int points2d_is_f64,
                        const double* extrinsics, const double* intrinsics9, const double* extra_params, double max_reproj_error,
                        double min_tri_angle_deg, int check_triangle, double hard_max, uint8_t* out_valid,
                        uint8_t* out_detail, void* workspace, size_t ws_bytes, void* stream) {
  VGG_REQUIRE(points3d && points2d && extrinsics && intrinsics9 && out_valid && workspace, "null pointer");
  VGG_REQUIRE(S >= 1 && P > 0 && ws_bytes >= (size_t)S * 24, "bad sizes");
  cudaStream_t st = (cudaStream_t)stream;
  g_launch_count = 0;
  double* centers = reinterpret_cast<double*>(workspace);
  proj_centers_kernel<<<(S + 127) / 128, 128, 0, st>>>(S, extrinsics, centers);
  VGG_LAUNCH_CHECK();
  const int W = (S + 31) / 32;
  const size_t smem = sizeof(uint32_t) * 8 * W;
  const double cosmin = cos(min_tri_angle_deg * (kPi / 180.0));
  const double e2 = max_reproj_error * max_reproj_error;
  if (points2d_is_f64)
    filter_points_kernel<double><<<(P + 7) / 8, 256, smem, st>>>(S, P, points3d, (const double*)points2d, extrinsics, centers,
                                                                 intrinsics9, extra_params, e2, cosmin, check_triangle, hard_max,
                                                                 out_valid, out_detail);
  else
    filter_points_kernel<float><<<(P + 7) / 8, 256, smem, st>>>(S, P, points3d, (const float*)points2d, extrinsics, centers,
                                                                intrinsics9, extra_params, e2, cosmin, check_triangle, hard_max,
                                                                out_valid, out_detail);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

int vgg_filter_observations(int S, int N, const vgg_ba_obs_list* obs, const double* points3d, const double* extrinsics,
                            const double* intrinsics9, const double* extra_params, double max_reproj_error,
                            double min_tri_angle_deg, uint8_t* out_keep, uint8_t* out_valid, void* workspace,
                            size_t ws_bytes, void* stream) {
  VGG_REQUIRE(obs && points3d && extrinsics && intrinsics9 && out_keep && out_valid && workspace && obs->track_start,
              "null pointer");
  VGG_REQUIRE(S >= 1 && N >= 0 && ws_bytes >= (size_t)S * 24, "bad sizes");
  VGG_REQUIRE(obs->M >= 0 && obs->M < ((int64_t)1 << 30) && (obs->M == 0 || (obs->uv && obs->frame)),
              "observation list: need 0 <= M < 2^30 and its uv and frame arrays");
  cudaStream_t st = (cudaStream_t)stream;
  g_launch_count = 0;
  if (N == 0) return VGG_OK;
  double* centers = reinterpret_cast<double*>(workspace);
  proj_centers_kernel<<<(S + 127) / 128, 128, 0, st>>>(S, extrinsics, centers);
  VGG_LAUNCH_CHECK();
  filter_obs_list_kernel<<<(N + 7) / 8, 256, 0, st>>>(S, N, obs->uv, obs->frame, obs->track_start, points3d, extrinsics,
                                                      centers, intrinsics9, extra_params,
                                                      max_reproj_error * max_reproj_error,
                                                      cos(min_tri_angle_deg * (kPi / 180.0)), out_keep, out_valid);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

int vgg_project_points(int S, int P, const double* points3d, const double* extrinsics, const double* intrinsics9,
                       const double* extra_params, double* out_points2d, double* out_points_cam, void* stream) {
  VGG_REQUIRE(points3d && extrinsics && (out_points2d || out_points_cam), "null pointer");
  VGG_REQUIRE(!out_points2d || intrinsics9, "intrinsics needed for 2D output");
  cudaStream_t st = (cudaStream_t)stream;
  g_launch_count = 0;
  const size_t total = (size_t)S * P;
  project_points_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(S, P, points3d, extrinsics, intrinsics9, extra_params,
                                                                         out_points2d, out_points_cam);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

int vgg_normalize_tracks(int S, int N, const void* tracks, const void* focal2, const void* pp2, int is_f64, void* out,
                         void* stream) {
  VGG_REQUIRE(tracks && focal2 && pp2 && out, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  g_launch_count = 0;
  const size_t total = (size_t)S * N * 2;
  if (is_f64)
    normalize_tracks_kernel<double><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(S, N, (const double*)tracks, (const double*)focal2,
                                                                                      (const double*)pp2, (double*)out);
  else
    normalize_tracks_kernel<float><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(S, N, (const float*)tracks, (const float*)focal2,
                                                                                    (const float*)pp2, (float*)out);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

int vgg_undistort_simple_radial(int S, int N, const double* tracks_normalized, const double* extra_params,
                                int max_iterations, double max_step_norm, double rel_step_size, double* out,
                                int* iterations_run, void* workspace, size_t ws_bytes, void* stream) {
  VGG_REQUIRE(tracks_normalized && extra_params && out && workspace && ws_bytes >= 16, "null pointer");
  VGG_REQUIRE(max_iterations >= 1 && max_iterations <= 128, "max_iterations must be in [1,128]");
  cudaStream_t st = (cudaStream_t)stream;
  g_launch_count = 0;
  unsigned long long* notconv = reinterpret_cast<unsigned long long*>(workspace);
  VGG_CUDA_CHECK(cudaMemsetAsync(notconv, 0, 16, st));
  const size_t total = (size_t)S * N;
  const unsigned grid = (unsigned)((total + 127) / 128);
  undistort_kernel<<<grid, 128, 0, st>>>(S, N, tracks_normalized, extra_params, max_iterations, max_step_norm, rel_step_size, 0,
                                         notconv, 0, out);
  VGG_LAUNCH_CHECK();
  unsigned long long h[2];
  VGG_CUDA_CHECK(cudaMemcpyAsync(h, notconv, 16, cudaMemcpyDeviceToHost, st));
  VGG_CUDA_CHECK(cudaStreamSynchronize(st));
  int iters = max_iterations;
  for (int t = 0; t < max_iterations; ++t) {
    const bool nc = t < 64 ? ((h[0] >> t) & 1ull) : ((h[1] >> (t - 64)) & 1ull);
    if (!nc) { iters = t + 1; break; }
  }
  undistort_kernel<<<grid, 128, 0, st>>>(S, N, tracks_normalized, extra_params, max_iterations, max_step_norm, rel_step_size, 1,
                                         notconv, iters, out);
  VGG_LAUNCH_CHECK();
  if (iterations_run) *iterations_run = iters;
  return VGG_OK;
}

}  // extern "C"
