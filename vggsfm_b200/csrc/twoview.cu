// Batched two-view stage: 7-point / 8-point fundamental-matrix LO-RANSAC and the relative pose of every
// (frame 0, frame s) pair -- estimate_fundamental (vggsfm/two_view_geo/fundamental.py:43-183) and the decomposition /
// cheirality part of estimate_preliminary_cameras (estimate_preliminary.py:148-164, essential.py:36-83,
// utils.py:325-448).  The arithmetic is the one restated in oracle/twoview_oracle.py, float64 throughout.
//
// Launch sequence of vgg_estimate_fundamental (no host synchronisation in between):
//   tv_minimal_kernel   one thread per (pair, trial): 7-point solve, up to 3 candidates in registers; the CTA streams
//                       its pair's points through shared memory and keeps per candidate the inlier count, the sum of
//                       inlier residuals and whether any residual is NaN / inf.  Only those per-candidate numbers reach
//                       HBM; the candidate matrices are recomputed from the trial index where they are needed again.
//   tv_topk_kernel      one warp per pair: stable descending order of the counts (candidate index breaks ties), first
//                       lo_num kept -- a counting sort over the N+1 possible counts, histogram in the workspace.
//   tv_lo_kernel        one CTA per (pair, seed): the seed's inlier set, masked normalisation, the 9x9 normal matrix
//                       by block reductions, Jacobi -> smallest eigenvector, rank-2 projection, denormalisation; then
//                       the refined matrix is scored.  Run twice (second round from the top lo_num/2 of the first).
//   tv_select_kernel    one CTA per pair: residual indicator with the batch-wide `thres` (maximum of every candidate's
//                       mean inlier residual, NaN/inf -> 1e6, gathered by atomicMax in the scoring kernels), first
//                       argmax, then the winner's matrix, inlier mask and residuals.
#include <float.h>
#include <math.h>
#include "common.cuh"
#include "dev_probes.h"
#include "twoview_geom.h"

namespace vgg {

namespace {

constexpr int TV_TRIALS = 128;     // trials (threads) per CTA of the minimal kernel
constexpr int TV_TILE = 256;       // points per shared-memory tile of the minimal kernel
// one warp per (pair, seed): the 9x9 Jacobi runs on one lane, and with 32-thread CTAs 16 of them share an SM, so the
// solves of other seeds hide its latency (at 256 threads only 2 CTAs fit and the LO phase took 3x the scoring)
constexpr int TV_LO_THREADS = 32;
constexpr int TV_MAX_N = 190000;   // the LO kernel keeps a seed's inlier mask (N bytes) in dynamic shared memory
constexpr double TV_INVALID = 1e6;
constexpr float TV_MIN_DEPTH = 1.1920928955078125e-07f;        // torch.finfo(torch.float32).eps


// Sampson numerator and denominator with explicit roundings, so that every kernel gets the same bits for the same F
__device__ __forceinline__ void sampson_parts(const double* F, double x1, double y1, double x2, double y2, double& num,
                                              double& den) {
  const double l0 = __fma_rn(F[0], x1, __fma_rn(F[1], y1, F[2]));
  const double l1 = __fma_rn(F[3], x1, __fma_rn(F[4], y1, F[5]));
  const double l2 = __fma_rn(F[6], x1, __fma_rn(F[7], y1, F[8]));
  const double m0 = __fma_rn(F[0], x2, __fma_rn(F[3], y2, F[6]));
  const double m1 = __fma_rn(F[1], x2, __fma_rn(F[4], y2, F[7]));
  const double e = __fma_rn(x2, l0, __fma_rn(y2, l1, l2));
  num = __dmul_rn(e, e);
  den = __fma_rn(l0, l0, __fma_rn(l1, l1, __fma_rn(m0, m0, __dmul_rn(m1, m1))));
}

__device__ __forceinline__ double sampson_full(const double* F, double x1, double y1, double x2, double y2, int squared) {
  double num, den;
  sampson_parts(F, x1, y1, x2, y2, num, den);
  const double r = __ddiv_rn(num, den);
  return squared ? r : __dsqrt_rn(__dadd_rn(r, 1e-8));
}


// eigenvector of the smallest eigenvalue (the last such index on ties, like LAPACK's V[:, -1] of a zero matrix)
// (A and the n x n scratch V may live in shared memory: the 9 x 9 case of the LO kernel keeps them there)
template <int n>
__device__ void smallest_eigvec(double* A, double* V, double* v) {
  double w[n];
  jacobi_eig<n>(A, V, w);
  int k = 0;
#pragma unroll
  for (int i = 1; i < n; ++i)
    if (w[i] <= w[k]) k = i;
#pragma unroll
  for (int i = 0; i < n; ++i) v[i] = V[i * n + k];
}


template <typename TP>
__device__ void candidate_7pt(const TP* p1, const TP* p2, const int* samples, int trial, double* F3) {
  double2 a[7], b[7];
  for (int i = 0; i < 7; ++i) {
    const int id = samples[trial * 7 + i];
    a[i] = ldp(p1, id);
    b[i] = ldp(p2, id);
  }
  seven_point(a, b, F3);
}

__device__ __forceinline__ double indicator_mean(int cnt, double sum, bool bad) {
  if (bad || cnt == 0) return TV_INVALID;
  const double m = sum / (double)cnt;
  return isfinite(m) ? m : TV_INVALID;
}

// non-negative doubles order like their bit patterns
__device__ __forceinline__ void atomic_max_nonneg(unsigned long long* dst, double v) {
  atomicMax(dst, (unsigned long long)__double_as_longlong(v));
}

template <int NT>
__device__ double block_max(double v, double* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double m = red[0];
  for (int w = 1; w < NT / 32; ++w) m = fmax(m, red[w]);
  return m;
}

template <int NT, int NV>
__device__ void block_sums(double (&v)[NV], double* red /*[NT/32 * NV]*/) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = warp_sum(v[i]);
  __syncthreads();
  if (lane == 0)
#pragma unroll
    for (int i = 0; i < NV; ++i) red[warp * NV + i] = v[i];
  __syncthreads();
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    double s = 0.0;
    for (int w = 0; w < NT / 32; ++w) s += red[w * NV + i];
    v[i] = s;
  }
}

// -------------------------------------------------------------------------------------------------------------------
// 1. minimal solves + scoring
// -------------------------------------------------------------------------------------------------------------------
template <typename TP>
__global__ void __launch_bounds__(TV_TRIALS) tv_minimal_kernel(int N, int T, int K, const TP* __restrict__ p1,
                                                               const TP* __restrict__ p2,
                                                               const uint8_t* __restrict__ valid,
                                                               const int* __restrict__ samples, double thr, double pre,
                                                               int squared, int* __restrict__ cnt_out,
                                                               double* __restrict__ mean_out,
                                                               unsigned long long* __restrict__ thres_bits) {
  __shared__ double4 tile[TV_TILE];
  __shared__ uint8_t tval[TV_TILE];
  __shared__ double red[TV_TRIALS / 32];
  const int b = blockIdx.y, tid = threadIdx.x;
  const int trial = blockIdx.x * TV_TRIALS + tid;
  const bool active = trial < T;
  const TP* P1 = p1 + (size_t)b * N * 2;
  const TP* P2 = p2 + (size_t)b * N * 2;
  double F[27];
  if (active) candidate_7pt(P1, P2, samples, trial, F);
  else
    for (int i = 0; i < 27; ++i) F[i] = 0.0;
  int cnt[3] = {0, 0, 0};
  double sum[3] = {0.0, 0.0, 0.0};
  bool bad[3] = {false, false, false};
  const bool inval_in = TV_INVALID <= thr;
  for (int base = 0; base < N; base += TV_TILE) {
    const int nt = min(TV_TILE, N - base);
    __syncthreads();
    for (int i = tid; i < nt; i += TV_TRIALS) {
      const double2 a = ldp(P1, base + i), c = ldp(P2, base + i);
      tile[i] = make_double4(a.x, a.y, c.x, c.y);
      tval[i] = valid ? valid[(size_t)b * N + base + i] : 1;
    }
    __syncthreads();
    for (int j = 0; j < nt; ++j) {
      const double4 q = tile[j];
      if (!tval[j]) {                    // the reference's 1e6 overwrite (fundamental.py:102-104); uniform branch
        if (inval_in)
#pragma unroll
          for (int k = 0; k < 3; ++k) { cnt[k] += 1; sum[k] += TV_INVALID; }
        continue;
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        double num, den;
        sampson_parts(F + 9 * k, q.x, q.y, q.z, q.w, num, den);
        if (num <= pre * den) {          // only here can the residual reach the threshold
          double r = __ddiv_rn(num, den);
          if (!squared) r = __dsqrt_rn(__dadd_rn(r, 1e-8));
          if (r <= thr) { cnt[k] += 1; sum[k] += r; }
          bad[k] |= isnan(r);
        } else {
          bad[k] |= !(num <= DBL_MAX * den && den <= DBL_MAX);   // r = inf or NaN: the mean becomes NaN
        }
      }
    }
  }
  double mx = 0.0;
  if (active) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const size_t o = (size_t)b * K + 3 * trial + k;
      const double m = indicator_mean(cnt[k], sum[k], bad[k]);
      cnt_out[o] = cnt[k];
      mean_out[o] = m;
      mx = fmax(mx, m);
    }
  }
  mx = block_max<TV_TRIALS>(mx, red);
  if (tid == 0) atomic_max_nonneg(thres_bits, mx);
}

// -------------------------------------------------------------------------------------------------------------------
// 2. per-pair stable top-`take` by count (descending, lower candidate index first): counting sort, one warp per pair
// -------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32) tv_topk_kernel(int N, int K, int off, int nc, int take,
                                                     const int* __restrict__ cnt, int* __restrict__ seeds,
                                                     int seeds_stride, int* __restrict__ hist_all) {
  const int b = blockIdx.x, lane = threadIdx.x;
  int* hist = hist_all + (size_t)b * (N + 2);   // histogram, then the start position of each count
  const int* c = cnt + (size_t)b * K + off;
  for (int i = lane; i < N + 2; i += 32) hist[i] = 0;
  __syncwarp();
  for (int i = lane; i < nc; i += 32) atomicAdd(&hist[min(max(c[i], 0), N)], 1);
  __syncwarp();
  if (lane == 0) {                     // start[v] = number of candidates with a count above v
    int acc = 0;
    for (int v = N; v >= 0; --v) {
      const int h = hist[v];
      hist[v] = acc;
      acc += h;
    }
  }
  __syncwarp();
  for (int base = 0; base < nc; base += 32) {
    const int i = base + lane;
    const int v = i < nc ? min(max(c[i], 0), N) : -1 - lane;
    const unsigned same = __match_any_sync(0xffffffffu, v);
    const int before = __popc(same & ((1u << lane) - 1u));
    int pos = 0;
    if (i < nc) pos = hist[v] + before;
    __syncwarp();
    if (i < nc && before == 0) hist[v] += __popc(same);
    __syncwarp();
    if (i < nc && pos < take) seeds[(size_t)b * seeds_stride + pos] = i;
  }
}

// -------------------------------------------------------------------------------------------------------------------
// 3. local refinement: one CTA per (pair, seed)
// -------------------------------------------------------------------------------------------------------------------
struct LoShared {
  double F[27];
  double G[9];
  double A[81], V[81];
  double red[TV_LO_THREADS / 32 * 45];
  double t1[3], t2[3];
};

// round 1: seeds index the 3T minimal candidates, seed masks are the valid-masked inliers, and the raw (unmasked) count
// of each refined matrix is kept for round 2 (fundamental.py:131 ranks before the valid-mask overwrite).
// round 2: seeds index round-1 results, seed masks are raw inliers.
template <typename TP>
__global__ void __launch_bounds__(TV_LO_THREADS) tv_lo_kernel(int round, int N, int T, int K, int lo, int nseed,
                                                              const TP* __restrict__ p1, const TP* __restrict__ p2,
                                                              const uint8_t* __restrict__ valid,
                                                              const int* __restrict__ samples, double thr, int squared,
                                                              const int* __restrict__ seeds, double* __restrict__ Flo,
                                                              int* __restrict__ cnt_out, double* __restrict__ mean_out,
                                                              int* __restrict__ raw_cnt,
                                                              unsigned long long* __restrict__ thres_bits) {
  extern __shared__ uint8_t inl[];     // [N] inlier mask of the seed
  __shared__ LoShared sh;
  const int j = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const TP* P1 = p1 + (size_t)b * N * 2;
  const TP* P2 = p2 + (size_t)b * N * 2;
  const uint8_t* V = valid ? valid + (size_t)b * N : nullptr;
  const int lo2 = lo / 2;
  const int seed = seeds[(size_t)b * (round == 1 ? lo : lo2) + j];
  if (tid == 0) {
    if (round == 1) {
      candidate_7pt(P1, P2, samples, seed / 3, sh.F);
      for (int i = 0; i < 9; ++i) sh.G[i] = sh.F[9 * (seed % 3) + i];
    } else {
      for (int i = 0; i < 9; ++i) sh.G[i] = Flo[((size_t)b * (lo + lo2) + seed) * 9 + i];
    }
  }
  __syncthreads();
  // seed mask + masked mean (utils.py:203-210)
  double acc[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (int i = tid; i < N; i += TV_LO_THREADS) {
    const double2 a = ldp(P1, i), c = ldp(P2, i);
    bool in;
    if (round == 1 && V && !V[i]) in = TV_INVALID <= thr;
    else in = sampson_full(sh.G, a.x, a.y, c.x, c.y, squared) <= thr;
    inl[i] = in;
    if (in) { acc[0] += 1.0; acc[1] += a.x; acc[2] += a.y; acc[3] += c.x; acc[4] += c.y; }
  }
  block_sums<TV_LO_THREADS, 5>(acc, sh.red);
  const double n = acc[0];
  const double m1x = acc[1] / (n + 1e-8), m1y = acc[2] / (n + 1e-8), m2x = acc[3] / (n + 1e-8), m2y = acc[4] / (n + 1e-8);
  double d[2] = {0.0, 0.0};
  for (int i = tid; i < N; i += TV_LO_THREADS) {
    if (!inl[i]) continue;
    const double2 a = ldp(P1, i), c = ldp(P2, i);
    d[0] += sqrt((a.x - m1x) * (a.x - m1x) + (a.y - m1y) * (a.y - m1y));
    d[1] += sqrt((c.x - m2x) * (c.x - m2x) + (c.y - m2y) * (c.y - m2y));
  }
  block_sums<TV_LO_THREADS, 2>(d, sh.red);
  const double s1 = TV_SQRT2_F32 / (d[0] / (n + 1e-8) + 1e-8), s2 = TV_SQRT2_F32 / (d[1] / (n + 1e-8) + 1e-8);
  // 9x9 normal matrix, upper triangle (fundamental.py:303-313)
  double M[45];
#pragma unroll
  for (int k = 0; k < 45; ++k) M[k] = 0.0;
  for (int i = tid; i < N; i += TV_LO_THREADS) {
    if (!inl[i]) continue;
    const double2 a = ldp(P1, i), c = ldp(P2, i);
    const double x1 = (s1 * a.x + (-s1 * m1x)) * TV_HOM, y1 = (s1 * a.y + (-s1 * m1y)) * TV_HOM;
    const double x2 = (s2 * c.x + (-s2 * m2x)) * TV_HOM, y2 = (s2 * c.y + (-s2 * m2y)) * TV_HOM;
    const double row[9] = {x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, 1.0};
    int k = 0;
#pragma unroll
    for (int r = 0; r < 9; ++r)
#pragma unroll
      for (int q = r; q < 9; ++q) M[k++] += row[r] * row[q];
  }
  block_sums<TV_LO_THREADS, 45>(M, sh.red);
  if (tid == 0) {
    double* A = sh.A;
    double v[9];
    int k = 0;
    for (int r = 0; r < 9; ++r)
      for (int q = r; q < 9; ++q) { A[r * 9 + q] = A[q * 9 + r] = M[k++]; }
    smallest_eigvec<9>(A, sh.V, v);
    // rank-2 projection F - F v3 v3^T (= U diag(s1, s2, 0) V^T), v3 the smallest eigenvector of F^T F
    double FtF[9], W3[9], e[3];
    for (int r = 0; r < 3; ++r)
      for (int q = 0; q < 3; ++q) {
        double s = 0.0;
        for (int t = 0; t < 3; ++t) s += v[t * 3 + r] * v[t * 3 + q];
        FtF[r * 3 + q] = s;
      }
    smallest_eigvec<3>(FtF, W3, e);
    double Fp[9];
    for (int r = 0; r < 3; ++r) {
      const double fe = v[r * 3] * e[0] + v[r * 3 + 1] * e[1] + v[r * 3 + 2] * e[2];
      for (int q = 0; q < 3; ++q) Fp[r * 3 + q] = v[r * 3 + q] - fe * e[q];
    }
    const double t1[3] = {s1, m1x, m1y}, t2[3] = {s2, m2x, m2y};
    denormalize(Fp, t1, t2);
    if (Fp[8] < 0.0)
      for (int i = 0; i < 9; ++i) Fp[i] = -Fp[i];
    normalize_transformation(Fp);
    const int slot = (round == 1 ? 0 : lo) + j;
    for (int i = 0; i < 9; ++i) {
      sh.G[i] = Fp[i];
      Flo[((size_t)b * (lo + lo2) + slot) * 9 + i] = Fp[i];
    }
  }
  __syncthreads();
  // score the refined matrix: valid-masked count / sum / non-finite flag, and in round 1 the raw count
  double sc[4] = {0.0, 0.0, 0.0, 0.0};
  for (int i = tid; i < N; i += TV_LO_THREADS) {
    const double2 a = ldp(P1, i), c = ldp(P2, i);
    const double r = sampson_full(sh.G, a.x, a.y, c.x, c.y, squared);
    if (r <= thr) sc[3] += 1.0;
    if (V && !V[i]) {
      if (TV_INVALID <= thr) { sc[0] += 1.0; sc[1] += TV_INVALID; }
      continue;
    }
    if (r <= thr) { sc[0] += 1.0; sc[1] += r; }
    if (!isfinite(r)) sc[2] = 1.0;
  }
  block_sums<TV_LO_THREADS, 4>(sc, sh.red);
  if (tid == 0) {
    const size_t o = (size_t)b * K + 3 * (size_t)T + (round == 1 ? 0 : lo) + j;
    const int c = (int)(sc[0] + 0.5);
    const double m = indicator_mean(c, sc[1], sc[2] != 0.0);
    cnt_out[o] = c;
    mean_out[o] = m;
    if (round == 1) raw_cnt[(size_t)b * lo + j] = (int)(sc[3] + 0.5);
    atomic_max_nonneg(thres_bits, m);
  }
}

// -------------------------------------------------------------------------------------------------------------------
// 4. selection (utils.py:63-87, fundamental.py:164-181)
// -------------------------------------------------------------------------------------------------------------------
template <typename TP>
__global__ void __launch_bounds__(256) tv_select_kernel(int N, int T, int K, int Ku, int lo, const TP* __restrict__ p1,
                                                        const TP* __restrict__ p2, const uint8_t* __restrict__ valid,
                                                        const int* __restrict__ samples, double thr, int squared,
                                                        const int* __restrict__ cnt, const double* __restrict__ mean,
                                                        const double* __restrict__ Flo,
                                                        const unsigned long long* __restrict__ thres_bits,
                                                        double* __restrict__ fmat_out, int* __restrict__ num_out,
                                                        uint8_t* __restrict__ mask_out, double* __restrict__ res_out) {
  __shared__ double bv[8];
  __shared__ int bi[8];
  __shared__ double F[27];
  __shared__ double G[9];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const double thres = __longlong_as_double((long long)*thres_bits) + 1e-6;
  double best = -INFINITY;
  int besti = 0x7fffffff;
  for (int k = tid; k < Ku; k += 256) {
    const size_t o = (size_t)b * K + k;
    const double ind = (thres - mean[o]) / thres + (double)cnt[o];
    if (ind > best) { best = ind; besti = k; }       // k increases: the first maximum is kept
  }
  for (int off = 16; off >= 1; off >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, best, off);
    const int oi = __shfl_xor_sync(0xffffffffu, besti, off);
    if (ov > best || (ov == best && oi < besti)) { best = ov; besti = oi; }
  }
  if (lane == 0) { bv[warp] = best; bi[warp] = besti; }
  __syncthreads();
  const TP* P1 = p1 + (size_t)b * N * 2;
  const TP* P2 = p2 + (size_t)b * N * 2;
  if (tid == 0) {
    for (int w = 1; w < 8; ++w)
      if (bv[w] > best || (bv[w] == best && bi[w] < besti)) { best = bv[w]; besti = bi[w]; }
    if (besti < 3 * T) {
      candidate_7pt(P1, P2, samples, besti / 3, F);
      for (int i = 0; i < 9; ++i) G[i] = F[9 * (besti % 3) + i];
    } else {
      for (int i = 0; i < 9; ++i) G[i] = Flo[((size_t)b * (lo + lo / 2) + besti - 3 * T) * 9 + i];
    }
    for (int i = 0; i < 9; ++i) fmat_out[(size_t)b * 9 + i] = G[i];
  }
  __syncthreads();
  double c = 0.0;
  for (int i = tid; i < N; i += 256) {
    double r;
    if (valid && !valid[(size_t)b * N + i]) {
      r = TV_INVALID;
    } else {
      const double2 a = ldp(P1, i), q = ldp(P2, i);
      r = sampson_full(G, a.x, a.y, q.x, q.y, squared);
    }
    const bool in = r <= thr;
    res_out[(size_t)b * N + i] = r;
    mask_out[(size_t)b * N + i] = in;
    c += in ? 1.0 : 0.0;
  }
  double cc[1] = {c};
  block_sums<256, 1>(cc, bv);
  if (tid == 0) num_out[b] = (int)(cc[0] + 0.5);
}

// -------------------------------------------------------------------------------------------------------------------
// 5. relative pose: E = K2^T F K1, decomposition, cheirality vote (one CTA per pair)
// -------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cross3(const double* a, const double* b, double* o) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}

// One-sided (Hestenes) Jacobi on the m x n row-major A: plane rotations V make the columns of A V mutually orthogonal
// (to 4 eps relative), and A is overwritten by A V.  Working on A itself rather than on A^T A keeps the singular
// vectors accurate to about eps sigma_1 / gap instead of eps (sigma_1 / gap)^2.  A pair whose columns are already
// orthogonal, zero or not finite is left alone.
template <int m, int n>
__device__ void jacobi_svd(double* A, double* V) {
#pragma unroll
  for (int i = 0; i < n * n; ++i) V[i] = (i % (n + 1) == 0) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 30; ++sweep) {
    bool rotated = false;
#pragma unroll
    for (int p = 0; p < n; ++p)
#pragma unroll
      for (int q = p + 1; q < n; ++q) {
        double al = 0.0, be = 0.0, ga = 0.0;
#pragma unroll
        for (int k = 0; k < m; ++k) {
          al += A[k * n + p] * A[k * n + p];
          be += A[k * n + q] * A[k * n + q];
          ga += A[k * n + p] * A[k * n + q];
        }
        if (!(fabs(ga) > 4.0 * DBL_EPSILON * sqrt(al) * sqrt(be))) continue;
        const double zeta = (be - al) / (2.0 * ga);
        const double t = fabs(zeta) > 1e150 ? 0.5 / zeta
                                             : (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
#pragma unroll
        for (int k = 0; k < m; ++k) {
          const double ap = A[k * n + p], aq = A[k * n + q];
          A[k * n + p] = c * ap - s * aq;
          A[k * n + q] = s * ap + c * aq;
        }
#pragma unroll
        for (int k = 0; k < n; ++k) {
          const double vp = V[k * n + p], vq = V[k * n + q];
          V[k * n + p] = c * vp - s * vq;
          V[k * n + q] = s * vp + c * vq;
        }
        rotated = true;
      }
    if (!rotated) break;
  }
}

// 3x3 SVD of E by one-sided Jacobi; U, V row-major with singular vectors in the columns, descending order.  The third
// left vector is u0 x u1 (E has rank <= 2); the determinant fixes of the reference are then no-ops for U.  Where
// E v_i vanishes (rank <= 1, E = 0) the left vectors are completed to an orthonormal basis: u0 = e0 when E = 0, u1
// from the coordinate axis least aligned with u0 (E = 0 then gives U = V = I, as LAPACK does).
__device__ void svd3(const double* E, double* U, double* V) {
  double A[9], nrm[3];
  for (int i = 0; i < 9; ++i) A[i] = E[i];
  jacobi_svd<3, 3>(A, V);
  for (int i = 0; i < 3; ++i) nrm[i] = sqrt(A[i] * A[i] + A[3 + i] * A[3 + i] + A[6 + i] * A[6 + i]);
  int o[3] = {0, 1, 2};
  for (int i = 0; i < 3; ++i)
    for (int k = i + 1; k < 3; ++k)
      if (nrm[o[k]] > nrm[o[i]]) { const int t = o[i]; o[i] = o[k]; o[k] = t; }
  double W[9];
  for (int i = 0; i < 9; ++i) W[i] = V[i];
  for (int i = 0; i < 3; ++i)
    for (int r = 0; r < 3; ++r) V[r * 3 + i] = W[r * 3 + o[i]];
  double u[3][3];
  for (int i = 0; i < 2; ++i)
    for (int r = 0; r < 3; ++r) u[i][r] = nrm[o[i]] != 0.0 ? A[r * 3 + o[i]] / nrm[o[i]] : 0.0;   // NaN stays NaN
  if (nrm[o[0]] == 0.0) { u[0][0] = 1.0; u[0][1] = 0.0; u[0][2] = 0.0; }
  // re-orthogonalise u1 against u0 (equal singular values of an essential matrix), or complete it
  for (int pass = 0; pass < 2; ++pass) {
    double dp = u[0][0] * u[1][0] + u[0][1] * u[1][1] + u[0][2] * u[1][2], nn = 0.0;
    for (int r = 0; r < 3; ++r) { u[1][r] -= dp * u[0][r]; nn += u[1][r] * u[1][r]; }
    nn = sqrt(nn);
    if (pass == 0 && nn <= 0.5) {              // E v1 vanished (or lay along u0): the axis least aligned with u0
      int k = 0;
      for (int r = 1; r < 3; ++r)
        if (fabs(u[0][r]) < fabs(u[0][k])) k = r;
      for (int r = 0; r < 3; ++r) u[1][r] = r == k ? 1.0 : 0.0;
      continue;
    }
    for (int r = 0; r < 3; ++r) u[1][r] /= nn;
    break;
  }
  cross3(u[0], u[1], u[2]);
  for (int i = 0; i < 3; ++i)
    for (int r = 0; r < 3; ++r) U[r * 3 + i] = u[i][r];
}

template <typename TP>
__global__ void __launch_bounds__(128) tv_pose_kernel(int N, double width, double height, const TP* __restrict__ p1,
                                                      const TP* __restrict__ p2, const double* __restrict__ fmat,
                                                      double* __restrict__ R_out, double* __restrict__ t_out,
                                                      double* __restrict__ E_out, int* __restrict__ counts_out) {
  __shared__ double Rs[4][9], ts[4][3], maxd[4];
  __shared__ double red[4 * 4];
  const int b = blockIdx.x, tid = threadIdx.x;
  const double f = fmax(width, height), cx = width / 2.0, cy = height / 2.0;
  if (tid == 0) {
    const double* F = fmat + (size_t)b * 9;
    const double Kd[9] = {f, 0.0, cx, 0.0, f, cy, 0.0, 0.0, 1.0};
    double G[9], E[9];
    for (int r = 0; r < 3; ++r)
      for (int q = 0; q < 3; ++q) {
        double s = 0.0;
        for (int k = 0; k < 3; ++k) s += F[r * 3 + k] * Kd[k * 3 + q];
        G[r * 3 + q] = s;
      }
    for (int r = 0; r < 3; ++r)
      for (int q = 0; q < 3; ++q) {
        double s = 0.0;
        for (int k = 0; k < 3; ++k) s += Kd[k * 3 + r] * G[k * 3 + q];
        E[r * 3 + q] = s;
      }
    for (int i = 0; i < 9; ++i) E_out[(size_t)b * 9 + i] = E[i];
    double U[9], V[9];
    svd3(E, U, V);
    if (det3(V) < 0.0)                                  // Vt * maskt: last row of V^T = last column of V
      for (int r = 0; r < 3; ++r) V[r * 3 + 2] = -V[r * 3 + 2];
    if (det3(U) < 0.0)
      for (int r = 0; r < 3; ++r) U[r * 3 + 2] = -U[r * 3 + 2];
    // orientation pin: t = U[:, 2] with its largest-magnitude entry positive (U, V -> U P, V P, P = diag(-1, 1, -1))
    int im = 0;
    for (int r = 1; r < 3; ++r)
      if (fabs(U[r * 3 + 2]) > fabs(U[im * 3 + 2])) im = r;
    if (U[im * 3 + 2] < 0.0)
      for (int r = 0; r < 3; ++r) {
        U[r * 3] = -U[r * 3]; U[r * 3 + 2] = -U[r * 3 + 2];
        V[r * 3] = -V[r * 3]; V[r * 3 + 2] = -V[r * 3 + 2];
      }
    // R1 = U W V^T, R2 = U W^T V^T with W = [[0,-1,0],[1,0,0],[0,0,1]]: U W = [u1, -u0, u2], U W^T = [-u1, u0, u2]
    for (int r = 0; r < 3; ++r)
      for (int q = 0; q < 3; ++q) {
        const double a = U[r * 3 + 1] * V[q * 3] - U[r * 3] * V[q * 3 + 1] + U[r * 3 + 2] * V[q * 3 + 2];
        const double c = -U[r * 3 + 1] * V[q * 3] + U[r * 3] * V[q * 3 + 1] + U[r * 3 + 2] * V[q * 3 + 2];
        Rs[0][r * 3 + q] = Rs[1][r * 3 + q] = a;
        Rs[2][r * 3 + q] = Rs[3][r * 3 + q] = c;
      }
    for (int r = 0; r < 3; ++r) {
      ts[0][r] = ts[2][r] = U[r * 3 + 2];
      ts[1][r] = ts[3][r] = -U[r * 3 + 2];
    }
    for (int k = 0; k < 4; ++k) {
      double n2 = 0.0;
      for (int q = 0; q < 3; ++q) {
        const double v = Rs[k][q] * ts[k][0] + Rs[k][3 + q] * ts[k][1] + Rs[k][6 + q] * ts[k][2];
        n2 += v * v;
      }
      maxd[k] = 1000.0 * sqrt(n2);
    }
  }
  __syncthreads();
  double cnt[4] = {0.0, 0.0, 0.0, 0.0};
  const TP* P1 = p1 + (size_t)b * N * 2;
  const TP* P2 = p2 + (size_t)b * N * 2;
  for (int i = tid; i < N; i += 128) {
    const double2 a = ldp(P1, i), c = ldp(P2, i);
    const double x1 = (a.x - cx) / f, y1 = (a.y - cy) / f, x2 = (c.x - cx) / f, y2 = (c.y - cy) / f;
#pragma unroll 1
    for (int k = 0; k < 4; ++k) {
      const double* R = Rs[k];
      const double* t = ts[k];
      // two-view DLT (utils.py:366-395): rows of A, X = smallest right singular vector
      double A[16];
      A[0] = -1.0; A[1] = 0.0; A[2] = x1; A[3] = 0.0;
      A[4] = 0.0; A[5] = -1.0; A[6] = y1; A[7] = 0.0;
      for (int q = 0; q < 3; ++q) {
        A[8 + q] = x2 * R[6 + q] - R[q];
        A[12 + q] = y2 * R[6 + q] - R[3 + q];
      }
      A[11] = x2 * t[2] - t[0];
      A[15] = y2 * t[2] - t[1];
      double AtA[16], W4[16], v[4];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int q = 0; q < 4; ++q)
          AtA[r * 4 + q] = A[r] * A[q] + A[4 + r] * A[4 + q] + A[8 + r] * A[8 + q] + A[12 + r] * A[12 + q];
      bool fin = true;
#pragma unroll
      for (int q = 0; q < 16; ++q) fin = fin && isfinite(A[q]);
      if (!fin) continue;
      smallest_eigvec<4>(AtA, W4, v);
      const double X0 = v[0] / v[3], X1 = v[1] / v[3], X2 = v[2] / v[3];
      const double d1 = X2, d2 = R[6] * X0 + R[7] * X1 + R[8] * X2 + t[2];
      if (d1 > TV_MIN_DEPTH && d1 < maxd[k] && d2 > TV_MIN_DEPTH && d2 < maxd[k]) cnt[k] += 1.0;
    }
  }
  block_sums<128, 4>(cnt, red);
  if (tid == 0) {
    int kb = 0;
    for (int k = 1; k < 4; ++k)
      if (cnt[k] > cnt[kb]) kb = k;
    for (int i = 0; i < 9; ++i) R_out[(size_t)b * 9 + i] = Rs[kb][i];
    for (int i = 0; i < 3; ++i) t_out[(size_t)b * 3 + i] = ts[kb][i];
    if (counts_out)
      for (int k = 0; k < 4; ++k) counts_out[(size_t)b * 4 + k] = (int)(cnt[k] + 0.5);
  }
}

// inlier_by_fundamental (utils.py:300-322): Sampson inliers of every match under one matrix per pair
template <typename TP>
__global__ void __launch_bounds__(256) tv_inlier_kernel(int N, const TP* __restrict__ p1, const TP* __restrict__ p2,
                                                        const double* __restrict__ fmat, double thr, int squared,
                                                        uint8_t* __restrict__ mask_out) {
  const int b = blockIdx.y, i = blockIdx.x * 256 + threadIdx.x;
  if (i >= N) return;
  double F[9];
  for (int k = 0; k < 9; ++k) F[k] = fmat[(size_t)b * 9 + k];
  const double2 a = ldp(p1 + (size_t)b * N * 2, i), c = ldp(p2 + (size_t)b * N * 2, i);
  mask_out[(size_t)b * N + i] = sampson_full(F, a.x, a.y, c.x, c.y, squared) <= thr;
}

struct TvWork {
  int* cnt;
  double* mean;
  int* seeds1;
  int* seeds2;
  int* raw;
  double* Flo;
  unsigned long long* thres;
  int* samples;
  int* hist;
};

TvWork carve(void* ws, size_t bytes, int B, int N, int T, int lo, size_t* need) {
  Carver c(ws, bytes);
  const size_t K = 3 * (size_t)T + lo + lo / 2;
  TvWork w;
  w.cnt = c.take<int>((size_t)B * K);
  w.mean = c.take<double>((size_t)B * K);
  w.seeds1 = c.take<int>((size_t)B * lo);
  w.seeds2 = c.take<int>((size_t)B * (lo / 2 + 1));
  w.raw = c.take<int>((size_t)B * lo);
  w.Flo = c.take<double>((size_t)B * (lo + lo / 2) * 9);
  w.thres = c.take<unsigned long long>(1);
  w.samples = c.take<int>((size_t)T * 7);
  w.hist = c.take<int>((size_t)B * (N + 2));
  if (need) *need = align_up(c.off, 256);
  return w;
}

template <typename TP>
int estimate_fundamental_t(int B, int N, const TP* p1, const TP* p2, const uint8_t* valid, const int* samples, int T,
                           int lo, double thr, int squared, int second_refine, double* fmat, int* num, uint8_t* mask,
                           double* res, const TvWork& w, cudaStream_t st) {
  const int lo2 = second_refine ? lo / 2 : 0;
  // candidates of a pair: 3T minimal, lo first-round, lo/2 second-round (the slot range is kept when second_refine
  // is off; K_used excludes it from the selection)
  const int Kst = 3 * T + lo + lo / 2;
  const double pre = 2.0 * (squared ? thr : thr * thr);
  VGG_CUDA_CHECK(cudaMemsetAsync(w.thres, 0, sizeof(unsigned long long), st));
  tv_minimal_kernel<TP><<<dim3((T + TV_TRIALS - 1) / TV_TRIALS, B), TV_TRIALS, 0, st>>>(
      N, T, Kst, p1, p2, valid, samples, thr, pre, squared, w.cnt, w.mean, w.thres);
  VGG_LAUNCH_CHECK();
  tv_topk_kernel<<<B, 32, 0, st>>>(N, Kst, 0, 3 * T, lo, w.cnt, w.seeds1, lo, w.hist);
  VGG_LAUNCH_CHECK();
  tv_lo_kernel<TP><<<dim3(lo, B), TV_LO_THREADS, N, st>>>(1, N, T, Kst, lo, lo, p1, p2, valid, samples, thr, squared,
                                                          w.seeds1, w.Flo, w.cnt, w.mean, w.raw, w.thres);
  VGG_LAUNCH_CHECK();
  if (lo2 > 0) {
    tv_topk_kernel<<<B, 32, 0, st>>>(N, lo, 0, lo, lo2, w.raw, w.seeds2, lo / 2, w.hist);
    VGG_LAUNCH_CHECK();
    tv_lo_kernel<TP><<<dim3(lo2, B), TV_LO_THREADS, N, st>>>(2, N, T, Kst, lo, lo2, p1, p2, valid, samples, thr,
                                                             squared, w.seeds2, w.Flo, w.cnt, w.mean, w.raw, w.thres);
    VGG_LAUNCH_CHECK();
  }
  // without the second round the candidate list ends after the first one (row stride Kst, 3T + lo + lo2 used)
  tv_select_kernel<TP><<<B, 256, 0, st>>>(N, T, Kst, 3 * T + lo + lo2, lo, p1, p2, valid, samples, thr, squared, w.cnt, w.mean, w.Flo,
                                          w.thres, fmat, num, mask, res);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

}  // namespace

}  // namespace vgg

using namespace vgg;

extern "C" {

int vgg_twoview_workspace_bytes(int B, int N, int T, int lo_num, size_t* bytes) {
  VGG_REQUIRE(B >= 0 && N >= 0 && T >= 0 && lo_num >= 0 && bytes, "bad arguments");
  carve(nullptr, 0, B, N, T, lo_num, bytes);
  return VGG_OK;
}

int vgg_estimate_fundamental(int B, int N, const void* points1, const void* points2, int points_are_f64,
                             const uint8_t* valid_mask, const int32_t* samples, int T, int lo_num, double threshold,
                             int squared, int second_refine, double* fmat_out, int32_t* inlier_num_out,
                             uint8_t* inlier_mask_out, double* residuals_out, void* workspace, size_t ws_bytes,
                             void* stream) {
  VGG_REQUIRE(B >= 0 && N >= 7 && T >= 7, "estimate_fundamental: N and T must be at least 7");
  VGG_REQUIRE(lo_num >= 1 && lo_num <= 3 * T, "estimate_fundamental: lo_num must lie in [1, 3 T]");
  VGG_REQUIRE(N <= TV_MAX_N, "estimate_fundamental: at most 190000 points per pair (seed masks live in shared memory)");
  g_launch_count = 0;
  if (B == 0) return VGG_OK;
  VGG_REQUIRE(points1 && points2 && samples && fmat_out && inlier_num_out && inlier_mask_out && residuals_out &&
                  workspace, "null pointer");
  VGG_REQUIRE(threshold >= 0.0, "estimate_fundamental: negative threshold");
  for (size_t i = 0; i < (size_t)T * 7; ++i)
    VGG_REQUIRE(samples[i] >= 0 && samples[i] < N, "estimate_fundamental: sample index out of range [0, N)");
  size_t need = 0;
  carve(nullptr, 0, B, N, T, lo_num, &need);
  if (ws_bytes < need) {
    set_error("twoview workspace too small: need %zu bytes", need);
    return VGG_EWORKSPACE;
  }
  TvWork w = carve(workspace, ws_bytes, B, N, T, lo_num, nullptr);
  cudaStream_t st = (cudaStream_t)stream;
  VGG_CUDA_CHECK(cudaMemcpyAsync(w.samples, samples, (size_t)T * 7 * sizeof(int), cudaMemcpyHostToDevice, st));
  VGG_CUDA_CHECK(cudaFuncSetAttribute(tv_lo_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, TV_MAX_N));
  VGG_CUDA_CHECK(cudaFuncSetAttribute(tv_lo_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, TV_MAX_N));
  if (points_are_f64)
    return estimate_fundamental_t(B, N, (const double*)points1, (const double*)points2, valid_mask, w.samples, T, lo_num,
                                  threshold, squared, second_refine, fmat_out, inlier_num_out, inlier_mask_out,
                                  residuals_out, w, st);
  return estimate_fundamental_t(B, N, (const float*)points1, (const float*)points2, valid_mask, w.samples, T, lo_num,
                                threshold, squared, second_refine, fmat_out, inlier_num_out, inlier_mask_out,
                                residuals_out, w, st);
}

int vgg_fundamental_inliers(int B, int N, const void* points1, const void* points2, int points_are_f64,
                            const double* fmat, double threshold, int squared, uint8_t* inlier_mask_out, void* stream) {
  VGG_REQUIRE(B >= 0 && N >= 0, "bad arguments");
  g_launch_count = 0;
  if (B == 0 || N == 0) return VGG_OK;
  VGG_REQUIRE(points1 && points2 && fmat && inlier_mask_out, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((N + 255) / 256, B);
  if (points_are_f64)
    tv_inlier_kernel<double><<<grid, 256, 0, st>>>(N, (const double*)points1, (const double*)points2, fmat, threshold,
                                                   squared, inlier_mask_out);
  else
    tv_inlier_kernel<float><<<grid, 256, 0, st>>>(N, (const float*)points1, (const float*)points2, fmat, threshold,
                                                  squared, inlier_mask_out);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

int vgg_relative_pose_from_fundamental(int B, int N, const void* points1, const void* points2, int points_are_f64,
                                       const double* fmat, double width, double height, double* R_out, double* t_out,
                                       double* E_out, void* stream) {
  return vgg_dev_relative_pose_counts(B, N, points1, points2, points_are_f64, fmat, width, height, R_out, t_out, E_out,
                                      nullptr, stream);
}

int vgg_dev_relative_pose_counts(int B, int N, const void* points1, const void* points2, int points_are_f64,
                                 const double* fmat, double width, double height, double* R_out, double* t_out,
                                 double* E_out, int32_t* counts_out, void* stream) {
  VGG_REQUIRE(B >= 0 && N >= 0 && width > 0 && height > 0, "bad arguments");
  g_launch_count = 0;
  if (B == 0) return VGG_OK;
  VGG_REQUIRE(points1 && points2 && fmat && R_out && t_out && E_out, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (points_are_f64)
    tv_pose_kernel<double><<<B, 128, 0, st>>>(N, width, height, (const double*)points1, (const double*)points2, fmat,
                                              R_out, t_out, E_out, counts_out);
  else
    tv_pose_kernel<float><<<B, 128, 0, st>>>(N, width, height, (const float*)points1, (const float*)points2, fmat,
                                             R_out, t_out, E_out, counts_out);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

}  // extern "C"
