// Batched LO-MSAC fundamental matrix of the default two-view stage: poselib.estimate_fundamental as
// estimate_preliminary_cameras_poselib calls it (vggsfm/two_view_geo/estimate_preliminary.py:37-95), restated in
// oracle/poselib_oracle.py (float64 throughout; the header there lists every rule and every choice).
//
// PoseLib's loop is sequential, but whether a trial runs local optimisation (LO), and from which candidate, depends only
// on the minimal scores (running maximum of the inlier count, running minimum of the MSAC score), never on an LO result.
// Only the bookkeeping (best model, its score, dynamic_max_iter, the stop) depends on LO results.  So the trials run in
// chunks (the first one min_iterations + 1 trials, which is what a pair with a high inlier ratio needs):
//   ms_compact_kernel   one CTA per pair: the valid matches compacted in order, the shared scale, the scaled points.
//   per chunk:
//   ms_sample_kernel    one thread per live pair: the LCG draws of the chunk (the state persists across chunks).
//   ms_minimal_kernel   one thread per (pair, trial): 7-point solve (real roots), real focal check, MSAC count and score
//                       of every kept candidate, the pair's points streamed through shared memory.  Candidates are not
//                       stored; later kernels recompute them from the trial's sample.
//   ms_trigger_kernel   one warp per pair: prefix max / min scan over the chunk -> the trials that run LO, their seeds
//                       and the candidates that improve on the running minimal bests.
//   ms_lo_kernel        one CTA per (pair, trigger): truncated-loss LM with block reductions into the 7 x 7 normal
//                       equations, then the MSAC score of the result.
//   ms_resolve_kernel   one thread per pair: the bookkeeping over the chunk's triggers in trial order, and the stop.
//   ms_final_kernel     one CTA per pair: final LO, mask, Cauchy polish on the inliers, denormalisation.
// The host reads the largest trigger count and the number of live pairs once per chunk.
#include <float.h>
#include <math.h>
#include <algorithm>
#include "common.cuh"
#include "dev_probes.h"
#include "twoview_geom.h"

namespace vgg {

namespace {

constexpr int MS_TRIALS = 128;        // trials (threads) per CTA of the minimal kernel
constexpr int MS_TILE = 256;          // points per shared-memory tile of the minimal kernel
constexpr int MS_LO_THREADS = 256;    // threads of an LO / final CTA
constexpr int MS_MAX_CHUNK = 2048;    // trials per chunk at most (the workspace holds one chunk)
constexpr int MS_TRACE_CAP = 64;      // LO trials recorded per pair for vgg_dev_msac_trace
constexpr int MS_LO_ITERS = 25;
constexpr int MS_POLISH_ITERS = 100;
constexpr double MS_SUCCESS_PROB = 0.9999;
constexpr double MS_GRAD_TOL = 1e-10, MS_STEP_TOL = 1e-8;
constexpr double MS_LAMBDA0 = 1e-3, MS_MIN_LAMBDA = 1e-10, MS_MAX_LAMBDA = 1e10;

struct PairState {
  double best_min_score, model_score;
  double F[9];                 // best model (scaled frame)
  int best_min_cnt, model_cnt;
  int dyn, stopped, iterations;
  int src_kind, src_trial, src_slot;   // 0 none, 1 minimal candidate, 2 LO result
  int lo_runs;
};

struct Trig {
  int trial, seed, nimp;
  int icnt[3], islot[3];
  double isc[3];
};

struct MsWork {
  double4* pts;       // [B,N] scaled (x1, y1, x2, y2) of the valid matches, compacted
  int* idx;           // [B,N] original match index
  uint8_t* inl;       // [B,N] inliers of the final model
  int* nval;          // [B]
  double* scale;      // [B]
  unsigned long long* rng;   // [B]
  PairState* st;      // [B]
  int* samples;       // [B,C,7]
  int* cand;          // [B,C]   kept candidates: count | slot0 << 4 | slot1 << 8 | slot2 << 12
  int* mcnt;          // [B,C,3]
  double* msc;        // [B,C,3]
  Trig* trig;         // [B,C]
  int* ntrig;         // [B]
  double* loF;        // [B,C,9]
  int* locnt;         // [B,C]
  double* losc;       // [B,C]
  int* ctr;           // [2] largest trigger count, live pairs
  int* trace;         // [B, MS_TRACE_CAP]
};

int chunk_of(int max_iterations, int min_iterations) {
  return (int)std::max(1ll, std::min<long long>({(long long)max_iterations, (long long)min_iterations + 1,
                                                 (long long)MS_MAX_CHUNK}));
}

MsWork carve_ms(void* ws, size_t bytes, int B, int N, int C, size_t* need) {
  Carver c(ws, bytes);
  const size_t BN = (size_t)B * N, BC = (size_t)B * C;
  MsWork w;
  w.pts = c.take<double4>(BN);
  w.idx = c.take<int>(BN);
  w.inl = c.take<uint8_t>(BN);
  w.nval = c.take<int>(B);
  w.scale = c.take<double>(B);
  w.rng = c.take<unsigned long long>(B);
  w.st = c.take<PairState>(B);
  w.samples = c.take<int>(BC * 7);
  w.cand = c.take<int>(BC);
  w.mcnt = c.take<int>(BC * 3);
  w.msc = c.take<double>(BC * 3);
  w.trig = c.take<Trig>(BC);
  w.ntrig = c.take<int>(B);
  w.loF = c.take<double>(BC * 9);
  w.locnt = c.take<int>(BC);
  w.losc = c.take<double>(BC);
  w.ctr = c.take<int>(2);
  w.trace = c.take<int>((size_t)B * MS_TRACE_CAP);
  if (need) *need = align_up(c.off, 256);
  return w;
}

__device__ __forceinline__ double sq_sampson(const double* F, double4 q, double& e, double& den) {
  const double l0 = __fma_rn(F[0], q.x, __fma_rn(F[1], q.y, F[2]));
  const double l1 = __fma_rn(F[3], q.x, __fma_rn(F[4], q.y, F[5]));
  const double l2 = __fma_rn(F[6], q.x, __fma_rn(F[7], q.y, F[8]));
  const double m0 = __fma_rn(F[0], q.z, __fma_rn(F[3], q.w, F[6]));
  const double m1 = __fma_rn(F[1], q.z, __fma_rn(F[4], q.w, F[7]));
  e = __fma_rn(q.z, l0, __fma_rn(q.w, l1, l2));
  den = __fma_rn(l0, l0, __fma_rn(l1, l1, __fma_rn(m0, m0, __dmul_rn(m1, m1))));
  return __ddiv_rn(__dmul_rn(e, e), den);
}

// z component of e x a, for the Bougnoux sign test
__device__ __forceinline__ double cross_z(const double* e, double ax, double ay) { return e[0] * ay - e[1] * ax; }

// longest cross product of two columns of row-major M (orthogonal to its column space when M has rank 2)
__device__ void epipole(const double* M, double* e) {
  auto at = [&](int r, int c) { return M[r * 3 + c]; };
  double best = -1.0;
  const int pr[3][2] = {{0, 1}, {0, 2}, {1, 2}};
  for (int q = 0; q < 3; ++q) {
    const int i = pr[q][0], j = pr[q][1];
    const double c0 = at(1, i) * at(2, j) - at(2, i) * at(1, j);
    const double c1 = at(2, i) * at(0, j) - at(0, i) * at(2, j);
    const double c2 = at(0, i) * at(1, j) - at(1, i) * at(0, j);
    const double n = c0 * c0 + c1 * c1 + c2 * c2;
    if (n > best) { best = n; e[0] = c0; e[1] = c1; e[2] = c2; }
  }
}

// real focal check (Bougnoux, principal point at the origin): false when a focal length is imaginary or F not finite
__device__ bool real_focal(const double* F) {
  for (int i = 0; i < 9; ++i)
    if (!isfinite(F[i])) return false;
  double G[9];
  for (int view = 0; view < 2; ++view) {
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) G[r * 3 + c] = view == 0 ? F[r * 3 + c] : F[c * 3 + r];
    double e[3];
    epipole(G, e);
    const double n = cross_z(e, G[2], G[5]) * G[8];
    const double b0 = G[0] * G[6] + G[1] * G[7], b1 = G[3] * G[6] + G[4] * G[7];
    const double d = cross_z(e, b0, b1);
    if (n * d > 0.0) return false;
  }
  return true;
}

__device__ __forceinline__ void load7(const double4* P, const int* s, double2* a, double2* b) {
  for (int i = 0; i < 7; ++i) {
    const double4 q = P[s[i]];
    a[i] = make_double2(q.x, q.y);
    b[i] = make_double2(q.z, q.w);
  }
}

// kept candidates of a trial: F3 holds the 7-point slots, returns the count and the kept slots
__device__ int kept_candidates(const double4* P, const int* s, double* F3, int* slots) {
  double2 a[7], b[7];
  load7(P, s, a, b);
  const int nreal = seven_point(a, b, F3);
  int nk = 0;
  for (int k = 0; k < 3; ++k)
    if (k < nreal && real_focal(F3 + 9 * k)) slots[nk++] = k;
  return nk;
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

__device__ int dynamic_max_iter(int cnt, int n, int min_iterations, int max_iterations) {
  const double ratio = (double)cnt / (double)n;
  if (ratio >= 0.9999) return min_iterations;
  if (ratio <= 0.0001) return max_iterations;
  const double p = 1.0 - pow(ratio, 7.0);
  const double v = log(1.0 - MS_SUCCESS_PROB) / log(p);
  if (!(v < (double)max_iterations)) return max_iterations;
  return (int)ceil(v);
}

// -------------------------------------------------------------------------------------------------------------------
// 1. compaction and scale
// -------------------------------------------------------------------------------------------------------------------
template <typename TP>
__global__ void __launch_bounds__(256) ms_compact_kernel(int N, const TP* __restrict__ p1, const TP* __restrict__ p2,
                                                         const uint8_t* __restrict__ valid, double max_error,
                                                         unsigned long long seed, int max_iterations, MsWork w) {
  __shared__ int wsum[8];
  __shared__ int base_s;
  __shared__ double red[8 * 3];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const TP* P1 = p1 + (size_t)b * N * 2;
  const TP* P2 = p2 + (size_t)b * N * 2;
  double4* pts = w.pts + (size_t)b * N;
  int* idx = w.idx + (size_t)b * N;
  if (tid == 0) base_s = 0;
  double acc[3] = {0.0, 0.0, 0.0};   // sum of norms over finite matches, their count
  for (int t0 = 0; t0 < N; t0 += 256) {
    const int i = t0 + tid;
    const bool v = i < N && (valid == nullptr || valid[(size_t)b * N + i]);
    const unsigned bal = __ballot_sync(0xffffffffu, v);
    __syncthreads();
    if (lane == 0) wsum[warp] = __popc(bal);
    __syncthreads();
    int off = base_s;
    for (int q = 0; q < warp; ++q) off += wsum[q];
    off += __popc(bal & ((1u << lane) - 1u));
    if (v) {
      const double2 a = ldp(P1, i), c = ldp(P2, i);
      pts[off] = make_double4(a.x, a.y, c.x, c.y);
      idx[off] = i;
      if (isfinite(a.x) && isfinite(a.y) && isfinite(c.x) && isfinite(c.y)) {
        acc[0] += __dsqrt_rn(__dadd_rn(__dmul_rn(a.x, a.x), __dmul_rn(a.y, a.y)));
        acc[1] += __dsqrt_rn(__dadd_rn(__dmul_rn(c.x, c.x), __dmul_rn(c.y, c.y)));
        acc[2] += 1.0;
      }
    }
    __syncthreads();
    if (tid == 0)
      for (int q = 0; q < 8; ++q) base_s += wsum[q];
  }
  block_sums<256, 3>(acc, red);
  __syncthreads();
  const int n = base_s;
  double s = acc[2] > 0.0 ? (acc[0] + acc[1]) / (2.0 * acc[2]) / sqrt(2.0) : 1.0;
  if (!(isfinite(s) && s > 0.0)) s = 1.0;
  for (int i = tid; i < n; i += 256) {
    const double4 q = pts[i];
    pts[i] = make_double4(q.x / s, q.y / s, q.z / s, q.w / s);
  }
  if (tid == 0) {
    w.nval[b] = n;
    w.scale[b] = s;
    w.rng[b] = seed;
    PairState& st = w.st[b];
    st.best_min_score = DBL_MAX;
    st.model_score = DBL_MAX;
    st.best_min_cnt = 0;
    st.model_cnt = 0;
    st.dyn = max_iterations;
    st.stopped = n < 7;
    st.iterations = 0;
    st.src_kind = 0;
    st.src_trial = -1;
    st.src_slot = -1;
    st.lo_runs = 0;
    for (int k = 0; k < 9; ++k) st.F[k] = 0.0;
  }
}

// -------------------------------------------------------------------------------------------------------------------
// 2. sampler: PoseLib's RandomSampler (LCG mod 2^31, duplicates redrawn)
// -------------------------------------------------------------------------------------------------------------------
__global__ void ms_sample_kernel(int B, int C, int nt, MsWork w) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B || w.st[b].stopped) return;
  const unsigned long long n = (unsigned long long)w.nval[b];
  unsigned long long s = w.rng[b];
  int* out = w.samples + (size_t)b * C * 7;
  for (int t = 0; t < nt; ++t) {
    int smp[7];
    for (int i = 0; i < 7; ++i) {
      bool dup = true;
      while (dup) {
        s = (s * 1103515245ull + 12345ull) & 0x7fffffffull;
        smp[i] = (int)(s % n);
        dup = false;
        for (int j = 0; j < i; ++j) dup |= smp[j] == smp[i];
      }
      out[t * 7 + i] = smp[i];
    }
  }
  w.rng[b] = s;
}

// -------------------------------------------------------------------------------------------------------------------
// 3. minimal solves + MSAC scores
// -------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(MS_TRIALS) ms_minimal_kernel(int N, int C, int nt, double max_error, MsWork w) {
  __shared__ double4 tile[MS_TILE];
  const int b = blockIdx.y, tid = threadIdx.x;
  if (w.st[b].stopped) return;
  const int t = blockIdx.x * MS_TRIALS + tid;
  const bool active = t < nt;
  const int n = w.nval[b];
  const double thr = max_error / w.scale[b], thr2 = thr * thr, pre = 2.0 * thr2;
  const double4* P = w.pts + (size_t)b * N;
  double F3[27], F[27];
  int slots[3] = {0, 0, 0}, nk = 0;
  if (active) nk = kept_candidates(P, w.samples + ((size_t)b * C + t) * 7, F3, slots);
  for (int k = 0; k < 3; ++k)
    for (int i = 0; i < 9; ++i) F[9 * k + i] = k < nk ? F3[9 * slots[k] + i] : 0.0;
  int cnt[3] = {0, 0, 0};
  double sc[3] = {0.0, 0.0, 0.0};
  for (int base = 0; base < n; base += MS_TILE) {
    const int m = min(MS_TILE, n - base);
    __syncthreads();
    for (int i = tid; i < m; i += MS_TRIALS) tile[i] = P[base + i];
    __syncthreads();
    for (int j = 0; j < m; ++j) {
      const double4 q = tile[j];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double* G = F + 9 * k;
        const double l0 = __fma_rn(G[0], q.x, __fma_rn(G[1], q.y, G[2]));
        const double l1 = __fma_rn(G[3], q.x, __fma_rn(G[4], q.y, G[5]));
        const double l2 = __fma_rn(G[6], q.x, __fma_rn(G[7], q.y, G[8]));
        const double m0 = __fma_rn(G[0], q.z, __fma_rn(G[3], q.w, G[6]));
        const double m1 = __fma_rn(G[1], q.z, __fma_rn(G[4], q.w, G[7]));
        const double e = __fma_rn(q.z, l0, __fma_rn(q.w, l1, l2));
        const double num = __dmul_rn(e, e);
        const double den = __fma_rn(l0, l0, __fma_rn(l1, l1, __fma_rn(m0, m0, __dmul_rn(m1, m1))));
        double add = thr2;
        if (num <= pre * den) {          // only here can r^2 fall below thr^2
          const double r2 = __ddiv_rn(num, den);
          if (r2 < thr2) { cnt[k] += 1; add = r2; }
        }
        sc[k] += add;
      }
    }
  }
  if (active) {
    const size_t o = (size_t)b * C + t;
    w.cand[o] = nk | (slots[0] << 4) | (slots[1] << 8) | (slots[2] << 12);
    for (int k = 0; k < 3; ++k) {
      w.mcnt[o * 3 + k] = cnt[k];
      w.msc[o * 3 + k] = sc[k];
    }
  }
}

// -------------------------------------------------------------------------------------------------------------------
// 4. triggers: which trials run LO, from which seed, and which candidates improve the running minimal bests
// -------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32) ms_trigger_kernel(int C, int nt, MsWork w) {
  const int b = blockIdx.x, lane = threadIdx.x;
  PairState& st = w.st[b];
  if (st.stopped) return;
  int run_c = st.best_min_cnt;
  double run_s = st.best_min_score;
  int ntr = 0;
  for (int base = 0; base < nt; base += 32) {
    const int t = base + lane;
    const size_t o = (size_t)b * C + t;
    int nk = 0, cw = 0, c[3] = {0, 0, 0};
    double s[3] = {0.0, 0.0, 0.0};
    if (t < nt) {
      cw = w.cand[o];
      nk = cw & 15;
      for (int k = 0; k < nk; ++k) { c[k] = w.mcnt[o * 3 + k]; s[k] = w.msc[o * 3 + k]; }
    }
    int lc = -1;
    double ls = DBL_MAX;
    for (int k = 0; k < nk; ++k) { lc = max(lc, c[k]); ls = fmin(ls, s[k]); }
    // inclusive warp scans, then exclusive
    int ic = lc;
    double is = ls;
    for (int d = 1; d < 32; d <<= 1) {
      const int oc = __shfl_up_sync(0xffffffffu, ic, d);
      const double os = __shfl_up_sync(0xffffffffu, is, d);
      if (lane >= d) { ic = max(ic, oc); is = fmin(is, os); }
    }
    int ec = __shfl_up_sync(0xffffffffu, ic, 1);
    double es = __shfl_up_sync(0xffffffffu, is, 1);
    if (lane == 0) { ec = -1; es = DBL_MAX; }
    int cur_c = max(run_c, ec);
    double cur_s = fmin(run_s, es);
    Trig tr;
    tr.trial = t;
    tr.seed = -1;
    tr.nimp = 0;
    for (int k = 0; k < nk; ++k) {
      const bool more = c[k] > cur_c, better = s[k] < cur_s;
      if (more) cur_c = c[k];
      if (better) cur_s = s[k];
      if (more || better) {
        const int slot = (cw >> (4 + 4 * k)) & 15;
        tr.icnt[tr.nimp] = c[k];
        tr.isc[tr.nimp] = s[k];
        tr.islot[tr.nimp] = slot;
        tr.nimp++;
        tr.seed = slot;
      }
    }
    const unsigned bal = __ballot_sync(0xffffffffu, tr.seed >= 0);
    if (tr.seed >= 0) w.trig[(size_t)b * C + ntr + __popc(bal & ((1u << lane) - 1u))] = tr;
    ntr += __popc(bal);
    run_c = max(run_c, __shfl_sync(0xffffffffu, ic, 31));
    run_s = fmin(run_s, __shfl_sync(0xffffffffu, is, 31));
  }
  if (lane == 0) {
    st.best_min_cnt = run_c;
    st.best_min_score = run_s;
    w.ntrig[b] = ntr;
    atomicMax(&w.ctr[0], ntr);
  }
}

// -------------------------------------------------------------------------------------------------------------------
// LM on the factorised F (one CTA): truncated loss over all matches, or Cauchy over the flagged subset
// -------------------------------------------------------------------------------------------------------------------
struct LmShared {
  double F[9], A[9], Bm[9], G[63];
  double red[MS_LO_THREADS / 32 * 36];
  double sig;
  int go;
};

__device__ void mat3_mul(const double* a, const double* b, double* o) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) o[r * 3 + c] = a[r * 3] * b[c] + a[r * 3 + 1] * b[3 + c] + a[r * 3 + 2] * b[6 + c];
}

__device__ void rodrigues(const double* v, double* R) {
  const double t2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
  for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
  if (t2 == 0.0) return;
  const double t = sqrt(t2), a = sin(t) / t, h = sin(0.5 * t), c = 2.0 * h * h / t2;
  const double K[9] = {0.0, -v[2], v[1], v[2], 0.0, -v[0], -v[1], v[0], 0.0};
  double K2[9];
  mat3_mul(K, K, K2);
  for (int i = 0; i < 9; ++i) R[i] += a * K[i] + c * K2[i];
}

// derivative basis at F = A + sig Bm: [e_k]x F, -F [e_k]x, Bm
__device__ void deriv_basis(const double* F, const double* Bm, double* G) {
  for (int k = 0; k < 3; ++k) {
    double* Gw = G + 9 * k;
    double* Gv = G + 9 * (3 + k);
    for (int j = 0; j < 3; ++j) {           // columns of [e_k]x F: e_k x F[:, j]
      const double c[3] = {F[j], F[3 + j], F[6 + j]};
      const double x[3] = {k == 0 ? 0.0 : (k == 1 ? c[2] : -c[1]), k == 0 ? -c[2] : (k == 1 ? 0.0 : c[0]),
                           k == 0 ? c[1] : (k == 1 ? -c[0] : 0.0)};
      for (int i = 0; i < 3; ++i) Gw[i * 3 + j] = x[i];
    }
    for (int i = 0; i < 3; ++i) {           // rows of -F [e_k]x: e_k x F[i, :]
      const double r[3] = {F[i * 3], F[i * 3 + 1], F[i * 3 + 2]};
      Gv[i * 3 + 0] = k == 0 ? 0.0 : (k == 1 ? r[2] : -r[1]);
      Gv[i * 3 + 1] = k == 0 ? -r[2] : (k == 1 ? 0.0 : r[0]);
      Gv[i * 3 + 2] = k == 0 ? r[1] : (k == 1 ? -r[0] : 0.0);
    }
  }
  for (int i = 0; i < 9; ++i) G[54 + i] = Bm[i];
}

// one pass at sh.F / sh.G: v[0..27] lower JtJ, v[28..34] Jtr, v[35] cost (every thread gets the sums)
__device__ void lm_pass(const double4* P, int n, const uint8_t* sub, bool cauchy, double c2, LmShared& sh,
                        double (&v)[36]) {
  for (int q = 0; q < 36; ++q) v[q] = 0.0;
  for (int i = threadIdx.x; i < n; i += MS_LO_THREADS) {
    if (sub && !sub[i]) continue;
    const double4 q = P[i];
    double e, den;
    const double r2 = sq_sampson(sh.F, q, e, den);
    double wgt;
    if (cauchy) {
      wgt = 1.0 / (1.0 + r2 / c2);
      v[35] += c2 * log1p(r2 / c2);
    } else {
      const bool in = r2 < c2;
      wgt = in ? 1.0 : 0.0;
      v[35] += in ? r2 : c2;
    }
    if (!(wgt > 0.0)) continue;
    const double* F = sh.F;
    const double l0 = F[0] * q.x + F[1] * q.y + F[2], l1 = F[3] * q.x + F[4] * q.y + F[5];
    const double m0 = F[0] * q.z + F[3] * q.w + F[6], m1 = F[1] * q.z + F[4] * q.w + F[7];
    const double sq = sqrt(den), r = e / sq, kk = e / den;
    const double x1[3] = {q.x, q.y, 1.0}, x2[3] = {q.z, q.w, 1.0}, l[2] = {l0, l1}, m[2] = {m0, m1};
    double dF[9];
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        double t = (a < 2 ? l[a] * x1[c] : 0.0) + (c < 2 ? m[c] * x2[a] : 0.0);
        dF[a * 3 + c] = (x2[a] * x1[c] - kk * t) / sq;
      }
    double J[7];
#pragma unroll
    for (int p = 0; p < 7; ++p) {
      double s = 0.0;
#pragma unroll
      for (int k = 0; k < 9; ++k) s += dF[k] * sh.G[p * 9 + k];
      J[p] = s;
    }
    int o = 0;
#pragma unroll
    for (int p = 0; p < 7; ++p) {
#pragma unroll
      for (int s2 = 0; s2 <= p; ++s2) v[o++] += wgt * J[p] * J[s2];
      v[28 + p] += wgt * r * J[p];
    }
  }
  block_sums<MS_LO_THREADS, 36>(v, sh.red);
}

// refines sh.F in place (whole CTA); sh.F must be set and visible on entry
__device__ void lm_refine(const double4* P, int n, const uint8_t* sub, bool cauchy, double c2, int iters,
                          LmShared& sh) {
  if (threadIdx.x == 0) {
    // factorisation: V from the eigenvectors of F^T F, u_i = F v_i / s_i
    double M[9], V[9], ev[3];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c)
        M[r * 3 + c] = sh.F[r] * sh.F[c] + sh.F[3 + r] * sh.F[3 + c] + sh.F[6 + r] * sh.F[6 + c];
    jacobi_eig<3>(M, V, ev);
    int o[3] = {0, 1, 2};
    for (int i = 0; i < 3; ++i)
      for (int k = i + 1; k < 3; ++k)
        if (ev[o[k]] > ev[o[i]]) { const int t = o[i]; o[i] = o[k]; o[k] = t; }
    double u[2][3], s[2];
    for (int q = 0; q < 2; ++q) {
      const double* vv = V;
      double nn = 0.0;
      for (int r = 0; r < 3; ++r) {
        u[q][r] = sh.F[r * 3] * vv[o[q]] + sh.F[r * 3 + 1] * vv[3 + o[q]] + sh.F[r * 3 + 2] * vv[6 + o[q]];
        nn += u[q][r] * u[q][r];
      }
      s[q] = sqrt(nn);
    }
    sh.go = s[1] > 0.0 && isfinite(s[0]) && isfinite(s[1]);
    if (sh.go) {
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) {
          sh.A[r * 3 + c] = u[0][r] / s[0] * V[c * 3 + o[0]];
          sh.Bm[r * 3 + c] = u[1][r] / s[1] * V[c * 3 + o[1]];
        }
      sh.sig = s[1] / s[0];
      for (int i = 0; i < 9; ++i) sh.F[i] = sh.A[i] + sh.sig * sh.Bm[i];
      deriv_basis(sh.F, sh.Bm, sh.G);
    }
  }
  __syncthreads();
  if (!sh.go) return;
  double v[36];
  lm_pass(P, n, sub, cauchy, c2, sh, v);
  // thread 0 keeps the accepted state
  double JtJ[28], Jtr[7], cost = v[35], lam = MS_LAMBDA0;
  double A[9], Bm[9], sig = sh.sig;
  for (int q = 0; q < 28; ++q) JtJ[q] = v[q];
  for (int q = 0; q < 7; ++q) Jtr[q] = v[28 + q];
  for (int i = 0; i < 9; ++i) { A[i] = sh.A[i]; Bm[i] = sh.Bm[i]; }
  for (int it = 0; it < iters; ++it) {
    __syncthreads();
    if (threadIdx.x == 0) {
      sh.go = 0;
      double g = 0.0;
      for (int q = 0; q < 7; ++q) g += Jtr[q] * Jtr[q];
      if (sqrt(g) >= MS_GRAD_TOL) {
        // Cholesky of JtJ + lam I (lower, packed row-wise like JtJ)
        double L[7][7], sol[7];
        bool ok = true;
        for (int i = 0; i < 7 && ok; ++i)
          for (int j = 0; j <= i; ++j) {
            double a = JtJ[i * (i + 1) / 2 + j] + (i == j ? lam : 0.0);
            for (int k = 0; k < j; ++k) a -= L[i][k] * L[j][k];
            if (i == j) {
              if (!(a > 0.0)) { ok = false; break; }
              L[i][i] = sqrt(a);
            } else {
              L[i][j] = a / L[j][j];
            }
          }
        if (ok) {
          double y[7];
          for (int i = 0; i < 7; ++i) {
            double a = Jtr[i];
            for (int k = 0; k < i; ++k) a -= L[i][k] * y[k];
            y[i] = a / L[i][i];
          }
          for (int i = 6; i >= 0; --i) {
            double a = y[i];
            for (int k = i + 1; k < 7; ++k) a -= L[k][i] * sol[k];
            sol[i] = a / L[i][i];
          }
          double st = 0.0;
          for (int i = 0; i < 7; ++i) { sol[i] = -sol[i]; st += sol[i] * sol[i]; }
          if (sqrt(st) >= MS_STEP_TOL) {
            double Rw[9], Rv[9], T1[9];
            rodrigues(sol, Rw);
            rodrigues(sol + 3, Rv);
            double RvT[9];
            for (int r = 0; r < 3; ++r)
              for (int c = 0; c < 3; ++c) RvT[r * 3 + c] = Rv[c * 3 + r];
            mat3_mul(Rw, A, T1);
            mat3_mul(T1, RvT, sh.A);
            mat3_mul(Rw, Bm, T1);
            mat3_mul(T1, RvT, sh.Bm);
            sh.sig = sig + sol[6];
            for (int i = 0; i < 9; ++i) sh.F[i] = sh.A[i] + sh.sig * sh.Bm[i];
            deriv_basis(sh.F, sh.Bm, sh.G);
            sh.go = 1;
          }
        }
      }
    }
    __syncthreads();
    if (!sh.go) break;
    lm_pass(P, n, sub, cauchy, c2, sh, v);
    if (threadIdx.x == 0) {
      if (v[35] < cost) {
        cost = v[35];
        for (int q = 0; q < 28; ++q) JtJ[q] = v[q];
        for (int q = 0; q < 7; ++q) Jtr[q] = v[28 + q];
        for (int i = 0; i < 9; ++i) { A[i] = sh.A[i]; Bm[i] = sh.Bm[i]; }
        sig = sh.sig;
        lam = fmax(MS_MIN_LAMBDA, lam / 10.0);
      } else {
        lam = fmin(MS_MAX_LAMBDA, lam * 10.0);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int i = 0; i < 9; ++i) sh.F[i] = A[i] + sig * Bm[i];
  __syncthreads();
}

// MSAC count and score of sh.F over all matches (every thread gets them)
__device__ void msac_score(const double4* P, int n, double thr2, LmShared& sh, int& cnt, double& score) {
  double v[2] = {0.0, 0.0};
  for (int i = threadIdx.x; i < n; i += MS_LO_THREADS) {
    double e, den;
    const double r2 = sq_sampson(sh.F, P[i], e, den);
    if (r2 < thr2) { v[0] += 1.0; v[1] += r2; } else { v[1] += thr2; }
  }
  block_sums<MS_LO_THREADS, 2>(v, sh.red);
  cnt = (int)(v[0] + 0.5);
  score = v[1];
}

// -------------------------------------------------------------------------------------------------------------------
// 5. LO of the chunk's triggers
// -------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(MS_LO_THREADS) ms_lo_kernel(int N, int C, double max_error, MsWork w) {
  __shared__ LmShared sh;
  const int j = blockIdx.x, b = blockIdx.y;
  if (w.st[b].stopped || j >= w.ntrig[b]) return;
  const Trig& tr = w.trig[(size_t)b * C + j];
  const double4* P = w.pts + (size_t)b * N;
  const int n = w.nval[b];
  const double thr = max_error / w.scale[b], thr2 = thr * thr;
  if (threadIdx.x == 0) {
    double2 a[7], c[7];
    double F3[27];
    load7(P, w.samples + ((size_t)b * C + tr.trial) * 7, a, c);
    seven_point(a, c, F3);
    for (int i = 0; i < 9; ++i) sh.F[i] = F3[9 * tr.seed + i];
  }
  __syncthreads();
  lm_refine(P, n, nullptr, false, thr2, MS_LO_ITERS, sh);
  int cnt;
  double score;
  msac_score(P, n, thr2, sh, cnt, score);
  if (threadIdx.x == 0) {
    const size_t o = (size_t)b * C + j;
    for (int i = 0; i < 9; ++i) w.loF[o * 9 + i] = sh.F[i];
    w.locnt[o] = cnt;
    w.losc[o] = score;
  }
}

// -------------------------------------------------------------------------------------------------------------------
// 6. bookkeeping in trial order, stop
// -------------------------------------------------------------------------------------------------------------------
__global__ void ms_resolve_kernel(int B, int N, int C, int it0, int nt, int max_iterations, int min_iterations, MsWork w) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  PairState& st = w.st[b];
  if (st.stopped) return;
  const int n = w.nval[b], ntr = w.ntrig[b];
  int pos = it0, dyn = st.dyn, stop = -1;
  int kind = 0, trial = -1, slot = -1, lo_j = -1;   // source of the best model, if it changed in this chunk
  double ms = st.model_score;
  int mc = st.model_cnt;
  for (int j = 0; j < ntr; ++j) {
    const Trig& tr = w.trig[(size_t)b * C + j];
    const int T = it0 + tr.trial;
    const int at = max(pos, max(min_iterations, dyn) + 1);
    if (at <= T) { stop = at; break; }
    for (int k = 0; k < tr.nimp; ++k)
      if (tr.isc[k] < ms) { ms = tr.isc[k]; mc = tr.icnt[k]; kind = 1; trial = tr.trial; slot = tr.islot[k]; }
    const size_t o = (size_t)b * C + j;
    if (w.losc[o] < ms) { ms = w.losc[o]; mc = w.locnt[o]; kind = 2; trial = tr.trial; lo_j = j; }
    dyn = dynamic_max_iter(mc, n, min_iterations, max_iterations);
    if (st.lo_runs < MS_TRACE_CAP) w.trace[(size_t)b * MS_TRACE_CAP + st.lo_runs] = T;
    st.lo_runs++;
    pos = T + 1;
  }
  if (stop < 0) {
    const int at = max(pos, max(min_iterations, dyn) + 1);
    if (at <= it0 + nt) stop = at;
    else if (it0 + nt >= max_iterations) stop = max_iterations;
  }
  if (kind != 0) {
    st.src_kind = kind;
    st.src_trial = it0 + trial;
    st.src_slot = slot;
    if (kind == 2) {
      for (int i = 0; i < 9; ++i) st.F[i] = w.loF[((size_t)b * C + lo_j) * 9 + i];
    } else {                          // a minimal candidate: recompute it from the trial's sample
      double2 a[7], c[7];
      double F3[27];
      load7(w.pts + (size_t)b * N, w.samples + ((size_t)b * C + trial) * 7, a, c);
      seven_point(a, c, F3);
      for (int i = 0; i < 9; ++i) st.F[i] = F3[9 * slot + i];
    }
  }
  st.model_score = ms;
  st.model_cnt = mc;
  st.dyn = dyn;
  if (stop >= 0) {
    st.stopped = 1;
    st.iterations = stop;
  } else {
    atomicAdd(&w.ctr[1], 1);
  }
}

// -------------------------------------------------------------------------------------------------------------------
// 7. final LO, mask, polish, denormalisation
// -------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(MS_LO_THREADS) ms_final_kernel(int N, double max_error, MsWork w,
                                                                 double* __restrict__ fmat_out,
                                                                 int* __restrict__ num_out,
                                                                 uint8_t* __restrict__ mask_out,
                                                                 int* __restrict__ iter_out) {
  __shared__ LmShared sh;
  __shared__ double Fm[9];
  const int b = blockIdx.x, tid = threadIdx.x;
  const PairState& st = w.st[b];
  const int n = w.nval[b];
  if (n < 7 || st.src_kind == 0) {
    if (tid < 9) fmat_out[(size_t)b * 9 + tid] = 0.0;
    if (tid == 0) { num_out[b] = 0; iter_out[b] = n < 7 ? 0 : st.iterations; }
    return;
  }
  const double4* P = w.pts + (size_t)b * N;
  const double s = w.scale[b], thr = max_error / s, thr2 = thr * thr;
  if (tid < 9) { sh.F[tid] = st.F[tid]; Fm[tid] = st.F[tid]; }
  __syncthreads();
  lm_refine(P, n, nullptr, false, thr2, MS_LO_ITERS, sh);
  int cnt;
  double score;
  msac_score(P, n, thr2, sh, cnt, score);
  if (tid < 9 && score < st.model_score) Fm[tid] = sh.F[tid];
  __syncthreads();
  if (tid < 9) sh.F[tid] = Fm[tid];
  __syncthreads();
  uint8_t* inl = w.inl + (size_t)b * N;
  double c[1] = {0.0};
  for (int i = tid; i < n; i += MS_LO_THREADS) {
    double e, den;
    const bool in = sq_sampson(sh.F, P[i], e, den) < thr2;
    inl[i] = in;
    if (in) { mask_out[(size_t)b * N + w.idx[(size_t)b * N + i]] = 1; c[0] += 1.0; }
  }
  block_sums<MS_LO_THREADS, 1>(c, sh.red);
  const int num = (int)(c[0] + 0.5);
  __syncthreads();
  if (num > 7) lm_refine(P, n, inl, true, 1.0 / (s * s), MS_POLISH_ITERS, sh);
  if (tid == 0) {
    const double t[3] = {1.0 / s, 1.0 / s, 1.0};
    double G[9], nn = 0.0;
    for (int r = 0; r < 3; ++r)
      for (int q = 0; q < 3; ++q) { G[r * 3 + q] = sh.F[r * 3 + q] * t[r] * t[q]; nn += G[r * 3 + q] * G[r * 3 + q]; }
    nn = sqrt(nn);
    int im = 0;
    for (int i = 0; i < 9; ++i) {
      G[i] /= nn;
      if (fabs(G[i]) > fabs(G[im])) im = i;
    }
    const double sg = G[im] < 0.0 ? -1.0 : 1.0;
    for (int i = 0; i < 9; ++i) fmat_out[(size_t)b * 9 + i] = sg * G[i];
    num_out[b] = num;
    iter_out[b] = st.iterations;
  }
}

template <typename TP>
int run_msac(int B, int N, const TP* p1, const TP* p2, const uint8_t* valid, double max_error, int max_iterations,
             int min_iterations, unsigned long long seed, double* fmat, int* num, uint8_t* mask, int* iters,
             const MsWork& w, int C, cudaStream_t st) {
  VGG_CUDA_CHECK(cudaMemsetAsync(mask, 0, (size_t)B * N, st));
  ms_compact_kernel<TP><<<B, 256, 0, st>>>(N, p1, p2, valid, max_error, seed, max_iterations, w);
  VGG_LAUNCH_CHECK();
  int h[2];
  for (int it0 = 0; it0 < max_iterations;) {
    const int nt = std::min(C, max_iterations - it0);
    VGG_CUDA_CHECK(cudaMemsetAsync(w.ctr, 0, 2 * sizeof(int), st));
    ms_sample_kernel<<<(B + 127) / 128, 128, 0, st>>>(B, C, nt, w);
    VGG_LAUNCH_CHECK();
    ms_minimal_kernel<<<dim3((nt + MS_TRIALS - 1) / MS_TRIALS, B), MS_TRIALS, 0, st>>>(N, C, nt, max_error, w);
    VGG_LAUNCH_CHECK();
    ms_trigger_kernel<<<B, 32, 0, st>>>(C, nt, w);
    VGG_LAUNCH_CHECK();
    VGG_CUDA_CHECK(cudaMemcpyAsync(h, w.ctr, sizeof(int), cudaMemcpyDeviceToHost, st));
    VGG_CUDA_CHECK(cudaStreamSynchronize(st));
    if (h[0] > 0) {
      ms_lo_kernel<<<dim3(h[0], B), MS_LO_THREADS, 0, st>>>(N, C, max_error, w);
      VGG_LAUNCH_CHECK();
    }
    ms_resolve_kernel<<<(B + 127) / 128, 128, 0, st>>>(B, N, C, it0, nt, max_iterations, min_iterations, w);
    VGG_LAUNCH_CHECK();
    VGG_CUDA_CHECK(cudaMemcpyAsync(h + 1, w.ctr + 1, sizeof(int), cudaMemcpyDeviceToHost, st));
    VGG_CUDA_CHECK(cudaStreamSynchronize(st));
    it0 += nt;
    if (h[1] == 0) break;
  }
  ms_final_kernel<<<B, MS_LO_THREADS, 0, st>>>(N, max_error, w, fmat, num, mask, iters);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

}  // namespace

}  // namespace vgg

using namespace vgg;

extern "C" {

int vgg_msac_fundamental_workspace_bytes(int B, int N, int max_iterations, int min_iterations, size_t* bytes) {
  VGG_REQUIRE(B >= 0 && N >= 0 && max_iterations >= 1 && min_iterations >= 0 && bytes, "bad arguments");
  VGG_REQUIRE((long long)B * N < (1ll << 31), "estimate_fundamental_msac: B * N must stay below 2^31");
  carve_ms(nullptr, 0, B, N, chunk_of(max_iterations, min_iterations), bytes);
  return VGG_OK;
}

int vgg_estimate_fundamental_msac(int B, int N, const void* points1, const void* points2, int points_are_f64,
                                  const uint8_t* valid_mask, double max_error, int max_iterations, int min_iterations,
                                  unsigned long long seed, double* fmat_out, int32_t* inlier_num_out,
                                  uint8_t* inlier_mask_out, int32_t* iterations_out, void* workspace, size_t ws_bytes,
                                  void* stream) {
  VGG_REQUIRE(B >= 0 && N >= 0, "estimate_fundamental_msac: negative size");
  VGG_REQUIRE((long long)B * N < (1ll << 31), "estimate_fundamental_msac: B * N must stay below 2^31");
  VGG_REQUIRE(max_iterations >= 1 && min_iterations >= 0, "estimate_fundamental_msac: bad iteration limits");
  VGG_REQUIRE(max_error > 0.0 && isfinite(max_error), "estimate_fundamental_msac: max_error must be positive");
  g_launch_count = 0;
  if (B == 0) return VGG_OK;
  VGG_REQUIRE(points1 && points2 && fmat_out && inlier_num_out && inlier_mask_out && iterations_out && workspace,
              "null pointer");
  const int C = chunk_of(max_iterations, min_iterations);
  size_t need = 0;
  carve_ms(nullptr, 0, B, N, C, &need);
  if (ws_bytes < need) {
    set_error("msac workspace too small: need %zu bytes", need);
    return VGG_EWORKSPACE;
  }
  MsWork w = carve_ms(workspace, ws_bytes, B, N, C, nullptr);
  cudaStream_t st = (cudaStream_t)stream;
  if (points_are_f64)
    return run_msac(B, N, (const double*)points1, (const double*)points2, valid_mask, max_error, max_iterations,
                    min_iterations, seed, fmat_out, inlier_num_out, inlier_mask_out, iterations_out, w, C, st);
  return run_msac(B, N, (const float*)points1, (const float*)points2, valid_mask, max_error, max_iterations,
                  min_iterations, seed, fmat_out, inlier_num_out, inlier_mask_out, iterations_out, w, C, st);
}

int vgg_dev_msac_trace(int B, int N, int max_iterations, int min_iterations, const void* workspace, int cap,
                       int32_t* lo_runs_host, int32_t* win_trial_host, int32_t* lo_trials_host) {
  VGG_REQUIRE(B >= 0 && N >= 0 && max_iterations >= 1 && min_iterations >= 0 && workspace && cap >= 0, "bad arguments");
  const int C = chunk_of(max_iterations, min_iterations);
  MsWork w = carve_ms(const_cast<void*>(workspace), ~(size_t)0, B, N, C, nullptr);
  VGG_CUDA_CHECK(cudaDeviceSynchronize());
  for (int b = 0; b < B; ++b) {
    PairState s;
    VGG_CUDA_CHECK(cudaMemcpy(&s, w.st + b, sizeof(PairState), cudaMemcpyDeviceToHost));
    lo_runs_host[b] = s.lo_runs;
    win_trial_host[b] = s.src_kind == 0 ? -1 : s.src_trial;
    const int m = std::min(std::min(s.lo_runs, MS_TRACE_CAP), cap);
    for (int k = 0; k < cap; ++k) lo_trials_host[(size_t)b * cap + k] = -1;
    if (m > 0)
      VGG_CUDA_CHECK(cudaMemcpy(lo_trials_host + (size_t)b * cap, w.trace + (size_t)b * MS_TRACE_CAP, m * sizeof(int),
                                cudaMemcpyDeviceToHost));
  }
  return VGG_OK;
}

}  // extern "C"
