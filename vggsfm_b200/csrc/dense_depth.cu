// Dense depth stage: align_dense_depth_maps (vggsfm/utils/utils.py:635-770) as batched kernels over every frame of a
// call, restated in oracle/dense_depth_oracle.py (which the header there lists rule by rule).
//
//   dd_samples_kernel   one thread per sparse observation: half-to-even pixel rounding, bounds, nearest-pixel lookup of
//                       the monocular disparity, the depth clip and the target disparity 1/depth (utils.py:669-690).
//   dd_median_kernel    one CTA per frame: np.median of the targets by two 8-bit radix selects over the bit patterns.
//   per chunk of trials (the host draws the samples; see DESIGN §3 for the random-number pin):
//   dd_trial_kernel     one CTA per (frame, trial): sklearn's float32 two-point LinearRegression fit, the inlier count
//                       and the R^2 of the inlier subset.  Nothing of size frames x trials x points is stored.
//   dd_resolve_kernel   one thread per live frame: RANSACRegressor.fit's bookkeeping over the chunk in trial order and
//                       the dynamic stop (sklearn/linear_model/_ransac.py).
//   dd_final_kernel     one CTA per frame: the winner's inlier mask and the OLS fit with intercept on it.
//   dd_apply_kernel     one HBM pass over the disparity maps: rescale in place, clip, depth = 1/disp, valid counts per
//                       tile for the unprojection's compaction.
//   dd_unproject_kernel one pass over the depth maps: valid pixels in row-major order through cam_from_img, times
//                       depth, through the inverse pose, with their colour / 255.
#include <float.h>
#include <math.h>
#include "common.cuh"

namespace vgg {

namespace {

constexpr int DD_THREADS = 256;
constexpr int DD_TILE = 2048;              // pixels per CTA of the apply / unproject kernels (8 per thread)
constexpr int DD_MAX_CHUNK = 4096;         // trials per chunk at most

struct DdState {
  double max_trials;                       // min(max_trials, _dynamic_max_trials(...)); may be +inf
  double score_best;
  int n_trials, n_best, has_best, pad;
  float c, b;                              // the best trial's float32 model
};

struct DdTrial {
  double score;
  float c, b;
  int n, pad;
};

// LinearRegression().fit on two samples as sklearn runs it for a float32 X: y cast to float32, both centred in float32
// by their float32 means, then LAPACK sgelsd on the 2 x 1 system (Householder QR via slarfg / slapy2, Q^T b, then
// slalsd's scaling by 1/R).  Every operation rounds separately, like the Fortran it restates.
__device__ __forceinline__ void fit_two(float x0, float x1, double y0d, double y1d, float* c_out, float* b_out) {
  const float y0 = (float)y0d, y1 = (float)y1d;
  const float xm = __fmul_rn(__fadd_rn(x0, x1), 0.5f), ym = __fmul_rn(__fadd_rn(y0, y1), 0.5f);
  const float a0 = __fsub_rn(x0, xm), a1 = __fsub_rn(x1, xm);
  const float b0 = __fsub_rn(y0, ym), b1 = __fsub_rn(y1, ym);
  float R = a0, bb = b0;
  if (a1 != 0.f) {
    const float w = fmaxf(fabsf(a0), fabsf(a1)), z = fminf(fabsf(a0), fabsf(a1));
    float nrm = w;
    if (z != 0.f) {
      const float q = __fdiv_rn(z, w);
      nrm = __fmul_rn(w, __fsqrt_rn(__fadd_rn(1.f, __fmul_rn(q, q))));
    }
    const float beta = -copysignf(nrm, a0);
    const float tau = __fdiv_rn(__fsub_rn(beta, a0), beta);
    const float v1 = __fmul_rn(a1, __fdiv_rn(1.f, __fsub_rn(a0, beta)));
    const float wk = __fadd_rn(b0, __fmul_rn(b1, v1));
    bb = __fadd_rn(b0, __fmul_rn(-tau, wk));
    R = beta;
  }
  const float c = (R == 0.f) ? 0.f : __fmul_rn(bb, __fdiv_rn(1.f, R));
  *c_out = c;
  *b_out = __fsub_rn(ym, __fmul_rn(xm, c));
}

// estimator.predict (float32 X @ coef_ + intercept_), then loss "squared_error" against the float64 target
__device__ __forceinline__ double sq_residual(float x, double y, float c, float b) {
  const double d = __dsub_rn(y, (double)__fadd_rn(__fmul_rn(x, c), b));
  return __dmul_rn(d, d);
}

template <typename T>
__device__ T block_sum(T v, T* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[wid] = v;
  __syncthreads();
  T s = 0;
  if (threadIdx.x == 0) {
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += red[i];
    red[0] = s;
  }
  __syncthreads();
  return red[0];
}

// r2_score(y, y_pred) of the inlier subset (force_finite): 1 - SSres / SStot around the subset mean
// (skipped, score -inf, below `need` inliers: such a trial can no longer be kept)
__device__ double inlier_r2(const float* x, const double* y, int n, double th, float c, float b, int need,
                            int* cnt_out) {
  __shared__ double redd[DD_THREADS / 32];
  __shared__ int redi[DD_THREADS / 32];
  int cnt = 0;
  double sy = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    if (sq_residual(x[i], y[i], c, b) <= th) { ++cnt; sy += y[i]; }
  cnt = block_sum(cnt, redi);
  sy = block_sum(sy, redd);
  *cnt_out = cnt;
  if (cnt == 0 || cnt < need) return -INFINITY;
  // no contractions: with two inliers every sum below is order-independent, so the score equals numpy's bitwise
  const double mean = __ddiv_rn(sy, (double)cnt);
  double ssr = 0.0, sst = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const double r2 = sq_residual(x[i], y[i], c, b);
    if (r2 <= th) {
      ssr = __dadd_rn(ssr, r2);
      const double e = __dsub_rn(y[i], mean);
      sst = __dadd_rn(sst, __dmul_rn(e, e));
    }
  }
  ssr = block_sum(ssr, redd);
  sst = block_sum(sst, redd);
  if (sst == 0.0) return ssr == 0.0 ? 1.0 : 0.0;
  return __dsub_rn(1.0, __ddiv_rn(ssr, sst));
}

__global__ void __launch_bounds__(DD_THREADS) dd_samples_kernel(
    int n_total, const int32_t* __restrict__ uvd_frame, const double* __restrict__ uvd, double depth_min,
    double depth_max, const int64_t* __restrict__ map_offsets, const int32_t* __restrict__ map_hw,
    const float* __restrict__ disp, float* __restrict__ x_out, double* __restrict__ y_out, uint8_t* __restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_total) return;
  const int f = uvd_frame[i];
  const int H = map_hw[2 * f], W = map_hw[2 * f + 1];
  const double u = rint(uvd[3 * i]), v = rint(uvd[3 * i + 1]), d = uvd[3 * i + 2];
  float s = 0.f;
  if (u >= 0.0 && u < (double)W && v >= 0.0 && v < (double)H)
    s = disp[map_offsets[f] + (int64_t)v * W + (int64_t)u];
  const double dc = d < depth_min ? depth_min : (d > depth_max ? depth_max : d);   // np.clip keeps NaN
  keep[i] = s > 0.f;
  x_out[i] = s;
  y_out[i] = 1.0 / dc;
}

// k-th smallest of n non-negative doubles: their bit patterns order like the values
__device__ double radix_select(const double* y, int n, int k) {
  __shared__ int hist[256];
  __shared__ int sel_bin, sel_k;
  unsigned long long prefix = 0, mask = 0;
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const unsigned long long bits = (unsigned long long)__double_as_longlong(y[i]);
      if ((bits & mask) == prefix) atomicAdd(&hist[(bits >> shift) & 255], 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int acc = 0, bin = 0;
      for (; bin < 255 && acc + hist[bin] <= k; ++bin) acc += hist[bin];
      sel_bin = bin;
      sel_k = k - acc;
    }
    __syncthreads();
    prefix |= (unsigned long long)sel_bin << shift;
    mask |= 255ull << shift;
    k = sel_k;
    __syncthreads();
  }
  return __longlong_as_double((long long)prefix);
}

__global__ void __launch_bounds__(DD_THREADS) dd_median_kernel(const int32_t* __restrict__ offsets,
                                                               const double* __restrict__ y, double divisor,
                                                               double* __restrict__ med) {
  const int f = blockIdx.x, o = offsets[f], n = offsets[f + 1] - o;
  if (n == 0) { if (threadIdx.x == 0) med[f] = __longlong_as_double(0x7ff8000000000000ll); return; }
  const double lo = radix_select(y + o, n, (n - 1) / 2);
  const double hi = (n & 1) ? lo : radix_select(y + o, n, n / 2);
  // np.median: the mean of the two middle values for an even count; then the caller's divisor (utils.py:695)
  if (threadIdx.x == 0) med[f] = __ddiv_rn((n & 1) ? lo : __ddiv_rn(__dadd_rn(lo, hi), 2.0), divisor);
}

__global__ void dd_init_kernel(int F, double max_trials, DdState* st) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  DdState s;
  s.max_trials = max_trials;
  s.score_best = -INFINITY;
  s.n_trials = 0; s.n_best = 1; s.has_best = 0; s.pad = 0;
  s.c = 0.f; s.b = 0.f;
  st[f] = s;
}

__global__ void __launch_bounds__(DD_THREADS) dd_trial_kernel(
    const int32_t* __restrict__ offsets, const float* __restrict__ x, const double* __restrict__ y,
    const double* __restrict__ thresh, const int32_t* __restrict__ frames, int T, const int32_t* __restrict__ samples,
    const DdState* __restrict__ st, DdTrial* __restrict__ res) {
  const int t = blockIdx.x, r = blockIdx.y, f = frames[r];
  const int o = offsets[f], n = offsets[f + 1] - o;
  const int64_t k = (int64_t)r * T + t;
  const int i0 = samples[2 * k], i1 = samples[2 * k + 1];
  float c, b;
  fit_two(x[o + i0], x[o + i1], y[o + i0], y[o + i1], &c, &b);
  int cnt;
  const double score = inlier_r2(x + o, y + o, n, thresh[f], c, b, st[f].n_best, &cnt);
  if (threadIdx.x == 0) {
    DdTrial tr;
    tr.score = score; tr.c = c; tr.b = b; tr.n = cnt; tr.pad = 0;
    res[k] = tr;
  }
}

// sklearn's _dynamic_max_trials(n_inliers, n_samples, min_samples=2, probability=0.99)
__device__ double dynamic_max_trials(int n_inliers, int n_samples) {
  const double ratio = (double)n_inliers / (double)n_samples;
  const double nom = fmax(DBL_EPSILON, 1.0 - 0.99);
  const double denom = fmax(DBL_EPSILON, 1.0 - ratio * ratio);
  if (nom == 1.0) return 0.0;
  if (denom == 1.0) return INFINITY;
  return fabs(ceil(log(nom) / log(denom)));
}

__global__ void dd_resolve_kernel(int R, const int32_t* __restrict__ offsets, const int32_t* __restrict__ frames, int T,
                                  const DdTrial* __restrict__ res, DdState* __restrict__ st,
                                  uint8_t* __restrict__ running) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const int f = frames[r], n = offsets[f + 1] - offsets[f];
  DdState s = st[f];
  for (int t = 0; t < T && s.n_trials < s.max_trials; ++t) {
    s.n_trials++;
    const DdTrial tr = res[(int64_t)r * T + t];
    if (tr.n < s.n_best) continue;
    if (tr.n == s.n_best && tr.score < s.score_best) continue;
    s.n_best = tr.n; s.score_best = tr.score; s.c = tr.c; s.b = tr.b; s.has_best = 1;
    s.max_trials = fmin(s.max_trials, dynamic_max_trials(s.n_best, n));
  }
  st[f] = s;
  running[f] = s.n_trials < s.max_trials;
}

__global__ void __launch_bounds__(DD_THREADS) dd_final_kernel(
    const int32_t* __restrict__ offsets, const float* __restrict__ x, const double* __restrict__ y,
    const double* __restrict__ thresh, const DdState* __restrict__ st, float* __restrict__ scale,
    float* __restrict__ shift, int32_t* __restrict__ n_trials, int32_t* __restrict__ n_inliers,
    uint8_t* __restrict__ mask) {
  __shared__ double redd[DD_THREADS / 32];
  __shared__ int redi[DD_THREADS / 32];
  const int f = blockIdx.x, o = offsets[f], n = offsets[f + 1] - o;
  const DdState s = st[f];
  const double th = thresh[f];
  int cnt = 0;
  double sx = 0.0, sy = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const bool in = s.has_best && sq_residual(x[o + i], y[o + i], s.c, s.b) <= th;
    mask[o + i] = in;
    if (in) { ++cnt; sx += x[o + i]; sy += (float)y[o + i]; }
  }
  cnt = block_sum(cnt, redi);
  sx = block_sum(sx, redd);
  sy = block_sum(sy, redd);
  if (!s.has_best || cnt == 0) {
    if (threadIdx.x == 0) { scale[f] = 0.f; shift[f] = 0.f; n_trials[f] = s.n_trials; n_inliers[f] = s.has_best ? 0 : -1; }
    return;
  }
  // LinearRegression on the inliers: float32 means, float32 centring, the 1-column least squares accumulated in float64
  const float xm = (float)(sx / cnt), ym = (float)(sy / cnt);
  double sxy = 0.0, sxx = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    if (mask[o + i]) {
      const double a = __fsub_rn(x[o + i], xm), bq = __fsub_rn((float)y[o + i], ym);
      sxy += a * bq;
      sxx += a * a;
    }
  sxy = block_sum(sxy, redd);
  sxx = block_sum(sxx, redd);
  if (threadIdx.x == 0) {
    const float c = sxx == 0.0 ? 0.f : (float)(sxy / sxx);
    scale[f] = c;
    shift[f] = __fsub_rn(ym, __fmul_rn(xm, c));
    n_trials[f] = s.n_trials;
    n_inliers[f] = cnt;
  }
}

__device__ __forceinline__ int frame_tile(const int64_t* tile_offsets, int F, int64_t tile) {
  int lo = 0, hi = F - 1;                  // the frame f with tile_offsets[f] <= tile < tile_offsets[f + 1]
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (tile_offsets[mid] <= tile) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// numpy: disp[nz] = disp[nz] * scale + shift with float32 scale / shift (float32 ops); keep 0 < disp <= 10000;
// depth = float32(1 / disp), 0 elsewhere
__global__ void __launch_bounds__(DD_THREADS) dd_apply_kernel(
    int F, const int64_t* __restrict__ map_offsets, const int64_t* __restrict__ tile_offsets,
    const float* __restrict__ scale, const float* __restrict__ shift, float* __restrict__ disp,
    float* __restrict__ depth, int32_t* __restrict__ tile_counts) {
  __shared__ int redi[DD_THREADS / 32];
  const int64_t tile = blockIdx.x;
  const int f = frame_tile(tile_offsets, F, tile);
  const int64_t base = map_offsets[f], npix = map_offsets[f + 1] - base;
  const int64_t p0 = (tile - tile_offsets[f]) * DD_TILE;
  const float sc = scale[f], sh = shift[f];
  int cnt = 0;
#pragma unroll
  for (int k = 0; k < DD_TILE / DD_THREADS; ++k) {
    const int64_t p = p0 + k * DD_THREADS + threadIdx.x;
    if (p < npix) {
      float d = disp[base + p];
      if (d != 0.f) d = __fadd_rn(__fmul_rn(d, sc), sh);
      const bool ok = d > 0.f && d <= 10000.f;
      if (!ok) d = 0.f;
      disp[base + p] = d;
      depth[base + p] = ok ? __fdiv_rn(1.f, d) : 0.f;
      cnt += ok;
    }
  }
  if (tile_counts) {
    cnt = block_sum(cnt, redi);
    if (threadIdx.x == 0) tile_counts[tile] = cnt;
  }
}

// pycolmap Camera.cam_from_img for SIMPLE_RADIAL: COLMAP's IterativeUndistortion (Newton with central-difference
// Jacobian, 100 iterations, stop when |step|^2 < 1e-10) [3P-memory, parity unpinned]
__device__ void radial_undistort(double k, double* u, double* v) {
  const double x0 = *u, y0 = *v;
  double x = x0, y = y0;
  auto dist = [k](double a, double b, double* da, double* db) {
    const double r2 = a * a + b * b, rad = k * r2;
    *da = a * rad; *db = b * rad;
  };
  for (int it = 0; it < 100; ++it) {
    const double s0 = fmax(DBL_EPSILON, fabs(1e-6 * x)), s1 = fmax(DBL_EPSILON, fabs(1e-6 * y));
    double dx, dy, a0, a1, b0, b1, c0, c1, e0, e1;
    dist(x, y, &dx, &dy);
    dist(x - s0, y, &a0, &a1);
    dist(x + s0, y, &b0, &b1);
    dist(x, y - s1, &c0, &c1);
    dist(x, y + s1, &e0, &e1);
    const double J00 = 1 + (b0 - a0) / (2 * s0), J01 = (e0 - c0) / (2 * s1);
    const double J10 = (b1 - a1) / (2 * s0), J11 = 1 + (e1 - c1) / (2 * s1);
    const double r0 = x + dx - x0, r1 = y + dy - y0;
    const double det = J00 * J11 - J01 * J10;
    const double st0 = (J11 * r0 - J01 * r1) / det, st1 = (J00 * r1 - J10 * r0) / det;
    x -= st0;
    y -= st1;
    if (st0 * st0 + st1 * st1 < 1e-10) break;
  }
  *u = x;
  *v = y;
}

// out = R p + t with the terms added left to right, as Rigid3d.__mul__ of vggsfm_b200.reconstruction does
__device__ __forceinline__ double rowdot(const double* R, double p0, double p1, double p2, double t) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(R[0], p0), __dmul_rn(R[1], p1)), __dmul_rn(R[2], p2)), t);
}

__global__ void __launch_bounds__(DD_THREADS) dd_unproject_kernel(
    int F, const int64_t* __restrict__ map_offsets, const int32_t* __restrict__ map_hw,
    const int64_t* __restrict__ tile_offsets, const int64_t* __restrict__ tile_base, const float* __restrict__ depth,
    const uint8_t* __restrict__ rgb, const int32_t* __restrict__ cam_model, const double* __restrict__ cam_params,
    const double* __restrict__ world_from_cam, double* __restrict__ out) {
  __shared__ int warp_cnt[DD_THREADS / 32];
  const int64_t tile = blockIdx.x;
  const int f = frame_tile(tile_offsets, F, tile);
  const int64_t base = map_offsets[f], npix = map_offsets[f + 1] - base;
  const int W = map_hw[2 * f + 1];
  const int64_t p0 = (tile - tile_offsets[f]) * DD_TILE;
  const double fl = cam_params[4 * f], cx = cam_params[4 * f + 1], cy = cam_params[4 * f + 2];
  const double kr = cam_params[4 * f + 3];
  const bool radial = cam_model[f] == VGG_SIMPLE_RADIAL;
  const double* P = world_from_cam + 12 * f;   // [R | t] of cam_from_world.inverse(), row-major 3 x 4
  // frame f's points are out[6 fb ..] as one [2, M_f, 3] block: xyz rows, then rgb rows
  const int64_t fb = tile_base[tile_offsets[f]], Mf = tile_base[tile_offsets[f + 1]] - fb;
  double* xyz = out + 6 * fb;
  double* col = xyz + 3 * Mf;
  int64_t pos = tile_base[tile] - fb;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int k = 0; k < DD_TILE / DD_THREADS; ++k) {
    const int64_t p = p0 + k * DD_THREADS + threadIdx.x;
    const float d = p < npix ? depth[base + p] : 0.f;
    const bool ok = d != 0.f;
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    __syncthreads();
    if (lane == 0) warp_cnt[wid] = __popc(bal);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < DD_THREADS / 32; ++w) { before += w < wid ? warp_cnt[w] : 0; total += warp_cnt[w]; }
    if (ok) {
      const int64_t o = pos + before + __popc(bal & ((1u << lane) - 1u));
      const double px = (double)(p % W), py = (double)(p / W);
      double u = __ddiv_rn(__dsub_rn(px, cx), fl), v = __ddiv_rn(__dsub_rn(py, cy), fl);
      if (radial) radial_undistort(kr, &u, &v);
      const double z = (double)d, X = __dmul_rn(u, z), Y = __dmul_rn(v, z);
      xyz[3 * o] = rowdot(P, X, Y, z, P[3]);
      xyz[3 * o + 1] = rowdot(P + 4, X, Y, z, P[7]);
      xyz[3 * o + 2] = rowdot(P + 8, X, Y, z, P[11]);
      const uint8_t* c = rgb + 3 * (base + p);
      col[3 * o] = c[0] / 255.0;
      col[3 * o + 1] = c[1] / 255.0;
      col[3 * o + 2] = c[2] / 255.0;
    }
    pos += total;
  }
}

struct DdWork {
  DdState* st;
  DdTrial* trials;
};

size_t carve_dd(int F, void* ws, size_t bytes, DdWork* w) {
  Carver c(ws, bytes);
  w->st = c.take<DdState>((size_t)F);
  w->trials = c.take<DdTrial>((size_t)F * DD_MAX_CHUNK);
  return c.off;
}

}  // namespace

}  // namespace vgg

using namespace vgg;

extern "C" {

int vgg_depth_sparse_samples(int n_total, const int32_t* uvd_frame, const double* uvd, double depth_min,
                             double depth_max, const int64_t* map_offsets, const int32_t* map_hw, const float* disp,
                             float* x_out, double* y_out, uint8_t* keep_out, void* stream) {
  VGG_REQUIRE(n_total >= 0, "n_total must be non-negative");
  if (n_total == 0) return 0;
  dd_samples_kernel<<<(n_total + DD_THREADS - 1) / DD_THREADS, DD_THREADS, 0, (cudaStream_t)stream>>>(
      n_total, uvd_frame, uvd, depth_min, depth_max, map_offsets, map_hw, disp, x_out, y_out, keep_out);
  VGG_LAUNCH_CHECK();
  return 0;
}

int vgg_depth_median(int F, const int32_t* offsets, const double* y, double divisor, double* median_out,
                     void* stream) {
  VGG_REQUIRE(F >= 0, "F must be non-negative");
  if (F == 0) return 0;
  dd_median_kernel<<<F, DD_THREADS, 0, (cudaStream_t)stream>>>(offsets, y, divisor, median_out);
  VGG_LAUNCH_CHECK();
  return 0;
}

int vgg_depth_ransac_workspace_bytes(int F, size_t* bytes) {
  VGG_REQUIRE(F >= 0 && bytes, "F must be non-negative");
  DdWork w;
  *bytes = carve_dd(F, nullptr, 0, &w);
  return 0;
}

int vgg_depth_ransac_max_chunk(void) { return DD_MAX_CHUNK; }

int vgg_depth_ransac_begin(int F, int max_trials, void* workspace, size_t ws_bytes, void* stream) {
  VGG_REQUIRE(F >= 0 && max_trials >= 1, "F must be non-negative and max_trials positive");
  DdWork w;
  VGG_REQUIRE(workspace && carve_dd(F, workspace, ws_bytes, &w) <= ws_bytes, "workspace too small");
  if (F == 0) return 0;
  dd_init_kernel<<<(F + 127) / 128, 128, 0, (cudaStream_t)stream>>>(F, (double)max_trials, w.st);
  VGG_LAUNCH_CHECK();
  return 0;
}

int vgg_depth_ransac_chunk(int F, const int32_t* offsets, const float* x, const double* y, const double* threshold,
                           int R, const int32_t* frames, int T, const int32_t* samples, uint8_t* running_out,
                           void* workspace, size_t ws_bytes, void* stream) {
  VGG_REQUIRE(R >= 0 && R <= F && T >= 1 && T <= DD_MAX_CHUNK, "R must lie in [0, F] and T in [1, max chunk]");
  VGG_REQUIRE(R <= 65535, "at most 65535 live frames per chunk");
  DdWork w;
  VGG_REQUIRE(workspace && carve_dd(F, workspace, ws_bytes, &w) <= ws_bytes, "workspace too small");
  if (R == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  dd_trial_kernel<<<dim3(T, R), DD_THREADS, 0, st>>>(offsets, x, y, threshold, frames, T, samples, w.st, w.trials);
  VGG_LAUNCH_CHECK();
  dd_resolve_kernel<<<(R + 127) / 128, 128, 0, st>>>(R, offsets, frames, T, w.trials, w.st, running_out);
  VGG_LAUNCH_CHECK();
  return 0;
}

int vgg_depth_ransac_finish(int F, const int32_t* offsets, const float* x, const double* y, const double* threshold,
                            float* scale_out, float* shift_out, int32_t* n_trials_out, int32_t* n_inliers_out,
                            uint8_t* inlier_mask_out, void* workspace, size_t ws_bytes, void* stream) {
  DdWork w;
  VGG_REQUIRE(F >= 0, "F must be non-negative");
  VGG_REQUIRE(workspace && carve_dd(F, workspace, ws_bytes, &w) <= ws_bytes, "workspace too small");
  if (F == 0) return 0;
  dd_final_kernel<<<F, DD_THREADS, 0, (cudaStream_t)stream>>>(offsets, x, y, threshold, w.st, scale_out, shift_out,
                                                              n_trials_out, n_inliers_out, inlier_mask_out);
  VGG_LAUNCH_CHECK();
  return 0;
}

int vgg_depth_tile_pixels(void) { return DD_TILE; }

int vgg_depth_apply(int F, int64_t n_tiles, const int64_t* map_offsets, const int64_t* tile_offsets,
                    const float* scale, const float* shift, float* disp, float* depth_out, int32_t* tile_counts,
                    void* stream) {
  VGG_REQUIRE(F >= 0 && n_tiles >= 0 && n_tiles < (1ll << 31), "bad frame or tile count");
  if (F == 0 || n_tiles == 0) return 0;
  dd_apply_kernel<<<(unsigned)n_tiles, DD_THREADS, 0, (cudaStream_t)stream>>>(F, map_offsets, tile_offsets, scale,
                                                                               shift, disp, depth_out, tile_counts);
  VGG_LAUNCH_CHECK();
  return 0;
}

int vgg_depth_unproject(int F, int64_t n_tiles, const int64_t* map_offsets, const int32_t* map_hw,
                        const int64_t* tile_offsets, const int64_t* tile_base, const float* depth, const uint8_t* rgb,
                        const int32_t* cam_model, const double* cam_params, const double* world_from_cam,
                        double* out, void* stream) {
  VGG_REQUIRE(F >= 0 && n_tiles >= 0 && n_tiles < (1ll << 31), "bad frame or tile count");
  if (F == 0 || n_tiles == 0) return 0;
  dd_unproject_kernel<<<(unsigned)n_tiles, DD_THREADS, 0, (cudaStream_t)stream>>>(
      F, map_offsets, map_hw, tile_offsets, tile_base, depth, rgb, cam_model, cam_params, world_from_cam, out);
  VGG_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
