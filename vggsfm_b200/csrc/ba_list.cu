// ITERATIVE_SCHUR on an observation list (vgg_ba_obs_list): the six kernels of the iterative LM loop that walk the dense
// [frames, points] grid, restated on a list whose memory is O(observations) instead of O(S N).  The solve around them is
// the grid's (csrc/ba_solve.cu lm_solve with the list, csrc/ba_pcg.cu): point_prep, the CG control, its fixed-order sums,
// cam_step, point_step, cam_update, gradmax and the shard hook run unchanged.
//
//   list_validate        the list's invariants, one pass, one flag word (launch_list_validate)
//   list_observed        points and frames with a non-empty segment (observed_kernel of the grid)
//   list_point_blocks    per point: g_p, H_pp                                  \  ba_build_blocks
//   list_frame_blocks    per frame: the camera record, the cost, g_s / H_ss    /
//   list_rhs_jacobi      per frame: rhs += Z q and the Schur-Jacobi blocks      \  pcg_rhs_jacobi
//   list_rhs_shared      per point: the shared-intrinsics rows of both          /
//   list_point_w         per point: w_n = W_n^T x, or t_n = M_n M_n^T w_n       backsub, pass 1 of pcg_schur
//   list_schur           per frame: qs -= Dc sum_n W_sn t_n                      pass 2 of pcg_schur
//   list_model_change    per point: -(J d)^T (f + J d / 2)                      pcg_model_change
//
// Every observation's residual and Jacobian come from obs_math (ba_obs.h), as in the grid kernels.  Two walks:
//   * point passes: one warp per point, its lanes over the point's segment [track_start[n], track_start[n+1]) (at most
//     S entries: one per frame), the sums reduced in the warp and stored without atomics;
//   * frame passes: CTA b takes positions [b LF_CHUNK, (b+1) LF_CHUNK) of frame_obs, which cover one or more frame
//     segments or a piece of a long one; per frame the CTA sums in registers, reduces through shared memory and adds
//     its partial with one RED per (CTA, frame, record entry), so a frame of any length costs ceil(len / LF_CHUNK) + 1
//     REDs per entry, never one per observation.
#include <stddef.h>
#include <algorithm>
#include "ba_obs.h"
#include "ba_pcg.h"
#include "common.cuh"

namespace vgg {

constexpr int LP_W = 8;           // point passes: warps (points) per CTA
constexpr int LF_T = 128;         // frame passes: threads per CTA
constexpr int LF_CHUNK = 1024;    // frame passes: frame_obs positions per CTA

// bits of the validation word
enum : int {
  LIST_BAD_TRACK_START = 1, LIST_BAD_POINT = 2, LIST_BAD_FRAME = 4, LIST_BAD_TRACK_ORDER = 8,
  LIST_BAD_FRAME_START = 16, LIST_BAD_FRAME_OBS = 32,
};

__device__ __forceinline__ void load_cam(const double* __restrict__ poses, const double* __restrict__ intr, int s,
                                         double (&cam)[16]) {
#pragma unroll
  for (int i = 0; i < 12; ++i) cam[i] = poses[(size_t)s * 12 + i];
#pragma unroll
  for (int i = 0; i < 4; ++i) cam[12 + i] = intr[(size_t)s * 4 + i];
}

// the frames that meet this CTA's positions [lo, hi) of frame_obs, in order: body(s, a, b) on the non-empty piece
// [a, b) of frame s.  Every thread of the CTA takes the same frames (body may synchronise the CTA).
template <class Body>
__device__ __forceinline__ void for_cta_frames(int S, const ObsList& L, Body body) {
  __shared__ int s_first;
  const int lo = blockIdx.x * LF_CHUNK, hi = min(L.M, lo + LF_CHUNK);
  if (threadIdx.x == 0) {
    int a = 0, b = S - 1;                       // the last frame whose segment starts at or before lo
    while (a < b) {
      const int m = (a + b + 1) >> 1;
      if (L.frame_start[m] <= lo) a = m;
      else b = m - 1;
    }
    s_first = a;
  }
  __syncthreads();
  for (int s = s_first; s < S; ++s) {
    const int fa = L.frame_start[s];
    if (fa >= hi) break;
    const int a = max(lo, fa), b = min(hi, L.frame_start[s + 1]);
    if (a < b) body(s, a, b);
  }
}

// the CTA's sum of v[K] (K <= LF_T): thread k < K returns entry k
template <int K>
__device__ __forceinline__ double cta_sum(double (&v)[K]) {
  constexpr int NW = LF_T / 32;
  __shared__ double red[K][NW];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const double s = warp_sum(v[k]);
    if (lane == 0) red[k][warp] = s;
  }
  __syncthreads();
  double r = 0.0;
  if ((int)threadIdx.x < K)
#pragma unroll
    for (int w = 0; w < NW; ++w) r += red[threadIdx.x][w];
  __syncthreads();
  return r;
}

// ------------------------------------------------------------------------------------------------
// One pass over every index of the list's arrays.  Together the checks prove that point[] names the segment of each
// observation and that frame_obs is the unique frame-major permutation of the list: an entry at position i of frame s's
// segment holds an observation of frame s, entries within a segment strictly increase, so frame_obs is injective and
// every frame's count of observations is at least its segment's length; the lengths add up to M, so the counts equal
// the lengths (the frame histogram is the frame_start differences) and frame_obs is a permutation.
__global__ void __launch_bounds__(256) list_validate_kernel(int S, int N, ObsList L, int* __restrict__ bad) {
  const int M = L.M, top = max(M - 1, max(N, S));
  int f = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= top; i += gridDim.x * blockDim.x) {
    if (i <= N) {
      const int t = L.track_start[i];
      if ((i == 0 && t != 0) || (i == N && t != M) || (i < N && L.track_start[i + 1] < t)) f |= LIST_BAD_TRACK_START;
    }
    if (i <= S) {
      const int t = L.frame_start[i];
      if ((i == 0 && t != 0) || (i == S && t != M) || (i < S && L.frame_start[i + 1] < t)) f |= LIST_BAD_FRAME_START;
    }
    if (i < M) {
      const int n = L.point[i];
      const bool n_ok = n >= 0 && n < N;
      const int seg_end = n_ok ? L.track_start[n + 1] : 0;
      if (!n_ok || L.track_start[n] > i || seg_end <= i) f |= LIST_BAD_POINT;
      const int fr = L.frame[i];
      if (fr < 0 || fr >= S) f |= LIST_BAD_FRAME;
      else if (i + 1 < M && i + 1 < seg_end && L.frame[i + 1] <= fr) f |= LIST_BAD_TRACK_ORDER;
      const int m = L.frame_obs[i];
      const int s = (m >= 0 && m < M) ? L.frame[m] : -1;
      if (s < 0 || s >= S || L.frame_start[s] > i || L.frame_start[s + 1] <= i) f |= LIST_BAD_FRAME_OBS;
      else if (i + 1 < M && i + 1 < L.frame_start[s + 1] && L.frame_obs[i + 1] <= m) f |= LIST_BAD_FRAME_OBS;
    }
  }
  if (f) atomicOr(bad, f);
}

// point_seen[n] = 1 / frame_seen[s] = 1.0 for a non-empty segment (both zeroed beforehand)
__global__ void list_observed_kernel(int S, int N, const int* __restrict__ track_start,
                                     const int* __restrict__ frame_start, uint8_t* __restrict__ point_seen,
                                     double* __restrict__ frame_seen) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N && track_start[i + 1] > track_start[i]) point_seen[i] = 1;
  if (i < S && frame_start[i + 1] > frame_start[i]) frame_seen[i] = 1.0;
}

// ------------------------------------------------------------------------------------------------
// g_p[n] = sum J_p^T r, H_pp[n] = sum J_p^T J_p (xx, xy, xz, yy, yz, zz) over the point's segment
template <int MODEL, int MODE, bool ROBUST>
__global__ void __launch_bounds__(LP_W * 32) list_point_blocks_kernel(
    int N, ObsList L, const double* __restrict__ poses, const double* __restrict__ intr,
    const double* __restrict__ points, const uint8_t* __restrict__ point_const, double* __restrict__ g_p,
    double* __restrict__ H_pp, BaLoss loss) {
  const int lane = threadIdx.x & 31, n = blockIdx.x * LP_W + (threadIdx.x >> 5);
  if (n >= N) return;
  const double X0 = points[(size_t)n * 3], X1 = points[(size_t)n * 3 + 1], X2 = points[(size_t)n * 3 + 2];
  const bool pc = point_const && point_const[n] != 0;
  double v[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) v[k] = 0.0;
  for (int m = L.track_start[n] + lane; m < L.track_start[n + 1]; m += 32) {
    double cam[16];
    load_cam(poses, intr, L.frame[m], cam);
    const float2 ob = L.uv[m];
    double jc0[8], jc1[8], jx0[3], jx1[3], rx, ry, oc;
    obs_math<MODEL, ROBUST>(cam, 1, X0, X1, X2, pc, ob.x, ob.y, true, jc0, jc1, jx0, jx1, rx, ry, loss, oc);
    v[0] += jx0[0] * rx + jx1[0] * ry;
    v[1] += jx0[1] * rx + jx1[1] * ry;
    v[2] += jx0[2] * rx + jx1[2] * ry;
    v[3] += jx0[0] * jx0[0] + jx1[0] * jx1[0];
    v[4] += jx0[0] * jx0[1] + jx1[0] * jx1[1];
    v[5] += jx0[0] * jx0[2] + jx1[0] * jx1[2];
    v[6] += jx0[1] * jx0[1] + jx1[1] * jx1[1];
    v[7] += jx0[1] * jx0[2] + jx1[1] * jx1[2];
    v[8] += jx0[2] * jx0[2] + jx1[2] * jx1[2];
  }
  const double r = warp_reduce_scatter<16>(v, lane);
  if (lane < 3) g_p[(size_t)n * 3 + lane] = r;
  else if (lane < 9) H_pp[(size_t)n * 6 + (lane - 3)] = r;
}

// camrec[s] += the frame's camera record (g_c | H_cc upper-packed | H_cs), cost += 0.5 sum rho, shared += (g_s, H_ss)
template <int MODEL, int MODE, bool ROBUST>
__global__ void __launch_bounds__(LF_T) list_frame_blocks_kernel(
    int S, ObsList L, const double* __restrict__ poses, const double* __restrict__ intr,
    const double* __restrict__ points, const uint8_t* __restrict__ point_const, double* __restrict__ cost,
    double* __restrict__ camrec, double* __restrict__ shared_out, BaLoss loss) {
  using C = BlkCfg<MODEL, MODE>;
  constexpr int DC = C::DC, NS = C::NS, KR = C::KR;
  double tot[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};          // cost, g_s (2), H_ss (xx, xy, yy)
  for_cta_frames(S, L, [&](int s, int a, int b) {
    double cam[16];
    load_cam(poses, intr, s, cam);
    double acc[KR];
#pragma unroll
    for (int k = 0; k < KR; ++k) acc[k] = 0.0;
    for (int j = a + threadIdx.x; j < b; j += LF_T) {
      const int m = L.frame_obs[j], n = L.point[m];
      const float2 ob = L.uv[m];
      double jc0[8], jc1[8], jx0[3], jx1[3], rx, ry, oc;
      obs_math<MODEL, ROBUST>(cam, 1, points[(size_t)n * 3], points[(size_t)n * 3 + 1], points[(size_t)n * 3 + 2],
                              point_const && point_const[n] != 0, ob.x, ob.y, true, jc0, jc1, jx0, jx1, rx, ry, loss, oc);
      tot[0] += oc;
      cam_accumulate<DC, NS, KR>(acc, jc0, jc1, rx, ry, std::make_integer_sequence<int, KR>{});
      if (NS > 0) {
        tot[1] += jc0[6] * rx + jc1[6] * ry;
        tot[3] += jc0[6] * jc0[6] + jc1[6] * jc1[6];
        if (NS > 1) {
          tot[2] += jc0[7] * rx + jc1[7] * ry;
          tot[4] += jc0[6] * jc0[7] + jc1[6] * jc1[7];
          tot[5] += jc0[7] * jc0[7] + jc1[7] * jc1[7];
        }
      }
    }
    const double r = cta_sum<KR>(acc);
    if ((int)threadIdx.x < KR && r != 0.0) atomicAdd(&camrec[(size_t)s * KR + threadIdx.x], r);
  });
  const double r = cta_sum<6>(tot);
  if (threadIdx.x == 0 && r != 0.0) atomicAdd(cost, r);
  else if (NS > 0 && threadIdx.x >= 1 && threadIdx.x < 6 && r != 0.0) atomicAdd(&shared_out[threadIdx.x - 1], r);
}

// ------------------------------------------------------------------------------------------------
// per frame: rhs[row] += (Z q)[row] and acc[block] += Z_b Z_b^T (upper entries) over the frame's observations, Z = W M
// (pcg_rhs_jacobi_kernel of the grid, csrc/ba_pcg.cu)
template <int MODEL, int MODE, bool ROBUST>
__global__ void __launch_bounds__(LF_T) list_rhs_jacobi_kernel(
    int S, ObsList L, const double* __restrict__ poses, const double* __restrict__ intr,
    const double* __restrict__ points, const uint8_t* __restrict__ point_const, const double* __restrict__ M,
    const double* __restrict__ q, double* __restrict__ rhs, double* __restrict__ acc, BaLoss loss) {
  using C = BlkCfg<MODEL, MODE>;
  constexpr int DC = C::DC;
  constexpr int NI = DC - 6, NIU = NI * (NI + 1) / 2;
  constexpr int NB = 12 + NIU;                              // upper entries of the frame's blocks: 6 + 6 + intrinsics
  for_cta_frames(S, L, [&](int s, int a, int b) {
    double cam[16];
    load_cam(poses, intr, s, cam);
    double v[DC + NB];                                      // Z q | block entries
#pragma unroll
    for (int k = 0; k < DC + NB; ++k) v[k] = 0.0;
    for (int j = a + threadIdx.x; j < b; j += LF_T) {
      const int m = L.frame_obs[j], n = L.point[m];
      const float2 ob = L.uv[m];
      double jc0[8], jc1[8], jx0[3], jx1[3], rx, ry, oc;
      obs_math<MODEL, ROBUST>(cam, 1, points[(size_t)n * 3], points[(size_t)n * 3 + 1], points[(size_t)n * 3 + 2],
                              point_const && point_const[n] != 0, ob.x, ob.y, true, jc0, jc1, jx0, jx1, rx, ry, loss, oc);
      const double* mm = M + (size_t)n * 9;
      const double q0 = q[(size_t)n * 3], q1 = q[(size_t)n * 3 + 1], q2 = q[(size_t)n * 3 + 2];
      double z[DC][3];
#pragma unroll
      for (int i = 0; i < DC; ++i) {
        const double w0 = w_entry(jc0, jc1, jx0, jx1, i, 0), w1 = w_entry(jc0, jc1, jx0, jx1, i, 1),
                     w2 = w_entry(jc0, jc1, jx0, jx1, i, 2);
        z[i][0] = w0 * mm[0];
        z[i][1] = w0 * mm[1] + w1 * mm[4];
        z[i][2] = w0 * mm[2] + w1 * mm[5] + w2 * mm[8];
        v[i] += z[i][0] * q0 + z[i][1] * q1 + z[i][2] * q2;
      }
      int k = DC;
#pragma unroll
      for (int blk = 0; blk < 3; ++blk) {
        const int r0 = 3 * blk, nb = blk < 2 ? 3 : NI;
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
          for (int c = a; c < 3; ++c)
            if (a < nb && c < nb) {
              v[k] += z[r0 + a][0] * z[r0 + c][0] + z[r0 + a][1] * z[r0 + c][1] + z[r0 + a][2] * z[r0 + c][2];
              ++k;
            }
      }
    }
    const double r = cta_sum<DC + NB>(v);
    const int t = threadIdx.x;
    if (t < DC) {
      if (r != 0.0) atomicAdd(&rhs[(size_t)s * DC + t], r);
    } else if (t < DC + NB && r != 0.0) {
      const int k = t - DC, blk = k < 6 ? 0 : (k < 12 ? 1 : 2), nb = blk < 2 ? 3 : NI;
      atomicAdd(&acc[(size_t)(3 * s + blk) * 9 + pack_row(nb, k - 6 * blk) * 3 + pack_col(nb, k - 6 * blk)], r);
    }
  });
}

// per point: the shared-intrinsics rows of the same, zs = (sum_s W_sn[shared rows]) M_n; rhs[S DC + j] += zs_j q_n and
// acc[3 S] += zs zs^T, summed over the CTA's points and added once per CTA
template <int MODEL, int MODE, bool ROBUST>
__global__ void __launch_bounds__(LP_W * 32, 1) list_rhs_shared_kernel(
    int S, int N, ObsList L, const double* __restrict__ poses, const double* __restrict__ intr,
    const double* __restrict__ points, const uint8_t* __restrict__ point_const, const double* __restrict__ M,
    const double* __restrict__ q, double* __restrict__ rhs, double* __restrict__ acc, BaLoss loss) {
  using C = BlkCfg<MODEL, MODE>;
  constexpr int DC = C::DC, NS = C::NS > 0 ? C::NS : 1, NO = NS + NS * (NS + 1) / 2;
  __shared__ double red[NO][LP_W];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n = blockIdx.x * LP_W + warp;
  double w[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) w[e] = 0.0;
  if (n < N) {
    const double X0 = points[(size_t)n * 3], X1 = points[(size_t)n * 3 + 1], X2 = points[(size_t)n * 3 + 2];
    const bool pc = point_const && point_const[n] != 0;
    const int m1 = L.track_start[n + 1];
#pragma unroll 1
    for (int m = L.track_start[n] + lane; m < m1; m += 32) {
      double cam[16];
      load_cam(poses, intr, L.frame[m], cam);
      const float2 ob = L.uv[m];
      double jc0[8], jc1[8], jx0[3], jx1[3], rx, ry, oc;
      obs_math<MODEL, ROBUST>(cam, 1, X0, X1, X2, pc, ob.x, ob.y, true, jc0, jc1, jx0, jx1, rx, ry, loss, oc);
#pragma unroll
      for (int e = 0; e < 3 * NS; ++e) w[e] += w_entry(jc0, jc1, jx0, jx1, 6 + e / 3, e % 3);
    }
  }
  const double r = warp_reduce_scatter<8>(w, lane);       // lane e < 3 NS: sum of w[e]
  double ws[3 * NS];
#pragma unroll
  for (int e = 0; e < 3 * NS; ++e) ws[e] = __shfl_sync(0xffffffffu, r, e);
  if (lane == 0) {
    double zs[NS][3];
    const double* mm = M + (size_t)n * 9;
    const double* qq = q + (size_t)n * 3;
#pragma unroll
    for (int j = 0; j < NS; ++j) {
      const double w0 = ws[3 * j], w1 = ws[3 * j + 1], w2 = ws[3 * j + 2];
      zs[j][0] = n < N ? w0 * mm[0] : 0.0;
      zs[j][1] = n < N ? w0 * mm[1] + w1 * mm[4] : 0.0;
      zs[j][2] = n < N ? w0 * mm[2] + w1 * mm[5] + w2 * mm[8] : 0.0;
      red[j][warp] = n < N ? zs[j][0] * qq[0] + zs[j][1] * qq[1] + zs[j][2] * qq[2] : 0.0;
    }
    int k = NS;
#pragma unroll
    for (int a = 0; a < NS; ++a)
#pragma unroll
      for (int c = a; c < NS; ++c) red[k++][warp] = zs[a][0] * zs[c][0] + zs[a][1] * zs[c][1] + zs[a][2] * zs[c][2];
  }
  __syncthreads();
  if ((int)threadIdx.x < NO) {
    const int k = threadIdx.x;
    double v = 0.0;
#pragma unroll
    for (int i = 0; i < LP_W; ++i) v += red[k][i];
    if (v != 0.0) {
      if (k < NS) atomicAdd(&rhs[(size_t)S * DC + k], v);
      else atomicAdd(&acc[(size_t)(3 * S) * 9 + pack_row(NS, k - NS) * 3 + pack_col(NS, k - NS)], v);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// per point: w_n = sum_s W_sn^T x_s (+ the shared-intrinsics rows); M = null: out[n] = w_n (backsub's wacc), otherwise
// out[n] = M_n M_n^T w_n, zero for a constant point (pass 1 of the matvec's Schur part; cg: return when the CG is done)
template <int MODEL, int MODE, bool ROBUST>
__global__ void __launch_bounds__(LP_W * 32) list_point_w_kernel(
    int S, int N, ObsList L, const double* __restrict__ poses, const double* __restrict__ intr,
    const double* __restrict__ points, const uint8_t* __restrict__ point_const, const double* __restrict__ x,
    const double* __restrict__ M, double* __restrict__ out, const double* __restrict__ cg, BaLoss loss) {
  if (cg && cg[CG_DONE] != 0.0) return;
  using C = BlkCfg<MODEL, MODE>;
  constexpr int DC = C::DC, NS = C::NS;
  const int lane = threadIdx.x & 31, n = blockIdx.x * LP_W + (threadIdx.x >> 5);
  if (n >= N) return;
  const double X0 = points[(size_t)n * 3], X1 = points[(size_t)n * 3 + 1], X2 = points[(size_t)n * 3 + 2];
  const bool pc = point_const && point_const[n] != 0;
  double xsh[2] = {0.0, 0.0};
#pragma unroll
  for (int j = 0; j < NS; ++j) xsh[j] = x[(size_t)S * DC + j];
  double w[4] = {0.0, 0.0, 0.0, 0.0};
  for (int m = L.track_start[n] + lane; m < L.track_start[n + 1]; m += 32) {
    const int s = L.frame[m];
    double cam[16];
    load_cam(poses, intr, s, cam);
    const float2 ob = L.uv[m];
    double jc0[8], jc1[8], jx0[3], jx1[3], rx, ry, oc;
    obs_math<MODEL, ROBUST>(cam, 1, X0, X1, X2, pc, ob.x, ob.y, true, jc0, jc1, jx0, jx1, rx, ry, loss, oc);
    const double* d = x + (size_t)s * DC;
#pragma unroll
    for (int i = 0; i < DC; ++i) {
      const double di = __ldg(d + i);
      w[0] = fma(w_entry(jc0, jc1, jx0, jx1, i, 0), di, w[0]);
      w[1] = fma(w_entry(jc0, jc1, jx0, jx1, i, 1), di, w[1]);
      w[2] = fma(w_entry(jc0, jc1, jx0, jx1, i, 2), di, w[2]);
    }
#pragma unroll
    for (int j = 0; j < NS; ++j) {
      w[0] = fma(w_entry(jc0, jc1, jx0, jx1, 6 + j, 0), xsh[j], w[0]);
      w[1] = fma(w_entry(jc0, jc1, jx0, jx1, 6 + j, 1), xsh[j], w[1]);
      w[2] = fma(w_entry(jc0, jc1, jx0, jx1, 6 + j, 2), xsh[j], w[2]);
    }
  }
  const double r = warp_reduce_scatter<4>(w, lane);       // lane c < 3: sum of w[c]
  if (!M) {
    if (lane < 3) out[(size_t)n * 3 + lane] = r;
    return;
  }
  const double a0 = __shfl_sync(0xffffffffu, r, 0), a1 = __shfl_sync(0xffffffffu, r, 1),
               a2 = __shfl_sync(0xffffffffu, r, 2);
  if (lane < 3) {
    double t = 0.0;
    if (!pc) {
      const double* m = M + (size_t)n * 9;
      const double y0 = m[0] * a0;
      const double y1 = m[1] * a0 + m[4] * a1;
      const double y2 = m[2] * a0 + m[5] * a1 + m[8] * a2;
      t = lane == 0 ? m[0] * y0 + m[1] * y1 + m[2] * y2 : (lane == 1 ? m[4] * y1 + m[5] * y2 : m[8] * y2);
    }
    out[(size_t)n * 3 + lane] = t;
  }
}

// per frame: qs[row] -= sc[row] (sum_n W_sn t_n)[row] for free rows (pass 2 of the matvec's Schur part; qs zeroed by
// pcg_hcc); the shared-intrinsics rows sum over every observation and are added once per CTA
template <int MODEL, int MODE, bool ROBUST>
__global__ void __launch_bounds__(LF_T) list_schur_kernel(
    int S, ObsList L, const double* __restrict__ poses, const double* __restrict__ intr,
    const double* __restrict__ points, const uint8_t* __restrict__ point_const, const double* __restrict__ tp,
    const double* __restrict__ sc, const uint8_t* __restrict__ pconst, double* __restrict__ qs,
    const double* __restrict__ cg, BaLoss loss) {
  if (cg[CG_DONE] != 0.0) return;
  using C = BlkCfg<MODEL, MODE>;
  constexpr int DC = C::DC, NS = C::NS;
  double vsh[2] = {0.0, 0.0};
  for_cta_frames(S, L, [&](int s, int a, int b) {
    double cam[16];
    load_cam(poses, intr, s, cam);
    double v[DC];
#pragma unroll
    for (int i = 0; i < DC; ++i) v[i] = 0.0;
    for (int j = a + threadIdx.x; j < b; j += LF_T) {
      const int m = L.frame_obs[j], n = L.point[m];
      const float2 ob = L.uv[m];
      double jc0[8], jc1[8], jx0[3], jx1[3], rx, ry, oc;
      obs_math<MODEL, ROBUST>(cam, 1, points[(size_t)n * 3], points[(size_t)n * 3 + 1], points[(size_t)n * 3 + 2],
                              point_const && point_const[n] != 0, ob.x, ob.y, true, jc0, jc1, jx0, jx1, rx, ry, loss, oc);
      const double t0 = tp[(size_t)n * 3], t1 = tp[(size_t)n * 3 + 1], t2 = tp[(size_t)n * 3 + 2];
#pragma unroll
      for (int i = 0; i < DC; ++i)
        v[i] += w_entry(jc0, jc1, jx0, jx1, i, 0) * t0 + w_entry(jc0, jc1, jx0, jx1, i, 1) * t1 +
                w_entry(jc0, jc1, jx0, jx1, i, 2) * t2;
#pragma unroll
      for (int k = 0; k < NS; ++k)
        vsh[k] += w_entry(jc0, jc1, jx0, jx1, 6 + k, 0) * t0 + w_entry(jc0, jc1, jx0, jx1, 6 + k, 1) * t1 +
                  w_entry(jc0, jc1, jx0, jx1, 6 + k, 2) * t2;
    }
    const double r = cta_sum<DC>(v);
    if ((int)threadIdx.x < DC) {
      const size_t row = (size_t)s * DC + threadIdx.x;
      if (!pconst[row] && r != 0.0) atomicAdd(&qs[row], -sc[row] * r);
    }
  });
  if (NS > 0) {
    const double r = cta_sum<2>(vsh);
    if ((int)threadIdx.x < NS) {
      const size_t row = (size_t)S * DC + threadIdx.x;
      if (!pconst[row] && r != 0.0) atomicAdd(&qs[row], -sc[row] * r);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// per point: Ceres' model change -(J d)^T (f + J d / 2) over the point's segment, d_p recomputed with point_step's
// arithmetic (pcg_model_change_kernel of the grid); one RED per CTA
template <int MODEL, int MODE, bool ROBUST>
__global__ void __launch_bounds__(LP_W * 32) list_model_change_kernel(
    int S, int N, ObsList L, const double* __restrict__ poses, const double* __restrict__ intr,
    const double* __restrict__ points, const uint8_t* __restrict__ point_const, const double* __restrict__ M,
    const double* __restrict__ g_p, const double* __restrict__ wacc, const double* __restrict__ d_c,
    double* __restrict__ out, BaLoss loss) {
  using C = BlkCfg<MODEL, MODE>;
  constexpr int DC = C::DC, NS = C::NS;
  __shared__ double s_red[LP_W];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n = blockIdx.x * LP_W + warp;
  double accm = 0.0;
  if (n < N) {
    const double X0 = points[(size_t)n * 3], X1 = points[(size_t)n * 3 + 1], X2 = points[(size_t)n * 3 + 2];
    const bool pc = point_const && point_const[n] != 0;
    double d0 = 0.0, d1 = 0.0, d2 = 0.0;
    if (!pc) {
      const double* m = M + (size_t)n * 9;
      const double y0 = -(g_p[n * 3] + wacc[n * 3]), y1 = -(g_p[n * 3 + 1] + wacc[n * 3 + 1]),
                   y2 = -(g_p[n * 3 + 2] + wacc[n * 3 + 2]);
      const double t0 = m[0] * y0;
      const double t1 = m[1] * y0 + m[4] * y1;
      const double t2 = m[2] * y0 + m[5] * y1 + m[8] * y2;
      d0 = m[0] * t0 + m[1] * t1 + m[2] * t2;
      d1 = m[4] * t1 + m[5] * t2;
      d2 = m[8] * t2;
    }
    double dsh[2] = {0.0, 0.0};
#pragma unroll
    for (int j = 0; j < NS; ++j) dsh[j] = d_c[(size_t)S * DC + j];
    for (int m = L.track_start[n] + lane; m < L.track_start[n + 1]; m += 32) {
      const int s = L.frame[m];
      double cam[16];
      load_cam(poses, intr, s, cam);
      const float2 ob = L.uv[m];
      double jc0[8], jc1[8], jx0[3], jx1[3], rx, ry, oc;
      obs_math<MODEL, ROBUST>(cam, 1, X0, X1, X2, pc, ob.x, ob.y, true, jc0, jc1, jx0, jx1, rx, ry, loss, oc);
      const double* d = d_c + (size_t)s * DC;
      double e0 = jx0[0] * d0 + jx0[1] * d1 + jx0[2] * d2, e1 = jx1[0] * d0 + jx1[1] * d1 + jx1[2] * d2;
#pragma unroll
      for (int i = 0; i < DC; ++i) {
        const double di = __ldg(d + i);
        e0 = fma(jc0[i], di, e0);
        e1 = fma(jc1[i], di, e1);
      }
#pragma unroll
      for (int j = 0; j < NS; ++j) {
        e0 = fma(jc0[6 + j], dsh[j], e0);
        e1 = fma(jc1[6 + j], dsh[j], e1);
      }
      accm -= e0 * (rx + 0.5 * e0) + e1 * (ry + 0.5 * e1);
    }
  }
  accm = warp_sum(accm);
  if (lane == 0) s_red[warp] = accm;
  __syncthreads();
  if (threadIdx.x == 0) {
    double v = 0.0;
    for (int k = 0; k < LP_W; ++k) v += s_red[k];
    if (v != 0.0) atomicAdd(out, v);
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static unsigned point_ctas(int N) { return (unsigned)((N + LP_W - 1) / LP_W); }
static unsigned frame_ctas(int M) { return (unsigned)((M + LF_CHUNK - 1) / LF_CHUNK); }

int launch_list_validate(int S, int N, const ObsList& L, int* bad, cudaStream_t st) {
  const int top = std::max(L.M - 1, std::max(N, S));
  list_validate_kernel<<<std::min(1024, top / 256 + 1), 256, 0, st>>>(S, N, L, bad);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

int launch_list_observed(int S, int N, const ObsList& L, uint8_t* point_seen, double* frame_seen, cudaStream_t st) {
  list_observed_kernel<<<(std::max(S, N) + 255) / 256, 256, 0, st>>>(S, N, L.track_start, L.frame_start, point_seen,
                                                                      frame_seen);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

// the accumulators come in zeroed (lm_solve's eval): g_p and H_pp are stored, the rest added
int launch_list_blocks(const vgg_ba_problem* p, const ObsList& L, double* cost, double* camrec, double* g_p,
                       double* H_pp, double* shared_out, cudaStream_t st) {
  if (L.M == 0) return VGG_OK;
  const BaLoss loss = ba_loss_of(p);
  {
    VGG_PICK_BA_KERNEL(kern, list_point_blocks_kernel, p);
    kern<<<point_ctas(p->N), LP_W * 32, 0, st>>>(p->N, L, p->poses, p->intr, p->points, p->point_const, g_p, H_pp, loss);
    VGG_LAUNCH_CHECK();
  }
  VGG_PICK_BA_KERNEL(kern, list_frame_blocks_kernel, p);
  kern<<<frame_ctas(L.M), LF_T, 0, st>>>(p->S, L, p->poses, p->intr, p->points, p->point_const, cost, camrec,
                                          shared_out, loss);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

int launch_list_rhs_jacobi(const PcgOp& op, const double* q, const PcgBuffers& B, cudaStream_t st) {
  const vgg_ba_problem* p = op.p;
  const ObsList& L = *op.obs;
  if (L.M == 0) return VGG_OK;
  const BaLoss loss = ba_loss_of(p);
  {
    VGG_PICK_BA_KERNEL(kern, list_rhs_jacobi_kernel, p);
    kern<<<frame_ctas(L.M), LF_T, 0, st>>>(p->S, L, p->poses, p->intr, p->points, p->point_const, op.M, q, B.rhs, B.acc,
                                            loss);
    VGG_LAUNCH_CHECK();
  }
  if (op.ns > 0) {
    VGG_PICK_BA_KERNEL(kern, list_rhs_shared_kernel, p);
    kern<<<point_ctas(p->N), LP_W * 32, 0, st>>>(p->S, p->N, L, p->poses, p->intr, p->points, p->point_const, op.M, q,
                                                  B.rhs, B.acc, loss);
    VGG_LAUNCH_CHECK();
  }
  return VGG_OK;
}

int launch_list_schur(const PcgOp& op, const PcgBuffers& B, cudaStream_t st) {
  const vgg_ba_problem* p = op.p;
  const ObsList& L = *op.obs;
  if (L.M == 0) return VGG_OK;
  const BaLoss loss = ba_loss_of(p);
  {
    VGG_PICK_BA_KERNEL(kern, list_point_w_kernel, p);
    kern<<<point_ctas(p->N), LP_W * 32, 0, st>>>(p->S, p->N, L, p->poses, p->intr, p->points, p->point_const, B.u,
                                                  op.M, B.tp, B.cg, loss);
    VGG_LAUNCH_CHECK();
  }
  VGG_PICK_BA_KERNEL(kern, list_schur_kernel, p);
  kern<<<frame_ctas(L.M), LF_T, 0, st>>>(p->S, L, p->poses, p->intr, p->points, p->point_const, B.tp, op.sc_c,
                                          p->param_const, B.qs, B.cg, loss);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

int launch_list_backsub(const vgg_ba_problem* p, const ObsList& L, const double* d_c, double* wacc, cudaStream_t st) {
  if (L.M == 0) {
    VGG_CUDA_CHECK(cudaMemsetAsync(wacc, 0, sizeof(double) * 3 * (size_t)p->N, st));
    return VGG_OK;
  }
  VGG_PICK_BA_KERNEL(kern, list_point_w_kernel, p);
  kern<<<point_ctas(p->N), LP_W * 32, 0, st>>>(p->S, p->N, L, p->poses, p->intr, p->points, p->point_const, d_c,
                                                nullptr, wacc, nullptr, ba_loss_of(p));
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

int launch_list_model_change(const vgg_ba_problem* p, const ObsList& L, const double* M, const double* g_p,
                             const double* wacc, const double* d_c, double* out, cudaStream_t st) {
  VGG_CUDA_CHECK(cudaMemsetAsync(out, 0, sizeof(double), st));
  if (L.M == 0) return VGG_OK;
  VGG_PICK_BA_KERNEL(kern, list_model_change_kernel, p);
  kern<<<point_ctas(p->N), LP_W * 32, 0, st>>>(p->S, p->N, L, p->poses, p->intr, p->points, p->point_const, M, g_p,
                                                wacc, d_c, out, ba_loss_of(p));
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

}  // namespace vgg
