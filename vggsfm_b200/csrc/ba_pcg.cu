// ITERATIVE_SCHUR linear solver of the LM loop: preconditioned conjugate gradients on the reduced camera system without
// forming it.  Restates Ceres' IterativeSchurSolver with the SCHUR_JACOBI preconditioner and its
// ConjugateGradientsSolver (oracle/ba_pcg_oracle.py), in the scaled, damped variables of the direct path
// (csrc/ba_schur.cu scale_damp):
//
//   A = Dc (H_cc - sum_n Z_n Z_n^T) Dc + diag(clamp(diag(Dc H_cc Dc)))/radius,  Z_sn = W_sn M_n,  b = Dc rhs,
//   constant parameters pinned (identity rows and columns, zero right-hand side).
//
//   pcg_hc             per frame: rhs = -g, hdiag, gvec out of the camera records (no dense matrix)
//   pcg_rhs_jacobi     one pass over the observations: rhs += sum Z q and, per parameter block, sum Z_b Z_b^T
//                      (rotation, translation, per-frame intrinsics, shared intrinsics: Ceres' blocks)
//   pcg_init           per block: A_bb scaled and damped, inverted by a 3x3 Cholesky; b, x = 0, r = b, z = P r, rho
//   pcg_hcc / pcg_schur   q = A v: the camera-Hessian part per parameter row, then the Schur part per track CTA into its
//                      own vector qs, which pcg_alpha (or pcg_update after the residual reset) adds to q
//   pcg_alpha / pcg_xstep / pcg_update   the CG scalars and vectors
//   pcg_model_change   Ceres' model change -(J d)^T (f + J d / 2) of the inexact step, per observation
//
// W_sn is rebuilt per observation by obs_math (ba_obs.h), as z_build and backsub do; nothing is stored per observation.
// The CG scalars and its termination live on the device (pcg_state): every CG kernel returns at once when the state's
// done flag is set, and the host launches iterations in chunks of PCG_CHUNK, reading the flag once per chunk while the
// next chunk is already queued.
//
// Track shards (an all-reduce hook): each rank holds every camera and its own tracks, so what a rank builds from its
// observations is a partial sum -- the camera records, rhs / hdiag / gvec / acc of the assembly, the Schur part qs of
// every matvec and the model change.  The hook sums the assembly once per LM iteration (csrc/ba_solve.cu) and qs once per
// matvec (pcg_iteration); everything else in the CG is computed from summed data only.  Its scalars are sums over CTAs
// taken in a fixed order (reduce_fixed), so every rank forms the same bits, takes the same CG decisions and queues the
// same hook calls.  The single-GPU solve runs the same kernels without the hook.
#include <stddef.h>
#include <algorithm>
#include "ba_obs.h"
#include "ba_pcg.h"
#include "common.cuh"

namespace vgg {


__device__ __forceinline__ bool zero_or_inf(double v) { return v == 0.0 || isinf(v); }

// Sum of up to 3 per-thread values over the grid in a fixed order: each CTA adds its threads by warp shuffles and then
// its warps in index order into its own slots[K * blockIdx.x + k]; the CTA that finishes last adds the slots in CTA order
// into out[].  The bits depend on the inputs and the grid shape only, not on which CTA finishes first, so ranks holding
// the same data form the same sums.  Returns true in thread 0 of the last CTA, the only thread whose out[] is set.
template <int K>
__device__ bool reduce_fixed(const double (&v)[K], double* slots, unsigned* ticket, double (&out)[K]) {
  __shared__ double red[K][32];
  __shared__ bool last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const double s = warp_sum(v[k]);
    if (lane == 0) red[k][warp] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      double s = 0.0;
      for (int w = 0; w < nw; ++w) s += red[k][w];
      slots[(size_t)blockIdx.x * K + k] = s;
    }
    __threadfence();
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last || threadIdx.x != 0) return false;
  __threadfence();
#pragma unroll
  for (int k = 0; k < K; ++k) out[k] = 0.0;
  for (unsigned b = 0; b < gridDim.x; ++b)
#pragma unroll
    for (int k = 0; k < K; ++k) out[k] += __ldcg(slots + (size_t)b * K + k);
  *ticket = 0u;
  return true;
}
__device__ __forceinline__ void finish(double* cg, double term) {
  cg[CG_TERM] = term;
  cg[CG_DONE] = 1.0;
}

// ------------------------------------------------------------------------------------------------
// rhs = -g, hdiag = diag(H_cc), gvec = g (the entries of assemble_hc that the iterative solve needs)
__global__ void pcg_hc_kernel(int S, int dc, int ns, int KR, const double* __restrict__ camrec,
                              const double* __restrict__ shared_in, double* __restrict__ rhs,
                              double* __restrict__ hdiag, double* __restrict__ gvec) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < S * dc) {
    const double* rec = camrec + (size_t)(i / dc) * KR;
    const int a = i % dc;
    gvec[i] = rec[a];
    rhs[i] = -rec[a];
    hdiag[i] = rec[dc + a * dc - a * (a - 1) / 2];
  } else if (i < S * dc + ns) {
    const int j = i - S * dc;
    gvec[i] = shared_in[j];
    rhs[i] = -shared_in[j];
    hdiag[i] = shared_in[2 + (j == 0 ? 0 : 2)];
  }
}

// Preconditioner blocks: frame s has blocks 3 s (rotation), 3 s + 1 (translation), 3 s + 2 (per-frame intrinsics, empty
// otherwise); block 3 S holds the shared intrinsics.  Each block is 9 doubles (row-major 3x3).
__host__ __device__ __forceinline__ void pcg_block_rows(int b, int S, int dc, int ns, int* r0, int* nb) {
  if (b < 3 * S) {
    const int k = b % 3;
    *r0 = (b / 3) * dc + 3 * k;
    *nb = k < 2 ? 3 : dc - 6;
  } else {
    *r0 = S * dc;
    *nb = ns;
  }
}

// ------------------------------------------------------------------------------------------------
// One pass over the observations: rhs[row] += (Z q)[row] and acc[block] += sum_n Z_b Z_b^T (upper entries), Z = W M.
// Same CTA shape as z_build (ba_schur.cu): PJ_NT tracks per CTA, warps over the 32-frame groups, one lane per frame; a
// lane keeps its frame's sums in registers over the CTA's tracks and adds them once.
constexpr int PJ_NT = 8, PJ_W = 4;
template <int MODEL, int MODE, bool ROBUST>
__global__ void __launch_bounds__(PJ_W * 32) pcg_rhs_jacobi_kernel(
    int S, int N, const float* __restrict__ uv, const uint8_t* __restrict__ mask, const double* __restrict__ poses,
    const double* __restrict__ intr, const double* __restrict__ points, const uint8_t* __restrict__ point_const,
    const double* __restrict__ M, const double* __restrict__ q, double* __restrict__ rhs, double* __restrict__ acc,
    const int* __restrict__ fg_tracks, BaLoss loss) {
  using C = BlkCfg<MODEL, MODE>;
  constexpr int DC = C::DC, NS = C::NS;
  constexpr int NI = DC - 6, NIU = NI * (NI + 1) / 2;
  constexpr int NB = 12 + NIU;                              // upper entries of the frame's blocks: 6 + 6 + intrinsics
  __shared__ __align__(16) double s_cam[PJ_W][16 * 32];
  __shared__ double s_pt[PJ_NT][16];                        // X, Y, Z, constant flag | M (9) | q (3)
  __shared__ double s_ws[PJ_W][PJ_NT][3 * (NS > 0 ? NS : 1)];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n0 = blockIdx.x * PJ_NT, nt = min(PJ_NT, N - n0);
  const int ngroups = (S + 31) / 32;
  for (int e = threadIdx.x; e < PJ_NT * 16; e += blockDim.x) {
    const int t = e >> 4, k = e & 15, n = n0 + t;
    double v = 0.0;
    if (t < nt) {
      if (k < 3) v = points[(size_t)n * 3 + k];
      else if (k == 3) v = (point_const && point_const[n]) ? 1.0 : 0.0;
      else if (k < 13) v = M[(size_t)n * 9 + (k - 4)];
      else v = q[(size_t)n * 3 + (k - 13)];
    }
    s_pt[t][k] = v;
  }
  if (NS > 0)
    for (int e = threadIdx.x; e < PJ_W * PJ_NT * 3 * NS; e += blockDim.x) (&s_ws[0][0][0])[e] = 0.0;
  __syncthreads();
  double* pw = s_cam[warp];
  const float2* uv2 = reinterpret_cast<const float2*>(uv);
  for (int g = warp; g < ngroups; g += PJ_W) {
    if (fg_tracks && (n0 + nt <= fg_tracks[2 * g] || n0 >= fg_tracks[2 * g + 1])) continue;
    const int s = g * 32 + lane;
    const bool frame_ok = s < S;
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 12; ++i) pw[i * 32 + lane] = frame_ok ? poses[(size_t)s * 12 + i] : 0.0;
#pragma unroll
    for (int i = 0; i < 4; ++i) pw[(12 + i) * 32 + lane] = frame_ok ? intr[(size_t)s * 4 + i] : 0.0;
    __syncwarp();
    double zq[DC], ba[NB];
#pragma unroll
    for (int i = 0; i < DC; ++i) zq[i] = 0.0;
#pragma unroll
    for (int i = 0; i < NB; ++i) ba[i] = 0.0;
    bool any = false;
    for (int t = 0; t < nt; ++t) {
      const size_t o = (size_t)s * N + n0 + t;
      const bool valid = frame_ok && mask[o] != 0;
      if (!__any_sync(0xffffffffu, valid)) continue;
      any = any || valid;
      const float2 ob = frame_ok ? uv2[o] : make_float2(0.f, 0.f);
      const double* pt = s_pt[t];
      const double* m = pt + 4;
      double jc0[8], jc1[8], jx0[3], jx1[3], rx, ry, oc;
      obs_math<MODEL, ROBUST>(pw + lane, 32, pt[0], pt[1], pt[2], pt[3] != 0.0, ob.x, ob.y, valid, jc0, jc1, jx0, jx1,
                              rx, ry, loss, oc);
      double z[DC][3];
#pragma unroll
      for (int i = 0; i < DC; ++i) {
        const double w0 = w_entry(jc0, jc1, jx0, jx1, i, 0), w1 = w_entry(jc0, jc1, jx0, jx1, i, 1),
                     w2 = w_entry(jc0, jc1, jx0, jx1, i, 2);
        z[i][0] = w0 * m[0];
        z[i][1] = w0 * m[1] + w1 * m[4];
        z[i][2] = w0 * m[2] + w1 * m[5] + w2 * m[8];
        zq[i] += z[i][0] * m[9] + z[i][1] * m[10] + z[i][2] * m[11];
      }
      int k = 0;
#pragma unroll
      for (int blk = 0; blk < 3; ++blk) {
        const int r0 = 3 * blk, nb = blk < 2 ? 3 : NI;
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
          for (int c = a; c < 3; ++c)
            if (a < nb && c < nb) {
              ba[k] += z[r0 + a][0] * z[r0 + c][0] + z[r0 + a][1] * z[r0 + c][1] + z[r0 + a][2] * z[r0 + c][2];
              ++k;
            }
      }
      if (NS > 0) {
        double a8[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) a8[e] = e < 3 * NS ? w_entry(jc0, jc1, jx0, jx1, 6 + e / 3, e % 3) : 0.0;
        const double r = warp_reduce_scatter<8>(a8, lane);
        if (lane < 3 * NS) s_ws[warp][t][lane] += r;
      }
    }
    if (frame_ok && any) {
#pragma unroll
      for (int i = 0; i < DC; ++i)
        if (zq[i] != 0.0) atomicAdd(&rhs[(size_t)s * DC + i], zq[i]);
      int k = 0;
#pragma unroll
      for (int blk = 0; blk < 3; ++blk) {
        const int nb = blk < 2 ? 3 : NI;
        double* dst = acc + (size_t)(3 * s + blk) * 9;
#pragma unroll
        for (int a = 0; a < 3; ++a)
#pragma unroll
          for (int c = a; c < 3; ++c)
            if (a < nb && c < nb) {
              if (ba[k] != 0.0) atomicAdd(&dst[a * 3 + c], ba[k]);
              ++k;
            }
      }
    }
  }
  if (NS > 0) {
    __syncthreads();
    if ((int)threadIdx.x < nt) {
      const int t = threadIdx.x;
      const double* m = s_pt[t] + 4;
      double zs[NS > 0 ? NS : 1][3];
#pragma unroll
      for (int j = 0; j < NS; ++j) {
        double w[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          w[c] = 0.0;
#pragma unroll
          for (int v = 0; v < PJ_W; ++v) w[c] += s_ws[v][t][j * 3 + c];
        }
        zs[j][0] = w[0] * m[0];
        zs[j][1] = w[0] * m[1] + w[1] * m[4];
        zs[j][2] = w[0] * m[2] + w[1] * m[5] + w[2] * m[8];
        const double zqs = zs[j][0] * m[9] + zs[j][1] * m[10] + zs[j][2] * m[11];
        if (zqs != 0.0) atomicAdd(&rhs[(size_t)S * DC + j], zqs);
      }
      double* dst = acc + (size_t)(3 * S) * 9;
#pragma unroll
      for (int a = 0; a < NS; ++a)
#pragma unroll
        for (int c = a; c < NS; ++c) {
          const double v = zs[a][0] * zs[c][0] + zs[a][1] * zs[c][1] + zs[a][2] * zs[c][2];
          if (v != 0.0) atomicAdd(&dst[a * 3 + c], v);
        }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// entry (a, c) of the camera Hessian, a, c reduced-parameter rows
__device__ __forceinline__ double hcc_entry(int a, int c, int S, int dc, int ns, int KR, const double* camrec,
                                            const double* shared_in) {
  const int fa = a < S * dc ? a / dc : -1, fc = c < S * dc ? c / dc : -1;
  if (fa >= 0 && fc >= 0) {
    if (fa != fc) return 0.0;
    int i = a % dc, j = c % dc;
    if (i > j) { const int t = i; i = j; j = t; }
    return camrec[(size_t)fa * KR + dc + i * dc - i * (i - 1) / 2 + (j - i)];
  }
  if (fa < 0 && fc < 0) {
    int i = a - S * dc, j = c - S * dc;
    if (i > j) { const int t = i; i = j; j = t; }
    return shared_in[2 + (i == 0 ? j : 2)];
  }
  const int f = fa >= 0 ? fa : fc, i = (fa >= 0 ? a : c) % dc, j = (fa >= 0 ? c : a) - S * dc;
  return i < 6 ? camrec[(size_t)f * KR + dc + dc * (dc + 1) / 2 + i * ns + j] : 0.0;
}

// Per preconditioner block: A_bb = Dc (H_bb - acc_bb) Dc + damping, pinned rows identity, inverted through its
// Cholesky factor (a failed pivot fails the solve, as a failed factorisation does in the direct path); b = Dc rhs;
// x = 0, r = b, z = P r; rho = r.z and |b|^2 summed, and the last CTA starts the CG state.
__global__ void pcg_init_kernel(int S, int dc, int ns, int KR, const double* __restrict__ camrec,
                                const double* __restrict__ shared_in, const double* __restrict__ acc,
                                const double* __restrict__ rhs, const double* __restrict__ hdiag,
                                const double* __restrict__ sc, const uint8_t* __restrict__ pconst, double radius,
                                double min_diag, double max_diag, double* __restrict__ pinv, double* __restrict__ bvec,
                                double* __restrict__ x, double* __restrict__ r, double* __restrict__ z,
                                double* __restrict__ cg, double* __restrict__ slots) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  const int nblk = 3 * S + (ns > 0 ? 1 : 0);
  double part[3] = {0.0, 0.0, 0.0};       // r.z, |b|^2, failed blocks
  if (b < nblk) {
    int r0, nb;
    pcg_block_rows(b, S, dc, ns, &r0, &nb);
    double A[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    double bb[3] = {0, 0, 0};
    bool pin[3] = {true, true, true};
    for (int i = 0; i < nb; ++i) {
      pin[i] = pconst[r0 + i] != 0;
      bb[i] = pin[i] ? 0.0 : rhs[r0 + i] * sc[r0 + i];
    }
    for (int i = 0; i < nb; ++i)
      for (int j = 0; j < nb; ++j) {
        if (pin[i] || pin[j]) continue;
        const double ac = acc[(size_t)b * 9 + (i < j ? i * 3 + j : j * 3 + i)];
        double v = (hcc_entry(r0 + i, r0 + j, S, dc, ns, KR, camrec, shared_in) - ac) * sc[r0 + i] * sc[r0 + j];
        if (i == j) v += fmin(fmax(hdiag[r0 + i] * sc[r0 + i] * sc[r0 + i], min_diag), max_diag) / radius;
        A[i][j] = v;
      }
    // A = L L^T, then P = A^-1 = L^-T L^-1
    double L[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    bool bad = false;
    for (int j = 0; j < 3; ++j) {
      double d = A[j][j];
      for (int k = 0; k < j; ++k) d -= L[j][k] * L[j][k];
      bad = bad || !(d > 0.0);
      L[j][j] = sqrt(d);
      for (int i = j + 1; i < 3; ++i) {
        double v = A[i][j];
        for (int k = 0; k < j; ++k) v -= L[i][k] * L[j][k];
        L[i][j] = v / L[j][j];
      }
    }
    double Li[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    for (int i = 0; i < 3; ++i) {
      Li[i][i] = 1.0 / L[i][i];
      for (int j = 0; j < i; ++j) {
        double v = 0.0;
        for (int k = j; k < i; ++k) v -= L[i][k] * Li[k][j];
        Li[i][j] = v / L[i][i];
      }
    }
    double P[3][3];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        double v = 0.0;
        for (int k = (i > j ? i : j); k < 3; ++k) v += Li[k][i] * Li[k][j];
        P[i][j] = bad ? 0.0 : v;
      }
    for (int i = 0; i < 9; ++i) pinv[(size_t)b * 9 + i] = (&P[0][0])[i];
    for (int i = 0; i < nb; ++i) {
      double zi = 0.0;
      for (int j = 0; j < nb; ++j) zi += P[i][j] * bb[j];
      bvec[r0 + i] = bb[i];
      x[r0 + i] = 0.0;
      r[r0 + i] = bb[i];
      z[r0 + i] = zi;
      part[0] += bb[i] * zi;
      part[1] += bb[i] * bb[i];
    }
    part[2] = bad ? 1.0 : 0.0;
  }
  double sum[3];
  if (reduce_fixed<3>(part, slots, reinterpret_cast<unsigned*>(cg + CG_TICKET_SLOT), sum)) {
    const double rho = sum[0], bsq = sum[1], fails = sum[2];
    cg[CG_BB] = bsq;
    cg[CG_Q0] = 0.0;
    cg[CG_BETA] = 0.0;
    cg[CG_RHO] = rho;
    cg[CG_ZETA] = 0.0;
    cg[CG_RREL] = bsq > 0.0 ? 1.0 : 0.0;
    cg[CG_PRE_FAIL] = fails;
    cg[CG_ITERS] = 0.0;
    cg[CG_DONE] = 0.0;
    cg[CG_TERM] = -1.0;
    if (fails > 0.0) finish(cg, VGG_CG_FAILURE);                         // a preconditioner block is not positive definite
    else if (bsq == 0.0) finish(cg, VGG_CG_SUCCESS);                     // |b| = 0: x = 0
    else if (zero_or_inf(rho)) { cg[CG_ITERS] = 1.0; finish(cg, VGG_CG_FAILURE); }
  }
}

// ------------------------------------------------------------------------------------------------
// q = (camera-Hessian part of A) v, one thread per reduced-parameter row; the shared-intrinsics rows are sums over all
// frames and go to the extra last CTA.  pmode: v = z + beta p_old (beta = 0 on the first iteration, p_old zeroed), written
// to p_new; otherwise v = x (the residual reset).  u = Dc v with pinned entries zero goes to u for pcg_schur.
__device__ __forceinline__ double pcg_v(int k, bool pmode, const double* z, const double* p_old, const double* x,
                                        double beta) {
  return pmode ? z[k] + beta * p_old[k] : x[k];
}
__global__ void __launch_bounds__(256) pcg_hcc_kernel(int S, int dc, int ns, int KR, const double* __restrict__ camrec,
                                                      const double* __restrict__ shared_in,
                                                      const double* __restrict__ hdiag, const double* __restrict__ sc,
                                                      const uint8_t* __restrict__ pconst, double radius, double min_diag,
                                                      double max_diag, int pmode, const double* __restrict__ z,
                                                      const double* __restrict__ p_old, const double* __restrict__ x,
                                                      double* __restrict__ p_new, double* __restrict__ u,
                                                      double* __restrict__ q, double* __restrict__ qs,
                                                      const double* __restrict__ cg) {
  if (cg[CG_DONE] != 0.0) return;
  const double beta = cg[CG_BETA];
  const bool pm = pmode != 0;
  auto uval = [&](int k) { return pconst[k] ? 0.0 : sc[k] * pcg_v(k, pm, z, p_old, x, beta); };
  const int nrow = S * dc;
  const int frame_blocks = (nrow + 255) / 256;
  if ((int)blockIdx.x < frame_blocks) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= nrow) return;
    const int s = i / dc, a = i % dc;
    const double v = pcg_v(i, pm, z, p_old, x, beta);
    const double* rec = camrec + (size_t)s * KR;
    double y = 0.0;
    for (int c = 0; c < dc; ++c) {
      const int lo = a < c ? a : c, hi = a < c ? c : a;
      y += rec[dc + lo * dc - lo * (lo - 1) / 2 + (hi - lo)] * uval(s * dc + c);
    }
    if (a < 6)
      for (int j = 0; j < ns; ++j) y += rec[dc + dc * (dc + 1) / 2 + a * ns + j] * uval(nrow + j);
    const bool pin = pconst[i] != 0;
    const double damp = fmin(fmax(hdiag[i] * sc[i] * sc[i], min_diag), max_diag) / radius;
    if (pm) p_new[i] = v;
    u[i] = pin ? 0.0 : sc[i] * v;
    q[i] = pin ? v : sc[i] * y + damp * v;
    qs[i] = 0.0;
    return;
  }
  // shared-intrinsics rows: H_ss u_s + sum over frames of H_cs^T u_c
  double part[2] = {0.0, 0.0};
  for (int s = threadIdx.x; s < S; s += blockDim.x) {
    const double* rec = camrec + (size_t)s * KR + dc + dc * (dc + 1) / 2;
    for (int a = 0; a < 6; ++a) {
      const double ua = uval(s * dc + a);
      for (int j = 0; j < ns; ++j) part[j] += rec[a * ns + j] * ua;
    }
  }
  __shared__ double red[2][8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int j = 0; j < 2; ++j) {
    const double t = warp_sum(part[j]);
    if (lane == 0) red[j][warp] = t;
  }
  __syncthreads();
  if ((int)threadIdx.x < ns) {
    const int j = threadIdx.x, i = nrow + j;
    double y = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) y += red[j][w];
    for (int k = 0; k < ns; ++k) y += shared_in[2 + (j == 0 ? k : (k == 0 ? 1 : 2))] * uval(nrow + k);
    const double v = pcg_v(i, pm, z, p_old, x, beta);
    const bool pin = pconst[i] != 0;
    const double damp = fmin(fmax(hdiag[i] * sc[i] * sc[i], min_diag), max_diag) / radius;
    if (pm) p_new[i] = v;
    u[i] = pin ? 0.0 : sc[i] * v;
    q[i] = pin ? v : sc[i] * y + damp * v;
    qs[i] = 0.0;
  }
}

// qs[row] -= sc[row] (sum_n Z_n Z_n^T u)[row] for free rows (qs zeroed by pcg_hcc; q = its part + qs).  A CTA owns 32 tracks (one lane each); its warps take the
// frames in turn.  Pass 1 (as backsub): w_n = sum_s W_sn^T u_s; then t_n = M_n M_n^T w_n; pass 2: the frame's
// sum over the CTA's tracks of W_sn t_n, one warp reduce-scatter and one f64 RED per (CTA, frame parameter).
constexpr int PS_W = 16;
template <int MODEL, int MODE, bool ROBUST>
__global__ void __launch_bounds__(PS_W * 32) pcg_schur_kernel(
    int S, int N, const float* __restrict__ uv, const uint8_t* __restrict__ mask, const double* __restrict__ poses,
    const double* __restrict__ intr, const double* __restrict__ points, const uint8_t* __restrict__ point_const,
    const double* __restrict__ M, const double* __restrict__ sc, const uint8_t* __restrict__ pconst,
    const double* __restrict__ u, double* __restrict__ qs, const int* __restrict__ fg_tracks,
    const double* __restrict__ cg, BaLoss loss) {
  if (cg[CG_DONE] != 0.0) return;
  using C = BlkCfg<MODEL, MODE>;
  constexpr int DC = C::DC, NS = C::NS;
  __shared__ double s_cam[PS_W][16];
  __shared__ double s_acc[3][PS_W][32];
  __shared__ double s_t[3][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int nlo = blockIdx.x * 32, nhi = min(N, nlo + 32);
  const int n = nlo + lane;
  const bool track_ok = n < N;
  double X0 = 0.0, X1 = 0.0, X2 = 0.0;
  bool pc = true;
  if (track_ok) {
    X0 = points[(size_t)n * 3]; X1 = points[(size_t)n * 3 + 1]; X2 = points[(size_t)n * 3 + 2];
    pc = point_const && point_const[n] != 0;
  }
  double ush[2] = {0.0, 0.0};
#pragma unroll
  for (int j = 0; j < NS; ++j) ush[j] = u[(size_t)S * DC + j];
  const float2* uv2 = reinterpret_cast<const float2*>(uv);
  double* cam = s_cam[warp];
  auto skip = [&](int s) { return fg_tracks && (nhi <= fg_tracks[2 * (s >> 5)] || nlo >= fg_tracks[2 * (s >> 5) + 1]); };
  // ---- pass 1: w = sum_s W^T u_s
  double w0 = 0.0, w1 = 0.0, w2 = 0.0;
  for (int s = warp; s < S; s += nw) {
    if (skip(s)) continue;
    const size_t o = (size_t)s * N + n;
    const bool valid = track_ok && mask[o] != 0;
    if (!__any_sync(0xffffffffu, valid)) continue;
    const float2 ob = valid ? uv2[o] : make_float2(0.f, 0.f);
    __syncwarp();
    if (lane < 16) cam[lane] = lane < 12 ? poses[(size_t)s * 12 + lane] : intr[(size_t)s * 4 + (lane - 12)];
    __syncwarp();
    double jc0[8], jc1[8], jx0[3], jx1[3], rx, ry, oc;
    obs_math<MODEL, ROBUST>(cam, 1, X0, X1, X2, pc, ob.x, ob.y, valid, jc0, jc1, jx0, jx1, rx, ry, loss, oc);
    const double* d = u + (size_t)s * DC;
#pragma unroll
    for (int i = 0; i < DC; ++i) {
      const double di = __ldg(d + i);
      w0 = fma(w_entry(jc0, jc1, jx0, jx1, i, 0), di, w0);
      w1 = fma(w_entry(jc0, jc1, jx0, jx1, i, 1), di, w1);
      w2 = fma(w_entry(jc0, jc1, jx0, jx1, i, 2), di, w2);
    }
#pragma unroll
    for (int j = 0; j < NS; ++j) {
      w0 = fma(w_entry(jc0, jc1, jx0, jx1, 6 + j, 0), ush[j], w0);
      w1 = fma(w_entry(jc0, jc1, jx0, jx1, 6 + j, 1), ush[j], w1);
      w2 = fma(w_entry(jc0, jc1, jx0, jx1, 6 + j, 2), ush[j], w2);
    }
  }
  s_acc[0][warp][lane] = w0;
  s_acc[1][warp][lane] = w1;
  s_acc[2][warp][lane] = w2;
  __syncthreads();
  // ---- t = M M^T w per track (M upper triangular, row-major; zero for constant points)
  if (threadIdx.x < 32) {
    const int t = threadIdx.x;
    double a0 = 0.0, a1 = 0.0, a2 = 0.0;
    for (int v = 0; v < nw; ++v) {
      a0 += s_acc[0][v][t];
      a1 += s_acc[1][v][t];
      a2 += s_acc[2][v][t];
    }
    double t0 = 0.0, t1 = 0.0, t2 = 0.0;
    if (nlo + t < N && !(point_const && point_const[nlo + t])) {
      const double* m = M + (size_t)(nlo + t) * 9;
      const double y0 = m[0] * a0;
      const double y1 = m[1] * a0 + m[4] * a1;
      const double y2 = m[2] * a0 + m[5] * a1 + m[8] * a2;
      t0 = m[0] * y0 + m[1] * y1 + m[2] * y2;
      t1 = m[4] * y1 + m[5] * y2;
      t2 = m[8] * y2;
    }
    s_t[0][t] = t0;
    s_t[1][t] = t1;
    s_t[2][t] = t2;
  }
  __syncthreads();
  const double t0 = s_t[0][lane], t1 = s_t[1][lane], t2 = s_t[2][lane];
  // ---- pass 2: q_s -= Dc sum_n W_sn t_n
  double vsh[2] = {0.0, 0.0};
  for (int s = warp; s < S; s += nw) {
    if (skip(s)) continue;
    const size_t o = (size_t)s * N + n;
    const bool valid = track_ok && mask[o] != 0;
    if (!__any_sync(0xffffffffu, valid)) continue;
    const float2 ob = valid ? uv2[o] : make_float2(0.f, 0.f);
    __syncwarp();
    if (lane < 16) cam[lane] = lane < 12 ? poses[(size_t)s * 12 + lane] : intr[(size_t)s * 4 + (lane - 12)];
    __syncwarp();
    double jc0[8], jc1[8], jx0[3], jx1[3], rx, ry, oc;
    obs_math<MODEL, ROBUST>(cam, 1, X0, X1, X2, pc, ob.x, ob.y, valid, jc0, jc1, jx0, jx1, rx, ry, loss, oc);
    double a8[8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
      a8[i] = i < DC ? w_entry(jc0, jc1, jx0, jx1, i, 0) * t0 + w_entry(jc0, jc1, jx0, jx1, i, 1) * t1 +
                           w_entry(jc0, jc1, jx0, jx1, i, 2) * t2
                     : 0.0;
#pragma unroll
    for (int j = 0; j < NS; ++j)
      vsh[j] += w_entry(jc0, jc1, jx0, jx1, 6 + j, 0) * t0 + w_entry(jc0, jc1, jx0, jx1, 6 + j, 1) * t1 +
                w_entry(jc0, jc1, jx0, jx1, 6 + j, 2) * t2;
    const double r = warp_reduce_scatter<8>(a8, lane);
    if (lane < DC) {
      const size_t row = (size_t)s * DC + lane;
      if (!pconst[row] && r != 0.0) atomicAdd(&qs[row], -sc[row] * r);
    }
  }
  if (NS > 0) {
    __syncthreads();
#pragma unroll
    for (int j = 0; j < NS; ++j) {
      const double v = warp_sum(vsh[j]);
      if (lane == 0) s_acc[j][warp][0] = v;
    }
    __syncthreads();
    if ((int)threadIdx.x < NS) {
      const int j = threadIdx.x;
      double v = 0.0;
      for (int k = 0; k < nw; ++k) v += s_acc[j][k][0];
      const size_t row = (size_t)S * DC + j;
      if (!pconst[row] && v != 0.0) atomicAdd(&qs[row], -sc[row] * v);
    }
  }
}

// q += qs (the matvec's Schur part, summed over the ranks); pq = p.q; alpha = rho / pq.  p'q <= 0 (indefinite), an
// infinite p'q, or a zero or infinite alpha fail the solve.
__global__ void __launch_bounds__(256) pcg_alpha_kernel(int D, const double* __restrict__ p, double* __restrict__ q,
                                                        const double* __restrict__ qs, double* __restrict__ cg,
                                                        double* __restrict__ slots) {
  if (cg[CG_DONE] != 0.0) return;
  double part[1] = {0.0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < D; i += gridDim.x * blockDim.x) {
    const double qi = q[i] + qs[i];
    q[i] = qi;
    part[0] += p[i] * qi;
  }
  double sum[1];
  if (reduce_fixed<1>(part, slots, reinterpret_cast<unsigned*>(cg + CG_TICKET_SLOT), sum)) {
    const double pq = sum[0];
    const double alpha = cg[CG_RHO] / pq;
    cg[CG_ALPHA] = alpha;
    if (pq <= 0.0 || isinf(pq) || zero_or_inf(alpha)) {
      cg[CG_ITERS] += 1.0;
      finish(cg, VGG_CG_FAILURE);
    }
  }
}

// x += alpha p (the residual-reset iteration, before q = A x)
__global__ void pcg_xstep_kernel(int D, const double* __restrict__ p, double* __restrict__ x,
                                 const double* __restrict__ cg) {
  if (cg[CG_DONE] != 0.0) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < D) x[i] += cg[CG_ALPHA] * p[i];
}

// End of CG iteration i, one thread per preconditioner block: x += alpha p, r -= alpha q (reset: x already stepped,
// r = b - q with q = A x, its Schur part still in qs); z = P r; the last CTA forms Q1 = -x.(b + r), zeta = i (Q1 - Q0) / Q1 and the next rho and beta,
// in Ceres' order: zeta < eta with i >= min succeeds, then i >= max stops without convergence, then a zero or infinite
// rho or beta of iteration i + 1 fails.
__global__ void __launch_bounds__(256) pcg_update_kernel(int S, int dc, int ns, int reset, const double* __restrict__ pinv,
                                                         const double* __restrict__ bvec, const double* __restrict__ p,
                                                         const double* __restrict__ q, const double* __restrict__ qs,
                                                         double* __restrict__ x, double* __restrict__ r,
                                                         double* __restrict__ z, double eta, int min_it, int max_it,
                                                         double* __restrict__ cg, double* __restrict__ slots) {
  if (cg[CG_DONE] != 0.0) return;
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  const int nblk = 3 * S + (ns > 0 ? 1 : 0);
  const double alpha = cg[CG_ALPHA];
  double part[3] = {0.0, 0.0, 0.0};     // r.z, -x.(b + r), |r|^2
  if (b < nblk) {
    int r0, nb;
    pcg_block_rows(b, S, dc, ns, &r0, &nb);
    double rr[3] = {0, 0, 0};
    for (int i = 0; i < nb; ++i) {
      const int k = r0 + i;
      double xi = x[k], ri;
      if (reset) {
        ri = bvec[k] - (q[k] + qs[k]);
      } else {
        xi += alpha * p[k];
        x[k] = xi;
        ri = r[k] - alpha * q[k];
      }
      r[k] = ri;
      rr[i] = ri;
      part[1] -= xi * (bvec[k] + ri);
      part[2] += ri * ri;
    }
    const double* P = pinv + (size_t)b * 9;
    for (int i = 0; i < nb; ++i) {
      double zi = 0.0;
      for (int j = 0; j < nb; ++j) zi += P[i * 3 + j] * rr[j];
      z[r0 + i] = zi;
      part[0] += rr[i] * zi;
    }
  }
  double sum[3];
  if (reduce_fixed<3>(part, slots, reinterpret_cast<unsigned*>(cg + CG_TICKET_SLOT), sum)) {
    const double rho = sum[0], Q1 = sum[1], rsq = sum[2];
    const double i = cg[CG_ITERS] + 1.0;
    cg[CG_ITERS] = i;
    const double zeta = i * (Q1 - cg[CG_Q0]) / Q1;
    cg[CG_ZETA] = zeta;
    cg[CG_RREL] = sqrt(rsq / cg[CG_BB]);
    if (zeta < eta && i >= (double)min_it) {
      finish(cg, VGG_CG_SUCCESS);
      return;
    }
    cg[CG_Q0] = Q1;
    if (i >= (double)max_it) {
      finish(cg, VGG_CG_NO_CONVERGENCE);
      return;
    }
    const double beta = rho / cg[CG_RHO];
    if (zero_or_inf(rho) || zero_or_inf(beta)) {
      cg[CG_ITERS] = i + 1.0;
      finish(cg, VGG_CG_FAILURE);
      return;
    }
    cg[CG_RHO] = rho;
    cg[CG_BETA] = beta;
  }
}

// ------------------------------------------------------------------------------------------------
// Ceres' model change of a step: -(J d)^T (f + J d / 2) summed over the observations, d = (d_c, d_p) unscaled; d_p is
// recomputed from M, g_p and wacc with point_step's arithmetic (bit for bit the step the candidate took).  One lane per
// track, warps over the frames, as backsub.  With track shards this is the rank's part, summed with the candidate's cost.
template <int MODEL, int MODE, bool ROBUST>
__global__ void __launch_bounds__(PS_W * 32) pcg_model_change_kernel(
    int S, int N, const float* __restrict__ uv, const uint8_t* __restrict__ mask, const double* __restrict__ poses,
    const double* __restrict__ intr, const double* __restrict__ points, const uint8_t* __restrict__ point_const,
    const double* __restrict__ M, const double* __restrict__ g_p, const double* __restrict__ wacc,
    const double* __restrict__ d_c, const int* __restrict__ fg_tracks, double* __restrict__ out, BaLoss loss) {
  using C = BlkCfg<MODEL, MODE>;
  constexpr int DC = C::DC, NS = C::NS;
  __shared__ double s_cam[PS_W][16];
  __shared__ double s_red[PS_W];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int nlo = blockIdx.x * 32, nhi = min(N, nlo + 32);
  const int n = nlo + lane;
  const bool track_ok = n < N;
  double X0 = 0.0, X1 = 0.0, X2 = 0.0, d0 = 0.0, d1 = 0.0, d2 = 0.0;
  bool pc = true;
  if (track_ok) {
    X0 = points[(size_t)n * 3]; X1 = points[(size_t)n * 3 + 1]; X2 = points[(size_t)n * 3 + 2];
    pc = point_const && point_const[n] != 0;
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
  }
  double dsh[2] = {0.0, 0.0};
#pragma unroll
  for (int j = 0; j < NS; ++j) dsh[j] = d_c[(size_t)S * DC + j];
  const float2* uv2 = reinterpret_cast<const float2*>(uv);
  double* cam = s_cam[warp];
  double accm = 0.0;
  for (int s = warp; s < S; s += nw) {
    if (fg_tracks && (nhi <= fg_tracks[2 * (s >> 5)] || nlo >= fg_tracks[2 * (s >> 5) + 1])) continue;
    const size_t o = (size_t)s * N + n;
    const bool valid = track_ok && mask[o] != 0;
    if (!__any_sync(0xffffffffu, valid)) continue;
    const float2 ob = valid ? uv2[o] : make_float2(0.f, 0.f);
    __syncwarp();
    if (lane < 16) cam[lane] = lane < 12 ? poses[(size_t)s * 12 + lane] : intr[(size_t)s * 4 + (lane - 12)];
    __syncwarp();
    double jc0[8], jc1[8], jx0[3], jx1[3], rx, ry, oc;
    obs_math<MODEL, ROBUST>(cam, 1, X0, X1, X2, pc, ob.x, ob.y, valid, jc0, jc1, jx0, jx1, rx, ry, loss, oc);
    if (!valid) continue;
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
  accm = warp_sum(accm);
  if (lane == 0) s_red[warp] = accm;
  __syncthreads();
  if (threadIdx.x == 0) {
    double v = 0.0;
    for (int k = 0; k < nw; ++k) v += s_red[k];
    if (v != 0.0) atomicAdd(out, v);
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
int pcg_blocks(int S, int ns) { return 3 * S + (ns > 0 ? 1 : 0); }

// K partials per CTA of the fixed-order reductions: 3 per CTA of pcg_init / pcg_update, 1 per CTA of pcg_alpha
static int pcg_alpha_ctas(int D) { return std::min(132, (D + 255) / 256); }
size_t pcg_slot_doubles(int S, int dc, int ns) {
  return (size_t)std::max(3 * ((pcg_blocks(S, ns) + 255) / 256), pcg_alpha_ctas(S * dc + ns));
}

int launch_pcg_assemble(const PcgOp& op, const double* q, const PcgBuffers& B, cudaStream_t st) {
  const vgg_ba_problem* p = op.p;
  const int D = p->S * op.dc + op.ns;
  VGG_CUDA_CHECK(cudaMemsetAsync(B.acc, 0, sizeof(double) * 9 * (size_t)pcg_blocks(p->S, op.ns), st));
  pcg_hc_kernel<<<(D + 255) / 256, 256, 0, st>>>(p->S, op.dc, op.ns, op.KR, op.camrec, op.shared_in, B.rhs, B.hdiag, B.gvec);
  VGG_LAUNCH_CHECK();
  if (op.obs) return launch_list_rhs_jacobi(op, q, B, st);
  VGG_PICK_BA_KERNEL(kern, pcg_rhs_jacobi_kernel, p);
  const int nw = std::min(PJ_W, (p->S + 31) / 32);
  kern<<<(p->N + PJ_NT - 1) / PJ_NT, nw * 32, 0, st>>>(p->S, p->N, p->uv, p->mask, p->poses, p->intr, p->points,
                                                        p->point_const, op.M, q, B.rhs, B.acc, op.fg_tracks, ba_loss_of(p));
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

int launch_pcg_init(const PcgOp& op, const PcgBuffers& B, double* bvec, cudaStream_t st) {
  const int S = op.p->S, nblk = pcg_blocks(S, op.ns);
  VGG_CUDA_CHECK(cudaMemsetAsync(B.cg, 0, sizeof(double) * PCG_STATE_DOUBLES, st));
  pcg_init_kernel<<<(nblk + 255) / 256, 256, 0, st>>>(S, op.dc, op.ns, op.KR, op.camrec, op.shared_in, B.acc, B.rhs,
                                                      B.hdiag, op.sc_c, op.p->param_const, op.radius, op.min_diag,
                                                      op.max_diag, B.pinv, bvec, B.x, B.r, B.z, B.cg, B.slots);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

// q = A v (pmode: v = z + beta p_old, stored to p_new; otherwise v = x)
int launch_pcg_matvec(const PcgOp& op, int pmode, const double* p_old, double* p_new, const PcgBuffers& B,
                      cudaStream_t st) {
  const vgg_ba_problem* p = op.p;
  const int nrow = p->S * op.dc;
  pcg_hcc_kernel<<<(nrow + 255) / 256 + (op.ns > 0 ? 1 : 0), 256, 0, st>>>(
      p->S, op.dc, op.ns, op.KR, op.camrec, op.shared_in, B.hdiag, op.sc_c, p->param_const, op.radius, op.min_diag,
      op.max_diag, pmode, B.z, p_old, B.x, p_new, B.u, B.q, B.qs, B.cg);
  VGG_LAUNCH_CHECK();
  if (op.obs) return launch_list_schur(op, B, st);
  VGG_PICK_BA_KERNEL(kern, pcg_schur_kernel, p);
  const int nw = std::min(PS_W, p->S);
  kern<<<(p->N + 31) / 32, nw * 32, 0, st>>>(p->S, p->N, p->uv, p->mask, p->poses, p->intr, p->points, p->point_const,
                                             op.M, op.sc_c, p->param_const, B.u, B.qs, op.fg_tracks, B.cg,
                                             ba_loss_of(p));
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

// q += qs outside the CG (vgg_dev_pcg_probe: the whole product of one matvec)
__global__ void pcg_combine_kernel(int D, double* __restrict__ q, const double* __restrict__ qs) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < D) q[i] += qs[i];
}
int launch_pcg_combine(int D, double* q, const double* qs, cudaStream_t st) {
  pcg_combine_kernel<<<(D + 255) / 256, 256, 0, st>>>(D, q, qs);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

// One CG iteration i (1-based); iteration i reads p[(i + 1) & 1] and writes p[i & 1].  With track shards, the Schur
// part qs of each matvec is summed over the ranks before pcg_alpha (or pcg_update after the reset) adds it to q: one
// reduction per iteration, two on the reset iteration.
static int pcg_iteration(const PcgOp& op, const vgg_ba_linear_solver& lin, const PcgBuffers& B, double* bvec,
                         const Ranks& ranks, int i, cudaStream_t st) {
  int rc;
  const int S = op.p->S, D = S * op.dc + op.ns;
  const int nblk = pcg_blocks(S, op.ns);
  double* p_new = B.p[i & 1];
  const double* p_old = B.p[(i + 1) & 1];
  if ((rc = launch_pcg_matvec(op, 1, p_old, p_new, B, st))) return rc;
  if ((rc = ranks.sum(B.qs, (size_t)D))) return rc;
  pcg_alpha_kernel<<<pcg_alpha_ctas(D), 256, 0, st>>>(D, p_new, B.q, B.qs, B.cg, B.slots);
  VGG_LAUNCH_CHECK();
  const bool reset = i % PCG_RESET_PERIOD == 0;
  if (reset) {
    pcg_xstep_kernel<<<(D + 255) / 256, 256, 0, st>>>(D, p_new, B.x, B.cg);
    VGG_LAUNCH_CHECK();
    if ((rc = launch_pcg_matvec(op, 0, nullptr, nullptr, B, st))) return rc;
    if ((rc = ranks.sum(B.qs, (size_t)D))) return rc;
  }
  pcg_update_kernel<<<(nblk + 255) / 256, 256, 0, st>>>(S, op.dc, op.ns, reset ? 1 : 0, B.pinv, bvec, p_new, B.q, B.qs,
                                                        B.x, B.r, B.z, lin.eta, lin.min_linear_solver_iterations,
                                                        lin.max_linear_solver_iterations, B.cg, B.slots);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

// The CG loop after launch_pcg_init: chunks of PCG_CHUNK iterations; the done flag of chunk c is copied to the host
// behind it and read only after chunk c + 1 has been queued, so the GPU does not wait for the host between chunks.
// Iterations past the end are kernels that return at once (and reductions of a vector nobody reads: the done flag is
// the same on every rank, so every rank queues the same chunks).  The solution is B.x.
int pcg_run(const PcgOp& op, const vgg_ba_linear_solver& lin, const PcgBuffers& B, double* bvec, const Ranks& ranks,
            cudaStream_t st) {
  static thread_local double* h_flag = nullptr;
  static thread_local cudaEvent_t ev[2] = {nullptr, nullptr};
  if (!h_flag) {
    VGG_CUDA_CHECK(cudaHostAlloc(reinterpret_cast<void**>(&h_flag), sizeof(double) * 2, cudaHostAllocDefault));
    VGG_CUDA_CHECK(cudaEventCreateWithFlags(&ev[0], cudaEventDisableTiming));
    VGG_CUDA_CHECK(cudaEventCreateWithFlags(&ev[1], cudaEventDisableTiming));
  }
  const size_t D = (size_t)(op.p->S * op.dc + op.ns);
  VGG_CUDA_CHECK(cudaMemsetAsync(B.p[0], 0, sizeof(double) * D, st));
  VGG_CUDA_CHECK(cudaMemsetAsync(B.p[1], 0, sizeof(double) * D, st));
  // Ceres' loop runs its first iteration before it tests max_num_iterations
  const int max_it = std::max(1, lin.max_linear_solver_iterations);
  const int nchunks = (max_it + PCG_CHUNK - 1) / PCG_CHUNK;
  int rc;
  auto queue_chunk = [&](int c) -> int {
    for (int j = 1; j <= PCG_CHUNK; ++j)
      if ((rc = pcg_iteration(op, lin, B, bvec, ranks, c * PCG_CHUNK + j, st))) return rc;
    VGG_CUDA_CHECK(cudaMemcpyAsync(h_flag + (c & 1), B.cg + CG_DONE, sizeof(double), cudaMemcpyDeviceToHost, st));
    VGG_CUDA_CHECK(cudaEventRecord(ev[c & 1], st));
    return VGG_OK;
  };
  if ((rc = queue_chunk(0))) return rc;
  for (int c = 0; c < nchunks; ++c) {
    if (c + 1 < nchunks && (rc = queue_chunk(c + 1))) return rc;
    VGG_CUDA_CHECK(cudaEventSynchronize(ev[c & 1]));
    if (h_flag[c & 1] != 0.0) break;
  }
  return VGG_OK;
}

int launch_pcg_model_change(const vgg_ba_problem* p, const double* M, const double* g_p, const double* wacc,
                            const double* d_c, const int* fg_tracks, double* out, cudaStream_t st) {
  VGG_PICK_BA_KERNEL(kern, pcg_model_change_kernel, p);
  const int nw = std::min(PS_W, p->S);
  VGG_CUDA_CHECK(cudaMemsetAsync(out, 0, sizeof(double), st));
  kern<<<(p->N + 31) / 32, nw * 32, 0, st>>>(p->S, p->N, p->uv, p->mask, p->poses, p->intr, p->points, p->point_const,
                                             M, g_p, wacc, d_c, fg_tracks, out, ba_loss_of(p));
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

}  // namespace vgg
