// Schur-complement reduce, reduced-system preparation and back-substitution kernels.
//
// Replaces the Ceres SchurEliminator + DENSE_SCHUR/SPARSE_SCHUR Cholesky that
// pycolmap.bundle_adjustment runs on the host (vggsfm/utils/triangulation.py:1050,1142).
//
//   point_prep      per point: V = Dp H_pp Dp + diag(clamp(diag))/radius, 3x3 Cholesky,
//                   M = Dp L^-T, q = M^T g_p
//   assemble_hc     camera Hessian/gradient from the per-frame records into the dense reduced system
//   z_build         Zt[3n+c][row] = (W[n][row][:] M_n)[c]   (k-major operand for the SYRK), W rebuilt per observation,
//                   rhs[row] += Z[row] . q
//   syrk_f64        Sraw -= Zt^T Zt on the upper 128x128 tiles, mirrored into the lower triangle: FP64 tensor cores
//                   (DMMA 16x8x16), bulk-copy/mbarrier ring, persistent over a k-split work list, f64 RED epilogue
//   scale_damp      A = Dc Sraw Dc + diag(clamp(diag(Dc Hcc Dc)))/radius, constant parameters pinned
//   cam_step / backsub_partial / point_step / cam_update   back-substitution and the candidate state
#include <stddef.h>
#include <algorithm>
#include <vector>
#include "ba_lm.h"
#include "ba_obs.h"
#include "common.cuh"
#include "dev_probes.h"
#include "syrk_work.h"

namespace vgg {

// Add v to one element of the reduced-system buffer.  Single GPU: plain f64 RED on the local copy.  Track-sharded
// multi-GPU ("fabric" mode): ONE multimem reduction on the NVSwitch multicast address, which lands the addend in every
// rank's copy of the buffer -- the all-reduce of the reduced camera system happens inside the kernels that
// produce it (assemble, z_build, SYRK epilogue), tile by tile, instead of in a separate NCCL call afterwards.
__device__ __forceinline__ void ar_add(double* local, double* mc, double v) {
  if (mc) asm volatile("multimem.red.relaxed.sys.global.add.f64 [%0], %1;" ::"l"(mc), "d"(v) : "memory");
  else atomicAdd(local, v);
}
__device__ __forceinline__ void ar_put(double* local, double* mc, double v) {   // buffer is zero beforehand
  if (mc) asm volatile("multimem.red.relaxed.sys.global.add.f64 [%0], %1;" ::"l"(mc), "d"(v) : "memory");
  else *local = v;
}

// ------------------------------------------------------------------------------------------------
__global__ void jacobi_scale_points_kernel(int N, const double* __restrict__ H_pp, double* __restrict__ sc_p, int enable) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const double* h = H_pp + (size_t)n * 6;
  sc_p[n * 3 + 0] = enable ? 1.0 / (1.0 + sqrt(h[0])) : 1.0;
  sc_p[n * 3 + 1] = enable ? 1.0 / (1.0 + sqrt(h[3])) : 1.0;
  sc_p[n * 3 + 2] = enable ? 1.0 / (1.0 + sqrt(h[5])) : 1.0;
}

__global__ void jacobi_scale_cams_kernel(int D, const double* __restrict__ hdiag, double* __restrict__ sc_c, int enable) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D) return;
  sc_c[i] = enable ? 1.0 / (1.0 + sqrt(hdiag[i])) : 1.0;
}

// ------------------------------------------------------------------------------------------------
// per point: M (3x3 row-major) = Dp L^-T, q = M^T g_p, dpp = clamped scaled diagonal
__global__ void point_prep_kernel(int N, const double* __restrict__ H_pp, const double* __restrict__ g_p,
                                  const double* __restrict__ sc_p, const uint8_t* __restrict__ point_const,
                                  double radius, double min_diag, double max_diag, double* __restrict__ M,
                                  double* __restrict__ q, double* __restrict__ dpp, double* __restrict__ scal) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  double* Mo = M + (size_t)n * 9;
  if (point_const && point_const[n]) {
#pragma unroll
    for (int i = 0; i < 9; ++i) Mo[i] = 0.0;
    q[n * 3] = q[n * 3 + 1] = q[n * 3 + 2] = 0.0;
    dpp[n * 3] = dpp[n * 3 + 1] = dpp[n * 3 + 2] = 0.0;
    return;
  }
  const double* h = H_pp + (size_t)n * 6;
  const double s0 = sc_p[n * 3], s1 = sc_p[n * 3 + 1], s2 = sc_p[n * 3 + 2];
  double v00 = h[0] * s0 * s0, v01 = h[1] * s0 * s1, v02 = h[2] * s0 * s2;
  double v11 = h[3] * s1 * s1, v12 = h[4] * s1 * s2, v22 = h[5] * s2 * s2;
  const double d0 = fmin(fmax(v00, min_diag), max_diag);
  const double d1 = fmin(fmax(v11, min_diag), max_diag);
  const double d2 = fmin(fmax(v22, min_diag), max_diag);
  dpp[n * 3] = d0; dpp[n * 3 + 1] = d1; dpp[n * 3 + 2] = d2;
  v00 += d0 / radius; v11 += d1 / radius; v22 += d2 / radius;
  // Cholesky V = L L^T
  bool bad = !(v00 > 0.0);
  const double l00 = sqrt(v00);
  const double l10 = v01 / l00, l20 = v02 / l00;
  const double t11 = v11 - l10 * l10;
  bad = bad || !(t11 > 0.0);
  const double l11 = sqrt(t11);
  const double l21 = (v12 - l20 * l10) / l11;
  const double t22 = v22 - l20 * l20 - l21 * l21;
  bad = bad || !(t22 > 0.0);
  const double l22 = sqrt(t22);
  if (bad) {
    atomicAdd(&scal[SCAL_PT_FAIL], 1.0);
#pragma unroll
    for (int i = 0; i < 9; ++i) Mo[i] = 0.0;
    q[n * 3] = q[n * 3 + 1] = q[n * 3 + 2] = 0.0;
    return;
  }
  // Linv (lower)
  const double i00 = 1.0 / l00, i11 = 1.0 / l11, i22 = 1.0 / l22;
  const double i10 = -l10 * i00 * i11;
  const double i21 = -l21 * i11 * i22;
  const double i20 = -(l20 * i00 + l21 * i10) * i22;
  // M = Dp Linv^T : M[r][c] = s_r * Linv[c][r]
  const double m00 = s0 * i00, m01 = s0 * i10, m02 = s0 * i20;
  const double m11 = s1 * i11, m12 = s1 * i21;
  const double m22 = s2 * i22;
  Mo[0] = m00; Mo[1] = m01; Mo[2] = m02;
  Mo[3] = 0.0; Mo[4] = m11; Mo[5] = m12;
  Mo[6] = 0.0; Mo[7] = 0.0; Mo[8] = m22;
  const double g0 = g_p[n * 3], g1 = g_p[n * 3 + 1], g2 = g_p[n * 3 + 2];
  q[n * 3 + 0] = m00 * g0;
  q[n * 3 + 1] = m01 * g0 + m11 * g1;
  q[n * 3 + 2] = m02 * g0 + m12 * g1 + m22 * g2;
}

// ------------------------------------------------------------------------------------------------
// camera records -> dense reduced system (both triangles of the diagonal blocks and borders),
// rhs = -g, hdiag, gvec.  One CTA per frame, plus one for the shared-intrinsics block.
__global__ void assemble_hc_kernel(int S, int dc, int ns, int KR, int Dpad, const double* __restrict__ camrec,
                                   const double* __restrict__ shared_in, double* __restrict__ Sraw,
                                   double* __restrict__ rhs, double* __restrict__ hdiag, double* __restrict__ gvec,
                                   ptrdiff_t mc_off) {
  const int s = blockIdx.x;
  const int tid = threadIdx.x;
#define VGG_PUT(ptr, val) ar_put((ptr), mc_off ? (ptr) + mc_off : nullptr, (val))
  if (s < S) {
    const double* rec = camrec + (size_t)s * KR;
    const int base = s * dc;
    if (tid < dc) {
      VGG_PUT(&gvec[base + tid], rec[tid]);
      VGG_PUT(&rhs[base + tid], -rec[tid]);
    }
    if (tid < dc * dc) {
      const int i = tid / dc, j = tid % dc;
      const int a = i < j ? i : j, b = i < j ? j : i;
      const int idx = dc + a * dc - a * (a - 1) / 2 + (b - a);
      const double val = rec[idx];
      VGG_PUT(&Sraw[(size_t)(base + i) * Dpad + base + j], val);
      if (i == j) VGG_PUT(&hdiag[base + i], val);
    }
    if (tid < 6 * ns) {
      const int i = tid / ns, j = tid % ns;
      const double val = rec[dc + dc * (dc + 1) / 2 + tid];
      VGG_PUT(&Sraw[(size_t)(S * dc + j) * Dpad + base + i], val);
      VGG_PUT(&Sraw[(size_t)(base + i) * Dpad + S * dc + j], val);
    }
  } else if (ns > 0) {
    const int base = S * dc;
    if (tid < ns) {
      VGG_PUT(&gvec[base + tid], shared_in[tid]);
      VGG_PUT(&rhs[base + tid], -shared_in[tid]);
    }
    if (tid < ns * ns) {
      const int i = tid / ns, j = tid % ns;
      const int a = i < j ? i : j, b = i < j ? j : i;
      const double val = shared_in[2 + (a == 0 ? b : 2)];
      VGG_PUT(&Sraw[(size_t)(base + i) * Dpad + base + j], val);
      if (i == j) VGG_PUT(&hdiag[base + i], val);
    }
  }
#undef VGG_PUT
}

// ------------------------------------------------------------------------------------------------
// Schur operand straight from the observations: Zt[(3n+c)*Dpad + s*dc+i] = (W_sn M_n)[i][c], W_sn = J_c^T J_p of
// observation (s, n) rebuilt by obs_math (ba_obs.h) -- no stored coupling blocks -- and rhs[row] += sum_{n,c} Z q.
// A CTA owns ZB_NT tracks and all frames; its warps take the 32-frame groups in turn, one lane per frame, so the blocks
// of one (track, group) are 32*dc contiguous doubles of each of the three Zt rows: staged in shared memory, written
// with 16-byte stores.  A lane reads the ZB_NT observations of its frame, 8 B each and consecutive in uv, so every
// sector it pulls from HBM is used whole.  The shared-intrinsics columns are sums over all frames: each warp reduces
// its groups' share per track, the CTA adds the warps' shares at the end.
// Rows that no observation reaches (masked everywhere in a frame group; band skip of sequential problems) are not
// written: the mask is fixed during a solve and Zt is zeroed once before it, so they hold the zero they would get.
constexpr int ZB_NT = 8;     // tracks per CTA
constexpr int ZB_W = 4;      // warps per CTA
template <int MODEL, int MODE, bool ROBUST>
__global__ void __launch_bounds__(ZB_W * 32) z_build_kernel(
    int S, int N, int Dpad, const float* __restrict__ uv, const uint8_t* __restrict__ mask,
    const double* __restrict__ poses, const double* __restrict__ intr, const double* __restrict__ points,
    const uint8_t* __restrict__ point_const, const double* __restrict__ M, const double* __restrict__ q,
    double* __restrict__ Zt, double* __restrict__ rhs, ptrdiff_t mc_off, const int* __restrict__ fg_tracks, BaLoss loss) {
  using C = BlkCfg<MODEL, MODE>;
  constexpr int DC = C::DC, NS = C::NS;
  constexpr int ZR = 32 * DC;                      // Zt columns of one frame group
  __shared__ __align__(16) double s_cam[ZB_W][16 * 32];   // per warp: pose | f, cx, cy, k, transposed (one frame per lane)
  __shared__ __align__(16) double s_z[ZB_W][3 * ZR];      // per warp: the three Zt rows of one (track, frame group)
  __shared__ double s_pt[ZB_NT][16];                      // per track: X, Y, Z, constant flag | M (9) | q (3)
  __shared__ double s_ws[ZB_W][ZB_NT][3 * (NS > 0 ? NS : 1)];   // per warp and track: its frames' share of W_s
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n0 = blockIdx.x * ZB_NT, nt = min(ZB_NT, N - n0);
  const int ngroups = (S + 31) / 32;
  for (int e = threadIdx.x; e < ZB_NT * 16; e += blockDim.x) {
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
    for (int e = threadIdx.x; e < ZB_W * ZB_NT * 3 * NS; e += blockDim.x) (&s_ws[0][0][0])[e] = 0.0;
  __syncthreads();
  double* pw = s_cam[warp];
  double* zs = s_z[warp];
  const float2* uv2 = reinterpret_cast<const float2*>(uv);
  for (int g = warp; g < ngroups; g += ZB_W) {
    if (fg_tracks && (n0 + nt <= fg_tracks[2 * g] || n0 >= fg_tracks[2 * g + 1])) continue;
    const int s = g * 32 + lane;
    const bool frame_ok = s < S;
    const int cnt = min(32, S - g * 32) * DC;      // Zt columns of the frames of this group that exist
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 12; ++i) pw[i * 32 + lane] = frame_ok ? poses[(size_t)s * 12 + i] : 0.0;
#pragma unroll
    for (int i = 0; i < 4; ++i) pw[(12 + i) * 32 + lane] = frame_ok ? intr[(size_t)s * 4 + i] : 0.0;
    __syncwarp();
    double zq[DC];
#pragma unroll
    for (int i = 0; i < DC; ++i) zq[i] = 0.0;
    for (int t = 0; t < nt; ++t) {
      const size_t o = (size_t)s * N + n0 + t;
      const bool valid = frame_ok && mask[o] != 0;
      if (!__any_sync(0xffffffffu, valid)) continue;
      const float2 ob = frame_ok ? uv2[o] : make_float2(0.f, 0.f);
      const double* pt = s_pt[t];
      const double* m = pt + 4;                    // M upper triangular (row-major), then q
      double jc0[8], jc1[8], jx0[3], jx1[3], rx, ry, oc;
      obs_math<MODEL, ROBUST>(pw + lane, 32, pt[0], pt[1], pt[2], pt[3] != 0.0, ob.x, ob.y, valid, jc0, jc1, jx0, jx1,
                              rx, ry, loss, oc);
#pragma unroll
      for (int i = 0; i < DC; ++i) {
        const double w0 = w_entry(jc0, jc1, jx0, jx1, i, 0), w1 = w_entry(jc0, jc1, jx0, jx1, i, 1),
                     w2 = w_entry(jc0, jc1, jx0, jx1, i, 2);
        const double z0 = w0 * m[0];
        const double z1 = w0 * m[1] + w1 * m[4];
        const double z2 = w0 * m[2] + w1 * m[5] + w2 * m[8];
        zs[lane * DC + i] = z0;
        zs[ZR + lane * DC + i] = z1;
        zs[2 * ZR + lane * DC + i] = z2;
        zq[i] += z0 * m[9] + z1 * m[10] + z2 * m[11];
      }
      if (NS > 0) {
        double a[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) a[k] = k < 3 * NS ? w_entry(jc0, jc1, jx0, jx1, 6 + k / 3, k % 3) : 0.0;
        const double r = warp_reduce_scatter<8>(a, lane);
        if (lane < 3 * NS) s_ws[warp][t][lane] += r;
      }
      __syncwarp();
      double* dst = Zt + (size_t)(3 * (n0 + t)) * Dpad + (size_t)g * ZR;
#pragma unroll
      for (int c = 0; c < 3; ++c, dst += Dpad) {
        const double* src = zs + c * ZR;
        for (int e = 2 * lane; e + 1 < cnt; e += 64)
          *reinterpret_cast<double2*>(dst + e) = *reinterpret_cast<const double2*>(src + e);
        if ((cnt & 1) && lane == 0) dst[cnt - 1] = src[cnt - 1];
      }
      __syncwarp();
    }
    if (frame_ok) {
#pragma unroll
      for (int i = 0; i < DC; ++i) {
        double* r = &rhs[(size_t)s * DC + i];
        if (zq[i] != 0.0) ar_add(r, mc_off ? r + mc_off : nullptr, zq[i]);
      }
    }
  }
  if (NS > 0) {
    __syncthreads();
    if ((int)threadIdx.x < nt * NS) {
      const int t = threadIdx.x / NS, j = threadIdx.x % NS;
      double w[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        w[c] = 0.0;
#pragma unroll
        for (int v = 0; v < ZB_W; ++v) w[c] += s_ws[v][t][j * 3 + c];
      }
      const double* m = s_pt[t] + 4;
      const double z0 = w[0] * m[0];
      const double z1 = w[0] * m[1] + w[1] * m[4];
      const double z2 = w[0] * m[2] + w[1] * m[5] + w[2] * m[8];
      double* zo = Zt + (size_t)(3 * (n0 + t)) * Dpad + (size_t)S * DC + j;
      zo[0] = z0;
      zo[Dpad] = z1;
      zo[2 * (size_t)Dpad] = z2;
      const double zq = z0 * m[9] + z1 * m[10] + z2 * m[11];
      double* r = &rhs[(size_t)S * DC + j];
      if (zq != 0.0) ar_add(r, mc_off ? r + mc_off : nullptr, zq);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Schur SYRK on the FP64 tensor cores: Sraw -= Zt^T Zt with mma.sync.m16n8k16.f64 (SASS DMMA.16x8x16, the full-rate FP64
// MMA of sm_90a; m8n8k4 issues at half of it).  Persistent, one CTA per SM, over a host-built list of (upper tile
// bi <= bj, k range) items:
//   warp 0      producer: one 1 KB bulk copy (cp.async.bulk) per k-row and operand into a ring of SF_STAGES stages of
//               SF_BK k-rows, completing on the stage's mbarrier; Zt is read as z_build wrote it ([Kpad][Dpad]).  The
//               rest of its warpgroup only hands its registers over (setmaxnreg)
//   warps 4-11  2 x 4 warps of 64 x 32 outputs (4 x 4 MMA tiles, 64 accumulator doubles per lane), then syrk_red_upper
// Diagonal tiles load one operand.  The row stride of SF_LDS = 132 doubles is 4 doubles (mod the 128-byte bank row), so
// the four k-rows one fragment load touches fall into disjoint quarters of the banks.
constexpr int SF_BM = 128, SF_BK = 16, SF_LDS = 132, SF_STAGES = 4, SF_MMA_WARPS = 8;
constexpr int SF_THREADS = 128 + SF_MMA_WARPS * 32;
constexpr int SF_STAGE_DOUBLES = 2 * SF_BK * SF_LDS;
constexpr size_t SF_SMEM_BYTES = sizeof(double) * SF_STAGES * SF_STAGE_DOUBLES + sizeof(uint64_t) * 2 * SF_STAGES;

struct SyrkWork {
  int bi, bj, kb0, kb1;        // upper tile (row block bi <= column block bj), k blocks of 64 rows [kb0, kb1)
};

__global__ void __launch_bounds__(SF_THREADS, 1)
    syrk_f64_kernel(const SyrkWork* __restrict__ work, int nwork, int Kpad, int Dpad, const double* __restrict__ Zt,
                    double* __restrict__ Cmat, ptrdiff_t mc_off, const __grid_constant__ FabricDev fd) {
  extern __shared__ __align__(16) double sf_smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(sf_smem + SF_STAGES * SF_STAGE_DOUBLES);
  uint64_t* empty = full + SF_STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < SF_STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], SF_MMA_WARPS);        // one arrive per MMA warp
    }
    mbar_fence_init();
  }
  __syncthreads();

  int stage = 0, phase = 0;
  if (warp < 4) {
    // ===== producer: lanes 0-15 copy the k-rows of operand bi, lanes 16-31 those of bj =====
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp > 0) return;
    const int row = lane & (SF_BK - 1), opnd = lane / SF_BK;
    for (int w = blockIdx.x; w < nwork; w += gridDim.x) {
      const SyrkWork wk = work[w];
      const bool diag = wk.bi == wk.bj;
      const int k1 = min(Kpad, wk.kb1 * 64);
      for (int k = wk.kb0 * 64; k < k1; k += SF_BK) {
        mbar_wait(&empty[stage], phase ^ 1);
        if (lane == 0) mbar_expect_tx(&full[stage], (diag ? 1u : 2u) * SF_BK * SF_BM * (uint32_t)sizeof(double));
        __syncwarp();
        if (opnd == 0 || !diag)
          tma_load_1d(sf_smem + stage * SF_STAGE_DOUBLES + (opnd * SF_BK + row) * SF_LDS,
                      Zt + (size_t)(k + row) * Dpad + (opnd ? wk.bj : wk.bi) * SF_BM, SF_BM * sizeof(double), &full[stage]);
        if (++stage == SF_STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }

  // ===== MMA warps =====
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int wm = (warp - 4) >> 2, wn = warp & 3;
  const int g = lane >> 2, t = lane & 3;
  for (int w = blockIdx.x; w < nwork; w += gridDim.x) {
    const SyrkWork wk = work[w];
    const bool diag = wk.bi == wk.bj;
    const int k1 = min(Kpad, wk.kb1 * 64);
    double acc[4][4][4];
#pragma unroll
    for (int mt = 0; mt < 4; ++mt)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int h = 0; h < 4; ++h) acc[mt][nt][h] = 0.0;
    for (int k = wk.kb0 * 64; k < k1; k += SF_BK) {
      mbar_wait(&full[stage], phase);
      const double* as = sf_smem + stage * SF_STAGE_DOUBLES + t * SF_LDS + wm * 64 + g;
      const double* bs = sf_smem + stage * SF_STAGE_DOUBLES + (diag ? 0 : SF_BK * SF_LDS) + t * SF_LDS + wn * 32 + g;
      double b[4][4];
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int j = 0; j < 4; ++j) b[nt][j] = bs[4 * j * SF_LDS + nt * 8];
#pragma unroll
      for (int mt = 0; mt < 4; ++mt) {
        double a[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) a[i] = as[4 * (i >> 1) * SF_LDS + mt * 16 + 8 * (i & 1)];
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) dmma_m16n8k16(acc[mt][nt], a, b[nt]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[stage]);
      if (++stage == SF_STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }
#pragma unroll
    for (int mt = 0; mt < 4; ++mt)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int h = 0; h < 4; ++h) {
          const int r = wk.bi * SF_BM + wm * 64 + mt * 16 + g + 8 * (h >> 1);
          const int col = wk.bj * SF_BM + wn * 32 + nt * 8 + 2 * t + (h & 1);
          syrk_red_upper(Cmat, Dpad, r, col, wk.bj, diag, acc[mt][nt][h], mc_off, fd);
        }
  }
}

// ------------------------------------------------------------------------------------------------
// A (in place) = sc_i sc_j Sraw + diag; constant parameters pinned; b = sc * rhs.  Lower triangle only.
__global__ void scale_damp_kernel(int D, int Dpad, double* __restrict__ A, const double* __restrict__ rhs,
                                  const double* __restrict__ hdiag, const double* __restrict__ sc,
                                  const uint8_t* __restrict__ pconst, double radius, double min_diag, double max_diag,
                                  double* __restrict__ bvec) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = blockIdx.y;
  if (j >= D || j > i) return;
  const bool ci = pconst[i] != 0, cj = pconst[j] != 0;
  double v;
  if (ci || cj) {
    v = (i == j) ? 1.0 : 0.0;
  } else {
    v = A[(size_t)i * Dpad + j] * sc[i] * sc[j];
    if (i == j) v += fmin(fmax(hdiag[i] * sc[i] * sc[i], min_diag), max_diag) / radius;
  }
  A[(size_t)i * Dpad + j] = v;
  if (i == j) {
    // The scaled right-hand side also becomes row D of the matrix (in the workspace rhs IS row D, so this scales it in
    // place): the factorisation of the bordered matrix [[A, b], [b^T, c]] = [[L, 0], [y^T, .]] leaves y = L^-1 b there,
    // i.e. the forward substitution comes out of the factorisation for free (csrc/ba_solve.cu).  c only has to exceed
    // y^T y.
    const double b = ci ? 0.0 : rhs[i] * sc[i];
    bvec[i] = b;
    A[(size_t)D * Dpad + i] = b;
    if (i == 0) A[(size_t)D * Dpad + D] = 1e300;
  }
}

// d_c = sc * dcs ; the camera slots of scal (csrc/ba_lm.h): the model term, |d_c|^2 and the non-finite count
__global__ void cam_step_kernel(int D, const double* __restrict__ dcs, size_t dcs_stride, const double* __restrict__ sc,
                                const double* __restrict__ hdiag, const double* __restrict__ gvec,
                                const uint8_t* __restrict__ pconst, double radius, double min_diag, double max_diag,
                                double* __restrict__ d_c, double* __restrict__ scal) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double a = 0, b = 0, bad = 0;
  if (i < D) {
    const double x = pconst[i] ? 0.0 : dcs[(size_t)i * dcs_stride];
    const double dc = x * sc[i];
    d_c[i] = dc;
    if (!isfinite(x)) bad = 1.0;
    const double dcc = fmin(fmax(hdiag[i] * sc[i] * sc[i], min_diag), max_diag);
    a = pconst[i] ? 0.0 : (x * x * dcc / radius - dc * gvec[i]);
    b = dc * dc;
  }
  a = warp_sum(a); b = warp_sum(b); bad = warp_sum(bad);
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&scal[SCAL_CAM_QUAD], a);
    atomicAdd(&scal[SCAL_CAM_STEP2], b);
    if (bad > 0) atomicAdd(&scal[SCAL_CAM_BAD], bad);
  }
}

// wacc[n] = W_n^T d_c = sum_s J_p,sn^T (J_c,sn d_c,s + J_intr,sn d_shared), each block rebuilt from its observation
// (obs_math, ba_obs.h).  One lane per track, so the observation loads are coalesced and the sum stays in the lane; the
// warps of a CTA take the frames in turn (a frame's camera and step are broadcasts) and add up at the end.  Frames in
// which none of the CTA's tracks is visible (band skip of sequential problems, or all masked) are passed over.
constexpr int BS_W = 16;     // warps per CTA
template <int MODEL, int MODE, bool ROBUST>
__global__ void __launch_bounds__(BS_W * 32) backsub_kernel(
    int S, int N, const float* __restrict__ uv, const uint8_t* __restrict__ mask, const double* __restrict__ poses,
    const double* __restrict__ intr, const double* __restrict__ points, const uint8_t* __restrict__ point_const,
    const double* __restrict__ d_c, double* __restrict__ wacc, const int* __restrict__ fg_tracks, BaLoss loss) {
  using C = BlkCfg<MODEL, MODE>;
  constexpr int DC = C::DC, NS = C::NS;
  __shared__ double s_cam[BS_W][16];
  __shared__ double s_acc[3][BS_W][32];
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
  double dsh[2] = {0.0, 0.0};
#pragma unroll
  for (int j = 0; j < NS; ++j) dsh[j] = d_c[(size_t)S * DC + j];
  const float2* uv2 = reinterpret_cast<const float2*>(uv);
  double* cam = s_cam[warp];
  double w0 = 0.0, w1 = 0.0, w2 = 0.0;
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
    const double* d = d_c + (size_t)s * DC;
#pragma unroll
    for (int i = 0; i < DC; ++i) {
      const double di = __ldg(d + i);
      w0 = fma(w_entry(jc0, jc1, jx0, jx1, i, 0), di, w0);
      w1 = fma(w_entry(jc0, jc1, jx0, jx1, i, 1), di, w1);
      w2 = fma(w_entry(jc0, jc1, jx0, jx1, i, 2), di, w2);
    }
#pragma unroll
    for (int j = 0; j < NS; ++j) {
      w0 = fma(w_entry(jc0, jc1, jx0, jx1, 6 + j, 0), dsh[j], w0);
      w1 = fma(w_entry(jc0, jc1, jx0, jx1, 6 + j, 1), dsh[j], w1);
      w2 = fma(w_entry(jc0, jc1, jx0, jx1, 6 + j, 2), dsh[j], w2);
    }
  }
  s_acc[0][warp][lane] = w0;
  s_acc[1][warp][lane] = w1;
  s_acc[2][warp][lane] = w2;
  __syncthreads();
  // 3 x 32 sums; a CTA of fewer than three warps (S < 3) takes several
  for (int e = threadIdx.x; e < 96; e += blockDim.x) {
    const int c = e >> 5, t = e & 31;
    double r = 0.0;
    for (int v = 0; v < nw; ++v) r += s_acc[c][v][t];
    if (nlo + t < N) wacc[(size_t)(nlo + t) * 3 + c] = r;
  }
}

// d_p = M M^T (-(g_p + w)); candidate = X + d_p; scal[SCAL_PT_QUAD] += sum dps^2 dpp/r - d_p.g_p,
// scal[SCAL_PT_STEP2] += |d_p|^2.  A constant point (point_const: given constant, or seen by no valid observation) is
// SELECTED out: its step and both terms are exact zeros and its candidate is X bit for bit, whatever wacc, g_p and sc_p
// hold for it (M = 0 alone would give 0 * NaN = NaN for a point whose coordinates are not in the problem).
__global__ void point_step_kernel(int N, const double* __restrict__ M, const double* __restrict__ g_p,
                                  const double* __restrict__ wacc, const double* __restrict__ sc_p,
                                  const double* __restrict__ dpp, const uint8_t* __restrict__ point_const,
                                  const double* __restrict__ X, double radius, double* __restrict__ Xc,
                                  double* __restrict__ scal) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  double a = 0, b = 0;
  if (n < N) {
    const bool pc = point_const && point_const[n];
    const double* m = M + (size_t)n * 9;
    const double g0 = g_p[n * 3], g1 = g_p[n * 3 + 1], g2 = g_p[n * 3 + 2];
    const double y0 = -(g0 + wacc[n * 3]), y1 = -(g1 + wacc[n * 3 + 1]), y2 = -(g2 + wacc[n * 3 + 2]);
    // t = M^T y (M upper triangular)
    const double t0 = m[0] * y0;
    const double t1 = m[1] * y0 + m[4] * y1;
    const double t2 = m[2] * y0 + m[5] * y1 + m[8] * y2;
    const double d0 = m[0] * t0 + m[1] * t1 + m[2] * t2;
    const double d1 = m[4] * t1 + m[5] * t2;
    const double d2 = m[8] * t2;
    Xc[n * 3] = pc ? X[n * 3] : X[n * 3] + d0;
    Xc[n * 3 + 1] = pc ? X[n * 3 + 1] : X[n * 3 + 1] + d1;
    Xc[n * 3 + 2] = pc ? X[n * 3 + 2] : X[n * 3 + 2] + d2;
    const double s0 = sc_p[n * 3], s1 = sc_p[n * 3 + 1], s2 = sc_p[n * 3 + 2];
    const double e0 = d0 / s0, e1 = d1 / s1, e2 = d2 / s2;
    a = pc ? 0.0 : (e0 * e0 * dpp[n * 3] + e1 * e1 * dpp[n * 3 + 1] + e2 * e2 * dpp[n * 3 + 2]) / radius -
                       (d0 * g0 + d1 * g1 + d2 * g2);
    b = pc ? 0.0 : d0 * d0 + d1 * d1 + d2 * d2;
  }
  a = warp_sum(a); b = warp_sum(b);
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&scal[SCAL_PT_QUAD], a);
    atomicAdd(&scal[SCAL_PT_STEP2], b);
  }
}

// candidate cameras: R <- Exp(2 delta) R, t <- t + dt, intrinsics.  A parameter whose step is exactly zero (a constant
// one, and every parameter of a frame that no valid observation sees) is copied, so that it comes back bit for bit as
// given even when it is NaN or inf.
__global__ void cam_update_kernel(int S, int dc, int ns, int model, const double* __restrict__ d_c,
                                  const double* __restrict__ poses, const double* __restrict__ intr,
                                  double* __restrict__ poses_c, double* __restrict__ intr_c) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S) return;
  const double* d = d_c + (size_t)s * dc;
  const double p0 = 2.0 * d[0], p1 = 2.0 * d[1], p2 = 2.0 * d[2];
  const double th2 = p0 * p0 + p1 * p1 + p2 * p2;
  const double th = sqrt(th2);
  double a, b;
  if (th < 1e-12) {
    a = 1.0 - th2 / 6.0;
    b = 0.5 - th2 / 24.0;
  } else {
    a = sin(th) / th;
    b = (1.0 - cos(th)) / th2;
  }
  // E = I + a K + b K^2
  const bool rot = p0 != 0.0 || p1 != 0.0 || p2 != 0.0;
  double E[9];
  E[0] = 1.0 + b * (-(p1 * p1 + p2 * p2)); E[1] = -a * p2 + b * p0 * p1;           E[2] = a * p1 + b * p0 * p2;
  E[3] = a * p2 + b * p0 * p1;             E[4] = 1.0 + b * (-(p0 * p0 + p2 * p2)); E[5] = -a * p0 + b * p1 * p2;
  E[6] = -a * p1 + b * p0 * p2;            E[7] = a * p0 + b * p1 * p2;            E[8] = 1.0 + b * (-(p0 * p0 + p1 * p1));
  const double* P = poses + (size_t)s * 12;
  double* Q = poses_c + (size_t)s * 12;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      Q[i * 4 + j] = rot ? E[i * 3] * P[j] + E[i * 3 + 1] * P[4 + j] + E[i * 3 + 2] * P[8 + j] : P[i * 4 + j];
  Q[3] = d[3] != 0.0 ? P[3] + d[3] : P[3];
  Q[7] = d[4] != 0.0 ? P[7] + d[4] : P[7];
  Q[11] = d[5] != 0.0 ? P[11] + d[5] : P[11];
  const int ni = (model == VGG_SIMPLE_PINHOLE) ? 1 : 2;
  double f = intr[s * 4], k = intr[s * 4 + 3];
  const double* di = dc > 6 ? d + 6 : d_c + (size_t)S * dc;   // per-frame or shared intrinsics step
  if (dc > 6 || ns > 0) {
    if (di[0] != 0.0) f += di[0];
    if (ni > 1 && di[1] != 0.0) k += di[1];
  }
  intr_c[s * 4] = f;
  intr_c[s * 4 + 1] = intr[s * 4 + 1];
  intr_c[s * 4 + 2] = intr[s * 4 + 2];
  intr_c[s * 4 + 3] = k;
}

// gradient of the candidate camera block out of its records
__global__ void extract_gvec_kernel(int S, int dc, int ns, int KR, const double* __restrict__ camrec,
                                    const double* __restrict__ shared_in, double* __restrict__ gvec) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int D = S * dc + ns;
  if (i >= D) return;
  gvec[i] = (i < S * dc) ? camrec[(size_t)(i / dc) * KR + (i % dc)] : shared_in[i - S * dc];
}

// scal[SCAL_GMAX_C] = max |gvec| over free parameters, scal[SCAL_GMAX_P] = max |g_p| over variable points, taken over
// the bit patterns: non-negative doubles order like them, and fabs(NaN) is a positive NaN, which orders above +inf --
// so a NaN gradient entry gives a NaN max-norm (that never passes gradient_tolerance) where fmax would drop it.
__global__ void gradmax_kernel(int D, int N, const double* __restrict__ gvec, const uint8_t* __restrict__ pconst,
                               const double* __restrict__ g_p, const uint8_t* __restrict__ point_const,
                               double* __restrict__ scal) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long mc = 0, mp = 0;
  if (i < D && !pconst[i]) mc = (unsigned long long)__double_as_longlong(fabs(gvec[i]));
  if (i < N * 3 && !(point_const && point_const[i / 3])) mp = (unsigned long long)__double_as_longlong(fabs(g_p[i]));
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    mc = max(mc, __shfl_xor_sync(0xffffffffu, mc, off));
    mp = max(mp, __shfl_xor_sync(0xffffffffu, mp, off));
  }
  if ((threadIdx.x & 31) == 0) {
    atomicMax(reinterpret_cast<unsigned long long*>(&scal[SCAL_GMAX_C]), mc);
    atomicMax(reinterpret_cast<unsigned long long*>(&scal[SCAL_GMAX_P]), mp);
  }
}

// ------------------------------------------------------------------------------------------------
// host-side launch helpers used by ba_solve.cu
// ------------------------------------------------------------------------------------------------
int launch_jacobi_scale_points(int N, const double* H_pp, double* sc_p, int enable, cudaStream_t st) {
  jacobi_scale_points_kernel<<<(N + 255) / 256, 256, 0, st>>>(N, H_pp, sc_p, enable);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}
int launch_jacobi_scale_cams(int D, const double* hdiag, double* sc_c, int enable, cudaStream_t st) {
  jacobi_scale_cams_kernel<<<(D + 255) / 256, 256, 0, st>>>(D, hdiag, sc_c, enable);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}
int launch_point_prep(int N, const double* H_pp, const double* g_p, const double* sc_p, const uint8_t* point_const,
                      double radius, double min_diag, double max_diag, double* M, double* q, double* dpp,
                      double* scal, cudaStream_t st) {
  point_prep_kernel<<<(N + 127) / 128, 128, 0, st>>>(N, H_pp, g_p, sc_p, point_const, radius, min_diag, max_diag, M, q,
                                                     dpp, scal);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}
int launch_assemble_hc(int S, int dc, int ns, int KR, int Dpad, const double* camrec, const double* shared_in,
                       double* Sraw, double* rhs, double* hdiag, double* gvec, ptrdiff_t mc_off, cudaStream_t st) {
  assemble_hc_kernel<<<S + (ns > 0 ? 1 : 0), 64, 0, st>>>(S, dc, ns, KR, Dpad, camrec, shared_in, Sraw, rhs, hdiag, gvec,
                                                          mc_off);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}
int launch_z_build(const vgg_ba_problem* p, int Dpad, const double* M, const double* q, double* Zt, double* rhs,
                   ptrdiff_t mc_off, const int* fg_tracks, cudaStream_t st) {
  VGG_PICK_BA_KERNEL(kern, z_build_kernel, p);
  const int nw = std::min(ZB_W, (p->S + 31) / 32);
  kern<<<(p->N + ZB_NT - 1) / ZB_NT, nw * 32, 0, st>>>(p->S, p->N, Dpad, p->uv, p->mask, p->poses, p->intr, p->points,
                                                        p->point_const, M, q, Zt, rhs, mc_off, fg_tracks, ba_loss_of(p));
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

// work list of the last shape / band hint, kept on the device until either changes
struct SyrkF64State {
  int dev = -1, Kpad = -1, Dpad = -1, sms = 0, nwork = 0;
  std::vector<int> ranges;
  SyrkWork* work_dev = nullptr;
  size_t work_cap = 0;
};
thread_local SyrkF64State g_sf;

// the work list of launch_syrk for nworkers persistent CTAs (ranges: the band hint, empty = dense)
static std::vector<SyrkWork> syrk_f64_work(int Kpad, int Dpad, const std::vector<int>& ranges, int nworkers) {
  const int nb = Dpad / SF_BM, KB = (Kpad + 63) / 64;
  // equal-length items, longest first: the CTAs of a wave advance through k together, so Zt is read from HBM about
  // once and from L2 by the other tiles of its column block
  std::vector<SyrkWork> work;
  build_work_list<SyrkWork>({1}, syrk_tile_jobs(nb, ranges), KB, nworkers, KB, 1,
                            [](const SyrkTileJob& j, int, int k0, int k1) { return SyrkWork{j.bi, j.bj, k0, k1}; }, &work);
  return work;
}

// Cmat -= Zt^T Zt: Zt [Kpad][Dpad] (Dpad % 128 == 0, Kpad % 16 == 0), Cmat [Dpad][Dpad] row-major, LOWER triangle (or
// the fabric destinations of fd / mc_off, see syrk_red_upper).  kb_ranges: [lo, hi) k-block range per 128-column row
// block of Zt outside which the block is exactly zero (csrc/ba_solve.cu, compute_band_hint); any other size = dense.
int launch_syrk(int Kpad, int Dpad, const double* Zt, double* Cmat, ptrdiff_t mc_off, const std::vector<int>& kb_ranges,
                const FabricDev& fd, cudaStream_t st) {
  VGG_REQUIRE(Dpad % SF_BM == 0 && Kpad % SF_BK == 0, "syrk: Dpad must be a multiple of 128 and Kpad of 16");
  const int nb = Dpad / SF_BM;
  SyrkF64State& hs = g_sf;
  const std::vector<int> ranges = (int)kb_ranges.size() == 2 * nb ? kb_ranges : std::vector<int>();
  int dev = 0;
  VGG_CUDA_CHECK(cudaGetDevice(&dev));
  if (hs.dev != dev || hs.Kpad != Kpad || hs.Dpad != Dpad || hs.ranges != ranges) {
    VGG_CUDA_CHECK(cudaDeviceGetAttribute(&hs.sms, cudaDevAttrMultiProcessorCount, dev));
    VGG_CUDA_CHECK(cudaFuncSetAttribute(syrk_f64_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SF_SMEM_BYTES));
    const std::vector<SyrkWork> work = syrk_f64_work(Kpad, Dpad, ranges, hs.sms);
    // a kernel in flight (on any stream) may still read the previous list
    VGG_CUDA_CHECK(cudaDeviceSynchronize());
    if (hs.dev != dev || work.size() > hs.work_cap) {
      if (hs.work_dev) cudaFree(hs.work_dev);
      hs.work_dev = nullptr;
      hs.work_cap = std::max<size_t>(work.size(), 1);
      VGG_CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&hs.work_dev), sizeof(SyrkWork) * hs.work_cap));
    }
    if (!work.empty())
      VGG_CUDA_CHECK(cudaMemcpy(hs.work_dev, work.data(), sizeof(SyrkWork) * work.size(), cudaMemcpyHostToDevice));
    hs.nwork = (int)work.size();
    hs.dev = dev;
    hs.Kpad = Kpad;
    hs.Dpad = Dpad;
    hs.ranges = ranges;
  }
  if (hs.nwork == 0) return VGG_OK;
  syrk_f64_kernel<<<std::min(hs.sms, hs.nwork), SF_THREADS, SF_SMEM_BYTES, st>>>(hs.work_dev, hs.nwork, Kpad, Dpad, Zt, Cmat,
                                                                               mc_off, fd);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}
int launch_scale_damp(int D, int Dpad, double* A, const double* rhs, const double* hdiag, const double* sc,
                      const uint8_t* pconst, double radius, double min_diag, double max_diag, double* bvec,
                      cudaStream_t st) {
  dim3 grid((D + 255) / 256, D);
  scale_damp_kernel<<<grid, 256, 0, st>>>(D, Dpad, A, rhs, hdiag, sc, pconst, radius, min_diag, max_diag, bvec);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}
int launch_cam_step(int D, const double* dcs, size_t dcs_stride, const double* sc, const double* hdiag, const double* gvec,
                    const uint8_t* pconst, double radius, double min_diag, double max_diag, double* d_c, double* scal,
                    cudaStream_t st) {
  cam_step_kernel<<<(D + 255) / 256, 256, 0, st>>>(D, dcs, dcs_stride, sc, hdiag, gvec, pconst, radius, min_diag, max_diag, d_c, scal);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}
int launch_backsub(const vgg_ba_problem* p, const double* d_c, double* wacc, const int* fg_tracks, cudaStream_t st) {
  VGG_PICK_BA_KERNEL(kern, backsub_kernel, p);
  const int nw = std::min(BS_W, p->S);
  kern<<<(p->N + 31) / 32, nw * 32, 0, st>>>(p->S, p->N, p->uv, p->mask, p->poses, p->intr, p->points, p->point_const,
                                             d_c, wacc, fg_tracks, ba_loss_of(p));
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}
int launch_point_step(int N, const double* M, const double* g_p, const double* wacc, const double* sc_p,
                      const double* dpp, const uint8_t* point_const, const double* X, double radius, double* Xc,
                      double* scal, cudaStream_t st) {
  point_step_kernel<<<(N + 127) / 128, 128, 0, st>>>(N, M, g_p, wacc, sc_p, dpp, point_const, X, radius, Xc, scal);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}
int launch_cam_update(int S, int dc, int ns, int model, const double* d_c, const double* poses, const double* intr,
                      double* poses_c, double* intr_c, cudaStream_t st) {
  cam_update_kernel<<<(S + 127) / 128, 128, 0, st>>>(S, dc, ns, model, d_c, poses, intr, poses_c, intr_c);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}
int launch_extract_gvec(int S, int dc, int ns, int KR, const double* camrec, const double* shared_in, double* gvec,
                        cudaStream_t st) {
  const int D = S * dc + ns;
  extract_gvec_kernel<<<(D + 255) / 256, 256, 0, st>>>(S, dc, ns, KR, camrec, shared_in, gvec);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}
int launch_gradmax(int D, int N, const double* gvec, const uint8_t* pconst, const double* g_p,
                   const uint8_t* point_const, double* scal, cudaStream_t st) {
  const int n = D > N * 3 ? D : N * 3;
  gradmax_kernel<<<(n + 255) / 256, 256, 0, st>>>(D, N, gvec, pconst, g_p, point_const, scal);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

}  // namespace vgg

extern "C" {

/* development probes (csrc/dev_probes.h): the in-loop Schur SYRK on its own, dense / with the given band hint */
int vgg_dev_syrk_f64(int Kpad, int Dpad, const double* Zt, double* Cmat, void* stream) {
  return vgg_dev_syrk_f64_band(Kpad, Dpad, Zt, Cmat, stream, nullptr, 0);
}

int vgg_dev_syrk_f64_band(int Kpad, int Dpad, const double* Zt, double* Cmat, void* stream, const int* ranges, int count) {
  using namespace vgg;
  g_launch_count = 0;
  VGG_REQUIRE(Zt && Cmat && Kpad > 0 && Dpad > 0 && (ranges || count <= 0), "bad argument");
  return launch_syrk(Kpad, Dpad, Zt, Cmat, 0, std::vector<int>(ranges, ranges + std::max(count, 0)), FabricDev{},
                     static_cast<cudaStream_t>(stream));
}

/* development probe (csrc/dev_probes.h): the work list launch_syrk builds for nworkers CTAs, host only */
int vgg_dev_syrk_work_list(int Kpad, int Dpad, const int* ranges, int count, int nworkers, int* items, int cap,
                           int* nwork) {
  using namespace vgg;
  VGG_REQUIRE(Kpad > 0 && Kpad % SF_BK == 0 && Dpad > 0 && Dpad % SF_BM == 0 && nworkers > 0 && nwork &&
                  (ranges || count <= 0),
              "bad argument");
  std::vector<int> r(ranges, ranges + std::max(count, 0));
  if ((int)r.size() != 2 * (Dpad / SF_BM)) r.clear();
  const std::vector<SyrkWork> work = syrk_f64_work(Kpad, Dpad, r, nworkers);
  *nwork = (int)work.size();
  if (!items) return VGG_OK;
  VGG_REQUIRE((int)work.size() <= cap, "work list longer than cap");
  for (size_t i = 0; i < work.size(); ++i) {
    items[4 * i] = work[i].bi;
    items[4 * i + 1] = work[i].bj;
    items[4 * i + 2] = work[i].kb0;
    items[4 * i + 3] = work[i].kb1;
  }
  return VGG_OK;
}

}  // extern "C"
