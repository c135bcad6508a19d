// Levenberg-Marquardt driver (Ceres TrustRegionMinimizer + LevenbergMarquardtStrategy semantics) and
// the C-ABI entry points of the bundle-adjustment path.  The loop body is ~14 kernel launches per
// iteration on one stream and ONE small device->host read (accept/reject scalars); track shards on
// other GPUs join through the caller's all-reduce hook (NCCL over NVLink, see vggsfm_b200/dist.py).
#include <cublas_v2.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <map>
#include <vector>
#include "ba_lm.h"
#include "ba_pcg.h"
#include "common.cuh"
#include "dev_probes.h"

namespace vgg {

static thread_local char g_err[512] = "";
thread_local long long g_launch_count = 0;
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// kernels (ba_blocks.cu / ba_schur.cu)
int ba_build_blocks(const vgg_ba_problem* p, double* cost, double* camrec, double* g_p, double* H_pp, double* W,
                    double* shared_out, int tracks_per_warp, const int* fg_tracks, cudaStream_t stream,
                    bool outputs_zeroed = false);
int launch_jacobi_scale_points(int N, const double* H_pp, double* sc_p, int enable, cudaStream_t st);
int launch_jacobi_scale_cams(int D, const double* hdiag, double* sc_c, int enable, cudaStream_t st);
int launch_point_prep(int N, const double* H_pp, const double* g_p, const double* sc_p, const uint8_t* point_const,
                      double radius, double min_diag, double max_diag, double* M, double* q, double* dpp,
                      double* scal, cudaStream_t st);
int launch_assemble_hc(int S, int dc, int ns, int KR, int Dpad, const double* camrec, const double* shared_in,
                       double* Sraw, double* rhs, double* hdiag, double* gvec, ptrdiff_t mc_off, cudaStream_t st);
int launch_z_build(const vgg_ba_problem* p, int Dpad, const double* M, const double* q, double* Zt, double* rhs,
                   ptrdiff_t mc_off, const int* fg_tracks, cudaStream_t st);
int launch_syrk(int Kpad, int Dpad, const double* Zt, double* Cmat, ptrdiff_t mc_off, const std::vector<int>& kb_ranges,
                const FabricDev& fd, cudaStream_t st);
int launch_scale_damp(int D, int Dpad, double* A, const double* rhs, const double* hdiag, const double* sc,
                      const uint8_t* pconst, double radius, double min_diag, double max_diag, double* bvec,
                      cudaStream_t st);
int launch_cam_step(int D, const double* dcs, size_t dcs_stride, const double* sc, const double* hdiag, const double* gvec,
                    const uint8_t* pconst, double radius, double min_diag, double max_diag, double* d_c, double* scal,
                    cudaStream_t st);
int launch_backsub(const vgg_ba_problem* p, const double* d_c, double* wacc, const int* fg_tracks, cudaStream_t st);
int launch_point_step(int N, const double* M, const double* g_p, const double* wacc, const double* sc_p,
                      const double* dpp, const uint8_t* point_const, const double* X, double radius, double* Xc,
                      double* scal, cudaStream_t st);
int launch_cam_update(int S, int dc, int ns, int model, const double* d_c, const double* poses, const double* intr,
                      double* poses_c, double* intr_c, cudaStream_t st);
int launch_extract_gvec(int S, int dc, int ns, int KR, const double* camrec, const double* shared_in, double* gvec,
                        cudaStream_t st);
int launch_gradmax(int D, int N, const double* gvec, const uint8_t* pconst, const double* g_p,
                   const uint8_t* point_const, double* scal, cudaStream_t st);

int launch_trsv_upper(int n, int lda, const double* A, const double* y, size_t y_stride, double* x, long long* stamps,
                      cudaStream_t st);
size_t chol_workspace_doubles(int n);
int chol_lower_inplace(int n, int lda, double* A, double* Ldiag, int* info, const std::vector<int>& end_blk,
                       int arrow_blk, cudaStream_t st);
int launch_fabric_barrier(const FabricDev& fd, size_t flags_off, unsigned long long epoch, int* err, cudaStream_t st);
int launch_fabric_gather(const FabricDev& fd, int nrows, int nmat, int ncols_vec, int lda, cudaStream_t st);
int launch_fabric_allreduce(const FabricDev& fd, size_t flags_off, size_t mail_off, int mail_len, int parity,
                            unsigned long long epoch, double* vec, int count, int max_slot, int* err, cudaStream_t st);

// gathers the accept/reject scalars into one record (csrc/ba_lm.h) so the host reads them with ONE copy
__global__ void pack_scalars_kernel(const double* __restrict__ scal, const double* __restrict__ small,
                                    const int* __restrict__ info, const double* __restrict__ cg,
                                    double* __restrict__ out) {
  const int i = threadIdx.x;
  if (i < VGG_REC(small)) out[i] = scal[i];
  else if (i < VGG_REC(chol_info)) out[i] = small[i - VGG_REC(small)];
  else if (i <= VGG_REC(trsv_info)) out[i] = (double)info[i - VGG_REC(chol_info)];   // INFO_CHOL, INFO_TRSV
  else if (i == VGG_REC(xnorm_c)) out[i] = scal[SCAL_XNORM_C];
  else if (i == VGG_REC(fabric_timeout)) out[i] = (double)info[INFO_FABRIC];
  else if (i < (int)(sizeof(LmRecord) / sizeof(double)) && cg) out[i] = cg[i - VGG_REC(cg)];
}

// |x|^2 of Ceres' reduced program in ambient coordinates (ParameterToleranceReached: step_norm <= tol * (|x| + tol)):
// unit quaternion + translation of every image whose block is not constant, non-constant camera blocks (f,cx,cy[,k]),
// free points.  Only launched when parameter_tolerance > 0 (COLMAP's BA default is 0).  One CTA; the camera part goes to
// cam_out[0], the point part to pts_out[0]: with track shards the cameras are the same on every rank but the points are
// this rank's, so the point part has to be summed over the ranks before |x| is formed.
__global__ void xnorm_kernel(int S, int N, int dc, int ns, int model, const uint8_t* __restrict__ pconst,
                             const uint8_t* __restrict__ point_const, const double* __restrict__ poses,
                             const double* __restrict__ intr, const double* __restrict__ pts,
                             double* __restrict__ cam_out, double* __restrict__ pts_out) {
  double acc = 0.0, acc_p = 0.0;
  const int np = model == VGG_SIMPLE_RADIAL ? 4 : 3;
  for (int s = threadIdx.x; s < S; s += blockDim.x) {
    const uint8_t* c = pconst + (size_t)s * dc;
    if (!(c[0] && c[1] && c[2])) acc += 1.0;
    if (!(c[3] && c[4] && c[5])) {
      const double* P = poses + (size_t)s * 12;
      acc += P[3] * P[3] + P[7] * P[7] + P[11] * P[11];
    }
    if (dc > 6) {
      bool all_const = true;
      for (int i = 6; i < dc; ++i) all_const = all_const && c[i];
      if (!all_const)
        for (int i = 0; i < np; ++i) acc += intr[(size_t)s * 4 + i] * intr[(size_t)s * 4 + i];
    }
  }
  if (threadIdx.x == 0 && ns > 0) {
    bool all_const = true;
    for (int i = 0; i < ns; ++i) all_const = all_const && pconst[(size_t)S * dc + i];
    if (!all_const)
      for (int i = 0; i < np; ++i) acc += intr[i] * intr[i];
  }
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    if (point_const && point_const[n]) continue;
    acc_p += pts[3 * (size_t)n] * pts[3 * (size_t)n] + pts[3 * (size_t)n + 1] * pts[3 * (size_t)n + 1] +
             pts[3 * (size_t)n + 2] * pts[3 * (size_t)n + 2];
  }
  __shared__ double red[2][32];
  acc = warp_sum(acc);
  acc_p = warp_sum(acc_p);
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = acc;
    red[1][threadIdx.x >> 5] = acc_p;
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    const bool in = threadIdx.x < (blockDim.x >> 5);
    const double v = warp_sum(in ? red[0][threadIdx.x] : 0.0), vp = warp_sum(in ? red[1][threadIdx.x] : 0.0);
    if (threadIdx.x == 0) {
      cam_out[0] = v;
      pts_out[0] = vp;
    }
  }
}

// CUDA events of one solve, destroyed on every exit path
struct EventPair {
  cudaEvent_t a = nullptr, b = nullptr;
  ~EventPair() {
    if (a) cudaEventDestroy(a);
    if (b) cudaEventDestroy(b);
  }
};

static double* pinned_scalars() {
  static thread_local double* h = nullptr;
  if (!h) {
    if (cudaHostAlloc(reinterpret_cast<void**>(&h), sizeof(double) * REC_CAP, cudaHostAllocDefault) != cudaSuccess) {
      h = nullptr;
      set_error("cudaHostAlloc for the scalar read-back failed");
    }
  }
  return h;
}

// The problem's robust loss: an unknown type, or a robust one whose scale a is not finite and > 0 with a^2 a normal
// number (so that b = a^2 and c = 1 / b are finite and nonzero), is VGG_EINVAL before anything is launched.
static int check_loss(const vgg_ba_problem* p) {
  const int t = p->loss_function_type;
  const double a = p->loss_function_scale;
  VGG_REQUIRE(t == VGG_LOSS_TRIVIAL || t == VGG_LOSS_SOFT_L1 || t == VGG_LOSS_CAUCHY,
              "loss_function_type must be VGG_LOSS_TRIVIAL, VGG_LOSS_SOFT_L1 or VGG_LOSS_CAUCHY");
  VGG_REQUIRE(t == VGG_LOSS_TRIVIAL || (isfinite(a) && a > 0.0 && isnormal(a * a)),
              "loss_function_scale of a robust loss must be finite and > 0 (a^2 a normal double)");
  return VGG_OK;
}

// sizes of S frames and N points; Dpad leaves >= 2 spare slots after D (row D: the bordered right-hand side)
struct Dims {
  int dc, ns, KR, D, Dpad, Kpad;
};
static int dims_of(int model, int mode, int S, int N, Dims* d) {
  VGG_REQUIRE((model == VGG_SIMPLE_PINHOLE || model == VGG_SIMPLE_RADIAL) &&
                  (mode == VGG_INTR_CONST || mode == VGG_INTR_PER_FRAME || mode == VGG_INTR_SHARED),
              "bad camera_model/intr_mode");
  const int ni = model == VGG_SIMPLE_PINHOLE ? 1 : 2;
  d->dc = mode == VGG_INTR_PER_FRAME ? 6 + ni : 6;
  d->ns = mode == VGG_INTR_SHARED ? ni : 0;
  d->KR = d->dc + d->dc * (d->dc + 1) / 2 + 6 * d->ns;
  d->D = S * d->dc + d->ns;
  d->Dpad = (int)align_up((size_t)d->D + 2, 128);
  d->Kpad = (int)align_up((size_t)3 * N, 16);
  return VGG_OK;
}

// ------------------------------------------------------------------------------------------------
// workspace layout
// ------------------------------------------------------------------------------------------------
// Accumulators of one evaluation.  The coupling blocks W are not among them: z_build and backsub rebuild each one from
// its observation (csrc/ba_obs.h).
struct BlockSet {
  double *cost, *camrec, *g_p, *H_pp, *shared;
};
struct Layout : Dims {
  int S, N;
  BlockSet blk[2];
  double *poses[2], *intr[2], *points[2];
  double *sc_c, *sc_p, *M, *q, *dpp, *wacc, *d_c, *bvec, *Zt;
  double *AR;        // the reduced system (reduced_view)
  double *small;     // [SMALL_VEC + Dpad]: the candidate's all-reduce (csrc/ba_lm.h)
  double *scal;      // [SCAL_DOUBLES]
  double *packed;    // [REC_CAP]: the record the host reads
  double *chol_diag;
  int *dev_info;
  uint8_t *pconst, *point_const;   // [Dpad], [N]: the solve's constant flags (observed_kernel / effective_const_kernel)
  PcgBuffers pcg;                  // iterative layout only (Zt, AR and chol_diag are then null)
  size_t bytes;
};

// iterative: the layout of vgg_ba_solve_iterative -- the same buffers without the Schur operand Zt, the reduced system
// AR and the factorisation workspace, plus the O(S + N) buffers of csrc/ba_pcg.cu: its O(D) vectors, the Schur-Jacobi
// blocks, a copy of the camera records (summed over track shards) and the per-CTA slots of its fixed-order reductions.
// list: the iterative layout of vgg_ba_solve_iterative_obs, which adds the point pass's [N, 3] of the list matvec.
static int make_layout(int S, int N, int model, int mode, void* base, size_t cap, Layout* L, bool iterative = false,
                       bool list = false) {
  if (const int rc = dims_of(model, mode, S, N, L)) return rc;
  const int KR = L->KR, dc = L->dc, ns = L->ns;
  L->S = S;
  L->N = N;
  Carver c(base, cap);
  for (int b = 0; b < 2; ++b) {
    L->blk[b].cost = c.take<double>(8);
    L->blk[b].shared = c.take<double>(8);
    L->blk[b].camrec = c.take<double>((size_t)S * KR);
    L->blk[b].g_p = c.take<double>((size_t)N * 3);
    L->blk[b].H_pp = c.take<double>((size_t)N * 6);
    L->poses[b] = c.take<double>((size_t)S * 12);
    L->intr[b] = c.take<double>((size_t)S * 4);
    L->points[b] = c.take<double>((size_t)N * 3);
  }
  L->sc_c = c.take<double>(L->Dpad);
  L->sc_p = c.take<double>((size_t)N * 3);
  L->M = c.take<double>((size_t)N * 9);
  L->q = c.take<double>((size_t)N * 3);
  L->dpp = c.take<double>((size_t)N * 3);
  L->wacc = c.take<double>((size_t)N * 3);
  L->d_c = c.take<double>(L->Dpad);
  L->bvec = c.take<double>(L->Dpad);
  L->Zt = iterative ? nullptr : c.take<double>((size_t)L->Kpad * L->Dpad);
  L->AR = iterative ? nullptr : c.take<double>(reduced_doubles(L->D, L->Dpad));
  L->small = c.take<double>(SMALL_VEC + (size_t)L->Dpad);
  L->scal = c.take<double>(SCAL_DOUBLES);
  L->packed = c.take<double>(REC_CAP);
  L->chol_diag = iterative ? nullptr : c.take<double>(chol_workspace_doubles(L->D + 1));
  L->dev_info = c.take<int>(INFO_INTS);
  L->pconst = c.take<uint8_t>(L->Dpad);
  L->point_const = c.take<uint8_t>((size_t)N);
  L->pcg = PcgBuffers{};
  if (iterative) {
    PcgBuffers& B = L->pcg;
    // the region the hook sums once per LM iteration, back to back: rhs | hdiag | gvec | acc | shared | camrec
    for (double** v : {&B.rhs, &B.hdiag, &B.gvec}) *v = c.take<double>(L->Dpad);
    B.acc = c.take<double>(9 * (size_t)pcg_blocks(S, ns));
    B.shared = c.take<double>(8);
    B.camrec = c.take<double>((size_t)S * KR);
    B.red_doubles = (size_t)(B.camrec + (size_t)S * KR - B.rhs);
    for (double** v : {&B.x, &B.r, &B.z, &B.q, &B.qs, &B.u, &B.p[0], &B.p[1]}) *v = c.take<double>(L->Dpad);
    B.pinv = c.take<double>(9 * (size_t)pcg_blocks(S, ns));
    B.cg = c.take<double>(PCG_STATE_DOUBLES);
    B.slots = c.take<double>(pcg_slot_doubles(S, dc, ns));
    B.tp = list ? c.take<double>((size_t)N * 3) : nullptr;
  }
  L->bytes = align_up(c.off, 256);
  if (base && c.off > cap) {
    set_error("workspace too small: need %zu bytes, have %zu", c.off, cap);
    return VGG_EWORKSPACE;
  }
  return VGG_OK;
}

static cublasHandle_t get_cublas() {
  static thread_local cublasHandle_t h = nullptr;
  if (!h) {
    if (cublasCreate(&h) != CUBLAS_STATUS_SUCCESS) h = nullptr;
  }
  return h;
}

// Layout of the symmetric allocation of the fabric (doubles): two copies of the reduced system (iteration parity, so a
// rank may zero the next copy while a slow peer still pulls from the previous one), the mailboxes of the small
// all-reduce (2 parities x 8 source ranks), one row of 64-bit barrier flags.
struct FabricLayout {
  size_t arc, mail_off, flags_off, total;
  int mail_len;
};
static FabricLayout fabric_layout(int D, int Dpad) {
  FabricLayout f;
  f.arc = align_up(reduced_doubles(D, Dpad), 256);
  f.mail_len = Dpad + 64;
  f.mail_off = 2 * f.arc;
  f.flags_off = align_up(f.mail_off + (size_t)2 * 8 * f.mail_len, 32);
  f.total = f.flags_off + 64;
  return f;
}

// Run-time state of the fabric (csrc/fabric.cu): reduce-scatter + gather of the reduced system, in-kernel barriers and
// small all-reduces -- no NCCL call and no host callback inside the LM loop.
struct Fabric {
  FabricDev base{};                 // peer[r] = base of rank r's symmetric allocation
  FabricLayout lay{};
  double* ar_local = nullptr;       // this rank's copy of the symmetric allocation
  ptrdiff_t mc_off = 0;             // multicast twin of a local address, minus the address
  unsigned long long* epoch = nullptr;
  int small_parity = 0;
  int* err = nullptr;
  FabricDev at(size_t off) const {
    FabricDev f = base;
    for (int r = 0; r < f.world; ++r) f.peer[r] += off;
    return f;
  }
  int barrier(cudaStream_t st) { return launch_fabric_barrier(base, lay.flags_off, ++*epoch, err, st); }
  int allreduce(double* vec, int count, int max_slot, cudaStream_t st) {
    small_parity ^= 1;
    return launch_fabric_allreduce(base, lay.flags_off, lay.mail_off, lay.mail_len, small_parity, ++*epoch, vec, count,
                                   max_slot, err, st);
  }
};

int Ranks::sum(double* vec, size_t count) const {
  if (fab) return fab->allreduce(vec, (int)count, -1, st);
  return fn ? fn(user, vec, count, 0, st) : VGG_OK;
}
int Ranks::max(double* slot) const {
  if (fab) return fab->allreduce(slot, 1, 0, st);
  return fn ? fn(user, slot, 1, 1, st) : VGG_OK;
}
template <class Gradmax>
int Ranks::candidate(double* small, size_t count, double* scal, Gradmax gradmax) const {
  int rc;
  if (!fab) return (rc = sum(small, count)) || (rc = gradmax()) ? rc : max(scal + SCAL_GMAX_P);
  // one in-kernel all-reduce: the point-gradient max rides in its max slot; the camera max is taken from the sum
  if ((rc = gradmax())) return rc;
  VGG_CUDA_CHECK(cudaMemcpyAsync(small + SMALL_GMAX_P, scal + SCAL_GMAX_P, sizeof(double), cudaMemcpyDeviceToDevice, st));
  if ((rc = fab->allreduce(small, (int)count, SMALL_GMAX_P, st))) return rc;
  VGG_CUDA_CHECK(cudaMemsetAsync(scal + SCAL_GMAX_C, 0, sizeof(double) * 2, st));
  if ((rc = gradmax())) return rc;
  VGG_CUDA_CHECK(cudaMemcpyAsync(scal + SCAL_GMAX_P, small + SMALL_GMAX_P, sizeof(double), cudaMemcpyDeviceToDevice, st));
  return VGG_OK;
}

// The band structure of one solve (compute_band_hint), passed to the launchers that use it; empty / null = dense.
//   kb_ranges             SYRK k-block range per 128-column row block of Zt (launch_syrk)
//   end_blk, arrow_blk    block structure of the reduced system (chol_lower_inplace)
//   dev                   device table for ba_blocks / z_build / backsub (fg_tracks, also kept on the host)
//   kb_rows               reduced-system row range per k-block (vgg_dev_last_band_hint only)
struct BandPlan {
  int nb = 0, KB = 0, ngroups = 0, arrow_blk = 0;
  std::vector<int> kb_ranges, end_blk, kb_rows, fg_tracks;
  BandDev dev{nullptr};
};
// the plan of the most recent solve or vgg_dev_schur_build on this thread (vgg_dev_last_band_hint): the tests compare it
// with oracle/band_oracle.py
static thread_local BandPlan g_band_last;

// first / last visible point of every frame (N / -1 when the frame sees nothing): the band structure of sequential
// (video) problems, where a point lives for a few windows and the dense [S, N] grid is mostly masked out
__global__ void __launch_bounds__(256) frame_point_range_kernel(int S, int N, const uint8_t* __restrict__ mask,
                                                                int* __restrict__ out) {
  __shared__ int s_lo[256], s_hi[256];
  const int s = blockIdx.x;
  int lo = N, hi = -1;
  for (int n = threadIdx.x; n < N; n += 256)
    if (mask[(size_t)s * N + n]) {
      lo = min(lo, n);
      hi = max(hi, n);
    }
  s_lo[threadIdx.x] = lo;
  s_hi[threadIdx.x] = hi;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) {
      s_lo[threadIdx.x] = min(s_lo[threadIdx.x], s_lo[threadIdx.x + w]);
      s_hi[threadIdx.x] = max(s_hi[threadIdx.x], s_hi[threadIdx.x + w]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    out[2 * s] = s_lo[0];
    out[2 * s + 1] = s_hi[0];
  }
}

// Which points and frames at least one valid observation sees: point_seen[n] = 1 / frame_seen[s] = 1.0 (both zeroed
// beforehand; frame_seen is a double so that track shards can sum it with the small all-reduce).  grid.y takes the frames
// in chunks of OBS_FRAMES, one lane per point, so the mask reads are coalesced.
constexpr int OBS_FRAMES = 16;
__global__ void __launch_bounds__(256) observed_kernel(int S, int N, const uint8_t* __restrict__ mask,
                                                       uint8_t* __restrict__ point_seen, double* __restrict__ frame_seen) {
  const int n = blockIdx.x * 256 + threadIdx.x;
  const int s0 = blockIdx.y * OBS_FRAMES, s1 = min(S, s0 + OBS_FRAMES);
  bool seen = false;
  for (int s = s0; s < s1; ++s) {
    const bool m = n < N && mask[(size_t)s * N + n] != 0;
    seen = seen || m;
    if (__any_sync(0xffffffffu, m) && (threadIdx.x & 31) == 0) frame_seen[s] = 1.0;
  }
  if (seen) point_seen[n] = 1;
}

// The constant flags the solve runs with: a point that no valid observation sees, and every camera parameter of a frame
// that sees nothing, count as constant whatever the caller's flags say.  Ceres leaves such blocks out of the problem, so
// they must not reach |x| (parameter tolerance), the step or the gradient norm -- their values may be NaN or inf.
// point_const holds point_seen on entry and is rewritten in place.
__global__ void effective_const_kernel(int S, int N, int dc, int D, const uint8_t* __restrict__ param_const,
                                       const uint8_t* __restrict__ user_point_const, const double* __restrict__ frame_seen,
                                       uint8_t* __restrict__ pconst, uint8_t* __restrict__ point_const) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < D) pconst[i] = param_const[i] || (i < S * dc && frame_seen[i / dc] == 0.0);
  if (i < N) point_const[i] = (user_point_const && user_point_const[i]) || !point_const[i];
}

// Per 128-column row block of Zt: the 64-row k-block range outside which the block is exactly zero (Zt row 3n+c belongs to
// point n; column d < S*dc to frame d / dc; the shared-intrinsics columns see every point).  Leaves the hint empty when
// the grid is (nearly) dense.  One small kernel + a 8 S byte read-back per solve.  *plan must come in empty (dense).
static int compute_band_hint(const vgg_ba_problem* prob, int dc, int D, int Dpad, int Kpad, bool multi_rank, cudaStream_t st,
                             BandPlan* plan) {
  const int S = prob->S, N = prob->N, nb = Dpad / 128, KB = (Kpad + 63) / 64;
  plan->nb = nb;
  plan->KB = KB;
  plan->ngroups = (S + 31) / 32;
  if (nb < 6 || N < 1024) return VGG_OK;
  static thread_local int* dev = nullptr;
  static thread_local int cap = 0;
  if (cap < 2 * S) {
    if (dev) cudaFree(dev);
    VGG_CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&dev), sizeof(int) * 2 * (size_t)S));
    cap = 2 * S;
  }
  frame_point_range_kernel<<<S, 256, 0, st>>>(S, N, prob->mask, dev);
  VGG_LAUNCH_CHECK();
  std::vector<int> fr(2 * (size_t)S);
  VGG_CUDA_CHECK(cudaMemcpyAsync(fr.data(), dev, sizeof(int) * fr.size(), cudaMemcpyDeviceToHost, st));
  VGG_CUDA_CHECK(cudaStreamSynchronize(st));
  std::vector<int> rg(2 * (size_t)nb);
  for (int rb = 0; rb < nb; ++rb) {
    const int d0 = rb * 128, d1 = std::min(D, d0 + 128) - 1;
    int lo = KB, hi = 0;
    if (d1 >= d0) {
      if (d1 >= S * dc) {
        lo = 0;
        hi = KB;
      } else {
        for (int f = d0 / dc; f <= d1 / dc; ++f) {
          if (fr[2 * f + 1] < 0) continue;
          lo = std::min(lo, 3 * fr[2 * f] / 64);
          hi = std::max(hi, (3 * fr[2 * f + 1] + 2) / 64 + 1);
        }
      }
    }
    if (hi <= lo) lo = hi = 0;
    rg[2 * rb] = lo;
    rg[2 * rb + 1] = std::min(hi, KB);
  }
  // worth it only if a good part of the tile x k volume disappears
  double kept = 0.0, all = 0.0;
  for (int bi = 0; bi < nb; ++bi)
    for (int bj = 0; bj <= bi; ++bj) {
      all += KB;
      kept += std::max(0, std::min(rg[2 * bi + 1], rg[2 * bj + 1]) - std::max(rg[2 * bi], rg[2 * bj]));
    }
  if (kept < 0.7 * all) {
    plan->kb_ranges = rg;
    // the same structure for the factorisation: block (i, b) of the reduced system is non-zero iff the k ranges of row
    // blocks i and b meet; the blocks from the first shared-intrinsics column on (and the bordered right-hand-side row)
    // are the dense "arrow".  end[b] = one past the last band block of column b, made non-decreasing (the envelope
    // Cholesky fills) and >= b + 2 so that block row b + 1 always counts as band.
    // Multi-GPU solves: the ranges above describe THIS rank's tracks only, which is all the kernels that touch its W / Zt
    // need; the reduced system it factors is the sum over ranks, so the factorisation keeps the dense structure there.
    const int arrow = (S * dc) / 128;
    if (arrow >= 4 && !multi_rank) {
      std::vector<int> end(nb);
      int prev = 0;
      for (int b = 0; b < nb; ++b) {
        int e = b;
        if (b < arrow) {
          for (int i = b + 1; i < arrow; ++i)
            if (std::min(rg[2 * i + 1], rg[2 * b + 1]) > std::max(rg[2 * i], rg[2 * b])) e = i;
          e = std::max(e + 1, std::min(b + 2, arrow));
          e = std::max(e, prev);
          e = std::min(e, arrow);
        } else {
          e = nb;
        }
        end[b] = e;
        prev = e;
      }
      plan->end_blk = end;
      plan->arrow_blk = arrow;
      // the per-k-block row ranges (reported by vgg_dev_last_band_hint) and the per-frame-group track ranges, the device
      // table of the kernels that walk the dense [frames, points] grid
      const int ngroups = (S + 31) / 32;
      std::vector<int> t_kb(2 * (size_t)KB, 0), t_fg(2 * (size_t)ngroups, 0);
      for (int kb = 0; kb < KB; ++kb) {
        int first = -1, last = -1;
        for (int rb = 0; rb < arrow; ++rb)
          if (rg[2 * rb] <= kb && kb < rg[2 * rb + 1]) {
            if (first < 0) first = rb;
            last = rb;
          }
        t_kb[2 * kb] = first < 0 ? 0 : first * 128;
        t_kb[2 * kb + 1] = first < 0 ? 0 : (last + 1) * 128;
      }
      for (int g = 0; g < ngroups; ++g) {
        int lo = N, hi = 0;
        for (int f = 32 * g; f < std::min(S, 32 * g + 32); ++f) {
          if (fr[2 * f + 1] < 0) continue;
          lo = std::min(lo, fr[2 * f]);
          hi = std::max(hi, fr[2 * f + 1] + 1);
        }
        t_fg[2 * g] = hi > lo ? lo : 0;
        t_fg[2 * g + 1] = hi > lo ? hi : 0;
      }
      static thread_local int* tdev = nullptr;
      static thread_local size_t tcap = 0;
      if (tcap < t_fg.size()) {
        if (tdev) cudaFree(tdev);
        VGG_CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&tdev), sizeof(int) * t_fg.size()));
        tcap = t_fg.size();
      }
      VGG_CUDA_CHECK(cudaMemcpyAsync(tdev, t_fg.data(), sizeof(int) * t_fg.size(), cudaMemcpyHostToDevice, st));
      VGG_CUDA_CHECK(cudaStreamSynchronize(st));           // pageable source
      plan->dev = BandDev{tdev};
      plan->kb_rows = t_kb;
      plan->fg_tracks = t_fg;
    }
  }
  return VGG_OK;
}

// Schur complement of blk onto the reduced system R at the given radius; p: the problem at the state blk was evaluated
// at (z_build rebuilds the coupling blocks from it); fd: where the SYRK epilogue sends each row block in a fabric solve,
// fab: that solve's fabric (null otherwise); syrk = false stops after z_build (vgg_dev_schur_build with Zt filled with a
// NaN sentinel: the SYRK adds every non-zero product, so sentinels left in the padding columns [D, Dpad) would send it
// past the reduced system's rows)
static int schur_build(const Layout& L, const Reduced& R, const vgg_ba_problem& p, const BlockSet& b,
                       const BandPlan& band, const FabricDev& fd, double radius, double min_diag, double max_diag,
                       cudaStream_t st, Fabric* fab = nullptr, bool syrk = true) {
  int rc;
  const ptrdiff_t mc_off = fab ? fab->mc_off : 0;
  if ((rc = launch_point_prep(L.N, b.H_pp, b.g_p, L.sc_p, p.point_const, radius, min_diag, max_diag, L.M, L.q, L.dpp,
                              L.scal, st)))
    return rc;
  VGG_CUDA_CHECK(cudaMemsetAsync(R.S, 0, sizeof(double) * reduced_doubles(L.D, L.Dpad), st));
  // fabric mode: every rank's copy must be zero before anyone's reductions land in it
  if (fab && (rc = fab->barrier(st))) return rc;
  if ((rc = launch_assemble_hc(L.S, L.dc, L.ns, L.KR, L.Dpad, b.camrec, b.shared, R.S, R.rhs, R.hdiag, R.gvec, mc_off, st)))
    return rc;
  if ((rc = launch_z_build(&p, L.Dpad, L.M, L.q, L.Zt, R.rhs, mc_off, band.dev.fg_tracks, st))) return rc;
  if (syrk && (rc = launch_syrk(L.Kpad, L.Dpad, L.Zt, R.S, mc_off, band.kb_ranges, fd, st))) return rc;
  // ... and all reductions must have landed before anyone reads its copy
  if (fab && (rc = fab->barrier(st))) return rc;
  return VGG_OK;
}

// The one schur_build of vgg_ba_schur and vgg_dev_schur_build, into the buffers of *L.  band null: the dense plan, and
// the last band plan is left alone; otherwise the plan of prob->mask when `banded`, recorded as the last one.
static int schur_probe(const vgg_ba_problem* prob, const double* camrec, const double* g_p, const double* H_pp,
                       const double* shared_in, const double* scale_p, double radius, double min_diag, double max_diag,
                       BandPlan* band, bool banded, bool zt_nan, void* workspace, size_t ws_bytes, cudaStream_t st,
                       Layout* L) {
  if (const int rc = check_loss(prob)) return rc;
  g_launch_count = 0;
  int rc = make_layout(prob->S, prob->N, prob->camera_model, prob->intr_mode, workspace, ws_bytes, L);
  if (rc) return rc;
  BandPlan dense;
  if (band && banded && (rc = compute_band_hint(prob, L->dc, L->D, L->Dpad, L->Kpad, false, st, band))) return rc;
  if (band) g_band_last = *band;
  const BlockSet b{nullptr, const_cast<double*>(camrec), const_cast<double*>(g_p), const_cast<double*>(H_pp),
                   const_cast<double*>(shared_in)};
  VGG_CUDA_CHECK(cudaMemcpyAsync(L->sc_p, scale_p, sizeof(double) * (size_t)L->N * 3, cudaMemcpyDeviceToDevice, st));
  // all-ones bytes: a NaN, so that the entries z_build writes can be told from the ones it leaves
  VGG_CUDA_CHECK(cudaMemsetAsync(L->Zt, zt_nan ? 0xff : 0, sizeof(double) * (size_t)L->Kpad * L->Dpad, st));
  VGG_CUDA_CHECK(cudaMemsetAsync(L->scal, 0, sizeof(double) * SCAL_DOUBLES, st));
  return schur_build(*L, reduced_view(L->AR, L->D, L->Dpad), *prob, b, band ? *band : dense, FabricDev{}, radius,
                     min_diag, max_diag, st, nullptr, !zt_nan);
}

static int copy_out(double* dst, const double* src, size_t n, cudaStream_t st) {
  if (dst) VGG_CUDA_CHECK(cudaMemcpyAsync(dst, src, sizeof(double) * n, cudaMemcpyDeviceToDevice, st));
  return VGG_OK;
}

}  // namespace vgg

using namespace vgg;

extern "C" {

const char* vgg_last_error(void) { return g_err; }
int vgg_version(void) { return 102; }

void vgg_ba_default_options(vgg_ba_options* o) {
  memset(o, 0, sizeof(*o));
  o->max_num_iterations = 100;
  o->max_num_consecutive_invalid_steps = 10;
  o->jacobi_scaling = 1;
  o->function_tolerance = 0.0;
  o->gradient_tolerance = 1e-4;
  o->parameter_tolerance = 0.0;
  o->initial_trust_region_radius = 1e4;
  o->max_trust_region_radius = 1e16;
  o->min_trust_region_radius = 1e-32;
  o->min_relative_decrease = 1e-3;
  o->min_lm_diagonal = 1e-6;
  o->max_lm_diagonal = 1e32;
}

int vgg_ba_dims(int camera_model, int intr_mode, int* dc, int* ns) {
  Dims d;
  if (const int rc = dims_of(camera_model, intr_mode, 0, 0, &d)) return rc;
  if (dc) *dc = d.dc;
  if (ns) *ns = d.ns;
  return VGG_OK;
}

int vgg_ba_camrec_len(int camera_model, int intr_mode) {
  Dims d;
  if (const int rc = dims_of(camera_model, intr_mode, 0, 0, &d)) return rc;
  return d.KR;
}

static int workspace_bytes(int S, int N, int camera_model, int intr_mode, size_t* bytes, bool iterative,
                           bool list = false) {
  VGG_REQUIRE(S > 0 && N > 0 && bytes, "S, N must be positive");
  Layout L;
  const int rc = make_layout(S, N, camera_model, intr_mode, nullptr, 0, &L, iterative, list);
  if (!rc) *bytes = L.bytes;
  return rc;
}

int vgg_ba_workspace_bytes(int S, int N, int camera_model, int intr_mode, size_t* bytes) {
  return workspace_bytes(S, N, camera_model, intr_mode, bytes, false);
}

int vgg_ba_build_blocks(const vgg_ba_problem* prob, double* cost, double* camrec, double* g_p, double* H_pp, double* W,
                        double* shared_out, int tracks_per_warp, void* stream) {
  return vgg_dev_build_blocks_band(prob, cost, camrec, g_p, H_pp, W, shared_out, tracks_per_warp, nullptr, 0, stream);
}

/* development probe (csrc/dev_probes.h): vgg_ba_build_blocks with the band table of the solve's block kernel */
int vgg_dev_build_blocks_band(const vgg_ba_problem* prob, double* cost, double* camrec, double* g_p, double* H_pp,
                              double* W, double* shared_out, int tracks_per_warp, const int* fg_tracks, int count,
                              void* stream) {
  VGG_REQUIRE(prob && cost && camrec && g_p && H_pp && shared_out, "null pointer");
  if (const int rc = check_loss(prob)) return rc;
  // a warp's first track t0 = chunk * tracks_per_warp + 4k is the 16-byte (uv) / 4-byte (mask) cp.async offset
  VGG_REQUIRE(tracks_per_warp >= 0 && tracks_per_warp % 4 == 0, "tracks_per_warp must be 0 (choose) or a multiple of 4");
  VGG_REQUIRE(!fg_tracks || count == 2 * ((prob->S + 31) / 32), "fg_tracks needs 2 entries per group of 32 frames");
  cudaStream_t st = (cudaStream_t)stream;
  g_launch_count = 0;
  static thread_local int* tdev = nullptr;
  static thread_local int tcap = 0;
  if (fg_tracks) {
    // a launch of an earlier call, on any stream, may still read the table
    VGG_CUDA_CHECK(cudaDeviceSynchronize());
    if (tcap < count) {
      if (tdev) cudaFree(tdev);
      tdev = nullptr;
      VGG_CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&tdev), sizeof(int) * (size_t)count));
      tcap = count;
    }
    VGG_CUDA_CHECK(cudaMemcpyAsync(tdev, fg_tracks, sizeof(int) * (size_t)count, cudaMemcpyHostToDevice, st));
    VGG_CUDA_CHECK(cudaStreamSynchronize(st));           // pageable source
  }
  return ba_build_blocks(prob, cost, camrec, g_p, H_pp, W, shared_out, tracks_per_warp, fg_tracks ? tdev : nullptr, st);
}

int vgg_ba_schur(const vgg_ba_problem* prob, const double* camrec, const double* g_p, const double* H_pp,
                 const double* shared_in, const double* scale_p, double radius, double min_diag,
                 double max_diag, void* workspace, size_t ws_bytes, double* Sraw, double* rhs, int* Dpad_out,
                 void* stream) {
  VGG_REQUIRE(prob && workspace && Sraw && rhs, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  Layout L;
  int rc = schur_probe(prob, camrec, g_p, H_pp, shared_in, scale_p, radius, min_diag, max_diag, nullptr, false, false,
                       workspace, ws_bytes, st, &L);
  if (rc) return rc;
  const Reduced R = reduced_view(L.AR, L.D, L.Dpad);
  if ((rc = copy_out(Sraw, R.S, (size_t)L.D * L.Dpad, st)) || (rc = copy_out(rhs, R.rhs, L.Dpad, st))) return rc;
  if (Dpad_out) *Dpad_out = L.Dpad;
  return VGG_OK;
}

/* development probe (csrc/dev_probes.h): schur_build as the LM loop runs it, with its intermediate buffers */
int vgg_dev_schur_build(const vgg_ba_problem* prob, const double* camrec, const double* g_p, const double* H_pp,
                        const double* shared_in, const double* scale_p, double radius, double min_diag, double max_diag,
                        int banded, int zt_nan, void* workspace, size_t ws_bytes, double* M, double* q, double* dpp,
                        double* scal, double* Zt, double* Sraw, double* rhs, void* stream) {
  VGG_REQUIRE(prob && camrec && g_p && H_pp && shared_in && scale_p && workspace, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  Layout L;
  BandPlan band;
  int rc = schur_probe(prob, camrec, g_p, H_pp, shared_in, scale_p, radius, min_diag, max_diag, &band, banded, zt_nan,
                       workspace, ws_bytes, st, &L);
  if (rc) return rc;
  const Reduced R = reduced_view(L.AR, L.D, L.Dpad);
  const size_t N = (size_t)L.N;
  if ((rc = copy_out(M, L.M, 9 * N, st)) || (rc = copy_out(q, L.q, 3 * N, st)) ||
      (rc = copy_out(dpp, L.dpp, 3 * N, st)) || (rc = copy_out(scal, L.scal, SCAL_DOUBLES, st)) ||
      (rc = copy_out(Zt, L.Zt, (size_t)L.Kpad * L.Dpad, st)) || (rc = copy_out(Sraw, R.S, (size_t)L.D * L.Dpad, st)) ||
      (rc = copy_out(rhs, R.rhs, L.Dpad, st)))
    return rc;
  VGG_CUDA_CHECK(cudaStreamSynchronize(st));
  return VGG_OK;
}

int vgg_cholesky_lower(int n, int lda, double* A, void* workspace, size_t ws_bytes, int* info_host, void* stream) {
  return vgg_dev_cholesky_band(n, lda, A, workspace, ws_bytes, info_host, stream, nullptr, 0, 0);
}

/* development probe (csrc/dev_probes.h): vgg_cholesky_lower of a banded + arrow matrix */
int vgg_dev_cholesky_band(int n, int lda, double* A, void* workspace, size_t ws_bytes, int* info_host, void* stream,
                          const int* end_blk, int count, int arrow_blk) {
  VGG_REQUIRE(A && workspace && n > 0 && lda >= n && (end_blk || count <= 0), "bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  g_launch_count = 0;
  const size_t need = sizeof(double) * chol_workspace_doubles(n) + 256;
  if (ws_bytes < need) {
    set_error("cholesky workspace too small: need %zu bytes", need);
    return VGG_EWORKSPACE;
  }
  int* info = reinterpret_cast<int*>(workspace);
  double* diag = reinterpret_cast<double*>(reinterpret_cast<char*>(workspace) + 256);
  int rc = chol_lower_inplace(n, lda, A, diag, info, std::vector<int>(end_blk, end_blk + std::max(count, 0)),
                              count > 0 ? arrow_blk : 0, st);
  if (rc) return rc;
  if (info_host) {
    VGG_CUDA_CHECK(cudaMemcpyAsync(info_host, info, sizeof(int), cudaMemcpyDeviceToHost, st));
    VGG_CUDA_CHECK(cudaStreamSynchronize(st));
  }
  return VGG_OK;
}

int vgg_ba_reduced_system_doubles(int S, int camera_model, int intr_mode, size_t* doubles) {
  Dims d;
  VGG_REQUIRE(doubles, "null pointer");
  if (const int rc = dims_of(camera_model, intr_mode, S, 0, &d)) return rc;
  *doubles = reduced_doubles(d.D, d.Dpad);
  return VGG_OK;
}

int vgg_ba_fabric_doubles(int S, int camera_model, int intr_mode, size_t* doubles) {
  Dims d;
  VGG_REQUIRE(doubles, "null pointer");
  if (const int rc = dims_of(camera_model, intr_mode, S, 0, &d)) return rc;
  *doubles = fabric_layout(d.D, d.Dpad).total;
  return VGG_OK;
}

int vgg_ba_solve(const vgg_ba_problem* prob, const vgg_ba_options* opt_in, void* workspace, size_t ws_bytes,
                 vgg_allreduce_fn allreduce, void* ar_user, vgg_ba_summary* summary, double* trace, void* stream) {
  return vgg_ba_solve_fabric(prob, opt_in, workspace, ws_bytes, allreduce, ar_user, nullptr, summary, trace, stream);
}

// a fabric solve's state from the caller's description; the barrier epoch lives as long as the allocation
static int attach_fabric(const vgg_ba_fabric& f, const Layout& L, Fabric* fab) {
  static thread_local std::map<const double*, unsigned long long> fabric_epochs;
  VGG_REQUIRE(f.ar_doubles >= reduced_doubles(L.D, L.Dpad), "fabric buffer too small (vgg_ba_reduced_system_doubles)");
  const FabricLayout lay = fabric_layout(L.D, L.Dpad);
  VGG_REQUIRE(f.world > 1 && f.world <= 8 && f.peer_base[0] && f.total_doubles >= lay.total,
              "fabric needs its peer table: world in 2..8, peer_base set, total_doubles >= vgg_ba_fabric_doubles");
  fab->lay = lay;
  fab->ar_local = f.ar_local;
  fab->mc_off = f.ar_multicast - f.ar_local;
  fab->base = FabricDev{f.world, f.rank, {}};
  for (int r = 0; r < f.world; ++r) fab->base.peer[r] = f.peer_base[r];
  fab->epoch = &fabric_epochs[f.peer_base[f.rank]];
  fab->err = L.dev_info + INFO_FABRIC;
  return VGG_OK;
}

// What the steps of one solve's LM loop share
struct LmContext {
  const Layout& L;
  const vgg_ba_options& opt;
  const BandPlan& band;
  const Ranks& ranks;
  const ObsList* obs;     // the observation list of a list solve, else null (the problem's grid)
};

// a linear step as cam_step reads it: the scaled camera step (entries stride apart), diag(H_cc) and the gradient
struct LinStep {
  const double *dcs, *hdiag, *gvec;
  size_t stride;
};

// DENSE_SCHUR: schur_build, the exchange of the reduced system over the ranks, its scaled and damped bordered form, the
// Cholesky and the backward substitution.  first: the camera Jacobi scale is taken from this hdiag.
static int direct_step(const LmContext& c, const vgg_ba_problem& pcur, const BlockSet& b, int it, double radius,
                       bool first, LinStep* out) {
  const Layout& L = c.L;
  const int D = L.D;
  Fabric* fab = c.ranks.fab;
  const cudaStream_t st = c.ranks.st;
  int rc;
  // a fabric solve alternates two copies of the reduced system (fabric_layout); fd: where the SYRK sends each row block
  const size_t off = fab ? (size_t)(it & 1) * fab->lay.arc : 0;
  const Reduced R = reduced_view(fab ? fab->ar_local + off : L.AR, D, L.Dpad);
  const FabricDev fd = fab ? fab->at(off) : FabricDev{};
  if ((rc = schur_build(L, R, pcur, b, c.band, fd, radius, c.opt.min_lm_diagonal, c.opt.max_lm_diagonal, st, fab)))
    return rc;
  // fabric: every row block is complete on its owner, pull the others (rows 0..D incl. the rhs row, hdiag, gvec)
  if ((rc = fab ? launch_fabric_gather(fd, D + 3, D + 1, D, L.Dpad, st) : c.ranks.sum(R.S, reduced_doubles(D, L.Dpad))))
    return rc;
  if (first && (rc = launch_jacobi_scale_cams(D, R.hdiag, L.sc_c, c.opt.jacobi_scaling, st))) return rc;
  if ((rc = launch_scale_damp(D, L.Dpad, R.S, R.rhs, R.hdiag, L.sc_c, pcur.param_const, radius, c.opt.min_lm_diagonal,
                              c.opt.max_lm_diagonal, L.bvec, st)))
    return rc;
  // Factor the reduced system with the in-repo blocked Cholesky (csrc/chol.cu) on the row-major LOWER triangle of the
  // BORDERED matrix of order D+1 -- scale_damp put the scaled right-hand side into row D, so the factorisation leaves
  // y = L^-1 b there (and, mirrored like every panel, in column D): the forward substitution costs nothing and only the
  // backward substitution L^T x = y remains.  (cuSOLVER potrf on the same matrix took 1.05 ms at n = 2403, this 0.93.)
  if ((rc = chol_lower_inplace(D + 1, L.Dpad, R.S, L.chol_diag, L.dev_info + INFO_CHOL, c.band.end_blk, c.band.arrow_blk, st)))
    return rc;
  // Backward substitution on U = L^T (the row-major upper triangle), y = column D of the buffer: the own kernel
  // (csrc/trsv.cu, block rows chained through the solution), cuBLAS beyond its one co-resident wave of D/64 CTAs.
  VGG_CUDA_CHECK(cudaMemsetAsync(L.dev_info + INFO_TRSV, 0, sizeof(int), st));
  *out = LinStep{L.bvec, R.hdiag, R.gvec, 1};
  if (D <= 7000) return launch_trsv_upper(D, L.Dpad, R.S, R.S + D, (size_t)L.Dpad, L.bvec, nullptr, st);
  cublasHandle_t cb = get_cublas();
  if (!cb || cublasSetStream(cb, st) != CUBLAS_STATUS_SUCCESS) {
    set_error("cublasCreate / cublasSetStream failed");
    return VGG_ESOLVER;
  }
  if (cublasDtrsv(cb, CUBLAS_FILL_MODE_LOWER, CUBLAS_OP_T, CUBLAS_DIAG_NON_UNIT, D, R.S, L.Dpad, R.S + D, L.Dpad) !=
      CUBLAS_STATUS_SUCCESS) {
    set_error("cublasDtrsv failed to launch");
    return VGG_ESOLVER;
  }
  g_launch_count += 1;
  *out = LinStep{R.S + D, R.hdiag, R.gvec, (size_t)L.Dpad};
  return VGG_OK;
}

// ITERATIVE_SCHUR: the point blocks as schur_build prepares them, then the reduced right-hand side and the Schur-Jacobi
// blocks in one pass over the observations, and CG on the implicit reduced system (csrc/ba_pcg.cu)
static int iterative_step(const LmContext& c, const vgg_ba_linear_solver& lin, const vgg_ba_problem& pcur,
                          const BlockSet& b, double radius, bool first, LinStep* out) {
  const Layout& L = c.L;
  const PcgBuffers& B = L.pcg;
  const cudaStream_t st = c.ranks.st;
  int rc;
  if ((rc = launch_point_prep(L.N, b.H_pp, b.g_p, L.sc_p, pcur.point_const, radius, c.opt.min_lm_diagonal,
                              c.opt.max_lm_diagonal, L.M, L.q, L.dpp, L.scal, st)))
    return rc;
  PcgOp op{&pcur, L.dc, L.ns, L.KR, b.camrec, b.shared, L.M, L.sc_c, radius, c.opt.min_lm_diagonal,
           c.opt.max_lm_diagonal, c.band.dev.fg_tracks, c.obs};
  if ((rc = launch_pcg_assemble(op, L.q, B, st))) return rc;
  // track shards: the assembly and a copy of the camera records are this rank's partial sums, summed in one call.
  // The copy, not b itself: after a rejected step b is evaluated again and would be summed twice.
  if (c.ranks.sharded()) {
    VGG_CUDA_CHECK(cudaMemcpyAsync(B.shared, b.shared, sizeof(double) * 8, cudaMemcpyDeviceToDevice, st));
    VGG_CUDA_CHECK(cudaMemcpyAsync(B.camrec, b.camrec, sizeof(double) * (size_t)L.S * L.KR, cudaMemcpyDeviceToDevice, st));
    if ((rc = c.ranks.sum(B.rhs, B.red_doubles))) return rc;
    op.camrec = B.camrec;
    op.shared_in = B.shared;
  }
  if (first && (rc = launch_jacobi_scale_cams(L.D, B.hdiag, L.sc_c, c.opt.jacobi_scaling, st))) return rc;
  if ((rc = launch_pcg_init(op, B, L.bvec, st)) || (rc = pcg_run(op, lin, B, L.bvec, c.ranks, st))) return rc;
  *out = LinStep{B.x, B.hdiag, B.gvec, 1};
  return VGG_OK;
}

// The candidate's record, summed over the ranks: its cost, the point-side model terms, the iterative solve's model
// change, the point part of |x|^2 and the candidate's camera gradient, and from that the gradient max-norms
static int reduce_candidate(const LmContext& c, const vgg_ba_problem& pcur, int cur, bool iterative) {
  const Layout& L = c.L;
  const BlockSet& bn = L.blk[cur ^ 1];
  const cudaStream_t st = c.ranks.st;
  const size_t count = SMALL_VEC + (size_t)L.Dpad;
  int rc;
  VGG_CUDA_CHECK(cudaMemsetAsync(L.small, 0, sizeof(double) * count, st));
  if (iterative &&
      (rc = c.obs ? launch_list_model_change(&pcur, *c.obs, L.M, L.blk[cur].g_p, L.wacc, L.d_c, L.small + SMALL_MODEL_CHANGE,
                                             st)
                  : launch_pcg_model_change(&pcur, L.M, L.blk[cur].g_p, L.wacc, L.d_c, c.band.dev.fg_tracks,
                                            L.small + SMALL_MODEL_CHANGE, st)))
    return rc;
  VGG_CUDA_CHECK(cudaMemcpyAsync(L.small + SMALL_COST, bn.cost, sizeof(double), cudaMemcpyDeviceToDevice, st));
  VGG_CUDA_CHECK(cudaMemcpyAsync(L.small + SMALL_PT_QUAD, L.scal + SCAL_PT_QUAD, sizeof(double) * 2, cudaMemcpyDeviceToDevice, st));
  VGG_CUDA_CHECK(cudaMemcpyAsync(L.small + SMALL_PT_FAIL, L.scal + SCAL_PT_FAIL, sizeof(double), cudaMemcpyDeviceToDevice, st));
  if ((rc = launch_extract_gvec(L.S, L.dc, L.ns, L.KR, bn.camrec, bn.shared, L.small + SMALL_VEC, st))) return rc;
  if (c.opt.parameter_tolerance > 0.0) {
    // |x|^2 of the current state: the camera part stays in scal, the point part (this rank's points) is summed, so
    // every rank tests the parameter tolerance against the same |x|
    xnorm_kernel<<<1, 1024, 0, st>>>(L.S, L.N, L.dc, L.ns, pcur.camera_model, pcur.param_const, pcur.point_const,
                                      pcur.poses, pcur.intr, pcur.points, L.scal + SCAL_XNORM_C, L.small + SMALL_XNORM_P);
    VGG_LAUNCH_CHECK();
  }
  return c.ranks.candidate(L.small, count, L.scal, [&] {
    return launch_gradmax(L.D, L.N, L.small + SMALL_VEC, pcur.param_const, bn.g_p, pcur.point_const, L.scal, st);
  });
}

struct LmState {
  double cost, radius, decrease_factor;
  int invalid_steps;
};

// Ceres' TrustRegionMinimizer + LevenbergMarquardtStrategy rules on iteration it's record: updates s and the trace rows,
// sets summary->termination when the solve stops, and returns true when the candidate becomes the state.
static bool lm_decide(const LmRecord& r, const vgg_ba_options& opt, bool iterative, int it, LmState* s,
                      vgg_ba_summary* summary, double* trace, double* cg_trace) {
  const double c_cost = r.cost();
  const double step_norm = sqrt(r.scal[SCAL_CAM_STEP2] + r.small[SMALL_PT_STEP2]);
  // the iterative solve takes Ceres' model change -(J d)^T (f + J d / 2); 0.5 * quad holds for an exact solve only
  const double model_change =
      iterative ? r.small[SMALL_MODEL_CHANGE] : 0.5 * (r.scal[SCAL_CAM_QUAD] + r.small[SMALL_PT_QUAD]);
  const bool solver_bad = r.chol_info != 0 || r.trsv_info != 0 || r.scal[SCAL_CAM_BAD] > 0 ||
                          r.small[SMALL_PT_FAIL] > 0 || (iterative && r.cg[CG_TERM] == VGG_CG_FAILURE);
  if (iterative && cg_trace) memcpy(cg_trace + (size_t)(it - 1) * 4, r.cg + CG_ITERS, sizeof(double) * 4);
  double* tr = trace ? trace + (size_t)(it - 1) * 8 : nullptr;
  if (tr) {
    tr[0] = it; tr[1] = s->cost; tr[2] = c_cost; tr[3] = model_change; tr[4] = 0; tr[5] = s->radius; tr[6] = step_norm;
    tr[7] = 0;
  }
  if (solver_bad || !(model_change > 0.0) || !isfinite(c_cost)) {
    // Ceres: invalid step -> LevenbergMarquardtStrategy::StepIsInvalid
    if (tr) tr[7] = 2;
    if (++s->invalid_steps >= opt.max_num_consecutive_invalid_steps) summary->termination = VGG_BA_FAILURE;
    else s->radius *= 0.5;
    return false;
  }
  s->invalid_steps = 0;
  const double cost_change = s->cost - c_cost;
  const double rho = cost_change / model_change;
  if (tr) tr[4] = rho;
  // Ceres ParameterToleranceReached(): step_norm <= tol * (|x| + tol), |x| over the non-constant blocks in ambient
  // coordinates (xnorm_kernel, only launched when the tolerance is non-zero -- COLMAP's default is 0)
  const double x_norm = opt.parameter_tolerance > 0.0 ? sqrt(r.xnorm_c + r.small[SMALL_XNORM_P]) : 0.0;
  if (step_norm <= opt.parameter_tolerance * (x_norm + opt.parameter_tolerance)) {
    summary->termination = VGG_BA_CONVERGENCE_PARAMETER;
    return false;
  }
  if (fabs(cost_change) <= opt.function_tolerance * s->cost) {
    // Ceres 2.x TrustRegionMinimizer::Minimize returns from FunctionToleranceReached() before IsStepSuccessful() /
    // HandleSuccessfulStep(): the candidate of the terminating iteration is discarded
    summary->termination = VGG_BA_CONVERGENCE_FUNCTION;
    return false;
  }
  if (!(rho > opt.min_relative_decrease)) {
    s->radius = s->radius / s->decrease_factor;
    s->decrease_factor *= 2.0;
    return false;
  }
  s->cost = c_cost;
  summary->successful++;
  if (tr) tr[7] = 1;
  s->radius = fmin(opt.max_trust_region_radius, s->radius / fmax(1.0 / 3.0, 1.0 - pow(2.0 * rho - 1.0, 3.0)));
  s->decrease_factor = 2.0;
  if (r.gmax() <= opt.gradient_tolerance) summary->termination = VGG_BA_CONVERGENCE_GRADIENT;
  return true;
}

// The checks of vgg_ba_solve_iterative_obs on a list (csrc/ba_list.cu list_validate_kernel): one kernel, one read of
// its flag word (dev_flag, a zeroed int of the workspace)
static int check_list(int S, int N, const ObsList& ol, int* dev_flag, cudaStream_t st) {
  int rc;
  if ((rc = launch_list_validate(S, N, ol, dev_flag, st))) return rc;
  int bad = 0;
  VGG_CUDA_CHECK(cudaMemcpyAsync(&bad, dev_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
  VGG_CUDA_CHECK(cudaStreamSynchronize(st));
  if (bad) {
    set_error("malformed observation list:%s%s%s%s%s%s", bad & 1 ? " track_start (ends or order)" : "",
              bad & 2 ? " point[] (not the owner of its track segment)" : "", bad & 4 ? " frame outside [0, S)" : "",
              bad & 8 ? " frames not strictly increasing within a point" : "",
              bad & 16 ? " frame_start (ends or order)" : "",
              bad & 32 ? " frame_obs (not its segment's frame, or not strictly increasing)" : "");
    return VGG_EINVAL;
  }
  return VGG_OK;
}

// The LM loop of both linear solvers: lin = null solves the reduced camera system directly (direct_step, DENSE_SCHUR),
// otherwise by PCG (iterative_step, ITERATIVE_SCHUR; fabric null).  Everything else is the same code for both.
// list: the observations as a list (ITERATIVE_SCHUR only; prob->uv and prob->mask null), checked before the loop.
static int lm_solve(const vgg_ba_problem* prob, const vgg_ba_options* opt_in, const vgg_ba_linear_solver* lin,
                    void* workspace, size_t ws_bytes, vgg_allreduce_fn allreduce, void* ar_user,
                    const vgg_ba_fabric* fabric, vgg_ba_summary* summary, double* trace, double* cg_trace, void* stream,
                    const vgg_ba_obs_list* list = nullptr) {
  VGG_REQUIRE(prob && workspace && summary, "null pointer");
  VGG_REQUIRE(prob->param_const && prob->poses && prob->intr && prob->points, "null problem array");
  if (list) {
    VGG_REQUIRE(!prob->uv && !prob->mask, "a list solve takes no grid: prob->uv and prob->mask must be NULL");
    VGG_REQUIRE(lin && !fabric, "the observation list runs ITERATIVE_SCHUR only");
    // 2^30: the kernels' 32-bit list indices stay clear of overflow after any loop or grid stride
    VGG_REQUIRE(list->M >= 0 && list->M < ((int64_t)1 << 30), "observation list: need 0 <= M < 2^30");
    VGG_REQUIRE(list->track_start && list->frame_start &&
                    (list->M == 0 || (list->uv && list->frame && list->point && list->frame_obs)),
                "observation list: null array");
  } else {
    VGG_REQUIRE(prob->uv && prob->mask, "null problem array");
  }
  if (const int rc = check_loss(prob)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  g_launch_count = 0;
  vgg_ba_options opt;
  if (opt_in) opt = *opt_in;
  else vgg_ba_default_options(&opt);
  Layout L;
  int rc = make_layout(prob->S, prob->N, prob->camera_model, prob->intr_mode, workspace, ws_bytes, &L, lin != nullptr,
                       list != nullptr);
  if (rc) return rc;
  ObsList ol{};
  if (list) {
    ol = ObsList{(int)list->M, reinterpret_cast<const float2*>(list->uv), list->frame, list->point, list->track_start,
                 list->frame_start, list->frame_obs};
    VGG_CUDA_CHECK(cudaMemsetAsync(L.dev_info, 0, sizeof(int) * INFO_INTS, st));
    if ((rc = check_list(prob->S, prob->N, ol, L.dev_info + INFO_LIST, st))) return rc;
  }
  const ObsList* obs = list ? &ol : nullptr;
  const int S = L.S, N = L.N, D = L.D;
  Fabric fab;
  const bool fab_on = fabric && fabric->ar_local && fabric->ar_multicast;
  if (fab_on && (rc = attach_fabric(*fabric, L, &fab))) return rc;
  const Ranks ranks{fab_on ? &fab : nullptr, allreduce, ar_user, st};
  // the constant flags of this solve (unobserved points and frames added); every kernel below reads these, not the
  // caller's.  Frames are summed over track shards: a frame is in the problem if any rank sees it.
  const vgg_ba_problem* const caller = prob;
  vgg_ba_problem pe = *prob;
  pe.param_const = L.pconst;
  pe.point_const = L.point_const;
  prob = &pe;
  BandPlan band;
  // the iterative solve factors nothing: each rank's band tables describe its own tracks, which is all its kernels read.
  // A list solve has no grid to skip: its kernels walk the observations only.
  if (!list && (rc = compute_band_hint(prob, L.dc, D, L.Dpad, L.Kpad, !lin && (allreduce != nullptr || fabric != nullptr),
                                       st, &band)))
    return rc;
  g_band_last = band;
  const LmContext c{L, opt, band, ranks, obs};
  const size_t small_count = SMALL_VEC + (size_t)L.Dpad;

  VGG_CUDA_CHECK(cudaMemsetAsync(L.point_const, 0, (size_t)N, st));
  VGG_CUDA_CHECK(cudaMemsetAsync(L.small, 0, sizeof(double) * small_count, st));
  if (obs) {
    if ((rc = launch_list_observed(S, N, *obs, L.point_const, L.small + SMALL_VEC, st))) return rc;
  } else {
    observed_kernel<<<dim3((N + 255) / 256, (S + OBS_FRAMES - 1) / OBS_FRAMES), 256, 0, st>>>(S, N, pe.mask, L.point_const,
                                                                                             L.small + SMALL_VEC);
    VGG_LAUNCH_CHECK();
  }
  if ((rc = ranks.sum(L.small, small_count))) return rc;
  effective_const_kernel<<<(std::max(D, N) + 255) / 256, 256, 0, st>>>(S, N, L.dc, D, caller->param_const,
                                                                       caller->point_const, L.small + SMALL_VEC,
                                                                       L.pconst, L.point_const);
  VGG_LAUNCH_CHECK();

  EventPair evs;
  VGG_CUDA_CHECK(cudaEventCreate(&evs.a));
  VGG_CUDA_CHECK(cudaEventCreate(&evs.b));
  const cudaEvent_t ev0 = evs.a, ev1 = evs.b;
  VGG_CUDA_CHECK(cudaEventRecord(ev0, st));

  int cur = 0;
  VGG_CUDA_CHECK(cudaMemcpyAsync(L.poses[0], prob->poses, sizeof(double) * (size_t)S * 12, cudaMemcpyDeviceToDevice, st));
  VGG_CUDA_CHECK(cudaMemcpyAsync(L.intr[0], prob->intr, sizeof(double) * (size_t)S * 4, cudaMemcpyDeviceToDevice, st));
  VGG_CUDA_CHECK(cudaMemcpyAsync(L.points[0], prob->points, sizeof(double) * (size_t)N * 3, cudaMemcpyDeviceToDevice, st));
  if (!lin) VGG_CUDA_CHECK(cudaMemsetAsync(L.Zt, 0, sizeof(double) * (size_t)L.Kpad * L.Dpad, st));
  // the padding of the summed region (alignment gaps, rows past D) is never written: zero it once, so the sums over the
  // ranks add zeros there
  if (lin) VGG_CUDA_CHECK(cudaMemsetAsync(L.pcg.rhs, 0, sizeof(double) * L.pcg.red_doubles, st));
  VGG_CUDA_CHECK(cudaMemsetAsync(L.d_c, 0, sizeof(double) * L.Dpad, st));

  // the problem at state `which` (buffer set of the current state or the candidate)
  auto state = [&](int which) {
    vgg_ba_problem p = *prob;
    p.poses = L.poses[which];
    p.intr = L.intr[which];
    p.points = L.points[which];
    return p;
  };
  auto eval = [&](int which) -> int {
    const vgg_ba_problem p = state(which);
    const BlockSet& b = L.blk[which];
    // cost | shared | camrec | g_p | H_pp are carved back to back: one memset covers all accumulators
    const size_t acc_bytes = reinterpret_cast<char*>(b.H_pp + (size_t)N * 6) - reinterpret_cast<char*>(b.cost);
    VGG_CUDA_CHECK(cudaMemsetAsync(b.cost, 0, acc_bytes, st));
    if (obs) return launch_list_blocks(&p, *obs, b.cost, b.camrec, b.g_p, b.H_pp, b.shared, st);
    return ba_build_blocks(&p, b.cost, b.camrec, b.g_p, b.H_pp, nullptr, b.shared, 0, band.dev.fg_tracks, st, true);
  };
  double* h_rec = pinned_scalars();
  if (!h_rec) return VGG_ECUDA;
  const LmRecord& rec = *reinterpret_cast<const LmRecord*>(h_rec);
  VGG_CUDA_CHECK(cudaMemsetAsync(L.dev_info, 0, sizeof(int) * INFO_INTS, st));
  auto read_record = [&]() -> int {
    pack_scalars_kernel<<<1, 32, 0, st>>>(L.scal, L.small, L.dev_info, L.pcg.cg, L.packed);
    VGG_LAUNCH_CHECK();
    VGG_CUDA_CHECK(cudaMemcpyAsync(h_rec, L.packed, sizeof(double) * (lin ? REC_DOUBLES_CG : REC_DOUBLES),
                                   cudaMemcpyDeviceToHost, st));
    VGG_CUDA_CHECK(cudaStreamSynchronize(st));
    if (rec.fabric_timeout != 0.0) {
      set_error("fabric barrier timed out: a peer rank did not arrive");
      return VGG_ECUDA;
    }
    return VGG_OK;
  };

  // the initial cost and gradient max-norm, summed over the ranks
  const BlockSet& b0 = L.blk[cur];
  if ((rc = eval(cur))) return rc;
  if ((rc = launch_jacobi_scale_points(N, b0.H_pp, L.sc_p, opt.jacobi_scaling, st))) return rc;
  VGG_CUDA_CHECK(cudaMemsetAsync(L.small, 0, sizeof(double) * small_count, st));
  VGG_CUDA_CHECK(cudaMemcpyAsync(L.small + SMALL_COST, b0.cost, sizeof(double), cudaMemcpyDeviceToDevice, st));
  if ((rc = launch_extract_gvec(S, L.dc, L.ns, L.KR, b0.camrec, b0.shared, L.small + SMALL_VEC, st))) return rc;
  if ((rc = ranks.sum(L.small, small_count))) return rc;
  VGG_CUDA_CHECK(cudaMemsetAsync(L.scal + SCAL_GMAX_C, 0, sizeof(double) * 2, st));
  if ((rc = launch_gradmax(D, N, L.small + SMALL_VEC, prob->param_const, b0.g_p, prob->point_const, L.scal, st)) ||
      (rc = ranks.max(L.scal + SCAL_GMAX_P)) || (rc = read_record()))
    return rc;

  LmState s{rec.cost(), opt.initial_trust_region_radius, 2.0, 0};
  memset(summary, 0, sizeof(*summary));
  summary->initial_cost = s.cost;
  summary->termination = rec.gmax() <= opt.gradient_tolerance ? VGG_BA_CONVERGENCE_GRADIENT : VGG_BA_NO_CONVERGENCE;
  int it = 0;
  bool have_scale_c = false;

  while (summary->termination == VGG_BA_NO_CONVERGENCE) {
    if (it >= opt.max_num_iterations) break;
    if (s.radius < opt.min_trust_region_radius) {
      summary->termination = VGG_BA_MIN_TRUST_REGION;
      break;
    }
    ++it;
    const int cand = cur ^ 1;
    VGG_CUDA_CHECK(cudaMemsetAsync(L.scal, 0, sizeof(double) * SCAL_DOUBLES, st));
    const vgg_ba_problem pcur = state(cur);
    LinStep ls;
    if ((rc = lin ? iterative_step(c, *lin, pcur, L.blk[cur], s.radius, !have_scale_c, &ls)
                  : direct_step(c, pcur, L.blk[cur], it, s.radius, !have_scale_c, &ls)))
      return rc;
    have_scale_c = true;
    if ((rc = launch_cam_step(D, ls.dcs, ls.stride, L.sc_c, ls.hdiag, ls.gvec, prob->param_const, s.radius,
                              opt.min_lm_diagonal, opt.max_lm_diagonal, L.d_c, L.scal, st)) ||
        (rc = obs ? launch_list_backsub(&pcur, *obs, L.d_c, L.wacc, st)
                  : launch_backsub(&pcur, L.d_c, L.wacc, band.dev.fg_tracks, st)) ||
        (rc = launch_point_step(N, L.M, L.blk[cur].g_p, L.wacc, L.sc_p, L.dpp, prob->point_const, L.points[cur],
                                s.radius, L.points[cand], L.scal, st)) ||
        (rc = launch_cam_update(S, L.dc, L.ns, prob->camera_model, L.d_c, L.poses[cur], L.intr[cur], L.poses[cand],
                                L.intr[cand], st)) ||
        (rc = eval(cand)) || (rc = reduce_candidate(c, pcur, cur, lin != nullptr)) || (rc = read_record()))
      return rc;
    if (lm_decide(rec, opt, lin != nullptr, it, &s, summary, trace, cg_trace)) cur = cand;
  }

  VGG_CUDA_CHECK(cudaMemcpyAsync(prob->poses, L.poses[cur], sizeof(double) * (size_t)S * 12, cudaMemcpyDeviceToDevice, st));
  VGG_CUDA_CHECK(cudaMemcpyAsync(prob->intr, L.intr[cur], sizeof(double) * (size_t)S * 4, cudaMemcpyDeviceToDevice, st));
  VGG_CUDA_CHECK(cudaMemcpyAsync(prob->points, L.points[cur], sizeof(double) * (size_t)N * 3, cudaMemcpyDeviceToDevice, st));
  VGG_CUDA_CHECK(cudaEventRecord(ev1, st));
  VGG_CUDA_CHECK(cudaEventSynchronize(ev1));
  float ms = 0;
  VGG_CUDA_CHECK(cudaEventElapsedTime(&ms, ev0, ev1));
  summary->iterations = it;
  summary->final_cost = s.cost;
  summary->final_radius = s.radius;
  summary->device_ms = ms;
  summary->kernel_launches = g_launch_count;
  return VGG_OK;
}

int vgg_ba_solve_fabric(const vgg_ba_problem* prob, const vgg_ba_options* opt_in, void* workspace, size_t ws_bytes,
                        vgg_allreduce_fn allreduce, void* ar_user, const vgg_ba_fabric* fabric, vgg_ba_summary* summary,
                        double* trace, void* stream) {
  return lm_solve(prob, opt_in, nullptr, workspace, ws_bytes, allreduce, ar_user, fabric, summary, trace, nullptr, stream);
}

void vgg_ba_default_linear_solver(vgg_ba_linear_solver* lin) {
  lin->type = VGG_BA_DENSE_SCHUR;
  lin->min_linear_solver_iterations = 0;
  lin->max_linear_solver_iterations = 500;
  lin->eta = 0.1;
}

int vgg_ba_workspace_bytes_iterative(int S, int N, int camera_model, int intr_mode, size_t* bytes) {
  return workspace_bytes(S, N, camera_model, intr_mode, bytes, true);
}

int vgg_ba_solve_iterative(const vgg_ba_problem* prob, const vgg_ba_options* opt, const vgg_ba_linear_solver* lin,
                           void* workspace, size_t ws_bytes, vgg_ba_summary* summary, double* trace, double* cg_trace,
                           void* stream) {
  return vgg_ba_solve_iterative_sharded(prob, opt, lin, workspace, ws_bytes, nullptr, nullptr, summary, trace, cg_trace,
                                        stream);
}

static int check_iterative(const vgg_ba_linear_solver* lin) {
  VGG_REQUIRE(lin && lin->type == VGG_BA_ITERATIVE_SCHUR, "vgg_ba_solve_iterative needs lin->type = VGG_BA_ITERATIVE_SCHUR");
  VGG_REQUIRE(lin->min_linear_solver_iterations >= 0 &&
                  lin->max_linear_solver_iterations >= lin->min_linear_solver_iterations && lin->eta > 0.0 &&
                  isfinite(lin->eta),
              "linear solver options: need 0 <= min <= max iterations and a positive finite eta");
  return VGG_OK;
}

int vgg_ba_solve_iterative_sharded(const vgg_ba_problem* prob, const vgg_ba_options* opt,
                                   const vgg_ba_linear_solver* lin, void* workspace, size_t ws_bytes,
                                   vgg_allreduce_fn allreduce, void* allreduce_user, vgg_ba_summary* summary,
                                   double* trace, double* cg_trace, void* stream) {
  if (const int rc = check_iterative(lin)) return rc;
  return lm_solve(prob, opt, lin, workspace, ws_bytes, allreduce, allreduce_user, nullptr, summary, trace, cg_trace,
                  stream);
}

int vgg_ba_workspace_bytes_obs(int S, int N, int camera_model, int intr_mode, size_t* bytes) {
  return workspace_bytes(S, N, camera_model, intr_mode, bytes, true, true);
}

int vgg_ba_solve_iterative_obs(const vgg_ba_problem* prob, const vgg_ba_obs_list* obs, const vgg_ba_options* opt,
                               const vgg_ba_linear_solver* lin, void* workspace, size_t ws_bytes,
                               vgg_allreduce_fn allreduce, void* allreduce_user, vgg_ba_summary* summary,
                               double* trace, double* cg_trace, void* stream) {
  VGG_REQUIRE(obs, "null observation list");
  if (const int rc = check_iterative(lin)) return rc;
  return lm_solve(prob, opt, lin, workspace, ws_bytes, allreduce, allreduce_user, nullptr, summary, trace, cg_trace,
                  stream, obs);
}

/* development probe (csrc/dev_probes.h): the preparation of the iterative solve and one product of its reduced
 * operator, at the given blocks, scales and radius, with the flags of prob taken as the solve's effective ones */
int vgg_dev_pcg_probe(const vgg_ba_problem* prob, const double* camrec, const double* g_p, const double* H_pp,
                      const double* shared_in, const double* scale_p, const double* scale_c, double radius,
                      double min_diag, double max_diag, const double* x_in, void* workspace, size_t ws_bytes,
                      double* y_out, double* b_out, double* pinv_out, double* state_out, void* stream) {
  VGG_REQUIRE(prob && camrec && g_p && H_pp && shared_in && scale_p && scale_c && x_in && workspace, "null pointer");
  VGG_REQUIRE(prob->param_const, "null param_const");
  if (const int rc = check_loss(prob)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  g_launch_count = 0;
  Layout L;
  int rc = make_layout(prob->S, prob->N, prob->camera_model, prob->intr_mode, workspace, ws_bytes, &L, true);
  if (rc) return rc;
  const int D = L.D;
  const PcgOp op{prob, L.dc, L.ns, L.KR, camrec, shared_in, L.M, L.sc_c, radius, min_diag, max_diag, nullptr};
  VGG_CUDA_CHECK(cudaMemcpyAsync(L.sc_p, scale_p, sizeof(double) * (size_t)L.N * 3, cudaMemcpyDeviceToDevice, st));
  VGG_CUDA_CHECK(cudaMemcpyAsync(L.sc_c, scale_c, sizeof(double) * (size_t)D, cudaMemcpyDeviceToDevice, st));
  VGG_CUDA_CHECK(cudaMemsetAsync(L.scal, 0, sizeof(double) * SCAL_DOUBLES, st));
  if ((rc = launch_point_prep(L.N, H_pp, g_p, L.sc_p, prob->point_const, radius, min_diag, max_diag, L.M, L.q, L.dpp,
                              L.scal, st)))
    return rc;
  if ((rc = launch_pcg_assemble(op, L.q, L.pcg, st))) return rc;
  if ((rc = launch_pcg_init(op, L.pcg, L.bvec, st))) return rc;
  if (state_out)
    VGG_CUDA_CHECK(cudaMemcpyAsync(state_out, L.pcg.cg, sizeof(double) * PCG_STATE_DOUBLES, cudaMemcpyDeviceToDevice, st));
  VGG_CUDA_CHECK(cudaMemsetAsync(L.pcg.cg + CG_DONE, 0, sizeof(double), st));   // the product runs whatever init decided
  VGG_CUDA_CHECK(cudaMemcpyAsync(L.pcg.x, x_in, sizeof(double) * (size_t)D, cudaMemcpyDeviceToDevice, st));
  if ((rc = launch_pcg_matvec(op, 0, nullptr, nullptr, L.pcg, st))) return rc;
  if ((rc = launch_pcg_combine(D, L.pcg.q, L.pcg.qs, st))) return rc;
  if ((rc = copy_out(y_out, L.pcg.q, D, st)) || (rc = copy_out(b_out, L.bvec, D, st)) ||
      (rc = copy_out(pinv_out, L.pcg.pinv, 9 * (size_t)pcg_blocks(prob->S, L.ns), st)))
    return rc;
  VGG_CUDA_CHECK(cudaStreamSynchronize(st));
  return VGG_OK;
}

/* development probe (csrc/dev_probes.h): the band hint of the most recent solve on this thread */
int vgg_dev_last_band_hint(int* meta, int* rb_range, int* end_blk, int* kb_rows, int* fg_tracks) {
  VGG_REQUIRE(meta, "null pointer");
  const BandPlan& r = g_band_last;
  const int m[8] = {!r.kb_ranges.empty(), !r.end_blk.empty(), !r.fg_tracks.empty(), r.nb, r.KB, r.ngroups, r.arrow_blk, 0};
  memcpy(meta, m, sizeof(m));
  auto put = [](int* dst, const std::vector<int>& v) {
    if (dst && !v.empty()) memcpy(dst, v.data(), sizeof(int) * v.size());
  };
  put(rb_range, r.kb_ranges);
  put(end_blk, r.end_blk);
  put(kb_rows, r.kb_rows);
  put(fg_tracks, r.fg_tracks);
  return VGG_OK;
}

}  // extern "C"
