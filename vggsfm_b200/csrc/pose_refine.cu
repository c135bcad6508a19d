// Batched absolute-pose refinement (motion-only bundle adjustment), one CTA per frame.
//
// Replaces the per-frame python loop around pycolmap.pose_refinement in
//   vggsfm/utils/triangulation.py:260-479 (refine_pose) and :482-647 (init_refine_pose):
// S sequential CPU Ceres solves with a .cpu() sync each become one launch in which every frame runs its
// own trust-region LM (Ceres semantics, CauchyLoss(1), 6..8 unknowns) entirely on chip: the 8x8 normal
// equations are accumulated over the frame's inlier correspondences in registers, reduced through
// shuffles + shared memory, solved by one thread, and the candidate is re-evaluated by the whole CTA.
// The points [P,3] are shared by all S CTAs (L2-resident); per-frame traffic is uv [P,2] f32 + mask [P].
#include "common.cuh"

namespace vgg {

namespace {

constexpr int PT = 256;            // threads per CTA
constexpr int PW = PT / 32;
constexpr int NACC = 45;           // 36 (H upper) + 8 (g) + 1 (cost)

struct Cam {
  double R[9], t[3], f, cx, cy, k;
};

__device__ __forceinline__ void load_cam(Cam& c, const double* pose, const double* intr) {
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int j = 0; j < 3; ++j) c.R[i * 3 + j] = pose[i * 4 + j];
    c.t[i] = pose[i * 4 + 3];
  }
  c.f = intr[0]; c.cx = intr[1]; c.cy = intr[2]; c.k = intr[3];
}

// residual of one correspondence; returns false when the depth is not positive (used by the pre-filter only)
template <int MODEL>
__device__ __forceinline__ void project(const Cam& c, const double X[3], double RX[3], double& u, double& v,
                                        double& iz, double& d, double& r2, double& pz) {
#pragma unroll
  for (int i = 0; i < 3; ++i) RX[i] = c.R[i * 3] * X[0] + c.R[i * 3 + 1] * X[1] + c.R[i * 3 + 2] * X[2];
  pz = RX[2] + c.t[2];
  iz = 1.0 / pz;
  u = (RX[0] + c.t[0]) * iz;
  v = (RX[1] + c.t[1]) * iz;
  r2 = u * u + v * v;
  d = (MODEL == VGG_SIMPLE_RADIAL) ? 1.0 + c.k * r2 : 1.0;
}

__device__ __forceinline__ void block_reduce(double (&acc)[NACC], int n, double* red, double* tot) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int i = 0; i < n; ++i) {
    const double s = warp_sum(acc[i]);
    if (lane == 0) red[w * NACC + i] = s;
  }
  __syncthreads();
  if (threadIdx.x < n) {
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < PW; ++k) s += red[k * NACC + threadIdx.x];
    tot[threadIdx.x] = s;
  }
  __syncthreads();
}

// 8x8 SPD solve in place (A lower used), returns false on a non-positive pivot
__device__ bool chol_solve8(double* A, double* b) {
  for (int j = 0; j < 8; ++j) {
    double d = A[j * 8 + j];
    for (int k = 0; k < j; ++k) d -= A[j * 8 + k] * A[j * 8 + k];
    if (!(d > 0.0)) return false;
    d = sqrt(d);
    A[j * 8 + j] = d;
    for (int i = j + 1; i < 8; ++i) {
      double s = A[i * 8 + j];
      for (int k = 0; k < j; ++k) s -= A[i * 8 + k] * A[j * 8 + k];
      A[i * 8 + j] = s / d;
    }
  }
  for (int i = 0; i < 8; ++i) {
    double s = b[i];
    for (int k = 0; k < i; ++k) s -= A[i * 8 + k] * b[k];
    b[i] = s / A[i * 8 + i];
  }
  for (int i = 7; i >= 0; --i) {
    double s = b[i];
    for (int k = i + 1; k < 8; ++k) s -= A[k * 8 + i] * b[k];
    b[i] = s / A[i * 8 + i];
  }
  return true;
}

__device__ void plus_cam(const double* pose, const double* intr, const double* dl, double* pose_c, double* intr_c) {
  const double p0 = 2.0 * dl[0], p1 = 2.0 * dl[1], p2 = 2.0 * dl[2];
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
  double E[9];
  E[0] = 1.0 + b * (-(p1 * p1 + p2 * p2)); E[1] = -a * p2 + b * p0 * p1;           E[2] = a * p1 + b * p0 * p2;
  E[3] = a * p2 + b * p0 * p1;             E[4] = 1.0 + b * (-(p0 * p0 + p2 * p2)); E[5] = -a * p0 + b * p1 * p2;
  E[6] = -a * p1 + b * p0 * p2;            E[7] = a * p0 + b * p1 * p2;            E[8] = 1.0 + b * (-(p0 * p0 + p1 * p1));
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j)
      pose_c[i * 4 + j] = E[i * 3] * pose[j] + E[i * 3 + 1] * pose[4 + j] + E[i * 3 + 2] * pose[8 + j];
    pose_c[i * 4 + 3] = pose[i * 4 + 3] + dl[3 + i];
  }
  intr_c[0] = intr[0] + dl[6];
  intr_c[1] = intr[1];
  intr_c[2] = intr[2];
  intr_c[3] = intr[3] + dl[7];
}

enum { ST_EVAL_CAND = 0, ST_RETRY = 1, ST_DONE = 2, ST_ACCEPT = 3 };

struct Shared {
  double red[PW * NACC];
  double tot[NACC];
  double pose[12], intr[4], pose_c[12], intr_c[4];
  double H[64], g[8], sc[8], dd[8], y[8], delta[8];
  double cost, radius, decrease, model_change;
  int state, it, invalid, successful, termination, count;
};

template <int MODEL>
__global__ void __launch_bounds__(PT) pose_refine_kernel(int S, int P, const float* __restrict__ uv,
                                                         const uint8_t* __restrict__ inlier,
                                                         const uint8_t* __restrict__ frame_flags,
                                                         const double* __restrict__ points, double* __restrict__ poses,
                                                         double* __restrict__ intr, vgg_pose_options opt,
                                                         uint8_t* __restrict__ used, double* __restrict__ summary_d,
                                                         int32_t* __restrict__ summary_i) {
  __shared__ Shared sh;
  const int s = blockIdx.x;
  const int tid = threadIdx.x;
  const uint8_t flags = frame_flags[s];
  const float2* uvs = reinterpret_cast<const float2*>(uv) + (size_t)s * P;
  const uint8_t* inl = inlier + (size_t)s * P;
  uint8_t* use = used + (size_t)s * P;
  const double bsc = opt.loss_function_scale * opt.loss_function_scale;
  const bool free_f = (flags & 2) != 0;
  const bool free_k = (flags & 4) != 0 && MODEL == VGG_SIMPLE_RADIAL;

  if (tid < 12) sh.pose[tid] = poses[(size_t)s * 12 + tid];
  if (tid < 4) sh.intr[tid] = intr[(size_t)s * 4 + tid];
  __syncthreads();

  // ---- effective inlier mask: visibility/geometry mask AND (depth > 0, squared error <= max^2) at the input pose
  //      (triangulation.py:298-315); counted against min_inliers (:386 "> 100", :585 "> 50")
  {
    Cam c;
    load_cam(c, sh.pose, sh.intr);
    const double thr = opt.max_reproj_error * opt.max_reproj_error;
    int cnt = 0;
    for (int p = tid; p < P; p += PT) {
      uint8_t m = inl[p];
      if (m && opt.max_reproj_error > 0.0) {
        const double X[3] = {points[(size_t)p * 3], points[(size_t)p * 3 + 1], points[(size_t)p * 3 + 2]};
        double RX[3], u, v, iz, d, r2, pz;
        project<MODEL>(c, X, RX, u, v, iz, d, r2, pz);
        const float2 o = uvs[p];
        const double rx = c.f * d * u + c.cx - (double)o.x, ry = c.f * d * v + c.cy - (double)o.y;
        double e = rx * rx + ry * ry;
        if (pz <= 0.0) e = 1e9;
        m = (e <= thr) ? 1 : 0;
      }
      use[p] = m;
      cnt += m;
    }
    double accn[NACC];  // `use` is re-read below by the thread that wrote it: no barrier needed for it
    accn[0] = (double)cnt;
    block_reduce(accn, 1, sh.red, sh.tot);
  }
  const int count = (int)(sh.tot[0] + 0.5);
  __syncthreads();
  if (!(flags & 1) || count <= opt.min_inliers) {
    if (tid == 0) {
      summary_d[s * 4 + 0] = 0.0; summary_d[s * 4 + 1] = 0.0; summary_d[s * 4 + 2] = 0.0; summary_d[s * 4 + 3] = (double)count;
      summary_i[s * 4 + 0] = 0; summary_i[s * 4 + 1] = 0;
      summary_i[s * 4 + 2] = (flags & 1) ? VGG_POSE_FEW_INLIERS : VGG_POSE_SKIPPED;
      summary_i[s * 4 + 3] = 0;
    }
    return;
  }

  // ---- evaluation of the robustified normal equations / cost at a camera held in shared memory
  auto evaluate = [&](const double* pose_sm, const double* intr_sm, bool jac) {
    Cam c;
    load_cam(c, pose_sm, intr_sm);
    double acc[NACC];
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = 0.0;
    for (int p = tid; p < P; p += PT) {
      if (!use[p]) continue;
      const double X[3] = {points[(size_t)p * 3], points[(size_t)p * 3 + 1], points[(size_t)p * 3 + 2]};
      double RX[3], u, v, iz, d, r2, pz;
      project<MODEL>(c, X, RX, u, v, iz, d, r2, pz);
      const float2 o = uvs[p];
      const double rx = c.f * d * u + c.cx - (double)o.x, ry = c.f * d * v + c.cy - (double)o.y;
      const double sq = rx * rx + ry * ry;
      acc[44] += 0.5 * bsc * log1p(sq / bsc);
      if (!jac) continue;
      const double w = 1.0 / (1.0 + sq / bsc);      // rho'; Corrector with rho'' <= 0 scales r and J by sqrt(rho')
      const double k = (MODEL == VGG_SIMPLE_RADIAL) ? c.k : 0.0;
      const double a00 = c.f * (d + 2.0 * k * u * u), a01 = c.f * (2.0 * k * u * v), a11 = c.f * (d + 2.0 * k * v * v);
      double J0[8], J1[8];
      const double j00 = a00 * iz, j01 = a01 * iz, j02 = -(a00 * u + a01 * v) * iz;
      const double j10 = a01 * iz, j11 = a11 * iz, j12 = -(a01 * u + a11 * v) * iz;
      J0[0] = 2.0 * (-RX[2] * j01 + RX[1] * j02); J1[0] = 2.0 * (-RX[2] * j11 + RX[1] * j12);
      J0[1] = 2.0 * (RX[2] * j00 - RX[0] * j02);  J1[1] = 2.0 * (RX[2] * j10 - RX[0] * j12);
      J0[2] = 2.0 * (-RX[1] * j00 + RX[0] * j01); J1[2] = 2.0 * (-RX[1] * j10 + RX[0] * j11);
      J0[3] = j00; J0[4] = j01; J0[5] = j02;
      J1[3] = j10; J1[4] = j11; J1[5] = j12;
      J0[6] = free_f ? d * u : 0.0;
      J1[6] = free_f ? d * v : 0.0;
      J0[7] = free_k ? c.f * u * r2 : 0.0;
      J1[7] = free_k ? c.f * v * r2 : 0.0;
      int q = 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const double wi0 = w * J0[i], wi1 = w * J1[i];
#pragma unroll
        for (int j = i; j < 8; ++j) acc[q++] += wi0 * J0[j] + wi1 * J1[j];
        acc[36 + i] += wi0 * rx + wi1 * ry;
      }
    }
    if (jac) {
      block_reduce(acc, NACC, sh.red, sh.tot);
    } else {
      double a1[NACC];
      a1[0] = acc[44];
      block_reduce(a1, 1, sh.red, sh.tot);
    }
  };

  // thread 0: unpack H,g,cost from tot after a full evaluation
  auto unpack = [&]() {
    int q = 0;
    for (int i = 0; i < 8; ++i)
      for (int j = i; j < 8; ++j) {
        sh.H[i * 8 + j] = sh.tot[q];
        sh.H[j * 8 + i] = sh.tot[q];
        ++q;
      }
    for (int i = 0; i < 8; ++i) sh.g[i] = sh.tot[36 + i];
    sh.cost = sh.tot[44];
  };
  auto grad_max = [&]() {
    double m = 0.0;
    for (int i = 0; i < 8; ++i) {
      const bool fr = i < 6 || (i == 6 ? free_f : free_k);
      if (fr) m = fmax(m, fabs(sh.g[i]));
    }
    return m;
  };

  evaluate(sh.pose, sh.intr, true);
  if (tid == 0) {
    unpack();
    for (int i = 0; i < 8; ++i) sh.sc[i] = 1.0 / (1.0 + sqrt(sh.H[i * 8 + i]));
    sh.radius = opt.initial_trust_region_radius;
    sh.decrease = 2.0;
    sh.it = 0; sh.invalid = 0; sh.successful = 0; sh.termination = VGG_BA_NO_CONVERGENCE;
    summary_d[s * 4 + 0] = sh.cost;
    sh.state = ST_EVAL_CAND;
    // a non-finite residual at the start (NaN observation, point on the camera plane) fails the solve before the first
    // iteration, as Ceres' initial evaluation does; grad_max() would drop the NaNs (fmax) and report convergence
    bool finite = isfinite(sh.cost);
    for (int i = 0; i < 8; ++i)
      if (i < 6 || (i == 6 ? free_f : free_k)) finite = finite && isfinite(sh.g[i]);
    if (!finite) {
      sh.termination = VGG_BA_FAILURE;
      sh.state = ST_DONE;
    } else if (grad_max() <= opt.gradient_tolerance) {
      sh.termination = VGG_BA_CONVERGENCE_GRADIENT;
      sh.state = ST_DONE;
    }
  }
  auto read_state = [&]() {
    __syncthreads();
    const int v = sh.state;
    __syncthreads();
    return v;
  };

  while (read_state() != ST_DONE) {
    // ---- trust-region step (one thread; 8 unknowns)
    if (tid == 0) {
      if (sh.it >= opt.max_num_iterations) {
        sh.state = ST_DONE;
      } else if (sh.radius < opt.min_trust_region_radius) {
        sh.termination = VGG_BA_MIN_TRUST_REGION;
        sh.state = ST_DONE;
      } else {
        sh.it++;
        double A[64], b[8];
        for (int i = 0; i < 8; ++i) {
          const bool fi = i < 6 || (i == 6 ? free_f : free_k);
          for (int j = 0; j < 8; ++j) {
            const bool fj = j < 6 || (j == 6 ? free_f : free_k);
            A[i * 8 + j] = (fi && fj) ? sh.H[i * 8 + j] * sh.sc[i] * sh.sc[j] : 0.0;
          }
          const double di = fmin(fmax(sh.H[i * 8 + i] * sh.sc[i] * sh.sc[i], opt.min_lm_diagonal), opt.max_lm_diagonal);
          sh.dd[i] = di;
          if (fi) {
            A[i * 8 + i] += di / sh.radius;
            b[i] = -sh.g[i] * sh.sc[i];
          } else {
            A[i * 8 + i] = 1.0;
            b[i] = 0.0;
          }
        }
        bool ok = chol_solve8(A, b);
        double mc = 0.0;
        if (ok) {
          for (int i = 0; i < 8; ++i) {
            const bool fi = i < 6 || (i == 6 ? free_f : free_k);
            sh.y[i] = b[i];
            sh.delta[i] = b[i] * sh.sc[i];
            if (!isfinite(sh.delta[i])) ok = false;
            mc += (fi ? b[i] * b[i] * sh.dd[i] / sh.radius : 0.0) - sh.delta[i] * sh.g[i];
          }
          mc *= 0.5;
          if (!(mc > 0.0)) ok = false;
        }
        if (!ok) {
          sh.invalid++;
          if (sh.invalid >= opt.max_num_consecutive_invalid_steps) {
            sh.termination = VGG_BA_FAILURE;
            sh.state = ST_DONE;
          } else {
            sh.radius *= 0.5;
            sh.state = ST_RETRY;
          }
        } else {
          sh.invalid = 0;
          sh.model_change = mc;
          plus_cam(sh.pose, sh.intr, sh.delta, sh.pose_c, sh.intr_c);
          sh.state = ST_EVAL_CAND;
        }
      }
    }
    const int st1 = read_state();
    if (st1 == ST_DONE) break;
    if (st1 == ST_RETRY) continue;

    // ---- candidate cost (whole CTA), then the Ceres accept / reject / convergence rules
    evaluate(sh.pose_c, sh.intr_c, false);
    if (tid == 0) {
      const double c_cost = sh.tot[0];
      const double nd = sqrt(sh.delta[0] * sh.delta[0] + sh.delta[1] * sh.delta[1] + sh.delta[2] * sh.delta[2]);
      double sn = 2.0 - 2.0 * cos(nd);
      for (int i = 3; i < 8; ++i) sn += sh.delta[i] * sh.delta[i];
      const double step_norm = sqrt(sn);
      double xn = 1.0 + sh.pose[3] * sh.pose[3] + sh.pose[7] * sh.pose[7] + sh.pose[11] * sh.pose[11] +
                  sh.intr[0] * sh.intr[0] + sh.intr[1] * sh.intr[1] + sh.intr[2] * sh.intr[2];
      if (MODEL == VGG_SIMPLE_RADIAL) xn += sh.intr[3] * sh.intr[3];
      const double x_norm = sqrt(xn);
      const double cost_change = sh.cost - c_cost;
      const double rho = cost_change / sh.model_change;
      const bool good = rho > opt.min_relative_decrease;
      sh.state = ST_EVAL_CAND;
      if (step_norm <= opt.parameter_tolerance * (x_norm + opt.parameter_tolerance)) {
        sh.termination = VGG_BA_CONVERGENCE_PARAMETER;
        sh.state = ST_DONE;
      } else if (fabs(cost_change) <= opt.function_tolerance * sh.cost) {
        // Ceres 2.x TrustRegionMinimizer::Minimize returns from FunctionToleranceReached() BEFORE IsStepSuccessful() /
        // HandleSuccessfulStep(): the candidate of the terminating iteration is discarded, x stays the last accepted point
        sh.termination = VGG_BA_CONVERGENCE_FUNCTION;
        sh.state = ST_DONE;
      } else if (good) {
        for (int i = 0; i < 12; ++i) sh.pose[i] = sh.pose_c[i];
        for (int i = 0; i < 4; ++i) sh.intr[i] = sh.intr_c[i];
        sh.successful++;
        const double t = 2.0 * rho - 1.0;
        sh.radius = fmin(opt.max_trust_region_radius, sh.radius / fmax(1.0 / 3.0, 1.0 - t * t * t));
        sh.decrease = 2.0;
        sh.state = ST_ACCEPT;
      } else {
        sh.radius /= sh.decrease;
        sh.decrease *= 2.0;
      }
    }
    if (read_state() == ST_ACCEPT) {
      evaluate(sh.pose, sh.intr, true);
      if (tid == 0) {
        unpack();
        sh.state = ST_EVAL_CAND;
        if (grad_max() <= opt.gradient_tolerance) {
          sh.termination = VGG_BA_CONVERGENCE_GRADIENT;
          sh.state = ST_DONE;
        }
      }
    }
  }

  if (tid < 12) poses[(size_t)s * 12 + tid] = sh.pose[tid];
  if (tid < 4) intr[(size_t)s * 4 + tid] = sh.intr[tid];
  if (tid == 0) {
    summary_d[s * 4 + 1] = sh.cost;
    summary_d[s * 4 + 2] = sh.radius;
    summary_d[s * 4 + 3] = (double)count;
    summary_i[s * 4 + 0] = sh.it;
    summary_i[s * 4 + 1] = sh.successful;
    summary_i[s * 4 + 2] = sh.termination;
    summary_i[s * 4 + 3] = 0;
  }
}

}  // namespace
}  // namespace vgg

extern "C" {

void vgg_pose_default_options(vgg_pose_options* o) {
  if (!o) return;
  o->max_num_iterations = 100;
  o->max_num_consecutive_invalid_steps = 5;
  o->min_inliers = 0;
  o->reserved = 0;
  o->function_tolerance = 1e-6;
  o->gradient_tolerance = 1.0;
  o->parameter_tolerance = 1e-8;
  o->initial_trust_region_radius = 1e4;
  o->max_trust_region_radius = 1e16;
  o->min_trust_region_radius = 1e-32;
  o->min_relative_decrease = 1e-3;
  o->min_lm_diagonal = 1e-6;
  o->max_lm_diagonal = 1e32;
  o->loss_function_scale = 1.0;
  o->max_reproj_error = 0.0;
}

int vgg_pose_refinement(int S, int P, int camera_model, const float* uv, const uint8_t* inlier,
                        const uint8_t* frame_flags, const double* points, double* poses, double* intr,
                        const vgg_pose_options* opt, uint8_t* inlier_used, double* summary_d, int32_t* summary_i,
                        void* stream) {
  using namespace vgg;
  g_launch_count = 0;
  VGG_REQUIRE(S >= 0 && P >= 0, "negative size");
  VGG_REQUIRE(camera_model == VGG_SIMPLE_PINHOLE || camera_model == VGG_SIMPLE_RADIAL, "camera model");
  VGG_REQUIRE(opt != nullptr, "options");
  if (S == 0) return VGG_OK;
  VGG_REQUIRE(uv && inlier && frame_flags && points && poses && intr && inlier_used && summary_d && summary_i,
              "null pointer");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (camera_model == VGG_SIMPLE_PINHOLE)
    pose_refine_kernel<VGG_SIMPLE_PINHOLE><<<S, PT, 0, st>>>(S, P, uv, inlier, frame_flags, points, poses, intr, *opt,
                                                             inlier_used, summary_d, summary_i);
  else
    pose_refine_kernel<VGG_SIMPLE_RADIAL><<<S, PT, 0, st>>>(S, P, uv, inlier, frame_flags, points, poses, intr, *opt,
                                                            inlier_used, summary_d, summary_i);
  VGG_LAUNCH_CHECK();
  return VGG_OK;
}

}  // extern "C"
