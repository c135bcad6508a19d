/*
 * vggsfm_b200 -- C ABI of the H100-native (sm_90a) geometry hot path for VGGSfM.
 *
 * The reference (facebookresearch/vggsfm @ e1d9d2e) has no FFI of its own: its seam for this path
 * is ordinary Python symbols plus the pycolmap object API (SURVEY.md section 8b).  Every entry
 * point below names the reference call site it replaces.  All pointers are DEVICE pointers owned
 * by the caller unless marked "host"; `stream` is a cudaStream_t passed as void*; no entry point
 * allocates device memory (the caller passes a workspace sized by the matching *_workspace_bytes).
 * Return value: 0 on success, negative VGG_E* on error; vgg_last_error() gives the message.
 *
 * Layouts (row-major, densely packed):
 *   observations  uv   float  [S,N,2]   pixels (or normalised coordinates where stated)
 *                 mask uint8  [S,N]     1 = observation participates
 *   cameras       poses  double [S,12]  cam_from_world R|t, 3x4 row-major
 *                 intr   double [S,4]   f, cx, cy, k   (k unused for SIMPLE_PINHOLE)
 *   points        double [N,3]
 */
#ifndef VGGSFM_B200_H
#define VGGSFM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VGG_OK 0
#define VGG_EINVAL (-1)
#define VGG_ECUDA (-2)
#define VGG_EWORKSPACE (-3)
#define VGG_ESOLVER (-4)

#define VGG_SIMPLE_PINHOLE 0
#define VGG_SIMPLE_RADIAL 1

#define VGG_INTR_CONST 0      /* intrinsics held constant (video_runner.py:813-815)            */
#define VGG_INTR_PER_FRAME 1  /* one pycolmap.Camera per frame (tensor_to_pycolmap.py:78-110)  */
#define VGG_INTR_SHARED 2     /* shared_camera=True: one Camera for all frames                 */

const char* vgg_last_error(void);
int vgg_version(void);

/* ------------------------------------------------------------------------------------------- */
/* Bundle adjustment: replaces pycolmap.bundle_adjustment(reconstruction, ba_options)           */
/* (vggsfm/utils/triangulation.py:213,1050,1142; vggsfm/runners/video_runner.py:508,1321-1331)  */
/* and the tensor<->Reconstruction marshalling around it (tensor_to_pycolmap.py:16-214).        */
/* ------------------------------------------------------------------------------------------- */

typedef struct vgg_ba_problem {
  int32_t S, N;
  int32_t camera_model;        /* VGG_SIMPLE_* */
  int32_t intr_mode;           /* VGG_INTR_*   */
  const float* uv;             /* [S,N,2] pixels */
  const uint8_t* mask;         /* [S,N] */
  const uint8_t* param_const;  /* [S*dc+ns] 1 = reduced parameter held constant (gauge, fixed poses) */
  const uint8_t* point_const;  /* [N] 1 = point held constant (video_runner.py:821-829), or NULL */
  double* poses;               /* [S,12] in/out */
  double* intr;                /* [S,4]  in/out */
  double* points;              /* [N,3]  in/out */
} vgg_ba_problem;

/* Ceres solver options as COLMAP's BundleAdjustmentOptions sets them (triangulation_helpers.py:626-635). */
typedef struct vgg_ba_options {
  int32_t max_num_iterations;
  int32_t max_num_consecutive_invalid_steps;
  int32_t jacobi_scaling;
  int32_t reserved;
  double function_tolerance, gradient_tolerance, parameter_tolerance;
  double initial_trust_region_radius, max_trust_region_radius, min_trust_region_radius;
  double min_relative_decrease, min_lm_diagonal, max_lm_diagonal;
} vgg_ba_options;

typedef struct vgg_ba_summary {
  int32_t iterations, successful, termination, reserved;
  double initial_cost, final_cost, final_radius;
  double device_ms;            /* CUDA-event time of the LM loop on `stream` */
  int64_t kernel_launches;     /* kernels of this library launched by the call */
} vgg_ba_summary;

/* termination codes */
#define VGG_BA_NO_CONVERGENCE 0
#define VGG_BA_CONVERGENCE_GRADIENT 1
#define VGG_BA_CONVERGENCE_FUNCTION 2
#define VGG_BA_CONVERGENCE_PARAMETER 3
#define VGG_BA_MIN_TRUST_REGION 4
#define VGG_BA_FAILURE 5

/* Sum/max all-reduce hook over track shards (one process per GPU).  `buf` is a device pointer
 * inside the caller's workspace; op 0 = sum, 1 = max, on `stream`.  NULL = single GPU. */
typedef int (*vgg_allreduce_fn)(void* user, double* buf, size_t count, int op, void* stream);

/* Fused reduction over NVLink/NVSwitch: the reduced camera system [D x Dpad | rhs | diag | g] lives in symmetric
 * (peer-mapped) memory and is reduced by the kernels that produce it, so the LM loop needs no separate collective.
 * ar_local and ar_multicast address the same allocation (e.g. torch.distributed._symmetric_memory); the assemble /
 * Schur kernels add the small blocks with multimem.red on the multicast address.  The SYRK reduce-scatters the lower
 * triangle's 128-row blocks onto their owners (block b -> rank b mod world) with system-scope REDs over NVLink, every
 * rank gathers the others by peer loads, and the barriers and the small cost/gradient all-reduces are kernels on the
 * same allocation -- no NCCL call, no host callback inside the LM loop, inbound traffic per GPU independent of the
 * number of ranks, bit-identical systems on all ranks.  The all-reduce hook is not called. */
typedef struct vgg_ba_fabric {
  double* ar_local;
  double* ar_multicast;
  size_t ar_doubles;     /* >= vgg_ba_reduced_system_doubles() */
  /* world in 2..8, rank = this process.  peer_base[r] = rank r's base address of the SAME symmetric allocation
   * (ar_local == peer_base[rank]), which must hold total_doubles >= vgg_ba_fabric_doubles() and be zero-filled once
   * when it is created.  vgg_ba_solve_fabric returns VGG_EINVAL without them. */
  int32_t world, rank;
  double* peer_base[8];
  size_t total_doubles;
} vgg_ba_fabric;

void vgg_ba_default_options(vgg_ba_options* opt);
int vgg_ba_dims(int camera_model, int intr_mode, int* dc, int* ns);
int vgg_ba_workspace_bytes(int S, int N, int camera_model, int intr_mode, size_t* bytes);

/* Fused residual + analytic 2x(dc+3) Jacobian + normal-equation block kernel (one launch).
 * Outputs (all double): cost[1]; camrec[S,KR] = per frame (g_c[dc] | H_cc upper-packed | H_cs[6,ns]);
 * g_p[N,3]; H_pp[N,6] (xx,xy,xz,yy,yz,zz); W[N, pitch, 3] track-major coupling blocks J_c^T J_p with
 * row = s*dc+i (shared-intrinsics rows at S*dc..) and pitch = D rounded up to even, D = S*dc+ns;
 * shared[8] = (g_s[2], H_ss xx,xy,yy).  KR = vgg_ba_camrec_len().  The last int argument is the number of
 * tracks each warp walks: 0 = choose, otherwise a positive multiple of 4 (the observation loads of a warp are
 * vectorised over 4 tracks); any other value returns VGG_EINVAL before anything is launched. */
int vgg_ba_camrec_len(int camera_model, int intr_mode);
int vgg_ba_build_blocks(const vgg_ba_problem* prob, double* cost, double* camrec, double* g_p,
                        double* H_pp, double* W, double* shared, int tracks_per_warp, void* stream);

/* Schur complement of the point blocks onto the camera system (second kernel of the path):
 * given the blocks above (without W: the coupling blocks are rebuilt from prob's observations and state), the Jacobi
 * scales and the trust-region radius, writes
 * Sraw[D,Dpad] (symmetric, only the row-major lower triangle valid) = H_cc - sum_j W_j V_j^-1 W_j^T and rhs[Dpad] =
 * -(g_c - sum_j W_j V_j^-1 g_pj).  Exposed for the parity tests and profiling. */
int vgg_ba_schur(const vgg_ba_problem* prob, const double* camrec, const double* g_p,
                 const double* H_pp, const double* shared, const double* scale_p,
                 double radius, double min_diag, double max_diag, void* workspace, size_t ws_bytes,
                 double* Sraw, double* rhs, int* Dpad_out, void* stream);

/* Blocked Cholesky of the reduced camera system (csrc/chol.cu): in-place factorisation of the row-major
 * lower triangle of A [n x n], leading dimension lda (any even lda >= n, A 16-byte aligned), replacing the potrf inside
 * Ceres' DENSE_SCHUR.  On return the lower triangle holds L and the strict upper triangle L^T.  Nothing outside the
 * n x n matrix is read or written, and the input in the strict upper triangle is never used (it may hold anything).
 * workspace >= ceil(n/128)*131072 + 1024 bytes (n <= 24000); *info_host = 0, the 1-based index of the failing pivot, or
 * INT_MAX if the in-kernel hand-off between CTAs stalled (bounded spin; never seen, reported instead of hanging). */
int vgg_cholesky_lower(int n, int lda, double* A, void* workspace, size_t ws_bytes, int* info_host, void* stream);

/* The Schur SYRK step on the INT8 tensor cores (csrc/syrk_i8.cu): Cmat[Dpad,Dpad] -= Zt^T Zt for Zt double [Kpad,Dpad]
 * (Dpad a multiple of 128), FP64-equivalent through `slices` (3..7; 7 = 54 fractional bits) int8
 * Ozaki slices on wgmma s8 with exact int32 accumulation in registers.  The row-major LOWER triangle is written.
 * vgg_ba_solve runs the FP64 tensor-core SYRK of csrc/ba_schur.cu instead (faster on H100); this one is kept for the
 * parity tests and profiling. */
int vgg_syrk_ozaki_workspace_bytes(int Kpad, int Dpad, int slices, size_t* bytes);
int vgg_syrk_ozaki(int Kpad, int Dpad, const double* Zt, double* Cmat, int slices, void* workspace, size_t ws_bytes,
                   void* stream);
/* Whole Levenberg-Marquardt solve (Ceres trust-region semantics).  `trace` is a HOST array
 * [max_num_iterations, 8] (it, cost, candidate_cost, model_change, rho, radius, step_norm, flags) or NULL. */
int vgg_ba_solve(const vgg_ba_problem* prob, const vgg_ba_options* opt, void* workspace,
                 size_t ws_bytes, vgg_allreduce_fn allreduce, void* allreduce_user,
                 vgg_ba_summary* summary, double* trace, void* stream);
int vgg_ba_reduced_system_doubles(int S, int camera_model, int intr_mode, size_t* doubles);
int vgg_ba_fabric_doubles(int S, int camera_model, int intr_mode, size_t* doubles);
int vgg_ba_solve_fabric(const vgg_ba_problem* prob, const vgg_ba_options* opt, void* workspace,
                        size_t ws_bytes, vgg_allreduce_fn allreduce, void* allreduce_user,
                        const vgg_ba_fabric* fabric, vgg_ba_summary* summary, double* trace, void* stream);

/* ------------------------------------------------------------------------------------------- */
/* Absolute-pose refinement: replaces the per-frame loop around pycolmap.pose_refinement        */
/* (vggsfm/utils/triangulation.py:260-479 refine_pose, :482-647 init_refine_pose).               */
/* ------------------------------------------------------------------------------------------- */

/* COLMAP AbsolutePoseRefinementOptions + the Ceres defaults behind it, plus the two pre-filters the
 * reference applies around the call: max_reproj_error > 0 ANDs the mask with (depth > 0 and squared
 * reprojection error <= max^2) at the input camera (triangulation.py:298-315); a frame is refined only
 * when its effective inlier count is > min_inliers (:386, :585). */
typedef struct vgg_pose_options {
  int32_t max_num_iterations;
  int32_t max_num_consecutive_invalid_steps;
  int32_t min_inliers;
  int32_t reserved;
  double function_tolerance, gradient_tolerance, parameter_tolerance;
  double initial_trust_region_radius, max_trust_region_radius, min_trust_region_radius;
  double min_relative_decrease, min_lm_diagonal, max_lm_diagonal;
  double loss_function_scale;   /* ceres::CauchyLoss scale */
  double max_reproj_error;      /* pixels; <= 0 disables the pre-filter */
} vgg_pose_options;

#define VGG_POSE_SKIPPED 6       /* frame_flags bit0 clear */
#define VGG_POSE_FEW_INLIERS 7   /* effective inliers <= min_inliers: pose left unchanged */

void vgg_pose_default_options(vgg_pose_options* opt);

/* One launch, one CTA per frame.  uv float [S,P,2] pixels; inlier uint8 [S,P]; frame_flags uint8 [S]
 * (bit0 refine this frame, bit1 refine_focal_length, bit2 refine_extra_params); points double [P,3]
 * (constant); poses [S,12] / intr [S,4] in/out.  Outputs: inlier_used uint8 [S,P] (the effective mask),
 * summary_d double [S,4] = (initial_cost, final_cost, final_radius, effective inliers), summary_i int32
 * [S,4] = (iterations, successful steps, termination VGG_BA_* / VGG_POSE_*, 0). */
int vgg_pose_refinement(int S, int P, int camera_model, const float* uv, const uint8_t* inlier,
                        const uint8_t* frame_flags, const double* points, double* poses, double* intr,
                        const vgg_pose_options* opt, uint8_t* inlier_used, double* summary_d, int32_t* summary_i,
                        void* stream);

/* ------------------------------------------------------------------------------------------- */
/* Triangulation side (float64, like the reference's real pipeline: models/triangulator.py:91) */
/* ------------------------------------------------------------------------------------------- */

/* triangulate_tracks / triangulate_tracks_single_chunk (vggsfm/utils/triangulation.py:677-956):
 * fused LORANSAC.  extrinsics [S,12]; tracks_normalized double [S,N,2]; track_vis/track_score float
 * [S,N] (score may be NULL); pairs int32 [H0,2] = the hypothesis frame pairs drawn on the host exactly
 * like triangulation.py:804-813 (CPU torch.randperm).  Outputs: points double [N,3], inlier_num
 * int64 [N], inlier_mask uint8 [N,S]. */
int vgg_tri_workspace_bytes(int S, int N, int H0, int lo_num, size_t* bytes);
int vgg_triangulate_tracks(int S, int N, const double* extrinsics, const double* tracks_normalized,
                           const float* track_vis, const float* track_score, const int32_t* pairs, int H0,
                           int lo_num, double max_angular_error_deg, double min_tri_angle_deg, double* out_points,
                           int64_t* out_inlier_num, uint8_t* out_inlier_mask, void* workspace, size_t ws_bytes,
                           void* stream);

/* triangulate_by_pair (triangulation.py:45-135): frame 0 against frames 1..S-1.  Outputs [S-1,N,3],
 * cheirality uint8 [S-1,N] (1 = in front of both), angle double [S-1,N] degrees.  workspace >= S*24 B. */
int vgg_triangulate_by_pair(int S, int N, const double* extrinsics, const double* tracks_normalized,
                            double* out_points, uint8_t* out_cheirality, double* out_angle_deg, void* workspace,
                            size_t ws_bytes, void* stream);

/* filter_all_points3D / _single_chunk (vggsfm/utils/triangulation_helpers.py:133-307).  points2d is
 * float or double [S,P,2]; intrinsics9 [S,9] row-major K; extra_params [S] SIMPLE_RADIAL k or NULL;
 * out_valid uint8 [P]; out_detail uint8 [S,P] or NULL (return_detail).  workspace >= S*24 B. */
int vgg_filter_points3d(int S, int P, const double* points3d, const void* points2d, int points2d_is_f64,
                        const double* extrinsics, const double* intrinsics9, const double* extra_params,
                        double max_reproj_error, double min_tri_angle_deg, int check_triangle, double hard_max,
                        uint8_t* out_valid, uint8_t* out_detail, void* workspace, size_t ws_bytes, void* stream);

/* project_3D_points / img_from_cam (triangulation_helpers.py:311-395): out_points2d [S,P,2] and/or
 * out_points_cam [S,3,P] (either may be NULL). */
int vgg_project_points(int S, int P, const double* points3d, const double* extrinsics, const double* intrinsics9,
                       const double* extra_params, double* out_points2d, double* out_points_cam, void* stream);

/* cam_from_img without distortion (triangulation_helpers.py:398-428): (uv - pp)/f in the input
 * precision (is_f64 selects float/double for tracks, focal2 [S,2], pp2 [S,2] and out). */
int vgg_normalize_tracks(int S, int N, const void* tracks, const void* focal2, const void* pp2, int is_f64, void* out,
                         void* stream);

/* iterative_undistortion (vggsfm/utils/distortion.py:27-99) for SIMPLE_RADIAL, with the reference's
 * semantics: damped Newton with a central-difference Jacobian and ONE global stop when the largest
 * squared step over all observations is < max_step_norm.  workspace >= 16 B. */
int vgg_undistort_simple_radial(int S, int N, const double* tracks_normalized, const double* extra_params,
                                int max_iterations, double max_step_norm, double rel_step_size, double* out,
                                int* iterations_run, void* workspace, size_t ws_bytes, void* stream);

/* pycolmap.absolute_pose_estimation for the frames refine_pose cannot refine (vggsfm/utils/triangulation.py:404-433:
 * estimate_focal_length = True, ransac.max_error = 12) and for the video runner's PnP alignment
 * (vggsfm/runners/video_runner.py:985-998): P3P + LO-RANSAC, batched over frames AND over COLMAP's 31 focal-length
 * factors (0.2 + 4.8 (i/30)^2) in one launch, on caller-drawn minimal samples (u_samples double [num_trials,3], uniform
 * in [0,1), mapped to the frame's usable points).  uv float [S,P,2] pixels, mask uint8 [S,P] usable observations,
 * frame_flags uint8 [S] (0 = skip the frame), points double [P,3], intr double [S,4] = f,cx,cy,k.
 * Out: pose_out double [S,12] (R|t, written for successful frames only), focal_out double [S] (prior focal x best
 * factor), num_inliers_out int32 [S] (0 = no model: the reference's `None`), inlier_out uint8 [S,P].
 * The non-linear refinement COLMAP runs afterwards is vgg_pose_refinement.  P <= 9751 per call: the
 * frame's usable points live in 21 P + 16 bytes of dynamic shared memory, capped at 200 KB; a larger P returns
 * VGG_EINVAL before anything is launched. */
int vgg_pnp_workspace_bytes(int S, int estimate_focal_length, size_t* bytes);
int vgg_absolute_pose_estimation(int S, int P, int camera_model, const float* uv, const uint8_t* mask,
                                 const uint8_t* frame_flags, const double* points, const double* intr,
                                 const double* u_samples, int num_trials, int estimate_focal_length, double max_error,
                                 double* pose_out, double* focal_out, int* num_inliers_out, uint8_t* inlier_out,
                                 void* workspace, size_t ws_bytes, void* stream);

/* ------------------------------------------------------------------------------------------- */
/* Two-view stage (float64 arithmetic; float or double tracks)                                 */
/* ------------------------------------------------------------------------------------------- */

/* estimate_fundamental (vggsfm/two_view_geo/fundamental.py:43-183) for B pairs at once: 7-point minimal solves on
 * caller-drawn samples (int32 [T,7], HOST memory: generate_samples, utils.py:39-60), Sampson scoring, two rounds of
 * 8-point local refinement from the top lo_num (then lo_num/2) candidates, the residual indicator with its batch-wide
 * threshold (utils.py:63-87), first argmax.  points1/points2 [B,N,2] float (points_are_f64 = 0) or double,
 * valid_mask uint8 [B,N] or NULL, threshold = max_error^2 (squared) or max_error.  Outputs: fmat_out double [B,3,3],
 * inlier_num_out int32 [B], inlier_mask_out uint8 [B,N], residuals_out double [B,N] (1e6 at invalid matches).
 * VGG_EINVAL before any launch when N < 7, T < 7, lo_num outside [1, 3T], N > 190000 or a sample is outside [0, N). */
int vgg_twoview_workspace_bytes(int B, int N, int T, int lo_num, size_t* bytes);
int vgg_estimate_fundamental(int B, int N, const void* points1, const void* points2, int points_are_f64,
                             const uint8_t* valid_mask, const int32_t* samples, int T, int lo_num, double threshold,
                             int squared, int second_refine, double* fmat_out, int32_t* inlier_num_out,
                             uint8_t* inlier_mask_out, double* residuals_out, void* workspace, size_t ws_bytes,
                             void* stream);

/* inlier_by_fundamental (utils.py:300-322): inlier_mask_out uint8 [B,N] = Sampson residual of (points1, points2)
 * under fmat double [B,3,3] <= threshold (squared distance, or its square root + eps when squared = 0). */
int vgg_fundamental_inliers(int B, int N, const void* points1, const void* points2, int points_are_f64,
                            const double* fmat, double threshold, int squared, uint8_t* inlier_mask_out, void* stream);

/* estimate_preliminary.py:148-164: E = K^T F K with the default K (f = max(W, H), principal point (W/2, H/2)),
 * decompose_essential_matrix (essential.py:36-83) and remove_cheirality (utils.py:325-448) over all N matches of the
 * pair.  Out: R_out double [B,3,3], t_out double [B,3], E_out double [B,3,3]. */
int vgg_relative_pose_from_fundamental(int B, int N, const void* points1, const void* points2, int points_are_f64,
                                       const double* fmat, double width, double height, double* R_out, double* t_out,
                                       double* E_out, void* stream);

/* poselib.estimate_fundamental as estimate_preliminary_cameras_poselib (vggsfm/two_view_geo/estimate_preliminary.py:37-95)
 * calls it, for B pairs at once: LO-MSAC over the valid matches with PoseLib's seeded sampler, the real-root 7-point
 * solver with the real focal check, truncated-loss LM local optimisation, PoseLib's dynamic stopping rule, and a
 * Cauchy polish on the inliers (restated in oracle/poselib_oracle.py).  points1/points2 [B,N,2] float
 * (points_are_f64 = 0) or double pixels, valid_mask uint8 [B,N] or NULL (all valid), max_error = the epipolar threshold
 * in pixels (Sampson distance), max_iterations / min_iterations as RansacOptions, seed = RansacOptions.seed (the
 * reference uses the defaults: min_iterations 1000, seed 0).  Outputs: fmat_out double [B,3,3] (|F|_F = 1, entry of
 * largest magnitude positive; 0 when a pair has fewer than 7 valid matches or no model), inlier_num_out int32 [B],
 * inlier_mask_out uint8 [B,N] (invalid matches 0), iterations_out int32 [B] (RANSAC iterations run).  The call
 * synchronises with `stream` once per chunk of trials.  VGG_EINVAL before any launch when B or N is negative,
 * B * N >= 2^31, max_iterations < 1, min_iterations < 0 or max_error is not positive and finite. */
int vgg_msac_fundamental_workspace_bytes(int B, int N, int max_iterations, int min_iterations, size_t* bytes);
int vgg_estimate_fundamental_msac(int B, int N, const void* points1, const void* points2, int points_are_f64,
                                  const uint8_t* valid_mask, double max_error, int max_iterations, int min_iterations,
                                  unsigned long long seed, double* fmat_out, int32_t* inlier_num_out,
                                  uint8_t* inlier_mask_out, int32_t* iterations_out, void* workspace, size_t ws_bytes,
                                  void* stream);

/* ------------------------------------------------------------------------------------------- */
/* Tracker correlation inner loop (float32 math on float or half feature pyramids)             */
/* ------------------------------------------------------------------------------------------- */

/* CorrBlock.__init__ (vggsfm/models/track_modules/blocks.py:339-361): feature pyramid by repeated
 * avg_pool2d(2,2), stored channels-last [BS,H_l,W_l,C] per level in `elem_size` bytes per element
 * (4 = float, 2 = half as under the reference's fp16 autocast, runners/runner.py:418).
 * fmaps_nchw is float [BS,C,H,W].  The half pyramid needs a float scratch (sizes from *_bytes). */
int vgg_corr_pyramid_bytes(int BS, int C, int H, int W, int num_levels, int elem_size, size_t* pyramid_bytes,
                           size_t* scratch_bytes);
int vgg_corr_build_pyramid(int BS, int C, int H, int W, int num_levels, const float* fmaps_nchw, int elem_size,
                           void* pyramid, void* scratch, void* stream);

/* CorrBlock.corr + CorrBlock.sample fused (blocks.py:363-416; border_padding=1 gives
 * EfficientCorrBlock.sample, :433-471).  targets float [BS,N,C], coords float [BS,N,2] (x,y) in level-0
 * pixels, out float [BS,N,num_levels*(2r+1)^2] with out[a*(2r+1)+b] sampled at (x+a-r, y+b-r).  Coordinates follow
 * grid_sample on CUDA: a NaN or ±inf coordinate reads 0 with zero padding; border padding clamps it (NaN -> 0).
 * BS * N == 0 returns VGG_OK without a launch, and the pointers may then be null (also for vgg_corr_tc_sample). */
int vgg_corr_sample(int BS, int N, int C, int H, int W, int num_levels, int radius, const void* pyramid, int elem_size,
                    const float* targets, const float* coords, int border_padding, float* out, void* stream);

/* The same CorrBlock.corr + CorrBlock.sample for the coarse tracker's C = 128 maps ON THE TENSOR CORES
 * (csrc/corr_tc.cu: wgmma f16 M=64 x N=256 x K=128 per warpgroup into registers, footprint extraction from the register
 * accumulators; the dense fp16 product of blocks.py:413 without ever storing the volume).  Zero padding only; map width a
 * power of two.  vgg_corr_tc_build turns the HALF channels-last pyramid of vgg_corr_build_pyramid into operand tile
 * images once per CorrBlock (tile_bytes from vgg_corr_tc_bytes); vgg_corr_tc_sample needs `target_bytes` of scratch for
 * the fp16 target tiles of the call.  Same targets / coords / out layout as vgg_corr_sample. */
int vgg_corr_tc_supported(int C, int H, int W, int num_levels, int radius);
int vgg_corr_tc_bytes(int BS, int C, int H, int W, int num_levels, int N, size_t* tile_bytes, size_t* target_bytes);
int vgg_corr_tc_build(int BS, int C, int H, int W, int num_levels, const void* pyramid_half, void* tiles, void* stream);
int vgg_corr_tc_sample(int BS, int N, int C, int H, int W, int num_levels, int radius, const void* tiles, const float* targets,
                       const float* coords, void* target_tiles, float* out, void* stream);

/* sample_features4d (vggsfm/models/utils.py:415-447; colour read-back at models/triangulator.py:324, query
 * features in the tracker): bilinear sampling, align_corners=True, border padding.  input float [B,C,H,W],
 * coords float [B,R,2] (x,y) pixels, out float [B,R,C]. */
int vgg_sample_features4d(int B, int C, int H, int W, int R, const float* input_nchw, const float* coords, float* out,
                          void* stream);

/* ------------------------------------------------------------------------------------------- */
/* Dense depth stage (align_dense_depth_maps, vggsfm/utils/utils.py:635-770), all frames per call */
/* ------------------------------------------------------------------------------------------- */

/* Frames' disparity maps are one CSR: frame f is float32 [H_f, W_f] row-major at map_offsets[f] (int64 [F+1]),
 * map_hw int32 [F,2] = (H_f, W_f).  Sparse samples are a CSR too: int32 offsets [F+1] into the per-sample arrays. */

/* utils.py:669-690: per observation i of frame uvd_frame[i], uvd double [n,3] = (u, v, depth): np.round (half to
 * even) of (u, v), bounds 0 <= u < W, 0 <= v < H, nearest-pixel disparity x_out (0 when out of bounds),
 * y_out = 1 / clip(depth, depth_min, depth_max), keep_out = x_out > 0. */
int vgg_depth_sparse_samples(int n_total, const int32_t* uvd_frame, const double* uvd, double depth_min,
                             double depth_max, const int64_t* map_offsets, const int32_t* map_hw, const float* disp,
                             float* x_out, double* y_out, uint8_t* keep_out, void* stream);

/* np.median(y) / divisor per frame (utils.py:695; the median is the mean of the two middle values for an even count,
 * NaN for none), each step one IEEE double operation.  y >= 0. */
int vgg_depth_median(int F, const int32_t* offsets, const double* y, double divisor, double* median_out,
                     void* stream);

/* RANSACRegressor(LinearRegression(), min_samples=2, residual_threshold=threshold[f], max_trials, loss=
 * "squared_error").fit(x[:, None], y) per frame (utils.py:700-709), x float32, y double.  begin() resets every frame;
 * each chunk() evaluates T trials (T <= vgg_depth_ransac_max_chunk()) of the R live frames `frames` int32 [R], the
 * trial's two sample indices in samples int32 [R,T,2] (drawn by the caller), and writes running_out uint8 [F] for
 * those frames (1 while n_trials < max_trials).  finish() writes scale / shift float32 [F] (coef_[0], intercept_),
 * n_trials / n_inliers int32 [F] (n_inliers -1 when no trial was kept: sklearn's "could not find a valid consensus
 * set") and inlier_mask uint8 in the sample CSR.  The final fit centres on numpy's float32 pairwise means of the
 * inliers, bitwise.  The workspace holds the per-frame state and one chunk's trials. */
int vgg_depth_ransac_workspace_bytes(int F, size_t* bytes);
int vgg_depth_ransac_max_chunk(void);
int vgg_depth_ransac_begin(int F, int max_trials, void* workspace, size_t ws_bytes, void* stream);
int vgg_depth_ransac_chunk(int F, const int32_t* offsets, const float* x, const double* y, const double* threshold,
                           int R, const int32_t* frames, int T, const int32_t* samples, uint8_t* running_out,
                           void* workspace, size_t ws_bytes, void* stream);
int vgg_depth_ransac_finish(int F, const int32_t* offsets, const float* x, const double* y, const double* threshold,
                            float* scale_out, float* shift_out, int32_t* n_trials_out, int32_t* n_inliers_out,
                            uint8_t* inlier_mask_out, void* workspace, size_t ws_bytes, void* stream);

/* utils.py:712-724 in one pass: disp != 0 -> disp * scale[f] + shift[f] (float32 ops, written back in place),
 * kept where 0 < disp <= 10000 and 0 elsewhere; depth_out = float32(1 / disp), 0 where disp == 0 or where 1 / disp
 * overflows to +inf (the reference zeroes infinite depths).  Frame f spans
 * the tiles tile_offsets[f] .. tile_offsets[f+1] (int64 [F+1]) of vgg_depth_tile_pixels() pixels each;
 * tile_counts int32 [n_tiles] (may be NULL) receives each tile's valid-pixel count. */
int vgg_depth_tile_pixels(void);
int vgg_depth_apply(int F, int64_t n_tiles, const int64_t* map_offsets, const int64_t* tile_offsets,
                    const float* scale, const float* shift, float* disp, float* depth_out, int32_t* tile_counts,
                    void* stream);

/* utils.py:728-765 (visual_dense_point_cloud): valid pixels (disp != 0: the rescaled disparity that
 * vgg_depth_apply wrote, so a valid pixel whose depth is 0 is still a point) in row-major order, compacted by
 * tile_base int64 [n_tiles + 1] (exclusive prefix of tile_counts): pixel (x, y) without +0.5 through cam_from_img
 * (cam_model VGG_SIMPLE_*, cam_params double [F,4] = f, cx, cy, k), times depth, through world_from_cam double
 * [F,3,4] (cam_from_world.inverse()).  Frame f's M_f points are one [2, M_f, 3] block of `out` double starting at
 * 6 * tile_base[tile_offsets[f]]: the world points, then rgb uint8 [pixels,3] / 255. */
int vgg_depth_unproject(int F, int64_t n_tiles, const int64_t* map_offsets, const int32_t* map_hw,
                        const int64_t* tile_offsets, const int64_t* tile_base, const float* depth, const float* disp,
                        const uint8_t* rgb,
                        const int32_t* cam_model, const double* cam_params, const double* world_from_cam,
                        double* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif
