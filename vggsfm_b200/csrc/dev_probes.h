// Development probes (NOT part of the public C ABI in include/vggsfm_b200.h): exported from the library for
// tools/syrk_i8_check.py, tools/microbench.py, bench.py's roofline and the tests only.
#pragma once
#ifdef __cplusplus
extern "C" {
#endif
/* Kernel-only timing of ba_blocks_kernel: while enabled, every build_blocks call records a CUDA event pair on its stream
 * directly around the kernel launch (the accumulator memsets before it are outside); last_ms waits for the second event
 * and returns the elapsed milliseconds of the most recent launch. */
int vgg_dev_blocks_timing(int enable);
int vgg_dev_blocks_last_ms(double* ms);
/* One-CTA probe of the in-shared-memory POTRF128 of csrc/chol.cu: A_host row-major SPD 128 x 128, L_host its factor,
 * prof13_host[0..5] = cycles per phase seen by warp 0, [6..11] by warp 1 (0 first leaf, 1 TRSM of the micro-panel,
 * 2 look-ahead section work, 3 wait at its barrier, 4 rank-32 DMMA update, 5 first leaf of the next sub-panel),
 * [12] = total cycles of the last of `reps` passes. */
int vgg_dev_chol128_probe(int reps, const double* A_host, double* L_host, long long* prof13_host);
/* The Schur SYRK of the LM loop (csrc/ba_schur.cu, FP64 tensor cores): Cmat -= Zt^T Zt into the row-major LOWER triangle
 * of Cmat [Dpad][Dpad] for Zt [Kpad][Dpad] (device pointers; Dpad % 128 == 0, Kpad % 16 == 0). */
int vgg_dev_syrk_f64(int Kpad, int Dpad, const double* Zt, double* Cmat, void* stream);
/* vgg_dev_syrk_f64 with a band hint, as vgg_ba_solve computes it from the visibility mask: ranges_host[2*rb], [2*rb+1]
 * = the 64-row k-block range outside which the 128-column row block rb of Zt is exactly zero (count = 2 * Dpad/128;
 * NULL, 0 = dense). */
int vgg_dev_syrk_f64_band(int Kpad, int Dpad, const double* Zt, double* Cmat, void* stream, const int* ranges_host,
                          int count);
/* Backward substitution U x = y (csrc/trsv.cu).  A_dev: row-major upper triangle, lda columns (the strictly lower
 * triangle is never read); y_dev[i * y_stride] = y_i.  stamps_host == NULL: the launcher of the LM loop (sentinel fill +
 * kernel), then a device synchronise.  Otherwise the kernel alone with per-block-row timestamps (ns, 6 per block row of
 * 64 rows: entry, diagonal block loaded, inverse ready, every x_j consumed, x_b published, right-hand side ready). */
int vgg_dev_trsv_probe(int n, int lda, const double* A_dev, const double* y_dev, size_t y_stride, double* x_dev,
                       long long* stamps_host);
/* Band hint of the most recent vgg_ba_solve (or vgg_dev_schur_build) on the calling thread (csrc/ba_solve.cu,
 * compute_band_hint).  meta_host[0..7] = {SYRK k-range hint active, factorisation band set, device tables for
 * ba_blocks / z_build / backsub made, nb (128-column row blocks), KB (64-row k blocks), frame groups of 32, arrow_blk, 0}.
 * Each non-null array receives its table if it was made: rb_range[2 nb], end_blk[nb], kb_rows[2 KB],
 * fg_tracks[2 groups]. */
int vgg_dev_last_band_hint(int* meta_host, int* rb_range, int* end_blk, int* kb_rows, int* fg_tracks);
/* vgg_cholesky_lower of a banded + arrow matrix: end_blk_host[b] = one past the last band block (128 rows) of block
 * column b, arrow_blk = first block of the dense arrow (NULL, 0 = dense). */
int vgg_dev_cholesky_band(int n, int lda, double* A, void* workspace, size_t ws_bytes, int* info_host, void* stream,
                          const int* end_blk_host, int count, int arrow_blk);
/* Trace of the most recent vgg_estimate_fundamental_msac on `workspace` (same B, N and iteration limits; waits for the
 * device): per pair the number of trials that ran local optimisation, the trial whose model won (-1: none) and the
 * first min(cap, 64) of those trials in order (-1 padded), all host arrays. */
int vgg_dev_msac_trace(int B, int N, int max_iterations, int min_iterations, const void* workspace, int cap,
                       int32_t* lo_runs_host, int32_t* win_trial_host, int32_t* lo_trials_host);
/* vgg_relative_pose_from_fundamental that also writes the cheirality vote: counts_dev[4 b + k] = points in front of both
 * cameras inside the depth window for candidate k (R1 t, R1 -t, R2 t, R2 -t) of pair b (device int32 [B, 4]). */
int vgg_dev_relative_pose_counts(int B, int N, const void* points1, const void* points2, int points_are_f64,
                                 const double* fmat, double width, double height, double* R_out, double* t_out,
                                 double* E_out, int32_t* counts_dev, void* stream);

/* vgg_ba_build_blocks with the band table of the LM solve's block kernel: fg_tracks_host[2g], [2g+1] = the track range
 * [lo, hi) outside which frame group g (32 frames) sees nothing (count = 2 * ceil(S/32); NULL, 0 = dense).  With a
 * table and tracks_per_warp = 0 the kernel runs the banded sizing of the solve (64 tracks per warp; the warps whose
 * track chunk misses their group's range return at once).  W = NULL runs the solve's variant, which stores no W.
 * The table goes to a device buffer that the next call with a table rewrites after a device synchronise. */
int vgg_dev_build_blocks_band(const vgg_ba_problem* prob, double* cost, double* camrec, double* g_p, double* H_pp,
                              double* W, double* shared, int tracks_per_warp, const int* fg_tracks_host, int count,
                              void* stream);
/* One schur_build of the LM loop (csrc/ba_solve.cu) at the given state, Jacobi point scales (device [N,3]) and radius:
 * point_prep, assemble_hc, z_build, syrk_f64 with the launchers of the solve.  banded = 0: dense plan; otherwise the
 * plan compute_band_hint makes from prob->mask (then also reported by vgg_dev_last_band_hint).  zt_nan = 1 fills Zt
 * with all-ones bytes (a NaN) instead of zeros before z_build, so the entries it writes can be told from the ones it
 * leaves; the SYRK is then not run (it adds every non-zero product, so a sentinel left in the padding columns would
 * reach rows beyond the reduced system) and Sraw holds assemble_hc's camera blocks only.  Each non-null device output
 * receives a copy: M [N,9] (row-major upper triangular), q [N,3], dpp [N,3], scal [16] (slot SCAL_PT_FAIL = 6 of csrc/ba_lm.h:
 * points whose 3x3 factorisation failed), Zt [Kpad,Dpad], Sraw [D,Dpad] (lower triangle valid), rhs [Dpad]; Kpad = 3N rounded up to 16, Dpad as in
 * vgg_ba_schur.  workspace as vgg_ba_workspace_bytes.  Waits for the device. */
int vgg_dev_schur_build(const vgg_ba_problem* prob, const double* camrec, const double* g_p, const double* H_pp,
                        const double* shared, const double* scale_p, double radius, double min_diag, double max_diag,
                        int banded, int zt_nan, void* workspace, size_t ws_bytes, double* M, double* q, double* dpp,
                        double* scal, double* Zt, double* Sraw, double* rhs, void* stream);
/* The work list of the Schur SYRK (csrc/ba_schur.cu launch_syrk, csrc/syrk_work.h) for nworkers persistent CTAs, on
 * the host, no launch: items_host[4w..4w+3] = (bi, bj, kb0, kb1) of item w (upper tile bi <= bj, k blocks [kb0, kb1)
 * of 64 rows), in the order CTAs take them (item w goes to CTA w mod nworkers).  ranges_host / count: the band hint of
 * vgg_dev_syrk_f64_band.  *nwork = the length; items_host = NULL only queries it, otherwise cap must cover it. */
int vgg_dev_syrk_work_list(int Kpad, int Dpad, const int* ranges_host, int count, int nworkers, int* items_host,
                           int cap, int* nwork);

/* The iterative solve's preparation at the given blocks (as vgg_ba_schur takes them), point scales scale_p [N,3], camera
 * scales scale_c [D] and radius, with prob->param_const / point_const taken as the solve's effective flags; then one
 * product y = A x of the scaled, damped reduced operator (csrc/ba_pcg.cu).  Outputs (device, each may be NULL): y_out [D],
 * b_out [D] (scaled right-hand side, pinned entries 0), pinv_out [9 * (3 S + (ns > 0))] (the inverted Schur-Jacobi
 * blocks, row-major 3x3: rotation, translation, intrinsics of each frame, then the shared block), state_out [32] (the CG
 * state after its initialisation).  workspace from vgg_ba_workspace_bytes_iterative. */
int vgg_dev_pcg_probe(const vgg_ba_problem* prob, const double* camrec, const double* g_p, const double* H_pp,
                      const double* shared_in, const double* scale_p, const double* scale_c, double radius,
                      double min_diag, double max_diag, const double* x_in, void* workspace, size_t ws_bytes,
                      double* y_out, double* b_out, double* pinv_out, double* state_out, void* stream);

#ifdef __cplusplus
}
#endif
