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
/* vgg_syrk_ozaki (csrc/syrk_i8.cu) with the band hint of vgg_dev_syrk_f64_band. */
int vgg_dev_syrk_ozaki_band(int Kpad, int Dpad, const double* Zt, double* Cmat, int slices, void* workspace,
                            size_t ws_bytes, void* stream, const int* ranges_host, int count);
/* Backward substitution U x = y (csrc/trsv.cu).  A_dev: row-major upper triangle, lda columns (the strictly lower
 * triangle is never read); y_dev[i * y_stride] = y_i.  stamps_host == NULL: the launcher of the LM loop (sentinel fill +
 * kernel), then a device synchronise.  Otherwise the kernel alone with per-block-row timestamps (ns, 6 per block row of
 * 64 rows: entry, diagonal block loaded, inverse ready, every x_j consumed, x_b published, right-hand side ready). */
int vgg_dev_trsv_probe(int n, int lda, const double* A_dev, const double* y_dev, size_t y_stride, double* x_dev,
                       long long* stamps_host);
/* Band hint of the most recent vgg_ba_solve on the calling thread (csrc/ba_solve.cu, compute_band_hint).
 * meta_host[0..7] = {SYRK k-range hint active, factorisation band set, device tables for
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

#ifdef __cplusplus
}
#endif
