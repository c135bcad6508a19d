// What the LM driver (csrc/ba_solve.cu) and its kernels (csrc/ba_schur.cu, csrc/ba_pcg.cu) agree on: scalar slots, the
// host's record, the reduced-system buffer and the reduction over the ranks of a track-sharded solve.
#pragma once
#include <math.h>
#include <stddef.h>
#include "common.cuh"

namespace vgg {

// scal[SCAL_DOUBLES]: this rank's scalars of one LM iteration (cam_step, point_step, gradmax, point_prep, xnorm_kernel)
enum : int {
  SCAL_CAM_QUAD = 0, SCAL_CAM_STEP2 = 1, SCAL_PT_QUAD = 2, SCAL_PT_STEP2 = 3, SCAL_GMAX_C = 4, SCAL_GMAX_P = 5,
  SCAL_PT_FAIL = 6, SCAL_CAM_BAD = 7, SCAL_XNORM_C = 8, SCAL_DOUBLES = 16,
};
// small[SMALL_VEC + Dpad]: what the candidate sums over the ranks, then from SMALL_VEC the frame flags (before the loop)
// or the candidate's camera gradient; SMALL_GMAX_P is the max slot of the fabric's all-reduce
enum : int {
  SMALL_COST = 0, SMALL_PT_QUAD = 1, SMALL_PT_STEP2 = 2, SMALL_PT_FAIL = 3, SMALL_GMAX_P = 4, SMALL_XNORM_P = 5,
  SMALL_MODEL_CHANGE = 6, SMALL_VEC = 8,
};
// int info[INFO_INTS]; INFO_LIST: the flag word of an observation list's check (before the loop)
enum : int { INFO_CHOL = 0, INFO_TRSV = 1, INFO_FABRIC = 2, INFO_LIST = 3, INFO_INTS = 4 };

// The record pack_scalars_kernel gathers for the host's one read per iteration (cg: the CG state of csrc/ba_pcg.h).
// The host reads REC_DOUBLES of it, REC_DOUBLES_CG in an iterative solve, into a buffer of REC_CAP.
struct LmRecord {
  double scal[8], small[8], chol_info, trsv_info, xnorm_c, fabric_timeout, cg[5];
  double cost() const { return small[SMALL_COST]; }
  // max of the camera and point gradient max-norms; a NaN in either (gradmax_kernel keeps them) stays NaN, so that a
  // NaN gradient is never taken for convergence
  double gmax() const {
    return isnan(scal[SCAL_GMAX_C]) || isnan(scal[SCAL_GMAX_P]) ? NAN : fmax(scal[SCAL_GMAX_C], scal[SCAL_GMAX_P]);
  }
};
#define VGG_REC(field) ((int)(offsetof(LmRecord, field) / sizeof(double)))
enum : int { REC_DOUBLES = 24, REC_DOUBLES_CG = 28, REC_CAP = 32 };

// the reduced-system buffer [D x Dpad matrix | rhs | hdiag | gvec], each vector Dpad long
struct Reduced {
  double *S, *rhs, *hdiag, *gvec;
};
inline size_t reduced_doubles(int D, int Dpad) { return (size_t)D * Dpad + 3 * (size_t)Dpad; }
inline Reduced reduced_view(double* base, int D, int Dpad) {
  return Reduced{base, base + (size_t)D * Dpad, base + (size_t)(D + 1) * Dpad, base + (size_t)(D + 2) * Dpad};
}

// Sums and maxima over the ranks of a track-sharded solve: in-kernel over the fabric (csrc/fabric.cu), else through the
// caller's all-reduce hook, else (one GPU) nothing.  Defined in csrc/ba_solve.cu.
struct Fabric;
struct Ranks {
  Fabric* fab;
  vgg_allreduce_fn fn;
  void* user;
  cudaStream_t st;
  bool sharded() const { return fab || fn; }
  int sum(double* vec, size_t count) const;
  int max(double* slot) const;
  // small[0, count) summed and scal[SCAL_GMAX_P] maximised around gradmax(), which fills scal's max-norms
  template <class Gradmax>
  int candidate(double* small, size_t count, double* scal, Gradmax gradmax) const;
};

}  // namespace vgg
