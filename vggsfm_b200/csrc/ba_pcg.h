// The iterative (PCG) linear solver of the LM loop, csrc/ba_pcg.cu; used by csrc/ba_solve.cu.
#pragma once
#include "ba_lm.h"

namespace vgg {

constexpr int PCG_CHUNK = 10;             // CG iterations queued between two reads of the done flag
constexpr int PCG_RESET_PERIOD = 10;      // Ceres' residual_reset_period: r = b - A x every 10th iteration
constexpr int PCG_STATE_DOUBLES = 32;

// slots of the CG state (PcgBuffers::cg); [1..4] are what the host reads after each LM iteration (slot 0 is unused: the
// model change goes to the small all-reduce of the candidate, launch_pcg_model_change)
enum : int {
  CG_ITERS = 1, CG_TERM = 2, CG_ZETA = 3, CG_RREL = 4, CG_DONE = 5, CG_RHO = 6, CG_BETA = 7,
  CG_ALPHA = 8, CG_Q0 = 9, CG_BB = 10, CG_PRE_FAIL = 11,
  CG_TICKET_SLOT = 24,      // unsigned counter of the kernel's finished CTAs (reset by the last one)
};

// Device buffers of one solve (all [Dpad] unless noted), carved by make_layout in csrc/ba_solve.cu.  With track shards
// the partial sums of a rank are rhs | hdiag | gvec | acc | shared | camrec, carved back to back from `rhs` on:
// [rhs, rhs + red_doubles) is the one region the all-reduce hook sums once per LM iteration.
struct PcgBuffers {
  double *rhs, *hdiag, *gvec;   // reduced right-hand side (unscaled), diag(H_cc), camera gradient
  double *acc;                  // [9 * pcg_blocks]: sum Z_b Z_b^T of the Schur-Jacobi blocks
  double *shared, *camrec;      // [8], [S * KR]: copy of the camera records (H_cc, g) summed with the above
  size_t red_doubles;
  double *x, *r, *z, *q, *u;    // CG vectors; u = Dc v, the operand of the Schur part of the matvec
  double *qs;                   // Schur part of the matvec (summed over the ranks before it joins q)
  double *p[2];                 // search direction, alternating between iterations
  double *pinv;                 // [9 * pcg_blocks]: inverted preconditioner blocks
  double *cg;                   // [PCG_STATE_DOUBLES] scalars and termination
  double *slots;                // [pcg_slot_doubles]: per-CTA partials of the fixed-order CG reductions
  double *tp;                   // [N * 3]: t_n = M_n M_n^T W_n^T u of the list matvec's point pass (list solve only)
};

// A validated vgg_ba_obs_list (csrc/ba_list.cu), M < 2^30: point-major uv / frame / point, frame-major frame_obs
struct ObsList {
  int M;
  const float2* uv;
  const int *frame, *point, *track_start, *frame_start, *frame_obs;
};

// the reduced operator of one LM iteration: the state, its camera records, point blocks M, camera scales and damping
struct PcgOp {
  const vgg_ba_problem* p;
  int dc, ns, KR;
  const double *camrec, *shared_in, *M, *sc_c;
  double radius, min_diag, max_diag;
  const int* fg_tracks;
  const ObsList* obs;           // the observation list, or null: the problem's grid
};

int pcg_blocks(int S, int ns);
size_t pcg_slot_doubles(int S, int dc, int ns);
int launch_pcg_assemble(const PcgOp& op, const double* q, const PcgBuffers& B, cudaStream_t st);
int launch_pcg_init(const PcgOp& op, const PcgBuffers& B, double* bvec, cudaStream_t st);
int launch_pcg_matvec(const PcgOp& op, int pmode, const double* p_old, double* p_new, const PcgBuffers& B,
                      cudaStream_t st);
int launch_pcg_combine(int D, double* q, const double* qs, cudaStream_t st);
int pcg_run(const PcgOp& op, const vgg_ba_linear_solver& lin, const PcgBuffers& B, double* bvec, const Ranks& ranks,
            cudaStream_t st);
int launch_pcg_model_change(const vgg_ba_problem* p, const double* M, const double* g_p, const double* wacc,
                            const double* d_c, const int* fg_tracks, double* out, cudaStream_t st);

// the same steps on an observation list (csrc/ba_list.cu); *bad (zeroed by the caller) gets a non-zero word of
// LIST_BAD_* bits for a malformed list
int launch_list_validate(int S, int N, const ObsList& L, int* bad, cudaStream_t st);
int launch_list_observed(int S, int N, const ObsList& L, uint8_t* point_seen, double* frame_seen, cudaStream_t st);
int launch_list_blocks(const vgg_ba_problem* p, const ObsList& L, double* cost, double* camrec, double* g_p,
                       double* H_pp, double* shared_out, cudaStream_t st);
int launch_list_rhs_jacobi(const PcgOp& op, const double* q, const PcgBuffers& B, cudaStream_t st);
int launch_list_schur(const PcgOp& op, const PcgBuffers& B, cudaStream_t st);
int launch_list_backsub(const vgg_ba_problem* p, const ObsList& L, const double* d_c, double* wacc, cudaStream_t st);
int launch_list_model_change(const vgg_ba_problem* p, const ObsList& L, const double* M, const double* g_p,
                             const double* wacc, const double* d_c, double* out, cudaStream_t st);

}  // namespace vgg
