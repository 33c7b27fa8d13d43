/*
 * cpd_b200.h -- C ABI of libcpd_b200.so: the CPD EM hot path on one H100 (sm_90a).
 *
 * The reference (neka-nat/probreg v0.3.7) has no C/FFI boundary for this path: the seam
 * is Python-level (probreg/cpd.py) plus one pybind11 module (probreg/_math).  Each entry
 * point below names the reference interface it stands in for.  All host pointers are
 * caller-owned, C-order, `double`; nothing is retained after a call returns.  One handle
 * owns one CUDA device + one stream and is not re-entrant.  Every function returns 0 on
 * success and a negative code on failure; cpd_last_error() then describes the failure.
 * There is no CPU fallback: without a CUDA device cpd_create fails.
 *
 * Coordinates are D = 2 or 3; clouds are (count x D) row-major.
 */
#ifndef CPD_B200_H
#define CPD_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct cpd_ctx cpd_ctx;

enum { CPD_OK = 0, CPD_ERR_ARG = -1, CPD_ERR_CUDA = -2, CPD_ERR_STATE = -3, CPD_ERR_NCCL = -4 };

/* transformation families: probreg/cpd.py:123 (RigidCPD), :195 (AffineCPD), :247 (NonRigidCPD) */
enum { CPD_TF_RIGID = 0, CPD_TF_AFFINE = 1, CPD_TF_NONRIGID = 2 };

/* Result of one M-step == probreg/cpd.py:18 MstepResult(transformation, sigma2, q) flattened.
 * rigid : rot (D x D row-major in lin[0..D*D)), t, scale            (cpd.py:192)
 * affine: b   (D x D row-major in lin),          t, scale == 1      (cpd.py:244)          */
typedef struct cpd_params {
    double lin[9];
    double t[3];
    double scale;
    double sigma2;
    double q;
    double n_p;       /* EstepResult.n_p of the E-step that fed this M-step (cpd.py:88) */
} cpd_params;

const char* cpd_last_error(void);
int cpd_version(void);

/* Number of CUDA devices visible (0 => every other call fails). */
int cpd_device_count(void);

/* -- handle ---------------------------------------------------------------------------
 * stream == NULL: the handle creates its own non-blocking stream.  Otherwise `stream` is a
 * cudaStream_t the caller owns (e.g. torch.cuda.current_stream().cuda_stream).
 * Replaces the backend selection of CoherentPointDrift.__init__ (cpd.py:42-59).        */
int cpd_create(cpd_ctx** out, int device, int dim, void* stream);
void cpd_destroy(cpd_ctx* h);

/* CoherentPointDrift.set_source (cpd.py:61-62) / the `source` ctor argument.            */
int cpd_set_source(cpd_ctx* h, const double* source, int64_t m);

/* The `target` argument of registration()/expectation_step (cpd.py:71,106).
 * `target` holds THIS handle's shard (n_local rows); n_global is the N of cpd.py:79.
 * frame_origin (D doubles) is the common origin all ranks centre on; NULL => the shard mean
 * (only valid when n_local == n_global).                                                */
int cpd_set_target(cpd_ctx* h, const double* target, int64_t n_local, int64_t n_global,
                   const double* frame_origin);

/* math_utils.squared_kernel_sum (math_utils.py:28-29 -> _math.squared_kernel,
 * cc/math_utils_py.cc:14) evaluated in closed form, FP64, on the device, over the handle's
 * source and (all ranks') target.  Multi-rank handles all-reduce the target sums.       */
int cpd_sigma2_init(cpd_ctx* h, double* sigma2);

/* Set the state the EM loop starts from: family, RigidCPD(update_scale=...) (cpd.py:136),
 * the outlier weight w of registration() (cpd.py:106), tf_init_params (cpd.py:149-152:
 * lin = rot or b, t, scale) and sigma2 / q of _initialize (cpd.py:145-153).             */
int cpd_set_state(cpd_ctx* h, int tf_kind, int update_scale, double w, const cpd_params* init);

/* One EM iteration == the loop body cpd.py:111-113: transform(source) -> expectation_step
 * -> maximization_step, entirely on the device; `out` receives the new MstepResult.
 * out may be NULL (no host sync).                                                       */
int cpd_em_step(cpd_ctx* h, cpd_params* out);

/* CoherentPointDrift.registration (cpd.py:106-120) without callbacks: at most maxiter
 * iterations, stopping after the first one with |q - q_prev| < tol.  trace (may be NULL)
 * receives 2 doubles (sigma2, q) per iteration run.                                     */
int cpd_em_run(cpd_ctx* h, int maxiter, double tol, cpd_params* out, int* iters_run, double* trace);

/* CoherentPointDrift.expectation_step(t_source, target, sigma2, w) (cpd.py:71-88) against the
 * handle's target shard.  t_source is m x D (m as given to cpd_set_source).  Any of
 * pt1 (n_local), p1 (m), px (m x D) may be NULL.  In a multi-rank handle p1/px/n_p are
 * all-reduced so every rank receives the global sums; pt1 stays per-shard.              */
int cpd_estep(cpd_ctx* h, const double* t_source, double sigma2, double w,
              double* pt1, double* p1, double* px, double* n_p);

/* RigidCPD._maximization_step (cpd.py:160-192) / AffineCPD._maximization_step (:219-244)
 * from a caller-supplied EstepResult (host arrays as returned by cpd_estep) against the
 * handle's source and target.                                                           */
int cpd_mstep(cpd_ctx* h, int tf_kind, int update_scale, const double* pt1, const double* p1,
              const double* px, double n_p, cpd_params* out);

/* BayesianCoherentPointDrift.expectation_step(t_source, target, scale, alpha, sigma_mat, sigma2, w) (probreg/bcpd.py:53-72)
 * against the handle's target shard: the same two passes with a per-source weight alpha_m exp(-scale^2 sigma_mm D / 2 sigma2)
 * (1 - w) and the constant w / N.  alpha: m; sigma_diag: the m diagonal entries of sigma_mat (the only ones bcpd.py:61 reads).
 * Out (any may be NULL): nu_d (n_local), nu (m), px (m x D), n_p; x_hat of the reference's EstepResult is px / nu.        */
int cpd_bcpd_estep(cpd_ctx* h, const double* t_source, double scale, const double* alpha, const double* sigma_diag, double sigma2,
                   double w, double* nu_d, double* nu, double* px, double* n_p);

/* Copies of the last E-step's reductions (device -> host), valid after cpd_em_step/run. */
int cpd_last_estep(cpd_ctx* h, double* pt1, double* p1, double* px, double* n_p);

/* NonRigidCPD with a dense G (cpd.py:247-303, transformation.py:81-102), resident on the device.
 * cpd_nonrigid_begin: after cpd_set_source/target; builds G (float32, like _math.rbf_kernel), W = 0
 * (cpd.py:281) and starts from sigma2 (cpd.py:279).  cpd_nonrigid_step: one loop body of cpd.py:111-113 --
 * T = Y + G W, E-step, the M x M solve of cpd.py:296 (cuSOLVER LU), sigma2 of cpd.py:298-301; returns the
 * new sigma2 (== q, cpd.py:303).  cpd_nonrigid_get: W (m x D) and/or the moved source Y + G W.      */
int cpd_nonrigid_begin(cpd_ctx* h, double beta, double lmd, double sigma2, double w);
int cpd_nonrigid_step(cpd_ctx* h, double* sigma2_out);
int cpd_nonrigid_get(cpd_ctx* h, double* w_out, double* moved_out);
/* NonRigidCPD._maximization_step (cpd.py:284-303; with priors set: ConstrainedNonRigidCPD's, cpd.py:376-404) from a caller-supplied
 * EstepResult (host arrays as cpd_estep returns them) and the sigma2 that E-step used; after a *_begin on this handle.  The
 * new W / moved source are read with cpd_nonrigid_get; *sigma2_out == q (cpd.py:303).                                            */
int cpd_nonrigid_mstep(cpd_ctx* h, const double* pt1, const double* p1, const double* px, double sigma2_p, double* sigma2_out);

/* NonRigidCPD with G replaced by a rank-K factorisation G ~= Q Bc Q^T (csrc/lowrank.cuh; BASELINE configuration 5, no
 * reference counterpart: the reference only has the dense solve of cpd.py:296).  Same life cycle as the dense path:
 * cpd_nonrigid_lowrank_begin instead of cpd_nonrigid_begin, then cpd_nonrigid_step / cpd_nonrigid_get.  Q comes from a
 * randomised range finder (seeded, `power_iters` subspace iterations, 2 is plenty) on products G X formed on the fly, so
 * nothing of size M x M is stored; each M-step is a K x K solve: symmetric positive definite on the factor Q L, Bc ~= L L^T, in one
 * CTA for rank <= 228, else (or with CPD_B200_LR_CORE=lu) the LU of the unsymmetric form.  rank is clamped to M; rank <= 1024.
 * cpd_nonrigid_lowrank_get: the rank in use, Q (m x rank row-major, caller's point order) and Bc (rank x rank, symmetric; L L^T in
 * the default form: positive semi-definite, exactly the core the iteration uses); any may be NULL. */
int cpd_nonrigid_lowrank_begin(cpd_ctx* h, double beta, double lmd, double sigma2, double w, int rank, int power_iters, uint64_t seed);
int cpd_nonrigid_lowrank_get(cpd_ctx* h, int* rank_out, double* q_out, double* bcore_out);

/* Another registration with the same source (one template, many targets): resets W = 0 (cpd.py:281), the moved source, sigma2, w,
 * lmd and the priors, and keeps G / the low-rank factors of the last cpd_nonrigid_*begin.  The caller vouches that the source
 * coordinates on the handle are the ones that begin saw.                                                                      */
int cpd_nonrigid_restart(cpd_ctx* h, double lmd, double sigma2, double w);

/* Correspondence priors of ConstrainedNonRigidCPD (cpd.py:364-374: p1_tilde = row sums of the indicator matrix, px_tilde =
 * its product with the target; cpd.py:390-396: both enter the system and the right-hand side scaled by sigma2 / alpha).
 * Call after cpd_nonrigid_begin / cpd_nonrigid_lowrank_begin; p1_tilde: m, px_tilde: m x D; both NULL switches priors off. */
int cpd_nonrigid_set_prior(cpd_ctx* h, double alpha, const double* p1_tilde, const double* px_tilde);

/* _math.rbf_kernel (cc/math_utils_py.cc:15 -> cc/math_utils.cc:17-19):
 * out[i*ny + j] = exp(-|x_i - y_j|^2 / (2*beta)) as float32, x: nx x D, y: ny x D.       */
int cpd_rbf_kernel(int device, const double* x, int64_t nx, const double* y, int64_t ny, int dim,
                   double beta, float* out);

/* _math.inverse_multiquadric_kernel (cc/math_utils_py.cc -> cc/math_utils.cc:37-39): out[i*ny + j] = (|x_i - y_j|^2 + c)^(-1/2),
 * float32 (used by CombinedBCPD._initialize, bcpd.py:113).                                                                   */
int cpd_imq_kernel(int device, const double* x, int64_t nx, const double* y, int64_t ny, int dim, double c, float* out);

/* gauss_transform._gauss_transform_direct / GaussTransform.compute (gauss_transform.py:10-16, 47-60), evaluated
 * exactly (no IFGT): out[c*n + i] = sum_j weights[c*m + j] * exp(-|target_i - source_j|^2 / h^2).        */
int cpd_gauss_transform(int device, const double* source, int64_t m, const double* target, int64_t n, int dim, double h,
                        const double* weights, int k, double* out);

/* math_utils.squared_kernel_sum on two host clouds without a handle.                    */
int cpd_squared_kernel_sum(int device, const double* x, int64_t nx, const double* y, int64_t ny,
                           int dim, double* out);

/* -- multi-GPU: one process per GPU, targets sharded, sources replicated -------------------
 * cpd_comm_unique_id fills 128 bytes (an ncclUniqueId) on one rank; after it has been
 * distributed (any side channel), every rank calls cpd_comm_create ONCE -- a collective -- and
 * attaches the communicator to as many handles as it likes.  From then on cpd_em_step /
 * cpd_estep / cpd_sigma2_init issue one ncclAllReduce(sum, double) on the handle's stream.
 * The communicator outlives the handles; destroy it explicitly (or let the process exit).   */
int cpd_comm_unique_id(char id[128]);
int cpd_comm_create(void** comm, int device, int world_size, int rank, const char id[128]);
int cpd_comm_destroy(void* comm);
int cpd_comm_attach(cpd_ctx* h, void* comm, int world_size, int rank);
/* Fused exchange for the EM loop (single node): each rank exports a 64-byte cudaIpcMemHandle of its
 * mailbox (cpd_p2p_local_handle), the handles of all ranks are concatenated in rank order and given to
 * cpd_p2p_attach.  cpd_em_step then reduces the moments, exchanges them through NVLink peer memory and runs
 * the M-step in ONE kernel; the NCCL communicator is still used for the M-sized sums of cpd_estep and for
 * cpd_sigma2_init.  Every rank must have attached before any rank calls cpd_em_step.              */
int cpd_p2p_local_handle(cpd_ctx* h, char out[64]);
int cpd_p2p_attach(cpd_ctx* h, const char* handles, int world_size, int rank);
int cpd_p2p_detach(cpd_ctx* h);      /* back to ncclAllReduce for the moments (e.g. when a peer could not map the mailboxes) */

/* Host-only: the work list {tile, first unit, end unit, partial slot} a pass over ntiles i-tiles x nunits sub-chunks of j-records is
 * launched with on `slots` resident CTAs (csrc/cpd_b200.cu: build_work); last_tile_cost in (0, 1]: the share of the last tile's
 * warps that hold i-points.  items may be NULL to query the counts.                                                     */
int cpd_plan_work(int ntiles, int nunits, int slots, double last_tile_cost, int* items, int capacity, int* n_items, int* max_slots);

/* -- measurement helpers (bench.py): CUDA events on the handle's stream ---------------- */
int cpd_timer_start(cpd_ctx* h);
int cpd_timer_stop(cpd_ctx* h, float* ms);           /* synchronises */
int cpd_sync(cpd_ctx* h);
/* a pool of CUDA events on the handle's stream: record slot `idx` (0 <= idx < 8192) now; elapsed
 * ms between two recorded slots (the caller synchronises first, e.g. cpd_sync).             */
int cpd_event_record(cpd_ctx* h, int idx);
int cpd_event_elapsed(cpd_ctx* h, int idx_start, int idx_stop, float* ms);
/* duration of the last run of each kernel stage, ms (events recorded when profiling is on):
 * [0] pack [1] pass1 [2] finalize1 [3] pass2 [4] finalize2 [5] moments+mstep (+allreduce)  */
int cpd_set_profiling(cpd_ctx* h, int on);
int cpd_stage_times(cpd_ctx* h, float ms[6]);
/* the last cpd_nonrigid_lowrank_begin run with profiling on: ms of [0] the G X products [1] the orthonormalisations [2] Bc       */
int cpd_lowrank_setup_times(cpd_ctx* h, float ms[3]);
/* launches issued by this handle since creation (kernels only).                         */
int64_t cpd_launch_count(cpd_ctx* h);
/* overwrite `bytes` of scratch to evict L2 (bench hygiene); 0 => default 256 MiB.        */
int cpd_flush_l2(cpd_ctx* h, int64_t bytes);
/* Issue-rate micro-benchmarks for the roofline denominators: out[0] = FFMA TFLOP/s, out[1] =
 * MUFU.EX2 Gop/s, out[2] = SM clock MHz seen by the probe, out[3] = SM count, out[4] = packed
 * FFMA2 TFLOP/s, out[5..7] = Gpairs/s of synthetic (11 FP32 + 1 MUFU), packed (6 FFMA2-class + 2
 * MUFU per 2 pairs) and (7 FP32 + 1 MUFU) instruction mixes, out[8] = TFLOP/s of FFMA2 and scalar
 * FFMA interleaved 1:1.                                                                     */
int cpd_microbench(int device, double out[9]);

#ifdef __cplusplus
}
#endif
#endif /* CPD_B200_H */
