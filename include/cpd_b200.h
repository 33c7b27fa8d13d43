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
 * lin = rot or b, t, scale) and sigma2 / q of _initialize (cpd.py:145-153).
 * The EM loop and the non-rigid loop share the device state: this call (and cpd_mstep)
 * ends a non-rigid loop on the handle, and cpd_nonrigid_*begin / cpd_nonrigid_restart end
 * this loop.  A later call on the ended loop fails with CPD_ERR_STATE, naming the call.  */
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

/* CombinedBCPD.registration (probreg/bcpd.py:82-156) resident on the device, after cpd_set_source / cpd_set_target.
 * gmat_inv: the caller's m x m float32 inverse of the IMQ kernel matrix (row-major, caller's point order; bcpd.py:113-114).  It is
 * uploaded once and kept in float32; the handle holds it, the FP64 precision matrix A and the posterior covariance Sigma: about
 * 20 m^2 bytes (8 GB at m = 20k).  lmd, k > 0, sigma2 > 0, 0 <= w < 1.
 * Starts from the reference's _initialize: identity similarity, v = 0, alpha = 1/m, diag(sigma_mat) = 1, the given sigma2.
 * Refused (CPD_ERR_STATE) on a handle with a communicator attached: the loop runs on one GPU.                               */
int cpd_bcpd_begin(cpd_ctx* h, const float* gmat_inv, double lmd, double k, double sigma2, double w);
/* One loop body: E-step on T(y) = s R (y + v) + t, then the M-step of bcpd.py:125-156 (Sigma = A^-1 by cuSOLVER's LU and a solve
 * against the identity; v = ratio Sigma r without a division by nu, so a source no target explains keeps v finite).
 * *sigma2_out: the new sigma2.  The target may be set again between two steps (any count); the loop goes on from its state.
 * Fails with CPD_ERR_STATE before cpd_bcpd_begin, after the source was set again, when getrf finds U exactly singular or getrs
 * fails, or when the new sigma2 is not a positive finite number; after such a failure every step fails until the next
 * cpd_bcpd_begin.                                                                                                               */
int cpd_bcpd_step(cpd_ctx* h, double* sigma2_out);
/* The current state, caller's order; any pointer may be NULL.  sim: lin = rot, t, scale, sigma2 (n_p: of the last E-step).
 * v_out, moved_out (s R (y + v) + t): m x D;  alpha_out, sigma_diag_out: m.                                                    */
int cpd_bcpd_get(cpd_ctx* h, cpd_params* sim, double* v_out, double* moved_out, double* alpha_out, double* sigma_diag_out);
/* The same loop with the kernel matrix replaced by a rank-K factorisation G ~= Q Bc Q^T of the inverse multiquadric
 * G_ij = (|y_i - y_j|^2 + c)^(-1/2) (CombinedBCPD uses c = 1): no G^-1, nothing of size M x M on the device or the host, and a
 * K x K M-step (csrc/bcpd.cuh).  Sound where G is numerically of low rank -- source clouds of extent up to a few sqrt(c); the dense
 * loop above stays for the others.  The factors come from the low-rank set-up of cpd_nonrigid_lowrank_begin (randomised range
 * finder, `power_iters` subspace iterations, seeded) with the IMQ kernel; set-up times go to cpd_lowrank_setup_times.
 * Same preconditions and starting state as cpd_bcpd_begin; c > 0, rank 1..1024 (clamped to m), power_iters 0..8.
 * cpd_bcpd_step / cpd_bcpd_get then run and read the low-rank loop, with the same failure rules (a singular K x K factor, a failed
 * solve or a sigma2 that is not a positive finite number stop it until the next begin).  The handle's low-rank factors are
 * shared with non-rigid CPD: this call ends a non-rigid loop on the handle, a later cpd_nonrigid_*begin ends this loop (its next
 * step fails and says why), and cpd_bcpd_begin returns the handle to the dense loop.
 * cpd_bcpd_lowrank_get: the rank in use, Q (m x rank, row-major, caller's order) and Bc = L L^T (rank x rank); any may be NULL.  */
int cpd_bcpd_lowrank_begin(cpd_ctx* h, double c, double lmd, double k, double sigma2, double w, int rank, int power_iters, uint64_t seed);
int cpd_bcpd_lowrank_get(cpd_ctx* h, int* rank_out, double* q_out, double* bcore_out);

/* GMMTree (probreg/gmmtree.py, probreg/cc/gmmtree.cc; csrc/gmmtree.cuh), 3-D only, one GPU (a handle with a communicator attached
 * is refused with CPD_ERR_STATE).  A tree of tree_level = L (1..5) levels has n_total = 8 (8^L - 1) / 7 nodes (pi, mu, Sigma);
 * level l holds the 8^(l+1) nodes from 8 (8^l - 1) / 7, and the children of node j start at 8 (j + 1).
 * cpd_gmmtree_build: buildGmmTree on the handle's source, in FP64 (pdfs, log-likelihood, moments), every reduction in a fixed
 * order (bit-identical runs on one device).  Where it departs from the reference: the 8^L leaves are seeded from leaf_seeds
 * (8^L point indices into the source, caller's order) instead of Eigen's random draw, which reads out of bounds for L >= 2; and
 * each level stops after maxiter (>= 1) EM iterations if |q - q_prev| < lambda_s has not stopped it before.  iters_per_level (L
 * ints, may be NULL): the iterations each level ran.  lambda_d: the m0 below which a node dies (the reference passes 1e-4).
 * The tree does not depend on the source once built: cpd_set_source keeps it.
 * cpd_gmmtree_nodes: the current tree, pi (n_total), mu (n_total x 3), cov (n_total x 3 x 3), in the caller's coordinates; any
 * may be NULL.  cpd_gmmtree_load installs a caller's tree of the same layout instead (all finite) -- to test the E-step alone.
 * cpd_gmmtree_assign: per source point (caller's order, m int32) the node it was assigned to in the last E-step of the build's
 * last level (the leaf level); refused after a load or once the source count has changed.
 * cpd_gmmtree_estep: gmmTreeRegEstep on the handle's target moved by z = rot x + t (rot row-major 3 x 3): each point descends
 * from the root to the argmax child until a node of complexity (smallest eigenvalue / trace of Sigma) <= lambda_c, and adds
 * (gamma, gamma z, gamma z z^T) to that node only.  moments: n_total x 13 (m0, m1[3], m2[3][3] row-major).
 * cpd_gmmtree_times: with profiling on (cpd_set_profiling), ms of each level of the last build (level_ms[l], l < L; 0 beyond)
 * and of the last cpd_gmmtree_estep; either pointer may be NULL.
 * Refused with CPD_ERR_ARG: a 2-D handle, tree_level outside 1..5, a seed outside 0..m-1, a non-finite parameter, source or
 * target; with CPD_ERR_STATE: no source (build), no tree or no target (E-step).                                                */
int cpd_gmmtree_build(cpd_ctx* h, int tree_level, double lambda_s, double lambda_d, const int64_t* leaf_seeds, int maxiter,
                      int* iters_per_level);
int cpd_gmmtree_nodes(cpd_ctx* h, double* pi, double* mu, double* cov);
int cpd_gmmtree_load(cpd_ctx* h, int tree_level, const double* pi, const double* mu, const double* cov);
int cpd_gmmtree_assign(cpd_ctx* h, int32_t* node);
int cpd_gmmtree_estep(cpd_ctx* h, const double rot[9], const double t[3], double lambda_c, double* moments);
int cpd_gmmtree_times(cpd_ctx* h, float level_ms[5], float* estep_ms);

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
/* Test / diagnostic entry (like cpd_plan_work): out = G x for the G of the last low-rank set-up on this handle: the Gaussian of
 * cpd_nonrigid_lowrank_begin's beta or the inverse multiquadric of cpd_bcpd_lowrank_begin's c, on its source points (the source
 * must not have changed since).  x and out are m x cols (1 <= cols <= 1024), row-major, in the
 * caller's point order.  kernel 0: the exact integer-digit product on the tensor cores (csrc/gram_i8.cuh), 1: the CUDA-core kernel
 * (csrc/lowrank.cuh); the call goes straight to it, without the first-use self-check.  world = 1, rank = 0: every row; otherwise
 * only the rows that rank `rank` of a `world`-rank handle forms are filled and the others are zero (there is no exchange).  The
 * factors and the iteration state are left as they were.  The CPU emulation of the test-suite has no tensor-core product: kernel 0
 * fails there with CPD_ERR_STATE. */
int cpd_lowrank_gram_product(cpd_ctx* h, const double* x, int cols, int kernel, int world, int rank, double* out);

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

/* GMMReg (probreg/l2dist_regs.py, cost_functions.py, features.py; csrc/l2dist.cuh), FP64, every reduction in a fixed order
 * (bit-identical runs on one device).
 * cpd_gmm_fit: features.GMM's sklearn GaussianMixture(k, covariance_type="spherical", init_params="random_from_data",
 * reg_covar, tol, max_iter, n_init=1).fit on the handle's source (2-D or 3-D).  seeds: k distinct point indices (caller's order)
 * where the one-hot initial responsibilities sit; the initial weights are nk / N, unnormalised, as sklearn leaves them.  Each
 * iteration: E-step (per-point log-sum-exp, lower bound = its mean), M-step (weights nk / sum nk), then the stop test
 * |lb - lb_prev| < tol.  The pair arithmetic runs in the handle's centred frame; the M-step forms sklearn's parameters in the
 * caller's frame in residual form (no avg_X2 - 2 avg_X mu + mu^2 cancellation).  Outputs (any may be NULL): weights (k), means
 * (k x D, caller's frame), variances (k), n_iter, lower_bounds (max_iter doubles, the first n_iter written).  Refused with
 * CPD_ERR_ARG: k outside 1..m, a seed outside 0..m-1 or repeated, reg_covar < 0 or non-finite, NaN tol, max_iter < 1, a
 * non-finite source; with CPD_ERR_STATE: no source.
 * cpd_l2_dist: compute_l2_dist (cost_functions.py:33-41) without a handle, by direct FP64 pair sums (the reference's Gauss
 * transform is a float32 IFGT): with z = (2 pi sigma^2)^(D/2) and e_ij = exp(-|mu_s,i - mu_t,j|^2 / (2 sigma^2)),
 * f = -sum_i phi_s,i sum_j (phi_t,j / z) e_ij and g_i = phi_s,i sum_j (phi_t,j / z) e_ij (mu_s,i - mu_t,j) / (2 sigma^2)
 * (g: ns x D).  Refused: dim not 2 or 3, an empty mixture, sigma <= 0 or non-finite, a non-finite mean or weight.
 * cpd_tps_kernel: _math.tps_kernel_2d / _3d (cc/math_utils.cc:21-30), float32 like the reference: 2-D r^2 log r (0 where
 * r^2 <= 1e-9; the log of the float32 r is taken in FP64 and rounded once), 3-D -r.  out: nx x ny.                          */
int cpd_gmm_fit(cpd_ctx* h, int k, const int64_t* seeds, double reg_covar, double tol, int max_iter, double* weights, double* means,
                double* variances, int* n_iter, double* lower_bounds);
int cpd_l2_dist(int device, const double* mu_s, int64_t ns, const double* phi_s, const double* mu_t, int64_t nt, const double* phi_t,
                int dim, double sigma, double* f, double* g);
int cpd_tps_kernel(int device, const double* x, int64_t nx, const double* y, int64_t ny, int dim, float* out);

/* SVR (probreg/l2dist_regs.py RigidSVR / TPSSVR, features.py OneClassSVM; csrc/ocsvm.cuh), without a handle.
 * cpd_ocsvm_fit: sklearn's OneClassSVM(kernel="rbf", nu, gamma, tol).fit on x (n x dim, row-major), the one-class dual
 * min 1/2 a^T Q a subject to 0 <= a_i <= 1, sum a = nu n, Q_ij = exp(-gamma |x_i - x_j|^2), by libsvm's SMO with second-order
 * working-set selection and no shrinking (where measured, sklearn's shrinking gives the same a).  sklearn's path is kept: its
 * sample-weighted start, the kernel on the raw coordinates in the caller's order rounded to float32 (libsvm's Qfloat), ties
 * to the larger index, its clipped two-variable step.  FP64 otherwise, every reduction in a fixed order (bit-identical runs on
 * one device).  Outputs: alpha (n, every point; the support is alpha > 0), rho (libsvm's; sklearn's intercept_ = -rho; +inf
 * when every alpha is 1, which sklearn refuses), n_iter (updates made; n_iter = max_iter means the cap was reached and alpha
 * is the current iterate; libsvm's cap is max(10^7, 100 n)).  Refused with CPD_ERR_ARG: dim not 2 or 3, n < 1, nu outside
 * (0, 1], gamma <= 0 or non-finite, tol <= 0 or NaN, max_iter < 1, a non-finite coordinate.                                 */
int cpd_ocsvm_fit(int device, const double* x, int64_t n, int dim, double nu, double gamma, double tol, int64_t max_iter, double* alpha,
                  double* rho, int64_t* n_iter);

/* math_utils.squared_kernel_sum on two host clouds without a handle.                    */
int cpd_squared_kernel_sum(int device, const double* x, int64_t nx, const double* y, int64_t ny,
                           int dim, double* out);

/* FilterReg (probreg/filterreg.py, gaussian_filtering.py; csrc/lattice.cuh), without a handle.  The permutohedral lattice is the
 * reference's x86-64 build (third_party/permutohedral, SSE path) reproduced bit for bit: the same vertex set and lattice size,
 * including the vertices of the zero padding lanes of its 4-point blocks, and the same float32 splat, blur and slice, with
 * compute()'s dispatch (seqCompute for 1-2 value channels, sseCompute for 3 or more).
 * cpd_lattice_filter: Permutohedral(feature, with_blur) over n points (n x d float32, row-major, |feature| < 1e8), then
 *   filter(values) of vs = 1..8 channels (n x vs float32) into out (n x vs).  values == NULL: only *lattice_size.
 * cpd_filterreg_estep: FilterReg.expectation_step (filterreg.py:78-108) on t_source (m x d) and target (n x d): the features
 *   float32(x / sqrt(sigma2)), the blurred lattice, rebuilt without blur when its size exceeds n * alpha (*with_blur tells which),
 *   and m0 (m), m1 (m x d), m2 (m, update_sigma2 only; |y|^2 in FP64 rounded once) and nx (m x d, target_normals != NULL only)
 *   read at the sources.  stage_ms (NULL or 6 floats): ms of [0] elevation [1] sort [2] vertex numbering and blur neighbours
 *   [3] splat [4] blur [5] slice, of the last lattice built.                                                                  */
int cpd_lattice_filter(int device, const float* feature, int64_t n, int d, const float* values, int vs, int with_blur, float* out,
                       int64_t* lattice_size);
int cpd_filterreg_estep(int device, const double* t_source, int64_t m, const double* target, int64_t n, int d,
                        const double* target_normals, double sigma2, int update_sigma2, double alpha, float* m0, float* m1, float* m2,
                        float* nx, int* with_blur, float* stage_ms);
/* The FilterReg loop (filterreg.py:120-147) with the clouds resident on the device.  cpd_filterreg_begin uploads source (m x d),
 * target (n x d) and target_normals (n x d, NULL for pt2pt) once.  cpd_filterreg_step(h, rot (d x d row-major), t, sigma2, w, moments)
 * moves the source in FP64 (x' = ((R00 x + R01 y) + R02 z) + t0, no FMA), runs the E-step of cpd_filterreg_estep on it and
 * reduces the M-step's sums (filterreg.py:163-196) over the sources with m0 != 0 in FP64, fixed order, into 49 doubles:
 *   [0] survivors  [1] S wt  [2..4] S wt x  [5..7] S wt y  [8] S wt^2  [9] S wt |x - y|  [10] S (m0 |x|^2 - 2 x.m1 + m2) / (m0 + c)
 *   [11] S m0 / (m0 + c)  [12..20] S wt^2 (x - mc)(y - tc)^T (3 x 3, mc, tc the wt-weighted centres)
 *   [21..41] S wt J J^T (upper triangle, row by row)  [42..47] S wt r J  [48] S wt^2 r^2   (point to plane, 3-D with normals)
 * with y = m1 / m0, c = w / (1 - w) n / m (2 pi sigma2)^(d/2), wt = sqrt(m0 / (m0 + c) / sigma2), n = nx / m0, r = n.(y - x),
 * J = [x cross n, n]; coordinates past d are 0.  Only these doubles cross per step.  cpd_filterreg_get reads the last E-step's
 * m0, m1, m2, nx (NULL: skipped), the blur decision, the device bytes the handle holds and the last step's stage times.      */
typedef struct cpd_fr cpd_fr;
int cpd_filterreg_begin(cpd_fr** out, int device, const double* source, int64_t m, const double* target, int64_t n, int d,
                        const double* target_normals, int update_sigma2, double alpha);
int cpd_filterreg_step(cpd_fr* h, const double* rot, const double* t, double sigma2, double w, double* moments);
int cpd_filterreg_get(cpd_fr* h, float* m0, float* m1, float* m2, float* nx, int* with_blur, int64_t* device_bytes, float* stage_ms);
void cpd_filterreg_end(cpd_fr* h);

/* Many independent rigid / affine registrations in one call, without a handle (no reference counterpart: the reference registers
 * one pair at a time).  Pair k is source rows [src_off[k], src_off[k+1]) of src and target rows [tgt_off[k], tgt_off[k+1]) of tgt
 * (both row-major, D = dim; src_off[0] = tgt_off[0] = 0; npairs + 1 offsets each).  Per pair exactly what cpd_sigma2_init +
 * cpd_set_state + cpd_em_run(maxiter, tol) compute for it: sigma2_0 in closed form, q_0 = 1 + N D / 2 log sigma2_0 (cpd.py:148),
 * then at most maxiter EM iterations, stopping after the first one with |q - q_prev| < tol.  init (NULL: identity, t = 0,
 * scale = 1) holds npairs starting transformations (lin = rot or b, t, scale; scale is ignored for affine); sigma2 and q of init
 * are not read.  out (npairs): the last MstepResult of each pair (the start state when maxiter = 0); iters (npairs): the
 * iterations each pair ran.  One CTA owns one pair for its whole registration (csrc/batch.cuh): one launch and one read-back for
 * the batch, and a pair's result does not depend on the other pairs, its position or the batch size.
 * Refused with CPD_ERR_ARG before anything runs, naming the pair: an empty cloud, a non-finite coordinate or initial transformation,
 * sigma2_0 = 0 (all points of both clouds identical), m or n > 2^16 or m n > 2^26 (such a pair belongs to the handle's
 * loop); and dim not 2 or 3,
 * w outside [0, 1), maxiter < 0, tf_kind not rigid or affine (CPD_TF_NONRIGID has its own message).                             */
int cpd_batch_register(int device, int dim, int npairs, const double* src, const int64_t* src_off, const double* tgt,
                       const int64_t* tgt_off, int tf_kind, int update_scale, double w, int maxiter, double tol,
                       const cpd_params* init, cpd_params* out, int* iters);

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
/* the last cpd_bcpd_step run with profiling on, ms: [0] E-step [1] building the precision matrix [2] getrf [3] getrs against the
 * identity [4] the rest of the M-step.  In low-rank mode: [0] E-step [1] St and Rt (and the K x K system) [2] getrf (K) [3] getrs (K)
 * [4] the rest (v, diag Sigma, mixing weights, similarity, sigma2)                                                              */
int cpd_bcpd_step_times(cpd_ctx* h, float ms[5]);
/* the last low-rank set-up (cpd_nonrigid_lowrank_begin or cpd_bcpd_lowrank_begin) run with profiling on: ms of [0] the G X
 * products [1] the orthonormalisations [2] Bc and its factor                                                                     */
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
