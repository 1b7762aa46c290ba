/*
 * pinn_b200.h -- C ABI of libpinn_b200.so: the H100-native PINN training core.
 *
 * The reference (pierremtb/PINNs-TF2.0) has no FFI; its de-facto boundary is the Python class surface
 * of utils/neuralnetwork.py, utils/custom_lbfgs.py and the per-PDE subclasses.  Each entry point below
 * replaces the reference code cited next to it (paths relative to the reference repo root) and is what a
 * ctypes/cffi binding on the reference side would bind (see INTEGRATION.md).
 *
 * Conventions
 *   - every function returns 0 on success, <0 on error; the message is in pinn_last_error() (thread-local);
 *     no C++ exception crosses this boundary;
 *   - all floating point is IEEE fp64 (the reference runs float64: utils/neuralnetwork.py:24-26);
 *   - host buffers are borrowed for the duration of the call only; output buffers are caller-owned,
 *     C-contiguous;
 *   - the handle owns all device memory, one CUDA stream and (world > 1) one NCCL communicator; it is not
 *     thread-safe; one process per GPU;
 *   - functions that return a host scalar/array synchronise the handle's stream; the others only enqueue;
 *   - what a handle returns depends only on its CURRENT inputs (points, targets, constants, stage matrices, residual spec,
 *     source, weights, optimiser state), never on the calls that brought it there: after any order of setter, evaluation and
 *     optimiser calls it equals, bit for bit, a fresh handle fed the same inputs, and a refused call changes nothing
 *     (tests/test_gpu_handle_state.py).
 *
 * Flat parameter layout (utils/neuralnetwork.py:68-89 get_weights/set_weights, :97-100 flat gradient):
 *   for each Dense layer in order: W.flatten() (row-major [in,out]) then b;  identification appends
 *   [lambda_1, lambda_2] (1d-burgers/ide_cont_burgers.py:98-107).
 */
#ifndef PINN_B200_H
#define PINN_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pinn_handle pinn_t;

/* PDE ids: which fused residual kernel a handle runs. */
enum {
  PINN_BURGERS_INF = 0, /* 1d-burgers/inf_cont_burgers.py:48-98   f = u_t + u u_x - nu u_xx              */
  PINN_BURGERS_IDE = 1, /* 1d-burgers/ide_cont_burgers.py:47-118  f = u_t + l1 u u_x - exp(l2) u_xx      */
  PINN_NLS_INF = 2,     /* 1dcomplex-schrodinger/inf_cont_schrodinger.py:46-135                          */
  PINN_BURGERS_DISC = 3, /* 1d-burgers/inf_disc_burgers.py:49-127  discrete time, q-stage implicit Runge-Kutta:
                           net [1, ..., q+1] on x only; U_0 = U_1 + dt (U U_x - nu U_xx) IRK^T; SSE losses          */
  PINN_BURGERS_IDE_DISC = 4 /* 1d-burgers/ide_disc_burgers.py:48-203  discrete-time identification: net [1, ..., q], two
                           snapshots; N = l1 U U_x - exp(l2) U_xx; U_0 = U + dt N alpha^T, U_1 = U - dt N (beta-alpha)^T;
                           loss = sum (U_0 - u_0)^2 + sum (U_1 - u_1)^2; flat vector ends with [lambda_1, lambda_2]   */,
  PINN_KDV_IDE_DISC = 5, /* discrete_time_identification (KdV)/KdV.py of PINNs/main (fp64 restatement): as BURGERS_IDE_DISC
                           with u_t + l1 u u_x + exp(l2) u_xxx = 0, i.e. N = l1 U U_x + exp(l2) U_xxx; net [1, ..., q]    */
  PINN_AC_DISC = 6      /* discrete_time_inference (AC)/AC.py of PINNs/main (fp64 restatement): net [1, ..., q+1] on x;
                           N = k U^3 - k U - d U_xx; U_0 = U_1 + dt N IRK^T; loss = sum (U_0 - u_0)^2 + sum over all q+1
                           outputs of (U_1(lb) - U_1(ub))^2 + (d/dx U_1(lb) - d/dx U_1(ub))^2 (periodic in value and slope) */,
  PINN_NS_IDE = 7       /* continuous_time_identification (Navier-Stokes)/NavierStokes.py of PINNs/main (fp64 restatement): net
                           [3, ..., 2] maps (x, y, t) to (psi, p); u = psi_y, v = -psi_x;
                           f_u = u_t + l1 (u u_x + v u_y) + p_x - l2 (u_xx + u_yy), f_v = v_t + l1 (u v_x + v v_y) + p_y - l2 (v_xx + v_yy);
                           loss = sum (u - u_d)^2 + sum (v - v_d)^2 + sum f_u^2 + sum f_v^2 over the data points (parts: data, 0,
                           residual); flat vector ends with the raw [lambda_1, lambda_2]; one GPU only (world == 1)          */,
  PINN_POLY_INF = 8,    /* user-defined residual (pinn_set_residual) on a net [2, ..., 1]:
                           f = sum_k c_k kappa_k u^a_k u_x^b_k u_t^c_k u_xx^d_k - s(x, t); every kappa_k = 1; s is an
                           array (pinn_set_source) or a table the device evaluates (pinn_set_source_terms);
                           loss structure of BURGERS_INF (data term of pinn_set_data + mean f^2 over pinn_set_collocation)  */
  PINN_POLY_IDE = 9     /* as POLY_INF with kappa_k in {1, l1, l2, e^l1, e^l2}; loss structure of BURGERS_IDE (the residual on the
                           data points); flat vector ends with the raw [lambda_1, lambda_2].  Both poly ids run on the generic
                           fused kernel and on one GPU only (world == 1)                                                    */
};

/* L-BFGS stop reasons (utils/custom_lbfgs.py:73-76,154-156,192-215). */
enum {
  PINN_LBFGS_RUNNING = 0,
  PINN_LBFGS_MAX_ITER = 1,
  PINN_LBFGS_MAX_EVAL = 2,
  PINN_LBFGS_OPTIMALITY = 3,
  PINN_LBFGS_STEP_TOL = 4,
  PINN_LBFGS_F_TOL = 5,
  PINN_LBFGS_NO_PROGRESS = 6,
  PINN_LBFGS_INITIAL_OPTIMALITY = 7
};

const char* pinn_last_error(void);
const char* pinn_version(void);

/* NeuralNetwork.__init__ (utils/neuralnetwork.py:8-47): layers = hp["layers"]; lb/ub feed the normalising
 * Lambda (:29-30).  rank/world/nccl_uid: data-parallel sharding of the collocation set (new capability,
 * SURVEY 8(e)); nccl_uid = 128-byte ncclUniqueId from pinn_nccl_unique_id on rank 0, NULL when world==1.  world > 1 is
 * accepted for BURGERS_INF and NLS_INF only (DESIGN.md section 5).
 * lb and ub hold max(2, layers[0]) entries: (x, t), or (x, y, t) for NS_IDE. */
int pinn_create(pinn_t** out, int pde_id, int n_layers, const int* layers, const double* lb, const double* ub,
                int device, int rank, int world, const void* nccl_uid);
int pinn_destroy(pinn_t* h);
int pinn_nccl_unique_id(void* out128);

/* Fused NVLink push exchange (world > 1; replaces reduce -> ncclAllReduce -> Adam by ONE kernel per evaluation): every rank
 * owns a small IPC-exported exchange buffer; the tail kernel of an evaluation reduces the per-CTA partials, STORES the
 * result into every peer's buffer over NVLink (P2P stores, nobody pulls), waits on its local flags, sums the ranks' vectors
 * in a fixed order (bitwise identical on all ranks) and applies Adam in the same pass.  Usage: each rank calls
 * pinn_p2p_export (64-byte cudaIpcMemHandle), the handles are all-gathered by the caller's control plane, then each rank
 * calls pinn_p2p_connect(handles[world][64]).  All ranks must use the same path: if mapping fails anywhere, every rank
 * calls pinn_p2p_enable(h, 0) and the NCCL communicator of pinn_create carries the exchange instead. */
int pinn_p2p_export(pinn_t* h, void* out64);
int pinn_p2p_connect(pinn_t* h, const void* handles, int world);
int pinn_p2p_enable(pinn_t* h, int on);

/* Number of entries of the flat parameter vector (net params [+2 for identification]). */
int64_t pinn_num_params(const pinn_t* h);

/* PDE constants.  BURGERS_INF: p[0] = nu (inf_cont_burgers.py:52,111).  BURGERS_DISC: p = [nu, dt]
 * (inf_disc_burgers.py:53-54).  BURGERS_IDE_DISC and KDV_IDE_DISC: p = [dt] (ide_disc_burgers.py:52).
 * AC_DISC: p = [dt, d, k].  Others take none. */
int pinn_set_pde_params(pinn_t* h, const double* p, int n);
/* get_params(numpy=True): BURGERS_INF -> [nu] (inf_cont_burgers.py:92-93); BURGERS_IDE and BURGERS_IDE_DISC ->
 * [lambda_1, exp(lambda_2)] read from the trained flat vector (ide_cont_burgers.py:109-114, ide_disc_burgers.py:138-143);
 * KDV_IDE_DISC -> [lambda_1, exp(lambda_2)] likewise; BURGERS_DISC -> [nu, dt]; AC_DISC -> [dt, d, k];
 * NS_IDE and POLY_IDE -> the raw [lambda_1, lambda_2]. */
int pinn_get_params(pinn_t* h, double* p, int n);
/* BURGERS_DISC: the implicit Runge-Kutta stage matrix IRK_weights, (q+1) x q row-major (inf_disc_burgers.py:56,86);
 * q+1 must equal the network's output width.
 * BURGERS_IDE_DISC: irk = [M_0 ; M_1], 2q x q row-major, with M_0 = IRK_alpha and M_1 = -(IRK_beta - IRK_alpha) (the caller
 * forms the difference exactly as the reference does -- in the tables' float32, ide_disc_burgers.py:107 -- and folds the sign
 * of N' = -N into it); q must equal the network's output width. */
/* KDV_IDE_DISC takes the BURGERS_IDE_DISC layout, AC_DISC the BURGERS_DISC one. */
int pinn_set_irk(pinn_t* h, const double* irk, int q);

/* Point, target and weight inputs are not checked for finiteness: NaN and +-Inf propagate as in the reference (DESIGN §1,
 * "Non-finite values"). */
/* Collocation points of THIS rank: x_f, t_f (inf_cont_burgers.py:55-56; inf_cont_schrodinger.py:56-57).
 * n_global = N_f over all ranks (the MSE_f denominator); pass n when world == 1. */
int pinn_set_collocation(pinn_t* h, const double* x, const double* t, int64_t n, int64_t n_global);

/* Zero-copy variant for per-step resampling (the e2e path of bench.py): x, t must be PINNED host memory
 * (pinn_host_alloc); nothing is copied -- the fused kernel reads the batch straight over PCIe (prefetched one tile ahead).
 * The buffers must stay valid and unchanged until the next synchronising call.  Burgers inference kernel only. */
int pinn_set_collocation_mapped(pinn_t* h, const double* x_pinned, const double* t_pinned, int64_t n, int64_t n_global);

/* BURGERS_INF, NLS_INF, POLY_INF: replace this rank's collocation set by rows [first, first + n) of Latin-hypercube draw `draw`
 * of `seed` over [lb, ub] of pinn_create, with N = n_global strata per dimension (DESIGN §4.6).  Enqueue only: no host buffer,
 * no synchronisation (except when the collocation region has to grow, as for pinn_set_collocation).  n_global is also the MSE_f
 * denominator, as in pinn_set_collocation; 1 <= n_global <= 2^53 and 0 <= first <= first + n <= n_global.  Replaces a mapped
 * batch.  POLY_INF: an array source resets to zero and a source table is evaluated at the new set, as for every new set of
 * residual points.  The drawn set is a current input of the
 * handle, defined by (seed, draw, first, n, n_global, lb, ub): the handle equals a fresh one fed the same points through
 * pinn_set_collocation.  The row rule: one Philox4x32-10 block of (row, draw) under the seed gives two 53-bit uniforms, two
 * keyed Feistel permutations of [0, n_global) give the strata, and x_d = lb_d + (ub_d - lb_d) * ((stratum + u) / n_global). */
int pinn_draw_collocation(pinn_t* h, uint64_t seed, uint64_t draw, int64_t first, int64_t n, int64_t n_global);
/* BURGERS_INF, NLS_INF, POLY_INF, one GPU: residual-based adaptive resampling (RAD, Wu et al., CMAME 403, 2023; DESIGN §4.7).  Replaces
 * the collocation set by n points drawn, with replacement, from a pool with probability proportional to a quantised
 * eps(x)^k / E[eps^k] + c, where eps is the PDE residual at the handle's current weights.  Enqueue only, like
 * pinn_draw_collocation: no host buffer, no synchronisation (except when the collocation region or the pool scratch has to grow).
 * n is also the MSE_f denominator.  Replaces a mapped batch.  The handle then equals a fresh one fed the same points through
 * pinn_set_collocation.  The draw, step by step (every integer step is exact, so it does not depend on a reduction order):
 *   1. pool: rows [0, n_pool) of Latin-hypercube draw `draw` of `seed` with n_pool strata, i.e. what
 *      pinn_draw_collocation(h, seed, draw, 0, n_pool, n_pool) stores;
 *   2. f_i at pool point i, from the weights after every step already enqueued: bit for bit the value pinn_residual returns;
 *   3. r_i = |f_i| (BURGERS_INF, POLY_INF) or sqrt(f_u^2 + f_v^2) (NLS_INF), each operation rounded; a_i = r_i^k as left-to-right rounded
 *      products (k = 0: a_i = 1);
 *   4. amax = the largest finite a_i (0 if none); A_i = 2^24 if a_i is not finite, else floor((a_i / amax) * 2^24) as a uint64
 *      (0 when amax = 0); S = sum A_i; C' = floor(c * (double)S / n_pool) (one rounded fp64 multiply, one rounded divide);
 *      Q_i = A_i + C', T = sum Q_i, and every Q_i = 1 if T = 0;
 *   5. row j: one Philox4x32-10 block (w0, w1, w2, w3) with counter (lo j, hi j, lo draw, hi draw) and key
 *      (lo seed ^ 0xBF58476D, hi seed ^ 0x1CE4E5B9); target = mulhi64(w0 << 32 | w1, T), in [0, T); row j is pool point i for
 *      the least i whose inclusive prefix Q_0 + ... + Q_i exceeds target.
 * Points with Q_i = 0 are never drawn; a non-finite residual takes the largest weight.  Up to the 2^-24 quantisation Q_i / T is
 * RAD's (a_i / mean a + c) / (n_pool (1 + c)).  Unlike Wu et al. the draw is with replacement: a point may appear more than once.
 * POLY_INF: f is the residual spec's sum in pinn_residual's order, each product and sum rounded, minus the source table's s at
 * the pool point; the table is then evaluated at the drawn set.  Refused (the handle is left unchanged) for the identification,
 * discrete-time and Navier-Stokes models, for POLY_INF without a residual spec or with an array source (pinn_set_source: values
 * at the stored points say nothing about a pool), for world > 1, and unless 0 <= k <= 4, c is finite in [0, 1024],
 * 1 <= n_pool <= 2^29 and n >= 0. */
int pinn_draw_collocation_rad(pinn_t* h, uint64_t seed, uint64_t draw, int64_t n_pool, int64_t n, int k, double c);
/* The stored collocation set, however it got there (upload, mapped batch, draw): x, t hold n doubles each; n must equal
 * pinn_num_residual_points(h).  Synchronises.  (A POLY_INF source that a table cannot express is evaluated on a set read back
 * here and stored with pinn_set_source.) */
int pinn_get_collocation(pinn_t* h, double* x, double* t, int64_t n);

/* Data term: X_u,u of fit(X_u,u) (utils/neuralnetwork.py:138-146).  X is (n,in_dim) row-major; in_dim==1
 * reproduces the Lambda's broadcast of a (N,1) input to (x, t:=x) (quirk Q1, inf_cont_schrodinger.py:164).
 * u is (n,out_dim).  For BURGERS_IDE these are also the residual points (ide_cont_burgers.py:88-91,116-118).
 * weight: 1 on the rank that owns the (replicated) data term, 0 elsewhere.
 * AC_DISC: x_0 (n,1) and u_0 (n,1); the periodic pair is (lb[0], ub[0]) of pinn_create, so it needs no pinn_set_boundary.
 * NS_IDE: X (n,3) = (x, y, t) and u (n,2) = (u, v); these are also the residual points (no collocation, boundary, stage matrix
 * or snapshot calls, and no PDE constants). */
int pinn_set_data(pinn_t* h, const double* X, int64_t n, int in_dim, const double* u, int out_dim, double weight);

/* BURGERS_IDE_DISC and KDV_IDE_DISC: snapshot `which` (0: (x_0,u_0) at t_0, 1: (x_1,u_1) at t_1 = t_0 + dt) of fit(x_0,u_0,x_1,u_1)
 * (ide_disc_burgers.py:149-156); x and u are (n,1), u broadcasts over the q stages.  pinn_set_data == snapshot 0. */
int pinn_set_snapshot(pinn_t* h, int which, const double* x, int64_t n, const double* u);

/* POLY_INF / POLY_IDE: the residual f = sum_k coef[k] kappa_k u^e0 u_x^e1 u_t^e2 u_xx^e3 - s.  n_terms in 1..16; exps is
 * n_terms x 4 row-major in the order (u, u_x, u_t, u_xx), each 0..3, no all-zero row; kind[k] in 0..4 selects kappa_k =
 * 1, lambda_1, lambda_2, exp(lambda_1), exp(lambda_2) (raw trainable lambdas; POLY_INF takes kind 0 only); coef finite.  The
 * spec may be replaced at any time; evaluating a poly handle before it is set is an error. */
int pinn_set_residual(pinn_t* h, int n_terms, const double* coef, const int* kind, const int* exps);
/* POLY_INF / POLY_IDE: the source s at the stored residual points, n == pinn_num_residual_points(h).  Storing new residual
 * points (pinn_set_collocation, pinn_draw_collocation and pinn_draw_collocation_rad for POLY_INF, pinn_set_data for POLY_IDE)
 * resets the source to zero, so a source never outlives the points it was computed for.  Removes a source table. */
int pinn_set_source(pinn_t* h, const double* s, int64_t n);
/* POLY_INF / POLY_IDE: the source as a function the device evaluates (DESIGN §4.8), a sum of n_terms separable terms
 *   s(x, t) = sum_k a_k x^p_k t^q_k X_k(x) T_k(t) exp(alpha_k x + gamma_k x^2 + beta_k t + delta_k t^2),
 * X_k one of 1, sin(omega_k x + phi_k), cos(omega_k x + phi_k) and T_k one of 1, sin(nu_k t + psi_k), cos(nu_k t + psi_k).
 * form[k] = p_k | q_k << 2 | xkind_k << 4 | tkind_k << 6 with p, q in 0..3 and the kinds 0: 1, 1: sin, 2: cos; par is
 * n_terms x 9 row-major (a, omega, phi, nu, psi, alpha, gamma, beta, delta), every entry finite; 0 <= n_terms <= 16.  A refused
 * call changes nothing.  Evaluation order, every product and sum rounded on its own (no contraction):
 *   m = a; m *= x, p times; m *= t, q times; m *= X(omega * x + phi); m *= T(nu * t + psi);
 *   m *= exp(((alpha * x + gamma * (x * x)) + beta * t) + delta * (t * t)), omitted when alpha, gamma, beta and delta are all 0;
 *   s = ((0 + m_0) + m_1) + ... in term order.
 * exp is CUDA's exp; sin and cos are CUDA's sin and cos for arguments of magnitude below 2^31 (the library's fast path,
 * restated bit for bit) and NaN from 2^31 on.  Non-finite x or t propagate into s.  A table is a function and follows the
 * points: setting it evaluates it at the stored residual points, and every new set of residual points (pinn_set_collocation,
 * pinn_draw_collocation, pinn_draw_collocation_rad for POLY_INF; pinn_set_data for POLY_IDE) is evaluated again, enqueued
 * (only a growing source array synchronises).  Setting a table removes an array source (pinn_set_source) and vice versa;
 * n_terms = 0 removes both.  A handle with a table equals a fresh one fed the same points and pinn_set_source of
 * pinn_get_source. */
int pinn_set_source_terms(pinn_t* h, int n_terms, const int* form, const double* par);
/* POLY_INF / POLY_IDE: the stored source at the residual points, however it was formed (array, table or none: zeros);
 * n == pinn_num_residual_points(h).  Synchronises. */
int pinn_get_source(pinn_t* h, double* s, int64_t n);

/* NLS periodic-boundary times tb (N_b,1): X_lb=(lb0,tb), X_ub=(ub0,tb) (inf_cont_schrodinger.py:50-53).
 * BURGERS_DISC: the boundary positions x_1 on which sum(net(x_1)^2) is imposed (inf_disc_burgers.py:57,99). */
int pinn_set_boundary(pinn_t* h, const double* tb, int64_t n_b);

/* get_weights / set_weights (utils/neuralnetwork.py:68-89; ide_cont_burgers.py:98-107). */
int pinn_set_weights(pinn_t* h, const double* w, int64_t n);
int pinn_get_weights(pinn_t* h, double* w, int64_t n);

/* grad(X,u) / get_loss_and_flat_grad closure (utils/neuralnetwork.py:55-59, 91-103) with the subclass loss
 * (inf_cont_burgers.py:59-62 | ide_cont_burgers.py:88-91 | inf_cont_schrodinger.py:107-129).
 * ONE fused kernel launch (+ partial reduction, + allreduce when world > 1).  w_or_null: weights to load
 * first (the closure's set_weights(w)); grad_out: P doubles or NULL; parts_out: 3 doubles
 * (mse_u|mse_0, mse_b, mse_f) or NULL. */
int pinn_loss_grad(pinn_t* h, const double* w_or_null, double* loss_out, double* grad_out_or_null,
                   double* parts_out_or_null);

/* tf_optimization_step (utils/neuralnetwork.py:112-116) with TF-2.0 Keras Adam semantics
 * (alpha_t = lr sqrt(1-b2^t)/(1-b1^t); m += (g-m)(1-b1); v += (g^2-v)(1-b2); w -= alpha_t m/(sqrt(v)+eps)).
 * loss_out == NULL: fully asynchronous (one launch on a single GPU with the specialised Burgers kernel -- the last CTAs of the
 * fused kernel reduce the partials and apply Adam --, two launches otherwise; no host sync; the loss goes to a device ring, see
 * pinn_last_loss).  The loss is the one evaluated BEFORE the update, as in the reference. */
int pinn_adam_step(pinn_t* h, double lr, double b1, double b2, double eps, double* loss_out_or_null);

/* n consecutive asynchronous Adam steps (the body of tf_optimization's epoch loop, utils/neuralnetwork.py:105-110, without the
 * per-epoch logger call) enqueued by ONE call: for small point sets the per-call cost of a binding (ctypes: several microseconds)
 * is comparable to the step itself.  Losses go to the device ring as for pinn_adam_step(loss_out == NULL). */
int pinn_adam_steps(pinn_t* h, int n, double lr, double b1, double b2, double eps);
int pinn_adam_reset(pinn_t* h);
/* Loss values of the last n asynchronous Adam steps are kept in a device ring; read the most recent one. */
int pinn_last_loss(pinn_t* h, double* loss_out);

/* nt_optimization_steps -> lbfgs() (utils/neuralnetwork.py:131-136, utils/custom_lbfgs.py:39-236):
 * device-resident two-loop recursion, fixed step (no line search exists in the reference), first step
 * min(1,1/|g|_1), history only pushed when y.s > 1e-10, last update not followed by an evaluation so the
 * model keeps the weights of iteration maxIter-1.  log_cb(it, f, ud) is called for every iteration the
 * reference would have logged (custom_lbfgs.py:217-218), in order, in batches of `sync_every` iterations
 * (1 = after each iteration, like the reference).  Returns iteration/evaluation counts and stop reason. */
typedef void (*pinn_log_cb)(int iter, double f, void* user);
int pinn_lbfgs(pinn_t* h, int max_iter, double learning_rate, int n_correction, double tol_fun, double tol_x,
               int sync_every, pinn_log_cb log_cb, void* user, int* n_iter_out, int* n_eval_out, int* reason_out,
               double* x_final_or_null);

/* f_hist of the last pinn_lbfgs run (custom_lbfgs.py:66-67,186-187: the initial f and the f of every evaluation, including
 * the ones that hit a stop test and were therefore not logged).  *n_out = number of evaluations; f_hist_out may be NULL to
 * query the count.  pinn_lbfgs(max_iter = 0) is a run too (lbfgs() returns before it evaluates anything): the history is
 * empty after it, not that of the run before. */
int pinn_lbfgs_history(pinn_t* h, double* f_hist_out, int capacity, int* n_out);

/* lbfgs() for an ARBITRARY opfunc (utils/custom_lbfgs.py:39-236 takes any closure x -> (f, g)): a stand-alone device-resident
 * optimiser object.  The caller evaluates its objective wherever it likes; the iterate, the (s, y) history ring and the
 * two-loop recursion live on the device and run through the same kernel as pinn_lbfgs, with the reference's control flow
 * and quirks.  Protocol:  create(x0) -> f,g = opfunc(x0) -> feed(f, g) -> while status == PINN_LBFGS_RUNNING:
 * f,g = opfunc(x_next); feed(f, g).  feed() returns in x_next the point to evaluate next or, once status != 0, the vector
 * lbfgs() returns; logged_iter >= 1 names the iteration the reference would have logged after this evaluation (with its f),
 * -1 none.  max_eval == 0 selects the reference default 1.25 * max_iter.  The default (literal, single-CTA) kernel takes
 * n <= 32768; with PINN_LBFGS=gram (Gram-matrix formulation) n may be larger, up to 2^30. */
typedef struct pinn_lbfgs_handle pinn_lbfgs_t;
int pinn_lbfgs_create(pinn_lbfgs_t** out, int device, int64_t n, const double* x0, int max_iter, double learning_rate,
                      int n_correction, double tol_fun, double tol_x, double max_eval);
int pinn_lbfgs_feed(pinn_lbfgs_t* s, double f, const double* g, double* x_next, int* status_out, int* n_iter_out, int* n_eval_out,
                    int* logged_iter_out, double* logged_f_out);
int pinn_lbfgs_f_hist(pinn_lbfgs_t* s, double* f_hist_out, int capacity, int* n_out);
int pinn_lbfgs_destroy(pinn_lbfgs_t* s);

/* predict (utils/neuralnetwork.py:151-153): forward only on (n,in_dim) points -> (n,out_dim); NS_IDE: (psi, p). */
int pinn_predict(pinn_t* h, const double* X, int64_t n, int in_dim, double* out);
/* f_model on the stored residual points (inf_cont_burgers.py:65-90,95-98): the collocation set, or the data points for
 * identification (ide_cont_burgers.py:88-91).  f_out: n_rows * n_res doubles (n_res = 1 Burgers, 2 NLS: f_u then f_v per
 * point; NS_IDE: f_u then f_v per data point); n_rows must equal pinn_num_residual_points(h) -- a mismatch is an error, never
 * a short or long write. */
int64_t pinn_num_residual_points(const pinn_t* h);
int pinn_residual(pinn_t* h, double* f_out, int64_t n_rows);
/* u, u_x, u_t, u_xx at arbitrary points (parity probes): out is (n, 4*out_dim), [u.., u_x.., u_t.., u_xx..].
 * NS_IDE: X is (n,3) and out is (n, 13*2): the 13 streams value, x, y, t, xx, xy, yy, xt, yt, xxx, xxy, xyy, yyy in that order,
 * each block (psi, p). */
int pinn_derivatives(pinn_t* h, const double* X, int64_t n, double* out);

int pinn_sync(pinn_t* h);

/* Pinned host memory for callers that want true async H2D (bench e2e leg). */
int pinn_host_alloc(void** out, int64_t bytes);
int pinn_host_free(void* p);

/* Measurement hooks (bench.py): device-side CUDA-event timing of `iters` back-to-back launches of the fused
 * loss/grad kernel alone, on the handle's stream; and the number of kernels this library has launched. */
int pinn_time_loss_grad_kernel(pinn_t* h, int iters, float* ms_total_out);
int64_t pinn_launch_count(const pinn_t* h);
/* CUDA events on the handle's stream (bench.py times steps on the device, not by wall clock), and an L2
 * flush (a 256 MB memset on the same stream) to put between timed iterations. */
int pinn_event_record(pinn_t* h, int idx);
int pinn_event_elapsed_ms(pinn_t* h, int i, int j, float* ms_out);
int pinn_flush_l2(pinn_t* h);
/* Test hook: the kernels' branch-free fp64 tanh evaluated on the device (tests compare it with libm). */
int pinn_test_tanh(const double* x, int n, double* y);
/* Kernel configuration string (grid, block, dynamic smem, registers) for DESIGN/bench reporting. */
int pinn_kernel_info(pinn_t* h, char* buf, int buflen);

#ifdef __cplusplus
}
#endif
#endif /* PINN_B200_H */
