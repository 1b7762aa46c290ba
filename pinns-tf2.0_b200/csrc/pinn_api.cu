// libpinn_b200.so -- C ABI (include/pinn_b200.h) over the fused sm_90a PINN kernels.
#include "../../include/pinn_b200.h"

#include <cuda_runtime.h>
#include <dlfcn.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <string>
#include <mutex>
#include <vector>

#include "burgers_fused.cuh"
#include "burgers_fused_v2.cuh"
#include "nls_fused.cuh"
#include "optim_kernels.cuh"
#include "generic_fused.cuh"
#include "navier_stokes_fused.cuh"
#include "lhs_draw.cuh"
#include "rad_sample.cuh"
#include "source_terms.cuh"

namespace {

thread_local std::string g_err;
int fail(const std::string& m) { g_err = m; return -1; }

// Live handles of this process.  A launch with the in-kernel tail (fused_tail) keeps its last CTAs spinning on their SMs until the
// launch's stragglers arrive; two such launches running CONCURRENTLY on one device (two handles, two streams) could fill every SM
// with spinning CTAs while both still have CTAs waiting for an SM.  So a handle uses the in-kernel tail only while no OTHER handle on
// the same device has such a launch in flight (checked with cudaStreamQuery); otherwise it falls back to the tail kernel.
std::mutex g_live_mu;
std::vector<struct pinn_handle*> g_live;

#define CUDA_TRY(expr)                                                                                         \
  do {                                                                                                         \
    cudaError_t _e = (expr);                                                                                   \
    if (_e != cudaSuccess)                                                                                     \
      return fail(std::string(#expr) + ": " + cudaGetErrorString(_e) + " (" __FILE__ ":" + std::to_string(__LINE__) + ")"); \
  } while (0)

// ---- NCCL, resolved at run time (torch's bundled libnccl.so.2 is already in the process under torchrun;
// otherwise the system one is opened).  Only the five entry points the path needs.
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(ncclUniqueId*) = nullptr;
  int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  bool load(std::string& why) {
    if (lib) return true;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
      lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (lib) break;
    }
    if (!lib) { why = std::string("dlopen(libnccl.so.2) failed: ") + dlerror(); return false; }
    GetUniqueId = (decltype(GetUniqueId))dlsym(lib, "ncclGetUniqueId");
    CommInitRank = (decltype(CommInitRank))dlsym(lib, "ncclCommInitRank");
    AllReduce = (decltype(AllReduce))dlsym(lib, "ncclAllReduce");
    CommDestroy = (decltype(CommDestroy))dlsym(lib, "ncclCommDestroy");
    GetErrorString = (decltype(GetErrorString))dlsym(lib, "ncclGetErrorString");
    if (!GetUniqueId || !CommInitRank || !AllReduce || !CommDestroy) { why = "NCCL symbols missing"; return false; }
    return true;
  }
};
NcclApi g_nccl;
constexpr int NCCL_FLOAT64 = 8;   // ncclDouble
constexpr int NCCL_SUM = 0;       // ncclSum

constexpr int LOSS_RING = 4096;

// One L-BFGS iteration on the device (stop tests of the pending evaluation, history update, direction, step).
// Default: the single-CTA kernel that follows the reference's loop literally (lbfgs_iterate).
// PINN_LBFGS=gram selects the Gram-matrix formulation (lbfgs_dots -> lbfgs_solve -> lbfgs_apply: every SM reads its slice of
// the history, so it takes less time per iteration, and it has no 32768-entry limit).  It is not the default: the literal
// kernel is the reference's loop term by term.  Long fixed-step runs diverge from some starting points in BOTH modes
// (profiles/lbfgs_stability_h100.jsonl); the step-by-step replay in tests/test_gpu_optimizer_replay.py keeps both kernels
// within their fp64 error bound up to the divergence (DESIGN.md section 4.3).
bool lbfgs_serial() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("PINN_LBFGS"); v = (e && !strcmp(e, "gram")) ? 0 : 1; }
  return v == 1;
}

// The arguments of one L-BFGS run after the reference's defaults (utils/custom_lbfgs.py:49-55).
struct LbfgsConfig {
  int max_iter, n_corr;
  double lr, tol_fun, tol_x, max_eval;
};

// Applies those defaults to the caller's arguments (0 = default) and refuses what the device kernels cannot run: more than
// 128 history pairs, more than 32768 entries in the single-CTA kernel.  `who` names the entry point in the messages.
int lbfgs_config(const char* who, int64_t n, int max_iter, double lr, int n_corr, double tol_fun, double tol_x, double max_eval,
                 LbfgsConfig* c) {
  const std::string w(who);
  if (lbfgs_serial() && n > 32 * 1024) return fail(w + ": vector too large for the single-CTA L-BFGS kernel (32768 entries)");
  if (n > (1 << 30)) return fail(w + ": vector too large");
  if (n_corr <= 0) n_corr = 100;                                             // :52 (`or 100`)
  if (n_corr > 128) return fail(w + ": n_correction > 128 not supported");
  *c = LbfgsConfig{max_iter, n_corr, lr == 0.0 ? 1.0 : lr,                   // :55
                   tol_fun == 0.0 ? 1e-5 : tol_fun,                          // :50
                   tol_x == 0.0 ? 1e-19 : tol_x,                             // :51
                   max_eval == 0.0 ? max_iter * 1.25 : max_eval};            // :49
  return 0;
}

// Iterations whose stop tests have run: all < n_iter, plus n_iter itself unless its evaluation is pending.
int lbfgs_tested(const pinn::LbfgsState& s) { return s.pending ? s.n_iter - 1 : s.n_iter; }

// The device state of L-BFGS runs (optim_kernels.cuh): the LbfgsState, the vectors of an iteration, the (s, y) history ring,
// f_hist, the per-iteration log flags and the Gram formulation's buffers.  The buffers only grow, so an owner that runs
// L-BFGS again reuses them.
struct DeviceLbfgs {
  pinn::LbfgsState* st = nullptr;
  double *g_old = nullptr, *d = nullptr, *x_final = nullptr, *S = nullptr, *Y = nullptr, *f_hist = nullptr;
  int* logged = nullptr;
  double *SY = nullptr, *YY = nullptr, *part = nullptr;   // Gram formulation (lbfgs_dots / lbfgs_solve / lbfgs_apply)
  int n_cap = 0, corr_cap = 0, iter_cap = 0, part_stride = 0;

  int reserve(int n, int n_corr, int max_iter) {
    if (!st) CUDA_TRY(cudaMalloc((void**)&st, sizeof(pinn::LbfgsState)));
    if (n > n_cap || n_corr > corr_cap) {
      if (n < n_cap) n = n_cap;
      if (n_corr < corr_cap) n_corr = corr_cap;
      for (double* b : {g_old, d, x_final, S, Y, SY, YY, part}) if (b) cudaFree(b);
      g_old = d = x_final = S = Y = SY = YY = part = nullptr;
      const size_t NS = (size_t)n_corr + 1;                 // + the spare history slot of the Gram formulation
      const size_t nb = (n + pinn::LB_CHUNK - 1) / pinn::LB_CHUNK;
      part_stride = pinn::LB_NSCAL + 4 * n_corr + 1;
      CUDA_TRY(cudaMalloc((void**)&g_old, (size_t)n * 8));
      CUDA_TRY(cudaMalloc((void**)&d, (size_t)n * 8));
      CUDA_TRY(cudaMalloc((void**)&x_final, (size_t)n * 8));
      CUDA_TRY(cudaMalloc((void**)&S, NS * n * 8));
      CUDA_TRY(cudaMalloc((void**)&Y, NS * n * 8));
      CUDA_TRY(cudaMalloc((void**)&SY, NS * NS * 8));
      CUDA_TRY(cudaMalloc((void**)&YY, NS * NS * 8));
      CUDA_TRY(cudaMalloc((void**)&part, nb * part_stride * 8));
      if ((size_t)n_corr * n_corr * 8 > 48 * 1024)
        CUDA_TRY(cudaFuncSetAttribute(pinn::lbfgs_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, n_corr * n_corr * 8));
      n_cap = n; corr_cap = n_corr;
    }
    if (max_iter + 2 > iter_cap) {
      if (f_hist) cudaFree(f_hist);
      if (logged) cudaFree(logged);
      f_hist = nullptr; logged = nullptr;
      CUDA_TRY(cudaMalloc((void**)&f_hist, (size_t)(max_iter + 2) * 8));
      CUDA_TRY(cudaMalloc((void**)&logged, (size_t)(max_iter + 2) * 4));
      iter_cap = max_iter + 2;
    }
    return 0;
  }

  // Clears f_hist and the log flags and writes the initial state of a run (after reserve).
  int start(cudaStream_t stream, const LbfgsConfig& c) {
    CUDA_TRY(cudaMemsetAsync(logged, 0, (size_t)(c.max_iter + 2) * 4, stream));
    CUDA_TRY(cudaMemsetAsync(f_hist, 0, (size_t)(c.max_iter + 2) * 8, stream));
    pinn::LbfgsState s{};
    s.pending = 1;                               // the initial evaluation comes first
    s.max_iter = c.max_iter; s.n_corr = c.n_corr; s.max_eval = c.max_eval;
    s.lr = c.lr; s.tol_fun = c.tol_fun; s.tol_x = c.tol_x; s.h_diag = 1.0;
    CUDA_TRY(cudaMemcpyAsync(st, &s, sizeof(s), cudaMemcpyHostToDevice, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));     // s is a stack object
    return 0;
  }

  // One iteration on the P-vector w, whose gradient and loss parts are R = [g | 3 loss parts].
  int iterate(cudaStream_t stream, double* w, const double* R, int P, long long* launches) const {
    if (lbfgs_serial()) {
#define LB_LAUNCH(E, NT) pinn::lbfgs_iterate<E, NT><<<1, NT, 0, stream>>>(st, w, R, P, g_old, d, S, Y, x_final, f_hist, logged)
      if (P <= 12 * 256) LB_LAUNCH(12, 256);        // Burgers-size vectors: 8 warps, 12 entries per thread
      else if (P <= 8 * 1024) LB_LAUNCH(8, 1024);
      else LB_LAUNCH(32, 1024);
#undef LB_LAUNCH
      if (cudaGetLastError() != cudaSuccess) return fail("lbfgs_iterate launch failed");
      if (launches) *launches += 1;
      return 0;
    }
    const int nb = (P + pinn::LB_CHUNK - 1) / pinn::LB_CHUNK;
    pinn::lbfgs_dots<<<nb, pinn::LB_DOT_THREADS, 0, stream>>>(st, R, P, g_old, d, S, Y, part, part_stride);
    pinn::lbfgs_solve<<<1, 128, (size_t)corr_cap * corr_cap * 8, stream>>>(st, R, P, part, nb, part_stride, SY, YY, f_hist, logged);
    pinn::lbfgs_apply<<<nb, pinn::LB_CHUNK, 0, stream>>>(st, w, R, P, g_old, d, S, Y, x_final);
    if (cudaGetLastError() != cudaSuccess) return fail("L-BFGS iteration launch failed");
    if (launches) *launches += 3;
    return 0;
  }

  void release() {
    for (double* b : {g_old, d, x_final, S, Y, f_hist, SY, YY, part}) if (b) cudaFree(b);
    if (logged) cudaFree(logged);
    if (st) cudaFree(st);
    *this = DeviceLbfgs{};
  }
};

// The fused loss/gradient kernel a handle runs, chosen once in pinn_create.
enum class Kernel {
  BurgersV2,      // specialised Burgers DMMA kernel, warp-specialised (default for the Burgers net)
  BurgersV1,      // specialised Burgers DMMA kernel, single-role (PINN_BURGERS_KERNEL=v1)
  Schrodinger,    // specialised NLS DMMA kernel
  Generic,        // any other layer list, and the discrete-time and polynomial residual heads
  NavierStokes,
};

// Grow-only per-CTA scratch of the generic, Schrodinger and Navier-Stokes kernels (activations, adjoints, seeds).  A handle
// runs one kernel, so one set serves it; it is regrown only when the points per CTA exceed those it was sized for.
struct Scratch {
  double *H = nullptr, *A = nullptr, *S = nullptr;
  long long pts = 0;

  int reserve(long long pts_per_cta, size_t h_bytes, size_t a_bytes, size_t s_bytes) {
    if (pts_per_cta <= pts) return 0;
    release();
    CUDA_TRY(cudaMalloc((void**)&H, h_bytes));
    CUDA_TRY(cudaMalloc((void**)&A, a_bytes));
    CUDA_TRY(cudaMalloc((void**)&S, s_bytes));
    pts = pts_per_cta;
    return 0;
  }

  void release() {
    for (double* b : {H, A, S}) if (b) cudaFree(b);
    *this = Scratch{};
  }
};

}  // namespace

struct pinn_handle {
  int pde = 0, device = 0, rank = 0, world = 1;
  std::vector<int> layers;
  double lb[3] = {0, 0, 0}, ub[3] = {1, 1, 1};    // NS_IDE: (x, y, t); the other models use the first two
  int P_net = 0, P = 0;             // net parameters; P = P_net (+2 identification)
  double nu = 0.0, dt = 0.0;        // AC_DISC: nu holds d
  double kc = 0.0;                  // AC_DISC: k
  double* d_irk = nullptr;          // DISC: (q+1) x q stage matrix
  int irk_q = 0;
  std::vector<double> h_x0;         // DISC, AC: data x positions (host copy for re-assembly); IDE_DISC, KdV: snapshot 0 (x_1 lives in h_tb)
  std::vector<double> h_u0, h_u1;   // IDE_DISC: targets of the two snapshots
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int n_sm = 0;
  long long launches = 0;
  bool tail_inflight = false;   // a launch with the in-kernel tail may still be running on this handle's stream
  pinn::ReduceMap last_map{};       // reduction map / grid / stride of the most recent fused launch (record_launch)
  int last_grid = 0, last_stride = 0;
  Kernel kernel = Kernel::Generic;
  Scratch scratch;

  // parameters and optimiser state
  double* d_w = nullptr;            // WPAD-padded flat weights
  int w_cap = 0;
  double* d_R = nullptr;            // [P grad | 3 loss parts | pad]
  double* d_partials = nullptr;
  int n_cta = 0, pstride = 0;
  double *d_m = nullptr, *d_v = nullptr;
  int* d_step = nullptr;
  double* d_loss_ring = nullptr;
  long long adam_steps = 0;

  // point sets (device SoA x[], t[]).  Layout: [data region, capacity dcap | collocation region, capacity ccap];
  // data points are stored right-aligned in their region so that [data | collocation] is contiguous:
  // kernel point 0 is at offset dcap - n_d.  A per-step collocation upload touches only its own region.
  double *d_x = nullptr, *d_t = nullptr, *d_u = nullptr;
  long long dcap = 0, ccap = 0, u_cap = 0;
  long long n_c = 0, n_c_global = 0, n_d = 0, n_b = 0;
  int d_out_dim = 1;
  double data_weight = 1.0;
  std::vector<double> h_tb;                 // NLS boundary times
  std::vector<double> h_icx, h_ict;         // NLS initial-condition points (host copy for re-assembly)
  const double *map_x = nullptr, *map_t = nullptr;   // zero-copy collocation block (device aliases of pinned host memory)
  long long n_aux = 0;                      // points stored in the data region (Burgers: n_d; NLS: n0p + 2 n_b)
  std::vector<double> stage_x, stage_t;     // host staging of the data-region block (upload_points)

  // measurement
  std::vector<cudaEvent_t> events;
  double* d_flush = nullptr;
  size_t flush_bytes = 0;

  // L-BFGS
  DeviceLbfgs lbfgs;
  std::vector<double> lb_fhist;             // f of every evaluation of the last pinn_lbfgs run (custom_lbfgs.py f_hist)

  // scratch for predict / derivatives
  double *d_px = nullptr, *d_pout = nullptr;
  long long px_cap = 0, pout_cap = 0;
  double* d_pscr = nullptr;                 // NS probe: streams of two layers [2][13][maxw][chunk]
  long long pscr_cap = 0;
  double* d_nsX = nullptr;                  // NS: training points [n][3] = (x, y, t); targets [n][2] in d_u
  long long nsx_cap = 0;
  double* d_rad = nullptr;                  // pinn_draw_collocation_rad: pool x, t, r^k, segment prefixes, block maxima and sums
  long long rad_cap = 0;

  // POLY_INF / POLY_IDE: the residual's term table (n == 0: not set yet) and the source: an array of values at the residual
  // points (h_src, copied to d_src; empty: none) or a table the device evaluates into d_src at every new set of points
  // (src_tab.n == 0: none).  At most one of the two is set.
  pinn::generic::PolySpec poly{};
  std::vector<double> h_src;
  pinn::source::Table src_tab{};
  double* d_src = nullptr;
  long long src_cap = 0;

  ncclComm_t comm = nullptr;
  // NVLink push exchange in the tail of every evaluation (optim_kernels.cuh: exchange_block)
  double* d_xchg = nullptr;            // [2][world][slot_len] doubles, then [2][world][n_blocks] u64 flags (IPC-exported)
  bool p2p_ready = false, p2p_mapped = false;
  pinn::XchgPeers peers{};
  void* peer_base[pinn::P2P_MAX] = {nullptr};
  int* d_xseq = nullptr;               // evaluations published to the peers
  int* d_p2p_err = nullptr;
};

namespace {

// What each model is, indexed by pde id.  Host code branches on these fields; a switch on the pde is left only where the models
// compute different things (the residual formulas, the constants, the layout of a re-assembled point block).
enum class Out { One, Two, QPlus1, Q };   // network outputs: exactly 1, exactly 2, q+1 >= 2 (IRK inference), q >= 1 (IRK identification)
enum class Res { None, Data, Colloc };    // residual points: none (discrete-time), the data points, the collocation set

struct Model {
  int in_dim;             // 1: x, 2: (x, t), 3: (x, y, t)
  Out out;
  int head_cap;           // widest output layer (the IRK head may be q+1 = 501 wide)
  int n_lambda;           // trained lambdas behind the net parameters: P = P_net + n_lambda
  Res residual;           // Res::Colloc: the model has a collocation set (pinn_set_collocation); no other model has one
  bool boundary;          // pinn_set_boundary
  bool snapshots;         // two snapshots (pinn_set_snapshot)
  bool irk;               // a stage matrix (pinn_set_irk)
  bool poly;              // a user-defined polynomial residual (pinn_set_residual, pinn_set_source) on generic::fused_loss_grad<true>
  Kernel kernel;          // the specialised kernel that runs the model's BASELINE net (Generic: none)
  const char* no_shard;   // why world must be 1 (nullptr: the model may be sharded)
};

// Sharding (utils/sharding.py) splits the collocation rows with the global 1/N_f and weights the replicated terms by the data
// weight.  The discrete-time heads have no collocation set and sum every term without a data weight, and Burgers
// identification puts its residual on the data points with the local 1/n_d: sharded, each of them counts the wrong loss.
constexpr const char* NO_SHARD_DISC = "pinn_create: the discrete-time models run on one GPU (world must be 1): they have no "
                                      "collocation set to shard and their heads read no data weight";
constexpr Model MODELS[10] = {
    /* BURGERS_INF      */ {2, Out::One, pinn::MAXW_WIDE, 0, Res::Colloc, false, false, false, false, Kernel::BurgersV2, nullptr},
    /* BURGERS_IDE      */ {2, Out::One, pinn::MAXW_WIDE, 2, Res::Data, false, false, false, false, Kernel::BurgersV2,
                            "pinn_create: the Burgers identification model runs on one GPU (world must be 1): its residual sits on "
                            "the data points, which carry no data weight"},
    /* NLS_INF          */ {2, Out::Two, pinn::MAXW_WIDE, 0, Res::Colloc, true, false, false, false, Kernel::Schrodinger, nullptr},
    /* BURGERS_DISC     */ {1, Out::QPlus1, 512, 0, Res::None, true, false, true, false, Kernel::Generic, NO_SHARD_DISC},
    /* BURGERS_IDE_DISC */ {1, Out::Q, 512, 2, Res::None, false, true, true, false, Kernel::Generic, NO_SHARD_DISC},
    /* KDV_IDE_DISC     */ {1, Out::Q, 512, 2, Res::None, false, true, true, false, Kernel::Generic, NO_SHARD_DISC},
    /* AC_DISC          */ {1, Out::QPlus1, 512, 0, Res::None, false, false, true, false, Kernel::Generic, NO_SHARD_DISC},
    /* NS_IDE           */ {3, Out::Two, pinn::MAXW_WIDE, 2, Res::Data, false, false, false, false, Kernel::NavierStokes,
                            "pinn_create: the Navier-Stokes identification model runs on one GPU (world must be 1)"},
    /* POLY_INF         */ {2, Out::One, pinn::MAXW_WIDE, 0, Res::Colloc, false, false, false, true, Kernel::Generic,
                            "pinn_create: the polynomial residual models run on one GPU (world must be 1)"},
    /* POLY_IDE         */ {2, Out::One, pinn::MAXW_WIDE, 2, Res::Data, false, false, false, true, Kernel::Generic,
                            "pinn_create: the polynomial residual models run on one GPU (world must be 1)"},
};
static_assert(sizeof(MODELS) / sizeof(MODELS[0]) == PINN_POLY_IDE + 1, "one MODELS row per pde id");

const Model& model(const pinn_t* h) { return MODELS[h->pde]; }

bool is_burgers_net(const std::vector<int>& L) {
  if (L.size() != 10 || L[0] != 2 || L[9] != 1) return false;
  for (int i = 1; i <= 8; i++) if (L[i] != 20) return false;
  return true;
}
bool is_nls_net(const std::vector<int>& L) {
  if (L.size() != 6 || L[0] != 2 || L[5] != 2) return false;
  for (int i = 1; i <= 4; i++) if (L[i] != 100) return false;
  return true;
}

int nls_launch_eval(pinn_t* h, const int* run_flag);
int generic_launch_eval(pinn_t* h, const int* run_flag);
int ns_launch_eval(pinn_t* h, const int* run_flag);

// after a stream synchronisation: has the fused P2P exchange reported a peer that never published?
int check_p2p(pinn_t* h) {
  if (!h->p2p_ready) return 0;
  int e = 0;
  if (cudaMemcpy(&e, h->d_p2p_err, 4, cudaMemcpyDeviceToHost) != cudaSuccess) return fail("reading the P2P error flag failed");
  if (e) return fail("P2P exchange timed out waiting for a peer rank (a rank died or the evaluation counts diverged); "
                     "weights and optimiser state were left untouched by that step");
  return 0;
}

pinn::NetDesc net_desc(const pinn_t* h) {
  pinn::NetDesc nd{};
  nd.n_layers = (int)h->layers.size() - 1;
  int o = 0;
  for (int l = 0; l < nd.n_layers; l++) {
    nd.dims[l] = h->layers[l];
    nd.woff[l] = o; o += h->layers[l] * h->layers[l + 1];
    nd.boff[l] = o; o += h->layers[l + 1];
  }
  nd.dims[nd.n_layers] = h->layers.back();
  nd.lb0 = h->lb[0]; nd.lb1 = h->lb[1];
  nd.dx0 = h->ub[0] - h->lb[0]; nd.dx1 = h->ub[1] - h->lb[1];
  return nd;
}

int ensure(double** p, long long* cap, long long need) {
  if (need <= *cap) return 0;
  if (*p) cudaFree(*p);
  *p = nullptr;
  long long c = need + need / 8 + 64;
  if (cudaMalloc((void**)p, (size_t)c * sizeof(double)) != cudaSuccess) return fail("cudaMalloc failed");
  *cap = c;
  return 0;
}

// grow the point arrays, preserving both regions
int ensure_points(pinn_t* h, long long need_d, long long need_c) {
  if (need_d <= h->dcap && need_c <= h->ccap && h->d_x) return 0;
  long long nd = h->dcap, nc = h->ccap;
  if (need_d > nd) nd = need_d + need_d / 4 + 1024;
  if (need_c > nc) nc = need_c + need_c / 8 + 1024;
  if (nd < 1024) nd = 1024;
  double *nx = nullptr, *nt = nullptr;
  CUDA_TRY(cudaMalloc((void**)&nx, (size_t)(nd + nc) * 8));
  CUDA_TRY(cudaMalloc((void**)&nt, (size_t)(nd + nc) * 8));
  if (h->d_x) {
    if (h->n_aux) {
      CUDA_TRY(cudaMemcpyAsync(nx + nd - h->n_aux, h->d_x + h->dcap - h->n_aux, h->n_aux * 8, cudaMemcpyDeviceToDevice, h->stream));
      CUDA_TRY(cudaMemcpyAsync(nt + nd - h->n_aux, h->d_t + h->dcap - h->n_aux, h->n_aux * 8, cudaMemcpyDeviceToDevice, h->stream));
    }
    // the device-resident collocation block: nothing to preserve while the batch is a zero-copy mapping of pinned host
    // memory (n_c then counts the HOST batch and ccap may be 0), and never more than the old region held
    const long long keep_c = h->map_x ? 0 : (h->n_c < h->ccap ? h->n_c : h->ccap);
    if (keep_c) {
      CUDA_TRY(cudaMemcpyAsync(nx + nd, h->d_x + h->dcap, keep_c * 8, cudaMemcpyDeviceToDevice, h->stream));
      CUDA_TRY(cudaMemcpyAsync(nt + nd, h->d_t + h->dcap, keep_c * 8, cudaMemcpyDeviceToDevice, h->stream));
    }
    CUDA_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_x); cudaFree(h->d_t);
  }
  h->d_x = nx; h->d_t = nt; h->dcap = nd; h->ccap = nc;
  return 0;
}

// Writes the staged block (stage_x, stage_t) right-aligned into the data region, growing the point arrays for it and for the
// current collocation set first; kernel point 0 then sits at dcap - n_aux.
int upload_points(pinn_t* h) {
  const long long n = (long long)h->stage_x.size();
  if (ensure_points(h, n, h->n_c)) return -1;
  if (n) {
    CUDA_TRY(cudaMemcpyAsync(h->d_x + h->dcap - n, h->stage_x.data(), n * 8, cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(cudaMemcpyAsync(h->d_t + h->dcap - n, h->stage_t.data(), n * 8, cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(cudaStreamSynchronize(h->stream));
  }
  h->n_aux = n;
  return 0;
}

// The data-region blocks that are re-assembled from host copies whenever one of their parts changes.
//   Schrodinger: [initial-condition points | pad to even | (lb_k, ub_k) pairs] (inf_cont_schrodinger.py:50-53 builds
//                X_lb = (0*tb+lb0, tb), X_ub = (0*tb+ub0, tb)); the pairs are adjacent and must not straddle a CTA.
//   Allen-Cahn: [x_0 | pad to even | lb, ub]: the periodic pair starts at an even index, so it never straddles a CTA.
//   other discrete-time models: [x_0 data points | x_1 boundary points or snapshot].  t is unused in all three 1-D layouts.
int assemble_points(pinn_t* h) {
  const long long n0 = h->n_d, n0p = (n0 + 1) & ~1LL;
  std::vector<double> &x = h->stage_x, &t = h->stage_t;
  switch (h->pde) {
    case PINN_NLS_INF:
      x.assign(n0p + 2 * h->n_b, 0.0); t.assign(x.size(), 0.0);
      for (long long i = 0; i < n0; i++) { x[i] = h->h_icx[i]; t[i] = h->h_ict[i]; }
      if (n0p > n0) { x[n0] = h->lb[0]; t[n0] = h->lb[1]; }     // inert alignment point
      for (long long k = 0; k < h->n_b; k++) {
        // x as the reference forms it, 0 * tb + lb0: NaN for an infinite or NaN tb, lb0 (ub0) for every finite one
        x[n0p + 2 * k] = 0.0 * h->h_tb[k] + h->lb[0];     t[n0p + 2 * k] = h->h_tb[k];
        x[n0p + 2 * k + 1] = 0.0 * h->h_tb[k] + h->ub[0]; t[n0p + 2 * k + 1] = h->h_tb[k];
      }
      break;
    case PINN_AC_DISC:
      x.assign(n0 > 0 ? n0p + 2 : 0, 0.0); t.assign(x.size(), 0.0);
      for (long long i = 0; i < n0; i++) x[i] = h->h_x0[i];
      if (n0 > 0) {
        for (long long i = n0; i < n0p; i++) x[i] = h->lb[0];    // inert alignment point
        x[n0p] = h->lb[0]; x[n0p + 1] = h->ub[0];
      }
      break;
    default:
      x.assign(n0 + h->n_b, 0.0); t.assign(x.size(), 0.0);
      for (long long i = 0; i < n0; i++) x[i] = h->h_x0[i];
      for (long long i = 0; i < h->n_b; i++) x[n0 + i] = h->h_tb[i];
      break;
  }
  return upload_points(h);
}

// Copies n doubles from the caller's buffer into the grow-only device buffer *p and waits: the buffer is only borrowed.
int upload(pinn_t* h, double** p, long long* cap, const double* src, long long n) {
  if (n <= 0) return 0;
  if (ensure(p, cap, n)) return -1;
  CUDA_TRY(cudaMemcpyAsync(*p, src, n * 8, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  return 0;
}

// POLY_INF / POLY_IDE with a source table: enqueues s at the stored residual points into d_src (the collocation set, or the
// data points for POLY_IDE).  Called whenever those points or the table change; only a growing d_src synchronises.
int fill_source(pinn_t* h) {
  const long long n = pinn_num_residual_points(h);
  if (h->src_tab.n == 0 || n == 0) return 0;
  if (ensure(&h->d_src, &h->src_cap, n)) return -1;
  const long long off = model(h).residual == Res::Data ? h->dcap - h->n_d : h->dcap;
  const long long blocks = (n + pinn::source::THREADS - 1) / pinn::source::THREADS;
  const int grid = (int)(blocks < 8LL * h->n_sm ? blocks : 8LL * h->n_sm);     // one wave of 256-thread blocks, grid-stride beyond
  pinn::source::eval_kernel<<<grid, pinn::source::THREADS, 0, h->stream>>>(h->src_tab, h->d_x + off, h->d_t + off, h->d_src,
                                                                            (uint64_t)n);
  CUDA_TRY(cudaGetLastError());
  h->launches++;
  return 0;
}

// Records h's most recent fused launch for the tail that reduces it (make_tail, launch_tail): the grid, the stride of the
// partial vectors and the ReduceMap -- the p_net net-gradient entries, then the partial-vector entries of the two trained lambdas
// (lam; nullptr when there are none) and of the data, boundary and residual loss parts.
void record_launch(pinn_t* h, int grid, int stride, int p_net, const int* lam, int l_data, int l_bnd, int l_res) {
  pinn::ReduceMap map{};
  map.p_net = p_net;
  if (lam) { map.extra_src[map.n_extra++] = lam[0]; map.extra_src[map.n_extra++] = lam[1]; }
  for (int s : {l_data, l_bnd, l_res}) map.extra_src[map.n_extra++] = s;
  map.n_out = map.p_net + map.n_extra;
  h->last_map = map; h->last_grid = grid; h->last_stride = stride;
}

struct AdamArgs { double lr, b1, b2, eps; };

// The tail of h's most recent fused launch (h->last_map): with Adam when ad != nullptr, with the P2P exchange when world > 1 and
// the peers are connected.
int make_tail(pinn_t* h, const AdamArgs* ad, pinn::Tail* tl) {
  *tl = pinn::Tail{};
  tl->R = h->d_R; tl->map = h->last_map; tl->step = h->d_step;
  tl->w = h->d_w; tl->m = h->d_m; tl->v = h->d_v; tl->P = h->P;
  tl->loss_ring = h->d_loss_ring; tl->ring = LOSS_RING;
  if (ad) { tl->adam = 1; tl->lr = ad->lr; tl->b1 = ad->b1; tl->b2 = ad->b2; tl->eps = ad->eps; }
  if (h->world > 1 && h->p2p_ready) {
    if ((tl->map.n_out + 31) / 32 != h->peers.n_blocks || tl->map.n_out > h->peers.slot_len)
      return fail("internal: exchange buffer geometry mismatch");
    tl->xchg = 1; tl->peers = h->peers; tl->xseq = h->d_xseq; tl->err = h->d_p2p_err;
  }
  return 0;
}

// The tail of an evaluation: fixed-order reduction of the per-CTA partials into R = [grad | loss parts] on every rank,
// optionally fused with the Adam update.
// (Evaluations of the specialised Burgers kernel do all of this in their own last CTAs -- fused_tail -- and never get here.)
//   world == 1, or P2P : reduce_tail -- reduction (+ NVLink all-to-all push + rank-ordered sum) (+ Adam) in ONE kernel
//   world > 1, NCCL    : reduce_tail + ncclAllReduce(P+3 doubles) (+ adam_update)
int launch_tail(pinn_t* h, const int* run_flag, const AdamArgs* ad) {
  const bool nccl = h->world > 1 && !h->p2p_ready;
  pinn::Tail tl;
  if (make_tail(h, nccl ? nullptr : ad, &tl)) return -1;
  const int nb = (tl.map.n_out + 31) / 32;
  const int grid = tl.xchg && nb > 2 * h->n_sm ? 2 * h->n_sm : nb;   // certainly co-resident: <= 2 blocks of 256 threads per SM
  pinn::reduce_tail<<<grid, 256, 0, h->stream>>>(h->d_partials, h->last_grid, h->last_stride, tl, run_flag);
  CUDA_TRY(cudaGetLastError());
  h->launches++;
  if (!nccl) return 0;
  // one exchange over [gradient | loss parts] (SURVEY 8(e)).  A skipped evaluation (L-BFGS stopped) still takes part with
  // stale but rank-identical participation so that ranks never diverge.
  int rc = g_nccl.AllReduce(h->d_R, h->d_R, (size_t)h->P + 3, NCCL_FLOAT64, NCCL_SUM, h->comm, h->stream);
  if (rc != 0) return fail(std::string("ncclAllReduce: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "error"));
  if (ad) {
    if (make_tail(h, ad, &tl)) return -1;
    pinn::adam_update<<<(h->P + 127) / 128, 128, 0, h->stream>>>(tl);
    CUDA_TRY(cudaGetLastError());
    h->launches++;
  }
  return 0;
}

// true when no other live handle on h's device may still be running a launch with the in-kernel tail
bool tail_slot_free(pinn_t* h) {
  std::lock_guard<std::mutex> lk(g_live_mu);
  for (pinn_t* o : g_live) {
    if (o == h || o->device != h->device || !o->tail_inflight) continue;
    if (cudaStreamQuery(o->stream) == cudaSuccess) o->tail_inflight = false;
    else return false;
  }
  (void)cudaGetLastError();               // cudaErrorNotReady from the query is not an error of ours
  return true;
}

// v2 kernel with tail_done != nullptr: the launch also reduces the partials (+ exchanges them, + applies Adam when ad != nullptr) in
// its last CTAs (fused_tail); *tail_done tells the caller that no tail kernel is needed.  PINN_FUSED_TAIL=0 keeps the tail kernel.
int burgers_launch_eval(pinn_t* h, const int* run_flag, const AdamArgs* ad = nullptr, bool* tail_done = nullptr) {
  namespace B = pinn::burgers;
  const bool ide = model(h).residual == Res::Data;
  const bool v2 = h->kernel == Kernel::BurgersV2;
  const long long n_total = ide ? h->n_d : h->n_d + h->n_c;
  if (n_total <= 0) return fail("no points set (pinn_set_collocation / pinn_set_data)");
  B::Args a{};
  a.w = h->d_w;
  a.x = h->d_x + (h->dcap - h->n_d); a.t = h->d_t + (h->dcap - h->n_d); a.utgt = h->d_u;
  a.xc = h->map_x; a.tc = h->map_t;
  if (h->map_x && !v2) return fail("zero-copy collocation needs the v2 Burgers kernel");
  a.n_total = n_total;
  a.c0 = ide ? 0 : h->n_d;
  a.n_c = ide ? h->n_d : h->n_c;
  a.d0 = 0;
  a.n_d = h->n_d;
  const long long nfg = ide ? h->n_d : h->n_c_global;
  a.wf = nfg > 0 ? 1.0 / (double)nfg : 0.0;
  a.wd = h->n_d > 0 ? h->data_weight / (double)h->n_d : 0.0;
  a.lb0 = h->lb[0]; a.lb1 = h->lb[1];
  a.dx0 = h->ub[0] - h->lb[0]; a.dx1 = h->ub[1] - h->lb[1];
  a.nu = h->nu; a.ide = ide ? 1 : 0;
  a.partials = h->d_partials;
  a.run_flag = run_flag;
  // v2: tile-granular distribution inside the kernel (any grid <= tiles); v1: rounds of 32 points striped over the CTAs
  a.chains = 4;
  const long long n_tiles = (n_total + B::TILE - 1) / B::TILE;
  const long long rounds = (n_total + B::ROUND - 1) / B::ROUND;
  const long long units = v2 ? n_tiles : rounds;
  int grid = (int)(units < h->n_cta ? units : h->n_cta);
  const int lam[2] = {B::IDX_DL1, B::IDX_DL2};
  record_launch(h, grid, B::PSTRIDE, B::P_NET, ide ? lam : nullptr, B::IDX_LD, 3023, B::IDX_LF);   // (3023: the boundary part, always 0)
  static const bool fused_tail_on = [] { const char* e = getenv("PINN_FUSED_TAIL"); return !(e && e[0] == '0'); }();
  // every evaluation of the v2 kernel carries its own tail: Adam steps (ad != nullptr) and plain evaluations (L-BFGS, loss/gradient
  // queries; a launch skipped through run_flag skips its tail with it, exactly like the stand-alone tail kernel)
  if (tail_done && fused_tail_on && (h->world == 1 || h->p2p_ready) && v2 && grid <= h->n_sm && tail_slot_free(h)) {
    if (make_tail(h, ad, &a.tail)) return -1;
    a.tail.enabled = 1;
    h->tail_inflight = true;
    *tail_done = true;
  }
  if (v2)
    pinn::burgers2::fused_loss_grad<<<grid, pinn::burgers2::THREADS, pinn::burgers2::SMEM_BYTES, h->stream>>>(a);
  else
    B::fused_loss_grad<<<grid, B::THREADS, B::SMEM_BYTES, h->stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  h->launches++;
  return 0;
}

// one evaluation: the fused loss/gradient kernel of the handle's PDE, then (unless fused_only) the tail
int launch_eval(pinn_t* h, const int* run_flag, bool fused_only = false, const AdamArgs* ad = nullptr) {
  int rc = 0;
  bool tail_done = false;
  switch (h->kernel) {
    case Kernel::BurgersV2:
    case Kernel::BurgersV1: rc = burgers_launch_eval(h, run_flag, ad, fused_only ? nullptr : &tail_done); break;
    case Kernel::Schrodinger: rc = nls_launch_eval(h, run_flag); break;
    case Kernel::Generic: rc = generic_launch_eval(h, run_flag); break;
    case Kernel::NavierStokes: rc = ns_launch_eval(h, run_flag); break;
  }
  if (rc) return -1;
  if (fused_only || tail_done) return 0;
  return launch_tail(h, run_flag, ad);
}

int generic_launch_eval(pinn_t* h, const int* run_flag) {
  namespace G = pinn::generic;
  const Model& m = model(h);
  if (m.irk && (!h->d_irk || h->irk_q + (m.out == Out::QPlus1 ? 1 : 0) != h->layers.back()))
    return fail("discrete-time model: call pinn_set_irk first");
  if (m.poly && h->poly.n == 0) return fail("polynomial residual model: call pinn_set_residual first (no residual is set)");
  const bool ide = m.residual == Res::Data;
  // the kernel's points: the block right-aligned in the data region, then the collocation set (n_c is 0 for models without one)
  const long long n_total = h->n_aux + h->n_c;
  if (n_total <= 0) return fail("no points set (pinn_set_collocation / pinn_set_data)");
  const long long per = (n_total + h->n_cta - 1) / h->n_cta;
  // points per CTA: a multiple of 16 for large sets; small sets (the discrete-time models have ~250 points) are spread over as
  // many CTAs as possible -- an even count, because NLS boundary pairs (lb_k, ub_k) are adjacent and must not straddle a CTA
  const long long pts = per >= 16 ? (per + 15) / 16 * 16 : (per + 1) / 2 * 2;
  // only CTAs that own points are launched: every CTA writes (and the tail kernel reads) a full partial vector
  const int grid = (int)((n_total + pts - 1) / pts);
  pinn::NetDesc nd = net_desc(h);
  int maxw = 0; long long hsum = 0;
  for (int l = 0; l < nd.n_layers - 1; l++) { hsum += 4 * pts * nd.dims[l + 1]; if (nd.dims[l + 1] > maxw) maxw = nd.dims[l + 1]; }
  const int out_w = nd.dims[nd.n_layers];
  if (out_w > maxw) maxw = out_w;                 // the IRK head reuses the adjoint scratch for N, N-bar and 2(U_0 - u_0)
  const long long a_per = 4 * pts * maxw;
  // sized for the largest grid (all CTAs)
  if (h->scratch.reserve(pts, (size_t)h->n_cta * hsum * 8, (size_t)h->n_cta * 2 * a_per * 8, (size_t)h->n_cta * 2 * pts * 4 * out_w * 8))
    return -1;
  G::Args a{};
  a.w = h->d_w; a.nd = nd;
  a.x = h->d_x + (h->dcap - h->n_aux); a.t = h->d_t + (h->dcap - h->n_aux); a.tgt = h->d_u;
  a.n_total = n_total; a.pde = h->pde;
  a.in_dim = m.in_dim; a.dt = h->dt; a.irk = h->d_irk;
  a.o3 = h->pde == PINN_KDV_IDE_DISC ? 1 : 0; a.kc = h->kc;
  a.c0 = ide ? 0 : h->n_d; a.n_c = ide ? h->n_d : h->n_c; a.d0 = 0; a.n_d = h->n_d;
  const long long nfg = ide ? h->n_d : h->n_c_global;
  a.wf = nfg > 0 ? 1.0 / (double)nfg : 0.0;
  a.wd = h->n_d > 0 ? h->data_weight / (double)h->n_d : 0.0;
  a.nu = h->nu;
  a.n0 = h->n_d; a.n0p = (h->n_d + 1) & ~1LL; a.nb = h->n_b;
  a.w0 = h->n_d > 0 ? h->data_weight / (double)h->n_d : 0.0;
  a.wb = h->n_b > 0 ? h->data_weight / (double)h->n_b : 0.0;
  if (h->pde == PINN_NLS_INF && h->n_aux != a.n0p + 2 * a.nb) return fail("internal: NLS auxiliary block out of date");
  a.p_net = h->P_net;
  a.scrH = h->scratch.H; a.scrA = h->scratch.A; a.scrS = h->scratch.S;
  a.h_per_cta = hsum; a.a_per_cta = a_per;
  a.pts = (int)pts; a.maxw = maxw;
  static const bool generic_dfma = [] { const char* e = getenv("PINN_GENERIC_DFMA"); return e && e[0] == '1'; }();
  a.dmma = generic_dfma ? 0 : 1;
  a.partials = h->d_partials; a.pstride = h->pstride; a.run_flag = run_flag;
  if (m.poly) {
    a.poly = h->poly;
    a.src = h->h_src.empty() && h->src_tab.n == 0 ? nullptr : h->d_src;
    G::fused_loss_grad<true><<<grid, G::THREADS, 0, h->stream>>>(a);
  } else {
    G::fused_loss_grad<false><<<grid, G::THREADS, 0, h->stream>>>(a);
  }
  CUDA_TRY(cudaGetLastError());
  h->launches++;
  const int lam[2] = {h->P_net, h->P_net + 1};
  record_launch(h, grid, h->pstride, h->P_net, m.n_lambda ? lam : nullptr, h->P_net + 3, h->P_net + 4, h->P_net + 5);
  return 0;
}

// Navier-Stokes identification: every data point also carries the residual term.  A CTA per SM (the kernel is built for one
// 256-thread CTA per SM), points split evenly; only CTAs that own points are launched.
int ns_launch_eval(pinn_t* h, const int* run_flag) {
  namespace S = pinn::nsid;
  const long long n_total = h->n_d;
  if (n_total <= 0) return fail("no points set (pinn_set_data)");
  const long long pts = (n_total + h->n_cta - 1) / h->n_cta;
  const int grid = (int)((n_total + pts - 1) / pts);
  pinn::NetDesc nd = net_desc(h);
  int maxw = 0; long long hsum = 0;
  for (int l = 0; l < nd.n_layers - 1; l++) { hsum += S::NST * pts * nd.dims[l + 1]; if (nd.dims[l + 1] > maxw) maxw = nd.dims[l + 1]; }
  const long long a_per = S::NST * pts * maxw;
  if (h->scratch.reserve(pts, (size_t)h->n_cta * hsum * 8, (size_t)h->n_cta * 2 * a_per * 8, (size_t)h->n_cta * 2 * pts * S::SEEDW * 8))
    return -1;
  S::Args a{};
  a.w = h->d_w; a.nd = nd;
  for (int c = 0; c < 3; c++) { a.lb[c] = h->lb[c]; a.sc[c] = 2.0 / (h->ub[c] - h->lb[c]); }
  a.X = h->d_nsX; a.tgt = h->d_u; a.n_total = n_total; a.p_net = h->P_net;
  a.scrH = h->scratch.H; a.scrA = h->scratch.A; a.scrS = h->scratch.S;
  a.h_per_cta = hsum; a.a_per_cta = a_per; a.pts = (int)pts;
  a.partials = h->d_partials; a.pstride = h->pstride; a.run_flag = run_flag;
  S::fused_loss_grad<<<grid, S::THREADS, 0, h->stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  h->launches++;
  const int lam[2] = {h->P_net, h->P_net + 1};
  record_launch(h, grid, h->pstride, h->P_net, lam, h->P_net + 2, h->P_net + 3, h->P_net + 4);
  return 0;
}

// NS probe (pinn_predict / pinn_derivatives / pinn_residual): mode 0 (psi, p), 1 all 13 streams, 2 (f_u, f_v); X is [n][3] on
// the device.  Chunks of points keep the two-layer stream scratch within 256 MB.
int ns_probe(pinn_t* h, const double* dX, int64_t n, int mode, double* out_host) {
  namespace S = pinn::nsid;
  const int per = mode == 1 ? S::SEEDW : 2;
  if (ensure(&h->d_pout, &h->pout_cap, n * per)) return -1;
  pinn::NetDesc nd = net_desc(h);
  int maxw = 1;
  for (int l = 1; l < nd.n_layers; l++) maxw = nd.dims[l] > maxw ? nd.dims[l] : maxw;
  long long chunk = (32LL << 20) / (2LL * S::NST * maxw);
  if (chunk > n) chunk = n;
  if (ensure(&h->d_pscr, &h->pscr_cap, 2LL * S::NST * maxw * chunk)) return -1;
  S::Probe pr{};
  for (int c = 0; c < 3; c++) { pr.lb[c] = h->lb[c]; pr.sc[c] = 2.0 / (h->ub[c] - h->lb[c]); }
  pr.p_net = h->P_net; pr.maxw = maxw; pr.mode = mode; pr.chunk = chunk;
  for (long long c0 = 0; c0 < n; c0 += chunk) {
    const long long m = n - c0 < chunk ? n - c0 : chunk;
    S::probe_forward<<<(int)((m + 127) / 128), 128, 0, h->stream>>>(h->d_w, nd, pr, dX + 3 * c0, m, h->d_pout + per * c0, h->d_pscr);
    CUDA_TRY(cudaGetLastError());
    h->launches++;
  }
  CUDA_TRY(cudaMemcpyAsync(out_host, h->d_pout, n * per * 8, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  return 0;
}

int nls_launch_eval(pinn_t* h, const int* run_flag) {
  namespace N = pinn::nls;
  const long long n0 = h->n_d, n0p = (n0 + 1) & ~1LL, nb = h->n_b;
  const long long n_total = h->n_aux + h->n_c;
  if (n_total <= 0) return fail("no points set (pinn_set_collocation / pinn_set_data / pinn_set_boundary)");
  if (h->n_aux != n0p + 2 * nb) return fail("internal: NLS auxiliary block out of date");
  const int grid = h->n_cta;
  long long per = (n_total + grid - 1) / grid;
  const int pts = (int)((per + N::RPTS - 1) / N::RPTS * N::RPTS);
  if (h->scratch.reserve(pts, (size_t)grid * 16 * pts * N::W * 8, (size_t)grid * 8 * pts * N::W * 8, (size_t)grid * pts * 8 * 8))
    return -1;
  N::Args a{};
  a.w = h->d_w;
  a.x = h->d_x + (h->dcap - h->n_aux); a.t = h->d_t + (h->dcap - h->n_aux); a.uv0 = h->d_u;
  a.n_total = n_total; a.n0 = n0; a.n0p = n0p; a.nb = nb; a.nc = h->n_c;
  a.w0 = n0 > 0 ? h->data_weight / (double)n0 : 0.0;
  a.wb = nb > 0 ? h->data_weight / (double)nb : 0.0;
  a.wf = h->n_c_global > 0 ? 1.0 / (double)h->n_c_global : 0.0;
  a.lb0 = h->lb[0]; a.lb1 = h->lb[1]; a.dx0 = h->ub[0] - h->lb[0]; a.dx1 = h->ub[1] - h->lb[1];
  a.scratchH = h->scratch.H; a.scratchA = h->scratch.A; a.scratchS = h->scratch.S;
  // the kernel derives its point range from a.pts, so keep the distribution even when the scratch is larger
  a.pts = pts;
  a.partials = h->d_partials; a.run_flag = run_flag;
  N::fused_loss_grad<<<grid, N::THREADS, N::SMEM_BYTES, h->stream>>>(a);
  CUDA_TRY(cudaGetLastError());
  h->launches++;
  record_launch(h, grid, N::PSTRIDE, N::P_NET, nullptr, N::IDX_L0, N::IDX_LB, N::IDX_LF);
  return 0;
}

}  // namespace

extern "C" {

const char* pinn_last_error(void) { return g_err.c_str(); }
const char* pinn_version(void) { return "pinn_b200 0.1 (sm_90a, fp64 DMMA)"; }

int pinn_p2p_export(pinn_t* h, void* out64) {
  if (!h || !out64) return fail("pinn_p2p_export: null argument");
  if (h->world < 2 || h->world > pinn::P2P_MAX) return fail("pinn_p2p_export: needs 2..8 ranks");
  CUDA_TRY(cudaSetDevice(h->device));
  if (!h->d_xchg) {
    const int n = h->P + 3;
    h->peers.world = h->world; h->peers.rank = h->rank;
    h->peers.slot_len = ((n + 15) / 16) * 16;
    h->peers.n_blocks = (n + 31) / 32;
    const size_t data_bytes = (size_t)2 * h->world * h->peers.slot_len * 8;
    const size_t flag_bytes = (size_t)2 * h->world * h->peers.n_blocks * 8;
    CUDA_TRY(cudaMalloc((void**)&h->d_xchg, data_bytes + flag_bytes));
    CUDA_TRY(cudaMemset(h->d_xchg, 0, data_bytes + flag_bytes));
    CUDA_TRY(cudaMalloc((void**)&h->d_p2p_err, 4));
    CUDA_TRY(cudaMemset(h->d_p2p_err, 0, 4));
    CUDA_TRY(cudaMalloc((void**)&h->d_xseq, 4));
    CUDA_TRY(cudaMemset(h->d_xseq, 0, 4));
    CUDA_TRY(cudaDeviceSynchronize());
  }
  cudaIpcMemHandle_t hd;
  CUDA_TRY(cudaIpcGetMemHandle(&hd, h->d_xchg));
  static_assert(sizeof(hd) == 64, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(out64, &hd, 64);
  return 0;
}

int pinn_p2p_connect(pinn_t* h, const void* handles, int world) {
  if (!h || !handles) return fail("pinn_p2p_connect: null argument");
  if (world != h->world || world < 2 || world > pinn::P2P_MAX) return fail("pinn_p2p_connect: world must match pinn_create (2..8)");
  if (!h->d_xchg) return fail("pinn_p2p_connect: call pinn_p2p_export first");
  CUDA_TRY(cudaSetDevice(h->device));
  const size_t data_doubles = (size_t)2 * world * h->peers.slot_len;
  for (int r = 0; r < world; r++) {
    void* base = nullptr;
    if (r == h->rank) {
      base = h->d_xchg;
    } else {
      cudaIpcMemHandle_t hd;
      memcpy(&hd, (const char*)handles + (size_t)r * 64, 64);
      cudaError_t e = cudaIpcOpenMemHandle(&base, hd, cudaIpcMemLazyEnablePeerAccess);
      if (e != cudaSuccess) { cudaGetLastError(); return fail(std::string("cudaIpcOpenMemHandle(rank ") + std::to_string(r) + "): " + cudaGetErrorString(e)); }
      h->peer_base[r] = base;
    }
    h->peers.data[r] = (double*)base;
    h->peers.flag[r] = reinterpret_cast<unsigned long long*>((double*)base + data_doubles);
  }
  h->p2p_mapped = true;
  h->p2p_ready = true;
  return 0;
}

int pinn_p2p_enable(pinn_t* h, int on) {
  if (!h) return fail("null handle");
  if (on && !h->p2p_mapped) return fail("pinn_p2p_enable: call pinn_p2p_connect first");
  h->p2p_ready = on != 0;
  return 0;
}

int pinn_nccl_unique_id(void* out128) {
  std::string why;
  if (!g_nccl.load(why)) return fail(why);
  ncclUniqueId id;
  int rc = g_nccl.GetUniqueId(&id);
  if (rc != 0) return fail("ncclGetUniqueId failed");
  memcpy(out128, &id, 128);
  return 0;
}

int pinn_create(pinn_t** out, int pde_id, int n_layers, const int* layers, const double* lb, const double* ub,
                int device, int rank, int world, const void* nccl_uid) {
  if (!out || !layers || !lb || !ub) return fail("pinn_create: null argument");
  if (n_layers < 3 || n_layers > pinn::MAXL) return fail("pinn_create: need 3..16 layer sizes");
  if (pde_id < 0 || pde_id > 9) return fail("pinn_create: unknown pde_id");
  const Model& m = MODELS[pde_id];
  if (world > 1 && m.no_shard) return fail(m.no_shard);
  const int q = layers[n_layers - 1];
  if (m.poly && (layers[0] != 2 || q != 1))
    return fail("pinn_create: unknown pde_id for a [" + std::to_string(layers[0]) + ", ..., " + std::to_string(q) +
                "] net: the polynomial residual models (8, 9) take a net [2, ..., 1]: (x, t) -> u");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail("pinn_create: no CUDA device -- this library has no CPU fallback");
  if (device < 0 || device >= ndev) return fail("pinn_create: bad device index");
  for (int i = 0; i < n_layers; i++)
    if (layers[i] < 1 || layers[i] > (i == n_layers - 1 ? m.head_cap : pinn::MAXW_WIDE))
      return fail("pinn_create: layer width out of range (1..256; IRK head <= 512)");
  if (m.in_dim == 3 ? (layers[0] != 3 || q != 2) : layers[0] != m.in_dim)
    return fail(m.in_dim == 3   ? "pinn_create: the Navier-Stokes identification model needs a net [3, ..., 2]: (x, y, t) -> (psi, p)"
                : m.in_dim == 1 ? "pinn_create: the discrete-time model takes a 1-D input (x)"
                                : "pinn_create: input dimension must be 2 (x,t)");
  double lo[3] = {0.0, 0.0, 0.0}, hi[3] = {1.0, 1.0, 1.0};     // an axis the model does not have (t of a 1-D net) keeps [0, 1]
  for (int c = 0; c < m.in_dim; c++) { lo[c] = lb[c]; hi[c] = ub[c]; }
  if (!(hi[0] > lo[0]) || !(hi[1] > lo[1]) || !(hi[2] > lo[2])) return fail("pinn_create: need ub > lb");
  switch (m.out) {
    case Out::One: if (q != 1) return fail("pinn_create: the Burgers problems need 1 network output (u)"); break;
    case Out::Two: if (q != 2) return fail("pinn_create: the Schrodinger problem needs 2 network outputs (u, v)"); break;
    case Out::QPlus1: if (q < 2) return fail("pinn_create: the discrete-time model needs q+1 >= 2 outputs"); break;
    case Out::Q: if (q < 1) return fail("pinn_create: the discrete-time identification model needs q >= 1 outputs"); break;
  }
  if (world > 1 && !nccl_uid) return fail("pinn_create: world > 1 needs an ncclUniqueId");

  // the specialised DMMA kernels run their model's BASELINE net; any other layer list runs on the generic kernel
  const std::vector<int> L(layers, layers + n_layers);
  const char* fg = getenv("PINN_FORCE_GENERIC");
  const bool force = fg && fg[0] == '1';
  Kernel kernel = m.kernel;
  if (kernel == Kernel::Schrodinger && (force || !is_nls_net(L))) kernel = Kernel::Generic;
  if (kernel == Kernel::BurgersV2) {
    const char* kv = getenv("PINN_BURGERS_KERNEL");
    if (force || !is_burgers_net(L)) kernel = Kernel::Generic;
    else if (kv && (!strcmp(kv, "v1") || !strcmp(kv, "1"))) kernel = Kernel::BurgersV1;
  }

  pinn_t* h = new pinn_t();
  h->pde = pde_id; h->device = device; h->rank = rank; h->world = world < 1 ? 1 : world;
  h->layers = L;
  for (int c = 0; c < 3; c++) { h->lb[c] = lo[c]; h->ub[c] = hi[c]; }
  h->kernel = kernel;
  h->P_net = 0;
  for (int l = 0; l + 1 < n_layers; l++) h->P_net += layers[l] * layers[l + 1] + layers[l + 1];
  h->P = h->P_net + m.n_lambda;

#define CREATE_TRY(expr)                                                                          \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) {                                                                      \
      fail(std::string(#expr) + ": " + cudaGetErrorString(_e));                                   \
      pinn_destroy(h);                                                                            \
      return -1;                                                                                  \
    }                                                                                             \
  } while (0)
  CREATE_TRY(cudaSetDevice(device));
  cudaDeviceProp prop;
  CREATE_TRY(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    fail(std::string("pinn_create: device '") + prop.name + "' is not sm_90 (Hopper); this library is built for sm_90a only");
    pinn_destroy(h);
    return -1;
  }
  h->n_sm = prop.multiProcessorCount;
  CREATE_TRY(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  CREATE_TRY(cudaEventCreate(&h->ev0));
  CREATE_TRY(cudaEventCreate(&h->ev1));
  h->w_cap = ((h->P + 3 + 63) / 64) * 64 + 64;
  if (h->w_cap < pinn::burgers::WPAD) h->w_cap = pinn::burgers::WPAD;
  if (h->w_cap < pinn::nls::WPAD + 64) h->w_cap = pinn::nls::WPAD + 64;
  CREATE_TRY(cudaMalloc((void**)&h->d_w, h->w_cap * 8));
  CREATE_TRY(cudaMemset(h->d_w, 0, h->w_cap * 8));
  CREATE_TRY(cudaMalloc((void**)&h->d_R, h->w_cap * 8));
  CREATE_TRY(cudaMemset(h->d_R, 0, h->w_cap * 8));
  CREATE_TRY(cudaMalloc((void**)&h->d_m, h->w_cap * 8));
  CREATE_TRY(cudaMalloc((void**)&h->d_v, h->w_cap * 8));
  CREATE_TRY(cudaMemset(h->d_m, 0, h->w_cap * 8));
  CREATE_TRY(cudaMemset(h->d_v, 0, h->w_cap * 8));
  CREATE_TRY(cudaMalloc((void**)&h->d_step, 16));
  CREATE_TRY(cudaMemset(h->d_step, 0, 16));
  CREATE_TRY(cudaMalloc((void**)&h->d_loss_ring, LOSS_RING * 8));
  CREATE_TRY(cudaMemset(h->d_loss_ring, 0, LOSS_RING * 8));
  switch (h->kernel) {
    case Kernel::BurgersV2:
      h->n_cta = h->n_sm;
      h->pstride = pinn::burgers::PSTRIDE;
      CREATE_TRY(cudaFuncSetAttribute(pinn::burgers2::fused_loss_grad, cudaFuncAttributeMaxDynamicSharedMemorySize, pinn::burgers2::SMEM_BYTES));
      break;
    case Kernel::BurgersV1:
      h->n_cta = h->n_sm;
      h->pstride = pinn::burgers::PSTRIDE;
      CREATE_TRY(cudaFuncSetAttribute(pinn::burgers::fused_loss_grad, cudaFuncAttributeMaxDynamicSharedMemorySize, pinn::burgers::SMEM_BYTES));
      break;
    case Kernel::Schrodinger:
      h->n_cta = pinn::nls::grid_size(h->n_sm);
      h->pstride = pinn::nls::PSTRIDE;
      CREATE_TRY(cudaFuncSetAttribute(pinn::nls::fused_loss_grad, cudaFuncAttributeMaxDynamicSharedMemorySize, pinn::nls::SMEM_BYTES));
      break;
    case Kernel::Generic:
    case Kernel::NavierStokes:
      h->n_cta = (h->kernel == Kernel::Generic ? 2 : 1) * h->n_sm;     // CTAs of 256 threads: two per SM, or one (Navier-Stokes)
      h->pstride = ((h->P_net + 8 + 15) / 16) * 16;
      break;
  }
  CREATE_TRY(cudaMalloc((void**)&h->d_partials, (size_t)h->n_cta * h->pstride * 8));
  CREATE_TRY(cudaMemset(h->d_partials, 0, (size_t)h->n_cta * h->pstride * 8));
  if (h->world > 1) {
    std::string why;
    if (!g_nccl.load(why)) { fail(why); pinn_destroy(h); return -1; }
    ncclUniqueId id;
    memcpy(&id, nccl_uid, 128);
    int rc = g_nccl.CommInitRank(&h->comm, h->world, id, h->rank);
    if (rc != 0) { fail(std::string("ncclCommInitRank: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "error")); pinn_destroy(h); return -1; }
  }
  { std::lock_guard<std::mutex> lk(g_live_mu); g_live.push_back(h); }
  *out = h;
  return 0;
}

int pinn_destroy(pinn_t* h) {
  if (!h) return 0;
  {
    std::lock_guard<std::mutex> lk(g_live_mu);
    for (size_t i = 0; i < g_live.size(); i++)
      if (g_live[i] == h) { g_live.erase(g_live.begin() + i); break; }
  }
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  for (int r = 0; r < pinn::P2P_MAX; r++) if (h->peer_base[r]) cudaIpcCloseMemHandle(h->peer_base[r]);
  if (h->d_xchg) cudaFree(h->d_xchg);
  if (h->d_p2p_err) cudaFree(h->d_p2p_err);
  if (h->d_xseq) cudaFree(h->d_xseq);
  if (h->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(h->comm);
  double* bufs[] = {h->d_w, h->d_R, h->d_partials, h->d_m, h->d_v, h->d_loss_ring, h->d_x, h->d_t, h->d_u, h->d_irk,
                    h->d_px, h->d_pout, h->d_pscr, h->d_nsX, h->d_src, h->d_rad};
  for (double* b : bufs) if (b) cudaFree(b);
  if (h->d_step) cudaFree(h->d_step);
  h->scratch.release();
  h->lbfgs.release();
  for (cudaEvent_t e : h->events) cudaEventDestroy(e);
  if (h->d_flush) cudaFree(h->d_flush);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return 0;
}

int64_t pinn_num_params(const pinn_t* h) { return h ? h->P : -1; }

int pinn_set_pde_params(pinn_t* h, const double* p, int n) {
  if (!h) return fail("null handle");
  switch (h->pde) {
    case PINN_BURGERS_INF:
      if (n != 1 || !p) return fail("pinn_set_pde_params: BURGERS_INF takes exactly one parameter (nu)");
      h->nu = p[0];
      return 0;
    case PINN_BURGERS_DISC:
      if (n != 2 || !p) return fail("pinn_set_pde_params: BURGERS_DISC takes [nu, dt]");
      h->nu = p[0]; h->dt = p[1];
      return 0;
    case PINN_BURGERS_IDE_DISC:
    case PINN_KDV_IDE_DISC:
      if (n != 1 || !p) return fail("pinn_set_pde_params: the discrete-time identification models take [dt]");
      h->dt = p[0];
      return 0;
    case PINN_AC_DISC:
      if (n != 3 || !p) return fail("pinn_set_pde_params: AC_DISC takes [dt, d, k]");
      h->dt = p[0]; h->nu = p[1]; h->kc = p[2];
      return 0;
  }
  if (n != 0) return fail("pinn_set_pde_params: this PDE takes no constants");
  return 0;
}

int pinn_get_params(pinn_t* h, double* p, int n) {
  if (!h || !p) return fail("pinn_get_params: null argument");
  switch (h->pde) {
    case PINN_BURGERS_INF:
      if (n != 1) return fail("pinn_get_params: BURGERS_INF has one parameter (nu)");
      p[0] = h->nu;                                   // inf_cont_burgers.py:92-93
      return 0;
    case PINN_BURGERS_IDE:
    case PINN_BURGERS_IDE_DISC:
    case PINN_KDV_IDE_DISC: {
      if (n != 2) return fail("pinn_get_params: identification has two parameters (lambda_1, exp(lambda_2))");
      CUDA_TRY(cudaSetDevice(h->device));
      double lam[2];
      CUDA_TRY(cudaMemcpyAsync(lam, h->d_w + h->P_net, 16, cudaMemcpyDeviceToHost, h->stream));
      CUDA_TRY(cudaStreamSynchronize(h->stream));
      p[0] = lam[0]; p[1] = std::exp(lam[1]);         // ide_cont_burgers.py:109-114, ide_disc_burgers.py:138-143
      return 0;
    }
    case PINN_NS_IDE:
    case PINN_POLY_IDE:
      if (n != 2) return fail(h->pde == PINN_NS_IDE ? "pinn_get_params: NS_IDE has two parameters (lambda_1, lambda_2)"
                                                    : "pinn_get_params: POLY_IDE has two parameters (the raw lambda_1, lambda_2)");
      CUDA_TRY(cudaSetDevice(h->device));
      CUDA_TRY(cudaMemcpyAsync(p, h->d_w + h->P_net, 16, cudaMemcpyDeviceToHost, h->stream));
      CUDA_TRY(cudaStreamSynchronize(h->stream));
      return 0;
    case PINN_BURGERS_DISC:
      if (n != 2) return fail("pinn_get_params: BURGERS_DISC has two constants (nu, dt)");
      p[0] = h->nu; p[1] = h->dt;
      return 0;
    case PINN_AC_DISC:
      if (n != 3) return fail("pinn_get_params: AC_DISC has three constants (dt, d, k)");
      p[0] = h->dt; p[1] = h->nu; p[2] = h->kc;
      return 0;
  }
  if (n != 0) return fail("pinn_get_params: this PDE has no parameters");
  return 0;
}

int pinn_set_irk(pinn_t* h, const double* irk, int q) {
  if (!h || !irk) return fail("pinn_set_irk: null argument");
  if (!model(h).irk) return fail("pinn_set_irk: only the discrete-time models have stage matrices");
  const bool idd = model(h).out == Out::Q;                         // identification: a net [1, ..., q]
  if (!idd && q + 1 != h->layers.back()) return fail("pinn_set_irk: q+1 must equal the network's output width");
  if (idd && q != h->layers.back()) return fail("pinn_set_irk: q must equal the network's output width");
  const size_t n_rows = idd ? (size_t)2 * q : (size_t)q + 1;      // identification: [M_0 ; M_1], each q x q
  CUDA_TRY(cudaSetDevice(h->device));
  if (h->d_irk) cudaFree(h->d_irk);
  h->d_irk = nullptr;
  CUDA_TRY(cudaMalloc((void**)&h->d_irk, n_rows * q * 8));
  CUDA_TRY(cudaMemcpy(h->d_irk, irk, n_rows * q * 8, cudaMemcpyHostToDevice));
  h->irk_q = q;
  return 0;
}

int pinn_set_collocation(pinn_t* h, const double* x, const double* t, int64_t n, int64_t n_global) {
  if (!h) return fail("null handle");
  if (model(h).residual == Res::Data)
    return fail("pinn_set_collocation: identification uses the data points as residual points");
  if (model(h).residual == Res::None)
    return fail("pinn_set_collocation: the discrete-time models have no collocation set (snapshot / boundary points only)");
  if (n < 0 || (n > 0 && (!x || !t))) return fail("pinn_set_collocation: bad arguments");
  if (n_global < n) return fail("pinn_set_collocation: n_global < n");
  CUDA_TRY(cudaSetDevice(h->device));
  if (ensure_points(h, h->n_aux, n)) return -1;
  if (n) {
    // straight from the caller's buffer into the collocation region (truly asynchronous when it is pinned)
    CUDA_TRY(cudaMemcpyAsync(h->d_x + h->dcap, x, n * 8, cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(cudaMemcpyAsync(h->d_t + h->dcap, t, n * 8, cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(cudaStreamSynchronize(h->stream));   // the buffers are only borrowed for the call
  }
  h->n_c = n; h->n_c_global = n_global;
  h->map_x = h->map_t = nullptr;
  h->h_src.clear();                               // POLY_INF: new residual points, an array source is 0 until set again
  return fill_source(h);                          // ... and a table follows them
}

int pinn_draw_collocation(pinn_t* h, uint64_t seed, uint64_t draw, int64_t first, int64_t n, int64_t n_global) {
  if (!h) return fail("null handle");
  if (model(h).residual == Res::Data)
    return fail("pinn_draw_collocation: identification uses the data points as residual points");
  if (model(h).residual == Res::None)
    return fail("pinn_draw_collocation: the discrete-time models have no collocation set (snapshot / boundary points only)");
  if (n_global < 1 || n_global > (1LL << 53)) return fail("pinn_draw_collocation: n_global must be in 1..2^53");
  if (first < 0 || n < 0 || first > n_global || n > n_global - first)
    return fail("pinn_draw_collocation: the rows [first, first + n) must lie in [0, n_global)");
  CUDA_TRY(cudaSetDevice(h->device));
  if (ensure_points(h, h->n_aux, n)) return -1;
  if (n) {
    pinn::lhs::Args a{};
    a.x = h->d_x + h->dcap; a.t = h->d_t + h->dcap;
    a.seed = seed; a.draw = draw; a.first = (uint64_t)first; a.n = (uint64_t)n; a.n_global = (uint64_t)n_global;
    a.lb0 = h->lb[0]; a.lb1 = h->lb[1]; a.dx0 = h->ub[0] - h->lb[0]; a.dx1 = h->ub[1] - h->lb[1];
    a.m = pinn::lhs::half_bits((uint64_t)n_global);
    const long long blocks = (n + pinn::lhs::THREADS - 1) / pinn::lhs::THREADS;
    const int grid = (int)(blocks < 8LL * h->n_sm ? blocks : 8LL * h->n_sm);     // one wave of 256-thread blocks, grid-stride beyond
    pinn::lhs::draw_kernel<<<grid, pinn::lhs::THREADS, 0, h->stream>>>(a);
    CUDA_TRY(cudaGetLastError());
    h->launches++;
  }
  h->n_c = n; h->n_c_global = n_global;
  h->map_x = h->map_t = nullptr;
  h->h_src.clear();                               // POLY_INF: new residual points, an array source is 0 until set again
  return fill_source(h);                          // ... and a table follows them
}

static int launch_forward_generic(pinn_t* h, const double* dx, const double* dt, int64_t n, int in_dim, int ns);

int pinn_draw_collocation_rad(pinn_t* h, uint64_t seed, uint64_t draw, int64_t n_pool, int64_t n, int k, double c) {
  if (!h) return fail("null handle");
  const Model& m = model(h);
  if (m.residual == Res::Data)
    return fail("pinn_draw_collocation_rad: identification uses the data points as residual points");
  if (m.residual == Res::None)
    return fail("pinn_draw_collocation_rad: the discrete-time models have no collocation set (snapshot / boundary points only)");
  if (m.poly && h->poly.n == 0)
    return fail("pinn_draw_collocation_rad: POLY_INF has no residual spec to weight the pool by (call pinn_set_residual first)");
  if (m.poly && !h->h_src.empty())
    return fail("pinn_draw_collocation_rad: POLY_INF's source is an array of values at the stored points, which says nothing about "
                "a pool drawn on the device; give it as a table the device evaluates (pinn_set_source_terms)");
  if (h->world > 1)
    return fail("pinn_draw_collocation_rad: runs on one GPU (world must be 1): the weights are normalised over the whole pool");
  if (k < 0 || k > 4) return fail("pinn_draw_collocation_rad: k must be in 0..4");
  if (!(c >= 0.0 && c <= pinn::rad::MAX_C)) return fail("pinn_draw_collocation_rad: c must be finite and in [0, 1024]");
  if (n_pool < 1 || n_pool > pinn::rad::MAX_POOL) return fail("pinn_draw_collocation_rad: n_pool must be in 1..2^29");
  if (n < 0) return fail("pinn_draw_collocation_rad: n must be >= 0");
  CUDA_TRY(cudaSetDevice(h->device));
  if (n) {
    using namespace pinn;
    const long long blocks = (n_pool + rad::THREADS - 1) / rad::THREADS;
    const int grid = (int)(blocks < rad::MAX_BLOCKS ? blocks : rad::MAX_BLOCKS);
    if (ensure(&h->d_rad, &h->rad_cap, 4 * n_pool + 2 * rad::MAX_BLOCKS)) return -1;
    if (ensure_points(h, h->n_aux, n)) return -1;
    double* px = h->d_rad;
    double* pt = px + n_pool;
    // the pool: what pinn_draw_collocation(seed, draw, 0, n_pool, n_pool) stores
    lhs::Args l{};
    l.x = px; l.t = pt;
    l.seed = seed; l.draw = draw; l.first = 0; l.n = (uint64_t)n_pool; l.n_global = (uint64_t)n_pool;
    l.lb0 = h->lb[0]; l.lb1 = h->lb[1]; l.dx0 = h->ub[0] - h->lb[0]; l.dx1 = h->ub[1] - h->lb[1];
    l.m = lhs::half_bits((uint64_t)n_pool);
    const int lgrid = (int)(blocks < 8LL * h->n_sm ? blocks : 8LL * h->n_sm);
    lhs::draw_kernel<<<lgrid, lhs::THREADS, 0, h->stream>>>(l);
    CUDA_TRY(cudaGetLastError());
    h->launches++;
    // its probe streams from the weights after every step already enqueued, as pinn_residual forms them
    if (launch_forward_generic(h, px, pt, n_pool, 2, 4)) return -1;
    rad::Args a{};
    a.streams = h->d_pout; a.px = px; a.pt = pt;
    a.a = pt + n_pool;
    a.lp = reinterpret_cast<uint64_t*>(a.a + n_pool);
    a.bmax = a.a + 2 * n_pool;
    a.bsum = reinterpret_cast<uint64_t*>(a.bmax + rad::MAX_BLOCKS);
    a.x = h->d_x + h->dcap; a.t = h->d_t + h->dcap;
    a.n_pool = (uint64_t)n_pool; a.seg = (uint64_t)((n_pool + grid - 1) / grid); a.n = (uint64_t)n;
    a.seed = seed; a.draw = draw; a.grid = grid;
    a.nls = h->pde == PINN_NLS_INF; a.k = k; a.nu = h->nu; a.c = c;
    if (m.poly) {
      // f of the residual spec minus the table's s at every pool point (source_terms.cuh)
      source::PoolArgs pa{a, h->poly, h->src_tab};
      source::pool_head_kernel<<<grid, source::THREADS, 0, h->stream>>>(pa);
    } else {
      rad::head_kernel<<<grid, rad::THREADS, 0, h->stream>>>(a);
    }
    CUDA_TRY(cudaGetLastError());
    rad::quantise_kernel<<<grid, rad::THREADS, 0, h->stream>>>(a);
    CUDA_TRY(cudaGetLastError());
    const long long rows = (n + rad::THREADS - 1) / rad::THREADS;
    rad::pick_kernel<<<(int)(rows < 8LL * h->n_sm ? rows : 8LL * h->n_sm), rad::THREADS, 0, h->stream>>>(a);
    CUDA_TRY(cudaGetLastError());
    h->launches += 3;
  }
  h->n_c = n; h->n_c_global = n;
  h->map_x = h->map_t = nullptr;
  return fill_source(h);                          // POLY_INF: the table follows the new set
}

int pinn_get_collocation(pinn_t* h, double* x, double* t, int64_t n) {
  if (!h) return fail("null handle");
  if (model(h).residual != Res::Colloc) return fail("pinn_get_collocation: this model has no collocation set");
  if (n != h->n_c)
    return fail("pinn_get_collocation: the output buffers hold " + std::to_string(n) + " rows but " + std::to_string(h->n_c) +
                " collocation points are stored (pinn_num_residual_points)");
  if (n == 0) return 0;
  if (!x || !t) return fail("pinn_get_collocation: null argument");
  CUDA_TRY(cudaSetDevice(h->device));
  // a mapped batch is read through its device alias: the copy is ordered after the launches that still read it
  const double* sx = h->map_x ? h->map_x : h->d_x + h->dcap;
  const double* st = h->map_t ? h->map_t : h->d_t + h->dcap;
  CUDA_TRY(cudaMemcpyAsync(x, sx, (size_t)n * 8, cudaMemcpyDefault, h->stream));
  CUDA_TRY(cudaMemcpyAsync(t, st, (size_t)n * 8, cudaMemcpyDefault, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  return 0;
}

int pinn_set_collocation_mapped(pinn_t* h, const double* x_pinned, const double* t_pinned, int64_t n, int64_t n_global) {
  if (!h) return fail("null handle");
  if ((h->kernel != Kernel::BurgersV2 && h->kernel != Kernel::BurgersV1) || model(h).residual != Res::Colloc)
    return fail("pinn_set_collocation_mapped: zero-copy collocation is implemented for the fused Burgers inference kernel only");
  if (n <= 0 || !x_pinned || !t_pinned || n_global < n) return fail("pinn_set_collocation_mapped: bad arguments");
  CUDA_TRY(cudaSetDevice(h->device));
  void *dx = nullptr, *dt = nullptr;
  if (cudaHostGetDevicePointer(&dx, (void*)x_pinned, 0) != cudaSuccess || cudaHostGetDevicePointer(&dt, (void*)t_pinned, 0) != cudaSuccess) {
    cudaGetLastError();
    return fail("pinn_set_collocation_mapped: the buffers must be pinned host memory (pinn_host_alloc / cudaHostAlloc)");
  }
  if (ensure_points(h, h->n_aux, 0)) return -1;
  // the kernel that is about to be enqueued reads the caller's buffers: they must stay valid and unchanged until the
  // next synchronising call (pinn_adam_step with a loss pointer, pinn_loss_grad, pinn_sync)
  h->map_x = (const double*)dx; h->map_t = (const double*)dt;
  h->n_c = n; h->n_c_global = n_global;
  return 0;
}

int pinn_set_data(pinn_t* h, const double* X, int64_t n, int in_dim, const double* u, int out_dim, double weight) {
  if (!h) return fail("null handle");
  if (n < 0 || (n > 0 && (!X || !u))) return fail("pinn_set_data: bad arguments");
  const Model& m = model(h);
  if (m.in_dim == 3) {
    // X (n,3) = (x, y, t), u (n,2) = (u, v); these points also carry the residual term
    if (in_dim != 3 || out_dim != 2) return fail("pinn_set_data: the Navier-Stokes model takes X (n,3) = (x, y, t) and u (n,2) = (u, v)");
    CUDA_TRY(cudaSetDevice(h->device));
    if (upload(h, &h->d_nsX, &h->nsx_cap, X, 3 * n) || upload(h, &h->d_u, &h->u_cap, u, 2 * n)) return -1;
    h->n_d = n; h->d_out_dim = 2; h->data_weight = weight;
    return 0;
  }
  if (in_dim != 1 && in_dim != 2) return fail("pinn_set_data: in_dim must be 1 (broadcast quirk) or 2");
  if (m.snapshots) return pinn_set_snapshot(h, 0, X, n, u);
  if (m.in_dim == 1) {
    // x_0 (n,1) and u_0 (n,1): the snapshot the q stages are fitted to (inf_disc_burgers.py:98-101; u_0 broadcasts)
    if (in_dim != 1 || out_dim != 1) return fail("pinn_set_data: the discrete-time model takes x_0 (n,1) and u_0 (n,1)");
    CUDA_TRY(cudaSetDevice(h->device));
    h->h_x0.assign(X, X + n);
    if (upload(h, &h->d_u, &h->u_cap, u, n)) return -1;
    h->n_d = n; h->d_out_dim = 1; h->data_weight = weight;
    return assemble_points(h);
  }
  if (out_dim != h->layers.back()) return fail("pinn_set_data: out_dim does not match the network head");
  CUDA_TRY(cudaSetDevice(h->device));
  // the Schrodinger block is re-assembled with the boundary pairs, so it keeps host copies; the others are staged directly
  std::vector<double>& x = m.boundary ? h->h_icx : h->stage_x;
  std::vector<double>& t = m.boundary ? h->h_ict : h->stage_t;
  x.resize(n); t.resize(n);
  for (int64_t i = 0; i < n; i++) {
    x[i] = X[i * in_dim];
    t[i] = in_dim == 1 ? X[i] : X[i * in_dim + 1];   // quirk Q1: the (N,1) input is broadcast by the Lambda, t := x
  }
  if (upload(h, &h->d_u, &h->u_cap, u, n * out_dim)) return -1;
  h->n_d = n; h->d_out_dim = out_dim; h->data_weight = weight;
  if (m.boundary) return assemble_points(h);
  // shrinking/growing the data set moves its right-aligned start; the collocation region is untouched
  if (upload_points(h)) return -1;
  if (m.residual != Res::Data) return 0;
  h->h_src.clear();                                // new residual points: an array source is 0 until set again
  return fill_source(h);                           // ... and a table follows them
}

int pinn_set_residual(pinn_t* h, int n_terms, const double* coef, const int* kind, const int* exps) {
  if (!h) return fail("null handle");
  if (!model(h).poly) return fail("pinn_set_residual: only the polynomial residual models (POLY_INF, POLY_IDE) take a residual spec");
  if (n_terms < 1 || n_terms > pinn::generic::POLY_MAXT)
    return fail("pinn_set_residual: n_terms = " + std::to_string(n_terms) + " is outside 1..16");
  if (!coef || !kind || !exps) return fail("pinn_set_residual: null argument");
  pinn::generic::PolySpec s{};
  s.n = n_terms;
  for (int k = 0; k < n_terms; k++) {
    const std::string term = "pinn_set_residual: term " + std::to_string(k) + ": ";
    if (!std::isfinite(coef[k])) return fail(term + "the coefficient is not finite");
    if (kind[k] < 0 || kind[k] > 4) return fail(term + "kind " + std::to_string(kind[k]) + " is outside 0..4 (1, l1, l2, e^l1, e^l2)");
    if (kind[k] != 0 && model(h).n_lambda == 0)
      return fail(term + "POLY_INF has no trainable lambdas: every kind must be 0 (use POLY_IDE for l1, l2, e^l1, e^l2)");
    int code = kind[k], any = 0;
    for (int j = 0; j < 4; j++) {
      const int e = exps[4 * k + j];
      if (e < 0 || e > 3) return fail(term + "exponent " + std::to_string(e) + " of stream " + std::to_string(j) + " is outside 0..3");
      code |= e << (3 + 2 * j);
      any |= e;
    }
    if (!any) return fail(term + "all four exponents are 0 (a constant term belongs in the source)");
    s.code[k] = code;
    s.coef[k] = coef[k];
  }
  h->poly = s;
  return 0;
}

int pinn_set_source(pinn_t* h, const double* src, int64_t n) {
  if (!h) return fail("null handle");
  if (!model(h).poly) return fail("pinn_set_source: only the polynomial residual models (POLY_INF, POLY_IDE) take a source");
  const int64_t want = pinn_num_residual_points(h);
  if (n != want)
    return fail("pinn_set_source: " + std::to_string(n) + " values given but " + std::to_string(want) +
                " residual points are stored (pinn_num_residual_points)");
  if (n > 0 && !src) return fail("pinn_set_source: null argument");
  CUDA_TRY(cudaSetDevice(h->device));
  if (upload(h, &h->d_src, &h->src_cap, src, n)) return -1;
  h->h_src.assign(src, src + n);
  h->src_tab.n = 0;                               // an array replaces a table
  return 0;
}

int pinn_set_source_terms(pinn_t* h, int n_terms, const int* form, const double* par) {
  namespace S = pinn::source;
  if (!h) return fail("null handle");
  if (!model(h).poly)
    return fail("pinn_set_source_terms: only the polynomial residual models (POLY_INF, POLY_IDE) take a source");
  if (n_terms < 0 || n_terms > S::MAXT)
    return fail("pinn_set_source_terms: n_terms = " + std::to_string(n_terms) + " is outside 0..16");
  if (n_terms > 0 && (!form || !par)) return fail("pinn_set_source_terms: null argument");
  static const char* const PAR[S::NPAR] = {"a", "omega", "phi", "nu", "psi", "alpha", "gamma", "beta", "delta"};
  S::Table tb{};
  tb.n = n_terms;
  for (int k = 0; k < n_terms; k++) {
    const std::string term = "pinn_set_source_terms: term " + std::to_string(k) + ": ";
    const int f = form[k];
    if (f < 0 || f > 255) return fail(term + "form " + std::to_string(f) + " is outside 0..255 (p | q << 2 | X kind << 4 | T kind << 6)");
    if (((f >> 4) & 3) == 3) return fail(term + "X kind 3 is outside 0..2 (1, sin, cos)");
    if (((f >> 6) & 3) == 3) return fail(term + "T kind 3 is outside 0..2 (1, sin, cos)");
    tb.form[k] = f;
    for (int j = 0; j < S::NPAR; j++) {
      const double v = par[S::NPAR * k + j];
      if (!std::isfinite(v)) return fail(term + "parameter " + PAR[j] + " is not finite");
      tb.par[S::NPAR * k + j] = v;
    }
  }
  CUDA_TRY(cudaSetDevice(h->device));
  h->h_src.clear();                               // a table replaces an array
  h->src_tab = tb;
  return fill_source(h);
}

int pinn_get_source(pinn_t* h, double* s, int64_t n) {
  if (!h) return fail("null handle");
  if (!model(h).poly) return fail("pinn_get_source: only the polynomial residual models (POLY_INF, POLY_IDE) have a source");
  const int64_t want = pinn_num_residual_points(h);
  if (n != want)
    return fail("pinn_get_source: the output buffer holds " + std::to_string(n) + " values but " + std::to_string(want) +
                " residual points are stored (pinn_num_residual_points)");
  if (n == 0) return 0;
  if (!s) return fail("pinn_get_source: null argument");
  CUDA_TRY(cudaSetDevice(h->device));
  if (h->src_tab.n) CUDA_TRY(cudaMemcpyAsync(s, h->d_src, (size_t)n * 8, cudaMemcpyDeviceToHost, h->stream));
  else if (!h->h_src.empty()) memcpy(s, h->h_src.data(), (size_t)n * 8);
  else for (int64_t i = 0; i < n; i++) s[i] = 0.0;
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  return 0;
}

int pinn_set_snapshot(pinn_t* h, int which, const double* x, int64_t n, const double* u) {
  if (!h) return fail("null handle");
  if (!model(h).snapshots) return fail("pinn_set_snapshot: only the discrete-time identification models have two snapshots");
  if ((which != 0 && which != 1) || n < 0 || (n > 0 && (!x || !u))) return fail("pinn_set_snapshot: bad arguments");
  CUDA_TRY(cudaSetDevice(h->device));
  // host copies of both snapshots: the device blocks [x_0 | x_1] and [u_0 | u_1] are re-assembled whenever one changes
  (which == 0 ? h->h_x0 : h->h_tb).assign(x, x + n);
  (which == 0 ? h->h_u0 : h->h_u1).assign(u, u + n);
  h->n_d = (long long)h->h_x0.size();
  h->n_b = (long long)h->h_tb.size();
  h->d_out_dim = 1; h->data_weight = 1.0;
  std::vector<double> u01(h->h_u0);
  u01.insert(u01.end(), h->h_u1.begin(), h->h_u1.end());
  if (upload(h, &h->d_u, &h->u_cap, u01.data(), (long long)u01.size())) return -1;
  return assemble_points(h);
}

int pinn_set_boundary(pinn_t* h, const double* tb, int64_t n_b) {
  if (!h) return fail("null handle");
  if (h->pde == PINN_AC_DISC) return fail("pinn_set_boundary: the Allen-Cahn model's periodic pair is (lb, ub) of pinn_create");
  if (!model(h).boundary) return fail("pinn_set_boundary: only the NLS and discrete-time inference problems have a boundary term");
  if (n_b < 0 || (n_b > 0 && !tb)) return fail("pinn_set_boundary: bad arguments");
  h->h_tb.assign(tb, tb + n_b);
  h->n_b = n_b;
  CUDA_TRY(cudaSetDevice(h->device));
  return assemble_points(h);
}

int pinn_set_weights(pinn_t* h, const double* w, int64_t n) {
  if (!h || !w) return fail("pinn_set_weights: null argument");
  if (n != h->P) return fail("pinn_set_weights: expected " + std::to_string(h->P) + " values, got " + std::to_string(n));
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaMemcpyAsync(h->d_w, w, n * 8, cudaMemcpyHostToDevice, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  return 0;
}

int pinn_get_weights(pinn_t* h, double* w, int64_t n) {
  if (!h || !w) return fail("pinn_get_weights: null argument");
  if (n != h->P) return fail("pinn_get_weights: expected " + std::to_string(h->P) + " values, got " + std::to_string(n));
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaMemcpyAsync(w, h->d_w, n * 8, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  return 0;
}

int pinn_loss_grad(pinn_t* h, const double* w_or_null, double* loss_out, double* grad_out_or_null,
                   double* parts_out_or_null) {
  if (!h) return fail("null handle");
  CUDA_TRY(cudaSetDevice(h->device));
  if (w_or_null) CUDA_TRY(cudaMemcpyAsync(h->d_w, w_or_null, h->P * 8, cudaMemcpyHostToDevice, h->stream));
  if (launch_eval(h, nullptr)) return -1;
  double parts[3];
  CUDA_TRY(cudaMemcpyAsync(parts, h->d_R + h->P, 24, cudaMemcpyDeviceToHost, h->stream));
  if (grad_out_or_null) CUDA_TRY(cudaMemcpyAsync(grad_out_or_null, h->d_R, h->P * 8, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  if (check_p2p(h)) return -1;
  if (loss_out) *loss_out = parts[0] + parts[1] + parts[2];
  if (parts_out_or_null) { parts_out_or_null[0] = parts[0]; parts_out_or_null[1] = parts[1]; parts_out_or_null[2] = parts[2]; }
  return 0;
}

int pinn_adam_step(pinn_t* h, double lr, double b1, double b2, double eps, double* loss_out_or_null) {
  if (!h) return fail("null handle");
  CUDA_TRY(cudaSetDevice(h->device));
  // fused kernel, then the tail: ONE more kernel on a single GPU (reduce + Adam) and with the NVLink push exchange
  // (reduce + exchange + Adam); reduce + ncclAllReduce + Adam on the NCCL path
  const AdamArgs ad{lr, b1, b2, eps};
  if (launch_eval(h, nullptr, false, &ad)) return -1;
  h->adam_steps++;
  if (loss_out_or_null) {
    CUDA_TRY(cudaMemcpyAsync(loss_out_or_null, h->d_loss_ring + ((h->adam_steps - 1) % LOSS_RING), 8, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(cudaStreamSynchronize(h->stream));
    if (check_p2p(h)) return -1;
  }
  return 0;
}

int pinn_adam_steps(pinn_t* h, int n, double lr, double b1, double b2, double eps) {
  if (!h) return fail("null handle");
  if (n < 0) return fail("pinn_adam_steps: n < 0");
  CUDA_TRY(cudaSetDevice(h->device));
  const AdamArgs ad{lr, b1, b2, eps};
  for (int i = 0; i < n; i++) {
    if (launch_eval(h, nullptr, false, &ad)) return -1;
    h->adam_steps++;
  }
  return 0;
}

int pinn_adam_reset(pinn_t* h) {
  if (!h) return fail("null handle");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaMemsetAsync(h->d_m, 0, h->w_cap * 8, h->stream));
  CUDA_TRY(cudaMemsetAsync(h->d_v, 0, h->w_cap * 8, h->stream));
  CUDA_TRY(cudaMemsetAsync(h->d_step, 0, 16, h->stream));
  h->adam_steps = 0;
  return 0;
}

int pinn_last_loss(pinn_t* h, double* loss_out) {
  if (!h || !loss_out) return fail("null argument");
  if (h->adam_steps == 0) return fail("pinn_last_loss: no Adam step has run");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaMemcpyAsync(loss_out, h->d_loss_ring + ((h->adam_steps - 1) % LOSS_RING), 8, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  if (check_p2p(h)) return -1;
  return 0;
}

int pinn_lbfgs(pinn_t* h, int max_iter, double learning_rate, int n_correction, double tol_fun, double tol_x,
               int sync_every, pinn_log_cb log_cb, void* user, int* n_iter_out, int* n_eval_out, int* reason_out,
               double* x_final_or_null) {
  if (!h) return fail("null handle");
  if (n_iter_out) *n_iter_out = 0;
  if (n_eval_out) *n_eval_out = 0;
  if (reason_out) *reason_out = PINN_LBFGS_RUNNING;
  if (max_iter == 0) { h->lb_fhist.clear(); return 0; }             // custom_lbfgs.py:43-44: a run with no evaluation
  if (max_iter < 0) return fail("pinn_lbfgs: max_iter < 0");
  const int P = h->P;
  LbfgsConfig cfg;
  if (lbfgs_config("pinn_lbfgs", P, max_iter, learning_rate, n_correction, tol_fun, tol_x, 0.0, &cfg)) return -1;
  if (sync_every < 1) sync_every = 1;
  CUDA_TRY(cudaSetDevice(h->device));
  DeviceLbfgs& lb = h->lbfgs;
  if (lb.reserve(P, cfg.n_corr, max_iter) || lb.start(h->stream, cfg)) return -1;
  const int* run_flag = &lb.st->status;
  if (launch_eval(h, run_flag)) return -1;      // initial f, g (:65)

  std::vector<double> fh(max_iter + 2);
  std::vector<int> lg(max_iter + 2);
  pinn::LbfgsState st{};
  int reported = 0;
  while (true) {
    for (int b = 0; b < sync_every; b++) {
      if (lb.iterate(h->stream, h->d_w, h->d_R, P, &h->launches)) return -1;
      if (launch_eval(h, run_flag)) return -1;
    }
    CUDA_TRY(cudaMemcpyAsync(&st, lb.st, sizeof(st), cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(cudaMemcpyAsync(fh.data(), lb.f_hist, (size_t)(max_iter + 2) * 8, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(cudaMemcpyAsync(lg.data(), lb.logged, (size_t)(max_iter + 2) * 4, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(cudaStreamSynchronize(h->stream));
    if (check_p2p(h)) return -1;
    const int upto = lbfgs_tested(st);
    for (int it = reported + 1; it <= upto; it++)
      if (lg[it] && log_cb) log_cb(it, fh[it], user);
    if (upto > reported) reported = upto;
    if (st.status != 0) break;
  }
  h->lb_fhist.assign(fh.begin(), fh.begin() + (st.n_eval < (int)fh.size() ? st.n_eval : (int)fh.size()));
  if (n_iter_out) *n_iter_out = st.n_iter;
  if (n_eval_out) *n_eval_out = st.n_eval;
  if (reason_out) *reason_out = st.status;
  if (x_final_or_null) {
    // x after the loop: differs from the model weights only when the loop ended on max_iter (the last update
    // is not evaluated, utils/custom_lbfgs.py:176-182; utils/neuralnetwork.py:131-136 ignores the return).
    const double* src = (st.status == PINN_LBFGS_MAX_ITER) ? lb.x_final : h->d_w;
    CUDA_TRY(cudaMemcpyAsync(x_final_or_null, src, (size_t)P * 8, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(cudaStreamSynchronize(h->stream));
  }
  return 0;
}

int pinn_lbfgs_history(pinn_t* h, double* f_hist_out, int capacity, int* n_out) {
  if (!h || !n_out) return fail("pinn_lbfgs_history: null argument");
  const int n = (int)h->lb_fhist.size();
  *n_out = n;
  if (f_hist_out) {
    if (capacity < n) return fail("pinn_lbfgs_history: buffer too small");
    for (int i = 0; i < n; i++) f_hist_out[i] = h->lb_fhist[i];
  }
  return 0;
}

// generic thread-per-point forward of n >= 1 device points into h->d_pout, [n][ns][no], enqueued on h->stream: interleaved
// X[n][in_dim] in dx (dt == nullptr) or a SoA range (dx, dt)
static int launch_forward_generic(pinn_t* h, const double* dx, const double* dt, int64_t n, int in_dim, int ns) {
  if (ensure(&h->d_pout, &h->pout_cap, n * h->layers.back() * ns)) return -1;
  pinn::NetDesc nd = net_desc(h);
  const int threads = 64;
  const int blocks = (int)((n + threads - 1) / threads);
  int maxw = 0;
  for (int l = 1; l < nd.n_layers; l++) maxw = nd.dims[l] > maxw ? nd.dims[l] : maxw;
  const int o3 = h->pde == PINN_KDV_IDE_DISC ? 1 : 0;        // KdV: the t column block carries u_xxx
  // per-thread activation arrays sized for the widest hidden layer: the 128-wide instantiation for every net that fits
  if (maxw <= pinn::MAXW) {
    if (ns == 1) pinn::mlp_forward_generic<1, pinn::MAXW><<<blocks, threads, 0, h->stream>>>(h->d_w, nd, dx, dt, n, in_dim, h->d_pout, o3);
    else pinn::mlp_forward_generic<4, pinn::MAXW><<<blocks, threads, 0, h->stream>>>(h->d_w, nd, dx, dt, n, in_dim, h->d_pout, o3);
  } else {
    if (ns == 1) pinn::mlp_forward_generic<1, pinn::MAXW_WIDE><<<blocks, threads, 0, h->stream>>>(h->d_w, nd, dx, dt, n, in_dim, h->d_pout, o3);
    else pinn::mlp_forward_generic<4, pinn::MAXW_WIDE><<<blocks, threads, 0, h->stream>>>(h->d_w, nd, dx, dt, n, in_dim, h->d_pout, o3);
  }
  CUDA_TRY(cudaGetLastError());
  h->launches++;
  return 0;
}

// generic thread-per-point forward on host points (X != nullptr) or on a device SoA range (dx, dt)
static int forward_generic(pinn_t* h, const double* X, const double* dx, const double* dt, int64_t n, int in_dim, double* out,
                           int ns) {
  if (!h || !out || (!X && !dx)) return fail("null argument");
  if (n <= 0) return 0;
  if (in_dim != 1 && in_dim != 2) return fail("in_dim must be 1 or 2");
  CUDA_TRY(cudaSetDevice(h->device));
  if (X) {
    if (ensure(&h->d_px, &h->px_cap, n * in_dim)) return -1;
    CUDA_TRY(cudaMemcpyAsync(h->d_px, X, n * in_dim * 8, cudaMemcpyHostToDevice, h->stream));
    dx = h->d_px; dt = nullptr;
  }
  if (launch_forward_generic(h, dx, dt, n, in_dim, ns)) return -1;
  CUDA_TRY(cudaMemcpyAsync(out, h->d_pout, n * h->layers.back() * ns * 8, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  return 0;
}

// NS handles: the probe kernel on host points X (n,3)
static int forward_ns(pinn_t* h, const double* X, int64_t n, int in_dim, double* out, int mode) {
  if (!h || !out || !X) return fail("null argument");
  if (in_dim != 3) return fail("the Navier-Stokes model takes X (n,3) = (x, y, t)");
  if (n <= 0) return 0;
  CUDA_TRY(cudaSetDevice(h->device));
  if (ensure(&h->d_px, &h->px_cap, n * 3)) return -1;
  CUDA_TRY(cudaMemcpyAsync(h->d_px, X, n * 3 * 8, cudaMemcpyHostToDevice, h->stream));
  return ns_probe(h, h->d_px, n, mode, out);
}

int pinn_predict(pinn_t* h, const double* X, int64_t n, int in_dim, double* out) {
  if (h && h->kernel == Kernel::NavierStokes) return forward_ns(h, X, n, in_dim, out, 0);
  return forward_generic(h, X, nullptr, nullptr, n, in_dim, out, 1);
}

int pinn_derivatives(pinn_t* h, const double* X, int64_t n, double* out) {
  if (h && h->kernel == Kernel::NavierStokes) return forward_ns(h, X, n, 3, out, 1);
  return forward_generic(h, X, nullptr, nullptr, n, h ? h->layers[0] : 2, out, 4);
}

int64_t pinn_num_residual_points(const pinn_t* h) {
  if (!h) return -1;
  switch (model(h).residual) {
    case Res::Data: return h->n_d;
    case Res::Colloc: return h->n_c;
    case Res::None: break;
  }
  return 0;
}

int pinn_residual(pinn_t* h, double* f_out, int64_t n_rows) {
  if (!h || !f_out) return fail("null argument");
  const Res res = model(h).residual;
  const bool poly = model(h).poly;
  if (res == Res::None) return fail("pinn_residual: not defined for the discrete-time models");
  if (poly && h->poly.n == 0) return fail("pinn_residual: call pinn_set_residual first (no residual is set)");
  const int64_t n = pinn_num_residual_points(h);
  if (n_rows != n)
    return fail("pinn_residual: the output buffer holds " + std::to_string(n_rows) + " rows but " + std::to_string(n) +
                " residual points are stored (pinn_num_residual_points)");
  if (n == 0) return 0;
  if (h->kernel == Kernel::NavierStokes) {
    CUDA_TRY(cudaSetDevice(h->device));
    return ns_probe(h, h->d_nsX, n, 2, f_out);
  }
  const bool ide = res == Res::Data;
  const long long off = ide ? h->dcap - h->n_d : h->dcap;
  std::vector<double> D(n * 4 * h->layers.back());
  const double* rx = (!ide && h->map_x) ? h->map_x : h->d_x + off;
  const double* rt = (!ide && h->map_t) ? h->map_t : h->d_t + off;
  if (forward_generic(h, nullptr, rx, rt, n, 2, D.data(), 4)) return -1;
  if (h->pde == PINN_NLS_INF) {
    for (int64_t i = 0; i < n; i++) {
      const double* d = &D[i * 8];
      const double u = d[0], v = d[1], ut = d[4], vt = d[5], uxx = d[6], vxx = d[7];
      const double h2 = u * u + v * v;
      f_out[2 * i] = ut + 0.5 * vxx + h2 * v;
      f_out[2 * i + 1] = vt - 0.5 * uxx - h2 * u;
    }
    return 0;
  }
  if (poly) {
    // the kernel head's f, term by term on the host: sum_k c_k kappa_k prod_j v_j^e_kj - s
    std::vector<double> tab_src;
    if (h->src_tab.n) {
      tab_src.resize(n);
      if (pinn_get_source(h, tab_src.data(), n)) return -1;
    }
    const double* src = h->src_tab.n ? tab_src.data() : h->h_src.empty() ? nullptr : h->h_src.data();
    double lam[2] = {0.0, 0.0};
    if (ide) CUDA_TRY(cudaMemcpy(lam, h->d_w + h->P_net, 16, cudaMemcpyDeviceToHost));
    const double kv[5] = {1.0, lam[0], lam[1], std::exp(lam[0]), std::exp(lam[1])};
    for (int64_t i = 0; i < n; i++) {
      const double* d = &D[i * 4];
      double f = 0.0;
      for (int k = 0; k < h->poly.n; k++) {
        const int code = h->poly.code[k];
        double m = h->poly.coef[k];
        for (int j = 0; j < 4; j++)
          for (int e = (code >> (3 + 2 * j)) & 3; e > 0; e--) m *= d[j];
        f += kv[code & 7] * m;
      }
      f_out[i] = src ? f - src[i] : f;
    }
    return 0;
  }
  double l1 = 1.0, kap = h->nu;
  if (ide) {
    double lam[2];
    CUDA_TRY(cudaMemcpy(lam, h->d_w + h->P_net, 16, cudaMemcpyDeviceToHost));
    l1 = lam[0]; kap = std::exp(lam[1]);
  }
  for (int64_t i = 0; i < n; i++) {
    const double* d = &D[i * 4];
    f_out[i] = d[2] + l1 * d[0] * d[1] - kap * d[3];
  }
  return 0;
}

int pinn_sync(pinn_t* h) {
  if (!h) return fail("null handle");
  CUDA_TRY(cudaSetDevice(h->device));
  CUDA_TRY(cudaStreamSynchronize(h->stream));
  return check_p2p(h);
}

int pinn_host_alloc(void** out, int64_t bytes) {
  if (!out || bytes <= 0) return fail("pinn_host_alloc: bad arguments");
  CUDA_TRY(cudaHostAlloc(out, (size_t)bytes, cudaHostAllocDefault));
  return 0;
}
int pinn_host_free(void* p) {
  if (p) CUDA_TRY(cudaFreeHost(p));
  return 0;
}

int pinn_time_loss_grad_kernel(pinn_t* h, int iters, float* ms_total_out) {
  if (!h || !ms_total_out || iters < 1) return fail("pinn_time_loss_grad_kernel: bad arguments");
  CUDA_TRY(cudaSetDevice(h->device));
  const int world = h->world;
  h->world = 1;   // kernel only: no collective inside the timed region
  CUDA_TRY(cudaEventRecord(h->ev0, h->stream));
  int rc = 0;
  for (int i = 0; i < iters && rc == 0; i++) rc = launch_eval(h, nullptr, true);
  h->world = world;
  if (rc) return -1;
  CUDA_TRY(cudaEventRecord(h->ev1, h->stream));
  CUDA_TRY(cudaEventSynchronize(h->ev1));
  CUDA_TRY(cudaEventElapsedTime(ms_total_out, h->ev0, h->ev1));
  return 0;
}

int pinn_event_record(pinn_t* h, int idx) {
  if (!h || idx < 0 || idx >= 65536) return fail("pinn_event_record: bad arguments");
  CUDA_TRY(cudaSetDevice(h->device));
  while ((int)h->events.size() <= idx) {
    cudaEvent_t e;
    CUDA_TRY(cudaEventCreate(&e));
    h->events.push_back(e);
  }
  CUDA_TRY(cudaEventRecord(h->events[idx], h->stream));
  return 0;
}

int pinn_event_elapsed_ms(pinn_t* h, int i, int j, float* ms_out) {
  if (!h || !ms_out || i < 0 || j < 0 || i >= (int)h->events.size() || j >= (int)h->events.size())
    return fail("pinn_event_elapsed_ms: bad arguments");
  CUDA_TRY(cudaEventSynchronize(h->events[j]));
  CUDA_TRY(cudaEventElapsedTime(ms_out, h->events[i], h->events[j]));
  return 0;
}

int pinn_flush_l2(pinn_t* h) {
  if (!h) return fail("null handle");
  CUDA_TRY(cudaSetDevice(h->device));
  if (!h->d_flush) {
    h->flush_bytes = (size_t)128 << 20;   // > 2x the 50 MB L2
    CUDA_TRY(cudaMalloc((void**)&h->d_flush, h->flush_bytes));
  }
  CUDA_TRY(cudaMemsetAsync(h->d_flush, 0, h->flush_bytes, h->stream));
  return 0;
}

int pinn_test_tanh(const double* x, int n, double* y) {
  if (!x || !y || n < 1) return fail("pinn_test_tanh: bad arguments");
  double *dx = nullptr, *dy = nullptr;
  CUDA_TRY(cudaMalloc((void**)&dx, (size_t)n * 8));
  CUDA_TRY(cudaMalloc((void**)&dy, (size_t)n * 8));
  CUDA_TRY(cudaMemcpy(dx, x, (size_t)n * 8, cudaMemcpyHostToDevice));
  pinn::tanh_fast_kernel<<<(n + 255) / 256, 256>>>(dx, n, dy);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpy(y, dy, (size_t)n * 8, cudaMemcpyDeviceToHost));
  cudaFree(dx); cudaFree(dy);
  return 0;
}

int64_t pinn_launch_count(const pinn_t* h) { return h ? h->launches : -1; }

int pinn_kernel_info(pinn_t* h, char* buf, int buflen) {
  if (!h || !buf || buflen < 1) return fail("bad arguments");
  cudaFuncAttributes fa{};
  int smem = 0, threads = 0;
  switch (h->kernel) {
    case Kernel::BurgersV2:
      CUDA_TRY(cudaFuncGetAttributes(&fa, pinn::burgers2::fused_loss_grad));
      smem = pinn::burgers2::SMEM_BYTES; threads = pinn::burgers2::THREADS;
      break;
    case Kernel::BurgersV1:
      CUDA_TRY(cudaFuncGetAttributes(&fa, pinn::burgers::fused_loss_grad));
      smem = pinn::burgers::SMEM_BYTES; threads = pinn::burgers::THREADS;
      break;
    case Kernel::Schrodinger:
      CUDA_TRY(cudaFuncGetAttributes(&fa, pinn::nls::fused_loss_grad));
      smem = pinn::nls::SMEM_BYTES; threads = pinn::nls::THREADS;
      break;
    case Kernel::Generic:
      if (model(h).poly) CUDA_TRY(cudaFuncGetAttributes(&fa, pinn::generic::fused_loss_grad<true>));
      else CUDA_TRY(cudaFuncGetAttributes(&fa, pinn::generic::fused_loss_grad<false>));
      smem = 0; threads = pinn::generic::THREADS;
      break;
    case Kernel::NavierStokes:
      CUDA_TRY(cudaFuncGetAttributes(&fa, pinn::nsid::fused_loss_grad));
      smem = 0; threads = pinn::nsid::THREADS;
      break;
  }
  snprintf(buf, buflen, "{\"grid\": %d, \"block\": %d, \"dyn_smem\": %d, \"regs\": %d, \"local_bytes\": %zu, \"sms\": %d}",
           h->n_cta, threads, smem, fa.numRegs, fa.localSizeBytes, h->n_sm);
  return 0;
}

// -----------------------------------------------------------------------------------------------------------------
// Stand-alone device-resident L-BFGS for ANY objective (utils/custom_lbfgs.py:39 takes an arbitrary `opfunc`): the caller
// evaluates f and g wherever it likes and feeds them in; the vectors, the (s, y) history ring and the two-loop recursion
// stay on the device and run through the SAME kernels (DeviceLbfgs) the PINN handles use.
// -----------------------------------------------------------------------------------------------------------------
struct pinn_lbfgs_handle {
  int device = 0, n = 0;
  cudaStream_t stream = nullptr;
  double *d_x = nullptr, *d_R = nullptr;   // the iterate; [g | f 0 0], laid out as a model's reduced vector
  DeviceLbfgs lb;
  int reported = 0;
};

int pinn_lbfgs_destroy(pinn_lbfgs_t* s) {
  if (!s) return 0;
  cudaSetDevice(s->device);
  if (s->stream) cudaStreamSynchronize(s->stream);
  if (s->d_x) cudaFree(s->d_x);
  if (s->d_R) cudaFree(s->d_R);
  s->lb.release();
  if (s->stream) cudaStreamDestroy(s->stream);
  delete s;
  return 0;
}

int pinn_lbfgs_create(pinn_lbfgs_t** out, int device, int64_t n, const double* x0, int max_iter, double learning_rate,
                      int n_correction, double tol_fun, double tol_x, double max_eval) {
  if (!out || !x0 || n < 1) return fail("pinn_lbfgs_create: bad arguments");
  if (max_iter < 1) return fail("pinn_lbfgs_create: max_iter must be >= 1 (lbfgs() returns before anything for maxIter == 0)");
  LbfgsConfig cfg;
  if (lbfgs_config("pinn_lbfgs_create", n, max_iter, learning_rate, n_correction, tol_fun, tol_x, max_eval, &cfg)) return -1;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail("pinn_lbfgs_create: no CUDA device -- this library has no CPU fallback");
  if (device < 0 || device >= ndev) return fail("pinn_lbfgs_create: bad device index");
  pinn_lbfgs_t* s = new pinn_lbfgs_t();
  s->device = device; s->n = (int)n;
  auto setup = [&]() -> int {
    CUDA_TRY(cudaSetDevice(device));
    CUDA_TRY(cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking));
    const size_t nb = ((size_t)n + 8) * 8;
    CUDA_TRY(cudaMalloc((void**)&s->d_x, nb));
    CUDA_TRY(cudaMalloc((void**)&s->d_R, nb));
    CUDA_TRY(cudaMemsetAsync(s->d_R, 0, nb, s->stream));
    CUDA_TRY(cudaMemcpyAsync(s->d_x, x0, (size_t)n * 8, cudaMemcpyHostToDevice, s->stream));
    if (s->lb.reserve((int)n, cfg.n_corr, max_iter)) return -1;
    return s->lb.start(s->stream, cfg);
  };
  if (setup()) { pinn_lbfgs_destroy(s); return -1; }
  *out = s;
  return 0;
}

int pinn_lbfgs_feed(pinn_lbfgs_t* s, double f, const double* g, double* x_next, int* status_out, int* n_iter_out, int* n_eval_out,
                    int* logged_iter_out, double* logged_f_out) {
  if (!s || !g || !x_next || !status_out) return fail("pinn_lbfgs_feed: null argument");
  CUDA_TRY(cudaSetDevice(s->device));
  const int n = s->n;
  const double tail[3] = {f, 0.0, 0.0};          // the kernel reads f as the sum of three loss parts behind the gradient
  CUDA_TRY(cudaMemcpyAsync(s->d_R, g, (size_t)n * 8, cudaMemcpyHostToDevice, s->stream));
  CUDA_TRY(cudaMemcpyAsync(s->d_R + n, tail, 24, cudaMemcpyHostToDevice, s->stream));
  if (s->lb.iterate(s->stream, s->d_x, s->d_R, n, nullptr)) return -1;
  pinn::LbfgsState st{};
  CUDA_TRY(cudaMemcpyAsync(&st, s->lb.st, sizeof(st), cudaMemcpyDeviceToHost, s->stream));
  CUDA_TRY(cudaStreamSynchronize(s->stream));
  *status_out = st.status;
  if (n_iter_out) *n_iter_out = st.n_iter;
  if (n_eval_out) *n_eval_out = st.n_eval;
  // the iteration whose stop tests have just run (custom_lbfgs.py:217-218 logs it only if none of them fired)
  const int tested = lbfgs_tested(st);
  int logged_it = -1;
  double logged_f = 0.0;
  // (at most one iteration is newly logged per evaluation; when the loop ends on max_iter, `tested` also covers the final,
  // never-evaluated and never-logged iteration)
  for (int it = s->reported + 1; it <= tested && it >= 1; it++) {
    int flag = 0;
    CUDA_TRY(cudaMemcpy(&flag, s->lb.logged + it, 4, cudaMemcpyDeviceToHost));
    if (flag) { logged_it = it; logged_f = f; }
  }
  if (tested > s->reported) s->reported = tested;
  if (logged_iter_out) *logged_iter_out = logged_it;
  if (logged_f_out) *logged_f_out = logged_f;
  // where to evaluate next (status 0), or the vector lbfgs() returns: the last update when the loop ended on max_iter
  const double* src = (st.status == PINN_LBFGS_MAX_ITER) ? s->lb.x_final : s->d_x;
  CUDA_TRY(cudaMemcpy(x_next, src, (size_t)n * 8, cudaMemcpyDeviceToHost));
  return 0;
}

int pinn_lbfgs_f_hist(pinn_lbfgs_t* s, double* f_hist_out, int capacity, int* n_out) {
  if (!s || !n_out) return fail("pinn_lbfgs_f_hist: null argument");
  CUDA_TRY(cudaSetDevice(s->device));
  pinn::LbfgsState st{};
  CUDA_TRY(cudaMemcpy(&st, s->lb.st, sizeof(st), cudaMemcpyDeviceToHost));
  *n_out = st.n_eval;
  if (f_hist_out) {
    if (capacity < st.n_eval) return fail("pinn_lbfgs_f_hist: buffer too small");
    if (st.n_eval) CUDA_TRY(cudaMemcpy(f_hist_out, s->lb.f_hist, (size_t)st.n_eval * 8, cudaMemcpyDeviceToHost));
  }
  return 0;
}

}  // extern "C"
