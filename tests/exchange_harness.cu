// W simulated ranks of the multi-GPU evaluation tail on ONE GPU (tests/test_gpu_exchange_sim.py).
//
// The product device code runs unchanged: pinn::reduce_tail, pinn::adam_update and pinn::fused_tail (through a wrapper kernel
// that does what the end of the Burgers kernel does).  Each rank has its own stream and its own buffers, laid out as pinn_api.cu
// lays them out: partials [n_cta][stride]; R, w, m, v; step[3], the loss ring, xseq and err; and an exchange buffer as
// pinn_p2p_export allocates it (data [2][world][slot_len] doubles, then flags [2][world][n_blocks] u64).  XchgPeers points at the
// other ranks' plain device allocations instead of IPC mappings, so the exchange's stores, flags and waits cross streams of one
// device instead of NVLink.
//
// Every enqueue launches all ranks of an evaluation, and refuses a set of grids that the device cannot hold resident at once:
// the tail CTAs of one rank spin on the flags of the others, so they may only wait for CTAs that are already running.
#include <cuda_runtime.h>

#include "optim_kernels.cuh"

namespace {

__global__ void fused_tail_kernel(const double* __restrict__ partials, int stride, const pinn::Tail tl, const int* __restrict__ run_flag) {
  __shared__ double red[512];
  if (run_flag && *run_flag != 0) return;
  pinn::fused_tail(tl, partials, stride, red);
}

constexpr int RING = 16;
constexpr int N_INTS = 5;      // snapshot integers: step[0..2], xseq, err

struct Rank {
  cudaStream_t s = nullptr;
  double *partials = nullptr, *R = nullptr, *w = nullptr, *m = nullptr, *v = nullptr, *ring = nullptr, *xchg = nullptr;
  int *step = nullptr, *xseq = nullptr, *err = nullptr, *run_flag = nullptr;
  double* snap = nullptr;      // [n_snap][n_out + 3 P + RING]
  int* snap_i = nullptr;       // [n_snap][N_INTS]
  int n_cta[64] = {0};         // per slot
};

struct Sim {
  int world, n_out, P, stride, max_cta, n_slots, n_snap, sms, occ_reduce, occ_fused;
  pinn::ReduceMap map;
  pinn::XchgPeers peers;
  Rank r[pinn::P2P_MAX];
  size_t snap_len() const { return (size_t)n_out + 3 * (size_t)P + RING; }
};

int g_err = 0;
int ck(cudaError_t e) {
  if (e != cudaSuccess && !g_err) g_err = (int)e;
  return e == cudaSuccess ? 0 : -1;
}

pinn::Tail make_tail(const Sim& S, int rank, int adam, const double* hp) {
  const Rank& q = S.r[rank];
  pinn::Tail tl{};
  tl.R = q.R; tl.map = S.map; tl.step = q.step;
  tl.w = q.w; tl.m = q.m; tl.v = q.v; tl.P = S.P;
  tl.loss_ring = q.ring; tl.ring = RING;
  if (adam) { tl.adam = 1; tl.lr = hp[0]; tl.b1 = hp[1]; tl.b2 = hp[2]; tl.eps = hp[3]; }
  tl.xchg = 1;
  tl.peers = S.peers;
  tl.peers.rank = rank;
  tl.xseq = q.xseq; tl.err = q.err;
  return tl;
}

}  // namespace

extern "C" {

int xh_last_cuda_error(void) { return g_err; }

// map: R[i] = column i for i < p_net, column extra_src[i - p_net] above (pinn::ReduceMap); n_out = P + 3 as in the product.
void* xh_create(int world, int n_out, int p_net, int n_extra, const int* extra_src, int stride, int max_cta, int n_slots, int n_snap) {
  if (world < 1 || world > pinn::P2P_MAX || n_extra < 0 || n_extra > 8 || p_net + n_extra != n_out || n_out < 4 || n_slots > 64)
    return nullptr;
  Sim* S = new Sim();
  S->world = world; S->n_out = n_out; S->P = n_out - 3; S->stride = stride; S->max_cta = max_cta;
  S->n_slots = n_slots; S->n_snap = n_snap;
  S->map = pinn::ReduceMap{};
  S->map.n_out = n_out; S->map.p_net = p_net; S->map.n_extra = n_extra;
  for (int i = 0; i < n_extra; i++) S->map.extra_src[i] = extra_src[i];
  int dev = 0;
  ck(cudaGetDevice(&dev));
  ck(cudaDeviceGetAttribute(&S->sms, cudaDevAttrMultiProcessorCount, dev));
  ck(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&S->occ_reduce, pinn::reduce_tail, 256, 0));
  ck(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&S->occ_fused, fused_tail_kernel, 256, 0));
  // exchange geometry of pinn_p2p_export
  S->peers = pinn::XchgPeers{};
  S->peers.world = world;
  S->peers.slot_len = ((n_out + 15) / 16) * 16;
  S->peers.n_blocks = (n_out + 31) / 32;
  const size_t data_doubles = (size_t)2 * world * S->peers.slot_len;
  const size_t xchg_bytes = data_doubles * 8 + (size_t)2 * world * S->peers.n_blocks * 8;
  for (int k = 0; k < world; k++) {
    Rank& q = S->r[k];
    ck(cudaStreamCreateWithFlags(&q.s, cudaStreamNonBlocking));
    ck(cudaMalloc((void**)&q.partials, (size_t)n_slots * max_cta * stride * 8));
    ck(cudaMalloc((void**)&q.run_flag, (size_t)n_slots * 4));
    ck(cudaMalloc((void**)&q.R, (size_t)n_out * 8));
    ck(cudaMalloc((void**)&q.w, (size_t)S->P * 8));
    ck(cudaMalloc((void**)&q.m, (size_t)S->P * 8));
    ck(cudaMalloc((void**)&q.v, (size_t)S->P * 8));
    ck(cudaMalloc((void**)&q.ring, RING * 8));
    ck(cudaMalloc((void**)&q.step, 3 * 4));
    ck(cudaMalloc((void**)&q.xseq, 4));
    ck(cudaMalloc((void**)&q.err, 4));
    ck(cudaMalloc((void**)&q.xchg, xchg_bytes));
    ck(cudaMalloc((void**)&q.snap, (size_t)n_snap * S->snap_len() * 8));
    ck(cudaMalloc((void**)&q.snap_i, (size_t)n_snap * N_INTS * 4));
    ck(cudaMemset(q.partials, 0, (size_t)n_slots * max_cta * stride * 8));
    ck(cudaMemset(q.run_flag, 0, (size_t)n_slots * 4));
    ck(cudaMemset(q.R, 0, (size_t)n_out * 8));
    ck(cudaMemset(q.ring, 0, RING * 8));
    ck(cudaMemset(q.step, 0, 3 * 4));
    ck(cudaMemset(q.xseq, 0, 4));
    ck(cudaMemset(q.err, 0, 4));
    ck(cudaMemset(q.xchg, 0, xchg_bytes));
    S->peers.data[k] = q.xchg;
    S->peers.flag[k] = reinterpret_cast<unsigned long long*>(q.xchg + data_doubles);
  }
  ck(cudaDeviceSynchronize());
  if (g_err) return nullptr;
  return S;
}

// sms, blocks of reduce_tail per SM, blocks of the fused wrapper per SM
int xh_info(void* h, int* out3) {
  const Sim* S = (const Sim*)h;
  out3[0] = S->sms; out3[1] = S->occ_reduce; out3[2] = S->occ_fused;
  return 0;
}

// partials of `rank` for evaluation slot `slot`: n_cta x stride doubles; run_flag != 0 skips the evaluation
int xh_load(void* h, int rank, int slot, const double* partials, int n_cta, int run_flag) {
  Sim* S = (Sim*)h;
  if (rank < 0 || rank >= S->world || slot < 0 || slot >= S->n_slots || n_cta < 1 || n_cta > S->max_cta) return -1;
  Rank& q = S->r[rank];
  if (ck(cudaDeviceSynchronize())) return -1;      // the ranks' streams do not order against this copy
  q.n_cta[slot] = n_cta;
  if (ck(cudaMemcpy(q.partials + (size_t)slot * S->max_cta * S->stride, partials, (size_t)n_cta * S->stride * 8, cudaMemcpyHostToDevice)))
    return -1;
  return ck(cudaMemcpy(q.run_flag + slot, &run_flag, 4, cudaMemcpyHostToDevice));
}

// optimiser state of `rank`: w, m, v (P each) and the completed step count
int xh_set_state(void* h, int rank, const double* w, const double* m, const double* v, int step0) {
  Sim* S = (Sim*)h;
  if (rank < 0 || rank >= S->world) return -1;
  Rank& q = S->r[rank];
  const int st[3] = {step0, 0, 0};
  if (ck(cudaDeviceSynchronize()) || ck(cudaMemcpy(q.w, w, (size_t)S->P * 8, cudaMemcpyHostToDevice)) || ck(cudaMemcpy(q.m, m, (size_t)S->P * 8, cudaMemcpyHostToDevice)) ||
      ck(cudaMemcpy(q.v, v, (size_t)S->P * 8, cudaMemcpyHostToDevice)) || ck(cudaMemcpy(q.step, st, 12, cudaMemcpyHostToDevice)))
    return -1;
  return 0;
}

// One evaluation on every rank, enqueued without a host synchronisation, then a snapshot of every rank's state into `snap`.
//   form 0: reduce_tail with grid[rank] blocks;  form 1: fused_tail in a launch of n_cta CTAs (grid ignored);
//   form 2: adam_update on the R already in place (the NCCL path after its all-reduce; no exchange).
// hp = (lr, b1, b2, eps) when adam != 0.  Returns -2 when the grids could not all be resident at once (nothing is launched).
int xh_enqueue(void* h, int slot, int form, const int* grid, int adam, const double* hp, int snap) {
  Sim* S = (Sim*)h;
  if (slot < 0 || slot >= S->n_slots || snap < 0 || snap >= S->n_snap || form < 0 || form > 2) return -1;
  long long total = 0;
  for (int k = 0; k < S->world; k++) {
    if (S->r[k].n_cta[slot] < 1) return -1;
    const int g = form == 0 ? grid[k] : form == 1 ? S->r[k].n_cta[slot] : 0;
    if (form == 0 && g < 1) return -1;
    total += g;
  }
  const int occ = form == 0 ? S->occ_reduce : S->occ_fused;
  if (total > (long long)occ * S->sms) return -2;
  for (int k = 0; k < S->world; k++) {
    Rank& q = S->r[k];
    const double* part = q.partials + (size_t)slot * S->max_cta * S->stride;
    const int* rf = q.run_flag + slot;
    if (form == 0) {
      pinn::reduce_tail<<<grid[k], 256, 0, q.s>>>(part, q.n_cta[slot], S->stride, make_tail(*S, k, adam, hp), rf);
    } else if (form == 1) {
      fused_tail_kernel<<<q.n_cta[slot], 256, 0, q.s>>>(part, S->stride, make_tail(*S, k, adam, hp), rf);
    } else {
      pinn::Tail tl = make_tail(*S, k, 1, hp);
      tl.xchg = 0;
      pinn::adam_update<<<(S->P + 127) / 128, 128, 0, q.s>>>(tl);
    }
    if (ck(cudaGetLastError())) return -1;
  }
  for (int k = 0; k < S->world; k++) {
    Rank& q = S->r[k];
    double* d = q.snap + (size_t)snap * S->snap_len();
    ck(cudaMemcpyAsync(d, q.R, (size_t)S->n_out * 8, cudaMemcpyDeviceToDevice, q.s));
    ck(cudaMemcpyAsync(d + S->n_out, q.w, (size_t)S->P * 8, cudaMemcpyDeviceToDevice, q.s));
    ck(cudaMemcpyAsync(d + S->n_out + S->P, q.m, (size_t)S->P * 8, cudaMemcpyDeviceToDevice, q.s));
    ck(cudaMemcpyAsync(d + S->n_out + 2 * (size_t)S->P, q.v, (size_t)S->P * 8, cudaMemcpyDeviceToDevice, q.s));
    ck(cudaMemcpyAsync(d + S->n_out + 3 * (size_t)S->P, q.ring, RING * 8, cudaMemcpyDeviceToDevice, q.s));
    int* di = q.snap_i + (size_t)snap * N_INTS;
    ck(cudaMemcpyAsync(di, q.step, 12, cudaMemcpyDeviceToDevice, q.s));
    ck(cudaMemcpyAsync(di + 3, q.xseq, 4, cudaMemcpyDeviceToDevice, q.s));
    ck(cudaMemcpyAsync(di + 4, q.err, 4, cudaMemcpyDeviceToDevice, q.s));
  }
  return g_err ? -1 : 0;
}

int xh_sync(void* h) {
  Sim* S = (Sim*)h;
  for (int k = 0; k < S->world; k++) ck(cudaStreamSynchronize(S->r[k].s));
  return g_err ? -1 : 0;
}

// snapshot `snap` of `rank`: out = [R (n_out) | w | m | v (P each) | loss ring (16)], ints = [step0, step1, step2, xseq, err]
int xh_read(void* h, int rank, int snap, double* out, int* ints) {
  Sim* S = (Sim*)h;
  if (rank < 0 || rank >= S->world || snap < 0 || snap >= S->n_snap) return -1;
  const Rank& q = S->r[rank];
  if (ck(cudaMemcpy(out, q.snap + (size_t)snap * S->snap_len(), S->snap_len() * 8, cudaMemcpyDeviceToHost))) return -1;
  return ck(cudaMemcpy(ints, q.snap_i + (size_t)snap * N_INTS, N_INTS * 4, cudaMemcpyDeviceToHost));
}

// the flags of `rank`'s exchange buffer: [2 parities][world][n_blocks]
int xh_read_flags(void* h, int rank, unsigned long long* out) {
  Sim* S = (Sim*)h;
  if (rank < 0 || rank >= S->world) return -1;
  return ck(cudaMemcpy(out, S->peers.flag[rank], (size_t)2 * S->world * S->peers.n_blocks * 8, cudaMemcpyDeviceToHost));
}

int xh_destroy(void* h) {
  Sim* S = (Sim*)h;
  if (!S) return 0;
  for (int k = 0; k < S->world; k++) {
    Rank& q = S->r[k];
    if (q.s) cudaStreamSynchronize(q.s);
    for (void* p : {(void*)q.partials, (void*)q.run_flag, (void*)q.R, (void*)q.w, (void*)q.m, (void*)q.v, (void*)q.ring, (void*)q.step,
                    (void*)q.xseq, (void*)q.err, (void*)q.xchg, (void*)q.snap, (void*)q.snap_i})
      cudaFree(p);
    if (q.s) cudaStreamDestroy(q.s);
  }
  delete S;
  return 0;
}

}  // extern "C"
