// Cross-CTA reduction, on-device Adam (TF-2.0 semantics) and the device-resident two-loop L-BFGS.
// Replaces: utils/neuralnetwork.py:112-116 (+ Keras Adam), utils/custom_lbfgs.py:39-236.
#pragma once
#include "pinn_common.cuh"

namespace pinn {

// Layout of the reduced vector R: [0, P) gradient; [P, P+3) loss parts (data|ic, boundary, residual).
// It is contiguous so that one ncclAllReduce(P+3) covers gradient and loss.

struct LbfgsState {
  int status;       // PINN_LBFGS_*; 0 = running
  int n_iter;
  int n_eval;
  int k;            // history length
  int head;         // ring slot of the oldest pair
  int pending;      // 1: an evaluation has been enqueued whose stop tests have not run yet
  int max_iter;
  int n_corr;
  double max_eval;
  double lr, tol_fun, tol_x;
  double h_diag, t, f, f_old;
  double ro[128];   // 1 / (y_i . s_i) per ring slot, cached when the pair is pushed (same dot product the reference
                    // recomputes every iteration, utils/custom_lbfgs.py:121-123)
  // ---- Gram-matrix formulation (lbfgs_dots / lbfgs_solve / lbfgs_apply): physical history slots 0..n_corr (one spare)
  int free_slot;    // physical slot that receives the candidate pair of the next iteration
  int apply;        // what lbfgs_apply has to do: 0 nothing, 1 move the model weights, 2 write x_final (last iteration)
  int slot[129];    // physical slot of the pair of age i (0 = oldest), i < k
  double c_g;       // direction d = c_g g + sum_m ca[m] s_m + cb[m] y_m  (m = age)
  double ca[128], cb[128];
};

// ------------------------------------------------------------------------------------------------
// The rules of the reference routine (utils/custom_lbfgs.py:39-236) that both L-BFGS formulations below share.
// ------------------------------------------------------------------------------------------------
// Stop tests of the evaluation that has just completed, in the reference's order: initial optimality after the first
// evaluation (:65-76), then max_eval (:195), optimality (:200-204), step below tolX (:206-210) and f change below tolX
// (:212-215).  g1 = |g|_1, s1 = |d t|_1 (not read for the initial evaluation).  Returns the status, 0 = keep going.
__device__ __forceinline__ int lbfgs_eval_status(const LbfgsState* st, int n_iter, int n_eval, double g1, double s1, double f_new) {
  if (n_iter == 0) return g1 <= st->tol_fun ? 7 : 0;
  if ((double)n_eval >= st->max_eval) return 2;
  if (g1 <= st->tol_fun) return 3;
  if (s1 <= st->tol_x) return 4;
  if (fabs(f_new - st->f_old) < st->tol_x) return 5;
  return 0;
}

// Thread 0's record of that evaluation: f_hist, and the log flag of its iteration (:217-218: an iteration is logged after its
// stop tests, and only if none of them fired).
__device__ __forceinline__ void lbfgs_record_eval(LbfgsState* st, int n_iter, int n_eval, double f_new, int status,
                                                  double* f_hist, int* logged) {
  st->n_eval = n_eval;
  st->f = f_new;
  st->pending = 0;
  f_hist[n_eval - 1] = f_new;
  if (n_iter > 0 && status == 0) logged[n_iter] = 1;
  st->status = status;
}

// The step of iteration n_iter from g.d and |g|_1: no progress along d stops the run (:154-156, status 6); the step length
// is min(1, 1/|g|_1) on the first iteration and the fixed learning rate after (:159-163); the last iteration's update goes
// to x_final instead of the model and is never evaluated (:176-182, status 1 at :192).
struct LbfgsStep {
  bool stop, last;
  double t;
};
__device__ __forceinline__ LbfgsStep lbfgs_step(const LbfgsState* st, int n_iter, double gtd, double g1) {
  LbfgsStep s;
  s.stop = gtd > -st->tol_x;
  s.t = (n_iter == 1) ? fmin(1.0, 1.0 / g1) : st->lr;
  s.last = n_iter == st->max_iter;
  return s;
}
// Thread 0's record of the step (f_old = f precedes the progress test, :144-145).
__device__ __forceinline__ void lbfgs_record_step(LbfgsState* st, int n_iter, const LbfgsStep& s) {
  st->n_iter = n_iter;
  st->f_old = st->f;
  if (s.stop) { st->status = 6; return; }
  st->t = s.t;
  if (s.last) st->status = 1;
  else st->pending = 1;
}

// ------------------------------------------------------------------------------------------------
// reduce the per-CTA partial vectors (fixed order -> deterministic).  src index map: gradient entries
// [0,P_net) map 1:1; extra entries are gathered through `extra_src` (parameter and loss-part slots).
// ------------------------------------------------------------------------------------------------
struct ReduceMap {
  int n_out;          // entries of R to produce
  int p_net;          // first p_net entries copy 1:1
  int extra_src[8];   // source column for R[p_net + i]
  int n_extra;
};

// Fixed-order sum of the per-CTA partials, 32 entries per block of 256 threads: warp w adds the partials of CTAs w, w+8, ...
// for entry `lane` (every load is one coalesced 256-byte row segment, all of a thread's loads are independent), the eight
// warp sums meet in shared memory and are combined as ((0+1)+(2+3))+((4+5)+(6+7)) -- deterministic, and the same order as
// the 8-lanes-per-entry shuffle tree of round 1 (which read 8 x 32 bytes per load and was slower).
// Contains ONE block barrier; returns the total of entry (threadIdx.x & 31) to every thread.
__device__ __forceinline__ double combine8(const double* red, int lane) {
  return ((red[lane] + red[32 + lane]) + (red[64 + lane] + red[96 + lane])) +
         ((red[128 + lane] + red[160 + lane]) + (red[192 + lane] + red[224 + lane]));
}
__device__ __forceinline__ double reduce_block_entries(const double* __restrict__ partials, int n_cta, int stride, int src, bool ok,
                                                       double* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double s = 0.0;
  if (ok) {
    const double* col = partials + src;
#pragma unroll 8
    for (int b = warp; b < n_cta; b += 8) s += __ldcg(col + (size_t)b * stride);   // L2: other CTAs of a running launch may have written it
  }
  red[warp * 32 + lane] = s;
  __syncthreads();
  return combine8(red, lane);
}

// ------------------------------------------------------------------------------------------------
// Adam (ResourceApplyAdam of TF 2.0):  alpha_t = lr sqrt(1-b2^t)/(1-b1^t); m += (g-m)(1-b1);
// v += (g^2-v)(1-b2); w -= alpha_t m / (sqrt(v)+eps).   step[0] = t (completed steps).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void adam_entry(double* w, double* m, double* v, double g, int i, int t, double lr, double b1,
                                           double b2, double eps) {
  const double alpha = lr * sqrt(1.0 - pow(b2, (double)t)) / (1.0 - pow(b1, (double)t));
  const double mi = m[i] + (g - m[i]) * (1.0 - b1);
  const double vi = v[i] + (g * g - v[i]) * (1.0 - b2);
  m[i] = mi;
  v[i] = vi;
  w[i] -= (mi * alpha) / (sqrt(vi) + eps);
}

// ------------------------------------------------------------------------------------------------
// Reduce -> all-to-all PUSH over NVLink peer memory -> (Adam) in the tail of every evaluation (multi-GPU, one process per
// GPU): one launch per rank and evaluation instead of a reduction + ncclAllReduce + adam_update.
//
// Every rank owns an IPC-exported exchange buffer   data[2 parities][world][slot_len] doubles, flag[2][world][n_blocks] u64.
// Block b of rank r reduces its 32 entries of the per-CTA partials (fixed order), STORES them into slot [parity][r] of EVERY
// rank's buffer (warp k of a block writes its 32 entries to peer k: remote stores are fire-and-forget, nobody pulls), fences, and
// raises flag[parity][r][b] = seq on every peer.  It then waits on its LOCAL flags of all ranks for the same block --
// a local spin, no NVLink round trips -- sums the world slots in a fixed butterfly order (bitwise identical on all ranks,
// so replicated optimiser state never diverges) and applies Adam to its entries in the same pass.
// seq / parity come from a device-side counter of published evaluations (identical on all ranks), so an evaluation that
// is skipped on the device (L-BFGS stopped: *run_flag != 0 on every rank alike) consumes neither.  Two parities suffice: a
// rank publishes evaluation k+1 only after it has seen every peer's evaluation k, and a peer publishes k only after it
// has finished consuming k-1 (stream order), so slot parity (k+1)&1 is no longer being read anywhere.
// The wait is bounded (~20 s by the global timer): a dead peer raises *err instead of hanging the GPU, and the update is
// skipped; the host reports it at the next synchronising call.
// ------------------------------------------------------------------------------------------------
constexpr int P2P_MAX = 8;
struct XchgPeers {
  double* data[P2P_MAX];                 // peer exchange buffers
  unsigned long long* flag[P2P_MAX];
  int world, rank;
  int slot_len;                          // doubles per (parity, rank) slot
  int n_blocks;                          // flags per (parity, rank)
};

__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// One 32-entry virtual block of the exchange, executed by a whole block of 256 threads: local reduction of the partials, push
// to every rank, publication, wait for every rank's copy, rank-ordered sum, optional Adam.  red/red2: 256 doubles each.
struct AdamDev {
  int on;
  double *w, *m, *v;
  int P, t;
  double lr, b1, b2, eps;
};
__device__ __forceinline__ void exchange_block(int vb, const double* __restrict__ partials, int n_cta, int stride, const ReduceMap& map,
                                               const XchgPeers& peers, unsigned long long seq, int* __restrict__ err,
                                               double* __restrict__ R, const AdamDev& ad, double* red, double* red2, bool& dead) {
  const int parity = (int)(seq & 1);
  const int lane = threadIdx.x & 31, sub = threadIdx.x >> 5;       // entry within the virtual block; warp = partial slice, then peer rank
  const int i = vb * 32 + lane;
  const bool ok = i < map.n_out;
  const int src = ok ? (i < map.p_net ? i : map.extra_src[i - map.p_net]) : 0;
  const double s = reduce_block_entries(partials, n_cta, stride, src, ok, red);   // every warp holds the 32 local sums
  // ---- push: warp k stores the 32 entries into rank k's buffer (one 256-byte row), slot [parity][my rank]
  const size_t slot = ((size_t)parity * peers.world + peers.rank) * peers.slot_len;
  if (ok && sub < peers.world) peers.data[sub][slot + i] = s;
  // publication: the block barrier orders every thread's data stores before the flag writers, whose release at system
  // scope (fence + store) is cumulative over what they have observed through the barrier -- ONE system-scope fence per
  // block and peer instead of one per thread
  __syncthreads();
  if (threadIdx.x < peers.world) {
    __threadfence_system();
    st_release_sys(peers.flag[threadIdx.x] + ((size_t)parity * peers.world + peers.rank) * peers.n_blocks + vb, seq);
  }
  // ---- wait for every rank's copy of this virtual block's entries (local flags)
  if (threadIdx.x < peers.world) {
    const unsigned long long* f = peers.flag[peers.rank] + ((size_t)parity * peers.world + threadIdx.x) * peers.n_blocks + vb;
    const unsigned long long t0 = globaltimer_ns();
    while (ld_acquire_sys(f) < seq) {
      if (globaltimer_ns() - t0 > 20000000000ULL) { atomicExch(err, 1); break; }
      __nanosleep(32);
    }
  }
  __syncthreads();
  dead = dead || *(volatile int*)err != 0;        // a peer never published: leave R, weights and optimiser state untouched
  // ---- sum over ranks: warp k loads rank k's 32 values from the LOCAL buffer, combined in the fixed order of combine8
  double part = 0.0;
  if (ok && sub < peers.world)
    part = __ldcv(peers.data[peers.rank] + ((size_t)parity * peers.world + sub) * peers.slot_len + i);
  red2[sub * 32 + lane] = part;
  __syncthreads();
  const double tot = combine8(red2, lane);
  if (ok && sub == 0 && !dead) {
    R[i] = tot;
    if (ad.on && i < ad.P) adam_entry(ad.w, ad.m, ad.v, tot, i, ad.t, ad.lr, ad.b1, ad.b2, ad.eps);
  }
}

// ------------------------------------------------------------------------------------------------
// The tail of an evaluation: the fixed-order reduction of the per-CTA partials into R = [grad | loss parts], 32 entries at a
// time, with the exchange between ranks (world > 1, P2P) and the Adam update (Adam steps) in the same pass.  It runs either as
// the stand-alone kernel reduce_tail or in the last CTAs of the fused loss/gradient launch (fused_tail); both run tail_block
// and tail_finish, so the two forms give the same bits.
// ------------------------------------------------------------------------------------------------
struct Tail {
  int enabled;            // fused kernels: run fused_tail at the end of the launch
  double* R;
  ReduceMap map;
  int adam;               // 1: Adam step (update, loss ring, step counter); 0: evaluation only (L-BFGS, loss/gradient queries)
  double *w, *m, *v;
  int P;
  double lr, b1, b2, eps;
  double* loss_ring;
  int ring;
  int xchg;               // 1: exchange with the other ranks over peer memory
  XchgPeers peers;
  int* xseq;              // evaluations published to the peers so far (identical on all ranks)
  int* err;               // raised when a peer never published
  int* step;              // [0] completed Adam steps, [1] participants done, [2] fused_tail's tickets (both counters left at 0)
};

// One 32-entry block vb of R, executed by a whole block of 256 threads.  red: 512 doubles of shared memory.  t (the Adam step
// being taken) and seq (the exchange's sequence number) are read once per participant by the caller: only tail_finish advances
// them, after every participant's last block.
__device__ __forceinline__ void tail_block(const Tail& tl, int vb, const double* __restrict__ partials, int n_cta, int stride,
                                           double* red, int t, unsigned long long seq) {
  const AdamDev ad{tl.adam, tl.w, tl.m, tl.v, tl.P, t, tl.lr, tl.b1, tl.b2, tl.eps};
  if (tl.xchg) {
    bool dead = false;                  // *err only ever goes from 0 to 1: the flag of one block is the flag of all later ones
    exchange_block(vb, partials, n_cta, stride, tl.map, tl.peers, seq, tl.err, tl.R, ad, red, red + 256, dead);
  } else {
    const int i = vb * 32 + (threadIdx.x & 31);
    const bool ok = i < tl.map.n_out;
    const int src = ok ? (i < tl.map.p_net ? i : tl.map.extra_src[i - tl.map.p_net]) : 0;
    const double s = reduce_block_entries(partials, n_cta, stride, src, ok, red);
    if (ok && threadIdx.x < 32) {
      tl.R[i] = s;
      if (ad.on && i < ad.P) adam_entry(ad.w, ad.m, ad.v, s, i, t, ad.lr, ad.b1, ad.b2, ad.eps);
    }
  }
  __syncthreads();                      // red is rewritten by the next block of entries
}

// Called by all threads of each of the n_part participants after its last block.  The last participant to finish writes the
// loss (its three parts live in possibly different blocks) and advances the step to t, resets the counters and advances the
// exchange sequence, so no participant can observe an advanced counter.
__device__ __forceinline__ void tail_finish(const Tail& tl, int n_part, int t) {
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int done = atomicAdd(tl.step + 1, 1);
    if (done == n_part - 1) {
      __threadfence();
      if (tl.adam && !(tl.xchg && *(volatile int*)tl.err != 0)) {     // a peer never published: optimiser state untouched
        const volatile double* Rv = tl.R;
        tl.loss_ring[(t - 1) % tl.ring] = Rv[tl.P] + Rv[tl.P + 1] + Rv[tl.P + 2];
        *(volatile int*)tl.step = t;
      }
      tl.step[1] = 0;
      tl.step[2] = 0;
      if (tl.xchg) *(volatile int*)tl.xseq = *(volatile int*)tl.xseq + 1;
      __threadfence();
    }
  }
}

// The stand-alone tail, one launch after the fused kernel.  With the exchange the grid is capped at a size that is certainly
// co-resident (the host passes min(n_vblocks, 2 x SMs)); every block walks the 32-entry "virtual blocks" vb = blockIdx.x,
// blockIdx.x + gridDim.x, ... in increasing order.  A block waiting for the peers' copy of vb therefore only depends on peers'
// blocks that wait for SMALLER virtual blocks: no cycle, whatever the order in which the hardware dispatches blocks on the
// different GPUs.
__global__ void reduce_tail(const double* __restrict__ partials, int n_cta, int stride, const Tail tl, const int* __restrict__ run_flag) {
  __shared__ double red[512];
  if (run_flag && *run_flag != 0) return;          // identical on every rank (replicated L-BFGS state)
  const int nb = (tl.map.n_out + 31) / 32;
  const int t = tl.adam ? *(volatile int*)tl.step + 1 : 0;
  const unsigned long long seq = tl.xchg ? (unsigned long long)(*(volatile int*)tl.xseq) + 1 : 0;
  for (int vb = blockIdx.x; vb < nb; vb += gridDim.x) tail_block(tl, vb, partials, n_cta, stride, red, t, seq);
  tail_finish(tl, gridDim.x, t);
}

// Adam on an R that is already complete (NCCL path: after the all-reduce).
__global__ void adam_update(const Tail tl) {
  const int t = tl.step[0] + 1;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < tl.P) adam_entry(tl.w, tl.m, tl.v, tl.R[i], i, t, tl.lr, tl.b1, tl.b2, tl.eps);
  tail_finish(tl, gridDim.x, t);
}

// ------------------------------------------------------------------------------------------------
// The tail INSIDE the fused loss/gradient launch (specialised Burgers kernel): every CTA takes a ticket after writing its
// partial vector; the last K to arrive (one per 32-entry block when the grid is large enough) wait for the stragglers and then
// run the tail on their blocks -- no second launch, no kernel boundary in the middle of a step.  Every CTA of the launch must
// be resident (grid <= number of SMs, one CTA per SM), which holds for the persistent kernels that use it.  Across GPUs a tail
// CTA that waits for the peers' copy of block vb depends on the peers' tail CTA that owns vb, which exists as soon as enough of
// the peer's CTAs have finished -- the peers' kernels run to completion independently of the exchange, so there is no cycle.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Called by ALL threads of every CTA after the CTA's partial vector has been written.  red: >= 512 doubles of shared memory
// nobody else uses any more.
__device__ __forceinline__ void fused_tail(const Tail& tl, const double* __restrict__ partials, int stride, double* red) {
  __shared__ int s_slot;
  const int nb = (tl.map.n_out + 31) / 32;
  const int K = (int)gridDim.x < nb ? (int)gridDim.x : nb;            // tail CTAs: the last K to arrive
  int* tickets = tl.step + 2;
  __threadfence();                                                    // this thread's partial entries, device-wide
  __syncthreads();
  if (threadIdx.x == 0) {
    const int ticket = atomicAdd(tickets, 1);
    const int slot = ticket - ((int)gridDim.x - K);
    if (slot >= 0)
      while (ld_acquire_gpu(tickets) < (int)gridDim.x) __nanosleep(40);  // every partial vector is complete
    s_slot = slot;
  }
  __syncthreads();
  const int slot = s_slot;
  if (slot < 0) return;
  const int t = tl.adam ? *(volatile int*)tl.step + 1 : 0;
  const unsigned long long seq = tl.xchg ? (unsigned long long)(*(volatile int*)tl.xseq) + 1 : 0;
  for (int vb = slot; vb < nb; vb += K) tail_block(tl, vb, partials, (int)gridDim.x, stride, red, t, seq);
  tail_finish(tl, K, t);
}

// ------------------------------------------------------------------------------------------------
// L-BFGS iteration kernel: ONE CTA; each thread keeps EPT entries of the working vector in registers.
// Runs (a) the stop tests of the previous iteration's evaluation, (b) the memory update and two-loop
// recursion, (c) the step, exactly in the reference order (utils/custom_lbfgs.py:81-221).
// ------------------------------------------------------------------------------------------------
// Block-wide sum in a fixed order, ONE barrier per call: the per-warp partials go to alternating halves of `red`, so a
// call never overwrites values another warp may still be reading (a warp can be at most one call ahead).
template <int NT>
__device__ __forceinline__ double block_sum_t(double v, double* red, int& phase) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* buf = red + (phase & 1) * 32;
  phase++;
  if (lane == 0) buf[warp] = v;
  __syncthreads();
  constexpr int NW = NT / 32;
  double s = (lane < NW) ? buf[lane] : 0.0;
#pragma unroll
  for (int m = NW / 2; m > 0; m >>= 1) s += shfl_xor_d(s, m);
  return __shfl_sync(0xffffffffu, s, 0);   // every thread holds the total
}

template <int EPT, int LB_THREADS>
__global__ void __launch_bounds__(LB_THREADS, 1)
lbfgs_iterate(LbfgsState* __restrict__ st, double* __restrict__ w, const double* __restrict__ R, int P,
              double* __restrict__ g_old, double* __restrict__ d, double* __restrict__ S, double* __restrict__ Y,
              double* __restrict__ x_final, double* __restrict__ f_hist, int* __restrict__ logged) {
  __shared__ double red[64];
  __shared__ double ro[128], al[128];
  int red_phase = 0;
  auto block_sum = [&](double v, double*) { return block_sum_t<LB_THREADS>(v, red, red_phase); };
  const int tid = threadIdx.x;
  if (st->status != 0) return;

  double gv[EPT];
#pragma unroll
  for (int e = 0; e < EPT; e++) {
    const int i = tid + e * LB_THREADS;
    gv[e] = i < P ? R[i] : 0.0;
  }
  const double f_new = R[P] + R[P + 1] + R[P + 2];

  // ---- (a) bookkeeping + stop tests for the evaluation that has just completed
  if (st->pending) {
    const int n_iter = st->n_iter;
    const int n_eval = st->n_eval + 1;
    double a1 = 0.0;
#pragma unroll
    for (int e = 0; e < EPT; e++) a1 += fabs(gv[e]);
    a1 = block_sum(a1, red);
    int status;
    if (n_iter == 0) status = lbfgs_eval_status(st, n_iter, n_eval, a1, 0.0, f_new);   // no step yet, so no |d t|_1
    else {
      double a2 = 0.0;
      const double t = st->t;
#pragma unroll
      for (int e = 0; e < EPT; e++) {
        const int i = tid + e * LB_THREADS;
        a2 += i < P ? fabs(d[i] * t) : 0.0;
      }
      a2 = block_sum(a2, red);
      status = lbfgs_eval_status(st, n_iter, n_eval, a1, a2, f_new);
    }
    __syncthreads();
    if (tid == 0) lbfgs_record_eval(st, n_iter, n_eval, f_new, status, f_hist, logged);
    __syncthreads();
    if (status != 0) return;
  }

  // ---- (b) direction
  const int n_iter = st->n_iter + 1;
  const int n_corr = st->n_corr;
  double dv[EPT];
  if (n_iter == 1) {                                                     // :91-95
#pragma unroll
    for (int e = 0; e < EPT; e++) dv[e] = -gv[e];
  } else {
    const double t_prev = st->t;
    double yv[EPT], sv[EPT];
    double ys = 0.0, yy = 0.0;
#pragma unroll
    for (int e = 0; e < EPT; e++) {
      const int i = tid + e * LB_THREADS;
      yv[e] = i < P ? gv[e] - g_old[i] : 0.0;                            // :98
      sv[e] = i < P ? d[i] * t_prev : 0.0;                               // :99
      ys += yv[e] * sv[e];
      yy += yv[e] * yv[e];
    }
    ys = block_sum(ys, red);
    int k = st->k, head = st->head;
    double h_diag = st->h_diag;
    if (ys > 1e-10) {                                                    // :102-114
      yy = block_sum(yy, red);
      int slot;
      if (k == n_corr) { slot = head; head = (head + 1) % n_corr; }      // drop the oldest pair
      else { slot = (head + k) % n_corr; k++; }
#pragma unroll
      for (int e = 0; e < EPT; e++) {
        const int i = tid + e * LB_THREADS;
        if (i < P) { S[(size_t)slot * P + i] = sv[e]; Y[(size_t)slot * P + i] = yv[e]; }
      }
      h_diag = ys / yy;
      if (tid == 0) st->ro[slot] = 1.0 / ys;
      __syncthreads();
    }
    // ro_i (i = 0 oldest) from the per-slot cache
    for (int i = tid; i < k; i += LB_THREADS) ro[i] = st->ro[(head + i) % n_corr];
    __syncthreads();
    double qv[EPT];
#pragma unroll
    for (int e = 0; e < EPT; e++) qv[e] = -gv[e];                        // :130
    // first loop (:131-133), newest to oldest; the next pair is prefetched while the current reduction runs
    double sn[EPT], yn[EPT];
    if (k > 0) {
      const size_t base = (size_t)((head + k - 1) % n_corr) * P;
#pragma unroll
      for (int e = 0; e < EPT; e++) {
        const int j = tid + e * LB_THREADS;
        sn[e] = j < P ? S[base + j] : 0.0;
        yn[e] = j < P ? Y[base + j] : 0.0;
      }
    }
    for (int i = k - 1; i >= 0; i--) {
      double sc[EPT], yc[EPT];
#pragma unroll
      for (int e = 0; e < EPT; e++) { sc[e] = sn[e]; yc[e] = yn[e]; }
      if (i > 0) {
        const size_t base = (size_t)((head + i - 1) % n_corr) * P;
#pragma unroll
        for (int e = 0; e < EPT; e++) {
          const int j = tid + e * LB_THREADS;
          sn[e] = j < P ? S[base + j] : 0.0;
          yn[e] = j < P ? Y[base + j] : 0.0;
        }
      }
      double a = 0.0;
#pragma unroll
      for (int e = 0; e < EPT; e++) a += sc[e] * qv[e];
      a = block_sum(a, red) * ro[i];
      if (tid == 0) al[i] = a;
#pragma unroll
      for (int e = 0; e < EPT; e++) qv[e] -= a * yc[e];
    }
    __syncthreads();
#pragma unroll
    for (int e = 0; e < EPT; e++) qv[e] *= h_diag;                       // :136
    // second loop (:137-139), oldest to newest
    if (k > 0) {
      const size_t base = (size_t)(head % n_corr) * P;
#pragma unroll
      for (int e = 0; e < EPT; e++) {
        const int j = tid + e * LB_THREADS;
        sn[e] = j < P ? S[base + j] : 0.0;
        yn[e] = j < P ? Y[base + j] : 0.0;
      }
    }
    for (int i = 0; i < k; i++) {
      double sc[EPT], yc[EPT];
#pragma unroll
      for (int e = 0; e < EPT; e++) { sc[e] = sn[e]; yc[e] = yn[e]; }
      if (i + 1 < k) {
        const size_t base = (size_t)((head + i + 1) % n_corr) * P;
#pragma unroll
        for (int e = 0; e < EPT; e++) {
          const int j = tid + e * LB_THREADS;
          sn[e] = j < P ? S[base + j] : 0.0;
          yn[e] = j < P ? Y[base + j] : 0.0;
        }
      }
      double a = 0.0;
#pragma unroll
      for (int e = 0; e < EPT; e++) a += yc[e] * qv[e];
      const double be = block_sum(a, red) * ro[i];
      const double c = al[i] - be;
#pragma unroll
      for (int e = 0; e < EPT; e++) qv[e] += c * sc[e];
    }
#pragma unroll
    for (int e = 0; e < EPT; e++) dv[e] = qv[e];
    if (tid == 0) { st->k = k; st->head = head; st->h_diag = h_diag; }
  }

  // ---- (c) step
  double gtd = 0.0, a1 = 0.0;
#pragma unroll
  for (int e = 0; e < EPT; e++) { gtd += gv[e] * dv[e]; a1 += fabs(gv[e]); }
  gtd = block_sum(gtd, red);                                             // :151
  a1 = block_sum(a1, red);
  // g_old = g, f_old = f happen before the progress test (:144-145)
#pragma unroll
  for (int e = 0; e < EPT; e++) {
    const int i = tid + e * LB_THREADS;
    if (i < P) { g_old[i] = gv[e]; d[i] = dv[e]; }
  }
  const LbfgsStep step = lbfgs_step(st, n_iter, gtd, a1);
  if (!step.stop) {
#pragma unroll
    for (int e = 0; e < EPT; e++) {
      const int i = tid + e * LB_THREADS;
      if (i < P) {
        const double xn = w[i] + step.t * dv[e];                         // :174
        if (step.last) x_final[i] = xn;
        else w[i] = xn;
      }
    }
  }
  __syncthreads();
  if (tid == 0) lbfgs_record_step(st, n_iter, step);
}

// ------------------------------------------------------------------------------------------------
// L-BFGS, Gram-matrix formulation: the same iteration as lbfgs_iterate (utils/custom_lbfgs.py:81-221, same stop tests, same
// quirks), re-associated so that nothing sequential touches a P-vector.  lbfgs_iterate is one CTA whose 2 x n_corr dependent
// dot products each stream an (s, y) pair through ONE SM (4.8 MB of history per iteration at n_corr = 50, P = 3021:
// SM<->L2 bandwidth bound).  Here
//   lbfgs_dots   (P/256 CTAs): y = g - g_old, s = d t into the spare history slot; per-CTA partial sums of ALL dot products
//                the iteration needs -- s_m.y, y_m.y, s_m.g, y_m.g for every stored pair m, y.s, y.y, s.g, y.g, g.g, |g|_1,
//                |s|_1 -- the history is read once, by all SMs in parallel;
//   lbfgs_solve  (1 CTA): fixed-order sum of the partials, the stop tests, the curvature test and history bookkeeping, the
//                Gram matrices SY[a][b] = s_a.y_b, YY[a][b] = y_a.y_b (one new row/column per accepted pair), and the two-loop
//                recursion in COEFFICIENT space:  al_i = ro_i (-s_i.g - sum_{m>i} al_m SY[i][m]);
//                y_i.q = -y_i.g - sum_m al_m YY[i][m];  be_i = ro_i (H y_i.q + sum_{m<i} (al_m - be_m) SY[m][i]);
//                d = -H g - H sum al_m y_m + sum (al_m - be_m) s_m;  g.d from the same numbers;
//   lbfgs_apply  (P/256 CTAs): d as that linear combination (history read once more, in parallel), g_old = g, x += t d.
// Mathematically identical to the reference's loop; rounding differs at the 1e-16 level (different association), which a
// fixed-step L-BFGS amplifies about tenfold per ten iterations -- as between any two fp64 implementations (DESIGN.md section 1).
// ------------------------------------------------------------------------------------------------
constexpr int LB_CHUNK = 256;       // entries per CTA of lbfgs_dots / lbfgs_apply
constexpr int LB_NSCAL = 7;         // scalar dots: |g|_1, g.g, |s|_1, y.s, y.y, s.g, y.g;  then 4 per stored pair

constexpr int LB_DOT_THREADS = 512;  // lbfgs_dots: 16 warps share a 256-entry chunk (the dot products are latency-bound)

__global__ void __launch_bounds__(LB_DOT_THREADS)
lbfgs_dots(const LbfgsState* __restrict__ st, const double* __restrict__ R, int P, const double* __restrict__ g_old,
           const double* __restrict__ d, double* __restrict__ S, double* __restrict__ Y, double* __restrict__ part, int part_stride) {
  __shared__ double sg[LB_CHUNK], sy[LB_CHUNK], ss[LB_CHUNK];
  if (st->status != 0) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool have_step = st->n_iter > 0;             // false: this is the initial evaluation, there is no pair to form
  const int k = st->k;
  if (tid < LB_CHUNK) {
    const int i = blockIdx.x * LB_CHUNK + tid;
    const double gi = i < P ? R[i] : 0.0;
    double yi = 0.0, si = 0.0;
    if (have_step && i < P) {
      yi = gi - g_old[i];                             // custom_lbfgs.py:98
      si = d[i] * st->t;                              // :99
      const size_t o = (size_t)st->free_slot * P + i;
      S[o] = si; Y[o] = yi;
    }
    sg[tid] = gi; sy[tid] = yi; ss[tid] = si;
  }
  __syncthreads();
  double* out = part + (size_t)blockIdx.x * part_stride;
  constexpr int NW = LB_DOT_THREADS / 32, EPL = LB_CHUNK / 32;
  // scalar dots: warps 0..6, one each; lanes stride the chunk; fixed shuffle tree -> deterministic
  if (warp < LB_NSCAL) {
    double acc = 0.0;
#pragma unroll
    for (int e = 0; e < EPL; e++) {
      const int t = lane + 32 * e;
      const double gg = sg[t], yy = sy[t], sv = ss[t];
      acc += warp == 0 ? fabs(gg) : warp == 1 ? gg * gg : warp == 2 ? fabs(sv) : warp == 3 ? yy * sv : warp == 4 ? yy * yy
                                                                                   : warp == 5 ? sv * gg : yy * gg;
    }
    acc = warp_sum(acc);
    if (lane == 0) out[warp] = acc;
  }
  if (!have_step) return;
  // stored pairs: warp takes ages m = warp, warp + 16, ...; the four dot products of a pair (s_m.y, y_m.y, s_m.g, y_m.g) share
  // their 2 x 8 loads per lane, all in flight together
  for (int m = warp; m < k; m += NW) {
    const size_t base = (size_t)st->slot[m] * P + (size_t)blockIdx.x * LB_CHUNK;
    double sv[EPL], yv[EPL];
#pragma unroll
    for (int e = 0; e < EPL; e++) {
      const int t = lane + 32 * e;
      const bool in = blockIdx.x * LB_CHUNK + t < P;
      sv[e] = in ? S[base + t] : 0.0;
      yv[e] = in ? Y[base + t] : 0.0;
    }
    double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
#pragma unroll
    for (int e = 0; e < EPL; e++) {
      const int t = lane + 32 * e;
      a0 = fma(sv[e], sy[t], a0); a1 = fma(yv[e], sy[t], a1);
      a2 = fma(sv[e], sg[t], a2); a3 = fma(yv[e], sg[t], a3);
    }
    a0 = warp_sum(a0); a1 = warp_sum(a1); a2 = warp_sum(a2); a3 = warp_sum(a3);
    if (lane == 0) {
      double* o = out + LB_NSCAL + 4 * m;
      o[0] = a0; o[1] = a1; o[2] = a2; o[3] = a3;
    }
  }
}

__global__ void __launch_bounds__(128)
lbfgs_solve(LbfgsState* __restrict__ st, const double* __restrict__ R, int P, const double* __restrict__ part, int n_blocks,
            int part_stride, double* __restrict__ SY, double* __restrict__ YY, double* __restrict__ f_hist, int* __restrict__ logged) {
  extern __shared__ double sy_s[];          // SY of the live pairs in AGE order, [k][k]: the recurrences below walk it serially
  __shared__ double dots[LB_NSCAL + 4 * 128];
  __shared__ double al[128], dl[128], sgv[128], ygv[128], yq[128], rov[128];
  __shared__ int pslot[128];
  if (st->status != 0) return;
  const int tid = threadIdx.x;
  const bool have_step = st->n_iter > 0;
  int k = st->k;
  const int ndots = LB_NSCAL + (have_step ? 4 * k : 0);
  for (int j = tid; j < ndots; j += blockDim.x) {
    double sacc = 0.0;
    for (int b = 0; b < n_blocks; b++) sacc += part[(size_t)b * part_stride + j];
    dots[j] = sacc;
  }
  for (int m = tid; m < k; m += blockDim.x) pslot[m] = st->slot[m];
  __syncthreads();
  const double f_new = R[P] + R[P + 1] + R[P + 2];
  const double a1 = dots[0];
  const int NS = st->n_corr + 1;
  // ---- (a) bookkeeping + stop tests of the evaluation that has just completed
  if (st->pending) {
    const int n_iter = st->n_iter, n_eval = st->n_eval + 1;
    const int status = lbfgs_eval_status(st, n_iter, n_eval, a1, dots[2], f_new);
    __syncthreads();
    if (tid == 0) {
      lbfgs_record_eval(st, n_iter, n_eval, f_new, status, f_hist, logged);
      if (status != 0) st->apply = 0;
    }
    if (status != 0) return;
  }
  // ---- (b) history update and direction coefficients
  const int n_iter = st->n_iter + 1;
  const int n_corr = st->n_corr;
  double h_diag = st->h_diag;
  double gtd;
  if (n_iter == 1) {                                                     // :91-95  d = -g
    gtd = -dots[1];
    if (tid == 0) { st->c_g = -1.0; }
  } else {
    const double ys = dots[3];
    const int p_new = st->free_slot;
    int shift = 0;                           // ages move down by one when the oldest pair is dropped
    int k_new = k, free_next = p_new;
    const bool accept = ys > 1e-10;                                      // :102-114
    if (accept) {
      if (k == n_corr) { shift = 1; free_next = pslot[0]; k_new = k; }
      else { k_new = k + 1; free_next = k_new <= n_corr ? k_new : n_corr; }
      h_diag = ys / dots[4];
    }
    __syncthreads();
    // Gram entries of the new pair against the stored ones (read at their OLD ages), then the age tables in their NEW order
    if (accept) {
      for (int m = tid; m < k; m += blockDim.x) {
        const int pm = pslot[m];
        SY[(size_t)pm * NS + p_new] = dots[LB_NSCAL + 4 * m + 0];        // s_m . y_new
        YY[(size_t)pm * NS + p_new] = dots[LB_NSCAL + 4 * m + 1];        // y_m . y_new (symmetric)
        YY[(size_t)p_new * NS + pm] = dots[LB_NSCAL + 4 * m + 1];
      }
      if (tid == 0) { SY[(size_t)p_new * NS + p_new] = ys; YY[(size_t)p_new * NS + p_new] = dots[4]; }
    }
    for (int m = tid; m < k; m += blockDim.x) {
      if (m >= shift) { sgv[m - shift] = dots[LB_NSCAL + 4 * m + 2]; ygv[m - shift] = dots[LB_NSCAL + 4 * m + 3]; }
    }
    __syncthreads();
    int my_slot = -1;
    if (tid < k_new) {
      if (accept && tid == k_new - 1) { my_slot = p_new; sgv[tid] = dots[5]; ygv[tid] = dots[6]; }
      else my_slot = pslot[tid + shift];
    }
    __syncthreads();
    if (tid < k_new) pslot[tid] = my_slot;
    __threadfence_block();
    __syncthreads();
    k = k_new;
    // stage SY[age a][age b] (only a <= b is ever used: s of the older pair against y of the newer one) -- all loads in flight
    // together instead of one dependent global load per step of the serial recurrences
    for (int e = tid; e < k * k; e += blockDim.x) {
      const int a = e / k, b = e - a * k;
      sy_s[e] = a <= b ? SY[(size_t)pslot[a] * NS + pslot[b]] : 0.0;
    }
    __syncthreads();
    if (tid < k) rov[tid] = 1.0 / sy_s[tid * k + tid];                        // ro_i = 1 / (y_i . s_i)   (:121-123)
    __syncthreads();
    // first loop (:131-133), newest to oldest.  Thread m accumulates  -s_m.g - sum_{j>m} al_j SY[m][j]  as the al_j appear.
    double accm = tid < k ? -sgv[tid] : 0.0;
    for (int j = k - 1; j >= 0; j--) {
      if (tid == j) al[j] = accm * rov[j];
      __syncthreads();
      if (tid < j) accm = fma(-al[j], sy_s[tid * k + j], accm);
    }
    // y_i . q  with q = -g - sum_m al_m y_m
    if (tid < k) {
      double v = -ygv[tid];
      const double* yrow = YY + (size_t)pslot[tid] * NS;
#pragma unroll 8
      for (int m = 0; m < k; m++) v = fma(-al[m], yrow[pslot[m]], v);      // independent loads, in flight together
      yq[tid] = v;
    }
    __syncthreads();
    // second loop (:137-139), oldest to newest.  Thread i accumulates  H y_i.q + sum_{m<i} (al_m - be_m) SY[m][i].
    double acci = tid < k ? h_diag * yq[tid] : 0.0;
    for (int m = 0; m < k; m++) {
      if (tid == m) dl[m] = al[m] - acci * rov[m];                       // al_m - be_m
      __syncthreads();
      if (tid > m && tid < k) acci = fma(dl[m], sy_s[m * k + tid], acci);
    }
    // g . d = -H g.g - H sum al_m y_m.g + sum (al_m - be_m) s_m.g       (:151)
    double gsum = 0.0;
    if (tid == 0) {
      gsum = -h_diag * dots[1];
      for (int m = 0; m < k; m++) gsum = fma(-h_diag * al[m], ygv[m], gsum);
      for (int m = 0; m < k; m++) gsum = fma(dl[m], sgv[m], gsum);
      dots[0] = gsum;                      // broadcast through shared memory (a1 was copied out above)
    }
    __syncthreads();
    gtd = dots[0];
    if (tid < k) { st->ca[tid] = dl[tid]; st->cb[tid] = -h_diag * al[tid]; st->slot[tid] = pslot[tid]; }
    if (tid == 0) { st->c_g = -h_diag; st->k = k; st->h_diag = h_diag; st->free_slot = free_next; }
  }
  if (n_iter == 1 && tid == 0) { st->k = 0; st->free_slot = 0; }
  // ---- (c) step
  __syncthreads();
  if (tid == 0) {
    const LbfgsStep step = lbfgs_step(st, n_iter, gtd, a1);
    lbfgs_record_step(st, n_iter, step);
    st->apply = step.stop ? 0 : step.last ? 2 : 1;
  }
}

__global__ void __launch_bounds__(LB_CHUNK)
lbfgs_apply(LbfgsState* __restrict__ st, double* __restrict__ w, const double* __restrict__ R, int P, double* __restrict__ g_old,
            double* __restrict__ d, const double* __restrict__ S, const double* __restrict__ Y, double* __restrict__ x_final) {
  __shared__ double ca[128], cb[128];
  __shared__ int ps[128];
  const int apply = st->apply;
  if (apply == 0) return;                  // a stop test fired (or the optimiser was already stopped): nothing moves
  const int k = st->k;
  for (int m = threadIdx.x; m < k; m += blockDim.x) { ca[m] = st->ca[m]; cb[m] = st->cb[m]; ps[m] = st->slot[m]; }
  __syncthreads();
  const int i = blockIdx.x * LB_CHUNK + threadIdx.x;
  if (i >= P) return;
  const double gi = R[i];
  double dv = st->c_g * gi;
#pragma unroll 8
  for (int m = 0; m < k; m++) {            // 2k independent loads per entry; the fixed order of the FMAs keeps d reproducible
    const size_t o = (size_t)ps[m] * P + i;
    dv = fma(ca[m], S[o], dv);
    dv = fma(cb[m], Y[o], dv);
  }
  g_old[i] = gi; d[i] = dv;                // :144, the direction of this step (s of the next iteration = d t)
  const double xn = fma(st->t, dv, w[i]);                                // :174
  if (apply == 2) x_final[i] = xn;         // no evaluation follows (:176-182): the model keeps the previous weights
  else w[i] = xn;
}

// ------------------------------------------------------------------------------------------------
// Generic (any layer sizes, hidden width <= MAXW_WIDE) thread-per-point kernels, off the per-step path:
// forward (predict, utils/neuralnetwork.py:151-153) and forward Taylor-mode derivatives (parity probes,
// f_model on the stored points).  Weights are read through the read-only path (warp-uniform addresses).
// ------------------------------------------------------------------------------------------------
constexpr int MAXW = 128;        // per-thread activation arrays of mlp_forward_generic for the nets that fit
constexpr int MAXW_WIDE = 256;   // widest hidden layer of any generic net (second instantiation above MAXW)
constexpr int MAXL = 16;

// Third-order mode of 1-D nets (the idle t slot carries the xxx stream):
//   a_xxx = s (z_xxx - 6 a z_x z_xx - 2 (1 - 3a^2) z_x^3);  this returns the bracket.
__device__ __forceinline__ double xxx_bracket(double a, double zx, double zxx, double zxxx) {
  return fma(-6.0 * a * zx, zxx, fma(-2.0 * fma(-3.0 * a, a, 1.0) * zx * zx, zx, zxxx));
}

struct NetDesc {
  int n_layers;            // number of Dense layers
  int dims[MAXL + 1];      // layer sizes
  int woff[MAXL], boff[MAXL];
  double lb0, lb1, dx0, dx1;
};

// NS = 1: values only; NS = 4: (h, h_x, h_t, h_xx), or (h, h_x, h_xxx, h_xx) with o3 (1-D nets).  W: widest hidden layer.
template <int NS, int W>
__global__ void mlp_forward_generic(const double* __restrict__ w, NetDesc nd, const double* __restrict__ X,
                                    const double* __restrict__ Tsoa, long long n, int in_dim, double* __restrict__ out,
                                    int o3) {
  // points either interleaved X[n][in_dim] (Tsoa == nullptr) or SoA (X = x[n], Tsoa = t[n])
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  double h[NS][W], z[NS][W];
  const double x = Tsoa ? X[p] : X[p * in_dim];
  const double t = Tsoa ? Tsoa[p] : (in_dim == 1 ? x : X[p * in_dim + 1]);
  h[0][0] = 2.0 * (x - nd.lb0) / nd.dx0 - 1.0;
  h[0][1] = nd.dims[0] == 2 ? 2.0 * (t - nd.lb1) / nd.dx1 - 1.0 : 0.0;   // 1-D nets (discrete-time models) ignore t
  if (NS == 4) {
    h[1][0] = 2.0 / nd.dx0; h[1][1] = 0.0;
    h[2][0] = 0.0;          h[2][1] = 2.0 / nd.dx1;
    h[3][0] = 0.0;          h[3][1] = 0.0;
  }
  for (int l = 0; l < nd.n_layers; l++) {
    const int fi = nd.dims[l], fo = nd.dims[l + 1];
    const double* Wl = w + nd.woff[l];
    const double* bl = w + nd.boff[l];
    if (l == nd.n_layers - 1) {
      // linear head: written straight to the output (it may be wider than MAXW, e.g. q+1 = 501 IRK stages)
      for (int j = 0; j < fo; j++) {
        double acc[NS];
        acc[0] = __ldg(bl + j);
#pragma unroll
        for (int s = 1; s < NS; s++) acc[s] = 0.0;
        for (int i = 0; i < fi; i++) {
          const double wv = __ldg(Wl + i * fo + j);
#pragma unroll
          for (int s = 0; s < NS; s++) acc[s] = fma(h[s][i], wv, acc[s]);
        }
#pragma unroll
        for (int s = 0; s < NS; s++) out[p * (NS * fo) + s * fo + j] = acc[s];
      }
      return;
    }
    for (int j = 0; j < fo; j++) {
      double acc[NS];
      acc[0] = __ldg(bl + j);
#pragma unroll
      for (int s = 1; s < NS; s++) acc[s] = 0.0;
      for (int i = 0; i < fi; i++) {
        const double wv = __ldg(Wl + i * fo + j);
#pragma unroll
        for (int s = 0; s < NS; s++) acc[s] = fma(h[s][i], wv, acc[s]);
      }
#pragma unroll
      for (int s = 0; s < NS; s++) z[s][j] = acc[s];
    }
    const bool last = (l == nd.n_layers - 1);
    for (int j = 0; j < fo; j++) {
      if (last) {
#pragma unroll
        for (int s = 0; s < NS; s++) h[s][j] = z[s][j];
      } else {
        const double a = tanh(z[0][j]);
        h[0][j] = a;
        if (NS == 4) {
          const double sd = fma(-a, a, 1.0);
          const double zx = z[1][j];
          h[1][j] = sd * zx;
          h[2][j] = sd * (o3 ? xxx_bracket(a, zx, z[3][j], z[2][j]) : z[2][j]);
          h[3][j] = sd * fma(-2.0 * a * zx, zx, z[3][j]);
        }
      }
    }
  }
  const int no = nd.dims[nd.n_layers];
  for (int s = 0; s < NS; s++)
    for (int j = 0; j < no; j++) out[p * (NS * no) + s * no + j] = h[s][j];
}


__global__ void tanh_fast_kernel(const double* __restrict__ x, int n, double* __restrict__ y) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = tanh_fast(x[i]);
}

}  // namespace pinn
