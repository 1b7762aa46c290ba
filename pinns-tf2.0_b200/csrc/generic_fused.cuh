// Generic fused PINN loss + gradient kernel: ANY tanh MLP [2, w_1, ..., w_k, out] (hidden widths <= 256, <= 15 Dense layers),
// PDE heads: Burgers inference / identification (out = 1), Schrodinger (out = 2), and the discrete-time (implicit
// Runge-Kutta) models on 1-D nets [1, ..., q(+1)] (q+1 <= 512 outputs): Burgers inference and identification
// (1d-burgers/inf_disc_burgers.py, ide_disc_burgers.py), KdV identification and Allen-Cahn inference; and, in the POLY
// instantiation, a user-defined polynomial residual in (u, u_x, u_t, u_xx) on nets [2, ..., 1] (pde 8, 9); fp64, sm_90a.
//
// Purpose: hp["layers"] is user-configurable in the reference (1d-burgers/inf_cont_burgers.py:23-34); the DMMA kernels
// (burgers_fused_v2.cuh, nls_fused.cuh) are specialised for the two BASELINE nets.  This kernel keeps the path a drop-in
// for every other layer list, and doubles as an independent on-GPU cross-check of the specialised kernels
// (PINN_FORCE_GENERIC=1).  It is a correctness-first fallback: plain DFMA, one launch, persistent CTAs.
//
// Structure (same mathematics as the specialised kernels: forward Taylor streams h, h_x, h_t, h_xx and the hand-derived
// reverse sweep, SURVEY Appendix A): a CTA owns a contiguous block of points and walks the network layer by layer;
// activations live in a per-CTA global scratch.
//   F_l   thread per (point, unit): 4 stream dot products over the previous layer (weights through the read-only path,
//         activations broadcast within the warp), tanh + Taylor epilogue
//   HEAD  linear head, PDE residual / data / boundary terms, loss parts, seeds
//   B_l   Z-bar (division-free backward formula) -> weight gradient (thread per weight entry, loop over the CTA's points;
//         written once per CTA) -> input adjoint (thread per (point, unit))
// Third-order mode (o3, KdV): a 1-D net has no t stream, so its slot carries h_xxx instead (input h_xxx = 0).  Only the
// tanh epilogue of the forward and the Z-bar formulas change; every contraction is the same 4-stream one.
#pragma once
#include "optim_kernels.cuh"

namespace pinn {
namespace generic {

constexpr int THREADS = 256;
constexpr int MAXOUT = 2;
constexpr int POLY_MAXT = 16;

// A polynomial residual (pinn_set_residual): term k is coef[k] * kappa * u^e0 u_x^e1 u_t^e2 u_xx^e3 with
// code[k] = kind | e0 << 3 | e1 << 5 | e2 << 7 | e3 << 9, kind 0..4 selecting kappa = 1, l1, l2, e^l1, e^l2 (raw lambdas).
struct PolySpec {
  int n;
  int code[POLY_MAXT];
  double coef[POLY_MAXT];
};

struct Args {
  const double* w;
  NetDesc nd;
  const double* x;
  const double* t;
  const double* tgt;          // data targets [n_d][out]
  long long n_total;
  int pde;                    // PINN_BURGERS_INF / PINN_BURGERS_IDE / PINN_NLS_INF / PINN_BURGERS_DISC (3) / PINN_BURGERS_IDE_DISC (4)
                              // / PINN_KDV_IDE_DISC (5) / PINN_AC_DISC (6) / PINN_POLY_INF (8) / PINN_POLY_IDE (9)
  int in_dim;                 // 2 (x,t), or 1 (x only: discrete-time models)
  int o3;                     // third-order mode: the t slot carries the xxx stream (KdV)
  double dt;                  // DISC, AC: time step;  irk: (q+1) x q stage matrix, q = out - 1;  IDE_DISC, KdV: [M_0 ; M_1], each q x q, q = out
  double kc;                  // AC: k of k u^3 - k u (its d is in nu)
  const double* irk;
  // Burgers: points [d0, d0+n_d) carry the data term, [c0, c0+n_c) the residual term
  long long c0, n_c, d0, n_d;
  double wf, wd, nu;
  // NLS: [ic n0 | pad to n0p | (lb,ub) pairs 2 nb | collocation];  AC: [x_0 n_d | pad to n0p | (lb, ub)]
  long long n0, n0p, nb;
  double w0, wb;
  int p_net;                  // network parameters (identification: lambdas at p_net, p_net+1)
  double* scrH;               // [grid][sum_l 4*pts*w_l]   outputs of the hidden layers
  double* scrA;               // [grid][2][4*pts*maxw]     adjoints / Z-bar
  double* scrS;               // [grid][2][pts*4*out]      head outputs, seeds
  long long h_per_cta, a_per_cta;
  int pts, maxw;
  int dmma;                   // hidden-to-hidden layers on DMMA.8x8x4 (default); 0: plain DFMA everywhere (PINN_GENERIC_DFMA=1)
  double* partials;           // [grid][pstride]: [grad p_net | dl1 dl2 - part0 part1 part2]
  int pstride;
  const int* run_flag;
  // PINN_POLY_INF (8) / PINN_POLY_IDE (9), read only by fused_loss_grad<true>: the residual's term table, and the source s at
  // the residual points [n_c] (nullptr: s = 0)
  PolySpec poly;
  const double* src;
};

// Polynomial residual head (DESIGN 4.4d): f = sum_k c_k kappa_k u^a u_x^b u_t^c u_xx^d - s.  A stream's power v^e and its
// derivative e v^(e-1) are picked from the powers formed once per point, never by dividing by v (u may be 0).
__device__ __forceinline__ double pick_pow(double v, double v2, double v3, int e) {
  return e == 0 ? 1.0 : (e == 1 ? v : (e == 2 ? v2 : v3));
}
__device__ __forceinline__ double pick_dpow(double v, double v2, int e) {
  return e == 0 ? 0.0 : (e == 1 ? 1.0 : (e == 2 ? 2.0 * v : 3.0 * v2));
}

// ---- DMMA.8x8x4 building block for the hidden layers: operands straight from global memory (the per-CTA scratch is L1/L2
// resident, the weights come through the read-only path); no shared-memory staging, so it works for any width.
constexpr int NTW = 4;                       // N tiles (of 8 columns) per work item

// C[s][j] += A_s[8 rows x K] * B[K x 8 columns of tile j],  s = 4 streams sharing the B fragments.
//   A_s(row g, k) = arow[s * sstride + k]  (arow already points at this lane's row);  B(k, n) = B[k * ldk + n * ldn]
// k >= K / n >= N contribute zero through B (the A address is clamped, its value is finite).
__device__ __forceinline__ void dmma_rows(double (&C)[4][NTW][2], const double* arow, size_t sstride, int K, const double* B,
                                          size_t ldk, size_t ldn, int n0, int N, int ntn, int g, int q) {
  const double* bp[NTW];
  bool bok[NTW];
#pragma unroll
  for (int j = 0; j < NTW; j++) {
    const int n = n0 + 8 * j + g;
    bok[j] = j < ntn && n < N;
    bp[j] = B + (size_t)(n < N ? n : N - 1) * ldn;
  }
  const double* ap = arow + q;
  const int kfull = K >> 2;
  // full k-steps: no guard on k
#pragma unroll 4
  for (int ks = 0; ks < kfull; ks++) {
    double a[4], b[NTW];
#pragma unroll
    for (int st = 0; st < 4; st++) a[st] = ap[st * sstride + 4 * ks];
#pragma unroll
    for (int j = 0; j < NTW; j++) b[j] = bok[j] ? __ldg(bp[j] + (size_t)(4 * ks + q) * ldk) : 0.0;
#pragma unroll
    for (int j = 0; j < NTW; j++)
      if (j < ntn) {
#pragma unroll
        for (int st = 0; st < 4; st++) dmma(C[st][j], a[st], b[j]);
      }
  }
  if (K & 3) {
    const int k = 4 * kfull + q;
    const bool kok = k < K;
    const int kc = kok ? k : K - 1;
    double a[4], b[NTW];
#pragma unroll
    for (int st = 0; st < 4; st++) a[st] = arow[st * sstride + kc];
#pragma unroll
    for (int j = 0; j < NTW; j++) b[j] = (bok[j] && kok) ? __ldg(bp[j] + (size_t)kc * ldk) : 0.0;
#pragma unroll
    for (int j = 0; j < NTW; j++)
      if (j < ntn) {
#pragma unroll
        for (int st = 0; st < 4; st++) dmma(C[st][j], a[st], b[j]);
      }
  }
}

// work items are handed out through a shared-memory counter (every output element is produced by exactly one warp in a
// fixed summation order, so the result does not depend on which warp takes which item)
__device__ __forceinline__ int next_item(int* ctr, int lane) {
  int it = 0;
  if (lane == 0) it = atomicAdd(ctr, 1);
  return __shfl_sync(0xffffffffu, it, 0);
}

__device__ __forceinline__ void block_reduce_store(double v, double* red, double* dst) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < THREADS / 32; i++) s += red[i];
    *dst = s;
  }
}

// Discrete-time IRK heads (pde 3..6), out of line: this code runs once per evaluation, and inlined it would take registers
// from the hidden-layer loops.  Returns (part0, part1, d/d lambda_1, d/d lambda_2) of this thread.
struct HeadSums { double part0, part1, gl1, gl2; };
struct DiscArgs { const double* irk; const double* tgt; long long n_d, n0p; double dt, nu, kc; int pde; };
__device__ __noinline__ HeadSums disc_head(const DiscArgs p, int npts, int out, long long base, const double* OUTV, double* SEED,
                                          double* NB, double* RB, double l1, double kap) {
  const int tid = threadIdx.x, lane = tid & 31;
  double part0 = 0.0, part1 = 0.0, gl1 = 0.0, gl2 = 0.0;
  // Discrete-time IRK heads.  OUTV[pt] = [U (out) | U_x | (t: 0; KdV: U_xxx) | U_xx].
  // pde 3, inference (1d-burgers/inf_disc_burgers.py:61-101), out = q+1:
  //   N_j = U_j U_x,j - nu U_xx,j (j < q);  U_0,k = U_k + dt sum_j N_j IRK[k][j];  loss = sum (U_0 - u_0)^2 on the data
  //   points + sum U^2 on the boundary points.
  // pde 4, identification (1d-burgers/ide_disc_burgers.py:81-115), out = q, two snapshots [x_0 (n_d) | x_1]:
  //   N_j = l1 U_j U_x,j - e^{l2} U_xx,j;  snapshot s: pred_k = U_k + dt sum_j N_j M_s[k][j] with M_0 = alpha and
  //   M_1 = -(beta - alpha) (the sign of N' = -N folded into the matrix);  loss = sum (pred - u_s)^2 over points and stages.
  // pde 5, KdV identification: as pde 4 with N_j = l1 U_j U_x,j + e^{l2} U_xxx,j (third-order mode).
  // pde 6, Allen-Cahn inference: as pde 3 with N_j = k U_j^3 - k U_j - d U_xx,j; the boundary term is the periodic pair
  //   (lb, ub) at [n0p, n0p + 2): sum_k (U_k(lb) - U_k(ub))^2 + (U_x,k(lb) - U_x,k(ub))^2 over all q+1 outputs.
  // Scratch: NB[pt][q] (N, then N-bar), RB[pt][out] (2 x residual).
  const bool kdv = p.pde == 5, ac = p.pde == 6;
  const bool idd = p.pde == 4 || kdv;
  const int q = idd ? out : out - 1;
  for (int idx = tid; idx < npts * q; idx += THREADS) {
    const int pt = idx / q, j = idx - pt * q;
    const double* o = OUTV + (size_t)pt * 4 * out;
    if (kdv) NB[idx] = fma(l1 * o[j], o[out + j], kap * o[2 * out + j]);
    else if (ac) NB[idx] = fma(p.kc * o[j], o[j] * o[j], -p.kc * o[j]) - p.nu * o[3 * out + j];
    else NB[idx] = l1 * o[j] * o[out + j] - kap * o[3 * out + j];       // inference: l1 = 1, kap = nu
  }
  __syncthreads();
  // (i) stage products  S[pt][k] = sum_j N[pt][j] M_pt[k][j]  -> RB.  One warp per (point, stage), lanes over j: the rows of the
  // stage matrix are read coalesced and all 16 loads of a lane are in flight at once (q <= 512).  (Round 1: a thread per
  // (point, stage) walking its own row -- 41 % of this model's step.)
  for (int it = tid >> 5; it < npts * out; it += THREADS / 32) {
    const int pt = it / out, k = it - pt * out;
    const long long gp = base + pt;
    if (idd || gp < p.n_d) {
      const double* nrow = NB + (size_t)pt * q;
      const double* irow = p.irk + ((idd && gp >= p.n_d) ? (size_t)q * q : 0) + (size_t)k * q;
      double mv[16], nv[16];
#pragma unroll
      for (int c = 0; c < 16; c++) {
        const int j = lane + 32 * c;
        mv[c] = j < q ? __ldg(irow + j) : 0.0;
        nv[c] = j < q ? nrow[j] : 0.0;
      }
      double acc = 0.0;
#pragma unroll
      for (int c = 0; c < 16; c++) acc = fma(nv[c], mv[c], acc);
      acc = warp_sum(acc);
      if (lane == 0) RB[it] = acc;
    }
  }
  __syncthreads();
  for (int idx = tid; idx < npts * out; idx += THREADS) {
    const int pt = idx / out, k = idx - pt * out;
    const long long gp = base + pt;
    const double uk = OUTV[(size_t)pt * 4 * out + k];
    if (idd || gp < p.n_d) {
      const bool second = idd && gp >= p.n_d;
      const double r = fma(p.dt, RB[idx], uk) - __ldg(p.tgt + gp);  // targets: [u_0 | u_1]
      if (second) part1 = fma(r, r, part1); else part0 = fma(r, r, part0);
      RB[idx] = 2.0 * r;
    } else if (ac) {
      // periodic pair: lb at an even offset from n0p, its ub partner next to it in the same CTA (pts and n0p are even)
      double dv = 0.0;
      if (gp >= p.n0p) {
        const bool is_lb = ((gp - p.n0p) & 1) == 0;
        const double* o = OUTV + (size_t)pt * 4 * out;
        const double* op = o + (is_lb ? 4 * out : -4 * out);
        dv = o[k] - op[k];
        const double dx = o[out + k] - op[out + k];
        if (is_lb) part1 = fma(dv, dv, fma(dx, dx, part1));
      }
      RB[idx] = 2.0 * dv;                  // 0 on the alignment pad
    } else {
      part1 = fma(uk, uk, part1);
      RB[idx] = 2.0 * uk;                  // boundary point: d/dU of sum U^2
    }
  }
  __syncthreads();
  // (ii) N-bar[pt][j] = dt sum_k RB[pt][k] M_pt[k][j]: thread per (point, column j) (coalesced over j), the k loop unrolled so
  // that 16 independent matrix loads are in flight per thread
  for (int idx = tid; idx < npts * q; idx += THREADS) {
    const int pt = idx / q, j = idx - pt * q;
    const long long gp = base + pt;
    double acc = 0.0;
    if (idd || gp < p.n_d) {
      const double* rrow = RB + (size_t)pt * out;
      const double* mcol = p.irk + ((idd && gp >= p.n_d) ? (size_t)q * q : 0) + j;
      double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
      int k = 0;
      for (; k + 16 <= out; k += 16) {
        double mv[16];
#pragma unroll
        for (int c = 0; c < 16; c++) mv[c] = __ldg(mcol + (size_t)(k + c) * q);
#pragma unroll
        for (int c = 0; c < 16; c += 4) {
          a0 = fma(rrow[k + c], mv[c], a0);
          a1 = fma(rrow[k + c + 1], mv[c + 1], a1);
          a2 = fma(rrow[k + c + 2], mv[c + 2], a2);
          a3 = fma(rrow[k + c + 3], mv[c + 3], a3);
        }
      }
      for (; k < out; k++) a0 = fma(rrow[k], __ldg(mcol + (size_t)k * q), a0);
      acc = ((a0 + a1) + (a2 + a3)) * p.dt;
    }
    NB[idx] = acc;                          // N-bar (0 on boundary points)
  }
  __syncthreads();
  for (int idx = tid; idx < npts * out; idx += THREADS) {
    const int pt = idx / out, k = idx - pt * out;
    const double* o = OUTV + (size_t)pt * 4 * out;
    const double nb_ = k < q ? NB[(size_t)pt * q + k] : 0.0;
    double* sdp = SEED + (size_t)pt * 4 * out;
    if (kdv) {
      sdp[k] = fma(nb_ * l1, o[out + k], RB[idx]);
      sdp[out + k] = nb_ * l1 * o[k];
      sdp[2 * out + k] = kap * nb_;
      sdp[3 * out + k] = 0.0;
      gl1 = fma(nb_ * o[k], o[out + k], gl1);
      gl2 = fma(kap * nb_, o[2 * out + k], gl2);
    } else if (ac) {
      const long long gp = base + pt;
      double sx = 0.0;                                               // slope seed of the periodic pair: 2 (U_x - U_x(partner))
      if (gp >= p.n0p) sx = 2.0 * (o[out + k] - o[(((gp - p.n0p) & 1) == 0 ? 4 * out : -4 * out) + out + k]);
      sdp[k] = fma(nb_, fma(3.0 * p.kc * o[k], o[k], -p.kc), RB[idx]);
      sdp[out + k] = sx;
      sdp[2 * out + k] = 0.0;
      sdp[3 * out + k] = -p.nu * nb_;
    } else {
      sdp[k] = fma(nb_ * l1, o[out + k], RB[idx]);
      sdp[out + k] = nb_ * l1 * o[k];
      sdp[2 * out + k] = 0.0;
      sdp[3 * out + k] = -kap * nb_;
      gl1 = fma(nb_ * o[k], o[out + k], gl1);                       // d/d lambda_1, d/d lambda_2 (raw); unused for pde 3
      gl2 = fma(-kap * nb_, o[3 * out + k], gl2);
    }
  }
  __syncthreads();
  return {part0, part1, gl1, gl2};
}

// POLY = false: the hard-wired heads (pde 0..6).  POLY = true: the polynomial residual head (pde 8, 9) in an instantiation of
// its own, so the code of the hard-wired models does not change with it.
template <bool POLY>
__global__ void __launch_bounds__(THREADS, 2) fused_loss_grad(const Args p) {
  __shared__ double red[THREADS / 32];
  __shared__ int work_ctr;
  if (p.run_flag && *p.run_flag != 0) return;
  const int tid = threadIdx.x, lane = tid & 31;
  const int g = lane >> 2, q = lane & 3;
  const NetDesc& nd = p.nd;
  const int L = nd.n_layers;                 // Dense layers; hidden 0..L-2, head L-1
  const int out = nd.dims[L];
  const int pts = p.pts;
  const long long base = (long long)blockIdx.x * pts;
  const long long navail = p.n_total - base;
  const int npts = navail <= 0 ? 0 : (navail < pts ? (int)navail : pts);
  double* Hs = p.scrH + (size_t)blockIdx.x * p.h_per_cta;
  double* A0 = p.scrA + (size_t)blockIdx.x * 2 * p.a_per_cta;
  double* A1 = A0 + p.a_per_cta;
  double* OUTV = p.scrS + (size_t)blockIdx.x * 2 * pts * 4 * out;
  double* SEED = OUTV + (size_t)pts * 4 * out;
  double* outp = p.partials + (size_t)blockIdx.x * p.pstride;
  const double sc0 = 2.0 / nd.dx0, sc1 = 2.0 / nd.dx1;
  const bool ide = p.pde == 1 || p.pde == 4 || p.pde == 5;
  const bool o3 = p.o3 != 0;
  const double l1 = ide ? p.w[p.p_net] : 1.0;
  const double kap = ide ? exp(p.w[p.p_net + 1]) : p.nu;

  // layer-l output slab: [4][pts][w_l]  (offsets in shared memory: a dynamically indexed per-thread array would live on the stack)
  __shared__ size_t hoff[MAXL];
  if (tid == 0) {
    size_t o = 0;
    for (int l = 0; l < L - 1; l++) { hoff[l] = o; o += (size_t)4 * pts * nd.dims[l + 1]; }
  }
  __syncthreads();

  // ======================================= forward: hidden layers =======================================
  for (int l = 0; l < L - 1; l++) {
    const int fi = nd.dims[l], fo = nd.dims[l + 1];
    const double* Wl = p.w + nd.woff[l];
    const double* bl = p.w + nd.boff[l];
    const double* Hp = l > 0 ? Hs + hoff[l - 1] : nullptr;
    double* Ho = Hs + hoff[l];
    const size_t sp = (size_t)pts * fi, so = (size_t)pts * fo;
    if (l > 0 && p.dmma) {
      // [4 streams x 8 points] x [fi x fo] on the tensor pipe: item = (group of 8 points, group of <= NTW column tiles)
      const int nt = (fo + 7) >> 3, ngrp = (nt + NTW - 1) / NTW, tpg = (nt + ngrp - 1) / ngrp;
      const int items = ((npts + 7) >> 3) * ngrp;
      if (tid == 0) work_ctr = 0;
      __syncthreads();
      for (int it = next_item(&work_ctr, lane); it < items; it = next_item(&work_ctr, lane)) {
        const int pgp = it / ngrp, grp = it - pgp * ngrp;
        const int n0 = 8 * grp * tpg, ntn = min(tpg, nt - grp * tpg);
        const int pt = 8 * pgp + g, ptc = pt < npts ? pt : npts - 1;
        double C[4][NTW][2];
#pragma unroll
        for (int j = 0; j < NTW; j++)
#pragma unroll
          for (int e = 0; e < 2; e++) {
            const int u = n0 + 8 * j + 2 * q + e;
            C[0][j][e] = (j < ntn && u < fo) ? __ldg(bl + u) : 0.0;
            C[1][j][e] = C[2][j][e] = C[3][j][e] = 0.0;
          }
        dmma_rows(C, Hp + (size_t)ptc * fi, sp, fi, Wl, fo, 1, n0, fo, ntn, g, q);
        if (pt < npts) {
#pragma unroll
          for (int j = 0; j < NTW; j++)
#pragma unroll
            for (int e = 0; e < 2; e++) {
              const int u = n0 + 8 * j + 2 * q + e;
              if (j < ntn && u < fo) {
                const double a = tanh_fast(C[0][j][e]);
                const double sd = fma(-a, a, 1.0), zx = C[1][j][e];
                double* o = Ho + (size_t)pt * fo + u;
                o[0] = a;
                o[so] = sd * zx;
                o[2 * so] = sd * (o3 ? xxx_bracket(a, zx, C[3][j][e], C[2][j][e]) : C[2][j][e]);
                o[3 * so] = sd * fma(-2.0 * a * zx, zx, C[3][j][e]);
              }
            }
        }
      }
    } else
    for (int idx = tid; idx < npts * fo; idx += THREADS) {
      const int pt = idx / fo, j = idx - pt * fo;
      double z = __ldg(bl + j), zx = 0.0, zt = 0.0, zxx = 0.0;
      if (l == 0) {
        const double xh = 2.0 * (__ldg(p.x + base + pt) - nd.lb0) / nd.dx0 - 1.0;   // utils/neuralnetwork.py:29-30
        const double th = p.in_dim == 2 ? 2.0 * (__ldg(p.t + base + pt) - nd.lb1) / nd.dx1 - 1.0 : 0.0;
        const double w0 = __ldg(Wl + j), w1 = p.in_dim == 2 ? __ldg(Wl + fo + j) : 0.0;
        z = fma(xh, w0, fma(th, w1, z));
        zx = sc0 * w0;
        zt = sc1 * w1;
      } else {
        const double* h0 = Hp + (size_t)pt * fi;
        for (int i = 0; i < fi; i++) {
          const double wv = __ldg(Wl + (size_t)i * fo + j);
          z = fma(h0[i], wv, z);
          zx = fma(h0[sp + i], wv, zx);
          zt = fma(h0[2 * sp + i], wv, zt);
          zxx = fma(h0[3 * sp + i], wv, zxx);
        }
      }
      const double a = tanh_fast(z);
      const double s = fma(-a, a, 1.0);
      double* o = Ho + (size_t)pt * fo + j;
      o[0] = a;
      o[so] = s * zx;
      o[2 * so] = s * (o3 ? xxx_bracket(a, zx, zxx, zt) : zt);
      o[3 * so] = s * fma(-2.0 * a * zx, zx, zxx);
    }
    __syncthreads();
  }

  // ======================================= head + PDE terms =======================================
  const int fl = nd.dims[L - 1];                         // width of the last hidden layer
  const double* Hl = Hs + hoff[L - 2];
  const size_t sl = (size_t)pts * fl;
  const double* Wh = p.w + nd.woff[L - 1];
  for (int idx = tid; idx < npts * 4 * out; idx += THREADS) {
    const int pt = idx / (4 * out), so_ = idx - pt * 4 * out, s = so_ / out, o = so_ - s * out;
    const double* h = Hl + s * sl + (size_t)pt * fl;
    double acc = s == 0 ? __ldg(p.w + nd.boff[L - 1] + o) : 0.0;
#pragma unroll 10
    for (int i = 0; i < fl; i++) acc = fma(h[i], __ldg(Wh + (size_t)i * out + o), acc);
    OUTV[idx] = acc;
  }
  __syncthreads();
  double part0 = 0.0, part1 = 0.0, part2 = 0.0, gl1 = 0.0, gl2 = 0.0;
  if (!POLY && p.pde >= 3) {
    const DiscArgs da{p.irk, p.tgt, p.n_d, p.n0p, p.dt, p.nu, p.kc, p.pde};
    const HeadSums hs = disc_head(da, npts, out, base, OUTV, SEED, A0, A1, l1, kap);
    part0 = hs.part0; part1 = hs.part1; gl1 = hs.gl1; gl2 = hs.gl2;
    __syncthreads();
  } else
  for (int pt = tid; pt < npts; pt += THREADS) {
    const long long gp = base + pt;
    const double* o = OUTV + (size_t)pt * 4 * out;
    double sd[4 * MAXOUT];
#pragma unroll
    for (int c = 0; c < 4 * MAXOUT; c++) sd[c] = 0.0;
    if (POLY) {
      // polynomial residual (DESIGN 4.4d), BURGERS_INF / BURGERS_IDE loss structure: o = [u, u_x, u_t, u_xx]
      const bool res = gp >= p.c0 && gp < p.c0 + p.n_c;
      const double wf = res ? p.wf : 0.0;
      const bool has_d = gp >= p.d0 && gp < p.d0 + p.n_d;
      const double wd = has_d ? p.wd : 0.0;
      const double r = has_d ? o[0] - __ldg(p.tgt + (gp - p.d0)) : 0.0;
      const bool lam = p.pde == 9;                              // POLY_IDE: raw lambdas behind the net parameters
      const double l1 = lam ? p.w[p.p_net] : 0.0, l2 = lam ? p.w[p.p_net + 1] : 0.0;
      const double e1 = lam ? exp(l1) : 1.0, e2 = lam ? exp(l2) : 1.0;
      double v[4], v2[4], v3[4];
#pragma unroll
      for (int j = 0; j < 4; j++) { v[j] = o[j]; v2[j] = v[j] * v[j]; v3[j] = v2[j] * v[j]; }
      // f, df/dv_j = sum_k c_k kappa_k e_kj v_j^(e_kj - 1) prod_{i != j} v_i^e_ki, and df/d lambda_i (d e^l / dl = e^l)
      double f = 0.0, d0 = 0.0, d1 = 0.0, d2 = 0.0, d3 = 0.0, f1 = 0.0, f2 = 0.0;
      for (int k = 0; k < p.poly.n; k++) {
        const int code = p.poly.code[k];
        const int kind = code & 7, a0 = (code >> 3) & 3, a1 = (code >> 5) & 3, a2 = (code >> 7) & 3, a3 = (code >> 9) & 3;
        const double q0 = pick_pow(v[0], v2[0], v3[0], a0), q1 = pick_pow(v[1], v2[1], v3[1], a1);
        const double q2 = pick_pow(v[2], v2[2], v3[2], a2), q3 = pick_pow(v[3], v2[3], v3[3], a3);
        const double q01 = q0 * q1, q23 = q2 * q3;
        const double m = p.poly.coef[k] * (q01 * q23);
        const double kv = kind == 0 ? 1.0 : (kind == 1 ? l1 : (kind == 2 ? l2 : (kind == 3 ? e1 : e2)));
        const double ck = p.poly.coef[k] * kv;
        f = fma(kv, m, f);
        d0 = fma(ck * pick_dpow(v[0], v2[0], a0), q1 * q23, d0);
        d1 = fma(ck * pick_dpow(v[1], v2[1], a1), q0 * q23, d1);
        d2 = fma(ck * pick_dpow(v[2], v2[2], a2), q01 * q3, d2);
        d3 = fma(ck * pick_dpow(v[3], v2[3], a3), q01 * q2, d3);
        if (kind == 1 || kind == 3) f1 = fma(kind == 1 ? 1.0 : e1, m, f1);
        else if (kind != 0) f2 = fma(kind == 2 ? 1.0 : e2, m, f2);
      }
      if (res && p.src) f -= __ldg(p.src + (gp - p.c0));
      f = res ? f : 0.0;                                        // selected, not weighted by 0: see the Burgers head
      const double c = 2.0 * wf * f;
      sd[0] = fma(c, d0, 2.0 * wd * r);
      sd[1] = c * d1;
      sd[2] = c * d2;
      sd[3] = c * d3;
      part0 = fma(wd * r, r, part0);
      part2 = fma(wf * f, f, part2);
      gl1 = fma(c, f1, gl1);
      gl2 = fma(c, f2, gl2);
    } else if (p.pde != 2) {
      // Burgers (inf_cont_burgers.py:59-90 / ide_cont_burgers.py:56-91): outputs o = [u, u_x, u_t, u_xx]
      const double u = o[0], ux = o[1], ut = o[2], uxx = o[3];
      const bool res = gp >= p.c0 && gp < p.c0 + p.n_c;
      const double wf = res ? p.wf : 0.0;
      const bool has_d = gp >= p.d0 && gp < p.d0 + p.n_d;
      const double wd = has_d ? p.wd : 0.0;
      const double r = has_d ? u - __ldg(p.tgt + (gp - p.d0)) : 0.0;
      // f is selected, not weighted by 0, off the residual set: 0 * NaN or 0 * Inf would reach the data part
      const double f = res ? ut + l1 * u * ux - kap * uxx : 0.0;
      const double c = 2.0 * wf * f;
      sd[0] = fma(c * l1, ux, 2.0 * wd * r);
      sd[1] = c * l1 * u;
      sd[2] = c;
      sd[3] = -c * kap;
      part0 = fma(wd * r, r, part0);
      part2 = fma(wf * f, f, part2);
      gl1 = fma(c * u, ux, gl1);
      gl2 = fma(-c * kap, uxx, gl2);
    } else {
      // Schrodinger (inf_cont_schrodinger.py:79-129): o = [u, v, u_x, v_x, u_t, v_t, u_xx, v_xx]
      if (gp < p.n0) {
        const double ru = o[0] - __ldg(p.tgt + 2 * gp), rv = o[1] - __ldg(p.tgt + 2 * gp + 1);
        part0 += p.w0 * (ru * ru + rv * rv);
        sd[0] = 2.0 * p.w0 * ru; sd[1] = 2.0 * p.w0 * rv;
      } else if (gp < p.n0p) {
        // alignment padding: inert
      } else if (gp < p.n0p + 2 * p.nb) {
        const bool is_lb = ((gp - p.n0p) & 1) == 0;
        const double* op = is_lb ? o + 8 : o - 8;
        const double sgn = is_lb ? 1.0 : -1.0;
        double acc = 0.0;
#pragma unroll
        for (int c = 0; c < 4; c++) {
          const double d = sgn * (o[c] - op[c]);
          acc = fma(d, d, acc);
          sd[c] = sgn * 2.0 * p.wb * d;
        }
        if (is_lb) part1 += p.wb * acc;
      } else {
        const double u = o[0], v = o[1], ut = o[4], vt = o[5], uxx = o[6], vxx = o[7];
        const double h2 = u * u + v * v;
        const double fu = ut + 0.5 * vxx + h2 * v;
        const double fv = vt - 0.5 * uxx - h2 * u;
        part2 += p.wf * (fu * fu + fv * fv);
        const double cu = 2.0 * p.wf * fu, cv = 2.0 * p.wf * fv;
        sd[0] = cu * 2.0 * u * v - cv * (3.0 * u * u + v * v);
        sd[1] = cu * (u * u + 3.0 * v * v) - cv * 2.0 * u * v;
        sd[4] = cu; sd[5] = cv;
        sd[6] = -0.5 * cv; sd[7] = 0.5 * cu;
      }
    }
#pragma unroll
    for (int c = 0; c < 4 * MAXOUT; c++)
      if (c < 4 * out) SEED[(size_t)pt * 4 * out + c] = sd[c];
  }
  block_reduce_store(part0, red, outp + p.p_net + 3);
  block_reduce_store(part1, red, outp + p.p_net + 4);
  block_reduce_store(part2, red, outp + p.p_net + 5);
  block_reduce_store(gl1, red, outp + p.p_net + 0);
  block_reduce_store(gl2, red, outp + p.p_net + 1);
  __syncthreads();

  // ======================================= head: gradient and input adjoint =======================================
  for (int e = tid; e < (fl + 1) * out; e += THREADS) {
    const int i = e / out, o = e - i * out;
    double acc = 0.0;
    for (int pt = 0; pt < npts; pt++) {
      const double* sd = SEED + (size_t)pt * 4 * out;
      if (i < fl) {
#pragma unroll
        for (int s = 0; s < 4; s++) acc = fma(Hl[s * sl + (size_t)pt * fl + i], sd[s * out + o], acc);
      } else {
        acc += sd[o];
      }
    }
    if (i < fl) outp[nd.woff[L - 1] + i * out + o] = acc;
    else outp[nd.boff[L - 1] + o] = acc;
  }
  double* Acur = A0;      // adjoint of the current layer's outputs: [4][pts][w]
  double* Aoth = A1;
  if (out >= 64) {
    // wide heads (discrete-time models: out = q or q+1): a warp per (point, unit), lanes over the outputs -- coalesced rows of
    // the head weights, all loads of a lane in flight at once (out <= 512), four stream sums reduced by shuffles
    for (int it = tid >> 5; it < npts * fl; it += THREADS / 32) {
      const int pt = it / fl, i = it - pt * fl;
      const double* sd = SEED + (size_t)pt * 4 * out;
      const double* wr = Wh + (size_t)i * out;
      double a4[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll 4
      for (int c = 0; c < 16; c++) {
        const int o = lane + 32 * c;
        if (o < out) {
          const double wv = __ldg(wr + o);
#pragma unroll
          for (int s = 0; s < 4; s++) a4[s] = fma(sd[s * out + o], wv, a4[s]);
        }
      }
#pragma unroll
      for (int s = 0; s < 4; s++) {
        const double v = warp_sum(a4[s]);
        if (lane == 0) Acur[s * sl + (size_t)pt * fl + i] = v;
      }
    }
  } else
  for (int idx = tid; idx < npts * fl; idx += THREADS) {
    const int pt = idx / fl, i = idx - pt * fl;
    const double* sd = SEED + (size_t)pt * 4 * out;
#pragma unroll
    for (int s = 0; s < 4; s++) {
      double acc = 0.0;
      for (int o = 0; o < out; o++) acc = fma(sd[s * out + o], __ldg(Wh + (size_t)i * out + o), acc);
      Acur[s * sl + (size_t)pt * fl + i] = acc;
    }
  }
  __syncthreads();

  // ======================================= backward: hidden layers =======================================
  for (int l = L - 2; l >= 0; l--) {
    const int fi = nd.dims[l], fo = nd.dims[l + 1];
    const double* Wl = p.w + nd.woff[l];
    const double* Ho = Hs + hoff[l];
    const double* Hp = l > 0 ? Hs + hoff[l - 1] : nullptr;
    const size_t so = (size_t)pts * fo, sp = (size_t)pts * fi;
    // the layer inputs were written a whole forward pass ago: start pulling them towards L2 for the weight gradient below
    if (l > 0 && p.dmma && tid == 0) {
      const size_t bytes = (size_t)4 * pts * fi * 8;
      for (size_t o = 0; o < bytes; o += 65536) prefetch_l2_bulk(reinterpret_cast<const char*>(Hp) + o, (uint32_t)min((size_t)65536, bytes - o));
    }
    // (1) Z-bar
    if (p.o3) {
      // third-order mode (t slot = xxx stream: at = a_xxx, Bt its adjoint), in layer outputs the t-stream formula plus
      //   Z += -6 a_x a_xx Bt,  Z_x += -6 u2 Bt,  Z_xx += -6 a a_x Bt;  Z_xxx = s Bt
      for (int idx = tid; idx < npts * fo; idx += THREADS) {
        const size_t q = idx;
        const double a = Ho[q], ax = Ho[so + q], at = Ho[2 * so + q], axx = Ho[3 * so + q];
        const double B0 = Acur[q], Bx = Acur[so + q], Bt = Acur[2 * so + q], Bxx = Acur[3 * so + q];
        const double s = fma(-a, a, 1.0);
        const double u1 = fma(ax, Bx, at * Bt);
        const double u2 = fma(a, axx, ax * ax);
        double z = fma(-2.0 * a, u1, s * B0);
        z = fma(-2.0 * Bxx, u2, z);
        Aoth[q] = fma(-6.0 * ax * axx, Bt, z);
        Aoth[so + q] = fma(-6.0 * u2, Bt, fma(-4.0 * a * ax, Bxx, s * Bx));
        Aoth[2 * so + q] = s * Bt;
        Aoth[3 * so + q] = fma(-6.0 * a * ax, Bt, s * Bxx);
      }
    } else
    for (int idx = tid; idx < npts * fo; idx += THREADS) {
      const size_t q = idx;                               // == pt*fo + j
      const double a = Ho[q], ax = Ho[so + q], at = Ho[2 * so + q], axx = Ho[3 * so + q];
      const double B0 = Acur[q], Bx = Acur[so + q], Bt = Acur[2 * so + q], Bxx = Acur[3 * so + q];
      const double s = fma(-a, a, 1.0);
      const double u1 = fma(ax, Bx, at * Bt);
      const double u2 = fma(a, axx, ax * ax);
      double z = fma(-2.0 * a, u1, s * B0);
      z = fma(-2.0 * Bxx, u2, z);
      Aoth[q] = z;
      Aoth[so + q] = fma(-4.0 * a * ax, Bxx, s * Bx);
      Aoth[2 * so + q] = s * Bt;
      Aoth[3 * so + q] = s * Bxx;
    }
    __syncthreads();
    if (l > 0 && p.dmma) {
      // (2)+(3) on the tensor pipe, one item list: weight-gradient items (long: K = 4 streams x points) first, then the
      // input-adjoint items.  Both only read Z-bar (Aoth), the layer inputs and W_l; the adjoint overwrites Acur.
      const int nto = (fo + 7) >> 3, ngo = (nto + NTW - 1) / NTW, tpo = (nto + ngo - 1) / ngo;     // column tiles over fo
      const int nti = (fi + 7) >> 3, ngi = (nti + NTW - 1) / NTW, tpi = (nti + ngi - 1) / ngi;     // column tiles over fi
      const int mt_w = (fi + 1 + 7) >> 3;                                                          // row tiles of [W_l ; b_l]
      const int items_w = mt_w * ngo, items = items_w + ((npts + 7) >> 3) * ngi;
      if (tid == 0) work_ctr = 0;
      __syncthreads();
      for (int it = next_item(&work_ctr, lane); it < items; it = next_item(&work_ctr, lane)) {
        if (it < items_w) {
          // G[i][j] = sum_{s, pt} Hin[s][pt][i] Z[s][pt][j];  row fi: ones on the value stream (bias)
          const int mt = it / ngo, grp = it - mt * ngo;
          const int n0 = 8 * grp * tpo, ntn = min(tpo, nto - grp * tpo);
          const int i = 8 * mt + g, ic = i < fi ? i : fi - 1;
          double G[NTW][2];
#pragma unroll
          for (int j = 0; j < NTW; j++) G[j][0] = G[j][1] = 0.0;
          int nc[NTW];
#pragma unroll
          for (int j = 0; j < NTW; j++) { const int n = n0 + 8 * j + g; nc[j] = n < fo ? n : fo - 1; }
          const int kfull = npts >> 2;
          for (int st = 0; st < 4; st++) {
            const double* hq = Hp + st * sp + ic + (size_t)q * fi;           // row pt0 + q of the layer inputs
            const double* zq = Aoth + st * so + (size_t)q * fo;              // ... and of Z-bar
            const double one = st == 0 ? 1.0 : 0.0;
            const bool bias_row = i == fi;                                   // rows beyond fi are never stored
            const double* hp = hq;
            const double* zp[NTW];
#pragma unroll
            for (int j = 0; j < NTW; j++) zp[j] = zq + nc[j];
            const size_t hs = (size_t)4 * fi, zs = (size_t)4 * fo;           // one k-step = 4 points further down
#pragma unroll 4
            for (int kk = 0; kk < kfull; kk++) {
              const double hv = *hp;
              hp += hs;
              const double a = bias_row ? one : hv;
              double b[NTW];
#pragma unroll
              for (int j = 0; j < NTW; j++) {
                b[j] = j < ntn ? *zp[j] : 0.0;
                zp[j] += zs;
              }
#pragma unroll
              for (int j = 0; j < NTW; j++)
                if (j < ntn) dmma(G[j], a, b[j]);
            }
            if (npts & 3) {
              const int pt = 4 * kfull + q;
              const bool ok = pt < npts;
              const size_t ptc = ok ? pt : npts - 1;
              const double hv = Hp[st * sp + ic + ptc * fi];
              const double a = bias_row ? one : hv;
              double b[NTW];
#pragma unroll
              for (int j = 0; j < NTW; j++) b[j] = (ok && j < ntn) ? Aoth[st * so + ptc * fo + nc[j]] : 0.0;
#pragma unroll
              for (int j = 0; j < NTW; j++)
                if (j < ntn) dmma(G[j], a, b[j]);
            }
          }
#pragma unroll
          for (int j = 0; j < NTW; j++)
#pragma unroll
            for (int e = 0; e < 2; e++) {
              const int n = n0 + 8 * j + 2 * q + e;
              if (j < ntn && n < fo) {
                if (i < fi) outp[nd.woff[l] + i * fo + n] = G[j][e];
                else if (i == fi) outp[nd.boff[l] + n] = G[j][e];
              }
            }
        } else {
          // A-bar[l-1][s][pt][i] = sum_j Z[s][pt][j] W_l[i][j]
          const int ia = it - items_w;
          const int pgp = ia / ngi, grp = ia - pgp * ngi;
          const int n0 = 8 * grp * tpi, ntn = min(tpi, nti - grp * tpi);
          const int pt = 8 * pgp + g, ptc = pt < npts ? pt : npts - 1;
          double C[4][NTW][2];
#pragma unroll
          for (int st = 0; st < 4; st++)
#pragma unroll
            for (int j = 0; j < NTW; j++) C[st][j][0] = C[st][j][1] = 0.0;
          dmma_rows(C, Aoth + (size_t)ptc * fo, so, fo, Wl, 1, fo, n0, fi, ntn, g, q);
          if (pt < npts) {
#pragma unroll
            for (int j = 0; j < NTW; j++)
#pragma unroll
              for (int e = 0; e < 2; e++) {
                const int i = n0 + 8 * j + 2 * q + e;
                if (j < ntn && i < fi) {
                  double* a = Acur + (size_t)pt * fi + i;
                  a[0] = C[0][j][e]; a[sp] = C[1][j][e]; a[2 * sp] = C[2][j][e]; a[3 * sp] = C[3][j][e];
                }
              }
          }
        }
      }
      __syncthreads();
      continue;
    }
    // (2) weight gradient: thread per entry (i, j), i == fi is the bias
    for (int e = tid; e < (fi + 1) * fo; e += THREADS) {
      const int i = e / fo, j = e - i * fo;
      double acc = 0.0;
      for (int pt = 0; pt < npts; pt++) {
        const double* z = Aoth + (size_t)pt * fo + j;
        if (i == fi) {
          acc += z[0];
        } else if (l == 0) {
          const double xh = 2.0 * (__ldg(p.x + base + pt) - nd.lb0) / nd.dx0 - 1.0;
          const double th = p.in_dim == 2 ? 2.0 * (__ldg(p.t + base + pt) - nd.lb1) / nd.dx1 - 1.0 : 0.0;
          acc += i == 0 ? fma(xh, z[0], sc0 * z[so]) : fma(th, z[0], sc1 * z[2 * so]);
        } else {
          const double* h = Hp + (size_t)pt * fi + i;
          acc = fma(h[0], z[0], acc);
          acc = fma(h[sp], z[so], acc);
          acc = fma(h[2 * sp], z[2 * so], acc);
          acc = fma(h[3 * sp], z[3 * so], acc);
        }
      }
      if (i < fi) outp[nd.woff[l] + i * fo + j] = acc;
      else outp[nd.boff[l] + j] = acc;
    }
    // (3) input adjoint (overwrites the adjoint of this layer's outputs, which is no longer needed)
    __syncthreads();
    if (l > 0) {
      for (int idx = tid; idx < npts * fi; idx += THREADS) {
        const int pt = idx / fi, i = idx - pt * fi;
        const double* z = Aoth + (size_t)pt * fo;
        double b0 = 0.0, bx = 0.0, bt = 0.0, bxx = 0.0;
        for (int j = 0; j < fo; j++) {
          const double wv = __ldg(Wl + (size_t)i * fo + j);
          b0 = fma(z[j], wv, b0);
          bx = fma(z[so + j], wv, bx);
          bt = fma(z[2 * so + j], wv, bt);
          bxx = fma(z[3 * so + j], wv, bxx);
        }
        double* a = Acur + (size_t)pt * fi + i;
        a[0] = b0; a[sp] = bx; a[2 * sp] = bt; a[3 * sp] = bxx;
      }
      __syncthreads();
    }
  }
  if (tid == 0) outp[p.p_net + 2] = 0.0;
}

}  // namespace generic
}  // namespace pinn
