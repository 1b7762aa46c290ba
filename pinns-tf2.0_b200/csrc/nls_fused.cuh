// Fused nonlinear-Schrodinger PINN loss + gradient kernel for the [2, 100 x 4, 2] tanh MLP, fp64, sm_90a.
//
// Replaces (reference file:line): 1dcomplex-schrodinger/inf_cont_schrodinger.py:60-76 (uvx_model), :79-105 (f_model),
// :107-129 (loss: mse_0 + mse_b + mse_f), and the outer tape of utils/neuralnetwork.py:55-59.
//
// One launch, one persistent CTA per SM.  The 100x100 fp64 weight matrices (80 KB each, 246 KB in total) do not fit
// in shared memory together, so a CTA owns a contiguous block of points and walks the network LAYER BY LAYER:
//   F0        layer 0 (2 -> 100), direct;                              outputs -> scratch H[0]
//   F1..F3    W_l staged once per pass with ONE TMA bulk copy; 16-point rounds of H[l-1] stream in through
//             cp.async (double buffered); DMMA GEMM [64 rows x 100] x [100 x 100]; tanh + Taylor streams in the
//             epilogue;                                                outputs -> scratch H[l]
//   OUT       (head outputs come out of the F3 epilogue) residuals f_u, f_v, initial/boundary terms, loss parts, seeds
//   B3..B1    per round: Z-bar[l] (activation adjoint of layer l, from scratch) and H[l-1] stream in through cp.async;
//             input adjoint A-bar[l-1] = Z-bar W_l^T (DMMA) stays in registers and is turned into Z-bar[l-1] in the
//             epilogue with the H[l-1] values of the staged slab -> scratch (so A-bar never round-trips through global
//             memory and H[l] is not re-read);  weight gradient G_l += H[l-1]^T Z-bar (DMMA, K = 64 rows per round).
//             The 13x13 output tiles of G_l are OWNED by warps, so their accumulators stay in registers for the whole
//             pass over the CTA's points and are written once (bias gradient = virtual ones-row 100).
//             The l = 3 pass stages H[3] instead and turns it into Z-bar[3] IN the slab (seeds x head weights, one block
//             barrier more per round), accumulating the head gradient from the same shared-memory values.
//   B0        layer-0 gradient from Z-bar[0], direct.
// The activations (4 streams x 100 units x 4 layers = 12.8 KB per point) live in a per-CTA global scratch that is
// streamed, not re-read: algorithmic HBM traffic is 16 B/point, implementation traffic ~67 KB/point (DESIGN.md 4.5).
//
// Point list: [initial-condition points n0 | boundary pairs (lb_k, ub_k) interleaved, 2 nb | collocation nc].
// Every point is carried with 4 streams (value, x, t, xx); only the seeds differ.
#pragma once
#include "pinn_common.cuh"

namespace pinn {
namespace nls {

constexpr int W = 100;                // hidden width
constexpr int NT = 13;                // N tiles of 8 (104)
constexpr int KS = 25;                // k-steps of 4
constexpr int P_NET = 30802;
constexpr int WPAD = 30816;
constexpr int PSTRIDE = 30816;        // [P_NET grad | mse_0, mse_b, mse_f | pad]
constexpr int IDX_L0 = 30802, IDX_LB = 30803, IDX_LF = 30804;
constexpr int THREADS = 256;
constexpr int WARPS = 8;
constexpr int RPTS = 16;              // points per round
constexpr int RROWS = 4 * RPTS;       // 64 rows per round
constexpr int SLAB = RROWS * W;       // doubles per staged round tile (51.2 KB)

__host__ __device__ constexpr int woff(int l) { return l == 0 ? 0 : (l <= 3 ? 300 + (l - 1) * 10100 : 30600); }
__host__ __device__ constexpr int boff(int l) { return l == 0 ? 200 : (l <= 3 ? 300 + (l - 1) * 10100 + 10000 : 30800); }

// shared memory (doubles): W_l | two staging slabs | barrier
constexpr int SM_W = 0;
constexpr int SM_S0 = SM_W + W * W;
constexpr int SM_S1 = SM_S0 + SLAB;
constexpr int SM_RED = SM_S1 + SLAB;
constexpr int SM_W4 = SM_RED + 64;          // head weights W_4 (100 x 2)
constexpr int SM_HO = SM_W4 + 2 * W;        // head-output partials of a forward round: [2 (round parity)][4 warps][16 points][8]
constexpr int SM_GH = SM_HO + 2 * 4 * RPTS * 8;   // head-gradient accumulators [2 point halves][2 outputs][128 units]
constexpr int SM_BAR = SM_GH + 2 * 2 * 128;
constexpr int SM_DOUBLES = SM_BAR + 8;    // mbarriers: weights, slab S0, slab S1 (forward); Z lo, Z hi, H, lo-halves-free (backward)
constexpr int SMEM_BYTES = SM_DOUBLES * 8;     // 182,928 B

inline int grid_size(int n_sm) { return n_sm; }

struct Args {
  const double* w;
  const double* x;
  const double* t;
  const double* uv0;        // [n0][2]
  long long n_total, n0, n0p, nb, nc;   // n0p: n0 rounded up to even (start of the boundary-pair block)
  double w0, wb, wf;        // aux/n0, aux/nb, 1/nc_global
  double lb0, lb1, dx0, dx1;
  double* scratchH;         // [grid][4 layers][4 streams][pts][W]
  double* scratchA;         // [grid][2 buffers][4 streams][pts][W]
  double* scratchS;         // [grid][pts][8]  seeds (u,v | u_x,v_x | u_t,v_t | u_xx,v_xx)
  int pts;                  // points per CTA (multiple of 16)
  double* partials;         // [grid][PSTRIDE]
  const int* run_flag;
};

__device__ __forceinline__ int prow(int g) { return (g & 4) | ((g & 1) << 1) | ((g & 2) >> 1); }

// stage one round (16 points x 4 streams x 100 units) of a scratch layer [4][pts][W] into a slab [64 rows][W],
// row = 16*s + p.  Each stream block is contiguous on both sides (12 800 B): four TMA bulk copies completing on one
// mbarrier, issued by ONE thread (the per-thread cp.async form cost 19 k instructions per warp, 2/3 of the DMMA count).
__device__ __forceinline__ void stage_round_tma(double* slab, const double* src, int pts, int p0, uint64_t* bar) {
  mbar_expect_tx(bar, RROWS * W * 8);
#pragma unroll
  for (int s = 0; s < 4; s++) tma_bulk_g2s(slab + 16 * s * W, src + ((size_t)s * pts + p0) * W, RPTS * W * 8, bar);
}

// half a round: streams 2*half, 2*half+1 (rows 32*half .. 32*half+31 of the slab)
__device__ __forceinline__ void stage_half_tma(double* slab, const double* src, int pts, int p0, int half, uint64_t* bar) {
  mbar_expect_tx(bar, RROWS * W * 4);
#pragma unroll
  for (int s = 2 * half; s < 2 * half + 2; s++) tma_bulk_g2s(slab + 16 * s * W, src + ((size_t)s * pts + p0) * W, RPTS * W * 8, bar);
}

// warp -> (point group, N tiles) for the row-parallel GEMMs (forward, input adjoint): 2 groups x 13 tiles over 8 warps;
// the 4-tile warp sits on a different sub-partition in each group (loads 7,7,6,6).
__device__ __forceinline__ void gemm_role(int warp, int& pg, int& nt0, int& ntn) {
  pg = warp >> 2;
  const int k = warp & 3;
  if (pg == 0) { nt0 = k == 0 ? 0 : 3 * k + 1; ntn = k == 0 ? 4 : 3; }
  else { nt0 = k == 0 ? 0 : (k == 1 ? 3 : 3 * k + 1); ntn = k == 1 ? 4 : 3; }
}

// C[s][j][:] (+)= A(rows of group pg, streams s) * B,   B[k][n] = Wsm[k*ldk + n*ldn];  n >= 100 reads as zero
// streams S_LO .. S_HI-1 only (the backward pass runs the two stream halves separately: the second half of the slab lands
// while the first is being multiplied)
template <int S_LO = 0, int S_HI = 4>
__device__ __forceinline__ void gemm_rows(double (&C)[4][4][2], const double* slab, const double* Wsm, int ldk, int ldn,
                                          int pg, int nt0, int ntn, int lane) {
  const int g = lane >> 2, q = lane & 3;
  const int prow_g = prow(g);
#pragma unroll 5
  for (int ks = 0; ks < KS; ks++) {
    double a[4], b[4];
#pragma unroll
    for (int s = S_LO; s < S_HI; s++) a[s] = slab[(16 * s + 8 * pg + prow_g) * W + 4 * ks + q];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int n = 8 * (nt0 + j) + g;
      b[j] = (j < ntn && n < W) ? Wsm[(4 * ks + q) * ldk + n * ldn] : 0.0;
    }
#pragma unroll
    for (int j = 0; j < 4; j++)
      if (j < ntn) {
#pragma unroll
        for (int s = S_LO; s < S_HI; s++) dmma(C[s][j], a[s], b[j]);
      }
  }
}

__device__ __forceinline__ void load_weights_tma(double* Wsm, const double* src, uint64_t* bar, uint32_t& phase) {
  fence_proxy_async();                   // this thread's scratch / slab writes of the previous phase precede the TMA reads below
  __syncthreads();                       // everybody is done with the previous contents of Wsm and of the slabs
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, W * W * 8);
    tma_bulk_g2s(Wsm, src, W * W * 8, bar);
  }
  mbar_wait(bar, phase);
  phase ^= 1;
}

// activation adjoint of one tanh unit carried with its (value, x, t, xx) streams (division-free form, SURVEY Appendix A):
// outputs (a, a_x, a_t, a_xx), adjoint of the outputs (A0, Ax, At, Axx)  ->  adjoint of the pre-activation streams
__device__ __forceinline__ void zbar(double (&z)[4], double a, double ax, double at, double axx, double A0, double Ax, double At,
                                     double Axx) {
  const double s = fma(-a, a, 1.0);
  const double u1 = fma(ax, Ax, at * At);
  const double u2 = fma(a, axx, ax * ax);
  double zz = fma(-2.0 * a, u1, s * A0);
  zz = fma(-2.0 * Axx, u2, zz);
  z[0] = zz;
  z[1] = fma(-4.0 * a * ax, Axx, s * Ax);
  z[2] = s * At;
  z[3] = s * Axx;
}

// normalised coordinates of point pt of this CTA (utils/neuralnetwork.py:29-30); padded points replicate the last valid one
__device__ __forceinline__ void norm_coords(const Args& p, long long base, int npts, int npad, int pt, double& xh, double& th) {
  xh = th = 0.0;
  if (pt < npad) {
    const long long gp = base + (pt < npts ? pt : npts - 1);
    xh = 2.0 * (__ldg(p.x + gp) - p.lb0) / p.dx0 - 1.0;
    th = 2.0 * (__ldg(p.t + gp) - p.lb1) / p.dx1 - 1.0;
  }
}

__global__ void __launch_bounds__(THREADS, 1) fused_loss_grad(const Args p) {
  extern __shared__ __align__(16) double sm[];
  if (p.run_flag && *p.run_flag != 0) return;
  double* Wsm = sm + SM_W;
  double* S0 = sm + SM_S0;
  double* S1 = sm + SM_S1;
  double* red = sm + SM_RED;
  double* W4s = sm + SM_W4;
  double* HO = sm + SM_HO;
  double* GH = sm + SM_GH;
  uint64_t* bar = reinterpret_cast<uint64_t*>(sm + SM_BAR);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, q = lane & 3;
  uint64_t* bar0 = bar + 1;                // slab S0
  uint64_t* bar1 = bar + 2;                // slab S1
  uint64_t* bZl = bar + 3;                 // backward: Z-bar slab, streams 0-1 / 2-3; H slab (two half copies); lo halves free
  uint64_t* bZh = bar + 4;
  uint64_t* bH = bar + 5;
  uint64_t* bFree = bar + 6;
  uint32_t wphase = 0, ph0 = 0, ph1 = 0, phZl = 0, phZh = 0, phH = 0, phF = 0;
  if (tid == 0) {
    mbar_init(bar, 1); mbar_init(bar0, 1); mbar_init(bar1, 1);
    mbar_init(bZl, 1); mbar_init(bZh, 1); mbar_init(bH, 2); mbar_init(bFree, WARPS);
  }
  __syncthreads();

  for (int i = tid; i < 2 * W; i += THREADS) W4s[i] = __ldg(p.w + woff(4) + i);
  for (int i = tid; i < 2 * 2 * 128; i += THREADS) GH[i] = 0.0;
  const int pts = p.pts;
  const long long base = (long long)blockIdx.x * pts;              // first point of this CTA
  long long navail = p.n_total - base;
  const int npts = navail <= 0 ? 0 : (navail < pts ? (int)navail : pts);   // valid points
  const int nrounds = (npts + RPTS - 1) / RPTS;
  double* H = p.scratchH + (size_t)blockIdx.x * 16 * pts * W;      // H[l][s][pt][W]
  double* A = p.scratchA + (size_t)blockIdx.x * 8 * pts * W;       // A[buf][s][pt][W]
  double* SEED = p.scratchS + (size_t)blockIdx.x * pts * 8;
  double* outp = p.partials + (size_t)blockIdx.x * PSTRIDE;
  const double sc0 = 2.0 / p.dx0, sc1 = 2.0 / p.dx1;
  const size_t LSZ = (size_t)4 * pts * W;                          // one layer of H
  const size_t SSZ = (size_t)pts * W;                              // one stream

  // =============================== F0: layer 0 (2 -> 100), direct ===============================
  // warp per point, lanes over the units (lane, lane+32, lane+64, lane+96): the input normalisation (two fp64 divisions)
  // is evaluated once per point and warp, the layer-0 weights are per-lane constants
  {
    double w0c[4], w1c[4], bc[4];
#pragma unroll
    for (int c = 0; c < 4; c++) {
      const int u = lane + 32 * c;
      w0c[c] = u < W ? __ldg(p.w + u) : 0.0;
      w1c[c] = u < W ? __ldg(p.w + W + u) : 0.0;
      bc[c] = u < W ? __ldg(p.w + 2 * W + u) : 0.0;
    }
    const int npad0 = nrounds * RPTS;
    for (int chunk = 0; warp + WARPS * 32 * chunk < npad0; chunk++) {
      // the lanes fetch and normalise the coordinates of the warp's next 32 points in one go (no load latency per point)
      double xl, tl;
      norm_coords(p, base, npts, npad0, warp + WARPS * (32 * chunk + lane), xl, tl);
#pragma unroll 2
      for (int i = 0; i < 32; i++) {
      const int pt = warp + WARPS * (32 * chunk + i);
      if (pt >= npad0) break;
      const double xh = __shfl_sync(0xffffffffu, xl, i), th = __shfl_sync(0xffffffffu, tl, i);
#pragma unroll
      for (int c = 0; c < 4; c++) {
        const int u = lane + 32 * c;
        if (u < W) {
          const double a = tanh_fast(fma(xh, w0c[c], fma(th, w1c[c], bc[c])));
          const double s = fma(-a, a, 1.0), zx = sc0 * w0c[c], zt = sc1 * w1c[c];
          H[0 * SSZ + (size_t)pt * W + u] = a;
          H[1 * SSZ + (size_t)pt * W + u] = s * zx;
          H[2 * SSZ + (size_t)pt * W + u] = s * zt;
          H[3 * SSZ + (size_t)pt * W + u] = -2.0 * a * s * zx * zx;
        }
      }
      }
    }
  }
  __syncthreads();

  int pg, nt0, ntn;
  gemm_role(warp, pg, nt0, ntn);
  const int myp = 8 * pg + prow(g);                                 // this lane's point within a round

  // =============================== F1..F3: hidden layers ===============================
  for (int l = 1; l <= 3; l++) {
    load_weights_tma(Wsm, p.w + woff(l), bar, wphase);
    const double* Hin = H + (size_t)(l - 1) * LSZ;
    double* Hout = H + (size_t)l * LSZ;
    const double* bias = p.w + boff(l);
    if (nrounds > 0 && tid == 0) stage_round_tma(S0, Hin, pts, 0, bar0);
    for (int r = 0; r < nrounds; r++) {
      double* cur = (r & 1) ? S1 : S0;
      // the other slab was last read in round r-1 (block barrier at its end): refill it while this round computes
      if (r + 1 < nrounds && tid == 0) stage_round_tma((r & 1) ? S0 : S1, Hin, pts, (r + 1) * RPTS, (r & 1) ? bar0 : bar1);
      if (r & 1) { mbar_wait(bar1, ph1); ph1 ^= 1; } else { mbar_wait(bar0, ph0); ph0 ^= 1; }
      double C[4][4][2];
#pragma unroll
      for (int j = 0; j < 4; j++)
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const int u = 8 * (nt0 + j) + 2 * q + e;
          C[0][j][e] = (j < ntn && u < W) ? __ldg(bias + u) : 0.0;
          C[1][j][e] = C[2][j][e] = C[3][j][e] = 0.0;
        }
      gemm_rows(C, cur, Wsm, W, 1, pg, nt0, ntn, lane);
      const int pt = r * RPTS + myp;
      double ho[8] = {0, 0, 0, 0, 0, 0, 0, 0};        // l == 3: this lane's share of the head outputs out[pt][2 s + o]
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int u = 8 * (nt0 + j) + 2 * q;
        if (j < ntn && u < W) {
          double o[4][2];
#pragma unroll
          for (int e = 0; e < 2; e++) {
            const double a = tanh_fast(C[0][j][e]);
            const double s = fma(-a, a, 1.0), zx = C[1][j][e];
            o[0][e] = a;
            o[1][e] = s * zx;
            o[2][e] = s * C[2][j][e];
            o[3][e] = s * fma(-2.0 * a * zx, zx, C[3][j][e]);
          }
#pragma unroll
          for (int s = 0; s < 4; s++)
            *reinterpret_cast<double2*>(Hout + s * SSZ + (size_t)pt * W + u) = make_double2(o[s][0], o[s][1]);
          if (l == 3) {
            const double2 wa = *reinterpret_cast<const double2*>(W4s + 2 * u);          // W4[u][0..1]
            const double2 wb = *reinterpret_cast<const double2*>(W4s + 2 * u + 2);      // W4[u+1][0..1]
#pragma unroll
            for (int s = 0; s < 4; s++) {
              ho[2 * s] = fma(o[s][0], wa.x, fma(o[s][1], wb.x, ho[2 * s]));
              ho[2 * s + 1] = fma(o[s][0], wa.y, fma(o[s][1], wb.y, ho[2 * s + 1]));
            }
          }
        }
      }
      if (l == 3) {
        // head (100 -> 2) from the values still in registers: quad reduction, then one partial per warp of the point group
        double* hop = HO + (r & 1) * (4 * RPTS * 8);
#pragma unroll
        for (int c = 0; c < 8; c++) {
          ho[c] += shfl_xor_d(ho[c], 1);
          ho[c] += shfl_xor_d(ho[c], 2);
        }
        if (q == 0) {
#pragma unroll
          for (int c = 0; c < 8; c++) hop[((warp & 3) * RPTS + myp) * 8 + c] = ho[c];
        }
      }
      __syncthreads();
      if (l == 3 && tid < RPTS * 8) {
        // fixed-order sum over the four warps of a point group -> OUTV (the adjoint scratch is still unused at this point);
        // the partial buffer alternates with the round, so the next round's writers cannot overtake these reads
        const double* hop = HO + (r & 1) * (4 * RPTS * 8);
        const int pp = tid >> 3, c = tid & 7;
        double v = c < 2 ? __ldg(p.w + boff(4) + c) : 0.0;
#pragma unroll
        for (int k = 0; k < 4; k++) v += hop[(k * RPTS + pp) * 8 + c];
        A[(r * RPTS + pp) * 8 + c] = v;
      }
    }
  }

  // =============================== OUT: head (100 -> 2), residuals, seeds ===============================
  {
    // head outputs out[pt][2s+o]: written to OUTV by the F3 epilogue
    double* OUTV = A;
    __syncthreads();
    double l0 = 0.0, lbd = 0.0, lf = 0.0;
    // one thread per point; a boundary point reads its partner's outputs (pairs are adjacent and never straddle a
    // CTA: the pair block starts at the even index n0p and CTA ranges start at multiples of 16)
    for (int pt = tid; pt < nrounds * RPTS; pt += THREADS) {
      const long long gp = base + pt;
      double sd[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      const double* o = OUTV + pt * 8;
      if (pt >= npts) {
        // padding point of the last round: inert
      } else if (gp < p.n0) {                                          // initial condition (:118-119)
        const double ru = o[0] - __ldg(p.uv0 + 2 * gp), rv = o[1] - __ldg(p.uv0 + 2 * gp + 1);
        l0 += p.w0 * (ru * ru + rv * rv);
        sd[0] = 2.0 * p.w0 * ru; sd[1] = 2.0 * p.w0 * rv;
      } else if (gp < p.n0p) {
        // alignment padding between the initial-condition block and the boundary pairs: inert
      } else if (gp < p.n0p + 2 * p.nb) {                              // periodic boundary (:120-123)
        const bool is_lb = ((gp - p.n0p) & 1) == 0;
        const double* op = is_lb ? o + 8 : o - 8;                      // partner outputs
        const double sgn = is_lb ? 1.0 : -1.0;
        double acc = 0.0;
#pragma unroll
        for (int c = 0; c < 4; c++) {                                  // u, v, u_x, v_x: lb minus ub
          const double d = sgn * (o[c] - op[c]);
          acc = fma(d, d, acc);
          sd[c] = sgn * 2.0 * p.wb * d;
        }
        if (is_lb) lbd += p.wb * acc;
      } else {                                                         // collocation (:79-105)
        const double u = o[0], v = o[1], ut = o[4], vt = o[5], uxx = o[6], vxx = o[7];
        const double h2 = u * u + v * v;
        const double fu = ut + 0.5 * vxx + h2 * v;                     // :101
        const double fv = vt - 0.5 * uxx - h2 * u;                     // :102
        lf += p.wf * (fu * fu + fv * fv);
        const double cu = 2.0 * p.wf * fu, cv = 2.0 * p.wf * fv;
        sd[0] = cu * 2.0 * u * v - cv * (3.0 * u * u + v * v);
        sd[1] = cu * (u * u + 3.0 * v * v) - cv * 2.0 * u * v;
        sd[4] = cu; sd[5] = cv;
        sd[6] = -0.5 * cv; sd[7] = 0.5 * cu;
      }
#pragma unroll
      for (int c = 0; c < 8; c++) SEED[pt * 8 + c] = sd[c];
    }
    __syncthreads();
    // loss parts
    l0 = warp_sum(l0); lbd = warp_sum(lbd); lf = warp_sum(lf);
    if (lane == 0) { red[warp * 3 + 0] = l0; red[warp * 3 + 1] = lbd; red[warp * 3 + 2] = lf; }
    __syncthreads();
    if (tid < 3) {
      double s = 0.0;
      for (int w8 = 0; w8 < WARPS; w8++) s += red[w8 * 3 + tid];
      outp[IDX_L0 + tid] = s;
    }
    // head bias gradient: sum_pt seed[pt][0][o]  (the head weight gradient and Z-bar[3] are formed in the l = 3 pass below)
    if (tid < 2) {
      double gb = 0.0;
      for (int pt = 0; pt < nrounds * RPTS; pt++) gb += SEED[pt * 8 + tid];
      outp[boff(4) + tid] = gb;
    }
    __syncthreads();
  }

  // =============================== B3..B1: hidden layers, reverse ===============================
  // weight-gradient tile ownership (13 x 13 tiles of G_l): warps 0-3 own the 3 x 7 block (M tiles 3b..3b+2, N tiles 0..6),
  // warps 4-7 the 3 x 6 block (N tiles 7..12) plus a strip of the last M tile (rows 96..103: units 96-99 and the
  // ones-row 100 = bias): N tiles {0-2}, {3-5}, {6-8}, {9-12}  ->  21, 21, 21, 21, 21, 21, 21, 22 tiles.
  const int wb = warp & 3;                       // M band
  const bool wide = warp < 4;                    // 7 N tiles (else 6 + strip)
  const int n_first = wide ? 0 : 7;
  const int sn0 = 3 * wb;                        // strip: first N tile
  const int snn = wide ? 0 : (wb == 3 ? 4 : 3);  // strip: number of N tiles
  for (int l = 3; l >= 1; l--) {
    load_weights_tma(Wsm, p.w + woff(l), bar, wphase);
    const double* Hin = H + (size_t)(l - 1) * LSZ;                  // inputs of layer l: A operand of the weight gradient, and
                                                                     // the outputs the activation adjoint of layer l-1 needs
    // Z-bar[l], written by the pass above; l = 3: H[3], turned into Z-bar[3] in the slab
    const double* Zin = l == 3 ? H + (size_t)3 * LSZ : A + (size_t)(l & 1) * 4 * SSZ;
    double* Zout = A + (size_t)((l & 1) ^ 1) * 4 * SSZ;              // Z-bar[l-1]
    double G[3][7][2], GS[4][2];
#pragma unroll
    for (int m = 0; m < 3; m++)
#pragma unroll
      for (int n = 0; n < 7; n++) G[m][n][0] = G[m][n][1] = 0.0;
#pragma unroll
    for (int n = 0; n < 4; n++) GS[n][0] = GS[n][1] = 0.0;

    if (nrounds > 0 && tid == 0) {
      stage_half_tma(S1, Zin, pts, 0, 0, bZl); stage_half_tma(S1, Zin, pts, 0, 1, bZh);
      stage_half_tma(S0, Hin, pts, 0, 0, bH); stage_half_tma(S0, Hin, pts, 0, 1, bH);
    }
    for (int r = 0; r < nrounds; r++) {
      const int pt = r * RPTS + myp;
      // pull the next round's slabs towards L2 while this round computes (they are loaded into S1/S0 when the round is over)
      if (tid < 8 && r + 1 < nrounds) {
        const double* src = (tid < 4 ? Zin : Hin) + (size_t)(tid & 3) * SSZ + (size_t)(r + 1) * RPTS * W;
        prefetch_l2_bulk(src, RPTS * W * 8);
      }
      // (3) input adjoint: A-bar[l-1] = Z-bar * W_l^T   (K = units of layer l), streams 0-1 then 2-3: the lo halves of the
      // slabs were refilled in the middle of the previous round's weight gradient, the hi halves at its end
      double C[4][4][2];
#pragma unroll
      for (int s = 0; s < 4; s++)
#pragma unroll
        for (int j = 0; j < 4; j++) C[s][j][0] = C[s][j][1] = 0.0;
      mbar_wait(bZl, phZl); phZl ^= 1;
      if (l == 3) {
        // the slab holds H[3] (outputs of the last hidden layer): per (point, unit)
        //   A-bar[3][s] = sum_o seed[pt][s][o] W4[u][o]  ->  Z-bar[3] written back in place;
        //   head gradient G4[u][o] += sum_s H3[s] seed[pt][s][o]   (accumulators in shared memory, one slot per thread)
        mbar_wait(bZh, phZh); phZh ^= 1;
        const int u = tid & 127, ph = tid >> 7;
        if (u < W) {
          const double w40 = W4s[2 * u], w41 = W4s[2 * u + 1];
          double g0 = 0.0, g1 = 0.0;
#pragma unroll 2
          for (int pp = 8 * ph; pp < 8 * ph + 8; pp++) {
            const double* sdp = SEED + (size_t)(r * RPTS + pp) * 8;
            double hv[4], ab[4], z[4];
#pragma unroll
            for (int s = 0; s < 4; s++) {
              hv[s] = S1[(16 * s + pp) * W + u];
              const double s0 = sdp[2 * s], s1 = sdp[2 * s + 1];
              g0 = fma(hv[s], s0, g0);
              g1 = fma(hv[s], s1, g1);
              ab[s] = fma(s0, w40, s1 * w41);
            }
            zbar(z, hv[0], hv[1], hv[2], hv[3], ab[0], ab[1], ab[2], ab[3]);
#pragma unroll
            for (int s = 0; s < 4; s++) S1[(16 * s + pp) * W + u] = z[s];
          }
          GH[(ph * 2 + 0) * 128 + u] += g0;
          GH[(ph * 2 + 1) * 128 + u] += g1;
        }
        fence_proxy_async();                         // these generic writes precede the TMA refills of the slab
        __syncthreads();
        gemm_rows<0, 4>(C, S1, Wsm, 1, W, pg, nt0, ntn, lane);
      } else {
        gemm_rows<0, 2>(C, S1, Wsm, 1, W, pg, nt0, ntn, lane);
        mbar_wait(bZh, phZh); phZh ^= 1;
        gemm_rows<2, 4>(C, S1, Wsm, 1, W, pg, nt0, ntn, lane);
      }
      mbar_wait(bH, phH); phH ^= 1;                  // H_r (both halves)
      // (3b) Z-bar[l-1] for this lane's point and units from A-bar (registers) and H[l-1] (slab S0) -> scratch
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int u = 8 * (nt0 + j) + 2 * q;
        if (j < ntn && u < W) {
          double2 h[4];
#pragma unroll
          for (int s = 0; s < 4; s++) h[s] = *reinterpret_cast<const double2*>(S0 + (16 * s + myp) * W + u);
          double z0[4], z1[4];
          zbar(z0, h[0].x, h[1].x, h[2].x, h[3].x, C[0][j][0], C[1][j][0], C[2][j][0], C[3][j][0]);
          zbar(z1, h[0].y, h[1].y, h[2].y, h[3].y, C[0][j][1], C[1][j][1], C[2][j][1], C[3][j][1]);
#pragma unroll
          for (int s = 0; s < 4; s++)
            *reinterpret_cast<double2*>(Zout + s * SSZ + (size_t)pt * W + u) = make_double2(z0[s], z1[s]);
        }
      }
      // (4) weight gradient: G[i][j] += sum_rows S0[row][i] * S1[row][j]   (unit i == 100: ones on the value stream)
#pragma unroll 1
      for (int hf = 0; hf < 2; hf++) {
#pragma unroll 2
      for (int ks = 8 * hf; ks < 8 * hf + 8; ks++) {
        const double* ar = S0 + (4 * ks + q) * W;
        const double* br = S1 + (4 * ks + q) * W;
        double av[3], bv[7];
#pragma unroll
        for (int m = 0; m < 3; m++) av[m] = ar[8 * (3 * wb + m) + g];
#pragma unroll
        for (int n = 0; n < 7; n++) {
          const int ju = 8 * (n_first + n) + g;
          bv[n] = ((n < 6 || wide) && ju < W) ? br[ju] : 0.0;
        }
#pragma unroll
        for (int m = 0; m < 3; m++) {
#pragma unroll
          for (int n = 0; n < 6; n++) dmma(G[m][n], av[m], bv[n]);
          if (wide) dmma(G[m][6], av[m], bv[6]);
        }
        if (!wide) {
          const int iu = 96 + g;
          const double as = iu < W ? ar[iu] : ((iu == W && ks < 4) ? 1.0 : 0.0);   // rows 0..15 are the value stream
#pragma unroll
          for (int n = 0; n < 4; n++) {
            if (n < snn) {
              const int ju = 8 * (sn0 + n) + g;
              dmma(GS[n], as, ju < W ? br[ju] : 0.0);
            }
          }
        }
      }
        if (hf == 0) {
          // rows 0..31 (streams 0-1) of both slabs are dead once every warp is past them: refill them now
          if (lane == 0) mbar_arrive(bFree);
          if (tid == 0) {
            if (r + 1 < nrounds) {
              mbar_wait(bFree, phF);
              stage_half_tma(S1, Zin, pts, (r + 1) * RPTS, 0, bZl);
              stage_half_tma(S0, Hin, pts, (r + 1) * RPTS, 0, bH);
            }
            phF ^= 1;
          }
        }
      }
      __syncthreads();                               // the hi halves are free
      if (r + 1 < nrounds && tid == 0) {
        stage_half_tma(S1, Zin, pts, (r + 1) * RPTS, 1, bZh);
        stage_half_tma(S0, Hin, pts, (r + 1) * RPTS, 1, bH);
      }
    }
    if (l == 3) {
      // head weight gradient: the two point halves in a fixed order (the last round's barrier ordered the accumulators)
      for (int i = tid; i < 2 * W; i += THREADS) {
        const int u = i >> 1, o = i & 1;
        outp[woff(4) + i] = GH[(0 * 2 + o) * 128 + u] + GH[(1 * 2 + o) * 128 + u];
      }
    }
    // (5) flush this warp's tiles of G_l
#pragma unroll
    for (int m = 0; m < 3; m++) {
      const int iu = 8 * (3 * wb + m) + g;                   // < 96
#pragma unroll
      for (int n = 0; n < 7; n++) {
        if (n < 6 || wide) {
#pragma unroll
          for (int e = 0; e < 2; e++) {
            const int ju = 8 * (n_first + n) + 2 * q + e;
            if (ju < W) outp[woff(l) + iu * W + ju] = G[m][n][e];
          }
        }
      }
    }
    if (!wide) {
      const int iu = 96 + g;
#pragma unroll
      for (int n = 0; n < 4; n++) {
        if (n < snn) {
#pragma unroll
          for (int e = 0; e < 2; e++) {
            const int ju = 8 * (sn0 + n) + 2 * q + e;
            if (ju < W) {
              if (iu < W) outp[woff(l) + iu * W + ju] = GS[n][e];
              else if (iu == W) outp[boff(l) + ju] = GS[n][e];
            }
          }
        }
      }
    }
  }

  // =============================== B0: layer-0 gradient, direct ===============================
  __syncthreads();
  {
    // warp w takes the points pt = w, w+8, ...; lane covers units lane, lane+32, lane+64, lane+96 (coalesced rows);
    // many independent loads in flight per thread, then a fixed-order combine over the 8 warps.
    const double* Z0 = A;                                  // Z-bar[0]: scratch buffer 0, written by the l = 1 pass
    double gx[4] = {0, 0, 0, 0}, gt[4] = {0, 0, 0, 0}, gb[4] = {0, 0, 0, 0};
    const int npad = nrounds * RPTS;
    for (int chunk = 0; warp + WARPS * 32 * chunk < npad; chunk++) {
      double xl, tl;
      norm_coords(p, base, npts, npad, warp + WARPS * (32 * chunk + lane), xl, tl);
#pragma unroll 4
      for (int i = 0; i < 32; i++) {
        const int pt = warp + WARPS * (32 * chunk + i);
        if (pt >= npad) break;
        const double xh = __shfl_sync(0xffffffffu, xl, i), th = __shfl_sync(0xffffffffu, tl, i);
#pragma unroll
        for (int c = 0; c < 4; c++) {
          const int u = lane + 32 * c;
          if (u < W) {
            const size_t o = (size_t)pt * W + u;
            const double z = Z0[o], zbx = Z0[SSZ + o], zbt = Z0[2 * SSZ + o];
            gx[c] = fma(xh, z, fma(sc0, zbx, gx[c]));
            gt[c] = fma(th, z, fma(sc1, zbt, gt[c]));
            gb[c] += z;
          }
        }
      }
    }
    double* comb = S0;                                       // [warp][3][128]
#pragma unroll
    for (int c = 0; c < 4; c++) {
      const int u = lane + 32 * c;
      comb[(warp * 3 + 0) * 128 + u] = gx[c];
      comb[(warp * 3 + 1) * 128 + u] = gt[c];
      comb[(warp * 3 + 2) * 128 + u] = gb[c];
    }
    __syncthreads();
    for (int i = tid; i < 3 * W; i += THREADS) {
      const int which = i / W, u = i - which * W;
      double sum = 0.0;
#pragma unroll
      for (int w8 = 0; w8 < WARPS; w8++) sum += comb[(w8 * 3 + which) * 128 + u];
      outp[(which == 0 ? woff(0) : (which == 1 ? woff(0) + W : boff(0))) + u] = sum;
    }
  }
}

}  // namespace nls
}  // namespace pinn
