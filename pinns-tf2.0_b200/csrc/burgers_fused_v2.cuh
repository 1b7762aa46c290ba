// Fused Burgers PINN loss + gradient kernel, v2: warp-specialised (sm_90a, fp64 DMMA on Hopper's 16x8 shapes).
//
// Same mathematics as burgers_fused.cuh (v1, kept on m8n8k4 as a cross-check), re-organised so that the FP64 pipe of every
// SM sub-partition always has two warps to draw from and nobody waits at a block barrier.  Its GEMMs run on DMMA.16x8x4
// (chain) and DMMA.16x8x8 (weight gradient), which issue twice the FMAs per cycle of DMMA.8x8x4 on the H100
// (profiles/microbench/fp64_peak_h100.jsonl).  Per 8-point tile: 210 DMMA.16x8x4 forward, 210 input adjoint and
// 140 DMMA.16x8x8 weight gradient (v1: 420 + 420 + 504 DMMA.8x8x4).
//
//   warps 0-3  "chain" warps  : own an 8-point tile each; forward DMMA chain through the 8 tanh layers, residual,
//                               seeds, then the backward chain (activation adjoints + input-adjoint DMMAs).  At
//                               every backward layer they stage Z-bar (the adjoint of the pre-activations, 4
//                               streams x 8 points x 20 units) into a 2-slot ring in shared memory and signal an
//                               mbarrier.  The stash written during the forward pass holds the layer OUTPUTS
//                               (a, a_x, a_t, a_xx) in [row][unit] layout, which is both what the division-free
//                               backward formula needs and the A operand of the weight-gradient GEMM.
//   warps 4-7  "wgrad" warps  : consume (stash[l-1], Z-bar_l) pairs of all four chain warps and run the
//                               weight-gradient GEMM  G_l[i][j] += sum_rows H_{l-1}[row][i] Zbar_l[row][j]  with DMMA.16x8x8
//                               (G_l is 21 input rows incl. the bias ones-row x 20 units; 5 tiles of 16 x 8 per layer, one
//                               of them transposed, see first_tile; K = the 32 staged rows).  The 35 output tiles of layers
//                               1..7 are OWNED by warps, 9/9/9/8; operand column pointers are chosen once per task (padded
//                               lanes point into a ones/zeros page), so the unrolled k loop has no predicates.
//                               Accumulators live in registers for the whole kernel: no shared-memory accumulator, no
//                               atomics, no cross-warp reduction, and a fixed summation order (deterministic results).
//
// Register layout of a chain warp ("V5").  A DMMA accumulator fragment (lane = 4g+q) holds point g, units 8nt+2q+e; hidden
// width 20 makes the third N tile half padding (units 20..23 in lanes q >= 2).  Between the GEMMs the 20 units of a point
// are therefore kept as FIVE values per lane and stream: j = 2nt+e for the first two tiles and, for j = 4, unit
// {16,18,17,19}[q] -- one quad shuffle moves the odd units of tile 2 from lanes q < 2 to lanes q >= 2.  This is exactly
// the A-operand layout of k-step j of the next GEMM (the contraction index is permuted: k-step j contracts the units the
// four lanes of a quad hold in slot j), so accumulators chain from layer to layer in registers, and the activation
// arithmetic (tanh and the Taylor/adjoint formulas) runs on 5 instead of 6 values per lane -- no lane computes padding.
// The m16n8k4 chain GEMMs stack two streams in one M = 16 tile (mma_layer5), whose fragment halves are these same layouts.
//
// Backward through a tanh layer in terms of its outputs (s = 1 - a^2; A* = adjoints of the outputs):
//   Z_xx = s A_xx;  Z_t = s A_t;  Z_x = s A_x - 4 a a_x A_xx;
//   Z    = s A - 2 a (a_x A_x + a_t A_t) - 2 A_xx (a a_xx + a_x^2)
// (algebraically identical to SURVEY Appendix A; no division by s, so saturated units are safe).
//
// Work distribution is tile-granular (8 points): the tiles are dealt evenly to the CTAs and round-robin to a CTA's four chain
// warps, so the slowest CTA carries at most one tile more than the others and small sets spread over all SMs.
//
// The tail of the evaluation runs in this launch too (optim_kernels.cuh: fused_tail): the last CTAs to finish reduce the per-CTA
// partial vectors in a fixed order, exchange them with the other ranks over NVLink (multi-GPU) and apply Adam (Adam steps).
//
// Alternatives tried on the previous target GPU with DMMA.8x8x4 and dropped there as slower or equal (not re-measured on H100
// or with the 16x8 shapes): 3-slot ring, holding the weight-gradient DMMAs back while the co-resident chain
// warp is in a DMMA phase (the weight-gradient warps starve), publishing Z-bar after the chain warp's own input-adjoint GEMM,
// output units 16..19 of the chain GEMMs (or columns 16..19 of the weight-gradient tile rows) as FMAs + a quad reduce-scatter
// instead of the half-padded third DMMA tile (DFMA interleaved with DMMA costs more than it saves), spreading the
// weight-gradient DMMAs with __nanosleep between k-steps, and a THREE-warps-per-sub-partition variant that splits every tile's
// chain between two half-warps (N tiles {0,2} / {1}, A operands from shared memory, roles alternating per layer; 384 threads x
// 168 registers: pair barriers and the A-operand LDS cost more than the added latency hiding bought).
// Tried on the H100 and dropped as slower (DESIGN §6): each layer's elementwise work fused slot by slot with the GEMM that
// consumes it (k-step j right after slot j; staging, ring arrive and the next layer's loads after the DMMA issue;
// profiles/experiments/burgers_chain_slotwise.patch).  Bit-identical, 51 instead of 13 DMMA.16x8x4 next to FP64 arithmetic in
// the SASS, and 0.5 % slower: DMMA.16x8 interleaved with DFMA in one warp costs more than the latency it hides.  Fully
// unrolled layer loops (no spills; 9-11 k instead of 7 k SASS instructions): forward +5 %, backward +1 %, both +18 %.
// Backward ring wait, Z-bar staging and arrive moved after the input-adjoint DMMA issue (the counterpart of the forward
// staging under the GEMM, which is kept): +5 %, the weight-gradient warps get Z-bar later.
// Every chain GEMM moved to warps 4-7, each running a quarter of it (profiles/experiments/burgers_dmma_warps.patch): the chain
// warps keep only the elementwise work and hand the staged operands over by mbarrier; the DMMA warps poll every chain's requests
// and the weight-gradient tasks in their fixed order.  Bit-identical, no hang, 186 registers, no stack -- and 2.4 times slower
// (0.747 against 0.305 ms; the input-adjoint GEMMs alone moved: 0.470 ms).  One DMMA warp per sub-partition now serves 56
// requests per round one after another, ~500 cycles each (operand LDS, 5 dependent DMMAs, stores, hand-off), so its busy time
// alone exceeds the whole kernel's; the chain warps spend most of their time waiting for GEMM results (DESIGN §6).
#pragma once
#include "burgers_fused.cuh"

namespace pinn {
namespace burgers2 {

using burgers::W;
using burgers::NHID;
using burgers::P_NET;
using burgers::WPAD;
using burgers::TILE;
using burgers::PSTRIDE;
using burgers::IDX_DL1;
using burgers::IDX_DL2;
using burgers::IDX_LD;
using burgers::IDX_LF;
using burgers::woff;
using burgers::boff;
using burgers::prow;
using burgers::Args;

constexpr int CHAINS = 4;
constexpr int THREADS = 256;              // 4 chain warps + 4 wgrad warps
constexpr int ROUND = CHAINS * TILE;      // 32 points per full CTA round
#ifndef PINN_RING
#define PINN_RING 2
#endif
// timing ablations (they compute WRONG gradients on purpose; profiles/kernel_variants.py)
#ifndef PINN_ABL_NOWG
#define PINN_ABL_NOWG 0                   // weight-gradient warps only do the ring handshake
#endif
#ifndef PINN_ABL_NOACT
#define PINN_ABL_NOACT 0                  // no activation arithmetic in the chain warps
#endif
#ifndef PINN_ABL_NODMMA
#define PINN_ABL_NODMMA 0                 // no chain DMMAs
#endif
// phase profile (profiles/kernel_variants.py): every warp of CTAs 0 and 1 sums clock() deltas (SM cycles between issuing the
// marks) per phase over one launch and printf's them at its end
#ifndef PINN_PHASE_CLOCKS
#define PINN_PHASE_CLOCKS 0
#endif
constexpr int RING = PINN_RING;           // Z-bar ring slots per chain warp

// shared memory carve-up (doubles)
constexpr int STASH0 = 640;               // layer 0: outputs (a, a_x, a_t, a_xx) as [32 rows][20], like the other layers
constexpr int STASHL = 640;               // layers 1..6: outputs (a, a_x, a_t, a_xx) as [32 rows][20]
constexpr int STASH_PER_WARP = STASH0 + 6 * STASHL;   // 4480
constexpr int SM_W = 0;
constexpr int SM_STASH = SM_W + WPAD;
constexpr int SM_RING = SM_STASH + CHAINS * STASH_PER_WARP;
constexpr int RED_PER_WARP = 128;         // chain-warp partials: [0..4] scalars, [8..27] dW8, [32..91] dW0 (x row, t row), db0
constexpr int SM_RED = SM_RING + CHAINS * RING * 640;
constexpr int SM_BAR = SM_RED + CHAINS * RED_PER_WARP;      // 1 + 2*CHAINS*RING mbarriers
constexpr int SM_SPECIAL = SM_BAR + 1 + 2 * CHAINS * RING + 1;   // [32 rows][W] page: column 0 = the bias ones-row (1 on the value
                                                                 // stream's rows 0..7), column 1 = 0
constexpr int SM_DOUBLES = SM_SPECIAL + 32 * W;
constexpr int SMEM_BYTES = SM_DOUBLES * 8;   // ~217 KB

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Ring bookkeeping: chain warp c numbers its weight-gradient tasks T = 7*tile + J (J = 7 - layer, layers 7..1; the
// gradients of layer 0 and of the output layer are plain FMAs in the chain warp itself).  Task T lives in ring
// slot T % RING; it is the (T / RING)-th use of that slot, i.e. phase T / RING of the slot's full and empty barriers.
__device__ __forceinline__ uint64_t* bar_full(uint64_t* bars, int c, int slot) { return bars + 1 + (c * RING + slot) * 2; }
__device__ __forceinline__ uint64_t* bar_empty(uint64_t* bars, int c, int slot) { return bars + 2 + (c * RING + slot) * 2; }
__device__ __forceinline__ void wait_produced(uint64_t* bars, int c, int T) { mbar_wait(bar_full(bars, c, T % RING), (T / RING) & 1); }
__device__ __forceinline__ void wait_consumed(uint64_t* bars, int c, int T) { mbar_wait(bar_empty(bars, c, T % RING), (T / RING) & 1); }

// PINN_PHASE_CLOCKS: mark(k) adds the cycles since the previous mark to phase k.  Chain warps: forward GEMM, forward
// elementwise (+ staging), output layer, backward elementwise (+ staging), backward GEMM, ring waits; weight-gradient warps:
// DMMA tasks (phase 0), waits for Z-bar (phase 5).
enum { PH_FWD_GEMM, PH_FWD_ACT, PH_OUT, PH_BWD_ACT, PH_BWD_GEMM, PH_WAIT, N_PHASES };
struct PhaseClocks {
#if PINN_PHASE_CLOCKS
  unsigned acc[N_PHASES] = {}, t = (unsigned)clock();
  __device__ __forceinline__ void mark(int k) { const unsigned n = (unsigned)clock(); acc[k] += n - t; t = n; }
  __device__ __forceinline__ void report(int warp, int lane) const {
    if (blockIdx.x < 2 && lane == 0)
      printf("phase %d %d %u %u %u %u %u %u\n", blockIdx.x, warp, acc[0], acc[1], acc[2], acc[3], acc[4], acc[5]);
  }
#else
  __device__ __forceinline__ void mark(int) {}
  __device__ __forceinline__ void report(int, int) const {}
#endif
};

// ---------------------------------------------------------------------------------------------------
// chain warps: the V5 register layout
// ---------------------------------------------------------------------------------------------------
// hidden unit held in slot j of lane-quad position q (== the unit k-step j contracts for this lane)
__device__ __forceinline__ int unit5(int j, int q) { return j < 4 ? 8 * (j >> 1) + 2 * q + (j & 1) : (q < 2 ? 16 + 2 * q : 13 + 2 * q); }

// accumulator fragments (C layout) -> V5: slots 0..3 are the first two tiles, slot 4 gathers units 16..19 across the quad
__device__ __forceinline__ void c_to_v5(double (&V)[4][5], const double (&Z)[4][3][2], int lane) {
#pragma unroll
  for (int s = 0; s < 4; s++) {
    V[s][0] = Z[s][0][0]; V[s][1] = Z[s][0][1]; V[s][2] = Z[s][1][0]; V[s][3] = Z[s][1][1];
    const double odd = __shfl_sync(0xffffffffu, Z[s][2][1], (lane & ~3) | (lane & 1));   // units 17, 19 live in lanes q = 0, 1
    V[s][4] = (lane & 2) ? odd : Z[s][2][0];
  }
}

// Z[s][nt][:] += V_s * Bmat, Bmat[k][n] = Wl[k*ldk + n*ldn]  (forward: ldk = 20, ldn = 1; input adjoint: ldk = 1, ldn = 20,
// i.e. the transposed weight).  N columns >= 20 read as zero.  Two streams share one M = 16 tile (stream 2p in rows 0..7,
// stream 2p+1 in rows 8..15; the fragments are V5 and Z as they are): 5 k-steps x 2 stream pairs x 3 N tiles = 30 DMMA.16x8x4.
__device__ __forceinline__ void mma_layer5(double (&Z)[4][3][2], const double (&V)[4][5], const double* Wl, int ldk, int ldn,
                                           int lane) {
  const int g = lane >> 2, q = lane & 3;
#pragma unroll
  for (int ks = 0; ks < 5; ks++) {
    const int k = unit5(ks, q);
    double b[3];
#pragma unroll
    for (int nt = 0; nt < 3; nt++) {
      const int n = 8 * nt + g;
      b[nt] = (n < W) ? Wl[k * ldk + n * ldn] : 0.0;
    }
#pragma unroll
    for (int p = 0; p < 2; p++)
#pragma unroll
      for (int nt = 0; nt < 3; nt++) dmma16x8x4(Z[2 * p][nt], Z[2 * p + 1][nt], V[2 * p][ks], V[2 * p + 1][ks], b[nt]);
  }
}

// outputs of a tanh layer from its pre-activation streams (in place): (z, z_x, z_t, z_xx) -> (a, s z_x, s z_t, s (z_xx - 2 a z_x^2))
__device__ __forceinline__ void act_forward5(double (&V)[4][5]) {
  if (PINN_ABL_NOACT) return;
#pragma unroll
  for (int j = 0; j < 5; j++) {
    const double a = tanh_fast(V[0][j]);
    const double zx = V[1][j];
    const double s = fma(-a, a, 1.0);
    V[0][j] = a;
    V[1][j] = s * zx;
    V[2][j] = s * V[2][j];
    V[3][j] = s * fma(-2.0 * a * zx, zx, V[3][j]);
  }
}

// adjoints of the outputs (A, overwritten with the adjoints of the pre-activations) given the outputs H
__device__ __forceinline__ void act_backward5(double (&A)[4][5], const double (&H)[4][5]) {
  if (PINN_ABL_NOACT) return;
#pragma unroll
  for (int j = 0; j < 5; j++) {
    const double a = H[0][j], ax = H[1][j], at = H[2][j], axx = H[3][j];
    const double A0 = A[0][j], Ax = A[1][j], At = A[2][j], Axx = A[3][j];
    const double s = fma(-a, a, 1.0);
    const double u1 = fma(ax, Ax, at * At);
    const double u2 = fma(a, axx, ax * ax);
    double z = fma(-2.0 * a, u1, s * A0);
    z = fma(-2.0 * Axx, u2, z);
    A[0][j] = z;
    A[1][j] = fma(-4.0 * a * ax, Axx, s * Ax);
    A[2][j] = s * At;
    A[3][j] = s * Axx;
  }
}

// V5 <-> a staged [32 rows][20 units] tile T[row = 8 s + prow(g)][unit] (ld = 20): two 16-byte accesses for the first two
// N tiles and one 8-byte access for this lane's unit of 16..19 per stream; all bank-conflict-free with the prow() row order.
__device__ __forceinline__ void stage5(double* T, const double (&V)[4][5], int lane) {
  const int pg = prow(lane >> 2), q = lane & 3;
  const int u4 = unit5(4, q);
#pragma unroll
  for (int s = 0; s < 4; s++) {
    double* row = T + (8 * s + pg) * W;
    *reinterpret_cast<double2*>(row + 2 * q) = make_double2(V[s][0], V[s][1]);
    *reinterpret_cast<double2*>(row + 8 + 2 * q) = make_double2(V[s][2], V[s][3]);
    row[u4] = V[s][4];
  }
}
__device__ __forceinline__ void load5(double (&V)[4][5], const double* T, int lane) {
  const int pg = prow(lane >> 2), q = lane & 3;
  const int u4 = unit5(4, q);
#pragma unroll
  for (int s = 0; s < 4; s++) {
    const double* row = T + (8 * s + pg) * W;
    const double2 c0 = *reinterpret_cast<const double2*>(row + 2 * q);
    const double2 c1 = *reinterpret_cast<const double2*>(row + 8 + 2 * q);
    V[s][0] = c0.x; V[s][1] = c0.y; V[s][2] = c1.x; V[s][3] = c1.y;
    V[s][4] = row[u4];
  }
}

// ---------------------------------------------------------------------------------------------------
// wgrad warps
// ---------------------------------------------------------------------------------------------------
// Output tiles of hidden layer l (1..7): G_l[i][j] (i = input unit 0..19 or 20 = the bias row, j = unit 0..19), 5 tiles:
//   t = 0, 1, 4: rows i = 0..15 (M) x units j = 0..7 | 8..15 | 16..19 + padding (N tile nt = 0, 1, 2)
//   t = 2:       TRANSPOSED, C[j][i] = G_l[i][j] for units j = 0..15 (M) x rows i = 16..23 (N: units 16..19, the bias row, padding)
//   t = 3:       the corner, rows i = 16..20 + padding (M) x units j = 16..19 + padding (N)
// Tile t of layer l is number 5 (l - 1) + t of 35 and belongs to warp (5 (l - 1) + t) & 3: the first tile of warp wg is
// t1 = (wg - 5 (l - 1)) & 3 and, for t1 == 0, the second is tile 4 (same M tile as tile 0, so the two share the A fragments).
// Warp wg owns two tiles at the layers l with l - 1 == wg (mod 4): 9/9/9/8 tiles (36/36/36/32 DMMA.16x8x8 per chain tile),
// one warp per output element, accumulated in a fixed order.
__device__ __forceinline__ int first_tile(int l, int wg) { return (wg - 5 * (l - 1)) & 3; }

// one weight-gradient task: accumulate this warp's tiles of layer L for one chain warp's 8-point tile.  K = the 32 staged
// rows in 4 k-steps of 8: k-step st (= stream) contracts physical rows 8 st + q (k = q) and 8 st + 4 + q (k = q + 4), so a
// quad's lanes read 4 rows 20 doubles apart and the stash and ring loads are bank-conflict-free with the prow() row order.
// H[row][i] = output i of layer L-1 (i == 20: the bias ones-row on the value stream), Z[row][j] = Z-bar; the A operand is
// H^T (Z-bar^T for the transposed tile t = 2), the B operand Z-bar (H).  Operand pointers of padding rows and columns point
// into the ones/zeros page, so the unrolled loop is 6 (TWO: 8) LDS + 1 (2) DMMA per k-step without predicates.
template <bool TWO>
__device__ __forceinline__ void wgrad_task(double (&c1)[2][2], double (&c2)[2][2], int t1, const double* Aop, const double* ZB,
                                           const double* SP, int lane) {
  const int g = lane >> 2, q = lane & 3;
  auto hcol = [&](int i) { return (i < W ? Aop + i : (i == W ? SP : SP + 1)) + q * W; };   // [32 rows][W] outputs of layer L-1
  auto zcol = [&](int j) { return (j < W ? ZB + j : SP + 1) + q * W; };                     // [32 rows][W] Z-bar
  // tile t1: A rows (M) from ap0 (m = g) and ap1 (m = g + 8), B columns (N = g) from bp1; t1 == 0 with TWO: bp2 for tile 4
  const double* ap0 = t1 == 2 ? zcol(g) : hcol(t1 == 3 ? 16 + g : g);
  const double* ap1 = t1 == 2 ? zcol(8 + g) : hcol(t1 == 3 ? 24 + g : 8 + g);
  const double* bp1 = t1 == 2 ? hcol(16 + g) : zcol(t1 == 3 ? 16 + g : 8 * t1 + g);
  const double* bp2 = zcol(16 + g);
#pragma unroll
  for (int st = 0; st < 4; st++) {
    const int off = 8 * st * W, off4 = off + 4 * W;
    const double a0 = ap0[off], a1 = ap1[off], a2 = ap0[off4], a3 = ap1[off4];
    dmma16x8x8(c1[0], c1[1], a0, a1, a2, a3, bp1[off], bp1[off4]);
    if (TWO) dmma16x8x8(c2[0], c2[1], a0, a1, a2, a3, bp2[off], bp2[off4]);
  }
}

template <int L>
__device__ __forceinline__ void wgrad_layer(double (&c1)[2][2], double (&c2)[2][2], int wg, int it, int half, int cnt,
                                            const double* sm, uint64_t* bars, int lane, PhaseClocks& pc) {
  constexpr int J = 7 - L;                  // task index within a tile (layers 7..1)
  const int T = 7 * it + J;
  const int slot = T % RING;
  const int t1 = first_tile(L, wg);
#pragma unroll 1
  for (int c = 2 * half; c < 2 * half + 2; c++) {
    if (4 * it + c >= cnt) break;           // chain warp c has no tile in this round (the CTA's last round may be partial)
    wait_produced(bars, c, T);
    pc.mark(PH_WAIT);
    const double* stash = sm + SM_STASH + c * STASH_PER_WARP;
    const double* Aop = stash + (L - 1) * STASHL;         // outputs of layer L-1 (STASH0 == STASHL)
    const double* ZB = sm + SM_RING + (c * RING + slot) * 640;
    if (!PINN_ABL_NOWG) {                   // warp-uniform: t1 is a function of (layer, warp)
      if (t1 == 0) wgrad_task<true>(c1, c2, t1, Aop, ZB, sm + SM_SPECIAL, lane);
      else wgrad_task<false>(c1, c2, t1, Aop, ZB, sm + SM_SPECIAL, lane);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_empty(bars, c, slot));
    pc.mark(PH_FWD_GEMM);
  }
}

template <int L>
__device__ __forceinline__ void wgrad_flush_tile(const double (&acc)[2][2], int t, double* outp, int lane) {
  const int g = lane >> 2, q = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; h++)
#pragma unroll
    for (int e = 0; e < 2; e++) {
      const int m = 8 * h + g, n = 2 * q + e;           // C[m][n] of the tile
      const int i = t == 2 ? 16 + n : (t == 3 ? 16 + m : m);
      const int j = t == 2 ? m : (t >= 3 ? 16 + n : 8 * t + n);
      if (j < W) {
        if (i < W) outp[woff(L) + i * W + j] = acc[h][e];
        else if (i == W) outp[boff(L) + j] = acc[h][e];
      }
    }
}
template <int L>
__device__ __forceinline__ void wgrad_flush(const double (&c1)[2][2], const double (&c2)[2][2], int wg, double* outp, int lane) {
  const int t1 = first_tile(L, wg);
  wgrad_flush_tile<L>(c1, t1, outp, lane);
  if (t1 == 0) wgrad_flush_tile<L>(c2, 4, outp, lane);
}

// At most 252 registers so that the 8 warps fit the register file.  The 16x8 chain GEMMs take their A operand pairs and
// accumulators in aligned register groups, and left alone ptxas uses 254; with the cap it fits without spills (ptxas -v).
__global__ void __maxnreg__(252) fused_loss_grad(const Args p) {
  extern __shared__ __align__(16) double sm[];
  if (p.run_flag && *p.run_flag != 0) return;
  double* Wsm = sm + SM_W;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sm + SM_BAR);   // [0] weights TMA; then (full, empty) per (chain, slot)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, q = lane & 3;

  for (int i = threadIdx.x; i < 32 * W; i += THREADS) sm[SM_SPECIAL + i] = (i % W == 0 && i / W < 8) ? 1.0 : 0.0;
  if (threadIdx.x == 0) {
    mbar_init(bars, 1);
    for (int i = 0; i < CHAINS * RING; i++) {
      mbar_init(bars + 1 + 2 * i, 1);        // full: the producing chain warp's lane 0
      mbar_init(bars + 2 + 2 * i, 4);        // empty: lane 0 of each of the 4 wgrad warps
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(bars, WPAD * 8);
    tma_bulk_g2s(Wsm, p.w, WPAD * 8, bars);
  }
  mbar_wait(bars, 0);

  const double sc0 = 2.0 / p.dx0, sc1 = 2.0 / p.dx1;
  // Tile-granular distribution: the ceil(n/8) tiles are dealt to the CTAs as evenly as possible (the first `rem` CTAs take one
  // more), a CTA's tiles j = 0..cnt-1 go to chain warp j & 3 in round j >> 2.  No CTA runs a whole extra round for a few left-over
  // tiles (N_f = 100 000: 84.5 tiles per CTA = 21.1 rounds instead of 22 for the slowest CTA), and small sets spread over all SMs
  // (2000 points: 1-2 tiles per CTA).
  const long long tiles_total = (p.n_total + TILE - 1) / TILE;
  const long long tbase = tiles_total / gridDim.x, trem = tiles_total - tbase * gridDim.x;
  const int cnt = (int)(tbase + (blockIdx.x < trem ? 1 : 0));                                  // tiles of this CTA
  const long long first_tile = tbase * blockIdx.x + (blockIdx.x < trem ? blockIdx.x : trem);
  const int my_rounds = (cnt + CHAINS - 1) / CHAINS;
  double* outp = p.partials + (size_t)blockIdx.x * PSTRIDE;

  if (warp >= CHAINS) {
    // =========================================== wgrad warps ===========================================
    const int wg = warp & 3;
    PhaseClocks pc;
    // first tile of each layer, and the second tiles: x[(L - 1) >> 2] is layer L's for warp L - 1 (layers 1..4) and L - 5 (5..7)
    double a1[2][2], a2[2][2], a3[2][2], a4[2][2], a5[2][2], a6[2][2], a7[2][2], x[2][2][2];
#pragma unroll
    for (int h = 0; h < 2; h++)
#pragma unroll
      for (int e = 0; e < 2; e++) {
        a1[h][e] = a2[h][e] = a3[h][e] = a4[h][e] = a5[h][e] = a6[h][e] = a7[h][e] = 0.0;
#pragma unroll
        for (int k = 0; k < 2; k++) x[k][h][e] = 0.0;
      }
#pragma unroll 1
    // The chain warps are consumed in two halves (chains 0,1 then chains 2,3).  Ring back-pressure then shifts the
    // halves by one phase: while one half runs its forward pass (which produces no weight-gradient work), the other
    // half runs its backward pass and keeps these warps -- and the FP64 pipe of every sub-partition -- busy.
    for (int it2 = 0; it2 < 2 * my_rounds; it2++) {
      const int it = it2 >> 1, half = it2 & 1;
      wgrad_layer<7>(a7, x[1], wg, it, half, cnt, sm, bars, lane, pc);
      wgrad_layer<6>(a6, x[1], wg, it, half, cnt, sm, bars, lane, pc);
      wgrad_layer<5>(a5, x[1], wg, it, half, cnt, sm, bars, lane, pc);
      wgrad_layer<4>(a4, x[0], wg, it, half, cnt, sm, bars, lane, pc);
      wgrad_layer<3>(a3, x[0], wg, it, half, cnt, sm, bars, lane, pc);
      wgrad_layer<2>(a2, x[0], wg, it, half, cnt, sm, bars, lane, pc);
      wgrad_layer<1>(a1, x[0], wg, it, half, cnt, sm, bars, lane, pc);
    }
    wgrad_flush<1>(a1, x[0], wg, outp, lane);
    wgrad_flush<2>(a2, x[0], wg, outp, lane);
    wgrad_flush<3>(a3, x[0], wg, outp, lane);
    wgrad_flush<4>(a4, x[0], wg, outp, lane);
    wgrad_flush<5>(a5, x[1], wg, outp, lane);
    wgrad_flush<6>(a6, x[1], wg, outp, lane);
    wgrad_flush<7>(a7, x[1], wg, outp, lane);
    pc.report(warp, lane);
  } else {
    // =========================================== chain warps ===========================================
    const int c = warp;
    const int n_tiles = cnt > c ? (cnt - c + CHAINS - 1) / CHAINS : 0;      // tiles j = c, c + 4, ... of this CTA
    double* stash = sm + SM_STASH + c * STASH_PER_WARP;
    const double l1 = p.ide ? Wsm[P_NET] : 1.0;
    const double kap = p.ide ? exp(Wsm[P_NET + 1]) : p.nu;
    double loss_d = 0.0, loss_f = 0.0, gl1 = 0.0, gl2 = 0.0;
    double g8[5], gb8 = 0.0;                // output-layer weight gradient: per-lane partials over this lane's points
    double g0x[5], g0t[5], g0b[5];          // layer-0 weight gradient (rows x^, t^ of W_0 and b_0): likewise
#pragma unroll
    for (int j = 0; j < 5; j++) g8[j] = g0x[j] = g0t[j] = g0b[j] = 0.0;
    const int pg = prow(g);
    int u5[5];                              // the five hidden units of this lane
#pragma unroll
    for (int j = 0; j < 5; j++) u5[j] = unit5(j, q);
    // coordinates of this lane's point in tile `it`; the next tile's pair is prefetched one tile ahead so that neither
    // the L2/HBM latency nor (zero-copy mode: p.xc in pinned host memory) the PCIe latency is exposed
    auto load_xt = [&](int it, double& xo, double& to) {
      long long pt = (first_tile + 4 * it + c) * TILE + g;
      if (pt >= p.n_total) pt = p.n_total - 1;
      if (p.xc && pt >= p.c0 && pt < p.c0 + p.n_c) {
        xo = __ldg(p.xc + (pt - p.c0)); to = __ldg(p.tc + (pt - p.c0));
      } else {
        xo = __ldg(p.x + pt); to = __ldg(p.t + pt);
      }
    };
    double xr_next = 0.0, tr_next = 0.0;
    if (n_tiles > 0) load_xt(0, xr_next, tr_next);
    PhaseClocks pc;

#pragma unroll 1
    for (int it = 0; it < n_tiles; it++) {
      const long long pt = (first_tile + 4 * it + c) * TILE + g;
      const bool in_set = pt < p.n_total;
      const double xr = xr_next, tr = tr_next;
      if (it + 1 < n_tiles) load_xt(it + 1, xr_next, tr_next);
      const bool in_c = in_set && pt >= p.c0 && pt < p.c0 + p.n_c;
      const double wf = in_c ? p.wf : 0.0;
      const bool has_d = in_set && pt >= p.d0 && pt < p.d0 + p.n_d;
      const double wd = has_d ? p.wd : 0.0;
      const double ut = has_d ? __ldg(p.utgt + (pt - p.d0)) : 0.0;
      const double xh = 2.0 * (xr - p.lb0) / p.dx0 - 1.0;   // utils/neuralnetwork.py:29-30
      const double th = 2.0 * (tr - p.lb1) / p.dx1 - 1.0;

      double V[4][5];
      // ---------------- layer 0 (2 -> 20): direct
#pragma unroll
      for (int j = 0; j < 5; j++) {
        const double w0 = Wsm[u5[j]], w1 = Wsm[W + u5[j]], b = Wsm[2 * W + u5[j]];
        V[0][j] = fma(xh, w0, fma(th, w1, b));
        V[1][j] = sc0 * w0;
        V[2][j] = sc1 * w1;
        V[3][j] = 0.0;
      }
      act_forward5(V);
      pc.mark(PH_FWD_ACT);
      // ---------------- hidden layers 1..7: DMMA chain
#pragma unroll 1
      for (int l = 1; l < NHID; l++) {
        const double* Wl = Wsm + woff(l);
        double Z[4][3][2];
#pragma unroll
        for (int nt = 0; nt < 3; nt++)
#pragma unroll
          for (int e = 0; e < 2; e++) {
            const int col = 8 * nt + 2 * q + e;
            Z[0][nt][e] = (col < W) ? Wl[W * W + col] : 0.0;
            Z[1][nt][e] = Z[2][nt][e] = Z[3][nt][e] = 0.0;
          }
        if (!PINN_ABL_NODMMA) mma_layer5(Z, V, Wl, W, 1, lane);
        // The outputs of layer l-1 (V, the GEMM's A operand in registers) go to the stash while the DMMAs run: the stores, and for
        // l = 1 the wait below, sit under the GEMM instead of in series before it.  The stash is still the A operand of the
        // previous tile's weight-gradient tasks; slot 0 is read by the last of them, the layer-1 task (J = 6), and consumers
        // retire tasks in order, so once it is consumed every slot is free.
        pc.mark(PH_FWD_GEMM);
        if (l == 1 && it > 0) wait_consumed(bars, c, 7 * (it - 1) + 6);
        pc.mark(PH_WAIT);
        stage5(stash + (l - 1) * STASHL, V, lane);                  // STASH0 == STASHL
        pc.mark(PH_FWD_ACT);
        c_to_v5(V, Z, lane);
        pc.mark(PH_FWD_GEMM);
        act_forward5(V);
        pc.mark(PH_FWD_ACT);
      }
      // ---------------- output layer (20 -> 1), residual, seeds
      double A[4][5];
      {
        const double* W8 = Wsm + woff(8);
        double w8[5];
#pragma unroll
        for (int j = 0; j < 5; j++) w8[j] = W8[u5[j]];
        double out[4];
#pragma unroll
        for (int s = 0; s < 4; s++) {
          double acc = 0.0;
#pragma unroll
          for (int j = 0; j < 5; j++) acc = fma(V[s][j], w8[j], acc);
          acc += shfl_xor_d(acc, 1);
          acc += shfl_xor_d(acc, 2);
          out[s] = acc;
        }
        out[0] += Wsm[boff(8)];
        const double u = out[0], ux = out[1], utt = out[2], uxx = out[3];
        // f and r are selected, not weighted by 0, outside their sets: 0 * NaN or 0 * Inf would reach the other set's part
        const double f = in_c ? utt + l1 * u * ux - kap * uxx : 0.0;   // inf_cont_burgers.py:90 / ide_cont_burgers.py:85
        const double r = has_d ? u - ut : 0.0;
        const double cc = 2.0 * wf * f;
        double seed[4];
        seed[0] = fma(cc * l1, ux, 2.0 * wd * r);
        seed[1] = cc * l1 * u;
        seed[2] = cc;
        seed[3] = -cc * kap;
        if (q == 0 && in_set) {                              // a padded lane (clamped copy of the last point) adds nothing
          loss_d = fma(wd * r, r, loss_d);
          loss_f = fma(wf * f, f, loss_f);
          gl1 = fma(cc * u, ux, gl1);
          gl2 = fma(-cc * kap, uxx, gl2);
          gb8 += seed[0];
        }
        // output-layer weight gradient (per-lane partial over this lane's point) and adjoint of layer-7 outputs
#pragma unroll
        for (int j = 0; j < 5; j++) {
          double acc = g8[j];
#pragma unroll
          for (int s = 0; s < 4; s++) {
            acc = fma(V[s][j], seed[s], acc);
            A[s][j] = seed[s] * w8[j];
          }
          g8[j] = acc;
        }
      }
      pc.mark(PH_OUT);
      // ---------------- backward: layers 7..1 (task J = 7-l, ring slot J % RING); V holds the outputs of layer l (l = 7: still in
      // registers from the forward pass)
#pragma unroll 1
      for (int l = NHID - 1; l >= 1; l--) {
        const int T = 7 * it + (7 - l), slot = T % RING;
        act_backward5(A, V);                                                         // A := Z-bar
        pc.mark(PH_BWD_ACT);
        if (T >= RING) wait_consumed(bars, c, T - RING);                             // the slot's previous task is done
        pc.mark(PH_WAIT);
        stage5(sm + SM_RING + (c * RING + slot) * 640, A, lane);
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_full(bars, c, slot));
        pc.mark(PH_BWD_ACT);
        // adjoint of the layer inputs: A_new = Z-bar * W_l^T
        {
          const double* Wl = Wsm + woff(l);
          double An[4][3][2];
#pragma unroll
          for (int s = 0; s < 4; s++)
#pragma unroll
            for (int nt = 0; nt < 3; nt++) An[s][nt][0] = An[s][nt][1] = 0.0;
          if (!PINN_ABL_NODMMA) mma_layer5(An, A, Wl, 1, W, lane);
          // the outputs of layer l-1 (STASH0 == STASHL), loaded while the DMMAs are in flight: issued before the GEMM's
          // results are needed, their shared-memory latency is hidden instead of starting the next layer's arithmetic
          load5(V, stash + (l - 1) * STASHL, lane);
          c_to_v5(A, An, lane);
        }
        pc.mark(PH_BWD_GEMM);
      }
      // ---------------- backward: layer 0: its weight gradient is 3 rows (x^, t^, bias) -- 25 FMAs per lane here instead of 24
      // DMMAs in a weight-gradient warp
      {
        act_backward5(A, V);
#pragma unroll
        for (int j = 0; j < 5; j++) {
          g0x[j] = fma(xh, A[0][j], fma(sc0, A[1][j], g0x[j]));   // inputs: (x^, t^) on the value stream, (sc0, 0) on the x
          g0t[j] = fma(th, A[0][j], fma(sc1, A[2][j], g0t[j]));   // stream, (0, sc1) on the t stream, 0 on the xx stream
          g0b[j] += A[0][j];
        }
      }
      pc.mark(PH_BWD_ACT);
    }

    // ---------------- chain-warp partials: losses, identification gradients, output-layer gradient
    double* red = sm + SM_RED + c * RED_PER_WARP;
    loss_d = warp_sum(loss_d); loss_f = warp_sum(loss_f); gl1 = warp_sum(gl1); gl2 = warp_sum(gl2); gb8 = warp_sum(gb8);
#pragma unroll
    for (int j = 0; j < 5; j++) {
      double v = g8[j], vx = g0x[j], vt = g0t[j], vb = g0b[j];
      v += shfl_xor_d(v, 4); v += shfl_xor_d(v, 8); v += shfl_xor_d(v, 16);   // sum over the 8 points (g)
      vx += shfl_xor_d(vx, 4); vx += shfl_xor_d(vx, 8); vx += shfl_xor_d(vx, 16);
      vt += shfl_xor_d(vt, 4); vt += shfl_xor_d(vt, 8); vt += shfl_xor_d(vt, 16);
      vb += shfl_xor_d(vb, 4); vb += shfl_xor_d(vb, 8); vb += shfl_xor_d(vb, 16);
      if (g == 0) { red[8 + u5[j]] = v; red[32 + u5[j]] = vx; red[32 + W + u5[j]] = vt; red[32 + 2 * W + u5[j]] = vb; }
    }
    if (lane == 0) { red[0] = loss_d; red[1] = loss_f; red[2] = gl1; red[3] = gl2; red[4] = gb8; }
    pc.report(warp, lane);
  }

  __syncthreads();
  {
    const double* red = sm + SM_RED;
    constexpr int R = RED_PER_WARP;
    const int t = threadIdx.x;
    auto sum4 = [&](int i) { return red[i] + red[R + i] + red[2 * R + i] + red[3 * R + i]; };   // fixed order: chains 0..3
    if (t < W) outp[woff(8) + t] = sum4(8 + t);
    if (t >= 64 && t < 64 + 3 * W) outp[woff(0) + (t - 64)] = sum4(32 + (t - 64));   // W_0 (2 x 20, row-major) then b_0: flat 0..59
    if (t == 32) outp[boff(8)] = sum4(4);
    if (t == 33) outp[IDX_LD] = sum4(0);
    if (t == 34) outp[IDX_LF] = sum4(1);
    if (t == 35) outp[IDX_DL1] = sum4(2);
    if (t == 36) outp[IDX_DL2] = sum4(3);
    if (t == 37) outp[3023] = 0.0;
  }
  if (p.tail.enabled) fused_tail(p.tail, p.partials, PSTRIDE, sm + SM_STASH);     // the stash is dead; all 256 threads arrive
}

}  // namespace burgers2
}  // namespace pinn
