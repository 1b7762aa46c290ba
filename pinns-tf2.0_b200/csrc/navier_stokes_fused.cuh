// Continuous-time Navier-Stokes identification (PINNs/main/continuous_time_identification (Navier-Stokes)/NavierStokes.py,
// fp64 restatement): fused loss + gradient kernel for any tanh MLP [3, w_1, ..., w_k, 2] (hidden widths <= 256, <= 15 Dense
// layers) on 13 forward Taylor streams, and the thread-per-point probe kernel behind pinn_predict / pinn_derivatives /
// pinn_residual for these handles; fp64, sm_90a.
//
// Streams (multi-indices over (x, y, t); the same order in the C ABI's probe layout and here):
//   0 value, 1 x, 2 y, 3 t, 4 xx, 5 xy, 6 yy, 7 xt, 8 yt, 9 xxx, 10 xxy, 11 xyy, 12 yyy
// The t stream exists only to form xt and yt.  Per tanh layer, s = 1 - a^2, sigma2 = -2as, sigma3 = -2s(1 - 3a^2):
//   a_i = s z_i;  a_ij = s z_ij + sigma2 z_i z_j;  a_ijk = s z_ijk + sigma2 (z_ij z_k + z_ik z_j + z_jk z_i) + sigma3 z_i z_j z_k
// Reverse, division-free in the stored layer outputs: perturbing z_beta by d adds d x^beta / beta! to z, so
//   d a_alpha / d z_beta = C(alpha, beta) s_(alpha - beta),   s_gamma = d^gamma (1 - a^2) = -d^gamma (a^2)  (Leibniz in a-streams)
//   Z-bar_beta = sum over alpha >= beta of C(alpha, beta) s_(alpha - beta) A-bar_alpha         (written out in zbar_streams)
// KdV's 1-D identity  d a_xxx / dz = -2a a_xxx - 6 a_x a_xx  is the case alpha = xxx, beta = 0.
//
// Structure (the layer-outer design of generic_fused.cuh, which makes it width-agnostic): a CTA owns a contiguous block of
// points; the 13 streams of every hidden layer go to a per-CTA global scratch [layer][13][pts][w], so the rows
// (stream, point) of a layer are one row-major [13 pts x w] matrix.  Phases  F_0 (direct, K = 3) -> F_l -> HEAD -> B_l -> B_0.
// GEMMs on DMMA.16x8x4 (pinn_common.cuh), item lists handed out through a shared counter:
//   F_l          item = (16 points, 8 columns): the 13 stream tiles of those points share every B fragment, so one lane ends
//                with all 13 streams of its (point, unit) pairs and applies the tanh rules in registers
//   input adj.   the same tile shape over Z-bar x W_l^T
//   weight grad  item = (16 rows of [W_l ; b_l], 8 columns), K = 13 streams x the CTA's points in a fixed order: every output
//                element comes from exactly one warp, so the result is bitwise reproducible
#pragma once
#include "generic_fused.cuh"

namespace pinn {
namespace nsid {

constexpr int THREADS = 256;
constexpr int NST = 13;                   // Taylor streams
constexpr int OUT = 2;                    // (psi, p)
constexpr int SEEDW = NST * OUT;          // head outputs / seeds per point: [stream][psi, p]

struct Args {
  const double* w;
  NetDesc nd;                 // dims / offsets (its lb/dx fields are unused: 3 inputs)
  double lb[3], sc[3];        // input box: h = sc (X - lb) - 1, sc = 2 / (ub - lb)
  const double* X;            // [n][3] = (x, y, t)
  const double* tgt;          // [n][2] = (u, v)
  long long n_total;
  int p_net;                  // lambda_1, lambda_2 at p_net, p_net + 1 (raw)
  double* scrH;               // [grid][sum_l 13 pts w_l]
  double* scrA;               // [grid][2][13 pts maxw]
  double* scrS;               // [grid][2][pts][26]   head outputs, seeds
  long long h_per_cta, a_per_cta;
  int pts;
  double* partials;           // [grid][pstride]: [grad p_net | dl1 dl2 | part0 part1 part2]
  int pstride;
  const int* run_flag;
};

// the 13 output streams of a tanh unit from a = tanh(z) and the 13 pre-activation streams
__device__ __forceinline__ void tanh_streams(double a, const double (&z)[NST], double (&o)[NST]) {
  const double s = fma(-a, a, 1.0);
  const double s2 = -2.0 * a * s;
  const double s3 = -2.0 * s * fma(-3.0 * a, a, 1.0);
  const double zx = z[1], zy = z[2], zt = z[3];
  o[0] = a;
  o[1] = s * zx;
  o[2] = s * zy;
  o[3] = s * zt;
  o[4] = fma(s2 * zx, zx, s * z[4]);
  o[5] = fma(s2 * zx, zy, s * z[5]);
  o[6] = fma(s2 * zy, zy, s * z[6]);
  o[7] = fma(s2 * zx, zt, s * z[7]);
  o[8] = fma(s2 * zy, zt, s * z[8]);
  o[9] = fma(s3 * zx * zx, zx, fma(s2, 3.0 * z[4] * zx, s * z[9]));
  o[10] = fma(s3 * zx * zx, zy, fma(s2, fma(z[4], zy, 2.0 * z[5] * zx), s * z[10]));
  o[11] = fma(s3 * zx * zy, zy, fma(s2, fma(2.0 * z[5], zy, z[6] * zx), s * z[11]));
  o[12] = fma(s3 * zy * zy, zy, fma(s2, 3.0 * z[6] * zy, s * z[12]));
}

// Z-bar of the 13 pre-activation streams from the stored outputs A and their adjoints B (see the header comment)
__device__ __forceinline__ void zbar_streams(const double (&A)[NST], const double (&B)[NST], double (&Z)[NST]) {
  const double a = A[0];
  double S[NST];                                    // s_gamma = -d^gamma (a^2)
  S[0] = fma(-a, a, 1.0);
  S[1] = -2.0 * a * A[1];
  S[2] = -2.0 * a * A[2];
  S[3] = -2.0 * a * A[3];
  S[4] = -2.0 * fma(a, A[4], A[1] * A[1]);
  S[5] = -2.0 * fma(a, A[5], A[1] * A[2]);
  S[6] = -2.0 * fma(a, A[6], A[2] * A[2]);
  S[7] = -2.0 * fma(a, A[7], A[1] * A[3]);
  S[8] = -2.0 * fma(a, A[8], A[2] * A[3]);
  S[9] = -2.0 * fma(a, A[9], 3.0 * A[4] * A[1]);
  S[10] = -2.0 * fma(a, A[10], fma(A[4], A[2], 2.0 * A[5] * A[1]));
  S[11] = -2.0 * fma(a, A[11], fma(2.0 * A[5], A[2], A[6] * A[1]));
  S[12] = -2.0 * fma(a, A[12], 3.0 * A[6] * A[2]);
  const double s = S[0];
  double z0 = 0.0;
#pragma unroll
  for (int k = 0; k < NST; k++) z0 = fma(S[k], B[k], z0);
  Z[0] = z0;
  // x:  x, xx (2), xy, xt, xxx (3), xxy (2), xyy
  Z[1] = fma(s, B[1], fma(2.0 * S[1], B[4], fma(S[2], B[5], fma(S[3], B[7], fma(3.0 * S[4], B[9], fma(2.0 * S[5], B[10], S[6] * B[11]))))));
  // y:  y, xy, yy (2), yt, xxy, xyy (2), yyy (3)
  Z[2] = fma(s, B[2], fma(S[1], B[5], fma(2.0 * S[2], B[6], fma(S[3], B[8], fma(S[4], B[10], fma(2.0 * S[5], B[11], 3.0 * S[6] * B[12]))))));
  Z[3] = fma(s, B[3], fma(S[1], B[7], S[2] * B[8]));                                  // t:  t, xt, yt
  Z[4] = fma(s, B[4], fma(3.0 * S[1], B[9], S[2] * B[10]));                           // xx: xx, xxx (3), xxy
  Z[5] = fma(s, B[5], fma(2.0 * S[1], B[10], 2.0 * S[2] * B[11]));                    // xy: xy, xxy (2), xyy (2)
  Z[6] = fma(s, B[6], fma(S[1], B[11], 3.0 * S[2] * B[12]));                          // yy: yy, xyy, yyy (3)
#pragma unroll
  for (int k = 7; k < NST; k++) Z[k] = s * B[k];                                      // xt, yt and the third order
}

// C[s] += A_s (16 rows x K) * B (K x 8 columns), the 13 streams sharing every B fragment (DMMA.16x8x4).
//   A_s(row r, k) = X[s * sstride + r * lda + k] with this lane's rows r_lo (= g) and r_hi (= g + 8) already clamped to valid
//   rows;  B(k, n) = B[k * ldk + n * ldn] at this lane's column n (clamped; nok = false makes it zero).  k >= K contributes zero
//   through B (the A address is clamped, its value finite).
__device__ __forceinline__ void gemm13(double (&C)[NST][2][2], const double* X, size_t sstride, int lda, int K, const double* B,
                                       size_t ldk, size_t ldn, int n, bool nok, int r_lo, int r_hi, int q) {
  const double* xl = X + (size_t)r_lo * lda;
  const double* xh = X + (size_t)r_hi * lda;
  const double* bp = B + (size_t)n * ldn;
  const int kfull = K >> 2;
#pragma unroll 1
  for (int ks = 0; ks < kfull; ks++) {
    const int k = 4 * ks + q;
    const double b = nok ? __ldg(bp + (size_t)k * ldk) : 0.0;
#pragma unroll
    for (int s = 0; s < NST; s++) dmma16x8x4(C[s][0], C[s][1], xl[s * sstride + k], xh[s * sstride + k], b);
  }
  if (K & 3) {
    const int k = 4 * kfull + q;
    const bool kok = k < K;
    const int kc = kok ? k : K - 1;
    const double b = (nok && kok) ? __ldg(bp + (size_t)kc * ldk) : 0.0;
#pragma unroll
    for (int s = 0; s < NST; s++) dmma16x8x4(C[s][0], C[s][1], xl[s * sstride + kc], xh[s * sstride + kc], b);
  }
}

__global__ void __launch_bounds__(THREADS, 1) fused_loss_grad(const Args p) {
  __shared__ double red[THREADS / 32];
  __shared__ int work_ctr;
  __shared__ size_t hoff[MAXL];
  if (p.run_flag && *p.run_flag != 0) return;
  const int tid = threadIdx.x, lane = tid & 31;
  const int g = lane >> 2, q = lane & 3;
  const NetDesc& nd = p.nd;
  const int L = nd.n_layers;                 // Dense layers; hidden 0..L-2, head L-1
  const int pts = p.pts;
  const long long base = (long long)blockIdx.x * pts;
  const long long navail = p.n_total - base;
  const int npts = navail <= 0 ? 0 : (navail < pts ? (int)navail : pts);
  double* Hs = p.scrH + (size_t)blockIdx.x * p.h_per_cta;
  double* A0 = p.scrA + (size_t)blockIdx.x * 2 * p.a_per_cta;
  double* A1 = A0 + p.a_per_cta;
  double* OUTV = p.scrS + (size_t)blockIdx.x * 2 * pts * SEEDW;
  double* SEED = OUTV + (size_t)pts * SEEDW;
  double* outp = p.partials + (size_t)blockIdx.x * p.pstride;
  const double l1 = p.w[p.p_net], l2 = p.w[p.p_net + 1];

  if (tid == 0) {
    size_t o = 0;
    for (int l = 0; l < L - 1; l++) { hoff[l] = o; o += (size_t)NST * pts * nd.dims[l + 1]; }
  }
  __syncthreads();

  // ======================================= forward: hidden layers =======================================
  for (int l = 0; l < L - 1; l++) {
    const int fi = nd.dims[l], fo = nd.dims[l + 1];
    const double* Wl = p.w + nd.woff[l];
    const double* bl = p.w + nd.boff[l];
    double* Ho = Hs + hoff[l];
    const size_t so = (size_t)pts * fo;
    if (l == 0) {
      // K = 3: thread per (point, unit); the first-order input streams are constant, the higher ones zero
      for (int idx = tid; idx < npts * fo; idx += THREADS) {
        const int pt = idx / fo, j = idx - pt * fo;
        const double* xp = p.X + 3 * (base + pt);
        double z[NST], o[NST];
#pragma unroll
        for (int s = 0; s < NST; s++) z[s] = 0.0;
        z[0] = __ldg(bl + j);
#pragma unroll
        for (int i = 0; i < 3; i++) {
          const double wv = __ldg(Wl + i * fo + j);
          z[0] = fma(fma(p.sc[i], __ldg(xp + i) - p.lb[i], -1.0), wv, z[0]);
          z[1 + i] = p.sc[i] * wv;
        }
        tanh_streams(tanh_fast(z[0]), z, o);
#pragma unroll
        for (int s = 0; s < NST; s++) Ho[s * so + (size_t)pt * fo + j] = o[s];
      }
      __syncthreads();
      continue;
    }
    const double* Hp = Hs + hoff[l - 1];
    const size_t sp = (size_t)pts * fi;
    const int nt = (fo + 7) >> 3;
    const int items = ((npts + 15) >> 4) * nt;
    if (tid == 0) work_ctr = 0;
    __syncthreads();
    for (int it = generic::next_item(&work_ctr, lane); it < items; it = generic::next_item(&work_ctr, lane)) {
      const int pt0 = 16 * (it / nt), n0 = 8 * (it - (it / nt) * nt);
      const int n = n0 + g;
      double C[NST][2][2];
#pragma unroll
      for (int e = 0; e < 2; e++) {
        const int u = n0 + 2 * q + e;
        C[0][0][e] = C[0][1][e] = u < fo ? __ldg(bl + u) : 0.0;
      }
#pragma unroll
      for (int s = 1; s < NST; s++) C[s][0][0] = C[s][0][1] = C[s][1][0] = C[s][1][1] = 0.0;
      gemm13(C, Hp, sp, fi, fi, Wl, fo, 1, n < fo ? n : fo - 1, n < fo, min(pt0 + g, npts - 1), min(pt0 + g + 8, npts - 1), q);
#pragma unroll
      for (int hf = 0; hf < 2; hf++)
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const int pt = pt0 + g + 8 * hf, u = n0 + 2 * q + e;
          if (pt < npts && u < fo) {
            double z[NST], o[NST];
#pragma unroll
            for (int s = 0; s < NST; s++) z[s] = C[s][hf][e];
            tanh_streams(tanh_fast(z[0]), z, o);
#pragma unroll
            for (int s = 0; s < NST; s++) Ho[s * so + (size_t)pt * fo + u] = o[s];
          }
        }
    }
    __syncthreads();
  }

  // ======================================= head + Navier-Stokes terms =======================================
  const int fl = nd.dims[L - 1];
  const double* Hl = Hs + hoff[L - 2];
  const size_t sl = (size_t)pts * fl;
  const double* Wh = p.w + nd.woff[L - 1];
  for (int idx = tid; idx < npts * SEEDW; idx += THREADS) {
    const int pt = idx / SEEDW, r = idx - pt * SEEDW, s = r >> 1, o = r & 1;
    const double* h = Hl + s * sl + (size_t)pt * fl;
    double acc = s == 0 ? __ldg(p.w + nd.boff[L - 1] + o) : 0.0;
    for (int i = 0; i < fl; i++) acc = fma(h[i], __ldg(Wh + 2 * i + o), acc);
    OUTV[idx] = acc;
  }
  __syncthreads();
  double part0 = 0.0, part2 = 0.0, gl1 = 0.0, gl2 = 0.0;
  for (int pt = tid; pt < npts; pt += THREADS) {
    const double* O = OUTV + (size_t)pt * SEEDW;          // O[2 s] = psi stream s, O[2 s + 1] = p stream s
    const double px = O[2], py = O[4], pxx = O[8], pxy = O[10], pyy = O[12], pxt = O[14], pyt = O[16];
    const double pxxx = O[18], pxxy = O[20], pxyy = O[22], pyyy = O[24];
    const double qx = O[3], qy = O[5];
    const double e_u = py - __ldg(p.tgt + 2 * (base + pt)), e_v = -px - __ldg(p.tgt + 2 * (base + pt) + 1);
    const double adv_u = fma(py, pxy, -px * pyy), adv_v = fma(px, pxy, -py * pxx);
    const double lap_u = pxxy + pyyy, lap_v = pxxx + pxyy;
    const double f_u = fma(-l2, lap_u, fma(l1, adv_u, pyt + qx));
    const double f_v = fma(l2, lap_v, fma(l1, adv_v, qy - pxt));
    part0 = fma(e_u, e_u, fma(e_v, e_v, part0));
    part2 = fma(f_u, f_u, fma(f_v, f_v, part2));
    const double cu = 2.0 * f_u, cv = 2.0 * f_v;
    gl1 = fma(cu, adv_u, fma(cv, adv_v, gl1));
    gl2 = fma(-cu, lap_u, fma(cv, lap_v, gl2));
    double* S = SEED + (size_t)pt * SEEDW;
    const double lcu = l1 * cu, lcv = l1 * cv;
    S[0] = 0.0;                         S[1] = 0.0;
    S[2] = fma(lcv, pxy, fma(-lcu, pyy, -2.0 * e_v));  S[3] = cu;          // x
    S[4] = fma(-lcv, pxx, fma(lcu, pxy, 2.0 * e_u));   S[5] = cv;          // y
    S[6] = 0.0;                         S[7] = 0.0;                        // t
    S[8] = -lcv * py;                   S[9] = 0.0;                        // xx
    S[10] = fma(lcu, py, lcv * px);     S[11] = 0.0;                       // xy
    S[12] = -lcu * px;                  S[13] = 0.0;                       // yy
    S[14] = -cv;                        S[15] = 0.0;                       // xt
    S[16] = cu;                         S[17] = 0.0;                       // yt
    S[18] = l2 * cv;                    S[19] = 0.0;                       // xxx
    S[20] = -l2 * cu;                   S[21] = 0.0;                       // xxy
    S[22] = l2 * cv;                    S[23] = 0.0;                       // xyy
    S[24] = -l2 * cu;                   S[25] = 0.0;                       // yyy
  }
  generic::block_reduce_store(gl1, red, outp + p.p_net + 0);
  generic::block_reduce_store(gl2, red, outp + p.p_net + 1);
  generic::block_reduce_store(part0, red, outp + p.p_net + 2);
  generic::block_reduce_store(part2, red, outp + p.p_net + 4);
  if (tid == 0) outp[p.p_net + 3] = 0.0;
  __syncthreads();

  // ======================================= head: gradient and input adjoint =======================================
  for (int e = tid; e < (fl + 1) * OUT; e += THREADS) {
    const int i = e >> 1, o = e & 1;
    double acc = 0.0;
    for (int pt = 0; pt < npts; pt++) {
      const double* sd = SEED + (size_t)pt * SEEDW + o;
      if (i < fl) {
#pragma unroll
        for (int s = 0; s < NST; s++) acc = fma(Hl[s * sl + (size_t)pt * fl + i], sd[2 * s], acc);
      } else {
        acc += sd[0];
      }
    }
    if (i < fl) outp[nd.woff[L - 1] + 2 * i + o] = acc;
    else outp[nd.boff[L - 1] + o] = acc;
  }
  double* Acur = A0;      // adjoint of the current layer's outputs: [13][pts][w]
  double* Aoth = A1;
  for (int idx = tid; idx < npts * fl; idx += THREADS) {
    const int pt = idx / fl, i = idx - pt * fl;
    const double* sd = SEED + (size_t)pt * SEEDW;
    const double w0 = __ldg(Wh + 2 * i), w1 = __ldg(Wh + 2 * i + 1);
#pragma unroll
    for (int s = 0; s < NST; s++) Acur[s * sl + (size_t)pt * fl + i] = fma(sd[2 * s], w0, sd[2 * s + 1] * w1);
  }
  __syncthreads();

  // ======================================= backward: hidden layers =======================================
  for (int l = L - 2; l >= 0; l--) {
    const int fi = nd.dims[l], fo = nd.dims[l + 1];
    const double* Wl = p.w + nd.woff[l];
    const double* Ho = Hs + hoff[l];
    const size_t so = (size_t)pts * fo, sp = (size_t)pts * fi;
    // (1) Z-bar
    for (int idx = tid; idx < npts * fo; idx += THREADS) {
      double A[NST], B[NST], Z[NST];
#pragma unroll
      for (int s = 0; s < NST; s++) { A[s] = Ho[s * so + idx]; B[s] = Acur[s * so + idx]; }
      zbar_streams(A, B, Z);
#pragma unroll
      for (int s = 0; s < NST; s++) Aoth[s * so + idx] = Z[s];
    }
    __syncthreads();
    if (l == 0) {
      // first layer: thread per entry (i, j), i == 3 is the bias; input streams as in the forward
      for (int e = tid; e < 4 * fo; e += THREADS) {
        const int i = e / fo, j = e - i * fo;
        double acc = 0.0;
        for (int pt = 0; pt < npts; pt++) {
          const double* z = Aoth + (size_t)pt * fo + j;
          if (i == 3) acc += z[0];
          else acc += fma(fma(p.sc[i], __ldg(p.X + 3 * (base + pt) + i) - p.lb[i], -1.0), z[0], p.sc[i] * z[(1 + i) * so]);
        }
        if (i < 3) outp[nd.woff[0] + i * fo + j] = acc;
        else outp[nd.boff[0] + j] = acc;
      }
      break;
    }
    // (2)+(3) on the tensor pipe, one item list: weight-gradient items (long: K = 13 streams x points) first, then the
    // input-adjoint items.  Both only read Z-bar (Aoth), the layer inputs and W_l; the adjoint overwrites Acur.
    const double* Hp = Hs + hoff[l - 1];
    const int nto = (fo + 7) >> 3, nti = (fi + 7) >> 3;
    const int items_w = ((fi + 1 + 15) >> 4) * nto, items = items_w + ((npts + 15) >> 4) * nti;
    if (tid == 0) work_ctr = 0;
    __syncthreads();
    for (int it = generic::next_item(&work_ctr, lane); it < items; it = generic::next_item(&work_ctr, lane)) {
      if (it < items_w) {
        // G[i][j] = sum_{s, pt} Hin[s][pt][i] Z[s][pt][j];  row fi: ones on the value stream (bias)
        const int mt = it / nto, n0 = 8 * (it - mt * nto);
        const int i_lo = 16 * mt + g, i_hi = i_lo + 8;
        const int ic_lo = min(i_lo, fi - 1), ic_hi = min(i_hi, fi - 1);
        const int n = n0 + g;
        const bool nok = n < fo;
        const int nc = nok ? n : fo - 1;
        double lo[2] = {0.0, 0.0}, hi[2] = {0.0, 0.0};
        const int kfull = npts >> 2;
#pragma unroll 1
        for (int s = 0; s < NST; s++) {
          const double one = s == 0 ? 1.0 : 0.0;
          const double* hq = Hp + s * sp + (size_t)q * fi;            // row pt0 + q of the layer inputs
          const double* zq = Aoth + s * so + (size_t)q * fo + nc;     // ... and of Z-bar
#pragma unroll 4
          for (int kk = 0; kk < kfull; kk++) {
            const double a_lo = i_lo == fi ? one : hq[ic_lo];
            const double a_hi = i_hi == fi ? one : hq[ic_hi];
            const double b = nok ? *zq : 0.0;
            dmma16x8x4(lo, hi, a_lo, a_hi, b);
            hq += 4 * fi;
            zq += 4 * fo;
          }
          if (npts & 3) {
            const bool ok = 4 * kfull + q < npts;
            const double a_lo = ok ? (i_lo == fi ? one : hq[ic_lo]) : 0.0;
            const double a_hi = ok ? (i_hi == fi ? one : hq[ic_hi]) : 0.0;
            const double b = (ok && nok) ? *zq : 0.0;
            dmma16x8x4(lo, hi, a_lo, a_hi, b);
          }
        }
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const int j = n0 + 2 * q + e;
          if (j < fo) {
            if (i_lo < fi) outp[nd.woff[l] + i_lo * fo + j] = lo[e];
            else if (i_lo == fi) outp[nd.boff[l] + j] = lo[e];
            if (i_hi < fi) outp[nd.woff[l] + i_hi * fo + j] = hi[e];
            else if (i_hi == fi) outp[nd.boff[l] + j] = hi[e];
          }
        }
      } else {
        // A-bar[l-1][s][pt][i] = sum_j Z[s][pt][j] W_l[i][j]
        const int ia = it - items_w;
        const int pt0 = 16 * (ia / nti), n0 = 8 * (ia - (ia / nti) * nti);
        const int n = n0 + g;
        double C[NST][2][2];
#pragma unroll
        for (int s = 0; s < NST; s++) C[s][0][0] = C[s][0][1] = C[s][1][0] = C[s][1][1] = 0.0;
        gemm13(C, Aoth, so, fo, fo, Wl, 1, fo, n < fi ? n : fi - 1, n < fi, min(pt0 + g, npts - 1), min(pt0 + g + 8, npts - 1), q);
#pragma unroll
        for (int hf = 0; hf < 2; hf++)
#pragma unroll
          for (int e = 0; e < 2; e++) {
            const int pt = pt0 + g + 8 * hf, i = n0 + 2 * q + e;
            if (pt < npts && i < fi) {
#pragma unroll
              for (int s = 0; s < NST; s++) Acur[s * sp + (size_t)pt * fi + i] = C[s][hf][e];
            }
          }
      }
    }
    __syncthreads();                                // Acur now holds A-bar of layer l-1
  }
}

// ---- probe: thread per point, off the per-step path (pinn_predict / pinn_derivatives / pinn_residual).
// mode 0: (psi, p) [n][2];  mode 1: all 13 streams [n][13][2];  mode 2: residuals (f_u, f_v) [n][2] with the lambdas of w.
// The streams of the current and the previous layer live in a global scratch [2][13][maxw][chunk] (coalesced over points).
struct Probe {
  double lb[3], sc[3];
  int p_net, maxw, mode;
  long long chunk;
};

__global__ void __launch_bounds__(128) probe_forward(const double* __restrict__ w, NetDesc nd, Probe pr, const double* __restrict__ X,
                                                     long long n, double* __restrict__ out, double* __restrict__ scr) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const int nst = pr.mode == 0 ? 1 : NST;
  const long long ch = pr.chunk;
  const size_t sstr = (size_t)pr.maxw * ch, bstr = (size_t)NST * sstr;
  double* cur = scr;
  double* nxt = scr + bstr;
  const int L = nd.n_layers;
  for (int l = 0; l < L - 1; l++) {
    const int fi = nd.dims[l], fo = nd.dims[l + 1];
    const double* Wl = w + nd.woff[l];
    const double* bl = w + nd.boff[l];
    for (int j = 0; j < fo; j++) {
      double z[NST], o[NST];
#pragma unroll
      for (int s = 0; s < NST; s++) z[s] = 0.0;
      z[0] = __ldg(bl + j);
      if (l == 0) {
#pragma unroll
        for (int i = 0; i < 3; i++) {
          const double wv = __ldg(Wl + i * fo + j);
          z[0] = fma(fma(pr.sc[i], X[3 * p + i] - pr.lb[i], -1.0), wv, z[0]);
          z[1 + i] = pr.sc[i] * wv;
        }
      } else {
        for (int i = 0; i < fi; i++) {
          const double wv = __ldg(Wl + i * fo + j);
#pragma unroll
          for (int s = 0; s < NST; s++)
            if (s < nst) z[s] = fma(cur[s * sstr + (size_t)i * ch + p], wv, z[s]);
        }
      }
      tanh_streams(tanh(z[0]), z, o);
#pragma unroll
      for (int s = 0; s < NST; s++)
        if (s < nst) nxt[s * sstr + (size_t)j * ch + p] = o[s];
    }
    double* t = cur; cur = nxt; nxt = t;
  }
  const int fl = nd.dims[L - 1];
  const double* Wh = w + nd.woff[L - 1];
  double O[NST][OUT];
#pragma unroll
  for (int o = 0; o < OUT; o++) {
    O[0][o] = __ldg(w + nd.boff[L - 1] + o);
#pragma unroll
    for (int s = 1; s < NST; s++) O[s][o] = 0.0;
  }
  for (int i = 0; i < fl; i++) {
    const double w0 = __ldg(Wh + 2 * i), w1 = __ldg(Wh + 2 * i + 1);
#pragma unroll
    for (int s = 0; s < NST; s++)
      if (s < nst) {
        const double h = cur[s * sstr + (size_t)i * ch + p];
        O[s][0] = fma(h, w0, O[s][0]);
        O[s][1] = fma(h, w1, O[s][1]);
      }
  }
  if (pr.mode == 1) {
#pragma unroll
    for (int s = 0; s < NST; s++) { out[p * SEEDW + 2 * s] = O[s][0]; out[p * SEEDW + 2 * s + 1] = O[s][1]; }
  } else if (pr.mode == 2) {
    const double l1 = w[pr.p_net], l2 = w[pr.p_net + 1];
    const double px = O[1][0], py = O[2][0], pxx = O[4][0], pxy = O[5][0], pyy = O[6][0];
    out[2 * p] = fma(-l2, O[10][0] + O[12][0], fma(l1, fma(py, pxy, -px * pyy), O[8][0] + O[1][1]));
    out[2 * p + 1] = fma(l2, O[9][0] + O[11][0], fma(l1, fma(px, pxy, -py * pxx), O[2][1] - O[7][0]));
  } else {
    out[2 * p] = O[0][0];
    out[2 * p + 1] = O[0][1];
  }
}

}  // namespace nsid
}  // namespace pinn
