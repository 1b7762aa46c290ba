// Residual-based adaptive resampling of the collocation set on the device (pinn_draw_collocation_rad; DESIGN §4.7).
//
// After the pool (rows [0, n_pool) of a Latin-hypercube draw, lhs::draw_kernel) and its probe streams (mlp_forward_generic<4, W>)
// are on the device, three kernels finish the draw:
//   head_kernel     f at every pool point, in the operation order of pinn_residual's host head and explicitly rounded, so f is
//                   the value pinn_residual returns bit for bit; r = |f| (Burgers) or sqrt(f_u^2 + f_v^2) (Schrodinger);
//                   a = r^k as left-to-right products (k = 0: 1); one maximum of the finite a per block.
//   quantise_kernel amax over the block maxima; A = 2^24 for a non-finite a, else floor((a / amax) * 2^24) (0 when amax = 0);
//                   block b owns the contiguous segment [b seg, (b + 1) seg) and writes the inclusive prefix of A within it
//                   and the segment's sum.
//   pick_kernel     the exclusive prefix of the segment sums gives S = sum A and the global prefix of A; C' = floor(c S / n_pool)
//                   and Q = A + C' (every Q = 1 when T = S + n_pool C' = 0) make the inclusive prefix of Q at i
//                   P_i = prefix_A(i) + (i + 1) C'.  Row j draws target = mulhi64(w0 << 32 | w1, T) from one Philox4x32-10
//                   block with counter (lo j, hi j, lo draw, hi draw) and key (lo seed ^ RAD_SALT0, hi seed ^ RAD_SALT1), takes
//                   the least i with P_i > target by binary search, and copies pool point i to the collocation region.
// Every integer step is exact (A <= 2^24, S <= n_pool 2^24 <= 2^53, T < 2^64), so the picks do not depend on the grid or on the
// order of any sum.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "lhs_draw.cuh"

namespace pinn {
namespace rad {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;
constexpr int MAX_BLOCKS = 1024;                 // grid of head_kernel and quantise_kernel: pick_kernel keeps their sums in smem
constexpr long long MAX_POOL = 1LL << 29;        // keeps S <= 2^53 (exact in fp64) and T < 2^64 with c <= MAX_C
constexpr double MAX_C = 1024.0;
constexpr double SCALE = 0x1p24;                 // the weight of a point with a = amax, and of a non-finite a
// the pick key differs from both keys of the LHS draw: (lo seed, hi seed) and (lo seed ^ KEY_SALT0, hi seed ^ KEY_SALT1)
constexpr uint32_t RAD_SALT0 = 0xBF58476Du, RAD_SALT1 = 0x1CE4E5B9u;
static_assert(RAD_SALT0 != lhs::KEY_SALT0 || RAD_SALT1 != lhs::KEY_SALT1, "the pick key must differ from the permutation key");

struct Args {
  const double* streams;          // [n_pool][4][no] of mlp_forward_generic<4, W>: (h, h_x, h_t, h_xx) per output
  const double *px, *pt;          // the pool
  double* a;                      // [n_pool] r^k
  uint64_t* lp;                   // [n_pool] inclusive prefix of A within each segment
  double* bmax;                   // [grid] largest finite a of each head block
  uint64_t* bsum;                 // [grid] sum of A over each segment
  double *x, *t;                  // rows [0, n) of the new collocation set
  uint64_t n_pool, seg, n, seed, draw;
  int grid;                       // blocks of head_kernel and quantise_kernel (<= MAX_BLOCKS)
  int nls;                        // 0: Burgers f = u_t + u u_x - nu u_xx; 1: Schrodinger (f_u, f_v)
  int k;                          // 0..4
  double nu, c;
};

// inclusive scan of one value per thread over the block; total = the block's sum.  s holds WARPS entries.
__device__ __forceinline__ uint64_t block_scan(uint64_t v, uint64_t* s, uint64_t& total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint64_t y = __shfl_up_sync(0xFFFFFFFFu, v, o);
    if (lane >= o) v += y;
  }
  if (lane == 31) s[w] = v;
  __syncthreads();
  uint64_t before = 0, all = 0;
#pragma unroll
  for (int j = 0; j < WARPS; j++) {
    const uint64_t sj = s[j];
    before += j < w ? sj : 0;
    all += sj;
  }
  __syncthreads();                // s is reused by the next call
  total = all;
  return before + v;
}

// the block's maximum of non-negative finite values, returned to every thread.  s holds WARPS entries.
__device__ __forceinline__ double block_max(double m, double* s) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xFFFFFFFFu, m, o));
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = m;
  __syncthreads();
  m = s[0];
#pragma unroll
  for (int j = 1; j < WARPS; j++) m = fmax(m, s[j]);
  return m;
}

__global__ void __launch_bounds__(THREADS) head_kernel(Args a) {
  __shared__ double s[WARPS];
  double m = 0.0;
  for (uint64_t i = (uint64_t)blockIdx.x * THREADS + threadIdx.x; i < a.n_pool; i += (uint64_t)gridDim.x * THREADS) {
    double r;
    if (a.nls) {
      // pinn_residual: h2 = u*u + v*v; f_u = ut + 0.5*vxx + h2*v; f_v = vt - 0.5*uxx - h2*u
      const double* d = a.streams + i * 8;
      const double u = d[0], v = d[1], ut = d[4], vt = d[5], uxx = d[6], vxx = d[7];
      const double h2 = __dadd_rn(__dmul_rn(u, u), __dmul_rn(v, v));
      const double fu = __dadd_rn(__dadd_rn(ut, __dmul_rn(0.5, vxx)), __dmul_rn(h2, v));
      const double fv = __dsub_rn(__dsub_rn(vt, __dmul_rn(0.5, uxx)), __dmul_rn(h2, u));
      r = __dsqrt_rn(__dadd_rn(__dmul_rn(fu, fu), __dmul_rn(fv, fv)));
    } else {
      // pinn_residual: d[2] + l1 * d[0] * d[1] - kap * d[3] with l1 = 1, kap = nu
      const double* d = a.streams + i * 4;
      r = fabs(__dsub_rn(__dadd_rn(d[2], __dmul_rn(__dmul_rn(1.0, d[0]), d[1])), __dmul_rn(a.nu, d[3])));
    }
    double p = a.k ? r : 1.0;
    for (int j = 1; j < a.k; j++) p = __dmul_rn(p, r);
    a.a[i] = p;
    if (isfinite(p)) m = fmax(m, p);
  }
  m = block_max(m, s);
  if (threadIdx.x == 0) a.bmax[blockIdx.x] = m;
}

__global__ void __launch_bounds__(THREADS) quantise_kernel(Args a) {
  __shared__ double sm[WARPS];
  __shared__ uint64_t ss[WARPS];
  double m = 0.0;
  for (int b = threadIdx.x; b < a.grid; b += THREADS) m = fmax(m, a.bmax[b]);
  const double amax = block_max(m, sm);
  const uint64_t lo = min((uint64_t)blockIdx.x * a.seg, a.n_pool), hi = min(lo + a.seg, a.n_pool);
  uint64_t carry = 0;
  for (uint64_t base = lo; base < hi; base += THREADS) {
    const uint64_t i = base + threadIdx.x;
    uint64_t A = 0;
    if (i < hi) {
      const double v = a.a[i];
      if (!isfinite(v)) A = (uint64_t)SCALE;
      else if (amax > 0.0) A = __double2ull_rz(__dmul_rn(__ddiv_rn(v, amax), SCALE));    // floor: the value is in [0, 2^24]
    }
    uint64_t total;
    const uint64_t inc = block_scan(A, ss, total);
    if (i < hi) a.lp[i] = carry + inc;
    carry += total;
  }
  if (threadIdx.x == 0) a.bsum[blockIdx.x] = carry;
}

__global__ void __launch_bounds__(THREADS) pick_kernel(Args a) {
  __shared__ uint64_t base[MAX_BLOCKS];
  __shared__ uint64_t ss[WARPS];
  uint64_t S = 0;
  for (int b0 = 0; b0 < a.grid; b0 += THREADS) {
    const int b = b0 + threadIdx.x;
    const uint64_t v = b < a.grid ? a.bsum[b] : 0;
    uint64_t total;
    const uint64_t inc = block_scan(v, ss, total);
    if (b < a.grid) base[b] = S + inc - v;
    S += total;
  }
  __syncthreads();
  // C' = floor(c S / n_pool): (double)S and (double)n_pool are exact, the product and the quotient are rounded
  uint64_t cq = __double2ull_rz(__ddiv_rn(__dmul_rn(a.c, (double)S), (double)a.n_pool));
  if (S == 0 && cq == 0) cq = 1;                                  // T = 0: every Q_i = 1 (every A_i is 0)
  const uint64_t T = S + a.n_pool * cq;
  const uint32_t k0 = (uint32_t)a.seed ^ RAD_SALT0, k1 = (uint32_t)(a.seed >> 32) ^ RAD_SALT1;
  const uint32_t dlo = (uint32_t)a.draw, dhi = (uint32_t)(a.draw >> 32);
  for (uint64_t j = (uint64_t)blockIdx.x * THREADS + threadIdx.x; j < a.n; j += (uint64_t)gridDim.x * THREADS) {
    const lhs::Block w = lhs::philox((uint32_t)j, (uint32_t)(j >> 32), dlo, dhi, k0, k1);
    const uint64_t target = __umul64hi(((uint64_t)w.w0 << 32) | w.w1, T);     // in [0, T)
    uint64_t lo = 0, hi = a.n_pool - 1;                                          // P_{n_pool - 1} = T > target
    while (lo < hi) {
      const uint64_t mid = lo + (hi - lo) / 2;
      if (base[mid / a.seg] + a.lp[mid] + (mid + 1) * cq > target) hi = mid;
      else lo = mid + 1;
    }
    a.x[j] = a.px[lo];
    a.t[j] = a.pt[lo];
  }
}

}  // namespace rad
}  // namespace pinn
