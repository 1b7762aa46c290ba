// Latin-hypercube collocation draw on the device (pinn_draw_collocation; DESIGN §4.6).
//
// A draw is a pure function of (seed, draw, N, lb, ub); row i of it is
//   u_d  = 53-bit uniform of Philox4x32-10 with counter (lo(i), hi(i), lo(draw), hi(draw)) and key (lo(seed), hi(seed)):
//          u_x = ((w0 >> 11) << 32 | w1) * 2^-53, u_t = ((w2 >> 11) << 32 | w3) * 2^-53;
//   p_d  = pi_d(i), a keyed permutation of [0, N): a balanced Feistel network on 2m bits (4^m >= N, m >= 1) with ROUNDS rounds,
//          round function = word 0 of Philox4x32-10 on (R, round | d << 8, lo(draw), hi(draw)) under the key
//          (lo(seed) ^ KEY_SALT0, hi(seed) ^ KEY_SALT1), cycle-walked down to [0, N);
//   x_d  = lb_d + (ub_d - lb_d) * ((p_d + u_d) / N), in fp64 and in that order (explicitly rounded: no FMA contraction).
// Each dimension then holds exactly one point per stratum [k/N, (k+1)/N].  Rows are independent, so a shard [first, first + n)
// computes its rows without the others and the union of the shards is the whole-set draw.  Philox and the Feistel network
// are written out here rather than taken from curand so that a host restatement can follow the same integer steps.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pinn {
namespace lhs {

constexpr int THREADS = 256;
constexpr int ROUNDS = 4;                       // Feistel rounds (4 rounds of a pseudo-random function: a pseudo-random permutation)
constexpr uint32_t KEY_SALT0 = 0x5851F42Du, KEY_SALT1 = 0x4C957F2Du;

struct Args {
  double *x, *t;                  // rows [first, first + n) go to x[0..n), t[0..n)
  uint64_t seed, draw, first, n, n_global;
  double lb0, lb1, dx0, dx1;      // dx = ub - lb
  int m;                          // half width of the Feistel domain in bits: the least m >= 1 with 4^m >= n_global
};

struct Block { uint32_t w0, w1, w2, w3; };

// Philox4x32-10 (Salmon et al., SC'11; the Random123 constants)
__device__ __forceinline__ Block philox(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; r++) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return Block{c0, c1, c2, c3};
}

__device__ __forceinline__ double uniform53(uint32_t a, uint32_t b) {
  return (double)(((uint64_t)(a >> 11) << 32) | b) * 0x1p-53;      // exact: a 53-bit integer times a power of two
}

// pi_d(i) for i < N: the Feistel network, re-applied until the value falls below N.  The walk follows the cycle of the
// 4^m-point permutation through i, which returns to i < N, so it ends; on average over a draw it takes at most 4^m / N
// applications (< 4 for N >= 2).
__device__ __forceinline__ uint64_t permute(uint64_t v, const Args& a, uint32_t d, uint32_t kf0, uint32_t kf1) {
  const uint32_t half = (1u << a.m) - 1u;
  const uint32_t dlo = (uint32_t)a.draw, dhi = (uint32_t)(a.draw >> 32);
  do {
    uint32_t L = (uint32_t)(v >> a.m), R = (uint32_t)v & half;
#pragma unroll
    for (uint32_t r = 0; r < ROUNDS; r++) {
      const uint32_t f = philox(R, r | (d << 8), dlo, dhi, kf0, kf1).w0 & half;
      const uint32_t nr = L ^ f;
      L = R; R = nr;
    }
    v = ((uint64_t)L << a.m) | R;
  } while (v >= a.n_global);
  return v;
}

__device__ __forceinline__ double place(double lb, double dx, uint64_t p, double u, double N) {
  return __dadd_rn(lb, __dmul_rn(dx, __ddiv_rn(__dadd_rn((double)p, u), N)));
}

__global__ void __launch_bounds__(THREADS) draw_kernel(Args a) {
  const uint32_t s0 = (uint32_t)a.seed, s1 = (uint32_t)(a.seed >> 32);
  const uint32_t dlo = (uint32_t)a.draw, dhi = (uint32_t)(a.draw >> 32);
  const double N = (double)a.n_global;                                // exact: n_global <= 2^53
  for (uint64_t k = (uint64_t)blockIdx.x * THREADS + threadIdx.x; k < a.n; k += (uint64_t)gridDim.x * THREADS) {
    const uint64_t i = a.first + k;
    const Block w = philox((uint32_t)i, (uint32_t)(i >> 32), dlo, dhi, s0, s1);
    const uint64_t px = permute(i, a, 0, s0 ^ KEY_SALT0, s1 ^ KEY_SALT1);
    const uint64_t pt = permute(i, a, 1, s0 ^ KEY_SALT0, s1 ^ KEY_SALT1);
    a.x[k] = place(a.lb0, a.dx0, px, uniform53(w.w0, w.w1), N);
    a.t[k] = place(a.lb1, a.dx1, pt, uniform53(w.w2, w.w3), N);
  }
}

// the least m >= 1 with 4^m >= n (n <= 2^53, so m <= 27 and both halves fit 32 bits)
inline int half_bits(uint64_t n) {
  int m = 1;
  while (m < 27 && (n - 1) >> (2 * m)) m++;
  return m;
}

}  // namespace lhs
}  // namespace pinn
