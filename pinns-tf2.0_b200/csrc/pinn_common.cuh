// Shared device helpers for the fused PINN kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pinn {

// ---- FP64 tensor-core MMA: D(8x8) += A(8x4) * B(4x8); SASS DMMA.8x8x4 (the FP64 MMA shape these kernels are written
// for; SASS DMMA.8x8x4 on sm_90a).  Fragment ownership, lane = 4*g + q:
//   A[row g][col q]      B[row q][col g]      C/D[row g][cols 2q, 2q+1]
__device__ __forceinline__ void dmma(double (&c)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c[0]), "+d"(c[1])
               : "d"(a), "d"(b));
}

// ---- Hopper's 16x8 FP64 MMA shapes; SASS DMMA.16x8x4 / DMMA.16x8x8, native on sm_90a and twice the FMA rate of DMMA.8x8x4
// there (profiles/microbench/fp64_peak_h100.jsonl).  The accumulator is two 8x8 halves laid out like the m8n8k4 C fragment:
//   C/D: lo = [row g][cols 2q, 2q+1],  hi = [row g+8][cols 2q, 2q+1]
// m16n8k4,  D(16x8) += A(16x4) * B(4x8):   a_lo = A[g][q], a_hi = A[g+8][q];   b = B[q][g]
__device__ __forceinline__ void dmma16x8x4(double (&lo)[2], double (&hi)[2], double a_lo, double a_hi, double b) {
  asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
               : "+d"(lo[0]), "+d"(lo[1]), "+d"(hi[0]), "+d"(hi[1])
               : "d"(a_lo), "d"(a_hi), "d"(b));
}
// m16n8k8,  D(16x8) += A(16x8) * B(8x8):   a0 = A[g][q], a1 = A[g+8][q], a2 = A[g][q+4], a3 = A[g+8][q+4];
//                                          b0 = B[q][g], b1 = B[q+4][g]
__device__ __forceinline__ void dmma16x8x8(double (&lo)[2], double (&hi)[2], double a0, double a1, double a2, double a3,
                                           double b0, double b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+d"(lo[0]), "+d"(lo[1]), "+d"(hi[0]), "+d"(hi[1])
               : "d"(a0), "d"(a1), "d"(a2), "d"(a3), "d"(b0), "d"(b1));
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier + TMA bulk copy (global -> shared, 1-D): SASS UBLKCP.  Used to stage the flat weight
// vector into shared memory with a single asynchronous copy.
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// asynchronous L2 prefetch of a contiguous global range (16-byte aligned, size a multiple of 16): one instruction, no registers
__device__ __forceinline__ void prefetch_l2_bulk(const void* src_gmem, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src_gmem), "r"(bytes) : "memory");
}

__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// orders this thread's earlier generic-proxy writes (shared and global) before later async-proxy (TMA) accesses
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  }
}

// ---- branch-free fp64 tanh (<= 2.5 ulp, full relative accuracy down to denormals), built so that several
// evaluations interleave (no divergent branches; libdevice tanh serialises into 11-cycle DFMA chains):
//   em = expm1(-2|x|) = 2^n p(r) + (2^n - 1),  p(r) = e^r - 1 (degree-13 Taylor, |r| <= ln2/2)
//   tanh|x| = -em / (2 + em),  division by MUFU.RCP64H seed + 1 Newton step + one residual correction.
#ifndef PINN_TANH_NEWTON1
#define PINN_TANH_NEWTON1 1               // one Newton step on the reciprocal seed instead of two: the residual correction of the
#endif                                    // quotient squares the remaining error once more (measured: <= 4 ulp kept, -1 % kernel time)
__device__ __forceinline__ double tanh_fast(double x) {
  // tanh(20) rounds to 1.0.  A NaN fails the test and flows through to copysign (NaN in, NaN out, as libm); fmin would return
  // 20 and make it +-1.  The compiler folds the select after -2|x|, so the FP64-pipe instruction counts are fmin's.
  const double ax = fabs(x) > 20.0 ? 20.0 : fabs(x);
  const double y = -2.0 * ax;
  const double SHIFT = 6755399441055744.0;      // 1.5 * 2^52: round-to-nearest-integer trick
  const double t = fma(y, 1.4426950408889634, SHIFT);
  const int n = __double2loint(t);
  const double nd = t - SHIFT;
  double r = fma(nd, -6.93147180369123816490e-01, y);
  r = fma(nd, -1.90821492927058770002e-10, r);
  double q = 1.6059043836821613e-10;            // 1/13!
  q = fma(q, r, 2.08767569878681e-09);          // 1/12!
  q = fma(q, r, 2.505210838544172e-08);         // 1/11!
  q = fma(q, r, 2.755731922398589e-07);         // 1/10!
  q = fma(q, r, 2.7557319223985893e-06);        // 1/9!
  q = fma(q, r, 2.48015873015873e-05);          // 1/8!
  q = fma(q, r, 0.0001984126984126984);         // 1/7!
  q = fma(q, r, 0.001388888888888889);          // 1/6!
  q = fma(q, r, 0.008333333333333333);          // 1/5!
  q = fma(q, r, 0.041666666666666664);          // 1/4!
  q = fma(q, r, 0.16666666666666666);           // 1/3!
  q = fma(q, r, 0.5);                           // 1/2!
  const double p = fma(r * r, q, r);            // e^r - 1
  const double scale = __hiloint2double((1023 + n) << 20, 0);   // 2^n, n in [-58, 0]
  const double em = fma(scale, p, scale - 1.0);
  const double den = 2.0 + em;                  // in [1, 2]
  double rc;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(rc) : "d"(den));
  double e = fma(-den, rc, 1.0);
  rc = fma(rc, e, rc);
#if !PINN_TANH_NEWTON1
  e = fma(-den, rc, 1.0);
  rc = fma(rc, e, rc);
#endif
  const double num = -em;
  double qd = num * rc;
  qd = fma(fma(-den, qd, num), rc, qd);
  return copysign(qd, x);
}

__device__ __forceinline__ double shfl_xor_d(double v, int m) { return __shfl_xor_sync(0xffffffffu, v, m); }
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) v += shfl_xor_d(v, m);
  return v;
}

}  // namespace pinn
