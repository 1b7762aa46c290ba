// FP64 pipe microbenchmark for H100 (sm_90a): DFMA peak, DMMA.8x8x4 peak, dependent-chain
// latencies, and whether DFMA and DMMA issue concurrently; then the same for the 16x8 shapes
// (DMMA.16x8x4/8/16) and a check of their fragment layouts.  Gives the roofline denominator for
// the fused PINN kernels (MEASURED_PEAKS.json carries no FP64 figure).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_peak fp64_peak.cu
#include <cstdio>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); return 1; } } while (0)

template <int ILP>
__global__ void dfma_kernel(double* out, int iters, double x) {
  double acc[ILP];
#pragma unroll
  for (int i = 0; i < ILP; i++) acc[i] = threadIdx.x * 1e-9 + i;
  double m = x;
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < ILP; i++) acc[i] = fma(acc[i], m, 1e-30);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < ILP; i++) s += acc[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

template <int ILP>
__global__ void dmma_kernel(double* out, int iters, double x) {
  double c0[ILP], c1[ILP];
#pragma unroll
  for (int i = 0; i < ILP; i++) { c0[i] = 0; c1[i] = 0; }
  double a = x * 1e-3 + threadIdx.x * 1e-12, b = x * 1e-3;
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < ILP; i++) dmma(c0[i], c1[i], a, b);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < ILP; i++) s += c0[i] + c1[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// mixed: per iteration NM DMMAs and NF DFMAs (independent chains)
template <int NM, int NF>
__global__ void mixed_kernel(double* out, int iters, double x) {
  double c0[NM + 1], c1[NM + 1], f[NF + 1];
#pragma unroll
  for (int i = 0; i < NM; i++) { c0[i] = 0; c1[i] = 0; }
#pragma unroll
  for (int i = 0; i < NF; i++) f[i] = i + threadIdx.x * 1e-9;
  double a = x * 1e-3 + threadIdx.x * 1e-12, b = x * 1e-3;
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < NM; i++) dmma(c0[i], c1[i], a, b);
#pragma unroll
    for (int i = 0; i < NF; i++) f[i] = fma(f[i], x, 1e-30);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < NM; i++) s += c0[i] + c1[i];
#pragma unroll
  for (int i = 0; i < NF; i++) s += f[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// ---- the Hopper FP64 MMA shapes.  S: 0 = m8n8k4, 1 = m16n8k4, 2 = m16n8k8, 3 = m16n8k16.  Fragments (lane = 4g + q):
// A a_i = (row g + 8 (i & 1), col q + 4 (i >> 1)) for M = 16 (m8n8k4: a0 = (g, q)); B b_i = (row q + 4 i, col g);
// C c_i = (row g + 8 (i >> 1), col 2q + (i & 1)).  layout_check() verifies these against a host GEMM.
template <int S> struct Shape;
template <> struct Shape<0> { static constexpr int M = 8, K = 4, NA = 1, NB = 1, NC = 2; static constexpr const char* name = "m8n8k4"; };
template <> struct Shape<1> { static constexpr int M = 16, K = 4, NA = 2, NB = 1, NC = 4; static constexpr const char* name = "m16n8k4"; };
template <> struct Shape<2> { static constexpr int M = 16, K = 8, NA = 4, NB = 2, NC = 4; static constexpr const char* name = "m16n8k8"; };
template <> struct Shape<3> { static constexpr int M = 16, K = 16, NA = 8, NB = 4, NC = 4; static constexpr const char* name = "m16n8k16"; };

template <int S>
__device__ __forceinline__ void mma_s(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
  if (S == 0)
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(c[0]), "+d"(c[1]) : "d"(a[0]), "d"(b[0]));
  else if (S == 1)
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(b[0]));
  else if (S == 2)
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
  else
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
                 "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                   "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

template <int S, int ILP>
__global__ void mma_kernel(double* out, int iters, double x) {
  double c[ILP][4], a[8], b[4];
#pragma unroll
  for (int i = 0; i < ILP; i++) c[i][0] = c[i][1] = c[i][2] = c[i][3] = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) a[i] = x * 1e-3 + threadIdx.x * 1e-12 + i * 1e-9;
#pragma unroll
  for (int i = 0; i < 4; i++) b[i] = x * 1e-3 + i * 1e-9;
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < ILP; i++) mma_s<S>(c[i], a, b);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < ILP; i++) s += c[i][0] + c[i][1] + c[i][2] + c[i][3];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int S, int NM, int NF>
__global__ void mixed_mma_kernel(double* out, int iters, double x) {
  double c[NM + 1][4], a[8], b[4], f[NF + 1];
#pragma unroll
  for (int i = 0; i < NM; i++) c[i][0] = c[i][1] = c[i][2] = c[i][3] = 0;
#pragma unroll
  for (int i = 0; i < NF; i++) f[i] = i + threadIdx.x * 1e-9;
#pragma unroll
  for (int i = 0; i < 8; i++) a[i] = x * 1e-3 + threadIdx.x * 1e-12 + i * 1e-9;
#pragma unroll
  for (int i = 0; i < 4; i++) b[i] = x * 1e-3 + i * 1e-9;
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < NM; i++) mma_s<S>(c[i], a, b);
#pragma unroll
    for (int i = 0; i < NF; i++) f[i] = fma(f[i], x, 1e-30);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < NM; i++) s += c[i][0] + c[i][1] + c[i][2] + c[i][3];
#pragma unroll
  for (int i = 0; i < NF; i++) s += f[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// one warp: C = A B with A[m][k] = m + 16 k + 1, B[k][n] = (k + 1) (n + 2) (exact in fp64), fragments as documented above
template <int S>
__global__ void layout_kernel(double* c_out) {
  using Sh = Shape<S>;
  const int g = threadIdx.x >> 2, q = threadIdx.x & 3;
  double a[8] = {0, 0, 0, 0, 0, 0, 0, 0}, b[4] = {0, 0, 0, 0}, c[4] = {0, 0, 0, 0};
  for (int i = 0; i < Sh::NA; i++) {
    const int m = g + (Sh::M == 16 ? 8 * (i & 1) : 0), k = q + 4 * (Sh::M == 16 ? i >> 1 : i);
    a[i] = m + 16 * k + 1;
  }
  for (int i = 0; i < Sh::NB; i++) b[i] = (q + 4 * i + 1) * (g + 2);
  mma_s<S>(c, a, b);
  for (int i = 0; i < Sh::NC; i++) c_out[(g + 8 * (i >> 1)) * 8 + 2 * q + (i & 1)] = c[i];
}

template <int S>
int layout_check(double* dev) {
  using Sh = Shape<S>;
  CK(cudaMemset(dev, 0, 16 * 8 * sizeof(double)));
  layout_kernel<S><<<1, 32>>>(dev);
  double c[128];
  CK(cudaMemcpy(c, dev, sizeof(c), cudaMemcpyDeviceToHost));
  int bad = 0;
  for (int m = 0; m < Sh::M; m++)
    for (int n = 0; n < 8; n++) {
      double r = 0;
      for (int k = 0; k < Sh::K; k++) r += (double)(m + 16 * k + 1) * ((k + 1) * (n + 2));
      bad += c[m * 8 + n] != r;
    }
  printf("{\"shape\": \"%s\", \"fragment_layout_ok\": %s}\n", Sh::name, bad ? "false" : "true");
  return 0;
}

// FP32 FFMA for context
template <int ILP>
__global__ void ffma_kernel(float* out, int iters, float x) {
  float acc[ILP];
#pragma unroll
  for (int i = 0; i < ILP; i++) acc[i] = threadIdx.x * 1e-9f + i;
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int i = 0; i < ILP; i++) acc[i] = fmaf(acc[i], x, 1e-30f);
  }
  float s = 0;
#pragma unroll
  for (int i = 0; i < ILP; i++) s += acc[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <typename F>
float time_ms(F launch, int reps = 5) {
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  launch(); cudaDeviceSynchronize();
  float best = 1e30f;
  for (int r = 0; r < reps; r++) {
    cudaEventRecord(e0); launch(); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1); if (ms < best) best = ms;
  }
  return best;
}

// per shape: throughput at 1, 2 and 4 warps per sub-partition (ILP 8), the ILP sweep at one warp per sub-partition, and
// the DMMA + DFMA mix.  "cyc_per_256fma" = issue cycles of one sub-partition per 256 FMAs (DMMA.8x8x4 = 1 instruction),
// at the maximum SM clock.
template <int S>
int shape_sweep(int sms, int clk_khz, double* out) {
  using Sh = Shape<S>;
  const int iters = 4096;
  const double fma_per_op = Sh::M * 8.0 * Sh::K;
  const double cyc_per_ms = clk_khz;   // kHz = cycles per ms
  for (int wpsp : {1, 2, 4}) {
    const int grid = sms * 4, threads = 32 * wpsp;
    float ms = time_ms([&] { mma_kernel<S, 8><<<grid, threads>>>(out, iters, 0.999); });
    CK(cudaGetLastError());
    const double ops_per_smsp = (double)wpsp * 8 * iters;
    printf("{\"shape\": \"%s\", \"warps_per_smsp\": %d, \"tflops\": %.2f, \"cyc_per_op\": %.2f, \"cyc_per_256fma\": %.2f}\n", Sh::name,
           wpsp, 2.0 * fma_per_op * ops_per_smsp * 4 * sms / ms / 1e9, ms * cyc_per_ms / ops_per_smsp,
           ms * cyc_per_ms / ops_per_smsp * 256.0 / fma_per_op);
  }
  {
    const int grid = sms * 4, threads = 32;
    float m1 = time_ms([&] { mma_kernel<S, 1><<<grid, threads>>>(out, iters, 0.999); });
    float m2 = time_ms([&] { mma_kernel<S, 2><<<grid, threads>>>(out, iters, 0.999); });
    float m4 = time_ms([&] { mma_kernel<S, 4><<<grid, threads>>>(out, iters, 0.999); });
    float m8 = time_ms([&] { mma_kernel<S, 8><<<grid, threads>>>(out, iters, 0.999); });
    CK(cudaGetLastError());
    printf("{\"shape\": \"%s\", \"one_warp_per_smsp\": true, \"cyc_per_op\": {\"ilp1\": %.2f, \"ilp2\": %.2f, \"ilp4\": %.2f, \"ilp8\": %.2f}}\n",
           Sh::name, m1 * cyc_per_ms / iters, m2 * cyc_per_ms / iters / 2, m4 * cyc_per_ms / iters / 4, m8 * cyc_per_ms / iters / 8);
  }
  for (int wpsp : {1, 2}) {
    const int grid = sms * 4, threads = 32 * wpsp;
    float mm = time_ms([&] { mixed_mma_kernel<S, 8, 0><<<grid, threads>>>(out, iters, 0.999); });
    float ff = time_ms([&] { mixed_mma_kernel<S, 0, 16><<<grid, threads>>>(out, iters, 0.999); });
    float mf = time_ms([&] { mixed_mma_kernel<S, 8, 16><<<grid, threads>>>(out, iters, 0.999); });
    CK(cudaGetLastError());
    printf("{\"shape\": \"%s\", \"warps_per_smsp\": %d, \"ms_dmma8\": %.4f, \"ms_dfma16\": %.4f, \"ms_both\": %.4f, \"overlap\": %.2f}\n",
           Sh::name, wpsp, mm, ff, mf, (mm + ff - mf) / (mm < ff ? mm : ff));
  }
  return 0;
}

int main() {
  cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
  int sms = prop.multiProcessorCount;
  int clk_khz = 0; cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
  printf("{\"device\": \"%s\", \"sms\": %d, \"max_clock_mhz\": %.0f}\n", prop.name, sms, clk_khz / 1e3);
  double* out; CK(cudaMalloc(&out, sizeof(double) * sms * 64 * 1024));
  const int iters = 4096;
  // sweep warps per SM for DFMA and DMMA at ILP 8
  int wps[] = {1, 2, 4, 8, 16, 32};
  for (int w : wps) {
    int threads = 32 * (w < 4 ? 1 : w / 4) ; int blocks_per_sm = w < 4 ? w : 4;
    int grid = sms * blocks_per_sm;
    float ms = time_ms([&] { dfma_kernel<8><<<grid, threads>>>(out, iters, 0.999); });
    double flops = 2.0 * grid * threads * 8.0 * iters;
    float ms2 = time_ms([&] { dmma_kernel<8><<<grid, threads>>>(out, iters, 0.999); });
    double flops2 = 2.0 * 256.0 * grid * (threads / 32) * 8.0 * iters;
    printf("{\"warps_per_sm\": %d, \"dfma_tflops\": %.2f, \"dmma_tflops\": %.2f}\n", w, flops / ms / 1e9, flops2 / ms2 / 1e9);
  }
  // ILP sweep at 4 warps/SM (1 per SMSP): exposes latency
  {
    int grid = sms * 4, threads = 32;
    float a1 = time_ms([&] { dfma_kernel<1><<<grid, threads>>>(out, iters, 0.999); });
    float a2 = time_ms([&] { dfma_kernel<2><<<grid, threads>>>(out, iters, 0.999); });
    float a4 = time_ms([&] { dfma_kernel<4><<<grid, threads>>>(out, iters, 0.999); });
    float a16 = time_ms([&] { dfma_kernel<16><<<grid, threads>>>(out, iters, 0.999); });
    float m1 = time_ms([&] { dmma_kernel<1><<<grid, threads>>>(out, iters, 0.999); });
    float m2 = time_ms([&] { dmma_kernel<2><<<grid, threads>>>(out, iters, 0.999); });
    float m4 = time_ms([&] { dmma_kernel<4><<<grid, threads>>>(out, iters, 0.999); });
    float m12 = time_ms([&] { dmma_kernel<12><<<grid, threads>>>(out, iters, 0.999); });
    // ns per dependent op = ms*1e6/iters/ILP... report cycles at max clock
    double cyc = clk_khz * 1e3 * 1e-3;  // cycles per ms
    printf("{\"one_warp_per_smsp\": true, \"dfma_cyc_per_op\": {\"ilp1\": %.2f, \"ilp2\": %.2f, \"ilp4\": %.2f, \"ilp16\": %.2f}, "
           "\"dmma_cyc_per_op\": {\"ilp1\": %.2f, \"ilp2\": %.2f, \"ilp4\": %.2f, \"ilp12\": %.2f}}\n",
           a1 * cyc / iters / 1, a2 * cyc / iters / 2, a4 * cyc / iters / 4, a16 * cyc / iters / 16,
           m1 * cyc / iters / 1, m2 * cyc / iters / 2, m4 * cyc / iters / 4, m12 * cyc / iters / 12);
  }
  // mixed at 4 and 8 warps/SM
  for (int w : {4, 8, 16}) {
    int threads = 32 * (w / 4), grid = sms * 4;
    float mm = time_ms([&] { mixed_kernel<8, 0><<<grid, threads>>>(out, iters, 0.999); });
    float ff = time_ms([&] { mixed_kernel<0, 16><<<grid, threads>>>(out, iters, 0.999); });
    float mf = time_ms([&] { mixed_kernel<8, 16><<<grid, threads>>>(out, iters, 0.999); });
    printf("{\"warps_per_sm\": %d, \"ms_dmma8\": %.4f, \"ms_dfma16\": %.4f, \"ms_both\": %.4f, \"overlap\": %.2f}\n", w, mm, ff, mf,
           (mm + ff - mf) / (mm < ff ? mm : ff));
  }
  {
    int grid = sms * 4, threads = 256;
    float ms = time_ms([&] { ffma_kernel<8><<<grid, threads>>>((float*)out, iters, 0.999f); });
    printf("{\"ffma_tflops\": %.2f}\n", 2.0 * grid * threads * 8.0 * iters / ms / 1e9);
  }
  if (layout_check<0>(out) || layout_check<1>(out) || layout_check<2>(out) || layout_check<3>(out)) return 1;
  if (shape_sweep<0>(sms, clk_khz, out) || shape_sweep<1>(sms, clk_khz, out) || shape_sweep<2>(sms, clk_khz, out) ||
      shape_sweep<3>(sms, clk_khz, out))
    return 1;
  return 0;
}
