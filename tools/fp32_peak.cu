// fp32_peak.cu -- micro-benchmark of the CUDA-core fp32 pipe on the box the bench runs on (SURVEY.md 8d: "measure both with a
// micro-benchmark before quoting fractions").  Independent FMA chains per thread, no memory traffic:
//   ffma3   d = fma(a, b, d) with three register operands (what K8's inner loop issues)
//   ffma2   fma.rn.f32x2 (packed pair, FFMA2)
//   fadd    d = d + a
//   mix     K8's per-test mix: 9 FFMA + 5 FADD + 3 SHF + 1 FMNMX
// Prints lane-operations per second (one FMA = one lane-operation) and per clock per SM.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 tools/fp32_peak.cu -o fp32_peak && ./fp32_peak
#include <cstdio>
#include <cuda_runtime.h>

template <int MODE>
__global__ void __launch_bounds__(256) k(float* out, int iters, float a0, float b0) {
  float d[8], a = a0 + threadIdx.x * 1e-9f, b = b0;
  unsigned long long p[4];
  unsigned w = threadIdx.x;
#pragma unroll
  for (int i = 0; i < 8; ++i) d[i] = (float)i;
#pragma unroll
  for (int i = 0; i < 4; ++i) asm("mov.b64 %0, {%1, %2};" : "=l"(p[i]) : "f"(d[2 * i]), "f"(d[2 * i + 1]));
  unsigned long long pa, pb;
  asm("mov.b64 %0, {%1, %2};" : "=l"(pa) : "f"(a), "f"(a));
  asm("mov.b64 %0, {%1, %2};" : "=l"(pb) : "f"(b), "f"(b));
  for (int it = 0; it < iters; ++it) {
    if (MODE == 0) {
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int i = 0; i < 8; ++i) d[i] = __fmaf_rn(a, d[i], b);
    } else if (MODE == 1) {
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int i = 0; i < 4; ++i) asm volatile("fma.rn.f32x2 %0, %1, %0, %2;" : "+l"(p[i]) : "l"(pa), "l"(pb));
    } else if (MODE == 2) {
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int i = 0; i < 8; ++i) d[i] = __fadd_rn(d[i], a);
    } else {
#pragma unroll
      for (int i = 0; i < 8; i += 2) {  // 4 "tests": 9 FFMA + 5 FADD + 3 SHF + 1 FMNMX each
        float x = d[i], y = d[i + 1];
        x = __fmaf_rn(a, x, b); x = __fmaf_rn(b, x, a); x = __fmaf_rn(a, x, y); y = __fmaf_rn(a, y, b); y = __fmaf_rn(b, y, a);
        y = __fmaf_rn(a, y, x); float u = __fadd_rn(x, a), v = __fadd_rn(y, b);
        float D = __fadd_rn(u, -v), s = __fadd_rn(u, v);
        float g = __fmaf_rn(a, s, b), t = __fmaf_rn(D, D, g), q = __fmaf_rn(D, a, b);
        float ww = __fadd_rn(t, -q);
        w = __funnelshift_l(__float_as_uint(t), w, 1); w = __funnelshift_l(__float_as_uint(s), w, 1); w = __funnelshift_l(__float_as_uint(ww), w, 1);
        d[i] = fminf(x, s); d[i + 1] = ww;
      }
    }
  }
  float acc = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) acc += d[i];
#pragma unroll
  for (int i = 0; i < 4; ++i) { float lo, hi; asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(p[i])); acc += lo + hi; }
  if (acc == 123.456f || w == 0x12345u) out[threadIdx.x] = acc;
}

template <int MODE>
double run(const char* name, double lane_ops_per_iter, int sms, double clk_ghz) {
  float* out;
  cudaMalloc(&out, 4096);
  const int iters = 20000, blocks = sms * 8;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  k<MODE><<<blocks, 256>>>(out, 100, 1.0001f, 0.5f);
  cudaDeviceSynchronize();
  cudaEventRecord(e0);
  k<MODE><<<blocks, 256>>>(out, iters, 1.0001f, 0.5f);
  cudaEventRecord(e1);
  cudaDeviceSynchronize();
  float ms = 0;
  cudaEventElapsedTime(&ms, e0, e1);
  const double ops = lane_ops_per_iter * iters * (double)blocks * 256;
  const double rate = ops / (ms * 1e-3);
  printf("{\"mode\": \"%s\", \"lane_ops_per_s\": %.4e, \"lane_ops_per_clk_per_sm\": %.1f, \"ms\": %.3f}\n", name, rate, rate / (sms * clk_ghz * 1e9), ms);
  cudaFree(out);
  return rate;
}

int main() {
  cudaDeviceProp pr;
  cudaGetDeviceProperties(&pr, 0);
  int clk_khz = 0;
  cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
  const double ghz = clk_khz * 1e-6;
  printf("{\"device\": \"%s\", \"sms\": %d, \"clock_ghz\": %.3f}\n", pr.name, pr.multiProcessorCount, ghz);
  run<0>("ffma 3-register (1 lane-op each)", 32, pr.multiProcessorCount, ghz);
  run<1>("ffma2 packed (2 lane-ops each)", 32, pr.multiProcessorCount, ghz);
  run<2>("fadd", 32, pr.multiProcessorCount, ghz);
  run<3>("K8 mix: 14 fp32-pipe ops of 18 instructions per test (fp32-pipe lane-ops counted)", 4 * 14, pr.multiProcessorCount, ghz);
  return 0;
}
