// ubench3.cu -- pipe probes for sm_90a (H100): FP64 (DFMA) vs wide integer multiply (IMAD.WIDE) issue rates, how
// they overlap with each other and with ALU work, and the DFMA-based 256-bit multiplier (kgx_field_fp64.cuh) against the
// integer one (kgx_field.cuh), alone and mixed.  Cycles are MEASURED (clock64 of one thread per CTA + globaltimer), not
// derived from a nominal clock.   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/ubench3 scripts/ubench3.cu
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>
#include "../kangaroo_b200/csrc/kgx_field.cuh"
#include "../kangaroo_b200/csrc/kgx_field_fp64.cuh"
using namespace kgx;

#define N 8
// V: 0 IMAD.WIDE x8 | 1 DFMA x8 | 2 IMAD.WIDE x8 + DFMA x8 | 3 IMAD.WIDE x8 + LOP3 x8 | 4 IMAD.WIDE x8 + LOP3 x16
//    5 DFMA x8 + LOP3 x8 | 6 DFMA x8 + LOP3 x16 | 7 LOP3 x16 | 8 IMAD.WIDE x8 + FFMA x8 | 9 FFMA x16 | 10 DFMA x8 + IADD3.X-style 64-bit adds x8
//    11 IMAD.WIDE x8 + DFMA x4 | 12 IMAD.WIDE x8 + DFMA x16 | 13 DADD x8 | 14 IMAD.WIDE x4 + DFMA x8 + LOP3 x8
template <int V> __global__ void probe(int iters, unsigned long long* cyc, u32* sink) {
  const u32 seed = blockIdx.x * blockDim.x + threadIdx.x + 1u;
  u64 acc[N]; u32 x[N], y[2 * N]; double d[2 * N], e[N]; float f[2 * N];
#pragma unroll
  for (int k = 0; k < N; k++) { acc[k] = seed * (k + 3u); x[k] = seed + k * 1315423911u; e[k] = 1.0 + 1e-9 * (seed + k); }
#pragma unroll
  for (int k = 0; k < 2 * N; k++) { y[k] = seed * (k + 1); d[k] = 1.0 + 1e-7 * k; f[k] = 1.0f + 1e-3f * k; }
  u32 m1 = seed * 7u + 5u; double dm = 1.0000001; float fm = 1.0001f;
  const long long t0 = clock64();
  for (int it = 0; it < iters; it++) {
    m1 = m1 * 0x9E3779B1u + 12345u;
    constexpr int NI = (V == 0 || V == 2 || V == 3 || V == 4 || V == 8 || V == 11 || V == 12) ? 8 : (V == 14 ? 4 : 0);
    constexpr int ND = (V == 1 || V == 2 || V == 5 || V == 6 || V == 10 || V == 14) ? 8 : (V == 11 ? 4 : (V == 12 ? 16 : 0));
    constexpr int NL = (V == 3 || V == 5 || V == 14) ? 8 : ((V == 4 || V == 6 || V == 7) ? 16 : 0);
    constexpr int NF = (V == 8) ? 8 : (V == 9 ? 16 : 0);
#pragma unroll
    for (int k = 0; k < 16; k++) {
      if (k < NI) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[k]) : "r"(x[k]), "r"(m1));
      if (k < ND) asm volatile("fma.rz.f64 %0, %1, %2, %0;" : "+d"(d[k]) : "d"(e[k & 7]), "d"(dm));
      if (k < NL) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(y[k]) : "r"(m1), "r"(x[k & 7]));
      if (k < NF) asm volatile("fma.rn.f32 %0, %1, %2, %0;" : "+f"(f[k]) : "f"(f[(k + 1) & 15]), "f"(fm));
      if (V == 10 && k < 8) asm volatile("add.cc.u32 %0, %0, %2;\n\taddc.u32 %1, %1, %3;" : "+r"(y[2 * k]), "+r"(y[2 * k + 1]) : "r"(m1), "r"(x[k]));
      if (V == 13 && k < 8) asm volatile("add.rz.f64 %0, %0, %1;" : "+d"(d[k]) : "d"(dm));
    }
  }
  const long long t1 = clock64();
  if (threadIdx.x == 0) cyc[blockIdx.x] = (unsigned long long)(t1 - t0);
  u64 s = 0; double ds = 0; float fs = 0;
#pragma unroll
  for (int k = 0; k < N; k++) s ^= acc[k];
#pragma unroll
  for (int k = 0; k < 2 * N; k++) { s ^= y[k]; ds += d[k]; fs += f[k]; }
  if (s == 0x1234567ull) sink[0] = (u32)s;
  if (ds == 1.5) sink[1] = 1u;
  if (fs == 2.5f) sink[2] = 2u;
}

__device__ __forceinline__ void fe_mul_fp64(u32* r, const u32* a, const u32* b) {
  double da[5], db[5]; u32 w[16];
  fe_to_d52(da, a); fe_to_d52(db, b);
  kgx_mul512_d52(w, da, db);
  kgx_fold(r, w);
}
__device__ __forceinline__ void fe_sqr_fp64(u32* r, const u32* a) {
  double da[5]; u32 w[16];
  fe_to_d52(da, a);
  kgx_sqr512_d52(w, da);
  kgx_fold(r, w);
}

// kind 0: fe_mul chains (integer) | 1: fe_mul_fp64 chains | 2: one integer chain + one fp64 chain per thread (independent data)
// 3: warp-specialised: even warps integer, odd warps fp64 | 4: fe_sqr int | 5: fe_sqr fp64 | 6: 2 int : 1 fp64 per thread
__global__ void __launch_bounds__(128) mulbench(int kind, int iters, unsigned long long* cyc, u32* sink) {
  const u32 seed = blockIdx.x * blockDim.x + threadIdx.x + 1u;
  u32 a[8], b[8], c[8], d[8];
#pragma unroll
  for (int w = 0; w < 8; w++) { a[w] = seed * (2654435761u + w); b[w] = seed * (40503u + 7u * w) + w; c[w] = a[w] ^ 0x55aa55aau; d[w] = b[w] + 77u * w; }
  const long long t0 = clock64();
  const bool odd = (threadIdx.x >> 5) & 1;
  if (kind == 0) for (int it = 0; it < iters; it++) { fe_mul(a, a, b); fe_mul(b, b, a); }
  else if (kind == 1) for (int it = 0; it < iters; it++) { fe_mul_fp64(a, a, b); fe_mul_fp64(b, b, a); }
  else if (kind == 2) for (int it = 0; it < iters; it++) { fe_mul(a, a, b); fe_mul_fp64(c, c, d); fe_mul(b, b, a); fe_mul_fp64(d, d, c); }
  else if (kind == 3) { if (odd) for (int it = 0; it < iters; it++) { fe_mul_fp64(a, a, b); fe_mul_fp64(b, b, a); } else for (int it = 0; it < iters; it++) { fe_mul(a, a, b); fe_mul(b, b, a); } }
  else if (kind == 4) for (int it = 0; it < iters; it++) { fe_sqr(a, a); fe_sqr(b, b); }
  else if (kind == 5) for (int it = 0; it < iters; it++) { fe_sqr_fp64(a, a); fe_sqr_fp64(b, b); }
  else if (kind == 6) for (int it = 0; it < iters; it++) { fe_mul(a, a, b); fe_mul(b, b, a); fe_mul_fp64(c, c, d); }
  const long long t1 = clock64();
  if (threadIdx.x == 0) cyc[blockIdx.x] = (unsigned long long)(t1 - t0);
  u32 s = 0;
#pragma unroll
  for (int w = 0; w < 8; w++) s ^= a[w] ^ b[w] ^ c[w] ^ d[w];
  if (s == 0x12345u) sink[0] = s;
}

__global__ void check_kernel(int n, int* bad) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  u32 a[8], b[8], r0[8], r1[8];
  u32 s = i * 2654435761u + 12345u;
#pragma unroll
  for (int w = 0; w < 8; w++) { s = s * 1664525u + 1013904223u; a[w] = s; s = s * 1664525u + 1013904223u; b[w] = s; }
  if ((i & 15) == 0) { for (int w = 0; w < 8; w++) a[w] = 0xFFFFFFFFu; }
  if ((i & 31) == 1) { for (int w = 0; w < 8; w++) b[w] = 0xFFFFFFFFu; }
  if ((i & 63) == 2) { for (int w = 1; w < 8; w++) a[w] = 0; }
  fe_mul(r0, a, b); fe_mul_fp64(r1, a, b);
  bool ok = true;
  for (int w = 0; w < 8; w++) ok &= (r0[w] == r1[w]);
  fe_sqr(r0, a); fe_sqr_fp64(r1, a);
  for (int w = 0; w < 8; w++) ok &= (r0[w] == r1[w]);
  if (!ok) atomicAdd(bad, 1);
}

static double run_cycles(unsigned long long* dcyc, int blocks) {
  unsigned long long* h = (unsigned long long*)malloc(blocks * 8);
  cudaMemcpy(h, dcyc, blocks * 8, cudaMemcpyDeviceToHost);
  double s = 0; for (int i = 0; i < blocks; i++) s += (double)h[i];
  free(h); return s / blocks;
}

template <int V> static void run_probe(const char* name, double ops_per_iter, int sms, int wps, unsigned long long* dcyc, u32* sink) {
  const int threads = 128, blocks = sms * (wps * 4 * 32 / threads), iters = 4000;
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  probe<V><<<blocks, threads>>>(iters / 8, dcyc, sink); cudaDeviceSynchronize();
  cudaEventRecord(a); probe<V><<<blocks, threads>>>(iters, dcyc, sink); cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b);
  const double cyc = run_cycles(dcyc, blocks);
  const double lane_ops = ops_per_iter * iters * (double)blocks * threads;
  // per SM per clock, from the measured per-CTA cycle count (all CTAs resident at once: blocks = sms * CTAs/SM)
  printf("%-46s wps=%2d  %8.3f ms  %9.0f cyc  eff.clk %.0f MHz  %7.2f counted-ops/clk/SM\n", name, wps, ms, cyc, cyc / (ms * 1e3),
         lane_ops / sms / cyc);
}

int main() {
  cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
  const int sms = prop.multiProcessorCount;
  printf("%s, %d SMs\n", prop.name, sms);
  unsigned long long* dcyc; cudaMalloc(&dcyc, 8 * 65536); u32* sink; cudaMalloc(&sink, 64);
  for (int wps = 4; wps <= 8; wps += 4) {
    run_probe<0>("V0  IMAD.WIDE x8 (count IMAD.WIDE)", 8, sms, wps, dcyc, sink);
    run_probe<1>("V1  DFMA x8 (count DFMA)", 8, sms, wps, dcyc, sink);
    run_probe<13>("V13 DADD x8 (count DADD)", 8, sms, wps, dcyc, sink);
    run_probe<2>("V2  IMAD.WIDE x8 + DFMA x8 (count 8)", 8, sms, wps, dcyc, sink);
    run_probe<11>("V11 IMAD.WIDE x8 + DFMA x4 (count 8)", 8, sms, wps, dcyc, sink);
    run_probe<12>("V12 IMAD.WIDE x8 + DFMA x16 (count 8)", 8, sms, wps, dcyc, sink);
    run_probe<3>("V3  IMAD.WIDE x8 + LOP3 x8 (count 8)", 8, sms, wps, dcyc, sink);
    run_probe<4>("V4  IMAD.WIDE x8 + LOP3 x16 (count 8)", 8, sms, wps, dcyc, sink);
    run_probe<5>("V5  DFMA x8 + LOP3 x8 (count 8)", 8, sms, wps, dcyc, sink);
    run_probe<6>("V6  DFMA x8 + LOP3 x16 (count 8)", 8, sms, wps, dcyc, sink);
    run_probe<7>("V7  LOP3 x16 (count 16)", 16, sms, wps, dcyc, sink);
    run_probe<8>("V8  IMAD.WIDE x8 + FFMA x8 (count 8)", 8, sms, wps, dcyc, sink);
    run_probe<9>("V9  FFMA x16 (count 16)", 16, sms, wps, dcyc, sink);
    run_probe<10>("V10 DFMA x8 + 64-bit int add x8 (count 8)", 8, sms, wps, dcyc, sink);
    run_probe<14>("V14 IMAD.WIDE x4 + DFMA x8 + LOP3 x8 (count 8)", 8, sms, wps, dcyc, sink);
  }
  // correctness of the FP64 multiplier against the integer one on the device
  int* dbad; cudaMalloc(&dbad, 4); cudaMemset(dbad, 0, 4);
  check_kernel<<<4096, 256>>>(4096 * 256, dbad);
  int bad = -1; cudaMemcpy(&bad, dbad, 4, cudaMemcpyDeviceToHost);
  printf("fe_mul_fp64 / fe_sqr_fp64 vs integer fe_mul / fe_sqr on %d operands: %d mismatches  (%s)\n", 4096 * 256, bad, cudaGetErrorString(cudaGetLastError()));
  const char* names[] = {"fe_mul int x2", "fe_mul fp64 x2", "1 int + 1 fp64 per thread (x2)", "warp-specialised int | fp64", "fe_sqr int x2", "fe_sqr fp64 x2", "2 int + 1 fp64 per thread"};
  const double per_iter[] = {2, 2, 4, 2, 2, 2, 3};
  for (int ctas = 2; ctas <= 4; ctas++) {
    for (int kind = 0; kind < 7; kind++) {
      const int blocks = sms * ctas, threads = 128, iters = 2000;
      cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
      mulbench<<<blocks, threads>>>(kind, iters / 8, dcyc, sink); cudaDeviceSynchronize();
      cudaEventRecord(a); mulbench<<<blocks, threads>>>(kind, iters, dcyc, sink); cudaEventRecord(b); cudaEventSynchronize(b);
      float ms; cudaEventElapsedTime(&ms, a, b);
      const double cyc = run_cycles(dcyc, blocks);
      const double ops = per_iter[kind] * iters * (double)blocks * threads;
      printf("mul %-34s %d CTA/SM x128: %8.3f ms  %.3e mult/s  %7.1f cyc/mult/warp/SMSP (cyc %.0f)\n", names[kind], ctas, ms, ops / (ms * 1e-3),
             cyc / (per_iter[kind] * iters) / (ctas * 4 / 4.0) , cyc);
    }
  }
  printf("done: %s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
