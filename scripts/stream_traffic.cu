// stream_traffic.cu -- HBM traffic twin of the stream kernel (kangaroo_b200/csrc/kgx_kernel.cuh, stream_kernel): the same
// grid (2 CTAs of 128 threads per SM, one tile each), the same [tile][g][chunk][T] state planes and [tile][g][2][T] prefix
// planes, the same alternating-direction sweep over the G kangaroos of a thread, the same register ping-pong and the same
// two-instruction L2 prefetch of the pair pfDist kangaroos ahead -- with the field arithmetic replaced by XORs.  Every
// loaded word feeds a store, so no load is dead.  The time it takes is what the memory system alone needs to move one
// launch's planes, i.e. the GJump/s ceiling HBM puts on the real kernel.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scripts/stream_traffic scripts/stream_traffic.cu
//   scripts/stream_traffic [G=128] [passes=64] [pfDist=2] [reps=7]
//
// Plane sets, in designed bytes per jump:
//   224   : read prefix/x/y/d, write x'/y'/d'/prefix'
//   194.5 : read prefix/x/y, write x'/y'/prefix' and one jump-log byte; at the end of the launch every kangaroo's 64 log
//           bytes are folded into its distance (d read + write)
//   162.5 : the 194.5 set with one prefix product per pair of kangaroos instead of one per kangaroo
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <algorithm>
#include <vector>
#include <cuda_runtime.h>

typedef unsigned int u32;
constexpr int T = 128, CHUNKS = 5, LOG_RUNS = 64;
constexpr int SMEM_PAD = 100 * 1024;   // dynamic shared memory that pins the twin to 2 CTAs per SM, like the real kernel's registers

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #call, cudaGetErrorString(e_)); exit(1); } } while (0)

template <int SET> struct Set {
  static constexpr int NS = SET == 0 ? 5 : 4;              // state planes a jump reads and writes
  static constexpr bool PAIR = SET == 2;                   // one prefix per pair
  static constexpr bool LOG = SET != 0;                    // jump-log byte + end-of-launch fold
  static constexpr int NPL = 2 * NS + (PAIR ? 2 : 4);      // 128-byte-line planes of a pair: 14, 12, 10
};

struct Ld { uint4 c[CHUNKS + 2]; };

template <int SET>
__device__ __forceinline__ void load(Ld& k, const uint4* sg, const uint4* pg, bool withPre) {
#pragma unroll
  for (int c = 0; c < Set<SET>::NS; c++) k.c[c] = sg[c * T];
  if (withPre) { k.c[CHUNKS] = pg[0]; k.c[CHUNKS + 1] = pg[T]; }
}

template <int SET>
__device__ __forceinline__ void body(const Ld& k, uint4* sg, uint4* pg, uint8_t* lg, bool withPre, u32& acc) {
  u32 a = acc;
#pragma unroll
  for (int c = 0; c < Set<SET>::NS; c++) a ^= k.c[c].x ^ k.c[c].y ^ k.c[c].z ^ k.c[c].w;
  if (withPre) a ^= k.c[CHUNKS].x ^ k.c[CHUNKS + 1].w;
#pragma unroll
  for (int c = 0; c < Set<SET>::NS; c++) sg[c * T] = make_uint4(k.c[c].x ^ a, k.c[c].y, k.c[c].z, k.c[c].w + a);
  if (withPre) { pg[0] = make_uint4(k.c[CHUNKS].x + a, k.c[CHUNKS].y, k.c[CHUNKS].z, k.c[CHUNKS].w); pg[T] = k.c[CHUNKS + 1]; }
  if (Set<SET>::LOG) lg[0] = (uint8_t)(a & 63u);
  acc = a * 0x9E3779B1u + 1u;
}

template <int SET>
__global__ void __launch_bounds__(T, 2) twin(uint4* state, uint4* pre, uint8_t* jlog, int G, int passes, int pfDist) {
  using S = Set<SET>;
  const int t = threadIdx.x, lane = t & 31;
  const size_t tile = blockIdx.x;
  uint4* st = state + tile * ((size_t)G * CHUNKS * T) + t;
  const int npre = S::PAIR ? G / 2 : G;                                   // prefix slots per thread
  uint4* pr = pre + tile * ((size_t)npre * 2 * T) + t;
  uint8_t* lt = jlog + tile * ((size_t)LOG_RUNS * G * T) + t;
  const size_t runStride = (size_t)G * T;
  u32 acc = t;
  int backward = 1, logged = 0;
  for (int pass = 0; pass < passes; pass++) {
    const int g0 = backward ? G - 1 : 0;
    const ptrdiff_t ds = backward ? -(ptrdiff_t)(CHUNKS * T) : (ptrdiff_t)(CHUNKS * T);
    const ptrdiff_t dk = backward ? -(ptrdiff_t)T : (ptrdiff_t)T;
    // prefix pointer step per kangaroo (per pair in the pair set, where only the first member of a pair touches it)
    const ptrdiff_t dp = backward ? -(ptrdiff_t)(2 * T) : (ptrdiff_t)(2 * T);
    uint4* sg = st + (size_t)g0 * (CHUNKS * T);
    uint4* pg = pr + (size_t)(S::PAIR ? g0 / 2 : g0) * (2 * T);
    uint8_t* lg = lt + (size_t)logged * runStride + (size_t)g0 * T;
    // L2 prefetch: lane -> (plane, line) of the pair pfDist kangaroos ahead; plane k of a pair: the first member's state planes,
    // the second's, then the prefix planes.  Two instructions (planes lane/4 and 8 + lane/4).
    const ptrdiff_t lineOff = (ptrdiff_t)((lane & 3) * 8) - lane;
    const uint4* q[2];
    ptrdiff_t qs[2];
    bool qon[2];
    for (int h = 0; h < 2; h++) {
      const int k = 8 * h + (lane >> 2);
      qon[h] = k < S::NPL;
      if (k < 2 * S::NS) {
        const int m = k / S::NS;
        q[h] = sg + (ptrdiff_t)(pfDist + m) * ds + (k % S::NS) * T + lineOff;
        qs[h] = 2 * ds;
      } else {
        const int r = k - 2 * S::NS;
        q[h] = S::PAIR ? pg + (ptrdiff_t)(pfDist / 2) * dp + (r & 1) * T + lineOff
                       : pg + (ptrdiff_t)(pfDist + r / 2) * dp + (r & 1) * T + lineOff;
        qs[h] = S::PAIR ? dp : 2 * dp;
      }
    }
    Ld A, B;
    load<SET>(A, sg, pg, true);
#pragma unroll 1
    for (int i = 0; i < G; i += 2) {
      if (pfDist > 0 && i + pfDist + 1 < G) {
        if (qon[0]) asm volatile("prefetch.global.L2 [%0];" ::"l"(q[0]));
        if (qon[1]) asm volatile("prefetch.global.L2 [%0];" ::"l"(q[1]));
      }
      q[0] += qs[0]; q[1] += qs[1];
      uint4* pgB = S::PAIR ? pg : pg + dp;
      load<SET>(B, sg + ds, pgB, !S::PAIR);
      body<SET>(A, sg, pg, lg, true, acc);
      uint4* pgN = S::PAIR ? pg + dp : pg + 2 * dp;
      if (i + 2 < G) load<SET>(A, sg + 2 * ds, pgN, true);
      body<SET>(B, sg + ds, pgB, lg + dk, !S::PAIR, acc);
      sg += 2 * ds; pg = pgN; lg += 2 * dk;
    }
    backward ^= 1;
    if (S::LOG && (++logged == LOG_RUNS || pass == passes - 1)) {      // fold: d chunk read + write, 64 log bytes read
#pragma unroll 1
      for (int g = 0; g < G; g++) {
        const uint8_t* l = lt + (size_t)g * T;
        u32 b[LOG_RUNS];
#pragma unroll
        for (int r = 0; r < LOG_RUNS; r++) b[r] = l[(size_t)r * runStride];
        uint4* dptr = st + (size_t)(g * CHUNKS + 4) * T;
        uint4 d = *dptr;
#pragma unroll
        for (int r = 0; r < LOG_RUNS; r++) if (r < logged) { d.x += b[r]; d.y ^= d.x; }
        *dptr = d;
      }
      logged = 0;
    }
  }
  if (acc == 0x12345678u) state[0].x = acc;
}

template <int SET>
static void run(const char* name, double bytesPerJump, uint4* state, uint4* pre, uint8_t* jlog, int tiles, int G, int passes, int pfDist, int reps) {
  CK(cudaFuncSetAttribute(twin<SET>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_PAD));
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  std::vector<float> ms;
  for (int it = 0; it < reps + 2; it++) {                     // 2 warm-up launches
    CK(cudaEventRecord(a));
    twin<SET><<<tiles, T, SMEM_PAD>>>(state, pre, jlog, G, passes, pfDist);
    CK(cudaEventRecord(b));
    CK(cudaEventSynchronize(b));
    CK(cudaGetLastError());
    float m; CK(cudaEventElapsedTime(&m, a, b));
    if (it >= 2) ms.push_back(m);
  }
  std::sort(ms.begin(), ms.end());
  const double jumps = (double)tiles * T * G * passes;
  const double med = ms[ms.size() / 2], best = ms[0];
  printf("{\"set\": \"%s\", \"bytes_per_jump\": %.1f, \"ms_median\": %.3f, \"ms_min\": %.3f, \"ms_max\": %.3f, "
         "\"tb_s_median\": %.3f, \"gjump_s_ceiling_median\": %.2f, \"gjump_s_ceiling_best\": %.2f}\n",
         name, bytesPerJump, med, best, ms.back(), bytesPerJump * jumps / (med * 1e-3) / 1e12, jumps / (med * 1e-3) / 1e9,
         jumps / (best * 1e-3) / 1e9);
  CK(cudaEventDestroy(a)); CK(cudaEventDestroy(b));
}

int main(int argc, char** argv) {
  const int G = argc > 1 ? atoi(argv[1]) : 128, passes = argc > 2 ? atoi(argv[2]) : 64;
  const int pfDist = argc > 3 ? atoi(argv[3]) : 2, reps = argc > 4 ? atoi(argv[4]) : 7;
  if (G < 2 || (G & 1) || passes < 1 || pfDist < 0 || reps < 1) { fprintf(stderr, "bad arguments\n"); return 2; }
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  const int tiles = 2 * prop.multiProcessorCount;                       // the default herd: one tile per CTA, 2 CTAs per SM
  const size_t n = (size_t)tiles * T * G;
  uint4 *state, *pre; uint8_t* jlog;
  CK(cudaMalloc(&state, n * CHUNKS * 16));
  CK(cudaMalloc(&pre, n * 32));
  CK(cudaMalloc(&jlog, n * LOG_RUNS));
  CK(cudaMemset(state, 1, n * CHUNKS * 16)); CK(cudaMemset(pre, 2, n * 32)); CK(cudaMemset(jlog, 0, n * LOG_RUNS));
  printf("{\"device\": \"%s\", \"sms\": %d, \"kangaroos\": %zu, \"G\": %d, \"passes\": %d, \"pf\": %d, \"l2_mb\": %.0f, "
         "\"footprint_mb\": %.0f}\n", prop.name, prop.multiProcessorCount, n, G, passes, pfDist, prop.l2CacheSize / 1048576.0,
         n * (CHUNKS * 16 + 32 + LOG_RUNS) / 1e6);
  {   // what the card sustains on a plain device-to-device copy of the state (read + write), for scale
    cudaEvent_t a, b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
    const size_t half = n * CHUNKS * 8;
    float best = 1e30f;
    for (int it = 0; it < reps + 1; it++) {
      CK(cudaEventRecord(a));
      CK(cudaMemcpyAsync((char*)state + half, state, half, cudaMemcpyDeviceToDevice));
      CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b));
      float m; CK(cudaEventElapsedTime(&m, a, b));
      if (it > 0) best = std::min(best, m);
    }
    printf("{\"set\": \"d2d memcpy\", \"tb_s_best\": %.3f}\n", 2.0 * half / (best * 1e-3) / 1e12);
    CK(cudaEventDestroy(a)); CK(cudaEventDestroy(b));
  }
  run<0>("224", 224.0, state, pre, jlog, tiles, G, passes, pfDist, reps);
  run<1>("194.5", 194.5, state, pre, jlog, tiles, G, passes, pfDist, reps);
  run<2>("162.5", 162.5, state, pre, jlog, tiles, G, passes, pfDist, reps);
  CK(cudaFree(state)); CK(cudaFree(pre)); CK(cudaFree(jlog));
  return 0;
}
