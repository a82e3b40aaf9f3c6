// kgx_engine.cu -- host side of the H100 jump engine behind the C ABI of include/kgx.h.
//
// Replaces the host half of the reference's GPU/GPUEngine.cu (ctor/dtor :144-263, SetKangaroos/GetKangaroos/
// SetKangaroo :381-538, callKernel :540-557, SetParams :559-590, Launch :607-679) with a stream-ordered
// design: one non-blocking stream per engine, device-side pack/unpack kernels instead of per-block host
// transposes, double-buffered DP slabs so the readback of launch i overlaps launch i+1, CUDA-event timing of
// every launch.  No CPU fallback exists: every entry point fails when CUDA does.
#include <cuda_runtime.h>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <unistd.h>
#include "../../include/kgx.h"
#include "kgx_kernel.cuh"
#include "kgx_herd.cuh"
#include "kgx_ckpt.cuh"
#include "kgx_testhooks.cuh"

using namespace kgx;

static char g_create_err[256] = "";

// Every compiled jump-kernel instantiation.  Resident tile kernels: T, K = the tile geometry (KGX_CFG="T,K"); the first entry
// is the default, the largest tile of 128 threads that still fits two CTAs per SM.  Stream kernels: ctasPerSM (KGX_STREAM_CTAS)
// and warpInv (KGX_STREAM_INV) select them, K is the group size chosen at engine creation.  sym: the symmetric-mode
// (USE_SYMMETRY) instantiation, compiled for the default geometry and the 2-CTA warp-inverse stream kernel only.
struct KernelEntry {
  int kind, T, K, ctasPerSM;
  bool warpInv, sym;
  void (*fn)(LaunchParams);
  int smem, ctasPerTile;     // dynamic shared memory; CTAs sharing one tile (the cluster kernel's 2)
};
#define KGX_RESIDENT(T_, K_, SYM_) { KGX_KERNEL_RESIDENT, T_, K_, Cfg<T_, K_>::CTAS_PER_SM, false, SYM_, jump_kernel<T_, K_, SYM_>, Cfg<T_, K_>::SMEM_BYTES, 1 }
#define KGX_STREAM(CTAS_, WARPINV_, SYM_) { KGX_KERNEL_STREAM, 128, 0, CTAS_, WARPINV_, SYM_, stream_kernel<128, CTAS_, WARPINV_, SYM_>, 0, 1 }
static const KernelEntry g_kernels[] = {
  KGX_RESIDENT(128, 7, false), KGX_RESIDENT(128, 7, true), KGX_RESIDENT(128, 4, false), KGX_RESIDENT(128, 5, false),
  KGX_RESIDENT(64, 7, false), KGX_RESIDENT(64, 5, false), KGX_RESIDENT(64, 6, false), KGX_RESIDENT(64, 4, false),
  KGX_RESIDENT(96, 6, false), KGX_RESIDENT(256, 3, false), KGX_RESIDENT(32, 8, false), KGX_RESIDENT(32, 12, false),
  KGX_STREAM(2, true, false), KGX_STREAM(2, false, false), KGX_STREAM(3, true, false), KGX_STREAM(3, false, false),
  KGX_STREAM(2, true, true),
  { KGX_KERNEL_TMEM, CfgCl::T, CfgCl::K * CfgCl::CLUSTER, 2, false, false, jump_kernel_cluster, CfgCl::SMEM_BYTES, CfgCl::CLUSTER },
};

// The instantiation of kernel kind `kind` for tile geometry T,K (resident), or ctas and warpInv (stream), in symmetric mode
// or not; NULL when none is compiled.  The symmetric stream kernel always takes the warp inverse, whatever warpInv says.
static const KernelEntry* find_kernel(int kind, int T, int K, int ctas, bool warpInv, bool sym) {
  for (const KernelEntry& k : g_kernels) {
    if (k.kind != kind || k.sym != sym) continue;
    if (kind == KGX_KERNEL_RESIDENT && (k.T != T || k.K != K)) continue;
    if (kind == KGX_KERNEL_STREAM && (k.ctasPerSM != ctas || (!sym && k.warpInv != warpInv))) continue;
    return &k;
  }
  return nullptr;
}

struct kgx_engine {
  int dev = 0, groups = 0, tpg = 0, sms = 0;
  int T = 0, K = 0;          // state layout: tiles of T x K kangaroos (the stream kernel's K is its group size)
  int kind = 0;              // KGX_KERNEL_STREAM / _RESIDENT / _TMEM
  const KernelEntry* kern = nullptr;   // the instantiation kgx_launch_async launches
  u64 n = 0, nPadded = 0;
  u32 numTiles = 0, maxFound = 0;
  int nRun = KGX_NB_RUN;
  uint4* state = nullptr;
  uint4* pre = nullptr;      // streaming mode: prefix-product scratch
  uint8_t* jlog = nullptr;   // streaming mode: jump-index log, LOG_RUNS bytes per kangaroo (kgx_kernel.cuh stream_fold)
  int streamCtas = 2;
  bool symmetry = false;     // USE_SYMMETRY engine mode (kgx_set_symmetry): class switch + cycle rule, signed distances
  int symRule = 0;           // KGX_SYM_LASTJUMP / KGX_SYM_CLASS
  int pfDist = 2;            // KGX_STREAM_PF: L2 prefetch distance of the stream kernel in kangaroos (0 = off).  H100 SXM at
                             // 700 W, default herd, kernel time (scripts/sweep2.py, one run each): 0 -> 11.54, 1 -> 12.33,
                             // 2 -> 12.88, 3 -> 12.42, 4 -> 11.65 GJump/s; 3 CTAs/SM at distance 2: 12.39
  uint8_t* aux = nullptr;    // symmetric mode: lastJump per slot
  bool warpInv = true;       // stream kernel: one warp-wide shuffle-butterfly inverse per pass (false: one per thread)
  u32* slab[2] = {nullptr, nullptr};   // DP slabs [count][maxFound*14]
  u32* slabPinned = nullptr;
  u32* dp40 = nullptr;       // [count][maxFound x 10 words]: converted records of the last completed launch
  u32* jtab = nullptr;
  u32* herdTab = nullptr;    // 256 x 16 words: 2^i * G (built on first kgx_create_herd)
  uint4 *stgX = nullptr, *stgY = nullptr, *stgD = nullptr;   // device staging (AoS, kIdx order)
  u64 dpMask = 0;
  bool haveParams = false, inflight = false;
  int cur = 0;                 // slab the in-flight (or last) launch writes
  int done = -1;               // slab of the most recently completed launch
  cudaStream_t stream = nullptr, copyStream = nullptr;
  cudaEvent_t evStart[2] = {nullptr, nullptr}, evStop[2] = {nullptr, nullptr};
  cudaEvent_t evSnap = nullptr;   // snapshot (checkpoint) staging complete
  bool snapPending = false;
  u64* herdRecs = nullptr;        // n x 96-byte work-file records (kgx_snapshot_export / kgx_import); kept, like the staging, for the next save
  bool snapConverted = false;     // herdRecs holds the pending snapshot
  // multi-key herd (kgx_create_herd_multi / kgx_retarget): none of it is jump-kernel state
  u32* keys = nullptr;            // key table: keyCap x 16 words (x, y); the first nKeys hold the herd's keys
  uint16_t* targets = nullptr;    // n: key of every wild kangaroo, kIdx order
  u32* rtDelta = nullptr;         // keyCap x 16 words: keys[to[j]] - keys[from] of the retarget in stream order
  u32* rtTo = nullptr;            // keyCap: to[j] | infinity flag
  u32 nKeys = 0, keyCap = 0;      // nKeys == 0: no key table (a herd of kgx_create_herd or kgx_upload)
  uint16_t* snapTargets = nullptr; // n: the targets of the pending snapshot (kgx_snapshot_begin on a herd with a key table)
  bool snapHasTargets = false;
  int firstType = 0;
  float lastMs = 0.f;
  unsigned long long* prof = nullptr;   // KGX_PROF=1: phase cycle counters
  u64 launches = 0;
  size_t slabBytes = 0, stateBytes = 0;
  char err[256] = "";
};

#define CK(e, call)                                                                            \
  do {                                                                                         \
    cudaError_t _s = (call);                                                                   \
    if (_s != cudaSuccess) {                                                                   \
      snprintf((e)->err, sizeof((e)->err), "%s: %s", #call, cudaGetErrorString(_s));           \
      return -1;                                                                               \
    }                                                                                          \
  } while (0)

// state byte of a fresh kangaroo in symmetric mode: lastJump = NB_JUMP (none yet) / symClass = 0
static int aux_init(const kgx_engine* e) { return e->symRule == KGX_SYM_CLASS ? 0 : 32; }
#ifndef KGX_DEFAULT_STREAM
#define KGX_DEFAULT_STREAM 1   // streaming kernel for large herds; KGX_MODE=resident selects the tile kernel
#endif

extern "C" {

int kgx_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int kgx_grid_default(int dev, int* x, int* y) {
  if (*x > 0 && *y > 0) return 0;
  int n = kgx_device_count();
  if (n == 0 || dev >= n) return -1;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return -1;
  if (*x <= 0) *x = 2 * prop.multiProcessorCount;   // GPUEngine.cu:301
  if (*y <= 0) *y = 128;                            // GPUEngine.cu:303 (sm_90 is not in the reference's core table)
  return 0;
}

int kgx_device_info(int dev, char* buf, int buflen) {
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return -1;
  snprintf(buf, buflen, "%s|%d|%d|%d|%.1f", prop.name, prop.multiProcessorCount, prop.major, prop.minor,
           (double)prop.totalGlobalMem / 1048576.0);
  return 0;
}

const char* kgx_last_error(kgx_engine* e) { return e ? e->err : g_create_err; }

void kgx_destroy(kgx_engine* e) {
  if (!e) return;
  cudaSetDevice(e->dev);
  if (e->stream) cudaStreamSynchronize(e->stream);
  cudaFree(e->dp40); cudaFree(e->herdTab); cudaFree(e->state); cudaFree(e->pre); cudaFree(e->jlog); cudaFree(e->slab[0]); cudaFree(e->slab[1]); cudaFree(e->jtab);
  cudaFree(e->stgX); cudaFree(e->stgY); cudaFree(e->stgD); cudaFree(e->aux); cudaFree(e->herdRecs);
  cudaFree(e->keys); cudaFree(e->targets); cudaFree(e->rtDelta); cudaFree(e->rtTo); cudaFree(e->snapTargets);
  if (e->slabPinned) cudaFreeHost(e->slabPinned);
  for (int i = 0; i < 2; i++) { if (e->evStart[i]) cudaEventDestroy(e->evStart[i]); if (e->evStop[i]) cudaEventDestroy(e->evStop[i]); }
  if (e->evSnap) cudaEventDestroy(e->evSnap);
  if (e->stream) cudaStreamDestroy(e->stream);
  if (e->copyStream) cudaStreamDestroy(e->copyStream);
  delete e;
}

kgx_engine* kgx_create(int dev, int groups, int threads_per_group, uint32_t max_found) {
  return kgx_create_ex(dev, groups, threads_per_group, max_found, KGX_KERNEL_AUTO, 0);
}

// kernel: KGX_KERNEL_AUTO / _STREAM / _RESIDENT; stream_g: kangaroos per thread of the stream kernel (0 = adaptive).
// The environment (KGX_MODE, KGX_STREAM_G, KGX_CFG) only fills in what the arguments leave on "auto".
kgx_engine* kgx_create_ex(int dev, int groups, int threads_per_group, uint32_t max_found, int kernel, int stream_g) {
  kgx_engine* e = new kgx_engine();
  auto fail = [&](const char* what, cudaError_t s) -> kgx_engine* {
    snprintf(g_create_err, sizeof g_create_err, "kgx_create: %s: %s", what, cudaGetErrorString(s));
    cudaGetLastError();   // do not leave a sticky error behind for the next engine of this process
    kgx_destroy(e);
    return nullptr;
  };
  if (groups <= 0 || threads_per_group <= 0 || max_found == 0) {
    snprintf(g_create_err, sizeof g_create_err, "kgx_create: bad arguments");
    delete e; return nullptr;
  }
  int cnt = 0;
  cudaError_t s = cudaGetDeviceCount(&cnt);
  if (s != cudaSuccess || cnt == 0) {
    snprintf(g_create_err, sizeof g_create_err, "kgx_create: no CUDA device (%s)", cudaGetErrorString(s));
    cudaGetLastError(); delete e; return nullptr;
  }
  if ((s = cudaSetDevice(dev)) != cudaSuccess) return fail("cudaSetDevice", s);
  cudaDeviceProp prop;
  if ((s = cudaGetDeviceProperties(&prop, dev)) != cudaSuccess) return fail("cudaGetDeviceProperties", s);
  e->dev = dev; e->groups = groups; e->tpg = threads_per_group; e->sms = prop.multiProcessorCount;
  e->n = (u64)groups * (u64)threads_per_group * KGX_GPU_GRP_SIZE;
  e->T = g_kernels[0].T; e->K = g_kernels[0].K;
  if (const char* env = getenv("KGX_CFG")) {
    int t = 0, k = 0;
    if (sscanf(env, "%d,%d", &t, &k) != 2 || !find_kernel(KGX_KERNEL_RESIDENT, t, k, 0, false, false)) {
      snprintf(g_create_err, sizeof g_create_err, "kgx_create: KGX_CFG=%s is not a compiled tile geometry", env); delete e; return nullptr;
    }
    e->T = t; e->K = k;
  }
  {
    const char* mode = getenv("KGX_MODE");
    if (kernel == KGX_KERNEL_STREAM) mode = "stream";
    else if (kernel == KGX_KERNEL_RESIDENT) mode = "resident";
    else if (kernel == KGX_KERNEL_TMEM) mode = "tmem";
    else if (kernel != KGX_KERNEL_AUTO) { snprintf(g_create_err, sizeof g_create_err, "kgx_create_ex: bad kernel selector %d", kernel); delete e; return nullptr; }
    // default: the streaming kernel for herds of 400 k kangaroos and more (it wants many kangaroos per thread on every
    // SM to amortise the per-thread inverse), the shared-memory tile kernel below that (its inverse is shared by a whole
    // tile, so it keeps its rate on herds too small to give every stream thread a long group)
    if (!mode) e->kind = KGX_DEFAULT_STREAM != 0 && e->n >= 400000ull ? KGX_KERNEL_STREAM : KGX_KERNEL_RESIDENT;
    else if (!strcmp(mode, "stream")) e->kind = KGX_KERNEL_STREAM;
    else if (!strcmp(mode, "resident")) e->kind = KGX_KERNEL_RESIDENT;
    else if (!strcmp(mode, "tmem")) e->kind = KGX_KERNEL_TMEM;
    else { snprintf(g_create_err, sizeof g_create_err, "kgx_create: KGX_MODE must be stream, resident or tmem"); delete e; return nullptr; }
    if (e->kind == KGX_KERNEL_STREAM) {
      // kangaroos per thread: 128 (the reference's GPU_GRP_SIZE) when the herd fills two CTAs per SM with it; smaller
      // herds get a smaller group so that the grid still covers the chip (one wave of 2 CTAs/SM), at the price of more
      // inversions per jump.  KGX_STREAM_G overrides.
      int ctas = 2;
      if (const char* sc = getenv("KGX_STREAM_CTAS")) ctas = atoi(sc);
      if (ctas != 2 && ctas != 3) { snprintf(g_create_err, sizeof g_create_err, "kgx_create: KGX_STREAM_CTAS must be 2 or 3"); delete e; return nullptr; }
      bool invChosen = false;
      if (const char* si = getenv("KGX_STREAM_INV")) {
        invChosen = true;
        if (!strcmp(si, "thread")) e->warpInv = false;
        else if (strcmp(si, "warp")) { snprintf(g_create_err, sizeof g_create_err, "kgx_create: KGX_STREAM_INV must be warp or thread"); delete e; return nullptr; }
      }
      const u64 slots = (u64)ctas * prop.multiProcessorCount * 128;       // threads of one wave
      long long g = (long long)((e->n + slots - 1) / slots);               // round UP: never more tiles than one wave
      g = (g + 1) & ~1LL;
      if (g > 128) g = 128;
      if (g < 2) g = 2;
      if (stream_g > 0) g = stream_g;
      else if (const char* sg = getenv("KGX_STREAM_G")) g = atoi(sg);
      if (g < 2 || g > 4096 || (g & 1)) { snprintf(g_create_err, sizeof g_create_err, "kgx_create: stream group size (KGX_STREAM_G) must be an even number in [2, 4096]"); delete e; return nullptr; }
      // group inverse: the warp-wide shuffle butterfly (one uniform inverse per warp and pass) for long groups, one inverse per
      // thread for short ones, where the butterfly's 10 extra multiplications per lane weigh more than lane divergence inside
      // the variable-time inverse
      if (!invChosen) e->warpInv = g >= 64;
      if (const char* pf = getenv("KGX_STREAM_PF")) e->pfDist = atoi(pf);
      e->streamCtas = ctas;
      e->K = (int)g;
    }
  }
  e->kern = find_kernel(e->kind, e->T, e->K, e->streamCtas, e->warpInv, false);   // every non-symmetric selection is compiled
  e->T = e->kern->T;
  if (e->kind != KGX_KERNEL_STREAM) e->K = e->kern->K;
  const u64 TILE = (u64)e->T * e->K;
  e->numTiles = (u32)((e->n + TILE - 1) / TILE);
  e->nPadded = (u64)e->numTiles * TILE;
  e->maxFound = max_found;
  e->stateBytes = (size_t)e->nPadded * CHUNKS * 16;
  e->slabBytes = (size_t)max_found * KGX_ITEM_SIZE + 4;
  if ((s = cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking)) != cudaSuccess) return fail("cudaStreamCreate", s);
  if ((s = cudaStreamCreateWithFlags(&e->copyStream, cudaStreamNonBlocking)) != cudaSuccess) return fail("cudaStreamCreate", s);
  for (int i = 0; i < 2; i++) {
    if ((s = cudaEventCreate(&e->evStart[i])) != cudaSuccess) return fail("cudaEventCreate", s);
    if ((s = cudaEventCreateWithFlags(&e->evStop[i], cudaEventBlockingSync)) != cudaSuccess) return fail("cudaEventCreate", s);
  }
  if ((s = cudaMalloc(&e->state, e->stateBytes)) != cudaSuccess) return fail("cudaMalloc(state)", s);
  if (e->kind == KGX_KERNEL_STREAM && (s = cudaMalloc(&e->pre, (size_t)e->nPadded * 32)) != cudaSuccess) return fail("cudaMalloc(pre)", s);
  if (e->kind == KGX_KERNEL_STREAM && (s = cudaMalloc(&e->jlog, (size_t)e->nPadded * LOG_RUNS)) != cudaSuccess) return fail("cudaMalloc(jlog)", s);
  for (int i = 0; i < 2; i++) {
    if ((s = cudaMalloc(&e->slab[i], e->slabBytes)) != cudaSuccess) return fail("cudaMalloc(slab)", s);
    if ((s = cudaMemsetAsync(e->slab[i], 0, 4, e->stream)) != cudaSuccess) return fail("cudaMemset(slab)", s);  // Check.cpp:526 collects before any launch
  }
  if ((s = cudaMalloc(&e->jtab, JT_WORDS * 4)) != cudaSuccess) return fail("cudaMalloc(jtab)", s);
  if (getenv("KGX_PROF")) {
    if ((s = cudaMalloc(&e->prof, 64)) != cudaSuccess) return fail("cudaMalloc(prof)", s);
    cudaMemset(e->prof, 0, 64);
  }
  if ((s = cudaHostAlloc(&e->slabPinned, e->slabBytes, cudaHostAllocDefault)) != cudaSuccess) return fail("cudaHostAlloc", s);
  if ((s = cudaFuncSetAttribute(e->kern->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, e->kern->smem)) != cudaSuccess)
    return fail("cudaFuncSetAttribute(smem)", s);
  if ((s = cudaStreamSynchronize(e->stream)) != cudaSuccess) return fail("sync", s);
  return e;
}

uint64_t kgx_num_kangaroos(kgx_engine* e) { return e->n; }
int kgx_kernel_kind(kgx_engine* e) { return e->kind; }
uint64_t kgx_memory_bytes(kgx_engine* e) {
  return e->stateBytes + (e->pre ? e->nPadded * 32 : 0) + (e->jlog ? e->nPadded * LOG_RUNS : 0) + 2 * e->slabBytes + JT_WORDS * 4 +
         (e->targets ? e->n * 4 : 0) + (u64)e->keyCap * (64 + 64 + 4);
}
uint32_t kgx_max_found(kgx_engine* e) { return e->maxFound; }
float kgx_last_launch_ms(kgx_engine* e) { return e->lastMs; }
uint64_t kgx_kernel_launches(kgx_engine* e) { return e->launches; }
// debug: read and reset the phase counters (KGX_PROF=1): serial, modinv, parallel cycles, tile-steps
int kgx_debug_prof(kgx_engine* e, uint64_t out[4]) {
  if (!e->prof) return -1;
  cudaStreamSynchronize(e->stream);
  cudaMemcpy(out, e->prof, 32, cudaMemcpyDeviceToHost);
  cudaMemset(e->prof, 0, 64);
  return 0;
}
int kgx_set_jumps_per_launch(kgx_engine* e, int n_run) {
  if (n_run <= 0) { snprintf(e->err, sizeof e->err, "kgx_set_jumps_per_launch: n_run must be > 0"); return -1; }
  e->nRun = n_run; return 0;
}

// USE_SYMMETRY engine mode (SURVEY 8f/f4).  Must be chosen before the herd is uploaded: it allocates the lastJump bytes,
// switches the jump kernels to their symmetric instantiation and makes every distance crossing the ABI a SIGNED 128-bit
// two's complement value (no wild-offset bias).
int kgx_set_symmetry(kgx_engine* e, int on) {
  CK(e, cudaSetDevice(e->dev));
  if (e->inflight) { snprintf(e->err, sizeof e->err, "kgx_set_symmetry: a launch is in flight"); return -1; }
  const KernelEntry* kern = find_kernel(e->kind, e->T, e->K, e->streamCtas, e->warpInv, on != 0);
  if (!kern) {
    if (e->kind == KGX_KERNEL_TMEM) snprintf(e->err, sizeof e->err, "kgx_set_symmetry: the cluster tile kernel has no symmetric instantiation");
    else if (e->kind == KGX_KERNEL_STREAM) snprintf(e->err, sizeof e->err, "kgx_set_symmetry: the symmetric stream kernel is the 2-CTA variant only");
    else snprintf(e->err, sizeof e->err, "kgx_set_symmetry: tile geometry %d,%d has no symmetric instantiation", e->T, e->K);
    return -1;
  }
  if (on != 0 && on != KGX_SYM_LASTJUMP && on != KGX_SYM_CLASS) { snprintf(e->err, sizeof e->err, "kgx_set_symmetry: mode must be 0, 1 (lastJump rule) or 2 (symClass rule)"); return -1; }
  if (on && !e->aux) CK(e, cudaMalloc(&e->aux, e->nPadded));
  if (on) CK(e, cudaMemsetAsync(e->aux, on == KGX_SYM_CLASS ? 0 : 32, e->nPadded, e->stream));
  e->symRule = on;
  if (on) e->nKeys = 0;        // a multi-key herd is not available in symmetric mode (kgx_create_herd_multi): drop its table
  CK(e, cudaFuncSetAttribute(kern->fn, cudaFuncAttributeMaxDynamicSharedMemorySize, kern->smem));
  e->kern = kern;
  e->symmetry = on != 0;
  return 0;
}
int kgx_get_symmetry(kgx_engine* e) { return e->symmetry ? e->symRule : 0; }

// word w (0..7 jpx, 8..15 jpy, 16..19 jd) of jump j in the device table: uint4 jt[w / 4][j], component w % 4 (kgx_kernel.cuh)
static inline int jt_word(int w, int j) { return ((w >> 2) * 32 + j) * 4 + (w & 3); }

int kgx_set_params(kgx_engine* e, uint64_t dp_mask, const uint64_t* jd, const uint64_t* jpx, const uint64_t* jpy) {
  CK(e, cudaSetDevice(e->dev));
  u32 tab[JT_WORDS];
  for (int j = 0; j < 32; j++) {
    for (int w = 0; w < 8; w++) {
      tab[jt_word(w, j)] = (u32)(jpx[4 * j + w / 2] >> (32 * (w & 1)));
      tab[jt_word(8 + w, j)] = (u32)(jpy[4 * j + w / 2] >> (32 * (w & 1)));
    }
    for (int w = 0; w < 4; w++) tab[jt_word(16 + w, j)] = (u32)(jd[2 * j + w / 2] >> (32 * (w & 1)));
  }
  CK(e, cudaStreamSynchronize(e->stream));   // a running kernel may still read the old table
  CK(e, cudaMemcpy(e->jtab, tab, sizeof tab, cudaMemcpyHostToDevice));
  e->dpMask = dp_mask;
  e->haveParams = true;
  return 0;
}

static int ensure_staging(kgx_engine* e) {
  if (e->stgX) return 0;
  CK(e, cudaMalloc(&e->stgX, e->n * 32));
  CK(e, cudaMalloc(&e->stgY, e->n * 32));
  CK(e, cudaMalloc(&e->stgD, e->n * 16));
  return 0;
}
static void free_staging(kgx_engine* e) {
  cudaFree(e->stgX); cudaFree(e->stgY); cudaFree(e->stgD);
  e->stgX = e->stgY = e->stgD = nullptr;
}

int kgx_upload(kgx_engine* e, const uint64_t* px, const uint64_t* py, const uint64_t* d) {
  CK(e, cudaSetDevice(e->dev));
  if (e->snapPending) { snprintf(e->err, sizeof e->err, "kgx_upload: snapshot pending (read it first)"); return -1; }
  if (ensure_staging(e)) return -1;
  CK(e, cudaMemcpyAsync(e->stgX, px, e->n * 32, cudaMemcpyHostToDevice, e->stream));
  CK(e, cudaMemcpyAsync(e->stgY, py, e->n * 32, cudaMemcpyHostToDevice, e->stream));
  CK(e, cudaMemcpyAsync(e->stgD, d, e->n * 16, cudaMemcpyHostToDevice, e->stream));
  u32 blocks = (u32)((e->nPadded + 255) / 256);
  pack_kernel<<<blocks, 256, 0, e->stream>>>(e->state, e->stgX, e->stgY, e->stgD, e->n, e->nPadded, e->T, e->K, e->aux, aux_init(e));
  e->launches++;
  CK(e, cudaGetLastError());
  CK(e, cudaStreamSynchronize(e->stream));
  free_staging(e);
  return 0;
}

int kgx_download(kgx_engine* e, uint64_t* px, uint64_t* py, uint64_t* d) {
  CK(e, cudaSetDevice(e->dev));
  if (e->snapPending) { snprintf(e->err, sizeof e->err, "kgx_download: snapshot pending (read it first)"); return -1; }
  if (ensure_staging(e)) return -1;
  u32 blocks = (u32)((e->n + 255) / 256);
  unpack_kernel<<<blocks, 256, 0, e->stream>>>(e->state, e->stgX, e->stgY, e->stgD, e->n, e->T, e->K);   // stream order: after the in-flight launch
  e->launches++;
  CK(e, cudaGetLastError());
  CK(e, cudaMemcpyAsync(px, e->stgX, e->n * 32, cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaMemcpyAsync(py, e->stgY, e->n * 32, cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaMemcpyAsync(d, e->stgD, e->n * 16, cudaMemcpyDeviceToHost, e->stream));
  CK(e, cudaStreamSynchronize(e->stream));
  free_staging(e);
  return 0;
}

// ---- asynchronous checkpoint (SURVEY 8f/f3; reference: SolveKeyGPU parks on saveMutex while GetKangaroos copies the
// whole herd with blocking memcpys, Kangaroo.cpp:618-626).  kgx_snapshot_begin() enqueues, in stream order (i.e. after the
// launch in flight), a device-side copy of the herd into kIdx-ordered staging and returns at once; later launches run
// on; kgx_snapshot_read() waits for that copy only and moves it to the host on the copy stream.
int kgx_snapshot_begin(kgx_engine* e) {
  CK(e, cudaSetDevice(e->dev));
  if (e->snapPending) { snprintf(e->err, sizeof e->err, "kgx_snapshot_begin: previous snapshot not read"); return -1; }
  if (ensure_staging(e)) return -1;
  if (!e->evSnap) CK(e, cudaEventCreateWithFlags(&e->evSnap, cudaEventBlockingSync | cudaEventDisableTiming));
  u32 blocks = (u32)((e->n + 255) / 256);
  unpack_kernel<<<blocks, 256, 0, e->stream>>>(e->state, e->stgX, e->stgY, e->stgD, e->n, e->T, e->K);
  e->launches++;
  CK(e, cudaGetLastError());
  // the targets of a multi-key herd, in the same stream order: a kgx_retarget queued after this call changes e->targets only
  if (e->nKeys) CK(e, cudaMemcpyAsync(e->snapTargets, e->targets, e->n * 2, cudaMemcpyDeviceToDevice, e->stream));
  CK(e, cudaEventRecord(e->evSnap, e->stream));
  e->snapPending = true;
  e->snapConverted = false;
  e->snapHasTargets = e->nKeys != 0;
  return 0;
}

int kgx_snapshot_read(kgx_engine* e, uint64_t* px, uint64_t* py, uint64_t* d) {
  CK(e, cudaSetDevice(e->dev));
  if (!e->snapPending) { snprintf(e->err, sizeof e->err, "kgx_snapshot_read: no snapshot pending"); return -1; }
  CK(e, cudaStreamWaitEvent(e->copyStream, e->evSnap, 0));
  CK(e, cudaMemcpyAsync(px, e->stgX, e->n * 32, cudaMemcpyDeviceToHost, e->copyStream));
  CK(e, cudaMemcpyAsync(py, e->stgY, e->n * 32, cudaMemcpyDeviceToHost, e->copyStream));
  CK(e, cudaMemcpyAsync(d, e->stgD, e->n * 16, cudaMemcpyDeviceToHost, e->copyStream));
  CK(e, cudaStreamSynchronize(e->copyStream));
  e->snapPending = false;
  free_staging(e);
  return 0;
}

// Work-file records of the pending snapshot (kgx_ckpt.cuh).  The first call converts the whole snapshot on the copy stream
// (after the snapshot's unpack, concurrently with the jump launches queued since); every call copies records
// [first, first+count) to dst (host or device memory of this engine's GPU).  The call whose range ends at n releases the
// snapshot.  The staging (stgX/stgY/stgD, 80 B per kangaroo) and herdRecs (96 B per kangaroo) stay allocated for the next
// save: cudaFree synchronises the device and would wait for the jump launch in flight.
int kgx_snapshot_export(kgx_engine* e, const uint64_t wild_offset[2], uint64_t first, uint64_t count, void* dst) {
  CK(e, cudaSetDevice(e->dev));
  if (e->symmetry) { snprintf(e->err, sizeof e->err, "kgx_snapshot_export: not available in symmetric mode (signed distances)"); return -1; }
  if (!e->snapPending) { snprintf(e->err, sizeof e->err, "kgx_snapshot_export: no snapshot pending"); return -1; }
  if (first > e->n || count > e->n - first) { snprintf(e->err, sizeof e->err, "kgx_snapshot_export: range [%llu, +%llu) outside the herd", (unsigned long long)first, (unsigned long long)count); return -1; }
  if (!e->snapConverted) {
    if (!e->herdRecs) CK(e, cudaMalloc(&e->herdRecs, e->n * 96));
    CK(e, cudaStreamWaitEvent(e->copyStream, e->evSnap, 0));
    herd_export_kernel<<<4 * e->sms, 256, 0, e->copyStream>>>(reinterpret_cast<const u32*>(e->stgX), reinterpret_cast<const u32*>(e->stgY),
                                                             reinterpret_cast<const u32*>(e->stgD), e->herdRecs, e->n, wild_offset[0], wild_offset[1]);
    e->launches++;
    CK(e, cudaGetLastError());
    e->snapConverted = true;
  }
  if (count) CK(e, cudaMemcpyAsync(dst, e->herdRecs + first * 12, count * 96, cudaMemcpyDefault, e->copyStream));
  CK(e, cudaStreamSynchronize(e->copyStream));
  if (first + count == e->n) { e->snapPending = false; e->snapConverted = false; }
  return 0;
}

int kgx_snapshot_export_targets(kgx_engine* e, uint64_t first, uint64_t count, uint16_t* dst) {
  CK(e, cudaSetDevice(e->dev));
  if (!e->snapPending) { snprintf(e->err, sizeof e->err, "kgx_snapshot_export_targets: no snapshot pending"); return -1; }
  if (!e->snapHasTargets) { snprintf(e->err, sizeof e->err, "kgx_snapshot_export_targets: the snapshot's herd has no key table (kgx_create_herd_multi)"); return -1; }
  if (first > e->n || count > e->n - first) { snprintf(e->err, sizeof e->err, "kgx_snapshot_export_targets: range [%llu, +%llu) outside the herd", (unsigned long long)first, (unsigned long long)count); return -1; }
  CK(e, cudaStreamWaitEvent(e->copyStream, e->evSnap, 0));
  if (count) CK(e, cudaMemcpyAsync(dst, e->snapTargets + first, count * 2, cudaMemcpyDeviceToHost, e->copyStream));
  CK(e, cudaStreamSynchronize(e->copyStream));
  return 0;
}

// The device key table of a multi-key herd, grown to n_keys, and the per-kangaroo targets (kgx_create_herd_multi,
// kgx_import_multi).  The snapshot's copy of the targets is allocated with them: kgx_snapshot_begin allocates nothing.
static int ensure_key_table(kgx_engine* e, uint32_t n_keys) {
  if (n_keys > e->keyCap) {
    cudaFree(e->keys); cudaFree(e->rtDelta); cudaFree(e->rtTo);
    e->keys = e->rtDelta = e->rtTo = nullptr;
    e->keyCap = 0;
    CK(e, cudaMalloc(&e->keys, (size_t)n_keys * 64));
    CK(e, cudaMalloc(&e->rtDelta, (size_t)n_keys * 64));
    CK(e, cudaMalloc(&e->rtTo, (size_t)n_keys * 4));
    e->keyCap = n_keys;
  }
  if (!e->targets) CK(e, cudaMalloc(&e->targets, e->n * 2));
  if (!e->snapTargets) CK(e, cudaMalloc(&e->snapTargets, e->n * 2));
  // load the retarget kernels now: kgx_retarget must not be the first launch of a kernel, which can wait for the device
  cudaFuncAttributes fa;
  CK(e, cudaFuncGetAttributes(&fa, retarget_delta_kernel));
  CK(e, cudaFuncGetAttributes(&fa, retarget_kernel));
  return 0;
}

// Replace kangaroos 0..count-1 by `count` work-file records (host memory), in stream order after the launch in flight.
// Nothing changes when a record's biased distance does not fit in 128 bits (error) or, with verify != 0, when any position
// differs from d*G (tame) / key + d*G (wild): *mismatches then says how many do (0 = imported).  keys: n_keys x 8 limbs;
// targets NULL: one key; else wild record i is checked against keys[targets[i]], and on success the key table and the
// targets of kangaroos 0..count-1 are installed (kgx_import_multi).
static int import_records(kgx_engine* e, const char* what, const uint64_t wild_offset[2], const void* recs, uint64_t count,
                          const uint64_t* keys, uint32_t n_keys, const uint16_t* targets, int verify, uint64_t* mismatches) {
  CK(e, cudaSetDevice(e->dev));
  if (mismatches) *mismatches = 0;
  if (e->symmetry) { snprintf(e->err, sizeof e->err, "%s: not available in symmetric mode (signed distances)", what); return -1; }
  if (e->snapPending) { snprintf(e->err, sizeof e->err, "%s: snapshot pending (export it first)", what); return -1; }
  if (count > e->n) { snprintf(e->err, sizeof e->err, "%s: %llu records for a herd of %llu", what, (unsigned long long)count, (unsigned long long)e->n); return -1; }
  if (targets) {
    if (n_keys == 0 || n_keys > KGX_MAX_KEYS) { snprintf(e->err, sizeof e->err, "%s: n_keys must be in [1, %d]", what, KGX_MAX_KEYS); return -1; }
    for (u64 i = 0; i < count; i++)
      if (targets[i] >= n_keys) {
        snprintf(e->err, sizeof e->err, "%s: target %u of record %llu is not below n_keys = %u", what, targets[i], (unsigned long long)i, n_keys);
        return -1;
      }
    if (count < e->n && !e->nKeys) {
      snprintf(e->err, sizeof e->err, "%s: %llu records for a herd of %llu without a key table (kgx_create_herd_multi first)", what,
               (unsigned long long)count, (unsigned long long)e->n);
      return -1;
    }
  }
  if (count == 0) return 0;
  if (verify && !e->herdTab) {
    CK(e, cudaMalloc(&e->herdTab, 256 * 16 * 4));
    herd_table_kernel<<<1, 32, 0, e->stream>>>(e->herdTab);
    e->launches++;
    CK(e, cudaGetLastError());
  }
  if (!e->herdRecs) CK(e, cudaMalloc(&e->herdRecs, e->n * 96));
  if (ensure_staging(e)) return -1;
  u32 *scal = nullptr, *vx = nullptr, *vy = nullptr, *dKey = nullptr;
  uint16_t* dTg = nullptr;
  unsigned long long* flags = nullptr;     // [0] lowest out-of-range index (~0 = none), [1] mismatches
  auto body = [&]() -> int {
    CK(e, cudaMalloc(&scal, count * 32));
    CK(e, cudaMalloc(&flags, 16));
    const unsigned long long init[2] = {~0ull, 0ull};
    CK(e, cudaMemcpyAsync(flags, init, 16, cudaMemcpyHostToDevice, e->stream));
    CK(e, cudaMemcpyAsync(e->herdRecs, recs, count * 96, cudaMemcpyHostToDevice, e->stream));
    unpack_kernel<<<(u32)((e->n + 255) / 256), 256, 0, e->stream>>>(e->state, e->stgX, e->stgY, e->stgD, e->n, e->T, e->K);
    e->launches++;
    CK(e, cudaGetLastError());
    herd_import_kernel<<<4 * e->sms, 256, 0, e->stream>>>(e->herdRecs, count, wild_offset[0], wild_offset[1], reinterpret_cast<u32*>(e->stgX),
                                                         reinterpret_cast<u32*>(e->stgY), reinterpret_cast<u32*>(e->stgD), scal, flags);
    e->launches++;
    CK(e, cudaGetLastError());
    if (verify) {
      CK(e, cudaMalloc(&vx, count * 32));
      CK(e, cudaMalloc(&vy, count * 32));
      CK(e, cudaMalloc(&dKey, (size_t)n_keys * 64));
      CK(e, cudaMemcpyAsync(dKey, keys, (size_t)n_keys * 64, cudaMemcpyHostToDevice, e->stream));
      if (targets) {
        CK(e, cudaMalloc(&dTg, count * 2));
        CK(e, cudaMemcpyAsync(dTg, targets, count * 2, cudaMemcpyHostToDevice, e->stream));
      }
      herd_kernel<<<(u32)((count + 127) / 128), 128, 0, e->stream>>>(e->herdTab, scal, dKey, dTg, 0, count, vx, vy, 0, nullptr);
      e->launches++;
      CK(e, cudaGetLastError());
      herd_compare_kernel<<<4 * e->sms, 256, 0, e->stream>>>(reinterpret_cast<u32*>(e->stgX), reinterpret_cast<u32*>(e->stgY), vx, vy, count, flags + 1);
      e->launches++;
      CK(e, cudaGetLastError());
    }
    unsigned long long res[2];
    CK(e, cudaMemcpyAsync(res, flags, 16, cudaMemcpyDeviceToHost, e->stream));
    CK(e, cudaStreamSynchronize(e->stream));
    if (res[0] != ~0ull) {
      snprintf(e->err, sizeof e->err, "kgx_import: record %llu: distance does not fit the engine's 128-bit form (a file of another range?)", res[0]);
      return -1;
    }
    if (mismatches) *mismatches = res[1];
    if (res[1]) return 0;
    if (targets) {                         // verified: install the key table and the targets, as kgx_create_herd_multi does
      if (ensure_key_table(e, n_keys)) return -1;
      CK(e, cudaMemcpyAsync(e->keys, keys, (size_t)n_keys * 64, cudaMemcpyHostToDevice, e->stream));
      CK(e, cudaMemcpyAsync(e->targets, targets, count * 2, cudaMemcpyHostToDevice, e->stream));
    }
    pack_kernel<<<(u32)((e->nPadded + 255) / 256), 256, 0, e->stream>>>(e->state, e->stgX, e->stgY, e->stgD, e->n, e->nPadded, e->T, e->K, e->aux, aux_init(e));
    e->launches++;
    CK(e, cudaGetLastError());
    CK(e, cudaStreamSynchronize(e->stream));
    if (targets) { e->nKeys = n_keys; e->firstType = 0; }
    return 0;
  };
  const int rc = body();
  cudaFree(scal); cudaFree(vx); cudaFree(vy); cudaFree(dKey); cudaFree(dTg); cudaFree(flags);
  free_staging(e);
  return rc;
}

int kgx_import(kgx_engine* e, const uint64_t wild_offset[2], const void* recs, uint64_t count, const uint64_t keyx[4],
               const uint64_t keyy[4], int verify, uint64_t* mismatches) {
  uint64_t key[8];
  memcpy(key, keyx, 32); memcpy(key + 4, keyy, 32);
  return import_records(e, "kgx_import", wild_offset, recs, count, key, 1, nullptr, verify, mismatches);
}

int kgx_import_multi(kgx_engine* e, const uint64_t wild_offset[2], const void* recs, uint64_t count, const uint64_t* keys,
                     uint32_t n_keys, const uint16_t* targets, int verify, uint64_t* mismatches) {
  return import_records(e, "kgx_import_multi", wild_offset, recs, count, keys, n_keys, targets, verify, mismatches);
}

int kgx_patch(kgx_engine* e, uint64_t kidx, const uint64_t px[4], const uint64_t py[4], const uint64_t d[2]) {
  CK(e, cudaSetDevice(e->dev));
  if (kidx >= e->n) { snprintf(e->err, sizeof e->err, "kgx_patch: kidx out of range"); return -1; }
  PatchArgs a;
  memcpy(&a.c[0], px, 32); memcpy(&a.c[2], py, 32); memcpy(&a.c[4], d, 16);
  patch_kernel<<<1, 32, 0, e->stream>>>(e->state, kidx, a, e->T, e->K, e->aux, aux_init(e));   // stream order == the reference's blocking memcpy order (Kangaroo.cpp:607)
  e->launches++;
  CK(e, cudaGetLastError());
  // padding slots replicate kangaroo (s % n): keep them walking their stale copy -- harmless, their DPs are dropped.
  return 0;
}

// Kangaroo::CreateHerd on the device (Kangaroo.cpp:670-738): positions d*G (tame) / key + d*G (wild) for all n
// kangaroos straight into the engine state.  scalars: n x 4 limbs (d mod group order, exactly what the reference
// feeds ComputePublicKeys); d128: n x 2 limbs (the biased distances to store).  keys: n_keys x 8 limbs (x, y); targets
// NULL: one key, no key table kept; else the wild term of kangaroo i is keys[targets[i]] and the table and the targets stay
// in the engine for kgx_retarget.
static int create_herd(kgx_engine* e, const char* what, const uint64_t* scalars, const uint64_t* d128, const uint64_t* keys,
                       uint32_t n_keys, const uint16_t* targets, int first_type) {
  CK(e, cudaSetDevice(e->dev));
  if (e->snapPending) { snprintf(e->err, sizeof e->err, "%s: snapshot pending (read it first)", what); return -1; }
  e->nKeys = 0;
  if (!e->herdTab) {
    CK(e, cudaMalloc(&e->herdTab, 256 * 16 * 4));
    herd_table_kernel<<<1, 32, 0, e->stream>>>(e->herdTab);
    e->launches++;
    CK(e, cudaGetLastError());
  }
  if (ensure_staging(e)) return -1;
  u32 *dScal = nullptr, *dKey = nullptr;
  auto body = [&]() -> int {      // CK returns from the lambda, so the scratch buffers are always released below
    CK(e, cudaMalloc(&dScal, e->n * 32));
    if (targets) {
      if (ensure_key_table(e, n_keys)) return -1;
      CK(e, cudaMemcpyAsync(e->keys, keys, (size_t)n_keys * 64, cudaMemcpyHostToDevice, e->stream));
      CK(e, cudaMemcpyAsync(e->targets, targets, e->n * 2, cudaMemcpyHostToDevice, e->stream));
    } else {
      CK(e, cudaMalloc(&dKey, 64));
      CK(e, cudaMemcpyAsync(dKey, keys, 64, cudaMemcpyHostToDevice, e->stream));
    }
    CK(e, cudaMemcpyAsync(dScal, scalars, e->n * 32, cudaMemcpyHostToDevice, e->stream));
    CK(e, cudaMemcpyAsync(e->stgD, d128, e->n * 16, cudaMemcpyHostToDevice, e->stream));
    herd_kernel<<<(u32)((e->n + 127) / 128), 128, 0, e->stream>>>(e->herdTab, dScal, targets ? e->keys : dKey, targets ? e->targets : nullptr,
                                                                 first_type, e->n, reinterpret_cast<u32*>(e->stgX), reinterpret_cast<u32*>(e->stgY),
                                                                 e->symmetry ? 1 : 0, reinterpret_cast<u32*>(e->stgD));
    e->launches++;
    CK(e, cudaGetLastError());
    u32 blocks = (u32)((e->nPadded + 255) / 256);
    pack_kernel<<<blocks, 256, 0, e->stream>>>(e->state, e->stgX, e->stgY, e->stgD, e->n, e->nPadded, e->T, e->K, e->aux, aux_init(e));
    e->launches++;
    CK(e, cudaGetLastError());
    CK(e, cudaStreamSynchronize(e->stream));
    return 0;
  };
  const int rc = body();
  cudaFree(dScal); cudaFree(dKey);
  free_staging(e);
  if (rc == 0 && targets) { e->nKeys = n_keys; e->firstType = first_type; }
  return rc;
}

int kgx_create_herd(kgx_engine* e, const uint64_t* scalars, const uint64_t* d128, const uint64_t keyx[4], const uint64_t keyy[4], int first_type) {
  uint64_t key[8];
  memcpy(key, keyx, 32); memcpy(key + 4, keyy, 32);
  return create_herd(e, "kgx_create_herd", scalars, d128, key, 1, nullptr, first_type);
}

int kgx_create_herd_multi(kgx_engine* e, const uint64_t* scalars, const uint64_t* d128, const uint64_t* keys, uint32_t n_keys,
                          const uint16_t* targets, int first_type) {
  if (e->symmetry) { snprintf(e->err, sizeof e->err, "kgx_create_herd_multi: not available in symmetric mode"); return -1; }
  if (n_keys == 0 || n_keys > KGX_MAX_KEYS) { snprintf(e->err, sizeof e->err, "kgx_create_herd_multi: n_keys must be in [1, %d]", KGX_MAX_KEYS); return -1; }
  for (u64 i = 0; i < e->n; i++)
    if (targets[i] >= n_keys) {
      snprintf(e->err, sizeof e->err, "kgx_create_herd_multi: target %u of kangaroo %llu is not below n_keys = %u", targets[i], (unsigned long long)i, n_keys);
      return -1;
    }
  return create_herd(e, "kgx_create_herd_multi", scalars, d128, keys, n_keys, targets, first_type);
}

// Moves the wild kangaroos of key `from` to the keys in `to`, in stream order after the launch in flight (like kgx_patch),
// without waiting for it: the destination list reaches the device as kernel parameters (retarget_delta_kernel), one
// affine addition per moved kangaroo follows (retarget_kernel).
int kgx_retarget(kgx_engine* e, uint32_t from, const uint16_t* to, uint32_t n_to) {
  CK(e, cudaSetDevice(e->dev));
  if (e->symmetry) { snprintf(e->err, sizeof e->err, "kgx_retarget: not available in symmetric mode"); return -1; }
  if (!e->nKeys) { snprintf(e->err, sizeof e->err, "kgx_retarget: the herd has no key table (kgx_create_herd_multi)"); return -1; }
  if (from >= e->nKeys) { snprintf(e->err, sizeof e->err, "kgx_retarget: key %u is not below n_keys = %u", from, e->nKeys); return -1; }
  if (n_to == 0 || n_to > e->nKeys) { snprintf(e->err, sizeof e->err, "kgx_retarget: n_to must be in [1, n_keys = %u]", e->nKeys); return -1; }
  for (u32 j = 0; j < n_to; j++)
    if (to[j] >= e->nKeys) { snprintf(e->err, sizeof e->err, "kgx_retarget: to[%u] = %u is not below n_keys = %u", j, to[j], e->nKeys); return -1; }
  for (u32 j0 = 0; j0 < n_to; j0 += RETARGET_CHUNK) {
    const u32 cnt = n_to - j0 < (u32)RETARGET_CHUNK ? n_to - j0 : (u32)RETARGET_CHUNK;
    RetargetChunk c;
    memset(&c, 0, sizeof c);
    memcpy(c.to, to + j0, (size_t)cnt * 2);
    retarget_delta_kernel<<<(cnt + 127) / 128, 128, 0, e->stream>>>(e->keys, from, c, j0, cnt, e->rtDelta, e->rtTo);
    e->launches++;
    CK(e, cudaGetLastError());
  }
  retarget_kernel<<<(u32)((e->n + 255) / 256), 256, 0, e->stream>>>(e->state, e->T, e->K, e->n, e->firstType, e->targets, from,
                                                                   e->rtDelta, e->rtTo, n_to);
  e->launches++;
  CK(e, cudaGetLastError());
  return 0;
}

int kgx_targets(kgx_engine* e, uint16_t* out) {
  CK(e, cudaSetDevice(e->dev));
  if (e->symmetry) { snprintf(e->err, sizeof e->err, "kgx_targets: not available in symmetric mode"); return -1; }
  if (!e->nKeys) { snprintf(e->err, sizeof e->err, "kgx_targets: the herd has no key table (kgx_create_herd_multi)"); return -1; }
  CK(e, cudaMemcpyAsync(out, e->targets, e->n * 2, cudaMemcpyDeviceToHost, e->stream));   // stream order: after the retargets
  CK(e, cudaStreamSynchronize(e->stream));
  return 0;
}

int kgx_launch_async(kgx_engine* e) {
  CK(e, cudaSetDevice(e->dev));
  if (!e->haveParams) { snprintf(e->err, sizeof e->err, "kgx_launch_async: kgx_set_params not called"); return -1; }
  if (e->inflight) { snprintf(e->err, sizeof e->err, "kgx_launch_async: previous launch not collected"); return -1; }
  int sidx = e->cur ^ 1;
  LaunchParams p;
  p.state = e->state; p.jtab = e->jtab; p.out = e->slab[sidx]; p.dpMask = e->dpMask; p.nKangaroos = e->n;
  p.numTiles = e->numTiles; p.maxFound = e->maxFound; p.nRun = e->nRun; p.prof = e->prof; p.pre = e->pre; p.G = e->K; p.aux = e->aux; p.symRule = e->symRule; p.pfDist = e->pfDist; p.jlog = e->jlog;
  CK(e, cudaMemsetAsync(e->slab[sidx], 0, 4, e->stream));            // GPUEngine.cu:543
  CK(e, cudaEventRecord(e->evStart[sidx], e->stream));
  const KernelEntry& k = *e->kern;
  u32 grid = (u32)(k.ctasPerSM * e->sms);
  if (grid > e->numTiles * k.ctasPerTile) grid = e->numTiles * k.ctasPerTile;
  k.fn<<<grid, k.T, k.smem, e->stream>>>(p);
  e->launches++;
  CK(e, cudaGetLastError());
  CK(e, cudaEventRecord(e->evStop[sidx], e->stream));
  e->cur = sidx;
  e->inflight = true;
  return 0;
}

int kgx_collect(kgx_engine* e, kgx_item* items, uint32_t cap, uint32_t* n_items, uint32_t* n_found, int spin, int relaunch) {
  CK(e, cudaSetDevice(e->dev));
  *n_items = 0; *n_found = 0;
  int sidx = e->cur;
  if (e->inflight) {
    if (spin) {
      cudaError_t q;
      while ((q = cudaEventQuery(e->evStop[sidx])) == cudaErrorNotReady) { }
      CK(e, q);                                       // anything but success / not-ready is a failed launch
    } else {
      CK(e, cudaEventSynchronize(e->evStop[sidx]));   // blocking-sync event: the host thread sleeps (GPUEngine.cu:620-629)
    }
    CK(e, cudaGetLastError());
    CK(e, cudaEventElapsedTime(&e->lastMs, e->evStart[sidx], e->evStop[sidx]));
    e->inflight = false;
    e->done = sidx;
  }
  if (relaunch) { if (kgx_launch_async(e)) return -1; }   // second half of GPUEngine::Launch, issued BEFORE the readback
  // read back slab `sidx` (the new launch writes the other slab)
  // (on its own stream, so it does not queue behind the kernel just started)
  CK(e, cudaMemcpyAsync(e->slabPinned, e->slab[sidx], 4, cudaMemcpyDeviceToHost, e->copyStream));
  CK(e, cudaStreamSynchronize(e->copyStream));
  u32 found = e->slabPinned[0];
  *n_found = found;
  u32 nrec = found > e->maxFound ? e->maxFound : found;
  if (nrec > cap) nrec = cap;
  if (nrec) {
    CK(e, cudaMemcpyAsync(e->slabPinned + 1, e->slab[sidx] + 1, (size_t)nrec * KGX_ITEM_SIZE, cudaMemcpyDeviceToHost, e->copyStream));
    CK(e, cudaStreamSynchronize(e->copyStream));
    memcpy(items, e->slabPinned + 1, (size_t)nrec * KGX_ITEM_SIZE);
  }
  *n_items = nrec;
  return 0;
}

int kgx_sync(kgx_engine* e) {
  CK(e, cudaSetDevice(e->dev));
  CK(e, cudaStreamSynchronize(e->stream));
  if (e->inflight) {
    CK(e, cudaEventElapsedTime(&e->lastMs, e->evStart[e->cur], e->evStop[e->cur]));
    e->inflight = false; e->done = e->cur;
  }
  return 0;
}

// HashTable::Convert on the device for the most recently completed launch (SURVEY 8f/f1).  wild_offset: 2 limbs.
// Returns the device pointer of [u32 count][count x 40-byte DP records] through *out (valid until the next call).
int kgx_convert_dps(kgx_engine* e, const uint64_t wild_offset[2], void** out) {
  CK(e, cudaSetDevice(e->dev));
  if (!e->dp40) CK(e, cudaMalloc(&e->dp40, (size_t)e->maxFound * 40 + 4));
  const int sidx = e->done >= 0 ? e->done : e->cur;
  dp_convert_kernel<<<64, 256, 0, e->copyStream>>>(e->slab[sidx], e->dp40, e->maxFound, wild_offset[0], wild_offset[1], e->symmetry ? 1 : 0);
  e->launches++;
  CK(e, cudaGetLastError());
  CK(e, cudaStreamSynchronize(e->copyStream));
  *out = e->dp40;
  return 0;
}

void* kgx_dp_slab_device(kgx_engine* e) { return e->done >= 0 ? (void*)e->slab[e->done] : (void*)e->slab[e->cur]; }

// ---- test / microbench hooks ----
#define CKH(call) do { cudaError_t _s = (call); if (_s != cudaSuccess) { snprintf(g_create_err, sizeof g_create_err, "%s: %s", #call, cudaGetErrorString(_s)); return -1; } } while (0)

int kgx_test_field(int dev, int op, int n, const uint64_t* a, const uint64_t* b, uint64_t* out) {
  if (op < KGX_TF_MUL || op > KGX_TF_SYM_NEXT_AUX || n <= 0) {
    snprintf(g_create_err, sizeof g_create_err, "kgx_test_field: bad op %d or count %d", op, n);
    return -1;
  }
  CKH(cudaSetDevice(dev));
  u32 *da, *db, *dout;
  CKH(cudaMalloc(&da, (size_t)n * 32)); CKH(cudaMalloc(&db, (size_t)n * 32)); CKH(cudaMalloc(&dout, (size_t)n * 32));
  CKH(cudaMemcpy(da, a, (size_t)n * 32, cudaMemcpyHostToDevice));
  CKH(cudaMemcpy(db, b, (size_t)n * 32, cudaMemcpyHostToDevice));
  test_field_kernel<<<(n + 127) / 128, 128>>>(op, n, da, db, dout);
  CKH(cudaGetLastError());
  CKH(cudaMemcpy(out, dout, (size_t)n * 32, cudaMemcpyDeviceToHost));
  cudaFree(da); cudaFree(db); cudaFree(dout);
  return 0;
}

int kgx_test_dp_convert(int dev, uint32_t count, uint32_t max_found, const void* recs56, const uint64_t wild_offset[2],
                        int signed_mode, void* out) {
  if (max_found == 0) { snprintf(g_create_err, sizeof g_create_err, "kgx_test_dp_convert: max_found must be > 0"); return -1; }
  CKH(cudaSetDevice(dev));
  const u32 stored = count < max_found ? count : max_found;
  const size_t slabBytes = 4 + (size_t)max_found * KGX_ITEM_SIZE, outBytes = 4 + (size_t)max_found * 40;
  u32 *slab = nullptr, *out40 = nullptr;
  auto body = [&]() -> int {
    CKH(cudaMalloc(&slab, slabBytes));
    CKH(cudaMalloc(&out40, outBytes));
    CKH(cudaMemset(slab, 0, slabBytes));
    CKH(cudaMemset(out40, 0xFF, outBytes));
    CKH(cudaMemcpy(slab, &count, 4, cudaMemcpyHostToDevice));
    if (stored) CKH(cudaMemcpy(slab + 1, recs56, (size_t)stored * KGX_ITEM_SIZE, cudaMemcpyHostToDevice));
    dp_convert_kernel<<<64, 256>>>(slab, out40, max_found, wild_offset[0], wild_offset[1], signed_mode ? 1 : 0);   // kgx_convert_dps's launch
    CKH(cudaGetLastError());
    CKH(cudaMemcpy(out, out40, outBytes, cudaMemcpyDeviceToHost));
    return 0;
  };
  const int rc = body();
  cudaFree(slab); cudaFree(out40);
  return rc;
}

int kgx_bench_raw(int dev, int kind, int iters, float* ms, double* ops) {
  CKH(cudaSetDevice(dev));
  cudaDeviceProp prop; CKH(cudaGetDeviceProperties(&prop, dev));
  u32* sink; CKH(cudaMalloc(&sink, 4));
  cudaEvent_t a, b; CKH(cudaEventCreate(&a)); CKH(cudaEventCreate(&b));
  const int blocks = prop.multiProcessorCount * 8, threads = 256;
  bench_raw_kernel<<<blocks, threads>>>(kind, iters / 8 + 1, sink);   // warm-up
  CKH(cudaDeviceSynchronize());
  CKH(cudaEventRecord(a));
  bench_raw_kernel<<<blocks, threads>>>(kind, iters, sink);
  CKH(cudaEventRecord(b));
  CKH(cudaEventSynchronize(b));
  CKH(cudaGetLastError());
  CKH(cudaEventElapsedTime(ms, a, b));
  double per_thread = kind == 0 ? 8.0 * iters : (kind == 3 ? 1.0 * iters : 2.0 * iters);
  *ops = per_thread * (double)blocks * threads;
  cudaFree(sink); cudaEventDestroy(a); cudaEventDestroy(b);
  return 0;
}

}  // extern "C"

#include "kgx_bucketsort.cuh"  // work-file order for a block of buckets (the table's save and the merge)
#include "kgx_worktool.cuh"  // work-file check and merge (kgx_work_*)
#include "kgx_partition.cuh" // a rank's DP records grouped by the shard that owns them (kgx_dp_partition)
#include "kgx_resolver.cuh"  // the persistent collision resolver (kgx_resolver_*), which the table's resolving add runs
#include "kgx_dptable.cuh"   // the device-resident DP table (kgx_dptable_*)
