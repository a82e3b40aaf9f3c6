// GPUEngine_b200.cpp -- drop-in implementation of the reference's `class GPUEngine` on top of libkgx.so.
//
// The class declaration is the reference's own, UNCHANGED header GPU/GPUEngine.h:40-84 (found on the include path
// at build time: -I$KANGAROO_REF; this file replaces GPU/GPUEngine.cu in the link).  Every member keeps the
// semantics documented in SURVEY.md 8(b); the private data members of the verbatim header are reused as opaque
// storage (inputKangaroo -> kgx_engine*, outputItemPinned -> kgx_item staging) because the header cannot change.
//
// With this object and libkgx.so the reference's main.cpp / Kangaroo.cpp / Check.cpp / HashTable.cpp / SECPK1 build
// and run unmodified:  see kangaroo_b200/csrc/build_dropin.sh and INTEGRATION.md.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <thread>
#include <vector>
#include "GPU/GPUEngine.h"
#include "../../include/kgx.h"

#define KGX(e) (reinterpret_cast<kgx_engine*>(e))

static void int_to_limbs(uint64_t* dst, Int* v, int limbs) { for (int i = 0; i < limbs; i++) dst[i] = v->bits64[i]; }

// Distance marshalling across the C ABI.
//   default build : the reference's convention -- wild (odd kIdx) distances biased by wildOffset mod n on the way in and
//                   un-biased on the way out (GPUEngine.cu:407-411, 477, 526, 672), 128 bits unsigned on the device.
//   USE_SYMMETRY  : the engine is switched to kgx_set_symmetry(1); distances change sign on the device, so they travel as
//                   SIGNED 128-bit values: d mod n above n/2 is negative (the same test HashTable::Convert uses,
//                   HashTable.cpp:84-92).  The wild offset the host passes (rangeWidthDiv4, Kangaroo.cpp:548-550) is not
//                   applied: with sign switches a bias does not commute with negation, which is one of the reasons the
//                   reference's own symmetric GPU path cannot pass its `-check` (DESIGN.md, symmetry).
static void dist_to_abi(uint64_t dst[2], Int* d, bool wild, Int* wildOffset) {
#ifdef USE_SYMMETRY
  (void)wild; (void)wildOffset;
  if (d->bits64[3] > 0x7FFFFFFFFFFFFFFFULL) {
    Int t; t.Set(d); t.ModNegK1order();                       // |d|
    dst[0] = ~t.bits64[0] + 1; dst[1] = ~t.bits64[1] + (dst[0] == 0 ? 1 : 0);
  } else { dst[0] = d->bits64[0]; dst[1] = d->bits64[1]; }
#else
  Int dOff; dOff.Set(d);
  if (wild) dOff.ModAddK1order(wildOffset);
  dst[0] = dOff.bits64[0]; dst[1] = dOff.bits64[1];
#endif
}
static void dist_from_abi(Int* d, const uint64_t src[2], bool wild, Int* wildOffset) {
  d->SetInt32(0);
#ifdef USE_SYMMETRY
  (void)wild; (void)wildOffset;
  if (src[1] >> 63) {
    uint64_t m0 = ~src[0] + 1, m1 = ~src[1] + (m0 == 0 ? 1 : 0);
    d->bits64[0] = m0; d->bits64[1] = m1;
    d->ModNegK1order();
  } else { d->bits64[0] = src[0]; d->bits64[1] = src[1]; }
#else
  d->bits64[0] = src[0]; d->bits64[1] = src[1];
  if (wild) d->ModSubK1order(wildOffset);
#endif
}

void GPUEngine::SetWildOffset(Int* offset) { wildOffset.Set(offset); }        // GPUEngine.cu:140-142

GPUEngine::GPUEngine(int nbThreadGroup, int nbThreadPerGroup, int gpuId, uint32_t maxFound) {   // GPUEngine.cu:144-253
  this->nbThreadPerGroup = nbThreadPerGroup;
  this->nbThread = nbThreadGroup * nbThreadPerGroup;
  this->maxFound = maxFound;
  this->outputSize = maxFound * ITEM_SIZE + 4;
  initialised = false; lostWarning = false;
  inputKangaroo = NULL; inputKangarooPinned = NULL; outputItem = NULL; outputItemPinned = NULL; jumpPinned = NULL;
  kangarooSize = 0; kangarooSizePinned = 0; jumpSize = NB_JUMP * 8 * 4; dpMask = 0;
  wildOffset.SetInt32(0);
  kgx_engine* e = kgx_create(gpuId, nbThreadGroup, nbThreadPerGroup, maxFound);
  if (!e) { printf("GPUEngine: %s\n", kgx_last_error(NULL)); return; }        // callers never check (Kangaroo.cpp:523-526)
  inputKangaroo = reinterpret_cast<uint64_t*>(e);
#ifdef USE_SYMMETRY
  // Which of the reference's two symmetric jump rules the engine runs (include/kgx.h): the one its working path uses
  // (SolveKeyCPU: symClass) unless KGX_SYM_RULE=lastjump asks for the device/Check.cpp rule -- `-check` needs the latter.
  int symRule = KGX_SYM_CLASS;
  if (const char* r = getenv("KGX_SYM_RULE")) {
    if (!strcmp(r, "lastjump")) symRule = KGX_SYM_LASTJUMP;
    else if (strcmp(r, "symclass")) printf("GPUEngine: KGX_SYM_RULE must be lastjump or symclass (using symclass)\n");
  }
  if (kgx_set_symmetry(e, symRule) != 0) { printf("GPUEngine: %s\n", kgx_last_error(e)); kgx_destroy(e); inputKangaroo = NULL; return; }
#endif
  outputItemPinned = reinterpret_cast<uint32_t*>(new kgx_item[maxFound]);
  kangarooSize = (uint32_t)kgx_memory_bytes(e);
  char info[256] = "", name[200] = "?"; int sms = 0;
  if (kgx_device_info(gpuId, info, sizeof info) == 0) { char* bar = strchr(info, '|'); if (bar) { *bar = 0; sms = atoi(bar + 1); } strncpy(name, info, sizeof name - 1); }
  char tmp[512];
  snprintf(tmp, sizeof tmp, "GPU #%d %s (%dx%d cores) Grid(%dx%d)", gpuId, name, sms, 128, nbThreadGroup, nbThreadPerGroup);
  deviceName = std::string(tmp);
  initialised = true;
}

GPUEngine::~GPUEngine() {
  if (inputKangaroo) kgx_destroy(KGX(inputKangaroo));
  if (outputItemPinned) delete[] reinterpret_cast<kgx_item*>(outputItemPinned);
}

int GPUEngine::GetMemory() { return (int)(inputKangaroo ? kgx_memory_bytes(KGX(inputKangaroo)) : 0); }   // int, as the reference (overflows > 2 GB)
int GPUEngine::GetGroupSize() { return GPU_GRP_SIZE; }
int GPUEngine::GetNbThread() { return nbThread; }

bool GPUEngine::GetGridSize(int gpuId, int* x, int* y) {                       // GPUEngine.cu:275-309
  if (*x <= 0 || *y <= 0) {
    if (kgx_device_count() == 0) { printf("GPUEngine: There are no available device(s) that support CUDA\n"); return false; }
    if (kgx_grid_default(gpuId, x, y) != 0) { printf("GPUEngine::GetGridSize() Invalid gpuId\n"); return false; }
  }
  return true;
}

void* GPUEngine::AllocatePinnedMemory(size_t size) { return malloc(size); }    // unused by every caller (SURVEY 8b)
void GPUEngine::FreePinnedMemory(void* buff) { free(buff); }

void GPUEngine::PrintCudaInfo() {                                              // GPUEngine.cu:331-375 (-l)
  int n = kgx_device_count();
  if (n == 0) { printf("GPUEngine: There are no available device(s) that support CUDA\n"); return; }
  for (int i = 0; i < n; i++) {
    char info[256];
    if (kgx_device_info(i, info, sizeof info) != 0) continue;
    char name[200]; int sms, maj, min; double mb;
    char* p = strchr(info, '|'); *p = 0; strncpy(name, info, sizeof name - 1); name[sizeof name - 1] = 0;
    sscanf(p + 1, "%d|%d|%d|%lf", &sms, &maj, &min, &mb);
    printf("GPU #%d %s (%dx%d cores) (Cap %d.%d) (%.1f MB) (%s)\n", i, name, sms, 128, maj, min, mb, "Multiple host threads");
  }
}

void GPUEngine::SetParams(uint64_t dpMask, Int* distance, Int* px, Int* py) {  // GPUEngine.cu:559-590
  this->dpMask = dpMask;
  if (!inputKangaroo) return;
  uint64_t jd[NB_JUMP * 2], jx[NB_JUMP * 4], jy[NB_JUMP * 4];
  for (int i = 0; i < NB_JUMP; i++) { int_to_limbs(jd + 2 * i, &distance[i], 2); int_to_limbs(jx + 4 * i, &px[i], 4); int_to_limbs(jy + 4 * i, &py[i], 4); }
  if (kgx_set_params(KGX(inputKangaroo), dpMask, jd, jx, jy) != 0) printf("GPUEngine: SetParams: %s\n", kgx_last_error(KGX(inputKangaroo)));
}

// Int <-> limb marshalling of a whole herd (4.3 M kangaroos x 3 Int on the default H100 grid) on several host threads: the
// checkpoint path (Kangaroo.cpp:618-626) parks the GPU thread on GetKangaroos, so its duration is GPU idle time.
template <typename F>
static void parallel_for(uint64_t n, F body) {
  unsigned nt = std::thread::hardware_concurrency();
  nt = nt == 0 ? 1 : (nt > 16 ? 16 : nt);
  if (n < 65536) nt = 1;
  std::vector<std::thread> th;
  const uint64_t chunk = (n + nt - 1) / nt;
  for (unsigned t = 1; t < nt; t++) th.emplace_back([=] { const uint64_t a = t * chunk, b = a + chunk < n ? a + chunk : n; for (uint64_t i = a; i < b; i++) body(i); });
  for (uint64_t i = 0; i < (chunk < n ? chunk : n); i++) body(i);
  for (auto& x : th) x.join();
}

void GPUEngine::SetKangaroos(Int* px, Int* py, Int* d) {                        // GPUEngine.cu:381-433
  if (!inputKangaroo) return;
  const uint64_t n = kgx_num_kangaroos(KGX(inputKangaroo));
  std::unique_ptr<uint64_t[]> ax(new uint64_t[n * 4]), ay(new uint64_t[n * 4]), ad(new uint64_t[n * 2]);
  Int* wo = &wildOffset;
  uint64_t *bx = ax.get(), *by = ay.get(), *bd = ad.get();
  parallel_for(n, [=](uint64_t i) {
    int_to_limbs(bx + 4 * i, &px[i], 4); int_to_limbs(by + 4 * i, &py[i], 4);
    dist_to_abi(bd + 2 * i, &d[i], i % 2 == WILD, wo);
  });
  if (kgx_upload(KGX(inputKangaroo), bx, by, bd) != 0) printf("GPUEngine: SetKangaroos: %s\n", kgx_last_error(KGX(inputKangaroo)));
}

void GPUEngine::GetKangaroos(Int* px, Int* py, Int* d) {                        // GPUEngine.cu:435-491
  if (!inputKangaroo) { printf("GPUEngine: GetKangaroos: Cannot retreive kangaroos, mem has been freed\n"); return; }
  const uint64_t n = kgx_num_kangaroos(KGX(inputKangaroo));
  std::unique_ptr<uint64_t[]> ax(new uint64_t[n * 4]), ay(new uint64_t[n * 4]), ad(new uint64_t[n * 2]);
  uint64_t *bx = ax.get(), *by = ay.get(), *bd = ad.get();
  if (kgx_download(KGX(inputKangaroo), bx, by, bd) != 0) { printf("GPUEngine: GetKangaroos: %s\n", kgx_last_error(KGX(inputKangaroo))); return; }
  Int* wo = &wildOffset;
  parallel_for(n, [=](uint64_t i) {
    for (int k = 0; k < 4; k++) { px[i].bits64[k] = bx[4 * i + k]; py[i].bits64[k] = by[4 * i + k]; }
    px[i].bits64[4] = 0; py[i].bits64[4] = 0;
    dist_from_abi(&d[i], bd + 2 * i, i % 2 == WILD, wo);
  });
}

void GPUEngine::SetKangaroo(uint64_t kIdx, Int* px, Int* py, Int* d) {          // GPUEngine.cu:493-538
  if (!inputKangaroo) return;
  uint64_t x[4], y[4], dd[2];
  int_to_limbs(x, px, 4); int_to_limbs(y, py, 4);
  dist_to_abi(dd, d, kIdx % 2 == WILD, &wildOffset);
  if (kgx_patch(KGX(inputKangaroo), kIdx, x, y, dd) != 0) printf("GPUEngine: SetKangaroo: %s\n", kgx_last_error(KGX(inputKangaroo)));
}

// The reference prints a CUDA error on every failing call (GPUEngine.cu:549-553); its callers ignore the result and
// keep looping (Kangaroo.cpp:572-575), so an engine that could not be created must at least say so -- once.
static bool no_engine(const char* where) {
  static bool said = false;
  if (!said) { printf("GPUEngine: %s: engine not initialised (%s)\n", where, kgx_last_error(NULL)); said = true; }
  return false;
}

bool GPUEngine::callKernel() {                                                  // GPUEngine.cu:540-557
  if (!inputKangaroo) return no_engine("Kernel");
  if (kgx_launch_async(KGX(inputKangaroo)) != 0) { printf("GPUEngine: Kernel: %s\n", kgx_last_error(KGX(inputKangaroo))); return false; }
  return true;
}

bool GPUEngine::callKernelAndWait() {                                           // GPUEngine.cu:592-605
  bool ok = callKernel();
  if (inputKangaroo && kgx_sync(KGX(inputKangaroo)) != 0) { printf("GPUEngine: callKernelAndWait: %s\n", kgx_last_error(KGX(inputKangaroo))); return false; }
  return ok;
}

bool GPUEngine::Launch(std::vector<ITEM>& hashFound, bool spinWait) {            // GPUEngine.cu:607-679
  hashFound.clear();
  if (!inputKangaroo) return no_engine("Launch");
  kgx_item* items = reinterpret_cast<kgx_item*>(outputItemPinned);
  uint32_t nItems = 0, nFound = 0;
  // waits for the launch in flight, starts the next one, then reads the finished slab back (double buffered)
  if (kgx_collect(KGX(inputKangaroo), items, maxFound, &nItems, &nFound, spinWait ? 1 : 0, 1) != 0) {
    printf("GPUEngine: Launch: %s\n", kgx_last_error(KGX(inputKangaroo)));
    return false;
  }
  if (nFound > maxFound && !lostWarning) {
    printf("\nWarning, %d items lost\nHint: Search with less threads (-g) or increse dp (-d)\n", (nFound - maxFound));
    lostWarning = true;
  }
  hashFound.reserve(nItems);
  for (uint32_t i = 0; i < nItems; i++) {
    ITEM it;
    it.kIdx = items[i].kidx;
    for (int k = 0; k < 4; k++) it.x.bits64[k] = items[i].x[k];
    it.x.bits64[4] = 0;
    dist_from_abi(&it.d, items[i].d, it.kIdx % 2 == WILD, &wildOffset);
    hashFound.push_back(it);
  }
  return true;
}
