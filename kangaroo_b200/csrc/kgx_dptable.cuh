// kgx_dptable.cuh -- the rank-0 distinguished-point table in the memory of one GPU (C ABI: include/kgx.h, kgx_dptable_*).
//
// Semantics: exactly those of the reference's HashTable::Add driven record by record in arrival order (HashTable.cpp:262-307)
// with kgx_ingest.cpp's event mapping (kgx_ingest.cpp:68-83): 2^18 buckets h = x.bits64[2] & 0x3FFFF, one ENTRY {x, d} per
// distinct x of a bucket, per-bucket nbItem / maxItem counted like the reference (maxItem 16 on the first Add of a bucket, +4
// on every later Add -- stored or not -- that finds nbItem >= maxItem - 1), and work files that are byte for byte what
// HashTable::SaveTable writes (buckets in order, entries sorted by unsigned (x.hi, x.lo)).  The file format is
// kgx_workfile.h's; a save orders each chunk of whole buckets with kgx_bucketsort.cuh's sort.
// A table may hold a range of buckets only (kgx_dptable_create_range): one shard of the sharded table, which saves and loads
// its range as a piece of a work file at an offset.
//
// Layout (fixed capacity C entries, no growth):
//   ent[C]      32-byte entries {x, d}, dense in insertion order; ent_h[C] their bucket
//   slots[N]    open-addressing index over (h, x), N = C + C/2 (load <= 2/3), linear probing: 64-bit word
//               (entry index << 32) | tag, tag = (h + 1) | 13 bits of x.hi << 19, 0 = empty
//   nb/mx[2^18] the reference's nbItem / maxItem
// 48 bytes per entry of capacity, plus 2 MB of bucket counters and the save scratch (SAVE_CHUNK entries, 56 bytes each,
// and the save's selection of SAVE_SELECT entries, 4 bytes each, with its 2^18 bucket cursors).
// With KGX_DPT_HOST_ENTRIES (kgx_dptable_create_ex), ent[C] is mapped, pinned host memory that the kernels reach through its
// device pointer, and the GPU holds 16 bytes per entry.  An add touches an entry only to write a new one and to read one
// back when a probe meets a slot of the same tag; probes, tags and counters stay on the device.
//
// A save goes through the table in passes.  Each pass takes whole save chunks of consecutive buckets, at most SAVE_SELECT
// entries in all, and groups their entries by bucket in one scan of ent_h: the bucket counts are nbItem, their prefix sums
// (on the host) start one cursor per bucket, and each entry of the pass's buckets takes the next place of its bucket.  Each
// chunk's entries are then a contiguous run of the selection, sorted and gathered on their own (kgx_bucketsort.cuh).  Four
// chunks always fit a pass and two neighbouring chunks hold more than SAVE_CHUNK entries, so a save reads ent_h at most
// count / 2^22 + 1 times, about count / SAVE_SELECT when buckets are small against a chunk.
//
// One add call, stream-ordered on the caller's stream:
//   1. key  = h of every record (2^18 for a malformed one), value = arrival index (rank segments in order, then records)
//   2. stable radix sort by key: the records of one bucket together, in arrival order
//   3. one thread per bucket present walks its records in order: the reference's sequence of Add calls on that bucket, with
//      the (h, x) index in place of its binary search.  Buckets never share an entry, so threads of different buckets only
//      meet in the index, where an insert claims an empty slot with a CAS after its entry is written.
//   4. the events, written at their arrival index, are compacted in arrival order; the first `cap` go back to the host.
//      kgx_dptable_add_resolve runs a resolver (kgx_resolver.cuh) over those `cap` on the same stream first, so that each
//      collision goes back with its key and private key in the same copy.
#include <cub/cub.cuh>
#include "kgx_workfile.h"
#include "kgx_bucketsort.cuh"

namespace kgx_dpt {

using kgx_wf::Entry;
using kgx_wf::NBUCKET;
typedef unsigned long long ull;
constexpr uint64_t TYPE_BIT = 0x4000000000000000ull;    // b126 of the tagged distance: herd type (HashTable::CalcDistAndType)
constexpr uint64_t SAVE_CHUNK = 1ull << 21;             // entries per device->host chunk of a save / host->device chunk of a load
constexpr uint64_t SAVE_SELECT = 1ull << 23;            // entries one select pass of a save groups (32 MB of indices)

struct Res { ull count; uint32_t nsel; uint32_t bad; };
struct Ranks { uint32_t n; uint32_t pre[KGX_DPT_MAX_RANKS + 1]; };

__device__ __forceinline__ uint32_t rank_of(const Ranks& R, uint32_t i) {
  uint32_t lo = 0, hi = R.n - 1;                        // the last rank whose segment starts at or before i
  while (lo < hi) {
    const uint32_t m = (lo + hi + 1) >> 1;
    if (R.pre[m] <= i) lo = m; else hi = m - 1;
  }
  return lo;
}

__device__ __forceinline__ const uint64_t* record(const uint8_t* recs, uint64_t stride, const Ranks& R, uint32_t i, uint32_t r) {
  return reinterpret_cast<const uint64_t*>(recs + ((uint64_t)r * stride + (i - R.pre[r])) * 40ull);
}

__host__ __device__ __forceinline__ uint32_t slot_tag(uint32_t h, uint64_t x1) { return (h + 1) | ((uint32_t)(x1 >> 51) << 19); }

__device__ __forceinline__ uint64_t slot_home(uint32_t h, uint64_t x0, uint64_t x1, uint64_t nslots) {
  uint64_t k = (x0 ^ (x1 * 0x9E3779B97F4A7C15ull) ^ ((uint64_t)h << 40)) * 0xD6E8FEB86659FD93ull;
  k ^= k >> 32;
  return __umul64hi(k, nslots);
}

__device__ __forceinline__ void index_insert(ull* slots, uint64_t nslots, uint64_t home, ull word) {
  uint64_t p = home;
  while (atomicCAS(&slots[p], 0ull, word) != 0ull)
    if (++p == nslots) p = 0;
}

__global__ void k_keys(const uint8_t* recs, uint64_t stride, Ranks R, uint32_t n, uint32_t lo, uint32_t hi, uint32_t* keys,
                       uint32_t* vals, uint8_t* evFlag, Res* res) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t h = (uint32_t)(record(recs, stride, R, i, rank_of(R, i))[0] >> 32);
  const bool in = h >= lo && h < hi;                    // [lo, hi): the table's buckets, all 2^18 but in a shard
  keys[i] = in ? h : NBUCKET;
  vals[i] = i;
  evFlag[i] = 0;
  if (!in) res->bad = 1;                                // skipped, like kgx_ingest.cpp's workers; the call returns -1
}

// one thread per bucket present in the call: HashTable::Add(h, x, d) for each of its records in arrival order
__global__ void k_insert(const uint32_t* keys, const uint32_t* vals, uint32_t n, const uint8_t* recs, uint64_t stride, Ranks R,
                         Entry* ent, uint32_t* ent_h, ull* slots, uint64_t nslots, uint32_t* nb, uint32_t* mx, Res* res,
                         kgx_dp_event* evArr, uint8_t* evFlag) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint32_t h = keys[j];
  if (h >= NBUCKET || (j > 0 && keys[j - 1] == h)) return;
  uint32_t nbv = nb[h], mxv = mx[h];
  for (uint32_t k = j; k < n && keys[k] == h; k++) {
    const uint32_t i = vals[k], r = rank_of(R, i);
    const uint64_t* rec = record(recs, stride, R, i, r);
    const uint64_t w0 = rec[0], x0 = rec[1], x1 = rec[2], d0 = rec[3], d1 = rec[4];
    const uint32_t tag = slot_tag(h, x1);
    const uint64_t home = slot_home(h, x0, x1, nslots);
    if (mxv == 0) mxv = 16;                             // HashTable.cpp:264-267
    if (nbv != 0) {
      if (nbv >= mxv - 1) mxv += 4;                     // HashTable.cpp:275-278: before the search, whatever it finds
      uint64_t p = home;
      for (;;) {
        const ull s = *reinterpret_cast<volatile ull*>(&slots[p]);
        if (s == 0) break;
        if ((uint32_t)s == tag) {
          const Entry* e = ent + (s >> 32);
          if (__ldcg(&e->x0) == x0 && __ldcg(&e->x1) == x1) {
            const uint64_t o0 = __ldcg(&e->d0), o1 = __ldcg(&e->d1);
            kgx_dp_event ev;
            ev.rank = r; ev.kidx = (uint32_t)w0; ev.h = h;
            ev.d_new[0] = d0; ev.d_new[1] = d1;
            if (o0 == d0 && o1 == d1) {                 // ADD_DUPLICATE
              ev.kind = KGX_DPT_EV_RESET; ev.d_old[0] = 0; ev.d_old[1] = 0;
            } else {                                    // ADD_COLLISION: same herd -> reset (Kangaroo.cpp:258-262)
              ev.kind = ((o1 ^ d1) & TYPE_BIT) ? KGX_DPT_EV_COLLISION : KGX_DPT_EV_RESET;
              ev.d_old[0] = o0; ev.d_old[1] = o1;
            }
            evArr[i] = ev;
            evFlag[i] = 1;
            goto next;
          }
        }
        if (++p == nslots) p = 0;
      }
    }
    {                                                   // ADD_OK: a new entry
      const ull e = atomicAdd(&res->count, 1ull);
      ent[e] = Entry{x0, x1, d0, d1};
      ent_h[e] = h;
      __threadfence();                                  // the entry before the slot that publishes it
      index_insert(slots, nslots, home, (e << 32) | tag);
      nbv++;
    }
  next:;
  }
  nb[h] = nbv; mx[h] = mxv;
}

__global__ void k_events_out(const kgx_dp_event* evArr, const uint32_t* sel, const Res* res, uint32_t cap, kgx_dp_event* out) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < cap && t < res->nsel) out[t] = evArr[sel[t]];
}

// a load: entries [first, first + n) are already in ent / ent_h
__global__ void k_index_entries(const Entry* ent, const uint32_t* ent_h, uint64_t first, uint64_t n, ull* slots, uint64_t nslots) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const uint64_t e = first + t;
  const Entry v = ent[e];
  const uint32_t h = ent_h[e];
  index_insert(slots, nslots, slot_home(h, v.x0, v.x1, nslots), ((ull)e << 32) | slot_tag(h, v.x1));
}

// a save's select pass: the entries of buckets [b0, b1) grouped by bucket, cursor[h] the next place of bucket h in sel
__global__ void k_save_select(const uint32_t* ent_h, uint64_t count, uint32_t b0, uint32_t b1, uint32_t* cursor, uint32_t* sel) {
  const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= count) return;
  const uint32_t h = ent_h[e];
  if (h >= b0 && h < b1) sel[atomicAdd(&cursor[h], 1u)] = (uint32_t)e;
}

inline uint64_t slots_for(uint64_t capacity) { return capacity + capacity / 2 + 64; }
inline uint64_t save_chunk_for(uint64_t capacity) { return capacity < SAVE_CHUNK ? (capacity ? capacity : 1) : SAVE_CHUNK; }
inline uint64_t save_select_for(uint64_t capacity) { return capacity < SAVE_SELECT ? (capacity ? capacity : 1) : SAVE_SELECT; }

}  // namespace kgx_dpt

static char g_dpt_create_err[256] = "";

struct kgx_dptable {
  int dev = 0;
  uint32_t lo = 0, hi = kgx_dpt::NBUCKET;                 // the buckets the table holds (a shard of the sharded table: a range)
  uint64_t capacity = 0, nslots = 0, count = 0;           // count: host mirror of res->count after the last call
  int flags = 0;
  kgx_dpt::Entry* ent = nullptr;                           // as the kernels reach it: device memory, or entHost mapped
  kgx_dpt::Entry* entHost = nullptr;                       // KGX_DPT_HOST_ENTRIES: the pinned entries (else null)
  uint64_t hostBytes = 0;
  uint32_t* ent_h = nullptr;
  kgx_dpt::ull* slots = nullptr;
  uint32_t *nb = nullptr, *mx = nullptr;
  kgx_dpt::Res* res = nullptr;                             // device
  kgx_dpt::Res* resHost = nullptr;                         // pinned
  // add scratch, grown to the largest call so far
  uint32_t scratchN = 0, evCap = 0;
  uint32_t *keyIn = nullptr, *keyOut = nullptr, *valIn = nullptr, *valOut = nullptr, *sel = nullptr;
  kgx_dp_event *evArr = nullptr, *evOut = nullptr;
  kgx_dp_event_key* evKey = nullptr;                       // kgx_dptable_add_resolve's events, evCap of them
  uint8_t* evFlag = nullptr;
  void* cubTmp = nullptr;
  size_t cubTmpBytes = 0;
  uint64_t scratchBytes = 0;
  // save / load scratch: chunk entries on the device, pinned on the host; the select pass's selection and bucket cursors
  uint64_t chunk = 0, select = 0;
  uint32_t *sIdxA = nullptr, *sIdxB = nullptr, *sSel = nullptr, *sCursor = nullptr;
  uint64_t *sKeyA = nullptr, *sKeyB = nullptr;
  kgx_dpt::Entry* sOut = nullptr;
  void* sTmp = nullptr;
  size_t sTmpBytes = 0;
  kgx_dpt::Entry* hostEnt = nullptr;                       // pinned, chunk entries (allocated by the first save or load)
  uint32_t* hostH = nullptr;
  uint64_t bytes = 0;
  char err[256] = "";
};

#define DPT_CK(t, call)                                                                        \
  do {                                                                                         \
    cudaError_t _s = (call);                                                                   \
    if (_s != cudaSuccess) {                                                                   \
      snprintf((t)->err, sizeof((t)->err), "%s: %s", #call, cudaGetErrorString(_s));           \
      return -3;                                                                               \
    }                                                                                          \
  } while (0)

static int dpt_alloc(kgx_dptable* t, void** p, size_t n) {
  cudaError_t s = cudaMalloc(p, n ? n : 1);
  if (s != cudaSuccess) {
    snprintf(t->err, sizeof t->err, "cudaMalloc(%zu bytes): %s", n, cudaGetErrorString(s));
    cudaGetLastError();
    *p = nullptr;
    return -3;
  }
  t->bytes += n;
  return 0;
}

static void dpt_free_scratch(kgx_dptable* t) {
  cudaFree(t->keyIn); cudaFree(t->keyOut); cudaFree(t->valIn); cudaFree(t->valOut); cudaFree(t->sel);
  cudaFree(t->evArr); cudaFree(t->evFlag); cudaFree(t->cubTmp);
  t->keyIn = t->keyOut = t->valIn = t->valOut = t->sel = nullptr;
  t->evArr = nullptr; t->evFlag = nullptr; t->cubTmp = nullptr;
  t->bytes -= t->scratchBytes;
  t->scratchN = 0; t->cubTmpBytes = 0; t->scratchBytes = 0;
}

// grow-only per-call scratch for n records (rounded up to a power of two).  Every add ends with a synchronisation of its
// stream, so no earlier call still reads the scratch freed here.
static int dpt_scratch(kgx_dptable* t, uint32_t n) {
  if (n <= t->scratchN) return 0;
  dpt_free_scratch(t);
  const uint64_t before = t->bytes;
  uint32_t m = 1024;
  while (m < n) m <<= 1;
  size_t a = 0, b = 0;
  DPT_CK(t, cub::DeviceRadixSort::SortPairs(nullptr, a, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)m, 0, 19));
  DPT_CK(t, cub::DeviceSelect::Flagged(nullptr, b, (uint32_t*)nullptr, (uint8_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)m));
  const size_t tmp = a > b ? a : b;
  if (dpt_alloc(t, (void**)&t->keyIn, 4ull * m) || dpt_alloc(t, (void**)&t->keyOut, 4ull * m) || dpt_alloc(t, (void**)&t->valIn, 4ull * m) ||
      dpt_alloc(t, (void**)&t->valOut, 4ull * m) || dpt_alloc(t, (void**)&t->sel, 4ull * m) ||
      dpt_alloc(t, (void**)&t->evArr, sizeof(kgx_dp_event) * (size_t)m) || dpt_alloc(t, (void**)&t->evFlag, m) ||
      dpt_alloc(t, &t->cubTmp, tmp)) {
    t->scratchBytes = t->bytes - before;
    dpt_free_scratch(t);
    return -3;
  }
  t->scratchN = m; t->cubTmpBytes = tmp; t->scratchBytes = t->bytes - before;
  return 0;
}

static int dpt_reset(kgx_dptable* t, cudaStream_t st) {
  DPT_CK(t, cudaMemsetAsync(t->slots, 0, 8ull * t->nslots, st));
  DPT_CK(t, cudaMemsetAsync(t->nb, 0, 4ull * kgx_dpt::NBUCKET, st));
  DPT_CK(t, cudaMemsetAsync(t->mx, 0, 4ull * kgx_dpt::NBUCKET, st));
  DPT_CK(t, cudaMemsetAsync(t->res, 0, sizeof(kgx_dpt::Res), st));
  DPT_CK(t, cudaStreamSynchronize(st));
  t->count = 0;
  return 0;
}

static int dpt_pinned(kgx_dptable* t) {
  if (t->hostEnt) return 0;
  DPT_CK(t, cudaHostAlloc((void**)&t->hostEnt, sizeof(kgx_dpt::Entry) * t->chunk, cudaHostAllocDefault));
  DPT_CK(t, cudaHostAlloc((void**)&t->hostH, 4ull * t->chunk, cudaHostAllocDefault));
  return 0;
}

extern "C" {

uint64_t kgx_dptable_bytes_for_ex(uint64_t capacity, int flags, uint64_t* host_bytes) {
  const uint64_t c = kgx_dpt::save_chunk_for(capacity), ent = sizeof(kgx_dpt::Entry) * capacity;
  const bool host = flags & KGX_DPT_HOST_ENTRIES;
  if (host_bytes) *host_bytes = host ? ent : 0;
  return (host ? 0 : ent) + 4 * capacity + 8 * kgx_dpt::slots_for(capacity) + 8ull * kgx_dpt::NBUCKET +
         4 * kgx_dpt::save_select_for(capacity) + 4ull * kgx_dpt::NBUCKET +
         c * (4 + 4 + 8 + 8 + sizeof(kgx_dpt::Entry)) + 2 * 8 * c + (64ull << 20);   // the last two: radix-sort scratch, estimated
}

uint64_t kgx_dptable_bytes_for(uint64_t capacity) { return kgx_dptable_bytes_for_ex(capacity, 0, nullptr); }

const char* kgx_dptable_last_error(kgx_dptable* t) { return t ? t->err : g_dpt_create_err; }

void kgx_dptable_destroy(kgx_dptable* t) {
  if (!t) return;
  cudaSetDevice(t->dev);
  cudaDeviceSynchronize();
  if (t->entHost) cudaFreeHost(t->entHost);
  else cudaFree(t->ent);
  cudaFree(t->ent_h); cudaFree(t->slots); cudaFree(t->nb); cudaFree(t->mx); cudaFree(t->res);
  dpt_free_scratch(t);
  cudaFree(t->evOut); cudaFree(t->evKey);
  cudaFree(t->sIdxA); cudaFree(t->sIdxB); cudaFree(t->sSel); cudaFree(t->sCursor); cudaFree(t->sKeyA); cudaFree(t->sKeyB); cudaFree(t->sOut); cudaFree(t->sTmp);
  if (t->resHost) cudaFreeHost(t->resHost);
  if (t->hostEnt) cudaFreeHost(t->hostEnt);
  if (t->hostH) cudaFreeHost(t->hostH);
  delete t;
}

// the pinned entries of a KGX_DPT_HOST_ENTRIES table, mapped into the device's address space
static int dpt_alloc_host_entries(kgx_dptable* t) {
  const size_t n = sizeof(kgx_dpt::Entry) * t->capacity;
  cudaError_t s = cudaHostAlloc((void**)&t->entHost, n, cudaHostAllocMapped);
  if (s == cudaSuccess) s = cudaHostGetDevicePointer((void**)&t->ent, t->entHost, 0);
  if (s != cudaSuccess) {
    snprintf(t->err, sizeof t->err, "cudaHostAlloc(%zu bytes, mapped): %s", n, cudaGetErrorString(s));
    cudaGetLastError();
    return -3;
  }
  t->hostBytes = n;
  return 0;
}

kgx_dptable* kgx_dptable_create_ex(int dev, uint64_t capacity, uint32_t lo, uint32_t hi, int flags) {
  if (lo >= hi || hi > kgx_dpt::NBUCKET) {
    snprintf(g_dpt_create_err, sizeof g_dpt_create_err, "kgx_dptable_create_range: buckets [%u, %u) are not a range of [0, 2^18)", lo, hi);
    return nullptr;
  }
  if (flags & ~KGX_DPT_HOST_ENTRIES) {
    snprintf(g_dpt_create_err, sizeof g_dpt_create_err, "kgx_dptable_create_ex: unknown flags 0x%x", flags);
    return nullptr;
  }
  int cnt = 0;
  cudaError_t s = cudaGetDeviceCount(&cnt);
  if (s != cudaSuccess || cnt == 0) {
    snprintf(g_dpt_create_err, sizeof g_dpt_create_err, "kgx_dptable_create: no CUDA device (%s)", cudaGetErrorString(s));
    cudaGetLastError();
    return nullptr;
  }
  if (capacity == 0 || capacity >= 0xFFFFFFFFull) {
    snprintf(g_dpt_create_err, sizeof g_dpt_create_err, "kgx_dptable_create: capacity %llu is not in 1 .. 2^32-2 entries",
             (unsigned long long)capacity);
    return nullptr;
  }
  if ((s = cudaSetDevice(dev)) != cudaSuccess) {
    snprintf(g_dpt_create_err, sizeof g_dpt_create_err, "kgx_dptable_create: cudaSetDevice(%d): %s", dev, cudaGetErrorString(s));
    cudaGetLastError();
    return nullptr;
  }
  kgx_dptable* t = new kgx_dptable();
  t->dev = dev; t->lo = lo; t->hi = hi; t->flags = flags;
  t->capacity = capacity; t->nslots = kgx_dpt::slots_for(capacity);
  t->chunk = kgx_dpt::save_chunk_for(capacity);
  t->select = kgx_dpt::save_select_for(capacity);
  const uint64_t c = t->chunk;
  t->sTmpBytes = kgx_wf::bucket_sort_scratch(c);
  bool ok = (flags & KGX_DPT_HOST_ENTRIES) ? !dpt_alloc_host_entries(t) : !dpt_alloc(t, (void**)&t->ent, sizeof(kgx_dpt::Entry) * capacity);
  ok = ok && !dpt_alloc(t, (void**)&t->ent_h, 4ull * capacity) &&
       !dpt_alloc(t, (void**)&t->slots, 8ull * t->nslots) && !dpt_alloc(t, (void**)&t->nb, 4ull * kgx_dpt::NBUCKET) &&
       !dpt_alloc(t, (void**)&t->mx, 4ull * kgx_dpt::NBUCKET) && !dpt_alloc(t, (void**)&t->res, sizeof(kgx_dpt::Res)) &&
       !dpt_alloc(t, (void**)&t->sIdxA, 4ull * c) && !dpt_alloc(t, (void**)&t->sIdxB, 4ull * c) &&
       !dpt_alloc(t, (void**)&t->sSel, 4ull * t->select) && !dpt_alloc(t, (void**)&t->sCursor, 4ull * kgx_dpt::NBUCKET) &&
       !dpt_alloc(t, (void**)&t->sKeyA, 8ull * c) &&
       !dpt_alloc(t, (void**)&t->sKeyB, 8ull * c) && !dpt_alloc(t, (void**)&t->sOut, sizeof(kgx_dpt::Entry) * c) &&
       !dpt_alloc(t, &t->sTmp, t->sTmpBytes);
  if (ok && cudaHostAlloc((void**)&t->resHost, sizeof(kgx_dpt::Res), cudaHostAllocDefault) != cudaSuccess) {
    snprintf(t->err, sizeof t->err, "cudaHostAlloc failed");
    ok = false;
  }
  if (ok) ok = dpt_reset(t, 0) == 0;
  if (!ok) {
    uint64_t hb = 0;
    const uint64_t db = kgx_dptable_bytes_for_ex(capacity, flags, &hb);
    if (hb)
      snprintf(g_dpt_create_err, sizeof g_dpt_create_err, "kgx_dptable_create(%llu entries, %.2f GB + %.2f GB pinned host): %.160s",
               (unsigned long long)capacity, db / 1e9, hb / 1e9, t->err);
    else
      snprintf(g_dpt_create_err, sizeof g_dpt_create_err, "kgx_dptable_create(%llu entries, %.2f GB): %.180s",
               (unsigned long long)capacity, db / 1e9, t->err);
    cudaGetLastError();
    kgx_dptable_destroy(t);
    return nullptr;
  }
  return t;
}

kgx_dptable* kgx_dptable_create_range(int dev, uint64_t capacity, uint32_t lo, uint32_t hi) {
  return kgx_dptable_create_ex(dev, capacity, lo, hi, 0);
}

kgx_dptable* kgx_dptable_create(int dev, uint64_t capacity) { return kgx_dptable_create_ex(dev, capacity, 0, kgx_dpt::NBUCKET, 0); }

uint64_t kgx_dptable_count(kgx_dptable* t) { return t->count; }
uint64_t kgx_dptable_capacity(kgx_dptable* t) { return t->capacity; }
uint64_t kgx_dptable_host_bytes(kgx_dptable* t) { return t->hostBytes; }
uint64_t kgx_dptable_memory_bytes(kgx_dptable* t) {
  return t->bytes + (t->evOut ? (sizeof(kgx_dp_event) + sizeof(kgx_dp_event_key)) * (uint64_t)t->evCap : 0);
}

// the first `cap` events of an add on the device, plain and with their keys (grow-only; every add ends with a
// synchronisation of its stream, so no earlier call still writes the buffers freed here)
static int dpt_events(kgx_dptable* t, uint32_t cap) {
  if (cap <= t->evCap) return 0;
  cudaFree(t->evOut); cudaFree(t->evKey);
  t->evOut = nullptr; t->evKey = nullptr; t->evCap = 0;
  DPT_CK(t, cudaMalloc((void**)&t->evOut, sizeof(kgx_dp_event) * (size_t)cap));
  DPT_CK(t, cudaMalloc((void**)&t->evKey, sizeof(kgx_dp_event_key) * (size_t)cap));
  t->evCap = cap;
  return 0;
}

int kgx_dptable_reserve(kgx_dptable* t, uint32_t n_records, uint32_t cap) {
  DPT_CK(t, cudaSetDevice(t->dev));
  if (n_records >= 0x80000000u) {
    snprintf(t->err, sizeof t->err, "kgx_dptable_reserve: %u records (at most 2^31-1)", n_records);
    return -3;
  }
  if (n_records && dpt_scratch(t, n_records)) return -3;
  return dpt_events(t, cap);
}

// kgx_dptable_add (r null: ev holds kgx_dp_event) and kgx_dptable_add_resolve (ev holds kgx_dp_event_key)
static int dpt_add(kgx_dptable* t, const void* recs, const uint32_t* counts, uint32_t n_ranks, uint64_t stride, const kgx_resolver* r,
                   void* ev, uint32_t cap, uint32_t* n_ev, void* stream) {
  using namespace kgx_dpt;
  *n_ev = 0;
  if (r && r->dev != t->dev) {
    snprintf(t->err, sizeof t->err, "kgx_dptable_add_resolve: the resolver is on device %d, the table on device %d", r->dev, t->dev);
    return -3;
  }
  if (n_ranks == 0 || n_ranks > KGX_DPT_MAX_RANKS) {
    snprintf(t->err, sizeof t->err, "kgx_dptable_add: %u ranks (1 .. %d)", n_ranks, KGX_DPT_MAX_RANKS);
    return -3;
  }
  Ranks R;
  R.n = n_ranks;
  uint64_t n64 = 0;
  for (uint32_t r = 0; r < n_ranks; r++) {
    if (counts[r] > stride && n_ranks > 1) {
      snprintf(t->err, sizeof t->err, "kgx_dptable_add: rank %u has %u records, more than the stride %llu", r, counts[r], (unsigned long long)stride);
      return -3;
    }
    R.pre[r] = (uint32_t)n64;
    n64 += counts[r];
  }
  R.pre[n_ranks] = (uint32_t)n64;
  if (n64 >= 0x80000000ull) {
    snprintf(t->err, sizeof t->err, "kgx_dptable_add: %llu records in one call (at most 2^31-1)", (unsigned long long)n64);
    return -3;
  }
  if (t->count + n64 > t->capacity) {                      // checked before anything runs: a full table changes nothing
    snprintf(t->err, sizeof t->err, "DP table full: %llu entries + %llu records of this call > capacity %llu",
             (unsigned long long)t->count, (unsigned long long)n64, (unsigned long long)t->capacity);
    return -2;
  }
  const uint32_t n = (uint32_t)n64;
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  DPT_CK(t, cudaSetDevice(t->dev));
  if (dpt_scratch(t, n)) return -3;
  if (dpt_events(t, cap)) return -3;
  const uint8_t* rp = static_cast<const uint8_t*>(recs);
  DPT_CK(t, cudaMemsetAsync(&t->res->nsel, 0, 8, st));
  const uint32_t B = 256, G = (n + B - 1) / B;
  k_keys<<<G, B, 0, st>>>(rp, stride, R, n, t->lo, t->hi, t->keyIn, t->valIn, t->evFlag, t->res);
  DPT_CK(t, cudaGetLastError());
  size_t tb = t->cubTmpBytes;
  DPT_CK(t, cub::DeviceRadixSort::SortPairs(t->cubTmp, tb, t->keyIn, t->keyOut, t->valIn, t->valOut, (int)n, 0, 19, st));
  k_insert<<<G, B, 0, st>>>(t->keyOut, t->valOut, n, rp, stride, R, t->ent, t->ent_h, t->slots, t->nslots, t->nb, t->mx, t->res,
                            t->evArr, t->evFlag);
  DPT_CK(t, cudaGetLastError());
  tb = t->cubTmpBytes;
  DPT_CK(t, cub::DeviceSelect::Flagged(t->cubTmp, tb, t->valIn, t->evFlag, t->sel, &t->res->nsel, (int)n, st));
  const uint32_t nout = cap < n ? cap : n;
  if (nout) {
    k_events_out<<<(nout + B - 1) / B, B, 0, st>>>(t->evArr, t->sel, t->res, cap, t->evOut);
    DPT_CK(t, cudaGetLastError());
    if (r) DPT_CK(t, kgx_wt::resolve_events(r, t->evOut, &t->res->nsel, nout, t->evKey, st));
  }
  DPT_CK(t, cudaMemcpyAsync(t->resHost, t->res, sizeof(Res), cudaMemcpyDeviceToHost, st));
  DPT_CK(t, cudaStreamSynchronize(st));
  t->count = t->resHost->count;
  *n_ev = t->resHost->nsel;
  const uint32_t ncopy = *n_ev < cap ? *n_ev : cap;
  if (ncopy) {
    if (r) DPT_CK(t, cudaMemcpyAsync(ev, t->evKey, sizeof(kgx_dp_event_key) * (size_t)ncopy, cudaMemcpyDeviceToHost, st));
    else DPT_CK(t, cudaMemcpyAsync(ev, t->evOut, sizeof(kgx_dp_event) * (size_t)ncopy, cudaMemcpyDeviceToHost, st));
    DPT_CK(t, cudaStreamSynchronize(st));
  }
  return t->resHost->bad ? -1 : 0;
}

int kgx_dptable_add(kgx_dptable* t, const void* recs, const uint32_t* counts, uint32_t n_ranks, uint64_t stride, kgx_dp_event* ev,
                    uint32_t cap, uint32_t* n_ev, void* stream) {
  return dpt_add(t, recs, counts, n_ranks, stride, nullptr, ev, cap, n_ev, stream);
}

int kgx_dptable_add_resolve(kgx_dptable* t, const void* recs, const uint32_t* counts, uint32_t n_ranks, uint64_t stride, kgx_resolver* r,
                            kgx_dp_event_key* ev, uint32_t cap, uint32_t* n_ev, void* stream) {
  if (!r) {
    snprintf(t->err, sizeof t->err, "kgx_dptable_add_resolve: no resolver");
    return -3;
  }
  return dpt_add(t, recs, counts, n_ranks, stride, r, ev, cap, n_ev, stream);
}

// The buckets [b0, b1) of the table, each nbItem, maxItem and its entries (HashTable::SaveTable, HashTable.cpp:375-396), to f
// in chunks of whole buckets: a select pass groups the entries of several chunks by bucket, then each chunk is sorted by
// (h, x.hi, x.lo) and copied out.  -> 0, -3 on a CUDA error (text in t->err), or 1 when a write failed (errno tells).
static int dpt_write_buckets(kgx_dptable* t, FILE* f, uint32_t b0, uint32_t b1, cudaStream_t st) {
  using namespace kgx_dpt;
  using namespace kgx_wf;
  if (dpt_pinned(t)) return -3;
  uint32_t* nbH = (uint32_t*)malloc(12ull * NBUCKET);
  if (!nbH) { snprintf(t->err, sizeof t->err, "out of host memory"); return -3; }
  uint32_t* mxH = nbH + NBUCKET;
  uint32_t* curH = mxH + NBUCKET;                         // a pass's bucket cursors: where each bucket starts in the selection
  if (cudaMemcpy(nbH, t->nb, 4ull * NBUCKET, cudaMemcpyDeviceToHost) != cudaSuccess ||
      cudaMemcpy(mxH, t->mx, 4ull * NBUCKET, cudaMemcpyDeviceToHost) != cudaSuccess) {
    free(nbH);
    snprintf(t->err, sizeof t->err, "kgx_dptable_save_work: bucket counters: %s", cudaGetErrorString(cudaGetLastError()));
    return -3;
  }
  bool ok = true;
  int rc = 0;
  const uint32_t end = b1;
  uint32_t p0 = b0, p1 = b0;                              // the buckets of the current select pass
  while (ok && rc == 0 && b0 < end) {
    uint64_t m = 0;
    b1 = b0;
    while (b1 < end && (m + nbH[b1] <= t->chunk || b1 == b0)) m += nbH[b1++];
    if (m > t->chunk) {                                   // one bucket larger than a chunk
      snprintf(t->err, sizeof t->err, "kgx_dptable_save_work: bucket %u holds %llu entries, more than a save chunk (%llu)", b0,
               (unsigned long long)m, (unsigned long long)t->chunk);
      rc = -3;
      break;
    }
    if (m && b0 >= p1) {                                  // a new select pass: whole chunks from b0, at most t->select entries
      uint64_t sel = 0;
      p0 = p1 = b0;
      for (uint32_t c1 = b0; c1 < end && sel < t->select;) {
        uint64_t cm = 0;
        uint32_t c2 = c1;
        while (c2 < end && (cm + nbH[c2] <= t->chunk || c2 == c1)) cm += nbH[c2++];
        if (cm > t->chunk || sel + cm > t->select) break;
        sel += cm;
        c1 = p1 = c2;
      }
      uint32_t run = 0;
      for (uint32_t h = p0; h < p1; h++) { curH[h] = run; run += nbH[h]; }
      const uint32_t B = 256;
      bool good = cudaMemcpyAsync(t->sCursor + p0, curH + p0, 4ull * (p1 - p0), cudaMemcpyHostToDevice, st) == cudaSuccess;
      if (good) k_save_select<<<(unsigned)((t->count + B - 1) / B), B, 0, st>>>(t->ent_h, t->count, p0, p1, t->sCursor, t->sSel);
      if (!good || cudaGetLastError() != cudaSuccess) {
        snprintf(t->err, sizeof t->err, "kgx_dptable_save_work: %s", cudaGetErrorString(cudaGetLastError()));
        rc = -3;
        break;
      }
    }
    if (m) {
      const uint32_t n = (uint32_t)m, B = 256, G = (n + B - 1) / B;
      uint32_t* order = nullptr;
      bool good = bucket_sort(t->ent, t->ent_h, t->sSel + curH[b0], n, b0, b1, t->sIdxA, t->sIdxB, t->sKeyA, t->sKeyB, t->sTmp,
                              t->sTmpBytes, st, &order) == cudaSuccess;
      if (good) bucket_gather<<<G, B, 0, st>>>(t->ent, order, n, t->sOut);
      good = good && cudaMemcpyAsync(t->hostEnt, t->sOut, sizeof(Entry) * m, cudaMemcpyDeviceToHost, st) == cudaSuccess &&
             cudaStreamSynchronize(st) == cudaSuccess;
      if (!good) {
        snprintf(t->err, sizeof t->err, "kgx_dptable_save_work: %s", cudaGetErrorString(cudaGetLastError()));
        rc = -3;
        break;
      }
    }
    uint64_t off = 0;
    for (uint32_t b = b0; ok && b < b1; b++) {
      ok = write_bucket(f, nbH[b], mxH[b], t->hostEnt + off);
      off += nbH[b];
    }
    b0 = b1;
  }
  free(nbH);
  return rc ? rc : (ok ? 0 : 1);
}

int kgx_dptable_save_work(kgx_dptable* t, const char* path, uint32_t dp_bits, const uint64_t range_start[4], const uint64_t range_end[4],
                          const uint64_t keyx[4], const uint64_t keyy[4], uint64_t total_count, double total_time, uint64_t total_walk,
                          void* stream) {
  using namespace kgx_dpt;
  using namespace kgx_wf;
  cudaStream_t st = (cudaStream_t)stream;
  DPT_CK(t, cudaSetDevice(t->dev));
  DPT_CK(t, cudaStreamSynchronize(st));                    // every add queued on this stream is in the table
  if (dpt_pinned(t)) return -3;
  errno = 0;
  FILE* f = fopen(path, "wb");
  if (!f) { const int e = io_error(); snprintf(t->err, sizeof t->err, "%s: %s", path, strerror(-e)); return e; }
  setvbuf(f, nullptr, _IOFBF, 1 << 22);
  bool ok = write_header(f, make_header(dp_bits, range_start, range_end, keyx, keyy, total_count, total_time));
  int rc = ok ? dpt_write_buckets(t, f, 0, NBUCKET, st) : 0;   // every bucket: those out of a shard's range are empty
  if (rc == 1) { ok = false; rc = 0; }
  ok = ok && fwrite(&total_walk, 8, 1, f) == 1;           // Backup.cpp:530-531 / 549-551
  ok = fflush(f) == 0 && ok;
  int err = rc ? rc : (ok ? 0 : io_error());
  if (fclose(f) != 0 && err == 0) err = io_error();
  if (err < 0 && err != -3) snprintf(t->err, sizeof t->err, "%s: %s", path, strerror(-err));
  return err;
}

uint64_t kgx_dptable_piece_bytes(kgx_dptable* t) { return 8ull * (t->hi - t->lo) + sizeof(kgx_dpt::Entry) * t->count; }

int kgx_dptable_save_range(kgx_dptable* t, const char* path, uint64_t offset, void* stream) {
  using namespace kgx_wf;
  cudaStream_t st = (cudaStream_t)stream;
  DPT_CK(t, cudaSetDevice(t->dev));
  DPT_CK(t, cudaStreamSynchronize(st));
  errno = 0;
  FILE* f = fopen(path, "r+b");                           // the file exists: its header and the other pieces stay
  if (!f) { const int e = io_error(); snprintf(t->err, sizeof t->err, "%s: %s", path, strerror(-e)); return e; }
  setvbuf(f, nullptr, _IOFBF, 1 << 22);
  bool ok = fseeko(f, (off_t)offset, SEEK_SET) == 0;
  int rc = ok ? dpt_write_buckets(t, f, t->lo, t->hi, st) : 0;
  if (rc == 1) { ok = false; rc = 0; }
  ok = ok && fflush(f) == 0 && fsync(fileno(f)) == 0;
  int err = rc ? rc : (ok ? 0 : io_error());
  if (fclose(f) != 0 && err == 0) err = io_error();
  if (err < 0 && err != -3) snprintf(t->err, sizeof t->err, "%s: %s", path, strerror(-err));
  return err;
}

// HashTable::LoadTable (HashTable.cpp:439-459) of the table's buckets [lo, hi): the others are walked past.  More than
// max_entries entries in the range: -ENOSPC and an empty table, like any failed load.  The entries are read into the pinned
// chunk buffer and copied to the device, or with host entries read straight into their place in ent; either way the index
// is rebuilt on the device.
static int dpt_load(kgx_dptable* t, const char* path, uint64_t max_entries, uint32_t* dp_bits, uint64_t range_start[4],
                    uint64_t range_end[4], uint64_t keyx[4], uint64_t keyy[4], uint64_t* total_count, double* total_time,
                    uint64_t* nb_walk, uint64_t* walk_offset, cudaStream_t st) {
  using namespace kgx_dpt;
  using namespace kgx_wf;
  DPT_CK(t, cudaSetDevice(t->dev));
  DPT_CK(t, cudaStreamSynchronize(st));
  if (dpt_reset(t, st)) return -3;                         // HashTable::LoadTable starts with Reset()
  if (dpt_pinned(t)) return -3;
  if (max_entries > t->capacity) max_entries = t->capacity;
  errno = 0;
  FILE* f = fopen(path, "rb");
  if (!f) { const int e = io_error(); snprintf(t->err, sizeof t->err, "%s: %s", path, strerror(-e)); return e; }
  setvbuf(f, nullptr, _IOFBF, 1 << 22);
  WorkHeader hd;                                          // Kangaroo::LoadWork (Backup.cpp:149-207)
  uint64_t walk = 0, off = 0;
  bool ok = read_header(f, hd);
  uint32_t* nbH = (uint32_t*)malloc(8ull * NBUCKET);
  if (!nbH) { fclose(f); snprintf(t->err, sizeof t->err, "out of host memory"); return -ENOMEM; }
  uint32_t* mxH = nbH + NBUCKET;
  int rc = 0;
  uint64_t staged = 0, total = 0;
  auto flush = [&]() -> bool {                            // staged entries -> ent[count ..], then into the index
    if (!staged) return true;
    if (t->count + staged > t->capacity) {
      rc = -ENOSPC;
      return false;
    }
    const uint64_t B = 256;
    bool good = (t->entHost || cudaMemcpyAsync(t->ent + t->count, t->hostEnt, sizeof(Entry) * staged, cudaMemcpyHostToDevice, st) ==
                                   cudaSuccess) &&
                cudaMemcpyAsync(t->ent_h + t->count, t->hostH, 4 * staged, cudaMemcpyHostToDevice, st) == cudaSuccess;
    if (good) k_index_entries<<<(unsigned)((staged + B - 1) / B), (unsigned)B, 0, st>>>(t->ent, t->ent_h, t->count, staged, t->slots, t->nslots);
    good = good && cudaStreamSynchronize(st) == cudaSuccess;    // the pinned buffers are refilled next
    if (!good) { rc = -3; snprintf(t->err, sizeof t->err, "kgx_dptable_load_work: %s", cudaGetErrorString(cudaGetLastError())); return false; }
    t->count += staged;
    staged = 0;
    return true;
  };
  for (uint32_t h = 0; ok && h < NBUCKET; h++) {
    ok = read_bucket_head(f, nbH[h], mxH[h]);
    if (ok && (h < t->lo || h >= t->hi)) {                 // another shard's bucket
      ok = nbH[h] == 0 || fseeko(f, (off_t)nbH[h] * (off_t)sizeof(Entry), SEEK_CUR) == 0;
      nbH[h] = mxH[h] = 0;
      continue;
    }
    uint32_t left = ok ? nbH[h] : 0;
    total += left;
    if (ok && total > max_entries) { rc = -ENOSPC; ok = false; break; }
    while (ok && left) {
      if (staged == t->chunk && !flush()) { ok = false; break; }
      const uint32_t k = (uint32_t)std::min<uint64_t>(left, t->chunk - staged);
      // total <= max_entries <= capacity: the entries read fit, host ones straight in ent
      ok = fread((t->entHost ? t->entHost + t->count : t->hostEnt) + staged, sizeof(Entry), k, f) == k;
      for (uint32_t q = 0; q < k; q++) t->hostH[staged + q] = h;
      staged += k;
      left -= k;
    }
  }
  ok = ok && flush();
  ok = ok && fread(&walk, 8, 1, f) == 1 && walks_complete(f, walk, off);
  fclose(f);
  if (ok) {
    ok = cudaMemcpy(t->nb, nbH, 4ull * NBUCKET, cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(t->mx, mxH, 4ull * NBUCKET, cudaMemcpyHostToDevice) == cudaSuccess;
    const ull c = t->count;
    ok = ok && cudaMemcpy(&t->res->count, &c, 8, cudaMemcpyHostToDevice) == cudaSuccess;
    if (!ok) rc = -3;
  }
  free(nbH);
  if (!ok) {
    if (rc == -ENOSPC && max_entries < t->capacity)
      snprintf(t->err, sizeof t->err, "%s: buckets [%u, %u) hold more than %llu entries", path, t->lo, t->hi, (unsigned long long)max_entries);
    else if (rc == -ENOSPC)
      snprintf(t->err, sizeof t->err, "%s holds more than the table's capacity of %llu entries", path, (unsigned long long)t->capacity);
    else if (rc == 0)
      snprintf(t->err, sizeof t->err, "%s is not a complete HEADW work file", path);
    dpt_reset(t, st);
    return rc ? rc : -EINVAL;
  }
  get_header(hd, dp_bits, range_start, range_end, keyx, keyy, total_count, total_time);
  if (nb_walk) *nb_walk = walk;
  if (walk_offset) *walk_offset = off;
  return 0;
}

int kgx_dptable_load_work(kgx_dptable* t, const char* path, uint32_t* dp_bits, uint64_t range_start[4], uint64_t range_end[4],
                          uint64_t keyx[4], uint64_t keyy[4], uint64_t* total_count, double* total_time, uint64_t* nb_walk,
                          uint64_t* walk_offset, void* stream) {
  return dpt_load(t, path, t->capacity, dp_bits, range_start, range_end, keyx, keyy, total_count, total_time, nb_walk, walk_offset,
                  (cudaStream_t)stream);
}

int kgx_dptable_load_range(kgx_dptable* t, const char* path, uint32_t* dp_bits, uint64_t range_start[4], uint64_t range_end[4],
                           uint64_t keyx[4], uint64_t keyy[4], uint64_t* total_count, double* total_time, uint64_t* nb_walk,
                           uint64_t* walk_offset, uint64_t max_entries, void* stream) {
  return dpt_load(t, path, max_entries, dp_bits, range_start, range_end, keyx, keyy, total_count, total_time, nb_walk, walk_offset,
                  (cudaStream_t)stream);
}

}  // extern "C"
