// kgx_partition.cuh -- one rank's 40-byte DP records (kgx_convert_dps) grouped by the rank that owns their bucket, for the
// sharded DP table (C ABI: include/kgx.h, kgx_dp_partition).  Rank r of W owns the buckets [floor(r*2^18/W),
// floor((r+1)*2^18/W)); a record with h >= 2^18 is malformed, counted and dropped.  The partition is stable: each group keeps
// the records' input order, so a shard meets the records of each of its buckets in the order the single table would.
//
// Three passes over tiles of 256 records, on the caller's stream:
//   1. per tile, a histogram of owners (W + 1 bins, the last one the malformed records), stored owner-major
//   2. an exclusive scan of it: the position of (owner, tile) in the grouped output
//   3. per tile, each record's rank among the tile's records of its owner (warp match + per-warp counts) -> its slot
#include <cub/cub.cuh>
#include "kgx_workfile.h"

namespace kgx_part {

constexpr uint32_t TILE = 256, WARPS = TILE / 32;

__host__ __device__ __forceinline__ uint32_t owner_of(uint32_t h, uint32_t world) {
  return (uint32_t)(((uint64_t)(h + 1) * world - 1) / kgx_wf::NBUCKET);   // the last r with floor(r*2^18/W) <= h
}

__device__ __forceinline__ uint32_t dest_of(const uint8_t* recs, uint32_t i, uint32_t world) {
  const uint32_t h = reinterpret_cast<const uint32_t*>(recs + 40ull * i)[1];
  return h < kgx_wf::NBUCKET ? owner_of(h, world) : world;
}

// Where record i goes: its owner, or `world` for a record left out (the malformed ones here; the wrong ones of
// kgx_resolver_verify_partition, whose Dest reads the check's flags)
struct ByBucket {
  const uint8_t* recs;
  __device__ __forceinline__ uint32_t operator()(uint32_t i, uint32_t world) const { return dest_of(recs, i, world); }
};

template <class Dest>
__global__ void k_hist(Dest dest, uint32_t n, uint32_t world, uint32_t ntiles, uint32_t* hist) {
  __shared__ uint32_t cnt[KGX_DPT_MAX_RANKS + 1];
  for (uint32_t d = threadIdx.x; d <= world; d += blockDim.x) cnt[d] = 0;
  __syncthreads();
  const uint32_t i = blockIdx.x * TILE + threadIdx.x;
  if (i < n) atomicAdd(&cnt[dest(i, world)], 1u);
  __syncthreads();
  for (uint32_t d = threadIdx.x; d <= world; d += blockDim.x) hist[(uint64_t)d * ntiles + blockIdx.x] = cnt[d];
}

// stride 0: the groups packed one after another; else group d starts at record d * stride.  left: null, or the indices of the
// first `cap` records left out, in input order
template <class Dest>
__global__ void k_scatter(const uint8_t* recs, Dest dest, uint32_t n, uint32_t world, uint32_t ntiles, const uint32_t* pos, uint64_t stride,
                          uint8_t* out, uint32_t* left, uint32_t cap) {
  __shared__ uint32_t wcnt[WARPS][KGX_DPT_MAX_RANKS + 1];
  const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (uint32_t k = threadIdx.x; k < WARPS * (world + 1); k += blockDim.x) wcnt[k / (world + 1)][k % (world + 1)] = 0;
  __syncthreads();
  const uint32_t i = blockIdx.x * TILE + threadIdx.x;
  const uint32_t d = i < n ? dest(i, world) : 0xFFFFFFFFu;
  const uint32_t peers = __match_any_sync(0xFFFFFFFFu, d);
  if (i < n && lane == __ffs(peers) - 1) wcnt[w][d] = __popc(peers);
  __syncthreads();
  if (i >= n || (d == world && !left)) return;
  uint32_t r = __popc(peers & ((1u << lane) - 1));
  for (uint32_t v = 0; v < w; v++) r += wcnt[v][d];
  const uint64_t p = pos[(uint64_t)d * ntiles + blockIdx.x];
  if (d == world) {                                       // the record's number among those left out
    const uint64_t b = p - pos[(uint64_t)world * ntiles] + r;
    if (b < cap) left[b] = i;
    return;
  }
  const uint64_t slot = stride ? d * stride + (p - pos[(uint64_t)d * ntiles]) + r : p + r;
  // 32-bit words: kgx_convert_dps's records follow its u32 count, so they are 4-byte aligned only
  const uint32_t* s4 = reinterpret_cast<const uint32_t*>(recs + 40ull * i);
  uint32_t* o4 = reinterpret_cast<uint32_t*>(out + 40ull * slot);
#pragma unroll
  for (int k = 0; k < 10; k++) o4[k] = s4[k];
}

__global__ void k_counts(const uint32_t* hist, const uint32_t* pos, uint32_t world, uint32_t ntiles, uint32_t* counts) {
  const uint32_t d = threadIdx.x + blockIdx.x * blockDim.x;
  if (d > world) return;
  const uint64_t last = (uint64_t)(world + 1) * ntiles - 1;
  const uint32_t end = d < world ? pos[(uint64_t)(d + 1) * ntiles] : pos[last] + hist[last];
  counts[d] = end - pos[(uint64_t)d * ntiles];
}

inline uint32_t tiles_for(uint32_t n) { return n ? (n + TILE - 1) / TILE : 1; }

inline size_t scan_bytes(uint32_t n, uint32_t world) {
  size_t b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, b, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)((uint64_t)(world + 1) * tiles_for(n)));
  return b;
}

inline uint64_t align256(uint64_t v) { return (v + 255) & ~255ull; }

// the three passes and the counts on st, scratch as kgx_dp_partition_scratch_bytes(n, world) lays it out -> 0 or -3
template <class Dest>
int run(const uint8_t* recs, Dest dest, uint32_t n, uint32_t world, uint64_t stride, void* out, uint32_t* counts, uint32_t* left,
        uint32_t cap, void* scratch, uint64_t scratch_bytes, cudaStream_t st) {
  const uint32_t nt = tiles_for(n);
  const uint64_t cells = (uint64_t)(world + 1) * nt;
  uint8_t* s = static_cast<uint8_t*>(scratch);
  uint32_t* hist = reinterpret_cast<uint32_t*>(s);
  uint32_t* pos = reinterpret_cast<uint32_t*>(s + align256(4 * cells));
  void* tmp = s + 2 * align256(4 * cells);
  size_t tb = scratch_bytes - 2 * align256(4 * cells);
  k_hist<<<nt, TILE, 0, st>>>(dest, n, world, nt, hist);
  if (cudaGetLastError() != cudaSuccess) return -3;
  if (cub::DeviceScan::ExclusiveSum(tmp, tb, hist, pos, (int)cells, st) != cudaSuccess) return -3;
  if (n) k_scatter<<<nt, TILE, 0, st>>>(recs, dest, n, world, nt, pos, stride, static_cast<uint8_t*>(out), left, cap);
  k_counts<<<(world + 1 + 255) / 256, 256, 0, st>>>(hist, pos, world, nt, counts);
  return cudaGetLastError() == cudaSuccess ? 0 : -3;
}

}  // namespace kgx_part

extern "C" {

uint64_t kgx_dp_partition_scratch_bytes(uint32_t n, uint32_t world) {
  using namespace kgx_part;
  if (world == 0 || world > KGX_DPT_MAX_RANKS) return 0;
  const uint64_t cells = (uint64_t)(world + 1) * tiles_for(n);
  return 2 * align256(4 * cells) + align256(scan_bytes(n, world));
}

int kgx_dp_partition(const void* recs, uint32_t n, uint32_t world, uint64_t stride, void* out, uint32_t* counts, void* scratch,
                     uint64_t scratch_bytes, void* stream) {
  using namespace kgx_part;
  if (world == 0 || world > KGX_DPT_MAX_RANKS || n >= 0x80000000u || (stride != 0 && stride < n) ||
      scratch_bytes < kgx_dp_partition_scratch_bytes(n, world))
    return -1;
  const uint8_t* in = static_cast<const uint8_t*>(recs);
  return run(in, ByBucket{in}, n, world, stride, out, counts, nullptr, 0, scratch, scratch_bytes, (cudaStream_t)stream);
}

}  // extern "C"
