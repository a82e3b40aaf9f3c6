// kgx_bucketsort.cuh -- a block of whole buckets of entries into work-file order (HashTable::SaveTable: buckets in order,
// entries by unsigned (x.hi, x.lo)) for the device table's save and the merge.  Three stable CUB radix passes over entry
// indices -- x.lo, x.hi, then the bucket -- so entries of equal (bucket, x) keep the order they came in.
#pragma once
#include <cub/cub.cuh>
#include "kgx_workfile.h"

namespace kgx_wf {

// pass 0: key[t] = x.lo, pass 1: x.hi, pass 2: the bucket - b0 (u32 keys) of entry e = idx[t] (e = t when idx is null).
// Pass 0 also writes val[t] = e, the values its sort carries.
__global__ void bucket_sort_key(const Entry* ent, const uint32_t* hs, const uint32_t* idx, uint32_t n, int pass, uint32_t b0,
                                uint64_t* key, uint32_t* val) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const uint32_t e = idx ? idx[t] : t;
  if (pass == 0) { key[t] = ent[e].x0; val[t] = e; }
  else if (pass == 1) key[t] = ent[e].x1;
  else reinterpret_cast<uint32_t*>(key)[t] = hs[e] - b0;
}

// out[t] = ent[idx[t]]
__global__ void bucket_gather(const Entry* ent, const uint32_t* idx, uint32_t n, Entry* out) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n) out[t] = ent[idx[t]];
}

// radix-sort scratch bytes for blocks of up to n entries
static size_t bucket_sort_scratch(uint64_t n) {
  size_t a = 0, b = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, a, (uint64_t*)nullptr, (uint64_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)n, 0, 64);
  cub::DeviceRadixSort::SortPairs(nullptr, b, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)n, 0, 19);
  return a > b ? a : b;
}

// The n entries ent[idx[t]] (ent[t] when idx is null) of buckets [b0, b1), hs[e] the bucket of entry e, sorted on stream st.
// Scratch: idxA / idxB of n indices (idxA may be idx), keyA / keyB of n keys, tmp of tmpBytes >= bucket_sort_scratch(n).
// *order: the sorted entry indices (idxB).
static cudaError_t bucket_sort(const Entry* ent, const uint32_t* hs, const uint32_t* idx, uint32_t n, uint32_t b0, uint32_t b1,
                               uint32_t* idxA, uint32_t* idxB, uint64_t* keyA, uint64_t* keyB, void* tmp, size_t tmpBytes,
                               cudaStream_t st, uint32_t** order) {
  const uint32_t T = 256, G = (n + T - 1) / T;
  int bits = 1;
  while ((1u << bits) < b1 - b0) bits++;
  size_t tb = tmpBytes;
  cudaError_t s;
  bucket_sort_key<<<G, T, 0, st>>>(ent, hs, idx, n, 0, b0, keyA, idxA);
  if ((s = cub::DeviceRadixSort::SortPairs(tmp, tb, keyA, keyB, idxA, idxB, (int)n, 0, 64, st)) != cudaSuccess) return s;
  bucket_sort_key<<<G, T, 0, st>>>(ent, hs, idxB, n, 1, b0, keyA, nullptr);
  tb = tmpBytes;
  if ((s = cub::DeviceRadixSort::SortPairs(tmp, tb, keyA, keyB, idxB, idxA, (int)n, 0, 64, st)) != cudaSuccess) return s;
  bucket_sort_key<<<G, T, 0, st>>>(ent, hs, idxA, n, 2, b0, keyA, nullptr);
  tb = tmpBytes;
  if ((s = cub::DeviceRadixSort::SortPairs(tmp, tb, (uint32_t*)keyA, (uint32_t*)keyB, idxA, idxB, (int)n, 0, bits, st)) != cudaSuccess)
    return s;
  *order = idxB;
  return cudaSuccess;
}

}  // namespace kgx_wf
