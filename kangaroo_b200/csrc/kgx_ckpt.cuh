// kgx_ckpt.cuh -- the herd in the reference's work-file form, converted on the device (checkpoint / resume).
//
// Record = what Kangaroo::SaveWork writes per kangaroo and FetchWalks reads back (Backup.cpp:536-539, 211-223):
// {x[4], y[4], d[4]} little-endian u64 limbs, 96 bytes, d = the distance mod n with the wild offset removed -- what
// GetKangaroos returns (GPUEngine.cu:477).  The engine keeps the biased 128-bit form (GPUEngine.cu:407-411), so
//   export: d = biased - wildOffset (mod n) for odd kIdx, biased for even kIdx      (256-bit result)
//   import: biased = (d mod n) + wildOffset (mod n) for odd kIdx, d mod n for even   (must fit in 128 bits)
#pragma once
#include "kgx_curve.cuh"   // kOrder, sub256, add256, ge_order

namespace kgx {

// staging (AoS u32, kIdx order: x 8 words, y 8 words, biased d 4 words) -> records rec[n][12] (u64)
__global__ void herd_export_kernel(const u32* __restrict__ px, const u32* __restrict__ py, const u32* __restrict__ d128,
                                   u64* __restrict__ rec, u64 n, u64 wo0, u64 wo1) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
    const u32* x = px + i * 8; const u32* y = py + i * 8; const u32* dv = d128 + i * 4;
    u64* o = rec + i * 12;
#pragma unroll
    for (int k = 0; k < 4; k++) {
      o[k] = (u64)x[2 * k] | ((u64)x[2 * k + 1] << 32);
      o[4 + k] = (u64)y[2 * k] | ((u64)y[2 * k + 1] << 32);
    }
    u64 d[4] = {(u64)dv[0] | ((u64)dv[1] << 32), (u64)dv[2] | ((u64)dv[3] << 32), 0, 0};
    if (i & 1ull) {
      const u64 wo[4] = {wo0, wo1, 0, 0};
      if (sub256(d, d, wo)) { u64 nn[4] = {kOrder[0], kOrder[1], kOrder[2], kOrder[3]}; add256(d, d, nn); }   // below zero: + n
    }
#pragma unroll
    for (int k = 0; k < 4; k++) o[8 + k] = d[k];
  }
}

// records [count][12] -> staging slots 0..count-1 (x, y, biased d) and scal[count][8 words] = d mod n (the scalar the
// position must equal d*G [+ key] for).  *bad (initialised to ~0) receives the lowest index whose biased distance needs
// more than 128 bits -- a record of another range.
__global__ void herd_import_kernel(const u64* __restrict__ rec, u64 count, u64 wo0, u64 wo1, u32* __restrict__ px,
                                   u32* __restrict__ py, u32* __restrict__ d128, u32* __restrict__ scal,
                                   unsigned long long* bad) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (u64)gridDim.x * blockDim.x) {
    const u64* r = rec + i * 12;
    u64 d[4] = {r[8], r[9], r[10], r[11]};
    if (ge_order(d)) { u64 nn[4] = {kOrder[0], kOrder[1], kOrder[2], kOrder[3]}; sub256(d, d, nn); }
    u64 b[4] = {d[0], d[1], d[2], d[3]};
    if (i & 1ull) {
      const u64 wo[4] = {wo0, wo1, 0, 0};
      const u64 c = add256(b, b, wo);
      if (c || ge_order(b)) { u64 nn[4] = {kOrder[0], kOrder[1], kOrder[2], kOrder[3]}; sub256(b, b, nn); }
    }
    if (b[2] | b[3]) atomicMin(bad, (unsigned long long)i);
#pragma unroll
    for (int k = 0; k < 4; k++) {
      px[i * 8 + 2 * k] = (u32)r[k]; px[i * 8 + 2 * k + 1] = (u32)(r[k] >> 32);
      py[i * 8 + 2 * k] = (u32)r[4 + k]; py[i * 8 + 2 * k + 1] = (u32)(r[4 + k] >> 32);
      scal[i * 8 + 2 * k] = (u32)d[k]; scal[i * 8 + 2 * k + 1] = (u32)(d[k] >> 32);
    }
#pragma unroll
    for (int k = 0; k < 2; k++) { d128[i * 4 + 2 * k] = (u32)b[k]; d128[i * 4 + 2 * k + 1] = (u32)(b[k] >> 32); }
  }
}

// count the slots whose (x, y) differ from the recomputed (vx, vy)
__global__ void herd_compare_kernel(const u32* __restrict__ px, const u32* __restrict__ py, const u32* __restrict__ vx,
                                    const u32* __restrict__ vy, u64 count, unsigned long long* mismatches) {
  for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (u64)gridDim.x * blockDim.x) {
    u32 diff = 0;
#pragma unroll
    for (int w = 0; w < 8; w++) diff |= (px[i * 8 + w] ^ vx[i * 8 + w]) | (py[i * 8 + w] ^ vy[i * 8 + w]);
    if (diff) atomicAdd(mismatches, 1ull);
  }
}

}  // namespace kgx
