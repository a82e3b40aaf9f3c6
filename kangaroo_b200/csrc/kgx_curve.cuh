// kgx_curve.cuh -- secp256k1 on the device, one copy for herd creation, the checkpoint conversion and the work-file check:
// the field helpers of the group law, the mixed and the affine add (both following the group law at equal x), G and n.
#pragma once
#include "kgx_field.cuh"
#include "kgx_modinv.h"

namespace kgx {

__device__ __forceinline__ void fe_neg(u32* r, const u32* a) {
  u32 z[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  fe_sub(r, z, a);
}
__device__ __forceinline__ void fe_dbl(u32* r, const u32* a) {   // 2a mod p
  u32 n[8];
  fe_neg(n, a);
  fe_sub(r, a, n);
}

// a == 0 (mod p)?  fe_mul / fe_sub results live in [0, 2^256): the only representatives of 0 are 0 and p.
__device__ __forceinline__ bool fe_is_zero_modp(const u32* a) {
  const u32 orv = a[0] | a[1] | a[2] | a[3] | a[4] | a[5] | a[6] | a[7];
  const u32 andv = a[2] & a[3] & a[4] & a[5] & a[6] & a[7];
  return orv == 0u || (andv == 0xFFFFFFFFu && a[1] == 0xFFFFFFFEu && a[0] == 0xFFFFFC2Fu);
}

// canonical residue: fe_mul / fe_sub leave values < 2^256 congruent mod p; subtract p once if needed
// (subtracting p mod 2^256 == adding 0x1000003D1)
__device__ __forceinline__ void fe_canon(u32* V) {
  const u32 pm[8] = {0xFFFFFC2Fu, 0xFFFFFFFEu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
  bool ge = true;
  for (int w = 7; w >= 0; w--) { if (V[w] != pm[w]) { ge = V[w] > pm[w]; break; } }
  if (ge) {
    u64 acc = (u64)V[0] + 0x3D1u; V[0] = (u32)acc;
    acc = (u64)V[1] + 1u + (acc >> 32); V[1] = (u32)acc;
    for (int w = 2; w < 8; w++) { acc = (u64)V[w] + (acc >> 32); V[w] = (u32)acc; }
  }
}

// the generator G, affine
__device__ __forceinline__ void set_g(u32* x, u32* y) {
  const u32 gx[8] = {0x16F81798u, 0x59F2815Bu, 0x2DCE28D9u, 0x029BFCDBu, 0xCE870B07u, 0x55A06295u, 0xF9DCBBACu, 0x79BE667Eu};
  const u32 gy[8] = {0xFB10D4B8u, 0x9C47D08Fu, 0xA6855419u, 0xFD17B448u, 0x0E1108A8u, 0x5DA4FBFCu, 0x26A3C465u, 0x483ADA77u};
#pragma unroll
  for (int w = 0; w < 8; w++) { x[w] = gx[w]; y[w] = gy[w]; }
}

// (X, Y, Z) += (qx, qy) in Jacobian + affine coordinates, the point at infinity as the flag inf.
//   H = x2 Z^2 - X ; R = y2 Z^3 - Y ; X3 = R^2 - H^3 - 2 X H^2 ; Y3 = R (X H^2 - X3) - Y H^3 ; Z3 = Z H
// Same x: the term equals the accumulator (a doubling) or its negative (the point at infinity) -- the group law, where the
// reference's AddDirect (SECP256K1.cpp:238-262) would divide by zero.
__device__ __forceinline__ void jac_add_affine(u32* X, u32* Y, u32* Z, bool& inf, const u32* qx, const u32* qy) {
  if (inf) { fe_copy(X, qx); fe_copy(Y, qy); fe_set_one(Z); inf = false; return; }
  u32 zz[8], u2[8], s2[8], h[8], r[8], hh[8], hhh[8], v[8], t[8];
  fe_sqr(zz, Z);
  fe_mul(u2, qx, zz);
  fe_mul(s2, qy, zz); fe_mul(s2, s2, Z);
  fe_sub(h, u2, X);
  fe_sub(r, s2, Y);
  if (fe_is_zero_modp(h)) {
    if (!fe_is_zero_modp(r)) { inf = true; return; }
    // Jacobian doubling, a = 0: S = 4 X Y^2 ; M = 3 X^2 ; X' = M^2 - 2S ; Y' = M (S - X') - 8 Y^4 ; Z' = 2 Y Z
    u32 yy[8], S[8], M[8], m2[8], y4[8], nx[8], ny[8], nz[8];
    fe_sqr(yy, Y);
    fe_mul(S, X, yy); fe_dbl(S, S); fe_dbl(S, S);
    fe_sqr(m2, X); fe_dbl(M, m2); { u32 ng[8]; fe_neg(ng, m2); fe_sub(M, M, ng); }
    fe_sqr(nx, M); fe_sub(nx, nx, S); fe_sub(nx, nx, S);
    fe_sqr(y4, yy); fe_dbl(y4, y4); fe_dbl(y4, y4); fe_dbl(y4, y4);
    fe_sub(ny, S, nx); fe_mul(ny, ny, M); fe_sub(ny, ny, y4);
    fe_mul(nz, Y, Z); fe_dbl(nz, nz);
    fe_copy(X, nx); fe_copy(Y, ny); fe_copy(Z, nz);
    return;
  }
  fe_sqr(hh, h);
  fe_mul(hhh, hh, h);
  fe_mul(v, X, hh);
  fe_sqr(t, r);
  fe_sub(t, t, hhh);
  fe_sub(t, t, v); fe_sub(t, t, v);            // X3
  fe_sub(v, v, t);
  fe_mul(v, v, r);
  fe_mul(hhh, hhh, Y);
  fe_sub(Y, v, hhh);                           // Y3
  fe_mul(Z, Z, h);                             // Z3
  fe_copy(X, t);
}

// (x1, y1) += (x2, y2) in affine coordinates with one inverse; canonical result.  Same x: doubling when the points are
// equal, the point at infinity (returns false, x1 / y1 then meaningless) when they are opposite -- the group law, as
// jac_add_affine.
__device__ bool affine_add(u32* x1, u32* y1, const u32* x2, const u32* y2) {
  u32 num[8], den[8], s[8], t[8];
  fe_sub(den, x2, x1);
  fe_sub(num, y2, y1);
  if (fe_is_zero_modp(den)) {
    if (!fe_is_zero_modp(num)) return false;
    // s = 3 x^2 / 2 y
    fe_sqr(t, x1);
    fe_dbl(num, t); fe_neg(s, t); fe_sub(num, num, s);
    fe_dbl(den, y1);
  }
  modinv256(t, den);
  fe_mul(s, num, t);
  fe_sqr(t, s); fe_sub(t, t, x1); fe_sub(t, t, x2);     // x3 = s^2 - x1 - x2
  fe_sub(num, x1, t); fe_mul(num, num, s); fe_sub(y1, num, y1);   // y3 = s (x1 - x3) - y1
  fe_copy(x1, t);
  fe_canon(x1);
  fe_canon(y1);
  return true;
}

// ---- the group order n, as 4 u64 limbs: kOrderHost for host code, kOrder (the same value) for the device ----------------
constexpr u64 kOrderHost[4] = {0xBFD25E8CD0364141ull, 0xBAAEDCE6AF48A03Bull, 0xFFFFFFFFFFFFFFFEull, 0xFFFFFFFFFFFFFFFFull};
__device__ __constant__ u64 kOrder[4] = {kOrderHost[0], kOrderHost[1], kOrderHost[2], kOrderHost[3]};

// r = a - b (mod 2^256); returns the borrow
__host__ __device__ __forceinline__ u64 sub256(u64* r, const u64* a, const u64* b) {
  u64 br = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const u64 t = a[k] - b[k];
    const u64 b1 = a[k] < b[k];
    r[k] = t - br;
    br = b1 | (t < br);
  }
  return br;
}
// r = a + b (mod 2^256); returns the carry
__host__ __device__ __forceinline__ u64 add256(u64* r, const u64* a, const u64* b) {
  u64 c = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const u64 t = a[k] + b[k];
    const u64 c1 = t < a[k];
    r[k] = t + c;
    c = c1 | (r[k] < t);
  }
  return c;
}
// a >= b
__host__ __device__ __forceinline__ bool ge256(const u64* a, const u64* b) {
#pragma unroll
  for (int k = 3; k >= 0; k--) if (a[k] != b[k]) return a[k] > b[k];
  return true;
}
__device__ __forceinline__ bool ge_order(const u64* a) { return ge256(a, kOrder); }

}  // namespace kgx
