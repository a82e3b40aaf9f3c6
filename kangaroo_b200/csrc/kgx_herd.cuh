// kgx_herd.cuh -- herd creation on the device (SURVEY.md 8f row f2; reference: Kangaroo::CreateHerd,
// Kangaroo.cpp:670-738, which calls Secp256K1::ComputePublicKeys + AddDirect on the CPU: 12 s per 2^21 kangaroos,
// README.md:398).  pos = d*G for tame kangaroos, key + d*G for wild ones; the affine result is unique, so instead of
// the reference's 32x256-entry byte table walk this uses a 256-entry table of 2^i*G built on the device, Jacobian
// mixed additions over the set bits of d, and ONE inversion per kangaroo.
#pragma once
#include "kgx_curve.cuh"
#include "kgx_kernel.cuh"

namespace kgx {

// tab[i] = 2^i * G (affine, 16 words each: x then y), i = 0..255.  One thread; 255 affine doublings.
__global__ void herd_table_kernel(u32* tab) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  u32 x[8], y[8];
  set_g(x, y);
  for (int i = 0; i < 256; i++) {
    for (int w = 0; w < 8; w++) { tab[i * 16 + w] = x[w]; tab[i * 16 + 8 + w] = y[w]; }
    // s = 3x^2 / 2y ; x' = s^2 - 2x ; y' = s (x - x') - y     (SECP256K1.cpp:438-466 DoubleDirect)
    u32 t[8], t3[8], y2[8], s[8], nx[8], ny[8];
    fe_sqr(t, x);
    fe_dbl(t3, t); { u32 n[8]; fe_neg(n, t); fe_sub(t3, t3, n); }
    fe_dbl(y2, y);
    modinv256(y2, y2);
    fe_mul(s, t3, y2);
    fe_sqr(nx, s);
    fe_sub(nx, nx, x); fe_sub(nx, nx, x);
    fe_sub(ny, x, nx); fe_mul(ny, ny, s); fe_sub(ny, ny, y);
    // canonicalise (table entries are compared against nothing, but keep them in [0,p) like the reference)
    fe_copy(x, nx); fe_copy(y, ny);
  }
}

// One thread per kangaroo: (x,y) = d*G [+ key].  scal: n x 8 words (d mod group order).  keys: the key table, 16 words
// (x then y) per key; the wild term of kangaroo i is key targets[i], or key 0 when targets is NULL (a single-key herd).
// Kangaroo i is wild when (i + firstType) is odd.  Writes AoS px,py (n x 8 words each) in kIdx order.
// sym != 0 (USE_SYMMETRY herd, Kangaroo.cpp:730-734): a point whose y is in the upper half is replaced by its negative and
// the stored (signed 128-bit) distance dist[i] is negated with it.
__global__ void herd_kernel(const u32* __restrict__ tab, const u32* __restrict__ scal, const u32* __restrict__ keys,
                            const uint16_t* __restrict__ targets, int firstType, u64 n, u32* px, u32* py, int sym, u32* dist) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  u32 k[8];
#pragma unroll
  for (int w = 0; w < 8; w++) k[w] = scal[i * 8 + w];
  u32 X[8], Y[8], Z[8];
  bool inf = true;
  const bool wild = ((i + (u64)firstType) & 1ull) != 0;
  const int nterms = 256 + (wild ? 1 : 0);
  for (int b = 0; b < nterms; b++) {
    const u32* q;
    if (b < 256) {
      if (!((k[b >> 5] >> (b & 31)) & 1u)) continue;
      q = tab + b * 16;
    } else {
      q = keys + (targets ? 16u * targets[i] : 0u);
    }
    u32 qx[8], qy[8];
#pragma unroll
    for (int w = 0; w < 8; w++) { qx[w] = q[w]; qy[w] = q[8 + w]; }
    // two table terms never share an x for a scalar < n; the key term does when d*G == +-key (a wild kangaroo created on
    // the key itself), and jac_add_affine then follows the group law
    jac_add_affine(X, Y, Z, inf, qx, qy);
  }
  if (inf) {
    // scalar 0 (tame) or d*G == -key (wild): the point at infinity has no affine form; store (0, 0) -- not on the curve,
    // the walk from it is meaningless but harmless (probability ~2^-rangePower; the reference stores an equally
    // meaningless Z = 0 projective conversion, SECP256K1.cpp:59-87).
#pragma unroll
    for (int w = 0; w < 8; w++) { px[i * 8 + w] = 0; py[i * 8 + w] = 0; }
    return;
  }
  u32 zi[8], zi2[8];
  modinv256(zi, Z);
  fe_sqr(zi2, zi);
  fe_mul(X, X, zi2);
  fe_mul(zi2, zi2, zi);
  fe_mul(Y, Y, zi2);
  fe_canon(X);
  fe_canon(Y);
  if (sym) {
    const u32 neg = fe_gt_half_mask(Y);
    fe_cneg(Y, neg);
    u32 d[4] = {dist[i * 4], dist[i * 4 + 1], dist[i * 4 + 2], dist[i * 4 + 3]};
    d128_cneg(d, neg);
    dist[i * 4] = d[0]; dist[i * 4 + 1] = d[1]; dist[i * 4 + 2] = d[2]; dist[i * 4 + 3] = d[3];
  }
#pragma unroll
  for (int w = 0; w < 8; w++) { px[i * 8 + w] = X[w]; py[i * 8 + w] = Y[w]; }
}

// ---- multi-key herd: moving the wild kangaroos of a solved key to other keys (kgx_retarget) ----------------------------
// The destination list of one kgx_retarget travels as kernel parameters, copied at launch: the call returns without
// waiting for the launch in flight and leaves no host buffer behind that the device still has to read.
constexpr int RETARGET_CHUNK = 1024;
struct RetargetChunk { uint16_t to[RETARGET_CHUNK]; };

// delta[j0 + j] = keys[to[j]] - keys[from] (16 words), rtTo[j0 + j] = to[j], bit 31 set when the difference is the point
// at infinity (the same key listed twice: the moved kangaroo keeps its point).
__global__ void retarget_delta_kernel(const u32* __restrict__ keys, u32 from, RetargetChunk c, u32 j0, u32 cnt, u32* delta,
                                      u32* rtTo) {
  const u32 j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= cnt) return;
  const u32 b = c.to[j];
  u32 x[8], y[8], fx[8], fy[8];
#pragma unroll
  for (int w = 0; w < 8; w++) { x[w] = keys[16 * b + w]; y[w] = keys[16 * b + 8 + w]; fx[w] = keys[16 * from + w]; fy[w] = keys[16 * from + 8 + w]; }
  fe_neg(fy, fy);
  const bool inf = !affine_add(x, y, fx, fy);
#pragma unroll
  for (int w = 0; w < 8; w++) { delta[16 * (j0 + j) + w] = x[w]; delta[16 * (j0 + j) + 8 + w] = y[w]; }
  rtTo[j0 + j] = b | (inf ? 0x80000000u : 0u);
}

// Every wild kangaroo s < n (kIdx order; wild when s + firstType is odd) whose target is `from` moves to key
// b = rtTo[(s >> 1) % nTo]: its point gets keys[b] - keys[from] added in place in the tile layout (slot_chunks), its
// distance stays, its target becomes b.  Padding slots are left stale, like patch_kernel leaves them.
__global__ void retarget_kernel(uint4* state, int T, int K, u64 n, int firstType, uint16_t* targets, u32 from,
                                const u32* __restrict__ delta, const u32* __restrict__ rtTo, u32 nTo) {
  const u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n || !((s + (u64)firstType) & 1ull) || targets[s] != from) return;
  const u32 j = (u32)((s >> 1) % nTo);
  const u32 tj = rtTo[j];
  targets[s] = (uint16_t)(tj & 0xFFFFu);
  if (tj >> 31) return;
  uint4* st = slot_chunks(state, s, T, K);
  uint4 c[4];
#pragma unroll
  for (int k = 0; k < 4; k++) c[k] = st[k * T];
  u32 x[8] = {c[0].x, c[0].y, c[0].z, c[0].w, c[1].x, c[1].y, c[1].z, c[1].w};
  u32 y[8] = {c[2].x, c[2].y, c[2].z, c[2].w, c[3].x, c[3].y, c[3].z, c[3].w};
  if (!affine_add(x, y, delta + 16 * j, delta + 16 * j + 8)) {
    // keys[b] + d*G is the point at infinity: stored as (0, 0), as herd_kernel does
#pragma unroll
    for (int w = 0; w < 8; w++) { x[w] = 0; y[w] = 0; }
  }
  st[0] = make_uint4(x[0], x[1], x[2], x[3]);
  st[T] = make_uint4(x[4], x[5], x[6], x[7]);
  st[2 * T] = make_uint4(y[0], y[1], y[2], y[3]);
  st[3 * T] = make_uint4(y[4], y[5], y[6], y[7]);
}

}  // namespace kgx
