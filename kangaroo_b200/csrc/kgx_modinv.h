// kgx_modinv.h -- modular inverse mod p = 2^256 - 0x1000003D1, variable time, host+device.
//
// Replaces the reference's GPU/GPUMath.h:700-803 (_ModInv: DRS62 "delayed right shift" divsteps on 64-bit
// limbs, which sm_90a has to emulate).  Algorithm and structure: the Bernstein-Yang "safegcd" divstep iteration in
// the variable-time signed-30-bit-limb form published by libsecp256k1 (src/modinv32_impl.h, MIT licence, P. Wuille):
// divsteps_30_var / update_de_30 / update_fg_30 / normalize_30 and the f*g*(f^2-2) 6-bit inverse trick follow that
// design -- third-party public code, NOT the reference -- re-typed here for one fixed modulus p (constants folded,
// host+device, static register indexing).  Batches of 30 divsteps on the low words, 2x2 transition matrices with
// 32-bit signed entries applied to (f,g) and (d,e) held as 9 signed 30-bit limbs, so every product is one native
// 32x32->64 IMAD.WIDE.  Result contract = the reference's: the canonical inverse in [0,p), and inv(0) = 0
// (GPUMath.h:785-801, IntMod.cpp:560-569).  Inputs are expected in [0, 2^256); the jump path only feeds products of
// fe_mul, i.e. values < 2^256 congruent to their residue.  (Input exactly p is not reduced first: the host twin
// returns 1 for it, not 0 -- unreachable from the jump path, probability 2^-256.)
//
// In the jump kernel every lane of the inverting warp runs this on the SAME value (the tile product after
// the butterfly), so all data-dependent control flow is warp-uniform: no divergence.
// Compiles as plain C++ for the CPU unit test (tests/test_abi_cpu.py via csrc/kgx_hosttest.cpp).
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define KGX_HD __host__ __device__ __forceinline__
#else
#define KGX_HD static inline
#endif

namespace kgx {

struct s30 { int32_t v[9]; };
struct t2x2 { int32_t u, v, q, r; };

KGX_HD int ctz32(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return __ffs((int)x) - 1;
#else
  return __builtin_ctz(x);
#endif
}

// 30 divsteps on the low words; returns new eta and the transition matrix scaled by 2^30.
KGX_HD int32_t divsteps_30_var(int32_t eta, uint32_t f0, uint32_t g0, t2x2* t) {
  uint32_t u = 1, v = 0, q = 0, r = 1;
  uint32_t f = f0, g = g0, m, w;
  int i = 30, limit, zeros;
  for (;;) {
    zeros = ctz32(g | (0xFFFFFFFFu << i));
    g >>= zeros; u <<= zeros; v <<= zeros; eta -= zeros; i -= zeros;
    if (i == 0) break;
    if (eta < 0) {
      uint32_t tmp;
      eta = -eta;
      tmp = f; f = g; g = 0u - tmp;
      tmp = u; u = q; q = 0u - tmp;
      tmp = v; v = r; r = 0u - tmp;
    }
    // cancel up to 6 low bits of g at once: w = -g/f mod 2^limit, with f*(f*f-2) == -1/f mod 64
    limit = (eta + 1) > i ? i : (eta + 1);
    m = (0xFFFFFFFFu >> (32 - limit)) & 63u;
    w = (f * g * (f * f - 2u)) & m;
    g += f * w; q += u * w; r += v * w;
  }
  t->u = (int32_t)u; t->v = (int32_t)v; t->q = (int32_t)q; t->r = (int32_t)r;
  return eta;
}

// p in signed-30 form: limbs {-977, -4, 0, 0, 0, 0, 0, 0, 65536}
#define KGX_P0 (-977)
#define KGX_P1 (-4)
#define KGX_P8 (65536)
#define KGX_PINV30 0x2DDACACFu  // p^-1 mod 2^30

// (d,e) <- t * (d,e) / 2^30 mod p
KGX_HD void update_de_30(s30* d, s30* e, const t2x2* t) {
  const int32_t M30 = (int32_t)(0xFFFFFFFFu >> 2);
  const int32_t u = t->u, v = t->v, q = t->q, r = t->r;
  int32_t di, ei, md, me, sd, se;
  int64_t cd, ce;
  sd = d->v[8] >> 31; se = e->v[8] >> 31;
  md = (u & sd) + (v & se);
  me = (q & sd) + (r & se);
  di = d->v[0]; ei = e->v[0];
  cd = (int64_t)u * di + (int64_t)v * ei;
  ce = (int64_t)q * di + (int64_t)r * ei;
  md -= (int32_t)((KGX_PINV30 * (uint32_t)cd + (uint32_t)md) & (uint32_t)M30);
  me -= (int32_t)((KGX_PINV30 * (uint32_t)ce + (uint32_t)me) & (uint32_t)M30);
  cd += (int64_t)KGX_P0 * md;
  ce += (int64_t)KGX_P0 * me;
  cd >>= 30; ce >>= 30;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (int i = 1; i < 9; ++i) {
    di = d->v[i]; ei = e->v[i];
    cd += (int64_t)u * di + (int64_t)v * ei;
    ce += (int64_t)q * di + (int64_t)r * ei;
    if (i == 1) { cd += (int64_t)KGX_P1 * md; ce += (int64_t)KGX_P1 * me; }
    if (i == 8) { cd += (int64_t)KGX_P8 * md; ce += (int64_t)KGX_P8 * me; }
    d->v[i - 1] = (int32_t)cd & M30; cd >>= 30;
    e->v[i - 1] = (int32_t)ce & M30; ce >>= 30;
  }
  d->v[8] = (int32_t)cd;
  e->v[8] = (int32_t)ce;
}

// (f,g) <- t * (f,g) / 2^30 on the first len limbs
template <int LEN>
KGX_HD void update_fg_30(s30* f, s30* g, const t2x2* t) {
  const int32_t M30 = (int32_t)(0xFFFFFFFFu >> 2);
  const int32_t u = t->u, v = t->v, q = t->q, r = t->r;
  int32_t fi, gi;
  int64_t cf, cg;
  fi = f->v[0]; gi = g->v[0];
  cf = (int64_t)u * fi + (int64_t)v * gi;
  cg = (int64_t)q * fi + (int64_t)r * gi;
  cf >>= 30; cg >>= 30;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (int i = 1; i < LEN; ++i) {
    fi = f->v[i]; gi = g->v[i];
    cf += (int64_t)u * fi + (int64_t)v * gi;
    cg += (int64_t)q * fi + (int64_t)r * gi;
    f->v[i - 1] = (int32_t)cf & M30; cf >>= 30;
    g->v[i - 1] = (int32_t)cg & M30; cg >>= 30;
  }
  f->v[LEN - 1] = (int32_t)cf;
  g->v[LEN - 1] = (int32_t)cg;
}

// r <- r * sign(f) normalised into [0,p)
KGX_HD void normalize_30(s30* r, int32_t sign) {
  const int32_t M30 = (int32_t)(0xFFFFFFFFu >> 2);
  int32_t r0 = r->v[0], r1 = r->v[1], r2 = r->v[2], r3 = r->v[3], r4 = r->v[4], r5 = r->v[5], r6 = r->v[6], r7 = r->v[7],
          r8 = r->v[8];
  int32_t cond_add, cond_negate;
  cond_add = r8 >> 31;
  r0 += KGX_P0 & cond_add; r1 += KGX_P1 & cond_add; r8 += KGX_P8 & cond_add;
  cond_negate = sign >> 31;
  r0 = (r0 ^ cond_negate) - cond_negate; r1 = (r1 ^ cond_negate) - cond_negate; r2 = (r2 ^ cond_negate) - cond_negate;
  r3 = (r3 ^ cond_negate) - cond_negate; r4 = (r4 ^ cond_negate) - cond_negate; r5 = (r5 ^ cond_negate) - cond_negate;
  r6 = (r6 ^ cond_negate) - cond_negate; r7 = (r7 ^ cond_negate) - cond_negate; r8 = (r8 ^ cond_negate) - cond_negate;
  r1 += r0 >> 30; r0 &= M30; r2 += r1 >> 30; r1 &= M30; r3 += r2 >> 30; r2 &= M30; r4 += r3 >> 30; r3 &= M30;
  r5 += r4 >> 30; r4 &= M30; r6 += r5 >> 30; r5 &= M30; r7 += r6 >> 30; r6 &= M30; r8 += r7 >> 30; r7 &= M30;
  cond_add = r8 >> 31;
  r0 += KGX_P0 & cond_add; r1 += KGX_P1 & cond_add; r8 += KGX_P8 & cond_add;
  r1 += r0 >> 30; r0 &= M30; r2 += r1 >> 30; r1 &= M30; r3 += r2 >> 30; r2 &= M30; r4 += r3 >> 30; r3 &= M30;
  r5 += r4 >> 30; r4 &= M30; r6 += r5 >> 30; r5 &= M30; r7 += r6 >> 30; r6 &= M30; r8 += r7 >> 30; r7 &= M30;
  r->v[0] = r0; r->v[1] = r1; r->v[2] = r2; r->v[3] = r3; r->v[4] = r4; r->v[5] = r5; r->v[6] = r6; r->v[7] = r7; r->v[8] = r8;
}

// in/out: 8 x u32 little-endian words (any value < 2^256); out: canonical inverse, 0 -> 0.
KGX_HD void modinv256(uint32_t out[8], const uint32_t in[8]) {
  const uint32_t M30 = 0xFFFFFFFFu >> 2;
  s30 d = {{0, 0, 0, 0, 0, 0, 0, 0, 0}}, e = {{1, 0, 0, 0, 0, 0, 0, 0, 0}};
  s30 f = {{KGX_P0, KGX_P1, 0, 0, 0, 0, 0, 0, KGX_P8}};
  s30 g;
  // 8 x 32 -> 9 x 30
  g.v[0] = (int32_t)(in[0] & M30);
  g.v[1] = (int32_t)(((in[0] >> 30) | (in[1] << 2)) & M30);
  g.v[2] = (int32_t)(((in[1] >> 28) | (in[2] << 4)) & M30);
  g.v[3] = (int32_t)(((in[2] >> 26) | (in[3] << 6)) & M30);
  g.v[4] = (int32_t)(((in[3] >> 24) | (in[4] << 8)) & M30);
  g.v[5] = (int32_t)(((in[4] >> 22) | (in[5] << 10)) & M30);
  g.v[6] = (int32_t)(((in[5] >> 20) | (in[6] << 12)) & M30);
  g.v[7] = (int32_t)(((in[6] >> 18) | (in[7] << 14)) & M30);
  g.v[8] = (int32_t)(in[7] >> 16);
  int32_t eta = -1;
  // full-length updates keep every loop fully unrolled with static register indexing (no local memory);
  // the batch count is data dependent (about 18 for random input; 25 bounds any 256-bit input).
  // KGX_INV_UNROLL batches run between two convergence tests: once g == 0 a further batch is the matrix (2^30, 0; 0, 1),
  // which leaves f and d unchanged (d at most re-normalised by +p), so testing less often is still exact.  The idea was to
  // let batch k+1's divsteps (which need only the low limbs of f, g) overlap the tail of batch k's 9-limb updates; the
  // extra batches run idle once g == 0, so by default the test stays after every batch.
#ifndef KGX_INV_UNROLL
#define KGX_INV_UNROLL 1
#endif
  for (int it = 0; it < (26 + KGX_INV_UNROLL - 1) / KGX_INV_UNROLL; ++it) {
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int k = 0; k < KGX_INV_UNROLL; ++k) {
      t2x2 t;
      eta = divsteps_30_var(eta, (uint32_t)f.v[0], (uint32_t)g.v[0], &t);
      update_de_30(&d, &e, &t);
      update_fg_30<9>(&f, &g, &t);
    }
    int32_t cond = g.v[0] | g.v[1] | g.v[2] | g.v[3] | g.v[4] | g.v[5] | g.v[6] | g.v[7] | g.v[8];
    if (cond == 0) break;
  }
  // gcd is |f| = 1 for invertible input; for 0 f = +-p and d = 0.
  normalize_30(&d, f.v[8]);
  out[0] = (uint32_t)d.v[0] | ((uint32_t)d.v[1] << 30);
  out[1] = ((uint32_t)d.v[1] >> 2) | ((uint32_t)d.v[2] << 28);
  out[2] = ((uint32_t)d.v[2] >> 4) | ((uint32_t)d.v[3] << 26);
  out[3] = ((uint32_t)d.v[3] >> 6) | ((uint32_t)d.v[4] << 24);
  out[4] = ((uint32_t)d.v[4] >> 8) | ((uint32_t)d.v[5] << 22);
  out[5] = ((uint32_t)d.v[5] >> 10) | ((uint32_t)d.v[6] << 20);
  out[6] = ((uint32_t)d.v[6] >> 12) | ((uint32_t)d.v[7] << 18);
  out[7] = ((uint32_t)d.v[7] >> 14) | ((uint32_t)d.v[8] << 16);
}

}  // namespace kgx
