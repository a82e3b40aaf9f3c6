// kgx_field.cuh -- secp256k1 field arithmetic for sm_90a, 8 x 32-bit limbs, written from scratch.
//
// Replaces the reference's GPU/GPUMath.h (ModSub256 :476-516, _ModMult :810-907, _ModSqr :909-1019).
// The reference works on 4 x u64 limbs with 64-bit PTX multiplies that ptxas lowers to chains of
// 32x32 IMAD.WIDE.U32; here the 32-bit structure is explicit: every carry chain is ONE asm block of
// mad.lo.cc / madc.hi.cc pairs on an even/odd column split, which ptxas fuses into
// IMAD.WIDE.U32.X with predicate carries (65 IMAD.WIDE + 16 IADD3 for the 256x256->512 product).
//
// Result conventions (SURVEY.md App. A.3, bit-exact with IntMod.cpp:873-942):
//   fe_mul / fe_sqr : R1 = lo + hi*0x1000003D1 (exact, 290 bits); out = (R1 mod 2^256 + (R1>>256)*0x1000003D1) mod 2^256
//                     -- no final conditional subtraction, last carry dropped.
//   fe_sub          : a - b mod 2^256, plus p if the subtraction borrowed.
#pragma once
#include <cstdint>

typedef uint32_t u32;
typedef uint64_t u64;

#define KGX_C 0x3D1u  // 0x1000003D1 = 2^32 + 0x3D1

#include "kgx_chains.cuh"   // generated carry-chain primitives kgx_chain_{pairs}_{fresh words}_{carry: a|n|x}

// 512 -> 256 fold, see header comment. w[16] little-endian 32-bit words (w is consumed).
__device__ __forceinline__ void kgx_fold(u32* r, u32* w) {
  const u32 c = KGX_C;
  // E' = w[0..7] + {h0,h2,h4,h6} * c  (h = w[8..15]); e8 = carry
  u32 e[10];
#pragma unroll
  for (int i = 0; i < 8; i++) e[i] = w[i];
  kgx_chain_4_0_n(e, c, w[8], w[10], w[12], w[14]);
  // O'' = h (the 2^32 part of 0x1000003D1, words 1..8) + {h1,h3,h5,h7} * c (pairs at words 1,3,5,7): the products are
  // accumulated straight INTO a copy of h -- one chain, no separate 9-instruction addition.  Every multiplicand h_(2k+1) is read
  // for the last time by the instruction that overwrites its own accumulator word, so the copy may share its registers.
  u32 o[9];
#pragma unroll
  for (int i = 0; i < 8; i++) o[i] = w[8 + i];
  kgx_chain_4_0_n(o, c, w[9], w[11], w[13], w[15]);
  // R1 = E' + (O'' << 32): words 1..9
  asm("add.cc.u32  %0, %0, %9;\n\t"
      "addc.cc.u32 %1, %1, %10;\n\t"
      "addc.cc.u32 %2, %2, %11;\n\t"
      "addc.cc.u32 %3, %3, %12;\n\t"
      "addc.cc.u32 %4, %4, %13;\n\t"
      "addc.cc.u32 %5, %5, %14;\n\t"
      "addc.cc.u32 %6, %6, %15;\n\t"
      "addc.cc.u32 %7, %7, %16;\n\t"
      "addc.u32    %8, %17, 0;"
      : "+r"(e[1]), "+r"(e[2]), "+r"(e[3]), "+r"(e[4]), "+r"(e[5]), "+r"(e[6]), "+r"(e[7]), "+r"(e[8]), "=&r"(e[9])
      : "r"(o[0]), "r"(o[1]), "r"(o[2]), "r"(o[3]), "r"(o[4]), "r"(o[5]), "r"(o[6]), "r"(o[7]), "r"(o[8]));
  // second fold: top = e8 + e9*2^32 (e9 <= 2) ; V = top*(2^32+c) = e8*c + (e8 + e9*c)*2^32 + e9*2^64 ; r = R1[0..7] + V,
  // last carry dropped.  One wide multiply (e8*c) + one small 32-bit multiply (e9*c < 2^12).
  u32 v0, v1, v2;
  asm("{\n\t"
      ".reg .u32 q;\n\t"
      ".reg .u64 pw;\n\t"
      "mul.wide.u32   pw, %3, %5;\n\t"
      "mov.b64        {%0, %1}, pw;\n\t"
      "mul.lo.u32     q, %4, %5;\n\t"
      "add.cc.u32     %1, %1, %3;\n\t"
      "addc.u32       %2, %4, 0;\n\t"
      "add.cc.u32     %1, %1, q;\n\t"
      "addc.u32       %2, %2, 0;\n\t"
      "}"
      : "=&r"(v0), "=&r"(v1), "=&r"(v2)
      : "r"(e[8]), "r"(e[9]), "r"(c));
  asm("add.cc.u32  %0, %0, %8;\n\t"
      "addc.cc.u32 %1, %1, %9;\n\t"
      "addc.cc.u32 %2, %2, %10;\n\t"
      "addc.cc.u32 %3, %3, 0;\n\t"
      "addc.cc.u32 %4, %4, 0;\n\t"
      "addc.cc.u32 %5, %5, 0;\n\t"
      "addc.cc.u32 %6, %6, 0;\n\t"
      "addc.u32    %7, %7, 0;"
      : "+r"(e[0]), "+r"(e[1]), "+r"(e[2]), "+r"(e[3]), "+r"(e[4]), "+r"(e[5]), "+r"(e[6]), "+r"(e[7])
      : "r"(v0), "r"(v1), "r"(v2));
#pragma unroll
  for (int i = 0; i < 8; i++) r[i] = e[i];
}

// w[0..15] = E + (O << 32) where E[i] sits at word i and O[i] at word i+1 (E15 may be passed as 0).
__device__ __forceinline__ void kgx_merge_eo(u32* w, const u32* E, u32 E15, const u32* O) {
  w[0] = E[0];
  asm("add.cc.u32  %0, %15, %30;\n\t"
      "addc.cc.u32 %1, %16, %31;\n\t"
      "addc.cc.u32 %2, %17, %32;\n\t"
      "addc.cc.u32 %3, %18, %33;\n\t"
      "addc.cc.u32 %4, %19, %34;\n\t"
      "addc.cc.u32 %5, %20, %35;\n\t"
      "addc.cc.u32 %6, %21, %36;\n\t"
      "addc.cc.u32 %7, %22, %37;\n\t"
      "addc.cc.u32 %8, %23, %38;\n\t"
      "addc.cc.u32 %9, %24, %39;\n\t"
      "addc.cc.u32 %10, %25, %40;\n\t"
      "addc.cc.u32 %11, %26, %41;\n\t"
      "addc.cc.u32 %12, %27, %42;\n\t"
      "addc.cc.u32 %13, %28, %43;\n\t"
      "addc.u32    %14, %29, %44;"
      : "=&r"(w[1]), "=&r"(w[2]), "=&r"(w[3]), "=&r"(w[4]), "=&r"(w[5]), "=&r"(w[6]), "=&r"(w[7]), "=&r"(w[8]),
        "=&r"(w[9]), "=&r"(w[10]), "=&r"(w[11]), "=&r"(w[12]), "=&r"(w[13]), "=&r"(w[14]), "=&r"(w[15])
      : "r"(E[1]), "r"(E[2]), "r"(E[3]), "r"(E[4]), "r"(E[5]), "r"(E[6]), "r"(E[7]), "r"(E[8]), "r"(E[9]),
        "r"(E[10]), "r"(E[11]), "r"(E[12]), "r"(E[13]), "r"(E[14]), "r"(E15),
        "r"(O[0]), "r"(O[1]), "r"(O[2]), "r"(O[3]), "r"(O[4]), "r"(O[5]), "r"(O[6]), "r"(O[7]), "r"(O[8]),
        "r"(O[9]), "r"(O[10]), "r"(O[11]), "r"(O[12]), "r"(O[13]), "r"(O[14]));
}

// 256 x 256 -> 512 schoolbook on the even/odd column split; every accumulator word is written before it is
// read (no zero-initialisation), every row is one carry chain.
__device__ __forceinline__ void kgx_mul512(u32* w, const u32* a, const u32* b) {
  u32 E[16], O[15];
  // A chain whose TOP word is fresh (addend 0) can never carry out: hi(a*b) <= 0xFFFFFFFE, so hi + carry-in fits.  Those rows use
  // the _x variants (no carry word); the word above is then created by the NEXT row of the same parity, whose top word does
  // have an addend (_n: carry -> fresh word).  One instruction less per row pair than materialising an always-zero carry.
  kgx_chain_4_8_x(E + 0, b[0], a[0], a[2], a[4], a[6]);   // row 0 even j -> words 0..7   (all new)
  kgx_chain_4_8_x(O + 0, b[0], a[1], a[3], a[5], a[7]);   // row 0 odd  j -> words 1..8   (all new)
  kgx_chain_4_2_x(E + 2, b[1], a[1], a[3], a[5], a[7]);   // row 1 odd  j -> words 2..9,  E8 E9 new (no carry out of a fresh top)
  kgx_chain_4_0_n(O + 0, b[1], a[0], a[2], a[4], a[6]);   // row 1 even j -> words 1..8,  carry -> O8 new
  kgx_chain_4_0_n(E + 2, b[2], a[0], a[2], a[4], a[6]);   // row 2        words 2..9,  carry -> E10 new
  kgx_chain_4_1_x(O + 2, b[2], a[1], a[3], a[5], a[7]);   //              O9 new
  kgx_chain_4_1_x(E + 4, b[3], a[1], a[3], a[5], a[7]);   // row 3        E11 new
  kgx_chain_4_0_n(O + 2, b[3], a[0], a[2], a[4], a[6]);   //              carry -> O10 new
  kgx_chain_4_0_n(E + 4, b[4], a[0], a[2], a[4], a[6]);   // row 4        carry -> E12 new
  kgx_chain_4_1_x(O + 4, b[4], a[1], a[3], a[5], a[7]);   //              O11 new
  kgx_chain_4_1_x(E + 6, b[5], a[1], a[3], a[5], a[7]);   // row 5        E13 new
  kgx_chain_4_0_n(O + 4, b[5], a[0], a[2], a[4], a[6]);   //              carry -> O12 new
  kgx_chain_4_0_n(E + 6, b[6], a[0], a[2], a[4], a[6]);   // row 6        carry -> E14 new
  kgx_chain_4_1_x(O + 6, b[6], a[1], a[3], a[5], a[7]);   //              O13 new
  kgx_chain_4_1_x(E + 8, b[7], a[1], a[3], a[5], a[7]);   // row 7        E15 new, no carry out of word 15
  kgx_chain_4_0_n(O + 6, b[7], a[0], a[2], a[4], a[6]);   //              carry -> O14 new
  kgx_merge_eo(w, E, E[15], O);
}

__device__ __forceinline__ void fe_mul(u32* r, const u32* a, const u32* b) {
  u32 w[16];
  kgx_mul512(w, a, b);
  kgx_fold(r, w);
}

// a^2 as 28 cross products (computed once, doubled) + 8 squares: 36 IMAD.WIDE instead of 64.
// Same exact 512-bit value as a*a, hence the same folded result (GPUMath.h:909-1019 / IntMod.cpp:1030-1234).
__device__ __forceinline__ void kgx_sqr512(u32* w, const u32* a) {
  u32 E[16], O[15];
  // E[i] sits at word i, O[i] at word i+1; product a_i*a_j lands at word i+j.  E0 E1 are never written (zero).
  // (same rule as kgx_mul512: a chain with a fresh top word cannot carry out -> _x; the word above is created by the next chain
  //  of that parity with a real top addend -> _n.  E14 and O14 are never written: they are zero.)
  kgx_chain_4_8_x(O + 0, a[0], a[1], a[3], a[5], a[7]);   // 0x{1,3,5,7} -> words 1,3,5,7   O0..O7 new
  kgx_chain_3_6_x(E + 2, a[0], a[2], a[4], a[6]);         // 0x{2,4,6}   -> words 2,4,6     E2..E7 new
  kgx_chain_3_0_n(O + 2, a[1], a[2], a[4], a[6]);         // 1x{2,4,6}   -> words 3,5,7     carry -> O8 new
  kgx_chain_3_2_x(E + 4, a[1], a[3], a[5], a[7]);         // 1x{3,5,7}   -> words 4,6,8     E8 E9 new
  kgx_chain_3_1_x(O + 4, a[2], a[3], a[5], a[7]);         // 2x{3,5,7}   -> words 5,7,9     O9 new
  kgx_chain_2_0_n(E + 6, a[2], a[4], a[6]);               // 2x{4,6}     -> words 6,8       carry -> E10 new
  kgx_chain_2_0_n(O + 6, a[3], a[4], a[6]);               // 3x{4,6}     -> words 7,9       carry -> O10 new
  kgx_chain_2_1_x(E + 8, a[3], a[5], a[7]);               // 3x{5,7}     -> words 8,10      E11 new
  kgx_chain_2_1_x(O + 8, a[4], a[5], a[7]);               // 4x{5,7}     -> words 9,11      O11 new
  kgx_chain_1_0_n(E + 10, a[4], a[6]);                    // 4x6         -> word 10         carry -> E12 new
  kgx_chain_1_0_n(O + 10, a[5], a[6]);                    // 5x6         -> word 11         carry -> O12 new
  kgx_chain_1_1_x(E + 12, a[5], a[7]);                    // 5x7         -> word 12         E13 new
  kgx_chain_1_1_x(O + 12, a[6], a[7]);                    // 6x7         -> word 13         O13 new
  E[14] = 0; O[14] = 0;
  // C = E + (O << 32), words 1..15 (words 0 and, from E, 1 are zero)
  u32 c[16];
  c[1] = O[0];
  asm("add.cc.u32  %0, %14, %27;\n\t"
      "addc.cc.u32 %1, %15, %28;\n\t"
      "addc.cc.u32 %2, %16, %29;\n\t"
      "addc.cc.u32 %3, %17, %30;\n\t"
      "addc.cc.u32 %4, %18, %31;\n\t"
      "addc.cc.u32 %5, %19, %32;\n\t"
      "addc.cc.u32 %6, %20, %33;\n\t"
      "addc.cc.u32 %7, %21, %34;\n\t"
      "addc.cc.u32 %8, %22, %35;\n\t"
      "addc.cc.u32 %9, %23, %36;\n\t"
      "addc.cc.u32 %10, %24, %37;\n\t"
      "addc.cc.u32 %11, %25, %38;\n\t"
      "addc.cc.u32 %12, %26, %39;\n\t"
      "addc.u32    %13, 0, %40;"
      : "=&r"(c[2]), "=&r"(c[3]), "=&r"(c[4]), "=&r"(c[5]), "=&r"(c[6]), "=&r"(c[7]), "=&r"(c[8]),
        "=&r"(c[9]), "=&r"(c[10]), "=&r"(c[11]), "=&r"(c[12]), "=&r"(c[13]), "=&r"(c[14]), "=&r"(c[15])
      : "r"(E[2]), "r"(E[3]), "r"(E[4]), "r"(E[5]), "r"(E[6]), "r"(E[7]), "r"(E[8]), "r"(E[9]),
        "r"(E[10]), "r"(E[11]), "r"(E[12]), "r"(E[13]), "r"(E[14]),
        "r"(O[1]), "r"(O[2]), "r"(O[3]), "r"(O[4]), "r"(O[5]), "r"(O[6]), "r"(O[7]), "r"(O[8]),
        "r"(O[9]), "r"(O[10]), "r"(O[11]), "r"(O[12]), "r"(O[13]), "r"(O[14]));
  // 2C by funnel shifts (no carry chain); word 0 of 2C is zero
  u32 c2[16];
  c2[1] = c[1] << 1;
#pragma unroll
  for (int i = 15; i >= 2; i--) c2[i] = __funnelshift_l(c[i - 1], c[i], 1);
  // + squares a_i^2 at words (2i, 2i+1)
  asm("mul.lo.u32     %0, %16, %16;\n\t"
      "mad.hi.cc.u32  %1, %16, %16, %24;\n\t"
      "madc.lo.cc.u32 %2, %17, %17, %25;\n\t"
      "madc.hi.cc.u32 %3, %17, %17, %26;\n\t"
      "madc.lo.cc.u32 %4, %18, %18, %27;\n\t"
      "madc.hi.cc.u32 %5, %18, %18, %28;\n\t"
      "madc.lo.cc.u32 %6, %19, %19, %29;\n\t"
      "madc.hi.cc.u32 %7, %19, %19, %30;\n\t"
      "madc.lo.cc.u32 %8, %20, %20, %31;\n\t"
      "madc.hi.cc.u32 %9, %20, %20, %32;\n\t"
      "madc.lo.cc.u32 %10, %21, %21, %33;\n\t"
      "madc.hi.cc.u32 %11, %21, %21, %34;\n\t"
      "madc.lo.cc.u32 %12, %22, %22, %35;\n\t"
      "madc.hi.cc.u32 %13, %22, %22, %36;\n\t"
      "madc.lo.cc.u32 %14, %23, %23, %37;\n\t"
      "madc.hi.u32    %15, %23, %23, %38;"
      : "=&r"(w[0]), "=&r"(w[1]), "=&r"(w[2]), "=&r"(w[3]), "=&r"(w[4]), "=&r"(w[5]), "=&r"(w[6]), "=&r"(w[7]),
        "=&r"(w[8]), "=&r"(w[9]), "=&r"(w[10]), "=&r"(w[11]), "=&r"(w[12]), "=&r"(w[13]), "=&r"(w[14]), "=&r"(w[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(a[4]), "r"(a[5]), "r"(a[6]), "r"(a[7]),
        "r"(c2[1]), "r"(c2[2]), "r"(c2[3]), "r"(c2[4]), "r"(c2[5]), "r"(c2[6]), "r"(c2[7]),
        "r"(c2[8]), "r"(c2[9]), "r"(c2[10]), "r"(c2[11]), "r"(c2[12]), "r"(c2[13]), "r"(c2[14]), "r"(c2[15]));
}

__device__ __forceinline__ void fe_sqr(u32* r, const u32* a) {
  u32 w[16];
  kgx_sqr512(w, a);
  kgx_fold(r, w);
}

// r = a - b (mod 2^256), + p if borrow.   GPUMath.h:476-494 semantics.
__device__ __forceinline__ void fe_sub(u32* r, const u32* a, const u32* b) {
  u32 t0, t1, t2, t3, t4, t5, t6, t7, m;
  asm("sub.cc.u32  %0, %9, %17;\n\t"
      "subc.cc.u32 %1, %10, %18;\n\t"
      "subc.cc.u32 %2, %11, %19;\n\t"
      "subc.cc.u32 %3, %12, %20;\n\t"
      "subc.cc.u32 %4, %13, %21;\n\t"
      "subc.cc.u32 %5, %14, %22;\n\t"
      "subc.cc.u32 %6, %15, %23;\n\t"
      "subc.cc.u32 %7, %16, %24;\n\t"
      "subc.u32    %8, 0, 0;"
      : "=&r"(t0), "=&r"(t1), "=&r"(t2), "=&r"(t3), "=&r"(t4), "=&r"(t5), "=&r"(t6), "=&r"(t7), "=&r"(m)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(a[4]), "r"(a[5]), "r"(a[6]), "r"(a[7]),
        "r"(b[0]), "r"(b[1]), "r"(b[2]), "r"(b[3]), "r"(b[4]), "r"(b[5]), "r"(b[6]), "r"(b[7]));
  // + p (mod 2^256)  ==  - 0x1000003D1
  u32 k0 = m & KGX_C, k1 = m & 1u;
  asm("sub.cc.u32  %0, %0, %8;\n\t"
      "subc.cc.u32 %1, %1, %9;\n\t"
      "subc.cc.u32 %2, %2, 0;\n\t"
      "subc.cc.u32 %3, %3, 0;\n\t"
      "subc.cc.u32 %4, %4, 0;\n\t"
      "subc.cc.u32 %5, %5, 0;\n\t"
      "subc.cc.u32 %6, %6, 0;\n\t"
      "subc.u32    %7, %7, 0;"
      : "+r"(t0), "+r"(t1), "+r"(t2), "+r"(t3), "+r"(t4), "+r"(t5), "+r"(t6), "+r"(t7)
      : "r"(k0), "r"(k1));
  r[0] = t0; r[1] = t1; r[2] = t2; r[3] = t3; r[4] = t4; r[5] = t5; r[6] = t6; r[7] = t7;
}

// 128-bit distance accumulate (GPUMath.h:119-121 Add128): wraps silently.
__device__ __forceinline__ void d128_add(u32* d, u32 j0, u32 j1, u32 j2, u32 j3) {
  asm("add.cc.u32  %0, %0, %4;\n\t"
      "addc.cc.u32 %1, %1, %5;\n\t"
      "addc.cc.u32 %2, %2, %6;\n\t"
      "addc.u32    %3, %3, %7;"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
      : "r"(j0), "r"(j1), "r"(j2), "r"(j3));
}

// ---- USE_SYMMETRY helpers (SURVEY 8f/f4; reference: Int::ModPositiveK1 IntMod.cpp:1270-1283, GPUMath.h:518-531) ----
// mask = 0xFFFFFFFF when y > (p-1)/2 (the reference CPU test: 2y - p >= 0), else 0.  (p-1)/2 = 2^255 - 0x800001E9.
__device__ __forceinline__ u32 fe_gt_half_mask(const u32* y) {
  u32 t, m;
  asm("{\n\t"
      ".reg .u32 t;\n\t"
      "sub.cc.u32  t, 0x7FFFFE17, %1;\n\t"
      "subc.cc.u32 t, 0xFFFFFFFF, %2;\n\t"
      "subc.cc.u32 t, 0xFFFFFFFF, %3;\n\t"
      "subc.cc.u32 t, 0xFFFFFFFF, %4;\n\t"
      "subc.cc.u32 t, 0xFFFFFFFF, %5;\n\t"
      "subc.cc.u32 t, 0xFFFFFFFF, %6;\n\t"
      "subc.cc.u32 t, 0xFFFFFFFF, %7;\n\t"
      "subc.cc.u32 t, 0x7FFFFFFF, %8;\n\t"
      "subc.u32    %0, 0, 0;\n\t"
      "}"
      : "=r"(m)
      : "r"(y[0]), "r"(y[1]), "r"(y[2]), "r"(y[3]), "r"(y[4]), "r"(y[5]), "r"(y[6]), "r"(y[7]));
  (void)t;
  return m;      // borrow -> 0xFFFFFFFF
}
// y = mask ? p - y : y   (p - y = ~y - 0x1000003D0 for y <= p)
__device__ __forceinline__ void fe_cneg(u32* y, u32 m) {
  u32 k0 = m & 0x3D0u, k1 = m & 1u;
  u32 t0 = y[0] ^ m, t1 = y[1] ^ m, t2 = y[2] ^ m, t3 = y[3] ^ m, t4 = y[4] ^ m, t5 = y[5] ^ m, t6 = y[6] ^ m, t7 = y[7] ^ m;
  asm("sub.cc.u32  %0, %0, %8;\n\t"
      "subc.cc.u32 %1, %1, %9;\n\t"
      "subc.cc.u32 %2, %2, 0;\n\t"
      "subc.cc.u32 %3, %3, 0;\n\t"
      "subc.cc.u32 %4, %4, 0;\n\t"
      "subc.cc.u32 %5, %5, 0;\n\t"
      "subc.cc.u32 %6, %6, 0;\n\t"
      "subc.u32    %7, %7, 0;"
      : "+r"(t0), "+r"(t1), "+r"(t2), "+r"(t3), "+r"(t4), "+r"(t5), "+r"(t6), "+r"(t7)
      : "r"(k0), "r"(k1));
  y[0] = t0; y[1] = t1; y[2] = t2; y[3] = t3; y[4] = t4; y[5] = t5; y[6] = t6; y[7] = t7;
}
// signed 128-bit distance: d = mask ? -d : d  (two's complement; the symmetric engine keeps distances signed instead of the
// reference's biased-unsigned form, whose ModNeg256Order writes 256 bits into a 128-bit slot, GPUMath.h:533-547)
__device__ __forceinline__ void d128_cneg(u32* d, u32 m) {
  u32 t0 = d[0] ^ m, t1 = d[1] ^ m, t2 = d[2] ^ m, t3 = d[3] ^ m;
  asm("sub.cc.u32  %0, %0, %4;\n\t"
      "subc.cc.u32 %1, %1, %4;\n\t"
      "subc.cc.u32 %2, %2, %4;\n\t"
      "subc.u32    %3, %3, %4;"
      : "+r"(t0), "+r"(t1), "+r"(t2), "+r"(t3)
      : "r"(m));
  d[0] = t0; d[1] = t1; d[2] = t2; d[3] = t3;
}

__device__ __forceinline__ void fe_copy(u32* r, const u32* a) {
#pragma unroll
  for (int i = 0; i < 8; i++) r[i] = a[i];
}
__device__ __forceinline__ void fe_set_one(u32* r) {
  r[0] = 1;
#pragma unroll
  for (int i = 1; i < 8; i++) r[i] = 0;
}
