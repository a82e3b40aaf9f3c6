/*
 * kgx_oracle.h -- CPU restatement of the reference kangaroo jump path (TEST INFRASTRUCTURE ONLY).
 *
 * This is the parity oracle for the H100 jump engine.  It is NOT part of the product: only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load it.
 * Every function cites the reference file:line (of the reference sources) whose algorithm it restates.
 *
 * Pinned against: SURVEY.md Appendix C golden vectors (jump table rangePower=64, 1024-jump
 * trajectory), the known answers of the reference's sample inputs, and -- in the build container --
 * the reference's own SECPK1 code compiled into oracle/_ref/libkref.so (tests/test_oracle_vs_ref.py).
 *
 * All field elements are 4 x u64 little-endian limbs (reference Int::bits64[0..3], SECPK1/Int.h:190).
 */
#ifndef KGX_ORACLE_H
#define KGX_ORACLE_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define KGO_NB_JUMP 32 /* Constants.h:29 */

/* ---- field GF(p), p = 2^256 - 0x1000003D1 (SECPK1/SECP256K1.cpp:29) ---- */
void kgo_mod_sub(uint64_t r[4], const uint64_t a[4], const uint64_t b[4]);   /* IntMod.cpp:95-99, GPUMath.h:476-494 */
void kgo_mod_mul(uint64_t r[4], const uint64_t a[4], const uint64_t b[4]);   /* IntMod.cpp:873-942 (fold, no final subtract) */
void kgo_mod_sqr(uint64_t r[4], const uint64_t a[4]);                        /* IntMod.cpp:1126-1234 */
void kgo_mod_inv(uint64_t r[4], const uint64_t a[4]);                        /* canonical inverse, 0 -> 0 (IntMod.cpp:368-569 result contract) */
void kgo_mod_neg(uint64_t r[4], const uint64_t a[4]);
void kgo_batch_inv(uint64_t *v, uint64_t *scratch, int n);                   /* IntGroup.cpp:36-58; v = n x 4 limbs in place */

/* ---- scalars mod group order n (SECP256K1.cpp:38) ---- */
void kgo_order_add(uint64_t r[4], const uint64_t a[4], const uint64_t b[4]); /* IntMod.cpp:1245-1257 ModAddK1order */
void kgo_order_sub(uint64_t r[4], const uint64_t a[4], const uint64_t b[4]); /* IntMod.cpp:1259-1263 ModSubK1order */

/* ---- curve (affine; infinity not represented except where noted) ---- */
void kgo_ec_add(uint64_t rx[4], uint64_t ry[4], const uint64_t ax[4], const uint64_t ay[4],
                const uint64_t bx[4], const uint64_t by[4]);                 /* SECP256K1.cpp:232-262 AddDirect */
void kgo_ec_dbl(uint64_t rx[4], uint64_t ry[4], const uint64_t ax[4], const uint64_t ay[4]); /* SECP256K1.cpp DoubleDirect */
/* k*G for k in [1,n); returns 0 on success, -1 for k == 0 (point at infinity). SECP256K1.cpp:59-87 */
int  kgo_ec_mul_g(uint64_t rx[4], uint64_t ry[4], const uint64_t k[4]);
int  kgo_ec_on_curve(const uint64_t x[4], const uint64_t y[4]);

/* ---- MT19937 exactly as SECPK1/Random.cpp:33-117 (one global state) ---- */
void     kgo_rseed(uint32_t seed);
uint32_t kgo_rndl(void);
void     kgo_rand_bits(uint64_t r[4], int nbit);                             /* Int.cpp:988-1001 Int::Rand(int) */

/* ---- search set-up ---- */
/* Kangaroo.cpp:742-832 CreateJumpTable (non-symmetry build).  Re-seeds MT with 0x600DCAFE.
 * jd: 32 x 2 limbs (128-bit), jpx/jpy: 32 x 4 limbs. Returns the number of draws used. */
int  kgo_create_jump_table(int range_power, uint64_t *jd, uint64_t *jpx, uint64_t *jpy);
/* Kangaroo.cpp:670-738 CreateHerd: d from the CURRENT MT state, type alternates starting at first_type;
 * wild kangaroos get d - width/2 (mod n) and start at key + d*G.  d is 4 limbs (mod n). */
void kgo_create_herd(int n, int range_power, const uint64_t range_width_div2[4],
                     const uint64_t keyx[4], const uint64_t keyy[4], int first_type,
                     uint64_t *px, uint64_t *py, uint64_t *d);
/* Kangaroo.cpp:154-164 SetDP */
uint64_t kgo_dp_mask(int dp_bits);

/* ---- the jump loop ---- */
typedef struct {
  uint64_t x[4];
  uint64_t d[4];   /* CPU convention: 256-bit mod n; GPU convention: low 2 limbs used */
  uint64_t kidx;
  uint32_t jump;   /* jump number (1-based within this call) at which the DP fired */
  uint32_t pad;
} kgo_dp_t;

/* Kangaroo.cpp:375-433 SolveKeyCPU inner loop (CPU convention: d += jD mod n, 256-bit), batched
 * inverse over groups of `grp` kangaroos (reference: CPU_GRP_SIZE=1024).  Runs `njumps` jumps on all
 * n kangaroos in place; DPs appended to dps (capacity max_dp); returns total DP count (may exceed max_dp). */
uint64_t kgo_jump_cpu(int n, int njumps, int grp, uint64_t *px, uint64_t *py, uint64_t *d,
                      const uint64_t *jd, const uint64_t *jpx, const uint64_t *jpy,
                      uint64_t dp_mask, kgo_dp_t *dps, uint64_t max_dp);
/* GPUCompute.h:45-109 device convention: d is 128-bit (2 limbs, wraps), already biased by wildOffset. */
uint64_t kgo_jump_gpu_conv(int n, int njumps, int grp, uint64_t *px, uint64_t *py, uint64_t *d128,
                      const uint64_t *jd, const uint64_t *jpx, const uint64_t *jpy,
                      uint64_t dp_mask, kgo_dp_t *dps, uint64_t max_dp);
/* Check.cpp:534-586 formulation: one AddDirect (own inversion) per kangaroo per jump. */
void kgo_jump_single(uint64_t x[4], uint64_t y[4], uint64_t d[4],
                     const uint64_t *jd, const uint64_t *jpx, const uint64_t *jpy);

/* HashTable.cpp:75-100 Convert: (x,d,type) -> bucket h, 128-bit x, tagged 128-bit d */
void kgo_hash_convert(const uint64_t x[4], const uint64_t d[4], uint32_t type,
                      uint64_t *h, uint64_t X[2], uint64_t D[2]);

/* Multi-threaded timing leg for bench.py (port of the SolveKeyCPU inner loop, `threads` pthreads,
 * each on its own 1024-kangaroo group). Returns total jumps done; seconds in *sec. */
uint64_t kgo_bench_cpu(int threads, int jumps_per_kangaroo, int range_power, double *sec);

/* ---- USE_SYMMETRY restatement (Constants.h:25; Kangaroo.cpp:742-832, 670-738 sym branches; Check.cpp:534-556) ---- */
int  kgo_mod_positive(uint64_t y[4]);                                        /* IntMod.cpp:1270-1283 ModPositiveK1 */
void kgo_order_neg(uint64_t r[4], const uint64_t d[4]);                      /* IntMod.cpp:1265-1268 ModNegK1order */
int  kgo_create_jump_table_sym(int range_power, uint64_t *jd, uint64_t *jpx, uint64_t *jpy, uint64_t uv[2]);
void kgo_create_herd_sym(int n, int range_power, const uint64_t range_width_div4[4], const uint64_t keyx[4], const uint64_t keyy[4],
                         int first_type, uint64_t *px, uint64_t *py, uint64_t *d);
uint64_t kgo_jump_sym(int n, int njumps, int grp, uint64_t *px, uint64_t *py, uint64_t *d, uint8_t *last_jump,
                      const uint64_t *jd, const uint64_t *jpx, const uint64_t *jpy, uint64_t dp_mask, kgo_dp_t *dps, uint64_t max_dp,
                      int rule /* 1 = lastJump (Check.cpp:536-541), 2 = symClass (Kangaroo.cpp:381-384) */);

#ifdef __cplusplus
}
#endif
#endif
