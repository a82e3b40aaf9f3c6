// kgx_worktool.cuh -- checking and merging HEADW work files on one GPU (C ABI: include/kgx.h, kgx_work_*).
//
// Check (the reference's -wcheck, Check.cpp:33-108, 290-411): every stored DP {x lo 128, tagged d} of bucket h is OK iff
// S = +-|d|*G (+ K for a wild entry, K = keyToSearch = P - start*G) has S.x.bits64[2] & 0x3FFFF == h and the low 128 bits
// of S.x equal x.  |d| < 2^126, so S comes from a fixed-base comb: 32 windows of 4 bits, 15 affine points each
// (j * 2^(4w) * G, 30 KB in shared memory), added from the lowest window up with mixed Jacobian additions.  The partial sum
// of windows < w has a scalar below 2^(4w) and the next term one of at least 2^(4w), so two comb terms never meet the equal
// or opposite point; only the final +K can (S = +-K), and there the group law is followed: a doubling, or the point at
// infinity, which is counted wrong.  Affine x comes from Montgomery's batch inverse over each thread's GROUP entries.
// Walk records {x, y, d mod n} are checked by the same comb, magnitude min(d, n - d), compared projectively (no inverse):
// OK as tame when (x, y) = d*G, as wild when (x, y) = K + d*G.
//
// Merge (the reference's -wm / -wmdir, Merge.cpp:33-346, HashTable::MergeH): the inputs stream through in blocks of whole
// buckets, each bucket's entries uploaded in input order.  A stable radix sort by (h, x.hi, x.lo) keeps that order among
// equal keys; one scan keeps the first entry of every run of equal (h, x) -- the earliest input's, as the reference's
// pairwise merges do -- and classifies each later one against it: equal tagged d = a duplicate ("Dead kangaroo"), else a
// collision returned to the host.  The kept entries are compacted, counted per bucket and written with maxItem = nbItem
// rounded up to a multiple of 4 (HashTable.cpp:204-209).  Batch work files merge through the same blocks, each block's
// collisions resolved against every key on the device (wt_resolve_kernel, around wt_resolve_pair, which the persistent
// resolver of kgx_resolver.cuh shares).  The file format is kgx_workfile.h's, the block sort
// kgx_bucketsort.cuh's (shared with the device table's save) and the group law kgx_curve.cuh's (shared with herd creation).
#include <vector>
#include <algorithm>
#include <string>
#include <thrust/iterator/counting_iterator.h>
#include "kgx_workfile.h"
#include "kgx_bucketsort.cuh"
#include "kgx_curve.cuh"

namespace kgx_wt {

using ::u32;
using ::u64;
using kgx_wf::Entry;
using kgx_wf::NBUCKET;
typedef unsigned long long ull;
constexpr int COMB_W = 32, COMB_J = 15, COMB_WORDS = COMB_W * COMB_J * 16;   // 480 affine points, 16 words each
constexpr int CHECK_THREADS = 128, GROUP = 8;                                 // entries per thread share one inverse
constexpr uint64_t DEFAULT_CHUNK = 1ull << 21, DEFAULT_BLOCK = 1ull << 22;

struct Coll { uint32_t h, seq; uint64_t d_first[2], d_other[2]; };
struct MergeRes { ull dup, ncoll; };

// tab[(w * 15 + j - 1) * 16]: j * 2^(4w) * G, affine x then y, canonical.  Thread w builds window w.
__global__ void wt_comb_kernel(u32* tab) {
  const int w = threadIdx.x;
  if (w >= COMB_W) return;
  u32 bx[8], by[8];
  kgx::set_g(bx, by);
  for (int i = 0; i < 4 * w; i++) {                 // 2^(4w) * G
    u32 cx[8], cy[8];
    fe_copy(cx, bx); fe_copy(cy, by);
    kgx::affine_add(bx, by, cx, cy);
  }
  u32 x[8], y[8];
  fe_copy(x, bx); fe_copy(y, by);
  for (int j = 1; j <= COMB_J; j++) {
    u32* o = tab + (w * COMB_J + j - 1) * 16;
    for (int k = 0; k < 8; k++) { o[k] = x[k]; o[8 + k] = y[k]; }
    if (j < COMB_J) kgx::affine_add(x, y, bx, by);
  }
}

// m * G for a 128-bit m (4 words) from the comb in shared memory, lowest window first
__device__ __forceinline__ void wt_comb_mul(const u32* sc, const u32* m, u32* X, u32* Y, u32* Z, bool& inf) {
  inf = true;
#pragma unroll 1
  for (int w = 0; w < COMB_W; w++) {
    const u32 nib = (m[w >> 3] >> (4 * (w & 7))) & 15u;
    if (nib) {
      const u32* q = sc + (w * COMB_J + nib - 1) * 16;
      kgx::jac_add_affine(X, Y, Z, inf, q, q + 8);
    }
  }
}

__device__ __forceinline__ void wt_load_comb(u32* sc, const u32* comb) {
  for (int i = threadIdx.x; i < COMB_WORDS; i += blockDim.x) sc[i] = comb[i];
  __syncthreads();
}

// How wt_check_entries_kernel reads record i and reports it: d() gives its tagged distance (d1: bit 63 the sign, bit 62 the
// type, the rest |d| with d0), same() whether x (S.x, 8 words, canonical) is its (bucket, x lo 128), done() the verdict.
// Work-file entries: Entry + hs[i]; bad[i] = 1 when wrong, *nbad counts them.
struct EntryCheck {
  const Entry* ent;
  const uint32_t* hs;
  uint8_t* bad;
  ull* nbad;
  __device__ __forceinline__ void d(uint64_t i, u64& d0, u64& d1) const { d0 = ent[i].d0; d1 = ent[i].d1; }
  __device__ __forceinline__ bool same(uint64_t i, const u32* x) const {
    const Entry e = ent[i];
    return (x[4] & 0x3FFFFu) == hs[i] && (((u64)x[1] << 32) | x[0]) == e.x0 && (((u64)x[3] << 32) | x[2]) == e.x1;
  }
  __device__ __forceinline__ void done(uint64_t i, bool wrong) const {
    bad[i] = wrong;
    if (wrong) atomicAdd(nbad, 1ull);
  }
};

// 40-byte DP records {u32 kIdx; u32 h; u128 x; u128 tagged d} (Kangaroo.h:94-101), 8-byte aligned, as 5 words each:
// good[i] = 1 when record i is right.  h >= 2^18 never equals the 18 bits of S.x, so a malformed record is wrong.
struct Dp40Check {
  const u64* rec;
  uint32_t* good;
  __device__ __forceinline__ void d(uint64_t i, u64& d0, u64& d1) const { d0 = rec[5 * i + 3]; d1 = rec[5 * i + 4]; }
  __device__ __forceinline__ bool same(uint64_t i, const u32* x) const {
    return (x[4] & 0x3FFFFu) == (uint32_t)(rec[5 * i] >> 32) && (((u64)x[1] << 32) | x[0]) == rec[5 * i + 1] &&
           (((u64)x[3] << 32) | x[2]) == rec[5 * i + 2];
  }
  __device__ __forceinline__ void done(uint64_t i, bool wrong) const { good[i] = !wrong; }
};

// Records of a table (Src: EntryCheck, Dp40Check): record i is wrong unless S = +-|d|*G (+ K when wild) is not the point at
// infinity and src.same(i, S.x).  K: 16 words (x, y), kinf = K is the point at infinity.  Block b checks records
// [b * 128 * GROUP, (b + 1) * 128 * GROUP); thread t those at t + g * 128, g < GROUP, with one inverse for its group
// (records at infinity, past n or wrong, are left out of the product).
template <class Src>
__global__ void __launch_bounds__(CHECK_THREADS) wt_check_entries_kernel(const u32* __restrict__ comb, const Src src, uint64_t n,
                                                                        const u32* __restrict__ K, int kinf) {
  using namespace kgx;
  __shared__ u32 sc[COMB_WORDS];
  wt_load_comb(sc, comb);
  const uint64_t base = (uint64_t)blockIdx.x * (CHECK_THREADS * GROUP) + threadIdx.x;
  u32 X[GROUP][8], Z[GROUP][8], acc[GROUP][8];
  bool inf[GROUP];
  u32 run[8];
  fe_set_one(run);
#pragma unroll 1
  for (int g = 0; g < GROUP; g++) {
    const uint64_t i = base + (uint64_t)g * CHECK_THREADS;
    inf[g] = true;
    if (i < n) {
      u64 d0, d1;
      src.d(i, d0, d1);
      const bool wild = (d1 >> 62) & 1, neg = d1 >> 63;
      const u32 m[4] = {(u32)d0, (u32)(d0 >> 32), (u32)d1, (u32)(d1 >> 32) & 0x3FFFFFFFu};
      u32 Y[8];
      bool f;
      wt_comb_mul(sc, m, X[g], Y, Z[g], f);
      if (neg && !f) { u32 t[8]; fe_neg(t, Y); fe_copy(Y, t); }
      if (wild && !kinf) jac_add_affine(X[g], Y, Z[g], f, K, K + 8);
      inf[g] = f;
      if (!f) fe_mul(run, run, Z[g]);
    }
    fe_copy(acc[g], run);
  }
  u32 inv[8];
  modinv256(inv, run);
#pragma unroll 1
  for (int g = GROUP - 1; g >= 0; g--) {
    const uint64_t i = base + (uint64_t)g * CHECK_THREADS;
    if (i >= n) continue;
    bool wrong = true;
    if (!inf[g]) {
      u32 zi[8], x[8];
      if (g > 0) fe_mul(zi, inv, acc[g - 1]); else fe_copy(zi, inv);
      fe_mul(inv, inv, Z[g]);
      fe_sqr(zi, zi);
      fe_mul(x, X[g], zi);
      fe_canon(x);
      wrong = !src.same(i, x);
    }
    src.done(i, wrong);
  }
}

__device__ __forceinline__ bool wt_proj_eq(const u32* X, const u32* Y, const u32* Z, const u32* x, const u32* y) {
  using namespace kgx;
  u32 zz[8], t[8];
  fe_sqr(zz, Z);
  fe_mul(t, x, zz);
  fe_sub(t, X, t);
  if (!fe_is_zero_modp(t)) return false;
  fe_mul(zz, zz, Z);
  fe_mul(t, y, zz);
  fe_sub(t, Y, t);
  return fe_is_zero_modp(t);
}

// Walk records (96 bytes: x[4], y[4], d[4] limbs): res[i] = 1 tame OK, 2 wild OK, 0 wrong; cnt = {tame, wild, wrong}.
// bad[i] = 1 when wrong.  d >= n or min(d, n - d) >= 2^128 is wrong: engine distances are 128-bit.  K: the key table (16 words
// per key), kinfs[k] = key k is the point at infinity; record i is checked against key tg[i] (a batch file's targets), or key
// 0 when tg is null.
__global__ void __launch_bounds__(CHECK_THREADS) wt_check_walks_kernel(const u32* __restrict__ comb, const u32* __restrict__ recs,
                                                                      uint64_t n, const u32* __restrict__ K, const int* __restrict__ kinfs,
                                                                      const uint16_t* __restrict__ tg, uint8_t* res, uint8_t* bad, ull* cnt) {
  using namespace kgx;
  __shared__ u32 sc[COMB_WORDS];
  wt_load_comb(sc, comb);
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const u32* r = recs + i * 24;
    u32 x[8], y[8];
    for (int k = 0; k < 8; k++) { x[k] = r[k]; y[k] = r[8 + k]; }
    const u64* r64 = reinterpret_cast<const u64*>(r);
    u64 d[4] = {r64[8], r64[9], r64[10], r64[11]};
    int kind = 0;
    if (!ge_order(d)) {
      u64 nd[4];                                        // n - d
      const u64 nn[4] = {kOrder[0], kOrder[1], kOrder[2], kOrder[3]};
      sub256(nd, nn, d);
      const bool dle = ge256(nd, d);                    // d <= n - d ?
      const u64* m = dle ? d : nd;
      if ((m[2] | m[3]) == 0) {
        const u32 mw[4] = {(u32)m[0], (u32)(m[0] >> 32), (u32)m[1], (u32)(m[1] >> 32)};
        u32 X[8], Y[8], Z[8];
        bool f;
        wt_comb_mul(sc, mw, X, Y, Z, f);
        if (!dle && !f) { u32 t[8]; fe_neg(t, Y); fe_copy(Y, t); }
        if (!f && wt_proj_eq(X, Y, Z, x, y)) kind = 1;
        else {
          const u32 t = tg ? tg[i] : 0u;
          if (!kinfs[t]) jac_add_affine(X, Y, Z, f, K + 16 * t, K + 16 * t + 8);
          if (!f && wt_proj_eq(X, Y, Z, x, y)) kind = 2;
        }
      }
    }
    res[i] = (uint8_t)kind;
    bad[i] = kind == 0;
    atomicAdd(&cnt[kind == 0 ? 2 : kind - 1], 1ull);
  }
}

// key checks: *ok (set to 1 by the caller) is cleared when one of the n keys (x, y) is off the curve; K = key + s*G (s = -start
// mod n, 8 words) is left to herd_kernel
__global__ void wt_on_curve_kernel(const u32* keys, uint32_t n, int* ok) {
  using namespace kgx;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u32* key = keys + 16 * i;
  u32 l[8], r[8], s[8], seven[8] = {7, 0, 0, 0, 0, 0, 0, 0};
  fe_sqr(l, key + 8);
  fe_sqr(r, key);
  fe_mul(r, r, key);
  fe_neg(s, seven);
  fe_sub(r, r, s);                                      // x^3 + 7
  fe_sub(l, l, r);
  bool canon = true;                                    // coordinates must be below p, as the reference's EC() check reads them
  u32 t[8];
  for (int c = 0; c < 2; c++) { fe_copy(t, key + 8 * c); fe_canon(t); for (int k = 0; k < 8; k++) canon = canon && t[k] == key[8 * c + k]; }
  if (!(fe_is_zero_modp(l) && canon)) atomicAnd(ok, 0);
}

// Table entries of a batch file: as wt_check_entries_kernel, one entry per thread, but a wild entry is OK when S = +-|d|*G
// plus any of the n_keys keys K (16 words each; kinfs[k]: K is the point at infinity, then S itself) passes the test.  S is
// made affine once; then every key costs one affine addition, whose inverses are batched over KB keys at a time.  The group
// law is followed as in wt_check_entries_kernel: S at infinity (|d| = 0) gives K itself; K = S is a doubling, whose slope
// 3 x_S^2 / 2 y_S takes the key's place in the batched inverse; K = -S gives infinity, no match (its factor is 1, so that
// it leaves the other keys' inverses intact).  The scan stops at the first key that matches.
constexpr int KB = 8;
__global__ void __launch_bounds__(CHECK_THREADS) wt_check_entries_multi_kernel(const u32* __restrict__ comb, const Entry* __restrict__ ent,
                                                                              const uint32_t* __restrict__ hs, uint64_t n,
                                                                              const u32* __restrict__ K, const int* __restrict__ kinfs,
                                                                              uint32_t n_keys, uint8_t* bad, ull* nbad) {
  using namespace kgx;
  __shared__ u32 sc[COMB_WORDS];
  wt_load_comb(sc, comb);
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Entry e = ent[i];
  const uint32_t h = hs[i];
  auto match = [&](u32* x) { fe_canon(x); return (x[4] & 0x3FFFFu) == h && (((u64)x[1] << 32) | x[0]) == e.x0 && (((u64)x[3] << 32) | x[2]) == e.x1; };
  const bool wild = (e.d1 >> 62) & 1, neg = e.d1 >> 63;
  const u32 m[4] = {(u32)e.d0, (u32)(e.d0 >> 32), (u32)e.d1, (u32)(e.d1 >> 32) & 0x3FFFFFFFu};
  u32 X[8], Y[8], Z[8];
  bool f, ok = false;
  wt_comb_mul(sc, m, X, Y, Z, f);
  if (f && wild) {                                  // S at infinity: S + K = K
#pragma unroll 1
    for (uint32_t k = 0; k < n_keys && !ok; k++)
      if (!kinfs[k]) { u32 x[8]; fe_copy(x, K + 16 * k); ok = match(x); }
  } else if (!f) {
    u32 zi[8], z2[8];
    modinv256(zi, Z);
    fe_sqr(z2, zi);
    fe_mul(X, X, z2);
    fe_mul(z2, z2, zi);
    fe_mul(Y, Y, z2);
    fe_canon(X);
    fe_canon(Y);
    if (neg) { u32 t[8]; fe_neg(t, Y); fe_copy(Y, t); fe_canon(Y); }
    if (!wild) {
      u32 x[8];
      fe_copy(x, X);
      ok = match(x);
    } else {
      // key k's factor in the batched inverse -> 0: no addition (a missing key, K at infinity or K = -S; factor 1),
      // 1: an addition (x_K - x_S), 2: a doubling, K = S (2 y_S)
      auto factor = [&](uint32_t k, u32* dx) -> int {
        fe_set_one(dx);
        if (k >= n_keys || kinfs[k]) return 0;
        fe_sub(dx, K + 16 * k, X);
        if (!fe_is_zero_modp(dx)) return 1;
        u32 dy[8];
        fe_sub(dy, K + 16 * k + 8, Y);
        if (fe_is_zero_modp(dy)) { fe_dbl(dx, Y); return 2; }
        fe_set_one(dx);
        return 0;
      };
#pragma unroll 1
      for (uint32_t k0 = 0; k0 < n_keys && !ok; k0 += KB) {
        u32 acc[KB][8], run[8];
        fe_set_one(run);
#pragma unroll
        for (int j = 0; j < KB; j++) {            // prefix products of the factors
          u32 dx[8];
          factor(k0 + j, dx);
          fe_mul(run, run, dx);
          fe_copy(acc[j], run);
        }
        u32 inv[8];
        modinv256(inv, run);
#pragma unroll
        for (int j = KB - 1; j >= 0; j--) {
          const uint32_t k = k0 + j;
          u32 dx[8], di[8];
          const int add = factor(k, dx);
          if (j > 0) fe_mul(di, inv, acc[j - 1]); else fe_copy(di, inv);   // 1 / dx
          fe_mul(inv, inv, dx);
          if (k < n_keys && kinfs[k]) { u32 x[8]; fe_copy(x, X); ok = ok || match(x); }
          if (!add) continue;
          u32 lam[8], x3[8], t[8];
          if (add == 2) {                                 // 3 x_S^2
            u32 ng[8];
            fe_sqr(t, X);
            fe_dbl(lam, t); fe_neg(ng, t); fe_sub(lam, lam, ng);
          } else {
            fe_sub(lam, K + 16 * k + 8, Y);
          }
          fe_mul(lam, lam, di);
          fe_sqr(x3, lam);
          fe_sub(x3, x3, X);
          fe_sub(t, x3, K + 16 * k);
          ok = ok || match(t);
        }
      }
    }
  }
  bad[i] = !ok;
  if (!ok) atomicAdd(nbad, 1ull);
}

// ---- merge ----
// ord: the block's entries in (h, x) order, input order among equals.  keep[i] = first of its run; later entries are
// duplicates or collisions against that first one.  nb[h - b0] counts the kept entries of each bucket.
__global__ void wt_merge_scan(const Entry* ent, const uint32_t* hs, const uint32_t* ord, uint32_t n, uint32_t b0, uint8_t* keep,
                              uint32_t* nb, MergeRes* res, Coll* coll) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t e = ord[i];
  const Entry v = ent[e];
  const uint32_t h = hs[e];
  uint32_t f = i;
  while (f > 0) {
    const uint32_t p = ord[f - 1];
    if (hs[p] != h || ent[p].x0 != v.x0 || ent[p].x1 != v.x1) break;
    f--;
  }
  keep[i] = f == i;
  if (f == i) { atomicAdd(&nb[h - b0], 1u); return; }
  const Entry w = ent[ord[f]];
  if (w.d0 == v.d0 && w.d1 == v.d1) { atomicAdd(&res->dup, 1ull); return; }
  const ull c = atomicAdd(&res->ncoll, 1ull);
  coll[c] = Coll{h, i, {w.d0, w.d1}, {v.d0, v.d1}};
}

// ---- batch merge: every tame/wild collision resolved against all keys (kgi_resolve_multi's result, on the device) ----
// kgi_resolve_multi tries the four candidates +-Td +-Wd of Kangaroo::CheckKey against every key K and its negative and
// reports the first key in input order that one of them hits.  With t = |Td| and w = |Wd| (both < 2^126) the candidates are
// +-m1 and +-m2, m1 = t + w and m2 = |t - w| (< 2^127), so the keys hit are those whose x is the x of m1*G or of m2*G, and
// the sign of y gives s = +-m with s*G = K; the private key is s + start (mod n).  m = 0 gives the point at infinity, which the
// host stores as (0, 0), as the key table stores a key at infinity; no point of the curve has x = 0, so (0, 0) matches those
// keys only.
constexpr uint32_t NO_KEY = 0xFFFFFFFFu;
struct Hit { uint32_t h, seq, key, reserved; uint64_t priv[4], d_first[2], d_other[2]; };
struct Start { u64 v[4]; };                            // the range start, below n

__device__ __forceinline__ int wt_cmp8(const u32* a, const u32* b) {
  for (int w = 7; w >= 0; w--) if (a[w] != b[w]) return a[w] < b[w] ? -1 : 1;
  return 0;
}

// The first key (input order) that is (x, y) or its negative -> its index (NO_KEY: none), neg = it is -(x, y).  kx: the
// n keys' x, 8 words each, ascending, equal x in input order; ki: their indices; K: 16 words per key, by index.
__device__ uint32_t wt_find_key(const u32* kx, const uint32_t* ki, const u32* K, uint32_t n, const u32* x, const u32* y, bool& neg) {
  using namespace kgx;
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (wt_cmp8(kx + 8ull * mid, x) < 0) lo = mid + 1; else hi = mid;
  }
  u32 ny[8];
  fe_neg(ny, y);
  fe_canon(ny);
  for (; lo < n && wt_cmp8(kx + 8ull * lo, x) == 0; lo++) {
    const uint32_t k = ki[lo];
    if (wt_cmp8(K + 16ull * k + 8, y) == 0) { neg = false; return k; }
    if (wt_cmp8(K + 16ull * k + 8, ny) == 0) { neg = true; return k; }
  }
  return NO_KEY;
}

// One collision (two tagged distances, in either order) -> the key it hits (NO_KEY: none, same-herd included) and, with a key,
// its private key in priv (else 0).  sc: the comb in shared memory.  The two points share one inverse.
__device__ uint32_t wt_resolve_pair(const u32* sc, const u64* d_first, const u64* d_other, const u32* __restrict__ kx,
                                    const uint32_t* __restrict__ ki, const u32* __restrict__ K, uint32_t n_keys, const Start& start,
                                    u64* priv) {
  using namespace kgx;
  const u64 M = 0x3FFFFFFFFFFFFFFFull;
  const bool cross = ((d_first[1] ^ d_other[1]) >> 62) & 1;
  uint32_t key = NO_KEY;
  for (int w = 0; w < 4; w++) priv[w] = 0;
  if (cross) {                                         // a tame/wild pair
    const u64 a[2] = {d_first[0], d_first[1] & M}, b[2] = {d_other[0], d_other[1] & M};
    u64 m[2][2];
    m[0][0] = a[0] + b[0];
    m[0][1] = a[1] + b[1] + (m[0][0] < a[0]);
    const bool age = a[1] != b[1] ? a[1] > b[1] : a[0] >= b[0];
    const u64* p = age ? a : b;
    const u64* q = age ? b : a;
    m[1][0] = p[0] - q[0];
    m[1][1] = p[1] - q[1] - (p[0] < q[0]);
    u32 X[2][8], Y[2][8], Z[2][8];
    bool inf[2];
    for (int j = 0; j < 2; j++) {
      const u32 mw[4] = {(u32)m[j][0], (u32)(m[j][0] >> 32), (u32)m[j][1], (u32)(m[j][1] >> 32)};
      wt_comb_mul(sc, mw, X[j], Y[j], Z[j], inf[j]);
    }
    u32 zi[2][8], t[8];                                  // 1/Z of each finite point, from one inverse
    if (!inf[0] && !inf[1]) {
      fe_mul(t, Z[0], Z[1]);
      modinv256(t, t);
      fe_mul(zi[0], t, Z[1]);
      fe_mul(zi[1], t, Z[0]);
    } else {
      for (int j = 0; j < 2; j++) if (!inf[j]) modinv256(zi[j], Z[j]);
    }
    bool neg = false;
    int hit = -1;
    for (int j = 0; j < 2; j++) {
      u32 x[8] = {0, 0, 0, 0, 0, 0, 0, 0}, y[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (!inf[j]) {
        fe_sqr(t, zi[j]);
        fe_mul(x, X[j], t);
        fe_mul(t, t, zi[j]);
        fe_mul(y, Y[j], t);
        fe_canon(x);
        fe_canon(y);
      }
      bool ng = false;
      const uint32_t k = wt_find_key(kx, ki, K, n_keys, x, y, ng);
      if (k < key) { key = k; neg = ng; hit = j; }
    }
    if (hit >= 0) {                                      // s = +-m, priv = s + start (mod n)
      u64 s[4] = {m[hit][0], m[hit][1], 0, 0};
      if (neg && (s[0] | s[1])) { const u64 nn[4] = {kOrder[0], kOrder[1], kOrder[2], kOrder[3]}; sub256(s, nn, s); }
      const u64 cy = add256(priv, s, start.v);
      if (cy || ge_order(priv)) { const u64 nn[4] = {kOrder[0], kOrder[1], kOrder[2], kOrder[3]}; sub256(priv, priv, nn); }
    }
  }
  return key;
}

// The batch merge: one collision per thread, classified as cnt = {same herd, no key, key already solved, hit}; every hit on a
// key not in solved is appended to hits.
__global__ void __launch_bounds__(CHECK_THREADS) wt_resolve_kernel(const u32* __restrict__ comb, const Coll* __restrict__ coll, uint32_t n,
                                                                  const u32* __restrict__ kx, const uint32_t* __restrict__ ki,
                                                                  const u32* __restrict__ K, uint32_t n_keys, Start start,
                                                                  const uint8_t* solved, ull* cnt, Hit* hits) {
  __shared__ u32 sc[COMB_WORDS];
  wt_load_comb(sc, comb);
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Coll c = coll[i];
  const bool cross = ((c.d_first[1] ^ c.d_other[1]) >> 62) & 1;
  u64 priv[4];
  const uint32_t key = wt_resolve_pair(sc, c.d_first, c.d_other, kx, ki, K, n_keys, start, priv);
  if (!cross) atomicAdd(&cnt[0], 1ull);
  else if (key == NO_KEY) atomicAdd(&cnt[1], 1ull);
  else if (solved[key]) atomicAdd(&cnt[2], 1ull);
  else {
    const ull slot = atomicAdd(&cnt[3], 1ull);
    Hit& o = hits[slot];
    o.h = c.h; o.seq = c.seq; o.key = key; o.reserved = 0;
    for (int w = 0; w < 4; w++) o.priv[w] = priv[w];
    o.d_first[0] = c.d_first[0]; o.d_first[1] = c.d_first[1];
    o.d_other[0] = c.d_other[0]; o.d_other[1] = c.d_other[1];
  }
}

}  // namespace kgx_wt

static char g_wt_err[512] = "";

#define WT_CK(call)                                                                                   \
  do {                                                                                                \
    cudaError_t _s = (call);                                                                          \
    if (_s != cudaSuccess) {                                                                          \
      snprintf(g_wt_err, sizeof g_wt_err, "%s: %s", #call, cudaGetErrorString(_s));                   \
      cudaGetLastError();                                                                             \
      return -3;                                                                                      \
    }                                                                                                 \
  } while (0)

namespace kgx_wt {

// device scratch that lives for one call: freed on every return path
struct DevBufs {
  std::vector<void*> d, h;
  ~DevBufs() { for (void* p : d) cudaFree(p); for (void* p : h) cudaFreeHost(p); }
  template <class T> int dev(T** p, size_t n) {
    if (cudaMalloc((void**)p, n ? n : 1) != cudaSuccess) {
      snprintf(g_wt_err, sizeof g_wt_err, "cudaMalloc(%zu bytes): %s", n, cudaGetErrorString(cudaGetLastError()));
      return -3;
    }
    d.push_back(*p);
    return 0;
  }
  template <class T> int host(T** p, size_t n) {
    if (cudaHostAlloc((void**)p, n ? n : 1, cudaHostAllocDefault) != cudaSuccess) {
      snprintf(g_wt_err, sizeof g_wt_err, "cudaHostAlloc(%zu bytes): %s", n, cudaGetErrorString(cudaGetLastError()));
      return -3;
    }
    h.push_back(*p);
    return 0;
  }
};

static int set_device(int dev) {
  int cnt = 0;
  cudaError_t s = cudaGetDeviceCount(&cnt);
  if (s != cudaSuccess || cnt == 0) {
    snprintf(g_wt_err, sizeof g_wt_err, "no CUDA device (%s)", cudaGetErrorString(s));
    cudaGetLastError();
    return -3;
  }
  WT_CK(cudaSetDevice(dev));
  return 0;
}

// n public keys (8 limbs each: x, y) -> *ok = all on the curve.  With K: K (n x 16 words on the device) = key - start*G, and
// kinfs (device) and hinf (host, when given) = K is the point at infinity.  herd_kernel makes odd slots wild, so key k is
// computed in slot 2k + 1.
static int keys_setup(DevBufs& B, const uint64_t* keys, uint32_t n, const uint64_t rs[4], cudaStream_t st, int* ok, u32** K = nullptr,
                      int** kinfs = nullptr, std::vector<int>* hinf = nullptr) {
  u32 *dKeys, *tab, *scal, *px, *py;
  uint16_t* tg;
  int* dOk;
  if (B.dev(&dKeys, 64ull * n) || B.dev(&dOk, 4)) return -3;
  const int one = 1;
  WT_CK(cudaMemcpyAsync(dKeys, keys, 64ull * n, cudaMemcpyHostToDevice, st));
  WT_CK(cudaMemcpyAsync(dOk, &one, 4, cudaMemcpyHostToDevice, st));
  wt_on_curve_kernel<<<(n + 127) / 128, 128, 0, st>>>(dKeys, n, dOk);
  WT_CK(cudaGetLastError());
  WT_CK(cudaMemcpyAsync(ok, dOk, 4, cudaMemcpyDeviceToHost, st));
  WT_CK(cudaStreamSynchronize(st));
  if (!K || !*ok) return 0;
  if (B.dev(&tab, 256 * 16 * 4) || B.dev(&scal, 64ull * n) || B.dev(&px, 64ull * n) || B.dev(&py, 64ull * n) || B.dev(&tg, 4ull * n) ||
      B.dev(K, 64ull * n) || B.dev(kinfs, 4ull * n))
    return -3;
  using kgx::kOrderHost;
  u64 a[4], s[4] = {0, 0, 0, 0};
  memcpy(a, rs, 32);
  if (kgx::ge256(a, kOrderHost)) kgx::sub256(a, a, kOrderHost);
  if (a[0] | a[1] | a[2] | a[3]) kgx::sub256(s, kOrderHost, a);
  std::vector<uint64_t> hs(8ull * n);
  std::vector<uint16_t> ht(2ull * n);
  for (uint32_t k = 0; k < n; k++) {
    memcpy(&hs[8ull * k], s, 32); memcpy(&hs[8ull * k + 4], s, 32);
    ht[2 * k] = ht[2 * k + 1] = (uint16_t)k;
  }
  WT_CK(cudaMemcpyAsync(scal, hs.data(), 64ull * n, cudaMemcpyHostToDevice, st));
  WT_CK(cudaMemcpyAsync(tg, ht.data(), 4ull * n, cudaMemcpyHostToDevice, st));
  kgx::herd_table_kernel<<<1, 32, 0, st>>>(tab);
  kgx::herd_kernel<<<(2 * n + 127) / 128, 128, 0, st>>>(tab, scal, dKeys, tg, 0, 2ull * n, px, py, 0, nullptr);
  WT_CK(cudaGetLastError());
  std::vector<uint32_t> hx(16ull * n), hy(16ull * n), hk(16ull * n);
  std::vector<int> own;
  std::vector<int>& inf = hinf ? *hinf : own;
  inf.assign(n, 0);
  WT_CK(cudaMemcpyAsync(hx.data(), px, 64ull * n, cudaMemcpyDeviceToHost, st));
  WT_CK(cudaMemcpyAsync(hy.data(), py, 64ull * n, cudaMemcpyDeviceToHost, st));
  WT_CK(cudaStreamSynchronize(st));
  for (uint32_t k = 0; k < n; k++) {
    bool z = true;
    for (int w = 0; w < 8; w++) {
      hk[16ull * k + w] = hx[16ull * k + 8 + w];
      hk[16ull * k + 8 + w] = hy[16ull * k + 8 + w];
      z = z && hk[16ull * k + w] == 0 && hk[16ull * k + 8 + w] == 0;
    }
    inf[k] = z;                                         // herd_kernel stores the point at infinity as (0, 0)
  }
  WT_CK(cudaMemcpyAsync(*K, hk.data(), 64ull * n, cudaMemcpyHostToDevice, st));
  WT_CK(cudaMemcpyAsync(*kinfs, inf.data(), 4ull * n, cudaMemcpyHostToDevice, st));
  WT_CK(cudaStreamSynchronize(st));
  return 0;
}

static int build_comb(DevBufs& B, u32** comb, cudaStream_t st) {
  if (B.dev(comb, COMB_WORDS * 4)) return -3;
  wt_comb_kernel<<<1, 32, 0, st>>>(*comb);
  WT_CK(cudaGetLastError());
  return 0;
}

static unsigned check_blocks(uint64_t n) { return (unsigned)((n + CHECK_THREADS * GROUP - 1) / (CHECK_THREADS * GROUP)); }

// wt_find_key's index of n keys (hk: 16 words per key, x then y, by index): *kx = their x in ascending order, equal x in input
// order, *ki = the key indices in that order, both on the device; order (host) = the same indices
static int key_index(DevBufs& B, const std::vector<uint32_t>& hk, uint32_t n, u32** kx, uint32_t** ki, std::vector<uint32_t>& order) {
  order.resize(n);
  for (uint32_t k = 0; k < n; k++) order[k] = k;
  auto less = [&hk](uint32_t a, uint32_t b) {
    for (int w = 7; w >= 0; w--) if (hk[16ull * a + w] != hk[16ull * b + w]) return hk[16ull * a + w] < hk[16ull * b + w];
    return false;
  };
  std::stable_sort(order.begin(), order.end(), less);
  std::vector<uint32_t> sx(8ull * n);
  for (uint32_t j = 0; j < n; j++) memcpy(&sx[8ull * j], &hk[16ull * order[j]], 32);
  if (B.dev(kx, 32ull * n) || B.dev(ki, 4ull * n)) return -3;
  WT_CK(cudaMemcpy(*kx, sx.data(), 32ull * n, cudaMemcpyHostToDevice));
  WT_CK(cudaMemcpy(*ki, order.data(), 4ull * n, cudaMemcpyHostToDevice));
  return 0;
}

// (a + b) mod n and (a - b) mod n for a, b < n
static void add_mod_n(u64* r, const u64* a, const u64* b) {
  if (kgx::add256(r, a, b) || kgx::ge256(r, kgx::kOrderHost)) kgx::sub256(r, r, kgx::kOrderHost);
}
static void sub_mod_n(u64* r, const u64* a, const u64* b) {
  u64 t[4];
  if (kgx::sub256(t, a, b)) kgx::add256(t, t, kgx::kOrderHost);
  memcpy(r, t, 32);
}

// *bad = the first key k with solved[k] whose priv[k] * G is not its public key (x, y: keys, 8 limbs per key), or -1; herd_kernel
// makes even slots tame, so the j-th solved key is computed in slot 2j
static int privs_check(DevBufs& B, const std::vector<uint64_t>& keys, const std::vector<uint8_t>& solved, const std::vector<uint64_t>& privs,
                       uint32_t n, int64_t* bad) {
  *bad = -1;
  std::vector<uint32_t> sel;
  for (uint32_t k = 0; k < n; k++) if (solved[k]) sel.push_back(k);
  if (sel.empty()) return 0;
  const uint64_t m = sel.size();
  u32 *tab, *scal, *px, *py;
  if (B.dev(&tab, 256 * 16 * 4) || B.dev(&scal, 64 * m) || B.dev(&px, 64 * m) || B.dev(&py, 64 * m)) return -3;
  std::vector<uint64_t> hs(8 * m, 0);
  for (uint64_t j = 0; j < m; j++) memcpy(&hs[8 * j], &privs[4ull * sel[j]], 32);
  WT_CK(cudaMemcpy(scal, hs.data(), 64 * m, cudaMemcpyHostToDevice));
  kgx::herd_table_kernel<<<1, 32>>>(tab);
  kgx::herd_kernel<<<(unsigned)((2 * m + 127) / 128), 128>>>(tab, scal, tab, nullptr, 0, 2 * m, px, py, 0, nullptr);
  WT_CK(cudaGetLastError());
  std::vector<uint64_t> hx(8 * m), hy(8 * m);
  WT_CK(cudaMemcpy(hx.data(), px, 64 * m, cudaMemcpyDeviceToHost));
  WT_CK(cudaMemcpy(hy.data(), py, 64 * m, cudaMemcpyDeviceToHost));
  for (uint64_t j = 0; j < m && *bad < 0; j++)
    if (memcmp(&hx[8 * j], &keys[8ull * sel[j]], 32) || memcmp(&hy[8 * j], &keys[8ull * sel[j] + 4], 32)) *bad = sel[j];
  return 0;
}

// Input i of a merge, checked before anything is written (Merge.cpp:56-143): opened into fs[i], positioned after its header
// hd[i], and refused when it is of the other kind (a batch work file in a plain merge, a plain one in a batch merge), of
// another version than the first input, with its key off the curve (a plain merge; a batch merge checks its block's keys) or
// of another range.  *nk: its key count (a batch merge).
static int merge_input(DevBufs& B, const char* const* paths, uint32_t i, bool batch, std::vector<FILE*>& fs,
                       std::vector<kgx_wf::WorkHeader>& hd, uint32_t* nk) {
  errno = 0;
  fs[i] = fopen(paths[i], "rb");
  if (!fs[i]) { const int e = kgx_wf::io_error(); snprintf(g_wt_err, sizeof g_wt_err, "%s: %s", paths[i], strerror(-e)); return e; }
  setvbuf(fs[i], nullptr, _IOFBF, 1 << 22);
  if (!kgx_wf::read_header(fs[i], hd[i])) { snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: %s is not a HEADW work file", paths[i]); return -1; }
  *nk = 0;
  const int bf = kgx_batch_read(paths[i], nk, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
  if (batch && bf < 0) return bf;
  if (batch && bf == 0) {
    snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: %s is a plain HEADW work file: batch work files merge only with batch work files", paths[i]);
    return -1;
  }
  if (!batch && bf == 1) {
    snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: %s is a batch work file (%u keys): merging batch files is not supported", paths[i], *nk);
    return -1;
  }
  if (hd[i].version != hd[0].version) { snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: cannot merge workfile of different version (%s)", paths[i]); return -1; }
  if (!batch) {
    uint64_t key[8];
    memcpy(key, hd[i].kx, 32); memcpy(key + 4, hd[i].ky, 32);
    int ok = 0;
    if (keys_setup(B, key, 1, hd[i].rs, 0, &ok)) return -3;
    if (!ok) { snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: key of %s does not lie on elliptic curve", paths[i]); return -1; }
  }
  if (memcmp(hd[i].rs, hd[0].rs, 32) || memcmp(hd[i].re, hd[0].re, 32)) {
    snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: File range differs (%s, %s)", paths[0], paths[i]);
    return -1;
  }
  return 0;
}

// The merge proper, after every input was checked (fs: the inputs, positioned after their headers hd): writes tmp_path (the
// header, the merged table, a kangaroo count of 0, then whatever tail(out) writes) and fills info but n_listed.  on_coll(n, dColl)
// gets each block's n > 0 collisions on the device (legacy default stream), before the next block is read; its nonzero
// result ends the merge with that code.  On failure tmp_path is removed.
template <class OnColl, class Tail>
static int merge_stream(DevBufs& B, std::vector<FILE*>& fs, const char* const* paths, const std::vector<kgx_wf::WorkHeader>& hd,
                        uint32_t n_paths, const char* tmp_path, uint64_t block_entries, kgx_work_merge_info* info, OnColl on_coll,
                        Tail tail) {
  const uint64_t C = block_entries;
  Entry *hIn, *dIn, *dOut, *hOut;
  uint32_t *hH, *dH, *idxA, *idxB, *dNsel, *dNb, *hNb;
  uint64_t *keyA, *keyB;
  uint8_t* keep;
  MergeRes* dRes;
  Coll* dColl;
  size_t tC = 0;
  WT_CK(cub::DeviceSelect::Flagged(nullptr, tC, (uint32_t*)nullptr, (uint8_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)C));
  const size_t tmpBytes = std::max(kgx_wf::bucket_sort_scratch(C), tC);
  void* dTmp;
  if (B.host(&hIn, 32 * C) || B.dev(&dIn, 32 * C) || B.dev(&dOut, 32 * C) || B.host(&hOut, 32 * C) || B.host(&hH, 4 * C) ||
      B.dev(&dH, 4 * C) || B.dev(&idxA, 4 * C) || B.dev(&idxB, 4 * C) || B.dev(&dNsel, 4) || B.dev(&dNb, 4ull * NBUCKET) ||
      B.host(&hNb, 4ull * NBUCKET) || B.dev(&keyA, 8 * C) || B.dev(&keyB, 8 * C) || B.dev(&keep, C) || B.dev(&dRes, sizeof(MergeRes)) ||
      B.dev(&dColl, sizeof(Coll) * C) || B.dev(&dTmp, tmpBytes))
    return -3;
  errno = 0;
  FILE* out = fopen(tmp_path, "wb");
  if (!out) { const int e = kgx_wf::io_error(); snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: Cannot open %s for writing: %s", tmp_path, strerror(-e)); return e; }
  setvbuf(out, nullptr, _IOFBF, 1 << 22);
  kgx_wf::WorkHeader oh = hd[0];                      // the first input's range and key, written as version 0
  oh.count = 0;
  oh.time = 0;
  for (uint32_t i = 0; i < n_paths; i++) { oh.dp = std::min(oh.dp, hd[i].dp); oh.count += hd[i].count; oh.time += hd[i].time; }
  bool okw = kgx_wf::write_header(out, oh);
  int rc = 0;
  uint64_t fill = 0;
  uint32_t b0 = 0;
  // one block: entries of buckets [b0, b1) in hIn (bucket by bucket, inputs in order within a bucket) -> the merged buckets
  auto flush = [&](uint32_t b1) -> int {
    const uint32_t n = (uint32_t)fill, T = 256, G = (n + T - 1) / T;
    WT_CK(cudaMemsetAsync(dNb, 0, 4ull * (b1 - b0)));
    if (n) {
      WT_CK(cudaMemcpyAsync(dIn, hIn, 32ull * n, cudaMemcpyHostToDevice));
      WT_CK(cudaMemcpyAsync(dH, hH, 4ull * n, cudaMemcpyHostToDevice));
      WT_CK(cudaMemsetAsync(dRes, 0, sizeof(MergeRes)));
      uint32_t* ord;                                    // the legacy default stream, as every other call of the merge
      WT_CK(kgx_wf::bucket_sort(dIn, dH, nullptr, n, b0, b1, idxA, idxB, keyA, keyB, dTmp, tmpBytes, 0, &ord));
      wt_merge_scan<<<G, T>>>(dIn, dH, ord, n, b0, keep, dNb, dRes, dColl);
      size_t tb = tmpBytes;
      WT_CK(cub::DeviceSelect::Flagged(dTmp, tb, ord, keep, idxA, dNsel, (int)n));
      WT_CK(cudaGetLastError());
      MergeRes r;
      uint32_t nk = 0;
      WT_CK(cudaMemcpy(&r, dRes, sizeof r, cudaMemcpyDeviceToHost));
      WT_CK(cudaMemcpy(&nk, dNsel, 4, cudaMemcpyDeviceToHost));
      kgx_wf::bucket_gather<<<(nk + T - 1) / T, T>>>(dIn, idxA, nk, dOut);
      WT_CK(cudaGetLastError());
      WT_CK(cudaMemcpy(hOut, dOut, 32ull * nk, cudaMemcpyDeviceToHost));
      WT_CK(cudaMemcpy(hNb, dNb, 4ull * (b1 - b0), cudaMemcpyDeviceToHost));
      info->duplicates += r.dup;
      info->collisions += r.ncoll;
      if (r.ncoll) {
        const int e = on_coll((uint32_t)r.ncoll, dColl);
        if (e) return e;
      }
    } else {
      memset(hNb, 0, 4ull * (b1 - b0));
    }
    uint64_t off = 0;
    for (uint32_t b = b0; okw && b < b1; b++) {
      const uint32_t nb = hNb[b - b0];
      okw = kgx_wf::write_bucket(out, nb, (nb + 3) & ~3u, hOut + off);
      off += nb;
      info->entries += nb;
    }
    info->blocks++;
    b0 = b1;
    fill = 0;
    return 0;
  };
  std::vector<uint32_t> nbs(n_paths);
  for (uint32_t h = 0; rc == 0 && okw && h < NBUCKET; h++) {
    uint64_t sum = 0;
    for (uint32_t i = 0; i < n_paths; i++) {
      uint32_t mx;
      if (!kgx_wf::read_bucket_head(fs[i], nbs[i], mx)) {
        snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: the table of %s is cut short", paths[i]);
        rc = -1;
        break;
      }
      sum += nbs[i];
    }
    if (rc) break;
    if (sum > C) {
      snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: bucket %u holds %llu entries over the inputs, more than a merge block (%llu)", h,
               (unsigned long long)sum, (unsigned long long)C);
      rc = -1;
      break;
    }
    if (fill + sum > C && (rc = flush(h)) != 0) break;
    for (uint32_t i = 0; i < n_paths && rc == 0; i++) {
      if (nbs[i] && fread(hIn + fill, 32, nbs[i], fs[i]) != nbs[i]) {
        snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: the table of %s is cut short", paths[i]);
        rc = -1;
      }
      for (uint32_t q = 0; q < nbs[i]; q++) hH[fill + q] = h;
      fill += nbs[i];
    }
  }
  if (rc == 0 && okw) rc = flush(NBUCKET);
  const uint64_t zero = 0;                              // the kangaroo count: 0, so that loaders of -ws files take the result
  okw = okw && fwrite(&zero, 8, 1, out) == 1;
  okw = okw && tail(out);
  okw = fflush(out) == 0 && okw;
  const int ioerr = kgx_wf::io_error();
  okw = (fclose(out) == 0) && okw;
  if (rc == 0 && !okw) { snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: %s: %s", tmp_path, strerror(-ioerr)); rc = ioerr; }
  if (rc) { remove(tmp_path); return rc; }
  info->dp_bits = oh.dp;
  info->total_count = oh.count;
  info->total_time = oh.time;
  return 0;
}


}  // namespace kgx_wt

extern "C" {

const char* kgx_work_last_error(void) { return g_wt_err; }

int kgx_work_comb(int dev, uint64_t* out) {
  using namespace kgx_wt;
  if (set_device(dev)) return -3;
  DevBufs B;
  u32* comb;
  if (build_comb(B, &comb, 0)) return -3;
  WT_CK(cudaMemcpy(out, comb, COMB_WORDS * 4, cudaMemcpyDeviceToHost));
  return 0;
}

int kgx_work_check_records(int dev, int walks, const void* recs, const uint32_t* hs, uint64_t n, const uint64_t keyx[4],
                           const uint64_t keyy[4], const uint64_t range_start[4], uint8_t* out) {
  using namespace kgx_wt;
  if (set_device(dev)) return -3;
  DevBufs B;
  uint64_t key[8];
  memcpy(key, keyx, 32); memcpy(key + 4, keyy, 32);
  int ok = 0, *Kinfs;
  u32 *K, *comb;
  std::vector<int> kinf;
  if (keys_setup(B, key, 1, range_start, 0, &ok, &K, &Kinfs, &kinf)) return -3;
  if (!ok) { snprintf(g_wt_err, sizeof g_wt_err, "kgx_work_check_records: the key does not lie on the curve"); return -1; }
  if (build_comb(B, &comb, 0)) return -3;
  if (n == 0) return 0;
  uint8_t *dRes, *dBad;
  ull* cnt;
  void* dRec;
  if (B.dev(&dRec, n * (walks ? 96 : 32)) || B.dev(&dRes, n) || B.dev(&dBad, n) || B.dev(&cnt, 24)) return -3;
  WT_CK(cudaMemcpy(dRec, recs, n * (walks ? 96 : 32), cudaMemcpyHostToDevice));
  WT_CK(cudaMemset(cnt, 0, 24));
  if (walks) {
    wt_check_walks_kernel<<<(unsigned)std::min<uint64_t>((n + 127) / 128, 4096), 128>>>(comb, (const u32*)dRec, n, K, Kinfs, nullptr, dRes,
                                                                                         dBad, cnt);
  } else {
    uint32_t* dH;
    if (B.dev(&dH, 4 * n)) return -3;
    WT_CK(cudaMemcpy(dH, hs, 4 * n, cudaMemcpyHostToDevice));
    wt_check_entries_kernel<<<check_blocks(n), CHECK_THREADS>>>(comb, EntryCheck{(const Entry*)dRec, dH, dBad, cnt}, n, K, kinf[0]);
  }
  WT_CK(cudaGetLastError());
  WT_CK(cudaMemcpy(out, walks ? dRes : dBad, n, cudaMemcpyDeviceToHost));
  return 0;
}

int kgx_work_check(int dev, const char* path, uint64_t chunk, kgx_work_check_info* info, uint32_t* wrong_entries, uint64_t* wrong_walks,
                   uint32_t cap) {
  using namespace kgx_wt;
  memset(info, 0, sizeof *info);
  if (set_device(dev)) return -3;
  if (chunk == 0) chunk = DEFAULT_CHUNK;
  if (chunk >= 0x40000000ull) { snprintf(g_wt_err, sizeof g_wt_err, "kgx_work_check: chunk of %llu entries (at most 2^30-1)", (unsigned long long)chunk); return -1; }
  errno = 0;
  FILE* f = fopen(path, "rb");
  if (!f) { const int e = kgx_wf::io_error(); snprintf(g_wt_err, sizeof g_wt_err, "%s: %s", path, strerror(-e)); return e; }
  struct Closer { FILE* f; ~Closer() { fclose(f); } } closer{f};
  setvbuf(f, nullptr, _IOFBF, 1 << 22);
  kgx_wf::WorkHeader hd;
  if (!kgx_wf::read_header(f, hd)) { snprintf(g_wt_err, sizeof g_wt_err, "%s is not a HEADW work file", path); return -1; }
  info->dp_bits = hd.dp;
  DevBufs B;
  cudaStream_t st;
  WT_CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  struct StreamGuard { cudaStream_t s; ~StreamGuard() { cudaStreamSynchronize(s); cudaStreamDestroy(s); } } sg{st};
  // the file's keys: the header key, or every key of a batch file's block, with every kangaroo's target
  uint64_t hkey[8];
  memcpy(hkey, hd.kx, 32); memcpy(hkey + 4, hd.ky, 32);
  kgx_wf::BatchInfo bi;
  std::vector<uint64_t> bkeys;
  std::vector<uint16_t> btg;
  char berr[256] = "";
  FILE* g = fopen(path, "rb");
  if (!g) { const int e = kgx_wf::io_error(); snprintf(g_wt_err, sizeof g_wt_err, "%s: %s", path, strerror(-e)); return e; }
  int bf = kgx_wf::batch_find(g, bi, berr, sizeof berr);
  if (bf == 1) {
    bkeys.resize(8ull * bi.n_keys);
    btg.resize(bi.nb_walk);
    if (kgx_wf::batch_read(g, bi, bkeys.data(), nullptr, nullptr, btg.data(), berr, sizeof berr)) bf = -1;
  }
  fclose(g);
  const bool batch = bf == 1;
  // the header key is checked first, a batch file's too; a damaged batch block is reported after it
  int ok = 0, *Kinfs;
  u32 *K, *comb;
  std::vector<int> kinf;
  if (keys_setup(B, hkey, 1, hd.rs, st, &ok, batch ? nullptr : &K, &Kinfs, &kinf)) return -3;
  if (!ok) { snprintf(g_wt_err, sizeof g_wt_err, "CheckWorkFile: key1 does not lie on elliptic curve"); return -1; }
  if (bf < 0) { snprintf(g_wt_err, sizeof g_wt_err, "%s: %s", path, berr); return -1; }
  if (batch) {
    if (keys_setup(B, bkeys.data(), bi.n_keys, hd.rs, st, &ok, &K, &Kinfs, &kinf)) return -3;
    if (!ok) { snprintf(g_wt_err, sizeof g_wt_err, "CheckWorkFile: a key of the batch block does not lie on elliptic curve"); return -1; }
    info->n_keys = bi.n_keys;
  }
  if (build_comb(B, &comb, st)) return -3;
  // two buffers: the host fills one from disk while the device checks the other
  const uint64_t wchunk = chunk / 3 ? chunk / 3 : 1;    // walks per chunk: 96-byte records in the 32-byte entries' room
  Entry *hEnt[2], *dEnt[2];
  uint32_t *hH[2], *dH[2], *dSel[2], *hSel[2], *dNsel[2], *hNsel[2];
  uint8_t *dBad[2], *dRes[2];
  uint16_t* dTg[2] = {nullptr, nullptr};
  ull *dCnt[2], *hCnt[2];
  std::vector<uint32_t> hIdx[2];
  size_t selTmp = 0;
  void* dTmp[2];
  WT_CK(cub::DeviceSelect::Flagged(nullptr, selTmp, thrust::counting_iterator<uint32_t>(0), (uint8_t*)nullptr, (uint32_t*)nullptr,
                                   (uint32_t*)nullptr, (int)chunk));
  cudaEvent_t done[2];
  for (int b = 0; b < 2; b++) {
    if (B.host(&hEnt[b], 32 * chunk) || B.dev(&dEnt[b], 32 * chunk) || B.host(&hH[b], 4 * chunk) || B.dev(&dH[b], 4 * chunk) ||
        B.dev(&dBad[b], chunk) || B.dev(&dRes[b], chunk) || B.dev(&dNsel[b], 4) ||
        B.host(&hSel[b], 4ull * (cap + 1)) || B.host(&hNsel[b], 4) || B.dev(&dCnt[b], 24) || B.host(&hCnt[b], 24) ||
        B.dev(&dTmp[b], selTmp) || B.dev(&dSel[b], 4 * chunk) || (batch && B.dev(&dTg[b], 2 * wchunk)))
      return -3;
    hIdx[b].resize(chunk);
    WT_CK(cudaEventCreateWithFlags(&done[b], cudaEventDisableTiming));
  }
  struct EvGuard { cudaEvent_t* e; ~EvGuard() { cudaEventDestroy(e[0]); cudaEventDestroy(e[1]); } } eg{done};
  uint64_t pending_n[2] = {0, 0}, pending_first[2] = {0, 0};
  int pending_kind[2] = {-1, -1};
  uint32_t nwe = 0, nww = 0;
  auto submit = [&](int b, int kind, uint64_t n, uint64_t first) -> int {
    WT_CK(cudaMemsetAsync(dCnt[b], 0, 24, st));
    if (kind == 0) {
      WT_CK(cudaMemcpyAsync(dEnt[b], hEnt[b], 32 * n, cudaMemcpyHostToDevice, st));
      WT_CK(cudaMemcpyAsync(dH[b], hH[b], 4 * n, cudaMemcpyHostToDevice, st));
      if (batch)
        wt_check_entries_multi_kernel<<<(unsigned)((n + CHECK_THREADS - 1) / CHECK_THREADS), CHECK_THREADS, 0, st>>>(
            comb, dEnt[b], dH[b], n, K, Kinfs, bi.n_keys, dBad[b], dCnt[b]);
      else
        wt_check_entries_kernel<<<check_blocks(n), CHECK_THREADS, 0, st>>>(comb, EntryCheck{dEnt[b], dH[b], dBad[b], dCnt[b]}, n, K, kinf[0]);
    } else {
      WT_CK(cudaMemcpyAsync(dEnt[b], hEnt[b], 96 * n, cudaMemcpyHostToDevice, st));
      if (batch) WT_CK(cudaMemcpyAsync(dTg[b], btg.data() + first, 2 * n, cudaMemcpyHostToDevice, st));
      wt_check_walks_kernel<<<(unsigned)std::min<uint64_t>((n + 127) / 128, 4096), 128, 0, st>>>(comb, (const u32*)dEnt[b], n, K, Kinfs,
                                                                                                   dTg[b], dRes[b], dBad[b], dCnt[b]);
    }
    WT_CK(cudaGetLastError());
    size_t tb = selTmp;
    WT_CK(cub::DeviceSelect::Flagged(dTmp[b], tb, thrust::counting_iterator<uint32_t>(0), dBad[b], dSel[b], dNsel[b], (int)n, st));
    WT_CK(cudaMemcpyAsync(hNsel[b], dNsel[b], 4, cudaMemcpyDeviceToHost, st));
    if (cap) WT_CK(cudaMemcpyAsync(hSel[b], dSel[b], 4ull * std::min<uint64_t>(cap, n), cudaMemcpyDeviceToHost, st));
    WT_CK(cudaMemcpyAsync(hCnt[b], dCnt[b], 24, cudaMemcpyDeviceToHost, st));
    WT_CK(cudaEventRecord(done[b], st));
    pending_n[b] = n; pending_kind[b] = kind; pending_first[b] = first;
    return 0;
  };
  auto drain = [&](int b) -> int {                     // wait for buffer b's chunk and count it
    if (pending_kind[b] < 0) return 0;
    WT_CK(cudaEventSynchronize(done[b]));
    const uint32_t ns = std::min<uint32_t>(*hNsel[b], cap);
    if (pending_kind[b] == 0) {
      info->entries += pending_n[b];
      info->wrong_entries += hCnt[b][0];
      for (uint32_t k = 0; k < ns && nwe < cap; k++, nwe++) {
        wrong_entries[2 * nwe] = hH[b][hSel[b][k]];
        wrong_entries[2 * nwe + 1] = hIdx[b][hSel[b][k]];
      }
    } else {
      info->walks += pending_n[b];
      info->walks_tame += hCnt[b][0];
      info->walks_wild += hCnt[b][1];
      info->wrong_walks += hCnt[b][2];
      for (uint32_t k = 0; k < ns && nww < cap; k++, nww++) wrong_walks[nww] = pending_first[b] + hSel[b][k];
    }
    pending_kind[b] = -1;
    return 0;
  };
  int cur = 0;
  uint64_t fill = 0;
  bool okr = true;
  for (uint32_t h = 0; okr && h < NBUCKET; h++) {      // HashTable::LoadTable order; buckets may span chunks
    uint32_t nb = 0, mx = 0;
    okr = kgx_wf::read_bucket_head(f, nb, mx);
    uint32_t done_in_bucket = 0;
    while (okr && done_in_bucket < nb) {
      if (fill == 0 && drain(cur)) return -3;           // the buffer is free once its previous chunk was counted
      const uint32_t k = (uint32_t)std::min<uint64_t>(nb - done_in_bucket, chunk - fill);
      okr = fread(hEnt[cur] + fill, 32, k, f) == k;
      for (uint32_t q = 0; q < k; q++) { hH[cur][fill + q] = h; hIdx[cur][fill + q] = done_in_bucket + q; }
      fill += k;
      done_in_bucket += k;
      if (fill == chunk) {
        if (submit(cur, 0, fill, 0)) return -3;
        cur ^= 1;
        fill = 0;
      }
    }
  }
  if (!okr) { snprintf(g_wt_err, sizeof g_wt_err, "%s: the table is cut short", path); return -1; }
  if (fill) {
    if (submit(cur, 0, fill, 0)) return -3;
    cur ^= 1;
    fill = 0;
  }
  uint64_t nwalk = 0;
  if (fread(&nwalk, 8, 1, f) == 1) {                    // files the reference's -wm wrote end right after the table
    info->has_walk_count = 1;
    for (uint64_t first = 0; first < nwalk;) {
      if (drain(cur)) return -3;
      const uint64_t k = std::min<uint64_t>(nwalk - first, wchunk);
      if (fread(hEnt[cur], 96, k, f) != k) { snprintf(g_wt_err, sizeof g_wt_err, "%s: the kangaroo block is cut short", path); return -1; }
      if (submit(cur, 1, k, first)) return -3;
      cur ^= 1;
      first += k;
    }
  }
  if (drain(cur) || drain(cur ^ 1)) return -3;         // the older chunk first: wrong records are listed in file order
  info->n_wrong_entries_listed = nwe;
  info->n_wrong_walks_listed = nww;
  return 0;
}

int kgx_work_merge(int dev, const char* const* paths, uint32_t n_paths, const char* tmp_path, uint64_t block_entries,
                   kgx_work_merge_info* info, kgx_work_collision* coll, uint32_t cap) {
  using namespace kgx_wt;
  memset(info, 0, sizeof *info);
  if (n_paths < 2) { snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: at least two work files are needed, %u given", n_paths); return -1; }
  if (block_entries == 0) block_entries = DEFAULT_BLOCK;
  if (block_entries >= 0x40000000ull) { snprintf(g_wt_err, sizeof g_wt_err, "kgx_work_merge: block of %llu entries (at most 2^30-1)", (unsigned long long)block_entries); return -1; }
  if (set_device(dev)) return -3;
  std::vector<FILE*> fs(n_paths, nullptr);
  struct Closer { std::vector<FILE*>& v; ~Closer() { for (FILE* f : v) if (f) fclose(f); } } closer{fs};
  std::vector<kgx_wf::WorkHeader> hd(n_paths);
  DevBufs B;
  for (uint32_t i = 0; i < n_paths; i++) {
    uint32_t nk;
    if (const int e = merge_input(B, paths, i, false, fs, hd, &nk)) return e;
    if (memcmp(hd[i].kx, hd[0].kx, 32) || memcmp(hd[i].ky, hd[0].ky, 32)) {
      snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: key differs, multiple keys not yet supported (%s, %s)", paths[0], paths[i]);
      return -1;
    }
  }
  std::vector<Coll> hColl;
  const int rc = merge_stream(
      B, fs, paths, hd, n_paths, tmp_path, block_entries, info,
      [&](uint32_t n, const Coll* dColl) -> int {
        const size_t c0 = hColl.size();
        hColl.resize(c0 + n);
        WT_CK(cudaMemcpy(hColl.data() + c0, dColl, sizeof(Coll) * n, cudaMemcpyDeviceToHost));
        std::sort(hColl.begin() + c0, hColl.end(), [](const Coll& a, const Coll& b) { return a.h != b.h ? a.h < b.h : a.seq < b.seq; });
        if (hColl.size() > cap) hColl.resize(cap);
        return 0;
      },
      [](FILE*) { return true; });
  if (rc) return rc;
  info->n_listed = (uint32_t)hColl.size();
  for (size_t k = 0; k < hColl.size(); k++) {
    coll[k].h = hColl[k].h;
    coll[k].reserved = 0;
    memcpy(coll[k].d_first, hColl[k].d_first, 16);
    memcpy(coll[k].d_other, hColl[k].d_other, 16);
  }
  return 0;
}

uint64_t kgx_batch_block_bytes(uint32_t n_keys, uint64_t nb_walk) { return kgx_wf::batch_block_bytes(n_keys, nb_walk); }

int kgx_batch_block(const uint64_t* keys, const uint8_t* solved, const uint64_t* privs, uint32_t n_keys, const uint16_t* targets,
                    uint64_t nb_walk, uint64_t offset, void* out) {
  if (n_keys == 0 || n_keys > kgx_wf::BATCH_MAX_KEYS) { snprintf(g_wt_err, sizeof g_wt_err, "kgx_batch_block: n_keys must be in [1, %u]", kgx_wf::BATCH_MAX_KEYS); return -1; }
  for (uint64_t i = 0; i < nb_walk; i++)
    if (targets[i] >= n_keys) { snprintf(g_wt_err, sizeof g_wt_err, "kgx_batch_block: target %u of kangaroo %llu is not below n_keys = %u", targets[i], (unsigned long long)i, n_keys); return -1; }
  kgx_wf::batch_encode(keys, solved, privs, n_keys, targets, nb_walk, offset, static_cast<uint8_t*>(out));
  return 0;
}

int kgx_batch_read(const char* path, uint32_t* n_keys, uint64_t* nb_walk, uint64_t* offset, uint64_t* keys, uint8_t* solved,
                   uint64_t* privs, uint16_t* targets) {
  errno = 0;
  FILE* f = fopen(path, "rb");
  if (!f) { const int e = kgx_wf::io_error(); snprintf(g_wt_err, sizeof g_wt_err, "%s: %s", path, strerror(-e)); return e; }
  kgx_wf::BatchInfo bi;
  char err[256] = "";
  int rc = kgx_wf::batch_find(f, bi, err, sizeof err);
  if (rc == 1 && (keys || solved || privs || targets) && kgx_wf::batch_read(f, bi, keys, solved, privs, targets, err, sizeof err)) rc = -1;
  fclose(f);
  if (rc < 0) { snprintf(g_wt_err, sizeof g_wt_err, "%s: %s", path, err); return -1; }
  if (n_keys) *n_keys = bi.n_keys;
  if (nb_walk) *nb_walk = bi.nb_walk;
  if (offset) *offset = bi.offset;
  return rc;
}

int kgx_work_merge_batch(int dev, const char* const* paths, uint32_t n_paths, const char* tmp_path, uint64_t block_entries,
                         kgx_work_merge_info* info, kgx_batch_merge_info* binfo, kgx_batch_key_result* keys_out, uint32_t cap_keys) {
  using namespace kgx_wt;
  memset(info, 0, sizeof *info);
  memset(binfo, 0, sizeof *binfo);
  if (n_paths < 2) { snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: at least two work files are needed, %u given", n_paths); return -1; }
  if (block_entries == 0) block_entries = DEFAULT_BLOCK;
  if (block_entries >= 0x40000000ull) { snprintf(g_wt_err, sizeof g_wt_err, "kgx_work_merge_batch: block of %llu entries (at most 2^30-1)", (unsigned long long)block_entries); return -1; }
  if (set_device(dev)) return -3;
  std::vector<FILE*> fs(n_paths, nullptr);
  struct Closer { std::vector<FILE*>& v; ~Closer() { for (FILE* f : v) if (f) fclose(f); } } closer{fs};
  std::vector<kgx_wf::WorkHeader> hd(n_paths);
  DevBufs B;
  // every input is checked before anything is written: its HEADW part, then its batch block
  uint32_t n = 0;
  std::vector<uint64_t> keys, ki, privs, pi;             // the first input's keys; privs: the union of the recorded ones
  std::vector<uint8_t> solved, si;
  for (uint32_t i = 0; i < n_paths; i++) {
    uint32_t nk;
    if (const int e = merge_input(B, paths, i, true, fs, hd, &nk)) return e;
    if (i == 0) n = nk;
    if (nk != n) { snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: %s holds %u keys, %s %u: the key lists differ", paths[i], nk, paths[0], n); return -1; }
    ki.assign(8ull * n, 0); pi.assign(4ull * n, 0); si.assign(n, 0);
    const int rb = kgx_batch_read(paths[i], nullptr, nullptr, nullptr, ki.data(), si.data(), pi.data(), nullptr);
    if (rb < 0) return rb;
    if (i == 0) { keys = ki; privs.assign(4ull * n, 0); solved.assign(n, 0); }
    for (uint32_t k = 0; k < n; k++) {
      if (memcmp(&ki[8ull * k], &keys[8ull * k], 64)) {
        snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: key #%u of %s differs from key #%u of %s: the key lists differ", k, paths[i], k, paths[0]);
        return -1;
      }
      if (!si[k]) continue;
      if (kgx::ge256(&pi[4ull * k], kgx::kOrderHost)) {
        snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: the private key of key #%u in %s is not below the group order", k, paths[i]);
        return -1;
      }
      if (solved[k] && memcmp(&pi[4ull * k], &privs[4ull * k], 32)) {
        snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: two inputs record different private keys for key #%u (%s, %s)", k, paths[i],
                 paths[0]);
        return -1;
      }
      solved[k] = 1;
      memcpy(&privs[4ull * k], &pi[4ull * k], 32);
    }
  }
  if (kgx::ge256(hd[0].rs, kgx::kOrderHost)) { snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: the range start of %s is not below the group order", paths[0]); return -1; }
  if (n > cap_keys) { snprintf(g_wt_err, sizeof g_wt_err, "kgx_work_merge_batch: %u keys, room for %u results", n, cap_keys); return -1; }
  int ok = 0;
  u32* K;
  int* kinfs;
  if (keys_setup(B, keys.data(), n, hd[0].rs, 0, &ok, &K, &kinfs)) return -3;
  if (!ok) { snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: a key of %s does not lie on elliptic curve", paths[0]); return -1; }
  int64_t bad = -1;
  if (privs_check(B, keys, solved, privs, n, &bad)) return -3;
  if (bad >= 0) { snprintf(g_wt_err, sizeof g_wt_err, "MergeWork: the private key recorded for key #%lld does not give its public key", (long long)bad); return -1; }
  // K on the host, its index on the device; keys with the same x (the same point or its negative) form one class
  std::vector<uint32_t> hk(16ull * n), order, pos(n);
  WT_CK(cudaMemcpy(hk.data(), K, 64ull * n, cudaMemcpyDeviceToHost));
  u32* kx;
  uint32_t* kidx;
  if (key_index(B, hk, n, &kx, &kidx, order)) return -3;
  for (uint32_t j = 0; j < n; j++) pos[order[j]] = j;
  std::vector<kgx_batch_key_result> res(n);
  memset(res.data(), 0, sizeof(kgx_batch_key_result) * n);
  for (uint32_t k = 0; k < n; k++)
    if (solved[k]) { res[k].status = 1; memcpy(res[k].priv, &privs[4ull * k], 32); binfo->solved_in_inputs++; }
  u32* comb;
  uint8_t* dSolved;
  ull* dCnt;
  Hit* dHits;
  const uint64_t C = block_entries;
  if (build_comb(B, &comb, 0) || B.dev(&dSolved, n) || B.dev(&dCnt, 32) || B.dev(&dHits, sizeof(Hit) * C)) return -3;
  WT_CK(cudaMemcpy(dSolved, solved.data(), n, cudaMemcpyHostToDevice));
  Start st;
  memcpy(st.v, hd[0].rs, 32);
  std::vector<Hit> hits;
  auto on_coll = [&](uint32_t nc, const Coll* dColl) -> int {
    WT_CK(cudaMemset(dCnt, 0, 32));
    wt_resolve_kernel<<<(nc + CHECK_THREADS - 1) / CHECK_THREADS, CHECK_THREADS>>>(comb, dColl, nc, kx, kidx, K, n, st, dSolved, dCnt,
                                                                                   dHits);
    WT_CK(cudaGetLastError());
    ull cnt[4];
    WT_CK(cudaMemcpy(cnt, dCnt, 32, cudaMemcpyDeviceToHost));
    binfo->same_herd += cnt[0];
    binfo->no_key += cnt[1];
    binfo->already_solved += cnt[2];
    if (!cnt[3]) return 0;
    hits.resize(cnt[3]);
    WT_CK(cudaMemcpy(hits.data(), dHits, sizeof(Hit) * cnt[3], cudaMemcpyDeviceToHost));
    std::sort(hits.begin(), hits.end(), [](const Hit& a, const Hit& b) { return a.h != b.h ? a.h < b.h : a.seq < b.seq; });
    for (const Hit& t : hits) {
      if (solved[t.key]) { binfo->already_solved++; continue; }
      binfo->solving++;
      // the hit key is the first of its class; the others get priv (the same point) or 2 * start - priv (its negative)
      u64 neg[4], s2[4];
      add_mod_n(s2, hd[0].rs, hd[0].rs);
      sub_mod_n(neg, s2, t.priv);
      for (uint32_t j = pos[t.key]; j < n && !memcmp(&hk[16ull * order[j]], &hk[16ull * t.key], 32); j++) {
        const uint32_t k = order[j];
        if (solved[k]) continue;
        solved[k] = 1;
        kgx_batch_key_result& r = res[k];
        r.status = 2;
        r.h = t.h;
        memcpy(r.priv, memcmp(&hk[16ull * k + 8], &hk[16ull * t.key + 8], 32) ? neg : t.priv, 32);
        memcpy(r.d_first, t.d_first, 16);
        memcpy(r.d_other, t.d_other, 16);
        memcpy(&privs[4ull * k], r.priv, 32);
        binfo->solved_by_merge++;
      }
    }
    WT_CK(cudaMemcpy(dSolved, solved.data(), n, cudaMemcpyHostToDevice));
    return 0;
  };
  auto tail = [&](FILE* out) -> bool {                  // the batch block: every key, no kangaroo
    const long off = ftell(out);
    if (off < 0) return false;
    std::vector<uint8_t> blk(kgx_wf::batch_block_bytes(n, 0));
    const uint16_t no_target = 0;
    kgx_wf::batch_encode(keys.data(), solved.data(), privs.data(), n, &no_target, 0, (uint64_t)off, blk.data());
    return fwrite(blk.data(), 1, blk.size(), out) == blk.size();
  };
  const int rc = merge_stream(B, fs, paths, hd, n_paths, tmp_path, block_entries, info, on_coll, tail);
  if (rc) return rc;
  binfo->n_keys = n;
  binfo->left = n - binfo->solved_in_inputs - binfo->solved_by_merge;
  memcpy(keys_out, res.data(), sizeof(kgx_batch_key_result) * n);
  return 0;
}

}  // extern "C"
