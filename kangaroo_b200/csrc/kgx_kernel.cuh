// kgx_kernel.cuh -- the kangaroo jump kernels for sm_90a (H100).
//
// Replace the reference's GPU/GPUCompute.h:22-117 (ComputeKangaroos) + comp_kangaroos (GPUEngine.cu:35-40).
// Same mathematics (SURVEY.md App. A.2), different machine mapping:
//
//   reference      : every thread owns 128 kangaroos in LOCAL memory (18.5 KB stack/thread): px/py/dx/subp arrays are
//                    re-read and re-written through L1/L2 several times per jump (~416 B/jump), three passes.
//   stream_kernel  : (default for herds >= 4e5 kangaroos, kgx_engine.cu) every thread owns G kangaroos that live in HBM as
//                    coalesced 16-byte SoA chunks; ONE fused pass per jump reads prefix/x/y and writes x'/y'/next prefix
//                    and a one-byte jump-index log entry (the distances are folded from the log at the end of the launch;
//                    ~194.5 B/jump) with the next kangaroo prefetched into a second register buffer and the pair two
//                    trips ahead pulled into L2; no barriers.  Group inverse once per G jumps: the 32 lane products of a warp
//                    are multiplied by a shuffle butterfly and ONE warp-uniform safegcd inverse serves 32*G kangaroos
//                    (WARPINV), or every thread inverts its own product (short groups).
//   jump_kernel    : (resident; default for small herds) a CTA of T threads owns a tile of T*K kangaroos whose whole
//                    state stays in SHARED memory for all NB_RUN jumps of a launch (HBM 2.5 B/jump).  The batch inverse
//                    spans the tile: per-thread chains -> per-lane chains across the warps -> XOR-butterfly product over
//                    the 32 lanes with warp shuffles -> ONE warp-uniform inverse per tile per jump -> back down the tree;
//                    several CTAs per SM overlap one tile's serial inverse with another's parallel phase.
//   jump_kernel_cluster : (opt-in) the resident kernel with one 1792-kangaroo tile spread over the shared memory of a 2-CTA
//                    thread-block cluster; one inverse per tile through distributed shared memory.
//   SYM instantiations of the first two add the reference's USE_SYMMETRY paths (class switch + lastJump / symClass rule).
//
//   All three make the same fused per-kangaroo pass: back-substitution of this jump's inverse, the affine add (one copy:
//   kangaroo_jump), the distance update, the DP test, and the *next* jump's dx / prefix product (next_dx; accumulated in
//   the order of this pass, consumed in reverse by the next): 5 ModMult + 1 ModSqr + 7 ModSub per jump.  The two tile
//   kernels are one body (tile_body) that differs only in rows per CTA and the inverse step, and every group inverse uses
//   the same lane butterfly (butterfly_up / butterfly_down).  DESIGN.md 3 has the measurements.
#pragma once
#include "kgx_field.cuh"
#include "kgx_modinv.h"
#include <cooperative_groups.h>

namespace kgx {

constexpr int CHUNKS = 5;         // 16-byte chunks per kangaroo in HBM: x0 x1 y0 y1 d
constexpr int JT_WORDS = 20 * 32; // jump table as uint4 jt[5][32] = {jpx lo, jpx hi, jpy lo, jpy hi, jd} x 32 jumps: one LDS.128 per half element

// Tile geometry of one CTA: T threads (W = T/32 warps), K kangaroos per thread.  Shared memory (uint4 units):
//   X[K][2][T] Y[K][2][T] P[K][2][T] D[K][T] TOT[2][T] then the jump table (u32 view), then the symmetric mode's state
//   bytes [K][T] (the cluster kernel's CfgCl puts its exchange slots there instead).
template <int T_, int K_>
struct Cfg {
  static constexpr int T = T_, K = K_, W = T_ / 32, TILE = T_ * K_;
  static constexpr int S_X = 0;
  static constexpr int S_Y = S_X + K * 2 * T;
  static constexpr int S_P = S_Y + K * 2 * T;
  static constexpr int S_D = S_P + K * 2 * T;
  static constexpr int S_TOT = S_D + K * T;
  static constexpr int S_JT = S_TOT + 2 * T;
  static constexpr int LJ_OFF = S_JT * 16 + JT_WORDS * 4;          // symmetric mode: lastJump bytes [K][T]
  static constexpr int SMEM_BYTES = LJ_OFF + K * T;
  static constexpr int CTAS_PER_SM = (227 * 1024) / (SMEM_BYTES + 1024);
};

struct LaunchParams {
  uint4* state;          // [numTiles][K][CHUNKS][T]
  const u32* jtab;       // JT_WORDS words
  u32* out;              // DP slab: [count][maxFound * 14 words]
  u64 dpMask;
  u64 nKangaroos;        // real (unpadded) count: DPs of padding slots are dropped
  u32 numTiles;
  u32 maxFound;
  int nRun;
  uint4* pre;            // streaming kernel only: prefix-product scratch [numTiles][G][2][T]
  int G;                 // streaming kernel only: kangaroos per thread (even, chosen by the engine from the herd size)
  uint8_t* aux;          // symmetric mode only: one state byte per kangaroo, [numTiles][G or K][T] (see jump_index)
  int symRule;           // KGX_SYM_LASTJUMP / KGX_SYM_CLASS
  int pfDist;            // stream kernel: L2 prefetch distance in kangaroos (0 = off; KGX_STREAM_PF)
  uint8_t* jlog;         // stream kernel only: jump-index log [numTiles][LOG_RUNS][G][T] (see stream_fold)
  unsigned long long* prof;   // optional: [0]=sum serial cycles, [1]=sum modinv cycles, [2]=sum parallel cycles, [3]=tile-steps (warp 0 of every CTA)
};

__device__ __forceinline__ void lds_fe(u32* r, const uint4* base, int idx0, int idx1) {
  uint4 a = base[idx0], b = base[idx1];
  r[0] = a.x; r[1] = a.y; r[2] = a.z; r[3] = a.w; r[4] = b.x; r[5] = b.y; r[6] = b.z; r[7] = b.w;
}
__device__ __forceinline__ void sts_fe(uint4* base, int idx0, int idx1, const u32* r) {
  base[idx0] = make_uint4(r[0], r[1], r[2], r[3]);
  base[idx1] = make_uint4(r[4], r[5], r[6], r[7]);
}
__device__ __forceinline__ void unpack8(u32* r, const uint4& a, const uint4& b) {
  r[0] = a.x; r[1] = a.y; r[2] = a.z; r[3] = a.w; r[4] = b.x; r[5] = b.y; r[6] = b.z; r[7] = b.w;
}
// one half (4 limbs) of a jump-table element per LDS.128: tab[j] = low half, tab[32 + j] = high half
__device__ __forceinline__ void lds_jp4(u32* r, const uint4* tab, u32 j) {
  const uint4 a = tab[j], b = tab[32 + j];
  r[0] = a.x; r[1] = a.y; r[2] = a.z; r[3] = a.w; r[4] = b.x; r[5] = b.y; r[6] = b.z; r[7] = b.w;
}
__device__ __forceinline__ void shfl_xor_fe(u32* r, const u32* a, int mask) {
#pragma unroll
  for (int w = 0; w < 8; w++) r[w] = __shfl_xor_sync(0xffffffffu, a[w], mask);
}

__device__ __forceinline__ void fe_inv(u32* r, const u32* a) { modinv256(r, a); }

// USE_SYMMETRY jump selection.  The reference has TWO rules behind its compile-time switch, and the engine offers both
// (LaunchParams::symRule, one state byte per kangaroo in LaunchParams::aux):
//   KGX_SYM_LASTJUMP (1): the device rule (GPUCompute.h:53-58), which is also what Kangaroo::Check replays on the CPU
//       (Check.cpp:536-541): x mod 32, bumped by one when it repeats this kangaroo's previous jump.  aux = last jump index
//       (32 = none yet).  It only suppresses 2-cycles: on long walks kangaroos fall into longer fruitless cycles and stop
//       producing new distinguished points -- measured: the USE_SYMMETRY build does not solve in64 with it.
//   KGX_SYM_CLASS (2): the rule of the reference's working symmetric path, SolveKeyCPU (Kangaroo.cpp:381-384, 422-428):
//       x mod 16 + 16 * symClass, where symClass flips at every class switch, so that the jump taken after a negation comes
//       from the other half of the table (distances multiples of u, resp. v: Kangaroo.cpp:763-806).  aux = symClass.
#ifndef KGX_SYM_LASTJUMP
#define KGX_SYM_LASTJUMP 1
#define KGX_SYM_CLASS    2
#endif
template <bool SYM>
__device__ __forceinline__ u32 jump_index(u32 x0, u32 aux, int rule) {
  if (!SYM) return x0 & 31u;
  const u32 j0 = x0 & 31u;
  const u32 jl = (j0 == aux) ? ((aux + 1u) & 31u) : j0;
  const u32 jc = (x0 & 15u) | ((aux & 1u) << 4);
  return rule == KGX_SYM_CLASS ? jc : jl;
}
// state byte after a jump with index j that did (neg != 0) or did not switch class
__device__ __forceinline__ u32 sym_next_aux(u32 aux, u32 j, u32 neg, int rule) {
  return rule == KGX_SYM_CLASS ? ((aux ^ neg) & 1u) : j;
}

// XOR butterfly over the 32 lanes of a warp: v becomes the product of all 32 lanes' v (identical in every lane) and sib[l]
// keeps the sibling factor of round l.  butterfly_down walks it back: the inverse of that product becomes the inverse of this
// lane's own v.
__device__ __forceinline__ void butterfly_up(u32* v, u32 (*sib)[8]) {
#pragma unroll
  for (int l = 0; l < 5; l++) {
    shfl_xor_fe(sib[l], v, 1 << l);
    fe_mul(v, v, sib[l]);
  }
}
__device__ __forceinline__ void butterfly_down(u32* inv, u32 (*sib)[8]) {
#pragma unroll
  for (int l = 4; l >= 0; l--) fe_mul(inv, inv, sib[l]);
}

// Warp 0's tree over the T per-thread products in sTot.  tile_reduce: lane l chains the totals of threads {l, l+32, ...}
// (one per warp: conflict-free; c[w] = tw[0]*...*tw[w]) and the butterfly multiplies the 32 lane chains into v, the
// product of all T.  tile_walk_back takes inv = 1 / v back down the same tree and writes the T inverses to sTot.
template <int T, int W>
__device__ __forceinline__ void tile_reduce(u32* v, u32 (*tw)[8], u32 (*c)[8], u32 (*sib)[8], const uint4* sTot, int lane) {
#pragma unroll
  for (int w = 0; w < W; w++) lds_fe(tw[w], sTot, 32 * w + lane, T + 32 * w + lane);
  fe_copy(c[0], tw[0]);
#pragma unroll
  for (int w = 1; w < W; w++) fe_mul(c[w], c[w - 1], tw[w]);
  fe_copy(v, c[W - 1]);
  butterfly_up(v, sib);
}
template <int T, int W>
__device__ __forceinline__ void tile_walk_back(uint4* sTot, u32* inv, u32 (*tw)[8], u32 (*c)[8], u32 (*sib)[8], int lane) {
  butterfly_down(inv, sib);       // -> 1 / c[W-1] of this lane
#pragma unroll
  for (int w = W - 1; w >= 1; w--) {
    u32 o[8];
    fe_mul(o, inv, c[w - 1]);     // 1 / tw[w]
    sts_fe(sTot, 32 * w + lane, T + 32 * w + lane, o);
    fe_mul(inv, inv, tw[w]);      // 1 / c[w-1]
  }
  sts_fe(sTot, lane, T + lane, inv);
}

// Warp 0 only: turn the T per-thread products in sTot into their T inverses (in place) with one warp-uniform inverse.
template <int T, int W>
__device__ __noinline__ void tile_inverse(uint4* sTot, int lane, unsigned long long* prof) {
  u32 tw[W][8], c[W][8], sib[5][8], v[8], inv[8];
  tile_reduce<T, W>(v, tw, c, sib, sTot, lane);
  long long tq0 = prof ? clock64() : 0;
  fe_inv(inv, v);                 // identical in all 32 lanes
  if (prof && lane == 0) atomicAdd(prof + 1, (unsigned long long)(clock64() - tq0));
  tile_walk_back<T, W>(sTot, inv, tw, c, sib, lane);
}

// One jump of one kangaroo: the arithmetic of the fused pass that every jump kernel shares.  pre holds the product of the
// dx accumulated before this kangaroo in the pass (clobbered: it becomes 1/dx); strip takes this dx out of the running
// inverse I, which the last kangaroo of a pass can skip.  y comes as its two 16-byte halves and is read only after the
// inverse step, so that a tile kernel's shared-memory load of y does not hold 8 registers across it.  Returns (rx, ry), the jump index j and, in symmetric mode, the
// class-switch mask (all ones when the point was negated); the caller applies the jump to the distance and the state byte.
template <bool SYM>
__device__ __forceinline__ u32 kangaroo_jump(u32* rx, u32* ry, u32& j, const u32* x, const uint4& y0, const uint4& y1, u32* pre,
                                             u32* I, bool strip, u32 aux, const uint4* jt, int rule) {
  u32 y[8], jx[8], jy[8], dx[8], s[8];
  j = jump_index<SYM>(x[0], aux, rule);
  lds_jp4(jx, jt, j);
  fe_sub(dx, x, jx);
  fe_mul(pre, pre, I);                     // 1/dx
  if (strip) fe_mul(I, I, dx);             // strip this dx from the running inverse
  unpack8(y, y0, y1);
  lds_jp4(jy, jt + 64, j);
  fe_sub(s, y, jy);                        // dy
  fe_mul(s, s, pre);                       // s = dy/dx
  fe_sqr(rx, s);
  fe_sub(rx, rx, jx);
  fe_sub(rx, rx, x);                       // rx = s^2 - jx - x
  fe_sub(ry, x, rx);
  fe_mul(ry, ry, s);
  fe_sub(ry, ry, y);                       // ry = s (x - rx) - y
  if (!SYM) return 0u;
  const u32 neg = fe_gt_half_mask(ry);     // equivalence class switch (Check.cpp:551-556): y > (p-1)/2 -> (x, p - y), d -> -d
  fe_cneg(ry, neg);
  return neg;
}

// dx of the next jump of the kangaroo at x with state byte aux.
template <bool SYM>
__device__ __forceinline__ void next_dx(u32* dx, const u32* x, u32 aux, const uint4* jt, int rule) {
  u32 jx[8];
  lds_jp4(jx, jt, jump_index<SYM>(x[0], aux, rule));
  fe_sub(dx, x, jx);
}

// Tile kernels: appends dx to the chain P and stores the product of the dx before it at (i0, i1) of sP (first: a new chain).
__device__ __forceinline__ void chain_dx(uint4* sP, int i0, int i1, u32* P, const u32* dx, bool first) {
  if (first) {
    u32 one[8]; fe_set_one(one);
    sts_fe(sP, i0, i1, one);
    fe_copy(P, dx);
  } else {
    sts_fe(sP, i0, i1, P);
    fe_mul(P, P, dx);
  }
}

// DP record at position pos of the slab (GPUMath.h:173-188 layout): x (8 words), distance (4 words), kIdx (2 words).
__device__ __forceinline__ void put_dp_record(u32* out, u32 pos, const u32* x, const u32* d, u64 kidx) {
  u32* o = out + 1 + (size_t)pos * 14;
#pragma unroll
  for (int w = 0; w < 8; w++) o[w] = x[w];
  o[8] = d[0]; o[9] = d[1]; o[10] = d[2]; o[11] = d[3];
  o[12] = (u32)kidx; o[13] = (u32)(kidx >> 32);
}

// The body of both tile kernels.  A tile of CTAS * K rows of T kangaroos is spread over CTAS CTAs; this one holds rows
// rank * K .. rank * K + K - 1 in its shared memory (Cfg<T, K> layout) for all nRun jumps of the launch.  inverse(sTot, t)
// turns the T thread totals in sTot into their inverses; every thread calls it, between two barriers.
template <int T, int K, int CTAS, bool SYM, class Inverse>
__device__ __forceinline__ void tile_body(const LaunchParams& p, u32 rank, Inverse inverse) {
  using C = Cfg<T, K>;
  constexpr int TILE = T * K * CTAS;
  extern __shared__ uint4 smem[];
  uint8_t* sL = reinterpret_cast<uint8_t*>(smem) + C::LJ_OFF;
  uint4* sX = smem + C::S_X;
  uint4* sY = smem + C::S_Y;
  uint4* sP = smem + C::S_P;
  uint4* sD = smem + C::S_D;
  uint4* sTot = smem + C::S_TOT;
  uint4* jt = smem + C::S_JT;
  const int t = threadIdx.x;
  const u32 mlo = (u32)p.dpMask, mhi = (u32)(p.dpMask >> 32);

  for (int i = t; i < JT_WORDS; i += T) reinterpret_cast<u32*>(jt)[i] = p.jtab[i];

  for (u32 tile = blockIdx.x / CTAS; tile < p.numTiles; tile += gridDim.x / CTAS) {   // the CTAs of a tile walk the same tiles
    __syncthreads();   // jump table visible; previous tile's shared state fully consumed
    const u32 row0 = rank * K;   // this CTA's first row in the tile: slot tile * TILE + (row0 + g) * T + t
    uint4* gsrc = p.state + (size_t)tile * (CTAS * K * CHUNKS * T) + (size_t)row0 * (CHUNKS * T);
#pragma unroll
    for (int g = 0; g < K; g++) {
      sX[(g * 2 + 0) * T + t] = gsrc[(g * CHUNKS + 0) * T + t];
      sX[(g * 2 + 1) * T + t] = gsrc[(g * CHUNKS + 1) * T + t];
      sY[(g * 2 + 0) * T + t] = gsrc[(g * CHUNKS + 2) * T + t];
      sY[(g * 2 + 1) * T + t] = gsrc[(g * CHUNKS + 3) * T + t];
      sD[g * T + t] = gsrc[(g * CHUNKS + 4) * T + t];
      if (SYM) sL[g * T + t] = p.aux[(size_t)tile * TILE + (row0 + g) * T + t];
    }
    // prologue: forward chain of dx; sP[g] = product of the dx before g
    u32 P[8];
    {
      u32 x[8], dx[8];
#pragma unroll 1
      for (int g = 0; g < K; g++) {
        const int i0 = (g * 2) * T + t, i1 = (g * 2 + 1) * T + t;
        lds_fe(x, sX, i0, i1);
        next_dx<SYM>(dx, x, SYM ? (u32)sL[g * T + t] : 0u, jt, p.symRule);
        chain_dx(sP, i0, i1, P, dx, g == 0);
      }
      sts_fe(sTot, t, T + t, P);
    }
    int backward = 1;   // the pass after a forward accumulation consumes in reverse order
    long long tp0 = 0;

    for (int run = 0; run < p.nRun; run++) {
      long long tp1 = (p.prof && t == 0) ? clock64() : 0;
      if (p.prof && t == 0 && run > 0) atomicAdd(p.prof + 2, (unsigned long long)(tp1 - tp0));
      __syncthreads();
      long long ts0 = (p.prof && t == 0) ? clock64() : 0;
      inverse(sTot, t);
      if (p.prof && t == 0) { atomicAdd(p.prof + 0, (unsigned long long)(clock64() - ts0)); atomicAdd(p.prof + 3, 1ull); }
      __syncthreads();
      tp0 = (p.prof && t == 0) ? clock64() : 0;
      u32 I[8];
      lds_fe(I, sTot, t, T + t);
      const bool last = (run == p.nRun - 1);
#pragma unroll 1
      for (int i = 0; i < K; i++) {
        const int g = backward ? (K - 1 - i) : i;
        const int i0 = (g * 2) * T + t, i1 = (g * 2 + 1) * T + t;
        u32 x[8], pre[8], rx[8], ry[8], j;
        lds_fe(x, sX, i0, i1);
        lds_fe(pre, sP, i0, i1);
        const u32 aux0 = SYM ? (u32)sL[g * T + t] : 0u;
        const u32 neg = kangaroo_jump<SYM>(rx, ry, j, x, sY[i0], sY[i1], pre, I, i != K - 1, aux0, jt, p.symRule);
        uint4 dv = sD[g * T + t];
        u32 d[4] = {dv.x, dv.y, dv.z, dv.w};
        const uint4 jd = jt[128 + j];
        d128_add(d, jd.x, jd.y, jd.z, jd.w);
        u32 aux1 = 0;
        if (SYM) {                               // signed 128-bit distance: negated after the add
          d128_cneg(d, neg);
          aux1 = sym_next_aux(aux0, j, neg, p.symRule);
          sL[g * T + t] = (uint8_t)aux1;
        }
        sts_fe(sX, i0, i1, rx);
        sts_fe(sY, i0, i1, ry);
        sD[g * T + t] = make_uint4(d[0], d[1], d[2], d[3]);
        if (((rx[7] & mhi) | (rx[6] & mlo)) == 0u) {          // GPUCompute.h:96
          const u64 kidx = (u64)tile * TILE + (u64)(row0 + g) * T + (u64)t;
          if (kidx < p.nKangaroos) {
            const u32 pos = atomicAdd(p.out, 1u);
            if (pos < p.maxFound) put_dp_record(p.out, pos, rx, d, kidx);
          }
        }
        if (!last) {                             // next jump's dx and prefix, accumulated in THIS order
          u32 dx[8];
          next_dx<SYM>(dx, rx, aux1, jt, p.symRule);
          chain_dx(sP, i0, i1, P, dx, i == 0);
        }
      }
      if (!last) sts_fe(sTot, t, T + t, P);
      backward ^= 1;
    }

    uint4* gdst = gsrc;
#pragma unroll
    for (int g = 0; g < K; g++) {
      gdst[(g * CHUNKS + 0) * T + t] = sX[(g * 2 + 0) * T + t];
      gdst[(g * CHUNKS + 1) * T + t] = sX[(g * 2 + 1) * T + t];
      gdst[(g * CHUNKS + 2) * T + t] = sY[(g * 2 + 0) * T + t];
      gdst[(g * CHUNKS + 3) * T + t] = sY[(g * 2 + 1) * T + t];
      gdst[(g * CHUNKS + 4) * T + t] = sD[g * T + t];
      if (SYM) p.aux[(size_t)tile * TILE + (row0 + g) * T + t] = sL[g * T + t];
    }
  }
}

// Resident tile kernel: a CTA of T threads owns a tile of T * K kangaroos; warp 0 inverts the tile product.
template <int T, int K, bool SYM>
__global__ void __launch_bounds__(T, Cfg<T, K>::CTAS_PER_SM) jump_kernel(LaunchParams p) {
  tile_body<T, K, 1, SYM>(p, 0, [&](uint4* sTot, int t) {
    if (t < 32) tile_inverse<T, Cfg<T, K>::W>(sTot, t & 31, p.prof);
  });
}

// =====================================================================================================
// Cluster tile kernel (KGX_MODE=tmem / KGX_KERNEL_TMEM; the selector keeps its name).  One tile of 1792 kangaroos (14 rows
// of T = 128) is shared by the two CTAs of a thread-block cluster, each holding 7 rows -- x, y, prefix products and distances
// -- in its own shared memory (105 KB, so two CTAs fit on one SM).  The tile still takes ONE inverse per jump: each CTA
// reduces its 128 thread totals to one product (tile_reduce), the two products meet through distributed shared memory
// across a cluster barrier, both CTAs invert the same tile product and walk their own tree back.  That doubles the
// kangaroos per inverse of a 2-CTA-per-SM resident tile without needing more shared memory per SM.  Everything else is
// tile_body (no symmetric instantiation).
// =====================================================================================================
// A CTA's layout is Cfg<128, 7>'s, with the exchange slots (2 x 2 uint4: this CTA's product, double-buffered) where the
// resident layout keeps its state bytes.
struct CfgCl : Cfg<128, 7> {
  static constexpr int CLUSTER = 2;
  static constexpr int XCH_OFF = LJ_OFF;
  static constexpr int SMEM_BYTES = XCH_OFF + 4 * 16;
};

// Called by every thread of both CTAs (it contains a cluster barrier).  Warp 0 turns the T totals of sTot into their
// inverses like tile_inverse, but with the product of BOTH CTAs' totals inverted: `mine` is this CTA's exchange slot,
// `peer` the same slot of the other CTA (distributed shared memory).
template <int T, int W>
__device__ __noinline__ void cluster_tile_inverse(uint4* sTot, uint4* mine, const uint4* peer, int t) {
  const int lane = t & 31;
  u32 tw[W][8], c[W][8], v[8], sib[5][8];
  if (t < 32) {
    tile_reduce<T, W>(v, tw, c, sib, sTot, lane);
    if (lane == 0) sts_fe(mine, 0, 1, v);         // product of this CTA's 128 totals
  }
  cooperative_groups::this_cluster().sync();      // release / acquire: both products are visible cluster-wide
  if (t < 32) {
    u32 pv[8], inv[8];
    lds_fe(pv, peer, 0, 1);
    fe_mul(inv, v, pv);
    fe_inv(inv, inv);                             // 1 / tile product, identical in both CTAs
    fe_mul(inv, inv, pv);                         // -> 1 / this CTA's product
    tile_walk_back<T, W>(sTot, inv, tw, c, sib, lane);
  }
}

__global__ void __cluster_dims__(CfgCl::CLUSTER, 1, 1) __launch_bounds__(CfgCl::T, 2) jump_kernel_cluster(LaunchParams p) {
  extern __shared__ uint4 smem[];
  cooperative_groups::cluster_group cluster = cooperative_groups::this_cluster();
  const u32 rank = cluster.block_rank();
  uint4* xch = smem + CfgCl::XCH_OFF / 16;
  const uint4* xchPeer = cluster.map_shared_rank(xch, rank ^ 1u);
  // Exchange slot of the next tile inverse.  It alternates on EVERY call, across tile boundaries too: a CTA can only write
  // a slot again after the cluster barrier of the call in between, which its partner passes only after reading that slot.
  u32 slot = 0;
  tile_body<CfgCl::T, CfgCl::K, CfgCl::CLUSTER, false>(p, rank, [&](uint4* sTot, int t) {
    cluster_tile_inverse<CfgCl::T, CfgCl::W>(sTot, xch + 2 * slot, xchPeer + 2 * slot, t);
    slot ^= 1u;
  });
  cluster.sync();   // the other CTA may still read this CTA's exchange slot
}

// =====================================================================================================
// Streaming variant: every THREAD owns a private Montgomery group of G kangaroos that live in HBM
// ([tile][g][chunk][t], 16-byte chunks, lanes contiguous -> every warp access is one 512-byte line set).
// No barriers, no cross-thread traffic: a thread inverts its own group product (lanes diverge inside the
// variable-time safegcd, other warps fill the pipes meanwhile) and then makes ONE fused pass over its G
// kangaroos per jump: read prefix/x/y (96 B), write x'/y'/next prefix (96 B) and one jump-log byte, software-prefetching
// the next kangaroo while the current one is in the multiplier.  The distance chunk stays out of the hot loop: the
// log is folded into it at the end of the launch (stream_fold), so at every launch boundary the state holds the exact
// distance.  HBM traffic ~194.5 B/jump instead of 2.5, but no serial section at all; selected with KGX_MODE=stream
// (see DESIGN.md for the measured trade-off).
// =====================================================================================================
struct KangLoad { uint4 p0, p1, x0, x1, y0, y1; u32 lj; };

// Runs a jump-log window holds.  A thread folds its log into the distances after its tile's last run and after every
// LOG_RUNS runs, so the log takes LOG_RUNS bytes per kangaroo whatever kgx_set_jumps_per_launch says.
constexpr int LOG_RUNS = 64;


// sg / pg point at this thread's column of kangaroo g: sg = st + g*CHUNKS*T, pg = pr + g*2*T (running pointers: the
// hot loop does no index multiplications -- IMAD shares the binding pipe)
template <int T, bool SYM>
__device__ __forceinline__ void stream_load(KangLoad& k, const uint4* sg, const uint4* pg, const uint8_t* ag) {
  k.p0 = pg[0]; k.p1 = pg[T];
  k.x0 = sg[0]; k.x1 = sg[T];
  k.y0 = sg[2 * T]; k.y1 = sg[3 * T];
  if (SYM) k.lj = ag[0];
}

// Replays one jump-log byte on a distance: bits 0-4 the jump index, bit 5 the class switch of symmetric mode -- exactly
// the distance update of the jump (d += jD[j]; d = -d after a switch).
template <bool SYM>
__device__ __forceinline__ void replay_jump(u32* d, u32 b, const uint4* jt) {
  const uint4 jd = jt[128 + (b & 31u)];
  d128_add(d, jd.x, jd.y, jd.z, jd.w);
  if (SYM) d128_cneg(d, 0u - ((b >> 5) & 1u));
}

// Replays the first n (<= LOG_RUNS) bytes of one kangaroo's log window on its distance: l = the window's first byte, its
// runs lie runStride bytes apart.  The bytes are loaded in two batches of LOG_RUNS / 2 before any of a batch is applied
// (the window is always allocated), so the replay waits for two memory latencies, not one per jump.  The log is read
// with ordinary loads: this thread wrote it in this launch.
template <bool SYM>
__device__ __forceinline__ void replay_window(u32* d, const uint8_t* l, size_t runStride, int n, const uint4* jt) {
  constexpr int HALF = LOG_RUNS / 2;
#pragma unroll
  for (int h = 0; h < LOG_RUNS; h += HALF) {
    u32 b[HALF];
#pragma unroll
    for (int r = 0; r < HALF; r++) b[r] = l[(size_t)(h + r) * runStride];
#pragma unroll
    for (int r = 0; r < HALF; r++)
      if (h + r < n) replay_jump<SYM>(d, b[r], jt);
  }
}

// DP record append (GPUCompute.h:96-105, GPUMath.h:173-188): rare path (2^-dp per jump), kept out of line so the jump loop
// stays one basic block.  The record is re-read from the kangaroo's own state chunks, which stream_body has just
// written (same thread, program order): the hot loop keeps neither x' nor d' alive for it -- no local-memory home, no
// extra registers.  d' is the distance of the last fold plus the `runs` + 1 log bytes of this window, the last one at lg.
template <int T, bool SYM>
__device__ __noinline__ void emit_dp_from_state(u32* out, const u32 maxFound, const u64 nKangaroos, const uint4* sg, const uint8_t* lg,
                                                int runs, size_t runStride, const uint4* jt, u64 kidx) {
  if (kidx >= nKangaroos) return;                      // padding slot
  const u32 pos = atomicAdd(out, 1u);
  if (pos >= maxFound) return;                         // GPUEngine.cu:641-648: counted, not stored
  const uint4 x0 = sg[0], x1 = sg[T], dv = sg[4 * T];
  u32 x[8], d[4] = {dv.x, dv.y, dv.z, dv.w};
  replay_window<SYM>(d, lg - (ptrdiff_t)runs * (ptrdiff_t)runStride, runStride, runs + 1, jt);
  unpack8(x, x0, x1);
  put_dp_record(out, pos, x, d, kidx);
}

// Folds the `runs` logged jumps of this thread's G kangaroos into their distance chunks.  st / lt: this thread's column
// of the tile's state and log.  Every warp load of the log is one 32-byte sector; the next kangaroo's log lines are
// pulled into L2 while one is replayed (lane l: runs l and l + 32).
template <int T, bool SYM>
__device__ __noinline__ void stream_fold(uint4* st, const uint8_t* lt, const int G, const int runs, const uint4* jt) {
  const size_t runStride = (size_t)G * T;
  const int lane = threadIdx.x & 31;
  const uint8_t* pf = lt - threadIdx.x + (size_t)lane * runStride;
#pragma unroll 1
  for (int g = 0; g < G; g++) {
    const uint8_t* l = lt + (size_t)g * T;
    if (g + 1 < G) {
      asm volatile("prefetch.global.L2 [%0];" ::"l"(pf + (size_t)(g + 1) * T));
      asm volatile("prefetch.global.L2 [%0];" ::"l"(pf + (size_t)(g + 1) * T + 32 * runStride));
    }
    uint4* dp = st + (size_t)(g * CHUNKS + 4) * T;
    const uint4 dv = *dp;
    u32 d[4] = {dv.x, dv.y, dv.z, dv.w};
    replay_window<SYM>(d, l, runStride, runs, jt);
    *dp = make_uint4(d[0], d[1], d[2], d[3]);
  }
}

// One kangaroo of the fused pass (see the file header): back-substitute, jump, log the jump, start the next chain.
// Branch-free: returns whether the new point is distinguished (x' is in the state chunks for emit_dp_from_state).
template <int T, bool SYM>
__device__ __forceinline__ bool stream_body(const KangLoad& cur, uint4* sg, uint4* pg, uint8_t* ag, uint8_t* lg, const uint4* jt, u32* I,
                                            u32* P, const u32 mlo, const u32 mhi, const int rule) {
  u32 x[8], pre[8], dx[8], rx[8], ry[8], j;
  unpack8(x, cur.x0, cur.x1);
  unpack8(pre, cur.p0, cur.p1);
  // I is stripped after the last kangaroo of a pass too: unused, but one branch fewer
  const u32 neg = kangaroo_jump<SYM>(rx, ry, j, x, cur.y0, cur.y1, pre, I, true, cur.lj, jt, rule);
  u32 auxn = 0;
  if (SYM) {
    auxn = sym_next_aux(cur.lj, j, neg, rule);
    ag[0] = (uint8_t)auxn;                 // lastJump / symClass
  }
  lg[0] = (uint8_t)(j | (neg & 32u));      // jump-log byte (replay_jump): the distance update happens in the fold
  sg[0] = make_uint4(rx[0], rx[1], rx[2], rx[3]);
  sg[T] = make_uint4(rx[4], rx[5], rx[6], rx[7]);
  sg[2 * T] = make_uint4(ry[0], ry[1], ry[2], ry[3]);
  sg[3 * T] = make_uint4(ry[4], ry[5], ry[6], ry[7]);
  // next jump's dx and prefix product, accumulated in THIS order (P starts at 1 for the first kangaroo of a pass)
  next_dx<SYM>(dx, rx, auxn, jt, rule);
  pg[0] = make_uint4(P[0], P[1], P[2], P[3]);
  pg[T] = make_uint4(P[4], P[5], P[6], P[7]);
  fe_mul(P, P, dx);
  return ((rx[7] & mhi) | (rx[6] & mlo)) == 0u;          // GPUCompute.h:96
}

// Group inverse of the stream kernel.  WARPINV = false: every thread inverts the product of its own G kangaroos (lanes
// diverge inside the variable-time safegcd).  WARPINV = true: the 32 lane products are multiplied together by an XOR
// butterfly (5 shuffle rounds, every lane keeps the sibling factor of each round), ONE warp-uniform inverse is computed
// -- no divergence, 32 x fewer inversions -- and the butterfly is walked back: 10 multiplications per lane per pass buy
// a Montgomery group of 32*G kangaroos (north_star: "batch-inverse prefix/suffix products done with warp shuffles so one
// inverse amortises over the whole group").  Same canonical inverses either way (SURVEY.md App. A.4).
template <bool WARPINV>
__device__ __forceinline__ void stream_group_inverse(u32* I, const u32* P) {
  if (!WARPINV) { fe_inv(I, P); return; }
  u32 v[8], sib[5][8];
  fe_copy(v, P);
  butterfly_up(v, sib);
  fe_inv(I, v);                                  // identical in all 32 lanes
  butterfly_down(I, sib);                        // -> 1 / (this lane's own product)
}

template <int T, int CTAS, bool WARPINV, bool SYM>
__global__ void __launch_bounds__(T, CTAS) stream_kernel(LaunchParams p) {
  const int G = p.G;     // even: the fused pass is unrolled by two
  __shared__ uint4 jt[JT_WORDS / 4];
  const int t = threadIdx.x, lane = t & 31;
  const u32 mlo = (u32)p.dpMask, mhi = (u32)(p.dpMask >> 32);
  for (int i = t; i < JT_WORDS; i += T) reinterpret_cast<u32*>(jt)[i] = p.jtab[i];
  __syncthreads();

  for (u32 tile = blockIdx.x; tile < p.numTiles; tile += gridDim.x) {
    uint4* st = p.state + (size_t)tile * (G * CHUNKS * T) + t;
    uint4* pr = p.pre + (size_t)tile * (G * 2 * T) + t;
    const u64 kbase = (u64)tile * (T * G) + (u64)t;
    uint8_t* au = SYM ? (p.aux + (size_t)tile * ((size_t)G * T) + t) : nullptr;
    uint8_t* lt = p.jlog + (size_t)tile * ((size_t)LOG_RUNS * G * T) + t;    // [run][g] bytes of this thread's column
    const size_t runStride = (size_t)G * T;
    u32 P[8];
    fe_set_one(P);
    {   // prologue: forward chain, pr[g] = product of the dx before g
      u32 x[8], dx[8];
#pragma unroll 1
      for (int g = 0; g < G; g++) {
        unpack8(x, st[(g * CHUNKS + 0) * T], st[(g * CHUNKS + 1) * T]);
        next_dx<SYM>(dx, x, SYM ? (u32)au[(size_t)g * T] : 0u, jt, p.symRule);
        pr[(g * 2) * T] = make_uint4(P[0], P[1], P[2], P[3]); pr[(g * 2 + 1) * T] = make_uint4(P[4], P[5], P[6], P[7]);
        fe_mul(P, P, dx);
      }
    }
    int backward = 1;
    int logged = 0;                               // runs in the log since the last fold
    for (int run = 0; run < p.nRun; run++) {
      u32 I[8];
      stream_group_inverse<WARPINV>(I, P);       // 1 / (dx_0 ... dx_{G-1}) of this thread's G kangaroos
      fe_set_one(P);
      const int g0 = backward ? (G - 1) : 0;
      const ptrdiff_t ds = backward ? -(ptrdiff_t)(CHUNKS * T) : (ptrdiff_t)(CHUNKS * T);   // pointer steps per kangaroo
      const ptrdiff_t dp = backward ? -(ptrdiff_t)(2 * T) : (ptrdiff_t)(2 * T);
      const long long dk = backward ? -(long long)T : (long long)T;
      uint4* sg = st + (size_t)g0 * (CHUNKS * T);
      uint4* pg = pr + (size_t)g0 * (2 * T);
      uint8_t* ag = SYM ? (au + (size_t)g0 * T) : nullptr;
      uint8_t* lg = lt + (size_t)logged * runStride + (size_t)g0 * T;
      u64 kidx = kbase + (u64)g0 * T;
      KangLoad A, B;                              // ping-pong prefetch buffers (no register copies)
      stream_load<T, SYM>(A, sg, pg, ag);
      // L2 prefetch of the pair p.pfDist trips ahead (no registers held): a pair is 12 planes (2 x {x lo, x hi, y lo, y hi} of the
      // state, 2 x {lo, hi} of the prefix products) of 512 B per warp = 48 lines of 128 B.  Each LANE asks for a different line --
      // lane -> (plane lane/4, line lane%4) -- so two instructions cover the pair instead of one per plane (12).
      const int pl = lane >> 2;
      const ptrdiff_t lineOff = (ptrdiff_t)((lane & 3) * 8) - lane;                       // uint4 units, from this thread's own address
      const uint4* q1 = pl < 4 ? sg + (ptrdiff_t)p.pfDist * ds + pl * T + lineOff         // first kangaroo: 4 state planes,
                               : pg + (ptrdiff_t)p.pfDist * dp + (pl < 6 ? (pl - 4) * T : dp + (pl - 6) * T) + lineOff;   // both kangaroos' 2 prefix planes
      const uint4* q2 = sg + (ptrdiff_t)(p.pfDist + 1) * ds + pl * T + lineOff;          // second kangaroo: 4 state planes (lanes 0..15)
      const ptrdiff_t qs = 2 * (pl < 4 ? ds : dp);
      const bool q2on = pl < 4;
#pragma unroll 1
      for (int i = 0; i < G; i += 2) {
        if (p.pfDist > 0 && i + p.pfDist + 1 < G) {
          asm volatile("prefetch.global.L2 [%0];" ::"l"(q1));
          if (q2on) asm volatile("prefetch.global.L2 [%0];" ::"l"(q2));
        }
        q1 += qs; q2 += qs;
        stream_load<T, SYM>(B, sg + ds, pg + dp, ag + dk);
        const bool ha = stream_body<T, SYM>(A, sg, pg, ag, lg, jt, I, P, mlo, mhi, p.symRule);
        if (i + 2 < G) stream_load<T, SYM>(A, sg + 2 * ds, pg + 2 * dp, ag + 2 * dk);
        const bool hb = stream_body<T, SYM>(B, sg + ds, pg + dp, ag + dk, lg + dk, jt, I, P, mlo, mhi, p.symRule);
        if (__any_sync(0xffffffffu, ha | hb)) {      // warp-uniform: taken about once per 2^dp / 64 pairs
          if (ha) emit_dp_from_state<T, SYM>(p.out, p.maxFound, p.nKangaroos, sg, lg, logged, runStride, jt, kidx);
          if (hb) emit_dp_from_state<T, SYM>(p.out, p.maxFound, p.nKangaroos, sg + ds, lg + dk, logged, runStride, jt, kidx + dk);
          __syncwarp();   // the lanes back from a DP record rejoin their warp here.  Left to themselves they ran the rest of the
                          // launch as a separate group (the shuffles of the group inverse do not merge them): on the H100, 4 200
                          // DPs per launch cost a third of the kernel's speed.
        }
        sg += 2 * ds; pg += 2 * dp; lg += 2 * dk; kidx += 2 * dk;
        if (SYM) ag += 2 * dk;
      }
      backward ^= 1;
      if (++logged == LOG_RUNS || run == p.nRun - 1) {
        stream_fold<T, SYM>(st, lt, G, logged, jt);
        logged = 0;
      }
    }
  }
}

// ---- host AoS (kIdx order) <-> tile layout --------------------------------------------------------------
// slot s -> tile = s / TILE, g = (s % TILE) / T, t = s % T.  Padding slots (s >= n) replicate kangaroo s % n
// so that every tile is full of valid walkers; their DPs are dropped by the kidx < nKangaroos test.  The state byte of
// slot s (symmetric mode) is aux[s].
// Chunk 0 of slot s in the [tile][g][CHUNKS][T] layout of T x K tiles; chunk c is at [c * T].
template <class V>
__device__ __forceinline__ V* slot_chunks(V* state, u64 s, int T, int K) {
  const int TILE = T * K;
  const int r = (int)(s % TILE);
  return state + (s / TILE) * (K * CHUNKS * T) + (r / T) * (CHUNKS * T) + r % T;
}
__global__ void pack_kernel(uint4* state, const uint4* px, const uint4* py, const uint4* d, u64 n, u64 nPadded, int T, int K, uint8_t* aux, int auxInit) {
  u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= nPadded) return;
  u64 src = s < n ? s : s % n;
  uint4* dst = slot_chunks(state, s, T, K);
  dst[0] = px[2 * src];
  dst[T] = px[2 * src + 1];
  dst[2 * T] = py[2 * src];
  dst[3 * T] = py[2 * src + 1];
  dst[4 * T] = d[src];
  if (aux) aux[s] = (uint8_t)auxInit;   // lastJump = NB_JUMP: none yet (GPUEngine.cu:413-416) / symClass = 0 (Kangaroo.cpp:345-347)
}
__global__ void unpack_kernel(const uint4* state, uint4* px, uint4* py, uint4* d, u64 n, int T, int K) {
  u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const uint4* src = slot_chunks(state, s, T, K);
  px[2 * s] = src[0];
  px[2 * s + 1] = src[T];
  py[2 * s] = src[2 * T];
  py[2 * s + 1] = src[3 * T];
  d[s] = src[4 * T];
}
struct PatchArgs { uint4 c[CHUNKS]; };
__global__ void patch_kernel(uint4* state, u64 s, PatchArgs a, int T, int K, uint8_t* aux, int auxInit) {
  if (threadIdx.x < CHUNKS) slot_chunks(state, s, T, K)[threadIdx.x * T] = a.c[threadIdx.x];
  if (aux && threadIdx.x == 0) aux[s] = (uint8_t)auxInit;   // GPUEngine.cu:532-536
}

// ---- SURVEY 8f/f1: device-side HashTable::Convert (HashTable.cpp:75-100) -------------------------------------------
// 56-byte engine record {x[8 words], biased d[4 words], kIdx[2 words]} -> the reference's 40-byte wire/disk record
// DP {u32 kIdx; u32 h; int128 x; int128 d} (Kangaroo.h:94-101): h = x.bits64[2] & 0x3FFFF, x = 128 LSBs,
// d = |distance| (126 bits) | sign << 127 | type << 126 with distance = biased d - wildOffset for wild kangaroos
// (GPUEngine.cu:672) taken as a signed value (the reference forms it mod n and tests the top bit).
// signedMode (symmetric engine): the record's distance is a signed 128-bit two's complement value, no wild offset.
__global__ void dp_convert_kernel(const u32* __restrict__ slab, u32* __restrict__ out40, u32 maxFound, u64 wo0, u64 wo1, int signedMode) {
  const u32 cnt = min(slab[0], maxFound);
  if (blockIdx.x == 0 && threadIdx.x == 0) out40[0] = cnt;
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < cnt; i += gridDim.x * blockDim.x) {
    const u32* r = slab + 1 + (size_t)i * 14;
    u32* o = out40 + 1 + (size_t)i * 10;
    const u64 kidx = (u64)r[12] | ((u64)r[13] << 32);
    const u32 type = (u32)(kidx & 1ull);
    u64 d0 = (u64)r[8] | ((u64)r[9] << 32), d1 = (u64)r[10] | ((u64)r[11] << 32);
    u64 sign = 0;
    if (signedMode) {
      if (d1 >> 63) { d0 = ~d0 + 1; d1 = ~d1 + (d0 == 0); sign = 1ull << 63; }
    } else if (type) {                            // wild: subtract the offset, keep magnitude + sign
      const u64 b0 = d0 < wo0;
      u64 t0 = d0 - wo0, t1 = d1 - wo1 - b0;
      const bool neg = (d1 < wo1) || (d1 == wo1 && d0 < wo0);
      if (neg) { t0 = ~t0 + 1; t1 = ~t1 + (t0 == 0); sign = 1ull << 63; }
      d0 = t0; d1 = t1;
    }
    d1 = (d1 & 0x3FFFFFFFFFFFFFFFull) | sign | ((u64)type << 62);
    o[0] = (u32)kidx;
    o[1] = r[4] & 0x3FFFFu;                       // x.bits64[2] low word & HASH_MASK
    o[2] = r[0]; o[3] = r[1]; o[4] = r[2]; o[5] = r[3];
    o[6] = (u32)d0; o[7] = (u32)(d0 >> 32); o[8] = (u32)d1; o[9] = (u32)(d1 >> 32);
  }
}

// ---- microbench kernel (the unit-test kernel is in kgx_testhooks.cuh) ------------------------------------
// kind 0: dependent-free IMAD.WIDE.U32 issue-rate probe; kind 1: fe_mul chains; kind 2: fe_sqr chains; kind 3: fe_inv
__global__ void bench_raw_kernel(int kind, int iters, u32* sink) {
  const u32 seed = blockIdx.x * blockDim.x + threadIdx.x + 1u;
  if (kind == 0) {
    // 8 independent accumulators, multiplier changes every iteration so nothing can be hoisted:
    // measures the IMAD.WIDE.U32 issue rate of the fmaheavy pipe (the multiplier roofline of this engine).
    u64 acc[8];
    u32 x[8];
#pragma unroll
    for (int k = 0; k < 8; k++) { acc[k] = seed * (k + 3u); x[k] = seed + k * 1315423911u; }
    u32 m1 = seed * 7u + 5u;
    for (int it = 0; it < iters; it++) {
      m1 = m1 * 0x9E3779B1u + 12345u;
#pragma unroll
      for (int k = 0; k < 8; k++) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[k]) : "r"(x[k]), "r"(m1));
    }
    u64 s = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) s ^= acc[k];
    if (s == 0x1234567ull) sink[0] = (u32)s;
    return;
  }
  u32 a[8], b[8];
#pragma unroll
  for (int w = 0; w < 8; w++) { a[w] = seed * (2654435761u + w); b[w] = seed * (40503u + 7u * w) + w; }
  if (kind == 1) { for (int it = 0; it < iters; it++) { fe_mul(a, a, b); fe_mul(b, b, a); } }
  else if (kind == 2) { for (int it = 0; it < iters; it++) { fe_sqr(a, a); fe_sqr(b, b); } }
  else { for (int it = 0; it < iters; it++) { fe_inv(a, a); a[0] ^= b[0]; } }
  u32 s = 0;
#pragma unroll
  for (int w = 0; w < 8; w++) s ^= a[w] ^ b[w];
  if (s == 0x12345u) sink[0] = s;
}

}  // namespace kgx
