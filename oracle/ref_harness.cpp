/*
 * ref_harness.cpp -- thin C wrapper that drives the UNMODIFIED reference SECPK1 / HashTable code.
 *
 * TEST / BASELINE INFRASTRUCTURE ONLY.  Compiled by oracle/Makefile against the sources where they lie
 * under $KANGAROO_REF (nothing is copied into this repo) into oracle/_ref/libkref.so.  It exists to
 *   (1) pin oracle/kgx_oracle.c against the reference's own arithmetic (tests/test_oracle_vs_ref.py),
 *   (2) generate the committed fixtures under tests/golden/ (tests/golden/make_golden.py),
 *   (3) serve as the "reference" CPU baseline in bench.py (the SolveKeyCPU inner loop, Kangaroo.cpp:375-433,
 *       executed through the reference's Int / IntGroup classes on all host cores).
 * Only public reference API is called: Int, IntGroup, Point, Secp256K1, rseed/rndl, HashTable::Convert.
 * Kangaroo::CreateJumpTable / CreateHerd are private members (Kangaroo.h:166-167), so their bodies are
 * re-expressed here through the same public calls in the same order (Kangaroo.cpp:742-832, 670-738).
 */
#include <cstdint>
#include <cstring>
#include <cmath>
#include <vector>
#include <pthread.h>
#include <time.h>
#include "SECPK1/SECP256k1.h"
#include "SECPK1/IntGroup.h"
#include "SECPK1/Random.h"
#include "HashTable.h"
#include "Constants.h"

static Secp256K1 *secp = nullptr;

static void to_int(Int &r, const uint64_t *a, int limbs = 4) {
  r.SetInt32(0);
  for (int i = 0; i < limbs; i++) r.bits64[i] = a[i];
}
static void from_int(uint64_t *a, const Int &r, int limbs = 4) {
  for (int i = 0; i < limbs; i++) a[i] = r.bits64[i];
}

extern "C" {

void ref_init() {
  if (!secp) { secp = new Secp256K1(); secp->Init(); }
}
void ref_rseed(uint32_t s) { rseed(s); }
uint32_t ref_rndl() { return (uint32_t)rndl(); }
void ref_rand_bits(uint64_t r[4], int nbit) { Int a; a.Rand(nbit); from_int(r, a); }

void ref_mod_mul(uint64_t r[4], const uint64_t a[4], const uint64_t b[4]) {
  Int A, B, R; to_int(A, a); to_int(B, b); R.ModMulK1(&A, &B); from_int(r, R);
}
void ref_mod_sqr(uint64_t r[4], const uint64_t a[4]) {
  Int A, R; to_int(A, a); R.ModSquareK1(&A); from_int(r, R);
}
void ref_mod_sub(uint64_t r[4], const uint64_t a[4], const uint64_t b[4]) {
  Int A, B, R; to_int(A, a); to_int(B, b); R.ModSub(&A, &B); from_int(r, R);
}
void ref_mod_inv(uint64_t r[4], const uint64_t a[4]) {
  Int A; to_int(A, a); A.ModInv(); from_int(r, A);
}
void ref_order_add(uint64_t r[4], const uint64_t a[4], const uint64_t b[4]) {
  Int A, B; to_int(A, a); to_int(B, b); A.ModAddK1order(&B); from_int(r, A);
}
void ref_order_sub(uint64_t r[4], const uint64_t a[4], const uint64_t b[4]) {
  Int A, B; to_int(A, a); to_int(B, b); A.ModSubK1order(&B); from_int(r, A);
}
void ref_ec_mul_g(uint64_t rx[4], uint64_t ry[4], const uint64_t k[4]) {
  Int K; to_int(K, k); Point p = secp->ComputePublicKey(&K); from_int(rx, p.x); from_int(ry, p.y);
}
void ref_ec_add(uint64_t rx[4], uint64_t ry[4], const uint64_t ax[4], const uint64_t ay[4],
                const uint64_t bx[4], const uint64_t by[4]) {
  Int one; one.SetInt32(1);
  Int X1, Y1, X2, Y2; to_int(X1, ax); to_int(Y1, ay); to_int(X2, bx); to_int(Y2, by);
  Point a(&X1, &Y1, &one), b(&X2, &Y2, &one);
  Point r = secp->AddDirect(a, b);
  from_int(rx, r.x); from_int(ry, r.y);
}

/* Kangaroo.cpp:742-832 (non-symmetry branch), same calls in the same order. */
int ref_create_jump_table(int rangePower, uint64_t *jd, uint64_t *jpx, uint64_t *jpy) {
  int jumpBit = rangePower / 2 + 1;
  if (jumpBit > 128) jumpBit = 128;
  int maxRetry = 100; bool ok = false; double distAvg; int draws = 0;
  double maxAvg = pow(2.0, (double)jumpBit - 0.95);
  double minAvg = pow(2.0, (double)jumpBit - 1.05);
  Int jumpDistance[NB_JUMP];
  rseed(0x600DCAFE);
  while (!ok && maxRetry > 0) {
    Int totalDist; totalDist.SetInt32(0);
    for (int i = 0; i < NB_JUMP; ++i) {
      jumpDistance[i].Rand(jumpBit);
      if (jumpDistance[i].IsZero()) jumpDistance[i].SetInt32(1);
      totalDist.Add(&jumpDistance[i]);
    }
    distAvg = totalDist.ToDouble() / (double)(NB_JUMP);
    ok = distAvg > minAvg && distAvg < maxAvg;
    maxRetry--; draws++;
  }
  for (int i = 0; i < NB_JUMP; ++i) {
    Point J = secp->ComputePublicKey(&jumpDistance[i]);
    from_int(jd + 2 * i, jumpDistance[i], 2);
    from_int(jpx + 4 * i, J.x); from_int(jpy + 4 * i, J.y);
  }
  return draws;
}

/* Kangaroo.cpp:670-738 (non-symmetry branch). */
void ref_create_herd(int n, int rangePower, const uint64_t wdiv2[4], const uint64_t keyx[4], const uint64_t keyy[4],
                     int firstType, uint64_t *px, uint64_t *py, uint64_t *d) {
  Int W; to_int(W, wdiv2);
  Int one; one.SetInt32(1);
  Int KX, KY; to_int(KX, keyx); to_int(KY, keyy);
  Point key(&KX, &KY, &one);
  std::vector<Int> pk; std::vector<Point> S, Sp;
  Point Z; Z.Clear();
  for (int j = 0; j < n; j++) {
    Int dj; dj.Rand(rangePower);
    if ((j + firstType) % 2 == WILD) dj.ModSubK1order(&W);
    pk.push_back(dj);
    from_int(d + 4 * j, dj);
  }
  S = secp->ComputePublicKeys(pk);
  for (int j = 0; j < n; j++) Sp.push_back(((j + firstType) % 2 == TAME) ? Z : key);
  S = secp->AddDirect(Sp, S);
  for (int j = 0; j < n; j++) { from_int(px + 4 * j, S[j].x); from_int(py + 4 * j, S[j].y); }
}

typedef struct { uint64_t x[4]; uint64_t d[4]; uint64_t kidx; uint32_t jump; uint32_t pad; } ref_dp_t;

/* Kangaroo.cpp:375-433 through Int / IntGroup, group size grp (reference CPU_GRP_SIZE = 1024). */
static uint64_t jump_cpu_impl(int n, int njumps, int grp, Int *px, Int *py, Int *dist, Int *jD, Int *jPx, Int *jPy,
                              uint64_t dMask, ref_dp_t *dps, uint64_t max_dp) {
  uint64_t ndp = 0;
  IntGroup *g = new IntGroup(grp);
  Int *dx = new Int[grp];
  Int dy, rx, ry, _s, _p;
  for (int run = 0; run < njumps; run++) {
    for (int g0 = 0; g0 < n; g0 += grp) {
      int m = (n - g0 < grp) ? (n - g0) : grp;
      IntGroup *gg = g;
      if (m != grp) gg = new IntGroup(m);
      for (int i = 0; i < m; i++) {
        uint64_t jmp = px[g0 + i].bits64[0] % NB_JUMP;
        dx[i].ModSub(&px[g0 + i], &jPx[jmp]);
      }
      gg->Set(dx); gg->ModInv();
      for (int i = 0; i < m; i++) {
        int k = g0 + i;
        uint64_t jmp = px[k].bits64[0] % NB_JUMP;
        Int *p1x = &jPx[jmp], *p1y = &jPy[jmp], *p2x = &px[k], *p2y = &py[k];
        dy.ModSub(p2y, p1y);
        _s.ModMulK1(&dy, &dx[i]);
        _p.ModSquareK1(&_s);
        rx.ModSub(&_p, p1x);
        rx.ModSub(p2x);
        ry.ModSub(p2x, &rx);
        ry.ModMulK1(&_s);
        ry.ModSub(p2y);
        dist[k].ModAddK1order(&jD[jmp]);
        px[k].Set(&rx); py[k].Set(&ry);
        if ((px[k].bits64[3] & dMask) == 0) {
          if (dps && ndp < max_dp) {
            from_int(dps[ndp].x, px[k]); from_int(dps[ndp].d, dist[k]);
            dps[ndp].kidx = (uint64_t)k; dps[ndp].jump = (uint32_t)(run + 1); dps[ndp].pad = 0;
          }
          ndp++;
        }
      }
      if (gg != g) delete gg;
    }
  }
  delete g; delete[] dx;
  return ndp;
}

uint64_t ref_jump_cpu(int n, int njumps, int grp, uint64_t *px, uint64_t *py, uint64_t *d,
                      const uint64_t *jd, const uint64_t *jpx, const uint64_t *jpy,
                      uint64_t dp_mask, ref_dp_t *dps, uint64_t max_dp) {
  Int *X = new Int[n], *Y = new Int[n], *D = new Int[n];
  Int jD[NB_JUMP], jPx[NB_JUMP], jPy[NB_JUMP];
  for (int i = 0; i < n; i++) { to_int(X[i], px + 4 * i); to_int(Y[i], py + 4 * i); to_int(D[i], d + 4 * i); }
  for (int i = 0; i < NB_JUMP; i++) { to_int(jD[i], jd + 2 * i, 2); to_int(jPx[i], jpx + 4 * i); to_int(jPy[i], jpy + 4 * i); }
  uint64_t r = jump_cpu_impl(n, njumps, grp, X, Y, D, jD, jPx, jPy, dp_mask, dps, max_dp);
  for (int i = 0; i < n; i++) { from_int(px + 4 * i, X[i]); from_int(py + 4 * i, Y[i]); from_int(d + 4 * i, D[i]); }
  delete[] X; delete[] Y; delete[] D;
  return r;
}

/* Check.cpp:534-549: one AddDirect per kangaroo per jump. */
void ref_jump_single(uint64_t x[4], uint64_t y[4], uint64_t d[4], const uint64_t *jd, const uint64_t *jpx, const uint64_t *jpy) {
  Int one; one.SetInt32(1);
  Int X, Y, D; to_int(X, x); to_int(Y, y); to_int(D, d);
  uint64_t jmp = X.bits64[0] % NB_JUMP;
  Int JX, JY, JD; to_int(JX, jpx + 4 * jmp); to_int(JY, jpy + 4 * jmp); to_int(JD, jd + 2 * jmp, 2);
  Point J(&JX, &JY, &one), P(&X, &Y, &one);
  P = secp->AddDirect(P, J);
  D.ModAddK1order(&JD);
  from_int(x, P.x); from_int(y, P.y); from_int(d, D);
}

void ref_hash_convert(const uint64_t x[4], const uint64_t d[4], uint32_t type, uint64_t *h, uint64_t X[2], uint64_t D[2]) {
  Int XX, DD; to_int(XX, x); to_int(DD, d);
  int128_t ox, od;
  HashTable::Convert(&XX, &DD, type, h, &ox, &od);
  X[0] = ox.i64[0]; X[1] = ox.i64[1]; D[0] = od.i64[0]; D[1] = od.i64[1];
}

/* ---- CPU baseline: SolveKeyCPU inner loop on `threads` pthreads, CPU_GRP_SIZE=1024 kangaroos each ---- */
struct bench_arg { int jumps; Int *jD, *jPx, *jPy; Int *px, *py, *d; uint64_t done; };
static void *bench_thread(void *p) {
  bench_arg *a = (bench_arg *)p;
  jump_cpu_impl(1024, a->jumps, 1024, a->px, a->py, a->d, a->jD, a->jPx, a->jPy, ~0ULL, nullptr, 0);
  a->done = (uint64_t)1024 * (uint64_t)a->jumps;
  return nullptr;
}
uint64_t ref_bench_cpu(int threads, int jumps_per_kangaroo, int rangePower, double *sec) {
  ref_init();
  static uint64_t jd[64], jpx[128], jpy[128];
  ref_create_jump_table(rangePower, jd, jpx, jpy);
  static Int jD[NB_JUMP], jPx[NB_JUMP], jPy[NB_JUMP];
  for (int i = 0; i < NB_JUMP; i++) { to_int(jD[i], jd + 2 * i, 2); to_int(jPx[i], jpx + 4 * i); to_int(jPy[i], jpy + 4 * i); }
  std::vector<bench_arg> args(threads);
  std::vector<pthread_t> th(threads);
  rseed(12345);
  uint64_t zero[4] = {0, 0, 0, 0};
  for (int t = 0; t < threads; t++) {
    args[t].jumps = jumps_per_kangaroo; args[t].jD = jD; args[t].jPx = jPx; args[t].jPy = jPy;
    std::vector<uint64_t> x(4096), y(4096), d(4096);
    ref_create_herd(1024, rangePower, zero, zero, zero, TAME + 0, x.data(), y.data(), d.data());
    /* all-tame herd is fine for timing: wild rows would only add key to the start point */
    args[t].px = new Int[1024]; args[t].py = new Int[1024]; args[t].d = new Int[1024];
    for (int i = 0; i < 1024; i++) {
      /* odd rows were built as key(=0)+d*G with p1.x==0 -> pass-through (SECP256K1.cpp:300-302) */
      to_int(args[t].px[i], x.data() + 4 * i); to_int(args[t].py[i], y.data() + 4 * i); to_int(args[t].d[i], d.data() + 4 * i);
    }
  }
  struct timespec t0, t1;
  clock_gettime(CLOCK_MONOTONIC, &t0);
  for (int t = 0; t < threads; t++) pthread_create(&th[t], nullptr, bench_thread, &args[t]);
  uint64_t total = 0;
  for (int t = 0; t < threads; t++) { pthread_join(th[t], nullptr); total += args[t].done; }
  clock_gettime(CLOCK_MONOTONIC, &t1);
  *sec = (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
  for (int t = 0; t < threads; t++) { delete[] args[t].px; delete[] args[t].py; delete[] args[t].d; }
  return total;
}

/* ===== USE_SYMMETRY paths (Constants.h:25), driven through the same public reference API =====
 * The library itself is compiled WITHOUT the macro (SECPK1 / HashTable do not depend on it); the three private Kangaroo
 * members are re-expressed from their USE_SYMMETRY branches, call for call: CreateJumpTable (Kangaroo.cpp:742-832),
 * CreateHerd (:670-738) and the symmetric walk as Kangaroo::Check replays it on the CPU (Check.cpp:534-556). */
int ref_create_jump_table_sym(int rangePower, uint64_t *jd, uint64_t *jpx, uint64_t *jpy, uint64_t uv[2]) {
  int jumpBit = rangePower / 2;
  if (jumpBit > 128) jumpBit = 128;
  int maxRetry = 100; bool ok = false; double distAvg; int draws = 0;
  double maxAvg = pow(2.0, (double)jumpBit - 0.95);
  double minAvg = pow(2.0, (double)jumpBit - 1.05);
  Int jumpDistance[NB_JUMP];
  rseed(0x600DCAFE);
  Int old; old.Set(Int::GetFieldCharacteristic());
  Int u, v;
  u.SetInt32(1); u.ShiftL(jumpBit / 2); u.AddOne();
  while (!u.IsProbablePrime()) { u.AddOne(); u.AddOne(); }
  v.Set(&u); v.AddOne(); v.AddOne();
  while (!v.IsProbablePrime()) { v.AddOne(); v.AddOne(); }
  Int::SetupField(&old);
  if (uv) { uv[0] = u.bits64[0]; uv[1] = v.bits64[0]; }
  while (!ok && maxRetry > 0) {
    Int totalDist; totalDist.SetInt32(0);
    for (int i = 0; i < NB_JUMP / 2; ++i) {
      jumpDistance[i].Rand(jumpBit / 2); jumpDistance[i].Mult(&u);
      if (jumpDistance[i].IsZero()) jumpDistance[i].SetInt32(1);
      totalDist.Add(&jumpDistance[i]);
    }
    for (int i = NB_JUMP / 2; i < NB_JUMP; ++i) {
      jumpDistance[i].Rand(jumpBit / 2); jumpDistance[i].Mult(&v);
      if (jumpDistance[i].IsZero()) jumpDistance[i].SetInt32(1);
      totalDist.Add(&jumpDistance[i]);
    }
    distAvg = totalDist.ToDouble() / (double)(NB_JUMP);
    ok = distAvg > minAvg && distAvg < maxAvg;
    maxRetry--; draws++;
  }
  for (int i = 0; i < NB_JUMP; ++i) {
    Point J = secp->ComputePublicKey(&jumpDistance[i]);
    from_int(jd + 2 * i, jumpDistance[i], 2);
    from_int(jpx + 4 * i, J.x); from_int(jpy + 4 * i, J.y);
  }
  return draws;
}

void ref_create_herd_sym(int n, int rangePower, const uint64_t wdiv4[4], const uint64_t keyx[4], const uint64_t keyy[4],
                         int firstType, uint64_t *px, uint64_t *py, uint64_t *d) {
  Int W; to_int(W, wdiv4);
  Int one; one.SetInt32(1);
  Int KX, KY; to_int(KX, keyx); to_int(KY, keyy);
  Point key(&KX, &KY, &one);
  std::vector<Int> pk; std::vector<Point> S, Sp;
  Point Z; Z.Clear();
  std::vector<Int> dd(n);
  for (int j = 0; j < n; j++) {
    dd[j].Rand(rangePower - 1);                                   /* Tame in [0..N/2] */
    if ((j + firstType) % 2 == WILD) dd[j].ModSubK1order(&W);     /* Wild in [-N/4..N/4] */
    pk.push_back(dd[j]);
  }
  S = secp->ComputePublicKeys(pk);
  for (int j = 0; j < n; j++) Sp.push_back(((j + firstType) % 2 == TAME) ? Z : key);
  S = secp->AddDirect(Sp, S);
  for (int j = 0; j < n; j++) {
    Int X, Y; X.Set(&S[j].x); Y.Set(&S[j].y);
    if (Y.ModPositiveK1()) dd[j].ModNegK1order();                 /* Kangaroo.cpp:730-734 */
    from_int(px + 4 * j, X); from_int(py + 4 * j, Y); from_int(d + 4 * j, dd[j]);
  }
}

/* Check.cpp:534-556 (USE_SYMMETRY): one AddDirect per kangaroo per jump, lastJump cycle limiter, class switch. */
uint64_t ref_jump_sym(int n, int njumps, uint64_t *px, uint64_t *py, uint64_t *d, uint8_t *lastJump,
                      const uint64_t *jd, const uint64_t *jpx, const uint64_t *jpy, uint64_t dMask, ref_dp_t *dps, uint64_t max_dp) {
  Int one; one.SetInt32(1);
  Int jD[NB_JUMP], jPx[NB_JUMP], jPy[NB_JUMP];
  for (int i = 0; i < NB_JUMP; i++) { to_int(jD[i], jd + 2 * i, 2); to_int(jPx[i], jpx + 4 * i); to_int(jPy[i], jpy + 4 * i); }
  uint64_t ndp = 0;
  for (int r = 0; r < njumps; r++) {
    for (int i = 0; i < n; i++) {
      Int X, Y, D; to_int(X, px + 4 * i); to_int(Y, py + 4 * i); to_int(D, d + 4 * i);
      uint64_t jmp = (X.bits64[0] % NB_JUMP);
      if (jmp == lastJump[i]) jmp = (lastJump[i] + 1) % NB_JUMP;
      Point J(&jPx[jmp], &jPy[jmp], &one);
      Point P(&X, &Y, &one);
      P = secp->AddDirect(P, J);
      X.Set(&P.x); Y.Set(&P.y);
      D.ModAddK1order(&jD[jmp]);
      if (Y.ModPositiveK1()) D.ModNegK1order();
      lastJump[i] = (uint8_t)jmp;
      from_int(px + 4 * i, X); from_int(py + 4 * i, Y); from_int(d + 4 * i, D);
      if ((X.bits64[3] & dMask) == 0) {
        if (dps && ndp < max_dp) {
          from_int(dps[ndp].x, X); from_int(dps[ndp].d, D);
          dps[ndp].kidx = (uint64_t)i; dps[ndp].jump = (uint32_t)(r + 1); dps[ndp].pad = 0;
        }
        ndp++;
      }
    }
  }
  return ndp;
}

/* SolveKeyCPU's symmetric loop (Kangaroo.cpp:375-433, USE_SYMMETRY branches) through Int / IntGroup: jmp = x mod 16 + 16*symClass,
 * class switch toggles symClass. */
uint64_t ref_jump_symclass(int n, int njumps, int grp, uint64_t *px, uint64_t *py, uint64_t *d, uint8_t *symClass,
                           const uint64_t *jd, const uint64_t *jpx, const uint64_t *jpy, uint64_t dMask, ref_dp_t *dps, uint64_t max_dp) {
  Int *X = new Int[n], *Y = new Int[n], *D = new Int[n];
  Int jD[NB_JUMP], jPx[NB_JUMP], jPy[NB_JUMP];
  for (int i = 0; i < n; i++) { to_int(X[i], px + 4 * i); to_int(Y[i], py + 4 * i); to_int(D[i], d + 4 * i); }
  for (int i = 0; i < NB_JUMP; i++) { to_int(jD[i], jd + 2 * i, 2); to_int(jPx[i], jpx + 4 * i); to_int(jPy[i], jpy + 4 * i); }
  uint64_t ndp = 0;
  Int *dx = new Int[grp];
  Int dy, rx, ry, _s, _p;
  for (int run = 0; run < njumps; run++) {
    for (int g0 = 0; g0 < n; g0 += grp) {
      int m = (n - g0 < grp) ? (n - g0) : grp;
      IntGroup *gg = new IntGroup(m);
      for (int i = 0; i < m; i++) {
        uint64_t jmp = X[g0 + i].bits64[0] % (NB_JUMP / 2) + (NB_JUMP / 2) * symClass[g0 + i];
        dx[i].ModSub(&X[g0 + i], &jPx[jmp]);
      }
      gg->Set(dx); gg->ModInv();
      for (int i = 0; i < m; i++) {
        int k = g0 + i;
        uint64_t jmp = X[k].bits64[0] % (NB_JUMP / 2) + (NB_JUMP / 2) * symClass[k];
        Int *p1x = &jPx[jmp], *p1y = &jPy[jmp], *p2x = &X[k], *p2y = &Y[k];
        dy.ModSub(p2y, p1y);
        _s.ModMulK1(&dy, &dx[i]);
        _p.ModSquareK1(&_s);
        rx.ModSub(&_p, p1x);
        rx.ModSub(p2x);
        ry.ModSub(p2x, &rx);
        ry.ModMulK1(&_s);
        ry.ModSub(p2y);
        D[k].ModAddK1order(&jD[jmp]);
        if (ry.ModPositiveK1()) { D[k].ModNegK1order(); symClass[k] = !symClass[k]; }
        X[k].Set(&rx); Y[k].Set(&ry);
        if ((X[k].bits64[3] & dMask) == 0) {
          if (dps && ndp < max_dp) {
            from_int(dps[ndp].x, X[k]); from_int(dps[ndp].d, D[k]);
            dps[ndp].kidx = (uint64_t)k; dps[ndp].jump = (uint32_t)(run + 1); dps[ndp].pad = 0;
          }
          ndp++;
        }
      }
      delete gg;
    }
  }
  for (int i = 0; i < n; i++) { from_int(px + 4 * i, X[i]); from_int(py + 4 * i, Y[i]); from_int(d + 4 * i, D[i]); }
  delete[] dx; delete[] X; delete[] Y; delete[] D;
  return ndp;
}

} /* extern "C" */
