// kgx_ingest.cpp -- rank-0 distinguished-point ingest around the reference's UNCHANGED `class HashTable`
// (C ABI: include/kgx_ingest.h; SURVEY.md 8f row f1, host half).
//
// Built by build_ingest.sh against the reference sources (HashTable.cpp, SECPK1/*, Timer.cpp compiled where they lie -- the
// same arrangement as the drop-in binary, INTEGRATION.md); nothing of the reference is copied into this repository.
//
// Reference path being replaced (the driver, not the table): Kangaroo::SolveKeyGPU's DP loop, Kangaroo.cpp:594-612 --
//   LOCK(ghMutex); for every DP: AddToTable(x, d, type) -> HashTable::Add -> [ADD_COLLISION] CollisionCheck -> CheckKey x4
// one thread, one mutex, one malloc per entry.  Here the records of all GPUs arrive as one 40-byte-record buffer per step
// (already converted on the device, kgx_convert_dps) and are inserted by a pool of workers sharded by bucket
// (h mod workers): HashTable::Add(h, x, d) touches only E[h] (HashTable.cpp:262-307), so shards never share a bucket and
// no lock is taken.  The one shared field HashTable::Add writes -- kDist/kType on ADD_COLLISION -- is not read: the stored
// entry is looked up again by the owning worker.
#include <atomic>
#include <cerrno>
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>
#include "HashTable.h"               // reference header, found through -I$REF
#include "SECPK1/SECP256k1.h"
#include "../../include/kgx_ingest.h"
#include "kgx_workfile.h"

namespace {

struct DP40 { uint32_t kidx, h; int128_t x, d; };   // Kangaroo.h:94-101
static_assert(sizeof(DP40) == 40, "DP record must be 40 bytes");

struct Job {
  const DP40* recs = nullptr;
  uint32_t n = 0, rank = 0;
};

}  // namespace

struct kgi_table {
  HashTable* ht = nullptr;
  Secp256K1* secp = nullptr;
  int nthreads = 1;
  std::vector<std::thread> workers;
  std::vector<std::vector<kgi_event>> evs;
  std::mutex mu;
  std::condition_variable cvStart, cvDone;
  uint64_t generation = 0;
  int pending = 0;
  bool quit = false, bad = false;
  Job job;
};

// the stored entry with the same x in bucket h (binary search like HashTable::Add, HashTable.cpp:283-303)
static const ENTRY* find_entry(HashTable* ht, uint32_t h, const int128_t* x) {
  int st = 0, ed = (int)ht->E[h].nbItem - 1;
  while (st <= ed) {
    const int mi = (st + ed) / 2;
    const ENTRY* e = ht->E[h].items[mi];
    if (x->i64[1] == e->x.i64[1] && x->i64[0] == e->x.i64[0]) return e;
    const bool less = (x->i64[1] == e->x.i64[1]) ? (x->i64[0] < e->x.i64[0]) : (x->i64[1] < e->x.i64[1]);
    if (less) ed = mi - 1; else st = mi + 1;
  }
  return nullptr;
}

// Kangaroo::AddToTable(h, x, d) (Kangaroo.cpp:315-330) for one record, on the shard that owns bucket h
static void add_one(kgi_table* t, const DP40& r, uint32_t rank, std::vector<kgi_event>& out) {
  int128_t x = r.x, d = r.d;
  const int st = t->ht->Add((uint64_t)r.h, &x, &d);
  if (st == ADD_OK) return;
  kgi_event ev;
  memset(&ev, 0, sizeof ev);
  ev.rank = rank; ev.kidx = r.kidx; ev.h = r.h;
  ev.d_new[0] = d.i64[0]; ev.d_new[1] = d.i64[1];
  if (st == ADD_DUPLICATE) { ev.kind = KGI_EV_RESET; out.push_back(ev); return; }
  const ENTRY* old = find_entry(t->ht, r.h, &x);                 // ADD_COLLISION
  if (!old) return;
  ev.d_old[0] = old->d.i64[0]; ev.d_old[1] = old->d.i64[1];
  const uint64_t TYPE = 0x4000000000000000ULL;                  // HashTable::CalcDistAndType, b126
  ev.kind = ((old->d.i64[1] ^ d.i64[1]) & TYPE) ? KGI_EV_COLLISION : KGI_EV_RESET;   // same herd -> reset (Kangaroo.cpp:258-262)
  out.push_back(ev);
}

static void worker_main(kgi_table* t, int id) {
  uint64_t seen = 0;
  for (;;) {
    Job job;
    {
      std::unique_lock<std::mutex> lk(t->mu);
      t->cvStart.wait(lk, [&] { return t->quit || t->generation != seen; });
      if (t->quit) return;
      seen = t->generation;
      job = t->job;
    }
    std::vector<kgi_event>& out = t->evs[id];
    const uint32_t T = (uint32_t)t->nthreads;
    bool bad = false;
    for (uint32_t i = 0; i < job.n; i++) {
      const DP40& r = job.recs[i];
      if (r.h >= HASH_SIZE) { bad = true; continue; }
      if (r.h % T != (uint32_t)id) continue;
      add_one(t, r, job.rank, out);
    }
    {
      std::lock_guard<std::mutex> lk(t->mu);
      if (bad) t->bad = true;
      if (--t->pending == 0) t->cvDone.notify_all();
    }
  }
}

extern "C" {

kgi_table* kgi_create(int threads) {
  kgi_table* t = new kgi_table();
  if (threads <= 0) {
    unsigned hc = std::thread::hardware_concurrency();
    threads = hc == 0 ? 1 : (hc > 8 ? 8 : (int)hc);
  }
  if (threads > 64) threads = 64;
  t->nthreads = threads;
  t->ht = new HashTable();
  t->secp = new Secp256K1();
  t->secp->Init();                     // also installs the group order for Int::Mod*K1order (SECP256K1.cpp:29-41)
  t->evs.resize(threads);
  for (int i = 0; i < threads; i++) t->workers.emplace_back(worker_main, t, i);
  return t;
}

void kgi_destroy(kgi_table* t) {
  if (!t) return;
  {
    std::lock_guard<std::mutex> lk(t->mu);
    t->quit = true;
  }
  t->cvStart.notify_all();
  for (auto& w : t->workers) w.join();
  t->ht->Reset();
  delete t->ht;
  delete t->secp;
  delete t;
}

void kgi_reset(kgi_table* t) { t->ht->Reset(); }
uint64_t kgi_count(kgi_table* t) { return t->ht->GetNbItem(); }
int kgi_threads(kgi_table* t) { return t->nthreads; }

int kgi_add(kgi_table* t, const void* dp40, uint32_t n, uint32_t rank, kgi_event* ev, uint32_t cap, uint32_t* n_ev) {
  *n_ev = 0;
  if (n == 0) return 0;
  {
    std::lock_guard<std::mutex> lk(t->mu);
    t->job.recs = static_cast<const DP40*>(dp40);
    t->job.n = n; t->job.rank = rank;
    t->pending = t->nthreads;
    t->bad = false;
    for (auto& v : t->evs) v.clear();
    t->generation++;
  }
  t->cvStart.notify_all();
  {
    std::unique_lock<std::mutex> lk(t->mu);
    t->cvDone.wait(lk, [&] { return t->pending == 0; });
  }
  uint32_t k = 0;
  for (auto& v : t->evs)
    for (auto& e : v) { if (k < cap) ev[k] = e; k++; }
  *n_ev = k;
  return t->bad ? -1 : 0;
}

int kgi_add_items(kgi_table* t, const void* items56, uint32_t n, uint32_t rank, const uint64_t wild_offset[2],
                  kgi_event* ev, uint32_t cap, uint32_t* n_ev) {
  // GPUEngine::Launch's un-biasing (GPUEngine.cu:653-675) + HashTable::Convert (HashTable.cpp:75-100), with the reference's own Int
  struct Item56 { uint64_t x[4], d[2], kidx; };
  const Item56* it = static_cast<const Item56*>(items56);
  std::vector<DP40> recs(n);
  Int wo; wo.SetInt32(0); wo.bits64[0] = wild_offset[0]; wo.bits64[1] = wild_offset[1];
  for (uint32_t i = 0; i < n; i++) {
    Int x, d; x.SetInt32(0); d.SetInt32(0);
    for (int k = 0; k < 4; k++) x.bits64[k] = it[i].x[k];
    d.bits64[0] = it[i].d[0]; d.bits64[1] = it[i].d[1];
    const uint32_t type = (uint32_t)(it[i].kidx & 1);
    if (type) d.ModSubK1order(&wo);
    uint64_t h;
    HashTable::Convert(&x, &d, type, &h, &recs[i].x, &recs[i].d);
    recs[i].h = (uint32_t)h; recs[i].kidx = (uint32_t)it[i].kidx;
  }
  return kgi_add(t, recs.data(), n, rank, ev, cap, n_ev);
}

int kgi_resolve(kgi_table* t, const uint64_t d_old[2], const uint64_t d_new[2], const uint64_t keyx[4], const uint64_t keyy[4],
                const uint64_t range_start[4], uint64_t priv_out[4]) {
  int128_t a, b;
  a.i64[0] = d_old[0]; a.i64[1] = d_old[1]; b.i64[0] = d_new[0]; b.i64[1] = d_new[1];
  Int da, db; uint32_t ta, tb;
  HashTable::CalcDistAndType(a, &da, &ta);
  HashTable::CalcDistAndType(b, &db, &tb);
  if (ta == tb) return 0;                                        // Kangaroo.cpp:258-262
  Int Td, Wd;
  if (ta == 0) { Td.Set(&da); Wd.Set(&db); } else { Td.Set(&db); Wd.Set(&da); }
  Point key; key.Clear();
  key.x.SetInt32(0); key.y.SetInt32(0);
  for (int k = 0; k < 4; k++) { key.x.bits64[k] = keyx[k]; key.y.bits64[k] = keyy[k]; }
  key.z.SetInt32(1);
  Point keyNeg(key);
  keyNeg.y.ModNeg();
  Int start; start.SetInt32(0);
  for (int k = 0; k < 4; k++) start.bits64[k] = range_start[k];
  for (int type = 0; type < 4; type++) {                          // Kangaroo::CheckKey, Kangaroo.cpp:218-253
    Int d1(&Td), d2(&Wd);
    if (type & 1) d1.ModNegK1order();
    if (type & 2) d2.ModNegK1order();
    Int pk(&d1);
    pk.ModAddK1order(&d2);
    Point P = t->secp->ComputePublicKey(&pk);
    bool hit = false;
    if (P.equals(key)) hit = true;
    else if (P.equals(keyNeg)) { pk.ModNegK1order(); hit = true; }
    if (hit) {
      pk.ModAddK1order(&start);
      for (int k = 0; k < 4; k++) priv_out[k] = pk.bits64[k];
      return 1;
    }
  }
  return 0;
}

int kgi_resolve_multi(kgi_table* t, const uint64_t d_old[2], const uint64_t d_new[2], const uint64_t* keys, uint32_t n_keys,
                      const uint64_t range_start[4], uint32_t* key_index_out, uint64_t priv_out[4]) {
  int128_t a, b;
  a.i64[0] = d_old[0]; a.i64[1] = d_old[1]; b.i64[0] = d_new[0]; b.i64[1] = d_new[1];
  Int da, db; uint32_t ta, tb;
  HashTable::CalcDistAndType(a, &da, &ta);
  HashTable::CalcDistAndType(b, &db, &tb);
  if (ta == tb) return 0;
  Int Td, Wd;
  if (ta == 0) { Td.Set(&da); Wd.Set(&db); } else { Td.Set(&db); Wd.Set(&da); }
  // the four candidates of Kangaroo::CheckKey (Kangaroo.cpp:218-253), each one scalar multiplication, whatever n_keys is
  Int pk[4];
  Point P[4];
  Int negY[4];
  for (int type = 0; type < 4; type++) {
    Int d1(&Td), d2(&Wd);
    if (type & 1) d1.ModNegK1order();
    if (type & 2) d2.ModNegK1order();
    pk[type].Set(&d1);
    pk[type].ModAddK1order(&d2);
    P[type] = t->secp->ComputePublicKey(&pk[type]);
    negY[type].Set(&P[type].y);
    negY[type].ModNeg();
  }
  // then only comparisons per key: key k matches when a candidate is +-keys[k]; for that key the candidates are tried in
  // kgi_resolve's order, so both calls give the same private key
  for (uint32_t k = 0; k < n_keys; k++) {
    Int kx, ky;
    kx.SetInt32(0); ky.SetInt32(0);
    for (int w = 0; w < 4; w++) { kx.bits64[w] = keys[8 * k + w]; ky.bits64[w] = keys[8 * k + 4 + w]; }
    for (int type = 0; type < 4; type++) {
      if (!P[type].x.IsEqual(&kx)) continue;
      Int priv(&pk[type]);
      if (P[type].y.IsEqual(&ky)) { }
      else if (negY[type].IsEqual(&ky)) priv.ModNegK1order();
      else continue;
      Int start; start.SetInt32(0);
      for (int w = 0; w < 4; w++) start.bits64[w] = range_start[w];
      priv.ModAddK1order(&start);
      for (int w = 0; w < 4; w++) priv_out[w] = priv.bits64[w];
      *key_index_out = k;
      return 1;
    }
  }
  return 0;
}

int kgi_save_work_ex(kgi_table* t, const char* path, uint32_t dp_bits, const uint64_t range_start[4], const uint64_t range_end[4],
                     const uint64_t keyx[4], const uint64_t keyy[4], uint64_t total_count, double total_time, uint64_t total_walk) {
  using namespace kgx_wf;
  errno = 0;
  FILE* f = fopen(path, "wb");
  if (!f) return io_error();
  bool ok = write_header(f, make_header(dp_bits, range_start, range_end, keyx, keyy, total_count, total_time));
  if (ok) {
    t->ht->SaveTable(f, 0, HASH_SIZE, false);                     // HashTable.cpp:375-396 (ignores fwrite results: ferror below)
    ok = !ferror(f) && fwrite(&total_walk, 8, 1, f) == 1;         // Backup.cpp:530-531 / 549-551
  }
  ok = fflush(f) == 0 && ok;
  const int err = ok ? 0 : io_error();
  if (fclose(f) != 0 && ok) return io_error();
  return err;
}

int kgi_save_work(kgi_table* t, const char* path, uint32_t dp_bits, const uint64_t range_start[4], const uint64_t range_end[4],
                  const uint64_t keyx[4], const uint64_t keyy[4], uint64_t total_count, double total_time) {
  return kgi_save_work_ex(t, path, dp_bits, range_start, range_end, keyx, keyy, total_count, total_time, 0);
}

int kgi_load_work_ex(kgi_table* t, const char* path, uint32_t* dp_bits, uint64_t range_start[4], uint64_t range_end[4],
                     uint64_t keyx[4], uint64_t keyy[4], uint64_t* total_count, double* total_time, uint64_t* nb_walk,
                     uint64_t* walk_offset) {
  using namespace kgx_wf;
  errno = 0;
  FILE* f = fopen(path, "rb");
  if (!f) return io_error();
  WorkHeader hd;                                                  // Kangaroo::LoadWork (Backup.cpp:149-207)
  uint64_t walk = 0, off = 0;
  bool ok = read_header(f, hd);
  if (ok) {
    t->ht->LoadTable(f);                                          // HashTable.cpp (Reset + per-bucket read; ignores fread results)
    ok = !ferror(f) && !feof(f) && fread(&walk, 8, 1, f) == 1;
  }
  ok = ok && walks_complete(f, walk, off);
  fclose(f);
  if (!ok) { t->ht->Reset(); return -EINVAL; }
  get_header(hd, dp_bits, range_start, range_end, keyx, keyy, total_count, total_time);
  if (nb_walk) *nb_walk = walk;
  if (walk_offset) *walk_offset = off;
  return 0;
}

int kgi_load_work(kgi_table* t, const char* path, uint32_t* dp_bits, uint64_t* total_count, double* total_time) {
  return kgi_load_work_ex(t, path, dp_bits, nullptr, nullptr, nullptr, nullptr, total_count, total_time, nullptr, nullptr);
}

}  // extern "C"
