// kgx_workfile.h -- the reference's HEADW work-file format, one copy for the host table (kgx_ingest.cpp), the device table
// (kgx_dptable.cuh) and the work-file check and merge (kgx_worktool.cuh).  Plain host C++; every function is static, so
// neither library exports a symbol from here.  A file: the header (Backup.cpp:368-394), 2^18 buckets in order, each nbItem,
// maxItem and nbItem entries (HashTable.cpp:375-396), then a u64 kangaroo count and that many 96-byte records.
#pragma once
#include <cerrno>
#include <cstdint>
#include <cstdio>
#include <cstring>

namespace kgx_wf {

constexpr uint32_t HEADW_MAGIC = 0xFA6A8001u;           // Kangaroo.h:120
constexpr uint32_t NBUCKET = 1u << 18;                  // HASH_SIZE (HashTable.h)
constexpr uint64_t WALK_BYTES = 96;                     // one kangaroo: x[4], y[4], d[4] (Backup.cpp:536-539)

struct Entry { uint64_t x0, x1, d0, d1; };              // ENTRY {int128 x; int128 d}
static_assert(sizeof(Entry) == 32, "a table entry is 32 bytes");

// version is what a file holds; write_header always writes 0, as Kangaroo::SaveHeader does
struct WorkHeader {
  uint32_t version = 0, dp = 0;
  uint64_t rs[4] = {}, re[4] = {}, kx[4] = {}, ky[4] = {};
  uint64_t count = 0;
  double time = 0;
};

static inline WorkHeader make_header(uint32_t dp, const uint64_t rs[4], const uint64_t re[4], const uint64_t kx[4],
                                     const uint64_t ky[4], uint64_t count, double time) {
  WorkHeader h;
  h.dp = dp; h.count = count; h.time = time;
  memcpy(h.rs, rs, 32); memcpy(h.re, re, 32); memcpy(h.kx, kx, 32); memcpy(h.ky, ky, 32);
  return h;
}

// the header into the optional (null: not wanted) out-parameters of the C ABI's load calls
static inline void get_header(const WorkHeader& h, uint32_t* dp, uint64_t rs[4], uint64_t re[4], uint64_t kx[4], uint64_t ky[4],
                              uint64_t* count, double* time) {
  if (dp) *dp = h.dp;
  if (rs) memcpy(rs, h.rs, 32);
  if (re) memcpy(re, h.re, 32);
  if (kx) memcpy(kx, h.kx, 32);
  if (ky) memcpy(ky, h.ky, 32);
  if (count) *count = h.count;
  if (time) *time = h.time;
}

static inline bool write_header(FILE* f, const WorkHeader& h) {
  const uint32_t head = HEADW_MAGIC, version = 0;
  return fwrite(&head, 4, 1, f) == 1 && fwrite(&version, 4, 1, f) == 1 && fwrite(&h.dp, 4, 1, f) == 1 && fwrite(h.rs, 32, 1, f) == 1 &&
         fwrite(h.re, 32, 1, f) == 1 && fwrite(h.kx, 32, 1, f) == 1 && fwrite(h.ky, 32, 1, f) == 1 && fwrite(&h.count, 8, 1, f) == 1 &&
         fwrite(&h.time, 8, 1, f) == 1;
}

// false on a short read or another magic
static inline bool read_header(FILE* f, WorkHeader& h) {
  uint32_t head = 0;
  return fread(&head, 4, 1, f) == 1 && head == HEADW_MAGIC && fread(&h.version, 4, 1, f) == 1 && fread(&h.dp, 4, 1, f) == 1 &&
         fread(h.rs, 32, 1, f) == 1 && fread(h.re, 32, 1, f) == 1 && fread(h.kx, 32, 1, f) == 1 && fread(h.ky, 32, 1, f) == 1 &&
         fread(&h.count, 8, 1, f) == 1 && fread(&h.time, 8, 1, f) == 1;
}

static inline bool write_bucket(FILE* f, uint32_t nb, uint32_t mx, const Entry* e) {
  return fwrite(&nb, 4, 1, f) == 1 && fwrite(&mx, 4, 1, f) == 1 && (nb == 0 || fwrite(e, sizeof(Entry), nb, f) == nb);
}

// a bucket's nbItem and maxItem; its entries follow
static inline bool read_bucket_head(FILE* f, uint32_t& nb, uint32_t& mx) { return fread(&nb, 4, 1, f) == 1 && fread(&mx, 4, 1, f) == 1; }

// Right after the kangaroo count: offset = where the records start; true when all `walk` of them are there before the end
// of the file (Kangaroo::FetchWalks, Backup.cpp:211-223).
static inline bool walks_complete(FILE* f, uint64_t walk, uint64_t& offset) {
  const long off = ftell(f);
  offset = (uint64_t)off;
  if (!walk) return true;
  if (off < 0 || fseek(f, 0, SEEK_END) != 0) return false;
  const long end = ftell(f);
  return end >= off && (uint64_t)(end - off) / WALK_BYTES >= walk;
}

// a failed stdio call: -errno (EIO when the C library left errno at 0)
static inline int io_error() { return errno ? -errno : -EIO; }

}  // namespace kgx_wf
