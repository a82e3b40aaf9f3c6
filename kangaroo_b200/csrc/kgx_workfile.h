// kgx_workfile.h -- the reference's HEADW work-file format, one copy for the host table (kgx_ingest.cpp), the device table
// (kgx_dptable.cuh) and the work-file check and merge (kgx_worktool.cuh), and of the batch block that follows a batch work
// file's records (kgx_batch_block / kgx_batch_read, the solver's --batch-keys files).  Plain host C++; every function is
// static, so neither library exports a symbol from here.  A file: the header (Backup.cpp:368-394), 2^18 buckets in order,
// each nbItem, maxItem and nbItem entries (HashTable.cpp:375-396), then a u64 kangaroo count and that many 96-byte records.
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

// ---- batch work file (the solver's --batch-keys): a HEADW file as above (header key = input key 0, kangaroo records in
// file order, wild distances relative to each wild's own target key), followed by the batch block:
//   head    u32 BATCH_MAGIC, u32 BATCH_VERSION, u32 n_keys (1..65535), u32 0, u64 nb_walk (= the HEADW kangaroo count)
//   keys    n_keys x 104 bytes: public key x[4], y[4], private key[4] (u64 limbs; 0 when unsolved), u64 solved (0 / 1)
//   targets nb_walk x u16, the key index of every kangaroo in file order (tame ones 0), zero-padded to a multiple of 8 bytes
//   footer  u64 offset of the head from the start of the file, u32 BATCH_MAGIC, u32 BATCH_VERSION
// A reader finds the block from the end of the file.  The reference reads only the HEADW part (nbLoadedWalk records) and
// ignores what follows, so its -winfo, -wcheck and -i still take a batch file.
constexpr uint32_t BATCH_MAGIC = 0xBA7C4B01u;
constexpr uint32_t BATCH_VERSION = 1;
constexpr uint64_t BATCH_HEAD_BYTES = 24, BATCH_KEY_BYTES = 104, BATCH_FOOTER_BYTES = 16;
constexpr uint32_t BATCH_MAX_KEYS = 65535;

static inline uint64_t batch_targets_bytes(uint64_t nb_walk) { return (2 * nb_walk + 7) & ~7ull; }
static inline uint64_t batch_block_bytes(uint32_t n_keys, uint64_t nb_walk) {
  return BATCH_HEAD_BYTES + (uint64_t)n_keys * BATCH_KEY_BYTES + batch_targets_bytes(nb_walk) + BATCH_FOOTER_BYTES;
}

// the block into out (batch_block_bytes bytes).  keys: n_keys x 8 limbs (x, y); privs: n_keys x 4 limbs; solved: n_keys flags.
static inline void batch_encode(const uint64_t* keys, const uint8_t* solved, const uint64_t* privs, uint32_t n_keys,
                                const uint16_t* targets, uint64_t nb_walk, uint64_t offset, uint8_t* out) {
  uint8_t* p = out;
  auto put = [&p](const void* v, size_t n) { memcpy(p, v, n); p += n; };
  const uint32_t head[4] = {BATCH_MAGIC, BATCH_VERSION, n_keys, 0};
  put(head, 16);
  put(&nb_walk, 8);
  for (uint32_t k = 0; k < n_keys; k++) {
    const uint64_t zero[4] = {0, 0, 0, 0}, flag = solved[k] ? 1 : 0;
    put(keys + 8 * k, 64);
    put(solved[k] ? privs + 4 * k : zero, 32);
    put(&flag, 8);
  }
  if (nb_walk) put(targets, 2 * nb_walk);
  const uint64_t pad = batch_targets_bytes(nb_walk) - 2 * nb_walk;
  memset(p, 0, pad);
  p += pad;
  put(&offset, 8);
  const uint32_t tail[2] = {BATCH_MAGIC, BATCH_VERSION};
  put(tail, 8);
}

struct BatchInfo { uint32_t n_keys = 0; uint64_t nb_walk = 0, offset = 0; };

// Locates the batch block of an open work file: 1 = found (info filled, f positioned on its keys), 0 = a plain HEADW file (it
// ends with its kangaroo records, or right after its table), -1 = not a HEADW file or a damaged one, with the reason in err.
// The HEADW part is walked (header, bucket heads, kangaroo count) to find where its records end; the block must start
// exactly there, hold the same kangaroo count and end exactly at the end of the file.
static inline int batch_find(FILE* f, BatchInfo& info, char* err, size_t errlen) {
  WorkHeader h;
  if (fseek(f, 0, SEEK_SET) != 0 || !read_header(f, h)) { snprintf(err, errlen, "not a HEADW work file"); return -1; }
  for (uint32_t b = 0; b < NBUCKET; b++) {
    uint32_t nb, mx;
    if (!read_bucket_head(f, nb, mx) || (nb && fseek(f, (long)nb * (long)sizeof(Entry), SEEK_CUR) != 0)) {
      snprintf(err, errlen, "the table is cut short");
      return -1;
    }
  }
  const long tab_end = ftell(f);
  uint64_t nwalk = 0;
  const bool has_count = fread(&nwalk, 8, 1, f) == 1;
  if (fseek(f, 0, SEEK_END) != 0) { snprintf(err, errlen, "cannot seek"); return -1; }
  const uint64_t size = (uint64_t)ftell(f);
  if (!has_count) { if (size == (uint64_t)tab_end) return 0; snprintf(err, errlen, "the kangaroo count is cut short"); return -1; }
  const uint64_t rec_end = (uint64_t)tab_end + 8 + nwalk * WALK_BYTES;
  if (size < rec_end) { snprintf(err, errlen, "the kangaroo block is cut short (%llu records announced)", (unsigned long long)nwalk); return -1; }
  if (size == rec_end) return 0;
  uint64_t foot[2] = {0, 0};
  uint32_t head[4] = {0, 0, 0, 0};
  uint64_t hwalk = 0;
  if (size - rec_end < BATCH_HEAD_BYTES + BATCH_FOOTER_BYTES || fseek(f, (long)(size - BATCH_FOOTER_BYTES), SEEK_SET) != 0 ||
      fread(foot, 8, 2, f) != 2 || (uint32_t)foot[1] != BATCH_MAGIC) {
    snprintf(err, errlen, "%llu bytes follow the kangaroo records, but no batch block footer ends the file (cut short or damaged)",
             (unsigned long long)(size - rec_end));
    return -1;
  }
  if ((uint32_t)(foot[1] >> 32) != BATCH_VERSION) { snprintf(err, errlen, "batch block version %u (this program reads %u)", (uint32_t)(foot[1] >> 32), BATCH_VERSION); return -1; }
  if (foot[0] != rec_end) { snprintf(err, errlen, "the batch block footer points to offset %llu, the kangaroo records end at %llu", (unsigned long long)foot[0], (unsigned long long)rec_end); return -1; }
  if (fseek(f, (long)rec_end, SEEK_SET) != 0 || fread(head, 4, 4, f) != 4 || fread(&hwalk, 8, 1, f) != 1 || head[0] != BATCH_MAGIC ||
      head[1] != BATCH_VERSION) {
    snprintf(err, errlen, "the batch block head is damaged");
    return -1;
  }
  if (head[2] == 0 || head[2] > BATCH_MAX_KEYS || hwalk != nwalk || rec_end + batch_block_bytes(head[2], hwalk) != size) {
    snprintf(err, errlen, "the batch block (%u keys, %llu targets) does not match the file (%llu kangaroos, %llu bytes after them)",
             head[2], (unsigned long long)hwalk, (unsigned long long)nwalk, (unsigned long long)(size - rec_end));
    return -1;
  }
  info.n_keys = head[2];
  info.nb_walk = nwalk;
  info.offset = rec_end;
  return 1;
}

// After batch_find returned 1: the keys, solved flags, private keys and targets (any may be null: skipped).  -1 with the
// reason in err on a short read or a target that is not below n_keys.
static inline int batch_read(FILE* f, const BatchInfo& info, uint64_t* keys, uint8_t* solved, uint64_t* privs, uint16_t* targets,
                             char* err, size_t errlen) {
  if (fseek(f, (long)(info.offset + BATCH_HEAD_BYTES), SEEK_SET) != 0) { snprintf(err, errlen, "cannot seek"); return -1; }
  for (uint32_t k = 0; k < info.n_keys; k++) {
    uint64_t rec[13];
    if (fread(rec, 8, 13, f) != 13) { snprintf(err, errlen, "the batch block is cut short"); return -1; }
    if (rec[12] > 1) { snprintf(err, errlen, "key %u: solved flag %llu", k, (unsigned long long)rec[12]); return -1; }
    if (keys) memcpy(keys + 8 * k, rec, 64);
    if (privs) memcpy(privs + 4 * k, rec + 8, 32);
    if (solved) solved[k] = (uint8_t)rec[12];
  }
  if (!targets) return 0;
  if (info.nb_walk && fread(targets, 2, info.nb_walk, f) != info.nb_walk) { snprintf(err, errlen, "the batch block is cut short"); return -1; }
  for (uint64_t i = 0; i < info.nb_walk; i++)
    if (targets[i] >= info.n_keys) {
      snprintf(err, errlen, "kangaroo %llu: target %u is not below n_keys = %u", (unsigned long long)i, targets[i], info.n_keys);
      return -1;
    }
  return 0;
}

}  // namespace kgx_wf
