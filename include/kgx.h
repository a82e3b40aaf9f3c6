/*
 * kgx.h -- C ABI of the H100-native kangaroo jump engine (libkgx.so).
 *
 * This is the drop-in boundary for ONE path of JeanLucPons/Kangaroo: the GPU jump engine behind
 * `class GPUEngine` (reference GPU/GPUEngine.h:40-84, GPU/GPUEngine.cu).  The reference's interface is a C++
 * class taking host `Int` objects; the portable part of it is restated here as plain pointers and sizes so
 * that the C++ shim (kangaroo_b200/csrc/GPUEngine_b200.cu -> class GPUEngine, unchanged header), the
 * ctypes tests, bench.py and the NCCL rank driver all bind the same entry points.
 *
 * Conventions
 *   - field elements: 4 x uint64_t little-endian limbs (reference Int::bits64[0..3]);
 *   - distances: 2 x uint64_t, ALREADY biased by the wild offset for odd kIdx (the shim / Python host side
 *     adds and removes `wildOffset` exactly like GPUEngine.cu:407-411, 477, 526, 672);
 *   - kangaroo arrays are in kIdx order, n = groups * threads_per_group * KGX_GPU_GRP_SIZE entries
 *     (GPUEngine.cu:390-418); herd type = kIdx & 1;
 *   - every call returns 0 on success, a negative value on error with text in kgx_last_error();
 *     nothing throws, nothing falls back to the CPU: without a CUDA device kgx_create() fails.
 */
#ifndef KGX_H
#define KGX_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define KGX_NB_JUMP       32   /* Constants.h:29  */
#define KGX_GPU_GRP_SIZE  128  /* Constants.h:32  */
#define KGX_NB_RUN        64   /* Constants.h:35: jumps per kangaroo per launch */
#define KGX_ITEM_SIZE     56   /* GPUEngine.h:31: DP record {x[32], d[16], kIdx[8]} */

typedef struct kgx_engine kgx_engine;

/* DP record exactly as the reference kernel writes it (GPUMath.h:173-188, GPUEngine.cu:653-671). */
typedef struct {
  uint64_t x[4];
  uint64_t d[2];     /* biased 128-bit distance */
  uint64_t kidx;
} kgx_item;

/* --- static helpers (GPUEngine::GetGridSize / PrintCudaInfo, GPUEngine.cu:275-375) --- */
int  kgx_device_count(void);
/* Fills non-positive *x / *y with defaults: x = 2*SMs, y = 128 (GPUEngine.cu:301-303 on an unknown SM). */
int  kgx_grid_default(int dev, int* x, int* y);
/* "name|SMs|cc_major|cc_minor|totalMemMB" into buf */
int  kgx_device_info(int dev, char* buf, int buflen);

/* --- life cycle (GPUEngine ctor/dtor, GPUEngine.cu:144-263) --- */
kgx_engine* kgx_create(int dev, int groups, int threads_per_group, uint32_t max_found);
/* Same, with the jump kernel chosen by the caller instead of by herd size: KGX_KERNEL_STREAM = per-thread groups
 * streamed through HBM (the benchmarked kernel), KGX_KERNEL_RESIDENT = shared-memory tile kernel; stream_g = kangaroos
 * per thread of the stream kernel (even, 2..4096; 0 = adaptive).  Used by the parity tests to pin BOTH kernels to the
 * oracle and the reference fixtures on every grid. */
#define KGX_KERNEL_AUTO     0
#define KGX_KERNEL_STREAM   1
#define KGX_KERNEL_RESIDENT 2
#define KGX_KERNEL_TMEM     3   /* cluster tile kernel: one 1792-kangaroo tile in the shared memory of a 2-CTA cluster */
kgx_engine* kgx_create_ex(int dev, int groups, int threads_per_group, uint32_t max_found, int kernel, int stream_g);
/* 1 = stream kernel, 2 = resident kernel, 3 = cluster tile kernel (what kgx_create / kgx_create_ex resolved to) */
int         kgx_kernel_kind(kgx_engine* e);
void        kgx_destroy(kgx_engine* e);
const char* kgx_last_error(kgx_engine* e);      /* e may be NULL: error of the last failed kgx_create */
uint64_t    kgx_num_kangaroos(kgx_engine* e);   /* groups * threads_per_group * 128 */
uint64_t    kgx_memory_bytes(kgx_engine* e);    /* device bytes held (GPUEngine::GetMemory) */

/* --- USE_SYMMETRY engine mode (reference: compile-time switch Constants.h:25).  mode:
 *       0                    off
 *       KGX_SYM_LASTJUMP (1) the reference's DEVICE rule (GPUCompute.h:53-60, 91-94), which Kangaroo::Check replays on the CPU
 *                            (Check.cpp:534-556): jump = x mod 32, bumped when it repeats the previous jump of the kangaroo
 *       KGX_SYM_CLASS    (2) the rule of the reference's working symmetric path SolveKeyCPU (Kangaroo.cpp:381-384, 422-428):
 *                            jump = x mod 16 + 16 * symClass, symClass flipping at every class switch
 *     Both apply the equivalence-class switch after every jump (y > (p-1)/2 -> point negated, distance negated).  Distances
 *     crossing this ABI (upload, download, patch, create_herd, DP items) are then SIGNED 128-bit two's complement values and
 *     NO wild offset is applied (the reference's biased-unsigned device form cannot represent the sign changes: its
 *     ModNeg256Order writes 256 bits into a 128-bit slot, GPUMath.h:533-547).  The per-kangaroo rule state (lastJump /
 *     symClass) is reset by upload / patch / create_herd like GPUEngine.cu:413-416, 532-536.  Call before the herd is uploaded. --- */
#define KGX_SYM_LASTJUMP 1
#define KGX_SYM_CLASS    2
int kgx_set_symmetry(kgx_engine* e, int on);
int kgx_get_symmetry(kgx_engine* e);

/* --- GPUEngine::SetParams (GPUEngine.cu:559-590): jd 32x2, jpx/jpy 32x4 limbs --- */
int kgx_set_params(kgx_engine* e, uint64_t dp_mask, const uint64_t* jd, const uint64_t* jpx, const uint64_t* jpy);

/* --- GPUEngine::SetKangaroos / GetKangaroos / SetKangaroo (GPUEngine.cu:381-538) --- */
int kgx_upload(kgx_engine* e, const uint64_t* px, const uint64_t* py, const uint64_t* d);   /* n x 4, n x 4, n x 2 */
int kgx_download(kgx_engine* e, uint64_t* px, uint64_t* py, uint64_t* d);
int kgx_patch(kgx_engine* e, uint64_t kidx, const uint64_t px[4], const uint64_t py[4], const uint64_t d[2]);
/* Asynchronous GetKangaroos for checkpoints (SURVEY 8f/f3; Kangaroo.cpp:618-626, Backup.cpp:449-572): _begin snapshots the
 * herd in stream order (after the launch in flight) without blocking the caller or later launches; _read waits for that
 * snapshot only and copies it to the host arrays (kIdx order, distances still biased). */
int kgx_snapshot_begin(kgx_engine* e);
int kgx_snapshot_read(kgx_engine* e, uint64_t* px, uint64_t* py, uint64_t* d);

/* --- the herd as work-file records (Kangaroo::SaveWork -ws / FetchWalks, Backup.cpp:536-539, 211-223): 96 bytes per
 *     kangaroo, {x[4], y[4], d[4]} u64 limbs, d = distance mod n with the wild offset removed, kIdx order.  Both calls fail
 *     in symmetric mode.  wild_offset: 2 limbs (the bias of odd kIdx).
 * _export: after kgx_snapshot_begin, converts the snapshot on the device (copy stream; launches queued after the snapshot
 *     keep running) and copies records [first, first+count) to dst, host or device memory of the engine's GPU.  Call it
 *     in chunks; the call whose range ends at n releases the snapshot.  The engine then keeps the snapshot's staging
 *     (80 bytes per kangaroo) and the record buffer (96 bytes per kangaroo) for the next save: freeing device memory
 *     synchronises the device, which would stall the jump launches once per save.  kgx_destroy frees both.
 * _import: replaces kangaroos 0..count-1 (the rest of the herd is kept) in stream order after the launch in flight; recs:
 *     count x 96 bytes of host memory.  Fails, changing nothing, when a biased distance does not fit in 128 bits (a file of
 *     another range).  verify != 0 recomputes every position as d*G (even kIdx) / key + d*G (odd kIdx): *mismatches =
 *     records that differ, and the herd is only replaced when there are none. --- */
int kgx_snapshot_export(kgx_engine* e, const uint64_t wild_offset[2], uint64_t first, uint64_t count, void* dst);
int kgx_import(kgx_engine* e, const uint64_t wild_offset[2], const void* recs, uint64_t count, const uint64_t keyx[4],
               const uint64_t keyy[4], int verify, uint64_t* mismatches);

/* --- herd creation on the device (SURVEY 8f/f2; replaces the CPU side of Kangaroo::CreateHerd, Kangaroo.cpp:670-738):
 *     kangaroo i starts at scalars[i]*G, plus `key` when (i + first_type) is odd (wild).  scalars: n x 4 limbs (mod the
 *     group order), d128: n x 2 limbs stored as the (biased) distances. --- */
int kgx_create_herd(kgx_engine* e, const uint64_t* scalars, const uint64_t* d128, const uint64_t keyx[4], const uint64_t keyy[4], int first_type);

/* --- multi-key herd: one tame herd shared by several keys (the solver's --batch-keys).  Not in the reference, which solves
 *     the keys of an input file one after another with a new herd each (Kangaroo::Run, Kangaroo.cpp:1021-1066).
 * _create_herd_multi: kgx_create_herd with a key table of n_keys (1..KGX_MAX_KEYS) keys, keys: n_keys x 8 limbs (x[4], y[4]),
 *     and a target per kangaroo, targets: n entries in kIdx order, each below n_keys: wild kangaroo i starts at
 *     keys[targets[i]] + scalars[i]*G (the entries of tame kangaroos are not used).  The engine keeps the table and the
 *     targets (kgx_create_herd drops them).  Fails in symmetric mode.
 * _retarget: every wild kangaroo whose target is `from` moves to key b = to[(kIdx >> 1) % n_to] (1 <= n_to <= n_keys): its
 *     point gets keys[b] - keys[from] added, its distance stays, so it is at keys[b] + d*G again, and its target becomes b.
 *     Stream-ordered after the launch in flight, like kgx_patch, and the call does not wait for that launch.  Padding
 *     slots keep walking their old copy (their DPs are dropped).  kgx_upload / kgx_patch / kgx_import change no target.
 *     kgx_set_symmetry(on) drops the key table; _retarget and _targets fail in symmetric mode.
 * _targets: the n targets (kIdx order) after every retarget queued so far. --- */
#define KGX_MAX_KEYS 65535
int kgx_create_herd_multi(kgx_engine* e, const uint64_t* scalars, const uint64_t* d128, const uint64_t* keys, uint32_t n_keys,
                          const uint16_t* targets, int first_type);
int kgx_retarget(kgx_engine* e, uint32_t from, const uint16_t* to, uint32_t n_to);
int kgx_targets(kgx_engine* e, uint16_t* out);
/* --- checkpoint and resume of a multi-key herd (the solver's batch work files).
 * kgx_snapshot_begin on a herd with a key table also copies the targets, device to device in stream order with the state, so a
 *     kgx_retarget queued after it does not show in the snapshot.
 * _snapshot_export_targets: targets [first, first+count) of the pending snapshot (kIdx order) to dst (host memory); call it
 *     before the kgx_snapshot_export chunk that releases the snapshot.  Fails when the snapshot was taken without a key table.
 * _import_multi: kgx_import with a key table (keys: n_keys x 8 limbs, 1 <= n_keys <= KGX_MAX_KEYS) and a target per record
 *     (targets: count entries, each below n_keys): verify != 0 checks wild record i against keys[targets[i]] + d*G and tame ones
 *     against d*G, on the device.  On success the engine holds the key table and targets[0..count) as kgx_create_herd_multi
 *     leaves them (kgx_retarget and kgx_targets work); kangaroos count..n-1 keep their state and targets, so a partial import
 *     needs a herd of kgx_create_herd_multi with the same keys first.  Fails in symmetric mode; with mismatches nothing
 *     changes, key table and targets included. --- */
int kgx_snapshot_export_targets(kgx_engine* e, uint64_t first, uint64_t count, uint16_t* dst);
int kgx_import_multi(kgx_engine* e, const uint64_t wild_offset[2], const void* recs, uint64_t count, const uint64_t* keys,
                     uint32_t n_keys, const uint16_t* targets, int verify, uint64_t* mismatches);

/* --- GPUEngine::callKernel (GPUEngine.cu:540-557): zero the DP count, start NB_RUN jumps, asynchronous --- */
int kgx_launch_async(kgx_engine* e);
/* First half of GPUEngine::Launch (GPUEngine.cu:607-675): wait for the in-flight launch (sleeping unless
 * spin != 0), optionally start the NEXT launch before reading back (relaunch != 0; DP slabs are double
 * buffered so the copy overlaps the new kernel), then copy min(found, max_found, cap) records to `items`.
 * *n_items = records copied, *n_found = records the kernel wanted to write (may exceed max_found: lost). */
int kgx_collect(kgx_engine* e, kgx_item* items, uint32_t cap, uint32_t* n_items, uint32_t* n_found, int spin, int relaunch);
/* Blocks until every queued launch / copy finished. */
int kgx_sync(kgx_engine* e);

/* --- device-resident access for the multi-GPU DP gather and for bench.py (no host copies) --- */
/* Device pointer to the DP slab of the most recently COMPLETED launch: [u32 count][max_found x 56 B]. */
void*    kgx_dp_slab_device(kgx_engine* e);
uint32_t kgx_max_found(kgx_engine* e);
/* HashTable::Convert on the device (HashTable.cpp:75-100; SURVEY 8f/f1) for the most recently completed launch:
 * *out = device pointer to [u32 count][count x 40-byte DP {u32 kIdx; u32 h; u128 x; u128 tagged d}] (Kangaroo.h:94-101). */
int      kgx_convert_dps(kgx_engine* e, const uint64_t wild_offset[2], void** out);
/* Milliseconds the last completed launch spent on the device (CUDA events on the engine's stream). */
float    kgx_last_launch_ms(kgx_engine* e);
/* Jumps per launch override for tests (default KGX_NB_RUN). */
int      kgx_set_jumps_per_launch(kgx_engine* e, int n_run);
/* Number of kernels this engine has launched so far (jump + pack/unpack/patch), for bench.py's gpu_launches. */
uint64_t kgx_kernel_launches(kgx_engine* e);

/* --- device-resident DP table (kgx_dptable.cuh): the reference's HashTable (HashTable.cpp:262-307, 2^18 buckets of
 *     ENTRY {int128 x; int128 d}) in the memory of one GPU, fed the 40-byte records of kgx_convert_dps.  Every sequence of
 *     adds gives exactly the events, count, per-bucket nbItem / maxItem and work files of the host table of
 *     include/kgx_ingest.h (kgi_add / kgi_save_work_ex / kgi_load_work_ex) fed the same records in the same order.
 * _create: a table of `capacity` entries (fixed; 1 .. 2^32-2) on device dev; NULL without a device or memory, reason in
 *     kgx_dptable_last_error(NULL).  _bytes_for: device bytes a table of that capacity takes (48 per entry + fixed scratch:
 *     a save chunk of 2^21 entries at 56 bytes each, the save's selection of min(capacity, 2^23) entries at 4 bytes each).
 * _add: records of n_ranks rank segments (1 .. KGX_DPT_MAX_RANKS), segment r = counts[r] records at recs + r*stride*40
 *     (device memory; counts on the host), inserted in segment order then record order, stream-ordered on `stream`
 *     (a cudaStream_t; NULL = the legacy default stream); the call waits for its own work only.  Events in arrival order:
 *     the first `cap` are copied to ev (host), *n_ev = all of them.  Returns 0; -1 when records with h >= 2^18 were
 *     skipped (the others inserted, as kgi_add); -2 when count + records > capacity: nothing inserted, reason in
 *     kgx_dptable_last_error; -3 on a CUDA error.
 * _reserve: allocates now the per-call scratch of adds of up to n_records records (about 70 bytes per record) and of `cap`
 *     events (136 bytes each, for both kinds of add), which adds otherwise grow on demand; a caller that sizes the table to the free memory reserves first.
 * _save_work / _load_work: kgi_save_work_ex / kgi_load_work_ex on this table (same header arguments and results, same
 *     bytes; the entries move in bounded chunks through pinned memory), after the work queued on `stream`.  A load that
 *     holds more entries than the capacity fails with -ENOSPC and leaves the table empty, like any failed load. --- */
typedef struct kgx_dptable kgx_dptable;
typedef struct {                     /* = kgi_event (include/kgx_ingest.h) */
  uint32_t kind, rank, kidx, h;
  uint64_t d_old[2], d_new[2];
} kgx_dp_event;
#define KGX_DPT_EV_RESET     1
#define KGX_DPT_EV_COLLISION 2
#define KGX_DPT_MAX_RANKS    256
#define KGX_DPT_HOST_ENTRIES 1   /* kgx_dptable_create_ex: the 32-byte entries in mapped, pinned host memory */
/* --- the collision resolver on one GPU (kgx_resolver.cuh): kgi_resolve_multi's result without the host.
 * _create: keys K = key - start*G (n_keys x 8 limbs, x then y; the point at infinity as (0, 0); 1 <= n_keys <= KGX_MAX_KEYS)
 *     and a range start below the group order n.  Builds the fixed-base comb and the keys' index by x once, on device dev,
 *     and waits for them.  NULL on bad arguments or a CUDA error, reason in kgx_resolver_last_error(NULL).
 * _run: n collisions in device memory, pairs = n x 4 limbs {d_first[2], d_other[2]} of tagged distances (either order) ->
 *     key_out[i] (device, n entries) = the first key in input order that one of the four candidates +-Td +-Wd * G hits (the
 *     key or its negative), KGX_NO_KEY when none does or both distances are of one herd; priv_out (device, n x 4 limbs) = its
 *     private key, (+-m + start) mod n, 0 with no key.  Stream-ordered on `stream` (NULL = the legacy default stream), no
 *     allocation, no synchronisation.  -1: too many collisions; -3: a CUDA error, text in kgx_resolver_last_error(r).
 * _destroy frees the resolver after the runs queued on it.
 * _verify: a resolver of exactly one key (else -1) checks n received 40-byte DP records {u32 kIdx; u32 h; u128 x; u128 tagged d}
 *     (device memory, 8-byte aligned) by the rule of kgx_work_check: S = +-|d|*G (sign bit 127, |d| the low 126 bits), + K when
 *     the type bit 126 is set; a record is good iff h < 2^18, S is not the point at infinity, S.x.bits64[2] & 0x3FFFF == h and
 *     the low 128 bits of S.x equal x.  good (device, n x 40 bytes, 8-byte aligned) gets the good records in input order (a
 *     stable compaction), counts (device, 2 entries) = {good, bad}, bad_idx (device, cap entries) the indices of the first
 *     `cap` bad records in input order.  It is _verify_partition with W = 1 and stride 0.  scratch: device memory of at
 *     least kgx_resolver_verify_scratch_bytes(n) bytes (0: bad arguments), which is
 *     kgx_resolver_verify_partition_scratch_bytes(n, 1), 256-byte aligned (as cudaMalloc returns it; the flags, the
 *     partition's (owner, tile) counts and cub's scan storage of them live there).  Stream-ordered on `stream`, no
 *     allocation, no synchronisation.  -1: bad arguments; -3: a CUDA error, text in kgx_resolver_last_error(r).
 * _verify_partition: _verify and kgx_dp_partition in one call, for a DP table sharded over W tables (1 .. KGX_DPT_MAX_RANKS).
 *     The same check, then the good records grouped by the shard that owns their bucket (shard r of W holds the buckets
 *     [floor(r*2^18/W), floor((r+1)*2^18/W))), each group in input order, into out (device, 8-byte aligned): packed when
 *     stride = 0, else group r at record r * stride (stride >= n).  counts (device, W + 1 entries): the good records of each
 *     group, then the bad count; bad_idx (device, cap entries): the indices of the first `cap` bad records in input order.
 *     The result is byte for byte that of _verify followed by kgx_dp_partition of its good records.  scratch: at least
 *     kgx_resolver_verify_partition_scratch_bytes(n, W) bytes (0: bad arguments), 256-byte aligned.  Stream-ordered on
 *     `stream`, no allocation, no synchronisation.  -1: bad arguments; -3: a CUDA error, text in kgx_resolver_last_error(r). --- */
typedef struct kgx_resolver kgx_resolver;
#define KGX_NO_KEY 0xFFFFFFFFu
kgx_resolver* kgx_resolver_create(int dev, const uint64_t* keys, uint32_t n_keys, const uint64_t range_start[4]);
void          kgx_resolver_destroy(kgx_resolver* r);
const char*   kgx_resolver_last_error(kgx_resolver* r);
int           kgx_resolver_run(kgx_resolver* r, const void* pairs, uint32_t n, uint32_t* key_out, uint64_t* priv_out, void* stream);
uint64_t      kgx_resolver_verify_scratch_bytes(uint32_t n);
int           kgx_resolver_verify(kgx_resolver* r, const void* recs, uint32_t n, void* good, uint32_t* counts, uint32_t* bad_idx,
                                  uint32_t cap, void* scratch, uint64_t scratch_bytes, void* stream);
uint64_t      kgx_resolver_verify_partition_scratch_bytes(uint32_t n, uint32_t world);
int           kgx_resolver_verify_partition(kgx_resolver* r, const void* recs, uint32_t n, uint32_t world, uint64_t stride, void* out,
                                            uint32_t* counts, uint32_t* bad_idx, uint32_t cap, void* scratch, uint64_t scratch_bytes,
                                            void* stream);
/* An event of kgx_dptable_add_resolve: the event of kgx_dptable_add, then for a collision event the resolver's key index and
 * private key, KGX_NO_KEY and 0 for any other event. */
typedef struct {
  kgx_dp_event ev;
  uint32_t key, reserved;
  uint64_t priv[4];
} kgx_dp_event_key;
kgx_dptable* kgx_dptable_create(int dev, uint64_t capacity);
void         kgx_dptable_destroy(kgx_dptable* t);
const char*  kgx_dptable_last_error(kgx_dptable* t);
uint64_t     kgx_dptable_count(kgx_dptable* t);
uint64_t     kgx_dptable_capacity(kgx_dptable* t);
uint64_t     kgx_dptable_memory_bytes(kgx_dptable* t);
uint64_t     kgx_dptable_bytes_for(uint64_t capacity);
int          kgx_dptable_reserve(kgx_dptable* t, uint32_t n_records, uint32_t cap);
int kgx_dptable_add(kgx_dptable* t, const void* recs, const uint32_t* counts, uint32_t n_ranks, uint64_t stride, kgx_dp_event* ev,
                    uint32_t cap, uint32_t* n_ev, void* stream);
/* _add_resolve: kgx_dptable_add (same inserts, events, counts and return codes) with the first `cap` events resolved by r on the
 *     same stream before the one copy of them to the host: ev gets kgx_dp_event_key records.  r must be on the table's device. */
int kgx_dptable_add_resolve(kgx_dptable* t, const void* recs, const uint32_t* counts, uint32_t n_ranks, uint64_t stride, kgx_resolver* r,
                            kgx_dp_event_key* ev, uint32_t cap, uint32_t* n_ev, void* stream);
int kgx_dptable_save_work(kgx_dptable* t, const char* path, uint32_t dp_bits, const uint64_t range_start[4], const uint64_t range_end[4],
                          const uint64_t keyx[4], const uint64_t keyy[4], uint64_t total_count, double total_time, uint64_t total_walk,
                          void* stream);
int kgx_dptable_load_work(kgx_dptable* t, const char* path, uint32_t* dp_bits, uint64_t range_start[4], uint64_t range_end[4],
                          uint64_t keyx[4], uint64_t keyy[4], uint64_t* total_count, double* total_time, uint64_t* nb_walk,
                          uint64_t* walk_offset, void* stream);
/* --- the sharded DP table: rank r of W holds the buckets [floor(r*2^18/W), floor((r+1)*2^18/W)) in a table of its own GPU.
 * _create_range: kgx_dptable_create for the buckets [lo, hi) only (lo < hi <= 2^18): _add skips a record of another bucket
 *     as malformed (-1), _save_work writes the other buckets empty, _load_work loads the range and walks past the rest.
 * _piece_bytes: the bytes of the table's piece of a work file, the nbItem, maxItem and entries of its buckets:
 *     8 * (hi - lo) + 32 * count.
 * _save_range: the piece written at byte `offset` of the existing file `path` (no header, no kangaroo count; the rest of
 *     the file is left as it is), after the work queued on `stream`, then flushed and fsynced.  The pieces of the W shards at
 *     offsets 156, 156 + piece 0, ... make the table of the file the single table writes for the same records.
 * _load_range: _load_work with a limit: more than max_entries entries in the range fail with -ENOSPC, and an empty table.
 *     The header arguments and the kangaroo count and offset are the file's, as _load_work returns them. --- */
kgx_dptable* kgx_dptable_create_range(int dev, uint64_t capacity, uint32_t lo, uint32_t hi);
uint64_t     kgx_dptable_piece_bytes(kgx_dptable* t);
int kgx_dptable_save_range(kgx_dptable* t, const char* path, uint64_t offset, void* stream);
int kgx_dptable_load_range(kgx_dptable* t, const char* path, uint32_t* dp_bits, uint64_t range_start[4], uint64_t range_end[4],
                           uint64_t keyx[4], uint64_t keyy[4], uint64_t* total_count, double* total_time, uint64_t* nb_walk,
                           uint64_t* walk_offset, uint64_t max_entries, void* stream);
/* --- the table's layout.
 * _create_ex: kgx_dptable_create_range with flags: 0 (= _create_range: everything on the device) or KGX_DPT_HOST_ENTRIES,
 *     which keeps the 32-byte entries in pinned host memory mapped into the device (cudaHostAllocMapped) and the index
 *     (24 bytes per 2/3 entry), the entries' buckets (4 bytes), the counters and all scratch on the device: 16 bytes of GPU
 *     memory per entry instead of 48.  Every call above works on either layout with exactly the same events, counts, return
 *     codes and file bytes; an add reads an entry from host memory only when a probe meets a slot of its tag, and a load
 *     reads the file's entries straight into the pinned buffer.  Unknown flags: NULL.  The pinned entries are freed by _destroy.
 * _bytes_for_ex: the device bytes of a table of that capacity and layout (_bytes_for(c) = _bytes_for_ex(c, 0, NULL)); the
 *     pinned host bytes of its entries (32 per entry, 0 on the device layout) in *host_bytes when not NULL.
 * _host_bytes: the pinned host bytes of the table's entries (0 on the device layout).  Saves and loads also pin 36 bytes per
 *     entry of a save chunk (at most 2^21 entries) on either layout, allocated by the first of them. --- */
kgx_dptable* kgx_dptable_create_ex(int dev, uint64_t capacity, uint32_t lo, uint32_t hi, int flags);
uint64_t     kgx_dptable_bytes_for_ex(uint64_t capacity, int flags, uint64_t* host_bytes);
uint64_t     kgx_dptable_host_bytes(kgx_dptable* t);
/* --- kgx_dp_partition (kgx_partition.cuh): n 40-byte DP records of kgx_convert_dps (device memory) grouped by the rank of W
 *     (1 .. KGX_DPT_MAX_RANKS) that owns their bucket, each group in input order (a stable partition), into out: packed when
 *     stride = 0, else group r at record r * stride (stride >= n).  recs and out need 4-byte alignment only (kgx_convert_dps's
 *     records follow its u32 count).  counts (device memory, W + 1 entries): the records of each
 *     group, then the malformed ones (h >= 2^18), which are left out.  scratch: device memory of at least
 *     kgx_dp_partition_scratch_bytes(n, W) bytes.  Stream-ordered on `stream`, the call does not wait.  -1: bad arguments;
 *     -3: a CUDA error. --- */
uint64_t kgx_dp_partition_scratch_bytes(uint32_t n, uint32_t world);
int kgx_dp_partition(const void* recs, uint32_t n, uint32_t world, uint64_t stride, void* out, uint32_t* counts, void* scratch,
                     uint64_t scratch_bytes, void* stream);

/* --- work-file tools on one GPU (kgx_worktool.cuh): the reference's -wcheck and -wm / -wmdir for HEADW files.  Without a
 *     device every call fails (-3); there is no CPU path.  Errors: a negative value, text in kgx_work_last_error().
 * _check: reads `path` in chunks of `chunk` entries (0 = 2^21) through two pinned buffers, so that the disk and the device
 *     overlap, and checks every table entry as Kangaroo::CheckHash does (Check.cpp:33-108): S = +-|d|*G, + K when wild
 *     (K = key - start*G), OK iff S.x.bits64[2] & 0x3FFFF == h and the low 128 bits of S.x equal the stored x.  A result at
 *     infinity is wrong.  Then every kangaroo record {x, y, d mod n}: OK as tame when (x, y) = d*G, as wild when
 *     (x, y) = K + d*G (by value, not by position), wrong otherwise or when min(d, n - d) >= 2^128.  A file that ends right
 *     after its table (the reference's -wm output) has no kangaroos: has_walk_count = 0.  The first `cap` wrong entries go to
 *     wrong_entries as (bucket, index in bucket) pairs in file order, the first `cap` wrong kangaroos' indices to wrong_walks.
 * _check_records: the same kernels on records in host memory (kind 0: n 32-byte entries with their buckets hs;
 *     kind 1: n 96-byte kangaroo records, hs unused) for a key and range start; out[i] = 1 for a wrong entry / 0 wrong,
 *     1 tame, 2 wild for a kangaroo.
 * _comb: the check's fixed-base table, 480 affine points j * 2^(4w) * G (w < 32, 1 <= j <= 15) as 8 limbs (x, y) each, at
 *     index w * 15 + j - 1.
 * _merge: merges n_paths >= 2 files in the order given, as the reference's pairwise MergeWork calls would (Merge.cpp:33-246,
 *     HashTable::MergeH): at equal x the entry of the earlier input is kept; a later one with the same tagged d is a
 *     duplicate, any other a collision.  Every input is checked first (HEADW, same version, key on the curve, same range,
 *     same key); nothing is written when one fails.  Writes tmp_path: header with the smallest dp and the summed count and
 *     time, the merged table (maxItem = nbItem rounded up to 4), then a kangaroo count of 0.  Inputs without a kangaroo count
 *     are accepted.  The inputs stream through the device in blocks of whole buckets of at most block_entries entries over
 *     all inputs (0 = 2^22); a bucket larger than that is refused and tmp_path removed.  The first `cap` collisions, ordered by
 *     bucket then x, go to coll.  A batch work file (kgx_workfile.h) is refused: kgx_work_merge_batch merges those.
 * A batch work file (_check reads it too: each kangaroo against its own target key K_t = keys[t] - start*G, each wild table
 *     entry accepted when it matches any key of the block, info->n_keys = the block's keys):
 * _batch_block_bytes / _batch_block: the block that follows the records of a file with nb_walk kangaroos whose records end
 *     at byte `offset`; keys: n_keys x 8 limbs (public x, y), solved: n_keys flags, privs: n_keys x 4 limbs (read where
 *     solved), targets: nb_walk key indices in file order.  Plain host code, no device needed.
 * _batch_read: 1 = `path` holds a batch block: *n_keys, *nb_walk, *offset and, where non-NULL, keys / solved / privs /
 *     targets (sized as above) are filled; 0 = a plain HEADW file; -1 = not a HEADW file, or a block cut short or damaged,
 *     reason in kgx_work_last_error(); -errno when the file cannot be opened.  No device needed. --- */
typedef struct {
  uint32_t dp_bits, has_walk_count;
  uint64_t entries, wrong_entries;
  uint64_t walks, walks_tame, walks_wild, wrong_walks;
  uint32_t n_wrong_entries_listed, n_wrong_walks_listed;
  uint32_t n_keys, reserved;   /* keys of a batch work file's block; 0 for a plain HEADW file */
} kgx_work_check_info;
typedef struct {
  uint32_t dp_bits, blocks;
  uint64_t entries, duplicates, collisions;
  uint64_t total_count;
  double total_time;
  uint32_t n_listed, reserved;
} kgx_work_merge_info;
typedef struct {
  uint32_t h, reserved;
  uint64_t d_first[2];   /* tagged distance of the kept entry */
  uint64_t d_other[2];   /* tagged distance of the later input's entry */
} kgx_work_collision;
const char* kgx_work_last_error(void);
int kgx_work_check(int dev, const char* path, uint64_t chunk, kgx_work_check_info* info, uint32_t* wrong_entries, uint64_t* wrong_walks,
                   uint32_t cap);
int kgx_work_check_records(int dev, int kind, const void* recs, const uint32_t* hs, uint64_t n, const uint64_t keyx[4],
                           const uint64_t keyy[4], const uint64_t range_start[4], uint8_t* out);
int kgx_work_comb(int dev, uint64_t* out);
int kgx_work_merge(int dev, const char* const* paths, uint32_t n_paths, const char* tmp_path, uint64_t block_entries,
                   kgx_work_merge_info* info, kgx_work_collision* coll, uint32_t cap);
uint64_t kgx_batch_block_bytes(uint32_t n_keys, uint64_t nb_walk);
int kgx_batch_block(const uint64_t* keys, const uint8_t* solved, const uint64_t* privs, uint32_t n_keys, const uint16_t* targets,
                    uint64_t nb_walk, uint64_t offset, void* out);
int kgx_batch_read(const char* path, uint32_t* n_keys, uint64_t* nb_walk, uint64_t* offset, uint64_t* keys, uint8_t* solved,
                   uint64_t* privs, uint16_t* targets);
/* --- merging batch work files: kgx_work_merge for files of many keys, every tame/wild collision resolved on the device.
 * _merge_batch: n_paths >= 2 batch work files of the same range, version and key list (same keys in the same order).  Refused
 *     before anything is written (-1, reason in kgx_work_last_error()): a plain HEADW file among them, another key count or
 *     order, another range or version, a range start not below the group order n, a key off the curve, a recorded private key
 *     that is not below n or does not give its public key, two inputs recording different private keys for one key, more keys
 *     than cap_keys.  The table is merged as kgx_work_merge merges the same files without their batch blocks (same blocks, same
 *     bytes; no collision is listed: info->n_listed = 0), and every collision of a block is resolved on the device before the
 *     next block, as kgi_resolve_multi resolves it against the keys K = key - start*G: the first key in input order that
 *     +-Td +-Wd * G hits.  In bucket then x order, a collision on a key not yet solved solves it and the keys listed before as
 *     the same point or its negative (the solver's classes: priv, or 2*start - priv for the negative); one on a key solved in an
 *     input or earlier in the merge changes nothing.  tmp_path gets the merged table, a kangaroo count of 0 and a batch block
 *     with every key, no kangaroo, solved = solved in an input or by the merge, privs as recorded or found.  binfo: the counts;
 *     keys[k] (n_keys entries): status 0 = unsolved, 1 = solved in an input (priv recorded), 2 = solved by this merge (priv, and
 *     h, d_first, d_other of the collision that solved its class).
 * _resolve: the merge's resolver on n collisions in host memory (d_first, d_other: n x 2 limbs of tagged distances) against
 *     n_keys (1..KGX_MAX_KEYS) keys K (n_keys x 8 limbs, keyToSearch = key - start*G, the point at infinity as (0, 0)) and a
 *     range start below n: key_out[i] = kgi_resolve_multi's key index for collision i, or 0xFFFFFFFF when it gives none (same
 *     herd included), priv_out (n x 4 limbs) = its private key (0 with no key).  A resolver created, run once and destroyed
 *     (the arrays are in host memory here). --- */
typedef struct {
  uint32_t n_keys, solved_in_inputs, solved_by_merge, left;
  uint64_t same_herd, no_key, already_solved, solving;   /* collisions by outcome; they sum to info->collisions */
} kgx_batch_merge_info;
typedef struct {
  uint32_t status, h;
  uint64_t priv[4];
  uint64_t d_first[2], d_other[2];
} kgx_batch_key_result;
int kgx_work_merge_batch(int dev, const char* const* paths, uint32_t n_paths, const char* tmp_path, uint64_t block_entries,
                         kgx_work_merge_info* info, kgx_batch_merge_info* binfo, kgx_batch_key_result* keys, uint32_t cap_keys);
int kgx_work_resolve(int dev, const uint64_t* d_first, const uint64_t* d_other, uint64_t n, const uint64_t* keys, uint32_t n_keys,
                     const uint64_t range_start[4], uint32_t* key_out, uint64_t* priv_out);

/* Debug (KGX_PROF=1 in the environment at kgx_create): phase cycle counters summed over warp 0 of every CTA:
 * out = {serial section, modular inverse alone, parallel phase, tile-steps}; resets them. -1 when disabled. */
int      kgx_debug_prof(kgx_engine* e, uint64_t out[4]);

/* --- device-side unit-test / microbenchmark hooks (kgx_field.cuh, kgx_modinv.h, kgx_herd.cuh, kgx_kernel.cuh) --- */
/* One device primitive per element.  a, b, out: n x 4 limbs on the HOST; "word k" is 32-bit word k of an element (word 0 =
 * low half of limb 0).  Results narrower than 256 bits fill the low words of out, the rest is 0.  Unknown op: error.
 *   MUL, SQR, SUB, INV     out = fe_mul(a,b) / fe_sqr(a) / fe_sub(a,b) / modinv256(a)
 *   *_INPLACE              the same through the aliased forms fe_mul(a,a,b) / fe_sqr(a,a) / fe_sub(a,a,b); out = a afterwards
 *   GT_HALF                word 0 = fe_gt_half_mask(a): 0xFFFFFFFF when a > (p-1)/2, else 0
 *   CNEG                   fe_cneg(a, mask = b word 0); out = a afterwards
 *   D128_ADD, D128_CNEG    128-bit distance in a words 0..3: d128_add(a, b words 0..3) / d128_cneg(a, mask = b word 0)
 *   IS_ZERO                word 0 = fe_is_zero_modp(a) (1 / 0)
 *   NEG, DBL               out = fe_neg(a) / fe_dbl(a)
 *   JUMP_INDEX             x0 = a word 0, aux = b word 0, rule = b word 1: word 0 = jump_index<symmetric>, word 1 = jump_index<plain>
 *   SYM_NEXT_AUX           j = a word 0, neg mask = a word 1, aux = b word 0, rule = b word 1: word 0 = sym_next_aux */
#define KGX_TF_MUL           0
#define KGX_TF_SQR           1
#define KGX_TF_SUB           2
#define KGX_TF_INV           3
#define KGX_TF_MUL_INPLACE   4
#define KGX_TF_SQR_INPLACE   5
#define KGX_TF_SUB_INPLACE   6
#define KGX_TF_GT_HALF       7
#define KGX_TF_CNEG          8
#define KGX_TF_D128_ADD      9
#define KGX_TF_D128_CNEG     10
#define KGX_TF_IS_ZERO       11
#define KGX_TF_NEG           12
#define KGX_TF_DBL           13
#define KGX_TF_JUMP_INDEX    14
#define KGX_TF_SYM_NEXT_AUX  15
int kgx_test_field(int dev, int op, int n, const uint64_t* a, const uint64_t* b, uint64_t* out);
/* The device HashTable::Convert (kgx_convert_dps) on crafted input: a DP slab [u32 count][max_found x 56-byte records] is
 * built from `count` and recs56 (min(count, max_found) records, kgx_item layout), converted with wild_offset (2 limbs) or,
 * with signed_mode != 0, as signed distances, and the whole [u32 count][max_found x 40-byte records] buffer is copied to
 * `out` (4 + max_found * 40 bytes; slots past the count keep the device fill 0xFF). */
int kgx_test_dp_convert(int dev, uint32_t count, uint32_t max_found, const void* recs56, const uint64_t wild_offset[2],
                        int signed_mode, void* out);
/* Raw device throughput probes: kind 0 = IMAD.WIDE.U32 issue rate (the multiplier roofline bench.py reports against),
 * 1 = ModMult chains, 2 = ModSqr chains, 3 = modular inverses.  *ms = device time, *ops = operations executed. */
int kgx_bench_raw(int dev, int kind, int iters, float* ms, double* ops);

#ifdef __cplusplus
}
#endif
#endif
