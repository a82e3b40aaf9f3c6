// kgx_resolver.cuh -- the collision resolver kept on one GPU (C ABI: include/kgx.h, kgx_resolver_*).
//
// kgx_resolver_create builds once what every resolve needs: the fixed-base comb (kgx_worktool.cuh, 30 KB), the keys
// K = key - start*G and their index sorted by x (wt_find_key's), and the range start.  A run is then one kernel,
// wt_resolve_pair per collision: kgi_resolve_multi's result, the first key in input order that +-Td +-Wd * G hits, and its
// private key.  Runs are stream-ordered on the caller's stream and allocate nothing, so the solver resolves every step's
// collisions on the device table's stream (kgx_dptable_add_resolve, kgx_dptable.cuh) and the host does no per-collision work.
// kgx_work_resolve is a resolver of one call.
//
// A resolver of one key also checks received DP records (kgx_resolver_verify, the server's check of what clients send): the
// stored-entry check of kgx_worktool.cuh (wt_check_entries_kernel, on Dp40Check records) flags each record, then
// kgx_dp_partition's passes (kgx_partition.cuh) run with the wrong records as the group left out: the good records grouped by
// the shard that owns their bucket (kgx_resolver_verify_partition; one group, in input order, for kgx_resolver_verify) and
// the bad indices, from one scan of (owner, tile) counts.

struct kgx_resolver {
  int dev = 0;
  uint32_t n_keys = 0;
  int kinf = 0;                                         // key 0's K is the point at infinity (the check needs it)
  kgx_wt::Start start;
  kgx_wt::u32 *comb = nullptr, *kx = nullptr, *K = nullptr;
  uint32_t* ki = nullptr;
  std::vector<void*> mem;                               // every device buffer above
  char err[256] = "";
};

namespace kgx_wt {

// pairs: n collisions, pair i = 4 words {d_first[2], d_other[2]} at pairs + 4i
__global__ void __launch_bounds__(CHECK_THREADS) wt_resolve_pairs_kernel(const u32* __restrict__ comb, const u64* __restrict__ pairs,
                                                                        uint32_t n, const u32* __restrict__ kx, const uint32_t* __restrict__ ki,
                                                                        const u32* __restrict__ K, uint32_t n_keys, Start start,
                                                                        uint32_t* key_out, u64* priv_out) {
  __shared__ u32 sc[COMB_WORDS];
  wt_load_comb(sc, comb);
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u64 a[2] = {pairs[4ull * i], pairs[4ull * i + 1]}, b[2] = {pairs[4ull * i + 2], pairs[4ull * i + 3]};
  u64 priv[4];
  key_out[i] = wt_resolve_pair(sc, a, b, kx, ki, K, n_keys, start, priv);
  for (int w = 0; w < 4; w++) priv_out[4ull * i + w] = priv[w];
}

// The device table's events of one add: the first min(*nsel, cap) of ev, each copied to out with its key -- a collision
// event's (d_old, d_new) resolved, NO_KEY for every other event.  The count is on the device, so the grid covers cap and the
// blocks past it return before they load the comb.
__global__ void __launch_bounds__(CHECK_THREADS) wt_resolve_events_kernel(const u32* __restrict__ comb, const kgx_dp_event* __restrict__ ev,
                                                                         const uint32_t* __restrict__ nsel, uint32_t cap,
                                                                         const u32* __restrict__ kx, const uint32_t* __restrict__ ki,
                                                                         const u32* __restrict__ K, uint32_t n_keys, Start start,
                                                                         kgx_dp_event_key* out) {
  const uint32_t n = *nsel < cap ? *nsel : cap;
  if (blockIdx.x * blockDim.x >= n) return;             // the whole block: before the comb's __syncthreads
  __shared__ u32 sc[COMB_WORDS];
  wt_load_comb(sc, comb);
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const kgx_dp_event e = ev[i];
  u64 priv[4] = {0, 0, 0, 0};
  uint32_t key = NO_KEY;
  if (e.kind == KGX_DPT_EV_COLLISION) key = wt_resolve_pair(sc, e.d_old, e.d_new, kx, ki, K, n_keys, start, priv);
  kgx_dp_event_key& o = out[i];
  o.ev = e;
  o.key = key;
  o.reserved = 0;
  for (int w = 0; w < 4; w++) o.priv[w] = priv[w];
}

// kgx_dptable_add_resolve's step, queued on st behind the events' compaction
static cudaError_t resolve_events(const kgx_resolver* r, const kgx_dp_event* ev, const uint32_t* nsel, uint32_t cap, kgx_dp_event_key* out,
                                  cudaStream_t st) {
  if (cap == 0) return cudaSuccess;
  wt_resolve_events_kernel<<<(cap + CHECK_THREADS - 1) / CHECK_THREADS, CHECK_THREADS, 0, st>>>(r->comb, ev, nsel, cap, r->kx, r->ki, r->K,
                                                                                               r->n_keys, r->start, out);
  return cudaGetLastError();
}

// kgx_resolver_verify_partition's destination of record i: the owner of its bucket when the check found it good (then
// h < 2^18, since h equals 18 bits of S.x), else the group left out
struct Verified {
  const uint8_t* recs;
  const uint32_t* good;
  __device__ __forceinline__ uint32_t operator()(uint32_t i, uint32_t world) const {
    return good[i] ? kgx_part::owner_of(reinterpret_cast<const uint32_t*>(recs + 40ull * i)[1], world) : world;
  }
};

// kgx_resolver_verify_partition, and kgx_resolver_verify as its world 1, stride 0; fn names the call in its error messages.
// scratch: the check's flags, then kgx_dp_partition_scratch_bytes(n, world) for the partition's passes.
static int verify_partition(const char* fn, kgx_resolver* r, const void* recs, uint32_t n, uint32_t world, uint64_t stride, void* out,
                            uint32_t* counts, uint32_t* bad_idx, uint32_t cap, void* scratch, uint64_t scratch_bytes, void* stream) {
  const char* why = nullptr;
  if (r->n_keys != 1) why = "the resolver must hold exactly one key";
  else if (n >= 0x80000000u) why = "at most 2^31-1 records";
  else if (world == 0 || world > KGX_DPT_MAX_RANKS) why = "world must be 1 .. KGX_DPT_MAX_RANKS";
  else if (stride != 0 && stride < n) why = "stride must be 0 or at least n";
  else if (((uintptr_t)recs | (uintptr_t)out) & 7) why = "the records and the output must be 8-byte aligned";
  else if ((uintptr_t)scratch & 255) why = "scratch must be 256-byte aligned";
  else if (scratch_bytes < kgx_resolver_verify_partition_scratch_bytes(n, world)) why = "scratch smaller than the call's _scratch_bytes";
  if (why) {
    snprintf(r->err, sizeof r->err, "%s: %s", fn, why);
    return -1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t s = cudaSetDevice(r->dev);
  uint8_t* sb = static_cast<uint8_t*>(scratch);
  uint32_t* flags = reinterpret_cast<uint32_t*>(sb);
  const uint8_t* in = static_cast<const uint8_t*>(recs);
  const uint64_t fb = kgx_part::align256(4ull * n);
  if (s == cudaSuccess && n > 0) {
    wt_check_entries_kernel<<<check_blocks(n), CHECK_THREADS, 0, st>>>(r->comb, Dp40Check{static_cast<const u64*>(recs), flags}, n, r->K,
                                                                      r->kinf);
    s = cudaGetLastError();
  }
  const int rc = s == cudaSuccess ? kgx_part::run(in, Verified{in, flags}, n, world, stride, out, counts, bad_idx, cap, sb + fb,
                                                  scratch_bytes - fb, st)
                                   : 0;
  if (s != cudaSuccess || rc) {
    snprintf(r->err, sizeof r->err, "%s: %s", fn, s != cudaSuccess ? cudaGetErrorString(s) : "a launch of the partition passes failed");
    cudaGetLastError();
    return -3;
  }
  return 0;
}

// the checks kgx_resolver_create and kgx_work_resolve share: -1 with the reason in g_wt_err, or 0
static int resolver_args(const char* fn, uint32_t n_keys, const uint64_t range_start[4]) {
  if (n_keys == 0 || n_keys > kgx_wf::BATCH_MAX_KEYS) { snprintf(g_wt_err, sizeof g_wt_err, "%s: n_keys must be in [1, %u]", fn, kgx_wf::BATCH_MAX_KEYS); return -1; }
  if (kgx::ge256(range_start, kgx::kOrderHost)) { snprintf(g_wt_err, sizeof g_wt_err, "%s: the range start is not below n", fn); return -1; }
  return 0;
}

}  // namespace kgx_wt

extern "C" {

kgx_resolver* kgx_resolver_create(int dev, const uint64_t* keys, uint32_t n_keys, const uint64_t range_start[4]) {
  using namespace kgx_wt;
  if (resolver_args("kgx_resolver_create", n_keys, range_start) || set_device(dev)) return nullptr;
  DevBufs B;
  u32 *comb, *kx, *K;
  uint32_t* ki;
  std::vector<uint32_t> order, hk(16ull * n_keys);
  memcpy(hk.data(), keys, 64ull * n_keys);
  if (build_comb(B, &comb, 0) || key_index(B, hk, n_keys, &kx, &ki, order) || B.dev(&K, 64ull * n_keys)) return nullptr;
  cudaError_t s = cudaMemcpy(K, keys, 64ull * n_keys, cudaMemcpyHostToDevice);
  if (s == cudaSuccess) s = cudaStreamSynchronize(0);   // the comb is built before a run on any other stream reads it
  if (s != cudaSuccess) {
    snprintf(g_wt_err, sizeof g_wt_err, "kgx_resolver_create: %s", cudaGetErrorString(s));
    cudaGetLastError();
    return nullptr;
  }
  kgx_resolver* r = new kgx_resolver();
  r->dev = dev;
  r->n_keys = n_keys;
  r->kinf = !(keys[0] | keys[1] | keys[2] | keys[3] | keys[4] | keys[5] | keys[6] | keys[7]);
  memcpy(r->start.v, range_start, 32);
  r->comb = comb; r->kx = kx; r->K = K; r->ki = ki;
  r->mem.swap(B.d);                                     // the resolver keeps them
  return r;
}

void kgx_resolver_destroy(kgx_resolver* r) {
  if (!r) return;
  cudaSetDevice(r->dev);
  for (void* p : r->mem) cudaFree(p);                   // cudaFree waits for the runs still queued
  delete r;
}

const char* kgx_resolver_last_error(kgx_resolver* r) { return r ? r->err : g_wt_err; }

int kgx_resolver_run(kgx_resolver* r, const void* pairs, uint32_t n, uint32_t* key_out, uint64_t* priv_out, void* stream) {
  using namespace kgx_wt;
  if (n >= 0x80000000u) { snprintf(r->err, sizeof r->err, "kgx_resolver_run: %u collisions (at most 2^31-1)", n); return -1; }
  if (n == 0) return 0;
  cudaError_t s = cudaSetDevice(r->dev);
  if (s == cudaSuccess) {
    wt_resolve_pairs_kernel<<<(n + CHECK_THREADS - 1) / CHECK_THREADS, CHECK_THREADS, 0, (cudaStream_t)stream>>>(
        r->comb, static_cast<const u64*>(pairs), n, r->kx, r->ki, r->K, r->n_keys, r->start, key_out, priv_out);
    s = cudaGetLastError();
  }
  if (s != cudaSuccess) {
    snprintf(r->err, sizeof r->err, "kgx_resolver_run: %s", cudaGetErrorString(s));
    return -3;
  }
  return 0;
}

uint64_t kgx_resolver_verify_scratch_bytes(uint32_t n) { return kgx_resolver_verify_partition_scratch_bytes(n, 1); }

int kgx_resolver_verify(kgx_resolver* r, const void* recs, uint32_t n, void* good, uint32_t* counts, uint32_t* bad_idx, uint32_t cap,
                        void* scratch, uint64_t scratch_bytes, void* stream) {
  return kgx_wt::verify_partition("kgx_resolver_verify", r, recs, n, 1, 0, good, counts, bad_idx, cap, scratch, scratch_bytes, stream);
}

uint64_t kgx_resolver_verify_partition_scratch_bytes(uint32_t n, uint32_t world) {
  const uint64_t part = kgx_dp_partition_scratch_bytes(n, world);
  return n >= 0x80000000u || part == 0 ? 0 : kgx_part::align256(4ull * n) + part;
}

int kgx_resolver_verify_partition(kgx_resolver* r, const void* recs, uint32_t n, uint32_t world, uint64_t stride, void* out,
                                  uint32_t* counts, uint32_t* bad_idx, uint32_t cap, void* scratch, uint64_t scratch_bytes, void* stream) {
  return kgx_wt::verify_partition("kgx_resolver_verify_partition", r, recs, n, world, stride, out, counts, bad_idx, cap, scratch,
                                  scratch_bytes, stream);
}

int kgx_work_resolve(int dev, const uint64_t* d_first, const uint64_t* d_other, uint64_t n, const uint64_t* keys, uint32_t n_keys,
                     const uint64_t range_start[4], uint32_t* key_out, uint64_t* priv_out) {
  using namespace kgx_wt;
  if (resolver_args("kgx_work_resolve", n_keys, range_start)) return -1;
  if (n >= 0x80000000ull) { snprintf(g_wt_err, sizeof g_wt_err, "kgx_work_resolve: %llu collisions (at most 2^31-1)", (unsigned long long)n); return -1; }
  kgx_resolver* r = kgx_resolver_create(dev, keys, n_keys, range_start);
  if (!r) return -3;
  struct Free { kgx_resolver* r; ~Free() { kgx_resolver_destroy(r); } } fr{r};
  if (n == 0) return 0;
  DevBufs B;
  u64 *dPairs, *dPriv;
  uint32_t* dKey;
  if (B.dev(&dPairs, 32 * n) || B.dev(&dKey, 4 * n) || B.dev(&dPriv, 32 * n)) return -3;
  std::vector<uint64_t> hp(4 * n);
  for (uint64_t i = 0; i < n; i++) {
    hp[4 * i] = d_first[2 * i]; hp[4 * i + 1] = d_first[2 * i + 1];
    hp[4 * i + 2] = d_other[2 * i]; hp[4 * i + 3] = d_other[2 * i + 1];
  }
  WT_CK(cudaMemcpy(dPairs, hp.data(), 32 * n, cudaMemcpyHostToDevice));
  if (kgx_resolver_run(r, dPairs, (uint32_t)n, dKey, dPriv, nullptr)) { snprintf(g_wt_err, sizeof g_wt_err, "%s", r->err); return -3; }
  WT_CK(cudaMemcpy(key_out, dKey, 4 * n, cudaMemcpyDeviceToHost));
  WT_CK(cudaMemcpy(priv_out, dPriv, 32 * n, cudaMemcpyDeviceToHost));
  return 0;
}

}  // extern "C"
