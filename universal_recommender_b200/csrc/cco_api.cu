// cco_api.cu -- C ABI (include/cco_b200.h) and host orchestration of the sm_90a CCO model builder.
//
// Replaces Mahout's SimilarityAnalysis.cooccurrencesIDSs / crossOccurrenceDownsampled as called from
// src/main/scala/URAlgorithm.scala:323-329,343-346.  No CPU fallback: every compute
// entry fails with CCO_E_CUDA when no CUDA device is usable.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <charconv>
#include <cmath>
#include <functional>
#include <memory>
#include <cub/cub.cuh>
#include <nvtx3/nvToolsExt.h>
#include <condition_variable>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/cco_b200.h"
#include "cco_kernels.cuh"
#include "cco_sampler.cuh"
#include "cco_format.cuh"
#include "cco_strings.cuh"
#include "cco_json.cuh"
#include "cco_events.cuh"
#include "cco_queries.cuh"
#include "cco_results.cuh"
#include "cco_index_pages.cuh"
#include "cco_index_write.cuh"
#include "cco_refresh.cuh"
#include "cco_intern.cuh"
#include "cco_snapshot.cuh"
#include "cco_clean.cuh"
#include "cco_erase.cuh"

namespace cco {

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
static int set_error(int code, const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof g_err, fmt, ap);
  va_end(ap);
  return code;
}
#define CK(expr)                                                                                      \
  do {                                                                                                \
    cudaError_t _e = (expr);                                                                          \
    if (_e != cudaSuccess)                                                                            \
      return set_error(_e == cudaErrorMemoryAllocation ? CCO_E_OOM : CCO_E_CUDA, "%s: %s (%s:%d)", #expr, \
                       cudaGetErrorString(_e), __FILE__, __LINE__);                                   \
  } while (0)
#define CKR(expr)            \
  do {                       \
    int _r = (expr);         \
    if (_r != CCO_OK) return _r; \
  } while (0)

// ------------------------------------------------------------------------------------------------
// NCCL, loaded lazily (only multi-GPU contexts need it)
// ------------------------------------------------------------------------------------------------
typedef struct ncclComm *ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
struct Nccl {
  void *h = nullptr;
  int (*GetUniqueId)(ncclUniqueId *) = nullptr;
  int (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
  int (*CommInitAll)(ncclComm_t *, int, const int *) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  int (*AllReduce)(const void *, void *, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*AllGather)(const void *, void *, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*Broadcast)(const void *, void *, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  const char *(*GetErrorString)(int) = nullptr;
};
static Nccl g_nccl;
static std::mutex g_nccl_mu;
static int load_nccl() {
  std::lock_guard<std::mutex> lk(g_nccl_mu);
  if (g_nccl.h) return CCO_OK;
  void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) return set_error(CCO_E_NCCL, "cannot load libnccl.so.2: %s", dlerror());
#define SYM(field, name)                                                         \
  *(void **)(&g_nccl.field) = dlsym(h, name);                                    \
  if (!g_nccl.field) return set_error(CCO_E_NCCL, "libnccl: missing symbol %s", name);
  SYM(GetUniqueId, "ncclGetUniqueId")
  SYM(CommInitRank, "ncclCommInitRank")
  SYM(CommInitAll, "ncclCommInitAll")
  SYM(CommDestroy, "ncclCommDestroy")
  SYM(AllReduce, "ncclAllReduce")
  SYM(AllGather, "ncclAllGather")
  SYM(Broadcast, "ncclBroadcast")
  SYM(GroupStart, "ncclGroupStart")
  SYM(GroupEnd, "ncclGroupEnd")
  SYM(GetErrorString, "ncclGetErrorString")
#undef SYM
  g_nccl.h = h;
  return CCO_OK;
}
constexpr int kNcclInt32 = 2, kNcclUint32 = 3, kNcclSum = 0, kNcclMax = 2;  // ncclInt32, ncclUint32, ncclSum, ncclMax (nccl.h enum values)

}  // namespace cco

using namespace cco;

// ------------------------------------------------------------------------------------------------
// context / result objects
// ------------------------------------------------------------------------------------------------
struct PinnedBuf {
  void *p;
  size_t cap;
  bool used;
};

// shared by the per-GPU member contexts of a group (single-process multi-GPU) context
struct GroupShared {
  int world = 0;
  std::mutex mu;
  std::condition_variable cv;
  int arrived = 0;
  unsigned long long generation = 0;
  std::vector<long long> totals;   // per rank: kept cells of the indicator being merged
  struct cco_result *merged = nullptr;
  int status = 0;                  // first failure of any member thread
  char err[512] = "";
  void barrier() {
    std::unique_lock<std::mutex> lk(mu);
    const unsigned long long g = generation;
    if (++arrived == world) {
      arrived = 0;
      ++generation;
      cv.notify_all();
    } else {
      cv.wait(lk, [&] { return generation != g; });
    }
  }
};

struct cco_ctx {
  int device = 0, rank = 0, world = 1;
  int sm_count = 0;
  size_t smem_optin = 0;
  cudaStream_t stream = nullptr, copy_stream = nullptr;
  cudaEvent_t ev[8] = {};
  cudaEvent_t tev[2] = {};
  cudaEvent_t copy_ev[2] = {};
  cudaStream_t bin_stream[8] = {};
  cudaStream_t sched_stream = nullptr;   // row scheduling of indicator i+1 runs here, beside the row kernels of indicator i
  cudaEvent_t bin_ev[9] = {};
  std::vector<PinnedBuf> pinned;
  std::mutex mu;
  ncclComm_t comm = nullptr;
  int launches = 0;
  int32_t key_range_cap = 0;   // cco_debug_key_range_cap: at most this many keys per key range (0 = off)
  uint64_t intern_mask = ~0ULL;   // cco_debug_intern_hash_bits: the intern hash of the logs begun from now on, truncated
  // mailbox for small device -> host results (mapped pinned memory written by k_mail_bytes).  Records are closed into
  // groups; a group is complete when its event has fired, so the host can wait for indicator i's numbers while the GPU
  // already runs indicator i + 1 (no stream-wide synchronisation).
  unsigned char *mail_h = nullptr, *mail_d = nullptr;
  size_t mail_used = 0;
  struct MailItem { void *dst; size_t off, n; int group; };
  std::vector<MailItem> mail_pending;
  std::vector<cudaEvent_t> mail_ev;
  int mail_group = 0;
  // optional caller-provided result arena (cco_config_t.result_arena): results are bump-allocated from it, e.g. a
  // shared-memory segment another process maps, so that no copy separates this rank's slice from the reader
  unsigned char *arena = nullptr;
  size_t arena_bytes = 0, arena_used = 0;
  int arena_live = 0;
  bool arena_registered = false;
  // small per-train device scratch comes from slabs the context keeps (bump allocation: no CUDA call per buffer), and the
  // per-train events come from a cached pool: a train of a small shape is bound by host API calls, not by its kernels
  struct Slab { unsigned char *p; size_t cap; };
  std::vector<Slab> slabs;
  size_t slab_idx = 0, slab_off = 0;
  bool slab_busy = false;
  std::vector<cudaEvent_t> ev_timing, ev_plain;
  size_t ev_timing_used = 0, ev_plain_used = 0;
  // group context: the leader owns one member context per GPU (members[0]->device = devices[0], ...)
  std::vector<cco_ctx *> members;
  GroupShared *gshared = nullptr;   // set on members

  void *pinned_get(size_t bytes, bool for_result = true) {
    std::lock_guard<std::mutex> lk(mu);
    if (bytes == 0) bytes = 16;
    if (arena && for_result) {
      const size_t off = (arena_used + 255) & ~(size_t)255;
      if (off + bytes <= arena_bytes) {
        arena_used = off + bytes;
        ++arena_live;
        return arena + off;
      }
    }
    int best = -1;
    for (size_t i = 0; i < pinned.size(); ++i)
      if (!pinned[i].used && pinned[i].cap >= bytes && (best < 0 || pinned[i].cap < pinned[best].cap)) best = (int)i;
    if (best >= 0) {
      pinned[best].used = true;
      return pinned[best].p;
    }
    void *p = nullptr;
    size_t cap = (bytes + (1u << 20) - 1) & ~((size_t)(1u << 20) - 1);
    if (cudaHostAlloc(&p, cap, cudaHostAllocPortable) != cudaSuccess) return nullptr;
    pinned.push_back({p, cap, true});
    return p;
  }
  void pinned_put(void *p) {
    std::lock_guard<std::mutex> lk(mu);
    if (arena && (unsigned char *)p >= arena && (unsigned char *)p < arena + arena_bytes) {
      if (--arena_live <= 0) { arena_live = 0; arena_used = 0; }   // every result freed: the arena starts over
      return;
    }
    for (auto &b : pinned)
      if (b.p == p) b.used = false;
  }
};

struct ResultMat {
  int64_t row_begin = 0, row_end = 0;
  int32_t n_cols = 0;
  int64_t *row_ptr = nullptr;
  int32_t *col = nullptr;
  double *llr = nullptr;
  int32_t *cnt = nullptr;
  int32_t key_ranges = 1;   // key ranges the indicator ran in
};
// A dataset holds, per event type, the block of user rows this context works on: the whole matrix on a single GPU,
// this rank's user block [row_base, row_base + n_local) in a multi-GPU job (each GPU uploads 1/N of the rows).
struct cco_dataset {
  cco_ctx *ctx = nullptr;
  int n_mats = 0;
  long long n_users = 0;           // U, global
  long long row_base = 0, n_local = 0;
  std::vector<long long> n_cols, nnz;   // nnz: stored entries of the WHOLE matrix as handed in
  std::vector<long long *> rp;   // device, indexable by local row 0 .. n_local (values index `col`)
  std::vector<int32_t *> col;    // device, indexable by the values of rp
  std::vector<void *> rp_alloc, col_alloc;   // what to free (rp/col may be offset views of these)
  std::vector<long long> q_lo, q_hi;         // per matrix: the offsets rp[0], rp[n_local] of the block (host-known)
  std::vector<cudaEvent_t> ready;  // per matrix: host->device copy finished (copy stream)
  bool h2d_pending = false;        // uploaded asynchronously: ms_h2d is read when the train joins
  bool validated = false;          // k_check_rows has run (and the rows are canonical)
  bool whole = false;              // rp_alloc / col_alloc hold the WHOLE matrices (device-built datasets, single-GPU uploads)
  float ms_h2d = 0;
  // cco_ingest_strings: [0] the user dictionary, [1 + t] the item dictionary of type t, in pinned memory of the context
  std::vector<cco_dictionary_t> dicts;
};

struct cco_result {
  cco_ctx *ctx = nullptr;
  std::vector<ResultMat> mats;
  cco_stats_t stats;
};

namespace cco {

// per-call device arena on top of the stream-ordered allocator
struct Arena {
  cudaStream_t s;
  cco_ctx *c;   // non-null: buffers up to kSlabMax bytes are bump-allocated from the context's slabs
  std::vector<void *> ptrs;
  std::vector<size_t> sizes;   // bytes of each of ptrs
  static constexpr size_t kSlabMax = 8u << 20, kSlabBytes = 64u << 20;
  explicit Arena(cudaStream_t st, cco_ctx *ctx = nullptr) : s(st), c(ctx && !ctx->slab_busy ? ctx : nullptr) {
    if (c) {
      c->slab_busy = true;
      c->slab_idx = 0;
      c->slab_off = 0;
    }
  }
  ~Arena() {
    for (void *p : ptrs) cudaFreeAsync(p, s);
    if (c) c->slab_busy = false;
  }
  void *bump(size_t bytes) {
    bytes = (bytes + 255) & ~(size_t)255;
    while (true) {
      if (c->slab_idx < c->slabs.size()) {
        cco_ctx::Slab &sl = c->slabs[c->slab_idx];
        if (c->slab_off + bytes <= sl.cap) {
          void *p = sl.p + c->slab_off;
          c->slab_off += bytes;
          return p;
        }
        ++c->slab_idx;
        c->slab_off = 0;
        continue;
      }
      void *p = nullptr;
      if (cudaMalloc(&p, kSlabBytes) != cudaSuccess) return nullptr;   // warm-up trains only; kept until cco_destroy
      c->slabs.push_back({(unsigned char *)p, kSlabBytes});
    }
  }
  template <typename T>
  int alloc(T **out, size_t n) {
    void *p = nullptr;
    size_t bytes = std::max<size_t>(n * sizeof(T), 16);
    if (c && bytes <= kSlabMax) {
      p = bump(bytes);
      if (!p) return set_error(CCO_E_OOM, "cudaMalloc(scratch slab) failed");
      *out = (T *)p;
      return CCO_OK;
    }
    cudaError_t e = cudaMallocAsync(&p, bytes, s);
    if (e != cudaSuccess) return set_error(CCO_E_OOM, "cudaMallocAsync(%zu bytes): %s", bytes, cudaGetErrorString(e));
    ptrs.push_back(p);
    sizes.push_back(bytes);
    *out = (T *)p;
    return CCO_OK;
  }
  // the buffer outlives the arena: its new owner frees it (never slab memory); -> its bytes
  size_t take(void *p) {
    for (size_t i = 0; i < ptrs.size(); ++i)
      if (ptrs[i] == p) {
        const size_t b = sizes[i];
        ptrs.erase(ptrs.begin() + i);
        sizes.erase(sizes.begin() + i);
        return b;
      }
    return 0;
  }
  void release(void *p) {   // slab memory is simply not reused within a train
    for (size_t i = 0; i < ptrs.size(); ++i)
      if (ptrs[i] == p) {
        cudaFreeAsync(p, s);
        ptrs.erase(ptrs.begin() + i);
        sizes.erase(sizes.begin() + i);
        return;
      }
  }
};
// cached events of a train (reset at its start)
static int pooled_event(cco_ctx *c, bool timing, cudaEvent_t *out) {
  std::vector<cudaEvent_t> &pool = timing ? c->ev_timing : c->ev_plain;
  size_t &used = timing ? c->ev_timing_used : c->ev_plain_used;
  if (used == pool.size()) {
    cudaEvent_t e;
    CK(timing ? cudaEventCreate(&e) : cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    pool.push_back(e);
  }
  *out = pool[used++];
  return CCO_OK;
}

// NVTX ranges per stage (SURVEY.md section 5: tracing); header-only NVTX3, a no-op unless a profiler is attached
static inline void nvtx_push(const char *name) { nvtxRangePushA(name); }
static inline void nvtx_pop() { nvtxRangePop(); }
struct NvtxRange {   // a range over one scope
  explicit NvtxRange(const char *name) { nvtx_push(name); }
  ~NvtxRange() { nvtx_pop(); }
};

static inline int grid_for(long long work_items, int block, int sm_count, int waves = 8) {
  long long g = (work_items + block - 1) / block;
  long long cap = (long long)sm_count * waves;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

constexpr size_t kMailBytes = 1 << 16;
// enqueue "copy n bytes from device to *dst_host"; the value is there after the group it belongs to has been waited for
static int mail_fetch(cco_ctx *c, void *dst_host, const void *src_dev, size_t n) {
  size_t off = (c->mail_used + 7) & ~(size_t)7;
  if (off + n > kMailBytes) return set_error(CCO_E_CUDA, "internal: mailbox overflow");
  k_mail_bytes<<<1, 128, 0, c->stream>>>(c->mail_d + off, (const unsigned char *)src_dev, (int)n);
  c->mail_pending.push_back({dst_host, off, n, c->mail_group});
  c->mail_used = off + n;
  return CCO_OK;
}
// close the current group: everything fetched so far is complete once the returned group's event has fired
static int mail_close(cco_ctx *c, int *group) {
  const int g = c->mail_group;
  while ((int)c->mail_ev.size() <= g) {
    cudaEvent_t e;
    CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    c->mail_ev.push_back(e);
  }
  CK(cudaEventRecord(c->mail_ev[g], c->stream));
  c->mail_group = g + 1;
  if (group) *group = g;
  return CCO_OK;
}
static int mail_wait_group(cco_ctx *c, int g) {
  CK(cudaEventSynchronize(c->mail_ev[g]));
  CK(cudaGetLastError());
  for (auto &m : c->mail_pending)
    if (m.group == g) memcpy(m.dst, c->mail_h + m.off, m.n);
  return CCO_OK;
}
static void mail_reset(cco_ctx *c) {
  c->mail_pending.clear();
  c->mail_used = 0;
  c->mail_group = 0;
}
// close + wait: the host needs the values now
static int mail_wait(cco_ctx *c) {
  int g = 0;
  CKR(mail_close(c, &g));
  return mail_wait_group(c, g);
}

struct DevRaw {  // a block of user rows of a matrix as uploaded (int64 row_ptr like the host)
  long long n_rows = 0;     // rows of the block (n_local)
  long long row_base = 0;   // global index of its first row
  int32_t n_cols = 0;
  long long nnz = 0;        // entries of the block
  long long q_base = 0;     // value of rp[0] (host-known): a rank's block keeps the caller's absolute offsets
  long long *rp = nullptr;  // indexable by local row
  int32_t *col = nullptr;   // indexable by rp values
};
struct DevMat {  // after canonicalise + downsample
  long long n_rows = 0;
  int32_t n_cols = 0;
  uint32_t *rp = nullptr;  // [n_rows+1]
  int32_t *col = nullptr;
  int32_t *marg = nullptr;  // post-sample column counts
};

template <typename T>
static int exclusive_sum(cco_ctx *c, Arena &ar, const T *in, T *out, long long n, cudaStream_t on = nullptr) {
  if (!on) on = c->stream;
  size_t tb = 0;
  CK(cub::DeviceScan::ExclusiveSum(nullptr, tb, in, out, n, on));
  void *tmp;
  CKR(ar.alloc((char **)&tmp, tb));   // a few KB: always slab memory when the arena has slabs
  CK(cub::DeviceScan::ExclusiveSum(tmp, tb, in, out, n, on));
  ar.release(tmp);
  return CCO_OK;
}
// sort (key, value) pairs of n entries by the low `bits` bits of the key, stably; the sorted arrays replace *k / *v
template <typename K, typename V>
static int sort_pairs(cco_ctx *c, Arena &ar, long long n, K **k, V **v, int bits) {
  cudaStream_t s = c->stream;
  K *k1;
  V *v1;
  CKR(ar.alloc(&k1, std::max<long long>(n, 1)));
  CKR(ar.alloc(&v1, std::max<long long>(n, 1)));
  cub::DoubleBuffer<K> kb(*k, k1);
  cub::DoubleBuffer<V> vb(*v, v1);
  size_t tbytes = 0;
  CK(cub::DeviceRadixSort::SortPairs(nullptr, tbytes, kb, vb, n, 0, bits, s));
  void *tmp;
  CKR(ar.alloc((char **)&tmp, tbytes));
  CK(cub::DeviceRadixSort::SortPairs(tmp, tbytes, kb, vb, n, 0, bits, s));
  c->launches++;
  ar.release(tmp);
  ar.release(kb.Alternate());
  ar.release(vb.Alternate());
  *k = kb.Current();
  *v = vb.Current();
  return CCO_OK;
}
static int bits_for(long long n) {
  int b = 1;
  while ((1LL << b) < n) ++b;
  return b;
}

// canonical CSR of n_rows rows from (row << 32 | col) keys: the n keys in k0 are radix-sorted on their low `bits` bits
// (k1: scratch of n keys), the first n_valid sorted keys lose their duplicates into `col` and give `rp` (keys past
// n_valid must sort after them).  The unique count comes back through the mailbox while the scatter runs.
static int keys_to_csr(cco_ctx *c, Arena &ar, unsigned long long *k0, unsigned long long *k1, long long n, int bits, long long n_valid,
                       long long n_rows, int32_t *col, long long *rp, long long *n_unique) {
  cudaStream_t s = c->stream;
  cub::DoubleBuffer<unsigned long long> db(k0, k1);
  size_t tb = 0;
  CK(cub::DeviceRadixSort::SortKeys(nullptr, tb, db, n, 0, bits, s));
  void *tmp;
  CKR(ar.alloc((char **)&tmp, tb));
  CK(cub::DeviceRadixSort::SortKeys(tmp, tb, db, n, 0, bits, s));
  ar.release(tmp);
  unsigned long long *sorted = db.Current(), *other = db.Alternate();
  uint32_t *flag, *pos;
  CKR(ar.alloc(&flag, n_valid + 1));
  CKR(ar.alloc(&pos, n_valid + 1));
  CK(cudaMemsetAsync(flag + n_valid, 0, 4, s));
  k_unique_flags<<<grid_for(n_valid, 256, c->sm_count), 256, 0, s>>>(n_valid, sorted, flag);
  CKR(exclusive_sum(c, ar, flag, pos, n_valid + 1));
  uint32_t nuq = 0;
  CKR(mail_fetch(c, &nuq, pos + n_valid, 4));
  k_unique_scatter<<<grid_for(n_valid, 256, c->sm_count), 256, 0, s>>>(n_valid, sorted, flag, pos, other, col);
  CKR(mail_wait(c));
  k_rowptr_from_keys<<<grid_for(n_rows + 1, 256, c->sm_count), 256, 0, s>>>(n_rows, nuq, other, rp);
  c->launches += 3;
  ar.release(flag);
  ar.release(pos);
  *n_unique = nuq;
  return CCO_OK;
}

// canonicalisation slow path: sort (row,col) keys, drop duplicates, rebuild row_ptr
static int canonicalize_device(cco_ctx *c, Arena &ar, DevRaw &m) {
  if (m.nnz == 0) return CCO_OK;
  unsigned long long *k0, *k1;
  CKR(ar.alloc(&k0, m.nnz));
  CKR(ar.alloc(&k1, m.nnz));
  k_expand_keys<<<grid_for(m.n_rows * kSG, 256, c->sm_count), 256, 0, c->stream>>>(m.n_rows, m.rp, m.col, k0);
  c->launches++;
  // the canonical block is rewritten 0-based at the start of its own column storage
  long long n_unique = 0;
  CKR(keys_to_csr(c, ar, k0, k1, m.nnz, 32 + bits_for(m.n_rows), m.nnz, m.n_rows, m.col + m.q_base, m.rp, &n_unique));
  m.col += m.q_base;
  m.q_base = 0;
  m.nnz = n_unique;
  CK(cudaGetLastError());
  ar.release(k0);
  ar.release(k1);
  return CCO_OK;
}

// rows with more than kHeavyRow entries of a block, listed once per train and matrix (k_list_heavy_rows)
struct HeavyRows {
  int32_t *list = nullptr;
  int *n = nullptr;
};
static int list_heavy_rows(cco_ctx *c, Arena &ar, const DevRaw &raw, HeavyRows *h) {
  CKR(ar.alloc(&h->list, std::max<long long>(raw.n_rows, 1)));
  CKR(ar.alloc(&h->n, 1));
  CK(cudaMemsetAsync(h->n, 0, 4, c->stream));
  if (raw.n_rows > 0) {
    k_list_heavy_rows<<<grid_for(raw.n_rows, 256, c->sm_count), 256, 0, c->stream>>>(raw.n_rows, raw.rp, h->list, h->n);
    c->launches++;
  }
  return CCO_OK;
}
// a row-parallel pass = one launch over the light rows (kSG lanes per row) + one over the listed heavy rows (a warp per
// row; a fixed few waves of CTAs loop over the list, whose length they read on the device)
static void launch_check(cco_ctx *c, const DevRaw &raw, const HeavyRows &h, int *flags) {
  if (raw.n_rows <= 0) return;
  const long long q_lo = raw.q_base, q_hi = raw.q_base + raw.nnz;
  k_check_rows<kSG><<<grid_for(raw.n_rows * kSG, 256, c->sm_count), 256, 0, c->stream>>>(raw.n_rows, raw.n_cols, raw.rp, raw.col, q_lo, q_hi,
                                                                                       nullptr, nullptr, flags);
  k_check_rows<32><<<c->sm_count * 4, 256, 0, c->stream>>>(raw.n_rows, raw.n_cols, raw.rp, raw.col, q_lo, q_hi, h.list, h.n, flags);
  c->launches += 2;
}
// per-matrix scratch of the two sampling passes: integer keep thresholds per column, one keep byte per stored entry
struct SampleScratch {
  unsigned long long *col_thr = nullptr;
  uint8_t *keep = nullptr;
};
static int sample_scratch(cco_ctx *c, Arena &ar, const DevRaw &raw, const int32_t *raw_counts, int32_t m, SampleScratch *sc) {
  CKR(ar.alloc(&sc->col_thr, std::max<int32_t>(raw.n_cols, 1)));
  CKR(ar.alloc(&sc->keep, std::max<long long>(raw.nnz, 1)));
  if (raw.n_cols > 0) {
    k_col_thresholds<<<grid_for(raw.n_cols, 256, c->sm_count, 4), 256, 0, c->stream>>>(raw.n_cols, raw_counts, m, sc->col_thr);
    c->launches++;
  }
  return CCO_OK;
}
// pass 1 (k_sample_count, cco_sampler.cuh): entry-parallel; `kept` must be zero for the block's rows; `bad` (nullable) is the
// device verdict of count_raw_columns -- a malformed matrix keeps nothing, so pass 2 can never write more than row_ptr promises
static void launch_count(cco_ctx *c, const DevRaw &raw, const SampleScratch &sc, int32_t m, int32_t seed, uint32_t flags, const int *bad,
                         uint32_t *kept, int32_t *new_counts) {
  if (raw.n_rows <= 0 || raw.nnz <= 0) return;
  const long long q_lo = raw.q_base, q_hi = raw.q_base + raw.nnz;
  const long long n_chunks = (raw.nnz + kSampleChunk - 1) / kSampleChunk;
  k_sample_count<<<grid_for(n_chunks * 32, 256, c->sm_count), 256, 0, c->stream>>>(raw.n_rows, raw.row_base, raw.rp, raw.col, raw.n_cols, q_lo, q_hi,
                                                                                  sc.col_thr, m, seed, flags, bad, kept, new_counts, sc.keep);
  c->launches++;
}
// pass 2: order-preserving compaction of the block's column indices by the keep bytes.  Kept entries keep their global
// order, so entry ranks inside the block are offsets from the block's first kept entry: `dst` is where that one goes.
static int launch_write(cco_ctx *c, Arena &ar, const DevRaw &raw, const SampleScratch &sc, int32_t *dst) {
  if (raw.n_rows <= 0 || raw.nnz <= 0) return CCO_OK;
  long long *n_sel;
  CKR(ar.alloc(&n_sel, 1));
  size_t tb = 0;
  CK(cub::DeviceSelect::Flagged(nullptr, tb, raw.col + raw.q_base, sc.keep, dst, n_sel, (long long)raw.nnz, c->stream));
  void *tmp;
  CKR(ar.alloc((char **)&tmp, tb));
  CK(cub::DeviceSelect::Flagged(tmp, tb, raw.col + raw.q_base, sc.keep, dst, n_sel, (long long)raw.nnz, c->stream));
  ar.release(tmp);
  c->launches += 2;   // init + select kernel
  return CCO_OK;
}

// Raw column counts (numNonZeroElementsPerColumn) of a block of user rows of every matrix, the one way the library counts
// them.  Matrices whose column space fits a CTA's shared memory as 16-bit counters are counted and row_ptr-checked by
// k_col_counts_smem, kHistSegs matrices per launch.  The others (C4: 1 M columns) take k_check_row_ptr and
// k_col_histogram_flat<true> into kHistCopies replicated copies, folded by one k_sum_copies.  *counts (allocated here):
// col_off[n] words, matrix i at col_off[i].  ready (nullable): per matrix, the event after which its block is on the
// device.  verdict (nullable: the block is validated already): 2 ints per matrix, [2i] set for a malformed matrix.
constexpr int kHistCopies = 16;
static bool hist_fits_smem(const cco_ctx *c, int32_t n_cols) { return ((size_t)n_cols + 1) / 2 * 4 <= c->smem_optin; }
static int count_raw_columns(cco_ctx *c, Arena &ar, const std::vector<DevRaw> &raw, const std::vector<long long> &col_off, const cudaEvent_t *ready,
                             int *verdict, int32_t **counts_out) {
  cudaStream_t s = c->stream;
  const int n_mats = (int)raw.size();
  const long long total_cols = col_off[n_mats];
  const long long copy_stride = std::max<long long>(total_cols, 1);
  bool copies = false;
  for (int i = 0; i < n_mats; ++i) copies = copies || (raw[i].n_rows > 0 && !hist_fits_smem(c, raw[i].n_cols));
  const int n_copies = copies ? kHistCopies : 1;
  int32_t *counts;
  CKR(ar.alloc(&counts, (size_t)copy_stride * n_copies));
  CK(cudaMemsetAsync(counts, 0, sizeof(int32_t) * (size_t)copy_stride * n_copies, s));
  *counts_out = counts;
  // shared-memory path: CTAs of a batch go to its matrices in proportion to their entries, each at least
  // kHistMinEntries, so that no CTA spends more time zeroing and flushing its counters than counting
  std::vector<int> fit;
  for (int i = 0; i < n_mats; ++i)
    if (raw[i].n_rows > 0 && hist_fits_smem(c, raw[i].n_cols)) fit.push_back(i);
  for (size_t b0 = 0; b0 < fit.size(); b0 += kHistSegs) {
    const size_t b1 = std::min(fit.size(), b0 + kHistSegs);
    HistBatch hb{};
    long long nnz_sum = 0;
    int32_t max_cols = 0;
    for (size_t t = b0; t < b1; ++t) {
      nnz_sum += raw[fit[t]].nnz;
      max_cols = std::max(max_cols, raw[fit[t]].n_cols);
    }
    const size_t smem = ((size_t)max_cols + 1) / 2 * 4;
    const int per_sm = std::max(1, std::min<int>(2048 / kHistThreads, (int)(c->smem_optin / std::max<size_t>(smem + 1024, 1))));
    const long long target = (long long)c->sm_count * per_sm;
    for (size_t t = b0; t < b1; ++t) {
      const int i = fit[t];
      if (ready) CK(cudaStreamWaitEvent(s, ready[i], 0));   // async upload: matrix i has landed
      // CCO_FLAG_ASSUME_CANONICAL skips the canonicalisation, not the safety net: a malformed matrix still fails the call
      // (until the verdict is read, the counts skip ids outside the column space and the sampler keeps nothing)
      const long long share = nnz_sum > 0 ? (target * raw[i].nnz + nnz_sum - 1) / nnz_sum : 1;
      const long long need = (raw[i].nnz + kHistMinEntries - 1) / kHistMinEntries;
      HistSeg &g = hb.seg[hb.n++];
      g.col = raw[i].col + raw[i].q_base;
      g.rp = raw[i].rp;
      g.nnz = raw[i].nnz;
      g.n_rows = raw[i].n_rows;
      g.q_lo = raw[i].q_base;
      g.q_hi = raw[i].q_base + raw[i].nnz;
      g.counts = counts + col_off[i];
      g.verdict = verdict ? verdict + 2 * i : nullptr;
      g.n_cols = raw[i].n_cols;
      g.cta0 = hb.cta_end;
      hb.cta_end += (int32_t)std::max(1LL, std::min(share, need));
    }
    CK(cudaFuncSetAttribute(k_col_counts_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_col_counts_smem<<<hb.cta_end, kHistThreads, smem, s>>>(hb);
    c->launches++;
  }
  for (int i = 0; i < n_mats && copies; ++i) {
    if (raw[i].n_rows == 0 || hist_fits_smem(c, raw[i].n_cols)) continue;
    if (ready) CK(cudaStreamWaitEvent(s, ready[i], 0));
    int *v = verdict ? verdict + 2 * i : nullptr;
    if (v) {
      k_check_row_ptr<<<grid_for(raw[i].n_rows, 256, c->sm_count), 256, 0, s>>>(raw[i].n_rows, raw[i].rp, raw[i].q_base, raw[i].q_base + raw[i].nnz, v);
      c->launches++;
    }
    if (raw[i].nnz > 0) {
      // warp-aggregated (__match_any_sync) before the atomics: Zipf-hot columns take one atomic per warp instead of per lane
      k_col_histogram_flat<true><<<grid_for(raw[i].nnz, 256, c->sm_count), 256, 0, s>>>(raw[i].nnz, raw[i].col + raw[i].q_base, raw[i].n_cols,
                                                                                       counts + col_off[i], kHistCopies, copy_stride, v);
      c->launches++;
    }
  }
  if (copies) {
    k_sum_copies<<<grid_for(total_cols, 256, c->sm_count), 256, 0, s>>>(total_cols, kHistCopies, copy_stride, counts);
    c->launches++;
  }
  if (ready)   // every block has landed before anything after the counts reads it (also the ones with no rows)
    for (int i = 0; i < n_mats; ++i) CK(cudaStreamWaitEvent(s, ready[i], 0));
  return CCO_OK;
}

static int nccl_check(int rc, const char *what) {
  if (rc != 0) return set_error(CCO_E_NCCL, "%s: %s", what, g_nccl.GetErrorString(rc));
  return CCO_OK;
}

// sampleDownAndBinarize of every matrix from the final (on several GPUs: all-reduced) raw column counts.  Rank r holds
// and samples only its block of users; every rank ends with the whole sampled matrices.  The same steps on any number of
// GPUs, each ending at one stage event:
//   [0] pass 1 of every matrix: keep bytes, kept counts per user, post-sample column counts
//   [1] on several GPUs the all-gather of the kept counts (all matrices) and the all-reduce of the post-sample column
//       counts (the marginals: nothing is re-counted on the gathered matrix); then the row_ptr scan of every matrix
//   [2] pass 2 of every matrix: on one GPU straight into the sampled matrix, on several into this rank's slot of a
//       gather buffer.  NCCL's all-gather moves equal counts per rank, so the slots are padded to the largest SAMPLED
//       block (2-3x smaller than the raw blocks at the 10M-user shapes); the block edges come from the scanned row_ptr
//       through one mailbox record (an event wait, not a stream sync)
//   [3] on several GPUs the all-gather of the column blocks and a pack kernel
static int downsample_all(cco_ctx *c, Arena &ar, const std::vector<DevRaw> &raw, const int *d_check /* [2 * n_mats] */, long long U,
                          const int32_t *raw_counts, int32_t *marg_all, const std::vector<long long> &col_off,
                          const cco_indicator_params_t *params, int32_t seed, uint32_t flags, std::vector<DevMat> &dm,
                          const cudaEvent_t *stage_ev /* [4] */) {
  cudaStream_t s = c->stream;
  const int W = c->world, r = c->rank, n_mats = (int)raw.size();
  const long long S = (U + W - 1) / W;
  std::vector<uint32_t *> kept(n_mats, nullptr);
  std::vector<SampleScratch> sc(n_mats);
  for (int i = 0; i < n_mats; ++i) {
    DevMat *out = &dm[i];
    out->n_rows = U;
    out->n_cols = raw[i].n_cols;
    out->marg = marg_all + col_off[i];
    CKR(ar.alloc(&kept[i], (size_t)(W * S + 1)));
    CKR(ar.alloc(&out->rp, U + 1));
    CK(cudaMemsetAsync(kept[i], 0, sizeof(uint32_t) * (size_t)(W * S + 1), s));
    CKR(sample_scratch(c, ar, raw[i], raw_counts + col_off[i], params[i].max_interactions, &sc[i]));
    launch_count(c, raw[i], sc[i], params[i].max_interactions, seed, flags, d_check + 2 * i, kept[i], out->marg);
  }
  CK(cudaEventRecord(stage_ev[0], s));
  if (W > 1) {
    if (S > 0) {
      g_nccl.GroupStart();
      for (int i = 0; i < n_mats; ++i) {
        int rc = g_nccl.AllGather(kept[i] + (size_t)r * S, kept[i], (size_t)S, kNcclUint32, c->comm, s);
        if (rc != 0) { g_nccl.GroupEnd(); return nccl_check(rc, "ncclAllGather(kept counts)"); }
      }
      CKR(nccl_check(g_nccl.GroupEnd(), "ncclGroupEnd(kept counts)"));
    }
    if (col_off[n_mats] > 0)
      CKR(nccl_check(g_nccl.AllReduce(marg_all, marg_all, (size_t)col_off[n_mats], kNcclInt32, kNcclSum, c->comm, s), "ncclAllReduce(marginals)"));
  }
  std::vector<uint32_t> edge((size_t)n_mats * (W + 1), 0);
  for (int i = 0; i < n_mats; ++i) {
    CKR(exclusive_sum(c, ar, kept[i], dm[i].rp, U + 1));
    ar.release(kept[i]);
    if (W > 1)
      for (int q = 0; q <= W; ++q) CKR(mail_fetch(c, &edge[(size_t)i * (W + 1) + q], dm[i].rp + std::min<long long>((long long)q * S, U), 4));
  }
  CK(cudaEventRecord(stage_ev[1], s));
  if (W > 1) CKR(mail_wait(c));
  std::vector<long long> cap(n_mats, 0);
  std::vector<int32_t *> gathered(n_mats, nullptr);
  for (int i = 0; i < n_mats; ++i) {
    if (W == 1) {
      CKR(ar.alloc(&dm[i].col, std::max<long long>(raw[i].nnz, 1)));
      CKR(launch_write(c, ar, raw[i], sc[i], dm[i].col));
    } else {
      for (int q = 0; q < W; ++q) cap[i] = std::max<long long>(cap[i], (long long)edge[(size_t)i * (W + 1) + q + 1] - edge[(size_t)i * (W + 1) + q]);
      CKR(ar.alloc(&dm[i].col, std::max<long long>(edge[(size_t)i * (W + 1) + W], 1)));
      if (cap[i] > 0) {
        CKR(ar.alloc(&gathered[i], (size_t)(cap[i] * W)));
        // kept entries keep their order: this rank's block goes to its slot relative to the block's first entry
        CKR(launch_write(c, ar, raw[i], sc[i], gathered[i] + (size_t)r * cap[i]));
      }
    }
    ar.release(sc[i].col_thr);
    ar.release(sc[i].keep);
  }
  CK(cudaEventRecord(stage_ev[2], s));
  if (W > 1) {
    g_nccl.GroupStart();
    for (int i = 0; i < n_mats; ++i) {
      if (!gathered[i]) continue;
      int rc = g_nccl.AllGather(gathered[i] + (size_t)r * cap[i], gathered[i], (size_t)cap[i], kNcclInt32, c->comm, s);
      if (rc != 0) { g_nccl.GroupEnd(); return nccl_check(rc, "ncclAllGather(column blocks)"); }
    }
    CKR(nccl_check(g_nccl.GroupEnd(), "ncclGroupEnd(column blocks)"));
    for (int i = 0; i < n_mats; ++i) {
      if (!gathered[i]) continue;
      dim3 grid((unsigned)std::max(1, std::min(c->sm_count * 8 / W, 1024)), (unsigned)W);
      k_pack_blocks<<<grid, 256, 0, s>>>(W, S, U, cap[i], dm[i].rp, gathered[i], dm[i].col);
      c->launches++;
      ar.release(gathered[i]);
    }
  }
  CK(cudaEventRecord(stage_ev[3], s));
  CK(cudaGetLastError());
  return CCO_OK;
}

// ---- row-kernel configurations -----------------------------------------------------------------

struct BinCfg {
  int group;    // threads that own one row: 32 (warp), 256 or 1024 (whole CTA)
  int slots;    // table words per group
  int cap;      // distinct keys a hashed table may hold per pass
  int cbuf;     // candidate buffer entries per group
  int caux, keep_max, final_max;
  bool dense;
  bool bitmap;    // bitmap rows (use_bitmap): slots = repeat-table words, then bm_words of bitmap and top_k singles
  bool sorted;    // sorted rows (use_sorted): the table holds a row's keys and the radix sort's second buffer
  int bm_words;
  size_t region;  // shared-memory bytes per group
  size_t smem;    // per CTA
  int ctas_per_sm;
};

static int next_pow2(int x) {
  int p = 1;
  while (p < x) p <<= 1;
  return p;
}

template <int GROUP>
static int launch_rows_t(cco_ctx *c, const RowArgs &a, BinCfg &cfg, cudaStream_t st) {
  constexpr int CTA = GROUP == 32 ? 64 : GROUP;   // warp-owned rows: two independent warps per CTA (fine-grained smem packing)
  int occ = 1;
  void (*kern)(const RowArgs) = cfg.dense ? k_rows<GROUP, true> : k_rows<GROUP, false>;
  if constexpr (GROUP == 512 || GROUP == 256)
    if (cfg.bitmap) kern = k_rows<GROUP, false, true>;
  if constexpr (GROUP == 32)
    if (cfg.sorted) kern = k_rows<32, false, false, true>;
  CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cfg.smem));
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, CTA, cfg.smem));
  // 4 waves of CTAs over the work-sorted row list: a CTA that draws cheap rows retires early and the hardware
  // scheduler backfills, which balances the tail better than one persistent wave
  kern<<<c->sm_count * std::max(occ, 1) * 4, CTA, cfg.smem, st>>>(a);
  cfg.ctas_per_sm = occ;
  c->launches++;
  CK(cudaGetLastError());
  return CCO_OK;
}
static int launch_rows(cco_ctx *c, const RowArgs &a, BinCfg &cfg, cudaStream_t st) {
  switch (cfg.group) {
    case 1024: return launch_rows_t<1024>(c, a, cfg, st);
    case 512: return launch_rows_t<512>(c, a, cfg, st);
    case 256: return launch_rows_t<256>(c, a, cfg, st);
    case 128: return launch_rows_t<128>(c, a, cfg, st);
    case 32: return launch_rows_t<32>(c, a, cfg, st);
  }
  return set_error(CCO_E_INVALID_ARG, "internal: bad bin config");
}

static BinCfg make_cfg(cco_ctx *c, int group, int want_slots, int top_k, int n_cols_b) {
  BinCfg f;
  const int groups = group == 32 ? 2 : 1;
  f.group = group;
  f.final_max = next_pow2(top_k);
  f.cbuf = next_pow2(top_k + std::max(group, 128) + (group == 32 ? 64 : 0));
  if (group == 32 && top_k + 32 <= 96) f.cbuf = 128;  // small top_k: a 128-entry buffer doubles the warps per SM
  f.keep_max = std::max(f.final_max, (f.cbuf - group) / 2);
  f.caux = group == 32 ? 0 : f.keep_max;
  // candidates, x12/x11 tables, ctrl, radix-select histogram (aliased by the level-1 cut bins), queues
  size_t fixed = (size_t)(f.cbuf + f.caux) * 16 + 2 * 256 + 512 + 1024 + (size_t)(group / 32) * 256;
  size_t avail = (c->smem_optin - 1024) / groups;  // slack for static shared memory
  int max_slots = (int)((avail - fixed) / 4) & ~1023;
  f.slots = std::min(want_slots, max_slots);
  f.cap = f.slots / 2;  // load factor <= 1/2: higher load factors lengthen the probe chains
  f.dense = n_cols_b <= f.slots;
  f.bitmap = false;
  f.sorted = false;
  f.bm_words = 0;
  f.region = (fixed + (size_t)f.slots * 4 + 15) & ~(size_t)15;
  f.smem = f.region * groups;
  f.ctas_per_sm = 1;
  return f;
}

// Bitmap rows (DESIGN.md 3.1): a hashed CTA-owned bin whose rows all take the key path with an exact cut counts each cell's
// first product into a bitmap over the keys and hashes only the repeats.  Its table then holds at most max_w / 2 cells at
// load factor <= 1/2, i.e. max_w words (rounded to the per-warp segments), next to ceil(n_cols_b / 32) bitmap words and
// top_k singles.  The bin switches only when that fits in the shared memory of its current table: same CTAs per SM.
// Only the 512- and 256-thread bins are candidates (their gain at C3 is in DESIGN.md 3.2): the 128-thread bin's table
// is too small to hold a 100 K-column bitmap, and the 1024-thread bins were not tried.
static bool use_bitmap(BinCfg &f, uint32_t max_w, int top_k, int n_cols_b) {
  if (f.dense || (f.group != 512 && f.group != 256)) return false;
  const long long seg = 32LL * (f.group / 32);
  const long long rep = (std::max<long long>(max_w, 64) + seg - 1) / seg * seg;
  const long long bm = ((long long)n_cols_b + 31) / 32;
  if (rep + bm + top_k > f.slots) return false;
  f.bitmap = true;
  f.slots = (int)rep;
  f.bm_words = (int)bm;
  return true;
}

// Sorted rows (DESIGN.md 3.1): a hashed warp-owned bin whose rows all take the key path with an exact cut sorts each row's
// keys instead of hashing them.  The radix sort ping-pongs between two max_w-word halves that end where the table ends and
// reach back over the select histogram and the evaluation queues (256 + 64 words, dead while a row counts); the second half,
// which holds the cells the score stage reads, stays inside the table.  The table so shrinks to max(2 max_w - 320, max_w)
// words -- bin 5 (max_w 1024) from 2048 to 1728, one more CTA per SM.  One packed u16 histogram per key digit lives in the
// candidate buffer (also dead while a row counts).  Digits as sort_digits (cco_kernels.cuh): ceil(key bits / 9) passes.
static bool use_sorted(BinCfg &f, uint32_t max_w, int count_bits) {
  constexpr int kAliased = 256 + 64;   // k_rows: hist + wqueue (NW = 1) lie right below the table
  if (f.dense || f.group != 32 || max_w > 1024u) return false;
  const int slots = std::max(2 * (int)max_w - kAliased, (int)max_w);
  const int kb = 32 - count_bits, passes = (kb + 8) / 9;
  const int dbits = std::max((kb + passes - 1) / passes, 6);
  if (slots > f.slots || (long long)passes << (dbits - 1) > 4LL * f.cbuf) return false;
  f.sorted = true;
  f.region -= (size_t)(f.slots - slots) * 4;
  f.smem = f.region * 2;
  f.slots = slots;
  return true;
}

// ---- exactness of the level-1 cut and the dominance filter under fp64 rounding (DESIGN.md 3.1) ---------------------------
// eps bounds |computed - real| of one LLR as k_rows (and llr_cells) evaluates it, u = 2^-53, M = N ln N:
//   * xlogx(x) = fl(x * log(x)) with the device log within 1 ulp: relative error <= 2u + u + 2u^2 < 3.01u.  The terms
//     enter the LLR as xN (once, net: the three copies are the same computed value) and three groups whose arguments
//     sum to N -- {ra, N - ra}, {cb, N - cb}, {k11, k12, k21, k22} -- and x ln x is superadditive, so each group sums
//     to <= M: the terms contribute <= 4 * 3.01u M.
//   * ten additions / subtractions, eight with |result| <= M and two (sre, sre - mat_e) with |result| <= 2M:
//     <= 12u M.  (The same holds for the ENTROPY_VARARGS order: its partial sums are also <= M.)
//   * the final * 2 is exact: eps <= 2 (12.04 + 12) u M + O(u^2 M) < 64u M = 2^-47 M.  A computed 0 (the clamp of
//     s < mat_e) only happens when the real LLR is below eps too.
static double llr_error_bound(long long n_users) {
  const double n = (double)n_users;
  return n > 1.0 ? std::ldexp(n * std::log(n), -47) : 0.0;
}
// The cut drops k11 == 1 cells of colB c + 1 (and above) because they rank below cells of colB c.  Real-valued, with
// r = rowA <= R = max rowA and c + 1 <= C = max colB:
//   -dLLR/dx = 2 [-ln(1 - 1/x) - ln((N - x) / (N - x - r + 1))] >= 2 [1/x - (r - 1) / (N - x - r + 1)]
// (-ln(1 - t) >= t and ln(1 + t) <= t), which decreases in x and in r, so over x in [c, c + 1]
//   LLR(c) - LLR(c + 1) >= G1 = 2 [1/C - (R - 1) / (N - C - R + 1)]      (when N - C - R + 1 > 0).
// When R C comes close to N / 2, G1 vanishes; there the dropped cell's side of the cut (2 r (c + 1) < N, so
// N - x - r + 1 >= r x) gives -dLLR/dx >= 2 / (r x), hence a gap >= 2 / (r (c + 1)) >= G2 = 2 / min(R C, N / 2).
// If max(G1, G2) > 2 eps, the computed values are strictly decreasing in colB too, and the cut (colB or key) is exact
// for them.  Otherwise the rows run without it (same output, more evaluations).  With the default m = 500 every
// marginal is ~560 and G1 ~ 3.5e-3, above 2 eps for every N < 2^31 (2 eps = 6.6e-4 there; 2.3e-6 at C4).  The cut goes
// off only when max colB nears 1 / eps: ~7.6e4 at N = 1e8, ~3000 at N = 2^31.
static bool cut_exact(long long n_users, int32_t max_marg_a, int32_t max_marg_b) {
  const double n = (double)n_users, r = (double)max_marg_a, c = (double)max_marg_b;
  if (r <= 0.0 || c <= 0.0) return true;
  double g = 2.0 / std::min(r * c, 0.5 * n);
  const double d = n - c - r + 1.0;
  if (d > 0.0) g = std::max(g, 2.0 * (1.0 / c - (r - 1.0) / d));
  return g > 2.0 * llr_error_bound(n_users);
}

// ---- bins of one indicator (or of one key range of it) -----------------------------------------------------------------
struct BinPlan {
  std::vector<BinCfg> cfgs;
  int32_t *d_bounds = nullptr;   // [bins + 3] row-list bounds, filled on the device by k_bin_bounds (allocated if null)
};
// the packed (key << count_bits | count) word for keys 0 .. n_keys - 1 and counts up to k11_max: false = it does not fit
static bool packed_bits(long long n_keys, long long k11_max, int *key_bits, int *count_bits) {
  int kb = 1;
  while (((1LL << kb) - 1) <= n_keys) ++kb;  // keys <= 2^kb - 2
  *key_bits = kb;
  *count_bits = 32 - kb;
  return *count_bits >= 1 && k11_max < (1LL << *count_bits);
}
static int plan_bins(cco_ctx *c, Arena &ar, int32_t n_items_a, int32_t n_cols_b, int count_bits, int32_t max_marg_a,
                     int32_t max_marg_b, long long n_users, int k_eff, bool emit_all, const uint32_t *sorted_work, cudaStream_t ss,
                     BinPlan *bp) {
  const bool warp_ok = k_eff + 32 <= 256;  // warp-owned rows keep a 256-entry candidate buffer
  // Work bins, largest rows first.  {threads that own a row, table words, largest row work w the bin takes}.
  // Bin 0 is the multi-pass bin (same config as bin 1).  Rows up to 1024 products are WARP-owned: no CTA barrier
  // anywhere in their count / compact / score / select pipeline; larger rows need the table and the parallelism of a CTA.
  struct BinSpec { int group, slots; uint32_t max_w; };
  std::vector<BinSpec> spec = {{1024, 1 << 20, 0xffffffffu}, {1024, 1 << 20, 0xffffffffu}, {512, 16384, 8192u}, {256, 8192, 4096u}};
  if (warp_ok) {
    // rows of 1025..2048 products: a 128-thread CTA shares one 4096-word table -- a warp-owned 4096-word table leaves
    // too few warps per SM; up to 1024 products rows are warp-owned
    spec.push_back({128, 4096, 2048u});
    spec.push_back({32, 2048, 1024u});
    spec.push_back({32, 1024, 512u});
    spec.push_back({32, 512, 256u});
  } else {
    spec.push_back({128, 4096, 2048u});
  }
  const int kBins = (int)spec.size();
  std::vector<BinCfg> &cfgs = bp->cfgs;
  cfgs.resize(kBins);
  for (int b = 0; b < kBins; ++b) cfgs[b] = make_cfg(c, spec[b].group, spec[b].slots, k_eff, n_cols_b);
  // thresholds on w, descending: bin b takes rows with h_thr[b-1] >= w > h_thr[b]; a hashed table also needs w <= cap
  std::vector<uint32_t> h_thr(kBins);
  for (int b = 0; b < kBins; ++b) {
    const BinCfg &f = cfgs[std::min(b + 1, kBins - 1)];   // h_thr[b] = upper limit of bin b+1
    uint32_t lim = b + 1 < kBins ? spec[b + 1].max_w : 0u;
    if (b + 1 < kBins && !f.dense) lim = std::min<uint32_t>(lim, (uint32_t)f.cap);
    h_thr[b] = lim;
    if (b > 0) h_thr[b] = std::min(h_thr[b], h_thr[b - 1]);
  }
  // bitmap and sorted rows: the k11 = 1 cells are cut by key, so every row must be keyed (2 rowA colB < N for the largest of both)
  // and the cut exact
  const bool bitmap_ok = !emit_all && cut_exact(n_users, max_marg_a, max_marg_b) &&
                         2ull * (unsigned long long)std::max(max_marg_a, 0) * (unsigned long long)std::max(max_marg_b, 0) <
                             (unsigned long long)n_users;
  for (int b = 1; b < kBins && bitmap_ok; ++b) {
    use_bitmap(cfgs[b], h_thr[b - 1], k_eff, n_cols_b);
    use_sorted(cfgs[b], h_thr[b - 1], count_bits);
  }
  if (!bp->d_bounds) CKR(ar.alloc(&bp->d_bounds, kBins + 3));   // key ranges reuse one across ranges
  BinThresholds bt;
  memset(&bt, 0, sizeof bt);
  for (int b = 0; b < kBins; ++b) bt.t[b] = h_thr[b];
  k_bin_bounds<<<1, 32, 0, ss>>>(n_items_a, sorted_work, kBins, bt, bp->d_bounds);
  c->launches++;
  return CCO_OK;
}
// the bins touch disjoint rows: run them concurrently (tails of one bin overlap the bulk of another); s joins them all
static int launch_bins(cco_ctx *c, const RowArgs &a, BinPlan &bp, cudaStream_t s) {
  std::vector<BinCfg> &cfgs = bp.cfgs;
  CK(cudaEventRecord(c->bin_ev[8], s));
  for (int b = 0; b < (int)cfgs.size(); ++b) {
    if (b == 0 && cfgs[1].dense) continue;                 // dense L takes every large row in bin 1
    RowArgs ab = a;
    ab.bin_bounds = bp.d_bounds;
    ab.bin = b;
    ab.slots = cfgs[b].slots;
    ab.cap = cfgs[b].cap;
    ab.tsize_x16 = 32;
    ab.cbuf = cfgs[b].cbuf;
    ab.caux = cfgs[b].caux;
    ab.keep_max = cfgs[b].keep_max;
    ab.final_max = cfgs[b].final_max;
    ab.group_smem_bytes = (int32_t)cfgs[b].region;
    ab.bm_words = cfgs[b].bm_words;
    CK(cudaStreamWaitEvent(c->bin_stream[b], c->bin_ev[8], 0));
    CKR(launch_rows(c, ab, cfgs[b], c->bin_stream[b]));
    CK(cudaEventRecord(c->bin_ev[b], c->bin_stream[b]));
    CK(cudaStreamWaitEvent(s, c->bin_ev[b], 0));
  }
  return CCO_OK;
}

// (n_cols_b - 1) >> key_shift < kCutBins: the first level of the key cut
static int key_shift_for(int32_t n_cols_b) {
  int sh = 0;
  while (((long long)std::max(n_cols_b - 1, 0) >> sh) >= kCutBins) ++sh;
  return sh;
}

// ---- key ranges (DESIGN.md 3.1 "key ranges") -----------------------------------------------------------------------------
// Keys number B' columns by (colB ascending, column id ascending), so colB never decreases with the key and a key range
// [k0, k1) has its largest colB at k1 - 1.  The range's counts fit the packed word when bitlen(k1 - k0 + 1) +
// bitlen(min(max rowA, colB(k1 - 1))) <= 32 (packed_bits).  Any sub-range of a range that fits fits too, so cutting
// greedily from key 0 upward, each range as long as it fits (and at most max_keys keys when max_keys > 0), gives the
// fewest ranges.  first_key_of_cb[c] (c in [0, max_marg_b + 1]) = first key whose colB >= c, as k_col_order builds it.
// False when a single key's counts do not fit.
struct KeyRange { int32_t k0, k1, max_marg; };
static bool plan_key_ranges(const int32_t *first_key_of_cb, int32_t max_marg_b, int32_t n_keys, int32_t max_marg_a,
                            int32_t max_keys, std::vector<KeyRange> *plan) {
  const int32_t *fk_end = first_key_of_cb + (size_t)max_marg_b + 2;
  auto marg = [&](int32_t k) { return (int32_t)(std::upper_bound(first_key_of_cb, fk_end, k) - first_key_of_cb) - 1; };
  auto fits = [&](int32_t k0, int32_t k1) {
    int kb, cb;
    return packed_bits((long long)k1 - k0, std::min<long long>(max_marg_a, marg(k1 - 1)), &kb, &cb);
  };
  plan->clear();
  for (int32_t k0 = 0; k0 < n_keys;) {
    const int32_t top = max_keys > 0 ? (int32_t)std::min<long long>(n_keys, (long long)k0 + max_keys) : n_keys;
    if (!fits(k0, k0 + 1)) return false;
    int32_t lo = k0 + 1, hi = top;   // the largest k1 in [lo, hi] that fits
    while (lo < hi) {
      const int32_t mid = lo + (hi - lo + 1) / 2;
      if (fits(k0, mid)) lo = mid; else hi = mid - 1;
    }
    plan->push_back({k0, lo, marg(lo - 1)});
    k0 = lo;
  }
  return true;
}

// ---- one indicator = rows [lo, hi) of A'^T B' on this rank ---------------------------------------------------------------
// enqueue_indicator puts everything of one indicator on the stream without a single host round trip (the rank partition,
// the bin bounds and the packed sizes stay on the device); finish_indicator waits for that indicator's mailbox record
// only -- while the GPU already runs the next indicator -- and starts the device->host copy of its packed arrays.
struct IndicatorState {
  int mail_group = -1;
  long long rec[7] = {0, 0, 0, 0, 0, 0, 0};   // k_indicator_record
  cudaEvent_t packed = nullptr;                // compaction done (the copy stream waits for it)
  long long *out_ptr = nullptr;                // [n_items_a + 1], 0 outside the rank's rows
  int32_t *p_col = nullptr, *p_cnt = nullptr;
  double *p_llr = nullptr;
  int32_t n_items_a = 0, n_cols_b = 0;
  int n_ranges = 1;                            // key ranges the indicator ran in
  bool emit_all = false;
};

static int enqueue_indicator(cco_ctx *c, Arena &ar, const uint32_t *at_ptr, const int32_t *at_users, int32_t n_items_a,
                             const int32_t *marg_a, int32_t max_marg_a, int32_t max_marg_b, const DevMat &B, long long n_users,
                             bool self, const cco_indicator_params_t &prm, uint32_t flags, bool emit_all, cudaEvent_t inputs_ready,
                             cudaEvent_t ev_begin, cudaEvent_t ev_end, IndicatorState *st) {
  cudaStream_t s = c->stream;
  const int32_t n_cols_b = B.n_cols;
  const int rank = c->rank, world = c->world;
  st->n_items_a = n_items_a;
  st->n_cols_b = n_cols_b;
  st->emit_all = emit_all;
  // 1. work per output row, rank partition, schedule --------------------------------------------------
  // The schedule reads only the prepared matrices, so it does not have to queue behind the previous indicator's row
  // kernels: with `inputs_ready` (recorded on s once the preparation is complete) it runs on the scheduling stream and s
  // joins it before the bins launch.  Everything it touches must then be slab memory (no stream-ordered allocation on s).
  uint32_t *row_work, *masked, *sorted_work;
  unsigned long long *work64;
  long long *work_prefix;
  int32_t *ids, *rows_sorted, *d_pb = nullptr;
  size_t sort_tb = 0, order_tb = 0;
  if (n_items_a > 0)
    CK(cub::DeviceRadixSort::SortPairsDescending(nullptr, sort_tb, (const uint32_t *)nullptr, (uint32_t *)nullptr, (const int32_t *)nullptr,
                                                 (int32_t *)nullptr, n_items_a, 0, 32, s));
  int cb_bits = 1;   // colB <= max_marg_b: the column-order sort looks at these key bits only
  while ((1LL << cb_bits) <= (long long)max_marg_b) ++cb_bits;
  cub::DoubleBuffer<uint32_t> order_cb(nullptr, nullptr);
  cub::DoubleBuffer<int32_t> order_id(nullptr, nullptr);
  if (n_cols_b > 0) CK(cub::DeviceRadixSort::SortPairs(nullptr, order_tb, order_cb, order_id, n_cols_b, 0, cb_bits, s));
  const bool beside = inputs_ready && ar.c && ((size_t)n_items_a + 1) * 8 <= Arena::kSlabMax && sort_tb <= Arena::kSlabMax &&
                      (size_t)n_cols_b * 4 <= Arena::kSlabMax && order_tb <= Arena::kSlabMax &&
                      ((size_t)max_marg_b + 2) * 4 <= Arena::kSlabMax;
  cudaStream_t ss = beside ? c->sched_stream : s;
  if (beside) CK(cudaStreamWaitEvent(ss, inputs_ready, 0));
  CKR(ar.alloc(&row_work, n_items_a + 1));
  CKR(ar.alloc(&masked, n_items_a + 1));
  CKR(ar.alloc(&work64, n_items_a + 1));
  CKR(ar.alloc(&work_prefix, n_items_a + 1));
  CKR(ar.alloc(&ids, n_items_a + 1));
  CKR(ar.alloc(&sorted_work, n_items_a + 1));
  CKR(ar.alloc(&rows_sorted, n_items_a + 1));
  CK(cudaMemsetAsync(work64 + n_items_a, 0, 8, ss));
  k_row_work<<<grid_for((long long)n_items_a * kSG, 256, c->sm_count), 256, 0, ss>>>(n_items_a, at_ptr, at_users, B.rp,
                                                                                  row_work, work64, ids, nullptr);
  c->launches++;
  CKR(exclusive_sum(c, ar, (const long long *)work64, work_prefix, (long long)n_items_a + 1, ss));
  if (world > 1) {
    // contiguous item ranges balanced by work prefix, identical on every rank; they never leave the device
    CKR(ar.alloc(&d_pb, world + 1));
    k_partition_rows<<<1, ((world + 1 + 31) / 32) * 32, 0, ss>>>(work_prefix, n_items_a, world, d_pb);
    c->launches++;
  }
  k_mask_work<<<grid_for(n_items_a, 256, c->sm_count), 256, 0, ss>>>(n_items_a, row_work, d_pb, rank, masked);
  c->launches++;
  if (n_items_a > 0) {
    void *tmp;
    CKR(ar.alloc((char **)&tmp, sort_tb));
    CK(cub::DeviceRadixSort::SortPairsDescending(tmp, sort_tb, masked, sorted_work, ids, rows_sorted, n_items_a, 0, 32, ss));
    ar.release(tmp);
  }
  // 2. packed word and bins -------------------------------------------------------------------------
  const int k_eff = emit_all ? 1 : prm.top_k;
  // a co-occurrence count is bounded by both marginals: k11 <= min(rowA, colB) <= min(max rowA, max colB).  With the
  // reference's default downsampling (m = 500) that is ~560, i.e. 10 count bits next to 22 key bits (4M columns).
  int key_bits, count_bits;
  const long long k11_max = std::min<long long>(max_marg_a, max_marg_b);
  const bool fits = packed_bits(n_cols_b, k11_max, &key_bits, &count_bits);
  // key ranges: the counts do not fit and the caller accepts the ranges' cost, or the debug cap forces them
  const bool split = n_cols_b > 0 && (c->key_range_cap > 0 || (!fits && (flags & CCO_FLAG_KEY_RANGES)));
  if (!fits && !split)
    return set_error(CCO_E_UNSUPPORTED,
                     "co-occurrence counts up to %lld over %d columns do not fit the packed 32-bit accumulator word "
                     "(key %d bits + count %d bits): lower maxItemsPerUser/maxEventsPerEventType for this event type, "
                     "or train it in key ranges with CCO_FLAG_KEY_RANGES (\"Limits\" in include/cco_b200.h)",
                     k11_max, n_cols_b, key_bits, count_bits);
  st->n_ranges = 1;
  BinPlan bins;
  if (!split)
    CKR(plan_bins(c, ar, n_items_a, n_cols_b, count_bits, max_marg_a, max_marg_b, n_users, k_eff, emit_all, sorted_work, ss, &bins));
  // column order of B' (DESIGN.md 3.1, step 3): key = rank under (colB ascending, column id ascending), from a stable
  // sort of the final post-sample marginals (identical on every rank).  B' is relabelled to keys IN PLACE: every B' is
  // this train's own sampled copy, and A' (the B' of the self indicator) has already been transposed.  Like the
  // schedule, it runs beside the previous indicator's row kernels.
  int32_t *key_of_col, *first_key_of_cb, *order_id0, *order_id1;
  uint32_t *order_cb0, *order_cb1;
  const int32_t n_order = std::max<int32_t>(n_cols_b, 1);
  CKR(ar.alloc(&key_of_col, n_order));
  CKR(ar.alloc(&first_key_of_cb, (size_t)max_marg_b + 2));
  CKR(ar.alloc(&order_cb0, n_order));
  CKR(ar.alloc(&order_cb1, n_order));
  CKR(ar.alloc(&order_id0, n_order));
  CKR(ar.alloc(&order_id1, n_order));
  order_cb = cub::DoubleBuffer<uint32_t>(order_cb0, order_cb1);
  order_id = cub::DoubleBuffer<int32_t>(order_id0, order_id1);
  if (n_cols_b > 0) {
    k_col_order_init<<<grid_for(n_cols_b, 256, c->sm_count, 4), 256, 0, ss>>>(n_cols_b, B.marg, order_cb0, order_id0);
    void *tmp;
    CKR(ar.alloc((char **)&tmp, order_tb));
    CK(cub::DeviceRadixSort::SortPairs(tmp, order_tb, order_cb, order_id, n_cols_b, 0, cb_bits, ss));
    ar.release(tmp);
    k_col_order<<<grid_for(n_cols_b, 256, c->sm_count, 4), 256, 0, ss>>>(n_cols_b, max_marg_b, order_cb.Current(), order_id.Current(),
                                                                        key_of_col, first_key_of_cb);
    k_relabel_cols<<<c->sm_count * 8, 256, 0, ss>>>(B.rp + B.n_rows, key_of_col, B.col);
    c->launches += 3;
  }
  const int32_t *marg_key = reinterpret_cast<const int32_t *>(order_cb.Current()), *col_of_key = order_id.Current();
  if (beside) {
    cudaEvent_t scheduled;
    CKR(pooled_event(c, false, &scheduled));
    CK(cudaEventRecord(scheduled, ss));
    CK(cudaStreamWaitEvent(s, scheduled, 0));
  }
  // per-column constants of B' for the fused LLR, in key order
  ColTerm *col_terms;
  CKR(ar.alloc(&col_terms, std::max<int32_t>(n_cols_b, 1)));
  if (n_cols_b > 0) {
    k_col_terms<<<grid_for(n_cols_b, 256, c->sm_count, 4), 256, 0, s>>>(n_cols_b, marg_key, col_of_key, n_users, flags, col_terms);
    c->launches++;
  }
  // 3. outputs ----------------------------------------------------------------------------------------
  int32_t stride = emit_all ? n_cols_b : std::min<int32_t>(prm.top_k, n_cols_b);
  if (stride < 1) stride = 1;
  int32_t *o_col, *o_cnt, *o_len;
  double *o_llr = nullptr;
  unsigned long long *d_distinct;
  int *d_err;
  size_t cells = (size_t)std::max(n_items_a, 1) * stride;
  CKR(ar.alloc(&o_col, cells));
  CKR(ar.alloc(&o_cnt, cells));
  if (!emit_all) CKR(ar.alloc(&o_llr, cells));
  CKR(ar.alloc(&o_len, n_items_a + 1));
  CKR(ar.alloc(&d_distinct, 2));
  CKR(ar.alloc(&d_err, 1));
  CK(cudaMemsetAsync(o_len, 0, sizeof(int32_t) * ((size_t)n_items_a + 1), s));
  CK(cudaMemsetAsync(d_distinct, 0, 16, s));
  CK(cudaMemsetAsync(d_err, 0, 4, s));
  RowArgs a;
  memset(&a, 0, sizeof a);
  a.at_ptr = at_ptr;
  a.at_users = at_users;
  a.b_ptr = B.rp;
  a.b_col = B.col;
  a.marg_a = marg_a;
  a.marg_b = marg_key;
  a.key_of_col = key_of_col;
  a.first_key_of_cb = first_key_of_cb;
  a.key_shift = key_shift_for(n_cols_b);
  a.max_marg_b = max_marg_b;
  a.col_terms = col_terms;
  a.rows_sorted = rows_sorted;
  a.row_work = row_work;
  a.n_cols_b = n_cols_b;
  a.n_users = n_users;
  a.self = self ? 1 : 0;
  a.top_k = k_eff;
  a.has_min_llr = prm.has_min_llr;
  a.min_llr = prm.min_llr;
  a.cut_ok = cut_exact(n_users, max_marg_a, max_marg_b) ? 1 : 0;
  a.llr_eps2 = 2.0 * llr_error_bound(n_users);
  a.flags = flags;
  a.count_bits = count_bits;
  a.out_stride = stride;
  a.out_col = o_col;
  a.out_llr = o_llr;
  a.out_cnt = o_cnt;
  a.out_len = o_len;
  a.stat_distinct = d_distinct;
  a.stat_evaluated = d_distinct + 1;
  a.err_flag = d_err;
  a.emit_all = emit_all ? 1 : 0;
  a.key_base = 0;
  if (ev_begin) CK(cudaEventRecord(ev_begin, s));
  if (!split) {
    if (n_items_a > 0) CKR(launch_bins(c, a, bins, s));
  } else {
    // 2b. key ranges (DESIGN.md 3.1 "key ranges"): the plan is cut on the host from first_key_of_cb, read together with
    // nnz(B') in one round trip (a plain copy: max colB + 2 ints can outgrow the mailbox).  The marginals are all-reduced,
    // so every rank cuts the same plan.
    const int32_t n_fk = max_marg_b + 2;
    int32_t *h_fk = (int32_t *)c->pinned_get(sizeof(int32_t) * ((size_t)n_fk + 1), false);
    if (!h_fk) return set_error(CCO_E_OOM, "pinned host allocation failed");
    struct PutBack { cco_ctx *c; void *p; ~PutBack() { c->pinned_put(p); } } put_back{c, h_fk};
    CK(cudaMemcpyAsync(h_fk, first_key_of_cb, sizeof(int32_t) * (size_t)n_fk, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(h_fk + n_fk, B.rp + B.n_rows, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    std::vector<KeyRange> plan;
    if (!plan_key_ranges(h_fk, max_marg_b, n_cols_b, max_marg_a, c->key_range_cap, &plan))
      return set_error(CCO_E_UNSUPPORTED,
                       "co-occurrence counts up to %lld do not fit the packed 32-bit accumulator word even in a key range of one "
                       "column (at most 2^30 - 1): lower maxItemsPerUser/maxEventsPerEventType for this event type "
                       "(\"Limits\" in include/cco_b200.h)", k11_max);
    const long long nnz_b = (long long)(uint32_t)h_fk[n_fk], U = B.n_rows;
    st->n_ranges = (int)plan.size();
    // Everything the ranges need is allocated once, here: one range's B'_r at a time, the running top-k next to one
    // range's rows, and one set of scratch (scan and sort storage, the range's first_key_of_cb, the bin bounds) reused
    // by every range -- memory does not grow with the number of ranges.
    uint32_t *r_cnt, *r_ptr;
    int32_t *r_col, *fk_r, *t_col = nullptr, *t_cnt = nullptr, *t_len = nullptr;
    double *t_llr = nullptr;
    void *scan_tmp, *sort_tmp;
    size_t scan_tb = 0;
    CKR(ar.alloc(&r_cnt, U + 1));
    CKR(ar.alloc(&r_ptr, U + 1));
    CK(cub::DeviceScan::ExclusiveSum(nullptr, scan_tb, r_cnt, r_ptr, U + 1, s));
    CKR(ar.alloc(&r_col, std::max<long long>(nnz_b, 1)));
    CKR(ar.alloc(&fk_r, (size_t)max_marg_b + 2));
    CKR(ar.alloc((char **)&scan_tmp, scan_tb));
    CKR(ar.alloc((char **)&sort_tmp, sort_tb));
    BinPlan bp;
    if (plan.size() > 1) {
      CKR(ar.alloc(&t_col, cells));
      CKR(ar.alloc(&t_cnt, cells));
      if (!emit_all) CKR(ar.alloc(&t_llr, cells));
      CKR(ar.alloc(&t_len, n_items_a + 1));
    }
    const int split_grid = grid_for(U * 32, 256, c->sm_count);
    for (size_t r = 0; r < plan.size(); ++r) {
      const KeyRange kr = plan[r];
      const int32_t n_r = kr.k1 - kr.k0;
      k_split_range<false><<<split_grid, 256, 0, s>>>(U, B.rp, B.col, kr.k0, kr.k1, r_cnt, nullptr);
      CK(cub::DeviceScan::ExclusiveSum(scan_tmp, scan_tb, r_cnt, r_ptr, U + 1, s));
      k_split_range<true><<<split_grid, 256, 0, s>>>(U, B.rp, B.col, kr.k0, kr.k1, r_ptr, r_col);
      c->launches += 2;
      // the range's schedule: products per row over B'_r, masked to this rank's rows (the partition of the whole B')
      k_row_work<<<grid_for((long long)n_items_a * kSG, 256, c->sm_count), 256, 0, s>>>(n_items_a, at_ptr, at_users, r_ptr, row_work,
                                                                                     work64, ids, nullptr);
      k_mask_work<<<grid_for(n_items_a, 256, c->sm_count), 256, 0, s>>>(n_items_a, row_work, d_pb, rank, masked);
      c->launches += 2;
      if (n_items_a > 0)
        CK(cub::DeviceRadixSort::SortPairsDescending(sort_tmp, sort_tb, masked, sorted_work, ids, rows_sorted, n_items_a, 0, 32, s));
      k_range_first_keys<<<grid_for((long long)kr.max_marg + 2, 256, c->sm_count), 256, 0, s>>>(kr.max_marg + 2, first_key_of_cb, kr.k0,
                                                                                             n_r, fk_r);
      c->launches++;
      int kb_r, cbits_r;
      packed_bits(n_r, std::min<long long>(max_marg_a, kr.max_marg), &kb_r, &cbits_r);
      CKR(plan_bins(c, ar, n_items_a, n_r, cbits_r, max_marg_a, kr.max_marg, n_users, k_eff, emit_all, sorted_work, s, &bp));
      // the range as a view of B': keys rebased by k0, the per-key tables offset by k0 (the output keeps column ids)
      RowArgs ar_r = a;
      ar_r.b_ptr = r_ptr;
      ar_r.b_col = r_col;
      ar_r.marg_b = marg_key + kr.k0;
      ar_r.col_terms = col_terms + kr.k0;
      ar_r.first_key_of_cb = fk_r;
      ar_r.key_base = kr.k0;
      ar_r.key_shift = key_shift_for(n_r);
      ar_r.max_marg_b = kr.max_marg;
      ar_r.n_cols_b = n_r;
      ar_r.cut_ok = cut_exact(n_users, max_marg_a, kr.max_marg) ? 1 : 0;
      ar_r.count_bits = cbits_r;
      if (r > 0) {   // later ranges write beside the running result and are merged into it
        ar_r.out_col = t_col;
        ar_r.out_llr = t_llr;
        ar_r.out_cnt = t_cnt;
        ar_r.out_len = t_len;
        CK(cudaMemsetAsync(t_len, 0, sizeof(int32_t) * ((size_t)n_items_a + 1), s));
      }
      if (n_items_a > 0) CKR(launch_bins(c, ar_r, bp, s));
      if (r > 0 && n_items_a > 0) {
        k_merge_range<<<grid_for((long long)n_items_a * 32, 256, c->sm_count), 256, 0, s>>>(n_items_a, stride, k_eff, emit_all ? 1 : 0, o_col,
                                                                                         o_llr, o_cnt, o_len, t_col, t_llr, t_cnt, t_len);
        c->launches++;
      }
    }
  }
  if (ev_end) CK(cudaEventRecord(ev_end, s));
  // 4. pack ---------------------------------------------------------------------------------------------
  long long *len64, *rec_d;
  CKR(ar.alloc(&len64, n_items_a + 1));
  CKR(ar.alloc(&st->out_ptr, n_items_a + 1));
  CKR(ar.alloc(&rec_d, 8));
  k_len_to_i64<<<grid_for((long long)n_items_a + 1, 256, c->sm_count), 256, 0, s>>>(n_items_a, o_len, d_pb, rank, len64);
  c->launches++;
  CKR(exclusive_sum(c, ar, len64, st->out_ptr, (long long)n_items_a + 1));
  // the packed size is only known on the device: the buffers take the worst case (every row of the item space full)
  CKR(ar.alloc(&st->p_col, cells));
  if (!(flags & CCO_FLAG_RESULT_NO_COUNT) || emit_all) CKR(ar.alloc(&st->p_cnt, cells));
  if (!emit_all && !(flags & CCO_FLAG_RESULT_NO_LLR)) CKR(ar.alloc(&st->p_llr, cells));
  if (n_items_a > 0) {
    k_compact_rows<<<grid_for((long long)n_items_a * 32, 256, c->sm_count), 256, 0, s>>>(n_items_a, stride, st->out_ptr, o_col, o_llr,
                                                                                      o_cnt, st->p_col, st->p_llr, st->p_cnt);
    c->launches++;
  }
  k_indicator_record<<<1, 32, 0, s>>>(n_items_a, d_pb, rank, st->out_ptr, work_prefix, d_distinct, d_err, rec_d);
  c->launches++;
  CKR(mail_fetch(c, st->rec, rec_d, sizeof(long long) * 7));
  CKR(mail_close(c, &st->mail_group));
  if (!st->packed) CK(cudaEventCreateWithFlags(&st->packed, cudaEventDisableTiming));
  CK(cudaEventRecord(st->packed, s));
  CK(cudaGetLastError());
  // the strided buffers are dead once k_compact_rows has been enqueued (stream order)
  for (void *p : {(void *)o_col, (void *)o_cnt, (void *)o_llr, (void *)len64})
    if (p) ar.release(p);
  return CCO_OK;
}

struct IndicatorOut {
  int64_t row_begin = 0, row_end = 0;
  int64_t nnz = 0;
  int64_t products = 0, distinct = 0, evaluated = 0;
};

// wait for the indicator's record, allocate its host arrays, start the device->host copies on the copy stream
static int finish_indicator(cco_ctx *c, IndicatorState *st, uint32_t flags, int index, ResultMat *rm, IndicatorOut *io) {
  CKR(mail_wait_group(c, st->mail_group));
  const int32_t lo = (int32_t)st->rec[0], hi = (int32_t)st->rec[1];
  const long long total = st->rec[2];
  io->row_begin = lo;
  io->row_end = hi;
  io->nnz = total;
  io->products = st->rec[3];
  io->distinct = st->rec[4];
  io->evaluated = st->rec[5];
  if (st->rec[6]) return set_error(CCO_E_CUDA, "internal: shared-memory hash table overflow");
  const int32_t n_my = hi - lo;
  cudaStream_t cs = c->copy_stream;
  CK(cudaStreamWaitEvent(cs, st->packed, 0));
  GroupShared *gs = c->gshared;
  int64_t *h_rp;
  int32_t *h_col, *h_cnt = nullptr;
  double *h_llr = nullptr;
  long long base = 0;
  if (gs) {
    // group mode: every rank's slice lands in ONE set of host arrays (rank 0 of the group allocates them once all
    // ranks know their sizes); row pointers are rebased on the device by the cells of the ranks before this one
    {
      std::lock_guard<std::mutex> lk(gs->mu);
      gs->totals[c->rank] = total;
    }
    gs->barrier();
    long long grand = 0;
    for (int q = 0; q < gs->world; ++q) {
      if (q < c->rank) base += gs->totals[q];
      grand += gs->totals[q];
    }
    ResultMat &mm = gs->merged->mats[index];
    if (c->rank == 0) {
      cco_ctx *owner = gs->merged->ctx;
      mm.row_begin = 0;
      mm.row_end = st->n_items_a;
      mm.n_cols = st->n_cols_b;
      mm.row_ptr = (int64_t *)owner->pinned_get(sizeof(int64_t) * ((size_t)st->n_items_a + 1));
      mm.col = (int32_t *)owner->pinned_get(sizeof(int32_t) * (size_t)std::max<long long>(grand, 1));
      if (st->p_cnt) mm.cnt = (int32_t *)owner->pinned_get(sizeof(int32_t) * (size_t)std::max<long long>(grand, 1));
      if (st->p_llr) mm.llr = (double *)owner->pinned_get(sizeof(double) * (size_t)std::max<long long>(grand, 1));
      mm.key_ranges = st->n_ranges;   // every rank cuts the same plan
    }
    gs->barrier();
    if (!mm.row_ptr || !mm.col || (st->p_cnt && !mm.cnt) || (st->p_llr && !mm.llr)) return set_error(CCO_E_OOM, "pinned host allocation failed");
    h_rp = mm.row_ptr + lo;
    h_col = mm.col + base;
    h_cnt = mm.cnt ? mm.cnt + base : nullptr;
    h_llr = mm.llr ? mm.llr + base : nullptr;
    if (base != 0 && n_my >= 0) {
      k_add_i64<<<grid_for((long long)n_my + 1, 256, c->sm_count, 2), 256, 0, cs>>>((long long)n_my + 1, base, st->out_ptr + lo);
      c->launches++;
    }
    rm->row_begin = lo;   // the member's own record (stats only; the arrays belong to the merged result)
    rm->row_end = hi;
    rm->n_cols = st->n_cols_b;
    rm->key_ranges = st->n_ranges;
  } else {
    rm->row_begin = lo;
    rm->row_end = hi;
    rm->n_cols = st->n_cols_b;
    rm->key_ranges = st->n_ranges;
    rm->row_ptr = (int64_t *)c->pinned_get(sizeof(int64_t) * ((size_t)n_my + 1));
    rm->col = (int32_t *)c->pinned_get(sizeof(int32_t) * (size_t)std::max<long long>(total, 1));
    if (st->p_cnt) rm->cnt = (int32_t *)c->pinned_get(sizeof(int32_t) * (size_t)std::max<long long>(total, 1));
    if (st->p_llr) rm->llr = (double *)c->pinned_get(sizeof(double) * (size_t)std::max<long long>(total, 1));
    if (!rm->row_ptr || !rm->col || (st->p_cnt && !rm->cnt) || (st->p_llr && !rm->llr))
      return set_error(CCO_E_OOM, "pinned host allocation failed");
    h_rp = rm->row_ptr;
    h_col = rm->col;
    h_cnt = rm->cnt;
    h_llr = rm->llr;
  }
  // out_ptr is 0 up to row lo, so out_ptr[lo .. hi] are the row pointers of this rank's slice relative to its first row
  CK(cudaMemcpyAsync(h_rp, st->out_ptr + lo, sizeof(int64_t) * ((size_t)n_my + 1), cudaMemcpyDeviceToHost, cs));
  if (total > 0 && !(flags & CCO_FLAG_RESULT_ON_DEVICE)) {
    CK(cudaMemcpyAsync(h_col, st->p_col, sizeof(int32_t) * (size_t)total, cudaMemcpyDeviceToHost, cs));
    if (h_cnt) CK(cudaMemcpyAsync(h_cnt, st->p_cnt, sizeof(int32_t) * (size_t)total, cudaMemcpyDeviceToHost, cs));
    if (h_llr) CK(cudaMemcpyAsync(h_llr, st->p_llr, sizeof(double) * (size_t)total, cudaMemcpyDeviceToHost, cs));
  }
  return CCO_OK;
}

static int validate_host(int32_t n_mats, const cco_csr_t *mats, const cco_indicator_params_t *params) {
  if (n_mats < 1 || !mats || !params) return set_error(CCO_E_INVALID_ARG, "need at least the primary matrix and its params");
  for (int i = 0; i < n_mats; ++i) {
    const cco_csr_t &m = mats[i];
    if (!m.row_ptr) return set_error(CCO_E_INVALID_ARG, "matrix %d: null row_ptr", i);
    if (m.n_rows < 0 || m.n_rows >= 0x7fffffffLL) return set_error(CCO_E_INVALID_ARG, "matrix %d: n_rows out of range", i);
    if (m.n_cols < 0 || m.n_cols >= 0x7ffffffe) return set_error(CCO_E_INVALID_ARG, "matrix %d: n_cols out of range", i);
    if (m.n_rows != mats[0].n_rows)
      return set_error(CCO_E_SHAPE_MISMATCH, "matrix %d has %lld rows, the primary has %lld: all event types share the user dictionary",
                       i, (long long)m.n_rows, (long long)mats[0].n_rows);
    if (m.row_ptr[0] != 0) return set_error(CCO_E_INVALID_ARG, "matrix %d: row_ptr[0] != 0", i);
    long long nnz = m.row_ptr[m.n_rows];
    if (nnz < 0 || nnz >= 0xffffffffLL) return set_error(CCO_E_UNSUPPORTED, "matrix %d: nnz %lld outside [0, 2^32)", i, nnz);
    if (nnz > 0 && !m.col_idx) return set_error(CCO_E_INVALID_ARG, "matrix %d: null col_idx", i);
    if (params[i].max_interactions < 1) return set_error(CCO_E_INVALID_ARG, "matrix %d: max_interactions must be >= 1", i);
    if (params[i].top_k < 1) return set_error(CCO_E_INVALID_ARG, "matrix %d: top_k must be >= 1", i);
    if (params[i].top_k > CCO_MAX_TOP_K)
      return set_error(CCO_E_UNSUPPORTED, "matrix %d: top_k %d > CCO_MAX_TOP_K (%d)", i, params[i].top_k, CCO_MAX_TOP_K);
    if (params[i].has_min_llr && params[i].min_llr != params[i].min_llr)
      return set_error(CCO_E_INVALID_ARG, "matrix %d: min_llr is NaN", i);
  }
  return CCO_OK;
}

// the block of user rows rank r of a W-rank job works on
static inline void user_block(long long U, int W, int r, long long *lo, long long *hi) {
  const long long S = (U + W - 1) / W;
  *lo = std::min<long long>((long long)r * S, U);
  *hi = std::min<long long>(*lo + S, U);
}

static void dataset_release(cco_dataset *d) {
  if (!d) return;
  cudaSetDevice(d->ctx->device);
  for (auto p : d->rp_alloc)
    if (p) cudaFreeAsync(p, d->ctx->stream);
  for (auto p : d->col_alloc)
    if (p) cudaFreeAsync(p, d->ctx->stream);
  for (auto e : d->ready)
    if (e) cudaEventDestroy(e);
  for (auto &dc : d->dicts) {
    if (dc.offsets) d->ctx->pinned_put((void *)dc.offsets);
    if (dc.bytes) d->ctx->pinned_put((void *)dc.bytes);
  }
  delete d;
}

// the block of user rows of matrix i that the dataset holds
static DevRaw block_of(const cco_dataset *d, int i) {
  DevRaw r;
  r.n_rows = d->n_local;
  r.row_base = d->row_base;
  r.n_cols = (int32_t)d->n_cols[i];
  r.q_base = d->q_lo[i];
  r.nnz = d->q_hi[i] - d->q_lo[i];
  r.rp = d->rp[i];
  r.col = d->col[i];
  return r;
}

// device check of the uploaded block(s) + canonicalisation of unsorted / duplicated rows (synchronous).  In a multi-GPU
// job the "malformed" verdict is all-reduced so that every rank fails (or proceeds) together.
static int dataset_validate(cco_ctx *c, cco_dataset *d, bool canonicalise) {
  cudaStream_t s = c->stream;
  const int n_mats = d->n_mats;
  mail_reset(c);   // the canonicalisation reads its unique counts through the mailbox
  Arena ar(s);
  int *d_flags;
  CKR(ar.alloc(&d_flags, 2 * n_mats));
  CK(cudaMemsetAsync(d_flags, 0, sizeof(int) * 2 * n_mats, s));
  for (int i = 0; i < n_mats; ++i) {
    CK(cudaStreamWaitEvent(s, d->ready[i], 0));
    if (d->n_local == 0) continue;
    const DevRaw r = block_of(d, i);
    HeavyRows hv;
    CKR(list_heavy_rows(c, ar, r, &hv));
    launch_check(c, r, hv, d_flags + 2 * i);
  }
  if (c->world > 1)
    CKR(nccl_check(g_nccl.AllReduce(d_flags, d_flags, (size_t)(2 * n_mats), kNcclInt32, kNcclMax, c->comm, s), "ncclAllReduce(check flags)"));
  std::vector<int> h(2 * n_mats);
  CK(cudaMemcpyAsync(h.data(), d_flags, sizeof(int) * 2 * n_mats, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  for (int i = 0; i < n_mats; ++i)
    if (h[2 * i]) return set_error(CCO_E_INVALID_ARG, "matrix %d: row_ptr not monotone or column index out of [0, n_cols)", i);
  if (canonicalise)
    for (int i = 0; i < n_mats; ++i)
      if (h[2 * i + 1] && d->n_local > 0) {
        // (the flag is all-reduced: every rank canonicalises its own block, the blocks are independent)
        DevRaw r = block_of(d, i);
        CKR(canonicalize_device(c, ar, r));
        d->col[i] = r.col;
        d->q_lo[i] = 0;
        d->q_hi[i] = r.nnz;
        if (c->world == 1) d->nnz[i] = r.nnz;
      }
  CK(cudaStreamSynchronize(s));
  d->validated = canonicalise;
  return CCO_OK;
}

// host CSR -> device: this rank's block of user rows only (the dataset owns its buffers until cco_dataset_free)
static int dataset_upload(cco_ctx *c, int32_t n_mats, const cco_csr_t *mats, uint32_t flags, cco_dataset **out, bool async = false) {
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  cco_dataset *d = new cco_dataset();
  d->ctx = c;
  d->n_mats = n_mats;
  d->n_users = mats[0].n_rows;
  long long u_lo, u_hi;
  user_block(d->n_users, c->world, c->rank, &u_lo, &u_hi);
  d->row_base = u_lo;
  d->n_local = u_hi - u_lo;
  d->whole = c->world == 1;
  d->rp.assign(n_mats, nullptr);
  d->col.assign(n_mats, nullptr);
  d->rp_alloc.assign(n_mats, nullptr);
  d->col_alloc.assign(n_mats, nullptr);
  d->n_cols.assign(n_mats, 0);
  d->nnz.assign(n_mats, 0);
  d->q_lo.assign(n_mats, 0);
  d->q_hi.assign(n_mats, 0);
  d->ready.assign(n_mats, nullptr);
  struct G {
    cco_dataset *d;
    bool ok = false;
    ~G() {
      if (!ok) dataset_release(d);
    }
  } g{d};
  // allocations are ordered on the main stream; the copies run on the copy stream (H2D engine) so that the caller
  // of the async form can start preparing matrix i while matrix i+1 is still in flight
  cudaStream_t cs = c->copy_stream;
  for (int i = 0; i < n_mats; ++i) {
    const cco_csr_t &m = mats[i];
    d->n_cols[i] = m.n_cols;
    d->nnz[i] = m.row_ptr[m.n_rows];
    const long long q0 = m.row_ptr[u_lo], q1 = m.row_ptr[u_hi];
    d->q_lo[i] = q0;
    d->q_hi[i] = q1;
    void *p = nullptr;
    cudaError_t e = cudaMallocAsync(&p, sizeof(int64_t) * ((size_t)d->n_local + 1), s);
    if (e != cudaSuccess) return set_error(CCO_E_OOM, "cudaMallocAsync row_ptr: %s", cudaGetErrorString(e));
    d->rp_alloc[i] = p;
    d->rp[i] = (long long *)p;
    e = cudaMallocAsync(&p, sizeof(int32_t) * (size_t)std::max<long long>(q1 - q0, 4), s);
    if (e != cudaSuccess) return set_error(CCO_E_OOM, "cudaMallocAsync col_idx: %s", cudaGetErrorString(e));
    d->col_alloc[i] = p;
    d->col[i] = (int32_t *)p - q0;   // the block keeps the caller's absolute offsets: col[rp[r]] addresses its own storage
    CK(cudaEventCreateWithFlags(&d->ready[i], cudaEventDisableTiming));
  }
  CK(cudaEventRecord(c->copy_ev[0], s));
  CK(cudaStreamWaitEvent(cs, c->copy_ev[0], 0));
  CK(cudaEventRecord(c->ev[6], cs));
  for (int i = 0; i < n_mats; ++i) {
    const cco_csr_t &m = mats[i];
    const long long q0 = m.row_ptr[u_lo], q1 = m.row_ptr[u_hi];
    CK(cudaMemcpyAsync(d->rp_alloc[i], m.row_ptr + u_lo, sizeof(int64_t) * ((size_t)d->n_local + 1), cudaMemcpyHostToDevice, cs));
    if (q1 > q0)
      CK(cudaMemcpyAsync(d->col_alloc[i], m.col_idx + q0, sizeof(int32_t) * (size_t)(q1 - q0), cudaMemcpyHostToDevice, cs));
    CK(cudaEventRecord(d->ready[i], cs));
  }
  CK(cudaEventRecord(c->ev[7], cs));
  if (async && (flags & CCO_FLAG_ASSUME_CANONICAL)) {
    d->h2d_pending = true;   // the malformed-input check runs inside the train, next to the first pass over the data
    g.ok = true;
    *out = d;
    return CCO_OK;
  }
  CKR(dataset_validate(c, d, !(flags & CCO_FLAG_ASSUME_CANONICAL)));
  CK(cudaEventElapsedTime(&d->ms_h2d, c->ev[6], c->ev[7]));
  g.ok = true;
  *out = d;
  return CCO_OK;
}

// The train's preparation of the dataset's matrices on this rank: raw column counts and the malformed-input verdict,
// sampleDownAndBinarize, the transpose of A' and the largest marginals.  c->ev[1] and c->ev[2] bracket it on the stream,
// stage[k] ends cco_stats_t.ms_prep_stage[k].  It ends in the preparation's one host round trip: the packed-word check
// of the indicators needs the largest marginals.
struct Prepared {
  std::vector<DevMat> dm;          // the sampled matrices, all users
  uint32_t *at_ptr = nullptr;      // A'^T: [n_items_a + 1] offsets into at_users
  int32_t *at_users = nullptr;
  int32_t *raw_counts = nullptr;   // raw column counts, matrix i at the sum of the earlier matrices' n_cols
  std::vector<int32_t> max_marg;   // largest post-sample column count per matrix
  std::vector<uint32_t> nnz;       // entries per sampled matrix
  cudaEvent_t stage[7] = {};
};
static int prepare(cco_ctx *c, Arena &ar, const cco_dataset *ds, const cco_indicator_params_t *params, int32_t seed, uint32_t flags,
                   Prepared *p) {
  cudaStream_t s = c->stream;
  const int n_mats = ds->n_mats;
  const long long n_users = ds->n_users;
  std::vector<DevRaw> raw(n_mats);
  for (int i = 0; i < n_mats; ++i) raw[i] = block_of(ds, i);
  for (auto &e : p->stage) CKR(pooled_event(c, true, &e));
  auto mark = [&](int k) { return cudaEventRecord(p->stage[k], s); };
  CK(cudaEventRecord(c->ev[1], s));
  nvtx_push("cco:prepare");
  // raw column counts: this rank histograms its user block; ONE allreduce sums all matrices' counts
  long long total_cols = 0;
  std::vector<long long> col_off(n_mats + 1, 0);
  for (int i = 0; i < n_mats; ++i) {
    col_off[i] = total_cols;
    total_cols += raw[i].n_cols;
  }
  col_off[n_mats] = total_cols;
  const long long copy_stride = std::max<long long>(total_cols, 1);
  int32_t *marg_all;
  int *d_check;
  CKR(ar.alloc(&marg_all, (size_t)copy_stride));
  CKR(ar.alloc(&d_check, 2 * n_mats));
  CK(cudaMemsetAsync(marg_all, 0, sizeof(int32_t) * (size_t)copy_stride, s));
  CK(cudaMemsetAsync(d_check, 0, sizeof(int) * 2 * n_mats, s));
  CKR(count_raw_columns(c, ar, raw, col_off, ds->ready.data(), ds->validated ? nullptr : d_check, &p->raw_counts));
  CK(mark(0));
  if (c->world > 1) {
    if (total_cols > 0)
      CKR(nccl_check(g_nccl.AllReduce(p->raw_counts, p->raw_counts, (size_t)total_cols, kNcclInt32, kNcclSum, c->comm, s), "ncclAllReduce(raw counts)"));
    CKR(nccl_check(g_nccl.AllReduce(d_check, d_check, (size_t)(2 * n_mats), kNcclInt32, kNcclMax, c->comm, s), "ncclAllReduce(check flags)"));
  }
  CK(mark(1));
  // sampleDownAndBinarize every matrix
  std::vector<DevMat> &dm = p->dm;
  dm.assign(n_mats, DevMat());
  CKR(downsample_all(c, ar, raw, d_check, n_users, p->raw_counts, marg_all, col_off, params, seed, flags, dm, &p->stage[2]));
  // `drmA.t`
  const int32_t n_items_a = dm[0].n_cols;
  uint32_t *cursor;
  int32_t *d_max;
  CKR(ar.alloc(&p->at_ptr, n_items_a + 1));
  CKR(ar.alloc(&cursor, n_items_a + 1));
  CKR(ar.alloc(&d_max, n_mats));
  CKR(ar.alloc(&p->at_users, std::max<long long>(ds->nnz[0], 1)));
  CK(cudaMemsetAsync(d_max, 0, 4 * (size_t)n_mats, s));
  {
    uint32_t *marg_pad;
    CKR(ar.alloc(&marg_pad, n_items_a + 1));
    CK(cudaMemcpyAsync(marg_pad, dm[0].marg, sizeof(int32_t) * (size_t)n_items_a, cudaMemcpyDeviceToDevice, s));
    CK(cudaMemsetAsync(marg_pad + n_items_a, 0, 4, s));
    CKR(exclusive_sum(c, ar, marg_pad, p->at_ptr, (long long)n_items_a + 1));
    ar.release(marg_pad);
  }
  CK(cudaMemcpyAsync(cursor, p->at_ptr, sizeof(uint32_t) * ((size_t)n_items_a + 1), cudaMemcpyDeviceToDevice, s));
  k_transpose_entries<<<grid_for((ds->nnz[0] + kSampleChunk - 1) / kSampleChunk * 32, 256, c->sm_count), 256, 0, s>>>(n_users, dm[0].rp,
                                                                                                                     dm[0].col, cursor, p->at_users);
  c->launches++;
  for (int i = 0; i < n_mats; ++i)
    if (dm[i].n_cols > 0) {
      k_max_i32<<<grid_for(dm[i].n_cols, 256, c->sm_count, 2), 256, 0, s>>>(dm[i].n_cols, dm[i].marg, d_max + i);
      c->launches++;
    }
  p->max_marg.assign(n_mats, 0);
  p->nnz.assign(n_mats, 0);
  std::vector<int> h_check(2 * n_mats, 0);
  CKR(mail_fetch(c, p->max_marg.data(), d_max, 4 * (size_t)n_mats));
  CKR(mail_fetch(c, h_check.data(), d_check, sizeof(int) * 2 * (size_t)n_mats));
  for (int i = 0; i < n_mats; ++i) CKR(mail_fetch(c, &p->nnz[i], dm[i].rp + n_users, 4));
  CK(mark(6));
  CK(cudaEventRecord(c->ev[2], s));
  nvtx_pop();
  CKR(mail_wait(c));
  for (int i = 0; i < n_mats; ++i)
    if (h_check[2 * i]) return set_error(CCO_E_INVALID_ARG, "matrix %d: row_ptr not monotone or column index out of [0, n_cols)", i);
  return CCO_OK;
}

// The whole hot path on this rank, for the block of users the dataset holds.
static int train_dataset(cco_ctx *c, const cco_dataset *ds, const cco_indicator_params_t *params, int32_t seed, uint32_t flags,
                         cco_result **out) {
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  const int n_mats = ds->n_mats;
  mail_reset(c);
  c->ev_timing_used = c->ev_plain_used = 0;
  Arena ar(s, c);
  struct CopyJoin {  // destroyed before `ar`: no packed buffer is freed while the copy stream still reads it
    cco_ctx *c;
    ~CopyJoin() {
      cudaStreamSynchronize(c->copy_stream);
      cudaStreamSynchronize(c->sched_stream);   // error paths: no schedule kernel outlives the train's slab memory
    }
  } copy_join{c};
  cco_result *res = new cco_result();
  res->ctx = c;
  res->mats.resize(n_mats);
  memset(&res->stats, 0, sizeof res->stats);
  struct Guard {
    cco_result *r;
    bool ok = false;
    ~Guard() {
      if (!ok) cco_result_free(r);
    }
  } guard{res};
  std::vector<IndicatorState> ist(n_mats);
  for (auto &x : ist) CKR(pooled_event(c, false, &x.packed));
  cco_stats_t &st = res->stats;
  st.n_mats = n_mats;
  st.n_users = ds->n_users;
  st.ms_h2d = ds->ms_h2d;
  const bool h2d_pending = ds->h2d_pending;
  const long long n_users = ds->n_users;
  for (int i = 0; i < n_mats; ++i) st.nnz_in_total += ds->nnz[i];
  Prepared p;
  CKR(prepare(c, ar, ds, params, seed, flags, &p));
  for (int i = 0; i < n_mats && i < 16; ++i) st.nnz_downsampled[i] = p.nnz[i];

  // indicators, software-pipelined: indicator i+1 is on the stream before the host waits for indicator i's record
  const int32_t n_items_a = p.dm[0].n_cols;
  std::vector<IndicatorOut> io(n_mats);
  std::vector<cudaEvent_t> ev_rows(2 * n_mats, nullptr);
  for (auto &e : ev_rows) CKR(pooled_event(c, true, &e));
  for (int i = 0; i < n_mats; ++i) {
    nvtx_push("cco:indicator");
    CKR(enqueue_indicator(c, ar, p.at_ptr, p.at_users, n_items_a, p.dm[0].marg, p.max_marg[0], p.max_marg[i], p.dm[i], n_users, i == 0,
                          params[i], flags, false, c->ev[2], ev_rows[2 * i], ev_rows[2 * i + 1], &ist[i]));
    nvtx_pop();
    if (i > 0) CKR(finish_indicator(c, &ist[i - 1], flags, i - 1, &res->mats[i - 1], &io[i - 1]));
  }
  CKR(finish_indicator(c, &ist[n_mats - 1], flags, n_mats - 1, &res->mats[n_mats - 1], &io[n_mats - 1]));
  CK(cudaEventRecord(c->copy_ev[1], c->copy_stream));
  CK(cudaStreamWaitEvent(s, c->copy_ev[1], 0));
  CK(cudaEventRecord(c->ev[3], s));
  CK(cudaStreamSynchronize(s));
  CK(cudaStreamSynchronize(c->copy_stream));
  for (int i = 0; i < n_mats && i < 16; ++i) {
    st.products[i] = io[i].products;
    st.distinct_cells[i] = io[i].distinct;
    st.llr_evaluated[i] = io[i].evaluated;
    st.out_nnz[i] = io[i].nnz;
    CK(cudaEventElapsedTime(&st.ms_indicator[i], ev_rows[2 * i], ev_rows[2 * i + 1]));
  }
  if (h2d_pending) CK(cudaEventElapsedTime(&st.ms_h2d, c->ev[6], c->ev[7]));
  CK(cudaEventElapsedTime(&st.ms_prep_stage[0], c->ev[1], p.stage[0]));
  for (int k = 1; k <= 6; ++k) CK(cudaEventElapsedTime(&st.ms_prep_stage[k], p.stage[k - 1], p.stage[k]));
  CK(cudaEventElapsedTime(&st.ms_prepare, c->ev[1], c->ev[2]));
  CK(cudaEventElapsedTime(&st.ms_cooccurrence, c->ev[2], c->ev[3]));
  CK(cudaEventElapsedTime(&st.ms_total, c->ev[1], c->ev[3]));
  if (!h2d_pending) st.ms_total += st.ms_h2d;  // async upload overlaps the prepare stage: already inside the bracket
  st.n_kernel_launches = c->launches;
  guard.ok = true;
  *out = res;
  return CCO_OK;
}

static int train_impl(cco_ctx *c, int32_t n_mats, const cco_csr_t *mats, const cco_indicator_params_t *params, int32_t seed,
                      uint32_t flags, cco_result **out) {
  c->launches = 0;
  cco_dataset *ds = nullptr;
  CKR(dataset_upload(c, n_mats, mats, flags, &ds, /*async=*/true));
  int rc = train_dataset(c, ds, params, seed, flags, out);
  cudaStreamSynchronize(c->copy_stream);  // the caller's host buffers are free again when cco_train returns
  dataset_release(ds);
  return rc;
}

// cco_train on a group context: one host thread per GPU runs the per-rank train on its member context (same host
// matrices, each thread uploads its block of users); the slices meet in one merged result owned by the leader.
static int train_group(cco_ctx *leader, int32_t n_mats, const cco_csr_t *mats, const cco_indicator_params_t *params, int32_t seed,
                       uint32_t flags, cco_result **out) {
  const int W = (int)leader->members.size();
  GroupShared *gs = leader->members[0]->gshared;
  cco_result *merged = new cco_result();
  merged->ctx = leader;
  merged->mats.resize(n_mats);
  memset(&merged->stats, 0, sizeof merged->stats);
  gs->merged = merged;
  gs->totals.assign(W, 0);
  gs->status = CCO_OK;
  gs->err[0] = 0;
  std::vector<cco_result *> part(W, nullptr);
  std::vector<std::thread> th;
  for (int r = 0; r < W; ++r)
    th.emplace_back([&, r]() {
      int rc = train_impl(leader->members[r], n_mats, mats, params, seed, flags, &part[r]);
      if (rc != CCO_OK) {
        std::lock_guard<std::mutex> lk(gs->mu);
        if (gs->status == CCO_OK) {
          gs->status = rc;
          snprintf(gs->err, sizeof gs->err, "GPU %d: %s", leader->members[r]->device, cco_last_error());
        }
      }
    });
  for (auto &t : th) t.join();
  gs->merged = nullptr;
  if (gs->status != CCO_OK) {
    for (auto p : part)
      if (p) cco_result_free(p);
    cco_result_free(merged);
    return set_error(gs->status, "%s", gs->err);
  }
  cco_stats_t &st = merged->stats;
  st = part[0]->stats;
  for (int r = 1; r < W; ++r) {
    const cco_stats_t &p = part[r]->stats;
    for (int i = 0; i < 16; ++i) {
      st.products[i] += p.products[i];
      st.distinct_cells[i] += p.distinct_cells[i];
      st.out_nnz[i] += p.out_nnz[i];
      st.llr_evaluated[i] += p.llr_evaluated[i];
      st.ms_indicator[i] = std::max(st.ms_indicator[i], p.ms_indicator[i]);
    }
    st.ms_h2d = std::max(st.ms_h2d, p.ms_h2d);
    st.ms_prepare = std::max(st.ms_prepare, p.ms_prepare);
    st.ms_cooccurrence = std::max(st.ms_cooccurrence, p.ms_cooccurrence);
    st.ms_total = std::max(st.ms_total, p.ms_total);
    st.n_kernel_launches += p.n_kernel_launches;
  }
  for (auto p : part) cco_result_free(p);
  *out = merged;
  return CCO_OK;
}

}  // namespace cco

// ================================================================================================
// C ABI
// ================================================================================================
extern "C" {

int cco_abi_version(void) { return CCO_ABI_VERSION; }
const char *cco_last_error(void) { return g_err; }
const char *cco_status_string(int s) {
  switch (s) {
    case CCO_OK: return "ok";
    case CCO_E_INVALID_ARG: return "invalid argument";
    case CCO_E_CUDA: return "CUDA error";
    case CCO_E_NCCL: return "NCCL error";
    case CCO_E_OOM: return "out of memory";
    case CCO_E_SHAPE_MISMATCH: return "shape mismatch";
    case CCO_E_UNSUPPORTED: return "unsupported";
  }
  return "unknown";
}

int cco_device_count(void) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) return set_error(CCO_E_CUDA, "cudaGetDeviceCount: %s", cudaGetErrorString(e));
  int ok = 0;
  for (int i = 0; i < n; ++i) {
    cudaDeviceProp p;
    if (cudaGetDeviceProperties(&p, i) == cudaSuccess && p.major == 9 && p.minor == 0) ++ok;
  }
  return ok;
}

int cco_nccl_unique_id(unsigned char out[128]) {
  if (!out) return set_error(CCO_E_INVALID_ARG, "null output");
  CKR(load_nccl());
  ncclUniqueId id;
  int r = g_nccl.GetUniqueId(&id);
  if (r != 0) return set_error(CCO_E_NCCL, "ncclGetUniqueId: %s", g_nccl.GetErrorString(r));
  memcpy(out, id.internal, 128);
  return CCO_OK;
}

// streams, events, mailbox, memory pool of one per-GPU context (the NCCL communicator is attached by the caller)
static int ctx_init_device(cco_ctx *c) {
  CK(cudaSetDevice(c->device));
  CK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
  for (auto &ev : c->ev) CK(cudaEventCreate(&ev));
  for (auto &ev : c->tev) CK(cudaEventCreate(&ev));
  for (auto &ev : c->copy_ev) CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  for (auto &st : c->bin_stream) CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  // The schedule and column order of indicator i+1 are short dependent kernels on the path to its row kernels; at the
  // highest priority their CTAs are dispatched ahead of the queued CTAs of indicator i's row kernels.
  int lo_pri = 0, hi_pri = 0;
  CK(cudaDeviceGetStreamPriorityRange(&lo_pri, &hi_pri));
  CK(cudaStreamCreateWithPriority(&c->sched_stream, cudaStreamNonBlocking, hi_pri));
  for (auto &ev : c->bin_ev) CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  CK(cudaHostAlloc((void **)&c->mail_h, kMailBytes, cudaHostAllocMapped | cudaHostAllocPortable));
  CK(cudaHostGetDevicePointer((void **)&c->mail_d, c->mail_h, 0));
  cudaMemPool_t pool;
  CK(cudaDeviceGetDefaultMemPool(&pool, c->device));
  uint64_t thr = UINT64_MAX;  // keep freed blocks: steady-state trains allocate nothing
  CK(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
  return CCO_OK;
}

static int check_device(int device, cudaDeviceProp *p) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0)
    return set_error(CCO_E_CUDA, "no CUDA device (%s): this library has no CPU fallback",
                     e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
  if (device < 0 || device >= n) return set_error(CCO_E_INVALID_ARG, "device %d not in [0,%d)", device, n);
  CK(cudaGetDeviceProperties(p, device));
  if (p->major != 9 || p->minor != 0)   // sm_90a code runs on compute capability 9.0 only
    return set_error(CCO_E_CUDA, "device %d is sm_%d%d; this build contains sm_90a code only", device, p->major, p->minor);
  return CCO_OK;
}

static int create_failed(cco_ctx *c, int st) {
  char keep[sizeof g_err];
  memcpy(keep, g_err, sizeof keep);   // cco_destroy must not clobber the message
  cco_destroy(c);
  memcpy(g_err, keep, sizeof keep);
  return st;
}

int cco_create(const cco_config_t *cfg, cco_ctx_t **out) {
  if (!cfg || !out) return set_error(CCO_E_INVALID_ARG, "null argument");
  if (cfg->world_size < 1 || cfg->rank < 0 || cfg->rank >= cfg->world_size)
    return set_error(CCO_E_INVALID_ARG, "bad rank/world_size %d/%d", cfg->rank, cfg->world_size);
  if (cfg->world_size > 1023) return set_error(CCO_E_UNSUPPORTED, "world_size %d > 1023", cfg->world_size);
  cudaDeviceProp p;
  CKR(check_device(cfg->device, &p));
  if (cfg->world_size > 1 && !cfg->nccl_unique_id) return set_error(CCO_E_INVALID_ARG, "world_size > 1 needs nccl_unique_id");
  cco_ctx *c = new cco_ctx();
  c->device = cfg->device;
  c->rank = cfg->rank;
  c->world = cfg->world_size;
  c->sm_count = p.multiProcessorCount;
  c->smem_optin = p.sharedMemPerBlockOptin;
  // every failure below releases what was created so far (cco_destroy tolerates a half-built context)
  auto init = [&]() -> int {
    CKR(ctx_init_device(c));
    if (cfg->result_arena && cfg->result_arena_bytes > 0) {
      // caller-provided result memory (e.g. a shared-memory segment the reading process maps): page-lock it so the
      // device->host copies of the indicators land there directly
      CK(cudaHostRegister(cfg->result_arena, cfg->result_arena_bytes, cudaHostRegisterPortable));
      c->arena = (unsigned char *)cfg->result_arena;
      c->arena_bytes = cfg->result_arena_bytes;
      c->arena_registered = true;
    }
    if (c->world > 1) {
      CKR(load_nccl());
      ncclUniqueId id;
      memcpy(id.internal, cfg->nccl_unique_id, 128);
      int rc = g_nccl.CommInitRank(&c->comm, c->world, id, c->rank);
      if (rc != 0) return set_error(CCO_E_NCCL, "ncclCommInitRank: %s", g_nccl.GetErrorString(rc));
    }
    return CCO_OK;
  };
  const int st = init();
  if (st != CCO_OK) return create_failed(c, st);
  *out = c;
  return CCO_OK;
}

// One context over several GPUs of this process (what a single JVM thread can drive): member r runs on devices[r] with
// its own streams; the communicator comes from ncclCommInitAll; cco_train runs one host thread per member.
int cco_create_group(int32_t n_devices, const int32_t *devices, cco_ctx_t **out) {
  if (!devices || !out || n_devices < 1) return set_error(CCO_E_INVALID_ARG, "bad argument");
  if (n_devices > 1023) return set_error(CCO_E_UNSUPPORTED, "more than 1023 devices");
  std::vector<cudaDeviceProp> props(n_devices);
  for (int r = 0; r < n_devices; ++r) {
    CKR(check_device(devices[r], &props[r]));
    for (int q = 0; q < r; ++q)
      if (devices[q] == devices[r]) return set_error(CCO_E_INVALID_ARG, "device %d listed twice", devices[r]);
  }
  cco_ctx *leader = new cco_ctx();
  leader->device = devices[0];
  leader->world = 1;
  GroupShared *gs = new GroupShared();
  gs->world = n_devices;
  auto init = [&]() -> int {
    std::vector<ncclComm_t> comms(n_devices, nullptr);
    if (n_devices > 1) {
      CKR(load_nccl());
      std::vector<int> devs(devices, devices + n_devices);
      int rc = g_nccl.CommInitAll(comms.data(), n_devices, devs.data());
      if (rc != 0) return set_error(CCO_E_NCCL, "ncclCommInitAll: %s", g_nccl.GetErrorString(rc));
    }
    for (int r = 0; r < n_devices; ++r) {
      cco_ctx *m = new cco_ctx();
      m->device = devices[r];
      m->rank = r;
      m->world = n_devices;
      m->sm_count = props[r].multiProcessorCount;
      m->smem_optin = props[r].sharedMemPerBlockOptin;
      m->comm = comms[r];
      m->gshared = gs;
      leader->members.push_back(m);
      CKR(ctx_init_device(m));
    }
    CK(cudaSetDevice(devices[0]));
    return CCO_OK;
  };
  const int st = init();
  if (st != CCO_OK) {
    if (leader->members.empty()) delete gs;
    return create_failed(leader, st);
  }
  *out = leader;
  return CCO_OK;
}

int cco_destroy(cco_ctx_t *c) {
  if (!c) return CCO_OK;
  if (!c->members.empty()) {
    GroupShared *gs = c->members[0]->gshared;
    for (cco_ctx *m : c->members) {
      m->gshared = nullptr;
      cco_destroy(m);
    }
    c->members.clear();
    delete gs;
  }
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  if (c->copy_stream) cudaStreamSynchronize(c->copy_stream);
  if (c->comm) g_nccl.CommDestroy(c->comm);
  for (auto &b : c->pinned) cudaFreeHost(b.p);
  if (c->arena_registered) cudaHostUnregister(c->arena);
  if (c->mail_h) cudaFreeHost(c->mail_h);
  for (auto &ev : c->mail_ev) cudaEventDestroy(ev);
  for (auto &ev : c->ev_timing) cudaEventDestroy(ev);
  for (auto &ev : c->ev_plain) cudaEventDestroy(ev);
  for (auto &sl : c->slabs) cudaFree(sl.p);
  for (auto &ev : c->ev)
    if (ev) cudaEventDestroy(ev);
  for (auto &ev : c->tev)
    if (ev) cudaEventDestroy(ev);
  for (auto &ev : c->copy_ev)
    if (ev) cudaEventDestroy(ev);
  for (auto &st : c->bin_stream)
    if (st) cudaStreamDestroy(st);
  if (c->sched_stream) cudaStreamDestroy(c->sched_stream);
  for (auto &ev : c->bin_ev)
    if (ev) cudaEventDestroy(ev);
  if (c->stream) cudaStreamDestroy(c->stream);
  if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
  delete c;
  return CCO_OK;
}

int cco_host_alloc(cco_ctx_t *c, size_t bytes, void **out) {
  if (!c || !out) return set_error(CCO_E_INVALID_ARG, "null argument");
  CK(cudaSetDevice(c->device));
  void *p = c->pinned_get(bytes, /*for_result=*/false);
  if (!p) return set_error(CCO_E_OOM, "cudaHostAlloc(%zu) failed", bytes);
  *out = p;
  return CCO_OK;
}
int cco_host_free(cco_ctx_t *c, void *p) {
  if (!c) return set_error(CCO_E_INVALID_ARG, "null context");
  if (p) c->pinned_put(p);
  return CCO_OK;
}

int cco_train(cco_ctx_t *ctx, int32_t n_mats, const cco_csr_t *mats, const cco_indicator_params_t *params, int32_t seed,
              uint32_t flags, cco_result_t **out) {
  if (!ctx || !out) return set_error(CCO_E_INVALID_ARG, "null argument");
  *out = nullptr;
  CKR(validate_host(n_mats, mats, params));   // everything the host can check, before any GPU (or thread) starts
  if (!ctx->members.empty()) return train_group(ctx, n_mats, mats, params, seed, flags, out);
  return train_impl(ctx, n_mats, mats, params, seed, flags, out);
}

int cco_cooccurrences_idss(cco_ctx_t *ctx, int32_t n_mats, const cco_csr_t *mats, int32_t seed,
                           int32_t max_interesting_items_per_thing, int32_t max_num_interactions, uint32_t flags,
                           cco_result_t **out) {
  if (n_mats < 1) return set_error(CCO_E_INVALID_ARG, "need at least the primary matrix");
  std::vector<cco_indicator_params_t> p(n_mats);
  for (auto &q : p) {
    q.max_interactions = max_num_interactions;
    q.top_k = max_interesting_items_per_thing;
    q.has_min_llr = 0;
    q.min_llr = 0.0;
  }
  return cco_train(ctx, n_mats, mats, p.data(), seed, flags, out);
}

int cco_dataset_shape(const cco_dataset_t *ds, int32_t i, int64_t *n_rows, int32_t *n_cols, int64_t *nnz) {
  if (!ds || i < 0 || i >= ds->n_mats) return set_error(CCO_E_INVALID_ARG, "bad dataset/index");
  if (n_rows) *n_rows = ds->n_users;
  if (n_cols) *n_cols = (int32_t)ds->n_cols[i];
  if (nnz) *nnz = ds->nnz[i];
  return CCO_OK;
}

int cco_dataset_download(const cco_dataset_t *ds, int32_t i, int64_t **row_ptr, int32_t **col_idx) {
  if (!ds || !row_ptr || !col_idx || i < 0 || i >= ds->n_mats) return set_error(CCO_E_INVALID_ARG, "bad argument");
  if (!ds->whole) return set_error(CCO_E_UNSUPPORTED, "this dataset holds one rank's block of users only");
  cco_ctx *c = ds->ctx;
  CK(cudaSetDevice(c->device));
  int64_t *rp = (int64_t *)malloc(sizeof(int64_t) * ((size_t)ds->n_users + 1));
  int32_t *ci = (int32_t *)malloc(sizeof(int32_t) * (size_t)std::max<long long>(ds->nnz[i], 1));
  if (!rp || !ci) return set_error(CCO_E_OOM, "malloc failed");
  CK(cudaStreamSynchronize(c->copy_stream));
  CK(cudaMemcpyAsync(rp, ds->rp_alloc[i], sizeof(int64_t) * ((size_t)ds->n_users + 1), cudaMemcpyDeviceToHost, c->stream));
  if (ds->nnz[i] > 0)
    CK(cudaMemcpyAsync(ci, ds->col_alloc[i], sizeof(int32_t) * (size_t)ds->nnz[i], cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  *row_ptr = rp;
  *col_idx = ci;
  return CCO_OK;
}

// Preparator.prepare on the device (SURVEY.md 8f-1): histogram + scans for the dictionaries, one radix sort + unique
// per event type for the binary CSR.  The events of a type reach the device through `fill` (a host->device copy for
// cco_ingest, the generator kernel for cco_synth_ingest) right before the type is processed.
struct IngestSource {
  int n_types = 0;
  long long n_users_raw = 0;
  std::vector<long long> n_events;
  std::vector<int32_t> n_items_raw;
  bool keep_item_space = false;   // synthetic workloads: the item dictionary is the raw id space (identity map)
  // fill(t, d_user, d_item): enqueue on the context's stream whatever puts type t's raw events into the two arrays
  std::function<int(int, long long *, int32_t *)> fill;
};

// an empty device-built dataset of n_types matrices: canonical by construction, every rank holds the whole matrices
static cco_dataset *ingest_dataset_new(cco_ctx *c, int n_types) {
  cco_dataset *d = new cco_dataset();
  d->ctx = c;
  d->n_mats = n_types;
  d->rp.assign(n_types, nullptr);
  d->col.assign(n_types, nullptr);
  d->rp_alloc.assign(n_types, nullptr);
  d->col_alloc.assign(n_types, nullptr);
  d->q_lo.assign(n_types, 0);
  d->q_hi.assign(n_types, 0);
  d->n_cols.assign(n_types, 0);
  d->nnz.assign(n_types, 0);
  d->ready.assign(n_types, nullptr);
  d->validated = true;   // built here: canonical by construction
  d->whole = true;
  return d;
}

// binary CSR of matrix t (n_users rows) from the (user << 32 | item) keys of its ne events in k0 (dropped events carry ~0,
// `kept` do not): radix sort, unique, row_ptr.  k1 is scratch of ne keys.
static int ingest_csr(cco_ctx *c, Arena &ar, cco_dataset *d, int t, long long ne, uint32_t n_users, unsigned long long *k0,
                      unsigned long long *k1, unsigned long long kept) {
  cudaStream_t s = c->stream;
  void *p = nullptr;
  cudaError_t e = cudaMallocAsync(&p, sizeof(int64_t) * ((size_t)n_users + 1), s);
  if (e != cudaSuccess) return set_error(CCO_E_OOM, "cudaMallocAsync row_ptr: %s", cudaGetErrorString(e));
  d->rp[t] = (long long *)p;
  d->rp_alloc[t] = p;
  e = cudaMallocAsync(&p, sizeof(int32_t) * (size_t)std::max<unsigned long long>(kept, 4), s);
  if (e != cudaSuccess) return set_error(CCO_E_OOM, "cudaMallocAsync col_idx: %s", cudaGetErrorString(e));
  d->col[t] = (int32_t *)p;
  d->col_alloc[t] = p;
  CK(cudaEventCreateWithFlags(&d->ready[t], cudaEventDisableTiming));
  long long n_unique = 0;
  if (kept > 0)   // dropped events carry the key ~0 and sort to the end: all 64 bits take part
    CKR(keys_to_csr(c, ar, k0, k1, ne, 64, (long long)kept, n_users, d->col[t], d->rp[t], &n_unique));
  else
    CK(cudaMemsetAsync(d->rp[t], 0, sizeof(int64_t) * ((size_t)n_users + 1), s));
  d->nnz[t] = n_unique;
  CK(cudaEventRecord(d->ready[t], s));
  return CCO_OK;
}

// every rank of a multi-GPU job builds the whole matrices (the events are all here) and then works on its block of
// users like an uploaded dataset does; the block's entry offsets come from row_ptr
static int ingest_blocks(cco_ctx *c, cco_dataset *d, uint32_t n_users) {
  const int n_types = d->n_mats;
  long long u_lo, u_hi;
  user_block(n_users, c->world, c->rank, &u_lo, &u_hi);
  d->row_base = u_lo;
  d->n_local = u_hi - u_lo;
  for (int t = 0; t < n_types; ++t) {
    CKR(mail_fetch(c, &d->q_lo[t], d->rp[t] + u_lo, 8));
    CKR(mail_fetch(c, &d->q_hi[t], d->rp[t] + u_hi, 8));
  }
  CKR(mail_wait(c));
  for (int t = 0; t < n_types; ++t) d->rp[t] += u_lo;   // views of the block; rp_alloc / col_alloc keep the whole matrices
  return CCO_OK;
}

static int ingest_core(cco_ctx *c, const IngestSource &src, int32_t min_events_per_user, int32_t *user_map,
                       int32_t *const *item_maps, cco_dataset **out) {
  const int n_types = src.n_types;
  const long long n_users_raw = src.n_users_raw;
  *out = nullptr;
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  mail_reset(c);
  Arena ar(s);
  cco_dataset *d = ingest_dataset_new(c, n_types);
  struct G {
    cco_dataset *d;
    bool ok = false;
    ~G() {
      if (!ok) dataset_release(d);
    }
  } g{d};
  const long long nu = std::max<long long>(n_users_raw, 1);
  int32_t *cnt, *d_user_map;
  uint32_t *uflag, *upos;
  CKR(ar.alloc(&cnt, nu));
  CKR(ar.alloc(&uflag, nu + 1));
  CKR(ar.alloc(&upos, nu + 1));
  CKR(ar.alloc(&d_user_map, nu));
  uint32_t n_users = 0;
  for (int t = 0; t < n_types; ++t) {
    const long long ne = src.n_events[t], ni = std::max<int32_t>(src.n_items_raw[t], 1);
    long long *d_user;
    int32_t *d_item;
    CKR(ar.alloc(&d_user, std::max<long long>(ne, 1)));
    CKR(ar.alloc(&d_item, std::max<long long>(ne, 1)));
    if (ne > 0) CKR(src.fill(t, d_user, d_item));
    if (t == 0) {
      // user dictionary from the primary events (duplicates count: Preparator.scala:129-132)
      CK(cudaMemsetAsync(cnt, 0, sizeof(int32_t) * (size_t)nu, s));
      CK(cudaMemsetAsync(uflag, 0, sizeof(uint32_t) * ((size_t)nu + 1), s));
      if (ne > 0) k_ingest_count_users<<<grid_for(ne, 256, c->sm_count), 256, 0, s>>>(ne, d_user, cnt);
      const int32_t need = min_events_per_user > 1 ? min_events_per_user : 1;
      if (n_users_raw > 0)
        k_ingest_user_flags<<<grid_for(n_users_raw, 256, c->sm_count), 256, 0, s>>>(n_users_raw, cnt, need, uflag);
      CKR(exclusive_sum(c, ar, uflag, upos, nu + 1));
      if (n_users_raw > 0)
        k_ingest_make_map<<<grid_for(n_users_raw, 256, c->sm_count), 256, 0, s>>>(n_users_raw, uflag, upos, d_user_map);
      c->launches += 3;
      CKR(mail_fetch(c, &n_users, upos + n_users_raw, 4));
      if (n_users_raw > 0 && user_map)
        CK(cudaMemcpyAsync(user_map, d_user_map, sizeof(int32_t) * (size_t)n_users_raw, cudaMemcpyDeviceToHost, s));
      CKR(mail_wait(c));
      d->n_users = n_users;
    }
    uint32_t *iflag, *ipos;
    int32_t *d_item_map;
    CKR(ar.alloc(&iflag, ni + 1));
    CKR(ar.alloc(&ipos, ni + 1));
    CKR(ar.alloc(&d_item_map, ni));
    if (src.keep_item_space) {
      CK(cudaMemsetAsync(iflag + ni, 0, 4, s));
      k_fill_u32<<<grid_for(ni, 256, c->sm_count), 256, 0, s>>>(ni, 1u, iflag);
    } else {
      CK(cudaMemsetAsync(iflag, 0, sizeof(uint32_t) * ((size_t)ni + 1), s));
      if (ne > 0) k_ingest_item_flags<<<grid_for(ne, 256, c->sm_count), 256, 0, s>>>(ne, d_user, d_item, d_user_map, iflag);
    }
    CKR(exclusive_sum(c, ar, iflag, ipos, ni + 1));
    k_ingest_make_map<<<grid_for(ni, 256, c->sm_count), 256, 0, s>>>(src.n_items_raw[t], iflag, ipos, d_item_map);
    uint32_t n_items = 0;
    CKR(mail_fetch(c, &n_items, ipos + src.n_items_raw[t], 4));
    if (src.n_items_raw[t] > 0 && item_maps && item_maps[t])
      CK(cudaMemcpyAsync(item_maps[t], d_item_map, sizeof(int32_t) * (size_t)src.n_items_raw[t], cudaMemcpyDeviceToHost, s));
    // sort surviving (user, item) keys, drop duplicates, rebuild row_ptr
    unsigned long long *k0, *k1, *d_kept;
    CKR(ar.alloc(&k0, std::max<long long>(ne, 1)));
    CKR(ar.alloc(&k1, std::max<long long>(ne, 1)));
    CKR(ar.alloc(&d_kept, 1));
    CK(cudaMemsetAsync(d_kept, 0, 8, s));
    if (ne > 0) k_ingest_keys<<<grid_for(ne, 256, c->sm_count), 256, 0, s>>>(ne, d_user, d_item, d_user_map, d_item_map, k0, d_kept);
    c->launches += 3;
    unsigned long long kept = 0;
    CKR(mail_fetch(c, &kept, d_kept, 8));
    CKR(mail_wait(c));
    ar.release(d_user);   // the raw events are dead once the keys exist
    ar.release(d_item);
    d->n_cols[t] = n_items;
    CKR(ingest_csr(c, ar, d, t, ne, n_users, k0, k1, kept));
    ar.release(k0);
    ar.release(k1);
    ar.release(iflag);
    ar.release(ipos);
    ar.release(d_item_map);
  }
  CKR(ingest_blocks(c, d, n_users));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  g.ok = true;
  *out = d;
  return CCO_OK;
}

int cco_ingest(cco_ctx_t *c, int32_t n_types, const cco_events_t *ev, int64_t n_users_raw, int32_t min_events_per_user,
               int32_t *user_map, int32_t *const *item_maps, cco_dataset_t **out) {
  if (!c || !ev || !user_map || !item_maps || !out || n_types < 1) return set_error(CCO_E_INVALID_ARG, "bad argument");
  if (n_users_raw < 0 || n_users_raw >= 0x7fffffffLL) return set_error(CCO_E_INVALID_ARG, "n_users_raw out of range");
  IngestSource src;
  src.n_types = n_types;
  src.n_users_raw = n_users_raw;
  for (int t = 0; t < n_types; ++t) {
    if (ev[t].n_events < 0 || ev[t].n_events >= 0xffffffffLL || ev[t].n_items_raw < 0)
      return set_error(CCO_E_INVALID_ARG, "type %d: bad event count / item space", t);
    if (ev[t].n_events > 0 && (!ev[t].user || !ev[t].item)) return set_error(CCO_E_INVALID_ARG, "type %d: null event arrays", t);
    if (!item_maps[t] && ev[t].n_items_raw > 0) return set_error(CCO_E_INVALID_ARG, "type %d: null item_map", t);
    // ids are range-checked on the host: they index device arrays
    for (int64_t i = 0; i < ev[t].n_events; ++i)
      if (ev[t].user[i] < 0 || ev[t].user[i] >= n_users_raw || ev[t].item[i] < 0 || ev[t].item[i] >= ev[t].n_items_raw)
        return set_error(CCO_E_INVALID_ARG, "type %d: user or item id out of range at event %lld", t, (long long)i);
    src.n_events.push_back(ev[t].n_events);
    src.n_items_raw.push_back(ev[t].n_items_raw);
  }
  cudaStream_t s = c->stream;
  src.fill = [&](int t, long long *d_user, int32_t *d_item) -> int {
    CK(cudaMemcpyAsync(d_user, ev[t].user, sizeof(int64_t) * (size_t)ev[t].n_events, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_item, ev[t].item, sizeof(int32_t) * (size_t)ev[t].n_events, cudaMemcpyHostToDevice, s));
    return CCO_OK;
  };
  return ingest_core(c, src, min_events_per_user, user_map, item_maps, out);
}

// The synthetic workload of bench.py / the tests (SURVEY.md 8d spec; synth.py holds the numpy twin of the stream):
// event e of a type draws  h1 = mix64(mix64(seed) + (e + 1) * golden), h2 = mix64(h1 ^ 0x6a09e667f3bcc909);
// user = user_perm[upper_bound(user_cdf, u01(h1))], item = item_perm[upper_bound(item_cdf, u01(h2))]; the events are
// generated straight into HBM and go through the same ingest as cco_ingest.
int cco_synth_ingest(cco_ctx_t *c, int32_t n_types, const cco_synth_type_t *types, int64_t n_users_raw, const double *user_cdf,
                     const int32_t *user_perm, int32_t min_events_per_user, int32_t keep_item_space, cco_dataset_t **out) {
  if (!c || !types || !out || n_types < 1 || !user_cdf || !user_perm) return set_error(CCO_E_INVALID_ARG, "bad argument");
  if (n_users_raw < 1 || n_users_raw >= 0x7fffffffLL) return set_error(CCO_E_INVALID_ARG, "n_users_raw out of range");
  IngestSource src;
  src.n_types = n_types;
  src.n_users_raw = n_users_raw;
  src.keep_item_space = keep_item_space != 0;
  for (int t = 0; t < n_types; ++t) {
    if (types[t].n_events < 0 || types[t].n_events >= 0xffffffffLL || types[t].n_items < 1 || !types[t].item_cdf || !types[t].item_perm)
      return set_error(CCO_E_INVALID_ARG, "type %d: bad generator spec", t);
    src.n_events.push_back(types[t].n_events);
    src.n_items_raw.push_back(types[t].n_items);
  }
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  double *d_ucdf = nullptr, *d_icdf = nullptr;
  int32_t *d_uperm = nullptr, *d_iperm = nullptr;
  int32_t max_items = 1;
  for (int t = 0; t < n_types; ++t) max_items = std::max(max_items, types[t].n_items);
  auto drop = [&]() {
    for (void *p : {(void *)d_ucdf, (void *)d_icdf, (void *)d_uperm, (void *)d_iperm})
      if (p) cudaFreeAsync(p, s);
  };
  auto up = [&]() -> int {
    CK(cudaMallocAsync((void **)&d_ucdf, sizeof(double) * (size_t)n_users_raw, s));
    CK(cudaMallocAsync((void **)&d_uperm, sizeof(int32_t) * (size_t)n_users_raw, s));
    CK(cudaMallocAsync((void **)&d_icdf, sizeof(double) * (size_t)max_items, s));
    CK(cudaMallocAsync((void **)&d_iperm, sizeof(int32_t) * (size_t)max_items, s));
    CK(cudaMemcpyAsync(d_ucdf, user_cdf, sizeof(double) * (size_t)n_users_raw, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_uperm, user_perm, sizeof(int32_t) * (size_t)n_users_raw, cudaMemcpyHostToDevice, s));
    return CCO_OK;
  };
  int rc = up();
  if (rc != CCO_OK) { drop(); return rc; }
  src.fill = [&](int t, long long *d_user, int32_t *d_item) -> int {
    CK(cudaMemcpyAsync(d_icdf, types[t].item_cdf, sizeof(double) * (size_t)types[t].n_items, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_iperm, types[t].item_perm, sizeof(int32_t) * (size_t)types[t].n_items, cudaMemcpyHostToDevice, s));
    k_synth_events<<<grid_for(types[t].n_events, 256, c->sm_count), 256, 0, s>>>(types[t].n_events, types[t].seed, d_ucdf, d_uperm,
                                                                                (int32_t)n_users_raw, d_icdf, d_iperm, types[t].n_items,
                                                                                d_user, d_item);
    c->launches++;
    CK(cudaGetLastError());
    return CCO_OK;
  };
  rc = ingest_core(c, src, min_events_per_user, nullptr, nullptr, out);
  drop();
  return rc;
}

// ---- SURVEY.md 8f-1 on string ids: cco_ingest_strings (kernels in cco_strings.cuh) ------------------------------------
namespace cco {
// one column of string ids in HBM
struct DevStrCol {
  long long n = 0, base = 0;   // base = the caller's offsets[0]: byte offsets index the uploaded buffer as off[i] - base
  long long *off = nullptr;    // [n + 1], the caller's values
  uint64_t *w = nullptr;       // bytes [off[0], off[n]) as 8-byte words, 16 bytes of padding
  uint64_t *hash = nullptr;    // [n]
};
// the host-side checks of a column (the device checks that no offset decreases before any kernel reads bytes through them)
static int str_check_host(long long n, const int64_t *off, const char *bytes, int t, const char *what) {
  if (n < 0) return set_error(CCO_E_INVALID_ARG, "type %d: negative event count", t);
  if (n >= 0x7fffffffLL) return set_error(CCO_E_UNSUPPORTED, "type %d: %lld events, string ingest takes < 2^31 per type", t, n);
  if (n == 0) return CCO_OK;
  if (!off) return set_error(CCO_E_INVALID_ARG, "type %d: null %s offsets", t, what);
  if (off[0] < 0) return set_error(CCO_E_INVALID_ARG, "type %d: %s offsets[0] = %lld is negative", t, what, (long long)off[0]);
  if (off[0] > off[n])
    return set_error(CCO_E_INVALID_ARG, "type %d: %s offsets[0] = %lld > offsets[n] = %lld", t, what, (long long)off[0], (long long)off[n]);
  if (off[n] > off[0] && !bytes) return set_error(CCO_E_INVALID_ARG, "type %d: null %s bytes", t, what);
  return CCO_OK;
}
static int str_upload(cco_ctx *c, Arena &ar, long long n, const int64_t *off, const char *bytes, DevStrCol *col) {
  cudaStream_t s = c->stream;
  col->n = n;
  col->base = n > 0 ? off[0] : 0;
  const long long nb = n > 0 ? off[n] - off[0] : 0;
  CKR(ar.alloc(&col->off, n + 1));
  CKR(ar.alloc(&col->w, (nb + 16 + 7) / 8));
  CKR(ar.alloc(&col->hash, std::max<long long>(n, 1)));
  if (n > 0) {
    CK(cudaMemcpyAsync(col->off, off, sizeof(int64_t) * ((size_t)n + 1), cudaMemcpyHostToDevice, s));
    if (nb > 0) CK(cudaMemcpyAsync(col->w, bytes + off[0], (size_t)nb, cudaMemcpyHostToDevice, s));
  }
  return CCO_OK;
}
static void str_release(Arena &ar, DevStrCol &col) {
  ar.release(col.off);
  ar.release(col.w);
  ar.release(col.hash);
}
// launch the decreasing-offset check of a column into *bad
static void str_check_device(cco_ctx *c, const DevStrCol &col, int *bad) {
  if (col.n == 0) return;
  k_str_check<<<grid_for(col.n, 256, c->sm_count), 256, 0, c->stream>>>(col.n, col.off, bad);
  c->launches++;
}
static void str_hash(cco_ctx *c, const DevStrCol &col, uint64_t mask) {
  if (col.n == 0) return;
  k_str_hash<<<grid_for(col.n, 256, c->sm_count), 256, 0, c->stream>>>(col.n, col.off, col.base, col.w, mask, col.hash);
  c->launches++;
}

// the string table of one column and the dictionary it defines
struct StrTable {
  long long cap = 0;                // power of two, > 1.5 x the ids inserted
  uint32_t *table = nullptr;        // [cap]: index of the id that claimed the slot, kStrEmpty
  uint32_t *slot_of = nullptr;      // [n]: slot of each id, kStrEmpty for gated ids
  uint32_t *first = nullptr;        // [cap]: first index of the slot's string
  uint32_t *count = nullptr;        // [cap]: ids of the slot (primary user column only)
  int32_t *rank_of_slot = nullptr;  // [cap]: dictionary id, -1
  uint32_t *first_sorted = nullptr; // [n_groups]: first index of each dictionary entry, in dictionary order
  long long n_groups = 0;
};
static void str_table_release(Arena &ar, StrTable &tb) {
  for (void *p : {(void *)tb.table, (void *)tb.slot_of, (void *)tb.first, (void *)tb.count, (void *)tb.rank_of_slot, (void *)tb.first_sorted})
    if (p) ar.release(p);
  tb = StrTable();
}
// Group the ids of a column by string (exact: hash, then bytes), keep the groups with >= need ids (counting) or all of them,
// number them by first appearance, and write each id's dictionary id (-1: gated or filtered out).  gate[i] < 0 keeps id i
// out of the table, so `first` is the first appearance among the ids that pass the gate.
static int str_group(cco_ctx *c, Arena &ar, const DevStrCol &col, const int32_t *gate, bool counting, uint32_t need, StrTable *tb,
                     int32_t *id) {
  cudaStream_t s = c->stream;
  const long long n = col.n;
  long long cap = 64;
  while (cap < n + n / 2 + 1) cap <<= 1;
  tb->cap = cap;
  CKR(ar.alloc(&tb->table, cap));
  CKR(ar.alloc(&tb->slot_of, std::max<long long>(n, 1)));
  CKR(ar.alloc(&tb->first, cap));
  CKR(ar.alloc(&tb->rank_of_slot, cap));
  CK(cudaMemsetAsync(tb->table, 0xff, sizeof(uint32_t) * (size_t)cap, s));
  CK(cudaMemsetAsync(tb->first, 0xff, sizeof(uint32_t) * (size_t)cap, s));
  CK(cudaMemsetAsync(tb->rank_of_slot, 0xff, sizeof(int32_t) * (size_t)cap, s));
  if (counting) {
    CKR(ar.alloc(&tb->count, cap));
    CK(cudaMemsetAsync(tb->count, 0, sizeof(uint32_t) * (size_t)cap, s));
  }
  if (n > 0) {
    k_str_insert<<<grid_for(n, 256, c->sm_count), 256, 0, s>>>(n, col.off, col.base, col.w, col.hash, gate, (uint64_t)cap - 1, tb->table,
                                                              tb->slot_of, tb->first, tb->count);
    c->launches++;
  }
  uint32_t *flag, *pos;
  CKR(ar.alloc(&flag, cap + 1));
  CKR(ar.alloc(&pos, cap + 1));
  CK(cudaMemsetAsync(flag + cap, 0, 4, s));
  k_str_flags<<<grid_for(cap, 256, c->sm_count), 256, 0, s>>>(cap, tb->table, tb->count, need, flag);
  CKR(exclusive_sum(c, ar, flag, pos, cap + 1));
  uint32_t ng = 0;
  CKR(mail_fetch(c, &ng, pos + cap, 4));
  CKR(mail_wait(c));
  tb->n_groups = ng;
  CKR(ar.alloc(&tb->first_sorted, std::max<long long>(ng, 1)));
  if (ng > 0) {
    uint32_t *k0, *v0, *v1;
    CKR(ar.alloc(&k0, ng));
    CKR(ar.alloc(&v0, ng));
    CKR(ar.alloc(&v1, ng));
    k_str_compact<<<grid_for(cap, 256, c->sm_count), 256, 0, s>>>(cap, flag, pos, tb->first, k0, v0);
    // first indices are distinct: the sort by them is the dictionary order
    int bits = 1;
    while ((1LL << bits) < n) ++bits;
    cub::DoubleBuffer<uint32_t> kb(k0, tb->first_sorted), vb(v0, v1);
    size_t tbytes = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, tbytes, kb, vb, (long long)ng, 0, bits, s));
    void *tmp;
    CKR(ar.alloc((char **)&tmp, tbytes));
    CK(cub::DeviceRadixSort::SortPairs(tmp, tbytes, kb, vb, (long long)ng, 0, bits, s));
    ar.release(tmp);
    if (kb.Current() != tb->first_sorted)
      CK(cudaMemcpyAsync(tb->first_sorted, kb.Current(), sizeof(uint32_t) * ng, cudaMemcpyDeviceToDevice, s));
    k_str_rank<<<grid_for(ng, 256, c->sm_count), 256, 0, s>>>(ng, vb.Current(), tb->rank_of_slot);
    c->launches += 3;
    ar.release(k0);
    ar.release(v0);
    ar.release(v1);
  }
  if (n > 0) {
    k_str_ids<<<grid_for(n, 256, c->sm_count), 256, 0, s>>>(n, tb->slot_of, tb->rank_of_slot, id);
    c->launches++;
  }
  ar.release(flag);
  ar.release(pos);
  return CCO_OK;
}
// the dictionary of a grouped column as offsets + bytes in pinned host memory of the context (copies enqueued on the stream)
static int str_dictionary(cco_ctx *c, Arena &ar, const DevStrCol &col, const StrTable &tb, cco_dictionary_t *out) {
  cudaStream_t s = c->stream;
  const long long ng = tb.n_groups;
  long long *len, *off;
  CKR(ar.alloc(&len, ng + 1));
  CKR(ar.alloc(&off, ng + 1));
  CK(cudaMemsetAsync(len + ng, 0, 8, s));
  if (ng > 0) {
    k_str_dict_len<<<grid_for(ng, 256, c->sm_count), 256, 0, s>>>(ng, tb.first_sorted, col.off, len);
    c->launches++;
  }
  CKR(exclusive_sum(c, ar, len, off, ng + 1));
  long long total = 0;
  CKR(mail_fetch(c, &total, off + ng, 8));
  CKR(mail_wait(c));
  unsigned char *bytes;
  CKR(ar.alloc(&bytes, std::max<long long>(total, 1)));
  if (ng > 0 && total > 0) {
    k_str_dict_gather<<<grid_for(ng, 256, c->sm_count), 256, 0, s>>>(ng, tb.first_sorted, col.off, col.base,
                                                                    (const unsigned char *)col.w, off, bytes);
    c->launches++;
  }
  out->n = ng;
  out->offsets = (const int64_t *)c->pinned_get(sizeof(int64_t) * ((size_t)ng + 1), /*for_result=*/false);
  if (!out->offsets) return set_error(CCO_E_OOM, "pinned host allocation failed");
  out->bytes = (const char *)c->pinned_get((size_t)std::max<long long>(total, 1), /*for_result=*/false);
  if (!out->bytes) return set_error(CCO_E_OOM, "pinned host allocation failed");
  CK(cudaMemcpyAsync((void *)out->offsets, off, sizeof(int64_t) * ((size_t)ng + 1), cudaMemcpyDeviceToHost, s));
  if (total > 0) CK(cudaMemcpyAsync((void *)out->bytes, bytes, (size_t)total, cudaMemcpyDeviceToHost, s));
  ar.release(len);
  ar.release(off);
  ar.release(bytes);   // stream-ordered: freed after the copy
  return CCO_OK;
}

// type t of the dataset from each event's user and item dictionary ids (-1: dropped): the (user, item) keys, then the
// CSR; uid and iid are released
static int ingest_ids_csr(cco_ctx *c, Arena &ar, cco_dataset *d, int t, long long ne, uint32_t n_users, int32_t *uid, int32_t *iid) {
  cudaStream_t s = c->stream;
  unsigned long long *k0, *k1, *d_kept;
  CKR(ar.alloc(&k0, std::max<long long>(ne, 1)));
  CKR(ar.alloc(&k1, std::max<long long>(ne, 1)));
  CKR(ar.alloc(&d_kept, 1));
  CK(cudaMemsetAsync(d_kept, 0, 8, s));
  if (ne > 0) {
    k_str_keys<<<grid_for(ne, 256, c->sm_count), 256, 0, s>>>(ne, uid, iid, k0, d_kept);
    c->launches++;
  }
  unsigned long long kept = 0;
  CKR(mail_fetch(c, &kept, d_kept, 8));
  CKR(mail_wait(c));
  ar.release(uid);
  ar.release(iid);
  CKR(ingest_csr(c, ar, d, t, ne, n_users, k0, k1, kept));
  ar.release(k0);
  ar.release(k1);
  return CCO_OK;
}

// the user and item columns of type t in HBM: uploaded from the caller's arrays, or views of an event log's columns
using StrColumns = std::function<int(Arena &, int, DevStrCol *, DevStrCol *)>;

static int ingest_strings_core(cco_ctx *c, int32_t n_types, const StrColumns &columns, int32_t min_events_per_user, cco_dataset **out) {
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  NvtxRange nvtx("cco:ingest_strings");
  mail_reset(c);
  Arena ar(s);
  cco_dataset *d = ingest_dataset_new(c, n_types);
  d->dicts.assign((size_t)n_types + 1, cco_dictionary_t{0, nullptr, nullptr});
  struct G {
    cco_dataset *d;
    bool ok = false;
    ~G() {
      if (!ok) {
        cudaStreamSynchronize(d->ctx->stream);   // no dictionary copy still writes the pinned buffers released here
        dataset_release(d);
      }
    }
  } g{d};
  const uint32_t need = min_events_per_user > 1 ? (uint32_t)min_events_per_user : 1u;
  DevStrCol pu;   // the primary user column and its table stay resident: later types look their users up there
  StrTable ut;
  uint32_t n_users = 0;
  for (int t = 0; t < n_types; ++t) {
    DevStrCol uc, ic;
    CKR(columns(ar, t, &uc, &ic));
    const long long ne = uc.n;
    str_hash(c, uc, ~0ULL);
    str_hash(c, ic, ~0ULL);
    int32_t *uid, *iid;
    CKR(ar.alloc(&uid, std::max<long long>(ne, 1)));
    CKR(ar.alloc(&iid, std::max<long long>(ne, 1)));
    if (t == 0) {
      // user dictionary: primary users with >= need events (duplicates count, Preparator.scala:129-132), first appearance order
      CKR(str_group(c, ar, uc, nullptr, true, need, &ut, uid));
      if (ut.n_groups >= 0x7fffffffLL) return set_error(CCO_E_UNSUPPORTED, "%lld users: the user space must stay < 2^31 - 1", ut.n_groups);
      n_users = (uint32_t)ut.n_groups;
      d->n_users = n_users;
      CKR(str_dictionary(c, ar, uc, ut, &d->dicts[0]));
      pu = uc;
    } else if (ne > 0) {
      // secondary events of users outside the dictionary are dropped (Preparator.scala:175-178)
      k_str_lookup<<<grid_for(ne, 256, c->sm_count), 256, 0, s>>>(ne, uc.off, uc.base, uc.w, uc.hash, pu.off, pu.base, pu.w, pu.hash,
                                                                   (uint64_t)ut.cap - 1, ut.table, ut.rank_of_slot, uid);
      c->launches++;
    }
    // item dictionary of type t: items with a surviving event, ordered by first surviving appearance
    StrTable it;
    CKR(str_group(c, ar, ic, uid, false, 0, &it, iid));
    if (it.n_groups >= 0x7ffffffeLL) return set_error(CCO_E_UNSUPPORTED, "type %d: %lld items, at most 2^31 - 2", t, it.n_groups);
    d->n_cols[t] = it.n_groups;
    CKR(str_dictionary(c, ar, ic, it, &d->dicts[1 + t]));
    str_table_release(ar, it);
    if (t > 0) str_release(ar, uc);
    str_release(ar, ic);
    CKR(ingest_ids_csr(c, ar, d, t, ne, n_users, uid, iid));
  }
  CKR(ingest_blocks(c, d, n_users));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  g.ok = true;
  *out = d;
  return CCO_OK;
}
}  // namespace cco

int cco_ingest_strings(cco_ctx_t *c, int32_t n_types, const cco_string_events_t *ev, int32_t min_events_per_user, cco_dataset_t **out) {
  if (!c || !ev || !out || n_types < 1) return set_error(CCO_E_INVALID_ARG, "bad argument");
  *out = nullptr;
  if (!c->members.empty()) return set_error(CCO_E_UNSUPPORTED, "resident datasets are per GPU: ingest on a per-GPU context");
  for (int t = 0; t < n_types; ++t) {
    CKR(str_check_host(ev[t].n_events, ev[t].user_offsets, ev[t].user_bytes, t, "user"));
    CKR(str_check_host(ev[t].n_events, ev[t].item_offsets, ev[t].item_bytes, t, "item"));
  }
  const StrColumns upload = [c, ev](Arena &ar, int t, DevStrCol *uc, DevStrCol *ic) -> int {
    const long long ne = ev[t].n_events;
    CKR(str_upload(c, ar, ne, ev[t].user_offsets, ev[t].user_bytes, uc));
    CKR(str_upload(c, ar, ne, ev[t].item_offsets, ev[t].item_bytes, ic));
    int *bad;
    CKR(ar.alloc(&bad, 1));
    CK(cudaMemsetAsync(bad, 0, sizeof(int), c->stream));
    str_check_device(c, *uc, bad);
    str_check_device(c, *ic, bad);
    int h_bad = 0;
    CKR(mail_fetch(c, &h_bad, bad, 4));
    CKR(mail_wait(c));
    if (h_bad) return set_error(CCO_E_INVALID_ARG, "type %d: offsets decrease", t);
    return CCO_OK;
  };
  return ingest_strings_core(c, n_types, upload, min_events_per_user, out);
}

int cco_dataset_dictionary(const cco_dataset_t *ds, int32_t which, cco_dictionary_t *out) {
  if (!ds || !out) return set_error(CCO_E_INVALID_ARG, "null argument");
  if (ds->dicts.empty()) return set_error(CCO_E_INVALID_ARG, "this dataset was not built from strings (cco_ingest_strings)");
  if (which < -1 || which >= ds->n_mats) return set_error(CCO_E_INVALID_ARG, "dictionary %d not in [-1, %d)", which, ds->n_mats);
  *out = ds->dicts[(size_t)which + 1];
  return CCO_OK;
}

int cco_debug_string_ids(cco_ctx_t *c, int64_t n, const int64_t *offsets, const char *bytes, int32_t hash_bits, int32_t *ids) {
  if (!c || (n > 0 && !ids)) return set_error(CCO_E_INVALID_ARG, "bad argument");
  if (hash_bits < 0 || hash_bits > 64) return set_error(CCO_E_INVALID_ARG, "hash_bits %d not in [0, 64]", hash_bits);
  if (!c->members.empty()) return set_error(CCO_E_UNSUPPORTED, "per-GPU contexts only");
  CKR(str_check_host(n, offsets, bytes, 0, "id"));
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  mail_reset(c);
  Arena ar(s);
  DevStrCol col;
  CKR(str_upload(c, ar, n, offsets, bytes, &col));
  int *bad;
  CKR(ar.alloc(&bad, 1));
  CK(cudaMemsetAsync(bad, 0, sizeof(int), s));
  str_check_device(c, col, bad);
  int h_bad = 0;
  CKR(mail_fetch(c, &h_bad, bad, 4));
  CKR(mail_wait(c));
  if (h_bad) return set_error(CCO_E_INVALID_ARG, "offsets decrease");
  str_hash(c, col, hash_bits == 64 ? ~0ULL : (1ULL << hash_bits) - 1);
  int32_t *d_ids;
  CKR(ar.alloc(&d_ids, std::max<long long>(n, 1)));
  StrTable tb;
  CKR(str_group(c, ar, col, nullptr, false, 0, &tb, d_ids));
  if (n > 0) CK(cudaMemcpyAsync(ids, d_ids, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  return CCO_OK;
}

// copy matrix i of a resident dataset into caller-provided host arrays (pinned ones from cco_host_alloc copy at PCIe speed)
int cco_dataset_copy_to_host(const cco_dataset_t *ds, int32_t i, int64_t *row_ptr, int32_t *col_idx) {
  if (!ds || !row_ptr || i < 0 || i >= ds->n_mats) return set_error(CCO_E_INVALID_ARG, "bad argument");
  if (ds->nnz[i] > 0 && !col_idx) return set_error(CCO_E_INVALID_ARG, "null col_idx");
  if (!ds->whole) return set_error(CCO_E_UNSUPPORTED, "this dataset holds one rank's block of users only");
  cco_ctx *c = ds->ctx;
  CK(cudaSetDevice(c->device));
  CK(cudaStreamSynchronize(c->copy_stream));
  CK(cudaMemcpyAsync(row_ptr, ds->rp_alloc[i], sizeof(int64_t) * ((size_t)ds->n_users + 1), cudaMemcpyDeviceToHost, c->stream));
  if (ds->nnz[i] > 0)
    CK(cudaMemcpyAsync(col_idx, ds->col_alloc[i], sizeof(int32_t) * (size_t)ds->nnz[i], cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return CCO_OK;
}

int cco_partition_rows(const int64_t *work_prefix, int32_t n_items, int32_t world_size, int32_t *bounds) {
  if (!work_prefix || !bounds || n_items < 0 || world_size < 1) return set_error(CCO_E_INVALID_ARG, "bad argument");
  // weight of row i = its products + 1 (so rows without work are spread too); contiguous ranges of equal weight
  const long long total = (long long)work_prefix[n_items] + n_items;
  for (int r = 0; r <= world_size; ++r) {
    if (r == 0) { bounds[r] = 0; continue; }
    if (r == world_size) { bounds[r] = n_items; continue; }
    const long long target = (long long)((__int128)total * r / world_size);
    int lo = 0, hi = n_items;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if ((long long)work_prefix[mid] + mid < target) lo = mid + 1; else hi = mid;
    }
    bounds[r] = lo;
  }
  return CCO_OK;
}

int cco_dataset_upload(cco_ctx_t *ctx, int32_t n_mats, const cco_csr_t *mats, uint32_t flags, cco_dataset_t **out) {
  if (!ctx || !out) return set_error(CCO_E_INVALID_ARG, "null argument");
  if (!ctx->members.empty()) return set_error(CCO_E_UNSUPPORTED, "resident datasets are per GPU: use cco_train on a group context");
  *out = nullptr;
  std::vector<cco_indicator_params_t> p(std::max(n_mats, 1), cco_indicator_params_t{1, 1, 0, 0.0});
  CKR(validate_host(n_mats, mats, p.data()));
  return dataset_upload(ctx, n_mats, mats, flags, out);
}
int cco_dataset_free(cco_dataset_t *ds) {
  dataset_release(ds);
  return CCO_OK;
}
int cco_train_dataset(cco_ctx_t *ctx, const cco_dataset_t *ds, const cco_indicator_params_t *params, int32_t seed,
                      uint32_t flags, cco_result_t **out) {
  if (!ctx || !ds || !params || !out) return set_error(CCO_E_INVALID_ARG, "null argument");
  if (ds->ctx != ctx) return set_error(CCO_E_INVALID_ARG, "dataset belongs to another context");
  *out = nullptr;
  for (int i = 0; i < ds->n_mats; ++i) {
    if (params[i].max_interactions < 1) return set_error(CCO_E_INVALID_ARG, "matrix %d: max_interactions must be >= 1", i);
    if (params[i].top_k < 1) return set_error(CCO_E_INVALID_ARG, "matrix %d: top_k must be >= 1", i);
    if (params[i].top_k > CCO_MAX_TOP_K)
      return set_error(CCO_E_UNSUPPORTED, "matrix %d: top_k %d > CCO_MAX_TOP_K (%d)", i, params[i].top_k, CCO_MAX_TOP_K);
  }
  ctx->launches = 0;
  return train_dataset(ctx, ds, params, seed, flags, out);
}
int cco_timer_start(cco_ctx_t *ctx) {
  if (!ctx) return set_error(CCO_E_INVALID_ARG, "null context");
  CK(cudaSetDevice(ctx->device));
  CK(cudaEventRecord(ctx->tev[0], ctx->stream));
  return CCO_OK;
}
int cco_timer_stop(cco_ctx_t *ctx, float *ms) {
  if (!ctx || !ms) return set_error(CCO_E_INVALID_ARG, "null argument");
  CK(cudaSetDevice(ctx->device));
  CK(cudaEventRecord(ctx->tev[1], ctx->stream));
  CK(cudaEventSynchronize(ctx->tev[1]));
  CK(cudaEventElapsedTime(ms, ctx->tev[0], ctx->tev[1]));
  return CCO_OK;
}

int cco_result_num_matrices(const cco_result_t *r) { return r ? (int)r->mats.size() : set_error(CCO_E_INVALID_ARG, "null result"); }

int cco_result_row_range(const cco_result_t *r, int32_t i, int64_t *row_begin, int64_t *row_end) {
  if (!r || i < 0 || i >= (int)r->mats.size()) return set_error(CCO_E_INVALID_ARG, "bad result/index");
  if (row_begin) *row_begin = r->mats[i].row_begin;
  if (row_end) *row_end = r->mats[i].row_end;
  return CCO_OK;
}

int cco_result_key_ranges(const cco_result_t *r, int32_t i, int32_t *n_ranges) {
  if (!r || i < 0 || i >= (int)r->mats.size() || !n_ranges) return set_error(CCO_E_INVALID_ARG, "bad result/index");
  *n_ranges = r->mats[i].key_ranges;
  return CCO_OK;
}

int cco_result_matrix(const cco_result_t *r, int32_t i, int64_t *n_rows, int32_t *n_cols, const int64_t **row_ptr,
                      const int32_t **col_idx, const double **llr, const int32_t **count) {
  if (!r || i < 0 || i >= (int)r->mats.size()) return set_error(CCO_E_INVALID_ARG, "bad result/index");
  const ResultMat &m = r->mats[i];
  if (n_rows) *n_rows = m.row_end - m.row_begin;
  if (n_cols) *n_cols = m.n_cols;
  if (row_ptr) *row_ptr = m.row_ptr;
  if (col_idx) *col_idx = m.col;
  if (llr) *llr = m.llr;
  if (count) *count = m.cnt;
  return CCO_OK;
}

int cco_result_stats(const cco_result_t *r, cco_stats_t *out) {
  if (!r || !out) return set_error(CCO_E_INVALID_ARG, "null argument");
  *out = r->stats;
  return CCO_OK;
}

int cco_result_free(cco_result_t *r) {
  if (!r) return CCO_OK;
  for (auto &m : r->mats) {
    for (void *p : {(void *)m.row_ptr, (void *)m.col, (void *)m.llr, (void *)m.cnt})
      if (p) r->ctx->pinned_put(p);
  }
  delete r;
  return CCO_OK;
}

// ---- SURVEY.md 8f-2: indicator model -> Elasticsearch bulk body (cco_format.cuh) --------------------------------------
namespace cco {
static int upload_dict(cco_ctx *c, Arena &ar, const cco_dictionary_t &d, DevDict *raw) {
  if (d.n < 0 || (d.n > 0 && (!d.offsets || (d.offsets[d.n] > 0 && !d.bytes)))) return set_error(CCO_E_INVALID_ARG, "bad dictionary");
  long long *off;
  unsigned char *bytes;
  const long long nb = d.n > 0 ? d.offsets[d.n] : 0;
  CKR(ar.alloc(&off, d.n + 1));
  CKR(ar.alloc(&bytes, std::max<long long>(nb, 1)));
  if (d.n > 0) {
    CK(cudaMemcpyAsync(off, d.offsets, sizeof(int64_t) * ((size_t)d.n + 1), cudaMemcpyHostToDevice, c->stream));
    if (nb > 0) CK(cudaMemcpyAsync(bytes, d.bytes, (size_t)nb, cudaMemcpyHostToDevice, c->stream));
  } else {
    CK(cudaMemsetAsync(off, 0, 8, c->stream));
  }
  raw->off = off;
  raw->bytes = bytes;
  raw->n = d.n;
  return CCO_OK;
}
// a few host strings as a device dictionary; waits for the copies, since the flattened strings are local
static int upload_strings(cco_ctx *c, Arena &ar, const std::vector<std::string> &strs, DevDict *raw) {
  std::vector<int64_t> off(strs.size() + 1, 0);
  std::string blob;
  for (size_t i = 0; i < strs.size(); ++i) {
    blob += strs[i];
    off[i + 1] = (int64_t)blob.size();
  }
  CKR(upload_dict(c, ar, cco_dictionary_t{(int64_t)strs.size(), off.data(), blob.data()}, raw));
  CK(cudaStreamSynchronize(c->stream));
  return CCO_OK;
}
// JSON-escape every string of a device dictionary (two passes: lengths, scan, bytes)
static int escape_dict(cco_ctx *c, Arena &ar, const DevDict &raw, DevDict *esc) {
  long long *len, *off;
  CKR(ar.alloc(&len, raw.n + 1));
  CKR(ar.alloc(&off, raw.n + 1));
  CK(cudaMemsetAsync(len + raw.n, 0, 8, c->stream));
  if (raw.n > 0) {
    k_escape_len<<<grid_for(raw.n, 256, c->sm_count), 256, 0, c->stream>>>(raw.n, raw.off, raw.bytes, len);
    c->launches++;
  }
  CKR(exclusive_sum(c, ar, len, off, raw.n + 1));
  long long total = 0;
  CK(cudaMemcpyAsync(&total, off + raw.n, 8, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  unsigned char *bytes;
  CKR(ar.alloc(&bytes, std::max<long long>(total, 1)));
  if (raw.n > 0) {
    k_escape_write<<<grid_for(raw.n, 256, c->sm_count), 256, 0, c->stream>>>(raw.n, raw.off, raw.bytes, off, bytes);
    c->launches++;
  }
  esc->off = off;
  esc->bytes = bytes;
  esc->n = raw.n;
  ar.release(len);
  return CCO_OK;
}
}  // namespace cco

namespace cco {
// PopModel's bucket edges for one ranking window (Joda integer millisecond arithmetic)
static PopArgs pop_args(int mode, long long start_ms, long long end_ms, int32_t n_keys) {
  PopArgs a;
  memset(&a, 0, sizeof a);
  a.n_items = n_keys;
  const long long dur = end_ms - start_ms;
  if (mode == CCO_POP_POPULAR) {
    a.n_buckets = 1;
    a.edge[0] = start_ms;
    a.edge[1] = end_ms;
  } else if (mode == CCO_POP_TRENDING) {   // PopModel.scala:134-138: halfInterval = durationMillis / 2
    a.n_buckets = 2;
    a.edge[0] = start_ms;
    a.edge[1] = start_ms + dur / 2;
    a.edge[2] = end_ms;
  } else {                                  // PopModel.scala:159-164: older = dur / 3, middle = the same length, newer = the rest
    a.n_buckets = 3;
    a.edge[0] = start_ms;
    a.edge[1] = start_ms + dur / 3;
    a.edge[2] = a.edge[1] + dur / 3;
    a.edge[3] = end_ms;
  }
  return a;
}

// one section of a combined key column (key_column), e.g. the row dictionary, the property items or one ranking stream.  A
// device section (the decoded ids of an index body) is already in HBM: offsets from 0, nbytes bytes.
struct KeySection {
  long long n;
  const int64_t *off;
  const char *bytes;
  bool device = false;
  long long nbytes = 0;
  long long base = 0;   // device: off[0] (bytes points at that byte)
  long long byte_count() const { return n == 0 ? 0 : device ? nbytes : off[n] - off[0]; }
};
// one ranking stream: the target ids of one event name's ranking events and their times, both on the host (a
// cco_ranking_stream_t) or both in HBM (an event log's columns) as items.device says; per ranking, its streams in order
struct Stream {
  KeySection items;
  const int64_t *time;
};
using Streams = std::vector<std::vector<Stream>>;
// the properties of an event log (cco_format_model_log): the columns of cco_item_properties_t in HBM, built on the device
struct DevProps {
  KeySection items;
  const int32_t *field;
  const long long *voff;   // from 0
  const unsigned char *vals;
};

// One string column of the sections in order: offsets from 0, bytes as 8-byte words with 16 bytes of padding.  A host
// section's offsets are checked on the device into *bad; the caller reads that verdict before any kernel reads bytes
// through the key column.
static int key_column(cco_ctx *c, Arena &ar, const std::vector<KeySection> &sec, int *bad, DevStrCol *key) {
  cudaStream_t s = c->stream;
  long long N = 0, nb = 0, max_n = 0;
  for (const KeySection &k : sec) {
    N += k.n;
    nb += k.byte_count();
    max_n = std::max(max_n, k.n);
  }
  key->n = N;
  key->base = 0;
  CKR(ar.alloc(&key->off, N + 1));
  CKR(ar.alloc(&key->w, (nb + 16 + 7) / 8));
  CKR(ar.alloc(&key->hash, std::max<long long>(N, 1)));
  CK(cudaMemsetAsync(key->off, 0, 8, s));
  long long *tmp_off;
  CKR(ar.alloc(&tmp_off, max_n + 1));
  // every section: raw offsets -> decreasing check -> rebased into the key column; bytes appended to the word buffer
  long long at = 0, byte_at = 0;
  for (const KeySection &k : sec) {
    if (k.n == 0) continue;
    const long long kb = k.byte_count();
    if (k.device) {
      k_rebase<<<grid_for(k.n + 1, 256, c->sm_count), 256, 0, s>>>(k.n + 1, (const long long *)k.off, byte_at - k.base, key->off + at);
      c->launches++;
      if (kb > 0) CK(cudaMemcpyAsync((char *)key->w + byte_at, k.bytes, (size_t)kb, cudaMemcpyDeviceToDevice, s));
      at += k.n;
      byte_at += kb;
      continue;
    }
    CK(cudaMemcpyAsync(tmp_off, k.off, sizeof(int64_t) * ((size_t)k.n + 1), cudaMemcpyHostToDevice, s));
    k_str_check<<<grid_for(k.n, 256, c->sm_count), 256, 0, s>>>(k.n, tmp_off, bad);
    k_rebase<<<grid_for(k.n + 1, 256, c->sm_count), 256, 0, s>>>(k.n + 1, tmp_off, byte_at - k.off[0], key->off + at);
    c->launches += 2;
    if (kb > 0) CK(cudaMemcpyAsync((char *)key->w + byte_at, k.bytes + k.off[0], (size_t)kb, cudaMemcpyHostToDevice, s));
    at += k.n;
    byte_at += kb;
  }
  ar.release(tmp_off);
  return CCO_OK;
}

// The model part of FormatArgs (cco_format_model, cco_rerank_model): group the item ids of every source, score the
// rankings per group, sort the properties, and list the documents of items without a row.  The caller's host columns have
// passed str_check_host.  unique_rows: two rows with the same id are CCO_E_INVALID_ARG (the documents of an old index).
static int model_fields(cco_ctx *c, Arena &ar, FormatArgs *fa, const KeySection &rows, const cco_item_properties_t *props,
                        int32_t n_rank, const cco_ranking_t *rk, const Streams &st, bool extra_docs, bool unique_rows = false,
                        const DevProps *dp = nullptr) {
  cudaStream_t s = c->stream;
  mail_reset(c);
  const long long R = rows.n, P = props ? props->n : 0;
  std::vector<KeySection> sec;
  sec.push_back(rows);
  sec.push_back(dp ? dp->items : KeySection{P, P > 0 ? props->item_offsets : nullptr, P > 0 ? props->item_bytes : nullptr});
  std::vector<long long> rank_begin(n_rank + 1);   // ranking k's events are key entries R + P + [rank_begin[k], rank_begin[k + 1])
  long long E = 0;
  for (int k = 0; k < n_rank; ++k) {
    rank_begin[k] = E;
    for (const Stream &q : st[k]) {
      sec.push_back(q.items);
      E += q.items.n;
    }
  }
  rank_begin[n_rank] = E;
  const long long N = R + P + E;
  int *bad;
  CKR(ar.alloc(&bad, 1));
  CK(cudaMemsetAsync(bad, 0, sizeof(int), s));
  DevStrCol key;
  CKR(key_column(c, ar, sec, bad, &key));
  // property fields and values
  int32_t *d_field = nullptr;
  if (dp && P > 0) {   // built on the device: nothing to copy or check
    d_field = (int32_t *)dp->field;
    fa->val_off = dp->voff;
    fa->val_base = 0;
    fa->vals = dp->vals;
  } else if (P > 0) {
    const long long vb = props->value_offsets[P] - props->value_offsets[0];
    long long *d_voff;
    unsigned char *d_vals;
    CKR(ar.alloc(&d_field, P));
    CKR(ar.alloc(&d_voff, P + 1));
    CKR(ar.alloc(&d_vals, std::max<long long>(vb, 1)));
    CK(cudaMemcpyAsync(d_field, props->field, sizeof(int32_t) * (size_t)P, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_voff, props->value_offsets, sizeof(int64_t) * ((size_t)P + 1), cudaMemcpyHostToDevice, s));
    if (vb > 0) CK(cudaMemcpyAsync(d_vals, props->value_bytes + props->value_offsets[0], (size_t)vb, cudaMemcpyHostToDevice, s));
    k_str_check<<<grid_for(P, 256, c->sm_count), 256, 0, s>>>(P, d_voff, bad);
    k_prop_check<<<grid_for(P, 256, c->sm_count), 256, 0, s>>>(P, d_field, props->n_fields, d_voff, bad);
    c->launches += 2;
    fa->val_off = d_voff;
    fa->val_base = props->value_offsets[0];
    fa->vals = d_vals;
  }
  // event times, all rankings' streams in order
  long long *d_t;
  CKR(ar.alloc(&d_t, std::max<long long>(E, 1)));
  for (int k = 0; k < n_rank; ++k) {
    long long e = rank_begin[k];
    for (const Stream &q : st[k]) {
      if (q.items.n > 0)
        CK(cudaMemcpyAsync(d_t + e, q.time, sizeof(int64_t) * (size_t)q.items.n,
                           q.items.device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s));
      e += q.items.n;
    }
  }
  // the device verdict comes before any kernel reads bytes through the offsets
  int h_bad = 0;
  CKR(mail_fetch(c, &h_bad, bad, 4));
  CKR(mail_wait(c));
  if (h_bad & 1) return set_error(CCO_E_INVALID_ARG, "offsets decrease");
  if (h_bad & 2) return set_error(CCO_E_INVALID_ARG, "a property field index is outside [0, %d)", props->n_fields);
  if (h_bad & 4) return set_error(CCO_E_INVALID_ARG, "an empty property value (values are JSON text)");

  // 1. item key space: one exact grouping by string over every source, numbered by first appearance
  str_hash(c, key, ~0ULL);
  int32_t *gid;
  CKR(ar.alloc(&gid, std::max<long long>(N, 1)));
  StrTable tb;
  CKR(str_group(c, ar, key, nullptr, false, 0, &tb, gid));
  const long long G = tb.n_groups;
  if (unique_rows && R > 0) {
    unsigned long long *dup, h_dup = ~0ULL;
    CKR(ar.alloc(&dup, 1));
    CK(cudaMemsetAsync(dup, 0xff, 8, s));
    k_dup_rows<<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, gid, tb.first_sorted, dup);
    c->launches++;
    CKR(mail_fetch(c, &h_dup, dup, 8));
    CKR(mail_wait(c));
    if (h_dup != ~0ULL)
      return set_error(CCO_E_INVALID_ARG, "document %llu: its _id is the _id of document %llu", h_dup >> 32, h_dup & 0xffffffffULL);
  }
  fa->n_groups = G;
  fa->row_group = gid + fa->row_id_base;
  // 2. properties: sorted by (group, field), stable in the triple index, so the last triple of each run wins
  if (P > 0) {
    unsigned long long *key;
    int32_t *tri, *pbeg, *pend;
    CKR(ar.alloc(&key, P));
    CKR(ar.alloc(&tri, P));
    CKR(ar.alloc(&pbeg, G));
    CKR(ar.alloc(&pend, G));
    CK(cudaMemsetAsync(pbeg, 0, sizeof(int32_t) * (size_t)G, s));
    CK(cudaMemsetAsync(pend, 0, sizeof(int32_t) * (size_t)G, s));
    k_prop_keys<<<grid_for(P, 256, c->sm_count), 256, 0, s>>>(P, gid + R, d_field, key, tri);
    CKR(sort_pairs(c, ar, P, &key, &tri, 32 + bits_for(G)));
    k_prop_ranges<<<grid_for(P, 256, c->sm_count), 256, 0, s>>>(P, key, pbeg, pend);
    c->launches += 2;
    fa->pkey = key;
    fa->ptri = tri;
    fa->pbeg = pbeg;
    fa->pend = pend;
  }
  // 3. rankings: PopModel histograms over the groups; random ones from the popular histogram, the properties and the hash
  fa->n_rank = n_rank;
  if (n_rank > 0) {
    long long *score;
    unsigned char *pmask, *present;
    int32_t *counts;
    unsigned long long *tot;
    CKR(ar.alloc(&score, (size_t)n_rank * G));
    CKR(ar.alloc(&pmask, G));
    CKR(ar.alloc(&present, G));
    CKR(ar.alloc(&counts, (size_t)3 * G));
    CKR(ar.alloc(&tot, 4));
    CK(cudaMemsetAsync(pmask, 0, (size_t)G, s));
    for (int k = 0; k < n_rank; ++k) {
      const bool random = rk[k].mode == CCO_POP_RANDOM;
      const PopArgs pa = pop_args(random ? CCO_POP_POPULAR : rk[k].mode, rk[k].start_ms, rk[k].end_ms, (int32_t)G);
      const long long ne = rank_begin[k + 1] - rank_begin[k];
      CK(cudaMemsetAsync(counts, 0, sizeof(int32_t) * (size_t)pa.n_buckets * G, s));
      CK(cudaMemsetAsync(tot, 0, 32, s));
      if (ne > 0) {
        k_pop_count<<<grid_for(ne, 256, c->sm_count), 256, 0, s>>>(ne, gid + R + P + rank_begin[k], d_t + rank_begin[k], pa, counts, tot);
        c->launches++;
      }
      if (random) {
        k_random_score<<<grid_for(G, 256, c->sm_count), 256, 0, s>>>(G, counts, fa->pbeg, fa->pend, tb.first_sorted, key.hash,
                                                                    rk[k].start_ms, rk[k].end_ms, score + (size_t)k * G, present);
        fa->rank_scale[k] = 15;
      } else {
        k_pop_score<long long><<<grid_for(G, 256, c->sm_count), 256, 0, s>>>(pa, rk[k].mode, counts, tot, score + (size_t)k * G, present);
      }
      k_rank_mask<<<grid_for(G, 256, c->sm_count), 256, 0, s>>>(G, present, k, pmask);
      c->launches += 2;
    }
    ar.release(counts);
    ar.release(present);
    fa->score = score;
    fa->pmask = pmask;
  }
  // 4. documents of items without a row, in order of first appearance (only the result that begins at row 0 writes them)
  fa->n_extra = 0;
  if (extra_docs && G > 0) {
    uint32_t *flag, *pos;
    CKR(ar.alloc(&flag, G + 1));
    CKR(ar.alloc(&pos, G + 1));
    CK(cudaMemsetAsync(flag + G, 0, 4, s));
    k_extra_flags<<<grid_for(G, 256, c->sm_count), 256, 0, s>>>(G, tb.first_sorted, R, fa->pbeg, fa->pend, fa->pmask, flag);
    c->launches++;
    CKR(exclusive_sum(c, ar, flag, pos, G + 1));
    uint32_t n_extra = 0;
    CKR(mail_fetch(c, &n_extra, pos + G, 4));
    CKR(mail_wait(c));
    if (n_extra > 0) {
      int32_t *extra_group;
      uint32_t *extra_first;
      long long *len, *off;
      CKR(ar.alloc(&extra_group, n_extra));
      CKR(ar.alloc(&extra_first, n_extra));
      CKR(ar.alloc(&len, (long long)n_extra + 1));
      CKR(ar.alloc(&off, (long long)n_extra + 1));
      k_extra_compact<<<grid_for(G, 256, c->sm_count), 256, 0, s>>>(G, flag, pos, tb.first_sorted, extra_group, extra_first);
      CK(cudaMemsetAsync(len + n_extra, 0, 8, s));
      k_str_dict_len<<<grid_for(n_extra, 256, c->sm_count), 256, 0, s>>>(n_extra, extra_first, key.off, len);
      CKR(exclusive_sum(c, ar, len, off, (long long)n_extra + 1));
      long long total = 0;
      CKR(mail_fetch(c, &total, off + n_extra, 8));
      CKR(mail_wait(c));
      unsigned char *bytes;
      CKR(ar.alloc(&bytes, std::max<long long>(total, 1)));
      k_str_dict_gather<<<grid_for(n_extra, 256, c->sm_count), 256, 0, s>>>(n_extra, extra_first, key.off, 0, (const unsigned char *)key.w,
                                                                           off, bytes);
      c->launches += 3;
      const DevDict raw = {off, bytes, (long long)n_extra};
      CKR(escape_dict(c, ar, raw, &fa->extra_ids));
      fa->extra_group = extra_group;
      fa->n_extra = (int32_t)n_extra;
    }
  }
  return CCO_OK;
}

// host checks of the model inputs (the device checks decreasing offsets, field indices and empty values).  st: the
// rankings' streams; empty for rankings that hold their streams (cco_ranking_t), which are listed into it as they are checked
static int model_check_host(const cco_dictionary_t *row_ids, const cco_item_properties_t *props, int32_t n_rank, const cco_ranking_t *rk,
                            Streams *st, bool dev_props = false) {
  if (n_rank < 0 || (n_rank > 0 && !rk)) return set_error(CCO_E_INVALID_ARG, "bad rankings");
  if (n_rank > kMaxRankings) return set_error(CCO_E_UNSUPPORTED, "%d rankings, at most %d", n_rank, kMaxRankings);
  long long total = row_ids->n;
  CKR(str_check_host(row_ids->n, row_ids->offsets, row_ids->bytes, -1, "row id"));
  if (props) {
    if (props->n < 0 || props->n_fields < 0 || (props->n_fields > 0 && !props->field_names)) return set_error(CCO_E_INVALID_ARG, "bad properties");
    for (int f = 0; f < props->n_fields; ++f) {
      if (!props->field_names[f]) return set_error(CCO_E_INVALID_ARG, "null field name %d", f);
      for (int h = 0; h < f; ++h)
        if (!strcmp(props->field_names[h], props->field_names[f]))
          return set_error(CCO_E_INVALID_ARG, "field names %d and %d are both \"%s\"", h, f, props->field_names[f]);
    }
    if (props->n > 0 && !dev_props) {
      if (!props->field) return set_error(CCO_E_INVALID_ARG, "null property field indices");
      CKR(str_check_host(props->n, props->item_offsets, props->item_bytes, -1, "property item"));
      CKR(str_check_host(props->n, props->value_offsets, props->value_bytes, -1, "property value"));
    }
    total += props->n;
  }
  const bool listed = !st->empty();
  st->resize(n_rank);
  for (int k = 0; k < n_rank; ++k) {
    const cco_ranking_t &r = rk[k];
    if (!r.name) return set_error(CCO_E_INVALID_ARG, "ranking %d: null name", k);
    if (r.mode < CCO_POP_POPULAR || r.mode > CCO_POP_RANDOM)
      return set_error(CCO_E_INVALID_ARG, "ranking %d: mode must be CCO_POP_POPULAR, _TRENDING, _HOT or _RANDOM", k);
    if (r.end_ms < r.start_ms) return set_error(CCO_E_INVALID_ARG, "ranking %d: end before start (Joda Interval would throw)", k);
    if (!listed) {
      if (r.n_streams < 1 || !r.streams) return set_error(CCO_E_INVALID_ARG, "ranking %d: needs at least one stream", k);
      for (int q = 0; q < r.n_streams; ++q) {
        const cco_ranking_stream_t &h = r.streams[q];
        (*st)[k].push_back({{h.n_events, h.item_offsets, h.item_bytes}, h.time_ms});
      }
    }
    for (const Stream &q : (*st)[k]) {
      if (!q.items.device) {
        CKR(str_check_host(q.items.n, q.items.off, q.items.bytes, k, "ranking item"));
        if (q.items.n > 0 && !q.time) return set_error(CCO_E_INVALID_ARG, "ranking %d: null event times", k);
      }
      total += q.items.n;
      if (total >= 0x7fffffffLL) break;
    }
    if (total >= 0x7fffffffLL) break;
  }
  if (total >= 0x7fffffffLL) return set_error(CCO_E_UNSUPPORTED, "rows + property triples + ranking events must stay < 2^31 per call");
  return CCO_OK;
}

// The names of FormatArgs: event names, field names and ranking names escaped as one more tiny dictionary, and (model) who
// beats whom where names repeat.
static int model_names(cco_ctx *c, Arena &ar, FormatArgs *fa, int n_ind, const char *const *names, bool model,
                       const cco_item_properties_t *props, int32_t n_rank, const cco_ranking_t *rk) {
  cudaStream_t s = c->stream;
  const int n_fields = props ? props->n_fields : 0;
  std::vector<std::string> all_names(names, names + n_ind);
  if (model) {
    for (int f = 0; f < n_fields; ++f) all_names.push_back(props->field_names[f]);
    for (int k = 0; k < n_rank; ++k) all_names.push_back(rk[k].name);
  }
  const int n_all = (int)all_names.size();
  std::vector<long long> eoff(n_all + 1);
  DevDict nraw, nesc;
  CKR(upload_strings(c, ar, all_names, &nraw));
  CKR(escape_dict(c, ar, nraw, &nesc));
  CK(cudaMemcpyAsync(eoff.data(), nesc.off, sizeof(long long) * ((size_t)n_all + 1), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  fa->names = nesc.bytes;
  for (int i = 0; i <= n_ind; ++i) fa->name_off[i] = (int32_t)eoff[i];
  if (model) {
    fa->field_off = nesc.off + n_ind;
    for (int k = 0; k <= n_rank; ++k) fa->rank_name_off[k] = (int32_t)eoff[n_ind + n_fields + k];
  }
  if (model) {
    // precedence, lowest to highest: indicators < properties < rankings (a later ranking beats an earlier one) < "id".
    // The names are few, so the host resolves who beats whom and the device only checks presence per document.
    auto same = [](const char *x, const char *y) { return strcmp(x, y) == 0; };
    std::vector<uint16_t> fclash(std::max(n_fields, 1), 0);
    for (int f = 0; f < n_fields; ++f) {
      if (same(props->field_names[f], "id")) fclash[f] |= kClashId;
      for (int k = 0; k < n_rank; ++k)
        if (same(props->field_names[f], rk[k].name)) fclash[f] |= (uint16_t)(1u << k);
    }
    for (int i = 0; i < n_ind; ++i) {
      fa->ind_field[i] = -1;
      for (int f = 0; f < n_fields; ++f)
        if (same(names[i], props->field_names[f])) fa->ind_field[i] = f;
      for (int k = 0; k < n_rank; ++k)
        if (same(names[i], rk[k].name)) fa->ind_rank[i] |= (uint8_t)(1u << k);
    }
    for (int k = 0; k < n_rank; ++k) {
      if (same(rk[k].name, "id")) fa->rank_clash[k] |= kClashId;
      for (int l = k + 1; l < n_rank; ++l)
        if (same(rk[k].name, rk[l].name)) fa->rank_clash[k] |= (uint16_t)(1u << l);
    }
    uint16_t *d_fclash;
    CKR(ar.alloc(&d_fclash, fclash.size()));
    CK(cudaMemcpyAsync(d_fclash, fclash.data(), sizeof(uint16_t) * fclash.size(), cudaMemcpyHostToDevice, s));
    fa->field_clash = d_fclash;
    CK(cudaStreamSynchronize(s));   // fclash is a local
  }
  return CCO_OK;
}

// The total bytes at d_out into pinned memory of `owner` (released with cco_host_free on that context), then the wait for
// stream s; `also` may enqueue more copies before the wait.  On failure the pinned memory is given back.
static int body_to_host(cco_ctx *owner, cudaStream_t s, const unsigned char *d_out, long long total, char **out_bytes, int64_t *out_len,
                        const std::function<int()> &also = nullptr) {
  char *host = (char *)owner->pinned_get((size_t)std::max<long long>(total, 1), /*for_result=*/false);
  if (!host) return set_error(CCO_E_OOM, "pinned host allocation failed");
  const int st = [&]() -> int {
    if (total > 0) CK(cudaMemcpyAsync(host, d_out, (size_t)total, cudaMemcpyDeviceToHost, s));
    if (also) CKR(also());
    CK(cudaStreamSynchronize(s));
    CK(cudaGetLastError());
    return CCO_OK;
  }();
  if (st != CCO_OK) {
    owner->pinned_put(host);
    return st;
  }
  *out_bytes = host;
  *out_len = total;
  return CCO_OK;
}

// cco_format_es_bulk == format_model without properties and rankings: one set of document kernels
static int format_model(cco_ctx_t *ctx, const cco_result_t *res, int32_t n_names, const char *const *names, const cco_dictionary_t *row_ids,
                        const cco_dictionary_t *col_ids, const cco_item_properties_t *props, int32_t n_rank, const cco_ranking_t *rk,
                        char **out_bytes, int64_t *out_len, const char *range, Streams st = {}, const DevProps *dp = nullptr) {
  if (!ctx || !res || !names || !row_ids || !col_ids || !out_bytes || !out_len) return set_error(CCO_E_INVALID_ARG, "null argument");
  const int n_ind = (int)res->mats.size();
  if (n_names != n_ind) return set_error(CCO_E_INVALID_ARG, "%d event names for %d indicators", n_names, n_ind);
  if (n_ind < 1 || n_ind > kMaxFormatIndicators) return set_error(CCO_E_UNSUPPORTED, "1..%d indicators", kMaxFormatIndicators);
  cco_ctx *c = ctx->members.empty() ? ctx : ctx->members[0];   // a group's merged model is formatted on its first GPU
  const int64_t row_lo = res->mats[0].row_begin, row_hi = res->mats[0].row_end;
  for (int i = 0; i < n_ind; ++i) {
    const ResultMat &m = res->mats[i];
    if (m.row_begin != row_lo || m.row_end != row_hi) return set_error(CCO_E_INVALID_ARG, "indicators cover different row ranges");
    if (!m.row_ptr || (m.row_ptr[row_hi - row_lo] > 0 && !m.col)) return set_error(CCO_E_INVALID_ARG, "indicator %d has no column array on the host", i);
    if (col_ids[i].n < m.n_cols) return set_error(CCO_E_INVALID_ARG, "column dictionary %d has %lld ids for %d columns", i, (long long)col_ids[i].n, m.n_cols);
    if (!names[i]) return set_error(CCO_E_INVALID_ARG, "null event name");
  }
  if (row_ids->n < row_hi) return set_error(CCO_E_INVALID_ARG, "row dictionary has %lld ids, rows go up to %lld", (long long)row_ids->n, (long long)row_hi);
  const bool model = (props && props->n > 0) || n_rank > 0;
  if (model) CKR(model_check_host(row_ids, props, n_rank, rk, &st, dp != nullptr));
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Arena ar(s);
  NvtxRange nvtx(range);
  FormatArgs fa;
  memset(&fa, 0, sizeof fa);
  fa.n_rows = (int32_t)(row_hi - row_lo);
  fa.row_id_base = row_lo;
  fa.n_ind = n_ind;
  DevDict raw;
  CKR(upload_dict(c, ar, *row_ids, &raw));
  CKR(escape_dict(c, ar, raw, &fa.row_ids));
  CKR(model_names(c, ar, &fa, n_ind, names, model, props, n_rank, rk));
  if (model) CKR(model_fields(c, ar, &fa, KeySection{row_ids->n, row_ids->offsets, row_ids->bytes}, props, n_rank, rk, st, row_lo == 0, false, dp));
  for (int i = 0; i < n_ind; ++i) {
    const ResultMat &m = res->mats[i];
    CKR(upload_dict(c, ar, col_ids[i], &raw));
    CKR(escape_dict(c, ar, raw, &fa.col_ids[i]));
    const long long n_my = row_hi - row_lo, nnz = m.row_ptr[n_my] - m.row_ptr[0];
    long long *d_rp;
    int32_t *d_col;
    CKR(ar.alloc(&d_rp, n_my + 1));
    CKR(ar.alloc(&d_col, std::max<long long>(nnz, 1)));
    CK(cudaMemcpyAsync(d_rp, m.row_ptr, sizeof(int64_t) * ((size_t)n_my + 1), cudaMemcpyHostToDevice, s));
    if (nnz > 0) CK(cudaMemcpyAsync(d_col, m.col + m.row_ptr[0], sizeof(int32_t) * (size_t)nnz, cudaMemcpyHostToDevice, s));
    if (m.row_ptr[0] != 0) {   // a group member's slice is rebased inside the merged arrays: bring it back to 0
      k_add_i64<<<grid_for(n_my + 1, 256, c->sm_count, 2), 256, 0, s>>>(n_my + 1, -(long long)m.row_ptr[0], d_rp);
      c->launches++;
    }
    fa.row_ptr[i] = d_rp;
    fa.col[i] = d_col;
  }
  const int32_t n_docs = fa.n_rows + fa.n_extra;
  long long *doc_len, *doc_off;
  CKR(ar.alloc(&doc_len, (long long)n_docs + 1));
  CKR(ar.alloc(&doc_off, (long long)n_docs + 1));
  CK(cudaMemsetAsync(doc_len + n_docs, 0, 8, s));
  if (n_docs > 0) {
    k_doc_len<<<grid_for(n_docs, 256, c->sm_count), 256, 0, s>>>(fa, n_docs, doc_len);
    c->launches++;
  }
  CKR(exclusive_sum(c, ar, doc_len, doc_off, (long long)n_docs + 1));
  long long total = 0;
  CK(cudaMemcpyAsync(&total, doc_off + n_docs, 8, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  unsigned char *d_out;
  CKR(ar.alloc(&d_out, std::max<long long>(total, 1)));
  if (n_docs > 0 && total > 0) {
    k_doc_write<<<grid_for((long long)n_docs * 32, 256, c->sm_count), 256, 0, s>>>(fa, n_docs, doc_off, d_out);
    c->launches++;
  }
  return body_to_host(ctx, s, d_out, total, out_bytes, out_len);
}

// ---- cco_rerank_model: an existing index with fresh rankings and properties (calcPop), kernels in cco_json.cuh ---------
// the message of a tokenizer / action verdict: span = err >> 8 is a line (lines) or a document
static int json_error(unsigned long long err, bool lines) {
  const long long span = (long long)(err >> 8), doc = lines ? span / 2 : span;
  const int code = (int)(err & 0xff);
  const char *part = lines && (span & 1) ? "source" : "action";
  if (code == kJsonLongLine) return set_error(CCO_E_UNSUPPORTED, "document %lld: the %s line is longer than 2^31 - 1 bytes", doc, part);
  if (!lines || code == kJsonAction)
    return set_error(CCO_E_INVALID_ARG, "document %lld: the action line is not {\"index\":{...}} with a string \"_id\" member", doc);
  if (code == kJsonNotObject) return set_error(CCO_E_INVALID_ARG, "document %lld: the %s line is not a JSON object", doc, part);
  if (code == kJsonString)
    return set_error(CCO_E_INVALID_ARG, "document %lld: a string of the %s line is unterminated or holds a bad escape or a raw byte < 0x20",
                     doc, part);
  return set_error(CCO_E_INVALID_ARG, "document %lld: the %s line is not one JSON object (unbalanced brackets or an unexpected token)",
                   doc, part);
}
// one tokenizer run over n object spans: count, verdict (*verdict = ~0: every span is one object), then, when the verdict
// is clean and the members are fewer than limit, write.  moff[s] = first member of span s, *total = all members
static int json_members(cco_ctx *c, Arena &ar, long long n, const long long *sb, const long long *se, const unsigned char *body,
                        long long limit, unsigned long long *verdict, long long **moff_out, JMember **mem_out, long long *total_out) {
  cudaStream_t s = c->stream;
  long long *cnt, *moff;
  unsigned long long *err;
  CKR(ar.alloc(&cnt, n + 1));
  CKR(ar.alloc(&moff, n + 1));
  CKR(ar.alloc(&err, 1));
  CK(cudaMemsetAsync(cnt + n, 0, 8, s));
  CK(cudaMemsetAsync(err, 0xff, 8, s));
  const int grid = grid_for(n * 32, 256, c->sm_count);
  if (n > 0) {
    k_json_members<<<grid, 256, 0, s>>>(n, sb, se, body, MemberSink<false>{cnt, nullptr, nullptr}, err);
    c->launches++;
  }
  CKR(exclusive_sum(c, ar, cnt, moff, n + 1));
  long long total = 0;
  CKR(mail_fetch(c, verdict, err, 8));
  CKR(mail_fetch(c, &total, moff + n, 8));
  CKR(mail_wait(c));
  *total_out = total;
  if (*verdict != ~0ULL || total >= limit) return CCO_OK;
  JMember *mem;
  CKR(ar.alloc(&mem, std::max<long long>(total, 1)));
  if (total > 0) {
    k_json_members<<<grid, 256, 0, s>>>(n, sb, se, body, MemberSink<true>{nullptr, moff, mem}, err);
    c->launches++;
  }
  ar.release(cnt);
  *moff_out = moff;
  *mem_out = mem;
  return CCO_OK;
}
// the lines of the len bytes of w (bytes [len, round_up(len, 8) + 16) are zero): every '\n' ends one; open_tail: a last
// line without it ends at len.  -> *L lines and, when there are any, their spans [sb, se)
static int split_lines(cco_ctx *c, Arena &ar, const uint64_t *w, long long len, bool open_tail, long long *L, long long **sb,
                       long long **se) {
  cudaStream_t s = c->stream;
  const long long NW = (len + 7) / 8, n_chunks = (NW + kNlChunkWords - 1) / kNlChunkWords;
  long long *cc, *coff, *nl;
  CKR(ar.alloc(&cc, n_chunks + 1));
  CKR(ar.alloc(&coff, n_chunks + 1));
  CK(cudaMemsetAsync(cc + n_chunks, 0, 8, s));
  if (NW > 0) {
    k_nl_count<<<grid_for(n_chunks * 32, 256, c->sm_count), 256, 0, s>>>(NW, w, cc);
    c->launches++;
  }
  CKR(exclusive_sum(c, ar, cc, coff, n_chunks + 1));
  *L = 0;
  CKR(mail_fetch(c, L, coff + n_chunks, 8));
  CKR(mail_wait(c));
  CKR(ar.alloc(&nl, *L + 1));
  if (*L > 0) {
    k_nl_write<<<grid_for(n_chunks * 32, 256, c->sm_count), 256, 0, s>>>(NW, w, coff, nl);
    c->launches++;
  }
  if (open_tail) {
    CK(cudaMemcpyAsync(nl + *L, &len, 8, cudaMemcpyHostToDevice, s));
    ++*L;
  }
  if (*L == 0) return CCO_OK;
  CKR(ar.alloc(sb, *L));
  CKR(ar.alloc(se, *L));
  k_line_spans<<<grid_for(*L, 256, c->sm_count), 256, 0, s>>>(*L, nl, *sb, *se);
  c->launches++;
  return CCO_OK;
}
// the strings [m.nb, m.ne) of n members decoded into a string column (offsets from 0, 8-byte words, 16 bytes of padding)
static int json_decode(cco_ctx *c, Arena &ar, long long n, const JMember *m, const unsigned char *body, DevStrCol *col, long long *bytes) {
  cudaStream_t s = c->stream;
  long long *len;
  CKR(ar.alloc(&len, n + 1));
  CKR(ar.alloc(&col->off, n + 1));
  CKR(ar.alloc(&col->hash, std::max<long long>(n, 1)));
  CK(cudaMemsetAsync(len + n, 0, 8, s));
  const int grid = grid_for(n, 256, c->sm_count);
  if (n > 0) k_json_unescape<false><<<grid, 256, 0, s>>>(n, m, body, len, nullptr, nullptr);
  CKR(exclusive_sum(c, ar, len, col->off, n + 1));
  long long total = 0;
  CKR(mail_fetch(c, &total, col->off + n, 8));
  CKR(mail_wait(c));
  CKR(ar.alloc(&col->w, (total + 16 + 7) / 8));
  if (n > 0 && total > 0) k_json_unescape<true><<<grid, 256, 0, s>>>(n, m, body, nullptr, col->off, (unsigned char *)col->w);
  c->launches += 2;
  ar.release(len);
  col->n = n;
  col->base = 0;
  *bytes = total;
  return CCO_OK;
}

// the documents of an index body parsed on the device: its lines' members and the decoded member names and _ids
struct BulkDocs {
  const unsigned char *body = nullptr;   // the body as 8-byte words with 16 bytes of zero padding
  long long D = 0, M1 = 0;               // documents, members of all lines
  long long *line_moff = nullptr;        // [2 D + 1]: line l's members are [line_moff[l], line_moff[l + 1])
  JMember *mem = nullptr;                // [M1]
  DevStrCol names, ids;                  // decoded member names [M1] and _ids [D] (offsets from 0)
  long long ids_bytes = 0;
  const long long *line_b = nullptr;     // [2 D]: the first byte of each line
};
// upload, line split, members, the action / _id checks and the decoded names and ids (cco_rerank_model's grammar; the
// messages name the 0-based document).  extra entries share the 2^31 limit with the documents; `what` names them.
static int bulk_parse(cco_ctx *c, Arena &ar, const char *body, int64_t body_len, long long extra, const char *what, BulkDocs *bd) {
  cudaStream_t s = c->stream;
  // 1. the body, once, into 8-byte words with 16 bytes of zero padding
  const long long NW = (body_len + 7) / 8;
  uint64_t *w;
  CKR(ar.alloc(&w, NW + 2));
  CK(cudaMemsetAsync(w + body_len / 8, 0, sizeof(uint64_t) * (size_t)(NW + 2 - body_len / 8), s));
  if (body_len > 0) CK(cudaMemcpyAsync(w, body, (size_t)body_len, cudaMemcpyHostToDevice, s));
  const unsigned char *bb = (const unsigned char *)w;
  bd->body = bb;
  // 2. line bounds
  long long L = 0, *sb = nullptr, *se = nullptr;
  CKR(split_lines(c, ar, w, body_len, false, &L, &sb, &se));
  if (L & 1) return set_error(CCO_E_INVALID_ARG, "the body has %lld lines: lines come in (action, source) pairs", L);
  const long long D = L / 2;
  if (D + extra >= 0x7fffffffLL) return set_error(CCO_E_UNSUPPORTED, "documents + %s must stay < 2^31 per call", what);
  bd->D = D;
  bd->line_b = sb;
  if (D == 0) return CCO_OK;
  // 3. members of every line; the verdict on the whole body comes before anything reads through the spans
  unsigned long long *err, h_err = 0;
  CKR(json_members(c, ar, L, sb, se, bb, 0x7fffffffLL, &h_err, &bd->line_moff, &bd->mem, &bd->M1));
  if (h_err != ~0ULL) return json_error(h_err, true);
  if (bd->M1 >= 0x7fffffffLL) return set_error(CCO_E_UNSUPPORTED, "%lld members in the body, at most 2^31 - 2", bd->M1);
  // 4. member names decoded; each action is {"index":{...}} and its "_id" is a string
  long long name_bytes = 0;
  CKR(json_decode(c, ar, bd->M1, bd->mem, bb, &bd->names, &name_bytes));
  long long *ib, *ie;
  CKR(ar.alloc(&ib, D));
  CKR(ar.alloc(&ie, D));
  CKR(ar.alloc(&err, 1));
  CK(cudaMemsetAsync(err, 0xff, 8, s));
  k_action_check<<<grid_for(D, 256, c->sm_count), 256, 0, s>>>(D, bd->line_moff, bd->mem, bd->names.off, (const unsigned char *)bd->names.w,
                                                               bb, ib, ie, err);
  c->launches++;
  CKR(mail_fetch(c, &h_err, err, 8));
  CKR(mail_wait(c));
  if (h_err != ~0ULL) return json_error(h_err, false);
  long long *imoff, M2 = 0, iname_bytes = 0;
  JMember *imem, *id_span;
  CKR(json_members(c, ar, D, ib, ie, bb, 0x7fffffffLL, &h_err, &imoff, &imem, &M2));
  if (h_err != ~0ULL) return json_error(h_err, false);
  if (M2 >= 0x7fffffffLL) return set_error(CCO_E_UNSUPPORTED, "%lld members in the body, at most 2^31 - 2", M2);
  DevStrCol inames;
  CKR(json_decode(c, ar, M2, imem, bb, &inames, &iname_bytes));
  CKR(ar.alloc(&id_span, D));
  k_pick_id<<<grid_for(D, 256, c->sm_count), 256, 0, s>>>(D, imoff, imem, inames.off, (const unsigned char *)inames.w, bb, id_span, err);
  c->launches++;
  CKR(mail_fetch(c, &h_err, err, 8));
  CKR(mail_wait(c));
  if (h_err != ~0ULL) return json_error(h_err, false);
  return json_decode(c, ar, D, id_span, bb, &bd->ids, &bd->ids_bytes);
}
// the decoded member names of a body against a small host table of names: *ngid = each member's name group, *entry_of =
// each group's table entry (-1: not in the table)
static int member_entries(cco_ctx *c, Arena &ar, const DevStrCol &names, const std::vector<std::string> &entries, int32_t **ngid,
                          int32_t **entry_of) {
  DevDict traw;
  CKR(upload_strings(c, ar, entries, &traw));
  str_hash(c, names, ~0ULL);
  CKR(ar.alloc(ngid, std::max<long long>(names.n, 1)));
  StrTable nt;
  CKR(str_group(c, ar, names, nullptr, false, 0, &nt, *ngid));
  CKR(ar.alloc(entry_of, std::max<long long>(nt.n_groups, 1)));
  if (nt.n_groups > 0) {
    k_name_entry<<<grid_for(nt.n_groups, 256, c->sm_count), 256, 0, c->stream>>>(nt.n_groups, nt.first_sorted, names.off, (const unsigned char *)names.w,
                                                                                (int)entries.size(), traw.off, traw.bytes, *entry_of);
    c->launches++;
  }
  return CCO_OK;
}

static int rerank_model(cco_ctx_t *ctx, const char *body, int64_t body_len, const cco_item_properties_t *props, int32_t n_rank,
                        const cco_ranking_t *rk, char **out_bytes, int64_t *out_len, Streams st = {}, const DevProps *dp = nullptr) {
  if (!ctx || !out_bytes || !out_len || body_len < 0 || (body_len > 0 && !body)) return set_error(CCO_E_INVALID_ARG, "null argument or negative length");
  if (!ctx->members.empty()) return set_error(CCO_E_UNSUPPORTED, "per-GPU contexts only");
  if (body_len > 0 && body[body_len - 1] != '\n') return set_error(CCO_E_INVALID_ARG, "the body does not end in a newline");
  const cco_dictionary_t no_rows = {0, nullptr, nullptr};
  CKR(model_check_host(&no_rows, props, n_rank, rk, &st, dp != nullptr));
  long long fresh = props ? props->n : 0;   // property triples + ranking events, checked < 2^31 by model_check_host
  for (const std::vector<Stream> &r : st)
    for (const Stream &q : r) fresh += q.items.n;
  cco_ctx *c = ctx;
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Arena ar(s);
  NvtxRange nvtx("cco:rerank_model");
  mail_reset(c);
  // 1-4. the documents: members, decoded names and _ids
  BulkDocs bd;
  CKR(bulk_parse(c, ar, body, body_len, fresh, "property triples + ranking events", &bd));
  const long long D = bd.D, M1 = bd.M1;
  const unsigned char *bb = bd.body;
  FormatArgs fa;
  memset(&fa, 0, sizeof fa);
  RerankArgs ra;
  memset(&ra, 0, sizeof ra);
  ra.body = bb;
  DevStrCol &ids = bd.ids, &names = bd.names;
  const long long ids_bytes = bd.ids_bytes;
  ra.line_moff = bd.line_moff;
  ra.mem = bd.mem;
  // 5. join: the decoded ids are the row section of the key column (a group with two of them is a repeated _id)
  CKR(model_names(c, ar, &fa, 0, nullptr, true, props, n_rank, rk));
  fa.n_rows = (int32_t)D;
  const DevDict raw_ids = {ids.off, (const unsigned char *)ids.w, D};
  CKR(escape_dict(c, ar, raw_ids, &fa.row_ids));
  const KeySection rows{D, (const int64_t *)ids.off, (const char *)ids.w, true, ids_bytes};
  CKR(model_fields(c, ar, &fa, rows, props, n_rank, rk, st, true, true, dp));
  // 6. member names -> the distinct names of the fields, the rankings and "id"
  if (D > 0) {
    std::vector<std::string> ent;
    std::vector<int32_t> ent_field;
    std::vector<uint8_t> ent_rank, ent_id;
    auto entry = [&](const char *nm) {
      for (size_t t = 0; t < ent.size(); ++t)
        if (ent[t] == nm) return (int)t;
      ent.push_back(nm);
      ent_field.push_back(-1);
      ent_rank.push_back(0);
      ent_id.push_back(0);
      return (int)ent.size() - 1;
    };
    for (int f = 0; props && f < props->n_fields; ++f) ent_field[entry(props->field_names[f])] = f;
    for (int k = 0; k < n_rank; ++k) ent_rank[entry(rk[k].name)] |= (uint8_t)(1u << k);
    ent_id[entry("id")] = 1;
    const int T = (int)ent.size();
    int32_t *d_field, *ngid, *entry_of, *ment;
    uint8_t *d_rank, *d_id, *mkeep;
    CKR(ar.alloc(&d_field, T));
    CKR(ar.alloc(&d_rank, T));
    CKR(ar.alloc(&d_id, T));
    CK(cudaMemcpyAsync(d_field, ent_field.data(), sizeof(int32_t) * T, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_rank, ent_rank.data(), T, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_id, ent_id.data(), T, cudaMemcpyHostToDevice, s));
    CKR(member_entries(c, ar, names, ent, &ngid, &entry_of));   // its wait for the upload also covers these local tables
    CKR(ar.alloc(&ment, std::max<long long>(M1, 1)));
    CKR(ar.alloc(&mkeep, std::max<long long>(M1, 1)));
    k_member_info<<<grid_for(D * 32, 256, c->sm_count), 256, 0, s>>>(D, ra.line_moff, ngid, entry_of, d_id, ment, mkeep);
    c->launches++;
    ra.ment = ment;
    ra.mkeep = mkeep;
    ra.ent_field = d_field;
    ra.ent_rank = d_rank;
  }
  // 7. documents: the old ones merged, then the new items' as cco_format_model writes them
  const long long X = fa.n_extra, n_docs = D + X;
  FormatArgs fx = fa;   // the new items only
  fx.n_rows = 0;
  long long *doc_len, *doc_off;
  CKR(ar.alloc(&doc_len, n_docs + 1));
  CKR(ar.alloc(&doc_off, n_docs + 1));
  CK(cudaMemsetAsync(doc_len + n_docs, 0, 8, s));
  if (D > 0) {
    k_rerank_len<<<grid_for(D, 256, c->sm_count), 256, 0, s>>>(fa, ra, (int32_t)D, doc_len);
    c->launches++;
  }
  if (X > 0) {
    k_doc_len<<<grid_for(X, 256, c->sm_count), 256, 0, s>>>(fx, (int32_t)X, doc_len + D);
    c->launches++;
  }
  CKR(exclusive_sum(c, ar, doc_len, doc_off, n_docs + 1));
  long long total = 0;
  CKR(mail_fetch(c, &total, doc_off + n_docs, 8));
  CKR(mail_wait(c));
  unsigned char *d_out;
  CKR(ar.alloc(&d_out, std::max<long long>(total, 1)));
  if (D > 0) {
    k_rerank_write<<<grid_for(D * 32, 256, c->sm_count), 256, 0, s>>>(fa, ra, (int32_t)D, doc_off, d_out);
    c->launches++;
  }
  if (X > 0) {
    k_doc_write<<<grid_for(X * 32, 256, c->sm_count), 256, 0, s>>>(fx, (int32_t)X, doc_off + D, d_out);
    c->launches++;
  }
  return body_to_host(c, s, d_out, total, out_bytes, out_len);
}
}  // namespace cco

int cco_rerank_model(cco_ctx_t *ctx, const char *body, int64_t body_len, const cco_item_properties_t *props, int32_t n_rankings,
                     const cco_ranking_t *rankings, char **out_bytes, int64_t *out_len) {
  return rerank_model(ctx, body, body_len, props, n_rankings, rankings, out_bytes, out_len);
}

int cco_format_es_bulk(cco_ctx_t *ctx, const cco_result_t *res, int32_t n_names, const char *const *names,
                       const cco_dictionary_t *row_ids, const cco_dictionary_t *col_ids, char **out_bytes, int64_t *out_len) {
  return format_model(ctx, res, n_names, names, row_ids, col_ids, nullptr, 0, nullptr, out_bytes, out_len, "cco:format_es_bulk");
}

int cco_format_model(cco_ctx_t *ctx, const cco_result_t *res, int32_t n_names, const char *const *names, const cco_dictionary_t *row_ids,
                     const cco_dictionary_t *col_ids, const cco_item_properties_t *props, int32_t n_rankings, const cco_ranking_t *rankings,
                     char **out_bytes, int64_t *out_len) {
  return format_model(ctx, res, n_names, names, row_ids, col_ids, props, n_rankings, rankings, out_bytes, out_len, "cco:format_model");
}

// ---- cco_event_log_*: a PredictionIO event export parsed on the device (kernels in cco_events.cuh) ---------------------
// One string column of the log, partitioned by event name (file order inside a name): offsets from 0 and 8-byte words with
// 16 bytes of padding, in HBM; boff[g] = the byte offset of name g's first entry (host copy, n_names + 1 entries).
struct EvCol {
  long long *off = nullptr;
  uint64_t *w = nullptr;
  std::vector<long long> boff;
};
// what one parsed chunk of a streamed read keeps until finish: its retained columns, partitioned by the names known when
// it was parsed (train_at / rank_at: that many names + 1)
struct EvSeg {
  EvCol tu, ti, ri;
  long long *rtime = nullptr;
  long long *tline = nullptr, *rline = nullptr;   // removeDuplicates: the global line of each training / ranking entry
  long long *ttime = nullptr;                       // history retention: each training entry's time (and tline its line)
  long long *tkey = nullptr;                        // interned ids: each training entry's (user key << 32 | item key)
  std::vector<long long> train_at, rank_at;
};
// the intern table of one id column (CCO_LOG_INTERN_IDS; kernels in cco_intern.cuh): key k's string is the heap's bytes
// [off[k], off[k + 1]) (words w, 16 bytes of padding), its hash hash[k]; table: cap slots, each a key or kStrEmpty
struct InternTable {
  long long n = 0, kcap = 0;        // keys; capacity of off (+ 1) and hash
  long long bytes = 0, bcap = 0;    // heap bytes; capacity of w (+ 16 bytes)
  long long cap = 0;
  long long *off = nullptr;
  uint64_t *w = nullptr, *hash = nullptr;
  uint32_t *table = nullptr;
  DevStrCol heap() const {
    DevStrCol v;
    v.n = n;
    v.off = off;
    v.w = w;
    return v;
  }
};
extern "C++" {
namespace cco {
struct SnapImage;
struct SnapLoad;
void snap_delete(SnapImage *);
void snap_delete(SnapLoad *);
struct SnapFree {
  template <typename T>
  void operator()(T *p) const { snap_delete(p); }
};
}  // namespace cco
}  // extern "C++"
struct cco_event_log {
  cco_ctx *ctx = nullptr;
  long long n_lines = 0, n_prop = 0, n_ignored = 0;
  std::vector<int64_t> name_off;   // the distinct event names, first appearance order
  std::string name_bytes;
  std::vector<int64_t> n_train, n_rank;        // per name
  std::vector<long long> train_at, rank_at;    // per name + 1: first event of the name in the partitioned columns
  EvCol tu, ti, ri;                            // training users, training items, ranking items
  long long *rtime = nullptr;                  // ranking event times, partitioned as ri
  // the aggregated properties: n_triples (item, field, value text) triples in HBM (cco_item_properties_t's columns,
  // offsets from 0), the field names on the host
  long long n_prop_items = 0, n_prop_fields = 0, n_triples = 0;
  int32_t *p_field = nullptr;
  long long *p_voff = nullptr, *p_ioff = nullptr, p_ibytes_n = 0;
  unsigned char *p_vals = nullptr, *p_ibytes = nullptr;
  std::vector<std::string> field_names;
  std::vector<void *> dev;                     // what to free
  std::vector<size_t> dev_bytes;               // the bytes of each (cco_event_log_resident_bytes)
  // the read in progress (cco_event_log_begin / _append / _finish): staging of cap bytes (+ 24 of padding) holding
  // `staged` bytes, the last '\n' among them at last_nl (-1: none); lines parsed so far; per chunk one segment; the
  // property-event lines (each ending in '\n') and their global lines, aggregated at finish
  unsigned char *stage = nullptr;
  long long cap = 0, staged = 0, last_nl = -1;
  std::vector<EvSeg> segs;
  std::unordered_map<std::string, int> name_code;
  unsigned char *pb = nullptr;
  long long pb_len = 0, pb_cap = 0;
  std::vector<long long> prop_line;
  // the eventWindow (cco_event_log_begin_window): lines at or before cutoff expire ($set / $unset excepted); with dedup
  // each retained line leaves a WinRec (n_rec of them) for removeDuplicates at finish, and the layout keeps each
  // retained entry's global line (tline / rline) until the columns are compacted
  long long cutoff = INT64_MIN;
  bool dedup = false;
  long long n_expired = 0, n_dup = 0;
  WinRec *rec = nullptr;
  long long n_rec = 0, rec_cap = 0;
  long long *tline = nullptr, *rline = nullptr;
  // history retention (CCO_LOG_KEEP_HISTORY): every training entry's time and global line, partitioned as tu / ti; tline
  // then outlives finish
  bool history = false;
  long long *ttime = nullptr;
  // interned ids (CCO_LOG_INTERN_IDS): one table for the users and one for the items of the training entries, and tkey
  // (user key << 32 | item key) per training entry, partitioned as tu / ti.  After every finish the tables hold exactly
  // the ids of the retained entries.  intern_mask: the context's cco_debug_intern_hash_bits when the read began.
  bool intern = false;
  uint64_t intern_mask = ~0ULL;
  InternTable users, items;
  long long *tkey = nullptr;
  // extendable logs (CCO_LOG_EXTENDABLE): rec (one record per retained line, with or without dedup), tline / rline and the
  // property lines (pb, prop_line) outlive finish; dup_time holds the eventTimes of the non-exempt lines removeDuplicates
  // dropped, which a later cutoff turns into expired lines; chunk0 is the staging cco_event_log_extend reopens with
  bool extendable = false;
  long long chunk0 = 0;
  long long *dup_time = nullptr;
  long long n_dup_time = 0;
  long long n_erased = 0;                      // retained lines cco_event_log_erase took out, over the log's life
  // the property events' item ids, which a log read without CCO_LOG_EXTENDABLE keeps after the aggregation (a snapshot
  // carries them, so that a loaded log holds the bytes the saved one holds)
  EvCol pitem;
  // snapshots (cco_event_log_save / cco_event_log_load_*): the image of the finished log, built at the first save call
  // after a finish; the state of a load in progress
  std::unique_ptr<cco::SnapImage, cco::SnapFree> snap;
  std::unique_ptr<cco::SnapLoad, cco::SnapFree> load;
  bool finished = false;
  int cleaners = 0;                            // open cco_event_log_clean_begin cleaners: extend and free refuse meanwhile
  int fail = CCO_OK;                           // a failed append / finish: every later call returns it with fail_msg
  std::string fail_msg;
  int code_of(const char *name) const {
    const size_t n = strlen(name);
    for (size_t g = 0; g + 1 < name_off.size(); ++g)
      if ((size_t)(name_off[g + 1] - name_off[g]) == n && !memcmp(name_bytes.data() + name_off[g], name, n)) return (int)g;
    return -1;
  }
  // the entries [at[g], at[g] + n) of a column as a string column the ingest and key kernels read (no copy)
  DevStrCol view(const EvCol &col, int g, const std::vector<long long> &at, long long n) const {
    DevStrCol v;
    v.n = g >= 0 ? n : 0;
    const long long b0 = g >= 0 ? col.boff[g] : 0;
    v.base = b0 & ~7LL;
    v.off = col.off + (g >= 0 ? at[g] : 0);
    v.w = col.w + v.base / 8;
    return v;
  }
};

namespace cco {
static void event_log_release(cco_event_log *lg) {
  if (!lg) return;
  cudaSetDevice(lg->ctx->device);
  for (void *p : lg->dev) cudaFreeAsync(p, lg->ctx->stream);
  cudaStreamSynchronize(lg->ctx->stream);
  delete lg;
}
static int event_error(unsigned long long err) {
  const long long line = (long long)(err >> 8);
  switch ((unsigned)(err & 0xff)) {
    case kJsonLongLine: return set_error(CCO_E_UNSUPPORTED, "line %lld: longer than 2^31 - 1 bytes", line);
    case kJsonNotObject: return set_error(CCO_E_INVALID_ARG, "line %lld: not a JSON object (a blank line is not an event)", line);
    case kJsonString:
      return set_error(CCO_E_INVALID_ARG, "line %lld: a string is unterminated or holds a bad escape or a raw byte < 0x20", line);
    case kEvMissing:
      return set_error(CCO_E_INVALID_ARG, "line %lld: an event needs \"event\", \"entityType\", \"entityId\" and \"eventTime\"", line);
    case kEvType:
      return set_error(CCO_E_INVALID_ARG, "line %lld: a member has the wrong type (event, entityType, entityId, eventTime: string; "
                       "targetEntityType, targetEntityId: string or null; properties: object)", line);
    case kEvTime_:
      return set_error(CCO_E_INVALID_ARG, "line %lld: eventTime is not YYYY-MM-DDThh:mm:ss[.fraction](Z|+hh:mm|+hhmm|+hh)", line);
    case kEvEmptyId: return set_error(CCO_E_INVALID_ARG, "line %lld: Empty user or item ID", line);
    case kEvTarget: return set_error(CCO_E_INVALID_ARG, "line %lld: targetEntityType and targetEntityId must be given together", line);
    default:
      return set_error(CCO_E_INVALID_ARG, "line %lld: not one JSON object (unbalanced brackets or an unexpected token)", line);
  }
}
static int log_keep(Arena &ar, cco_event_log *lg, void *p) {
  lg->dev_bytes.push_back(ar.take(p));
  lg->dev.push_back(p);
  return CCO_OK;
}
// a buffer the log kept, freed before the log is
static void log_drop(cco_event_log *lg, void *p) {
  for (size_t i = 0; p && i < lg->dev.size(); ++i)
    if (lg->dev[i] == p) {
      cudaFreeAsync(p, lg->ctx->stream);
      lg->dev.erase(lg->dev.begin() + i);
      lg->dev_bytes.erase(lg->dev_bytes.begin() + i);
      return;
    }
}
// a buffer kept by the log grown to cap (+ pad) entries, its first keep entries copied; the old one is freed
extern "C++" {
template <typename T>
static int log_grow(cco_event_log *lg, Arena &ar, T **buf, long long cap, long long keep, long long pad) {
  T *p;
  CKR(ar.alloc(&p, cap + pad));
  CKR(log_keep(ar, lg, p));
  if (keep > 0) CK(cudaMemcpyAsync(p, *buf, sizeof(T) * (size_t)keep, cudaMemcpyDeviceToDevice, lg->ctx->stream));
  log_drop(lg, *buf);
  *buf = p;
  return CCO_OK;
}
}  // extern "C++"
// the entries i < n with keep[i] != 0, in order -> idx[0 .. count); the count stays on the device in (*pos)[n].  keep
// has n + 1 entries.
static int select_flagged(cco_ctx *c, Arena &ar, long long n, uint32_t *keep, uint32_t **pos, uint32_t **idx) {
  CKR(ar.alloc(pos, n + 1));
  CKR(ar.alloc(idx, n));
  CK(cudaMemsetAsync(keep + n, 0, 4, c->stream));
  CKR(exclusive_sum(c, ar, (const uint32_t *)keep, *pos, n + 1));
  k_win_scatter<<<grid_for(n, 256, c->sm_count), 256, 0, c->stream>>>(n, keep, *pos, *idx);
  c->launches++;
  return CCO_OK;
}
// the lines carrying flag bit `want` by event name, file order inside a name -> idx[0 .. count)
static int event_partition(cco_ctx *c, Arena &ar, long long L, const uint8_t *flag, uint8_t want, const int32_t *code, uint32_t n_names,
                           uint32_t **idx) {
  uint32_t *key;
  CKR(ar.alloc(&key, L));
  CKR(ar.alloc(idx, L));
  k_event_keys<<<grid_for(L, 256, c->sm_count), 256, 0, c->stream>>>(L, flag, want, code, n_names, key, *idx);
  c->launches++;
  CKR(sort_pairs(c, ar, L, &key, idx, bits_for((long long)n_names + 1)));
  ar.release(key);
  return CCO_OK;
}
// boff[g] = off[at[g]]: the byte offset of each name's first entry in a column, on the host
static int name_boff(cco_ctx *c, Arena &ar, const long long *off, const std::vector<long long> &at, std::vector<long long> *boff) {
  cudaStream_t s = c->stream;
  boff->assign(at.size(), 0);
  std::vector<uint32_t> at32(at.begin(), at.end());
  uint32_t *d_at;
  long long *d_b;
  CKR(ar.alloc(&d_at, at.size()));
  CKR(ar.alloc(&d_b, at.size()));
  CK(cudaMemcpyAsync(d_at, at32.data(), sizeof(uint32_t) * at.size(), cudaMemcpyHostToDevice, s));
  k_gather_i64<<<grid_for((long long)at.size(), 256, c->sm_count), 256, 0, s>>>((long long)at.size(), d_at, off, d_b);
  c->launches++;
  CK(cudaMemcpyAsync(boff->data(), d_b, sizeof(long long) * at.size(), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));   // at32 is a local
  return CCO_OK;
}
// member k's string of the listed lines decoded into a column kept by the log; boff at the names' first entries
static int event_column(cco_ctx *c, Arena &ar, cco_event_log *lg, long long n, const uint32_t *idx, int k, const long long *sb,
                        const int2 *span, const unsigned char *body, const std::vector<long long> &at, EvCol *col) {
  cudaStream_t s = c->stream;
  JMember *jm;
  CKR(ar.alloc(&jm, std::max<long long>(n, 1)));
  if (n > 0) {
    k_event_strings<<<grid_for(n, 256, c->sm_count), 256, 0, s>>>(n, idx, k, sb, span, body, jm);
    c->launches++;
  }
  DevStrCol d;
  long long nb = 0;
  CKR(json_decode(c, ar, n, jm, body, &d, &nb));
  ar.release(jm);
  ar.release(d.hash);
  CKR(log_keep(ar, lg, d.off));
  CKR(log_keep(ar, lg, d.w));
  col->off = d.off;
  col->w = d.w;
  return name_boff(c, ar, d.off, at, &col->boff);
}

// PEventStore.aggregateProperties over the property events ($set / $unset / $delete of items) of a read log, in
// (eventTime, line) order: a $set merges its members (the later value of a field wins), a $unset removes the fields it
// names, a $delete drops what the item had.  Result, kept by the log: (item, field, value text) triples in the order of
// the items' first property event (line order), each item's fields in the order their names first appear among the
// members of $set / $unset properties; an item whose final state exists without a field gets one triple of the field "id"
// (never written: "id" wins) so that it has a document and is a random-rank candidate.  Values are the members' trimmed
// JSON text, spliced verbatim.  Field numbers follow first appearance in the triples.  gline[l]: the global line of line l,
// named by an error.
static int event_properties(cco_ctx *c, Arena &ar, cco_event_log *lg, long long L, const uint8_t *flag, const long long *tm,
                            const long long *sb, const int2 *span, const unsigned char *bb, const long long *gline) {
  cudaStream_t s = c->stream;
  const long long NP = lg->n_prop;
  uint32_t *keep, *pos, *pl;   // property event -> line, line order
  CKR(ar.alloc(&keep, L + 1));
  k_win_flag_keep<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, flag, kEvProperty, keep);
  c->launches++;
  CKR(select_flagged(c, ar, L, keep, &pos, &pl));
  ar.release(keep);
  ar.release(pos);
  // items, grouped exactly in order of first appearance
  EvCol pcol;
  CKR(event_column(c, ar, lg, NP, pl, kEvEntityId, sb, span, bb, std::vector<long long>{0, NP}, &pcol));
  DevStrCol pc;
  pc.n = NP;
  pc.off = pcol.off;
  pc.w = pcol.w;
  CKR(ar.alloc(&pc.hash, NP));
  str_hash(c, pc, ~0ULL);
  int32_t *pg;
  CKR(ar.alloc(&pg, NP));
  StrTable it;
  CKR(str_group(c, ar, pc, nullptr, false, 0, &it, pg));
  const long long G = it.n_groups;
  // kinds, and each event's position in the (eventTime, line) order (a stable sort by time of events in line order)
  uint8_t *pk;
  long long *pt;
  CKR(ar.alloc(&pk, NP));
  CKR(ar.alloc(&pt, NP));
  k_gather_u8<<<grid_for(NP, 256, c->sm_count), 256, 0, s>>>(NP, pl, flag, pk);
  k_gather_i64<<<grid_for(NP, 256, c->sm_count), 256, 0, s>>>(NP, pl, tm, pt);
  unsigned long long *tk;
  uint32_t *tv;
  CKR(ar.alloc(&tk, NP));
  CKR(ar.alloc(&tv, NP));
  k_prop_time_keys<<<grid_for(NP, 256, c->sm_count), 256, 0, s>>>(NP, pt, tk, tv);
  c->launches += 3;
  CKR(sort_pairs(c, ar, NP, &tk, &tv, 64));
  int32_t *ord, *last_del, *last_set;
  CKR(ar.alloc(&ord, NP));
  CKR(ar.alloc(&last_del, G));
  CKR(ar.alloc(&last_set, G));
  CK(cudaMemsetAsync(last_del, 0xff, sizeof(int32_t) * (size_t)G, s));
  CK(cudaMemsetAsync(last_set, 0xff, sizeof(int32_t) * (size_t)G, s));
  k_prop_scatter_ord<<<grid_for(NP, 256, c->sm_count), 256, 0, s>>>(NP, tv, ord);
  k_prop_last<<<grid_for(NP, 256, c->sm_count), 256, 0, s>>>(NP, pk, pg, ord, last_del, last_set);
  unsigned long long *cnt, h_cnt[2] = {0, 0};
  CKR(ar.alloc(&cnt, 2));
  CK(cudaMemsetAsync(cnt, 0, 16, s));
  k_prop_counts<<<grid_for(std::max(NP, G), 256, c->sm_count), 256, 0, s>>>(NP, pk, kEvPropObj, G, last_del, last_set, cnt);
  c->launches += 3;
  CKR(mail_fetch(c, h_cnt, cnt, 16));
  CKR(mail_wait(c));
  const long long Q = (long long)h_cnt[0];
  lg->n_prop_items = (long long)h_cnt[1];
  // members of the properties objects of $set / $unset events; the verdict names the line
  uint32_t *qi;
  CKR(ar.alloc(&keep, NP + 1));
  k_win_flag_keep<<<grid_for(NP, 256, c->sm_count), 256, 0, s>>>(NP, pk, kEvPropObj, keep);
  c->launches++;
  CKR(select_flagged(c, ar, NP, keep, &pos, &qi));
  ar.release(keep);
  ar.release(pos);
  long long *qb, *qe, *moff, M = 0;
  unsigned long long h_err = 0;
  CKR(ar.alloc(&qb, std::max<long long>(Q, 1)));
  CKR(ar.alloc(&qe, std::max<long long>(Q, 1)));
  if (Q > 0) {
    k_prop_spans<<<grid_for(Q, 256, c->sm_count), 256, 0, s>>>(Q, qi, pl, sb, span, qb, qe);
    c->launches++;
  }
  JMember *mem;
  CKR(json_members(c, ar, Q, qb, qe, bb, 0x7fffffffLL - G, &h_err, &moff, &mem, &M));
  if (h_err != ~0ULL) {
    uint32_t q = 0, line = 0;
    CK(cudaMemcpy(&q, qi + (h_err >> 8), 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(&line, pl + q, 4, cudaMemcpyDeviceToHost));
    return event_error(((unsigned long long)gline[line] << 8) | (h_err & 0xff));
  }
  if (M + G >= 0x7fffffffLL) return set_error(CCO_E_UNSUPPORTED, "%lld property members, at most 2^31 - 2 with the items", M);
  uint32_t *mev;
  int32_t *mf;
  CKR(ar.alloc(&mev, std::max<long long>(M, 1)));
  CKR(ar.alloc(&mf, std::max<long long>(M, 1)));
  if (M > 0) {
    k_prop_member_event<<<grid_for(Q, 256, c->sm_count), 256, 0, s>>>(Q, moff, qi, mev);
    c->launches++;
  }
  // field names decoded and grouped exactly; the few distinct ones go to the host once
  DevStrCol nm;
  long long nm_bytes = 0;
  CKR(json_decode(c, ar, M, mem, bb, &nm, &nm_bytes));
  str_hash(c, nm, ~0ULL);
  StrTable ft;
  CKR(str_group(c, ar, nm, nullptr, false, 0, &ft, mf));
  const long long NF = ft.n_groups;
  cco_dictionary_t fd;
  CKR(str_dictionary(c, ar, nm, ft, &fd));
  CK(cudaStreamSynchronize(s));
  std::vector<std::string> fname;
  for (long long f = 0; f < NF; ++f) fname.emplace_back(fd.bytes + fd.offsets[f], (size_t)(fd.offsets[f + 1] - fd.offsets[f]));
  c->pinned_put((void *)fd.offsets);
  c->pinned_put((void *)fd.bytes);
  // members in (eventTime, line, member) order, then stably by (item, field) with one presence entry per item last
  const long long N = M + G;
  uint32_t *k1, *v1, *v2;
  unsigned long long *k2;
  CKR(ar.alloc(&k1, std::max<long long>(M, 1)));
  CKR(ar.alloc(&v1, std::max<long long>(M, 1)));
  CKR(ar.alloc(&k2, N + 1));
  CKR(ar.alloc(&v2, N + 1));
  if (M > 0) {
    k_prop_keys1<<<grid_for(M, 256, c->sm_count), 256, 0, s>>>(M, mev, ord, k1, v1);
    c->launches++;
    CKR(sort_pairs(c, ar, M, &k1, &v1, bits_for(NP)));
  }
  k_prop_keys2<<<grid_for(N, 256, c->sm_count), 256, 0, s>>>(M, G, v1, mev, pg, mf, k2, v2);
  c->launches++;
  CKR(sort_pairs(c, ar, N, &k2, &v2, 32 + bits_for(G)));
  uint32_t *has;
  CKR(ar.alloc(&keep, N + 1));
  CKR(ar.alloc(&pos, N + 1));
  CKR(ar.alloc(&has, G));
  CK(cudaMemsetAsync(has, 0, sizeof(uint32_t) * (size_t)G, s));
  CK(cudaMemsetAsync(keep + N, 0, 4, s));
  k_prop_win<<<grid_for(N, 256, c->sm_count), 256, 0, s>>>(M, G, k2, v2, mev, pk, ord, last_del, keep, has);
  k_prop_presence<<<grid_for(N, 256, c->sm_count), 256, 0, s>>>(M, G, k2, last_del, last_set, has, keep);
  c->launches += 2;
  CKR(exclusive_sum(c, ar, keep, pos, N + 1));
  uint32_t T = 0;
  CKR(mail_fetch(c, &T, pos + N, 4));
  CKR(mail_wait(c));
  lg->n_triples = T;
  auto drop_items = [&] {   // an extendable log aggregates at every finish: the item column goes once the triples are built
    if (!lg->extendable) {
      lg->pitem.off = pcol.off;
      lg->pitem.w = pcol.w;
      return;
    }
    log_drop(lg, pcol.off);
    log_drop(lg, pcol.w);
  };
  if (T == 0) {
    drop_items();
    return CCO_OK;
  }
  uint32_t *titem, *first;
  int32_t *tfield;
  long long *vb, *ve;
  CKR(ar.alloc(&titem, T));
  CKR(ar.alloc(&tfield, T));
  CKR(ar.alloc(&vb, T));
  CKR(ar.alloc(&ve, T));
  CKR(ar.alloc(&first, NF + 1));
  CK(cudaMemsetAsync(first, 0xff, sizeof(uint32_t) * (size_t)(NF + 1), s));
  k_prop_triples<<<grid_for(N, 256, c->sm_count), 256, 0, s>>>(M, G, keep, pos, k2, v2, mev, it.first_sorted, mem, (int32_t)NF, titem, tfield,
                                                             vb, ve, first);
  c->launches++;
  // field numbers by first appearance in the triples; the presence field is "id" (a property of that name included)
  std::vector<uint32_t> h_first((size_t)NF + 1);
  CK(cudaMemcpyAsync(h_first.data(), first, sizeof(uint32_t) * h_first.size(), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  long long f_id = NF;
  for (long long f = 0; f < NF; ++f)
    if (fname[f] == "id") f_id = f;
  // a property named "id" is a field of the aggregated properties only if some item keeps it
  const bool id_kept = f_id < NF && h_first[f_id] != ~0u, presence = h_first[NF] != ~0u;
  h_first[f_id] = std::min(h_first[f_id], h_first[NF]);
  std::vector<long long> used;
  for (long long f = 0; f < NF; ++f)
    if (h_first[f] != ~0u) used.push_back(f);
  if (f_id == NF && h_first[NF] != ~0u) used.push_back(NF);
  std::sort(used.begin(), used.end(), [&](long long a, long long b) { return h_first[a] < h_first[b]; });
  std::vector<int32_t> remap((size_t)NF + 1, 0);
  lg->field_names.clear();
  for (size_t k = 0; k < used.size(); ++k) {
    remap[used[k]] = (int32_t)k;
    lg->field_names.push_back(used[k] == NF ? std::string("id") : fname[used[k]]);
  }
  remap[NF] = remap[f_id];
  lg->n_prop_fields = (long long)used.size() - (presence && !id_kept ? 1 : 0);
  int32_t *d_remap;
  CKR(ar.alloc(&d_remap, NF + 1));
  CK(cudaMemcpyAsync(d_remap, remap.data(), sizeof(int32_t) * remap.size(), cudaMemcpyHostToDevice, s));
  k_remap_i32<<<grid_for(T, 256, c->sm_count), 256, 0, s>>>(T, d_remap, tfield);
  // value texts and item ids of the triples as columns (offsets from 0)
  long long *len, *voff, *ioff, vtotal = 0, itotal = 0;
  CKR(ar.alloc(&len, (long long)T + 1));
  CKR(ar.alloc(&voff, (long long)T + 1));
  CKR(ar.alloc(&ioff, (long long)T + 1));
  CK(cudaMemsetAsync(len + T, 0, 8, s));
  k_prop_value_len<<<grid_for(T, 256, c->sm_count), 256, 0, s>>>(T, vb, ve, len);
  CKR(exclusive_sum(c, ar, len, voff, (long long)T + 1));
  k_str_dict_len<<<grid_for(T, 256, c->sm_count), 256, 0, s>>>(T, titem, pcol.off, len);
  CKR(exclusive_sum(c, ar, len, ioff, (long long)T + 1));
  c->launches += 3;
  CKR(mail_fetch(c, &vtotal, voff + T, 8));
  CKR(mail_fetch(c, &itotal, ioff + T, 8));
  CKR(mail_wait(c));
  unsigned char *vals, *ibytes;
  CKR(ar.alloc(&vals, std::max<long long>(vtotal, 1)));
  CKR(ar.alloc(&ibytes, std::max<long long>(itotal, 1)));
  k_prop_value_copy<<<grid_for(T, 256, c->sm_count), 256, 0, s>>>(T, vb, voff, bb, vals);
  k_str_dict_gather<<<grid_for(T, 256, c->sm_count), 256, 0, s>>>(T, titem, pcol.off, 0, (const unsigned char *)pcol.w, ioff, ibytes);
  c->launches += 2;
  for (void *p : {(void *)tfield, (void *)voff, (void *)vals, (void *)ioff, (void *)ibytes}) CKR(log_keep(ar, lg, p));
  lg->p_field = tfield;
  lg->p_voff = voff;
  lg->p_vals = vals;
  lg->p_ioff = ioff;
  lg->p_ibytes = ibytes;
  lg->p_ibytes_n = itotal;
  drop_items();
  return CCO_OK;
}

// steps 2-4 of a read over the len bytes of w (bytes [len, round_up(len, 8) + 16) are zero): lines (every '\n' ends one;
// open_tail: a last line without it ends at len), the seven members an event is read through, then types, times and the
// selection.  Each verdict comes before anything reads through the parsed spans; an error names the global line
// line_base + l.
struct EvLines {
  long long L = 0;
  long long *sb = nullptr, *se = nullptr, *tm = nullptr;
  int2 *span = nullptr;
  int2 *xspan = nullptr;   // with_x: the spans of "prId" and "tags" (EventSinkX)
  uint8_t *flag = nullptr;
};
static int event_lines(cco_ctx *c, Arena &ar, const uint64_t *w, long long len, bool open_tail, long long line_base, EvLines *ev,
                       bool with_x = false) {
  cudaStream_t s = c->stream;
  const unsigned char *bb = (const unsigned char *)w;
  const unsigned long long base = (unsigned long long)line_base << 8;
  CKR(split_lines(c, ar, w, len, open_tail, &ev->L, &ev->sb, &ev->se));
  const long long L = ev->L;
  if (L > 0x7fffffffLL) return set_error(CCO_E_UNSUPPORTED, "%lld lines in one parsed chunk, at most 2^31 - 1", L);
  if (L == 0) return CCO_OK;
  unsigned long long *err, h_err = 0;
  CKR(ar.alloc(&ev->span, L * kEvSlots));
  CKR(ar.alloc(&err, 1));
  CK(cudaMemsetAsync(ev->span, 0xff, sizeof(int2) * (size_t)L * kEvSlots, s));
  CK(cudaMemsetAsync(err, 0xff, 8, s));
  if (with_x) {
    CKR(ar.alloc(&ev->xspan, L * kEvXSlots));
    CK(cudaMemsetAsync(ev->xspan, 0xff, sizeof(int2) * (size_t)L * kEvXSlots, s));
    k_json_members<<<grid_for(L * 32, 256, c->sm_count), 256, 0, s>>>(L, ev->sb, ev->se, bb, EventSinkX{ev->span, ev->xspan, bb}, err);
  } else {
    k_json_members<<<grid_for(L * 32, 256, c->sm_count), 256, 0, s>>>(L, ev->sb, ev->se, bb, EventSink{ev->span, bb}, err);
  }
  c->launches++;
  CKR(mail_fetch(c, &h_err, err, 8));
  CKR(mail_wait(c));
  if (h_err != ~0ULL) return event_error(h_err + base);
  CKR(ar.alloc(&ev->flag, L));
  CKR(ar.alloc(&ev->tm, L));
  k_event_check<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, ev->sb, ev->span, bb, ev->flag, ev->tm, err);
  c->launches++;
  CKR(mail_fetch(c, &h_err, err, 8));
  CKR(mail_wait(c));
  if (h_err != ~0ULL) return event_error(h_err + base);
  return CCO_OK;
}

// zero the word that holds byte `len` of a buffer and the 16 bytes after it, so that the newline passes, which read whole
// words, see no stale byte past len
static int event_pad(cco_ctx *c, unsigned char *buf, long long len) {
  CK(cudaMemsetAsync(buf + len, 0, (size_t)(((len + 7) & ~7LL) + 16 - len), c->stream));
  return CCO_OK;
}

// removeDuplicates: the global line of each of the n entries of a chunk's column (idx: the chunk lines), kept by the log
static int win_entry_lines(cco_event_log *lg, Arena &ar, long long n, const uint32_t *idx, long long base, long long **out) {
  CKR(ar.alloc(out, std::max<long long>(n, 1)));
  CKR(log_keep(ar, lg, *out));
  if (n > 0) {
    k_win_lines<<<grid_for(n, 256, lg->ctx->sm_count), 256, 0, lg->ctx->stream>>>(n, idx, base, *out);
    lg->ctx->launches++;
  }
  return CCO_OK;
}
// removeDuplicates, per chunk: the identity hash of every retained line (not expired) into lg->rec.  The identity is the
// decoded event, entityType, entityId, targetEntityType, targetEntityId and prId (null = absent), the tags text (absent,
// null = []) and the set of the properties' top-level members (decoded name, trimmed value text; the last of a repeated
// name; absent = {}).  A properties object the tokenizer cannot split (the line is read all the same) is its text.
// win_idents: the records of the R chunk lines ridx (bytes bb) -> out[0 .. R); win_records also in the event log's cleaner
static int win_idents(cco_ctx *c, Arena &ar, const EvLines &ev, const unsigned char *bb, const int32_t *code, long long base, long long R,
                      const uint32_t *ridx, WinRec *out);
static int win_records(cco_event_log *lg, Arena &ar, const EvLines &ev, const int32_t *code, long long base) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  const long long L = ev.L;
  uint32_t *keep, *pos, *ridx;
  CKR(ar.alloc(&keep, L + 1));
  k_win_keep_lines<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, ev.flag, keep);
  c->launches++;
  CKR(select_flagged(c, ar, L, keep, &pos, &ridx));
  uint32_t R32 = 0;
  CKR(mail_fetch(c, &R32, pos + L, 4));
  CKR(mail_wait(c));
  ar.release(keep);
  ar.release(pos);
  const long long R = R32;
  if (R == 0) return CCO_OK;
  if (lg->n_rec + R > lg->rec_cap) {   // grow geometrically
    lg->rec_cap = std::max(2 * lg->rec_cap, lg->n_rec + R);
    CKR(log_grow(lg, ar, &lg->rec, lg->rec_cap, lg->n_rec, 0));
  }
  CKR(win_idents(c, ar, ev, lg->stage, code, base, R, ridx, lg->rec + lg->n_rec));
  lg->n_rec += R;
  return CCO_OK;
}
static int win_idents(cco_ctx *c, Arena &ar, const EvLines &ev, const unsigned char *bb, const int32_t *code, long long base, long long R,
                      const uint32_t *ridx, WinRec *out) {
  cudaStream_t s = c->stream;
  // the properties' members: count pass with each span's verdict, then the members of the well-formed spans
  long long *pb, *pe, *mcnt, *moff;
  int *codes;
  unsigned long long *err;
  CKR(ar.alloc(&pb, R));
  CKR(ar.alloc(&pe, R));
  CKR(ar.alloc(&mcnt, R + 1));
  CKR(ar.alloc(&moff, R + 1));
  CKR(ar.alloc(&codes, R));
  CKR(ar.alloc(&err, 1));
  CK(cudaMemsetAsync(mcnt + R, 0, 8, s));
  k_win_prop_spans<<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, ridx, ev.sb, ev.span, pb, pe);
  k_json_members<<<grid_for(R * 32, 256, c->sm_count), 256, 0, s>>>(R, pb, pe, bb, WinMemberSink<false>{mcnt, codes, nullptr, nullptr}, err);
  c->launches += 2;
  CKR(exclusive_sum(c, ar, mcnt, moff, R + 1));
  long long M = 0;
  CKR(mail_fetch(c, &M, moff + R, 8));
  CKR(mail_wait(c));
  JMember *mem;
  CKR(ar.alloc(&mem, std::max<long long>(M, 1)));
  if (M > 0) {
    k_json_members<<<grid_for(R * 32, 256, c->sm_count), 256, 0, s>>>(R, pb, pe, bb, WinMemberSink<true>{nullptr, codes, moff, mem}, err);
    c->launches++;
  }
  // decoded strings (six per line, then the member names) and raw texts (tags, unsplit properties, member values), hashed
  const long long ND = kWinStr * R + M, NR = 2 * R + M;
  JMember *jm;
  CKR(ar.alloc(&jm, ND));
  k_win_strings<<<grid_for(ND, 256, c->sm_count), 256, 0, s>>>(R, ridx, ev.sb, ev.span, ev.xspan, bb, M, mem, jm);
  c->launches++;
  DevStrCol d;
  long long d_bytes = 0;
  CKR(json_decode(c, ar, ND, jm, bb, &d, &d_bytes));
  ar.release(jm);
  ulonglong2 *hd, *hr;
  long long *rb, *re;
  CKR(ar.alloc(&hd, ND));
  CKR(ar.alloc(&hr, NR));
  CKR(ar.alloc(&rb, NR));
  CKR(ar.alloc(&re, NR));
  k_win_hash<<<grid_for(ND * 32, 256, c->sm_count), 256, 0, s>>>(ND, d.off, d.off + 1, d.w, hd);
  k_win_raw_ranges<<<grid_for(NR, 256, c->sm_count), 256, 0, s>>>(R, ridx, ev.sb, ev.span, ev.xspan, codes, M, mem, rb, re);
  k_win_hash<<<grid_for(NR * 32, 256, c->sm_count), 256, 0, s>>>(NR, rb, re, (const uint64_t *)bb, hr);
  c->launches += 3;
  str_release(ar, d);
  // the set of members: the last of each (line, name) -- sorted by name hash, then stably by line -- summed per line
  unsigned long long *acc;
  CKR(ar.alloc(&acc, 2 * R));
  CK(cudaMemsetAsync(acc, 0, sizeof(unsigned long long) * 2 * (size_t)R, s));
  if (M > 0) {
    uint32_t *mline, *v, *k32;
    unsigned long long *k64;
    CKR(ar.alloc(&mline, M));
    CKR(ar.alloc(&v, M));
    CKR(ar.alloc(&k64, M));
    CKR(ar.alloc(&k32, M));
    k_win_member_line<<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, moff, mline);
    k_win_name_keys<<<grid_for(M, 256, c->sm_count), 256, 0, s>>>(M, hd + kWinStr * R, k64, v);
    c->launches += 2;
    CKR(sort_pairs(c, ar, M, &k64, &v, 64));
    k_win_line_keys<<<grid_for(M, 256, c->sm_count), 256, 0, s>>>(M, v, mline, k32);
    c->launches++;
    CKR(sort_pairs(c, ar, M, &k32, &v, bits_for(R)));
    k_win_props<<<grid_for(M, 256, c->sm_count), 256, 0, s>>>(M, v, mline, hd + kWinStr * R, hr + 2 * R, acc);
    c->launches++;
  }
  k_win_ident<<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, ridx, base, ev.sb, ev.span, ev.xspan, bb, hd, hr, codes, acc, ev.tm, ev.flag,
                                                          code, out);
  c->launches++;
  return CCO_OK;
}
// extendable logs without removeDuplicates, per chunk: what expiry needs of every retained line (a WinRec without a hash)
static int ext_records(cco_event_log *lg, Arena &ar, const EvLines &ev, const int32_t *code, long long base) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  const long long L = ev.L;
  uint32_t *keep, *pos, *ridx, R32 = 0;
  CKR(ar.alloc(&keep, L + 1));
  k_win_keep_lines<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, ev.flag, keep);
  c->launches++;
  CKR(select_flagged(c, ar, L, keep, &pos, &ridx));
  CKR(mail_fetch(c, &R32, pos + L, 4));
  CKR(mail_wait(c));
  const long long R = R32;
  if (R == 0) return CCO_OK;
  if (lg->n_rec + R > lg->rec_cap) {   // grow geometrically
    lg->rec_cap = std::max(2 * lg->rec_cap, lg->n_rec + R);
    CKR(log_grow(lg, ar, &lg->rec, lg->rec_cap, lg->n_rec, 0));
  }
  k_ext_line_recs<<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, ridx, base, ev.tm, ev.flag, code, lg->rec + lg->n_rec);
  c->launches++;
  lg->n_rec += R;
  return CCO_OK;
}

// ---- interned logs: intern tables per chunk and their refit at finish (kernels in cco_intern.cuh) --------------------------
// the slots of a table for n keys: a power of two, at most half full
static long long intern_slots(long long n) {
  long long cap = 64;
  while (cap < 2 * n) cap <<= 1;
  return cap;
}
// tb's keys in a new table of cap slots, inserted from their stored hashes; the old table is freed
static int intern_rehash(cco_event_log *lg, Arena &ar, InternTable *tb, long long cap) {
  cco_ctx *c = lg->ctx;
  uint32_t *t;
  CKR(ar.alloc(&t, cap));
  CKR(log_keep(ar, lg, t));
  CK(cudaMemsetAsync(t, 0xff, sizeof(uint32_t) * (size_t)cap, c->stream));
  if (tb->n > 0) {
    k_intern_rehash<<<grid_for(tb->n, 256, c->sm_count), 256, 0, c->stream>>>(tb->n, tb->hash, (uint64_t)cap - 1, t);
    c->launches++;
  }
  log_drop(lg, tb->table);
  tb->table = t;
  tb->cap = cap;
  return CCO_OK;
}
// the n ids of one column of a chunk's segment interned into tb: the strings new to tb take the next keys in the order
// of their first entry, their bytes join the heap; each entry's key -> half[2 i]
static int intern_column(cco_event_log *lg, Arena &ar, InternTable *tb, const EvCol &col, long long n, uint32_t *half) {
  if (n == 0) return CCO_OK;
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  if (intern_slots(tb->n + n) > tb->cap) CKR(intern_rehash(lg, ar, tb, intern_slots(tb->n + n)));
  uint64_t *hash;
  uint32_t *slot_of, *flag, *pos, *idx, K = 0;
  CKR(ar.alloc(&hash, n));
  CKR(ar.alloc(&slot_of, n));
  CKR(ar.alloc(&flag, n + 1));
  k_str_hash<<<grid_for(n, 256, c->sm_count), 256, 0, s>>>(n, col.off, 0, col.w, lg->intern_mask, hash);
  k_intern_claim<<<grid_for(n, 256, c->sm_count), 256, 0, s>>>(n, col.off, col.w, hash, tb->off, tb->w, tb->hash, (uint64_t)tb->cap - 1,
                                                               tb->table, slot_of);
  k_intern_first<<<grid_for(n, 256, c->sm_count), 256, 0, s>>>(n, slot_of, tb->table, flag);
  c->launches += 3;
  CKR(select_flagged(c, ar, n, flag, &pos, &idx));
  CKR(mail_fetch(c, &K, pos + n, 4));
  CKR(mail_wait(c));
  if (tb->n + K >= (long long)kInternNew) return set_error(CCO_E_UNSUPPORTED, "%lld distinct ids: an interned log takes < 2^31", tb->n + K);
  if (K > 0) {
    long long *len, *noff, total = 0;
    CKR(ar.alloc(&len, (long long)K + 1));
    CKR(ar.alloc(&noff, (long long)K + 1));
    CK(cudaMemsetAsync(len + K, 0, 8, s));
    k_str_dict_len<<<grid_for(K, 256, c->sm_count), 256, 0, s>>>(K, idx, col.off, len);
    c->launches++;
    CKR(exclusive_sum(c, ar, len, noff, (long long)K + 1));
    CKR(mail_fetch(c, &total, noff + K, 8));
    CKR(mail_wait(c));
    if (tb->n + K > tb->kcap) {   // grow geometrically
      const long long kc = std::max(2 * tb->kcap, tb->n + K);
      CKR(log_grow(lg, ar, &tb->off, kc, tb->n > 0 ? tb->n + 1 : 0, 1));
      CKR(log_grow(lg, ar, &tb->hash, kc, tb->n, 0));
      tb->kcap = kc;
    }
    if (tb->bytes + total > tb->bcap) {
      const long long bc = std::max(2 * tb->bcap, tb->bytes + total);
      CKR(log_grow(lg, ar, &tb->w, (bc + 7) / 8, (tb->bytes + 7) / 8, 2));
      tb->bcap = bc;
    }
    k_intern_new<<<grid_for(K, 256, c->sm_count), 256, 0, s>>>(K, idx, slot_of, hash, (uint32_t)tb->n, tb->table, tb->hash);
    k_intern_heap_off<<<grid_for((long long)K + 1, 256, c->sm_count), 256, 0, s>>>(K, noff, tb->bytes, tb->off + tb->n);
    c->launches += 2;
    if (total > 0) {
      k_str_dict_gather<<<grid_for(K, 256, c->sm_count), 256, 0, s>>>(K, idx, col.off, 0, (const unsigned char *)col.w, noff,
                                                                      (unsigned char *)tb->w + tb->bytes);
      c->launches++;
    }
    tb->n += K;
    tb->bytes += total;
  }
  k_intern_keys<<<grid_for(n, 256, c->sm_count), 256, 0, s>>>(n, slot_of, tb->table, half);
  c->launches++;
  CK(cudaStreamSynchronize(s));
  return CCO_OK;
}
// the keys live[k] != 0 of tb kept, renumbered in key order (pos: their new numbers, idx: the old key of each new one):
// the heap and hashes gathered as exact fits, the table rebuilt at intern_slots of the count
static int intern_refit_table(cco_event_log *lg, Arena &ar, InternTable *tb, const uint32_t *pos, const uint32_t *idx) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  uint32_t K = 0;
  long long total = 0;
  CK(cudaMemcpyAsync(&K, pos + tb->n, 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  long long *len, *off;
  uint64_t *w, *h;
  CKR(ar.alloc(&len, (long long)K + 1));
  CKR(ar.alloc(&off, (long long)K + 1));
  CK(cudaMemsetAsync(len + K, 0, 8, s));
  if (K > 0) {
    k_str_dict_len<<<grid_for(K, 256, c->sm_count), 256, 0, s>>>(K, idx, tb->off, len);
    c->launches++;
  }
  CKR(exclusive_sum(c, ar, len, off, (long long)K + 1));
  CK(cudaMemcpyAsync(&total, off + K, 8, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CKR(ar.alloc(&w, (total + 16 + 7) / 8));
  CKR(ar.alloc(&h, std::max<long long>(K, 1)));
  if (K > 0) {
    if (total > 0) {
      k_str_dict_gather<<<grid_for(K, 256, c->sm_count), 256, 0, s>>>(K, idx, tb->off, 0, (const unsigned char *)tb->w, off, (unsigned char *)w);
      c->launches++;
    }
    k_gather_i64<<<grid_for(K, 256, c->sm_count), 256, 0, s>>>(K, idx, (const long long *)tb->hash, (long long *)h);
    c->launches++;
  }
  for (void *p : {(void *)off, (void *)w, (void *)h}) CKR(log_keep(ar, lg, p));
  for (void *p : {(void *)tb->off, (void *)tb->w, (void *)tb->hash}) log_drop(lg, p);
  tb->off = off;
  tb->w = w;
  tb->hash = h;
  tb->n = tb->kcap = K;
  tb->bytes = tb->bcap = total;
  return intern_rehash(lg, ar, tb, intern_slots(K));
}
// at the end of every finish: the tables keep exactly the ids of the retained training entries, sized by their counts only
static int intern_refit(cco_event_log *lg) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  Arena ar(s);
  const long long E = lg->train_at.back();
  InternTable *tbs[2] = {&lg->users, &lg->items};
  uint32_t *live[2], *pos[2], *idx[2];
  for (int x = 0; x < 2; ++x) {
    CKR(ar.alloc(&live[x], tbs[x]->n + 1));
    CK(cudaMemsetAsync(live[x], 0, sizeof(uint32_t) * (size_t)(tbs[x]->n + 1), s));
  }
  if (E > 0) {
    k_intern_live<<<grid_for(E, 256, c->sm_count), 256, 0, s>>>(E, (const unsigned long long *)lg->tkey, live[0], live[1]);
    c->launches++;
  }
  for (int x = 0; x < 2; ++x) CKR(select_flagged(c, ar, tbs[x]->n, live[x], &pos[x], &idx[x]));
  if (E > 0) {
    k_intern_remap<<<grid_for(E, 256, c->sm_count), 256, 0, s>>>(E, pos[0], pos[1], (unsigned long long *)lg->tkey);
    c->launches++;
  }
  for (int x = 0; x < 2; ++x) CKR(intern_refit_table(lg, ar, tbs[x], pos[x], idx[x]));
  CK(cudaStreamSynchronize(s));
  return CCO_OK;
}

// the event names of a chunk's lines: decoded and grouped exactly -> *code (each line's group, numbered by first
// appearance in the chunk) and the groups' names on the host
static int chunk_names(cco_ctx *c, Arena &ar, const EvLines &ev, const unsigned char *bb, int32_t **code, std::vector<std::string> *out) {
  cudaStream_t s = c->stream;
  const long long L = ev.L;
  JMember *jm;
  CKR(ar.alloc(&jm, L));
  k_event_strings<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, nullptr, kEvName, ev.sb, ev.span, bb, jm);
  c->launches++;
  DevStrCol names;
  long long name_bytes = 0;
  CKR(json_decode(c, ar, L, jm, bb, &names, &name_bytes));
  ar.release(jm);
  str_hash(c, names, ~0ULL);
  CKR(ar.alloc(code, L));
  StrTable nt;
  CKR(str_group(c, ar, names, nullptr, false, 0, &nt, *code));
  const long long NC = nt.n_groups;
  cco_dictionary_t nd;
  CKR(str_dictionary(c, ar, names, nt, &nd));
  CK(cudaStreamSynchronize(s));
  out->clear();
  for (long long k = 0; k < NC; ++k) out->emplace_back(nd.bytes + nd.offsets[k], (size_t)(nd.offsets[k + 1] - nd.offsets[k]));
  c->pinned_put((void *)nd.offsets);
  c->pinned_put((void *)nd.bytes);
  str_table_release(ar, nt);
  str_release(ar, names);
  return CCO_OK;
}
// code[l] = remap[code[l]] for the L lines of a chunk
static int chunk_remap(cco_ctx *c, Arena &ar, long long L, const std::vector<int32_t> &remap, int32_t *code) {
  cudaStream_t s = c->stream;
  int32_t *d_remap;
  CKR(ar.alloc(&d_remap, (long long)remap.size()));
  CK(cudaMemcpyAsync(d_remap, remap.data(), sizeof(int32_t) * remap.size(), cudaMemcpyHostToDevice, s));
  k_remap_i32<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, d_remap, code);
  c->launches++;
  return CCO_OK;
}

// one chunk of a streamed read, the first len staged bytes: every line parsed, the names numbered globally, the counts
// added, the training and ranking events decoded into one new segment, the property-event lines appended to lg->pb
static int event_chunk(cco_event_log *lg, long long len, bool open_tail) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  mail_reset(c);
  Arena ar(s);
  CKR(event_pad(c, lg->stage, len));
  EvLines ev;
  const long long base = lg->n_lines;
  CKR(event_lines(c, ar, (const uint64_t *)lg->stage, len, open_tail, base, &ev, lg->dedup));
  const long long L = ev.L;
  if (L == 0) return CCO_OK;
  const unsigned char *bb = lg->stage;
  if (lg->cutoff != INT64_MIN) {   // the eventWindow's duration: expired lines lose their selection
    unsigned long long *nx, h_nx = 0;
    CKR(ar.alloc(&nx, 1));
    CK(cudaMemsetAsync(nx, 0, 8, s));
    k_win_expire<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, ev.sb, ev.span, bb, ev.tm, lg->cutoff, ev.flag, nx);
    c->launches++;
    CKR(mail_fetch(c, &h_nx, nx, 8));
    CKR(mail_wait(c));
    lg->n_expired += (long long)h_nx;
  }
  // 5. event names: decoded, grouped exactly, numbered by first appearance in the chunk; the few distinct ones go to the
  // host, where names new to the log take the next codes (chunks arrive in order: the order of the whole read)
  int32_t *code;
  std::vector<std::string> cnames;
  CKR(chunk_names(c, ar, ev, bb, &code, &cnames));
  std::vector<int32_t> remap(cnames.size());
  for (size_t k = 0; k < cnames.size(); ++k) {
    const std::string &nm = cnames[k];
    auto it = lg->name_code.find(nm);
    if (it == lg->name_code.end()) {
      it = lg->name_code.emplace(nm, (int)lg->name_off.size() - 1).first;
      lg->name_bytes += nm;
      lg->name_off.push_back((int64_t)lg->name_bytes.size());
    }
    remap[k] = it->second;
  }
  const long long NG = (long long)lg->name_off.size() - 1;
  CKR(chunk_remap(c, ar, L, remap, code));
  // 6. counts per name
  unsigned long long *cnt;
  CKR(ar.alloc(&cnt, 2 * NG + 2));
  CK(cudaMemsetAsync(cnt, 0, sizeof(unsigned long long) * (size_t)(2 * NG + 2), s));
  k_event_counts<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, ev.flag, code, (int32_t)NG, cnt);
  c->launches++;
  std::vector<unsigned long long> h_cnt((size_t)(2 * NG + 2));
  CK(cudaMemcpyAsync(h_cnt.data(), cnt, sizeof(unsigned long long) * h_cnt.size(), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));   // remap and h_cnt are locals
  lg->n_train.resize(NG, 0);
  lg->n_rank.resize(NG, 0);
  lg->segs.emplace_back();
  EvSeg &sg = lg->segs.back();
  sg.train_at.assign(NG + 1, 0);
  sg.rank_at.assign(NG + 1, 0);
  for (long long n = 0; n < NG; ++n) {
    lg->n_train[n] += (int64_t)h_cnt[2 * n];
    lg->n_rank[n] += (int64_t)h_cnt[2 * n + 1];
    sg.train_at[n + 1] = sg.train_at[n] + (long long)h_cnt[2 * n];
    sg.rank_at[n + 1] = sg.rank_at[n] + (long long)h_cnt[2 * n + 1];
  }
  const long long NP = (long long)h_cnt[2 * NG];
  lg->n_prop += NP;
  lg->n_ignored += (long long)h_cnt[2 * NG + 1];
  lg->n_lines += L;
  if (lg->dedup) CKR(win_records(lg, ar, ev, code, base));
  else if (lg->extendable) CKR(ext_records(lg, ar, ev, code, base));
  // 7. training and ranking events partitioned by name, file order inside a name: decoded ids and times
  uint32_t *idx;
  CKR(event_partition(c, ar, L, ev.flag, kEvTraining, code, (uint32_t)NG, &idx));
  CKR(event_column(c, ar, lg, sg.train_at[NG], idx, kEvEntityId, ev.sb, ev.span, bb, sg.train_at, &sg.tu));
  CKR(event_column(c, ar, lg, sg.train_at[NG], idx, kEvTargetId, ev.sb, ev.span, bb, sg.train_at, &sg.ti));
  if (lg->dedup || lg->history || lg->extendable) CKR(win_entry_lines(lg, ar, sg.train_at[NG], idx, base, &sg.tline));
  if (lg->intern) {   // the chunk's lines have their verdicts: its training ids take their keys
    const long long NT = sg.train_at[NG];
    CKR(ar.alloc(&sg.tkey, std::max<long long>(NT, 1)));
    CKR(log_keep(ar, lg, sg.tkey));
    CKR(intern_column(lg, ar, &lg->users, sg.tu, NT, (uint32_t *)sg.tkey + 1));
    CKR(intern_column(lg, ar, &lg->items, sg.ti, NT, (uint32_t *)sg.tkey));
  }
  if (lg->history) {
    const long long NT = sg.train_at[NG];
    CKR(ar.alloc(&sg.ttime, std::max<long long>(NT, 1)));
    CKR(log_keep(ar, lg, sg.ttime));
    if (NT > 0) {
      k_gather_i64<<<grid_for(NT, 256, c->sm_count), 256, 0, s>>>(NT, idx, ev.tm, sg.ttime);
      c->launches++;
    }
  }
  ar.release(idx);
  CKR(event_partition(c, ar, L, ev.flag, kEvRanking, code, (uint32_t)NG, &idx));
  const long long NR = sg.rank_at[NG];
  CKR(event_column(c, ar, lg, NR, idx, kEvTargetId, ev.sb, ev.span, bb, sg.rank_at, &sg.ri));
  CKR(ar.alloc(&sg.rtime, std::max<long long>(NR, 1)));
  CKR(log_keep(ar, lg, sg.rtime));
  if (NR > 0) {
    k_gather_i64<<<grid_for(NR, 256, c->sm_count), 256, 0, s>>>(NR, idx, ev.tm, sg.rtime);
    c->launches++;
  }
  if (lg->dedup || lg->extendable) CKR(win_entry_lines(lg, ar, NR, idx, base, &sg.rline));
  ar.release(idx);
  // 8. the property-event lines, in line order, for the aggregation at finish (see event_log_finish)
  if (NP > 0) {
    uint32_t *keep, *pos;
    CKR(ar.alloc(&keep, L + 1));
    k_win_flag_keep<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, ev.flag, kEvProperty, keep);
    c->launches++;
    CKR(select_flagged(c, ar, L, keep, &pos, &idx));
    long long *len8, *off;
    CKR(ar.alloc(&len8, NP + 1));
    CKR(ar.alloc(&off, NP + 1));
    CK(cudaMemsetAsync(len8 + NP, 0, 8, s));
    k_line_len<<<grid_for(NP, 256, c->sm_count), 256, 0, s>>>(NP, idx, ev.sb, ev.se, len8);
    c->launches++;
    CKR(exclusive_sum(c, ar, len8, off, NP + 1));
    long long total = 0;
    std::vector<uint32_t> h_idx((size_t)NP);
    CK(cudaMemcpyAsync(&total, off + NP, 8, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(h_idx.data(), idx, sizeof(uint32_t) * (size_t)NP, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    if (lg->pb_len + total > lg->pb_cap) {   // grow geometrically; 24 bytes of padding for event_pad
      lg->pb_cap = std::max(2 * lg->pb_cap, lg->pb_len + total);
      CKR(log_grow(lg, ar, &lg->pb, lg->pb_cap, lg->pb_len, 24));
    }
    k_line_gather<<<grid_for(NP * 32, 256, c->sm_count), 256, 0, s>>>(NP, idx, ev.sb, ev.se, bb, off, lg->pb + lg->pb_len);
    c->launches++;
    lg->pb_len += total;
    for (uint32_t l : h_idx) lg->prop_line.push_back(base + (long long)l);
  }
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  return CCO_OK;
}

// one retained column of every segment, concatenated name-major (segments in order inside a name) into *out; the
// segments' buffers of the column are freed as soon as it is built, so that the peak stays near one column above the
// retained bytes.  at: each segment's entry offsets per name (train_at or rank_at); gat: the same for the whole log.
static int event_cat_column(cco_event_log *lg, EvCol EvSeg::*col, std::vector<long long> EvSeg::*at, const std::vector<long long> &gat,
                            EvCol *out) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  Arena ar(s);
  const long long NG = (long long)gat.size() - 1;
  std::vector<CatPiece> bytes, ents;
  out->boff.assign(NG + 1, 0);
  long long b = 0, e = 0;
  for (long long g = 0; g < NG; ++g) {
    out->boff[g] = b;
    for (EvSeg &sg : lg->segs) {
      const std::vector<long long> &sa = sg.*at;
      if (g + 1 >= (long long)sa.size()) continue;   // a name first seen in a later chunk
      const EvCol &sc = sg.*col;
      CatPiece p{sc.w, sc.off, sc.boff[g], b, sc.boff[g + 1] - sc.boff[g], sa[g], e, sa[g + 1] - sa[g], true};
      if (p.nb > 0) bytes.push_back(p);
      if (p.ne > 0) ents.push_back(p);
      b += p.nb;
      e += p.ne;
    }
  }
  out->boff[NG] = b;
  const long long NW = (b + 7) / 8 + 2;
  CKR(ar.alloc(&out->off, e + 1));
  CKR(ar.alloc(&out->w, NW));
  CatPiece *d_p;
  CKR(ar.alloc(&d_p, bytes.size() + ents.size()));
  CK(cudaMemcpyAsync(d_p, bytes.data(), sizeof(CatPiece) * bytes.size(), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(d_p + bytes.size(), ents.data(), sizeof(CatPiece) * ents.size(), cudaMemcpyHostToDevice, s));
  k_cat_words<<<grid_for(NW, 256, c->sm_count), 256, 0, s>>>(NW, b, d_p, (int)bytes.size(), out->w);
  k_cat_entries<<<grid_for(e + 1, 256, c->sm_count), 256, 0, s>>>(e, b, d_p + bytes.size(), (int)ents.size(), out->off);
  c->launches += 2;
  CK(cudaStreamSynchronize(s));   // the pieces are locals
  CKR(log_keep(ar, lg, out->off));
  CKR(log_keep(ar, lg, out->w));
  for (EvSeg &sg : lg->segs) {
    log_drop(lg, (sg.*col).off);
    log_drop(lg, (sg.*col).w);
  }
  return CCO_OK;
}
// one per-entry column of every segment (the ranking times; with removeDuplicates also the entries' global lines),
// name-major, as the string columns of the same partition (at)
static int event_cat_times(cco_event_log *lg, long long **out, long long *EvSeg::*col = &EvSeg::rtime,
                           std::vector<long long> EvSeg::*at = &EvSeg::rank_at) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  Arena ar(s);
  const long long NG = (long long)lg->name_off.size() - 1;
  std::vector<CatPiece> ents;
  long long e = 0;
  for (long long g = 0; g < NG; ++g)
    for (EvSeg &sg : lg->segs) {
      const std::vector<long long> &sa = sg.*at;
      if (g + 1 >= (long long)sa.size() || sa[g + 1] == sa[g]) continue;
      ents.push_back(CatPiece{nullptr, sg.*col, 0, 0, 0, sa[g], e, sa[g + 1] - sa[g], false});
      e += ents.back().ne;
    }
  CKR(ar.alloc(out, std::max<long long>(e, 1)));
  CatPiece *d_p;
  CKR(ar.alloc(&d_p, ents.size()));
  CK(cudaMemcpyAsync(d_p, ents.data(), sizeof(CatPiece) * ents.size(), cudaMemcpyHostToDevice, s));
  if (e > 0) {
    k_cat_entries<<<grid_for(e, 256, c->sm_count), 256, 0, s>>>(e, -1, d_p, (int)ents.size(), *out);
    c->launches++;
  }
  CK(cudaStreamSynchronize(s));
  CKR(log_keep(ar, lg, *out));
  for (EvSeg &sg : lg->segs) log_drop(lg, sg.*col);
  return CCO_OK;
}

// the drop bitmap over the global lines, kept by the log until finish ends
static int win_bitmap(cco_event_log *lg, Arena &ar, uint32_t **bitmap) {
  const long long words = lg->n_lines / 32 + 1;
  CKR(ar.alloc(bitmap, words));
  CKR(log_keep(ar, lg, *bitmap));
  CK(cudaMemsetAsync(*bitmap, 0, sizeof(uint32_t) * (size_t)words, lg->ctx->stream));
  return CCO_OK;
}
// removeDuplicates at finish: the records of every chunk sorted by (hash, time desc, line desc); all but the first of each
// run are dropped -> *bitmap over the global lines (made here when null); *n_prop_drop += the property lines among the
// drops, *n_new = all of them.
// An extendable log keeps its records (ext_split_records takes the dropped ones out).
static int win_mark(cco_event_log *lg, uint32_t **bitmap, long long *n_prop_drop, long long *n_new) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  Arena ar(s);
  const long long N = lg->n_rec, NG = (long long)lg->name_off.size() - 1;
  if (!*bitmap) CKR(win_bitmap(lg, ar, bitmap));
  std::vector<unsigned long long> h_cnt((size_t)(2 * NG + 3), 0);
  if (N > 1) {
    unsigned long long *key, *cnt;
    uint32_t *val;
    CKR(ar.alloc(&key, N));
    CKR(ar.alloc(&val, N));
    k_win_key_time<<<grid_for(N, 256, c->sm_count), 256, 0, s>>>(N, lg->rec, key, val);
    c->launches++;
    CKR(sort_pairs(c, ar, N, &key, &val, 64));
    for (int high : {1, 0}) {
      k_win_key_hash<<<grid_for(N, 256, c->sm_count), 256, 0, s>>>(N, lg->rec, val, high, key);
      c->launches++;
      CKR(sort_pairs(c, ar, N, &key, &val, 64));
    }
    CKR(ar.alloc(&cnt, 2 * NG + 3));
    CK(cudaMemsetAsync(cnt, 0, sizeof(unsigned long long) * h_cnt.size(), s));
    k_win_mark<<<grid_for(N, 256, c->sm_count), 256, 0, s>>>(N, lg->rec, val, (int32_t)NG, *bitmap, cnt);
    c->launches++;
    CK(cudaMemcpyAsync(h_cnt.data(), cnt, sizeof(unsigned long long) * h_cnt.size(), cudaMemcpyDeviceToHost, s));
  }
  CK(cudaStreamSynchronize(s));
  *n_prop_drop += (long long)h_cnt[2 * NG];
  lg->n_prop -= (long long)h_cnt[2 * NG];
  lg->n_ignored -= (long long)h_cnt[2 * NG + 1];
  *n_new = (long long)h_cnt[2 * NG + 2];
  lg->n_dup += *n_new;
  if (!lg->extendable) {
    log_drop(lg, lg->rec);
    lg->rec = nullptr;
  }
  return CCO_OK;
}

// ---- extendable logs: the retained part under a later cutoff (kernels k_ext_* in cco_events.cuh) ---------------------------
// per event name: 1 for "$set" and "$unset", which never expire
static int ext_exempt(cco_event_log *lg, Arena &ar, uint8_t **out) {
  const long long NG = (long long)lg->name_off.size() - 1;
  std::vector<uint8_t> h((size_t)std::max<long long>(NG, 1), 0);
  for (long long g = 0; g < NG; ++g) {
    const std::string nm(lg->name_bytes.data() + lg->name_off[g], (size_t)(lg->name_off[g + 1] - lg->name_off[g]));
    h[g] = nm == "$set" || nm == "$unset";
  }
  CKR(ar.alloc(out, h.size()));
  CK(cudaMemcpyAsync(*out, h.data(), h.size(), cudaMemcpyHostToDevice, lg->ctx->stream));
  CK(cudaStreamSynchronize(lg->ctx->stream));   // h is a local
  return CCO_OK;
}
// the records idx[0 .. K) become the log's records (an exact fit: expired and dropped ones are freed)
static int ext_keep_records(cco_event_log *lg, Arena &ar, long long K, const uint32_t *idx) {
  cco_ctx *c = lg->ctx;
  WinRec *r;
  CKR(ar.alloc(&r, std::max<long long>(K, 1)));
  if (K > 0) {
    k_ext_gather_rec<<<grid_for(K, 256, c->sm_count), 256, 0, c->stream>>>(K, idx, lg->rec, r);
    c->launches++;
  }
  CKR(log_keep(ar, lg, r));
  log_drop(lg, lg->rec);
  lg->rec = r;
  lg->n_rec = lg->rec_cap = K;
  return CCO_OK;
}
// the cutoff applied to what earlier finishes retained: a record at or before it whose name is not exempt expires (its
// line goes into *bitmap, made here), and an earlier duplicate drop at or before it counts as expired from now on, as a
// whole read under this cutoff counts it.  *n_x: the lines that expired, *n_px: of them property events.  The lines
// parsed since the last finish were judged under this cutoff already and pass unchanged.
static int ext_expire(cco_event_log *lg, const uint8_t *exempt, uint32_t **bitmap, long long *n_x, long long *n_px) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  Arena ar(s);
  CKR(win_bitmap(lg, ar, bitmap));
  *n_x = *n_px = 0;
  const long long N = lg->n_rec, D = lg->n_dup_time;
  if (lg->cutoff == INT64_MIN || (N == 0 && D == 0)) return CCO_OK;
  unsigned long long *cnt, h_cnt[4] = {0, 0, 0, 0};
  uint32_t *keep, *pos, *idx, *dkeep, *dpos, *didx, K = 0, KD = 0;
  CKR(ar.alloc(&cnt, 4));
  CK(cudaMemsetAsync(cnt, 0, sizeof(h_cnt), s));
  CKR(ar.alloc(&keep, N + 1));
  CKR(ar.alloc(&dkeep, D + 1));
  if (N > 0) {
    k_ext_expire<<<grid_for(N, 256, c->sm_count), 256, 0, s>>>(N, lg->rec, lg->cutoff, exempt, *bitmap, keep, cnt);
    c->launches++;
  }
  CKR(select_flagged(c, ar, N, keep, &pos, &idx));
  if (D > 0) {
    k_ext_expire_times<<<grid_for(D, 256, c->sm_count), 256, 0, s>>>(D, lg->dup_time, lg->cutoff, dkeep, cnt + 3);
    c->launches++;
  }
  CKR(select_flagged(c, ar, D, dkeep, &dpos, &didx));
  CK(cudaMemcpyAsync(h_cnt, cnt, sizeof(h_cnt), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(&K, pos + N, 4, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(&KD, dpos + D, 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (h_cnt[0] > 0) CKR(ext_keep_records(lg, ar, K, idx));
  if (h_cnt[3] > 0) {
    long long *t;
    CKR(ar.alloc(&t, std::max<uint32_t>(KD, 1)));
    if (KD > 0) {
      k_gather_i64<<<grid_for(KD, 256, c->sm_count), 256, 0, s>>>(KD, didx, lg->dup_time, t);
      c->launches++;
    }
    CKR(log_keep(ar, lg, t));
    log_drop(lg, lg->dup_time);
    lg->dup_time = t;
    lg->n_dup_time = KD;
  }
  CK(cudaStreamSynchronize(s));
  *n_x = (long long)h_cnt[0];
  *n_px = (long long)h_cnt[1];
  lg->n_expired += (long long)(h_cnt[0] + h_cnt[3]);
  lg->n_dup -= (long long)h_cnt[3];
  lg->n_prop -= (long long)h_cnt[1];
  lg->n_ignored -= (long long)h_cnt[2];
  return CCO_OK;
}
// after win_mark: the records whose line it dropped leave the log; the eventTimes of the non-exempt ones join dup_time
static int ext_split_records(cco_event_log *lg, const uint8_t *exempt, const uint32_t *bitmap) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  Arena ar(s);
  const long long N = lg->n_rec;
  uint32_t *keep, *dup, *pos, *idx, *dpos, *didx, K = 0, KD = 0;
  long long *tm;
  CKR(ar.alloc(&keep, N + 1));
  CKR(ar.alloc(&dup, N + 1));
  CKR(ar.alloc(&tm, N));
  k_ext_dup_split<<<grid_for(N, 256, c->sm_count), 256, 0, s>>>(N, lg->rec, bitmap, exempt, keep, dup, tm);
  c->launches++;
  CKR(select_flagged(c, ar, N, keep, &pos, &idx));
  CKR(select_flagged(c, ar, N, dup, &dpos, &didx));
  CK(cudaMemcpyAsync(&K, pos + N, 4, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(&KD, dpos + N, 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CKR(ext_keep_records(lg, ar, K, idx));
  if (KD > 0) {
    CKR(log_grow(lg, ar, &lg->dup_time, lg->n_dup_time + KD, lg->n_dup_time, 0));
    k_gather_i64<<<grid_for(KD, 256, c->sm_count), 256, 0, s>>>(KD, didx, tm, lg->dup_time + lg->n_dup_time);
    c->launches++;
    lg->n_dup_time += KD;
  }
  CK(cudaStreamSynchronize(s));
  return CCO_OK;
}
// after the aggregation: the property lines that are still selected (ev: pb parsed, dropped lines with flag 0) become pb,
// an exact fit, and prop_line follows them
static int ext_keep_property_lines(cco_event_log *lg, Arena &ar, const EvLines &ev) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  const long long L = ev.L;
  uint32_t *keep, *pos, *idx, K = 0;
  CKR(ar.alloc(&keep, L + 1));
  k_win_flag_keep<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, ev.flag, kEvProperty, keep);
  c->launches++;
  CKR(select_flagged(c, ar, L, keep, &pos, &idx));
  CK(cudaMemcpyAsync(&K, pos + L, 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (K == (uint32_t)L) return CCO_OK;   // nothing left the window
  long long *len8, *off, total = 0;
  CKR(ar.alloc(&len8, (long long)K + 1));
  CKR(ar.alloc(&off, (long long)K + 1));
  CK(cudaMemsetAsync(len8 + K, 0, 8, s));
  if (K > 0) {
    k_line_len<<<grid_for(K, 256, c->sm_count), 256, 0, s>>>(K, idx, ev.sb, ev.se, len8);
    c->launches++;
  }
  CKR(exclusive_sum(c, ar, len8, off, (long long)K + 1));
  std::vector<uint32_t> h_idx((size_t)K);
  CK(cudaMemcpyAsync(&total, off + K, 8, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(h_idx.data(), idx, sizeof(uint32_t) * (size_t)K, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  unsigned char *pb;
  CKR(ar.alloc(&pb, total + 24));
  if (K > 0) {
    k_line_gather<<<grid_for((long long)K * 32, 256, c->sm_count), 256, 0, s>>>(K, idx, ev.sb, ev.se, lg->pb, off, pb);
    c->launches++;
  }
  CKR(log_keep(ar, lg, pb));
  log_drop(lg, lg->pb);
  lg->pb = pb;
  lg->pb_len = lg->pb_cap = total;
  std::vector<long long> pl((size_t)K);
  for (uint32_t k = 0; k < K; ++k) pl[k] = lg->prop_line[h_idx[k]];
  lg->prop_line.swap(pl);
  CK(cudaStreamSynchronize(s));
  return CCO_OK;
}
// a string column's entries idx[0 .. K) gathered into a new column kept by the log (the old one is freed); boff at the
// names' first entries at
static int win_gather_column(cco_event_log *lg, Arena &ar, long long K, const uint32_t *idx, const std::vector<long long> &at, EvCol *col) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  long long *len, *off, total = 0;
  CKR(ar.alloc(&len, K + 1));
  CKR(ar.alloc(&off, K + 1));
  CK(cudaMemsetAsync(len + K, 0, 8, s));
  if (K > 0) {
    k_str_dict_len<<<grid_for(K, 256, c->sm_count), 256, 0, s>>>(K, idx, col->off, len);
    c->launches++;
  }
  CKR(exclusive_sum(c, ar, len, off, K + 1));
  CK(cudaMemcpyAsync(&total, off + K, 8, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  uint64_t *w;
  CKR(ar.alloc(&w, (total + 16 + 7) / 8));
  if (K > 0 && total > 0) {
    k_str_dict_gather<<<grid_for(K, 256, c->sm_count), 256, 0, s>>>(K, idx, col->off, 0, (const unsigned char *)col->w, off, (unsigned char *)w);
    c->launches++;
  }
  CKR(name_boff(c, ar, off, at, &col->boff));
  CKR(log_keep(ar, lg, off));
  CKR(log_keep(ar, lg, w));
  log_drop(lg, col->off);
  log_drop(lg, col->w);
  col->off = off;
  col->w = w;
  return CCO_OK;
}
// the name-partitioned entries whose line survives the bitmap: columns c1 (and c2), the times (nullable) and at, compacted
static int win_compact(cco_event_log *lg, const uint32_t *bitmap, const long long *line, std::vector<long long> &at, EvCol *c1, EvCol *c2,
                       long long **times, long long **times2 = nullptr, long long **times3 = nullptr) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  Arena ar(s);
  const long long n = at.back(), NA = (long long)at.size();
  if (n == 0) return CCO_OK;
  uint32_t *keep, *pos, *idx;
  CKR(ar.alloc(&keep, n + 1));
  k_win_entry_keep<<<grid_for(n, 256, c->sm_count), 256, 0, s>>>(n, line, bitmap, keep);
  c->launches++;
  CKR(select_flagged(c, ar, n, keep, &pos, &idx));
  long long *d_at, *d_nat;
  CKR(ar.alloc(&d_at, NA));
  CKR(ar.alloc(&d_nat, NA));
  CK(cudaMemcpyAsync(d_at, at.data(), sizeof(long long) * (size_t)NA, cudaMemcpyHostToDevice, s));
  k_win_at<<<grid_for(NA, 256, c->sm_count), 256, 0, s>>>(NA, d_at, pos, d_nat);
  c->launches++;
  std::vector<long long> nat((size_t)NA);
  CK(cudaMemcpyAsync(nat.data(), d_nat, sizeof(long long) * (size_t)NA, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));   // at and nat are host vectors
  const long long K = nat.back();
  CKR(win_gather_column(lg, ar, K, idx, nat, c1));
  if (c2) CKR(win_gather_column(lg, ar, K, idx, nat, c2));
  for (long long **tp : {times, times2, times3}) {
    if (!tp) continue;
    long long *t;
    CKR(ar.alloc(&t, std::max<long long>(K, 1)));
    if (K > 0) {
      k_gather_i64<<<grid_for(K, 256, c->sm_count), 256, 0, s>>>(K, idx, *tp, t);
      c->launches++;
    }
    CK(cudaStreamSynchronize(s));
    CKR(log_keep(ar, lg, t));
    log_drop(lg, *tp);
    *tp = t;
  }
  at = nat;
  return CCO_OK;
}
// the property lines gathered for finish lose their selection where dropped; first the members of every properties object
// among them are checked, so that a dropped line fails as it fails without the window (event_properties' error)
static int win_drop_property_lines(cco_event_log *lg, Arena &ar, const EvLines &ev, const uint32_t *bitmap) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  const long long L = ev.L;
  uint32_t *keep, *pos, *qi, Q = 0;
  CKR(ar.alloc(&keep, L + 1));
  k_win_flag_keep<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, ev.flag, kEvPropObj, keep);
  c->launches++;
  CKR(select_flagged(c, ar, L, keep, &pos, &qi));
  CKR(mail_fetch(c, &Q, pos + L, 4));
  CKR(mail_wait(c));
  long long *gl;
  CKR(ar.alloc(&gl, L));
  CK(cudaMemcpyAsync(gl, lg->prop_line.data(), sizeof(long long) * (size_t)L, cudaMemcpyHostToDevice, s));
  if (Q > 0) {
    long long *qb, *qe, *mcnt;
    unsigned long long *err, h_err = 0;
    CKR(ar.alloc(&qb, Q));
    CKR(ar.alloc(&qe, Q));
    CKR(ar.alloc(&mcnt, Q));
    CKR(ar.alloc(&err, 1));
    CK(cudaMemsetAsync(err, 0xff, 8, s));
    k_win_obj_spans<<<grid_for(Q, 256, c->sm_count), 256, 0, s>>>(Q, qi, ev.sb, ev.span, qb, qe);
    k_json_members<<<grid_for((long long)Q * 32, 256, c->sm_count), 256, 0, s>>>(Q, qb, qe, lg->pb, MemberSink<false>{mcnt, nullptr, nullptr}, err);
    c->launches += 2;
    CKR(mail_fetch(c, &h_err, err, 8));
    CKR(mail_wait(c));
    if (h_err != ~0ULL) {
      uint32_t line = 0;
      CK(cudaMemcpy(&line, qi + (h_err >> 8), 4, cudaMemcpyDeviceToHost));
      return event_error(((unsigned long long)lg->prop_line[line] << 8) | (h_err & 0xff));
    }
  }
  k_win_drop_lines<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, gl, bitmap, ev.flag);
  c->launches++;
  CK(cudaStreamSynchronize(s));   // prop_line is read by the copy
  return CCO_OK;
}

// the staging is full: parse it up to its last '\n' and carry the bytes after it to its front, or, when it holds no '\n'
// (one line fills it), double it
static int event_flush(cco_event_log *lg) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  Arena ar(s);
  if (lg->last_nl < 0) {
    if (lg->staged >= (1LL << 31)) return event_error(((unsigned long long)lg->n_lines << 8) | kJsonLongLine);
    lg->cap *= 2;
    return log_grow(lg, ar, &lg->stage, lg->cap, lg->staged, 24);
  }
  const long long P = lg->last_nl + 1, carry = lg->staged - P;
  unsigned char *tmp = nullptr;
  if (carry > 0) {   // through scratch: the carry may overlap its destination
    CKR(ar.alloc(&tmp, carry));
    CK(cudaMemcpyAsync(tmp, lg->stage + P, (size_t)carry, cudaMemcpyDeviceToDevice, s));
  }
  CKR(event_chunk(lg, P, false));
  if (carry > 0) CK(cudaMemcpyAsync(lg->stage, tmp, (size_t)carry, cudaMemcpyDeviceToDevice, s));
  lg->staged = carry;
  lg->last_nl = -1;
  return CCO_OK;
}

static int event_log_begin(cco_ctx *c, int64_t chunk_bytes, cco_event_log **out) {
  CK(cudaSetDevice(c->device));
  cco_event_log *lg = new cco_event_log();
  lg->ctx = c;
  lg->name_off.assign(1, 0);
  lg->train_at.assign(1, 0);
  lg->rank_at.assign(1, 0);
  lg->cap = lg->chunk0 = std::max<int64_t>(chunk_bytes, 1);
  Arena ar(c->stream);
  const int rc = ar.alloc(&lg->stage, lg->cap + 24);
  if (rc != CCO_OK) {
    delete lg;
    return rc;
  }
  log_keep(ar, lg, lg->stage);
  *out = lg;
  return CCO_OK;
}

static int event_log_append(cco_event_log *lg, const char *bytes, int64_t len) {
  cco_ctx *c = lg->ctx;
  CK(cudaSetDevice(c->device));
  NvtxRange nvtx("cco:event_log_append");
  while (len > 0) {
    if (lg->staged == lg->cap) CKR(event_flush(lg));
    const long long take = std::min<long long>(len, lg->cap - lg->staged);
    CK(cudaMemcpyAsync(lg->stage + lg->staged, bytes, (size_t)take, cudaMemcpyHostToDevice, c->stream));
    const void *nl = memrchr(bytes, '\n', (size_t)take);
    if (nl) lg->last_nl = lg->staged + ((const char *)nl - bytes);
    lg->staged += take;
    bytes += take;
    len -= take;
  }
  CK(cudaStreamSynchronize(c->stream));   // the bytes are copied: the caller may reuse its buffer
  return CCO_OK;
}

// the carried tail as the last chunk (its last line need not end in '\n'), the per-name limits, the retained columns
// name-major, then the properties: event_properties once over the property-event lines of every chunk as a small log in
// line order, so that the (eventTime, line) rule sees them as the whole read does
static int event_log_finish(cco_event_log *lg) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  CK(cudaSetDevice(c->device));
  NvtxRange nvtx("cco:event_log_finish");
  if (lg->staged > 0) CKR(event_chunk(lg, lg->staged, lg->last_nl != lg->staged - 1));
  log_drop(lg, lg->stage);
  lg->stage = nullptr;
  lg->staged = 0;
  const long long NG = (long long)lg->name_off.size() - 1;
  lg->train_at.assign(NG + 1, 0);
  lg->rank_at.assign(NG + 1, 0);
  for (long long n = 0; n < NG; ++n) {
    if (lg->n_rank[n] >= 0x7fffffffLL)
      return set_error(CCO_E_UNSUPPORTED, "event name %lld: %lld events, at most 2^31 - 2 per name", n, (long long)lg->n_rank[n]);
    lg->train_at[n + 1] = lg->train_at[n] + lg->n_train[n];
    lg->rank_at[n + 1] = lg->rank_at[n] + lg->n_rank[n];
  }
  uint32_t *drop = nullptr;   // removeDuplicates (and an extendable log's expiry): the dropped global lines
  long long n_prop_drop = 0, n_drop = 0;   // dropped property lines, all dropped lines
  Arena ear(s);
  uint8_t *exempt = nullptr;
  if (lg->extendable) {   // what earlier finishes retained, under the current cutoff
    long long n_x = 0, n_px = 0;
    CKR(ext_exempt(lg, ear, &exempt));
    CKR(ext_expire(lg, exempt, &drop, &n_x, &n_px));
    n_drop += n_x;
    n_prop_drop += n_px;
  }
  if (lg->dedup) {
    long long n_new = 0;
    mail_reset(c);
    CKR(win_mark(lg, &drop, &n_prop_drop, &n_new));
    n_drop += n_new;
    if (lg->extendable && n_new > 0) CKR(ext_split_records(lg, exempt, drop));
  }
  if (lg->segs.size() == 1) {   // one chunk: its segment is the layout
    EvSeg &sg = lg->segs[0];
    lg->tu = sg.tu;
    lg->ti = sg.ti;
    lg->ri = sg.ri;
    lg->rtime = sg.rtime;
    lg->tline = sg.tline;
    lg->rline = sg.rline;
    lg->ttime = sg.ttime;
    lg->tkey = sg.tkey;
  } else if (lg->segs.size() > 1) {
    CKR(event_cat_column(lg, &EvSeg::tu, &EvSeg::train_at, lg->train_at, &lg->tu));
    CKR(event_cat_column(lg, &EvSeg::ti, &EvSeg::train_at, lg->train_at, &lg->ti));
    CKR(event_cat_column(lg, &EvSeg::ri, &EvSeg::rank_at, lg->rank_at, &lg->ri));
    CKR(event_cat_times(lg, &lg->rtime));
    if (lg->dedup || lg->history || lg->extendable) CKR(event_cat_times(lg, &lg->tline, &EvSeg::tline, &EvSeg::train_at));
    if (lg->dedup || lg->extendable) CKR(event_cat_times(lg, &lg->rline, &EvSeg::rline, &EvSeg::rank_at));
    if (lg->history) CKR(event_cat_times(lg, &lg->ttime, &EvSeg::ttime, &EvSeg::train_at));
    if (lg->intern) CKR(event_cat_times(lg, &lg->tkey, &EvSeg::tkey, &EvSeg::train_at));
  }
  lg->segs.clear();
  if (drop && n_drop > 0) {   // the retained columns without the dropped lines' entries
    CKR(win_compact(lg, drop, lg->tline, lg->train_at, &lg->tu, &lg->ti, lg->history ? &lg->ttime : nullptr,
                    lg->history || lg->extendable ? &lg->tline : nullptr, lg->intern ? &lg->tkey : nullptr));
    CKR(win_compact(lg, drop, lg->rline, lg->rank_at, &lg->ri, nullptr, &lg->rtime, lg->extendable ? &lg->rline : nullptr));
    for (long long n = 0; n < NG; ++n) {
      lg->n_train[n] = lg->train_at[n + 1] - lg->train_at[n];
      lg->n_rank[n] = lg->rank_at[n + 1] - lg->rank_at[n];
    }
  }
  if (!lg->history && !lg->extendable) {
    log_drop(lg, lg->tline);
    lg->tline = nullptr;
  }
  if (lg->intern) CKR(intern_refit(lg));
  if (!lg->extendable) {
    log_drop(lg, lg->rline);
    lg->rline = nullptr;
  }
  if (lg->n_prop > 0) {
    mail_reset(c);
    Arena ar(s);
    CKR(event_pad(c, lg->pb, lg->pb_len));
    EvLines ev;
    CKR(event_lines(c, ar, (const uint64_t *)lg->pb, lg->pb_len, false, 0, &ev));   // judged once already
    if (n_prop_drop > 0) CKR(win_drop_property_lines(lg, ar, ev, drop));
    CKR(event_properties(c, ar, lg, ev.L, ev.flag, ev.tm, ev.sb, ev.span, lg->pb, lg->prop_line.data()));
    if (lg->extendable) CKR(ext_keep_property_lines(lg, ar, ev));
    CK(cudaStreamSynchronize(s));
  }
  log_drop(lg, drop);
  if (!lg->extendable || lg->n_prop == 0) {
    log_drop(lg, lg->pb);
    lg->pb = nullptr;
    lg->pb_len = lg->pb_cap = 0;
    lg->prop_line = std::vector<long long>();
  }
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  lg->finished = true;
  return CCO_OK;
}

// a finished extendable log reopened for append / finish: its retained layout becomes the first segment of the next
// finish, which concatenates the new chunks' segments after it name-major, re-expires it under the new cutoff and
// deduplicates it together with them; the aggregated properties are rebuilt then
static int event_log_extend(cco_event_log *lg, const cco_event_window_t *w) {
  cco_ctx *c = lg->ctx;
  CK(cudaSetDevice(c->device));
  NvtxRange nvtx("cco:event_log_extend");
  Arena ar(c->stream);
  lg->cap = lg->chunk0;
  CKR(ar.alloc(&lg->stage, lg->cap + 24));
  CKR(log_keep(ar, lg, lg->stage));
  lg->staged = 0;
  lg->last_nl = -1;
  if (w) lg->cutoff = w->cutoff_ms;
  EvSeg sg;
  sg.tu = lg->tu;
  sg.ti = lg->ti;
  sg.ri = lg->ri;
  sg.rtime = lg->rtime;
  sg.tline = lg->tline;
  sg.rline = lg->rline;
  sg.ttime = lg->ttime;
  sg.tkey = lg->tkey;
  sg.train_at = lg->train_at;
  sg.rank_at = lg->rank_at;
  lg->segs.assign(1, sg);
  for (void *p : {(void *)lg->p_field, (void *)lg->p_voff, (void *)lg->p_vals, (void *)lg->p_ioff, (void *)lg->p_ibytes}) log_drop(lg, p);
  lg->p_field = nullptr;
  lg->p_voff = lg->p_ioff = nullptr;
  lg->p_vals = lg->p_ibytes = nullptr;
  lg->p_ibytes_n = lg->n_triples = lg->n_prop_items = lg->n_prop_fields = 0;
  lg->field_names.clear();
  lg->finished = false;
  return CCO_OK;
}

// ---- cco_event_log_erase: the lines of erased users and items taken out of a finished extendable log (cco_erase.cuh) ----
// one id list of the caller (Arrow layout, checked on the host) on the device as a column with offsets from 0
static int erase_upload(cco_ctx *c, Arena &ar, int64_t n, const int64_t *off, const char *bytes, EvCol *col) {
  std::vector<long long> o((size_t)n + 1, 0);
  for (int64_t i = 1; i <= n; ++i) o[i] = off[i] - off[0];
  CKR(ar.alloc(&col->off, n + 1));
  CKR(ar.alloc(&col->w, (o[n] + 16 + 7) / 8));
  CK(cudaMemcpyAsync(col->off, o.data(), sizeof(long long) * o.size(), cudaMemcpyHostToDevice, c->stream));
  if (o[n] > 0) CK(cudaMemcpyAsync(col->w, bytes + off[0], (size_t)o[n], cudaMemcpyHostToDevice, c->stream));
  CK(cudaStreamSynchronize(c->stream));   // o is a local
  return CCO_OK;
}
// the n ids of col probed in table tb: bit line[i] of bits for each found id (line null: the bit of its key)
static void erase_probe(cco_event_log *lg, long long n, const long long *off, const uint64_t *w, const InternTable &tb, const long long *line,
                        uint32_t *bits) {
  if (n == 0 || tb.n == 0) return;
  cco_ctx *c = lg->ctx;
  k_erase_probe<<<grid_for(n, 256, c->sm_count), 256, 0, c->stream>>>(n, off, w, lg->intern_mask, tb.off, tb.w, tb.hash, (uint64_t)tb.cap - 1,
                                                                       tb.table, line, bits);
  c->launches++;
}
// a zeroed bitmap of n bits in the arena
static int erase_bits(cco_ctx *c, Arena &ar, long long n, uint32_t **bits) {
  const long long words = n / 32 + 1;
  CKR(ar.alloc(bits, words));
  CK(cudaMemsetAsync(*bits, 0, sizeof(uint32_t) * (size_t)words, c->stream));
  return CCO_OK;
}
// Mark, then drop through the extend's finish pipeline: the records, the training and ranking columns, the property lines and
// their aggregation, the intern tables.  Nothing marked: the log is left untouched, its snapshot image included.
static int event_log_erase(cco_event_log *lg, int64_t n_users, const int64_t *user_off, const char *user_bytes, int64_t n_items,
                           const int64_t *item_off, const char *item_bytes, cco_event_erase_stats_t *stats) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  CK(cudaSetDevice(c->device));
  NvtxRange nvtx("cco:event_log_erase");
  mail_reset(c);
  Arena ar(s);
  EvCol eu, ei;
  CKR(erase_upload(c, ar, n_users, user_off, user_bytes, &eu));
  CKR(erase_upload(c, ar, n_items, item_off, item_bytes, &ei));
  uint32_t *drop = nullptr;
  CKR(win_bitmap(lg, ar, &drop));
  // the erase sets: intern tables of the ids, their buffers the log's until the erase ends
  InternTable su, si;
  uint32_t *half;
  CKR(ar.alloc(&half, 2 * std::max<int64_t>(std::max(n_users, n_items), 1)));
  auto drop_set = [&](InternTable &tb) {
    for (void *p : {(void *)tb.off, (void *)tb.w, (void *)tb.hash, (void *)tb.table}) log_drop(lg, p);
  };
  auto release = [&] {
    drop_set(su);
    drop_set(si);
    log_drop(lg, drop);
  };
  int rc = [&]() -> int {
    const long long E = lg->train_at.back(), R = lg->rank_at.back();
    CKR(intern_column(lg, ar, &si, ei, n_items, half));
    if (lg->intern) {   // the erase ids' keys in the log's own tables, then 8 bytes per training entry
      uint32_t *ub, *ib;
      CKR(erase_bits(c, ar, lg->users.n, &ub));
      CKR(erase_bits(c, ar, lg->items.n, &ib));
      erase_probe(lg, n_users, eu.off, eu.w, lg->users, nullptr, ub);
      erase_probe(lg, n_items, ei.off, ei.w, lg->items, nullptr, ib);
      if (E > 0 && (n_users > 0 || n_items > 0)) {
        k_erase_keys<<<grid_for(E, 256, c->sm_count), 256, 0, s>>>(E, (const unsigned long long *)lg->tkey, ub, ib, lg->tline, drop);
        c->launches++;
      }
    } else {
      CKR(intern_column(lg, ar, &su, eu, n_users, half));
      erase_probe(lg, E, lg->tu.off, lg->tu.w, su, lg->tline, drop);
      erase_probe(lg, E, lg->ti.off, lg->ti.w, si, lg->tline, drop);
    }
    erase_probe(lg, R, lg->ri.off, lg->ri.w, si, lg->rline, drop);
    // property events by their entityId: the retained property lines parsed as every finish parses them
    Arena par(s);
    EvLines ev;
    if (lg->n_prop > 0 && si.n > 0) {
      CKR(event_pad(c, lg->pb, lg->pb_len));
      CKR(event_lines(c, par, (const uint64_t *)lg->pb, lg->pb_len, false, 0, &ev));
      JMember *jm;
      CKR(par.alloc(&jm, ev.L));
      k_event_strings<<<grid_for(ev.L, 256, c->sm_count), 256, 0, s>>>(ev.L, nullptr, kEvEntityId, ev.sb, ev.span, lg->pb, jm);
      c->launches++;
      DevStrCol ids;
      long long nb = 0;
      CKR(json_decode(c, par, ev.L, jm, lg->pb, &ids, &nb));
      long long *gl;
      CKR(par.alloc(&gl, ev.L));
      CK(cudaMemcpyAsync(gl, lg->prop_line.data(), sizeof(long long) * (size_t)ev.L, cudaMemcpyHostToDevice, s));
      erase_probe(lg, ev.L, ids.off, ids.w, si, gl, drop);
      CK(cudaStreamSynchronize(s));   // prop_line is read by the copy
    }
    // the records of the marked lines: nothing marked leaves the log as it was
    const long long N = lg->n_rec;
    unsigned long long *cnt, h_cnt[3] = {0, 0, 0};
    uint32_t *keep, *pos, *idx, K = 0;
    CKR(ar.alloc(&cnt, 3));
    CK(cudaMemsetAsync(cnt, 0, sizeof(h_cnt), s));
    CKR(ar.alloc(&keep, N + 1));
    if (N > 0) {
      k_erase_records<<<grid_for(N, 256, c->sm_count), 256, 0, s>>>(N, lg->rec, drop, keep, cnt);
      c->launches++;
    }
    CKR(select_flagged(c, ar, N, keep, &pos, &idx));
    CK(cudaMemcpyAsync(h_cnt, cnt, sizeof(h_cnt), cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(&K, pos + N, 4, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    if (h_cnt[0] == 0) return CCO_OK;
    lg->snap.reset();   // the image is of the log before the erase
    CKR(ext_keep_records(lg, ar, K, idx));
    lg->n_erased += (long long)h_cnt[0];
    lg->n_prop -= (long long)h_cnt[1];
    lg->n_ignored -= (long long)h_cnt[2];
    const long long NG = (long long)lg->name_off.size() - 1;
    CKR(win_compact(lg, drop, lg->tline, lg->train_at, &lg->tu, &lg->ti, lg->history ? &lg->ttime : nullptr, &lg->tline,
                    lg->intern ? &lg->tkey : nullptr));
    CKR(win_compact(lg, drop, lg->rline, lg->rank_at, &lg->ri, nullptr, &lg->rtime, &lg->rline));
    for (long long g = 0; g < NG; ++g) {
      lg->n_train[g] = lg->train_at[g + 1] - lg->train_at[g];
      lg->n_rank[g] = lg->rank_at[g + 1] - lg->rank_at[g];
    }
    if (lg->intern) CKR(intern_refit(lg));
    if (h_cnt[1] > 0) {   // the aggregation again, over the property lines left
      for (void *p : {(void *)lg->p_field, (void *)lg->p_voff, (void *)lg->p_vals, (void *)lg->p_ioff, (void *)lg->p_ibytes}) log_drop(lg, p);
      lg->p_field = nullptr;
      lg->p_voff = lg->p_ioff = nullptr;
      lg->p_vals = lg->p_ibytes = nullptr;
      lg->p_ibytes_n = lg->n_triples = lg->n_prop_items = lg->n_prop_fields = 0;
      lg->field_names.clear();
      if (lg->n_prop > 0) {
        mail_reset(c);
        CKR(win_drop_property_lines(lg, par, ev, drop));
        CKR(event_properties(c, par, lg, ev.L, ev.flag, ev.tm, ev.sb, ev.span, lg->pb, lg->prop_line.data()));
        CKR(ext_keep_property_lines(lg, par, ev));
      } else {
        log_drop(lg, lg->pb);
        lg->pb = nullptr;
        lg->pb_len = lg->pb_cap = 0;
        lg->prop_line = std::vector<long long>();
      }
    }
    if (stats) {
      stats->n_lines = (int64_t)h_cnt[0];
      stats->n_training = E - lg->train_at.back();
      stats->n_ranking = R - lg->rank_at.back();
      stats->n_property_events = (int64_t)h_cnt[1];
    }
    return CCO_OK;
  }();
  if (rc == CCO_OK) {
    CK(cudaStreamSynchronize(s));
    CK(cudaGetLastError());
  }
  release();
  CK(cudaStreamSynchronize(s));
  return rc;
}

// the rankings of cco_format_model_log / cco_rerank_model_log as cco_ranking_t without streams + the log's streams
static int log_rankings(const cco_event_log *lg, int32_t n_rank, const cco_log_ranking_t *lr, std::vector<cco_ranking_t> *rk, Streams *ls) {
  if (n_rank < 0 || (n_rank > 0 && !lr)) return set_error(CCO_E_INVALID_ARG, "bad rankings");
  rk->assign((size_t)std::max(n_rank, 0), cco_ranking_t{});
  ls->assign((size_t)std::max(n_rank, 0), {});
  const int NG = (int)lg->n_rank.size();
  for (int k = 0; k < n_rank; ++k) {
    const cco_log_ranking_t &r = lr[k];
    (*rk)[k] = cco_ranking_t{r.name, r.mode, 0, r.start_ms, r.end_ms, nullptr};
    std::vector<int> codes;
    if (r.mode == CCO_POP_RANDOM) {   // calcRandom reads every event name
      for (int g = 0; g < NG; ++g) codes.push_back(g);
    } else {
      if (r.n_event_names < 0 || (r.n_event_names > 0 && !r.event_names)) return set_error(CCO_E_INVALID_ARG, "ranking %d: bad event names", k);
      for (int q = 0; q < r.n_event_names; ++q) {
        if (!r.event_names[q]) return set_error(CCO_E_INVALID_ARG, "ranking %d: null event name", k);
        codes.push_back(lg->code_of(r.event_names[q]));
      }
    }
    for (int g : codes) {
      if (g < 0) continue;   // a name without events: an empty stream
      Stream st;
      st.items.n = lg->n_rank[g];
      st.items.off = (const int64_t *)(lg->ri.off + lg->rank_at[g]);
      st.items.bytes = (const char *)lg->ri.w + lg->ri.boff[g];
      st.items.device = true;
      st.items.base = lg->ri.boff[g];
      st.items.nbytes = lg->ri.boff[g + 1] - lg->ri.boff[g];
      st.time = (const int64_t *)(lg->rtime + lg->rank_at[g]);
      (*ls)[k].push_back(st);
    }
  }
  return CCO_OK;
}
// a failed log answers every call with its first error's message; a log in progress is not read before finish
static int log_state(const cco_event_log *lg, bool want_finished) {
  if (lg->fail != CCO_OK) return set_error(CCO_E_INVALID_ARG, "the read of this log failed: %s", lg->fail_msg.c_str());
  if (lg->load) return set_error(CCO_E_INVALID_ARG, "the log is being loaded (cco_event_log_load_finish)");
  if (lg->finished != want_finished)
    return set_error(CCO_E_INVALID_ARG, want_finished ? "the log is not finished (cco_event_log_finish)" : "the log is finished");
  return CCO_OK;
}
static int log_fail(cco_event_log *lg, int rc) {
  if (rc != CCO_OK) {
    lg->fail = rc;
    lg->fail_msg = g_err;
  }
  return rc;
}
}  // namespace cco

int cco_event_log_begin(cco_ctx_t *ctx, int64_t chunk_bytes, cco_event_log_t **out) {
  return cco_event_log_begin_window(ctx, chunk_bytes, nullptr, out);
}

int cco_event_log_begin_window(cco_ctx_t *ctx, int64_t chunk_bytes, const cco_event_window_t *w, cco_event_log_t **out) {
  if (!ctx || !out || chunk_bytes < 1) return set_error(CCO_E_INVALID_ARG, "null argument or chunk_bytes < 1");
  *out = nullptr;
  if (w && (w->remove_duplicates != 0 && w->remove_duplicates != 1))
    return set_error(CCO_E_INVALID_ARG, "remove_duplicates is %d, not 0 or 1", (int)w->remove_duplicates);
  if (w && w->reserved != 0) return set_error(CCO_E_INVALID_ARG, "the window's reserved field must be 0");
  if (!ctx->members.empty()) return set_error(CCO_E_UNSUPPORTED, "an event log is resident on one GPU: read it on a per-GPU context");
  CKR(event_log_begin(ctx, chunk_bytes, out));
  if (w) {
    (*out)->cutoff = w->cutoff_ms;
    (*out)->dedup = w->remove_duplicates != 0;
  }
  return CCO_OK;
}

int cco_event_log_window_stats(const cco_event_log_t *lg, int64_t *n_expired, int64_t *n_duplicates) {
  if (!lg || !n_expired || !n_duplicates) return set_error(CCO_E_INVALID_ARG, "null argument");
  CKR(log_state(lg, true));
  *n_expired = lg->n_expired;
  *n_duplicates = lg->n_dup;
  return CCO_OK;
}

int cco_event_log_append(cco_event_log_t *lg, const char *bytes, int64_t len) {
  if (!lg || len < 0 || (len > 0 && !bytes)) return set_error(CCO_E_INVALID_ARG, "null argument or negative length");
  CKR(log_state(lg, false));
  return log_fail(lg, event_log_append(lg, bytes, len));
}

int cco_event_log_finish(cco_event_log_t *lg) {
  if (!lg) return set_error(CCO_E_INVALID_ARG, "null argument");
  CKR(log_state(lg, false));
  return log_fail(lg, event_log_finish(lg));
}

int cco_event_log_extend(cco_event_log_t *lg, const cco_event_window_t *w) {
  if (!lg) return set_error(CCO_E_INVALID_ARG, "null argument");
  CKR(log_state(lg, true));
  if (!lg->extendable) return set_error(CCO_E_INVALID_ARG, "the log was read without CCO_LOG_EXTENDABLE (cco_event_log_begin_ex)");
  if (lg->cleaners > 0) return set_error(CCO_E_INVALID_ARG, "a cleaner of the log is open (cco_event_log_clean_free)");
  lg->snap.reset();   // the image is of the log as it was finished
  if (w) {
    if (w->reserved != 0) return set_error(CCO_E_INVALID_ARG, "the window's reserved field must be 0");
    if ((w->remove_duplicates != 0) != lg->dedup || (w->remove_duplicates != 0 && w->remove_duplicates != 1))
      return set_error(CCO_E_INVALID_ARG, "remove_duplicates is %d: an extend keeps the first read's (%d)", (int)w->remove_duplicates, (int)lg->dedup);
    if (w->cutoff_ms < lg->cutoff)
      return set_error(CCO_E_INVALID_ARG, "cutoff %lld is before the log's %lld: expired lines are gone", (long long)w->cutoff_ms, lg->cutoff);
  }
  return log_fail(lg, event_log_extend(lg, w));
}

// the host checks of one id list of cco_event_log_erase
static int erase_ids_check(const char *what, int64_t n, const int64_t *off, const char *bytes) {
  if (n < 0) return set_error(CCO_E_INVALID_ARG, "%s: a negative count", what);
  if (n == 0) return CCO_OK;
  if (off[0] < 0) return set_error(CCO_E_INVALID_ARG, "%s: offsets[0] = %lld is negative", what, (long long)off[0]);
  for (int64_t i = 0; i < n; ++i)
    if (off[i + 1] < off[i]) return set_error(CCO_E_INVALID_ARG, "%s: offsets[%lld] = %lld decreases", what, (long long)i + 1, (long long)off[i + 1]);
  if (off[n] > off[0] && !bytes) return set_error(CCO_E_INVALID_ARG, "null argument");
  return CCO_OK;
}

int cco_event_log_erase(cco_event_log_t *lg, int64_t n_users, const int64_t *user_offsets, const char *user_bytes, int64_t n_items,
                        const int64_t *item_offsets, const char *item_bytes, cco_event_erase_stats_t *stats) {
  if (!lg || (n_users > 0 && !user_offsets) || (n_items > 0 && !item_offsets)) return set_error(CCO_E_INVALID_ARG, "null argument");
  if (stats) *stats = cco_event_erase_stats_t{0, 0, 0, 0};
  if (!lg->ctx->members.empty()) return set_error(CCO_E_UNSUPPORTED, "an event log is resident on one GPU");
  CKR(log_state(lg, true));
  if (!lg->extendable) return set_error(CCO_E_INVALID_ARG, "the log was read without CCO_LOG_EXTENDABLE (cco_event_log_begin_ex)");
  if (lg->cleaners > 0) return set_error(CCO_E_INVALID_ARG, "a cleaner of the log is open (cco_event_log_clean_free)");
  CKR(erase_ids_check("users", n_users, user_offsets, user_bytes));
  CKR(erase_ids_check("items", n_items, item_offsets, item_bytes));
  return log_fail(lg, event_log_erase(lg, n_users, user_offsets, user_bytes, n_items, item_offsets, item_bytes, stats));
}

int cco_event_log_erased(const cco_event_log_t *lg, int64_t *n_erased) {
  if (!lg || !n_erased) return set_error(CCO_E_INVALID_ARG, "null argument");
  CKR(log_state(lg, true));
  *n_erased = lg->n_erased;
  return CCO_OK;
}

int cco_event_log_intern_stats(const cco_event_log_t *lg, int64_t *n_user_keys, int64_t *n_item_keys) {
  if (!lg || !n_user_keys || !n_item_keys) return set_error(CCO_E_INVALID_ARG, "null argument");
  CKR(log_state(lg, true));
  if (!lg->intern) return set_error(CCO_E_INVALID_ARG, "the log was read without CCO_LOG_INTERN_IDS (cco_event_log_begin_ex)");
  *n_user_keys = lg->users.n;
  *n_item_keys = lg->items.n;
  return CCO_OK;
}

int cco_event_log_resident_bytes(const cco_event_log_t *lg, int64_t *bytes) {
  if (!lg || !bytes) return set_error(CCO_E_INVALID_ARG, "null argument");
  CKR(log_state(lg, true));
  int64_t b = 0;
  for (size_t x : lg->dev_bytes) b += (int64_t)x;
  *bytes = b;
  return CCO_OK;
}

int cco_event_log_read(cco_ctx_t *ctx, const char *bytes, int64_t len, cco_event_log_t **out) {
  if (!ctx || !out || len < 0 || (len > 0 && !bytes)) return set_error(CCO_E_INVALID_ARG, "null argument or negative length");
  *out = nullptr;
  if (!ctx->members.empty()) return set_error(CCO_E_UNSUPPORTED, "an event log is resident on one GPU: read it on a per-GPU context");
  NvtxRange nvtx("cco:event_log_read");
  cco_event_log *lg = nullptr;
  CKR(event_log_begin(ctx, std::max<int64_t>(len, 1), &lg));
  int rc = event_log_append(lg, bytes, len);
  if (rc == CCO_OK) rc = event_log_finish(lg);
  if (rc != CCO_OK) {
    event_log_release(lg);
    return rc;
  }
  *out = lg;
  return CCO_OK;
}

int cco_event_log_info(const cco_event_log_t *lg, cco_event_log_info_t *out) {
  if (!lg || !out) return set_error(CCO_E_INVALID_ARG, "null argument");
  CKR(log_state(lg, true));
  out->n_lines = lg->n_lines;
  out->names = cco_dictionary_t{(int64_t)lg->n_train.size(), lg->name_off.data(), lg->name_bytes.data()};
  out->n_training = lg->n_train.data();
  out->n_ranking = lg->n_rank.data();
  out->n_property_events = lg->n_prop;
  out->n_property_items = lg->n_prop_items;
  out->n_property_fields = lg->n_prop_fields;
  out->n_ignored = lg->n_ignored;
  return CCO_OK;
}

namespace cco {
// the entries [0, n) of one key column (entry e's key: key2[2 e] < n_keys) grouped by key, gated entries (gate[e] < 0)
// left out: the keys with >= need entries (counting; duplicates count) or every key met, numbered by their first entry
// -> rank[key] (-1: not numbered), id[e] (-1: gated or not numbered), the keys in dictionary order (tb->first_sorted, as
// str_dictionary reads it: the heap's strings are indexed by key)
static int key_group(cco_ctx *c, Arena &ar, long long n, const uint32_t *key2, long long n_keys, const int32_t *gate, bool counting,
                     uint32_t need, StrTable *tb, int32_t *rank, int32_t *id) {
  cudaStream_t s = c->stream;
  uint32_t *first, *count = nullptr, *flag, *pos;
  CKR(ar.alloc(&first, std::max<long long>(n_keys, 1)));
  CK(cudaMemsetAsync(first, 0xff, sizeof(uint32_t) * (size_t)n_keys, s));
  if (counting) {
    CKR(ar.alloc(&count, std::max<long long>(n_keys, 1)));
    CK(cudaMemsetAsync(count, 0, sizeof(uint32_t) * (size_t)n_keys, s));
  }
  CK(cudaMemsetAsync(rank, 0xff, sizeof(int32_t) * (size_t)n_keys, s));
  if (n > 0) {
    k_intern_first_count<<<grid_for(n, 256, c->sm_count), 256, 0, s>>>(n, key2, gate, first, count);
    c->launches++;
  }
  CKR(ar.alloc(&flag, n_keys + 1));
  CKR(ar.alloc(&pos, n_keys + 1));
  CK(cudaMemsetAsync(flag + n_keys, 0, 4, s));
  if (n_keys > 0) {
    k_str_flags<<<grid_for(n_keys, 256, c->sm_count), 256, 0, s>>>(n_keys, first, count, need, flag);   // first: kStrEmpty = no entry
    c->launches++;
  }
  CKR(exclusive_sum(c, ar, flag, pos, n_keys + 1));
  uint32_t ng = 0;
  CKR(mail_fetch(c, &ng, pos + n_keys, 4));
  CKR(mail_wait(c));
  tb->n_groups = ng;
  if (ng > 0) {
    uint32_t *k0, *v0;
    CKR(ar.alloc(&k0, ng));
    CKR(ar.alloc(&v0, ng));
    k_str_compact<<<grid_for(n_keys, 256, c->sm_count), 256, 0, s>>>(n_keys, flag, pos, first, k0, v0);
    c->launches++;
    CKR(sort_pairs(c, ar, ng, &k0, &v0, bits_for(n)));   // first entries are distinct: the sort by them is the dictionary order
    k_str_rank<<<grid_for(ng, 256, c->sm_count), 256, 0, s>>>(ng, v0, rank);
    c->launches++;
    ar.release(k0);
    tb->first_sorted = v0;
  }
  if (n > 0) {
    k_intern_ids<<<grid_for(n, 256, c->sm_count), 256, 0, s>>>(n, key2, gate, rank, id);
    c->launches++;
  }
  ar.release(first);
  ar.release(count);
  ar.release(flag);
  ar.release(pos);
  return CCO_OK;
}
// cco_event_log_ingest on an interned log: ingest_strings_core's rules over the entries' keys, integer passes only; the
// dictionaries are the heaps' strings gathered in dictionary order
static int ingest_keys_core(cco_ctx *c, const cco_event_log *lg, const std::vector<int> &codes, int32_t min_events_per_user, cco_dataset **out) {
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  NvtxRange nvtx("cco:ingest_keys");
  mail_reset(c);
  Arena ar(s);
  const int n_types = (int)codes.size();
  cco_dataset *d = ingest_dataset_new(c, n_types);
  d->dicts.assign((size_t)n_types + 1, cco_dictionary_t{0, nullptr, nullptr});
  struct G {
    cco_dataset *d;
    bool ok = false;
    ~G() {
      if (!ok) {
        cudaStreamSynchronize(d->ctx->stream);   // no dictionary copy still writes the pinned buffers released here
        dataset_release(d);
      }
    }
  } g{d};
  const uint32_t need = min_events_per_user > 1 ? (uint32_t)min_events_per_user : 1u;
  const long long NU = lg->users.n, NI = lg->items.n;
  int32_t *urank, *irank;
  CKR(ar.alloc(&urank, std::max<long long>(NU, 1)));
  CKR(ar.alloc(&irank, std::max<long long>(NI, 1)));
  uint32_t n_users = 0;
  for (int t = 0; t < n_types; ++t) {
    const int gc = codes[t];
    const long long ne = gc >= 0 ? lg->n_train[gc] : 0;
    // entry e's item key at k2[2 e], its user key at k2[2 e + 1]
    const uint32_t *k2 = ne > 0 ? (const uint32_t *)(lg->tkey + lg->train_at[gc]) : nullptr;
    int32_t *uid, *iid;
    CKR(ar.alloc(&uid, std::max<long long>(ne, 1)));
    CKR(ar.alloc(&iid, std::max<long long>(ne, 1)));
    if (t == 0) {
      // user dictionary: primary users with >= need events (duplicates count, Preparator.scala:129-132), first appearance order
      StrTable ut;
      CKR(key_group(c, ar, ne, k2 ? k2 + 1 : nullptr, NU, nullptr, true, need, &ut, urank, uid));
      if (ut.n_groups >= 0x7fffffffLL) return set_error(CCO_E_UNSUPPORTED, "%lld users: the user space must stay < 2^31 - 1", ut.n_groups);
      n_users = (uint32_t)ut.n_groups;
      d->n_users = n_users;
      CKR(str_dictionary(c, ar, lg->users.heap(), ut, &d->dicts[0]));
      ar.release(ut.first_sorted);
    } else if (ne > 0) {
      // secondary events of users outside the dictionary are dropped (Preparator.scala:175-178)
      k_intern_ids<<<grid_for(ne, 256, c->sm_count), 256, 0, s>>>(ne, k2 + 1, nullptr, urank, uid);
      c->launches++;
    }
    // item dictionary of type t: items with a surviving event, ordered by first surviving appearance
    StrTable it;
    CKR(key_group(c, ar, ne, k2, NI, uid, false, 0, &it, irank, iid));
    if (it.n_groups >= 0x7ffffffeLL) return set_error(CCO_E_UNSUPPORTED, "type %d: %lld items, at most 2^31 - 2", t, it.n_groups);
    d->n_cols[t] = it.n_groups;
    CKR(str_dictionary(c, ar, lg->items.heap(), it, &d->dicts[1 + t]));
    ar.release(it.first_sorted);
    CKR(ingest_ids_csr(c, ar, d, t, ne, n_users, uid, iid));
  }
  CKR(ingest_blocks(c, d, n_users));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  g.ok = true;
  *out = d;
  return CCO_OK;
}
}  // namespace cco

int cco_event_log_ingest(cco_ctx_t *c, const cco_event_log_t *lg, int32_t n_names, const char *const *names, int32_t min_events_per_user,
                         cco_dataset_t **out) {
  if (!c || !lg || !names || !out || n_names < 1) return set_error(CCO_E_INVALID_ARG, "bad argument");
  *out = nullptr;
  if (!c->members.empty() || lg->ctx != c) return set_error(CCO_E_UNSUPPORTED, "ingest a log on the per-GPU context that read it");
  CKR(log_state(lg, true));
  std::vector<int> codes(n_names);
  for (int t = 0; t < n_names; ++t) {
    if (!names[t]) return set_error(CCO_E_INVALID_ARG, "null event name %d", t);
    codes[t] = lg->code_of(names[t]);
  }
  if (lg->intern) return ingest_keys_core(c, lg, codes, min_events_per_user, out);
  const StrColumns view = [lg, &codes](Arena &ar, int t, DevStrCol *uc, DevStrCol *ic) -> int {
    const int g = codes[t];
    const long long n = g >= 0 ? lg->n_train[g] : 0;
    *uc = lg->view(lg->tu, g, lg->train_at, n);
    *ic = lg->view(lg->ti, g, lg->train_at, n);
    CKR(ar.alloc(&uc->hash, std::max<long long>(n, 1)));
    CKR(ar.alloc(&ic->hash, std::max<long long>(n, 1)));
    return CCO_OK;
  };
  return ingest_strings_core(c, n_names, view, min_events_per_user, out);
}

namespace cco {
// the log's aggregated properties as format_model takes them: a host shell (count, field names) + the device columns
struct LogProps {
  std::vector<const char *> names;
  cco_item_properties_t shell;
  DevProps dev;
};
static void log_props(const cco_event_log *lg, LogProps *p) {
  for (const std::string &f : lg->field_names) p->names.push_back(f.c_str());
  p->shell = cco_item_properties_t{lg->n_triples, nullptr, nullptr, nullptr, nullptr, nullptr, (int32_t)p->names.size(), p->names.data()};
  p->dev.items = KeySection{lg->n_triples, (const int64_t *)lg->p_ioff, (const char *)lg->p_ibytes, true, lg->p_ibytes_n, 0};
  p->dev.field = lg->p_field;
  p->dev.voff = lg->p_voff;
  p->dev.vals = lg->p_vals;
}
}  // namespace cco

int cco_format_model_log(cco_ctx_t *ctx, const cco_result_t *res, int32_t n_names, const char *const *names,
                         const cco_dictionary_t *row_ids, const cco_dictionary_t *col_ids, const cco_event_log_t *lg, int32_t n_rankings,
                         const cco_log_ranking_t *rankings, char **out_bytes, int64_t *out_len) {
  if (!ctx || !lg) return set_error(CCO_E_INVALID_ARG, "null argument");
  if (!ctx->members.empty() || lg->ctx != ctx) return set_error(CCO_E_UNSUPPORTED, "format on the per-GPU context that read the log");
  CKR(log_state(lg, true));
  std::vector<cco_ranking_t> rk;
  Streams ls;
  CKR(log_rankings(lg, n_rankings, rankings, &rk, &ls));
  LogProps lp;
  log_props(lg, &lp);
  const bool any = lg->n_triples > 0;
  return format_model(ctx, res, n_names, names, row_ids, col_ids, any ? &lp.shell : nullptr, n_rankings, rk.data(), out_bytes, out_len,
                      "cco:format_model_log", std::move(ls), any ? &lp.dev : nullptr);
}

int cco_rerank_model_log(cco_ctx_t *ctx, const char *body, int64_t body_len, const cco_event_log_t *lg, int32_t n_rankings,
                         const cco_log_ranking_t *rankings, char **out_bytes, int64_t *out_len) {
  if (!ctx || !lg) return set_error(CCO_E_INVALID_ARG, "null argument");
  if (!ctx->members.empty() || lg->ctx != ctx) return set_error(CCO_E_UNSUPPORTED, "rerank on the per-GPU context that read the log");
  CKR(log_state(lg, true));
  std::vector<cco_ranking_t> rk;
  Streams ls;
  CKR(log_rankings(lg, n_rankings, rankings, &rk, &ls));
  LogProps lp;
  log_props(lg, &lp);
  const bool any = lg->n_triples > 0;
  return rerank_model(ctx, body, body_len, any ? &lp.shell : nullptr, n_rankings, rk.data(), out_bytes, out_len, std::move(ls),
                      any ? &lp.dev : nullptr);
}

// ---- cco_refresh_properties: fresh item properties written into the old documents, kernels in cco_refresh.cuh ----------
namespace cco {
static int refresh_names(int32_t n, const char *const *names, const char *what) {
  if (n < 0 || (n > 0 && !names)) return set_error(CCO_E_INVALID_ARG, "bad %s names", what);
  for (int k = 0; k < n; ++k)
    if (!names[k]) return set_error(CCO_E_INVALID_ARG, "%s name %d is null", what, k);
  return CCO_OK;
}
// the outputs into pinned memory of c, one device-to-host copy each, then one wait; on failure every buffer goes back
static int refresh_to_host(cco_ctx *c, const unsigned char *const src[5], const long long bytes[5], void *dst[5]) {
  cudaStream_t s = c->stream;
  for (int k = 0; k < 5; ++k) dst[k] = nullptr;
  const int st = [&]() -> int {
    for (int k = 0; k < 5; ++k) {
      dst[k] = c->pinned_get((size_t)std::max<long long>(bytes[k], 1), /*for_result=*/false);
      if (!dst[k]) return set_error(CCO_E_OOM, "pinned host allocation failed");
      if (bytes[k] > 0) CK(cudaMemcpyAsync(dst[k], src[k], (size_t)bytes[k], cudaMemcpyDeviceToHost, s));
    }
    CK(cudaStreamSynchronize(s));
    CK(cudaGetLastError());
    return CCO_OK;
  }();
  if (st != CCO_OK)
    for (int k = 0; k < 5; ++k)
      if (dst[k]) c->pinned_put(dst[k]);
  return st;
}

static int refresh_properties(cco_ctx_t *ctx, const char *body, int64_t body_len, const cco_item_properties_t *props,
                              const cco_refresh_params_t *prm, cco_refresh_out_t *out, const DevProps *dp = nullptr) {
  if (!ctx || !prm || !out || body_len < 0 || (body_len > 0 && !body)) return set_error(CCO_E_INVALID_ARG, "null argument or negative length");
  memset(out, 0, sizeof *out);
  if (!ctx->members.empty()) return set_error(CCO_E_UNSUPPORTED, "per-GPU contexts only");
  if (body_len > 0 && body[body_len - 1] != '\n') return set_error(CCO_E_INVALID_ARG, "the body does not end in a newline");
  CKR(refresh_names(prm->n_correlators, prm->correlators, "correlator"));
  CKR(refresh_names(prm->n_rankings, prm->rankings, "ranking"));
  const cco_dictionary_t no_rows = {0, nullptr, nullptr};
  Streams st;
  CKR(model_check_host(&no_rows, props, 0, nullptr, &st, dp != nullptr));
  const int n_fields = props ? props->n_fields : 0;
  for (int f = 0; f < n_fields; ++f)   // cco_format_model would let it replace the array; a refresh has none to put back
    for (int i = 0; i < prm->n_correlators; ++i)
      if (!strcmp(props->field_names[f], prm->correlators[i]))
        return set_error(CCO_E_UNSUPPORTED, "property field \"%s\" is named like a correlator: a refresh keeps the correlator arrays",
                         props->field_names[f]);
  cco_ctx *c = ctx;
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Arena ar(s);
  NvtxRange nvtx("cco:refresh_properties");
  mail_reset(c);
  // 1. the old documents: members, decoded names and _ids (cco_rerank_model's grammar and checks)
  BulkDocs bd;
  CKR(bulk_parse(c, ar, body, body_len, props ? props->n : 0, "property triples", &bd));
  const long long D = bd.D, M1 = bd.M1;
  // 2. join: the decoded ids are the row section of the key column, the properties sorted per item as cco_format_model
  FormatArgs fa;
  memset(&fa, 0, sizeof fa);
  CKR(model_names(c, ar, &fa, 0, nullptr, true, props, 0, nullptr));
  fa.n_rows = (int32_t)D;
  const DevDict raw_ids = {bd.ids.off, (const unsigned char *)bd.ids.w, D};
  CKR(escape_dict(c, ar, raw_ids, &fa.row_ids));
  const KeySection rows{D, (const int64_t *)bd.ids.off, (const char *)bd.ids.w, true, bd.ids_bytes};
  CKR(model_fields(c, ar, &fa, rows, props, 0, nullptr, st, true, true, dp));
  // a field named "id" or like a computed ranking is not written (kClashId: prop_written skips it)
  std::vector<uint16_t> fclash(std::max(n_fields, 1), 0);
  for (int f = 0; f < n_fields; ++f) {
    if (!strcmp(props->field_names[f], "id")) fclash[f] = kClashId;
    for (int k = 0; k < prm->n_rankings; ++k)
      if (!strcmp(props->field_names[f], prm->rankings[k])) fclash[f] = kClashId;
  }
  uint16_t *d_fclash;
  CKR(ar.alloc(&d_fclash, fclash.size()));
  CK(cudaMemcpyAsync(d_fclash, fclash.data(), sizeof(uint16_t) * fclash.size(), cudaMemcpyHostToDevice, s));
  fa.field_clash = d_fclash;
  // 3. member names -> correlator, computed ranking or other; "id" and members followed by one of the same name are skipped
  RefreshArgs ra;
  memset(&ra, 0, sizeof ra);
  ra.body = bd.body;
  ra.line_moff = bd.line_moff;
  ra.mem = bd.mem;
  ra.line_b = bd.line_b;
  ra.body_len = body_len;
  std::vector<std::string> ent;
  std::vector<uint8_t> ent_cls, ent_id;
  auto entry = [&](const char *nm, uint8_t cls, uint8_t id) {
    for (size_t t = 0; t < ent.size(); ++t)
      if (ent[t] == nm) return;
    ent.push_back(nm);
    ent_cls.push_back(cls);
    ent_id.push_back(id);
  };
  entry("id", kRefreshOther, 1);
  for (int i = 0; i < prm->n_correlators; ++i) entry(prm->correlators[i], kRefreshCorrelator, 0);
  for (int k = 0; k < prm->n_rankings; ++k) entry(prm->rankings[k], kRefreshRanking, 0);
  if (D > 0) {
    const int T = (int)ent.size();
    int32_t *ngid, *entry_of, *ment;
    uint8_t *d_cls, *d_id, *mkeep;
    CKR(ar.alloc(&d_cls, T));
    CKR(ar.alloc(&d_id, T));
    CK(cudaMemcpyAsync(d_cls, ent_cls.data(), T, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_id, ent_id.data(), T, cudaMemcpyHostToDevice, s));
    CKR(member_entries(c, ar, bd.names, ent, &ngid, &entry_of));   // its wait for the upload also covers these local tables
    CKR(ar.alloc(&ment, std::max<long long>(M1, 1)));
    CKR(ar.alloc(&mkeep, std::max<long long>(M1, 1)));
    k_member_info<<<grid_for(D * 32, 256, c->sm_count), 256, 0, s>>>(D, ra.line_moff, ngid, entry_of, d_id, ment, mkeep);
    c->launches++;
    ra.ment = ment;
    ra.mkeep = mkeep;
    ra.ent_cls = d_cls;
  }
  CK(cudaStreamSynchronize(s));   // fclash, ent_cls and ent_id are locals
  // 4. the refreshed body: the old documents rewritten (deleted ones: 0 bytes), then the new items as cco_format_model writes them
  const long long X = fa.n_extra, N = D + X;
  FormatArgs fx = fa;   // the new items only
  fx.n_rows = 0;
  long long *doc_len, *doc_off;
  CKR(ar.alloc(&doc_len, N + 1));
  CKR(ar.alloc(&doc_off, N + 1));
  CK(cudaMemsetAsync(doc_len + N, 0, 8, s));
  if (D > 0) k_refresh_len<<<grid_for(D * 32, 256, c->sm_count), 256, 0, s>>>(fa, ra, (int32_t)D, doc_len);
  if (X > 0) k_doc_len<<<grid_for(X, 256, c->sm_count), 256, 0, s>>>(fx, (int32_t)X, doc_len + D);
  c->launches += (D > 0) + (X > 0);
  CKR(exclusive_sum(c, ar, doc_len, doc_off, N + 1));
  long long total = 0;
  CKR(mail_fetch(c, &total, doc_off + N, 8));
  CKR(mail_wait(c));
  unsigned char *d_full;
  CKR(ar.alloc(&d_full, std::max<long long>(total, 1)));
  if (D > 0) k_refresh_write<<<grid_for(D * 32, 256, c->sm_count), 256, 0, s>>>(fa, ra, (int32_t)D, doc_off, d_full);
  if (X > 0) k_doc_write<<<grid_for(X * 32, 256, c->sm_count), 256, 0, s>>>(fx, (int32_t)X, doc_off + D, d_full);
  c->launches += (D > 0) + (X > 0);
  // 5. the diff against the old source lines, the delta and deleted lists
  uint32_t *flag, *fpos, *del, *dpos;
  CKR(ar.alloc(&flag, N + 1));
  CKR(ar.alloc(&fpos, N + 1));
  CKR(ar.alloc(&del, N + 1));
  CKR(ar.alloc(&dpos, N + 1));
  CK(cudaMemsetAsync(flag, 0, sizeof(uint32_t) * (size_t)(N + 1), s));
  CK(cudaMemsetAsync(del, 0, sizeof(uint32_t) * (size_t)(N + 1), s));
  if (N > 0) {
    k_refresh_diff<<<grid_for(N * 32, 256, c->sm_count), 256, 0, s>>>(fa, ra, (int32_t)D, (int32_t)N, doc_off, d_full, flag, del);
    c->launches++;
  }
  CKR(exclusive_sum(c, ar, flag, fpos, N + 1));
  CKR(exclusive_sum(c, ar, del, dpos, N + 1));
  uint32_t n_delta = 0, n_changed = 0, n_deleted = 0;
  CKR(mail_fetch(c, &n_delta, fpos + N, 4));
  CKR(mail_fetch(c, &n_changed, fpos + D, 4));
  CKR(mail_fetch(c, &n_deleted, dpos + N, 4));
  CKR(mail_wait(c));
  uint32_t *pick;
  long long *se, *dlen, *doff, *xlen, *xoff;
  int64_t *changed, *deleted;
  CKR(ar.alloc(&pick, std::max<long long>(n_delta, 1)));
  CKR(ar.alloc(&se, std::max<long long>(N, 1)));
  CKR(ar.alloc(&changed, std::max<long long>(n_changed, 1)));
  CKR(ar.alloc(&deleted, std::max<long long>(n_deleted, 1)));
  CKR(ar.alloc(&dlen, (long long)n_delta + 1));
  CKR(ar.alloc(&doff, (long long)n_delta + 1));
  CKR(ar.alloc(&xlen, (long long)n_deleted + 1));
  CKR(ar.alloc(&xoff, (long long)n_deleted + 1));
  CK(cudaMemsetAsync(dlen + n_delta, 0, 8, s));
  CK(cudaMemsetAsync(xlen + n_deleted, 0, 8, s));
  if (N > 0) {
    k_refresh_lists<<<grid_for(N, 256, c->sm_count), 256, 0, s>>>((int32_t)D, (int32_t)N, flag, fpos, del, dpos, doc_off, pick, se, changed, deleted);
    c->launches++;
  }
  if (n_delta > 0) {
    k_line_len<<<grid_for(n_delta, 256, c->sm_count), 256, 0, s>>>(n_delta, pick, doc_off, se, dlen);
    c->launches++;
  }
  if (n_deleted > 0) {
    k_refresh_del_len<<<grid_for(n_deleted, 256, c->sm_count), 256, 0, s>>>(n_deleted, deleted, fa.row_ids, xlen);
    c->launches++;
  }
  CKR(exclusive_sum(c, ar, dlen, doff, (long long)n_delta + 1));
  CKR(exclusive_sum(c, ar, xlen, xoff, (long long)n_deleted + 1));
  long long delta_bytes = 0, del_bytes = 0;
  CKR(mail_fetch(c, &delta_bytes, doff + n_delta, 8));
  CKR(mail_fetch(c, &del_bytes, xoff + n_deleted, 8));
  CKR(mail_wait(c));
  unsigned char *d_delta, *d_del;
  CKR(ar.alloc(&d_delta, std::max<long long>(delta_bytes, 1)));
  CKR(ar.alloc(&d_del, std::max<long long>(del_bytes, 1)));
  if (n_delta > 0) {
    k_line_gather<<<grid_for((long long)n_delta * 32, 256, c->sm_count), 256, 0, s>>>(n_delta, pick, doc_off, se, d_full, doff, d_delta);
    c->launches++;
  }
  if (n_deleted > 0) {
    k_refresh_del_write<<<grid_for((long long)n_deleted * 32, 256, c->sm_count), 256, 0, s>>>(n_deleted, deleted, fa.row_ids, xoff, d_del);
    c->launches++;
  }
  // 6. one device-to-host copy per output
  const unsigned char *src[5] = {d_full, d_delta, d_del, (const unsigned char *)changed, (const unsigned char *)deleted};
  const long long bytes[5] = {total, delta_bytes, del_bytes, 8LL * n_changed, 8LL * n_deleted};
  void *dst[5];
  CKR(refresh_to_host(c, src, bytes, dst));
  out->n_docs = N - n_deleted;
  out->n_changed = n_changed;
  out->n_new = X;
  out->n_deleted = n_deleted;
  out->n_unchanged = D - n_deleted - n_changed;
  out->body = (char *)dst[0];
  out->body_len = total;
  out->delta = (char *)dst[1];
  out->delta_len = delta_bytes;
  out->deletes = (char *)dst[2];
  out->deletes_len = del_bytes;
  out->changed = (int64_t *)dst[3];
  out->deleted = (int64_t *)dst[4];
  return CCO_OK;
}
}  // namespace cco

int cco_refresh_properties(cco_ctx_t *ctx, const char *body, int64_t body_len, const cco_item_properties_t *props,
                           const cco_refresh_params_t *params, cco_refresh_out_t *out) {
  return refresh_properties(ctx, body, body_len, props, params, out);
}

int cco_refresh_properties_log(cco_ctx_t *ctx, const char *body, int64_t body_len, const cco_event_log_t *lg,
                               const cco_refresh_params_t *params, cco_refresh_out_t *out) {
  if (!ctx || !lg) return set_error(CCO_E_INVALID_ARG, "null argument");
  if (!ctx->members.empty() || lg->ctx != ctx) return set_error(CCO_E_UNSUPPORTED, "refresh on the per-GPU context that read the log");
  CKR(log_state(lg, true));
  LogProps lp;
  log_props(lg, &lp);
  const bool any = lg->n_triples > 0;
  return refresh_properties(ctx, body, body_len, any ? &lp.shell : nullptr, params, out, any ? &lp.dev : nullptr);
}

namespace cco {
// json4s 3.2's quote of a name (the escaping of uq_escape, on the host), quotes included
static std::string uq_quote(const char *s) {
  std::string o = "\"";
  const unsigned char *b = (const unsigned char *)s;
  const size_t n = strlen(s);
  char hex[8];
  for (size_t i = 0; i < n; ++i) {
    const unsigned char x = b[i];
    unsigned cp = 0xffffffffu;
    if (x == '"' || x == '\\') { o += '\\'; o += (char)x; continue; }
    if (x == '\b') { o += "\\b"; continue; }
    if (x == '\f') { o += "\\f"; continue; }
    if (x == '\n') { o += "\\n"; continue; }
    if (x == '\r') { o += "\\r"; continue; }
    if (x == '\t') { o += "\\t"; continue; }
    if (x < 0x20) cp = x;
    else if (x == 0xC2 && i + 1 < n && b[i + 1] >= 0x80 && b[i + 1] <= 0x9F) cp = b[++i];
    else if (x == 0xE2 && i + 2 < n && b[i + 1] >= 0x80 && b[i + 1] <= 0x83 && (b[i + 2] & 0xC0) == 0x80) {
      cp = 0x2000u | ((unsigned)(b[i + 1] & 0x3F) << 6) | (b[i + 2] & 0x3F);
      i += 2;
    }
    if (cp != 0xffffffffu) {
      snprintf(hex, sizeof hex, "\\u%04x", cp);
      o += hex;
    } else {
      o += (char)x;
    }
  }
  return o + "\"";
}

// the text every query template starts with (up to the should clauses), and the one after the must_not ids
static std::string query_head(const char *header, const char *head) {
  return std::string(header) + "\n" + head + ",\"query\":{\"bool\":{\"should\":[";
}
static std::string query_tail(const char *must_not, const char *sort) {
  return std::string("],\"boost\":0}}") + (*must_not ? std::string(",") + must_not : std::string()) +
         "],\"minimum_should_match\":1}},\"sort\":" + sort + "}\n";
}

// The R records of a query builder, one warp each: the length pass, the record offsets (each record < 2^31 bytes) on the
// host, the write pass and the body on the host; `also` as in body_to_host.  On failure every pinned buffer taken here is
// given back.
extern "C++" {
template <class Args>
static int emit_records(cco_ctx *c, Arena &ar, long long R, void (*len_pass)(Args, const long long *, long long *, unsigned char *),
                        void (*write_pass)(Args, const long long *, long long *, unsigned char *), const Args &a, char **out_body,
                        int64_t *out_len, int64_t **out_offsets, int64_t *out_n, const std::function<int()> &also = nullptr) {
  cudaStream_t s = c->stream;
  const int grid = grid_for(R * 32, 256, c->sm_count);
  long long *rlen, *roff;
  CKR(ar.alloc(&rlen, R + 1));
  CKR(ar.alloc(&roff, R + 1));
  CK(cudaMemsetAsync(rlen + R, 0, 8, s));
  if (R > 0) {
    len_pass<<<grid, 256, 0, s>>>(a, nullptr, rlen, nullptr);
    c->launches++;
  }
  CKR(exclusive_sum(c, ar, rlen, roff, R + 1));
  int64_t *ho = (int64_t *)c->pinned_get(sizeof(int64_t) * ((size_t)R + 1), /*for_result=*/false);
  if (!ho) return set_error(CCO_E_OOM, "pinned host allocation failed");
  const int st = [&]() -> int {
    CK(cudaMemcpyAsync(ho, roff, sizeof(int64_t) * ((size_t)R + 1), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    for (long long r = 0; r < R; ++r)
      if (ho[r + 1] - ho[r] >= (1LL << 31))
        return set_error(CCO_E_UNSUPPORTED, "record %lld has %lld bytes, at most 2^31 - 1", r, (long long)(ho[r + 1] - ho[r]));
    const long long total = ho[R];
    unsigned char *d_out;
    CKR(ar.alloc(&d_out, std::max<long long>(total, 1)));
    if (R > 0 && total > 0) {
      write_pass<<<grid, 256, 0, s>>>(a, roff, nullptr, d_out);
      c->launches++;
    }
    return body_to_host(c, s, d_out, total, out_body, out_len, also);
  }();
  if (st != CCO_OK) {
    c->pinned_put(ho);
    return st;
  }
  *out_offsets = ho;
  *out_n = R;
  return CCO_OK;
}
}  // extern "C++"

static int uq_check_host(const cco_user_query_t *q, int64_t n_users, const int64_t *uoff, const char *ubytes) {
  if (q->n_names < 0 || q->n_names > kUqMaxNames) return set_error(CCO_E_INVALID_ARG, "%d query event names, 0..%d", (int)q->n_names, kUqMaxNames);
  if (q->n_names > 0 && (!q->names || !q->limits)) return set_error(CCO_E_INVALID_ARG, "null names or limits");
  for (int k = 0; k < q->n_names; ++k) {
    if (!q->names[k] || !*q->names[k]) return set_error(CCO_E_INVALID_ARG, "query event name %d is null or empty", k);
    if (q->limits[k] < 0) return set_error(CCO_E_INVALID_ARG, "query event name %d: negative limit %d", k, (int)q->limits[k]);
  }
  if (q->n_history_names < 0 || q->n_history_names > q->n_names)
    return set_error(CCO_E_INVALID_ARG, "n_history_names = %d is outside [0, %d]", (int)q->n_history_names, (int)q->n_names);
  if (q->n_blacklist_names < 0 || (q->n_blacklist_names > 0 && !q->blacklist_names)) return set_error(CCO_E_INVALID_ARG, "bad blacklist names");
  for (int b = 0; b < q->n_blacklist_names; ++b)
    if (!q->blacklist_names[b]) return set_error(CCO_E_INVALID_ARG, "blacklist name %d is null", b);
  if (q->history_in_must != 0 && q->history_in_must != 1) return set_error(CCO_E_INVALID_ARG, "history_in_must must be 0 or 1");
  if (!q->head || !q->should || !q->must || !q->must_not || !q->sort || !q->header) return set_error(CCO_E_INVALID_ARG, "a null fragment");
  if (!*q->should) return set_error(CCO_E_INVALID_ARG, "the should fragment is empty");
  CKR(str_check_host(q->n_blacklist_items, q->blacklist_item_offsets, q->blacklist_item_bytes, 0, "blacklist item"));
  if (uoff) CKR(str_check_host(n_users, uoff, ubytes, 0, "user"));
  else if (n_users != 0) return set_error(CCO_E_INVALID_ARG, "n_users without user offsets");
  return CCO_OK;
}

// The history stage of the user-query builders: every training event of the query names, the users' history lists and
// their blacklisted items, in HBM.  The log's users and items are grouped exactly; the groups number the user table (ut)
// and the item table (it) that records and ids are looked up in.
struct UqHistory {
  long long E = 0, G = 0, B = 0;   // events of the query names, users among them, blacklisted events
  StrTable ut, it;
  DevStrCol tu, ti;                // the log's training user and item columns (hashed when E > 0)
  uint32_t *ent = nullptr, *hord = nullptr, *bord = nullptr, *gord = nullptr;
  uint8_t *keep_h = nullptr, *keep_b = nullptr, *qr = nullptr;
  int32_t *uid = nullptr, *iid = nullptr, *d_limit = nullptr;
  long long *ln = nullptr, *hstart = nullptr, *bstart = nullptr;
  unsigned long long *bkey = nullptr;
};
// per query name: its events are blacklisted (a blacklist name; a repeated query name reads the same events: once)
static std::vector<uint8_t> uq_black_names(int nq, const char *const *names, int n_blacklist_names, const char *const *blacklist_names) {
  std::vector<uint8_t> black(std::max(nq, 1), 0);
  for (int k = 0; k < nq; ++k) {
    bool earlier = false;
    for (int j = 0; j < k; ++j) earlier |= strcmp(names[j], names[k]) == 0;
    for (int b = 0; b < n_blacklist_names && !earlier; ++b)
      if (strcmp(blacklist_names[b], names[k]) == 0) black[k] = 1;
  }
  return black;
}
static int uq_blacklist(cco_ctx *c, Arena &ar, int nq, const std::vector<uint8_t> &black, UqHistory *h);
static int uq_history(cco_ctx *c, Arena &ar, const cco_event_log *lg, int nq, const char *const *names, const int32_t *limits,
                      const std::vector<uint8_t> &black, UqHistory *h) {
  cudaStream_t s = c->stream;
  std::vector<int> code(nq);
  for (int k = 0; k < nq; ++k) code[k] = lg->code_of(names[k]);
  // 2. the training events of the query names, name-major
  std::vector<long long> qoff(nq + 1, 0), qbase(std::max(nq, 1), 0);
  for (int k = 0; k < nq; ++k) {
    const long long n = code[k] >= 0 ? lg->n_train[code[k]] : 0;
    qbase[k] = code[k] >= 0 ? lg->train_at[code[k]] : 0;
    qoff[k + 1] = qoff[k] + n;
  }
  const long long E = qoff[nq];
  if (E >= 0x7fffffffLL) return set_error(CCO_E_UNSUPPORTED, "%lld training events of the query names, at most 2^31 - 2", E);
  const long long NT = lg->train_at.back();
  h->E = E;
  long long &G = h->G;
  StrTable &ut = h->ut, &it = h->it;
  DevStrCol &tu = h->tu, &ti = h->ti;
  uint32_t *&ent = h->ent, *&gord = h->gord, *&hord = h->hord;
  uint8_t *&qr = h->qr, *&keep_h = h->keep_h;
  int32_t *&uid = h->uid, *&iid = h->iid, *&d_limit = h->d_limit;
  long long *tm = nullptr, *&ln = h->ln, *&hstart = h->hstart;
  CKR(ar.alloc(&d_limit, std::max(nq, 1)));
  if (nq > 0) CK(cudaMemcpyAsync(d_limit, limits, sizeof(int32_t) * (size_t)nq, cudaMemcpyHostToDevice, s));
  if (E > 0) {
    long long *d_qoff, *d_qbase;
    CKR(ar.alloc(&d_qoff, nq + 1));
    CKR(ar.alloc(&d_qbase, nq));
    CK(cudaMemcpyAsync(d_qoff, qoff.data(), sizeof(long long) * (size_t)(nq + 1), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_qbase, qbase.data(), sizeof(long long) * (size_t)nq, cudaMemcpyHostToDevice, s));
    CKR(ar.alloc(&ent, E));
    CKR(ar.alloc(&qr, E));
    k_uq_select<<<grid_for(E, 256, c->sm_count), 256, 0, s>>>(E, nq, d_qoff, d_qbase, ent, qr);
    c->launches++;
    // 3. users and items grouped exactly (hash, then bytes) over the log's columns, gated to the query names' events
    int32_t *gate, *ugid, *igid;
    CKR(ar.alloc(&gate, NT));
    CK(cudaMemsetAsync(gate, 0xff, sizeof(int32_t) * (size_t)NT, s));
    for (int k = 0; k < nq; ++k)
      if (code[k] >= 0 && lg->n_train[code[k]] > 0)
        CK(cudaMemsetAsync(gate + lg->train_at[code[k]], 0, sizeof(int32_t) * (size_t)lg->n_train[code[k]], s));
    tu = lg->view(lg->tu, 0, lg->train_at, NT);
    ti = lg->view(lg->ti, 0, lg->train_at, NT);
    CKR(ar.alloc(&tu.hash, NT));
    CKR(ar.alloc(&ti.hash, NT));
    CKR(ar.alloc(&ugid, NT));
    CKR(ar.alloc(&igid, NT));
    str_hash(c, tu, ~0ULL);
    str_hash(c, ti, ~0ULL);
    CKR(str_group(c, ar, tu, gate, false, 0, &ut, ugid));
    CKR(str_group(c, ar, ti, gate, false, 0, &it, igid));
    G = ut.n_groups;
    if (G * (long long)nq >= (1LL << 32)) return set_error(CCO_E_UNSUPPORTED, "%lld users x %d names, at most 2^32 segments", G, nq);
    // 4. per event: user, item, time, line
    CKR(ar.alloc(&uid, E));
    CKR(ar.alloc(&iid, E));
    CKR(ar.alloc(&tm, E));
    CKR(ar.alloc(&ln, E));
    k_uq_gather<<<grid_for(E, 256, c->sm_count), 256, 0, s>>>(E, ent, ugid, igid, lg->ttime, lg->tline, uid, iid, tm, ln);
    c->launches++;
    // 5. latest first: line desc, then stably time desc
    unsigned long long *key;
    CKR(ar.alloc(&key, E));
    CKR(ar.alloc(&gord, E));
    k_uq_key_line<<<grid_for(E, 256, c->sm_count), 256, 0, s>>>(E, lg->n_lines, ln, key, gord);
    c->launches++;
    CKR(sort_pairs(c, ar, E, &key, &gord, bits_for(lg->n_lines)));
    k_uq_key_time<<<grid_for(E, 256, c->sm_count), 256, 0, s>>>(E, gord, tm, key);
    c->launches++;
    CKR(sort_pairs(c, ar, E, &key, &gord, 64));
    // 6. history order: stably by (user, name rank); segment starts
    CKR(ar.alloc(&hord, E));
    CK(cudaMemcpyAsync(hord, gord, sizeof(uint32_t) * (size_t)E, cudaMemcpyDeviceToDevice, s));
    k_uq_key_seg<<<grid_for(E, 256, c->sm_count), 256, 0, s>>>(E, nq, gord, uid, qr, key);
    c->launches++;
    CKR(sort_pairs(c, ar, E, &key, &hord, bits_for(G * nq)));
    long long *cnt;
    CKR(ar.alloc(&cnt, G * nq + 1));
    CKR(ar.alloc(&hstart, G * nq + 1));
    CK(cudaMemsetAsync(cnt, 0, sizeof(long long) * (size_t)(G * nq + 1), s));
    k_uq_count<<<grid_for(E, 256, c->sm_count), 256, 0, s>>>(E, key, cnt);
    c->launches++;
    CKR(exclusive_sum(c, ar, cnt, hstart, G * nq + 1));
    // 7. the first limit[q] of each segment, each item at its oldest position among them
    unsigned long long *k2;
    uint32_t *p2;
    CKR(ar.alloc(&k2, E));
    CKR(ar.alloc(&p2, E));
    CKR(ar.alloc(&keep_h, E));
    CK(cudaMemsetAsync(keep_h, 0, (size_t)E, s));
    k_uq_hist_keys<<<grid_for(E, 256, c->sm_count), 256, 0, s>>>(E, nq, key, hstart, d_limit, hord, iid, k2, p2);
    c->launches++;
    CKR(sort_pairs(c, ar, E, &k2, &p2, 64));
    k_uq_first<<<grid_for(E, 256, c->sm_count), 256, 0, s>>>(E, k2, p2, keep_h);
    c->launches++;
    ar.release(k2);
    ar.release(p2);
  }
  return uq_blacklist(c, ar, nq, black, h);
}
// 8. blacklist: the events of the names flagged in black latest first, stably by user; each item's newest position (into
//    h's bstart, bord, keep_b, bkey, B)
static int uq_blacklist(cco_ctx *c, Arena &ar, int nq, const std::vector<uint8_t> &black, UqHistory *h) {
  cudaStream_t s = c->stream;
  const long long E = h->E, G = h->G;
  long long &B = h->B;
  uint32_t *&bord = h->bord, *gord = h->gord;
  uint8_t *&keep_b = h->keep_b;
  long long *&bstart = h->bstart;
  unsigned long long *&bkey = h->bkey;
  if (E > 0) {
    uint8_t *d_black;
    CKR(ar.alloc(&d_black, nq));
    CK(cudaMemcpyAsync(d_black, black.data(), (size_t)nq, cudaMemcpyHostToDevice, s));
    uint32_t *flag, *pos, *bidx;
    CKR(ar.alloc(&flag, E + 1));
    k_uq_flag_black<<<grid_for(E, 256, c->sm_count), 256, 0, s>>>(E, gord, h->qr, d_black, flag);
    c->launches++;
    CKR(select_flagged(c, ar, E, flag, &pos, &bidx));
    uint32_t B32 = 0;
    CKR(mail_fetch(c, &B32, pos + E, 4));
    CKR(mail_wait(c));
    B = B32;
    CKR(ar.alloc(&bkey, std::max<long long>(B, 1)));
    CKR(ar.alloc(&bord, std::max<long long>(B, 1)));
    CKR(ar.alloc(&bstart, G + 1));
    CKR(ar.alloc(&keep_b, std::max<long long>(B, 1)));
    long long *bcnt;
    CKR(ar.alloc(&bcnt, G + 1));
    CK(cudaMemsetAsync(bcnt, 0, sizeof(long long) * (size_t)(G + 1), s));
    if (B > 0) {
      k_uq_key_user<<<grid_for(B, 256, c->sm_count), 256, 0, s>>>(B, bidx, gord, h->uid, bkey, bord);
      c->launches++;
      CKR(sort_pairs(c, ar, B, &bkey, &bord, bits_for(G)));
      k_uq_count<<<grid_for(B, 256, c->sm_count), 256, 0, s>>>(B, bkey, bcnt);
      uint32_t *p3;
      CKR(ar.alloc(&p3, B));
      k_uq_black_keys<<<grid_for(B, 256, c->sm_count), 256, 0, s>>>(B, bord, h->uid, h->iid, bkey, p3);
      c->launches += 2;
      CKR(sort_pairs(c, ar, B, &bkey, &p3, 64));
      CK(cudaMemsetAsync(keep_b, 0, (size_t)B, s));
      k_uq_first<<<grid_for(B, 256, c->sm_count), 256, 0, s>>>(B, bkey, p3, keep_b);
      c->launches++;
    }
    CKR(exclusive_sum(c, ar, bcnt, bstart, G + 1));
  }
  return CCO_OK;
}
// the user group of each of R records (-1: no training event of a query name); uc holds the records' user ids
static int uq_record_users(cco_ctx *c, const UqHistory &h, const DevStrCol &uc, long long R, int32_t *rec_uid) {
  cudaStream_t s = c->stream;
  if (R > 0 && h.E > 0) {
    str_hash(c, uc, ~0ULL);
    k_str_lookup<<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, uc.off, uc.base, uc.w, uc.hash, h.tu.off, h.tu.base, h.tu.w, h.tu.hash,
                                                              (uint64_t)h.ut.cap - 1, h.ut.table, h.ut.rank_of_slot, rec_uid);
    c->launches++;
  } else if (R > 0) {
    CK(cudaMemsetAsync(rec_uid, 0xff, sizeof(int32_t) * (size_t)R, s));
  }
  return CCO_OK;
}
// the history lists as the record kernel reads them
static UqArgs uq_args(const UqHistory &h, const cco_event_log *lg, int nq) {
  UqArgs a{};
  a.nq = nq;
  a.limit = h.d_limit;
  a.hstart = h.hstart;
  a.hord = h.hord;
  a.keep_h = h.keep_h;
  a.ent = h.ent;
  a.ioff = h.E > 0 ? lg->ti.off : nullptr;
  a.ibytes = h.E > 0 ? (const unsigned char *)lg->ti.w : nullptr;
  return a;
}
// every user with an event of a query name, in order of their first line: the rows' user groups (*rec_uid [h.G]) and, when
// users is not null, their ids
static int uq_every_user(cco_ctx *c, Arena &ar, const cco_event_log *lg, const UqHistory &h, int32_t **rec_uid, cco_dictionary_t *users) {
  cudaStream_t s = c->stream;
  const long long R = h.G;
  if (R > 0) {
    unsigned long long *mn, *uk;
    CKR(ar.alloc(&mn, R));
    CKR(ar.alloc(&uk, R));
    CK(cudaMemsetAsync(mn, 0xff, sizeof(unsigned long long) * (size_t)R, s));
    k_uq_min_line<<<grid_for(h.E, 256, c->sm_count), 256, 0, s>>>(h.E, h.uid, h.ln, mn);
    k_uq_user_keys<<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, mn, uk, *rec_uid);
    c->launches += 2;
    CKR(sort_pairs(c, ar, R, &uk, rec_uid, bits_for(lg->n_lines)));
  }
  if (!users) return CCO_OK;
  uint32_t *ue;
  long long *len, *off, total = 0;
  CKR(ar.alloc(&ue, std::max<long long>(R, 1)));
  CKR(ar.alloc(&len, R + 1));
  CKR(ar.alloc(&off, R + 1));
  CK(cudaMemsetAsync(len + R, 0, 8, s));
  if (R > 0) {
    k_uq_user_entry<<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, *rec_uid, h.ut.first_sorted, ue);
    k_str_dict_len<<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, ue, h.tu.off, len);
    c->launches += 2;
  }
  CKR(exclusive_sum(c, ar, len, off, R + 1));
  CK(cudaMemcpyAsync(&total, off + R, 8, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  unsigned char *ub;
  CKR(ar.alloc(&ub, std::max<long long>(total, 1)));
  if (R > 0 && total > 0) {
    k_str_dict_gather<<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, ue, h.tu.off, h.tu.base, (const unsigned char *)h.tu.w, off, ub);
    c->launches++;
  }
  int64_t *ho = (int64_t *)c->pinned_get(sizeof(int64_t) * ((size_t)R + 1), /*for_result=*/false);
  char *hb = (char *)c->pinned_get((size_t)std::max<long long>(total, 1), /*for_result=*/false);
  if (!ho || !hb) return set_error(CCO_E_OOM, "pinned host allocation failed");
  CK(cudaMemcpyAsync(ho, off, sizeof(int64_t) * ((size_t)R + 1), cudaMemcpyDeviceToHost, s));
  if (total > 0) CK(cudaMemcpyAsync(hb, ub, (size_t)total, cudaMemcpyDeviceToHost, s));
  *users = cco_dictionary_t{R, ho, hb};
  return CCO_OK;
}
}  // namespace cco

int cco_event_log_begin_ex(cco_ctx_t *ctx, int64_t chunk_bytes, const cco_event_window_t *w, uint32_t flags, cco_event_log_t **out) {
  if (flags & ~(uint32_t)(CCO_LOG_KEEP_HISTORY | CCO_LOG_EXTENDABLE | CCO_LOG_INTERN_IDS))
    return set_error(CCO_E_INVALID_ARG, "unknown flags 0x%x", (unsigned)flags);
  CKR(cco_event_log_begin_window(ctx, chunk_bytes, w, out));
  (*out)->history = (flags & CCO_LOG_KEEP_HISTORY) != 0;
  (*out)->extendable = (flags & CCO_LOG_EXTENDABLE) != 0;
  (*out)->intern = (flags & CCO_LOG_INTERN_IDS) != 0;
  (*out)->intern_mask = ctx->intern_mask;
  return CCO_OK;
}

namespace cco {
static int iq_check_host(const cco_item_query_t *q, int64_t n_items, const int64_t *ioff, const char *ibytes) {
  if (q->n_names < 1 || q->n_names > kUqMaxNames) return set_error(CCO_E_INVALID_ARG, "%d model event names, 1..%d", (int)q->n_names, kUqMaxNames);
  if (!q->names) return set_error(CCO_E_INVALID_ARG, "null names");
  for (int k = 0; k < q->n_names; ++k)
    if (!q->names[k] || !*q->names[k]) return set_error(CCO_E_INVALID_ARG, "model event name %d is null or empty", k);
  if (q->max_query_events < 1) return set_error(CCO_E_INVALID_ARG, "max_query_events = %d, at least 1", (int)q->max_query_events);
  if ((q->similar_in_must != 0 && q->similar_in_must != 1) || (q->exclude_self != 0 && q->exclude_self != 1))
    return set_error(CCO_E_INVALID_ARG, "similar_in_must and exclude_self must be 0 or 1");
  if (!q->head || !q->should_head || !q->should || !q->must_head || !q->must || !q->must_not || !q->sort || !q->header)
    return set_error(CCO_E_INVALID_ARG, "a null fragment");
  CKR(str_check_host(q->n_blacklist_items, q->blacklist_item_offsets, q->blacklist_item_bytes, 0, "blacklist item"));
  if (ioff) CKR(str_check_host(n_items, ioff, ibytes, 0, "item"));
  else if (n_items != 0) return set_error(CCO_E_INVALID_ARG, "n_items without item offsets");
  return CCO_OK;
}

// the documents' side of an item query: _ids are unique (gid: the key column's groups, the documents first)
static int iq_unique_ids(cco_ctx *c, Arena &ar, long long D, const int32_t *gid, const StrTable &tb) {
  cudaStream_t s = c->stream;
  if (D > 0) {
    unsigned long long *dup, h_dup = ~0ULL;
    CKR(ar.alloc(&dup, 1));
    CK(cudaMemsetAsync(dup, 0xff, 8, s));
    k_dup_rows<<<grid_for(D, 256, c->sm_count), 256, 0, s>>>(D, gid, tb.first_sorted, dup);
    c->launches++;
    CKR(mail_fetch(c, &h_dup, dup, 8));
    CKR(mail_wait(c));
    if (h_dup != ~0ULL)
      return set_error(CCO_E_INVALID_ARG, "document %llu: its _id is the _id of document %llu", h_dup >> 32, h_dup & 0xffffffffULL);
  }
  return CCO_OK;
}
// The similar-items lists of the queried documents: per document the last source member of each distinct model name,
// checked as an array of strings (only where queried[d]) and its elements decoded.  Element list (d, t) is
// dec[eoff[d * T + t] .. eoff[d * T + t + 1]); model name j is distinct name name_entry[j].
struct IqDocs {
  int T = 0;
  std::vector<int32_t> name_entry;
  long long *eoff = nullptr;   // [D * T + 1]
  DevStrCol dec;
};
static int iq_documents(cco_ctx *c, Arena &ar, const BulkDocs &bd, int n_names, const char *const *names, const uint8_t *queried,
                        IqDocs *o) {
  cudaStream_t s = c->stream;
  // 9. the distinct model names; per document the last source member of each
  std::vector<std::string> ent;
  std::vector<int32_t> &name_entry = o->name_entry;
  name_entry.assign(n_names, 0);
  for (int j = 0; j < n_names; ++j) {
    size_t t = 0;
    while (t < ent.size() && ent[t] != names[j]) ++t;
    if (t == ent.size()) ent.push_back(names[j]);
    name_entry[j] = (int32_t)t;
  }
  const int T = (int)ent.size();
  o->T = T;
  const long long D = bd.D, DT = D * T;
  long long *&eoff = o->eoff;
  CKR(ar.alloc(&eoff, DT + 1));
  CK(cudaMemsetAsync(eoff, 0, sizeof(long long) * (size_t)(DT + 1), s));
  DevStrCol &dec = o->dec;
  if (D > 0) {
    int32_t *ngid, *entry_of, *pick;
    CKR(member_entries(c, ar, bd.names, ent, &ngid, &entry_of));
    CKR(ar.alloc(&pick, DT));
    k_iq_pick<<<grid_for(D, 256, c->sm_count), 256, 0, s>>>(D, T, bd.line_moff, ngid, entry_of, pick);
    c->launches++;
    // 10. the queried documents' picked values: the verdict comes before anything reads through the element spans
    long long *cnt, NE = 0;
    unsigned long long *err, h_err = ~0ULL;
    CKR(ar.alloc(&cnt, DT + 1));
    CKR(ar.alloc(&err, 1));
    CK(cudaMemsetAsync(cnt + DT, 0, 8, s));
    CK(cudaMemsetAsync(err, 0xff, 8, s));
    const int agrid = grid_for(DT * 32, 256, c->sm_count);
    k_iq_array<false><<<agrid, 256, 0, s>>>(DT, T, queried, pick, bd.mem, bd.body, cnt, nullptr, nullptr, err);
    c->launches++;
    CKR(exclusive_sum(c, ar, cnt, eoff, DT + 1));
    CKR(mail_fetch(c, &h_err, err, 8));
    CKR(mail_fetch(c, &NE, eoff + DT, 8));
    CKR(mail_wait(c));
    if (h_err != ~0ULL)
      return set_error(CCO_E_INVALID_ARG, "document %lld: its \"%s\" member is not an array of strings", (long long)(h_err / T),
                       ent[h_err % T].c_str());
    JMember *elem;
    CKR(ar.alloc(&elem, std::max<long long>(NE, 1)));
    if (NE > 0) {
      k_iq_array<true><<<agrid, 256, 0, s>>>(DT, T, queried, pick, bd.mem, bd.body, nullptr, eoff, elem, err);
      c->launches++;
    }
    long long dec_bytes = 0;
    CKR(json_decode(c, ar, NE, elem, bd.body, &dec, &dec_bytes));
  }
  return CCO_OK;
}

static int is_check_host(const cco_item_set_query_t *q, long long n_sets, const int64_t *soff, long long n_elements, const int64_t *eoff,
                         const char *ebytes) {
  if (q->with_set != 0 && q->with_set != 1) return set_error(CCO_E_INVALID_ARG, "with_set must be 0 or 1");
  if (q->with_set && (!q->name || !*q->name)) return set_error(CCO_E_INVALID_ARG, "the set clause's name is null or empty");
  if (!q->head || !q->should_head || !q->should_tail || !q->must || !q->must_not || !q->sort || !q->header)
    return set_error(CCO_E_INVALID_ARG, "a null fragment");
  CKR(str_check_host(q->n_blacklist_items, q->blacklist_item_offsets, q->blacklist_item_bytes, 0, "blacklist item"));
  if (n_sets < 0 || n_elements < 0) return set_error(CCO_E_INVALID_ARG, "negative set or element count");
  if (n_sets >= 0x7fffffffLL) return set_error(CCO_E_UNSUPPORTED, "%lld sets, at most 2^31 - 2", n_sets);
  if (!soff) return set_error(CCO_E_INVALID_ARG, "null set offsets");
  if (soff[0] < 0 || soff[0] > soff[n_sets] || soff[n_sets] > n_elements)
    return set_error(CCO_E_INVALID_ARG, "set offsets [0] = %lld and [n_sets] = %lld are not within [0, n_elements = %lld] in order",
                     (long long)soff[0], (long long)soff[n_sets], n_elements);
  const long long NE = soff[n_sets] - soff[0];
  if (NE + q->n_blacklist_items >= 0x7fffffffLL)
    return set_error(CCO_E_UNSUPPORTED, "%lld elements + %lld blacklist items, at most 2^31 - 2", NE, (long long)q->n_blacklist_items);
  if (NE > 0) CKR(str_check_host(NE, eoff ? eoff + soff[0] : nullptr, ebytes, 0, "element"));
  return CCO_OK;
}

// What cco_event_log_user_queries, cco_item_queries and cco_item_set_queries add when they render their queries as rows of
// a mixed batch, each row with one member: the NVTX range; an item query's head clauses, written before the history and
// the similar items of should and must; the members the body's size check names; and a row source that is not a column,
// every user of the history or every document of the body, whose rows are fixed once they are known, with *keys (nullable)
// listing them.
enum : int { kMqColumns = 0, kMqEveryUser, kMqEveryDoc };
struct MqSingle {
  const char *range = "cco:mixed_queries";
  const char *should_head = "", *must_head = "";
  const char *what = "items + blacklist items + elements";
  int rows = kMqColumns;
  cco_dictionary_t *keys = nullptr;
};

// the record template of a mixed query, 13 + n_history_names + n_model_names pieces: 0 head and "should":[, 1 boosted,
// 2 should_tail, 3 must, 4 "],"must":[, 5 the ids clause up to its values, 6 the rest of the record, 7 the end of a history
// clause, 8 the end of a similar-items clause, 9 / 10 the start / end of the set clause, 11 / 12 should's / must's head,
// 13 + j the start of query name j's history clause, 13 + n_history_names + j the start of model name j's similar-items
// clause (see include/cco_b200.h)
static std::vector<std::string> mq_template(const cco_mixed_query_t *q, const MqSingle &x) {
  auto end = [](bool in_must, const char *boost) {
    return in_must ? std::string("],\"boost\":0}}") : boost ? std::string("],\"boost\":") + boost + "}}" : std::string("]}}");
  };
  std::vector<std::string> t(13);
  t[0] = query_head(q->header, q->head);
  t[1] = q->boosted;
  t[2] = q->should_tail;
  t[3] = q->must;
  t[4] = "],\"must\":[";
  t[5] = "],\"must_not\":[{\"ids\":{\"values\":[";
  t[6] = query_tail(q->must_not, q->sort);
  t[7] = end(q->history_in_must != 0, q->history_boost);
  t[8] = end(q->similar_in_must != 0, q->similar_boost);
  if (q->with_set) {
    t[9] = "{\"terms\":{" + uq_quote(q->set_name) + ":[";
    t[10] = end(false, q->set_boost);
  }
  t[11] = x.should_head;
  t[12] = x.must_head;
  for (int j = 0; j < q->n_history_names; ++j) t.push_back("{\"terms\":{" + uq_quote(q->names[j]) + ":[");
  for (int j = 0; j < q->n_model_names; ++j) t.push_back("{\"terms\":{" + uq_quote(q->model_names[j]) + ":[");
  return t;
}

// whether any of the R rows has the member: a column is given and its bitmap (nullptr: every row) has a bit set
static bool mq_any(long long R, const int64_t *off, const uint8_t *valid) {
  if (!off || R == 0) return false;
  if (!valid) return true;
  for (long long r = 0; r < R; ++r)
    if ((valid[r >> 3] >> (r & 7)) & 1) return true;
  return false;
}

static int mq_check_host(const cco_mixed_query_t *q, long long R, const int64_t *uoff, const char *ubytes, const int64_t *ioff,
                         const char *ibytes, const int64_t *soff, long long n_elements, const int64_t *eoff, const char *ebytes) {
  // the history, as uq_check_host
  if (q->n_names < 0 || q->n_names > kUqMaxNames) return set_error(CCO_E_INVALID_ARG, "%d query event names, 0..%d", (int)q->n_names, kUqMaxNames);
  if (q->n_names > 0 && (!q->names || (uoff && !q->limits))) return set_error(CCO_E_INVALID_ARG, "null names or limits");
  for (int k = 0; k < q->n_names; ++k) {
    if (!q->names[k] || !*q->names[k]) return set_error(CCO_E_INVALID_ARG, "query event name %d is null or empty", k);
    if (uoff && q->limits[k] < 0) return set_error(CCO_E_INVALID_ARG, "query event name %d: negative limit %d", k, (int)q->limits[k]);
  }
  if (q->n_history_names < 0 || q->n_history_names > q->n_names)
    return set_error(CCO_E_INVALID_ARG, "n_history_names = %d is outside [0, %d]", (int)q->n_history_names, (int)q->n_names);
  if (q->n_blacklist_names < 0 || (q->n_blacklist_names > 0 && !q->blacklist_names)) return set_error(CCO_E_INVALID_ARG, "bad blacklist names");
  for (int b = 0; b < q->n_blacklist_names; ++b)
    if (!q->blacklist_names[b]) return set_error(CCO_E_INVALID_ARG, "blacklist name %d is null", b);
  if (q->history_in_must != 0 && q->history_in_must != 1) return set_error(CCO_E_INVALID_ARG, "history_in_must must be 0 or 1");
  // the similar items, as iq_check_host; an item column needs a model name
  if (q->n_model_names < (ioff ? 1 : 0) || q->n_model_names > kUqMaxNames)
    return set_error(CCO_E_INVALID_ARG, "%d model event names, %d..%d", (int)q->n_model_names, ioff ? 1 : 0, kUqMaxNames);
  if (q->n_model_names > 0 && !q->model_names) return set_error(CCO_E_INVALID_ARG, "null names");
  for (int k = 0; k < q->n_model_names; ++k)
    if (!q->model_names[k] || !*q->model_names[k]) return set_error(CCO_E_INVALID_ARG, "model event name %d is null or empty", k);
  if (q->max_query_events < 1) return set_error(CCO_E_INVALID_ARG, "max_query_events = %d, at least 1", (int)q->max_query_events);
  if ((q->similar_in_must != 0 && q->similar_in_must != 1) || (q->exclude_self != 0 && q->exclude_self != 1))
    return set_error(CCO_E_INVALID_ARG, "similar_in_must and exclude_self must be 0 or 1");
  // the set clause, as is_check_host
  if (q->with_set != 0 && q->with_set != 1) return set_error(CCO_E_INVALID_ARG, "with_set must be 0 or 1");
  if (q->with_set && (!q->set_name || !*q->set_name)) return set_error(CCO_E_INVALID_ARG, "the set clause's name is null or empty");
  if (!q->head || !q->boosted || !q->should_tail || !q->must || !q->must_not || !q->sort || !q->header)
    return set_error(CCO_E_INVALID_ARG, "a null fragment");
  CKR(str_check_host(q->n_blacklist_items, q->blacklist_item_offsets, q->blacklist_item_bytes, 0, "blacklist item"));
  // the rows
  if (R < 0 || n_elements < 0) return set_error(CCO_E_INVALID_ARG, "negative row or element count");
  if (R >= 0x7fffffffLL) return set_error(CCO_E_UNSUPPORTED, "%lld rows, at most 2^31 - 2", R);
  if (uoff) CKR(str_check_host(R, uoff, ubytes, 0, "user"));
  if (ioff) CKR(str_check_host(R, ioff, ibytes, 0, "item"));
  long long NE = 0;
  if (soff) {
    if (soff[0] < 0 || soff[0] > soff[R] || soff[R] > n_elements)
      return set_error(CCO_E_INVALID_ARG, "set offsets [0] = %lld and [n_sets] = %lld are not within [0, n_elements = %lld] in order",
                       (long long)soff[0], (long long)soff[R], n_elements);
    NE = soff[R] - soff[0];
    if (NE > 0) CKR(str_check_host(NE, eoff ? eoff + soff[0] : nullptr, ebytes, 0, "element"));
  }
  const long long NI = ioff ? R : 0;
  if (NI + q->n_blacklist_items + NE >= 0x7fffffffLL)
    return set_error(CCO_E_UNSUPPORTED, "%lld items + %lld blacklist items + %lld elements, at most 2^31 - 2", NI, (long long)q->n_blacklist_items, NE);
  return CCO_OK;
}

// The rows of a mixed batch in HBM, as the two callers stage them: mixed_queries' columns (one template, one shared
// blacklistItems list) and a query file's lines (a template and a blacklistItems list per row).
struct MqRows {
  long long R = 0, NI = 0, NL = 0, NE = 0;   // rows; key entries of the items (R or 0), the lists and the elements
  std::vector<KeySection> sec;              // the items, the lists' entries, the elements (the key column after the _ids)
  DevStrCol uc;                             // the users (uc.n = R when a user column is given)
  bool col[3] = {false, false, false};      // a user, item, set column is given
  const uint8_t *valid[3] = {nullptr, nullptr, nullptr};   // device LSB-first bitmaps, nullptr: every row
  long long *soff = nullptr;                // [R + 1] 0-based element index of each row's set, nullptr: all 0
  long long *loff = nullptr;                // [lists + 1] entry index of each list
  bool list_shared = true;                  // one list for every row, else list r is row r's
  int32_t *rec_tpl = nullptr;               // [R] template of each row, nullptr: all 0
  std::vector<uint8_t> tpl_user;            // per template: a row with a user reads it
  MqSingle one;
};

// the union of the query names of the templates a row with a user reads, their limits, each template's history names in
// it and each distinct blacklist name mask over it (template -> mask)
struct MqNames {
  std::vector<const char *> names;
  std::vector<int32_t> limits, hbeg{0}, hname, tmask;
  std::vector<std::vector<uint8_t>> masks;
};
static int mq_names(const std::vector<const cco_mixed_query_t *> &tq, const std::vector<uint8_t> &tpl_user, bool single, MqNames *o) {
  const int T = (int)tq.size();
  auto find = [&](const char *n) {
    for (size_t k = 0; k < o->names.size(); ++k)
      if (strcmp(o->names[k], n) == 0) return (int)k;
    return -1;
  };
  for (int t = 0; t < T; ++t) {   // the union: cco_mixed_queries keeps its names as given (a repeated one reads the same events)
    if (!tpl_user[t]) continue;
    const cco_mixed_query_t *q = tq[t];
    for (int j = 0; j < q->n_names; ++j) {
      const int x = single ? -1 : find(q->names[j]);
      if (x >= 0) {
        if (o->limits[x] != q->limits[j])
          return set_error(CCO_E_INVALID_ARG, "template %d: query event name \"%s\" has limit %d, another template %d", t, q->names[j],
                           (int)q->limits[j], (int)o->limits[x]);
        continue;
      }
      if ((int)o->names.size() == kUqMaxNames)
        return set_error(CCO_E_UNSUPPORTED, "more than %d distinct query event names over the templates with a user", kUqMaxNames);
      o->names.push_back(q->names[j]);
      o->limits.push_back(q->limits[j]);
    }
  }
  for (int t = 0; t < T; ++t) {
    const cco_mixed_query_t *q = tq[t];
    for (int j = 0; j < q->n_history_names; ++j) o->hname.push_back(!tpl_user[t] ? -1 : single ? j : find(q->names[j]));
    o->hbeg.push_back((int32_t)o->hname.size());
  }
  // masks: the union names that are this template's query names and blacklist names (first occurrence only)
  const int nq = (int)o->names.size();
  o->tmask.assign(T, 0);
  for (int t = 0; t < T; ++t) {
    if (!tpl_user[t]) continue;
    const cco_mixed_query_t *q = tq[t];
    std::vector<uint8_t> m(std::max(nq, 1), 0);
    if (single) {
      m = uq_black_names(q->n_names, q->names, q->n_blacklist_names, q->blacklist_names);
    } else {
      for (int k = 0; k < nq; ++k) {
        bool in_q = false, in_b = false;
        for (int j = 0; j < q->n_names && !in_q; ++j) in_q = strcmp(q->names[j], o->names[k]) == 0;
        for (int b = 0; b < q->n_blacklist_names && !in_b; ++b) in_b = strcmp(q->blacklist_names[b], o->names[k]) == 0;
        m[k] = in_q && in_b;
      }
    }
    size_t x = 0;
    while (x < o->masks.size() && o->masks[x] != m) ++x;
    if (x == o->masks.size()) o->masks.push_back(m);
    o->tmask[t] = (int32_t)x;
  }
  return CCO_OK;
}

// Steps shared by every query builder: the documents, one key column (_ids, items, blacklistItems, elements), the history
// over the union of the templates' names, each row's members, the lists' and sets' first occurrences, and the records.
// *bad holds the device verdict on the caller's offsets so far.
static int mixed_render(cco_ctx *c, Arena &ar, const cco_event_log *lg, const char *body, int64_t body_len,
                        const std::vector<const cco_mixed_query_t *> &tq, MqRows &in, int *bad, char **out_body, int64_t *out_len,
                        int64_t **out_offsets, int64_t *out_n) {
  cudaStream_t s = c->stream;
  const long long NI = in.NI, NL = in.NL, NE = in.NE;
  long long R = in.R;
  const cco_mixed_query_t *q0 = tq[0];
  const int T = (int)tq.size();
  bool any_user = false;
  for (uint8_t x : in.tpl_user) any_user |= x != 0;
  // 1. the documents of the index body: members, decoded names and _ids
  BulkDocs bd;
  if (body) CKR(bulk_parse(c, ar, body, body_len, NI + NL + NE, in.one.what, &bd));
  const long long D = bd.D;
  if (in.one.rows == kMqEveryDoc) R = D;   // row r is document r, its item key entry r (its own _id)
  // 2. one key column of the decoded _ids, the items, blacklistItems and the elements
  std::vector<KeySection> sec{KeySection{D, (const int64_t *)bd.ids.off, (const char *)bd.ids.w, true, bd.ids_bytes}};
  sec.insert(sec.end(), in.sec.begin(), in.sec.end());
  DevStrCol key;
  int h_bad = 0;
  CKR(key_column(c, ar, sec, bad, &key));
  CKR(mail_fetch(c, &h_bad, bad, 4));
  CKR(mail_wait(c));
  if (h_bad) return set_error(CCO_E_INVALID_ARG, "decreasing offsets in the users, the items, the sets, the elements or the blacklist items");
  // 3. one exact grouping over the key column: _ids are unique
  str_hash(c, key, ~0ULL);
  int32_t *gid;
  CKR(ar.alloc(&gid, std::max<long long>(key.n, 1)));
  StrTable tb;
  CKR(str_group(c, ar, key, nullptr, false, 0, &tb, gid));
  CKR(iq_unique_ids(c, ar, D, gid, tb));
  // 4. blacklistItems: each entry's first occurrence within its list and each list's sorted (list << 32 | group) keys,
  //    from one stable sort (membership is a search of the row's list)
  const long long n_lists = in.list_shared ? 1 : R;
  uint8_t *first_in_list;
  unsigned long long *lkey;
  CKR(ar.alloc(&first_in_list, std::max<long long>(NL, 1)));
  CKR(ar.alloc(&lkey, std::max<long long>(NL, 1)));
  if (NL > 0) {
    uint32_t *p2;
    CKR(ar.alloc(&p2, NL));
    CK(cudaMemsetAsync(first_in_list, 0, (size_t)NL, s));
    k_is_keys<<<grid_for(NL, 256, c->sm_count), 256, 0, s>>>(NL, n_lists, in.loff, gid + D + NI, lkey, p2);
    c->launches++;
    CKR(sort_pairs(c, ar, NL, &lkey, &p2, 32 + bits_for(n_lists)));
    k_uq_first<<<grid_for(NL, 256, c->sm_count), 256, 0, s>>>(NL, lkey, p2, first_in_list);
    c->launches++;
  }
  // 5. the history over the union of names, when a row has a user; each row's user group; one user blacklist per mask
  MqNames nm;
  CKR(mq_names(tq, in.tpl_user, T == 1 && in.list_shared, &nm));
  const int nq = (int)nm.names.size();
  UqHistory h;
  std::vector<MqBlack> hb;
  if (any_user) {
    CKR(uq_history(c, ar, lg, nq, nm.names.data(), nm.limits.data(), nm.masks[0], &h));
    hb.push_back(MqBlack{h.bstart, h.bkey, h.bord, h.keep_b});
    for (size_t m = 1; m < nm.masks.size(); ++m) {
      CKR(uq_blacklist(c, ar, nq, nm.masks[m], &h));
      hb.push_back(MqBlack{h.bstart, h.bkey, h.bord, h.keep_b});
    }
  }
  if (hb.empty()) hb.push_back(MqBlack{nullptr, nullptr, nullptr, nullptr});
  if (in.one.rows == kMqEveryUser) R = h.G;
  int32_t *rec_uid;
  CKR(ar.alloc(&rec_uid, std::max<long long>(R, 1)));
  if (in.one.rows == kMqEveryUser) CKR(uq_every_user(c, ar, lg, h, &rec_uid, in.one.keys));
  else if (any_user) CKR(uq_record_users(c, h, in.uc, R, rec_uid));
  else if (R > 0) CK(cudaMemsetAsync(rec_uid, 0xff, sizeof(int32_t) * (size_t)R, s));
  // a caller without sets or templates: every row's set is empty and its template 0
  long long *soff = in.soff;
  int32_t *rec_tpl = in.rec_tpl;
  if (!soff) {
    CKR(ar.alloc(&soff, R + 1));
    CK(cudaMemsetAsync(soff, 0, sizeof(long long) * ((size_t)R + 1), s));
  }
  if (!rec_tpl) {
    CKR(ar.alloc(&rec_tpl, std::max<long long>(R, 1)));
    CK(cudaMemsetAsync(rec_tpl, 0, sizeof(int32_t) * (size_t)std::max<long long>(R, 1), s));
  }
  // 6. each row's members and document; the queried documents
  int32_t *rec_doc, *rec_key;
  uint8_t *rec_set, *queried;
  CKR(ar.alloc(&rec_doc, std::max<long long>(R, 1)));
  CKR(ar.alloc(&rec_key, std::max<long long>(R, 1)));
  CKR(ar.alloc(&rec_set, std::max<long long>(R, 1)));
  CKR(ar.alloc(&queried, std::max<long long>(D, 1)));
  CK(cudaMemsetAsync(queried, 0, (size_t)std::max<long long>(D, 1), s));
  if (R > 0) {
    k_mq_rows<<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, in.valid[0], in.valid[1], in.valid[2], in.col[0], in.col[1], in.col[2], D,
                                                           in.one.rows == kMqEveryDoc ? 0 : D, gid, tb.first_sorted, rec_uid, rec_doc,
                                                           rec_key, rec_set, queried);
    c->launches++;
  }
  // 7. the queried documents' similar-items lists (the model names are the algorithm's: every template has the same)
  IqDocs docs;
  CKR(iq_documents(c, ar, bd, q0->n_model_names, q0->model_names, queried, &docs));
  // 8. the items, blacklistItems and elements in the log's item table: the user's blacklist is a group test there
  int32_t *klog;
  CKR(ar.alloc(&klog, std::max<long long>(key.n, 1)));
  CK(cudaMemsetAsync(klog, 0xff, sizeof(int32_t) * (size_t)std::max<long long>(key.n, 1), s));
  if (h.E > 0 && key.n > D) {
    k_str_lookup<<<grid_for(key.n - D, 256, c->sm_count), 256, 0, s>>>(key.n - D, key.off + D, key.base, key.w, key.hash + D, h.ti.off, h.ti.base,
                                                                       h.ti.w, h.ti.hash, (uint64_t)h.it.cap - 1, h.it.table,
                                                                       h.it.rank_of_slot, klog + D);
    c->launches++;
  }
  // 9. each element's first occurrence within its set: the first of each run of (row, group) keys after a stable sort
  uint8_t *first_in_set;
  CKR(ar.alloc(&first_in_set, std::max<long long>(NE, 1)));
  if (NE > 0) {
    unsigned long long *k2;
    uint32_t *p2;
    CKR(ar.alloc(&k2, NE));
    CKR(ar.alloc(&p2, NE));
    CK(cudaMemsetAsync(first_in_set, 0, (size_t)NE, s));
    k_is_keys<<<grid_for(NE, 256, c->sm_count), 256, 0, s>>>(NE, R, soff, gid + D + NI + NL, k2, p2);
    c->launches++;
    CKR(sort_pairs(c, ar, NE, &k2, &p2, 32 + bits_for(R)));
    k_uq_first<<<grid_for(NE, 256, c->sm_count), 256, 0, s>>>(NE, k2, p2, first_in_set);
    c->launches++;
    ar.release(k2);
    ar.release(p2);
  }
  // 10. every template's pieces and per-template arrays, then a length pass, the record offsets and a write pass: one warp
  //     per row
  std::vector<std::string> pieces;
  std::vector<int32_t> tpiece(T);
  std::vector<uint8_t> tflag(T);
  for (int t = 0; t < T; ++t) {
    const cco_mixed_query_t *q = tq[t];
    tpiece[t] = (int32_t)pieces.size();
    std::vector<std::string> p = mq_template(q, in.one);
    pieces.insert(pieces.end(), p.begin(), p.end());
    tflag[t] = (uint8_t)((q->history_in_must ? kMqHistInMust : 0) | (q->similar_in_must ? kMqSimilarInMust : 0) |
                         (q->exclude_self ? kMqExcludeSelf : 0) | (q->with_set ? kMqWithSet : 0));
  }
  int32_t *d_entry, *d_tpiece, *d_hbeg, *d_hname, *d_tmask;
  uint8_t *d_tflag;
  MqBlack *d_black;
  auto up = [&](auto **dst, const auto &v) -> int {
    CKR(ar.alloc(dst, std::max<size_t>(v.size(), 1)));
    if (!v.empty()) CK(cudaMemcpyAsync(*dst, v.data(), sizeof(v[0]) * v.size(), cudaMemcpyHostToDevice, s));
    return CCO_OK;
  };
  CKR(up(&d_entry, docs.name_entry));
  CKR(up(&d_tpiece, tpiece));
  CKR(up(&d_hbeg, nm.hbeg));
  CKR(up(&d_hname, nm.hname));
  CKR(up(&d_tmask, nm.tmask));
  CKR(up(&d_tflag, tflag));
  CKR(up(&d_black, hb));
  DevDict tp;
  CKR(upload_strings(c, ar, pieces, &tp));   // waits for the copies above too: the host vectors are local
  MqArgs a{};
  a.n_rec = R;
  a.rec_uid = rec_uid;
  a.rec_doc = rec_doc;
  a.rec_key = rec_key;
  a.rec_set = rec_set;
  a.rec_tpl = rec_tpl;
  a.h = uq_args(h, lg, nq);
  a.tpiece = d_tpiece;
  a.hbeg = d_hbeg;
  a.hname = d_hname;
  a.tflag = d_tflag;
  a.tmask = d_tmask;
  a.black = d_black;
  a.kgid = gid;
  a.koff = key.off;
  a.kbytes = (const unsigned char *)key.w;
  a.klog = klog;
  a.line_moff = bd.line_moff;
  a.T = docs.T;
  a.n_names = q0->n_model_names;
  a.name_entry = d_entry;
  a.eoff = docs.eoff;
  a.doff = docs.dec.off;
  a.dbytes = (const unsigned char *)docs.dec.w;
  a.slice = q0->max_query_events;
  a.list_at = D + NI;
  a.loff = in.loff;
  a.list_shared = in.list_shared;
  a.first_in_list = first_in_list;
  a.lkey = lkey;
  a.soff = soff;
  a.elem_at = D + NI + NL;
  a.first_in_set = first_in_set;
  a.toff = tp.off;
  a.tbytes = tp.bytes;
  return emit_records(c, ar, R, k_mq_record<false>, k_mq_record<true>, a, out_body, out_len, out_offsets, out_n, [&]() -> int {
    if (in.one.rows != kMqEveryDoc || !in.one.keys) return CCO_OK;
    // the documents' decoded _ids, in body order
    int64_t *io = (int64_t *)c->pinned_get(sizeof(int64_t) * ((size_t)D + 1), /*for_result=*/false);
    char *ib = (char *)c->pinned_get((size_t)std::max<long long>(bd.ids_bytes, 1), /*for_result=*/false);
    if (!io || !ib) return set_error(CCO_E_OOM, "pinned host allocation failed");
    io[0] = 0;
    if (D > 0) CK(cudaMemcpyAsync(io, bd.ids.off, sizeof(int64_t) * ((size_t)D + 1), cudaMemcpyDeviceToHost, s));
    if (bd.ids_bytes > 0) CK(cudaMemcpyAsync(ib, bd.ids.w, (size_t)bd.ids_bytes, cudaMemcpyDeviceToHost, s));
    *in.one.keys = cco_dictionary_t{D, io, ib};
    return CCO_OK;
  });
}

static int mixed_queries(cco_ctx *c, const cco_event_log *lg, const char *body, int64_t body_len, const cco_mixed_query_t *q, long long R,
                         const int64_t *uoff, const char *ubytes, const uint8_t *uval, const int64_t *ioff, const char *ibytes,
                         const uint8_t *ival, const int64_t *set_off, const int64_t *eoff, const char *ebytes, const uint8_t *sval,
                         bool any_user, const MqSingle &one, char **out_body, int64_t *out_len, int64_t **out_offsets, int64_t *out_n) {
  cudaStream_t s = c->stream;
  CK(cudaSetDevice(c->device));
  Arena ar(s);
  NvtxRange nvtx(one.range);
  mail_reset(c);
  MqRows in;
  in.one = one;
  in.R = R;
  in.NI = ioff ? R : 0;
  in.NL = q->n_blacklist_items;
  const long long s0 = set_off ? set_off[0] : 0;
  in.NE = set_off ? set_off[R] - s0 : 0;
  // the users, the validity bitmaps, the set offsets 0-based and the one shared list; every column's offsets are checked
  // on the device before any kernel reads through them
  int *bad;
  CKR(ar.alloc(&bad, 1));
  CK(cudaMemsetAsync(bad, 0, sizeof(int), s));
  if (uoff) {
    CKR(str_upload(c, ar, R, uoff, ubytes, &in.uc));
    str_check_device(c, in.uc, bad);
  }
  const uint8_t *h_valid[3] = {uval, ival, sval};
  for (int k = 0; k < 3; ++k)
    if (h_valid[k] && R > 0) {
      uint8_t *d;
      CKR(ar.alloc(&d, (R + 7) / 8));
      CK(cudaMemcpyAsync(d, h_valid[k], (size_t)(R + 7) / 8, cudaMemcpyHostToDevice, s));
      in.valid[k] = d;
    }
  in.col[0] = uoff != nullptr || one.rows == kMqEveryUser;
  in.col[1] = ioff != nullptr || one.rows == kMqEveryDoc;
  in.col[2] = set_off != nullptr;
  if (set_off) {
    long long *stmp;
    CKR(ar.alloc(&in.soff, R + 1));
    CKR(ar.alloc(&stmp, R + 1));
    CK(cudaMemcpyAsync(stmp, set_off, sizeof(int64_t) * ((size_t)R + 1), cudaMemcpyHostToDevice, s));
    if (R > 0) {
      k_str_check<<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, stmp, bad);
      c->launches++;
    }
    k_rebase<<<grid_for(R + 1, 256, c->sm_count), 256, 0, s>>>(R + 1, stmp, -s0, in.soff);
    c->launches++;
  }
  const long long lo[2] = {0, in.NL};
  CKR(ar.alloc(&in.loff, 2));
  CK(cudaMemcpyAsync(in.loff, lo, sizeof lo, cudaMemcpyHostToDevice, s));
  in.sec = {KeySection{in.NI, ioff, ibytes}, KeySection{in.NL, q->blacklist_item_offsets, q->blacklist_item_bytes},
            KeySection{in.NE, eoff ? eoff + s0 : nullptr, ebytes}};
  in.tpl_user = {(uint8_t)(any_user ? 1 : 0)};
  CK(cudaStreamSynchronize(s));   // lo is local
  return mixed_render(c, ar, lg, body, body_len, {q}, in, bad, out_body, out_len, out_offsets, out_n);
}
}  // namespace cco

int cco_mixed_queries(cco_ctx_t *ctx, const cco_event_log_t *lg, const char *index_body, int64_t index_len, const cco_mixed_query_t *q,
                      int64_t n_rows, const int64_t *user_offsets, const char *user_bytes, const uint8_t *user_validity,
                      const int64_t *item_offsets, const char *item_bytes, const uint8_t *item_validity, const int64_t *set_offsets,
                      int64_t n_elements, const int64_t *elem_offsets, const char *elem_bytes, const uint8_t *set_validity, char **out_body,
                      int64_t *out_len, int64_t **out_offsets, int64_t *out_n) {
  if (!ctx || !q || !out_body || !out_len || !out_offsets || !out_n || index_len < 0 || (index_len > 0 && !index_body))
    return set_error(CCO_E_INVALID_ARG, "null argument or negative length");
  if (!ctx->members.empty()) return set_error(CCO_E_UNSUPPORTED, "per-GPU contexts only");
  if (lg && lg->ctx != ctx) return set_error(CCO_E_INVALID_ARG, "the log was read on another context");
  if (lg) CKR(log_state(lg, true));
  if (index_len > 0 && index_body[index_len - 1] != '\n') return set_error(CCO_E_INVALID_ARG, "the body does not end in a newline");
  CKR(mq_check_host(q, n_rows, user_offsets, user_bytes, item_offsets, item_bytes, set_offsets, n_elements, elem_offsets, elem_bytes));
  const bool any_user = mq_any(n_rows, user_offsets, user_validity);
  if (any_user && !lg) return set_error(CCO_E_INVALID_ARG, "a row has a user: its history needs a log (cco_event_log_begin_ex, CCO_LOG_KEEP_HISTORY)");
  if (any_user && !lg->history)
    return set_error(CCO_E_INVALID_ARG, "the log was read without history retention (cco_event_log_begin_ex, CCO_LOG_KEEP_HISTORY)");
  if (mq_any(n_rows, item_offsets, item_validity) && !index_body)
    return set_error(CCO_E_INVALID_ARG, "a row has an item: its similar items need an index body");
  return mixed_queries(ctx, lg, index_body, index_len, q, n_rows, user_offsets, user_bytes, user_validity, item_offsets, item_bytes,
                       item_validity, set_offsets, elem_offsets, elem_bytes, set_validity, any_user, MqSingle{}, out_body, out_len,
                       out_offsets, out_n);
}

// ---- the single builders: each query a row of a mixed batch with one member -------------------------------------------
int cco_event_log_user_queries(cco_ctx_t *ctx, const cco_event_log_t *lg, const cco_user_query_t *q, int64_t n_users,
                               const int64_t *user_offsets, const char *user_bytes, char **out_body, int64_t *out_len,
                               int64_t **out_offsets, int64_t *out_n, cco_dictionary_t *out_users) {
  if (!ctx || !lg || !q || !out_body || !out_len || !out_offsets || !out_n) return set_error(CCO_E_INVALID_ARG, "null argument");
  if (!ctx->members.empty() || lg->ctx != ctx) return set_error(CCO_E_UNSUPPORTED, "build queries on the per-GPU context that read the log");
  CKR(log_state(lg, true));
  CKR(uq_check_host(q, n_users, user_offsets, user_bytes));
  if (!lg->history) return set_error(CCO_E_INVALID_ARG, "the log was read without history retention (cco_event_log_begin_ex, CCO_LOG_KEEP_HISTORY)");
  if (out_users) *out_users = cco_dictionary_t{0, nullptr, nullptr};
  cco_mixed_query_t m{};
  m.n_names = q->n_names;
  m.n_history_names = q->n_history_names;
  m.names = q->names;
  m.limits = q->limits;
  m.n_blacklist_names = q->n_blacklist_names;
  m.history_in_must = q->history_in_must;
  m.blacklist_names = q->blacklist_names;
  m.history_boost = q->boost;
  m.max_query_events = 1;
  m.head = q->head;
  m.boosted = q->should;
  m.should_tail = "";
  m.must = q->must;
  m.must_not = q->must_not;
  m.sort = q->sort;
  m.header = q->header;
  m.n_blacklist_items = q->n_blacklist_items;
  m.blacklist_item_offsets = q->blacklist_item_offsets;
  m.blacklist_item_bytes = q->blacklist_item_bytes;
  MqSingle one;
  one.range = "cco:user_queries";
  if (!user_offsets) {
    one.rows = kMqEveryUser;
    one.keys = out_users;
  }
  // the history is built even for no row
  return mixed_queries(ctx, lg, nullptr, 0, &m, user_offsets ? n_users : 0, user_offsets, user_bytes, nullptr, nullptr, nullptr, nullptr,
                       nullptr, nullptr, nullptr, nullptr, true, one, out_body, out_len, out_offsets, out_n);
}

int cco_item_queries(cco_ctx_t *ctx, const char *index_body, int64_t index_len, const cco_item_query_t *q, int64_t n_items,
                     const int64_t *item_offsets, const char *item_bytes, char **out_body, int64_t *out_len, int64_t **out_offsets,
                     int64_t *out_n, cco_dictionary_t *out_items) {
  if (!ctx || !q || !out_body || !out_len || !out_offsets || !out_n || index_len < 0 || (index_len > 0 && !index_body))
    return set_error(CCO_E_INVALID_ARG, "null argument or negative length");
  if (!ctx->members.empty()) return set_error(CCO_E_UNSUPPORTED, "per-GPU contexts only");
  if (index_len > 0 && index_body[index_len - 1] != '\n') return set_error(CCO_E_INVALID_ARG, "the body does not end in a newline");
  CKR(iq_check_host(q, n_items, item_offsets, item_bytes));
  if (out_items) *out_items = cco_dictionary_t{0, nullptr, nullptr};
  cco_mixed_query_t m{};
  m.n_model_names = q->n_names;
  m.model_names = q->names;
  m.max_query_events = q->max_query_events;
  m.similar_in_must = q->similar_in_must;
  m.similar_boost = q->similar_boost;
  m.exclude_self = q->exclude_self;
  m.head = q->head;
  m.boosted = "";
  m.should_tail = q->should;
  m.must = q->must;
  m.must_not = q->must_not;
  m.sort = q->sort;
  m.header = q->header;
  m.n_blacklist_items = q->n_blacklist_items;
  m.blacklist_item_offsets = q->blacklist_item_offsets;
  m.blacklist_item_bytes = q->blacklist_item_bytes;
  MqSingle one;
  one.range = "cco:item_queries";
  one.should_head = q->should_head;
  one.must_head = q->must_head;
  one.what = "items + blacklist items";
  if (!item_offsets) {
    one.rows = kMqEveryDoc;
    one.keys = out_items;
  }
  // an empty body, NULL or not, holds no document
  return mixed_queries(ctx, nullptr, index_len > 0 ? index_body : "", index_len, &m, item_offsets ? n_items : 0, nullptr, nullptr, nullptr,
                       item_offsets, item_bytes, nullptr, nullptr, nullptr, nullptr, nullptr, false, one, out_body, out_len, out_offsets,
                       out_n);
}

int cco_item_set_queries(cco_ctx_t *ctx, const cco_item_set_query_t *q, int64_t n_sets, const int64_t *set_offsets, int64_t n_elements,
                         const int64_t *elem_offsets, const char *elem_bytes, char **out_body, int64_t *out_len, int64_t **out_offsets,
                         int64_t *out_n) {
  if (!ctx || !q || !out_body || !out_len || !out_offsets || !out_n) return set_error(CCO_E_INVALID_ARG, "null argument");
  if (!ctx->members.empty()) return set_error(CCO_E_UNSUPPORTED, "per-GPU contexts only");
  CKR(is_check_host(q, n_sets, set_offsets, n_elements, elem_offsets, elem_bytes));
  cco_mixed_query_t m{};
  m.max_query_events = 1;
  m.set_name = q->name;
  m.with_set = q->with_set;
  m.set_boost = q->boost;
  m.head = q->head;
  m.boosted = q->should_head;
  m.should_tail = q->should_tail;
  m.must = q->must;
  m.must_not = q->must_not;
  m.sort = q->sort;
  m.header = q->header;
  m.n_blacklist_items = q->n_blacklist_items;
  m.blacklist_item_offsets = q->blacklist_item_offsets;
  m.blacklist_item_bytes = q->blacklist_item_bytes;
  MqSingle one;
  one.range = "cco:item_set_queries";
  return mixed_queries(ctx, nullptr, nullptr, 0, &m, n_sets, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, set_offsets, elem_offsets,
                       elem_bytes, nullptr, false, one, out_body, out_len, out_offsets, out_n);
}

// ---- batchpredict query files: the lines read on the device, the templates planned by the caller, the rows rendered -----
struct cco_query_file {
  cco_ctx *ctx = nullptr;
  long long L = 0, NL = 0, NE = 0, rows_bytes = 0;
  std::vector<void *> dev;
  DevStrCol uc, rows;                  // decoded users [L]; decoded items [L], blacklistItems entries [NL], elements [NE]
  long long *soff = nullptr, *loff = nullptr;
  uint8_t *bits = nullptr;             // 3 LSB-first bitmaps of (L + 7) / 8 bytes: user, item, set present
  int32_t *tid = nullptr;              // [L] template by first appearance
  std::vector<int64_t> key_off, first_line, first_member;   // first_member: [3 T] first line with a user, item, set; -1
  std::string key_bytes;
};

namespace cco {
static const char *const kQfNames[kQfMembers] = {"user", "item", "itemSet", "blacklistItems", "withRanks", "fields", "dateRange",
                                                 "currentDate", "returnSelf", "num", "from", "eventNames", "userBias", "itemBias",
                                                 "itemSetBias"};
static int qf_line_error(unsigned long long err) {
  const long long line = (long long)(err >> 8);
  switch ((unsigned)(err & 0xff)) {
    case kJsonLongLine: return set_error(CCO_E_UNSUPPORTED, "line %lld: longer than 2^31 - 1 bytes", line);
    case kJsonNotObject: return set_error(CCO_E_INVALID_ARG, "line %lld: not a JSON object (an empty line is not a query)", line);
    case kJsonString:
      return set_error(CCO_E_INVALID_ARG, "line %lld: not one JSON object (a string is unterminated or holds a bad escape or a raw byte < 0x20)", line);
    default: return set_error(CCO_E_INVALID_ARG, "line %lld: not one JSON object", line);
  }
}
static int qf_keep(Arena &ar, cco_query_file *qf, void *p) {
  ar.take(p);
  qf->dev.push_back(p);
  return CCO_OK;
}
// the array members of every line picked in pick (-1: none) -> element spans at elem, per-line offsets eoff [L + 1]
static int qf_arrays(cco_ctx *c, Arena &ar, long long L, const uint8_t *ones, const int32_t *pick, const JMember *mem, const unsigned char *bb,
                     const char *what, long long **eoff, long long *n, JMember **elem) {
  cudaStream_t s = c->stream;
  long long *cnt;
  unsigned long long *err, h_err = ~0ULL;
  CKR(ar.alloc(&cnt, L + 1));
  CKR(ar.alloc(eoff, L + 1));
  CKR(ar.alloc(&err, 1));
  CK(cudaMemsetAsync(cnt + L, 0, 8, s));
  CK(cudaMemsetAsync(err, 0xff, 8, s));
  const int grid = grid_for(L * 32, 256, c->sm_count);
  if (L > 0) k_iq_array<false><<<grid, 256, 0, s>>>(L, 1, ones, pick, mem, bb, cnt, nullptr, nullptr, err);
  CKR(exclusive_sum(c, ar, cnt, *eoff, L + 1));
  CKR(mail_fetch(c, &h_err, err, 8));
  CKR(mail_fetch(c, n, *eoff + L, 8));
  CKR(mail_wait(c));
  if (h_err != ~0ULL) return set_error(CCO_E_INVALID_ARG, "line %lld: \"%s\" is not an array of strings", (long long)h_err, what);
  CKR(ar.alloc(elem, std::max<long long>(*n, 1)));
  if (*n > 0) k_iq_array<true><<<grid, 256, 0, s>>>(L, 1, ones, pick, mem, bb, nullptr, *eoff, *elem, err);
  c->launches += 2;
  return CCO_OK;
}
static int query_file_read(cco_ctx *c, const char *bytes, int64_t len, cco_query_file *qf) {
  cudaStream_t s = c->stream;
  CK(cudaSetDevice(c->device));
  Arena ar(s);
  NvtxRange nvtx("cco:query_file_read");
  mail_reset(c);
  // 1. the file as 8-byte words with 16 bytes of zero padding; its lines (a final '\n' opens none)
  const long long NW = (len + 7) / 8;
  uint64_t *w;
  CKR(ar.alloc(&w, NW + 2));
  CK(cudaMemsetAsync(w + len / 8, 0, sizeof(uint64_t) * (size_t)(NW + 2 - len / 8), s));
  if (len > 0) CK(cudaMemcpyAsync(w, bytes, (size_t)len, cudaMemcpyHostToDevice, s));
  const unsigned char *bb = (const unsigned char *)w;
  long long L = 0, *sb = nullptr, *se = nullptr;
  CKR(split_lines(c, ar, w, len, len > 0 && bytes[len - 1] != '\n', &L, &sb, &se));
  if (L >= 0x7fffffffLL) return set_error(CCO_E_UNSUPPORTED, "%lld lines, at most 2^31 - 2", L);
  qf->L = L;
  // 2. every line one object (the verdict before anything reads through the spans); member names decoded and matched
  long long *moff = nullptr, M = 0;
  JMember *mem = nullptr;
  unsigned long long h_err = ~0ULL;
  if (L > 0) {
    CKR(json_members(c, ar, L, sb, se, bb, 0x7fffffffLL, &h_err, &moff, &mem, &M));
    if (h_err != ~0ULL) return qf_line_error(h_err);
    if (M >= 0x7fffffffLL) return set_error(CCO_E_UNSUPPORTED, "%lld members in the file, at most 2^31 - 2", M);
  }
  DevStrCol names;
  long long name_bytes = 0;
  CKR(json_decode(c, ar, M, mem, bb, &names, &name_bytes));
  int32_t *ngid, *entry_of;
  CKR(member_entries(c, ar, names, std::vector<std::string>(kQfNames, kQfNames + kQfMembers), &ngid, &entry_of));
  // 3. per line: the known members, once each, null = absent; user and item are strings
  JMember *uspan;
  int32_t *pick_set, *pick_list, *tmem;
  uint8_t *has, *ones;
  unsigned long long *err;
  const long long L1 = std::max<long long>(L, 1);
  CKR(ar.alloc(&uspan, L1));
  CKR(ar.alloc(&pick_set, L1));
  CKR(ar.alloc(&pick_list, L1));
  CKR(ar.alloc(&tmem, L1 * kQfTemplateMembers));
  CKR(ar.alloc(&has, L1));
  CKR(ar.alloc(&ones, L1));
  CKR(ar.alloc(&err, 1));
  CK(cudaMemsetAsync(ones, 1, (size_t)L1, s));
  CK(cudaMemsetAsync(err, 0xff, 8, s));
  // the item spans go first in the decoded row column, the list entries and the elements after them (sized below)
  JMember *ispan;
  CKR(ar.alloc(&ispan, L1));
  if (L > 0) {
    k_qf_lines<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, moff, mem, ngid, entry_of, bb, uspan, ispan, pick_set, pick_list, tmem, has, err);
    c->launches++;
  }
  CKR(mail_fetch(c, &h_err, err, 8));
  CKR(mail_wait(c));
  if (h_err != ~0ULL) {
    const long long line = (long long)(h_err >> 16);
    const int t = (int)((h_err >> 8) & 0xff);
    if ((h_err & 0xff) == kQfRepeated) return set_error(CCO_E_INVALID_ARG, "line %lld: the member \"%s\" is repeated", line, kQfNames[t]);
    if (t == kQfWithRanks) return set_error(CCO_E_INVALID_ARG, "line %lld: \"withRanks\" is not true or false", line);
    return set_error(CCO_E_INVALID_ARG, "line %lld: \"%s\" is not a string", line, kQfNames[t]);
  }
  // 4. blacklistItems and itemSet: arrays of strings, their element spans
  JMember *lel, *sel;
  CKR(qf_arrays(c, ar, L, ones, pick_list, mem, bb, "blacklistItems", &qf->loff, &qf->NL, &lel));
  CKR(qf_arrays(c, ar, L, ones, pick_set, mem, bb, "itemSet", &qf->soff, &qf->NE, &sel));
  if (L + qf->NL + qf->NE >= 0x7fffffffLL)
    return set_error(CCO_E_UNSUPPORTED, "%lld lines + %lld blacklist items + %lld elements, at most 2^31 - 2", L, qf->NL, qf->NE);
  // 5. the strings decoded: the users; the items, the blacklistItems entries and the elements in one column
  JMember *rs;
  const long long NR = L + qf->NL + qf->NE;
  CKR(ar.alloc(&rs, std::max<long long>(NR, 1)));
  if (L > 0) CK(cudaMemcpyAsync(rs, ispan, sizeof(JMember) * (size_t)L, cudaMemcpyDeviceToDevice, s));
  if (qf->NL > 0) CK(cudaMemcpyAsync(rs + L, lel, sizeof(JMember) * (size_t)qf->NL, cudaMemcpyDeviceToDevice, s));
  if (qf->NE > 0) CK(cudaMemcpyAsync(rs + L + qf->NL, sel, sizeof(JMember) * (size_t)qf->NE, cudaMemcpyDeviceToDevice, s));
  long long ub = 0;
  CKR(json_decode(c, ar, L, uspan, bb, &qf->uc, &ub));
  CKR(json_decode(c, ar, NR, rs, bb, &qf->rows, &qf->rows_bytes));
  // 6. template keys: the template members' raw spans in order, '\0' between them; template ids by first appearance
  DevStrCol key;
  long long *klen, total = 0;
  CKR(ar.alloc(&klen, L + 1));
  CKR(ar.alloc(&key.off, L + 1));
  CKR(ar.alloc(&key.hash, L1));
  CK(cudaMemsetAsync(klen + L, 0, 8, s));
  if (L > 0) k_qf_key<false><<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, tmem, mem, bb, klen, nullptr, nullptr);
  CKR(exclusive_sum(c, ar, klen, key.off, L + 1));
  CKR(mail_fetch(c, &total, key.off + L, 8));
  CKR(mail_wait(c));
  CKR(ar.alloc(&key.w, (total + 16 + 7) / 8));
  if (L > 0 && total > 0) k_qf_key<true><<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, tmem, mem, bb, nullptr, key.off, (unsigned char *)key.w);
  c->launches += 2;
  key.n = L;
  str_hash(c, key, ~0ULL);
  CKR(ar.alloc(&qf->tid, L1));
  StrTable tb;
  CKR(str_group(c, ar, key, nullptr, false, 0, &tb, qf->tid));
  const long long T = tb.n_groups;
  // 7. per template: the key, its first line, its first line with a user, an item, a set; the rows' validity bitmaps
  long long *first, *dlen, *doff;
  CKR(ar.alloc(&first, std::max<long long>(3 * T, 1)));
  CKR(ar.alloc(&dlen, T + 1));
  CKR(ar.alloc(&doff, T + 1));
  CK(cudaMemsetAsync(first, 0xff, sizeof(long long) * (size_t)std::max<long long>(3 * T, 1), s));
  CK(cudaMemsetAsync(dlen + T, 0, 8, s));
  CKR(ar.alloc(&qf->bits, 3 * ((L + 7) / 8) + 1));
  if (L > 0) {
    k_qf_first<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, qf->tid, has, first);
    k_qf_bits<<<grid_for((L + 7) / 8, 256, c->sm_count), 256, 0, s>>>(L, has, qf->bits);
    k_str_dict_len<<<grid_for(T, 256, c->sm_count), 256, 0, s>>>(T, tb.first_sorted, key.off, dlen);
    c->launches += 3;
  }
  CKR(exclusive_sum(c, ar, dlen, doff, T + 1));
  qf->key_off.assign(T + 1, 0);
  CK(cudaMemcpyAsync(qf->key_off.data(), doff, sizeof(int64_t) * (size_t)(T + 1), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  unsigned char *kb;
  CKR(ar.alloc(&kb, std::max<long long>(qf->key_off[T], 1)));
  if (T > 0 && qf->key_off[T] > 0) {
    k_str_dict_gather<<<grid_for(T, 256, c->sm_count), 256, 0, s>>>(T, tb.first_sorted, key.off, key.base, (const unsigned char *)key.w, doff, kb);
    c->launches++;
  }
  qf->key_bytes.resize((size_t)qf->key_off[T]);
  std::vector<uint32_t> fs(T);
  qf->first_member.assign(3 * T, -1);
  if (qf->key_off[T] > 0) CK(cudaMemcpyAsync(&qf->key_bytes[0], kb, (size_t)qf->key_off[T], cudaMemcpyDeviceToHost, s));
  if (T > 0) {
    CK(cudaMemcpyAsync(fs.data(), tb.first_sorted, sizeof(uint32_t) * (size_t)T, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(qf->first_member.data(), first, sizeof(int64_t) * (size_t)(3 * T), cudaMemcpyDeviceToHost, s));
  }
  CK(cudaStreamSynchronize(s));
  qf->first_line.assign(fs.begin(), fs.end());
  for (void *p : {(void *)qf->uc.off, (void *)qf->uc.w, (void *)qf->uc.hash, (void *)qf->rows.off, (void *)qf->rows.w, (void *)qf->rows.hash,
                  (void *)qf->soff, (void *)qf->loff, (void *)qf->bits, (void *)qf->tid})
    CKR(qf_keep(ar, qf, p));
  return CCO_OK;
}

static int query_file_queries(cco_ctx *c, const cco_query_file *qf, const cco_event_log *lg, const char *body, int64_t body_len,
                              const std::vector<const cco_mixed_query_t *> &tq, char **out_body, int64_t *out_len, int64_t **out_offsets,
                              int64_t *out_n) {
  cudaStream_t s = c->stream;
  CK(cudaSetDevice(c->device));
  Arena ar(s);
  NvtxRange nvtx("cco:query_file_queries");
  mail_reset(c);
  const long long L = qf->L, T = (long long)tq.size();
  if (L == 0) {   // no line: an empty body
    int64_t *ho = (int64_t *)c->pinned_get(sizeof(int64_t), /*for_result=*/false);
    if (!ho) return set_error(CCO_E_OOM, "pinned host allocation failed");
    ho[0] = 0;
    const int st = body_to_host(c, s, nullptr, 0, out_body, out_len);
    if (st != CCO_OK) {
      c->pinned_put(ho);
      return st;
    }
    *out_offsets = ho;
    *out_n = 0;
    return CCO_OK;
  }
  MqRows in;
  in.R = L;
  in.NI = L;
  in.NL = qf->NL;
  in.NE = qf->NE;
  in.sec = {KeySection{L + qf->NL + qf->NE, (const int64_t *)qf->rows.off, (const char *)qf->rows.w, true, qf->rows_bytes}};
  in.uc = qf->uc;
  const long long nb = (L + 7) / 8;
  for (int k = 0; k < 3; ++k) {
    in.col[k] = true;
    in.valid[k] = qf->bits + k * nb;
  }
  in.soff = qf->soff;
  in.loff = qf->loff;
  in.list_shared = false;
  in.rec_tpl = qf->tid;
  in.tpl_user.resize(T);
  for (long long t = 0; t < T; ++t) in.tpl_user[t] = qf->first_member[3 * t] >= 0;
  int *bad;
  CKR(ar.alloc(&bad, 1));
  CK(cudaMemsetAsync(bad, 0, sizeof(int), s));
  return mixed_render(c, ar, lg, body, body_len, tq, in, bad, out_body, out_len, out_offsets, out_n);
}
}  // namespace cco

int cco_query_file_read(cco_ctx_t *ctx, const char *bytes, int64_t len, cco_query_file_t **out) {
  if (!ctx || !out || len < 0 || (len > 0 && !bytes)) return set_error(CCO_E_INVALID_ARG, "null argument or negative length");
  if (!ctx->members.empty()) return set_error(CCO_E_UNSUPPORTED, "per-GPU contexts only");
  *out = nullptr;
  cco_query_file *qf = new cco_query_file();
  qf->ctx = ctx;
  const int st = query_file_read(ctx, bytes, len, qf);
  if (st != CCO_OK) {
    cco_query_file_free(qf);
    return st;
  }
  *out = qf;
  return CCO_OK;
}

int cco_query_file_templates(const cco_query_file_t *qf, int64_t *n_lines, int64_t *n_templates, const int64_t **key_offsets,
                             const char **key_bytes, const int64_t **first_line, const int64_t **first_member_line) {
  if (!qf || !n_lines || !n_templates || !key_offsets || !key_bytes || !first_line || !first_member_line)
    return set_error(CCO_E_INVALID_ARG, "null argument");
  *n_lines = qf->L;
  *n_templates = (int64_t)qf->first_line.size();
  *key_offsets = qf->key_off.data();
  *key_bytes = qf->key_bytes.data();
  *first_line = qf->first_line.data();
  *first_member_line = qf->first_member.data();
  return CCO_OK;
}

int cco_query_file_queries(cco_ctx_t *ctx, const cco_query_file_t *qf, const cco_event_log_t *lg, const char *index_body, int64_t index_len,
                           int64_t n_templates, const cco_mixed_query_t *templates, char **out_body, int64_t *out_len, int64_t **out_offsets,
                           int64_t *out_n) {
  if (!ctx || !qf || !out_body || !out_len || !out_offsets || !out_n || index_len < 0 || (index_len > 0 && !index_body) ||
      (n_templates > 0 && !templates))
    return set_error(CCO_E_INVALID_ARG, "null argument or negative length");
  if (qf->ctx != ctx) return set_error(CCO_E_INVALID_ARG, "the query file was read on another context");
  if (lg && lg->ctx != ctx) return set_error(CCO_E_INVALID_ARG, "the log was read on another context");
  if (lg) CKR(log_state(lg, true));
  if (index_len > 0 && index_body[index_len - 1] != '\n') return set_error(CCO_E_INVALID_ARG, "the body does not end in a newline");
  const long long T = (long long)qf->first_line.size();
  if (n_templates != T) return set_error(CCO_E_INVALID_ARG, "%lld templates given, the file has %lld", (long long)n_templates, T);
  static const int64_t zero[1] = {0};
  std::vector<const cco_mixed_query_t *> tq;
  long long user_line = -1, item_line = -1;
  for (long long t = 0; t < T; ++t) {
    const cco_mixed_query_t *q = &templates[t];
    const long long fu = qf->first_member[3 * t], fi = qf->first_member[3 * t + 1];
    const int st = mq_check_host(q, 0, fu >= 0 ? zero : nullptr, nullptr, fi >= 0 ? zero : nullptr, nullptr, nullptr, 0, nullptr, nullptr);
    if (st != CCO_OK) return set_error(st, "line %lld: %s", (long long)qf->first_line[t], std::string(cco_last_error()).c_str());
    if (q->n_blacklist_items != 0) return set_error(CCO_E_INVALID_ARG, "template %lld: blacklistItems are the lines' own", t);
    if (q->n_model_names != templates[0].n_model_names || q->max_query_events != templates[0].max_query_events)
      return set_error(CCO_E_INVALID_ARG, "template %lld: the model names and max_query_events are the algorithm's, the same in every template", t);
    for (int k = 0; k < q->n_model_names; ++k)
      if (strcmp(q->model_names[k], templates[0].model_names[k]) != 0)
        return set_error(CCO_E_INVALID_ARG, "template %lld: the model names are the algorithm's, the same in every template", t);
    if (fu >= 0 && (user_line < 0 || fu < user_line)) user_line = fu;
    if (fi >= 0 && (item_line < 0 || fi < item_line)) item_line = fi;
    tq.push_back(q);
  }
  if (user_line >= 0 && !lg)
    return set_error(CCO_E_INVALID_ARG, "line %lld: a row has a user: its history needs a log (cco_event_log_begin_ex, CCO_LOG_KEEP_HISTORY)", user_line);
  if (user_line >= 0 && !lg->history)
    return set_error(CCO_E_INVALID_ARG, "line %lld: the log was read without history retention (cco_event_log_begin_ex, CCO_LOG_KEEP_HISTORY)", user_line);
  if (item_line >= 0 && !index_body) return set_error(CCO_E_INVALID_ARG, "line %lld: a row has an item: its similar items need an index body", item_line);
  return query_file_queries(ctx, qf, lg, index_body, index_len, tq, out_body, out_len, out_offsets, out_n);
}

int cco_query_file_free(cco_query_file_t *qf) {
  if (!qf) return CCO_OK;
  cudaSetDevice(qf->ctx->device);
  for (void *p : qf->dev) cudaFreeAsync(p, qf->ctx->stream);
  cudaStreamSynchronize(qf->ctx->stream);
  delete qf;
  return CCO_OK;
}

int cco_event_log_free(cco_event_log_t *lg) {
  if (lg && lg->cleaners > 0) return set_error(CCO_E_INVALID_ARG, "a cleaner of the log is open (cco_event_log_clean_free)");
  event_log_release(lg);
  return CCO_OK;
}

// ---- cco_event_log_clean_*: the log's kept lines copied out of its source bytes (kernels in cco_clean.cuh) ------------------
struct cco_event_clean {
  cco_event_log *lg = nullptr;
  uint32_t flags = 0;
  // the staging, as the log's read stages (cap bytes + 24 of padding, `staged` of them, the last '\n' at last_nl)
  unsigned char *stage = nullptr;
  long long cap = 0, staged = 0, last_nl = -1;
  uint32_t *keep_bits = nullptr;   // one bit per global line of the log: set for the line of every retained record
  uint32_t *fold_bits = nullptr;   // compressProperties: the same, set for the lines folded into fold_out
  std::string fold_out;            // compressProperties: the folded lines, rendered at begin, written at finish
  long long n_read = 0;            // lines read so far
  long long n_rec_done = 0;        // records matched so far (the kept lines read)
  std::vector<int32_t> name_remap; // the log's code of each name, by its chunk-local number (rebuilt per chunk)
  // pinned output of the current call (from the context's pool): out_len bytes of out_cap
  unsigned char *out = nullptr;
  long long out_len = 0, out_cap = 0;
  cco_event_clean_stats_t stats{};
  bool finished = false;
  int fail = CCO_OK;
  std::string fail_msg;
  std::vector<void *> dev;
};

namespace cco {
static void clean_release(cco_event_clean *x) {
  cco_ctx *c = x->lg->ctx;
  cudaSetDevice(c->device);
  for (void *p : x->dev) cudaFreeAsync(p, c->stream);
  cudaStreamSynchronize(c->stream);
  if (x->out) c->pinned_put(x->out);
  x->lg->cleaners--;
  delete x;
}
// room for n more bytes in the pinned output, its first out_len bytes kept
static int clean_out_room(cco_event_clean *x, long long n) {
  if (x->out_len + n <= x->out_cap) return CCO_OK;
  const long long cap = std::max(2 * x->out_cap, x->out_len + n);
  cco_ctx *c = x->lg->ctx;
  unsigned char *p = (unsigned char *)c->pinned_get((size_t)cap, false);   // the context's pool: reused by the next clean
  if (!p) return set_error(CCO_E_OOM, "cudaHostAlloc(%lld bytes) for the cleaned lines failed", cap);
  if (x->out_len > 0) memcpy(p, x->out, (size_t)x->out_len);
  if (x->out) c->pinned_put(x->out);
  x->out = p;
  x->out_cap = cap;
  return CCO_OK;
}
static int clean_mismatch(unsigned long long err) {
  const long long line = (long long)(err >> 8);
  const char *what = (err & 0xff) == kClTime ? "eventTime" : (err & 0xff) == kClName ? "event name"
                     : (err & 0xff) == kClSelection ? "selection (entity and target types, ids, event kind)" : "identity";
  return set_error(CCO_E_INVALID_ARG, "line %lld: its %s differs from the log's record of the line: the source is not what the log read",
                   line, what);
}
// one chunk, the first len staged bytes: parsed and checked as the read parses them, the kept lines checked against their
// records and appended to the pinned output
static int clean_chunk(cco_event_clean *x, long long len, bool open_tail) {
  cco_event_log *lg = x->lg;
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  mail_reset(c);
  Arena ar(s);
  CKR(event_pad(c, x->stage, len));
  EvLines ev;
  const long long base = x->n_read;
  CKR(event_lines(c, ar, (const uint64_t *)x->stage, len, open_tail, base, &ev, lg->dedup));
  const long long L = ev.L;
  if (L == 0) return CCO_OK;
  if (base + L > lg->n_lines)
    return set_error(CCO_E_INVALID_ARG, "line %lld: past the %lld lines the log read", lg->n_lines, lg->n_lines);
  const unsigned char *bb = x->stage;
  int32_t *code;
  std::vector<std::string> cnames;
  CKR(chunk_names(c, ar, ev, bb, &code, &cnames));
  x->name_remap.assign(cnames.size(), 0);
  for (size_t k = 0; k < cnames.size(); ++k) {
    auto it = lg->name_code.find(cnames[k]);
    if (it == lg->name_code.end()) {   // the first line of the name: found on the device
      unsigned long long *first;
      CKR(ar.alloc(&first, 1));
      CK(cudaMemsetAsync(first, 0xff, 8, s));
      k_clean_first_code<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, code, (int32_t)k, first);
      c->launches++;
      unsigned long long h_first = 0;
      CKR(mail_fetch(c, &h_first, first, 8));
      CKR(mail_wait(c));
      return set_error(CCO_E_INVALID_ARG, "line %lld: an event name the log did not read: the source is not what the log read",
                       base + (long long)h_first);
    }
    x->name_remap[k] = it->second;
  }
  CKR(chunk_remap(c, ar, L, x->name_remap, code));
  // the kept lines of the chunk and their records
  uint32_t *keep, *pos, *kidx, K32 = 0;
  CKR(ar.alloc(&keep, L + 1));
  k_clean_keep<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, base, x->keep_bits, keep);
  c->launches++;
  CKR(select_flagged(c, ar, L, keep, &pos, &kidx));
  CKR(mail_fetch(c, &K32, pos + L, 4));
  CKR(mail_wait(c));
  const long long K = K32;
  x->n_read += L;
  if (K == 0) return CCO_OK;
  WinRec *ident = nullptr;
  if (lg->dedup) {
    CKR(ar.alloc(&ident, K));
    CKR(win_idents(c, ar, ev, bb, code, base, K, kidx, ident));
  }
  unsigned long long *err, h_err = 0;
  CKR(ar.alloc(&err, 1));
  CK(cudaMemsetAsync(err, 0xff, 8, s));
  k_clean_check<<<grid_for(K, 256, c->sm_count), 256, 0, s>>>(K, kidx, base, lg->rec + x->n_rec_done, ev.tm, ev.flag, code, ident, err);
  c->launches++;
  CKR(mail_fetch(c, &h_err, err, 8));
  // the compaction: each kept line and its '\n'
  long long *len8, *off, total = 0;
  CKR(ar.alloc(&len8, K + 1));
  CKR(ar.alloc(&off, K + 1));
  CK(cudaMemsetAsync(len8 + K, 0, 8, s));
  k_clean_len<<<grid_for(K, 256, c->sm_count), 256, 0, s>>>(K, kidx, base, ev.sb, ev.se, x->fold_bits, len8);
  c->launches++;
  CKR(exclusive_sum(c, ar, len8, off, K + 1));
  CKR(mail_fetch(c, &total, off + K, 8));
  CKR(mail_wait(c));
  if (h_err != ~0ULL) return clean_mismatch(h_err);
  x->n_rec_done += K;
  if (total == 0) return CCO_OK;
  unsigned char *d_out;
  CKR(ar.alloc(&d_out, (total + 7) / 8 * 8));
  k_clean_compact<<<grid_for(K * 32, 256, c->sm_count), 256, 0, s>>>(K, kidx, ev.sb, ev.se, (const uint64_t *)bb, off, d_out);
  c->launches++;
  CKR(clean_out_room(x, total));
  CK(cudaMemcpyAsync(x->out + x->out_len, d_out, (size_t)total, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  x->out_len += total;
  x->stats.n_bytes += total;
  return CCO_OK;
}
// the staging is full: as event_flush, through clean_chunk
static int clean_flush(cco_event_clean *x) {
  cco_ctx *c = x->lg->ctx;
  cudaStream_t s = c->stream;
  Arena ar(s);
  if (x->last_nl < 0) {
    if (x->staged >= (1LL << 31)) return event_error(((unsigned long long)x->n_read << 8) | kJsonLongLine);
    unsigned char *p;
    CKR(ar.alloc(&p, 2 * x->cap + 24));
    ar.take(p);
    CK(cudaMemcpyAsync(p, x->stage, (size_t)x->staged, cudaMemcpyDeviceToDevice, s));
    for (void *&d : x->dev)
      if (d == x->stage) d = p;
    cudaFreeAsync(x->stage, s);
    x->stage = p;
    x->cap *= 2;
    return CCO_OK;
  }
  const long long P = x->last_nl + 1, carry = x->staged - P;
  unsigned char *tmp = nullptr;
  if (carry > 0) {
    CKR(ar.alloc(&tmp, carry));
    CK(cudaMemcpyAsync(tmp, x->stage + P, (size_t)carry, cudaMemcpyDeviceToDevice, s));
  }
  CKR(clean_chunk(x, P, false));
  if (carry > 0) CK(cudaMemcpyAsync(x->stage, tmp, (size_t)carry, cudaMemcpyDeviceToDevice, s));
  x->staged = carry;
  x->last_nl = -1;
  return CCO_OK;
}
// compressProperties over the log's retained item property lines (lg->pb, their global lines lg->prop_line): the $set /
// $unset lines of each foldable entity marked in fold_bits and rendered as one line each into fold_out (kernels k_fold_*)
static int clean_fold(cco_event_clean *x) {
  cco_event_log *lg = x->lg;
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  mail_reset(c);
  Arena ar(s);
  CKR(event_pad(c, lg->pb, lg->pb_len));
  EvLines ev;
  CKR(event_lines(c, ar, (const uint64_t *)lg->pb, lg->pb_len, false, 0, &ev));   // judged when the log read them
  const long long L = ev.L;
  if (L == 0) return CCO_OK;
  if (L != (long long)lg->prop_line.size()) return set_error(CCO_E_INVALID_ARG, "internal: %lld property lines, %zu line numbers", L, lg->prop_line.size());
  const unsigned char *pb = lg->pb;
  // 1. the entities: decoded entityIds grouped exactly (hash, then the strings compared), numbered by first line
  JMember *jm;
  CKR(ar.alloc(&jm, L));
  k_event_strings<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, nullptr, kEvEntityId, ev.sb, ev.span, pb, jm);
  c->launches++;
  DevStrCol ids;
  long long id_bytes = 0;
  CKR(json_decode(c, ar, L, jm, pb, &ids, &id_bytes));
  str_hash(c, ids, ~0ULL);
  int32_t *gcode;
  CKR(ar.alloc(&gcode, L));
  StrTable gt;
  CKR(str_group(c, ar, ids, nullptr, false, 0, &gt, gcode));
  const long long G = gt.n_groups;
  // 2. foldable groups (no pin, two or more $set / $unset lines), ranked in order of their first line; their lines
  uint32_t *cnt, *pin, *gkeep, *gpos, *gidx, R32 = 0;
  CKR(ar.alloc(&cnt, G));
  CKR(ar.alloc(&pin, G));
  CKR(ar.alloc(&gkeep, G + 1));
  CK(cudaMemsetAsync(cnt, 0, sizeof(uint32_t) * (size_t)G, s));
  CK(cudaMemsetAsync(pin, 0, sizeof(uint32_t) * (size_t)G, s));
  k_fold_count<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, ev.flag, gcode, cnt, pin);
  k_fold_groups<<<grid_for(G, 256, c->sm_count), 256, 0, s>>>(G, cnt, pin, gkeep);
  c->launches += 2;
  CKR(select_flagged(c, ar, G, gkeep, &gpos, &gidx));
  long long *gline;
  uint8_t *fl;
  CKR(ar.alloc(&gline, L));
  CKR(ar.alloc(&fl, L + 1));
  CK(cudaMemcpyAsync(gline, lg->prop_line.data(), sizeof(long long) * (size_t)L, cudaMemcpyHostToDevice, s));
  k_fold_lines<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, ev.flag, gcode, gkeep, gline, fl, x->fold_bits);
  c->launches++;
  CKR(mail_fetch(c, &R32, gpos + G, 4));
  CKR(mail_wait(c));
  const long long R = R32;
  if (R == 0) return CCO_OK;
  uint32_t *lkeep, *lpos, *idx, F32 = 0;
  CKR(ar.alloc(&lkeep, L + 1));
  k_win_flag_keep<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, fl, kFoldLine, lkeep);
  c->launches++;
  CKR(select_flagged(c, ar, L, lkeep, &lpos, &idx));
  CKR(mail_fetch(c, &F32, lpos + L, 4));
  CKR(mail_wait(c));
  const long long F = F32;
  // 3. the fold order: (group rank, eventTime, line) -- sorted by time, then stably by rank (idx is in line order)
  unsigned long long *k1;
  uint32_t *k2, *v, *gr;
  CKR(ar.alloc(&k1, F));
  CKR(ar.alloc(&k2, F));
  CKR(ar.alloc(&v, F));
  CKR(ar.alloc(&gr, F));
  k_fold_keys<<<grid_for(F, 256, c->sm_count), 256, 0, s>>>(F, idx, ev.tm, gcode, gpos, k1, k2, v);
  c->launches++;
  CKR(sort_pairs(c, ar, F, &k1, &v, 64));
  k_fold_key2<<<grid_for(F, 256, c->sm_count), 256, 0, s>>>(F, v, k2, gr);
  c->launches++;
  CKR(sort_pairs(c, ar, F, &gr, &v, bits_for(R)));
  uint32_t *place, *first_set, *last;
  const uint32_t *rank_of_line = k2;   // each folded line's group rank, in folded-line order
  CKR(ar.alloc(&place, F));
  CKR(ar.alloc(&first_set, R));
  CKR(ar.alloc(&last, R));
  CK(cudaMemsetAsync(first_set, 0xff, sizeof(uint32_t) * (size_t)R, s));
  k_fold_first<<<grid_for(F, 256, c->sm_count), 256, 0, s>>>(F, v, gr, idx, fl, place, first_set, last);
  c->launches++;
  // 4. the members of the folded lines' properties (count pass with each object's verdict, then the members)
  long long *ob, *oe, *mcnt, *moff;
  int *codes;
  unsigned long long *err;
  CKR(ar.alloc(&ob, F));
  CKR(ar.alloc(&oe, F));
  CKR(ar.alloc(&mcnt, F + 1));
  CKR(ar.alloc(&moff, F + 1));
  CKR(ar.alloc(&codes, F));
  CKR(ar.alloc(&err, 1));
  CK(cudaMemsetAsync(mcnt + F, 0, 8, s));
  k_win_prop_spans<<<grid_for(F, 256, c->sm_count), 256, 0, s>>>(F, idx, ev.sb, ev.span, ob, oe);
  k_json_members<<<grid_for(F * 32, 256, c->sm_count), 256, 0, s>>>(F, ob, oe, pb, WinMemberSink<false>{mcnt, codes, nullptr, nullptr}, err);
  c->launches += 2;
  CKR(exclusive_sum(c, ar, mcnt, moff, F + 1));
  long long M = 0;
  CKR(mail_fetch(c, &M, moff + F, 8));
  CKR(mail_wait(c));
  JMember *mem;
  CKR(ar.alloc(&mem, std::max<long long>(M, 1)));
  uint32_t *members = nullptr, P32 = 0;
  long long *gmoff;
  CKR(ar.alloc(&gmoff, R + 1));
  CK(cudaMemsetAsync(gmoff, 0, sizeof(long long) * (size_t)(R + 1), s));
  DevStrCol names;
  if (M > 0) {
    k_json_members<<<grid_for(F * 32, 256, c->sm_count), 256, 0, s>>>(F, ob, oe, pb, WinMemberSink<true>{nullptr, codes, moff, mem}, err);
    c->launches++;
    // 5. the names, decoded and grouped exactly; members sorted by (rank, name, place, index)
    JMember *nm;
    CKR(ar.alloc(&nm, M));
    k_win_strings<<<grid_for(M, 256, c->sm_count), 256, 0, s>>>(0, nullptr, nullptr, nullptr, nullptr, pb, M, mem, nm);
    c->launches++;
    long long name_bytes = 0;
    CKR(json_decode(c, ar, M, nm, pb, &names, &name_bytes));
    str_hash(c, names, ~0ULL);
    int32_t *ncode;
    CKR(ar.alloc(&ncode, M));
    StrTable nt;
    CKR(str_group(c, ar, names, nullptr, false, 0, &nt, ncode));
    uint32_t *mline, *mv, *keep, *kpos, *kidx;
    unsigned long long *mk1, *mk2, *mk2s, *ins;
    CKR(ar.alloc(&mline, M));
    CKR(ar.alloc(&mv, M));
    CKR(ar.alloc(&mk1, M));
    CKR(ar.alloc(&mk2, M));
    CKR(ar.alloc(&mk2s, M));
    k_win_member_line<<<grid_for(F, 256, c->sm_count), 256, 0, s>>>(F, moff, mline);
    k_fold_mkeys<<<grid_for(M, 256, c->sm_count), 256, 0, s>>>(M, mline, moff, place, rank_of_line, ncode, mk1, mk2, mv);
    c->launches += 2;
    CKR(sort_pairs(c, ar, M, &mk1, &mv, 64));
    k_fold_mkey2<<<grid_for(M, 256, c->sm_count), 256, 0, s>>>(M, mv, mk2, mk2s);
    c->launches++;
    CKR(sort_pairs(c, ar, M, &mk2s, &mv, 64));
    // 6. per (group, name) run: in the line or not, where inserted, which value; then the members in insertion order
    CKR(ar.alloc(&keep, M + 1));
    CKR(ar.alloc(&ins, M));
    uint32_t *vm;
    CKR(ar.alloc(&vm, M));
    k_fold_runs<<<grid_for(M, 256, c->sm_count), 256, 0, s>>>(M, mk2s, mv, mline, moff, place, idx, fl, first_set, keep, ins, vm);
    c->launches++;
    CKR(select_flagged(c, ar, M, keep, &kpos, &kidx));
    CKR(mail_fetch(c, &P32, kpos + M, 4));
    CKR(mail_wait(c));
    const long long P = P32;
    if (P > 0) {
      // sorted by insertion, then stably by rank: each folded line's members in insertion order
      unsigned long long *ok1;
      uint32_t *or32, *om, *perm, *r2, *ocnt;
      CKR(ar.alloc(&ok1, P));
      CKR(ar.alloc(&or32, P));
      CKR(ar.alloc(&om, P));
      CKR(ar.alloc(&perm, P));
      CKR(ar.alloc(&r2, P));
      CKR(ar.alloc(&members, P));
      CKR(ar.alloc(&ocnt, R + 1));
      CK(cudaMemsetAsync(ocnt, 0, sizeof(uint32_t) * (size_t)(R + 1), s));
      k_fold_okeys<<<grid_for(P, 256, c->sm_count), 256, 0, s>>>(P, kidx, mk2s, ins, vm, ok1, or32, om, perm, ocnt);
      c->launches++;
      CKR(sort_pairs(c, ar, P, &ok1, &perm, 64));
      k_fold_gather2<<<grid_for(P, 256, c->sm_count), 256, 0, s>>>(P, perm, or32, om, r2, members);
      c->launches++;
      CKR(sort_pairs(c, ar, P, &r2, &members, bits_for(R)));
      long long *c64;
      CKR(ar.alloc(&c64, R + 1));
      k_fold_count64<<<grid_for(R + 1, 256, c->sm_count), 256, 0, s>>>(R, ocnt, c64);
      c->launches++;
      CKR(exclusive_sum(c, ar, c64, gmoff, R + 1));
    }
  }
  // 7. the entity id of each folded group (its first line's) and the two render passes
  DevDict gid;
  {
    uint32_t *first_line;
    long long *len, *goff;
    CKR(ar.alloc(&first_line, R));
    CKR(ar.alloc(&len, R + 1));
    CKR(ar.alloc(&goff, R + 1));
    k_fold_group_line<<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, gidx, gt.first_sorted, first_line, ids.off, len);
    c->launches++;
    CK(cudaMemsetAsync(len + R, 0, 8, s));
    CKR(exclusive_sum(c, ar, len, goff, R + 1));
    long long total = 0;
    CKR(mail_fetch(c, &total, goff + R, 8));
    CKR(mail_wait(c));
    unsigned char *gb;
    CKR(ar.alloc(&gb, std::max<long long>(total, 1)));
    k_str_dict_gather<<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, first_line, ids.off, 0, (const unsigned char *)ids.w, goff, gb);
    c->launches++;
    gid = DevDict{goff, gb, R};
  }
  long long *rlen, *roff, total = 0;
  CKR(ar.alloc(&rlen, R + 1));
  CKR(ar.alloc(&roff, R + 1));
  CK(cudaMemsetAsync(rlen + R, 0, 8, s));
  const long long *noff = M > 0 ? names.off : nullptr;
  const unsigned char *nb = M > 0 ? (const unsigned char *)names.w : nullptr;
  k_fold_render<false><<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, last, first_set, idx, ev.sb, ev.span, pb, gid.off, gid.bytes, gmoff, members,
                                                                     noff, nb, mem, nullptr, rlen, nullptr);
  c->launches++;
  CKR(exclusive_sum(c, ar, rlen, roff, R + 1));
  CKR(mail_fetch(c, &total, roff + R, 8));
  CKR(mail_wait(c));
  unsigned char *d_out;
  CKR(ar.alloc(&d_out, std::max<long long>(total, 1)));
  k_fold_render<true><<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, last, first_set, idx, ev.sb, ev.span, pb, gid.off, gid.bytes, gmoff, members,
                                                                    noff, nb, mem, roff, nullptr, d_out);
  c->launches++;
  x->fold_out.resize((size_t)total);
  CK(cudaMemcpyAsync(&x->fold_out[0], d_out, (size_t)total, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  x->stats.n_folded = F;
  x->stats.n_compressed = R;
  return CCO_OK;
}
static int clean_begin(cco_event_log *lg, uint32_t flags, cco_event_clean **out) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  CK(cudaSetDevice(c->device));
  NvtxRange nvtx("cco:event_clean");
  std::unique_ptr<cco_event_clean> x(new cco_event_clean());
  x->lg = lg;
  x->flags = flags;
  x->cap = lg->chunk0;
  Arena ar(s);
  const long long NB = (lg->n_lines + 31) / 32;
  CKR(ar.alloc(&x->stage, x->cap + 24));
  CKR(ar.alloc(&x->keep_bits, std::max<long long>(NB, 1)));
  for (void *p : {(void *)x->stage, (void *)x->keep_bits}) {
    ar.take(p);
    x->dev.push_back(p);
  }
  CK(cudaMemsetAsync(x->keep_bits, 0, sizeof(uint32_t) * (size_t)std::max<long long>(NB, 1), s));
  if (lg->n_rec > 0) {
    k_clean_bitmap<<<grid_for(lg->n_rec, 256, c->sm_count), 256, 0, s>>>(lg->n_rec, lg->rec, x->keep_bits);
    c->launches++;
  }
  CK(cudaStreamSynchronize(s));
  if ((flags & CCO_CLEAN_COMPRESS_PROPERTIES) && lg->n_prop > 0) {
    CKR(ar.alloc(&x->fold_bits, std::max<long long>(NB, 1)));
    ar.take(x->fold_bits);
    x->dev.push_back(x->fold_bits);
    CK(cudaMemsetAsync(x->fold_bits, 0, sizeof(uint32_t) * (size_t)std::max<long long>(NB, 1), s));
    CKR(clean_fold(x.get()));
  }
  x->stats.n_expired = lg->n_expired;
  x->stats.n_duplicates = lg->n_dup;
  lg->cleaners++;
  *out = x.release();
  return CCO_OK;
}
static int clean_append(cco_event_clean *x, const char *bytes, int64_t len) {
  cco_ctx *c = x->lg->ctx;
  CK(cudaSetDevice(c->device));
  NvtxRange nvtx("cco:event_clean");
  x->out_len = 0;
  while (len > 0) {
    if (x->staged == x->cap) CKR(clean_flush(x));
    const long long take = std::min<long long>(len, x->cap - x->staged);
    CK(cudaMemcpyAsync(x->stage + x->staged, bytes, (size_t)take, cudaMemcpyHostToDevice, c->stream));
    const void *nl = memrchr(bytes, '\n', (size_t)take);
    if (nl) x->last_nl = x->staged + ((const char *)nl - bytes);
    x->staged += take;
    bytes += take;
    len -= take;
  }
  CK(cudaStreamSynchronize(c->stream));   // the bytes are copied: the caller may reuse its buffer
  return CCO_OK;
}
static int clean_finish(cco_event_clean *x) {
  cco_event_log *lg = x->lg;
  CK(cudaSetDevice(lg->ctx->device));
  NvtxRange nvtx("cco:event_clean");
  x->out_len = 0;
  if (x->staged > 0) CKR(clean_chunk(x, x->staged, x->last_nl != x->staged - 1));
  x->staged = 0;
  if (x->n_read != lg->n_lines)
    return set_error(CCO_E_INVALID_ARG, "line %lld: the source ends after %lld lines, the log read %lld", x->n_read, x->n_read, lg->n_lines);
  const long long F = (long long)x->fold_out.size();
  if (F > 0) {
    CKR(clean_out_room(x, F));
    memcpy(x->out + x->out_len, x->fold_out.data(), (size_t)F);
    x->out_len += F;
    x->stats.n_bytes += F;
  }
  x->stats.n_lines = x->n_read;
  x->stats.n_written = lg->n_rec - x->stats.n_folded + x->stats.n_compressed;
  x->finished = true;
  return CCO_OK;
}
static int clean_state(const cco_event_clean *x) {
  if (x->fail != CCO_OK) return set_error(CCO_E_INVALID_ARG, "the cleaner failed: %s", x->fail_msg.c_str());
  if (x->finished) return set_error(CCO_E_INVALID_ARG, "the cleaner is finished");
  return CCO_OK;
}
static int clean_fail(cco_event_clean *x, int rc) {
  if (rc != CCO_OK) {
    x->fail = rc;
    x->fail_msg = g_err;
  }
  return rc;
}
}  // namespace cco

int cco_event_log_clean_begin(cco_event_log_t *lg, uint32_t flags, cco_event_clean_t **out) {
  if (!lg || !out) return set_error(CCO_E_INVALID_ARG, "null argument");
  *out = nullptr;
  if (flags & ~(uint32_t)CCO_CLEAN_COMPRESS_PROPERTIES) return set_error(CCO_E_INVALID_ARG, "unknown flags 0x%x", (unsigned)flags);
  if (!lg->ctx->members.empty()) return set_error(CCO_E_UNSUPPORTED, "an event log is resident on one GPU");
  CKR(log_state(lg, true));
  if (!lg->extendable) return set_error(CCO_E_INVALID_ARG, "the log was read without CCO_LOG_EXTENDABLE (cco_event_log_begin_ex)");
  return clean_begin(lg, flags, out);
}

int cco_event_log_clean_append(cco_event_clean_t *x, const char *bytes, int64_t len, const char **out, int64_t *out_len) {
  if (!x || len < 0 || (len > 0 && !bytes) || !out || !out_len) return set_error(CCO_E_INVALID_ARG, "null argument or negative length");
  *out = nullptr;
  *out_len = 0;
  CKR(clean_state(x));
  CKR(clean_fail(x, clean_append(x, bytes, len)));
  *out = (const char *)x->out;
  *out_len = x->out_len;
  return CCO_OK;
}

int cco_event_log_clean_finish(cco_event_clean_t *x, const char **out, int64_t *out_len, cco_event_clean_stats_t *stats) {
  if (!x || !out || !out_len || !stats) return set_error(CCO_E_INVALID_ARG, "null argument");
  *out = nullptr;
  *out_len = 0;
  CKR(clean_state(x));
  CKR(clean_fail(x, clean_finish(x)));
  *out = (const char *)x->out;
  *out_len = x->out_len;
  *stats = x->stats;
  return CCO_OK;
}

int cco_event_log_clean_free(cco_event_clean_t *x) {
  if (x) clean_release(x);
  return CCO_OK;
}

// ---- event log snapshots (cco_event_log_save / cco_event_log_load_*; layout in include/cco_b200.h) --------------------
namespace cco {
constexpr char kSnapMagic[8] = {'C', 'C', 'O', 'L', 'O', 'G', 'S', 'N'};
constexpr uint32_t kSnapVersion = CCO_SNAPSHOT_VERSION;
constexpr long long kSnapHead = 64, kSnapEntry = 40, kSnapAlign = 256, kSnapStateWords = 16;
constexpr long long kSnapStage = 32LL << 20;   // pinned staging of a save, per buffer (two)
enum SnapKind : uint32_t {
  kSnState = 1, kSnNames, kSnCounts, kSnFields, kSnPropLines,   // host sections
  kSnTuOff, kSnTuBytes, kSnTiOff, kSnTiBytes, kSnRiOff, kSnRiBytes, kSnRtime, kSnTline, kSnRline, kSnTtime, kSnTkey, kSnRecords,
  kSnDupTime, kSnPropBytes, kSnPField, kSnPVoff, kSnPVals, kSnPIoff, kSnPIbytes, kSnPItemOff, kSnPItemBytes, kSnUserOff,
  kSnUserBytes, kSnItemOff, kSnItemBytes,
  kSnEnd
};
static const char *const kSnName[kSnEnd] = {"", "state", "names", "counts", "fields", "property_lines", "train_users.offsets",
  "train_users.bytes", "train_items.offsets", "train_items.bytes", "rank_items.offsets", "rank_items.bytes", "rank_times",
  "train_lines", "rank_lines", "train_times", "train_keys", "records", "duplicate_times", "property_bytes", "properties.fields",
  "properties.value_offsets", "properties.values", "properties.item_offsets", "properties.item_bytes",
  "property_items.offsets", "property_items.bytes", "user_keys.offsets", "user_keys.bytes", "item_keys.offsets",
  "item_keys.bytes"};
static bool snap_host_kind(uint32_t k) { return k >= kSnState && k <= kSnPropLines; }
// string bytes carry 16 bytes of padding past a whole word, the property lines 24 (event_pad)
static bool snap_str_bytes(uint32_t k) {
  return k == kSnTuBytes || k == kSnTiBytes || k == kSnRiBytes || k == kSnPItemBytes || k == kSnUserBytes || k == kSnItemBytes;
}
// the least device bytes a section of len bytes takes (what the log allocates for it)
static long long snap_need(uint32_t k, long long len) {
  if (snap_str_bytes(k)) return std::max<long long>((len + 23) / 8 * 8, 16);
  if (k == kSnPropBytes) return len + 24;
  return std::max<long long>(len, k == kSnRecords ? (long long)sizeof(WinRec) : 16);
}

struct SnapSec {
  uint32_t kind = 0;
  long long off = 0, len = 0, alloc = 0;   // alloc: device bytes (0: a host section)
  uint64_t sum = 0;
  unsigned char *dev = nullptr;
  std::string host;
};
struct SnapImage {
  std::string head;   // header + table, zero-padded to the first section
  std::vector<SnapSec> secs;
  long long total = 0;
};
struct SnapLoad {
  std::string head;
  long long pos = 0, total = -1, n_sec = 0;
  bool table = false;
  std::vector<SnapSec> secs;
  long long pb_newlines = 0;
  unsigned char pb_last = 0;
};
}  // namespace cco
extern "C++" {
namespace cco {
void snap_delete(SnapImage *p) { delete p; }
void snap_delete(SnapLoad *p) { delete p; }
template <typename T>
static void snap_put(std::string *s, T v) {
  s->append((const char *)&v, sizeof v);
}
template <typename T>
static T snap_get(const std::string &s, long long at) {
  T v;
  memcpy(&v, s.data() + at, sizeof v);
  return v;
}
}  // namespace cco
}  // extern "C++"
namespace cco {

static uint64_t snap_sum_host(const unsigned char *p, long long len) {
  uint64_t h = snap_mix((uint64_t)len);
  for (long long i = 0; i * 8 < len; ++i) {
    uint64_t w = 0;
    memcpy(&w, p + 8 * i, (size_t)std::min<long long>(8, len - 8 * i));
    h += snap_mix(w ^ (uint64_t)i * kSnapGolden);
  }
  return h;
}
// a list of strings: n, offsets [n + 1] from 0, bytes
static std::string snap_strings(const std::vector<std::string> &v) {
  std::string s;
  snap_put<int64_t>(&s, (int64_t)v.size());
  int64_t o = 0;
  snap_put<int64_t>(&s, 0);
  for (const std::string &x : v) snap_put<int64_t>(&s, o += (int64_t)x.size());
  for (const std::string &x : v) s += x;
  return s;
}
static int snap_unstrings(const SnapSec &sc, std::vector<std::string> *out) {
  const std::string &s = sc.host;
  const long long L = (long long)s.size();
  const int64_t n = L >= 8 ? snap_get<int64_t>(s, 0) : -1;
  if (n < 0 || n > (L - 16) / 8) return set_error(CCO_E_INVALID_ARG, "snapshot section %s: a bad string count", kSnName[sc.kind]);
  const long long b0 = 16 + 8 * n;
  int64_t prev = 0;
  out->clear();
  for (int64_t i = 0; i < n; ++i) {
    const int64_t o = snap_get<int64_t>(s, 8 * (i + 2));
    if (o < prev || b0 + o > L) return set_error(CCO_E_INVALID_ARG, "snapshot section %s: string %lld has a bad offset", kSnName[sc.kind], (long long)i);
    out->emplace_back(s.data() + b0 + prev, (size_t)(o - prev));
    prev = o;
  }
  if (snap_get<int64_t>(s, 8) != 0 || b0 + prev != L)
    return set_error(CCO_E_INVALID_ARG, "snapshot section %s: the offsets disagree with its length", kSnName[sc.kind]);
  return CCO_OK;
}
// the log field a device section fills
static void **snap_slot(cco_event_log *lg, uint32_t k) {
  switch (k) {
    case kSnTuOff: return (void **)&lg->tu.off;
    case kSnTuBytes: return (void **)&lg->tu.w;
    case kSnTiOff: return (void **)&lg->ti.off;
    case kSnTiBytes: return (void **)&lg->ti.w;
    case kSnRiOff: return (void **)&lg->ri.off;
    case kSnRiBytes: return (void **)&lg->ri.w;
    case kSnRtime: return (void **)&lg->rtime;
    case kSnTline: return (void **)&lg->tline;
    case kSnRline: return (void **)&lg->rline;
    case kSnTtime: return (void **)&lg->ttime;
    case kSnTkey: return (void **)&lg->tkey;
    case kSnRecords: return (void **)&lg->rec;
    case kSnDupTime: return (void **)&lg->dup_time;
    case kSnPropBytes: return (void **)&lg->pb;
    case kSnPField: return (void **)&lg->p_field;
    case kSnPVoff: return (void **)&lg->p_voff;
    case kSnPVals: return (void **)&lg->p_vals;
    case kSnPIoff: return (void **)&lg->p_ioff;
    case kSnPIbytes: return (void **)&lg->p_ibytes;
    case kSnPItemOff: return (void **)&lg->pitem.off;
    case kSnPItemBytes: return (void **)&lg->pitem.w;
    case kSnUserOff: return (void **)&lg->users.off;
    case kSnUserBytes: return (void **)&lg->users.w;
    case kSnItemOff: return (void **)&lg->items.off;
    case kSnItemBytes: return (void **)&lg->items.w;
    default: return nullptr;
  }
}
// the offsets section paired with a bytes section
static uint32_t snap_off_of(uint32_t k) {
  switch (k) {
    case kSnTuBytes: case kSnTiBytes: case kSnRiBytes: case kSnPVals: case kSnPIbytes: case kSnPItemBytes: case kSnUserBytes:
    case kSnItemBytes: return k - 1;
    default: return 0;
  }
}

// the checksums of the device sections, one k_snap_sum pass over all of them
static int snap_device_sums(cco_ctx *c, std::vector<SnapSec *> &secs) {
  cudaStream_t s = c->stream;
  std::vector<SnapSpan> sp;
  long long at = 0;
  for (SnapSec *x : secs) {
    sp.push_back(SnapSpan{x->dev, x->len, at});
    at += ((x->len + 7) / 8 + 31) / 32 * 32;
  }
  if (sp.empty()) return CCO_OK;
  Arena ar(s);
  SnapSpan *d_sp;
  unsigned long long *d_sum;
  CKR(ar.alloc(&d_sp, sp.size()));
  CKR(ar.alloc(&d_sum, sp.size()));
  std::vector<unsigned long long> h((size_t)sp.size(), 0);
  CK(cudaMemcpyAsync(d_sp, sp.data(), sizeof(SnapSpan) * sp.size(), cudaMemcpyHostToDevice, s));
  CK(cudaMemsetAsync(d_sum, 0, sizeof(unsigned long long) * sp.size(), s));
  if (at > 0) {
    k_snap_sum<<<grid_for(at, 256, c->sm_count), 256, 0, s>>>((int)sp.size(), d_sp, at, d_sum);
    c->launches++;
  }
  CK(cudaMemcpyAsync(h.data(), d_sum, sizeof(unsigned long long) * h.size(), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  for (size_t i = 0; i < secs.size(); ++i) secs[i]->sum = h[i] + snap_mix((uint64_t)secs[i]->len);
  return CCO_OK;
}

// the image of a finished log: host sections serialised, device sections measured and hashed, the layout and header
static int snap_image(cco_event_log *lg) {
  if (lg->snap) return CCO_OK;
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  CK(cudaStreamSynchronize(s));
  std::unique_ptr<SnapImage, SnapFree> im(new SnapImage());
  auto host = [&](uint32_t k, std::string v) {
    SnapSec x;
    x.kind = k;
    x.len = (long long)v.size();
    x.host = std::move(v);
    x.sum = snap_sum_host((const unsigned char *)x.host.data(), x.len);
    im->secs.push_back(std::move(x));
  };
  std::string st;
  const int64_t flags = (lg->history ? CCO_LOG_KEEP_HISTORY : 0) | (lg->extendable ? CCO_LOG_EXTENDABLE : 0) | (lg->intern ? CCO_LOG_INTERN_IDS : 0);
  const int64_t w[kSnapStateWords] = {flags, lg->dedup, lg->cutoff, lg->chunk0, lg->n_lines, lg->n_prop, lg->n_ignored, lg->n_prop_items,
                                      lg->n_prop_fields, lg->n_expired, lg->n_dup, (int64_t)lg->intern_mask, lg->n_erased, 0, 0, 0};
  st.assign((const char *)w, sizeof w);
  host(kSnState, st);
  const long long NG = (long long)lg->name_off.size() - 1;
  std::vector<std::string> names;
  for (long long g = 0; g < NG; ++g) names.emplace_back(lg->name_bytes.data() + lg->name_off[g], (size_t)(lg->name_off[g + 1] - lg->name_off[g]));
  host(kSnNames, snap_strings(names));
  std::string cnt;
  for (int64_t v : lg->n_train) snap_put<int64_t>(&cnt, v);
  for (int64_t v : lg->n_rank) snap_put<int64_t>(&cnt, v);
  host(kSnCounts, cnt);
  host(kSnFields, snap_strings(lg->field_names));
  if (lg->pb) host(kSnPropLines, std::string((const char *)lg->prop_line.data(), sizeof(long long) * lg->prop_line.size()));
  // device sections: entries from the counters, string bytes from the last offset
  const long long NT = lg->train_at.back(), NR = lg->rank_at.back(), T = lg->n_triples;
  auto last_off = [&](const long long *off, long long n, long long *v) -> int {
    CK(cudaMemcpy(v, off + n, 8, cudaMemcpyDeviceToHost));
    return CCO_OK;
  };
  std::vector<SnapSec *> dev;
  for (uint32_t k = kSnTuOff; k < kSnEnd; ++k) {
    void *p = *snap_slot(lg, k);
    if (!p) continue;
    long long n = 0;
    switch (k) {
      case kSnTuOff: case kSnTiOff: n = 8 * (NT + 1); break;
      case kSnRiOff: n = 8 * (NR + 1); break;
      case kSnRtime: case kSnRline: n = 8 * NR; break;
      case kSnTline: case kSnTtime: case kSnTkey: n = 8 * NT; break;
      case kSnRecords: n = (long long)sizeof(WinRec) * lg->n_rec; break;
      case kSnDupTime: n = 8 * lg->n_dup_time; break;
      case kSnPropBytes: n = lg->pb_len; break;
      case kSnPField: n = 4 * T; break;
      case kSnPVoff: case kSnPIoff: n = 8 * (T + 1); break;
      case kSnPItemOff: n = 8 * (lg->n_prop + 1); break;
      case kSnUserOff: n = 8 * (lg->users.n + 1); break;
      case kSnItemOff: n = 8 * (lg->items.n + 1); break;
      default: CKR(last_off((const long long *)*snap_slot(lg, snap_off_of(k)), im->secs.back().len / 8 - 1, &n));
    }
    SnapSec x;
    x.kind = k;
    x.len = n;
    x.dev = (unsigned char *)p;
    for (size_t i = 0; i < lg->dev.size(); ++i)
      if (lg->dev[i] == p) x.alloc = (long long)lg->dev_bytes[i];
    if (x.alloc < snap_need(k, n)) return set_error(CCO_E_CUDA, "internal: section %s holds %lld bytes of %lld", kSnName[k], x.alloc, n);
    im->secs.push_back(std::move(x));
  }
  for (SnapSec &x : im->secs)
    if (x.dev) dev.push_back(&x);
  CKR(snap_device_sums(c, dev));
  const long long NS = (long long)im->secs.size();
  long long at = (kSnapHead + kSnapEntry * NS + kSnapAlign - 1) / kSnapAlign * kSnapAlign;
  for (SnapSec &x : im->secs) {
    x.off = at;
    at = (at + x.len + kSnapAlign - 1) / kSnapAlign * kSnapAlign;
  }
  im->total = im->secs.back().off + im->secs.back().len;
  std::string &h = im->head;
  h.append(kSnapMagic, 8);
  snap_put<uint32_t>(&h, kSnapVersion);
  snap_put<uint32_t>(&h, CCO_ABI_VERSION);
  snap_put<uint32_t>(&h, (uint32_t)NS);
  snap_put<uint32_t>(&h, 0);
  snap_put<int64_t>(&h, im->total);
  h.resize(kSnapHead, '\0');
  for (const SnapSec &x : im->secs) {
    snap_put<uint32_t>(&h, x.kind);
    snap_put<uint32_t>(&h, 0);
    snap_put<int64_t>(&h, x.off);
    snap_put<int64_t>(&h, x.len);
    snap_put<int64_t>(&h, x.alloc);
    snap_put<uint64_t>(&h, x.sum);
  }
  const uint64_t hs = snap_sum_host((const unsigned char *)h.data(), (long long)h.size());
  memcpy(&h[32], &hs, 8);
  h.resize((size_t)im->secs[0].off, '\0');
  lg->snap = std::move(im);
  return CCO_OK;
}

// bytes [offset, offset + len) of the image -> dst; device sections through two pinned buffers on the copy stream
static int snap_save(cco_event_log *lg, long long offset, unsigned char *dst, long long len) {
  cco_ctx *c = lg->ctx;
  const SnapImage &im = *lg->snap;
  const long long end = offset + len;
  long long cur = offset;   // dst holds the image's bytes [offset, cur)
  auto gap = [&](long long a) {   // zeros up to a (the padding before a section)
    a = std::min(a, end);
    if (a > cur) memset(dst + (cur - offset), 0, (size_t)(a - cur));
    cur = std::max(cur, a);
  };
  if (offset < (long long)im.head.size()) {
    cur = std::min(end, (long long)im.head.size());
    memcpy(dst, im.head.data() + offset, (size_t)(cur - offset));
  }
  for (const SnapSec &x : im.secs) {
    const long long a = std::max(x.off, cur), b = std::min(x.off + x.len, end);
    if (a >= b) continue;
    gap(a);
    if (!x.dev) {
      memcpy(dst + (a - offset), x.host.data() + (a - x.off), (size_t)(b - a));
      cur = b;
      continue;
    }
    const long long piece = std::min(kSnapStage, b - a);
    unsigned char *buf[2] = {(unsigned char *)c->pinned_get((size_t)piece, false), nullptr};
    if (b - a > piece) buf[1] = (unsigned char *)c->pinned_get((size_t)piece, false);
    struct Put {
      cco_ctx *c;
      unsigned char **b;
      ~Put() {
        for (int i = 0; i < 2; ++i)
          if (b[i]) c->pinned_put(b[i]);
      }
    } put{c, buf};
    if (!buf[0] || (b - a > piece && !buf[1])) return set_error(CCO_E_OOM, "pinned host allocation failed");
    long long prev = -1, prev_n = 0;
    int j = 0;
    for (long long q = a; q < b; q += piece, ++j) {
      const long long n = std::min(piece, b - q);
      CK(cudaMemcpyAsync(buf[j & 1], x.dev + (q - x.off), (size_t)n, cudaMemcpyDeviceToHost, c->copy_stream));
      CK(cudaEventRecord(c->copy_ev[j & 1], c->copy_stream));
      if (prev >= 0) {
        CK(cudaEventSynchronize(c->copy_ev[(j - 1) & 1]));
        memcpy(dst + (prev - offset), buf[(j - 1) & 1], (size_t)prev_n);
      }
      prev = q;
      prev_n = n;
    }
    CK(cudaEventSynchronize(c->copy_ev[(j - 1) & 1]));
    memcpy(dst + (prev - offset), buf[(j - 1) & 1], (size_t)prev_n);
    cur = b;
  }
  gap(end);
  return CCO_OK;
}

// ---- load ---------------------------------------------------------------------------------------------------------------
static const char *snap_name(uint32_t k) { return k > 0 && k < kSnEnd ? kSnName[k] : "?"; }
// the header and the section table, complete: checked before anything is allocated; then the device sections' buffers
static int snap_table(cco_event_log *lg) {
  SnapLoad &ld = *lg->load;
  const std::string &h = ld.head;
  const long long NS = ld.n_sec, tab = kSnapHead + kSnapEntry * NS;
  std::string z = h;
  memset(&z[32], 0, 8);
  if (snap_sum_host((const unsigned char *)z.data(), tab) != snap_get<uint64_t>(h, 32))
    return set_error(CCO_E_INVALID_ARG, "snapshot header: checksum mismatch");
  long long prev_end = tab;
  uint32_t prev_kind = 0;
  for (long long i = 0; i < NS; ++i) {
    const long long e = kSnapHead + kSnapEntry * i;
    SnapSec x;
    x.kind = snap_get<uint32_t>(h, e);
    x.off = snap_get<int64_t>(h, e + 8);
    x.len = snap_get<int64_t>(h, e + 16);
    x.alloc = snap_get<int64_t>(h, e + 24);
    x.sum = snap_get<uint64_t>(h, e + 32);
    const char *nm = snap_name(x.kind);
    if (x.kind <= prev_kind || x.kind >= kSnEnd || snap_get<uint32_t>(h, e + 4) != 0)
      return set_error(CCO_E_INVALID_ARG, "snapshot section table: entry %lld has kind %u (unknown, repeated or out of order)", i, x.kind);
    if (x.off % kSnapAlign != 0) return set_error(CCO_E_INVALID_ARG, "snapshot section %s: offset %lld is not 256-byte aligned", nm, x.off);
    if (x.off < prev_end) return set_error(CCO_E_INVALID_ARG, "snapshot section %s: overlaps the section table or the section before it", nm);
    if (x.len < 0 || x.len > ld.total - x.off)
      return set_error(CCO_E_INVALID_ARG, "snapshot section %s: [%lld, +%lld) runs past the end (%lld bytes)", nm, x.off, x.len, ld.total);
    if (snap_host_kind(x.kind) ? x.alloc != 0 : (x.alloc < snap_need(x.kind, x.len) || x.alloc > 2 * snap_need(x.kind, x.len) + 4096))
      return set_error(CCO_E_INVALID_ARG, "snapshot section %s: %lld device bytes for %lld bytes", nm, x.alloc, x.len);
    prev_end = x.off + x.len;
    prev_kind = x.kind;
    ld.secs.push_back(std::move(x));
  }
  if (prev_end != ld.total) return set_error(CCO_E_INVALID_ARG, "snapshot: %lld bytes, its last section ends at %lld", ld.total, prev_end);
  cco_ctx *c = lg->ctx;
  Arena ar(c->stream);
  for (SnapSec &x : ld.secs) {
    if (!x.alloc) {
      x.host.reserve((size_t)x.len);
      continue;
    }
    CKR(ar.alloc(&x.dev, (size_t)x.alloc));
    CKR(log_keep(ar, lg, x.dev));
  }
  CK(cudaStreamSynchronize(c->stream));   // the copies run on the copy stream
  for (SnapSec &x : ld.secs)
    if (x.dev) CK(cudaMemsetAsync(x.dev, 0, (size_t)x.alloc, c->copy_stream));
  ld.table = true;
  return CCO_OK;
}
static int snap_append(cco_event_log *lg, const unsigned char *bytes, long long len) {
  cco_ctx *c = lg->ctx;
  CK(cudaSetDevice(c->device));
  SnapLoad &ld = *lg->load;
  while (len > 0 && !ld.table) {
    const long long want = ld.head.size() < (size_t)kSnapHead ? kSnapHead : kSnapHead + kSnapEntry * ld.n_sec;
    const long long take = std::min(len, want - (long long)ld.head.size());
    ld.head.append((const char *)bytes, (size_t)take);
    ld.pos += take;
    bytes += take;
    len -= take;
    if ((long long)ld.head.size() == kSnapHead && want == kSnapHead) {
      const std::string &h = ld.head;
      if (memcmp(h.data(), kSnapMagic, 8) != 0) return set_error(CCO_E_INVALID_ARG, "snapshot header: not an event log snapshot (bad magic)");
      if (snap_get<uint32_t>(h, 8) != kSnapVersion)
        return set_error(CCO_E_INVALID_ARG, "snapshot header: format version %u, this library reads %u", snap_get<uint32_t>(h, 8), kSnapVersion);
      if (snap_get<uint32_t>(h, 12) != CCO_ABI_VERSION)
        return set_error(CCO_E_INVALID_ARG, "snapshot header: ABI version %u, this library is %u", snap_get<uint32_t>(h, 12), (unsigned)CCO_ABI_VERSION);
      ld.n_sec = snap_get<uint32_t>(h, 16);
      ld.total = snap_get<int64_t>(h, 24);
      if (ld.n_sec < 1 || ld.n_sec >= kSnEnd) return set_error(CCO_E_INVALID_ARG, "snapshot header: %lld sections", ld.n_sec);
      if (ld.total < kSnapHead + kSnapEntry * ld.n_sec) return set_error(CCO_E_INVALID_ARG, "snapshot header: %lld bytes, shorter than its section table", ld.total);
    }
    if ((long long)ld.head.size() == kSnapHead + kSnapEntry * ld.n_sec && ld.n_sec > 0) CKR(snap_table(lg));
  }
  if (len == 0) return CCO_OK;
  if (len > ld.total - ld.pos) return set_error(CCO_E_INVALID_ARG, "snapshot: bytes past its end (%lld bytes)", ld.total);
  const long long a = ld.pos, b = a + len;
  for (SnapSec &x : ld.secs) {
    const long long p = std::max(a, x.off), q = std::min(b, x.off + x.len);
    if (p >= q) continue;
    const unsigned char *src = bytes + (p - a);
    if (!x.dev) {
      x.host.append((const char *)src, (size_t)(q - p));
      continue;
    }
    CK(cudaMemcpyAsync(x.dev + (p - x.off), src, (size_t)(q - p), cudaMemcpyHostToDevice, c->copy_stream));
    if (x.kind == kSnPropBytes) {   // the lines a later finish parses: counted here, checked against property_lines
      for (const unsigned char *r = src, *e = src + (q - p); (r = (const unsigned char *)memchr(r, '\n', (size_t)(e - r))); ++r) ++ld.pb_newlines;
      ld.pb_last = src[q - p - 1];
    }
  }
  ld.pos = b;
  CK(cudaStreamSynchronize(c->copy_stream));   // the bytes are copied: the caller may reuse its buffer
  return CCO_OK;
}

// the checks of a complete snapshot and the log built from it
static int snap_finish(cco_event_log *lg) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  CK(cudaSetDevice(c->device));
  NvtxRange nvtx("cco:event_log_load");
  SnapLoad &ld = *lg->load;
  if (!ld.table) return set_error(CCO_E_INVALID_ARG, "snapshot truncated at byte %lld: the header and section table are incomplete", ld.pos);
  if (ld.pos < ld.total) {
    for (const SnapSec &x : ld.secs)
      if (x.off + x.len > ld.pos)
        return set_error(CCO_E_INVALID_ARG, "snapshot truncated at byte %lld of %lld: section %s is incomplete", ld.pos, ld.total, kSnName[x.kind]);
  }
  CK(cudaStreamSynchronize(c->copy_stream));
  SnapSec *sec[kSnEnd] = {};
  std::vector<SnapSec *> dev;
  for (SnapSec &x : ld.secs) {
    sec[x.kind] = &x;
    if (x.dev) dev.push_back(&x);
  }
  std::vector<uint64_t> want;
  for (SnapSec *x : dev) want.push_back(x->sum);
  for (SnapSec &x : ld.secs)
    if (!x.dev && snap_sum_host((const unsigned char *)x.host.data(), x.len) != x.sum)
      return set_error(CCO_E_INVALID_ARG, "snapshot section %s: checksum mismatch", kSnName[x.kind]);
  mail_reset(c);
  CKR(snap_device_sums(c, dev));
  for (size_t i = 0; i < dev.size(); ++i)
    if (dev[i]->sum != want[i]) return set_error(CCO_E_INVALID_ARG, "snapshot section %s: checksum mismatch", kSnName[dev[i]->kind]);
  // host state
  for (uint32_t k : {kSnState, kSnNames, kSnCounts, kSnFields})
    if (!sec[k]) return set_error(CCO_E_INVALID_ARG, "snapshot section %s: missing", kSnName[k]);
  if (sec[kSnState]->len != 8 * kSnapStateWords) return set_error(CCO_E_INVALID_ARG, "snapshot section state: %lld bytes, not %lld", sec[kSnState]->len, 8 * kSnapStateWords);
  int64_t st[kSnapStateWords];
  memcpy(st, sec[kSnState]->host.data(), sizeof st);
  const int64_t flags = st[0];
  if (flags & ~(int64_t)(CCO_LOG_KEEP_HISTORY | CCO_LOG_EXTENDABLE | CCO_LOG_INTERN_IDS))
    return set_error(CCO_E_INVALID_ARG, "snapshot section state: unknown flags 0x%llx", (long long)flags);
  bool counters_ok = (st[1] == 0 || st[1] == 1) && st[3] >= 1;
  for (int i = 4; i <= 10; ++i) counters_ok = counters_ok && st[i] >= 0;
  counters_ok = counters_ok && st[12] >= 0;
  for (int i = 13; i < kSnapStateWords; ++i) counters_ok = counters_ok && st[i] == 0;
  if (!counters_ok) return set_error(CCO_E_INVALID_ARG, "snapshot section state: a counter is out of range");
  lg->history = flags & CCO_LOG_KEEP_HISTORY;
  lg->extendable = flags & CCO_LOG_EXTENDABLE;
  lg->intern = flags & CCO_LOG_INTERN_IDS;
  lg->dedup = st[1] != 0;
  lg->cutoff = st[2];
  lg->chunk0 = st[3];
  lg->n_lines = st[4];
  lg->n_prop = st[5];
  lg->n_ignored = st[6];
  lg->n_prop_items = st[7];
  lg->n_prop_fields = st[8];
  lg->n_expired = st[9];
  lg->n_dup = st[10];
  lg->intern_mask = (uint64_t)st[11];
  lg->n_erased = st[12];
  std::vector<std::string> names;
  CKR(snap_unstrings(*sec[kSnNames], &names));
  const long long NG = (long long)names.size();
  for (long long g = 0; g < NG; ++g) {
    if (!lg->name_code.emplace(names[g], (int)g).second)
      return set_error(CCO_E_INVALID_ARG, "snapshot section names: name %lld repeats an earlier one", g);
    lg->name_bytes += names[g];
    lg->name_off.push_back((int64_t)lg->name_bytes.size());
  }
  if (sec[kSnCounts]->len != 16 * NG) return set_error(CCO_E_INVALID_ARG, "snapshot section counts: %lld bytes for %lld names", sec[kSnCounts]->len, NG);
  lg->n_train.resize(NG);
  lg->n_rank.resize(NG);
  memcpy(lg->n_train.data(), sec[kSnCounts]->host.data(), 8 * (size_t)NG);
  memcpy(lg->n_rank.data(), sec[kSnCounts]->host.data() + 8 * NG, 8 * (size_t)NG);
  lg->train_at.assign(NG + 1, 0);
  lg->rank_at.assign(NG + 1, 0);
  for (long long g = 0; g < NG; ++g) {
    if (lg->n_train[g] < 0 || lg->n_train[g] >= 0x7fffffffLL || lg->n_rank[g] < 0 || lg->n_rank[g] >= 0x7fffffffLL)
      return set_error(CCO_E_INVALID_ARG, "snapshot section counts: name %lld has %lld training and %lld ranking events", g, (long long)lg->n_train[g],
                       (long long)lg->n_rank[g]);
    lg->train_at[g + 1] = lg->train_at[g] + lg->n_train[g];
    lg->rank_at[g + 1] = lg->rank_at[g] + lg->n_rank[g];
  }
  CKR(snap_unstrings(*sec[kSnFields], &lg->field_names));
  for (size_t f = 0; f < lg->field_names.size(); ++f)
    for (size_t g = 0; g < f; ++g)
      if (lg->field_names[f] == lg->field_names[g]) return set_error(CCO_E_INVALID_ARG, "snapshot section fields: field %zu repeats an earlier one", f);
  if (lg->n_prop_fields > (long long)lg->field_names.size()) return set_error(CCO_E_INVALID_ARG, "snapshot section state: more property fields than field names");
  // which sections the flags allow, and the length each must have
  const long long NT = lg->train_at.back(), NR = lg->rank_at.back();
  const long long T = sec[kSnPField] ? sec[kSnPField]->len / 4 : 0;
  const long long UK = sec[kSnUserOff] ? sec[kSnUserOff]->len / 8 - 1 : 0, IK = sec[kSnItemOff] ? sec[kSnItemOff]->len / 8 - 1 : 0;
  for (uint32_t k = kSnPropLines; k < kSnEnd; ++k) {
    bool allowed = true;
    long long want_len = -1, n_entries = -1;   // -1: any length (the paired offsets decide the bytes)
    switch (k) {
      case kSnPropLines: case kSnPropBytes: case kSnRecords: case kSnRline: allowed = lg->extendable; break;
      case kSnDupTime: allowed = lg->extendable && lg->dedup; break;
      case kSnTline: allowed = lg->history || lg->extendable; break;
      case kSnTtime: allowed = lg->history; break;
      case kSnTkey: case kSnUserOff: case kSnUserBytes: case kSnItemOff: case kSnItemBytes: allowed = lg->intern; break;
      case kSnPItemOff: case kSnPItemBytes: allowed = !lg->extendable; break;
      default: break;
    }
    switch (k) {
      case kSnTuOff: case kSnTiOff: n_entries = NT; want_len = 8 * (NT + 1); break;
      case kSnRiOff: n_entries = NR; want_len = 8 * (NR + 1); break;
      case kSnRtime: case kSnRline: n_entries = NR; want_len = 8 * NR; break;
      case kSnTline: case kSnTtime: case kSnTkey: n_entries = NT; want_len = 8 * NT; break;
      case kSnPVoff: case kSnPIoff: n_entries = T; want_len = 8 * (T + 1); break;
      case kSnPItemOff: n_entries = lg->n_prop; want_len = 8 * (lg->n_prop + 1); break;
      case kSnPropLines: n_entries = lg->n_prop; want_len = 8 * lg->n_prop; break;
      default: break;
    }
    SnapSec *x = sec[k];
    const char *nm = kSnName[k];
    if (x && !allowed) return set_error(CCO_E_INVALID_ARG, "snapshot section %s: not part of a log with flags 0x%llx", nm, (long long)flags);
    if (!x) {   // an absent column holds no entries
      const uint32_t ko = snap_off_of(k);
      if (allowed && (n_entries > 0 || (ko && sec[ko]) || (lg->intern && (k == kSnUserOff || k == kSnItemOff))))
        return set_error(CCO_E_INVALID_ARG, "snapshot section %s: missing", nm);
      continue;
    }
    if (snap_off_of(k) && !sec[snap_off_of(k)]) return set_error(CCO_E_INVALID_ARG, "snapshot section %s: its offsets are missing", nm);
    if ((k == kSnPVoff || k == kSnPIoff || k == kSnPVals || k == kSnPIbytes) && !sec[kSnPField])
      return set_error(CCO_E_INVALID_ARG, "snapshot section %s: the property fields are missing", nm);
    if (want_len >= 0 && x->len != want_len)
      return set_error(CCO_E_INVALID_ARG, "snapshot section %s: %lld bytes, its counters give %lld", nm, x->len, want_len);
    const long long unit = k == kSnRecords ? (long long)sizeof(WinRec) : k == kSnPField ? 4 : (k == kSnUserOff || k == kSnItemOff || k == kSnDupTime) ? 8 : 1;
    if (x->len % unit != 0 || ((k == kSnUserOff || k == kSnItemOff) && x->len < 8))
      return set_error(CCO_E_INVALID_ARG, "snapshot section %s: %lld bytes is not a whole number of entries", nm, x->len);
    if (k == kSnPField && T == 0) return set_error(CCO_E_INVALID_ARG, "snapshot section %s: present without entries", nm);
  }
  if (sec[kSnPropBytes]) {
    const long long NP = sec[kSnPropLines] ? sec[kSnPropLines]->len / 8 : 0;
    if (ld.pb_newlines != NP || ld.pb_last != '\n' || NP == 0)
      return set_error(CCO_E_INVALID_ARG, "snapshot section property_bytes: its lines disagree with property_lines");
  } else if (lg->extendable && lg->n_prop > 0) {
    return set_error(CCO_E_INVALID_ARG, "snapshot section property_bytes: missing");
  }
  if (sec[kSnPropLines]) {
    lg->prop_line.resize((size_t)lg->n_prop);
    memcpy(lg->prop_line.data(), sec[kSnPropLines]->host.data(), 8 * (size_t)lg->n_prop);
    for (long long i = 0; i < lg->n_prop; ++i)
      if (lg->prop_line[i] < 0 || lg->prop_line[i] >= lg->n_lines || (i > 0 && lg->prop_line[i] <= lg->prop_line[i - 1]))
        return set_error(CCO_E_INVALID_ARG, "snapshot section property_lines: line %lld is out of order or >= the line count", i);
  }
  // device checks: one k_snap_check over every checked section, its verdict before anything reads through an offset
  std::vector<SnapTask> tk;
  std::vector<uint32_t> tkind;
  long long at = 0;
  auto task = [&](uint32_t k, int kind, long long n, long long bound, long long bound2) {
    if (!sec[k] || n <= 0) return;
    tk.push_back(SnapTask{sec[k]->dev, n, at, bound, bound2, kind});
    tkind.push_back(k);
    at += n;
  };
  for (uint32_t k : {kSnTuBytes, kSnTiBytes, kSnRiBytes, kSnPVals, kSnPIbytes, kSnPItemBytes, kSnUserBytes, kSnItemBytes}) {
    const uint32_t ko = snap_off_of(k);
    if (sec[ko]) task(ko, kSnapOffsets, sec[ko]->len / 8, sec[k] ? sec[k]->len : 0, 0);
  }
  task(kSnTline, kSnapBelow, NT, lg->n_lines, 0);
  task(kSnRline, kSnapBelow, NR, lg->n_lines, 0);
  task(kSnTkey, kSnapKeys, NT, UK, IK);
  task(kSnPField, kSnapFields, T, (long long)lg->field_names.size(), 0);
  task(kSnRecords, kSnapRecords, sec[kSnRecords] ? sec[kSnRecords]->len / (long long)sizeof(WinRec) : 0, lg->n_lines, NG);
  if (!tk.empty()) {
    Arena ar(s);
    SnapTask *d_tk;
    unsigned long long *bad, h_bad = ~0ULL;
    CKR(ar.alloc(&d_tk, tk.size()));
    CKR(ar.alloc(&bad, 1));
    CK(cudaMemcpyAsync(d_tk, tk.data(), sizeof(SnapTask) * tk.size(), cudaMemcpyHostToDevice, s));
    CK(cudaMemsetAsync(bad, 0xff, 8, s));
    k_snap_check<<<grid_for(at, 256, c->sm_count), 256, 0, s>>>((int)tk.size(), d_tk, at, bad);
    c->launches++;
    CKR(mail_fetch(c, &h_bad, bad, 8));
    CKR(mail_wait(c));
    if (h_bad != ~0ULL) {
      const SnapTask &t = tk[h_bad >> 40];
      const long long i = (long long)(h_bad & ((1ULL << 40) - 1));
      const char *nm = kSnName[tkind[h_bad >> 40]];
      switch (t.kind) {
        case kSnapOffsets:
          return set_error(CCO_E_INVALID_ARG, "snapshot section %s: offset %lld decreases, does not start at 0 or does not end at the %lld bytes", nm, i, t.bound);
        case kSnapBelow: return set_error(CCO_E_INVALID_ARG, "snapshot section %s: entry %lld is not a line of the log (%lld lines)", nm, i, t.bound);
        case kSnapKeys: return set_error(CCO_E_INVALID_ARG, "snapshot section %s: entry %lld holds a key >= its table's key count", nm, i);
        case kSnapFields: return set_error(CCO_E_INVALID_ARG, "snapshot section %s: entry %lld is not a field of the %lld names", nm, i, t.bound);
        default:
          return set_error(CCO_E_INVALID_ARG, "snapshot section %s: record %lld is out of line order, >= the line count or of a name >= %lld", nm, i, t.bound2);
      }
    }
  }
  // the log: the sections are its buffers
  for (SnapSec *x : dev) *snap_slot(lg, x->kind) = x->dev;
  lg->n_triples = T;
  lg->p_ibytes_n = sec[kSnPIbytes] ? sec[kSnPIbytes]->len : 0;
  if (sec[kSnRecords]) {
    lg->n_rec = sec[kSnRecords]->len / (long long)sizeof(WinRec);
    lg->rec_cap = sec[kSnRecords]->alloc / (long long)sizeof(WinRec);
  }
  lg->n_dup_time = sec[kSnDupTime] ? sec[kSnDupTime]->len / 8 : 0;
  if (sec[kSnPropBytes]) {
    lg->pb_len = sec[kSnPropBytes]->len;
    lg->pb_cap = sec[kSnPropBytes]->alloc - 24;
  }
  Arena ar(s);
  for (auto cl : {std::make_pair(&lg->tu, &lg->train_at), std::make_pair(&lg->ti, &lg->train_at), std::make_pair(&lg->ri, &lg->rank_at)}) {
    if (cl.first->off) CKR(name_boff(c, ar, cl.first->off, *cl.second, &cl.first->boff));
    else cl.first->boff.assign(NG + 1, 0);
  }
  // the intern tables: the stored strings hashed and claimed into empty tables, each its own key; a string stored twice
  // would claim one slot for both
  if (lg->intern) {
    InternTable *tbs[2] = {&lg->users, &lg->items};
    for (int x = 0; x < 2; ++x) {
      InternTable *tb = tbs[x];
      const uint32_t ko = x == 0 ? kSnUserOff : kSnItemOff;
      const long long K = sec[ko]->len / 8 - 1;
      tb->n = tb->kcap = K;
      tb->bytes = tb->bcap = sec[ko + 1]->len;
      tb->cap = intern_slots(K);
      CKR(ar.alloc(&tb->hash, std::max<long long>(K, 1)));
      CKR(log_keep(ar, lg, tb->hash));
      CKR(ar.alloc(&tb->table, tb->cap));
      CKR(log_keep(ar, lg, tb->table));
      CK(cudaMemsetAsync(tb->table, 0xff, sizeof(uint32_t) * (size_t)tb->cap, s));
      if (K == 0) continue;
      uint64_t *hash;
      uint32_t *slot_of, *flag, *pos, *idx, KN = 0;
      CKR(ar.alloc(&hash, K));
      CKR(ar.alloc(&slot_of, K));
      CKR(ar.alloc(&flag, K + 1));
      k_str_hash<<<grid_for(K, 256, c->sm_count), 256, 0, s>>>(K, tb->off, 0, tb->w, lg->intern_mask, hash);
      k_intern_claim<<<grid_for(K, 256, c->sm_count), 256, 0, s>>>(K, tb->off, tb->w, hash, tb->off, tb->w, tb->hash, (uint64_t)tb->cap - 1,
                                                                   tb->table, slot_of);
      k_intern_first<<<grid_for(K, 256, c->sm_count), 256, 0, s>>>(K, slot_of, tb->table, flag);
      c->launches += 3;
      CKR(select_flagged(c, ar, K, flag, &pos, &idx));
      CKR(mail_fetch(c, &KN, pos + K, 4));
      CKR(mail_wait(c));
      if (KN != (uint32_t)K) return set_error(CCO_E_INVALID_ARG, "snapshot section %s: an id is stored twice", kSnName[ko + 1]);
      k_intern_new<<<grid_for(K, 256, c->sm_count), 256, 0, s>>>(K, idx, slot_of, hash, 0, tb->table, tb->hash);
      c->launches++;
    }
  }
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  lg->load.reset();
  lg->finished = true;
  return CCO_OK;
}
// a failed load keeps no device memory: the log answers with its message until it is freed
static int snap_fail(cco_event_log *lg, int rc) {
  if (rc == CCO_OK) return rc;
  log_fail(lg, rc);
  cudaSetDevice(lg->ctx->device);
  cudaStreamSynchronize(lg->ctx->copy_stream);
  for (void *p : lg->dev) cudaFreeAsync(p, lg->ctx->stream);
  cudaStreamSynchronize(lg->ctx->stream);
  lg->dev.clear();
  lg->dev_bytes.clear();
  lg->load.reset();
  return rc;
}
}  // namespace cco

int cco_event_log_save_size(cco_event_log_t *lg, int64_t *bytes) {
  if (!lg || !bytes) return set_error(CCO_E_INVALID_ARG, "null argument");
  CKR(log_state(lg, true));
  CK(cudaSetDevice(lg->ctx->device));
  CKR(snap_image(lg));
  *bytes = lg->snap->total;
  return CCO_OK;
}

int cco_event_log_save(cco_event_log_t *lg, int64_t offset, void *dst, int64_t len) {
  if (!lg || offset < 0 || len < 0 || (len > 0 && !dst)) return set_error(CCO_E_INVALID_ARG, "null argument, or a negative offset or length");
  CKR(log_state(lg, true));
  CK(cudaSetDevice(lg->ctx->device));
  NvtxRange nvtx("cco:event_log_save");
  CKR(snap_image(lg));
  if (len > lg->snap->total - offset)
    return set_error(CCO_E_INVALID_ARG, "bytes [%lld, %lld) of a %lld-byte snapshot", (long long)offset, (long long)(offset + len), lg->snap->total);
  return snap_save(lg, offset, (unsigned char *)dst, len);
}

int cco_event_log_load_begin(cco_ctx_t *ctx, cco_event_log_t **out) {
  if (!ctx || !out) return set_error(CCO_E_INVALID_ARG, "null argument");
  *out = nullptr;
  if (!ctx->members.empty()) return set_error(CCO_E_UNSUPPORTED, "an event log is resident on one GPU: load it on a per-GPU context");
  CK(cudaSetDevice(ctx->device));
  cco_event_log *lg = new cco_event_log();
  lg->ctx = ctx;
  lg->name_off.assign(1, 0);
  lg->train_at.assign(1, 0);
  lg->rank_at.assign(1, 0);
  lg->load.reset(new SnapLoad());
  *out = lg;
  return CCO_OK;
}

int cco_event_log_load_append(cco_event_log_t *lg, const void *bytes, int64_t len) {
  if (!lg || len < 0 || (len > 0 && !bytes)) return set_error(CCO_E_INVALID_ARG, "null argument or negative length");
  if (lg->fail != CCO_OK) return set_error(CCO_E_INVALID_ARG, "the load of this log failed: %s", lg->fail_msg.c_str());
  if (!lg->load) return set_error(CCO_E_INVALID_ARG, "the log is not being loaded (cco_event_log_load_begin)");
  return snap_fail(lg, snap_append(lg, (const unsigned char *)bytes, len));
}

int cco_event_log_load_finish(cco_event_log_t *lg) {
  if (!lg) return set_error(CCO_E_INVALID_ARG, "null argument");
  if (lg->fail != CCO_OK) return set_error(CCO_E_INVALID_ARG, "the load of this log failed: %s", lg->fail_msg.c_str());
  if (!lg->load) return set_error(CCO_E_INVALID_ARG, "the log is not being loaded (cco_event_log_load_begin)");
  return snap_fail(lg, snap_finish(lg));
}

// ---- SURVEY.md 8f-3: PopModel rank histograms -------------------------------------------------------------------------
int cco_pop_model(cco_ctx_t *ctx, int32_t mode, int64_t n_events, const int32_t *item, const int64_t *time_ms, int32_t n_items,
                  int64_t start_ms, int64_t end_ms, double *score, unsigned char *present) {
  if (!ctx || n_events < 0 || n_items < 0 || (n_events > 0 && (!item || !time_ms)) || (n_items > 0 && (!score || !present)))
    return set_error(CCO_E_INVALID_ARG, "bad argument");
  if (mode < CCO_POP_POPULAR || mode > CCO_POP_HOT) return set_error(CCO_E_INVALID_ARG, "mode must be CCO_POP_POPULAR, _TRENDING or _HOT");
  if (end_ms < start_ms) return set_error(CCO_E_INVALID_ARG, "end before start (Joda Interval would throw)");
  if (n_items == 0) return CCO_OK;
  cco_ctx *c = ctx->members.empty() ? ctx : ctx->members[0];
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Arena ar(s);
  NvtxRange nvtx("cco:pop_model");
  const PopArgs a = pop_args(mode, start_ms, end_ms, n_items);
  int32_t *d_item, *d_counts;
  long long *d_t;
  unsigned long long *d_tot;
  double *d_score;
  unsigned char *d_present;
  CKR(ar.alloc(&d_item, std::max<long long>(n_events, 1)));
  CKR(ar.alloc(&d_t, std::max<long long>(n_events, 1)));
  CKR(ar.alloc(&d_counts, (size_t)a.n_buckets * n_items));
  CKR(ar.alloc(&d_tot, 4));
  CKR(ar.alloc(&d_score, n_items));
  CKR(ar.alloc(&d_present, n_items));
  CK(cudaMemsetAsync(d_counts, 0, sizeof(int32_t) * (size_t)a.n_buckets * n_items, s));
  CK(cudaMemsetAsync(d_tot, 0, 32, s));
  if (n_events > 0) {
    CK(cudaMemcpyAsync(d_item, item, sizeof(int32_t) * (size_t)n_events, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_t, time_ms, sizeof(int64_t) * (size_t)n_events, cudaMemcpyHostToDevice, s));
    k_pop_count<<<grid_for(n_events, 256, c->sm_count), 256, 0, s>>>(n_events, d_item, d_t, a, d_counts, d_tot);
    c->launches++;
  }
  k_pop_score<double><<<grid_for(n_items, 256, c->sm_count), 256, 0, s>>>(a, mode, d_counts, d_tot, d_score, d_present);
  c->launches++;
  CK(cudaMemcpyAsync(score, d_score, sizeof(double) * (size_t)n_items, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(present, d_present, (size_t)n_items, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  return CCO_OK;
}

void cco_free(void *p) { free(p); }

// ---- debug / parity entries ------------------------------------------------------------------------
int cco_debug_llr(cco_ctx_t *c, int64_t n, const int64_t *k11, const int64_t *k12, const int64_t *k21, const int64_t *k22,
                  uint32_t flags, double *out) {
  if (!c || n < 0 || (n > 0 && (!k11 || !k12 || !k21 || !k22 || !out))) return set_error(CCO_E_INVALID_ARG, "bad argument");
  if (n == 0) return CCO_OK;
  for (int64_t i = 0; i < n; ++i)
    if (k11[i] < 0 || k12[i] < 0 || k21[i] < 0 || k22[i] < 0)
      return set_error(CCO_E_INVALID_ARG, "negative count at %lld (Preconditions.checkArgument in LogLikelihood)", (long long)i);
  CK(cudaSetDevice(c->device));
  Arena ar(c->stream);
  long long *d[4];
  double *dout;
  const int64_t *h[4] = {k11, k12, k21, k22};
  for (int j = 0; j < 4; ++j) {
    CKR(ar.alloc(&d[j], n));
    CK(cudaMemcpyAsync(d[j], h[j], sizeof(int64_t) * (size_t)n, cudaMemcpyHostToDevice, c->stream));
  }
  CKR(ar.alloc(&dout, n));
  k_debug_llr<<<(unsigned)((n + 255) / 256), 256, 0, c->stream>>>(n, d[0], d[1], d[2], d[3], flags, dout);
  CK(cudaMemcpyAsync(out, dout, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  CK(cudaGetLastError());
  return CCO_OK;
}

int cco_debug_rank_text(cco_ctx_t *c, int64_t n, const int64_t *v, int32_t scale, int64_t *offsets, char *bytes) {
  if (!c || n < 0 || !offsets || (n > 0 && (!v || !bytes))) return set_error(CCO_E_INVALID_ARG, "bad argument");
  if (scale != 0 && scale != 15) return set_error(CCO_E_INVALID_ARG, "scale %d is neither 0 nor 15", scale);
  for (int64_t i = 0; i < n; ++i)
    if (scale == 0 ? (v[i] <= -(1LL << 53) || v[i] >= (1LL << 53)) : (v[i] < 0 || v[i] >= 1000000000000000LL))
      return set_error(CCO_E_INVALID_ARG, "value %lld at %lld is outside the range of scale %d", (long long)v[i], (long long)i, scale);
  offsets[0] = 0;
  if (n == 0) return CCO_OK;
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  Arena ar(s);
  long long *d_v;
  unsigned char *d_slot;
  int32_t *d_len;
  CKR(ar.alloc(&d_v, n));
  CKR(ar.alloc(&d_slot, 32 * n));
  CKR(ar.alloc(&d_len, n));
  CK(cudaMemcpyAsync(d_v, v, sizeof(int64_t) * (size_t)n, cudaMemcpyHostToDevice, s));
  k_debug_rank_text<<<grid_for(n, 256, c->sm_count), 256, 0, s>>>(n, d_v, scale, d_slot, d_len);
  std::vector<unsigned char> slot((size_t)32 * n);
  std::vector<int32_t> len((size_t)n);
  CK(cudaMemcpyAsync(slot.data(), d_slot, slot.size(), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(len.data(), d_len, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  for (int64_t i = 0; i < n; ++i) {
    if (len[i] < 1 || len[i] > 32) return set_error(CCO_E_CUDA, "text %lld has length %d", (long long)i, len[i]);
    memcpy(bytes + offsets[i], slot.data() + 32 * (size_t)i, (size_t)len[i]);
    offsets[i + 1] = offsets[i] + len[i];
  }
  return CCO_OK;
}

int cco_debug_downsample(cco_ctx_t *c, const cco_csr_t *m, int32_t max_interactions, int32_t seed, uint32_t flags,
                         int64_t **row_ptr, int32_t **col_idx, int32_t *raw_col_counts, int32_t *new_col_counts) {
  if (!c || !m || !row_ptr || !col_idx) return set_error(CCO_E_INVALID_ARG, "null argument");
  if (c->world != 1 || !c->members.empty()) return set_error(CCO_E_UNSUPPORTED, "debug entries need a single-GPU context");
  cco_indicator_params_t prm = {max_interactions, 1, 0, 0.0};
  CKR(validate_host(1, m, &prm));
  CK(cudaSetDevice(c->device));
  mail_reset(c);
  c->ev_timing_used = c->ev_plain_used = 0;
  cco_dataset *ds = nullptr;
  CKR(dataset_upload(c, 1, m, flags, &ds));
  struct DG { cco_dataset *d; ~DG() { dataset_release(d); } } dg{ds};
  Arena ar(c->stream);
  Prepared p;   // the raw counts, the verdict and the sample exactly as the train makes them
  CKR(prepare(c, ar, ds, &prm, seed, flags, &p));
  const DevMat &dm = p.dm[0];
  std::vector<uint32_t> rp32((size_t)m->n_rows + 1);
  CK(cudaMemcpyAsync(rp32.data(), dm.rp, sizeof(uint32_t) * rp32.size(), cudaMemcpyDeviceToHost, c->stream));
  if (raw_col_counts && m->n_cols > 0)
    CK(cudaMemcpyAsync(raw_col_counts, p.raw_counts, sizeof(int32_t) * (size_t)m->n_cols, cudaMemcpyDeviceToHost, c->stream));
  if (new_col_counts && m->n_cols > 0)
    CK(cudaMemcpyAsync(new_col_counts, dm.marg, sizeof(int32_t) * (size_t)m->n_cols, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  CK(cudaGetLastError());
  size_t nnz = rp32[m->n_rows];
  int64_t *rp = (int64_t *)malloc(sizeof(int64_t) * rp32.size());
  int32_t *ci = (int32_t *)calloc(std::max<size_t>(nnz, 1), sizeof(int32_t));
  if (!rp || !ci) return set_error(CCO_E_OOM, "malloc failed");
  for (size_t i = 0; i < rp32.size(); ++i) rp[i] = rp32[i];
  // (kept counts beyond the matrix's entries show in row_ptr; the copy stays inside the sampled columns, the tail stays 0)
  const size_t n_copy = std::min<size_t>(nnz, (size_t)ds->nnz[0]);
  if (n_copy) CK(cudaMemcpy(ci, dm.col, sizeof(int32_t) * n_copy, cudaMemcpyDeviceToHost));
  *row_ptr = rp;
  *col_idx = ci;
  return CCO_OK;
}

// one rank's share of downsample_all on one GPU: the rank that owns users [row_lo, row_hi) samples them with
// row_base = row_lo, absolute entry offsets, the whole matrix's raw counts and kept counts indexed by global user
int cco_debug_downsample_block(cco_ctx_t *c, const cco_csr_t *m, int64_t row_lo, int64_t row_hi, const int32_t *raw_col_counts,
                               int32_t max_interactions, int32_t seed, uint32_t flags, int64_t *kept_per_row, int32_t **col_idx,
                               int32_t *new_col_counts) {
  if (!c || !m || !col_idx || (m->n_rows > 0 && !kept_per_row) || (m->n_cols > 0 && (!raw_col_counts || !new_col_counts)))
    return set_error(CCO_E_INVALID_ARG, "null argument");
  if (c->world != 1 || !c->members.empty()) return set_error(CCO_E_UNSUPPORTED, "debug entries need a single-GPU context");
  cco_indicator_params_t prm = {max_interactions, 1, 0, 0.0};
  CKR(validate_host(1, m, &prm));
  if (row_lo < 0 || row_hi < row_lo || row_hi > m->n_rows)
    return set_error(CCO_E_INVALID_ARG, "rows [%lld, %lld) outside [0, %lld)", (long long)row_lo, (long long)row_hi, (long long)m->n_rows);
  CK(cudaSetDevice(c->device));
  mail_reset(c);
  cudaStream_t s = c->stream;
  cco_dataset *ds = nullptr;
  CKR(dataset_upload(c, 1, m, flags, &ds));
  struct DG { cco_dataset *d; ~DG() { dataset_release(d); } } dg{ds};
  Arena ar(s);
  const long long U = ds->n_users;
  const int32_t width = std::max<int32_t>(m->n_cols, 1);
  long long q[2] = {0, 0};   // the block's entries, from the (possibly canonicalised) device row_ptr
  CK(cudaMemcpyAsync(&q[0], ds->rp[0] + row_lo, sizeof(long long), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(&q[1], ds->rp[0] + row_hi, sizeof(long long), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  DevRaw blk;
  blk.n_rows = row_hi - row_lo;
  blk.row_base = row_lo;
  blk.n_cols = m->n_cols;
  blk.q_base = q[0];
  blk.nnz = q[1] - q[0];
  blk.rp = ds->rp[0] + row_lo;
  blk.col = ds->col[0];   // indexable by absolute offsets, as a rank's upload is
  int32_t *counts, *marg, *dst;
  uint32_t *kept;
  CKR(ar.alloc(&counts, width));
  CKR(ar.alloc(&marg, width));
  CKR(ar.alloc(&kept, U + 1));
  CKR(ar.alloc(&dst, std::max<long long>(blk.nnz, 1)));
  if (m->n_cols > 0) CK(cudaMemcpyAsync(counts, raw_col_counts, sizeof(int32_t) * (size_t)m->n_cols, cudaMemcpyHostToDevice, s));
  CK(cudaMemsetAsync(marg, 0, sizeof(int32_t) * (size_t)width, s));
  CK(cudaMemsetAsync(kept, 0, sizeof(uint32_t) * ((size_t)U + 1), s));
  SampleScratch sc;
  CKR(sample_scratch(c, ar, blk, counts, max_interactions, &sc));
  launch_count(c, blk, sc, max_interactions, seed, flags, nullptr, kept, marg);
  CKR(launch_write(c, ar, blk, sc, dst));
  std::vector<uint32_t> hk((size_t)U + 1);
  CK(cudaMemcpyAsync(hk.data(), kept, sizeof(uint32_t) * hk.size(), cudaMemcpyDeviceToHost, s));
  if (m->n_cols > 0) CK(cudaMemcpyAsync(new_col_counts, marg, sizeof(int32_t) * (size_t)m->n_cols, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  // the train lays the block's columns out by the scanned kept counts: as many as they sum to
  size_t n_kept = 0;
  for (long long r = 0; r < U; ++r) {
    kept_per_row[r] = hk[r];
    if (r >= row_lo && r < row_hi) n_kept += hk[r];
  }
  int32_t *ci = (int32_t *)calloc(std::max<size_t>(n_kept, 1), sizeof(int32_t));
  if (!ci) return set_error(CCO_E_OOM, "malloc failed");
  const size_t n_copy = std::min<size_t>(n_kept, (size_t)blk.nnz);   // (kept counts beyond the block's entries: the tail stays 0)
  if (n_copy) {
    cudaError_t e = cudaMemcpy(ci, dst, sizeof(int32_t) * n_copy, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) {
      free(ci);
      return set_error(CCO_E_CUDA, "cudaMemcpy: %s", cudaGetErrorString(e));
    }
  }
  *col_idx = ci;
  return CCO_OK;
}

int cco_debug_key_range_cap(cco_ctx_t *c, int32_t max_keys) {
  if (!c || max_keys < 0) return set_error(CCO_E_INVALID_ARG, "null context or negative cap");
  c->key_range_cap = max_keys;
  for (cco_ctx *m : c->members) m->key_range_cap = max_keys;
  return CCO_OK;
}

int cco_debug_intern_hash_bits(cco_ctx_t *c, int32_t bits) {
  if (!c || bits < 0 || bits > 64) return set_error(CCO_E_INVALID_ARG, "null context or hash bits %d not in [0, 64]", bits);
  c->intern_mask = bits == 64 ? ~0ULL : (1ULL << bits) - 1;
  return CCO_OK;
}

int cco_debug_cooccurrence(cco_ctx_t *c, const cco_csr_t *a, const cco_csr_t *b, int64_t **row_ptr, int32_t **col_idx,
                           int32_t **count) {
  if (!c || !a || !b || !row_ptr || !col_idx || !count) return set_error(CCO_E_INVALID_ARG, "null argument");
  if (c->world != 1 || !c->members.empty()) return set_error(CCO_E_UNSUPPORTED, "debug entries need a single-GPU context");
  cco_csr_t two[2] = {*a, *b};
  cco_indicator_params_t prm[2] = {{0x7fffffff, 1, 0, 0.0}, {0x7fffffff, 1, 0, 0.0}};
  CKR(validate_host(2, two, prm));
  CK(cudaSetDevice(c->device));
  mail_reset(c);
  c->ev_timing_used = c->ev_plain_used = 0;
  cco_dataset *ds = nullptr;
  CKR(dataset_upload(c, 2, two, 0, &ds));
  struct DG { cco_dataset *d; ~DG() { dataset_release(d); } } dg{ds};
  Arena ar(c->stream);
  struct CopyJoin {
    cco_ctx *c;
    ~CopyJoin() { cudaStreamSynchronize(c->copy_stream); }
  } copy_join{c};
  // the train's preparation with the identity sample (m = INT_MAX): the device CSR, marginals and A'^T
  Prepared prep;
  CKR(prepare(c, ar, ds, prm, 0, 0, &prep));
  const int32_t n_items_a = prep.dm[0].n_cols;
  ResultMat rm;
  IndicatorOut io;
  IndicatorState ist;
  struct EG { IndicatorState &x; ~EG() { if (x.packed) cudaEventDestroy(x.packed); } } eg{ist};
  cco_indicator_params_t p1 = {0x7fffffff, 1, 0, 0.0};
  auto put = [&]() {
    for (void *p : {(void *)rm.row_ptr, (void *)rm.col, (void *)rm.llr, (void *)rm.cnt})
      if (p) c->pinned_put(p);
  };
  int rc = enqueue_indicator(c, ar, prep.at_ptr, prep.at_users, n_items_a, prep.dm[0].marg, prep.max_marg[0], prep.max_marg[1], prep.dm[1],
                             a->n_rows, false, p1, 0, true, nullptr, nullptr, nullptr, &ist);
  if (rc == CCO_OK) rc = finish_indicator(c, &ist, 0, 0, &rm, &io);
  cudaStreamSynchronize(c->copy_stream);
  if (rc != CCO_OK) {
    put();
    return rc;
  }
  size_t nnz = (size_t)rm.row_ptr[n_items_a];
  int64_t *rp = (int64_t *)malloc(sizeof(int64_t) * ((size_t)n_items_a + 1));
  int32_t *ci = (int32_t *)malloc(sizeof(int32_t) * std::max<size_t>(nnz, 1));
  int32_t *cn = (int32_t *)malloc(sizeof(int32_t) * std::max<size_t>(nnz, 1));
  if (!rp || !ci || !cn) {
    put();
    return set_error(CCO_E_OOM, "malloc failed");
  }
  memcpy(rp, rm.row_ptr, sizeof(int64_t) * ((size_t)n_items_a + 1));
  // cells of a row come back in table order: sort each row by column for the caller
  std::vector<std::pair<int32_t, int32_t>> tmp;
  for (int32_t r = 0; r < n_items_a; ++r) {
    size_t lo = (size_t)rp[r], hi = (size_t)rp[r + 1];
    tmp.resize(hi - lo);
    for (size_t q = lo; q < hi; ++q) tmp[q - lo] = {rm.col[q], rm.cnt[q]};
    std::sort(tmp.begin(), tmp.end());
    for (size_t q = lo; q < hi; ++q) {
      ci[q] = tmp[q - lo].first;
      cn[q] = tmp[q - lo].second;
    }
  }
  put();
  *row_ptr = rp;
  *col_idx = ci;
  *count = cn;
  return CCO_OK;
}

// ---- what the readers of Elasticsearch responses share (search results, index pages, index write) ---------------------
extern "C++" {
namespace cco {

// A reader's first failure, repeated by every later call but free; a finished reader refuses every call but free.
struct ReaderLatch {
  bool failed = false, finished = false;
  std::string msg;
  int code = CCO_OK;
  int fail(int st) {
    failed = true;
    code = st;
    msg = cco_last_error();
    return st;
  }
  int state(const char *finished_msg) const {
    if (failed) return set_error(code == CCO_OK ? CCO_E_INVALID_ARG : code, "%s", msg.c_str());
    if (finished) return set_error(CCO_E_INVALID_ARG, "%s", finished_msg);
    return CCO_OK;
  }
};

// Response bodies on their way to the device, in one or two slots: per slot a pinned staging buffer and a device buffer,
// each grown to the largest body so far, and the event of the copy.  A body is padded with spaces to whole 64-byte words
// and one word more, as the structural passes read it, and copied on the copy stream.  A slot's next put reuses its
// buffers, so the slot's last body must have been read by then.
struct BodyStage {
  char *pinned[2] = {};
  size_t pinned_cap[2] = {};
  unsigned char *dev[2] = {};
  size_t dev_cap[2] = {};
  cudaEvent_t copied[2] = {};

  int init() {
    for (cudaEvent_t &e : copied)
      if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) return set_error(CCO_E_CUDA, "cudaEventCreate failed");
    return CCO_OK;
  }
  // what names the body in a refusal ("page 3 of 812 bytes"), copy_of in a failed copy ("page 3")
  int put(cco_ctx *c, int slot, const char *bytes, long long len, const char *what, const char *copy_of) {
    const size_t padded = (size_t)((len + 63) / 64 * 64) + 64;
    size_t free_b = 0, total_b = 0;
    CK(cudaMemGetInfo(&free_b, &total_b));
    if (padded > total_b / 4) return set_error(CCO_E_UNSUPPORTED, "%s: at most a quarter of the device's memory", what);
    if (pinned_cap[slot] < padded) {
      if (pinned[slot]) cudaFreeHost(pinned[slot]);
      pinned[slot] = nullptr;
      pinned_cap[slot] = 0;
      if (cudaHostAlloc((void **)&pinned[slot], padded, cudaHostAllocPortable) != cudaSuccess)
        return set_error(CCO_E_OOM, "cudaHostAlloc(%zu) failed", padded);
      pinned_cap[slot] = padded;
    }
    if (dev_cap[slot] < padded) {
      if (dev[slot]) cudaFree(dev[slot]);
      dev[slot] = nullptr;
      dev_cap[slot] = 0;
      if (cudaMalloc((void **)&dev[slot], padded) != cudaSuccess) return set_error(CCO_E_UNSUPPORTED, "%s does not fit the device", what);
      dev_cap[slot] = padded;
    }
    if (len > 0) memcpy(pinned[slot], bytes, (size_t)len);
    memset(pinned[slot] + len, ' ', padded - (size_t)len);
    if (cudaMemcpyAsync(dev[slot], pinned[slot], padded, cudaMemcpyHostToDevice, c->copy_stream) != cudaSuccess ||
        cudaEventRecord(copied[slot], c->copy_stream) != cudaSuccess)
      return set_error(CCO_E_CUDA, "the copy of %s failed", copy_of);
    return CCO_OK;
  }
  int wait(cudaStream_t s, int slot) const {
    CK(cudaStreamWaitEvent(s, copied[slot], 0));
    return CCO_OK;
  }
  const char *host(int slot) const { return pinned[slot]; }
  void release(cco_ctx *c) {
    cudaStreamSynchronize(c->copy_stream);
    for (int i = 0; i < 2; ++i) {
      if (pinned[i]) cudaFreeHost(pinned[i]);
      if (dev[i]) cudaFree(dev[i]);
      if (copied[i]) cudaEventDestroy(copied[i]);
    }
  }
};

static const char *sr_message(int code) {
  switch (code) {
    case kSrSyntax: return "malformed JSON";
    case kSrString: return "a string holds a bad escape or a raw byte < 0x20";
    case kSrUnbalanced: return "unbalanced or mismatched brackets";
    case kSrNoResponses: return "the top level is not an object with one \"responses\" array";
    case kSrElement: return "a responses element is not an object";
    case kSrStatus: return "status is not a 32-bit integer";
    case kSrHitsNotArray: return "hits.hits is not an array";
    case kSrHitNotObject: return "a hits.hits element is not an object";
    case kSrNoId: return "the hit has no string _id";
    case kSrRepeated: return "a repeated _id or _score";
    case kSrNoScore: return "_score is missing, null or not a number";
    case kSrBadRank: return "a rank is not a number";
    case kSrLine: return "the query line is not one JSON object";
    case kSrWithRanks: return "the query line's withRanks is not true, false or null";
    case kSrLineRepeated: return "the query line repeats withRanks";
    case kSrLineDeep: return "the query line nests deeper than 64 levels";
    case kSrOpenString: return "a string is not closed";
    case kSrNotObject: return "the top level is not an object";
    case kSrEsError: return "Elasticsearch returned an error";
    case kSrRepeatedId: return "a repeated _id";
    case kIpTimedOut: return "the search timed out (timed_out is true)";
    case kIpShards: return "_shards.failed is not 0";
    case kIpHitsNotArray: return "hits.hits is neither an array nor absent";
    case kIpNoSource: return "the hit has no _source";
    case kIpSourceNotObject: return "_source is not an object";
    case kIwNoItems: return "the response has no \"items\" array";
    case kIwItemNotObject: return "an items element is not an object";
    case kIwNotIndex: return "the item is not {\"index\":{...}}";
    case kIwNoId: return "the item has no string _id";
    case kIwIdMismatch: return "the item's _id is not the document's _id";
    case kIwNoStatus: return "the item has no status";
    case kIwRepeatedStatus: return "a repeated status";
    case kIwBadStatus: return "the status is not a 32-bit integer";
  }
  return "malformed response";
}

// The structural index of a body on the device, padded as BodyStage pads it: the byte positions pos[m] and depths dep[m]
// (in ar) of the entries at depth <= max_depth.  *bad = ~0, or (byte offset << 8 | kSr* code) of a malformed body.  The
// passes' scratch is released before it returns.
struct SrIndex {
  long long *pos = nullptr;
  unsigned char *dep = nullptr;
  long long m = 0;
};
static int sr_index(cco_ctx *c, Arena &ar, const unsigned char *body, long long len, int max_depth, SrIndex *ix, unsigned long long *bad) {
  cudaStream_t s = c->stream;
  const long long NW = (len + 63) / 64, n_chunks = (NW + kSrChunkWords - 1) / kSrChunkWords;
  unsigned long long *err;
  SrFun *fun, *pre;
  long long *cnt, *coff;
  CKR(ar.alloc(&err, 1));
  CKR(ar.alloc(&fun, n_chunks + 1));
  CKR(ar.alloc(&pre, n_chunks + 1));
  CKR(ar.alloc(&cnt, n_chunks + 1));
  CKR(ar.alloc(&coff, n_chunks + 1));
  CK(cudaMemsetAsync(err, 0xff, 8, s));
  CK(cudaMemsetAsync(cnt + n_chunks, 0, 8, s));
  SrFun fin = sr_identity();
  if (n_chunks > 0) {
    const int grid = grid_for(n_chunks * 32, 256, c->sm_count);
    k_sr_chunk<<<grid, 256, 0, s>>>(NW, (const uint4 *)body, fun);
    k_sr_scan<<<1, kSrScanThreads, 0, s>>>(n_chunks, fun, pre);
    k_sr_index<false><<<grid, 256, 0, s>>>(NW, (const uint4 *)body, pre, max_depth, cnt, nullptr, nullptr, nullptr, err);
    c->launches += 3;
    CKR(mail_fetch(c, &fin, pre + n_chunks - 1, sizeof(SrFun)));
  }
  CKR(exclusive_sum(c, ar, cnt, coff, n_chunks + 1));
  ix->m = 0;
  *bad = ~0ULL;
  CKR(mail_fetch(c, &ix->m, coff + n_chunks, 8));
  CKR(mail_fetch(c, bad, err, 8));
  CKR(mail_wait(c));
  if (*bad == ~0ULL && (fin.f[0] >> 1)) *bad = (unsigned long long)len << 8 | kSrOpenString;
  if (*bad == ~0ULL && fin.d[0] != 0) *bad = (unsigned long long)len << 8 | kSrUnbalanced;
  if (*bad == ~0ULL) {
    CKR(ar.alloc(&ix->pos, ix->m + 1));
    CKR(ar.alloc(&ix->dep, ix->m + 1));
    if (ix->m > 0) {
      k_sr_index<true><<<grid_for(n_chunks * 32, 256, c->sm_count), 256, 0, s>>>(NW, (const uint4 *)body, pre, max_depth, nullptr, coff, ix->pos,
                                                                                  ix->dep, err);
      c->launches++;
    }
  }
  for (void *p : {(void *)err, (void *)fun, (void *)pre, (void *)cnt, (void *)coff}) ar.release(p);
  return CCO_OK;
}

// A buffer of n bytes from the context's pinned pool for the caller, who frees it with cco_host_free: a copy of src, or
// left for the caller to fill when src is null.
template <typename T>
static int pinned_give(cco_ctx *c, T **out, const void *src, size_t n) {
  *out = (T *)c->pinned_get(std::max<size_t>(n, 1), /*for_result=*/false);
  if (!*out) return set_error(CCO_E_OOM, "pinned host allocation failed");
  if (src && n) memcpy(*out, src, n);
  return CCO_OK;
}

// a valid raw JSON string as UTF-8, a surrogate that is not part of a pair in its 3-byte form (k_json_unescape's rules)
static std::string sr_unescape(const char *p, long long n) {
  std::string o;
  auto hex4 = [](const char *q) { return (unsigned)strtoul(std::string(q, 4).c_str(), nullptr, 16); };
  for (long long i = 0; i < n;) {
    if (p[i] != '\\') {
      o += p[i++];
      continue;
    }
    const char x = p[i + 1];
    if (x != 'u') {
      o += x == 'b' ? '\b' : x == 'f' ? '\f' : x == 'n' ? '\n' : x == 'r' ? '\r' : x == 't' ? '\t' : x;
      i += 2;
      continue;
    }
    unsigned cp = hex4(p + i + 2);
    i += 6;
    if (cp >= 0xd800 && cp < 0xdc00 && i + 6 <= n && p[i] == '\\' && p[i + 1] == 'u') {
      const unsigned lo = hex4(p + i + 2);
      if (lo >= 0xdc00 && lo < 0xe000) {
        cp = 0x10000 + ((cp - 0xd800) << 10) + (lo - 0xdc00);
        i += 6;
      }
    }
    if (cp < 0x80) {
      o += (char)cp;
    } else if (cp < 0x800) {
      o += (char)(0xc0 | cp >> 6);
      o += (char)(0x80 | (cp & 0x3f));
    } else if (cp < 0x10000) {
      o += (char)(0xe0 | cp >> 12);
      o += (char)(0x80 | (cp >> 6 & 0x3f));
      o += (char)(0x80 | (cp & 0x3f));
    } else {
      o += (char)(0xf0 | cp >> 18);
      o += (char)(0x80 | (cp >> 12 & 0x3f));
      o += (char)(0x80 | (cp >> 6 & 0x3f));
      o += (char)(0x80 | (cp & 0x3f));
    }
  }
  return o;
}

}  // namespace cco
}  // extern "C++"

// ---- cco_search_results: _msearch response bodies -> PredictedResults, kernels in cco_results.cuh ----------------------
struct cco_search_results {
  cco_ctx *ctx = nullptr;
  int n_rank = 0;
  uint32_t flags = 0;
  std::string names, qnames;           // ranking names (UTF-8) and their json4s quotes, each followed by ':'
  int name_off[9] = {}, qname_off[9] = {};
  BodyStage stage;                     // the last two bodies
  long long n_bodies = 0;
  bool pending = false;                // the last appended body is copied, not yet read
  long long p_len = 0, p_rec = 0;
  std::vector<uint8_t> p_ranks;        // its records' withRanks, one byte each (without query lines)
  bool p_has_lines = false;            // its records' query lines (rebased offsets and bytes, copied at append)
  std::vector<int64_t> p_loff;
  std::string p_lines;
  ReaderLatch latch;
  // what the read bodies gave, records and hits numbered across bodies
  std::vector<int64_t> hit_off{0}, total, id_off{0}, text_off{0};
  std::vector<int32_t> status;
  std::vector<double> score, ranks;
  std::string id_bytes, text;
  long long n_exact = 0;
};

extern "C++" {
namespace cco {

static int sr_count_check(long long n, const char *what) {
  if (n >= (1LL << 31)) return set_error(CCO_E_UNSUPPORTED, "%lld %s in one body: at most 2^31 - 1", n, what);
  return CCO_OK;
}
// the exact path: strtod (correctly rounded; an underflow is a zero, not an error) and std::to_chars' digits, the
// shortest that give the same double back and of those the nearest to it (what Python's repr prints)
static int sr_exact_value(const char *t, long long n, SrNum *o) {
  std::string s(t, (size_t)n);
  const double v = strtod(s.c_str(), nullptr);
  if (std::isinf(v)) return 1;
  SrNum r = {v, 0ULL, 0, 0, s[0] == '-', 0};
  if (v != 0) {
    char buf[40];
    const std::to_chars_result tc = std::to_chars(buf, buf + sizeof buf - 1, std::fabs(v), std::chars_format::scientific);
    *tc.ptr = 0;
    const char *e = strchr(buf, 'e');
    unsigned long long dig = 0;
    int nd = 0;
    for (const char *q = buf; q < e; ++q)
      if (*q != '.') {
        dig = dig * 10 + (unsigned)(*q - '0');
        ++nd;
      }
    int e10 = atoi(e + 1) - (nd - 1);
    while (dig % 10 == 0) {
      dig /= 10;
      ++e10;
      --nd;
    }
    r.dig = dig;
    r.e10 = e10;
    r.nd = nd;
  }
  *o = r;
  return 0;
}
// the exact path's spans [b, e) of text converted into val -> the first entry out of the range of a double, or -1
static long long sr_exact_values(const char *text, const std::vector<SrExact> &xs, std::vector<SrNum> &val) {
  val.resize(xs.size());
  for (size_t i = 0; i < xs.size(); ++i)
    if (sr_exact_value(text + xs[i].b, xs[i].e - xs[i].b, &val[i])) return (long long)i;
  return -1;
}
template <typename T>
static void sr_append(std::vector<T> &dst, const T *src, long long n, T delta = T()) {
  const size_t at = dst.size();
  dst.resize(at + (size_t)n);
  for (long long i = 0; i < n; ++i) dst[at + i] = src[i] + delta;
}
// the compaction of the index entries with lo_dep <= dep <= hi_dep strictly between entries lo and hi
static int sr_select(cco_ctx *c, Arena &ar, long long m, const unsigned char *dep, int lo_dep, int hi_dep, long long lo, long long hi,
                     long long **out, long long *n) {
  cudaStream_t s = c->stream;
  long long *flag, *off;
  CKR(ar.alloc(&flag, m + 1));
  CKR(ar.alloc(&off, m + 1));
  CK(cudaMemsetAsync(flag + m, 0, 8, s));
  if (m > 0) k_sr_flag<<<grid_for(m, 256, c->sm_count), 256, 0, s>>>(m, dep, lo_dep, hi_dep, lo, hi, flag);
  CKR(exclusive_sum(c, ar, flag, off, m + 1));
  CKR(mail_fetch(c, n, off + m, 8));
  CKR(mail_wait(c));
  CKR(ar.alloc(out, *n + 1));
  if (m > 0) k_sr_compact<<<grid_for(m, 256, c->sm_count), 256, 0, s>>>(m, flag, off, *out);
  c->launches += 2;
  ar.release(flag);
  ar.release(off);
  return CCO_OK;
}

// Read the pending body (device slot h->n_bodies - 1 & 1): its records go after the ones read so far.
static int sr_read(cco_search_results *h) {
  cco_ctx *c = h->ctx;
  cudaStream_t s = c->stream;
  const int slot = (int)((h->n_bodies - 1) & 1);
  const long long len = h->p_len, body_no = h->n_bodies - 1, rec_base = (long long)h->status.size(),
                  hit_base = h->hit_off.back();
  const unsigned char *body = h->stage.dev[slot];
  const char *hbody = h->stage.host(slot);
  CKR(h->stage.wait(s, slot));
  mail_reset(c);   // every fetch below is waited for before the next body
  Arena ar(s);
  NvtxRange nvtx("cco:search_results");
  auto byte_error = [&](unsigned long long e) {
    return set_error(CCO_E_INVALID_ARG, "response body %lld, byte %lld: %s", body_no, (long long)(e >> 8), sr_message((int)(e & 0xff)));
  };
  SrIndex ix;
  unsigned long long e0 = ~0ULL;
  CKR(sr_index(c, ar, body, len, kSrMaxDepth, &ix, &e0));
  if (e0 != ~0ULL) return byte_error(e0);
  const long long m = ix.m, *pos = ix.pos;
  const unsigned char *dep = ix.dep;
  unsigned long long *err;
  CKR(ar.alloc(&err, 4));
  CK(cudaMemsetAsync(err, 0xff, 32, s));
  // the top level and the responses array
  long long *top, nt = 0, ends[2] = {-1, -1}, *d_ends;
  CKR(sr_select(c, ar, m, dep, 0, 1, -1, m, &top, &nt));
  CKR(ar.alloc(&d_ends, 2));
  k_sr_top<<<1, 32, 0, s>>>(SrIdx{pos, dep, body, top}, nt, len, d_ends, err);
  c->launches++;
  CKR(mail_fetch(c, &e0, err, 8));
  CKR(mail_fetch(c, ends, d_ends, 16));
  CKR(mail_wait(c));
  if (e0 != ~0ULL) return byte_error(e0);
  // one record per element
  long long *el, n2 = 0;
  CKR(sr_select(c, ar, m, dep, 2, 2, ends[0], ends[1], &el, &n2));
  long long *eflag, *erank, n_rec = 0;
  CKR(ar.alloc(&eflag, n2 + 1));
  CKR(ar.alloc(&erank, n2 + 1));
  CK(cudaMemsetAsync(eflag + n2, 0, 8, s));
  k_sr_elems<<<grid_for(n2 + 1, 256, c->sm_count), 256, 0, s>>>(SrIdx{pos, dep, body, el}, n2, ends[0], ends[1], eflag, err);
  c->launches++;
  CKR(exclusive_sum(c, ar, eflag, erank, n2 + 1));
  CKR(mail_fetch(c, &e0, err, 8));
  CKR(mail_fetch(c, &n_rec, erank + n2, 8));
  CKR(mail_wait(c));
  if (e0 != ~0ULL) return byte_error(e0);
  CKR(sr_count_check(n_rec, "records"));
  if (h->p_rec >= 0 && n_rec != h->p_rec)
    return set_error(CCO_E_INVALID_ARG, "response body %lld: %lld response elements for %lld records", body_no, n_rec, h->p_rec);
  if (h->p_rec < 0) h->p_ranks.assign((size_t)n_rec, (h->flags & CCO_SR_WITH_RANKS) ? 1 : 0);
  // the query lines: checked, their withRanks read, numbers beyond the fast path converted here
  SrLines q = {nullptr, nullptr, nullptr, nullptr, 0};
  uint8_t *wr;
  CKR(ar.alloc(&wr, n_rec + 1));
  if (h->p_has_lines) {
    const long long lb = (long long)h->p_lines.size(), cap = lb / 2 + 1;
    unsigned char *d_lines;
    long long *d_loff;
    SrExact *lx;
    CKR(ar.alloc(&d_lines, lb + 1));
    CKR(ar.alloc(&d_loff, n_rec + 1));
    CKR(ar.alloc(&lx, cap));
    if (lb > 0) CK(cudaMemcpyAsync(d_lines, h->p_lines.data(), (size_t)lb, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_loff, h->p_loff.data(), 8 * ((size_t)n_rec + 1), cudaMemcpyHostToDevice, s));
    CK(cudaMemsetAsync(err + 3, 0, 8, s));
    q.bytes = d_lines;
    q.off = d_loff;
    if (n_rec > 0) {
      k_sr_lines<<<grid_for(n_rec, 128, c->sm_count), 128, 0, s>>>(n_rec, q, wr, lx, err + 3, err + 2);
      c->launches++;
    }
    unsigned long long e2 = ~0ULL, nx = 0;
    CKR(mail_fetch(c, &e2, err + 2, 8));
    CKR(mail_fetch(c, &nx, err + 3, 8));
    CKR(mail_wait(c));
    if (e2 != ~0ULL)
      return set_error(CCO_E_INVALID_ARG, "record %lld: %s", rec_base + (long long)(e2 >> 8), sr_message((int)(e2 & 0xff)));
    if (nx > 0) {
      std::vector<SrExact> xs((size_t)nx);
      CK(cudaMemcpyAsync(xs.data(), lx, sizeof(SrExact) * (size_t)nx, cudaMemcpyDeviceToHost, s));
      CK(cudaStreamSynchronize(s));
      std::sort(xs.begin(), xs.end(), [](const SrExact &x, const SrExact &y) { return x.b < y.b; });
      std::vector<SrNum> xval;
      const long long bad = sr_exact_values(h->p_lines.data(), xs, xval);
      if (bad >= 0) {
        const SrExact &x = xs[(size_t)bad];
        const long long r = (long long)(std::upper_bound(h->p_loff.begin(), h->p_loff.end(), (int64_t)x.b) - h->p_loff.begin()) - 1;
        return set_error(CCO_E_INVALID_ARG, "record %lld: the query line's %.*s is out of the range of a double", rec_base + r,
                         (int)std::min<long long>(x.e - x.b, 64), h->p_lines.data() + x.b);
      }
      std::vector<long long> xpos((size_t)nx);
      for (size_t i = 0; i < xs.size(); ++i) xpos[i] = xs[i].b;
      long long *d_xpos;
      SrNum *d_xval;
      CKR(ar.alloc(&d_xpos, (long long)nx));
      CKR(ar.alloc(&d_xval, (long long)nx));
      CK(cudaMemcpyAsync(d_xpos, xpos.data(), 8 * (size_t)nx, cudaMemcpyHostToDevice, s));
      CK(cudaMemcpyAsync(d_xval, xval.data(), sizeof(SrNum) * (size_t)nx, cudaMemcpyHostToDevice, s));
      CK(cudaStreamSynchronize(s));   // the host vectors go out of scope
      q.xpos = d_xpos;
      q.xval = d_xval;
      q.nx = (long long)nx;
      h->n_exact += (long long)nx;
    }
  } else if (n_rec > 0) {
    CK(cudaMemcpyAsync(wr, h->p_ranks.data(), (size_t)n_rec, cudaMemcpyHostToDevice, s));
  }
  SrArgs a;
  memset(&a, 0, sizeof a);
  a.x = SrIdx{pos, dep, body, nullptr};
  a.n_rec = n_rec;
  a.n_rank = h->n_rank;
  memcpy(a.name_off, h->name_off, sizeof a.name_off);
  long long *ropen, *rclose, *nh, *hoff;
  int32_t *st;
  long long *tot;
  unsigned char *names;
  CKR(ar.alloc(&ropen, n_rec + 1));
  CKR(ar.alloc(&rclose, n_rec + 1));
  CKR(ar.alloc(&nh, n_rec + 1));
  CKR(ar.alloc(&hoff, n_rec + 1));
  CKR(ar.alloc(&st, n_rec + 1));
  CKR(ar.alloc(&tot, n_rec + 1));
  CKR(ar.alloc(&names, h->names.size() + 1));
  if (!h->names.empty()) CK(cudaMemcpyAsync(names, h->names.data(), h->names.size(), cudaMemcpyHostToDevice, s));
  a.ropen = ropen;
  a.rclose = rclose;
  a.with_ranks = wr;
  a.names = names;
  CK(cudaMemsetAsync(nh + n_rec, 0, 8, s));
  if (n2 > 0) k_sr_records<<<grid_for(n2, 256, c->sm_count), 256, 0, s>>>(n2, el, eflag, erank, ropen, rclose);
  const int rgrid = grid_for(n_rec * 32, 256, c->sm_count);
  if (n_rec > 0) k_sr_resp<false><<<rgrid, 256, 0, s>>>(a, st, tot, nh, nullptr, nullptr, nullptr, nullptr, err + 1);
  c->launches += 2;
  CKR(exclusive_sum(c, ar, nh, hoff, n_rec + 1));
  long long n_hits = 0;
  unsigned long long e1 = ~0ULL;
  CKR(mail_fetch(c, &e1, err + 1, 8));
  CKR(mail_fetch(c, &n_hits, hoff + n_rec, 8));
  CKR(mail_wait(c));
  if (e1 != ~0ULL)
    return set_error(CCO_E_INVALID_ARG, "record %lld: %s", rec_base + (long long)(e1 >> 8), sr_message((int)(e1 & 0xff)));
  CKR(sr_count_check(n_hits, "hits"));
  long long *hopen, *hclose;
  int32_t *hrec;
  JMember *idm;
  SrNum *sc, *rk;
  uint8_t *hr;
  SrExact *xl;
  const long long n_slots = n_hits * (1 + h->n_rank);
  CKR(ar.alloc(&hopen, n_hits + 1));
  CKR(ar.alloc(&hclose, n_hits + 1));
  CKR(ar.alloc(&hrec, n_hits + 1));
  CKR(ar.alloc(&idm, n_hits + 1));
  CKR(ar.alloc(&sc, n_hits + 1));
  CKR(ar.alloc(&rk, n_hits * h->n_rank + 1));
  CKR(ar.alloc(&hr, n_hits + 1));
  CKR(ar.alloc(&xl, n_slots + 1));
  CK(cudaMemsetAsync(err + 3, 0, 8, s));   // the exact-path count
  if (n_rec > 0 && n_hits > 0) {
    k_sr_resp<true><<<rgrid, 256, 0, s>>>(a, nullptr, nullptr, nullptr, hoff, hopen, hclose, hrec, err + 1);
    k_sr_hit<<<grid_for(n_hits * 32, 256, c->sm_count), 256, 0, s>>>(a, n_hits, hopen, hclose, hrec, idm, sc, rk, hr, xl, err + 3, err + 2);
    c->launches += 2;
  }
  unsigned long long e2 = ~0ULL, nx = 0;
  CKR(mail_fetch(c, &e2, err + 2, 8));
  CKR(mail_fetch(c, &nx, err + 3, 8));
  CKR(mail_wait(c));
  std::vector<int64_t> hh((size_t)n_rec + 1);
  CK(cudaMemcpyAsync(hh.data(), hoff, 8 * ((size_t)n_rec + 1), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  auto hit_where = [&](long long hit, char *buf, size_t n) {
    const long long r = (long long)(std::upper_bound(hh.begin(), hh.end(), (int64_t)hit) - hh.begin()) - 1;
    snprintf(buf, n, "record %lld hit %lld", rec_base + r, hit - hh[(size_t)r]);
  };
  char where[96];
  if (e2 != ~0ULL) {
    hit_where((long long)(e2 >> 8), where, sizeof where);
    return set_error(CCO_E_INVALID_ARG, "%s: %s", where, sr_message((int)(e2 & 0xff)));
  }
  // numbers beyond the fast path, on the host
  if (nx > 0) {
    std::vector<SrExact> xs((size_t)nx);
    CK(cudaMemcpyAsync(xs.data(), xl, sizeof(SrExact) * (size_t)nx, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    std::vector<SrNum> val;
    const long long bad = sr_exact_values(hbody, xs, val);
    if (bad >= 0) {
      const SrExact &x = xs[(size_t)bad];
      hit_where(x.slot < n_hits ? x.slot : (x.slot - n_hits) / std::max(h->n_rank, 1), where, sizeof where);
      return set_error(CCO_E_INVALID_ARG, "%s: %.*s is out of the range of a double", where, (int)std::min<long long>(x.e - x.b, 64), hbody + x.b);
    }
    std::vector<long long> slot_h((size_t)nx);
    for (size_t i = 0; i < xs.size(); ++i) slot_h[i] = xs[i].slot;
    long long *d_slot;
    SrNum *d_val;
    CKR(ar.alloc(&d_slot, (long long)nx));
    CKR(ar.alloc(&d_val, (long long)nx));
    CK(cudaMemcpyAsync(d_slot, slot_h.data(), 8 * (size_t)nx, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_val, val.data(), sizeof(SrNum) * (size_t)nx, cudaMemcpyHostToDevice, s));
    k_sr_exact_put<<<grid_for((long long)nx, 256, c->sm_count), 256, 0, s>>>((long long)nx, d_slot, d_val, n_hits, sc, rk);
    c->launches++;
    CK(cudaStreamSynchronize(s));   // the host vectors go out of scope
    h->n_exact += (long long)nx;
  }
  // the ids decoded, the value columns
  DevStrCol ids;
  long long id_total = 0;
  CKR(json_decode(c, ar, n_hits, idm, body, &ids, &id_total));
  double *sv, *rv;
  CKR(ar.alloc(&sv, n_hits + 1));
  CKR(ar.alloc(&rv, n_hits * h->n_rank + 1));
  if (n_hits > 0) {
    k_sr_values<<<grid_for(n_hits, 256, c->sm_count), 256, 0, s>>>(n_hits, h->n_rank, sc, rk, hr, sv, rv);
    c->launches++;
  }
  // the text
  long long text_total = 0, *rec_off = nullptr;
  unsigned char *d_text = nullptr;
  if (h->flags & CCO_SR_TEXT) {
    SrText t;
    memset(&t, 0, sizeof t);
    unsigned char *qn;
    CKR(ar.alloc(&qn, h->qnames.size() + 1));
    if (!h->qnames.empty()) CK(cudaMemcpyAsync(qn, h->qnames.data(), h->qnames.size(), cudaMemcpyHostToDevice, s));
    t.id_off = ids.off;
    t.id_bytes = (const unsigned char *)ids.w;
    t.score = sc;
    t.rank = rk;
    t.has_rank = hr;
    t.hrec = hrec;
    t.rec_hoff = hoff;
    t.n_rank = h->n_rank;
    t.qnames = qn;
    memcpy(t.qname_off, h->qname_off, sizeof t.qname_off);
    long long *tl, *toff;
    CKR(ar.alloc(&tl, n_hits + 1));
    CKR(ar.alloc(&toff, n_hits + 1));
    CKR(ar.alloc(&rec_off, n_rec + 1));
    CK(cudaMemsetAsync(tl + n_hits, 0, 8, s));
    const int hgrid = grid_for(n_hits, 256, c->sm_count), rg = grid_for(n_rec + 1, 256, c->sm_count);
    long long *eoff = nullptr;   // batchpredict lines: the echoes' offsets
    if (h->flags & CCO_SR_BATCHPREDICT) {
      long long *el;
      CKR(ar.alloc(&el, n_rec + 1));
      CKR(ar.alloc(&eoff, n_rec + 1));
      CK(cudaMemsetAsync(el + n_rec, 0, 8, s));
      if (n_rec > 0) k_sr_echo_len<<<grid_for(n_rec, 128, c->sm_count), 128, 0, s>>>(n_rec, q, el);
      CKR(exclusive_sum(c, ar, el, eoff, n_rec + 1));
      c->launches++;
    }
    if (n_hits > 0) k_sr_hit_text<false><<<hgrid, 256, 0, s>>>(t, eoff, n_hits, tl, nullptr, nullptr, nullptr);
    CKR(exclusive_sum(c, ar, tl, toff, n_hits + 1));
    k_sr_rec_text<false><<<rg, 256, 0, s>>>(n_rec, hoff, toff, eoff, q, rec_off, nullptr);
    CKR(mail_fetch(c, &text_total, rec_off + n_rec, 8));
    CKR(mail_wait(c));
    CKR(ar.alloc(&d_text, text_total + 1));
    if (n_hits > 0) k_sr_hit_text<true><<<hgrid, 256, 0, s>>>(t, eoff, n_hits, nullptr, toff, rec_off, d_text);
    k_sr_rec_text<true><<<rg, 256, 0, s>>>(n_rec, hoff, toff, eoff, q, rec_off, d_text);
    c->launches += 4;
  }
  // to the host, after the records read so far
  std::vector<int64_t> idoff((size_t)n_hits + 1), toff_h((size_t)n_rec + 1), tot_h((size_t)n_rec);
  std::vector<int32_t> st_h((size_t)n_rec);
  const size_t at_id = h->id_bytes.size(), at_text = h->text.size(), at_sc = h->score.size(), at_rk = h->ranks.size();
  h->id_bytes.resize(at_id + (size_t)id_total);
  h->score.resize(at_sc + (size_t)n_hits);
  h->ranks.resize(at_rk + (size_t)(n_hits * h->n_rank));
  h->text.resize(at_text + (size_t)text_total);
  CK(cudaMemcpyAsync(idoff.data(), ids.off, 8 * ((size_t)n_hits + 1), cudaMemcpyDeviceToHost, s));
  if (id_total > 0) CK(cudaMemcpyAsync(&h->id_bytes[at_id], ids.w, (size_t)id_total, cudaMemcpyDeviceToHost, s));
  if (n_hits > 0) CK(cudaMemcpyAsync(&h->score[at_sc], sv, 8 * (size_t)n_hits, cudaMemcpyDeviceToHost, s));
  if (n_hits * h->n_rank > 0) CK(cudaMemcpyAsync(&h->ranks[at_rk], rv, 8 * (size_t)(n_hits * h->n_rank), cudaMemcpyDeviceToHost, s));
  if (n_rec > 0) {
    CK(cudaMemcpyAsync(st_h.data(), st, 4 * (size_t)n_rec, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(tot_h.data(), tot, 8 * (size_t)n_rec, cudaMemcpyDeviceToHost, s));
  }
  if (rec_off) {
    CK(cudaMemcpyAsync(toff_h.data(), rec_off, 8 * ((size_t)n_rec + 1), cudaMemcpyDeviceToHost, s));
    if (text_total > 0) CK(cudaMemcpyAsync(&h->text[at_text], d_text, (size_t)text_total, cudaMemcpyDeviceToHost, s));
  }
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  sr_append(h->hit_off, hh.data() + 1, n_rec, (int64_t)hit_base);
  sr_append(h->status, st_h.data(), n_rec);
  sr_append(h->total, tot_h.data(), n_rec);
  sr_append(h->id_off, idoff.data() + 1, n_hits, (int64_t)at_id);
  if (rec_off) sr_append(h->text_off, toff_h.data() + 1, n_rec, (int64_t)at_text);
  return CCO_OK;
}

}  // namespace cco
}  // extern "C++"

int cco_search_results_begin(cco_ctx_t *ctx, const cco_search_results_params_t *params, cco_search_results_t **out) {
  if (!ctx || !params || !out || (params->n_rankings > 0 && !params->ranking_names)) return set_error(CCO_E_INVALID_ARG, "null argument");
  if (!ctx->members.empty()) return set_error(CCO_E_UNSUPPORTED, "per-GPU contexts only");
  if (params->n_rankings < 0 || params->n_rankings > CCO_MAX_RANKINGS)
    return set_error(CCO_E_INVALID_ARG, "%d rankings: 0 .. %d", params->n_rankings, CCO_MAX_RANKINGS);
  if (params->flags & ~(uint32_t)(CCO_SR_WITH_RANKS | CCO_SR_TEXT | CCO_SR_BATCHPREDICT))
    return set_error(CCO_E_INVALID_ARG, "unknown flags %#x", params->flags);
  *out = nullptr;
  CK(cudaSetDevice(ctx->device));
  cco_search_results *h = new cco_search_results();
  h->ctx = ctx;
  h->flags = params->flags;
  for (int k = 0; k < params->n_rankings; ++k) {
    const char *nm = params->ranking_names[k];
    if (!nm) {
      delete h;
      return set_error(CCO_E_INVALID_ARG, "null ranking name");
    }
    bool repeat = false;   // a name listed twice is one member, at its first place
    for (int j = 0; j < k; ++j) repeat = repeat || !strcmp(nm, params->ranking_names[j]);
    if (repeat) continue;
    const int at = h->n_rank++;
    h->names += nm;
    h->name_off[at + 1] = (int)h->names.size();
    std::string q(strlen(nm) * 6 + 3, '\0');   // json4s' quote of the name, then ':'
    q[0] = '"';
    const long long n = uq_escape((const unsigned char *)nm, (long long)strlen(nm), (unsigned char *)&q[1]);
    q.resize((size_t)n + 1);
    q += "\":";
    h->qnames += q;
    h->qname_off[at + 1] = (int)h->qnames.size();
  }
  if (h->stage.init() != CCO_OK) {
    cco_search_results_free(h);
    return set_error(CCO_E_CUDA, "cudaEventCreate failed");
  }
  *out = h;
  return CCO_OK;
}

int cco_search_results_append(cco_search_results_t *h, const char *body, int64_t len, int64_t n_records, const int64_t *line_offsets,
                              const char *line_bytes, const uint8_t *with_ranks) {
  if (!h || len < 0 || (len > 0 && !body) || (with_ranks && n_records < 0)) return set_error(CCO_E_INVALID_ARG, "null argument or negative length");
  CKR(h->latch.state("the results are finished"));
  if (n_records >= (1LL << 31)) return h->latch.fail(set_error(CCO_E_UNSUPPORTED, "%lld records in one body: at most 2^31 - 1", (long long)n_records));
  if (line_offsets && (n_records < 0 || with_ranks)) return set_error(CCO_E_INVALID_ARG, "query lines need n_records >= 0 and no with_ranks bitmap");
  if ((h->flags & CCO_SR_BATCHPREDICT) && !line_offsets) return set_error(CCO_E_INVALID_ARG, "batchpredict lines need the query lines");
  if (line_offsets) {
    for (long long r = 0; r < n_records; ++r)
      if (line_offsets[r + 1] < line_offsets[r]) return set_error(CCO_E_INVALID_ARG, "query line %lld: decreasing offsets", r);
    if (line_offsets[n_records] > line_offsets[0] && !line_bytes) return set_error(CCO_E_INVALID_ARG, "null line bytes");
  }
  cco_ctx *c = h->ctx;
  CK(cudaSetDevice(c->device));
  // this slot last held the body before the previous one, which has been read
  char what[64], copy_of[48];
  snprintf(what, sizeof what, "a response body of %lld bytes", (long long)len);
  snprintf(copy_of, sizeof copy_of, "response body %lld", h->n_bodies);
  int st = h->stage.put(c, (int)(h->n_bodies & 1), body, len, what, copy_of);
  // the previous body is read while this one is copied
  if (st == CCO_OK && h->pending) st = sr_read(h);
  if (st != CCO_OK) return h->latch.fail(st);
  ++h->n_bodies;
  h->pending = true;
  h->p_len = len;
  h->p_rec = n_records;
  h->p_ranks.clear();
  h->p_has_lines = line_offsets != nullptr;
  h->p_loff.clear();
  h->p_lines.clear();
  if (line_offsets) {
    h->p_loff.resize((size_t)n_records + 1);
    for (long long r = 0; r <= n_records; ++r) h->p_loff[(size_t)r] = line_offsets[r] - line_offsets[0];
    h->p_lines.assign(line_bytes ? line_bytes + line_offsets[0] : "", (size_t)(line_offsets[n_records] - line_offsets[0]));
  } else if (n_records >= 0) {
    h->p_ranks.resize((size_t)n_records);
    for (long long r = 0; r < n_records; ++r)
      h->p_ranks[(size_t)r] = with_ranks ? (with_ranks[r >> 3] >> (r & 7)) & 1 : ((h->flags & CCO_SR_WITH_RANKS) ? 1 : 0);
  }
  return CCO_OK;
}

int cco_search_results_finish(cco_search_results_t *h, cco_search_results_out_t *out) {
  if (!h || !out) return set_error(CCO_E_INVALID_ARG, "null argument");
  CKR(h->latch.state("the results are finished"));
  cco_ctx *c = h->ctx;
  CK(cudaSetDevice(c->device));
  if (h->pending) {
    const int st = sr_read(h);
    if (st != CCO_OK) return h->latch.fail(st);
    h->pending = false;
  }
  h->latch.finished = true;
  memset(out, 0, sizeof *out);
  const long long R = (long long)h->status.size(), H = h->hit_off.back();
  std::vector<void *> got;   // handed back to the pool when a later one fails
  auto give = [&](void **dst, const void *src, size_t n) {
    if (pinned_give(c, dst, src, n) != CCO_OK) return false;
    got.push_back(*dst);
    return true;
  };
  bool ok = give((void **)&out->hit_offsets, h->hit_off.data(), 8 * (size_t)(R + 1)) && give((void **)&out->status, h->status.data(), 4 * (size_t)R) &&
            give((void **)&out->total, h->total.data(), 8 * (size_t)R) && give((void **)&out->id_offsets, h->id_off.data(), 8 * (size_t)(H + 1)) &&
            give((void **)&out->id_bytes, h->id_bytes.data(), h->id_bytes.size()) && give((void **)&out->score, h->score.data(), 8 * (size_t)H) &&
            give((void **)&out->ranks, h->ranks.data(), 8 * h->ranks.size());
  if (ok && (h->flags & CCO_SR_TEXT))
    ok = give((void **)&out->text_offsets, h->text_off.data(), 8 * (size_t)(R + 1)) && give((void **)&out->text, h->text.data(), h->text.size());
  if (!ok) {
    for (void *p : got) c->pinned_put(p);
    memset(out, 0, sizeof *out);
    return set_error(CCO_E_OOM, "pinned host allocation failed");
  }
  out->n_records = R;
  out->n_hits = H;
  out->n_rankings = h->n_rank;
  out->n_exact = h->n_exact;
  return CCO_OK;
}

int cco_search_results_free(cco_search_results_t *h) {
  if (!h) return CCO_OK;
  cudaSetDevice(h->ctx->device);
  h->stage.release(h->ctx);
  delete h;
  return CCO_OK;
}

// ---- cco_index_pages: _search / _search/scroll response pages -> the model index's bulk body, kernels in
// cco_index_pages.cuh ----------------------------------------------------------------------------------------------------
struct cco_index_pages {
  cco_ctx *ctx = nullptr;
  BodyStage stage;                     // the last two pages
  long long n_pages = 0;
  // the pending page (the last appended): its hits are known, its documents are written by the next append or by finish
  bool pending = false;
  Arena *p_ar = nullptr;               // its index and hit brackets
  long long p_len = 0, p_hits = 0;
  const long long *p_pos = nullptr, *p_hopen = nullptr, *p_hclose = nullptr;
  const unsigned char *p_dep = nullptr;
  std::string scroll_id;               // the last page's, decoded
  long long total = -1, n_docs = 0;
  char *out = nullptr;                 // the documents so far (the context's pinned memory, handed to the caller by finish)
  size_t out_cap = 0, out_len = 0;
  ReaderLatch latch;
};

extern "C++" {
namespace cco {

// The new page (slot h->n_pages & 1, copied on the copy stream): its structural index down to the _source brackets and the
// top walk.  Leaves it pending with its hit count; *sid = its _scroll_id's raw inside (sid[0] < 0: absent).
static int ip_top(cco_index_pages *h, long long len, long long *n_hits, long long sid[2]) {
  cco_ctx *c = h->ctx;
  cudaStream_t s = c->stream;
  const int slot = (int)(h->n_pages & 1);
  const long long page_no = h->n_pages;
  const unsigned char *page = h->stage.dev[slot];
  CKR(h->stage.wait(s, slot));
  mail_reset(c);
  h->p_ar = new Arena(s);
  Arena &ar = *h->p_ar;
  NvtxRange nvtx("cco:index_pages");
  auto byte_error = [&](long long at, int code) {
    return set_error(CCO_E_INVALID_ARG, "page %lld, byte %lld: %s", page_no, at, sr_message(code));
  };
  SrIndex ix;
  unsigned long long e0 = ~0ULL;
  CKR(sr_index(c, ar, page, len, kIpMaxDepth, &ix, &e0));
  if (e0 != ~0ULL) return byte_error((long long)(e0 >> 8), (int)(e0 & 0xff));
  const long long m = ix.m, *pos = ix.pos;
  const unsigned char *dep = ix.dep;
  // the top walk over the entries down to the hits' brackets
  long long *top, nt = 0, *hopen, *hclose;
  CKR(sr_select(c, ar, m, dep, 0, kIpTopDepth, -1, m, &top, &nt));
  CKR(ar.alloc(&hopen, nt / 2 + 1));
  CKR(ar.alloc(&hclose, nt / 2 + 1));
  IpTop *d_top, r;
  CKR(ar.alloc(&d_top, 1));
  k_ip_top<<<1, 32, 0, s>>>(SrIdx{pos, dep, page, top}, nt, len, d_top, hopen, hclose);
  c->launches++;
  CKR(mail_fetch(c, &r, d_top, sizeof r));
  CKR(mail_wait(c));
  ar.release(top);
  if (r.code == kSrNotObject || r.code == kIpTimedOut || r.code == kIpShards || r.code == kIpHitsNotArray)
    return set_error(CCO_E_INVALID_ARG, "page %lld: %s", page_no, sr_message(r.code));
  if (r.code == kSrEsError) {
    if (r.has_status) return set_error(CCO_E_INVALID_ARG, "page %lld: %s (status %lld)", page_no, sr_message(r.code), r.status);
    return set_error(CCO_E_INVALID_ARG, "page %lld: %s", page_no, sr_message(r.code));
  }
  if (r.code) return byte_error(r.bad, r.code);
  if (r.n_hits >= (1LL << 31)) return set_error(CCO_E_UNSUPPORTED, "page %lld: %lld hits in one page: at most 2^31 - 1", page_no, r.n_hits);
  if (page_no == 0) h->total = r.total;
  h->p_len = len;
  h->p_hits = r.n_hits;
  h->p_pos = pos;
  h->p_dep = dep;
  h->p_hopen = hopen;
  h->p_hclose = hclose;
  h->pending = true;
  *n_hits = r.n_hits;
  sid[0] = r.sid_b;
  sid[1] = r.sid_e;
  return CCO_OK;
}

// The pending page's documents: each hit's _id and _source, the documents written on the device and appended to h->out.
static int ip_docs(cco_index_pages *h) {
  cco_ctx *c = h->ctx;
  cudaStream_t s = c->stream;
  const long long page_no = h->n_pages - 1, n = h->p_hits;
  const unsigned char *page = h->stage.dev[page_no & 1];
  h->pending = false;
  Arena &ar = *h->p_ar;
  mail_reset(c);
  NvtxRange nvtx("cco:index_pages");
  if (n > 0) {
    unsigned long long *err;
    CKR(ar.alloc(&err, 4));
    CK(cudaMemsetAsync(err, 0xff, 24, s));
    CK(cudaMemsetAsync(err + 3, 0, 8, s));
    JMember *idm;
    long long *sb, *se;
    CKR(ar.alloc(&idm, n));
    CKR(ar.alloc(&sb, n));
    CKR(ar.alloc(&se, n));
    k_ip_hit<<<grid_for(n * 32, 256, c->sm_count), 256, 0, s>>>(SrIdx{h->p_pos, h->p_dep, page, nullptr}, n, h->p_hopen, h->p_hclose, idm, sb, se,
                                                                err, err + 1);
    c->launches++;
    unsigned long long e_hit = ~0ULL, e_byte = ~0ULL;
    CKR(mail_fetch(c, &e_hit, err, 8));
    CKR(mail_fetch(c, &e_byte, err + 1, 8));
    DevStrCol ids;
    long long id_total = 0;
    CKR(json_decode(c, ar, n, idm, page, &ids, &id_total));   // waits for the fetches above
    if (e_byte != ~0ULL)
      return set_error(CCO_E_INVALID_ARG, "page %lld, byte %lld: %s", page_no, (long long)(e_byte >> 8), sr_message((int)(e_byte & 0xff)));
    if (e_hit != ~0ULL) return set_error(CCO_E_INVALID_ARG, "page %lld, hit %lld: %s", page_no, (long long)(e_hit >> 8), sr_message((int)(e_hit & 0xff)));
    IpDocs a = {page, sb, se, ids.off, (const unsigned char *)ids.w};
    long long *len, *off;
    CKR(ar.alloc(&len, n + 1));
    CKR(ar.alloc(&off, n + 1));
    CK(cudaMemsetAsync(len + n, 0, 8, s));
    const int grid = grid_for(n * 32, 256, c->sm_count);
    k_ip_doc<false><<<grid, 256, 0, s>>>(a, n, len, nullptr, nullptr, err + 2, err + 3);
    c->launches++;
    CKR(exclusive_sum(c, ar, len, off, n + 1));
    long long total = 0;
    unsigned long long e_str = ~0ULL, max_line = 0;
    CKR(mail_fetch(c, &total, off + n, 8));
    CKR(mail_fetch(c, &e_str, err + 2, 8));
    CKR(mail_fetch(c, &max_line, err + 3, 8));
    CKR(mail_wait(c));
    if (e_str != ~0ULL) {
      const long long at = (long long)(e_str >> 8);
      std::vector<long long> sb_h((size_t)n);
      CK(cudaMemcpyAsync(sb_h.data(), sb, 8 * (size_t)n, cudaMemcpyDeviceToHost, s));
      CK(cudaStreamSynchronize(s));
      const long long hit = (long long)(std::upper_bound(sb_h.begin(), sb_h.end(), at) - sb_h.begin()) - 1;
      return set_error(CCO_E_INVALID_ARG, "page %lld, hit %lld, byte %lld: a _source string holds a bad escape or a raw byte < 0x20", page_no,
                       hit, at);
    }
    if (max_line >= (1ULL << 31))
      return set_error(CCO_E_UNSUPPORTED, "page %lld: a document line of %llu bytes: at most 2^31 - 1", page_no, max_line);
    if (h->out_len + (size_t)total > h->out_cap) {   // from the context's pinned pool, so a later read reuses it
      const size_t cap = std::max<size_t>(h->out_cap * 2, std::max<size_t>(h->out_len + (size_t)total, 1u << 20));
      char *p = (char *)c->pinned_get(cap, /*for_result=*/false);
      if (!p) return set_error(CCO_E_OOM, "pinned host allocation of %zu bytes failed", cap);
      if (h->out_len) memcpy(p, h->out, h->out_len);
      if (h->out) c->pinned_put(h->out);
      h->out = p;
      h->out_cap = cap;
    }
    unsigned char *d_out;
    CKR(ar.alloc(&d_out, total + 1));
    k_ip_doc<true><<<grid, 256, 0, s>>>(a, n, nullptr, off, d_out, nullptr, nullptr);
    c->launches++;
    CK(cudaMemcpyAsync(h->out + h->out_len, d_out, (size_t)total, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    CK(cudaGetLastError());
    h->out_len += (size_t)total;
    h->n_docs += n;
  }
  delete h->p_ar;   // the page's index is freed in stream order
  h->p_ar = nullptr;
  return CCO_OK;
}
}  // namespace cco
}  // extern "C++"

int cco_index_pages_begin(cco_ctx_t *ctx, cco_index_pages_t **out) {
  if (!ctx || !out) return set_error(CCO_E_INVALID_ARG, "null argument");
  if (!ctx->members.empty()) return set_error(CCO_E_UNSUPPORTED, "per-GPU contexts only");
  *out = nullptr;
  CK(cudaSetDevice(ctx->device));
  cco_index_pages *h = new cco_index_pages();
  h->ctx = ctx;
  if (h->stage.init() != CCO_OK) {
    cco_index_pages_free(h);
    return set_error(CCO_E_CUDA, "cudaEventCreate failed");
  }
  *out = h;
  return CCO_OK;
}

int cco_index_pages_append(cco_index_pages_t *h, const char *page, int64_t len, int64_t *n_hits, const char **scroll_id,
                           int64_t *scroll_id_len) {
  if (!h || len < 0 || (len > 0 && !page) || !n_hits || !scroll_id || !scroll_id_len)
    return set_error(CCO_E_INVALID_ARG, "null argument or negative length");
  CKR(h->latch.state("the index pages are finished"));
  *n_hits = 0;
  *scroll_id = nullptr;
  *scroll_id_len = 0;
  cco_ctx *c = h->ctx;
  CK(cudaSetDevice(c->device));
  // this slot last held the page before the previous one, whose documents are written
  const int slot = (int)(h->n_pages & 1);
  char what[80], copy_of[48];
  snprintf(what, sizeof what, "page %lld of %lld bytes", h->n_pages, (long long)len);
  snprintf(copy_of, sizeof copy_of, "page %lld", h->n_pages);
  int st = h->stage.put(c, slot, page, len, what, copy_of);
  // the previous page's documents are written while this one is copied
  if (st == CCO_OK && h->pending) st = ip_docs(h);
  if (st != CCO_OK) return h->latch.fail(st);
  long long n = 0, sid[2] = {-1, -1};
  st = ip_top(h, len, &n, sid);
  ++h->n_pages;
  if (st != CCO_OK) return h->latch.fail(st);
  *n_hits = n;
  if (sid[0] >= 0) {
    h->scroll_id = sr_unescape(h->stage.host(slot) + sid[0], sid[1] - sid[0]);
    *scroll_id = h->scroll_id.data();
    *scroll_id_len = (int64_t)h->scroll_id.size();
  }
  return CCO_OK;
}

int cco_index_pages_finish(cco_index_pages_t *h, cco_index_pages_out_t *out) {
  if (!h || !out) return set_error(CCO_E_INVALID_ARG, "null argument");
  CKR(h->latch.state("the index pages are finished"));
  cco_ctx *c = h->ctx;
  CK(cudaSetDevice(c->device));
  if (h->pending) {
    const int st = ip_docs(h);
    if (st != CCO_OK) return h->latch.fail(st);
  }
  memset(out, 0, sizeof *out);
  if (!h->out) {   // an empty index: an empty body
    h->out = (char *)c->pinned_get(1, /*for_result=*/false);
    if (!h->out) return set_error(CCO_E_OOM, "pinned host allocation failed");
  }
  h->latch.finished = true;
  out->n_docs = h->n_docs;
  out->total = h->total;
  out->body = h->out;
  out->body_len = (int64_t)h->out_len;
  h->out = nullptr;
  h->out_cap = h->out_len = 0;
  return CCO_OK;
}

int cco_index_pages_free(cco_index_pages_t *h) {
  if (!h) return CCO_OK;
  cudaSetDevice(h->ctx->device);
  cudaStreamSynchronize(h->ctx->stream);
  delete h->p_ar;
  h->stage.release(h->ctx);
  if (h->out) h->ctx->pinned_put(h->out);
  delete h;
  return CCO_OK;
}

// ---- cco_index_write: the model index written into Elasticsearch (URModel.save, EsClient.hotSwap), kernels in
// cco_index_write.cuh ----------------------------------------------------------------------------------------------------
struct cco_index_write {
  cco_ctx *ctx = nullptr;
  Arena *ar = nullptr;                 // the body, its parse, the statuses and the retry lists, for the session
  BodyStage stage;                     // the response being read, in slot 0
  BulkDocs bd;
  int32_t *status = nullptr;           // [D] on the device: each document's latest status, 0 if never answered
  char *hbody = nullptr;               // the body in pinned memory: retry bodies are gathered from it
  long long len = 0, max_docs = 0, max_bytes = 0;
  std::vector<long long> doc_b;        // [D + 1]: the first byte of each document's action line, len at D
  struct Req {
    int round;                         // -1: the documents [b, e); else the positions [b, e) of retry round `round`
    long long b, e;
    bool answered;
  };
  std::vector<Req> reqs;
  long long n_first = 0;               // requests of the body itself
  std::vector<long long> first_db, first_bb;
  std::vector<std::vector<long long>> round_docs;   // the documents of each retry round, ascending
  std::vector<long long *> round_ddocs;             // their device copies
  std::unordered_map<long long, std::pair<std::string, std::string>> errors;   // each document's latest error.type, .reason
  ReaderLatch latch;
};

extern "C++" {
namespace cco {

// The greedy cut of documents of the given sizes into requests of at most max_docs documents and max_bytes bytes; a
// document larger than max_bytes is a request of its own.  db / bb: the requests' first document and byte, then the ends.
static void iw_cut(const std::vector<long long> &size, long long max_docs, long long max_bytes, std::vector<long long> &db,
                   std::vector<long long> &bb) {
  db.assign(1, 0);
  bb.assign(1, 0);
  long long n = 0, bytes = 0, at = 0;
  for (size_t k = 0; k < size.size(); ++k) {
    if (n > 0 && (n == max_docs || bytes + size[k] > max_bytes)) {
      db.push_back((long long)k);
      bb.push_back(at);
      n = 0;
      bytes = 0;
    }
    ++n;
    bytes += size[k];
    at += size[k];
  }
  if (n > 0) {
    db.push_back((long long)size.size());
    bb.push_back(at);
  }
}
// The body on the device: its documents checked as cco_rerank_model checks them (a repeated _id included), the documents'
// first bytes on the host, and the requests of the body itself.
static int iw_begin(cco_index_write *h, const char *body, long long len) {
  cco_ctx *c = h->ctx;
  cudaStream_t s = c->stream;
  h->ar = new Arena(s);
  Arena &ar = *h->ar;
  NvtxRange nvtx("cco:index_write");
  mail_reset(c);
  BulkDocs &bd = h->bd;
  CKR(bulk_parse(c, ar, body, len, 0, "nothing", &bd));
  const long long D = bd.D;
  h->doc_b.assign((size_t)D + 1, len);
  CKR(ar.alloc(&h->status, std::max<long long>(D, 1)));
  CK(cudaMemsetAsync(h->status, 0, sizeof(int32_t) * (size_t)std::max<long long>(D, 1), s));
  if (D > 0) {
    str_hash(c, bd.ids, ~0ULL);
    int32_t *gid;
    CKR(ar.alloc(&gid, D));
    StrTable tb;
    CKR(str_group(c, ar, bd.ids, nullptr, false, 0, &tb, gid));
    CKR(iq_unique_ids(c, ar, D, gid, tb));
    str_table_release(ar, tb);
    ar.release(gid);
    CK(cudaMemcpy2DAsync(h->doc_b.data(), sizeof(long long), bd.line_b, 2 * sizeof(long long), sizeof(long long), (size_t)D,
                         cudaMemcpyDeviceToHost, s));
  }
  if (pinned_give(c, &h->hbody, body, (size_t)len) != CCO_OK) return set_error(CCO_E_OOM, "pinned host allocation of %lld bytes failed", len);
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  std::vector<long long> size((size_t)D);
  for (long long d = 0; d < D; ++d) size[d] = h->doc_b[d + 1] - h->doc_b[d];
  iw_cut(size, h->max_docs, h->max_bytes, h->first_db, h->first_bb);
  h->n_first = (long long)h->first_db.size() - 1;
  for (long long q = 0; q < h->n_first; ++q) h->reqs.push_back({-1, h->first_db[q], h->first_db[q + 1], false});
  return CCO_OK;
}

// esFields: the distinct decoded names of the document lines' members in first-appearance order, escaped; "id" last when
// no document line has it.
static int iw_fields(cco_index_write *h, int64_t *n_out, int64_t **name_offsets, char **name_bytes) {
  cco_ctx *c = h->ctx;
  cudaStream_t s = c->stream;
  Arena ar(s);
  NvtxRange nvtx("cco:index_write");
  mail_reset(c);
  const BulkDocs &bd = h->bd;
  const long long D = bd.D;
  long long ng = 0, total = 0;
  DevDict esc = {nullptr, nullptr, 0};
  if (D > 0 && bd.M1 > 0) {
    int32_t *gate, *gid;
    CKR(ar.alloc(&gate, bd.M1));
    CKR(ar.alloc(&gid, bd.M1));
    k_iw_gate<<<grid_for(2 * D, 256, c->sm_count), 256, 0, s>>>(2 * D, bd.line_moff, gate);
    c->launches++;
    str_hash(c, bd.names, ~0ULL);
    StrTable tb;
    CKR(str_group(c, ar, bd.names, gate, false, 0, &tb, gid));
    ng = tb.n_groups;
    long long *len, *off;
    CKR(ar.alloc(&len, ng + 1));
    CKR(ar.alloc(&off, ng + 1));
    CK(cudaMemsetAsync(len + ng, 0, 8, s));
    if (ng > 0) {
      k_str_dict_len<<<grid_for(ng, 256, c->sm_count), 256, 0, s>>>(ng, tb.first_sorted, bd.names.off, len);
      c->launches++;
    }
    CKR(exclusive_sum(c, ar, len, off, ng + 1));
    long long raw_total = 0;
    CKR(mail_fetch(c, &raw_total, off + ng, 8));
    CKR(mail_wait(c));
    unsigned char *raw;
    CKR(ar.alloc(&raw, std::max<long long>(raw_total, 1)));
    if (ng > 0 && raw_total > 0) {
      k_str_dict_gather<<<grid_for(ng, 256, c->sm_count), 256, 0, s>>>(ng, tb.first_sorted, bd.names.off, bd.names.base,
                                                                      (const unsigned char *)bd.names.w, off, raw);
      c->launches++;
    }
    CKR(escape_dict(c, ar, DevDict{off, raw, ng}, &esc));   // waits for its total
    CK(cudaMemcpyAsync(&total, esc.off + ng, 8, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
  }
  int64_t *ho;
  char *hb;
  CKR(pinned_give(c, &ho, nullptr, sizeof(int64_t) * ((size_t)ng + 2)));
  CKR(pinned_give(c, &hb, nullptr, (size_t)total + 2));
  ho[0] = 0;
  if (ng > 0) {
    CK(cudaMemcpyAsync(ho, esc.off, sizeof(int64_t) * ((size_t)ng + 1), cudaMemcpyDeviceToHost, s));
    if (total > 0) CK(cudaMemcpyAsync(hb, esc.bytes, (size_t)total, cudaMemcpyDeviceToHost, s));
  }
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  bool has_id = false;
  for (long long k = 0; k < ng && !has_id; ++k) has_id = ho[k + 1] - ho[k] == 2 && hb[ho[k]] == 'i' && hb[ho[k] + 1] == 'd';
  if (D > 0 && !has_id) {   // save adds "id" to every document (URModel.scala:73)
    hb[total] = 'i';
    hb[total + 1] = 'd';
    ho[++ng] = total + 2;
  }
  *n_out = ng;
  *name_offsets = ho;
  *name_bytes = hb;
  return CCO_OK;
}

// One _bulk response body for request q: its structural index, the top walk, one warp per item.
static int iw_response(cco_index_write *h, long long q, const char *resp, long long len) {
  cco_ctx *c = h->ctx;
  cudaStream_t s = c->stream;
  if (q < 0 || q >= (long long)h->reqs.size())
    return set_error(CCO_E_INVALID_ARG, "request %lld is out of range: there are %lld requests", q, (long long)h->reqs.size());
  cco_index_write::Req &rq = h->reqs[q];
  if (rq.answered) return set_error(CCO_E_INVALID_ARG, "request %lld is answered twice", q);
  const long long n_docs = rq.e - rq.b;
  char what[96], copy_of[48];
  snprintf(what, sizeof what, "request %lld: a response of %lld bytes", q, len);
  snprintf(copy_of, sizeof copy_of, "the response to request %lld", q);
  CKR(h->stage.put(c, 0, resp, len, what, copy_of));
  CKR(h->stage.wait(s, 0));
  const unsigned char *page = h->stage.dev[0];
  Arena ar(s);
  NvtxRange nvtx("cco:index_write");
  mail_reset(c);
  auto byte_error = [&](long long at, int code) {
    return set_error(CCO_E_INVALID_ARG, "request %lld, byte %lld: %s", q, at, sr_message(code));
  };
  // the structural index down to the members of an item's error
  SrIndex ix;
  unsigned long long e0 = ~0ULL;
  CKR(sr_index(c, ar, page, len, kIwMaxDepth, &ix, &e0));
  if (e0 != ~0ULL) return byte_error((long long)(e0 >> 8), (int)(e0 & 0xff));
  const long long m = ix.m, *pos = ix.pos;
  const unsigned char *dep = ix.dep;
  // the top walk over the entries down to the items' brackets
  long long *top, nt = 0, *iopen, *iclose;
  CKR(sr_select(c, ar, m, dep, 0, kIwTopDepth, -1, m, &top, &nt));
  CKR(ar.alloc(&iopen, nt / 2 + 1));
  CKR(ar.alloc(&iclose, nt / 2 + 1));
  IwTop *d_top, r;
  CKR(ar.alloc(&d_top, 1));
  k_iw_top<<<1, 32, 0, s>>>(SrIdx{pos, dep, page, top}, nt, len, d_top, iopen, iclose);
  c->launches++;
  CKR(mail_fetch(c, &r, d_top, sizeof r));
  CKR(mail_wait(c));
  if (r.code == kSrNotObject || r.code == kIwNoItems) return set_error(CCO_E_INVALID_ARG, "request %lld: %s", q, sr_message(r.code));
  if (r.code == kSrEsError) {
    if (r.has_status) return set_error(CCO_E_INVALID_ARG, "request %lld: %s (status %lld)", q, sr_message(r.code), r.status);
    return set_error(CCO_E_INVALID_ARG, "request %lld: %s", q, sr_message(r.code));
  }
  if (r.code) return byte_error(r.bad, r.code);
  if (r.n_items != n_docs)
    return set_error(CCO_E_INVALID_ARG, "request %lld: %lld items for %lld documents", q, r.n_items, n_docs);
  if (n_docs > 0) {
    const long long *ddocs = rq.round < 0 ? nullptr : h->round_ddocs[rq.round] + rq.b;
    const IwItems it = {ddocs, rq.round < 0 ? rq.b : 0, h->bd.ids.off, (const unsigned char *)h->bd.ids.w};
    unsigned long long *err;
    IwFail *fail;
    CKR(ar.alloc(&err, 4));
    CKR(ar.alloc(&fail, n_docs));
    CK(cudaMemsetAsync(err, 0xff, 24, s));
    CK(cudaMemsetAsync(err + 3, 0, 8, s));
    k_iw_item<<<grid_for(n_docs * 32, 256, c->sm_count), 256, 0, s>>>(SrIdx{pos, dep, page, nullptr}, n_docs, iopen, iclose, it, h->status, fail,
                                                                      err + 3, err + 1, err + 2);
    c->launches++;
    unsigned long long e_item = ~0ULL, e_byte = ~0ULL, nf = 0;
    CKR(mail_fetch(c, &e_item, err + 1, 8));
    CKR(mail_fetch(c, &e_byte, err + 2, 8));
    CKR(mail_fetch(c, &nf, err + 3, 8));
    CKR(mail_wait(c));
    if (e_byte != ~0ULL) return byte_error((long long)(e_byte >> 8), (int)(e_byte & 0xff));
    if (e_item != ~0ULL)
      return set_error(CCO_E_INVALID_ARG, "request %lld, item %lld: %s", q, (long long)(e_item >> 8), sr_message((int)(e_item & 0xff)));
    if (nf > 0) {   // failures are few: their error texts are decoded on the host, from the caller's response
      std::vector<IwFail> hf((size_t)nf);
      CK(cudaMemcpyAsync(hf.data(), fail, sizeof(IwFail) * (size_t)nf, cudaMemcpyDeviceToHost, s));
      CK(cudaStreamSynchronize(s));
      for (const IwFail &f : hf) {
        const long long doc = rq.round < 0 ? rq.b + f.item : h->round_docs[rq.round][rq.b + f.item];
        h->errors[doc] = {f.tb < 0 ? std::string() : sr_unescape(resp + f.tb, f.te - f.tb),
                          f.rb < 0 ? std::string() : sr_unescape(resp + f.rb, f.re - f.rb)};
      }
    }
  }
  CK(cudaGetLastError());
  rq.answered = true;
  return CCO_OK;
}

static int iw_statuses(cco_index_write *h, int32_t *out) {
  if (h->bd.D > 0) CK(cudaMemcpyAsync(out, h->status, sizeof(int32_t) * (size_t)h->bd.D, cudaMemcpyDeviceToHost, h->ctx->stream));
  CK(cudaStreamSynchronize(h->ctx->stream));
  return CCO_OK;
}

// The documents whose latest status is 429 as a new body, gathered from the pinned copy, and its requests.
static int iw_retry(cco_index_write *h, cco_index_write_retry_t *out) {
  cco_ctx *c = h->ctx;
  const long long D = h->bd.D;
  std::vector<int32_t> st((size_t)D);
  CKR(iw_statuses(h, st.data()));
  std::vector<long long> docs, size;
  for (long long d = 0; d < D; ++d)
    if (st[d] == 429) {
      docs.push_back(d);
      size.push_back(h->doc_b[d + 1] - h->doc_b[d]);
    }
  std::vector<long long> db, bb;
  iw_cut(size, h->max_docs, h->max_bytes, db, bb);
  char *body;
  CKR(pinned_give(c, &body, nullptr, (size_t)bb.back()));
  long long at = 0;
  for (size_t k = 0; k < docs.size(); ++k) {
    memcpy(body + at, h->hbody + h->doc_b[docs[k]], (size_t)size[k]);
    at += size[k];
  }
  long long *dd = nullptr;
  if (!docs.empty()) {
    CKR(h->ar->alloc(&dd, docs.size()));
    CK(cudaMemcpyAsync(dd, docs.data(), sizeof(long long) * docs.size(), cudaMemcpyHostToDevice, c->stream));
    CK(cudaStreamSynchronize(c->stream));
  }
  const int round = (int)h->round_docs.size();
  h->round_docs.push_back(docs);
  h->round_ddocs.push_back(dd);
  memset(out, 0, sizeof *out);
  out->first_request = (int64_t)h->reqs.size();
  for (size_t k = 0; k + 1 < db.size(); ++k) h->reqs.push_back({round, db[k], db[k + 1], false});
  out->n_docs = (int64_t)docs.size();
  out->body = body;
  out->body_len = at;
  out->n_requests = (int64_t)db.size() - 1;
  CKR(pinned_give(c, &out->doc, docs.data(), sizeof(int64_t) * docs.size()));
  CKR(pinned_give(c, &out->doc_begin, db.data(), sizeof(int64_t) * db.size()));
  CKR(pinned_give(c, &out->byte_begin, bb.data(), sizeof(int64_t) * bb.size()));
  return CCO_OK;
}

static int iw_finish(cco_index_write *h, cco_index_write_out_t *out) {
  cco_ctx *c = h->ctx;
  const long long D = h->bd.D;
  memset(out, 0, sizeof *out);
  int32_t *st;
  CKR(pinned_give(c, &st, nullptr, sizeof(int32_t) * (size_t)D));
  out->status = st;
  CKR(iw_statuses(h, st));
  std::vector<int64_t> edoc, toff{0}, roff{0};
  std::string tb, rb;
  for (long long d = 0; d < D; ++d) {
    if (st[d] >= 200 && st[d] < 300) {
      ++out->n_ok;
      continue;
    }
    ++(st[d] == 429 ? out->n_rejected : out->n_failed);
    edoc.push_back(d);
    auto e = h->errors.find(d);
    if (e != h->errors.end()) {
      tb += e->second.first;
      rb += e->second.second;
    }
    toff.push_back((int64_t)tb.size());
    roff.push_back((int64_t)rb.size());
  }
  out->n_docs = D;
  out->n_errors = (int64_t)edoc.size();
  CKR(pinned_give(c, &out->error_doc, edoc.data(), sizeof(int64_t) * edoc.size()));
  CKR(pinned_give(c, &out->type_offsets, toff.data(), sizeof(int64_t) * toff.size()));
  CKR(pinned_give(c, &out->reason_offsets, roff.data(), sizeof(int64_t) * roff.size()));
  CKR(pinned_give(c, &out->type_bytes, tb.data(), tb.size()));
  CKR(pinned_give(c, &out->reason_bytes, rb.data(), rb.size()));
  return CCO_OK;
}

}  // namespace cco
}  // extern "C++"

int cco_index_write_begin(cco_ctx_t *ctx, const char *body, int64_t len, const cco_index_write_params_t *params, cco_index_write_t **out) {
  if (!ctx || !out || !params || len < 0 || (len > 0 && !body)) return set_error(CCO_E_INVALID_ARG, "null argument or negative length");
  *out = nullptr;
  if (params->max_docs < 1 || params->max_bytes < 1)
    return set_error(CCO_E_INVALID_ARG, "max_docs = %lld and max_bytes = %lld: both must be at least 1", (long long)params->max_docs,
                     (long long)params->max_bytes);
  if (!ctx->members.empty()) return set_error(CCO_E_UNSUPPORTED, "per-GPU contexts only");
  if (len > 0 && body[len - 1] != '\n') return set_error(CCO_E_INVALID_ARG, "the body does not end in a newline");
  CK(cudaSetDevice(ctx->device));
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  if ((size_t)len > total_b / 4)
    return set_error(CCO_E_UNSUPPORTED, "a body of %lld bytes: at most a quarter of the device's memory", (long long)len);
  cco_index_write *h = new cco_index_write();
  h->ctx = ctx;
  h->len = len;
  h->max_docs = params->max_docs;
  h->max_bytes = params->max_bytes;
  int st = h->stage.init();
  if (st == CCO_OK) st = iw_begin(h, body, len);
  if (st != CCO_OK) {
    const std::string msg = cco_last_error();
    cco_index_write_free(h);
    return set_error(st, "%s", msg.c_str());
  }
  *out = h;
  return CCO_OK;
}

int cco_index_write_fields(cco_index_write_t *h, int64_t *n, int64_t **name_offsets, char **name_bytes) {
  if (!h || !n || !name_offsets || !name_bytes) return set_error(CCO_E_INVALID_ARG, "null argument");
  CKR(h->latch.state("the index write is finished"));
  CK(cudaSetDevice(h->ctx->device));
  const int st = iw_fields(h, n, name_offsets, name_bytes);
  return st == CCO_OK ? st : h->latch.fail(st);
}

int cco_index_write_requests(cco_index_write_t *h, int64_t *n_requests, int64_t **doc_begin, int64_t **byte_begin) {
  if (!h || !n_requests || !doc_begin || !byte_begin) return set_error(CCO_E_INVALID_ARG, "null argument");
  CKR(h->latch.state("the index write is finished"));
  int st = pinned_give(h->ctx, doc_begin, h->first_db.data(), sizeof(int64_t) * h->first_db.size());
  if (st == CCO_OK) st = pinned_give(h->ctx, byte_begin, h->first_bb.data(), sizeof(int64_t) * h->first_bb.size());
  if (st != CCO_OK) return h->latch.fail(st);
  *n_requests = h->n_first;
  return CCO_OK;
}

int cco_index_write_response(cco_index_write_t *h, int64_t request, const char *resp, int64_t len) {
  if (!h || len < 0 || (len > 0 && !resp)) return set_error(CCO_E_INVALID_ARG, "null argument or negative length");
  CKR(h->latch.state("the index write is finished"));
  CK(cudaSetDevice(h->ctx->device));
  const int st = iw_response(h, request, resp, len);
  return st == CCO_OK ? st : h->latch.fail(st);
}

int cco_index_write_retry(cco_index_write_t *h, cco_index_write_retry_t *out) {
  if (!h || !out) return set_error(CCO_E_INVALID_ARG, "null argument");
  CKR(h->latch.state("the index write is finished"));
  CK(cudaSetDevice(h->ctx->device));
  const int st = iw_retry(h, out);
  return st == CCO_OK ? st : h->latch.fail(st);
}

int cco_index_write_finish(cco_index_write_t *h, cco_index_write_out_t *out) {
  if (!h || !out) return set_error(CCO_E_INVALID_ARG, "null argument");
  CKR(h->latch.state("the index write is finished"));
  CK(cudaSetDevice(h->ctx->device));
  const int st = iw_finish(h, out);
  if (st != CCO_OK) return h->latch.fail(st);
  h->latch.finished = true;
  return CCO_OK;
}

int cco_index_write_free(cco_index_write_t *h) {
  if (!h) return CCO_OK;
  cudaSetDevice(h->ctx->device);
  cudaStreamSynchronize(h->ctx->stream);
  delete h->ar;
  cudaStreamSynchronize(h->ctx->stream);
  h->stage.release(h->ctx);
  if (h->hbody) h->ctx->pinned_put(h->hbody);
  delete h;
  return CCO_OK;
}


}  // extern "C"
