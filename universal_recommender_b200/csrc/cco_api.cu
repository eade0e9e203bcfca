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
#include <cmath>
#include <functional>
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
    *out = (T *)p;
    return CCO_OK;
  }
  void take(void *p) {   // the buffer outlives the arena: its new owner frees it (never slab memory)
    for (size_t i = 0; i < ptrs.size(); ++i)
      if (ptrs[i] == p) {
        ptrs.erase(ptrs.begin() + i);
        return;
      }
  }
  void release(void *p) {   // slab memory is simply not reused within a train
    for (size_t i = 0; i < ptrs.size(); ++i)
      if (ptrs[i] == p) {
        cudaFreeAsync(p, s);
        ptrs.erase(ptrs.begin() + i);
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
  // 2. bins -----------------------------------------------------------------------------------------
  const int k_eff = emit_all ? 1 : prm.top_k;
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
  std::vector<BinCfg> cfgs(kBins);
  for (int b = 0; b < kBins; ++b) cfgs[b] = make_cfg(c, spec[b].group, spec[b].slots, k_eff, n_cols_b);
  BinCfg &cfgL = cfgs[1];
  // packed word: key bits must leave room for the largest possible count
  int key_bits = 1;
  while (((1LL << key_bits) - 1) <= (long long)n_cols_b) ++key_bits;  // keys <= 2^kb - 2
  int count_bits = 32 - key_bits;
  // a co-occurrence count is bounded by both marginals: k11 <= min(rowA, colB) <= min(max rowA, max colB).  With the
  // reference's default downsampling (m = 500) that is ~560, i.e. 10 count bits next to 22 key bits (4M columns).
  const long long k11_max = std::min<long long>(max_marg_a, max_marg_b);
  if (count_bits < 1 || k11_max >= (1LL << count_bits))
    return set_error(CCO_E_UNSUPPORTED,
                     "co-occurrence counts up to %lld over %d columns do not fit the packed 32-bit accumulator word "
                     "(key %d bits + count %d bits): lower maxItemsPerUser/maxEventsPerEventType for this event type "
                     "(\"Limits\" in include/cco_b200.h)", k11_max, n_cols_b, key_bits, count_bits);
  // thresholds on w, descending: bin b takes rows with h_thr[b-1] >= w > h_thr[b]; a hashed table also needs w <= cap
  std::vector<uint32_t> h_thr(kBins);
  for (int b = 0; b < kBins; ++b) {
    const BinCfg &f = cfgs[std::min(b + 1, kBins - 1)];   // h_thr[b] = upper limit of bin b+1
    uint32_t lim = b + 1 < kBins ? spec[b + 1].max_w : 0u;
    if (b + 1 < kBins && !f.dense) lim = std::min<uint32_t>(lim, (uint32_t)f.cap);
    h_thr[b] = lim;
    if (b > 0) h_thr[b] = std::min(h_thr[b], h_thr[b - 1]);
  }
  // bitmap rows: the k11 = 1 cells are cut by key, so every row must be keyed (2 rowA colB < N for the largest of both)
  // and the cut exact
  const bool bitmap_ok = !emit_all && cut_exact(n_users, max_marg_a, max_marg_b) &&
                         2ull * (unsigned long long)std::max(max_marg_a, 0) * (unsigned long long)std::max(max_marg_b, 0) <
                             (unsigned long long)n_users;
  for (int b = 1; b < kBins && bitmap_ok; ++b) use_bitmap(cfgs[b], h_thr[b - 1], k_eff, n_cols_b);
  int32_t *d_bounds;
  CKR(ar.alloc(&d_bounds, kBins + 3));
  BinThresholds bt;
  memset(&bt, 0, sizeof bt);
  for (int b = 0; b < kBins; ++b) bt.t[b] = h_thr[b];
  k_bin_bounds<<<1, 32, 0, ss>>>(n_items_a, sorted_work, kBins, bt, d_bounds);
  c->launches++;
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
  a.key_shift = 0;
  while (((long long)std::max(n_cols_b - 1, 0) >> a.key_shift) >= kCutBins) ++a.key_shift;
  a.max_marg_b = max_marg_b;
  a.col_terms = col_terms;
  a.rows_sorted = rows_sorted;
  a.row_work = row_work;
  a.bin_bounds = d_bounds;
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
  if (ev_begin) CK(cudaEventRecord(ev_begin, s));
  if (n_items_a > 0) {
    // the bins touch disjoint rows: run them concurrently (tails of one bin overlap the bulk of another)
    CK(cudaEventRecord(c->bin_ev[8], s));
    for (int b = 0; b < kBins; ++b) {
      if (b == 0 && cfgL.dense) continue;                 // dense L takes every large row in bin 1
      RowArgs ab = a;
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
  } else {
    rm->row_begin = lo;
    rm->row_end = hi;
    rm->n_cols = st->n_cols_b;
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

// the user and item columns of type t in HBM: uploaded from the caller's arrays, or views of an event log's columns
using StrColumns = std::function<int(Arena &, int, DevStrCol *, DevStrCol *)>;

static int ingest_strings_core(cco_ctx *c, int32_t n_types, const StrColumns &columns, int32_t min_events_per_user, cco_dataset **out) {
  CK(cudaSetDevice(c->device));
  cudaStream_t s = c->stream;
  nvtx_push("cco:ingest_strings");
  struct Pop { ~Pop() { nvtx_pop(); } } pop;
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

// one section of the combined key column: the row dictionary, the property items or one ranking stream.  A device
// section (the decoded ids of an old index, cco_rerank_model) is already in HBM: offsets from 0, nbytes bytes.
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
  long long nb = 0;
  for (const KeySection &k : sec) nb += k.byte_count();
  DevStrCol key;
  key.n = N;
  key.base = 0;
  CKR(ar.alloc(&key.off, N + 1));
  CKR(ar.alloc(&key.w, (nb + 16 + 7) / 8));
  CKR(ar.alloc(&key.hash, std::max<long long>(N, 1)));
  CK(cudaMemsetAsync(key.off, 0, 8, s));
  int *bad;
  CKR(ar.alloc(&bad, 1));
  CK(cudaMemsetAsync(bad, 0, sizeof(int), s));
  long long *tmp_off;
  long long max_n = 0;
  for (const KeySection &k : sec) max_n = std::max(max_n, k.n);
  CKR(ar.alloc(&tmp_off, max_n + 1));
  // every section: raw offsets -> decreasing check -> rebased into the key column; bytes appended to the word buffer
  long long at = 0, byte_at = 0;
  for (const KeySection &k : sec) {
    if (k.n == 0) continue;
    const long long kb = k.byte_count();
    if (k.device) {
      k_rebase<<<grid_for(k.n + 1, 256, c->sm_count), 256, 0, s>>>(k.n + 1, (const long long *)k.off, byte_at - k.base, key.off + at);
      c->launches++;
      if (kb > 0) CK(cudaMemcpyAsync((char *)key.w + byte_at, k.bytes, (size_t)kb, cudaMemcpyDeviceToDevice, s));
      at += k.n;
      byte_at += kb;
      continue;
    }
    CK(cudaMemcpyAsync(tmp_off, k.off, sizeof(int64_t) * ((size_t)k.n + 1), cudaMemcpyHostToDevice, s));
    k_str_check<<<grid_for(k.n, 256, c->sm_count), 256, 0, s>>>(k.n, tmp_off, bad);
    k_rebase<<<grid_for(k.n + 1, 256, c->sm_count), 256, 0, s>>>(k.n + 1, tmp_off, byte_at - k.off[0], key.off + at);
    c->launches += 2;
    if (kb > 0) CK(cudaMemcpyAsync((char *)key.w + byte_at, k.bytes + k.off[0], (size_t)kb, cudaMemcpyHostToDevice, s));
    at += k.n;
    byte_at += kb;
  }
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
  ar.release(tmp_off);

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
  std::vector<const char *> all_names(names, names + n_ind);
  if (model) {
    for (int f = 0; f < n_fields; ++f) all_names.push_back(props->field_names[f]);
    for (int k = 0; k < n_rank; ++k) all_names.push_back(rk[k].name);
  }
  const int n_all = (int)all_names.size();
  std::vector<long long> eoff(n_all + 1);
  {
    std::vector<int64_t> noff(n_all + 1, 0);
    std::string blob;
    for (int i = 0; i < n_all; ++i) {
      blob += all_names[i];
      noff[i + 1] = (int64_t)blob.size();
    }
    cco_dictionary_t nd = {n_all, noff.data(), blob.data()};
    DevDict nraw, nesc;
    CKR(upload_dict(c, ar, nd, &nraw));
    CK(cudaStreamSynchronize(s));   // noff / blob are locals
    CKR(escape_dict(c, ar, nraw, &nesc));
    CK(cudaMemcpyAsync(eoff.data(), nesc.off, sizeof(long long) * ((size_t)n_all + 1), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    fa->names = nesc.bytes;
    for (int i = 0; i <= n_ind; ++i) fa->name_off[i] = (int32_t)eoff[i];
    if (model) {
      fa->field_off = nesc.off + n_ind;
      for (int k = 0; k <= n_rank; ++k) fa->rank_name_off[k] = (int32_t)eoff[n_ind + n_fields + k];
    }
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
  nvtx_push(range);
  struct Pop { ~Pop() { nvtx_pop(); } } pop;
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
  char *host = (char *)ctx->pinned_get((size_t)std::max<long long>(total, 1), /*for_result=*/false);
  if (!host) return set_error(CCO_E_OOM, "pinned host allocation failed");
  if (total > 0) CK(cudaMemcpyAsync(host, d_out, (size_t)total, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  *out_bytes = host;
  *out_len = total;
  return CCO_OK;
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
  nvtx_push("cco:rerank_model");
  struct Pop { ~Pop() { nvtx_pop(); } } pop;
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
  KeySection rows;
  rows.n = D;
  rows.off = (const int64_t *)ids.off;
  rows.bytes = (const char *)ids.w;
  rows.device = true;
  rows.nbytes = ids_bytes;
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
    std::vector<int64_t> toff(T + 1, 0);
    std::string tblob;
    for (int t = 0; t < T; ++t) {
      tblob += ent[t];
      toff[t + 1] = (int64_t)tblob.size();
    }
    const cco_dictionary_t td = {T, toff.data(), tblob.data()};
    DevDict traw;
    int32_t *d_field;
    uint8_t *d_rank, *d_id;
    CKR(upload_dict(c, ar, td, &traw));
    CKR(ar.alloc(&d_field, T));
    CKR(ar.alloc(&d_rank, T));
    CKR(ar.alloc(&d_id, T));
    CK(cudaMemcpyAsync(d_field, ent_field.data(), sizeof(int32_t) * T, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_rank, ent_rank.data(), T, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_id, ent_id.data(), T, cudaMemcpyHostToDevice, s));
    CK(cudaStreamSynchronize(s));   // the table is local
    str_hash(c, names, ~0ULL);
    int32_t *ngid, *entry_of, *ment;
    uint8_t *mkeep;
    CKR(ar.alloc(&ngid, std::max<long long>(M1, 1)));
    StrTable nt;
    CKR(str_group(c, ar, names, nullptr, false, 0, &nt, ngid));
    CKR(ar.alloc(&entry_of, std::max<long long>(nt.n_groups, 1)));
    CKR(ar.alloc(&ment, std::max<long long>(M1, 1)));
    CKR(ar.alloc(&mkeep, std::max<long long>(M1, 1)));
    if (nt.n_groups > 0)
      k_name_entry<<<grid_for(nt.n_groups, 256, c->sm_count), 256, 0, s>>>(nt.n_groups, nt.first_sorted, names.off,
                                                                           (const unsigned char *)names.w, T, traw.off, traw.bytes, entry_of);
    k_member_info<<<grid_for(D * 32, 256, c->sm_count), 256, 0, s>>>(D, ra.line_moff, ngid, entry_of, d_id, ment, mkeep);
    c->launches += 2;
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
  char *host = (char *)ctx->pinned_get((size_t)std::max<long long>(total, 1), /*for_result=*/false);
  if (!host) return set_error(CCO_E_OOM, "pinned host allocation failed");
  if (total > 0) CK(cudaMemcpyAsync(host, d_out, (size_t)total, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  *out_bytes = host;
  *out_len = total;
  return CCO_OK;
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
  std::vector<long long> train_at, rank_at;
};
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
  bool finished = false;
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
  ar.take(p);
  lg->dev.push_back(p);
  return CCO_OK;
}
// a buffer the log kept, freed before the log is
static void log_drop(cco_event_log *lg, void *p) {
  for (size_t i = 0; p && i < lg->dev.size(); ++i)
    if (lg->dev[i] == p) {
      cudaFreeAsync(p, lg->ctx->stream);
      lg->dev.erase(lg->dev.begin() + i);
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
  if (T == 0) return CCO_OK;
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
static int win_records(cco_event_log *lg, Arena &ar, const EvLines &ev, const int32_t *code, long long base) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  const long long L = ev.L;
  const unsigned char *bb = lg->stage;
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
  if (lg->n_rec + R > lg->rec_cap) {   // grow geometrically
    lg->rec_cap = std::max(2 * lg->rec_cap, lg->n_rec + R);
    CKR(log_grow(lg, ar, &lg->rec, lg->rec_cap, lg->n_rec, 0));
  }
  k_win_ident<<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, ridx, base, ev.sb, ev.span, ev.xspan, bb, hd, hr, codes, acc, ev.tm, ev.flag,
                                                          code, lg->rec + lg->n_rec);
  c->launches++;
  lg->n_rec += R;
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
  JMember *jm;
  CKR(ar.alloc(&jm, L));
  k_event_strings<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, nullptr, kEvName, ev.sb, ev.span, bb, jm);
  c->launches++;
  DevStrCol names;
  long long name_bytes = 0;
  CKR(json_decode(c, ar, L, jm, bb, &names, &name_bytes));
  ar.release(jm);
  str_hash(c, names, ~0ULL);
  int32_t *code;
  CKR(ar.alloc(&code, L));
  StrTable nt;
  CKR(str_group(c, ar, names, nullptr, false, 0, &nt, code));
  const long long NC = nt.n_groups;
  cco_dictionary_t nd;
  CKR(str_dictionary(c, ar, names, nt, &nd));
  CK(cudaStreamSynchronize(s));
  std::vector<int32_t> remap((size_t)NC);
  for (long long k = 0; k < NC; ++k) {
    std::string nm(nd.bytes + nd.offsets[k], (size_t)(nd.offsets[k + 1] - nd.offsets[k]));
    auto it = lg->name_code.find(nm);
    if (it == lg->name_code.end()) {
      it = lg->name_code.emplace(nm, (int)lg->name_off.size() - 1).first;
      lg->name_bytes += nm;
      lg->name_off.push_back((int64_t)lg->name_bytes.size());
    }
    remap[k] = it->second;
  }
  c->pinned_put((void *)nd.offsets);
  c->pinned_put((void *)nd.bytes);
  str_table_release(ar, nt);
  str_release(ar, names);
  const long long NG = (long long)lg->name_off.size() - 1;
  int32_t *d_remap;
  CKR(ar.alloc(&d_remap, NC));
  CK(cudaMemcpyAsync(d_remap, remap.data(), sizeof(int32_t) * (size_t)NC, cudaMemcpyHostToDevice, s));
  k_remap_i32<<<grid_for(L, 256, c->sm_count), 256, 0, s>>>(L, d_remap, code);
  c->launches++;
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
  // 7. training and ranking events partitioned by name, file order inside a name: decoded ids and times
  uint32_t *idx;
  CKR(event_partition(c, ar, L, ev.flag, kEvTraining, code, (uint32_t)NG, &idx));
  CKR(event_column(c, ar, lg, sg.train_at[NG], idx, kEvEntityId, ev.sb, ev.span, bb, sg.train_at, &sg.tu));
  CKR(event_column(c, ar, lg, sg.train_at[NG], idx, kEvTargetId, ev.sb, ev.span, bb, sg.train_at, &sg.ti));
  if (lg->dedup || lg->history) CKR(win_entry_lines(lg, ar, sg.train_at[NG], idx, base, &sg.tline));
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
  if (lg->dedup) CKR(win_entry_lines(lg, ar, NR, idx, base, &sg.rline));
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

// removeDuplicates at finish: the records of every chunk sorted by (hash, time desc, line desc); all but the first of each
// run are dropped -> *bitmap over the global lines (kept by the log until finish ends); the counts of the drops
static int win_mark(cco_event_log *lg, uint32_t **bitmap, long long *n_prop_dup) {
  cco_ctx *c = lg->ctx;
  cudaStream_t s = c->stream;
  Arena ar(s);
  const long long N = lg->n_rec, NG = (long long)lg->name_off.size() - 1, words = lg->n_lines / 32 + 1;
  CKR(ar.alloc(bitmap, words));
  CKR(log_keep(ar, lg, *bitmap));
  CK(cudaMemsetAsync(*bitmap, 0, sizeof(uint32_t) * (size_t)words, s));
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
  *n_prop_dup = (long long)h_cnt[2 * NG];
  lg->n_prop -= (long long)h_cnt[2 * NG];
  lg->n_ignored -= (long long)h_cnt[2 * NG + 1];
  lg->n_dup = (long long)h_cnt[2 * NG + 2];
  log_drop(lg, lg->rec);
  lg->rec = nullptr;
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
                       long long **times, long long **times2 = nullptr) {
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
  for (long long **tp : {times, times2}) {
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
  lg->cap = std::max<int64_t>(chunk_bytes, 1);
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
  nvtx_push("cco:event_log_append");
  struct Pop { ~Pop() { nvtx_pop(); } } pop;
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
  nvtx_push("cco:event_log_finish");
  struct Pop { ~Pop() { nvtx_pop(); } } pop;
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
  uint32_t *drop = nullptr;   // removeDuplicates: the dropped global lines
  long long n_prop_dup = 0;
  if (lg->dedup) {
    mail_reset(c);
    CKR(win_mark(lg, &drop, &n_prop_dup));
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
  } else if (lg->segs.size() > 1) {
    CKR(event_cat_column(lg, &EvSeg::tu, &EvSeg::train_at, lg->train_at, &lg->tu));
    CKR(event_cat_column(lg, &EvSeg::ti, &EvSeg::train_at, lg->train_at, &lg->ti));
    CKR(event_cat_column(lg, &EvSeg::ri, &EvSeg::rank_at, lg->rank_at, &lg->ri));
    CKR(event_cat_times(lg, &lg->rtime));
    if (lg->dedup || lg->history) CKR(event_cat_times(lg, &lg->tline, &EvSeg::tline, &EvSeg::train_at));
    if (lg->dedup) CKR(event_cat_times(lg, &lg->rline, &EvSeg::rline, &EvSeg::rank_at));
    if (lg->history) CKR(event_cat_times(lg, &lg->ttime, &EvSeg::ttime, &EvSeg::train_at));
  }
  lg->segs.clear();
  if (drop && lg->n_dup > 0) {   // the retained columns without the dropped lines' entries
    CKR(win_compact(lg, drop, lg->tline, lg->train_at, &lg->tu, &lg->ti, lg->history ? &lg->ttime : nullptr,
                    lg->history ? &lg->tline : nullptr));
    CKR(win_compact(lg, drop, lg->rline, lg->rank_at, &lg->ri, nullptr, &lg->rtime));
    for (long long n = 0; n < NG; ++n) {
      lg->n_train[n] = lg->train_at[n + 1] - lg->train_at[n];
      lg->n_rank[n] = lg->rank_at[n + 1] - lg->rank_at[n];
    }
  }
  if (!lg->history) {
    log_drop(lg, lg->tline);
    lg->tline = nullptr;
  }
  log_drop(lg, lg->rline);
  lg->rline = nullptr;
  if (lg->n_prop > 0) {
    mail_reset(c);
    Arena ar(s);
    CKR(event_pad(c, lg->pb, lg->pb_len));
    EvLines ev;
    CKR(event_lines(c, ar, (const uint64_t *)lg->pb, lg->pb_len, false, 0, &ev));   // judged once already
    if (n_prop_dup > 0) CKR(win_drop_property_lines(lg, ar, ev, drop));
    CKR(event_properties(c, ar, lg, ev.L, ev.flag, ev.tm, ev.sb, ev.span, lg->pb, lg->prop_line.data()));
    CK(cudaStreamSynchronize(s));
  }
  log_drop(lg, drop);
  log_drop(lg, lg->pb);
  lg->pb = nullptr;
  lg->prop_line = std::vector<long long>();
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  lg->finished = true;
  return CCO_OK;
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

int cco_event_log_read(cco_ctx_t *ctx, const char *bytes, int64_t len, cco_event_log_t **out) {
  if (!ctx || !out || len < 0 || (len > 0 && !bytes)) return set_error(CCO_E_INVALID_ARG, "null argument or negative length");
  *out = nullptr;
  if (!ctx->members.empty()) return set_error(CCO_E_UNSUPPORTED, "an event log is resident on one GPU: read it on a per-GPU context");
  nvtx_push("cco:event_log_read");
  struct Pop { ~Pop() { nvtx_pop(); } } pop;
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

// the record template: n_history_names + 2 pieces around the history lists and the blacklist (see include/cco_b200.h)
static std::vector<std::string> uq_template(const cco_user_query_t *q) {
  std::vector<std::string> t(1);
  const int k = q->n_history_names;
  auto clause = [&](const char *rest, bool hist) {
    bool any = false;
    for (int j = 0; hist && j < k; ++j) {
      if (any) t.back() += ",";
      t.back() += "{\"terms\":{" + uq_quote(q->names[j]) + ":[";
      t.emplace_back("]");
      if (q->history_in_must) t.back() += ",\"boost\":0";
      else if (q->boost) t.back() += std::string(",\"boost\":") + q->boost;
      t.back() += "}}";
      any = true;
    }
    if (*rest) {
      if (any) t.back() += ",";
      t.back() += rest;
    }
  };
  t.back() += std::string(q->header) + "\n" + q->head + ",\"query\":{\"bool\":{\"should\":[";
  clause(q->should, !q->history_in_must);
  t.back() += "],\"must\":[";
  clause(q->must, q->history_in_must != 0);
  t.back() += "],\"must_not\":[{\"ids\":{\"values\":[";
  t.emplace_back("],\"boost\":0}}");
  if (*q->must_not) t.back() += std::string(",") + q->must_not;
  t.back() += std::string("],\"minimum_should_match\":1}},\"sort\":") + q->sort + "}\n";
  return t;
}

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

static int user_queries(cco_ctx *c, const cco_event_log *lg, const cco_user_query_t *q, int64_t n_users, const int64_t *uoff,
                        const char *ubytes, char **out_body, int64_t *out_len, int64_t **out_offsets, int64_t *out_n,
                        cco_dictionary_t *out_users) {
  cudaStream_t s = c->stream;
  const int nq = q->n_names;
  std::vector<int> code(nq);
  std::vector<uint8_t> black(std::max(nq, 1), 0);
  for (int k = 0; k < nq; ++k) {
    code[k] = lg->code_of(q->names[k]);
    bool earlier = false;   // a repeated query name reads the same events: blacklist them once
    for (int j = 0; j < k; ++j) earlier |= strcmp(q->names[j], q->names[k]) == 0;
    for (int b = 0; b < q->n_blacklist_names && !earlier; ++b)
      if (strcmp(q->blacklist_names[b], q->names[k]) == 0) black[k] = 1;
  }
  CK(cudaSetDevice(c->device));
  mail_reset(c);
  Arena ar(s);
  nvtx_push("cco:user_queries");
  struct Pop { ~Pop() { nvtx_pop(); } } pop;
  // 1. the caller's columns, checked on the device before any kernel reads bytes through their offsets
  DevStrCol lc, uc;
  CKR(str_upload(c, ar, q->n_blacklist_items, q->blacklist_item_offsets, q->blacklist_item_bytes, &lc));
  if (uoff) CKR(str_upload(c, ar, n_users, uoff, ubytes, &uc));
  int *bad, h_bad = 0;
  CKR(ar.alloc(&bad, 1));
  CK(cudaMemsetAsync(bad, 0, 4, s));
  str_check_device(c, lc, bad);
  if (uoff) str_check_device(c, uc, bad);
  CKR(mail_fetch(c, &h_bad, bad, 4));
  CKR(mail_wait(c));
  if (h_bad) return set_error(CCO_E_INVALID_ARG, "decreasing offsets in the blacklist items or the users");
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
  long long G = 0;
  StrTable ut, it;
  DevStrCol tu, ti;
  uint32_t *ent = nullptr, *gord = nullptr, *hord = nullptr, *bord = nullptr;
  uint8_t *qr = nullptr, *keep_h = nullptr, *keep_b = nullptr, *d_black = nullptr;
  int32_t *uid = nullptr, *iid = nullptr, *d_limit = nullptr;
  long long *tm = nullptr, *ln = nullptr, *hstart = nullptr, *bstart = nullptr;
  unsigned long long *bkey = nullptr;
  long long B = 0;
  CKR(ar.alloc(&d_limit, std::max(nq, 1)));
  if (nq > 0) CK(cudaMemcpyAsync(d_limit, q->limits, sizeof(int32_t) * (size_t)nq, cudaMemcpyHostToDevice, s));
  if (E > 0) {
    long long *d_qoff, *d_qbase;
    CKR(ar.alloc(&d_qoff, nq + 1));
    CKR(ar.alloc(&d_qbase, nq));
    CKR(ar.alloc(&d_black, nq));
    CK(cudaMemcpyAsync(d_qoff, qoff.data(), sizeof(long long) * (size_t)(nq + 1), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_qbase, qbase.data(), sizeof(long long) * (size_t)nq, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(d_black, black.data(), (size_t)nq, cudaMemcpyHostToDevice, s));
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
    // 8. blacklist: the blacklisted names' events latest first, stably by user; each item's newest position
    uint32_t *flag, *pos, *bidx;
    CKR(ar.alloc(&flag, E + 1));
    k_uq_flag_black<<<grid_for(E, 256, c->sm_count), 256, 0, s>>>(E, gord, qr, d_black, flag);
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
      k_uq_key_user<<<grid_for(B, 256, c->sm_count), 256, 0, s>>>(B, bidx, gord, uid, bkey, bord);
      c->launches++;
      CKR(sort_pairs(c, ar, B, &bkey, &bord, bits_for(G)));
      k_uq_count<<<grid_for(B, 256, c->sm_count), 256, 0, s>>>(B, bkey, bcnt);
      uint32_t *p3;
      CKR(ar.alloc(&p3, B));
      k_uq_black_keys<<<grid_for(B, 256, c->sm_count), 256, 0, s>>>(B, bord, uid, iid, bkey, p3);
      c->launches += 2;
      CKR(sort_pairs(c, ar, B, &bkey, &p3, 64));
      CK(cudaMemsetAsync(keep_b, 0, (size_t)B, s));
      k_uq_first<<<grid_for(B, 256, c->sm_count), 256, 0, s>>>(B, bkey, p3, keep_b);
      c->launches++;
    }
    CKR(exclusive_sum(c, ar, bcnt, bstart, G + 1));
  }
  // 9. blacklistItems: item groups of the log (membership is a group test), repeats within the list dropped
  const long long NL = q->n_blacklist_items;
  int32_t *lgid;
  uint8_t *keep_l;
  CKR(ar.alloc(&lgid, std::max<long long>(NL, 1)));
  CKR(ar.alloc(&keep_l, std::max<long long>(NL, 1)));
  if (NL > 0) {
    str_hash(c, lc, ~0ULL);
    if (E > 0) {
      k_str_lookup<<<grid_for(NL, 256, c->sm_count), 256, 0, s>>>(NL, lc.off, lc.base, lc.w, lc.hash, ti.off, ti.base, ti.w, ti.hash,
                                                                 (uint64_t)it.cap - 1, it.table, it.rank_of_slot, lgid);
      c->launches++;
    } else {
      CK(cudaMemsetAsync(lgid, 0xff, sizeof(int32_t) * (size_t)NL, s));
    }
    StrTable lt;
    int32_t *lid;
    CKR(ar.alloc(&lid, NL));
    CKR(str_group(c, ar, lc, nullptr, false, 0, &lt, lid));
    k_uq_list_first<<<grid_for(NL, 256, c->sm_count), 256, 0, s>>>(NL, lid, lt.first_sorted, keep_l);
    c->launches++;
  }
  // 10. the records' users
  long long R = 0;
  int32_t *rec_uid;
  if (uoff) {
    R = n_users;
    CKR(ar.alloc(&rec_uid, std::max<long long>(R, 1)));
    if (R > 0 && E > 0) {
      str_hash(c, uc, ~0ULL);
      k_str_lookup<<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, uc.off, uc.base, uc.w, uc.hash, tu.off, tu.base, tu.w, tu.hash,
                                                                (uint64_t)ut.cap - 1, ut.table, ut.rank_of_slot, rec_uid);
      c->launches++;
    } else if (R > 0) {
      CK(cudaMemsetAsync(rec_uid, 0xff, sizeof(int32_t) * (size_t)R, s));
    }
  } else {   // every user with an event of a query name, by first line
    R = G;
    CKR(ar.alloc(&rec_uid, std::max<long long>(R, 1)));
    if (R > 0) {
      unsigned long long *mn, *uk;
      CKR(ar.alloc(&mn, G));
      CKR(ar.alloc(&uk, G));
      CK(cudaMemsetAsync(mn, 0xff, sizeof(unsigned long long) * (size_t)G, s));
      k_uq_min_line<<<grid_for(E, 256, c->sm_count), 256, 0, s>>>(E, uid, ln, mn);
      k_uq_user_keys<<<grid_for(G, 256, c->sm_count), 256, 0, s>>>(G, mn, uk, rec_uid);
      c->launches += 2;
      CKR(sort_pairs(c, ar, G, &uk, &rec_uid, bits_for(lg->n_lines)));
    }
    if (out_users) {
      uint32_t *ue;
      long long *len, *off, total = 0;
      CKR(ar.alloc(&ue, std::max<long long>(R, 1)));
      CKR(ar.alloc(&len, R + 1));
      CKR(ar.alloc(&off, R + 1));
      CK(cudaMemsetAsync(len + R, 0, 8, s));
      if (R > 0) {
        k_uq_user_entry<<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, rec_uid, ut.first_sorted, ue);
        k_str_dict_len<<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, ue, tu.off, len);
        c->launches += 2;
      }
      CKR(exclusive_sum(c, ar, len, off, R + 1));
      CK(cudaMemcpyAsync(&total, off + R, 8, cudaMemcpyDeviceToHost, s));
      CK(cudaStreamSynchronize(s));
      unsigned char *ub;
      CKR(ar.alloc(&ub, std::max<long long>(total, 1)));
      if (R > 0 && total > 0) {
        k_str_dict_gather<<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, ue, tu.off, tu.base, (const unsigned char *)tu.w, off, ub);
        c->launches++;
      }
      int64_t *ho = (int64_t *)c->pinned_get(sizeof(int64_t) * ((size_t)R + 1), /*for_result=*/false);
      char *hb = (char *)c->pinned_get((size_t)std::max<long long>(total, 1), /*for_result=*/false);
      if (!ho || !hb) return set_error(CCO_E_OOM, "pinned host allocation failed");
      CK(cudaMemcpyAsync(ho, off, sizeof(int64_t) * ((size_t)R + 1), cudaMemcpyDeviceToHost, s));
      if (total > 0) CK(cudaMemcpyAsync(hb, ub, (size_t)total, cudaMemcpyDeviceToHost, s));
      *out_users = cco_dictionary_t{R, ho, hb};
    }
  }
  // 11. the template, then a length pass, the record offsets and a write pass: one warp per record
  const std::vector<std::string> tp = uq_template(q);
  std::vector<long long> toff(tp.size() + 1, 0);
  std::string tb;
  for (size_t j = 0; j < tp.size(); ++j) {
    tb += tp[j];
    toff[j + 1] = (long long)tb.size();
  }
  long long *d_toff;
  unsigned char *d_tb;
  CKR(ar.alloc(&d_toff, (long long)toff.size()));
  CKR(ar.alloc(&d_tb, std::max<long long>((long long)tb.size(), 1)));
  CK(cudaMemcpyAsync(d_toff, toff.data(), sizeof(long long) * toff.size(), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(d_tb, tb.data(), tb.size(), cudaMemcpyHostToDevice, s));
  UqArgs a;
  a.n_rec = R;
  a.rec_uid = rec_uid;
  a.nq = nq;
  a.n_kept = q->n_history_names;
  a.limit = d_limit;
  a.hstart = hstart;
  a.hord = hord;
  a.keep_h = keep_h;
  a.bstart = bstart;
  a.bord = bord;
  a.keep_b = keep_b;
  a.bkey = bkey;
  a.B = B;
  a.ent = ent;
  a.ioff = E > 0 ? lg->ti.off : nullptr;
  a.ibytes = E > 0 ? (const unsigned char *)lg->ti.w : nullptr;
  a.n_list = NL;
  a.loff = lc.off;
  a.lbase = lc.base;
  a.lbytes = (const unsigned char *)lc.w;
  a.lgid = lgid;
  a.keep_l = keep_l;
  a.toff = d_toff;
  a.tbytes = d_tb;
  long long *rlen, *roff;
  CKR(ar.alloc(&rlen, R + 1));
  CKR(ar.alloc(&roff, R + 1));
  CK(cudaMemsetAsync(rlen + R, 0, 8, s));
  if (R > 0) {
    k_uq_record<false><<<grid_for(R * 32, 256, c->sm_count), 256, 0, s>>>(a, nullptr, rlen, nullptr);
    c->launches++;
  }
  CKR(exclusive_sum(c, ar, rlen, roff, R + 1));
  int64_t *ho = (int64_t *)c->pinned_get(sizeof(int64_t) * ((size_t)R + 1), /*for_result=*/false);
  if (!ho) return set_error(CCO_E_OOM, "pinned host allocation failed");
  CK(cudaMemcpyAsync(ho, roff, sizeof(int64_t) * ((size_t)R + 1), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  for (long long r = 0; r < R; ++r)
    if (ho[r + 1] - ho[r] >= (1LL << 31)) {
      c->pinned_put(ho);
      return set_error(CCO_E_UNSUPPORTED, "record %lld has %lld bytes, at most 2^31 - 1", r, (long long)(ho[r + 1] - ho[r]));
    }
  const long long total = ho[R];
  unsigned char *d_out;
  CKR(ar.alloc(&d_out, std::max<long long>(total, 1)));
  if (R > 0 && total > 0) {
    k_uq_record<true><<<grid_for(R * 32, 256, c->sm_count), 256, 0, s>>>(a, roff, nullptr, d_out);
    c->launches++;
  }
  char *host = (char *)c->pinned_get((size_t)std::max<long long>(total, 1), /*for_result=*/false);
  if (!host) return set_error(CCO_E_OOM, "pinned host allocation failed");
  if (total > 0) CK(cudaMemcpyAsync(host, d_out, (size_t)total, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  *out_body = host;
  *out_len = total;
  *out_offsets = ho;
  *out_n = R;
  return CCO_OK;
}
}  // namespace cco

int cco_event_log_begin_ex(cco_ctx_t *ctx, int64_t chunk_bytes, const cco_event_window_t *w, uint32_t flags, cco_event_log_t **out) {
  if (flags & ~(uint32_t)CCO_LOG_KEEP_HISTORY) return set_error(CCO_E_INVALID_ARG, "unknown flags 0x%x", (unsigned)flags);
  CKR(cco_event_log_begin_window(ctx, chunk_bytes, w, out));
  (*out)->history = (flags & CCO_LOG_KEEP_HISTORY) != 0;
  return CCO_OK;
}

int cco_event_log_user_queries(cco_ctx_t *ctx, const cco_event_log_t *lg, const cco_user_query_t *q, int64_t n_users,
                               const int64_t *user_offsets, const char *user_bytes, char **out_body, int64_t *out_len,
                               int64_t **out_offsets, int64_t *out_n, cco_dictionary_t *out_users) {
  if (!ctx || !lg || !q || !out_body || !out_len || !out_offsets || !out_n) return set_error(CCO_E_INVALID_ARG, "null argument");
  if (!ctx->members.empty() || lg->ctx != ctx) return set_error(CCO_E_UNSUPPORTED, "build queries on the per-GPU context that read the log");
  CKR(log_state(lg, true));
  CKR(uq_check_host(q, n_users, user_offsets, user_bytes));
  if (!lg->history) return set_error(CCO_E_INVALID_ARG, "the log was read without history retention (cco_event_log_begin_ex, CCO_LOG_KEEP_HISTORY)");
  if (out_users) *out_users = cco_dictionary_t{0, nullptr, nullptr};
  return user_queries(ctx, lg, q, n_users, user_offsets, user_bytes, out_body, out_len, out_offsets, out_n, out_users);
}

namespace cco {
// the record template of an item query, 9 + n_names pieces: 0 head and "should":[, 1 should_head, 2 should, 3 "must":[,
// 4 must_head, 5 must, 6 the ids clause up to its values, 7 the rest of the record, 8 the end of a similar-items clause,
// 9 + j the start of model name j's clause (see include/cco_b200.h)
static std::vector<std::string> iq_template(const cco_item_query_t *q) {
  std::vector<std::string> t(9 + q->n_names);
  t[0] = std::string(q->header) + "\n" + q->head + ",\"query\":{\"bool\":{\"should\":[";
  t[1] = q->should_head;
  t[2] = q->should;
  t[3] = "],\"must\":[";
  t[4] = q->must_head;
  t[5] = q->must;
  t[6] = "],\"must_not\":[{\"ids\":{\"values\":[";
  t[7] = std::string("],\"boost\":0}}") + (*q->must_not ? std::string(",") + q->must_not : std::string()) +
         "],\"minimum_should_match\":1}},\"sort\":" + q->sort + "}\n";
  t[8] = q->similar_in_must ? "],\"boost\":0}}" : q->similar_boost ? std::string("],\"boost\":") + q->similar_boost + "}}" : "]}}";
  for (int j = 0; j < q->n_names; ++j) t[9 + j] = "{\"terms\":{" + uq_quote(q->names[j]) + ":[";
  return t;
}

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

static int item_queries(cco_ctx *c, const char *body, int64_t body_len, const cco_item_query_t *q, int64_t n_items, const int64_t *ioff,
                        const char *ibytes, char **out_body, int64_t *out_len, int64_t **out_offsets, int64_t *out_n,
                        cco_dictionary_t *out_items) {
  cudaStream_t s = c->stream;
  CK(cudaSetDevice(c->device));
  Arena ar(s);
  nvtx_push("cco:item_queries");
  struct Pop { ~Pop() { nvtx_pop(); } } pop;
  mail_reset(c);
  const bool all = ioff == nullptr;
  const long long NI = all ? 0 : n_items, NL = q->n_blacklist_items;
  // 1-4. the documents: members, decoded names and _ids
  BulkDocs bd;
  CKR(bulk_parse(c, ar, body, body_len, NI + NL, "items + blacklist items", &bd));
  const long long D = bd.D, R = all ? D : NI;
  // 5. one key column: the decoded _ids, the items, blacklistItems; the caller's offsets are checked on the device before
  //    any kernel reads bytes through them
  const long long NK = D + NI + NL;
  const long long nb = bd.ids_bytes + (NI > 0 ? ioff[NI] - ioff[0] : 0) +
                       (NL > 0 ? q->blacklist_item_offsets[NL] - q->blacklist_item_offsets[0] : 0);
  DevStrCol key;
  key.n = NK;
  key.base = 0;
  CKR(ar.alloc(&key.off, NK + 1));
  CKR(ar.alloc(&key.w, (nb + 16 + 7) / 8));
  CKR(ar.alloc(&key.hash, std::max<long long>(NK, 1)));
  CK(cudaMemsetAsync(key.off, 0, 8, s));
  int *bad, h_bad = 0;
  CKR(ar.alloc(&bad, 1));
  CK(cudaMemsetAsync(bad, 0, sizeof(int), s));
  long long at = 0, byte_at = 0;
  if (D > 0) {
    k_rebase<<<grid_for(D + 1, 256, c->sm_count), 256, 0, s>>>(D + 1, bd.ids.off, 0, key.off);
    c->launches++;
    if (bd.ids_bytes > 0) CK(cudaMemcpyAsync(key.w, bd.ids.w, (size_t)bd.ids_bytes, cudaMemcpyDeviceToDevice, s));
    at = D;
    byte_at = bd.ids_bytes;
  }
  for (int k = 0; k < 2; ++k) {
    const long long n = k ? NL : NI;
    const int64_t *off = k ? q->blacklist_item_offsets : ioff;
    const char *bytes = k ? q->blacklist_item_bytes : ibytes;
    if (n == 0) continue;
    long long *tmp;
    CKR(ar.alloc(&tmp, n + 1));
    CK(cudaMemcpyAsync(tmp, off, sizeof(int64_t) * ((size_t)n + 1), cudaMemcpyHostToDevice, s));
    k_str_check<<<grid_for(n, 256, c->sm_count), 256, 0, s>>>(n, tmp, bad);
    k_rebase<<<grid_for(n + 1, 256, c->sm_count), 256, 0, s>>>(n + 1, tmp, byte_at - off[0], key.off + at);
    c->launches += 2;
    const long long kb = off[n] - off[0];
    if (kb > 0) CK(cudaMemcpyAsync((char *)key.w + byte_at, bytes + off[0], (size_t)kb, cudaMemcpyHostToDevice, s));
    at += n;
    byte_at += kb;
  }
  CKR(mail_fetch(c, &h_bad, bad, 4));
  CKR(mail_wait(c));
  if (h_bad) return set_error(CCO_E_INVALID_ARG, "decreasing offsets in the items or the blacklist items");
  // 6. one exact grouping over the key column; a group that holds two documents is a repeated _id
  str_hash(c, key, ~0ULL);
  int32_t *gid;
  CKR(ar.alloc(&gid, std::max<long long>(NK, 1)));
  StrTable tb;
  CKR(str_group(c, ar, key, nullptr, false, 0, &tb, gid));
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
  // 7. blacklistItems: each group's first list index (membership and repeats are group tests)
  const long long G = tb.n_groups;
  uint32_t *first_in_list;
  CKR(ar.alloc(&first_in_list, std::max<long long>(G, 1)));
  CK(cudaMemsetAsync(first_in_list, 0xff, sizeof(uint32_t) * (size_t)std::max<long long>(G, 1), s));
  if (NL > 0) {
    k_iq_black<<<grid_for(NL, 256, c->sm_count), 256, 0, s>>>(NL, D + NI, gid, first_in_list);
    c->launches++;
  }
  // 8. the records' documents; the queried documents
  int32_t *rec_doc, *rec_key;
  uint8_t *queried;
  CKR(ar.alloc(&rec_doc, std::max<long long>(R, 1)));
  CKR(ar.alloc(&rec_key, std::max<long long>(R, 1)));
  CKR(ar.alloc(&queried, std::max<long long>(D, 1)));
  CK(cudaMemsetAsync(queried, 0, (size_t)std::max<long long>(D, 1), s));
  if (R > 0) {
    k_iq_rec<<<grid_for(R, 256, c->sm_count), 256, 0, s>>>(R, D, all, gid, tb.first_sorted, rec_doc, rec_key, queried);
    c->launches++;
  }
  // 9. the distinct model names; per document the last source member of each
  std::vector<std::string> ent;
  std::vector<int32_t> name_entry(q->n_names);
  for (int j = 0; j < q->n_names; ++j) {
    size_t t = 0;
    while (t < ent.size() && ent[t] != q->names[j]) ++t;
    if (t == ent.size()) ent.push_back(q->names[j]);
    name_entry[j] = (int32_t)t;
  }
  const int T = (int)ent.size();
  const long long DT = D * T;
  long long *eoff;
  CKR(ar.alloc(&eoff, DT + 1));
  CK(cudaMemsetAsync(eoff, 0, sizeof(long long) * (size_t)(DT + 1), s));
  DevStrCol dec;
  if (D > 0) {
    std::vector<int64_t> toff(T + 1, 0);
    std::string tblob;
    for (int t = 0; t < T; ++t) {
      tblob += ent[t];
      toff[t + 1] = (int64_t)tblob.size();
    }
    const cco_dictionary_t td = {T, toff.data(), tblob.data()};
    DevDict traw;
    CKR(upload_dict(c, ar, td, &traw));
    CK(cudaStreamSynchronize(s));   // the table is local
    str_hash(c, bd.names, ~0ULL);
    int32_t *ngid, *entry_of, *pick;
    CKR(ar.alloc(&ngid, std::max<long long>(bd.M1, 1)));
    StrTable nt;
    CKR(str_group(c, ar, bd.names, nullptr, false, 0, &nt, ngid));
    CKR(ar.alloc(&entry_of, std::max<long long>(nt.n_groups, 1)));
    CKR(ar.alloc(&pick, DT));
    if (nt.n_groups > 0)
      k_name_entry<<<grid_for(nt.n_groups, 256, c->sm_count), 256, 0, s>>>(nt.n_groups, nt.first_sorted, bd.names.off,
                                                                           (const unsigned char *)bd.names.w, T, traw.off, traw.bytes, entry_of);
    k_iq_pick<<<grid_for(D, 256, c->sm_count), 256, 0, s>>>(D, T, bd.line_moff, ngid, entry_of, pick);
    c->launches += 2;
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
  // 11. the template, then a length pass, the record offsets and a write pass: one warp per record
  const std::vector<std::string> tp = iq_template(q);
  std::vector<long long> toff(tp.size() + 1, 0);
  std::string tbl;
  for (size_t j = 0; j < tp.size(); ++j) {
    tbl += tp[j];
    toff[j + 1] = (long long)tbl.size();
  }
  long long *d_toff;
  unsigned char *d_tb;
  int32_t *d_entry;
  CKR(ar.alloc(&d_toff, (long long)toff.size()));
  CKR(ar.alloc(&d_tb, std::max<long long>((long long)tbl.size(), 1)));
  CKR(ar.alloc(&d_entry, q->n_names));
  CK(cudaMemcpyAsync(d_toff, toff.data(), sizeof(long long) * toff.size(), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(d_tb, tbl.data(), tbl.size(), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(d_entry, name_entry.data(), sizeof(int32_t) * (size_t)q->n_names, cudaMemcpyHostToDevice, s));
  IqArgs a;
  a.n_rec = R;
  a.rec_doc = rec_doc;
  a.rec_key = rec_key;
  a.kgid = gid;
  a.koff = key.off;
  a.kbytes = (const unsigned char *)key.w;
  a.line_moff = bd.line_moff;
  a.T = T;
  a.n_names = q->n_names;
  a.name_entry = d_entry;
  a.eoff = eoff;
  a.doff = dec.off;
  a.dbytes = (const unsigned char *)dec.w;
  a.slice = q->max_query_events;
  a.in_must = q->similar_in_must;
  a.exclude_self = q->exclude_self;
  a.n_list = NL;
  a.list_at = D + NI;
  a.first_in_list = first_in_list;
  a.toff = d_toff;
  a.tbytes = d_tb;
  long long *rlen, *roff;
  CKR(ar.alloc(&rlen, R + 1));
  CKR(ar.alloc(&roff, R + 1));
  CK(cudaMemsetAsync(rlen + R, 0, 8, s));
  if (R > 0) {
    k_iq_record<false><<<grid_for(R * 32, 256, c->sm_count), 256, 0, s>>>(a, nullptr, rlen, nullptr);
    c->launches++;
  }
  CKR(exclusive_sum(c, ar, rlen, roff, R + 1));
  int64_t *ho = (int64_t *)c->pinned_get(sizeof(int64_t) * ((size_t)R + 1), /*for_result=*/false);
  if (!ho) return set_error(CCO_E_OOM, "pinned host allocation failed");
  CK(cudaMemcpyAsync(ho, roff, sizeof(int64_t) * ((size_t)R + 1), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  for (long long r = 0; r < R; ++r)
    if (ho[r + 1] - ho[r] >= (1LL << 31)) {
      c->pinned_put(ho);
      return set_error(CCO_E_UNSUPPORTED, "record %lld has %lld bytes, at most 2^31 - 1", r, (long long)(ho[r + 1] - ho[r]));
    }
  const long long total = ho[R];
  unsigned char *d_out;
  CKR(ar.alloc(&d_out, std::max<long long>(total, 1)));
  if (R > 0 && total > 0) {
    k_iq_record<true><<<grid_for(R * 32, 256, c->sm_count), 256, 0, s>>>(a, roff, nullptr, d_out);
    c->launches++;
  }
  char *host = (char *)c->pinned_get((size_t)std::max<long long>(total, 1), /*for_result=*/false);
  if (!host) return set_error(CCO_E_OOM, "pinned host allocation failed");
  if (total > 0) CK(cudaMemcpyAsync(host, d_out, (size_t)total, cudaMemcpyDeviceToHost, s));
  if (all && out_items) {   // the documents' decoded _ids, in body order
    int64_t *io = (int64_t *)c->pinned_get(sizeof(int64_t) * ((size_t)D + 1), /*for_result=*/false);
    char *ib = (char *)c->pinned_get((size_t)std::max<long long>(bd.ids_bytes, 1), /*for_result=*/false);
    if (!io || !ib) return set_error(CCO_E_OOM, "pinned host allocation failed");
    io[0] = 0;
    if (D > 0) CK(cudaMemcpyAsync(io, bd.ids.off, sizeof(int64_t) * ((size_t)D + 1), cudaMemcpyDeviceToHost, s));
    if (bd.ids_bytes > 0) CK(cudaMemcpyAsync(ib, bd.ids.w, (size_t)bd.ids_bytes, cudaMemcpyDeviceToHost, s));
    *out_items = cco_dictionary_t{D, io, ib};
  }
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  *out_body = host;
  *out_len = total;
  *out_offsets = ho;
  *out_n = R;
  return CCO_OK;
}
}  // namespace cco

int cco_item_queries(cco_ctx_t *ctx, const char *index_body, int64_t index_len, const cco_item_query_t *q, int64_t n_items,
                     const int64_t *item_offsets, const char *item_bytes, char **out_body, int64_t *out_len, int64_t **out_offsets,
                     int64_t *out_n, cco_dictionary_t *out_items) {
  if (!ctx || !q || !out_body || !out_len || !out_offsets || !out_n || index_len < 0 || (index_len > 0 && !index_body))
    return set_error(CCO_E_INVALID_ARG, "null argument or negative length");
  if (!ctx->members.empty()) return set_error(CCO_E_UNSUPPORTED, "per-GPU contexts only");
  if (index_len > 0 && index_body[index_len - 1] != '\n') return set_error(CCO_E_INVALID_ARG, "the body does not end in a newline");
  CKR(iq_check_host(q, n_items, item_offsets, item_bytes));
  if (out_items) *out_items = cco_dictionary_t{0, nullptr, nullptr};
  return item_queries(ctx, index_body, index_len, q, n_items, item_offsets, item_bytes, out_body, out_len, out_offsets, out_n, out_items);
}

int cco_event_log_free(cco_event_log_t *lg) {
  event_log_release(lg);
  return CCO_OK;
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
  nvtx_push("cco:pop_model");
  struct Pop { ~Pop() { nvtx_pop(); } } pop;
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

}  // extern "C"
