// cco_sampler.cuh -- pass 1 of sampleDownAndBinarize, entry-parallel.
//
// Reference: Mahout 0.13.0 SimilarityAnalysis.sampleDownAndBinarize as called from
// src/main/scala/URAlgorithm.scala:323-329, 343-346 (SURVEY.md 8a, H2); the sampler itself is the
// counter-based one of include/cco_b200.h "Sampler" (bit-identical to the CPU restatement's).
//
// The row-parallel form (k_downsample_count<SG> in cco_kernels.cuh: 8 lanes per user row) is issue-bound, not HBM-bound:
// four independent rows per warp diverge on trip count and on the rate branches, so most lanes of a warp idle, and the
// rows above 256 entries need a warp-per-row launch whose duration is the longest row's dependent chain (it does not
// shrink when users are sharded).
// Here a warp walks a CHUNK of consecutive stored entries, whatever rows they belong to:
//   * the first row of the chunk comes from a 32-ary search on row_ptr (4 probe rounds at 1 M rows);
//   * the warp keeps a WINDOW of 32 consecutive rows in registers: lane i owns row (base + i) -- its [start, end), its
//     integer keep threshold and its hash prefix, computed once per row instead of once per lane;
//   * each lane finds the row of its entry by a 5-step binary search over the window's row ends (shuffles), pulls the
//     row's constants from the owner lane, decides, writes the keep byte, bumps the post-sample column count;
//   * the owner lane counts the kept entries of its row from the ballot and a lane-range mask -- no shuffles, no atomics
//     inside the chunk; one atomicAdd per (row, window) when the window slides or the chunk ends (rows may straddle chunks).
// Every lane does useful work on every entry, rows of any length are split evenly over warps, and the kernel only
// dereferences entry offsets inside [q_lo, q_hi): a malformed row_ptr (reported by count_raw_columns) cannot send it out of bounds.
// Pass 2 is an order-preserving stream compaction by the keep bytes (cub::DeviceSelect::Flagged in cco_api.cu): kept
// entries keep their global order, so their rank inside the block is their offset from the block's first kept entry.
//
// These kernels supersede k_downsample_count / k_downsample_write, and k_col_counts_smem / k_col_histogram_flat (the raw
// counts of the train and of every debug entry, cco_api.cu count_raw_columns) supersede k_col_histogram; the old ones stay in cco_kernels.cuh
// unreferenced: bench.py names the row-kernel build a line was measured on by that file's hash (source_build_id).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "cco_kernels.cuh"

namespace cco {

constexpr int kSampleChunk = 256;   // stored entries per warp visit

// largest r in [0, n_rows) with rp[r] <= q (the row holding entry q when row_ptr is monotone); warp-uniform
template <typename P>
__device__ __forceinline__ long long warp_find_row(const P *__restrict__ rp, long long n_rows, long long q, int lane) {
  long long lo = 0, hi = n_rows;
  while (hi - lo > 1) {
    const long long step = (hi - lo + 31) / 32;
    const long long p = lo + lane * step;
    const bool ok = p < hi && (long long)rp[p] <= q;
    const unsigned b = __ballot_sync(0xffffffffu, ok) | 1u;   // lane 0 probes rp[lo] <= q, the loop invariant
    const int top = 31 - __clz(b);
    lo += top * step;
    hi = hi < lo + step ? hi : lo + step;
  }
  return lo;
}

__global__ void __launch_bounds__(256) k_sample_count(long long n_rows, long long row_base, const long long *__restrict__ rp,
                                                      const int32_t *__restrict__ col, int32_t n_cols, long long q_lo, long long q_hi,
                                                      const unsigned long long *__restrict__ col_thr, int32_t m, int32_t seed, uint32_t flags,
                                                      const int *__restrict__ bad /* nullable: the validation verdict (count_raw_columns) */,
                                                      uint32_t *__restrict__ kept_per_row /* zeroed */, int32_t *__restrict__ new_counts,
                                                      uint8_t *__restrict__ keep_flag) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  const long long n_chunks = (q_hi - q_lo + kSampleChunk - 1) / kSampleChunk;
  const bool intdiv = (flags & CCO_FLAG_ROWRATE_INTDIV) != 0;
  const long long kNoRow = 0x7fffffffffffffffLL;
  if (n_rows <= 0) return;
  if (bad && *bad) {
    // malformed matrix (the call fails once the host reads the verdict): keep nothing, so that pass 2 writes nothing
    for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < q_hi - q_lo; q += (long long)gridDim.x * blockDim.x) keep_flag[q] = 0;
    return;
  }
  for (long long chunk = warp; chunk < n_chunks; chunk += n_warps) {
    const long long Q0 = q_lo + chunk * kSampleChunk;
    const long long Q1 = Q0 + kSampleChunk < q_hi ? Q0 + kSampleChunk : q_hi;
    long long base = warp_find_row(rp, n_rows, Q0, lane);
    long long start_i, end_i;
    unsigned long long t_i, x_i;
    uint32_t kept_i;
    // lane i takes over row base + i
#define CCO_LOAD_WINDOW()                                                                                   \
  {                                                                                                         \
    const long long r = base + lane;                                                                        \
    start_i = end_i = kNoRow;                                                                               \
    t_i = kKeepAlways;                                                                                      \
    x_i = 0;                                                                                                \
    if (r < n_rows) {                                                                                       \
      start_i = rp[r];                                                                                      \
      end_i = rp[r + 1];                                                                                    \
      const long long d = end_i - start_i;                                                                  \
      if (d > (long long)m) t_i = rate_threshold(row_sample_rate(d, m, intdiv)); /* d <= m: rate 1, no division */ \
      x_i = mix64(((uint64_t)(uint32_t)seed << 32) | (uint64_t)(uint32_t)(row_base + r));                   \
    }                                                                                                       \
    kept_i = 0;                                                                                             \
  }
#define CCO_FLUSH_WINDOW()                                                                                  \
  if (kept_i) atomicAdd(&kept_per_row[row_base + base + lane], kept_i);
    CCO_LOAD_WINDOW()
    for (long long qb = Q0; qb < Q1; qb += 32) {
      const long long q = qb + lane;
      bool pending = q < Q1;
      const int32_t j = pending ? col[q] : 0;
      unsigned long long t_col = kKeepAlways;
      if (pending && (uint32_t)j < (uint32_t)n_cols) t_col = col_thr[j];
      while (true) {
        // rows of the window that end at or before q (row ends are non-decreasing): 0..32
        int idx = 0;
#pragma unroll
        for (int step = 16; step > 0; step >>= 1) {
          const long long v = __shfl_sync(0xffffffffu, end_i, idx + step - 1);
          if (v <= q) idx += step;
        }
        {
          const long long v = __shfl_sync(0xffffffffu, end_i, idx);   // idx <= 31 here
          if (v <= q) idx += 1;
        }
        const int src = idx & 31;
        const unsigned long long t_row = __shfl_sync(0xffffffffu, t_i, src);
        const unsigned long long x_row = __shfl_sync(0xffffffffu, x_i, src);
        const bool here = pending && idx < 32;
        const bool real_row = base + idx < n_rows;   // an entry past the last row's end (malformed row_ptr) is dropped
        bool keep = false;
        if (here) {
          // (ids outside [0, n_cols) belong to a malformed matrix: dropped here, reported by count_raw_columns)
          keep = real_row && (uint32_t)j < (uint32_t)n_cols && keep_entry_thr(t_row, t_col, x_row, (uint32_t)j);
          keep_flag[q - q_lo] = keep ? 1 : 0;   // pass 2 compacts by these decisions
          if (keep && new_counts) atomicAdd(&new_counts[j], 1);
        }
        const unsigned kb = __ballot_sync(0xffffffffu, keep);
        // the owner lane counts its row's kept entries of this batch: lanes [a, b) hold entries [start_i, end_i)
        const int a = start_i <= qb ? 0 : (start_i >= qb + 32 ? 32 : (int)(start_i - qb));
        const int b = end_i <= qb ? 0 : (end_i >= qb + 32 ? 32 : (int)(end_i - qb));
        if (b > a) {
          const unsigned below_b = b >= 32 ? 0xffffffffu : ((1u << b) - 1u);
          const unsigned below_a = (1u << a) - 1u;   // a < b <= 32, so a <= 31
          kept_i += __popc(kb & below_b & ~below_a);
        }
        pending = pending && !here;
        if (!__any_sync(0xffffffffu, pending)) break;
        // some entries lie beyond the window: slide it
        CCO_FLUSH_WINDOW()
        base += 32;
        if (base >= n_rows) {   // entries past the last row (malformed row_ptr): not kept
          if (pending) keep_flag[q - q_lo] = 0;
          kept_i = 0;
          start_i = end_i = kNoRow;
          break;
        }
        CCO_LOAD_WINDOW()
      }
      if (base >= n_rows) {
        // malformed tail: every later entry of the chunk is dropped as well
        for (long long q2 = qb + 32 + lane; q2 < Q1; q2 += 32) keep_flag[q2 - q_lo] = 0;
        break;
      }
    }
    if (base < n_rows && base + lane < n_rows) { CCO_FLUSH_WINDOW() }
#undef CCO_LOAD_WINDOW
#undef CCO_FLUSH_WINDOW
  }
}

// ---- validation + raw column counts of a not yet validated block, entry-parallel ------------------------------------------
// The in-train safety net needs only "malformed or not" (canonical order is the caller's promise under
// CCO_FLAG_ASSUME_CANONICAL, and the synchronous upload canonicalises): row_ptr is checked per row, column ids are checked
// by the pass that reads every column id anyway -- the raw column histogram (numNonZeroElementsPerColumn).
__global__ void k_check_row_ptr(long long n_rows, const long long *__restrict__ rp, long long q_lo, long long q_hi, int *flags) {
  int bad = 0;
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < n_rows; r += (long long)gridDim.x * blockDim.x) {
    const long long s = rp[r], e = rp[r + 1];
    if (e < s || s < q_lo || e > q_hi) bad = 1;
  }
  if (bad) atomicOr(&flags[0], 1);
}
// counts[j] += 1 for every stored entry of the block (col = the block's first entry, n entries); ids outside [0, n_cols)
// are skipped and, with `flags`, reported.  Replicated counters as in k_col_histogram.  AGG: aggregate equal ids of a warp
// first (__match_any_sync).
template <bool AGG>
__global__ void k_col_histogram_flat(long long n, const int32_t *__restrict__ col, int32_t n_cols, int32_t *__restrict__ counts, int n_copies,
                                     long long copy_stride, int *flags /* nullable */) {
  int32_t *mine = counts + (long long)(blockIdx.x % n_copies) * copy_stride;
  const int lane = threadIdx.x & 31;
  int bad = 0;
  for (long long q0 = blockIdx.x * (long long)blockDim.x + (threadIdx.x & ~31); q0 < n; q0 += (long long)gridDim.x * blockDim.x) {
    const long long q = q0 + lane;
    const bool act = q < n;
    const int32_t j = act ? col[q] : -1;
    const bool ok = act && (uint32_t)j < (uint32_t)n_cols;
    if (act && !ok) bad = 1;
    if (AGG) {
      const unsigned om = __ballot_sync(0xffffffffu, ok);
      if (ok) {
        const unsigned peers = __match_any_sync(om, j);
        if ((__ffs(peers) - 1) == lane) atomicAdd(&mine[j], __popc(peers));
      }
    } else if (ok) {
      atomicAdd(&mine[j], 1);
    }
  }
  if (flags && bad) atomicOr(&flags[0], 1);
}

// ---- `drmA.t`, entry-parallel ----------------------------------------------------------------------------------------------
// users[cursor[j]++] = u for every entry (u, j) of the sampled primary matrix.  A warp walks chunks of kSampleChunk
// entries with k_sample_count's window of 32 rows (lane i holds the end of row base + i), so every lane scatters one
// entry per batch whatever the row lengths (about 5 kept entries per user at C3).  The order of users inside an item's
// list is not fixed; nothing downstream depends on it.
__global__ void __launch_bounds__(256) k_transpose_entries(long long n_rows, const uint32_t *__restrict__ rp, const int32_t *__restrict__ col,
                                                           uint32_t *__restrict__ cursor, int32_t *__restrict__ users) {
  if (n_rows <= 0) return;
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  const long long nnz = rp[n_rows];
  const long long n_chunks = (nnz + kSampleChunk - 1) / kSampleChunk;
  for (long long chunk = warp; chunk < n_chunks; chunk += n_warps) {
    const long long Q0 = chunk * kSampleChunk;
    const long long Q1 = Q0 + kSampleChunk < nnz ? Q0 + kSampleChunk : nnz;
    long long base = warp_find_row(rp, n_rows, Q0, lane);
    long long end_i = base + lane < n_rows ? (long long)rp[base + lane + 1] : 0x7fffffffffffffffLL;
    for (long long qb = Q0; qb < Q1; qb += 32) {
      const long long q = qb + lane;
      bool pending = q < Q1;
      const int32_t j = pending ? col[q] : 0;
      while (true) {
        int idx = 0;   // rows of the window that end at or before q
#pragma unroll
        for (int step = 16; step > 0; step >>= 1) {
          const long long v = __shfl_sync(0xffffffffu, end_i, idx + step - 1);
          if (v <= q) idx += step;
        }
        if (__shfl_sync(0xffffffffu, end_i, idx & 31) <= q) idx += 1;
        const bool here = pending && idx < 32;
        if (here) users[atomicAdd(&cursor[j], 1u)] = (int32_t)(base + idx);
        pending = pending && !here;
        if (!__any_sync(0xffffffffu, pending)) break;
        base += 32;   // entries of rows past the window (a well-formed row_ptr: they lie in rows < n_rows)
        end_i = base + lane < n_rows ? (long long)rp[base + lane + 1] : 0x7fffffffffffffffLL;
      }
    }
  }
}

// ---- raw column counts in shared memory, one launch over a batch of matrices ----------------------------------------------
// When a matrix's column space fits a CTA's shared memory as 16-bit counters (n_cols <= ~116 K on H100), each CTA counts
// an even slice of its matrix's entries privately and adds its counters to the global counts once, at the end: Zipf-hot
// columns cost shared-memory atomics instead of contended L2 atomics, and nothing is replicated or summed afterwards.
// A counter that reaches 2^15 hands 2^15 to the global count at once (hist_add), so no 16-bit counter can overflow
// whatever the slice length.  The same CTAs check their share of the matrix's row_ptr (k_check_row_ptr's test).
constexpr int kHistSegs = 8;                     // matrices per launch
constexpr int kHistThreads = 1024;
constexpr long long kHistMinEntries = 1 << 16;   // entries per CTA at least: zeroing and flushing cost ~n_cols / CTA
struct HistSeg {
  const int32_t *col;   // the block's first entry
  const long long *rp;  // the block's row_ptr (n_rows + 1 values in [q_lo, q_hi] when well formed)
  long long nnz, n_rows, q_lo, q_hi;
  int32_t *counts;      // the matrix's raw counts: atomicAdd
  int *verdict;         // nullable: [0] |= malformed
  int32_t n_cols;
  int32_t cta0;         // first CTA of the matrix; the next segment's cta0 (or HistBatch::cta_end) ends it
};
struct HistBatch {
  HistSeg seg[kHistSegs];
  int32_t n, cta_end;
};
__device__ __forceinline__ void hist_add(uint32_t *h, int32_t j, int32_t *g) {
  const int sh = (j & 1) << 4;
  const uint32_t old = atomicAdd(&h[j >> 1], 1u << sh);
  if (((old >> sh) & 0xffffu) == 0x7fffu) {
    // this add took the counter to 2^15: it moves 2^15 to the global count; the other threads of the CTA cannot add
    // the further 2^15 that would overflow it before the subtraction lands
    atomicAdd(&g[j], 0x8000);
    atomicSub(&h[j >> 1], 0x8000u << sh);
  }
}
__global__ void __launch_bounds__(kHistThreads) k_col_counts_smem(const HistBatch b) {
  extern __shared__ uint32_t h[];   // two 16-bit counters per word: column j in word j / 2, half j % 2
  int i = 0;
  while (i + 1 < b.n && (int)blockIdx.x >= b.seg[i + 1].cta0) ++i;
  const HistSeg &s = b.seg[i];
  const long long n_ctas = (i + 1 < b.n ? b.seg[i + 1].cta0 : b.cta_end) - s.cta0, k = blockIdx.x - s.cta0;
  const int words = (s.n_cols + 1) >> 1;
  for (int w = threadIdx.x; w < words; w += blockDim.x) h[w] = 0;
  int bad = 0;
  if (s.verdict) {
    const long long r1 = s.n_rows * (k + 1) / n_ctas;
    for (long long r = s.n_rows * k / n_ctas + threadIdx.x; r < r1; r += blockDim.x) {
      const long long a = s.rp[r], e = s.rp[r + 1];
      if (e < a || a < s.q_lo || e > s.q_hi) bad = 1;
    }
  }
  __syncthreads();
  const long long q0 = s.nnz * k / n_ctas, q1 = s.nnz * (k + 1) / n_ctas;
  constexpr int U = 8;   // loads in flight per thread
  for (long long q = q0 + threadIdx.x; q < q1; q += U * kHistThreads) {
    int32_t j[U];
#pragma unroll
    for (int u = 0; u < U; ++u) j[u] = q + u * kHistThreads < q1 ? s.col[q + u * kHistThreads] : -1;
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if ((uint32_t)j[u] < (uint32_t)s.n_cols) hist_add(h, j[u], s.counts);
      else if (q + u * kHistThreads < q1) bad = 1;   // outside [0, n_cols): skipped, reported
    }
  }
  if (__syncthreads_or(bad) && threadIdx.x == 0 && s.verdict) atomicOr(&s.verdict[0], 1);
  for (int w = threadIdx.x; w < words; w += blockDim.x) {
    const uint32_t v = h[w];
    if (v & 0xffffu) atomicAdd(&s.counts[2 * w], (int32_t)(v & 0xffffu));
    if (v >> 16) atomicAdd(&s.counts[2 * w + 1], (int32_t)(v >> 16));
  }
}

}  // namespace cco
