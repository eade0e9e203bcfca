// cco_kernels.cuh -- hand-written sm_90a kernels of the CCO train hot path.
//
// Reference semantics (what each stage replaces) -- Apache Mahout 0.13.0 SimilarityAnalysis,
// called from src/main/scala/URAlgorithm.scala:323-329,343-346 (SURVEY.md 8a):
//   input validation           -> k_check_rows; canonicalisation slow path k_expand_keys / k_unique_* / k_rowptr_from_keys
//   H2 sampleDownAndBinarize   -> k_downsample_count / k_downsample_write (row ranges: whole matrix or a rank's user block)
//   H3 numNonZeroElementsPerColumn -> k_col_histogram (raw, before the allreduce), k_downsample_count or
//                                 k_col_histogram_u32 (post-sample)
//   `drmA.t`                   -> k_transpose_entries (cco_sampler.cuh)
//   scheduling                 -> k_row_work, k_bin_bounds, k_partition_rows; column order of B' k_col_order_init /
//                                 k_col_order / k_relabel_cols; per-column LLR constants k_col_terms
//   H4 A'^T B' counts, H5 LLR, H6 top-k -> k_rows<GROUP, DENSE> (one fused kernel, nothing materialised)
//   result assembly            -> k_len_to_i64, k_compact_rows; small device->host results k_mail_bytes
//
// Everything here is integer/byte work plus scalar fp64; no tensor cores (DESIGN.md 3.2).  The accumulator, the
// candidate buffer, the select histogram and the LLR tables of a row live in shared memory; B' and the per-column
// terms are gathered from L2/HBM.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace cco {

// ------------------------------------------------------------------------------------------------
// device views
// ------------------------------------------------------------------------------------------------
struct RowArgs {
  // A'^T: users of every primary item
  const uint32_t *at_ptr;
  const int32_t *at_users;
  // B' (CSR over users)
  const uint32_t *b_ptr;
  const int32_t *b_col;   // column KEYS (k_col_order): B' relabelled by the order (colB ascending, column id ascending)
  const int32_t *marg_a;  // colA, downsampled, per primary item
  const int32_t *marg_b;  // colB, downsampled, per column key (ascending)
  const int32_t *key_of_col;       // column id -> key (the diagonal of A'^T A')
  const int32_t *first_key_of_cb;  // [c] = first key whose colB >= c, for c in [0, max_marg_b + 1]
  int32_t key_shift;      // (n_cols_b - 1) >> key_shift < kCutBins: first level of the key cut
  const uint2 *ext;       // experiment (tools/experiments/cco_rows2.cuh): (start, len) of B'[u] per (item, user) pair; unused
  int32_t max_marg_b;     // largest colB (bounds every co-occurrence count together with rowA)
  // schedule: items sorted by estimated work, descending; bin b = rows_sorted[bin_bounds[b], bin_bounds[b+1])
  const int32_t *rows_sorted;
  const uint32_t *row_work;  // by item: w_a = sum_{u in a} degB'(u), saturated at 2^32-1
  const int32_t *bin_bounds;
  int32_t bin;
  int32_t n_cols_b;
  long long n_users;  // N
  int32_t self;       // A'^T A': skip the diagonal
  int32_t top_k;
  int32_t has_min_llr;
  double min_llr;
  int32_t cut_ok;    // the level-1 cut is exact for the computed LLRs at this (N, max rowA, max colB): cut_exact (cco_api.cu)
  double llr_eps2;   // 2 eps: eps bounds |computed - real| of one fp64 LLR at this N (llr_error_bound, cco_api.cu)
  uint32_t flags;
  int32_t count_bits;  // packed hash word = (key << count_bits) | count
  int32_t slots;       // hash/dense table words in shared memory
  int32_t cap;         // max distinct keys per pass for hashed rows (load-factor bound)
  int32_t tsize_x16;   // table words per expected distinct key, in sixteenths (32 = load factor 1/2)
  int32_t cbuf;        // candidate buffer entries per group (power of two, >= top_k + GROUP)
  int32_t caux;        // scratch entries for the out-of-place compaction of the radix select (0 for warps)
  int32_t keep_max;    // M: a prune keeps between top_k and max(M, top_k) candidates
  int32_t final_max;   // the final sort runs on at most this many candidates (next_pow2(top_k))
  int32_t group_smem_bytes;  // shared memory of one group (multiple of 16)
  const struct ColTerm *col_terms;  // per column key: {columnEntropy, xLogX(colB - 1), colB, column id}
  // outputs, strided
  int32_t out_stride;
  int32_t *out_col;
  double *out_llr;
  int32_t *out_cnt;
  int32_t *out_len;
  unsigned long long *stat_distinct;
  unsigned long long *stat_evaluated;  // cells whose fp64 LLR was actually evaluated (after the dominance filter)
  int *err_flag;     // set to 1 if a hash table overflowed (result invalid)
  int32_t emit_all;  // debug: write every non-zero cell (col,count), no LLR/top-k
  int32_t bm_words;  // bitmap rows (k_rows<..., BITMAP>): words of the key bitmap, ceil(n_cols_b / 32); else 0
  int32_t key_base;  // key ranges (DESIGN.md 3.1): first global key of this view; its keys are key_of_col - key_base
};

constexpr uint32_t kEmpty = 0xffffffffu;

__device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z ^= z >> 30;
  z *= 0xbf58476d1ce4e5b9ULL;
  z ^= z >> 27;
  z *= 0x94d049bb133111ebULL;
  z ^= z >> 31;
  return z;
}
// sampler of include/cco_b200.h "Sampler" (bit-identical to oracle/cco_oracle.c orc_hash64/orc_u01)
__device__ __forceinline__ double sample_u01(int32_t seed, uint32_t u, uint32_t j) {
  uint64_t x = mix64(((uint64_t)(uint32_t)seed << 32) | (uint64_t)u);
  uint64_t h = mix64(x + (uint64_t)j * 0x9e3779b97f4a7c15ULL);
  return __dmul_rn((double)(h >> 11), 0x1.0p-53);
}
__device__ __forceinline__ uint32_t hash32(uint32_t x) {
  x ^= x >> 16;
  x *= 0x7feb352dU;
  x ^= x >> 15;
  x *= 0x846ca68bU;
  x ^= x >> 16;
  return x;
}

// ------------------------------------------------------------------------------------------------
// LogLikelihood (Mahout mahout-math LogLikelihood.java; SURVEY.md A.3).  __dmul_rn/__dsub_rn keep
// nvcc from contracting x*log(x) - ... into FMAs so the evaluation order matches the JVM's.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double xlogx(long long x) {
  return x == 0 ? 0.0 : __dmul_rn((double)x, log((double)x));
}
// counts inside the row kernel are < 2^31 (n_rows < 2^31 is validated): the 32-bit conversion is exact and cheaper
__device__ __forceinline__ double xlogx_u32(uint32_t x) {
  return x == 0 ? 0.0 : __dmul_rn((double)x, log((double)x));
}
__device__ __forceinline__ double entropy2(long long a, long long b, bool varargs) {
  if (varargs) return __dsub_rn(xlogx(a + b), __dadd_rn(__dadd_rn(0.0, xlogx(a)), xlogx(b)));
  return __dsub_rn(__dsub_rn(xlogx(a + b), xlogx(a)), xlogx(b));
}
__device__ __forceinline__ double entropy4(long long a, long long b, long long c, long long d, bool varargs) {
  if (varargs) {
    double r = __dadd_rn(__dadd_rn(__dadd_rn(__dadd_rn(0.0, xlogx(a)), xlogx(b)), xlogx(c)), xlogx(d));
    return __dsub_rn(xlogx(a + b + c + d), r);
  }
  return __dsub_rn(__dsub_rn(__dsub_rn(__dsub_rn(xlogx(a + b + c + d), xlogx(a)), xlogx(b)), xlogx(c)), xlogx(d));
}
__device__ __forceinline__ double llr_cells(long long k11, long long k12, long long k21, long long k22, bool varargs) {
  double row_e = entropy2(k11 + k12, k21 + k22, varargs);
  double col_e = entropy2(k11 + k21, k12 + k22, varargs);
  double mat_e = entropy4(k11, k12, k21, k22, varargs);
  double s = __dadd_rn(row_e, col_e);
  if (s < mat_e) return 0.0;  // round off error
  return __dmul_rn(2.0, __dsub_rn(s, mat_e));
}

__global__ void k_debug_llr(long long n, const long long *k11, const long long *k12, const long long *k21,
                            const long long *k22, uint32_t flags, double *out) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) out[i] = llr_cells(k11[i], k12[i], k21[i], k22[i], (flags & CCO_FLAG_ENTROPY_VARARGS) != 0);
}

// ------------------------------------------------------------------------------------------------
// Row-parallel passes over a CSR matrix: SG lanes cooperate on one user row.
// ------------------------------------------------------------------------------------------------
constexpr int kSG = 8;  // lanes per user row in the preparation passes (avg row ~10-30 entries)

// Row-parallel passes give a row to a sub-group of kSG lanes.  A user with thousands of entries would keep one sub-group
// busy long after the rest of the grid has drained (Zipf users: the top row of C3 has ~6 K entries, of C4 ~40 K) -- and
// that tail does not shrink when the users are sharded over GPUs.  Rows above kHeavyRow entries are therefore listed once
// (k_list_heavy_rows) and handled by a second launch of the same kernel with a whole warp per listed row.
constexpr int kHeavyRow = 256;
__global__ void k_list_heavy_rows(long long n_rows, const long long *__restrict__ rp, int32_t *__restrict__ list, int *__restrict__ n_list) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < n_rows; r += (long long)gridDim.x * blockDim.x)
    if (rp[r + 1] - rp[r] > kHeavyRow) list[atomicAdd(n_list, 1)] = (int32_t)r;
}
// the rows one launch walks: every light row (list == nullptr) or the listed heavy ones
#define CCO_ROW_LOOP_BEGIN(SG)                                                                         \
  const int lane = threadIdx.x % SG;                                                                   \
  long long it = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / SG;                              \
  const long long stride = (long long)gridDim.x * blockDim.x / SG;                                     \
  const long long n_it = list ? (long long)*n_list : n_rows;                                           \
  for (; it < n_it; it += stride) {                                                                    \
    const long long row = list ? (long long)list[it] : it;
#define CCO_ROW_LOOP_END }

// flags[0] |= malformed (row_ptr not monotone / outside [q_lo, q_hi] / column out of range), flags[1] |= not canonical
template <int SG>
__global__ void k_check_rows(long long n_rows, int32_t n_cols, const long long *__restrict__ rp, const int32_t *__restrict__ col,
                             long long q_lo, long long q_hi, const int32_t *__restrict__ list, const int *__restrict__ n_list, int *flags) {
  int bad = 0, unsorted = 0;
  CCO_ROW_LOOP_BEGIN(SG)
    long long s = rp[row], e = rp[row + 1];
    if (e < s || s < q_lo || e > q_hi) { bad = 1; continue; }   // never dereference an offset outside the uploaded block
    if (!list && e - s > kHeavyRow) continue;
    for (long long q = s + lane; q < e; q += SG) {
      int32_t c = col[q];
      if (c < 0 || c >= n_cols) bad = 1;
      if (q > s && col[q - 1] >= c) unsorted = 1;
    }
  CCO_ROW_LOOP_END
  if (bad) atomicOr(&flags[0], 1);
  if (unsorted) atomicOr(&flags[1], 1);
}

// raw column counts c_j of rows [row_begin,row_end) (numNonZeroElementsPerColumn of the raw matrix)
// The counters are REPLICATED (n_copies arrays, copy_stride apart, chosen by CTA): with Zipf-skewed items 8 % of all
// entries hit one column, and its atomics serialise in one L2 slice;
// k_sum_copies folds the copies back into copy 0.
__global__ void k_col_histogram(long long row_begin, long long row_end, const long long *__restrict__ rp,
                                const int32_t *__restrict__ col, int32_t n_cols, int32_t *__restrict__ counts, int n_copies,
                                long long copy_stride) {
  // element-parallel over the contiguous slice rp[row_begin]..rp[row_end]; warp-uniform trip count
  const long long s = rp[row_begin], e = rp[row_end];
  const int lane = threadIdx.x & 31;
  int32_t *mine = counts + (long long)(blockIdx.x % n_copies) * copy_stride;
  for (long long q0 = s + blockIdx.x * (long long)blockDim.x + (threadIdx.x & ~31); q0 < e;
       q0 += (long long)gridDim.x * blockDim.x) {
    const long long q = q0 + lane;
    const bool act = q < e;
    const unsigned am = __ballot_sync(0xffffffffu, act);
    if (act) {
      int32_t c = col[q];
      // warp-aggregate lanes hitting the same column (Zipf-hot columns)
      unsigned peers = __match_any_sync(am, c);
      // (an out-of-range id of a not yet validated matrix is skipped here and reported by k_check_rows)
      if ((__ffs(peers) - 1) == lane && (uint32_t)c < (uint32_t)n_cols) atomicAdd(&mine[c], __popc(peers));
    }
  }
}
__global__ void k_sum_copies(long long n, int n_copies, long long copy_stride, int32_t *__restrict__ counts) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int32_t acc = counts[i];
    for (int k = 1; k < n_copies; ++k) acc += counts[i + k * copy_stride];
    counts[i] = acc;
  }
}

// column histogram of the entries [*lo, *hi) of a column-index array (bounds read on the device, 32-bit offsets)
__global__ void k_col_histogram_u32(const uint32_t *__restrict__ lo, const uint32_t *__restrict__ hi,
                                    const int32_t *__restrict__ col, int32_t *__restrict__ counts) {
  const long long s = *lo, e = *hi;
  const int lane = threadIdx.x & 31;
  for (long long q0 = s + blockIdx.x * (long long)blockDim.x + (threadIdx.x & ~31); q0 < e;
       q0 += (long long)gridDim.x * blockDim.x) {
    const long long q = q0 + lane;
    const bool act = q < e;
    const unsigned am = __ballot_sync(0xffffffffu, act);
    if (act) {
      const int32_t c = col[q];
      const unsigned peers = __match_any_sync(am, c);
      if ((__ffs(peers) - 1) == lane) atomicAdd(&counts[c], __popc(peers));
    }
  }
}

__device__ __forceinline__ double row_sample_rate(long long d, int32_t m, bool intdiv) {
  if (d <= 0) return 1.0;
  const long long md = d < m ? d : (long long)m;
  return intdiv ? (double)(md / d) : __ddiv_rn((double)md, (double)d);
}
// The sampler keeps (u, j) iff u01 <= min(rowRate, colRate) with u01 = (h >> 11) * 2^-53 (include/cco_b200.h "Sampler";
// bit-identical to oracle/cco_oracle.c orc_downsample).  u01 is a 53-bit integer scaled by a power of two, so the
// comparison is exactly  (h >> 11) <= floor(rate * 2^53): rates become integer thresholds -- one per column (k_col_thresholds,
// once per train) and one per row -- and an entry costs one mix64 and one integer compare, no fp64 division.  A rate of
// 1 (row and column within m) gets the threshold 2^53: u01 < 1 always passes, the hash is not even computed.
constexpr unsigned long long kKeepAlways = 1ULL << 53;
__device__ __forceinline__ unsigned long long rate_threshold(double rate) {
  if (rate >= 1.0) return kKeepAlways;
  return (unsigned long long)floor(__dmul_rn(rate, 0x1.0p53));   // exact: a power-of-two scaling, then the integer part
}
__global__ void k_col_thresholds(int32_t n_cols, const int32_t *__restrict__ raw_counts, int32_t m, unsigned long long *__restrict__ thr) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n_cols; j += gridDim.x * blockDim.x) {
    const int32_t c = raw_counts[j];
    thr[j] = c <= m ? kKeepAlways : rate_threshold(__ddiv_rn((double)m, (double)c));
  }
}
__device__ __forceinline__ bool keep_entry_thr(unsigned long long t_row, unsigned long long t_col, uint64_t x_row, uint32_t j) {
  const unsigned long long t = t_row < t_col ? t_row : t_col;
  if (t >= kKeepAlways) return true;
  const uint64_t h = mix64(x_row + (uint64_t)j * 0x9e3779b97f4a7c15ULL);
  return (h >> 11) <= t;
}

// pass 1 of sampleDownAndBinarize: kept entries per row + post-sample column marginals.
// The matrix handed in is a block of n_rows user rows (the whole matrix on one GPU, this rank's user block otherwise);
// row_base = global index of its first user: the sampler hashes GLOBAL user ids and kept_per_row is indexed globally.
template <int SG>
__global__ void k_downsample_count(long long n_rows, long long row_base, const long long *__restrict__ rp, const int32_t *__restrict__ col,
                                   int32_t n_cols, long long q_lo, long long q_hi, const unsigned long long *__restrict__ col_thr, int32_t m,
                                   int32_t seed, uint32_t flags, const int32_t *__restrict__ list, const int *__restrict__ n_list,
                                   uint32_t *__restrict__ kept_per_row, int32_t *__restrict__ new_counts, uint8_t *__restrict__ keep_flag) {
  const unsigned sg_mask = SG == 32 ? 0xffffffffu : (((1u << SG) - 1u) << ((threadIdx.x & 31) / SG * SG));
  const bool intdiv = (flags & CCO_FLAG_ROWRATE_INTDIV) != 0;
  // all lanes of a sub-group share `row`, so loop trip counts are sub-group uniform
  CCO_ROW_LOOP_BEGIN(SG)
    long long s = rp[row], e = rp[row + 1], d = e - s;
    if (!list && d > kHeavyRow) continue;
    if (d < 0 || s < q_lo || e > q_hi) continue;   // malformed row_ptr: k_check_rows reports it
    const unsigned long long t_row = rate_threshold(row_sample_rate(d, m, intdiv));
    const uint32_t g = (uint32_t)(row_base + row);
    const uint64_t x_row = mix64(((uint64_t)(uint32_t)seed << 32) | (uint64_t)g);
    uint32_t kept = 0;
    for (long long q0 = s; q0 < e; q0 += SG) {
      long long q = q0 + lane;
      bool keep = false;
      int32_t j = 0;
      if (q < e) {
        j = col[q];
        // (ids outside [0, n_cols) belong to a malformed matrix: dropped here, reported by k_check_rows)
        keep = (uint32_t)j < (uint32_t)n_cols && keep_entry_thr(t_row, col_thr[j], x_row, (uint32_t)j);
        keep_flag[q - q_lo] = keep ? 1 : 0;   // pass 2 compacts by these decisions instead of hashing again
      }
      if (keep && new_counts) atomicAdd(&new_counts[j], 1);
      kept += __popc(__ballot_sync(sg_mask, keep) & sg_mask);
    }
    if (lane == 0) kept_per_row[g] = kept;
  CCO_ROW_LOOP_END
}

// pass 2: ordered compaction by the recorded decisions (ascending columns are preserved).  new_ptr is the GLOBAL row
// pointer of the sampled matrix; out_base (nullable) points at the entry the output buffer starts at (this rank's block
// offset when the block is written into a send buffer, null = 0 when it is written in place).
template <int SG>
__global__ void k_downsample_write(long long n_rows, long long row_base, const long long *__restrict__ rp, const int32_t *__restrict__ col,
                                   long long q_lo, long long q_hi, const uint8_t *__restrict__ keep_flag,
                                   const int32_t *__restrict__ list, const int *__restrict__ n_list,
                                   const uint32_t *__restrict__ new_ptr, const uint32_t *__restrict__ out_base, int32_t *__restrict__ new_col) {
  const int sg_shift = SG == 32 ? 0 : (threadIdx.x & 31) / SG * SG;
  const unsigned sg_mask = SG == 32 ? 0xffffffffu : (((1u << SG) - 1u) << sg_shift);
  const uint32_t base = out_base ? *out_base : 0u;
  CCO_ROW_LOOP_BEGIN(SG)
    long long s = rp[row], e = rp[row + 1], d = e - s;
    if (!list && d > kHeavyRow) continue;
    if (d < 0 || s < q_lo || e > q_hi) continue;
    uint32_t w = new_ptr[row_base + row] - base;
    for (long long q0 = s; q0 < e; q0 += SG) {
      long long q = q0 + lane;
      bool keep = false;
      int32_t j = 0;
      if (q < e) {
        j = col[q];
        keep = keep_flag[q - q_lo] != 0;
      }
      unsigned b = (__ballot_sync(sg_mask, keep) & sg_mask) >> sg_shift;
      if (keep) new_col[w + __popc(b & ((1u << lane) - 1u))] = j;
      w += __popc(b);
    }
  CCO_ROW_LOOP_END
}

// multi-GPU: every rank sampled its user block into a padded send buffer; after the all-gather the W padded blocks
// (cap entries apart) are packed into the contiguous column array of the sampled matrix.  Block q holds users
// [q * S, min((q + 1) * S, U)): its length is new_ptr[end] - new_ptr[begin], read here -- no host round trip.
__global__ void k_pack_blocks(int world, long long S, long long U, long long cap, const uint32_t *__restrict__ new_ptr,
                              const int32_t *__restrict__ gathered, int32_t *__restrict__ new_col) {
  for (int q = blockIdx.y; q < world; q += gridDim.y) {
    const long long u0 = min((long long)q * S, U), u1 = min(u0 + S, U);
    const uint32_t lo = new_ptr[u0], hi = new_ptr[u1];
    const int32_t *src = gathered + (long long)q * cap;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < hi - lo; i += gridDim.x * blockDim.x) new_col[lo + i] = src[i];
  }
}

// w_a = sum over users of item a of degB'(u)  (= products of output row a), saturating; also P
__global__ void k_row_work(int32_t n_items, const uint32_t *__restrict__ at_ptr, const int32_t *__restrict__ at_users,
                           const uint32_t *__restrict__ b_ptr, uint32_t *__restrict__ row_work,
                           unsigned long long *__restrict__ work64, int32_t *__restrict__ item_ids,
                           uint2 *__restrict__ ext) {
  const int lane = threadIdx.x % kSG;
  const unsigned sg_mask = ((1u << kSG) - 1u) << ((threadIdx.x & 31) / kSG * kSG);
  int item = (blockIdx.x * blockDim.x + threadIdx.x) / kSG;
  const int stride = gridDim.x * blockDim.x / kSG;
  for (; item < n_items; item += stride) {
    uint32_t s = at_ptr[item], e = at_ptr[item + 1];
    unsigned long long w = 0;
    for (uint32_t q = s + lane; q < e; q += kSG) {
      int32_t u = at_users[q];
      const uint32_t bs = b_ptr[u], bl = b_ptr[u + 1] - bs;
      w += bl;
      if (ext) ext[q] = make_uint2(bs, bl);   // the row kernel streams these instead of gathering b_ptr twice per user
    }
#pragma unroll
    for (int o = kSG / 2; o > 0; o >>= 1) w += __shfl_xor_sync(sg_mask, w, o);
    if (lane == 0) {
      row_work[item] = w > 0xffffffffULL ? 0xffffffffu : (uint32_t)w;
      work64[item] = w;
      item_ids[item] = item;
    }
  }
}

// bin boundaries inside the work-descending row list: bin b holds rows whose distinct-cell bound
// D = min(w, n_cols_b) satisfies thresholds[b-1] >= D > thresholds[b]  (thresholds descending)
struct BinThresholds {
  uint32_t t[12];  // by value in the launch parameters: no host->device copy, no host sync
};
__global__ void k_bin_bounds(int32_t n_rows, const uint32_t *__restrict__ sorted_work, int32_t n_bins,
                             const BinThresholds thresholds, int32_t *__restrict__ bounds) {
  int b = threadIdx.x;
  if (b > n_bins) return;
  if (b == 0) { bounds[0] = 0; return; }
  // first index whose work <= thresholds[b-1]  (sorted descending).  The last bin ends at the first row WITHOUT work:
  // rows of other ranks (masked to zero by k_mask_work) and empty rows need no kernel, their out_len is preset to 0.
  uint32_t t = b == n_bins ? 0u : thresholds.t[b - 1];
  int lo = 0, hi = n_rows;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (sorted_work[mid] > t) lo = mid + 1; else hi = mid;
  }
  bounds[b] = lo;
}

// ------------------------------------------------------------------------------------------------
// Per-column constants of B' for the fused LLR: columnEntropy = entropy(cb, N - cb) depends only on the
// column, so it is evaluated once per column (same operations, same bits) instead of once per cell.
// ------------------------------------------------------------------------------------------------
struct __align__(16) ColTerm {
  double col_e;     // entropy(cb, N - cb)
  double x_cbm1;    // xLogX(cb - 1): the k21 term of every k11 == 1 cell of this column
  int32_t cb;
  int32_t col;      // original column id (what the output rows hold)
  int32_t pad[2];
};
// terms in key order: marg_key[k] = colB and col_of_key[k] = column id of key k (k_col_order)
__global__ void k_col_terms(int32_t n_cols, const int32_t *__restrict__ marg_key, const int32_t *__restrict__ col_of_key,
                            long long n_users, uint32_t flags, ColTerm *__restrict__ out) {
  const bool varargs = (flags & CCO_FLAG_ENTROPY_VARARGS) != 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_cols; i += gridDim.x * blockDim.x) {
    long long cb = marg_key[i];
    ColTerm t;
    t.col_e = entropy2(cb, n_users - cb, varargs);
    t.x_cbm1 = cb >= 1 ? xlogx(cb - 1) : 0.0;
    t.cb = (int32_t)cb;
    t.col = col_of_key[i];
    t.pad[0] = t.pad[1] = 0;
    out[i] = t;
  }
}

// ---- column order of B' (DESIGN.md 3.1, step 3) -------------------------------------------------------------------
// key = rank of a column under (colB ascending, column id ascending).  k_col_order_init writes the (colB, id) pairs a
// stable radix sort by colB turns into marg_key / col_of_key; k_col_order inverts the permutation and tabulates the
// first key of every colB value.
__global__ void k_col_order_init(int32_t n_cols, const int32_t *__restrict__ marg, uint32_t *__restrict__ cb_out,
                                 int32_t *__restrict__ id_out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_cols; i += gridDim.x * blockDim.x) {
    cb_out[i] = (uint32_t)marg[i];
    id_out[i] = i;
  }
}
__global__ void k_col_order(int32_t n_cols, int32_t max_cb, const uint32_t *__restrict__ marg_key, const int32_t *__restrict__ col_of_key,
                            int32_t *__restrict__ key_of_col, int32_t *__restrict__ first_key_of_cb) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n_cols; k += gridDim.x * blockDim.x) {
    key_of_col[col_of_key[k]] = k;
    // key k is the first key of every colB value in (marg_key[k - 1], marg_key[k]]; the last key also closes the table
    const int32_t cb = (int32_t)marg_key[k], lo = k == 0 ? 0 : (int32_t)marg_key[k - 1] + 1;
    for (int32_t c = lo; c <= cb; ++c) first_key_of_cb[c] = k;
    if (k == n_cols - 1)
      for (int32_t c = cb + 1; c <= max_cb + 1; ++c) first_key_of_cb[c] = n_cols;
  }
}
// B' column ids -> keys, in place; the entry count is read on the device (*end = row_ptr[U])
__global__ void k_relabel_cols(const uint32_t *__restrict__ end, const int32_t *__restrict__ key_of_col, int32_t *__restrict__ col) {
  const long long n = *end;
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x)
    col[q] = key_of_col[col[q]];
}

// ------------------------------------------------------------------------------------------------
// The fused row kernel.  A GROUP of threads (one warp, or a whole CTA of 256 / 1024 threads) owns one
// primary item a at a time and keeps everything for that row in shared memory:
//   count  : for u in users(a): for b in B'[u]: table[b]++     products flattened over lanes by a prefix sum +
//                                                               shuffle search; CTA-owned rows split them evenly over warps
//   compact: occupied table words -> dense per-warp lists (in place)
//   score  : LLR(k11, colA[a], colB[b], N) in fp64, in registers, 2 logs per cell (the other xLogX terms
//            are per-row / per-column / small-integer tables holding bit-identical values)
//   select : running top-k under the total order (llr desc, col asc): threshold-pruned candidate buffer
// DENSE: table indexed by b directly (n_cols_b <= slots); otherwise a packed open-addressing hash
// (key << count_bits | count), multi-pass over hash partitions when the row's distinct-cell bound
// exceeds the table capacity.  Nothing of A'^T B' is ever written to HBM except the kept top-k.
// ------------------------------------------------------------------------------------------------
// candidate entry, 16 bytes so that the sort moves it with one LDS.128 / STS.128:
//   x,y = low/high word of the fp64 LLR bit pattern (positive doubles order like unsigned integers),
//   z = column, w = k11
__device__ __forceinline__ bool cand_better(const uint4 &p, const uint4 &q) {
  return p.y > q.y || (p.y == q.y && (p.x > q.x || (p.x == q.x && p.z < q.z)));
}

template <int GROUP>
__device__ __forceinline__ void group_sync() {
  if (GROUP == 32) __syncwarp(); else __syncthreads();
}

// bitonic sort of the candidate buffer, best first; pads [n, n2) with key 0 (never valid: LLR > 0)
template <int GROUP>
__device__ void sort_candidates(uint4 *tk, int n, int gtid) {
  int n2 = 1;
  while (n2 < n) n2 <<= 1;
  for (int i = n + gtid; i < n2; i += GROUP) tk[i] = make_uint4(0u, 0u, 0xffffffffu, 0u);
  group_sync<GROUP>();
  for (int k2 = 2; k2 <= n2; k2 <<= 1) {
    for (int j = k2 >> 1; j > 0; j >>= 1) {
      for (int t = gtid; t < (n2 >> 1); t += GROUP) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
        const int p = i | j;
        const bool up = (i & k2) == 0;
        const uint4 ei = tk[i], ep = tk[p];
        const bool swap = up ? cand_better(ep, ei) : cand_better(ei, ep);
        if (swap) { tk[i] = ep; tk[p] = ei; }
      }
      group_sync<GROUP>();
    }
  }
}

// ---- candidate reduction: MSB-first 8-bit radix select on the composite key (llr hi, llr lo, ~col) ----------
// Keeps every candidate >= a threshold T chosen so that  top_k <= kept <= max(M, top_k)  (exactly top_k when the
// key is fully resolved; keys are unique because columns are).  Cost: a few histogram passes over the buffer
// instead of a full sort.  Returns the kept count; the threshold entry goes to thr (same layout as a candidate).
__device__ __forceinline__ uint32_t cand_word(const uint4 &e, int wi) { return wi == 0 ? e.y : (wi == 1 ? e.x : ~e.z); }

template <int GROUP>
__device__ int reduce_candidates(uint4 *tk, uint4 *aux, int n, int k, int M, int *hist, int *ctrl, int gtid) {
  // ctrl[16..18] = prefix words, ctrl[24] = D, ctrl[25] = c_gt, ctrl[26] = c_D, ctrl[27] = output cursor
  volatile int *vc = ctrl;
  uint32_t pre0 = 0u, pre1 = 0u, pre2 = 0u;
  int nb = 0, above = 0, kept = n;
  while (true) {
    for (int i = gtid; i < 256; i += GROUP) hist[i] = 0;
    group_sync<GROUP>();
    const int wi = nb >> 5, sh = 24 - (nb & 31);
    for (int i = gtid; i < n; i += GROUP) {
      const uint4 e = tk[i];
      const uint32_t w0 = e.y, w1 = e.x, w2 = ~e.z;
      bool match;
      if (nb == 0) match = true;
      else if (nb < 32) match = (w0 >> (32 - nb)) == (pre0 >> (32 - nb));
      else if (nb == 32) match = w0 == pre0;
      else if (nb < 64) match = w0 == pre0 && (w1 >> (64 - nb)) == (pre1 >> (64 - nb));
      else if (nb == 64) match = w0 == pre0 && w1 == pre1;
      else match = w0 == pre0 && w1 == pre1 && (w2 >> (96 - nb)) == (pre2 >> (96 - nb));
      // digit = byte (sh / 8) of the key word, extracted with PRMT: ptxas 12.9 turned `(word >> 24) & 255` of the
      // peeled nb == 0 pass into an index by the WHOLE word in one inlining context (compute-sanitizer: invalid shared atomic)
      if (match) atomicAdd(&hist[__byte_perm(cand_word(e, wi), 0u, 0x4440u | (uint32_t)(sh >> 3))], 1);
    }
    group_sync<GROUP>();
    if (gtid < 32) {
      // lane l owns digits 255-8l .. 248-8l (descending); find the digit holding the (k-above)-th best
      int c[8], ssum = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) { c[j] = hist[255 - 8 * gtid - j]; ssum += c[j]; }
      int incl = ssum;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, d);
        if (gtid >= d) incl += v;
      }
      const int excl = incl - ssum, need = k - above;
      if (excl < need && need <= incl) {
        int run = excl;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (run < need && run + c[j] >= need) { ctrl[24] = 255 - 8 * gtid - j; ctrl[25] = run; ctrl[26] = c[j]; }
          run += c[j];
        }
      }
    }
    group_sync<GROUP>();
    const int D = vc[24], c_gt = vc[25], c_d = vc[26];
    if (wi == 0) pre0 |= (uint32_t)D << sh; else if (wi == 1) pre1 |= (uint32_t)D << sh; else pre2 |= (uint32_t)D << sh;
    nb += 8;
    kept = above + c_gt + c_d;
    if (kept <= M || nb == 96) break;
    above += c_gt;
    group_sync<GROUP>();
  }
  // keep e iff key(e) >= prefix (low bits zero)
  if (gtid == 0) ctrl[27] = 0;
  group_sync<GROUP>();
  if (GROUP == 32) {
    // single warp: in-place batch compaction (reads of a batch complete before its writes)
    int w = 0;
    for (int i0 = 0; i0 < n; i0 += 32) {
      const int i = i0 + gtid;
      uint4 e = make_uint4(0u, 0u, 0u, 0u);
      bool keep = false;
      if (i < n) {
        e = tk[i];
        const uint32_t w0 = e.y, w1 = e.x, w2 = ~e.z;
        keep = w0 > pre0 || (w0 == pre0 && (w1 > pre1 || (w1 == pre1 && w2 >= pre2)));
      }
      const unsigned m = __ballot_sync(0xffffffffu, keep);
      __syncwarp();
      if (keep) tk[w + __popc(m & ((1u << gtid) - 1u))] = e;
      w += __popc(m);
      __syncwarp();
    }
  } else {
    for (int i = gtid; i < n; i += GROUP) {
      const uint4 e = tk[i];
      const uint32_t w0 = e.y, w1 = e.x, w2 = ~e.z;
      const bool keep = w0 > pre0 || (w0 == pre0 && (w1 > pre1 || (w1 == pre1 && w2 >= pre2)));
      if (keep) aux[atomicAdd(&ctrl[27], 1)] = e;
    }
    group_sync<GROUP>();
    for (int i = gtid; i < kept; i += GROUP) tk[i] = aux[i];
  }
  if (gtid == 0) {
    ctrl[0] = kept;
    ctrl[4] = (int)pre1; ctrl[5] = (int)pre0; ctrl[6] = (int)~pre2; ctrl[7] = 0;  // threshold as a candidate entry
    ctrl[1] = 1;
  }
  group_sync<GROUP>();
  return kept;
}

constexpr int kCutBins = 512;   // level-1 integer cut: u16 colB bins; they alias the 1 KB radix-select histogram (dead until the score loop)
constexpr int kDomLevels = 15;  // dominance filter keeps cfail[1..15] in ctrl[41..55]
constexpr int kX12N = 31;  // x12tab[j] = xLogX(ra - j) for j < 31; x12tab[31] = xLogX(N - ra)

// One warp: the smallest of the kCutBins u16 bins of h1 at which the running count reaches `need` -> ctrl[9]
// (0x7fffffff if the bins hold fewer cells), and the cells in the bins below it -> ctrl[10].
__device__ __forceinline__ void cut_find(const uint32_t *h1, uint32_t need, int lane, int *ctrl) {
  // lane l owns bins [16 l, 16 l + 16): 8 words
  uint32_t sum = 0;
  for (int wi = 0; wi < 8; ++wi) { const uint32_t v = h1[lane * 8 + wi]; sum += (v & 0xffffu) + (v >> 16); }
  uint32_t incl = sum;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += v;
  }
  const uint32_t excl = incl - sum;
  int found = 0x7fffffff;
  uint32_t below = 0;
  if (excl < need && incl >= need) {
    uint32_t run = excl;
    for (int wi = 0; wi < 8; ++wi) {
      const uint32_t v = h1[lane * 8 + wi];
      if (run + (v & 0xffffu) >= need) { found = lane * 16 + 2 * wi; below = run; break; }
      run += v & 0xffffu;
      if (run + (v >> 16) >= need) { found = lane * 16 + 2 * wi + 1; below = run; break; }
      run += v >> 16;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {   // at most one lane found the bin
    found = min(found, __shfl_xor_sync(0xffffffffu, found, o));
    below = max(below, __shfl_xor_sync(0xffffffffu, below, o));
  }
  if (lane == 0) { ctrl[9] = found; ctrl[10] = (int)below; }
}

template <int GROUP, bool DENSE>
__device__ __forceinline__ void accumulate(uint32_t *table, uint32_t tsize, uint32_t b, int cbits, uint32_t n_pass,
                                           uint32_t pass, int *err_flag) {
  if (DENSE) {
    atomicAdd(&table[b], 1u);
    return;
  }
  if (n_pass > 1 && ((b * 0x85ebca6bu) >> 12) % n_pass != pass) return;
  uint32_t slot = __umulhi(b * 0x9e3779b1u, tsize);
  const uint32_t want = b << cbits;
  uint32_t probes = 0;
  while (true) {
    const uint32_t w = *reinterpret_cast<volatile uint32_t *>(&table[slot]);
    if ((w >> cbits) == b && w != kEmpty) { atomicAdd(&table[slot], 1u); return; }
    if (w == kEmpty) {
      const uint32_t old = atomicCAS(&table[slot], kEmpty, want | 1u);
      if (old == kEmpty) return;
      if ((old >> cbits) == b) { atomicAdd(&table[slot], 1u); return; }
    }
    slot = (slot + 1 == tsize) ? 0 : slot + 1;
    if (++probes > tsize) { atomicOr(err_flag, 1); return; }
  }
}

// Count the products [p_lo, p_hi) of a window of up to 32 users held in registers: lane l holds user l's first product
// index `off` (non-decreasing over the lanes, lane 0's <= p_lo; unused lanes hold 0xffffffff) and the start `s` of its
// B' row.  Each lane finds the user of its product by a 5-step shuffle search, then gathers the column.
// BITMAP: the first product of a cell sets its bit in `seen`; only the later products of a cell reach the hash table, which
// so holds k11 - 1 for exactly the cells with k11 >= 2.
template <int GROUP, bool DENSE, bool BITMAP>
__device__ __forceinline__ void count_window(const RowArgs &a, uint32_t *table, uint32_t *seen, uint32_t tsize, int cbits,
                                             uint32_t n_pass, uint32_t pass, uint32_t off, uint32_t s, uint32_t p_lo,
                                             uint32_t p_hi, int lane) {
  for (uint32_t p0 = p_lo; p0 < p_hi; p0 += 64) {
    // two products per lane per trip (two independent gathers in flight)
    uint32_t bb[2];
    bool act[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t p = p0 + h * 32 + lane;
      int j = 0;
#pragma unroll
      for (int st = 16; st > 0; st >>= 1) {
        const int c = j + st;
        const uint32_t v = __shfl_sync(0xffffffffu, off, c);
        if (v <= p) j = c;
      }
      const uint32_t sj = __shfl_sync(0xffffffffu, s, j), oj = __shfl_sync(0xffffffffu, off, j);
      act[h] = p < p_hi;
      bb[h] = act[h] ? (uint32_t)a.b_col[sj + (p - oj)] : 0u;
    }
    if (BITMAP) {
      uint32_t old[2];   // both atomics issue before either result is needed
#pragma unroll
      for (int h = 0; h < 2; ++h) old[h] = act[h] ? atomicOr(&seen[bb[h] >> 5], 1u << (bb[h] & 31u)) : 0u;
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (act[h] && ((old[h] >> (bb[h] & 31u)) & 1u)) accumulate<GROUP, false>(table, tsize, bb[h], cbits, 1u, 0u, a.err_flag);
    } else {
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (act[h]) accumulate<GROUP, DENSE>(table, tsize, bb[h], cbits, n_pass, pass, a.err_flag);
    }
  }
}

// ---- sorted rows (warp-owned rows keyed with an exact cut; DESIGN.md 3.1 "sorted rows") ------------------------------------
// The row's keys are sorted by an LSD radix sort over `passes` digits of `dbits` bits.  Each digit has a histogram of
// 2^dbits u16 bins packed two to a word (a warp-owned row has at most 1024 products); all of them are counted while the
// keys are gathered.
struct SortDigits {
  int passes, dbits, hwords;   // hwords = 2^(dbits - 1): words of one digit's histogram, 32 .. 256
};
__device__ __forceinline__ SortDigits sort_digits(int cbits) {
  const int kb = 32 - cbits;
  SortDigits d;
  d.passes = (kb + 8) / 9;
  d.dbits = max((kb + d.passes - 1) / d.passes, 6);
  d.hwords = 1 << (d.dbits - 1);
  return d;
}
__device__ __forceinline__ void digit_count(uint32_t *h, const SortDigits &sd, uint32_t b) {
  for (int p = 0; p < sd.passes; ++p) {
    const uint32_t dg = (b >> (p * sd.dbits)) & ((1u << sd.dbits) - 1u);
    atomicAdd(&h[p * sd.hwords + (dg >> 1)], 1u << (16u * (dg & 1u)));
  }
}

// Gather the products [0, p_hi) of a window of up to 32 users (registers as in count_window) to keys[p] in product order,
// counting every digit of every key into the histograms h.  Nothing waits on a gathered key here (no probe), so each lane
// keeps kGatherDepth gathers in flight.
constexpr int kGatherDepth = 4;
__device__ __forceinline__ void gather_window(const RowArgs &a, uint32_t *keys, uint32_t *h, const SortDigits &sd, uint32_t off,
                                              uint32_t s, uint32_t p_hi, int lane) {
  for (uint32_t p0 = 0; p0 < p_hi; p0 += 32 * kGatherDepth) {
    uint32_t bb[kGatherDepth];
    bool act[kGatherDepth];
#pragma unroll
    for (int hh = 0; hh < kGatherDepth; ++hh) {
      const uint32_t p = p0 + hh * 32 + lane;
      int j = 0;
#pragma unroll
      for (int st = 16; st > 0; st >>= 1) {
        const int c = j + st;
        const uint32_t v = __shfl_sync(0xffffffffu, off, c);
        if (v <= p) j = c;
      }
      const uint32_t sj = __shfl_sync(0xffffffffu, s, j), oj = __shfl_sync(0xffffffffu, off, j);
      act[hh] = p < p_hi;
      bb[hh] = act[hh] ? (uint32_t)a.b_col[sj + (p - oj)] : 0u;
    }
#pragma unroll
    for (int hh = 0; hh < kGatherDepth; ++hh)
      if (act[hh]) {
        keys[p0 + hh * 32 + lane] = bb[hh];
        digit_count(h, sd, bb[hh]);
      }
  }
}

// One warp: the counts of a packed u16 histogram of hwords words -> exclusive prefix sums, in place
__device__ __forceinline__ void digit_scan(uint32_t *h, int hwords, int lane) {
  const int per = hwords >> 5;
  uint32_t sum = 0;
  for (int j = 0; j < per; ++j) { const uint32_t v = h[lane * per + j]; sum += (v & 0xffffu) + (v >> 16); }
  uint32_t incl = sum;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += v;
  }
  uint32_t run = incl - sum;
  for (int j = 0; j < per; ++j) {
    const uint32_t v = h[lane * per + j], lo = v & 0xffffu;
    h[lane * per + j] = run | ((run + lo) << 16);
    run += lo + (v >> 16);
  }
  __syncwarp();
}

// Sorted rows: the row's w <= 1024 keys are in keys[0, w), keys[w, 2 w) is free, and h holds every digit's counts.  A
// stable LSD radix sort orders them (equal digits of one 32-key batch keep their lane order: match.any ranks them), and
// one pass over the sorted keys turns each run of equal keys into the packed word (key << cbits) | k11 at its last key,
// compacted to keys[w, w + n) -- the cells the filter reads.  The diagonal is dropped (the filter would skip it), and so
// is every k11 = 1 cell after the top_k-th other one: the singles are in key order, so those are exactly the cells
// beyond the level-1 key cut.  Returns n; *n_runs = the distinct cells.
__device__ uint32_t sort_runs(uint32_t *keys, uint32_t w, uint32_t *h, const SortDigits &sd, int cbits, int diag, int top_k,
                              uint32_t *n_runs, int lane) {
  const unsigned lt = (1u << lane) - 1u, le = (2u << lane) - 1u;
  uint32_t *src = keys, *dst = keys + w;
  for (int p = 0; p < sd.passes; ++p) {
    uint32_t *hp = h + p * sd.hwords;
    digit_scan(hp, sd.hwords, lane);
    const int sh = p * sd.dbits;
    for (uint32_t i0 = 0; i0 < w; i0 += 32) {
      const uint32_t i = i0 + lane;
      const bool valid = i < w;
      const uint32_t k = valid ? src[i] : 0u;
      const uint32_t dg = valid ? (k >> sh) & ((1u << sd.dbits) - 1u) : 0xffffffffu;
      const unsigned peers = __match_any_sync(0xffffffffu, dg);
      const uint32_t hsh = 16u * (dg & 1u);
      const uint32_t base = valid ? (hp[dg >> 1] >> hsh) & 0xffffu : 0u;
      __syncwarp();   // every lane has read its digit's offset before the batch's first lane of it moves it on
      if (valid) {
        const uint32_t r = __popc(peers & lt);
        dst[base + r] = k;
        if (r == 0) atomicAdd(&hp[dg >> 1], (uint32_t)__popc(peers) << hsh);
      }
      __syncwarp();
    }
    uint32_t *t = src; src = dst; dst = t;
  }
  // runs -> packed words at keys[w, w + n).  After an even number of passes that half is free; after an odd number it is
  // src itself, and the compaction is in place: the words of a batch go below the batch's last key (one word per run that
  // ends in or before it), and every later read is at or beyond the next batch.
  uint32_t *out = keys + w;
  uint32_t n = 0, n_single = 0, nr = 0, prev_key = kEmpty, head_pos = 0;
  for (uint32_t i0 = 0; i0 < w; i0 += 32) {
    const uint32_t i = i0 + lane;
    const bool valid = i < w;
    const uint32_t k = valid ? src[i] : kEmpty;   // keys are < 2^key_bits - 1: never kEmpty
    const uint32_t nk = i + 1 < w ? src[i + 1] : kEmpty;
    uint32_t pk = __shfl_up_sync(0xffffffffu, k, 1);
    if (lane == 0) pk = prev_key;
    const unsigned hm = __ballot_sync(0xffffffffu, valid && k != pk);
    nr += __popc(hm);
    const unsigned mine = hm & le;   // heads at or below this lane: the last one starts its run
    const uint32_t hpos = mine ? i0 + 31u - (uint32_t)__clz(mine) : head_pos;
    const uint32_t len = i + 1u - hpos;
    const bool off_diag = valid && k != nk && (int)k != diag;   // run ends here
    const bool single = off_diag && len == 1u;
    const unsigned sm = __ballot_sync(0xffffffffu, single);
    const bool keep = off_diag && (len > 1u || n_single + __popc(sm & lt) < (uint32_t)top_k);
    n_single += __popc(sm);
    const unsigned km = __ballot_sync(0xffffffffu, keep);
    prev_key = __shfl_sync(0xffffffffu, k, 31);
    head_pos = __shfl_sync(0xffffffffu, hpos, 31);
    __syncwarp();
    if (keep) out[n + __popc(km & lt)] = (k << cbits) | len;
    n += __popc(km);
    __syncwarp();
  }
  *n_runs = nr;
  return n;
}

// Minimum resident CTAs per SM that the register allocation must allow.  At top_k 50 make_cfg (cco_api.cu) fits 2 / 4 / 9
// hashed 512 / 256 / 128-thread CTAs per SM in shared memory; 8 instead of 9 keeps 64 registers (9 forces 56 and measured
// no faster).  Warp-owned rows run as 64-thread CTAs whose three bins fit 8 / 13 / 16 per SM: 12 is what their spill-free
// 80 registers allow, and a 16-CTA bound (64 registers) measured no faster.  Sorted rows need 72 registers (14 CTAs per
// SM) and their smaller tables fit 9 / 15 / 19.  DESIGN.md 3.2 lists registers and spills.
template <int GROUP>
struct RowsMinBlocks {
  static constexpr int value = GROUP == 512 ? 2 : GROUP == 256 ? 4 : GROUP == 128 ? 8 : GROUP == 32 ? 12 : 1;
};

// BITMAP (CTA-owned hashed bins whose rows are all on the key path with an exact cut; DESIGN.md 3.1 "bitmap rows"): the
// count sets one bit per cell in a bitmap over the keys and hashes only the repeated products; the level-1 key cut is the
// top_k-th set bit in key order, and only the k11 = 1 cells up to it are ever listed.
//
// SORTED (warp-owned hashed bins whose rows are all on the key path with an exact cut; DESIGN.md 3.1 "sorted rows"): the
// row's keys are gathered and sorted instead of hashed (sort_runs), which yields the counts, the compacted list and the
// level-1 key cut at once.
template <int GROUP, bool DENSE, bool BITMAP = false, bool SORTED = false>
__global__ void __launch_bounds__(GROUP == 32 ? 64 : GROUP, RowsMinBlocks<GROUP>::value) k_rows(const RowArgs a) {
  static_assert(!BITMAP || (GROUP > 32 && !DENSE), "bitmap rows are CTA-owned rows of a hashed bin");
  static_assert(!SORTED || (GROUP == 32 && !DENSE && !BITMAP), "sorted rows are warp-owned rows of a hashed bin");
  const int GROUPS = GROUP == 32 ? (int)(blockDim.x >> 5) : 1;  // warp-owned rows: several independent warps per CTA
  constexpr int NW = GROUP / 32;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int tid = threadIdx.x, lane = tid & 31;
  const int gid = tid / GROUP, gtid = tid % GROUP, gw = gtid >> 5;
  unsigned char *base = smem_raw + (size_t)gid * a.group_smem_bytes;
  uint4 *tk = reinterpret_cast<uint4 *>(base);
  uint4 *aux = tk + a.cbuf;                                  // a.caux entries (0 for warp-owned rows)
  double *x12tab = reinterpret_cast<double *>(aux + a.caux);
  double *x11tab = x12tab + 32;
  int *ctrl = reinterpret_cast<int *>(x11tab + 32);  // [0] ncand [1] have_thr [4..7] threshold entry [16..27] select state [40..55] dominance frontier [64..64+NW) per-warp list sizes
  int *hist = ctrl + 128;                                     // 256 bins of the radix select
  uint32_t *wqueue = reinterpret_cast<uint32_t *>(hist + 256);  // NW * 64 queued cells awaiting evaluation
  uint32_t *h1 = reinterpret_cast<uint32_t *>(hist);   // kCutBins/2 words: u16 histogram of colB over the strongly positive k11 == 1 cells
  uint32_t *table = wqueue + NW * 64;
  uint32_t *seen = table + a.slots;     // BITMAP: a.bm_words words, bit b = key b has a product in the row
  uint32_t *singles = seen + a.bm_words;  // BITMAP: top_k packed words, the k11 = 1 cells up to the key cut
  volatile int *vctrl = ctrl;

  const int row_begin = a.bin_bounds[a.bin], row_end = a.bin_bounds[a.bin + 1];
  const bool varargs = (a.flags & CCO_FLAG_ENTROPY_VARARGS) != 0;
  const int cbits = a.count_bits;
  const uint32_t cmask = (1u << cbits) - 1u;
  const int prune_limit = a.cbuf - GROUP;
  const long long N = a.n_users;
  const double xN = xlogx(N);
  unsigned long long distinct_local = 0, evaluated_local = 0;
  if (gtid < 32) x11tab[gtid] = xlogx((long long)gtid);
  uint32_t *dhist = reinterpret_cast<uint32_t *>(tk);   // SORTED: the digit histograms (the candidates are dead until the score stage)
  const SortDigits sd = sort_digits(cbits);

  for (int ri = row_begin + blockIdx.x * GROUPS + gid; ri < row_end; ri += gridDim.x * GROUPS) {
    const int item = a.rows_sorted[ri];
    const uint32_t u_begin = a.at_ptr[item], u_end = a.at_ptr[item + 1];
    const long long ra = a.marg_a[item];
    int diag = -1;   // the key of the A'^T A' diagonal cell, -1 when it lies outside this key range
    if (a.self) {
      const int d = a.key_of_col[item] - a.key_base;
      if ((unsigned)d < (unsigned)a.n_cols_b) diag = d;
    }
    // Key path: 2 rowA colB < N for every column of B' (every row at C3 / C4), so every cell is strongly positive and both
    // the level-1 cut and the dominance filter are monotone in colB -- hence in the key.  They compare keys, and no cell
    // gathers its colB.  Other rows read colB from marg_b[key].
    const bool keyed = 2ull * (unsigned long long)ra * (unsigned long long)a.max_marg_b < (unsigned long long)N;
    // table sized to the row: load factor <= 1/2 of the distinct-cell bound D = min(w, n_cols_b)
    uint32_t n_pass = 1, tsize = (uint32_t)a.n_cols_b;
    if (!DENSE && !SORTED) {
      const uint32_t w = a.row_work[item];
      // BITMAP: the table holds only cells with k11 >= 2, each of at least two of the w products (one pass: the host
      // sizes a.slots for the bin's largest w)
      const uint32_t dcells = BITMAP ? w / 2u : w;
      const uint32_t dbound = dcells < (uint32_t)a.n_cols_b ? dcells : (uint32_t)a.n_cols_b;
      n_pass = BITMAP ? 1u : (dbound + (uint32_t)a.cap - 1u) / (uint32_t)a.cap;
      if (n_pass == 0) n_pass = 1;
      tsize = n_pass > 1 ? (uint32_t)a.slots
                         : (uint32_t)min((unsigned long long)a.slots,
                                         max(((unsigned long long)dbound * (unsigned long long)a.tsize_x16) >> 4, 64ull));
      tsize = min((uint32_t)a.slots, (tsize + 32u * NW - 1u) / (32u * NW) * (32u * NW));
    }
    group_sync<GROUP>();  // previous row fully done with shared memory
    if (gtid < 32) {
      const long long v = (gtid < kX12N) ? ra - gtid : N - ra;
      x12tab[gtid] = v >= 0 ? xlogx(v) : 0.0;
    }
    if (gtid == 0) { ctrl[0] = 0; ctrl[1] = 0; }
    if (gtid < 16) ctrl[40 + gtid] = 0x7fffffff;
    int emitted = 0;

    for (uint32_t pass = 0; pass < n_pass; ++pass) {
      // ---- clear --------------------------------------------------------------------------------------
      if (SORTED)
        for (int i = lane; i < sd.passes * sd.hwords; i += 32) dhist[i] = 0u;
      else
        for (uint32_t i = gtid; i < tsize; i += GROUP) table[i] = DENSE ? 0u : kEmpty;
      if (BITMAP)
        for (int i = gtid; i < a.bm_words; i += GROUP) seen[i] = 0u;
      group_sync<GROUP>();
      // ---- count -------------------------------------------------------------------------------------------
      // SORTED: the row's w keys and the sort's second half end where the table ends, reaching back over the dead select
      // histogram and evaluation queues (the host sizes a.slots >= max(2 max_w - 320, max_w)); the cells the filter reads
      // end up in the second half, inside the table
      uint32_t *keys = table + a.slots - 2u * (SORTED ? a.row_work[item] : 0u);
      uint32_t n_keys = 0;   // SORTED: the keys gathered so far
      if (NW == 1) {
        // warp-owned row: 32-user chunks, the products of a chunk flattened over the lanes by a warp prefix sum
        for (uint32_t c0 = u_begin; c0 < u_end; c0 += 32) {
          const uint32_t i = c0 + lane;
          uint32_t s = 0, len = 0;
          if (i < u_end) {
            const int32_t u = a.at_users[i];
            s = a.b_ptr[u];
            len = a.b_ptr[u + 1] - s;
          }
          uint32_t off = len;
#pragma unroll
          for (int d = 1; d < 32; d <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, off, d);
            if (lane >= d) off += v;
          }
          const uint32_t total = __shfl_sync(0xffffffffu, off, 31);
          off = i < u_end ? off - len : 0xffffffffu;  // exclusive
          if (SORTED) {
            gather_window(a, keys + n_keys, dhist, sd, off, s, total, lane);
            n_keys += total;
          } else {
            count_window<GROUP, DENSE, BITMAP>(a, table, seen, tsize, cbits, n_pass, pass, off, s, 0u, total, lane);
          }
        }
      } else {
        // CTA-owned row: the count barrier waits for the busiest warp, and B' degrees are Zipf-skewed, so the warps
        // split the PRODUCTS of a window of GROUP users evenly (not the users).  Thread t loads user t of the window;
        // a CTA scan of the degrees goes to `wofs` = (B' row start, first product) per user, which aliases the
        // evaluation queues (dead until the score stage).  Warp g counts products [g T / NW, (g + 1) T / NW) of the
        // window's T, 32 users at a time in registers.
        uint2 *wofs = reinterpret_cast<uint2 *>(wqueue);   // GROUP entries = NW * 64 words
        int *wsum = hist;                                  // NW warp totals (the select histogram is dead here)
        for (uint32_t w0 = u_begin; w0 < u_end; w0 += GROUP) {
          const uint32_t nwin = min((uint32_t)GROUP, u_end - w0);
          uint32_t s = 0, len = 0;
          if ((uint32_t)gtid < nwin) {
            const int32_t u = a.at_users[w0 + gtid];
            s = a.b_ptr[u];
            len = a.b_ptr[u + 1] - s;
          }
          uint32_t incl = len;
#pragma unroll
          for (int d = 1; d < 32; d <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += v;
          }
          if (lane == 31) wsum[gw] = (int)incl;
          __syncthreads();
          uint32_t wpre = lane < NW ? (uint32_t)wsum[lane] : 0u;
#pragma unroll
          for (int d = 1; d < NW; d <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, wpre, d);
            if (lane >= d) wpre += v;
          }
          const uint32_t T = __shfl_sync(0xffffffffu, wpre, NW - 1);
          const uint32_t before = gw == 0 ? 0u : __shfl_sync(0xffffffffu, wpre, gw - 1);
          wofs[gtid] = make_uint2(s, before + incl - len);
          __syncthreads();
          const uint32_t p_lo = (uint32_t)((unsigned long long)T * gw / NW);
          const uint32_t p_hi = (uint32_t)((unsigned long long)T * (gw + 1) / NW);
          if (p_lo < p_hi) {
            // first user of the warp's range: the last one whose first product is <= p_lo
            uint32_t lo = 0, hi = nwin - 1;
            while (lo < hi) {
              const uint32_t mid = (lo + hi + 1) >> 1;
              if (wofs[mid].y <= p_lo) lo = mid; else hi = mid - 1;
            }
            for (uint32_t j0 = lo, p = p_lo; p < p_hi; j0 += 32) {
              const uint2 e = j0 + lane < nwin ? wofs[j0 + lane] : make_uint2(0u, 0xffffffffu);
              const uint32_t wend = min(p_hi, j0 + 32 < nwin ? wofs[j0 + 32].y : T);
              count_window<GROUP, DENSE, BITMAP>(a, table, seen, tsize, cbits, n_pass, pass, e.y, e.x, p, wend, lane);
              p = wend;
            }
          }
          __syncthreads();   // wofs / wsum are rewritten by the next window
        }
      }
      group_sync<GROUP>();
      // ---- compact: each warp packs the occupied words of its own table segment, in place ----------------
      const uint32_t seg = (((tsize + NW - 1) / NW) + 31u) & ~31u;
      const uint32_t seg_lo = min((uint32_t)gw * seg, tsize), seg_hi = min(seg_lo + seg, tsize);
      uint32_t n_mine = 0;
      const uint32_t *list = table;   // the cells the filter reads (SORTED: the second half of the sort)
      if (SORTED) {
        uint32_t n_runs;
        n_mine = sort_runs(keys, n_keys, dhist, sd, cbits, diag, a.top_k, &n_runs, lane);
        list = keys + n_keys;
        if (lane == 0) distinct_local += n_runs;
      }
      for (uint32_t pos = seg_lo; pos < seg_hi && !SORTED; pos += 32) {
        const uint32_t idx = pos + lane;
        uint32_t w = DENSE ? 0u : kEmpty;
        if (idx < seg_hi) w = table[idx];
        const bool valid = DENSE ? (w != 0u) : (w != kEmpty);
        const uint32_t word = DENSE ? ((idx << cbits) | w) : w;
        const unsigned m = __ballot_sync(0xffffffffu, valid);
        __syncwarp();
        if (valid) {
          // BITMAP: the table counted k11 - 1; the cell leaves the bitmap, which keeps the k11 = 1 cells only
          table[seg_lo + n_mine + __popc(m & ((1u << lane) - 1u))] = BITMAP ? word + 1u : word;
          if (BITMAP) atomicAnd(&seen[(word >> cbits) >> 5], ~(1u << ((word >> cbits) & 31u)));
        }
        n_mine += __popc(m);
        __syncwarp();
      }
      if (lane == 0 && !SORTED) distinct_local += n_mine;
      uint32_t n_list = n_mine;   // cells this warp filters: its compacted table words, then (BITMAP) its singles
      const uint32_t *singles_mine = singles;
      if (BITMAP) {
        // ---- singles and the level-1 key cut (exact; DESIGN.md 3.1 "bitmap rows") -----------------------------------
        // The bitmap now holds the k11 = 1 cells.  Without the diagonal, the first top_k set bits in key order are the
        // cells at or below the key cut (all of them when there are fewer): one CTA prefix sum of popcounts over
        // contiguous word ranges, and each thread lists the bits of its range that fall below top_k.
        group_sync<GROUP>();
        if (gtid == 0 && diag >= 0) {
          const uint32_t bit = 1u << ((uint32_t)diag & 31u);
          if (seen[diag >> 5] & bit) {
            seen[diag >> 5] &= ~bit;
            ++distinct_local;
          }
        }
        group_sync<GROUP>();
        const uint32_t nbw = (uint32_t)a.bm_words, per = (nbw + GROUP - 1u) / GROUP;
        const uint32_t w_lo = min((uint32_t)gtid * per, nbw), w_hi = min(w_lo + per, nbw);
        uint32_t cnt = 0;
        for (uint32_t i = w_lo; i < w_hi; ++i) cnt += __popc(seen[i]);
        distinct_local += cnt;
        uint32_t incl = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
          if (lane >= d) incl += v;
        }
        int *wsum = hist;   // the select histogram is dead until the score stage
        if (lane == 31) wsum[gw] = (int)incl;
        __syncthreads();
        uint32_t wpre = lane < NW ? (uint32_t)wsum[lane] : 0u;
#pragma unroll
        for (int d = 1; d < NW; d <<= 1) {
          const uint32_t v = __shfl_up_sync(0xffffffffu, wpre, d);
          if (lane >= d) wpre += v;
        }
        const uint32_t total = __shfl_sync(0xffffffffu, wpre, NW - 1);
        const uint32_t before = gw == 0 ? 0u : __shfl_sync(0xffffffffu, wpre, gw - 1);
        const uint32_t n_single = min(total, (uint32_t)a.top_k);
        uint32_t o = before + incl - cnt;
        for (uint32_t i = w_lo; i < w_hi && o < n_single; ++i)
          for (uint32_t m = seen[i]; m != 0u && o < n_single; m &= m - 1u)
            singles[o++] = (((i << 5) | (uint32_t)(__ffs(m) - 1)) << cbits) | 1u;
        __syncthreads();   // wsum is the select histogram again; the singles are complete
        const uint32_t s_lo = (uint32_t)((unsigned long long)n_single * gw / NW);
        const uint32_t s_hi = (uint32_t)((unsigned long long)n_single * (gw + 1) / NW);
        singles_mine = singles + s_lo;
        n_list = n_mine + (s_hi - s_lo);
      }
      if (!BITMAP && !SORTED && a.emit_all) {
        // debug: every non-zero cell of the row (col, count), unordered
        int basepos = 0;
        if (lane == 0) basepos = atomicAdd(&ctrl[0], (int)n_mine);
        basepos = __shfl_sync(0xffffffffu, basepos, 0);
        for (uint32_t q = lane; q < n_mine; q += 32) {
          const uint32_t word = table[seg_lo + q];
          const size_t o = (size_t)item * a.out_stride + emitted + basepos + q;
          a.out_col[o] = a.col_terms[word >> cbits].col;
          a.out_cnt[o] = (int32_t)(word & cmask);
        }
        group_sync<GROUP>();
        emitted += vctrl[0];
        group_sync<GROUP>();
        if (gtid == 0) ctrl[0] = 0;
        group_sync<GROUP>();
        continue;
      }
      // ---- level-1 integer cut (exact; DESIGN.md 3.1) ---------------------------------------------------------------
      // On the strongly positive side (2*rowA*colB < N) the real LLR of k11 == 1 cells is strictly decreasing in colB, so
      // the smallest colB c1 with >= top_k such cells at or below it bounds the row's k-th best from below: k11 == 1 cells
      // with colB > c1 can never be kept and are dropped by an integer compare in the filter stage.
      // Key path: c1 is the k-th smallest KEY of those cells (MSB-first radix select, 9 key bits per level): ties in
      // colB are ordered by column id, the output's tie order, so the cut is exact and drops ties beyond the k-th too.
      // Both hold for the COMPUTED fp64 values only when adjacent colB values are further apart than the evaluation
      // error: the host checks that once per indicator (a.cut_ok) and otherwise the row runs without the cut.
      int cut1 = 0x7fffffff;   // (BITMAP, SORTED: the singles list is already cut)
      if (!BITMAP && !SORTED && a.cut_ok && a.row_work[item] < 65536u) {   // u16 bins cannot overflow
        int sh = keyed ? a.key_shift : 0, hi_sh = 32;   // level: bins over key bits [sh, hi_sh) of keys matching `prefix` above
        uint32_t prefix = 0, need = (uint32_t)a.top_k;
        while (true) {
          for (int i = gtid; i < kCutBins / 2; i += GROUP) h1[i] = 0u;
          group_sync<GROUP>();
          for (uint32_t q0 = 0; q0 < n_mine; q0 += 32) {
            const uint32_t q = q0 + lane;
            if (q < n_mine) {
              const uint32_t word = table[seg_lo + q];
              const uint32_t b = word >> cbits;
              if ((word & cmask) == 1u && (int)b != diag) {
                uint32_t bin = kCutBins;
                if (keyed) {
                  if (((unsigned long long)(b ^ prefix) >> hi_sh) == 0) bin = (b >> sh) & (kCutBins - 1);
                } else {
                  const uint32_t cb = (uint32_t)a.marg_b[b];
                  if (cb < (uint32_t)kCutBins && 2ull * (unsigned long long)ra * cb < (unsigned long long)N) bin = cb;
                }
                if (bin < (uint32_t)kCutBins) atomicAdd(&h1[bin >> 1], 1u << (16u * (bin & 1u)));
              }
            }
          }
          group_sync<GROUP>();
          if (gtid < 32) cut_find(h1, need, lane, ctrl);
          group_sync<GROUP>();
          const int found = vctrl[9];
          if (!keyed || found == 0x7fffffff) { cut1 = found; break; }
          prefix |= (uint32_t)found << sh;
          need -= (uint32_t)vctrl[10];
          if (sh == 0) { cut1 = (int)prefix; break; }
          hi_sh = sh;
          sh = sh > 9 ? sh - 9 : 0;
        }
      }
      // ---- score + select -----------------------------------------------------------------------------------
      const double x_ra = x12tab[0], x_nra = x12tab[kX12N];
      const double row_e = varargs ? __dsub_rn(xN, __dadd_rn(__dadd_rn(0.0, x_ra), x_nra))
                                   : __dsub_rn(__dsub_rn(xN, x_ra), x_nra);
      // Two stages per warp so that the fp64 evaluation always runs on full warps:
      //   filter  : 32 cells at a time through the exact dominance filter (integer work only); survivors are queued
      //   evaluate: 32 queued cells at a time -> LLR -> threshold test -> candidate buffer
      // One evaluation batch per round, then (CTA-owned rows) one barrier that also decides whether any warp has work.
      uint32_t *wq = wqueue + gw * 64;
      uint32_t pos = 0;
      int qn = 0;
      while (true) {
        while (qn < 32 && pos < n_list) {
          const uint32_t q = pos + lane;
          bool surv = false;
          uint32_t word = 0;
          if (q < n_list) {
            word = (!BITMAP || q < n_mine) ? list[seg_lo + q] : singles_mine[q - n_mine];
            const uint32_t b = word >> cbits, k11 = word & cmask;
            if ((int)b != diag) {
              // Dominance filter (exact, DESIGN.md "dominance"): for fixed rowA and N, on the positively associated
              // side (rowA*cb < k11*N) the real LLR grows with k11 and shrinks with cb, so every evaluated cell (k, c) that
              // fails by more than 2 eps proves that all cells (k' <= k, c' >= c) fail too; cfail[k'] = smallest such c.
              // Key path: every cell is on that side, cfail holds first_key_of_cb[c], and key >= it iff colB >= c.
              if (keyed) {
                surv = !(k11 <= (uint32_t)kDomLevels && (int)b >= vctrl[40 + k11]);
                if (k11 == 1u && (int)b > cut1) surv = false;   // beyond the level-1 key cut
              } else {
                const long long cb = a.marg_b[b];
                const bool pos_side = (unsigned long long)ra * (unsigned long long)cb < (unsigned long long)k11 * (unsigned long long)N;
                surv = !(pos_side && k11 <= (uint32_t)kDomLevels && (int)cb >= vctrl[40 + k11]);
                if (k11 == 1u && (int)cb > cut1 && 2ull * (unsigned long long)ra * (unsigned long long)cb < (unsigned long long)N)
                  surv = false;   // beyond the level-1 integer cut
              }
            }
          }
          const unsigned m = __ballot_sync(0xffffffffu, surv);
          if (surv) wq[qn + __popc(m & ((1u << lane) - 1u))] = word;
          qn += __popc(m);
          pos += 32;
          __syncwarp();
        }
        const int take = qn < 32 ? qn : 32;
        bool pass_ok = false;
        uint4 e = make_uint4(0u, 0u, 0u, 0u);
        if (lane < take) {
          const uint32_t word = wq[qn - take + lane];
          const uint32_t b = word >> cbits, k11 = word & cmask;
          const ColTerm ct = a.col_terms[b];
          const long long cb = ct.cb;
          const bool pos_side = (unsigned long long)ra * (unsigned long long)cb < (unsigned long long)k11 * (unsigned long long)N;
          const uint32_t kf = k11 < (uint32_t)kDomLevels ? k11 : (uint32_t)kDomLevels;
          ++evaluated_local;
          const long long k21 = cb - k11, k22 = N - ra - cb + k11;
          const double x11 = k11 < 32 ? x11tab[k11] : xlogx_u32(k11);
          const double x12 = k11 < kX12N ? x12tab[k11] : xlogx_u32((uint32_t)(ra - k11));
          const double x21 = k11 == 1 ? ct.x_cbm1 : xlogx_u32((uint32_t)k21), x22 = xlogx_u32((uint32_t)k22);
          double mat_e;
          if (varargs)
            mat_e = __dsub_rn(xN, __dadd_rn(__dadd_rn(__dadd_rn(__dadd_rn(0.0, x11), x12), x21), x22));
          else
            mat_e = __dsub_rn(__dsub_rn(__dsub_rn(__dsub_rn(xN, x11), x12), x21), x22);
          const double sre = __dadd_rn(row_e, ct.col_e);
          const double v = (sre < mat_e) ? 0.0 : __dmul_rn(2.0, __dsub_rn(sre, mat_e));
          const bool min_ok = !a.has_min_llr || v >= a.min_llr;
          pass_ok = v > 0.0 && min_ok;
          // (cells whose LLR rounds to 0 are cancellation noise: they teach nothing)
          // A failing cell proves that the cells it dominates fail only if it misses the bar T (minLLR or the running
          // threshold) by more than 2 eps: their computed LLR is at most v + 2 eps (DESIGN.md 3.1, "dominance").
          const double vm = __dadd_rn(v, a.llr_eps2);
          bool strict_fail = v > 0.0 && !min_ok && vm < a.min_llr;
          const unsigned long long key = (unsigned long long)__double_as_longlong(v);
          e = make_uint4((uint32_t)key, (uint32_t)(key >> 32), (uint32_t)ct.col, k11);
          if (pass_ok && vctrl[1]) {
            const uint4 thr = make_uint4((uint32_t)vctrl[4], (uint32_t)vctrl[5], (uint32_t)vctrl[6], (uint32_t)vctrl[7]);
            pass_ok = !cand_better(thr, e);
            strict_fail = vm < __hiloint2double((int)thr.y, (int)thr.x);
          }
          if (strict_fail && pos_side) {
            const int f = keyed ? a.first_key_of_cb[cb] : (int)cb;
            for (uint32_t kk = kf; kk >= 1 && f < vctrl[40 + kk]; --kk) atomicMin(&ctrl[40 + kk], f);
          }
        }
        qn -= take;
        const unsigned m = __ballot_sync(0xffffffffu, pass_ok);
        int basepos_round = 0;
        if (m) {
          int basepos = 0;
          if (lane == 0) basepos = atomicAdd(&ctrl[0], __popc(m));
          basepos = __shfl_sync(0xffffffffu, basepos, 0);
          if (pass_ok) tk[basepos + __popc(m & ((1u << lane) - 1u))] = e;
          basepos_round = basepos;
        }
        const bool more = qn > 0 || pos < n_list;
        // Both decisions of this round are taken from barrier results (CTA-uniform by construction).  Re-reading ctrl[0]
        // after the barrier raced with warps that had already looped back and appended (or with warp 0's single-warp
        // select storing the kept count): warps of one CTA could disagree on `n > prune_limit` and pair different
        // barriers.  `mine` = the counter right after this warp's own append (0 if it appended nothing): the counter only
        // grows inside a round, so the largest `mine` is its final value.
        int mine = 0;
        if (m) mine = basepos_round + __popc(m);
        bool any_more, need_prune;
        if (GROUP == 32) {
          __syncwarp();
          any_more = more;
          need_prune = mine > prune_limit;
        } else {
          any_more = __syncthreads_or(more ? 1 : 0) != 0;
          need_prune = __syncthreads_or(mine > prune_limit ? 1 : 0) != 0;
        }
        if (need_prune) {
          const int n = vctrl[0];   // nobody appends until every warp has left this branch
          if (GROUP > 32 && n <= 512) {
            // small buffer: one warp runs the whole select (no CTA barriers inside), the others wait once
            if (gw == 0) reduce_candidates<32>(tk, aux, n, a.top_k, a.keep_max, hist, ctrl, lane);
            group_sync<GROUP>();
          } else {
            reduce_candidates<GROUP>(tk, aux, n, a.top_k, a.keep_max, hist, ctrl, gtid);
          }
        }
        if (!any_more) break;
      }
      group_sync<GROUP>();
    }
    // ---- final select + write -------------------------------------------------------------------------------
    if (a.emit_all) {
      if (gtid == 0) a.out_len[item] = emitted;
    } else {
      int n = vctrl[0];
      if (n > 0) {
        if (GROUP > 32 && n <= 512) {
          if (gw == 0) {
            int m = n;
            if (m > a.final_max) m = reduce_candidates<32>(tk, aux, m, a.top_k, a.final_max, hist, ctrl, lane);
            sort_candidates<32>(tk, m, lane);
            if (lane == 0) ctrl[0] = m;
          }
          group_sync<GROUP>();
          n = vctrl[0];
        } else {
          if (n > a.final_max) n = reduce_candidates<GROUP>(tk, aux, n, a.top_k, a.final_max, hist, ctrl, gtid);
          sort_candidates<GROUP>(tk, n, gtid);
        }
        const int keep = n < a.top_k ? n : a.top_k;
        for (int i = gtid; i < keep; i += GROUP) {
          const size_t o = (size_t)item * a.out_stride + i;
          const uint4 e = tk[i];
          a.out_col[o] = (int32_t)e.z;
          a.out_llr[o] = __longlong_as_double((long long)(((unsigned long long)e.y << 32) | e.x));
          a.out_cnt[o] = (int32_t)e.w;
        }
        if (gtid == 0) a.out_len[item] = keep;
      } else if (gtid == 0) {
        a.out_len[item] = 0;
      }
    }
  }
  for (int o = 16; o > 0; o >>= 1) distinct_local += __shfl_xor_sync(0xffffffffu, distinct_local, o);
  if (lane == 0 && distinct_local) atomicAdd(a.stat_distinct, distinct_local);
  for (int o = 16; o > 0; o >>= 1) evaluated_local += __shfl_xor_sync(0xffffffffu, evaluated_local, o);
  if (lane == 0 && evaluated_local) atomicAdd(a.stat_evaluated, evaluated_local);
}

// packed output: gather the strided per-row results into CSR order (out_ptr = exclusive scan of the masked row lengths:
// rows outside this rank's range have length 0 there and are skipped)
__global__ void k_compact_rows(int32_t n_items, int32_t stride, const long long *__restrict__ out_ptr,
                               const int32_t *__restrict__ col, const double *__restrict__ llr, const int32_t *__restrict__ cnt,
                               int32_t *__restrict__ p_col, double *__restrict__ p_llr, int32_t *__restrict__ p_cnt) {
  // one warp per row
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int item = warp; item < n_items; item += nwarps) {
    const long long o = out_ptr[item];
    const int n = (int)(out_ptr[item + 1] - o);
    size_t src = (size_t)item * stride;
    for (int i = lane; i < n; i += 32) {
      p_col[o + i] = col[src + i];
      if (p_llr) p_llr[o + i] = llr[src + i];
      if (p_cnt) p_cnt[o + i] = cnt[src + i];
    }
  }
}

// ---- key ranges (DESIGN.md 3.1): an indicator whose counts do not fit the packed word runs once per key range ----------
// B'_r = the entries of B' whose key lies in [k0, k1), rebased to key - k0, over the same users.  One warp per user row;
// WRITE = false counts them into r_ptr[u] (and r_ptr[n_rows] = 0, so an exclusive scan turns the counts into row pointers),
// WRITE = true writes them at r_ptr[u] in the order of B'[u].
template <bool WRITE>
__global__ void k_split_range(long long n_rows, const uint32_t *__restrict__ b_ptr, const int32_t *__restrict__ b_col, int32_t k0,
                              int32_t k1, uint32_t *__restrict__ r_ptr, int32_t *__restrict__ r_col) {
  const int lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * blockDim.x / 32;
  if (!WRITE && blockIdx.x == 0 && threadIdx.x == 0) r_ptr[n_rows] = 0u;
  for (long long u = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / 32; u < n_rows; u += stride) {
    const uint32_t s = b_ptr[u], e = b_ptr[u + 1];
    uint32_t w = WRITE ? r_ptr[u] : 0u;
    for (uint32_t q0 = s; q0 < e; q0 += 32) {
      const uint32_t q = q0 + lane;
      const int32_t key = q < e ? b_col[q] : -1;
      const bool in = key >= k0 && key < k1;
      const unsigned m = __ballot_sync(0xffffffffu, in);
      if (WRITE && in) r_col[w + __popc(m & ((1u << lane) - 1u))] = key - k0;
      w += __popc(m);
    }
    if (!WRITE && lane == 0) r_ptr[u] = w;
  }
}
// first_key_of_cb of a key range: [c] = first key of the range whose colB >= c, for c in [0, max colB of the range + 1]
__global__ void k_range_first_keys(int32_t n, const int32_t *__restrict__ first_key_of_cb, int32_t k0, int32_t n_keys,
                                   int32_t *__restrict__ out) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x)
    out[c] = min(max(first_key_of_cb[c] - k0, 0), n_keys);
}
// Merge range r's strided rows (r_*) into the running result (col / llr / cnt / len), in place, one warp per row.
// Top-k rows: both lists are sorted by (llr desc, col asc) and hold distinct columns, so the first min(top_k, la + lb)
// entries of their merge are the top-k over both ranges.  Output position p takes A[i] or B[p - i], i = the merge-path
// co-rank of p; positions are filled from the end, 32 at a time, and every read of a chunk lies at or below its positions
// while every later write lies below the chunk: the merge can overwrite A in place.
// emit_all rows: the ranges' cells are appended (that mode's rows are unordered).
__device__ __forceinline__ bool merge_before(double la, int32_t ca, double lb, int32_t cb) {
  return la > lb || (la == lb && ca < cb);
}
__global__ void k_merge_range(int32_t n_items, int32_t stride, int32_t top_k, int32_t emit_all, int32_t *__restrict__ col,
                              double *__restrict__ llr, int32_t *__restrict__ cnt, int32_t *__restrict__ len,
                              const int32_t *__restrict__ r_col, const double *__restrict__ r_llr, const int32_t *__restrict__ r_cnt,
                              const int32_t *__restrict__ r_len) {
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int item = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; item < n_items; item += nwarps) {
    const int la = len[item], lb = r_len[item];
    if (lb == 0) continue;
    int32_t *A_col = col + (size_t)item * stride, *A_cnt = cnt + (size_t)item * stride;
    const int32_t *B_col = r_col + (size_t)item * stride, *B_cnt = r_cnt + (size_t)item * stride;
    if (emit_all) {
      for (int j = lane; j < lb; j += 32) {
        A_col[la + j] = B_col[j];
        A_cnt[la + j] = B_cnt[j];
      }
      if (lane == 0) len[item] = la + lb;
      continue;
    }
    double *A_llr = llr + (size_t)item * stride;
    const double *B_llr = r_llr + (size_t)item * stride;
    const int n = min(top_k, la + lb);
    for (int base = (n - 1) & ~31; base >= 0; base -= 32) {
      const int p = base + lane;
      int32_t oc = 0, on = 0;
      double ol = 0.0;
      if (p < n) {
        int lo = max(0, p - lb), hi = min(p, la);
        while (lo < hi) {   // co-rank: the number of A entries among the first p outputs
          const int mid = (lo + hi) >> 1;
          if (merge_before(A_llr[mid], A_col[mid], B_llr[p - 1 - mid], B_col[p - 1 - mid])) lo = mid + 1; else hi = mid;
        }
        const int i = lo, j = p - lo;
        const bool from_a = j >= lb || (i < la && merge_before(A_llr[i], A_col[i], B_llr[j], B_col[j]));
        if (from_a) { oc = A_col[i]; ol = A_llr[i]; on = A_cnt[i]; } else { oc = B_col[j]; ol = B_llr[j]; on = B_cnt[j]; }
      }
      __syncwarp();
      if (p < n) { A_col[p] = oc; A_llr[p] = ol; A_cnt[p] = on; }
      __syncwarp();
    }
    if (lane == 0) len[item] = n;
  }
}

// ---- canonicalisation slow path (unsorted / duplicated input rows) -------------------------------
__global__ void k_expand_keys(long long n_rows, const long long *__restrict__ rp, const int32_t *__restrict__ col,
                              unsigned long long *__restrict__ keys) {
  const int lane = threadIdx.x % kSG;
  long long row = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / kSG;
  const long long stride = (long long)gridDim.x * blockDim.x / kSG;
  const long long q_base = rp[0];   // a rank's user block keeps the caller's absolute offsets
  for (; row < n_rows; row += stride) {
    long long s = rp[row], e = rp[row + 1];
    for (long long q = s + lane; q < e; q += kSG) keys[q - q_base] = ((unsigned long long)row << 32) | (uint32_t)col[q];
  }
}
__global__ void k_unique_flags(long long n, const unsigned long long *__restrict__ keys, uint32_t *__restrict__ flag) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    flag[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1u : 0u;
}
__global__ void k_unique_scatter(long long n, const unsigned long long *__restrict__ keys,
                                 const uint32_t *__restrict__ flag, const uint32_t *__restrict__ pos,
                                 unsigned long long *__restrict__ out_keys, int32_t *__restrict__ out_col) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    if (flag[i]) { out_keys[pos[i]] = keys[i]; out_col[pos[i]] = (int32_t)(keys[i] & 0xffffffffULL); }
}
// row_ptr[r] = first index whose key >= (r << 32)
__global__ void k_rowptr_from_keys(long long n_rows, long long n_unique, const unsigned long long *__restrict__ keys,
                                   long long *__restrict__ rp) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r <= n_rows; r += (long long)gridDim.x * blockDim.x) {
    unsigned long long t = (unsigned long long)r << 32;
    long long lo = 0, hi = n_unique;
    while (lo < hi) {
      long long mid = (lo + hi) >> 1;
      if (keys[mid] < t) lo = mid + 1; else hi = mid;
    }
    rp[r] = lo;
  }
}

// small device -> host results go through a mapped pinned "mailbox" written by this kernel, not through the D2H copy
// engine: a few-byte cudaMemcpyAsync would queue behind the multi-megabyte indicator copies of the previous
// indicator (one DMA FIFO per direction) and stall the launch pipeline behind them.
__global__ void k_mail_bytes(unsigned char *__restrict__ dst_mapped, const unsigned char *__restrict__ src, int n) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) dst_mapped[i] = src[i];
  __threadfence_system();
}

// device twin of cco_partition_rows (cco_api.cu): contiguous item ranges of equal (products + 1 per row)
__global__ void k_partition_rows(const long long *__restrict__ work_prefix, int32_t n_items, int32_t world, int32_t *bounds) {
  const int r = threadIdx.x;
  if (r > world) return;
  if (r == 0) { bounds[0] = 0; return; }
  if (r == world) { bounds[r] = n_items; return; }
  const long long total = work_prefix[n_items] + n_items;
  const long long target = (long long)((__int128)total * r / world);
  int lo = 0, hi = n_items;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (work_prefix[mid] + mid < target) lo = mid + 1; else hi = mid;
  }
  bounds[r] = lo;
}

// ---- ingest (SURVEY.md 8f-1: Preparator.prepare on integer-tokenised events) ---------------------------------------
// per-user event counts of the primary type (duplicates count: Preparator.scala:129-132)
__global__ void k_ingest_count_users(long long n, const long long *__restrict__ user, int32_t *__restrict__ counts) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    atomicAdd(&counts[user[i]], 1);
}
// flag[u] = 1 iff user u stays in the dictionary
__global__ void k_ingest_user_flags(long long n_users_raw, const int32_t *__restrict__ counts, int32_t need,
                                    uint32_t *__restrict__ flag) {
  for (long long u = blockIdx.x * (long long)blockDim.x + threadIdx.x; u < n_users_raw; u += (long long)gridDim.x * blockDim.x)
    flag[u] = counts[u] >= need ? 1u : 0u;
}
// map[i] = flag[i] ? pos[i] : -1
__global__ void k_ingest_make_map(long long n, const uint32_t *__restrict__ flag, const uint32_t *__restrict__ pos,
                                  int32_t *__restrict__ map) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    map[i] = flag[i] ? (int32_t)pos[i] : -1;
}
// items that still have an event of a surviving user (Preparator.scala:184)
__global__ void k_ingest_item_flags(long long n, const long long *__restrict__ user, const int32_t *__restrict__ item,
                                    const int32_t *__restrict__ user_map, uint32_t *__restrict__ item_flag) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    if (user_map[user[i]] >= 0) item_flag[item[i]] = 1u;
}
// key = (new user << 32 | new item) for surviving events, ~0 for dropped ones (they sort to the end)
__global__ void k_ingest_keys(long long n, const long long *__restrict__ user, const int32_t *__restrict__ item,
                              const int32_t *__restrict__ user_map, const int32_t *__restrict__ item_map,
                              unsigned long long *__restrict__ keys, unsigned long long *__restrict__ n_kept) {
  unsigned long long kept = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int32_t r = user_map[user[i]];
    if (r >= 0) {
      keys[i] = ((unsigned long long)(uint32_t)r << 32) | (uint32_t)item_map[item[i]];
      ++kept;
    } else {
      keys[i] = ~0ULL;
    }
  }
  for (int o = 16; o > 0; o >>= 1) kept += __shfl_xor_sync(0xffffffffu, kept, o);
  if ((threadIdx.x & 31) == 0 && kept) atomicAdd(n_kept, kept);
}

__global__ void k_fill_u32(long long n, uint32_t v, uint32_t *__restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) out[i] = v;
}

// ---- synthetic event streams (bench.py / tests; SURVEY.md 8d spec, numpy twin in synth.py) ---------------------------
// inclusive normalised CDF over ranks -> first rank whose CDF value exceeds u (numpy searchsorted side="right"), clipped
__device__ __forceinline__ int32_t cdf_upper_bound(const double *__restrict__ cdf, int32_t n, double u) {
  int32_t lo = 0, hi = n;
  while (lo < hi) {
    const int32_t mid = (int32_t)(((uint32_t)lo + (uint32_t)hi) >> 1);
    if (cdf[mid] <= u) lo = mid + 1; else hi = mid;
  }
  return lo < n ? lo : n - 1;
}
__global__ void k_synth_events(long long n_events, unsigned long long seed, const double *__restrict__ user_cdf,
                               const int32_t *__restrict__ user_perm, int32_t n_users, const double *__restrict__ item_cdf,
                               const int32_t *__restrict__ item_perm, int32_t n_items, long long *__restrict__ user,
                               int32_t *__restrict__ item) {
  const uint64_t base = mix64(seed);
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n_events; e += (long long)gridDim.x * blockDim.x) {
    const uint64_t h1 = mix64(base + (uint64_t)(e + 1) * 0x9e3779b97f4a7c15ULL);
    const uint64_t h2 = mix64(h1 ^ 0x6a09e667f3bcc909ULL);
    const double u1 = __dmul_rn((double)(h1 >> 11), 0x1.0p-53), u2 = __dmul_rn((double)(h2 >> 11), 0x1.0p-53);
    user[e] = user_perm[cdf_upper_bound(user_cdf, n_users, u1)];
    item[e] = item_perm[cdf_upper_bound(item_cdf, n_items, u2)];
  }
}

__global__ void k_max_i32(long long n, const int32_t *__restrict__ x, int32_t *__restrict__ out) {
  int32_t m = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    m = max(m, x[i]);
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(out, m);
}

// rank partition on the device: work of the rows outside this rank's [bounds[rank], bounds[rank + 1]) becomes 0, so they
// sort behind every row with work and fall out of the last bin; no bound ever travels to the host before the kernels run
__global__ void k_mask_work(int32_t n_items, const uint32_t *__restrict__ row_work, const int32_t *__restrict__ bounds, int rank,
                            uint32_t *__restrict__ masked) {
  const int32_t lo = bounds ? bounds[rank] : 0, hi = bounds ? bounds[rank + 1] : n_items;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_items; i += gridDim.x * blockDim.x)
    masked[i] = (i >= lo && i < hi) ? row_work[i] : 0u;
}

// kept-cell counts of this rank's rows as int64 (0 outside its range), input of the exclusive scan that gives row_ptr
__global__ void k_len_to_i64(int32_t n_items, const int32_t *__restrict__ len, const int32_t *__restrict__ bounds, int rank,
                             long long *__restrict__ out) {
  const int32_t lo = bounds ? bounds[rank] : 0, hi = bounds ? bounds[rank + 1] : n_items;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= n_items; i += gridDim.x * blockDim.x)
    out[i] = (i >= lo && i < hi) ? len[i] : 0;
}

// what the host needs from one indicator, in one mailbox record: [0] row_lo [1] row_hi [2] kept cells [3] products of the
// range [4] distinct cells [5] evaluated cells [6] hash-overflow flag
__global__ void k_indicator_record(int32_t n_items, const int32_t *__restrict__ bounds, int rank, const long long *__restrict__ out_ptr,
                                   const long long *__restrict__ work_prefix, const unsigned long long *__restrict__ distinct_eval,
                                   const int *__restrict__ err, long long *__restrict__ rec) {
  if (threadIdx.x || blockIdx.x) return;
  const int32_t lo = bounds ? bounds[rank] : 0, hi = bounds ? bounds[rank + 1] : n_items;
  rec[0] = lo;
  rec[1] = hi;
  rec[2] = out_ptr[n_items];
  rec[3] = work_prefix[hi] - work_prefix[lo];
  rec[4] = (long long)distinct_eval[0];
  rec[5] = (long long)distinct_eval[1];
  rec[6] = *err;
}

// group (single-process multi-GPU) mode: rebase this rank's row pointers by the cells of the ranks before it
__global__ void k_add_i64(long long n, long long v, long long *__restrict__ x) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) x[i] += v;
}

}  // namespace cco
