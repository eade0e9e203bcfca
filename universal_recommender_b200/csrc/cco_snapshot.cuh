// cco_snapshot.cuh -- event log snapshots (cco_event_log_save / cco_event_log_load_*): the section checksums and the
// structural checks of a loaded snapshot, each one launch over every device section.
//
//   k_snap_sum    the 64-bit checksum of every section (include/cco_b200.h): each section's words are laid out from a
//                 multiple of 32 in one flat index space, so that every warp iteration reads one section; lanes reduce
//                 their terms in registers and flush one atomicAdd per warp when the section changes
//   k_snap_check  the structural checks of a loaded snapshot (SnapCheck kinds) over every checked section; the first
//                 violation, as (check << 40 | entry), goes to one mailbox verdict by atomicMin.  It reads the sections'
//                 own entries only, never bytes through an offset, so the host has its verdict before anything does.
#pragma once

namespace cco {

// splitmix64's finaliser; the checksum of len bytes is snap_mix(len) + sum over words i of snap_mix(w_i ^ i * kSnapGolden)
__host__ __device__ __forceinline__ uint64_t snap_mix(uint64_t x) {
  x ^= x >> 30;
  x *= 0xbf58476d1ce4e5b9ULL;
  x ^= x >> 27;
  x *= 0x94d049bb133111ebULL;
  return x ^ (x >> 31);
}
constexpr uint64_t kSnapGolden = 0x9e3779b97f4a7c15ULL;

// one device section: len bytes at p (8-byte aligned), its words at [at, at + ceil(len / 8)) of the flat index
struct SnapSpan {
  const unsigned char *p;
  long long len, at;
};

__device__ __forceinline__ uint64_t snap_word(const SnapSpan &sp, long long i) {
  const long long b = i * 8;
  if (b + 8 <= sp.len) return ((const uint64_t *)sp.p)[i];
  uint64_t w = 0;
  for (long long k = b; k < sp.len; ++k) w |= (uint64_t)sp.p[k] << (8 * (k - b));
  return w;
}

template <typename T>
__device__ __forceinline__ int snap_find(const T *__restrict__ sp, int n, long long q) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (sp[mid].at <= q) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// sum[s] += the word terms of section s (the caller adds snap_mix(len)); n_flat: the flat index space, a multiple of 32
__global__ void k_snap_sum(int n_spans, const SnapSpan *__restrict__ sp, long long n_flat, unsigned long long *__restrict__ sum) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5, n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
  int cur = -1;
  uint64_t acc = 0;
  for (long long base = warp * 32; base < n_flat; base += n_warps * 32) {
    const int s = snap_find(sp, n_spans, base);   // warp-uniform: sections start at multiples of 32
    if (s != cur) {
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (cur >= 0 && lane == 0) atomicAdd(&sum[cur], (unsigned long long)acc);
      acc = 0;
      cur = s;
    }
    const long long i = base + lane - sp[s].at;
    if (i * 8 < sp[s].len) acc += snap_mix(snap_word(sp[s], i) ^ ((uint64_t)i * kSnapGolden));
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (cur >= 0 && lane == 0) atomicAdd(&sum[cur], (unsigned long long)acc);
}

enum SnapCheck : int {
  kSnapOffsets = 0,   // int64 [n + 1]: 0 at 0, never decreasing, bound at n
  kSnapBelow = 1,     // int64 [n]: each in [0, bound)
  kSnapKeys = 2,      // uint64 [n]: user key (high half) < bound, item key (low half) < bound2
  kSnapFields = 3,    // int32 [n]: each in [0, bound)
  kSnapRecords = 4,   // WinRec [n]: lines in [0, bound) strictly increasing, names in [0, bound2)
};
struct SnapTask {
  const void *p;
  long long n, at;          // entries checked, their first index in the flat index space
  long long bound, bound2;
  int kind;
};

__global__ void k_snap_check(int n_tasks, const SnapTask *__restrict__ tk, long long n_flat, unsigned long long *__restrict__ bad) {
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < n_flat; q += (long long)gridDim.x * blockDim.x) {
    const int t = snap_find(tk, n_tasks, q);
    const SnapTask &k = tk[t];
    const long long i = q - k.at;
    if (i >= k.n) continue;
    bool ok = true;
    switch (k.kind) {
      case kSnapOffsets: {
        const long long *o = (const long long *)k.p, v = o[i];
        ok = (i > 0 || v == 0) && (i + 1 < k.n ? o[i + 1] >= v : v == k.bound);
        break;
      }
      case kSnapBelow: {
        const long long v = ((const long long *)k.p)[i];
        ok = v >= 0 && v < k.bound;
        break;
      }
      case kSnapKeys: {
        const unsigned long long v = ((const unsigned long long *)k.p)[i];
        ok = (long long)(v >> 32) < k.bound && (long long)(uint32_t)v < k.bound2;
        break;
      }
      case kSnapFields: {
        const int32_t v = ((const int32_t *)k.p)[i];
        ok = v >= 0 && v < k.bound;
        break;
      }
      default: {
        const WinRec *r = (const WinRec *)k.p;
        const long long line = r[i].line;
        ok = line >= 0 && line < k.bound && r[i].code >= 0 && r[i].code < k.bound2 && (i == 0 || r[i - 1].line < line);
        break;
      }
    }
    if (!ok) atomicMin(bad, ((unsigned long long)t << 40) | (unsigned long long)i);
  }
}

}  // namespace cco
