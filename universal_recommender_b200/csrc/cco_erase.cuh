// cco_erase.cuh -- erasure from a resident extendable log (cco_event_log_erase): the lines of the erased users and items are
// marked in a bitmap over the global lines, then dropped by the extend's finish pipeline (records, columns, property lines,
// aggregation, intern refit).  The erase sets are intern tables (cco_intern.cuh) built from the caller's ids.
//   k_erase_probe    each id of a column looked up in an intern table (k_str_hash's hash, exact bytes); a found id sets bit
//                    line[i] of bits (the entry's global line), or, without line, the bit of the key it found (the erase
//                    ids looked up in an interned log's own tables give key bitmaps)
//   k_erase_keys     interned logs: a training entry whose user key or item key is marked sets its line's bit (8 bytes
//                    per entry, no string reads)
//   k_erase_records  the records whose line is marked leave: keep flags, and the erased lines counted by selection
#pragma once

namespace cco {

__device__ __forceinline__ void erase_set_bit(uint32_t *__restrict__ bits, long long b) { atomicOr(&bits[b >> 5], 1u << (b & 31)); }

__global__ void k_erase_probe(long long n, const long long *__restrict__ off, const uint64_t *__restrict__ w, uint64_t mask,
                              const long long *__restrict__ koff, const uint64_t *__restrict__ kw, const uint64_t *__restrict__ khash,
                              uint64_t cap_mask, const uint32_t *__restrict__ table, const long long *__restrict__ line,
                              uint32_t *__restrict__ bits) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long a = off[i], len = off[i + 1] - a;
    const uint64_t h = str_hash_at(w, a, len) & mask;
    uint64_t s = (h ^ (h >> 29)) & cap_mask;
    while (true) {
      const uint32_t r = table[s];
      if (r == kStrEmpty) break;
      if (khash[r] == h && koff[r + 1] - koff[r] == len && str_equal(kw, koff[r], w, a, len)) {
        erase_set_bit(bits, line ? line[i] : (long long)r);
        break;
      }
      s = (s + 1) & cap_mask;
    }
  }
}

__global__ void k_erase_keys(long long n, const unsigned long long *__restrict__ tkey, const uint32_t *__restrict__ user_bits,
                             const uint32_t *__restrict__ item_bits, const long long *__restrict__ line, uint32_t *__restrict__ bitmap) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = tkey[e];
    const uint32_t u = (uint32_t)(k >> 32), i = (uint32_t)k;
    if (((user_bits[u >> 5] >> (u & 31)) & 1u) | ((item_bits[i >> 5] >> (i & 31)) & 1u)) erase_set_bit(bitmap, line[e]);
  }
}

// keep[i] = record i's line is not marked; cnt[0] += the erased records, cnt[1] += of them property events, cnt[2] += ignored
__global__ void k_erase_records(long long N, const WinRec *__restrict__ rec, const uint32_t *__restrict__ bitmap,
                                uint32_t *__restrict__ keep, unsigned long long *__restrict__ cnt) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long base = blockIdx.x * (long long)blockDim.x; base < N; base += stride) {
    const long long i = base + threadIdx.x;
    bool x = false;
    if (i < N) {
      const WinRec &r = rec[i];
      x = win_dropped(bitmap, r.line);
      keep[i] = x ? 0u : 1u;
      if (x && (r.flag & kEvProperty)) atomicAdd(&cnt[1], 1ULL);
      if (x && !r.flag) atomicAdd(&cnt[2], 1ULL);
    }
    const unsigned m = __ballot_sync(0xffffffffu, x);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(&cnt[0], (unsigned long long)__popc(m));
  }
}

}  // namespace cco
