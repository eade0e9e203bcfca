// cco_strings.cuh -- string-keyed ingest (SURVEY.md 8f-1): Preparator.prepare on (user id, item id) byte strings.
//
// A column is n ids in the Arrow large_string layout: id i = bytes[off[i] - base .. off[i + 1] - base), the byte buffer
// uploaded into 8-byte words with 16 bytes of padding so that word loads may read past the last id.
//   k_str_check    offsets that decrease -> flag (the host checks off[0] >= 0 and off[0] <= off[n])
//   k_str_hash     64-bit keyed hash per id (mix64 over 8-byte words), truncated to `mask` (collision tests)
//   k_str_insert   open-addressing table over the ids: a slot holds the index of the id that claimed it; an id joins a slot
//                  when hash AND bytes are equal, so groups are exact whatever the hash does.  Per slot: first index
//                  (atomicMin) and, for the primary user column, the event count.  A gate (user id < 0) keeps dropped
//                  events out, which makes `first` the first *surviving* appearance of an item.
//   k_str_lookup   secondary user columns: probe the primary user table (read-only), -1 for unknown / filtered users
//   k_str_flags / k_str_compact / k_str_rank / k_str_ids   passing slots -> (first, slot), sorted by first = dictionary
//                  order, rank per slot, id per event
//   k_str_keys     (user << 32 | item) per surviving event, ~0 for dropped ones (the CSR tail of cco_ingest follows)
//   k_str_dict_len / k_str_dict_gather   dictionary strings (first appearance of each id) into one contiguous buffer
#pragma once

namespace cco {

constexpr uint32_t kStrEmpty = 0xffffffffu;

// word k of the id that starts at byte a of the word buffer
__device__ __forceinline__ uint64_t str_word(const uint64_t *__restrict__ w, long long a, long long k) {
  const long long q = (a >> 3) + k;
  const int sh = (int)(a & 7) * 8;
  const uint64_t lo = w[q];
  return sh ? (lo >> sh) | (w[q + 1] << (64 - sh)) : lo;
}
__device__ __forceinline__ uint64_t str_mask_tail(uint64_t x, long long remaining) {
  return remaining >= 8 ? x : x & ((1ULL << (8 * remaining)) - 1);
}
// bytes of id a (in wa) == bytes of id b (in wb), both of length len
__device__ __forceinline__ bool str_equal(const uint64_t *__restrict__ wa, long long a, const uint64_t *__restrict__ wb, long long b,
                                          long long len) {
  for (long long k = 0; k * 8 < len; ++k)
    if (str_mask_tail(str_word(wa, a, k) ^ str_word(wb, b, k), len - k * 8) != 0) return false;
  return true;
}

__global__ void k_str_check(long long n, const long long *__restrict__ off, int *__restrict__ bad) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    if (off[i + 1] < off[i]) *bad = 1;
}

// k_str_hash's hash of the id of len bytes at byte a of w, before the mask
__device__ __forceinline__ uint64_t str_hash_at(const uint64_t *__restrict__ w, long long a, long long len) {
  uint64_t h = 0x243f6a8885a308d3ULL;
  for (long long k = 0; k * 8 < len; ++k) h = mix64(h ^ str_mask_tail(str_word(w, a, k), len - k * 8)) + 0x9e3779b97f4a7c15ULL;
  return mix64(h ^ (uint64_t)len);
}
__global__ void k_str_hash(long long n, const long long *__restrict__ off, long long base, const uint64_t *__restrict__ w,
                           uint64_t mask, uint64_t *__restrict__ hash) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long a = off[i] - base, len = off[i + 1] - off[i];
    hash[i] = str_hash_at(w, a, len) & mask;
  }
}

__global__ void k_str_insert(long long n, const long long *__restrict__ off, long long base, const uint64_t *__restrict__ w,
                             const uint64_t *__restrict__ hash, const int32_t *__restrict__ gate, uint64_t cap_mask,
                             uint32_t *__restrict__ table, uint32_t *__restrict__ slot_of, uint32_t *__restrict__ first,
                             uint32_t *__restrict__ count) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (gate && gate[i] < 0) {
      slot_of[i] = kStrEmpty;
      continue;
    }
    const uint64_t h = hash[i];
    const long long a = off[i] - base, len = off[i + 1] - off[i];
    uint64_t s = (h ^ (h >> 29)) & cap_mask;
    while (true) {
      uint32_t r = table[s];
      if (r == kStrEmpty) {
        r = atomicCAS(&table[s], kStrEmpty, (uint32_t)i);
        if (r == kStrEmpty) break;   // claimed
      }
      // a claimed slot never changes: compare against the id that claimed it
      if (hash[r] == h && off[r + 1] - off[r] == len && str_equal(w, off[r] - base, w, a, len)) break;
      s = (s + 1) & cap_mask;
    }
    slot_of[i] = (uint32_t)s;
    atomicMin(&first[s], (uint32_t)i);
    if (count) atomicAdd(&count[s], 1u);
  }
}

__global__ void k_str_lookup(long long n, const long long *__restrict__ off, long long base, const uint64_t *__restrict__ w,
                             const uint64_t *__restrict__ hash, const long long *__restrict__ ref_off, long long ref_base,
                             const uint64_t *__restrict__ ref_w, const uint64_t *__restrict__ ref_hash, uint64_t cap_mask,
                             const uint32_t *__restrict__ table, const int32_t *__restrict__ rank_of_slot, int32_t *__restrict__ id) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const uint64_t h = hash[i];
    const long long a = off[i] - base, len = off[i + 1] - off[i];
    uint64_t s = (h ^ (h >> 29)) & cap_mask;
    int32_t out = -1;
    while (true) {
      const uint32_t r = table[s];
      if (r == kStrEmpty) break;
      if (ref_hash[r] == h && ref_off[r + 1] - ref_off[r] == len && str_equal(ref_w, ref_off[r] - ref_base, w, a, len)) {
        out = rank_of_slot[s];
        break;
      }
      s = (s + 1) & cap_mask;
    }
    id[i] = out;
  }
}

// flag[s] = 1 iff slot s holds an id that enters the dictionary (count == nullptr: every claimed slot)
__global__ void k_str_flags(long long cap, const uint32_t *__restrict__ table, const uint32_t *__restrict__ count, uint32_t need,
                            uint32_t *__restrict__ flag) {
  for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < cap; s += (long long)gridDim.x * blockDim.x)
    flag[s] = table[s] != kStrEmpty && (!count || count[s] >= need) ? 1u : 0u;
}
__global__ void k_str_compact(long long cap, const uint32_t *__restrict__ flag, const uint32_t *__restrict__ pos,
                              const uint32_t *__restrict__ first, uint32_t *__restrict__ key, uint32_t *__restrict__ slot) {
  for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < cap; s += (long long)gridDim.x * blockDim.x)
    if (flag[s]) {
      key[pos[s]] = first[s];
      slot[pos[s]] = (uint32_t)s;
    }
}
__global__ void k_str_rank(long long n_groups, const uint32_t *__restrict__ slot_sorted, int32_t *__restrict__ rank_of_slot) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < n_groups; k += (long long)gridDim.x * blockDim.x)
    rank_of_slot[slot_sorted[k]] = (int32_t)k;
}
__global__ void k_str_ids(long long n, const uint32_t *__restrict__ slot_of, const int32_t *__restrict__ rank_of_slot,
                          int32_t *__restrict__ id) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    id[i] = slot_of[i] == kStrEmpty ? -1 : rank_of_slot[slot_of[i]];
}

__global__ void k_str_keys(long long n, const int32_t *__restrict__ uid, const int32_t *__restrict__ iid,
                           unsigned long long *__restrict__ keys, unsigned long long *__restrict__ n_kept) {
  unsigned long long kept = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int32_t r = uid[i];
    if (r >= 0) {
      keys[i] = ((unsigned long long)(uint32_t)r << 32) | (uint32_t)iid[i];
      ++kept;
    } else {
      keys[i] = ~0ULL;
    }
  }
  for (int o = 16; o > 0; o >>= 1) kept += __shfl_xor_sync(0xffffffffu, kept, o);
  if ((threadIdx.x & 31) == 0 && kept) atomicAdd(n_kept, kept);
}

// dictionary entry k = the id at event first_sorted[k]; len[n_groups] is the scan's tail (set by the caller)
__global__ void k_str_dict_len(long long n_groups, const uint32_t *__restrict__ first_sorted, const long long *__restrict__ off,
                               long long *__restrict__ len) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < n_groups; k += (long long)gridDim.x * blockDim.x) {
    const uint32_t e = first_sorted[k];
    len[k] = off[e + 1] - off[e];
  }
}
__global__ void k_str_dict_gather(long long n_groups, const uint32_t *__restrict__ first_sorted, const long long *__restrict__ off,
                                  long long base, const unsigned char *__restrict__ bytes, const long long *__restrict__ out_off,
                                  unsigned char *__restrict__ out) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < n_groups; k += (long long)gridDim.x * blockDim.x) {
    const uint32_t e = first_sorted[k];
    const long long a = off[e] - base, len = off[e + 1] - off[e], o = out_off[k];
    for (long long j = 0; j < len; ++j) out[o + j] = bytes[a + j];
  }
}

}  // namespace cco
