// cco_intern.cuh -- interned event logs (CCO_LOG_INTERN_IDS): every distinct user id and item id of the training entries
// has a 32-bit key, so that cco_event_log_ingest builds its dictionaries and matrices with integer passes only.
//
// An intern table is open addressing over k_str_hash's hash of the id, with an exact byte compare against the table's
// string heap (the 8-byte-word layout of DevStrCol, 16 bytes of padding); a slot holds a key, or, while a chunk is being
// interned, kInternNew | the chunk entry that claimed it.  Per chunk:
//   k_intern_claim     each entry finds its string's key, or claims a slot for it; entries of one new string keep the
//                      smallest entry index (atomicMin), which makes the numbering deterministic
//   k_intern_first     flag the entries that own a claimed slot: the chunk's new strings, in first-appearance order
//   k_intern_new       the flagged entries' slots become keys n_old + k; their hashes are stored for rehashing
//   k_intern_keys      each entry's key into one 32-bit half of the entry's (user key << 32 | item key) word
//   k_intern_heap_off  the new strings' heap offsets (their bytes follow through k_str_dict_gather)
//   k_intern_rehash    a table rebuilt from the stored hashes (growth, and the refit at finish)
// At finish (the refit to the live keys):
//   k_intern_live      mark the keys the retained entries hold
//   k_intern_remap     renumber the entries' keys by the scan of the marks
// Key-path ingest, over direct-indexed arrays of the key space:
//   k_intern_first_count  first entry (atomicMin) and, for primary users, the entry count of every key, warp-aggregated
//                         with __match_any_sync (ids are power-law distributed)
//   k_intern_ids          each entry's dictionary id through the key's rank (-1: gated, or the key is not in the dictionary)
#pragma once

namespace cco {

constexpr uint32_t kInternNew = 0x80000000u;

__global__ void k_intern_claim(long long n, const long long *__restrict__ off, const uint64_t *__restrict__ w,
                               const uint64_t *__restrict__ hash, const long long *__restrict__ koff, const uint64_t *__restrict__ kw,
                               const uint64_t *__restrict__ khash, uint64_t cap_mask, uint32_t *__restrict__ table,
                               uint32_t *__restrict__ slot_of) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const uint64_t h = hash[i];
    const long long a = off[i], len = off[i + 1] - a;
    uint64_t s = (h ^ (h >> 29)) & cap_mask;
    while (true) {
      uint32_t r = table[s];
      if (r == kStrEmpty) {
        r = atomicCAS(&table[s], kStrEmpty, kInternNew | (uint32_t)i);
        if (r == kStrEmpty) break;   // claimed
      }
      if (r & kInternNew) {
        // claimed in this chunk: the slot only ever moves to a smaller entry of the same string
        const long long j = r & ~kInternNew;
        if (hash[j] == h && off[j + 1] - off[j] == len && str_equal(w, off[j], w, a, len)) {
          atomicMin(&table[s], kInternNew | (uint32_t)i);
          break;
        }
      } else if (khash[r] == h && koff[r + 1] - koff[r] == len && str_equal(kw, koff[r], w, a, len)) {
        break;
      }
      s = (s + 1) & cap_mask;
    }
    slot_of[i] = (uint32_t)s;
  }
}
__global__ void k_intern_first(long long n, const uint32_t *__restrict__ slot_of, const uint32_t *__restrict__ table,
                               uint32_t *__restrict__ flag) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    flag[i] = table[slot_of[i]] == (kInternNew | (uint32_t)i) ? 1u : 0u;
}
__global__ void k_intern_new(long long k_new, const uint32_t *__restrict__ idx, const uint32_t *__restrict__ slot_of,
                             const uint64_t *__restrict__ hash, uint32_t n_old, uint32_t *__restrict__ table, uint64_t *__restrict__ khash) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < k_new; k += (long long)gridDim.x * blockDim.x) {
    const uint32_t i = idx[k];
    table[slot_of[i]] = n_old + (uint32_t)k;
    khash[n_old + k] = hash[i];
  }
}
// key of entry i -> half[2 i] (half: the user or the item half of the entries' 64-bit key words)
__global__ void k_intern_keys(long long n, const uint32_t *__restrict__ slot_of, const uint32_t *__restrict__ table,
                              uint32_t *__restrict__ half) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    half[2 * i] = table[slot_of[i]];
}
// koff[k] = at + off[k] for k in [0, n]
__global__ void k_intern_heap_off(long long n, const long long *__restrict__ off, long long at, long long *__restrict__ koff) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k <= n; k += (long long)gridDim.x * blockDim.x)
    koff[k] = at + off[k];
}
__global__ void k_intern_rehash(long long n_keys, const uint64_t *__restrict__ khash, uint64_t cap_mask, uint32_t *__restrict__ table) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < n_keys; k += (long long)gridDim.x * blockDim.x) {
    const uint64_t h = khash[k];
    uint64_t s = (h ^ (h >> 29)) & cap_mask;
    while (atomicCAS(&table[s], kStrEmpty, (uint32_t)k) != kStrEmpty) s = (s + 1) & cap_mask;
  }
}

__global__ void k_intern_live(long long n, const unsigned long long *__restrict__ tkey, uint32_t *__restrict__ live_u,
                              uint32_t *__restrict__ live_i) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = tkey[e];
    live_u[k >> 32] = 1u;
    live_i[(uint32_t)k] = 1u;
  }
}
__global__ void k_intern_remap(long long n, const uint32_t *__restrict__ new_u, const uint32_t *__restrict__ new_i,
                               unsigned long long *__restrict__ tkey) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = tkey[e];
    tkey[e] = ((unsigned long long)new_u[k >> 32] << 32) | new_i[(uint32_t)k];
  }
}

// key2[2 e]: the key of entry e.  The lanes of one key in a warp hold consecutive entries, so its lowest lane holds the
// smallest of them.
__global__ void k_intern_first_count(long long n, const uint32_t *__restrict__ key2, const int32_t *__restrict__ gate,
                                     uint32_t *__restrict__ first, uint32_t *__restrict__ count) {
  const int lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long base = blockIdx.x * (long long)blockDim.x; base < n; base += stride) {
    const long long e = base + threadIdx.x;
    const long long k = e < n && (!gate || gate[e] >= 0) ? (long long)key2[2 * e] : -1;
    const unsigned same = __match_any_sync(0xffffffffu, k);
    if (k >= 0 && lane == __ffs(same) - 1) {
      atomicMin(&first[k], (uint32_t)e);
      if (count) atomicAdd(&count[k], (uint32_t)__popc(same));
    }
  }
}
__global__ void k_intern_ids(long long n, const uint32_t *__restrict__ key2, const int32_t *__restrict__ gate,
                             const int32_t *__restrict__ rank, int32_t *__restrict__ id) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x)
    id[e] = gate && gate[e] < 0 ? -1 : rank[key2[2 * e]];
}

}  // namespace cco
