// cco_clean.cuh -- a resident extendable log's cleaned events written back as a compacted export
// (cco_event_log_clean_*): a second streaming pass over the source bytes the log has read, which copies out the lines
// the log keeps.  The lines are parsed with the read's kernels (cco_events.cuh); the kernels here only select, check and
// copy them.
//   k_clean_first_code per chunk: the first line of an event name the log does not know
//   k_clean_bitmap    at begin: one bit per global line the log read, set for the line of every retained record
//   k_clean_keep      per chunk: keep[l] = the bit of the chunk's line l
//   k_clean_check     per chunk: each kept line against its record (eventTime, event name, selection, and under
//                     removeDuplicates the 128-bit identity) -> the first mismatching global line into the error word
//   k_clean_len       per chunk: each kept line's output bytes (0 for a line compressProperties folds)
//   k_clean_compact   per chunk: the kept lines' bytes, each followed by one '\n', packed into the output; one warp per
//                     line over the output's 8-byte words, so that no thread walks a long line
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace cco {

// mismatch kinds of a kept line (the low byte of the error word; the global line above it)
enum : unsigned { kClTime = 1, kClName = 2, kClSelection = 3, kClIdentity = 4 };

__global__ void k_clean_bitmap(long long n, const WinRec *__restrict__ rec, uint32_t *__restrict__ bitmap) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    atomicOr(&bitmap[rec[i].line >> 5], 1u << (rec[i].line & 31));
}
__global__ void k_clean_keep(long long n, long long base, const uint32_t *__restrict__ bitmap, uint32_t *__restrict__ keep) {
  for (long long l = blockIdx.x * (long long)blockDim.x + threadIdx.x; l < n; l += (long long)gridDim.x * blockDim.x) {
    const long long g = base + l;
    keep[l] = (bitmap[g >> 5] >> (g & 31)) & 1u;
  }
}
// *first = min line l with code[l] == k (a name the log does not know)
__global__ void k_clean_first_code(long long n, const int32_t *__restrict__ code, int32_t k, unsigned long long *__restrict__ first) {
  for (long long l = blockIdx.x * (long long)blockDim.x + threadIdx.x; l < n; l += (long long)gridDim.x * blockDim.x)
    if (code[l] == k) atomicMin(first, (unsigned long long)l);
}
// kept line k (chunk line idx[k]) is record rec[k]; ident (removeDuplicates: the line's own record, hashed as the read
// hashed it, else null) carries the identity to compare
__global__ void k_clean_check(long long n, const uint32_t *__restrict__ idx, long long base, const WinRec *__restrict__ rec,
                              const long long *__restrict__ tm, const uint8_t *__restrict__ flag, const int32_t *__restrict__ code,
                              const WinRec *__restrict__ ident, unsigned long long *__restrict__ err) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
    const long long l = idx[k];
    const WinRec &r = rec[k];
    unsigned bad = 0;
    if (tm[l] != r.time) bad = kClTime;
    else if (code[l] != r.code) bad = kClName;
    else if ((uint32_t)flag[l] != r.flag) bad = kClSelection;
    else if (ident && (ident[k].h0 != r.h0 || ident[k].h1 != r.h1)) bad = kClIdentity;
    if (bad) atomicMin(err, ((unsigned long long)(base + l) << 8) | bad);
  }
}
// len[k] = the output bytes of kept line k: its bytes and a '\n', none for a line folded by compressProperties (fold: a
// bitmap over the global lines, null without compression)
__global__ void k_clean_len(long long n, const uint32_t *__restrict__ idx, long long base, const long long *__restrict__ sb,
                            const long long *__restrict__ se, const uint32_t *__restrict__ fold, long long *__restrict__ len) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
    const long long l = idx[k], g = base + l;
    len[k] = fold && ((fold[g >> 5] >> (g & 31)) & 1u) ? 0 : se[l] - sb[l] + 1;
  }
}
// kept line k: the bytes [sb, se) of chunk line idx[k] and a '\n' to out[off[k], off[k + 1]) (none when that is empty).  The words wholly inside
// the line are stored whole (a funnel shift of two source words); the first and last words, which it may share with its
// neighbours, byte by byte.  w: the staging as words (24 bytes of padding); out: 8-byte aligned.
__global__ void k_clean_compact(long long n, const uint32_t *__restrict__ idx, const long long *__restrict__ sb, const long long *__restrict__ se,
                                const uint64_t *__restrict__ w, const long long *__restrict__ off, unsigned char *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const unsigned char *src = (const unsigned char *)w;
  for (long long k = warp; k < n; k += nwarps) {
    const long long l = idx[k], b = sb[l], o = off[k], e = off[k + 1];   // '\n' at e - 1
    if (e == o) continue;
    for (long long q = (o >> 3) + lane; q * 8 < e; q += 32) {
      const long long p = q * 8;
      if (p >= o && p + 8 <= e) {
        uint64_t x = str_word(w, b + (p - o), 0);
        if (p + 8 == e) x = (x & 0x00ffffffffffffffULL) | (0x0aULL << 56);
        ((uint64_t *)out)[q] = x;
      } else {
        for (long long j = p > o ? p : o; j < p + 8 && j < e; ++j) out[j] = j == e - 1 ? '\n' : src[b + (j - o)];
      }
    }
  }
}

// ---- compressProperties (CCO_CLEAN_COMPRESS_PROPERTIES), at begin over the log's retained item property lines ----------
// Lines 0 .. L-1 are the log's property lines (line order), gcode[l] the exact group of their decoded entityId.
//   k_fold_count    per group: $set / $unset lines and a pin ($delete, or a $set / $unset with a target)
//   k_fold_lines    the $set / $unset lines of foldable groups (not pinned, two or more): flag, fold bitmap over the global lines
//   k_fold_keys     sort keys of the fold order: (eventTime, line), then the group's output rank
//   k_fold_first    per folded group: the first $set's and the last line's place in the fold order
//   k_fold_mkeys    sort keys of the members: (fold place, member index), then (group rank, name)
//   k_fold_runs     one thread per (group, name) run, in fold order: does the name end up in the line, where was it inserted
//                   (Python dict order: {**cur, **props}, removed by an $unset after the first $set), and its last value
//   k_fold_render   size pass and write pass of the folded lines, one thread per line
enum : uint8_t { kFoldLine = 1, kFoldSet = 2 };
__global__ void k_fold_count(long long L, const uint8_t *__restrict__ flag, const int32_t *__restrict__ gcode, uint32_t *__restrict__ cnt,
                             uint32_t *__restrict__ pin) {
  for (long long l = blockIdx.x * (long long)blockDim.x + threadIdx.x; l < L; l += (long long)gridDim.x * blockDim.x) {
    const uint8_t f = flag[l];
    const int g = gcode[l];
    if ((f & kEvDelete) || ((f & (kEvSet | kEvUnset)) && (f & kEvRanking))) pin[g] = 1;
    else if (f & (kEvSet | kEvUnset)) atomicAdd(&cnt[g], 1u);
  }
}
__global__ void k_fold_groups(long long G, const uint32_t *__restrict__ cnt, const uint32_t *__restrict__ pin, uint32_t *__restrict__ keep) {
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < G; g += (long long)gridDim.x * blockDim.x)
    keep[g] = !pin[g] && cnt[g] >= 2 ? 1u : 0u;
}
// fl[l] = kFoldLine (| kFoldSet) for a folded line, its global line into the fold bitmap
__global__ void k_fold_lines(long long L, const uint8_t *__restrict__ flag, const int32_t *__restrict__ gcode, const uint32_t *__restrict__ gkeep,
                             const long long *__restrict__ gline, uint8_t *__restrict__ fl, uint32_t *__restrict__ bitmap) {
  for (long long l = blockIdx.x * (long long)blockDim.x + threadIdx.x; l < L; l += (long long)gridDim.x * blockDim.x) {
    uint8_t x = 0;
    if (gkeep[gcode[l]] && (flag[l] & (kEvSet | kEvUnset))) {
      x = kFoldLine | ((flag[l] & kEvSet) ? kFoldSet : 0);
      atomicOr(&bitmap[gline[l] >> 5], 1u << (gline[l] & 31));
    }
    fl[l] = x;
  }
}
// the F folded lines idx[i]: key1 = eventTime (signed order), key2 = the group's rank among the folded groups
__global__ void k_fold_keys(long long F, const uint32_t *__restrict__ idx, const long long *__restrict__ tm, const int32_t *__restrict__ gcode,
                            const uint32_t *__restrict__ grank, unsigned long long *__restrict__ key1, uint32_t *__restrict__ key2,
                            uint32_t *__restrict__ val) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < F; i += (long long)gridDim.x * blockDim.x) {
    key1[i] = (unsigned long long)tm[idx[i]] ^ 0x8000000000000000ULL;
    key2[i] = grank[gcode[idx[i]]];
    val[i] = (uint32_t)i;
  }
}
__global__ void k_fold_key2(long long F, const uint32_t *__restrict__ val, const uint32_t *__restrict__ key2, uint32_t *__restrict__ out) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < F; k += (long long)gridDim.x * blockDim.x) out[k] = key2[val[k]];
}
// place[i] = the fold place of folded line i (its position in the sorted order); per group rank r: first_set[r] = the
// least place of a $set, last[r] = the folded line at its last place
__global__ void k_fold_first(long long F, const uint32_t *__restrict__ sorted, const uint32_t *__restrict__ gr, const uint32_t *__restrict__ idx,
                             const uint8_t *__restrict__ fl, uint32_t *__restrict__ place, uint32_t *__restrict__ first_set,
                             uint32_t *__restrict__ last) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < F; k += (long long)gridDim.x * blockDim.x) {
    const uint32_t i = sorted[k], r = gr[k];
    place[i] = (uint32_t)k;
    if (fl[idx[i]] & kFoldSet) atomicMin(&first_set[r], (uint32_t)k);
    if (k + 1 == F || gr[k + 1] != r) last[r] = i;
  }
}
// member m (of folded line mline[m], its index m - moff[mline[m]] in the line): key1 = (place, index), key2 = (rank, name)
__global__ void k_fold_mkeys(long long M, const uint32_t *__restrict__ mline, const long long *__restrict__ moff, const uint32_t *__restrict__ place,
                             const uint32_t *__restrict__ rank_of_line, const int32_t *__restrict__ ncode, unsigned long long *__restrict__ key1,
                             unsigned long long *__restrict__ key2, uint32_t *__restrict__ val) {
  for (long long m = blockIdx.x * (long long)blockDim.x + threadIdx.x; m < M; m += (long long)gridDim.x * blockDim.x) {
    const uint32_t i = mline[m];
    key1[m] = ((unsigned long long)place[i] << 32) | (uint32_t)(m - moff[i]);
    key2[m] = ((unsigned long long)rank_of_line[i] << 32) | (uint32_t)ncode[m];
    val[m] = (uint32_t)m;
  }
}
__global__ void k_fold_mkey2(long long M, const uint32_t *__restrict__ val, const unsigned long long *__restrict__ key2, unsigned long long *__restrict__ out) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < M; k += (long long)gridDim.x * blockDim.x) out[k] = key2[val[k]];
}
// members sorted by (rank, name, place, index): the thread at the start of each run walks it.  keep[k] = the name is in
// the folded line; ins[k] = (place, index) of its insertion; vm[k] = the member whose value it has
__global__ void k_fold_runs(long long M, const unsigned long long *__restrict__ key2, const uint32_t *__restrict__ val,
                            const uint32_t *__restrict__ mline, const long long *__restrict__ moff, const uint32_t *__restrict__ place,
                            const uint32_t *__restrict__ idx, const uint8_t *__restrict__ fl, const uint32_t *__restrict__ first_set,
                            uint32_t *__restrict__ keep, unsigned long long *__restrict__ ins, uint32_t *__restrict__ vm) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < M; k += (long long)gridDim.x * blockDim.x) {
    keep[k] = 0;
    if (k > 0 && key2[k - 1] == key2[k]) continue;
    const uint32_t r = (uint32_t)(key2[k] >> 32), fs = first_set[r];
    const bool set_group = fs != 0xffffffffu;
    bool present = false;
    unsigned long long at = 0;
    uint32_t v = 0;
    for (long long j = k; j < M && key2[j] == key2[k]; ++j) {
      const uint32_t m = val[j], i = mline[m];
      const unsigned long long here = ((unsigned long long)place[i] << 32) | (uint32_t)(m - moff[i]);
      const bool is_set = fl[idx[i]] & kFoldSet;
      if (!set_group || is_set) {
        if (!present) at = here;
        present = true;
        v = m;
      } else if (place[i] > fs) {   // an $unset after the first $set
        present = false;
      }
    }
    keep[k] = present ? 1u : 0u;
    ins[k] = at;
    vm[k] = v;
  }
}
// the P kept runs kidx[p]: their insertion key, group rank and value member, a permutation to sort, and the count per rank
__global__ void k_fold_okeys(long long P, const uint32_t *__restrict__ kidx, const unsigned long long *__restrict__ key2,
                             const unsigned long long *__restrict__ ins, const uint32_t *__restrict__ vm, unsigned long long *__restrict__ k1,
                             uint32_t *__restrict__ r32, uint32_t *__restrict__ val, uint32_t *__restrict__ perm, uint32_t *__restrict__ cnt) {
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < P; p += (long long)gridDim.x * blockDim.x) {
    const uint32_t k = kidx[p];
    k1[p] = ins[k];
    r32[p] = (uint32_t)(key2[k] >> 32);
    val[p] = vm[k];
    perm[p] = (uint32_t)p;
    atomicAdd(&cnt[r32[p]], 1u);
  }
}
__global__ void k_fold_gather2(long long n, const uint32_t *__restrict__ perm, const uint32_t *__restrict__ a, const uint32_t *__restrict__ b,
                               uint32_t *__restrict__ a2, uint32_t *__restrict__ b2) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
    a2[k] = a[perm[k]];
    b2[k] = b[perm[k]];
  }
}
// out[r] = cnt[r] (r < R), out[R] = 0: the members per folded line, for the exclusive sum
__global__ void k_fold_count64(long long R, const uint32_t *__restrict__ cnt, long long *__restrict__ out) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r <= R; r += (long long)gridDim.x * blockDim.x)
    out[r] = r < R ? (long long)cnt[r] : 0;
}
// folded line r: the first property line of its group (gidx[r]) and the length of that line's decoded entityId
__global__ void k_fold_group_line(long long R, const uint32_t *__restrict__ gidx, const uint32_t *__restrict__ first_sorted,
                                  uint32_t *__restrict__ first_line, const long long *__restrict__ id_off, long long *__restrict__ len) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < R; r += (long long)gridDim.x * blockDim.x) {
    const uint32_t l = first_sorted[gidx[r]];
    first_line[r] = l;
    len[r] = id_off[l + 1] - id_off[l];
  }
}
// folded line r: {"event":"$set"|"$unset","entityType":"item","entityId":<id>,"properties":{<name>:<value>,...},
// "eventTime":<the last folded event's eventTime text>}\n; strings through json4s' quote (uq_escape).  kWrite false: the
// lengths into len[r]
template <bool kWrite>
__global__ void k_fold_render(long long R, const uint32_t *__restrict__ last, const uint32_t *__restrict__ first_set, const uint32_t *__restrict__ idx,
                              const long long *__restrict__ sb, const int2 *__restrict__ span, const unsigned char *__restrict__ pb,
                              const long long *__restrict__ id_off, const unsigned char *__restrict__ id_bytes, const long long *__restrict__ gmoff,
                              const uint32_t *__restrict__ members, const long long *__restrict__ name_off, const unsigned char *__restrict__ names,
                              const JMember *__restrict__ mem, const long long *__restrict__ off, long long *__restrict__ len,
                              unsigned char *__restrict__ out) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < R; r += (long long)gridDim.x * blockDim.x) {
    unsigned char *o = kWrite ? out + off[r] : nullptr;
    long long n = 0;
    auto lit = [&](const char *x) {
      for (; *x; ++x, ++n)
        if (kWrite) o[n] = (unsigned char)*x;
    };
    auto raw = [&](long long b, long long e) {
      for (long long q = b; q < e; ++q, ++n)
        if (kWrite) o[n] = pb[q];
    };
    auto quoted = [&](const unsigned char *s, long long k) {
      lit("\"");
      n += uq_escape(s, k, kWrite ? o + n : nullptr);
      lit("\"");
    };
    lit(first_set[r] != 0xffffffffu ? "{\"event\":\"$set\"" : "{\"event\":\"$unset\"");
    lit(",\"entityType\":\"item\",\"entityId\":");
    quoted(id_bytes + id_off[r], id_off[r + 1] - id_off[r]);
    lit(",\"properties\":{");
    for (long long j = gmoff[r]; j < gmoff[r + 1]; ++j) {
      const uint32_t m = members[j];
      if (j > gmoff[r]) lit(",");
      quoted(names + name_off[m], name_off[m + 1] - name_off[m]);
      lit(":");
      raw(mem[m].vb, mem[m].ve);
    }
    lit("},\"eventTime\":");
    const uint32_t l = idx[last[r]];
    const int2 t = span[l * kEvSlots + kEvTime];
    raw(sb[l] + t.x, sb[l] + t.y);
    lit("}\n");
    if (!kWrite) len[r] = n;
  }
}

}  // namespace cco
