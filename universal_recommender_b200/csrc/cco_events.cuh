// cco_events.cuh -- a PredictionIO event export (`pio export`: JSON lines, one event per line) parsed on the device
// (cco_event_log_read), the DataSource of the reference (DataSource.scala:65-102) without its event store.
//   k_json_members + EventSink     the tokenizer of cco_json.cuh with a sink that keeps, per line, the value spans of the
//                                  seven members an event is read through (the last of a repeated name), nothing else
//   k_event_check                  per line: member types, eventTime -> epoch ms, the selection (training / ranking /
//                                  property event) and the empty-id rule, verdict into the error word
//   k_event_strings                the inside of one member's string per line (or per listed line) as JMember spans for
//                                  k_json_unescape
//   k_event_keys / k_event_counts  partition keys by event name, per-name counts of training and ranking events
//   k_prop_*                       PEventStore.aggregateProperties of the items' $set / $unset / $delete events: the
//                                  (eventTime, line) order, the last $delete and $set per item, the members of the
//                                  properties objects sorted by (item, field) after that order, the winning member per
//                                  (item, field), one presence entry per item left without a field, the triples
//   k_line_len / k_line_gather     streamed reads: the property-event lines of each chunk, kept for the aggregation at finish
//   k_cat_words / k_cat_entries    streamed reads: the chunks' name-partitioned columns concatenated name-major at finish
//   k_ext_*                        extendable logs: the retained part re-expired under a later cutoff at each finish
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace cco {

// the members of an event line that are read; every other member is skipped
enum : int { kEvName = 0, kEvEntityType, kEvEntityId, kEvTargetType, kEvTargetId, kEvTime, kEvProps, kEvSlots };
// error codes of an event line (after the tokenizer's kJson* codes)
enum : unsigned { kEvMissing = 6, kEvType = 7, kEvTime_ = 8, kEvEmptyId = 9, kEvTarget = 10 };
// line flags
enum : uint8_t { kEvTraining = 1, kEvRanking = 2, kEvProperty = 4, kEvSet = 8, kEvUnset = 16, kEvDelete = 32, kEvPropObj = 64 };

// the next decoded unit of the raw string bytes [q, e) (escapes validated by the tokenizer): a code point for an escape,
// else the raw byte (a UTF-8 lead or continuation byte is >= 0x80 and never equals an ASCII unit)
__device__ __forceinline__ unsigned json_next_unit(const unsigned char *__restrict__ body, long long &q) {
  const unsigned c = body[q];
  if (c != '\\') {
    ++q;
    return c;
  }
  const unsigned x = body[q + 1];
  if (x != 'u') {
    q += 2;
    return x == 'b' ? 8 : x == 'f' ? 12 : x == 'n' ? 10 : x == 'r' ? 13 : x == 't' ? 9 : x;
  }
  const unsigned cp = json_hex4(body + q + 2);
  q += 6;
  return cp;   // a surrogate stays >= 0x80: it never equals an ASCII literal
}
// the raw string bytes [q, e) decode to the ASCII literal lit of n bytes
__device__ __forceinline__ bool json_str_is(const unsigned char *__restrict__ body, long long q, long long e, const char *lit, int n) {
  for (int k = 0; k < n; ++k) {
    if (q >= e || json_next_unit(body, q) != (unsigned char)lit[k]) return false;
  }
  return q == e;
}

__device__ __forceinline__ int event_slot(const unsigned char *__restrict__ body, long long nb, long long ne) {
  if (json_str_is(body, nb, ne, "event", 5)) return kEvName;
  if (json_str_is(body, nb, ne, "entityType", 10)) return kEvEntityType;
  if (json_str_is(body, nb, ne, "entityId", 8)) return kEvEntityId;
  if (json_str_is(body, nb, ne, "targetEntityType", 16)) return kEvTargetType;
  if (json_str_is(body, nb, ne, "targetEntityId", 14)) return kEvTargetId;
  if (json_str_is(body, nb, ne, "eventTime", 9)) return kEvTime;
  if (json_str_is(body, nb, ne, "properties", 10)) return kEvProps;
  return -1;
}
// span[l * kEvSlots + k] = value of member k of line l relative to the line's first byte, {-1, -1} when absent (memset
// by the caller); members arrive in order, so the last of a repeated name wins
struct EventSink {
  int2 *span;
  const unsigned char *body;
  __device__ void member(long long s, long long, long long b, const JMember &m) const {
    const int k = event_slot(body, m.nb, m.ne);
    if (k >= 0) span[s * kEvSlots + k] = make_int2((int)(m.vb - b), (int)(m.ve - b));
  }
  __device__ void end(long long, long long) const {}
};

// the value [vb, ve) is exactly one string
__device__ __forceinline__ bool json_is_string(const unsigned char *__restrict__ body, long long vb, long long ve) {
  if (ve - vb < 2 || body[vb] != '"') return false;
  long long q = vb + 1;
  while (q < ve - 1) {
    if (body[q] == '\\') q += 2;
    else if (body[q] == '"') return false;
    else ++q;
  }
  return q == ve - 1 && body[q] == '"';
}
__device__ __forceinline__ bool json_is_null(const unsigned char *__restrict__ body, long long vb, long long ve) {
  return ve - vb == 4 && body[vb] == 'n' && body[vb + 1] == 'u' && body[vb + 2] == 'l' && body[vb + 3] == 'l';
}

// Joda's extended date-time YYYY-MM-DDThh:mm:ss[.f{1,9}](Z|+hh:mm|+hhmm|+hh) (sign + or -), proleptic Gregorian,
// years 0000-9999 -> epoch milliseconds; fraction digits past the third are dropped (a floor: the fraction is positive)
__device__ __forceinline__ long long days_from_civil(long long y, unsigned m, unsigned d) {
  y -= m <= 2;
  const long long era = (y >= 0 ? y : y - 399) / 400;
  const unsigned yoe = (unsigned)(y - era * 400);
  const unsigned doy = (153 * (m + (m > 2 ? -3 : 9)) + 2) / 5 + d - 1;
  const unsigned doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
  return era * 146097 + (long long)doe - 719468;
}
__device__ __noinline__ bool parse_event_time(const unsigned char *__restrict__ body, long long q, long long e, long long *ms) {
  char t[40];
  int n = 0;
  while (q < e) {
    if (n == 40) return false;
    const unsigned u = json_next_unit(body, q);
    if (u >= 0x80) return false;
    t[n++] = (char)u;
  }
  auto dig = [&](int i, int k, int *v) {
    int x = 0;
    for (int j = i; j < i + k; ++j) {
      if (j >= n || t[j] < '0' || t[j] > '9') return false;
      x = x * 10 + (t[j] - '0');
    }
    *v = x;
    return true;
  };
  int Y, M, D, h, mi, s;
  if (n < 20 || !dig(0, 4, &Y) || t[4] != '-' || !dig(5, 2, &M) || t[7] != '-' || !dig(8, 2, &D) || t[10] != 'T' || !dig(11, 2, &h) ||
      t[13] != ':' || !dig(14, 2, &mi) || t[16] != ':' || !dig(17, 2, &s))
    return false;
  const bool leap = Y % 4 == 0 && (Y % 100 != 0 || Y % 400 == 0);
  const int mdays = M == 2 ? (leap ? 29 : 28) : (M == 4 || M == 6 || M == 9 || M == 11) ? 30 : 31;
  if (M < 1 || M > 12 || D < 1 || D > mdays || h > 23 || mi > 59 || s > 59) return false;
  int i = 19, frac = 0;
  if (t[i] == '.') {
    int k = 0;
    for (++i; i < n && t[i] >= '0' && t[i] <= '9'; ++i, ++k)
      if (k < 3) frac = frac * 10 + (t[i] - '0');
    if (k < 1 || k > 9) return false;
    for (; k < 3; ++k) frac *= 10;
  }
  int off = 0;
  if (i < n && t[i] == 'Z') {
    ++i;
  } else if (i < n && (t[i] == '+' || t[i] == '-')) {
    const int sign = t[i] == '-' ? -1 : 1;
    int oh, om = 0;
    if (!dig(i + 1, 2, &oh)) return false;
    i += 3;
    if (i < n && t[i] == ':') {
      if (!dig(i + 1, 2, &om)) return false;
      i += 3;
    } else if (i < n) {
      if (!dig(i, 2, &om)) return false;
      i += 2;
    }
    if (oh > 23 || om > 59) return false;
    off = sign * (oh * 60 + om);
  } else {
    return false;
  }
  if (i != n) return false;
  *ms = ((days_from_civil(Y, (unsigned)M, (unsigned)D) * 86400 + h * 3600 + mi * 60 + s) - (long long)off * 60) * 1000 + frac;
  return true;
}

// per line: types, time, selection; flags and times written for every line, the verdict into err
__global__ void k_event_check(long long n_lines, const long long *__restrict__ sb, const int2 *__restrict__ span,
                              const unsigned char *__restrict__ body, uint8_t *__restrict__ flag, long long *__restrict__ time,
                              unsigned long long *__restrict__ err) {
  for (long long l = blockIdx.x * (long long)blockDim.x + threadIdx.x; l < n_lines; l += (long long)gridDim.x * blockDim.x) {
    const long long b = sb[l];
    const int2 *sp = span + l * kEvSlots;
    unsigned code = 0;
    auto vb = [&](int k) { return b + sp[k].x; };
    auto ve = [&](int k) { return b + sp[k].y; };
    auto present = [&](int k) { return sp[k].x >= 0; };
    auto str = [&](int k) { return present(k) && json_is_string(body, vb(k), ve(k)); };
    // an optional string: absent or null counts as absent
    auto opt = [&](int k) { return present(k) && !json_is_null(body, vb(k), ve(k)); };
    for (int k : {kEvName, kEvEntityType, kEvEntityId, kEvTime})
      if (!code && !present(k)) code = kEvMissing;
    for (int k : {kEvName, kEvEntityType, kEvEntityId, kEvTime})
      if (!code && !str(k)) code = kEvType;
    for (int k : {kEvTargetType, kEvTargetId})
      if (!code && opt(k) && !str(k)) code = kEvType;
    if (!code && present(kEvProps) && (body[vb(kEvProps)] != '{' || body[ve(kEvProps) - 1] != '}')) code = kEvType;
    if (!code && opt(kEvTargetType) != opt(kEvTargetId)) code = kEvTarget;
    long long tm = 0;
    if (!code && !parse_event_time(body, vb(kEvTime) + 1, ve(kEvTime) - 1, &tm)) code = kEvTime_;
    uint8_t f = 0;
    if (!code) {
      const bool target = opt(kEvTargetId);
      const long long etb = vb(kEvEntityType) + 1, ete = ve(kEvEntityType) - 1;
      if (target) {
        f |= kEvRanking;
        const bool train = json_str_is(body, etb, ete, "user", 4) &&
                           json_str_is(body, vb(kEvTargetType) + 1, ve(kEvTargetType) - 1, "item", 4);
        if (train) {
          f |= kEvTraining;
          if (ve(kEvEntityId) - vb(kEvEntityId) == 2 || ve(kEvTargetId) - vb(kEvTargetId) == 2) code = kEvEmptyId;
        }
      }
      const long long nb = vb(kEvName) + 1, ne = ve(kEvName) - 1;
      if (json_str_is(body, etb, ete, "item", 4)) {
        const uint8_t kind = json_str_is(body, nb, ne, "$set", 4) ? kEvSet : json_str_is(body, nb, ne, "$unset", 6) ? kEvUnset
                             : json_str_is(body, nb, ne, "$delete", 7) ? kEvDelete : 0;
        if (kind) f |= kEvProperty | kind | (kind != kEvDelete && present(kEvProps) ? kEvPropObj : 0);
      }
    }
    if (code) atomicMin(err, ((unsigned long long)l << 8) | code);
    flag[l] = f;
    time[l] = tm;
  }
}

// out[i] = the inside of member k's string of line idx[i] (idx == nullptr: line i); absent or null -> empty
__global__ void k_event_strings(long long n, const uint32_t *__restrict__ idx, int k, const long long *__restrict__ sb,
                                const int2 *__restrict__ span, const unsigned char *__restrict__ body, JMember *__restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long l = idx ? (long long)idx[i] : i;
    const int2 v = span[l * kEvSlots + k];
    const bool s = v.x >= 0 && body[sb[l] + v.x] == '"';
    out[i] = s ? JMember{sb[l] + v.x + 1, sb[l] + v.y - 1, 0, 0} : JMember{0, 0, 0, 0};
  }
}

// key[l] = the line's event name code if it carries flag bit `want`, else `past` (sorted after them)
__global__ void k_event_keys(long long n_lines, const uint8_t *__restrict__ flag, uint8_t want, const int32_t *__restrict__ code,
                             uint32_t past, uint32_t *__restrict__ key, uint32_t *__restrict__ line) {
  for (long long l = blockIdx.x * (long long)blockDim.x + threadIdx.x; l < n_lines; l += (long long)gridDim.x * blockDim.x) {
    key[l] = (flag[l] & want) ? (uint32_t)code[l] : past;
    line[l] = (uint32_t)l;
  }
}
// cnt[2 g] += training events of name g, cnt[2 g + 1] += ranking events; cnt[2 n_names] += property events, cnt[2 n_names
// + 1] += ignored lines.  Lanes of a warp that add to the same counter add once (__match_any_sync).
__global__ void k_event_counts(long long n_lines, const uint8_t *__restrict__ flag, const int32_t *__restrict__ code, int32_t n_names,
                               unsigned long long *__restrict__ cnt) {
  const int lane = threadIdx.x & 31;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long base = blockIdx.x * (long long)blockDim.x; base < n_lines; base += stride) {
    const long long l = base + threadIdx.x;
    const uint8_t f = l < n_lines ? flag[l] : 0;
    const int g = l < n_lines ? code[l] : -1;
    for (int k = 0; k < 4; ++k) {
      int slot = -1;
      if (l < n_lines) {
        if (k == 0 && (f & kEvTraining)) slot = 2 * g;
        if (k == 1 && (f & kEvRanking)) slot = 2 * g + 1;
        if (k == 2 && (f & kEvProperty)) slot = 2 * n_names;
        if (k == 3 && !f) slot = 2 * n_names + 1;
      }
      const unsigned same = __match_any_sync(0xffffffffu, slot);
      if (slot >= 0 && lane == __ffs(same) - 1) atomicAdd(&cnt[slot], (unsigned long long)__popc(same));
    }
  }
}
__global__ void k_gather_i64(long long n, const uint32_t *__restrict__ idx, const long long *__restrict__ src, long long *__restrict__ dst) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) dst[i] = src[idx[i]];
}


// ---- property events: PEventStore.aggregateProperties on the device ----------------------------------------------------
// Property event i (line pl[i], line order) of item group pg[i] at position ord[i] of the (eventTime, line) order.
__global__ void k_prop_scatter_ord(long long n, const uint32_t *__restrict__ sorted, int32_t *__restrict__ ord) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) ord[sorted[k]] = (int32_t)k;
}
__global__ void k_prop_time_keys(long long n, const long long *__restrict__ t, unsigned long long *__restrict__ key, uint32_t *__restrict__ val) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    key[i] = (unsigned long long)t[i] ^ 0x8000000000000000ULL;
    val[i] = (uint32_t)i;
  }
}
// last_del[g] / last_set[g] = the latest position of a $delete / $set of group g (-1: none)
__global__ void k_prop_last(long long n, const uint8_t *__restrict__ kind, const int32_t *__restrict__ pg, const int32_t *__restrict__ ord,
                            int32_t *__restrict__ last_del, int32_t *__restrict__ last_set) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (kind[i] & kEvDelete) atomicMax(&last_del[pg[i]], ord[i]);
    if (kind[i] & kEvSet) atomicMax(&last_set[pg[i]], ord[i]);
  }
}
// the properties object of event qi[s] (an index into the property events) as a span of the body
__global__ void k_prop_spans(long long n, const uint32_t *__restrict__ qi, const uint32_t *__restrict__ pl, const long long *__restrict__ sb,
                             const int2 *__restrict__ span, long long *__restrict__ b, long long *__restrict__ e) {
  for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < n; s += (long long)gridDim.x * blockDim.x) {
    const long long l = pl[qi[s]];
    const int2 v = span[l * kEvSlots + kEvProps];
    b[s] = sb[l] + v.x;
    e[s] = sb[l] + v.y;
  }
}
// the property event of each member: mev[m] = qi[s] for m in [moff[s], moff[s + 1])
__global__ void k_prop_member_event(long long n, const long long *__restrict__ moff, const uint32_t *__restrict__ qi, uint32_t *__restrict__ mev) {
  for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < n; s += (long long)gridDim.x * blockDim.x)
    for (long long m = moff[s]; m < moff[s + 1]; ++m) mev[m] = qi[s];
}
// entries 0 .. M-1: members, keyed (group << 32 | field) and first ordered by the (eventTime, line) position of their event;
// entries M .. M+G-1: one presence entry per group, keyed (group << 32 | 0xffffffff), after its fields
__global__ void k_prop_keys1(long long M, const uint32_t *__restrict__ mev, const int32_t *__restrict__ ord, uint32_t *__restrict__ key,
                             uint32_t *__restrict__ val) {
  for (long long m = blockIdx.x * (long long)blockDim.x + threadIdx.x; m < M; m += (long long)gridDim.x * blockDim.x) {
    key[m] = (uint32_t)ord[mev[m]];
    val[m] = (uint32_t)m;
  }
}
__global__ void k_prop_keys2(long long M, long long G, const uint32_t *__restrict__ by_time, const uint32_t *__restrict__ mev,
                             const int32_t *__restrict__ pg, const int32_t *__restrict__ mf, unsigned long long *__restrict__ key,
                             uint32_t *__restrict__ val) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < M + G; k += (long long)gridDim.x * blockDim.x) {
    if (k < M) {
      const uint32_t m = by_time[k];
      key[k] = ((unsigned long long)(uint32_t)pg[mev[m]] << 32) | (uint32_t)mf[m];
      val[k] = m;
    } else {
      key[k] = ((unsigned long long)(k - M) << 32) | 0xffffffffULL;
      val[k] = (uint32_t)k;
    }
  }
}
// a member that ends its (group, field) run wins when its event is a $set after the group's last $delete; has[g] = 1
__global__ void k_prop_win(long long M, long long G, const unsigned long long *__restrict__ key, const uint32_t *__restrict__ val,
                           const uint32_t *__restrict__ mev, const uint8_t *__restrict__ kind, const int32_t *__restrict__ ord,
                           const int32_t *__restrict__ last_del, uint32_t *__restrict__ keep, uint32_t *__restrict__ has) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < M + G; k += (long long)gridDim.x * blockDim.x) {
    uint32_t w = 0;
    if ((uint32_t)key[k] != 0xffffffffu && key[k + 1] != key[k]) {   // entry M + G - 1 is a presence entry: k + 1 exists
      const uint32_t i = mev[val[k]];
      const int g = (int)(key[k] >> 32);
      if ((kind[i] & kEvSet) && ord[i] > last_del[g]) {
        w = 1;
        has[g] = 1;
      }
    }
    keep[k] = w;
  }
}
// a presence entry stays for an item whose final state exists (a $set after its last $delete) but holds no field
__global__ void k_prop_presence(long long M, long long G, const unsigned long long *__restrict__ key, const int32_t *__restrict__ last_del,
                                const int32_t *__restrict__ last_set, const uint32_t *__restrict__ has, uint32_t *__restrict__ keep) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < M + G; k += (long long)gridDim.x * blockDim.x) {
    if ((uint32_t)key[k] != 0xffffffffu) continue;
    const int g = (int)(key[k] >> 32);
    keep[k] = last_set[g] > last_del[g] && !has[g] ? 1u : 0u;
  }
}
// triple t (kept entry k at pos[k]): item = the item id of its event (presence: the group's first event), field, and the
// value text span (presence: none); first[f] = min triple index of field f (presence field: index n_fields)
__global__ void k_prop_triples(long long M, long long G, const uint32_t *__restrict__ keep, const uint32_t *__restrict__ pos,
                               const unsigned long long *__restrict__ key, const uint32_t *__restrict__ val, const uint32_t *__restrict__ mev,
                               const uint32_t *__restrict__ gfirst, const JMember *__restrict__ mem, int32_t n_fields,
                               uint32_t *__restrict__ titem, int32_t *__restrict__ tfield, long long *__restrict__ vb, long long *__restrict__ ve,
                               uint32_t *__restrict__ first) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < M + G; k += (long long)gridDim.x * blockDim.x) {
    if (!keep[k]) continue;
    const uint32_t t = pos[k];
    const bool presence = (uint32_t)key[k] == 0xffffffffu;
    const int f = presence ? n_fields : (int)(uint32_t)key[k];
    titem[t] = presence ? gfirst[key[k] >> 32] : mev[val[k]];
    tfield[t] = f;
    vb[t] = presence ? -1 : mem[val[k]].vb;
    ve[t] = presence ? -1 : mem[val[k]].ve;
    atomicMin(&first[f], t);
  }
}
// value text of each triple (presence: "null", never written) as a column: length pass, then copy pass
__global__ void k_prop_value_len(long long T, const long long *__restrict__ vb, const long long *__restrict__ ve, long long *__restrict__ len) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < T; t += (long long)gridDim.x * blockDim.x)
    len[t] = vb[t] < 0 ? 4 : ve[t] - vb[t];
}
__global__ void k_prop_value_copy(long long T, const long long *__restrict__ vb, const long long *__restrict__ off, const unsigned char *__restrict__ body,
                                  unsigned char *__restrict__ out) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < T; t += (long long)gridDim.x * blockDim.x) {
    const long long o = off[t], n = off[t + 1] - o;
    for (long long j = 0; j < n; ++j) out[o + j] = vb[t] < 0 ? (unsigned char)"null"[j] : body[vb[t] + j];
  }
}
__global__ void k_gather_u8(long long n, const uint32_t *__restrict__ idx, const uint8_t *__restrict__ src, uint8_t *__restrict__ dst) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) dst[i] = src[idx[i]];
}
// out[0] += entries with flag bit `want`; out[1] += groups whose final state exists (a $set after the last $delete)
__global__ void k_prop_counts(long long n, const uint8_t *__restrict__ flag, uint8_t want, long long G, const int32_t *__restrict__ last_del,
                              const int32_t *__restrict__ last_set, unsigned long long *__restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n || i < G; i += (long long)gridDim.x * blockDim.x) {
    if (i < n && (flag[i] & want)) atomicAdd(&out[0], 1ULL);
    if (i < G && last_set[i] > last_del[i]) atomicAdd(&out[1], 1ULL);
  }
}
__global__ void k_remap_i32(long long n, const int32_t *__restrict__ map, int32_t *__restrict__ x) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) x[i] = map[x[i]];
}

// ---- streamed reading ------------------------------------------------------------------------------------------------
// the property-event lines of a chunk, kept for the aggregation at finish: len[i] = bytes of line idx[i] + its '\n'
__global__ void k_line_len(long long n, const uint32_t *__restrict__ idx, const long long *__restrict__ sb, const long long *__restrict__ se,
                           long long *__restrict__ len) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    len[i] = se[idx[i]] - sb[idx[i]] + 1;
}
// one warp per listed line: its bytes to out + off[i], then a '\n' (the last line of a read may not have one)
__global__ void k_line_gather(long long n, const uint32_t *__restrict__ idx, const long long *__restrict__ sb, const long long *__restrict__ se,
                              const unsigned char *__restrict__ body, const long long *__restrict__ off, unsigned char *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long i = warp; i < n; i += nwarps) {
    const long long b = sb[idx[i]], m = se[idx[i]] - b;
    unsigned char *o = out + off[i];
    for (long long j = lane; j < m; j += 32) o[j] = body[b + j];
    if (lane == 0) o[m] = '\n';
  }
}

// One piece of a concatenation: the bytes [src_b, src_b + nb) of a segment's words go to [dst_b, dst_b + nb) of the
// output, and its entries [src_e, src_e + ne) of `e` to [dst_e, dst_e + ne), shifted by dst_b - src_b (offsets) or not
// (shift false: times).  Pieces are in output order.
struct CatPiece {
  const uint64_t *w;
  const long long *e;
  long long src_b, dst_b, nb, src_e, dst_e, ne;
  bool shift;
};
// the last piece whose start (`at` of the byte or the entry side) is <= x; pieces are sorted by it
template <bool kBytes>
__device__ __forceinline__ int cat_find(const CatPiece *__restrict__ pc, int np, long long x) {
  int lo = 0, hi = np - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if ((kBytes ? pc[mid].dst_b : pc[mid].dst_e) <= x) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}
// output word q of the concatenated bytes (pieces with nb > 0; words past `total` bytes are zero): a word inside one piece is
// a funnel shift of two source words (segments are not 8-byte aligned relative to each other), a word across pieces is
// assembled byte by byte
__global__ void k_cat_words(long long n_words, long long total, const CatPiece *__restrict__ pc, int np, uint64_t *__restrict__ out) {
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < n_words; q += (long long)gridDim.x * blockDim.x) {
    const long long pos = q * 8;
    if (pos >= total || np == 0) {
      out[q] = 0;
      continue;
    }
    int p = cat_find<true>(pc, np, pos);
    const CatPiece &a = pc[p];
    if (pos + 8 <= a.dst_b + a.nb) {
      const long long s = a.src_b + (pos - a.dst_b);
      const int sh = (int)(s & 7) * 8;
      const uint64_t lo = a.w[s >> 3];
      out[q] = sh ? (lo >> sh) | (a.w[(s >> 3) + 1] << (64 - sh)) : lo;
      continue;
    }
    uint64_t x = 0;
    for (int j = 0; j < 8; ++j) {
      const long long bp = pos + j;
      while (p < np && bp >= pc[p].dst_b + pc[p].nb) ++p;
      if (p == np || bp >= total) break;
      const unsigned char *src = (const unsigned char *)pc[p].w;
      x |= (uint64_t)src[pc[p].src_b + (bp - pc[p].dst_b)] << (8 * j);
    }
    out[q] = x;
  }
}
// output entry i of the concatenated offsets or times (pieces with ne > 0); last >= 0: out[n] = last
__global__ void k_cat_entries(long long n, long long last, const CatPiece *__restrict__ pc, int np, long long *__restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n + (last >= 0); i += (long long)gridDim.x * blockDim.x) {
    if (i == n) {
      out[n] = last;
      continue;
    }
    const CatPiece &a = pc[cat_find<false>(pc, np, i)];
    const long long v = a.e[a.src_e + (i - a.dst_e)];
    out[i] = a.shift ? v - a.src_b + a.dst_b : v;
  }
}

// ---- the DataSource's eventWindow (cco_event_log_begin_window) ------------------------------------------------------------
// PredictionIO's SelfCleaningDataSource.cleanPEvents, restated [RECALL, unverifiable here]: expiry (eventTime > cutoff, or
// the event is $set / $unset), then removeDuplicates (events equal but for eventId, eventTime and creationTime collapse to
// the one with the latest eventTime, ties to the later line).  Duplicates are found by a 128-bit identity hash per line
// (the bytes of earlier chunks are gone by finish):
//   k_win_expire                     an expired line loses its selection (flag kEvDropped) and is counted
//   EventSinkX                       EventSink plus the spans of "prId" and "tags", captured only when duplicates go
//   k_json_members + WinMemberSink   the top-level members of each retained line's properties, with the span's verdict
//   k_win_strings / k_win_raw_ranges the identity's decoded strings (json_decode) and raw value texts as byte ranges
//   k_win_hash                       128-bit hash of a byte range, one warp per range (no thread walks a long value)
//   k_win_props                      order-insensitive sum over the properties' members, the last of a repeated name only
//   k_win_ident                      the line's identity hash -> a WinRec (hash, time, global line, name, selection)
//   k_win_key_* / k_win_mark         at finish: records sorted by (hash, time desc, line desc), all but the first of each
//                                    run dropped into a bitmap over the global lines, the drops counted per selection
//   k_win_entry_keep / k_win_scatter the retained columns and the property lines compacted through the bitmap; with
//                                    k_win_flag_keep also every selection of lines by a flag bit in line order
enum : uint8_t { kEvDropped = 128 };   // an expired line: no selection, not ignored
enum : int { kEvPrId = 0, kEvTags, kEvXSlots };
constexpr int kWinStr = 6;             // decoded strings per line: event, entityType, entityId, targetEntityType, targetEntityId, prId

// what removeDuplicates keeps of a retained line
struct WinRec {
  uint64_t h0, h1;
  long long time, line;   // eventTime ms, global line
  int32_t code;           // event name
  uint32_t flag;          // selection flags
};

struct EventSinkX {
  int2 *span, *xspan;
  const unsigned char *body;
  __device__ void member(long long s, long long, long long b, const JMember &m) const {
    const int k = event_slot(body, m.nb, m.ne);
    if (k >= 0) {
      span[s * kEvSlots + k] = make_int2((int)(m.vb - b), (int)(m.ve - b));
      return;
    }
    const int x = json_str_is(body, m.nb, m.ne, "prId", 4) ? kEvPrId : json_str_is(body, m.nb, m.ne, "tags", 4) ? kEvTags : -1;
    if (x >= 0) xspan[s * kEvXSlots + x] = make_int2((int)(m.vb - b), (int)(m.ve - b));
  }
  __device__ void end(long long, long long) const {}
};

// lines at or before the cutoff whose event is neither $set nor $unset -> kEvDropped; *n_expired += them
__global__ void k_win_expire(long long n_lines, const long long *__restrict__ sb, const int2 *__restrict__ span,
                             const unsigned char *__restrict__ body, const long long *__restrict__ time, long long cutoff,
                             uint8_t *__restrict__ flag, unsigned long long *__restrict__ n_expired) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long base = blockIdx.x * (long long)blockDim.x; base < n_lines; base += stride) {
    const long long l = base + threadIdx.x;
    bool x = false;
    if (l < n_lines && time[l] <= cutoff) {
      const int2 v = span[l * kEvSlots + kEvName];
      const long long nb = sb[l] + v.x + 1, ne = sb[l] + v.y - 1;
      x = !json_str_is(body, nb, ne, "$set", 4) && !json_str_is(body, nb, ne, "$unset", 6);
      if (x) flag[l] = kEvDropped;
    }
    const unsigned m = __ballot_sync(0xffffffffu, x);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(n_expired, (unsigned long long)__popc(m));
  }
}
// keep[l] = line l is not expired
__global__ void k_win_keep_lines(long long n, const uint8_t *__restrict__ flag, uint32_t *__restrict__ keep) {
  for (long long l = blockIdx.x * (long long)blockDim.x + threadIdx.x; l < n; l += (long long)gridDim.x * blockDim.x)
    keep[l] = flag[l] != kEvDropped;
}
// out[pos[i]] = i for the kept i (pos = exclusive sum of keep)
__global__ void k_win_scatter(long long n, const uint32_t *__restrict__ keep, const uint32_t *__restrict__ pos, uint32_t *__restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    if (keep[i]) out[pos[i]] = (uint32_t)i;
}
// the properties object of retained line r (absent: an empty span, which the tokenizer calls not an object)
__global__ void k_win_prop_spans(long long R, const uint32_t *__restrict__ ridx, const long long *__restrict__ sb, const int2 *__restrict__ span,
                                 long long *__restrict__ b, long long *__restrict__ e) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < R; r += (long long)gridDim.x * blockDim.x) {
    const long long l = ridx[r];
    const int2 v = span[l * kEvSlots + kEvProps];
    b[r] = v.x >= 0 ? sb[l] + v.x : 0;
    e[r] = v.x >= 0 ? sb[l] + v.y : 0;
  }
}
// members of each span (count pass: count and verdict; write pass: the members of well-formed spans only)
template <bool kWrite>
struct WinMemberSink {
  long long *count;
  int *codes;
  const long long *moff;
  JMember *out;
  __device__ void member(long long s, long long n, long long, const JMember &m) const {
    if (kWrite && !codes[s]) out[moff[s] + n] = m;
  }
  __device__ void code(long long s, int c) const {
    if (!kWrite) codes[s] = c;
  }
  __device__ void end(long long s, long long n) const {
    if (!kWrite) count[s] = codes[s] ? 0 : n;
  }
};
// string i < 6 R: slot i % 6 of retained line i / 6, its inside when a string, its text when another value, empty when
// absent or null; string 6 R + m: the raw name of member m
__global__ void k_win_strings(long long R, const uint32_t *__restrict__ ridx, const long long *__restrict__ sb, const int2 *__restrict__ span,
                              const int2 *__restrict__ xspan, const unsigned char *__restrict__ body, long long M,
                              const JMember *__restrict__ mem, JMember *__restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < kWinStr * R + M; i += (long long)gridDim.x * blockDim.x) {
    if (i >= kWinStr * R) {
      const JMember &m = mem[i - kWinStr * R];
      out[i] = JMember{m.nb, m.ne, 0, 0};
      continue;
    }
    const long long l = ridx[i / kWinStr];
    const int k = (int)(i % kWinStr);
    const int2 v = k < kWinStr - 1 ? span[l * kEvSlots + k] : xspan[l * kEvXSlots + kEvPrId];
    const long long b = sb[l] + v.x, e = sb[l] + v.y;
    const bool present = v.x >= 0 && !json_is_null(body, b, e), str = present && body[b] == '"';
    out[i] = str ? JMember{b + 1, e - 1, 0, 0} : present ? JMember{b, e, 0, 0} : JMember{0, 0, 0, 0};
  }
}
// raw byte ranges: [0, R) the tags value, [R, 2 R) the properties text of a span the tokenizer could not split, [2 R, 2 R
// + M) the members' values (empty where unused)
__global__ void k_win_raw_ranges(long long R, const uint32_t *__restrict__ ridx, const long long *__restrict__ sb, const int2 *__restrict__ span,
                                 const int2 *__restrict__ xspan, const int *__restrict__ codes, long long M, const JMember *__restrict__ mem,
                                 long long *__restrict__ rb, long long *__restrict__ re) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < 2 * R + M; i += (long long)gridDim.x * blockDim.x) {
    long long b = 0, e = 0;
    if (i >= 2 * R) {
      b = mem[i - 2 * R].vb;
      e = mem[i - 2 * R].ve;
    } else {
      const long long r = i < R ? i : i - R, l = ridx[r];
      const int2 v = i < R ? xspan[l * kEvXSlots + kEvTags] : span[l * kEvSlots + kEvProps];
      if (v.x >= 0 && (i < R || codes[r])) {
        b = sb[l] + v.x;
        e = sb[l] + v.y;
      }
    }
    rb[i] = b;
    re[i] = e;
  }
}
// 128-bit hash of the bytes [rb[i], re[i]) of a word buffer (16 bytes of padding): the sum over its 8-byte words of a mix
// of (word, position), then the length -- one warp per range, each lane over every 32nd word
__device__ __forceinline__ ulonglong2 win_word(uint64_t x, uint64_t q) {
  return make_ulonglong2(mix64(x ^ mix64(q + 0x243f6a8885a308d3ULL)), mix64(mix64(x + q * 0x9e3779b97f4a7c15ULL) ^ 0x13198a2e03707344ULL));
}
__global__ void k_win_hash(long long n, const long long *__restrict__ rb, const long long *__restrict__ re, const uint64_t *__restrict__ w,
                           ulonglong2 *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long i = warp; i < n; i += nwarps) {
    const long long b = rb[i], len = re[i] - b;
    uint64_t a = 0, c = 0;
    for (long long k = lane; k * 8 < len; k += 32) {
      const ulonglong2 h = win_word(str_mask_tail(str_word(w, b, k), len - k * 8), (uint64_t)k);
      a += h.x;
      c += h.y;
    }
    for (int o = 16; o > 0; o >>= 1) {
      a += __shfl_xor_sync(0xffffffffu, a, o);
      c += __shfl_xor_sync(0xffffffffu, c, o);
    }
    if (lane == 0) out[i] = make_ulonglong2(mix64(a ^ mix64((uint64_t)len ^ 0xa4093822299f31d0ULL)), mix64(c + (uint64_t)len * 0x082efa98ec4e6c89ULL));
  }
}
// mline[m] = the retained line of member m
__global__ void k_win_member_line(long long R, const long long *__restrict__ moff, uint32_t *__restrict__ mline) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < R; r += (long long)gridDim.x * blockDim.x)
    for (long long m = moff[r]; m < moff[r + 1]; ++m) mline[m] = (uint32_t)r;
}
__global__ void k_win_name_keys(long long M, const ulonglong2 *__restrict__ hname, unsigned long long *__restrict__ key, uint32_t *__restrict__ val) {
  for (long long m = blockIdx.x * (long long)blockDim.x + threadIdx.x; m < M; m += (long long)gridDim.x * blockDim.x) {
    key[m] = hname[m].x;
    val[m] = (uint32_t)m;
  }
}
__global__ void k_win_line_keys(long long M, const uint32_t *__restrict__ val, const uint32_t *__restrict__ mline, uint32_t *__restrict__ key) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < M; k += (long long)gridDim.x * blockDim.x) key[k] = mline[val[k]];
}
// members sorted by (line, name hash, member order): the last of each (line, name) run adds a mix of (name, value) to
// its line's sum
__global__ void k_win_props(long long M, const uint32_t *__restrict__ val, const uint32_t *__restrict__ mline, const ulonglong2 *__restrict__ hname,
                            const ulonglong2 *__restrict__ hval, unsigned long long *__restrict__ acc) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < M; k += (long long)gridDim.x * blockDim.x) {
    const uint32_t m = val[k], r = mline[m];
    const ulonglong2 n = hname[m];
    if (k + 1 < M) {
      const uint32_t q = val[k + 1];
      if (mline[q] == r && hname[q].x == n.x && hname[q].y == n.y) continue;
    }
    const ulonglong2 v = hval[m];
    atomicAdd(&acc[2 * r], mix64(n.x ^ mix64(v.x + 0x452821e638d01377ULL)));
    atomicAdd(&acc[2 * r + 1], mix64(n.y + mix64(v.y ^ 0xbe5466cf34e90c6cULL)));
  }
}
// the identity hash of retained line r -> rec[r]
__global__ void k_win_ident(long long R, const uint32_t *__restrict__ ridx, long long line_base, const long long *__restrict__ sb,
                            const int2 *__restrict__ span, const int2 *__restrict__ xspan, const unsigned char *__restrict__ body,
                            const ulonglong2 *__restrict__ hdec, const ulonglong2 *__restrict__ hraw, const int *__restrict__ codes,
                            const unsigned long long *__restrict__ acc, const long long *__restrict__ tm, const uint8_t *__restrict__ flag,
                            const int32_t *__restrict__ code, WinRec *__restrict__ rec) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < R; r += (long long)gridDim.x * blockDim.x) {
    const long long l = ridx[r], b = sb[l];
    uint64_t a = 0x3707344a40938222ULL, c = 0x299f31d0082efa98ULL;
    auto add = [&](uint64_t x, uint64_t y) {
      a = mix64(a ^ x) + 0x9e3779b97f4a7c15ULL;
      c = mix64(c + y) ^ 0xc0ac29b7c97c50ddULL;
    };
    unsigned kinds = 0;   // per string slot: present, a string
    for (int k = 0; k < kWinStr; ++k) {
      const int2 v = k < kWinStr - 1 ? span[l * kEvSlots + k] : xspan[l * kEvXSlots + kEvPrId];
      const bool present = v.x >= 0 && !json_is_null(body, b + v.x, b + v.y);
      kinds |= (present ? 1u : 0u) << (2 * k);
      kinds |= (present && body[b + v.x] == '"' ? 2u : 0u) << (2 * k);
      add(hdec[kWinStr * r + k].x, hdec[kWinStr * r + k].y);
    }
    add(kinds, kinds);
    // tags: absent, null and [] are the empty list
    const int2 t = xspan[l * kEvXSlots + kEvTags];
    const bool no_tags = t.x < 0 || json_is_null(body, b + t.x, b + t.y) || (t.y - t.x == 2 && body[b + t.x] == '[' && body[b + t.x + 1] == ']');
    if (no_tags) add(1, 1);
    else add(hraw[r].x, hraw[r].y);
    // properties: absent is {}; the text of an object the tokenizer could not split stands for it
    const bool props = span[l * kEvSlots + kEvProps].x >= 0;
    if (props && codes[r]) add(hraw[R + r].x ^ 2, hraw[R + r].y ^ 2);
    else add(acc[2 * r], acc[2 * r + 1]);
    rec[r] = WinRec{mix64(a), mix64(c ^ a), tm[l], line_base + l, code[l], flag[l]};
  }
}
// at finish: keys of the (hash, time desc, line desc) order, sorted least significant first (records are in line order)
__global__ void k_win_key_time(long long N, const WinRec *__restrict__ rec, unsigned long long *__restrict__ key, uint32_t *__restrict__ val) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < N; i += (long long)gridDim.x * blockDim.x) {
    const long long j = N - 1 - i;
    key[i] = ~((unsigned long long)rec[j].time ^ 0x8000000000000000ULL);
    val[i] = (uint32_t)j;
  }
}
__global__ void k_win_key_hash(long long N, const WinRec *__restrict__ rec, const uint32_t *__restrict__ val, int high,
                               unsigned long long *__restrict__ key) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < N; k += (long long)gridDim.x * blockDim.x)
    key[k] = high ? rec[val[k]].h1 : rec[val[k]].h0;
}
// a record whose hash equals its predecessor's is a duplicate: its line goes into the bitmap, and cnt[2 g] / cnt[2 g + 1]
// (training / ranking events of name g), cnt[2 n_names] (property events), cnt[2 n_names + 1] (ignored lines) and
// cnt[2 n_names + 2] (all) count it
__global__ void k_win_mark(long long N, const WinRec *__restrict__ rec, const uint32_t *__restrict__ val, int32_t n_names,
                           uint32_t *__restrict__ bitmap, unsigned long long *__restrict__ cnt) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < N; k += (long long)gridDim.x * blockDim.x) {
    if (k == 0) continue;
    const WinRec &x = rec[val[k]], &p = rec[val[k - 1]];
    if (x.h0 != p.h0 || x.h1 != p.h1) continue;
    atomicOr(&bitmap[x.line >> 5], 1u << (x.line & 31));
    if (x.flag & kEvTraining) atomicAdd(&cnt[2 * x.code], 1ULL);
    if (x.flag & kEvRanking) atomicAdd(&cnt[2 * x.code + 1], 1ULL);
    if (x.flag & kEvProperty) atomicAdd(&cnt[2 * n_names], 1ULL);
    if (!x.flag) atomicAdd(&cnt[2 * n_names + 1], 1ULL);
    atomicAdd(&cnt[2 * n_names + 2], 1ULL);
  }
}
__device__ __forceinline__ bool win_dropped(const uint32_t *__restrict__ bitmap, long long line) {
  return (bitmap[line >> 5] >> (line & 31)) & 1;
}
// out[i] = base + idx[i]: the global line of each entry of a chunk's column
__global__ void k_win_lines(long long n, const uint32_t *__restrict__ idx, long long base, long long *__restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) out[i] = base + idx[i];
}
__global__ void k_win_entry_keep(long long n, const long long *__restrict__ line, const uint32_t *__restrict__ bitmap, uint32_t *__restrict__ keep) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    keep[i] = win_dropped(bitmap, line[i]) ? 0u : 1u;
}
// out[g] = pos[at[g]]: the kept entries before each name's first
__global__ void k_win_at(long long n, const long long *__restrict__ at, const uint32_t *__restrict__ pos, long long *__restrict__ out) {
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < n; g += (long long)gridDim.x * blockDim.x) out[g] = pos[at[g]];
}
// the property lines gathered at finish: a dropped one loses its selection
__global__ void k_win_drop_lines(long long n, const long long *__restrict__ gline, const uint32_t *__restrict__ bitmap, uint8_t *__restrict__ flag) {
  for (long long l = blockIdx.x * (long long)blockDim.x + threadIdx.x; l < n; l += (long long)gridDim.x * blockDim.x)
    if (win_dropped(bitmap, gline[l])) flag[l] = 0;
}
// the properties objects of the listed lines
__global__ void k_win_obj_spans(long long n, const uint32_t *__restrict__ idx, const long long *__restrict__ sb, const int2 *__restrict__ span,
                                long long *__restrict__ b, long long *__restrict__ e) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long l = idx[i];
    b[i] = sb[l] + span[l * kEvSlots + kEvProps].x;
    e[i] = sb[l] + span[l * kEvSlots + kEvProps].y;
  }
}
__global__ void k_win_flag_keep(long long n, const uint8_t *__restrict__ flag, uint8_t want, uint32_t *__restrict__ keep) {
  for (long long l = blockIdx.x * (long long)blockDim.x + threadIdx.x; l < n; l += (long long)gridDim.x * blockDim.x)
    keep[l] = (flag[l] & want) ? 1u : 0u;
}

// ---- extendable logs (CCO_LOG_EXTENDABLE, cco_event_log_extend) ------------------------------------------------------------
// A finished extendable log keeps one WinRec per retained line (without removeDuplicates its hash is 0), the global line of
// every training and ranking entry and the retained property-event lines.  At each finish:
//   k_ext_line_recs      per chunk, without removeDuplicates: the WinRec of every retained line (time, line, name, selection)
//   k_ext_expire         the records at or before the cutoff whose name is not exempt ($set / $unset) expire: their lines go
//                        into the drop bitmap, counted per selection; the rest are kept
//   k_ext_gather_rec     the kept records, in line order
//   k_ext_expire_times   the eventTimes of earlier duplicate drops (exempt names excluded) at or before the cutoff: a whole
//                        read under this cutoff calls those lines expired
//   k_ext_dup_split      after k_win_mark: the records whose line it dropped leave, and the times of the non-exempt ones stay
//                        for k_ext_expire_times
__global__ void k_ext_line_recs(long long R, const uint32_t *__restrict__ ridx, long long line_base, const long long *__restrict__ tm,
                                const uint8_t *__restrict__ flag, const int32_t *__restrict__ code, WinRec *__restrict__ rec) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < R; r += (long long)gridDim.x * blockDim.x) {
    const long long l = ridx[r];
    rec[r] = WinRec{0, 0, tm[l], line_base + l, code[l], flag[l]};
  }
}
// cnt[0] += expired records, cnt[1] += of them property events, cnt[2] += ignored lines
__global__ void k_ext_expire(long long N, const WinRec *__restrict__ rec, long long cutoff, const uint8_t *__restrict__ exempt,
                             uint32_t *__restrict__ bitmap, uint32_t *__restrict__ keep, unsigned long long *__restrict__ cnt) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long base = blockIdx.x * (long long)blockDim.x; base < N; base += stride) {
    const long long i = base + threadIdx.x;
    bool x = false;
    if (i < N) {
      const WinRec &r = rec[i];
      x = r.time <= cutoff && !exempt[r.code];
      keep[i] = x ? 0u : 1u;
      if (x) {
        atomicOr(&bitmap[r.line >> 5], 1u << (r.line & 31));
        if (r.flag & kEvProperty) atomicAdd(&cnt[1], 1ULL);
        if (!r.flag) atomicAdd(&cnt[2], 1ULL);
      }
    }
    const unsigned m = __ballot_sync(0xffffffffu, x);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(&cnt[0], (unsigned long long)__popc(m));
  }
}
__global__ void k_ext_gather_rec(long long n, const uint32_t *__restrict__ idx, const WinRec *__restrict__ src, WinRec *__restrict__ dst) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) dst[i] = src[idx[i]];
}
// keep[i] = time[i] > cutoff; *n_out += the others
__global__ void k_ext_expire_times(long long n, const long long *__restrict__ time, long long cutoff, uint32_t *__restrict__ keep,
                                   unsigned long long *__restrict__ n_out) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long base = blockIdx.x * (long long)blockDim.x; base < n; base += stride) {
    const long long i = base + threadIdx.x;
    const bool x = i < n && time[i] <= cutoff;
    if (i < n) keep[i] = x ? 0u : 1u;
    const unsigned m = __ballot_sync(0xffffffffu, x);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(n_out, (unsigned long long)__popc(m));
  }
}
// keep[i] = record i's line survived k_win_mark; dup[i] = it did not and its name is not exempt; time[i] its eventTime
__global__ void k_ext_dup_split(long long N, const WinRec *__restrict__ rec, const uint32_t *__restrict__ bitmap, const uint8_t *__restrict__ exempt,
                                uint32_t *__restrict__ keep, uint32_t *__restrict__ dup, long long *__restrict__ time) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < N; i += (long long)gridDim.x * blockDim.x) {
    const WinRec &r = rec[i];
    const bool d = win_dropped(bitmap, r.line);
    keep[i] = d ? 0u : 1u;
    dup[i] = d && !exempt[r.code] ? 1u : 0u;
    time[i] = r.time;
  }
}

}  // namespace cco
