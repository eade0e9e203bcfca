// cco_queries.cuh -- buildQuery (URAlgorithm.scala:563-839) on the device.  Every query builder renders its records as rows
// of a mixed batch (k_mq_record): cco_event_log_user_queries, cco_item_queries and cco_item_set_queries as rows with one
// member, cco_mixed_queries and cco_query_file_queries as rows with any.  The stages that feed it are listed with them: the
// training history an event log keeps (cco_event_log_begin_ex with CCO_LOG_KEEP_HISTORY), the similar items of a model
// index body, the set elements, then the mixed rows and the query file's lines.
//
// e = one training event of a query event name (name rank q); its user and item are dense group ids of the log's columns.
//   k_uq_select       e -> (log entry, name rank) over the query names' ranges of the name-partitioned columns
//   k_uq_gather       per e: user group, item group, time and global line of its log entry
//   k_uq_key_line / k_uq_key_time / k_uq_key_seg / k_uq_key_user   radix keys: line desc, time desc, (user, q), user
//   k_uq_count        segment sizes (histogram) -> scan -> segment starts
//   k_uq_hist_keys    the first `limit` of every (user, q) segment: (segment, item) keys, fed oldest first, so that the
//                     first of each run after the stable sort is the item's oldest position (distinct after the prepend)
//   k_uq_first        first of each run of equal keys -> keep flag
//   k_uq_min_line     each user's first line (the row order when every user is asked for)
//   k_uq_user_keys    (first line, user) pairs for that order's sort
//   k_uq_user_entry   the log entry that names each row's user, for the users' dictionary
#pragma once

namespace cco {

constexpr int kUqMaxNames = 64;

__global__ void k_uq_select(long long E, int nq, const long long *__restrict__ qoff, const long long *__restrict__ qbase,
                            uint32_t *__restrict__ ent, uint8_t *__restrict__ qr) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < E; e += (long long)gridDim.x * blockDim.x) {
    int lo = 0, hi = nq - 1;   // the last q with qoff[q] <= e
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (qoff[mid] <= e) lo = mid; else hi = mid - 1;
    }
    ent[e] = (uint32_t)(qbase[lo] + (e - qoff[lo]));
    qr[e] = (uint8_t)lo;
  }
}

__global__ void k_uq_gather(long long E, const uint32_t *__restrict__ ent, const int32_t *__restrict__ ugid, const int32_t *__restrict__ igid,
                            const long long *__restrict__ ttime, const long long *__restrict__ tline, int32_t *__restrict__ uid,
                            int32_t *__restrict__ iid, long long *__restrict__ tm, long long *__restrict__ ln) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < E; e += (long long)gridDim.x * blockDim.x) {
    const uint32_t x = ent[e];
    uid[e] = ugid[x];
    iid[e] = igid[x];
    tm[e] = ttime[x];
    ln[e] = tline[x];
  }
}

// keys of the first sort (line descending) over e = 0 .. E-1
__global__ void k_uq_key_line(long long E, long long n_lines, const long long *__restrict__ ln, unsigned long long *__restrict__ key,
                              uint32_t *__restrict__ val) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < E; e += (long long)gridDim.x * blockDim.x) {
    key[e] = (unsigned long long)(n_lines - 1 - ln[e]);
    val[e] = (uint32_t)e;
  }
}
// time descending, over the current order
__global__ void k_uq_key_time(long long E, const uint32_t *__restrict__ val, const long long *__restrict__ tm, unsigned long long *__restrict__ key) {
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < E; p += (long long)gridDim.x * blockDim.x)
    key[p] = ~((unsigned long long)tm[val[p]] ^ 0x8000000000000000ULL);
}
// (user, q) segment, over the current order
__global__ void k_uq_key_seg(long long E, int nq, const uint32_t *__restrict__ val, const int32_t *__restrict__ uid,
                             const uint8_t *__restrict__ qr, unsigned long long *__restrict__ key) {
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < E; p += (long long)gridDim.x * blockDim.x) {
    const uint32_t e = val[p];
    key[p] = (unsigned long long)uid[e] * (unsigned long long)nq + qr[e];
  }
}
// the blacklisted events (their name rank is flagged) in the current order -> keep flags
__global__ void k_uq_flag_black(long long E, const uint32_t *__restrict__ val, const uint8_t *__restrict__ qr, const uint8_t *__restrict__ black,
                                uint32_t *__restrict__ keep) {
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < E; p += (long long)gridDim.x * blockDim.x)
    keep[p] = black[qr[val[p]]] ? 1u : 0u;
}
// the selected positions' events with their user as key
__global__ void k_uq_key_user(long long B, const uint32_t *__restrict__ idx, const uint32_t *__restrict__ order, const int32_t *__restrict__ uid,
                              unsigned long long *__restrict__ key, uint32_t *__restrict__ val) {
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < B; p += (long long)gridDim.x * blockDim.x) {
    const uint32_t e = order[idx[p]];
    val[p] = e;
    key[p] = (unsigned long long)(uint32_t)uid[e];
  }
}
__global__ void k_uq_count(long long n, const unsigned long long *__restrict__ key, long long *__restrict__ cnt) {
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < n; p += (long long)gridDim.x * blockDim.x)
    atomicAdd((unsigned long long *)&cnt[key[p]], 1ULL);
}
// history: position p of the (user, q)-sorted order is taken iff it is among the first limit[q] of its segment; the taken
// ones get the key (segment << 32 | item), written at E - 1 - p so that the stable sort puts the oldest position first
__global__ void k_uq_hist_keys(long long E, int nq, const unsigned long long *__restrict__ seg, const long long *__restrict__ start,
                               const int32_t *__restrict__ limit, const uint32_t *__restrict__ val, const int32_t *__restrict__ iid,
                               unsigned long long *__restrict__ key, uint32_t *__restrict__ pos) {
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < E; p += (long long)gridDim.x * blockDim.x) {
    const unsigned long long s = seg[p];
    const bool taken = p - start[s] < (long long)limit[s % (unsigned long long)nq];
    key[E - 1 - p] = taken ? (s << 32) | (uint32_t)iid[val[p]] : ~0ULL;
    pos[E - 1 - p] = (uint32_t)p;
  }
}
// blacklist: (user << 32 | item) of the user-sorted blacklisted events, position as value
__global__ void k_uq_black_keys(long long B, const uint32_t *__restrict__ val, const int32_t *__restrict__ uid, const int32_t *__restrict__ iid,
                                unsigned long long *__restrict__ key, uint32_t *__restrict__ pos) {
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < B; p += (long long)gridDim.x * blockDim.x) {
    const uint32_t e = val[p];
    key[p] = ((unsigned long long)(uint32_t)uid[e] << 32) | (uint32_t)iid[e];
    pos[p] = (uint32_t)p;
  }
}
__global__ void k_uq_first(long long n, const unsigned long long *__restrict__ key, const uint32_t *__restrict__ pos, uint8_t *__restrict__ keep) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    if (key[i] != ~0ULL && (i == 0 || key[i - 1] != key[i])) keep[pos[i]] = 1;
}
__global__ void k_uq_min_line(long long E, const int32_t *__restrict__ uid, const long long *__restrict__ ln, unsigned long long *__restrict__ mn) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < E; e += (long long)gridDim.x * blockDim.x)
    atomicMin(&mn[uid[e]], (unsigned long long)ln[e]);
}
__global__ void k_uq_user_keys(long long G, const unsigned long long *__restrict__ mn, unsigned long long *__restrict__ key, int32_t *__restrict__ val) {
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < G; g += (long long)gridDim.x * blockDim.x) {
    key[g] = mn[g];
    val[g] = (int32_t)g;
  }
}
// the log entry that names each record's user (its group's first entry), for the users' dictionary
__global__ void k_uq_user_entry(long long R, const int32_t *__restrict__ rec_uid, const uint32_t *__restrict__ first_sorted, uint32_t *__restrict__ e) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < R; r += (long long)gridDim.x * blockDim.x)
    e[r] = first_sorted[rec_uid[r]];
}

// json4s 3.2 quote: '"' and '\' get a backslash, \b \f \n \r \t their short forms, every other code point below U+0020, in
// U+0080..U+009F (UTF-8 C2 80..C2 9F) and in U+2000..U+20FF (E2 80 80..E2 83 BF) becomes \u%04x in lowercase hex; the rest
// passes through.  o == nullptr: the length only.
__host__ __device__ __forceinline__ long long uq_escape(const unsigned char *__restrict__ s, long long n, unsigned char *o) {
  long long k = 0;
  for (long long i = 0; i < n; ++i) {
    const unsigned char b = s[i];
    unsigned cp = 0xffffffffu;
    unsigned char sh = 0;
    if (b == '"' || b == '\\') sh = b;
    else if (b == '\b') sh = 'b';
    else if (b == '\f') sh = 'f';
    else if (b == '\n') sh = 'n';
    else if (b == '\r') sh = 'r';
    else if (b == '\t') sh = 't';
    else if (b < 0x20) cp = b;
    else if (b == 0xC2 && i + 1 < n && s[i + 1] >= 0x80 && s[i + 1] <= 0x9F) {
      cp = s[i + 1];
      i += 1;
    } else if (b == 0xE2 && i + 2 < n && s[i + 1] >= 0x80 && s[i + 1] <= 0x83 && (s[i + 2] & 0xC0) == 0x80) {
      cp = 0x2000u | ((unsigned)(s[i + 1] & 0x3F) << 6) | (s[i + 2] & 0x3F);
      i += 2;
    }
    if (sh) {
      if (o) {
        o[k] = '\\';
        o[k + 1] = sh;
      }
      k += 2;
    } else if (cp != 0xffffffffu) {
      if (o) {
        o[k] = '\\';
        o[k + 1] = 'u';
        for (int d = 0; d < 4; ++d) o[k + 2 + d] = "0123456789abcdef"[(cp >> (12 - 4 * d)) & 15];
      }
      k += 6;
    } else {
      if (o) o[k] = b;
      k += 1;
    }
  }
  return k;
}

// the users' history lists
struct UqArgs {
  int nq;                          // query names
  const int32_t *limit;            // [nq]
  const long long *hstart;         // [G * nq + 1] segment starts in the (user, q) order
  const uint32_t *hord;            // [E] events in (user, q, time desc, line desc) order
  const uint8_t *keep_h;           // [E] by position: taken and the item's oldest taken position
  const uint32_t *ent;             // [E] log entry of each event
  const long long *ioff;           // the log's training item column
  const unsigned char *ibytes;
};

// the blacklisted items of the users under one set of blacklisted query names (uq_blacklist)
struct MqBlack {
  const long long *bstart;         // [G + 1]
  const unsigned long long *bkey;  // [B] (user << 32 | item), sorted
  const uint32_t *bord;            // [B] blacklisted events in (user, time desc, line desc) order
  const uint8_t *keep_b;           // [B] by position: the item's newest position
};

// whether user u's blacklisted items hold item group g
__device__ __forceinline__ bool uq_has(const MqBlack &a, int32_t u, int32_t g) {
  const unsigned long long x = ((unsigned long long)(uint32_t)u << 32) | (uint32_t)g;
  long long lo = a.bstart[u], hi = a.bstart[u + 1];
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (a.bkey[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo < a.bstart[u + 1] && a.bkey[lo] == x;
}

// One record, written by one warp at o (the write pass) or only measured (o == nullptr): cur is the warp-uniform byte count
// so far.
template <bool WRITE>
struct RecordOut {
  unsigned char *o;
  long long cur;
  int lane;
  // template piece j of the kernel's arguments (a.toff / a.tbytes, rendered on the host); whether it is not empty
  template <class Args>
  __device__ __forceinline__ bool piece(const Args &a, int j) {
    const long long t0 = a.toff[j], tl = a.toff[j + 1] - t0;
    if (WRITE)
      for (long long k = lane; k < tl; k += 32) o[cur + k] = a.tbytes[t0 + k];
    cur += tl;
    return tl > 0;
  }
  __device__ __forceinline__ void comma() {
    if (WRITE && lane == 0) o[cur] = ',';
    cur += 1;
  }
  // one list of quoted, comma-separated ids from n candidates; get(i, &ptr, &len) == false skips candidate i.  first is
  // warp-uniform.  The write tests o, not WRITE: testing WRITE here has made ptxas spill in a record kernel's write pass.
  template <class Get>
  __device__ __forceinline__ void list(long long n, const Get &get, bool &first) {
    for (long long b = 0; b < n; b += 32) {
      const long long i = b + lane;
      const unsigned char *p = nullptr;
      long long len = 0;
      const bool keep = i < n && get(i, &p, &len);
      const unsigned ball = __ballot_sync(0xffffffffu, keep);
      if (!ball) continue;
      const bool lead = first && lane == __ffs(ball) - 1;
      const long long el = keep ? uq_escape(p, len, nullptr) + 2 + (lead ? 0 : 1) : 0;
      long long x = el;
      for (int d = 1; d < 32; d <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d) x += y;
      }
      if (o && keep) {
        unsigned char *q = o + cur + x - el;
        if (!lead) *q++ = ',';
        *q++ = '"';
        q += uq_escape(p, len, q);
        *q = '"';
      }
      cur += __shfl_sync(0xffffffffu, x, 31);
      first = false;
    }
  }
};

// ---- the similar items of a model index body (parsed by cco_json.cuh) -------------------------------------------------
//   k_iq_pick      per document: the last source member of each model name (T distinct names), -1
//   k_iq_array     one warp per (queried document, name) value span: the array-of-strings grammar and the raw element spans,
//                  a count pass and a write pass; an error word for the first bad span
__global__ void k_iq_pick(long long n_docs, int T, const long long *__restrict__ line_moff, const int32_t *__restrict__ ngid,
                          const int32_t *__restrict__ entry_of, int32_t *__restrict__ pick) {
  for (long long d = blockIdx.x * (long long)blockDim.x + threadIdx.x; d < n_docs; d += (long long)gridDim.x * blockDim.x) {
    int32_t *p = pick + d * T;
    for (int t = 0; t < T; ++t) p[t] = -1;
    for (long long m = line_moff[2 * d + 1]; m < line_moff[2 * d + 2]; ++m) {
      const int32_t t = entry_of[ngid[m]];
      if (t >= 0) p[t] = (int32_t)m;
    }
  }
}
// Grammar of a picked value: '[' ws* ( ']' | string (ws* ',' ws* string)* ws* ']' ) -- the span is trimmed, its strings were
// validated by k_json_members.  The string and escape masks are k_json_members': escaped byte = an odd run of backslashes
// right before it, in string = prefix XOR of the unescaped quotes.  Events are the unescaped quotes and the non-whitespace
// bytes outside strings.  x = d * T + t; a span that is not queried or not picked counts 0 elements.
enum : int { kIaOpen = 0, kIaFirst, kIaString, kIaAfter, kIaNext, kIaDone };
template <bool kWrite>
__global__ void __launch_bounds__(256) k_iq_array(long long n, int T, const uint8_t *__restrict__ queried, const int32_t *__restrict__ pick,
                                                  const JMember *__restrict__ mem, const unsigned char *__restrict__ body,
                                                  long long *__restrict__ cnt, const long long *__restrict__ eoff, JMember *__restrict__ elem,
                                                  unsigned long long *__restrict__ err) {
  const int lane = threadIdx.x & 31;
  const unsigned below = (1u << lane) - 1, upto = 0xffffffffu >> (31 - lane);
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long x = warp; x < n; x += nwarps) {
    const int32_t m = queried[x / T] ? pick[x] : -1;
    if (m < 0) {
      if (!kWrite && lane == 0) cnt[x] = 0;
      continue;
    }
    const long long b = mem[m].vb, e = mem[m].ve;
    const long long at = kWrite ? eoff[x] : 0;
    int state = kIaOpen;
    long long k = 0, sb = 0;
    unsigned in_str = 0, bs_odd = 0;
    for (long long base = b; base < e && state >= 0; base += 32) {
      const long long p = base + lane;
      const unsigned c = p < e ? body[p] : ' ';
      const unsigned bsm = __ballot_sync(0xffffffffu, c == '\\');
      const unsigned nb = ~bsm & below;
      const unsigned esc = (nb ? lane - 1 - (31 - __clz(nb)) : lane + bs_odd) & 1;
      const unsigned qm = __ballot_sync(0xffffffffu, c == '"' && !esc);
      const bool uq = (qm >> lane) & 1;
      const bool S = (in_str ^ __popc(qm & upto)) & 1;
      const unsigned Sm = __ballot_sync(0xffffffffu, S);
      unsigned evm = __ballot_sync(0xffffffffu, uq || (p < e && !S && !json_ws(c)));
      while (evm && state >= 0) {
        const int i = __ffs(evm) - 1;
        evm &= evm - 1;
        const unsigned ci = __shfl_sync(0xffffffffu, c, i);
        const bool qi = (qm >> i) & 1, open_q = qi && ((Sm >> i) & 1);
        const long long pi = base + i;
        if (state == kIaOpen) {
          state = ci == '[' ? kIaFirst : -1;
        } else if (state == kIaFirst || state == kIaNext) {
          if (open_q) {
            sb = pi + 1;
            state = kIaString;
          } else {
            state = state == kIaFirst && ci == ']' ? kIaDone : -1;
          }
        } else if (state == kIaString) {   // the only event inside a string is its closing quote
          if (kWrite && lane == 0) elem[at + k] = JMember{sb, pi, 0, 0};
          ++k;
          state = kIaAfter;
        } else if (state == kIaAfter) {
          state = qi ? -1 : ci == ',' ? kIaNext : ci == ']' ? kIaDone : -1;
        } else {
          state = -1;   // anything after the closing bracket
        }
      }
      in_str = (in_str ^ __popc(qm)) & 1;
      if (~bsm) bs_odd = __clz(~bsm) & 1;
    }
    if (lane == 0) {
      if (state != kIaDone) atomicMin(err, (unsigned long long)x);
      if (!kWrite) cnt[x] = state == kIaDone ? k : 0;
    }
  }
}

// ---- the sets' elements and the blacklistItems lists ------------------------------------------------------------------
// "First occurrence within its set (list)" is the first of each run of (set << 32 | group) keys after one stable sort
// (k_uq_first).
//   k_is_keys      per element: the key (set << 32 | group), its position as value (the set by a search of the set offsets)
__global__ void k_is_keys(long long NE, long long n_sets, const long long *__restrict__ soff, const int32_t *__restrict__ egid,
                          unsigned long long *__restrict__ key, uint32_t *__restrict__ pos) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < NE; e += (long long)gridDim.x * blockDim.x) {
    long long lo = 0, hi = n_sets - 1;   // the last s with soff[s] <= e (the set holding e: soff[s] <= e < soff[s + 1])
    while (lo < hi) {
      const long long mid = (lo + hi + 1) >> 1;
      if (soff[mid] <= e) lo = mid; else hi = mid - 1;
    }
    key[e] = ((unsigned long long)lo << 32) | (uint32_t)egid[e];
    pos[e] = (uint32_t)e;
  }
}

// ---- the records: buildQuery for rows with any subset of {user, item, item set} ------------------------------------------
// The history comes from the history stage (UqHistory), the similar items from the documents' stage (IqDocs).
// One key column holds the decoded _ids, the items, blacklistItems and the set elements, grouped exactly; the items,
// blacklistItems and elements are also probed into the log's item table, so that every test of the exclusion list
// distinct(userBlacklisted ++ blacklistItems :+ item ++ itemSet) is a group test: the user's blacklist by uq_has,
// blacklistItems by first_in_list, the item by group equality, earlier in the set by first_in_set.
//   k_mq_rows      per row: which members it has (LSB-first validity bitmaps, nullptr: every row); its document; the queried
//                  documents flagged
//   k_mq_record    one warp per row: template pieces, history lists, similar-items lists, the set clause and the exclusion
//                  list; a length pass and a write pass (k_doc_len -> scan -> k_doc_write, as cco_format_model).  Ids
//                  are escaped as json4s 3.2 quotes them.
__device__ __forceinline__ bool mq_valid(const uint8_t *v, long long r) { return !v || ((v[r >> 3] >> (r & 7)) & 1); }

__global__ void k_mq_rows(long long R, const uint8_t *__restrict__ uvalid, const uint8_t *__restrict__ ivalid,
                          const uint8_t *__restrict__ svalid, int has_users, int has_items, int has_sets, long long D, long long item_at,
                          const int32_t *__restrict__ gid, const uint32_t *__restrict__ first_sorted, int32_t *__restrict__ rec_uid,
                          int32_t *__restrict__ rec_doc, int32_t *__restrict__ rec_key, uint8_t *__restrict__ rec_set,
                          uint8_t *__restrict__ queried) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < R; r += (long long)gridDim.x * blockDim.x) {
    if (!has_users || !mq_valid(uvalid, r)) rec_uid[r] = -1;
    int32_t d = -1, k = -1;
    if (has_items && mq_valid(ivalid, r)) {
      k = (int32_t)(item_at + r);
      const uint32_t f = first_sorted[gid[k]];
      if ((long long)f < D) d = (int32_t)f;
    }
    rec_doc[r] = d;
    rec_key[r] = k;
    if (d >= 0) queried[d] = 1;
    rec_set[r] = has_sets && mq_valid(svalid, r) ? 1 : 0;
  }
}

// A row reads everything that is not its own through its template tp = rec_tpl[r]: the template pieces from tpiece[tp] on
// (see mq_template), its history names hname[hbeg[tp] .. hbeg[tp + 1]) (indices into the union of query names that the
// history segments were built over), its flags and its user blacklist black[tmask[tp]].
enum : uint8_t { kMqHistInMust = 1, kMqSimilarInMust = 2, kMqExcludeSelf = 4, kMqWithSet = 8 };
struct MqArgs {
  long long n_rec;
  const int32_t *rec_uid;          // [n_rec] user group of the history, -1: no user or no history
  const int32_t *rec_doc;          // [n_rec] document, -1
  const int32_t *rec_key;          // [n_rec] key entry of the item, -1: no item
  const uint8_t *rec_set;          // [n_rec] the row has a set
  const int32_t *rec_tpl;          // [n_rec] template
  UqArgs h;                        // the history over the union of names
  const int32_t *tpiece;           // [T] first template piece
  const int32_t *hbeg;             // [T + 1]
  const int32_t *hname;            // [hbeg[T]] union name index, -1 for a template no row with a user reads
  const uint8_t *tflag;            // [T] kMq* bits
  const int32_t *tmask;            // [T] blacklist of the template's rows
  const MqBlack *black;
  const int32_t *kgid;             // key column: decoded _ids, items, blacklistItems, elements; group per entry
  const long long *koff;
  const unsigned char *kbytes;
  const int32_t *klog;             // per key entry: the log's item group, -1 (documents and unknown ids)
  const long long *line_moff;      // the source of document d has members iff line_moff[2 d + 2] > line_moff[2 d + 1]
  int T, n_names;                  // distinct model names; model names
  const int32_t *name_entry;
  const long long *eoff;           // [D * T + 1]
  const long long *doff;           // decoded elements of the documents
  const unsigned char *dbytes;
  long long slice;                 // max_query_events
  long long list_at;               // blacklistItems entry i is key entry list_at + i
  const long long *loff;           // list l is entries [loff[l], loff[l + 1]); row r reads list 0 (list_shared) or r
  int list_shared;
  const uint8_t *first_in_list;    // [entries] the entry is its string's first occurrence in its list
  const unsigned long long *lkey;  // [entries] (list << 32 | group), sorted: each list's groups, for membership
  const long long *soff;           // [n_rec + 1] 0-based element index of each row's set
  long long elem_at;               // element e is key entry elem_at + e
  const uint8_t *first_in_set;     // [elements] the element is its string's first occurrence in its set
  const long long *toff;           // template pieces of every template (see mq_template)
  const unsigned char *tbytes;
};

template <bool WRITE>
__global__ void __launch_bounds__(256, 1) k_mq_record(MqArgs a, const long long *__restrict__ rec_off, long long *__restrict__ rec_len,
                                                   unsigned char *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long r = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; r < a.n_rec; r += warps) {
    const int32_t u = a.rec_uid[r], d = a.rec_doc[r], key = a.rec_key[r], tp = a.rec_tpl[r];
    const int pb = a.tpiece[tp], h0n = a.hbeg[tp], n_kept = a.hbeg[tp + 1] - h0n;
    const unsigned fl = a.tflag[tp];
    const bool similar = d >= 0 && a.line_moff[2 * (long long)d + 2] > a.line_moff[2 * (long long)d + 1];
    const long long e0 = a.soff[r], ne = a.rec_set[r] ? a.soff[r + 1] - e0 : 0, k0 = a.elem_at + e0;
    const bool set_clause = (fl & kMqWithSet) && a.rec_set[r];
    RecordOut<WRITE> w{WRITE ? out + rec_off[r] : nullptr, 0, lane};
    // should (must = false) or must: the head, history, similar items, then should's boosted metadata, set clause and
    // constant_score, or must's tail, comma-separated
    auto section = [&](bool must) {
      bool any = w.piece(a, pb + (must ? 12 : 11));
      for (int j = 0; ((fl & kMqHistInMust) != 0) == must && j < n_kept; ++j) {
        if (any) w.comma();
        w.piece(a, pb + 13 + j);
        bool first = true;   // the history of name j, oldest first, each item at its first position
        if (u >= 0) {
          const int q = a.hname[h0n + j];
          const unsigned long long s = (unsigned long long)u * a.h.nq + q;
          const long long h0 = a.h.hstart[s], cnt = min(a.h.hstart[s + 1] - h0, (long long)a.h.limit[q]);
          w.list(cnt, [&](long long i, const unsigned char **p, long long *len) {
            const long long pos = h0 + cnt - 1 - i;
            if (!a.h.keep_h[pos]) return false;
            const uint32_t e = a.h.ent[a.h.hord[pos]];
            *p = a.h.ibytes + a.h.ioff[e];
            *len = a.h.ioff[e + 1] - a.h.ioff[e];
            return true;
          }, first);
        }
        w.piece(a, pb + 7);
        any = true;
      }
      for (int j = 0; similar && ((fl & kMqSimilarInMust) != 0) == must && j < a.n_names; ++j) {
        if (any) w.comma();
        w.piece(a, pb + 13 + n_kept + j);
        const long long x = (long long)d * a.T + a.name_entry[j], x0 = a.eoff[x], n = a.eoff[x + 1] - x0;
        bool first = true;
        w.list(n <= a.slice ? n : a.slice - 1, [&](long long i, const unsigned char **p, long long *len) {
          *p = a.dbytes + a.doff[x0 + i];
          *len = a.doff[x0 + i + 1] - a.doff[x0 + i];
          return true;
        }, first);
        w.piece(a, pb + 8);
        any = true;
      }
      const int tail = pb + (must ? 3 : 1);   // must's tail, or should's boosted metadata
      if (a.toff[tail + 1] > a.toff[tail]) {
        if (any) w.comma();
        w.piece(a, tail);
        any = true;
      }
      if (must) return;
      if (set_clause) {   // every element as given
        if (any) w.comma();
        w.piece(a, pb + 9);
        bool first = true;
        w.list(ne, [&](long long i, const unsigned char **p, long long *len) {
          *p = a.kbytes + a.koff[k0 + i];
          *len = a.koff[k0 + i + 1] - a.koff[k0 + i];
          return true;
        }, first);
        w.piece(a, pb + 10);
        any = true;
      }
      if (a.toff[pb + 3] > a.toff[pb + 2]) {
        if (any) w.comma();
        w.piece(a, pb + 2);
      }
    };
    w.piece(a, pb + 0);
    section(false);
    w.piece(a, pb + 4);
    section(true);
    w.piece(a, pb + 5);
    // the exclusion list: the user's blacklisted items newest first, blacklistItems, the item, the set; each id once
    const MqBlack bl = a.black[u >= 0 ? a.tmask[tp] : 0];
    auto in_user = [&](long long k) {
      const int32_t g = a.klog[k];
      return u >= 0 && g >= 0 && uq_has(bl, u, g);
    };
    const long long lr = a.list_shared ? 0 : r, l0 = a.loff[lr], l1 = a.loff[lr + 1];
    auto in_list = [&](int32_t g) {   // g is in the row's blacklistItems
      const unsigned long long x = ((unsigned long long)lr << 32) | (uint32_t)g;
      long long lo = l0, hi = l1;
      while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (a.lkey[mid] < x) lo = mid + 1; else hi = mid;
      }
      return lo < l1 && a.lkey[lo] == x;
    };
    bool first = true;
    if (u >= 0) {
      const long long b0 = bl.bstart[u];
      w.list(bl.bstart[u + 1] - b0, [&](long long i, const unsigned char **p, long long *len) {
        if (!bl.keep_b[b0 + i]) return false;
        const uint32_t e = a.h.ent[bl.bord[b0 + i]];
        *p = a.h.ibytes + a.h.ioff[e];
        *len = a.h.ioff[e + 1] - a.h.ioff[e];
        return true;
      }, first);
    }
    w.list(l1 - l0, [&](long long i, const unsigned char **p, long long *len) {
      const long long k = a.list_at + l0 + i;
      if (!a.first_in_list[l0 + i] || in_user(k)) return false;
      *p = a.kbytes + a.koff[k];
      *len = a.koff[k + 1] - a.koff[k];
      return true;
    }, first);
    const bool self = (fl & kMqExcludeSelf) && key >= 0;
    if (self && !in_list(a.kgid[key]) && !in_user(key))
      w.list(1, [&](long long, const unsigned char **p, long long *len) {
        *p = a.kbytes + a.koff[key];
        *len = a.koff[key + 1] - a.koff[key];
        return true;
      }, first);
    w.list(ne, [&](long long i, const unsigned char **p, long long *len) {
      const long long k = k0 + i;
      if (!a.first_in_set[e0 + i] || (self && a.kgid[k] == a.kgid[key]) || in_list(a.kgid[k]) || in_user(k)) return false;
      *p = a.kbytes + a.koff[k];
      *len = a.koff[k + 1] - a.koff[k];
      return true;
    }, first);
    w.piece(a, pb + 6);
    if (!WRITE && lane == 0) rec_len[r] = w.cur;
  }
}

// ---- cco_query_file_read: the lines of a batchpredict query file (tokenized by k_json_members) ------------------------
// Known members, by table entry (kQf*): the four row members, withRanks, then the template members in their fixed order.
//   k_qf_lines     one thread per line: each known member once, null = absent; user / item must be one string (its inside
//                  becomes a span for the decoder), itemSet / blacklistItems are picked for k_iq_array, withRanks must be
//                  true / false; the template members' raw value spans
//   k_qf_key<>     the template key of each line: the raw spans of the template members in order, separated by '\0' (an
//                  absent member leaves its place empty), a length pass and a write pass
//   k_qf_bits      per-line member flags -> LSB-first validity bitmaps (for k_mq_rows)
//   k_qf_first     per template: its first line with a user, with an item and with a set
enum : int { kQfUser = 0, kQfItem, kQfItemSet, kQfBlacklistItems, kQfWithRanks, kQfTemplate0 };
constexpr int kQfTemplateMembers = 10, kQfMembers = kQfTemplate0 + kQfTemplateMembers;
enum : unsigned { kQfRepeated = 16, kQfType = 17 };   // error codes next to the tokenizer's; the member entry rides in bits 8..15

__device__ __forceinline__ bool qf_literal(const unsigned char *b, const JMember &m, const char *lit, int n) {
  if (m.ve - m.vb != n) return false;
  for (int k = 0; k < n; ++k)
    if (b[m.vb + k] != (unsigned char)lit[k]) return false;
  return true;
}
__global__ void k_qf_lines(long long L, const long long *__restrict__ moff, const JMember *__restrict__ mem, const int32_t *__restrict__ ngid,
                           const int32_t *__restrict__ entry_of, const unsigned char *__restrict__ body, JMember *__restrict__ uspan,
                           JMember *__restrict__ ispan, int32_t *__restrict__ pick_set, int32_t *__restrict__ pick_list,
                           int32_t *__restrict__ tmem, uint8_t *__restrict__ has, unsigned long long *__restrict__ err) {
  for (long long l = blockIdx.x * (long long)blockDim.x + threadIdx.x; l < L; l += (long long)gridDim.x * blockDim.x) {
    int32_t at[kQfMembers];
    for (int t = 0; t < kQfMembers; ++t) at[t] = -1;
    unsigned seen = 0, code = 0, bad_t = 0;
    for (long long m = moff[l]; m < moff[l + 1] && !code; ++m) {
      const int32_t t = entry_of[ngid[m]];
      if (t < 0) continue;
      if ((seen >> t) & 1) {
        code = kQfRepeated;
        bad_t = t;
      }
      seen |= 1u << t;
      if (!qf_literal(body, mem[m], "null", 4)) at[t] = (int32_t)m;
    }
    for (int t = 0; t < 2 && !code; ++t) {   // user, item: one string
      const int32_t m = at[t];
      if (m < 0) continue;
      const long long b = mem[m].vb, e = mem[m].ve - 1;
      bool ok = body[b] == '"' && e > b && body[e] == '"';
      long long q = b + 1;
      while (ok && q < e) {
        if (body[q] == '\\') q += 2;
        else if (body[q] == '"') ok = false;
        else ++q;
      }
      ok = ok && q == e;
      if (!ok) {
        code = kQfType;
        bad_t = t;
      }
    }
    if (!code && at[kQfWithRanks] >= 0 && !qf_literal(body, mem[at[kQfWithRanks]], "true", 4) && !qf_literal(body, mem[at[kQfWithRanks]], "false", 5)) {
      code = kQfType;
      bad_t = kQfWithRanks;
    }
    if (code) atomicMin(err, ((unsigned long long)l << 16) | (bad_t << 8) | code);
    uspan[l] = at[kQfUser] >= 0 ? JMember{mem[at[kQfUser]].vb + 1, mem[at[kQfUser]].ve - 1, 0, 0} : JMember{0, 0, 0, 0};
    ispan[l] = at[kQfItem] >= 0 ? JMember{mem[at[kQfItem]].vb + 1, mem[at[kQfItem]].ve - 1, 0, 0} : JMember{0, 0, 0, 0};
    pick_set[l] = at[kQfItemSet];
    pick_list[l] = at[kQfBlacklistItems];
    for (int k = 0; k < kQfTemplateMembers; ++k) tmem[l * kQfTemplateMembers + k] = at[kQfTemplate0 + k];
    has[l] = (at[kQfUser] >= 0 ? 1 : 0) | (at[kQfItem] >= 0 ? 2 : 0) | (at[kQfItemSet] >= 0 ? 4 : 0);
  }
}
template <bool kWrite>
__global__ void k_qf_key(long long L, const int32_t *__restrict__ tmem, const JMember *__restrict__ mem, const unsigned char *__restrict__ body,
                         long long *__restrict__ len, const long long *__restrict__ off, unsigned char *__restrict__ out) {
  for (long long l = blockIdx.x * (long long)blockDim.x + threadIdx.x; l < L; l += (long long)gridDim.x * blockDim.x) {
    long long k = kWrite ? off[l] : 0;
    for (int t = 0; t < kQfTemplateMembers; ++t) {
      if (t) {
        if (kWrite) out[k] = 0;
        ++k;
      }
      const int32_t m = tmem[l * kQfTemplateMembers + t];
      if (m < 0) continue;
      for (long long p = mem[m].vb; p < mem[m].ve; ++p, ++k)
        if (kWrite) out[k] = body[p];
    }
    if (!kWrite) len[l] = k;
  }
}
__global__ void k_qf_bits(long long L, const uint8_t *__restrict__ has, uint8_t *__restrict__ bits) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (L + 7) / 8; i += (long long)gridDim.x * blockDim.x)
    for (int b = 0; b < 3; ++b) {
      unsigned v = 0;
      for (int j = 0; j < 8 && i * 8 + j < L; ++j) v |= (unsigned)((has[i * 8 + j] >> b) & 1) << j;
      bits[b * ((L + 7) / 8) + i] = (uint8_t)v;
    }
}
__global__ void k_qf_first(long long L, const int32_t *__restrict__ tid, const uint8_t *__restrict__ has, long long *__restrict__ first) {
  for (long long l = blockIdx.x * (long long)blockDim.x + threadIdx.x; l < L; l += (long long)gridDim.x * blockDim.x)
    for (int b = 0; b < 3; ++b)
      if ((has[l] >> b) & 1) atomicMin((unsigned long long *)&first[3 * (long long)tid[l] + b], (unsigned long long)l);
}

}  // namespace cco
