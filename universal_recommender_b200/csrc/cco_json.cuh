// cco_json.cuh -- the Elasticsearch bulk body of an existing model index, parsed on the device (cco_rerank_model).
//
// What the reference does with it (calcPop, URAlgorithm.scala:375-399): read the live index, join the fresh rankings and
// properties into every document by item id (URModel.scala:47-102) and write the index again.  The caller reads the index
// (cco_index_pages turns Elasticsearch's pages into the bulk body); this file splits that body into documents and
// top-level members:
//   k_nl_count / k_nl_write        '\n' positions: one warp per 2 KB chunk of the body's 8-byte words, a count pass and a
//                                  write pass around an exclusive scan of the chunk counts
//   k_json_members                 structural tokenizer, one warp per object span (a line, or the value of an action's
//                                  "index" member): the members' raw name spans and trimmed value spans, count pass + write
//                                  pass (the k_doc_len / k_doc_write idiom); a malformed span sets an error word
//   k_json_unescape                JSON string decoder (\" \\ \/ \b \f \n \r \t \uXXXX with surrogate pairs -> UTF-8), length
//                                  pass + write pass, one thread per string
//   k_action_check / k_pick_id     the action line is {"index":{..., "_id":"<string>", ...}}
//   k_name_entry / k_member_info   decoded member names -> the field / ranking / "id" table; repeated names (the last wins)
//   k_rerank_len / k_rerank_write  the merged documents of the old index (cco_format.cuh writes the new items' documents)
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace cco {

// one top-level member of an object: raw name bytes [nb, ne) (between the quotes, still escaped) and the value [vb, ve)
// without surrounding whitespace, as byte positions in the body
struct JMember {
  long long nb, ne, vb, ve;
};

// error word of a tokenizer run: min over bad spans of (span << 8 | code)
enum : unsigned { kJsonSyntax = 1, kJsonString = 2, kJsonNotObject = 3, kJsonAction = 4, kJsonLongLine = 5 };

// ---- line split ---------------------------------------------------------------------------------------------------------
constexpr int kNlChunkWords = 256;   // one warp: 8 steps of 32 words
__device__ __forceinline__ int nl_in_word(uint64_t x) {
  return (__popc(__vcmpeq4((unsigned)x, 0x0a0a0a0au)) + __popc(__vcmpeq4((unsigned)(x >> 32), 0x0a0a0a0au))) >> 3;
}
// the body's bytes past its end are zero in the last word
__global__ void k_nl_count(long long n_words, const uint64_t *__restrict__ w, long long *__restrict__ count) {
  const int lane = threadIdx.x & 31;
  const long long n_chunks = (n_words + kNlChunkWords - 1) / kNlChunkWords;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long ch = warp; ch < n_chunks; ch += nwarps) {
    int k = 0;
    for (int it = 0; it < kNlChunkWords / 32; ++it) {
      const long long q = ch * kNlChunkWords + it * 32 + lane;
      if (q < n_words) k += nl_in_word(w[q]);
    }
    for (int o = 16; o > 0; o >>= 1) k += __shfl_xor_sync(0xffffffffu, k, o);
    if (lane == 0) count[ch] = k;
  }
}
__global__ void k_nl_write(long long n_words, const uint64_t *__restrict__ w, const long long *__restrict__ chunk_off,
                           long long *__restrict__ pos) {
  const int lane = threadIdx.x & 31;
  const long long n_chunks = (n_words + kNlChunkWords - 1) / kNlChunkWords;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long ch = warp; ch < n_chunks; ch += nwarps) {
    long long at = chunk_off[ch];
    for (int it = 0; it < kNlChunkWords / 32; ++it) {
      const long long q = ch * kNlChunkWords + it * 32 + lane;
      const uint64_t x = q < n_words ? w[q] : 0;
      const int k = nl_in_word(x);
      int incl = k;
      for (int d = 1; d < 32; d <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += v;
      }
      long long o = at + incl - k;
      for (int j = 0; k && j < 8; ++j)
        if (((x >> (8 * j)) & 0xff) == 0x0a) pos[o++] = q * 8 + j;
      at += __shfl_sync(0xffffffffu, incl, 31);
    }
  }
}
// line l = [pos[l - 1] + 1, pos[l]) (the first starts at 0)
__global__ void k_line_spans(long long n_lines, const long long *__restrict__ pos, long long *__restrict__ sb, long long *__restrict__ se) {
  for (long long l = blockIdx.x * (long long)blockDim.x + threadIdx.x; l < n_lines; l += (long long)gridDim.x * blockDim.x) {
    sb[l] = l ? pos[l - 1] + 1 : 0;
    se[l] = pos[l];
  }
}

// ---- structural tokenizer --------------------------------------------------------------------------------------------
__device__ __forceinline__ bool json_ws(unsigned c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r'; }
__device__ __forceinline__ bool json_hex(unsigned c) { return c - '0' < 10u || (c | 0x20) - 'a' < 6u; }
// the escape that starts at the backslash at p is complete inside the span and one of \" \\ \/ \b \f \n \r \t \uXXXX
__device__ __noinline__ bool json_escape_ok(const unsigned char *__restrict__ body, long long p, long long e) {
  if (p + 1 >= e) return false;
  const unsigned x = body[p + 1];
  if (x == 'u') {
    if (p + 5 >= e) return false;
    for (int k = 2; k < 6; ++k)
      if (!json_hex(body[p + k])) return false;
    return true;
  }
  return x == '"' || x == '\\' || x == '/' || x == 'b' || x == 'f' || x == 'n' || x == 'r' || x == 't';
}

// Grammar of a span: ws* '{' ws* ( '}' | member (ws* ',' ws* member)* ws* '}' ) ws*, member = string ws* ':' ws* value.
// A value runs from its first byte to the last non-whitespace byte before the ',' or '}' that ends it at depth 1; its
// inside is not validated beyond the string rules (closed strings, valid escapes, no raw byte < 0x20) and bracket depth.
// One warp per span, 32 bytes per step; the state that crosses a step: in-string, the parity of a trailing backslash run,
// the depth, the last non-whitespace position and the member being read.
//   escaped byte   = an odd run of backslashes right before it (backslashes occur only inside strings, else an error)
//   in string      = prefix XOR of the unescaped quotes (the opening quote in, the closing quote out)
//   depth          = prefix count of '{' '[' minus '}' ']' outside strings (ballot popcounts)
// The bytes at depth <= 1 outside strings (and the quotes at depth 1) drive a small state machine, one event at a time.
enum : int { kJBefore = 0, kJFirst, kJNext, kJName, kJColon, kJValue0, kJValue, kJDone };
// a sink with a code(span, code) member is told each span's verdict (0: well formed); for the others this is a no-op
template <class Sink>
__device__ __forceinline__ auto sink_code(const Sink &sink, long long s, int code, int) -> decltype(sink.code(s, code), void()) {
  sink.code(s, code);
}
template <class Sink>
__device__ __forceinline__ void sink_code(const Sink &, long long, int, long) {}
// Every completed member goes to sink.member(span, index in span, span begin, member) on lane 0, and lane 0 calls
// sink.end(span, members) once per span; a malformed span sets the error word instead (its members may be partly sunk).
template <class Sink>
__global__ void k_json_members(long long n_spans, const long long *__restrict__ sb, const long long *__restrict__ se,
                               const unsigned char *__restrict__ body, const Sink sink, unsigned long long *__restrict__ err) {
  const int lane = threadIdx.x & 31;
  const unsigned below = (1u << lane) - 1, upto = 0xffffffffu >> (31 - lane);
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long s = warp; s < n_spans; s += nwarps) {
    const long long b = sb[s], e = se[s];
    int code = e - b > 0x7fffffffLL ? kJsonLongLine : 0;
    int state = kJBefore;
    long long n = 0, depth = 0, last_nonws = b - 1;
    JMember cur = {0, 0, 0, 0};
    unsigned in_str = 0, bs_odd = 0;
    for (long long base = b; base < e && !code; base += 32) {
      const long long p = base + lane;
      const unsigned c = p < e ? body[p] : ' ';
      const unsigned bsm = __ballot_sync(0xffffffffu, c == '\\');
      const unsigned nb = ~bsm & below;
      const unsigned esc = (nb ? lane - 1 - (31 - __clz(nb)) : lane + bs_odd) & 1;
      const unsigned qm = __ballot_sync(0xffffffffu, c == '"' && !esc);
      const bool uq = (qm >> lane) & 1;
      const bool S = (in_str ^ __popc(qm & upto)) & 1;   // inside a string, opening quote included
      const bool str = S || uq;
      const bool op = !str && (c == '{' || c == '['), cl = !str && (c == '}' || c == ']');
      const unsigned opm = __ballot_sync(0xffffffffu, op), clm = __ballot_sync(0xffffffffu, cl);
      const long long level = depth + __popc(opm & upto) - __popc(clm & upto) - (op ? 1 : 0);
      const bool nonws = p < e && !json_ws(c);
      bool bad = false;
      if (p < e && S && c < 0x20) bad = true;
      if (c == '\\') bad = !S || (!esc && !json_escape_ok(body, p, e));
      const unsigned Sm = __ballot_sync(0xffffffffu, S);
      const unsigned nwm = __ballot_sync(0xffffffffu, nonws);
      unsigned evm = __ballot_sync(0xffffffffu, nonws && (!S || uq) && level <= 1);
      if (__ballot_sync(0xffffffffu, bad)) code = kJsonString;
      while (evm && !code) {
        const int i = __ffs(evm) - 1;
        evm &= evm - 1;
        const unsigned ci = __shfl_sync(0xffffffffu, c, i);
        const long long li = __shfl_sync(0xffffffffu, level, i);
        const bool qi = (qm >> i) & 1, open_q = qi && ((Sm >> i) & 1);
        const long long pi = base + i;
        if (state == kJBefore) {
          if (ci == '{' && li == 0) state = kJFirst;
          else code = kJsonNotObject;
        } else if (state == kJFirst || state == kJNext) {
          if (open_q && li == 1) {
            cur.nb = pi + 1;
            state = kJName;
          } else if (state == kJFirst && ci == '}' && li == 0) {
            state = kJDone;
          } else {
            code = kJsonSyntax;
          }
        } else if (state == kJName) {   // the only event inside a name is its closing quote
          cur.ne = pi;
          state = kJColon;
        } else if (state == kJColon) {
          if (ci == ':' && !qi && li == 1) state = kJValue0;
          else code = kJsonSyntax;
        } else if (state == kJValue0) {
          if (li != 1 || (!qi && (ci == ',' || ci == ':'))) {
            code = kJsonSyntax;   // an empty value
          } else {
            cur.vb = pi;
            state = kJValue;
          }
        } else if (state == kJValue) {
          const bool comma = li == 1 && !qi && ci == ',';
          if (comma || li == 0) {
            if (li == 0 && ci != '}') {
              code = kJsonSyntax;
            } else {
              const unsigned lb = nwm & ((1u << i) - 1);
              cur.ve = (lb ? base + 31 - __clz(lb) : last_nonws) + 1;
              if (lane == 0) sink.member(s, n, b, cur);
              ++n;
              state = comma ? kJNext : kJDone;
            }
          } else if (li == 1 && !qi && ci == ':') {
            code = kJsonSyntax;
          }
        } else {
          code = kJsonSyntax;   // anything after the closing brace
        }
      }
      in_str = (in_str ^ __popc(qm)) & 1;
      depth += __popc(opm) - __popc(clm);
      if (nwm) last_nonws = base + 31 - __clz(nwm);
      if (~bsm) bs_odd = __clz(~bsm) & 1;
    }
    if (!code && state != kJDone) code = state == kJBefore ? kJsonNotObject : (in_str ? kJsonString : kJsonSyntax);
    if (lane == 0) {
      if (code) atomicMin(err, ((unsigned long long)s << 8) | (unsigned)code);
      sink_code(sink, s, code, 0);
      sink.end(s, n);
    }
  }
}
// the members of every span: count pass (count[s]) and write pass (out[moff[s] ..])
template <bool kWrite>
struct MemberSink {
  long long *count;
  const long long *moff;
  JMember *out;
  __device__ void member(long long s, long long n, long long, const JMember &m) const {
    if (kWrite) out[moff[s] + n] = m;
  }
  __device__ void end(long long s, long long n) const {
    if (!kWrite) count[s] = n;
  }
};

// ---- string decoder --------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned json_hex4(const unsigned char *__restrict__ p) {
  unsigned v = 0;
  for (int k = 0; k < 4; ++k) {
    const unsigned c = p[k];
    v = v * 16 + (c <= '9' ? c - '0' : (c | 0x20) - 'a' + 10);
  }
  return v;
}
// the raw bytes [m.nb, m.ne) of every string (escapes validated by k_json_members) as UTF-8; a surrogate that is not part
// of a pair is written as its 3-byte form (Python's "surrogatepass")
template <bool kWrite>
__global__ void k_json_unescape(long long n, const JMember *__restrict__ m, const unsigned char *__restrict__ body,
                                long long *__restrict__ len, const long long *__restrict__ off, unsigned char *__restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    long long q = m[i].nb, L = kWrite ? off[i] : 0;
    const long long e = m[i].ne;
    while (q < e) {
      const unsigned c = body[q];
      if (c != '\\') {
        if (kWrite) out[L] = (unsigned char)c;
        ++L;
        ++q;
        continue;
      }
      const unsigned x = body[q + 1];
      if (x != 'u') {
        if (kWrite) out[L] = (unsigned char)(x == 'b' ? 8 : x == 'f' ? 12 : x == 'n' ? 10 : x == 'r' ? 13 : x == 't' ? 9 : x);
        ++L;
        q += 2;
        continue;
      }
      unsigned cp = json_hex4(body + q + 2);
      q += 6;
      if (cp >= 0xd800 && cp < 0xdc00 && q + 6 <= e && body[q] == '\\' && body[q + 1] == 'u') {
        const unsigned lo = json_hex4(body + q + 2);
        if (lo >= 0xdc00 && lo < 0xe000) {
          cp = 0x10000 + ((cp - 0xd800) << 10) + (lo - 0xdc00);
          q += 6;
        }
      }
      const int k = cp < 0x80 ? 1 : cp < 0x800 ? 2 : cp < 0x10000 ? 3 : 4;
      if (kWrite) {
        if (k == 1) {
          out[L] = (unsigned char)cp;
        } else {
          for (int j = k - 1; j > 0; --j) {
            out[L + j] = (unsigned char)(0x80 | (cp & 0x3f));
            cp >>= 6;
          }
          out[L] = (unsigned char)((k == 2 ? 0xc0 : k == 3 ? 0xe0 : 0xf0) | cp);
        }
      }
      L += k;
    }
    if (!kWrite) len[i] = L;
  }
}

// decoded string i of a column (offsets + bytes) equals the literal lit
__device__ __forceinline__ bool dec_is(const long long *__restrict__ off, const unsigned char *__restrict__ bytes, long long i,
                                       const char *lit, int n) {
  if (off[i + 1] - off[i] != n) return false;
  for (int k = 0; k < n; ++k)
    if (bytes[off[i] + k] != (unsigned char)lit[k]) return false;
  return true;
}
// the action line of document d (line 2 d) is an object with exactly one member, named "index", whose value is an object:
// that value is the span of the second tokenizer run
__global__ void k_action_check(long long n_docs, const long long *__restrict__ line_moff, const JMember *__restrict__ mem,
                               const long long *__restrict__ name_off, const unsigned char *__restrict__ names,
                               const unsigned char *__restrict__ body, long long *__restrict__ ib, long long *__restrict__ ie,
                               unsigned long long *__restrict__ err) {
  for (long long d = blockIdx.x * (long long)blockDim.x + threadIdx.x; d < n_docs; d += (long long)gridDim.x * blockDim.x) {
    const long long m = line_moff[2 * d];
    const bool ok = line_moff[2 * d + 1] - m == 1 && dec_is(name_off, names, m, "index", 5) && body[mem[m].vb] == '{';
    if (!ok) atomicMin(err, ((unsigned long long)d << 8) | kJsonAction);
    ib[d] = ok ? mem[m].vb : 0;
    ie[d] = ok ? mem[m].ve : 0;
  }
}
// the "_id" of document d: the last member of that name in its "index" object, a string; ids[d] = its raw inside
__global__ void k_pick_id(long long n_docs, const long long *__restrict__ moff, const JMember *__restrict__ mem,
                          const long long *__restrict__ name_off, const unsigned char *__restrict__ names,
                          const unsigned char *__restrict__ body, JMember *__restrict__ ids, unsigned long long *__restrict__ err) {
  for (long long d = blockIdx.x * (long long)blockDim.x + threadIdx.x; d < n_docs; d += (long long)gridDim.x * blockDim.x) {
    long long pick = -1;
    for (long long m = moff[d]; m < moff[d + 1]; ++m)
      if (dec_is(name_off, names, m, "_id", 3)) pick = m;
    bool ok = pick >= 0 && body[mem[pick].vb] == '"';
    long long q = ok ? mem[pick].vb + 1 : 0;
    const long long e = ok ? mem[pick].ve - 1 : 0;
    while (ok && q < e) {   // the value is one string: its closing quote is its last byte
      if (body[q] == '\\') q += 2;
      else if (body[q] == '"') ok = false;
      else ++q;
    }
    ok = ok && q == e && body[e] == '"';
    if (!ok) atomicMin(err, ((unsigned long long)d << 8) | kJsonAction);
    ids[d] = ok ? JMember{mem[pick].vb + 1, e, 0, 0} : JMember{0, 0, 0, 0};
  }
}

// ---- member names -> fields, rankings, "id" -----------------------------------------------------------------------------
// entry[g] = the name table entry with the bytes of distinct member name g (its first member), -1
__global__ void k_name_entry(long long n_groups, const uint32_t *__restrict__ first_sorted, const long long *__restrict__ off,
                             const unsigned char *__restrict__ bytes, int n_entries, const long long *__restrict__ toff,
                             const unsigned char *__restrict__ tbytes, int32_t *__restrict__ entry) {
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < n_groups; g += (long long)gridDim.x * blockDim.x) {
    const uint32_t m = first_sorted[g];
    const long long a = off[m], len = off[m + 1] - a;
    int hit = -1;
    for (int t = 0; t < n_entries && hit < 0; ++t) {
      if (toff[t + 1] - toff[t] != len) continue;
      long long k = 0;
      while (k < len && bytes[a + k] == tbytes[toff[t] + k]) ++k;
      if (k == len) hit = t;
    }
    entry[g] = hit;
  }
}
// per member of document d's source (line 2 d + 1): its table entry, and whether it stays (not named "id", and no later
// member of the same name: json4s keeps the last).  One warp per document, the lanes over its members.
__global__ void k_member_info(long long n_docs, const long long *__restrict__ line_moff, const int32_t *__restrict__ gid,
                              const int32_t *__restrict__ entry_of, const uint8_t *__restrict__ ent_id, int32_t *__restrict__ ment,
                              uint8_t *__restrict__ mkeep) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long d = warp; d < n_docs; d += nwarps) {
    const long long m0 = line_moff[2 * d + 1], m1 = line_moff[2 * d + 2];
    for (long long m = m0 + lane; m < m1; m += 32) {
      const int32_t g = gid[m], t = entry_of[g];
      bool keep = !(t >= 0 && ent_id[t]);
      for (long long q = m + 1; keep && q < m1; ++q)
        if (gid[q] == g) keep = false;
      ment[m] = t;
      mkeep[m] = keep ? 1 : 0;
    }
  }
}

// ---- the documents of the old index --------------------------------------------------------------------------------------
// Per document, lowest to highest: fresh properties < old members < rankings (a later one beats an earlier one) < "id".
// Written: "id", the old members in their order (not "id", not named like a ranking present for the item, not followed by a
// member of the same name), the properties not named like any old member (cco_format.cuh's rules otherwise), the rankings.
struct RerankArgs {
  const long long *line_moff;   // [2 n_docs + 1]: line l's members are [line_moff[l], line_moff[l + 1])
  const JMember *mem;
  const int32_t *ment;          // table entry of each member's name, -1
  const uint8_t *mkeep;
  const int32_t *ent_field;     // per table entry: the property field of that name, -1
  const uint8_t *ent_rank;      // per table entry: bit k = ranking k has that name
  const unsigned char *body;
};
__device__ __forceinline__ bool member_written(const RerankArgs &r, long long m, unsigned mask) {
  return r.mkeep[m] && !(r.ment[m] >= 0 && (r.ent_rank[r.ment[m]] & mask));
}
__device__ __forceinline__ bool member_has_field(const RerankArgs &r, long long m0, long long m1, int f) {
  for (long long m = m0; m < m1; ++m)
    if (r.ment[m] >= 0 && r.ent_field[r.ment[m]] == f) return true;
  return false;
}
__device__ __forceinline__ bool rerank_prop_written(const FormatArgs &a, const RerankArgs &r, int g, int j, unsigned mask, long long m0,
                                                    long long m1) {
  return prop_last(a, g, j) && prop_written(a, j, mask) && !member_has_field(r, m0, m1, (int)(uint32_t)a.pkey[j]);
}

__global__ void k_rerank_len(const FormatArgs a, const RerankArgs r, int32_t n_docs, long long *__restrict__ doc_len) {
  for (int d = blockIdx.x * blockDim.x + threadIdx.x; d < n_docs; d += gridDim.x * blockDim.x) {
    const DocRef x = doc_ref(a, d);
    const unsigned mask = doc_rank_mask(a, x.g);
    const long long m0 = r.line_moff[2 * (long long)d + 1], m1 = r.line_moff[2 * (long long)d + 2];
    long long len = 17 + x.idl + 11 + x.idl + 1 + 2;
    for (long long m = m0; m < m1; ++m)
      if (member_written(r, m, mask)) len += (r.mem[m].ne - r.mem[m].nb) + 4 + (r.mem[m].ve - r.mem[m].vb);
    if (a.pbeg) {
      for (int j = a.pbeg[x.g]; j < a.pend[x.g]; ++j) {
        if (!rerank_prop_written(a, r, x.g, j, mask, m0, m1)) continue;
        const uint32_t f = (uint32_t)a.pkey[j];
        const int t = a.ptri[j];
        len += (a.field_off[f + 1] - a.field_off[f]) + 4 + (a.val_off[t + 1] - a.val_off[t]);
      }
    }
    for (int k = 0; k < a.n_rank; ++k) {
      if (!rank_written(a, k, mask)) continue;
      unsigned char txt[28];
      len += (a.rank_name_off[k + 1] - a.rank_name_off[k]) + 4 + java_double_text(a.score[(size_t)k * a.n_groups + x.g], a.rank_scale[k], txt);
    }
    doc_len[d] = len;
  }
}

// one warp per document, as k_doc_write
__global__ void k_rerank_write(const FormatArgs a, const RerankArgs r, int32_t n_docs, const long long *__restrict__ doc_off,
                               unsigned char *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int d = warp; d < n_docs; d += nwarps) {
    const DocRef x = doc_ref(a, d);
    const unsigned mask = doc_rank_mask(a, x.g);
    const long long m0 = r.line_moff[2 * (long long)d + 1], m1 = r.line_moff[2 * (long long)d + 2];
    unsigned char *w = out + doc_off[d];
    warp_lit(w, "{\"index\":{\"_id\":\"", 17, lane); w += 17;
    warp_copy(w, x.id, x.idl, lane); w += x.idl;
    warp_lit(w, "\"}}\n{\"id\":\"", 11, lane); w += 11;
    warp_copy(w, x.id, x.idl, lane); w += x.idl;
    warp_lit(w, "\"", 1, lane); w += 1;
    for (long long m = m0; m < m1; ++m) {   // old members, names and values as they were
      if (!member_written(r, m, mask)) continue;
      const JMember jm = r.mem[m];
      warp_lit(w, ",\"", 2, lane); w += 2;
      warp_copy(w, r.body + jm.nb, jm.ne - jm.nb, lane); w += jm.ne - jm.nb;
      warp_lit(w, "\":", 2, lane); w += 2;
      warp_copy(w, r.body + jm.vb, jm.ve - jm.vb, lane); w += jm.ve - jm.vb;
    }
    if (a.pbeg) {
      for (int j = a.pbeg[x.g]; j < a.pend[x.g]; ++j) {
        if (!rerank_prop_written(a, r, x.g, j, mask, m0, m1)) continue;
        const uint32_t f = (uint32_t)a.pkey[j];
        const int t = a.ptri[j];
        const long long nl = a.field_off[f + 1] - a.field_off[f], vl = a.val_off[t + 1] - a.val_off[t];
        warp_lit(w, ",\"", 2, lane); w += 2;
        warp_copy(w, a.names + a.field_off[f], nl, lane); w += nl;
        warp_lit(w, "\":", 2, lane); w += 2;
        warp_copy(w, a.vals + (a.val_off[t] - a.val_base), vl, lane); w += vl;
      }
    }
    for (int k = 0; k < a.n_rank; ++k) {
      if (!rank_written(a, k, mask)) continue;
      const int nl = a.rank_name_off[k + 1] - a.rank_name_off[k];
      unsigned char txt[28];
      const int tl = java_double_text(a.score[(size_t)k * a.n_groups + x.g], a.rank_scale[k], txt);
      warp_lit(w, ",\"", 2, lane); w += 2;
      warp_copy(w, a.names + a.rank_name_off[k], nl, lane); w += nl;
      warp_lit(w, "\":", 2, lane); w += 2;
      if (lane < tl) w[lane] = txt[lane];
      w += tl;
    }
    warp_lit(w, "}\n", 2, lane);
    __syncwarp();
  }
}

// a group of the key column that holds two old documents: dup = min over such documents d of (d << 32 | first document)
__global__ void k_dup_rows(long long n_rows, const int32_t *__restrict__ gid, const uint32_t *__restrict__ first_sorted,
                           unsigned long long *__restrict__ dup) {
  for (long long d = blockIdx.x * (long long)blockDim.x + threadIdx.x; d < n_rows; d += (long long)gridDim.x * blockDim.x) {
    const uint32_t f = first_sorted[gid[d]];
    if (f != (uint32_t)d) atomicMin(dup, ((unsigned long long)d << 32) | f);
  }
}

}  // namespace cco
