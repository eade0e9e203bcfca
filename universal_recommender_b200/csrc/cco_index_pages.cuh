// cco_index_pages.cuh -- the model index read back from Elasticsearch _search / _search/scroll response pages on the device
// (cco_index_pages_*): what EsClient.getRDD (esJsonRDD, EsClient.scala:464-470) hands calcPop and EsClient.getSource
// (EsClient.scala:394-442) hands the item queries, as the bulk body cco_format_model writes:
//   {"index":{"_id":"<_id>"}}\n<_source without whitespace outside strings>\n   per hit, in page order.
//
// A page is one JSON value, often one multi-MB line.  The structural passes of cco_results.cuh index it as they index an
// _msearch body, down to depth kIpMaxDepth only (top '{' -> hits '{' -> hits '[' -> hit '{' -> _source '{'): a hit's
// members and its _source's brackets enter the index, what _source holds does not.  Then:
//   k_ip_top                one warp over the entries down to the hits' brackets: _scroll_id, error, status, timed_out,
//                           _shards.failed, hits.total and hits.hits; the hits' bracket entries and their count
//   k_ip_hit                one warp per hit over its members: the raw _id and the bytes of its _source (sr_members)
//   k_ip_doc<kWrite>        one warp per hit, 32 bytes per step (length pass + write pass): the action line with the
//                           decoded _id re-escaped (json_escaped_len), then _source with the whitespace outside strings
//                           dropped and its strings checked as cco_rerank_model checks them
// Walks compare member names decoded and accept any member order; members they do not read are skipped by depth.
#include <cuda_runtime.h>
#include <stdint.h>

namespace cco {

constexpr int kIpMaxDepth = 4;   // the index: down to the _source brackets
constexpr int kIpTopDepth = 3;   // the top walk: down to the hits' brackets

// what is wrong with a page, beyond the kSr* codes of the walks
enum {
  kIpTimedOut = 32,     // timed_out is true
  kIpShards,            // _shards.failed is not 0
  kIpHitsNotArray,      // hits.hits is neither an array nor absent (null)
  kIpNoSource,          // a hit without _source
  kIpSourceNotObject,   // a hit whose _source is not an object
};

// the top walk's result
struct IpTop {
  long long n_hits;
  long long total;          // hits.total when exact (ES 7: relation "eq" or none), else -1
  long long sid_b, sid_e;   // the raw inside of _scroll_id; sid_b < 0: absent
  long long status;         // the first "status" member, when it is a 32-bit integer (has_status)
  int has_status;
  int code;                 // 0, a kSr* code at byte `bad`, kSrNotObject, kSrEsError or a kIp* code
  long long bad;
};

// One warp over the entries at depth <= kIpTopDepth (the list x.src[0 .. n)): the page is ws* '{' members '}' ws*.  Of a
// repeated member the first counts, except "error", which fails the page wherever it is.  hopen / hclose (n / 2 + 1
// entries each): the index entries of each hit's brackets.
__global__ void k_ip_top(SrIdx x, long long n, long long len, IpTop *__restrict__ out, long long *__restrict__ hopen,
                         long long *__restrict__ hclose) {
  if (threadIdx.x >= 32) return;
  const int lane = threadIdx.x;
  const unsigned char *b = x.body;
  IpTop r = {0, -1, -1, -1, 0, 0, 0, 0};
  long long first = 0;
  while (first < len && sr_ws(b[first])) ++first;
  if (n < 2 || x.pos[x.at(0)] != first || b[first] != '{') {
    r.code = kSrNotObject;
  } else if (x.dep[x.at(n - 1)] != 0 || b[x.pos[x.at(n - 1)]] != '}' || !sr_gap_ws(b, x.pos[x.at(n - 1)] + 1, len)) {
    r.code = kSrSyntax;
    r.bad = x.pos[x.at(n - 1)] + 1;
  } else {
    bool seen_sid = false, seen_status = false, seen_to = false, seen_shards = false, seen_hits = false;
    bool has_error = false, timed_out = false, shards_failed = false;
    int hits_kind = -1, code = 0;   // hits.hits: -1 absent or null; code: the first error of a nested walk, at byte nbad
    long long ha = -1, hb = -1, bad = 0, nbad = 0;
    auto nested = [&](int rc, long long at) {
      if (rc && !code) {
        code = rc;
        nbad = at;
      }
    };
    const int rc = sr_members(x, 0, n - 1, 1, &bad, [&](long long nb, long long ne, const SrVal &v) {
      if (sr_is(b, nb, ne, "error", 5)) {
        has_error = true;
      } else if (sr_is(b, nb, ne, "_scroll_id", 10) && !seen_sid) {
        seen_sid = true;
        if (v.kind == kVString) {
          r.sid_b = v.b;
          r.sid_e = v.e;
        }
      } else if (sr_is(b, nb, ne, "status", 6) && !seen_status) {
        seen_status = true;
        r.has_status = v.kind == kVScalar && sr_integer(b, v.b, v.e, -2147483648LL, 2147483647LL, &r.status);
      } else if (sr_is(b, nb, ne, "timed_out", 9) && !seen_to) {
        seen_to = true;
        timed_out = v.kind == kVScalar && v.e - v.b == 4 && b[v.b] == 't';
      } else if (sr_is(b, nb, ne, "_shards", 7) && !seen_shards) {
        seen_shards = true;
        if (v.kind != kVObject) return true;
        long long bad2 = 0;
        bool seen_failed = false;
        nested(sr_members(x, sr_walk_at(x.src, n, v.ob), sr_walk_at(x.src, n, v.oe), 2, &bad2, [&](long long nb2, long long ne2, const SrVal &w) {
                 if (!seen_failed && sr_is(b, nb2, ne2, "failed", 6)) {
                   seen_failed = true;
                   long long f = 1;
                   shards_failed = w.kind != kVScalar || !sr_integer(b, w.b, w.e, -1, 1, &f) || f != 0;
                 }
                 return true;
               }),
               bad2);
      } else if (sr_is(b, nb, ne, "hits", 4) && !seen_hits) {
        seen_hits = true;
        if (v.kind != kVObject) return true;
        long long bad2 = 0;
        bool seen_total = false, seen_inner = false;
        nested(sr_members(x, sr_walk_at(x.src, n, v.ob), sr_walk_at(x.src, n, v.oe), 2, &bad2, [&](long long nb2, long long ne2, const SrVal &w) {
                 if (sr_is(b, nb2, ne2, "total", 5) && !seen_total) {
                   seen_total = true;
                   if (w.kind == kVScalar) {
                     if (!sr_integer(b, w.b, w.e, -9223372036854775807LL, 9223372036854775807LL, &r.total)) r.total = -1;
                   } else if (w.kind == kVObject) {   // ES 7: {"value": n, "relation": "eq" | "gte"}
                     long long bad3 = 0, value = -1;
                     bool seen_value = false, seen_rel = false, exact = true;
                     nested(sr_members(x, sr_walk_at(x.src, n, w.ob), sr_walk_at(x.src, n, w.oe), 3, &bad3,
                                       [&](long long nb3, long long ne3, const SrVal &u) {
                                         if (!seen_value && sr_is(b, nb3, ne3, "value", 5)) {
                                           seen_value = true;
                                           if (u.kind != kVScalar ||
                                               !sr_integer(b, u.b, u.e, -9223372036854775807LL, 9223372036854775807LL, &value))
                                             exact = false;
                                         } else if (!seen_rel && sr_is(b, nb3, ne3, "relation", 8)) {
                                           seen_rel = true;
                                           exact = exact && u.kind == kVString && sr_is(b, u.b, u.e, "eq", 2);
                                         }
                                         return true;
                                       }),
                            bad3);
                     r.total = seen_value && exact ? value : -1;
                   }
                 } else if (sr_is(b, nb2, ne2, "hits", 4) && !seen_inner) {
                   seen_inner = true;
                   hits_kind = w.kind == kVScalar && sr_is_null(b, w.b, w.e) ? -1 : w.kind;
                   ha = w.ob;
                   hb = w.oe;
                 }
                 return true;
               }),
               bad2);
      }
      return true;
    });
    if (rc) {
      r.code = rc;
      r.bad = bad;
    } else if (code) {
      r.code = code;
      r.bad = nbad;
    } else if (has_error) {
      r.code = kSrEsError;
    } else if (timed_out) {
      r.code = kIpTimedOut;
    } else if (shards_failed) {
      r.code = kIpShards;
    } else if (hits_kind != -1 && hits_kind != kVArray) {
      r.code = kIpHitsNotArray;
    } else if (hits_kind == kVArray) {
      long long nh = 0;
      r.code = sr_objects(x, sr_walk_at(x.src, n, ha), sr_walk_at(x.src, n, hb), 3, kSrHitNotObject, &bad, &nh,
                          [&](long long k, long long o, long long c) {
                            if (lane == 0) {
                              hopen[k] = o;
                              hclose[k] = c;
                            }
                          });
      r.bad = bad;
      r.n_hits = r.code ? 0 : nh;
    }
  }
  if (lane == 0) *out = r;
}

// One warp per hit over its members (depth kIpMaxDepth): id[h] = the raw inside of its _id, [sb[h], se[h]) = the bytes of
// its first _source.  A malformed hit sets byte_err (byte offset << 8 | code), a hit without a string _id, with a repeated
// _id or without an object _source sets err (hit << 8 | code).
__global__ void k_ip_hit(SrIdx x, long long n_hits, const long long *__restrict__ hopen, const long long *__restrict__ hclose,
                         JMember *__restrict__ id, long long *__restrict__ sb, long long *__restrict__ se, unsigned long long *__restrict__ err,
                         unsigned long long *__restrict__ byte_err) {
  const int lane = threadIdx.x & 31;
  const unsigned char *b = x.body;
  for (long long h = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; h < n_hits; h += ((long long)gridDim.x * blockDim.x) >> 5) {
    int n_id = 0, n_src = 0;
    bool id_str = true, src_obj = false;
    long long ib = 0, ie = 0, s0 = 0, s1 = 0, bad = 0;
    const int rc = sr_members(x, hopen[h], hclose[h], kIpMaxDepth, &bad, [&](long long nb, long long ne, const SrVal &v) {
      if (sr_is(b, nb, ne, "_id", 3)) {
        id_str = id_str && v.kind == kVString;
        if (!n_id++) {
          ib = v.b;
          ie = v.e;
        }
      } else if (sr_is(b, nb, ne, "_source", 7) && !n_src++ && v.kind == kVObject) {
        src_obj = true;
        s0 = x.pos[v.ob];
        s1 = x.pos[v.oe] + 1;
      }
      return true;
    });
    const int code = rc ? 0 : !n_id || !id_str ? kSrNoId : n_id > 1 ? kSrRepeatedId : !n_src ? kIpNoSource : !src_obj ? kIpSourceNotObject : 0;
    if (lane == 0) {
      if (rc) sr_fail(byte_err, bad, rc);
      if (code) sr_fail(err, h, code);
      const bool ok = !rc && !code;
      id[h] = ok ? JMember{ib, ie, 0, 0} : JMember{0, 0, 0, 0};
      sb[h] = ok ? s0 : 0;
      se[h] = ok ? s1 : 0;
    }
  }
}

// ---- the documents -----------------------------------------------------------------------------------------------------
constexpr int kIpHead = 17, kIpMid = 4;   // {"index":{"_id":"  and  "}}\n ; a document ends with '\n'
struct IpDocs {
  const unsigned char *page;
  const long long *sb, *se;     // each hit's _source bytes in the page
  const long long *id_off;      // the decoded ids, id h = id[id_off[h] .. id_off[h + 1])
  const unsigned char *id;
};
__device__ __forceinline__ unsigned ip_prefix_xor(unsigned x) {
  x ^= x << 1;
  x ^= x << 2;
  x ^= x << 4;
  x ^= x << 8;
  x ^= x << 16;
  return x;
}
// One warp per hit.  Length pass: len[h] = the document's bytes, max_line = the longest _source line, err = the first byte
// (<< 8 | kSrString) of a _source string with a bad escape or a raw byte < 0x20, or of a backslash outside a string.  Write
// pass: the document at out + off[h].  _source goes 32 bytes per step; an odd run of backslashes escapes the byte after it
// (the run's parity is carried from step to step), the unescaped quotes' prefix XOR is the in-string mask (opening quote
// in, closing quote out), and whitespace outside strings is dropped.
template <bool kWrite>
__global__ void k_ip_doc(IpDocs a, long long n, long long *__restrict__ len, const long long *__restrict__ off, unsigned char *__restrict__ out,
                         unsigned long long *__restrict__ err, unsigned long long *__restrict__ max_line) {
  const int lane = threadIdx.x & 31;
  const unsigned below = (1u << lane) - 1;
  for (long long h = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; h < n; h += ((long long)gridDim.x * blockDim.x) >> 5) {
    long long w = kWrite ? off[h] : 0;
    if (kWrite && lane < kIpHead) out[w + lane] = (unsigned char)"{\"index\":{\"_id\":\""[lane];
    w += kIpHead;
    const long long i0 = a.id_off[h], i1 = a.id_off[h + 1];
    for (long long q = i0; q < i1; q += 32) {   // the id through json_escaped_len's escape
      const long long p = q + lane;
      const unsigned char c = p < i1 ? a.id[p] : 0;
      const int k = p < i1 ? json_escaped_len(c) : 0;
      int incl = k;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += y;
      }
      if (kWrite && k) {
        unsigned char *o = out + w + incl - k;
        if (k == 1) {
          o[0] = c;
        } else if (k == 2) {
          o[0] = '\\';
          o[1] = c;
        } else {
          o[0] = '\\'; o[1] = 'u'; o[2] = '0'; o[3] = '0';
          o[4] = (unsigned char)('0' + (c >> 4));   // c < 0x20
          o[5] = (unsigned char)((c & 15) < 10 ? '0' + (c & 15) : 'a' + (c & 15) - 10);
        }
      }
      w += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (kWrite && lane < kIpMid) out[w + lane] = (unsigned char)"\"}}\n"[lane];
    w += kIpMid;
    const long long line_at = w;
    const long long s0 = a.sb[h], s1 = a.se[h];
    unsigned in_str = 0, bs_odd = 0;
    for (long long base = s0; base < s1; base += 32) {
      const long long p = base + lane;
      const bool in = p < s1;
      const unsigned c = in ? a.page[p] : ' ';
      const unsigned bsm = __ballot_sync(0xffffffffu, c == '\\');
      const unsigned nbm = ~bsm & below;
      const unsigned esc = (nbm ? lane - 1 - (31 - __clz(nbm)) : lane + bs_odd) & 1;
      const unsigned qm = __ballot_sync(0xffffffffu, c == '"' && !esc);
      const unsigned sm = ip_prefix_xor(qm) ^ (in_str ? 0xffffffffu : 0u);
      const bool S = (sm >> lane) & 1, uq = (qm >> lane) & 1;
      const unsigned keepm = __ballot_sync(0xffffffffu, in && (S || !sr_ws(c)));
      if (!kWrite) {
        const bool bad = in && ((S && !uq && c < 0x20) || (c == '\\' && (!S || (!esc && !json_escape_ok(a.page, p, s1)))));
        const unsigned badm = __ballot_sync(0xffffffffu, bad);
        if (badm) {
          if (lane == 0) sr_fail(err, base + __ffs(badm) - 1, kSrString);
          break;
        }
      } else if ((keepm >> lane) & 1) {
        out[w + __popc(keepm & below)] = (unsigned char)c;
      }
      w += __popc(keepm);
      in_str = sm >> 31;
      if (~bsm) bs_odd = __clz(~bsm) & 1;
    }
    if (kWrite && lane == 0) out[w] = '\n';
    ++w;
    if (!kWrite && lane == 0) {
      len[h] = w;
      atomicMax(max_line, (unsigned long long)(w - 1 - line_at));
    }
  }
}

}  // namespace cco
