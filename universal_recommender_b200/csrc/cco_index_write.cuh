// cco_index_write.cuh -- the model index written into Elasticsearch as URModel.save / EsClient.hotSwap write it
// (URModel.scala:47-84, EsClient.scala:168-246, 257-362), the parts that read the body or the answers (cco_index_write_*):
//   k_iw_gate     the field scan's gate: the members of the document lines enter the name table, the action lines' do not;
//                 cco_strings.cuh's table (atomicMin first positions, sorted) then gives esFields in first-appearance order
//   k_iw_top      one warp over a _bulk response's entries down to the items' brackets: error, status and items
//   k_iw_item     one warp per item (sr_members): index._id against the document's decoded _id, index.status, and for an
//                 error item the raw insides of error.type and error.reason
// The response is indexed by cco_results.cuh's structural passes down to depth kIwMaxDepth (top '{' -> items '[' -> item
// '{' -> index '{' -> error '{' and its members); what error.caused_by holds never enters the index.  Walks compare member
// names decoded and accept any member order; members they do not read (_index, _type, _version, result, _shards, created,
// took, errors, ...) are skipped by depth.
#include <cuda_runtime.h>
#include <stdint.h>

namespace cco {

constexpr int kIwMaxDepth = 5;   // the index: down to the members of an item's error object
constexpr int kIwTopDepth = 2;   // the top walk: down to the items' brackets

// what is wrong with a _bulk response, beyond the kSr* codes of the walks
enum {
  kIwNoItems = 48,       // no "items" member, or it is not an array
  kIwItemNotObject,      // an items element that is not an object
  kIwNotIndex,           // an item whose one member is not an "index" object
  kIwNoId,               // an item without a string index._id
  kIwIdMismatch,         // index._id is not the document's _id
  kIwNoStatus,           // an item without index.status
  kIwRepeatedStatus,     // an item with two index.status members
  kIwBadStatus,          // index.status is not a 32-bit integer
};

// the top walk's result
struct IwTop {
  long long n_items;
  long long status;   // the first "status" member, when it is a 32-bit integer (has_status)
  int has_status;
  int code;           // 0, a kSr* code at byte `bad`, kSrNotObject, kSrEsError or a kIw* code
  long long bad;
};

// the items' side of one request: item i answers document docs ? docs[i] : doc0 + i
struct IwItems {
  const long long *docs;
  long long doc0;
  const long long *id_off;   // the body's decoded _ids: id d = id[id_off[d] .. id_off[d + 1])
  const unsigned char *id;
};
// an item whose status is not 2xx: the raw insides of its error.type and error.reason (b < 0: absent or not a string)
struct IwFail {
  long long item;
  long long tb, te, rb, re;
};

// The members of a document line enter the name table (gate 0), those of an action line do not (gate -1).
__global__ void k_iw_gate(long long n_lines, const long long *__restrict__ line_moff, int32_t *__restrict__ gate) {
  for (long long l = blockIdx.x * (long long)blockDim.x + threadIdx.x; l < n_lines; l += (long long)gridDim.x * blockDim.x) {
    const int32_t g = (l & 1) ? 0 : -1;
    for (long long m = line_moff[l]; m < line_moff[l + 1]; ++m) gate[m] = g;
  }
}

// One warp over the entries at depth <= kIwTopDepth (the list x.src[0 .. n)): the response is ws* '{' members '}' ws*.  Of
// a repeated member the first counts, except "error", which fails the response wherever it is.  iopen / iclose (n / 2 + 1
// entries each): the index entries of each item's brackets.
__global__ void k_iw_top(SrIdx x, long long n, long long len, IwTop *__restrict__ out, long long *__restrict__ iopen,
                         long long *__restrict__ iclose) {
  if (threadIdx.x >= 32) return;
  const int lane = threadIdx.x;
  const unsigned char *b = x.body;
  IwTop r = {0, 0, 0, 0, 0};
  long long first = 0;
  while (first < len && sr_ws(b[first])) ++first;
  if (n < 2 || x.pos[x.at(0)] != first || b[first] != '{') {
    r.code = kSrNotObject;
  } else if (x.dep[x.at(n - 1)] != 0 || b[x.pos[x.at(n - 1)]] != '}' || !sr_gap_ws(b, x.pos[x.at(n - 1)] + 1, len)) {
    r.code = kSrSyntax;
    r.bad = x.pos[x.at(n - 1)] + 1;
  } else {
    bool seen_status = false, seen_items = false, has_error = false;
    int items_kind = -1;
    long long ia = -1, ib = -1, bad = 0;
    const int rc = sr_members(x, 0, n - 1, 1, &bad, [&](long long nb, long long ne, const SrVal &v) {
      if (sr_is(b, nb, ne, "error", 5)) {
        has_error = true;
      } else if (sr_is(b, nb, ne, "status", 6) && !seen_status) {
        seen_status = true;
        r.has_status = v.kind == kVScalar && sr_integer(b, v.b, v.e, -2147483648LL, 2147483647LL, &r.status);
      } else if (sr_is(b, nb, ne, "items", 5) && !seen_items) {
        seen_items = true;
        items_kind = v.kind;
        ia = v.ob;
        ib = v.oe;
      }
      return true;
    });
    if (rc) {
      r.code = rc;
      r.bad = bad;
    } else if (has_error) {
      r.code = kSrEsError;
    } else if (items_kind != kVArray) {
      r.code = kIwNoItems;
    } else {
      long long ni = 0;
      r.code = sr_objects(x, sr_walk_at(x.src, n, ia), sr_walk_at(x.src, n, ib), 2, kIwItemNotObject, &bad, &ni,
                          [&](long long k, long long o, long long c) {
                            if (lane == 0) {
                              iopen[k] = o;
                              iclose[k] = c;
                            }
                          });
      r.bad = bad;
      r.n_items = r.code ? 0 : ni;
    }
  }
  if (lane == 0) *out = r;
}

// One warp per item over its members (the whole index, depth kIwMaxDepth).  status[doc] = index.status; an item whose status
// is not 2xx appends an IwFail to fail[0 .. *n_fail).  A malformed item sets byte_err (byte offset << 8 | code), an item
// that breaks the rules sets err (item << 8 | code).
__global__ void k_iw_item(SrIdx x, long long n_items, const long long *__restrict__ iopen, const long long *__restrict__ iclose, IwItems it,
                          int32_t *__restrict__ status, IwFail *__restrict__ fail, unsigned long long *__restrict__ n_fail,
                          unsigned long long *__restrict__ err, unsigned long long *__restrict__ byte_err) {
  const int lane = threadIdx.x & 31;
  const unsigned char *b = x.body;
  for (long long i = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; i < n_items; i += ((long long)gridDim.x * blockDim.x) >> 5) {
    const long long doc = it.docs ? it.docs[i] : it.doc0 + i;
    int n_members = 0, n_id = 0, n_status = 0, nested = 0;
    bool index_obj = false, id_str = true, status_ok = true, seen_error = false, seen_type = false, seen_reason = false;
    long long ob = 0, oe = 0, idb = 0, ide = 0, st = 0, tb = -1, te = -1, rb = -1, re = -1, bad = 0, nbad = 0;
    int rc = sr_members(x, iopen[i], iclose[i], 3, &bad, [&](long long nb, long long ne, const SrVal &v) {
      if (!n_members++ && sr_is(b, nb, ne, "index", 5) && v.kind == kVObject) {
        index_obj = true;
        ob = v.ob;
        oe = v.oe;
      }
      return true;
    });
    if (!rc && index_obj && n_members == 1) {
      rc = sr_members(x, ob, oe, 4, &bad, [&](long long nb, long long ne, const SrVal &v) {
        if (sr_is(b, nb, ne, "_id", 3)) {
          id_str = id_str && v.kind == kVString;
          if (!n_id++) {
            idb = v.b;
            ide = v.e;
          }
        } else if (sr_is(b, nb, ne, "status", 6)) {
          if (!n_status++) status_ok = v.kind == kVScalar && sr_integer(b, v.b, v.e, -2147483648LL, 2147483647LL, &st);
        } else if (sr_is(b, nb, ne, "error", 5) && !seen_error) {
          seen_error = true;
          if (v.kind != kVObject) return true;
          long long bad2 = 0;
          const int rc2 = sr_members(x, v.ob, v.oe, 5, &bad2, [&](long long nb2, long long ne2, const SrVal &w) {
            if (sr_is(b, nb2, ne2, "type", 4) && !seen_type) {
              seen_type = true;
              if (w.kind == kVString) {
                tb = w.b;
                te = w.e;
              }
            } else if (sr_is(b, nb2, ne2, "reason", 6) && !seen_reason) {
              seen_reason = true;
              if (w.kind == kVString) {
                rb = w.b;
                re = w.e;
              }
            }
            return true;
          });
          if (rc2 && !nested) {   // reported after the walk: the callback cannot end it with an error
            nested = rc2;
            nbad = bad2;
          }
        }
        return true;
      });
    }
    if (!rc && nested) {
      rc = nested;
      bad = nbad;
    }
    int code = 0;
    if (!rc) {
      const long long i0 = it.id_off[doc], i1 = it.id_off[doc + 1];
      code = !index_obj || n_members != 1 ? kIwNotIndex
             : !n_id || !id_str          ? kIwNoId
             : n_id > 1                  ? kSrRepeatedId
             : !n_status                 ? kIwNoStatus
             : n_status > 1              ? kIwRepeatedStatus
             : !status_ok                ? kIwBadStatus
             : !sr_name_is(b, idb, ide, it.id + i0, (int)(i1 - i0)) ? kIwIdMismatch
                                                                     : 0;
    }
    if (lane == 0) {
      if (rc) sr_fail(byte_err, bad, rc);
      if (code) sr_fail(err, i, code);
      if (!rc && !code) {
        status[doc] = (int32_t)st;
        if (st < 200 || st >= 300) {
          const unsigned long long k = atomicAdd(n_fail, 1ULL);
          fail[k] = IwFail{i, tb, te, rb, re};
        }
      }
    }
  }
}

}  // namespace cco
