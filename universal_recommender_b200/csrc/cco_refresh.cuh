// cco_refresh.cuh -- item properties refreshed in the live model index (cco_refresh_properties), on the device.
//
// An old document keeps what only a train or a calcPop computes -- its correlator members and its computed ranking
// members, verbatim -- and takes the item's fresh properties in place of its old ones:
//   {"id":x, <correlator members>, <fresh properties>, <computed ranking members>}
// include/cco_b200.h states the rule.  The old index is parsed by cco_json.cuh (bulk_parse, k_member_info), the fresh
// properties are sorted by cco_format.cuh (model_fields), and the items without an old document are written by k_doc_write.
//   k_refresh_len / k_refresh_write   the rewritten old documents (0 bytes: deleted), one warp per document as k_rerank_write
//   k_refresh_diff                    one warp per document: is the rewritten source line the old one, byte for byte
//   k_refresh_lists                   the changed and new documents, the changed and the deleted ones, compacted
//   k_refresh_del_len / _write        the delete body, {"delete":{"_id":"<escaped id>"}} per deleted document
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace cco {

// the class of a member name: what the refresh does with an old member of that name
enum : uint8_t { kRefreshOther = 0, kRefreshCorrelator = 1, kRefreshRanking = 2 };

struct RefreshArgs {
  const long long *line_moff;   // [2 n_docs + 1]: line l's members are [line_moff[l], line_moff[l + 1])
  const JMember *mem;
  const int32_t *ment;          // table entry of each member's name, -1
  const uint8_t *mkeep;         // not "id", not followed by a member of the same name
  const uint8_t *ent_cls;       // per table entry: kRefresh*
  const unsigned char *body;
  const long long *line_b;      // [2 n_docs]: the first byte of each line
  long long body_len;
};
__device__ __forceinline__ int refresh_member_cls(const RefreshArgs &r, long long m) {
  return r.mkeep[m] && r.ment[m] >= 0 ? r.ent_cls[r.ment[m]] : kRefreshOther;
}
__device__ __forceinline__ bool refresh_has_props(const FormatArgs &a, int g) { return a.pbeg && a.pend[g] > a.pbeg[g]; }

// doc_len[d] = the bytes of old document d rewritten, 0 when it is deleted (no property state, no member besides "id")
__global__ void k_refresh_len(const FormatArgs a, const RefreshArgs r, int32_t n_docs, long long *__restrict__ doc_len) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int d = warp; d < n_docs; d += nwarps) {
    const DocRef x = doc_ref(a, d);
    const long long m0 = r.line_moff[2 * (long long)d + 1], m1 = r.line_moff[2 * (long long)d + 2];
    long long len = 0, n = 0;
    for (long long m = m0 + lane; m < m1; m += 32) {
      if (refresh_member_cls(r, m) == kRefreshOther) continue;
      len += (r.mem[m].ne - r.mem[m].nb) + 4 + (r.mem[m].ve - r.mem[m].vb);
      ++n;
    }
    if (a.pbeg) {
      for (int j = a.pbeg[x.g] + lane; j < a.pend[x.g]; j += 32) {
        if (!prop_last(a, x.g, j) || !prop_written(a, j, 0u)) continue;
        const uint32_t f = (uint32_t)a.pkey[j];
        const int t = a.ptri[j];
        len += (a.field_off[f + 1] - a.field_off[f]) + 4 + (a.val_off[t + 1] - a.val_off[t]);
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      len += __shfl_xor_sync(0xffffffffu, len, o);
      n += __shfl_xor_sync(0xffffffffu, n, o);
    }
    if (lane == 0) doc_len[d] = n == 0 && !refresh_has_props(a, x.g) ? 0 : 17 + x.idl + 11 + x.idl + 1 + 2 + len;
  }
}

__device__ __forceinline__ unsigned char *refresh_members(const RefreshArgs &r, long long m0, long long m1, int cls, unsigned char *w,
                                                          int lane) {
  for (long long m = m0; m < m1; ++m) {
    if (refresh_member_cls(r, m) != cls) continue;
    const JMember jm = r.mem[m];
    warp_lit(w, ",\"", 2, lane); w += 2;
    warp_copy(w, r.body + jm.nb, jm.ne - jm.nb, lane); w += jm.ne - jm.nb;
    warp_lit(w, "\":", 2, lane); w += 2;
    warp_copy(w, r.body + jm.vb, jm.ve - jm.vb, lane); w += jm.ve - jm.vb;
  }
  return w;
}

// one warp per kept document: "id", the correlator members, the fresh properties (cco_format.cuh's rules), the ranking members
__global__ void k_refresh_write(const FormatArgs a, const RefreshArgs r, int32_t n_docs, const long long *__restrict__ doc_off,
                                unsigned char *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int d = warp; d < n_docs; d += nwarps) {
    if (doc_off[d + 1] == doc_off[d]) continue;   // deleted
    const DocRef x = doc_ref(a, d);
    const long long m0 = r.line_moff[2 * (long long)d + 1], m1 = r.line_moff[2 * (long long)d + 2];
    unsigned char *w = out + doc_off[d];
    warp_lit(w, "{\"index\":{\"_id\":\"", 17, lane); w += 17;
    warp_copy(w, x.id, x.idl, lane); w += x.idl;
    warp_lit(w, "\"}}\n{\"id\":\"", 11, lane); w += 11;
    warp_copy(w, x.id, x.idl, lane); w += x.idl;
    warp_lit(w, "\"", 1, lane); w += 1;
    w = refresh_members(r, m0, m1, kRefreshCorrelator, w, lane);
    if (a.pbeg) {
      for (int j = a.pbeg[x.g]; j < a.pend[x.g]; ++j) {
        if (!prop_last(a, x.g, j) || !prop_written(a, j, 0u)) continue;
        const uint32_t f = (uint32_t)a.pkey[j];
        const int t = a.ptri[j];
        const long long nl = a.field_off[f + 1] - a.field_off[f], vl = a.val_off[t + 1] - a.val_off[t];
        warp_lit(w, ",\"", 2, lane); w += 2;
        warp_copy(w, a.names + a.field_off[f], nl, lane); w += nl;
        warp_lit(w, "\":", 2, lane); w += 2;
        warp_copy(w, a.vals + (a.val_off[t] - a.val_base), vl, lane); w += vl;
      }
    }
    w = refresh_members(r, m0, m1, kRefreshRanking, w, lane);
    warp_lit(w, "}\n", 2, lane);
    __syncwarp();
  }
}

// flag[d] = 1 for a document of the delta: an old one whose rewritten source line differs from its old source line, and
// every new one (d >= n_old); del[d] = 1 for a deleted old document.  One warp per document.
__global__ void k_refresh_diff(const FormatArgs a, const RefreshArgs r, int32_t n_old, int32_t n_docs, const long long *__restrict__ doc_off,
                               const unsigned char *__restrict__ out, uint32_t *__restrict__ flag, uint32_t *__restrict__ del) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int d = warp; d < n_docs; d += nwarps) {
    if (d >= n_old) {
      if (lane == 0) flag[d] = 1;
      continue;
    }
    const bool gone = doc_off[d + 1] == doc_off[d];
    bool differ = false;
    if (!gone) {
      const long long idl = a.row_ids.off[d + 1] - a.row_ids.off[d];
      const long long nb = doc_off[d] + 17 + idl + 4, ne = doc_off[d + 1] - 1;   // the new source line, without its '\n'
      const long long ob = r.line_b[2 * (long long)d + 1];
      const long long oe = (2 * (long long)d + 2 < 2 * (long long)n_old ? r.line_b[2 * (long long)d + 2] : r.body_len) - 1;
      const long long n = ne - nb;
      differ = n != oe - ob;
      for (long long k0 = 0; !differ && k0 < n; k0 += 32) {   // uniform over the warp
        const long long k = k0 + lane;
        differ = __any_sync(0xffffffffu, k < n && out[nb + k] != r.body[ob + k]);
      }
    }
    if (lane == 0) {
      flag[d] = differ ? 1u : 0u;
      del[d] = gone ? 1u : 0u;
    }
  }
}

// the compacted lists: pick[k] = the k-th delta document and se[d] = the last byte of document d before its final '\n'
// (k_line_gather's spans over the refreshed body); changed[k] / deleted[k] = the old numbers of the changed / deleted ones
__global__ void k_refresh_lists(int32_t n_old, int32_t n_docs, const uint32_t *__restrict__ flag, const uint32_t *__restrict__ fpos,
                                const uint32_t *__restrict__ del, const uint32_t *__restrict__ dpos, const long long *__restrict__ doc_off,
                                uint32_t *__restrict__ pick, long long *__restrict__ se, int64_t *__restrict__ changed,
                                int64_t *__restrict__ deleted) {
  for (int d = blockIdx.x * blockDim.x + threadIdx.x; d < n_docs; d += gridDim.x * blockDim.x) {
    se[d] = doc_off[d + 1] - 1;
    if (flag[d]) {
      pick[fpos[d]] = (uint32_t)d;
      if (d < n_old) changed[fpos[d]] = d;
    }
    if (d < n_old && del[d]) deleted[dpos[d]] = d;
  }
}

// {"delete":{"_id":"  = 18 bytes, the escaped id, "}}\n = 4
__global__ void k_refresh_del_len(long long n, const int64_t *__restrict__ deleted, const DevDict ids, long long *__restrict__ len) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    len[i] = 18 + (ids.off[deleted[i] + 1] - ids.off[deleted[i]]) + 4;
}
__global__ void k_refresh_del_write(long long n, const int64_t *__restrict__ deleted, const DevDict ids, const long long *__restrict__ off,
                                    unsigned char *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5, nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long i = warp; i < n; i += nwarps) {
    const long long q = deleted[i], idl = ids.off[q + 1] - ids.off[q];
    unsigned char *w = out + off[i];
    warp_lit(w, "{\"delete\":{\"_id\":\"", 18, lane); w += 18;
    warp_copy(w, ids.bytes + ids.off[q], idl, lane); w += idl;
    warp_lit(w, "\"}}\n", 4, lane);
  }
}

}  // namespace cco
