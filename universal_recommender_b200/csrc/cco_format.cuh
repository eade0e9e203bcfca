// cco_format.cuh -- SURVEY.md 8f-2: the indicator model as the Elasticsearch bulk body, assembled on the device.
//
// Reference (what this replaces, per item of the primary event):
//   IndexedDatasetConversions.toStringMapRDD   src/main/scala/package.scala:82-110
//       row -> non-zeros sorted by -LLR -> column id STRINGS (the LLR values are dropped); empty rows give an empty JArray
//   URModel.save: groupAll + ("id" -> itemId)    src/main/scala/URModel.scala:47-84, 87-102
//   EsClient.hotSwap: saveToEs(.., "es.mapping.id" -> "id")   src/main/scala/EsClient.scala:300-313
// One document per primary item, one keyword-array field per event name.  As elasticsearch-hadoop sends it:
//   {"index":{"_id":"<item>"}}\n
//   {"id":"<item>","<event 0>":["<col>","<col>",...],"<event 1>":[...]}\n
// The indicator rows arrive already ordered (llr desc, col asc), so the consumer's sortBy(-llr) is a no-op and the
// formatter only concatenates: dictionary strings are JSON-escaped once, then every document is a gather of byte ranges.
// HBM-bound byte work: two passes (lengths -> exclusive scan -> bytes), one warp per document.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace cco {

struct DevDict {            // id i = bytes[off[i] .. off[i + 1])
  const long long *off;
  const unsigned char *bytes;
  long long n;
};

// JSON string escaping (RFC 8259 minimum): '"' -> \" , '\\' -> \\\\ , bytes < 0x20 -> \u00xx (lower-case hex); everything
// else (UTF-8 included) passes through.  Same rule in the CPU restatement (oracle/format_oracle.py).
__device__ __forceinline__ int json_escaped_len(unsigned char ch) { return ch == '"' || ch == '\\' ? 2 : (ch < 0x20 ? 6 : 1); }

__global__ void k_escape_len(long long n, const long long *__restrict__ off, const unsigned char *__restrict__ bytes,
                             long long *__restrict__ out_len) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    long long len = 0;
    for (long long q = off[i]; q < off[i + 1]; ++q) len += json_escaped_len(bytes[q]);
    out_len[i] = len;
  }
}
__global__ void k_escape_write(long long n, const long long *__restrict__ off, const unsigned char *__restrict__ bytes,
                               const long long *__restrict__ out_off, unsigned char *__restrict__ out) {
  const char hex[] = "0123456789abcdef";
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    long long w = out_off[i];
    for (long long q = off[i]; q < off[i + 1]; ++q) {
      const unsigned char ch = bytes[q];
      if (ch == '"' || ch == '\\') {
        out[w++] = '\\';
        out[w++] = ch;
      } else if (ch < 0x20) {
        out[w++] = '\\'; out[w++] = 'u'; out[w++] = '0'; out[w++] = '0';
        out[w++] = hex[ch >> 4];
        out[w++] = hex[ch & 15];
      } else {
        out[w++] = ch;
      }
    }
  }
}

constexpr int kMaxFormatIndicators = 16;
constexpr int kMaxRankings = 8;
constexpr uint16_t kClashId = 0x100;   // the field is named "id": the document's own "id" wins over it
struct FormatArgs {
  int32_t n_rows;          // row documents = rows [0, n_rows) of every indicator (a rank's slice or the whole model)
  long long row_id_base;   // global item index of row 0 (the row dictionary is global)
  int32_t n_ind;
  DevDict row_ids;                              // escaped
  DevDict col_ids[kMaxFormatIndicators];        // escaped
  const long long *row_ptr[kMaxFormatIndicators];
  const int32_t *col[kMaxFormatIndicators];
  const unsigned char *names;                   // escaped event names, then field names, then ranking names, concatenated
  int32_t name_off[kMaxFormatIndicators + 1];
  // ---- the complete model (cco_format_model); row_group == nullptr: indicator fields only (cco_format_es_bulk) ----
  // Items are grouped by id string over the row dictionary, the property items and the ranking streams (str_group).
  int32_t n_extra;                              // documents after the rows: items without a row, by first appearance
  const int32_t *row_group;                     // [n_rows] item group of each row document
  const int32_t *extra_group;                   // [n_extra]
  DevDict extra_ids;                            // escaped ids of the extra documents
  int32_t ind_field[kMaxFormatIndicators];      // property field named like indicator i, -1
  uint8_t ind_rank[kMaxFormatIndicators];       // rankings named like indicator i (bit k)
  const long long *field_off;                   // names[field_off[f] .. field_off[f + 1]) = escaped field name f
  const uint16_t *field_clash;                  // [n_fields] bits 0-7: rankings of the same name; kClashId
  const unsigned long long *pkey;               // property triples sorted by (group << 32 | field), triple index within
  const int32_t *ptri;                          // triple index of each sorted entry
  const int32_t *pbeg, *pend;                   // [groups] each group's entries in pkey / ptri
  const long long *val_off;                     // [triples + 1] the caller's value offsets; value t = vals[val_off[t] - val_base ..]
  long long val_base;
  const unsigned char *vals;
  int32_t n_rank;
  long long n_groups;
  const long long *score;                       // [n_rank][n_groups]
  const unsigned char *pmask;                   // [n_groups] bit k: ranking k scores the group
  int32_t rank_name_off[kMaxRankings + 1];      // into names
  uint16_t rank_clash[kMaxRankings];            // bits: LATER rankings of the same name (they win); kClashId
  uint8_t rank_scale[kMaxRankings];             // ranking k's value is score · 10^-rank_scale[k]: 0, or 15 (random)
};

// Java's Double.toString of v · 10^-scale, for scale 0 (an integer-valued double, |v| < 2^53) or scale 15 (0 <= v < 10^15).
// Both values have at most 16 significant digits, which are their shortest round-trip digits (the decimal is the nearest
// double's shortest text), so the text is built from v alone: plain d.ddd with at least one fraction digit for
// 10^-3 <= |x| < 10^7, else computerised scientific notation d.ddd"E"n; trailing zeros of the digits are dropped
// (0.0, 12.0, 1.0E7, 1.2345678E7, 0.001, 0.12, 9.99E-4, 1.0E-15).  Returns the length (<= 25).
__device__ __forceinline__ int java_double_text(long long v, int scale, unsigned char *out) {
  unsigned long long u = v < 0 ? 0ULL - (unsigned long long)v : (unsigned long long)v;
  unsigned char d[20];
  int n = 0;
  do {
    d[n++] = (unsigned char)('0' + u % 10);
    u /= 10;
  } while (u);   // d[n - 1] is the leading digit
  const int e = v == 0 ? 0 : n - 1 - scale;   // decimal exponent of the leading digit
  int low = 0;   // trailing zeros after the leading digit
  while (low < n - 1 && d[low] == '0') ++low;
  int p = 0;
  if (v < 0) out[p++] = '-';
  if (e >= 0 && e < 7) {          // integer digits "." fraction digits (at least one)
    int k = n - 1;
    for (; k >= n - 1 - e; --k) out[p++] = d[k];
    out[p++] = '.';
    if (k < low) out[p++] = '0';
    for (; k >= low; --k) out[p++] = d[k];
    return p;
  }
  if (e < 0 && e >= -3) {         // "0." zeros digits
    out[p++] = '0';
    out[p++] = '.';
    for (int z = -1; z > e; --z) out[p++] = '0';
    for (int k = n - 1; k >= low; --k) out[p++] = d[k];
    return p;
  }
  out[p++] = d[n - 1];
  out[p++] = '.';
  if (low == n - 1) out[p++] = '0';
  for (int k = n - 2; k >= low; --k) out[p++] = d[k];
  out[p++] = 'E';
  if (e < 0) out[p++] = '-';
  const int ae = e < 0 ? -e : e;   // 7 .. 15 or 4 .. 15
  if (ae >= 10) out[p++] = (unsigned char)('0' + ae / 10);
  out[p++] = (unsigned char)('0' + ae % 10);
  return p;
}

// one document: a row of the slice (r >= 0) or an item without a row (r = -1); g = item group, -1 without one
struct DocRef {
  const unsigned char *id;
  long long idl;
  int r, g;
};
__device__ __forceinline__ DocRef doc_ref(const FormatArgs &a, int d) {
  DocRef x;
  if (d < a.n_rows) {
    const long long q = a.row_id_base + d;
    x.id = a.row_ids.bytes + a.row_ids.off[q];
    x.idl = a.row_ids.off[q + 1] - a.row_ids.off[q];
    x.r = d;
    x.g = a.row_group ? a.row_group[d] : -1;
  } else {
    const int e = d - a.n_rows;
    x.id = a.extra_ids.bytes + a.extra_ids.off[e];
    x.idl = a.extra_ids.off[e + 1] - a.extra_ids.off[e];
    x.r = -1;
    x.g = a.extra_group[e];
  }
  return x;
}
__device__ __forceinline__ unsigned doc_rank_mask(const FormatArgs &a, int g) { return g >= 0 && a.pmask ? a.pmask[g] : 0u; }
// sorted property entry j of group g is the last of its (group, field) run: the triple that wins
__device__ __forceinline__ bool prop_last(const FormatArgs &a, int g, int j) { return j + 1 >= a.pend[g] || a.pkey[j + 1] != a.pkey[j]; }
__device__ __forceinline__ bool prop_written(const FormatArgs &a, int j, unsigned mask) {
  const uint16_t c = a.field_clash[(uint32_t)a.pkey[j]];
  return !(c & kClashId) && !(c & mask);
}
__device__ __forceinline__ bool ind_written(const FormatArgs &a, int i, int g, unsigned mask) {
  if (g < 0) return true;
  if (a.ind_rank[i] & mask) return false;
  const int f = a.ind_field[i];
  if (f >= 0 && a.pbeg)
    for (int j = a.pbeg[g]; j < a.pend[g]; ++j)
      if ((int)(uint32_t)a.pkey[j] == f) return false;
  return true;
}
__device__ __forceinline__ bool rank_written(const FormatArgs &a, int k, unsigned mask) {
  return ((mask >> k) & 1u) && !(a.rank_clash[k] & kClashId) && !(a.rank_clash[k] & mask);
}

// {"index":{"_id":"  = 17 bytes ; "}}\n{"id":"  = 11 ; closing quote of the id = 1 ; per field  ,"name":[  = name + 5 and ] = 1 ;
// per element two quotes + a comma between elements ; per property or rank  ,"name":  = name + 4, then the value ; }\n = 2
__global__ void k_doc_len(const FormatArgs a, int32_t n_docs, long long *__restrict__ doc_len) {
  for (int d = blockIdx.x * blockDim.x + threadIdx.x; d < n_docs; d += gridDim.x * blockDim.x) {
    const DocRef x = doc_ref(a, d);
    const unsigned mask = doc_rank_mask(a, x.g);
    long long len = 17 + x.idl + 11 + x.idl + 1 + 2;
    for (int i = 0; x.r >= 0 && i < a.n_ind; ++i) {
      if (!ind_written(a, i, x.g, mask)) continue;
      len += (a.name_off[i + 1] - a.name_off[i]) + 5 + 1;
      const long long s = a.row_ptr[i][x.r], e = a.row_ptr[i][x.r + 1];
      for (long long q = s; q < e; ++q) {
        const int32_t c = a.col[i][q];
        len += a.col_ids[i].off[c + 1] - a.col_ids[i].off[c] + 2;
      }
      if (e > s) len += e - s - 1;
    }
    if (x.g >= 0 && a.pbeg) {
      for (int j = a.pbeg[x.g]; j < a.pend[x.g]; ++j) {
        if (!prop_last(a, x.g, j) || !prop_written(a, j, mask)) continue;
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

__device__ __forceinline__ void warp_copy(unsigned char *dst, const unsigned char *src, long long n, int lane) {
  for (long long i = lane; i < n; i += 32) dst[i] = src[i];
}
__device__ __forceinline__ void warp_lit(unsigned char *dst, const char *lit, int n, int lane) {
  if (lane < n) dst[lane] = (unsigned char)lit[lane];
}

// one warp per document: the lanes copy every byte range cooperatively; the write position advances uniformly
__global__ void k_doc_write(const FormatArgs a, int32_t n_docs, const long long *__restrict__ doc_off, unsigned char *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int d = warp; d < n_docs; d += nwarps) {
    const DocRef x = doc_ref(a, d);
    const unsigned mask = doc_rank_mask(a, x.g);
    const int r = x.r;
    unsigned char *w = out + doc_off[d];
    warp_lit(w, "{\"index\":{\"_id\":\"", 17, lane); w += 17;
    warp_copy(w, x.id, x.idl, lane); w += x.idl;
    warp_lit(w, "\"}}\n{\"id\":\"", 11, lane); w += 11;
    warp_copy(w, x.id, x.idl, lane); w += x.idl;
    warp_lit(w, "\"", 1, lane); w += 1;
    for (int i = 0; r >= 0 && i < a.n_ind; ++i) {
      if (!ind_written(a, i, x.g, mask)) continue;
      const int nl = a.name_off[i + 1] - a.name_off[i];
      warp_lit(w, ",\"", 2, lane); w += 2;
      warp_copy(w, a.names + a.name_off[i], nl, lane); w += nl;
      warp_lit(w, "\":[", 3, lane); w += 3;
      const long long s = a.row_ptr[i][r], e = a.row_ptr[i][r + 1];
      // elements: the lanes first agree on every element's offset inside the array (prefix sums of 32 at a time)
      for (long long q0 = s; q0 < e; q0 += 32) {
        const long long q = q0 + lane;
        long long el = 0;
        const unsigned char *src = nullptr;
        if (q < e) {
          const int32_t c = a.col[i][q];
          src = a.col_ids[i].bytes + a.col_ids[i].off[c];
          el = a.col_ids[i].off[c + 1] - a.col_ids[i].off[c];
        }
        long long mine = q < e ? el + 2 + (q > s ? 1 : 0) : 0;   // leading comma from the second element on
        long long incl = mine;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const long long v = __shfl_up_sync(0xffffffffu, incl, d);
          if (lane >= d) incl += v;
        }
        const long long total = __shfl_sync(0xffffffffu, incl, 31);
        if (q < e) {
          unsigned char *p = w + (incl - mine);
          if (q > s) *p++ = ',';
          *p++ = '"';
          for (long long k = 0; k < el; ++k) p[k] = src[k];   // ids are short (a few to a few dozen bytes)
          p[el] = '"';
        }
        w += total;
      }
      warp_lit(w, "]", 1, lane); w += 1;
    }
    if (x.g >= 0 && a.pbeg) {   // properties in field order, the value spliced as given
      for (int j = a.pbeg[x.g]; j < a.pend[x.g]; ++j) {
        if (!prop_last(a, x.g, j) || !prop_written(a, j, mask)) continue;
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

// ---- the complete model (cco_format_model): item key space, properties, document set ---------------------------------
// rebase one uploaded offset column into the combined key column: dst[i] = src[i] + delta
__global__ void k_rebase(long long n, const long long *__restrict__ src, long long delta, long long *__restrict__ dst) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) dst[i] = src[i] + delta;
}
// property triples: bit 1 = a field index out of range, bit 2 = an empty value (decreasing offsets: k_str_check)
__global__ void k_prop_check(long long n, const int32_t *__restrict__ field, int32_t n_fields, const long long *__restrict__ val_off,
                             int *__restrict__ bad) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    if ((uint32_t)field[t] >= (uint32_t)n_fields) atomicOr(bad, 2);
    if (val_off[t + 1] == val_off[t]) atomicOr(bad, 4);
  }
}
// sort key (group << 32 | field) and value (triple index) of every triple; group = key-column group of its item id
__global__ void k_prop_keys(long long n, const int32_t *__restrict__ group, const int32_t *__restrict__ field,
                            unsigned long long *__restrict__ key, int32_t *__restrict__ tri) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    key[t] = ((unsigned long long)(uint32_t)group[t] << 32) | (uint32_t)field[t];
    tri[t] = (int32_t)t;
  }
}
// each group's range of sorted entries (pbeg = pend = 0 beforehand for groups without a property)
__global__ void k_prop_ranges(long long n, const unsigned long long *__restrict__ key, int32_t *__restrict__ pbeg, int32_t *__restrict__ pend) {
  for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j < n; j += (long long)gridDim.x * blockDim.x) {
    const uint32_t g = (uint32_t)(key[j] >> 32);
    if (j == 0 || (uint32_t)(key[j - 1] >> 32) != g) pbeg[g] = (int32_t)j;
    if (j == n - 1 || (uint32_t)(key[j + 1] >> 32) != g) pend[g] = (int32_t)(j + 1);
  }
}
__global__ void k_rank_mask(long long n_groups, const unsigned char *__restrict__ present, int k, unsigned char *__restrict__ pmask) {
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < n_groups; g += (long long)gridDim.x * blockDim.x)
    if (present[g]) pmask[g] |= (unsigned char)(1u << k);
}
// flag[g] = 1 iff group g has no row (first appearance past the row dictionary) and a property or a score
__global__ void k_extra_flags(long long n_groups, const uint32_t *__restrict__ first_sorted, long long n_row_ids,
                              const int32_t *__restrict__ pbeg, const int32_t *__restrict__ pend, const unsigned char *__restrict__ pmask,
                              uint32_t *__restrict__ flag) {
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < n_groups; g += (long long)gridDim.x * blockDim.x)
    flag[g] = (long long)first_sorted[g] >= n_row_ids && ((pbeg && pend[g] > pbeg[g]) || (pmask && pmask[g])) ? 1u : 0u;
}
__global__ void k_extra_compact(long long n_groups, const uint32_t *__restrict__ flag, const uint32_t *__restrict__ pos,
                                const uint32_t *__restrict__ first_sorted, int32_t *__restrict__ extra_group, uint32_t *__restrict__ extra_first) {
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < n_groups; g += (long long)gridDim.x * blockDim.x)
    if (flag[g]) {
      extra_group[pos[g]] = (int32_t)g;
      extra_first[pos[g]] = first_sorted[g];
    }
}

// ---- SURVEY.md 8f-3: PopModel rank histograms (src/main/scala/PopModel.scala:113-182) -----------------------
// popular  = events per item in [start, end)                                              (calcPopular :113-122)
// trending = newer half - older half, items present in BOTH halves; nothing if the older half is empty   (:128-148)
// hot      = (newer - middle) - (middle - older) over thirds, items present in all three buckets; nothing if the older or
//            the middle third is empty                                                                  (:153-182)
// Bucket edges follow the reference's Joda arithmetic: integer millisecond division, [start, end) intervals
// (PEventStore.find: startTime inclusive, untilTime exclusive).
// The key of an event is an item index (cco_pop_model) or the item's key-column group (cco_format_model).  Scores are
// integers: the model path keeps them as int64 for the exact Double.toString text, cco_pop_model returns doubles.
struct PopArgs {
  long long edge[4];   // bucket b = [edge[b], edge[b + 1])
  int n_buckets;
  int32_t n_items;     // keys
};
__global__ void k_pop_count(long long n_events, const int32_t *__restrict__ item, const long long *__restrict__ t_ms, const PopArgs a,
                            int32_t *__restrict__ counts /* [n_buckets][n_items] */, unsigned long long *__restrict__ totals) {
  unsigned long long mine[3] = {0, 0, 0};
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n_events; e += (long long)gridDim.x * blockDim.x) {
    const long long t = t_ms[e];
    const int32_t j = item[e];
    if ((uint32_t)j >= (uint32_t)a.n_items) continue;
#pragma unroll
    for (int b = 0; b < 3; ++b)
      if (b < a.n_buckets && t >= a.edge[b] && t < a.edge[b + 1]) {
        atomicAdd(&counts[(size_t)b * a.n_items + j], 1);
        ++mine[b];
      }
  }
  for (int b = 0; b < 3; ++b) {
    unsigned long long v = mine[b];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0 && v) atomicAdd(&totals[b], v);
  }
}
template <typename Score>
__global__ void k_pop_score(const PopArgs a, int mode, const int32_t *__restrict__ counts, const unsigned long long *__restrict__ totals,
                            Score *__restrict__ score, unsigned char *__restrict__ present) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < a.n_items; j += gridDim.x * blockDim.x) {
    const long long c0 = counts[j], c1 = a.n_buckets > 1 ? counts[(size_t)a.n_items + j] : 0,
                    c2 = a.n_buckets > 2 ? counts[(size_t)2 * a.n_items + j] : 0;
    long long v = 0;          // |v| < 2^33: exact as a double too
    bool ok = false;
    if (mode == 0) {          // popular
      ok = c0 > 0;
      v = c0;
    } else if (mode == 1) {   // trending: buckets = (older, newer)
      ok = totals[0] > 0 && c0 > 0 && c1 > 0;
      v = c1 - c0;
    } else {                  // hot: buckets = (older, middle, newer)
      ok = totals[0] > 0 && totals[1] > 0 && c0 > 0 && c1 > 0 && c2 > 0;
      v = (c2 - c1) - (c1 - c0);
    }
    score[j] = ok ? (Score)v : (Score)0;
    present[j] = ok ? 1 : 0;
  }
}

// ---- random (uniqueRank, PopModel.calcRandom, PopModel.scala:98-110), cco_format_model only --------------------------
// Items: the targets of every event in [start, end) -- the ranking's streams are every event name's -- plus every item with
// a property triple.  Value: n · 10^-15, uniform in [0, 1), from the id and the window only (the reference's unseeded
// Random.nextDouble cannot be reproduced; these values are):
//   h = k_str_hash of the id (mask ~0),  r = mix64(h ^ mix64(start ^ mix64(end))),  n = floor(r · 10^15 / 2^64).
// counts = the popular histogram of the window; the group's hash is the hash of its first id in the key column.
__global__ void k_random_score(long long n_groups, const int32_t *__restrict__ counts, const int32_t *__restrict__ pbeg,
                               const int32_t *__restrict__ pend, const uint32_t *__restrict__ first_sorted,
                               const uint64_t *__restrict__ hash, long long start_ms, long long end_ms, long long *__restrict__ score,
                               unsigned char *__restrict__ present) {
  const uint64_t window = mix64((uint64_t)start_ms ^ mix64((uint64_t)end_ms));
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < n_groups; g += (long long)gridDim.x * blockDim.x) {
    const bool ok = counts[g] > 0 || (pbeg && pend[g] > pbeg[g]);
    const uint64_t r = mix64(hash[first_sorted[g]] ^ window);
    score[g] = ok ? (long long)__umul64hi(r, 1000000000000000ULL) : 0;
    present[g] = ok ? 1 : 0;
  }
}

}  // namespace cco
