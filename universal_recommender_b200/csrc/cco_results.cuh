// cco_results.cuh -- Elasticsearch _msearch response bodies read on the device (cco_search_results_*): the second half of
// URAlgorithm.predict (URAlgorithm.scala:484-529), from the search hits to the PredictedResult text.
//
// A response body is one JSON value, often one multi-GB line, so the event reader's tokenizer (one warp per line) does not
// apply.  The body is read as simdjson does, in 64-byte words:
//   k_sr_chunk              per word: the masks of '\\' '"' '{' '[' '}' ']' ':' ','; the word's effect on the state
//                           (escape carry, in string) and on the depth, for each of the four in-states (SrFun); one warp
//                           composes the 32 words of a chunk
//   k_sr_scan               an inclusive scan of the chunk functions gives every chunk's in-state and in-depth
//   k_sr_index<kWrite>      count pass + write pass of the structural index: the unescaped quotes and the brackets, ':' and
//                           ',' outside strings at depth <= 7 (top '{' -> responses '[' -> response '{' -> hits '{' -> hits
//                           '[' -> hit '{' -> _source '{'), with their depth; what _source's arrays hold never enters it
//   k_sr_top                one warp walks the depth <= 1 entries: the top-level object and its "responses" array
//   k_sr_elems              the depth-2 entries of the responses array: every element an object, one record each
//   k_sr_resp<kWrite>       one warp per record over its index entries: error / status / hits.total / hits.hits
//   k_sr_hit                one warp per hit: _id, _score and, for withRanks records, the ranking members of _source
//   k_sr_hit_text<kWrite>   the PredictedResult text, one thread per hit (length pass + write pass), k_sr_rec_text the
//                           record frames
// Walks compare member names decoded and accept any member order; members they do not know are skipped by depth.
#include <cuda_runtime.h>
#include <stdint.h>

namespace cco {

constexpr int kSrMaxDepth = 7;
constexpr int kSrChunkWords = 32;   // one warp, one 64-byte word per lane

// error codes of the walks; an error word is min over failures of (key << 8 | code), the key a byte offset, a record or a hit
enum {
  kSrSyntax = 1,        // malformed JSON at a byte offset
  kSrString,            // a bad escape or a raw byte < 0x20 in a string the walk reads
  kSrUnbalanced,        // a closing bracket without an opening one, or a mismatched pair
  kSrNoResponses,       // the top level is not an object with one "responses" array
  kSrElement,           // a responses element that is not an object
  kSrStatus,            // a status that is not a 32-bit integer
  kSrHitsNotArray,      // hits.hits is not an array (nor null)
  kSrHitNotObject,      // a hits.hits element that is not an object
  kSrNoId,              // a hit without a string _id
  kSrRepeated,          // a repeated _id or _score
  kSrNoScore,           // a hit whose _score is missing, null or not a number
  kSrBadRank,           // a ranking member that is present but neither a number nor null
};
// codes every reader shares (line errors take 16 .. 19, index pages 32 .., index write 48 ..)
enum {
  kSrOpenString = 20,   // the body ends inside a string
  kSrNotObject,         // the top level is not an object (index pages, index write)
  kSrEsError,           // a top-level "error" member (index pages, index write)
  kSrRepeatedId,        // a hit or item with two _id members (index pages, index write)
};

__device__ __forceinline__ void sr_fail(unsigned long long *w, long long key, int code) {
  atomicMin(w, ((unsigned long long)key << 8) | (unsigned)code);
}

// ---- structural index ----------------------------------------------------------------------------------------------
// state s = escape carry (bit 0: the word starts right after an odd run of backslashes) | in string (bit 1)
struct SrFun {
  unsigned char f[4];   // out-state of each in-state
  int d[4];             // depth change over the word for each in-state
};
__device__ __host__ __forceinline__ SrFun sr_identity() {
  SrFun r;
  for (int s = 0; s < 4; ++s) {
    r.f[s] = (unsigned char)s;
    r.d[s] = 0;
  }
  return r;
}
struct SrCompose {   // a then b
  __host__ __device__ __forceinline__ SrFun operator()(const SrFun &a, const SrFun &b) const {
    SrFun r;
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      r.f[s] = b.f[a.f[s]];
      r.d[s] = a.d[s] + b.d[a.f[s]];
    }
    return r;
  }
};

__device__ __forceinline__ uint64_t sr_bits4(unsigned m) { return (((m & 0x01010101u) * 0x01020408u) >> 24) & 0xfu; }
struct SrMasks {
  uint64_t bs, q, op, cl, sep;
};
// the word's masks; the body is padded with spaces to whole words
__device__ __forceinline__ SrMasks sr_masks(const uint4 *__restrict__ w) {
  SrMasks m = {0, 0, 0, 0, 0};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const uint4 v = w[k];
    const unsigned u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const unsigned x = u[j];
      const int sh = (k * 4 + j) * 4;
      m.bs |= sr_bits4(__vcmpeq4(x, 0x5c5c5c5cu)) << sh;
      m.q |= sr_bits4(__vcmpeq4(x, 0x22222222u)) << sh;
      m.op |= sr_bits4(__vcmpeq4(x, 0x7b7b7b7bu) | __vcmpeq4(x, 0x5b5b5b5bu)) << sh;
      m.cl |= sr_bits4(__vcmpeq4(x, 0x7d7d7d7du) | __vcmpeq4(x, 0x5d5d5d5du)) << sh;
      m.sep |= sr_bits4(__vcmpeq4(x, 0x3a3a3a3au) | __vcmpeq4(x, 0x2c2c2c2cu)) << sh;
    }
  }
  return m;
}
// escaped bytes of the word (preceded by an odd run of backslashes) for escape carry c; *cout: the carry out
__device__ __forceinline__ uint64_t sr_escaped(uint64_t bs, int c, int *cout) {
  if (!bs) {
    *cout = 0;
    return (uint64_t)c;
  }
  uint64_t esc = 0;
  int e = c;
  for (int i = 0; i < 64; ++i) {
    const uint64_t bit = 1ULL << i;
    if (e) {
      esc |= bit;
      e = 0;
    } else if (bs & bit) {
      e = 1;
    }
  }
  *cout = e;
  return esc;
}
__device__ __forceinline__ uint64_t sr_prefix_xor(uint64_t x) {
  x ^= x << 1;
  x ^= x << 2;
  x ^= x << 4;
  x ^= x << 8;
  x ^= x << 16;
  x ^= x << 32;
  return x;
}
// one word under both escape carries: its unescaped quotes uq[c], in-string bits from outside ins[c] (the opening quote
// in, the closing quote out), and its function
struct SrWord {
  SrMasks m;
  uint64_t uq[2], ins[2];
  SrFun F;
};
__device__ __forceinline__ void sr_word(const uint4 *__restrict__ w, SrWord &o) {
  o.m = sr_masks(w);
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    int co;
    const uint64_t esc = sr_escaped(o.m.bs, c, &co);
    o.uq[c] = o.m.q & ~esc;
    o.ins[c] = sr_prefix_xor(o.uq[c]);
    const int par = __popcll(o.uq[c]) & 1;
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      const uint64_t out = s ? o.ins[c] : ~o.ins[c];
      o.F.f[c | s << 1] = (unsigned char)(co | ((s ^ par) << 1));
      o.F.d[c | s << 1] = __popcll(o.m.op & out) - __popcll(o.m.cl & out);
    }
  }
}
__device__ __forceinline__ SrFun sr_shfl_up(const SrFun &a, int k) {
  SrFun r;
  unsigned packed = a.f[0] | a.f[1] << 8 | a.f[2] << 16 | (unsigned)a.f[3] << 24;
  packed = __shfl_up_sync(0xffffffffu, packed, k);
  for (int s = 0; s < 4; ++s) {
    r.f[s] = (unsigned char)(packed >> (8 * s));
    r.d[s] = __shfl_up_sync(0xffffffffu, a.d[s], k);
  }
  return r;
}
// inclusive warp scan of the lanes' functions (lane order = byte order)
__device__ __forceinline__ SrFun sr_warp_scan(SrFun x, int lane) {
#pragma unroll
  for (int k = 1; k < 32; k <<= 1) {
    const SrFun y = sr_shfl_up(x, k);
    if (lane >= k) x = SrCompose()(y, x);
  }
  return x;
}

__global__ void k_sr_chunk(long long n_words, const uint4 *__restrict__ body, SrFun *__restrict__ fun) {
  const int lane = threadIdx.x & 31;
  const long long n_chunks = (n_words + kSrChunkWords - 1) / kSrChunkWords;
  for (long long ch = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; ch < n_chunks; ch += ((long long)gridDim.x * blockDim.x) >> 5) {
    const long long wi = ch * kSrChunkWords + lane;
    SrFun F = sr_identity();
    if (wi < n_words) {
      SrWord o;
      sr_word(body + wi * 4, o);
      F = o.F;
    }
    F = sr_warp_scan(F, lane);
    if (lane == 31) fun[ch] = F;
  }
}

// inclusive scan of the chunk functions, one block of kSrScanThreads: each thread composes a contiguous run of chunks,
// thread 0 scans the runs' totals, then every thread rewrites its run with its prefix
constexpr int kSrScanThreads = 1024;
__global__ void __launch_bounds__(kSrScanThreads) k_sr_scan(long long n, const SrFun *__restrict__ in, SrFun *__restrict__ out) {
  __shared__ SrFun part[kSrScanThreads];
  const int t = threadIdx.x;
  const long long per = (n + kSrScanThreads - 1) / kSrScanThreads, lo = t * per, hi = lo + per < n ? lo + per : n;
  SrFun acc = sr_identity();
  for (long long i = lo; i < hi; ++i) acc = SrCompose()(acc, in[i]);
  part[t] = acc;
  __syncthreads();
  if (t == 0) {
    SrFun run = sr_identity();
    for (int k = 0; k < kSrScanThreads; ++k) {
      const SrFun x = part[k];
      part[k] = run;
      run = SrCompose()(run, x);
    }
  }
  __syncthreads();
  acc = part[t];
  for (long long i = lo; i < hi; ++i) {
    acc = SrCompose()(acc, in[i]);
    out[i] = acc;
  }
}

// count pass (cnt[chunk]) and write pass (pos / dep from coff[chunk]) of the entries at depth <= max_depth (kSrMaxDepth
// for an _msearch body); pre = inclusive scan of the chunk functions.
// A closing bracket with nothing open sets err (byte offset, kSrUnbalanced).
template <bool kWrite>
__global__ void k_sr_index(long long n_words, const uint4 *__restrict__ body, const SrFun *__restrict__ pre, int max_depth, long long *__restrict__ cnt,
                           const long long *__restrict__ coff, long long *__restrict__ pos, unsigned char *__restrict__ dep,
                           unsigned long long *__restrict__ err) {
  const int lane = threadIdx.x & 31;
  const long long n_chunks = (n_words + kSrChunkWords - 1) / kSrChunkWords;
  for (long long ch = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; ch < n_chunks; ch += ((long long)gridDim.x * blockDim.x) >> 5) {
    const long long wi = ch * kSrChunkWords + lane;
    const int st0 = ch ? pre[ch - 1].f[0] : 0;
    const int d0 = ch ? pre[ch - 1].d[0] : 0;
    SrWord o;
    SrFun F = sr_identity();
    if (wi < n_words) {
      sr_word(body + wi * 4, o);
      F = o.F;
    }
    const SrFun inc = sr_warp_scan(F, lane);
    SrFun exc = sr_shfl_up(inc, 1);
    if (lane == 0) exc = sr_identity();
    const int st = exc.f[st0];
    int d = d0 + exc.d[st0];
    long long n = 0, at = 0;
    uint64_t S = 0;
    const int c = st & 1;
    uint64_t ins = 0;
    if (wi < n_words) {
      ins = (st >> 1) ? ~o.ins[c] : o.ins[c];
      S = ((o.m.op | o.m.cl | o.m.sep) & ~ins) | o.uq[c];
    }
    if (kWrite) {   // this lane's first slot: the warp's exclusive sum of the lane counts, recounted
      uint64_t s2 = S;
      int dd = d;
      long long k = 0;
      while (s2) {
        const int i = __ffsll((long long)s2) - 1;
        s2 &= s2 - 1;
        const uint64_t bit = 1ULL << i;
        if (o.m.op & bit & ~ins) k += dd++ <= max_depth;
        else if (o.m.cl & bit & ~ins) k += --dd <= max_depth && dd >= 0;
        else k += dd <= max_depth;
      }
      long long x = k;
#pragma unroll
      for (int sft = 1; sft < 32; sft <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, x, sft);
        if (lane >= sft) x += y;
      }
      at = coff[ch] + x - k;
    }
    while (S) {
      const int i = __ffsll((long long)S) - 1;
      S &= S - 1;
      const uint64_t bit = 1ULL << i;
      const long long p = wi * 64 + i;
      int e;
      if (o.m.op & bit & ~ins) {
        e = d++;
      } else if (o.m.cl & bit & ~ins) {
        e = --d;
        if (d < 0) {
          if (!kWrite) sr_fail(err, p, kSrUnbalanced);
          continue;
        }
      } else {
        e = d;
      }
      if (e > max_depth) continue;
      if (kWrite) {
        pos[at] = p;
        dep[at] = (unsigned char)e;
        ++at;
      } else {
        ++n;
      }
    }
    if (!kWrite) {
#pragma unroll
      for (int sft = 16; sft > 0; sft >>= 1) n += __shfl_down_sync(0xffffffffu, n, sft);
      if (lane == 0) cnt[ch] = n;
    }
  }
}

// entries with lo_dep <= dep <= hi_dep and index in (lo, hi): flag[i] (for a compaction)
__global__ void k_sr_flag(long long m, const unsigned char *__restrict__ dep, int lo_dep, int hi_dep, long long lo, long long hi,
                          long long *__restrict__ flag) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < m; i += (long long)gridDim.x * blockDim.x)
    flag[i] = i > lo && i < hi && dep[i] >= lo_dep && dep[i] <= hi_dep;
}
__global__ void k_sr_compact(long long m, const long long *__restrict__ flag, const long long *__restrict__ off, long long *__restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < m; i += (long long)gridDim.x * blockDim.x)
    if (flag[i]) out[off[i]] = i;
}

// ---- walks -----------------------------------------------------------------------------------------------------------
struct SrIdx {
  const long long *pos;
  const unsigned char *dep;
  const unsigned char *body;
  const long long *src;   // nullable: walk a compacted list of entries
  __device__ __forceinline__ long long at(long long j) const { return src ? src[j] : j; }
};
__device__ __forceinline__ bool sr_ws(unsigned c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r'; }
__device__ __forceinline__ bool sr_gap_ws(const unsigned char *__restrict__ b, long long p, long long e) {
  for (; p < e; ++p)
    if (!sr_ws(b[p])) return false;
  return true;
}
// walk-order index of index entry e in the sorted entry list src[0 .. n)
__device__ __forceinline__ long long sr_walk_at(const long long *__restrict__ src, long long n, long long e) {
  long long lo = 0, hi = n - 1;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (src[mid] < e) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}
// the raw inside of a string: valid escapes, no raw byte < 0x20
__device__ __forceinline__ bool sr_string_ok(const unsigned char *__restrict__ b, long long p, long long e) {
  while (p < e) {
    const unsigned c = b[p];
    if (c < 0x20) return false;
    if (c != '\\') {
      ++p;
      continue;
    }
    const unsigned x = b[p + 1];
    if (x == 'u') {
      if (p + 6 > e) return false;
      for (int k = 2; k < 6; ++k) {
        const unsigned h = b[p + k];
        if (!(h - '0' < 10u || (h | 0x20) - 'a' < 6u)) return false;
      }
      p += 6;
    } else if (x == '"' || x == '\\' || x == '/' || x == 'b' || x == 'f' || x == 'n' || x == 'r' || x == 't') {
      p += 2;
    } else {
      return false;
    }
  }
  return true;
}
// the next code point of a valid raw string at *p, as UTF-8 into u (returns its length); surrogates as json_unescape does
__device__ __forceinline__ int sr_next_utf8(const unsigned char *__restrict__ b, long long *p, long long e, unsigned char *u) {
  const unsigned c = b[*p];
  if (c != '\\') {
    u[0] = (unsigned char)c;
    ++*p;
    return 1;
  }
  const unsigned x = b[*p + 1];
  if (x != 'u') {
    u[0] = (unsigned char)(x == 'b' ? 8 : x == 'f' ? 12 : x == 'n' ? 10 : x == 'r' ? 13 : x == 't' ? 9 : x);
    *p += 2;
    return 1;
  }
  unsigned cp = json_hex4(b + *p + 2);
  *p += 6;
  if (cp >= 0xd800 && cp < 0xdc00 && *p + 6 <= e && b[*p] == '\\' && b[*p + 1] == 'u') {
    const unsigned lo = json_hex4(b + *p + 2);
    if (lo >= 0xdc00 && lo < 0xe000) {
      cp = 0x10000 + ((cp - 0xd800) << 10) + (lo - 0xdc00);
      *p += 6;
    }
  }
  const int k = cp < 0x80 ? 1 : cp < 0x800 ? 2 : cp < 0x10000 ? 3 : 4;
  for (int j = k - 1; j > 0; --j) {
    u[j] = (unsigned char)(0x80 | (cp & 0x3f));
    cp >>= 6;
  }
  u[0] = (unsigned char)(k == 1 ? cp : (k == 2 ? 0xc0 : k == 3 ? 0xe0 : 0xf0) | cp);
  return k;
}
// the decoded raw string [p, e) equals the UTF-8 bytes lit[0 .. n)
__device__ __forceinline__ bool sr_name_is(const unsigned char *__restrict__ b, long long p, long long e, const unsigned char *lit, int n) {
  int i = 0;
  unsigned char u[4];
  while (p < e) {
    const int k = sr_next_utf8(b, &p, e, u);
    if (i + k > n) return false;
    for (int j = 0; j < k; ++j)
      if (u[j] != lit[i + j]) return false;
    i += k;
  }
  return i == n;
}
__device__ __forceinline__ bool sr_is(const unsigned char *b, long long p, long long e, const char *lit, int n) {
  return sr_name_is(b, p, e, (const unsigned char *)lit, n);
}

// a JSON number's text: the value for the exact fast path, and the shortest digits (value = dig * 10^e10, nd digits)
struct SrNum {
  double v;
  unsigned long long dig;
  int e10, nd;
  int neg, exact;   // exact: the host computes v, dig, e10 and nd from the text
};
// false when [p, e) is not a JSON number.  The exponent and the offset the mantissa's digits carry are summed in 64 bits;
// the exponent literal saturates at 2^59, beyond any digit offset, so a sum inside the fast path's window is exact, and a
// number outside it goes to the host, which reads the text itself.
__device__ __forceinline__ bool sr_number(const unsigned char *__restrict__ b, long long p, long long e, SrNum *o) {
  SrNum r = {0.0, 0ULL, 0, 0, 0, 0};
  long long e10 = 0;
  if (p < e && b[p] == '-') {
    r.neg = 1;
    ++p;
  }
  if (p >= e || b[p] - '0' >= 10u) return false;
  bool lost = false;
  auto digit = [&](unsigned d, bool frac) {
    if (r.dig == 0 && d == 0) {
      if (frac) --e10;
      return;
    }
    if (r.nd < 19) {
      r.dig = r.dig * 10 + d;
      ++r.nd;
      if (frac) --e10;
    } else {
      if (!frac) ++e10;
      if (d) lost = true;
    }
  };
  bool is_int = true;
  if (b[p] == '0') {
    ++p;
  } else {
    while (p < e && b[p] - '0' < 10u) digit(b[p++] - '0', false);
  }
  if (p < e && b[p] == '.') {
    is_int = false;
    ++p;
    if (p >= e || b[p] - '0' >= 10u) return false;
    while (p < e && b[p] - '0' < 10u) digit(b[p++] - '0', true);
  }
  if (p < e && (b[p] | 0x20) == 'e') {
    is_int = false;
    ++p;
    int sg = 1;
    if (p < e && (b[p] == '+' || b[p] == '-')) sg = b[p++] == '-' ? -1 : 1;
    if (p >= e || b[p] - '0' >= 10u) return false;
    long long x = 0;
    while (p < e && b[p] - '0' < 10u) {
      const unsigned d = b[p++] - '0';
      if (x < (1LL << 59)) x = x * 10 + d;   // x * 10 + 9 still fits
    }
    e10 += sg * x;
  }
  if (p != e) return false;
  if (r.dig == 0) {
    if (is_int) r.neg = 0;   // a JSON integer is a JInt: -0 is 0
    r.v = r.neg ? -0.0 : 0.0;
    *o = r;
    return true;
  }
  while (r.dig % 10 == 0) {
    r.dig /= 10;
    ++e10;
    --r.nd;
  }
  if (!lost && r.nd <= 15 && e10 >= -22 && e10 <= 22) {   // Clinger: both operands exact, one rounding
    r.e10 = (int)e10;
    const double p10[23] = {1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15,
                            1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};
    const double m = (double)r.dig;
    r.v = r.e10 >= 0 ? m * p10[r.e10] : m / p10[-r.e10];
    if (r.neg) r.v = -r.v;
  } else {
    r.exact = 1;
  }
  *o = r;
  return true;
}
// Java's Double.toString over the shortest digits (ur_model.java_double's layout); o == nullptr: the length only
__device__ __forceinline__ int sr_java_text(const SrNum &x, unsigned char *o) {
  unsigned char ds[20];
  int n = 0;
  for (unsigned long long u = x.dig; u; u /= 10) ds[n++] = (unsigned char)('0' + u % 10);   // ds[n - 1] leads
  int k = 0;
  auto put = [&](unsigned char ch) {
    if (o) o[k] = ch;
    ++k;
  };
  if (x.neg) put('-');
  if (n == 0) {
    put('0');
    put('.');
    put('0');
    return k;
  }
  const int point = n + x.e10;
  if (point >= -2 && point <= 7) {
    if (point <= 0) {
      put('0');
      put('.');
      for (int z = 0; z < -point; ++z) put('0');
      for (int i = n - 1; i >= 0; --i) put(ds[i]);
    } else if (point >= n) {
      for (int i = n - 1; i >= 0; --i) put(ds[i]);
      for (int z = 0; z < point - n; ++z) put('0');
      put('.');
      put('0');
    } else {
      for (int i = n - 1; i >= n - point; --i) put(ds[i]);
      put('.');
      for (int i = n - point - 1; i >= 0; --i) put(ds[i]);
    }
    return k;
  }
  put(ds[n - 1]);
  put('.');
  if (n == 1) put('0');
  for (int i = n - 2; i >= 0; --i) put(ds[i]);
  put('E');
  int ex = point - 1;
  if (ex < 0) {
    put('-');
    ex = -ex;
  }
  if (ex >= 100) put((unsigned char)('0' + ex / 100));
  if (ex >= 10) put((unsigned char)('0' + ex / 10 % 10));
  put((unsigned char)('0' + ex % 10));
  return k;
}
// a JSON integer that fits in [lo, hi]
__device__ __forceinline__ bool sr_integer(const unsigned char *__restrict__ b, long long p, long long e, long long lo, long long hi, long long *out) {
  const bool neg = p < e && b[p] == '-';
  if (neg) ++p;
  if (p >= e || (b[p] == '0' && p + 1 != e)) return false;
  // the magnitude may reach -lo (lo >= -2^63 + 1 is the callers' case, so it fits)
  const unsigned long long lim = neg ? (unsigned long long)(-lo) : (unsigned long long)hi;
  unsigned long long v = 0;
  for (; p < e; ++p) {
    const unsigned d = b[p] - '0';
    if (d >= 10u || v > (lim - d) / 10) return false;
    v = v * 10 + d;
  }
  *out = neg ? -(long long)v : (long long)v;
  return true;
}
__device__ __forceinline__ bool sr_scalar_ok(const unsigned char *__restrict__ b, long long p, long long e) {
  const long long n = e - p;
  if (n == 4 && b[p] == 't' && b[p + 1] == 'r' && b[p + 2] == 'u' && b[p + 3] == 'e') return true;
  if (n == 4 && b[p] == 'n' && b[p + 1] == 'u' && b[p + 2] == 'l' && b[p + 3] == 'l') return true;
  if (n == 5 && b[p] == 'f' && b[p + 1] == 'a' && b[p + 2] == 'l' && b[p + 3] == 's' && b[p + 4] == 'e') return true;
  SrNum x;
  return sr_number(b, p, e, &x);
}
__device__ __forceinline__ bool sr_is_null(const unsigned char *b, long long p, long long e) {
  return e - p == 4 && b[p] == 'n' && b[p + 1] == 'u' && b[p + 2] == 'l' && b[p + 3] == 'l';
}

enum { kVScalar = 0, kVString, kVObject, kVArray };
struct SrVal {
  int kind;
  long long b, e;     // scalar: the trimmed text; string: the raw inside
  long long ob, oe;   // object / array: the index entries of its brackets
};
// The members of the object whose brackets are entries lo and hi (in walk order), its members' syntax being the entries
// at depth `level` between them.  on(name_b, name_e, value) for every member in order; it returns false to stop.  All
// lanes of the warp run the walk in step.  -> 0, or an error code with *bad the byte offset.
template <class F>
__device__ int sr_members(const SrIdx &x, long long lo, long long hi, int level, long long *bad, F &&on) {
  const unsigned char *b = x.body;
  const int lane = threadIdx.x & 31;
  long long prev = x.pos[x.at(lo)] + 1;   // first byte after the last event
  long long nb = 0, ne = 0, ob = 0;
  int st = 0, kind = 0;
  for (long long base = lo + 1; base <= hi; base += 32) {
    const long long j = base + lane;
    const bool sig = j <= hi && (j == hi || x.dep[x.at(j)] == level);
    unsigned msk = __ballot_sync(0xffffffffu, sig);
    while (msk) {
      const long long jj = base + __ffs(msk) - 1;
      msk &= msk - 1;
      const long long e = x.at(jj), p = x.pos[e];
      const unsigned ch = b[p];
      if (jj == hi) {   // the closing bracket of the object
        if (ch != '}') return *bad = p, kSrUnbalanced;
        if (st == 3) {
          long long vb = prev, ve = p;
          while (vb < ve && sr_ws(b[vb])) ++vb;
          while (ve > vb && sr_ws(b[ve - 1])) --ve;
          if (vb == ve || !sr_scalar_ok(b, vb, ve)) return *bad = prev, kSrSyntax;
          on(nb, ne, SrVal{kVScalar, vb, ve, 0, 0});
          return 0;
        }
        if ((st != 0 && st != 7) || !sr_gap_ws(b, prev, p)) return *bad = prev, kSrSyntax;
        return 0;
      }
      bool ok = true;
      switch (st) {
        case 0:
        case 6:
          ok = ch == '"' && sr_gap_ws(b, prev, p);
          nb = p + 1;
          st = 1;
          break;
        case 1:
          ne = p;
          if (!sr_string_ok(b, nb, ne)) return *bad = nb, kSrString;
          st = 2;
          break;
        case 2:
          ok = ch == ':' && sr_gap_ws(b, prev, p);
          st = 3;
          break;
        case 3:
          if (ch == ',') {
            long long vb = prev, ve = p;
            while (vb < ve && sr_ws(b[vb])) ++vb;
            while (ve > vb && sr_ws(b[ve - 1])) --ve;
            if (vb == ve || !sr_scalar_ok(b, vb, ve)) return *bad = prev, kSrSyntax;
            if (!on(nb, ne, SrVal{kVScalar, vb, ve, 0, 0})) return 0;
            st = 6;
            break;
          }
          ok = sr_gap_ws(b, prev, p) && (ch == '"' || ch == '{' || ch == '[');
          ob = jj;
          kind = ch == '"' ? kVString : ch == '{' ? kVObject : kVArray;
          st = ch == '"' ? 4 : 5;
          break;
        case 4:
          if (!sr_string_ok(b, x.pos[x.at(ob)] + 1, p)) return *bad = x.pos[x.at(ob)] + 1, kSrString;
          if (!on(nb, ne, SrVal{kVString, x.pos[x.at(ob)] + 1, p, 0, 0})) return 0;
          st = 7;
          break;
        case 5:
          if (ch != (kind == kVObject ? '}' : ']')) return *bad = p, kSrUnbalanced;
          if (!on(nb, ne, SrVal{kind, 0, 0, x.at(ob), e})) return 0;
          st = 7;
          break;
        case 7:
          ok = ch == ',' && sr_gap_ws(b, prev, p);
          st = 6;
          break;
      }
      if (!ok) return *bad = p, kSrSyntax;
      prev = p + 1;
    }
  }
  return *bad = prev, kSrSyntax;   // not reached: hi is always an event
}
// The elements of the array whose brackets are index entries lo and hi, each an object: on(k, open, close) for element k.
// -> 0, or an error code (code_not_object for an element of another kind) with *bad the byte offset.
template <class F>
__device__ int sr_objects(const SrIdx &x, long long lo, long long hi, int level, int code_not_object, long long *bad, long long *n_out, F &&on) {
  const unsigned char *b = x.body;
  const int lane = threadIdx.x & 31;
  long long prev = x.pos[x.at(lo)] + 1, open = 0, n = 0;
  int st = 0;   // 0: start, 1: in an element, 2: after an element, 3: after ','
  for (long long base = lo + 1; base <= hi; base += 32) {
    const long long j = base + lane;
    const bool sig = j <= hi && (j == hi || x.dep[x.at(j)] == level);
    unsigned msk = __ballot_sync(0xffffffffu, sig);
    while (msk) {
      const long long jj = base + __ffs(msk) - 1;
      msk &= msk - 1;
      const long long e = x.at(jj), p = x.pos[e];
      const unsigned ch = b[p];
      if (jj == hi) {
        if (ch != ']') return *bad = p, kSrUnbalanced;
        if (!sr_gap_ws(b, prev, p)) return *bad = prev, code_not_object;
        if (st == 1 || st == 3) return *bad = p, kSrSyntax;
        *n_out = n;
        return 0;
      }
      if (st == 1) {
        if (ch != '}') return *bad = p, kSrUnbalanced;
        on(n, open, e);
        ++n;
        st = 2;
      } else if (st == 2) {
        if (!sr_gap_ws(b, prev, p)) return *bad = prev, code_not_object;
        if (ch != ',') return *bad = p, kSrSyntax;
        st = 3;
      } else {
        if (!sr_gap_ws(b, prev, p)) return *bad = prev, code_not_object;
        if (ch != '{') return *bad = p, ch == ',' ? kSrSyntax : code_not_object;
        open = e;
        st = 1;
      }
      prev = p + 1;
    }
  }
  return *bad = prev, kSrSyntax;
}

// ---- the top level ----------------------------------------------------------------------------------------------------
// One warp over the depth <= 1 entries (the list src[0 .. n)): the body is ws* '{' members '}' ws*, with one member named
// "responses" whose value is an array.  out[0..1] = its brackets' index entries.
__global__ void k_sr_top(SrIdx x, long long n, long long len, long long *__restrict__ out, unsigned long long *__restrict__ err) {
  if (threadIdx.x >= 32) return;
  const unsigned char *b = x.body;
  long long first = 0;
  while (first < len && sr_ws(b[first])) ++first;
  if (n < 2 || x.pos[x.at(0)] != first || b[first] != '{' || x.dep[x.at(0)] != 0) {
    if (threadIdx.x == 0) sr_fail(err, first, kSrNoResponses);
    return;
  }
  long long close = -1;   // the depth-0 entry after the opening one
  for (long long j = 1; j < n; ++j)
    if (x.dep[x.at(j)] == 0) {
      close = j;
      break;
    }
  if (close < 0 || !sr_gap_ws(b, x.pos[x.at(close)] + 1, len)) {
    if (threadIdx.x == 0) sr_fail(err, close < 0 ? len : x.pos[x.at(close)] + 1, kSrSyntax);
    return;
  }
  long long bad = 0, ra = -1, rb = -1;
  int found = 0;
  const int rc = sr_members(x, 0, close, 1, &bad, [&](long long nb, long long ne, const SrVal &v) {
    if (sr_is(b, nb, ne, "responses", 9)) {
      ++found;
      if (v.kind == kVArray) {
        ra = v.ob;
        rb = v.oe;
      }
    }
    return true;
  });
  if (threadIdx.x != 0) return;
  if (rc) sr_fail(err, bad, rc);
  else if (found != 1 || ra < 0) sr_fail(err, first, kSrNoResponses);
  else {
    out[0] = ra;
    out[1] = rb;
  }
}

// The depth-2 entries of the responses array (src[0 .. n), between its brackets ra and rb): each element an object.
// flag[j] = entry j opens one, for the count.
__global__ void k_sr_elems(SrIdx x, long long n, long long ra, long long rb, long long *__restrict__ flag, unsigned long long *__restrict__ err) {
  const unsigned char *b = x.body;
  for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j <= n; j += (long long)gridDim.x * blockDim.x) {
    const long long a = j == 0 ? ra : x.src[j - 1], c = j == n ? rb : x.src[j];
    const long long pa = x.pos[a], pc = x.pos[c];
    const unsigned ca = b[pa], cc = b[pc];
    if (j < n) flag[j] = cc == '{';
    bool ok;
    if (ca == '{') ok = cc == '}';   // the element's inside: deeper entries only
    else if (!sr_gap_ws(b, pa + 1, pc)) {
      sr_fail(err, pa + 1, kSrElement);
      continue;
    } else if (ca == '[') ok = cc == '{' || (cc == ']' && j == n);
    else if (ca == '}') ok = cc == ',' || (cc == ']' && j == n);
    else if (ca == ',') ok = cc == '{';
    else ok = false;
    if (!ok) sr_fail(err, cc == '}' || cc == ']' ? pc : pa, cc == '"' || cc == '[' || ca == '"' || ca == '[' && cc != '{' ? kSrElement : kSrSyntax);
  }
}
__global__ void k_sr_records(long long n, const long long *__restrict__ src, const long long *__restrict__ flag, const long long *__restrict__ rank,
                             long long *__restrict__ ropen, long long *__restrict__ rclose) {
  for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j < n; j += (long long)gridDim.x * blockDim.x)
    if (flag[j] && j + 1 < n) {
      ropen[rank[j]] = src[j];
      rclose[rank[j]] = src[j + 1];
    }
}

// ---- records and hits -------------------------------------------------------------------------------------------------
struct SrArgs {
  SrIdx x;
  long long n_rec;
  const long long *ropen, *rclose;
  const uint8_t *with_ranks;   // [n_rec]
  int n_rank;
  const unsigned char *names;  // ranking names, UTF-8, name k = names[name_off[k] .. name_off[k + 1])
  int name_off[9];
};
// one warp per record: status[r], total[r], nh[r] = its hits (0 for an error element or a status other than 200); write
// pass: the hits' bracket entries hopen / hclose and their record hrec, from hoff[r]
template <bool kWrite>
__global__ void k_sr_resp(SrArgs a, int32_t *__restrict__ status, long long *__restrict__ total, long long *__restrict__ nh,
                          const long long *__restrict__ hoff, long long *__restrict__ hopen, long long *__restrict__ hclose,
                          int32_t *__restrict__ hrec, unsigned long long *__restrict__ err) {
  const int lane = threadIdx.x & 31;
  const unsigned char *b = a.x.body;
  for (long long r = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; r < a.n_rec; r += ((long long)gridDim.x * blockDim.x) >> 5) {
    bool has_err = false, has_status = false, seen_hits = false, seen_total = false;
    long long st = 0, tot = -1, ha = -1, hb = -1, bad = 0;
    int hits_kind = -1;
    int rc = sr_members(a.x, a.ropen[r], a.rclose[r], 3, &bad, [&](long long nb, long long ne, const SrVal &v) {
      if (sr_is(b, nb, ne, "error", 5)) {
        has_err = true;
      } else if (sr_is(b, nb, ne, "status", 6)) {
        if (has_status) return true;
        has_status = true;
        if (v.kind != kVScalar || !sr_integer(b, v.b, v.e, -2147483648LL, 2147483647LL, &st)) {
          if (lane == 0) sr_fail(err, r, kSrStatus);
          st = 0;
        }
      } else if (sr_is(b, nb, ne, "hits", 4) && !seen_hits) {
        seen_hits = true;
        if (v.kind != kVObject) return true;
        long long bad2 = 0;
        bool seen_inner = false;
        const int rc2 = sr_members(a.x, v.ob, v.oe, 4, &bad2, [&](long long nb2, long long ne2, const SrVal &w) {
          if (sr_is(b, nb2, ne2, "total", 5) && !seen_total) {
            seen_total = true;
            if (w.kind == kVScalar) {
              if (!sr_integer(b, w.b, w.e, -9223372036854775807LL, 9223372036854775807LL, &tot)) tot = -1;
            } else if (w.kind == kVObject) {
              long long bad3 = 0;
              bool seen_value = false;
              const int rc3 = sr_members(a.x, w.ob, w.oe, 5, &bad3, [&](long long nb3, long long ne3, const SrVal &u) {
                if (!seen_value && sr_is(b, nb3, ne3, "value", 5)) {
                  seen_value = true;
                  if (u.kind != kVScalar || !sr_integer(b, u.b, u.e, -9223372036854775807LL, 9223372036854775807LL, &tot)) tot = -1;
                }
                return true;
              });
              if (rc3 && lane == 0) sr_fail(err, r, rc3);
            }
          } else if (sr_is(b, nb2, ne2, "hits", 4) && !seen_inner) {
            seen_inner = true;
            hits_kind = w.kind == kVScalar && sr_is_null(b, w.b, w.e) ? -1 : w.kind;
            ha = w.ob;
            hb = w.oe;
          }
          return true;
        });
        if (rc2 && lane == 0) sr_fail(err, r, rc2);
      }
      return true;
    });
    if (rc) {
      if (lane == 0) sr_fail(err, r, rc);
      continue;
    }
    long long n = 0;
    const bool empty = has_err || (has_status && st != 200) || hits_kind == -1;
    if (!empty && hits_kind != kVArray) {
      if (lane == 0) sr_fail(err, r, kSrHitsNotArray);
    } else if (!empty) {
      const long long base = kWrite ? hoff[r] : 0;
      rc = sr_objects(a.x, ha, hb, 5, kSrHitNotObject, &bad, &n, [&](long long k, long long o, long long c) {
        if (kWrite && lane == 0) {
          hopen[base + k] = o;
          hclose[base + k] = c;
          hrec[base + k] = (int32_t)r;
        }
      });
      if (rc) {
        if (lane == 0) sr_fail(err, r, rc);
        n = 0;
      }
    }
    if (!kWrite && lane == 0) {
      status[r] = (int32_t)st;
      total[r] = tot;
      nh[r] = n;
    }
  }
}

// one warp per hit: its _id (raw inside -> id[h]), _score and, for a withRanks record, the rankings of _source.  Numbers
// the fast path cannot give exactly are listed in xlist (slot: h for the score, n_hits + h * n_rank + k for rank k).
struct SrExact {
  long long slot, b, e;
};
__global__ void k_sr_hit(SrArgs a, long long n_hits, const long long *__restrict__ hopen, const long long *__restrict__ hclose,
                         const int32_t *__restrict__ hrec, JMember *__restrict__ id, SrNum *__restrict__ score, SrNum *__restrict__ rank,
                         uint8_t *__restrict__ has_rank, SrExact *__restrict__ xlist, unsigned long long *__restrict__ n_exact,
                         unsigned long long *__restrict__ err) {
  const int lane = threadIdx.x & 31;
  const unsigned char *b = a.x.body;
  for (long long h = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; h < n_hits; h += ((long long)gridDim.x * blockDim.x) >> 5) {
    int n_id = 0, n_score = 0, n_source = 0, code = 0;
    long long ib = 0, ie = 0;
    SrNum sc = {};
    unsigned seen = 0, present = 0;
    const bool ranks = a.n_rank > 0 && a.with_ranks[hrec[h]];
    long long bad = 0;
    const int rc = sr_members(a.x, hopen[h], hclose[h], 6, &bad, [&](long long nb, long long ne, const SrVal &v) {
      if (sr_is(b, nb, ne, "_id", 3)) {
        if (n_id++) code = code ? code : kSrRepeated;
        if (v.kind != kVString) code = code ? code : kSrNoId;
        ib = v.b;
        ie = v.e;
      } else if (sr_is(b, nb, ne, "_score", 6)) {
        if (n_score++) code = code ? code : kSrRepeated;
        if (v.kind != kVScalar || !sr_number(b, v.b, v.e, &sc)) code = code ? code : kSrNoScore;
        else if (sc.exact && n_score == 1 && lane == 0) {   // one slot per hit: a repeated _score is an error anyway
          const unsigned long long i = atomicAdd(n_exact, 1ULL);
          xlist[i] = SrExact{h, v.b, v.e};
        }
      } else if (sr_is(b, nb, ne, "_source", 7) && !n_source++ && ranks && v.kind == kVObject) {   // the first _source only
        long long bad2 = 0;
        const int rc2 = sr_members(a.x, v.ob, v.oe, 7, &bad2, [&](long long nb2, long long ne2, const SrVal &w) {
          for (int k = 0; k < a.n_rank; ++k) {
            if ((seen >> k & 1) || !sr_name_is(b, nb2, ne2, a.names + a.name_off[k], a.name_off[k + 1] - a.name_off[k])) continue;
            seen |= 1u << k;
            if (w.kind == kVScalar && sr_is_null(b, w.b, w.e)) continue;
            SrNum x;
            if (w.kind != kVScalar || !sr_number(b, w.b, w.e, &x)) {
              code = code ? code : kSrBadRank;
              continue;
            }
            present |= 1u << k;
            if (lane == 0) {
              rank[h * a.n_rank + k] = x;
              if (x.exact) {
                const unsigned long long i = atomicAdd(n_exact, 1ULL);
                xlist[i] = SrExact{n_hits + h * a.n_rank + k, w.b, w.e};
              }
            }
          }
          return true;
        });
        if (rc2) code = code ? code : rc2;
      }
      return true;
    });
    if (lane == 0) {
      if (rc) code = rc;
      else if (!code && !n_id) code = kSrNoId;
      else if (!code && !n_score) code = kSrNoScore;
      if (code) sr_fail(err, h, code);
      id[h] = JMember{ib, ie, 0, 0};
      score[h] = sc;
      has_rank[h] = (uint8_t)present;
    }
  }
}
// the host's exact values into their slots
__global__ void k_sr_exact_put(long long n, const long long *__restrict__ slot, const SrNum *__restrict__ val, long long n_hits,
                               SrNum *__restrict__ score, SrNum *__restrict__ rank) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long s = slot[i];
    if (s < n_hits) score[s] = val[i];
    else rank[s - n_hits] = val[i];
  }
}
// the double columns: score[h], rank[h * n_rank + k] (NaN where absent)
__global__ void k_sr_values(long long n_hits, int n_rank, const SrNum *__restrict__ score, const SrNum *__restrict__ rank,
                            const uint8_t *__restrict__ has_rank, double *__restrict__ sv, double *__restrict__ rv) {
  for (long long h = blockIdx.x * (long long)blockDim.x + threadIdx.x; h < n_hits; h += (long long)gridDim.x * blockDim.x) {
    sv[h] = score[h].v;
    for (int k = 0; k < n_rank; ++k) rv[h * n_rank + k] = (has_rank[h] >> k & 1) ? rank[h * n_rank + k].v : __longlong_as_double(0x7ff8000000000000LL);
  }
}

// ---- the PredictedResult text ----------------------------------------------------------------------------------------
// {"itemScores":[ hit, hit, ... ]}, hit = {"item":<quoted id>,"score":<double>[,"ranks":{<quoted name>:<double>,...}]}
constexpr int kSrHead = 15, kSrFoot = 2;   // {"itemScores":[  and  ]}
struct SrText {
  const long long *id_off;
  const unsigned char *id_bytes;
  const SrNum *score, *rank;
  const uint8_t *has_rank;
  const int32_t *hrec;
  const long long *rec_hoff;     // [n_rec + 1] first hit of each record
  int n_rank;
  const unsigned char *qnames;   // json4s-quoted names followed by ':'
  int qname_off[9];
};
__device__ __forceinline__ long long sr_lit(unsigned char *o, long long k, const char *s, int n) {
  if (o)
    for (int i = 0; i < n; ++i) o[k + i] = (unsigned char)s[i];
  return k + n;
}
// one hit's text (a leading ',' unless it is its record's first); o == nullptr: the length only
__device__ __forceinline__ long long sr_hit_text(const SrText &t, long long h, unsigned char *o) {
  long long k = 0;
  if (h != t.rec_hoff[t.hrec[h]]) k = sr_lit(o, k, ",", 1);
  k = sr_lit(o, k, "{\"item\":\"", 9);
  k += uq_escape(t.id_bytes + t.id_off[h], t.id_off[h + 1] - t.id_off[h], o ? o + k : nullptr);
  k = sr_lit(o, k, "\",\"score\":", 10);
  k += sr_java_text(t.score[h], o ? o + k : nullptr);
  const unsigned pr = t.has_rank[h];
  if (pr) {
    k = sr_lit(o, k, ",\"ranks\":{", 10);
    bool first = true;
    for (int r = 0; r < t.n_rank; ++r) {
      if (!(pr >> r & 1)) continue;
      if (!first) k = sr_lit(o, k, ",", 1);
      first = false;
      k = sr_lit(o, k, (const char *)t.qnames + t.qname_off[r], t.qname_off[r + 1] - t.qname_off[r]);
      k += sr_java_text(t.rank[h * t.n_rank + r], o ? o + k : nullptr);
    }
    k = sr_lit(o, k, "}", 1);
  }
  return sr_lit(o, k, "}", 1);
}
// ---- batchpredict lines -----------------------------------------------------------------------------------------------
// [RECALL] PredictionIO's BatchPredict line: {"query":<the query line re-rendered by json4s>,"prediction":<PredictedResult>}.
// The echo drops insignificant whitespace, decodes and re-quotes strings, prints integer literals as BigInt does (-0 -> 0)
// and other numbers as Double.toString; member order and repeated members are kept.
constexpr int kBpHead = 9, kBpMid = 14, kBpFoot = 1;   // {"query":  ,"prediction":  }
constexpr int kBpMaxDepth = 64;
enum { kSrLine = 16, kSrWithRanks, kSrLineRepeated, kSrLineDeep };   // line errors, keyed by the record
struct SrLines {
  const unsigned char *bytes;    // the body's query lines, line r = bytes[off[r] .. off[r + 1])
  const long long *off;
  const long long *xpos;         // sorted byte positions of the numbers the host converted, and their values
  const SrNum *xval;
  long long nx;
};
// the raw string from p (after its opening quote): its end (the closing quote), or -1 when it is bad or unclosed
__device__ __forceinline__ long long sr_line_string(const unsigned char *b, long long p, long long e) {
  while (p < e) {
    const unsigned c = b[p];
    if (c == '"') return p;
    if (c < 0x20) return -1;
    if (c != '\\') {
      ++p;
      continue;
    }
    if (p + 1 >= e) return -1;
    const unsigned x = b[p + 1];
    if (x == 'u') {
      if (p + 6 > e) return -1;
      for (int k = 2; k < 6; ++k) {
        const unsigned h = b[p + k];
        if (!(h - '0' < 10u || (h | 0x20) - 'a' < 6u)) return -1;
      }
      p += 6;
    } else if (x == '"' || x == '\\' || x == '/' || x == 'b' || x == 'f' || x == 'n' || x == 'r' || x == 't') {
      p += 2;
    } else {
      return -1;
    }
  }
  return -1;
}
__device__ __forceinline__ bool sr_num_byte(unsigned c) { return c - '0' < 10u || c == '-' || c == '+' || c == '.' || c == 'e' || c == 'E'; }
__device__ __forceinline__ bool sr_alpha(unsigned c) { return (c | 0x20) - 'a' < 26u; }
// One thread per line: the line is one JSON object (nesting below kBpMaxDepth); its top-level withRanks, when present and
// not null, is true or false and appears once (cco_query_file_read's rules) -> wr[r].  Numbers the fast path cannot give
// are listed in xlist (slot = -1, their byte positions in the lines).
__global__ void k_sr_lines(long long n, SrLines q, uint8_t *__restrict__ wr, SrExact *__restrict__ xlist, unsigned long long *__restrict__ n_exact,
                           unsigned long long *__restrict__ err) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < n; r += (long long)gridDim.x * blockDim.x) {
    const unsigned char *b = q.bytes;
    long long p = q.off[r];
    const long long e = q.off[r + 1];
    unsigned char stack[kBpMaxDepth];
    int depth = 0, st = 0;   // 0 value, 1 key or '}', 2 ':', 3 ',' or close, 4 key, 5 done
    int n_wr = 0, code = 0;
    bool is_wr = false;
    uint8_t w = 0;
    while (!code) {
      while (p < e && sr_ws(b[p])) ++p;
      if (p >= e) {
        if (st != 5) code = kSrLine;
        break;
      }
      const unsigned c = b[p];
      if (st == 5) {
        code = kSrLine;
      } else if (st == 1 || st == 4) {
        if (c == '}' && st == 1) {
          st = 3;
          --depth;
          ++p;
          if (depth == 0) st = 5;
          continue;
        }
        const long long z = c == '"' ? sr_line_string(b, p + 1, e) : -1;
        if (z < 0) {
          code = kSrLine;
          break;
        }
        is_wr = depth == 1 && sr_is(b, p + 1, z, "withRanks", 9);
        if (is_wr && n_wr++) code = kSrLineRepeated;
        p = z + 1;
        st = 2;
      } else if (st == 2) {
        if (c != ':') code = kSrLine;
        ++p;
        st = 0;
      } else if (st == 3) {
        if (c == ',') {
          st = stack[depth - 1] == '{' ? 4 : 0;
          ++p;
        } else if (c == (stack[depth - 1] == '{' ? '}' : ']')) {
          --depth;
          ++p;
          st = depth == 0 ? 5 : 3;
        } else {
          code = kSrLine;
        }
      } else {   // a value
        const bool wr_value = is_wr;
        is_wr = false;
        if (depth == 0 && c != '{') {
          code = kSrLine;
        } else if (c == '{' || c == '[') {
          if (depth == kBpMaxDepth) {
            code = kSrLineDeep;
            break;
          }
          if (wr_value) code = kSrWithRanks;
          stack[depth++] = (unsigned char)c;
          ++p;
          st = c == '{' ? 1 : 0;
          if (c == '[') {   // an empty array
            long long t = p;
            while (t < e && sr_ws(b[t])) ++t;
            if (t < e && b[t] == ']') {
              --depth;
              p = t + 1;
              st = 3;
            }
          }
        } else if (c == '"') {
          const long long z = sr_line_string(b, p + 1, e);
          if (z < 0) code = kSrLine;
          else if (wr_value) code = kSrWithRanks;
          p = z + 1;
          st = 3;
        } else {
          long long t = p;
          while (t < e && (sr_num_byte(b[t]) || sr_alpha(b[t]))) ++t;
          SrNum x;
          const bool lit_true = t - p == 4 && b[p] == 't' && b[p + 1] == 'r' && b[p + 2] == 'u' && b[p + 3] == 'e';
          const bool lit_false = t - p == 5 && b[p] == 'f' && b[p + 1] == 'a' && b[p + 2] == 'l' && b[p + 3] == 's' && b[p + 4] == 'e';
          if (lit_true || lit_false || sr_is_null(b, p, t)) {
            if (wr_value) w = lit_true;
          } else if (sr_number(b, p, t, &x)) {
            if (wr_value) code = kSrWithRanks;
            const bool integer = [&] {
              for (long long k = p; k < t; ++k)
                if (b[k] == '.' || (b[k] | 0x20) == 'e') return false;
              return true;
            }();
            if (!integer && x.exact) {
              const unsigned long long i = atomicAdd(n_exact, 1ULL);
              xlist[i] = SrExact{-1, p, t};
            }
          } else {
            code = kSrLine;
          }
          p = t;
          st = 3;
        }
        if (depth == 0 && st == 3) st = 5;
      }
    }
    if (code) sr_fail(err, r, code);
    wr[r] = w;
  }
}
// the echo of line r (checked by k_sr_lines); o == nullptr: the length only
__device__ __forceinline__ long long sr_echo(const SrLines &q, long long r, unsigned char *o) {
  const unsigned char *b = q.bytes;
  long long p = q.off[r], k = 0;
  const long long e = q.off[r + 1];
  while (p < e) {
    const unsigned c = b[p];
    if (sr_ws(c)) {
      ++p;
    } else if (c == '"') {
      const long long z = sr_line_string(b, p + 1, e);
      if (o) o[k] = '"';
      ++k;
      long long t = p + 1;
      unsigned char u[4];
      while (t < z) {   // one code point at a time, decoded, then through json4s' quote
        int n;
        if (b[t] == '\\') {
          n = sr_next_utf8(b, &t, z, u);
        } else {
          const unsigned x = b[t];
          n = x < 0xc0 ? 1 : x < 0xe0 ? 2 : x < 0xf0 ? 3 : 4;
          if (t + n > z) n = 1;
          for (int j = 0; j < n; ++j) u[j] = b[t + j];
          t += n;
        }
        k += uq_escape(u, n, o ? o + k : nullptr);
      }
      if (o) o[k] = '"';
      ++k;
      p = z + 1;
    } else if (c == '-' || c - '0' < 10u) {
      long long t = p;
      bool integer = true;
      while (t < e && sr_num_byte(b[t])) {
        if (b[t] == '.' || (b[t] | 0x20) == 'e') integer = false;
        ++t;
      }
      if (integer) {   // BigInt: the literal, but -0 is 0
        const bool minus_zero = t - p == 2 && b[p] == '-' && b[p + 1] == '0';
        for (long long j = p + minus_zero; j < t; ++j) {
          if (o) o[k] = b[j];
          ++k;
        }
      } else {
        SrNum x;
        sr_number(b, p, t, &x);
        if (x.exact) {   // the host's value: binary search by position
          long long lo = 0, hi = q.nx - 1;
          while (lo < hi) {
            const long long mid = (lo + hi) >> 1;
            if (q.xpos[mid] < p) lo = mid + 1;
            else hi = mid;
          }
          x = q.xval[lo];
        }
        k += sr_java_text(x, o ? o + k : nullptr);
      }
      p = t;
    } else {
      if (o) o[k] = (unsigned char)c;
      ++k;
      ++p;
    }
  }
  return k;
}
__global__ void k_sr_echo_len(long long n, SrLines q, long long *__restrict__ len) {
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < n; r += (long long)gridDim.x * blockDim.x) len[r] = sr_echo(q, r, nullptr);
}

// bytes of record r's text before its first hit: {"itemScores":[, after the echo frame for a batchpredict line
__device__ __forceinline__ long long sr_rec_head(const long long *eoff, long long r) {
  return kSrHead + (eoff ? kBpHead + kBpMid + eoff[r + 1] - eoff[r] : 0);
}
// length pass: len[h]; write pass: at rec_off[r] + head + (toff[h] - toff[first hit of r])
template <bool kWrite>
__global__ void k_sr_hit_text(SrText t, const long long *__restrict__ eoff, long long n_hits, long long *__restrict__ len,
                              const long long *__restrict__ toff, const long long *__restrict__ rec_off, unsigned char *__restrict__ out) {
  for (long long h = blockIdx.x * (long long)blockDim.x + threadIdx.x; h < n_hits; h += (long long)gridDim.x * blockDim.x) {
    if (!kWrite) {
      len[h] = sr_hit_text(t, h, nullptr);
      continue;
    }
    const int r = t.hrec[h];
    sr_hit_text(t, h, out + rec_off[r] + sr_rec_head(eoff, r) + toff[h] - toff[t.rec_hoff[r]]);
  }
}
// rec_off[r] = toff[first hit] + r * (frame bytes) + eoff[r] (the echoes before it, batchpredict lines only); write: the
// frame of each record, and its echo
template <bool kWrite>
__global__ void k_sr_rec_text(long long n_rec, const long long *__restrict__ rec_hoff, const long long *__restrict__ toff,
                              const long long *__restrict__ eoff, SrLines q, long long *__restrict__ rec_off, unsigned char *__restrict__ out) {
  const int frame = kSrHead + kSrFoot + (eoff ? kBpHead + kBpMid + kBpFoot : 0);
  for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r <= n_rec; r += (long long)gridDim.x * blockDim.x) {
    const long long at = toff[rec_hoff[r]] + r * frame + (eoff ? eoff[r] : 0);
    if (!kWrite) {
      rec_off[r] = at;
      continue;
    }
    if (r == n_rec) continue;
    long long k = at;
    if (eoff) {
      k = sr_lit(out, k, "{\"query\":", kBpHead);
      k += sr_echo(q, r, out + k);
      k = sr_lit(out, k, ",\"prediction\":", kBpMid);
      sr_lit(out, rec_off[r + 1] - kBpFoot, "}", kBpFoot);
    }
    sr_lit(out, k, "{\"itemScores\":[", kSrHead);
    sr_lit(out, rec_off[r + 1] - kSrFoot - (eoff ? kBpFoot : 0), "]}", kSrFoot);
  }
}

}  // namespace cco
