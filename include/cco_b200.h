/*
 * cco_b200.h -- C ABI of the H100-native (sm_90a) Correlated Cross-Occurrence (CCO) model builder.
 *
 * This is the drop-in boundary for the train hot path of actionml/universal-recommender.
 * It replaces the two calls the reference makes into Apache Mahout 0.13.0:
 *
 *   SimilarityAnalysis.cooccurrencesIDSs(Array[IndexedDataset], randomSeed,
 *       maxInterestingItemsPerThing, maxNumInteractions)       src/main/scala/URAlgorithm.scala:323-329
 *   SimilarityAnalysis.crossOccurrenceDownsampled(
 *       List[DownsamplableCrossOccurrenceDataset], randomSeed) src/main/scala/URAlgorithm.scala:343-346
 *
 * A Scala object with those two signatures marshals each IndexedDataset's matrix into CSR and
 * calls cco_train() over JNI (INTEGRATION.md has the stub); everything else in the reference
 * (engine.json, DataSource, Preparator, URModel, EsClient) is untouched.
 *
 * Plain C: pointers and sizes only, no CUDA/torch types.  All functions return 0 on success or
 * a negative cco_status_t; cco_last_error() gives the message (thread-local).  There is no CPU
 * fallback: every entry point that computes fails with CCO_E_CUDA when no sm_90 device exists.
 */
#ifndef CCO_B200_H
#define CCO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CCO_ABI_VERSION 2

typedef enum {
  CCO_OK = 0,
  CCO_E_INVALID_ARG = -1,    /* mirrors IllegalArgumentException / Preconditions.checkArgument in Mahout */
  CCO_E_CUDA = -2,           /* CUDA runtime / no usable device */
  CCO_E_NCCL = -3,
  CCO_E_OOM = -4,
  CCO_E_SHAPE_MISMATCH = -5, /* matrices do not share the user (row) space -- Preparator.scala:47-77 */
  CCO_E_UNSUPPORTED = -6
} cco_status_t;

/*
 * Input: one binary user x item matrix per event type, exactly what Preparator builds as
 * IndexedDatasetSpark (src/main/scala/Preparator.scala:160-214): every stored value is 1.0
 * (RandomAccessSparseVector.setQuick(col, 1.0), :201-208) so there is no values array;
 * n_rows is the size of the shared user dictionary (newRowCardinality, :213), including users
 * with no interaction in this event type.  Column indices may come in any order inside a row
 * and duplicates collapse (setQuick semantics).  The library never keeps host pointers.
 */
typedef struct {
  int64_t n_rows;         /* U, must be equal for all matrices of one call, < 2^31 (Mahout keys are Int) */
  int32_t n_cols;         /* I of this event type, < 2^31 - 1 */
  const int64_t *row_ptr; /* [n_rows + 1], row_ptr[0] == 0, monotone */
  const int32_t *col_idx; /* [row_ptr[n_rows]], each in [0, n_cols) */
} cco_csr_t;

/*
 * Per-matrix parameters = DownsamplableCrossOccurrenceDataset(iD, maxElementsPerRow,
 * maxInterestingElements, minLLROpt) as built at src/main/scala/URAlgorithm.scala:336-340.
 * Defaults in the reference: 500 / 50 / None (URAlgorithm.scala:54,56,338-340).
 */
typedef struct {
  int32_t max_interactions; /* m >= 1: maxItemsPerUser | maxEventsPerEventType */
  int32_t top_k;            /* k in [1, CCO_MAX_TOP_K]: maxCorrelatorsPerItem | maxCorrelatorsPerEventType */
  int32_t has_min_llr;      /* Option[Double].isDefined */
  double min_llr;           /* keep a cell only if llr >= min_llr */
} cco_indicator_params_t;

#define CCO_MAX_TOP_K 2048

/*
 * Limits (each one is a clean CCO_E_UNSUPPORTED with a message, never a wrong result):
 *  - top_k <= CCO_MAX_TOP_K;  stored entries per matrix < 2^32;  n_rows < 2^31 - 1 (Mahout row keys are Int).
 *  - packed accumulator word: a row's co-occurrence counts live in shared memory as (column << count_bits | count) in
 *    32 bits.  count <= min(largest primary-item marginal, largest column marginal of this event type) must fit next to
 *    the column id: bitlen(n_cols + 1) + bitlen(max count) <= 32.  After the reference's default downsampling (500) every
 *    marginal is <= ~560, i.e. 10 bits: item spaces up to 4M columns.  Without downsampling (m huge) a 1M-column space
 *    allows counts < 4096.
 */

/* cco_train flags */
enum {
  /* Row sample rate of sampleDownAndBinarize: 0 = real min(m,d)/d (default); 1 = literal
   * Int/Int division recalled from Mahout 0.13.0 (1 if d <= m else 0).  DESIGN.md "Downsampling". */
  CCO_FLAG_ROWRATE_INTDIV = 1,
  /* LogLikelihood.entropy evaluation order: 0 = left-to-right subtraction (default);
   * 2 = varargs form xLogX(sum) - (sum of xLogX).  Last-bit difference only. */
  CCO_FLAG_ENTROPY_VARARGS = 2,
  /* inputs are already canonical (columns strictly ascending inside each row): skip the check */
  CCO_FLAG_ASSUME_CANONICAL = 4,
  /* measurement only: leave the packed indicator arrays in HBM (col/llr/count host arrays are not
   * filled; row_ptr is).  Used for the device-resident throughput number of bench.py. */
  CCO_FLAG_RESULT_ON_DEVICE = 8,
  /* result contents.  The reference consumer keeps only the ordered column ids of each row (package.scala:100-108
   * drops the LLR values, nothing reads k11): NO_COUNT skips the count array (cco_result_matrix returns NULL for it),
   * NO_LLR skips the LLR array too -- 80 instead of 321 MB come back per train at C3. */
  CCO_FLAG_RESULT_NO_COUNT = 16,
  CCO_FLAG_RESULT_NO_LLR = 32
};

/*
 * Sampler (the repo's definition; Mahout's java.util.Random-per-Spark-block stream is not
 * reproducible by construction, SURVEY.md A.1).  For a stored (user u, item j) of a matrix with
 * raw row count d_u and raw column count c_j:
 *   mix64(z): z ^= z>>30; z *= 0xbf58476d1ce4e5b9; z ^= z>>27; z *= 0x94d049bb133111eb; z ^= z>>31
 *   h    = mix64( mix64(((uint64)(uint32)seed << 32) | (uint32)u) + (uint64)(uint32)j * 0x9e3779b97f4a7c15 )
 *   u01  = (double)(h >> 11) * 2^-53
 *   keep = u01 <= min( min(m,d_u)/d_u , min(m,c_j)/c_j )          (fp64, IEEE division)
 * Identity whenever every d_u <= m and c_j <= m -- the regime where parity with Mahout is exact.
 */

typedef struct {
  int32_t device;     /* CUDA device ordinal for this context */
  int32_t rank;       /* rank of this context in a multi-GPU job, 0 if world_size == 1 */
  int32_t world_size; /* number of cooperating contexts (one process per GPU) */
  int32_t reserved;
  /* world_size > 1: 128-byte NCCL unique id obtained from cco_nccl_unique_id() on rank 0 and
   * distributed by the host (any transport); ignored when world_size == 1 */
  const unsigned char *nccl_unique_id;
  /* optional (NULL / 0 = library-owned pinned memory): host memory the result arrays are placed in, e.g. a shared
   * segment another process maps, so that this rank's indicator slice reaches its reader without a copy.  The library
   * page-locks it (cudaHostRegister) for the life of the context; it is reused once every result has been freed. */
  void *result_arena;
  size_t result_arena_bytes;
} cco_config_t;

typedef struct cco_ctx cco_ctx_t;
typedef struct cco_result cco_result_t;
typedef struct cco_dataset cco_dataset_t;

/* Per-call statistics (the metrics/logging hook; replaces the logger.info dimension lines of
 * Preparator.scala:60,66,74 and feeds bench.py's roofline arithmetic). */
typedef struct {
  int64_t n_users;
  int64_t nnz_in_total;         /* stored entries handed in, all matrices */
  int64_t nnz_downsampled[16];  /* per matrix (first 16), after canonicalise + downsample */
  int64_t products[16];         /* per indicator: P(A',B') = sum_u degA'(u) * degB'(u), this rank's rows */
  int64_t distinct_cells[16];   /* per indicator: nnz(A'^T B') visited, this rank's rows */
  int64_t out_nnz[16];          /* per indicator: kept cells, this rank's rows */
  int64_t llr_evaluated[16];    /* per indicator: cells whose fp64 LLR was evaluated (rest: dominance-filtered) */
  /* CUDA-event times of this call.  ms_h2d: host->device copies (copy stream; overlaps ms_prepare in cco_train);
   * ms_prepare: histogram + allreduce + sampleDownAndBinarize + transpose; ms_cooccurrence: all indicators incl.
   * scheduling and result packing; ms_d2h: always 0 (the result copies overlap the next indicator on the copy
   * stream and are inside ms_cooccurrence / ms_total); ms_total: the whole call on the launch stream. */
  float ms_h2d, ms_prepare, ms_cooccurrence, ms_d2h, ms_total;
  float ms_indicator[16];       /* per indicator: row kernels only */
  int32_t n_kernel_launches;    /* kernels of this library launched by the call */
  int32_t n_mats;
  /* breakdown of ms_prepare, the same stages on any number of GPUs (on one GPU the collectives and the pack do not run:
   * [1] and [5] are empty and [3] holds the scans only): [0] input check + raw column histogram  [1] all-reduce of the raw counts
   * [2] sampleDownAndBinarize pass 1 (keep decisions, kept counts, marginals)  [3] kept-count all-gather + marginal
   * all-reduce + row_ptr scans  [4] pass 2 (ordered write)  [5] column-block all-gather + pack
   * [6] transpose of A' + largest marginals */
  float ms_prep_stage[8];
} cco_stats_t;

int cco_abi_version(void);
const char *cco_last_error(void);
const char *cco_status_string(int status);

/* number of sm_90 (H100) devices visible; <0 on CUDA failure */
int cco_device_count(void);

/* world_size > 1 only: fill 128 bytes on rank 0, hand them to every rank's cco_create */
int cco_nccl_unique_id(unsigned char out[128]);

int cco_create(const cco_config_t *cfg, cco_ctx_t **out);
/*
 * Group context: ONE context over several H100s of this process -- what the single Spark-driver thread of the reference
 * (URAlgorithm.scala:292-307) can drive through JNI.  cco_train / cco_cooccurrences_idss on it run one host thread per
 * GPU inside the library (NCCL communicator from ncclCommInitAll): each GPU uploads its block of user rows from the SAME
 * host matrices, computes a work-balanced range of primary-item rows, and copies its slice into ONE merged result (full
 * row range, one set of host arrays).  Resident datasets (cco_dataset_upload / cco_ingest) stay per-GPU APIs.
 */
int cco_create_group(int32_t n_devices, const int32_t *devices, cco_ctx_t **out);
int cco_destroy(cco_ctx_t *ctx);

/* Pinned host memory the caller can fill directly (e.g. wrapped as a direct ByteBuffer by the
 * JNI shim) so cco_train's host->device copies run at PCIe speed.  Optional. */
int cco_host_alloc(cco_ctx_t *ctx, size_t bytes, void **out);
int cco_host_free(cco_ctx_t *ctx, void *p);

/*
 * The whole hot path, mats[0] = primary (A):
 *   A' = sampleDownAndBinarize(A, seed, params[0].m); N = n_rows; colA = nnzPerColumn(A')
 *   out[0] = top-k_0 by LLR of A'^T A' (diagonal excluded), out[i] = top-k_i by LLR of A'^T B'_i
 * In a multi-GPU job every rank passes the same matrices; rank r computes a work-balanced range
 * of primary-item rows and its result holds only those rows (cco_result_row_range).
 * One call at a time per context.
 */
int cco_train(cco_ctx_t *ctx, int32_t n_mats, const cco_csr_t *mats, const cco_indicator_params_t *params,
              int32_t seed, uint32_t flags, cco_result_t **out);

/*
 * Split form of cco_train for callers that keep the matrices resident in HBM across trains
 * (the `drmA.checkpoint()` / cache() role in Mahout): upload once (host->device copy, validation,
 * canonicalisation), train any number of times with different parameters / seeds.
 * cco_train(...) == cco_dataset_upload + cco_train_dataset + cco_dataset_free.
 */
int cco_dataset_upload(cco_ctx_t *ctx, int32_t n_mats, const cco_csr_t *mats, uint32_t flags, cco_dataset_t **out);
int cco_train_dataset(cco_ctx_t *ctx, const cco_dataset_t *ds, const cco_indicator_params_t *params, int32_t seed,
                      uint32_t flags, cco_result_t **out);
int cco_dataset_free(cco_dataset_t *ds);

/*
 * Pure host helper (no GPU needed): the rank partition cco_train uses.  work_prefix[i] = products of primary items
 * [0, i) (exclusive prefix, n_items + 1 entries); bounds[r]..bounds[r+1] is rank r's contiguous item range, cut so
 * that every rank gets an equal share of (products + 1 per row).  Identical on every rank by construction.
 */
int cco_partition_rows(const int64_t *work_prefix, int32_t n_items, int32_t world_size, int32_t *bounds);

/*
 * Next row (SURVEY.md 8f-1), the ingest right before the boundary: Preparator.prepare + IndexedDatasetSpark.apply
 * (src/main/scala/Preparator.scala:44-87, 100-216) on integer-tokenised events.  Type 0 is the primary event: the
 * user dictionary = users with at least min_events_per_user primary events (duplicates counted, :129-132; 0/1 = any
 * primary event); every type is restricted to those users (:175-178); each type's item dictionary holds the items that
 * still have an event (:184); duplicates collapse (:201-208).  Dictionaries are in ascending raw-id order.
 * user_map [n_users_raw] and item_maps[t] [n_items_raw of t] are host arrays filled with the new id or -1.
 * The resulting dataset is resident in HBM and goes straight into cco_train_dataset.
 */
typedef struct {
  int64_t n_events;
  const int64_t *user; /* raw user id in [0, n_users_raw) */
  const int32_t *item; /* raw item id in [0, n_items_raw) */
  int32_t n_items_raw;
} cco_events_t;
int cco_ingest(cco_ctx_t *ctx, int32_t n_types, const cco_events_t *events, int64_t n_users_raw, int32_t min_events_per_user,
               int32_t *user_map, int32_t *const *item_maps, cco_dataset_t **out);
/*
 * Bench/test utility: the synthetic Zipf event streams of SURVEY.md 8(d) generated straight into HBM (no host event
 * arrays), then the same ingest as cco_ingest.  Stream of one event type, bit-identical to synth.py's numpy twin:
 *   h1 = mix64(mix64(seed) + (e + 1) * 0x9e3779b97f4a7c15), h2 = mix64(h1 ^ 0x6a09e667f3bcc909)      e = 0 .. n_events-1
 *   user = user_perm[upper_bound(user_cdf, (h1 >> 11) * 2^-53)], item = item_perm[upper_bound(item_cdf, (h2 >> 11) * 2^-53)]
 * cdf = inclusive, normalised cumulative weights over ranks; perm maps rank -> id.  All arrays are host pointers.
 * keep_item_space != 0: the item dictionary of every type is its raw id space (identity), not only the ids with an event.
 */
typedef struct {
  int64_t n_events;
  uint64_t seed;
  int32_t n_items;
  int32_t reserved;
  const double *item_cdf;   /* [n_items] */
  const int32_t *item_perm; /* [n_items] */
} cco_synth_type_t;
int cco_synth_ingest(cco_ctx_t *ctx, int32_t n_types, const cco_synth_type_t *types, int64_t n_users_raw, const double *user_cdf,
                     const int32_t *user_perm, int32_t min_events_per_user, int32_t keep_item_space, cco_dataset_t **out);
/* copy matrix i of a resident dataset into caller-provided host arrays ([n_rows + 1] and [nnz], see cco_dataset_shape) */
int cco_dataset_copy_to_host(const cco_dataset_t *ds, int32_t i, int64_t *row_ptr, int32_t *col_idx);
int cco_dataset_shape(const cco_dataset_t *ds, int32_t i, int64_t *n_rows, int32_t *n_cols, int64_t *nnz);
/* test helper: copy matrix i of a resident dataset back to the host (malloc'ed; free with cco_free) */
int cco_dataset_download(const cco_dataset_t *ds, int32_t i, int64_t **row_ptr, int32_t **col_idx);

/* CUDA-event stopwatch on the context's launch stream (what bench.py brackets its timed region with) */
int cco_timer_start(cco_ctx_t *ctx);
int cco_timer_stop(cco_ctx_t *ctx, float *ms);

/* SimilarityAnalysis.cooccurrencesIDSs convenience: one global (k, m) for every matrix */
int cco_cooccurrences_idss(cco_ctx_t *ctx, int32_t n_mats, const cco_csr_t *mats, int32_t seed,
                           int32_t max_interesting_items_per_thing, int32_t max_num_interactions,
                           uint32_t flags, cco_result_t **out);

/*
 * Result = List[IndexedDataset]; element i has rowIDs = A.columnIDs, columnIDs = B_i.columnIDs.
 * Indicator i as CSR over primary items: rows sorted by (llr desc, col asc), so the consumer's
 * sortBy(-llr) in package.scala:100-108 is a no-op.  count = k11 of each kept cell.
 * Pointers are owned by the result (pinned host memory) and live until cco_result_free.
 * row_ptr has (row_end - row_begin + 1) entries, relative to this rank's first row.
 */
int cco_result_num_matrices(const cco_result_t *r);
int cco_result_row_range(const cco_result_t *r, int32_t i, int64_t *row_begin, int64_t *row_end);
int cco_result_matrix(const cco_result_t *r, int32_t i, int64_t *n_rows, int32_t *n_cols,
                      const int64_t **row_ptr, const int32_t **col_idx, const double **llr,
                      const int32_t **count);
int cco_result_stats(const cco_result_t *r, cco_stats_t *out);
int cco_result_free(cco_result_t *r);

/*
 * Next row (SURVEY.md 8f-2): the model as the Elasticsearch bulk body, assembled on the device.  Replaces, per primary item,
 * IndexedDatasetConversions.toStringMapRDD (src/main/scala/package.scala:82-110: non-zeros ordered by -LLR, mapped to
 * column id strings, LLR dropped, empty rows -> empty array), URModel.save's groupAll + ("id" -> item)
 * (src/main/scala/URModel.scala:47-102) and the bulk serialisation of saveToEs with es.mapping.id = id
 * (src/main/scala/EsClient.scala:300-313).  One document per row of the result (a rank's slice or a merged model):
 *     {"index":{"_id":"<item>"}}\n{"id":"<item>","<names[0]>":["<col>",...],"<names[1]>":[...]}\n
 * Strings are JSON-escaped here ('"' and '\\' get a backslash, bytes < 0x20 become \u00xx, the rest passes through).
 * dictionaries: id i = bytes[offsets[i] .. offsets[i + 1]) (UTF-8); row_ids covers the primary item space, col_ids[i]
 * the item space of event i.  *out_bytes is pinned memory owned by the context: release it with cco_host_free.
 */
typedef struct {
  int64_t n;
  const int64_t *offsets; /* [n + 1] */
  const char *bytes;
} cco_dictionary_t;
int cco_format_es_bulk(cco_ctx_t *ctx, const cco_result_t *res, int32_t n_names, const char *const *names,
                       const cco_dictionary_t *row_ids, const cco_dictionary_t *col_ids, char **out_bytes, int64_t *out_len);

/*
 * SURVEY.md 8f-1 on string ids: Preparator.prepare (src/main/scala/Preparator.scala:44-87, 100-216) on (user id, item id)
 * byte strings, dictionaries included.  Type 0 is the primary event.  Exactly what the host mirror preparator.prepare returns:
 *  - user dictionary: users with >= max(min_events_per_user, 1) primary events (duplicates count, :129-132), ordered by
 *    first appearance in the primary stream;
 *  - events of type t survive iff their user is in the user dictionary (:175-178);
 *  - item dictionary of type t: items with a surviving event of type t, ordered by first appearance among those events;
 *  - matrix t: binary CSR over the user dictionary, duplicates collapsed, columns ascending.
 * Ids are arbitrary byte strings compared bytewise (UTF-8 of a Python str; the empty string is an id), in the Arrow
 * large_string layout: id e = bytes[offsets[e] .. offsets[e + 1]).  n_events < 2^31 per type.  Offsets below 0, decreasing
 * offsets and offsets[0] > offsets[n] give CCO_E_INVALID_ARG before any kernel reads bytes through them.  The dataset is
 * resident like one from cco_ingest (every rank of a multi-GPU job builds the whole matrices and works on its user block);
 * per-GPU contexts only, as every resident dataset.
 */
typedef struct {
  int64_t n_events;
  const int64_t *user_offsets; /* [n_events + 1] */
  const char *user_bytes;
  const int64_t *item_offsets; /* [n_events + 1] */
  const char *item_bytes;
} cco_string_events_t;
int cco_ingest_strings(cco_ctx_t *ctx, int32_t n_types, const cco_string_events_t *events, int32_t min_events_per_user,
                       cco_dataset_t **out);
/* which = -1: the user dictionary; which = t: the item dictionary of type t.  Pinned host memory owned by the dataset,
 * valid until cco_dataset_free.  CCO_E_INVALID_ARG on datasets that were not built from strings. */
int cco_dataset_dictionary(const cco_dataset_t *ds, int32_t which, cco_dictionary_t *out);

/*
 * Next row (SURVEY.md 8f-3): the backfill ranks of PopModel (src/main/scala/PopModel.scala:113-182) as per-item event
 * histograms over 1 / 2 / 3 time buckets of [start_ms, end_ms) -- what URAlgorithm.getRanksRDD (URAlgorithm.scala:537-560)
 * joins into the model.  events: (item index, event time in epoch milliseconds), already restricted to the ranking's event
 * names.  score[j] is meaningful iff present[j] != 0: `popular` lists the items with an event in the interval, `trending`
 * the items seen in both halves (newer - older), `hot` the items seen in all three thirds ((newer - middle) - (middle -
 * older)); `trending` / `hot` are empty when the older (or middle) bucket has no event at all, as in the reference.
 * RankingType.UserDefined is not a histogram and stays with the caller.  CCO_POP_RANDOM is accepted by cco_format_model only
 * (a random rank is keyed by id string; this entry works on item indices): see there.
 */
enum { CCO_POP_POPULAR = 0, CCO_POP_TRENDING = 1, CCO_POP_HOT = 2, CCO_POP_RANDOM = 3 };
int cco_pop_model(cco_ctx_t *ctx, int32_t mode, int64_t n_events, const int32_t *item, const int64_t *time_ms, int32_t n_items,
                  int64_t start_ms, int64_t end_ms, double *score, unsigned char *present);

/*
 * The complete model index (SURVEY.md 8f-2 + 8f-3): calcAll's propertiesRDD (URAlgorithm.scala:351-367) joined into the
 * documents of cco_format_es_bulk the way URModel.save's groupAll + ("id" -> item) does (URModel.scala:57-102).
 * Documents: every row of the result, then (only in the call whose result begins at row 0) every item without a row that
 * has a property or a score in a ranking, in order of first appearance (property items first, then the ranking streams in
 * order).  Items are matched by id string.  Fields: "id", the indicators in name order, the properties in field index order,
 * the rankings in order:
 *     {"index":{"_id":"<id>"}}\n{"id":"<id>"[,"<indicator>":[...]]*[,"<field>":<value>]*[,"<ranking>":<number>]*}\n
 * Where names repeat, precedence per document (lowest to highest): indicators < properties < rankings (a later ranking beats
 * an earlier one) < "id"; the lower field is not written.  Indicator names that repeat each other (or are "id") are written
 * as cco_format_es_bulk writes them.  Property values are JSON text, spliced verbatim (never parsed); ids and names are
 * JSON-escaped.  Rank numbers are Java's Double.toString of an integer: "-"?digits".0" below 10^7, else d.ddd"E"n with the
 * trailing zeros of the digits dropped (1.0E7, 1.2345678E7).  Without properties and rankings the body is byte-identical
 * to cco_format_es_bulk.
 * CCO_POP_RANDOM (RankingType.Random, PopModel.calcRandom, PopModel.scala:98-110): the items are the targets of every event
 * of the ranking's streams in [start_ms, end_ms) -- pass every event name's stream, as the reference ignores eventNames --
 * plus every item with a property triple.  The value is n · 10^-15, uniform in [0, 1), a function of the id bytes and the
 * window only: h = the id's 64-bit string hash (cco_strings.cuh k_str_hash), r = mix64(h ^ mix64((uint64)start_ms ^
 * mix64((uint64)end_ms))), n = floor(r · 10^15 / 2^64).  So the values repeat for a repeated window and change with it (an
 * ordinary train ends "now"), and every rank of a group writes the same value.  Text: Java's Double.toString of n / 10^15:
 * "0.0" for n = 0, "0." and n's 15 digits with the trailing zeros dropped for n >= 10^12 (0.001, 0.5, 0.123456789012345),
 * else d.ddd"E-"k (1.0E-15, 1.23E-13, 9.99999999999E-4).
 * Errors: CCO_E_INVALID_ARG for negative or decreasing offsets in any column, a field index outside [0, n_fields), an empty
 * value, repeated field names, end_ms < start_ms or a bad mode (decided on the device before any kernel reads bytes through
 * the offsets); CCO_E_UNSUPPORTED for more than CCO_MAX_RANKINGS rankings or rows + property triples + ranking events >= 2^31.
 */
typedef struct {
  int64_t n;                      /* (item, field, value) triples; a repeated (item, field) pair: the last triple wins */
  const int64_t *item_offsets;    /* [n + 1] item id t = item_bytes[item_offsets[t] .. item_offsets[t + 1]) */
  const char *item_bytes;
  const int32_t *field;           /* [n] index into field_names */
  const int64_t *value_offsets;   /* [n + 1] JSON text of value t, not empty */
  const char *value_bytes;
  int32_t n_fields;
  const char *const *field_names; /* [n_fields] distinct, NUL-terminated UTF-8 */
} cco_item_properties_t;
typedef struct {                  /* the events of one event name: target item ids and event times */
  int64_t n_events;
  const int64_t *item_offsets;    /* [n_events + 1] */
  const char *item_bytes;
  const int64_t *time_ms;         /* [n_events] epoch milliseconds */
} cco_ranking_stream_t;
typedef struct {                  /* one PopModel ranking over [start_ms, end_ms) of its streams, as cco_pop_model */
  const char *name;               /* the document field */
  int32_t mode;                   /* CCO_POP_*, CCO_POP_RANDOM included */
  int32_t n_streams;              /* >= 1 */
  int64_t start_ms, end_ms;
  const cco_ranking_stream_t *streams;
} cco_ranking_t;
#define CCO_MAX_RANKINGS 8
int cco_format_model(cco_ctx_t *ctx, const cco_result_t *res, int32_t n_names, const char *const *names,
                     const cco_dictionary_t *row_ids, const cco_dictionary_t *col_ids, const cco_item_properties_t *props /* nullable */,
                     int32_t n_rankings, const cco_ranking_t *rankings, char **out_bytes, int64_t *out_len);

/*
 * The rankings of an existing model index refreshed (calcPop, URAlgorithm.scala:375-399, recsModel "backfill"): the caller
 * reads the index and passes it as a bulk body such as cco_format_model writes; the body is parsed on the device and every
 * document gets the fresh rankings and properties, joined by item id the way cco_format_model joins them.  The rankings
 * and properties are those of cco_format_model, with its host and device checks; a random ranking covers the items of its
 * events and the property items, not the items found only in the old index.
 * Accepted body: lines ending in '\n' (an empty body has no documents), in (action, source) pairs.  The action is a JSON
 * object with exactly one member, "index", whose value is an object with a string member "_id" (the last "_id" if it
 * repeats; other members such as "_index" are ignored).  The source is a JSON object.  JSON whitespace, '\r' included, may
 * stand between tokens.  Strings must be closed and hold valid escapes and no raw byte < 0x20; scalars and the inside of
 * values are not validated further.  Names are compared decoded (\uXXXX, surrogate pairs, \/ ...); names and values of the
 * old documents are spliced verbatim.
 * Precedence per document, lowest to highest: fresh properties < members of the old document < rankings (a later ranking
 * beats an earlier one of the same name) < "id".  So a fresh property loses to an old member of the same name, and an old
 * rank member survives when the item has no score in that ranking.  Where a member name repeats, the last one wins.
 * Documents: the old ones in body order, then the items without an old document that have a property or a score, in order
 * of first appearance (property items first, then the ranking streams in order), written as cco_format_model writes them.
 * Fields of an old document: "id" (the decoded _id, escaped as every id), the old members in their order except "id", those
 * named like a ranking present for the item and those followed by a member of the same name, then the properties in field
 * index order except those named "id", like an old member or like a present ranking, then the rankings in order.
 *     {"index":{"_id":"<id>"}}\n{"id":"<id>"[,<old member>]*[,"<field>":<value>]*[,"<ranking>":<number>]*}\n
 * Errors: CCO_E_INVALID_ARG for an odd number of lines, a missing final newline, unbalanced brackets, an unterminated string,
 * a bad escape, an action that is not "index" or has no string "_id", a source that is not an object, an _id in two
 * documents (the message names the 0-based document; decided before anything reads through the parsed spans) and the input
 * errors of cco_format_model; CCO_E_UNSUPPORTED for a line of 2^31 or more bytes, 2^31 - 1 or more members in the body,
 * documents + property triples + ranking events >= 2^31, and group contexts.  out_bytes: pinned memory owned by the context,
 * released with cco_host_free.
 */
int cco_rerank_model(cco_ctx_t *ctx, const char *body, int64_t body_len, const cco_item_properties_t *props /* nullable */,
                     int32_t n_rankings, const cco_ranking_t *rankings, char **out_bytes, int64_t *out_len);

/*
 * A PredictionIO event export read on the device: the DataSource of the reference (DataSource.scala:65-102) and the event
 * reads of PopModel (PopModel.scala:184-195) over the interchange format `pio export` writes and `pio import` reads, JSON
 * lines, one event per line.  Reading the event store stays with the caller.  cco_event_log_read makes one host -> device
 * copy of the export and parses it there into a resident log (per-GPU contexts only, as every resident dataset):
 *  - lines end in '\n' (the last one may not); a '\r' before it is JSON whitespace; every line is one JSON object (a blank
 *    line is an error);
 *  - members read: "event", "entityType", "entityId", "eventTime" (strings, required), "targetEntityType" and
 *    "targetEntityId" (strings, null or absent; given together or not at all), "properties" (an object or absent); every
 *    other member is ignored.  Names are compared decoded; where a name repeats, the last one wins.  Strings are decoded
 *    (\uXXXX, surrogate pairs, short escapes), so ids compare as cco_ingest_strings compares them;
 *  - eventTime: Joda's extended date-time YYYY-MM-DDThh:mm:ss, an optional fraction of 1-9 digits (digits past the third
 *    are dropped: a floor on the time line), then Z, +hh:mm, +hhmm or +hh (sign + or -; the offset is subtracted); years
 *    0000-9999 of the proleptic Gregorian calendar, times before 1970 included;
 *  - training events (DataSource.scala:72-89): entityType "user" and targetEntityType "item", grouped by event name; an
 *    empty entityId or targetEntityId there is an error ("Empty user or item ID");
 *  - ranking events (PopModel.eventsRDD): every event with a targetEntityId, of any entity types, by event name;
 *  - property events: "$set", "$unset" and "$delete" with entityType "item", aggregated on the device as
 *    PEventStore.aggregateProperties does, in (eventTime, line) order -- ties go to the later line, the store's order for
 *    them being undefined: a $set merges its members (a later value of a field wins), a $unset removes the fields it
 *    names, a $delete drops what the item had.  An item whose final state exists keeps a document even without a field
 *    (an "id"-only one, and a random-rank candidate), as the reference's fieldsRDD lists it.  Values are the members'
 *    trimmed JSON text, spliced verbatim (the reference re-serialises them: number spellings and strings under a ranking
 *    name may differ).  Items are in order of their first property event, an item's fields in the order their names
 *    first appear among the members of $set / $unset properties;
 *  - every other line is counted and ignored.
 * Errors: CCO_E_INVALID_ARG for malformed JSON (nested values are checked for closed strings, valid escapes and bracket
 * balance only, as in cco_rerank_model), a missing or mistyped member, a bad time or an empty training id -- the message
 * names the first bad 0-based line, and the verdict comes before any kernel reads through the parsed spans;
 * CCO_E_UNSUPPORTED for more than 2^31 - 1 lines in one parsed chunk (see below; the whole of cco_event_log_read is one),
 * a line of 2^31 or more bytes, 2^31 - 1 or more ranking events of one name, 2^31 - 1 or more property members, and group
 * contexts.  Training events of one name are limited to < 2^31 by the ingest.  A log belongs to its context: free it
 * before cco_destroy of that context.
 *
 * Streamed reading: a log can be built from any split of the export's bytes, for exports larger than device or host
 * memory and for the part files `pio export` writes.  The result -- info, ingest, format and rerank -- is identical to
 * cco_event_log_read of the concatenated bytes, and so is the error code of a failed read; when exactly one line is bad
 * the message is the same and names the same global 0-based line.  When several lines are bad, a streamed log may name a
 * different one than the whole read: chunks are judged in order, each completely before the next.
 *  - cco_event_log_begin: an empty log with chunk_bytes of device staging.
 *  - cco_event_log_append: any number of bytes at any split point (mid-line, mid-escape, mid-UTF-8 sequence, between
 *    '\r' and '\n'); returns once they are copied, so the caller may reuse its buffer.  Whenever the staging is full its
 *    complete lines are parsed as one chunk and the unfinished line is carried to the next; a line longer than the
 *    staging doubles it.  Global line numbers are 64-bit: the 2^31 - 1 line limit holds per chunk.
 *  - cco_event_log_finish: parses the carried tail as the last line (which need not end in '\n'), lays the columns out
 *    and aggregates the properties.  Only then do info, ingest, format_model_log and rerank_model_log accept the log.
 * Before finish those return CCO_E_INVALID_ARG; after a failed append or finish every call but free returns
 * CCO_E_INVALID_ARG with the failure's message.  cco_event_log_read is begin(len) + append + finish.
 */
typedef struct cco_event_log cco_event_log_t;
int cco_event_log_read(cco_ctx_t *ctx, const char *bytes, int64_t len, cco_event_log_t **out);
int cco_event_log_begin(cco_ctx_t *ctx, int64_t chunk_bytes, cco_event_log_t **out);
int cco_event_log_append(cco_event_log_t *log, const char *bytes, int64_t len);
int cco_event_log_finish(cco_event_log_t *log);
typedef struct {
  int64_t n_lines;
  cco_dictionary_t names;          /* the distinct event names, in order of first appearance (owned by the log) */
  const int64_t *n_training;       /* [names.n] training events of each name */
  const int64_t *n_ranking;        /* [names.n] ranking events of each name */
  int64_t n_property_events;       /* $set / $unset / $delete events of items */
  int64_t n_property_items;        /* items whose final state exists (each gets a document) */
  int64_t n_property_fields;       /* distinct fields of the aggregated properties */
  int64_t n_ignored;               /* lines that are none of training, ranking or property events */
} cco_event_log_info_t;
/* arrays owned by the log, valid until cco_event_log_free */
int cco_event_log_info(const cco_event_log_t *log, cco_event_log_info_t *out);
/* cco_ingest_strings on the log's training events of the given names (type t = names[t]; a name without events is an
 * empty type): the same dataset and dictionaries as cco_ingest_strings on those columns, built from the columns in HBM. */
int cco_event_log_ingest(cco_ctx_t *ctx, const cco_event_log_t *log, int32_t n_names, const char *const *names, int32_t min_events_per_user,
                         cco_dataset_t **out);
typedef struct {                   /* a ranking over the log's ranking events: cco_ranking_t with event names for streams */
  const char *name;
  int32_t mode;                    /* CCO_POP_*; CCO_POP_RANDOM reads every event name of the log, in order of first appearance */
  int32_t n_event_names;           /* one stream per name (ignored when random); a name the log does not hold: an empty stream */
  int64_t start_ms, end_ms;
  const char *const *event_names;
} cco_log_ranking_t;
/* cco_format_model / cco_rerank_model with the properties aggregated from the log and the ranking streams read from it,
 * all in HBM (each stream: one event name's ranking events in line order).  Same documents, checks and errors; the log
 * must come from the same context. */
int cco_format_model_log(cco_ctx_t *ctx, const cco_result_t *res, int32_t n_names, const char *const *names,
                         const cco_dictionary_t *row_ids, const cco_dictionary_t *col_ids, const cco_event_log_t *log, int32_t n_rankings,
                         const cco_log_ranking_t *rankings, char **out_bytes, int64_t *out_len);
int cco_rerank_model_log(cco_ctx_t *ctx, const char *body, int64_t body_len, const cco_event_log_t *log, int32_t n_rankings,
                         const cco_log_ranking_t *rankings, char **out_bytes, int64_t *out_len);
int cco_event_log_free(cco_event_log_t *log);

/*
 * The DataSource's eventWindow (engine.json datasource.params.eventWindow, DataSource.scala:39,55,69-70): PredictionIO's
 * SelfCleaningDataSource cleans the event store before the training read, the property aggregation and PopModel's reads,
 * so all three selections see only the cleaned events.  Its rules, restated from PredictionIO 0.12's cleanPEvents
 * [RECALL, unverifiable here], in this order:
 *  - expiry (cutoff_ms > INT64_MIN): an event is kept iff eventTime > cutoff_ms (strictly), or its event is "$set" or
 *    "$unset" whatever its time.  A "$delete" is not exempt: an expired one is dropped, so the $sets before it count again.
 *    The caller computes cutoff_ms = now - Duration(duration).toMillis; the library parses no duration string;
 *  - compressProperties is assumed to preserve what aggregateProperties returns: it has no field here;
 *  - remove_duplicates: events equal in everything but eventId, eventTime and creationTime collapse to one, the one with
 *    the latest eventTime, ties to the later line (PredictionIO keeps an arbitrary one).  The identity: event, entityType,
 *    entityId, targetEntityType, targetEntityId and prId as decoded strings (null = absent), the text of tags (absent, null
 *    = []) and the properties as the set of their top-level members (decoded name, trimmed value text, the last of a
 *    repeated name; absent = {}).  Nested values compare by their trimmed text, where json4s compares numbers by value and
 *    objects without regard to member order; a `pio export` spells equal values alike, but for the member order of nested
 *    objects.  Since the bytes of earlier chunks are gone by finish, the identity is a 128-bit hash: two of n distinct
 *    events collide with probability about n^2 / 2^129 (10^-21 at 10^9 lines).
 * Parsing and checks are unchanged: an expired or duplicate line that is malformed fails as before, naming its line.  With
 * w == NULL (cco_event_log_begin) every output is identical to a read without the window.  info counts after the window:
 * expired and duplicate lines are in no count but the stats (n_lines still counts every line).  Any split of the bytes
 * gives the same log and stats, duplicates across chunks included.  The cleaned events are not written back.
 */
typedef struct {
  int64_t cutoff_ms;               /* INT64_MIN: nothing expires */
  int32_t remove_duplicates;       /* 0 or 1 */
  int32_t reserved;                /* 0 */
} cco_event_window_t;
int cco_event_log_begin_window(cco_ctx_t *ctx, int64_t chunk_bytes, const cco_event_window_t *w /* nullable */, cco_event_log_t **out);
/* after finish: the lines the window dropped as expired and as duplicates */
int cco_event_log_window_stats(const cco_event_log_t *log, int64_t *n_expired, int64_t *n_duplicates);

/*
 * User queries from the log (URAlgorithm.buildQuery for Query.user, URAlgorithm.scala:563-839): one Elasticsearch query per
 * user, built from the user's training events in HBM instead of one LEventStore.findByEntity read per user.
 *
 * History retention: cco_event_log_begin_ex with CCO_LOG_KEEP_HISTORY keeps each training event's eventTime and global
 * 0-based line next to the user and item columns (16 bytes per training event).  A log read without it is what
 * cco_event_log_begin_window reads, byte for byte and in device memory.  w as in cco_event_log_begin_window.
 */
enum { CCO_LOG_KEEP_HISTORY = 1 };
int cco_event_log_begin_ex(cco_ctx_t *ctx, int64_t chunk_bytes, const cco_event_window_t *w /* nullable */, uint32_t flags,
                           cco_event_log_t **out);
/*
 * The query of user u, for the query event names n_0 .. n_{k-1}:
 *  - history of n_q: u's training events of n_q, latest first (eventTime desc, ties to the later line), the first limits[q]
 *    of them reversed (oldest first), repeated items kept at their first position;
 *  - blacklist: the items of every training event of u whose name is among the names and the blacklist names, latest
 *    first, then the blacklist items, each item once (its first position);
 *  - the body record:  header \n head ,"query":{"bool":{"should":[S],"must":[M],"must_not":[{"ids":{"values":[blacklist],
 *    "boost":0}}(,must_not)?],"minimum_should_match":1}},"sort":sort} \n
 *    where the terms of the first n_history_names names, {"terms":{"<n_q>":[history],"boost":<boost>}} (without "boost" when
 *    boost is NULL) or {"terms":{"<n_q>":[history],"boost":0}} in must, come before the `should` (or `must`) fragment, all
 *    comma-separated.  Ids and names are escaped as json4s 3.2 quotes strings: '"' and '\' get a backslash, \b \f \n \r \t
 *    their short forms, every other code point below U+0020, in U+0080..U+009F and in U+2000..U+20FF \u%04x in lowercase.
 * Fragments are JSON text spliced verbatim: head ({"from":F,"size":N), should (must not be empty: the reference ends should
 * with a constant_score clause), must, must_not (may be empty), sort (an array), header (one _msearch header line).
 * Users: n_users ids in the Arrow large_string layout (a repeated or unknown user gets its record, an unknown one with an
 * empty history), or user_offsets == NULL: every user with a training event of a query name, in order of their first such
 * line; *out_users then lists them (pinned offsets and bytes, each released with cco_host_free; nullable otherwise).
 * Out: *out_body [*out_len] and *out_offsets [*out_n + 1] (record r = body[offsets[r] .. offsets[r + 1])), pinned memory
 * owned by the context, each released with cco_host_free.
 * Errors: CCO_E_INVALID_ARG for bad offsets in either column (decided on the device before any kernel reads bytes through
 * them), null or empty names, negative limits, n_history_names outside [0, n_names], a null fragment, more than 64 names and
 * a log read without CCO_LOG_KEEP_HISTORY; CCO_E_UNSUPPORTED for group contexts, 2^31 or more events of the names and a
 * record of 2^31 or more bytes.  A name the log does not hold has no history.
 */
typedef struct {
  int32_t n_names;
  int32_t n_history_names;           /* maxQueryEvents - 1 clamped to [0, n_names] */
  const char *const *names;          /* [n_names] the query event names */
  const int32_t *limits;             /* [n_names] history limit per name (maxItemsPerUser) */
  int32_t n_blacklist_names;
  int32_t history_in_must;           /* 0: should (userBias >= 0), 1: must (userBias < 0) */
  const char *const *blacklist_names;
  const char *boost;                 /* JSON number text or NULL */
  const char *head, *should, *must, *must_not, *sort, *header;
  int64_t n_blacklist_items;
  const int64_t *blacklist_item_offsets; /* [n + 1] */
  const char *blacklist_item_bytes;
} cco_user_query_t;
int cco_event_log_user_queries(cco_ctx_t *ctx, const cco_event_log_t *log, const cco_user_query_t *q, int64_t n_users,
                               const int64_t *user_offsets /* nullable: every user */, const char *user_bytes, char **out_body,
                               int64_t *out_len, int64_t **out_offsets, int64_t *out_n, cco_dictionary_t *out_users /* nullable */);

/*
 * Item queries from a model index (URAlgorithm.buildQuery for Query.item, user and itemSet absent, URAlgorithm.scala:563-792):
 * one Elasticsearch query per item, its similar items read from the index body instead of one EsClient.getSource round
 * trip per item.  index_body is an Elasticsearch bulk body as cco_format_model, cco_format_model_log and cco_rerank_model
 * write it, with cco_rerank_model's grammar, checks and messages (actions {"index":{..., "_id":"<string>"}}, sources JSON
 * objects, names compared decoded, the last of a repeated member name wins).
 *  - Documents by _id: a requested item matches the document whose decoded _id has the same bytes (UTF-8; a lone surrogate
 *    in its 3-byte form).  item_offsets == NULL: one record per document, in body order; *out_items then lists their
 *    decoded _ids (pinned offsets and bytes, each released with cco_host_free; nullable otherwise).  A repeated item gets a
 *    record each time.
 *  - Similar items: when the item has a document whose source has at least one member, one clause per model event name
 *    n_j, {"terms":{"<n_j>":[elements]}}, where the elements are those of the source's last member named n_j, which must be
 *    '[' string (',' string)* ']' or '[]' (JSON whitespace between tokens); a source without that member gives [].  A list
 *    of at most max_query_events elements is kept whole, a longer one keeps its first max_query_events - 1.  The clause ends
 *    in ,"boost":<similar_boost> when similar_boost is not NULL; with similar_in_must the clauses go to must instead, each
 *    with ,"boost":0.  An unknown item, or a document whose source is {}, has no similar-items clause.
 *  - Excluded ids: blacklistItems in order, each once, then the item itself when exclude_self and it is not among them.
 *  - The body record:
 *      header \n head ,"query":{"bool":{"should":[should_head, SIMILAR?, should],"must":[must_head, SIMILAR?, must],
 *      "must_not":[{"ids":{"values":[excluded],"boost":0}}(,must_not)?],"minimum_should_match":1}},"sort":sort} \n
 *    where SIMILAR stands in should unless similar_in_must, and in must then; the elements of each list are comma-separated
 *    and an empty piece leaves no comma.  Ids, elements and names are escaped as in cco_event_log_user_queries.
 * Fragments are JSON text spliced verbatim: head ({"from":F,"size":N), should_head / must_head (the clauses before the
 * similar items, e.g. buildQuery's empty user-history clauses; may be empty), should, must, must_not (may be empty), sort
 * (an array), header (one _msearch header line).  Items: n_items ids in the Arrow large_string layout.
 * Out: *out_body [*out_len] and *out_offsets [*out_n + 1] (record r = body[offsets[r] .. offsets[r + 1])), pinned memory
 * owned by the context, each released with cco_host_free.
 * Errors: CCO_E_INVALID_ARG for everything cco_rerank_model refuses in the body (same messages), an _id in two documents,
 * bad offsets in the items or the blacklist items (decided on the device before any kernel reads bytes through them), null
 * or empty names, more than 64 names, a null fragment, max_query_events < 1, and a queried document whose model-name
 * member is not an array of strings (the message names the 0-based document and the member; decided before anything reads
 * through the elements; an unqueried document is not checked); CCO_E_UNSUPPORTED for group contexts, documents + items +
 * blacklist items >= 2^31 and a record of 2^31 or more bytes.
 */
typedef struct {
  int32_t n_names;
  const char *const *names;          /* [n_names] the model event names = the index's indicator fields */
  int32_t max_query_events;          /* a longer list keeps its first max_query_events - 1 */
  int32_t similar_in_must;           /* 0: should (algorithm itemBias >= 0), 1: must (itemBias < 0) */
  const char *similar_boost;         /* JSON number text or NULL */
  int32_t exclude_self;              /* 1: the item is excluded (!returnSelf) */
  const char *head, *should_head, *should, *must_head, *must, *must_not, *sort, *header;  /* *_head may be "" */
  int64_t n_blacklist_items;
  const int64_t *blacklist_item_offsets; /* [n + 1] */
  const char *blacklist_item_bytes;
} cco_item_query_t;
int cco_item_queries(cco_ctx_t *ctx, const char *index_body, int64_t index_len, const cco_item_query_t *q, int64_t n_items,
                     const int64_t *item_offsets /* nullable: every document */, const char *item_bytes, char **out_body,
                     int64_t *out_len, int64_t **out_offsets, int64_t *out_n, cco_dictionary_t *out_items /* nullable */);

/*
 * Debug/parity entry (tests only): full integer co-occurrence matrix A^T B of two canonical
 * binary matrices computed by the same accumulation kernel as cco_train, no LLR, no top-k.
 * Output CSR over the columns of A with ascending column ids, malloc'ed; free with cco_free.
 */
int cco_debug_cooccurrence(cco_ctx_t *ctx, const cco_csr_t *a, const cco_csr_t *b, int64_t **row_ptr,
                           int32_t **col_idx, int32_t **count);
/* Debug/parity entry (tests only): sampleDownAndBinarize of one matrix on the device. */
int cco_debug_downsample(cco_ctx_t *ctx, const cco_csr_t *m, int32_t max_interactions, int32_t seed,
                         uint32_t flags, int64_t **row_ptr, int32_t **col_idx, int32_t *raw_col_counts,
                         int32_t *new_col_counts);
/* Debug/parity entry (tests only): one rank's share of the multi-GPU sampleDownAndBinarize, on one GPU.  The whole
 * matrix is uploaded (and canonicalised unless CCO_FLAG_ASSUME_CANONICAL); the users [row_lo, row_hi) are then sampled
 * as the rank owning that block samples them: by global user id, with raw_col_counts[n_cols] as the column counts (the
 * whole matrix's, as the all-reduce of the ranks' histograms gives them).  Out: kept_per_row[n_rows] (indexed by global
 * user, zero outside the block), *col_idx = the block's kept columns in order (as many as the block's kept counts sum
 * to, malloc'ed, free with cco_free), new_col_counts[n_cols] = the block's share of the post-sample column counts. */
int cco_debug_downsample_block(cco_ctx_t *ctx, const cco_csr_t *m, int64_t row_lo, int64_t row_hi,
                               const int32_t *raw_col_counts, int32_t max_interactions, int32_t seed, uint32_t flags,
                               int64_t *kept_per_row, int32_t **col_idx, int32_t *new_col_counts);
/* Debug/parity entry (tests only): the device LLR of n cells. */
int cco_debug_llr(cco_ctx_t *ctx, int64_t n, const int64_t *k11, const int64_t *k12, const int64_t *k21,
                  const int64_t *k22, uint32_t flags, double *out);
/* Debug/parity entry (tests only): the string-dictionary stage of cco_ingest_strings on one column, with the hash
 * truncated to hash_bits (0..64) bits so that distinct ids collide on purpose.  ids[e] = dictionary id of id e, the
 * dictionary ordered by first appearance; the result is the same for every hash_bits. */
int cco_debug_string_ids(cco_ctx_t *ctx, int64_t n, const int64_t *offsets, const char *bytes, int32_t hash_bits, int32_t *ids);
/* Debug/parity entry (tests only): the rank number text of cco_format_model, Java's Double.toString of v[i] * 10^-scale,
 * written by the device routine the document kernels call, once per value.  scale 0 (a histogram rank: |v[i]| < 2^53) or
 * 15 (a random rank: 0 <= v[i] < 10^15).  Text i = bytes[offsets[i] .. offsets[i + 1]), offsets[0] = 0; offsets holds
 * n + 1 entries and bytes 32 * n bytes, both the caller's (a text is at most 25 bytes long). */
int cco_debug_rank_text(cco_ctx_t *ctx, int64_t n, const int64_t *v, int32_t scale, int64_t *offsets, char *bytes);
void cco_free(void *p);

#ifdef __cplusplus
}
#endif
#endif /* CCO_B200_H */
