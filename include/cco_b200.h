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
 *    allows counts < 4096.  Without CCO_FLAG_KEY_RANGES an indicator past this bound is refused (CCO_E_UNSUPPORTED,
 *    the remedy named: lower maxItemsPerUser / maxEventsPerEventType); with it, the indicator is trained in column key
 *    ranges that each fit the word, bit for bit the result an unlimited word would give (see the flag).
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
  CCO_FLAG_RESULT_NO_LLR = 32,
  /* An indicator whose counts do not fit the packed accumulator word ("Limits") is trained in key ranges instead of
   * being refused: the columns, numbered by (colB ascending, column id ascending), are cut into the fewest contiguous
   * ranges whose counts fit, each range is scored on its own and the ranges' top-k lists are merged on the device.  The
   * result is bit for bit the unsplit one (LLR depends only on k11, colA, colB and N; ties keep the column-id order).
   * A flag, not automatic: the refusal is a documented contract, and without downsampling the number of ranges has no
   * useful bound (counts of 2^20 leave 12 key bits per range, each range a pass over B'), so the caller accepts that
   * cost.  Indicators whose word fits run exactly as without the flag.  Honoured by cco_train, cco_train_dataset,
   * cco_cooccurrences_idss, group contexts and multi-process ranks (every rank cuts the same plan).
   * llr_evaluated may differ from the unsplit run: the key cut and the dominance filter work per range. */
  CCO_FLAG_KEY_RANGES = 64
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
/* the number of key ranges indicator i ran in (CCO_FLAG_KEY_RANGES): 1 when its counts fit the packed word */
int cco_result_key_ranges(const cco_result_t *r, int32_t i, int32_t *n_ranges);
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
enum { CCO_LOG_KEEP_HISTORY = 1, CCO_LOG_EXTENDABLE = 2 };
int cco_event_log_begin_ex(cco_ctx_t *ctx, int64_t chunk_bytes, const cco_event_window_t *w /* nullable */, uint32_t flags,
                           cco_event_log_t **out);

/*
 * Extendable logs: a resident log that takes the newest lines of an export and a later cutoff without a re-read, for a
 * trainer that retrains on a schedule with a sliding eventWindow.  cco_event_log_begin_ex with CCO_LOG_EXTENDABLE (it
 * combines with CCO_LOG_KEEP_HISTORY) keeps, besides what the log holds anyway: each retained line's record (40 bytes:
 * its identity hash under remove_duplicates, eventTime, global line, name and selection), the global line of each
 * training and ranking entry (8 bytes each), the retained property-event lines (their bytes) and, under
 * remove_duplicates, the eventTime of each line dropped as a duplicate whose event is neither $set nor $unset (8 bytes).
 * A log read without the flag is what cco_event_log_begin_ex reads without it, byte for byte and in device memory.
 *
 * cco_event_log_extend reopens a finished extendable log for cco_event_log_append / cco_event_log_finish, staged in the
 * chunk_bytes the log was begun with; w == NULL keeps the current window.  Reading bytes A with window w1, then
 * extending with w2 and appending bytes B, gives after finish the log one read of A followed by B under w2 gives: info,
 * window_stats and every consumer's output (ingest, format_model_log, rerank_model_log, user_queries, mixed_queries,
 * query_file_queries).  B's first byte starts a line, as if A ended in '\n'; B's lines are numbered after A's, in
 * messages, in the (eventTime, line) rules and in history order.  Extends compose; one with no bytes only slides the
 * window.  Expiry comes first, then removeDuplicates (cco_event_log_begin_window), and three consequences follow:
 *  - duplicates across the seam: a line of B can drop a retained line of A, or be dropped for it, in either time order;
 *    at equal eventTime the later line, B's, stays.  So the record of every retained line survives finish, ignored and
 *    property-event lines included, since the counts of info name them;
 *  - stats re-attribution: a line dropped as a duplicate under the old cutoff whose eventTime is at or before the new one
 *    (and whose event is neither $set nor $unset) is an expired line for a whole read under the new cutoff; it moves from
 *    the duplicates to the expired lines of window_stats;
 *  - properties: a $delete that expires under the new cutoff lets the $sets before it count again, so the retained
 *    property-event lines stay resident and the aggregation runs again at every finish over old and new lines.  $set
 *    and $unset never expire.
 * All of it is exact because cutoffs only move forward: a line dropped under w1 is dropped under w2.  At finish only B
 * is parsed; the retained records, entries and property lines at or before the new cutoff are dropped and freed, the
 * retained records are deduplicated together with B's (one sort of all of them: the three 64-bit passes of removeDuplicates,
 * O(retained + new) per finish), the columns are concatenated name-major (the retained layout first, names new in B
 * after) and compacted, and the properties are aggregated again.
 * Errors: CCO_E_INVALID_ARG for a null log, a log read without CCO_LOG_EXTENDABLE, a log not finished or failed, a cutoff
 * below the current one, a remove_duplicates other than the first read's and a nonzero reserved field.  A failed append
 * or finish during an extend fails the log as it does any read: its resident state is lost, and every call but free
 * returns CCO_E_INVALID_ARG with the failure's message.
 * cco_event_log_resident_bytes: the device bytes a finished log holds (bounded by its retained lines, not by every line
 * ever appended).
 */
int cco_event_log_extend(cco_event_log_t *log, const cco_event_window_t *w /* nullable: keep the current window */);
int cco_event_log_resident_bytes(const cco_event_log_t *log, int64_t *bytes);

/*
 * Interned logs: retrains from a resident log at a cost set by its new lines plus integer passes.  cco_event_log_begin_ex
 * with CCO_LOG_INTERN_IDS (it combines with CCO_LOG_KEEP_HISTORY, CCO_LOG_EXTENDABLE and a window) gives every distinct
 * user id and item id of the training entries a 32-bit key as the lines are read: one table for the users (entityId),
 * one for the items (targetEntityId, shared by every event name).  Each chunk, and each extend, interns only its own
 * lines, and cco_event_log_ingest on the log then groups keys instead of strings.
 *
 * The invariant: for any export, window, chunking and sequence of extends, cco_event_log_ingest of an interned log, with
 * any names and any min_events_per_user, gives the dataset the same lines read once without the flag under the same
 * final window give -- the same dictionaries byte for byte and in the same order, the same matrices.  Every other
 * consumer (info, window_stats, format_model_log, rerank_model_log, user and mixed queries, query files,
 * refresh_properties_log) gives what it gives on that log.  After every finish, of a read or of an extend, the tables
 * hold exactly the distinct ids of the retained training entries (those of expired and duplicate lines are gone), and
 * their sizes are a fixed function of those counts and bytes: an extended interned log and a fresh interned extendable
 * read of the same lines hold the same bytes.  Key numbering is internal.
 *
 * Added device memory: 8 bytes per retained training entry (its user and item keys), and per table 24 to 32 bytes per
 * key (its string offset and hash, 8 bytes each, and 2 to 4 table slots of 4 bytes; at least 64 slots) plus the keys'
 * string bytes and 16 bytes of padding.
 *
 * cco_event_log_intern_stats: the live key counts of a finished interned log.  Errors: CCO_E_INVALID_ARG for a null
 * argument, a log not finished or failed, and a log read without CCO_LOG_INTERN_IDS; CCO_E_UNSUPPORTED for 2^31 or more
 * distinct ids in one table; group contexts refuse logs as before.
 */
enum { CCO_LOG_INTERN_IDS = 4 };
int cco_event_log_intern_stats(const cco_event_log_t *log, int64_t *n_user_keys, int64_t *n_item_keys);

/*
 * Snapshots: a finished log saved as one binary image and loaded back, so that a trainer restarts (after a deploy, a crash,
 * or on another GPU machine) without reading its export again.  The loaded log is the saved one: info, window_stats,
 * resident_bytes, intern_stats and every consumer's output are equal, and a loaded extendable log extends as the saved
 * one would.  Both sides stream in chunks, so neither needs the whole image in host memory.
 *  - cco_event_log_save_size: the image's exact length.  The image is built at the first save call after a finish
 *    (a hash pass over the device sections) and kept until the log is extended or freed.
 *  - cco_event_log_save: bytes [offset, offset + len) of the image into dst, any split; the device sections are copied on
 *    the context's copy stream through its pinned staging.
 *  - cco_event_log_load_begin / _append / _finish: a new log from the image's bytes, any split.  The sections are copied
 *    into their device buffers as they arrive; finish checks the whole image and builds the log.
 * Refused with CCO_E_INVALID_ARG: saving a log that is not finished or has failed.
 *
 * Layout (version CCO_SNAPSHOT_VERSION; integers little-endian; offsets from the image's first byte):
 *  - header, bytes [0, 64): the magic "CCOLOGSN" (8 bytes); u32 format version; u32 CCO_ABI_VERSION; u32 n_sections;
 *    u32 0; i64 total bytes; u64 the checksum of bytes [0, 64 + 40 n_sections) with these 8 bytes read as 0; 24 bytes 0.
 *  - section table, bytes [64, 64 + 40 n_sections): per section u32 kind; u32 0; i64 offset; i64 length; i64 device
 *    bytes (the buffer the loader allocates for it: its length plus the log's padding or growth room; 0 for a host
 *    section); u64 checksum.  Kinds ascend; offsets are multiples of 256 and sections do not overlap the table or each
 *    other; the last section ends at the total.  Bytes between sections are padding (zero when saved, not read).
 *  - checksum of n bytes: mix(n) + sum over words i of mix(w_i ^ (i * 0x9e3779b97f4a7c15)) mod 2^64, w_i the i-th 8-byte
 *    word (the last one zero-filled) and mix splitmix64's finaliser (x ^= x >> 30; x *= 0xbf58476d1ce4e5b9; x ^= x >> 27;
 *    x *= 0x94d049bb133111eb; x ^= x >> 31).
 *  - host sections (lists of strings: i64 n, i64 offsets [n + 1] from 0, the bytes):
 *      1 state: 16 i64: flags (CCO_LOG_*), remove_duplicates, cutoff_ms, chunk_bytes, n_lines, property events, ignored
 *        lines, property items, property fields, expired lines, duplicate lines, the intern hash mask, erased lines
 *        (cco_event_log_erased, >= 0; a reserved zero before erasure existed, so a library older than it refuses an image
 *        with erased lines: "a counter is out of range"), 3 zeros;
 *      2 names: the event names (a string list); 3 counts: training then ranking events per name (i64 each);
 *      4 fields: the aggregated properties' field names (a string list);
 *      5 property_lines: the global line of each retained property-event line (i64; CCO_LOG_EXTENDABLE).
 *  - device sections, present where the log holds the buffer (string columns: i64 offsets [n + 1] from 0 and the bytes):
 *      6-11 the training users, training items and ranking items (name-major, file order inside a name); 12 rank_times;
 *      13 train_lines (KEEP_HISTORY or EXTENDABLE); 14 rank_lines (EXTENDABLE); 15 train_times (KEEP_HISTORY);
 *      16 train_keys (INTERN_IDS: user key << 32 | item key); 17 records (EXTENDABLE: 40 bytes per retained line);
 *      18 duplicate_times (EXTENDABLE with remove_duplicates); 19 property_bytes (EXTENDABLE: the retained property-event
 *      lines); 20-24 the aggregated properties (i32 field of each triple, value offsets, values, item offsets, item
 *      bytes); 25-26 property_items (the property events' item ids a log without EXTENDABLE keeps); 27-30 the user and
 *      item keys' strings (INTERN_IDS; key k is string k).  The intern hash tables are not stored: the loader rebuilds
 *      them from the strings, so a snapshot of a log is independent of where its tables placed the keys.
 *
 * A snapshot is untrusted input: every damaged or inconsistent image is refused with CCO_E_INVALID_ARG and a message that
 * names the header or the section, and no kernel reads a byte through a stored offset before the host has the verdict
 * on it.  Refused: a wrong magic, format version or ABI version; a section table out of order, overlapping or past the
 * end; bytes past the end; an image shorter than its total at finish; a checksum mismatch; and any structural violation --
 * decreasing offsets or offsets that disagree with their bytes, name or field numbers out of range, keys >= their table's
 * count, an id stored twice in a key table, lines >= the line count, records out of line order, column lengths that
 * disagree with the counts, a section the flags do not allow or a missing one.  A failed load frees the device memory it
 * took; the log then answers every call but free with the failure's message.  CCO_E_UNSUPPORTED: group contexts, as for
 * every log.  A different format version is refused, never converted.
 */
#define CCO_SNAPSHOT_VERSION 1
int cco_event_log_save_size(cco_event_log_t *log, int64_t *bytes);
int cco_event_log_save(cco_event_log_t *log, int64_t offset, void *dst, int64_t len);
int cco_event_log_load_begin(cco_ctx_t *ctx, cco_event_log_t **out);
int cco_event_log_load_append(cco_event_log_t *log, const void *bytes, int64_t len);
int cco_event_log_load_finish(cco_event_log_t *log);

/*
 * Clean write-back: an extendable log's cleaned events written out as a compacted export, the part of PredictionIO's
 * SelfCleaningDataSource.cleanPersistedPEvents that writes the cleaned set back [RECALL, unverifiable here], so that the
 * export a trainer reads stops growing.  The log keeps one record per retained line (CCO_LOG_EXTENDABLE); the cleaner
 * reads the source bytes a second time and copies out exactly those lines, verbatim, each ending in '\n' (a last line or
 * a part without one gets one).  No resident state is added to the log, and the log is unchanged by a clean: its info,
 * window_stats, resident bytes, snapshot image and every consumer's output are the same before and after.
 *  - cco_event_log_clean_begin: a cleaner of a finished extendable log (read, extended or loaded).  It marks the log's
 *    retained lines in a bitmap of one bit per line read, and stages chunks as the log's read did.
 *  - cco_event_log_clean_append: the bytes the log has read, in order -- the first read's source, then each extend's --
 *    split anywhere.  *out / *out_len: the kept lines completed in this append, in pinned memory owned by the cleaner and
 *    valid until its next call.
 *  - cco_event_log_clean_finish: the rest; *stats as below.
 * The contract (events.clean_export is its host statement): reading the output under any later window w' (a cutoff at or
 * after the log's, the same removeDuplicates) gives the training events, the ranking events per name and the aggregated
 * properties that reading the whole source under w' gives, and without compression n_ignored and the order of
 * property-only items as well.
 * CCO_CLEAN_COMPRESS_PROPERTIES (compressProperties) folds, at begin, the $set / $unset lines of each item (entityType
 * "item") whose lines the log retained: an item with a retained $delete, with a $set / $unset that carries a target, or
 * with a single such line keeps its lines verbatim in place; every other item's lines become one line, written at finish
 * after all verbatim lines in the order of each item's first line: a $set of its aggregated state (or, for an item that
 * only unsets, an $unset of the union of the names, each with its last value), eventTime the last folded event's text,
 * strings through json4s' quote, values their trimmed text, no eventId.  Other entity types' lines are never folded: the
 * log keeps only the items' property lines, and no read looks at the others.  The folded lines are the log's own, so the
 * source's property members are not compared with them beyond the record check below.
 * The source is checked against the log as it is read: every line is parsed and checked as a read checks it, and each
 * kept line's eventTime, event name and selection must equal its record, and under remove_duplicates its 128-bit
 * identity too (without remove_duplicates the check does not cover ids, properties or other members).  A mismatch, a
 * line past the log's count, an event name the log did not read and a source that ends short at finish fail the cleaner
 * with CCO_E_INVALID_ARG naming the global 0-based line.
 * Errors: CCO_E_INVALID_ARG for a null argument, a log read without CCO_LOG_EXTENDABLE, not finished or failed, and
 * unknown flags; CCO_E_UNSUPPORTED for group contexts, as for every log.  While a cleaner of a log is open,
 * cco_event_log_extend and cco_event_log_free of the log refuse with CCO_E_INVALID_ARG: a caller frees every cleaner
 * before its log (the log would otherwise stay allocated), and every log before cco_destroy of its context.  A failed cleaner answers every
 * later call but free with its message.
 */
typedef struct cco_event_clean cco_event_clean_t;
enum { CCO_CLEAN_COMPRESS_PROPERTIES = 1 };
typedef struct {
  int64_t n_lines, n_written, n_expired, n_duplicates;   /* lines read; lines out; the log's window_stats */
  int64_t n_folded, n_compressed, n_bytes;               /* property lines folded; lines they became; bytes out (all three
                                                            in the output: n_written counts the lines they became) */
} cco_event_clean_stats_t;
int cco_event_log_clean_begin(cco_event_log_t *log, uint32_t flags, cco_event_clean_t **out);
int cco_event_log_clean_append(cco_event_clean_t *x, const char *bytes, int64_t len, const char **out, int64_t *out_len);
int cco_event_log_clean_finish(cco_event_clean_t *x, const char **out, int64_t *out_len, cco_event_clean_stats_t *stats);
int cco_event_log_clean_free(cco_event_clean_t *x);
/*
 * Erasure: the lines of given users and items taken out of a finished extendable log (read, extended or loaded), for bot
 * and test users, deletion requests and withdrawn products, without a re-read.  events.erased_line is the host statement
 * of which lines go.  A line is erased, whole (its training entry, ranking entry, property line, record and history
 * time), when
 *  1. it is a training event (entityType "user", targetEntityType "item") whose entityId is one of the users;
 *  2. its targetEntityId is one of the items, whatever its types (PopModel reads ranking events by id);
 *  3. it is a property event ($set / $unset / $delete of entityType "item") whose entityId is one of the items.
 * Ids compare decoded, as the log compares them; ids are bytes in the Arrow layout (id i = bytes[offsets[i] - offsets[0],
 * offsets[i + 1] - offsets[0])).  The rule is made of whole removeDuplicates groups (their identity holds entityId and
 * targetEntityId), and from that:
 *  - consumers: erasing set E from a log read from X under window w gives every consumer's output a fresh read of X - E
 *    (the export without E's lines) gives under w: ingest, format_model_log, rerank_model_log, user, mixed and query-file
 *    queries, refresh_properties_log and intern_stats.  An extend after the erase gives what a fresh read of (X - E) + B
 *    gives.  Erasure is not a block list: later extends read new lines of erased ids as any others;
 *  - counters: info's n_lines and window_stats are unchanged by an erase; info's training, ranking and property counts
 *    follow the retained lines; cco_event_log_erased counts the erased lines over the log's life, so that lines read =
 *    retained + expired + duplicates + erased holds for every log and across extends;
 *  - write-back: cco_event_log_clean_* of X after the erase writes events.clean_export(X - E, w, now, compress), byte for
 *    byte, with and without CCO_CLEAN_COMPRESS_PROPERTIES;
 *  - resident bytes: those of the fresh read, plus 8 for each duplicate eventTime the log keeps of a dropped duplicate of
 *    an erased line (the log holds no id for those lines; they still turn into expired lines under a later cutoff).
 * Limits: the log holds no entityId for a user's lines without an item target (a user $set, an event on a "user" or
 * "category" target) nor for lines that name an item only as entityId and are not property events, so these are not
 * erased and a write-back keeps them; a caller who must remove them filters the export.
 * On the device: the ids become two intern tables (users, items; cco_intern.cuh's table, exact byte compares); the
 * training entries are probed by string, or on an interned log by their keys (the ids looked up in the log's tables,
 * then 8 bytes per entry); the ranking entries and the retained property lines' entityIds are probed against the items.
 * The marked lines leave through the extend's finish: records, columns, property lines, aggregation and intern refit.
 * Ids the log does not hold, repeated ids and empty lists are fine; an erase that marks nothing leaves the log bit for
 * bit as it was, its snapshot image included.  Otherwise the saved image is rebuilt at the next save.
 * *stats (nullable): the lines erased, and the training, ranking and property events among them.
 * Errors: CCO_E_INVALID_ARG for a null log, null offsets with a positive count, null bytes with offsets that span bytes,
 * a negative count ("users: a negative count"), offsets[0] < 0 ("items: offsets[0] = -1 is negative"), decreasing
 * offsets ("users: offsets[3] = 2 decreases"), a log read without CCO_LOG_EXTENDABLE, a log not finished or failed, and a
 * log with an open cleaner (as cco_event_log_extend); CCO_E_UNSUPPORTED for group contexts, as for every log.  A failed
 * erase fails the log as a failed extend does.  cco_event_log_erased: CCO_E_INVALID_ARG for a null argument and a log
 * not finished or failed (0 for a log that never erased).
 */
typedef struct {
  int64_t n_lines, n_training, n_ranking, n_property_events;
} cco_event_erase_stats_t;
int cco_event_log_erase(cco_event_log_t *log, int64_t n_users, const int64_t *user_offsets, const char *user_bytes, int64_t n_items,
                        const int64_t *item_offsets, const char *item_bytes, cco_event_erase_stats_t *stats /* nullable */);
int cco_event_log_erased(const cco_event_log_t *log, int64_t *n_erased);
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
 * Item-set queries (URAlgorithm.buildQuery for Query.itemSet, user and item absent, URAlgorithm.scala:563-767): one
 * Elasticsearch query per item set ("shopping cart"), built for a whole batch of sets.  The sets are the caller's input;
 * nothing is read from a model or a history.
 *  - Sets: the Arrow list<large_string> layout.  Set s holds the elements [set_offsets[s], set_offsets[s + 1]) of a
 *    large_string column of n_elements ids; element e = elem_bytes[elem_offsets[e] .. elem_offsets[e + 1]).  Only the
 *    elements [set_offsets[0], set_offsets[n_sets]) are read.
 *  - The set clause, when with_set: {"terms":{"<name>":[elements]}}, the set's elements exactly as given (order and repeats
 *    kept, no slicing), ending in ,"boost":<boost> when boost is not NULL.  It always goes to should.
 *  - Excluded ids: blacklistItems in order, each once, then each element of the set that is not among them and did not
 *    appear earlier in the set (ids compare as bytes).  A repeated element is written twice in the set clause and once here.
 *  - The body record:
 *      header \n head ,"query":{"bool":{"should":[should_head, SET?, should_tail],"must":[must],
 *      "must_not":[{"ids":{"values":[excluded],"boost":0}}(,must_not)?],"minimum_should_match":1}},"sort":sort} \n
 *    where SET stands when with_set; the elements of should are comma-separated and an empty piece leaves no comma.  Ids,
 *    elements and the name are escaped as in cco_event_log_user_queries.
 * Fragments are JSON text spliced verbatim: head ({"from":F,"size":N), should_head (buildQuery's empty user-history clauses
 * when they go to should, then the boosted metadata; may be empty), should_tail (the constant_score clause), must (the
 * empty history clauses when they go to must, the filtering metadata and the date filters; may be empty), must_not (may be
 * empty), sort (an array), header (one _msearch header line).
 * Out: *out_body [*out_len] and *out_offsets [*out_n + 1] (record s = body[offsets[s] .. offsets[s + 1])), pinned memory
 * owned by the context, each released with cco_host_free.
 * Errors: CCO_E_INVALID_ARG for bad offsets in any column (set offsets that decrease or leave [0, n_elements], element or
 * blacklist item offsets that decrease; decided on the device before any kernel reads bytes through them), a null
 * fragment, and a null or empty name while with_set; CCO_E_UNSUPPORTED for group contexts, 2^31 or more sets, elements +
 * blacklist items >= 2^31 and a record of 2^31 or more bytes.
 */
typedef struct {
  const char *name;                  /* the set clause's field: the first model event name (may be NULL without with_set) */
  int32_t with_set;                  /* 0: no set clause (itemSetBias 0), 1: the clause is written */
  const char *boost;                 /* JSON number text or NULL */
  const char *head, *should_head, *should_tail, *must, *must_not, *sort, *header;  /* should_head, must may be "" */
  int64_t n_blacklist_items;
  const int64_t *blacklist_item_offsets; /* [n + 1] */
  const char *blacklist_item_bytes;
} cco_item_set_query_t;
int cco_item_set_queries(cco_ctx_t *ctx, const cco_item_set_query_t *q, int64_t n_sets, const int64_t *set_offsets, int64_t n_elements,
                         const int64_t *elem_offsets, const char *elem_bytes, char **out_body, int64_t *out_len, int64_t **out_offsets,
                         int64_t *out_n);

/*
 * Mixed queries (URAlgorithm.buildQuery for any combination of Query.user, Query.item and Query.itemSet,
 * URAlgorithm.scala:563-839): one Elasticsearch query per row, where each row of the batch may have a user, an item and an
 * item set, or any subset of them.  The batch shares one template.
 *  - Rows: n_rows; three optional columns, each with an optional validity bitmap (Arrow: LSB-first, bit r = 1 when row r
 *    has the member; NULL: every row has it).  A NULL offsets pointer means no row has the member.  users and items are
 *    large_string columns of n_rows ids; sets are list<large_string> as in cco_item_set_queries (set_offsets [n_rows + 1]
 *    into an element column of n_elements ids).  An absent set writes nothing; a present empty set writes [].
 *  - History (the row's user, as in cco_event_log_user_queries, from a log read with CCO_LOG_KEEP_HISTORY): the first
 *    n_history_names names get a terms clause, with the user's list, or [] for a row without a user or with a user the log
 *    does not know.  In should with history_boost (none when NULL), or in must with "boost":0 when history_in_must.
 *  - Similar items (the row's item, as in cco_item_queries, from index_body): one clause per model name when the item has a
 *    document whose source has a member; sliced to max_query_events; in should with similar_boost, or in must with
 *    "boost":0 when similar_in_must.
 *  - The set clause (as in cco_item_set_queries): {"terms":{"<set_name>":[elements]}} with ,"boost":<set_boost> when
 *    set_boost is not NULL, when with_set and the row has a set.
 *  - Excluded ids: the user's blacklisted items (newest first), blacklistItems, the item when exclude_self, the set's
 *    elements; each id once, at its first position (ids compare as bytes).
 *  - The body record:
 *      header \n head ,"query":{"bool":{"should":[HISTORY?, SIMILAR?, boosted, SET?, should_tail],"must":[HISTORY?,
 *      SIMILAR?, must],"must_not":[{"ids":{"values":[excluded],"boost":0}}(,must_not)?],"minimum_should_match":1}},
 *      "sort":sort} \n
 *    where the elements of should and must are comma-separated and an empty piece leaves no comma.  Ids, elements and
 *    names are escaped as in cco_event_log_user_queries.
 * log may be NULL when no row has a user; index_body may be NULL when no row has an item (index_len 0 with a non-NULL
 * body is an empty index: every item is unknown).  A given body is parsed with cco_item_queries' grammar and checks.
 * limits may be NULL when user_offsets is NULL.
 * Fragments are JSON text spliced verbatim: head ({"from":F,"size":N), boosted (the boosted metadata; may be empty),
 * should_tail (the constant_score clause), must (the filtering metadata and the date filters; may be empty), must_not (may
 * be empty), sort (an array), header (one _msearch header line).
 * Out: *out_body [*out_len] and *out_offsets [*out_n + 1] (record r = body[offsets[r] .. offsets[r + 1])), pinned memory
 * owned by the context, each released with cco_host_free.
 * Errors: CCO_E_INVALID_ARG for everything the three builders refuse (same messages where the cause is the same), a row
 * with a user but no log or a log without history, a log of another context, a row with an item but no index body, and
 * bad offsets in any column (decided on the device before any kernel reads through them); CCO_E_UNSUPPORTED for group
 * contexts, 2^31 or more rows, documents + items + blacklist items + elements >= 2^31, 2^31 or more training events of
 * the names and a record of 2^31 or more bytes.
 */
typedef struct {
  /* the history: cco_user_query_t's members */
  int32_t n_names;
  int32_t n_history_names;           /* maxQueryEvents - 1 clamped to [0, n_names] */
  const char *const *names;          /* [n_names] the query event names */
  const int32_t *limits;             /* [n_names] history limit per name; may be NULL without a user column */
  int32_t n_blacklist_names;
  int32_t history_in_must;           /* 0: should (userBias >= 0), 1: must (userBias < 0) */
  const char *const *blacklist_names;
  const char *history_boost;         /* JSON number text or NULL */
  /* the similar items: cco_item_query_t's members */
  int32_t n_model_names;
  const char *const *model_names;    /* [n_model_names] the index's indicator fields */
  int32_t max_query_events;
  int32_t similar_in_must;           /* 0: should (algorithm itemBias >= 0), 1: must (itemBias < 0) */
  const char *similar_boost;         /* JSON number text or NULL */
  int32_t exclude_self;              /* 1: the item is excluded (!returnSelf) */
  /* the set clause: cco_item_set_query_t's members */
  const char *set_name;              /* the first model event name (may be NULL without with_set) */
  int32_t with_set;                  /* 0: no set clause (itemSetBias 0), 1: the clause is written */
  const char *set_boost;             /* JSON number text or NULL */
  const char *head, *boosted, *should_tail, *must, *must_not, *sort, *header;  /* boosted, must may be "" */
  int64_t n_blacklist_items;
  const int64_t *blacklist_item_offsets; /* [n + 1] */
  const char *blacklist_item_bytes;
} cco_mixed_query_t;
int cco_mixed_queries(cco_ctx_t *ctx, const cco_event_log_t *log /* nullable */, const char *index_body /* nullable */, int64_t index_len,
                      const cco_mixed_query_t *q, int64_t n_rows,
                      const int64_t *user_offsets /* nullable */, const char *user_bytes, const uint8_t *user_validity /* nullable */,
                      const int64_t *item_offsets /* nullable */, const char *item_bytes, const uint8_t *item_validity /* nullable */,
                      const int64_t *set_offsets /* nullable */, int64_t n_elements, const int64_t *elem_offsets, const char *elem_bytes,
                      const uint8_t *set_validity /* nullable */, char **out_body, int64_t *out_len, int64_t **out_offsets,
                      int64_t *out_n);

/*
 * Batchpredict query files: one Query JSON object per line (`pio batchpredict --input`), each line with its own members.
 * Record r of the body is line r's query, exactly what cco_mixed_queries writes for a one-row batch whose template is the
 * line's members.
 *  - cco_query_file_read parses the file on the device with the event reader's line split and tokenizer: lines end at '\n'
 *    (a final one opens no line; an empty or blank line is an error), member names compare decoded, null is an absent
 *    member, unknown members are ignored, a repeated known member is an error.  The row members are checked and decoded
 *    there: user and item (a string), itemSet and blacklistItems (an array of strings); withRanks must be true or false and
 *    is otherwise ignored.  The other known members (fields, dateRange, currentDate, returnSelf, num, from, eventNames,
 *    userBias, itemBias, itemSetBias) form the line's template key: each member's raw value text in that order, '\0'
 *    between them, an absent one empty.  Keys get template ids by first appearance.
 *  - cco_query_file_templates hands out the T distinct keys (key t = key_bytes[key_offsets[t] .. key_offsets[t + 1])),
 *    the first line of each and first_member_line[3 t + k], the first line of template t with a user (k = 0), an item
 *    (k = 1) and a set (k = 2), -1 for none.  The pointers stay valid until cco_query_file_free.  The caller decodes and
 *    type-checks each key and renders its cco_mixed_query_t (limits are required for a template with a user; its
 *    blacklist items must be empty: the lines carry their own).
 *  - cco_query_file_queries renders every line with its template's fragments in one length pass and one write pass:
 *    the history is built once over the union of the query names of the templates with a user (at most 64; a name has
 *    one limit), the user's blacklist once per distinct mask of (template names x blacklist names), and each line's
 *    blacklistItems is its own list (each id once, at its first position across the four sources, as in
 *    cco_mixed_queries).  The model names and max_query_events must be the same in every template.
 * Errors name the 0-based line: CCO_E_INVALID_ARG for malformed JSON, a non-object line, a wrong type, a repeated member,
 * a line with a user but no log with history or with an item but no index body, and everything cco_mixed_queries
 * refuses; CCO_E_UNSUPPORTED for group contexts, 2^31 lines, lines + blacklist items + elements >= 2^31, a line or a
 * record of 2^31 bytes and more than 64 distinct query names.  Outputs as in cco_mixed_queries.
 */
typedef struct cco_query_file cco_query_file_t;
int cco_query_file_read(cco_ctx_t *ctx, const char *bytes, int64_t len, cco_query_file_t **out);
int cco_query_file_templates(const cco_query_file_t *qf, int64_t *n_lines, int64_t *n_templates, const int64_t **key_offsets,
                             const char **key_bytes, const int64_t **first_line, const int64_t **first_member_line);
int cco_query_file_queries(cco_ctx_t *ctx, const cco_query_file_t *qf, const cco_event_log_t *log /* nullable */,
                           const char *index_body /* nullable */, int64_t index_len, int64_t n_templates,
                           const cco_mixed_query_t *templates, char **out_body, int64_t *out_len, int64_t **out_offsets,
                           int64_t *out_n);
int cco_query_file_free(cco_query_file_t *qf);

/*
 * Search results: the Elasticsearch _msearch responses to query bodies read on the device into what URAlgorithm.predict
 * returns for each query (URAlgorithm.scala:484-529, EsClient.scala:370-385, Serving.scala:25-29).  Record r is element r
 * of a body's "responses" array, numbered across appends:
 *  - an element with an "error" member, or a "status" other than 200, has no hits (the reference's None);
 *  - otherwise every element of hits.hits, in order, is one hit: its _id decoded, its _score as the double nearest to
 *    ES's text (a JSON integer too), and for a withRanks record each ranking member of its "_source" that is a number
 *    (absent or null: none).  A missing or null hits.hits has no hits;
 *  - total is hits.total (a number, or ES 7's {"value": ...}), -1 when absent; status is the element's "status", 0 when
 *    absent.  Of a repeated member other than _id and _score the first counts.
 * With CCO_SR_TEXT the PredictedResult of every record is rendered as PredictionIO serves it:
 * {"itemScores":[{"item":"<id>","score":<double>,"ranks":{"<name>":<double>,...}}]}, ids and names through json4s' quote,
 * doubles as Java's Double.toString over the shortest digits, ranks in the order of the names and left out when a hit has
 * none.  Numbers with at most 15 significant digits and a decimal exponent within +-22 are converted on the device; the
 * others (n_exact) on the host, exactly.
 * Streaming: begin, any number of appends (one complete response body each; the next body's copy to the device overlaps
 * the read of the previous one, so a body's error may be returned by the next append or by finish), finish, free.  After
 * a failed append or finish every call but free fails with the same message.
 *  - n_records: the elements the body must hold (the queries of its _msearch request); -1: any number;
 *  - with_ranks: LSB-first bitmap over the body's records (nullable: CCO_SR_WITH_RANKS of params for every record);
 *  - line_offsets[n_records + 1] / line_bytes (nullable; then with_ranks must be NULL): the query-file lines of the body's
 *    records, line r = line_bytes[line_offsets[r] .. line_offsets[r + 1]).  Each line must be one JSON object; its
 *    withRanks, as cco_query_file_read reads it (true or false, null = absent, at most once), is the record's.  With
 *    CCO_SR_BATCHPREDICT record r's text is PredictionIO's BatchPredict output line [RECALL] without its newline:
 *    {"query":<line r re-rendered by json4s>,"prediction":<the PredictedResult>}.  The echo drops insignificant
 *    whitespace, decodes and re-quotes strings (json4s' quote), prints integer literals as BigInt does (-0 -> 0) and other
 *    numbers as the scores are printed; member order and repeated members are kept.  A line is checked for JSON syntax
 *    and nests at most 64 levels; its errors name the record.
 * Errors: CCO_E_INVALID_ARG for malformed JSON and a top level that is not an object with one "responses" array (with the
 * body's byte offset), a count mismatch, and, naming the record (and hit), a responses or hits.hits element that is not an
 * object, hits.hits that is neither an array nor null, a status that is not a 32-bit integer, a hit without a string _id,
 * a repeated _id or _score, a _score that is missing, null or not a number, a rank that is present but neither a number
 * nor null, and a number out of the range of a double.  Strings are checked for valid escapes and raw bytes where the reads
 * go (member names up to _source's, ids); what _source's values hold is checked for closed strings and bracket balance
 * only.  CCO_E_UNSUPPORTED for group contexts, a body larger than a quarter of the device's memory, and 2^31 or more
 * records or hits in one body.
 * Outputs (finish): pinned memory owned by the context, each array released with cco_host_free:
 *   hit_offsets[n_records + 1], status[n_records], total[n_records]; per hit the ids as an Arrow large_string (id_offsets
 *   [n_hits + 1], id_bytes), score[n_hits] and ranks[n_hits * n_rankings] (NaN where a hit has no such rank); with
 *   CCO_SR_TEXT text_offsets[n_records + 1] and text (record r = text[text_offsets[r] .. text_offsets[r + 1])), else NULL.
 */
#define CCO_SR_WITH_RANKS 1u         /* every record is a withRanks query */
#define CCO_SR_TEXT 2u               /* render the PredictedResult text */
#define CCO_SR_BATCHPREDICT 4u       /* with CCO_SR_TEXT: render batchpredict output lines (every append gives query lines) */
typedef struct {
  int32_t n_rankings;                /* 0 .. CCO_MAX_RANKINGS names, in ur_model.rankings_params order; a repeat is one member (the first) */
  const char *const *ranking_names;  /* UTF-8 */
  uint32_t flags;
} cco_search_results_params_t;
typedef struct {
  int64_t n_records, n_hits;
  int32_t n_rankings, reserved;
  int64_t n_exact;                   /* numbers converted on the host */
  int64_t *hit_offsets;
  int32_t *status;
  int64_t *total;
  int64_t *id_offsets;
  char *id_bytes;
  double *score, *ranks;
  int64_t *text_offsets;
  char *text;
} cco_search_results_out_t;
typedef struct cco_search_results cco_search_results_t;
int cco_search_results_begin(cco_ctx_t *ctx, const cco_search_results_params_t *params, cco_search_results_t **out);
int cco_search_results_append(cco_search_results_t *h, const char *body, int64_t len, int64_t n_records,
                              const int64_t *line_offsets /* nullable */, const char *line_bytes, const uint8_t *with_ranks /* nullable */);
int cco_search_results_finish(cco_search_results_t *h, cco_search_results_out_t *out);
int cco_search_results_free(cco_search_results_t *h);

/*
 * Index pages: the model index read back from Elasticsearch, as calcPop reads it (EsClient.getRDD / esJsonRDD,
 * EsClient.scala:464-470) and the item queries read a document (EsClient.getSource, EsClient.scala:394-442), turned into the
 * bulk body cco_format_model writes, which cco_rerank_model, cco_item_queries, cco_mixed_queries and cco_query_file_queries
 * take.  A page is one complete _search or _search/scroll response body (ES 5 .. 8, compact or ?pretty).  For every hit of
 * every page, in order, the body holds
 *   {"index":{"_id":"<_id>"}}\n<_source>\n
 *  - <_id> is the decoded _id (UTF-8, a lone surrogate in its 3-byte form) escaped as cco_format_model escapes ids;
 *  - <_source> is the hit's _source with the whitespace (space, \t, \n, \r) outside strings dropped: member order, repeated
 *    members, number spellings and string escapes are kept, so a compact _source is copied byte for byte.
 * A body this library wrote, paged as Elasticsearch returns it with compact sources, is read back byte for byte.  The
 * reader reads _scroll_id, error, status, timed_out, _shards.failed, hits.total and hits.hits of a page (of a repeated
 * member the first) and _id and _source of a hit (of a repeated _source the first); other members are skipped by depth.
 * Streaming: begin, an append per page, finish, free.  append returns the page's hit count and its decoded _scroll_id
 * (valid until the next call on h; NULL when absent), so a scroll loop is while (n_hits) append(the next scroll page).
 * The page's documents are written by the next append or by finish, so a page's later errors may come from either; after
 * a failed append or finish every call but free fails with the same message.
 * Errors, naming the 0-based page, and the hit or the byte offset where they apply: CCO_E_INVALID_ARG for malformed JSON,
 * a top level that is not an object, a top-level "error" member (with the page's status when it has one), timed_out true,
 * _shards.failed other than 0, hits.hits that is neither an array nor absent (null), a hit that is not an object, has no
 * string _id or a repeated _id, a hit without _source (_source disabled in the mapping or the request) or whose _source is
 * not an object, and a _source string with a bad escape or a raw byte < 0x20 (cco_rerank_model's string rules).  Inside
 * _source only the strings and the bracket balance are checked; the consumers read its members.  An _id on two pages is
 * not checked here: every consumer rejects it.  CCO_E_UNSUPPORTED for group contexts, a page larger than a quarter of the
 * device's memory, 2^31 or more hits in one page and a document line of 2^31 bytes or more.
 */
typedef struct cco_index_pages cco_index_pages_t;
typedef struct {
  int64_t n_docs;        /* documents written = hits read over all pages */
  int64_t total;         /* the first page's hits.total when exact (ES 7: relation "eq"), else -1 */
  char *body;            /* pinned, owned by the context, released with cco_host_free */
  int64_t body_len;
} cco_index_pages_out_t;
int cco_index_pages_begin(cco_ctx_t *ctx, cco_index_pages_t **out);
int cco_index_pages_append(cco_index_pages_t *h, const char *page, int64_t len, int64_t *n_hits,
                           const char **scroll_id /* decoded, valid until the next call on h; NULL if absent */,
                           int64_t *scroll_id_len);
int cco_index_pages_finish(cco_index_pages_t *h, cco_index_pages_out_t *out);
int cco_index_pages_free(cco_index_pages_t *h);

/*
 * Index write: the model index written into Elasticsearch as URModel.save and EsClient.hotSwap write it (URModel.scala:
 * 47-84, EsClient.scala:168-246, 257-362), every part that reads the body or the answers.  The HTTP calls stay with the
 * caller: it sends the byte ranges of the body as POST /<index>/<type>/_bulk requests and hands each response body back.
 *  - begin: the body, in the form cco_format_model, cco_rerank_model and cco_index_pages write ({"index":{..."_id":"<s>"...}}
 *    and one object line per document, each line ending in '\n'), checked with cco_rerank_model's rules (a repeated _id
 *    included); CCO_E_INVALID_ARG names the 0-based document.  The body stays on the device for the session.
 *  - fields: esFields (URModel.scala:78), every distinct decoded member name of the document lines in order of first
 *    appearance (document order, then member order), each escaped as cco_format_model escapes names; "id", which save
 *    adds to every document, goes last when no document line has it (and there is a document).
 *  - requests: the greedy cut of the body into _bulk requests of at most max_docs documents and max_bytes bytes (action and
 *    document lines); a document larger than max_bytes is a request of its own.  Request q holds the documents
 *    [doc_begin[q], doc_begin[q + 1]) and the bytes [byte_begin[q], byte_begin[q + 1]) of the body.
 *  - response: the body of the response to request q.  Requests are answered in any order, each once.  The response is
 *    one object whose "items" array holds one item per document of the request, in order; item i is {"index":{...}} with a
 *    string _id equal to document i's decoded _id, a 32-bit integer status and, for an error, error.type and error.reason
 *    (strings; caused_by and every other member are skipped).  ES 5 .. 8 shapes, compact or ?pretty, any member order.
 *    Each document's latest status is kept on the device.
 *  - retry: the documents whose latest status is 429, their lines in document order as a new body, cut by the same rule
 *    into requests numbered from first_request on; their responses are handed to response like the others.
 *  - finish: the latest status per document (0: never answered), the counts, and for every document whose latest status
 *    is not 2xx its index and the decoded error.type and error.reason of its latest error (empty when it had none).
 * Errors: CCO_E_INVALID_ARG naming the request (and the item or the byte offset where they apply) for malformed JSON, a
 * top level that is not an object, a top-level "error" member (with the response's status when it has one), a missing or
 * non-array "items", an item count other than the request's documents, an item that is not {"index":{...}}, a missing,
 * repeated or non-string _id, an _id that is not the document's, a missing, repeated or non-integer status, a request
 * number out of range and a request answered twice.  CCO_E_UNSUPPORTED for group contexts, a body or a response larger
 * than a quarter of the device's memory, and 2^31 or more documents or members.  After a failed call every call but free
 * fails with the same message.  Every pointer an out-structure receives is pinned memory of the context, released with
 * cco_host_free.
 */
typedef struct cco_index_write cco_index_write_t;
typedef struct {
  int64_t max_docs;      /* documents per request, >= 1 (elasticsearch-hadoop es.batch.size.entries: 1000) */
  int64_t max_bytes;     /* bytes per request, >= 1 (es.batch.size.bytes: 1 MiB) */
} cco_index_write_params_t;
typedef struct {
  int64_t n_docs;        /* documents to send again */
  int64_t *doc;          /* [n_docs] their indexes, ascending */
  char *body;            /* their lines, in document order */
  int64_t body_len;
  int64_t first_request; /* the number of the first retry request */
  int64_t n_requests;
  int64_t *doc_begin;    /* [n_requests + 1] positions in doc[] */
  int64_t *byte_begin;   /* [n_requests + 1] offsets in body */
} cco_index_write_retry_t;
typedef struct {
  int64_t n_docs;
  int32_t *status;       /* [n_docs] the latest status, 0 if never answered */
  int64_t n_ok;          /* 2xx */
  int64_t n_rejected;    /* 429 */
  int64_t n_failed;      /* anything else, never answered included */
  int64_t n_errors;      /* n_rejected + n_failed */
  int64_t *error_doc;    /* [n_errors] ascending */
  int64_t *type_offsets; /* [n_errors + 1], Arrow large_string */
  char *type_bytes;
  int64_t *reason_offsets;
  char *reason_bytes;
} cco_index_write_out_t;
int cco_index_write_begin(cco_ctx_t *ctx, const char *body, int64_t len, const cco_index_write_params_t *params,
                          cco_index_write_t **out);
int cco_index_write_fields(cco_index_write_t *h, int64_t *n, int64_t **name_offsets, char **name_bytes);
int cco_index_write_requests(cco_index_write_t *h, int64_t *n_requests, int64_t **doc_begin, int64_t **byte_begin);
int cco_index_write_response(cco_index_write_t *h, int64_t request, const char *resp, int64_t len);
int cco_index_write_retry(cco_index_write_t *h, cco_index_write_retry_t *out);
int cco_index_write_finish(cco_index_write_t *h, cco_index_write_out_t *out);
int cco_index_write_free(cco_index_write_t *h);

/*
 * Item properties refreshed in the live model index without a retrain: a `$set`, `$unset` or `$delete` reaches the
 * documents in place, and only the documents it changes are written again.  This is not calcPop (cco_rerank_model keeps
 * the reference's precedence, where an old member beats a fresh property); here the fresh properties win, and rankings and
 * correlators are never recomputed.
 * Inputs: the current index as a bulk body, with cco_rerank_model's grammar, checks and messages (a repeated _id is an
 * error); params: the correlator names (the model's event names) and the computed ranking names (the fields of the
 * popular, trending, hot and random rankings; a userDefined ranking's field is an ordinary property); the fresh
 * properties as (item, field, value) triples (cco_item_properties_t, as cco_format_model takes them), or a finished event
 * log's aggregated properties (cco_refresh_properties_log).
 * The rule, one document at a time.  An old document with id x is rewritten as
 *   {"index":{"_id":"<x>"}}\n{"id":"<x>"[,<correlator member>]*[,"<field>":<value>]*[,<ranking member>]*}\n
 *  1. "id" and x as cco_rerank_model writes them (the decoded _id, escaped as every id);
 *  2. its members named like a correlator, verbatim and in order;
 *  3. x's fresh properties by cco_format_model's rules: field index order, the last triple of an (item, field) wins, field
 *     "id" only marks that the item exists, and a field named like a computed ranking is not written;
 *  4. its members named like a computed ranking, verbatim and in order.
 * Every other old member is an old property and is dropped.  "id" and a member followed by a member of the same name are
 * skipped (json4s keeps the last).  A property field named like a correlator is CCO_E_UNSUPPORTED, naming the field:
 * cco_format_model would let it replace the correlator array, and a refresh has no array to put back.
 * Each document is then one of
 *  - deleted: the item has no triple and its rewritten document has no member besides "id" (cco_format_model would not
 *    write it);
 *  - changed: its rewritten source line differs from the old one byte for byte;
 *  - new: an item with a triple and no old document, written as cco_format_model writes a property-only item, in order of
 *    first appearance among the triples;
 *  - unchanged: everything else.
 * Outputs: body = the refreshed full index (the old documents in order without the deleted ones, then the new ones), which
 * the caller keeps for the next refresh, calcPop and item queries; delta = the changed and new documents, in the body's
 * order, which cco_index_write_begin takes; deletes = one {"delete":{"_id":"<id>"}} line per deleted document, the id
 * escaped as every id; changed / deleted = the old document numbers (0-based, ascending).  With params and properties
 * that made the body (the same triples cco_format_model was given, no random ranking), body is the input byte for byte
 * and delta and deletes are empty.  A new item gets no random (uniqueRank) value until the next calcPop.
 * Errors: those of cco_rerank_model on the body and of cco_format_model on the properties; CCO_E_INVALID_ARG for null
 * name arrays or names; CCO_E_UNSUPPORTED for a property named like a correlator, group contexts and documents + triples
 * >= 2^31.  Every pointer the out-structure receives is pinned memory of the context, released with cco_host_free.
 */
typedef struct {
  int32_t n_correlators;
  const char *const *correlators;   /* [n_correlators] NUL-terminated UTF-8 */
  int32_t n_rankings;
  const char *const *rankings;      /* [n_rankings] */
} cco_refresh_params_t;
typedef struct {
  int64_t n_docs;                   /* documents of body */
  int64_t n_changed, n_new, n_deleted, n_unchanged;
  char *body;
  int64_t body_len;
  char *delta;
  int64_t delta_len;
  char *deletes;
  int64_t deletes_len;
  int64_t *changed;                 /* [n_changed] */
  int64_t *deleted;                 /* [n_deleted] */
} cco_refresh_out_t;
int cco_refresh_properties(cco_ctx_t *ctx, const char *body, int64_t body_len, const cco_item_properties_t *props /* nullable */,
                           const cco_refresh_params_t *params, cco_refresh_out_t *out);
int cco_refresh_properties_log(cco_ctx_t *ctx, const char *body, int64_t body_len, const cco_event_log_t *log,
                               const cco_refresh_params_t *params, cco_refresh_out_t *out);

/*
 * Debug/parity entry (tests only): full integer co-occurrence matrix A^T B of two canonical
 * binary matrices computed by the same accumulation kernel as cco_train, no LLR, no top-k.
 * Output CSR over the columns of A with ascending column ids, malloc'ed; free with cco_free.
 */
int cco_debug_cooccurrence(cco_ctx_t *ctx, const cco_csr_t *a, const cco_csr_t *b, int64_t **row_ptr,
                           int32_t **col_idx, int32_t **count);
/* Debug entry (tests only): cap every key range (CCO_FLAG_KEY_RANGES) of this context's trains and debug entries at
 * max_keys keys, even where the packed word fits and without the flag, so that every row path can be run split; 0 = off.
 * On a group context it applies to every GPU of the group. */
int cco_debug_key_range_cap(cco_ctx_t *ctx, int32_t max_keys);
/* Debug entry (tests only): truncate the intern hash (CCO_LOG_INTERN_IDS) of the logs this context begins from now on to
 * its low `bits` bits (0..64; 64 = off), so that inserts collide and every key is found by its bytes. */
int cco_debug_intern_hash_bits(cco_ctx_t *ctx, int32_t bits);
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
