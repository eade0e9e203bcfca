/* Plain-C consumer of the event-log entries of include/cco_b200.h: read an export, list its names, ingest two of them and
 * format the model with the log's properties and a ranking over its streams.  Compiled by tests/test_events_abi.py. */
#include <stddef.h>

#include "cco_b200.h"

int train_half_from_an_export(cco_ctx_t *ctx, const char *bytes, int64_t len, const cco_result_t *res, const cco_dictionary_t *rows,
                              const cco_dictionary_t *cols, cco_dataset_t **ds, char **out, int64_t *out_len) {
  cco_event_log_t *log = NULL;
  cco_event_log_info_t info;
  const char *names[2] = {"purchase", "view"};
  const char *const stream_names[1] = {"purchase"};
  cco_log_ranking_t ranking = {"popRank", CCO_POP_POPULAR, 1, 0, 5000, stream_names};
  int rc = cco_event_log_read(ctx, bytes, len, &log);
  if (rc != CCO_OK) return rc;
  rc = cco_event_log_info(log, &info);
  if (rc == CCO_OK && info.names.n > 0 && info.n_training[0] >= 0 && info.n_ranking[0] >= 0 && info.n_property_events >= 0 &&
      info.n_property_items >= 0 && info.n_property_fields >= 0)
    rc = cco_event_log_ingest(ctx, log, 2, names, 3, ds);
  if (rc == CCO_OK) rc = cco_format_model_log(ctx, res, 2, names, rows, cols, log, 1, &ranking, out, out_len);
  if (rc == CCO_OK) rc = cco_rerank_model_log(ctx, *out, *out_len, log, 1, &ranking, out, out_len);
  cco_event_log_free(log);
  return rc;
}
