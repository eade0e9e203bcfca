/* Plain-C consumer of the streamed event-log entries of include/cco_b200.h: an export handed over in pieces (part files,
 * say), then ingested as a whole read would be.  Compiled by tests/test_event_stream_abi.py. */
#include <stddef.h>

#include "cco_b200.h"

int read_parts(cco_ctx_t *ctx, int n_parts, const char *const *parts, const int64_t *lens, cco_dataset_t **ds) {
  cco_event_log_t *log = NULL;
  cco_event_log_info_t info;
  const char *names[1] = {"purchase"};
  int rc = cco_event_log_begin(ctx, (int64_t)1 << 30, &log);
  if (rc != CCO_OK) return rc;
  for (int k = 0; rc == CCO_OK && k < n_parts; ++k) {
    rc = cco_event_log_append(log, parts[k], lens[k]);
    if (rc == CCO_OK && lens[k] > 0 && parts[k][lens[k] - 1] != '\n') rc = cco_event_log_append(log, "\n", 1);
  }
  if (rc == CCO_OK) rc = cco_event_log_finish(log);
  if (rc == CCO_OK) rc = cco_event_log_info(log, &info);
  if (rc == CCO_OK && info.n_lines > 0) rc = cco_event_log_ingest(ctx, log, 1, names, 0, ds);
  cco_event_log_free(log);
  return rc;
}
