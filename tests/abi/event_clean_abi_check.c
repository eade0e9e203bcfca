/* Plain-C consumer of the clean write-back entries of include/cco_b200.h: an extendable log's source read a second time
 * in pieces and its kept lines written to a FILE as they come.  Compiled by tests/test_event_clean_abi.py. */
#include <stddef.h>
#include <stdio.h>

#include "cco_b200.h"

int write_clean(cco_event_log_t *log, int n_parts, const char *const *parts, const int64_t *lens, FILE *out,
                cco_event_clean_stats_t *stats) {
  cco_event_clean_t *x = NULL;
  const char *bytes = NULL;
  int64_t len = 0;
  int rc = cco_event_log_clean_begin(log, 0, &x);
  if (rc != CCO_OK) return rc;
  for (int k = 0; rc == CCO_OK && k < n_parts; ++k) {
    rc = cco_event_log_clean_append(x, parts[k], lens[k], &bytes, &len);
    if (rc == CCO_OK && len > 0 && fwrite(bytes, 1, (size_t)len, out) != (size_t)len) rc = CCO_E_INVALID_ARG;
  }
  if (rc == CCO_OK) rc = cco_event_log_clean_finish(x, &bytes, &len, stats);
  if (rc == CCO_OK && len > 0 && fwrite(bytes, 1, (size_t)len, out) != (size_t)len) rc = CCO_E_INVALID_ARG;
  cco_event_log_clean_free(x);
  return rc;
}
