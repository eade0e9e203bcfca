/* Plain-C consumer of the eventWindow entries of include/cco_b200.h: an export read with expiry and duplicate removal,
 * then its drop counts.  Compiled and linked by tests/test_event_window.py. */
#include <stdint.h>
#include <stdio.h>

#include "cco_b200.h"

int read_windowed(cco_ctx_t *ctx, const char *bytes, int64_t len, int64_t now_ms, int64_t duration_ms, int64_t *n_expired,
                  int64_t *n_duplicates) {
  cco_event_window_t w = {now_ms - duration_ms, 1, 0};
  cco_event_log_t *log = NULL;
  int rc = cco_event_log_begin_window(ctx, len > 0 ? len : 1, &w, &log);
  if (rc != CCO_OK) return rc;
  rc = cco_event_log_append(log, bytes, len);
  if (rc == CCO_OK) rc = cco_event_log_finish(log);
  if (rc == CCO_OK) rc = cco_event_log_window_stats(log, n_expired, n_duplicates);
  cco_event_log_free(log);
  return rc;
}

int main(void) {
  /* without a context both entries refuse the call */
  cco_event_window_t w = {INT64_MIN, 0, 0};
  cco_event_log_t *log = NULL;
  int64_t x = 0, d = 0;
  if (cco_event_log_begin_window(NULL, 1, &w, &log) != CCO_E_INVALID_ARG) return 1;
  if (cco_event_log_window_stats(NULL, &x, &d) != CCO_E_INVALID_ARG) return 2;
  (void)read_windowed;
  printf("ok\n");
  return 0;
}
