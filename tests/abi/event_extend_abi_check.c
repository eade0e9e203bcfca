/* Plain-C consumer of the extendable event-log entries of include/cco_b200.h.  Without arguments: the entries refuse null
 * arguments before touching a device, and "ok" is printed.  With arguments  A B cutoff1 cutoff2 remove_duplicates : the
 * export file A is read as an extendable log under (cutoff1, remove_duplicates), extended with the file B under cutoff2,
 * finished, and "n_expired n_duplicates n_lines resident_bytes" is printed (cutoff -9223372036854775808: nothing expires).
 * Compiled by tests/test_event_extend.py, run on the device by tests/test_gpu_event_extend.py. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "cco_b200.h"

static char *slurp(const char *path, int64_t *len) {
  FILE *f = fopen(path, "rb");
  if (!f) return NULL;
  fseek(f, 0, SEEK_END);
  long n = ftell(f);
  fseek(f, 0, SEEK_SET);
  char *b = malloc((size_t)n + 1);
  if (b && fread(b, 1, (size_t)n, f) != (size_t)n) {
    free(b);
    b = NULL;
  }
  fclose(f);
  *len = n;
  return b;
}

static int run(const char *path_a, const char *path_b, int64_t cutoff1, int64_t cutoff2, int32_t dedup) {
  int64_t la = 0, lb = 0, n_expired = 0, n_dup = 0, resident = 0;
  char *a = slurp(path_a, &la), *b = slurp(path_b, &lb);
  if (!a || !b) return 20;
  cco_config_t cfg = {0, 0, 1, 0, NULL, NULL, 0};
  cco_ctx_t *ctx = NULL;
  cco_event_log_t *log = NULL;
  cco_event_window_t w1 = {cutoff1, dedup, 0}, w2 = {cutoff2, dedup, 0};
  cco_event_log_info_t info;
  int rc = cco_create(&cfg, &ctx);
  if (rc == CCO_OK) rc = cco_event_log_begin_ex(ctx, 1 << 16, &w1, CCO_LOG_EXTENDABLE, &log);
  if (rc == CCO_OK && la > 0) rc = cco_event_log_append(log, a, la);
  if (rc == CCO_OK) rc = cco_event_log_finish(log);
  if (rc == CCO_OK) rc = cco_event_log_extend(log, &w2);
  if (rc == CCO_OK && lb > 0) rc = cco_event_log_append(log, b, lb);
  if (rc == CCO_OK) rc = cco_event_log_finish(log);
  if (rc == CCO_OK) rc = cco_event_log_window_stats(log, &n_expired, &n_dup);
  if (rc == CCO_OK) rc = cco_event_log_info(log, &info);
  if (rc == CCO_OK) rc = cco_event_log_resident_bytes(log, &resident);
  if (rc == CCO_OK) printf("%lld %lld %lld %lld\n", (long long)n_expired, (long long)n_dup, (long long)info.n_lines, (long long)resident);
  else printf("error %d: %s\n", rc, cco_last_error());
  cco_event_log_free(log);
  if (ctx) cco_destroy(ctx);
  free(a);
  free(b);
  return rc == CCO_OK ? 0 : 21;
}

int main(int argc, char **argv) {
  if (argc == 6) return run(argv[1], argv[2], strtoll(argv[3], NULL, 10), strtoll(argv[4], NULL, 10), (int32_t)atoi(argv[5]));
  cco_event_window_t w = {0, 0, 0};
  int64_t bytes = 0;
  if (cco_event_log_extend(NULL, &w) != CCO_E_INVALID_ARG) return 1;
  if (cco_event_log_extend(NULL, NULL) != CCO_E_INVALID_ARG) return 2;
  if (cco_event_log_resident_bytes(NULL, &bytes) != CCO_E_INVALID_ARG) return 3;
  if (cco_event_log_begin_ex(NULL, 1, &w, CCO_LOG_EXTENDABLE | CCO_LOG_KEEP_HISTORY, NULL) != CCO_E_INVALID_ARG) return 4;
  printf("ok\n");
  return 0;
}
