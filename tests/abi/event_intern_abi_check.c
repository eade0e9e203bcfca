/* Plain-C consumer of the interned event-log entries of include/cco_b200.h.  Without arguments: the entries refuse null
 * arguments before touching a device, and "ok" is printed.  With arguments  A B cutoff1 cutoff2 : the export file A is
 * read as an interned extendable log under (cutoff1, removeDuplicates), extended with the file B under cutoff2, finished,
 * ingested for the names "buy" and "view", and "n_user_keys n_item_keys n_users n_items_buy n_items_view resident_bytes"
 * is printed.  Compiled and run on the device by tests/test_gpu_event_intern.py. */
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

static int run(const char *path_a, const char *path_b, int64_t cutoff1, int64_t cutoff2) {
  int64_t la = 0, lb = 0, n_user_keys = 0, n_item_keys = 0, resident = 0;
  char *a = slurp(path_a, &la), *b = slurp(path_b, &lb);
  if (!a || !b) return 20;
  cco_config_t cfg = {0, 0, 1, 0, NULL, NULL, 0};
  cco_ctx_t *ctx = NULL;
  cco_event_log_t *log = NULL;
  cco_dataset_t *ds = NULL;
  cco_event_window_t w1 = {cutoff1, 1, 0}, w2 = {cutoff2, 1, 0};
  const char *names[2] = {"buy", "view"};
  cco_dictionary_t users = {0, NULL, NULL}, buy = {0, NULL, NULL}, view = {0, NULL, NULL};
  int rc = cco_create(&cfg, &ctx);
  if (rc == CCO_OK) rc = cco_event_log_begin_ex(ctx, 1 << 16, &w1, CCO_LOG_EXTENDABLE | CCO_LOG_INTERN_IDS, &log);
  if (rc == CCO_OK && la > 0) rc = cco_event_log_append(log, a, la);
  if (rc == CCO_OK) rc = cco_event_log_finish(log);
  if (rc == CCO_OK) rc = cco_event_log_extend(log, &w2);
  if (rc == CCO_OK && lb > 0) rc = cco_event_log_append(log, b, lb);
  if (rc == CCO_OK) rc = cco_event_log_finish(log);
  if (rc == CCO_OK) rc = cco_event_log_intern_stats(log, &n_user_keys, &n_item_keys);
  if (rc == CCO_OK) rc = cco_event_log_resident_bytes(log, &resident);
  if (rc == CCO_OK) rc = cco_event_log_ingest(ctx, log, 2, names, 0, &ds);
  if (rc == CCO_OK) rc = cco_dataset_dictionary(ds, -1, &users);
  if (rc == CCO_OK) rc = cco_dataset_dictionary(ds, 0, &buy);
  if (rc == CCO_OK) rc = cco_dataset_dictionary(ds, 1, &view);
  if (rc == CCO_OK)
    printf("%lld %lld %lld %lld %lld %lld\n", (long long)n_user_keys, (long long)n_item_keys, (long long)users.n, (long long)buy.n,
           (long long)view.n, (long long)resident);
  else
    printf("error %d: %s\n", rc, cco_last_error());
  if (ds) cco_dataset_free(ds);
  cco_event_log_free(log);
  if (ctx) cco_destroy(ctx);
  free(a);
  free(b);
  return rc == CCO_OK ? 0 : 21;
}

int main(int argc, char **argv) {
  if (argc == 5) return run(argv[1], argv[2], strtoll(argv[3], NULL, 10), strtoll(argv[4], NULL, 10));
  int64_t u = 0, i = 0;
  if (cco_event_log_intern_stats(NULL, &u, &i) != CCO_E_INVALID_ARG) return 1;
  if (cco_debug_intern_hash_bits(NULL, 0) != CCO_E_INVALID_ARG) return 2;
  if (cco_event_log_begin_ex(NULL, 1, NULL, CCO_LOG_INTERN_IDS, NULL) != CCO_E_INVALID_ARG) return 3;
  printf("ok\n");
  return 0;
}
