/* Plain-C consumer of the event-log snapshot entries of include/cco_b200.h.  Without arguments: the entries refuse null
 * arguments before touching a device, and "ok" is printed.  With arguments  EXPORT SNAPSHOT chunk : the export file is
 * read as an extendable, interned log with history, saved to the file SNAPSHOT in blocks of `chunk` bytes, loaded back
 * from it in blocks of `chunk` bytes, and "n_lines resident_bytes(saved) resident_bytes(loaded) n_user_keys snapshot_bytes"
 * is printed.  Compiled and run on the device by tests/test_gpu_event_snapshot.py. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "cco_b200.h"

static int run(const char *export_path, const char *snap_path, int64_t chunk) {
  FILE *f = fopen(export_path, "rb");
  if (!f) return 20;
  char *buf = malloc((size_t)chunk);
  if (!buf) return 20;
  cco_config_t cfg = {0, 0, 1, 0, NULL, NULL, 0};
  cco_ctx_t *ctx = NULL;
  cco_event_log_t *log = NULL, *back = NULL;
  cco_event_log_info_t info;
  int64_t size = 0, rb = 0, rb2 = 0, uk = 0, ik = 0;
  size_t n;
  int rc = cco_create(&cfg, &ctx);
  if (rc == CCO_OK) rc = cco_event_log_begin_ex(ctx, 1 << 16, NULL, CCO_LOG_KEEP_HISTORY | CCO_LOG_EXTENDABLE | CCO_LOG_INTERN_IDS, &log);
  while (rc == CCO_OK && (n = fread(buf, 1, (size_t)chunk, f)) > 0) rc = cco_event_log_append(log, buf, (int64_t)n);
  fclose(f);
  if (rc == CCO_OK) rc = cco_event_log_finish(log);
  if (rc == CCO_OK) rc = cco_event_log_resident_bytes(log, &rb);
  if (rc == CCO_OK) rc = cco_event_log_save_size(log, &size);
  FILE *out = rc == CCO_OK ? fopen(snap_path, "wb") : NULL;
  for (int64_t off = 0; out && rc == CCO_OK && off < size; off += chunk) {
    const int64_t k = size - off < chunk ? size - off : chunk;
    rc = cco_event_log_save(log, off, buf, k);
    if (rc == CCO_OK && fwrite(buf, 1, (size_t)k, out) != (size_t)k) rc = 22;
  }
  if (out) fclose(out);
  FILE *in = rc == CCO_OK ? fopen(snap_path, "rb") : NULL;
  if (rc == CCO_OK) rc = cco_event_log_load_begin(ctx, &back);
  while (in && rc == CCO_OK && (n = fread(buf, 1, (size_t)chunk, in)) > 0) rc = cco_event_log_load_append(back, buf, (int64_t)n);
  if (in) fclose(in);
  if (rc == CCO_OK) rc = cco_event_log_load_finish(back);
  if (rc == CCO_OK) rc = cco_event_log_info(back, &info);
  if (rc == CCO_OK) rc = cco_event_log_resident_bytes(back, &rb2);
  if (rc == CCO_OK) rc = cco_event_log_intern_stats(back, &uk, &ik);
  if (rc == CCO_OK)
    printf("%lld %lld %lld %lld %lld\n", (long long)info.n_lines, (long long)rb, (long long)rb2, (long long)uk, (long long)size);
  else
    printf("error %d: %s\n", rc, cco_last_error());
  cco_event_log_free(back);
  cco_event_log_free(log);
  if (ctx) cco_destroy(ctx);
  free(buf);
  return rc == CCO_OK ? 0 : 21;
}

int main(int argc, char **argv) {
  if (argc == 4) return run(argv[1], argv[2], strtoll(argv[3], NULL, 10));
  int64_t b = 0;
  cco_event_log_t *log = NULL;
  char x = 0;
  if (cco_event_log_save_size(NULL, &b) != CCO_E_INVALID_ARG) return 1;
  if (cco_event_log_save(NULL, 0, &x, 1) != CCO_E_INVALID_ARG) return 2;
  if (cco_event_log_load_begin(NULL, &log) != CCO_E_INVALID_ARG) return 3;
  if (cco_event_log_load_append(NULL, &x, 1) != CCO_E_INVALID_ARG) return 4;
  if (cco_event_log_load_finish(NULL) != CCO_E_INVALID_ARG) return 5;
  if (CCO_SNAPSHOT_VERSION != 1) return 6;
  printf("ok\n");
  return 0;
}
