/* Plain-C consumer of the index-pages reader (include/cco_b200.h): a scroll of two pages, the second one empty, read into
 * the bulk body; the body released.  Compiled by tests/test_index_pages.py. */
#include <stddef.h>
#include <string.h>

#include "cco_b200.h"

int index_of_two_pages(cco_ctx_t *ctx, cco_index_pages_out_t *out) {
  static const char first[] = "{\"_scroll_id\":\"s1\",\"timed_out\":false,\"hits\":{\"total\":{\"value\":1,\"relation\":\"eq\"},"
                              "\"hits\":[{\"_id\":\"a\",\"_score\":null,\"_source\":{\"id\":\"a\",\"popRank\":2.0}}]}}";
  static const char last[] = "{\"_scroll_id\":\"s1\",\"hits\":{\"total\":{\"value\":1,\"relation\":\"eq\"},\"hits\":[]}}";
  const char *pages[2] = {first, last};
  const int64_t lens[2] = {(int64_t)(sizeof first - 1), (int64_t)(sizeof last - 1)};
  cco_index_pages_t *h = NULL;
  int rc = cco_index_pages_begin(ctx, &h);
  if (rc != CCO_OK) return rc;
  for (int p = 0; p < 2 && rc == CCO_OK; ++p) {
    int64_t n_hits = 0, sid_len = 0;
    const char *sid = NULL;
    rc = cco_index_pages_append(h, pages[p], lens[p], &n_hits, &sid, &sid_len);
    if (rc == CCO_OK && (sid == NULL || sid_len != 2 || memcmp(sid, "s1", 2) != 0)) rc = CCO_E_INVALID_ARG;
  }
  if (rc == CCO_OK) rc = cco_index_pages_finish(h, out);
  cco_index_pages_free(h);
  if (rc == CCO_OK && (out->n_docs != 1 || out->total != 1 || out->body == NULL)) rc = CCO_E_INVALID_ARG;
  return rc;
}

void release(cco_ctx_t *ctx, cco_index_pages_out_t *out) {
  cco_host_free(ctx, out->body);
  memset(out, 0, sizeof *out);
}
