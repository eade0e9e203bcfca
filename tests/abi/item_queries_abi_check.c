/* Plain-C consumer of cco_item_queries (include/cco_b200.h): the item queries of two items over a model index body, the
 * similar items boosted in should and the item itself excluded.  Compiled by tests/test_item_queries.py. */
#include <stddef.h>

#include "cco_b200.h"

int item_queries_of_an_index(cco_ctx_t *ctx, const char *index, int64_t index_len, char **body, int64_t *body_len, int64_t **offsets,
                             int64_t *n) {
  const char *const names[3] = {"purchase", "view", "category-pref"};
  const int64_t item_offsets[3] = {0, 8, 19};
  const int64_t no_offsets[1] = {0};
  cco_item_query_t q = {3, names, 3000, 0, "2.0", 1, "{\"from\":0,\"size\":4", "", "{\"constant_score\":{\"filter\":{\"match_all\":{}},\"boost\":0}}",
                        "", "", "", "[]", "{}", 0, no_offsets, NULL};
  cco_dictionary_t every = {0, NULL, NULL};
  int rc = cco_item_queries(ctx, index, index_len, &q, 2, item_offsets, "Iphone 4Ipad-retina", body, body_len, offsets, n, NULL);
  if (rc != CCO_OK) return rc;
  cco_host_free(ctx, *body);
  cco_host_free(ctx, *offsets);
  q.similar_in_must = 1;
  q.similar_boost = NULL;
  rc = cco_item_queries(ctx, index, index_len, &q, 0, NULL, NULL, body, body_len, offsets, n, &every);
  if (rc == CCO_OK && every.n == *n) {
    cco_host_free(ctx, (void *)every.offsets);
    cco_host_free(ctx, (void *)every.bytes);
  }
  return rc;
}
