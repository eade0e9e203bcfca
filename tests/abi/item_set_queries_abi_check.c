/* Plain-C consumer of cco_item_set_queries (include/cco_b200.h): the queries of two shopping carts, the second with a
 * repeated element, first with the set clause boosted, then without the clause (itemSetBias 0).  Compiled by
 * tests/test_item_set_queries.py. */
#include <stddef.h>

#include "cco_b200.h"

int item_set_queries_of_two_carts(cco_ctx_t *ctx, char **body, int64_t *body_len, int64_t **offsets, int64_t *n) {
  const int64_t set_offsets[3] = {0, 1, 4};
  const int64_t elem_offsets[5] = {0, 8, 22, 35, 49};
  const char *elems = "iPhone 6iPhone earbudsiPhone 6 caseiPhone earbuds";
  const int64_t no_offsets[1] = {0};
  cco_item_set_query_t q = {"purchase", 1, "2.0", "{\"from\":0,\"size\":4", "{\"terms\":{\"purchase\":[]}}",
                            "{\"constant_score\":{\"filter\":{\"match_all\":{}},\"boost\":0}}", "", "", "[]", "{}", 0, no_offsets, NULL};
  int rc = cco_item_set_queries(ctx, &q, 2, set_offsets, 4, elem_offsets, elems, body, body_len, offsets, n);
  if (rc != CCO_OK) return rc;
  cco_host_free(ctx, *body);
  cco_host_free(ctx, *offsets);
  q.with_set = 0;
  q.boost = NULL;
  return cco_item_set_queries(ctx, &q, 2, set_offsets, 4, elem_offsets, elems, body, body_len, offsets, n);
}
