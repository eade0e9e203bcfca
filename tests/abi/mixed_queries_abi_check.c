/* Plain-C consumer of cco_mixed_queries (include/cco_b200.h): three rows over a log and an index body -- a user with an
 * item, an item set alone (row 0 has no set: its validity bit is 0), and a row with no member -- then the same rows without
 * the set clause.  Compiled by tests/test_mixed_queries.py. */
#include <stddef.h>

#include "cco_b200.h"

int mixed_queries_of_three_rows(cco_ctx_t *ctx, const cco_event_log_t *log, const char *index_body, int64_t index_len, char **body,
                                int64_t *body_len, int64_t **offsets, int64_t *n) {
  const char *names[1] = {"purchase"};
  const int32_t limits[1] = {100};
  const int64_t user_offsets[4] = {0, 2, 2, 2};
  const uint8_t user_validity[1] = {0x1};
  const int64_t item_offsets[4] = {0, 8, 8, 8};
  const uint8_t item_validity[1] = {0x1};
  const int64_t set_offsets[4] = {0, 0, 2, 2};
  const uint8_t set_validity[1] = {0x2};
  const int64_t elem_offsets[3] = {0, 8, 12};
  const int64_t no_offsets[1] = {0};
  cco_mixed_query_t q = {1, 1, names, limits, 1, 0, names, NULL,
                         1, names, 1000, 0, NULL, 1,
                         "purchase", 1, "2.0",
                         "{\"from\":0,\"size\":4", "", "{\"constant_score\":{\"filter\":{\"match_all\":{}},\"boost\":0}}", "", "", "[]", "{}",
                         0, no_offsets, NULL};
  int rc = cco_mixed_queries(ctx, log, index_body, index_len, &q, 3, user_offsets, "u1", user_validity, item_offsets, "Iphone 4",
                             item_validity, set_offsets, 2, elem_offsets, "Iphone 6Soap", set_validity, body, body_len, offsets, n);
  if (rc != CCO_OK) return rc;
  cco_host_free(ctx, *body);
  cco_host_free(ctx, *offsets);
  q.with_set = 0;
  q.set_boost = NULL;
  return cco_mixed_queries(ctx, log, index_body, index_len, &q, 3, user_offsets, "u1", user_validity, item_offsets, "Iphone 4", item_validity,
                           set_offsets, 2, elem_offsets, "Iphone 6Soap", set_validity, body, body_len, offsets, n);
}
