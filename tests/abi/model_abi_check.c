/* Plain-C consumer of the complete-model entries of include/cco_b200.h: their structs fill from C99 and the calls type-check.
 * Compiled by tests/test_model_docs.py. */
#include <stddef.h>

#include "cco_b200.h"

int format_with_properties_and_rankings(cco_ctx_t *ctx, const cco_result_t *res, const cco_dictionary_t *rows,
                                        const cco_dictionary_t *cols, char **out, int64_t *len) {
  static const int64_t item_off[3] = {0, 6, 12}, value_off[3] = {0, 5, 10};
  static const int32_t field[2] = {0, 1};
  static const char *const field_names[2] = {"categories", "available"};
  static const int64_t ev_off[3] = {0, 6, 12}, ev_time[2] = {1000, 2000};
  const char *names[1] = {"purchase"};
  cco_item_properties_t props = {2, item_off, "item-1item-2", field, value_off, "[\"a\"]false", 2, field_names};
  cco_ranking_stream_t stream = {2, ev_off, "item-1item-3", ev_time};
  cco_ranking_t ranking = {"popRank", CCO_POP_POPULAR, 1, 0, 5000, &stream};
  return cco_format_model(ctx, res, 1, names, rows, cols, &props, 1, &ranking, out, len);
}

int rank_texts(cco_ctx_t *ctx, char *bytes /* 32 * 3 */, int64_t offsets[4]) {
  static const int64_t v[3] = {9999999, 10000000, -12000000};
  return cco_debug_rank_text(ctx, 3, v, 0, offsets, bytes);
}
