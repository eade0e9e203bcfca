/* Plain-C consumer of the search-results reader (include/cco_b200.h): one body of two responses with one ranking, the
 * second record withRanks, rendered as text; the outputs released.  Compiled by tests/test_predicted_results.py. */
#include <stddef.h>
#include <string.h>

#include "cco_b200.h"

int search_results_of_one_body(cco_ctx_t *ctx, cco_search_results_out_t *out) {
  static const char body[] = "{\"responses\":[{\"hits\":{\"hits\":[]}},{\"hits\":{\"total\":{\"value\":1},\"hits\":"
                             "[{\"_id\":\"a\",\"_score\":1,\"_source\":{\"popRank\":2.5}}]}}]}";
  const char *names[1] = {"popRank"};
  const uint8_t with_ranks[1] = {2};
  cco_search_results_params_t params = {1, names, CCO_SR_TEXT};
  cco_search_results_t *h = NULL;
  int rc = cco_search_results_begin(ctx, &params, &h);
  if (rc != CCO_OK) return rc;
  rc = cco_search_results_append(h, body, (int64_t)(sizeof body - 1), 2, NULL, NULL, with_ranks);
  if (rc == CCO_OK) rc = cco_search_results_finish(h, out);
  cco_search_results_free(h);
  if (rc == CCO_OK && (out->n_records != 2 || out->n_hits != 1 || out->n_rankings != 1 || out->text == NULL)) rc = CCO_E_INVALID_ARG;
  return rc;
}

/* the same body as batchpredict output lines: the records' query lines give their withRanks */
int batchpredict_lines_of_one_body(cco_ctx_t *ctx, cco_search_results_out_t *out) {
  static const char body[] = "{\"responses\":[{\"hits\":{\"hits\":[]}},{\"hits\":{\"hits\":[{\"_id\":\"a\",\"_score\":1}]}}]}";
  static const char lines[] = "{\"user\":\"u1\"}{\"item\":\"i1\",\"withRanks\":true}";
  const int64_t line_offsets[3] = {0, 13, (int64_t)(sizeof lines - 1)};
  cco_search_results_params_t params = {0, NULL, CCO_SR_TEXT | CCO_SR_BATCHPREDICT};
  cco_search_results_t *h = NULL;
  int rc = cco_search_results_begin(ctx, &params, &h);
  if (rc != CCO_OK) return rc;
  rc = cco_search_results_append(h, body, (int64_t)(sizeof body - 1), 2, line_offsets, lines, NULL);
  if (rc == CCO_OK) rc = cco_search_results_finish(h, out);
  cco_search_results_free(h);
  return rc;
}

void release(cco_ctx_t *ctx, cco_search_results_out_t *out) {
  void *arrays[9] = {out->hit_offsets, out->status, out->total, out->id_offsets, out->id_bytes, out->score, out->ranks,
                     out->text_offsets, out->text};
  for (size_t i = 0; i < 9; ++i) cco_host_free(ctx, arrays[i]);
  memset(out, 0, sizeof *out);
}
