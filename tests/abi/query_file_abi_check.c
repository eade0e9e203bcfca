/* Plain-C consumer of the query-file builder (include/cco_b200.h): read a two-line file, list its templates, render every
 * line with one template each, and free the file.  Compiled by tests/test_query_file.py. */
#include <stddef.h>

#include "cco_b200.h"

int query_file_of_two_lines(cco_ctx_t *ctx, const cco_event_log_t *log, const char *index_body, int64_t index_len,
                            const cco_mixed_query_t templates[2], char **body, int64_t *body_len, int64_t **offsets, int64_t *n) {
  static const char file[] = "{\"user\":\"u1\",\"blacklistItems\":[\"a\"]}\n{\"item\":\"i1\",\"num\":3}\n";
  cco_query_file_t *qf = NULL;
  int64_t n_lines = 0, n_templates = 0;
  const int64_t *key_offsets = NULL, *first_line = NULL, *first_member_line = NULL;
  const char *key_bytes = NULL;
  int rc = cco_query_file_read(ctx, file, (int64_t)(sizeof file - 1), &qf);
  if (rc != CCO_OK) return rc;
  rc = cco_query_file_templates(qf, &n_lines, &n_templates, &key_offsets, &key_bytes, &first_line, &first_member_line);
  if (rc == CCO_OK && (n_lines != 2 || n_templates != 2 || first_member_line[0] != 0 || first_member_line[3 + 1] != 1)) rc = CCO_E_INVALID_ARG;
  if (rc == CCO_OK) rc = cco_query_file_queries(ctx, qf, log, index_body, index_len, n_templates, templates, body, body_len, offsets, n);
  cco_query_file_free(qf);
  return rc;
}
