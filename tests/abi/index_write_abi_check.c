/* Plain-C consumer of the index-write session (include/cco_b200.h): a body of one document, its fields and requests, a
 * _bulk response, a retry round and the result; every pinned output released.  Compiled by tests/test_index_write_abi.py. */
#include <stddef.h>
#include <string.h>

#include "cco_b200.h"

int write_one_document(cco_ctx_t *ctx, cco_index_write_out_t *out) {
  static const char body[] = "{\"index\":{\"_id\":\"a\"}}\n{\"purchase\":[\"b\"],\"id\":\"a\"}\n";
  static const char resp[] = "{\"took\":3,\"errors\":false,\"items\":[{\"index\":{\"_index\":\"urindex_1\",\"_type\":\"items\","
                             "\"_id\":\"a\",\"_version\":1,\"result\":\"created\",\"status\":201}}]}";
  const cco_index_write_params_t params = {1000, 1 << 20};
  cco_index_write_t *h = NULL;
  int rc = cco_index_write_begin(ctx, body, (int64_t)(sizeof body - 1), &params, &h);
  if (rc != CCO_OK) return rc;
  int64_t n = 0, n_requests = 0;
  int64_t *name_offsets = NULL, *doc_begin = NULL, *byte_begin = NULL;
  char *name_bytes = NULL;
  rc = cco_index_write_fields(h, &n, &name_offsets, &name_bytes);
  if (rc == CCO_OK) {
    if (n != 2 || memcmp(name_bytes, "purchaseid", 10) != 0) rc = CCO_E_INVALID_ARG;
    cco_host_free(ctx, name_offsets);
    cco_host_free(ctx, name_bytes);
  }
  if (rc == CCO_OK) rc = cco_index_write_requests(h, &n_requests, &doc_begin, &byte_begin);
  if (rc == CCO_OK) {
    if (n_requests != 1 || doc_begin[1] != 1 || byte_begin[1] != (int64_t)(sizeof body - 1)) rc = CCO_E_INVALID_ARG;
    cco_host_free(ctx, doc_begin);
    cco_host_free(ctx, byte_begin);
  }
  if (rc == CCO_OK) rc = cco_index_write_response(h, 0, resp, (int64_t)(sizeof resp - 1));
  if (rc == CCO_OK) {
    cco_index_write_retry_t retry;
    rc = cco_index_write_retry(h, &retry);
    if (rc == CCO_OK) {
      if (retry.n_docs != 0 || retry.n_requests != 0 || retry.first_request != 1) rc = CCO_E_INVALID_ARG;
      cco_host_free(ctx, retry.doc);
      cco_host_free(ctx, retry.body);
      cco_host_free(ctx, retry.doc_begin);
      cco_host_free(ctx, retry.byte_begin);
    }
  }
  if (rc == CCO_OK) rc = cco_index_write_finish(h, out);
  cco_index_write_free(h);
  if (rc == CCO_OK && (out->n_docs != 1 || out->n_ok != 1 || out->status[0] != 201)) rc = CCO_E_INVALID_ARG;
  return rc;
}

void release(cco_ctx_t *ctx, cco_index_write_out_t *out) {
  cco_host_free(ctx, out->status);
  cco_host_free(ctx, out->error_doc);
  cco_host_free(ctx, out->type_offsets);
  cco_host_free(ctx, out->type_bytes);
  cco_host_free(ctx, out->reason_offsets);
  cco_host_free(ctx, out->reason_bytes);
  memset(out, 0, sizeof *out);
}
