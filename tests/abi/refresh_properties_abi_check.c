/* Plain-C consumer of cco_refresh_properties (include/cco_b200.h): a two-document index, one fresh property; the outputs
 * checked and every pinned buffer released.  Without arguments it checks the null-argument refusals only (no GPU);
 * with "run" it refreshes on device 0.  Built and run by tests/test_gpu_refresh_properties.py. */
#include <stdio.h>
#include <string.h>

#include "cco_b200.h"

static int run(void) {
  static const char body[] = "{\"index\":{\"_id\":\"a\"}}\n{\"id\":\"a\",\"buy\":[\"b\"],\"color\":\"red\",\"popRank\":2.0}\n"
                             "{\"index\":{\"_id\":\"b\"}}\n{\"id\":\"b\",\"color\":\"blue\"}\n";
  static const char want_body[] = "{\"index\":{\"_id\":\"a\"}}\n{\"id\":\"a\",\"buy\":[\"b\"],\"color\":\"green\",\"popRank\":2.0}\n";
  static const char want_deletes[] = "{\"delete\":{\"_id\":\"b\"}}\n";
  const int64_t item_offsets[2] = {0, 1}, value_offsets[2] = {0, 7};
  const int32_t field[1] = {0};
  const char *field_names[1] = {"color"}, *correlators[1] = {"buy"}, *rankings[1] = {"popRank"};
  const cco_item_properties_t props = {1, item_offsets, "a", field, value_offsets, "\"green\"", 1, field_names};
  const cco_refresh_params_t params = {1, correlators, 1, rankings};
  cco_config_t cfg = {0, 0, 1, 0, NULL, NULL, 0};
  cco_ctx_t *ctx = NULL;
  cco_refresh_out_t out;
  memset(&out, 0, sizeof out);
  int rc = cco_create(&cfg, &ctx);
  if (rc == CCO_OK) rc = cco_refresh_properties(ctx, body, (int64_t)(sizeof body - 1), &props, &params, &out);
  if (rc == CCO_OK) {
    const int ok = out.n_docs == 1 && out.n_changed == 1 && out.n_new == 0 && out.n_deleted == 1 && out.n_unchanged == 0 &&
                   out.body_len == (int64_t)(sizeof want_body - 1) && memcmp(out.body, want_body, sizeof want_body - 1) == 0 &&
                   out.delta_len == out.body_len && memcmp(out.delta, want_body, sizeof want_body - 1) == 0 &&
                   out.deletes_len == (int64_t)(sizeof want_deletes - 1) && memcmp(out.deletes, want_deletes, sizeof want_deletes - 1) == 0 &&
                   out.changed[0] == 0 && out.deleted[0] == 1;
    if (!ok) rc = CCO_E_INVALID_ARG;
    cco_host_free(ctx, out.body);
    cco_host_free(ctx, out.delta);
    cco_host_free(ctx, out.deletes);
    cco_host_free(ctx, out.changed);
    cco_host_free(ctx, out.deleted);
  }
  if (rc == CCO_OK) printf("ok\n");
  else printf("error %d: %s\n", rc, cco_last_error());
  if (ctx) cco_destroy(ctx);
  return rc == CCO_OK ? 0 : 21;
}

int main(int argc, char **argv) {
  if (argc == 2 && strcmp(argv[1], "run") == 0) return run();
  const cco_refresh_params_t params = {0, NULL, 0, NULL};
  cco_refresh_out_t out;
  if (cco_refresh_properties(NULL, "", 0, NULL, &params, &out) != CCO_E_INVALID_ARG) return 1;
  if (cco_refresh_properties_log(NULL, "", 0, NULL, &params, &out) != CCO_E_INVALID_ARG) return 2;
  printf("ok\n");
  return 0;
}
