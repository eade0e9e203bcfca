/* Plain-C consumer of the erase entries of include/cco_b200.h: the lines of a list of users (NUL-terminated ids, packed
 * into the Arrow layout here) taken out of a resident extendable log, and the balance of its counters checked.  Compiled by
 * tests/test_event_erase_abi.py. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "cco_b200.h"

int erase_users(cco_event_log_t *log, int n, const char *const *ids, cco_event_erase_stats_t *stats) {
  int64_t *off = malloc(sizeof(int64_t) * ((size_t)n + 1));
  size_t total = 0;
  for (int i = 0; i < n; ++i) total += strlen(ids[i]);
  char *bytes = malloc(total + 1);
  if (!off || !bytes) {
    free(off);
    free(bytes);
    return CCO_E_INVALID_ARG;
  }
  off[0] = 0;
  for (int i = 0; i < n; ++i) {
    const size_t k = strlen(ids[i]);
    memcpy(bytes + off[i], ids[i], k);
    off[i + 1] = off[i] + (int64_t)k;
  }
  const int rc = cco_event_log_erase(log, n, off, bytes, 0, NULL, NULL, stats);
  free(off);
  free(bytes);
  return rc;
}

/* lines read = retained + expired + duplicates + erased, with the retained lines counted by the caller */
int balanced(const cco_event_log_t *log, int64_t retained) {
  cco_event_log_info_t info;
  int64_t expired = 0, duplicates = 0, erased = 0;
  if (cco_event_log_info(log, &info) != CCO_OK || cco_event_log_window_stats(log, &expired, &duplicates) != CCO_OK ||
      cco_event_log_erased(log, &erased) != CCO_OK)
    return 0;
  return info.n_lines == retained + expired + duplicates + erased;
}
