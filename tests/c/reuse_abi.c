/* reuse_abi.c — cpbus_release_many, cpbus_subscribe_list and their group twins from plain C99, the way cgo-generated code
 * sees them: each entry point is taken with its declared type (a mismatch is a compile error under -Werror), and the argument
 * checks run before any device is looked at.  Exit code 0 = all checks passed.
 * Build: gcc -std=c99 -Wall -Wextra -Werror -pedantic -I include tests/c/reuse_abi.c -L containerpilot_b200 -lcpbus */
#include <stdio.h>

#include "cpbus.h"

int main(void) {
  int (*p_release)(cpbus_t*, const uint32_t*, uint32_t, int*, uint32_t*) = cpbus_release_many;
  int (*p_list)(cpbus_t*, const uint32_t*, const cpbus_pair*, const uint32_t*, uint32_t, uint32_t*) = cpbus_subscribe_list;
  int (*g_release)(cpbus_group_t*, const uint32_t*, uint32_t, int*, uint32_t*) = cpbus_group_release_many;
  int (*g_list)(cpbus_group_t*, const uint32_t*, const cpbus_pair*, const uint32_t*, uint32_t, uint32_t*) =
      cpbus_group_subscribe_list;
  const uint32_t ids[2] = {0, 1}, masks[2] = {CPBUS_MASK_ALL, 0}, n_pairs[2] = {1, 0};
  const cpbus_pair pairs[2 * CPBUS_MAX_PAIRS] = {{3, 7}};
  uint32_t out[2] = {5, 5}, applied = 7;
  int status[2] = {1, 1};
  int bad = 0;
#define CHECK(cond) do { if (!(cond)) { printf("failed: %s\n", #cond); bad++; } } while (0)
  CHECK(p_release(NULL, ids, 2, status, &applied) == CPBUS_EINVAL);
  CHECK(g_release(NULL, ids, 2, status, &applied) == CPBUS_EINVAL);
  CHECK(p_release(NULL, NULL, 0, NULL, NULL) == CPBUS_EINVAL);   /* the bus is checked first, also for n == 0 */
  CHECK(p_list(NULL, masks, pairs, n_pairs, 2, out) == CPBUS_EINVAL);
  CHECK(g_list(NULL, masks, pairs, n_pairs, 2, out) == CPBUS_EINVAL);
  CHECK(p_list(NULL, NULL, NULL, NULL, 2, out) == CPBUS_EINVAL);
  CHECK(status[0] == 1 && status[1] == 1 && applied == 7 && out[0] == 5 && out[1] == 5);   /* nothing written on a refusal */
  CHECK(cpbus_abi_version() == 2);
  printf(bad ? "FAILED (%d)\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
