/* bulk_membership_abi.c — cpbus_unsubscribe_many, cpbus_set_mask_many, cpbus_timer_cancel_many and their group twins from
 * plain C99, the way cgo-generated code sees them: each entry point is taken with its declared type (a mismatch is a compile
 * error under -Werror), and the argument checks run before any device is looked at.  Exit code 0 = all checks passed.
 * Build: gcc -std=c99 -Wall -Wextra -Werror -pedantic -I include tests/c/bulk_membership_abi.c -L containerpilot_b200 -lcpbus */
#include <stdio.h>

#include "cpbus.h"

int main(void) {
  int (*p_unsub)(cpbus_t*, const uint32_t*, uint32_t, int*, uint32_t*) = cpbus_unsubscribe_many;
  int (*p_mask)(cpbus_t*, const uint32_t*, const uint32_t*, uint32_t, int*, uint32_t*) = cpbus_set_mask_many;
  int (*p_cancel)(cpbus_t*, const uint32_t*, uint32_t, int*, uint32_t*) = cpbus_timer_cancel_many;
  int (*g_unsub)(cpbus_group_t*, const uint32_t*, uint32_t, int*, uint32_t*) = cpbus_group_unsubscribe_many;
  int (*g_mask)(cpbus_group_t*, const uint32_t*, const uint32_t*, uint32_t, int*, uint32_t*) = cpbus_group_set_mask_many;
  int (*g_cancel)(cpbus_group_t*, const uint32_t*, uint32_t, int*, uint32_t*) = cpbus_group_timer_cancel_many;
  const uint32_t ids[2] = {0, 1}, masks[2] = {CPBUS_MASK_ALL, 0};
  int status[2] = {1, 1};
  uint32_t applied = 7;
  int bad = 0;
#define CHECK(cond) do { if (!(cond)) { printf("failed: %s\n", #cond); bad++; } } while (0)
  CHECK(p_unsub(NULL, ids, 2, status, &applied) == CPBUS_EINVAL);
  CHECK(p_mask(NULL, ids, masks, 2, status, &applied) == CPBUS_EINVAL);
  CHECK(p_cancel(NULL, ids, 2, status, &applied) == CPBUS_EINVAL);
  CHECK(g_unsub(NULL, ids, 2, status, &applied) == CPBUS_EINVAL);
  CHECK(g_mask(NULL, ids, masks, 2, status, &applied) == CPBUS_EINVAL);
  CHECK(g_cancel(NULL, ids, 2, status, &applied) == CPBUS_EINVAL);
  CHECK(p_unsub(NULL, NULL, 0, NULL, NULL) == CPBUS_EINVAL);   /* the bus is checked first, also for n == 0 */
  CHECK(status[0] == 1 && status[1] == 1 && applied == 7);      /* nothing written on a refusal */
  CHECK(cpbus_abi_version() == 2);
  printf(bad ? "FAILED (%d)\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
