/* timer_add_list_abi.c — cpbus_timer_add_list, cpbus_group_timer_add_list and cpbus_timer_spec from plain C99, the way
 * cgo-generated code sees them: each entry point is taken with its declared type (a mismatch is a compile error under
 * -Werror), the struct's layout is printed for the caller to compare, and the argument checks run before any device is
 * looked at.  Exit code 0 = all checks passed.
 * Build: gcc -std=c99 -Wall -Wextra -Werror -pedantic -I include tests/c/timer_add_list_abi.c -L containerpilot_b200 -lcpbus */
#include <stddef.h>
#include <stdio.h>

#include "cpbus.h"

int main(void) {
  int (*p_list)(cpbus_t*, const cpbus_timer_spec*, uint32_t, uint32_t*, int*, uint32_t*) = cpbus_timer_add_list;
  int (*g_list)(cpbus_group_t*, const cpbus_timer_spec*, uint32_t, uint32_t*, int*, uint32_t*) = cpbus_group_timer_add_list;
  cpbus_timer_spec specs[2] = {{1000u, 0u, 7u, 0u, 0u}, {2000u, 1u, 8u, 1u, 0u}};
  uint32_t ids[2] = {5, 5}, applied = 7;
  int status[2] = {1, 1};
  int bad = 0;
#define CHECK(cond) do { if (!(cond)) { printf("failed: %s\n", #cond); bad++; } } while (0)
  printf("layout %u %u %u %u %u %u\n", (unsigned)sizeof(cpbus_timer_spec), (unsigned)offsetof(cpbus_timer_spec, period_ns),
         (unsigned)offsetof(cpbus_timer_spec, sub_id), (unsigned)offsetof(cpbus_timer_spec, source_id),
         (unsigned)offsetof(cpbus_timer_spec, oneshot), (unsigned)offsetof(cpbus_timer_spec, pad));
  CHECK(sizeof(cpbus_timer_spec) == 24);
  CHECK(p_list(NULL, specs, 2, ids, status, &applied) == CPBUS_EINVAL);
  CHECK(g_list(NULL, specs, 2, ids, status, &applied) == CPBUS_EINVAL);
  CHECK(p_list(NULL, NULL, 0, NULL, NULL, NULL) == CPBUS_EINVAL);   /* the bus is checked first, also for n == 0 */
  CHECK(g_list(NULL, NULL, 0, NULL, NULL, NULL) == CPBUS_EINVAL);
  CHECK(status[0] == 1 && status[1] == 1 && ids[0] == 5 && ids[1] == 5 && applied == 7);   /* nothing written on a refusal */
  CHECK(cpbus_abi_version() == 2);
  printf(bad ? "FAILED (%d)\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
