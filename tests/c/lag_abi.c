/* lag_abi.c — cpbus_lagging / cpbus_blockers and their group twins from plain C99, the way cgo-generated code sees them:
 * each entry point is taken with its declared type (a mismatch is a compile error under -Werror), the structs have the
 * documented layout, and every call refuses a NULL handle with CPBUS_EINVAL before it touches a device.  Exit code 0 = all
 * checks passed.
 * Build: gcc -std=c99 -Wall -Wextra -Werror -pedantic -I include tests/c/lag_abi.c -L containerpilot_b200 -lcpbus */
#include <stddef.h>
#include <stdio.h>

#include "cpbus.h"

int main(void) {
  int (*p_lagging)(cpbus_t*, uint32_t, uint32_t, uint32_t, uint32_t, cpbus_lag*, size_t, size_t*, uint32_t*,
                   cpbus_lag_summary*) = cpbus_lagging;
  int (*p_blockers)(cpbus_t*, uint32_t*, size_t, size_t*) = cpbus_blockers;
  int (*p_group_lagging)(cpbus_group_t*, uint32_t, uint32_t, uint32_t, uint32_t, cpbus_lag*, size_t, size_t*, uint32_t*,
                         cpbus_lag_summary*) = cpbus_group_lagging;
  int (*p_group_blockers)(cpbus_group_t*, uint32_t*, size_t, size_t*) = cpbus_group_blockers;
  cpbus_lag lag;
  cpbus_lag_summary sum;
  uint32_t id = 0;
  size_t n = 0;
  int bad = 0;
#define CHECK(cond) do { if (!(cond)) { printf("failed: %s\n", #cond); bad++; } } while (0)
  CHECK(sizeof(cpbus_lag) == 16);
  CHECK(offsetof(cpbus_lag, backlog) == 4 && offsetof(cpbus_lag, lost) == 8);
  CHECK(sizeof(cpbus_lag_summary) == 38 * 8);
  CHECK(offsetof(cpbus_lag_summary, hist) == 5 * 8);
  CHECK(p_lagging(NULL, 0, 1, 0, 1, &lag, 1, &n, &id, &sum) == CPBUS_EINVAL);
  CHECK(p_lagging(NULL, 0, 1, 0, 0, NULL, 0, &n, &id, NULL) == CPBUS_EINVAL);
  CHECK(p_blockers(NULL, &id, 1, &n) == CPBUS_EINVAL);
  CHECK(p_group_lagging(NULL, 0, 1, 0, 1, &lag, 1, &n, &id, &sum) == CPBUS_EINVAL);
  CHECK(p_group_blockers(NULL, &id, 1, &n) == CPBUS_EINVAL);
  printf(bad ? "FAILED (%d)\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
