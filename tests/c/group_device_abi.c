/* group_device_abi.c — cpbus_group_publish_device and _staged from plain C99, the way cgo-generated code sees them: each
 * entry point is taken with its declared type (a mismatch is a compile error under -Werror) next to its single-bus twin,
 * and the argument checks run before any device is looked at.  Exit code 0 = all checks passed.
 * Build: gcc -std=c99 -Wall -Wextra -Werror -pedantic -I include tests/c/group_device_abi.c -L containerpilot_b200 -lcpbus */
#include <stdio.h>

#include "cpbus.h"

int main(void) {
  int (*p_dev)(cpbus_t*, const void*, size_t, uint64_t) = cpbus_publish_device;
  int (*g_dev)(cpbus_group_t*, const void*, size_t, uint64_t) = cpbus_group_publish_device;
  int (*p_staged)(cpbus_t*, const void*, size_t, uint64_t, const void*, size_t) = cpbus_publish_device_staged;
  int (*g_staged)(cpbus_group_t*, const void*, size_t, uint64_t, const void*, size_t) = cpbus_group_publish_device_staged;
  static cpbus_event batch[4];
  int bad = 0;
#define CHECK(cond) do { if (!(cond)) { printf("failed: %s\n", #cond); bad++; } } while (0)
  CHECK(p_dev(NULL, batch, 4, 10) == CPBUS_EINVAL);
  CHECK(g_dev(NULL, batch, 4, 10) == CPBUS_EINVAL);
  CHECK(g_dev(NULL, NULL, 0, 10) == CPBUS_EINVAL);   /* the group is checked first, also for n == 0 */
  CHECK(p_staged(NULL, batch, 4, 10, NULL, 0) == CPBUS_EINVAL);
  CHECK(g_staged(NULL, batch, 4, 10, batch, 4) == CPBUS_EINVAL);
  CHECK(cpbus_abi_version() == 2);
  printf(bad ? "FAILED (%d)\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
