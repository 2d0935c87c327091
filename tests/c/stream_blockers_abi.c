/* stream_blockers_abi.c — cpbus_stream_blockers from plain C99, the way cgo-generated code sees it: the entry point is taken
 * with its declared type (a mismatch is a compile error under -Werror), and the calls that need no device refuse their
 * arguments with CPBUS_EINVAL.  Exit code 0 = all checks passed.
 * Build: gcc -std=c99 -Wall -Wextra -Werror -pedantic -I include tests/c/stream_blockers_abi.c -L containerpilot_b200 -lcpbus */
#include <stddef.h>
#include <stdio.h>

#include "cpbus.h"

int main(void) {
  int (*p_stream_blockers)(cpbus_stream_t*, uint32_t*, size_t, size_t*) = cpbus_stream_blockers;
  uint32_t id = 0;
  size_t n = 7;
  int bad = 0;
#define CHECK(cond) do { if (!(cond)) { printf("failed: %s\n", #cond); bad++; } } while (0)
  CHECK(p_stream_blockers(NULL, &id, 1, &n) == CPBUS_EINVAL);
  CHECK(p_stream_blockers(NULL, NULL, 0, &n) == CPBUS_EINVAL);
  CHECK(p_stream_blockers(NULL, &id, 1, NULL) == CPBUS_EINVAL);
  CHECK(cpbus_abi_version() == 2);
  printf(bad ? "FAILED (%d)\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
