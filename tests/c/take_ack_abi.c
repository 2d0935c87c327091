/* take_ack_abi.c — cpbus_take_ready, cpbus_ack_many and their group twins from plain C99, the way cgo-generated code sees
 * them: each entry point is taken with its declared type (a mismatch is a compile error under -Werror), and the argument
 * checks run before any device is looked at.  Exit code 0 = all checks passed.
 * Build: gcc -std=c99 -Wall -Wextra -Werror -pedantic -I include tests/c/take_ack_abi.c -L containerpilot_b200 -lcpbus */
#include <stdio.h>

#include "cpbus.h"

int main(void) {
  int (*p_take)(cpbus_t*, uint32_t, uint32_t, uint32_t, cpbus_event*, size_t, cpbus_ready*, size_t, size_t*, size_t*,
                uint32_t*) = cpbus_take_ready;
  int (*p_ack)(cpbus_t*, const uint32_t*, const uint32_t*, uint32_t, int*, uint32_t*) = cpbus_ack_many;
  int (*g_take)(cpbus_group_t*, uint32_t, uint32_t, uint32_t, cpbus_event*, size_t, cpbus_ready*, size_t, size_t*, size_t*,
                uint32_t*) = cpbus_group_take_ready;
  int (*g_ack)(cpbus_group_t*, const uint32_t*, const uint32_t*, uint32_t, int*, uint32_t*) = cpbus_group_ack_many;
  cpbus_event out[4];
  cpbus_ready ready[2];
  size_t n_ready = 5, total = 5;
  uint32_t next = 5;
  const uint32_t ids[2] = {0, 1}, counts[2] = {1, 0};
  int status[2] = {1, 1};
  uint32_t applied = 7;
  int bad = 0;
#define CHECK(cond) do { if (!(cond)) { printf("failed: %s\n", #cond); bad++; } } while (0)
  CHECK(p_take(NULL, 0, 1, 0, out, 4, ready, 2, &n_ready, &total, &next) == CPBUS_EINVAL);
  CHECK(g_take(NULL, 0, 1, 0, out, 4, ready, 2, &n_ready, &total, &next) == CPBUS_EINVAL);
  CHECK(n_ready == 5 && total == 5 && next == 5);               /* nothing written on a refusal */
  CHECK(p_ack(NULL, ids, counts, 2, status, &applied) == CPBUS_EINVAL);
  CHECK(g_ack(NULL, ids, counts, 2, status, &applied) == CPBUS_EINVAL);
  CHECK(p_ack(NULL, NULL, NULL, 0, NULL, NULL) == CPBUS_EINVAL);   /* the bus is checked first, also for n == 0 */
  CHECK(status[0] == 1 && status[1] == 1 && applied == 7);
  CHECK(sizeof(cpbus_ready) == 24);
  CHECK(cpbus_abi_version() == 2);
  printf(bad ? "FAILED (%d)\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
