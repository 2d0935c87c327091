/* drain_tickets_abi.c — cpbus_drain_ready_begin, cpbus_take_ready_begin and cpbus_drain_ready_end from plain C99, the way
 * cgo-generated code sees them: each entry point is taken with its declared type (a mismatch is a compile error under
 * -Werror), and the argument checks run before any device is looked at.  Exit code 0 = all checks passed.
 * Build: gcc -std=c99 -Wall -Wextra -Werror -pedantic -I include tests/c/drain_tickets_abi.c -L containerpilot_b200 -lcpbus */
#include <stdio.h>

#include "cpbus.h"

int main(void) {
  int (*p_drain)(cpbus_t*, uint32_t, uint32_t, uint32_t, size_t, size_t, uint32_t*) = cpbus_drain_ready_begin;
  int (*p_take)(cpbus_t*, uint32_t, uint32_t, uint32_t, size_t, size_t, uint32_t*) = cpbus_take_ready_begin;
  int (*p_end)(cpbus_t*, uint32_t, cpbus_event*, size_t, cpbus_ready*, size_t, size_t*, size_t*, uint32_t*) =
      cpbus_drain_ready_end;
  /* _end writes the output layout of cpbus_drain_ready: the same record, entry and count types */
  int (*p_sync)(cpbus_t*, uint32_t, uint32_t, uint32_t, cpbus_event*, size_t, cpbus_ready*, size_t, size_t*, size_t*,
                uint32_t*) = cpbus_drain_ready;
  cpbus_event out[4];
  cpbus_ready ready[2];
  size_t n_ready = 5, total = 5;
  uint32_t next = 5, ticket = 7;
  int bad = 0;
#define CHECK(cond) do { if (!(cond)) { printf("failed: %s\n", #cond); bad++; } } while (0)
  CHECK(p_drain(NULL, 0, 1, 0, 64, 2, &ticket) == CPBUS_EINVAL);
  CHECK(p_take(NULL, 0, 1, 0, 64, 2, &ticket) == CPBUS_EINVAL);
  CHECK(ticket == 7);                                             /* nothing written on a refusal */
  CHECK(p_end(NULL, 0, out, 4, ready, 2, &n_ready, &total, &next) == CPBUS_EINVAL);
  CHECK(p_sync(NULL, 0, 1, 0, out, 4, ready, 2, &n_ready, &total, &next) == CPBUS_EINVAL);
  CHECK(n_ready == 5 && total == 5 && next == 5);
  CHECK(sizeof(cpbus_ready) == 24 && sizeof(cpbus_event) == 32);
  CHECK(cpbus_abi_version() == 2);
  printf(bad ? "FAILED (%d)\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
