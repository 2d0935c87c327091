/* drop_missed_abi.c — CPBUS_CFG_DROP_MISSED_TICKS and the CPBUS_DUE_CATCHUP op of cpbus_due_trace from plain C99, the way
 * cgo-generated code sees them: the flag's value, and a trace in which a step of 95 ns across a 10 ns timer delivers one tick
 * instead of ten.  Exit code 0 = all checks passed.
 * Build: gcc -std=c99 -Wall -Wextra -Werror -pedantic -I include tests/c/drop_missed_abi.c -L containerpilot_b200 -lcpbus */
#include <stddef.h>
#include <stdio.h>

#include "cpbus.h"

int main(void) {
  int (*p_trace)(const cpbus_due_op*, size_t, uint32_t, uint32_t, cpbus_due_fire*, size_t, size_t*) = cpbus_due_trace;
  /* slot 0: periodic, 10 ns; slot 1: one-shot at 25 ns.  Launch to 5, catch up to 100, launch to 100. */
  const cpbus_due_op ops[4] = {{CPBUS_DUE_ARM, 0, 10}, {CPBUS_DUE_ONESHOT, 1, 25}, {CPBUS_DUE_LAUNCH, 0, 5},
                               {CPBUS_DUE_CATCHUP, 0, 100}};
  const cpbus_due_op launch = {CPBUS_DUE_LAUNCH, 0, 100};
  cpbus_due_op all[5];
  cpbus_due_fire out[4];
  size_t n = 0, i;
  int bad = 0;
#define CHECK(cond) do { if (!(cond)) { printf("failed: %s\n", #cond); bad++; } } while (0)
  CHECK(CPBUS_CFG_DROP_MISSED_TICKS == 0x10u);
  CHECK((CPBUS_CFG_DROP_MISSED_TICKS & (CPBUS_CFG_LOSSLESS | CPBUS_CFG_DIGEST | CPBUS_CFG_SPARSE_TICKS |
                                        CPBUS_CFG_SPARSE_RECORDS)) == 0);
  CHECK(CPBUS_DUE_CATCHUP == 6);
  for (i = 0; i < 4; i++) all[i] = ops[i];
  all[4] = launch;
  CHECK(p_trace(all, 5, 2, 1, out, 4, &n) == CPBUS_OK);
  CHECK(n == 2);
  if (n == 2) {   /* the periodic slot fires once, at 100, and next at 110; the one-shot is untouched */
    CHECK(out[0].launch == 1 && out[0].slot == 0 && out[0].ticks == 1 && out[0].next_due == 110);
    CHECK(out[1].launch == 1 && out[1].slot == 1 && out[1].ticks == 1 && out[1].next_due == UINT64_MAX);
  }
  all[3].value = 4;   /* a catch-up behind the last launch */
  CHECK(p_trace(all, 4, 2, 1, out, 4, &n) == CPBUS_EINVAL);
  printf(bad ? "FAILED (%d)\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
