/* sparse_abi.c — CPBUS_CFG_SPARSE_TICKS and cpbus_due_trace from plain C99, the way cgo-generated code sees them: the
 * entry point is taken with its declared type (a mismatch is a compile error under -Werror), the structs have the documented
 * layout, a group refuses the flag before it touches a device, and a two-launch trace fires what the header says.
 * Exit code 0 = all checks passed.
 * Build: gcc -std=c99 -Wall -Wextra -Werror -pedantic -I include tests/c/sparse_abi.c -L containerpilot_b200 -lcpbus */
#include <stddef.h>
#include <stdio.h>

#include "cpbus.h"

int main(void) {
  int (*p_trace)(const cpbus_due_op*, size_t, uint32_t, uint32_t, cpbus_due_fire*, size_t, size_t*) = cpbus_due_trace;
  cpbus_config cfg = {0};
  cpbus_group_t* g = NULL;
  const int32_t devices[1] = {0};
  /* slot 0: periodic, 10 ns; slot 1: one-shot at 25 ns; launches to 20 and 30 */
  const cpbus_due_op ops[5] = {{CPBUS_DUE_ARM, 0, 10}, {CPBUS_DUE_ONESHOT, 1, 25}, {CPBUS_DUE_LAUNCH, 0, 20},
                               {CPBUS_DUE_CLOCK, 0, 20}, {CPBUS_DUE_LAUNCH, 0, 30}};
  cpbus_due_fire out[4];
  size_t n = 0;
  int bad = 0;
#define CHECK(cond) do { if (!(cond)) { printf("failed: %s\n", #cond); bad++; } } while (0)
  CHECK(CPBUS_CFG_SPARSE_TICKS == 0x4u);
  CHECK((CPBUS_CFG_SPARSE_TICKS & (CPBUS_CFG_LOSSLESS | CPBUS_CFG_DIGEST)) == 0);
  CHECK(sizeof(cpbus_due_op) == 16 && offsetof(cpbus_due_op, value) == 8);
  CHECK(sizeof(cpbus_due_fire) == 32 && offsetof(cpbus_due_fire, slot) == 8 && offsetof(cpbus_due_fire, ticks) == 16);
  cfg.n_max_subs = 64; cfg.timers_per_sub = 1; cfg.flags = CPBUS_CFG_SPARSE_TICKS; cfg.device = -1;
  CHECK(cpbus_group_create(&cfg, devices, 1, &g) == CPBUS_EINVAL && g == NULL);
  CHECK(p_trace(ops, 5, 2, 1, out, 4, &n) == CPBUS_OK);
  CHECK(n == 3);
  if (n == 3) {
    CHECK(out[0].launch == 0 && out[0].slot == 0 && out[0].ticks == 2 && out[0].next_due == 30);
    CHECK(out[1].launch == 1 && out[1].slot == 0 && out[1].ticks == 1 && out[1].next_due == 40);
    CHECK(out[2].launch == 1 && out[2].slot == 1 && out[2].ticks == 1 && out[2].next_due == UINT64_MAX);
  }
  CHECK(p_trace(ops, 5, 2, 3, out, 4, &n) == CPBUS_EINVAL);   /* K = 3 */
  CHECK(p_trace(ops, 5, 1, 1, out, 4, &n) == CPBUS_EINVAL);   /* slot 1 out of range */
  printf(bad ? "FAILED (%d)\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
