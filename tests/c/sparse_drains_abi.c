/* sparse_drains_abi.c — CPBUS_CFG_SPARSE_DRAINS and cpbus_ready_trace from plain C99, the way cgo-generated code sees
 * them: the entry point is taken with its declared type (a mismatch is a compile error under -Werror), the op has the
 * documented layout, cpbus_create and cpbus_group_create refuse the flag without touching a device, and a small trace
 * comes out as the header says.  Exit code 0 = all checks passed.
 * Build: gcc -std=c99 -Wall -Wextra -Werror -pedantic -I include tests/c/sparse_drains_abi.c -L containerpilot_b200 -lcpbus */
#include <stddef.h>
#include <stdio.h>

#include "cpbus.h"

int main(void) {
  int (*p_trace)(const cpbus_ready_op*, size_t, const uint32_t*, size_t, uint32_t, size_t, uint32_t*, size_t, int64_t*,
                 size_t*) = cpbus_ready_trace;
  cpbus_config cfg = {0};
  cpbus_t* bus = NULL;
  cpbus_group_t* g = NULL;
  const int32_t devices[1] = {0};
  /* 8 mailboxes: a sparse launch to {2, 5}; a drain of everything that takes both; then a drain that needs no launch */
  const uint32_t ids[4] = {2, 5, 2, 5};
  cpbus_ready_op ops[5] = {{0}};
  uint32_t out[8];
  int64_t counts[5];
  size_t n = 0;
  int bad = 0;
#define CHECK(cond) do { if (!(cond)) { printf("failed: %s\n", #cond); bad++; } } while (0)
  ops[0].kind = CPBUS_READY_SPARSE; ops[0].ids = 0; ops[0].n_ids = 2;
  ops[1].kind = CPBUS_READY_DRAIN; ops[1].ticket = 1; ops[1].first = 0; ops[1].n = 8;
  ops[2].kind = CPBUS_READY_END; ops[2].ticket = 1; ops[2].ids = 2; ops[2].n_ids = 2; ops[2].cut = 8;
  ops[3].kind = CPBUS_READY_TAKE; ops[3].ticket = 2; ops[3].first = 0; ops[3].n = 8;
  ops[4].kind = CPBUS_READY_END; ops[4].ticket = 2; ops[4].cut = 8;
  CHECK(CPBUS_CFG_SPARSE_DRAINS == 0x20u);
  CHECK((CPBUS_CFG_SPARSE_DRAINS & (CPBUS_CFG_LOSSLESS | CPBUS_CFG_DIGEST | CPBUS_CFG_SPARSE_TICKS | CPBUS_CFG_SPARSE_RECORDS |
                                    CPBUS_CFG_DROP_MISSED_TICKS)) == 0);
  CHECK(sizeof(cpbus_ready_op) == 32 && offsetof(cpbus_ready_op, ids) == 16 && offsetof(cpbus_ready_op, cut) == 24);
  cfg.n_max_subs = 64; cfg.timers_per_sub = 1; cfg.flags = CPBUS_CFG_SPARSE_DRAINS; cfg.device = -1;
  CHECK(cpbus_create(&cfg, &bus) == CPBUS_EINVAL && bus == NULL);
  cfg.flags = CPBUS_CFG_SPARSE_DRAINS | CPBUS_CFG_SPARSE_TICKS;
  CHECK(cpbus_group_create(&cfg, devices, 1, &g) == CPBUS_EINVAL && g == NULL);
  CHECK(p_trace(ops, 5, ids, 4, 8, 1024, out, 8, counts, &n) == CPBUS_OK);
  CHECK(n == 2 && counts[1] == 2 && counts[3] == 0 && counts[0] == 0 && counts[2] == 0 && counts[4] == 0);
  if (n == 2) CHECK(out[0] == 2 && out[1] == 5);
  ops[4].ticket = 3;
  CHECK(p_trace(ops, 5, ids, 4, 8, 1024, out, 8, counts, &n) == CPBUS_ENOENT);
  CHECK(p_trace(ops, 5, ids, 4, 4, 1024, out, 8, counts, &n) == CPBUS_EINVAL); /* id 5 outside 4 mailboxes */
  printf(bad ? "FAILED (%d)\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
