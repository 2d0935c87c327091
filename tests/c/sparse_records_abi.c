/* sparse_records_abi.c — CPBUS_CFG_SPARSE_RECORDS and cpbus_sparse_plan from plain C99, the way cgo-generated code sees
 * them: the entry point is taken with its declared type (a mismatch is a compile error under -Werror), the plan entry has
 * the documented layout, cpbus_create and cpbus_group_create refuse the flag without touching a device, and a small plan
 * comes out as the header says.  Exit code 0 = all checks passed.
 * Build: gcc -std=c99 -Wall -Wextra -Werror -pedantic -I include tests/c/sparse_records_abi.c -L containerpilot_b200 -lcpbus */
#include <stddef.h>
#include <stdio.h>

#include "cpbus.h"

int main(void) {
  int (*p_plan)(const uint32_t*, const uint8_t*, uint32_t, const cpbus_pair*, const uint32_t*, uint32_t, const cpbus_event*,
                size_t, const uint32_t*, size_t, uint32_t, size_t, size_t, cpbus_plan_entry*, size_t, uint32_t*, size_t,
                size_t*, size_t*) = cpbus_sparse_plan;
  cpbus_config cfg = {0};
  cpbus_t* bus = NULL;
  cpbus_group_t* g = NULL;
  const int32_t devices[1] = {0};
  /* subscribers 0..3: mask {1}, mask {}, case {2, 7}, mask {2} (unsubscribed); records: code 1, {2, 7}, unicast to 1 */
  const uint32_t masks[4] = {1u << 1, 0u, 0u, 1u << 2};
  const uint8_t active[4] = {1, 1, 1, 0};
  cpbus_pair pairs[4 * CPBUS_MAX_PAIRS];
  const uint32_t n_pairs[4] = {0, 0, 1, 0};
  cpbus_event rec[3] = {{0}};
  const uint32_t due[1] = {1}; /* slot 1 of subscriber 0 (K = 2) */
  cpbus_plan_entry out[4];
  uint32_t idx[8];
  size_t n = 0, ni = 0;
  int bad = 0;
#define CHECK(cond) do { if (!(cond)) { printf("failed: %s\n", #cond); bad++; } } while (0)
  pairs[2 * CPBUS_MAX_PAIRS].code = 2; pairs[2 * CPBUS_MAX_PAIRS].source_id = 7;
  rec[0].code = 1; rec[0].target = CPBUS_TARGET_ALL;
  rec[1].code = 2; rec[1].source_id = 7; rec[1].target = CPBUS_TARGET_ALL;
  rec[2].code = 5; rec[2].target = 100 + 1; rec[2].flags = CPBUS_F_UNICAST;
  CHECK(CPBUS_CFG_SPARSE_RECORDS == 0x8u);
  CHECK((CPBUS_CFG_SPARSE_RECORDS & (CPBUS_CFG_LOSSLESS | CPBUS_CFG_DIGEST | CPBUS_CFG_SPARSE_TICKS)) == 0);
  CHECK(sizeof(cpbus_plan_entry) == 16 && offsetof(cpbus_plan_entry, first) == 8 && offsetof(cpbus_plan_entry, count) == 12);
  cfg.n_max_subs = 64; cfg.timers_per_sub = 1; cfg.flags = CPBUS_CFG_SPARSE_RECORDS; cfg.device = -1;
  CHECK(cpbus_create(&cfg, &bus) == CPBUS_EINVAL && bus == NULL);
  cfg.flags = CPBUS_CFG_SPARSE_RECORDS | CPBUS_CFG_SPARSE_TICKS;
  CHECK(cpbus_group_create(&cfg, devices, 1, &g) == CPBUS_EINVAL && g == NULL);
  CHECK(p_plan(masks, active, 4, pairs, n_pairs, 100, rec, 3, due, 1, 2, 32, 1024, out, 4, idx, 8, &n, &ni) == CPBUS_OK);
  CHECK(n == 3 && ni == 3);
  if (n == 3 && ni == 3) {
    CHECK(out[0].local == 0 && out[0].due_bits == 2 && out[0].first == 0 && out[0].count == 1 && idx[0] == 0);
    CHECK(out[1].local == 1 && out[1].due_bits == 0 && out[1].first == 1 && out[1].count == 1 && idx[1] == 2);
    CHECK(out[2].local == 2 && out[2].due_bits == 0 && out[2].first == 2 && out[2].count == 1 && idx[2] == 1);
  }
  CHECK(p_plan(masks, active, 4, pairs, n_pairs, 100, rec, 3, due, 1, 2, 2, 1024, out, 4, idx, 8, &n, &ni) == CPBUS_ENOSPC);
  CHECK(p_plan(masks, active, 4, pairs, n_pairs, 100, rec, 3, due, 1, 2, 32, 2, out, 4, idx, 8, &n, &ni) == CPBUS_ENOSPC);
  CHECK(p_plan(masks, active, 4, pairs, n_pairs, 100, rec, 3, due, 1, 3, 32, 1024, out, 4, idx, 8, &n, &ni) == CPBUS_EINVAL);
  printf(bad ? "FAILED (%d)\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
