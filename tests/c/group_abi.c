/* group_abi.c — the cpbus_group_* declarations of include/cpbus.h from plain C99, the way cgo-generated code sees them:
 * every entry point is taken with its declared type (a mismatch is a compile error under -Werror), and each refuses a NULL
 * group with CPBUS_EINVAL before it touches a device.  Exit code 0 = all checks passed.
 * Build: gcc -std=c99 -Wall -Wextra -Werror -pedantic -I include tests/c/group_abi.c -L containerpilot_b200 -lcpbus */
#include <stdio.h>

#include "cpbus.h"

int main(void) {
  int (*p_create)(const cpbus_config*, const int32_t*, uint32_t, cpbus_group_t**) = cpbus_group_create;
  int (*p_destroy)(cpbus_group_t*) = cpbus_group_destroy;
  int (*p_intern)(cpbus_group_t*, const char*, size_t, uint32_t*) = cpbus_group_intern;
  int (*p_intern_ephemeral)(cpbus_group_t*, const char*, size_t, uint32_t*) = cpbus_group_intern_ephemeral;
  int (*p_source)(cpbus_group_t*, uint32_t, char*, size_t, size_t*) = cpbus_group_source;
  int (*p_subscribe)(cpbus_group_t*, uint32_t, uint32_t*) = cpbus_group_subscribe;
  int (*p_subscribe_many)(cpbus_group_t*, const uint32_t*, uint32_t, uint32_t*) = cpbus_group_subscribe_many;
  int (*p_subscribe_pairs)(cpbus_group_t*, uint32_t, const cpbus_pair*, uint32_t, uint32_t*) = cpbus_group_subscribe_pairs;
  int (*p_subscribe_pairs_many)(cpbus_group_t*, const uint32_t*, const cpbus_pair*, const uint32_t*, uint32_t, uint32_t*) = cpbus_group_subscribe_pairs_many;
  int (*p_unsubscribe)(cpbus_group_t*, uint32_t) = cpbus_group_unsubscribe;
  int (*p_set_mask)(cpbus_group_t*, uint32_t, uint32_t) = cpbus_group_set_mask;
  int (*p_timer_add)(cpbus_group_t*, uint32_t, uint64_t, uint32_t, int, uint32_t*) = cpbus_group_timer_add;
  int (*p_timer_add_many)(cpbus_group_t*, uint32_t, uint32_t, uint64_t, const uint32_t*, uint32_t, int) = cpbus_group_timer_add_many;
  int (*p_timer_cancel)(cpbus_group_t*, uint32_t) = cpbus_group_timer_cancel;
  int (*p_publish)(cpbus_group_t*, const cpbus_event*, size_t) = cpbus_group_publish;
  int (*p_send)(cpbus_group_t*, uint32_t, const cpbus_event*) = cpbus_group_send;
  int (*p_advance)(cpbus_group_t*, uint64_t) = cpbus_group_advance;
  int (*p_flush)(cpbus_group_t*) = cpbus_group_flush;
  int (*p_sync)(cpbus_group_t*) = cpbus_group_sync;
  int (*p_drain)(cpbus_group_t*, uint32_t, cpbus_event*, size_t, size_t*, uint64_t*) = cpbus_group_drain;
  int (*p_drain_ready)(cpbus_group_t*, uint32_t, uint32_t, uint32_t, cpbus_event*, size_t, cpbus_ready*, size_t, size_t*, size_t*, uint32_t*) = cpbus_group_drain_ready;
  int (*p_consume_all)(cpbus_group_t*) = cpbus_group_consume_all;
  int (*p_peek_window)(cpbus_group_t*, uint32_t, cpbus_event*, size_t, size_t*) = cpbus_group_peek_window;
  int (*p_digest)(cpbus_group_t*, uint32_t, uint32_t, cpbus_digest_t*) = cpbus_group_digest;
  int (*p_digest_fold)(cpbus_group_t*, uint32_t, uint32_t, uint64_t*) = cpbus_group_digest_fold;
  int (*p_debug_events)(cpbus_group_t*, cpbus_event*, size_t, size_t*) = cpbus_group_debug_events;
  int (*p_stats)(cpbus_group_t*, cpbus_stats_t*) = cpbus_group_stats;
  int (*p_publish_counts)(cpbus_group_t*, cpbus_pair_count*, size_t, size_t*) = cpbus_group_publish_counts;
  cpbus_config cfg = {0};
  cpbus_group_t* g = NULL;
  uint32_t id = 0;
  size_t n = 0, m = 0;
  uint64_t u = 0, fold[4];
  cpbus_event ev;
  cpbus_stats_t st;
  cpbus_ready ready;
  cpbus_digest_t dg;
  cpbus_pair_count pc;
  int32_t dev = 0;
  int bad = 0;
  (void)u;
#define EXPECT_EINVAL(call) do { if ((call) != CPBUS_EINVAL) { printf("not EINVAL: %s\n", #call); bad++; } } while (0)
  EXPECT_EINVAL(p_create(NULL, &dev, 1, &g));
  EXPECT_EINVAL(p_create(&cfg, NULL, 1, &g));
  EXPECT_EINVAL(p_create(&cfg, &dev, 0, &g));
  EXPECT_EINVAL(p_destroy(NULL));
  EXPECT_EINVAL(p_intern(NULL, "a", 1, &id));
  EXPECT_EINVAL(p_intern_ephemeral(NULL, "a", 1, &id));
  EXPECT_EINVAL(p_source(NULL, 0, NULL, 0, &n));
  EXPECT_EINVAL(p_subscribe(NULL, CPBUS_MASK_ALL, &id));
  EXPECT_EINVAL(p_subscribe_many(NULL, &id, 1, &id));
  EXPECT_EINVAL(p_subscribe_pairs(NULL, 0, NULL, 0, &id));
  EXPECT_EINVAL(p_subscribe_pairs_many(NULL, &id, NULL, &id, 1, &id));
  EXPECT_EINVAL(p_unsubscribe(NULL, 0));
  EXPECT_EINVAL(p_set_mask(NULL, 0, 0));
  EXPECT_EINVAL(p_timer_add(NULL, 0, 1, 0, 0, &id));
  EXPECT_EINVAL(p_timer_add_many(NULL, 0, 1, 1, NULL, 0, 0));
  EXPECT_EINVAL(p_timer_cancel(NULL, 0));
  EXPECT_EINVAL(p_publish(NULL, &ev, 1));
  EXPECT_EINVAL(p_send(NULL, 0, &ev));
  EXPECT_EINVAL(p_advance(NULL, 1));
  EXPECT_EINVAL(p_flush(NULL));
  EXPECT_EINVAL(p_sync(NULL));
  EXPECT_EINVAL(p_drain(NULL, 0, &ev, 1, &n, &u));
  EXPECT_EINVAL(p_drain_ready(NULL, 0, 1, 0, &ev, 1024, &ready, 1, &n, &m, &id));
  EXPECT_EINVAL(p_consume_all(NULL));
  EXPECT_EINVAL(p_peek_window(NULL, 0, &ev, 1, &n));
  EXPECT_EINVAL(p_digest(NULL, 0, 1, &dg));
  EXPECT_EINVAL(p_digest_fold(NULL, 0, 1, fold));
  EXPECT_EINVAL(p_debug_events(NULL, &ev, 1, &n));
  EXPECT_EINVAL(p_stats(NULL, &st));
  EXPECT_EINVAL(p_publish_counts(NULL, &pc, 1, &n));
  if (g != NULL) { printf("a refused create wrote *out\n"); bad++; }
  printf(bad ? "FAILED (%d)\n" : "PASS\n", bad);
  return bad ? 1 : 0;
}
