/* lag_oracle.c — the oracle's side of the consumer backlog queries (cpbus_lagging, cpbus_blockers).  TEST INFRASTRUCTURE.
 *
 * The oracle itself (oracle/cpbus_oracle.c) is included whole, so that these two observers are built from its own state and
 * its own rules — `wants`, `mailbox_full`, `due_after` and the orc_advance timer walk — rather than from library code.  The
 * result is loaded next to oracle/libcpbus_oracle.so and called on the handles that library creates (the same source, hence
 * the same struct layout); tests/lag_oracle.py compiles and binds it.
 * Build: gcc -O2 -fPIC -std=gnu11 -shared -I oracle tests/c/lag_oracle.c -o liblag_oracle.so */
#include "../../oracle/cpbus_oracle.c"

/* Records the mailbox holds (delivered, not yet consumed); with mailbox_cap > 0 at most mailbox_cap, the ring. */
uint64_t orc_backlog(orc_bus* b, uint32_t gid) {
  orc_sub* s = sub_at(b, gid);
  if (!s) return 0;
  uint64_t held = s->count - s->consumed;
  return (b->cap && held > b->cap) ? b->cap : held;
}

/* Who the Go publisher would sit on next, at the current state.  Per subscriber, the timer goroutines' sends due by t come
 * first (orc_advance: oldest due first, ties by slot), then the publish or direct send of `next` (NULL: ticks only); each
 * send into a full mailbox blocks (subscriber.go:31).  Walks copies of the timers and of the fill level: nothing changes.
 * out receives the first `cap` ids, ascending; returns how many there are. */
size_t orc_blockers(orc_bus* b, const orc_event* next, uint64_t t, uint32_t* out, size_t cap) {
  size_t n = 0;
  if (!b->cap) return 0;   /* unbounded mailboxes never block */
  for (uint32_t i = 0; i < b->n_next; i++) {
    const orc_sub* s = &b->subs[i];
    if (!s->active) continue;
    orc_sub fill = *s;     /* only count / consumed change below: mailbox_full reads nothing else */
    int blocked = 0;
    if (s->n_active_timers) {
      orc_timer tm[8];     /* timers_per_sub <= 8 */
      for (uint32_t k = 0; k < b->K; k++) tm[k] = s->timers[k];
      for (;;) {
        int best = -1;
        for (uint32_t k = 0; k < b->K; k++) {
          if (!tm[k].active || tm[k].next_due > t || tm[k].next_due == ORC_NEVER) continue;
          if (best < 0 || tm[k].next_due < tm[best].next_due) best = (int)k;
        }
        if (best < 0) break;
        if (mailbox_full(b, &fill)) { blocked = 1; break; }
        fill.count++;
        if (tm[best].oneshot) tm[best].active = 0;
        else tm[best].next_due = due_after(tm[best].next_due, tm[best].period);
      }
    }
    if (!blocked && next) {
      const int want = next->target == ORC_TARGET_ALL ? wants(s, next->code, next->source_id) : next->target == b->base + i;
      blocked = want && mailbox_full(b, &fill);
    }
    if (blocked) {
      if (n < cap) out[n] = b->base + i;
      n++;
    }
  }
  return n;
}
