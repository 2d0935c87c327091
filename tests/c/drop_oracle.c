/* drop_oracle.c — the oracle's side of CPBUS_CFG_DROP_MISSED_TICKS.  TEST INFRASTRUCTURE.
 *
 * The oracle itself (oracle/cpbus_oracle.c) is included whole, so that the catch-up below works on its own timer state and
 * its firing loop (orc_advance) delivers what is left.  The result is loaded next to oracle/libcpbus_oracle.so and called on
 * the handles that library creates (the same source, hence the same struct layout); tests/drop_oracle.py compiles and binds it.
 * Build: gcc -O2 -fPIC -std=gnu11 -shared tests/c/drop_oracle.c -o libdrop_oracle.so
 *
 * The rule follows the Go runtime's ticker (Go 1.9, runtime/time.go): a ticker sends without blocking into a channel that
 * holds one tick, and after a late wake-up its next `when` is the first point of its grid after now.  NewEventTimer
 * (events/timer.go:40-71) reads that channel, so a clock step across several periods delivers one TimerExpired, the one due
 * last.  The oracle fires at advance time, so the step it catches up over is exactly (clock, now_ns]. */
#include "../../oracle/cpbus_oracle.c"

/* orc_advance with missed ticks dropped: every armed periodic timer with k >= 2 firings due in (clock, now_ns] first moves
 * k - 1 periods on, counting the skipped firings in its ordinal, so that orc_advance delivers only the last (due at the
 * largest point of its grid <= now_ns below ORC_NEVER).  Idempotent: a retry after ORC_EAGAIN finds nothing more to skip
 * for the same now_ns. */
int orc_advance_drop_missed(orc_bus* b, uint64_t now_ns) {
  if (now_ns < b->now) return ORC_EINVAL;
  const uint64_t w = now_ns < ORC_NEVER - 1 ? now_ns : ORC_NEVER - 1;
  for (uint32_t i = 0; i < b->n_next; i++) {
    orc_sub* s = &b->subs[i];
    if (!s->n_active_timers) continue;
    for (uint32_t k = 0; k < b->K; k++) {
      orc_timer* t = &s->timers[k];
      if (!t->active || t->oneshot || t->next_due == ORC_NEVER || t->next_due <= b->now || t->next_due > w) continue;
      if (w - t->next_due < t->period) continue;   /* one firing due: nothing to drop */
      const uint64_t skip = (w - t->next_due) / t->period;
      t->next_due += skip * t->period;
      t->fired += (uint32_t)skip;
    }
  }
  return orc_advance(b, now_ns);
}
