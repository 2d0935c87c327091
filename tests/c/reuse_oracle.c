/* reuse_oracle.c — the oracle's side of subscriber id reuse (cpbus_release_many, cpbus_subscribe_list).  TEST INFRASTRUCTURE.
 *
 * The oracle itself (oracle/cpbus_oracle.c) is included whole, so that a released slot and its next occupant are built from
 * its own state and its own subscribe (orc_subscribe_pairs) rather than from library code.  The result is loaded next to
 * oracle/libcpbus_oracle.so and called on the handles that library creates (the same source, hence the same struct layout);
 * tests/reuse_oracle.py compiles and binds it.
 * Build: gcc -O2 -fPIC -std=gnu11 -shared tests/c/reuse_oracle.c -o libreuse_oracle.so
 *
 * Ids behave like file descriptors: an unsubscribed subscriber's mailbox stays readable until it is released; a released
 * slot holds nothing (`ever` = 0 marks it) and is handed out again, lowest free id first, by orc_subscribe_list. */
#include "../../oracle/cpbus_oracle.c"

static int released(const orc_sub* s) { return !s->ever; }

/* 1 when gid was handed out and has been released since (and not handed out again) */
int orc_released(orc_bus* b, uint32_t gid) {
  orc_sub* s = sub_at(b, gid);
  return s && released(s);
}

/* ids ever handed out: the high-water mark of the id space */
uint32_t orc_high_water(orc_bus* b) { return b->n_next; }

/* 1 when gid is subscribed */
int orc_active(orc_bus* b, uint32_t gid) {
  orc_sub* s = sub_at(b, gid);
  return s && s->active;
}

/* armed timers over the whole bus */
uint32_t orc_n_timers(orc_bus* b) { return b->n_timers; }

/* ORC_ENOENT: never handed out or already released; ORC_EINVAL: still subscribed.  Otherwise the slot's records, count,
 * digest, mask and cases are gone and its timers idle (unsubscribing already disarmed them). */
int orc_release(orc_bus* b, uint32_t gid) {
  orc_sub* s = sub_at(b, gid);
  if (!s || released(s)) return ORC_ENOENT;
  if (s->active) return ORC_EINVAL;
  orc_timer* timers = s->timers;
  free(s->box);
  memset(s, 0, sizeof(*s));   /* ever = 0 */
  s->timers = timers;
  if (timers) memset(timers, 0, b->K * sizeof(orc_timer));
  return ORC_OK;
}

/* n subscribers on the lowest free ids (released slots ascending, then fresh ones), all or nothing: subscriber i gets masks[i]
 * and the first n_pairs[i] cases of row i of codes / sources (ORC_MAX_PAIRS per row; n_pairs NULL: none).  out[i] = its id. */
int orc_subscribe_list(orc_bus* b, const uint32_t* masks, const uint32_t* codes, const uint32_t* sources,
                       const uint32_t* n_pairs, uint32_t n, uint32_t* out) {
  uint64_t free_ids = b->n_max - b->n_next;
  for (uint32_t i = 0; i < b->n_next; i++) free_ids += released(&b->subs[i]);
  if (free_ids < n) return ORC_ENOSPC;
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t np = n_pairs ? n_pairs[i] : 0;
    if (np > ORC_MAX_PAIRS) return ORC_EINVAL;
    for (uint32_t j = 0; j < np; j++) if (codes[(size_t)i * ORC_MAX_PAIRS + j] >= ORC_N_CODES) return ORC_EINVAL;
  }
  uint32_t scan = 0;
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t np = n_pairs ? n_pairs[i] : 0;
    const uint32_t* c = np ? codes + (size_t)i * ORC_MAX_PAIRS : NULL;
    const uint32_t* src = np ? sources + (size_t)i * ORC_MAX_PAIRS : NULL;
    while (scan < b->n_next && !released(&b->subs[scan])) scan++;
    if (scan == b->n_next) {   /* a fresh id: the oracle's own subscribe */
      int rc = orc_subscribe_pairs(b, masks[i], c, src, np, &out[i]);
      if (rc) return rc;
      scan = b->n_next;
      continue;
    }
    orc_sub* s = &b->subs[scan];   /* a released slot: what orc_subscribe leaves in a fresh one, on the same timer array */
    s->active = 1; s->ever = 1; s->mask = masks[i];
    if (b->K && !s->timers) s->timers = (orc_timer*)calloc(b->K, sizeof(orc_timer));
    s->n_pairs = np;
    for (uint32_t j = 0; j < np; j++) { s->pair_code[j] = c[j]; s->pair_src[j] = src[j]; }
    b->done++;
    out[i] = b->base + scan++;
  }
  return ORC_OK;
}
