/*
 * cpbus_oracle.c — CPU oracle (TEST INFRASTRUCTURE, see cpbus_oracle.h).
 *
 * Plain-C restatement of /root/reference/events/{bus,subscriber,timer,events,
 * eventcode_string}.go under a virtual clock.  It processes one event at a
 * time exactly like the Go bus does; it has no notion of batches, shared
 * memory, filters pushed into kernels, or ring wrap tricks — so agreement with
 * the CUDA path is evidence about the CUDA path.
 */
#include "cpbus_oracle.h"

#include <stdlib.h>
#include <string.h>

#define ORC_TARGET_ALL 0xFFFFFFFFu
#define ORC_F_TICK 0x1u
#define ORC_F_UNICAST 0x2u
#define ORC_TIMER_EXPIRED 8u   /* events/events.go:30 */
#define ORC_METRIC 13u         /* events/events.go:35 */
#define ORC_N_CODES 17

/* ------------------------------------------------------------------ hash --- */
/* Spec of the delivered-sequence digest (shared by contract with
 * include/cpbus.h: cpbus_record_hash / cpbus_digest_multiplier).  Not from the
 * reference: the reference has no digest; it exists to compare 10^11-record
 * delivered sequences without retaining them. */
static const uint64_t K0 = 0x9E3779B97F4A7C15ull, K1 = 0xBF58476D1CE4E5B9ull,
                      K2 = 0x94D049BB133111EBull, K3 = 0xD6E8FEB86659FD93ull,
                      K4 = 0xA0761D6478BD642Full;
uint64_t orc_digest_multiplier(void) { return 0x9E3779B97F4A7C15ull; }

uint64_t orc_record_hash(const orc_event* e) {
  uint64_t w0 = e->seq, w1 = e->ts_ns;
  uint64_t w2 = (uint64_t)e->code | ((uint64_t)e->source_id << 32);
  uint64_t w3 = (uint64_t)e->target | ((uint64_t)e->flags << 32);
  uint64_t x = (w0 + K4) * K0; x ^= x >> 32;
  x = (x + w1) * K1; x ^= x >> 32;
  x = (x + w2) * K2; x ^= x >> 32;
  x = (x + w3) * K3; x ^= x >> 29;
  return x;
}

/* ---------------------------------------------------------------- state --- */
typedef struct orc_timer {
  int active, oneshot;
  uint64_t period, next_due;
  uint32_t source_id, fired;
} orc_timer;

typedef struct orc_sub {
  int active, ever;
  uint32_t mask;
  uint64_t count;      /* records ever delivered                       */
  uint64_t consumed;   /* records taken by orc_consume                 */
  uint64_t digest;
  orc_event* box;      /* keep_window==0: growable array; else ring[W] */
  size_t box_cap;
  orc_timer* timers;   /* [timers_per_sub] */
  uint32_t n_active_timers;
  uint32_t n_pairs;    /* second-level filter: exact {code, source} cases of the consumer's switch */
  uint32_t pair_code[ORC_MAX_PAIRS], pair_src[ORC_MAX_PAIRS];
} orc_sub;

struct orc_bus {
  /* events/bus.go:12-22 */
  orc_sub* subs;       /* registry map[*Subscriber]bool, keyed by id   */
  uint32_t n_max, n_next;
  int reload;
  long done;           /* sync.WaitGroup counter                        */
  int head, tail;      /* debug ring cursors                            */
  orc_event buf[10];   /* debug ring (code, source_id only are meaningful) */
  /* virtual clock + bookkeeping */
  uint64_t now, seq, deliveries, ticks;
  uint64_t by_code[ORC_N_CODES];
  uint64_t min_due;    /* early-out for orc_advance                      */
  uint32_t K, W, cap, base;
  uint32_t n_timers;
};

/* NewEventBus — events/bus.go:72-88: ring of 10 zero Events, head=-1, tail=0 */
orc_bus* orc_new(uint32_t n_max_subs, uint32_t timers_per_sub, uint32_t keep_window,
                 uint32_t mailbox_cap, uint32_t sub_id_base) {
  orc_bus* b = (orc_bus*)calloc(1, sizeof(*b));
  if (!b) return NULL;
  b->subs = (orc_sub*)calloc(n_max_subs ? n_max_subs : 1, sizeof(orc_sub));
  if (!b->subs) { free(b); return NULL; }
  b->n_max = n_max_subs; b->K = timers_per_sub; b->W = keep_window;
  b->cap = mailbox_cap; b->base = sub_id_base;
  b->head = -1; b->tail = 0; b->reload = 0;
  b->min_due = UINT64_MAX;
  return b;
}

void orc_free(orc_bus* b) {
  if (!b) return;
  for (uint32_t i = 0; i < b->n_next; i++) { free(b->subs[i].box); free(b->subs[i].timers); }
  free(b->subs); free(b);
}

static orc_sub* sub_at(orc_bus* b, uint32_t gid) {
  uint32_t i = gid - b->base;
  if (gid < b->base || i >= b->n_next) return NULL;
  return &b->subs[i];
}

/* Subscriber.Receive — events/subscriber.go:30-32: `sub.Rx <- event`, a FIFO
 * append to the subscriber's buffered channel. */
static void receive(orc_bus* b, orc_sub* s, const orc_event* e) {
  if (b->W == 0) {
    if (s->count >= s->box_cap) {
      size_t nc = s->box_cap ? s->box_cap * 2 : 64;
      s->box = (orc_event*)realloc(s->box, nc * sizeof(orc_event));
      s->box_cap = nc;
    }
    s->box[s->count] = *e;
  } else {
    if (!s->box) { s->box = (orc_event*)calloc(b->W, sizeof(orc_event)); s->box_cap = b->W; }
    s->box[s->count % b->W] = *e;
  }
  s->count++;
  s->digest = s->digest * orc_digest_multiplier() + orc_record_hash(e);
  b->deliveries++;
}

static int mailbox_full(const orc_bus* b, const orc_sub* s) {
  return b->cap && (s->count - s->consumed) >= b->cap;
}

/* enqueue — events/bus.go:24-31 */
static int ring_mod(int p) { return p % 10; }                 /* bus.go:56-58 */
static void enqueue(orc_bus* b, const orc_event* e) {
  b->buf[ring_mod(b->head + 1)] = *e;
  int old = b->head;
  b->head = (b->head + 1) % 10;
  if (old != -1 && b->head == b->tail) b->tail = ring_mod(b->tail + 1);
}

/* DebugEvents — events/bus.go:34-54 (without the 100 ms sleep) */
size_t orc_debug_events(orc_bus* b, orc_event* out, size_t cap) {
  size_t n = 0;
  for (;;) {
    if (b->head == -1) break;
    orc_event e = b->buf[ring_mod(b->tail)];
    if (b->tail == b->head) { b->head = -1; b->tail = 0; }
    else b->tail = ring_mod(b->tail + 1);
    if (e.code == 0 && e.source_id == 0) break;   /* event == NonEvent (events.go:45; "" interns to 0) */
    if (n < cap) out[n] = e;
    n++;
  }
  return n;
}

/* Register / Unregister — events/bus.go:91-102 */
int orc_register(orc_bus* b) { b->done++; return ORC_OK; }
int orc_unregister(orc_bus* b) { if (b->done <= 0) return ORC_ECLOSED; b->done--; return ORC_OK; }

/* Subscribe — events/bus.go:105-111.  mask is the pushed-down consumer switch
 * (SURVEY F3); 0x1FFFF is the reference behaviour. */
int orc_subscribe(orc_bus* b, uint32_t mask, uint32_t* sub_id) {
  if (b->n_next >= b->n_max) return ORC_ENOSPC;
  orc_sub* s = &b->subs[b->n_next];
  memset(s, 0, sizeof(*s));
  s->active = 1; s->ever = 1; s->mask = mask;
  if (b->K) s->timers = (orc_timer*)calloc(b->K, sizeof(orc_timer));
  if (sub_id) *sub_id = b->base + b->n_next;
  b->n_next++;
  b->done++;
  return ORC_OK;
}

/* A consumer's `switch event { case events.Event{Code, Source}: ... }` (jobs/jobs.go:188-231) compares whole
 * Event values: every case is an exact {code, source} pair.  A subscriber may push that down as well: a broadcast
 * event is wanted when its code is in `mask` (any source) OR {code, source_id} is one of the pairs. */
int orc_subscribe_pairs(orc_bus* b, uint32_t mask, const uint32_t* codes, const uint32_t* sources, uint32_t n_pairs,
                        uint32_t* sub_id) {
  if (n_pairs > ORC_MAX_PAIRS || (n_pairs && (!codes || !sources))) return ORC_EINVAL;
  for (uint32_t j = 0; j < n_pairs; j++) if (codes[j] >= ORC_N_CODES) return ORC_EINVAL;
  uint32_t id = 0;
  int r = orc_subscribe(b, mask, &id);
  if (r) return r;
  orc_sub* s = &b->subs[id - b->base];
  s->n_pairs = n_pairs;
  for (uint32_t j = 0; j < n_pairs; j++) { s->pair_code[j] = codes[j]; s->pair_src[j] = sources[j]; }
  if (sub_id) *sub_id = id;
  return ORC_OK;
}

/* A broadcast code >= ORC_N_CODES (possible only in complete records) is matched by no mask bit and no pair. */
static int wants(const orc_sub* s, uint32_t code, uint32_t source_id) {
  if (code < ORC_N_CODES && ((s->mask >> code) & 1u)) return 1;
  for (uint32_t j = 0; j < s->n_pairs; j++)
    if (s->pair_code[j] == code && s->pair_src[j] == source_id) return 1;
  return 0;
}

/* Unsubscribe — events/bus.go:114-122.  Done() on an already-unsubscribed
 * subscriber drives the WaitGroup negative => Go panics; here ORC_ECLOSED. */
int orc_unsubscribe(orc_bus* b, uint32_t gid) {
  orc_sub* s = sub_at(b, gid);
  if (!s) return ORC_ENOENT;
  if (!s->active) return ORC_ECLOSED;
  s->active = 0;
  for (uint32_t k = 0; k < b->K; k++)
    if (s->timers[k].active) { s->timers[k].active = 0; b->n_timers--; }
  s->n_active_timers = 0;
  b->done--;
  return ORC_OK;
}

void orc_set_reload(orc_bus* b) { b->reload = 1; }            /* bus.go:150-154 */
int orc_wait(orc_bus* b) { return b->done > 0 ? -1 : b->reload; }  /* bus.go:164-169 */

/* Publish — events/bus.go:125-140 */
int orc_publish(orc_bus* b, uint32_t code, uint32_t source_id) {
  orc_event e = { b->seq, b->now, code, source_id, ORC_TARGET_ALL, 0 };
  /* a full targeted mailbox blocks the publisher (subscriber.go:31); all-or-nothing here */
  if (b->cap)
    for (uint32_t i = 0; i < b->n_next; i++) {
      orc_sub* s = &b->subs[i];
      if (s->active && wants(s, code, source_id) && mailbox_full(b, s)) return ORC_EAGAIN;
    }
  if (code != ORC_METRIC && code < ORC_N_CODES) b->by_code[code]++;   /* bus.go:130-132 */
  for (uint32_t i = 0; i < b->n_next; i++) {                          /* bus.go:134-138 */
    orc_sub* s = &b->subs[i];
    if (!s->active) continue;
    if (wants(s, code, source_id)) receive(b, s, &e);
  }
  enqueue(b, &e);                                                     /* bus.go:139 */
  b->seq++;
  return ORC_OK;
}

/* direct mailbox write: `job.Rx <- ev` (jobs/jobs.go:262), watch.Receive(ev)
 * (watches/watches_test.go:48-50).  Never seen by the debug ring or the counter. */
int orc_receive(orc_bus* b, uint32_t gid, uint32_t code, uint32_t source_id) {
  orc_sub* s = sub_at(b, gid);
  if (!s) return ORC_ENOENT;
  if (!s->active) return ORC_ECLOSED;        /* send on closed channel: Go panics */
  if (mailbox_full(b, s)) return ORC_EAGAIN;
  orc_event e = { b->seq, b->now, code, source_id, gid, ORC_F_UNICAST };
  receive(b, s, &e);
  b->seq++;
  return ORC_OK;
}

/* Due times saturate: a sum past UINT64_MAX - 1 is ORC_NEVER, a due time that never comes (the timer stays armed). */
#define ORC_NEVER UINT64_MAX
static uint64_t due_after(uint64_t t, uint64_t period) {
  return period >= ORC_NEVER - t ? ORC_NEVER : t + period;
}

/* NewEventTimer (events/timer.go:40-71) / NewEventTimeout (timer.go:12-37):
 * first firing one period after creation; periodic repeats every period. */
int orc_timer_add(orc_bus* b, uint32_t gid, uint64_t period_ns, uint32_t source_id, int oneshot, uint32_t* timer_id) {
  orc_sub* s = sub_at(b, gid);
  if (!s) return ORC_ENOENT;
  if (!s->active) return ORC_ECLOSED;
  if (period_ns == 0) return ORC_EINVAL;
  for (uint32_t k = 0; k < b->K; k++) {
    if (s->timers[k].active) continue;
    orc_timer* t = &s->timers[k];
    t->active = 1; t->oneshot = oneshot; t->period = period_ns;
    t->next_due = due_after(b->now, period_ns); t->source_id = source_id; t->fired = 0;
    s->n_active_timers++; b->n_timers++;
    if (t->next_due < b->min_due) b->min_due = t->next_due;
    if (timer_id) *timer_id = (gid - b->base) * b->K + k;
    return ORC_OK;
  }
  return ORC_ENOSPC;
}

/* ctx cancel — timer.go:20-22 / 57-58 */
int orc_timer_cancel(orc_bus* b, uint32_t timer_id) {
  if (!b->K) return ORC_ENOENT;
  uint32_t i = timer_id / b->K, k = timer_id % b->K;
  if (i >= b->n_next) return ORC_ENOENT;
  orc_sub* s = &b->subs[i];
  if (!s->timers[k].active) return ORC_ENOENT;
  s->timers[k].active = 0; s->n_active_timers--; b->n_timers--;
  return ORC_OK;
}

/* The runtime clock reaching now_ns: every armed timer whose due time has
 * passed sends {TimerExpired, name} into its owner's rx (timer.go:31-33,
 * 59-67), oldest due first, ties by slot. */
int orc_advance(orc_bus* b, uint64_t now_ns) {
  if (now_ns < b->now) return ORC_EINVAL;
  if (b->n_timers && now_ns >= b->min_due) {
    uint64_t new_min = UINT64_MAX;
    for (uint32_t i = 0; i < b->n_next; i++) {
      orc_sub* s = &b->subs[i];
      if (!s->n_active_timers) continue;
      for (;;) {
        int best = -1;
        for (uint32_t k = 0; k < b->K; k++) {
          orc_timer* t = &s->timers[k];
          if (!t->active || t->next_due > now_ns || t->next_due == ORC_NEVER) continue;
          if (best < 0 || t->next_due < s->timers[best].next_due) best = (int)k;
        }
        if (best < 0) break;
        orc_timer* t = &s->timers[best];
        if (mailbox_full(b, s)) return ORC_EAGAIN;  /* timer goroutine sits in `rx <- event` */
        orc_event e = { t->fired, t->next_due, ORC_TIMER_EXPIRED, t->source_id, b->base + i, ORC_F_TICK };
        receive(b, s, &e);
        b->ticks++;
        t->fired++;
        if (t->oneshot) { t->active = 0; s->n_active_timers--; b->n_timers--; }
        else t->next_due = due_after(t->next_due, t->period);
      }
      for (uint32_t k = 0; k < b->K; k++)
        if (s->timers[k].active && s->timers[k].next_due < new_min) new_min = s->timers[k].next_due;
    }
    b->min_due = new_min;
  }
  b->now = now_ns;
  return ORC_OK;
}

int orc_publish_many(orc_bus* b, const uint32_t* codes, const uint32_t* sources, size_t n, uint64_t dt_ns) {
  for (size_t i = 0; i < n; i++) {
    if (dt_ns) { int r = orc_advance(b, b->now + dt_ns); if (r) return r; }
    int r = orc_publish(b, codes[i], sources[i]);
    if (r) return r;
  }
  return ORC_OK;
}

/* Complete records, as cpbus_publish_device / cpbus_stream_put(CPBUS_PUT_RAW) take them (bench traces, multi-GPU
 * streams): the clock first reaches each record's ts (timers due by then fire before it, timer.go:59-67); a broadcast
 * record is then delivered exactly like Publish (bus.go:125-140) and a unicast one like Receive (subscriber.go:30-32),
 * but with the record's OWN seq/ts.  A unicast target outside this shard is some other shard's business.  Finally the
 * clock reaches `watermark`.  The bus's own publish ordinal advances by one per record: the next host publish after n
 * records carries the previous ordinal + n, whatever seqs the records carried. */
int orc_publish_records(orc_bus* b, const orc_event* recs, size_t n, uint64_t watermark_ns) {
  for (size_t r = 0; r < n; r++) {
    const orc_event* e = &recs[r];
    if (e->ts_ns > b->now) { int rc = orc_advance(b, e->ts_ns); if (rc) return rc; }
    if (e->target == ORC_TARGET_ALL) {
      if (e->code != ORC_METRIC && e->code < ORC_N_CODES) b->by_code[e->code]++;
      for (uint32_t i = 0; i < b->n_next; i++) {
        orc_sub* s = &b->subs[i];
        if (s->active && wants(s, e->code, e->source_id)) receive(b, s, e);
      }
      enqueue(b, e);
    } else {
      orc_sub* s = sub_at(b, e->target);
      if (s && s->active) receive(b, s, e);
    }
    b->seq++;   /* every record takes one publish ordinal, whatever seq it carries */
  }
  if (watermark_ns > b->now) return orc_advance(b, watermark_ns);
  return ORC_OK;
}

/* ------------------------------------------------------------ observers --- */
uint64_t orc_count(orc_bus* b, uint32_t gid) { orc_sub* s = sub_at(b, gid); return s ? s->count : 0; }
uint64_t orc_digest(orc_bus* b, uint32_t gid) { orc_sub* s = sub_at(b, gid); return s ? s->digest : 0; }
uint64_t orc_now(orc_bus* b) { return b->now; }
uint64_t orc_total_deliveries(orc_bus* b) { return b->deliveries; }
uint64_t orc_total_ticks(orc_bus* b) { return b->ticks; }
uint64_t orc_published_by_code(orc_bus* b, uint32_t code) { return code < ORC_N_CODES ? b->by_code[code] : 0; }

size_t orc_mailbox(orc_bus* b, uint32_t gid, orc_event* out, size_t cap) {
  orc_sub* s = sub_at(b, gid);
  if (!s) return 0;
  uint64_t have = (b->W == 0 || s->count < b->W) ? s->count : b->W;
  uint64_t first = s->count - have;
  size_t n = 0;
  for (uint64_t j = first; j < s->count && n < cap; j++, n++)
    out[n] = b->W == 0 ? s->box[j] : s->box[j % b->W];
  return n;
}

size_t orc_consume(orc_bus* b, uint32_t gid, orc_event* out, size_t cap) {
  orc_sub* s = sub_at(b, gid);
  if (!s) return 0;
  size_t n = 0;
  while (s->consumed < s->count && n < cap) {
    if (b->W && s->count - s->consumed > b->W) { s->consumed = s->count - b->W; continue; }
    out[n++] = b->W == 0 ? s->box[s->consumed] : s->box[s->consumed % b->W];
    s->consumed++;
  }
  return n;
}

/* -------------------------------------------------------------- names ----- */
/* EventCode.String — events/eventcode_string.go:5-15 (stringer table) */
static const char* const CODE_NAMES[ORC_N_CODES] = {
  "None", "ExitSuccess", "ExitFailed", "Stopping", "Stopped", "StatusHealthy",
  "StatusUnhealthy", "StatusChanged", "TimerExpired", "EnterMaintenance",
  "ExitMaintenance", "Error", "Quit", "Metric", "Startup", "Shutdown", "Signal" };
const char* orc_code_name(int code) {
  return (code < 0 || code >= ORC_N_CODES) ? NULL : CODE_NAMES[code];
}

/* FromString — events/events.go:52-86 */
int orc_code_from_string(const char* n) {
  static const struct { const char* s; int c; } T[] = {
    {"exitSuccess", 1}, {"exitFailed", 2}, {"stopping", 3}, {"stopped", 4},
    {"healthy", 5}, {"unhealthy", 6}, {"changed", 7}, {"timerExpired", 8},
    {"enterMaintenance", 9}, {"exitMaintenance", 10}, {"error", 11}, {"quit", 12},
    {"startup", 14}, {"shutdown", 15}, {"SIGHUP", 16}, {"SIGUSR2", 16} };
  for (size_t i = 0; i < sizeof(T) / sizeof(T[0]); i++)
    if (strcmp(n, T[i].s) == 0) return T[i].c;
  return -1;   /* (None, error) */
}
