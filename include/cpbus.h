/*
 * cpbus.h — C-ABI of libcpbus, the H100-native event bus that sits behind
 * ContainerPilot's `events` package (reference: TritonDataCenter/containerpilot, events/).
 *
 * This header is the drop-in boundary (SURVEY.md §8b).  It is what a cgo shim
 * for package `events` binds (see INTEGRATION.md for the Go side).  Everything
 * is plain C: pointers + sizes, `int` status returns (0 = OK, negative =
 * CPBUS_E*), no exceptions, no torch types.  The library never keeps a caller
 * pointer past the call (cgo pointer rule).  One publisher thread at a time
 * per bus (the shim keeps `bus.lock`, reference events/bus.go:126); drain and
 * stats may be called from another thread between flushes.
 *
 * Record format (frozen): one 32-byte, 32-byte-aligned record = exactly one
 * HBM/L2 sector.  Go's `Event{Code EventCode; Source string}`
 * (events/events.go:10-13) maps to {code, source_id} through the host-side
 * intern table (cpbus_intern); seq/ts/target/flags are bus bookkeeping.
 */
#ifndef CPBUS_H
#define CPBUS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- event codes: events/events.go:21-39 (iota order is the wire value) ---- */
enum {
  CPBUS_NONE = 0, CPBUS_EXIT_SUCCESS, CPBUS_EXIT_FAILED, CPBUS_STOPPING,
  CPBUS_STOPPED, CPBUS_STATUS_HEALTHY, CPBUS_STATUS_UNHEALTHY,
  CPBUS_STATUS_CHANGED, CPBUS_TIMER_EXPIRED, CPBUS_ENTER_MAINTENANCE,
  CPBUS_EXIT_MAINTENANCE, CPBUS_ERROR, CPBUS_QUIT, CPBUS_METRIC,
  CPBUS_STARTUP, CPBUS_SHUTDOWN, CPBUS_SIGNAL,
  CPBUS_N_CODES /* 17 */
};

/* subscription mask: bit i set <=> subscriber wants EventCode i.
 * CPBUS_MASK_ALL reproduces the reference exactly (the reference bus has no
 * filter: events/bus.go:134-138 delivers every event to every subscriber). */
#define CPBUS_MASK_ALL 0x0001FFFFu

/* one exact case of a consumer's event switch: events.Event{Code, Source} (jobs/jobs.go:197-231) */
typedef struct cpbus_pair { uint32_t code, source_id; } cpbus_pair;
#define CPBUS_MAX_PAIRS 16

#define CPBUS_TARGET_ALL 0xFFFFFFFFu /* broadcast (EventBus.Publish)            */
#define CPBUS_F_TICK     0x1u        /* record produced by a timer (events/timer.go) */
#define CPBUS_F_UNICAST  0x2u        /* direct mailbox send (`sub.Rx <- ev`, jobs/jobs.go:262) */

typedef struct cpbus_event {
  uint64_t seq;       /* publish: global publish ordinal (0-based, bus lifetime).
                         tick: firing ordinal of that timer (0-based).          */
  uint64_t ts_ns;     /* virtual clock when published / due time of the tick    */
  uint32_t code;      /* EventCode                                              */
  uint32_t source_id; /* interned Event.Source                                  */
  uint32_t target;    /* CPBUS_TARGET_ALL, or the global subscriber id          */
  uint32_t flags;     /* CPBUS_F_*                                              */
} cpbus_event;        /* sizeof == 32 */

/* ---- status codes ---- */
enum {
  CPBUS_OK = 0,
  CPBUS_EINVAL = -1,   /* bad argument                                           */
  CPBUS_ENOMEM = -2,   /* host or device allocation failed                       */
  CPBUS_ECUDA = -3,    /* CUDA runtime error (cpbus_last_cuda_error has detail)  */
  CPBUS_EAGAIN = -4,   /* lossless mode: a targeted mailbox is full; drain+retry */
  CPBUS_ENOSPC = -5,   /* subscriber / timer / intern table capacity exhausted   */
  CPBUS_ENOENT = -6,   /* unknown subscriber / timer id                          */
  CPBUS_ECLOSED = -7,  /* subscriber already unsubscribed (Go: panic, bus.go:121)*/
  CPBUS_ENODEV = -8,   /* no CUDA device: there is NO CPU fallback               */
  CPBUS_EORDER = -9,   /* device batch not sorted by ts / clock moved backwards  */
  CPBUS_ETIMEDOUT = -10 /* stream mode: a batch never arrived (publisher stalled or the consumer fell a whole ring
                           behind); sticky: the bus reports it from every later stream call */
};

/* cpbus_config.flags */
#define CPBUS_CFG_LOSSLESS 0x1u /* reference semantics: never drop; a full mailbox
                                   stalls the publisher (events/subscriber.go:30-32).
                                   The library keeps a lower bound of the free room of
                                   the fullest mailbox: while a batch provably fits it
                                   goes straight to the fan-out; the admission kernel
                                   (and its host sync) runs only when the bound is used
                                   up, and refreshes it exactly.
                                   Without it the bus runs in overwrite-oldest
                                   throughput mode (no consumer needed).          */
#define CPBUS_CFG_DIGEST   0x2u /* maintain the per-subscriber order-sensitive
                                   64-bit digest in-kernel                       */
#define CPBUS_CFG_SPARSE_TICKS 0x4u /* a flush with no staged record costs what is due: the
                                   host keeps an index of the armed timer slots by due
                                   time; a flush with no tick due launches nothing, and
                                   one with a few due ticks launches one small kernel over
                                   the mailboxes that own them (the full fan-out past
                                   max(32, subscribers/1024) due slots, and in lossless mode when the
                                   room bound cannot prove that the ticks fit).  Results
                                   are those of a bus without the flag making the same
                                   calls, except cpbus_stats.batches, kernel_launches,
                                   admit_passes and admit_skipped.  Not supported on a
                                   group (cpbus_group_create) or with streams
                                   (cpbus_stream_create/_open/_attach): CPBUS_EINVAL. */
#define CPBUS_CFG_SPARSE_RECORDS 0x8u /* a flush with staged records that reach few
                                   mailboxes costs what it delivers: the host keeps an index
                                   of the subscribers by code (a count per code, and the list
                                   while it is short) and by exact {code, source} case, and
                                   such a flush launches one small kernel over exactly the
                                   mailboxes that take a record or own a due tick (the full
                                   fan-out past max(32, subscribers/1024) such mailboxes or
                                   past max(1024, subscribers/256) records planned, and in
                                   lossless mode when the room bound cannot prove that one
                                   mailbox's records and ticks fit).  Requires
                                   CPBUS_CFG_SPARSE_TICKS (CPBUS_EINVAL otherwise).  Results
                                   are those of a bus without the flag making the same calls,
                                   except cpbus_stats.batches, kernel_launches, admit_passes
                                   and admit_skipped; a flush that launched nothing (no
                                   mailbox takes anything) leaves the step result as it was.
                                   Device batches (cpbus_publish_device*) always take the
                                   full fan-out.  Not supported on a group: CPBUS_EINVAL. */
#define CPBUS_CFG_DROP_MISSED_TICKS 0x10u /* periodic timers drop missed ticks like Go's time.Ticker
                                   (NewEventTimer reads a ticker whose channel holds one tick,
                                   so a late wake-up delivers one tick, not a burst).  When
                                   cpbus_advance moves the clock from c to now, an armed periodic
                                   timer with k >= 2 firings due in (c, now] delivers only the
                                   last, due at d_last (the largest point of its grid <= now that
                                   is below UINT64_MAX), and next fires at d_last + period: the
                                   phase is kept.  The tick is the usual {seq, ts = d_last,
                                   TimerExpired, source, owner, F_TICK}, and seq stays the
                                   firing ordinal on the grid: the skipped firings are counted,
                                   so a gap of g between consecutive seqs of one timer means g
                                   ticks were dropped.  Firings due at or before c and one-shots
                                   are unaffected.  The bus compares each step with the shortest
                                   period armed since no timer was left armed (a lower bound: a
                                   cancel or an unsubscribe does not raise it).  A step no longer
                                   than that bound behaves exactly as without the flag.  A longer
                                   step first flushes what is staged and due at c, then runs one
                                   catch-up kernel; where it gives no timer two firings it
                                   delivers the same records as an unflagged bus, but the flush
                                   adds launches and, in lossless mode, may return CPBUS_EAGAIN
                                   where an unflagged bus would not (with the clock unchanged).
                                   The caller's step is the rule's resolution: a pump advancing
                                   every 1 ms with periods of seconds changes nothing in steady
                                   state.  The rule covers cpbus_advance, and cpbus_group_advance
                                   on a group created with the flag (which gives the flagged
                                   single bus's results).
                                   Valid with every other flag; a flagged sparse bus gives the
                                   results of a flagged dense twin.  Streams and device batches
                                   move the clock by watermarks no cpbus_advance sees, so
                                   cpbus_stream_create/_open/_attach and cpbus_publish_device
                                   /_staged return CPBUS_EINVAL on a flagged bus (the group's own
                                   internal streams excepted); lifting that is future work. */
#define CPBUS_CFG_SPARSE_DRAINS 0x20u /* cpbus_drain_ready / cpbus_take_ready (and their
                                   tickets) cost what the range can hold: the host keeps the
                                   mailboxes each sparse launch appended to and each drain
                                   emptied, and a ready call whose range holds no candidate
                                   launches nothing, copies nothing and does not synchronise
                                   (n_ready = total = 0, next_sub = start_sub; a _begin still
                                   takes a ticket slot), one with at most max(256,
                                   subscribers/4096) candidates scans only those, and otherwise
                                   the dense scan runs.  A full fan-out, a lossless partial
                                   flush or a device batch makes the candidates unknown (dense
                                   scans) until a drain that takes every ready mailbox of the
                                   whole subscribed range.  Results are those of a bus without
                                   the flag making the same calls, except
                                   cpbus_stats.kernel_launches.  Requires
                                   CPBUS_CFG_SPARSE_TICKS (CPBUS_EINVAL otherwise); not
                                   supported on a group: CPBUS_EINVAL. */

/* cpbus_config.store_path: how records reach the rings (all are bit-identical) */
enum {
  CPBUS_STORE_AUTO = 0, /* library default = best measured (see DESIGN.md)       */
  CPBUS_STORE_V4   = 1, /* lane pair per record, 16 B / lane, half-indexed loop  */
  CPBUS_STORE_V8   = 2, /* lane pair per record, record-indexed loop (default)   */
  CPBUS_STORE_BULK = 3  /* cp.async.bulk smem->global (TMA) for dense segments   */
};

typedef struct cpbus_config {
  uint32_t n_max_subs;     /* capacity of this shard's subscriber table           */
  uint32_t ring_cap;       /* records per mailbox; power of two, >= 64 (1024 = default; reference channel cap is 1000, jobs/jobs.go:23) */
  uint32_t batch_cap;      /* max events per flush; <= min(ring_cap/2, 1024), multiple of 32 */
  uint32_t timers_per_sub; /* timer slots per subscriber: 0,1,2,4,8               */
  uint32_t flags;          /* CPBUS_CFG_*                                         */
  int32_t  device;         /* CUDA device ordinal; -1 = current device            */
  uint32_t sub_id_base;    /* global id of this shard's subscriber 0 (multi-GPU:
                              contiguous shards, SURVEY.md §8e); sub_id_base +
                              n_max_subs <= 0xFFFFFFFF (CPBUS_EINVAL otherwise), so
                              no gid equals CPBUS_TARGET_ALL                      */
  uint32_t store_path;     /* CPBUS_STORE_*                                       */
  void*    stream;         /* cudaStream_t to run on; NULL = library-owned stream */
  uint32_t grid_ctas;      /* 0 = auto (multiple of the SM count)                 */
  uint32_t reserved[5];
} cpbus_config;

typedef struct cpbus_digest_t {
  uint64_t count;  /* records ever delivered to this mailbox (broadcast + unicast + ticks) */
  uint64_t digest; /* rolling h = h*P + H(record) over the delivered sequence (mod 2^64)  */
} cpbus_digest_t;

typedef struct cpbus_stats_t {
  uint64_t publishes;      /* events that entered Publish/Send                    */
  uint64_t deliveries;     /* 32-B records landed in mailboxes (incl. ticks)      */
  uint64_t ticks;          /* timer records among the deliveries                  */
  uint64_t batches;        /* fan-out launches                                    */
  uint64_t kernel_launches;/* all kernels this bus launched                       */
  uint64_t overwritten;    /* undrained records currently lost to overwrite-oldest:
                              sum over mailboxes of max(0, tail - ring_cap - head) */
  uint64_t published_by_code[CPBUS_N_CODES]; /* reconciliation of the Prometheus
                              `containerpilot_events` counter (events/bus.go:130-132) */
  uint32_t n_subs;         /* currently subscribed                                */
  uint32_t n_timers;       /* currently armed                                     */
  uint64_t now_ns;         /* virtual clock                                       */
  /* ABI v2 */
  uint64_t intern_entries; /* permanent Source strings held by the intern table  */
  uint64_t intern_bytes;   /* ... and their total length                          */
  uint64_t ephemeral_live; /* payload strings currently held by the bounded ephemeral region (cpbus_intern_ephemeral) */
  uint64_t ephemeral_recycled; /* ephemeral ids that have been recycled so far   */
  uint64_t admit_passes;   /* lossless mode: flushes that needed the admission kernel (+ one host sync) ... */
  uint64_t admit_skipped;  /* ... and flushes that provably fitted and went straight to the fan-out        */
  uint64_t admit_partial;  /* flushes that delivered only the prefix every mailbox could take (then EAGAIN)  */
  uint64_t device_splits;  /* slices launched for device batches one launch could not take (see cpbus_publish_device) */
} cpbus_stats_t;

typedef struct cpbus cpbus_t;

/* ---- lifecycle: NewEventBus (events/bus.go:72-88); reload = destroy+create (core/app.go:142) ---- */
int cpbus_create(const cpbus_config* cfg, cpbus_t** out);
int cpbus_destroy(cpbus_t* bus);

/* ---- Event.Source interning (events/events.go:12; SURVEY F7) ---- */
int cpbus_intern(cpbus_t* bus, const char* s, size_t len, uint32_t* source_id);
/* copies at most cap bytes; *len receives the full length.  CPBUS_ENOENT: unknown id, or an ephemeral id whose
 * slot has been recycled since. */
int cpbus_source(cpbus_t* bus, uint32_t source_id, char* out, size_t cap, size_t* len);
/* Payload strings that are NOT names: every POST /v3/metric publishes Event{Metric, "key|value"}
 * (control/endpoints.go:125-126) and each distinct value would otherwise live in the intern table for the bus's
 * lifetime (the reference keeps Metric out of its per-source counter for the same cardinality reason, events/bus.go:130).
 * Ephemeral ids come from a bounded region of CPBUS_EPHEMERAL_SLOTS strings that is recycled oldest-first: an id
 * (bit 31 set) stays resolvable until CPBUS_EPHEMERAL_SLOTS newer distinct payloads have been interned — far beyond the
 * lifetime of a record in a 1024-slot mailbox.  Equal strings that are both still live get the same id. */
#define CPBUS_EPHEMERAL_SLOTS 65536u
#define CPBUS_EPHEMERAL_BIT   0x80000000u
int cpbus_intern_ephemeral(cpbus_t* bus, const char* s, size_t len, uint32_t* source_id);

/* ---- membership: Subscribe/Unsubscribe (events/bus.go:105-122).  Ordered with
 *      publishes: any staged events are flushed first. ---- */
int cpbus_subscribe(cpbus_t* bus, uint32_t code_mask, uint32_t* sub_id);
int cpbus_subscribe_many(cpbus_t* bus, const uint32_t* code_masks, uint32_t n, uint32_t* first_sub_id);
/* Second-level filter (SURVEY.md §8f N3).  A consumer's `switch event { case events.Event{Code, Source}: ... }`
 * (jobs/jobs.go:188-231) compares whole Event values, so each case is an exact {code, source} pair.  The subscriber
 * receives a broadcast event when its code is in code_mask (any source) OR {code, source_id} equals one of the
 * n_pairs <= CPBUS_MAX_PAIRS pairs.  Unicast records and timer ticks bypass both levels, like a direct channel send.
 * CPBUS_EINVAL: n_pairs > CPBUS_MAX_PAIRS, a pair's code >= CPBUS_N_CODES, or pairs == NULL with n_pairs > 0. */
int cpbus_subscribe_pairs(cpbus_t* bus, uint32_t code_mask, const cpbus_pair* pairs, uint32_t n_pairs, uint32_t* sub_id);
/* bulk form for a whole fleet: subscriber i gets code_masks[i] and the first n_pairs[i] (<= CPBUS_MAX_PAIRS) entries of
 * row i of `pairs` (n rows of CPBUS_MAX_PAIRS entries; the rest of a row is ignored).  One upload instead of n calls. */
int cpbus_subscribe_pairs_many(cpbus_t* bus, const uint32_t* code_masks, const cpbus_pair* pairs, const uint32_t* n_pairs,
                               uint32_t n, uint32_t* first_sub_id);
int cpbus_unsubscribe(cpbus_t* bus, uint32_t sub_id);
/* Change a subscriber's code mask in place (ordered with publishes).  Mailbox, timers and exact cases are kept.  The
 * shims use it when a channel that only carried timer ticks (implicit mask-0 subscriber, see NewEventTimer in
 * INTEGRATION.md) is subscribed to the bus afterwards. */
int cpbus_set_mask(cpbus_t* bus, uint32_t sub_id, uint32_t code_mask);

/* ---- timers: NewEventTimer / NewEventTimeout (events/timer.go:40-71 / 12-37).
 *      The first firing is due at now + period_ns; a periodic timer then fires
 *      every period_ns, a one-shot exactly once.  cancel = ctx.Done().  A timer id carries a generation: cancelling an
 *      id whose slot has fired (one-shot) or been re-armed since returns CPBUS_ENOENT and touches nothing.
 *      Due times saturate: a first or re-armed due time past UINT64_MAX - 1 means "never" (the timer stays armed, counts
 *      in n_timers and can be cancelled, but does not fire). ---- */
int cpbus_timer_add(cpbus_t* bus, uint32_t sub_id, uint64_t period_ns, uint32_t source_id, int oneshot, uint32_t* timer_id);
/* one periodic timer per subscriber [first_sub, first_sub+n); source_ids[i] (or source_id0+i if NULL).  It arms slot 0 of
 * each subscriber, returns no timer ids and does not advance the slots' generations; cpbus_timer_add_list arms timers with
 * their own owners, periods and kinds and returns their ids. */
int cpbus_timer_add_many(cpbus_t* bus, uint32_t first_sub, uint32_t n, uint64_t period_ns, const uint32_t* source_ids, uint32_t source_id0, int oneshot);
int cpbus_timer_cancel(cpbus_t* bus, uint32_t timer_id);

/* ---- bulk membership changes: cpbus_unsubscribe / cpbus_set_mask / cpbus_timer_cancel for many ids in one call.
 * Each element is applied exactly as the single call would apply it, in array order, and the call goes on past an element
 * the single call would refuse without touching anything (CPBUS_ENOENT, CPBUS_ECLOSED).  status[i] (status may be NULL) =
 * what the single call would have returned for element i at its turn; *applied (may be NULL) = how many returned CPBUS_OK.
 * Loop equivalence: a bus that calls cpbus_X_many(ids, n) and a twin that calls cpbus_X(ids[i]) for i = 0 .. n-1 give the
 * same results afterwards (every later return code, drain, drain_ready, peek_window, digest, fold, lagging, blockers,
 * debug event and publish count, and every cpbus_stats field but batches, kernel_launches, admit_* and device_splits).  So:
 *  - an id listed twice acts twice: unsubscribe gives CPBUS_OK then CPBUS_ECLOSED; set_mask keeps the last mask; a timer
 *    id is cancelled once, and its second entry gets CPBUS_ENOENT;
 *  - ordered with publishes: one flush of the staged events runs first, where the first element that gets past its
 *    single call's up-front checks would run it (none gets past them: no flush).  In lossless mode its CPBUS_EAGAIN is
 *    returned with nothing applied, and status / applied are not written;
 *  - CPBUS_EINVAL (checked first): bus NULL, or an array NULL with n > 0.  n == 0: CPBUS_OK, the bus is not read.
 * The device work is one H2D copy of one entry per mailbox touched, one kernel launch and one stream synchronisation (none
 * when nothing is applied), instead of a synchronised round trip per id.  code_masks[i] goes with sub_ids[i]. ---- */
int cpbus_unsubscribe_many(cpbus_t* bus, const uint32_t* sub_ids, uint32_t n, int* status, uint32_t* applied);
int cpbus_set_mask_many(cpbus_t* bus, const uint32_t* sub_ids, const uint32_t* code_masks, uint32_t n, int* status,
                        uint32_t* applied);
int cpbus_timer_cancel_many(cpbus_t* bus, const uint32_t* timer_ids, uint32_t n, int* status, uint32_t* applied);

/* ---- bulk timer arming: cpbus_timer_add for many timers in one call, each with its own owner, period and kind.
 * Loop equivalence, as for the bulk membership calls above: a bus that calls cpbus_timer_add_list(specs, n) and a twin that
 * calls cpbus_timer_add(s.sub_id, s.period_ns, s.source_id, s.oneshot, &id) for each specs[i] in order give the same
 * statuses and ids and the same results afterwards (every later return code, drain, drain_ready, peek_window, digest,
 * fold, lagging, blockers, debug event and publish count, and every cpbus_stats field but batches, kernel_launches,
 * admit_* and device_splits).  So:
 *  - status[i] (status may be NULL) = what cpbus_timer_add would have returned for element i at its turn: CPBUS_EINVAL
 *    (period 0), CPBUS_ENOSPC (timers_per_sub == 0, or no free slot left), CPBUS_ENOENT (an id never handed out),
 *    CPBUS_ECLOSED (an unsubscribed owner) or CPBUS_OK.  The call goes on past refused elements; *applied (may be NULL)
 *    = how many got CPBUS_OK;
 *  - timer_ids[i] (timer_ids may be NULL) is written for each CPBUS_OK element and left as it was otherwise.  An element
 *    takes its owner's lowest free slot after the slots taken by earlier elements, so elements for one owner take
 *    successive slots until timers_per_sub runs out.  Each arming advances the slot's 6-bit generation, as cpbus_timer_add
 *    does: an id handed out before the slot was re-armed is stale for cpbus_timer_cancel / _cancel_many;
 *  - ordered with publishes: one flush of the staged events runs where the first element that gets past the up-front
 *    checks (period, timers_per_sub, id range) would run it (none gets past them: no flush), and then one-shots that have
 *    fired free their slots.  In lossless mode the flush's CPBUS_EAGAIN is returned with nothing applied, and status,
 *    timer_ids and applied are not written;
 *  - CPBUS_EINVAL (checked first): bus NULL, or specs NULL with n > 0.  n == 0: CPBUS_OK, the bus is not read.
 * The device work is one H2D copy of one entry per armed slot, one kernel launch and one stream synchronisation (none when
 * nothing is applied), instead of two synchronised copies per timer.  pad is ignored. ---- */
typedef struct cpbus_timer_spec {
  uint64_t period_ns;  /* > 0 */
  uint32_t sub_id;     /* owner */
  uint32_t source_id;  /* Event.Source of its ticks */
  uint32_t oneshot;    /* 0: periodic (NewEventTimer); else one-shot (NewEventTimeout) */
  uint32_t pad;
} cpbus_timer_spec;    /* 24 bytes */
int cpbus_timer_add_list(cpbus_t* bus, const cpbus_timer_spec* specs, uint32_t n, uint32_t* timer_ids, int* status,
                         uint32_t* applied);

/* ---- subscriber id reuse: ids behave like file descriptors.  An unsubscribed mailbox stays readable until it is released;
 * a released id goes back to a free set, and cpbus_subscribe_list hands free ids out again, lowest first.  The caller must not
 * use an id after releasing it: the next subscriber may already hold it.  cpbus_subscribe, _many, _pairs and _pairs_many
 * hand out fresh ids only and never reuse one; a program that never releases sees no difference anywhere.
 * cpbus_release_many: each element in array order; status[i] (status may be NULL): CPBUS_ENOENT (never handed out, or
 * already released, by an earlier element of the same call too), CPBUS_EINVAL (still subscribed: unsubscribe it first) or
 * CPBUS_OK; the call goes on past refused elements and *applied (may be NULL) = how many got CPBUS_OK.  Ordered with
 * publishes: one flush runs where the first element that passes these checks would run it (none passes: no flush); in
 * lossless mode its CPBUS_EAGAIN is returned with nothing applied and status / applied not written.  CPBUS_EINVAL (checked
 * first): bus NULL, or sub_ids NULL with n > 0.  n == 0: CPBUS_OK, the bus is not read.
 * A released id is in the state of an id never handed out: cpbus_send, _unsubscribe[_many], _set_mask[_many],
 * _timer_add[_list], _timer_add_many (a range that holds one), _drain, _peek_window and _ack_many refuse it with
 * CPBUS_ENOENT.  Range calls (drain_many, drain_ready, take_ready, lagging, digest, digest_fold) still take ranges up to
 * the highest id ever handed out and see a released mailbox as empty: count and digest 0, nothing to return, never lagging.  Its records are discarded (taken and not yet
 * acked ones too), and so are its take cursor and its exact cases.  Its timer slots keep their generations, and the next
 * arming advances them, so a timer id of the old occupant stays stale (CPBUS_ENOENT) and never cancels a new occupant's.
 * cpbus_subscribe_list: subscriber i gets code_masks[i] (code_masks NULL: CPBUS_MASK_ALL for all) and the first n_pairs[i]
 * cases of row i of `pairs`, laid out as for cpbus_subscribe_pairs_many (n_pairs NULL: no cases).  Ids are the lowest free
 * ones: released ids ascending, then fresh ones; sub_ids[i] receives subscriber i's id.  Each new subscriber starts as a
 * fresh cpbus_subscribe_pairs leaves it: empty mailbox with ring_cap slots of room, count and digest 0, no timers, its mask
 * and cases.  All or nothing: CPBUS_EINVAL (bus or sub_ids NULL, n == 0, n_pairs non-NULL with pairs NULL, n_pairs[i] >
 * CPBUS_MAX_PAIRS or a case's code >= CPBUS_N_CODES), CPBUS_ENOSPC (fewer than n ids free), and one flush first, ordered
 * with publishes, whose lossless CPBUS_EAGAIN applies nothing.
 * The device work of either call is one H2D copy of one entry per mailbox (plus the rows of new cases), one kernel launch and
 * one stream synchronisation; none when nothing is applied. ---- */
int cpbus_release_many(cpbus_t* bus, const uint32_t* sub_ids, uint32_t n, int* status, uint32_t* applied);
int cpbus_subscribe_list(cpbus_t* bus, const uint32_t* code_masks, const cpbus_pair* pairs, const uint32_t* n_pairs, uint32_t n,
                         uint32_t* sub_ids);

/* ---- the hot path: EventBus.Publish (events/bus.go:125-140) ---- */
/* Stages n events; only code/source_id are read from ev (seq, ts, target, flags
 * are stamped by the bus).  Flushes automatically whenever batch_cap is reached.
 * Lossless mode: if an automatic flush hits a full mailbox the call stops and returns
 * CPBUS_EAGAIN; events before the one that triggered the flush are staged, that one and
 * the rest are not (cpbus_stats.publishes tells how many were taken).  Publishing one
 * event per call, as the Go bus does, makes the retry point unambiguous.  cpbus_flush in
 * lossless mode blocks PER EVENT like the Go bus: when some mailbox lacks the room, the longest
 * prefix of the staged events that every targeted mailbox can take is delivered (with the timer
 * ticks due by its last event), the rest stays staged and the call returns CPBUS_EAGAIN; after the
 * consumers have drained, the next flush continues with the first undelivered event.
 * (Batches handed over in device memory, cpbus_publish_device, stay all-or-nothing: the caller owns them.) */
int cpbus_publish(cpbus_t* bus, const cpbus_event* ev, size_t n);
/* Direct mailbox write, bypassing the filter (`job.Rx <- ev`, jobs/jobs.go:262;
 * Subscriber.Receive, events/subscriber.go:30).  Ordered with publishes. */
int cpbus_send(cpbus_t* bus, uint32_t sub_id, const cpbus_event* ev);
/* Move the virtual clock; timers whose due time <= now_ns fire at the next flush,
 * ordered before any event published after this call.  On a CPBUS_CFG_DROP_MISSED_TICKS bus a step longer than the
 * shortest period drops the missed ticks (see the flag); in lossless mode it may return CPBUS_EAGAIN from the flush it makes
 * first, with the clock unchanged. */
int cpbus_advance(cpbus_t* bus, uint64_t now_ns);
/* Launch the fan-out for everything staged (async on the bus stream). */
int cpbus_flush(cpbus_t* bus);
int cpbus_sync(cpbus_t* bus);
/* Fan out a batch that is already resident in HBM (multi-GPU: the NCCL-broadcast
 * stream, SURVEY.md §8e; bench: device-resident trace).  Records are complete
 * (seq/ts/target/flags set by the producer), sorted by ts_ns, 32-byte aligned.
 * watermark_ns >= last ts; becomes the bus clock.  One launch takes up to batch_cap
 * records and a watermark step of up to 32/timers_per_sub periods of the fastest armed
 * timer; a batch beyond either is cut into several launches (the cut reads the records'
 * timestamps back, 8 bytes each: a slow path, counted in cpbus_stats.device_splits).
 * Lossless mode keeps the strict form: CPBUS_EINVAL / CPBUS_EORDER for such a batch.
 * A broadcast record whose code is >= CPBUS_N_CODES reaches no mailbox (no mask bit or pair selects it); it counts in
 * stats.publishes and the debug ring but not in published_by_code or cpbus_publish_counts.  The bus's seq advances by n. */
int cpbus_publish_device(cpbus_t* bus, const void* d_events, size_t n, uint64_t watermark_ns);
/* (Batches published this way are accounted for by the kernel itself: cpbus_stats.published_by_code,
 * cpbus_publish_counts and cpbus_debug_events see their broadcast events exactly as if they had gone through cpbus_publish.) */
/* Same, but d_events may point into ANOTHER GPU's HBM (the publisher's event stream, peer-mapped over
 * NVLink, e.g. through CUDA IPC): one CTA of the fan-out kernel pulls the batch across the link, stages it
 * locally and hands it to the other CTAs together with the batch descriptor — the broadcast of SURVEY.md §8e
 * fused into the fan-out launch, no collective call.  If d_next/n_next name a LATER batch (the next one, or better
 * the one after it), the same launch also pulls that batch (the NVLink transfer hides under this launch's stores) and
 * a later call given that pointer as its d_events starts from local memory; a batch pulled two launches earlier also
 * lets that launch's prologue overlap its predecessor (programmatic dependent launch).  The caller guarantees the peer batches are complete and stable while the
 * launch runs (throughput mode only). */
int cpbus_publish_device_staged(cpbus_t* bus, const void* d_events, size_t n, uint64_t watermark_ns,
                                const void* d_next, size_t n_next);

/* ---- the publisher's event stream across the GPUs of one box (one process per GPU) ----------------------------------
 * The subscriber set partitions into contiguous shards, one bus per GPU (cpbus_config.sub_id_base); every shard must see
 * the identical, totally ordered batch sequence (SURVEY.md §8e).  A stream is a ring of n_slots batch slots in the
 * PUBLISHER GPU's HBM, exported with CUDA IPC.  cpbus_stream_put copies a batch into the next slot and then releases it
 * by writing the slot header {seq, watermark, n} (stream-ordered after the payload).  cpbus_stream_fanout, called by
 * every rank including the publisher's, launches the ordinary fan-out kernel for the next batch of the stream: its lead
 * CTA acquires the header across NVLink (ld.acquire.sys, bounded wait), pulls the 32-byte records over the peer mapping,
 * stages them locally for the other CTAs and acknowledges the slot (st.release.sys into the publisher's memory) — the
 * broadcast is fused into the fan-out launch; there is no collective, no copy-engine op and no cross-stream wait on the
 * consumers' data path.  When the publisher runs >= 2 batches ahead, the lead CTA of batch q also pulls batch q+2 while
 * its own stores are in flight, so later launches start from local memory and keep their prologue overlapped with the
 * previous launch (programmatic dependent launch).
 *   publisher rank : cpbus_stream_create(bus, n_slots, n_consumers, &st, handle); send `handle` to the other ranks
 *   other ranks    : cpbus_stream_open(bus, handle, consumer_index (1..n_consumers-1), &st)
 *   every step     : [publisher] cpbus_stream_put(st, events, n, now_ns, flags)   (may run ahead by < n_slots batches)
 *                    [all ranks] cpbus_stream_fanout(st, n, now_ns)
 *   followers      : [ranks that are never told n, now_ns] cpbus_stream_fanout_next(st) — the kernel reads them from the slot
 *                    header; may be called ahead of the publisher (throughput mode; lossless: cpbus_stream_round_next)
 * Lossless mode (CPBUS_CFG_LOSSLESS): a stalled publish must stop at the same event on every shard — the shortest of the
 * prefixes the shards can take — so the fan-out is split in two and the driver takes the minimum in between:
 *   every step     : [publisher] cpbus_stream_put(st, events, n, now_ns, flags)
 *                    [all shards] cpbus_stream_admit(st, n, now_ns, &p_g)      m = min over the shards of p_g
 *                    [all shards] cpbus_stream_fanout_prefix(st, n, now_ns, m)
 *                    CPBUS_EAGAIN (from an admit, or from fanout_prefix: records remain): let the consumers drain, then admit
 *                    and fan out again with the same (n, now_ns); the batch resumes at its first undelivered record.
 * Where no one thread can take that minimum (one process per GPU), the shards agree on it through the publisher's memory:
 *   every step     : [publisher] cpbus_stream_put(st, events, n, now_ns, flags)
 *                    [all shards] cpbus_stream_admit(st, n, now_ns, &p)        CPBUS_EAGAIN: p = 0, stalled = 1
 *                    [all shards] cpbus_stream_offer(st, p, stalled)
 *                    [all shards] cpbus_stream_agree(st, &m)                  CPBUS_EAGAIN: some shard stalled, m = 0
 *                    [all shards] cpbus_stream_fanout_prefix(st, n, now_ns, m)   (skipped after CPBUS_EAGAIN from _agree)
 * An offer is one 64-bit word {round, stalled, prefix} stored (st.release.sys) into a spare word of the shard's ack sector;
 * the agree kernel acquires every shard's word of the current round (ld.acquire.sys, bounded by the stream timeout) and
 * the host waits for that one kernel.  Each stream counts its admission rounds (one per _agree, on every shard alike), so
 * a retry of the same batch never reads the previous round's offer.  Offers are split from the wait so that one thread
 * driving several attached shards can post every offer before it waits on any.
 * While the mailboxes provably have room, admission costs no kernel and no host sync (as for cpbus_flush).  A batch's slot
 * is acknowledged only when its last record has been fanned out, so the publisher cannot run more than n_slots batches
 * ahead of the slowest shard.  Plain cpbus_stream_fanout returns CPBUS_EINVAL on a lossless bus.
 * cpbus_stream_fanout must be told n and now_ns of every batch by the caller: SPMD drivers know them; others follow with
 * cpbus_stream_fanout_next, or ask cpbus_stream_poll, which reads them from the slot header (the kernel cross-checks n).  CPBUS_EAGAIN from _put: the slot's previous batch is still not acknowledged by every
 * consumer after the stream timeout (or at once with CPBUS_PUT_NOWAIT) — call again after the consumers have advanced.  CPBUS_ETIMEDOUT from _fanout/_status: an earlier stream
 * launch gave up waiting for its batch (bounded in-kernel wait, cpbus_stream_set_timeout) and delivered nothing; CPBUS_EORDER
 * from every stream call: a follower's batch was behind the clock or beyond the timer window (see _fanout_next). */
typedef struct cpbus_stream cpbus_stream_t;
#define CPBUS_PUT_STAMP 0x0u /* records are stamped like cpbus_publish: seq = running publish ordinal, ts = now_ns,
                                target = ALL, flags = 0; only code/source_id are read from the caller's records */
#define CPBUS_PUT_RAW   0x1u /* records are complete (as for cpbus_publish_device): copied verbatim */
#define CPBUS_PUT_NOWAIT 0x2u /* if the slot's previous batch is not yet acknowledged by every consumer, return
                                CPBUS_EAGAIN at once.  Default: wait for the consumers (their launches are queued, the
                                GPUs are busy) up to the stream timeout, then CPBUS_EAGAIN.  A single thread that drives
                                the publisher AND consumers (LocalShardedBus) must use NOWAIT or never run more than
                                n_slots batches ahead of its own fan-outs. */
int cpbus_stream_create(cpbus_t* bus, uint32_t n_slots, uint32_t n_consumers, cpbus_stream_t** out, unsigned char handle[64]);
int cpbus_stream_open(cpbus_t* bus, const unsigned char handle[64], uint32_t consumer_index, cpbus_stream_t** out);
/* same-process consumer (one host process driving several GPUs, as the cgo shim does): no IPC handle, the owner's ring is
 * used through peer access (enabled here if the two buses live on different GPUs) */
int cpbus_stream_attach(cpbus_t* bus, cpbus_stream_t* owner, uint32_t consumer_index, cpbus_stream_t** out);
int cpbus_stream_put(cpbus_stream_t* st, const cpbus_event* events, size_t n, uint64_t now_ns, uint32_t flags);
int cpbus_stream_fanout(cpbus_stream_t* st, size_t n, uint64_t now_ns);
/* Lossless stream.  *prefix = how many of the current batch's undelivered records this shard's mailboxes can take (every
 * record of the batch up to then, plus the ticks due by the last of them); the whole remainder means the batch can complete,
 * the ticks due by now_ns included.  Where only those trailing ticks do not fit (records older than now_ns), the last record
 * is held back; an empty remainder whose ticks do not fit gives CPBUS_EAGAIN.  First flushes the bus's own staged events
 * (CPBUS_EAGAIN propagates) and checks the clock like cpbus_stream_fanout (CPBUS_EORDER).  The admission kernel runs, on a
 * local copy of the remainder, only when the fast path cannot prove the fit.  On a throughput-mode bus it is the whole
 * remainder, with no kernel. */
int cpbus_stream_admit(cpbus_stream_t* st, size_t n, uint64_t now_ns, size_t* prefix);
/* Fan out the next m undelivered records of the current batch (n, now_ns = the batch's full shape, as for
 * cpbus_stream_fanout).  Returns CPBUS_OK when the batch is complete: the slot is acknowledged and the stream moves to the
 * next batch.  Returns CPBUS_EAGAIN when records remain (m == 0: nothing is launched): the caller lets consumers drain, then
 * admits and fans out again.  A partial launch's watermark is its last record's ts_ns, and the bus clock moves only that far
 * until the batch completes, so the ticks due after it go with the remainder.  m beyond the remainder: CPBUS_EINVAL (m is
 * the minimum of the shards' admitted prefixes; more than this shard admitted would overfill a mailbox).  An empty batch
 * has a remainder of 0: m = 0 completes it. */
int cpbus_stream_fanout_prefix(cpbus_stream_t* st, size_t n, uint64_t now_ns, size_t m);
/* Lossless stream across processes: post this shard's admitted prefix, then learn the minimum over all shards.
 * _offer is asynchronous (a one-thread kernel on the bus stream).  CPBUS_EINVAL: a throughput-mode bus, a second offer in
 * one round, a prefix beyond the remainder of the batch last admitted, or stalled != 0 with a prefix.
 * _agree waits for every shard's offer of this round and sets *m to the minimum prefix.  CPBUS_EAGAIN (*m = 0): some
 * shard stalled — let the consumers drain, then run the round again with the same (n, now_ns).  CPBUS_ETIMEDOUT: a shard
 * did not offer within the stream timeout; sticky, as for a batch that never arrives.  CPBUS_EINVAL: no offer this round,
 * or a throughput-mode bus. */
int cpbus_stream_offer(cpbus_stream_t* st, size_t prefix, int stalled);   /* async, stream-ordered */
int cpbus_stream_agree(cpbus_stream_t* st, size_t* m);                   /* waits for every shard's offer */
/* For a consumer whose driver does not know the batches' shapes: *ready = 1 and {n, now_ns} of the NEXT batch if the publisher
 * has released it, *ready = 0 otherwise (one 32-byte read of the slot header, synchronous).  Then cpbus_stream_fanout(st, n, now_ns). */
int cpbus_stream_poll(cpbus_stream_t* st, int* ready, size_t* n, uint64_t* now_ns);
/* Stream followers: a consumer that never learns the batches' shapes (a rank that holds only subscriber shards).
 * _fanout_next enqueues the fan-out of the stream's next batch on the bus stream and returns at once: the kernel's lead CTA
 * takes n and the watermark from the slot header it acquires anyway.  Call it several times in a row to run ahead of the
 * publisher; each launch waits in the kernel for its batch, bounded by the stream timeout.  The result equals
 * cpbus_stream_fanout(st, n, now_ns) with the header's n and watermark: mailboxes, digests, ticks, step result, the slot's
 * acknowledgement, published_by_code, cpbus_publish_counts and cpbus_debug_events.
 * The host learns what the launches took lazily: every call that reads or changes the bus's host state (publish, send,
 * advance, flush, sync, membership, timers, stats, drains, digests, debug events, publish counts, the other stream calls but
 * _put) first waits for the last outstanding follower and folds in their records; the asynchronous tickets
 * (cpbus_step_result_*, cpbus_digest_fold_begin/_end) do not.  At most 8 followers are outstanding; the 9th resolves first.
 * A followed batch whose watermark lies behind this bus's clock, or steps further than 32/timers_per_sub periods of the
 * fastest periodic timer, delivers nothing, fires no timer and is not acknowledged; every follower queued behind it does
 * nothing, and cpbus_stream_status and every later stream call on this bus return CPBUS_EORDER (sticky, as
 * CPBUS_ETIMEDOUT is for a batch that never arrives).  CPBUS_EINVAL: NULL, or a lossless bus (lossless followers queue
 * rounds with cpbus_stream_round_next). */
int cpbus_stream_fanout_next(cpbus_stream_t* st);
/* Lossless followers: one admission round enqueued on the bus stream, never waited for on the host.  The round takes this
 * shard's current batch — the first one it has not completely delivered when the round runs, which the host may not know
 * yet — and does on the device what one host-driven round does with the header's n and watermark: it acquires the slot
 * header (bounded wait), computes this shard's admissible prefix of the undelivered remainder by cpbus_stream_admit's rules,
 * posts the offer word, waits for every shard's offer of the same round (bounded by the stream timeout) and fans out the
 * agreed m records.  A partial round's watermark is its last record's; the batch's slot is acknowledged, and the device
 * cursor moves to the next batch, when the round completes it.  If any shard stalls, the round delivers nothing and fires
 * no timer.  Every shard must enqueue the same sequence of rounds (as with _offer / _agree; round numbers continue the
 * count of _agree, one per call); one round completes at most one batch.
 *   [all shards, per round]  cpbus_stream_round_next(st)        (queue several; one thread driving several shards queues
 *                                                                the same round on every shard before the next one)
 *   [now and then]           cpbus_stream_progress(st, &T_done, &offset, &stalled)   resolve; let the consumers drain
 * The host learns the outcomes lazily, through the followers' queue (at most 8 outstanding; the 9th call resolves first)
 * and the same per-launch records: every call that reads or changes host state resolves first, and then the bus state
 * (stream position, clock, publish counts and ordinals, room bound, admit_passes / _skipped / _partial, debug-ring
 * entries) is what the host-driven rounds with the same outcomes leave.  After resolution a driver may switch freely
 * between rounds and explicit admit / offer / agree / fanout_prefix.  While rounds are outstanding the device copy of the
 * room bound is authoritative; cpbus_consume_all does not wait for them: it is ordered behind them on the bus stream and
 * resets that copy there.  A round whose batch lies behind this bus's clock or beyond its timer window posts no offer and
 * sets the sticky CPBUS_EORDER; the rounds queued behind it do nothing, and the other shards' rounds give up waiting for
 * its offer (sticky CPBUS_ETIMEDOUT).  CPBUS_EINVAL: NULL, a throughput-mode bus, or an explicit offer pending. */
int cpbus_stream_round_next(cpbus_stream_t* st);
/* Resolves outstanding followers and rounds, then: *batches = batches this consumer has completely fanned out, *offset =
 * records of the next one already delivered (0 for throughput followers), *stalled_rounds = rounds so far that moved
 * nothing (some shard stalled, or the agreed prefix was 0).  A driver told only the number of batches T queues at most
 * T - *batches rounds at a time: never past the last batch, and every rank decides alike.  Returns the sticky stream error
 * (the outputs are set either way). */
int cpbus_stream_progress(cpbus_stream_t* st, uint64_t* batches, size_t* offset, uint64_t* stalled_rounds);
int cpbus_stream_status(cpbus_stream_t* st);                       /* CPBUS_OK or the sticky error */
int cpbus_stream_set_timeout(cpbus_stream_t* st, uint32_t microseconds);   /* in-kernel wait bound; default 2 s */
int cpbus_stream_close(cpbus_stream_t* st);                        /* importers close before the owner */

/* Buffers shared between the GPUs (processes) of one box, for the publisher's event stream: _alloc makes a
 * device buffer on this bus's GPU and returns a 64-byte CUDA IPC handle; _open, called on ANOTHER bus (another
 * process/GPU), maps it over NVLink and returns a pointer valid for cpbus_publish_device_staged there.
 * _close frees (owner) or unmaps (importer); cpbus_destroy closes what is left. */
int cpbus_shared_alloc(cpbus_t* bus, size_t bytes, void** dptr, unsigned char handle[64]);
int cpbus_shared_open(cpbus_t* bus, const unsigned char handle[64], void** dptr);
int cpbus_shared_close(cpbus_t* bus, void* dptr);

/* ---- consumer side ---- */
/* Mailbox -> host, FIFO (`<-sub.Rx`).  *lost = records overwritten before they
 * could be drained (always 0 in lossless mode). */
int cpbus_drain(cpbus_t* bus, uint32_t sub_id, cpbus_event* out, size_t cap, size_t* n, uint64_t* lost);
/* Bulk drain of mailboxes [first_sub, first_sub+n): one kernel gathers every undrained record into a staging
 * buffer (one atomic per mailbox), two D2H copies bring them back.  out[offsets[i] .. offsets[i]+counts[i]) is mailbox
 * i's run, FIFO.  A mailbox whose run does not fit into `cap` is left untouched (counts[i] = 0) for the next call;
 * *total = records returned.  Its index traffic is sized by n; a pump on a large fleet calls cpbus_drain_ready. */
int cpbus_drain_many(cpbus_t* bus, uint32_t first_sub, uint32_t n, cpbus_event* out, size_t cap,
                     uint32_t* offsets, uint32_t* counts, size_t* total);
/* Sparse drain: only the mailboxes that hold records.  Mailboxes [first_sub, first_sub+n) are examined in cyclic id order
 * starting at start_sub; a mailbox is ready when it has undrained records (throughput mode: from max(head, tail - ring_cap),
 * as cpbus_drain).  Ready mailboxes are taken in that order while their whole run still fits into `cap` records and
 * `ready_cap` entries; the first one that does not fit ends the call (a run is never split).  Entry i of ready[0 .. *n_ready)
 * is the i-th mailbox taken; its records are out[offset .. offset+count), FIFO, runs packed back to back (*total records).
 * Taken mailboxes are left empty (head = tail); nothing else changes.  *next_sub = the first mailbox not taken (the one
 * that did not fit), or start_sub when everything was taken: a pump passing it back as start_sub visits every mailbox.
 * The same state and arguments give byte-identical out and ready.  Cost: one read of the range's control blocks on the
 * device plus the records taken; host<->device traffic is 24*n_ready + 32*total bytes plus a constant; at most two stream
 * synchronisations (one, and no copy, when nothing is ready).  Runs on the bus stream behind every earlier fan-out.
 * CPBUS_EINVAL: a NULL pointer, n == 0, cap < ring_cap, cap > 0xFFFFFFFF, ready_cap == 0, or start_sub outside the range.
 * CPBUS_ENOENT: the range is not within this shard's subscribers. */
typedef struct cpbus_ready {
  uint32_t sub_id;   /* global id (sub_id_base applied)                                                  */
  uint32_t count;    /* records of this mailbox in out[offset .. offset+count), FIFO                      */
  uint32_t offset;   /* offsets increase with the entry index; runs are packed back to back                */
  uint32_t pad;      /* 0 */
  uint64_t lost;     /* throughput mode: records overwritten since the stored cursor (as cpbus_drain); 0 in lossless mode */
} cpbus_ready;       /* sizeof == 24 */
int cpbus_drain_ready(cpbus_t* bus, uint32_t first_sub, uint32_t n, uint32_t start_sub,
                      cpbus_event* out, size_t cap, cpbus_ready* ready, size_t ready_cap,
                      size_t* n_ready, size_t* total, uint32_t* next_sub);

/* ---- acknowledged drains (lossless mode): copy a mailbox's records out but keep their room until the consumer's channel
 * has them.  cpbus_drain_ready frees a mailbox as it copies it, so a pump that buffers on the host for a stalled consumer
 * never lets its mailbox fill, and the publisher never stalls on it.  Take and ack split that in two:
 * Each mailbox has a take cursor T (0 at subscribe); its effective value is taken = max(T, head), and its taken - head
 * HELD records are the ones copied out and not yet released.
 *  - cpbus_take_ready has the arguments, checks, walk, cuts, output layout and *next_sub rule of cpbus_drain_ready, but a
 *    mailbox is ready when tail > taken, its run is [taken, tail), and taking it sets T = tail and leaves head alone.
 *    cpbus_ready.lost and .pad are 0.  Like cpbus_drain_ready it runs on the bus stream behind every earlier launch and
 *    does not flush staged events.
 *  - cpbus_ack_many releases, for each element in array order, the oldest counts[i] held records of sub_ids[i] (head +=
 *    counts[i]).  status[i] (status may be NULL): CPBUS_ENOENT (an id this bus never handed out, or outside this shard),
 *    CPBUS_EINVAL (counts[i] exceeds what the mailbox holds at this element's turn: an id listed twice is checked against
 *    what its earlier elements left) or CPBUS_OK (counts[i] == 0 included).  The call goes on past refused elements;
 *    *applied (may be NULL) = how many got CPBUS_OK.  Unsubscribed mailboxes can be acked.  It does not flush.
 *    After ack(id, k) the bus is in the state a bus that never takes reaches with cpbus_drain(id, cap = k) at that point;
 *    only the take cursors differ.  The device work is one H2D copy of one entry per mailbox, one kernel launch and one
 *    stream synchronisation; none when no element with counts[i] > 0 names a mailbox of this bus, or before its first take.
 * Taking is invisible to everything else: held records stay in the ring, so a bus that takes and one that never drains
 * give the same return codes and CPBUS_EAGAIN points of every publish, flush, advance, send, membership and stream
 * admission call, the same blockers, stream_blockers and lagging (held records are backlog), windows, digests, folds, debug
 * events and every cpbus_stats field but kernel_launches.  cpbus_drain, _drain_many, _drain_ready and _consume_all read
 * from head, held records included; afterwards head >= T, so nothing is held.
 * A pump that takes, hands the records to its consumers' channels and acks what each channel accepted holds at most
 * ring_cap records per consumer, and a consumer that stops reading fills its mailbox and stalls the publisher.
 * CPBUS_EINVAL: as cpbus_drain_ready, or a throughput-mode bus (held records could be overwritten before their ack); for
 * ack_many, checked first, a NULL bus or an array NULL with n > 0.  ack_many with n == 0: CPBUS_OK, the bus is not read. */
int cpbus_take_ready(cpbus_t* bus, uint32_t first_sub, uint32_t n, uint32_t start_sub,
                     cpbus_event* out, size_t cap, cpbus_ready* ready, size_t ready_cap,
                     size_t* n_ready, size_t* total, uint32_t* next_sub);
int cpbus_ack_many(cpbus_t* bus, const uint32_t* sub_ids, const uint32_t* counts, uint32_t n, int* status, uint32_t* applied);
/* ---- drain tickets: cpbus_drain_ready and cpbus_take_ready split in two, so that a pump hands one step's records to its
 * channels while the next step's drain runs on the GPU.
 *  - _begin enqueues the call on the bus stream and returns a ticket: it sees every launch queued before it and none
 *    queued after.  Like the synchronous calls it resolves outstanding followers first and does not flush staged events.
 *    It never waits for the GPU, except to allocate or grow a ticket's host buffer while that ticket is free, or the
 *    bus's scan scratch while other tickets are outstanding (a larger n or ready_cap than before).  Cost: a memset, two
 *    launches, and no host<->device copy issued by the host: the gather kernel writes the records, the ready list and the
 *    header into the bus's pinned, mapped memory (the library keeps no caller pointer past a call).
 *  - _end(ticket, ...) waits for that ticket only, writes out, ready, *n_ready, *total and *next_sub and frees the ticket.
 *    They are byte-identical to what the synchronous call with the begin's arguments would have returned at the begin's
 *    place in stream order, whatever was called in between (publishes, flushes, advances, membership changes, acks, other
 *    drains and begins).  A bus that replaces each cpbus_drain_ready / cpbus_take_ready with _begin + _end, and one that
 *    does not, give the same results afterwards: every later return code, drain, window, digest, fold, lagging, blockers
 *    and debug event, and every cpbus_stats field but kernel_launches.  Cost: one event wait and host memcpys of
 *    24*n_ready + 32*total bytes.
 *  - One _end serves both begins; the tickets share one space.  At most 8 are outstanding: a 9th _begin returns
 *    CPBUS_ENOSPC and enqueues nothing (a drain's records have left their mailboxes, so no result is ever overwritten).
 *    Tickets may be ended in any order.  cpbus_destroy releases outstanding tickets: their records are lost, as records
 *    drained into a buffer nobody reads.
 *  - Memory: each of the 8 ticket slots keeps a pinned host buffer of 128 + 32*cap + 24*min(ready_cap, n) bytes for the
 *    largest call it has served; buffers never shrink and are freed by cpbus_destroy (eight tickets with cap = 2^22 hold
 *    about 1 GiB).
 * CPBUS_EINVAL (_begin): as the synchronous call — a NULL bus or ticket, n == 0, ready_cap == 0, cap < ring_cap,
 * cap > 0xFFFFFFFF, start_sub outside the range; cpbus_take_ready_begin also on a throughput-mode bus.  CPBUS_ENOENT
 * (_begin): the range is not within this shard's subscribers.
 * CPBUS_EINVAL (_end): a NULL pointer, or cap / ready_cap below the begin's (the ticket stays outstanding).  CPBUS_ENOENT
 * (_end): a ticket that is not outstanding (never begun, or already ended). */
int cpbus_drain_ready_begin(cpbus_t* bus, uint32_t first_sub, uint32_t n, uint32_t start_sub,
                            size_t cap, size_t ready_cap, uint32_t* ticket);
int cpbus_take_ready_begin(cpbus_t* bus, uint32_t first_sub, uint32_t n, uint32_t start_sub,
                           size_t cap, size_t ready_cap, uint32_t* ticket);
int cpbus_drain_ready_end(cpbus_t* bus, uint32_t ticket, cpbus_event* out, size_t cap,
                          cpbus_ready* ready, size_t ready_cap, size_t* n_ready, size_t* total, uint32_t* next_sub);
/* Consumer backlog, read-only: which subscribed mailboxes fall behind and by how much, without consuming anything (head never
 * moves; a drain after this call returns exactly what it would have returned without it).  Mailboxes [first_sub,
 * first_sub+n) are visited in cyclic id order from start_sub, as by cpbus_drain_ready; only subscribed ones count (the implicit
 * mask-0 timer mailboxes included).  out[0 .. *n_out) = the first `cap` mailboxes with backlog >= min_backlog, in that
 * order (min_backlog == 0: every subscribed mailbox).  *next_sub = the first such mailbox not returned, or start_sub when all
 * were: passing it back visits every lagging mailbox exactly once.  *sum (may be NULL) covers the whole range whatever cap
 * is.  Runs on the bus stream behind every earlier fan-out; does not flush staged events; the same state and arguments give
 * byte-identical outputs.  Cost: one read of the range's control blocks on the device; host traffic is 16 * n_out bytes
 * plus the summary and a constant; one stream synchronisation.
 * CPBUS_EINVAL: n == 0, start_sub outside the range, a NULL n_out / next_sub, or out == NULL with cap > 0.
 * CPBUS_ENOENT: the range is not within this shard's subscribers. */
typedef struct cpbus_lag {
  uint32_t sub_id;   /* global id (sub_id_base applied)                                                          */
  uint32_t backlog;  /* undrained records: tail - cursor, cursor = head (lossless) or max(head, tail - ring_cap)    */
  uint64_t lost;     /* throughput mode: cursor - head, exactly cpbus_ready.lost; 0 in lossless mode               */
} cpbus_lag;         /* sizeof == 16 */
typedef struct cpbus_lag_summary {
  uint64_t active;          /* subscribed mailboxes in the range                                                  */
  uint64_t lagging;         /* ... with backlog >= min_backlog                                                    */
  uint64_t backlog_total, backlog_max, lost_total;   /* over the subscribed mailboxes of the range                */
  uint64_t hist[33];        /* subscribed mailboxes by backlog: [0] = 0, [k] = [2^(k-1), 2^k)                     */
} cpbus_lag_summary;
int cpbus_lagging(cpbus_t* bus, uint32_t first_sub, uint32_t n, uint32_t start_sub, uint32_t min_backlog,
                  cpbus_lag* out, size_t cap, size_t* n_out, uint32_t* next_sub, cpbus_lag_summary* sum);
/* Lossless mode: the mailboxes the next flush cannot get past (what a Go goroutine dump shows as the channel the publisher
 * sits on).  The next unit U is the first staged record together with every tick due at or before its ts_ns; with nothing
 * staged, the ticks due by the bus clock that the next flush would fire.  A subscribed mailbox blocks when its share of U —
 * the ticks of its armed slots due by then, plus one if it takes the record (code mask, {code, source} case, or unicast
 * target) — exceeds its room ring_cap - (tail - head): its admissible prefix of the staged remainder is 0.
 * out[0 .. min(cap, *n)) = the smallest blocking global ids, ascending; *n = how many there are.  After CPBUS_EAGAIN from
 * cpbus_flush, cpbus_publish, cpbus_send, cpbus_advance or a membership / timer call, *n >= 1, and draining exactly these
 * mailboxes lets the next flush deliver at least U (U takes at most 32/timers_per_sub + 1 ticks per slot plus one record,
 * below ring_cap).  Changes no state and flushes nothing; no kernel when the room bound proves that U fits, and none in
 * throughput mode (*n = 0).  CPBUS_EINVAL: NULL bus or n, or out == NULL with cap > 0. */
int cpbus_blockers(cpbus_t* bus, uint32_t* out, size_t cap, size_t* n);
/* Lossless stream shard: the subscribed mailboxes of this shard that give it an admissible prefix of 0 for its current
 * batch, the one after the last it completed, at its stored offset.  (cpbus_blockers on a stream shard looks at the bus's
 * own staged records and clock, not at the stream.)  The next unit U is the undelivered remainder's, by cpbus_stream_admit's
 * rules with the batch's n and watermark from the slot header: with r >= 2 records left, the first of them with the ticks
 * due by its ts_ns; with r = 1, that record with the ticks due by the watermark (admit holds a last record back when those
 * ticks do not fit); with r = 0, the ticks due by the watermark.  A mailbox blocks when its share of U exceeds its room, as
 * for cpbus_blockers.  out[0 .. min(cap, *n)) = the smallest blocking global ids, ascending; *n = how many there are.
 * *n >= 1 exactly when cpbus_stream_admit(st, n_batch, watermark, &p) on this shard would return CPBUS_EAGAIN, or p = 0
 * with records left (with nothing staged on the bus itself), and draining exactly these mailboxes makes that admit return p >= 1, or complete
 * an empty remainder.  Outstanding followers and rounds are resolved first: after a stalled device round the answer is for
 * the batch and offset the device cursor holds.  A batch the publisher has not released yet, or whose watermark admission
 * refuses with CPBUS_EORDER, gives *n = 0.  Changes no state: no flush, admission, offer or room-bound change; reads the
 * slot header (and U's record, 32 bytes) across the link; no kernel when the room bound proves that U fits, and none in
 * throughput mode (*n = 0).  Returns the sticky stream error as cpbus_stream_status does.  CPBUS_EINVAL: NULL st or n, or
 * out == NULL with cap > 0. */
int cpbus_stream_blockers(cpbus_stream_t* st, uint32_t* out, size_t cap, size_t* n);
/* Device-side consumer: every mailbox is read to the end and its records are discarded (head = tail), ordered behind
 * every earlier fan-out on the bus stream.  For subscribers nobody reads, and for measuring the lossless mode with
 * consumers that keep up. */
int cpbus_consume_all(cpbus_t* bus);
/* Last min(cap, ring_cap, count) delivered records, oldest first, without consuming. */
int cpbus_peek_window(cpbus_t* bus, uint32_t sub_id, cpbus_event* out, size_t cap, size_t* n);
int cpbus_digest(cpbus_t* bus, uint32_t first_sub, uint32_t n, cpbus_digest_t* out);
/* XOR-fold / sum of (count, digest) over [first_sub, first_sub+n) computed on the
 * device: one 32-byte D2H instead of 16 B per subscriber. */
int cpbus_digest_fold(cpbus_t* bus, uint32_t first_sub, uint32_t n, uint64_t out[4]);
/* Split form: _begin enqueues the fold + the 32-byte D2H on the bus stream and returns a ticket
 * (up to 8 outstanding); _end waits for that ticket only.  Lets a caller read step i's result
 * while step i+1 is already running. */
int cpbus_digest_fold_begin(cpbus_t* bus, uint32_t first_sub, uint32_t n, uint32_t* ticket);
int cpbus_digest_fold_end(cpbus_t* bus, uint32_t ticket, uint64_t out[4]);

/* Result of the LAST fan-out launch, written by the kernel itself: out = {records delivered by that launch,
 * ticks among them, sum over every mailbox it appended to of fold32(new digest) with
 * fold32(x) = low32(x ^ (x >> 32)), launch ordinal}.
 * _begin enqueues a 256-byte D2H on the bus stream (up to 8 outstanding tickets), _end waits for it.
 * On a CPBUS_CFG_SPARSE_TICKS bus the sparse kernel of a flush (due ticks alone, or with CPBUS_CFG_SPARSE_RECORDS also
 * records) is such a launch too, and a flush that launched nothing leaves the result as it was. */
int cpbus_step_result_begin(cpbus_t* bus, uint32_t* ticket);
int cpbus_step_result_end(cpbus_t* bus, uint32_t ticket, uint64_t out[4]);

/* ---- observation ---- */
/* DebugEvents (events/bus.go:34-54): drains the 10-slot ring of the last published
 * events, oldest first, stopping at a NonEvent.  Host-side, no 100 ms sleep. */
int cpbus_debug_events(cpbus_t* bus, cpbus_event* out, size_t cap, size_t* n);
int cpbus_stats(cpbus_t* bus, cpbus_stats_t* out);
/* Publish counts by {code, source}: the label set of the reference's `containerpilot_events` counter
 * (events/bus.go:60-68,130-132; code Metric is excluded there and here).  Covers both host publishes and batches that
 * reached the bus in device memory (counted by the kernel).  Writes at most cap entries, *n = entries available.
 * Call it from the publisher's thread (or with the publisher quiescent): it reads the table cpbus_publish updates. */
typedef struct cpbus_pair_count { uint32_t code, source_id; uint64_t count; } cpbus_pair_count;
int cpbus_publish_counts(cpbus_t* bus, cpbus_pair_count* out, size_t cap, size_t* n);
/* HBM layout, for zero-copy inspection by tests/bench: `ring` = n_max_subs mailboxes of
 * ring_cap records each (mailbox s starts at ring + s*ring_cap*32 bytes; slot of the j-th
 * delivered record = j mod ring_cap); `ctl` = n_max_subs control blocks of 32 bytes:
 * {u64 tail (records ever delivered); u64 head (consumer cursor); u64 digest; u32 mask
 * (bit 31 = subscribed, bits 24..27 = timer slots in use); u32 pad}. */
int cpbus_device_ptrs(cpbus_t* bus, void** ring, void** ctl);

/* ---- one bus handle over the GPUs of a box: the group ------------------------------------------------------------
 * A group is G ordinary buses (shards) behind one handle, driven by one host thread (the single ContainerPilot process).
 * Shard g lives on devices[g] (devices may repeat: several shards on one GPU) and owns a contiguous slice of the global
 * subscriber ids, split as evenly as possible (the first n_max_subs % G shards take one more).  Shard 0 creates a stream
 * (cpbus_stream_create) and the others attach to it; every flush of the group is one RAW stream batch that every shard
 * fans out, so unicast sends travel in publish order and are delivered by the owning shard's kernel only.
 * cfg is interpreted exactly as by cpbus_create, with n_max_subs = the total over the shards; cfg->stream must be NULL
 * (each shard runs on its own library-owned stream) and n_max_subs >= n_devices.
 *
 * The contract: the cpbus_group_* twin of an entry point takes the same arguments and returns the same status codes as
 * the single-bus call.  Any sequence of these calls, run on a group of G shards and on one bus created with the same
 * cpbus_config, gives the same return codes, the same subscriber and timer ids, byte-identical drain, drain_ready (records,
 * ready list and next_sub), peek_window, digest, digest_fold, debug_events and publish_counts outputs, and the same
 * cpbus_stats except the launch-shaped counters (batches, kernel_launches, admit_passes, admit_skipped, admit_partial,
 * device_splits).  This holds in throughput mode and in lossless mode (CPBUS_CFG_LOSSLESS), including where CPBUS_EAGAIN
 * is returned and how many events cpbus_stats.publishes says a stalled publish took: the group stages, flushes, splits
 * clock steps and cuts lossless prefixes where the single bus does, and admits each flush on every shard before it puts
 * the part every shard can take into the stream.
 * The intern table is shard 0's; the other shards only ever see source ids.  debug_events, publish_counts and
 * published_by_code are the group's own host records, merged with what shard 0's kernel accounted of the device batches
 * (cpbus_group_publish_device*); deliveries, ticks and overwritten are sums over the shards.
 * Device batches: cpbus_group_publish_device and _staged keep every rule of the single-bus calls (flush first, the order
 * and argument checks, all-or-nothing in lossless mode, the same cut of a batch one launch cannot take, CPBUS_EINVAL on a
 * CPBUS_CFG_DROP_MISSED_TICKS group).  d_events may live in the HBM of any GPU in the group's device list (the group
 * enables peer access between them); each launch copies the batch into shard 0's stream slot on the device and every
 * shard fans it out, so d_events must stay unchanged until cpbus_group_sync returns.  d_next / n_next are checked as on
 * the single bus and otherwise have no effect: the shards read the stream slot, not d_events. */
typedef struct cpbus_group cpbus_group_t;
int cpbus_group_create(const cpbus_config* cfg, const int32_t* devices, uint32_t n_devices, cpbus_group_t** out);
int cpbus_group_destroy(cpbus_group_t* g);
int cpbus_group_intern(cpbus_group_t* g, const char* s, size_t len, uint32_t* source_id);
int cpbus_group_intern_ephemeral(cpbus_group_t* g, const char* s, size_t len, uint32_t* source_id);
int cpbus_group_source(cpbus_group_t* g, uint32_t source_id, char* out, size_t cap, size_t* len);
int cpbus_group_subscribe(cpbus_group_t* g, uint32_t code_mask, uint32_t* sub_id);
int cpbus_group_subscribe_many(cpbus_group_t* g, const uint32_t* code_masks, uint32_t n, uint32_t* first_sub_id);
int cpbus_group_subscribe_pairs(cpbus_group_t* g, uint32_t code_mask, const cpbus_pair* pairs, uint32_t n_pairs, uint32_t* sub_id);
int cpbus_group_subscribe_pairs_many(cpbus_group_t* g, const uint32_t* code_masks, const cpbus_pair* pairs,
                                     const uint32_t* n_pairs, uint32_t n, uint32_t* first_sub_id);
int cpbus_group_unsubscribe(cpbus_group_t* g, uint32_t sub_id);
int cpbus_group_set_mask(cpbus_group_t* g, uint32_t sub_id, uint32_t code_mask);
int cpbus_group_timer_add(cpbus_group_t* g, uint32_t sub_id, uint64_t period_ns, uint32_t source_id, int oneshot, uint32_t* timer_id);
int cpbus_group_timer_add_many(cpbus_group_t* g, uint32_t first_sub, uint32_t n, uint64_t period_ns, const uint32_t* source_ids,
                               uint32_t source_id0, int oneshot);
int cpbus_group_timer_cancel(cpbus_group_t* g, uint32_t timer_id);
/* the bulk membership calls: each shard with work takes its ids, in array order, in one call of the shard's bulk call */
int cpbus_group_unsubscribe_many(cpbus_group_t* g, const uint32_t* sub_ids, uint32_t n, int* status, uint32_t* applied);
int cpbus_group_set_mask_many(cpbus_group_t* g, const uint32_t* sub_ids, const uint32_t* code_masks, uint32_t n, int* status,
                              uint32_t* applied);
int cpbus_group_timer_cancel_many(cpbus_group_t* g, const uint32_t* timer_ids, uint32_t n, int* status, uint32_t* applied);
/* bulk timer arming: each shard with work takes its elements, in array order, in one cpbus_timer_add_list call; the ids
 * are global slots with their generation, as cpbus_group_timer_add returns them */
int cpbus_group_timer_add_list(cpbus_group_t* g, const cpbus_timer_spec* specs, uint32_t n, uint32_t* timer_ids, int* status,
                               uint32_t* applied);
/* subscriber id reuse: the group keeps the free set over global ids; each shard with work takes its elements, in array
 * order, in one cpbus_release_many / cpbus_subscribe_list call */
int cpbus_group_release_many(cpbus_group_t* g, const uint32_t* sub_ids, uint32_t n, int* status, uint32_t* applied);
int cpbus_group_subscribe_list(cpbus_group_t* g, const uint32_t* code_masks, const cpbus_pair* pairs, const uint32_t* n_pairs,
                               uint32_t n, uint32_t* sub_ids);
int cpbus_group_publish(cpbus_group_t* g, const cpbus_event* ev, size_t n);
int cpbus_group_send(cpbus_group_t* g, uint32_t sub_id, const cpbus_event* ev);
int cpbus_group_publish_device(cpbus_group_t* g, const void* d_events, size_t n, uint64_t watermark_ns);
int cpbus_group_publish_device_staged(cpbus_group_t* g, const void* d_events, size_t n, uint64_t watermark_ns,
                                      const void* d_next, size_t n_next);
int cpbus_group_advance(cpbus_group_t* g, uint64_t now_ns);
int cpbus_group_flush(cpbus_group_t* g);
int cpbus_group_sync(cpbus_group_t* g);
int cpbus_group_drain(cpbus_group_t* g, uint32_t sub_id, cpbus_event* out, size_t cap, size_t* n, uint64_t* lost);
int cpbus_group_drain_ready(cpbus_group_t* g, uint32_t first_sub, uint32_t n, uint32_t start_sub,
                            cpbus_event* out, size_t cap, cpbus_ready* ready, size_t ready_cap,
                            size_t* n_ready, size_t* total, uint32_t* next_sub);
/* acknowledged drains: _take_ready walks the shards as _drain_ready does; _ack_many gives each shard its elements, in array
 * order, in one cpbus_ack_many call */
int cpbus_group_take_ready(cpbus_group_t* g, uint32_t first_sub, uint32_t n, uint32_t start_sub,
                           cpbus_event* out, size_t cap, cpbus_ready* ready, size_t ready_cap,
                           size_t* n_ready, size_t* total, uint32_t* next_sub);
int cpbus_group_ack_many(cpbus_group_t* g, const uint32_t* sub_ids, const uint32_t* counts, uint32_t n, int* status,
                         uint32_t* applied);
/* _lagging walks the shards in the single call's cyclic order with the cap that is left (as _drain_ready) and sums the
 * summaries (backlog_max: the maximum); _blockers evaluates the group's staged remainder and clock on every shard. */
int cpbus_group_lagging(cpbus_group_t* g, uint32_t first_sub, uint32_t n, uint32_t start_sub, uint32_t min_backlog,
                        cpbus_lag* out, size_t cap, size_t* n_out, uint32_t* next_sub, cpbus_lag_summary* sum);
int cpbus_group_blockers(cpbus_group_t* g, uint32_t* out, size_t cap, size_t* n);
int cpbus_group_consume_all(cpbus_group_t* g);
int cpbus_group_peek_window(cpbus_group_t* g, uint32_t sub_id, cpbus_event* out, size_t cap, size_t* n);
int cpbus_group_digest(cpbus_group_t* g, uint32_t first_sub, uint32_t n, cpbus_digest_t* out);
int cpbus_group_digest_fold(cpbus_group_t* g, uint32_t first_sub, uint32_t n, uint64_t out[4]);
int cpbus_group_debug_events(cpbus_group_t* g, cpbus_event* out, size_t cap, size_t* n);
int cpbus_group_stats(cpbus_group_t* g, cpbus_stats_t* out);
int cpbus_group_publish_counts(cpbus_group_t* g, cpbus_pair_count* out, size_t cap, size_t* n);

/* ---- names: EventCode.String (events/eventcode_string.go:9-15), FromString (events/events.go:52-86) ---- */
const char* cpbus_code_name(int code);               /* NULL if out of range      */
int cpbus_code_from_string(const char* name);        /* code, or -1 if not valid  */

const char* cpbus_strerror(int status);
const char* cpbus_last_cuda_error(void);
uint32_t cpbus_abi_version(void);
/* 64-bit record hash and digest multiplier used by the in-kernel digest (so the
 * oracle and external checkers can reproduce it without reading kernel code) */
uint64_t cpbus_record_hash(const cpbus_event* ev);
uint64_t cpbus_digest_multiplier(void);
/* How cpbus_publish_device cuts a batch one launch cannot take, as a pure host function (no device needed): ts[0..n) = the
 * records' timestamps (sorted), now_ns = the bus clock, window_ns = the widest watermark step of one launch (UINT64_MAX: no
 * timer armed).  Slice k = records [ends[k-1], ends[k]) with watermark watermarks[k]; *n_slices = how many there are (the
 * first `cap` are written).  CPBUS_EORDER: unsorted, a record beyond watermark_ns, or watermark_ns < now_ns. */
int cpbus_split_plan(const uint64_t* ts, size_t n, uint32_t batch_cap, uint64_t now_ns, uint64_t watermark_ns, uint64_t window_ns,
                     size_t* ends, uint64_t* watermarks, size_t cap, size_t* n_slices);
/* The order in which the filtered (ORDERED) fan-out walks the mailboxes, as a pure host function (no device needed):
 * out[] receives the indices i < n with active[i] != 0 (active == NULL: all), grouped per block of `block` consecutive
 * subscribers (0 = the library's policy from n and ring_cap: one block up to 16 GiB of rings, 8-GiB blocks beyond;
 * 0xFFFFFFFF = one block), inside a block by code mask — equal masks adjacent — and, with heavy_first, masks with more
 * codes first.  out must have room for n indices; returns how many were written (0 on bad arguments).  Delivery
 * results never depend on this order. */
size_t cpbus_mask_order(const uint32_t* masks, const uint8_t* active, uint32_t n, uint32_t ring_cap, uint32_t block,
                        int heavy_first, uint32_t* out);
/* The due index of a CPBUS_CFG_SPARSE_TICKS bus, as a pure host function (no device needed): ops[0..n_ops) run in order
 * over a table of n_slots timer slots (slot = subscriber * K + k).  Each op is {kind, slot, value}:
 *   CPBUS_DUE_CLOCK     the clock becomes value (arming is relative to it)
 *   CPBUS_DUE_ARM       arm `slot` periodic with period value (> 0): first due = clock + value, saturating at "never"
 *   CPBUS_DUE_ONESHOT   arm `slot` as a one-shot due at clock + value
 *   CPBUS_DUE_DISARM    cancel `slot`
 *   CPBUS_DUE_UNSUB     disarm the K slots of subscriber `slot`
 *   CPBUS_DUE_LAUNCH    a launch to watermark value: every armed slot due at or before it fires
 *   CPBUS_DUE_CATCHUP   the clock becomes value, with the CPBUS_CFG_DROP_MISSED_TICKS catch-up and no firing: every
 *                       periodic slot due at d <= value whose next firing d + period is also <= value moves to the last
 *                       firing of its grid <= value (below UINT64_MAX); CPBUS_EINVAL when value is behind the last launch
 * Each LAUNCH appends, for every slot that fires, in ascending slot order, {launch ordinal (0-based), slot, ticks, next due
 * (UINT64_MAX: never, or a one-shot that is done)} to out; *n_out = how many entries there are (the first cap are written).
 * CPBUS_EINVAL: a slot out of range, a period of 0, K not in {1, 2, 4, 8}, or a launch behind the previous launch. */
enum { CPBUS_DUE_CLOCK = 0, CPBUS_DUE_ARM = 1, CPBUS_DUE_ONESHOT = 2, CPBUS_DUE_DISARM = 3, CPBUS_DUE_UNSUB = 4, CPBUS_DUE_LAUNCH = 5,
       CPBUS_DUE_CATCHUP = 6 };
typedef struct cpbus_due_op { uint32_t kind, slot; uint64_t value; } cpbus_due_op;                       /* sizeof == 16 */
typedef struct cpbus_due_fire { uint64_t launch; uint32_t slot, pad; uint64_t ticks, next_due; } cpbus_due_fire; /* sizeof == 32 */
int cpbus_due_trace(const cpbus_due_op* ops, size_t n_ops, uint32_t n_slots, uint32_t K, cpbus_due_fire* out, size_t cap,
                    size_t* n_out);
/* The plan of a CPBUS_CFG_SPARSE_RECORDS flush, as a pure host function (no device needed; the bus runs the same code over
 * its own index).  Subscriber l < n_subs is subscribed when active[l] != 0 (active == NULL: all), with code mask masks[l]
 * and, when pairs != NULL, the exact cases pairs[l * CPBUS_MAX_PAIRS + j] for j < n_pairs[l] (taken as stored: a case
 * matches whatever the mask holds).  It takes record i of records[0..n_records) when the record is broadcast (target ==
 * CPBUS_TARGET_ALL) and its code's bit is in the mask or {code, source_id} is one of its cases, or when the record is
 * unicast to its id sub_id_base + l.  due_slots[0..n_due) are timer slots (subscriber * K + k, K in {0, 1, 2, 4, 8}) due
 * in this flush.  The candidates are the subscribed mailboxes that take a record and the mailboxes of the due slots.
 * Each candidate, in ascending order, gets one entry {local index, bitmask of its due slots (bit k), first, count}: its
 * records are rec_idx[first .. first + count), ascending (batch order).  *n_out = candidates, *n_idx = records planned;
 * the first cap entries and the first idx_cap indices are written.
 * CPBUS_ENOSPC when the flush takes the full fan-out instead: more than max_mailboxes due slots or candidates (a broadcast
 * code with more than max_mailboxes subscribers ends the planning at once), or more than max_deliveries planned records.
 * CPBUS_EINVAL: a NULL array with a non-zero count, a due slot of a subscriber >= n_subs, n_pairs[l] > CPBUS_MAX_PAIRS,
 * or K not in {0, 1, 2, 4, 8}. */
typedef struct cpbus_plan_entry { uint32_t local, due_bits, first, count; } cpbus_plan_entry;   /* sizeof == 16 */
int cpbus_sparse_plan(const uint32_t* masks, const uint8_t* active, uint32_t n_subs, const cpbus_pair* pairs,
                      const uint32_t* n_pairs, uint32_t sub_id_base, const cpbus_event* records, size_t n_records,
                      const uint32_t* due_slots, size_t n_due, uint32_t K, size_t max_mailboxes, size_t max_deliveries,
                      cpbus_plan_entry* out, size_t cap, uint32_t* rec_idx, size_t idx_cap, size_t* n_out, size_t* n_idx);
/* The candidate index of a CPBUS_CFG_SPARSE_DRAINS bus, as a pure host function (no device needed; the bus runs the same
 * code): ops[0..n_ops) run in order over mailboxes [0, n_subs), all subscribed and empty at the start.  Each op is {kind,
 * ticket, first, n, ids, n_ids, cut}; ids[ids .. ids + n_ids) is the op's mailbox list (local indices):
 *   CPBUS_READY_SPARSE       a sparse launch that appends to the listed mailboxes
 *   CPBUS_READY_FULL         a launch that may append to any mailbox (fan-out, lossless partial flush, device batch)
 *   CPBUS_READY_DRAIN        a cpbus_drain_ready over [first, first + n), begun under `ticket` (any value not outstanding)
 *   CPBUS_READY_TAKE         the same for cpbus_take_ready
 *   CPBUS_READY_END          the end of `ticket`: the drain took the listed mailboxes, and cut >= its n when it took every
 *                            ready mailbox of its range
 *   CPBUS_READY_CONSUME_ALL  cpbus_consume_all
 *   CPBUS_READY_RELEASE      cpbus_release_many of the listed mailboxes
 * counts[i] is, for a DRAIN or TAKE op, the number of candidates its scan visits (0: no launch) or -1 for the dense scan
 * (unknown candidates, or more than list_cap of them in the range), and 0 for every other op.  The candidate lists, each
 * in ascending order, go to out one after the other; *n_out = their total length (the first cap are written).  A set
 * that grows past 4 * list_cap becomes unknown.  CPBUS_EINVAL: an unknown kind, a range or id outside [0, n_subs), an id
 * list outside ids[0 .. n_ids_total), list_cap == 0, or a DRAIN / TAKE under an outstanding ticket; CPBUS_ENOENT: an END
 * of a ticket not outstanding. */
enum { CPBUS_READY_SPARSE = 0, CPBUS_READY_FULL = 1, CPBUS_READY_DRAIN = 2, CPBUS_READY_TAKE = 3, CPBUS_READY_END = 4,
       CPBUS_READY_CONSUME_ALL = 5, CPBUS_READY_RELEASE = 6 };
typedef struct cpbus_ready_op { uint32_t kind, ticket, first, n, ids, n_ids; uint64_t cut; } cpbus_ready_op;   /* sizeof == 32 */
int cpbus_ready_trace(const cpbus_ready_op* ops, size_t n_ops, const uint32_t* ids, size_t n_ids_total, uint32_t n_subs,
                      size_t list_cap, uint32_t* out, size_t cap, int64_t* counts, size_t* n_out);

#ifdef __cplusplus
}
#endif
#endif /* CPBUS_H */
