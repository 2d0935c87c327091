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
/* one periodic timer per subscriber [first_sub, first_sub+n); source_ids[i] (or source_id0+i if NULL) */
int cpbus_timer_add_many(cpbus_t* bus, uint32_t first_sub, uint32_t n, uint64_t period_ns, const uint32_t* source_ids, uint32_t source_id0, int oneshot);
int cpbus_timer_cancel(cpbus_t* bus, uint32_t timer_id);

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
 * ordered before any event published after this call. */
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
 * _begin enqueues a 256-byte D2H on the bus stream (up to 8 outstanding tickets), _end waits for it. */
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
 * published_by_code are the group's own host records; deliveries, ticks and overwritten are sums over the shards. */
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
int cpbus_group_publish(cpbus_group_t* g, const cpbus_event* ev, size_t n);
int cpbus_group_send(cpbus_group_t* g, uint32_t sub_id, const cpbus_event* ev);
int cpbus_group_advance(cpbus_group_t* g, uint64_t now_ns);
int cpbus_group_flush(cpbus_group_t* g);
int cpbus_group_sync(cpbus_group_t* g);
int cpbus_group_drain(cpbus_group_t* g, uint32_t sub_id, cpbus_event* out, size_t cap, size_t* n, uint64_t* lost);
int cpbus_group_drain_ready(cpbus_group_t* g, uint32_t first_sub, uint32_t n, uint32_t start_sub,
                            cpbus_event* out, size_t cap, cpbus_ready* ready, size_t ready_cap,
                            size_t* n_ready, size_t* total, uint32_t* next_sub);
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

#ifdef __cplusplus
}
#endif
#endif /* CPBUS_H */
