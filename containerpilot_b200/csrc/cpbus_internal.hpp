// cpbus_internal.hpp — what the translation units of libcpbus share, and nothing else includes: the bus (struct cpbus)
// and the group (struct cpbus_group) with the host front end they share, the front end's templates, and one
// declaration for each internal function that one file defines and another calls.
//   cpbus.cu         the single bus: every kernel launch, the streams, drains and queries (the only file that compiles
//                    the device part of cpbus_kernels.cuh)
//   cpbus_group.cpp  the group (cpbus_group_*): host C++ over the single bus's entry points and the functions below
//   cpbus_host.cpp   the host-only planners of host_index.hpp and the exports that need no device
// Everything here compiles as plain C++ too: nothing that struct cpbus or HostFront depends on may sit under
// __CUDACC__, so that every file sees one layout.  The internals live in namespace cpbus_host, hidden from the
// library's dynamic symbol table; the entry points of include/cpbus.h are the only exports.
#pragma once
#include <cstdio>
#include <deque>
#include <mutex>
#include <new>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/cpbus.h"
#include "cpbus_kernels.cuh"
#include "cuda_owned.hpp"
#include "host_index.hpp"

using namespace cpbus_dev;
using namespace cuda_owned;

#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess) {                                                                       \
      snprintf(g_cuda_err, sizeof(g_cuda_err), "%s:%d %s: %s", __FILE__, __LINE__, #call,          \
               cudaGetErrorString(e_));                                                            \
      return CPBUS_ECUDA;                                                                          \
    }                                                                                              \
  } while (0)

// Nothing may unwind through the C boundary (cgo, ctypes): every status-returning entry point is a function-try-block.
#define CPBUS_CATCH                                                                                   \
  catch (const std::bad_alloc&) { return CPBUS_ENOMEM; }                                              \
  catch (...) { snprintf(g_cuda_err, sizeof(g_cuda_err), "unexpected C++ exception"); return CPBUS_ECUDA; }

namespace cpbus_host __attribute__((visibility("hidden"))) {

// The last CUDA failure of this thread (cpbus_last_cuda_error), defined once, in cpbus_host.cpp.
extern thread_local char g_cuda_err[256];

// debug ring entry awaiting enqueue: a concrete event, or "the broadcast events of device launch `launch`"
struct DbgItem { bool marker; unsigned long long launch; cpbus_event ev; };

// publish counts by (code << 32 | source_id): the label set of `containerpilot_events` (events/bus.go:131).  Flat
// open-addressing table (key + 1 stored, 0 = empty): an increment is one probe in the common case, and a burst of n
// events is counted in two passes (slots prefetched, then incremented) so that cache misses of a high-cardinality
// source set overlap instead of adding up (a std::unordered_map here cost ~40 ns per published event).
struct PairCounter {
  std::vector<uint64_t> keys, cnts;
  size_t used = 0;
  static uint64_t mix(uint64_t k) { k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; return k; }
  void grow() {
    std::vector<uint64_t> ok, oc;
    ok.swap(keys); oc.swap(cnts);
    const size_t cap = ok.empty() ? 1024 : ok.size() * 2;
    keys.assign(cap, 0); cnts.assign(cap, 0); used = 0;
    for (size_t i = 0; i < ok.size(); i++) if (ok[i]) add(ok[i] - 1, oc[i]);
  }
  void add(uint64_t key, uint64_t by) {
    if ((used + 1) * 2 > keys.size()) grow();
    const size_t mask = keys.size() - 1;
    for (size_t i = mix(key) & mask;; i = (i + 1) & mask) {
      if (keys[i] == key + 1) { cnts[i] += by; return; }
      if (!keys[i]) { keys[i] = key + 1; cnts[i] = by; used++; return; }
    }
  }
  void prefetch(uint64_t key) const { if (!keys.empty()) { const size_t i = mix(key) & (keys.size() - 1); __builtin_prefetch(&keys[i]); __builtin_prefetch(&cnts[i]); } }
};

// timer id = slot index (subscriber * K + k) | generation << 26: a late cancel from an old context cannot disarm a re-armed slot
constexpr uint32_t kTimerSlotBits = 26, kTimerSlotMask = (1u << kTimerSlotBits) - 1u;

// The host front end: what the single bus (cpbus) and the group (cpbus_group) keep over their whole id space, and what the
// rules below share — the clock window (max_window), timer arming and retirement, staging (stage_one), the publish loop
// (publish_burst), the clock's advance (advance_clock), the debug ring and the publish counts.
struct HostFront {
  uint32_t B = 0, K = 0;                  // batch_cap, timers per subscriber
  // clock and ordinals
  uint64_t now = 0, last_watermark = 0, seq = 0;
  size_t n_staged = 0;
  std::vector<HostTimer> h_timers;        // N*K, allocated on first timer
  std::vector<size_t> oneshot_idx;        // armed one-shot timers (index into h_timers)
  uint32_t n_timers = 0;
  uint64_t min_period = UINT64_MAX;       // conservative lower bound over armed periodic timers
  bool drop_missed = false;               // CPBUS_CFG_DROP_MISSED_TICKS: a long clock step drops missed periodic ticks
  // DebugEvents ring (events/bus.go:18-21, 24-54)
  int dbg_head = -1, dbg_tail = 0;
  cpbus_event dbg[10]{};
  std::deque<DbgItem> dbg_pending;        // debug-ring entries not yet enqueued (events, or markers of device batches)
  PairCounter pub_pairs;                  // host publishes by (code << 32 | source_id), Metric excluded (bus.go:130-132)
  uint64_t publishes = 0, published_by_code[CPBUS_N_CODES] = {};   // host publishes and sends; by code (Metric excluded)
};

}  // namespace cpbus_host

using namespace cpbus_host;

// The handles of include/cpbus.h keep default visibility, because the exported entry points take them, while their
// insides are hidden: callers only ever hold pointers to them, so GCC's warning about the mix does not apply.
#pragma GCC diagnostic push
#pragma GCC diagnostic ignored "-Wattributes"
struct cpbus_stream;

struct cpbus : HostFront {
  cpbus_config cfg{};
  int device = 0, sm_count = 132;
  size_t smem_per_sm = 228 * 1024, smem_reserved = 1024;   // shared memory per SM, and what the system keeps per CTA
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  uint32_t N = 0, R = 0;
  int store = CPBUS_STORE_V8;
  bool lossless = false, use_digest = false;

  // HBM-resident state (SoA, one entry per subscriber of this shard)
  DeviceBuf<cpbus_event> d_ring;          // N * R records: each mailbox is one contiguous 32*R-byte ring
  DeviceBuf<SubCtl> d_ctl;                // N control blocks: {tail, head, digest, mask}, one sector each
  DeviceBuf<DevTimer> d_timers;           // N * K
  DeviceBuf<DevStats> d_stats;
  DeviceBuf<uint64_t> d_pow;              // P^0..: digest multiplier powers, TMA-loaded by every CTA
  DeviceBuf<unsigned char> d_desc;        // per-launch batch descriptor (CTA 0 writes, the others read)
  DeviceBuf<unsigned long long> d_desc_ready;
  unsigned long long launch_seq = 0;
  DeviceBuf<cpbus_event> d_batch_local;    // staged ingest: CTA 0's local copy of a peer batch
  DeviceBuf<cpbus_event> d_admit_batch;    // lossless stream: local copy of a slot's undelivered records for the admission pass
  static constexpr int kPrefetch = 3;      // fused ingest: later batches pulled over NVLink by earlier launches
  DeviceBuf<cpbus_event> d_prefetch[kPrefetch];
  const void* pf_ptr[kPrefetch] = {};      // which peer batch sits in d_prefetch[i] ...
  size_t pf_n[kPrefetch] = {};
  unsigned long long pf_seq[kPrefetch] = {};   // ... and which launch wrote it
  int pf_next = 0;
  std::vector<void*> shared_owned, shared_mapped;   // cpbus_shared_alloc / cpbus_shared_open
  // stream mode (cpbus_stream_*): device-managed prefetch of later stream batches + sticky error word
  DeviceBuf<unsigned long long> d_pf_state;   // [kStreamPrefetch]: which stream batch sits in d_prefetch[i]
  DeviceBuf<cpbus_event> d_pf_buf;            // kStreamPrefetch x batch_cap records (one allocation)
  MappedBuf<unsigned int> h_err;              // kErr* bits written by the fan-out kernel
  uint32_t stream_spin_us = 0;                // bound of the in-kernel wait for a stream batch (0 = 2 s)
  // follower launches (cpbus_stream_fanout_next): enqueued without the batch's shape, resolved lazily (follow_resolve)
  static constexpr int kFollowMax = 8;        // outstanding at most; the next one resolves first
  // kind: a follower, a lossless round (cpbus_stream_round_next: rec indexes h_round) or a cpbus_consume_all issued
  // behind outstanding rounds (no record: it resets the room bound in order)
  enum FollowKind { kFollower, kRound, kConsumeAll };
  struct FollowPending { cpbus_stream* st; unsigned long long launch_seq; int rec; FollowKind kind; };
  std::vector<FollowPending> follow_q;        // outstanding, in launch order
  MappedBuf<RoundRec> h_round;                // kFollowMax records written by the round agree kernels
  DeviceBuf<RoundDev> d_round;                // lossless rounds: the device copy of the room bound and clock, round scratch
  MappedBuf<FollowRec> h_follow;              // kFollowMax records written by the lead CTAs
  DeviceBuf<unsigned long long> d_follow_clock;   // 4 words: {watermark, launch ordinal} by launch parity
  int follow_next = 0;
  CudaEvent follow_done;
  std::recursive_mutex follow_mu;              // the queue, when stats or drains on another thread resolve it
  // accounting of device-published batches (cpbus_publish_device*, cpbus_stream_fanout): done by the kernel's lead CTA
  DeviceBuf<DevPubAcct> d_acct;
  // pinned staging for cpbus_stats / cpbus_debug_events / cpbus_publish_counts: the fields of a DevPubAcct before pair_key
  PinnedBuf<unsigned char> h_acct;
  DevPubAcct* host_acct() const { return reinterpret_cast<DevPubAcct*>(h_acct.get()); }
  DeviceBuf<cpbus_event> d_drain;             // cpbus_drain_many staging (grown)
  DeviceBuf<uint2> d_drain_idx;
  // cpbus_drain_ready staging (records go to d_drain; grown): header + tile counter + tile status, ready list, ring
  // slot of each run, and the header the gather kernel hands to the host.  Drain tickets share the first three.
  DeviceBuf<unsigned long long> d_ready_lb;
  DeviceBuf<cpbus_ready> d_ready; DeviceBuf<uint32_t> d_ready_slot;
  MappedBuf<unsigned long long> h_ready_hdr;
  // drain tickets (cpbus_drain_ready_begin, cpbus_take_ready_begin, cpbus_drain_ready_end): per slot, the mapped host buffer
  // the ticket gather kernel writes ([header, 128 bytes | cap records | min(ready_cap, n) entries], grown only while the
  // slot is free), the event recorded behind that kernel, and what _end needs.  ticket = generation << 3 | slot.
  static constexpr int kDrainTickets = 8;
  struct DrainTicket {
    MappedBuf<unsigned char> buf;
    CudaEvent done;
    bool busy = false;
    uint32_t ticket = 0, first = 0, n = 0, start = 0;
    size_t cap = 0, ready_cap = 0;
    // CPBUS_CFG_SPARSE_DRAINS: the drain's place in the candidate index, its kind, whether it covers every subscribed
    // mailbox, and whether its range held no candidate (nothing was enqueued: _end returns the empty result)
    uint64_t place = 0;
    bool take = false, whole = false, none = false;
  };
  DrainTicket drain_tk[kDrainTickets];
  uint32_t drain_tk_gen = 0, drain_tk_busy = 0;
  // cpbus_lagging / cpbus_blockers: look-back and summary words sized for every subscriber, the header the scans hand to the
  // host, the blocker ids (lossless buses) and the lagging entries (grown)
  DeviceBuf<unsigned long long> d_lag_lb;
  MappedBuf<unsigned long long> h_lag_hdr;
  MappedBuf<uint32_t> h_block;
  MappedBuf<cpbus_lag> h_lag;
  uint32_t subs_per_warp = 0;             // 0 = auto
  uint32_t order_block = 0;               // mask order is built per block of this many consecutive subscribers (0 = one global order)
  bool pdl = true;                        // programmatic dependent launch of consecutive fan-outs
  CudaEvent launched;                     // recorded after the latest fan-out (step results are read on the copy stream)
  int hints = -1;                         // -1 auto; bit0: control blocks / timer slots evict_last in L2
  static constexpr int kFoldSlots = 8;
  DeviceBuf<unsigned long long> d_fold;   // kFoldSlots x 4 words
  CudaEvent fold_done[kFoldSlots];
  uint32_t fold_next = 0;
  static constexpr int kStage = 8;         // staging ring: the host may run several flushes ahead of the GPU
  static constexpr int kDevSlots = 64, kDevEpoch = 16;
  DeviceBuf<cpbus_event> d_stage;          // kDevSlots x batch_cap records: device side of the staging ring
  CudaEvent epoch_done[kDevSlots / kDevEpoch];   // on the bus stream, after the last fan-out of each epoch of slots
  uint32_t dev_slot = 0;
  PinnedBuf<cpbus_event> h_batch[kStage];  // staging
  CudaEvent h2d_done[kStage];              // on copy_stream: batch c has reached HBM
  CudaStream copy_stream;                  // H2D of batch i+1 overlaps the fan-out of batch i
  CudaStream result_stream;                // D2H of step results: must not queue in front of the next batch's H2D
  // per-launch results written by the fan-out kernel itself (no extra kernel to read a step's result)
  DeviceBuf<DevResultSlot> d_result;       // kResultRing x kResultSub slots
  PinnedBuf<DevResultSlot> h_result;       // kFoldSlots tickets x kResultSub
  CudaEvent result_done[8];
  uint32_t result_next = 0;
  PinnedBuf<DevStats> h_stats;
  PinnedBuf<unsigned long long> h_fold;
  int cur = 0;

  // registry mirror (events/bus.go:13 `registry map[*Subscriber]bool`)
  std::vector<uint32_t> h_mask;
  std::vector<uint8_t> h_active;
  std::vector<uint8_t> h_npairs;          // second-level filter: exact {code, source} cases per subscriber (empty until first use)
  DeviceBuf<uint2> d_pairs;               // N x CPBUS_MAX_PAIRS, allocated by the first cpbus_subscribe_pairs (pair_tables)
  uint32_t n_paired = 0;                  // active subscribers with a pair table
  DeviceBuf<uint32_t> d_order;            // active subscribers sorted by code mask (ORDERED fan-out)
  uint32_t n_order = 0, n_filtered = 0;   // n_filtered: active subscribers whose mask is not CPBUS_MASK_ALL
  bool order_dirty = true;
  uint32_t n_next = 0, n_active = 0;
  // subscriber id reuse (cpbus_release_many / cpbus_subscribe_list): released mailboxes below n_next, and the same ids as
  // a min-heap that cpbus_subscribe_list hands out lowest first; the device copy of the slot-reset list (grown)
  std::vector<uint8_t> h_released;
  std::vector<uint32_t> free_ids;
  DeviceBuf<unsigned char> d_reset;

  // lossless mode: a lower bound of the free slots of the FULLEST mailbox.  While a batch provably fits (bound >= what it
  // can append to one mailbox) the admission pass and its host sync are skipped; the bound is refreshed exactly whenever
  // the admission kernel does run, and reset by cpbus_consume_all.
  uint64_t room_lb = 0;

  // CPBUS_CFG_SPARSE_TICKS: the armed slots by due time, and the plan of a sparse flush (entries, record indices, and the
  // {mailbox, record} pairs it is sorted from), staged in pinned memory as [entries | indices] and copied on the copy stream
  // into a device buffer (both grown).  CPBUS_CFG_SPARSE_RECORDS: records are planned too, from the subscription
  // index.
  bool sparse = false, sparse_records = false;
  DueIndex due;
  std::vector<uint32_t> due_slots;
  SubIndex rec_index;
  std::vector<cpbus_plan_entry> plan;
  std::vector<uint32_t> plan_idx;
  std::vector<uint64_t> plan_pairs;
  PinnedBuf<unsigned char> h_plan; DeviceBuf<unsigned char> d_plan;
  CudaEvent plan_done;                    // on copy_stream: the plan (and the batch in front of it) has reached HBM
  CudaEvent records_done;                 // on the bus stream: the record kernel is done with the plan
  // CPBUS_CFG_DROP_MISSED_TICKS on a sparse bus: the slots a catch-up moves (host index), and their device copy (grown)
  std::vector<uint32_t> catchup_slots;
  DeviceBuf<uint32_t> d_catchup;
  // the bulk membership calls (cpbus_unsubscribe_many, ...): device copy of the coalesced per-mailbox list (grown)
  DeviceBuf<MemberOp> d_member;
  // cpbus_timer_add_list: device copy of the armed slots' list (grown)
  DeviceBuf<TimerArmOp> d_arm;
  // acknowledged drains (cpbus_take_ready / cpbus_ack_many): the take cursor of every mailbox, allocated (zero) by the first
  // take; the ack list ([entries | elements], pinned staging and its device copy, grown) and the statuses (grown)
  DeviceBuf<unsigned long long> d_taken;
  PinnedBuf<unsigned char> h_ack; DeviceBuf<unsigned char> d_ack;
  MappedBuf<int> h_ack_status;
  // CPBUS_CFG_SPARSE_DRAINS: the candidate index (read and written under mu, like the drains' scratch: launches take mu to
  // update it), the candidates of one drain, and the list the list scan reads ({mailbox, walk position}; host copy and
  // device copy, grown)
  bool sparse_drains = false;
  ReadyIndex ready_ix;
  std::vector<uint32_t> ready_cand;
  std::vector<uint2> ready_list;
  DeviceBuf<uint2> d_ready_list;

  // intern table (Event.Source string <-> u32)
  std::unordered_map<std::string, uint32_t> intern;
  std::vector<std::string> sources;
  size_t intern_bytes = 0;
  // bounded region for payload strings (Metric "key|value"): recycled oldest-first
  struct EphSlot { std::string s; uint32_t gen = 0; bool live = false; };
  std::vector<EphSlot> eph;
  std::unordered_map<std::string, uint32_t> eph_map;
  uint32_t eph_next = 0;
  uint64_t eph_live = 0, eph_recycled = 0;
  std::vector<cpbus_stream*> streams;     // open streams (closed by cpbus_destroy if the caller did not)

  cpbus_stats_t st{};
  std::mutex mu;   // drain/stats from a second thread
};

// The group: one bus handle over the GPUs of a box (include/cpbus.h: cpbus_group_*).  Its host front end is the single
// bus's, over the whole id space, and so are the rules that run on it (stage_one, publish_burst, advance_clock, the timer
// table that sets the clock window, the debug ring and publish counts); only its flush differs (flush_staged of a group).
// A flush becomes one RAW stream batch that every shard fans out in full: in lossless mode the group first runs the single
// bus's admission (admit) on every shard and puts only the prefix every shard can take, with the single bus's partial
// watermark.  (cpbus_stream_admit would hold a batch back until the ticks due by its watermark fit too, where a partial
// cpbus_flush delivers the records and stalls on the ticks alone.)
// Shard clocks: a shard's clock is its last launched watermark; a shard without timers is moved to the group clock with
// cpbus_advance right before a timer is armed on it (no launch: it has no timer window), so every shard's `now + period`
// is the single bus's.  A shard with timers already has the group clock there (the group has just flushed at `now`).
struct cpbus_group : HostFront {
  std::vector<cpbus*> shards;
  std::vector<cpbus_stream*> streams;   // streams[0] owns the ring (shard 0), the others are attached
  std::vector<uint32_t> first;          // global index (sub_id_base not applied) of each shard's subscriber 0; + a sentinel
  uint32_t base = 0, N = 0;
  bool lossless = false;
  uint32_t n_next = 0, n_active = 0;
  std::vector<uint32_t> free_ids;       // released global indices, a min-heap (cpbus_group_subscribe_list)
  std::vector<cpbus_event> staged;      // B records
  bool dev_counted = false;             // shard 0 has accounted a device batch (cpbus_group_publish_device)
};
#pragma GCC diagnostic pop

namespace cpbus_host __attribute__((visibility("hidden"))) {

// ---- defined in cpbus.cu ----
// entry, and the checks of configs, ids and subscription lists
int enter(cpbus* b);
int dev_guard(cpbus* b);
int config_check(const cpbus_config* cfg, uint32_t* R_out, uint32_t* B_out);
bool id_range(uint32_t base, uint32_t n_next, uint32_t first, uint64_t n, uint32_t* index);
int subscribe_list_check(const uint32_t* n_pairs, const cpbus_pair* pairs, uint32_t n);
// the timer table and the clock window of a host front end
uint64_t max_window(const HostFront* f);
bool flush_idle(HostFront* f, uint64_t w);
void retire_oneshots(HostFront* f, uint64_t w);
HostTimer& timer_arm(HostFront* f, size_t slot, uint64_t period, uint32_t source_id, bool oneshot);
void timer_disarm(HostFront* f, size_t slot, bool reset_bound);
// lossless admission on one bus: the room bound's fast path, and the admission pass
bool admit_fits(cpbus* b, uint32_t n, uint64_t w);
int admit_pass(cpbus* b, const cpbus_event* d_src, uint32_t n, uint64_t w, bool* ok, uint32_t* prefix);
// the stream: the put of a batch into the next slot, from host or device memory, and a consumer's launch of the next
// m records, with or without the accounting of a device-published batch
int stream_put(cpbus_stream* st, const cpbus_event* ev, size_t n, uint64_t now_ns, uint32_t flags, bool device_src);
int stream_fanout_prefix(cpbus_stream* st, size_t n, uint64_t now_ns, size_t m, bool account);
// the debug ring and the publish counts
void dbg_enqueue(HostFront* f, const cpbus_event& e);
void dbg_mark_device_batch(HostFront* f, unsigned long long launch);
int dbg_resolve(HostFront* f, cpbus* b);
size_t dbg_read(HostFront* f, cpbus_event* out, size_t cap);
int device_pairs(cpbus* b, std::vector<unsigned long long>& keys, std::vector<unsigned long long>& cnts);
void pair_counts(const HostFront* f, const unsigned long long* dev_keys, const unsigned long long* dev_cnts, size_t n_dev,
                 cpbus_pair_count* out, size_t cap, size_t* n);
// the bodies of the paged queries and of cpbus_ack_many on one bus, which a group runs shard by shard
int drain_ready_impl(cpbus_t* b, uint32_t first_sub, uint32_t n, uint32_t start_sub, cpbus_event* out, size_t cap,
                     cpbus_ready* ready, size_t ready_cap, size_t* n_ready, size_t* total, uint32_t* next_sub,
                     bool* all_taken, bool take = false);
// The cap check of every sparse drain (single bus, ticket or group; take: cpbus_take_ready's): a ready mailbox always fits
// an empty call (cap >= ring_cap), record offsets are 32-bit, and only a lossless bus holds records back for acks.
inline bool ready_cap_ok(size_t cap, uint32_t ring_cap, bool take, bool lossless) {
  return cap >= ring_cap && cap <= 0xFFFFFFFFull && (!take || lossless);
}
int ack_many_impl(cpbus* b, const uint32_t* sub_ids, const uint32_t* counts, uint32_t n, int* st);
void ack_statuses(const std::vector<int>& st, int* status, uint32_t* applied);
int lagging_impl(cpbus_t* b, uint32_t first_sub, uint32_t n, uint32_t start_sub, uint32_t min_backlog, cpbus_lag* out,
                 size_t cap, size_t* n_out, uint32_t* next_sub, cpbus_lag_summary* sum, bool* all_returned);
int blockers_impl(cpbus* b, const cpbus_event* rec, uint64_t t, uint32_t* out, size_t cap, size_t* n);

// ---- one overload per owner: the bus's in cpbus.cu, the group's in cpbus_group.cpp ----
// where the next staged record goes
cpbus_event* staging(cpbus* b);
cpbus_event* staging(cpbus_group* g);
// the flush of the staged records to watermark w
int flush_staged(cpbus* b, uint64_t w);
int flush_staged(cpbus_group* g, uint64_t w);
// CPBUS_CFG_DROP_MISSED_TICKS: the catch-up of a clock step to `now`
int catch_up(cpbus* b, uint64_t now);
int catch_up(cpbus_group* g, uint64_t now);

// stage_one, publish_burst and advance_clock run on the single bus and on the group alike (Owner = cpbus or cpbus_group):
// one body each, with the owner's own flush.
template <class Owner>
int stage_one(Owner* o, uint32_t code, uint32_t source_id, uint32_t target, uint32_t flags) {
  if (o->n_staged == o->B) { int rc = flush_staged(o, o->now); if (rc) return rc; }
  cpbus_event& e = staging(o)[o->n_staged++];
  e.seq = o->seq++; e.ts_ns = o->now; e.code = code; e.source_id = source_id; e.target = target; e.flags = flags;
  return CPBUS_OK;
}

// Publish a burst (events/bus.go:126-139): nothing of a burst with an invalid code is published.
template <class Owner>
int publish_burst(Owner* o, const cpbus_event* ev, size_t n) {
  for (size_t i = 0; i < n; i++) {   // counter slots of the whole burst: requested up front, touched in the loop below
    if (ev[i].code < CPBUS_N_CODES && ev[i].code != CPBUS_METRIC) o->pub_pairs.prefetch(((uint64_t)ev[i].code << 32) | ev[i].source_id);
  }
  // The debug ring holds 10 entries (events/bus.go:24-31): of a burst only the last 10 published can ever be seen, so only
  // those are enqueued — including when the call stops early (CPBUS_EAGAIN from an automatic flush in lossless mode).
  auto dbg_tail = [&](size_t published) {
    for (size_t j = published > 10 ? published - 10 : 0; j < published; j++) {
      cpbus_event e{};
      e.seq = o->seq - (published - j); e.ts_ns = o->now; e.code = ev[j].code; e.source_id = ev[j].source_id; e.target = CPBUS_TARGET_ALL;
      dbg_enqueue(o, e);
    }
  };
  for (size_t i = 0; i < n; i++) if (ev[i].code >= CPBUS_N_CODES) return CPBUS_EINVAL;
  for (size_t i = 0; i < n; i++) {
    const uint32_t code = ev[i].code;
    const int rc = stage_one(o, code, ev[i].source_id, CPBUS_TARGET_ALL, 0);
    if (rc) { dbg_tail(i); return rc; }
    if (code != CPBUS_METRIC) {                                  // events/bus.go:130-132
      o->published_by_code[code]++;
      o->pub_pairs.add(((uint64_t)code << 32) | ev[i].source_id, 1);
    }
    o->publishes++;
  }
  dbg_tail(n);                                                   // events/bus.go:139
  return CPBUS_OK;
}

// Move the clock to now_ns.  The kernel looks at <= 32/K candidate firings per timer slot per launch: every flush window is
// kept within that many periods of the fastest periodic timer (for a group, a stream batch never steps past a shard's window).
// CPBUS_CFG_DROP_MISSED_TICKS: only a step longer than the shortest period can hold two firings of one timer.  On such a
// step, what is due by the old clock is delivered on its own first (the previous step's window split keeps that flush within
// the window; CPBUS_EAGAIN leaves the clock where it was), then every periodic timer with missed firings moves to its last
// one, so the window split below launches at most one firing per slot.
template <class Owner>
int advance_clock(Owner* o, uint64_t now_ns) {
  if (now_ns < o->now) return CPBUS_EORDER;
  if (now_ns == o->now) return CPBUS_OK;
  if (o->drop_missed && o->n_timers && o->min_period != UINT64_MAX && now_ns - o->now > o->min_period) {
    int rc = flush_staged(o, o->now);
    if (rc || (rc = catch_up(o, now_ns))) return rc;
  }
  const uint64_t win = max_window(o);
  while (win != UINT64_MAX && now_ns - o->last_watermark > win) {
    o->now = o->last_watermark + win;
    const int rc = flush_staged(o, o->now); if (rc) return rc;
  }
  o->now = now_ns;
  return CPBUS_OK;
}

}  // namespace cpbus_host
