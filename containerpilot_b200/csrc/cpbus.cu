// cpbus.cu — libcpbus: C-ABI (include/cpbus.h) over the sm_90a (H100) kernels.
//
// Host-side bookkeeping that the reference keeps in Go (events/bus.go): the
// registry, the 10-slot debug ring, per-code publish counts, the Source intern
// table, the virtual clock, staging of published events into pinned batches.
// There is NO CPU data path: without a CUDA device cpbus_create fails with
// CPBUS_ENODEV, and nothing here touches oracle/.
#include "cpbus_kernels.cuh"

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

using namespace cpbus_dev;

namespace {

thread_local char g_cuda_err[256] = "";

#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess) {                                                                       \
      snprintf(g_cuda_err, sizeof(g_cuda_err), "%s:%d %s: %s", __FILE__, __LINE__, #call,          \
               cudaGetErrorString(e_));                                                            \
      return CPBUS_ECUDA;                                                                          \
    }                                                                                              \
  } while (0)

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

struct HostTimer { bool active = false, oneshot = false; uint8_t gen = 0; uint64_t period = 0, next_due = 0; uint32_t source_id = 0; };
// Due times saturate: one that would pass UINT64_MAX - 1 is kTimerIdle, "never".  The slot stays armed (it counts in
// n_timers and can be cancelled); the kernel never fires a tick due at kTimerIdle.
inline uint64_t due_after(uint64_t t, uint64_t period) { return period >= kTimerIdle - t ? kTimerIdle : t + period; }
// a one-shot due by watermark w has fired on the device and disarmed itself
inline bool oneshot_fired(uint64_t next_due, uint64_t w) { return next_due <= w && next_due != kTimerIdle; }
// timer id = slot index (subscriber * K + k) | generation << 26: a late cancel from an old context cannot disarm a re-armed slot
constexpr uint32_t kTimerSlotBits = 26, kTimerSlotMask = (1u << kTimerSlotBits) - 1u;

}  // namespace

struct cpbus_stream;

struct cpbus {
  cpbus_config cfg{};
  int device = 0, sm_count = 132;
  size_t smem_per_sm = 228 * 1024, smem_reserved = 1024;   // shared memory per SM, and what the system keeps per CTA
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  uint32_t N = 0, R = 0, B = 0, K = 0;
  int store = CPBUS_STORE_V8;
  bool lossless = false, use_digest = false;

  // HBM-resident state (SoA, one entry per subscriber of this shard)
  cpbus_event* d_ring = nullptr;          // N * R records: each mailbox is one contiguous 32*R-byte ring
  SubCtl* d_ctl = nullptr;                // N control blocks: {tail, head, digest, mask}, one sector each
  DevTimer* d_timers = nullptr;           // N * K
  DevStats* d_stats = nullptr;
  uint64_t* d_pow = nullptr;              // P^0..: digest multiplier powers, TMA-loaded by every CTA
  unsigned char* d_desc = nullptr;        // per-launch batch descriptor (CTA 0 writes, the others read)
  unsigned long long* d_desc_ready = nullptr;
  unsigned long long launch_seq = 0;
  cpbus_event* d_batch_local = nullptr;    // staged ingest: CTA 0's local copy of a peer batch
  cpbus_event* d_admit_batch = nullptr;    // lossless stream: local copy of a slot's undelivered records for the admission pass
  static constexpr int kPrefetch = 3;      // fused ingest: later batches pulled over NVLink by earlier launches
  cpbus_event* d_prefetch[kPrefetch] = {};
  const void* pf_ptr[kPrefetch] = {};      // which peer batch sits in d_prefetch[i] ...
  size_t pf_n[kPrefetch] = {};
  unsigned long long pf_seq[kPrefetch] = {};   // ... and which launch wrote it
  int pf_next = 0;
  std::vector<void*> shared_owned, shared_mapped;   // cpbus_shared_alloc / cpbus_shared_open
  // stream mode (cpbus_stream_*): device-managed prefetch of later stream batches + sticky error word
  unsigned long long* d_pf_state = nullptr;   // [kStreamPrefetch]: which stream batch sits in d_prefetch[i]
  cpbus_event* d_pf_buf = nullptr;            // kStreamPrefetch x batch_cap records (one allocation)
  unsigned int* h_err = nullptr;              // pinned + mapped: kErr* bits written by the fan-out kernel
  unsigned int* d_err = nullptr;              // device alias of h_err
  uint32_t stream_spin_us = 0;                // bound of the in-kernel wait for a stream batch (0 = 2 s)
  // follower launches (cpbus_stream_fanout_next): enqueued without the batch's shape, resolved lazily (follow_resolve)
  static constexpr int kFollowMax = 8;        // outstanding at most; the next one resolves first
  // kind: a follower, a lossless round (cpbus_stream_round_next: rec indexes h_round) or a cpbus_consume_all issued
  // behind outstanding rounds (no record: it resets the room bound in order)
  enum FollowKind { kFollower, kRound, kConsumeAll };
  struct FollowPending { cpbus_stream* st; unsigned long long launch_seq; int rec; FollowKind kind; };
  std::vector<FollowPending> follow_q;        // outstanding, in launch order
  RoundRec* h_round = nullptr;                // pinned + mapped: kFollowMax records written by the round agree kernels
  RoundRec* d_round_rec = nullptr;            // device alias of h_round
  RoundDev* d_round = nullptr;                // lossless rounds: the device copy of the room bound and clock, round scratch
  FollowRec* h_follow = nullptr;              // pinned + mapped: kFollowMax records written by the lead CTAs
  FollowRec* d_follow = nullptr;              // device alias of h_follow
  unsigned long long* d_follow_clock = nullptr;   // 4 words: {watermark, launch ordinal} by launch parity
  int follow_next = 0;
  cudaEvent_t follow_done = nullptr;
  std::recursive_mutex follow_mu;              // the queue, when stats or drains on another thread resolve it
  // accounting of device-published batches (cpbus_publish_device*, cpbus_stream_fanout): done by the kernel's lead CTA
  DevPubAcct* d_acct = nullptr;
  DevPubAcct* h_acct = nullptr;               // pinned staging for cpbus_stats / cpbus_debug_events / cpbus_publish_counts
  std::deque<DbgItem> dbg_pending;            // debug-ring entries not yet enqueued (events, or markers of device batches)
  PairCounter pub_pairs;                              // host publishes by (code << 32 | source_id), Metric excluded (bus.go:130-132)
  cpbus_event* d_drain = nullptr; size_t drain_cap = 0;        // cpbus_drain_many staging
  uint2* d_drain_idx = nullptr; size_t drain_idx_cap = 0;
  // cpbus_drain_ready staging (records go to d_drain): header + tile counter + tile status, ready list, ring slot of each run
  unsigned long long* d_ready_lb = nullptr; size_t ready_lb_tiles = 0;
  cpbus_ready* d_ready = nullptr; uint32_t* d_ready_slot = nullptr; size_t ready_stage_cap = 0;
  unsigned long long* h_ready_hdr = nullptr;   // pinned + mapped: the header the gather kernel hands to the host
  unsigned long long* d_ready_hdr = nullptr;   // device alias of h_ready_hdr
  uint32_t subs_per_warp = 0;             // 0 = auto
  uint32_t order_block = 0;               // mask order is built per block of this many consecutive subscribers (0 = one global order)
  bool pdl = true;                        // programmatic dependent launch of consecutive fan-outs
  cudaEvent_t launched = nullptr;         // recorded after the latest fan-out (step results are read on the copy stream)
  int hints = -1;                         // -1 auto; bit0: control blocks / timer slots evict_last in L2
  static constexpr int kFoldSlots = 8;
  unsigned long long* d_fold = nullptr;   // kFoldSlots x 4 words
  cudaEvent_t fold_done[kFoldSlots] = {};
  uint32_t fold_next = 0;
  static constexpr int kStage = 8;         // staging ring: the host may run several flushes ahead of the GPU
  static constexpr int kDevSlots = 64, kDevEpoch = 16;
  cpbus_event* d_stage = nullptr;          // kDevSlots x batch_cap records: device side of the staging ring
  cudaEvent_t epoch_done[kDevSlots / kDevEpoch] = {};   // on the bus stream, after the last fan-out of each epoch of slots
  uint32_t dev_slot = 0;
  cpbus_event* h_batch[kStage] = {};       // pinned staging
  cudaEvent_t h2d_done[kStage] = {};       // on copy_stream: batch c has reached HBM
  cudaStream_t copy_stream = nullptr;      // H2D of batch i+1 overlaps the fan-out of batch i
  cudaStream_t result_stream = nullptr;    // D2H of step results: must not queue in front of the next batch's H2D
  // per-launch results written by the fan-out kernel itself (no extra kernel to read a step's result)
  DevResultSlot* d_result = nullptr;       // kResultRing x kResultSub slots
  DevResultSlot* h_result = nullptr;       // pinned, kFoldSlots tickets x kResultSub
  cudaEvent_t result_done[8] = {};
  uint32_t result_next = 0;
  DevStats* h_stats = nullptr;            // pinned
  unsigned long long* h_fold = nullptr;   // pinned
  int cur = 0;
  size_t n_staged = 0;

  // registry mirror (events/bus.go:13 `registry map[*Subscriber]bool`)
  std::vector<uint32_t> h_mask;
  std::vector<uint8_t> h_active;
  std::vector<uint8_t> h_npairs;          // second-level filter: exact {code, source} cases per subscriber (empty until first use)
  uint2* d_pairs = nullptr;               // N x CPBUS_MAX_PAIRS, allocated by the first cpbus_subscribe_pairs
  uint32_t n_paired = 0;                  // active subscribers with a pair table
  uint32_t* d_order = nullptr;            // active subscribers sorted by code mask (ORDERED fan-out)
  uint32_t n_order = 0, n_filtered = 0;   // n_filtered: active subscribers whose mask is not CPBUS_MASK_ALL
  bool order_dirty = true;
  std::vector<size_t> oneshot_idx;        // armed one-shot timers (index into h_timers)
  std::vector<HostTimer> h_timers;        // N*K, allocated on first timer
  uint32_t n_next = 0, n_active = 0, n_timers = 0;
  uint64_t min_period = UINT64_MAX;       // conservative lower bound over armed periodic timers

  // clock and ordinals
  uint64_t now = 0, last_watermark = 0, seq = 0;
  // lossless mode: a lower bound of the free slots of the FULLEST mailbox.  While a batch provably fits (bound >= what it
  // can append to one mailbox) the admission pass and its host sync are skipped; the bound is refreshed exactly whenever
  // the admission kernel does run, and reset by cpbus_consume_all.
  uint64_t room_lb = 0;

  // DebugEvents ring (events/bus.go:18-21, 24-54)
  int dbg_head = -1, dbg_tail = 0;
  cpbus_event dbg[10]{};

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

namespace {

// counting sort of the active subscribers by their 17-bit code mask (stable: ids ascending inside a mask)
int rebuild_order(cpbus* b);

int dev_guard(cpbus* b) {
  CK(cudaSetDevice(b->device));
  return CPBUS_OK;
}

// Pinned host memory that the device writes through a mapping: *h and its device alias *d, set only on success.
template <class T>
cudaError_t mapped_alloc(size_t bytes, T** h, T** d) {
  void *ph = nullptr, *pd = nullptr;
  cudaError_t e = cudaHostAlloc(&ph, bytes, cudaHostAllocMapped);
  if (e != cudaSuccess) return e;
  if ((e = cudaHostGetDevicePointer(&pd, ph, 0)) != cudaSuccess) { cudaFreeHost(ph); return e; }
  *h = static_cast<T*>(ph); *d = static_cast<T*>(pd);
  return cudaSuccess;
}

// How long the host waits for a stream's consumers or publisher (cpbus_stream_set_timeout; 0 = 2 s).
std::chrono::microseconds stream_budget(const cpbus* b) {
  return std::chrono::microseconds(b->stream_spin_us ? b->stream_spin_us : 2000000u);
}

// The sticky stream error of this bus: a followed batch out of order (CPBUS_EORDER), otherwise a batch that never arrived or
// did not match its header (CPBUS_ETIMEDOUT).
int stream_error(const cpbus* b) {
  const unsigned int e = *(volatile const unsigned int*)b->h_err;
  return (e & kErrFollowOrder) ? CPBUS_EORDER : (e ? CPBUS_ETIMEDOUT : CPBUS_OK);
}

uint32_t mask_word(const cpbus* b, uint32_t local) {
  uint32_t hint = 0;
  if (b->K && !b->h_timers.empty())
    for (uint32_t k = 0; k < b->K; k++)
      if (b->h_timers[(size_t)local * b->K + k].active) hint = k + 1;
  if (!b->h_active[local]) return 0;
  const uint32_t pair_bit = (!b->h_npairs.empty() && b->h_npairs[local]) ? kPairBit : 0u;
  return (b->h_mask[local] & CPBUS_MASK_ALL) | (hint << kTimerHintShift) | pair_bit | kActiveBit;
}

void dbg_ring_put(cpbus* b, const cpbus_event& e) {   // events/bus.go:24-31
  b->dbg[(b->dbg_head + 1) % 10] = e;
  int old = b->dbg_head;
  b->dbg_head = (b->dbg_head + 1) % 10;
  if (old != -1 && b->dbg_head == b->dbg_tail) b->dbg_tail = (b->dbg_tail + 1) % 10;
}

// While the broadcast events of a device-published batch are still unknown to the host (a marker is pending), later
// enqueues queue up behind it so that the ring keeps the global publish order; cpbus_debug_events resolves them.
void dbg_enqueue(cpbus* b, const cpbus_event& e) {
  if (b->dbg_pending.empty()) { dbg_ring_put(b, e); return; }
  b->dbg_pending.push_back(DbgItem{false, 0ull, e});
  if (b->dbg_pending.size() > (size_t)kAcctDbgRing) b->dbg_pending.pop_front();
}

void dbg_mark_device_batch(cpbus* b, unsigned long long launch) {
  b->dbg_pending.push_back(DbgItem{true, launch, cpbus_event{}});
  if (b->dbg_pending.size() > (size_t)kAcctDbgRing) b->dbg_pending.pop_front();
}

// The mask order of the ORDERED build, host-only (exported as cpbus_mask_order so that it can be tested without a GPU).
// Equal masks become neighbours, so a warp's consecutive mailboxes share one filter pass.
//  * Blocks.  A GLOBAL order scatters the mailboxes that are written at the same time over the whole ring area (1,048,576
//    rings = 32 GiB = 16,384 2-MiB pages, all live at once); ordering block by block of consecutive subscribers keeps the
//    concurrently written rings within a few hundred pages, at the price of shorter runs.  Policy (block == 0): one global
//    order up to 16 GiB of rings, blocks of 8 GiB beyond.
//  * Heavy first.  Within a block a second, stable pass by the number of codes in the mask, most first: CTAs are dispatched
//    in block order, so the mailboxes that take the most records start first and the launch's last wave is made of the light
//    ones (shorter tail before the next launch may start); equal masks stay neighbours.
static void mask_order(const uint32_t* masks, const uint8_t* active, uint32_t n, uint32_t ring_cap, uint32_t block, bool heavy_first,
                       std::vector<uint32_t>& order) {
  order.clear();
  order.reserve(n);
  const uint64_t ring_bytes = (uint64_t)ring_cap * sizeof(cpbus_event);
  uint32_t blk = block;
  if (!blk) blk = (uint64_t)n * ring_bytes <= (16ull << 30) ? std::max(1u, n) : (uint32_t)std::max<uint64_t>(4096, (8ull << 30) / ring_bytes);
  if (block == 0xFFFFFFFFu) blk = std::max(1u, n);   // one global order (A/B)
  std::vector<uint32_t> count((size_t)CPBUS_MASK_ALL + 2), tmp;
  for (uint32_t lo = 0; lo < n; lo += blk) {
    const uint32_t hi = (uint32_t)std::min<uint64_t>((uint64_t)lo + blk, n);
    std::fill(count.begin(), count.end(), 0u);
    for (uint32_t i = lo; i < hi; i++) if (!active || active[i]) count[(masks[i] & CPBUS_MASK_ALL) + 1]++;
    for (size_t k = 1; k < count.size(); k++) count[k] += count[k - 1];
    const size_t base = order.size();
    order.resize(base + count.back());
    for (uint32_t i = lo; i < hi; i++) if (!active || active[i]) order[base + count[masks[i] & CPBUS_MASK_ALL]++] = i;
    if (heavy_first) {
      const size_t nb = order.size() - base;
      uint32_t pc_count[34] = {};
      for (size_t k = 0; k < nb; k++) pc_count[32 - __builtin_popcount(masks[order[base + k]] & CPBUS_MASK_ALL) + 1]++;
      for (int k = 1; k < 34; k++) pc_count[k] += pc_count[k - 1];
      tmp.resize(nb);
      for (size_t k = 0; k < nb; k++) tmp[pc_count[32 - __builtin_popcount(masks[order[base + k]] & CPBUS_MASK_ALL)]++] = order[base + k];
      std::copy(tmp.begin(), tmp.end(), order.begin() + base);
    }
  }
}

int rebuild_order(cpbus* b) {
  std::vector<uint32_t> order;
  static_assert(sizeof(b->h_active[0]) == 1, "h_active is a byte vector");
  mask_order(b->h_mask.data(), reinterpret_cast<const uint8_t*>(b->h_active.data()), b->n_next, b->R, b->order_block, /*heavy_first=*/true, order);
  b->n_order = (uint32_t)order.size();
  if (b->n_order) {
    CK(cudaMemcpyAsync(b->d_order, order.data(), (size_t)b->n_order * 4, cudaMemcpyHostToDevice, b->stream));
    CK(cudaStreamSynchronize(b->stream));
  }
  b->order_dirty = false;
  return CPBUS_OK;
}

constexpr int kFanoutMaxSmem = 200 * 1024;

enum { kLaunchPlain = 0, kLaunchFollow = 1, kLaunchRound = 2 };

template <int STORE, bool TIMERS, bool DIGEST, bool ORDERED, bool PAIRS = false>
int launch_fanout_t(cpbus* b, const FanoutParams& p, uint32_t grid, size_t smem, int kind) {
  static bool attr_done[3][64] = {};   // per instantiation AND per device: function attributes are per-device state
  void (*kernel)(FanoutParams) = kind == kLaunchRound  ? fanout_round_kernel<STORE, TIMERS, DIGEST, ORDERED, PAIRS>
                               : kind == kLaunchFollow ? fanout_follow_kernel<STORE, TIMERS, DIGEST, ORDERED, PAIRS>
                                                       : fanout_kernel<STORE, TIMERS, DIGEST, ORDERED, PAIRS>;
  const int dev = b->device & 63;
  if (!attr_done[kind][dev]) {
    CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kFanoutMaxSmem));
    attr_done[kind][dev] = true;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = smem; cfg.stream = b->stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;   // PDL: the next fan-out's prologue overlaps this one's tail
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  // (a round's fan-out reads what the agree kernel in front of it wrote: launched without PDL, see fanout_round_kernel)
  cfg.attrs = attr; cfg.numAttrs = b->pdl && kind != kLaunchRound ? 1 : 0;
  CK(cudaLaunchKernelEx(&cfg, kernel, p));
  CK(cudaGetLastError());
  return CPBUS_OK;
}

uint64_t max_window(const cpbus* b);

// Lossless rounds wait in the kernel: for the publisher's header (decide) and for the other shards' offers (agree).  With
// CUDA's lazy module loading, the first launch of a kernel loads it, and a load may wait for the kernels already running on
// the device — such as a round waiting for a batch that this very thread has yet to put, or for an offer that another shard
// of this thread has yet to queue.  So every kernel a lossless bus may launch while its rounds wait is loaded up front, once
// per device, when the bus is created.
template <int ST>
int preload_round_fanouts() {
  void (*ks[])(FanoutParams) = {
      fanout_round_kernel<ST, false, false, false>, fanout_round_kernel<ST, false, true, false>,
      fanout_round_kernel<ST, true, false, false>, fanout_round_kernel<ST, true, true, false>,
      fanout_round_kernel<ST, false, false, true>, fanout_round_kernel<ST, false, true, true>,
      fanout_round_kernel<ST, true, false, false, true>, fanout_round_kernel<ST, true, true, false, true>};
  for (auto k : ks) CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kFanoutMaxSmem));
  return CPBUS_OK;
}

int preload_round_kernels(cpbus* b) {
  static bool done[64] = {};
  static std::mutex mu;
  std::lock_guard<std::mutex> g(mu);
  if (done[b->device & 63]) return CPBUS_OK;
  int rc;
  if ((rc = preload_round_fanouts<CPBUS_STORE_V4>()) || (rc = preload_round_fanouts<CPBUS_STORE_V8>()) ||
      (rc = preload_round_fanouts<CPBUS_STORE_BULK>()))
    return rc;
  cudaFuncAttributes a;
  CK(cudaFuncGetAttributes(&a, stream_round_decide_kernel));
  CK(cudaFuncGetAttributes(&a, stream_round_admit_kernel));
  CK(cudaFuncGetAttributes(&a, stream_round_agree_kernel));
  CK(cudaFuncGetAttributes(&a, consume_all_kernel));     // cpbus_consume_all queues behind waiting rounds
  CK(cudaFuncGetAttributes(&a, digest_fold_kernel));     // as does cpbus_digest_fold_begin
  done[b->device & 63] = true;
  return CPBUS_OK;
}

// fan out `n` records at d_src with watermark w (all checks done by the caller)
struct StreamArgs {   // stream mode (cpbus_stream_fanout_prefix): where this batch's header / ack words live
  const StreamHdr* hdr = nullptr; unsigned long long* ack = nullptr; unsigned long long seq = 0;
  const StreamHdr* next_hdr = nullptr;
  uint32_t off = 0; bool final = true;   // records delivered before this launch; whether it completes the batch
  FollowRec* follow_rec = nullptr;       // follower launch (cpbus_stream_fanout_next): n and the watermark come from the header
  bool follow_from_host = false;         // ... and the previous watermark is the host clock rather than the clock words
  const RoundDev* round = nullptr;       // lossless round (cpbus_stream_round_next): m, the watermark and the source from the agree kernel
};

struct LaunchOpts {
  int staged = 0;                          // 1: the batch may live in a peer GPU's HBM; 2: a stream batch (`stream`)
  const cpbus_event* pf_src = nullptr;     // a later batch of pf_n records that this launch pulls into pf_dst
  cpbus_event* pf_dst = nullptr;
  uint32_t pf_n = 0;
  bool batch_dep = false;                  // the batch was written by the immediately preceding launch
  bool account = false;                    // the lead CTA accounts the batch (it did not pass through cpbus_publish)
  const StreamArgs* stream = nullptr;
};

int launch_fanout(cpbus* b, const cpbus_event* d_src, uint32_t n, uint64_t w, const LaunchOpts& o = {}) {
  const StreamArgs* sa = o.stream;
  if (b->n_next == 0 && !sa) return CPBUS_OK;
  if (n == 0 && b->n_timers == 0 && !sa) return CPBUS_OK;   // (a stream batch is always consumed: its slot must be acknowledged)
  FanoutParams p{};
  p.batch = d_src; p.ring = b->d_ring; p.ctl = b->d_ctl; p.timers = b->d_timers; p.stats = b->d_stats; p.pow_table = b->d_pow; p.launch_seq = ++b->launch_seq;
  p.desc = b->d_desc + (p.launch_seq & 1) * ((fanout_desc_bytes(2048) + 255) & ~(size_t)255);   // two descriptor buffers: launch i+1 may write while launch i reads
  p.desc_ready = b->d_desc_ready + (p.launch_seq & 1) * 16; p.w_now = w;
  p.result = b->d_result + (size_t)(p.launch_seq % kResultRing) * kResultSub;
  p.result_next = b->d_result + (size_t)((p.launch_seq + 1) % kResultRing) * kResultSub;
  p.batch_local = b->d_batch_local; p.staged = (uint32_t)o.staged;
  p.err_word = b->d_err; p.acct = o.account ? b->d_acct : nullptr;
  p.pf_state = b->d_pf_state; p.pf_buf = b->d_pf_buf; p.pf_stride = b->B; p.spin_us = b->stream_spin_us;
  if (sa) {
    p.stream_hdr = sa->hdr; p.stream_ack = sa->ack; p.stream_seq = sa->seq; p.stream_next_hdr = sa->next_hdr;
    p.stream_off = sa->off; p.stream_final = sa->final ? 1u : 0u;
  }
  const bool follow = sa && sa->follow_rec, round = sa && sa->round;
  const int kind = round ? kLaunchRound : follow ? kLaunchFollow : kLaunchPlain;
  p.round = round ? sa->round : nullptr;
  if (follow) {   // n = batch_cap sizes the launch; the kernel takes the batch's own n and watermark from the header
    p.follow_clock = b->d_follow_clock; p.follow_rec = sa->follow_rec; p.follow_window = max_window(b);
    p.follow_from_host = sa->follow_from_host ? 1u : 0u;
  }
  p.prefetch_src = o.pf_src; p.prefetch_dst = o.pf_dst; p.prefetch_n = o.pf_n;
  p.batch_dep = o.batch_dep ? 1u : 0u; p.n_ev = n;
  p.n_subs = b->n_next; p.ring_cap = b->R; p.K = b->K; p.sub_base = b->cfg.sub_id_base;
  p.use_digest = b->use_digest; p.lossless = b->lossless; p.timers_on = b->n_timers > 0 && b->K > 0;
  p.smem_cap = (n + 31u) & ~31u;
  // evict_last on control blocks / timer slots: they are re-read and re-written by every launch while the ring stream passes
  // through L2 once.  H100 (50 MB L2), 1,048,576 subscribers, 512-event batches, with the hint: config 5 (32 MiB of control
  // blocks, scattered by the mask order) 3.01 -> 2.90 ms per launch, config 3 (64 MiB with the timer slots) 6.41 -> 6.34 ms.
  // Kept up to 64 MiB of hot state, the largest footprint measured.
  const size_t hot_bytes = (size_t)b->n_next * (sizeof(SubCtl) + (p.timers_on ? b->K * sizeof(DevTimer) : 0));
  p.hints = b->hints >= 0 ? (uint32_t)b->hints : (hot_bytes <= (64u << 20) ? 1u : 0u);
  const uint32_t need = (b->n_next + kWarpsPerCta - 1) / kWarpsPerCta;
  uint32_t grid = b->cfg.grid_ctas ? std::max(1u, std::min(b->cfg.grid_ctas, need)) : 0u;
  int rc;
  // ORDERED build (no timers armed, at least one filtered subscriber): walk the mailboxes in code-mask order so that
  // equal masks are neighbours and share one filter pass (cost ~ deliveries + distinct masks, not subscribers x events)
  // PAIRS build (some subscriber has exact {code, source} cases): the timers build with the second-level test in its
  // general path; subscribers without a pair table take the same paths as before
  const bool pairs_on = b->n_paired > 0 && b->d_pairs;
  p.pairs = pairs_on ? b->d_pairs : nullptr;
  size_t smem = fanout_smem_bytes(p.smem_cap) + (pairs_on ? kPairFilterBytes : 0);   // + the batch's {code, source} presence filter
  if (!pairs_on && !p.timers_on && b->n_filtered > 0) {
    if (b->order_dirty) { const int rc_order = rebuild_order(b); if (rc_order) return rc_order; }
    if (b->n_order) {
      const uint32_t scale = std::max(1u, (p.n_ev + 128u) / 256u);
      // 512-event batches: 8 mailboxes per warp from 524,288 subscribers up, fewer for short launches (more, shorter CTAs)
      uint32_t spw = b->subs_per_warp ? std::min(32u, b->subs_per_warp)
                                      : std::max(4u, std::min(16u / scale, b->n_order / (20480u * scale)));
      p.order = b->d_order; p.n_order = b->n_order; p.spw = spw;
      const uint32_t warps = (b->n_order + spw - 1) / spw;
      grid = std::max(1u, (warps + kWarpsPerCta - 1) / kWarpsPerCta);
    }
  }
  if (pairs_on && !b->cfg.grid_ctas) {   // PAIRS build: lane-parallel triage over blocks of 32 mailboxes per warp turn
    const uint32_t blocks = (b->n_next + 31u) / 32u;
    grid = std::max(1u, std::min((blocks + kWarpsPerCta - 1) / kWarpsPerCta, (uint32_t)b->sm_count * 16u));
  }
  if (!pairs_on && !p.order) {
    // Plain build: CTA b owns subscribers [8 spw b, 8 spw (b + 1)).  Several waves of short-lived CTAs rather than one
    // persistent wave: the hardware CTA scheduler balances the SM speed spread for free.  Per-CTA setup here is a
    // descriptor copy + TMA wait, so the grid aims at 2-16 mailboxes per warp, scaled with the SM count.
    // (need == 0: a stream batch on a bus without subscribers still takes one CTA, which acknowledges it)
    uint32_t spw = b->subs_per_warp;
    if (grid) spw = std::max(1u, (need + grid - 1) / grid);   // a fixed grid: ranges cover every subscriber
    else if (!spw) {
      // ~constant bytes per warp: the counts above are for 256-event batches; a 512-event batch halves them
      const uint32_t scale = std::max(1u, (p.n_ev + 128u) / 256u);
      const uint32_t cap = std::max(1u, 16u / scale);
      spw = std::max(1u, std::min(cap, (need + (uint32_t)b->sm_count * 7 * scale) / ((uint32_t)b->sm_count * 14 * scale)));
    }
    p.spw = spw;
    grid = std::max(1u, (need + spw - 1) / spw);
    // The range's control blocks (and timer slots) are staged in shared memory stage_subs at a time, in what the batch
    // leaves of the shared memory at the residency that the batch plus the smallest round (one subscriber per warp)
    // allows, at most kCtasPerSm CTAs per SM.  Staging can therefore cost a resident CTA only where the batch
    // leaves less than that smallest round.
    const size_t off = fanout_stage_off(p.smem_cap);
    const size_t per_sub = sizeof(SubCtl) + (p.timers_on ? (size_t)b->K * sizeof(DevTimer) : 0);
    const size_t min_round = (size_t)kWarpsPerCta * per_sub;
    const size_t ctas = std::max<size_t>(1, std::min<size_t>(kCtasPerSm, b->smem_per_sm / (off + min_round + b->smem_reserved)));
    const size_t room = std::min<size_t>(kFanoutMaxSmem, b->smem_per_sm / ctas - b->smem_reserved) - off;   // >= min_round
    p.stage_subs = std::max<uint32_t>(kWarpsPerCta, (uint32_t)std::min<size_t>((size_t)kWarpsPerCta * spw, room / per_sub) & ~7u);
    smem = off + p.stage_subs * per_sub;
  }
  const int variant = pairs_on ? (p.use_digest ? 7 : 6) : (p.timers_on ? 2 : 0) | (p.use_digest ? 1 : 0) | (p.order ? 4 : 0);
#define CPBUS_DISPATCH(ST)                                                                \
  switch (variant) {                                                                     \
    case 0: rc = launch_fanout_t<ST, false, false, false>(b, p, grid, smem, kind); break;      \
    case 1: rc = launch_fanout_t<ST, false, true, false>(b, p, grid, smem, kind); break;       \
    case 2: rc = launch_fanout_t<ST, true, false, false>(b, p, grid, smem, kind); break;       \
    case 3: rc = launch_fanout_t<ST, true, true, false>(b, p, grid, smem, kind); break;        \
    case 4: rc = launch_fanout_t<ST, false, false, true>(b, p, grid, smem, kind); break;       \
    case 5: rc = launch_fanout_t<ST, false, true, true>(b, p, grid, smem, kind); break;        \
    case 6: rc = launch_fanout_t<ST, true, false, false, true>(b, p, grid, smem, kind); break; \
    default: rc = launch_fanout_t<ST, true, true, false, true>(b, p, grid, smem, kind); break; \
  }
  switch (b->store) {
    case CPBUS_STORE_V4: CPBUS_DISPATCH(CPBUS_STORE_V4); break;
    case CPBUS_STORE_BULK: CPBUS_DISPATCH(CPBUS_STORE_BULK); break;
    default: CPBUS_DISPATCH(CPBUS_STORE_V8); break;
  }
#undef CPBUS_DISPATCH
  if (rc) return rc;
  b->st.kernel_launches++;
  if (!round) b->st.batches++;   // (a round's batch counts when it is resolved, if it delivered)
  if (sa) return CPBUS_OK;       // (the caller folds a stream launch in once its outcome is known: stream_delivered)
  b->last_watermark = w;
  if (o.account && n) dbg_mark_device_batch(b, p.launch_seq);
  return CPBUS_OK;
}

// lossless admission (reference: the sender blocks on a full channel, events/subscriber.go:30-32)
// Fast path: true when n records with watermark w provably fit (or nothing has to be admitted) — no kernel, no sync.
bool admit_fits(cpbus* b, uint32_t n, uint64_t w) {
  if (!b->lossless || b->n_next == 0) return true;
  const uint64_t need = admit_need(n, w, b->last_watermark, b->min_period, b->K, b->n_timers && b->K);
  if (b->room_lb >= need) { b->room_lb -= need; b->st.admit_skipped++; return true; }
  return false;
}

// The admission pass (after admit_fits said no): one kernel over every mailbox of the shard, then a host sync.
int admit_pass(cpbus* b, const cpbus_event* d_src, uint32_t n, uint64_t w, bool* ok, uint32_t* prefix) {
  CK(cudaMemsetAsync(&b->d_stats->admit_overflow, 0, 4 * sizeof(unsigned long long), b->stream));   // overflow, overwritten, max_used, deficit
  const uint32_t threads = 256, grid = (b->n_next + threads - 1) / threads;
  admit_kernel<<<grid, threads, 0, b->stream>>>(d_src, n, w, b->d_ctl, b->d_timers, b->n_next, b->R, b->K,
                                                b->cfg.sub_id_base, b->n_timers > 0 && b->K > 0, b->d_stats,
                                                b->n_paired > 0 ? b->d_pairs : nullptr);
  CK(cudaGetLastError());
  b->st.kernel_launches++; b->st.admit_passes++;
  CK(cudaMemcpyAsync(&b->h_stats->admit_overflow, &b->d_stats->admit_overflow, 4 * sizeof(unsigned long long),
                     cudaMemcpyDeviceToHost, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  *ok = b->h_stats->admit_overflow == 0;
  if (!*ok && prefix) *prefix = n - (uint32_t)std::min<unsigned long long>(n, b->h_stats->admit_deficit);   // events every mailbox can still take
  const uint64_t used = b->h_stats->admit_max_used;            // fullest mailbox, this batch included
  // admitted: the batch is in; refused: nothing was appended, so the fullest mailbox holds at most `used` minus its share (>= 0):
  // keep the conservative figure either way
  b->room_lb = used >= b->R ? 0 : b->R - used;
  return CPBUS_OK;
}

int admit(cpbus* b, const cpbus_event* d_src, uint32_t n, uint64_t w, bool* ok, uint32_t* prefix = nullptr) {
  *ok = true;
  if (prefix) *prefix = n;
  if (admit_fits(b, n, w)) return CPBUS_OK;
  return admit_pass(b, d_src, n, w, ok, prefix);
}

// host mirror of one-shot timers that have fired on the device (events/timer.go:19-33):
// a one-shot whose due time is <= the last launched watermark has disarmed itself.
void retire_oneshots(cpbus* b, uint64_t w) {
  size_t keep = 0;
  for (size_t i = 0; i < b->oneshot_idx.size(); i++) {
    HostTimer& t = b->h_timers[b->oneshot_idx[i]];
    if (t.active && t.oneshot && oneshot_fired(t.next_due, w)) { t.active = false; b->n_timers--; continue; }
    if (t.active && t.oneshot) b->oneshot_idx[keep++] = b->oneshot_idx[i];
  }
  b->oneshot_idx.resize(keep);
  if (b->n_timers == 0) b->min_period = UINT64_MAX;
}

int flush_staged(cpbus* b, uint64_t w) {
  const uint32_t n = (uint32_t)b->n_staged;
  if (n == 0 && b->n_timers == 0) { b->last_watermark = std::max(b->last_watermark, w); return CPBUS_OK; }   // nothing armed: the watermark follows the clock
  if (n == 0 && w == b->last_watermark) return CPBUS_OK;
  const int c = b->cur;
  int rc;
  // Device staging is a long ring (kDevSlots batches): a slot is reused only kDevSlots flushes later, far beyond how far the
  // host can run ahead, so the H2D never has to wait for an old fan-out and lands within microseconds.  Reuse safety is a
  // host-side check once per epoch of kDevEpoch slots (almost always already satisfied).
  const uint32_t slot = b->dev_slot;
  cpbus_event* d_dst = b->d_stage + (size_t)slot * b->B;
  if (slot % cpbus::kDevEpoch == 0) CK(cudaEventSynchronize(b->epoch_done[slot / cpbus::kDevEpoch]));   // last round's users of this epoch are done
  if (n) {
    CK(cudaMemcpyAsync(d_dst, b->h_batch[c], (size_t)n * sizeof(cpbus_event), cudaMemcpyHostToDevice, b->copy_stream));
    CK(cudaEventRecord(b->h2d_done[c], b->copy_stream));
    // Give the 8-16 KiB copy up to 30 us to land.  If it has, the bus stream needs no wait node, consecutive fan-outs
    // stay adjacent in the stream and the next launch's prologue overlaps this one's tail (programmatic dependent launch).
    bool landed = false;
    const auto t_spin = std::chrono::steady_clock::now();
    do {
      const cudaError_t q = cudaEventQuery(b->h2d_done[c]);
      if (q == cudaSuccess) { landed = true; break; }
      if (q != cudaErrorNotReady) { CK(q); }
    } while (std::chrono::steady_clock::now() - t_spin < std::chrono::microseconds(30));
    if (!landed) CK(cudaStreamWaitEvent(b->stream, b->h2d_done[c], 0));
  }
  bool ok = true;
  uint32_t m = n;
  rc = admit(b, d_dst, n, w, &ok, &m);
  if (rc) return rc;
  if (!ok) {
    // Some mailbox lacks the room.  Like the Go bus, which blocks at the first event a full channel cannot take
    // (events/subscriber.go:30-32), deliver the longest prefix EVERY mailbox can take — with the ticks due by its last
    // event — keep the rest staged and report the stall; the caller lets the consumers run and flushes again.
    if (m == 0) return CPBUS_EAGAIN;
    const uint64_t w_part = b->h_batch[c][m - 1].ts_ns;
    rc = launch_fanout(b, d_dst, m, w_part);
    if (rc) return rc;
    if (slot % cpbus::kDevEpoch == cpbus::kDevEpoch - 1) CK(cudaEventRecord(b->epoch_done[slot / cpbus::kDevEpoch], b->stream));
    b->dev_slot = (slot + 1) % cpbus::kDevSlots;
    memmove(b->h_batch[c], b->h_batch[c] + m, (size_t)(n - m) * sizeof(cpbus_event));   // (the H2D of this buffer completed before the admission pass)
    b->n_staged = n - m;
    b->room_lb = 0;
    b->st.admit_partial++;
    return CPBUS_EAGAIN;
  }
  rc = launch_fanout(b, d_dst, n, w);
  if (rc) return rc;
  if (slot % cpbus::kDevEpoch == cpbus::kDevEpoch - 1) CK(cudaEventRecord(b->epoch_done[slot / cpbus::kDevEpoch], b->stream));
  b->dev_slot = (slot + 1) % cpbus::kDevSlots;
  b->n_staged = 0;
  b->cur = (b->cur + 1) % cpbus::kStage;
  CK(cudaEventSynchronize(b->h2d_done[b->cur]));   // the pinned buffer we are about to overwrite has left the host
  return CPBUS_OK;
}

uint64_t max_window(const cpbus* b) {
  if (!b->K || b->n_timers == 0 || b->min_period == UINT64_MAX) return UINT64_MAX;
  const uint64_t J = 32u / b->K;
  return b->min_period > UINT64_MAX / J ? UINT64_MAX : b->min_period * J;
}

int stage_one(cpbus* b, uint32_t code, uint32_t source_id, uint32_t target, uint32_t flags) {
  if (b->n_staged == b->B) { int rc = flush_staged(b, b->now); if (rc) return rc; }
  cpbus_event& e = b->h_batch[b->cur][b->n_staged++];
  e.seq = b->seq++; e.ts_ns = b->now; e.code = code; e.source_id = source_id; e.target = target; e.flags = flags;
  return CPBUS_OK;
}

bool is_pow2(uint32_t x) { return x && !(x & (x - 1)); }

}  // namespace

// outstanding followers and rounds that hold one of the kFollowMax records
static int follow_records(const cpbus* b) {
  int n = 0;
  for (const cpbus::FollowPending& f : b->follow_q) n += f.kind != cpbus::kConsumeAll ? 1 : 0;
  return n;
}

extern "C" {
static int follow_resolve(cpbus* b);
// The opening of the entry points that read or change host-side bus state: this bus's device, then the outstanding
// followers and rounds folded in (DESIGN.md §8, lazy resolution).
static int enter(cpbus* b) {
  const int rc = dev_guard(b);
  return rc ? rc : follow_resolve(b);
}
// Nothing may unwind through the C boundary (cgo, ctypes): every status-returning entry point is a function-try-block.
#define CPBUS_CATCH                                                                                   \
  catch (const std::bad_alloc&) { return CPBUS_ENOMEM; }                                              \
  catch (...) { snprintf(g_cuda_err, sizeof(g_cuda_err), "unexpected C++ exception"); return CPBUS_ECUDA; }

uint32_t cpbus_abi_version(void) { return 2; }
static int split_plan(const uint64_t* ts, size_t n, uint32_t batch_cap, uint64_t now, uint64_t watermark, uint64_t window,
                      std::vector<size_t>& end, std::vector<uint64_t>& wm);
int cpbus_split_plan(const uint64_t* ts, size_t n, uint32_t batch_cap, uint64_t now_ns, uint64_t watermark_ns, uint64_t window_ns,
                     size_t* ends, uint64_t* watermarks, size_t cap, size_t* n_slices) try {
  if ((!ts && n) || !n_slices || (cap && (!ends || !watermarks))) return CPBUS_EINVAL;
  std::vector<size_t> end; std::vector<uint64_t> wm;
  const int rc = split_plan(ts, n, batch_cap, now_ns, watermark_ns, window_ns, end, wm);
  if (rc) return rc;
  *n_slices = end.size();
  for (size_t k = 0; k < end.size() && k < cap; k++) { ends[k] = end[k]; watermarks[k] = wm[k]; }
  return CPBUS_OK;
} CPBUS_CATCH
size_t cpbus_mask_order(const uint32_t* masks, const uint8_t* active, uint32_t n, uint32_t ring_cap, uint32_t block, int heavy_first, uint32_t* out) {
  if (!masks || !out || !ring_cap) return 0;
  try {
    std::vector<uint32_t> order;
    mask_order(masks, active, n, ring_cap, block, heavy_first != 0, order);
    std::copy(order.begin(), order.end(), out);
    return order.size();
  } catch (const std::bad_alloc&) { return 0; }
}

const char* cpbus_last_cuda_error(void) { return g_cuda_err; }

const char* cpbus_strerror(int s) {
  switch (s) {
    case CPBUS_OK: return "ok";
    case CPBUS_EINVAL: return "invalid argument";
    case CPBUS_ENOMEM: return "out of memory";
    case CPBUS_ECUDA: return "CUDA error";
    case CPBUS_EAGAIN: return "mailbox full (lossless mode): drain and retry";
    case CPBUS_ENOSPC: return "capacity exhausted";
    case CPBUS_ENOENT: return "no such subscriber or timer";
    case CPBUS_ECLOSED: return "subscriber already unsubscribed";
    case CPBUS_ENODEV: return "no CUDA device (libcpbus has no CPU fallback)";
    case CPBUS_EORDER: return "clock moved backwards, batch unsorted or timer window exceeded";
    case CPBUS_ETIMEDOUT: return "stream batch never arrived (publisher stalled or consumer a whole ring behind)";
    default: return "unknown status";
  }
}

// EventCode.String — events/eventcode_string.go:5-15
const char* cpbus_code_name(int code) {
  static const char* const names[CPBUS_N_CODES] = {
      "None", "ExitSuccess", "ExitFailed", "Stopping", "Stopped", "StatusHealthy", "StatusUnhealthy", "StatusChanged",
      "TimerExpired", "EnterMaintenance", "ExitMaintenance", "Error", "Quit", "Metric", "Startup", "Shutdown", "Signal"};
  return (code < 0 || code >= CPBUS_N_CODES) ? nullptr : names[code];
}

// FromString — events/events.go:52-86
int cpbus_code_from_string(const char* name) try {
  if (!name) return -1;
  static const std::unordered_map<std::string, int> table = {
      {"exitSuccess", CPBUS_EXIT_SUCCESS}, {"exitFailed", CPBUS_EXIT_FAILED}, {"stopping", CPBUS_STOPPING},
      {"stopped", CPBUS_STOPPED}, {"healthy", CPBUS_STATUS_HEALTHY}, {"unhealthy", CPBUS_STATUS_UNHEALTHY},
      {"changed", CPBUS_STATUS_CHANGED}, {"timerExpired", CPBUS_TIMER_EXPIRED},
      {"enterMaintenance", CPBUS_ENTER_MAINTENANCE}, {"exitMaintenance", CPBUS_EXIT_MAINTENANCE},
      {"error", CPBUS_ERROR}, {"quit", CPBUS_QUIT}, {"startup", CPBUS_STARTUP}, {"shutdown", CPBUS_SHUTDOWN},
      {"SIGHUP", CPBUS_SIGNAL}, {"SIGUSR2", CPBUS_SIGNAL}};
  auto it = table.find(name);
  return it == table.end() ? -1 : it->second;
} CPBUS_CATCH

uint64_t cpbus_record_hash(const cpbus_event* e) {
  return record_hash_words(e->seq, e->ts_ns, (uint64_t)e->code | ((uint64_t)e->source_id << 32),
                           (uint64_t)e->target | ((uint64_t)e->flags << 32));
}
uint64_t cpbus_digest_multiplier(void) { return kDigestP; }

// The checks cpbus_create makes of a config (cpbus_group_create makes them of the total); R and B get the defaults applied.
static int config_check(const cpbus_config* cfg, uint32_t* R_out, uint32_t* B_out) {
  const uint32_t R = cfg->ring_cap ? cfg->ring_cap : 1024;
  const uint32_t B = cfg->batch_cap ? cfg->batch_cap : std::min(256u, R / 2);
  const uint32_t K = cfg->timers_per_sub;
  if (!cfg->n_max_subs || !is_pow2(R) || R < 64 || B == 0 || B > R / 2 || (B % 32) != 0 || B > 1024) return CPBUS_EINVAL;   // 1024: the kernel keeps one match word per 32-event chunk in a lane
  if (!(K == 0 || K == 1 || K == 2 || K == 4 || K == 8)) return CPBUS_EINVAL;
  if ((uint64_t)cfg->n_max_subs * std::max(K, 1u) > kTimerSlotMask) return CPBUS_EINVAL;   // timer ids keep 6 generation bits
  if (cfg->store_path > CPBUS_STORE_BULK) return CPBUS_EINVAL;
  if ((uint64_t)cfg->sub_id_base + cfg->n_max_subs > CPBUS_TARGET_ALL) return CPBUS_EINVAL;   // every gid stays below CPBUS_TARGET_ALL
  *R_out = R; *B_out = B;
  return CPBUS_OK;
}

int cpbus_create(const cpbus_config* cfg, cpbus_t** out) try {
  if (!cfg || !out) return CPBUS_EINVAL;
  *out = nullptr;
  uint32_t R = 0, B = 0;
  if (config_check(cfg, &R, &B)) return CPBUS_EINVAL;
  const uint32_t K = cfg->timers_per_sub;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    snprintf(g_cuda_err, sizeof(g_cuda_err), "no CUDA device visible");
    return CPBUS_ENODEV;
  }
  cpbus* b = new (std::nothrow) cpbus();
  if (!b) return CPBUS_ENOMEM;
  b->cfg = *cfg; b->cfg.ring_cap = R; b->cfg.batch_cap = B;
  b->N = cfg->n_max_subs; b->R = R; b->B = B; b->K = K;
  b->lossless = cfg->flags & CPBUS_CFG_LOSSLESS; b->use_digest = cfg->flags & CPBUS_CFG_DIGEST;
  b->room_lb = R;
  b->store = cfg->store_path == CPBUS_STORE_AUTO ? CPBUS_STORE_V8 : (int)cfg->store_path;
  if (const char* e = getenv("CPBUS_PDL")) b->pdl = atoi(e) != 0;
  if (const char* e = getenv("CPBUS_HINTS")) b->hints = atoi(e);
  if (const char* e = getenv("CPBUS_SUBS_PER_WARP")) b->subs_per_warp = (uint32_t)atoi(e);   // tuning knob for experiments
  if (const char* e = getenv("CPBUS_ORDER_BLOCK")) b->order_block = (uint32_t)atoll(e);
  int rc = CPBUS_OK;
  auto fail = [&](int code) { cpbus_destroy(b); return code; };
  if (cfg->device >= 0) b->device = cfg->device;
  else if (cudaGetDevice(&b->device) != cudaSuccess) return fail(CPBUS_ECUDA);
  if (b->device >= ndev) return fail(CPBUS_EINVAL);
  if ((rc = dev_guard(b))) return fail(rc);
  cudaDeviceProp prop{};
  if (cudaGetDeviceProperties(&prop, b->device) == cudaSuccess) {
    b->sm_count = prop.multiProcessorCount;
    b->smem_per_sm = prop.sharedMemPerMultiprocessor; b->smem_reserved = prop.reservedSharedMemPerBlock;
  }
  if (cfg->stream) b->stream = (cudaStream_t)cfg->stream;
  else {
    if (cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking) != cudaSuccess) return fail(CPBUS_ECUDA);
    b->own_stream = true;
  }
  const size_t N = b->N;
#define ALLOC(ptr, bytes)                                                                     \
  if (cudaMalloc((void**)&(ptr), (bytes)) != cudaSuccess) {                                   \
    snprintf(g_cuda_err, sizeof(g_cuda_err), "cudaMalloc(%zu) failed", (size_t)(bytes));     \
    return fail(CPBUS_ENOMEM);                                                                \
  }
  ALLOC(b->d_ring, N * R * sizeof(cpbus_event));
  ALLOC(b->d_ctl, N * sizeof(SubCtl)); ALLOC(b->d_order, N * 4);
  if (K) ALLOC(b->d_timers, N * K * sizeof(DevTimer));
  ALLOC(b->d_stats, sizeof(DevStats)); ALLOC(b->d_fold, 32 * cpbus::kFoldSlots); ALLOC(b->d_pow, kPowTableLen * 8);
  ALLOC(b->d_desc, 2 * ((fanout_desc_bytes(2048) + 255) & ~(size_t)255)); ALLOC(b->d_desc_ready, 256);
  if (cudaMemsetAsync(b->d_desc_ready, 0, 256, b->stream) != cudaSuccess) return fail(CPBUS_ECUDA);
  if (cudaStreamCreateWithFlags(&b->copy_stream, cudaStreamNonBlocking) != cudaSuccess) return fail(CPBUS_ECUDA);
  if (cudaStreamCreateWithFlags(&b->result_stream, cudaStreamNonBlocking) != cudaSuccess) return fail(CPBUS_ECUDA);
  if (cudaEventCreateWithFlags(&b->launched, cudaEventDisableTiming) != cudaSuccess) return fail(CPBUS_ECUDA);
  ALLOC(b->d_stage, (size_t)cpbus::kDevSlots * B * sizeof(cpbus_event));
  for (int i = 0; i < cpbus::kDevSlots / cpbus::kDevEpoch; i++)
    if (cudaEventCreateWithFlags(&b->epoch_done[i], cudaEventDisableTiming) != cudaSuccess) return fail(CPBUS_ECUDA);
  for (int i = 0; i < cpbus::kStage; i++) {
    if (cudaMallocHost((void**)&b->h_batch[i], (size_t)B * sizeof(cpbus_event)) != cudaSuccess) return fail(CPBUS_ENOMEM);
    if (cudaEventCreateWithFlags(&b->h2d_done[i], cudaEventDisableTiming) != cudaSuccess) return fail(CPBUS_ECUDA);
  }
  ALLOC(b->d_batch_local, (size_t)B * sizeof(cpbus_event));
  if (b->lossless) {
    ALLOC(b->d_admit_batch, (size_t)B * sizeof(cpbus_event));
    // lossless rounds (cpbus_stream_round_next): device state and the host records, allocated here rather than by the
    // first round, while no round of any shard can be waiting on the device
    ALLOC(b->d_round, sizeof(RoundDev));
    RoundDev init{};
    init.room_full = R;
    if (cudaMemcpyAsync(b->d_round, &init, sizeof(init), cudaMemcpyHostToDevice, b->stream) != cudaSuccess) return fail(CPBUS_ECUDA);
    if (mapped_alloc(sizeof(RoundRec) * cpbus::kFollowMax, &b->h_round, &b->d_round_rec) != cudaSuccess) return fail(CPBUS_ENOMEM);
    if ((rc = preload_round_kernels(b))) return fail(rc);
  } else {   // followers (cpbus_stream_fanout_next): their records and the clock words, zeroed
    if (mapped_alloc(sizeof(FollowRec) * cpbus::kFollowMax, &b->h_follow, &b->d_follow) != cudaSuccess) return fail(CPBUS_ENOMEM);
    ALLOC(b->d_follow_clock, 4 * sizeof(unsigned long long));
    if (cudaMemsetAsync(b->d_follow_clock, 0, 4 * sizeof(unsigned long long), b->stream) != cudaSuccess) return fail(CPBUS_ECUDA);
  }
  if (cudaEventCreateWithFlags(&b->follow_done, cudaEventDisableTiming) != cudaSuccess) return fail(CPBUS_ECUDA);
  ALLOC(b->d_pf_buf, (size_t)kStreamPrefetch * B * sizeof(cpbus_event)); ALLOC(b->d_pf_state, 64);
  ALLOC(b->d_acct, sizeof(DevPubAcct));
  if (cudaMemsetAsync(b->d_pf_state, 0, 64, b->stream) != cudaSuccess ||
      cudaMemsetAsync(b->d_acct, 0, sizeof(DevPubAcct), b->stream) != cudaSuccess) return fail(CPBUS_ECUDA);
  if (mapped_alloc(64, &b->h_err, &b->d_err) != cudaSuccess) return fail(CPBUS_ENOMEM);
  memset(b->h_err, 0, 64);
  if (cudaMallocHost((void**)&b->h_acct, offsetof(DevPubAcct, pair_key)) != cudaSuccess) return fail(CPBUS_ENOMEM);
  for (int i = 0; i < cpbus::kPrefetch; i++) ALLOC(b->d_prefetch[i], (size_t)B * sizeof(cpbus_event));
  ALLOC(b->d_result, sizeof(DevResultSlot) * kResultRing * kResultSub);
  if (cudaMemsetAsync(b->d_result, 0, sizeof(DevResultSlot) * kResultRing * kResultSub, b->stream) != cudaSuccess) return fail(CPBUS_ECUDA);
  if (cudaMallocHost((void**)&b->h_result, sizeof(DevResultSlot) * 8 * kResultSub) != cudaSuccess) return fail(CPBUS_ENOMEM);
  for (int i = 0; i < 8; i++)
    if (cudaEventCreateWithFlags(&b->result_done[i], cudaEventDisableTiming) != cudaSuccess) return fail(CPBUS_ECUDA);
#undef ALLOC
  if (cudaMallocHost((void**)&b->h_stats, sizeof(DevStats)) != cudaSuccess) return fail(CPBUS_ENOMEM);
  if (cudaMallocHost((void**)&b->h_fold, 32 * cpbus::kFoldSlots) != cudaSuccess) return fail(CPBUS_ENOMEM);
  for (int i = 0; i < cpbus::kFoldSlots; i++)
    if (cudaEventCreateWithFlags(&b->fold_done[i], cudaEventDisableTiming) != cudaSuccess) return fail(CPBUS_ECUDA);
  // rings are NOT cleared: a slot is only ever read after it has been written (head/tail bound every read)
  bool ok = cudaMemsetAsync(b->d_ctl, 0, N * sizeof(SubCtl), b->stream) == cudaSuccess &&
            cudaMemsetAsync(b->d_stats, 0, sizeof(DevStats), b->stream) == cudaSuccess &&
            (!K || cudaMemsetAsync(b->d_timers, 0xFF, N * K * sizeof(DevTimer), b->stream) == cudaSuccess) &&   // every slot idle
            cudaStreamSynchronize(b->stream) == cudaSuccess;
  if (!ok) return fail(CPBUS_ECUDA);
  {
    std::vector<uint64_t> pw(kPowTableLen);
    uint64_t x = 1;
    for (uint32_t i = 0; i < kPowTableLen; i++) { pw[i] = x; x *= kDigestP; }
    if (cudaMemcpyAsync(b->d_pow, pw.data(), kPowTableLen * 8, cudaMemcpyHostToDevice, b->stream) != cudaSuccess ||
        cudaStreamSynchronize(b->stream) != cudaSuccess) return fail(CPBUS_ECUDA);
  }
  b->h_mask.assign(N, 0);
  b->h_active.assign(N, 0);
  b->intern.emplace(std::string(), 0u);   // "" -> 0 so that NonEvent == {None, 0} (events/events.go:45)
  b->sources.emplace_back();
  *out = b;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_destroy(cpbus_t* b) try {
  if (!b) return CPBUS_EINVAL;
  follow_resolve(b);
  cudaSetDevice(b->device);
  if (b->stream) cudaStreamSynchronize(b->stream);
  while (!b->streams.empty()) cpbus_stream_close(b->streams.back());
  if (b->h_follow) cudaFreeHost(b->h_follow);
  cudaFree(b->d_follow_clock);
  if (b->h_round) cudaFreeHost(b->h_round);
  cudaFree(b->d_round);
  if (b->follow_done) cudaEventDestroy(b->follow_done);
  cudaFree(b->d_ring); cudaFree(b->d_ctl); cudaFree(b->d_order); cudaFree(b->d_pairs);
  cudaFree(b->d_timers); cudaFree(b->d_stats); cudaFree(b->d_fold); cudaFree(b->d_pow); cudaFree(b->d_desc); cudaFree(b->d_desc_ready);
  if (b->copy_stream) cudaStreamSynchronize(b->copy_stream);
  if (b->result_stream) { cudaStreamSynchronize(b->result_stream); cudaStreamDestroy(b->result_stream); }
  for (int i = 0; i < cpbus::kStage; i++) {
    if (b->h_batch[i]) cudaFreeHost(b->h_batch[i]);
    if (b->h2d_done[i]) cudaEventDestroy(b->h2d_done[i]);
  }
  cudaFree(b->d_stage);
  for (int i = 0; i < cpbus::kDevSlots / cpbus::kDevEpoch; i++) if (b->epoch_done[i]) cudaEventDestroy(b->epoch_done[i]);
  if (b->copy_stream) cudaStreamDestroy(b->copy_stream);
  if (b->launched) cudaEventDestroy(b->launched);
  cudaFree(b->d_drain); cudaFree(b->d_drain_idx);
  cudaFree(b->d_ready_lb); cudaFree(b->d_ready); cudaFree(b->d_ready_slot);
  if (b->h_ready_hdr) cudaFreeHost(b->h_ready_hdr);
  cudaFree(b->d_result); cudaFree(b->d_batch_local); cudaFree(b->d_admit_batch); cudaFree(b->d_pf_buf); cudaFree(b->d_pf_state); cudaFree(b->d_acct);
  if (b->h_err) cudaFreeHost(b->h_err);
  if (b->h_acct) cudaFreeHost(b->h_acct);
  for (int i = 0; i < cpbus::kPrefetch; i++) cudaFree(b->d_prefetch[i]);
  for (void* p : b->shared_mapped) cudaIpcCloseMemHandle(p);
  for (void* p : b->shared_owned) cudaFree(p);
  if (b->h_result) cudaFreeHost(b->h_result);
  for (int i = 0; i < 8; i++) if (b->result_done[i]) cudaEventDestroy(b->result_done[i]);
  if (b->h_stats) cudaFreeHost(b->h_stats);
  if (b->h_fold) cudaFreeHost(b->h_fold);
  for (int i = 0; i < cpbus::kFoldSlots; i++) if (b->fold_done[i]) cudaEventDestroy(b->fold_done[i]);
  if (b->own_stream && b->stream) cudaStreamDestroy(b->stream);
  delete b;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_intern(cpbus_t* b, const char* s, size_t len, uint32_t* source_id) try {
  if (!b || (!s && len) || !source_id) return CPBUS_EINVAL;
  std::string key(s ? s : "", len);
  auto it = b->intern.find(key);
  if (it != b->intern.end()) { *source_id = it->second; return CPBUS_OK; }
  if (b->sources.size() >= 0xFFFFFFF0u) return CPBUS_ENOSPC;
  if (b->sources.size() >= CPBUS_EPHEMERAL_BIT) return CPBUS_ENOSPC;   // permanent ids never carry the ephemeral bit
  const uint32_t id = (uint32_t)b->sources.size();
  b->sources.push_back(key);
  b->intern_bytes += key.size();
  b->intern.emplace(std::move(key), id);
  *source_id = id;
  return CPBUS_OK;
} CPBUS_CATCH

// Bounded region for payload strings (control/endpoints.go:125-126: Source = "key|value" of every posted metric).
// id = EPHEMERAL_BIT | generation(15) << 16 | slot(16); the slot's previous string is dropped when it is reused.
int cpbus_intern_ephemeral(cpbus_t* b, const char* s, size_t len, uint32_t* source_id) try {
  if (!b || (!s && len) || !source_id) return CPBUS_EINVAL;
  std::string key(s ? s : "", len);
  auto perm = b->intern.find(key);
  if (perm != b->intern.end()) { *source_id = perm->second; return CPBUS_OK; }   // already a name: keep one id per string
  auto it = b->eph_map.find(key);
  if (it != b->eph_map.end()) {
    const cpbus::EphSlot& e = b->eph[it->second];
    *source_id = CPBUS_EPHEMERAL_BIT | ((e.gen & 0x7FFFu) << 16) | it->second;
    return CPBUS_OK;
  }
  if (b->eph.empty()) b->eph.resize(CPBUS_EPHEMERAL_SLOTS);
  const uint32_t slot = b->eph_next;
  b->eph_next = (slot + 1) % CPBUS_EPHEMERAL_SLOTS;
  cpbus::EphSlot& e = b->eph[slot];
  if (e.live) { b->eph_map.erase(e.s); b->eph_recycled++; } else b->eph_live++;
  e.gen++; e.live = true; e.s = key;
  b->eph_map.emplace(std::move(key), slot);
  *source_id = CPBUS_EPHEMERAL_BIT | ((e.gen & 0x7FFFu) << 16) | slot;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_source(cpbus_t* b, uint32_t id, char* out, size_t cap, size_t* len) try {
  if (!b) return CPBUS_EINVAL;
  if (id & CPBUS_EPHEMERAL_BIT) {
    const uint32_t slot = id & 0xFFFFu, gen = (id >> 16) & 0x7FFFu;
    if (slot >= b->eph.size() || !b->eph[slot].live || (b->eph[slot].gen & 0x7FFFu) != gen) return CPBUS_ENOENT;   // recycled
    const std::string& s = b->eph[slot].s;
    if (len) *len = s.size();
    if (out && cap) memcpy(out, s.data(), std::min(cap, s.size()));
    return CPBUS_OK;
  }
  if (id >= b->sources.size()) return CPBUS_ENOENT;
  const std::string& s = b->sources[id];
  if (len) *len = s.size();
  if (out && cap) memcpy(out, s.data(), std::min(cap, s.size()));
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_subscribe_many(cpbus_t* b, const uint32_t* masks, uint32_t n, uint32_t* first_sub_id) try {
  if (!b || !n) return CPBUS_EINVAL;
  if ((uint64_t)b->n_next + n > b->N) return CPBUS_ENOSPC;
  int rc = enter(b); if (rc) return rc;
  if ((rc = flush_staged(b, b->now))) return rc;   // ordered with publishes (events/bus.go:105-107 takes the same lock)
  const uint32_t first = b->n_next;
  std::vector<SubCtl> blocks(n);
  memset(blocks.data(), 0, (size_t)n * sizeof(SubCtl));
  for (uint32_t i = 0; i < n; i++) {
    b->h_mask[first + i] = (masks ? masks[i] : CPBUS_MASK_ALL) & CPBUS_MASK_ALL;
    blocks[i].mask = b->h_mask[first + i] | kActiveBit;
    b->h_active[first + i] = 1;
    if (b->h_mask[first + i] != CPBUS_MASK_ALL) b->n_filtered++;
  }
  CK(cudaMemcpyAsync(b->d_ctl + first, blocks.data(), (size_t)n * sizeof(SubCtl), cudaMemcpyHostToDevice, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  b->n_next += n; b->n_active += n; b->order_dirty = true;
  if (first_sub_id) *first_sub_id = b->cfg.sub_id_base + first;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_subscribe(cpbus_t* b, uint32_t mask, uint32_t* sub_id) { return cpbus_subscribe_many(b, &mask, 1, sub_id); }

static int push_mask_words(cpbus* b, uint32_t first, uint32_t n);

int cpbus_subscribe_pairs(cpbus_t* b, uint32_t mask, const cpbus_pair* pairs, uint32_t n_pairs, uint32_t* sub_id) try {
  if (!b || n_pairs > CPBUS_MAX_PAIRS || (n_pairs && !pairs)) return CPBUS_EINVAL;
  for (uint32_t j = 0; j < n_pairs; j++) if (pairs[j].code >= CPBUS_N_CODES) return CPBUS_EINVAL;
  // a pair whose code is already in the mask adds nothing; what is left decides whether a table is needed at all
  uint2 row[CPBUS_MAX_PAIRS];
  uint32_t used = 0;
  for (uint32_t j = 0; j < n_pairs; j++)
    if (!((mask >> pairs[j].code) & 1u)) row[used++] = make_uint2(pairs[j].code, pairs[j].source_id);
  if (used == 0) return cpbus_subscribe_many(b, &mask, 1, sub_id);
  int rc = enter(b); if (rc) return rc;
  if (!b->d_pairs) {
    if (cudaMalloc((void**)&b->d_pairs, (size_t)b->N * CPBUS_MAX_PAIRS * sizeof(uint2)) != cudaSuccess) {
      snprintf(g_cuda_err, sizeof(g_cuda_err), "cudaMalloc(pair tables) failed");
      return CPBUS_ENOMEM;
    }
    CK(cudaMemsetAsync(b->d_pairs, 0xFF, (size_t)b->N * CPBUS_MAX_PAIRS * sizeof(uint2), b->stream));   // every slot unused
    b->h_npairs.assign(b->N, 0);
  }
  uint32_t id = 0;
  if ((rc = cpbus_subscribe_many(b, &mask, 1, &id))) return rc;
  const uint32_t l = id - b->cfg.sub_id_base;
  for (uint32_t j = used; j < CPBUS_MAX_PAIRS; j++) row[j] = make_uint2(kPairNone, kPairNone);
  CK(cudaMemcpyAsync(b->d_pairs + (size_t)l * CPBUS_MAX_PAIRS, row, sizeof(row), cudaMemcpyHostToDevice, b->stream));
  CK(cudaStreamSynchronize(b->stream));   // `row` is on the stack
  b->h_npairs[l] = (uint8_t)used; b->n_paired++;
  if ((rc = push_mask_words(b, l, 1))) return rc;
  if (sub_id) *sub_id = id;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_subscribe_pairs_many(cpbus_t* b, const uint32_t* masks, const cpbus_pair* pairs, const uint32_t* n_pairs,
                               uint32_t n, uint32_t* first_sub_id) try {
  if (!b || !n || !masks || !pairs || !n_pairs) return CPBUS_EINVAL;
  for (uint32_t i = 0; i < n; i++) {
    if (n_pairs[i] > CPBUS_MAX_PAIRS) return CPBUS_EINVAL;
    for (uint32_t j = 0; j < n_pairs[i]; j++) if (pairs[(size_t)i * CPBUS_MAX_PAIRS + j].code >= CPBUS_N_CODES) return CPBUS_EINVAL;
  }
  if ((uint64_t)b->n_next + n > b->N) return CPBUS_ENOSPC;
  int rc = enter(b); if (rc) return rc;
  if (!b->d_pairs) {
    if (cudaMalloc((void**)&b->d_pairs, (size_t)b->N * CPBUS_MAX_PAIRS * sizeof(uint2)) != cudaSuccess) {
      snprintf(g_cuda_err, sizeof(g_cuda_err), "cudaMalloc(pair tables) failed");
      return CPBUS_ENOMEM;
    }
    CK(cudaMemsetAsync(b->d_pairs, 0xFF, (size_t)b->N * CPBUS_MAX_PAIRS * sizeof(uint2), b->stream));   // every slot unused
    b->h_npairs.assign(b->N, 0);
  }
  uint32_t first = 0;
  if ((rc = cpbus_subscribe_many(b, masks, n, &first))) return rc;
  const uint32_t l0 = first - b->cfg.sub_id_base;
  std::vector<uint2> rows((size_t)n * CPBUS_MAX_PAIRS, make_uint2(kPairNone, kPairNone));
  uint32_t paired = 0;
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t m = masks[i] & CPBUS_MASK_ALL;
    uint32_t used = 0;
    for (uint32_t j = 0; j < n_pairs[i]; j++) {
      const cpbus_pair& pr = pairs[(size_t)i * CPBUS_MAX_PAIRS + j];
      if (!((m >> pr.code) & 1u)) rows[(size_t)i * CPBUS_MAX_PAIRS + used++] = make_uint2(pr.code, pr.source_id);
    }
    b->h_npairs[l0 + i] = (uint8_t)used;
    if (used) paired++;
  }
  CK(cudaMemcpyAsync(b->d_pairs + (size_t)l0 * CPBUS_MAX_PAIRS, rows.data(), rows.size() * sizeof(uint2), cudaMemcpyHostToDevice, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  b->n_paired += paired;
  if (paired && (rc = push_mask_words(b, l0, n))) return rc;
  if (first_sub_id) *first_sub_id = first;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_unsubscribe(cpbus_t* b, uint32_t sub_id) try {
  if (!b) return CPBUS_EINVAL;
  const uint32_t l = sub_id - b->cfg.sub_id_base;
  if (sub_id < b->cfg.sub_id_base || l >= b->n_next) return CPBUS_ENOENT;
  int rc = enter(b); if (rc) return rc;
  if ((rc = flush_staged(b, b->now))) return rc;
  // second Unsubscribe drives the WaitGroup negative in Go (events/bus.go:121) => panic
  if (!b->h_active[l]) return CPBUS_ECLOSED;
  b->h_active[l] = 0;
  if (b->h_mask[l] != CPBUS_MASK_ALL) b->n_filtered--;
  if (!b->h_npairs.empty() && b->h_npairs[l]) { b->h_npairs[l] = 0; b->n_paired--; }
  b->order_dirty = true;
  const uint32_t word = 0;
  CK(cudaMemcpyAsync(&b->d_ctl[l].mask, &word, 4, cudaMemcpyHostToDevice, b->stream));
  if (b->K && !b->h_timers.empty()) {
    for (uint32_t k = 0; k < b->K; k++) {
      HostTimer& t = b->h_timers[(size_t)l * b->K + k];
      if (t.active) { t.active = false; b->n_timers--; }
    }
    CK(cudaMemsetAsync(b->d_timers + (size_t)l * b->K, 0xFF, b->K * sizeof(DevTimer), b->stream));
  }
  CK(cudaStreamSynchronize(b->stream));
  b->n_active--;
  return CPBUS_OK;
} CPBUS_CATCH

// Change a subscriber's code mask in place (ordered with publishes like Subscribe): the subscriber keeps its mailbox,
// its timers and its exact cases.  Used when a mailbox that so far only received timer ticks / direct sends (mask 0:
// NewEventTimer on a channel that was not subscribed, watches/watches.go:37,71) is subscribed to the bus after all.
int cpbus_set_mask(cpbus_t* b, uint32_t sub_id, uint32_t mask) try {
  if (!b) return CPBUS_EINVAL;
  const uint32_t l = sub_id - b->cfg.sub_id_base;
  if (sub_id < b->cfg.sub_id_base || l >= b->n_next) return CPBUS_ENOENT;
  if (!b->h_active[l]) return CPBUS_ECLOSED;
  int rc = enter(b); if (rc) return rc;
  if ((rc = flush_staged(b, b->now))) return rc;
  mask &= CPBUS_MASK_ALL;
  if (b->h_mask[l] != CPBUS_MASK_ALL) b->n_filtered--;
  if (mask != CPBUS_MASK_ALL) b->n_filtered++;
  b->h_mask[l] = mask; b->order_dirty = true;
  return push_mask_words(b, l, 1);
} CPBUS_CATCH

static int push_mask_words(cpbus* b, uint32_t first, uint32_t n) {
  std::vector<uint32_t> words(n);
  for (uint32_t i = 0; i < n; i++) words[i] = mask_word(b, first + i);
  CK(cudaMemcpy2DAsync(&b->d_ctl[first].mask, sizeof(SubCtl), words.data(), 4, 4, n, cudaMemcpyHostToDevice, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  return CPBUS_OK;
}

int cpbus_timer_add(cpbus_t* b, uint32_t sub_id, uint64_t period_ns, uint32_t source_id, int oneshot, uint32_t* timer_id) try {
  if (!b || !period_ns) return CPBUS_EINVAL;
  if (!b->K) return CPBUS_ENOSPC;
  const uint32_t l = sub_id - b->cfg.sub_id_base;
  if (sub_id < b->cfg.sub_id_base || l >= b->n_next) return CPBUS_ENOENT;
  int rc = enter(b); if (rc) return rc;
  if ((rc = flush_staged(b, b->now))) return rc;
  if (b->h_timers.empty()) b->h_timers.resize((size_t)b->N * b->K);
  retire_oneshots(b, b->last_watermark);
  if (!b->h_active[l]) return CPBUS_ECLOSED;
  for (uint32_t k = 0; k < b->K; k++) {
    HostTimer& t = b->h_timers[(size_t)l * b->K + k];
    if (t.active) continue;
    t.active = true; t.oneshot = oneshot != 0; t.period = period_ns; t.next_due = due_after(b->now, period_ns); t.source_id = source_id;
    DevTimer d{}; d.next_due = t.next_due; d.period = oneshot ? 0 : period_ns; d.source_id = source_id; d.fired = 0;
    CK(cudaMemcpyAsync(b->d_timers + (size_t)l * b->K + k, &d, sizeof(d), cudaMemcpyHostToDevice, b->stream));
    CK(cudaStreamSynchronize(b->stream));
    b->n_timers++;
    if (!oneshot) b->min_period = std::min(b->min_period, period_ns);
    else b->oneshot_idx.push_back((size_t)l * b->K + k);
    t.gen = (uint8_t)((t.gen + 1) & 0x3F);
    if (timer_id) *timer_id = (l * b->K + k) | ((uint32_t)t.gen << kTimerSlotBits);
    return push_mask_words(b, l, 1);
  }
  return CPBUS_ENOSPC;
} CPBUS_CATCH

int cpbus_timer_add_many(cpbus_t* b, uint32_t first_sub, uint32_t n, uint64_t period_ns, const uint32_t* source_ids,
                         uint32_t source_id0, int oneshot) try {
  if (!b || !period_ns || !n) return CPBUS_EINVAL;
  if (!b->K) return CPBUS_ENOSPC;
  const uint32_t l0 = first_sub - b->cfg.sub_id_base;
  if (first_sub < b->cfg.sub_id_base || (uint64_t)l0 + n > b->n_next) return CPBUS_ENOENT;
  int rc = enter(b); if (rc) return rc;
  if ((rc = flush_staged(b, b->now))) return rc;
  if (b->h_timers.empty()) b->h_timers.resize((size_t)b->N * b->K);
  // bulk arm: uses slot 0 of each subscriber (must be free)
  retire_oneshots(b, b->last_watermark);
  for (uint32_t i = 0; i < n; i++) {
    if (!b->h_active[l0 + i]) return CPBUS_ECLOSED;
    if (b->h_timers[(size_t)(l0 + i) * b->K].active) return CPBUS_ENOSPC;
  }
  std::vector<DevTimer> dev((size_t)n * b->K);
  memset(dev.data(), 0, dev.size() * sizeof(DevTimer));
  CK(cudaMemcpyAsync(dev.data(), b->d_timers + (size_t)l0 * b->K, dev.size() * sizeof(DevTimer), cudaMemcpyDeviceToHost, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  for (uint32_t i = 0; i < n; i++) {
    HostTimer& t = b->h_timers[(size_t)(l0 + i) * b->K];
    t.active = true; t.oneshot = oneshot != 0; t.period = period_ns; t.next_due = due_after(b->now, period_ns);
    t.source_id = source_ids ? source_ids[i] : source_id0 + i;
    DevTimer& d = dev[(size_t)i * b->K];
    d.next_due = t.next_due; d.period = oneshot ? 0 : period_ns; d.source_id = t.source_id; d.fired = 0; d.pad[0] = d.pad[1] = 0;
    if (oneshot) b->oneshot_idx.push_back((size_t)(l0 + i) * b->K);
  }
  CK(cudaMemcpyAsync(b->d_timers + (size_t)l0 * b->K, dev.data(), dev.size() * sizeof(DevTimer), cudaMemcpyHostToDevice, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  b->n_timers += n;
  if (!oneshot) b->min_period = std::min(b->min_period, period_ns);
  return push_mask_words(b, l0, n);
} CPBUS_CATCH

int cpbus_timer_cancel(cpbus_t* b, uint32_t timer_id) try {
  if (!b) return CPBUS_EINVAL;
  if (!b->K || b->h_timers.empty()) return CPBUS_ENOENT;
  const uint32_t slot_index = timer_id & kTimerSlotMask, gen = timer_id >> kTimerSlotBits;
  const uint32_t l = slot_index / b->K, k = slot_index % b->K;
  if (l >= b->n_next) return CPBUS_ENOENT;
  int rc = enter(b); if (rc) return rc;
  if ((rc = flush_staged(b, b->now))) return rc;   // firings due before the cancel still happen
  retire_oneshots(b, b->last_watermark);
  HostTimer& t = b->h_timers[(size_t)l * b->K + k];
  if (!t.active || t.gen != gen) return CPBUS_ENOENT;   // already fired / cancelled, or the slot has been re-armed since
  t.active = false; b->n_timers--;
  CK(cudaMemsetAsync(b->d_timers + (size_t)l * b->K + k, 0xFF, sizeof(DevTimer), b->stream));
  CK(cudaStreamSynchronize(b->stream));
  if (b->n_timers == 0) b->min_period = UINT64_MAX;
  return push_mask_words(b, l, 1);
} CPBUS_CATCH

int cpbus_publish(cpbus_t* b, const cpbus_event* ev, size_t n) try {
  if (!b || (!ev && n)) return CPBUS_EINVAL;
  int rc = enter(b); if (rc) return rc;
  for (size_t i = 0; i < n; i++) {   // counter slots of the whole burst: requested up front, touched in the loop below
    if (ev[i].code < CPBUS_N_CODES && ev[i].code != CPBUS_METRIC) b->pub_pairs.prefetch(((uint64_t)ev[i].code << 32) | ev[i].source_id);
  }
  // The debug ring holds 10 entries (events/bus.go:24-31): of a burst only the last 10 published can ever be seen, so only
  // those are enqueued — including when the call stops early (CPBUS_EAGAIN from an automatic flush in lossless mode).
  auto dbg_tail = [&](size_t published) {
    for (size_t j = published > 10 ? published - 10 : 0; j < published; j++) {
      cpbus_event e{};
      e.seq = b->seq - (published - j); e.ts_ns = b->now; e.code = ev[j].code; e.source_id = ev[j].source_id; e.target = CPBUS_TARGET_ALL;
      dbg_enqueue(b, e);
    }
  };
  for (size_t i = 0; i < n; i++) if (ev[i].code >= CPBUS_N_CODES) return CPBUS_EINVAL;   // nothing of an invalid burst is published
  for (size_t i = 0; i < n; i++) {
    const uint32_t code = ev[i].code;
    if ((rc = stage_one(b, code, ev[i].source_id, CPBUS_TARGET_ALL, 0))) { dbg_tail(i); return rc; }
    if (code != CPBUS_METRIC) {                                  // events/bus.go:130-132
      b->st.published_by_code[code]++;
      b->pub_pairs.add(((uint64_t)code << 32) | ev[i].source_id, 1);
    }
    b->st.publishes++;
  }
  dbg_tail(n);                                                   // events/bus.go:139
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_send(cpbus_t* b, uint32_t sub_id, const cpbus_event* ev) try {
  if (!b || !ev || ev->code >= CPBUS_N_CODES) return CPBUS_EINVAL;
  const uint32_t l = sub_id - b->cfg.sub_id_base;
  if (sub_id < b->cfg.sub_id_base || l >= b->n_next) return CPBUS_ENOENT;
  if (!b->h_active[l]) return CPBUS_ECLOSED;   // the mailbox is gone (Go: send on a closed channel panics)
  int rc = enter(b); if (rc) return rc;
  if ((rc = stage_one(b, ev->code, ev->source_id, sub_id, CPBUS_F_UNICAST))) return rc;
  b->st.publishes++;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_advance(cpbus_t* b, uint64_t now_ns) try {
  if (!b) return CPBUS_EINVAL;
  int rc = follow_resolve(b); if (rc) return rc;   // the clock moves with the batches that followers fanned out
  if (now_ns < b->now) return CPBUS_EORDER;
  if (now_ns == b->now) return CPBUS_OK;
  if ((rc = dev_guard(b))) return rc;
  // the kernel looks at <= 32/K candidate firings per timer slot per launch: keep every
  // flush window within that many periods of the fastest periodic timer
  const uint64_t win = max_window(b);
  while (win != UINT64_MAX && now_ns - b->last_watermark > win) {
    b->now = b->last_watermark + win;
    if ((rc = flush_staged(b, b->now))) return rc;
  }
  b->now = now_ns;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_flush(cpbus_t* b) try {
  if (!b) return CPBUS_EINVAL;
  int rc = enter(b); if (rc) return rc;
  return flush_staged(b, b->now);
} CPBUS_CATCH

int cpbus_sync(cpbus_t* b) try {
  if (!b) return CPBUS_EINVAL;
  int rc = enter(b); if (rc) return rc;
  CK(cudaStreamSynchronize(b->stream));
  return CPBUS_OK;
} CPBUS_CATCH

static int publish_device_impl(cpbus_t* b, const void* d_events, size_t n, uint64_t watermark_ns, bool staged,
                               const void* d_next, size_t n_next);

// A device batch that one launch cannot take — more than batch_cap records, or a watermark further from the last one than the
// 32/K firings per timer slot a launch examines — is cut into slices that can (round 1 answered CPBUS_EINVAL / CPBUS_EORDER).
// The cut needs the records' timestamps: one strided D2H of 8 bytes per record, on this slow path only.  A slice ends at
// batch_cap records or at the window's edge, whichever comes first, and its watermark is its last record's timestamp (cut by
// size) or the edge (cut by time): ticks due by then are merged exactly where the unsplit launch would have put them, because
// a tick is ordered in front of every event with ts >= its due time and such events are either in this slice behind it or
// in a later one.  The host path does the same at cpbus_advance.  (events/timer.go:40-71 has no such limit: a Go timer
// that fell behind fires late, never "not at all".)
// The cut itself, host-only (exported as cpbus_split_plan so that it can be tested without a GPU): slice k = records
// [end[k-1], end[k]) launched with watermark wm[k].  `now` = the bus clock (= the last launched watermark once staged events
// are flushed), `window` = the widest watermark step one launch may take (UINT64_MAX: no timer armed).
static int split_plan(const uint64_t* ts, size_t n, uint32_t batch_cap, uint64_t now, uint64_t watermark, uint64_t window,
                      std::vector<size_t>& end, std::vector<uint64_t>& wm) {
  for (size_t i = 1; i < n; i++) if (ts[i] < ts[i - 1]) return CPBUS_EORDER;
  if (!batch_cap || !window) return CPBUS_EINVAL;
  if (watermark < now || (n && ts[n - 1] > watermark)) return CPBUS_EORDER;
  size_t i = 0;
  uint64_t lw = now;
  for (;;) {
    const uint64_t edge = (window == UINT64_MAX || watermark - lw <= window) ? watermark : lw + window;
    size_t j = std::upper_bound(ts + i, ts + n, edge) - ts;
    uint64_t w = edge;
    if (j - i > batch_cap) { j = i + batch_cap; w = std::max(ts[j - 1], lw); }   // (records older than the clock ride with it)
    end.push_back(j); wm.push_back(w);
    i = j; lw = w;
    if (j == n && w == watermark) return CPBUS_OK;
  }
}

static int publish_device_split(cpbus_t* b, const cpbus_event* d_events, size_t n, uint64_t watermark_ns, bool staged,
                                const void* d_next, size_t n_next) {
  std::vector<uint64_t> ts, wm;
  std::vector<size_t> end;
  ts.resize(n);
  if (n) {
    CK(cudaMemcpy2DAsync(ts.data(), 8, reinterpret_cast<const unsigned char*>(d_events) + offsetof(cpbus_event, ts_ns), sizeof(cpbus_event),
                         8, n, cudaMemcpyDeviceToHost, b->stream));
    CK(cudaStreamSynchronize(b->stream));
  }
  int rc = split_plan(ts.data(), n, b->B, b->now, watermark_ns, max_window(b), end, wm);   // (a one-shot retiring mid-way can only widen the window)
  if (rc) return rc;
  size_t i = 0;
  for (size_t k = 0; k < end.size(); k++) {
    const bool last = k + 1 == end.size();
    rc = publish_device_impl(b, d_events + i, end[k] - i, wm[k], staged, last ? d_next : nullptr, last ? n_next : 0);
    if (rc) return rc;
    b->st.device_splits++;
    i = end[k];
  }
  return CPBUS_OK;
}

static int publish_device_impl(cpbus_t* b, const void* d_events, size_t n, uint64_t watermark_ns, bool staged,
                               const void* d_next, size_t n_next) {
  if (!b || (!d_events && n) || ((uintptr_t)d_events & 31u) || n_next > b->B || ((uintptr_t)d_next & 31u)) return CPBUS_EINVAL;
  int rc = enter(b); if (rc) return rc;
  if ((rc = flush_staged(b, b->now))) return rc;
  if (watermark_ns < b->now) return CPBUS_EORDER;
  if (staged && b->lossless) return CPBUS_EINVAL;   // admission would have to read the peer batch: not supported
  if (n > b->B || watermark_ns - b->last_watermark > max_window(b)) {
    // lossless mode stays all-or-nothing per call (the caller owns the batch and could not tell how far a refused call got)
    if (b->lossless) return n > b->B ? CPBUS_EINVAL : CPBUS_EORDER;
    return publish_device_split(b, (const cpbus_event*)d_events, n, watermark_ns, staged, d_next, n_next);
  }
  bool ok = true;
  if ((rc = admit(b, (const cpbus_event*)d_events, (uint32_t)n, watermark_ns, &ok))) return rc;
  if (!ok) return CPBUS_EAGAIN;
  b->now = watermark_ns;
  const cpbus_event* src = (const cpbus_event*)d_events;
  bool dep = false;
  // Prefetch cache: a peer batch an earlier launch already pulled into d_prefetch[i].  An entry is good for ONE use, only
  // while it is recent (the caller may re-stamp or reuse the peer buffer later), and the newest match wins.
  for (int i = 0; i < cpbus::kPrefetch; i++)
    if (b->pf_ptr[i] && b->launch_seq - b->pf_seq[i] > (unsigned long long)cpbus::kPrefetch) b->pf_ptr[i] = nullptr;
  if (staged && n) {
    int hit = -1;
    for (int i = 0; i < cpbus::kPrefetch; i++)
      if (b->pf_ptr[i] == d_events && b->pf_n[i] == n && (hit < 0 || b->pf_seq[i] > b->pf_seq[hit])) hit = i;
    if (hit >= 0) {
      src = b->d_prefetch[hit];          // plain local launch
      staged = false;
      dep = b->pf_seq[hit] == b->launch_seq;   // written by the IMMEDIATELY preceding launch: its prologue must not run ahead
      for (int i = 0; i < cpbus::kPrefetch; i++) if (b->pf_ptr[i] == d_events) b->pf_ptr[i] = nullptr;   // consumed (and any older copy dropped)
    }
  }
  LaunchOpts o;
  o.staged = staged ? 1 : 0; o.pf_n = (uint32_t)n_next; o.batch_dep = dep; o.account = true;
  int slot = -1;
  if (d_next && n_next) {
    slot = b->pf_next;
    if (b->d_prefetch[slot] == src) slot = (slot + 1) % cpbus::kPrefetch;   // never overwrite the buffer this launch reads
    o.pf_src = (const cpbus_event*)d_next; o.pf_dst = b->d_prefetch[slot];
    for (int i = 0; i < cpbus::kPrefetch; i++) if (b->pf_ptr[i] == d_next) b->pf_ptr[i] = nullptr;   // superseded
  }
  const unsigned long long seq0 = b->launch_seq;
  if ((rc = launch_fanout(b, src, (uint32_t)n, watermark_ns, o))) return rc;
  // an empty batch with no timer armed launches nothing, so nothing pulled d_next: the cache must not claim it
  if (slot >= 0 && b->launch_seq != seq0) { b->pf_ptr[slot] = d_next; b->pf_n[slot] = n_next; b->pf_seq[slot] = b->launch_seq; b->pf_next = (slot + 1) % cpbus::kPrefetch; }
  b->st.publishes += n; b->seq += n;
  return CPBUS_OK;
}

int cpbus_publish_device(cpbus_t* b, const void* d_events, size_t n, uint64_t watermark_ns) try {
  return publish_device_impl(b, d_events, n, watermark_ns, false, nullptr, 0);
} CPBUS_CATCH

// Multi-GPU ingest fused into the fan-out kernel: d_events (and d_next) may point into ANOTHER GPU's HBM (the
// publisher's event stream, peer-mapped over NVLink).  One CTA pulls the batch across the link, stages it in local
// HBM and publishes it with the batch descriptor; if the caller names the NEXT batch, that one is pulled by the
// same launch while its stores are in flight, so the following call starts from local memory.  No collective.
int cpbus_publish_device_staged(cpbus_t* b, const void* d_events, size_t n, uint64_t watermark_ns, const void* d_next, size_t n_next) try {
  return publish_device_impl(b, d_events, n, watermark_ns, true, d_next, n_next);
} CPBUS_CATCH

// ---- buffers shared between the GPUs of one box (CUDA IPC; NVLink peer mapping on the importing side) ----
int cpbus_shared_alloc(cpbus_t* b, size_t bytes, void** dptr, unsigned char handle[64]) try {
  if (!b || !dptr || !handle || !bytes) return CPBUS_EINVAL;
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  int rc = dev_guard(b); if (rc) return rc;
  void* p = nullptr;
  if (cudaMalloc(&p, bytes) != cudaSuccess) { snprintf(g_cuda_err, sizeof(g_cuda_err), "cudaMalloc(%zu) failed", bytes); return CPBUS_ENOMEM; }
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) { cudaFree(p); snprintf(g_cuda_err, sizeof(g_cuda_err), "cudaIpcGetMemHandle: %s", cudaGetErrorString(e)); return CPBUS_ECUDA; }
  memcpy(handle, &h, 64);
  b->shared_owned.push_back(p);
  *dptr = p;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_shared_open(cpbus_t* b, const unsigned char handle[64], void** dptr) try {
  if (!b || !dptr || !handle) return CPBUS_EINVAL;
  int rc = dev_guard(b); if (rc) return rc;      // the IMPORTING device must be current: the mapping is made for it
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, 64);
  void* p = nullptr;
  CK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  b->shared_mapped.push_back(p);
  *dptr = p;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_shared_close(cpbus_t* b, void* dptr) try {
  if (!b || !dptr) return CPBUS_EINVAL;
  int rc = dev_guard(b); if (rc) return rc;
  CK(cudaStreamSynchronize(b->stream));
  for (int i = 0; i < cpbus::kPrefetch; i++) b->pf_ptr[i] = nullptr;   // prefetched copies of anything in that buffer are void
  for (size_t i = 0; i < b->shared_owned.size(); i++)
    if (b->shared_owned[i] == dptr) { cudaFree(dptr); b->shared_owned.erase(b->shared_owned.begin() + i); return CPBUS_OK; }
  for (size_t i = 0; i < b->shared_mapped.size(); i++)
    if (b->shared_mapped[i] == dptr) { cudaIpcCloseMemHandle(dptr); b->shared_mapped.erase(b->shared_mapped.begin() + i); return CPBUS_OK; }
  return CPBUS_ENOENT;
} CPBUS_CATCH

// ---- the publisher's event stream across the GPUs of one box (include/cpbus.h: cpbus_stream_*) ----
struct cpbus_stream {
  cpbus* bus = nullptr;
  bool owner = false, attached = false;      // attached: same-process consumer sharing the owner's pointer (peer access, no IPC)
  uint32_t n_slots = 0, n_consumers = 0, consumer = 0, B = 0;
  unsigned char* base = nullptr;             // the ring: local memory on the publisher, NVLink peer mapping elsewhere
  StreamHdr* hdr = nullptr;
  unsigned long long* ack = nullptr;         // consumer c's word is ack[4 * c] (one sector each)
  cpbus_event* payload = nullptr;
  unsigned long long put_seq = 0, get_seq = 0;   // batches released / fanned out so far (ordinals are 1-based)
  uint32_t get_off = 0;                      // lossless mode: records of batch get_seq + 1 already delivered
  uint32_t follow_out = 0;                   // follower launches of batches get_seq + 1 .. not yet resolved
  unsigned long long seen_seq = 0;           // highest batch whose release this consumer has seen from the host
  RoundCursor* d_cursor = nullptr;           // lossless rounds (cpbus_stream_round_next): {batch, offset} on the device
  unsigned long long stalled_rounds = 0;     // ... rounds resolved so far that moved nothing
  unsigned long long pub_seq = 0;            // publisher: publish ordinal stamped into the next record (CPBUS_PUT_STAMP)
  unsigned long long min_ack = 0;            // publisher: cached min over the consumers' acks
  // publisher staging: pinned payload + header buffers, copies on their own stream
  static constexpr int kStage = 8;
  cpbus_event* h_stage[kStage] = {};
  StreamHdr* h_hdr = nullptr;                // kStage headers
  unsigned long long* h_ack = nullptr;       // kStreamMaxConsumers x 4 words
  cudaEvent_t staged_done[kStage] = {};
  cudaStream_t put_stream = nullptr;
  // lossless across processes (cpbus_stream_offer / _agree): admission rounds agreed so far, and this round's state
  unsigned long long agree_round = 0;
  bool offered = false;
  unsigned long long admit_q = 0;            // batch ordinal and shape of the latest cpbus_stream_admit (bounds an offer)
  size_t admit_n = 0;
  StreamAgreeResult* h_agree = nullptr;      // pinned + mapped: written by the agree kernel
  StreamAgreeResult* d_agree = nullptr;      // device alias of h_agree
  cudaEvent_t agree_done = nullptr;
};

static int stream_bind(cpbus_stream* st) {
  st->hdr = reinterpret_cast<StreamHdr*>(st->base + stream_hdr_off());
  st->ack = reinterpret_cast<unsigned long long*>(st->base + stream_ack_off(st->n_slots));
  st->payload = reinterpret_cast<cpbus_event*>(st->base + stream_payload_off(st->n_slots));
  if (st->bus->lossless && cudaMalloc((void**)&st->d_cursor, sizeof(RoundCursor)) != cudaSuccess) {   // rounds' cursor
    snprintf(g_cuda_err, sizeof(g_cuda_err), "cudaMalloc(%zu) failed", sizeof(RoundCursor));
    return CPBUS_ENOMEM;
  }
  return CPBUS_OK;
}

int cpbus_stream_create(cpbus_t* b, uint32_t n_slots, uint32_t n_consumers, cpbus_stream_t** out, unsigned char handle[64]) try {
  if (!b || !out || !handle || n_slots < 4 || n_consumers == 0 || n_consumers > kStreamMaxConsumers) return CPBUS_EINVAL;
  *out = nullptr;
  int rc = dev_guard(b); if (rc) return rc;
  cpbus_stream* st = new (std::nothrow) cpbus_stream();
  if (!st) return CPBUS_ENOMEM;
  st->bus = b; st->owner = true; st->n_slots = n_slots; st->n_consumers = n_consumers; st->consumer = 0; st->B = b->B;
  st->pub_seq = b->seq;
  const size_t bytes = stream_bytes(n_slots, b->B);
  auto fail = [&](int code) { cpbus_stream_close(st); return code; };
  b->streams.push_back(st);
  if (cudaMalloc((void**)&st->base, bytes) != cudaSuccess) { snprintf(g_cuda_err, sizeof(g_cuda_err), "cudaMalloc(%zu) failed", bytes); return fail(CPBUS_ENOMEM); }
  if (cudaMemset(st->base, 0, stream_payload_off(n_slots)) != cudaSuccess) return fail(CPBUS_ECUDA);
  StreamMeta meta{}; meta.magic = kStreamMagic; meta.n_slots = n_slots; meta.batch_cap = b->B; meta.n_consumers = n_consumers;
  if (cudaMemcpy(st->base, &meta, sizeof(meta), cudaMemcpyHostToDevice) != cudaSuccess) return fail(CPBUS_ECUDA);
  cudaIpcMemHandle_t h;
  if (cudaIpcGetMemHandle(&h, st->base) != cudaSuccess) { snprintf(g_cuda_err, sizeof(g_cuda_err), "cudaIpcGetMemHandle failed"); return fail(CPBUS_ECUDA); }
  memcpy(handle, &h, 64);
  if ((rc = stream_bind(st))) return fail(rc);
  if (cudaStreamCreateWithFlags(&st->put_stream, cudaStreamNonBlocking) != cudaSuccess) return fail(CPBUS_ECUDA);
  for (int i = 0; i < cpbus_stream::kStage; i++) {
    if (cudaMallocHost((void**)&st->h_stage[i], (size_t)b->B * sizeof(cpbus_event)) != cudaSuccess) return fail(CPBUS_ENOMEM);
    if (cudaEventCreateWithFlags(&st->staged_done[i], cudaEventDisableTiming) != cudaSuccess) return fail(CPBUS_ECUDA);
  }
  if (cudaMallocHost((void**)&st->h_hdr, sizeof(StreamHdr) * cpbus_stream::kStage) != cudaSuccess) return fail(CPBUS_ENOMEM);
  if (cudaMallocHost((void**)&st->h_ack, (size_t)kStreamMaxConsumers * 32) != cudaSuccess) return fail(CPBUS_ENOMEM);
  *out = st;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_stream_open(cpbus_t* b, const unsigned char handle[64], uint32_t consumer_index, cpbus_stream_t** out) try {
  if (!b || !out || !handle || consumer_index == 0 || consumer_index >= kStreamMaxConsumers) return CPBUS_EINVAL;
  *out = nullptr;
  int rc = dev_guard(b); if (rc) return rc;      // the IMPORTING device must be current: the mapping is made for it
  cpbus_stream* st = new (std::nothrow) cpbus_stream();
  if (!st) return CPBUS_ENOMEM;
  st->bus = b; st->owner = false; st->consumer = consumer_index;
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, 64);
  cudaError_t e = cudaIpcOpenMemHandle((void**)&st->base, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) { snprintf(g_cuda_err, sizeof(g_cuda_err), "cudaIpcOpenMemHandle: %s", cudaGetErrorString(e)); delete st; return CPBUS_ECUDA; }
  StreamMeta meta{};
  e = cudaMemcpy(&meta, st->base, sizeof(meta), cudaMemcpyDeviceToHost);
  if (e != cudaSuccess || meta.magic != kStreamMagic || meta.batch_cap != b->B || consumer_index >= meta.n_consumers) {
    snprintf(g_cuda_err, sizeof(g_cuda_err), "stream meta mismatch (magic %x, batch_cap %u vs %u, consumers %u)", meta.magic, meta.batch_cap, b->B, meta.n_consumers);
    cudaIpcCloseMemHandle(st->base); delete st;
    return e != cudaSuccess ? CPBUS_ECUDA : CPBUS_EINVAL;
  }
  st->n_slots = meta.n_slots; st->n_consumers = meta.n_consumers; st->B = meta.batch_cap;
  if ((rc = stream_bind(st))) { cudaIpcCloseMemHandle(st->base); delete st; return rc; }
  b->streams.push_back(st);
  *out = st;
  return CPBUS_OK;
} CPBUS_CATCH

// Same-process consumer (one host process driving several GPUs, as a cgo shim would): no IPC handle — the owner's
// pointer is used directly, with peer access enabled when the consumer's bus lives on another GPU.
int cpbus_stream_attach(cpbus_t* b, cpbus_stream_t* owner, uint32_t consumer_index, cpbus_stream_t** out) try {
  if (!b || !owner || !owner->owner || !out || consumer_index == 0 || consumer_index >= owner->n_consumers) return CPBUS_EINVAL;
  if (b->B != owner->B) return CPBUS_EINVAL;
  *out = nullptr;
  int rc = dev_guard(b); if (rc) return rc;
  if (b->device != owner->bus->device) {
    int can = 0;
    CK(cudaDeviceCanAccessPeer(&can, b->device, owner->bus->device));
    if (!can) { snprintf(g_cuda_err, sizeof(g_cuda_err), "device %d cannot access device %d", b->device, owner->bus->device); return CPBUS_ECUDA; }
    const cudaError_t e = cudaDeviceEnablePeerAccess(owner->bus->device, 0);
    if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { CK(e); }
    cudaGetLastError();   // clear "already enabled"
  }
  cpbus_stream* st = new (std::nothrow) cpbus_stream();
  if (!st) return CPBUS_ENOMEM;
  st->bus = b; st->attached = true; st->consumer = consumer_index;
  st->n_slots = owner->n_slots; st->n_consumers = owner->n_consumers; st->B = owner->B; st->base = owner->base;
  if ((rc = stream_bind(st))) { delete st; return rc; }
  b->streams.push_back(st);
  *out = st;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_stream_close(cpbus_stream_t* st) try {
  if (!st) return CPBUS_EINVAL;
  cpbus* b = st->bus;
  follow_resolve(b);   // (teardown: the records of outstanding followers are folded in before the stream goes)
  cudaSetDevice(b->device);
  cudaStreamSynchronize(b->stream);
  if (st->put_stream) { cudaStreamSynchronize(st->put_stream); cudaStreamDestroy(st->put_stream); }
  for (int i = 0; i < cpbus_stream::kStage; i++) {
    if (st->h_stage[i]) cudaFreeHost(st->h_stage[i]);
    if (st->staged_done[i]) cudaEventDestroy(st->staged_done[i]);
  }
  if (st->h_hdr) cudaFreeHost(st->h_hdr);
  if (st->h_ack) cudaFreeHost(st->h_ack);
  if (st->h_agree) cudaFreeHost(st->h_agree);
  if (st->agree_done) cudaEventDestroy(st->agree_done);
  cudaFree(st->d_cursor);
  if (st->base) { if (st->owner) cudaFree(st->base); else if (!st->attached) cudaIpcCloseMemHandle(st->base); }
  b->streams.erase(std::remove(b->streams.begin(), b->streams.end(), st), b->streams.end());
  delete st;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_stream_set_timeout(cpbus_stream_t* st, uint32_t microseconds) try {
  if (!st) return CPBUS_EINVAL;
  st->bus->stream_spin_us = microseconds;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_stream_status(cpbus_stream_t* st) try {
  if (!st) return CPBUS_EINVAL;
  const int rc = follow_resolve(st->bus); if (rc) return rc;
  return stream_error(st->bus);
} CPBUS_CATCH

// Publisher: copy the batch into the next slot, then release it (header after payload, same stream).
int cpbus_stream_put(cpbus_stream_t* st, const cpbus_event* ev, size_t n, uint64_t now_ns, uint32_t flags) try {
  if (!st || !st->owner || (!ev && n) || n > st->B) return CPBUS_EINVAL;
  cpbus* b = st->bus;
  int rc = dev_guard(b); if (rc) return rc;
  const unsigned long long q = st->put_seq + 1;
  if (q > st->n_slots && st->min_ack + st->n_slots < q) {
    // The slot still holds batch q - n_slots: every consumer must have pulled it.  Acks are device words written by the
    // consumers' kernels; refresh the cached minimum, and — unless the caller asked not to wait — give consumers that
    // are merely behind (their launches are queued, the GPUs are busy) up to the stream timeout to get there.
    const auto t0 = std::chrono::steady_clock::now();
    for (;;) {
      CK(cudaMemcpyAsync(st->h_ack, st->ack, (size_t)st->n_consumers * 32, cudaMemcpyDeviceToHost, st->put_stream));
      CK(cudaStreamSynchronize(st->put_stream));
      unsigned long long m = ~0ull;
      for (uint32_t c = 0; c < st->n_consumers; c++) m = std::min(m, st->h_ack[4 * c]);
      st->min_ack = m;
      if (st->min_ack + st->n_slots >= q) break;
      if ((flags & CPBUS_PUT_NOWAIT) || std::chrono::steady_clock::now() - t0 > stream_budget(b) || *(volatile unsigned int*)b->h_err) return CPBUS_EAGAIN;
      std::this_thread::sleep_for(std::chrono::microseconds(20));
    }
  }
  const int s = (int)(q % cpbus_stream::kStage);
  CK(cudaEventSynchronize(st->staged_done[s]));   // the pinned buffers of batch q - kStage have left the host
  cpbus_event* dst = st->h_stage[s];
  if (flags & CPBUS_PUT_RAW) { if (n) memcpy(dst, ev, n * sizeof(cpbus_event)); }
  else {
    for (size_t i = 0; i < n; i++) {
      const uint32_t code = ev[i].code;
      if (code >= CPBUS_N_CODES) return CPBUS_EINVAL;
      dst[i].seq = st->pub_seq + i; dst[i].ts_ns = now_ns; dst[i].code = code; dst[i].source_id = ev[i].source_id;
      dst[i].target = CPBUS_TARGET_ALL; dst[i].flags = 0;
    }
  }
  const uint32_t slot = (uint32_t)(q % st->n_slots);
  if (n) CK(cudaMemcpyAsync(st->payload + (size_t)slot * st->B, dst, n * sizeof(cpbus_event), cudaMemcpyHostToDevice, st->put_stream));
  StreamHdr* hh = &st->h_hdr[s];
  memset(hh, 0, sizeof(*hh));
  hh->seq = q; hh->watermark = now_ns; hh->n = (uint32_t)n;
  if (!(flags & CPBUS_PUT_RAW)) st->pub_seq += n;
  CK(cudaMemcpyAsync(&st->hdr[slot], hh, sizeof(StreamHdr), cudaMemcpyHostToDevice, st->put_stream));   // the release: after the payload
  CK(cudaEventRecord(st->staged_done[s], st->put_stream));
  st->put_seq = q;
  return CPBUS_OK;
} CPBUS_CATCH

// Consumers that are NOT told n / now_ns by their driver: look at the next slot's header (one 32-byte copy across the link).
// *ready = 0: the publisher has not released that batch yet.
int cpbus_stream_poll(cpbus_stream_t* st, int* ready, size_t* n, uint64_t* now_ns) try {
  if (!st || !ready) return CPBUS_EINVAL;
  cpbus* b = st->bus;
  int rc = enter(b); if (rc) return rc;
  if ((rc = stream_error(b))) return rc;
  const unsigned long long q = st->get_seq + 1;
  StreamHdr h{};
  CK(cudaMemcpyAsync(&h, &st->hdr[q % st->n_slots], sizeof(h), cudaMemcpyDeviceToHost, b->result_stream));
  CK(cudaStreamSynchronize(b->result_stream));
  *ready = h.seq == q ? 1 : 0;
  if (*ready) { if (n) *n = h.n; if (now_ns) *now_ns = h.watermark; }
  return CPBUS_OK;
} CPBUS_CATCH

// Lossless stream, slow path only: before the host copies or reads records of batch q outside the fan-out kernel (which
// acquires the slot header itself), it waits until the publisher has released the batch — the payload lands before the
// header.  Bounded by the stream timeout; once per batch.
static int stream_wait_released(cpbus_stream* st, unsigned long long q, size_t n) {
  if (st->seen_seq >= q) return CPBUS_OK;
  cpbus* b = st->bus;
  const auto t0 = std::chrono::steady_clock::now();
  for (;;) {
    StreamHdr h{};
    CK(cudaMemcpyAsync(&h, &st->hdr[q % st->n_slots], sizeof(h), cudaMemcpyDeviceToHost, b->result_stream));
    CK(cudaStreamSynchronize(b->result_stream));
    if (h.seq == q) {
      if (h.n != n) return CPBUS_EINVAL;   // the caller's shape is not the released batch's
      st->seen_seq = q;
      return CPBUS_OK;
    }
    if (std::chrono::steady_clock::now() - t0 > stream_budget(b)) return CPBUS_ETIMEDOUT;
    std::this_thread::sleep_for(std::chrono::microseconds(20));
  }
}

// The checks every stream call makes before it admits or launches anything (clock, window, this bus's own staged events).
static int stream_enter(cpbus_stream* st, uint64_t now_ns) {
  cpbus* b = st->bus;
  int rc = enter(b); if (rc) return rc;
  if ((rc = stream_error(b))) return rc;
  if ((rc = flush_staged(b, b->now))) return rc;
  if (now_ns < b->now) return CPBUS_EORDER;
  if (now_ns - b->last_watermark > max_window(b)) return CPBUS_EORDER;
  return CPBUS_OK;
}

int cpbus_stream_admit(cpbus_stream_t* st, size_t n, uint64_t now_ns, size_t* prefix) try {
  if (!st || !prefix || n > st->B || st->get_off > n) return CPBUS_EINVAL;
  *prefix = 0;
  st->admit_q = st->get_seq + 1; st->admit_n = n;
  cpbus* b = st->bus;
  int rc = stream_enter(st, now_ns); if (rc) return rc;
  const uint32_t rem = (uint32_t)n - st->get_off;
  if (admit_fits(b, rem, now_ns)) { *prefix = rem; return CPBUS_OK; }   // no kernel, no sync
  // Slow path: the admission kernel reads the whole remainder from every CTA, so it runs on a local copy of it (one peer
  // copy on the bus stream) rather than over the link.  (Not d_batch_local: the fan-out kernel writes that one.)
  const unsigned long long q = st->get_seq + 1;
  if ((rc = stream_wait_released(st, q, n))) return rc;
  if (rem)
    CK(cudaMemcpyAsync(b->d_admit_batch, st->payload + (size_t)(q % st->n_slots) * st->B + st->get_off,
                       (size_t)rem * sizeof(cpbus_event), cudaMemcpyDefault, b->stream));
  bool ok = true;
  uint32_t m = rem;
  if ((rc = admit_pass(b, b->d_admit_batch, rem, now_ns, &ok, &m))) return rc;
  if (!ok && m == rem) {
    // Every record fits, but not the ticks due after the last of them (records older than now_ns, or none at all): the
    // batch cannot complete yet.  Hold back its last record, or report the stall when there is none.
    if (rem == 0) return CPBUS_EAGAIN;
    m = rem - 1;
  }
  *prefix = m;
  return CPBUS_OK;
} CPBUS_CATCH

// Consumer st's launch of batch q from record `off` of its slot: the header and this consumer's ack word and, without
// lossless mode, the batch after next for the kernel to prefetch (a lossless batch may take several launches, each reading
// its part of the slot, so lossless launches neither request nor take the prefetch).  Returns where the records start.
static const cpbus_event* stream_launch(const cpbus_stream* st, unsigned long long q, uint32_t off, bool final, StreamArgs& sa,
                                        LaunchOpts& o) {
  const cpbus* b = st->bus;
  const uint32_t slot = (uint32_t)(q % st->n_slots), slot2 = (uint32_t)((q + 2) % st->n_slots);
  sa.hdr = &st->hdr[slot]; sa.ack = &st->ack[4 * st->consumer]; sa.seq = q; sa.off = off; sa.final = final;
  o.staged = 2; o.account = true; o.stream = &sa;
  if (!b->lossless) {
    sa.next_hdr = &st->hdr[slot2];
    o.pf_src = st->payload + (size_t)slot2 * st->B; o.pf_dst = b->d_pf_buf + (size_t)((q + 2) % kStreamPrefetch) * b->B;
  }
  return st->payload + (size_t)slot * st->B + off;
}

// A stream launch that delivered m records with watermark w, folded into the host state; `final`: it completed its batch.
// The host-driven launch, a resolved follower and a resolved round all fold here, so each moves the host state exactly as
// the others with the same outcome do.
static void stream_delivered(cpbus* b, cpbus_stream* st, uint32_t m, uint64_t w, bool final, unsigned long long launch_seq) {
  b->st.publishes += m; b->seq += m;
  b->now = w; b->last_watermark = w;
  if (m) dbg_mark_device_batch(b, launch_seq);
  if (final) { st->get_seq++; st->get_off = 0; return; }
  st->get_off += m;
  b->room_lb = 0;
  b->st.admit_partial++;
}

// Fan out the next m undelivered records of the current batch (throughput mode: m = the whole batch, in one launch).
static int stream_fanout_prefix(cpbus_stream* st, size_t n, uint64_t now_ns, size_t m) {
  cpbus* b = st->bus;
  int rc = stream_enter(st, now_ns); if (rc) return rc;
  const bool final = m == n - st->get_off;
  if (m == 0 && !final) return CPBUS_EAGAIN;
  const unsigned long long q = st->get_seq + 1;
  StreamArgs sa;
  LaunchOpts o;
  const cpbus_event* src = stream_launch(st, q, st->get_off, final, sa, o);
  uint64_t w = now_ns;
  if (!final) {
    // Like a partial cpbus_flush: the watermark is the last delivered record's timestamp, so the ticks due after it go with
    // the remainder.  Read from the slot (8 bytes) rather than assumed to be now_ns: RAW records may be older.
    if ((rc = stream_wait_released(st, q, n))) return rc;
    uint64_t ts = 0;
    CK(cudaMemcpyAsync(&ts, &src[m - 1].ts_ns, sizeof(ts), cudaMemcpyDefault, b->result_stream));
    CK(cudaStreamSynchronize(b->result_stream));
    w = std::min(now_ns, std::max(ts, b->last_watermark));
  }
  // The clock follows the launched watermark.  Were it set to now_ns before the batch completes, the next call's flush of
  // this bus's own staged events would fire the ticks due by now_ns on their own, in front of the undelivered records and
  // without their admission.
  b->now = w;
  if ((rc = launch_fanout(b, src, (uint32_t)m, w, o))) return rc;
  stream_delivered(b, st, (uint32_t)m, w, final, b->launch_seq);
  return final ? CPBUS_OK : CPBUS_EAGAIN;
}

int cpbus_stream_fanout_prefix(cpbus_stream_t* st, size_t n, uint64_t now_ns, size_t m) try {
  if (!st || n > st->B || st->get_off > n || m > n - st->get_off) return CPBUS_EINVAL;
  return stream_fanout_prefix(st, n, now_ns, m);
} CPBUS_CATCH

// Every rank (the publisher's included): fan out the next batch of the stream to this GPU's shard.
int cpbus_stream_fanout(cpbus_stream_t* st, size_t n, uint64_t now_ns) try {
  if (!st || n > st->B || st->get_off > n) return CPBUS_EINVAL;
  if (st->bus->lossless) return CPBUS_EINVAL;   // without admission this shard could deliver more than another one does
  return stream_fanout_prefix(st, n, now_ns, n - st->get_off);
} CPBUS_CATCH

// Outstanding follower launches and lossless rounds: one wait on the last of them, then their records in launch order.  A
// launch that delivered moves the stream, the clock and the publish ordinals exactly as cpbus_stream_fanout with the
// header's shape does; an aborted one (and every follower behind it, each a no-op) changes nothing but the sticky error
// word.  A round moves the host state as the host-driven round with the same outcome (cpbus_stream_admit, _offer, _agree,
// then _fanout_prefix of the agreed prefix) would have moved it.
static void round_fold(cpbus* b, const cpbus::FollowPending& f) {
  const volatile RoundRec* r = &b->h_round[f.rec];
  cpbus_stream* st = f.st;
  const uint32_t status = r->status;
  if (status == kFollowAborted || status == kFollowSkipped) return;
  if (r->admit == kRoundAdmitPass) b->st.admit_passes++;
  else if (r->admit == kRoundAdmitSkipped) b->st.admit_skipped++;
  b->room_lb = r->room;
  if (status == kRoundStalled) { st->stalled_rounds++; return; }
  b->st.batches++;
  stream_delivered(b, st, r->m, r->watermark, status == kFollowDelivered, f.launch_seq);
}

static int follow_resolve(cpbus* b) {
  std::lock_guard<std::recursive_mutex> g(b->follow_mu);
  if (b->follow_q.empty()) return CPBUS_OK;
  int rc = dev_guard(b); if (rc) return rc;
  CK(cudaEventRecord(b->follow_done, b->stream));
  CK(cudaEventSynchronize(b->follow_done));
  std::vector<cpbus::FollowPending> q;
  q.swap(b->follow_q);
  bool missing = false;
  for (const cpbus::FollowPending& f : q) {
    if (f.kind == cpbus::kConsumeAll) { b->room_lb = b->R; continue; }
    f.st->follow_out--;
    if (f.kind == cpbus::kRound) {
      if (b->h_round[f.rec].status == kFollowPending) missing = true;
      else round_fold(b, f);
      continue;
    }
    const volatile FollowRec* r = &b->h_follow[f.rec];
    if (r->status == kFollowPending) missing = true;
    if (r->status == kFollowDelivered) stream_delivered(b, f.st, r->n, r->watermark, /*final=*/true, f.launch_seq);
  }
  if (missing) { snprintf(g_cuda_err, sizeof(g_cuda_err), "a follower launch or round completed without its record"); return CPBUS_ECUDA; }
  return CPBUS_OK;
}

// The opening of an enqueue (cpbus_stream_fanout_next, _round_next), under follow_mu: a free record (with kFollowMax
// outstanding, the queue is resolved first), record *ri marked pending.  The first launch after the host has resolved
// (*seed) starts from the host's state, this bus's own staged events flushed first as in the host-driven calls; the ones
// queued behind it take their predecessor's state on the device.
static int follow_begin(cpbus* b, cpbus::FollowKind kind, int* ri, bool* seed) {
  int rc = dev_guard(b); if (rc) return rc;
  if (follow_records(b) >= cpbus::kFollowMax && (rc = follow_resolve(b))) return rc;
  if ((rc = stream_error(b))) return rc;
  *seed = b->follow_q.empty();
  if (*seed && (rc = flush_staged(b, b->now))) return rc;
  *ri = b->follow_next;
  if (kind == cpbus::kRound) b->h_round[*ri].status = kFollowPending;
  else b->h_follow[*ri].status = kFollowPending;
  return CPBUS_OK;
}

// ... and its close: record ri joins the queue, behind the launch that writes it.
static void follow_end(cpbus_stream* st, cpbus::FollowKind kind, int ri) {
  cpbus* b = st->bus;
  b->follow_next = (ri + 1) % cpbus::kFollowMax;
  b->follow_q.push_back(cpbus::FollowPending{st, b->launch_seq, ri, kind});
  st->follow_out++;
}

// Every rank that does not know the batches' shapes: enqueue the fan-out of the stream's next not yet enqueued batch and
// return.  The lead CTA takes n and the watermark from the slot header; the host learns them when it next resolves.
int cpbus_stream_fanout_next(cpbus_stream_t* st) try {
  if (!st) return CPBUS_EINVAL;
  cpbus* b = st->bus;
  if (b->lossless) return CPBUS_EINVAL;   // lossless followers agree on every round, which syncs anyway
  std::lock_guard<std::recursive_mutex> g(b->follow_mu);
  int ri = 0; bool from_host = false;
  int rc = follow_begin(b, cpbus::kFollower, &ri, &from_host); if (rc) return rc;
  StreamArgs sa;
  LaunchOpts o;
  const cpbus_event* src = stream_launch(st, st->get_seq + 1 + st->follow_out, 0, /*final=*/true, sa, o);
  sa.follow_rec = b->d_follow + ri; sa.follow_from_host = from_host;
  if ((rc = launch_fanout(b, src, b->B, b->now, o))) return rc;
  follow_end(st, cpbus::kFollower, ri);
  return CPBUS_OK;
} CPBUS_CATCH

// Lossless stream, one admission round enqueued on the device: decide (one CTA), the exact admission pass (grid; every
// CTA returns at once on the fast path), offer + agree (one CTA), the fan-out of the agreed prefix.  The host learns the
// outcome when it next resolves (follow_resolve), like a follower's.
int cpbus_stream_round_next(cpbus_stream_t* st) try {
  if (!st) return CPBUS_EINVAL;
  cpbus* b = st->bus;
  if (!b->lossless || st->offered) return CPBUS_EINVAL;   // throughput mode needs no agreement; not inside an explicit round
  std::lock_guard<std::recursive_mutex> g(b->follow_mu);
  int ri = 0; bool seed_bus = false;
  int rc = follow_begin(b, cpbus::kRound, &ri, &seed_bus); if (rc) return rc;
  const bool seed_cur = st->follow_out == 0;   // likewise the stream's cursor, while none of this stream's rounds is queued
  RoundParams P{};
  P.dev = b->d_round; P.cur = st->d_cursor; P.rec = b->d_round_rec + ri;
  P.hdr = st->hdr; P.payload = st->payload; P.ack = st->ack;
  P.n_slots = st->n_slots; P.B = st->B; P.consumer = st->consumer; P.n_consumers = st->n_consumers;
  P.round = st->agree_round + 1;
  P.spin_us = b->stream_spin_us; P.err_word = b->d_err;
  P.admit_batch = b->d_admit_batch; P.ctl = b->d_ctl; P.timers = b->d_timers; P.stats = b->d_stats;
  P.pairs = b->n_paired > 0 ? b->d_pairs : nullptr;
  P.n_subs = b->n_next; P.ring_cap = b->R; P.K = b->K; P.sub_base = b->cfg.sub_id_base;
  P.timers_armed = b->n_timers > 0 && b->K > 0;
  P.min_period = b->min_period; P.window = max_window(b);
  P.seed_bus = seed_bus; P.seed_room = b->room_lb; P.seed_now = b->now; P.seed_wm = b->last_watermark;
  P.seed_cur = seed_cur; P.seed_batch = st->get_seq + 1; P.seed_off = st->get_off;
  stream_round_decide_kernel<<<1, kThreads, 0, b->stream>>>(P);
  CK(cudaGetLastError());
  b->st.kernel_launches++;
  if (b->n_next) {
    stream_round_admit_kernel<<<(b->n_next + 255) / 256, 256, 0, b->stream>>>(P);
    CK(cudaGetLastError());
    b->st.kernel_launches++;
  }
  stream_round_agree_kernel<<<1, kStreamMaxConsumers, 0, b->stream>>>(P);
  CK(cudaGetLastError());
  b->st.kernel_launches++;
  st->agree_round = P.round;
  StreamArgs sa;
  sa.ack = &st->ack[4 * st->consumer]; sa.round = b->d_round;
  LaunchOpts o;
  o.staged = 2; o.account = true; o.stream = &sa;
  rc = launch_fanout(b, st->payload, b->B, b->now, o);
  follow_end(st, cpbus::kRound, ri);   // (a failed launch leaves the round's record pending: the next resolution reports it)
  return rc;
} CPBUS_CATCH

int cpbus_stream_progress(cpbus_stream_t* st, uint64_t* batches, size_t* offset, uint64_t* stalled_rounds) try {
  if (!st || !batches || !offset || !stalled_rounds) return CPBUS_EINVAL;
  cpbus* b = st->bus;
  int rc = enter(b); if (rc) return rc;
  *batches = st->get_seq; *offset = st->get_off; *stalled_rounds = st->stalled_rounds;
  return stream_error(b);
} CPBUS_CATCH

// Lossless stream across processes, step 1 of the exchange: post this shard's admitted prefix for the current round.
// One-thread kernel on the bus stream (behind the admission pass when it ran); no host sync.
int cpbus_stream_offer(cpbus_stream_t* st, size_t prefix, int stalled) try {
  if (!st) return CPBUS_EINVAL;
  cpbus* b = st->bus;
  if (!b->lossless || st->offered) return CPBUS_EINVAL;   // throughput mode needs no agreement; one offer per round
  const size_t n = st->admit_q == st->get_seq + 1 ? st->admit_n : st->B;   // the batch's shape when this shard admitted it
  if (prefix > n - st->get_off || (stalled && prefix)) return CPBUS_EINVAL;
  int rc = dev_guard(b); if (rc) return rc;
  if ((rc = stream_error(b))) return rc;
  const unsigned long long r = st->agree_round + 1;
  stream_offer_kernel<<<1, 1, 0, b->stream>>>(st->ack + stream_offer_word_index(st->consumer, r),
                                              stream_offer_word(r, stalled ? 1u : 0u, (uint32_t)prefix));
  CK(cudaGetLastError());
  b->st.kernel_launches++;
  st->offered = true;
  return CPBUS_OK;
} CPBUS_CATCH

// Step 2: wait (in a one-CTA kernel, bounded by the stream timeout) for every shard's offer of this round; *m = the minimum.
// The host waits for that kernel only.  Every call completes the round, whatever it returns.
int cpbus_stream_agree(cpbus_stream_t* st, size_t* m) try {
  if (!st || !m) return CPBUS_EINVAL;
  *m = 0;
  cpbus* b = st->bus;
  if (!b->lossless || !st->offered) return CPBUS_EINVAL;
  int rc = dev_guard(b); if (rc) return rc;
  if ((rc = stream_error(b))) return rc;
  if (!st->h_agree) CK(mapped_alloc(sizeof(StreamAgreeResult), &st->h_agree, &st->d_agree));
  if (!st->agree_done) CK(cudaEventCreateWithFlags(&st->agree_done, cudaEventDisableTiming));
  const unsigned long long r = st->agree_round + 1;
  stream_agree_kernel<<<1, kStreamMaxConsumers, 0, b->stream>>>(st->ack, st->n_consumers, r, b->stream_spin_us, st->d_agree, b->d_err);
  CK(cudaGetLastError());
  b->st.kernel_launches++;
  st->agree_round = r; st->offered = false;
  CK(cudaEventRecord(st->agree_done, b->stream));
  CK(cudaEventSynchronize(st->agree_done));
  const volatile StreamAgreeResult* res = st->h_agree;
  if (res->status) return CPBUS_ETIMEDOUT;   // a shard never offered: the sticky error word is set, nothing goes out
  if (res->stalled) return CPBUS_EAGAIN;
  *m = res->m;
  return CPBUS_OK;
} CPBUS_CATCH

static int read_cursors(cpbus* b, uint32_t l, uint64_t* tail, uint64_t* head, uint64_t* lost = nullptr) {
  SubCtl c{};
  CK(cudaMemcpyAsync(&c, b->d_ctl + l, sizeof(SubCtl), cudaMemcpyDeviceToHost, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  *tail = c.tail;
  // overwrite-oldest: the consumer's cursor can never be older than the oldest record still in the ring
  *head = (!b->lossless && c.tail > b->R && c.tail - b->R > c.head) ? c.tail - b->R : c.head;
  if (lost) *lost = *head - c.head;   // records overwritten since the consumer's stored cursor
  return CPBUS_OK;
}

static int copy_slots(cpbus* b, uint32_t l, uint64_t from, size_t n, cpbus_event* out) {
  const cpbus_event* ring = b->d_ring + (size_t)l * b->R;
  const uint32_t s0 = (uint32_t)(from & (b->R - 1));
  const size_t first = std::min<size_t>(n, b->R - s0);
  if (first) CK(cudaMemcpyAsync(out, ring + s0, first * sizeof(cpbus_event), cudaMemcpyDeviceToHost, b->stream));
  if (n > first) CK(cudaMemcpyAsync(out + first, ring, (n - first) * sizeof(cpbus_event), cudaMemcpyDeviceToHost, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  return CPBUS_OK;
}

int cpbus_drain(cpbus_t* b, uint32_t sub_id, cpbus_event* out, size_t cap, size_t* n, uint64_t* lost) try {
  if (!b || !n || (!out && cap)) return CPBUS_EINVAL;
  const uint32_t l = sub_id - b->cfg.sub_id_base;
  if (sub_id < b->cfg.sub_id_base || l >= b->n_next) return CPBUS_ENOENT;
  std::lock_guard<std::mutex> g(b->mu);
  int rc = enter(b); if (rc) return rc;
  uint64_t tail = 0, head = 0;
  uint64_t gone = 0;
  if ((rc = read_cursors(b, l, &tail, &head, &gone))) return rc;
  if (lost) *lost = gone;
  const size_t take = (size_t)std::min<uint64_t>(tail - head, cap);
  if (take && (rc = copy_slots(b, l, head, take, out))) return rc;
  head += take;
  CK(cudaMemcpyAsync(&b->d_ctl[l].head, &head, 8, cudaMemcpyHostToDevice, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  *n = take;
  return CPBUS_OK;
} CPBUS_CATCH

// Bulk drain: everything undrained in mailboxes [first_sub, first_sub+n) in ONE kernel + two D2H copies.
// out receives the records (each mailbox's run contiguous and FIFO), offsets[i]/counts[i] say where mailbox i's run is.
int cpbus_drain_many(cpbus_t* b, uint32_t first_sub, uint32_t n, cpbus_event* out, size_t cap, uint32_t* offsets,
                     uint32_t* counts, size_t* total) try {
  if (!b || !n || !out || !cap || !offsets || !counts || !total || cap > 0xFFFFFFFFull) return CPBUS_EINVAL;
  const uint32_t l = first_sub - b->cfg.sub_id_base;
  if (first_sub < b->cfg.sub_id_base || (uint64_t)l + n > b->n_next) return CPBUS_ENOENT;
  std::lock_guard<std::mutex> g(b->mu);
  int rc = enter(b); if (rc) return rc;
  if (b->drain_cap < cap || b->drain_idx_cap < n) {   // device staging grows on demand and is kept
    if (b->drain_cap < cap) { cudaFree(b->d_drain); b->d_drain = nullptr; CK(cudaMalloc((void**)&b->d_drain, cap * sizeof(cpbus_event))); b->drain_cap = cap; }
    if (b->drain_idx_cap < n) { cudaFree(b->d_drain_idx); b->d_drain_idx = nullptr; CK(cudaMalloc((void**)&b->d_drain_idx, (size_t)n * sizeof(uint2) + 16)); b->drain_idx_cap = n; }
  }
  unsigned int* cursor = reinterpret_cast<unsigned int*>(b->d_drain_idx + n);
  CK(cudaMemsetAsync(cursor, 0, sizeof(unsigned int), b->stream));
  const uint32_t threads = 256, grid = std::min<uint32_t>((n + 7) / 8, (uint32_t)b->sm_count * 8);
  drain_many_kernel<<<grid, threads, 0, b->stream>>>(b->d_ctl, b->d_ring, l, n, b->R, b->lossless ? 1u : 0u, b->d_drain,
                                                     (uint32_t)cap, b->d_drain_idx, cursor);
  CK(cudaGetLastError());
  b->st.kernel_launches++;
  std::vector<uint2> idx(n);
  CK(cudaMemcpyAsync(idx.data(), b->d_drain_idx, (size_t)n * sizeof(uint2), cudaMemcpyDeviceToHost, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  size_t tot = 0, hi = 0;
  for (uint32_t i = 0; i < n; i++) {
    offsets[i] = idx[i].x; counts[i] = idx[i].y; tot += idx[i].y;
    hi = std::max<size_t>(hi, (size_t)idx[i].x + idx[i].y);
  }
  if (hi) CK(cudaMemcpyAsync(out, b->d_drain, hi * sizeof(cpbus_event), cudaMemcpyDeviceToHost, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  *total = tot;
  return CPBUS_OK;
} CPBUS_CATCH

// Sparse drain: only the mailboxes that hold records.  The scan kernel reads each control block of the range once and
// writes the ready list of the taken prefix; the gather kernel copies their runs and hands the 3-word header to the host
// through mapped pinned memory.  One sync reads the header; a second one follows the two copies sized by it.
// The body of cpbus_drain_ready, without its cap >= ring_cap check: a group hands each shard the cap its earlier shards
// left, which can be smaller.  *all_taken: every ready mailbox of the range was taken (then *next_sub = start_sub).
static int drain_ready_impl(cpbus_t* b, uint32_t first_sub, uint32_t n, uint32_t start_sub, cpbus_event* out, size_t cap,
                            cpbus_ready* ready, size_t ready_cap, size_t* n_ready, size_t* total, uint32_t* next_sub,
                            bool* all_taken);

int cpbus_drain_ready(cpbus_t* b, uint32_t first_sub, uint32_t n, uint32_t start_sub, cpbus_event* out, size_t cap,
                      cpbus_ready* ready, size_t ready_cap, size_t* n_ready, size_t* total, uint32_t* next_sub) try {
  if (!b || !out || !ready || !n_ready || !total || !next_sub || !n || !ready_cap) return CPBUS_EINVAL;
  if (cap < b->R || cap > 0xFFFFFFFFull) return CPBUS_EINVAL;   // cap >= ring_cap: a ready mailbox always fits an empty call
  bool all_taken = false;
  return drain_ready_impl(b, first_sub, n, start_sub, out, cap, ready, ready_cap, n_ready, total, next_sub, &all_taken);
} CPBUS_CATCH

static int drain_ready_impl(cpbus_t* b, uint32_t first_sub, uint32_t n, uint32_t start_sub, cpbus_event* out, size_t cap,
                            cpbus_ready* ready, size_t ready_cap, size_t* n_ready, size_t* total, uint32_t* next_sub,
                            bool* all_taken) {
  if (start_sub < first_sub || start_sub - first_sub >= n) return CPBUS_EINVAL;
  const uint32_t l = first_sub - b->cfg.sub_id_base;
  if (first_sub < b->cfg.sub_id_base || (uint64_t)l + n > b->n_next) return CPBUS_ENOENT;
  std::lock_guard<std::mutex> g(b->mu);
  int rc = enter(b); if (rc) return rc;
  const size_t rcap = std::min<size_t>(ready_cap, n);   // never more entries than mailboxes
  const uint32_t tiles = (n + kReadyTile - 1) / kReadyTile;
  // device staging grows on demand and is kept (the records share cpbus_drain_many's buffer)
  if (b->drain_cap < cap) {
    cudaFree(b->d_drain); b->d_drain = nullptr; b->drain_cap = 0;
    CK(cudaMalloc((void**)&b->d_drain, cap * sizeof(cpbus_event))); b->drain_cap = cap;
  }
  if (b->ready_stage_cap < rcap) {
    cudaFree(b->d_ready); cudaFree(b->d_ready_slot); b->d_ready = nullptr; b->d_ready_slot = nullptr; b->ready_stage_cap = 0;
    CK(cudaMalloc((void**)&b->d_ready, rcap * sizeof(cpbus_ready)));
    CK(cudaMalloc((void**)&b->d_ready_slot, rcap * sizeof(uint32_t)));
    b->ready_stage_cap = rcap;
  }
  if (b->ready_lb_tiles < tiles) {
    cudaFree(b->d_ready_lb); b->d_ready_lb = nullptr; b->ready_lb_tiles = 0;
    CK(cudaMalloc((void**)&b->d_ready_lb, (kReadyLbOffset + (size_t)tiles) * sizeof(unsigned long long)));
    b->ready_lb_tiles = tiles;
  }
  if (!b->h_ready_hdr) CK(mapped_alloc(64, &b->h_ready_hdr, &b->d_ready_hdr));
  CK(cudaMemsetAsync(b->d_ready_lb + kReadyHdrWords, 0, (kReadyLbOffset - kReadyHdrWords + (size_t)tiles) * sizeof(unsigned long long),
                     b->stream));
  const uint32_t rot = start_sub - first_sub;
  drain_ready_scan_kernel<<<tiles, kThreads, 0, b->stream>>>(b->d_ctl, l, n, rot, b->R, b->lossless ? 1u : 0u, b->cfg.sub_id_base,
                                                              cap, rcap, b->d_ready_lb, b->d_ready, b->d_ready_slot);
  CK(cudaGetLastError());
  const uint32_t gather_grid = (uint32_t)std::min<size_t>((size_t)b->sm_count * 4, (rcap + kWarpsPerCta - 1) / kWarpsPerCta);
  drain_ready_gather_kernel<<<gather_grid, kThreads, 0, b->stream>>>(b->d_ring, b->R, b->cfg.sub_id_base, b->d_ready,
                                                                      b->d_ready_slot, b->d_ready_lb, b->d_drain, b->d_ready_hdr);
  CK(cudaGetLastError());
  b->st.kernel_launches += 2;
  CK(cudaStreamSynchronize(b->stream));
  const size_t nr = (size_t)b->h_ready_hdr[0], tot = (size_t)b->h_ready_hdr[1];
  const uint64_t cut = b->h_ready_hdr[2];
  if (nr) {
    CK(cudaMemcpyAsync(ready, b->d_ready, nr * sizeof(cpbus_ready), cudaMemcpyDeviceToHost, b->stream));
    CK(cudaMemcpyAsync(out, b->d_drain, tot * sizeof(cpbus_event), cudaMemcpyDeviceToHost, b->stream));
    CK(cudaStreamSynchronize(b->stream));
  }
  *n_ready = nr; *total = tot;
  *all_taken = cut >= n;
  *next_sub = cut >= n ? start_sub : first_sub + (uint32_t)((rot + cut) % n);
  return CPBUS_OK;
}

// Device-side consumer: every mailbox of this shard is read to the end and its records are discarded.
int cpbus_consume_all(cpbus_t* b) try {
  if (!b) return CPBUS_EINVAL;
  std::lock_guard<std::mutex> g(b->mu);
  int rc = dev_guard(b); if (rc) return rc;
  std::lock_guard<std::recursive_mutex> gf(b->follow_mu);
  // Behind outstanding lossless rounds (the only thing a lossless bus queues) it does not wait: it is ordered behind them
  // on the bus stream, resets the device room bound there, and joins the queue so that resolution resets the host's in order.
  const bool behind_rounds = b->lossless && !b->follow_q.empty();
  if (!behind_rounds && (rc = follow_resolve(b))) return rc;
  if (b->n_next) {
    const uint32_t threads = 256, grid = std::min<uint32_t>((b->n_next + threads - 1) / threads, (uint32_t)b->sm_count * 8);
    consume_all_kernel<<<grid, threads, 0, b->stream>>>(b->d_ctl, b->n_next);
    CK(cudaGetLastError());
    b->st.kernel_launches++;
  }
  if (behind_rounds) {
    CK(cudaMemcpyAsync(&b->d_round->room, &b->d_round->room_full, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, b->stream));
    b->follow_q.push_back(cpbus::FollowPending{nullptr, 0ull, -1, cpbus::kConsumeAll});
  }
  b->room_lb = b->R;   // stream-ordered behind every earlier fan-out: from here on every mailbox is empty
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_peek_window(cpbus_t* b, uint32_t sub_id, cpbus_event* out, size_t cap, size_t* n) try {
  if (!b || !n || (!out && cap)) return CPBUS_EINVAL;
  const uint32_t l = sub_id - b->cfg.sub_id_base;
  if (sub_id < b->cfg.sub_id_base || l >= b->n_next) return CPBUS_ENOENT;
  std::lock_guard<std::mutex> g(b->mu);
  int rc = enter(b); if (rc) return rc;
  uint64_t tail = 0, head = 0;
  if ((rc = read_cursors(b, l, &tail, &head))) return rc;
  const size_t take = (size_t)std::min<uint64_t>(std::min<uint64_t>(tail, b->R), cap);
  if (take && (rc = copy_slots(b, l, tail - take, take, out))) return rc;
  *n = take;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_digest(cpbus_t* b, uint32_t first_sub, uint32_t n, cpbus_digest_t* out) try {
  if (!b || !out || !n) return CPBUS_EINVAL;
  const uint32_t l = first_sub - b->cfg.sub_id_base;
  if (first_sub < b->cfg.sub_id_base || (uint64_t)l + n > b->n_next) return CPBUS_ENOENT;
  std::lock_guard<std::mutex> g(b->mu);
  int rc = enter(b); if (rc) return rc;
  std::vector<SubCtl> c(n);
  CK(cudaMemcpyAsync(c.data(), b->d_ctl + l, (size_t)n * sizeof(SubCtl), cudaMemcpyDeviceToHost, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  for (uint32_t i = 0; i < n; i++) { out[i].count = c[i].tail; out[i].digest = c[i].digest; }
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_digest_fold_begin(cpbus_t* b, uint32_t first_sub, uint32_t n, uint32_t* ticket) try {
  if (!b || !ticket || !n) return CPBUS_EINVAL;
  const uint32_t l = first_sub - b->cfg.sub_id_base;
  if (first_sub < b->cfg.sub_id_base || (uint64_t)l + n > b->n_next) return CPBUS_ENOENT;
  std::lock_guard<std::mutex> g(b->mu);
  int rc = dev_guard(b); if (rc) return rc;
  const uint32_t slot = b->fold_next++ % cpbus::kFoldSlots;
  unsigned long long* d = b->d_fold + 4 * slot;
  CK(cudaMemsetAsync(d, 0, 32, b->stream));
  const uint32_t threads = 256, grid = std::min<uint32_t>((n + threads - 1) / threads, (uint32_t)b->sm_count * 4);
  digest_fold_kernel<<<grid, threads, 0, b->stream>>>(b->d_ctl, l, n, b->cfg.sub_id_base, d);
  CK(cudaGetLastError());
  b->st.kernel_launches++;
  CK(cudaMemcpyAsync(b->h_fold + 4 * slot, d, 32, cudaMemcpyDeviceToHost, b->stream));
  CK(cudaEventRecord(b->fold_done[slot], b->stream));
  *ticket = slot;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_digest_fold_end(cpbus_t* b, uint32_t ticket, uint64_t out[4]) try {
  if (!b || !out || ticket >= (uint32_t)cpbus::kFoldSlots) return CPBUS_EINVAL;
  int rc = dev_guard(b); if (rc) return rc;
  CK(cudaEventSynchronize(b->fold_done[ticket]));
  for (int i = 0; i < 4; i++) out[i] = b->h_fold[4 * ticket + i];
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_digest_fold(cpbus_t* b, uint32_t first_sub, uint32_t n, uint64_t out[4]) try {
  uint32_t ticket = 0;
  int rc = b ? follow_resolve(b) : CPBUS_OK;
  if (rc) return rc;
  rc = cpbus_digest_fold_begin(b, first_sub, n, &ticket);
  return rc ? rc : cpbus_digest_fold_end(b, ticket, out);
} CPBUS_CATCH

// The fan-out kernel leaves {deliveries, ticks, sum of the new digests} of each launch in a small ring;
// reading a step's result therefore costs one 256-byte D2H and no extra kernel.
int cpbus_step_result_begin(cpbus_t* b, uint32_t* ticket) try {
  if (!b || !ticket) return CPBUS_EINVAL;
  std::lock_guard<std::mutex> g(b->mu);
  int rc = dev_guard(b); if (rc) return rc;
  const uint32_t t = b->result_next++ % 8;
  const DevResultSlot* src = b->d_result + (size_t)(b->launch_seq % kResultRing) * kResultSub;
  // read it on a side stream, behind an event recorded after the launch: neither the next fan-out nor the next batch's
  // H2D queues behind this D2H
  CK(cudaEventRecord(b->launched, b->stream));
  CK(cudaStreamWaitEvent(b->result_stream, b->launched, 0));
  CK(cudaMemcpyAsync(b->h_result + (size_t)t * kResultSub, src, sizeof(DevResultSlot) * kResultSub, cudaMemcpyDeviceToHost, b->result_stream));
  CK(cudaEventRecord(b->result_done[t], b->result_stream));
  *ticket = t;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_step_result_end(cpbus_t* b, uint32_t ticket, uint64_t out[4]) try {
  if (!b || !out || ticket >= 8) return CPBUS_EINVAL;
  int rc = dev_guard(b); if (rc) return rc;
  CK(cudaEventSynchronize(b->result_done[ticket]));
  out[0] = out[1] = out[2] = out[3] = 0;
  for (int i = 0; i < kResultSub; i++) {
    const DevResultSlot& r = b->h_result[(size_t)ticket * kResultSub + i];
    out[0] += r.deliveries; out[1] += r.ticks; out[2] += r.digest_sum; out[3] += r.launch_seq;
  }
  return CPBUS_OK;
} CPBUS_CATCH

// DebugEvents — events/bus.go:34-54
// Broadcast events of device-published batches join the debug ring here, in publish order (the kernel's lead CTA kept
// the last 10 of each such batch; launches older than kAcctDbgRing are no longer resolvable and are skipped).
static int dbg_resolve(cpbus* b) {
  if (b->dbg_pending.empty()) return CPBUS_OK;
  bool any_marker = false;
  for (const DbgItem& it : b->dbg_pending) any_marker |= it.marker;
  if (any_marker) {
    int rc = dev_guard(b); if (rc) return rc;
    CK(cudaMemcpyAsync(b->h_acct->tail, b->d_acct->tail, sizeof(b->h_acct->tail), cudaMemcpyDeviceToHost, b->stream));
    CK(cudaStreamSynchronize(b->stream));
  }
  for (const DbgItem& it : b->dbg_pending) {
    if (!it.marker) { dbg_ring_put(b, it.ev); continue; }
    const DevDbgTail& t = b->h_acct->tail[it.launch % kAcctDbgRing];
    if (t.launch_seq != it.launch) continue;
    for (uint32_t j = 0; j < t.n_kept && j < (uint32_t)kAcctDbgKeep; j++) dbg_ring_put(b, t.ev[j]);
  }
  b->dbg_pending.clear();
  return CPBUS_OK;
}

int cpbus_debug_events(cpbus_t* b, cpbus_event* out, size_t cap, size_t* n) try {
  if (!b || !n || (!out && cap)) return CPBUS_EINVAL;
  { const int rc = follow_resolve(b); if (rc) return rc; }
  { const int rc = dbg_resolve(b); if (rc) return rc; }
  size_t k = 0;
  for (;;) {
    if (b->dbg_head == -1) break;
    const cpbus_event e = b->dbg[b->dbg_tail % 10];
    if (b->dbg_tail == b->dbg_head) { b->dbg_head = -1; b->dbg_tail = 0; }
    else b->dbg_tail = (b->dbg_tail + 1) % 10;
    if (e.code == CPBUS_NONE && e.source_id == 0) break;   // == NonEvent
    if (k < cap) out[k] = e;
    k++;
  }
  *n = k;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_stats(cpbus_t* b, cpbus_stats_t* out) try {
  if (!b || !out) return CPBUS_EINVAL;
  std::lock_guard<std::mutex> g(b->mu);
  int rc = enter(b); if (rc) return rc;
  CK(cudaMemsetAsync(&b->d_stats->overwritten, 0, sizeof(unsigned long long), b->stream));
  if (!b->lossless && b->n_next) {
    const uint32_t threads = 256, grid = std::min<uint32_t>((b->n_next + threads - 1) / threads, (uint32_t)b->sm_count * 4);
    overwritten_kernel<<<grid, threads, 0, b->stream>>>(b->d_ctl, b->n_next, b->R, &b->d_stats->overwritten);
    CK(cudaGetLastError());
  }
  CK(cudaMemcpyAsync(b->h_stats, b->d_stats, sizeof(DevStats), cudaMemcpyDeviceToHost, b->stream));
  CK(cudaMemcpyAsync(b->h_acct->by_code, b->d_acct->by_code, sizeof(b->h_acct->by_code), cudaMemcpyDeviceToHost, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  retire_oneshots(b, b->last_watermark);
  b->st.deliveries = b->st.ticks = 0;
  b->st.overwritten = b->h_stats->overwritten;
  for (int i = 0; i < kStatSlots; i++) { b->st.deliveries += b->h_stats->slot[i].deliveries; b->st.ticks += b->h_stats->slot[i].ticks; }
  b->st.n_subs = b->n_active; b->st.n_timers = b->n_timers; b->st.now_ns = b->now;
  b->st.intern_entries = b->sources.size(); b->st.intern_bytes = b->intern_bytes;
  b->st.ephemeral_live = b->eph_live; b->st.ephemeral_recycled = b->eph_recycled;
  *out = b->st;
  for (int c = 0; c < CPBUS_N_CODES; c++) out->published_by_code[c] += b->h_acct->by_code[c];   // device-published batches (kernel-counted)
  return CPBUS_OK;
} CPBUS_CATCH

// containerpilot_events{code, source} (events/bus.go:60-68,130-132): host publishes are counted in cpbus_publish, batches
// that arrive in device memory by the fan-out kernel's lead CTA (DevPubAcct).
int cpbus_publish_counts(cpbus_t* b, cpbus_pair_count* out, size_t cap, size_t* n) try {
  if (!b || !n || (!out && cap)) return CPBUS_EINVAL;
  std::lock_guard<std::mutex> g(b->mu);
  int rc = enter(b); if (rc) return rc;
  std::unordered_map<uint64_t, uint64_t> merged;
  for (size_t i = 0; i < b->pub_pairs.keys.size(); i++) if (b->pub_pairs.keys[i]) merged[b->pub_pairs.keys[i] - 1] += b->pub_pairs.cnts[i];
  if (b->launch_seq) {
    std::vector<unsigned long long> keys(kAcctPairSlots), cnts(kAcctPairSlots);
    CK(cudaMemcpyAsync(keys.data(), b->d_acct->pair_key, sizeof(unsigned long long) * kAcctPairSlots, cudaMemcpyDeviceToHost, b->stream));
    CK(cudaMemcpyAsync(cnts.data(), b->d_acct->pair_cnt, sizeof(unsigned long long) * kAcctPairSlots, cudaMemcpyDeviceToHost, b->stream));
    CK(cudaStreamSynchronize(b->stream));
    for (uint32_t i = 0; i < kAcctPairSlots; i++) if (keys[i]) merged[keys[i] - 1] += cnts[i];
  }
  std::vector<std::pair<uint64_t, uint64_t>> v(merged.begin(), merged.end());
  std::sort(v.begin(), v.end());
  for (size_t i = 0; i < v.size() && i < cap; i++) out[i] = cpbus_pair_count{(uint32_t)(v[i].first >> 32), (uint32_t)v[i].first, v[i].second};
  *n = v.size();
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_device_ptrs(cpbus_t* b, void** ring, void** ctl) try {
  if (!b) return CPBUS_EINVAL;
  if (ring) *ring = b->d_ring;
  if (ctl) *ctl = b->d_ctl;
  return CPBUS_OK;
} CPBUS_CATCH

// ---- the group: one bus handle over the GPUs of a box (include/cpbus.h: cpbus_group_*) ----------------------------------
// The group keeps the host state a single bus keeps for the whole id space — staged records, seq, clock, last launched
// watermark, the timer table that sets the clock window, debug ring and publish counts — and makes the flushes the single
// bus makes (flush_staged, stage_one, cpbus_advance).  A flush becomes one RAW stream batch that every shard fans out in
// full: in lossless mode the group first runs the single bus's admission (admit) on every shard and puts only the prefix
// every shard can take, with the single bus's partial watermark.  (cpbus_stream_admit would hold a batch back until the
// ticks due by its watermark fit too, where a partial cpbus_flush delivers the records and stalls on the ticks alone.)
// Shard clocks: a shard's clock is its last launched watermark; a shard without timers is moved to the group clock with
// cpbus_advance right before a timer is armed on it (no launch: it has no timer window), so every shard's `now + period`
// is the single bus's.  A shard with timers already has the group clock there (the group has just flushed at `now`).
struct cpbus_group {
  std::vector<cpbus*> shards;
  std::vector<cpbus_stream*> streams;   // streams[0] owns the ring (shard 0), the others are attached
  std::vector<uint32_t> first;          // global index (sub_id_base not applied) of each shard's subscriber 0; + a sentinel
  uint32_t base = 0, N = 0, B = 0, K = 0;
  bool lossless = false;
  uint32_t n_next = 0, n_active = 0;
  std::vector<cpbus_event> staged;      // B records
  size_t n_staged = 0;
  uint64_t now = 0, last_watermark = 0, seq = 0;
  // the single bus's timer bookkeeping over global slots (subscriber * K + k): what sets the clock window and when an empty
  // flush launches
  struct Slot { bool active = false, oneshot = false; uint64_t next_due = 0; };
  std::vector<Slot> timers;             // N * K, allocated on first use (as the single bus's h_timers)
  std::vector<size_t> oneshot_idx;
  uint32_t n_timers = 0;
  uint64_t min_period = UINT64_MAX;
  int dbg_head = -1, dbg_tail = 0;
  cpbus_event dbg[10]{};
  PairCounter pub_pairs;
  uint64_t publishes = 0, by_code[CPBUS_N_CODES] = {};
};

static uint32_t group_shard_of(const cpbus_group* g, uint32_t index) {   // index < N
  return (uint32_t)(std::upper_bound(g->first.begin(), g->first.end(), index) - g->first.begin()) - 1;
}

static uint64_t group_window(const cpbus_group* g) {   // max_window of the single bus
  if (!g->K || g->n_timers == 0 || g->min_period == UINT64_MAX) return UINT64_MAX;
  const uint64_t J = 32u / g->K;
  return g->min_period > UINT64_MAX / J ? UINT64_MAX : g->min_period * J;
}

// retire_oneshots of the single bus, for the group's table and, at the same moment, every shard's own: a shard's timer
// count (and so its window) then never lags the group's
static void group_retire(cpbus_group* g) {
  size_t keep = 0;
  for (size_t i = 0; i < g->oneshot_idx.size(); i++) {
    cpbus_group::Slot& t = g->timers[g->oneshot_idx[i]];
    if (t.active && t.oneshot && oneshot_fired(t.next_due, g->last_watermark)) { t.active = false; g->n_timers--; continue; }
    if (t.active && t.oneshot) g->oneshot_idx[keep++] = g->oneshot_idx[i];
  }
  g->oneshot_idx.resize(keep);
  if (g->n_timers == 0) g->min_period = UINT64_MAX;
  for (cpbus* s : g->shards) if (!s->h_timers.empty()) retire_oneshots(s, s->last_watermark);
}

// One launch of the single bus: the same early returns as launch_fanout, otherwise one stream batch on every shard.
static int group_launch(cpbus_group* g, const cpbus_event* ev, uint32_t n, uint64_t w) {
  if (g->n_next == 0) return CPBUS_OK;
  if (n == 0 && g->n_timers == 0) return CPBUS_OK;
  int rc = cpbus_stream_put(g->streams[0], ev, n, w, CPBUS_PUT_RAW);
  if (rc) return rc;
  for (cpbus_stream* st : g->streams)   // the whole batch: already admitted on every shard, so it completes in one launch
    if ((rc = cpbus_stream_fanout_prefix(st, n, w, n))) return rc;
  g->last_watermark = w;
  return CPBUS_OK;
}

// Lossless admission of the staged records on every shard (admit), the single bus's verdict being the conjunction and its
// prefix the minimum.  The records reach a shard's device only when its room bound cannot prove the fit.
static int group_admit(cpbus_group* g, uint32_t n, uint64_t w, bool* ok, uint32_t* m) {
  *ok = true; *m = n;
  for (cpbus* s : g->shards) {
    if (admit_fits(s, n, w)) continue;
    int rc = dev_guard(s); if (rc) return rc;
    if (n) CK(cudaMemcpyAsync(s->d_admit_batch, g->staged.data(), (size_t)n * sizeof(cpbus_event), cudaMemcpyHostToDevice, s->stream));
    bool ok_s = true;
    uint32_t m_s = n;
    if ((rc = admit_pass(s, s->d_admit_batch, n, w, &ok_s, &m_s))) return rc;
    if (!ok_s) { *ok = false; *m = std::min(*m, m_s); }
  }
  return CPBUS_OK;
}

// flush_staged of the single bus
static int group_flush(cpbus_group* g, uint64_t w) {
  const uint32_t n = (uint32_t)g->n_staged;
  if (n == 0 && g->n_timers == 0) { g->last_watermark = std::max(g->last_watermark, w); return CPBUS_OK; }
  if (n == 0 && w == g->last_watermark) return CPBUS_OK;
  bool ok = true;
  uint32_t m = n;
  int rc;
  if (g->lossless && (rc = group_admit(g, n, w, &ok, &m))) return rc;
  if (!ok) {
    if (m == 0) return CPBUS_EAGAIN;
    if ((rc = group_launch(g, g->staged.data(), m, g->staged[m - 1].ts_ns))) return rc;
    std::copy(g->staged.begin() + m, g->staged.begin() + n, g->staged.begin());
    g->n_staged = n - m;
    for (cpbus* s : g->shards) { s->room_lb = 0; s->st.admit_partial++; }
    return CPBUS_EAGAIN;
  }
  if ((rc = group_launch(g, g->staged.data(), n, w))) return rc;
  g->n_staged = 0;
  return CPBUS_OK;
}

// stage_one of the single bus: seq is one ordinal over publishes and sends
static int group_stage(cpbus_group* g, uint32_t code, uint32_t source_id, uint32_t target, uint32_t flags) {
  if (g->n_staged == g->B) { const int rc = group_flush(g, g->now); if (rc) return rc; }
  cpbus_event& e = g->staged[g->n_staged++];
  e.seq = g->seq++; e.ts_ns = g->now; e.code = code; e.source_id = source_id; e.target = target; e.flags = flags;
  return CPBUS_OK;
}

// the owning shard of global id `sub_id` and its local index; false: not a subscribed-so-far id
static bool group_locate(const cpbus_group* g, uint32_t sub_id, cpbus** s, uint32_t* l) {
  const uint32_t i = sub_id - g->base;
  if (sub_id < g->base || i >= g->n_next) return false;
  const uint32_t k = group_shard_of(g, i);
  *s = g->shards[k]; *l = i - g->first[k];
  return true;
}

// Arm timers on shard s: a shard without timers takes the group clock first (cpbus_advance launches nothing there).
static int group_shard_clock(cpbus_group* g, cpbus* s) {
  if (s->now == g->now) return CPBUS_OK;
  if (s->n_timers) return CPBUS_ECUDA;   // cannot happen: the group has just flushed at now, which moved this shard there
  return cpbus_advance(s, g->now);
}

int cpbus_group_destroy(cpbus_group_t* g) try {
  if (!g) return CPBUS_EINVAL;
  for (size_t i = g->streams.size(); i-- > 0;) if (g->streams[i]) cpbus_stream_close(g->streams[i]);   // importers first
  for (cpbus* s : g->shards) if (s) cpbus_destroy(s);
  delete g;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_create(const cpbus_config* cfg, const int32_t* devices, uint32_t n_devices, cpbus_group_t** out) try {
  if (!cfg || !devices || !n_devices || !out || cfg->stream || n_devices > kStreamMaxConsumers) return CPBUS_EINVAL;
  *out = nullptr;
  uint32_t R = 0, B = 0;
  if (config_check(cfg, &R, &B) || cfg->n_max_subs < n_devices) return CPBUS_EINVAL;
  cpbus_group* g = new (std::nothrow) cpbus_group();
  if (!g) return CPBUS_ENOMEM;
  g->base = cfg->sub_id_base; g->N = cfg->n_max_subs; g->B = B; g->K = cfg->timers_per_sub;
  g->lossless = cfg->flags & CPBUS_CFG_LOSSLESS;
  g->staged.resize(B);
  auto fail = [&](int code) { cpbus_group_destroy(g); return code; };
  const uint32_t each = g->N / n_devices, extra = g->N % n_devices;   // sharding.shard_range
  for (uint32_t k = 0; k < n_devices; k++) {
    const uint32_t first = k * each + std::min(k, extra), count = each + (k < extra ? 1u : 0u);
    cpbus_config c = *cfg;
    c.n_max_subs = count; c.device = devices[k]; c.sub_id_base = g->base + first;
    cpbus* s = nullptr;
    const int rc = cpbus_create(&c, &s);
    if (rc) return fail(rc);
    g->shards.push_back(s); g->first.push_back(first);
  }
  g->first.push_back(g->N);
  unsigned char handle[64];
  cpbus_stream* st0 = nullptr;
  int rc = cpbus_stream_create(g->shards[0], 8, n_devices, &st0, handle);
  if (rc) return fail(rc);
  g->streams.push_back(st0);
  for (uint32_t k = 1; k < n_devices; k++) {
    cpbus_stream* st = nullptr;
    if ((rc = cpbus_stream_attach(g->shards[k], st0, k, &st))) return fail(rc);
    g->streams.push_back(st);
  }
  *out = g;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_intern(cpbus_group_t* g, const char* s, size_t len, uint32_t* source_id) try {
  return g ? cpbus_intern(g->shards[0], s, len, source_id) : CPBUS_EINVAL;
} CPBUS_CATCH
int cpbus_group_intern_ephemeral(cpbus_group_t* g, const char* s, size_t len, uint32_t* source_id) try {
  return g ? cpbus_intern_ephemeral(g->shards[0], s, len, source_id) : CPBUS_EINVAL;
} CPBUS_CATCH
int cpbus_group_source(cpbus_group_t* g, uint32_t source_id, char* out, size_t cap, size_t* len) try {
  return g ? cpbus_source(g->shards[0], source_id, out, cap, len) : CPBUS_EINVAL;
} CPBUS_CATCH

// Subscribers [n_next, n_next + n) across the shards that own them; fn(shard, offset into the caller's arrays, count).
extern "C++" {
template <class Fn>
static int group_each_range(cpbus_group* g, uint32_t first_index, uint32_t n, Fn&& fn) {
  for (uint32_t done = 0; done < n;) {
    const uint32_t i = first_index + done, k = group_shard_of(g, i);
    const uint32_t cnt = std::min(n - done, g->first[k + 1] - i);
    const int rc = fn(g->shards[k], i - g->first[k], done, cnt);
    if (rc) return rc;
    done += cnt;
  }
  return CPBUS_OK;
}
}

int cpbus_group_subscribe_many(cpbus_group_t* g, const uint32_t* masks, uint32_t n, uint32_t* first_sub_id) try {
  if (!g || !n) return CPBUS_EINVAL;
  if ((uint64_t)g->n_next + n > g->N) return CPBUS_ENOSPC;
  int rc = group_flush(g, g->now); if (rc) return rc;
  const uint32_t first = g->n_next;
  rc = group_each_range(g, first, n, [&](cpbus* s, uint32_t, uint32_t off, uint32_t cnt) -> int {
    uint32_t id = 0;
    return cpbus_subscribe_many(s, masks ? masks + off : nullptr, cnt, &id);
  });
  if (rc) return rc;
  g->n_next += n; g->n_active += n;
  if (first_sub_id) *first_sub_id = g->base + first;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_subscribe(cpbus_group_t* g, uint32_t mask, uint32_t* sub_id) { return cpbus_group_subscribe_many(g, &mask, 1, sub_id); }

int cpbus_group_subscribe_pairs(cpbus_group_t* g, uint32_t mask, const cpbus_pair* pairs, uint32_t n_pairs, uint32_t* sub_id) try {
  if (!g || n_pairs > CPBUS_MAX_PAIRS || (n_pairs && !pairs)) return CPBUS_EINVAL;
  for (uint32_t j = 0; j < n_pairs; j++) if (pairs[j].code >= CPBUS_N_CODES) return CPBUS_EINVAL;
  if (g->n_next >= g->N) return CPBUS_ENOSPC;
  int rc = group_flush(g, g->now); if (rc) return rc;
  const uint32_t k = group_shard_of(g, g->n_next);
  uint32_t id = 0;
  if ((rc = cpbus_subscribe_pairs(g->shards[k], mask, pairs, n_pairs, &id))) return rc;
  g->n_next++; g->n_active++;
  if (sub_id) *sub_id = id;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_subscribe_pairs_many(cpbus_group_t* g, const uint32_t* masks, const cpbus_pair* pairs, const uint32_t* n_pairs,
                                     uint32_t n, uint32_t* first_sub_id) try {
  if (!g || !n || !masks || !pairs || !n_pairs) return CPBUS_EINVAL;
  for (uint32_t i = 0; i < n; i++) {
    if (n_pairs[i] > CPBUS_MAX_PAIRS) return CPBUS_EINVAL;
    for (uint32_t j = 0; j < n_pairs[i]; j++) if (pairs[(size_t)i * CPBUS_MAX_PAIRS + j].code >= CPBUS_N_CODES) return CPBUS_EINVAL;
  }
  if ((uint64_t)g->n_next + n > g->N) return CPBUS_ENOSPC;
  int rc = group_flush(g, g->now); if (rc) return rc;
  const uint32_t first = g->n_next;
  rc = group_each_range(g, first, n, [&](cpbus* s, uint32_t, uint32_t off, uint32_t cnt) -> int {
    uint32_t id = 0;
    return cpbus_subscribe_pairs_many(s, masks + off, pairs + (size_t)off * CPBUS_MAX_PAIRS, n_pairs + off, cnt, &id);
  });
  if (rc) return rc;
  g->n_next += n; g->n_active += n;
  if (first_sub_id) *first_sub_id = g->base + first;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_unsubscribe(cpbus_group_t* g, uint32_t sub_id) try {
  if (!g) return CPBUS_EINVAL;
  cpbus* s = nullptr; uint32_t l = 0;
  if (!group_locate(g, sub_id, &s, &l)) return CPBUS_ENOENT;
  int rc = group_flush(g, g->now); if (rc) return rc;
  if ((rc = cpbus_unsubscribe(s, sub_id))) return rc;
  if (g->K && !g->timers.empty())
    for (uint32_t k = 0; k < g->K; k++) {
      cpbus_group::Slot& t = g->timers[(size_t)(sub_id - g->base) * g->K + k];
      if (t.active) { t.active = false; g->n_timers--; }
    }
  g->n_active--;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_set_mask(cpbus_group_t* g, uint32_t sub_id, uint32_t mask) try {
  if (!g) return CPBUS_EINVAL;
  cpbus* s = nullptr; uint32_t l = 0;
  if (!group_locate(g, sub_id, &s, &l)) return CPBUS_ENOENT;
  if (!s->h_active[l]) return CPBUS_ECLOSED;
  const int rc = group_flush(g, g->now); if (rc) return rc;
  return cpbus_set_mask(s, sub_id, mask);
} CPBUS_CATCH

int cpbus_group_timer_add(cpbus_group_t* g, uint32_t sub_id, uint64_t period_ns, uint32_t source_id, int oneshot, uint32_t* timer_id) try {
  if (!g || !period_ns) return CPBUS_EINVAL;
  if (!g->K) return CPBUS_ENOSPC;
  cpbus* s = nullptr; uint32_t l = 0;
  if (!group_locate(g, sub_id, &s, &l)) return CPBUS_ENOENT;
  int rc = group_flush(g, g->now); if (rc) return rc;
  if (g->timers.empty()) g->timers.resize((size_t)g->N * g->K);
  group_retire(g);
  if (!s->h_active[l]) return CPBUS_ECLOSED;
  if ((rc = group_shard_clock(g, s))) return rc;
  uint32_t id = 0;
  if ((rc = cpbus_timer_add(s, sub_id, period_ns, source_id, oneshot, &id))) return rc;
  const uint32_t shard_base_slot = (sub_id - l - g->base) * g->K;   // global slot of the shard's slot 0
  const size_t slot = (size_t)(id & kTimerSlotMask) + shard_base_slot;
  cpbus_group::Slot& t = g->timers[slot];
  t.active = true; t.oneshot = oneshot != 0; t.next_due = due_after(g->now, period_ns);
  g->n_timers++;
  if (!oneshot) g->min_period = std::min(g->min_period, period_ns);
  else g->oneshot_idx.push_back(slot);
  if (timer_id) *timer_id = (uint32_t)slot | (id & ~kTimerSlotMask);
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_timer_add_many(cpbus_group_t* g, uint32_t first_sub, uint32_t n, uint64_t period_ns, const uint32_t* source_ids,
                               uint32_t source_id0, int oneshot) try {
  if (!g || !period_ns || !n) return CPBUS_EINVAL;
  if (!g->K) return CPBUS_ENOSPC;
  const uint32_t i0 = first_sub - g->base;
  if (first_sub < g->base || (uint64_t)i0 + n > g->n_next) return CPBUS_ENOENT;
  int rc = group_flush(g, g->now); if (rc) return rc;
  if (g->timers.empty()) g->timers.resize((size_t)g->N * g->K);
  group_retire(g);
  // the single bus checks every subscriber before it arms any
  for (uint32_t i = 0; i < n; i++) {
    cpbus* s = nullptr; uint32_t l = 0;
    group_locate(g, first_sub + i, &s, &l);
    if (!s->h_active[l]) return CPBUS_ECLOSED;
    if (g->timers[(size_t)(i0 + i) * g->K].active) return CPBUS_ENOSPC;
  }
  rc = group_each_range(g, i0, n, [&](cpbus* s, uint32_t l, uint32_t off, uint32_t cnt) -> int {
    const int rc_clock = group_shard_clock(g, s);
    if (rc_clock) return rc_clock;
    return cpbus_timer_add_many(s, s->cfg.sub_id_base + l, cnt, period_ns, source_ids ? source_ids + off : nullptr,
                                source_id0 + off, oneshot);
  });
  if (rc) return rc;
  for (uint32_t i = 0; i < n; i++) {
    const size_t slot = (size_t)(i0 + i) * g->K;
    cpbus_group::Slot& t = g->timers[slot];
    t.active = true; t.oneshot = oneshot != 0; t.next_due = due_after(g->now, period_ns);
    if (oneshot) g->oneshot_idx.push_back(slot);
  }
  g->n_timers += n;
  if (!oneshot) g->min_period = std::min(g->min_period, period_ns);
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_timer_cancel(cpbus_group_t* g, uint32_t timer_id) try {
  if (!g) return CPBUS_EINVAL;
  if (!g->K || g->timers.empty()) return CPBUS_ENOENT;
  const uint32_t slot = timer_id & kTimerSlotMask, i = slot / g->K;
  if (i >= g->n_next) return CPBUS_ENOENT;
  int rc = group_flush(g, g->now); if (rc) return rc;
  group_retire(g);
  const uint32_t k = group_shard_of(g, i);
  const uint32_t local = (slot - g->first[k] * g->K) | (timer_id & ~kTimerSlotMask);
  if ((rc = cpbus_timer_cancel(g->shards[k], local))) return rc;
  g->timers[slot].active = false; g->n_timers--;
  if (g->n_timers == 0) g->min_period = UINT64_MAX;
  return CPBUS_OK;
} CPBUS_CATCH

static void group_dbg_put(cpbus_group* g, const cpbus_event& e) {   // dbg_ring_put
  g->dbg[(g->dbg_head + 1) % 10] = e;
  const int old = g->dbg_head;
  g->dbg_head = (g->dbg_head + 1) % 10;
  if (old != -1 && g->dbg_head == g->dbg_tail) g->dbg_tail = (g->dbg_tail + 1) % 10;
}

int cpbus_group_publish(cpbus_group_t* g, const cpbus_event* ev, size_t n) try {
  if (!g || (!ev && n)) return CPBUS_EINVAL;
  auto dbg_tail = [&](size_t published) {   // as cpbus_publish: the last 10 of the burst
    for (size_t j = published > 10 ? published - 10 : 0; j < published; j++) {
      cpbus_event e{};
      e.seq = g->seq - (published - j); e.ts_ns = g->now; e.code = ev[j].code; e.source_id = ev[j].source_id; e.target = CPBUS_TARGET_ALL;
      group_dbg_put(g, e);
    }
  };
  for (size_t i = 0; i < n; i++) if (ev[i].code >= CPBUS_N_CODES) return CPBUS_EINVAL;
  for (size_t i = 0; i < n; i++) {
    const uint32_t code = ev[i].code;
    const int rc = group_stage(g, code, ev[i].source_id, CPBUS_TARGET_ALL, 0);
    if (rc) { dbg_tail(i); return rc; }
    if (code != CPBUS_METRIC) { g->by_code[code]++; g->pub_pairs.add(((uint64_t)code << 32) | ev[i].source_id, 1); }
    g->publishes++;
  }
  dbg_tail(n);
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_send(cpbus_group_t* g, uint32_t sub_id, const cpbus_event* ev) try {
  if (!g || !ev || ev->code >= CPBUS_N_CODES) return CPBUS_EINVAL;
  cpbus* s = nullptr; uint32_t l = 0;
  if (!group_locate(g, sub_id, &s, &l)) return CPBUS_ENOENT;
  if (!s->h_active[l]) return CPBUS_ECLOSED;
  const int rc = group_stage(g, ev->code, ev->source_id, sub_id, CPBUS_F_UNICAST);
  if (rc) return rc;
  g->publishes++;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_advance(cpbus_group_t* g, uint64_t now_ns) try {
  if (!g) return CPBUS_EINVAL;
  if (now_ns < g->now) return CPBUS_EORDER;
  if (now_ns == g->now) return CPBUS_OK;
  const uint64_t win = group_window(g);   // the single bus's grid: a stream batch never steps past a shard's window
  while (win != UINT64_MAX && now_ns - g->last_watermark > win) {
    g->now = g->last_watermark + win;
    const int rc = group_flush(g, g->now); if (rc) return rc;
  }
  g->now = now_ns;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_flush(cpbus_group_t* g) try {
  return g ? group_flush(g, g->now) : CPBUS_EINVAL;
} CPBUS_CATCH

int cpbus_group_sync(cpbus_group_t* g) try {
  if (!g) return CPBUS_EINVAL;
  for (cpbus* s : g->shards) { const int rc = cpbus_sync(s); if (rc) return rc; }
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_drain(cpbus_group_t* g, uint32_t sub_id, cpbus_event* out, size_t cap, size_t* n, uint64_t* lost) try {
  if (!g || !n || (!out && cap)) return CPBUS_EINVAL;
  cpbus* s = nullptr; uint32_t l = 0;
  if (!group_locate(g, sub_id, &s, &l)) return CPBUS_ENOENT;
  return cpbus_drain(s, sub_id, out, cap, n, lost);
} CPBUS_CATCH

// The first ready mailbox of [a, a + cnt) on shard s (cnt when none): where a walk with no room left stops.
static int group_first_ready(cpbus* s, uint32_t l, uint32_t cnt, uint32_t* at) {
  std::vector<SubCtl> c(cnt);
  int rc = dev_guard(s); if (rc) return rc;
  CK(cudaMemcpyAsync(c.data(), s->d_ctl + l, (size_t)cnt * sizeof(SubCtl), cudaMemcpyDeviceToHost, s->stream));
  CK(cudaStreamSynchronize(s->stream));
  *at = cnt;
  for (uint32_t i = 0; i < cnt; i++) if (c[i].tail > c[i].head) { *at = i; break; }
  return CPBUS_OK;
}

// The cyclic walk of cpbus_drain_ready over the shards: each piece of the walk that lies on one shard is drained there with
// the cap and ready entries still left, and the walk stops at the first mailbox that does not fit, as the single call does.
int cpbus_group_drain_ready(cpbus_group_t* g, uint32_t first_sub, uint32_t n, uint32_t start_sub, cpbus_event* out, size_t cap,
                            cpbus_ready* ready, size_t ready_cap, size_t* n_ready, size_t* total, uint32_t* next_sub) try {
  if (!g || !out || !ready || !n_ready || !total || !next_sub || !n || !ready_cap) return CPBUS_EINVAL;
  if (cap < g->shards[0]->R || cap > 0xFFFFFFFFull) return CPBUS_EINVAL;
  if (start_sub < first_sub || start_sub - first_sub >= n) return CPBUS_EINVAL;
  const uint32_t i0 = first_sub - g->base;
  if (first_sub < g->base || (uint64_t)i0 + n > g->n_next) return CPBUS_ENOENT;
  size_t nr = 0, tot = 0, ready_left = std::min<size_t>(ready_cap, n);
  const uint32_t rot = start_sub - first_sub;
  *next_sub = start_sub;
  for (uint32_t done = 0; done < n;) {
    const uint32_t i = i0 + (rot + done) % n;                       // global index of the walk's next mailbox
    const uint32_t k = group_shard_of(g, i);
    const uint32_t wrap = i0 + n - i;                               // the walk wraps to first_sub after this many
    const uint32_t cnt = std::min({n - done, g->first[k + 1] - i, wrap});
    cpbus* s = g->shards[k];
    const uint32_t l = i - g->first[k], a = g->base + i;
    if (ready_left == 0 || tot == cap) {                           // no room: the next ready mailbox ends the walk
      uint32_t at = cnt;
      const int rc = group_first_ready(s, l, cnt, &at); if (rc) return rc;
      if (at < cnt) { *next_sub = a + at; break; }
      done += cnt;
      continue;
    }
    size_t nr_s = 0, tot_s = 0;
    uint32_t next_s = a;
    bool all = false;
    const int rc = drain_ready_impl(s, a, cnt, a, out + tot, cap - tot, ready + nr, ready_left, &nr_s, &tot_s, &next_s, &all);
    if (rc) return rc;
    for (size_t j = 0; j < nr_s; j++) ready[nr + j].offset += (uint32_t)tot;
    nr += nr_s; tot += tot_s; ready_left -= nr_s;
    if (!all) { *next_sub = next_s; break; }
    done += cnt;
  }
  *n_ready = nr; *total = tot;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_consume_all(cpbus_group_t* g) try {
  if (!g) return CPBUS_EINVAL;
  for (cpbus* s : g->shards) { const int rc = cpbus_consume_all(s); if (rc) return rc; }
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_peek_window(cpbus_group_t* g, uint32_t sub_id, cpbus_event* out, size_t cap, size_t* n) try {
  if (!g || !n || (!out && cap)) return CPBUS_EINVAL;
  cpbus* s = nullptr; uint32_t l = 0;
  if (!group_locate(g, sub_id, &s, &l)) return CPBUS_ENOENT;
  return cpbus_peek_window(s, sub_id, out, cap, n);
} CPBUS_CATCH

int cpbus_group_digest(cpbus_group_t* g, uint32_t first_sub, uint32_t n, cpbus_digest_t* out) try {
  if (!g || !out || !n) return CPBUS_EINVAL;
  const uint32_t i0 = first_sub - g->base;
  if (first_sub < g->base || (uint64_t)i0 + n > g->n_next) return CPBUS_ENOENT;
  return group_each_range(g, i0, n, [&](cpbus* s, uint32_t l, uint32_t off, uint32_t cnt) -> int {
    return cpbus_digest(s, s->cfg.sub_id_base + l, cnt, out + off);
  });
} CPBUS_CATCH

int cpbus_group_digest_fold(cpbus_group_t* g, uint32_t first_sub, uint32_t n, uint64_t out[4]) try {
  if (!g || !out || !n) return CPBUS_EINVAL;
  const uint32_t i0 = first_sub - g->base;
  if (first_sub < g->base || (uint64_t)i0 + n > g->n_next) return CPBUS_ENOENT;
  uint64_t acc[4] = {0, 0, 0, 0};
  const int rc = group_each_range(g, i0, n, [&](cpbus* s, uint32_t l, uint32_t, uint32_t cnt) -> int {
    uint64_t part[4];
    const int rc_s = cpbus_digest_fold(s, s->cfg.sub_id_base + l, cnt, part);
    if (rc_s) return rc_s;
    acc[0] += part[0]; acc[1] += part[1]; acc[2] ^= part[2]; acc[3] += part[3];   // sums add, the hash term XORs
    return CPBUS_OK;
  });
  if (rc) return rc;
  for (int j = 0; j < 4; j++) out[j] = acc[j];
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_debug_events(cpbus_group_t* g, cpbus_event* out, size_t cap, size_t* n) try {   // cpbus_debug_events
  if (!g || !n || (!out && cap)) return CPBUS_EINVAL;
  size_t k = 0;
  for (;;) {
    if (g->dbg_head == -1) break;
    const cpbus_event e = g->dbg[g->dbg_tail % 10];
    if (g->dbg_tail == g->dbg_head) { g->dbg_head = -1; g->dbg_tail = 0; }
    else g->dbg_tail = (g->dbg_tail + 1) % 10;
    if (e.code == CPBUS_NONE && e.source_id == 0) break;
    if (k < cap) out[k] = e;
    k++;
  }
  *n = k;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_stats(cpbus_group_t* g, cpbus_stats_t* out) try {
  if (!g || !out) return CPBUS_EINVAL;
  cpbus_stats_t sum{}, s0{};
  for (cpbus* s : g->shards) {
    cpbus_stats_t x{};
    const int rc = cpbus_stats(s, &x); if (rc) return rc;
    if (s == g->shards[0]) s0 = x;   // the intern table's figures
    sum.deliveries += x.deliveries; sum.ticks += x.ticks; sum.overwritten += x.overwritten;
    sum.batches += x.batches; sum.kernel_launches += x.kernel_launches; sum.device_splits += x.device_splits;
    sum.admit_passes += x.admit_passes; sum.admit_skipped += x.admit_skipped; sum.admit_partial += x.admit_partial;
  }
  group_retire(g);
  sum.publishes = g->publishes;
  for (int c = 0; c < CPBUS_N_CODES; c++) sum.published_by_code[c] = g->by_code[c];
  sum.n_subs = g->n_active; sum.n_timers = g->n_timers; sum.now_ns = g->now;
  sum.intern_entries = s0.intern_entries; sum.intern_bytes = s0.intern_bytes;
  sum.ephemeral_live = s0.ephemeral_live; sum.ephemeral_recycled = s0.ephemeral_recycled;
  *out = sum;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_publish_counts(cpbus_group_t* g, cpbus_pair_count* out, size_t cap, size_t* n) try {
  if (!g || !n || (!out && cap)) return CPBUS_EINVAL;
  std::vector<std::pair<uint64_t, uint64_t>> v;
  for (size_t i = 0; i < g->pub_pairs.keys.size(); i++) if (g->pub_pairs.keys[i]) v.emplace_back(g->pub_pairs.keys[i] - 1, g->pub_pairs.cnts[i]);
  std::sort(v.begin(), v.end());
  for (size_t i = 0; i < v.size() && i < cap; i++) out[i] = cpbus_pair_count{(uint32_t)(v[i].first >> 32), (uint32_t)v[i].first, v[i].second};
  *n = v.size();
  return CPBUS_OK;
} CPBUS_CATCH

}  // extern "C"
