// cpbus.cu — libcpbus: C-ABI (include/cpbus.h) over the sm_90a (H100) kernels.
//
// Host-side bookkeeping that the reference keeps in Go (events/bus.go): the
// registry, the 10-slot debug ring, per-code publish counts, the Source intern
// table, the virtual clock, staging of published events into pinned batches.
// There is NO CPU data path: without a CUDA device cpbus_create fails with
// CPBUS_ENODEV, and nothing here touches oracle/.
//
// This file holds the single bus and its streams, and every kernel launch of the library; the group is
// cpbus_group.cpp, the host-only planners and exports cpbus_host.cpp, and what they share cpbus_internal.hpp.
#include "cpbus_internal.hpp"

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

int cpbus_host::dev_guard(cpbus* b) {
  CK(cudaSetDevice(b->device));
  return CPBUS_OK;
}

// How long the host waits for a stream's consumers or publisher (cpbus_stream_set_timeout; 0 = 2 s).
static std::chrono::microseconds stream_budget(const cpbus* b) {
  return std::chrono::microseconds(b->stream_spin_us ? b->stream_spin_us : 2000000u);
}

// The sticky stream error of this bus: a followed batch out of order (CPBUS_EORDER), otherwise a batch that never arrived or
// did not match its header (CPBUS_ETIMEDOUT).
static int stream_error(const cpbus* b) {
  const unsigned int e = *(volatile const unsigned int*)b->h_err;
  return (e & kErrFollowOrder) ? CPBUS_EORDER : (e ? CPBUS_ETIMEDOUT : CPBUS_OK);
}

static uint32_t mask_word(const cpbus* b, uint32_t local) {
  uint32_t hint = 0;
  if (b->K && !b->h_timers.empty())
    for (uint32_t k = 0; k < b->K; k++)
      if (b->h_timers[(size_t)local * b->K + k].active) hint = k + 1;
  if (!b->h_active[local]) return 0;
  const uint32_t pair_bit = (!b->h_npairs.empty() && b->h_npairs[local]) ? kPairBit : 0u;
  return (b->h_mask[local] & CPBUS_MASK_ALL) | (hint << kTimerHintShift) | pair_bit | kActiveBit;
}

static void dbg_ring_put(HostFront* f, const cpbus_event& e) {   // events/bus.go:24-31
  f->dbg[(f->dbg_head + 1) % 10] = e;
  int old = f->dbg_head;
  f->dbg_head = (f->dbg_head + 1) % 10;
  if (old != -1 && f->dbg_head == f->dbg_tail) f->dbg_tail = (f->dbg_tail + 1) % 10;
}

// While the broadcast events of a device-published batch are still unknown to the host (a marker is pending), later
// enqueues queue up behind it so that the ring keeps the global publish order; cpbus_debug_events resolves them.  (A group
// marks the device batches it launches, cpbus_group_publish_device, and resolves them against shard 0's accounting.)
void cpbus_host::dbg_enqueue(HostFront* f, const cpbus_event& e) {
  if (f->dbg_pending.empty()) { dbg_ring_put(f, e); return; }
  f->dbg_pending.push_back(DbgItem{false, 0ull, e});
  if (f->dbg_pending.size() > (size_t)kAcctDbgRing) f->dbg_pending.pop_front();
}

// DebugEvents (events/bus.go:34-54): empties the ring oldest first, up to a NonEvent; returns how many it read (the first
// cap of them go to out)
size_t cpbus_host::dbg_read(HostFront* f, cpbus_event* out, size_t cap) {
  size_t k = 0;
  for (;;) {
    if (f->dbg_head == -1) break;
    const cpbus_event e = f->dbg[f->dbg_tail % 10];
    if (f->dbg_tail == f->dbg_head) { f->dbg_head = -1; f->dbg_tail = 0; }
    else f->dbg_tail = (f->dbg_tail + 1) % 10;
    if (e.code == CPBUS_NONE && e.source_id == 0) break;   // == NonEvent
    if (k < cap) out[k] = e;
    k++;
  }
  return k;
}

void cpbus_host::dbg_mark_device_batch(HostFront* f, unsigned long long launch) {
  f->dbg_pending.push_back(DbgItem{true, launch, cpbus_event{}});
  if (f->dbg_pending.size() > (size_t)kAcctDbgRing) f->dbg_pending.pop_front();
}

// counting sort of the active subscribers by their 17-bit code mask (stable: ids ascending inside a mask)
static int rebuild_order(cpbus* b) {
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

// The ORDERED build (no timer armed, no pair table, at least one filtered subscriber) walks the mask order rebuild_order keeps
static bool ordered_build(const cpbus* b) {
  return !(b->n_paired > 0 && b->d_pairs) && !(b->n_timers > 0 && b->K > 0) && b->n_filtered > 0;
}

constexpr int kFanoutMaxSmem = 200 * 1024;

enum { kLaunchPlain = 0, kLaunchFollow = 1, kLaunchRound = 2 };

template <int STORE, bool TIMERS, bool DIGEST, bool ORDERED, bool PAIRS = false>
static int launch_fanout_t(cpbus* b, const FanoutParams& p, uint32_t grid, size_t smem, int kind) {
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

// Lossless rounds wait in the kernel: for the publisher's header (decide) and for the other shards' offers (agree).  With
// CUDA's lazy module loading, the first launch of a kernel loads it, and a load may wait for the kernels already running on
// the device — such as a round waiting for a batch that this very thread has yet to put, or for an offer that another shard
// of this thread has yet to queue.  So every kernel a lossless bus may launch while its rounds wait is loaded up front, once
// per device, when the bus is created.
template <int ST>
static int preload_round_fanouts() {
  void (*ks[])(FanoutParams) = {
      fanout_round_kernel<ST, false, false, false>, fanout_round_kernel<ST, false, true, false>,
      fanout_round_kernel<ST, true, false, false>, fanout_round_kernel<ST, true, true, false>,
      fanout_round_kernel<ST, false, false, true>, fanout_round_kernel<ST, false, true, true>,
      fanout_round_kernel<ST, true, false, false, true>, fanout_round_kernel<ST, true, true, false, true>};
  for (auto k : ks) CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kFanoutMaxSmem));
  return CPBUS_OK;
}

static int preload_round_kernels(cpbus* b) {
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
  CK(cudaFuncGetAttributes(&a, blockers_scan_kernel));   // a stalled publisher's query on another shard of this thread
  CK(cudaFuncGetAttributes(&a, lagging_scan_kernel));    // ... and the pump's
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

// The step-result sub-slots of launch ordinal `seq`: a launch adds into its own and zeroes its successor's.
static DevResultSlot* result_slot(const cpbus* b, unsigned long long seq) {
  return b->d_result + (size_t)(seq % kResultRing) * kResultSub;
}

// A launch (or a flush with nothing to launch) has reached watermark w: the clock, and the due index, follow it.
static void launched_to(cpbus* b, uint64_t w) {
  b->last_watermark = w;
  if (b->sparse) due_fire(b->due, b->h_timers, w, [](uint32_t, uint64_t, uint64_t) {});
}

static int launch_fanout(cpbus* b, const cpbus_event* d_src, uint32_t n, uint64_t w, const LaunchOpts& o = {}) {
  const StreamArgs* sa = o.stream;
  if (b->n_next == 0 && !sa) return CPBUS_OK;
  if (n == 0 && b->n_timers == 0 && !sa) return CPBUS_OK;   // (a stream batch is always consumed: its slot must be acknowledged)
  FanoutParams p{};
  p.batch = d_src; p.ring = b->d_ring; p.ctl = b->d_ctl; p.timers = b->d_timers; p.stats = b->d_stats; p.pow_table = b->d_pow; p.launch_seq = ++b->launch_seq;
  p.desc = b->d_desc + (p.launch_seq & 1) * ((fanout_desc_bytes(2048) + 255) & ~(size_t)255);   // two descriptor buffers: launch i+1 may write while launch i reads
  p.desc_ready = b->d_desc_ready + (p.launch_seq & 1) * 16; p.w_now = w;
  p.result = result_slot(b, p.launch_seq); p.result_next = result_slot(b, p.launch_seq + 1);
  p.batch_local = b->d_batch_local; p.staged = (uint32_t)o.staged;
  p.err_word = b->h_err.dev(); p.acct = o.account ? b->d_acct.get() : nullptr;
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
  p.pairs = pairs_on ? b->d_pairs.get() : nullptr;
  size_t smem = fanout_smem_bytes(p.smem_cap) + (pairs_on ? kPairFilterBytes : 0);   // + the batch's {code, source} presence filter
  if (ordered_build(b)) {
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
  // CPBUS_CFG_SPARSE_DRAINS: a drain on another thread sees the launch and the candidate index's update together
  std::unique_lock<std::mutex> ready_lock(b->mu, std::defer_lock);
  if (b->sparse_drains) ready_lock.lock();
#define CPBUS_DISPATCH(ST)                                                              \
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
  if (b->sparse_drains) b->ready_ix.full();   // any mailbox may have taken a record
  if (rc) return rc;
  b->st.kernel_launches++;
  if (!round) b->st.batches++;   // (a round's batch counts when it is resolved, if it delivered)
  if (sa) return CPBUS_OK;       // (the caller folds a stream launch in once its outcome is known: stream_delivered)
  launched_to(b, w);
  if (o.account && n) dbg_mark_device_batch(b, p.launch_seq);
  return CPBUS_OK;
}

// The host timer table, allocated by the first timer, and with it the due index.
static void timer_table(cpbus* b) {
  b->h_timers.resize((size_t)b->N * b->K);
  if (b->sparse) b->due.init(b->h_timers.size());
}

// Device staging is a long ring (kDevSlots batches): a slot is reused only kDevSlots flushes later, far beyond how far the
// host can run ahead, so the H2D never has to wait for an old fan-out and lands within microseconds.  Reuse safety is a
// host-side check once per epoch of kDevEpoch slots (almost always already satisfied).  stage_batch takes the next slot
// (*d_dst) and puts the n records of the current pinned buffer on their way into it; retire_slot follows the launch that
// reads the slot.
static int stage_batch(cpbus* b, uint32_t n, cpbus_event** d_dst) {
  const uint32_t slot = b->dev_slot;
  *d_dst = b->d_stage + (size_t)slot * b->B;
  if (slot % cpbus::kDevEpoch == 0) CK(cudaEventSynchronize(b->epoch_done[slot / cpbus::kDevEpoch]));   // last round's users of this epoch are done
  if (n) {
    CK(cudaMemcpyAsync(*d_dst, b->h_batch[b->cur], (size_t)n * sizeof(cpbus_event), cudaMemcpyHostToDevice, b->copy_stream));
    CK(cudaEventRecord(b->h2d_done[b->cur], b->copy_stream));
  }
  return CPBUS_OK;
}

static int retire_slot(cpbus* b) {
  const uint32_t slot = b->dev_slot;
  if (slot % cpbus::kDevEpoch == cpbus::kDevEpoch - 1) CK(cudaEventRecord(b->epoch_done[slot / cpbus::kDevEpoch], b->stream));
  b->dev_slot = (slot + 1) % cpbus::kDevSlots;
  return CPBUS_OK;
}

// Give the 8-16 KiB copy that `copied` marks up to 30 us to land.  If it has, the bus stream needs no wait node, consecutive
// fan-outs stay adjacent in the stream and the next launch's prologue overlaps this one's tail (programmatic dependent launch).
static int await_copy(cpbus* b, cudaEvent_t copied) {
  const auto t_spin = std::chrono::steady_clock::now();
  do {
    const cudaError_t q = cudaEventQuery(copied);
    if (q == cudaSuccess) return CPBUS_OK;
    if (q != cudaErrorNotReady) { CK(q); }
  } while (std::chrono::steady_clock::now() - t_spin < std::chrono::microseconds(30));
  CK(cudaStreamWaitEvent(b->stream, copied, 0));
  return CPBUS_OK;
}

// The staged batch has been launched whole: staging moves on to the next pinned buffer.
static int next_buffer(cpbus* b) {
  b->cur = (b->cur + 1) % cpbus::kStage;
  CK(cudaEventSynchronize(b->h2d_done[b->cur]));   // the pinned buffer we are about to overwrite has left the host
  return CPBUS_OK;
}

// CPBUS_CFG_SPARSE_TICKS: mailboxes (due slots, or candidates of a plan) and planned record deliveries beyond which a flush
// takes the full fan-out.  Measured on an H100 (DESIGN.md §4.6, §4.7): at 1,048,576 subscribers a dedicated tick kernel won
// at N/1,024 due slots and lost at N/128; the record kernel on timer-only plans costs the same as that kernel at N/1,024
// (the rows re-measured in §4.6), so the cap stays.
static size_t sparse_max(const cpbus* b) { return std::max<size_t>(32, b->n_next / 1024); }
static size_t sparse_max_deliveries(const cpbus* b) { return std::max<size_t>(1024, b->n_next / 256); }
// CPBUS_CFG_SPARSE_DRAINS: candidates in a drain's range beyond which it takes the dense scan, and a quarter of what the
// index keeps per set for a bus of n mailboxes.  Measured on an H100 at 1,048,576 mailboxes (DESIGN.md §4.13): the list
// scan beat the dense one up to 64 candidates, tied at 256 and lost from 1,024 on; the dense scan's cost grows with n.
static size_t ready_list_max(size_t n) { return std::max<size_t>(256, n / 4096); }

// The pinned plan buffer is free for `bytes`: the previous plan has left it, or both buffers are regrown (behind every
// kernel that may still read the old device buffer).
static int plan_room(cpbus* b, size_t bytes) {
  if (bytes <= b->d_plan.size() && bytes <= b->h_plan.size()) { CK(cudaEventSynchronize(b->plan_done)); return CPBUS_OK; }
  CK(cudaStreamSynchronize(b->stream)); CK(cudaStreamSynchronize(b->copy_stream));
  CK(b->d_plan.grow(bytes, 64 << 10));
  CK(b->h_plan.grow(bytes, 64 << 10));
  return CPBUS_OK;
}

// The record kernel over b->plan, to watermark w.  The plan goes up on the copy stream once the previous record kernel is
// done with the device buffer, and the kernel runs on the bus stream behind every earlier launch, without programmatic
// dependent launch.  With records staged, the batch takes the next device staging slot in front of the plan, the landing
// spin waits for both, and the staging buffer moves on.  A flush of due ticks alone has no batch: the bus stream waits for
// the plan.  A plan without a mailbox launches nothing and copies nothing.  The clock and the due index follow, as after a
// fan-out.
static int launch_sparse(cpbus* b, uint64_t w) {
  const size_t n_list = b->plan.size(), n_idx = b->plan_idx.size();
  const uint32_t n = (uint32_t)b->n_staged;
  if (n_list) {
    const size_t list_bytes = n_list * sizeof(cpbus_plan_entry), bytes = list_bytes + n_idx * sizeof(uint32_t);
    int rc = plan_room(b, bytes); if (rc) return rc;
    memcpy(b->h_plan, b->plan.data(), list_bytes);
    memcpy(b->h_plan + list_bytes, b->plan_idx.data(), n_idx * sizeof(uint32_t));
    cpbus_event* d_dst = nullptr;
    if (n && (rc = stage_batch(b, n, &d_dst))) return rc;
    CK(cudaStreamWaitEvent(b->copy_stream, b->records_done, 0));
    CK(cudaMemcpyAsync(b->d_plan, b->h_plan, bytes, cudaMemcpyHostToDevice, b->copy_stream));
    CK(cudaEventRecord(b->plan_done, b->copy_stream));
    if (n) { if ((rc = await_copy(b, b->plan_done))) return rc; }
    else CK(cudaStreamWaitEvent(b->stream, b->plan_done, 0));
    RecordScatterParams p{};
    p.list = reinterpret_cast<const uint4*>(b->d_plan.get()); p.n_list = (uint32_t)n_list;
    p.idx = reinterpret_cast<const uint32_t*>(b->d_plan + list_bytes); p.batch = d_dst;
    p.ring = b->d_ring; p.ctl = b->d_ctl; p.timers = b->d_timers; p.stats = b->d_stats; p.pow_table = b->d_pow;
    p.launch_seq = ++b->launch_seq;
    p.result = result_slot(b, p.launch_seq); p.result_next = result_slot(b, p.launch_seq + 1);
    p.w_now = w; p.ring_cap = b->R; p.K = b->K; p.sub_base = b->cfg.sub_id_base; p.use_digest = b->use_digest ? 1u : 0u;
    {
      // CPBUS_CFG_SPARSE_DRAINS: a drain on another thread sees the launch and its mailboxes in the index together
      std::unique_lock<std::mutex> ready_lock(b->mu, std::defer_lock);
      if (b->sparse_drains) ready_lock.lock();
      record_scatter_kernel<<<(uint32_t)((n_list + kWarpsPerCta - 1) / kWarpsPerCta), kThreads, 0, b->stream>>>(p);
      if (b->sparse_drains) b->ready_ix.add(&b->plan[0].local, n_list, sizeof(cpbus_plan_entry) / sizeof(uint32_t));
    }
    CK(cudaGetLastError());
    CK(cudaEventRecord(b->records_done, b->stream));
    b->st.kernel_launches++;
    if (n && (rc = retire_slot(b))) return rc;
  }
  b->n_staged = 0;
  // (n_next == 0: records staged on a bus without subscribers, which has no timer either; like the fan-out, the flush
  // launches nothing and leaves the watermark where it was.  A flush of due ticks alone always has subscribers.)
  if (b->n_next) launched_to(b, w);
  return n_list && n ? next_buffer(b) : CPBUS_OK;
}

// CPBUS_CFG_SPARSE_TICKS, with nothing staged or with CPBUS_CFG_SPARSE_RECORDS: true when the flush is done without the full
// fan-out (*rc = its status).  No record staged and no tick due in (last watermark, w]: no launch.  Otherwise the ticks due
// by w and the staged records are planned, and a plan within the caps launches the record kernel over its mailboxes (none:
// no launch).  False: the full fan-out follows, with admission and the partial prefix as before — past a cap, or (lossless)
// when the room bound cannot prove that the most one mailbox takes, records and ticks, fits.
static bool sparse_flush(cpbus* b, uint64_t w, int* rc) {
  *rc = CPBUS_OK;
  const bool ticks = b->due.min_due() <= w;
  if (!ticks && !b->n_staged) { b->last_watermark = w; return true; }
  const size_t max_m = sparse_max(b);
  std::vector<uint32_t>& due = b->due_slots;
  due.clear();
  if (ticks && !b->due.collect(w, max_m, &due)) return false;
  if (due.empty() && !b->n_staged) { launched_to(b, w); return true; }   // only stale entries in front (min_due is a lower bound): drop them
  if (!sparse_plan(b->rec_index, b->h_mask.data(), b->h_active.data(), b->n_next, b->cfg.sub_id_base, b->h_batch[b->cur],
                   b->n_staged, due, b->K, max_m, sparse_max_deliveries(b), b->plan_pairs, b->plan, b->plan_idx))
    return false;
  if (b->lossless) {
    uint64_t most = 0;   // the most one mailbox takes
    for (const cpbus_plan_entry& e : b->plan) {
      uint64_t take = e.count;
      for (uint32_t k = 0; k < b->K; k++) {
        if (!((e.due_bits >> k) & 1u)) continue;
        const HostTimer& t = b->h_timers[(size_t)e.local * b->K + k];
        take += t.oneshot ? 1 : due_ticks(t.next_due, t.period, w);
      }
      most = std::max(most, take);
    }
    if (b->room_lb < most) return false;
    b->room_lb -= most; b->st.admit_skipped++;
  }
  *rc = launch_sparse(b, w);
  return true;
}

// lossless admission (reference: the sender blocks on a full channel, events/subscriber.go:30-32)
// Fast path: true when n records with watermark w provably fit (or nothing has to be admitted) — no kernel, no sync.
bool cpbus_host::admit_fits(cpbus* b, uint32_t n, uint64_t w) {
  if (!b->lossless || b->n_next == 0) return true;
  const uint64_t need = admit_need(n, w, b->last_watermark, b->min_period, b->K, b->n_timers && b->K);
  if (b->room_lb >= need) { b->room_lb -= need; b->st.admit_skipped++; return true; }
  return false;
}

// The admission pass (after admit_fits said no): one kernel over every mailbox of the shard, then a host sync.
int cpbus_host::admit_pass(cpbus* b, const cpbus_event* d_src, uint32_t n, uint64_t w, bool* ok, uint32_t* prefix) {
  CK(cudaMemsetAsync(&b->d_stats->admit_overflow, 0, 4 * sizeof(unsigned long long), b->stream));   // overflow, overwritten, max_used, deficit
  const uint32_t threads = 256, grid = (b->n_next + threads - 1) / threads;
  admit_kernel<<<grid, threads, 0, b->stream>>>(d_src, n, w, b->d_ctl, b->d_timers, b->n_next, b->R, b->K,
                                                b->cfg.sub_id_base, b->n_timers > 0 && b->K > 0, b->d_stats,
                                                b->n_paired > 0 ? b->d_pairs.get() : nullptr);
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

static int admit(cpbus* b, const cpbus_event* d_src, uint32_t n, uint64_t w, bool* ok, uint32_t* prefix = nullptr) {
  *ok = true;
  if (prefix) *prefix = n;
  if (admit_fits(b, n, w)) return CPBUS_OK;
  return admit_pass(b, d_src, n, w, ok, prefix);
}

// host mirror of one-shot timers that have fired on the device (events/timer.go:19-33):
// a one-shot whose due time is <= the last launched watermark has disarmed itself.
void cpbus_host::retire_oneshots(HostFront* f, uint64_t w) {
  size_t keep = 0;
  for (size_t i = 0; i < f->oneshot_idx.size(); i++) {
    HostTimer& t = f->h_timers[f->oneshot_idx[i]];
    if (t.active && t.oneshot && oneshot_fired(t.next_due, w)) { t.active = false; f->n_timers--; continue; }
    if (t.active && t.oneshot) f->oneshot_idx[keep++] = f->oneshot_idx[i];
  }
  f->oneshot_idx.resize(keep);
  if (f->n_timers == 0) f->min_period = UINT64_MAX;
}

// Arm table slot `slot` (subscriber * K + k) at the clock: periodic timers bound the clock window, one-shots wait for
// retirement.
HostTimer& cpbus_host::timer_arm(HostFront* f, size_t slot, uint64_t period, uint32_t source_id, bool oneshot) {
  HostTimer& t = f->h_timers[slot];
  t.active = true; t.oneshot = oneshot; t.period = period; t.next_due = due_after(f->now, period); t.source_id = source_id;
  f->n_timers++;
  if (!oneshot) f->min_period = std::min(f->min_period, period);
  else f->oneshot_idx.push_back(slot);
  return t;
}

// Disarm table slot `slot` if it is armed.  A cancel (reset_bound) lets the window's bound go with the last timer; an
// unsubscribe keeps the stale bound, which narrows the window (and so the launch grid) until a cancel or a retirement.
void cpbus_host::timer_disarm(HostFront* f, size_t slot, bool reset_bound) {
  HostTimer& t = f->h_timers[slot];
  if (t.active) { t.active = false; f->n_timers--; }
  if (reset_bound && f->n_timers == 0) f->min_period = UINT64_MAX;
}

// True when a flush to watermark w launches nothing: no record is staged, and no timer is armed (the watermark then
// follows the clock) or the clock has not moved since the last launch.
bool cpbus_host::flush_idle(HostFront* f, uint64_t w) {
  if (f->n_staged) return false;
  if (f->n_timers == 0) { f->last_watermark = std::max(f->last_watermark, w); return true; }
  return w == f->last_watermark;
}

int cpbus_host::flush_staged(cpbus* b, uint64_t w) {
  if (flush_idle(b, w)) return CPBUS_OK;
  int rc;
  if (b->sparse && (!b->n_staged || b->sparse_records) && sparse_flush(b, w, &rc)) return rc;
  const uint32_t n = (uint32_t)b->n_staged;
  const int c = b->cur;
  cpbus_event* d_dst;
  if ((rc = stage_batch(b, n, &d_dst)) || (n && (rc = await_copy(b, b->h2d_done[c])))) return rc;
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
    if ((rc = launch_fanout(b, d_dst, m, w_part)) || (rc = retire_slot(b))) return rc;
    memmove(b->h_batch[c], b->h_batch[c] + m, (size_t)(n - m) * sizeof(cpbus_event));   // (the H2D of this buffer completed before the admission pass)
    b->n_staged = n - m;
    b->room_lb = 0;
    b->st.admit_partial++;
    return CPBUS_EAGAIN;
  }
  if ((rc = launch_fanout(b, d_dst, n, w)) || (rc = retire_slot(b))) return rc;
  b->n_staged = 0;
  return next_buffer(b);
}

cpbus_event* cpbus_host::staging(cpbus* b) { return b->h_batch[b->cur]; }

uint64_t cpbus_host::max_window(const HostFront* f) {
  if (!f->K || f->n_timers == 0 || f->min_period == UINT64_MAX) return UINT64_MAX;
  const uint64_t J = 32u / f->K;
  return f->min_period > UINT64_MAX / J ? UINT64_MAX : f->min_period * J;
}

// CPBUS_CFG_DROP_MISSED_TICKS: the catch-up of a clock step to `now`, after a flush to the old clock.  timer_catchup_kernel
// runs on the bus stream behind every earlier launch: over the whole slot table of a dense bus, and over exactly the slots
// that the due index moved (due_catchup) on a sparse one, where no slot moving means no launch.
int cpbus_host::catch_up(cpbus* b, uint64_t now) {
  if (!b->K || b->n_timers == 0 || b->h_timers.empty() || b->n_next == 0) return CPBUS_OK;
  const uint32_t* list = nullptr;
  size_t n = (size_t)b->n_next * b->K;
  if (b->sparse) {
    b->catchup_slots.clear();
    due_catchup(b->due, b->h_timers, now, &b->catchup_slots);
    n = b->catchup_slots.size();
    if (!n) return CPBUS_OK;
    if (n > b->d_catchup.size()) {   // (behind every kernel that may still read the old list)
      CK(cudaStreamSynchronize(b->stream));
      CK(b->d_catchup.grow(n, 1024));
    }
    // (pageable source: the call returns once the list has been taken, and the copy runs in stream order)
    CK(cudaMemcpyAsync(b->d_catchup, b->catchup_slots.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice, b->stream));
    list = b->d_catchup;
  }
  timer_catchup_kernel<<<(uint32_t)((n + kThreads - 1) / kThreads), kThreads, 0, b->stream>>>(b->d_timers, list, (uint32_t)n, now);
  CK(cudaGetLastError());
  b->st.kernel_launches++;
  return CPBUS_OK;
}


// Whether ids [first, first + n) lie in [base, base + n_next), the ids subscribed so far; *index = first - base.
bool cpbus_host::id_range(uint32_t base, uint32_t n_next, uint32_t first, uint64_t n, uint32_t* index) {
  *index = first - base;
  return first >= base && (uint64_t)*index + n <= n_next;
}

// Whether sub_id names a mailbox of this bus that was handed out and not released since; *l = its index.  A released id
// is refused as one never handed out; range calls keep n_next as their bound and see a released mailbox as empty.
static bool sub_index(const cpbus* b, uint32_t sub_id, uint32_t* l) {
  return id_range(b->cfg.sub_id_base, b->n_next, sub_id, 1, l) && !b->h_released[*l];
}

// cpbus_publish_counts: the host publish counts of f and n_dev device-counted pairs (key + 1 per slot, 0 = empty), merged by
// {code, source} and sorted; *n = how many pairs there are, the first cap of them go to out.
void cpbus_host::pair_counts(const HostFront* f, const unsigned long long* dev_keys, const unsigned long long* dev_cnts, size_t n_dev,
                             cpbus_pair_count* out, size_t cap, size_t* n) {
  std::unordered_map<uint64_t, uint64_t> merged;
  for (size_t i = 0; i < f->pub_pairs.keys.size(); i++) if (f->pub_pairs.keys[i]) merged[f->pub_pairs.keys[i] - 1] += f->pub_pairs.cnts[i];
  for (size_t i = 0; i < n_dev; i++) if (dev_keys[i]) merged[dev_keys[i] - 1] += dev_cnts[i];
  std::vector<std::pair<uint64_t, uint64_t>> v(merged.begin(), merged.end());
  std::sort(v.begin(), v.end());
  for (size_t i = 0; i < v.size() && i < cap; i++) out[i] = cpbus_pair_count{(uint32_t)(v[i].first >> 32), (uint32_t)v[i].first, v[i].second};
  *n = v.size();
}

static bool is_pow2(uint32_t x) { return x && !(x & (x - 1)); }

// outstanding followers and rounds that hold one of the kFollowMax records
static int follow_records(const cpbus* b) {
  int n = 0;
  for (const cpbus::FollowPending& f : b->follow_q) n += f.kind != cpbus::kConsumeAll ? 1 : 0;
  return n;
}

static int follow_resolve(cpbus* b);
// The opening of the entry points that read or change host-side bus state: this bus's device, then the outstanding
// followers and rounds folded in (DESIGN.md §8, lazy resolution).
int cpbus_host::enter(cpbus* b) {
  const int rc = dev_guard(b);
  return rc ? rc : follow_resolve(b);
}

// The checks cpbus_create makes of a config (cpbus_group_create makes them of the total); R and B get the defaults applied.
int cpbus_host::config_check(const cpbus_config* cfg, uint32_t* R_out, uint32_t* B_out) {
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
  if ((cfg->flags & CPBUS_CFG_SPARSE_RECORDS) && !(cfg->flags & CPBUS_CFG_SPARSE_TICKS)) return CPBUS_EINVAL;   // the due index finds the ticks
  if ((cfg->flags & CPBUS_CFG_SPARSE_DRAINS) && !(cfg->flags & CPBUS_CFG_SPARSE_TICKS)) return CPBUS_EINVAL;    // launches that know their mailboxes
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
  b->sparse = cfg->flags & CPBUS_CFG_SPARSE_TICKS;
  b->sparse_records = cfg->flags & CPBUS_CFG_SPARSE_RECORDS;
  b->sparse_drains = cfg->flags & CPBUS_CFG_SPARSE_DRAINS;
  b->drop_missed = cfg->flags & CPBUS_CFG_DROP_MISSED_TICKS;
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
  // device memory: CPBUS_ENOMEM, with the size the runtime refused
  auto alloc = [](auto& buf, size_t n) {
    if (buf.alloc(n) == cudaSuccess) return true;
    snprintf(g_cuda_err, sizeof(g_cuda_err), "cudaMalloc(%zu) failed", n * sizeof(*buf.get()));
    return false;
  };
  if (!alloc(b->d_ring, N * R) || !alloc(b->d_ctl, N) || !alloc(b->d_order, N) || (K && !alloc(b->d_timers, N * K)) ||
      !alloc(b->d_stats, 1) || !alloc(b->d_fold, 4 * cpbus::kFoldSlots) || !alloc(b->d_pow, kPowTableLen) ||
      !alloc(b->d_desc, 2 * ((fanout_desc_bytes(2048) + 255) & ~(size_t)255)) || !alloc(b->d_desc_ready, 32))
    return fail(CPBUS_ENOMEM);
  if (cudaMemsetAsync(b->d_desc_ready, 0, 256, b->stream) != cudaSuccess) return fail(CPBUS_ECUDA);
  if (b->copy_stream.create() != cudaSuccess || b->result_stream.create() != cudaSuccess || b->launched.create() != cudaSuccess)
    return fail(CPBUS_ECUDA);
  if (b->sparse && (b->plan_done.create() != cudaSuccess || b->records_done.create() != cudaSuccess)) return fail(CPBUS_ECUDA);
  if (!alloc(b->d_stage, (size_t)cpbus::kDevSlots * B)) return fail(CPBUS_ENOMEM);
  for (CudaEvent& e : b->epoch_done) if (e.create() != cudaSuccess) return fail(CPBUS_ECUDA);
  for (int i = 0; i < cpbus::kStage; i++) {
    if (b->h_batch[i].alloc(B) != cudaSuccess) return fail(CPBUS_ENOMEM);
    if (b->h2d_done[i].create() != cudaSuccess) return fail(CPBUS_ECUDA);
  }
  if (!alloc(b->d_batch_local, B)) return fail(CPBUS_ENOMEM);
  if (b->lossless) {
    // lossless rounds (cpbus_stream_round_next): device state and the host records, allocated here rather than by the
    // first round, while no round of any shard can be waiting on the device
    if (!alloc(b->d_admit_batch, B) || !alloc(b->d_round, 1)) return fail(CPBUS_ENOMEM);
    RoundDev init{};
    init.room_full = R;
    if (cudaMemcpyAsync(b->d_round, &init, sizeof(init), cudaMemcpyHostToDevice, b->stream) != cudaSuccess) return fail(CPBUS_ECUDA);
    if (b->h_round.alloc(cpbus::kFollowMax) != cudaSuccess) return fail(CPBUS_ENOMEM);
    if ((rc = preload_round_kernels(b))) return fail(rc);
  } else {   // followers (cpbus_stream_fanout_next): their records and the clock words, zeroed
    if (b->h_follow.alloc(cpbus::kFollowMax) != cudaSuccess || !alloc(b->d_follow_clock, 4)) return fail(CPBUS_ENOMEM);
    if (cudaMemsetAsync(b->d_follow_clock, 0, 4 * sizeof(unsigned long long), b->stream) != cudaSuccess) return fail(CPBUS_ECUDA);
  }
  if (b->follow_done.create() != cudaSuccess) return fail(CPBUS_ECUDA);
  if (!alloc(b->d_pf_buf, (size_t)kStreamPrefetch * B) || !alloc(b->d_pf_state, 8) || !alloc(b->d_acct, 1))
    return fail(CPBUS_ENOMEM);
  if (cudaMemsetAsync(b->d_pf_state, 0, 64, b->stream) != cudaSuccess ||
      cudaMemsetAsync(b->d_acct, 0, sizeof(DevPubAcct), b->stream) != cudaSuccess) return fail(CPBUS_ECUDA);
  if (b->h_err.alloc(16) != cudaSuccess) return fail(CPBUS_ENOMEM);
  memset(b->h_err, 0, 64);
  // cpbus_lagging / cpbus_blockers: allocated here, so that neither query allocates (or frees) while a round may wait
  if (!alloc(b->d_lag_lb, kLagLbOffset + (N + kReadyTile - 1) / kReadyTile) || b->h_lag_hdr.alloc(kLagHdrWords) != cudaSuccess ||
      (b->lossless && b->h_block.alloc(N) != cudaSuccess) || b->h_acct.alloc(offsetof(DevPubAcct, pair_key)) != cudaSuccess)
    return fail(CPBUS_ENOMEM);
  for (auto& d : b->d_prefetch) if (!alloc(d, B)) return fail(CPBUS_ENOMEM);
  if (!alloc(b->d_result, (size_t)kResultRing * kResultSub)) return fail(CPBUS_ENOMEM);
  if (cudaMemsetAsync(b->d_result, 0, sizeof(DevResultSlot) * kResultRing * kResultSub, b->stream) != cudaSuccess) return fail(CPBUS_ECUDA);
  if (b->h_result.alloc((size_t)8 * kResultSub) != cudaSuccess) return fail(CPBUS_ENOMEM);
  for (CudaEvent& e : b->result_done) if (e.create() != cudaSuccess) return fail(CPBUS_ECUDA);
  if (b->h_stats.alloc(1) != cudaSuccess || b->h_fold.alloc(4 * cpbus::kFoldSlots) != cudaSuccess) return fail(CPBUS_ENOMEM);
  for (CudaEvent& e : b->fold_done) if (e.create() != cudaSuccess) return fail(CPBUS_ECUDA);
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
  b->h_released.assign(N, 0);
  if (b->sparse_records) b->rec_index.init(N, 2 * std::max<size_t>(32, N / 1024));   // lists of up to twice the largest cap
  else if (b->sparse) b->rec_index.slot.assign(N, UINT32_MAX);
  if (b->sparse_drains) b->ready_ix.init(N, 4 * ready_list_max(N));
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
  if (b->copy_stream) cudaStreamSynchronize(b->copy_stream);
  if (b->result_stream) cudaStreamSynchronize(b->result_stream);
  while (!b->streams.empty()) cpbus_stream_close(b->streams.back());
  for (void* p : b->shared_mapped) cudaIpcCloseMemHandle(p);
  for (void* p : b->shared_owned) cudaFree(p);
  if (b->own_stream && b->stream) cudaStreamDestroy(b->stream);
  delete b;   // the owners free the bus's own memory, events and streams
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

// The host half of a subscription into mailbox l, fresh or reused, after the call's flush: the registry and the sparse
// record index.  The caller writes the control block.
static void subscribe_host(cpbus* b, uint32_t l, uint32_t mask) {
  b->h_mask[l] = mask & CPBUS_MASK_ALL;
  b->h_active[l] = 1;
  if (b->h_mask[l] != CPBUS_MASK_ALL) b->n_filtered++;
  if (b->sparse_records) b->rec_index.add_codes(l, b->h_mask[l]);
}

// The host half of subscriber l's exact cases, after subscribe_host, once the pair tables exist: the first n_pairs of
// `pairs` whose code is not in the mask go to row[0 ..) (the caller fills the rest with kPairNone), to the registry and to
// the sparse record index.  Returns how many there are.
static uint32_t pairs_host(cpbus* b, uint32_t l, const cpbus_pair* pairs, uint32_t n_pairs, uint2* row) {
  uint32_t used = 0;
  for (uint32_t j = 0; j < n_pairs; j++)
    if (!((b->h_mask[l] >> pairs[j].code) & 1u)) row[used++] = make_uint2(pairs[j].code, pairs[j].source_id);
  b->h_npairs[l] = (uint8_t)used;
  if (used) b->n_paired++;
  if (b->sparse_records && used) {
    uint64_t keys[CPBUS_MAX_PAIRS];
    for (uint32_t j = 0; j < used; j++) keys[j] = (uint64_t)row[j].x << 32 | row[j].y;
    b->rec_index.add_cases(l, keys, used);
  }
  return used;
}

int cpbus_subscribe_many(cpbus_t* b, const uint32_t* masks, uint32_t n, uint32_t* first_sub_id) try {
  if (!b || !n) return CPBUS_EINVAL;
  if ((uint64_t)b->n_next + n > b->N) return CPBUS_ENOSPC;
  int rc = enter(b); if (rc) return rc;
  if ((rc = flush_staged(b, b->now))) return rc;   // ordered with publishes (events/bus.go:105-107 takes the same lock)
  const uint32_t first = b->n_next;
  std::vector<SubCtl> blocks(n);
  memset(blocks.data(), 0, (size_t)n * sizeof(SubCtl));
  for (uint32_t i = 0; i < n; i++) {
    subscribe_host(b, first + i, masks ? masks[i] : CPBUS_MASK_ALL);
    blocks[i].mask = b->h_mask[first + i] | kActiveBit;
  }
  CK(cudaMemcpyAsync(b->d_ctl + first, blocks.data(), (size_t)n * sizeof(SubCtl), cudaMemcpyHostToDevice, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  b->n_next += n; b->n_active += n; b->order_dirty = true;
  if (first_sub_id) *first_sub_id = b->cfg.sub_id_base + first;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_subscribe(cpbus_t* b, uint32_t mask, uint32_t* sub_id) { return cpbus_subscribe_many(b, &mask, 1, sub_id); }

static int push_mask_words(cpbus* b, uint32_t first, uint32_t n) {
  std::vector<uint32_t> words(n);
  for (uint32_t i = 0; i < n; i++) words[i] = mask_word(b, first + i);
  CK(cudaMemcpy2DAsync(&b->d_ctl[first].mask, sizeof(SubCtl), words.data(), 4, 4, n, cudaMemcpyHostToDevice, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  return CPBUS_OK;
}

// The pair tables of every subscriber, allocated by the first subscription with pairs.
static int pair_tables(cpbus* b) {
  if (b->d_pairs) return CPBUS_OK;
  const size_t n = (size_t)b->N * CPBUS_MAX_PAIRS;
  if (b->d_pairs.alloc(n) != cudaSuccess) {
    snprintf(g_cuda_err, sizeof(g_cuda_err), "cudaMalloc(pair tables) failed");
    return CPBUS_ENOMEM;
  }
  CK(cudaMemsetAsync(b->d_pairs, 0xFF, n * sizeof(uint2), b->stream));   // every slot unused
  b->h_npairs.assign(b->N, 0);
  return CPBUS_OK;
}

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
  if ((rc = pair_tables(b))) return rc;
  uint32_t id = 0;
  if ((rc = cpbus_subscribe_many(b, &mask, 1, &id))) return rc;
  const uint32_t l = id - b->cfg.sub_id_base;
  for (uint32_t j = used; j < CPBUS_MAX_PAIRS; j++) row[j] = make_uint2(kPairNone, kPairNone);
  CK(cudaMemcpyAsync(b->d_pairs + (size_t)l * CPBUS_MAX_PAIRS, row, sizeof(row), cudaMemcpyHostToDevice, b->stream));
  CK(cudaStreamSynchronize(b->stream));   // `row` is on the stack
  b->h_npairs[l] = (uint8_t)used; b->n_paired++;
  if (b->sparse_records) {
    uint64_t keys[CPBUS_MAX_PAIRS];
    for (uint32_t j = 0; j < used; j++) keys[j] = (uint64_t)row[j].x << 32 | row[j].y;
    b->rec_index.add_cases(l, keys, used);
  }
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
  if ((rc = pair_tables(b))) return rc;
  uint32_t first = 0;
  if ((rc = cpbus_subscribe_many(b, masks, n, &first))) return rc;
  const uint32_t l0 = first - b->cfg.sub_id_base;
  std::vector<uint2> rows((size_t)n * CPBUS_MAX_PAIRS, make_uint2(kPairNone, kPairNone));
  uint32_t paired = 0;
  for (uint32_t i = 0; i < n; i++)
    if (pairs_host(b, l0 + i, pairs + (size_t)i * CPBUS_MAX_PAIRS, n_pairs[i], rows.data() + (size_t)i * CPBUS_MAX_PAIRS)) paired++;
  CK(cudaMemcpyAsync(b->d_pairs + (size_t)l0 * CPBUS_MAX_PAIRS, rows.data(), rows.size() * sizeof(uint2), cudaMemcpyHostToDevice, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  if (paired && (rc = push_mask_words(b, l0, n))) return rc;
  if (first_sub_id) *first_sub_id = first;
  return CPBUS_OK;
} CPBUS_CATCH

// The host half of cpbus_unsubscribe, after its flush: CPBUS_ECLOSED, or the registry, the sparse indexes and the timer
// table updated.  *clear = the timer slots whose device copies are to be disarmed: all K once the table exists.
static int unsubscribe_host(cpbus* b, uint32_t l, uint32_t* clear) {
  // second Unsubscribe drives the WaitGroup negative in Go (events/bus.go:121) => panic
  if (!b->h_active[l]) return CPBUS_ECLOSED;
  b->h_active[l] = 0;
  if (b->h_mask[l] != CPBUS_MASK_ALL) b->n_filtered--;
  if (!b->h_npairs.empty() && b->h_npairs[l]) { b->h_npairs[l] = 0; b->n_paired--; }
  if (b->sparse_records) {
    b->rec_index.remove_codes(l, b->h_mask[l], b->h_mask.data(), b->h_active.data());
    b->rec_index.remove_cases(l, b->h_active.data());
  }
  b->order_dirty = true;
  *clear = 0;
  if (b->K && !b->h_timers.empty()) {
    for (uint32_t k = 0; k < b->K; k++) {
      timer_disarm(b, (size_t)l * b->K + k, /*reset_bound=*/false);
      if (b->sparse) b->due.drop(l * b->K + k);
    }
    *clear = (1u << b->K) - 1u;
  }
  b->n_active--;
  return CPBUS_OK;
}

int cpbus_unsubscribe(cpbus_t* b, uint32_t sub_id) try {
  if (!b) return CPBUS_EINVAL;
  uint32_t l = 0, clear = 0;
  if (!sub_index(b, sub_id, &l)) return CPBUS_ENOENT;
  int rc = enter(b); if (rc) return rc;
  if ((rc = flush_staged(b, b->now))) return rc;
  if ((rc = unsubscribe_host(b, l, &clear))) return rc;
  const uint32_t word = 0;
  CK(cudaMemcpyAsync(&b->d_ctl[l].mask, &word, 4, cudaMemcpyHostToDevice, b->stream));
  if (clear) CK(cudaMemsetAsync(b->d_timers + (size_t)l * b->K, 0xFF, b->K * sizeof(DevTimer), b->stream));
  CK(cudaStreamSynchronize(b->stream));
  return CPBUS_OK;
} CPBUS_CATCH

// The host half of cpbus_set_mask, after its flush.
static void set_mask_host(cpbus* b, uint32_t l, uint32_t mask) {
  mask &= CPBUS_MASK_ALL;
  if (b->h_mask[l] != CPBUS_MASK_ALL) b->n_filtered--;
  if (mask != CPBUS_MASK_ALL) b->n_filtered++;
  const uint32_t old = b->h_mask[l];
  b->h_mask[l] = mask; b->order_dirty = true;
  if (b->sparse_records) {
    b->rec_index.add_codes(l, mask & ~old);
    b->rec_index.remove_codes(l, old & ~mask, b->h_mask.data(), b->h_active.data());
  }
}

// Change a subscriber's code mask in place (ordered with publishes like Subscribe): the subscriber keeps its mailbox,
// its timers and its exact cases.  Used when a mailbox that so far only received timer ticks / direct sends (mask 0:
// NewEventTimer on a channel that was not subscribed, watches/watches.go:37,71) is subscribed to the bus after all.
int cpbus_set_mask(cpbus_t* b, uint32_t sub_id, uint32_t mask) try {
  if (!b) return CPBUS_EINVAL;
  uint32_t l = 0;
  if (!sub_index(b, sub_id, &l)) return CPBUS_ENOENT;
  if (!b->h_active[l]) return CPBUS_ECLOSED;
  int rc = enter(b); if (rc) return rc;
  if ((rc = flush_staged(b, b->now))) return rc;
  set_mask_host(b, l, mask);
  return push_mask_words(b, l, 1);
} CPBUS_CATCH

int cpbus_timer_add(cpbus_t* b, uint32_t sub_id, uint64_t period_ns, uint32_t source_id, int oneshot, uint32_t* timer_id) try {
  if (!b || !period_ns) return CPBUS_EINVAL;
  if (!b->K) return CPBUS_ENOSPC;
  uint32_t l = 0;
  if (!sub_index(b, sub_id, &l)) return CPBUS_ENOENT;
  int rc = enter(b); if (rc) return rc;
  if ((rc = flush_staged(b, b->now))) return rc;
  if (b->h_timers.empty()) timer_table(b);
  retire_oneshots(b, b->last_watermark);
  if (!b->h_active[l]) return CPBUS_ECLOSED;
  for (uint32_t k = 0; k < b->K; k++) {
    if (b->h_timers[(size_t)l * b->K + k].active) continue;
    HostTimer& t = timer_arm(b, (size_t)l * b->K + k, period_ns, source_id, oneshot != 0);
    if (b->sparse) b->due.put(l * b->K + k, t.next_due);
    DevTimer d{}; d.next_due = t.next_due; d.period = oneshot ? 0 : period_ns; d.source_id = source_id; d.fired = 0;
    CK(cudaMemcpyAsync(b->d_timers + (size_t)l * b->K + k, &d, sizeof(d), cudaMemcpyHostToDevice, b->stream));
    CK(cudaStreamSynchronize(b->stream));
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
  uint32_t l0 = 0;
  if (!id_range(b->cfg.sub_id_base, b->n_next, first_sub, n, &l0)) return CPBUS_ENOENT;
  for (uint32_t i = 0; i < n; i++) if (b->h_released[l0 + i]) return CPBUS_ENOENT;   // as an id never handed out
  int rc = enter(b); if (rc) return rc;
  if ((rc = flush_staged(b, b->now))) return rc;
  if (b->h_timers.empty()) timer_table(b);
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
    const HostTimer& t = timer_arm(b, (size_t)(l0 + i) * b->K, period_ns, source_ids ? source_ids[i] : source_id0 + i, oneshot != 0);
    if (b->sparse) b->due.put((l0 + i) * b->K, t.next_due);
    DevTimer& d = dev[(size_t)i * b->K];
    d.next_due = t.next_due; d.period = oneshot ? 0 : period_ns; d.source_id = t.source_id; d.fired = 0; d.pad[0] = d.pad[1] = 0;
  }
  CK(cudaMemcpyAsync(b->d_timers + (size_t)l0 * b->K, dev.data(), dev.size() * sizeof(DevTimer), cudaMemcpyHostToDevice, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  return push_mask_words(b, l0, n);
} CPBUS_CATCH

// cpbus_timer_cancel's refusal before its flush (CPBUS_ENOENT: no such slot), or CPBUS_OK with the slot's mailbox and index
static int timer_cancel_check(const cpbus* b, uint32_t timer_id, uint32_t* l, uint32_t* k) {
  if (!b->K || b->h_timers.empty()) return CPBUS_ENOENT;
  const uint32_t slot_index = timer_id & kTimerSlotMask;
  *l = slot_index / b->K; *k = slot_index % b->K;
  return *l < b->n_next ? CPBUS_OK : CPBUS_ENOENT;
}

// The host half of cpbus_timer_cancel, after its flush and the one-shots' retirement.
static int timer_cancel_host(cpbus* b, uint32_t timer_id, uint32_t l, uint32_t k) {
  const HostTimer& t = b->h_timers[(size_t)l * b->K + k];
  if (!t.active || t.gen != timer_id >> kTimerSlotBits) return CPBUS_ENOENT;   // already fired / cancelled, or the slot has been re-armed since
  timer_disarm(b, (size_t)l * b->K + k, /*reset_bound=*/true);
  if (b->sparse) b->due.drop(l * b->K + k);
  return CPBUS_OK;
}

int cpbus_timer_cancel(cpbus_t* b, uint32_t timer_id) try {
  if (!b) return CPBUS_EINVAL;
  uint32_t l = 0, k = 0;
  int rc = timer_cancel_check(b, timer_id, &l, &k); if (rc) return rc;
  if ((rc = enter(b))) return rc;
  if ((rc = flush_staged(b, b->now))) return rc;   // firings due before the cancel still happen
  retire_oneshots(b, b->last_watermark);
  if ((rc = timer_cancel_host(b, timer_id, l, k))) return rc;
  CK(cudaMemsetAsync(b->d_timers + (size_t)l * b->K + k, 0xFF, sizeof(DevTimer), b->stream));
  CK(cudaStreamSynchronize(b->stream));
  return push_mask_words(b, l, 1);
} CPBUS_CATCH

// The bulk membership calls (cpbus_unsubscribe_many, cpbus_set_mask_many, cpbus_timer_cancel_many): each element as its
// single call would apply it, in array order.  check(i) is element i's refusal before the single call's flush (CPBUS_OK:
// none); the flush runs once, where the first element that passes its check would run it, then after_flush(), then
// apply(i, &l, &clear) for each element that passed: CPBUS_OK with its mailbox l and the timer slots it disarms, or its
// refusal.  The flush's CPBUS_EAGAIN (or an error) is returned with nothing applied and status / applied not written.
// Every mailbox an applied element touched then gets one membership_kernel entry with its final mask word: one H2D copy,
// one launch and one synchronisation, where the single calls take one synchronised round trip each.
template <class Check, class AfterFlush, class Apply>
static int membership_many(cpbus* b, uint32_t n, int* status, uint32_t* applied, Check&& check, AfterFlush&& after_flush,
                           Apply&& apply) {
  std::vector<int> st(n);
  bool any = false;
  for (uint32_t i = 0; i < n; i++) any |= (st[i] = check(i)) == CPBUS_OK;
  std::vector<uint64_t> touched;   // mailbox << 32 | timer slots disarmed, one per applied element
  if (any) {
    int rc = enter(b); if (rc) return rc;
    if ((rc = flush_staged(b, b->now))) return rc;
    after_flush();
    for (uint32_t i = 0; i < n; i++) {
      if (st[i] != CPBUS_OK) continue;
      uint32_t l = 0, clear = 0;
      if ((st[i] = apply(i, &l, &clear)) == CPBUS_OK) touched.push_back((uint64_t)l << 32 | clear);
    }
  }
  if (!touched.empty()) {
    std::sort(touched.begin(), touched.end());
    std::vector<MemberOp> ops;
    for (uint64_t t : touched) {
      const uint32_t l = (uint32_t)(t >> 32);
      if (ops.empty() || ops.back().local != l) ops.push_back(MemberOp{l, 0u, 0u, 0u});
      ops.back().clear_slots |= (uint32_t)t;
    }
    for (MemberOp& op : ops) op.mask_word = mask_word(b, op.local);
    CK(b->d_member.grow(ops.size(), 1024));   // (every bulk call ends in a synchronisation: no kernel reads the old list)
    // (pageable source: the call returns once the list has been taken, and the copy runs in stream order)
    CK(cudaMemcpyAsync(b->d_member, ops.data(), ops.size() * sizeof(MemberOp), cudaMemcpyHostToDevice, b->stream));
    membership_kernel<<<(uint32_t)((ops.size() + kThreads - 1) / kThreads), kThreads, 0, b->stream>>>(
        b->d_ctl, b->d_timers, b->d_member, (uint32_t)ops.size(), b->K);
    CK(cudaGetLastError());
    b->st.kernel_launches++;
    CK(cudaStreamSynchronize(b->stream));
  }
  uint32_t ok = 0;
  for (uint32_t i = 0; i < n; i++) ok += st[i] == CPBUS_OK ? 1u : 0u;
  if (status && n) memcpy(status, st.data(), (size_t)n * sizeof(int));
  if (applied) *applied = ok;
  return CPBUS_OK;
}

int cpbus_unsubscribe_many(cpbus_t* b, const uint32_t* sub_ids, uint32_t n, int* status, uint32_t* applied) try {
  if (!b || (!sub_ids && n)) return CPBUS_EINVAL;
  return membership_many(b, n, status, applied,
      [&](uint32_t i) { uint32_t l; return sub_index(b, sub_ids[i], &l) ? CPBUS_OK : CPBUS_ENOENT; },
      [] {},
      [&](uint32_t i, uint32_t* l, uint32_t* clear) { *l = sub_ids[i] - b->cfg.sub_id_base; return unsubscribe_host(b, *l, clear); });
} CPBUS_CATCH

int cpbus_set_mask_many(cpbus_t* b, const uint32_t* sub_ids, const uint32_t* code_masks, uint32_t n, int* status,
                        uint32_t* applied) try {
  if (!b || ((!sub_ids || !code_masks) && n)) return CPBUS_EINVAL;
  return membership_many(b, n, status, applied,
      [&](uint32_t i) {
        uint32_t l = 0;
        if (!sub_index(b, sub_ids[i], &l)) return CPBUS_ENOENT;
        return b->h_active[l] ? CPBUS_OK : CPBUS_ECLOSED;
      },
      [] {},
      [&](uint32_t i, uint32_t* l, uint32_t*) { *l = sub_ids[i] - b->cfg.sub_id_base; set_mask_host(b, *l, code_masks[i]); return CPBUS_OK; });
} CPBUS_CATCH

int cpbus_timer_cancel_many(cpbus_t* b, const uint32_t* timer_ids, uint32_t n, int* status, uint32_t* applied) try {
  if (!b || (!timer_ids && n)) return CPBUS_EINVAL;
  return membership_many(b, n, status, applied,
      [&](uint32_t i) { uint32_t l, k; return timer_cancel_check(b, timer_ids[i], &l, &k); },
      [&] { retire_oneshots(b, b->last_watermark); },
      [&](uint32_t i, uint32_t* l, uint32_t* clear) {
        uint32_t k = 0;
        timer_cancel_check(b, timer_ids[i], l, &k);
        *clear = 1u << k;
        return timer_cancel_host(b, timer_ids[i], *l, k);
      });
} CPBUS_CATCH

static_assert(sizeof(cpbus_timer_spec) == 24, "cpbus_timer_spec is part of the ABI");

// cpbus_timer_add's refusals before its flush: CPBUS_EINVAL, CPBUS_ENOSPC (no timer slots at all), CPBUS_ENOENT
static int timer_add_check(const cpbus* b, const cpbus_timer_spec& s) {
  if (!s.period_ns) return CPBUS_EINVAL;
  if (!b->K) return CPBUS_ENOSPC;
  uint32_t l = 0;
  return sub_index(b, s.sub_id, &l) ? CPBUS_OK : CPBUS_ENOENT;
}

// cpbus_timer_add for each element in array order, with one flush and one timer_arm_kernel launch: each applied element
// arms the host table (and the due index) as the single call does, and its slot gets one entry carrying its DevTimer image
// and the mailbox's final mask word.
int cpbus_timer_add_list(cpbus_t* b, const cpbus_timer_spec* specs, uint32_t n, uint32_t* timer_ids, int* status,
                         uint32_t* applied) try {
  if (!b || (!specs && n)) return CPBUS_EINVAL;
  std::vector<int> st(n);
  std::vector<uint32_t> ids(n);
  bool any = false;
  for (uint32_t i = 0; i < n; i++) any |= (st[i] = timer_add_check(b, specs[i])) == CPBUS_OK;
  std::vector<TimerArmOp> ops;
  if (any) {
    int rc = enter(b); if (rc) return rc;
    if ((rc = flush_staged(b, b->now))) return rc;
    if (b->h_timers.empty()) timer_table(b);
    // Once for the whole list, where the loop retires before every element: a one-shot armed here is due after the clock,
    // which no launched watermark passes, so the loop would retire none of this call's own one-shots between elements.
    retire_oneshots(b, b->last_watermark);
    for (uint32_t i = 0; i < n; i++) {
      if (st[i] != CPBUS_OK) continue;
      const cpbus_timer_spec& s = specs[i];
      const uint32_t l = s.sub_id - b->cfg.sub_id_base;
      if (!b->h_active[l]) { st[i] = CPBUS_ECLOSED; continue; }
      uint32_t k = 0;
      while (k < b->K && b->h_timers[(size_t)l * b->K + k].active) k++;
      if (k == b->K) { st[i] = CPBUS_ENOSPC; continue; }
      const uint32_t slot = l * b->K + k;
      HostTimer& t = timer_arm(b, slot, s.period_ns, s.source_id, s.oneshot != 0);
      if (b->sparse) b->due.put(slot, t.next_due);
      t.gen = (uint8_t)((t.gen + 1) & 0x3F);
      ids[i] = slot | ((uint32_t)t.gen << kTimerSlotBits);
      ops.push_back(TimerArmOp{t.next_due, s.oneshot ? 0 : s.period_ns, s.source_id, slot, l, 0u});
    }
  }
  if (!ops.empty()) {
    for (TimerArmOp& op : ops) op.mask_word = mask_word(b, op.local);
    CK(b->d_arm.grow(ops.size(), 1024));   // (every list call ends in a synchronisation: no kernel reads the old list)
    // (pageable source: the call returns once the list has been taken, and the copy runs in stream order)
    CK(cudaMemcpyAsync(b->d_arm, ops.data(), ops.size() * sizeof(TimerArmOp), cudaMemcpyHostToDevice, b->stream));
    timer_arm_kernel<<<(uint32_t)((ops.size() + kThreads - 1) / kThreads), kThreads, 0, b->stream>>>(
        b->d_ctl, b->d_timers, b->d_arm, (uint32_t)ops.size());
    CK(cudaGetLastError());
    b->st.kernel_launches++;
    CK(cudaStreamSynchronize(b->stream));
  }
  if (timer_ids)
    for (uint32_t i = 0; i < n; i++) if (st[i] == CPBUS_OK) timer_ids[i] = ids[i];
  if (status && n) memcpy(status, st.data(), (size_t)n * sizeof(int));
  if (applied) *applied = (uint32_t)ops.size();
  return CPBUS_OK;
} CPBUS_CATCH

// Subscriber id reuse.  Every mailbox a call touches gets one slot_reset_kernel entry: the list is [entries | pair rows],
// one H2D copy, one launch and one synchronisation (none when nothing is applied).  A reset mailbox has all ring_cap slots
// of room, so the lossless room bound (a lower bound of the fullest mailbox's room) stays valid without an update.
static int slot_reset(cpbus* b, const std::vector<SlotResetOp>& ops, const std::vector<uint2>& rows) {
  if (ops.empty()) return CPBUS_OK;
  const size_t head = ops.size() * sizeof(SlotResetOp), bytes = head + rows.size() * sizeof(uint2);
  std::vector<unsigned char> list(bytes);
  memcpy(list.data(), ops.data(), head);
  if (!rows.empty()) memcpy(list.data() + head, rows.data(), rows.size() * sizeof(uint2));
  CK(b->d_reset.grow(bytes, 4096));   // (every call ends in a synchronisation: no kernel reads the old list)
  // (pageable source: the call returns once the list has been taken, and the copy runs in stream order)
  CK(cudaMemcpyAsync(b->d_reset, list.data(), bytes, cudaMemcpyHostToDevice, b->stream));
  slot_reset_kernel<<<(uint32_t)((ops.size() + kThreads - 1) / kThreads), kThreads, 0, b->stream>>>(
      b->d_ctl, b->d_taken.get(), b->d_pairs.get(), b->K ? b->d_timers.get() : nullptr,
      reinterpret_cast<const SlotResetOp*>(b->d_reset.get()), (uint32_t)ops.size(),
      reinterpret_cast<const uint2*>(b->d_reset.get() + head), b->K);
  CK(cudaGetLastError());
  b->st.kernel_launches++;
  CK(cudaStreamSynchronize(b->stream));
  return CPBUS_OK;
}

// cpbus_release_many's refusal of element sub_id before its flush: CPBUS_ENOENT (never handed out, or released), CPBUS_EINVAL
// (still subscribed) or CPBUS_OK
static int release_check(const cpbus* b, uint32_t sub_id) {
  uint32_t l = 0;
  if (!sub_index(b, sub_id, &l)) return CPBUS_ENOENT;
  return b->h_active[l] ? CPBUS_EINVAL : CPBUS_OK;
}

// The host half of a release: mailbox l (unsubscribed) goes back to the state of a slot never handed out, and its id to the
// free set; its exact cases go to *touched for the call's one purge of the case lists (SubIndex::purge_released).  Unsubscribing already took it out of the registry's counts, the code lists, the due index and the timer table;
// the timer slots keep their generations, so an old occupant's timer ids stay stale.
static void release_host(cpbus* b, uint32_t l, std::vector<uint64_t>* touched) {
  b->h_released[l] = 1;
  b->free_ids.push_back(l);
  std::push_heap(b->free_ids.begin(), b->free_ids.end(), std::greater<uint32_t>());
  b->h_mask[l] = 0;
  if (!b->h_npairs.empty()) b->h_npairs[l] = 0;
  if (b->sparse_records) b->rec_index.release_cases(l, touched);
  if (b->K && !b->h_timers.empty())
    for (uint32_t k = 0; k < b->K; k++) {
      HostTimer& t = b->h_timers[(size_t)l * b->K + k];
      const uint8_t gen = t.gen;
      t = HostTimer{};
      t.gen = gen;
      if (b->sparse) b->due.drop(l * b->K + k);
    }
  b->order_dirty = true;
}

int cpbus_release_many(cpbus_t* b, const uint32_t* sub_ids, uint32_t n, int* status, uint32_t* applied) try {
  if (!b || (!sub_ids && n)) return CPBUS_EINVAL;
  std::vector<int> st(n);
  bool any = false;
  for (uint32_t i = 0; i < n; i++) any |= (st[i] = release_check(b, sub_ids[i])) == CPBUS_OK;
  std::vector<SlotResetOp> ops;
  if (any) {
    int rc = enter(b); if (rc) return rc;
    if ((rc = flush_staged(b, b->now))) return rc;   // ordered with publishes, like Unsubscribe
    std::vector<uint64_t> touched;   // the released subscribers' exact cases (sparse records)
    for (uint32_t i = 0; i < n; i++) {
      if (st[i] != CPBUS_OK) continue;
      const uint32_t l = sub_ids[i] - b->cfg.sub_id_base;
      if (b->h_released[l]) { st[i] = CPBUS_ENOENT; continue; }   // an earlier element released it
      release_host(b, l, &touched);
      ops.push_back(SlotResetOp{l, 0u, kResetNoRow, 0u});
    }
    if (!touched.empty()) b->rec_index.purge_released(touched, b->h_released.data());
  }
  const int rc = slot_reset(b, ops, {});
  if (rc) return rc;
  if (b->sparse_drains && !ops.empty()) {   // (after the reset: a drain between the two sees a superset)
    std::lock_guard<std::mutex> g(b->mu);
    b->ready_ix.released(&ops[0].local, ops.size(), sizeof(SlotResetOp) / sizeof(uint32_t));
  }
  if (status && n) memcpy(status, st.data(), (size_t)n * sizeof(int));
  if (applied) *applied = (uint32_t)ops.size();
  return CPBUS_OK;
} CPBUS_CATCH

// The argument checks of cpbus_subscribe_pairs_many, with pairs / n_pairs NULL meaning no cases
int cpbus_host::subscribe_list_check(const uint32_t* n_pairs, const cpbus_pair* pairs, uint32_t n) {
  if (!n_pairs) return CPBUS_OK;
  if (!pairs) return CPBUS_EINVAL;
  for (uint32_t i = 0; i < n; i++) {
    if (n_pairs[i] > CPBUS_MAX_PAIRS) return CPBUS_EINVAL;
    for (uint32_t j = 0; j < n_pairs[i]; j++) if (pairs[(size_t)i * CPBUS_MAX_PAIRS + j].code >= CPBUS_N_CODES) return CPBUS_EINVAL;
  }
  return CPBUS_OK;
}

int cpbus_subscribe_list(cpbus_t* b, const uint32_t* code_masks, const cpbus_pair* pairs, const uint32_t* n_pairs, uint32_t n,
                         uint32_t* sub_ids) try {
  if (!b || !n || !sub_ids || subscribe_list_check(n_pairs, pairs, n)) return CPBUS_EINVAL;
  if (b->free_ids.size() + (uint64_t)(b->N - b->n_next) < n) return CPBUS_ENOSPC;
  int rc = enter(b); if (rc) return rc;
  if ((rc = flush_staged(b, b->now))) return rc;   // ordered with publishes
  bool cases = false;   // some subscriber keeps a case its mask does not cover: it needs the pair tables
  for (uint32_t i = 0; n_pairs && !cases && i < n; i++) {
    const uint32_t m = code_masks ? code_masks[i] : CPBUS_MASK_ALL;
    for (uint32_t j = 0; j < n_pairs[i]; j++) cases |= !((m >> pairs[(size_t)i * CPBUS_MAX_PAIRS + j].code) & 1u);
  }
  if (cases && (rc = pair_tables(b))) return rc;
  std::vector<SlotResetOp> ops(n);
  std::vector<uint2> rows;
  uint2 row[CPBUS_MAX_PAIRS];
  for (uint32_t i = 0; i < n; i++) {   // lowest free id first: the released ones ascending, then fresh ones
    uint32_t l = b->n_next;
    if (!b->free_ids.empty()) {
      l = b->free_ids.front();
      std::pop_heap(b->free_ids.begin(), b->free_ids.end(), std::greater<uint32_t>());
      b->free_ids.pop_back();
      b->h_released[l] = 0;
    } else {
      b->n_next++;
    }
    subscribe_host(b, l, code_masks ? code_masks[i] : CPBUS_MASK_ALL);
    ops[i] = SlotResetOp{l, 0u, kResetNoRow, 0u};
    if (n_pairs && b->d_pairs) {
      for (uint2& r : row) r = make_uint2(kPairNone, kPairNone);
      if (pairs_host(b, l, pairs + (size_t)i * CPBUS_MAX_PAIRS, n_pairs[i], row)) {
        ops[i].row = (uint32_t)(rows.size() / CPBUS_MAX_PAIRS);
        rows.insert(rows.end(), row, row + CPBUS_MAX_PAIRS);
      }
    }
    ops[i].mask_word = mask_word(b, l);
    sub_ids[i] = b->cfg.sub_id_base + l;
  }
  b->n_active += n; b->order_dirty = true;
  return slot_reset(b, ops, rows);
} CPBUS_CATCH

int cpbus_publish(cpbus_t* b, const cpbus_event* ev, size_t n) try {
  if (!b || (!ev && n)) return CPBUS_EINVAL;
  int rc = enter(b); if (rc) return rc;
  return publish_burst(b, ev, n);
} CPBUS_CATCH

int cpbus_send(cpbus_t* b, uint32_t sub_id, const cpbus_event* ev) try {
  if (!b || !ev || ev->code >= CPBUS_N_CODES) return CPBUS_EINVAL;
  uint32_t l = 0;
  if (!sub_index(b, sub_id, &l)) return CPBUS_ENOENT;
  if (!b->h_active[l]) return CPBUS_ECLOSED;   // the mailbox is gone (Go: send on a closed channel panics)
  int rc = enter(b); if (rc) return rc;
  if ((rc = stage_one(b, ev->code, ev->source_id, sub_id, CPBUS_F_UNICAST))) return rc;
  b->publishes++;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_advance(cpbus_t* b, uint64_t now_ns) try {
  if (!b) return CPBUS_EINVAL;
  int rc = follow_resolve(b); if (rc) return rc;   // the clock moves with the batches that followers fanned out
  if (now_ns > b->now && (rc = dev_guard(b))) return rc;
  return advance_clock(b, now_ns);
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
  b->publishes += n; b->seq += n;
  return CPBUS_OK;
}

// (CPBUS_CFG_DROP_MISSED_TICKS: a device batch moves the clock by its watermark, which no cpbus_advance sees)
int cpbus_publish_device(cpbus_t* b, const void* d_events, size_t n, uint64_t watermark_ns) try {
  if (b && b->drop_missed) return CPBUS_EINVAL;
  return publish_device_impl(b, d_events, n, watermark_ns, false, nullptr, 0);
} CPBUS_CATCH

// Multi-GPU ingest fused into the fan-out kernel: d_events (and d_next) may point into ANOTHER GPU's HBM (the
// publisher's event stream, peer-mapped over NVLink).  One CTA pulls the batch across the link, stages it in local
// HBM and publishes it with the batch descriptor; if the caller names the NEXT batch, that one is pulled by the
// same launch while its stores are in flight, so the following call starts from local memory.  No collective.
int cpbus_publish_device_staged(cpbus_t* b, const void* d_events, size_t n, uint64_t watermark_ns, const void* d_next, size_t n_next) try {
  if (b && b->drop_missed) return CPBUS_EINVAL;
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
  DeviceBuf<RoundCursor> d_cursor;           // lossless rounds (cpbus_stream_round_next): {batch, offset} on the device
  unsigned long long stalled_rounds = 0;     // ... rounds resolved so far that moved nothing
  unsigned long long pub_seq = 0;            // publisher: publish ordinal stamped into the next record (CPBUS_PUT_STAMP)
  unsigned long long min_ack = 0;            // publisher: cached min over the consumers' acks
  // publisher staging: pinned payload + header buffers, copies on their own stream
  static constexpr int kStage = 8;
  PinnedBuf<cpbus_event> h_stage[kStage];
  PinnedBuf<StreamHdr> h_hdr;                // kStage headers
  PinnedBuf<unsigned long long> h_ack;       // kStreamMaxConsumers x 4 words
  CudaEvent staged_done[kStage];
  CudaStream put_stream;
  // lossless across processes (cpbus_stream_offer / _agree): admission rounds agreed so far, and this round's state
  unsigned long long agree_round = 0;
  bool offered = false;
  unsigned long long admit_q = 0;            // batch ordinal and shape of the latest cpbus_stream_admit (bounds an offer)
  size_t admit_n = 0;
  MappedBuf<StreamAgreeResult> h_agree;      // written by the agree kernel
  CudaEvent agree_done;
};

static int stream_bind(cpbus_stream* st) {
  st->hdr = reinterpret_cast<StreamHdr*>(st->base + stream_hdr_off());
  st->ack = reinterpret_cast<unsigned long long*>(st->base + stream_ack_off(st->n_slots));
  st->payload = reinterpret_cast<cpbus_event*>(st->base + stream_payload_off(st->n_slots));
  if (st->bus->lossless && st->d_cursor.alloc(1) != cudaSuccess) {   // rounds' cursor
    snprintf(g_cuda_err, sizeof(g_cuda_err), "cudaMalloc(%zu) failed", sizeof(RoundCursor));
    return CPBUS_ENOMEM;
  }
  return CPBUS_OK;
}

int cpbus_stream_create(cpbus_t* b, uint32_t n_slots, uint32_t n_consumers, cpbus_stream_t** out, unsigned char handle[64]) try {
  if (!b || !out || !handle || n_slots < 4 || n_consumers == 0 || n_consumers > kStreamMaxConsumers) return CPBUS_EINVAL;
  *out = nullptr;
  if (b->sparse) return CPBUS_EINVAL;   // stream launches move the clock on the device, past the host's due index
  if (b->drop_missed) return CPBUS_EINVAL;   // ... and by watermarks that no cpbus_advance sees
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
  if (st->put_stream.create() != cudaSuccess) return fail(CPBUS_ECUDA);
  for (int i = 0; i < cpbus_stream::kStage; i++) {
    if (st->h_stage[i].alloc(b->B) != cudaSuccess) return fail(CPBUS_ENOMEM);
    if (st->staged_done[i].create() != cudaSuccess) return fail(CPBUS_ECUDA);
  }
  if (st->h_hdr.alloc(cpbus_stream::kStage) != cudaSuccess || st->h_ack.alloc((size_t)kStreamMaxConsumers * 4) != cudaSuccess)
    return fail(CPBUS_ENOMEM);
  *out = st;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_stream_open(cpbus_t* b, const unsigned char handle[64], uint32_t consumer_index, cpbus_stream_t** out) try {
  if (!b || !out || !handle || consumer_index == 0 || consumer_index >= kStreamMaxConsumers) return CPBUS_EINVAL;
  *out = nullptr;
  if (b->sparse || b->drop_missed) return CPBUS_EINVAL;
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
  if (b->B != owner->B || b->sparse || b->drop_missed) return CPBUS_EINVAL;
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
  if (st->put_stream) cudaStreamSynchronize(st->put_stream);
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

// Publisher: copy the batch into the next slot, then release it (header after payload, same stream).  `device_src`: ev
// holds complete records in device memory (this GPU's or a peer's), copied into the slot as they are (CPBUS_PUT_RAW).
int cpbus_host::stream_put(cpbus_stream* st, const cpbus_event* ev, size_t n, uint64_t now_ns, uint32_t flags, bool device_src) {
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
  const cpbus_event* src = dst;
  if (device_src) src = ev;
  else if (flags & CPBUS_PUT_RAW) { if (n) memcpy(dst, ev, n * sizeof(cpbus_event)); }
  else {
    for (size_t i = 0; i < n; i++) {
      const uint32_t code = ev[i].code;
      if (code >= CPBUS_N_CODES) return CPBUS_EINVAL;
      dst[i].seq = st->pub_seq + i; dst[i].ts_ns = now_ns; dst[i].code = code; dst[i].source_id = ev[i].source_id;
      dst[i].target = CPBUS_TARGET_ALL; dst[i].flags = 0;
    }
  }
  const uint32_t slot = (uint32_t)(q % st->n_slots);
  if (n) CK(cudaMemcpyAsync(st->payload + (size_t)slot * st->B, src, n * sizeof(cpbus_event),
                            device_src ? cudaMemcpyDefault : cudaMemcpyHostToDevice, st->put_stream));
  StreamHdr* hh = &st->h_hdr[s];
  memset(hh, 0, sizeof(*hh));
  hh->seq = q; hh->watermark = now_ns; hh->n = (uint32_t)n;
  if (!(flags & CPBUS_PUT_RAW)) st->pub_seq += n;
  CK(cudaMemcpyAsync(&st->hdr[slot], hh, sizeof(StreamHdr), cudaMemcpyHostToDevice, st->put_stream));   // the release: after the payload
  CK(cudaEventRecord(st->staged_done[s], st->put_stream));
  st->put_seq = q;
  return CPBUS_OK;
}

int cpbus_stream_put(cpbus_stream_t* st, const cpbus_event* ev, size_t n, uint64_t now_ns, uint32_t flags) try {
  if (!st || !st->owner || (!ev && n) || n > st->B) return CPBUS_EINVAL;
  return stream_put(st, ev, n, now_ns, flags, false);
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
  b->publishes += m; b->seq += m;
  b->now = w; b->last_watermark = w;
  if (m) dbg_mark_device_batch(b, launch_seq);
  if (final) { st->get_seq++; st->get_off = 0; return; }
  st->get_off += m;
  b->room_lb = 0;
  b->st.admit_partial++;
}

// Fan out the next m undelivered records of the current batch (throughput mode: m = the whole batch, in one launch).
// `account`: the lead CTA accounts the records as a device-published batch (a group's shards: see group_launch).
int cpbus_host::stream_fanout_prefix(cpbus_stream* st, size_t n, uint64_t now_ns, size_t m, bool account) {
  cpbus* b = st->bus;
  int rc = stream_enter(st, now_ns); if (rc) return rc;
  const bool final = m == n - st->get_off;
  if (m == 0 && !final) return CPBUS_EAGAIN;
  const unsigned long long q = st->get_seq + 1;
  StreamArgs sa;
  LaunchOpts o;
  const cpbus_event* src = stream_launch(st, q, st->get_off, final, sa, o);
  o.account = account;
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
  return stream_fanout_prefix(st, n, now_ns, m, true);
} CPBUS_CATCH

// Every rank (the publisher's included): fan out the next batch of the stream to this GPU's shard.
int cpbus_stream_fanout(cpbus_stream_t* st, size_t n, uint64_t now_ns) try {
  if (!st || n > st->B || st->get_off > n) return CPBUS_EINVAL;
  if (st->bus->lossless) return CPBUS_EINVAL;   // without admission this shard could deliver more than another one does
  return stream_fanout_prefix(st, n, now_ns, n - st->get_off, true);
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
  sa.follow_rec = b->h_follow.dev() + ri; sa.follow_from_host = from_host;
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
  // The ORDERED build rebuilds its mask order, with a sync of the bus stream, at the first fan-out after a membership
  // change.  That sync must come before this round's kernels are queued: behind the agree kernel it would wait for offers
  // that other shards driven by this thread have not queued yet, until the stream timeout.  (A membership change resolves
  // every outstanding round, so nothing of this bus is waiting here when the order is stale.)
  if (b->order_dirty && ordered_build(b) && (rc = rebuild_order(b))) return rc;
  const bool seed_cur = st->follow_out == 0;   // likewise the stream's cursor, while none of this stream's rounds is queued
  RoundParams P{};
  P.dev = b->d_round; P.cur = st->d_cursor; P.rec = b->h_round.dev() + ri;
  P.hdr = st->hdr; P.payload = st->payload; P.ack = st->ack;
  P.n_slots = st->n_slots; P.B = st->B; P.consumer = st->consumer; P.n_consumers = st->n_consumers;
  P.round = st->agree_round + 1;
  P.spin_us = b->stream_spin_us; P.err_word = b->h_err.dev();
  P.admit_batch = b->d_admit_batch; P.ctl = b->d_ctl; P.timers = b->d_timers; P.stats = b->d_stats;
  P.pairs = b->n_paired > 0 ? b->d_pairs.get() : nullptr;
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
  if (!st->h_agree) CK(st->h_agree.alloc(1));
  if (!st->agree_done) CK(st->agree_done.create());
  const unsigned long long r = st->agree_round + 1;
  stream_agree_kernel<<<1, kStreamMaxConsumers, 0, b->stream>>>(st->ack, st->n_consumers, r, b->stream_spin_us, st->h_agree.dev(),
                                                                b->h_err.dev());
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
  uint32_t l = 0;
  if (!sub_index(b, sub_id, &l)) return CPBUS_ENOENT;
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
  uint32_t l = 0;
  if (!id_range(b->cfg.sub_id_base, b->n_next, first_sub, n, &l)) return CPBUS_ENOENT;
  std::lock_guard<std::mutex> g(b->mu);
  int rc = enter(b); if (rc) return rc;
  CK(b->d_drain.grow(cap));
  CK(b->d_drain_idx.grow((size_t)n + 2));   // n entries, then 16 bytes for the kernel's cursor
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
int cpbus_drain_ready(cpbus_t* b, uint32_t first_sub, uint32_t n, uint32_t start_sub, cpbus_event* out, size_t cap,
                      cpbus_ready* ready, size_t ready_cap, size_t* n_ready, size_t* total, uint32_t* next_sub) try {
  if (!b || !out || !ready || !n_ready || !total || !next_sub || !n || !ready_cap) return CPBUS_EINVAL;
  if (!ready_cap_ok(cap, b->R, false, b->lossless)) return CPBUS_EINVAL;
  bool all_taken = false;
  return drain_ready_impl(b, first_sub, n, start_sub, out, cap, ready, ready_cap, n_ready, total, next_sub, &all_taken);
} CPBUS_CATCH

int cpbus_take_ready(cpbus_t* b, uint32_t first_sub, uint32_t n, uint32_t start_sub, cpbus_event* out, size_t cap,
                     cpbus_ready* ready, size_t ready_cap, size_t* n_ready, size_t* total, uint32_t* next_sub) try {
  if (!b || !out || !ready || !n_ready || !total || !next_sub || !n || !ready_cap) return CPBUS_EINVAL;
  if (!ready_cap_ok(cap, b->R, true, b->lossless)) return CPBUS_EINVAL;
  bool all_taken = false;
  return drain_ready_impl(b, first_sub, n, start_sub, out, cap, ready, ready_cap, n_ready, total, next_sub, &all_taken, true);
} CPBUS_CATCH

// The range checks of a paged walk over ids [first_sub, first_sub + n) from start_sub (the sparse drains, cpbus_lagging):
// start_sub within the range (CPBUS_EINVAL), and the range within this shard (CPBUS_ENOENT); *l = the range's first mailbox.
static int walk_range(const cpbus* b, uint32_t first_sub, uint32_t n, uint32_t start_sub, uint32_t* l) {
  if (start_sub < first_sub || start_sub - first_sub >= n) return CPBUS_EINVAL;
  return id_range(b->cfg.sub_id_base, b->n_next, first_sub, n, l) ? CPBUS_OK : CPBUS_ENOENT;
}

// Where that walk goes on after a call that stopped at position `cut` (n or more: it did not stop, so at start_sub again)
static uint32_t walk_next(uint32_t first_sub, uint32_t n, uint32_t start_sub, uint64_t cut) {
  return cut >= n ? start_sub : first_sub + (uint32_t)(((uint64_t)(start_sub - first_sub) + cut) % n);
}

// CPBUS_CFG_SPARSE_DRAINS: b->ready_list = the candidates of b->ready_cand (ascending, in [l, l + n)) with their positions
// in the walk from rot, in position order: those at or after the start, then the ones before it.
static void ready_walk(cpbus* b, uint32_t l, uint32_t n, uint32_t rot) {
  const std::vector<uint32_t>& c = b->ready_cand;
  const size_t split = std::lower_bound(c.begin(), c.end(), l + rot) - c.begin();
  b->ready_list.clear();
  for (size_t i = split; i < c.size(); i++) b->ready_list.push_back(make_uint2(c[i], c[i] - l - rot));
  for (size_t i = 0; i < split; i++) b->ready_list.push_back(make_uint2(c[i], c[i] - l + (n - rot)));
}

// The host part of every sparse drain, synchronous or ticketed, up to its gather (the caller holds b->mu): resolution, the
// device scratch and the scan of mailboxes [l, l + n) from position rot, with at most rcap entries.  The gathers of
// outstanding tickets may still read the scratch on the bus stream, so a scratch buffer that has to grow while a ticket is
// outstanding waits for the stream first.  CPBUS_CFG_SPARSE_DRAINS: with no candidate in the range nothing is enqueued
// (*none = true); with few, the list scan reads only them; otherwise the dense scan runs.
static int ready_scan_enqueue(cpbus* b, uint32_t l, uint32_t n, uint32_t rot, size_t cap, size_t rcap, bool take, bool* none) {
  int rc = enter(b); if (rc) return rc;
  *none = false;
  if (take && !b->d_taken) {   // every cursor 0: max(0, head) = head, so nothing is held
    CK(b->d_taken.alloc(b->N));
    CK(cudaMemsetAsync(b->d_taken, 0, (size_t)b->N * sizeof(unsigned long long), b->stream));
  }
  const bool list = b->sparse_drains && b->ready_ix.candidates(take, l, n, ready_list_max(b->n_next), &b->ready_cand);
  if (list && b->ready_cand.empty()) { *none = true; return CPBUS_OK; }
  if (list) ready_walk(b, l, n, rot);
  const uint32_t tiles = list ? 1u : (n + kReadyTile - 1) / kReadyTile;
  const size_t m = list ? b->ready_list.size() : 0, lb_words = kReadyLbOffset + (list ? 0 : (size_t)tiles);
  if (b->drain_tk_busy && (rcap > b->d_ready.size() || rcap > b->d_ready_slot.size() || lb_words > b->d_ready_lb.size() ||
                           m > b->d_ready_list.size()))
    CK(cudaStreamSynchronize(b->stream));
  CK(b->d_ready.grow(rcap));
  CK(b->d_ready_slot.grow(rcap));
  CK(b->d_ready_lb.grow(lb_words));
  CK(b->d_ready_list.grow(m, 1024));
  const ReadyScan a{b->d_ctl, take ? b->d_taken.get() : nullptr, n, b->R, b->lossless ? 1u : 0u, b->cfg.sub_id_base, cap, rcap,
                    b->d_ready_lb, b->d_ready, b->d_ready_slot};
  if (list) {
    // (pageable source: the call returns once the list has been taken, and the copy runs in stream order)
    CK(cudaMemcpyAsync(b->d_ready_list, b->ready_list.data(), m * sizeof(uint2), cudaMemcpyHostToDevice, b->stream));
    (take ? ready_list_scan_kernel<true> : ready_list_scan_kernel<false>)<<<1, kThreads, 0, b->stream>>>(a, b->d_ready_list,
                                                                                                       (uint32_t)m);
  } else {
    CK(cudaMemsetAsync(b->d_ready_lb + kReadyHdrWords, 0, (lb_words - kReadyHdrWords) * sizeof(unsigned long long), b->stream));
    (take ? ready_scan_kernel<true> : ready_scan_kernel<false>)<<<tiles, kThreads, 0, b->stream>>>(a, l, rot);
  }
  CK(cudaGetLastError());
  return CPBUS_OK;
}

// CPBUS_CFG_SPARSE_DRAINS: whether [first_sub, first_sub + n) is every mailbox subscribed so far
static bool ready_whole(const cpbus* b, uint32_t first_sub, uint32_t n) {
  return first_sub == b->cfg.sub_id_base && n == b->n_next;
}

// CPBUS_CFG_SPARSE_DRAINS: the drain placed at `place` (take: a take_ready) has taken the mailboxes of ready[0..nr); all:
// every ready mailbox of its range, which covers every subscribed mailbox when whole.  The caller holds b->mu.
static void ready_drained(cpbus* b, bool take, uint64_t place, const cpbus_ready* ready, size_t nr, bool whole, bool all) {
  if (!b->sparse_drains) return;
  std::vector<uint32_t>& ids = b->ready_cand;
  ids.resize(nr);
  for (size_t i = 0; i < nr; i++) ids[i] = ready[i].sub_id - b->cfg.sub_id_base;
  b->ready_ix.drained(take, place, ids.data(), nr, 1, whole && all);
}

// The body of cpbus_drain_ready, without its cap >= ring_cap check: a group hands each shard the cap its earlier shards
// left, which can be smaller.  *all_taken: every ready mailbox of the range was taken (then *next_sub = start_sub).
// take: cpbus_take_ready's scan (the caller has checked that the bus is lossless).
int cpbus_host::drain_ready_impl(cpbus_t* b, uint32_t first_sub, uint32_t n, uint32_t start_sub, cpbus_event* out, size_t cap,
                                 cpbus_ready* ready, size_t ready_cap, size_t* n_ready, size_t* total, uint32_t* next_sub,
                                 bool* all_taken, bool take) {
  uint32_t l = 0;
  int rc = walk_range(b, first_sub, n, start_sub, &l); if (rc) return rc;
  std::lock_guard<std::mutex> g(b->mu);
  const size_t rcap = std::min<size_t>(ready_cap, n);   // never more entries than mailboxes
  const uint32_t rot = start_sub - first_sub;
  // the records share cpbus_drain_many's buffer; allocated before the scan, so that a refusal leaves every mailbox as it was
  if ((rc = dev_guard(b))) return rc;
  CK(b->d_drain.grow(cap));
  CK(b->h_ready_hdr.grow(8));
  const uint64_t place = b->ready_ix.place();
  bool none = false;
  if ((rc = ready_scan_enqueue(b, l, n, rot, cap, rcap, take, &none))) return rc;
  if (none) {
    ready_drained(b, take, place, nullptr, 0, ready_whole(b, first_sub, n), true);
    *n_ready = 0; *total = 0; *all_taken = true; *next_sub = start_sub;
    return CPBUS_OK;
  }
  const uint32_t gather_grid = (uint32_t)std::min<size_t>((size_t)b->sm_count * 4, (rcap + kWarpsPerCta - 1) / kWarpsPerCta);
  drain_ready_gather_kernel<<<gather_grid, kThreads, 0, b->stream>>>(b->d_ring, b->R, b->cfg.sub_id_base, b->d_ready,
                                                                      b->d_ready_slot, b->d_ready_lb, b->d_drain, b->h_ready_hdr.dev());
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
  ready_drained(b, take, place, ready, nr, ready_whole(b, first_sub, n), cut >= n);
  *n_ready = nr; *total = tot;
  *all_taken = cut >= n;
  *next_sub = walk_next(first_sub, n, start_sub, cut);
  return CPBUS_OK;
}

// Drain tickets: the scan of the synchronous call, then a gather that writes the records, the ready list and the header
// into the ticket's mapped host buffer; _end waits for the ticket's event and copies them out.
constexpr size_t kTicketHdrBytes = 128;   // the records start on a 128-byte line of the buffer

static int drain_ready_begin(cpbus_t* b, uint32_t first_sub, uint32_t n, uint32_t start_sub, size_t cap, size_t ready_cap,
                             uint32_t* ticket, bool take) {
  if (!b || !ticket || !n || !ready_cap || !ready_cap_ok(cap, b->R, take, b->lossless)) return CPBUS_EINVAL;
  uint32_t l = 0;
  int rc = walk_range(b, first_sub, n, start_sub, &l); if (rc) return rc;
  std::lock_guard<std::mutex> g(b->mu);
  if (b->drain_tk_busy == (uint32_t)cpbus::kDrainTickets) return CPBUS_ENOSPC;   // no result is ever overwritten
  uint32_t i = 0;
  while (b->drain_tk[i].busy) i++;
  cpbus::DrainTicket& t = b->drain_tk[i];
  const size_t rcap = std::min<size_t>(ready_cap, n);
  const size_t rec_bytes = cap * sizeof(cpbus_event);
  // the slot is free: no kernel writes its buffer, which may be replaced
  if ((rc = dev_guard(b))) return rc;
  CK(t.buf.grow(kTicketHdrBytes + rec_bytes + rcap * sizeof(cpbus_ready)));
  if (!(cudaEvent_t)t.done) CK(t.done.create());
  const uint32_t rot = start_sub - first_sub;
  const uint64_t place = b->ready_ix.place();
  bool none = false;
  if ((rc = ready_scan_enqueue(b, l, n, rot, cap, rcap, take, &none))) return rc;
  if (!none) {
    unsigned char* d = t.buf.dev();
    const uint32_t grid = (uint32_t)std::min<size_t>((size_t)b->sm_count * 4, ((cap + 15) / 16 + kWarpsPerCta - 1) / kWarpsPerCta);
    drain_ready_ticket_gather_kernel<<<grid, kThreads, 0, b->stream>>>(
        b->d_ring, b->R, b->cfg.sub_id_base, b->d_ready, b->d_ready_slot, b->d_ready_lb,
        reinterpret_cast<unsigned long long*>(d), reinterpret_cast<uint4*>(d + kTicketHdrBytes),
        reinterpret_cast<uint2*>(d + kTicketHdrBytes + rec_bytes));
    CK(cudaGetLastError());
    b->st.kernel_launches += 2;
    CK(cudaEventRecord(t.done, b->stream));
  }
  t.place = place; t.take = take; t.whole = ready_whole(b, first_sub, n); t.none = none;
  t.busy = true;
  b->drain_tk_busy++;
  t.ticket = (b->drain_tk_gen++ & 0x1FFFFFFFu) << 3 | i;
  t.first = first_sub; t.n = n; t.start = start_sub; t.cap = cap; t.ready_cap = ready_cap;
  *ticket = t.ticket;
  return CPBUS_OK;
}

int cpbus_drain_ready_begin(cpbus_t* b, uint32_t first_sub, uint32_t n, uint32_t start_sub, size_t cap, size_t ready_cap,
                            uint32_t* ticket) try {
  return drain_ready_begin(b, first_sub, n, start_sub, cap, ready_cap, ticket, false);
} CPBUS_CATCH

int cpbus_take_ready_begin(cpbus_t* b, uint32_t first_sub, uint32_t n, uint32_t start_sub, size_t cap, size_t ready_cap,
                           uint32_t* ticket) try {
  return drain_ready_begin(b, first_sub, n, start_sub, cap, ready_cap, ticket, true);
} CPBUS_CATCH

int cpbus_drain_ready_end(cpbus_t* b, uint32_t ticket, cpbus_event* out, size_t cap, cpbus_ready* ready, size_t ready_cap,
                          size_t* n_ready, size_t* total, uint32_t* next_sub) try {
  if (!b || !out || !ready || !n_ready || !total || !next_sub) return CPBUS_EINVAL;
  std::lock_guard<std::mutex> g(b->mu);
  cpbus::DrainTicket& t = b->drain_tk[ticket % cpbus::kDrainTickets];
  if (!t.busy || t.ticket != ticket) return CPBUS_ENOENT;
  if (cap < t.cap || ready_cap < t.ready_cap) return CPBUS_EINVAL;   // the ticket stays outstanding
  int rc = dev_guard(b); if (rc) return rc;
  size_t nr = 0, tot = 0;
  uint64_t cut = t.n;   // a ticket that enqueued nothing: its range held no candidate
  if (!t.none) {
    CK(cudaEventSynchronize(t.done));
    const unsigned char* h = t.buf.get();
    const volatile unsigned long long* hdr = reinterpret_cast<const volatile unsigned long long*>(h);
    nr = (size_t)hdr[0]; tot = (size_t)hdr[1]; cut = hdr[2];
    if (nr) {
      memcpy(ready, h + kTicketHdrBytes + t.cap * sizeof(cpbus_event), nr * sizeof(cpbus_ready));
      memcpy(out, h + kTicketHdrBytes, tot * sizeof(cpbus_event));
    }
  }
  ready_drained(b, t.take, t.place, ready, nr, t.whole, cut >= t.n);
  *n_ready = nr; *total = tot;
  *next_sub = walk_next(t.first, t.n, t.start, cut);
  t.busy = false;
  b->drain_tk_busy--;
  return CPBUS_OK;
} CPBUS_CATCH

// cpbus_ack_many on one bus (the caller has checked the arguments and that the bus is lossless): st[i] for every element.
// Unknown ids get CPBUS_ENOENT and count 0 gets CPBUS_OK on the host; the others go to ack_kernel, one entry per mailbox
// with its elements in array order.  Before the first take nothing is held, so they are refused without a launch.
int cpbus_host::ack_many_impl(cpbus* b, const uint32_t* sub_ids, const uint32_t* counts, uint32_t n, int* st) {
  std::vector<uint64_t> el;   // mailbox << 32 | element index: sorted, each mailbox's elements stay in array order
  for (uint32_t i = 0; i < n; i++) {
    uint32_t l = 0;
    if (!sub_index(b, sub_ids[i], &l)) st[i] = CPBUS_ENOENT;
    else if (counts[i] == 0) st[i] = CPBUS_OK;
    else if (!b->d_taken) st[i] = CPBUS_EINVAL;
    else el.push_back((uint64_t)l << 32 | i);
  }
  if (el.empty()) return CPBUS_OK;
  std::sort(el.begin(), el.end());
  std::vector<AckOp> ops;
  std::vector<uint2> elems(el.size());
  for (size_t j = 0; j < el.size(); j++) {
    const uint32_t l = (uint32_t)(el[j] >> 32), i = (uint32_t)el[j];
    if (ops.empty() || ops.back().local != l) ops.push_back(AckOp{l, (uint32_t)j, 0u, 0u});
    ops.back().n++;
    elems[j] = make_uint2(counts[i], i);
  }
  std::lock_guard<std::mutex> g(b->mu);
  int rc = enter(b); if (rc) return rc;
  const size_t op_bytes = ops.size() * sizeof(AckOp), bytes = op_bytes + elems.size() * sizeof(uint2);
  // (every call ends in a synchronisation: no copy or kernel reads the old list)
  CK(b->d_ack.grow(bytes, 16384));
  CK(b->h_ack.grow(bytes, 16384));
  CK(b->h_ack_status.grow(n, 1024));
  memcpy(b->h_ack, ops.data(), op_bytes);
  memcpy(b->h_ack + op_bytes, elems.data(), bytes - op_bytes);
  CK(cudaMemcpyAsync(b->d_ack, b->h_ack, bytes, cudaMemcpyHostToDevice, b->stream));
  ack_kernel<<<(uint32_t)((ops.size() + kThreads - 1) / kThreads), kThreads, 0, b->stream>>>(
      b->d_ctl, b->d_taken, reinterpret_cast<const AckOp*>(b->d_ack.get()), (uint32_t)ops.size(),
      reinterpret_cast<const uint2*>(b->d_ack + op_bytes), b->h_ack_status.dev());
  CK(cudaGetLastError());
  b->st.kernel_launches++;
  CK(cudaStreamSynchronize(b->stream));
  const volatile int* hs = b->h_ack_status;
  for (const uint2& e : elems) st[e.y] = hs[e.y];
  return CPBUS_OK;
}

// status (may be NULL) = st, *applied (may be NULL) = how many are CPBUS_OK
void cpbus_host::ack_statuses(const std::vector<int>& st, int* status, uint32_t* applied) {
  if (status) memcpy(status, st.data(), st.size() * sizeof(int));
  if (applied) *applied = (uint32_t)std::count(st.begin(), st.end(), CPBUS_OK);
}

int cpbus_ack_many(cpbus_t* b, const uint32_t* sub_ids, const uint32_t* counts, uint32_t n, int* status, uint32_t* applied) try {
  if (!b || ((!sub_ids || !counts) && n)) return CPBUS_EINVAL;
  if (n == 0) {
    if (applied) *applied = 0;
    return CPBUS_OK;
  }
  if (!b->lossless) return CPBUS_EINVAL;   // throughput mode: a held record could be overwritten before its ack
  std::vector<int> st(n);
  const int rc = ack_many_impl(b, sub_ids, counts, n, st.data());
  if (rc) return rc;
  ack_statuses(st, status, applied);
  return CPBUS_OK;
} CPBUS_CATCH

// The look-back scans of cpbus_lagging and cpbus_blockers over n mailboxes: their work buffer's counters and tile status are
// zeroed on the bus stream, and *tiles = the grid, one tile per kReadyTile mailboxes.
static cudaError_t lag_scan_reset(cpbus* b, uint32_t n, uint32_t* tiles) {
  *tiles = (n + kReadyTile - 1) / kReadyTile;
  return cudaMemsetAsync(b->d_lag_lb, 0, (kLagLbOffset + (size_t)*tiles) * sizeof(unsigned long long), b->stream);
}

// Consumer backlog: one read-only scan of the range's control blocks; the entries and the header {selected, cut position,
// summary} arrive in mapped pinned memory, so one sync is the only wait.  *all_returned: every lagging mailbox was returned.
int cpbus_host::lagging_impl(cpbus_t* b, uint32_t first_sub, uint32_t n, uint32_t start_sub, uint32_t min_backlog, cpbus_lag* out,
                             size_t cap, size_t* n_out, uint32_t* next_sub, cpbus_lag_summary* sum, bool* all_returned) {
  static_assert(sizeof(cpbus_lag) == 16 && sizeof(cpbus_lag_summary) == kLagSumWords * sizeof(unsigned long long), "C-ABI layout");
  uint32_t l = 0;
  int rc = walk_range(b, first_sub, n, start_sub, &l); if (rc) return rc;
  std::lock_guard<std::mutex> g(b->mu);
  if ((rc = enter(b))) return rc;
  const size_t ecap = std::min<size_t>(cap, n);   // never more entries than mailboxes
  CK(b->h_lag.grow(ecap));
  uint32_t tiles = 0;
  CK(lag_scan_reset(b, n, &tiles));
  const uint32_t rot = start_sub - first_sub;
  lagging_scan_kernel<<<tiles, kThreads, 0, b->stream>>>(b->d_ctl, l, n, rot, b->R, b->lossless ? 1u : 0u, b->cfg.sub_id_base,
                                                          min_backlog, ecap, b->d_lag_lb, b->h_lag.dev(), b->h_lag_hdr.dev());
  CK(cudaGetLastError());
  b->st.kernel_launches++;
  CK(cudaStreamSynchronize(b->stream));
  const volatile unsigned long long* hdr = b->h_lag_hdr;
  const uint64_t total = hdr[0], cut = hdr[1];
  const size_t got = (size_t)std::min<uint64_t>(total, ecap);
  if (got) memcpy(out, b->h_lag, got * sizeof(cpbus_lag));
  if (sum) {
    uint64_t w[kLagSumWords];
    for (uint32_t i = 0; i < kLagSumWords; i++) w[i] = hdr[2 + i];
    memcpy(sum, w, sizeof(w));
  }
  *n_out = got;
  *all_returned = total <= ecap;   // (then the cut position is n)
  *next_sub = walk_next(first_sub, n, start_sub, cut);
  return CPBUS_OK;
}

int cpbus_lagging(cpbus_t* b, uint32_t first_sub, uint32_t n, uint32_t start_sub, uint32_t min_backlog, cpbus_lag* out,
                  size_t cap, size_t* n_out, uint32_t* next_sub, cpbus_lag_summary* sum) try {
  if (!b || !n_out || !next_sub || !n || (!out && cap)) return CPBUS_EINVAL;
  bool all = false;
  return lagging_impl(b, first_sub, n, start_sub, min_backlog, out, cap, n_out, next_sub, sum, &all);
} CPBUS_CATCH

// The subscribed mailboxes of this shard that refuse the next unit U of a lossless flush: the record `rec` (NULL: ticks
// only) with the ticks due by t.  The caller holds b->mu and has resolved.  No kernel when the room bound proves that U fits
// (admit_fits without taking anything from the bound).
int cpbus_host::blockers_impl(cpbus* b, const cpbus_event* rec, uint64_t t, uint32_t* out, size_t cap, size_t* n) {
  *n = 0;
  const bool timers_on = b->n_timers > 0 && b->K > 0;
  if (b->n_next == 0 || b->room_lb >= admit_need(rec ? 1 : 0, t, b->last_watermark, b->min_period, b->K, timers_on)) return CPBUS_OK;
  uint32_t tiles = 0;
  CK(lag_scan_reset(b, b->n_next, &tiles));
  const size_t ecap = std::min<size_t>(cap, b->n_next);
  blockers_scan_kernel<<<tiles, kThreads, 0, b->stream>>>(b->d_ctl, b->d_timers, b->n_paired > 0 ? b->d_pairs.get() : nullptr, b->n_next,
                                                           b->R, b->K, b->cfg.sub_id_base, timers_on ? 1u : 0u, rec ? 1u : 0u,
                                                           rec ? *rec : cpbus_event{}, t, ecap, b->d_lag_lb, b->h_block.dev(),
                                                           b->h_lag_hdr.dev());
  CK(cudaGetLastError());
  b->st.kernel_launches++;
  CK(cudaStreamSynchronize(b->stream));
  const size_t total = (size_t)*(const volatile unsigned long long*)b->h_lag_hdr;
  if (total && ecap) memcpy(out, b->h_block, std::min(total, ecap) * sizeof(uint32_t));
  *n = total;
  return CPBUS_OK;
}

int cpbus_blockers(cpbus_t* b, uint32_t* out, size_t cap, size_t* n) try {
  if (!b || !n || (!out && cap)) return CPBUS_EINVAL;
  std::lock_guard<std::mutex> g(b->mu);
  int rc = enter(b); if (rc) return rc;
  *n = 0;
  if (!b->lossless) return CPBUS_OK;
  if (b->n_staged) {   // U = the first staged record with the ticks due by its ts_ns
    const cpbus_event e = b->h_batch[b->cur][0];
    return blockers_impl(b, &e, e.ts_ns, out, cap, n);
  }
  if (b->n_timers == 0 || b->now == b->last_watermark) return CPBUS_OK;   // the next flush launches nothing (flush_staged)
  return blockers_impl(b, nullptr, b->now, out, cap, n);
} CPBUS_CATCH

// The next unit of a lossless stream shard, by cpbus_stream_admit's rules: the undelivered remainder of its current batch
// (after resolution, the batch and offset the device cursor holds) with the watermark from the slot header.  r >= 2
// records: the first with the ticks due by its ts_ns; r = 1: that record with the ticks due by the watermark (admit holds
// a last record back when those do not fit); r = 0: the ticks due by the watermark.  The record is one 32-byte copy from
// the slot, local or peer-mapped, as cpbus_stream_admit copies the remainder.
int cpbus_stream_blockers(cpbus_stream_t* st, uint32_t* out, size_t cap, size_t* n) try {
  if (!st || !n || (!out && cap)) return CPBUS_EINVAL;
  *n = 0;
  cpbus* b = st->bus;
  std::lock_guard<std::mutex> g(b->mu);
  int rc = enter(b); if (rc) return rc;
  if ((rc = stream_error(b))) return rc;
  if (!b->lossless) return CPBUS_OK;
  const unsigned long long q = st->get_seq + 1;
  StreamHdr h{};
  CK(cudaMemcpyAsync(&h, &st->hdr[q % st->n_slots], sizeof(h), cudaMemcpyDeviceToHost, b->result_stream));
  CK(cudaStreamSynchronize(b->result_stream));
  if (h.seq != q) return CPBUS_OK;   // not released yet: the shard waits for the publisher, not for a consumer
  if (h.n > st->B || h.n < st->get_off) return CPBUS_EINVAL;
  // A watermark behind the clock or beyond the timer window makes admission fail with CPBUS_EORDER, not stall.
  if (h.watermark < b->now || h.watermark - b->last_watermark > max_window(b)) return CPBUS_OK;
  const uint32_t rem = h.n - st->get_off;
  if (rem == 0) return blockers_impl(b, nullptr, h.watermark, out, cap, n);
  cpbus_event e{};
  CK(cudaMemcpyAsync(&e, st->payload + (size_t)(q % st->n_slots) * st->B + st->get_off, sizeof(e), cudaMemcpyDefault,
                     b->result_stream));
  CK(cudaStreamSynchronize(b->result_stream));
  return blockers_impl(b, &e, rem == 1 ? h.watermark : e.ts_ns, out, cap, n);
} CPBUS_CATCH

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
  if (b->sparse_drains) b->ready_ix.consumed();
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_peek_window(cpbus_t* b, uint32_t sub_id, cpbus_event* out, size_t cap, size_t* n) try {
  if (!b || !n || (!out && cap)) return CPBUS_EINVAL;
  uint32_t l = 0;
  if (!sub_index(b, sub_id, &l)) return CPBUS_ENOENT;
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
  uint32_t l = 0;
  if (!id_range(b->cfg.sub_id_base, b->n_next, first_sub, n, &l)) return CPBUS_ENOENT;
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
  uint32_t l = 0;
  if (!id_range(b->cfg.sub_id_base, b->n_next, first_sub, n, &l)) return CPBUS_ENOENT;
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
  const DevResultSlot* src = result_slot(b, b->launch_seq);
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
// the last 10 of each such batch; launches older than kAcctDbgRing are no longer resolvable and are skipped).  f's markers
// name launches of bus b (f = b, or a group and its shard 0).
int cpbus_host::dbg_resolve(HostFront* f, cpbus* b) {
  if (f->dbg_pending.empty()) return CPBUS_OK;
  bool any_marker = false;
  for (const DbgItem& it : f->dbg_pending) any_marker |= it.marker;
  if (any_marker) {
    int rc = dev_guard(b); if (rc) return rc;
    CK(cudaMemcpyAsync(b->host_acct()->tail, b->d_acct->tail, sizeof(b->host_acct()->tail), cudaMemcpyDeviceToHost, b->stream));
    CK(cudaStreamSynchronize(b->stream));
  }
  for (const DbgItem& it : f->dbg_pending) {
    if (!it.marker) { dbg_ring_put(f, it.ev); continue; }
    const DevDbgTail& t = b->host_acct()->tail[it.launch % kAcctDbgRing];
    if (t.launch_seq != it.launch) continue;
    for (uint32_t j = 0; j < t.n_kept && j < (uint32_t)kAcctDbgKeep; j++) dbg_ring_put(f, t.ev[j]);
  }
  f->dbg_pending.clear();
  return CPBUS_OK;
}

int cpbus_debug_events(cpbus_t* b, cpbus_event* out, size_t cap, size_t* n) try {
  if (!b || !n || (!out && cap)) return CPBUS_EINVAL;
  { const int rc = follow_resolve(b); if (rc) return rc; }
  { const int rc = dbg_resolve(b, b); if (rc) return rc; }
  *n = dbg_read(b, out, cap);
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
  CK(cudaMemcpyAsync(b->host_acct()->by_code, b->d_acct->by_code, sizeof(b->host_acct()->by_code), cudaMemcpyDeviceToHost,
                     b->stream));
  CK(cudaStreamSynchronize(b->stream));
  retire_oneshots(b, b->last_watermark);
  b->st.deliveries = b->st.ticks = 0;
  b->st.overwritten = b->h_stats->overwritten;
  for (int i = 0; i < kStatSlots; i++) { b->st.deliveries += b->h_stats->slot[i].deliveries; b->st.ticks += b->h_stats->slot[i].ticks; }
  b->st.n_subs = b->n_active; b->st.n_timers = b->n_timers; b->st.now_ns = b->now;
  b->st.intern_entries = b->sources.size(); b->st.intern_bytes = b->intern_bytes;
  b->st.ephemeral_live = b->eph_live; b->st.ephemeral_recycled = b->eph_recycled;
  *out = b->st;
  out->publishes = b->publishes;
  for (int c = 0; c < CPBUS_N_CODES; c++)   // + device-published batches (kernel-counted)
    out->published_by_code[c] = b->published_by_code[c] + b->host_acct()->by_code[c];
  return CPBUS_OK;
} CPBUS_CATCH

// The {code, source} table of bus b's device-published batches (DevPubAcct), read back behind b's launches.
int cpbus_host::device_pairs(cpbus* b, std::vector<unsigned long long>& keys, std::vector<unsigned long long>& cnts) {
  keys.resize(kAcctPairSlots); cnts.resize(kAcctPairSlots);
  CK(cudaMemcpyAsync(keys.data(), b->d_acct->pair_key, sizeof(unsigned long long) * kAcctPairSlots, cudaMemcpyDeviceToHost, b->stream));
  CK(cudaMemcpyAsync(cnts.data(), b->d_acct->pair_cnt, sizeof(unsigned long long) * kAcctPairSlots, cudaMemcpyDeviceToHost, b->stream));
  CK(cudaStreamSynchronize(b->stream));
  return CPBUS_OK;
}

// containerpilot_events{code, source} (events/bus.go:60-68,130-132): host publishes are counted in cpbus_publish, batches
// that arrive in device memory by the fan-out kernel's lead CTA (DevPubAcct).
int cpbus_publish_counts(cpbus_t* b, cpbus_pair_count* out, size_t cap, size_t* n) try {
  if (!b || !n || (!out && cap)) return CPBUS_EINVAL;
  std::lock_guard<std::mutex> g(b->mu);
  int rc = enter(b); if (rc) return rc;
  std::vector<unsigned long long> keys, cnts;
  if (b->launch_seq && (rc = device_pairs(b, keys, cnts))) return rc;
  pair_counts(b, keys.data(), cnts.data(), keys.size(), out, cap, n);
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_device_ptrs(cpbus_t* b, void** ring, void** ctl) try {
  if (!b) return CPBUS_EINVAL;
  if (ring) *ring = b->d_ring;
  if (ctl) *ctl = b->d_ctl;
  return CPBUS_OK;
} CPBUS_CATCH
