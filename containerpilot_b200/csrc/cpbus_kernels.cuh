// cpbus_kernels.cuh — sm_90a (H100) kernels of the event bus hot path.
//
// Replaces the inner loop of EventBus.Publish (reference events/bus.go:134-138:
// `for subscriber := range bus.registry { subscriber.Receive(event) }`, one
// runtime.chansend per subscriber per event, events/subscriber.go:30-32) and the
// per-timer goroutines of events/timer.go:12-71, for a whole batch of events and
// all subscribers of this GPU's shard in one launch.
//
// Shape of the work: pure integer / byte movement, HBM-write bound.  No tensor
// cores.  One warp owns one subscriber (mailbox) at a time; the batch of 32-byte
// records is staged once per CTA into shared memory with a 1-D TMA bulk copy
// (cp.async.bulk + mbarrier); matches are found with warp ballots; every record
// is written as one full, aligned 32-byte sector (two 16-byte stores from one lane, or
// a lane pair) or, for dense runs, by TMA bulk stores straight out of the staged batch.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/cpbus.h"

namespace cpbus_dev {

constexpr int kWarpsPerCta = 8;
constexpr int kThreads = kWarpsPerCta * 32;
// Every variant of the fan-out kernel is held to 64 registers => 4 CTAs (32 warps) per SM.  ptxas (CUDA 12.9, sm_90a) spills
// nothing in the plain (dense and timers, with or without digest) and ORDERED variants, and 40-76 bytes in the PAIRS
// variants.  Occupancy is the biggest single lever (DESIGN.md §4.1).
constexpr int kCtasPerSm = 4;
constexpr uint32_t kActiveBit = 0x80000000u;   // mask word: subscriber is subscribed
constexpr int kTimerHintShift = 24;            // mask word bits 24..27: #timer slots to look at
constexpr uint32_t kPairBit = 0x10000000u;     // mask word bit 28: subscriber has a {code, source} pair table
constexpr uint32_t kPairNone = 0xFFFFFFFFu;    // code of an unused pair slot
// Fan-out staging: the `present` bit and histogram bucket of every broadcast code >= CPBUS_N_CODES.  The mask word never
// carries bit 17 (code mask in bits 0..16, bookkeeping from bit 24 up), so no mailbox selects such a record.
constexpr uint32_t kCodeOutOfRange = CPBUS_N_CODES;
static_assert(kCodeOutOfRange < (uint32_t)kTimerHintShift,"the out-of-range bit must lie between the code mask and the mask word's bookkeeping bits");
// PAIRS build: per-CTA presence filter over the batch's broadcast {code, source} keys (2 probes into 32,768 bits:
// ~0.1 % false positives at 512 events, never a false negative).  A pair-filtered mailbox whose cases are all absent
// from the batch is finished after 16 lanes x 2 shared-memory probes instead of a 512-event x 16-pair scan.
constexpr uint32_t kPairFilterWords = 1024;
constexpr uint32_t kPairFilterBytes = kPairFilterWords * 4;
__host__ __device__ inline uint32_t pair_key_hash(uint32_t code, uint32_t source_id) {
  uint32_t x = (source_id ^ (code << 27)) * 0x9E3779B1u;
  x ^= x >> 15; x *= 0x85EBCA77u; x ^= x >> 13;
  return x;   // probe bits: x & 32767 and (x >> 15) & 32767
}
constexpr uint64_t kDigestP = 0x9E3779B97F4A7C15ull;
constexpr uint32_t kPowTableLen = 2048 + 65 + 7;   // batch_cap <= 2048

// One timer slot (events/timer.go: one goroutine + ticker).  The first 16 bytes are all the fan-out kernel
// needs to decide whether anything fires; the second half is read only when a tick is actually emitted.
// Disarmed slot: next_due == kTimerIdle.  One-shot: period == 0.
struct __align__(32) DevTimer {
  uint64_t next_due;
  uint64_t period;
  uint32_t source_id;
  uint32_t fired;
  uint32_t pad[2];
};
constexpr uint64_t kTimerIdle = ~0ull;

// Statistics are spread over kStatSlots sector-sized slots: same-address REDs serialise at
// L2, distinct sectors do not.
constexpr int kStatSlots = 256;
struct __align__(32) DevStatSlot { unsigned long long deliveries, ticks, pad[2]; };
struct DevStats {
  DevStatSlot slot[kStatSlots];
  unsigned long long admit_overflow, overwritten;
  unsigned long long admit_max_used;   // lossless admission: max over mailboxes of (undrained records + what the batch would append)
  unsigned long long admit_deficit;    // ... and max over the mailboxes that lack room of (n - longest event prefix they can take)
};

// Accounting of batches that reach the bus already in device memory (cpbus_publish_device*, cpbus_stream_fanout).  What
// cpbus_publish does on the host for host-staged events (events/bus.go:128-139) the fan-out kernel's lead CTA does here:
// per-code publish counts (Metric excluded, bus.go:130), per-{code, source} counts (the label set of the
// `containerpilot_events` counter, bus.go:131) and the last 10 broadcast events of the batch for the debug ring (bus.go:139).
constexpr uint32_t kAcctPairSlots = 1u << 19;   // open addressing (8 MiB of HBM); key = (code << 32 | source_id) + 1, 0 = empty
constexpr int kAcctDbgRing = 64, kAcctDbgKeep = 10;
struct __align__(32) DevDbgTail {
  unsigned long long launch_seq;                 // written last: the slot belongs to this launch
  uint32_t n_broadcast, n_kept;
  cpbus_event ev[kAcctDbgKeep];                  // the batch's last n_kept broadcast events, oldest first
  uint32_t pad[4];
};
struct DevPubAcct {
  unsigned long long by_code[32];
  unsigned long long pair_overflow, pad[3];      // events whose {code, source} found no table slot
  DevDbgTail tail[kAcctDbgRing];
  unsigned long long pair_key[kAcctPairSlots];
  unsigned long long pair_cnt[kAcctPairSlots];
};

// Per-subscriber control block: exactly one 32-byte sector, read once and written once
// per subscriber per launch (the reference's hchan header: qcount/sendx/recvx, runtime/chan.go).
struct __align__(32) SubCtl {
  unsigned long long tail;    // records ever delivered to this mailbox
  unsigned long long head;    // consumer cursor (records ever drained / overwritten)
  unsigned long long digest;  // rolling order-sensitive digest of the delivered sequence
  uint32_t mask;              // code mask | timer hint << 24 | active bit 31
  uint32_t pad;
};

// Per-launch result ring, filled by the fan-out kernel (kResultSub sector-sized sub-slots per launch so
// that the per-CTA REDs do not serialise on one address; the host sums them).
constexpr int kResultRing = 64, kResultSub = 8;
struct __align__(32) DevResultSlot { unsigned long long deliveries, ticks, digest_sum, launch_seq; };

// Publisher's event stream shared between the GPUs of one box (cpbus_stream_*): a ring of batch slots in the publisher
// GPU's HBM.  A slot is complete when its header's seq equals the batch ordinal; the publisher writes the header AFTER
// the payload (stream-ordered copies), consumers' CTA 0 acquires it over NVLink, pulls the payload and acknowledges.
struct __align__(32) StreamHdr { unsigned long long seq, watermark; uint32_t n, pad[3]; };
struct __align__(32) StreamMeta { uint32_t magic, n_slots, batch_cap, n_consumers, pad[4]; };
constexpr uint32_t kStreamMagic = 0x53425043u;   // "CPBS"
constexpr uint32_t kStreamMaxConsumers = 64;
constexpr int kStreamPrefetch = 3;
constexpr unsigned int kErrStreamTimeout = 1u, kErrStreamShape = 2u;
// Follower launches (cpbus_stream_fanout_next) take n and the watermark from the slot header.  A followed batch behind the
// bus clock or beyond the shard's timer window sets kErrFollowOrder (CPBUS_EORDER from then on).  The device clock is a
// pair of {watermark, launch ordinal} words by launch parity: each follower launch's lead CTA writes its watermark (or
// kFollowPoison once a follower aborted: every follower after it is a no-op) into its own pair, and the next follower reads
// its predecessor's pair.  The per-launch record tells the host what the launch took.
constexpr unsigned int kErrFollowOrder = 4u;
constexpr unsigned long long kFollowPoison = ~0ull;
enum : uint32_t { kFollowDelivered = 0u, kFollowAborted = 1u, kFollowSkipped = 2u, kFollowPending = 0xFFFFFFFFu };
struct __align__(16) FollowRec { uint32_t n, status; unsigned long long watermark; };
// where the shape travels to the other CTAs: spare words of the descriptor summary {present, has_unicast, hist[32], pad[6]}
constexpr uint32_t kFollowN = 34, kFollowWLo = 35, kFollowWHi = 36;
__host__ __device__ inline size_t stream_hdr_off() { return sizeof(StreamMeta); }
__host__ __device__ inline size_t stream_ack_off(uint32_t n_slots) { return stream_hdr_off() + (size_t)n_slots * sizeof(StreamHdr); }
__host__ __device__ inline size_t stream_payload_off(uint32_t n_slots) { return stream_ack_off(n_slots) + (size_t)kStreamMaxConsumers * 32; }
__host__ __device__ inline size_t stream_bytes(uint32_t n_slots, uint32_t batch_cap) { return stream_payload_off(n_slots) + (size_t)n_slots * batch_cap * 32; }

// Lossless stream across processes (cpbus_stream_offer / _agree): consumer c posts its admitted prefix for admission round
// r as one word of its ack sector, word 1 + (r & 1).  Two words alternate because a shard that has finished round r may post
// its round r + 1 offer while a slower shard's agree kernel has not read the round r one yet; it cannot get to round r + 2
// before every shard has posted (hence finished agreeing on) round r + 1.  Word: r (31 bits) << 33 | stalled << 32 | prefix.
constexpr unsigned long long kOfferRoundMask = (1ull << 31) - 1;
__host__ __device__ inline uint32_t stream_offer_word_index(uint32_t consumer, unsigned long long round) {
  return 4u * consumer + 1u + (uint32_t)(round & 1ull);
}
__host__ __device__ inline unsigned long long stream_offer_word(unsigned long long round, uint32_t stalled, uint32_t prefix) {
  return ((round & kOfferRoundMask) << 33) | ((unsigned long long)(stalled ? 1u : 0u) << 32) | prefix;
}
// agree kernel -> host (pinned, mapped): the agreed prefix, the OR of the stall bits, 0 / kErrStreamTimeout
struct __align__(16) StreamAgreeResult { uint32_t m, stalled, status, pad; };

// Lossless admission fast path (host cpbus_stream_admit / cpbus_flush and the device round alike): the most one launch of
// n records with watermark w can append to ONE mailbox — every record, plus every firing of its K timer slots in the window.
__host__ __device__ inline uint64_t admit_need(uint64_t n, uint64_t w, uint64_t last_wm, uint64_t min_period, uint32_t K,
                                              bool timers_armed) {
  if (!timers_armed) return n;
  const uint64_t per_slot = (min_period != ~0ull && w > last_wm) ? (w - last_wm) / min_period + 2 : 2;
  return n + (uint64_t)K * per_slot;
}

// Lossless stream rounds on the device (cpbus_stream_round_next): decide (one CTA) -> exact admission pass (grid, exits at
// once on the fast path) -> offer + agree (one CTA) -> fan-out of the agreed prefix (fanout_round_kernel).  Each kernel
// hands the next one its result in RoundDev, on the bus stream; none of them is launched with programmatic dependent
// launch, so each starts after its predecessor has completed and its writes are visible.
// RoundDev: the device copy of the bus state the rounds move (authoritative while rounds are outstanding) and this round's
// scratch.  RoundCursor: a stream's position, {batch, records of it already delivered}.
struct __align__(16) RoundCursor { unsigned long long batch; uint32_t off, pad; };
enum : uint32_t { kRoundOk = 0u, kRoundSkip = 1u, kRoundAbort = 2u };                 // RoundDev::status (decide)
enum : uint32_t { kRoundAdmitNone = 0u, kRoundAdmitSkipped = 1u, kRoundAdmitPass = 2u };   // how the prefix was admitted
struct __align__(32) RoundDev {
  unsigned long long room;       // lower bound of the free slots of the fullest mailbox (cpbus::room_lb)
  unsigned long long now, last_wm;   // the bus clock and the last launched watermark
  unsigned long long poison;     // an earlier round aborted: every round queued behind it is a no-op
  unsigned long long room_full;  // ring_cap: what cpbus_consume_all copies into `room`, ordered on the stream
  // decide -> exact pass -> agree
  unsigned long long q, hw;      // this round's batch ordinal and its header's watermark
  uint32_t off, rem, status, admit;
  // agree -> fan-out: deliver m records from payload index src with watermark w; final: acknowledge batch q
  unsigned long long w;
  uint32_t go, m, src, final;
};
// per-round record for the host (pinned, mapped), written by the agree kernel.  status: kFollowDelivered (the batch is
// complete), kRoundPartial, kRoundStalled (nothing moved: some shard stalled, or the agreed prefix is 0), kFollowAborted,
// kFollowSkipped (queued behind an aborted round)
enum : uint32_t { kRoundPartial = 3u, kRoundStalled = 4u };
struct __align__(32) RoundRec { uint32_t m, status; unsigned long long watermark, room; uint32_t admit, pad; };
struct RoundParams {
  RoundDev* dev; RoundCursor* cur; RoundRec* rec;
  const StreamHdr* hdr; const cpbus_event* payload; unsigned long long* ack;   // the stream (peer pointers off the publisher)
  uint32_t n_slots, B, consumer, n_consumers;
  unsigned long long round;
  uint32_t spin_us; unsigned int* err_word;
  // admission
  cpbus_event* admit_batch; const SubCtl* ctl; const DevTimer* timers; DevStats* stats; const uint2* pairs;
  uint32_t n_subs, ring_cap, K, sub_base, timers_armed;
  uint64_t min_period, window;
  // the first round after the host resolved: the bus state and / or the cursor come from the host
  uint32_t seed_bus, seed_cur;
  unsigned long long seed_room, seed_now, seed_wm, seed_batch;
  uint32_t seed_off;
};
// where the round fan-out's source index travels to the other CTAs: a spare word of the descriptor summary
constexpr uint32_t kRoundSrc = 37;

struct FanoutParams {
  const cpbus_event* batch;   // n_ev records, sorted by ts (HBM)
  cpbus_event* ring;          // [n_subs][R]
  SubCtl* ctl;                // [n_subs]
  DevTimer* timers;           // [n_subs][K] or nullptr
  DevStats* stats;
  const uint64_t* pow_table;  // P^0 .. P^(kPowTableLen-1), computed once at cpbus_create
  unsigned char* desc;        // per-launch batch descriptor, written by CTA 0, read by every other CTA
  unsigned long long* desc_ready;   // holds the launch_seq whose descriptor is complete
  unsigned long long launch_seq;
  DevResultSlot* result;      // this launch's kResultSub sub-slots (zeroed by the previous launch)
  DevResultSlot* result_next; // next launch's sub-slots: CTA 0 zeroes them
  cpbus_event* batch_local;   // staged mode: CTA 0's local copy of a batch it pulled from a peer GPU
  uint32_t staged;            // 1: `batch` may live in another GPU's HBM (NVLink peer mapping): only CTA 0 reads it
  const cpbus_event* prefetch_src;   // next batch in the publisher GPU's HBM (peer pointer) or nullptr
  cpbus_event* prefetch_dst;         // local buffer it is pulled into while this launch's stores are in flight
  uint32_t prefetch_n;
  uint32_t batch_dep;         // 1: `batch` was produced by the previous launch (prefetch buffer): wait for it before staging
  const uint32_t* order;      // ORDERED build: active subscribers sorted by code mask (equal masks are neighbours)
  uint32_t n_order, spw;      // ... how many, and how many consecutive positions each warp takes (<= 32).  Plain build: CTA b
                              // owns subscribers [8 spw b, 8 spw (b + 1))
  uint32_t stage_subs;        // plain build: subscribers whose control blocks and timer slots are staged in shared memory at a time
  uint64_t w_now;             // watermark: timers due <= w_now fire in this launch
  uint32_t n_ev, n_subs, ring_cap, K, sub_base;
  uint32_t use_digest, lossless, timers_on;
  uint32_t smem_cap;          // n_ev rounded up to 32 (shared-memory carve-up)
  uint32_t hints;             // bit0: keep control blocks / timer slots in L2 (evict_last); bit1 (test hook): no CTA waits for
                              // CTA 0's descriptor, every CTA builds its own (the bounded-spin fallback path)
  const uint2* pairs;         // PAIRS build: [n_subs][CPBUS_MAX_PAIRS] exact {code, source_id} cases (unused slot: code = kPairNone)
  // ---- stream mode (staged == 2): the batch is slot `stream_seq % n_slots` of the publisher GPU's flagged ring ----
  const StreamHdr* stream_hdr;       // this batch's header in the publisher's HBM (peer pointer on the other GPUs)
  unsigned long long* stream_ack;    // this consumer's ack word in the publisher's HBM
  unsigned long long stream_seq;     // 1-based ordinal of the batch this launch fans out
  const StreamHdr* stream_next_hdr;  // header of batch stream_seq + 2 (prefetch_src = its payload), or nullptr
  uint32_t stream_off;               // records of this batch delivered by earlier launches (`batch` = slot payload + stream_off)
  uint32_t stream_final;             // 1: this launch completes the batch (header n == stream_off + n_ev) and acknowledges the slot
  unsigned long long* pf_state;      // [kStreamPrefetch] local: pf_state[q % 3] == q  <=>  batch q sits in pf_buf slot q % 3
  cpbus_event* pf_buf;               // kStreamPrefetch local buffers of pf_stride records
  uint32_t pf_stride;
  uint32_t spin_us;                  // bound of the cross-GPU flag wait (0 = default)
  unsigned int* err_word;            // host-mapped: sticky error bits (kErr*)
  DevPubAcct* acct;                  // non-null: this batch did not pass through cpbus_publish; the lead CTA accounts for it
  // ---- follower launch (fanout_follow_kernel only): n_ev and w_now come from the slot header ----
  unsigned long long* follow_clock;  // [4]: {watermark, launch ordinal} of the latest follower launch, by launch parity
  FollowRec* follow_rec;             // host-mapped: what this launch took (written by the lead CTA)
  uint64_t follow_window;            // widest watermark step of one launch (UINT64_MAX: no periodic timer armed)
  uint32_t follow_from_host;         // 1: the previous watermark is w_now (the host clock), not the clock words
  // ---- lossless round (fanout_round_kernel only): n, the watermark and the source come from the agree kernel ----
  const RoundDev* round;
};

// ---------------------------------------------------------------- helpers ---
__host__ __device__ inline uint64_t record_hash_words(uint64_t w0, uint64_t w1, uint64_t w2, uint64_t w3) {
  const uint64_t K0 = 0x9E3779B97F4A7C15ull, K1 = 0xBF58476D1CE4E5B9ull,
                 K2 = 0x94D049BB133111EBull, K3 = 0xD6E8FEB86659FD93ull,
                 K4 = 0xA0761D6478BD642Full;
  uint64_t x = (w0 + K4) * K0; x ^= x >> 32;
  x = (x + w1) * K1; x ^= x >> 32;
  x = (x + w2) * K2; x ^= x >> 32;
  x = (x + w3) * K3; x ^= x >> 29;
  return x;
}

__host__ __device__ inline uint64_t pow_p(uint32_t e) {
  uint64_t r = 1, b = kDigestP;
  while (e) { if (e & 1u) r *= b; b *= b; e >>= 1; }
  return r;
}

#ifdef __CUDACC__
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint64_t shfl64(uint64_t v, int src) {
  uint32_t lo = __shfl_sync(0xffffffffu, (uint32_t)v, src);
  uint32_t hi = __shfl_sync(0xffffffffu, (uint32_t)(v >> 32), src);
  return ((uint64_t)hi << 32) | lo;
}
__device__ __forceinline__ uint64_t warp_sum64(uint64_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    uint32_t lo = __shfl_xor_sync(0xffffffffu, (uint32_t)v, o);
    uint32_t hi = __shfl_xor_sync(0xffffffffu, (uint32_t)(v >> 32), o);
    v += ((uint64_t)hi << 32) | lo;
  }
  return v;
}
__device__ __forceinline__ void st_v4(void* dst, const uint4& a) {
  asm volatile("st.global.v4.b32 [%0], {%1,%2,%3,%4};" ::"l"(dst), "r"(a.x), "r"(a.y), "r"(a.z), "r"(a.w) : "memory");
}
// one full 32-byte sector per lane.  sm_90 has no 256-bit global store: the sector is written as two back-to-back
// 16-byte stores from the same lane, which L2 merges into one full-sector write (no read-for-ownership).
__device__ __forceinline__ void st_v8(void* dst, const uint4& a, const uint4& b) {
  st_v4(dst, a);
  st_v4(reinterpret_cast<unsigned char*>(dst) + 16, b);
}
// Warp-cooperative copy of staged records into a ring: lane l copies staged record i to ring slot (tail + out) & Rm if
// `valid`.  Every lane of the warp must call it.  One lane storing both 16-byte halves of its record leaves each store
// instruction with 32 half-filled sectors, and H100 then sustains about half of the lane-pair rate.  So the two lanes of
// a pair copy one record per instruction together, each lane loading from shared memory the half it stores: each of the
// two store instructions fills 16 whole 32-byte sectors.  Staged layout: planar (PL: half h of record i at s4[h * hi + i])
// or record-major (s4[2 * i + h]).
template <bool PL>
__device__ __forceinline__ void copy_record_pairs(const uint4* s4, uint32_t hi, cpbus_event* ring, uint32_t tail, uint32_t Rm,
                                                  uint32_t i, uint32_t out, bool valid) {
  const uint32_t h = threadIdx.x & 1u, ev = (threadIdx.x & 31u) & ~1u;
  const uint32_t pi = __shfl_xor_sync(0xffffffffu, i, 1), po = __shfl_xor_sync(0xffffffffu, out, 1);
  const uint32_t vm = __ballot_sync(0xffffffffu, valid);
  const uint32_t ie = h ? pi : i, oe = h ? po : out, io = h ? i : pi, oo = h ? out : po;   // the even / odd lane's record
  if ((vm >> ev) & 1u)
    st_v4(reinterpret_cast<unsigned char*>(ring + ((tail + oe) & Rm)) + 16u * h, PL ? s4[h * hi + ie] : s4[2u * ie + h]);
  if ((vm >> (ev + 1u)) & 1u)
    st_v4(reinterpret_cast<unsigned char*>(ring + ((tail + oo) & Rm)) + 16u * h, PL ? s4[h * hi + io] : s4[2u * io + h]);
}
// 32-byte sector / 16-byte half load/store with an L2 evict_last hint: control blocks and timer slots are
// re-read every launch, ring records are write-once streams
__device__ __forceinline__ uint64_t keep_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void ld_half(const void* src, uint4& a, bool hinted);
__device__ __forceinline__ void st_half(void* dst, const uint4& a, bool hinted);
// a whole 32-byte sector as two 16-byte accesses from one lane (sm_90 has no 256-bit global load/store)
__device__ __forceinline__ void ld_sector(const void* src, uint4& a, uint4& b, bool hinted) {
  ld_half(src, a, hinted);
  ld_half(reinterpret_cast<const unsigned char*>(src) + 16, b, hinted);
}
__device__ __forceinline__ void st_sector(void* dst, const uint4& a, const uint4& b, bool hinted) {
  st_half(dst, a, hinted);
  st_half(reinterpret_cast<unsigned char*>(dst) + 16, b, hinted);
}
__device__ __forceinline__ void ld_half(const void* src, uint4& a, bool hinted) {
  const uint64_t pol = hinted ? keep_policy() : 0ull;
  if (hinted)
    asm volatile("ld.global.L2::cache_hint.v4.b32 {%0,%1,%2,%3}, [%4], %5;" : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w) : "l"(src), "l"(pol));
  else
    asm volatile("ld.global.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w) : "l"(src));
}
__device__ __forceinline__ void st_half(void* dst, const uint4& a, bool hinted) {
  const uint64_t pol = hinted ? keep_policy() : 0ull;
  if (hinted)
    asm volatile("st.global.L2::cache_hint.v4.b32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(dst), "r"(a.x), "r"(a.y), "r"(a.z), "r"(a.w), "l"(pol) : "memory");
  else st_v4(dst, a);
}
// TMA 1-D bulk copies (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void* sdst, const void* gsrc, uint32_t bytes, uint64_t* mbar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(sdst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(mbar))
               : "memory");
}
// ... and with the evict_last L2 policy when `hinted`
__device__ __forceinline__ void bulk_g2s_hint(void* sdst, const void* gsrc, uint32_t bytes, uint64_t* mbar, bool hinted) {
  if (!hinted) { bulk_g2s(sdst, gsrc, bytes, mbar); return; }
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
                   smem_u32(sdst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(mbar)), "l"(keep_policy())
               : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* ssrc, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(ssrc)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_init(uint64_t* mbar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(mbar)), "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* mbar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(mbar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* mbar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "CPBUS_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra CPBUS_DONE;\n\t"
      "bra CPBUS_WAIT;\n\t"
      "CPBUS_DONE:\n\t}" ::"r"(smem_u32(mbar)),
      "r"(parity)
      : "memory");
}

// ------------------------------------------------------------- the kernel ---
// Shared memory carve-up (cap = smem_cap records):
//   [0, 32cap)            staged batch (TMA destination)
//   [32cap, 40cap)        record hashes H(e_i)
//   [40cap, 48cap)        {codebit, target} per event
//   [48cap, 56cap+16)     Q[i] = sum_{j<i} H(e_j) P^(n-1-j): prefix sums for O(#ticks) digests of dense runs
//   [.., +160)            descriptor summary {present, has_unicast, hist[32]} (lands with the descriptor's bulk copy)
//   [.., +4096)           PAIRS build only: presence filter of the batch's {code, source} keys (same bulk copy)
//   then                  powers P^0 .. P^(cap+64), BatchSummary (mbarriers, per-CTA accumulators), per-warp tick scratch
//   [fanout_stage_off, ..) plain build: control blocks [stage_subs], then timer slots [stage_subs][K] of the current round
struct BatchSummary {
  uint64_t mbar;
  uint64_t mbar_desc;      // the descriptor's bulk copy (CTAs other than the one that built it)
  uint64_t mbar_state;     // plain build: one phase per staging round of control blocks and timer slots
  uint32_t acc_deliv, acc_ticks, acc_pad[2];   // per-CTA statistics (flushed once at exit)
  uint32_t acc_dig_lo, acc_dig_hi;                     // sum of fold32(new digest), as two 16-bit-limb sums (native 32-bit atomics)
  uint32_t stream_local;   // stream mode: this batch was prefetched into local HBM by an earlier launch
  uint32_t own_desc;       // this CTA builds the descriptor itself (CTA 0, or the bounded wait for CTA 0 ran out)
  uint32_t abort_launch;   // the stream batch never arrived (publisher stalled): deliver nothing
  uint32_t pf_ok;
  uint64_t red[kWarpsPerCta];
};

__host__ __device__ inline size_t fanout_desc_bytes(uint32_t cap) { return (size_t)24 * cap + 16 + 160 + kPairFilterBytes; }

__host__ __device__ inline size_t fanout_smem_bytes(uint32_t cap) {
  const size_t scratch = (cap / 2u > 32u ? cap / 2u : 32u) * sizeof(uint32_t);
  return (size_t)cap * 56 + 16 + 160 + (size_t)(cap + 66) * 8 + sizeof(BatchSummary) + kWarpsPerCta * scratch + 128;
}
__host__ __device__ inline size_t fanout_stage_off(uint32_t cap) { return (fanout_smem_bytes(cap) + 127) & ~(size_t)127; }

// TIMERS=false compiles every timer/tick path out (the host knows when no timer is armed): fewer registers,
// one more resident CTA per SM.
// ORDERED (no-timer build only): warps walk the subscribers in code-mask order, so a run of mailboxes with the same
// mask shares one match/compaction pass and one digest polynomial — filtered fan-out then costs one copy per mailbox
// plus one filter pass per DISTINCT mask in the warp's block, instead of a filter pass per mailbox.
// PAIRS (second-level filter, jobs/jobs.go:188-231): a subscriber whose mask word carries kPairBit also takes the broadcast
// events that equal one of its exact {code, source} cases.  Such mailboxes go through the general two-pass path.
// Plain build (neither ORDERED nor PAIRS): CTA b owns one contiguous range of subscribers.  Their control blocks and timer
// slots arrive in shared memory by bulk copies, stage_subs subscribers per round, instead of as one scattered DRAM read per
// mailbox in the middle of the ring write stream.
// FOLLOW (fanout_follow_kernel, stream mode only): the host does not know the batch's shape.  The lead CTA reads n and the
// watermark from the slot header it acquires anyway, checks the watermark against the device clock (the previous follower's
// watermark) and publishes both with the descriptor; the batch always travels through the lead's local copy.
// ROUND (fanout_round_kernel, lossless stream rounds only; FOLLOW is set too): the shape is what this shard's round agreed
// on.  The lead CTA reads {m, watermark, source index, final} from RoundDev, which the agree kernel wrote earlier on the
// same stream; the kernel is launched without programmatic dependent launch, so that read needs no griddepcontrol.wait.
// A round that delivers nothing (a stall, a prefix of 0, an error) runs as an aborted launch: no record, no tick, no ack.
// The body is included once per kernel, so that the existing kernels are compiled from exactly the code they always were
// (an inlined device function in their place changes how ptxas allocates the PAIRS variants) and FOLLOW and ROUND cost
// them nothing.
template <int STORE, bool TIMERS, bool DIGEST, bool ORDERED, bool PAIRS = false>
__global__ void __launch_bounds__(kThreads, kCtasPerSm) fanout_kernel(const FanoutParams p) {
  constexpr bool FOLLOW = false, ROUND = false;
#include "cpbus_fanout_body.cuh"
}
// Stream follower (cpbus_stream_fanout_next): the same fan-out, shape and watermark taken from the slot header
template <int STORE, bool TIMERS, bool DIGEST, bool ORDERED, bool PAIRS = false>
__global__ void __launch_bounds__(kThreads, kCtasPerSm) fanout_follow_kernel(const FanoutParams p) {
  constexpr bool FOLLOW = true, ROUND = false;
#include "cpbus_fanout_body.cuh"
}
// Lossless stream round (cpbus_stream_round_next): the same fan-out of the prefix the shards agreed on
template <int STORE, bool TIMERS, bool DIGEST, bool ORDERED, bool PAIRS = false>
__global__ void __launch_bounds__(kThreads, kCtasPerSm) fanout_round_kernel(const FanoutParams p) {
  constexpr bool FOLLOW = true, ROUND = true;
#include "cpbus_fanout_body.cuh"
}

// Lossless mode (reference semantics, events/subscriber.go:30-32: a full channel
// blocks the sender): before a batch is fanned out, count for every mailbox what
// the batch would append and flag any that lacks the room.  Thread per subscriber.  (admit_kernel, and the exact pass
// of a lossless stream round, stream_round_admit_kernel)
__device__ __forceinline__ void admit_body(const cpbus_event* batch, uint32_t n_ev, uint64_t w_now, const SubCtl* ctl,
                                           const DevTimer* timers, uint32_t n_subs, uint32_t ring_cap, uint32_t K,
                                           uint32_t sub_base, uint32_t timers_on, DevStats* stats, const uint2* pairs) {
  __shared__ uint32_t hist[32];
  __shared__ uint32_t s_uni;
  __shared__ unsigned long long s_max;
  if (threadIdx.x < 32) hist[threadIdx.x] = 0;
  if (threadIdx.x == 0) { s_uni = 0; s_max = 0; }
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < n_ev; i += blockDim.x) {
    const uint32_t code = batch[i].code, target = batch[i].target;
    if (target == CPBUS_TARGET_ALL) { if (code < 32) atomicAdd(&hist[code], 1u); }
    else atomicAdd(&s_uni, 1u);
  }
  __syncthreads();
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  SubCtl c{};
  if (s < n_subs) c = ctl[s];
  const uint32_t m = c.mask;
  if (s < n_subs && (m & kActiveBit)) {
    uint64_t k = 0;
    for (uint32_t cc = 0; cc < CPBUS_N_CODES; cc++) if ((m >> cc) & 1u) k += hist[cc];
    if (pairs && (m & kPairBit)) {   // second-level filter: broadcast events outside the mask that equal an exact {code, source} case
      const uint2* my = pairs + (size_t)s * CPBUS_MAX_PAIRS;
      for (uint32_t i = 0; i < n_ev; i++) {
        const uint32_t code = batch[i].code;
        if (batch[i].target != CPBUS_TARGET_ALL || code >= CPBUS_N_CODES || ((m >> code) & 1u)) continue;
        const uint32_t src = batch[i].source_id;
        for (uint32_t j = 0; j < CPBUS_MAX_PAIRS; j++) {
          const uint2 pr = my[j];
          if (pr.x == kPairNone) break;
          if (pr.x == code && pr.y == src) { k++; break; }
        }
      }
    }
    if (s_uni) {
      const uint32_t gid = sub_base + s;
      for (uint32_t i = 0; i < n_ev; i++) if (batch[i].target == gid) k++;
    }
    const uint32_t nslots = timers_on ? min((m >> kTimerHintShift) & 0xFu, K) : 0u;
    // due times saturate at kTimerIdle - 1 (the fan-out kernel never fires a tick due at kTimerIdle): count up to there
    const uint64_t w_due = min(w_now, kTimerIdle - 1);
    for (uint32_t t = 0; t < nslots; t++) {
      const DevTimer tm = timers[(size_t)s * K + t];
      if (tm.next_due != kTimerIdle && tm.next_due <= w_due)
        k += tm.period ? (w_due - tm.next_due) / tm.period + 1u : 1u;
    }
    const unsigned long long used = c.tail - c.head + k;
    if (used > ring_cap) {
      atomicAdd(&stats->admit_overflow, 1ull);
      // Per-event blocking (events/subscriber.go:30-32: the publisher stalls at the FIRST event a full channel cannot take):
      // the longest prefix of the batch this mailbox has room for, its share of the ticks due by then included.  Events are
      // sorted by ts; a tick due at d sits in front of the first event with ts >= d.
      const unsigned long long room = ring_cap - min((unsigned long long)ring_cap, c.tail - c.head);
      const uint32_t gid = sub_base + s;
      unsigned long long taken = 0;
      uint32_t prefix = 0;
      for (uint32_t i = 0; i < n_ev; i++) {
        const cpbus_event e = batch[i];
        unsigned long long tks = 0;
        for (uint32_t t = 0; t < nslots; t++) {
          const DevTimer tm = timers[(size_t)s * K + t];
          const uint64_t ts = min(e.ts_ns, kTimerIdle - 1);
          if (tm.next_due != kTimerIdle && tm.next_due <= ts) tks += tm.period ? (ts - tm.next_due) / tm.period + 1u : 1u;
        }
        bool want;
        if (e.target == CPBUS_TARGET_ALL) {
          want = e.code < CPBUS_N_CODES && ((m >> e.code) & 1u);
          if (!want && pairs && (m & kPairBit)) {
            const uint2* my = pairs + (size_t)s * CPBUS_MAX_PAIRS;
            for (uint32_t j = 0; j < CPBUS_MAX_PAIRS && !want; j++) {
              const uint2 pr = my[j];
              if (pr.x == kPairNone) break;
              want = pr.x == e.code && pr.y == e.source_id;
            }
          }
        } else want = e.target == gid;
        if (taken + (want ? 1u : 0u) + tks > room) break;
        taken += want ? 1u : 0u;
        prefix = i + 1;
      }
      atomicMax(&stats->admit_deficit, (unsigned long long)(n_ev - prefix));
    }
    atomicMax(&s_max, used);
  }
  // how full the fullest mailbox would be after this batch: lets the host skip the admission pass (and its sync) for the
  // following batches while they provably fit
  __syncthreads();
  if (threadIdx.x == 0 && s_max) atomicMax(&stats->admit_max_used, s_max);
}
__global__ void admit_kernel(const cpbus_event* batch, uint32_t n_ev, uint64_t w_now, const SubCtl* ctl,
                             const DevTimer* timers, uint32_t n_subs, uint32_t ring_cap, uint32_t K, uint32_t sub_base,
                             uint32_t timers_on, DevStats* stats, const uint2* pairs) {
  admit_body(batch, n_ev, w_now, ctl, timers, n_subs, ring_cap, K, sub_base, timers_on, stats, pairs);
}

// Device-side consumer: every mailbox is read to the end and its records are discarded (head = tail).  Stands in for
// consumers that keep up (benchmarks of the lossless mode; subscribers whose events nobody reads).
__global__ void consume_all_kernel(SubCtl* ctl, uint32_t n) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) ctl[i].head = ctl[i].tail;
}

// Throughput mode: records that were overwritten before the consumer took them.  The fan-out kernel never
// touches `head` (it is consumer-owned); what has been lost is derived: max(0, tail - ring_cap - head).
__global__ void overwritten_kernel(const SubCtl* ctl, uint32_t n, uint32_t ring_cap, unsigned long long* out) {
  unsigned long long acc = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const SubCtl c = ctl[i];
    if (c.tail > ring_cap && c.tail - ring_cap > c.head) acc += c.tail - ring_cap - c.head;
  }
  acc = warp_sum64(acc);
  if ((threadIdx.x & 31) == 0 && acc) atomicAdd(out, acc);
}

// Bulk drain (the mailbox -> `chan Event` bridge for many subscribers at once): one warp per mailbox claims space in a
// contiguous staging buffer with a single atomic, copies its undrained records there in FIFO order and advances the
// consumer cursor.  index[s] = {offset in records, count}; a mailbox that does not fit entirely is left for the next call.
__global__ void drain_many_kernel(SubCtl* ctl, const cpbus_event* ring, uint32_t first, uint32_t n, uint32_t ring_cap,
                                  uint32_t lossless, cpbus_event* out, uint32_t out_cap, uint2* index, unsigned int* cursor) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t i = w; i < n; i += nw) {
    SubCtl* c = ctl + first + i;
    const unsigned long long tail = c->tail;
    unsigned long long head = c->head;
    if (!lossless && tail > ring_cap && tail - ring_cap > head) head = tail - ring_cap;   // overwritten before being taken
    const uint32_t avail = (uint32_t)(tail - head);
    uint32_t off = 0;
    if (lane == 0 && avail) off = atomicAdd(cursor, avail);
    off = __shfl_sync(0xffffffffu, off, 0);
    const bool fits = avail && off + avail <= out_cap;
    if (fits) {
      const cpbus_event* r = ring + (size_t)(first + i) * ring_cap;
      for (uint32_t j = lane; j < avail; j += 32) {
        const uint4* src = reinterpret_cast<const uint4*>(r + ((head + j) & (ring_cap - 1)));
        uint4* dst = reinterpret_cast<uint4*>(out + off + j);
        dst[0] = src[0]; dst[1] = src[1];
      }
    }
    if (lane == 0) {
      index[i] = make_uint2(fits ? off : 0u, fits ? avail : 0u);
      if (fits) c->head = tail;
    }
  }
}

// ---- sparse drain (cpbus_drain_ready) ----------------------------------------------------------------------------------
// Position p in [0, n) is mailbox first + (rot + p) mod n: the range in cyclic order from start_sub.  One single-pass scan
// kernel reads each control block once, numbers the ready mailboxes and their records in position order (decoupled
// look-back over tiles of kReadyTile positions), takes the prefix that fits and writes the ready list; a gather kernel
// then copies the taken runs.  A tile's status word: flag (bits 62-63: 1 = tile aggregate, 2 = inclusive prefix) | ready
// mailboxes (bits 33-61) | records (bits 0-32, saturating).  A shard has fewer than 2^29 mailboxes (each ring is at least
// 2 KiB), and a saturated record count exceeds every allowed cap (< 2^32), so neither field can mislead the cut.
constexpr uint32_t kReadyItems = 4, kReadyTile = kThreads * kReadyItems;
static_assert(kReadyItems * kWarpsPerCta == 32, "one lane per (item, warp) chunk of a tile");
constexpr unsigned long long kLbAgg = 1ull << 62, kLbIncl = 2ull << 62, kLbRecMax = (1ull << 33) - 1;
constexpr uint32_t kReadyHdrWords = 4, kReadyLbOffset = 8;   // lb buffer: [0..3] header, [4] tile counter, [8..] tile status

__device__ __forceinline__ unsigned long long lb_pack(unsigned long long flag, unsigned long long ready, unsigned long long rec) {
  return flag | (ready << 33) | (rec < kLbRecMax ? rec : kLbRecMax);
}

// hdr[0..2] = {mailboxes taken, records taken, position of the first ready mailbox that did not fit (n: none)}; exactly one
// thread writes it: the one holding that mailbox, or the last tile when everything fits.
__global__ void __launch_bounds__(kThreads) drain_ready_scan_kernel(SubCtl* __restrict__ ctl, uint32_t first, uint32_t n,
                                                                    uint32_t rot, uint32_t ring_cap, uint32_t lossless,
                                                                    uint32_t sub_base, unsigned long long cap,
                                                                    unsigned long long ready_cap, unsigned long long* lb,
                                                                    cpbus_ready* __restrict__ ready, uint32_t* __restrict__ slot) {
  __shared__ uint32_t s_tile;
  __shared__ uint32_t s_wr[32];              // per (item, warp) chunk: ready mailboxes, then their exclusive prefix in the tile
  __shared__ unsigned long long s_wc[32];    // ... and records
  __shared__ unsigned long long s_base_r, s_base_c;
  unsigned long long* hdr = lb;
  unsigned long long* status = lb + kReadyLbOffset;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // tiles are numbered in the order the CTAs start, so every predecessor a tile waits for is running or done
  if (threadIdx.x == 0) s_tile = atomicAdd(reinterpret_cast<unsigned int*>(lb + kReadyHdrWords), 1u);
  __syncthreads();
  const uint32_t tile = s_tile;
  uint32_t loc[kReadyItems], r_in[kReadyItems];
  unsigned long long tl[kReadyItems], cur[kReadyItems], hd[kReadyItems], c_in[kReadyItems];
#pragma unroll
  for (uint32_t k = 0; k < kReadyItems; k++) {   // item k of the tile = positions k*kThreads .. +kThreads: coalesced loads
    const uint32_t p = tile * kReadyTile + k * kThreads + threadIdx.x;
    unsigned long long t = 0, h = 0, c = 0;
    uint32_t l = 0;
    if (p < n) {
      unsigned long long q = (unsigned long long)rot + p;
      if (q >= n) q -= n;
      l = first + (uint32_t)q;
      const ulonglong2 th = *reinterpret_cast<const ulonglong2*>(ctl + l);   // {tail, head}
      t = th.x; h = th.y; c = h;
      if (!lossless && t > ring_cap && t - ring_cap > c) c = t - ring_cap;   // overwritten before being taken
    }
    loc[k] = l; tl[k] = t; hd[k] = h; cur[k] = c;
    uint32_t r = t != c ? 1u : 0u;
    unsigned long long s = t - c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t ro = __shfl_up_sync(0xffffffffu, r, o);
      const unsigned long long so = shfl64(s, (int)lane - o);
      if ((int)lane >= o) { r += ro; s += so; }
    }
    r_in[k] = r; c_in[k] = s;
    if (lane == 31) { s_wr[k * kWarpsPerCta + warp] = r; s_wc[k * kWarpsPerCta + warp] = s; }
  }
  __syncthreads();
  if (warp == 0) {
    const uint32_t r0 = s_wr[lane];
    const unsigned long long c0 = s_wc[lane];
    uint32_t r = r0;
    unsigned long long c = c0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t ro = __shfl_up_sync(0xffffffffu, r, o);
      const unsigned long long co = shfl64(c, (int)lane - o);
      if ((int)lane >= o) { r += ro; c += co; }
    }
    s_wr[lane] = r - r0; s_wc[lane] = c - c0;
    const unsigned long long agg_r = __shfl_sync(0xffffffffu, r, 31), agg_c = shfl64(c, 31);
    unsigned long long ex_r = 0, ex_c = 0;
    if (tile == 0) {
      if (lane == 0) *reinterpret_cast<volatile unsigned long long*>(status) = lb_pack(kLbIncl, agg_r, agg_c);
    } else {
      if (lane == 0) *reinterpret_cast<volatile unsigned long long*>(status + tile) = lb_pack(kLbAgg, agg_r, agg_c);
      // look back over windows of 32 predecessors until one has published its inclusive prefix (tile 0 always does)
      for (int pred = (int)tile - 1;; pred -= 32) {
        const int j = pred - (int)lane;
        unsigned long long v = kLbIncl;   // before tile 0: an empty inclusive prefix (never summed, tile 0 stops the walk)
        do {
          if (j >= 0) v = *reinterpret_cast<volatile unsigned long long*>(status + j);
        } while (__any_sync(0xffffffffu, (v >> 62) == 0));
        const uint32_t incl = __ballot_sync(0xffffffffu, (v >> 62) == 2);
        const uint32_t stop = incl ? (uint32_t)(__ffs(incl) - 1) : 31u;   // the nearest inclusive predecessor ends the walk
        ex_r += warp_sum64(lane <= stop ? (v >> 33) & ((1ull << 29) - 1) : 0ull);
        ex_c += warp_sum64(lane <= stop ? v & kLbRecMax : 0ull);
        ex_c = ex_c < kLbRecMax ? ex_c : kLbRecMax;
        if (incl) break;
      }
      if (lane == 0) *reinterpret_cast<volatile unsigned long long*>(status + tile) = lb_pack(kLbIncl, ex_r + agg_r, ex_c + agg_c);
    }
    if (lane == 0) {
      s_base_r = ex_r; s_base_c = ex_c;
      const unsigned long long all_r = ex_r + agg_r, all_c = ex_c + agg_c;
      if (tile == gridDim.x - 1 && all_r <= ready_cap && all_c <= cap) { hdr[0] = all_r; hdr[1] = all_c; hdr[2] = n; }
    }
  }
  __syncthreads();
#pragma unroll
  for (uint32_t k = 0; k < kReadyItems; k++) {
    const unsigned long long cnt = tl[k] - cur[k];
    if (!cnt) continue;
    const uint32_t chunk = k * kWarpsPerCta + warp;
    const unsigned long long r = s_base_r + s_wr[chunk] + r_in[k] - 1;        // entry index among the ready mailboxes
    const unsigned long long o = s_base_c + s_wc[chunk] + c_in[k] - cnt;      // first record of the run in `out`
    if (r < ready_cap && o + cnt <= cap) {
      ready[r] = cpbus_ready{sub_base + loc[k], (uint32_t)cnt, (uint32_t)o, 0u, cur[k] - hd[k]};
      slot[r] = (uint32_t)(cur[k] & (ring_cap - 1));
      ctl[loc[k]].head = tl[k];
    } else if (r == 0 || (r - 1 < ready_cap && o <= cap)) {   // its predecessor was taken: this one ends the call
      hdr[0] = r; hdr[1] = o; hdr[2] = tile * kReadyTile + k * kThreads + threadIdx.x;
    }
  }
}

// Copies the taken runs: one warp per ready entry, lane pairs per record (each pair writes one whole 32-byte sector), and
// hands the header to the host through mapped pinned memory.
__global__ void __launch_bounds__(kThreads) drain_ready_gather_kernel(const cpbus_event* __restrict__ ring, uint32_t ring_cap,
                                                                      uint32_t sub_base, const cpbus_ready* __restrict__ ready,
                                                                      const uint32_t* __restrict__ slot,
                                                                      const unsigned long long* __restrict__ hdr,
                                                                      cpbus_event* __restrict__ out, unsigned long long* h_hdr) {
  const unsigned long long n_ready = hdr[0];
  if (blockIdx.x == 0 && threadIdx.x < 3) h_hdr[threadIdx.x] = hdr[threadIdx.x];
  const uint32_t lane = threadIdx.x & 31, half = lane & 1;
  const unsigned long long nw = (gridDim.x * blockDim.x) >> 5;
  for (unsigned long long e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < n_ready; e += nw) {
    const cpbus_ready rd = ready[e];
    const uint32_t s0 = slot[e];
    const uint4* src = reinterpret_cast<const uint4*>(ring + (size_t)(rd.sub_id - sub_base) * ring_cap);
    uint4* dst = reinterpret_cast<uint4*>(out + rd.offset);
    uint32_t j = lane >> 1;
    for (; j + 16 < rd.count; j += 32) {   // two records per pair in flight
      const uint4 a = src[2 * ((s0 + j) & (ring_cap - 1)) + half], b = src[2 * ((s0 + j + 16) & (ring_cap - 1)) + half];
      dst[2 * j + half] = a; dst[2 * (j + 16) + half] = b;
    }
    if (j < rd.count) dst[2 * j + half] = src[2 * ((s0 + j) & (ring_cap - 1)) + half];
  }
}

// (count, digest) folds over a range of mailboxes: one 32-byte result instead of 16 B per subscriber
__global__ void digest_fold_kernel(const SubCtl* ctl, uint32_t first, uint32_t n, uint32_t sub_base,
                                   unsigned long long* out4) {
  unsigned long long c = 0, d = 0, x = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const unsigned long long t = ctl[first + i].tail, g = ctl[first + i].digest;
    c += t; d += g;
    x ^= record_hash_words(g, t, sub_base + first + i, 0);
  }
  c = warp_sum64(c); d = warp_sum64(d);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    uint32_t lo = __shfl_xor_sync(0xffffffffu, (uint32_t)x, o), hi = __shfl_xor_sync(0xffffffffu, (uint32_t)(x >> 32), o);
    x ^= ((unsigned long long)hi << 32) | lo;
  }
  if ((threadIdx.x & 31) == 0) { atomicAdd(&out4[0], c); atomicAdd(&out4[1], d); atomicXor(&out4[2], x); }
  if (blockIdx.x == 0 && threadIdx.x == 0) out4[3] = n;
}

// Lossless stream across processes: post this shard's offer word into the publisher's memory (peer mapping elsewhere).
// Stream-ordered behind the admission pass; the release orders nothing else, it makes the word itself visible system-wide.
__global__ void stream_offer_kernel(unsigned long long* word, unsigned long long value) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(word), "l"(value) : "memory");
}

// One CTA of kStreamMaxConsumers threads, lane c = consumer c: acquire every shard's offer of round `round` (bounded by the
// stream timeout), then the minimum prefix and the OR of the stall bits.  A missing offer sets the sticky error word.
// (stream_agree_kernel and stream_round_agree_kernel: every thread of the CTA calls it, thread 0 gets the result; flags:
// bit 0 some shard stalled, bit 1 some offer missing)
__device__ __forceinline__ void agree_offers(const unsigned long long* ack, uint32_t n_consumers, unsigned long long round,
                                             uint32_t spin_us, uint32_t& prefix, uint32_t& flags) {
  __shared__ uint32_t s_min[kStreamMaxConsumers / 32], s_flags[kStreamMaxConsumers / 32];
  const uint32_t c = threadIdx.x, lane = c & 31u, w = c >> 5;
  const unsigned long long tag = round & kOfferRoundMask;
  prefix = 0xFFFFFFFFu; flags = 0;
  if (c < n_consumers) {
    const unsigned long long* word = ack + stream_offer_word_index(c, round);
    const unsigned long long budget = (spin_us ? (unsigned long long)spin_us : 2000000ull) * 1000ull;
    unsigned long long v, t0, t1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    for (;;) {
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(word) : "memory");
      if ((v >> 33) == tag) break;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
      if (t1 - t0 > budget) break;
      __nanosleep(128);
    }
    if ((v >> 33) == tag) { prefix = (uint32_t)v; flags = (uint32_t)(v >> 32) & 1u; }
    else flags = 2u;
  }
  prefix = __reduce_min_sync(0xFFFFFFFFu, prefix);
  flags = __reduce_or_sync(0xFFFFFFFFu, flags);
  if (lane == 0) { s_min[w] = prefix; s_flags[w] = flags; }
  __syncthreads();
  if (c == 0)
    for (uint32_t i = 1; i < blockDim.x / 32; i++) { prefix = min(prefix, s_min[i]); flags |= s_flags[i]; }
}
__global__ void __launch_bounds__(kStreamMaxConsumers) stream_agree_kernel(const unsigned long long* ack, uint32_t n_consumers,
                                                                          unsigned long long round, uint32_t spin_us,
                                                                          StreamAgreeResult* out, unsigned int* err_word) {
  uint32_t prefix, flags;
  agree_offers(ack, n_consumers, round, spin_us, prefix, flags);
  if (threadIdx.x == 0) {
    const uint32_t status = (flags & 2u) ? kErrStreamTimeout : 0u;
    if (status) asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(err_word), "r"(status) : "memory");   // host-mapped, sticky
    out->m = flags ? 0u : prefix;
    out->stalled = flags & 1u;
    out->status = status;
  }
}

// ---- lossless stream rounds on the device (cpbus_stream_round_next) -----------------------------------------------------
// Step 1, one CTA: the cursor's batch header (acquired across the link, bounded by the stream timeout), the clock checks
// cpbus_stream_admit makes on the host, and the fast path against the device room bound.  When the bound cannot prove the
// fit, the CTA copies the remainder of the batch into local memory for the exact pass.  A batch that never arrives, that
// does not match the cursor, or that lies behind the clock or beyond the timer window poisons the bus's rounds and sets the
// sticky error word.
__global__ void __launch_bounds__(kThreads) stream_round_decide_kernel(const RoundParams P) {
  __shared__ uint32_t s_rem, s_src, s_pass;
  RoundDev* d = P.dev;
  if (threadIdx.x == 0) {
    if (P.seed_bus) { d->room = P.seed_room; d->now = P.seed_now; d->last_wm = P.seed_wm; d->poison = 0; }
    if (P.seed_cur) { P.cur->batch = P.seed_batch; P.cur->off = P.seed_off; }
    const unsigned long long q = P.cur->batch;
    const uint32_t off = P.cur->off;
    uint32_t status = kRoundOk, admit = kRoundAdmitNone, rem = 0;
    unsigned long long hw = 0;
    if (d->poison) status = kRoundSkip;
    else {
      const StreamHdr* h = P.hdr + q % P.n_slots;
      const unsigned long long budget = (P.spin_us ? (unsigned long long)P.spin_us : 2000000ull) * 1000ull;
      unsigned long long seen, t0, t1;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
      for (;;) {
        asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(&h->seq) : "memory");
        if (seen >= q) break;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        if (t1 - t0 > budget) break;
        __nanosleep(64);
      }
      unsigned int err = 0;
      if (seen != q) err = kErrStreamTimeout;
      else {
        uint32_t hn;
        asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(hn) : "l"(&h->n) : "memory");
        asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(hw) : "l"(&h->watermark) : "memory");
        if (hn > P.B || hn < off) err = kErrStreamShape;
        else if (hw < d->now || hw - d->last_wm > P.window) err = kErrFollowOrder;
        else rem = hn - off;
      }
      if (err) {
        asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(P.err_word), "r"(err) : "memory");   // host-mapped, sticky
        d->poison = 1;
        status = kRoundAbort;
      } else if (P.n_subs) {
        const uint64_t need = admit_need(rem, hw, d->last_wm, P.min_period, P.K, P.timers_armed != 0);
        if (d->room >= need) { d->room -= need; admit = kRoundAdmitSkipped; }
        else {
          admit = kRoundAdmitPass;
          P.stats->admit_overflow = 0; P.stats->overwritten = 0; P.stats->admit_max_used = 0; P.stats->admit_deficit = 0;
        }
      }
    }
    d->q = q; d->off = off; d->rem = rem; d->hw = hw; d->status = status; d->admit = admit;
    s_rem = rem; s_src = (uint32_t)(q % P.n_slots) * P.B + off; s_pass = admit == kRoundAdmitPass ? 1u : 0u;
  }
  __syncthreads();
  if (!s_pass) return;
  const uint4* src = reinterpret_cast<const uint4*>(P.payload + s_src);
  uint4* dst = reinterpret_cast<uint4*>(P.admit_batch);
  for (uint32_t i = threadIdx.x; i < 2u * s_rem; i += blockDim.x) {
    uint4 v;
    asm volatile("ld.global.relaxed.sys.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(src + i) : "memory");
    dst[i] = v;
  }
}

// Step 2, the grid: the exact admission pass over the local copy, when step 1 could not prove the fit.  On the fast path
// every CTA returns at once.
__global__ void stream_round_admit_kernel(const RoundParams P) {
  if (P.dev->admit != kRoundAdmitPass) return;   // CTA-uniform
  admit_body(P.admit_batch, P.dev->rem, P.dev->hw, P.ctl, P.timers, P.n_subs, P.ring_cap, P.K, P.sub_base, P.timers_armed,
             P.stats, P.pairs);
}

// Step 3, one CTA of kStreamMaxConsumers threads: this shard's admissible prefix (cpbus_stream_admit's rules), its offer
// word, the wait for every shard's offer of the round, and the round's outcome: the fan-out's shape in RoundDev, the
// cursor and the clock moved, the host's record.  A missing offer sets the sticky error word and poisons the bus's rounds.
__global__ void __launch_bounds__(kStreamMaxConsumers) stream_round_agree_kernel(const RoundParams P) {
  __shared__ uint32_t s_go;
  RoundDev* d = P.dev;
  if (threadIdx.x == 0) {
    s_go = d->status == kRoundOk ? 1u : 0u;
    if (s_go) {
      const uint32_t rem = d->rem;
      uint32_t p = rem, stalled = 0;
      if (d->admit == kRoundAdmitPass) {
        const bool ok = P.stats->admit_overflow == 0;
        if (!ok) p = rem - (uint32_t)min((unsigned long long)rem, P.stats->admit_deficit);
        const unsigned long long used = P.stats->admit_max_used;
        d->room = used >= P.ring_cap ? 0ull : P.ring_cap - used;
        // every record fits, but not the ticks due after the last of them: hold the last record back, or stall
        if (!ok && p == rem) { if (rem == 0) stalled = 1; else p = rem - 1; }
      }
      asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(P.ack + stream_offer_word_index(P.consumer, P.round)),
                   "l"(stream_offer_word(P.round, stalled, stalled ? 0u : p)) : "memory");
    }
  }
  __syncthreads();
  uint32_t m = 0, flags = 0;
  if (s_go) agree_offers(P.ack, P.n_consumers, P.round, P.spin_us, m, flags);   // (s_go is CTA-uniform)
  if (threadIdx.x != 0) return;
  uint32_t rs;
  unsigned long long w = 0;
  d->go = 0;
  if (!s_go) rs = d->status == kRoundSkip ? kFollowSkipped : kFollowAborted;
  else if (flags & 2u) {
    asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(P.err_word), "r"(kErrStreamTimeout) : "memory");   // host-mapped, sticky
    d->poison = 1;
    rs = kFollowAborted;
  } else if ((flags & 1u) || (m == 0 && d->rem != 0)) rs = kRoundStalled;
  else {
    const bool final = m == d->rem;
    const uint32_t src = (uint32_t)(d->q % P.n_slots) * P.B + d->off;
    w = d->hw;
    if (final) { P.cur->batch = d->q + 1; P.cur->off = 0; }
    else {
      // like a partial cpbus_stream_fanout_prefix: the watermark is the last delivered record's timestamp
      unsigned long long ts;
      asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(ts) : "l"(&P.payload[src + m - 1].ts_ns) : "memory");
      w = min(d->hw, max(ts, d->last_wm));
      d->room = 0;
      P.cur->off = d->off + m;
    }
    d->now = w; d->last_wm = w;
    d->go = 1; d->m = m; d->src = src; d->final = final ? 1u : 0u; d->w = w;
    rs = final ? kFollowDelivered : kRoundPartial;
  }
  volatile RoundRec* r = P.rec;
  r->m = d->go ? m : 0u; r->watermark = w; r->room = d->room; r->admit = d->admit;
  r->status = rs;
}
#endif  // __CUDACC__

}  // namespace cpbus_dev
