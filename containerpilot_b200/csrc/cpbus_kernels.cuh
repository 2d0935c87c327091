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
// variants.  Occupancy is the biggest single lever (DESIGN.md §4.1); the macro exists for A/B builds.
#ifndef CPBUS_CTAS_PER_SM
#define CPBUS_CTAS_PER_SM 4
#endif
// A/B build switches (build variants with -D...=0/1 and time them on one GPU; the defaults are the chosen variants)
#ifndef CPBUS_SWIZZLE
#define CPBUS_SWIZZLE 2      // shared-memory record reads with lanes 4-7 of each quarter warp fetching their halves in swapped order:
                             // 0 = never, 1 = every path, 2 = only gathered reads.  Only lds_record uses it, i.e. the per-lane
                             // reads of the CPBUS_ORD_RUNS variant; every other path copies records with copy_record_pairs.
                             // The swizzle removes the bank conflicts everywhere, but on the dense paths the two extra live
                             // registers per record cost more than the conflicts do.
#endif
#ifndef CPBUS_TICKS_REG
#define CPBUS_TICKS_REG 1    // dense+ticks copy loop: tick positions in registers (ballots) instead of shared-memory loads
#endif
#ifndef CPBUS_COLD_EARLY
#define CPBUS_COLD_EARLY 1   // PAIRS build: cold half of the timer slot loaded before the copy loop instead of after it (the plain
#endif                       // build reads it from its shared-memory staging)
#ifndef CPBUS_UNROLL2
#define CPBUS_UNROLL2 1      // dense+ticks loop: two 32-event chunks per iteration
#endif
#ifndef CPBUS_ORD_PF
#define CPBUS_ORD_PF 0       // ORDERED build: prefetch.L2 of the whole block's control blocks once the ids are known
#endif
#ifndef CPBUS_PLANAR
#define CPBUS_PLANAR 1       // the staged batch is re-laid in shared memory as two 16-byte planes (lo[i] = bytes 0-15 of record i, hi[i] =
#endif                       // bytes 16-31) before the copy loops: a lane's two LDS.128 are then conflict-free on the dense paths with no
                             // select and no extra register (the lane-swapped reads of CPBUS_SWIZZLE cost registers)
#ifndef CPBUS_ORD_RUNS
#define CPBUS_ORD_RUNS 0     // ORDERED build: process runs of equal masks as a unit (records read once, stored to every ring of the run).
                             // Bit-exact, but off by default: the rings then receive 1-2 KiB per visit instead of one contiguous
                             // multi-KiB append, which can cost more than the saved gathers.
#endif
constexpr uint32_t kActiveBit = 0x80000000u;   // mask word: subscriber is subscribed
constexpr int kTimerHintShift = 24;            // mask word bits 24..27: #timer slots to look at
constexpr uint32_t kPairBit = 0x10000000u;     // mask word bit 28: subscriber has a {code, source} pair table
constexpr uint32_t kPairNone = 0xFFFFFFFFu;    // code of an unused pair slot
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
// One lane reads one staged 32-byte record as two 16-byte shared-memory loads.  At a 32-byte lane stride the eight lanes
// of a quarter warp (one LDS.128 wavefront) touch only four distinct 16-byte bank groups: a 2-way conflict on every read.
// Lanes 4-7 of each quarter therefore fetch their two halves in the opposite order: each wavefront then covers all 32
// banks, and two selects per register put the halves back in place.  No re-layout of the TMA-staged batch is needed.
template <bool GATHER = false, bool PL = false>
__device__ __forceinline__ void lds_record(const uint4* s4, uint32_t i, uint32_t sw, uint4& a, uint4& b, uint32_t hi = 0) {
  if (PL) { a = s4[i]; b = s4[hi + i]; return; }   // planar staging: plane lo at s4, plane hi at s4 + hi
  if (CPBUS_SWIZZLE == 0 || (CPBUS_SWIZZLE == 2 && !GATHER)) {
    a = s4[2 * i]; b = s4[2 * i + 1];
    return;
  }
  const uint4 x = s4[2 * i + sw], y = s4[2 * i + (sw ^ 1u)];
  a.x = sw ? y.x : x.x; a.y = sw ? y.y : x.y; a.z = sw ? y.z : x.z; a.w = sw ? y.w : x.w;
  b.x = sw ? x.x : y.x; b.y = sw ? x.y : y.y; b.z = sw ? x.z : y.z; b.w = sw ? x.w : y.w;
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
template <int STORE, bool TIMERS, bool DIGEST, bool ORDERED, bool PAIRS = false>
__global__ void __launch_bounds__(kThreads, CPBUS_CTAS_PER_SM) fanout_kernel(const FanoutParams p) {
  constexpr bool STAGED = !ORDERED && !PAIRS;
  extern __shared__ __align__(128) unsigned char smem[];
  const uint32_t cap = p.smem_cap;
  cpbus_event* s_batch = reinterpret_cast<cpbus_event*>(smem);
  uint64_t* s_rhash = reinterpret_cast<uint64_t*>(smem + (size_t)cap * 32);
  uint2* s_meta = reinterpret_cast<uint2*>(smem + (size_t)cap * 40);
  uint64_t* s_q = reinterpret_cast<uint64_t*>(smem + (size_t)cap * 48);
  uint32_t* s_dsum = reinterpret_cast<uint32_t*>(s_q + cap + 2);        // descriptor summary: present, has_unicast, hist[32], pad (160 B)
  uint32_t* s_present = s_dsum + 40;                                  // PAIRS build: the batch's {code, source} presence filter (4 KiB), part of the descriptor
  uint64_t* s_pow = s_q + cap + 2 + 20 + (PAIRS ? kPairFilterWords / 2 : 0);   // 16-byte aligned (TMA destination)
  BatchSummary* s_sum = reinterpret_cast<BatchSummary*>(s_pow + cap + 66);
  uint32_t* s_tick = reinterpret_cast<uint32_t*>(s_sum + 1);
  const uint4* s_ctl4 = reinterpret_cast<const uint4*>(smem + fanout_stage_off(cap));   // STAGED: 2 halves per control block
  const uint4* s_tim4 = s_ctl4 + 2u * p.stage_subs;                                      // ... and per timer slot

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t n = p.n_ev;

  // ---- stage the batch: one elected thread drives the TMA engine ----
  // Programmatic dependent launch: this kernel may begin while the previous fan-out is still draining its last wave.
  // Everything up to `griddepcontrol.wait` touches only data that the previous launch never writes (the batch, the
  // power table, this launch's descriptor buffer, the publisher's stream); mailboxes, control blocks and timers come after it.
  if (p.batch_dep) asm volatile("griddepcontrol.wait;" ::: "memory");
  const bool stream = p.staged == 2u;
  const uint32_t pf_slot = stream ? (uint32_t)(p.stream_seq % kStreamPrefetch) : 0u;
  // position space: plain build = subscriber index, set per staging round; PAIRS build = subscriber index, set per triage
  // survivor; ORDERED build = index into p.order, one contiguous block of p.spw positions per warp (lane l keeps the id at
  // block position l: one coalesced load)
  uint32_t pos = ORDERED ? (blockIdx.x * kWarpsPerCta + warp) * p.spw : 0u;
  uint32_t my_ids = 0;
  if (ORDERED && pos + lane < min(pos + p.spw, p.n_order)) my_ids = __ldg(p.order + pos + lane);   // static data: safe before the wait
  if (tid == 0) {
    mbar_init(&s_sum->mbar, 1); mbar_init(&s_sum->mbar_desc, 1); mbar_init(&s_sum->mbar_state, 1);
    s_sum->acc_deliv = 0; s_sum->acc_ticks = 0; s_sum->acc_dig_lo = 0; s_sum->acc_dig_hi = 0;
    // stream mode: an earlier launch (two back, so it is complete and visible) may already hold this batch locally.  Not in
    // lossless mode (no launch prefetches there) and not for a resumed batch (stream_off > 0): those always read the slot
    s_sum->stream_local = (stream && !p.lossless && p.stream_off == 0 && __ldcg(p.pf_state + pf_slot) == p.stream_seq) ? 1u : 0u;
    s_sum->own_desc = blockIdx.x == 0 ? 1u : 0u; s_sum->abort_launch = 0;
  }
  __syncthreads();
  const bool stream_local = stream && s_sum->stream_local;
  // staged: the batch lives in another GPU's memory (or in the stream ring): CTA 0 pulls it once, stages it in local HBM
  // and every other CTA takes CTA 0's local copy after the descriptor flag (second mbarrier phase)
  const bool staged = p.staged && !stream_local;
  const cpbus_event* batch_src = stream_local ? p.pf_buf + (size_t)pf_slot * p.pf_stride : p.batch;
  if (tid == 0) {   // two bulk copies on one mbarrier: the batch and the powers P^0..P^(cap+64)
    const uint32_t pow_bytes = ((cap + 65u) * 8u + 15u) & ~15u;
    const bool direct = n && !staged;
    mbar_expect_tx(&s_sum->mbar, (direct ? n * 32u : 0u) + pow_bytes);
    if (direct) bulk_g2s(s_batch, batch_src, n * 32u, &s_sum->mbar);
    bulk_g2s(s_pow, p.pow_table, pow_bytes, &s_sum->mbar);
  }

  const bool keep = p.hints & 1u;
  // (the evict_last policy is materialised at each use — one instruction — rather than held in two registers)
  if (CPBUS_ORD_PF && ORDERED && pos + lane < min(pos + p.spw, p.n_order))   // mask order scatters the ids: lane l prefetches ITS mailbox's control block
    asm volatile("prefetch.global.L2 [%0];" ::"l"(p.ctl + my_ids));

  // ---- per-batch descriptor: computed ONCE per launch by CTA 0, copied by everyone else ----
  // descriptor = [rhash | meta | Q | summary {present, has_unicast, hist[32]}]: 24*cap + 16 + 160 bytes, the same layout in
  // shared memory and in HBM, so the copy is ONE bulk (TMA) transfer per CTA.  The flag word carries the launch ordinal and,
  // in bit 63, "aborted" (stream batch missing), so a consumer needs no second load to learn it.
  const uint32_t desc_bytes = 24u * cap + 16u + 160u + (PAIRS ? kPairFilterBytes : 0u);
  uint4* s_desc = reinterpret_cast<uint4*>(s_rhash);
  uint4* g_desc = reinterpret_cast<uint4*>(p.desc);
  constexpr unsigned long long kAbortBit = 1ull << 63;
  if (blockIdx.x != 0) {
    // Wait for CTA 0's descriptor — bounded.  CTA 0 is dispatched first and is resident in practice, but nothing
    // guarantees it (MPS time slicing, preemption, a future scheduler): when the wait runs out this CTA builds the
    // descriptor itself from the same batch (bit-identical result, only slower), so no CTA can spin forever.
    if (tid == 0) {
      unsigned long long seen = 0;
      if (!(p.hints & 2u)) {
        unsigned long long t0, t1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
        const unsigned long long budget = stream ? 4000000000ull : 200000ull;   // ns; a stream batch may legitimately be late
        do {
          asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(seen) : "l"(p.desc_ready) : "memory");
          if ((seen & ~kAbortBit) >= p.launch_seq) break;
          asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        } while (t1 - t0 < budget);
      }
      if ((seen & ~kAbortBit) < p.launch_seq) s_sum->own_desc = 1u;
      else {
        const bool ab = (seen & kAbortBit) != 0;
        s_sum->abort_launch = ab ? 1u : 0u;
        asm volatile("fence.proxy.async;" ::: "memory");             // CTA 0's generic-proxy stores -> our async-proxy reads
        mbar_expect_tx(&s_sum->mbar_desc, desc_bytes);
        bulk_g2s(s_desc, g_desc, desc_bytes, &s_sum->mbar_desc);
        if (staged && n && !ab) {
          mbar_wait(&s_sum->mbar, 0);                                // phase 0 (power table) is over
          mbar_expect_tx(&s_sum->mbar, n * 32u);
          bulk_g2s(s_batch, p.batch_local, n * 32u, &s_sum->mbar);
        }
      }
    }
    __syncthreads();
  }
  const bool own_desc = s_sum->own_desc != 0;   // CTA-uniform
  const bool lead = blockIdx.x == 0;            // the one CTA that publishes: descriptor, local batch copy, ack, result slot
  if (own_desc) {
    if (lead && tid < kResultSub * 4) reinterpret_cast<unsigned long long*>(p.result_next)[tid] = 0ull;   // next launch's result slot
    if (tid < 40) s_dsum[tid] = 0;
    if (stream && staged) {
      // the publisher releases a slot by writing its header after the payload; acquire it across the link (bounded)
      if (tid == 0) {
        unsigned long long seen, t0, t1;
        const unsigned long long budget = (p.spin_us ? (unsigned long long)p.spin_us : 2000000ull) * 1000ull;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
        for (;;) {
          asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(&p.stream_hdr->seq) : "memory");
          if (seen >= p.stream_seq) break;
          asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
          if (t1 - t0 > budget) break;
          __nanosleep(64);
        }
        unsigned int err = 0;
        if (seen != p.stream_seq) err = kErrStreamTimeout;   // never arrived (or the slot was already reused: the caller fell > n_slots behind)
        else {
          uint32_t hn;
          asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(hn) : "l"(&p.stream_hdr->n) : "memory");
          // a final launch takes the batch's last records; a partial one (lossless mode) leaves some behind
          if (p.stream_final ? hn != p.stream_off + n : hn <= p.stream_off + n) err = kErrStreamShape;
        }
        if (err) {
          s_sum->abort_launch = 1u;
          if (lead) asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p.err_word), "r"(err) : "memory");   // host-mapped, sticky
        }
      }
    }
    __syncthreads();
    const bool ab = s_sum->abort_launch != 0;
    if (staged && n && !ab) {   // peer pull: plain 16-byte loads on the NVLink-mapped pointer, into shared memory and the local copy
      const uint4* src = reinterpret_cast<const uint4*>(p.batch);
      uint4* loc = reinterpret_cast<uint4*>(p.batch_local);
      uint4* dst = reinterpret_cast<uint4*>(s_batch);
      for (uint32_t i = tid; i < 2 * n; i += kThreads) {
        uint4 v;
        asm volatile("ld.global.relaxed.sys.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(src + i) : "memory");
        dst[i] = v;
        if (lead) loc[i] = v;
      }
    }
    mbar_wait(&s_sum->mbar, 0);
    __syncthreads();
    if (lead && stream && tid == 0 && !ab && p.stream_final)   // the batch is out of the shared ring: the publisher may reuse the slot
      asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p.stream_ack), "l"(p.stream_seq) : "memory");
    const uint32_t nd = ab ? 0u : n;
    {
      uint32_t present = 0, uni = 0;
      for (uint32_t i = tid; i < nd; i += kThreads) {
        const ulonglong4 w = *reinterpret_cast<const ulonglong4*>(&s_batch[i]);
        s_rhash[i] = record_hash_words(w.x, w.y, w.z, w.w);
        const uint32_t code = (uint32_t)w.z, target = (uint32_t)w.w;
        uint32_t codebit = 0;
        if (target == CPBUS_TARGET_ALL) {
          if (code < 32) { codebit = 1u << code; atomicAdd(&s_dsum[2 + code], 1u); }
          present |= codebit;
        } else uni = 1;
        s_meta[i] = make_uint2(codebit, target);
      }
      present = __reduce_or_sync(0xffffffffu, present);
      uni = __reduce_or_sync(0xffffffffu, uni);
      if (lane == 0) { if (present) atomicOr(&s_dsum[0], present); if (uni) atomicOr(&s_dsum[1], 1u); }
    }
    __syncthreads();
    {   // Q: exclusive prefix sums of w_i = H(e_i) P^(n-1-i); Q[n] is the whole batch as one dense run
      const uint32_t E = (nd + kThreads - 1) / kThreads;
      const uint32_t lo = min(nd, (uint32_t)tid * E), hi = min(nd, lo + E);
      uint64_t sum = 0;
      for (uint32_t i = lo; i < hi; i++) sum += s_rhash[i] * s_pow[nd - 1 - i];
      uint64_t incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t l = __shfl_up_sync(0xffffffffu, (uint32_t)incl, o), h = __shfl_up_sync(0xffffffffu, (uint32_t)(incl >> 32), o);
        if (lane >= o) incl += ((uint64_t)h << 32) | l;
      }
      if (lane == 31) s_sum->red[warp] = incl;
      __syncthreads();
      uint64_t run = incl - sum;
      for (int w = 0; w < warp; w++) run += s_sum->red[w];
      for (uint32_t i = lo; i < hi; i++) { s_q[i] = run; run += s_rhash[i] * s_pow[nd - 1 - i]; }
      if (tid == 0) { uint64_t t = 0; for (int w = 0; w < kWarpsPerCta; w++) t += s_sum->red[w]; s_q[nd] = t; }
      __syncthreads();
    }
    if (PAIRS) {   // presence filter over the batch's broadcast {code, source} keys: built ONCE per launch, shipped with the descriptor
      for (uint32_t i = tid; i < kPairFilterWords; i += kThreads) s_present[i] = 0u;
      __syncthreads();
      for (uint32_t i = tid; i < nd; i += kThreads) {
        if (s_meta[i].y != CPBUS_TARGET_ALL) continue;
        const uint32_t h = pair_key_hash(s_batch[i].code, s_batch[i].source_id);
        atomicOr(&s_present[(h & 32767u) >> 5], 1u << (h & 31u));
        atomicOr(&s_present[((h >> 15) & 32767u) >> 5], 1u << ((h >> 15) & 31u));
      }
      __syncthreads();
    }
    if (lead) {
      for (uint32_t i = tid; i < desc_bytes / 16u; i += kThreads) g_desc[i] = s_desc[i];
      __threadfence();
      __syncthreads();
      if (tid == 0) {
        const unsigned long long flag = p.launch_seq | (ab ? kAbortBit : 0ull);
        asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p.desc_ready), "l"(flag) : "memory");
      }
    }
  } else {
    mbar_wait(&s_sum->mbar_desc, 0);
    mbar_wait(&s_sum->mbar, (staged && n && !s_sum->abort_launch) ? 1u : 0u);
  }
  // ---- planar re-layout of the staged batch (in place): record i = {lo[i], hi[i]}, lo at s4[i], hi at s4[cap + i] ----
  // At a 32-byte lane stride the eight lanes of an LDS.128 wavefront touch only four of the eight 16-byte bank groups
  // (2-way conflict on every record read); at a 16-byte stride they touch all
  // eight.  All 2n chunks are read into registers (n <= 1024: at most 8 per thread), barrier, then written to their
  // plane: two barriers and 8 shared-memory instructions per thread per CTA, against ~2000 record reads per thread.
  // Not in the ORDERED build: its gathered reads do no better on planes than with the lane-swapped halves, and not with
  // the bulk store path, which copies whole records out of shared memory.
  constexpr bool PLANAR = CPBUS_PLANAR && STORE != CPBUS_STORE_BULK && !ORDERED;
  const uint32_t hi_off = cap;                                         // in 16-byte units
  if (PLANAR && n) {
    uint4* sq = reinterpret_cast<uint4*>(s_batch);
    uint4 v[8];
    __syncthreads();                       // (own_desc CTAs: every reader of the record-major batch is done)
#pragma unroll
    for (int r = 0; r < 8; r++) { const uint32_t q = tid + r * kThreads; if (q < 2u * n) v[r] = sq[q]; }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 8; r++) { const uint32_t q = tid + r * kThreads; if (q < 2u * n) sq[(q & 1u) * hi_off + (q >> 1)] = v[r]; }
    __syncthreads();
  }
  // field reads from the staged batch, whichever layout it is in
  auto ev_ts = [&](uint32_t i) -> uint64_t {
    return PLANAR ? reinterpret_cast<const uint64_t*>(reinterpret_cast<const uint4*>(s_batch) + i)[1] : s_batch[i].ts_ns;
  };
  auto ev_code_src = [&](uint32_t i) -> uint2 {   // {code, source_id}
    return PLANAR ? reinterpret_cast<const uint2*>(reinterpret_cast<const uint4*>(s_batch) + hi_off + i)[0] : make_uint2(s_batch[i].code, s_batch[i].source_id);
  };
  const bool aborted = s_sum->abort_launch != 0;   // stream batch missing: this launch delivers nothing and fires no timer
  const uint32_t K = p.K, J = K ? 32u / K : 32u;   // candidate firings per timer slot per launch (host bounds the window)
  const uint32_t tk_slot = lane / J, tk_j = lane % J;
  const bool timers_on = TIMERS && p.timers_on && K;
  const uint32_t wstride = gridDim.x * kWarpsPerCta;
  uint32_t pos_end = (aborted || !ORDERED) ? 0u : min(pos + p.spw, p.n_order);
  const uint32_t pos_step = ORDERED ? 1u : kWarpsPerCta;   // (PAIRS: one position per triage turn)
  const uint32_t pos0 = pos;
  uint32_t s = ORDERED ? __shfl_sync(0xffffffffu, my_ids, 0) : pos;
  // ---- from here on the previous launch's results are needed: wait for it, then let the NEXT launch start its prologue
  // (the trigger comes after the wait so that a launch can never overlap its grand-parent: two descriptor buffers suffice)
  if (!p.batch_dep) asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;");
  // STAGED: this CTA's range is [rng_first, rng_end).  Thread 0 stages one round of it at a time (control blocks, then timer
  // slots) on mbar_state.
  const uint32_t rng_first = blockIdx.x * kWarpsPerCta * p.spw, rng_end = min(rng_first + kWarpsPerCta * p.spw, p.n_subs);
  auto stage_round = [&](uint32_t first) {
    if (!STAGED || tid != 0 || aborted || first >= rng_end) return;
    const uint32_t rn = min(p.stage_subs, rng_end - first);
    // the previous round's generic-proxy reads of the staging area are complete (barrier at the end of the turn)
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    const uint32_t tim_bytes = timers_on ? rn * K * (uint32_t)sizeof(DevTimer) : 0u;
    mbar_expect_tx(&s_sum->mbar_state, rn * (uint32_t)sizeof(SubCtl) + tim_bytes);
    bulk_g2s_hint(const_cast<uint4*>(s_ctl4), p.ctl + first, rn * (uint32_t)sizeof(SubCtl), &s_sum->mbar_state, keep);
    if (tim_bytes) bulk_g2s_hint(const_cast<uint4*>(s_tim4), p.timers + (size_t)first * K, tim_bytes, &s_sum->mbar_state, keep);
  };
  // ================= ORDERED build, no unicast in the batch: whole RUNS of equal masks at a time =================
  // The warp's block is <= 32 consecutive positions of the mask order; lane l owns position pos + l for the whole block
  // (its id is in my_ids, its control block in registers: ONE load instruction brings the block's control blocks in).
  // A run of L mailboxes with the same mask word shares the filter pass AND the record reads: each gathered record is
  // stored to all L rings back to back, so the index-list -> gather -> select chain is paid once per run, not per mailbox
  bool runs_done = false;
  if constexpr (ORDERED && !TIMERS && !PAIRS && CPBUS_ORD_RUNS) {
    if (!s_dsum[1]) {   // CTA-uniform: no unicast record in this batch
      runs_done = true;
      const uint32_t present_r = s_dsum[0];
      const uint32_t Rm_r = p.ring_cap - 1;
      const uint4* s4r = reinterpret_cast<const uint4*>(s_batch);
      const uint32_t swr = ((uint32_t)lane >> 2) & 1u;
      uint16_t* my_idx = reinterpret_cast<uint16_t*>(s_tick + warp * max(32u, cap / 2u));
      const uint32_t nb = pos < pos_end ? pos_end - pos : 0u;
      const bool mine = (uint32_t)lane < nb;
      uint4 ma = make_uint4(0, 0, 0, 0), mb = ma;
      if (mine) ld_sector(p.ctl + my_ids, ma, mb, keep);
      const uint32_t my_m = mine ? mb.z : 0u;
      const uint64_t p32 = s_pow[32];
      uint32_t j = 0;
      while (j < nb) {
        const uint32_t m = __shfl_sync(0xffffffffu, my_m, j);
        if (!(m & kActiveBit)) { j++; continue; }
        const uint32_t eq = __ballot_sync(0xffffffffu, mine && my_m == m) >> j;          // bit 0 = lane j itself
        const uint32_t L = (eq == 0xffffffffu) ? 32u : (uint32_t)__ffs(~eq) - 1u;          // consecutive mailboxes with this mask word
        const bool dense = (m & present_r) == present_r;
        uint32_t k = n;
        if (!dense) {   // pass 1: ballot 32 events at a time; matching lanes append their event index to the warp's scratch list
          uint32_t base = 0;
          const uint32_t nchunks = (n + 31) >> 5;
          for (uint32_t c0 = 0; c0 < nchunks; c0 += 4) {
            uint32_t cbit[4];
#pragma unroll
            for (uint32_t u = 0; u < 4; u++) {
              const uint32_t i = (c0 + u) * 32 + lane;
              cbit[u] = i < n ? s_meta[i].x : 0u;
            }
#pragma unroll
            for (uint32_t u = 0; u < 4; u++) {
              const bool match = (m & cbit[u]) != 0;
              const uint32_t w = __ballot_sync(0xffffffffu, match);
              if (match) my_idx[base + __popc(w & ((1u << lane) - 1u))] = (uint16_t)((c0 + u) * 32 + lane);
              base += __popc(w);
            }
          }
          k = base;
          __syncwarp();
        }
        // pass 2: lane -> output slot; every record read once, stored to the L rings of the run
        uint64_t acc = 0;
        for (uint32_t o0 = 0; o0 < k; o0 += 64) {   // warp-uniform trip count (the shuffles below need every lane)
          const uint32_t o = o0 + lane;
          const bool v0 = o < k, v1 = o + 32 < k;
          uint32_t i0 = o, i1 = o + 32;
          if (!dense) { i0 = v0 ? my_idx[o] : 0u; i1 = v1 ? my_idx[o + 32] : 0u; }
          uint4 a0, b0, a1, b1;
          if (v0) lds_record<true, PLANAR>(s4r, i0, swr, a0, b0, hi_off);
          if (v1) lds_record<true, PLANAR>(s4r, i1, swr, a1, b1, hi_off);
          if (DIGEST && !dense) {
            if (v0) acc = acc * p32 + s_rhash[i0];
            if (v1) acc = acc * p32 + s_rhash[i1];
          }
#pragma unroll 2
          for (uint32_t t = j; t < j + L; t++) {
            const uint32_t tl = __shfl_sync(0xffffffffu, ma.x, t);                        // low word of the tail: all the ring index needs
            const uint32_t id = __shfl_sync(0xffffffffu, my_ids, t);
            cpbus_event* ring = p.ring + (size_t)id * p.ring_cap;
            if (v0) st_v8(ring + ((tl + o) & Rm_r), a0, b0);
            if (v1) st_v8(ring + ((tl + o + 32) & Rm_r), a1, b1);
          }
        }
        uint64_t dsum = 0;
        if (DIGEST && k) {
          if (dense) dsum = s_q[n];
          else {   // per-lane Horner in P^32, then one power per lane: lane l wrote outputs l, l+32, ...; its last one is o_last
            const uint32_t cnt = k > (uint32_t)lane ? (k - lane + 31u) / 32u : 0u;
            dsum = cnt ? acc * s_pow[k - 1 - (lane + 32u * (cnt - 1u))] : 0ull;
            dsum = warp_sum64(dsum);
          }
        }
        if (k && (uint32_t)lane >= j && (uint32_t)lane < j + L) {   // each lane of the run writes ITS mailbox's control block back
          const uint64_t tail = ((uint64_t)ma.y << 32) | ma.x, dig = ((uint64_t)mb.y << 32) | mb.x;
          const uint64_t nt = tail + k;
          const uint64_t nd = DIGEST ? dig * s_pow[k] + dsum : dig;
          st_sector(p.ctl + my_ids, make_uint4((uint32_t)nt, (uint32_t)(nt >> 32), ma.z, ma.w),
                    make_uint4((uint32_t)nd, (uint32_t)(nd >> 32), mb.z, 0u), keep);
          atomicAdd(&s_sum->acc_deliv, k);
          if (DIGEST) {
            const uint32_t f = (uint32_t)nd ^ (uint32_t)(nd >> 32);
            atomicAdd(&s_sum->acc_dig_lo, f & 0xFFFFu);
            atomicAdd(&s_sum->acc_dig_hi, f >> 16);
          }
        }
        __syncwarp();   // my_idx is rewritten by the next run's pass 1
        j += L;
      }
    }
  }
  if (runs_done) pos = pos_end;   // nothing left for the per-mailbox loop below
  uint4 ca = make_uint4(0, 0, 0, 0), cb = ca, ta = ca;
  if (ORDERED && pos < pos_end) ld_sector(p.ctl + s, ca, cb, keep);   // software pipeline, stage 0: first control block
  const uint32_t present = s_dsum[0];
  const bool has_unicast = s_dsum[1] != 0;
  // PAIRS build: TRIAGE.  A fleet of pair-filtered subscribers (jobs/jobs.go:188-231: every consumer listens for a dozen exact
  // events) takes almost nothing from a given batch, so walking the mailboxes one per warp-iteration — control block, then
  // pair table, then 16 probes, each a dependent load — is all latency.
  // Instead lane l decides for mailbox 32*blk + l: one control-block load per lane, and only when the
  // code mask misses, its timer slots' due times and its pair row's probes into the presence filter.  The ballot of the
  // survivors drives the ordinary per-mailbox path below (control block handed over by shuffles); exactness is unchanged —
  // a survivor may still turn out to receive nothing.
  bool bulk_pending = false;
  uint32_t tri_blk = blockIdx.x * kWarpsPerCta + warp, tri_base = 0, tri_live = 0;
  uint4 tri_a = make_uint4(0, 0, 0, 0), tri_b = tri_a;
  uint32_t rnd_first = rng_first, rnd_phase = 0;   // STAGED: the current round starts at rnd_first
  for (;;) {   // PAIRS: one surviving mailbox per turn; plain build: one staging round per turn; ORDERED: exactly one turn
  if constexpr (STAGED) {
    if (aborted || rnd_first >= rng_end) break;   // CTA-uniform
    stage_round(rnd_first);
    mbar_wait(&s_sum->mbar_state, rnd_phase);
    rnd_phase ^= 1u;
    pos = rnd_first + warp; pos_end = rnd_first + min(p.stage_subs, rng_end - rnd_first);
  }
  if constexpr (PAIRS) {
    bool exhausted = aborted;
    while (!tri_live && !exhausted) {
      tri_base = tri_blk * 32u;
      if (tri_base >= p.n_subs) { exhausted = true; break; }
      tri_blk += wstride;
      const uint32_t sl = tri_base + lane;
      bool live = false;
      tri_a = make_uint4(0, 0, 0, 0); tri_b = tri_a;
      if (sl < p.n_subs) ld_sector(p.ctl + sl, tri_a, tri_b, keep);
      const uint32_t ml = tri_b.z;
      if (ml & kActiveBit) {
        live = has_unicast || (ml & present) != 0;
        if (!live && timers_on) {
          const uint32_t nsl = min((ml >> kTimerHintShift) & 0xFu, K);
          for (uint32_t t = 0; t < nsl && !live; t++) {
            uint4 h;
            ld_half(p.timers + (size_t)sl * K + t, h, keep);
            const uint64_t due = ((uint64_t)h.y << 32) | h.x;
            live = due != kTimerIdle && due <= p.w_now;
          }
        }
        if (!live && (ml & kPairBit)) {
          const uint4* row = reinterpret_cast<const uint4*>(p.pairs + (size_t)sl * CPBUS_MAX_PAIRS);
          for (uint32_t q = 0; q < CPBUS_MAX_PAIRS / 2 && !live; q++) {
            const uint4 v = __ldg(row + q);                      // two {code, source} cases
            if (v.x >= 32u) break;                               // used slots come first
            uint32_t h = pair_key_hash(v.x, v.y);
            live = ((s_present[(h & 32767u) >> 5] >> (h & 31u)) & (s_present[((h >> 15) & 32767u) >> 5] >> ((h >> 15) & 31u)) & 1u) != 0;
            if (live || v.z >= 32u) { if (!live) break; continue; }
            h = pair_key_hash(v.z, v.w);
            live = ((s_present[(h & 32767u) >> 5] >> (h & 31u)) & (s_present[((h >> 15) & 32767u) >> 5] >> ((h >> 15) & 31u)) & 1u) != 0;
          }
        }
      }
      tri_live = __ballot_sync(0xffffffffu, live);
    }
    if (exhausted) break;
    const uint32_t jl = (uint32_t)__ffs(tri_live) - 1u;
    tri_live &= tri_live - 1u;
    pos = tri_base + jl; pos_end = pos + 1u; s = pos;
    ca = make_uint4(__shfl_sync(0xffffffffu, tri_a.x, jl), __shfl_sync(0xffffffffu, tri_a.y, jl), __shfl_sync(0xffffffffu, tri_a.z, jl), __shfl_sync(0xffffffffu, tri_a.w, jl));
    cb = make_uint4(__shfl_sync(0xffffffffu, tri_b.x, jl), __shfl_sync(0xffffffffu, tri_b.y, jl), __shfl_sync(0xffffffffu, tri_b.z, jl), __shfl_sync(0xffffffffu, tri_b.w, jl));
    if (timers_on && tk_slot < K) ld_half(p.timers + (size_t)s * K + tk_slot, ta, keep);
  }
  const uint32_t Rm = p.ring_cap - 1;
  const uint4* s4 = reinterpret_cast<const uint4*>(s_batch);
  const uint32_t scratch_words = max(32u, cap / 2u);                   // per warp: 32 tick positions or cap u16 event indices
  uint32_t* my_tick = s_tick + warp * scratch_words;

  // ORDERED: software pipeline, the control block of the NEXT subscriber is in flight while the current one is being
  // written, so no DRAM round trip is exposed per subscriber.  STAGED: the round's state is in shared memory; halves are
  // re-read where they are needed rather than kept in registers across the copy loops.
  uint32_t run_mask = 0xffffffffu, run_k = 0;   // ORDERED: the filter pass of the previous mailbox, reusable while the mask repeats
  uint64_t run_sum = 0;
  for (; pos < pos_end; pos += pos_step) {
    const uint32_t si = pos - rnd_first;   // STAGED: staging index
    uint4 cur_a = ca, cur_b = cb;
    // half h of this subscriber's control block / of its timer slot tk_slot
    auto ctl_half = [&](uint32_t h) -> uint4 { return STAGED ? s_ctl4[2u * si + h] : (h ? cur_b : cur_a); };
    auto tim_half = [&](uint32_t h) -> uint4 {
      if (STAGED) return s_tim4[2u * (si * K + tk_slot) + h];
      if (!h) return ta;
      uint4 cold;
      ld_half(reinterpret_cast<const unsigned char*>(p.timers + (size_t)s * K + tk_slot) + 16, cold, keep);
      return cold;
    };
    if (STAGED) { cur_a = ctl_half(0); cur_b = ctl_half(1); }
    if (ORDERED) s = __shfl_sync(0xffffffffu, my_ids, (pos - pos0) & 31); else s = pos;
    if (ORDERED) {
      const uint32_t pn = pos + pos_step;
      if (pn < pos_end) ld_sector(p.ctl + __shfl_sync(0xffffffffu, my_ids, (pn - pos0) & 31), ca, cb, keep);
    }
    const uint32_t m = cur_b.z;
    if (!(m & kActiveBit)) continue;
    const uint64_t tail = ((uint64_t)cur_a.y << 32) | cur_a.x;
    cpbus_event* ring = p.ring + (size_t)s * p.ring_cap;
    const uint32_t gid = p.sub_base + s;
    const uint32_t nslots = timers_on ? min((m >> kTimerHintShift) & 0xFu, K) : 0u;
    // dense <=> this mailbox takes every record of the batch (the reference's only mode)
    const bool dense = !has_unicast && ((m & present) == present);

    // ---- timers: which ticks fire in (previous watermark, w_now] ----
    uint32_t n_ticks = 0, tk_mask = 0, tk_rank = 0, tk_src = 0, tk_fired = 0;
    bool tk_valid = false; uint64_t tk_due = 0, tk_period = 0;
    if (nslots) {
      uint64_t tk_due0 = kTimerIdle;
      if (TIMERS && tk_slot < nslots) {
        const uint4 hot = tim_half(0);
        tk_due0 = ((uint64_t)hot.y << 32) | hot.x; tk_period = ((uint64_t)hot.w << 32) | hot.z;
      }
      tk_due = tk_due0 + (uint64_t)tk_j * tk_period;
      tk_valid = tk_due0 != kTimerIdle && tk_due <= p.w_now && (tk_j == 0 || tk_period != 0);
      tk_mask = __ballot_sync(0xffffffffu, tk_valid);
      n_ticks = __popc(tk_mask);
      if (n_ticks) {

        // order simultaneous firings by (due, slot): rank = #valid ticks with a smaller key
        if (J == 32 || (tk_mask >> J) == 0) tk_rank = tk_j;       // only slot 0 fired
        else {
#pragma unroll 1
          for (int t = 0; t < 32; t++) {
            if (!((tk_mask >> t) & 1u)) continue;      // warp-uniform
            const uint64_t od = shfl64(tk_due, t);
            const uint32_t os = __shfl_sync(0xffffffffu, tk_slot, t);
            tk_rank += (od < tk_due || (od == tk_due && os < tk_slot)) ? 1u : 0u;
          }
        }
      }
    }
    uint32_t tk_pos = 0;   // events with ts < due stay in front of the tick (lower_bound over the sorted batch)
    if (tk_valid) {
      uint32_t lo = 0, hi = n;
      while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (ev_ts(mid) < tk_due) lo = mid + 1; else hi = mid;
      }
      tk_pos = lo;
    }

    // second-level filter: lane j < CPBUS_MAX_PAIRS holds this subscriber's j-th exact {code, source} case; the table
    // matters only if one of the cases is (probably) in this batch
    bool pair_live = false;
    if (PAIRS && (m & kPairBit) && !dense) {
      uint2 pr = make_uint2(kPairNone, 0u);
      if (lane < CPBUS_MAX_PAIRS) pr = __ldg(p.pairs + (size_t)s * CPBUS_MAX_PAIRS + lane);
      bool hit = false;
      if (pr.x < 32u) {
        const uint32_t h = pair_key_hash(pr.x, pr.y);
        hit = ((s_present[(h & 32767u) >> 5] >> (h & 31u)) & (s_present[((h >> 15) & 32767u) >> 5] >> ((h >> 15) & 31u)) & 1u) != 0;
      }
      pair_live = __any_sync(0xffffffffu, hit);
    }
    if (PAIRS && !pair_live && !has_unicast && n_ticks == 0 && (m & present) == 0) continue;   // nothing to append

    uint32_t k = 0;           // records appended to this mailbox by this launch
    uint64_t dsum = 0;        // sum of H(record) * P^(k-1-out) over them

    if (dense && n_ticks == 0) {
      // ================= dense run: copy the staged batch into the ring =================
      if (STORE == CPBUS_STORE_BULK) {
        if (lane == 0 && n) {
          const uint32_t slot0 = (uint32_t)tail & Rm;
          const uint32_t first = min(n, p.ring_cap - slot0);
          bulk_s2g(ring + slot0, s_batch, first * 32u);
          if (n > first) bulk_s2g(ring, s_batch + first, (n - first) * 32u);
          asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
        bulk_pending = true;
      } else if (STORE == CPBUS_STORE_V8) {
        for (uint32_t c0 = 0; c0 < n; c0 += 32)   // warp-uniform trip count (copy_record_pairs needs every lane)
          copy_record_pairs<PLANAR>(s4, hi_off, ring, (uint32_t)tail, Rm, c0 + lane, c0 + lane, c0 + lane < n);
      } else {
        for (uint32_t q = lane; q < 2 * n; q += 32) {   // lane pair per record: 512 contiguous bytes per instruction
          const uint4 v = PLANAR ? s4[(q & 1u) * hi_off + (q >> 1)] : s4[q];
          st_v4(reinterpret_cast<unsigned char*>(ring + (((uint32_t)tail + (q >> 1)) & Rm)) + (q & 1u) * 16u, v);
        }
      }
      k = n;
      if (DIGEST) dsum = s_q[n];
    } else if (dense) {
      // ================= dense run with interleaved ticks: O(#ticks) bookkeeping =================
      constexpr bool cold_early = CPBUS_COLD_EARLY && !STAGED;
      if (cold_early && TIMERS && tk_slot < nslots) {   // cold half of the timer slot {source_id, fired}: needed only for the tick records
        const uint4 cold = tim_half(1);                 // after the copy loop, but loaded HERE so that its DRAM round trip hides under the copy
        tk_src = cold.x; tk_fired = cold.y;
      }
      if (tk_valid) my_tick[tk_rank] = tk_pos;
      __syncwarp();
      k = n + n_ticks;
      // event i lands at i + #{ticks with pos <= i}.  Lane r keeps the r-th smallest tick position in a register, so per
      // 32-event chunk the count is two ballots and a bit mask — no shared-memory round trip in the copy loop (the my_tick[]
      // loads feeding these compares would otherwise stall it).
#if CPBUS_TICKS_REG
      const uint32_t T = (uint32_t)lane < n_ticks ? my_tick[lane] : 0xFFFFFFFFu;
      // destination of event i = c0 + lane of the chunk starting at c0
      auto slot_of = [&](uint32_t c0) -> uint32_t {
        const uint32_t before = __popc(__ballot_sync(0xffffffffu, T <= c0));          // ticks at or in front of the chunk's first event
        const bool in = T > c0 && T < c0 + 32u;                                        // ... strictly inside the chunk
        const uint32_t n_in = __popc(__ballot_sync(0xffffffffu, in));
        const uint32_t i = c0 + lane;
        uint32_t out = i + before;
        if (n_in) {
          const uint32_t bits = __reduce_or_sync(0xffffffffu, in ? 1u << (T - c0) : 0u);
          if (__popc(bits) == n_in) out += __popc(bits & ((2u << lane) - 1u));       // bit d <=> a tick at c0 + d <= i  <=>  d <= lane
          else                                                                         // several ticks share a position: count them one by one
            for (uint32_t t = before; t < n_ticks && my_tick[t] < c0 + 32u; t++) out += (my_tick[t] <= i) ? 1u : 0u;
        }
        return out;
      };
      uint32_t c0 = 0;
#if CPBUS_UNROLL2
#pragma unroll 1
      for (; c0 + 64 <= n; c0 += 64) {   // two chunks per iteration: both records' shared-memory loads are in flight before the selects
        const uint32_t o0 = slot_of(c0), o1 = slot_of(c0 + 32);
        copy_record_pairs<PLANAR>(s4, hi_off, ring, (uint32_t)tail, Rm, c0 + lane, o0, true);
        copy_record_pairs<PLANAR>(s4, hi_off, ring, (uint32_t)tail, Rm, c0 + 32 + lane, o1, true);
      }
#endif
#pragma unroll 1
      for (; c0 < n; c0 += 32) {
        const uint32_t out = slot_of(c0);
        copy_record_pairs<PLANAR>(s4, hi_off, ring, (uint32_t)tail, Rm, c0 + lane, out, c0 + lane < n);
      }
#else
      // Tick positions are sorted, so the count is warp-uniform for a whole 32-event chunk unless a tick falls strictly inside it
      uint32_t t_idx = 0;
#pragma unroll 1
      for (uint32_t c0 = 0; c0 < n; c0 += 32) {
        while (t_idx < n_ticks && my_tick[t_idx] <= c0) t_idx++;
        const uint32_t i = c0 + lane;
        uint32_t out = i + t_idx;
        for (uint32_t t = t_idx; t < n_ticks && my_tick[t] < c0 + 32; t++) out += (my_tick[t] <= i) ? 1u : 0u;
        copy_record_pairs<PLANAR>(s4, hi_off, ring, (uint32_t)tail, Rm, i, out, i < n);
      }
#endif
      if (!cold_early && TIMERS && tk_slot < nslots) {
        const uint4 cold = tim_half(1);
        tk_src = cold.x; tk_fired = cold.y;
      }
      if (tk_valid) {
        const uint32_t out = tk_pos + tk_rank;
        const uint64_t w0 = (uint64_t)tk_fired + tk_j, w1 = tk_due;
        const uint64_t w2 = (uint64_t)CPBUS_TIMER_EXPIRED | ((uint64_t)tk_src << 32);
        const uint64_t w3 = (uint64_t)gid | ((uint64_t)CPBUS_F_TICK << 32);
        const uint4 a = make_uint4((uint32_t)w0, (uint32_t)(w0 >> 32), (uint32_t)w1, (uint32_t)(w1 >> 32));
        const uint4 b = make_uint4((uint32_t)w2, (uint32_t)(w2 >> 32), (uint32_t)w3, (uint32_t)(w3 >> 32));
        st_v8(ring + (((uint32_t)tail + out) & Rm), a, b);
        if (DIGEST) {
          // the run of events in front of this tick keeps its internal weights and is shifted by the
          // ticks still to come: (Q[pos_r] - Q[pos_{r-1}]) * P^(n_ticks - r)
          const uint32_t prev = tk_rank ? my_tick[tk_rank - 1] : 0u;
          dsum = (s_q[tk_pos] - s_q[prev]) * s_pow[n_ticks - tk_rank] + record_hash_words(w0, w1, w2, w3) * s_pow[k - 1 - out];
          if (tk_rank == n_ticks - 1) dsum += s_q[n] - s_q[tk_pos];
        }
      }
      if (DIGEST) dsum = warp_sum64(dsum);
      __syncwarp();
    } else if (!(PAIRS && pair_live) && !has_unicast && n_ticks == 0) {
      if constexpr (!TIMERS) {
        // ================= filtered run: compact the matching event indices, then an output-centric copy =================
        // pass 1: ballot 32 events at a time; matching lanes append their event index to the warp's scratch list
        uint16_t* my_idx = reinterpret_cast<uint16_t*>(my_tick);
        const bool reuse = ORDERED && (m & CPBUS_MASK_ALL) == run_mask;   // same mask as the previous mailbox of this warp
        if (!reuse) {
          uint32_t base = 0;
          const uint32_t nchunks = (n + 31) >> 5;
          // code bits of 4 chunks are fetched up front: 4 independent shared-memory loads in flight instead of a
          // load -> test -> ballot chain per chunk
          for (uint32_t c0 = 0; c0 < nchunks; c0 += 4) {
            uint32_t cbit[4];
#pragma unroll
            for (uint32_t u = 0; u < 4; u++) {
              const uint32_t i = (c0 + u) * 32 + lane;
              cbit[u] = i < n ? s_meta[i].x : 0u;
            }
#pragma unroll
            for (uint32_t u = 0; u < 4; u++) {
              const bool match = (m & cbit[u]) != 0;
              const uint32_t w = __ballot_sync(0xffffffffu, match);
              if (match) my_idx[base + __popc(w & ((1u << lane) - 1u))] = (uint16_t)((c0 + u) * 32 + lane);
              base += __popc(w);
            }
          }
          run_k = base;
          __syncwarp();
        }
        k = run_k;
        // pass 2: lane -> output slot, so stores are fully coalesced and only ceil(k/32) iterations run.
        // Digest by per-lane Horner in P^32: acc_l = sum_it H(e) (P^32)^(nit_l-1-it); one power lookup per lane at the end.
        uint64_t acc = 0;
        const uint64_t p32 = s_pow[32];
        const bool hashing = DIGEST && !reuse;
        // warp-uniform trip count (copy_record_pairs needs every lane); the index list is read one iteration ahead, so the
        // records' shared-memory addresses are ready when the loop turns
        uint32_t i0 = (uint32_t)lane < k ? my_idx[lane] : 0u, i1 = lane + 32u < k ? my_idx[lane + 32] : 0u;
        for (uint32_t o0 = 0; o0 < k; o0 += 64) {
          const uint32_t o = o0 + lane;
          const bool v0 = o < k, v1 = o + 32 < k;
          const uint32_t n0 = o + 64 < k ? my_idx[o + 64] : 0u, n1 = o + 96 < k ? my_idx[o + 96] : 0u;
          copy_record_pairs<PLANAR>(s4, hi_off, ring, (uint32_t)tail, Rm, i0, o, v0);
          copy_record_pairs<PLANAR>(s4, hi_off, ring, (uint32_t)tail, Rm, i1, o + 32, v1);
          if (hashing) {
            if (v0) acc = acc * p32 + s_rhash[i0];
            if (v1) acc = acc * p32 + s_rhash[i1];
          }
          i0 = n0; i1 = n1;
        }
        if (DIGEST) {
          if (reuse) dsum = run_sum;
          else {
            // lane l wrote outputs l, l+32, ...: cnt of them, the last one at l + 32 (cnt - 1)
            const uint32_t cnt = k > (uint32_t)lane ? (k - lane + 31u) / 32u : 0u;
            dsum = cnt ? acc * s_pow[k - 1 - (lane + 32u * (cnt - 1u))] : 0ull;
            dsum = warp_sum64(dsum);
            if (ORDERED) run_sum = dsum;
          }
        }
        if (ORDERED) run_mask = m & CPBUS_MASK_ALL;
        __syncwarp();
      } else {
        // timers build: register budget is tighter (80, no spills) — single pass, ballot + running rank
        uint32_t kk = ((m >> lane) & 1u) ? s_dsum[2 + lane] : 0u;
        kk = __reduce_add_sync(0xffffffffu, kk);
        k = kk;
        uint32_t base = 0;
        const uint32_t nchunks = (n + 31) >> 5;
        for (uint32_t c = 0; c < nchunks; c++) {
          const uint32_t i = c * 32 + lane;
          const bool match = i < n && (m & s_meta[i].x) != 0;
          const uint32_t w = __ballot_sync(0xffffffffu, match);
          const uint32_t out = base + __popc(w & ((1u << lane) - 1u));
          if (DIGEST && match) dsum += s_rhash[i] * s_pow[k - 1 - out];
          copy_record_pairs<PLANAR>(s4, hi_off, ring, (uint32_t)tail, Rm, i, out, match);
          base += __popc(w);
        }
        if (DIGEST) dsum = warp_sum64(dsum);
      }
    } else {
      // ================= general run: filter + unicast + interleaved ticks, two passes =================
      const uint32_t nchunks = (n + 31) >> 5;
      uint2 my_pair = make_uint2(kPairNone, 0u);
      uint32_t n_pairs = 0, pair_codes = 0;
      if (PAIRS && pair_live) {   // rare: re-read the (cached) table rather than keep it live across the path selection
        if (lane < CPBUS_MAX_PAIRS) my_pair = __ldg(p.pairs + (size_t)s * CPBUS_MAX_PAIRS + lane);
        const bool used = my_pair.x < 32u;                       // the host packs used slots first
        n_pairs = __popc(__ballot_sync(0xffffffffu, used));
        pair_codes = __reduce_or_sync(0xffffffffu, used ? (1u << my_pair.x) : 0u);
      }
      uint32_t myword = 0;   // pass A: match bitmap, lane c keeps the ballot of chunk c
      for (uint32_t c = 0; c < nchunks; c++) {
        const uint32_t i = c * 32 + lane;
        bool match = false, cand = false;
        if (i < n) {
          const uint2 mt = s_meta[i];
          match = (mt.y == CPBUS_TARGET_ALL) ? ((m & mt.x) != 0) : (mt.y == gid);
          if (PAIRS) cand = !match && mt.y == CPBUS_TARGET_ALL && (mt.x & pair_codes) != 0;
        }
        if (PAIRS && n_pairs && __any_sync(0xffffffffu, cand)) {
          uint32_t ev_code = kPairNone - 1u, ev_src = 0;          // never equals a pair
          if (cand) { const uint2 cs = ev_code_src(i); ev_code = cs.x; ev_src = cs.y; }
          for (uint32_t j = 0; j < n_pairs; j++) {
            const uint32_t pc = __shfl_sync(0xffffffffu, my_pair.x, j), ps = __shfl_sync(0xffffffffu, my_pair.y, j);
            match = match || (ev_code == pc && ev_src == ps);
          }
        }
        const uint32_t w = __ballot_sync(0xffffffffu, match);
        if ((uint32_t)lane == c) myword = w;
      }
      uint32_t wcount = __popc(myword), wprefix = wcount;   // exclusive prefix of popcounts over chunks
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, wprefix, o);
        if (lane >= o) wprefix += t;
      }
      const uint32_t k_ev = __shfl_sync(0xffffffffu, wprefix, 31);
      wprefix -= wcount;
      uint32_t tk_mp = 0;    // matched events in front of each tick
      if (n_ticks) {
        const uint32_t pc = tk_pos >> 5;
        const uint32_t wsel = __shfl_sync(0xffffffffu, myword, pc & 31);
        const uint32_t psel = __shfl_sync(0xffffffffu, wprefix, pc & 31);
        tk_mp = (tk_pos >= n) ? k_ev : psel + __popc(wsel & ((1u << (tk_pos & 31u)) - 1u));
        if (tk_valid) my_tick[tk_rank] = tk_mp;
        __syncwarp();
      }
      k = k_ev + n_ticks;
      for (uint32_t c = 0; c < nchunks; c++) {   // pass B
        const uint32_t w = __shfl_sync(0xffffffffu, myword, c);
        const uint32_t wp = __shfl_sync(0xffffffffu, wprefix, c);
        if (!w) continue;                          // warp-uniform
        const bool mine = (w >> lane) & 1u;
        const uint32_t i = c * 32 + lane;
        uint32_t out = 0;
        if (mine) {
          const uint32_t mrank = wp + __popc(w & ((1u << lane) - 1u));
          out = mrank;
          for (uint32_t t = 0; t < n_ticks; t++) out += (my_tick[t] <= mrank) ? 1u : 0u;
          if (DIGEST) dsum += s_rhash[i] * s_pow[k - 1 - out];
        }
        copy_record_pairs<PLANAR>(s4, hi_off, ring, (uint32_t)tail, Rm, i, out, mine);
      }
      if (n_ticks) {
        if (TIMERS && tk_slot < nslots) {   // cold half of the timer slot {source_id, fired}: read late, only when something fires
          const uint4 cold = tim_half(1);
          tk_src = cold.x; tk_fired = cold.y;
        }
      }
      if (tk_valid) {   // the tick records themselves: {TimerExpired, name} (events/timer.go:31,60)
        const uint32_t out = tk_mp + tk_rank;
        const uint64_t w0 = (uint64_t)tk_fired + tk_j, w1 = tk_due;
        const uint64_t w2 = (uint64_t)CPBUS_TIMER_EXPIRED | ((uint64_t)tk_src << 32);
        const uint64_t w3 = (uint64_t)gid | ((uint64_t)CPBUS_F_TICK << 32);
        const uint4 a = make_uint4((uint32_t)w0, (uint32_t)(w0 >> 32), (uint32_t)w1, (uint32_t)(w1 >> 32));
        const uint4 b = make_uint4((uint32_t)w2, (uint32_t)(w2 >> 32), (uint32_t)w3, (uint32_t)(w3 >> 32));
        st_v8(ring + (((uint32_t)tail + out) & Rm), a, b);
        if (DIGEST) dsum += record_hash_words(w0, w1, w2, w3) * s_pow[k - 1 - out];
      }
      if (DIGEST) dsum = warp_sum64(dsum);
      __syncwarp();
    }

    if (n_ticks) {   // re-arm: one lane per slot writes its timer back (events/timer.go: ticker keeps running)
      const uint32_t slotmask = (J == 32 ? 0xffffffffu : ((1u << J) - 1u)) << (tk_slot * J);
      const uint32_t fired_here = __popc(tk_mask & slotmask);
      if (TIMERS && tk_j == 0 && tk_slot < nslots && fired_here) {
        unsigned char* t = reinterpret_cast<unsigned char*>(&p.timers[(size_t)s * K + tk_slot]);
        // this lane has tk_j == 0, so tk_due is the slot's next_due as loaded
        const uint64_t nd = tk_period ? tk_due + (uint64_t)fired_here * tk_period : kTimerIdle;   // one-shot disarms itself
        st_half(t, make_uint4((uint32_t)nd, (uint32_t)(nd >> 32), (uint32_t)tk_period, (uint32_t)(tk_period >> 32)), keep);
        st_half(t + 16, make_uint4(tk_src, tk_fired + fired_here, 0u, 0u), keep);
      }
    }
    if (lane == 0 && k) {   // one full-sector write of the control block
      const uint4 c0 = ctl_half(0), c1 = ctl_half(1);
      const uint64_t dig = ((uint64_t)c1.y << 32) | c1.x;
      const uint64_t nt = tail + k;
      const uint64_t nd = DIGEST ? dig * s_pow[k] + dsum : dig;
      st_sector(p.ctl + s, make_uint4((uint32_t)nt, (uint32_t)(nt >> 32), c0.z, c0.w),   // head: consumer-owned, passed through
                make_uint4((uint32_t)nd, (uint32_t)(nd >> 32), m, 0u), keep);
      atomicAdd(&s_sum->acc_deliv, k);
      if (DIGEST) {
        const uint32_t f = (uint32_t)nd ^ (uint32_t)(nd >> 32);
        atomicAdd(&s_sum->acc_dig_lo, f & 0xFFFFu);
        atomicAdd(&s_sum->acc_dig_hi, f >> 16);
      }
      if (TIMERS && n_ticks) atomicAdd(&s_sum->acc_ticks, n_ticks);
    }
  }

  if constexpr (ORDERED) break;
  if constexpr (STAGED) {
    __syncthreads();   // every warp is done with this round's staging before the next round overwrites it
    rnd_first += p.stage_subs;
  }
  }   // triage turns / staging rounds
  if (STORE == CPBUS_STORE_BULK && bulk_pending && lane == 0)
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // the staged batch must outlive the TMA reads
  __syncthreads();
  if (tid == 0) {   // one RED per counter per CTA, spread over kStatSlots sectors
    DevStatSlot* st = &p.stats->slot[blockIdx.x % kStatSlots];
    if (s_sum->acc_deliv) atomicAdd(&st->deliveries, (unsigned long long)s_sum->acc_deliv);
    if (s_sum->acc_ticks) atomicAdd(&st->ticks, (unsigned long long)s_sum->acc_ticks);
    DevResultSlot* rs = &p.result[blockIdx.x % kResultSub];
    if (s_sum->acc_deliv) atomicAdd(&rs->deliveries, (unsigned long long)s_sum->acc_deliv);
    if (s_sum->acc_ticks) atomicAdd(&rs->ticks, (unsigned long long)s_sum->acc_ticks);
    if (s_sum->acc_dig_lo | s_sum->acc_dig_hi) atomicAdd(&rs->digest_sum, (unsigned long long)s_sum->acc_dig_lo + ((unsigned long long)s_sum->acc_dig_hi << 16));
    if (blockIdx.x == 0) atomicAdd(&rs->launch_seq, p.launch_seq);
  }
  if (blockIdx.x == 0 && p.acct && !aborted) {
    // device-published batch: publish accounting (events/bus.go:128-139), done here — after the lead CTA's own mailboxes —
    // so that it never delays the fan-out (the staged batch and its descriptor are still intact in shared memory)
    if (tid < 32 && tid != CPBUS_METRIC && s_dsum[2 + tid]) atomicAdd(&p.acct->by_code[tid], (unsigned long long)s_dsum[2 + tid]);
    for (uint32_t i = tid; i < n; i += kThreads) {
      if (s_meta[i].y != CPBUS_TARGET_ALL) continue;
      const uint2 cs = ev_code_src(i);
      const uint32_t code = cs.x;
      if (code == CPBUS_METRIC || code >= 32u) continue;
      const unsigned long long key = (((unsigned long long)code << 32) | cs.y) + 1ull;
      uint32_t slot = pair_key_hash(code, cs.y) & (kAcctPairSlots - 1u);
      bool placed = false;
      for (int probe = 0; probe < 32 && !placed; probe++, slot = (slot + 1u) & (kAcctPairSlots - 1u)) {
        const unsigned long long old = atomicCAS(&p.acct->pair_key[slot], 0ull, key);
        if (old == 0ull || old == key) { atomicAdd(&p.acct->pair_cnt[slot], 1ull); placed = true; }
      }
      if (!placed) atomicAdd(&p.acct->pair_overflow, 1ull);   // table crowded (> ~10^5 distinct {code, source}): counted, not placed
    }
    if (tid == 0) {
      DevDbgTail* t = &p.acct->tail[p.launch_seq % kAcctDbgRing];
      uint32_t* idx = s_tick;                                      // every warp of this CTA is past its main loop (barrier above)
      uint32_t kept = 0, nb = 0;
      for (uint32_t c = 0; c < 32; c++) nb += s_dsum[2 + c];
      for (uint32_t i = n; i > 0 && kept < (uint32_t)kAcctDbgKeep; i--)
        if (s_meta[i - 1].y == CPBUS_TARGET_ALL) idx[kept++] = i - 1;
      for (uint32_t j = 0; j < kept; j++) {
        const uint32_t i = idx[kept - 1 - j];
        if (PLANAR) {
          uint4* o = reinterpret_cast<uint4*>(&t->ev[j]);
          o[0] = reinterpret_cast<const uint4*>(s_batch)[i]; o[1] = reinterpret_cast<const uint4*>(s_batch)[hi_off + i];
        } else t->ev[j] = s_batch[i];
      }
      t->n_broadcast = nb; t->n_kept = kept;
      __threadfence();
      t->launch_seq = p.launch_seq;
    }
  }
  if (blockIdx.x == 0 && p.prefetch_src) {
    // fused ingest: CTA 0 is done with its own mailboxes; pull a LATER batch across NVLink now.  The link round trip
    // hides under the stores of the CTAs still running, and that batch's launch starts from local memory.
    uint32_t pn = p.prefetch_n;
    bool go = true;
    if (stream) {   // stream mode: only if the publisher has already released batch seq+2 (never wait for it here)
      if (tid == 0) {
        unsigned long long seen; uint32_t hn = 0;
        asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(&p.stream_next_hdr->seq) : "memory");
        bool ok = !aborted && seen == p.stream_seq + 2;
        if (ok) {
          asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(hn) : "l"(&p.stream_next_hdr->n) : "memory");
          ok = hn <= p.pf_stride;
        }
        s_sum->pf_ok = ok ? hn + 1u : 0u;
      }
      __syncthreads();
      go = s_sum->pf_ok != 0; pn = go ? s_sum->pf_ok - 1u : 0u;
    }
    if (go) {
      const uint4* src = reinterpret_cast<const uint4*>(p.prefetch_src);
      uint4* dst = reinterpret_cast<uint4*>(p.prefetch_dst);
      for (uint32_t i = tid; i < 2 * pn; i += kThreads) {
        uint4 v;
        asm volatile("ld.global.relaxed.sys.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(src + i) : "memory");
        dst[i] = v;
      }
      if (stream) {   // publish "batch seq+2 is local" to the launch after next (complete and visible before its prologue runs)
        __threadfence();
        __syncthreads();
        if (tid == 0)
          asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p.pf_state + (p.stream_seq + 2) % kStreamPrefetch), "l"(p.stream_seq + 2) : "memory");
      }
    }
  }
}

// Lossless mode (reference semantics, events/subscriber.go:30-32: a full channel
// blocks the sender): before a batch is fanned out, count for every mailbox what
// the batch would append and flag any that lacks the room.  Thread per subscriber.
__global__ void admit_kernel(const cpbus_event* batch, uint32_t n_ev, uint64_t w_now, const SubCtl* ctl,
                             const DevTimer* timers, uint32_t n_subs, uint32_t ring_cap, uint32_t K, uint32_t sub_base,
                             uint32_t timers_on, DevStats* stats, const uint2* pairs) {
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
    for (uint32_t t = 0; t < nslots; t++) {
      const DevTimer tm = timers[(size_t)s * K + t];
      if (tm.next_due != kTimerIdle && tm.next_due <= w_now)
        k += tm.period ? (w_now - tm.next_due) / tm.period + 1u : 1u;
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
          if (tm.next_due != kTimerIdle && tm.next_due <= e.ts_ns) tks += tm.period ? (e.ts_ns - tm.next_due) / tm.period + 1u : 1u;
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
__global__ void __launch_bounds__(kStreamMaxConsumers) stream_agree_kernel(const unsigned long long* ack, uint32_t n_consumers,
                                                                          unsigned long long round, uint32_t spin_us,
                                                                          StreamAgreeResult* out, unsigned int* err_word) {
  __shared__ uint32_t s_min[kStreamMaxConsumers / 32], s_flags[kStreamMaxConsumers / 32];
  const uint32_t c = threadIdx.x, lane = c & 31u, w = c >> 5;
  const unsigned long long tag = round & kOfferRoundMask;
  uint32_t prefix = 0xFFFFFFFFu, flags = 0;   // flags: bit 0 stalled, bit 1 missing
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
  if (c == 0) {
    for (uint32_t i = 1; i < blockDim.x / 32; i++) { prefix = min(prefix, s_min[i]); flags |= s_flags[i]; }
    const uint32_t status = (flags & 2u) ? kErrStreamTimeout : 0u;
    if (status) asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(err_word), "r"(status) : "memory");   // host-mapped, sticky
    out->m = flags ? 0u : prefix;
    out->stalled = flags & 1u;
    out->status = status;
  }
}
#endif  // __CUDACC__

}  // namespace cpbus_dev
