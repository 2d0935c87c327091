// host_index.hpp — the host-only indexes of a bus and the planners that read them: the timer table's due-time
// arithmetic and the due index of a CPBUS_CFG_SPARSE_TICKS bus (DueIndex), the subscription index of a
// CPBUS_CFG_SPARSE_RECORDS bus (SubIndex), the drain candidates of a CPBUS_CFG_SPARSE_DRAINS bus (ReadyIndex), and the
// declarations of sparse_plan, split_plan and mask_order, which cpbus_host.cpp defines.  Plain C++17 with no device code:
// cpbus_due_trace, cpbus_sparse_plan, cpbus_ready_trace, cpbus_split_plan and cpbus_mask_order export this code so that it
// can be tested without a GPU.
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <map>
#include <unordered_map>
#include <vector>

#include "../../include/cpbus.h"
#include "cpbus_kernels.cuh"   // (its host part: kTimerIdle)

namespace cpbus_host __attribute__((visibility("hidden"))) {

using cpbus_dev::kTimerIdle;

struct HostTimer { bool active = false, oneshot = false; uint8_t gen = 0; uint64_t period = 0, next_due = 0; uint32_t source_id = 0; };
// Due times saturate: one that would pass UINT64_MAX - 1 is kTimerIdle, "never".  The slot stays armed (it counts in
// n_timers and can be cancelled); the kernel never fires a tick due at kTimerIdle.
inline uint64_t due_after(uint64_t t, uint64_t period) { return period >= kTimerIdle - t ? kTimerIdle : t + period; }
// a one-shot due by watermark w has fired on the device and disarmed itself
inline bool oneshot_fired(uint64_t next_due, uint64_t w) { return next_due <= w && next_due != kTimerIdle; }

// The due index of a CPBUS_CFG_SPARSE_TICKS bus: every armed slot whose next due time is not kTimerIdle, as {due, slot}
// entries in buckets of 2^kDueShift ns of due time (a calendar queue: a std::map from bucket to an unsorted vector of
// entries, with a lower bound of the bucket's due times).  Arming appends to one bucket, O(1) after the bucket's lookup;
// a launch to w takes the buckets wholly at or before w and scans the one that w falls in.  Nothing is removed from the
// middle of a bucket: a cancel, an unsubscribe or a re-arm bumps the slot's version, and an entry whose version is not the
// slot's any more is stale and skipped (32-bit versions, so a stale entry never passes for a live one the way a 6-bit
// timer-id generation could).  The whole index is rebuilt when stale entries outnumber the live ones.  A live slot's due
// time is also its HostTimer::next_due.  (A binary heap was measured first: at 10^6 slots each pop costs ~20 cache misses,
// ~2 us per due slot on the host; DESIGN.md §4.6.)
struct DueIndex {
  static constexpr int kDueShift = 20;   // ~1 ms of due time per bucket: the pump's step
  struct Entry { uint64_t due; uint32_t slot, ver; };
  struct Bucket { uint64_t lo = kTimerIdle; std::vector<Entry> e; };   // lo <= every live due in e
  std::map<uint64_t, Bucket> buckets;
  std::vector<uint32_t> ver;      // per slot
  std::vector<uint8_t> live;      // per slot: its current entry is in a bucket
  size_t n_live = 0, n_entries = 0;
  bool stale(const Entry& e) const { return ver[e.slot] != e.ver; }
  void init(size_t n_slots) { buckets.clear(); hot = nullptr; ver.assign(n_slots, 0); live.assign(n_slots, 0); n_live = n_entries = 0; }
  void drop(uint32_t slot) {
    ver[slot]++;
    if (live[slot]) { live[slot] = 0; n_live--; }
  }
  Bucket* hot = nullptr;          // the bucket the last insert went to (re-arms of one launch mostly share one)
  uint64_t hot_key = 0;
  void insert(const Entry& e) {
    const uint64_t k = e.due >> kDueShift;
    if (!hot || hot_key != k) { hot = &buckets[k]; hot_key = k; }
    hot->e.push_back(e); hot->lo = std::min(hot->lo, e.due);
    n_entries++;
  }
  void put(uint32_t slot, uint64_t due) {
    drop(slot);
    if (due == kTimerIdle) return;   // "never": not indexed, though the slot stays armed
    live[slot] = 1; n_live++;
    insert(Entry{due, slot, ver[slot]});
    if (n_entries > 2 * n_live + 64) compact();
  }
  void compact() {
    std::map<uint64_t, Bucket> old;
    old.swap(buckets);
    hot = nullptr; n_entries = 0;
    for (auto& kv : old) for (const Entry& e : kv.second.e) if (!stale(e)) insert(e);
  }
  // a lower bound of the earliest due time (kTimerIdle: nothing indexed); exact unless the first bucket holds stale entries
  uint64_t min_due() const { return buckets.empty() ? kTimerIdle : buckets.begin()->second.lo; }
  // The live slots due at or before w, appended to *out in no particular order, when there are at most cap of them (true);
  // false as soon as there are more.  Reads only the buckets that begin at or before w.
  bool collect(uint64_t w, size_t cap, std::vector<uint32_t>* out) const {
    size_t found = 0;
    for (auto it = buckets.begin(); it != buckets.end() && it->first <= (w >> kDueShift); ++it)
      for (const Entry& e : it->second.e)
        if (e.due <= w && !stale(e)) {
          if (++found > cap) return false;
          out->push_back(e.slot);
        }
    return true;
  }
};

// Firings of a periodic slot due at `due` <= w in one launch to w, as the kernel counts them: the candidates due + j *
// period <= w that do not reach kTimerIdle.  And the due time after k firings, saturating like the kernel's re-arm.
inline uint64_t due_ticks(uint64_t due, uint64_t period, uint64_t w) { return (std::min(w, kTimerIdle - 1) - due) / period + 1; }
inline uint64_t due_rearm(uint64_t due, uint64_t period, uint64_t k) {
  uint64_t step = 0;
  return (__builtin_mul_overflow(k, period, &step) || step >= kTimerIdle - due) ? kTimerIdle : due + step;
}

// After a launch to watermark w (any kernel that fires timers): every live slot due at or before w has fired on the device.
// A one-shot is done and leaves the index (retire_oneshots retires it in the host table as before); a periodic slot moves on
// by k = (w - due) / period + 1 periods into a later bucket.  on_fire(slot, ticks, next due) is told about each.  Each bucket
// that begins at or before w is taken out whole and its entries are fired, dropped as stale, or (only in the bucket w falls
// in) put back: O(due slots + that bucket), at most one pass over the table when every slot is due.
template <class F>
void due_fire(DueIndex& x, std::vector<HostTimer>& tm, uint64_t w, F&& on_fire) {
  const uint64_t last = w >> DueIndex::kDueShift;
  for (auto it = x.buckets.begin(); it != x.buckets.end() && it->first <= last;) {
    std::vector<DueIndex::Entry> v;
    v.swap(it->second.e);
    it = x.buckets.erase(it);   // (re-arms land after w, so in this bucket at the earliest: never in front of `it`)
    x.hot = nullptr;
    x.n_entries -= v.size();
    for (const DueIndex::Entry& e : v) {
      if (x.stale(e)) continue;
      if (e.due > w) { x.insert(e); continue; }
      HostTimer& t = tm[e.slot];
      if (t.oneshot) { x.drop(e.slot); on_fire(e.slot, (uint64_t)1, kTimerIdle); continue; }
      const uint64_t k = due_ticks(t.next_due, t.period, w);
      t.next_due = due_rearm(t.next_due, t.period, k);
      on_fire(e.slot, k, t.next_due);
      if (t.next_due == kTimerIdle) { x.drop(e.slot); continue; }
      x.ver[e.slot]++;   // a new entry for the slot, still live
      x.insert(DueIndex::Entry{t.next_due, e.slot, x.ver[e.slot]});
    }
  }
}

// CPBUS_CFG_DROP_MISSED_TICKS: the catch-up of a clock step to `now` in the due index, as timer_catchup_kernel does it on the
// device.  Every live periodic slot due at d <= now whose next firing is also <= now moves to d + k * period, k = (now - d) /
// period (below kTimerIdle: the kernel's candidates stop there too), under a new version; the slots that move are appended
// to *moved.  Reads the buckets that begin at or before now: O(entries due by now).
inline void due_catchup(DueIndex& x, std::vector<HostTimer>& tm, uint64_t now, std::vector<uint32_t>* moved) {
  const uint64_t w = std::min(now, kTimerIdle - 1);
  const size_t first = moved->size();
  for (auto it = x.buckets.begin(); it != x.buckets.end() && it->first <= (w >> DueIndex::kDueShift); ++it)
    for (const DueIndex::Entry& e : it->second.e) {
      if (x.stale(e) || e.due > w) continue;
      const HostTimer& t = tm[e.slot];
      if (!t.oneshot && w - e.due >= t.period) moved->push_back(e.slot);
    }
  for (size_t i = first; i < moved->size(); i++) {   // (put may rebuild the buckets: not while they are walked)
    HostTimer& t = tm[(*moved)[i]];
    t.next_due += (w - t.next_due) / t.period * t.period;
    x.put((*moved)[i], t.next_due);
  }
}

// The subscription index of a CPBUS_CFG_SPARSE_RECORDS bus: who takes a broadcast record, by code and by exact case.
//  * Per code: the count of subscribed mailboxes whose mask has the code's bit, and their list while the count is at most
//    `keep`.  A code past `keep` drops its list and keeps only the count: planning ends at once on such a code (it reaches
//    more mailboxes than the plan may), so an all-ones fleet holds 17 counts, not 17 N entries.  The list comes back by a scan
//    of the table when the plan next meets the code with few enough subscribers.  Entries are removed lazily: an entry is
//    live while its subscriber is subscribed and has the bit; `listed` (one word per subscriber) says which lists hold an
//    entry for it, so a bit that comes back revives the old entry instead of adding a second one, and a list is compacted
//    when its stale entries outnumber the live ones by 64.  Bound per code: 2 * min(count, keep) + 64 entries.
//  * Per exact case {code, source}: the subscribers with that case.  Cases are set at subscription and never change, so an
//    entry is live while its subscriber is subscribed; every subscriber's cases are kept (8 bytes each, the device table
//    keeps 8 too) so that an unsubscribe can find its lists, and a list is compacted when half of it is stale (+ 64).
//    A subscriber's cases sit in a segment of case_keys that a later occupant of its slot reuses when its cases fit, and
//    otherwise replaces by a segment of CPBUS_MAX_PAIRS: with slot reuse, at most n + CPBUS_MAX_PAIRS keys per slot.
//    Bound: 8 bytes per case subscribed so far, at most 8 * (n + CPBUS_MAX_PAIRS) per slot, and 2 * live + 64 entries per case.
// Maintenance is O(mask bits + cases) per subscriber and call, amortized.  `slot` (one word per subscriber, all UINT32_MAX
// between plans) maps a mailbox to its plan entry while a plan is built.  A CPBUS_CFG_SPARSE_TICKS bus without the records
// flag plans due ticks alone: it sizes `slot` and nothing else.
struct SubIndex {
  size_t keep = 0;
  uint32_t cnt[CPBUS_N_CODES] = {}, stale[CPBUS_N_CODES] = {};
  bool ok[CPBUS_N_CODES] = {};                       // list[c] is kept
  std::vector<uint32_t> list[CPBUS_N_CODES];
  std::vector<uint32_t> listed;                      // per subscriber: bit c <=> list[c] holds an entry for it
  struct Case { std::vector<uint32_t> subs; size_t stale = 0; };
  std::unordered_map<uint64_t, Case> cases;          // (code << 32 | source) -> subscribers
  std::vector<uint64_t> case_keys;                   // every subscriber's cases, in subscription order
  std::vector<uint32_t> case_first;                  // per subscriber (allocated with the first case): its cases in case_keys
  std::vector<uint8_t> case_n, case_cap;             // per subscriber: its cases, and the size of its segment
  std::vector<uint32_t> slot;                        // per subscriber: its entry in the plan being built (UINT32_MAX: none)

  static bool takes(const uint32_t* mask, const uint8_t* active, uint32_t l, uint32_t c) {
    return active[l] && ((mask[l] >> c) & 1u);
  }
  void init(size_t n, size_t keep_n) {
    keep = keep_n;
    listed.assign(n, 0); slot.assign(n, UINT32_MAX);
    for (uint32_t c = 0; c < CPBUS_N_CODES; c++) { cnt[c] = stale[c] = 0; ok[c] = true; list[c].clear(); }
    cases.clear(); case_keys.clear(); case_first.clear(); case_n.clear(); case_cap.clear();
  }
  void drop(uint32_t c) {
    for (uint32_t l : list[c]) listed[l] &= ~(1u << c);
    std::vector<uint32_t>().swap(list[c]);
    ok[c] = false; stale[c] = 0;
  }
  void compact(uint32_t c, const uint32_t* mask, const uint8_t* active) {
    size_t o = 0;
    for (uint32_t l : list[c]) {
      if (takes(mask, active, l, c)) list[c][o++] = l;
      else listed[l] &= ~(1u << c);
    }
    list[c].resize(o); stale[c] = 0;
  }
  void rebuild(uint32_t c, const uint32_t* mask, const uint8_t* active, uint32_t n) {
    list[c].clear();
    for (uint32_t l = 0; l < n; l++)
      if (takes(mask, active, l, c)) { list[c].push_back(l); listed[l] |= 1u << c; }
    ok[c] = true; stale[c] = 0;
  }
  // subscriber l has gained the codes in `bits` (it is subscribed and its mask has them)
  void add_codes(uint32_t l, uint32_t bits) {
    for (uint32_t c = 0; c < CPBUS_N_CODES; c++) {
      if (!((bits >> c) & 1u)) continue;
      cnt[c]++;
      if (!ok[c]) continue;
      if (cnt[c] > keep) { drop(c); continue; }
      if ((listed[l] >> c) & 1u) stale[c]--;   // its old entry is live again
      else { list[c].push_back(l); listed[l] |= 1u << c; }
    }
  }
  // subscriber l has lost the codes in `bits` (mask / active already say so)
  void remove_codes(uint32_t l, uint32_t bits, const uint32_t* mask, const uint8_t* active) {
    for (uint32_t c = 0; c < CPBUS_N_CODES; c++) {
      if (!((bits >> c) & 1u)) continue;
      cnt[c]--;
      if (!ok[c] || !((listed[l] >> c) & 1u)) continue;
      if (++stale[c] > cnt[c] + 64) compact(c, mask, active);
    }
  }
  // subscriber l (just subscribed) has the exact cases keys[0..n)
  void add_cases(uint32_t l, const uint64_t* keys, uint32_t n) {
    if (!n) return;
    if (case_first.empty()) { case_first.assign(listed.size(), 0); case_n.assign(listed.size(), 0); case_cap.assign(listed.size(), 0); }
    if (case_cap[l] < n) {   // a new segment: n keys for a slot's first subscriber with cases, the most a reused slot can need
      const uint32_t cap = case_cap[l] ? (uint32_t)CPBUS_MAX_PAIRS : n;
      case_first[l] = (uint32_t)case_keys.size(); case_cap[l] = (uint8_t)cap;
      case_keys.resize(case_keys.size() + cap);
    }
    case_n[l] = (uint8_t)n;
    for (uint32_t j = 0; j < n; j++) {
      case_keys[case_first[l] + j] = keys[j];
      Case& k = cases[keys[j]];
      if (k.subs.empty() || k.subs.back() != l) k.subs.push_back(l);   // (a case listed twice: one entry)
    }
  }
  // subscriber l has been unsubscribed (its cases stay recorded for release_cases)
  void remove_cases(uint32_t l, const uint8_t* active) {
    if (case_n.empty() || !case_n[l]) return;
    const uint64_t* keys = case_keys.data() + case_first[l];
    for (uint32_t j = 0; j < case_n[l]; j++) {
      if (std::find(keys, keys + j, keys[j]) != keys + j) continue;
      auto it = cases.find(keys[j]);
      Case& k = it->second;
      if (++k.stale * 2 <= k.subs.size() + 64) continue;
      size_t o = 0;
      for (uint32_t s : k.subs) if (active[s]) k.subs[o++] = s;
      k.subs.resize(o); k.stale = 0;
      if (!o) cases.erase(it);
    }
  }
  // subscriber l, unsubscribed, is being released (cpbus_release_many): its cases go to *touched, and purge_released then
  // takes the released subscribers' stale entries out of those lists, so that a later occupant of l with one of the same
  // cases is listed once
  void release_cases(uint32_t l, std::vector<uint64_t>* touched) {
    if (case_n.empty() || !case_n[l]) return;
    touched->insert(touched->end(), case_keys.begin() + case_first[l], case_keys.begin() + case_first[l] + case_n[l]);
    case_n[l] = 0;
  }
  // once per call: each touched list is filtered once, O(the touched lists' lengths) whatever number of its subscribers
  // the call released
  void purge_released(std::vector<uint64_t>& touched, const uint8_t* released) {
    std::sort(touched.begin(), touched.end());
    touched.erase(std::unique(touched.begin(), touched.end()), touched.end());
    for (uint64_t key : touched) {
      auto it = cases.find(key);
      if (it == cases.end()) continue;   // (compacted away)
      Case& k = it->second;
      size_t o = 0;
      for (uint32_t s : k.subs) if (!released[s]) k.subs[o++] = s;
      const size_t gone = k.subs.size() - o;   // stale entries: a released subscriber was unsubscribed
      k.subs.resize(o); k.stale = k.stale > gone ? k.stale - gone : 0;
      if (!o) cases.erase(it);
    }
  }
};

// The candidate index of a CPBUS_CFG_SPARSE_DRAINS bus: for each drain predicate a set of mailboxes that may hold records
// for it, or "unknown".  Set 0 (C_unread) serves cpbus_drain_ready: every mailbox that may have tail > head.  Set 1
// (C_untaken) serves cpbus_take_ready: every mailbox that may have tail > max(take cursor, head).  The invariant: at every
// point in stream order each mailbox with records for the predicate is in its set, or the set is unknown.
//  * Launches that append are numbered (`ord`).  A sparse launch stamps its mailboxes with its ordinal in both sets; any
//    other launch makes both unknown and records its ordinal as `blind`.
//  * A drain's place is the ordinal of the last launch in front of it in stream order (taken when it is enqueued).  When its
//    result is known it removes the mailboxes it took whose stamp is at most its place (a later launch may have refilled
//    the others).  A drain that took every ready mailbox of the whole subscribed range, with no blind launch after its
//    place, makes the set known: what holds records now was appended after its place, so it is the members stamped later.
//  * While unknown a set keeps stamping what sparse launches add, so that such a drain can make it known again.  A set of
//    more than `bound` members is emptied and made unknown (blind at the current ordinal).
// Drains of both kinds empty C_untaken; only cpbus_drain_ready empties C_unread.
struct ReadyIndex {
  // A set: per mailbox the ordinal of the launch that last added it (0: not a member), and the list of members, which may
  // also hold mailboxes removed since the list was last compacted (`listed`: in the list).  O(1) per added or removed
  // mailbox; a drain's candidates cost one pass over the list.
  struct Set {
    bool known = true;                               // a new bus: every mailbox is empty
    uint64_t blind = 0;                              // the last launch whose mailboxes may be missing from the set
    size_t live = 0;
    std::vector<uint64_t> stamp;
    std::vector<uint8_t> listed;
    std::vector<uint32_t> list;
    void put(uint32_t l, uint64_t o) {
      if (!stamp[l]) live++;
      stamp[l] = o;
      if (!listed[l]) { listed[l] = 1; list.push_back(l); }
    }
    void drop(uint32_t l) { if (stamp[l]) { stamp[l] = 0; live--; } }
    void clear() { for (uint32_t l : list) { stamp[l] = 0; listed[l] = 0; } list.clear(); live = 0; }
    void compact() {
      size_t o = 0;
      for (uint32_t l : list) { if (stamp[l]) list[o++] = l; else listed[l] = 0; }
      list.resize(o);
    }
    void tidy() { if (list.size() > 2 * live + 64) compact(); }
  };
  Set set[2];
  uint64_t ord = 0;
  size_t bound = 0;

  void init(size_t n, size_t bound_n) {
    bound = bound_n; ord = 0;
    for (Set& s : set) { s = Set{}; s.stamp.assign(n, 0); s.listed.assign(n, 0); }
  }
  uint64_t place() const { return ord; }
  void add(const uint32_t* ids, size_t n, size_t stride = 1) {
    ord++;
    for (Set& s : set) {
      for (size_t i = 0; i < n; i++) s.put(ids[i * stride], ord);
      if (s.live > bound) { s.clear(); s.known = false; s.blind = ord; }
    }
  }
  void full() {
    ord++;
    for (Set& s : set) { s.clear(); s.known = false; s.blind = ord; }
  }
  // a drain (take: a take_ready) placed at p took ids[0..n) (local indices, every `stride` words); complete: it took every
  // ready mailbox of the whole subscribed range
  void drained(bool take, uint64_t p, const uint32_t* ids, size_t n, size_t stride, bool complete) {
    for (int k = take ? 1 : 0; k < 2; k++) {
      Set& s = set[k];
      for (size_t i = 0; s.live && i < n; i++) {
        const uint32_t l = ids[i * stride];
        if (s.stamp[l] <= p) s.drop(l);
      }
      if (complete && s.blind <= p) {
        s.known = true;
        for (uint32_t l : s.list) if (s.stamp[l] <= p) s.drop(l);
        s.compact();
      } else {
        s.tidy();
      }
    }
  }
  void consumed() { for (Set& s : set) { s.clear(); s.known = true; } }
  void released(const uint32_t* ids, size_t n, size_t stride = 1) {
    for (Set& s : set) {
      for (size_t i = 0; i < n; i++) s.drop(ids[i * stride]);
      s.tidy();
    }
  }
  // The candidates of set `take` in [l, l + n), ascending, into *out: true when the set is known and holds at most cap of
  // them there; false for the dense scan.
  bool candidates(bool take, uint32_t l, uint32_t n, size_t cap, std::vector<uint32_t>* out) const {
    out->clear();
    const Set& s = set[take ? 1 : 0];
    if (!s.known) return false;
    for (uint32_t m : s.list)
      if (s.stamp[m] && m - l < n) {
        if (out->size() == cap) return false;
        out->push_back(m);
      }
    std::sort(out->begin(), out->end());
    return true;
  }
};

// The plan of a sparse record flush over index x (cpbus_host.cpp).
bool sparse_plan(SubIndex& x, const uint32_t* mask, const uint8_t* active, uint32_t n_subs, uint32_t base,
                 const cpbus_event* rec, size_t n, const std::vector<uint32_t>& due, uint32_t K, size_t max_m, size_t max_d,
                 std::vector<uint64_t>& pairs, std::vector<cpbus_plan_entry>& out, std::vector<uint32_t>& idx);
// The cut of a device batch into slices that one launch can take (cpbus_host.cpp).
int split_plan(const uint64_t* ts, size_t n, uint32_t batch_cap, uint64_t now, uint64_t watermark, uint64_t window,
               std::vector<size_t>& end, std::vector<uint64_t>& wm);
// The mask order of the ORDERED build (cpbus_host.cpp).
void mask_order(const uint32_t* masks, const uint8_t* active, uint32_t n, uint32_t ring_cap, uint32_t block, bool heavy_first,
                std::vector<uint32_t>& order);

}  // namespace cpbus_host
