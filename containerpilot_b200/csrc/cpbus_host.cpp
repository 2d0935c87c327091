// cpbus_host.cpp — libcpbus's host-only code: the planners over the indexes of host_index.hpp (sparse_plan, split_plan,
// mask_order) and the exports that need no device (status and code names, the record hash, and the planners and the
// due index driven from their arguments, so that they can be tested without a GPU).
#include "cpbus_internal.hpp"

#include <algorithm>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

thread_local char cpbus_host::g_cuda_err[256] = "";

// The plan of a sparse record flush (cpbus_sparse_plan is this function over an index built from its arguments).  For each
// record: a unicast record goes to its target if subscribed; a broadcast record to the live entries of its code's list and to
// the subscribers with its exact case whose mask lacks the code (the fan-out's rule: mask bit or case).  A code with more
// than max_m subscribers ends the planning at once, so a dense fleet costs O(records).  Each mailbox gets a plan entry the
// first time it turns up (x.slot maps it there), so the planning also ends as soon as a (max_m + 1)-th one does; the
// {mailbox, record} pairs are appended in record order.  The entries (at most max_m) are then sorted and the record indices
// scattered to them in that order: O(records planned + max_m log max_m), each entry's indices ascending.  False: the flush
// takes the full fan-out (more than max_m due slots or candidates, or more than max_d records planned).
bool cpbus_host::sparse_plan(SubIndex& x, const uint32_t* mask, const uint8_t* active, uint32_t n_subs, uint32_t base,
                             const cpbus_event* rec, size_t n, const std::vector<uint32_t>& due, uint32_t K, size_t max_m, size_t max_d,
                             std::vector<uint64_t>& pairs, std::vector<cpbus_plan_entry>& out, std::vector<uint32_t>& idx) {
  out.clear(); idx.clear(); pairs.clear();
  struct Reset {   // x.slot goes back to all UINT32_MAX whichever way the planning ends
    SubIndex& x; std::vector<cpbus_plan_entry>& out;
    ~Reset() { for (const cpbus_plan_entry& e : out) x.slot[e.local] = UINT32_MAX; }
  } reset{x, out};
  auto entry = [&](uint32_t l) -> cpbus_plan_entry* {   // nullptr: one mailbox too many
    uint32_t& s = x.slot[l];
    if (s == UINT32_MAX) {
      if (out.size() == max_m) return nullptr;
      s = (uint32_t)out.size();
      out.push_back(cpbus_plan_entry{l, 0u, 0u, 0u});
    }
    return &out[s];
  };
  if (due.size() > max_m) return false;
  for (uint32_t d : due) entry(d / K)->due_bits |= 1u << (d % K);
  auto take = [&](uint32_t l, size_t i) -> bool {
    cpbus_plan_entry* e = entry(l);
    if (!e) return false;
    e->count++;
    pairs.push_back((uint64_t)l << 32 | i);
    return true;
  };
  for (size_t i = 0; i < n; i++) {
    const cpbus_event& r = rec[i];
    if (r.target != CPBUS_TARGET_ALL) {
      const uint32_t l = r.target - base;
      if (r.target >= base && l < n_subs && active[l] && !take(l, i)) return false;
    } else if (r.code < CPBUS_N_CODES) {
      const uint32_t c = r.code;
      if (x.cnt[c] > max_m) return false;
      if (!x.ok[c]) x.rebuild(c, mask, active, n_subs);
      for (uint32_t l : x.list[c])
        if (SubIndex::takes(mask, active, l, c) && !take(l, i)) return false;
      if (!x.cases.empty()) {
        auto it = x.cases.find((uint64_t)c << 32 | r.source_id);
        if (it != x.cases.end())
          for (uint32_t l : it->second.subs)
            if (active[l] && !((mask[l] >> c) & 1u) && !take(l, i)) return false;
      }
    }
    if (pairs.size() > max_d) return false;
  }
  std::sort(out.begin(), out.end(), [](const cpbus_plan_entry& a, const cpbus_plan_entry& b) { return a.local < b.local; });
  uint32_t first = 0;
  for (uint32_t s = 0; s < out.size(); s++) {
    x.slot[out[s].local] = s;
    out[s].first = first; first += out[s].count; out[s].count = 0;
  }
  idx.resize(pairs.size());
  for (uint64_t p : pairs) {
    cpbus_plan_entry& e = out[x.slot[(uint32_t)(p >> 32)]];
    idx[e.first + e.count++] = (uint32_t)p;
  }
  return true;
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
void cpbus_host::mask_order(const uint32_t* masks, const uint8_t* active, uint32_t n, uint32_t ring_cap, uint32_t block, bool heavy_first,
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

// The cut itself, host-only (exported as cpbus_split_plan so that it can be tested without a GPU): slice k = records
// [end[k-1], end[k]) launched with watermark wm[k].  `now` = the bus clock (= the last launched watermark once staged events
// are flushed), `window` = the widest watermark step one launch may take (UINT64_MAX: no timer armed).
int cpbus_host::split_plan(const uint64_t* ts, size_t n, uint32_t batch_cap, uint64_t now, uint64_t watermark, uint64_t window,
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

uint32_t cpbus_abi_version(void) { return 2; }
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
// The due index of a sparse-ticks bus over a table of n_slots slots, driven by ops instead of the bus's entry points (arms
// start at the clock as timer_arm does; a launch fires what due_fire fires after a launch of the bus).
int cpbus_due_trace(const cpbus_due_op* ops, size_t n_ops, uint32_t n_slots, uint32_t K, cpbus_due_fire* out, size_t cap,
                    size_t* n_out) try {
  if ((!ops && n_ops) || !n_out || (cap && !out) || !(K == 1 || K == 2 || K == 4 || K == 8)) return CPBUS_EINVAL;
  std::vector<HostTimer> tm(n_slots);
  DueIndex x;
  x.init(n_slots);
  uint64_t clock = 0, last = 0, launches = 0;
  size_t n = 0;
  std::vector<cpbus_due_fire> fired;
  for (size_t i = 0; i < n_ops; i++) {
    const cpbus_due_op& op = ops[i];
    switch (op.kind) {
      case CPBUS_DUE_CLOCK: clock = op.value; break;
      case CPBUS_DUE_ARM:
      case CPBUS_DUE_ONESHOT: {
        if (op.slot >= n_slots || !op.value) return CPBUS_EINVAL;
        HostTimer& t = tm[op.slot];
        t.active = true; t.oneshot = op.kind == CPBUS_DUE_ONESHOT; t.period = op.value; t.next_due = due_after(clock, op.value);
        x.put(op.slot, t.next_due);
        break;
      }
      case CPBUS_DUE_DISARM:
        if (op.slot >= n_slots) return CPBUS_EINVAL;
        tm[op.slot].active = false; x.drop(op.slot);
        break;
      case CPBUS_DUE_UNSUB:
        if ((uint64_t)op.slot * K + K > n_slots) return CPBUS_EINVAL;
        for (uint32_t k = 0; k < K; k++) { tm[op.slot * K + k].active = false; x.drop(op.slot * K + k); }
        break;
      case CPBUS_DUE_CATCHUP: {
        if (op.value < last) return CPBUS_EINVAL;
        std::vector<uint32_t> moved;
        due_catchup(x, tm, op.value, &moved);
        clock = op.value;
        break;
      }
      case CPBUS_DUE_LAUNCH:
        if (op.value < last) return CPBUS_EINVAL;
        last = op.value;
        fired.clear();
        due_fire(x, tm, op.value, [&](uint32_t s, uint64_t ticks, uint64_t nd) {
          fired.push_back(cpbus_due_fire{launches, s, 0u, ticks, nd});
        });
        std::sort(fired.begin(), fired.end(), [](const cpbus_due_fire& a, const cpbus_due_fire& b) { return a.slot < b.slot; });
        for (const cpbus_due_fire& f : fired) { if (n < cap) out[n] = f; n++; }
        launches++;
        break;
      default: return CPBUS_EINVAL;
    }
  }
  *n_out = n;
  return CPBUS_OK;
} CPBUS_CATCH
// The candidate index of a sparse-drains bus over n_subs subscribed mailboxes, driven by ops instead of the bus's launches
// and drains (the bus's own list cap is max(256, subscribers / 4096), and its bound 4 times that).
int cpbus_ready_trace(const cpbus_ready_op* ops, size_t n_ops, const uint32_t* ids, size_t n_ids_total, uint32_t n_subs,
                      size_t list_cap, uint32_t* out, size_t cap, int64_t* counts, size_t* n_out) try {
  if ((!ops && n_ops) || (!ids && n_ids_total) || !n_out || (cap && !out) || (!counts && n_ops) || !list_cap) return CPBUS_EINVAL;
  ReadyIndex x;
  x.init(n_subs, 4 * list_cap);
  struct Open { uint64_t place; uint32_t first, n; bool take; };
  std::unordered_map<uint32_t, Open> open;
  std::vector<uint32_t> cand;
  size_t n = 0;
  for (size_t i = 0; i < n_ops; i++) {
    const cpbus_ready_op& op = ops[i];
    counts[i] = 0;
    if ((uint64_t)op.ids + op.n_ids > n_ids_total) return CPBUS_EINVAL;
    const uint32_t* list = ids + op.ids;
    for (uint32_t j = 0; j < op.n_ids; j++) if (list[j] >= n_subs) return CPBUS_EINVAL;
    switch (op.kind) {
      case CPBUS_READY_SPARSE: x.add(list, op.n_ids); break;
      case CPBUS_READY_FULL: x.full(); break;
      case CPBUS_READY_DRAIN:
      case CPBUS_READY_TAKE: {
        const bool take = op.kind == CPBUS_READY_TAKE;
        if (!op.n || (uint64_t)op.first + op.n > n_subs || open.count(op.ticket)) return CPBUS_EINVAL;
        open[op.ticket] = Open{x.place(), op.first, op.n, take};
        if (!x.candidates(take, op.first, op.n, list_cap, &cand)) { counts[i] = -1; break; }
        counts[i] = (int64_t)cand.size();
        for (uint32_t l : cand) { if (n < cap) out[n] = l; n++; }
        break;
      }
      case CPBUS_READY_END: {
        auto it = open.find(op.ticket);
        if (it == open.end()) return CPBUS_ENOENT;
        const Open o = it->second;
        open.erase(it);
        x.drained(o.take, o.place, list, op.n_ids, 1, op.cut >= o.n && o.first == 0 && o.n == n_subs);
        break;
      }
      case CPBUS_READY_CONSUME_ALL: x.consumed(); break;
      case CPBUS_READY_RELEASE: x.released(list, op.n_ids); break;
      default: return CPBUS_EINVAL;
    }
  }
  *n_out = n;
  return CPBUS_OK;
} CPBUS_CATCH
// The plan of a sparse-records flush over an index built from the arguments, with the bus's own planning code (keep =
// max_mailboxes: a code with more subscribers keeps only its count, as on a bus).
int cpbus_sparse_plan(const uint32_t* masks, const uint8_t* active, uint32_t n_subs, const cpbus_pair* pairs,
                      const uint32_t* n_pairs, uint32_t sub_id_base, const cpbus_event* records, size_t n_records,
                      const uint32_t* due_slots, size_t n_due, uint32_t K, size_t max_mailboxes, size_t max_deliveries,
                      cpbus_plan_entry* out, size_t cap, uint32_t* rec_idx, size_t idx_cap, size_t* n_out, size_t* n_idx) try {
  if ((!masks && n_subs) || (!records && n_records) || (!due_slots && n_due) || (pairs && !n_pairs) || !n_out || !n_idx ||
      (cap && !out) || (idx_cap && !rec_idx) || !(K == 0 || K == 1 || K == 2 || K == 4 || K == 8) || (!K && n_due))
    return CPBUS_EINVAL;
  for (size_t d = 0; d < n_due; d++) if (due_slots[d] / K >= n_subs) return CPBUS_EINVAL;
  if (pairs) for (uint32_t l = 0; l < n_subs; l++) if (n_pairs[l] > CPBUS_MAX_PAIRS) return CPBUS_EINVAL;
  std::vector<uint32_t> mask(n_subs);
  std::vector<uint8_t> act(n_subs, 1);
  for (uint32_t l = 0; l < n_subs; l++) { mask[l] = masks[l] & CPBUS_MASK_ALL; if (active) act[l] = active[l] ? 1 : 0; }
  SubIndex x;
  x.init(n_subs, max_mailboxes);
  for (uint32_t l = 0; l < n_subs; l++) {
    if (!act[l]) continue;
    x.add_codes(l, mask[l]);
    if (!pairs) continue;
    uint64_t keys[CPBUS_MAX_PAIRS];
    for (uint32_t j = 0; j < n_pairs[l]; j++) {
      const cpbus_pair& pr = pairs[(size_t)l * CPBUS_MAX_PAIRS + j];
      keys[j] = (uint64_t)pr.code << 32 | pr.source_id;
    }
    x.add_cases(l, keys, n_pairs[l]);
  }
  std::vector<uint32_t> due(due_slots, due_slots + n_due);
  std::sort(due.begin(), due.end());
  due.erase(std::unique(due.begin(), due.end()), due.end());
  std::vector<uint64_t> scratch;
  std::vector<cpbus_plan_entry> plan;
  std::vector<uint32_t> idx;
  if (!sparse_plan(x, mask.data(), act.data(), n_subs, sub_id_base, records, n_records, due, K, max_mailboxes, max_deliveries,
                   scratch, plan, idx))
    return CPBUS_ENOSPC;
  std::copy(plan.begin(), plan.begin() + std::min(cap, plan.size()), out);
  std::copy(idx.begin(), idx.begin() + std::min(idx_cap, idx.size()), rec_idx);
  *n_out = plan.size(); *n_idx = idx.size();
  return CPBUS_OK;
} CPBUS_CATCH

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
