// cpbus_group.cpp — the group: one bus handle over the GPUs of a box (include/cpbus.h: cpbus_group_*), host C++ over
// the single bus's entry points and the internals that cpbus_internal.hpp declares.  It launches no kernel itself: each
// of its launches is one stream batch that every shard fans out (group_launch).
#include "cpbus_internal.hpp"

#include <algorithm>
#include <cstring>
#include <functional>
#include <mutex>
#include <vector>

// One launch of the single bus: the same early returns as launch_fanout, otherwise one stream batch on every shard.
// `device`: ev is a batch in device memory (cpbus_group_publish_device), which shard 0's put stream copies into the slot.
// The group's host records hold every record it staged itself; a device batch is accounted where the single bus accounts
// it, by the kernel — by shard 0's launch alone, marked in the group's debug ring in call order.
static int group_launch(cpbus_group* g, const cpbus_event* ev, uint32_t n, uint64_t w, bool device = false) {
  if (g->n_next == 0) return CPBUS_OK;
  if (n == 0 && g->n_timers == 0) return CPBUS_OK;
  int rc = stream_put(g->streams[0], ev, n, w, CPBUS_PUT_RAW, device);
  if (rc) return rc;
  for (size_t k = 0; k < g->streams.size(); k++)   // the whole batch: already admitted on every shard, so it completes in one launch
    if ((rc = stream_fanout_prefix(g->streams[k], n, w, n, device && k == 0))) return rc;
  g->last_watermark = w;
  if (device && n) { dbg_mark_device_batch(g, g->shards[0]->launch_seq); g->dev_counted = true; }
  return CPBUS_OK;
}

// Lossless admission of n records at src (the staged records, or a device batch) on every shard (admit), the single bus's
// verdict being the conjunction and its prefix the minimum.  The records reach a shard's device only when its room bound
// cannot prove the fit.
static int group_admit(cpbus_group* g, const cpbus_event* src, uint32_t n, uint64_t w, bool* ok, uint32_t* m) {
  *ok = true; *m = n;
  for (cpbus* s : g->shards) {
    if (admit_fits(s, n, w)) continue;
    int rc = dev_guard(s); if (rc) return rc;
    if (n) CK(cudaMemcpyAsync(s->d_admit_batch, src, (size_t)n * sizeof(cpbus_event), cudaMemcpyDefault, s->stream));
    bool ok_s = true;
    uint32_t m_s = n;
    if ((rc = admit_pass(s, s->d_admit_batch, n, w, &ok_s, &m_s))) return rc;
    if (!ok_s) { *ok = false; *m = std::min(*m, m_s); }
  }
  return CPBUS_OK;
}

// The group's flush: the single bus's outcome (the whole staged batch, or in lossless mode the prefix every shard can take
// with the partial watermark), as one stream batch
int cpbus_host::flush_staged(cpbus_group* g, uint64_t w) {
  if (flush_idle(g, w)) return CPBUS_OK;
  const uint32_t n = (uint32_t)g->n_staged;
  bool ok = true;
  uint32_t m = n;
  int rc;
  if (g->lossless && (rc = group_admit(g, g->staged.data(), n, w, &ok, &m))) return rc;
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

cpbus_event* cpbus_host::staging(cpbus_group* g) { return g->staged.data(); }

// The group: the same catch-up on every shard that has timers (its shards are dense buses).
int cpbus_host::catch_up(cpbus_group* g, uint64_t now) {
  for (cpbus* s : g->shards) {
    if (!s->K || s->n_timers == 0) continue;
    int rc = dev_guard(s);
    if (rc || (rc = catch_up(s, now))) return rc;
  }
  return CPBUS_OK;
}

static uint32_t group_shard_of(const cpbus_group* g, uint32_t index) {   // index < N
  return (uint32_t)(std::upper_bound(g->first.begin(), g->first.end(), index) - g->first.begin()) - 1;
}

// retire_oneshots for the group's table and, at the same moment, every shard's own: a shard's timer count (and so its
// window) then never lags the group's
static void group_retire(cpbus_group* g) {
  retire_oneshots(g, g->last_watermark);
  for (cpbus* s : g->shards) if (!s->h_timers.empty()) retire_oneshots(s, s->last_watermark);
}

// the owning shard of global id `sub_id` and its local index; false: not a subscribed-so-far id, or a released one (*s and
// *l are still set when the id is below n_next)
static bool group_locate(const cpbus_group* g, uint32_t sub_id, cpbus** s, uint32_t* l) {
  uint32_t i = 0;
  if (!id_range(g->base, g->n_next, sub_id, 1, &i)) return false;
  const uint32_t k = group_shard_of(g, i);
  *s = g->shards[k]; *l = i - g->first[k];
  return !(*s)->h_released[*l];   // a released id is refused as one never handed out
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
  if (cfg->flags & CPBUS_CFG_SPARSE_TICKS) return CPBUS_EINVAL;   // the group's flush is a stream batch (see cpbus_stream_create)
  if (cfg->flags & CPBUS_CFG_SPARSE_RECORDS) return CPBUS_EINVAL;
  if (cfg->flags & CPBUS_CFG_SPARSE_DRAINS) return CPBUS_EINVAL;
  uint32_t R = 0, B = 0;
  if (config_check(cfg, &R, &B) || cfg->n_max_subs < n_devices) return CPBUS_EINVAL;
  cpbus_group* g = new (std::nothrow) cpbus_group();
  if (!g) return CPBUS_ENOMEM;
  g->base = cfg->sub_id_base; g->N = cfg->n_max_subs; g->B = B; g->K = cfg->timers_per_sub;
  g->lossless = cfg->flags & CPBUS_CFG_LOSSLESS;
  g->drop_missed = cfg->flags & CPBUS_CFG_DROP_MISSED_TICKS;   // the group catches its shards up itself (catch_up)
  g->staged.resize(B);
  auto fail = [&](int code) { cpbus_group_destroy(g); return code; };
  const uint32_t each = g->N / n_devices, extra = g->N % n_devices;   // sharding.shard_range
  for (uint32_t k = 0; k < n_devices; k++) {
    const uint32_t first = k * each + std::min(k, extra), count = each + (k < extra ? 1u : 0u);
    cpbus_config c = *cfg;
    c.n_max_subs = count; c.device = devices[k]; c.sub_id_base = g->base + first;
    c.flags &= ~CPBUS_CFG_DROP_MISSED_TICKS;   // (a flagged shard would refuse the group's streams)
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
  // a device batch (cpbus_group_publish_device) may live on any GPU of the group: peer access between every two of them
  // where the hardware has it, as cpbus_stream_attach enables it towards shard 0
  for (cpbus* a : g->shards)
    for (cpbus* b : g->shards) {
      if (a->device == b->device) continue;
      int can = 0;
      if (cudaSetDevice(a->device) != cudaSuccess || cudaDeviceCanAccessPeer(&can, a->device, b->device) != cudaSuccess) return fail(CPBUS_ECUDA);
      if (!can) continue;
      const cudaError_t e = cudaDeviceEnablePeerAccess(b->device, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return fail(CPBUS_ECUDA);
      cudaGetLastError();   // clear "already enabled"
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

// The cyclic walk of a paged query (cpbus_drain_ready, cpbus_lagging) over ids [first_sub, first_sub + n) from start_sub, in
// pieces that each lie on one shard: fn(shard, local index, id, count) returns CPBUS_OK to go on, kWalkEnd to end the walk,
// or an error.  The checks are the single call's; *next_sub is set to start_sub (the walk found no cut) before the first piece.
constexpr int kWalkEnd = 1;
template <class Fn>
static int group_walk(cpbus_group* g, uint32_t first_sub, uint32_t n, uint32_t start_sub, uint32_t* next_sub, Fn&& fn) {
  if (start_sub < first_sub || start_sub - first_sub >= n) return CPBUS_EINVAL;
  uint32_t i0 = 0;
  if (!id_range(g->base, g->n_next, first_sub, n, &i0)) return CPBUS_ENOENT;
  const uint32_t rot = start_sub - first_sub;
  *next_sub = start_sub;
  for (uint32_t done = 0; done < n;) {
    const uint32_t i = i0 + (rot + done) % n;                       // global index of the walk's next mailbox
    const uint32_t k = group_shard_of(g, i);
    const uint32_t wrap = i0 + n - i;                               // the walk wraps to first_sub after this many
    const uint32_t cnt = std::min({n - done, g->first[k + 1] - i, wrap});
    const int rc = fn(g->shards[k], i - g->first[k], g->base + i, cnt);
    if (rc) return rc == kWalkEnd ? CPBUS_OK : rc;
    done += cnt;
  }
  return CPBUS_OK;
}

int cpbus_group_subscribe_many(cpbus_group_t* g, const uint32_t* masks, uint32_t n, uint32_t* first_sub_id) try {
  if (!g || !n) return CPBUS_EINVAL;
  if ((uint64_t)g->n_next + n > g->N) return CPBUS_ENOSPC;
  int rc = flush_staged(g, g->now); if (rc) return rc;
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
  int rc = flush_staged(g, g->now); if (rc) return rc;
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
  int rc = flush_staged(g, g->now); if (rc) return rc;
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
  int rc = flush_staged(g, g->now); if (rc) return rc;
  if ((rc = cpbus_unsubscribe(s, sub_id))) return rc;
  if (g->K && !g->h_timers.empty())
    for (uint32_t k = 0; k < g->K; k++) timer_disarm(g, (size_t)(sub_id - g->base) * g->K + k, /*reset_bound=*/false);
  g->n_active--;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_set_mask(cpbus_group_t* g, uint32_t sub_id, uint32_t mask) try {
  if (!g) return CPBUS_EINVAL;
  cpbus* s = nullptr; uint32_t l = 0;
  if (!group_locate(g, sub_id, &s, &l)) return CPBUS_ENOENT;
  if (!s->h_active[l]) return CPBUS_ECLOSED;
  const int rc = flush_staged(g, g->now); if (rc) return rc;
  return cpbus_set_mask(s, sub_id, mask);
} CPBUS_CATCH

int cpbus_group_timer_add(cpbus_group_t* g, uint32_t sub_id, uint64_t period_ns, uint32_t source_id, int oneshot, uint32_t* timer_id) try {
  if (!g || !period_ns) return CPBUS_EINVAL;
  if (!g->K) return CPBUS_ENOSPC;
  cpbus* s = nullptr; uint32_t l = 0;
  if (!group_locate(g, sub_id, &s, &l)) return CPBUS_ENOENT;
  int rc = flush_staged(g, g->now); if (rc) return rc;
  if (g->h_timers.empty()) g->h_timers.resize((size_t)g->N * g->K);
  group_retire(g);
  if (!s->h_active[l]) return CPBUS_ECLOSED;
  if ((rc = group_shard_clock(g, s))) return rc;
  uint32_t id = 0;
  if ((rc = cpbus_timer_add(s, sub_id, period_ns, source_id, oneshot, &id))) return rc;
  const uint32_t shard_base_slot = (sub_id - l - g->base) * g->K;   // global slot of the shard's slot 0
  const size_t slot = (size_t)(id & kTimerSlotMask) + shard_base_slot;
  timer_arm(g, slot, period_ns, source_id, oneshot != 0);
  if (timer_id) *timer_id = (uint32_t)slot | (id & ~kTimerSlotMask);
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_timer_add_many(cpbus_group_t* g, uint32_t first_sub, uint32_t n, uint64_t period_ns, const uint32_t* source_ids,
                               uint32_t source_id0, int oneshot) try {
  if (!g || !period_ns || !n) return CPBUS_EINVAL;
  if (!g->K) return CPBUS_ENOSPC;
  uint32_t i0 = 0;
  if (!id_range(g->base, g->n_next, first_sub, n, &i0)) return CPBUS_ENOENT;
  for (uint32_t i = 0; i < n; i++) {   // a released id: as one never handed out
    cpbus* s = nullptr; uint32_t l = 0;
    if (!group_locate(g, first_sub + i, &s, &l)) return CPBUS_ENOENT;
  }
  int rc = flush_staged(g, g->now); if (rc) return rc;
  if (g->h_timers.empty()) g->h_timers.resize((size_t)g->N * g->K);
  group_retire(g);
  // the single bus checks every subscriber before it arms any
  for (uint32_t i = 0; i < n; i++) {
    cpbus* s = nullptr; uint32_t l = 0;
    group_locate(g, first_sub + i, &s, &l);
    if (!s->h_active[l]) return CPBUS_ECLOSED;
    if (g->h_timers[(size_t)(i0 + i) * g->K].active) return CPBUS_ENOSPC;
  }
  rc = group_each_range(g, i0, n, [&](cpbus* s, uint32_t l, uint32_t off, uint32_t cnt) -> int {
    const int rc_clock = group_shard_clock(g, s);
    if (rc_clock) return rc_clock;
    return cpbus_timer_add_many(s, s->cfg.sub_id_base + l, cnt, period_ns, source_ids ? source_ids + off : nullptr,
                                source_id0 + off, oneshot);
  });
  if (rc) return rc;
  for (uint32_t i = 0; i < n; i++)
    timer_arm(g, (size_t)(i0 + i) * g->K, period_ns, source_ids ? source_ids[i] : source_id0 + i, oneshot != 0);
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_timer_cancel(cpbus_group_t* g, uint32_t timer_id) try {
  if (!g) return CPBUS_EINVAL;
  if (!g->K || g->h_timers.empty()) return CPBUS_ENOENT;
  const uint32_t slot = timer_id & kTimerSlotMask, i = slot / g->K;
  if (i >= g->n_next) return CPBUS_ENOENT;
  int rc = flush_staged(g, g->now); if (rc) return rc;
  group_retire(g);
  const uint32_t k = group_shard_of(g, i);
  const uint32_t local = (slot - g->first[k] * g->K) | (timer_id & ~kTimerSlotMask);
  if ((rc = cpbus_timer_cancel(g->shards[k], local))) return rc;
  timer_disarm(g, slot, /*reset_bound=*/true);
  return CPBUS_OK;
} CPBUS_CATCH

// The group's bulk membership calls: the single group calls' loop.  check(i, &k) is element i's refusal before the group's
// flush (CPBUS_OK: none, and k = its shard); the group flushes once, where the first element that passes would, then
// after_flush(); then each shard with work takes its elements, in array order, in one call of the shard's bulk call:
// run(k, elements, their statuses), which also keeps the group's own records of the elements the shard applied.  Shards
// are independent, and the group's records of these calls (n_active, n_timers, min_period) end where the interleaved loop
// leaves them.
template <class Check, class AfterFlush, class Run>
static int group_membership_many(cpbus_group* g, uint32_t n, int* status, uint32_t* applied, Check&& check,
                                 AfterFlush&& after_flush, Run&& run) {
  std::vector<int> st(n);
  std::vector<std::vector<uint32_t>> work(g->shards.size());
  bool any = false;
  for (uint32_t i = 0; i < n; i++) {
    uint32_t k = 0;
    if ((st[i] = check(i, &k)) == CPBUS_OK) { work[k].push_back(i); any = true; }
  }
  if (any) {
    int rc = flush_staged(g, g->now); if (rc) return rc;
    after_flush();
    std::vector<int> st_k;
    for (uint32_t k = 0; k < g->shards.size(); k++) {
      if (work[k].empty()) continue;
      st_k.assign(work[k].size(), CPBUS_OK);
      if ((rc = run(k, work[k], st_k.data()))) return rc;
      for (size_t j = 0; j < work[k].size(); j++) st[work[k][j]] = st_k[j];
    }
  }
  uint32_t ok = 0;
  for (uint32_t i = 0; i < n; i++) ok += st[i] == CPBUS_OK ? 1u : 0u;
  if (status && n) memcpy(status, st.data(), (size_t)n * sizeof(int));
  if (applied) *applied = ok;
  return CPBUS_OK;
}

int cpbus_group_unsubscribe_many(cpbus_group_t* g, const uint32_t* sub_ids, uint32_t n, int* status, uint32_t* applied) try {
  if (!g || (!sub_ids && n)) return CPBUS_EINVAL;
  std::vector<uint32_t> ids;
  return group_membership_many(g, n, status, applied,
      [&](uint32_t i, uint32_t* k) {
        cpbus* s = nullptr; uint32_t l = 0;
        if (!group_locate(g, sub_ids[i], &s, &l)) return CPBUS_ENOENT;
        *k = group_shard_of(g, sub_ids[i] - g->base);
        return CPBUS_OK;
      },
      [] {},
      [&](uint32_t k, const std::vector<uint32_t>& el, int* st) -> int {
        ids.resize(el.size());
        for (size_t j = 0; j < el.size(); j++) ids[j] = sub_ids[el[j]];
        const int rc = cpbus_unsubscribe_many(g->shards[k], ids.data(), (uint32_t)ids.size(), st, nullptr);
        if (rc) return rc;
        for (size_t j = 0; j < el.size(); j++) {
          if (st[j] != CPBUS_OK) continue;
          if (g->K && !g->h_timers.empty())
            for (uint32_t t = 0; t < g->K; t++) timer_disarm(g, (size_t)(ids[j] - g->base) * g->K + t, /*reset_bound=*/false);
          g->n_active--;
        }
        return CPBUS_OK;
      });
} CPBUS_CATCH

int cpbus_group_set_mask_many(cpbus_group_t* g, const uint32_t* sub_ids, const uint32_t* code_masks, uint32_t n, int* status,
                              uint32_t* applied) try {
  if (!g || ((!sub_ids || !code_masks) && n)) return CPBUS_EINVAL;
  std::vector<uint32_t> ids, masks;
  return group_membership_many(g, n, status, applied,
      [&](uint32_t i, uint32_t* k) {
        cpbus* s = nullptr; uint32_t l = 0;
        if (!group_locate(g, sub_ids[i], &s, &l)) return CPBUS_ENOENT;
        if (!s->h_active[l]) return CPBUS_ECLOSED;
        *k = group_shard_of(g, sub_ids[i] - g->base);
        return CPBUS_OK;
      },
      [] {},
      [&](uint32_t k, const std::vector<uint32_t>& el, int* st) -> int {
        ids.resize(el.size()); masks.resize(el.size());
        for (size_t j = 0; j < el.size(); j++) { ids[j] = sub_ids[el[j]]; masks[j] = code_masks[el[j]]; }
        return cpbus_set_mask_many(g->shards[k], ids.data(), masks.data(), (uint32_t)ids.size(), st, nullptr);
      });
} CPBUS_CATCH

int cpbus_group_timer_cancel_many(cpbus_group_t* g, const uint32_t* timer_ids, uint32_t n, int* status, uint32_t* applied) try {
  if (!g || (!timer_ids && n)) return CPBUS_EINVAL;
  std::vector<uint32_t> ids;
  return group_membership_many(g, n, status, applied,
      [&](uint32_t i, uint32_t* k) {
        if (!g->K || g->h_timers.empty()) return CPBUS_ENOENT;
        const uint32_t slot = timer_ids[i] & kTimerSlotMask;
        if (slot / g->K >= g->n_next) return CPBUS_ENOENT;
        *k = group_shard_of(g, slot / g->K);
        return CPBUS_OK;
      },
      [&] { group_retire(g); },
      [&](uint32_t k, const std::vector<uint32_t>& el, int* st) -> int {
        ids.resize(el.size());   // the shard's own timer ids, as cpbus_group_timer_cancel maps them
        for (size_t j = 0; j < el.size(); j++)
          ids[j] = ((timer_ids[el[j]] & kTimerSlotMask) - g->first[k] * g->K) | (timer_ids[el[j]] & ~kTimerSlotMask);
        const int rc = cpbus_timer_cancel_many(g->shards[k], ids.data(), (uint32_t)ids.size(), st, nullptr);
        if (rc) return rc;
        for (size_t j = 0; j < el.size(); j++)
          if (st[j] == CPBUS_OK) timer_disarm(g, timer_ids[el[j]] & kTimerSlotMask, /*reset_bound=*/true);
        return CPBUS_OK;
      });
} CPBUS_CATCH

int cpbus_group_timer_add_list(cpbus_group_t* g, const cpbus_timer_spec* specs, uint32_t n, uint32_t* timer_ids, int* status,
                               uint32_t* applied) try {
  if (!g || (!specs && n)) return CPBUS_EINVAL;
  std::vector<int> st(n);
  std::vector<uint32_t> ids(n), shard_ids;
  std::vector<cpbus_timer_spec> shard_specs;
  const int rc = group_membership_many(g, n, st.data(), applied,
      [&](uint32_t i, uint32_t* k) {
        if (!specs[i].period_ns) return CPBUS_EINVAL;
        if (!g->K) return CPBUS_ENOSPC;
        cpbus* s = nullptr; uint32_t l = 0;
        if (!group_locate(g, specs[i].sub_id, &s, &l)) return CPBUS_ENOENT;
        *k = group_shard_of(g, specs[i].sub_id - g->base);
        return CPBUS_OK;
      },
      [&] {
        if (g->h_timers.empty()) g->h_timers.resize((size_t)g->N * g->K);
        group_retire(g);
      },
      [&](uint32_t k, const std::vector<uint32_t>& el, int* st_k) -> int {
        int rc_k = group_shard_clock(g, g->shards[k]); if (rc_k) return rc_k;
        shard_specs.resize(el.size()); shard_ids.resize(el.size());
        for (size_t j = 0; j < el.size(); j++) shard_specs[j] = specs[el[j]];
        rc_k = cpbus_timer_add_list(g->shards[k], shard_specs.data(), (uint32_t)el.size(), shard_ids.data(), st_k, nullptr);
        if (rc_k) return rc_k;
        for (size_t j = 0; j < el.size(); j++) {   // the group's slot and id, as cpbus_group_timer_add maps them
          if (st_k[j] != CPBUS_OK) continue;
          const cpbus_timer_spec& s = shard_specs[j];
          const size_t slot = (size_t)(shard_ids[j] & kTimerSlotMask) + (size_t)g->first[k] * g->K;
          timer_arm(g, slot, s.period_ns, s.source_id, s.oneshot != 0);
          ids[el[j]] = (uint32_t)slot | (shard_ids[j] & ~kTimerSlotMask);
        }
        return CPBUS_OK;
      });
  if (rc) return rc;
  if (timer_ids)
    for (uint32_t i = 0; i < n; i++) if (st[i] == CPBUS_OK) timer_ids[i] = ids[i];
  if (status && n) memcpy(status, st.data(), (size_t)n * sizeof(int));
  return CPBUS_OK;
} CPBUS_CATCH

// subscriber id reuse: each shard with work takes its elements, in array order, in one cpbus_release_many call; the group
// keeps the released global indices in its own free set
int cpbus_group_release_many(cpbus_group_t* g, const uint32_t* sub_ids, uint32_t n, int* status, uint32_t* applied) try {
  if (!g || (!sub_ids && n)) return CPBUS_EINVAL;
  std::vector<uint32_t> ids;
  return group_membership_many(g, n, status, applied,
      [&](uint32_t i, uint32_t* k) {
        cpbus* s = nullptr; uint32_t l = 0;
        if (!group_locate(g, sub_ids[i], &s, &l)) return CPBUS_ENOENT;
        if (s->h_active[l]) return CPBUS_EINVAL;
        *k = group_shard_of(g, sub_ids[i] - g->base);
        return CPBUS_OK;
      },
      [] {},
      [&](uint32_t k, const std::vector<uint32_t>& el, int* st) -> int {
        ids.resize(el.size());
        for (size_t j = 0; j < el.size(); j++) ids[j] = sub_ids[el[j]];
        const int rc = cpbus_release_many(g->shards[k], ids.data(), (uint32_t)ids.size(), st, nullptr);
        if (rc) return rc;
        for (size_t j = 0; j < el.size(); j++)
          if (st[j] == CPBUS_OK) {
            g->free_ids.push_back(ids[j] - g->base);
            std::push_heap(g->free_ids.begin(), g->free_ids.end(), std::greater<uint32_t>());
          }
        return CPBUS_OK;
      });
} CPBUS_CATCH

// The group hands out the lowest free global ids.  The shards fill in order, so the free ids of shard k's range are its own
// released ids and its own fresh ones, and the lowest of them are the ones shard k's cpbus_subscribe_list hands out: each
// shard with work takes its run of elements in one call.
int cpbus_group_subscribe_list(cpbus_group_t* g, const uint32_t* code_masks, const cpbus_pair* pairs, const uint32_t* n_pairs,
                               uint32_t n, uint32_t* sub_ids) try {
  if (!g || !n || !sub_ids || subscribe_list_check(n_pairs, pairs, n)) return CPBUS_EINVAL;
  if (g->free_ids.size() + (uint64_t)(g->N - g->n_next) < n) return CPBUS_ENOSPC;
  int rc = flush_staged(g, g->now); if (rc) return rc;
  std::vector<uint32_t> idx(n);   // global indices, ascending
  for (uint32_t i = 0; i < n; i++) {
    if (g->free_ids.empty()) { idx[i] = g->n_next++; continue; }
    idx[i] = g->free_ids.front();
    std::pop_heap(g->free_ids.begin(), g->free_ids.end(), std::greater<uint32_t>());
    g->free_ids.pop_back();
  }
  g->n_active += n;
  for (uint32_t i = 0; i < n;) {
    const uint32_t k = group_shard_of(g, idx[i]);
    uint32_t cnt = 1;
    while (i + cnt < n && idx[i + cnt] < g->first[k + 1]) cnt++;
    rc = cpbus_subscribe_list(g->shards[k], code_masks ? code_masks + i : nullptr, n_pairs ? pairs + (size_t)i * CPBUS_MAX_PAIRS : nullptr,
                              n_pairs ? n_pairs + i : nullptr, cnt, sub_ids + i);
    if (rc) return rc;
    for (uint32_t j = i; j < i + cnt; j++)
      if (sub_ids[j] != g->base + idx[j]) return CPBUS_ECUDA;   // cannot happen: the shard's lowest free ids are the group's
    i += cnt;
  }
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_publish(cpbus_group_t* g, const cpbus_event* ev, size_t n) try {
  if (!g || (!ev && n)) return CPBUS_EINVAL;
  return publish_burst(g, ev, n);
} CPBUS_CATCH

// Device batches on the group: publish_device_impl's rules on the group's host front (flush first, the order and argument
// checks, lossless all-or-nothing admission on every shard, the single bus's split), each launch one stream batch whose
// payload shard 0's put stream copies from d_events (group_launch).  The prefetch hints are checked as the single bus checks
// them; the fan-out kernels read shard 0's stream slot, and throughput-mode stream launches already pull the slot after
// next, so there is nothing for the hints to add.
static int group_publish_device(cpbus_group* g, const cpbus_event* d_events, size_t n, uint64_t watermark_ns, bool staged,
                                const void* d_next, size_t n_next);

// publish_device_split on the group: the records' timestamps are read on the stream of a shard on the batch's GPU
static int group_publish_device_split(cpbus_group* g, const cpbus_event* d_events, size_t n, uint64_t watermark_ns, bool staged,
                                      const void* d_next, size_t n_next) {
  std::vector<uint64_t> ts(n), wm;
  std::vector<size_t> end;
  cpbus* s = g->shards[0];
  if (n) {
    cudaPointerAttributes a{};
    CK(cudaPointerGetAttributes(&a, d_events));
    for (cpbus* x : g->shards) if (x->device == a.device) { s = x; break; }
    int rc = dev_guard(s); if (rc) return rc;
    CK(cudaMemcpy2DAsync(ts.data(), 8, reinterpret_cast<const unsigned char*>(d_events) + offsetof(cpbus_event, ts_ns), sizeof(cpbus_event),
                         8, n, cudaMemcpyDefault, s->stream));
    CK(cudaStreamSynchronize(s->stream));
  }
  int rc = split_plan(ts.data(), n, g->B, g->now, watermark_ns, max_window(g), end, wm);
  if (rc) return rc;
  size_t i = 0;
  for (size_t k = 0; k < end.size(); k++) {
    const bool last = k + 1 == end.size();
    rc = group_publish_device(g, d_events + i, end[k] - i, wm[k], staged, last ? d_next : nullptr, last ? n_next : 0);
    if (rc) return rc;
    g->shards[0]->st.device_splits++;
    i = end[k];
  }
  return CPBUS_OK;
}

static int group_publish_device(cpbus_group* g, const cpbus_event* d_events, size_t n, uint64_t watermark_ns, bool staged,
                                const void* d_next, size_t n_next) {
  if (!g || (!d_events && n) || ((uintptr_t)d_events & 31u) || n_next > g->B || ((uintptr_t)d_next & 31u)) return CPBUS_EINVAL;
  int rc = flush_staged(g, g->now); if (rc) return rc;
  if (watermark_ns < g->now) return CPBUS_EORDER;
  if (staged && g->lossless) return CPBUS_EINVAL;
  if (n > g->B || watermark_ns - g->last_watermark > max_window(g)) {
    if (g->lossless) return n > g->B ? CPBUS_EINVAL : CPBUS_EORDER;
    return group_publish_device_split(g, d_events, n, watermark_ns, staged, d_next, n_next);
  }
  bool ok = true;
  uint32_t m = (uint32_t)n;
  if (g->lossless && (rc = group_admit(g, d_events, (uint32_t)n, watermark_ns, &ok, &m))) return rc;
  if (!ok) return CPBUS_EAGAIN;   // (refused on some shard: nothing was put)
  g->now = watermark_ns;
  if ((rc = group_launch(g, d_events, (uint32_t)n, watermark_ns, true))) return rc;
  g->publishes += n; g->seq += n;
  return CPBUS_OK;
}

int cpbus_group_publish_device(cpbus_group_t* g, const void* d_events, size_t n, uint64_t watermark_ns) try {
  if (g && g->drop_missed) return CPBUS_EINVAL;
  return group_publish_device(g, (const cpbus_event*)d_events, n, watermark_ns, false, nullptr, 0);
} CPBUS_CATCH

int cpbus_group_publish_device_staged(cpbus_group_t* g, const void* d_events, size_t n, uint64_t watermark_ns, const void* d_next,
                                      size_t n_next) try {
  if (g && g->drop_missed) return CPBUS_EINVAL;
  return group_publish_device(g, (const cpbus_event*)d_events, n, watermark_ns, true, d_next, n_next);
} CPBUS_CATCH

int cpbus_group_send(cpbus_group_t* g, uint32_t sub_id, const cpbus_event* ev) try {
  if (!g || !ev || ev->code >= CPBUS_N_CODES) return CPBUS_EINVAL;
  cpbus* s = nullptr; uint32_t l = 0;
  if (!group_locate(g, sub_id, &s, &l)) return CPBUS_ENOENT;
  if (!s->h_active[l]) return CPBUS_ECLOSED;
  const int rc = stage_one(g, ev->code, ev->source_id, sub_id, CPBUS_F_UNICAST);
  if (rc) return rc;
  g->publishes++;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_advance(cpbus_group_t* g, uint64_t now_ns) try {
  return g ? advance_clock(g, now_ns) : CPBUS_EINVAL;
} CPBUS_CATCH

int cpbus_group_flush(cpbus_group_t* g) try {
  return g ? flush_staged(g, g->now) : CPBUS_EINVAL;
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
// take: ready as cpbus_take_ready sees it (records past the take cursor).
static int group_first_ready(cpbus* s, uint32_t l, uint32_t cnt, uint32_t* at, bool take = false) {
  std::vector<SubCtl> c(cnt);
  std::vector<unsigned long long> tk(cnt, 0ull);
  int rc = dev_guard(s); if (rc) return rc;
  CK(cudaMemcpyAsync(c.data(), s->d_ctl + l, (size_t)cnt * sizeof(SubCtl), cudaMemcpyDeviceToHost, s->stream));
  if (take && s->d_taken)
    CK(cudaMemcpyAsync(tk.data(), s->d_taken + l, (size_t)cnt * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s->stream));
  CK(cudaStreamSynchronize(s->stream));
  *at = cnt;
  for (uint32_t i = 0; i < cnt; i++) if (c[i].tail > std::max<uint64_t>(c[i].head, tk[i])) { *at = i; break; }
  return CPBUS_OK;
}

// The cyclic walk of cpbus_drain_ready (take: cpbus_take_ready) over the shards: each piece of the walk that lies on one
// shard is drained there with the cap and ready entries still left, and the walk stops at the first mailbox that does not
// fit, as the single call does.  The caller has checked the arguments.
static int group_drain_ready(cpbus_group* g, uint32_t first_sub, uint32_t n, uint32_t start_sub, cpbus_event* out, size_t cap,
                             cpbus_ready* ready, size_t ready_cap, size_t* n_ready, size_t* total, uint32_t* next_sub, bool take) {
  size_t nr = 0, tot = 0, ready_left = std::min<size_t>(ready_cap, n);
  const int rc = group_walk(g, first_sub, n, start_sub, next_sub, [&](cpbus* s, uint32_t l, uint32_t a, uint32_t cnt) -> int {
    if (ready_left == 0 || tot == cap) {                           // no room: the next ready mailbox ends the walk
      uint32_t at = cnt;
      const int rc_s = group_first_ready(s, l, cnt, &at, take); if (rc_s) return rc_s;
      if (at == cnt) return CPBUS_OK;
      *next_sub = a + at;
      return kWalkEnd;
    }
    size_t nr_s = 0, tot_s = 0;
    uint32_t next_s = a;
    bool all = false;
    const int rc_s = drain_ready_impl(s, a, cnt, a, out + tot, cap - tot, ready + nr, ready_left, &nr_s, &tot_s, &next_s, &all,
                                      take);
    if (rc_s) return rc_s;
    for (size_t j = 0; j < nr_s; j++) ready[nr + j].offset += (uint32_t)tot;
    nr += nr_s; tot += tot_s; ready_left -= nr_s;
    if (all) return CPBUS_OK;
    *next_sub = next_s;
    return kWalkEnd;
  });
  if (rc) return rc;
  *n_ready = nr; *total = tot;
  return CPBUS_OK;
}

int cpbus_group_drain_ready(cpbus_group_t* g, uint32_t first_sub, uint32_t n, uint32_t start_sub, cpbus_event* out, size_t cap,
                            cpbus_ready* ready, size_t ready_cap, size_t* n_ready, size_t* total, uint32_t* next_sub) try {
  if (!g || !out || !ready || !n_ready || !total || !next_sub || !n || !ready_cap) return CPBUS_EINVAL;
  if (!ready_cap_ok(cap, g->shards[0]->R, false, g->lossless)) return CPBUS_EINVAL;
  return group_drain_ready(g, first_sub, n, start_sub, out, cap, ready, ready_cap, n_ready, total, next_sub, false);
} CPBUS_CATCH

int cpbus_group_take_ready(cpbus_group_t* g, uint32_t first_sub, uint32_t n, uint32_t start_sub, cpbus_event* out, size_t cap,
                           cpbus_ready* ready, size_t ready_cap, size_t* n_ready, size_t* total, uint32_t* next_sub) try {
  if (!g || !out || !ready || !n_ready || !total || !next_sub || !n || !ready_cap) return CPBUS_EINVAL;
  if (!ready_cap_ok(cap, g->shards[0]->R, true, g->lossless)) return CPBUS_EINVAL;
  return group_drain_ready(g, first_sub, n, start_sub, out, cap, ready, ready_cap, n_ready, total, next_sub, true);
} CPBUS_CATCH

// Each shard with work takes its elements, in array order, in one cpbus_ack_many call; shards hold disjoint mailboxes, so
// the statuses are the single bus's.
int cpbus_group_ack_many(cpbus_group_t* g, const uint32_t* sub_ids, const uint32_t* counts, uint32_t n, int* status,
                         uint32_t* applied) try {
  if (!g || ((!sub_ids || !counts) && n)) return CPBUS_EINVAL;
  if (n == 0) {
    if (applied) *applied = 0;
    return CPBUS_OK;
  }
  if (!g->lossless) return CPBUS_EINVAL;
  std::vector<int> st(n);
  std::vector<std::vector<uint32_t>> work(g->shards.size());
  for (uint32_t i = 0; i < n; i++) {
    cpbus* s = nullptr; uint32_t l = 0;
    if (!group_locate(g, sub_ids[i], &s, &l)) st[i] = CPBUS_ENOENT;
    else work[group_shard_of(g, sub_ids[i] - g->base)].push_back(i);
  }
  std::vector<uint32_t> ids, cnts;
  std::vector<int> st_k;
  for (uint32_t k = 0; k < g->shards.size(); k++) {
    if (work[k].empty()) continue;
    ids.resize(work[k].size()); cnts.resize(work[k].size()); st_k.resize(work[k].size());
    for (size_t j = 0; j < work[k].size(); j++) { ids[j] = sub_ids[work[k][j]]; cnts[j] = counts[work[k][j]]; }
    const int rc = ack_many_impl(g->shards[k], ids.data(), cnts.data(), (uint32_t)ids.size(), st_k.data());
    if (rc) return rc;
    for (size_t j = 0; j < work[k].size(); j++) st[work[k][j]] = st_k[j];
  }
  ack_statuses(st, status, applied);
  return CPBUS_OK;
} CPBUS_CATCH

// The cyclic walk of cpbus_lagging over the shards: each piece on one shard is scanned with the cap still left; the first
// piece that could not return all of its lagging mailboxes sets next_sub, and every piece adds to the summary.
int cpbus_group_lagging(cpbus_group_t* g, uint32_t first_sub, uint32_t n, uint32_t start_sub, uint32_t min_backlog, cpbus_lag* out,
                        size_t cap, size_t* n_out, uint32_t* next_sub, cpbus_lag_summary* sum) try {
  if (!g || !n_out || !next_sub || !n || (!out && cap)) return CPBUS_EINVAL;
  cpbus_lag_summary acc{};
  size_t got = 0;
  bool cut = false;
  const int rc = group_walk(g, first_sub, n, start_sub, next_sub, [&](cpbus* s, uint32_t, uint32_t a, uint32_t cnt) -> int {
    cpbus_lag_summary part{};
    size_t n_s = 0;
    uint32_t next_s = a;
    bool all = false;
    const int rc_s = lagging_impl(s, a, cnt, a, min_backlog, out ? out + got : nullptr, cap - got, &n_s, &next_s, &part, &all);
    if (rc_s) return rc_s;
    got += n_s;
    if (!all && !cut) { *next_sub = next_s; cut = true; }
    acc.active += part.active; acc.lagging += part.lagging; acc.backlog_total += part.backlog_total;
    acc.backlog_max = std::max(acc.backlog_max, part.backlog_max); acc.lost_total += part.lost_total;
    for (int h = 0; h < 33; h++) acc.hist[h] += part.hist[h];
    return CPBUS_OK;
  });
  if (rc) return rc;
  *n_out = got;
  if (sum) *sum = acc;
  return CPBUS_OK;
} CPBUS_CATCH

// The group's next unit (its staged remainder and clock, as cpbus_blockers reads the single bus's) on every shard; the
// shards own ascending id ranges, so their lists concatenate in ascending order.
int cpbus_group_blockers(cpbus_group_t* g, uint32_t* out, size_t cap, size_t* n) try {
  if (!g || !n || (!out && cap)) return CPBUS_EINVAL;
  *n = 0;
  if (!g->lossless) return CPBUS_OK;
  const cpbus_event* rec = g->n_staged ? &g->staged[0] : nullptr;
  if (!rec && (g->n_timers == 0 || g->now == g->last_watermark)) return CPBUS_OK;   // the next flush launches nothing
  const uint64_t t = rec ? rec->ts_ns : g->now;
  size_t tot = 0;
  for (cpbus* s : g->shards) {
    std::lock_guard<std::mutex> lk(s->mu);
    int rc = enter(s); if (rc) return rc;
    const size_t used = std::min(tot, cap);
    size_t n_s = 0;
    if ((rc = blockers_impl(s, rec, t, out ? out + used : nullptr, cap - used, &n_s))) return rc;
    tot += n_s;
  }
  *n = tot;
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
  uint32_t i0 = 0;
  if (!id_range(g->base, g->n_next, first_sub, n, &i0)) return CPBUS_ENOENT;
  return group_each_range(g, i0, n, [&](cpbus* s, uint32_t l, uint32_t off, uint32_t cnt) -> int {
    return cpbus_digest(s, s->cfg.sub_id_base + l, cnt, out + off);
  });
} CPBUS_CATCH

int cpbus_group_digest_fold(cpbus_group_t* g, uint32_t first_sub, uint32_t n, uint64_t out[4]) try {
  if (!g || !out || !n) return CPBUS_EINVAL;
  uint32_t i0 = 0;
  if (!id_range(g->base, g->n_next, first_sub, n, &i0)) return CPBUS_ENOENT;
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
  const int rc = dbg_resolve(g, g->shards[0]); if (rc) return rc;
  *n = dbg_read(g, out, cap);
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
  for (int c = 0; c < CPBUS_N_CODES; c++)   // + device batches, accounted by shard 0's launches alone (group_launch)
    sum.published_by_code[c] = g->published_by_code[c] + s0.published_by_code[c];
  sum.n_subs = g->n_active; sum.n_timers = g->n_timers; sum.now_ns = g->now;
  sum.intern_entries = s0.intern_entries; sum.intern_bytes = s0.intern_bytes;
  sum.ephemeral_live = s0.ephemeral_live; sum.ephemeral_recycled = s0.ephemeral_recycled;
  *out = sum;
  return CPBUS_OK;
} CPBUS_CATCH

int cpbus_group_publish_counts(cpbus_group_t* g, cpbus_pair_count* out, size_t cap, size_t* n) try {
  if (!g || !n || (!out && cap)) return CPBUS_EINVAL;
  std::vector<unsigned long long> keys, cnts;
  if (g->dev_counted) {
    int rc = dev_guard(g->shards[0]);
    if (rc || (rc = device_pairs(g->shards[0], keys, cnts))) return rc;
  }
  pair_counts(g, keys.data(), cnts.data(), keys.size(), out, cap, n);
  return CPBUS_OK;
} CPBUS_CATCH

