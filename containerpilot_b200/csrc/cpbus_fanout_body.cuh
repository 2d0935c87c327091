// Body of fanout_kernel, fanout_follow_kernel and fanout_round_kernel (cpbus_kernels.cuh includes it inside each, with
// FOLLOW / ROUND = false / false, true / false and true / true).  Not a standalone header.
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
  uint32_t n = FOLLOW ? 0u : p.n_ev;   // FOLLOW: set from the descriptor summary (word kFollowN) once it is in
  uint64_t w_follow = 0;               // FOLLOW: the batch's watermark, in place of p.w_now
  unsigned long long round_ack = 0;    // ROUND, lead thread 0: the batch this launch completes (0: partial, no acknowledgement)

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
  const bool staged = FOLLOW || (p.staged && !stream_local);   // FOLLOW: a prefetched batch is pulled from local memory too
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
        // FOLLOW: the batch's size is in the descriptor the flag has just released (read from HBM: the bulk copy is in flight)
        const uint32_t n_copy = FOLLOW ? (ab ? 0u : *reinterpret_cast<const volatile uint32_t*>(p.desc + 24u * cap + 16u + 4u * kFollowN)) : n;
        if (staged && n_copy && !ab) {
          mbar_wait(&s_sum->mbar, 0);                                // phase 0 (power table) is over
          mbar_expect_tx(&s_sum->mbar, n_copy * 32u);
          bulk_g2s(s_batch, p.batch_local, n_copy * 32u, &s_sum->mbar);
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
    if constexpr (ROUND) {
      __syncthreads();   // thread 0 writes the shape into the summary below
      // The shape the shards agreed on, written by this shard's agree kernel (complete before this launch started: no PDL)
      if (tid == 0) {
        const volatile RoundDev* rd = p.round;
        if (!rd->go) s_sum->abort_launch = 1u;
        else {
          const unsigned long long w = rd->w;
          s_dsum[kFollowN] = rd->m; s_dsum[kFollowWLo] = (uint32_t)w; s_dsum[kFollowWHi] = (uint32_t)(w >> 32);
          s_dsum[kRoundSrc] = rd->src;
          if (lead && rd->final) round_ack = rd->q;
        }
      }
    } else if constexpr (FOLLOW) {
      __syncthreads();   // thread 0 writes the shape into the summary below
      // The clock: the host's, or the watermark the previous follower launch wrote (its lead did so before that launch let
      // this one start: acquired with its launch ordinal, bounded like the header).  Then the slot header, as below.
      if (tid == 0) {
        unsigned long long seen = 0, t0, t1, tag = 0, prev = p.w_now, hw = 0;
        const unsigned long long budget = (p.spin_us ? (unsigned long long)p.spin_us : 2000000ull) * 1000ull;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
        unsigned int err = 0;
        uint32_t hn = 0;
        if (!p.follow_from_host) {
          const unsigned long long* pw = p.follow_clock + 2u * (uint32_t)((p.launch_seq - 1ull) & 1ull);
          for (;;) {
            asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(tag) : "l"(pw + 1) : "memory");
            if (tag == p.launch_seq - 1ull) break;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
            if (t1 - t0 > budget) break;
            __nanosleep(64);
          }
          if (tag != p.launch_seq - 1ull) err = kErrStreamTimeout;
          else asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(prev) : "l"(pw) : "memory");
        }
        const bool skip = !err && prev == kFollowPoison;   // an earlier follower aborted: this one is a no-op
        if (!err && !skip) {
          for (;;) {
            asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(&p.stream_hdr->seq) : "memory");
            if (seen >= p.stream_seq) break;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
            if (t1 - t0 > budget) break;
            __nanosleep(64);
          }
          if (seen != p.stream_seq) err = kErrStreamTimeout;
          else {
            // the checks cpbus_stream_fanout makes on the host: the shape fits, the clock never moves backwards and the step
            // stays within the 32/K firings per timer slot that one launch examines
            asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(hn) : "l"(&p.stream_hdr->n) : "memory");
            asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(hw) : "l"(&p.stream_hdr->watermark) : "memory");
            if (hn > cap) err = kErrStreamShape;
            else if (hw < prev || hw - prev > p.follow_window) err = kErrFollowOrder;
            else { s_dsum[kFollowN] = hn; s_dsum[kFollowWLo] = (uint32_t)hw; s_dsum[kFollowWHi] = (uint32_t)(hw >> 32); }
          }
        }
        if (err || skip) s_sum->abort_launch = 1u;
        if (lead) {
          if (err) asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p.err_word), "r"(err) : "memory");   // host-mapped, sticky
          // this launch's clock pair (the next follower reads it), then what it took, for the host
          unsigned long long* pw = p.follow_clock + 2u * (uint32_t)(p.launch_seq & 1ull);
          asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(pw), "l"((err || skip) ? kFollowPoison : hw) : "memory");
          asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(pw + 1), "l"(p.launch_seq) : "memory");
          volatile FollowRec* rec = p.follow_rec;
          rec->n = (err || skip) ? 0u : hn; rec->watermark = hw;
          rec->status = skip ? kFollowSkipped : (err ? kFollowAborted : kFollowDelivered);
        }
      }
    } else if (stream && staged) {
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
    if constexpr (FOLLOW) {
      n = ab ? 0u : s_dsum[kFollowN];
      w_follow = ((uint64_t)s_dsum[kFollowWHi] << 32) | s_dsum[kFollowWLo];
    }
    if (staged && n && !ab) {   // peer pull: plain 16-byte loads on the NVLink-mapped pointer, into shared memory and the local copy
      const uint4* src = reinterpret_cast<const uint4*>(ROUND ? p.batch + s_dsum[kRoundSrc] : FOLLOW ? batch_src : p.batch);
      uint4* loc = reinterpret_cast<uint4*>(p.batch_local);
      uint4* dst = reinterpret_cast<uint4*>(s_batch);
      for (uint32_t i = tid; i < 2 * n; i += kThreads) {
        uint4 v;
        asm volatile("ld.global.relaxed.sys.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(src + i) : "memory");
        dst[i] = v;
        if (lead) loc[i] = v;
      }
      // the bulk store path reads s_batch through the async proxy (cp.async.bulk): order these generic writes before it
      if constexpr (STORE == CPBUS_STORE_BULK) asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    mbar_wait(&s_sum->mbar, 0);
    __syncthreads();
    if (lead && stream && tid == 0 && !ab && (ROUND ? round_ack != 0 : p.stream_final))   // the batch is out of the shared ring: the publisher may reuse the slot
      asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p.stream_ack), "l"(ROUND ? round_ack : p.stream_seq) : "memory");
    const uint32_t nd = ab ? 0u : n;
    {
      uint32_t present = 0, uni = 0;
      for (uint32_t i = tid; i < nd; i += kThreads) {
        const ulonglong4 w = *reinterpret_cast<const ulonglong4*>(&s_batch[i]);
        s_rhash[i] = record_hash_words(w.x, w.y, w.z, w.w);
        const uint32_t code = (uint32_t)w.z, target = (uint32_t)w.w;
        uint32_t codebit = 0;
        if (target == CPBUS_TARGET_ALL) {
          // a code outside the enum (only a complete record can carry one) takes bit / bucket kCodeOutOfRange, which no
          // control word carries: no mailbox selects it, dense runs are off for the batch and its publish is not counted
          const uint32_t c = min(code, kCodeOutOfRange);
          codebit = 1u << c; atomicAdd(&s_dsum[2 + c], 1u);
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
    if constexpr (FOLLOW) {
      n = s_sum->abort_launch ? 0u : s_dsum[kFollowN];
      w_follow = ((uint64_t)s_dsum[kFollowWHi] << 32) | s_dsum[kFollowWLo];
    }
    mbar_wait(&s_sum->mbar, (staged && n && !s_sum->abort_launch) ? 1u : 0u);
  }
  // ---- planar re-layout of the staged batch (in place): record i = {lo[i], hi[i]}, lo at s4[i], hi at s4[cap + i] ----
  // At a 32-byte lane stride the eight lanes of an LDS.128 wavefront touch only four of the eight 16-byte bank groups
  // (2-way conflict on every record read); at a 16-byte stride they touch all
  // eight.  All 2n chunks are read into registers (n <= 1024: at most 8 per thread), barrier, then written to their
  // plane: two barriers and 8 shared-memory instructions per thread per CTA, against ~2000 record reads per thread.
  // Not in the ORDERED build: its gathered reads do no better on planes, and not with the bulk store path, which copies
  // whole records out of shared memory.
  constexpr bool PLANAR = STORE != CPBUS_STORE_BULK && !ORDERED;
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
            live = due != kTimerIdle && due <= (FOLLOW ? w_follow : p.w_now);
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
      // due times saturate: a candidate whose sum passes UINT64_MAX - 1 never comes
      const uint64_t step = (uint64_t)tk_j * tk_period;
      tk_due = tk_due0 + step;
      const bool wraps = __umul64hi(tk_j, tk_period) != 0 || tk_due < step || tk_due == kTimerIdle;
      tk_valid = tk_due0 != kTimerIdle && !wraps && tk_due <= (FOLLOW ? w_follow : p.w_now) && (tk_j == 0 || tk_period != 0);
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
      constexpr bool cold_early = !STAGED;
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
#pragma unroll 1
      for (; c0 + 64 <= n; c0 += 64) {   // two chunks per iteration: both records' shared-memory loads are in flight before the selects
        const uint32_t o0 = slot_of(c0), o1 = slot_of(c0 + 32);
        copy_record_pairs<PLANAR>(s4, hi_off, ring, (uint32_t)tail, Rm, c0 + lane, o0, true);
        copy_record_pairs<PLANAR>(s4, hi_off, ring, (uint32_t)tail, Rm, c0 + 32 + lane, o1, true);
      }
#pragma unroll 1
      for (; c0 < n; c0 += 32) {
        const uint32_t out = slot_of(c0);
        copy_record_pairs<PLANAR>(s4, hi_off, ring, (uint32_t)tail, Rm, c0 + lane, out, c0 + lane < n);
      }
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
        // this lane has tk_j == 0, so tk_due is the slot's next_due as loaded.  A one-shot disarms itself; a periodic re-arm
        // past UINT64_MAX - 1 saturates to kTimerIdle (never fires again; the host still counts the slot as armed)
        const uint64_t step = (uint64_t)fired_here * tk_period;
        const uint64_t nd = (tk_period && __umul64hi(fired_here, tk_period) == 0 && step < kTimerIdle - tk_due) ? tk_due + step : kTimerIdle;
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
    if (tid < CPBUS_N_CODES && tid != CPBUS_METRIC && s_dsum[2 + tid]) atomicAdd(&p.acct->by_code[tid], (unsigned long long)s_dsum[2 + tid]);
    for (uint32_t i = tid; i < n; i += kThreads) {
      if (s_meta[i].y != CPBUS_TARGET_ALL) continue;
      const uint2 cs = ev_code_src(i);
      const uint32_t code = cs.x;
      if (code == CPBUS_METRIC || code >= CPBUS_N_CODES) continue;
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
      for (uint32_t c = 0; c <= kCodeOutOfRange; c++) nb += s_dsum[2 + c];
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
