"""SURVEY §8f N3 — second-level, source-aware filter on the device (`cpbus_subscribe_pairs`): a subscriber takes a
broadcast event when its code is in the mask OR {code, source} is one of its exact cases (the whole-Event cases of the
consumer's switch, jobs/jobs.go:188-231).  CUDA bus through the C-ABI against the CPU oracle, bit-exact."""
import numpy as np
import pytest

import oracle_binding as ob
import trace as tr
from containerpilot_b200 import _native as nat
from containerpilot_b200 import events as ev
from containerpilot_b200 import masks
from containerpilot_b200.bus import Bus, EVENT_DTYPE

pytestmark = pytest.mark.gpu


def publish_codes(bus, codes, srcs):
    e = np.zeros(len(codes), dtype=EVENT_DTYPE)
    e["code"], e["source_id"] = codes, srcs
    nat.check(bus.publish_many(e), "publish")


def test_pair_filter_semantics_and_errors():
    orc = ob.Oracle(4)
    subs = [(0, [(2, 7), (3, 9)]), (1 << 2, [(3, 9)]), (0, []), (nat.MASK_ALL, [(3, 9)])]
    for m, pr in subs:
        orc.subscribe(m, pr)
    with Bus(4, ring_cap=64, batch_cap=32) as bus:
        for m, pr in subs:
            bus.subscribe_pairs(m, pr)
        for code, src in [(2, 7), (2, 8), (3, 9), (3, 7), (4, 9), (3, 9)]:
            orc.publish(code, src); nat.check(bus.publish(code, src), "publish")
        nat.check(bus.flush(), "flush"); bus.sync()
        tr.compare(bus, orc, 4)
        assert [(int(r["code"]), int(r["source_id"])) for r in bus.peek_window(0)] == [(2, 7), (3, 9), (3, 9)]
        assert [(int(r["code"]), int(r["source_id"])) for r in bus.peek_window(1)] == [(2, 7), (2, 8), (3, 9), (3, 9)]
        assert len(bus.peek_window(2)) == 0 and len(bus.peek_window(3)) == 6
    with Bus(2) as bus:
        for bad in ([(17, 0)], [(1, 1)] * 17):
            with pytest.raises(nat.CpbusError) as e:
                bus.subscribe_pairs(0, bad)
            assert e.value.status == nat.EINVAL
        assert bus.subscribe_pairs(1 << 5, [(5, 3)]) == 0          # pair already covered by the mask: plain subscription


PAIR_TRACES = [(1, 0, 32, 0), (2, 1, 64, 0), (3, 2, 128, 0), (4, 4, 256, 0), (5, 8, 512, 0), (6, 0, 512, 0), (7, 0, 256, 0),
               (8, 2, 32, 0), (9, 0, 64, 1), (10, 2, 256, 1), (11, 1, 128, 3), (12, 4, 512, 3)]


@pytest.mark.parametrize("seed,K,batch_cap,grid_ctas", PAIR_TRACES,
                         ids=[f"{s}-{k}-{b}" + (f"-grid{g}" if g else "") for s, k, b, g in PAIR_TRACES])
def test_pair_filter_random_traces(seed, K, batch_cap, grid_ctas):
    """pairs mixed with plain masks, unicast sends, membership changes, clock advances and timers.  A fixed grid
    (grid_ctas) over ~1,000 subscribers makes every warp walk several blocks of 32 mailboxes in the triage loop, which the
    default grid does only above 540,672 subscribers on an H100"""
    n0 = 900 if grid_ctas else 24
    ops, n_total = tr.random_ops(seed + 900, n0, 4000, timers_per_sub=K, max_subs=n0 + 16, p_filter=0.8, p_send=0.04,
                                 n_sources=5, p_pairs=0.6)
    assert any(len(op) > 2 for op in ops if op[0] == "sub")
    assert not grid_ctas or (n_total + 31) // 32 > 8 * grid_ctas            # more triage blocks than warps
    orc = tr.run_oracle(ops, n0 + 16, timers_per_sub=K)
    with Bus(n0 + 16, ring_cap=4096, batch_cap=batch_cap, timers_per_sub=K, grid_ctas=grid_ctas) as bus:
        tr.run_bus(bus, ops)
        tr.compare(bus, orc, n_total, window=4096)


@pytest.mark.parametrize("store", [nat.STORE_V4, nat.STORE_BULK])
def test_pair_filter_other_store_paths(store):
    ops, n_total = tr.random_ops(977, 24, 3000, timers_per_sub=2, max_subs=40, p_filter=0.8, n_sources=5, p_pairs=0.6)
    orc = tr.run_oracle(ops, 40, timers_per_sub=2)
    with Bus(40, ring_cap=4096, batch_cap=128, timers_per_sub=2, store_path=store, digest=False) as bus:
        tr.run_bus(bus, ops)
        got = bus.digests(0, n_total)
        for s in range(n_total):
            assert int(got["count"][s]) == orc.count(s)
            assert bus.peek_window(s).tobytes() == orc.mailbox(s)[-4096:].tobytes()


def test_job_fleet_exact_cases_scaled():
    """A fleet of Job-shaped subscribers, each with the exact cases of its own switch (13-16 pairs, mask 0), plus Metric
    consumers (mask on Metric + 2 cases) and a few unfiltered ones: every mailbox equals the oracle's, and the device
    delivers a small fraction of what code masks alone would."""
    n_jobs, n_metric, n_all, n_events = 1500, 40, 8, 12_000
    names = ["", "global", "closed", "SIGHUP", "SIGUSR2"]
    for j in range(n_jobs):
        names += [f"job{j}", f"check.job{j}", f"job{j}.heartbeat", f"job{j}.run-every", f"job{j}.wait-timeout"]
    src_id = {s: i for i, s in enumerate(names)}
    rng = np.random.default_rng(0xC0DEB2A3)
    subs = []
    for j in range(n_jobs):
        dep = int(rng.integers(0, n_jobs))
        sw = masks.JobSwitch(f"job{j}", start_event=ev.Event(ev.ExitSuccess, f"job{dep}") if j % 3 else ev.GlobalStartup)
        m, cases = sw.cases()
        subs.append((m, [(e.Code, src_id[e.Source]) for e in cases]))
    for _ in range(n_metric):
        m, cases = masks.MetricSwitch().cases()
        subs.append((m, [(e.Code, src_id[e.Source]) for e in cases]))
    subs += [(nat.MASK_ALL, [])] * n_all
    rng.shuffle(subs)
    n_subs = len(subs)
    codes = rng.integers(1, 17, n_events).astype(np.uint32)
    srcs = rng.integers(0, len(names), n_events).astype(np.uint32)
    orc = ob.Oracle(n_subs, keep_window=1024)
    mask_only = 0
    hist = np.bincount(codes, minlength=17)
    for m, pr in subs:
        orc.subscribe(m, pr)
        cm = m
        for c, _ in pr:
            cm |= 1 << c
        mask_only += int(sum(int(hist[c]) for c in range(17) if (cm >> c) & 1))
    orc.publish_many(codes, srcs)
    with Bus(n_subs, ring_cap=1024, batch_cap=512) as bus:
        for m, pr in subs:
            bus.subscribe_pairs(m, pr)
        publish_codes(bus, codes, srcs)
        nat.check(bus.flush(), "flush"); bus.sync()
        st = tr.compare(bus, orc, n_subs)
        assert st["deliveries"] == orc.total_deliveries()
        assert st["deliveries"] < 0.05 * mask_only


def test_fleet_registered_in_one_call():
    """cpbus_subscribe_pairs_many == n calls of cpbus_subscribe_pairs (also mixed with plain subscriptions before and after)"""
    rng = np.random.default_rng(0xC0DEB2A4)
    n, n_events = 700, 6000
    subs = []
    for i in range(n):
        m = int(rng.integers(0, 1 << 17)) & int(rng.integers(0, 1 << 17)) if i % 5 else nat.MASK_ALL
        pr = [(int(rng.integers(0, 17)), int(rng.integers(0, 40))) for _ in range(int(rng.integers(0, 17)))] if i % 7 else []
        subs.append((m, pr))
    codes = rng.integers(0, 17, n_events).astype(np.uint32); srcs = rng.integers(0, 40, n_events).astype(np.uint32)
    orc = ob.Oracle(n + 2, keep_window=1024)
    orc.subscribe(1 << 3)
    for m, pr in subs:
        orc.subscribe(m, pr)
    orc.subscribe(0, [(4, 4)])
    orc.publish_many(codes, srcs)
    with Bus(n + 2, ring_cap=1024, batch_cap=256) as bus:
        assert bus.subscribe(1 << 3) == 0
        assert bus.subscribe_pairs_many([m for m, _ in subs], [pr for _, pr in subs]) == 1
        assert bus.subscribe_pairs(0, [(4, 4)]) == n + 1
        publish_codes(bus, codes, srcs)
        nat.check(bus.flush(), "flush"); bus.sync()
        tr.compare(bus, orc, n + 2)
        with pytest.raises(nat.CpbusError) as e:
            bus.subscribe_pairs_many([0], [[(17, 1)]])
        assert e.value.status == nat.EINVAL


def test_pair_filter_lossless_backpressure():
    """admission counts pair matches exactly: a full mailbox of a pair-filtered subscriber stalls the publisher"""
    orc = ob.Oracle(3)
    subs = [(0, [(1, 5), (2, 6)]), (1 << 3, [(1, 5)]), (nat.MASK_ALL, [])]
    for m, pr in subs:
        orc.subscribe(m, pr)
    with Bus(3, ring_cap=64, batch_cap=32, lossless=True) as bus:
        for m, pr in subs:
            bus.subscribe_pairs(m, pr)
        got = [[], [], []]
        n_block = 0
        for i in range(1500):
            code, src = 1 + i % 3, 5 + (i // 3) % 2
            orc.publish(code, src)
            while True:
                rc = bus.publish(code, src)
                if rc == nat.EAGAIN:
                    n_block += 1
                    got[2].append(bus.drain(2))
                    if n_block % 4 == 0:
                        got[0].append(bus.drain(0)); got[1].append(bus.drain(1))
                    continue
                nat.check(rc, "publish"); break
        while bus.flush() == nat.EAGAIN:
            for s in range(3):
                got[s].append(bus.drain(s))
        for s in range(3):
            got[s].append(bus.drain(s))
            assert np.concatenate(got[s]).tobytes() == orc.mailbox(s).tobytes()
        assert n_block > 5 and bus.stats()["overwritten"] == 0
        assert orc.count(0) == 500 and orc.count(1) == 750


def test_events_api_subscribe_with_cases():
    """the Go-shaped API: Subscriber.Subscribe(bus, mask, cases) with a Job's own switch"""
    bus = ev.NewEventBus()
    job, everything = ev.Subscriber(ev.Chan(1000)), ev.Subscriber(ev.Chan(1000))
    sw = masks.JobSwitch("web", start_event=ev.Event(ev.StatusHealthy, "watch.db"))
    m, cases = sw.cases()
    job.Subscribe(bus, m, cases)
    everything.Subscribe(bus)
    stream = [ev.Event(ev.ExitSuccess, "check.web"), ev.Event(ev.ExitSuccess, "check.api"), ev.Event(ev.StatusHealthy, "watch.db"),
              ev.Event(ev.StatusHealthy, "watch.cache"), ev.Event(ev.Metric, "m|1"), ev.Event(ev.Signal, "SIGHUP"),
              ev.Event(ev.Signal, "SIGTERM"), ev.Event(ev.Quit, "web"), ev.Event(ev.Quit, "api"), ev.GlobalShutdown]
    for e in stream:
        bus.Publish(e)
    assert job.Received() == [e for e in stream if sw.handles(e)]
    assert everything.Received() == stream
    job.Unsubscribe(); everything.Unsubscribe()
    bus.close()
