"""The reference's own bus tests, re-stated against the mirror of the `events`
API running on the CUDA bus (containerpilot_b200.events).  Each test cites the
Go test it follows."""
import json
import os
from collections import Counter

import pytest

from containerpilot_b200 import events
from containerpilot_b200.events import Event

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
G = json.load(open(os.path.join(HERE, "golden", "reference_vectors.json")))


class TestPublisher(events.Publisher):              # events/events_test.go:13-21
    __test__ = False

    def __init__(self, bus):
        super().__init__()
        self.Register(bus)


class TestSubscriber(events.Subscriber):            # events/events_test.go:23-37
    __test__ = False

    def __init__(self):
        super().__init__(events.Chan(100))
        self.results = []

    def Run(self, bus):                             # events_test.go:39-61 (the goroutine body, run on demand)
        self.Subscribe(bus)

    def Stop(self):
        self.results += self.Received()
        self.Unsubscribe()
        self.Rx.close()


def test_pub_sub_interfaces():
    """events/events_test.go:64-89"""
    bus = events.NewEventBus()
    tp = TestPublisher(bus)
    ts = TestSubscriber()
    ts.Run(bus)
    expected = [Event(events.Startup, "serviceA")]
    for e in expected:
        tp.Publish(e)
    ts.Stop()
    assert bus.DebugEvents() == expected
    assert ts.results == expected               # the Go test collects but never asserts this; we do
    tp.Unregister()
    assert bus.Wait() is False
    bus.close()


def test_publish_signal():
    """events/events_test.go:91-113"""
    bus = events.NewEventBus()
    ts = TestSubscriber()
    ts.Run(bus)
    signals = ["SIGHUP", "SIGUSR2"]
    expected = [Event(events.Signal, s) for s in signals]
    for s in signals:
        bus.PublishSignal(s)
    ts.Stop()
    assert bus.DebugEvents() == expected and ts.results == expected
    bus.close()


def test_job_run_safe_close_sequence():
    """jobs/jobs_test.go:15-48: publish after the only subscriber unsubscribed must not panic."""
    bus = events.NewEventBus()
    job_sub, job_pub = events.Subscriber(events.Chan(1000)), events.Publisher()
    job_sub.Subscribe(bus); job_pub.Register(bus)
    bus.Publish(events.GlobalStartup)
    job_pub.Publish(Event(events.Stopping, "myjob"))      # jobs/jobs.go:390
    job_sub.Unsubscribe(); job_pub.Unregister()           # jobs/jobs.go:411-412
    bus.Publish(Event(events.Stopped, "myjob"))           # jobs/jobs.go:415
    assert bus.Wait() is False
    assert bus.DebugEvents() == [events.GlobalStartup, Event(events.Stopping, "myjob"), Event(events.Stopped, "myjob")]
    job_pub.Bus.Publish(events.GlobalStartup)             # must not raise
    assert job_sub.Received() == [events.GlobalStartup, Event(events.Stopping, "myjob")]
    bus.close()


@pytest.mark.parametrize("vec", G["multiset"], ids=lambda v: v["name"])
def test_multiset_vectors(vec):
    bus = events.NewEventBus()
    sub = events.Subscriber(events.Chan(1000)); sub.Subscribe(bus)
    for code, src in vec.get("direct_receives", []):
        sub.Receive(Event(code, src))                     # watches/watches_test.go:48-50
    for code, src in vec["published"]:
        bus.Publish(Event(code, src))
    got = Counter(f"{e.Code}|{e.Source}" for e in bus.DebugEvents())
    assert dict(got) == vec["debug_events"]
    want = [Event(c, s) for c, s in vec.get("direct_receives", [])] + [Event(c, s) for c, s in vec["published"]]
    assert sub.Received() == want
    bus.close()


def test_closed_mailbox_panics_and_double_unsubscribe_panics():
    """events/bus.go:135-137 (send on closed Rx panics) and :121 (negative WaitGroup)."""
    bus = events.NewEventBus()
    sub = events.Subscriber(events.Chan(10)); sub.Subscribe(bus)
    sub.Rx.close()
    with pytest.raises(events.BusPanic):
        bus.Publish(events.GlobalStartup)
    sub.Unsubscribe()
    with pytest.raises(events.BusPanic):
        sub.Unsubscribe()
    with pytest.raises(events.BusPanic):
        bus.Subscribe(object())                           # bus.go:108 type assertion
    bus.close()


def test_timers_deliver_to_owner_only():
    """events/timer.go:12-71 under the virtual clock; names as in jobs/jobs.go:147-158."""
    bus = events.NewEventBus()
    job = events.Subscriber(events.Chan(1000)); job.Subscribe(bus)
    other = events.Subscriber(events.Chan(1000)); other.Subscribe(bus)
    ctx, cancel = events.WithCancel()
    events.NewEventTimer(ctx, job.Rx, 1_000_000_000, "myjob.heartbeat")
    events.NewEventTimeout(ctx, job.Rx, 2_500_000_000, "myjob.wait-timeout")
    bus.Publish(events.GlobalStartup)
    bus.Advance(3_000_000_000)
    bus.Publish(Event(events.StatusHealthy, "myjob"))
    hb, to = Event(events.TimerExpired, "myjob.heartbeat"), Event(events.TimerExpired, "myjob.wait-timeout")
    assert job.Received() == [events.GlobalStartup, hb, hb, to, hb, Event(events.StatusHealthy, "myjob")]
    assert other.Received() == [events.GlobalStartup, Event(events.StatusHealthy, "myjob")]
    cancel()                                              # ctx.Done(): timer.go:57-58
    bus.Advance(10_000_000_000)
    bus.Publish(events.GlobalShutdown)
    assert job.Received() == [events.GlobalShutdown]
    assert bus.DebugEvents() == [events.GlobalStartup, Event(events.StatusHealthy, "myjob"), events.GlobalShutdown]
    bus.close()


def test_from_string_and_names():
    for name, code in G["from_string"]["accepted"].items():
        assert events.FromString(name) == (code, None)
    code, err = events.FromString("bogus")
    assert code == events.None_ and "bogus is not a valid event code" in str(err)      # events.go:85
    assert [events.CodeString(i) for i in range(17)] == G["code_names"]["names"]
    assert events.CodeString(42) == "EventCode(42)"                                    # eventcode_string.go:11


def test_cpp_mirror_restates_reference_tests():
    """The compiled-language host side (containerpilot_b200/csrc/host/events.hpp, C++17 over the C-ABI):
    events_test.cc restates events/events_test.go + the jobs/control/watches vectors, with real
    bounded channels and consumer threads."""
    import subprocess
    exe = os.path.join(os.path.dirname(HERE), "containerpilot_b200", "csrc", "host", "events_test")
    assert os.path.exists(exe), "build with __graft_entry__.build()"
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.strip().endswith("PASS"), r.stdout + r.stderr


@pytest.mark.parametrize("body,status,expected", [
    ("{{\n", 422, {}),
    ('{"mymetric": 1.0}', 200, {Event(events.Metric, "mymetric|1"): 1}),
    ('{"mymetric": 1.5, "myothermetric": 2}', 200,
     {Event(events.Metric, "mymetric|1.5"): 1, Event(events.Metric, "myothermetric|2"): 1}),
])
def test_post_metric_as_one_batch(body, status, expected):
    """control/endpoints_test.go:104-145 through the batched handler (containerpilot_b200/ingest.py, SURVEY §8f N4)"""
    from containerpilot_b200 import ingest
    bus = events.NewEventBus()
    sensor = events.Subscriber(events.Chan(1000))
    sensor.Subscribe(bus, 1 << events.Metric)
    _, got_status = ingest.post_metric(bus, body)
    assert got_status == status
    got = Counter(e for e in bus.DebugEvents() if e != events.GlobalStartup)
    assert dict(got) == expected
    assert Counter(sensor.Received()) == Counter(expected)
    sensor.Unsubscribe()
    bus.close()


def test_post_metric_burst_is_one_fan_out():
    """a 200-key request costs one staging pass and one launch instead of 200 publishes"""
    import json as _json
    from containerpilot_b200 import ingest
    bus = events.NewEventBus(n_max_subs=8, batch_cap=256)
    subs = [events.Subscriber(events.Chan(1000)) for _ in range(4)]
    for s in subs:
        s.Subscribe(bus)
    body = _json.dumps({f"m{i}": i / 4 for i in range(200)})
    before = bus._bus.stats()["batches"]
    assert ingest.post_metric(bus, body) == (None, 200)
    bus.Flush()
    assert bus._bus.stats()["batches"] - before == 1
    want = [Event(events.Metric, f"m{i}|{ingest.go_sprint_v(i / 4)}") for i in range(200)]
    for s in subs:
        assert s.Received() == want
        s.Unsubscribe()
    bus.close()


# ---- watches/watches.go:65-101 restated as an actor on the mirror: a Watch keeps a PRIVATE channel that is not a bus
#      subscriber (watches.go:37), hands it to NewEventTimer (watches.go:71) and publishes Status* events on change ----
class Watch(events.Publisher):
    __test__ = False

    def __init__(self, name, poll_ns, backend):
        super().__init__()
        self.Name, self.poll_ns, self.backend = "watch." + name, poll_ns, backend
        self.rx = events.Chan(1000)                  # watches.go:39 — never passed to bus.Subscribe
        self.done = False

    def Run(self, pctx, bus):                        # watches.go:65-96
        self.Register(bus)
        self.ctx, self.cancel = events.WithCancel()
        self.timerSource = self.Name + ".poll"
        events.NewEventTimer(self.ctx, self.rx, self.poll_ns, self.timerSource)

    def Receive(self, event):                        # watches.go:99-101: `watch.rx <- event`
        self.rx.send(event)

    def pump(self):
        """the goroutine body of watches.go:73-95, run on demand (one pass over what the channel holds)"""
        for event in self.rx.recv_all():
            if self.done:
                break
            if event == events.QuitByTest:
                self.cancel(); self.Unregister(); self.done = True
                break
            if event == Event(events.TimerExpired, self.timerSource):
                changed, healthy = self.backend.check()
                if changed:
                    self.Publish(Event(events.StatusChanged, self.Name))
                    self.Publish(Event(events.StatusHealthy if healthy else events.StatusUnhealthy, self.Name))


class NoopDiscoveryBackend:                          # tests/mocks/discovery.go:6-22
    def __init__(self, val):
        self.Val, self.lastVal = val, False

    def check(self):
        changed = self.lastVal != self.Val
        self.lastVal = self.Val
        return changed, self.Val


def _run_watch_test(name, val):                      # watches/watches_test.go:41-58
    bus = events.NewEventBus()
    watch = Watch(name, 1_000_000_000, NoopDiscoveryBackend(val))
    watch.Run(None, bus)
    poll = Event(events.TimerExpired, watch.Name + ".poll")
    watch.Receive(poll)
    watch.Receive(poll)                              # "Ensure we can run it more than once"
    watch.Receive(events.QuitByTest)
    watch.pump()
    assert bus.Wait() is False
    got = {}
    for e in bus.DebugEvents():
        got[e] = got.get(e, 0) + 1
    bus.close()
    return got


def test_watch_poll_ok():
    """watches/watches_test.go:13-26"""
    got = _run_watch_test("mywatchOk", True)
    assert got.get(Event(events.StatusChanged, "watch.mywatchOk"), 0) == 1
    assert got.get(Event(events.StatusHealthy, "watch.mywatchOk"), 0) == 1


def test_watch_poll_fail():
    """watches/watches_test.go:28-39"""
    got = _run_watch_test("mywatchFail", False)
    assert got.get(Event(events.StatusChanged, "watch.mywatchFail"), 0) == 0
    assert got.get(Event(events.StatusUnhealthy, "watch.mywatchFail"), 0) == 0


def test_timer_on_a_channel_that_is_not_a_subscriber():
    """events/timer.go:40-71 takes any `chan Event`: the real ticker of a Watch (watches.go:71) fires into its private
    channel, interleaved in order with direct sends; broadcasts never land there; closing the channel ends the timer
    (timer.go:50-54: the goroutine recovers from the send on a closed channel and exits)."""
    bus = events.NewEventBus()
    other = TestSubscriber(); other.Run(bus)
    rx = events.Chan(1000)
    ctx, cancel = events.WithCancel()
    events.NewEventTimer(ctx, rx, 1000, "w.poll")
    events.NewEventTimeout(ctx, rx, 2500, "w.once")
    bus.Advance(1000)
    rx.send(Event(events.Quit, "direct"))
    bus.Publish(Event(events.Startup, "everyone"))   # a broadcast: must not reach the timer-only channel
    bus.Advance(3000)
    tick, once = Event(events.TimerExpired, "w.poll"), Event(events.TimerExpired, "w.once")
    assert rx.recv_all() == [tick, Event(events.Quit, "direct"), tick, once, tick]
    assert other.Received() == [Event(events.Startup, "everyone")]
    assert bus.Wait.__self__._done == 1              # the implicit mailbox is not in the WaitGroup (only `other` is)
    cancel()
    bus.Advance(5000)
    assert rx.recv_all() == []
    # subscribing the same channel afterwards keeps the mailbox (and opens the mask)
    ctx2, cancel2 = events.WithCancel()
    events.NewEventTimer(ctx2, rx, 1000, "w.again")
    late = events.Subscriber(rx)
    late.Subscribe(bus)
    bus.Advance(6000)
    bus.Publish(Event(events.Signal, "SIGHUP"))
    assert late.Received() == [Event(events.TimerExpired, "w.again"), Event(events.Signal, "SIGHUP")]
    rx2 = events.Chan(10)
    events.NewEventTimer(ctx2, rx2, 1000, "w.closed")
    rx2.close()                                      # timer goroutine would panic on its next send, recover and exit
    bus.Advance(9000)
    assert bus._bus.stats()["n_timers"] == 1         # only "w.again" is still armed
    cancel2()
    late.Unsubscribe(); other.Stop()
    bus.close()


def test_masks_derived_from_the_switches_run_on_the_cuda_bus():
    """N1 on hardware: subscribe with masks.job_mask() / METRIC_MASK through the CUDA bus and check that every event the
    consumer's switch would have handled is still delivered, in order (jobs/jobs.go:195-233, telemetry/metrics.go:97-106)."""
    import numpy as np
    from containerpilot_b200 import masks
    bus = events.NewEventBus(n_max_subs=16)
    sw = masks.JobSwitch("myjob", start_event=Event(events.StatusHealthy, "watch.db"), health_check_name="check.myjob",
                         stopping_wait_event=Event(events.Stopped, "db"), has_stopping_timeout=True)
    job_all, job_masked, job_exact, metric = (events.Subscriber(events.Chan()) for _ in range(4))
    job_all.Subscribe(bus)
    job_masked.Subscribe(bus, sw.mask())
    job_exact.Subscribe(bus, *sw.cases())                  # 17 cases: the one that does not fit widens the mask
    metric.Subscribe(bus, masks.METRIC_MASK)
    rng = np.random.default_rng(3)
    sources = ["myjob", "check.myjob", "myjob.run-every", "myjob.stopping-timeout", "watch.db", "db", "global", "closed",
               "SIGHUP", "SIGUSR2", "other", "m|1"]
    for _ in range(800):
        bus.Publish(Event(int(rng.integers(0, 17)), sources[int(rng.integers(0, len(sources)))]))
    full = job_all.Received()
    handled = [e for e in full if sw.handles(e)]
    assert Event(events.Stopping, "myjob.stopping-timeout") in handled
    assert [e for e in job_masked.Received() if sw.handles(e)] == handled and len(handled) > 0   # nothing the switch handles is lost, order kept
    assert [e for e in job_exact.Received() if sw.handles(e)] == handled
    ms = masks.MetricSwitch()
    assert [e for e in metric.Received() if ms.handles(e)] == [e for e in full if ms.handles(e)]
    job_exact.Unsubscribe()
    for s_ in (job_all, job_masked, metric):
        s_.Unsubscribe()
    bus.close()


def test_plain_c_caller_of_the_c_abi(tmp_path):
    """tests/c/abi_smoke.c — include/cpbus.h from C99, the way cgo-generated code calls it: the jobs_test.go:15-48 sequence, a
    periodic timer, a code mask, DebugEvents, the {code, source} counts; every check is inside the program."""
    import subprocess
    from test_abi import build_c_smoke
    r = subprocess.run([build_c_smoke(tmp_path)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and r.stdout.strip().endswith("PASS"), r.stdout + r.stderr
