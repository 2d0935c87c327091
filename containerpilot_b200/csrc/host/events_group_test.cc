// events_group_test.cc — the C++ mirror on a group of shards (EventBus with a device list): the same scenarios run on one
// bus and on three shards of GPU 0 must give the same answers, the pump (DrainAll over cpbus_group_drain_ready) included.
// Exit code 0 = all passed.  Needs a GPU (libcpbus has no CPU fallback).
#include <cstdio>
#include <memory>
#include <string>
#include <vector>

#include "events.hpp"

using namespace events;

static int failures = 0;
#define EXPECT(cond)                                                           \
  do {                                                                         \
    if (!(cond)) { std::printf("  FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); failures++; } \
  } while (0)

static const std::vector<int32_t> kOne = {}, kGroup = {0, 0, 0};

// DebugEvents: the last 10 published, oldest first (events/bus.go:34-54), with sends kept out of it
static std::vector<Event> DebugScenario(const std::vector<int32_t>& devices) {
  EventBus bus(devices, EventBus::Clock::Virtual, 8);
  Subscriber a, b;
  a.Rx = MakeChan(100); b.Rx = MakeChan(100);
  a.Subscribe(&bus); b.Subscribe(&bus);
  for (int i = 0; i < 14; i++) {
    bus.Publish(Event{(EventCode)(1 + i % 16), "src" + std::to_string(i)});
    b.Receive(Event{Signal, "direct" + std::to_string(i)});
  }
  std::vector<Event> out = bus.DebugEvents();
  Event e;
  while (a.Rx->Recv(&e)) out.push_back(e);
  while (b.Rx->Recv(&e)) out.push_back(e);
  a.Unsubscribe(); b.Unsubscribe();
  return out;
}

// A Job (jobs/jobs.go:147-231): exact cases, a heartbeat timer and a timeout, while a watcher's small channel fills and the
// publisher blocks until the pump has made room.
static std::vector<Event> JobScenario(const std::vector<int32_t>& devices) {
  EventBus bus(devices, EventBus::Clock::Virtual, 12, 64);
  std::vector<std::unique_ptr<Subscriber>> others;
  for (int i = 0; i < 8; i++) { others.emplace_back(new Subscriber()); others.back()->Rx = MakeChan(1000); others.back()->Subscribe(&bus); }
  Subscriber job;
  job.Rx = MakeChan(1000);
  job.Subscribe(&bus, 1u << Startup, {Event{StatusHealthy, "db"}, Event{Stopped, "db"}});
  Context ctx;
  NewEventTimer(ctx, job.Rx, std::chrono::seconds(1), "job.heartbeat");
  NewEventTimeout(ctx, job.Rx, std::chrono::milliseconds(2500), "job.wait-timeout");
  bus.Publish(GlobalStartup);
  bus.Advance(3'500'000'000ull);
  for (int i = 0; i < 300; i++) {   // more than a mailbox holds: Publish drains into the channels to make room
    bus.Publish(Event{StatusHealthy, i % 3 ? "web" : "db"});
    if (i % 50 == 0) { Event e; while (others[7]->Rx->Recv(&e)) {} }
  }
  bus.Publish(Event{Stopped, "db"});
  ctx.Cancel();
  bus.Advance(9'000'000'000ull);
  std::vector<Event> out;
  Event e;
  while (job.Rx->Recv(&e)) out.push_back(e);
  while (others[3]->Rx->Recv(&e)) out.push_back(e);
  for (const Event& d : bus.DebugEvents()) out.push_back(d);
  job.Unsubscribe();
  for (auto& s : others) s->Unsubscribe();
  return out;
}

// 5,000 subscribers of every event on three shards: each publish makes every mailbox ready, more than one drain call takes,
// so the pump resumes at next_sub across shard boundaries.
static bool FleetScenario(const std::vector<int32_t>& devices) {
  const int N = 5000, E = 5;
  EventBus bus(devices, EventBus::Clock::Virtual, N);
  std::vector<std::unique_ptr<Subscriber>> subs;
  for (int i = 0; i < N; i++) { subs.emplace_back(new Subscriber()); subs.back()->Rx = MakeChan(1000); subs.back()->Subscribe(&bus); }
  std::vector<Event> sent;
  for (int i = 0; i < E; i++) { Event e{(EventCode)(1 + i), "s" + std::to_string(i)}; sent.push_back(e); bus.Publish(e); }
  bool ok = true;
  for (auto& s : subs) {
    std::vector<Event> got;
    Event e;
    while (s->Rx->Recv(&e)) got.push_back(e);
    ok = ok && got == sent;
  }
  for (auto& s : subs) s->Unsubscribe();
  return ok && bus.Wait() == false;
}

int main() {
  std::printf("TestDebugEventsOnAGroup\n");
  const std::vector<Event> d1 = DebugScenario(kOne), dg = DebugScenario(kGroup);
  EXPECT(d1.size() == 10 + 14 + 28);   // ring, a's channel, b's channel (broadcasts + sends)
  EXPECT(d1 == dg);
  std::printf("TestJobOnAGroup\n");
  const std::vector<Event> j1 = JobScenario(kOne), jg = JobScenario(kGroup);
  EXPECT(!j1.empty());
  EXPECT(j1 == jg);
  std::printf("TestFleetOnAGroup\n");
  EXPECT(FleetScenario(kOne));
  EXPECT(FleetScenario(kGroup));
  std::printf(failures ? "FAILED (%d)\n" : "PASS\n", failures);
  return failures ? 1 : 0;
}
