// events_sparse_test.cc — the C++ mirror's pump (EventBus::DrainAll over cpbus_drain_ready) on fleets of thousands of
// subscribers: one where few mailboxes receive records, one where more mailboxes are ready than one drain call takes.
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

// 6,000 Job-shaped subscribers, each subscribed with the exact case {Quit, "job<i>"}; 40 of them receive records.  Half of
// the channels hold only 2 events, so records wait in `pending_` until the consumer has made room and the pump runs again.
static void TestSparseFleet() {
  std::printf("TestSparseFleet\n");
  const int N = 6000;
  EventBus bus(EventBus::Clock::Virtual, N);
  std::vector<std::unique_ptr<Subscriber>> subs;
  for (int i = 0; i < N; i++) {
    subs.emplace_back(new Subscriber());
    subs.back()->Rx = MakeChan(i % 2 ? 1000 : 2);
    subs.back()->Subscribe(&bus, 0u, {Event{Quit, "job" + std::to_string(i)}});
  }
  std::vector<std::vector<Event>> want(N), got(N);
  std::vector<int> hot;
  for (int k = 0; k < 40; k++) hot.push_back((k * 149 + 7) % N);
  for (int round = 0; round < 3; round++) {
    for (int h : hot) {
      const Event e{Quit, "job" + std::to_string(h)};
      bus.Publish(e);
      want[h].push_back(e);
    }
    const Event direct{Signal, "direct" + std::to_string(round)};   // `job.Rx <- ev`: bypasses the filter
    subs[hot[round]]->Receive(direct);
    want[hot[round]].push_back(direct);
  }
  uint64_t now = 0;
  for (int pass = 0; pass < 8; pass++) {   // consumers take what arrived; each Advance lets the pump move more
    for (int i = 0; i < N; i++) {
      Event e;
      while (subs[i]->Rx->Recv(&e)) got[i].push_back(e);
    }
    bus.Advance(now += 1000);
  }
  bool ok = true;
  for (int i = 0; i < N; i++) ok = ok && got[i] == want[i];
  EXPECT(ok);
  for (auto& s : subs) s->Unsubscribe();
  EXPECT(bus.Wait() == false);
}

// 5,000 subscribers of every event: each publish makes every mailbox ready, more than one drain call takes (4,096
// entries), so DrainAll resumes at next_sub.  Every channel gets every event in order.
static void TestMoreReadyThanOneCall() {
  std::printf("TestMoreReadyThanOneCall\n");
  const int N = 5000, E = 5;
  EventBus bus(EventBus::Clock::Virtual, N);
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
  EXPECT(ok);
  for (auto& s : subs) s->Unsubscribe();
  EXPECT(bus.Wait() == false);
}

int main() {
  TestSparseFleet();
  TestMoreReadyThanOneCall();
  std::printf(failures ? "FAILED (%d)\n" : "PASS\n", failures);
  return failures ? 1 : 0;
}
