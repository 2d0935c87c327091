// events_bulk_test.cc — EventBus::UnsubscribeMany (cpbus_unsubscribe_many) on one bus and on three shards of GPU 0: what
// was published before reaches every listed subscriber's channel, what is published after reaches only the others, and
// the subscriber table forgets exactly the listed ones (a never-subscribed entry is skipped).  Exit code 0 =
// all passed.  Needs a GPU (libcpbus has no CPU fallback).
#include <cstdio>
#include <vector>

#include "events.hpp"

using namespace events;

static int failures = 0;
#define EXPECT(cond)                                                           \
  do {                                                                         \
    if (!(cond)) { std::printf("  FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); failures++; } \
  } while (0)

static size_t Count(const ChanPtr& rx) {
  size_t n = 0;
  Event e;
  while (rx->Recv(&e)) n++;
  return n;
}

static void Scenario(const std::vector<int32_t>& devices) {
  EventBus bus(devices, EventBus::Clock::Virtual, 16, 64);
  std::vector<Subscriber> subs(6);
  for (Subscriber& s : subs) { s.Rx = MakeChan(1000); s.Subscribe(&bus); }
  Subscriber never;                                     // not subscribed: skipped by the bus call
  never.Rx = MakeChan(1000);
  bus.Register(nullptr);                                // one extra WaitGroup count for `never`
  bus.Publish(Event{StatusHealthy, "web"});
  bus.UnsubscribeMany({&subs[1], &subs[4], &subs[2], &never});
  for (size_t i = 0; i < subs.size(); i++) EXPECT(Count(subs[i].Rx) == 1);   // published before: delivered to all
  bus.Publish(Event{StatusUnhealthy, "web"});
  for (size_t i = 0; i < subs.size(); i++) {
    const bool gone = i == 1 || i == 2 || i == 4;
    EXPECT(Count(subs[i].Rx) == (gone ? 0u : 1u));
  }
  for (size_t i : {0u, 3u, 5u}) subs[i].Unsubscribe();
}

int main() {
  std::printf("TestUnsubscribeManyOnOneBus\n");
  Scenario({});
  std::printf("TestUnsubscribeManyOnAGroup\n");
  Scenario({0, 0, 0});
  std::printf(failures ? "FAILED (%d)\n" : "PASS\n", failures);
  return failures ? 1 : 0;
}
