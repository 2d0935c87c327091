// events_lag_test.cc — the C++ mirror's extensions Blocking() and Lagging() (cpbus_blockers / cpbus_lagging), on one bus
// and on three shards of GPU 0: a heartbeat timer fills its subscriber's 64-record mailbox while nobody pumps it, the clock
// step stalls, and Blocking() names that subscriber (and a timer-only channel's implicit one) while Lagging() reports the
// backlog.  Exit code 0 = all passed.  Needs a GPU (libcpbus has no CPU fallback).
#include <cstdio>
#include <stdexcept>
#include <vector>

#include "events.hpp"

using namespace events;

static int failures = 0;
#define EXPECT(cond)                                                           \
  do {                                                                         \
    if (!(cond)) { std::printf("  FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); failures++; } \
  } while (0)

static void Scenario(const std::vector<int32_t>& devices) {
  Context ctx;
  EventBus bus(devices, EventBus::Clock::Virtual, 8, 64);
  Subscriber quiet, busy;
  quiet.Rx = MakeChan(1000); busy.Rx = MakeChan(1000);
  quiet.Subscribe(&bus); busy.Subscribe(&bus);
  EXPECT(bus.Blocking().empty());
  EXPECT(bus.Lagging().empty());
  bus.Publish(Event{StatusHealthy, "web"});            // pumped into both channels at once
  EXPECT(bus.Lagging(0).size() == 2);
  ChanPtr watch = MakeChan(1000);                      // a Watch's private channel: an implicit timer-only mailbox
  NewEventTimer(ctx, busy.Rx, std::chrono::milliseconds(1), "busy.heartbeat");
  NewEventTimer(ctx, watch, std::chrono::milliseconds(1), "watch.poll");
  bool stalled = false;
  try {
    bus.Advance(1'000'000'000ull);                     // 1,000 ticks each: far more than a mailbox holds between pumps
  } catch (const std::runtime_error&) {
    stalled = true;                                    // the clock step stopped at a full mailbox (CPBUS_EAGAIN)
  }
  EXPECT(stalled);
  const std::vector<Subscriber*> blocking = bus.Blocking();
  EXPECT(blocking.size() == 2);
  EXPECT(!blocking.empty() && blocking[0] == &busy);
  EXPECT(blocking.size() == 2 && blocking[1]->Rx == watch);
  const std::vector<EventBus::Lag> lag = bus.Lagging();
  EXPECT(lag.size() == 2);
  EXPECT(!lag.empty() && lag[0].sub == &busy && lag[0].backlog == 64 && lag[0].lost == 0);
  EXPECT(lag.size() == 2 && lag[1].sub->Rx == watch && lag[1].backlog == 64);
  EXPECT(bus.Lagging(0).size() == 3);                  // quiet holds nothing: listed only with min_backlog 0
  EXPECT(bus.Blocking().size() == 2);                  // the queries changed nothing
}

int main() {
  std::printf("TestBlockingAndLaggingOnOneBus\n");
  Scenario({});
  std::printf("TestBlockingAndLaggingOnAGroup\n");
  Scenario({0, 0, 0});
  std::printf(failures ? "FAILED (%d)\n" : "PASS\n", failures);
  return failures ? 1 : 0;
}
