// events_reuse_test.cc — EventBus::ReuseIds (Unsubscribe releases the mailbox, Subscribe takes the lowest free id) on one
// bus.  10^5 Subscribe / Unsubscribe cycles on a bus of 4,096 subscribers, with a publish between cycles: no id runs out, and
// every record published while a subscriber was subscribed reaches its channel exactly once, in order, before its
// Unsubscribe returns.  With the option off the 4,097th Subscribe fails with CPBUS_ENOSPC, as before.  Exit code 0 = all
// passed.  Needs a GPU (libcpbus has no CPU fallback).
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

constexpr uint32_t kSubs = 4096, kMailbox = 64, kLive = 48;
constexpr int kCycles = 100000;

struct Live { std::unique_ptr<Subscriber> sub; int first; };   // first: the first publish it must receive

static void Churn() {
  EventBus bus(EventBus::Clock::Virtual, kSubs, kMailbox);
  bus.ReuseIds(true);
  std::vector<Live> live;
  int published = 0;
  uint32_t max_live = 0;
  bool exact = true;
  auto subscribe = [&] {
    Live l{std::make_unique<Subscriber>(), published};
    l.sub->Rx = MakeChan(4 * kLive);
    l.sub->Subscribe(&bus);
    live.push_back(std::move(l));
  };
  for (uint32_t i = 0; i < kLive; i++) subscribe();
  for (int c = 0; c < kCycles; c++) {
    bus.Publish(Event{StatusChanged, "e" + std::to_string(published++)});
    Live l = std::move(live[c % kLive]);
    l.sub->Unsubscribe();
    Event e;
    int want = l.first;
    while (l.sub->Rx->Recv(&e)) exact &= e.Source == "e" + std::to_string(want++);
    exact &= want == published;
    live[c % kLive] = Live{std::make_unique<Subscriber>(), published};
    live[c % kLive].sub->Rx = MakeChan(4 * kLive);
    live[c % kLive].sub->Subscribe(&bus);
    cpbus_stats_t st{};
    cpbus_stats(bus.handle(), &st);
    max_live = std::max<uint32_t>(max_live, (uint32_t)st.n_subs);
  }
  EXPECT(exact);
  EXPECT(max_live == kLive);
  // lowest free id first: each Subscribe took the id the Unsubscribe before it released, so ids [0, kLive) are all the
  // bus ever handed out
  cpbus_digest_t d{};
  EXPECT(cpbus_digest(bus.handle(), kLive - 1, 1, &d) == CPBUS_OK && cpbus_digest(bus.handle(), kLive, 1, &d) == CPBUS_ENOENT);
  for (Live& l : live) l.sub->Unsubscribe();
}

static void WithoutReuse() {
  EventBus bus(EventBus::Clock::Virtual, kSubs, kMailbox);
  std::vector<std::unique_ptr<Subscriber>> subs;
  bool refused = false;
  for (uint32_t i = 0; i <= kSubs && !refused; i++) {
    subs.push_back(std::make_unique<Subscriber>());
    subs.back()->Rx = MakeChan(4);
    try {
      subs.back()->Subscribe(&bus);
      subs.back()->Unsubscribe();
    } catch (const std::runtime_error& e) {
      refused = std::string(e.what()).find(cpbus_strerror(CPBUS_ENOSPC)) != std::string::npos;
      EXPECT(i == kSubs);
    }
  }
  EXPECT(refused);
}

int main() {
  std::printf("TestReuseIdsChurnOnOneBus\n");
  Churn();
  std::printf("TestWithoutReuseIdsTheIdsRunOut\n");
  WithoutReuse();
  std::printf(failures ? "FAILED (%d)\n" : "PASS\n", failures);
  return failures ? 1 : 0;
}
