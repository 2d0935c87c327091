// events_ack_test.cc — EventBus::AckOnDelivery (the pump over cpbus_take_ready + cpbus_ack_many) on one bus and on three
// shards of GPU 0.  A consumer stops reading and later resumes: the pump never holds more than mailbox_cap records for it;
// once channel capacity + mailbox_cap records wait for it, Blocking() names it and the next Publish blocks until it reads
// again; every record then arrives exactly once, in order.  With the option off the same consumer is buffered without
// bound and nothing blocks.  Exit code 0 = all passed.  Needs a GPU (libcpbus has no CPU fallback).
#include <atomic>
#include <chrono>
#include <cstdio>
#include <string>
#include <thread>
#include <vector>

#include "events.hpp"

using namespace events;

static int failures = 0;
#define EXPECT(cond)                                                           \
  do {                                                                         \
    if (!(cond)) { std::printf("  FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); failures++; } \
  } while (0)

constexpr uint32_t kMailbox = 64;
constexpr size_t kChan = 8;

static std::string Name(int i) { return "e" + std::to_string(i); }

// Stages one record without flushing it (the raw C-ABI): the next flush's unit, which cpbus_blockers evaluates.
static void Stage(EventBus& bus, int i) {
  const std::string s = Name(i);
  cpbus_event ev{};
  ev.code = StatusChanged;
  if (bus.group_handle()) {
    cpbus_group_intern(bus.group_handle(), s.data(), s.size(), &ev.source_id);
    EXPECT(cpbus_group_publish(bus.group_handle(), &ev, 1) == CPBUS_OK);
  } else {
    cpbus_intern(bus.handle(), s.data(), s.size(), &ev.source_id);
    EXPECT(cpbus_publish(bus.handle(), &ev, 1) == CPBUS_OK);
  }
}

static void Acknowledged(const std::vector<int32_t>& devices) {
  EventBus bus(devices, EventBus::Clock::Virtual, 16, kMailbox);
  bus.AckOnDelivery(true);
  Subscriber slow, fast;
  slow.Rx = MakeChan(kChan); slow.Subscribe(&bus);
  fast.Rx = MakeChan(100000); fast.Subscribe(&bus);
  const int queued = (int)(kChan + kMailbox);
  for (int i = 0; i < queued; i++) {
    bus.Publish(Event{StatusChanged, Name(i)});
    EXPECT(bus.Buffered(&slow) <= kMailbox);
  }
  EXPECT(slow.Rx->Len() == kChan && bus.Buffered(&slow) == kMailbox && bus.Buffered(&fast) == 0);
  EXPECT(bus.Blocking().empty());                        // nothing staged: the next flush has nothing to get past
  Stage(bus, queued);
  std::vector<Subscriber*> b = bus.Blocking();
  EXPECT(b.size() == 1 && b[0] == &slow);
  std::atomic<bool> done{false};
  std::thread pub([&] { bus.Publish(Event{StatusChanged, Name(queued + 1)}); done = true; });
  std::this_thread::sleep_for(std::chrono::milliseconds(300));
  EXPECT(!done);                                         // the publisher waits for the stopped consumer
  std::vector<std::string> got;                          // the consumer resumes
  Event e;
  while ((int)got.size() < queued + 2) {
    if (slow.Rx->Recv(&e)) got.push_back(e.Source);
    else if (done) bus.Advance(0);                       // the pump's next pass (a virtual bus pumps on every call)
    else std::this_thread::sleep_for(std::chrono::milliseconds(1));
  }
  pub.join();
  EXPECT(!slow.Rx->Recv(&e));
  bool in_order = true;
  for (int i = 0; i < queued + 2; i++) in_order &= got[i] == Name(i);
  EXPECT(in_order);
  size_t n_fast = 0;
  while (fast.Rx->Recv(&e)) in_order &= e.Source == Name((int)n_fast++);
  EXPECT(n_fast == (size_t)queued + 2 && in_order);
  EXPECT(bus.Buffered(&slow) == 0 && bus.Blocking().empty());
  slow.Unsubscribe(); fast.Unsubscribe();
}

static void Unacknowledged(const std::vector<int32_t>& devices) {
  EventBus bus(devices, EventBus::Clock::Virtual, 16, kMailbox);
  Subscriber slow;
  slow.Rx = MakeChan(kChan); slow.Subscribe(&bus);
  const int n = (int)(kChan + 3 * kMailbox);
  for (int i = 0; i < n; i++) bus.Publish(Event{StatusChanged, Name(i)});   // never blocks
  EXPECT(bus.Buffered(&slow) == (size_t)n - kChan);           // more than a mailbox: the host queue has no bound
  Stage(bus, n);
  EXPECT(bus.Blocking().empty());
  size_t got = 0;
  Event e;
  bool in_order = true;
  while (got < (size_t)n + 1) {
    if (slow.Rx->Recv(&e)) in_order &= e.Source == Name((int)got++);
    else bus.Advance(0);
  }
  EXPECT(in_order);
  slow.Unsubscribe();
}

int main() {
  std::printf("TestAckOnDeliveryOnOneBus\n");
  Acknowledged({});
  std::printf("TestAckOnDeliveryOnAGroup\n");
  Acknowledged({0, 0, 0});
  std::printf("TestWithoutAckTheHostQueueGrowsOnOneBus\n");
  Unacknowledged({});
  std::printf("TestWithoutAckTheHostQueueGrowsOnAGroup\n");
  Unacknowledged({0, 0, 0});
  std::printf(failures ? "FAILED (%d)\n" : "PASS\n", failures);
  return failures ? 1 : 0;
}
