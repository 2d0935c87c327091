// The owners of containerpilot_b200/csrc/cuda_owned.hpp, compiled with plain g++ against the CUDA runtime.
//   owned_buffers nodevice   every allocation is refused (run with no visible device)
//   owned_buffers device     on a GPU: floors, regrowth, a refused oversize request, moves
// Prints "ok" and exits 0, or names the first failed check and exits 1.
#include "cuda_owned.hpp"

#include <cstdio>
#include <cstring>
#include <utility>

using namespace cuda_owned;

#define CHECK(c)                                                   \
  do {                                                             \
    if (!(c)) {                                                    \
      std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #c);   \
      return 1;                                                    \
    }                                                              \
  } while (0)

template <class B>
static bool empty(const B& b) { return b.get() == nullptr && b.dev() == nullptr && b.size() == 0; }

// Without a device: every growth and allocation fails and leaves {nullptr, 0}.  (Without a device the runtime keeps its
// initialisation error as the last error for the life of the process, so consuming the error is checked on the device.)
template <class B>
static int refused(B& b) {
  CHECK(b.grow(10, 1024) != cudaSuccess);
  CHECK(empty(b));
  CHECK(b.alloc(16) != cudaSuccess);
  CHECK(empty(b));
  B moved(std::move(b));   // empty owners move and destroy harmlessly
  CHECK(empty(moved) && empty(b));
  b = std::move(moved);
  CHECK(empty(moved) && empty(b));
  return 0;
}

static int nodevice() {
  DeviceBuf<int> d;
  PinnedBuf<double> p;
  MappedBuf<unsigned long long> m;
  if (refused(d) || refused(p) || refused(m)) return 1;
  CudaEvent e;
  CudaStream s;
  CHECK(e.create() != cudaSuccess && (cudaEvent_t)e == nullptr);
  CHECK(s.create() != cudaSuccess && (cudaStream_t)s == nullptr);
  CudaEvent e2(std::move(e));
  CudaStream s2(std::move(s));
  CHECK((cudaEvent_t)e2 == nullptr && (cudaStream_t)s2 == nullptr);
  return 0;
}

static int device() {
  {
    DeviceBuf<int> d;
    CHECK(d.grow(10, 1024) == cudaSuccess && d.size() == 1024 && d.get() != nullptr && d.dev() == d.get());
    int* const p = d.get();
    CHECK(d.grow(1000, 1 << 20) == cudaSuccess && d.get() == p && d.size() == 1024);   // fits: kept, floor unused
    CHECK(d.grow(2000) == cudaSuccess && d.size() == 2000);
    // more than the device holds: an API error return, no kernel involved
    CHECK(d.grow((size_t)1 << 48) == cudaErrorMemoryAllocation);
    CHECK(empty(d));
    CHECK(cudaGetLastError() == cudaSuccess);
    CHECK(d.grow(10) == cudaSuccess && d.size() == 10 && d.get() != nullptr);
    DeviceBuf<unsigned char> big;
    CHECK(big.alloc((size_t)1 << 50) == cudaErrorMemoryAllocation && empty(big));
    CHECK(cudaGetLastError() == cudaSuccess);
  }
  {
    PinnedBuf<int> h;
    CHECK(h.grow(4, 16) == cudaSuccess && h.size() == 16 && h.get() != nullptr);
    for (int i = 0; i < 16; i++) h[i] = i;
    MappedBuf<int> m;
    CHECK(m.alloc(16) == cudaSuccess && m.get() != nullptr && m.dev() != nullptr);
    DeviceBuf<int> d;
    CHECK(d.alloc(16) == cudaSuccess);
    CHECK(cudaMemcpy(d, h, 16 * sizeof(int), cudaMemcpyHostToDevice) == cudaSuccess);
    CHECK(cudaMemcpy(m.dev(), d, 16 * sizeof(int), cudaMemcpyDeviceToDevice) == cudaSuccess);   // through the alias
    CHECK(std::memcmp(m.get(), h.get(), 16 * sizeof(int)) == 0);
  }
  {
    // a move hands the allocation over once: the source is empty, and no pointer is freed twice (a second cudaFree
    // of the same pointer would leave cudaErrorInvalidValue behind)
    DeviceBuf<int> a;
    CHECK(a.alloc(64) == cudaSuccess);
    int* const p = a.get();
    DeviceBuf<int> b(std::move(a));
    CHECK(empty(a) && b.get() == p && b.size() == 64);
    DeviceBuf<int> c;
    CHECK(c.alloc(8) == cudaSuccess);
    c = std::move(b);
    CHECK(empty(b) && c.get() == p && c.size() == 64);
    CudaStream s;
    CudaEvent e;
    CHECK(s.create() == cudaSuccess && e.create() == cudaSuccess);
    CudaStream s2(std::move(s));
    CudaEvent e2;
    e2 = std::move(e);
    CHECK((cudaStream_t)s == nullptr && (cudaEvent_t)e == nullptr);
    CHECK(cudaMemsetAsync(c, 0, 64 * sizeof(int), s2) == cudaSuccess && cudaEventRecord(e2, s2) == cudaSuccess);
    CHECK(cudaEventSynchronize(e2) == cudaSuccess);
  }
  CHECK(cudaGetLastError() == cudaSuccess);
  return 0;
}

int main(int argc, char** argv) {
  const bool dev = argc > 1 && std::strcmp(argv[1], "device") == 0;
  const int rc = dev ? device() : nodevice();
  if (rc == 0) std::printf("ok\n");
  return rc;
}
