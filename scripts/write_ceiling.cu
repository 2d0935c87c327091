// write_ceiling.cu — calibration: what does the GPU sustain for PURE HBM writes, and which
// store flavour / layout / occupancy gets the mailbox-append pattern closest to it?
// (A copy peak counts half reads, half writes.)  sm_90 has no 256-bit store: a "v8" sector is two 16-byte stores.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o write_ceiling write_ceiling.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); return 1; } } while (0)

enum { PLAIN = 0, CS = 1, WT = 2, NOALLOC = 3, EVICT_FIRST = 4 };
template <int F> __device__ __forceinline__ void st_v8(void* dst, uint32_t v, uint64_t pol) {
  if (F == PLAIN) { asm volatile("st.global.v4.b32 [%0], {%1,%1,%1,%1};" ::"l"(dst), "r"(v) : "memory"); asm volatile("st.global.v4.b32 [%0+16], {%1,%1,%1,%1};" ::"l"(dst), "r"(v) : "memory"); }
  if (F == CS) { asm volatile("st.global.cs.v4.b32 [%0], {%1,%1,%1,%1};" ::"l"(dst), "r"(v) : "memory"); asm volatile("st.global.cs.v4.b32 [%0+16], {%1,%1,%1,%1};" ::"l"(dst), "r"(v) : "memory"); }
  if (F == WT) { asm volatile("st.global.wt.v4.b32 [%0], {%1,%1,%1,%1};" ::"l"(dst), "r"(v) : "memory"); asm volatile("st.global.wt.v4.b32 [%0+16], {%1,%1,%1,%1};" ::"l"(dst), "r"(v) : "memory"); }
  if (F == NOALLOC) { asm volatile("st.global.L1::no_allocate.v4.b32 [%0], {%1,%1,%1,%1};" ::"l"(dst), "r"(v) : "memory"); asm volatile("st.global.L1::no_allocate.v4.b32 [%0+16], {%1,%1,%1,%1};" ::"l"(dst), "r"(v) : "memory"); }
  if (F == EVICT_FIRST) { asm volatile("st.global.L2::cache_hint.v4.b32 [%0], {%1,%1,%1,%1}, %2;" ::"l"(dst), "r"(v), "l"(pol) : "memory"); asm volatile("st.global.L2::cache_hint.v4.b32 [%0+16], {%1,%1,%1,%1}, %2;" ::"l"(dst), "r"(v), "l"(pol) : "memory"); }
}
__device__ __forceinline__ void st_v4(void* dst, uint32_t v) {
  asm volatile("st.global.v4.b32 [%0], {%1,%1,%1,%1};" ::"l"(dst), "r"(v) : "memory");
}
__global__ void linear_v4(uint4* p, size_t n16, uint32_t v) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x) st_v4(p + i, v);
}
// chunked: each warp owns one `chunk`-byte region at a time (the mailbox pattern), 32 B per lane per instruction
template <int F>
__global__ void chunked_v8(unsigned char* p, size_t n_chunks, uint32_t chunk, uint32_t stride, uint32_t v) {
  uint64_t pol = 0;
  if (F == EVICT_FIRST) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  const uint32_t lane = threadIdx.x & 31;
  const size_t w = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5, nw = ((size_t)gridDim.x * blockDim.x) >> 5;
  for (size_t c = w; c < n_chunks; c += nw) {
    unsigned char* base = p + c * stride;
    for (uint32_t o = lane * 32; o < chunk; o += 1024) st_v8<F>(base + o, v, pol);
  }
}
// persistent grid + dynamic claiming: each warp takes T chunks at a time from a global counter
__global__ void chunked_dyn(unsigned char* p, size_t n_chunks, uint32_t chunk, uint32_t stride, uint32_t v, unsigned long long* counter, uint32_t T) {
  const uint32_t lane = threadIdx.x & 31;
  for (;;) {
    unsigned long long c0 = 0;
    if (lane == 0) c0 = atomicAdd(counter, (unsigned long long)T);
    c0 = __shfl_sync(0xffffffffu, c0, 0);
    if (c0 >= n_chunks) break;
    for (uint32_t t = 0; t < T && c0 + t < n_chunks; t++) {
      unsigned char* base = p + (c0 + t) * stride;
      for (uint32_t o = lane * 32; o < chunk; o += 1024) st_v8<PLAIN>(base + o, v, 0);
    }
  }
}
// dynamic claiming with the NEXT claim in flight while the current chunks are written
__global__ void chunked_dyn_pf(unsigned char* p, size_t n_chunks, uint32_t chunk, uint32_t stride, uint32_t v, unsigned long long* counter, uint32_t T) {
  const uint32_t lane = threadIdx.x & 31;
  unsigned long long nxt = 0;
  if (lane == 0) nxt = atomicAdd(counter, (unsigned long long)T);
  for (;;) {
    unsigned long long c0 = __shfl_sync(0xffffffffu, nxt, 0);
    if (c0 >= n_chunks) break;
    if (lane == 0) nxt = atomicAdd(counter, (unsigned long long)T);   // result needed only next iteration
    for (uint32_t t = 0; t < T && c0 + t < n_chunks; t++) {
      unsigned char* base = p + (c0 + t) * stride;
      for (uint32_t o = lane * 32; o < chunk; o += 1024) st_v8<PLAIN>(base + o, v, 0);
    }
  }
}
// static persistent, but each warp owns a CONTIGUOUS block of chunks (tests address-order sensitivity)
__global__ void chunked_blocked(unsigned char* p, size_t n_chunks, uint32_t chunk, uint32_t stride, uint32_t v) {
  const uint32_t lane = threadIdx.x & 31;
  const size_t w = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5, nw = ((size_t)gridDim.x * blockDim.x) >> 5;
  const size_t per = (n_chunks + nw - 1) / nw;
  for (size_t c = w * per; c < (w + 1) * per && c < n_chunks; c++) {
    unsigned char* base = p + c * stride;
    for (uint32_t o = lane * 32; o < chunk; o += 1024) st_v8<PLAIN>(base + o, v, 0);
  }
}
// mailbox rings with a per-mailbox PHASE SKEW: mailbox c appends at ring offset (off0 + c*skew) mod 32 KiB (wraps inside
// its ring), and its 1 KiB pieces are written in an order rotated by `rot*c` — de-correlates the low address bits of
// concurrent stores across mailboxes (DRAM bank-level parallelism)
__global__ void chunked_skew(unsigned char* p, size_t n_chunks, uint32_t chunk, uint32_t off0, uint32_t skew, uint32_t rot, uint32_t v) {
  const uint32_t lane = threadIdx.x & 31;
  const size_t w = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5, nw = ((size_t)gridDim.x * blockDim.x) >> 5;
  const uint32_t pieces = chunk / 1024;
  for (size_t c = w; c < n_chunks; c += nw) {
    unsigned char* ring = p + c * 32768;
    const uint32_t start = (off0 + (uint32_t)c * skew) & 32767u;
    for (uint32_t k = 0; k < pieces; k++) {
      const uint32_t piece = (k + rot * (uint32_t)c) % pieces;
      st_v8<PLAIN>(ring + ((start + piece * 1024 + lane * 32) & 32767u), v, 0);
    }
  }
}
// persistent loop that waits for its own stores to drain after every chunk (what CTA exit does implicitly)
template <int FENCE>
__global__ void chunked_fenced(unsigned char* p, size_t n_chunks, uint32_t chunk, uint32_t stride, uint32_t v) {
  const uint32_t lane = threadIdx.x & 31;
  const size_t w = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5, nw = ((size_t)gridDim.x * blockDim.x) >> 5;
  for (size_t c = w; c < n_chunks; c += nw) {
    unsigned char* base = p + c * stride;
    for (uint32_t o = lane * 32; o < chunk; o += 1024) st_v8<PLAIN>(base + o, v, 0);
    if (FENCE == 1) __threadfence_block();
    if (FENCE == 2) __threadfence();
    if (FENCE == 3) asm volatile("fence.acq_rel.cta;" ::: "memory");
  }
}
int main() {
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  const size_t bytes = (size_t)4 << 30;
  unsigned char* d; CK(cudaMalloc(&d, bytes));
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  float ms;
  auto report = [&](const char* name, size_t b, int reps) { printf("%-58s %8.1f GB/s\n", name, b * (double)reps / (ms * 1e-3) / 1e9); };
  for (int it = 0; it < 2; it++) {
    cudaEventRecord(e0); for (int r = 0; r < 10; r++) CK(cudaMemsetAsync(d, r, bytes)); cudaEventRecord(e1); cudaEventSynchronize(e1);
    cudaEventElapsedTime(&ms, e0, e1);
  }
  report("cudaMemset 4 GiB", bytes, 10);
  for (int g : {sms * 4, sms * 8, sms * 16, sms * 64}) {
    cudaEventRecord(e0); for (int r = 0; r < 10; r++) linear_v4<<<g, 256>>>((uint4*)d, bytes / 16, r); cudaEventRecord(e1); cudaEventSynchronize(e1);
    cudaEventElapsedTime(&ms, e0, e1); char nm[64]; snprintf(nm, 64, "linear st.v4 grid=%d", g); report(nm, bytes, 10);
  }
  const size_t n_chunks = 65536;
  auto run = [&](auto kern, const char* flav, uint32_t chunk, uint32_t stride, int g) {
    const size_t b = n_chunks * chunk;
    cudaEventRecord(e0);
    for (int r = 0; r < 40; r++) {
      // mailbox layout: stride 32 KiB, append offset rotates; paged layout: stride == chunk, page base rotates
      unsigned char* base = stride == 32768 ? d + (size_t)(r % (32768 / chunk)) * chunk : d + (size_t)(r % 4) * n_chunks * chunk;
      kern<<<g, 256>>>(base, n_chunks, chunk, stride, r);
    }
    cudaEventRecord(e1); cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
    char nm[96]; snprintf(nm, 96, "chunk=%5u stride=%5u grid=%4d %s", chunk, stride, g, flav); report(nm, b, 40);
  };
  for (uint32_t chunk : {8192u}) for (uint32_t stride : {32768u, chunk}) for (int g : {sms * 3, sms * 4, sms * 8, sms * 16, sms * 32, sms * 64, 8192}) {
    run(chunked_v8<PLAIN>, "plain", chunk, stride, g);
    if (g <= sms * 4) run(chunked_v8<EVICT_FIRST>, "L2::evict_first", chunk, stride, g);
  }
  // fewer threads per CTA, more CTAs (128-thread CTAs)
  for (uint32_t stride : {32768u, 8192u}) for (int g : {sms * 16, sms * 64, 16384}) {
    const size_t b = n_chunks * 8192;
    cudaEventRecord(e0);
    for (int r = 0; r < 40; r++) chunked_v8<PLAIN><<<g, 128>>>(stride == 32768 ? d + (size_t)(r % 4) * 8192 : d + (size_t)(r % 4) * n_chunks * 8192, n_chunks, 8192, stride, r);
    cudaEventRecord(e1); cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
    char nm[96]; snprintf(nm, 96, "chunk= 8192 stride=%5u grid=%5d x128thr plain", stride, g); report(nm, b, 40);
  }
  {
    unsigned long long* ctr; CK(cudaMalloc(&ctr, 8 * 64));
    for (uint32_t stride : {32768u, 8192u}) for (uint32_t T : {1u, 4u, 16u}) for (int g : {sms * 3, sms * 4, sms * 8}) {
      const size_t b = n_chunks * 8192;
      cudaEventRecord(e0);
      for (int r = 0; r < 40; r++) {
        CK(cudaMemsetAsync(ctr, 0, 8));
        chunked_dyn<<<g, 256>>>(stride == 32768 ? d + (size_t)(r % 4) * 8192 : d + (size_t)(r % 4) * n_chunks * 8192, n_chunks, 8192, stride, r, ctr, T);
      }
      cudaEventRecord(e1); cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
      char nm[96]; snprintf(nm, 96, "DYNAMIC chunk=8192 stride=%5u grid=%4d claim=%u", stride, g, T); report(nm, b, 40);
    }
  }
  {
    unsigned long long* ctr; CK(cudaMalloc(&ctr, 8 * 64));
    for (uint32_t T : {2u, 4u, 8u}) for (int g : {sms * 3, sms * 4, sms * 8}) {
      const size_t b = n_chunks * 8192;
      cudaEventRecord(e0);
      for (int r = 0; r < 40; r++) { CK(cudaMemsetAsync(ctr, 0, 8)); chunked_dyn_pf<<<g, 256>>>(d + (size_t)(r % 4) * 8192, n_chunks, 8192, 32768, r, ctr, T); }
      cudaEventRecord(e1); cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
      char nm[96]; snprintf(nm, 96, "DYN+PREFETCH chunk=8192 stride=32768 grid=%4d claim=%u", g, T); report(nm, b, 40);
    }
    for (size_t nch : {(size_t)65536, (size_t)((sms * 3) * 8 * 18), (size_t)((sms * 3) * 8 * 19)}) for (int g : {sms * 3}) {
      const size_t b = nch * 8192;
      cudaEventRecord(e0);
      for (int r = 0; r < 40; r++) chunked_v8<PLAIN><<<g, 256>>>(d + (size_t)(r % 4) * 8192, nch, 8192, 32768, r);
      cudaEventRecord(e1); cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
      char nm[96]; snprintf(nm, 96, "STATIC strided n_chunks=%zu grid=%d", nch, g); report(nm, b, 40);
      cudaEventRecord(e0);
      for (int r = 0; r < 40; r++) chunked_blocked<<<g, 256>>>(d + (size_t)(r % 4) * 8192, nch, 8192, 32768, r);
      cudaEventRecord(e1); cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
      snprintf(nm, 96, "STATIC blocked n_chunks=%zu grid=%d", nch, g); report(nm, b, 40);
    }
  }
  for (int g : {sms * 3, sms * 4, sms * 8}) {
    const size_t b = n_chunks * 8192;
    auto go = [&](auto kern, const char* nm0) {
      cudaEventRecord(e0);
      for (int r = 0; r < 40; r++) kern<<<g, 256>>>(d + (size_t)(r % 4) * 8192, n_chunks, 8192, 32768, r);
      cudaEventRecord(e1); cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
      char nm[96]; snprintf(nm, 96, "FENCED %s grid=%d", nm0, g); report(nm, b, 40);
    };
    go(chunked_fenced<0>, "none          "); go(chunked_fenced<1>, "threadfence_block"); go(chunked_fenced<2>, "threadfence     "); go(chunked_fenced<3>, "fence.acq_rel.cta");
  }
  for (int g : {8192}) for (uint32_t skew : {0u, 8192u, 1024u, 1312u, 32u * 41u}) for (uint32_t rot : {0u, 1u}) {
    const size_t b = n_chunks * 8192;
    cudaEventRecord(e0);
    for (int r = 0; r < 40; r++) chunked_skew<<<g, 256>>>(d, n_chunks, 8192, (r % 4) * 8192, skew, rot, r);
    cudaEventRecord(e1); cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
    char nm[96]; snprintf(nm, 96, "SKEW grid=%4d skew=%5u rot=%u", g, skew, rot); report(nm, b, 40);
  }
  for (uint32_t chunk : {32768u}) for (int g : {sms * 4, sms * 8}) { run(chunked_v8<PLAIN>, "plain", chunk, 32768, g); run(chunked_v8<EVICT_FIRST>, "L2::evict_first", chunk, 32768, g); }
  CK(cudaGetLastError());
  return 0;
}
