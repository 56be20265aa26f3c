// alloc_probe.cu -- what do the allocation calls of the device-side setup cost on this GPU?
// nvcc -O2 -arch=sm_90a -o alloc_probe alloc_probe.cu ; ./alloc_probe
#include <cuda_runtime.h>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
static double now() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
int main() {
  cudaFree(0);
  cudaStream_t s; cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
  for (size_t gb : {1, 4, 8}) {
    const size_t bytes = gb << 30;
    void* p = nullptr;
    double t0 = now(); cudaMalloc(&p, bytes); double t1 = now(); cudaMemsetAsync(p, 0, bytes, s); cudaStreamSynchronize(s); double t2 = now();
    cudaFree(p); double t3 = now();
    printf("cudaMalloc %zu GB: %.2f ms, first memset %.2f ms, cudaFree %.2f ms\n", gb, t1 - t0, t2 - t1, t3 - t2);
  }
  cudaMemPool_t pool; cudaDeviceGetDefaultMemPool(&pool, 0);
  unsigned long long thr = ~0ULL; cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  for (int rep = 0; rep < 2; ++rep)
    for (size_t gb : {1, 4, 8}) {
      const size_t bytes = gb << 30;
      void* p = nullptr;
      double t0 = now(); cudaMallocAsync(&p, bytes, s); cudaStreamSynchronize(s); double t1 = now();
      cudaMemsetAsync(p, 0, bytes, s); cudaStreamSynchronize(s); double t2 = now();
      cudaFreeAsync(p, s); cudaStreamSynchronize(s); double t3 = now();
      printf("rep %d cudaMallocAsync %zu GB: %.2f ms, memset %.2f ms, cudaFreeAsync %.2f ms\n", rep, gb, t1 - t0, t2 - t1, t3 - t2);
    }
  { double t0 = now(); cudaMemPoolTrimTo(pool, 0); double t1 = now(); printf("trim pool: %.2f ms\n", t1 - t0); }
  // pageable / pinned H2D of 1 GB
  const size_t bytes = (size_t)1 << 30;
  void* d; cudaMalloc(&d, bytes);
  std::vector<char> h(bytes, 1);
  for (int rep = 0; rep < 2; ++rep) { double t0 = now(); cudaMemcpyAsync(d, h.data(), bytes, cudaMemcpyHostToDevice, s); cudaStreamSynchronize(s); double t1 = now();
    printf("pageable H2D 1 GB: %.2f ms (%.1f GB/s)\n", t1 - t0, 1.0737 / ((t1 - t0) * 1e-3)); }
  { double t0 = now(); cudaHostRegister(h.data(), bytes, cudaHostRegisterDefault); double t1 = now();
    cudaMemcpyAsync(d, h.data(), bytes, cudaMemcpyHostToDevice, s); cudaStreamSynchronize(s); double t2 = now();
    cudaHostUnregister(h.data()); double t3 = now();
    printf("cudaHostRegister 1 GB: %.2f ms, pinned H2D %.2f ms (%.1f GB/s), unregister %.2f ms\n", t1 - t0, t2 - t1, 1.0737 / ((t2 - t1) * 1e-3), t3 - t2); }
  { std::vector<char> h2(bytes); double t0 = now(); cudaMemcpyAsync(h2.data(), d, bytes, cudaMemcpyDeviceToHost, s); cudaStreamSynchronize(s); double t1 = now();
    printf("pageable D2H 1 GB: %.2f ms (%.1f GB/s)\n", t1 - t0, 1.0737 / ((t1 - t0) * 1e-3)); }
  // many small cudaMalloc / cudaFree
  { double t0 = now(); std::vector<void*> ps(200); for (auto& q : ps) cudaMalloc(&q, 64 << 20); double t1 = now(); for (auto q : ps) cudaFree(q); double t2 = now();
    printf("200 x cudaMalloc 64 MB: %.2f ms, 200 x cudaFree: %.2f ms\n", t1 - t0, t2 - t1); }
  return 0;
}
