// pcie_probe.cu -- what the host link gives this GPU, to choose the host-buffer pipeline (DESIGN.md section 6):
// SM loads/stores on mapped pinned memory (the zero-copy path) vs copy-engine DMA (the staged path), each
// direction alone and both at once.  nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/pcie_probe tools/pcie_probe.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } } while (0)

__global__ void __launch_bounds__(256) k_copy(uint4 *__restrict__ dst, const uint4 *__restrict__ src, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  for (; i + 3 * stride < n; i += 4 * stride) {
    uint4 a = src[i], b = src[i + stride], c = src[i + 2 * stride], d = src[i + 3 * stride];
    dst[i] = a; dst[i + stride] = b; dst[i + 2 * stride] = c; dst[i + 3 * stride] = d;
  }
  for (; i < n; i += stride) dst[i] = src[i];
}

int main(int argc, char **argv) {
  const size_t bytes = (argc > 1 ? atoll(argv[1]) : 2048ll) << 20, n = bytes / 16;
  uint4 *hA, *hB, *dA, *dB;
  CK(cudaHostAlloc(&hA, bytes, cudaHostAllocMapped));
  CK(cudaHostAlloc(&hB, bytes, cudaHostAllocMapped));
  CK(cudaMalloc(&dA, bytes));
  CK(cudaMalloc(&dB, bytes));
  memset(hA, 1, bytes); memset(hB, 2, bytes);
  CK(cudaMemset(dA, 3, bytes)); CK(cudaMemset(dB, 4, bytes));
  cudaStream_t s1, s2;
  CK(cudaStreamCreate(&s1)); CK(cudaStreamCreate(&s2));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  const int grids[] = {sms, sms * 4, sms * 16};
  auto timeit = [&](const char *name, auto fn, double gb_each_way, int ways) {
    fn(); cudaDeviceSynchronize();
    float best = 1e9;
    for (int r = 0; r < 3; r++) {
      cudaEventRecord(e0, 0); fn(); cudaEventRecord(e1, 0); cudaEventSynchronize(e1);   // legacy stream brackets both streams
      float ms; cudaEventElapsedTime(&ms, e0, e1); if (ms < best) best = ms;
    }
    printf("%-44s %8.2f ms  %6.1f GB/s per direction (%d direction%s)\n", name, best, gb_each_way / (best / 1e3), ways, ways > 1 ? "s" : "");
    return 0;
  };
  const double gb = bytes / 1e9;
  for (int g : grids) {
    char nm[96];
    snprintf(nm, sizeof nm, "SM  host->HBM   (grid %d)", g); timeit(nm, [&] { k_copy<<<g, 256, 0, s1>>>(dA, hA, n); }, gb, 1);
    snprintf(nm, sizeof nm, "SM  HBM->host   (grid %d)", g); timeit(nm, [&] { k_copy<<<g, 256, 0, s1>>>(hB, dB, n); }, gb, 1);
    snprintf(nm, sizeof nm, "SM  host->host  (grid %d)", g); timeit(nm, [&] { k_copy<<<g, 256, 0, s1>>>(hB, hA, n); }, gb, 2);
    snprintf(nm, sizeof nm, "SM  up + down, two kernels (grid %d each)", g);
    timeit(nm, [&] { k_copy<<<g, 256, 0, s1>>>(dA, hA, n); k_copy<<<g, 256, 0, s2>>>(hB, dB, n); }, gb, 2);
  }
  timeit("DMA H2D", [&] { cudaMemcpyAsync(dA, hA, bytes, cudaMemcpyHostToDevice, s1); }, gb, 1);
  timeit("DMA D2H", [&] { cudaMemcpyAsync(hB, dB, bytes, cudaMemcpyDeviceToHost, s1); }, gb, 1);
  timeit("DMA H2D + D2H", [&] { cudaMemcpyAsync(dA, hA, bytes, cudaMemcpyHostToDevice, s1); cudaMemcpyAsync(hB, dB, bytes, cudaMemcpyDeviceToHost, s2); }, gb, 2);
  timeit("SM up + DMA down", [&] { k_copy<<<sms * 4, 256, 0, s1>>>(dA, hA, n); cudaMemcpyAsync(hB, dB, bytes, cudaMemcpyDeviceToHost, s2); }, gb, 2);
  timeit("DMA up + SM down", [&] { cudaMemcpyAsync(dA, hA, bytes, cudaMemcpyHostToDevice, s1); k_copy<<<sms * 4, 256, 0, s2>>>(hB, dB, n); }, gb, 2);
  return 0;
}
