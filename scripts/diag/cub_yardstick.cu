// Diagnostic only (never linked into libmhb): what does the vendor's onesweep radix sort (cub::DeviceRadixSort) do per
// pass on this box for the bench's record count?  Yardstick for k_radix_pass3 (VERDICT r1, "What's weak" 5).
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o cub_yardstick.bin cub_yardstick.cu
//   ./cub_yardstick.bin [n_keys=1230000000]
#include <cub/cub.cuh>
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

__global__ void fill(uint64_t *a, size_t n, uint64_t seed) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    uint64_t x = (i + seed) * 0x9E3779B97F4A7C15ull; x ^= x >> 29; x *= 0xBF58476D1CE4E5B9ull; x ^= x >> 32;
    a[i] = x;
  }
}

template <typename K> static void run(size_t n, int begin_bit, int end_bit, const char *what) {
  K *a, *b;
  CK(cudaMalloc(&a, n * sizeof(K))); CK(cudaMalloc(&b, n * sizeof(K)));
  size_t tb = 0;
  cub::DoubleBuffer<K> db(a, b);
  CK(cub::DeviceRadixSort::SortKeys(nullptr, tb, db, n, begin_bit, end_bit));
  void *tmp; CK(cudaMalloc(&tmp, tb));
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  float best = 1e30f;
  for (int it = 0; it < 4; ++it) {
    fill<<<148 * 8, 256>>>((uint64_t *)a, n * sizeof(K) / 8, 1234 + it);
    db = cub::DoubleBuffer<K>(a, b);
    CK(cudaDeviceSynchronize());
    cudaEventRecord(e0);
    CK(cub::DeviceRadixSort::SortKeys(tmp, tb, db, n, begin_bit, end_bit));
    cudaEventRecord(e1); CK(cudaEventSynchronize(e1));
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    if (it > 0 && ms < best) best = ms;
  }
  int passes = (end_bit - begin_bit + 7) / 8;
  double gb = 2.0 * n * sizeof(K) / 1e9;
  // CUB onesweep = 1 histogram kernel reading the keys once + `passes` onesweep kernels
  printf("{\"what\": \"%s\", \"n\": %zu, \"key_bytes\": %zu, \"bits\": [%d, %d], \"passes\": %d, \"total_ms\": %.3f, "
         "\"ms_per_pass_incl_hist\": %.3f, \"gbs_per_pass_incl_hist\": %.1f, \"temp_bytes\": %zu}\n",
         what, n, sizeof(K), begin_bit, end_bit, passes, best, best / passes, gb / (best / passes * 1e-3), tb);
  cudaFree(a); cudaFree(b); cudaFree(tmp);
}

int main(int argc, char **argv) {
  size_t n = argc > 1 ? (size_t)atof(argv[1]) : 1230000000ull;
  run<uint64_t>(n, 8, 64, "cub SortKeys<u64> bits 8..64 (the count-record sort: 7 digit passes)");
  run<uint64_t>(n, 0, 64, "cub SortKeys<u64> bits 0..64");
  run<uint32_t>(n, 0, 32, "cub SortKeys<u32> bits 0..32");
  return 0;
}
