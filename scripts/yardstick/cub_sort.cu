// Library yardstick for the sort numbers in DESIGN.md §4: cub::DeviceRadixSort::SortKeys (CCCL shipped with CUDA 12.9, the
// one-sweep implementation) on the same key counts and widths the product's LSD passes handle.  Measurement aid only: the
// product does not link or call it.  Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o cub_sort cub_sort.cu
// Usage: cub_sort <n_keys> <n_columns> <bits: 32|64> [reps]  -> one JSON line (keys/s over all columns, ms per column).
#include <cub/device/device_radix_sort.cuh>
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <vector>

__global__ void fill(uint32_t* p, size_t n_words, uint32_t seed) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x, s = gridDim.x * (size_t)blockDim.x;
  for (; i < n_words; i += s) {
    uint64_t z = (i + 1) * 0x9E3779B97F4A7C15ull + seed;      // splitmix64
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    p[i] = (uint32_t)(z ^ (z >> 31));
  }
}

template <typename K> static int run(size_t n, int cols, int reps) {
  K *in, *out; void* tmp = nullptr; size_t tmp_bytes = 0;
  if (cudaMalloc(&in, n * sizeof(K) * cols) != cudaSuccess || cudaMalloc(&out, n * sizeof(K)) != cudaSuccess) { fprintf(stderr, "alloc failed\n"); return 1; }
  fill<<<132 * 8, 256>>>((uint32_t*)in, n * cols * (sizeof(K) / 4), 7u);
  cub::DeviceRadixSort::SortKeys(nullptr, tmp_bytes, in, out, n);
  cudaMalloc(&tmp, tmp_bytes);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  std::vector<float> ms;
  for (int r = 0; r < reps + 2; ++r) {                          // two warm-up rounds; every column is a fresh input > L2 apart
    cudaEventRecord(e0);
    for (int c = 0; c < cols; ++c) cub::DeviceRadixSort::SortKeys(tmp, tmp_bytes, in + (size_t)c * n, out, n);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float t; cudaEventElapsedTime(&t, e0, e1); if (r >= 2) ms.push_back(t);
  }
  if (cudaGetLastError() != cudaSuccess) { fprintf(stderr, "cuda error\n"); return 1; }
  float best = ms[0], sum = 0; for (float t : ms) { sum += t; if (t < best) best = t; }
  double mean = sum / ms.size();
  printf("{\"library\": \"cub::DeviceRadixSort::SortKeys\", \"cub_version\": %d, \"key_bits\": %d, \"n_keys\": %zu, \"columns\": %d, \"reps\": %d, "
         "\"ms_all_columns_mean\": %.4f, \"ms_all_columns_min\": %.4f, \"ms_per_column\": %.5f, \"gkeys_per_s\": %.3f}\n",
         CUB_VERSION, (int)sizeof(K) * 8, n, cols, reps, mean, best, mean / cols, (double)n * cols / mean / 1e6);
  return 0;
}

int main(int argc, char** argv) {
  if (argc < 4) { fprintf(stderr, "usage: cub_sort n_keys n_columns bits [reps]\n"); return 2; }
  size_t n = strtoull(argv[1], 0, 10); int cols = atoi(argv[2]), bits = atoi(argv[3]), reps = argc > 4 ? atoi(argv[4]) : 5;
  return bits == 64 ? run<uint64_t>(n, cols, reps) : run<uint32_t>(n, cols, reps);
}
