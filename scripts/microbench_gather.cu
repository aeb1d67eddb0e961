// Micro-benchmarks that bound the SpMV design on the GPU:
//   1. streaming read of a 96 MB + 64 MB (idx,val) pair        -> achievable HBM rate for the matrix stream
//   2. random 8-byte gathers from an 8 MB / 80 MB fp64 vector   -> L2 / HBM sector-gather rate (32 B per gather)
//   3. stream + gather together (the SpMV access pattern without any reduction)
// nvcc -O3 -gencode arch=compute_90a,code=sm_90a scripts/microbench_gather.cu -o microbench_gather
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

__global__ void k_stream(const int* __restrict__ idx, const double* __restrict__ val, size_t n, double* out)
{
  double acc = 0.0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    acc += __ldcs(val + i) * (double)__ldcs(idx + i);
  if (acc == 1.2345e-300) *out = acc;
}

template <int UNROLL>
__global__ void k_gather(const int* __restrict__ idx, const double* __restrict__ x, size_t n, double* out)
{
  double acc = 0.0;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  for (; i + (UNROLL - 1) * stride < n; i += UNROLL * stride) {
    int c[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) c[u] = __ldcs(idx + i + u * stride);
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) acc += __ldg(x + c[u]);
  }
  if (acc == 1.2345e-300) *out = acc;
}

template <int UNROLL>
__global__ void k_stream_gather(const int* __restrict__ idx, const double* __restrict__ val, const double* __restrict__ x,
                                size_t n, double* out)
{
  double acc = 0.0;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  for (; i + (UNROLL - 1) * stride < n; i += UNROLL * stride) {
    int c[UNROLL];
    double a[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) c[u] = __ldcs(idx + i + u * stride);
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) a[u] = __ldcs(val + i + u * stride);
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) acc += a[u] * __ldg(x + c[u]);
  }
  if (acc == 1.2345e-300) *out = acc;
}

template <typename F>
float time_it(F f, int reps)
{
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  for (int i = 0; i < 3; ++i) f();
  cudaEventRecord(a);
  for (int i = 0; i < reps; ++i) f();
  cudaEventRecord(b);
  cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b);
  return ms / reps;
}

int main()
{
  const size_t nnz = 8u << 20;  // 8M entries like configs[1]
  int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  for (size_t nvec : {size_t(1) << 20, size_t(10) << 20}) {
    std::vector<int> h(nnz);
    unsigned long long s = 88172645463325252ull;
    for (size_t i = 0; i < nnz; ++i) { s ^= s << 13; s ^= s >> 7; s ^= s << 17; h[i] = (int)(s % nvec); }
    int* idx; double *val, *x, *out;
    // two copies of the streams so that successive launches do not hit in L2 (flush by alternation)
    CK(cudaMalloc(&idx, 4 * nnz * sizeof(int)));
    CK(cudaMalloc(&val, 4 * nnz * sizeof(double)));
    CK(cudaMalloc(&x, nvec * sizeof(double)));
    CK(cudaMalloc(&out, 8));
    for (int c = 0; c < 4; ++c) CK(cudaMemcpy(idx + c * nnz, h.data(), nnz * sizeof(int), cudaMemcpyHostToDevice));
    CK(cudaMemset(val, 0, 4 * nnz * sizeof(double)));
    CK(cudaMemset(x, 0, nvec * sizeof(double)));
    printf("vector of %zu doubles (%.0f MB), %zu gathers per launch\n", nvec, nvec * 8e-6, nnz);
    for (int occ : {4, 8}) {
      const int grid = sms * occ, block = 256;
      int turn = 0;
      float ms = time_it([&] { k_stream<<<grid, block>>>(idx + (turn % 4) * nnz, val + (turn % 4) * nnz, nnz, out); ++turn; }, 40);
      printf("  grid %4d stream            : %7.2f us  %7.1f GB/s (12 B/entry)\n", grid, ms * 1e3, 12.0 * nnz / ms * 1e-6);
      ms = time_it([&] { k_gather<8><<<grid, block>>>(idx + (turn % 4) * nnz, x, nnz, out); ++turn; }, 40);
      printf("  grid %4d gather<8>         : %7.2f us  %7.2f Ggather/s  (%.1f GB/s of 32B sectors)\n", grid, ms * 1e3,
             nnz / ms * 1e-6, 32.0 * nnz / ms * 1e-6);
      ms = time_it([&] { k_gather<16><<<grid, block>>>(idx + (turn % 4) * nnz, x, nnz, out); ++turn; }, 40);
      printf("  grid %4d gather<16>        : %7.2f us  %7.2f Ggather/s\n", grid, ms * 1e3, nnz / ms * 1e-6);
      ms = time_it([&] { k_stream_gather<8><<<grid, block>>>(idx + (turn % 4) * nnz, val + (turn % 4) * nnz, x, nnz, out); ++turn; }, 40);
      printf("  grid %4d stream+gather<8>  : %7.2f us  %7.1f GB/s algorithmic (12 B/entry)\n", grid, ms * 1e3,
             12.0 * nnz / ms * 1e-6);
      ms = time_it([&] { k_stream_gather<16><<<grid, block>>>(idx + (turn % 4) * nnz, val + (turn % 4) * nnz, x, nnz, out); ++turn; }, 40);
      printf("  grid %4d stream+gather<16> : %7.2f us  %7.1f GB/s algorithmic\n", grid, ms * 1e3, 12.0 * nnz / ms * 1e-6);
    }
    cudaFree(idx); cudaFree(val); cudaFree(x); cudaFree(out);
  }
  return 0;
}
