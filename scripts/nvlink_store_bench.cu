// NVLink peer-store microbenchmark (measurement tool, not the product): how fast can SM-issued stores / the copy engines
// move a vector slice into a peer GPU's memory?  One process, all visible devices; every device stores into the NEXT one
// at the same time (the bidirectional pattern of the sharded PDHG attempt).
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a scripts/nvlink_store_bench.cu -o scripts/_bin/nvlink_store_bench
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <vector>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { std::printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); std::exit(1); } } while (0)

__global__ void k_store8(const double* __restrict__ src, double* __restrict__ dst, size_t n)
{
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) dst[i] = src[i] * 2.0;
}
__global__ void k_store16(const double2* __restrict__ src, double2* __restrict__ dst, size_t n2)
{
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += stride) {
    double2 v = src[i];
    v.x *= 2.0; v.y *= 2.0;
    dst[i] = v;
  }
}
// K1-like: 5 reads + 2 local writes per element, plus the remote store (what k_primal_step_bcast does)
__global__ void k_primal_like(const double* __restrict__ a, const double* __restrict__ b, const double* __restrict__ c,
                              const double* __restrict__ d, const double* __restrict__ e, double* __restrict__ o1,
                              double* __restrict__ o2, double* __restrict__ remote, size_t n)
{
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const double v = a[i] - 0.5 * (b[i] - c[i]);
    const double w = fmax(fmin(v, e[i]), d[i]);
    o1[i] = w;
    o2[i] = w - a[i] + w;
    if (remote) remote[i] = w - a[i] + w;
  }
}

int main(int argc, char** argv)
{
  int nd = 0;
  CK(cudaGetDeviceCount(&nd));
  int sms = 0;  // grids are multiples of the SM count
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  if (nd < 2) { std::printf("needs >= 2 devices\n"); return 0; }
  const size_t n = argc > 1 ? std::strtoull(argv[1], nullptr, 10) : 5000000;  // doubles per transfer
  std::vector<double*> src(nd), dst(nd), aux(nd);
  std::vector<cudaStream_t> st(nd);
  std::vector<cudaEvent_t> e0(nd), e1(nd);
  for (int d = 0; d < nd; ++d) {
    CK(cudaSetDevice(d));
    for (int p = 0; p < nd; ++p)
      if (p != d) { int ok = 0; cudaDeviceCanAccessPeer(&ok, d, p); if (ok) cudaDeviceEnablePeerAccess(p, 0); }
    cudaGetLastError();
    CK(cudaMalloc(&src[d], n * 8)); CK(cudaMalloc(&dst[d], n * 8)); CK(cudaMalloc(&aux[d], 7 * n * 8));
    CK(cudaMemset(src[d], 0, n * 8)); CK(cudaMemset(aux[d], 0, 7 * n * 8));
    CK(cudaStreamCreate(&st[d])); CK(cudaEventCreate(&e0[d])); CK(cudaEventCreate(&e1[d]));
  }
  auto run = [&](const char* name, int dirs, auto launch, size_t bytes = 0) {
    if (!bytes) bytes = n * 8;
    for (int rep = 0; rep < 3; ++rep) {
      for (int d = 0; d < dirs; ++d) { CK(cudaSetDevice(d)); CK(cudaEventRecord(e0[d], st[d])); for (int k = 0; k < 10; ++k) launch(d); CK(cudaEventRecord(e1[d], st[d])); }
      for (int d = 0; d < dirs; ++d) { CK(cudaSetDevice(d)); CK(cudaStreamSynchronize(st[d])); }
    }
    float worst = 0.f;
    for (int d = 0; d < dirs; ++d) { float ms = 0.f; CK(cudaEventElapsedTime(&ms, e0[d], e1[d])); worst = ms > worst ? ms : worst; }
    std::printf("%-52s %s  %8.1f us per transfer  %7.1f GB/s per direction\n", name, dirs > 1 ? "all devices at once" : "device 0 only     ",
                1e3 * worst / 10, bytes / (worst / 10 * 1e-3) / 1e9);
  };
  std::printf("%d devices, %zu doubles (%.1f MB) per transfer\n", nd, n, n * 8 / 1e6);
  for (int dirs : {1, nd}) {
    for (int grid : {sms * 4, sms * 8, sms * 16}) {
      char nm[128];
      std::snprintf(nm, sizeof nm, "SM stores  8 B/thread, grid %4d x 256", grid);
      run(nm, dirs, [&](int d) { k_store8<<<grid, 256, 0, st[d]>>>(src[d], dst[(d + 1) % nd], n); });
      std::snprintf(nm, sizeof nm, "SM stores 16 B/thread, grid %4d x 256", grid);
      run(nm, dirs, [&](int d) { k_store16<<<grid, 256, 0, st[d]>>>((const double2*)src[d], (double2*)dst[(d + 1) % nd], n / 2); });
    }
    run("copy engine (cudaMemcpyPeerAsync)", dirs, [&](int d) { CK(cudaMemcpyPeerAsync(dst[(d + 1) % nd], (d + 1) % nd, src[d], d, n * 8, st[d])); });
    run("local only: primal-like kernel, no remote store", dirs, [&](int d) {
      double* a = aux[d];
      k_primal_like<<<sms * 8, 256, 0, st[d]>>>(a, a + n, a + 2 * n, a + 3 * n, a + 4 * n, a + 5 * n, a + 6 * n, nullptr, n); });
    run("primal-like kernel + remote store of xbar", dirs, [&](int d) {
      double* a = aux[d];
      k_primal_like<<<sms * 8, 256, 0, st[d]>>>(a, a + n, a + 2 * n, a + 3 * n, a + 4 * n, a + 5 * n, a + 6 * n, dst[(d + 1) % nd], n); });
  }
  // fan-out: device 0 stores the same slice into EVERY other device (the all-gather pattern at nd ranks), everyone at once
  if (nd > 2) {
    std::printf("fan-out: every device stores its slice into all %d peers (egress = %d x slice)\n", nd - 1, nd - 1);
    const size_t ns = n / nd;
    run("SM stores 8 B/thread to all peers (GB/s = egress of one device)", nd, [&](int d) {
      for (int p = 1; p < nd; ++p) k_store8<<<sms * 2, 256, 0, st[d]>>>(src[d], dst[(d + p) % nd] + (size_t)d * ns, ns); }, ns * 8 * (nd - 1));
  }
  return 0;
}
