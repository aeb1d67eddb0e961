// Exploration: warp-synchronous row blocks (no __syncthreads, 2048 threads/SM) for configs[1].
// nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a scripts/spmv_warp_rows.cu -o /tmp/swr
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA %s at line %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

constexpr int T = 256, WPB = T / 32, WNNZ = 256;
__host__ __device__ constexpr int swz(int e) { return e ^ ((e >> 4) & 7); }

// EPI 0: y = A x.  EPI 1: K2-like epilogue (reads y, lc, uc; writes y'; accumulates dy^2).
template <int EPI, int MINB>
__global__ void __launch_bounds__(T, MINB) k_warp_rows(int n_wb, const int2* __restrict__ wdesc, const int* __restrict__ off,
                                                       const int* __restrict__ idx, const double* __restrict__ val,
                                                       const double* __restrict__ x, const double* __restrict__ yin,
                                                       const double* __restrict__ lc, const double* __restrict__ uc,
                                                       double sigma, double* __restrict__ yout, double* __restrict__ part)
{
  __shared__ double prod[WPB][WNNZ];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  double* pw = prod[w];
  double acc = 0.0;
  for (int wb = blockIdx.x * WPB + w; wb < n_wb; wb += gridDim.x * WPB) {
    const int2 d0 = __ldg(wdesc + wb), d1 = __ldg(wdesc + wb + 1);
    const int r0 = d0.x, lo = d0.y, r1 = d1.x, hi = d1.y;
    const int r = r0 + lane;
    int rs = 0, re = 0;
    double yi = 0, lo_b = 0, hi_b = 0;
    if (r < r1) {
      rs = __ldg(off + r) - lo;
      re = __ldg(off + r + 1) - lo;
      if (EPI == 1) { yi = yin[r]; lo_b = __ldcs(lc + r); hi_b = __ldcs(uc + r); }
    }
    int c[8]; double a[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) { const int e = lo + lane + 32 * k; c[k] = e < hi ? __ldcs(idx + e) : -1; }
#pragma unroll
    for (int k = 0; k < 8; ++k) { const int e = lo + lane + 32 * k; a[k] = e < hi ? __ldcs(val + e) : 0.0; }
#pragma unroll
    for (int k = 0; k < 8; ++k)
      if (c[k] >= 0) pw[swz(lane + 32 * k)] = a[k] * __ldcg(x + c[k]);
    __syncwarp();
    if (r < r1) {
      double s = 0.0;
      // batches of 8 INDEPENDENT shared loads, then the adds in order: one trip through the (gather-congested)
      // LSU queue per batch instead of one per element
      for (int p = rs; p < re; p += 8) {
        double v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = (p + j < re) ? pw[swz(p + j)] : 0.0;
#pragma unroll
        for (int j = 0; j < 8; ++j) s += v[j];
      }
      if (EPI == 0) {
        yout[r] = s;
      } else {
        double next      = yi - sigma * s;
        const double low = next + sigma * lo_b, up = next + sigma * hi_b;
        next             = fmax(low, fmin(up, 0.0));
        yout[r]          = next;
        const double dd  = next - yi;
        acc += dd * dd;
      }
    }
    __syncwarp();
  }
  if (EPI == 1) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) part[blockIdx.x * WPB + w] = acc;
  }
}

template <typename F>
float time_it(F f, int reps)
{
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  for (int i = 0; i < 3; ++i) f();
  CK(cudaDeviceSynchronize());
  cudaEventRecord(a);
  for (int i = 0; i < reps; ++i) f();
  cudaEventRecord(b); cudaEventSynchronize(b);
  CK(cudaGetLastError());
  float ms; cudaEventElapsedTime(&ms, a, b);
  return ms / reps * 1e3f;
}

int main(int argc, char** argv)
{
  const int rows = 1000000, cols = 1000000;
  const bool poisson = argc > 1;  // any argument: Poisson(8) row lengths (the transpose of a uniform matrix)
  std::vector<int> off(rows + 1, 0), idx; std::vector<double> val, x(cols);
  unsigned long long s = 88172645463325252ull;
  auto rnd = [&]() { s ^= s << 13; s ^= s >> 7; s ^= s << 17; return s; };
  if (!poisson) {
    for (int r = 0; r <= rows; ++r) off[r] = r * 8;
  } else {
    std::vector<int> cnt(rows, 0);
    for (size_t i = 0; i < (size_t)rows * 8; ++i) cnt[rnd() % rows]++;
    for (int r = 0; r < rows; ++r) off[r + 1] = off[r] + cnt[r];
  }
  const size_t nnz = off[rows];
  idx.resize(nnz); val.resize(nnz);
  for (size_t i = 0; i < nnz; ++i) { idx[i] = (int)(rnd() % cols); val[i] = (double)(rnd() % 1000) / 500.0 - 1.0; }
  for (int j = 0; j < cols; ++j) x[j] = (double)(rnd() % 1000) / 1000.0;
  // warp blocks: <= 256 nnz and <= 32 rows
  std::vector<int2> wd;
  for (int r = 0; r < rows;) {
    const int lo = off[r]; int r1 = r;
    while (r1 < rows && r1 - r < 32 && off[r1 + 1] - lo <= WNNZ) ++r1;
    if (r1 == r) { printf("long row unsupported in this experiment\n"); return 1; }
    wd.push_back(make_int2(r, lo)); r = r1;
  }
  wd.push_back(make_int2(rows, (int)nnz));
  const int n_wb = (int)wd.size() - 1;
  printf("%s rows: nnz %zu, %d warp blocks (%.1f nnz, %.1f rows per block)\n", poisson ? "Poisson(8)" : "uniform 8", nnz, n_wb,
         (double)nnz / n_wb, (double)rows / n_wb);
  std::vector<double> yref(rows);
  for (int r = 0; r < rows; ++r) { double t = 0; for (int p = off[r]; p < off[r + 1]; ++p) t += val[p] * x[idx[p]]; yref[r] = t; }

  int *doff, *didx[2]; int2* dwd; double *dval[2], *dx, *dy, *dy2, *dlc, *duc, *dpart;
  CK(cudaMalloc(&doff, (rows + 1) * 4)); CK(cudaMalloc(&dwd, wd.size() * 8));
  for (int c = 0; c < 2; ++c) { CK(cudaMalloc(&didx[c], nnz * 4 + 64)); CK(cudaMalloc(&dval[c], nnz * 8 + 64));
    CK(cudaMemcpy(didx[c], idx.data(), nnz * 4, cudaMemcpyHostToDevice)); CK(cudaMemcpy(dval[c], val.data(), nnz * 8, cudaMemcpyHostToDevice)); }
  CK(cudaMalloc(&dx, cols * 8)); CK(cudaMalloc(&dy, rows * 8)); CK(cudaMalloc(&dy2, rows * 8));
  CK(cudaMalloc(&dlc, rows * 8)); CK(cudaMalloc(&duc, rows * 8)); CK(cudaMalloc(&dpart, 1 << 20));
  CK(cudaMemcpy(doff, off.data(), (rows + 1) * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dwd, wd.data(), wd.size() * 8, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dx, x.data(), cols * 8, cudaMemcpyHostToDevice));
  CK(cudaMemset(dy2, 0, rows * 8)); CK(cudaMemset(dlc, 0, rows * 8)); CK(cudaMemset(duc, 0, rows * 8));
  int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  int turn = 0;
  std::vector<double> yy(rows);
  auto check = [&](const char* name) {
    CK(cudaMemcpy(yy.data(), dy, rows * 8, cudaMemcpyDeviceToHost));
    double mx = 0; for (int r = 0; r < rows; ++r) mx = fmax(mx, fabs(yy[r] - yref[r]));
    printf("      %s max |err| vs sequential CPU sum: %.3e\n", name, mx);
  };
  auto run = [&](auto kern, const char* name, bool chk) {
    int per_sm = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, T, 0);
    cudaFuncAttributes fa; cudaFuncGetAttributes(&fa, kern);
    for (int occ = per_sm; occ >= 4; occ -= 2) {
      float us = time_it([&] { kern<<<sms * occ, T>>>(n_wb, dwd, doff, didx[turn & 1], dval[turn & 1], dx, dy2, dlc, duc, 0.5, dy, dpart); ++turn; }, 30);
      printf("  %-34s regs %3d, %d CTA/SM: %6.1f us\n", name, fa.numRegs, occ, us);
    }
    if (chk) check(name);
  };
  run(k_warp_rows<0, 8>, "warp rows y=Ax (minb 8)", true);
  run(k_warp_rows<0, 6>, "warp rows y=Ax (minb 6)", false);
  run(k_warp_rows<1, 8>, "warp rows K2 epilogue (minb 8)", false);
  run(k_warp_rows<1, 6>, "warp rows K2 epilogue (minb 6)", false);
  run(k_warp_rows<1, 4>, "warp rows K2 epilogue (minb 4)", false);
  return 0;
}
