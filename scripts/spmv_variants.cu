// Stand-alone exploration of SpMV kernel shapes for configs[1] (1M x 1M, 8 nnz/row, random columns).
// y = A x only (no PDHG epilogue).  Prints microseconds per SpMV for each variant; results feed DESIGN.md.
// nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a scripts/spmv_variants.cu -o /tmp/spmv_variants
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA %s at line %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

constexpr int T = 256;

// ---------------------------------------------------------------- A: products in smem, thread per row (v1 shape)
template <int NNZ, bool CG>
__global__ void __launch_bounds__(T) k_smem_rows(int rows, const int* __restrict__ off, const int* __restrict__ idx,
                                                 const double* __restrict__ val, const double* __restrict__ x,
                                                 double* __restrict__ y, int rows_per_block)
{
  constexpr int K = NNZ / T;
  __shared__ double prod[NNZ + NNZ / 8];
  const int tid = threadIdx.x;
  const int nblocks = (rows + rows_per_block - 1) / rows_per_block;
  for (int b = blockIdx.x; b < nblocks; b += gridDim.x) {
    const int r0 = b * rows_per_block, r1 = min(rows, r0 + rows_per_block);
    const int lo = off[r0], hi = off[r1];
    int c[K]; double a[K];
#pragma unroll
    for (int k = 0; k < K; ++k) { const int e = lo + tid + k * T; c[k] = e < hi ? __ldcs(idx + e) : -1; }
#pragma unroll
    for (int k = 0; k < K; ++k) { const int e = lo + tid + k * T; a[k] = e < hi ? __ldcs(val + e) : 0.0; }
#pragma unroll
    for (int k = 0; k < K; ++k)
      if (c[k] >= 0) { const int p = tid + k * T; prod[p + (p >> 3)] = a[k] * (CG ? __ldcg(x + c[k]) : __ldg(x + c[k])); }
    __syncthreads();
    for (int r = r0 + tid; r < r1; r += T) {
      double s = 0.0;
      for (int p = off[r] - lo; p < off[r + 1] - lo; ++p) s += prod[p + (p >> 3)];
      y[r] = s;
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------- B: cp.async gathers into smem, software pipelined
__device__ __forceinline__ void cp_async8(void* smem, const void* g)
{
  const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(s), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem, const void* g)
{
  const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(s), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async16(void* smem, const void* g)
{
  const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// Stage s holds idx/val of a block (staged with 16-byte cp.async, needs lo % 4 == 0 here: uniform 8 nnz/row) and the
// gathered x entries.  Pipeline depth D blocks: idx/val of block i+2, gathers of block i+1, reduce of block i.
template <int NNZ, int LANES>
__global__ void __launch_bounds__(T) k_async_gather(int rows, const int* __restrict__ off, const int* __restrict__ idx,
                                                    const double* __restrict__ val, const double* __restrict__ x,
                                                    double* __restrict__ y, int rows_per_block)
{
  constexpr int K = NNZ / T;
  constexpr int S = 3;
  extern __shared__ __align__(16) unsigned char raw[];
  int* sidx    = reinterpret_cast<int*>(raw);                         // S x NNZ
  double* sval = reinterpret_cast<double*>(raw + S * NNZ * 4);        // S x NNZ
  double* sxg  = sval + S * NNZ;                                      // S x NNZ
  const int tid = threadIdx.x;
  const int nblocks = (rows + rows_per_block - 1) / rows_per_block;
  const int first = blockIdx.x, step = gridDim.x;
  auto stage_matrix = [&](int b, int s) {  // 16-byte async copies of idx / val (assumes 8 nnz/row alignment)
    if (b < nblocks) {
      const int r0 = b * rows_per_block, r1 = min(rows, r0 + rows_per_block);
      const int lo = off[r0], cnt = off[r1] - lo;
      for (int e = tid * 4; e < cnt; e += T * 4) cp_async16(sidx + s * NNZ + e, idx + lo + e);
      for (int e = tid * 2; e < cnt; e += T * 2) cp_async16(sval + s * NNZ + e, val + lo + e);
    }
    cp_commit();
  };
  auto stage_gathers = [&](int b, int s) {
    if (b < nblocks) {
      const int r0 = b * rows_per_block, r1 = min(rows, r0 + rows_per_block);
      const int cnt = off[r1] - off[r0];
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const int e = tid + k * T;
        if (e < cnt) cp_async8(sxg + s * NNZ + e, x + sidx[s * NNZ + e]);
      }
    }
    cp_commit();
  };
  // prologue
  stage_matrix(first, 0);
  stage_matrix(first + step, 1);
  cp_wait<1>();            // matrix of block 0 landed (this thread's part)
  __syncthreads();
  stage_gathers(first, 0);
  int it = 0;
  for (int b = first; b < nblocks; b += step, ++it) {
    const int s = it % S;
    stage_matrix(b + 2 * step, (it + 2) % S);   // group: matrix(it+2)
    cp_wait<2>();                                // matrix(it+1) landed for this thread   [groups outstanding: gath(it), mat(it+2)]... see note
    __syncthreads();
    stage_gathers(b + step, (it + 1) % S);       // group: gathers(it+1)
    cp_wait<2>();                                // gathers(it) landed for this thread
    __syncthreads();
    // reduce block `it`: LANES lanes per row, tree order
    const int r0 = b * rows_per_block, r1 = min(rows, r0 + rows_per_block);
    const int lo = off[r0];
    const int lane = tid % LANES, grp = tid / LANES;
    for (int r = r0 + grp; r < r1; r += T / LANES) {
      const int rs = off[r] - lo, re = off[r + 1] - lo;
      double s2 = 0.0;
      for (int p = rs + lane; p < re; p += LANES) s2 += sval[s * NNZ + p] * sxg[s * NNZ + p];
#pragma unroll
      for (int o = LANES / 2; o > 0; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
      if (lane == 0) y[r] = s2;
    }
    __syncthreads();
  }
  cp_wait<0>();
}

// ---------------------------------------------------------------- C: register gathers, no smem (rows of exactly 8)
template <bool CG>
__global__ void __launch_bounds__(T) k_row8(int rows, const int* __restrict__ idx, const double* __restrict__ val,
                                            const double* __restrict__ x, double* __restrict__ y)
{
  for (int r = blockIdx.x * T + threadIdx.x; r < rows; r += gridDim.x * T) {
    const int4 c0 = __ldcs(reinterpret_cast<const int4*>(idx + 8 * r));
    const int4 c1 = __ldcs(reinterpret_cast<const int4*>(idx + 8 * r) + 1);
    const double2* v = reinterpret_cast<const double2*>(val + 8 * r);
    const double2 a0 = __ldcs(v), a1 = __ldcs(v + 1), a2 = __ldcs(v + 2), a3 = __ldcs(v + 3);
    const int c[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
    double g[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) g[k] = CG ? __ldcg(x + c[k]) : __ldg(x + c[k]);
    double s = a0.x * g[0];
    s += a0.y * g[1]; s += a1.x * g[2]; s += a1.y * g[3]; s += a2.x * g[4]; s += a2.y * g[5]; s += a3.x * g[6]; s += a3.y * g[7];
    y[r] = s;
  }
}

__global__ void __launch_bounds__(T) k_row8x2(int rows, const int* __restrict__ idx, const double* __restrict__ val,
                                              const double* __restrict__ x, double* __restrict__ y)
{
  const int half = (rows + 1) / 2;
  for (int r = blockIdx.x * T + threadIdx.x; r < half; r += gridDim.x * T) {
    const int r2 = r + half;
    int c[16]; double a[16], g[16];
    const int4* p0 = reinterpret_cast<const int4*>(idx + 8 * (size_t)r);
    const int4* p1 = reinterpret_cast<const int4*>(idx + 8 * (size_t)(r2 < rows ? r2 : r));
    int4 q[4] = {__ldcs(p0), __ldcs(p0 + 1), __ldcs(p1), __ldcs(p1 + 1)};
#pragma unroll
    for (int i = 0; i < 4; ++i) { c[4 * i] = q[i].x; c[4 * i + 1] = q[i].y; c[4 * i + 2] = q[i].z; c[4 * i + 3] = q[i].w; }
#pragma unroll
    for (int k = 0; k < 16; ++k) g[k] = __ldcg(x + c[k]);
    const double2* v0 = reinterpret_cast<const double2*>(val + 8 * (size_t)r);
    const double2* v1 = reinterpret_cast<const double2*>(val + 8 * (size_t)(r2 < rows ? r2 : r));
#pragma unroll
    for (int i = 0; i < 4; ++i) { double2 t = __ldcs(v0 + i); a[2 * i] = t.x; a[2 * i + 1] = t.y; t = __ldcs(v1 + i); a[8 + 2 * i] = t.x; a[8 + 2 * i + 1] = t.y; }
    double s0 = 0, s1 = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) { s0 += a[k] * g[k]; s1 += a[8 + k] * g[8 + k]; }
    y[r] = s0;
    if (r2 < rows) y[r2] = s1;
  }
}
__global__ void __launch_bounds__(T) k_gather_only(int rows, const int* __restrict__ idx, const double* __restrict__ x, double* __restrict__ y)
{
  for (int r = blockIdx.x * T + threadIdx.x; r < rows; r += gridDim.x * T) {
    const int4 c0 = __ldcs(reinterpret_cast<const int4*>(idx + 8 * (size_t)r));
    const int4 c1 = __ldcs(reinterpret_cast<const int4*>(idx + 8 * (size_t)r) + 1);
    const int c[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
    double s = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) s += __ldcg(x + c[k]);
    y[r] = s;
  }
}
// microbench-like: coalesced idx/val, 16 per thread, accumulate per thread, one store per thread (no row structure)
__global__ void __launch_bounds__(T) k_coalesced_regs(size_t n, const int* __restrict__ idx, const double* __restrict__ val,
                                                      const double* __restrict__ x, double* __restrict__ y)
{
  const size_t stride = (size_t)gridDim.x * T;
  double acc = 0;
  size_t i = blockIdx.x * (size_t)T + threadIdx.x;
  for (; i + 15 * stride < n; i += 16 * stride) {
    int c[16]; double a[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) c[u] = __ldcs(idx + i + u * stride);
#pragma unroll
    for (int u = 0; u < 16; ++u) a[u] = __ldcs(val + i + u * stride);
#pragma unroll
    for (int u = 0; u < 16; ++u) acc += a[u] * __ldcg(x + c[u]);
  }
  y[blockIdx.x * T + threadIdx.x] = acc;
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

int main()
{
  const int rows = 1000000, cols = 1000000, k = 8;
  const size_t nnz = (size_t)rows * k;
  std::vector<int> off(rows + 1), idx(nnz); std::vector<double> val(nnz), x(cols);
  unsigned long long s = 88172645463325252ull;
  auto rnd = [&]() { s ^= s << 13; s ^= s >> 7; s ^= s << 17; return s; };
  for (int r = 0; r <= rows; ++r) off[r] = r * k;
  for (size_t i = 0; i < nnz; ++i) { idx[i] = (int)(rnd() % cols); val[i] = (double)(rnd() % 1000) / 500.0 - 1.0; }
  for (int j = 0; j < cols; ++j) x[j] = (double)(rnd() % 1000) / 1000.0;
  // two copies of the matrix, alternated, so that consecutive launches stream from DRAM (2 x 96 MB > L2)
  int *doff, *didx[2]; double *dval[2], *dx, *dy, *dyref;
  CK(cudaMalloc(&doff, (rows + 1) * 4));
  for (int c = 0; c < 2; ++c) { CK(cudaMalloc(&didx[c], nnz * 4 + 64)); CK(cudaMalloc(&dval[c], nnz * 8 + 64));
    CK(cudaMemcpy(didx[c], idx.data(), nnz * 4, cudaMemcpyHostToDevice)); CK(cudaMemcpy(dval[c], val.data(), nnz * 8, cudaMemcpyHostToDevice)); }
  CK(cudaMalloc(&dx, cols * 8)); CK(cudaMalloc(&dy, rows * 8)); CK(cudaMalloc(&dyref, rows * 8));
  CK(cudaMemcpy(doff, off.data(), (rows + 1) * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dx, x.data(), cols * 8, cudaMemcpyHostToDevice));
  int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  int turn = 0;
  std::vector<double> yref(rows), yy(rows);
  k_row8<false><<<sms * 8, T>>>(rows, didx[0], dval[0], dx, dyref);
  CK(cudaMemcpy(yref.data(), dyref, rows * 8, cudaMemcpyDeviceToHost));
  auto check = [&](const char* name) {
    CK(cudaMemcpy(yy.data(), dy, rows * 8, cudaMemcpyDeviceToHost));
    double mx = 0; for (int r = 0; r < rows; ++r) mx = fmax(mx, fabs(yy[r] - yref[r]));
    if (mx > 1e-12) printf("   !! %s max err %.3e\n", name, mx);
  };
  printf("SpMV 1M x 1M, 8 nnz/row: us per y = A x (matrix alternates between two copies)\n");
  for (int occ : {4, 6, 8}) {
    float us = time_it([&] { k_row8<false><<<sms * occ, T>>>(rows, didx[turn & 1], dval[turn & 1], dx, dy); ++turn; }, 30);
    printf("  row8 (thread/row, regs, ldg)   grid %4d : %6.1f us\n", sms * occ, us); check("row8");
    us = time_it([&] { k_row8<true><<<sms * occ, T>>>(rows, didx[turn & 1], dval[turn & 1], dx, dy); ++turn; }, 30);
    printf("  row8 (thread/row, regs, ldcg)  grid %4d : %6.1f us\n", sms * occ, us); check("row8cg");
  }
  {
    int per_sm = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_smem_rows<2048, false>, T, 0);
    float us = time_it([&] { k_smem_rows<2048, false><<<sms * per_sm, T>>>(rows, doff, didx[turn & 1], dval[turn & 1], dx, dy, 256); ++turn; }, 30);
    printf("  smem rows 2048/blk ldg   (%d CTA/SM)       : %6.1f us\n", per_sm, us); check("smem2048");
    us = time_it([&] { k_smem_rows<2048, true><<<sms * per_sm, T>>>(rows, doff, didx[turn & 1], dval[turn & 1], dx, dy, 256); ++turn; }, 30);
    printf("  smem rows 2048/blk ldcg  (%d CTA/SM)       : %6.1f us\n", per_sm, us); check("smem2048cg");
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_smem_rows<1024, false>, T, 0);
    us = time_it([&] { k_smem_rows<1024, false><<<sms * per_sm, T>>>(rows, doff, didx[turn & 1], dval[turn & 1], dx, dy, 128); ++turn; }, 30);
    printf("  smem rows 1024/blk ldg   (%d CTA/SM)       : %6.1f us\n", per_sm, us); check("smem1024");
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_smem_rows<512, false>, T, 0);
    us = time_it([&] { k_smem_rows<512, false><<<sms * per_sm, T>>>(rows, doff, didx[turn & 1], dval[turn & 1], dx, dy, 64); ++turn; }, 30);
    printf("  smem rows 512/blk ldg    (%d CTA/SM)       : %6.1f us\n", per_sm, us); check("smem512");
  }
  {
    int per_sm = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_smem_rows<4096, true>, T, 0);
    float us = time_it([&] { k_smem_rows<4096, true><<<sms * per_sm, T>>>(rows, doff, didx[turn & 1], dval[turn & 1], dx, dy, 512); ++turn; }, 30);
    printf("  smem rows 4096/blk ldcg  (%d CTA/SM)       : %6.1f us\n", per_sm, us); check("smem4096cg");
    for (int occ : {2, 3, 4, 6, 8}) {
      us = time_it([&] { k_smem_rows<2048, true><<<sms * occ, T>>>(rows, doff, didx[turn & 1], dval[turn & 1], dx, dy, 256); ++turn; }, 30);
      printf("  smem rows 2048/blk ldcg  grid %d x SMs      : %6.1f us\n", occ, us);
    }
    for (int occ : {4, 8}) {
      us = time_it([&] { k_row8x2<<<sms * occ, T>>>(rows, didx[turn & 1], dval[turn & 1], dx, dy); ++turn; }, 30);
      printf("  row8x2 (2 rows/thread in flight) grid %d x SMs : %6.1f us\n", occ, us); check("row8x2");
      us = time_it([&] { k_gather_only<<<sms * occ, T>>>(rows, didx[turn & 1], dx, dy); ++turn; }, 30);
      printf("  gather-only row8 (no val)       grid %d x SMs : %6.1f us\n", occ, us);
      us = time_it([&] { k_coalesced_regs<<<sms * occ, T>>>(nnz, didx[turn & 1], dval[turn & 1], dx, dy); ++turn; }, 30);
      printf("  coalesced idx/val + gather, sum in regs (no rows) grid %d x SMs : %6.1f us\n", occ, us);
    }
  }
  return 0;
}
