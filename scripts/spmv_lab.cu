// SpMV laboratory.
//
// Question: what does a row-structured fp64 CSR SpMV with uniformly random columns cost on the GPU at the sizes of
// BASELINE.json's configs[1] / configs[3], and how close can a kernel get to the rowless "stream + gather" ceiling?
// Candidates (all verified against a thread-per-row reference before they are timed):
//   base<RPL>     the round-1 production core (spmv_warp.cuh): coalesced loads, products parked in shared memory,
//                 one lane per row adds its products from shared memory
//   bicsr<CH,..>  "block-interleaved CSR": the matrix is stored per warp block of 32*CH slots so that a coalesced load
//                 hands lane l the CH CONSECUTIVE entries [CH*l, CH*l+CH) of the block; the row-end flag travels in bit 31
//                 of the column index.  Products stay in registers; each lane adds its chunk left to right, partial
//                 sums of rows that cross lanes are chained by shuffles, and only ONE double per row goes through shared
//                 memory (slot of the row's last entry) to reach the lane that runs the row epilogue.
//   gather<U>, stream_gather<U>   rowless ceilings (no reduction at all)
// nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Icuopt_b200/csrc -Iinclude scripts/spmv_lab.cu -o scripts/_bin/spmv_lab
#include "pdlp_kernels.cuh"

// ---- the round-1 core (spmv_warp.cuh of round 1), kept here as the baseline the new format is measured against ----
namespace cuopt_b200 {
constexpr int WARP_THREADS = 256;                // CTA size of the warp-block kernels
constexpr int WARP_PER_CTA = WARP_THREADS / 32;
constexpr int WARP_NNZ     = 256;                // nonzeros per warp block (8 per lane)
constexpr int WARP_KN      = WARP_NNZ / 32;
__host__ __device__ constexpr int warp_swz(int e) { return e ^ ((e >> 4) & 7); }

struct csr_warp_view_t {
  const int* off;
  const int* idx;
  const double* val;
  int n_wb;
  const int2* wdesc;  // n_wb + 1 entries {first row, first nnz}; entry n_wb = {rows, nnz}
};

// Walks this warp's blocks (static round robin over all warps of the grid).
//   pre_op(row)              -> payload P, issued before the matrix loads of the block
//   row_op(row, sum, P)      exactly once per row, by one lane
// `pw` = this warp's WARP_NNZ doubles of shared memory.
// RPL = rows per lane: 1 for the usual blocks of <= 32 rows; 8 for the "wide" schedule (<= 256 rows per block) that the
// host cuts for very sparse matrices (< 4 nonzeros per row: the transposed row shard A_g^T of a many-GPU solve has
// n rows but only nnz/G nonzeros), where blocks of 32 rows would leave 7 of the 8 gather slots of every lane idle.
// INIT: the row sum starts from P::init (a partial sum of the same row over earlier column blocks, see the gather
// blocking in pdlp_kernels.cuh) instead of 0, so that block after block the additions stay strictly left to right.
template <typename P, int RPL = 1, bool INIT = false, typename PreOp, typename RowOp>
__device__ __forceinline__ void spmv_warp_rows(const csr_warp_view_t& A,
                                               const double* __restrict__ x,
                                               double* pw,
                                               PreOp& pre_op,
                                               RowOp& row_op,
                                               unsigned long long gather_policy)
{
  const int lane   = threadIdx.x & 31;
  const int gwarp  = blockIdx.x * WARP_PER_CTA + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * WARP_PER_CTA;
  for (int wb = gwarp; wb < A.n_wb; wb += nwarps) {
    const int2 d0 = __ldg(A.wdesc + wb), d1 = __ldg(A.wdesc + wb + 1);
    const int r0 = d0.x, lo = d0.y, r1 = d1.x, hi = d1.y;
    if (hi - lo > WARP_NNZ) {
      // one long row: lanes stride over it, fixed xor tree at the end
      P pl;
      if (lane == 0) pl = pre_op(r0);
      double acc = 0.0;
      for (int e = lo + lane; e < hi; e += 32) acc += ld_stream(A.val + e) * ld_l2(x + ld_stream(A.idx + e), gather_policy);
      acc = warp_sum(acc);
      if (lane == 0) {
        if constexpr (INIT) acc = pl.init + acc;  // long rows are tree sums anyway
        row_op(r0, acc, pl);
      }
      continue;
    }
    int rs[RPL], re[RPL];
    P pl[RPL];
#pragma unroll
    for (int q = 0; q < RPL; ++q) {
      const int r = r0 + lane + 32 * q;
      rs[q] = re[q] = 0;
      if (r < r1) {
        rs[q] = __ldg(A.off + r) - lo;
        re[q] = __ldg(A.off + r + 1) - lo;
        pl[q] = pre_op(r);
      }
    }
    int c[WARP_KN];
    double a[WARP_KN];
#pragma unroll
    for (int k = 0; k < WARP_KN; ++k) {
      const int e = lo + lane + 32 * k;
      c[k]        = e < hi ? ld_stream(A.idx + e) : -1;
    }
#pragma unroll
    for (int k = 0; k < WARP_KN; ++k) {
      const int e = lo + lane + 32 * k;
      a[k]        = e < hi ? ld_stream(A.val + e) : 0.0;
    }
#pragma unroll
    for (int k = 0; k < WARP_KN; ++k)
      if (c[k] >= 0) pw[warp_swz(lane + 32 * k)] = a[k] * ld_l2(x + c[k], gather_policy);
    __syncwarp();
    if constexpr (RPL == 1) {
      if (r0 + lane < r1) {
        double s = 0.0;
        if constexpr (INIT) s = pl[0].init;
        for (int p = rs[0]; p < re[0]; p += 8) {
          double v[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] = (p + j < re[0]) ? pw[warp_swz(p + j)] : 0.0;
#pragma unroll
          for (int j = 0; j < 8; ++j) s += v[j];
        }
        row_op(r0 + lane, s, pl[0]);
      }
    } else {
#pragma unroll
      for (int q = 0; q < RPL; ++q) {
        const int r = r0 + lane + 32 * q;
        if (r < r1) {
          double s = 0.0;
          if constexpr (INIT) s = pl[q].init;
          for (int p = rs[q]; p < re[q]; ++p) s += pw[warp_swz(p)];
          row_op(r, s, pl[q]);
        }
      }
    }
    __syncwarp();
  }
}

}  // namespace cuopt_b200

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <string>
#include <vector>

using namespace cuopt_b200;

#define CK(x)                                                                      \
  do {                                                                             \
    cudaError_t e = (x);                                                           \
    if (e != cudaSuccess) {                                                        \
      printf("CUDA error %s at line %d\n", cudaGetErrorString(e), __LINE__);       \
      exit(1);                                                                     \
    }                                                                              \
  } while (0)

// ------------------------------------------------------------------------------------------------ host matrices
struct csr_host_t {
  int rows = 0, cols = 0;
  std::vector<int> off, idx;
  std::vector<double> val;
  size_t nnz() const { return idx.size(); }
};

static inline uint64_t splitmix(uint64_t& s)
{
  uint64_t z = (s += 0x9e3779b97f4a7c15ull);
  z          = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z          = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

csr_host_t make_fixed(int rows, int cols, int k, uint64_t seed)
{
  csr_host_t A;
  A.rows = rows;
  A.cols = cols;
  A.off.resize((size_t)rows + 1);
  A.idx.resize((size_t)rows * k);
  A.val.resize((size_t)rows * k);
  for (int r = 0; r <= rows; ++r) A.off[r] = r * k;
#pragma omp parallel for schedule(static)
  for (int r = 0; r < rows; ++r) {
    uint64_t s0 = seed * 0x632be59bd9b4e019ull + (uint64_t)r;  // decorrelate the rows: hash the row number first
    uint64_t s  = splitmix(s0);
    int* c     = A.idx.data() + (size_t)r * k;
    for (int j = 0; j < k; ++j) c[j] = (int)(splitmix(s) % (uint64_t)cols);
    std::sort(c, c + k);
    for (int j = 0; j < k; ++j) A.val[(size_t)r * k + j] = ((double)(splitmix(s) >> 11) / 9007199254740992.0) * 2.0 - 1.0;
  }
  return A;
}

csr_host_t transpose(const csr_host_t& A)
{
  csr_host_t T;
  T.rows = A.cols;
  T.cols = A.rows;
  T.off.assign((size_t)T.rows + 1, 0);
  T.idx.resize(A.nnz());
  T.val.resize(A.nnz());
  for (size_t p = 0; p < A.nnz(); ++p) T.off[A.idx[p] + 1]++;
  for (int r = 0; r < T.rows; ++r) T.off[r + 1] += T.off[r];
  std::vector<int> cur(T.off.begin(), T.off.end() - 1);
  for (int r = 0; r < A.rows; ++r)
    for (int p = A.off[r]; p < A.off[r + 1]; ++p) {
      const int q = cur[A.idx[p]]++;
      T.idx[q]    = r;
      T.val[q]    = A.val[p];
    }
  return T;
}

// entries with column in [c0, c1) (column indices stay global, like the production gather blocks)
csr_host_t column_block(const csr_host_t& A, int c0, int c1)
{
  csr_host_t B;
  B.rows = A.rows;
  B.cols = A.cols;
  B.off.assign((size_t)A.rows + 1, 0);
  for (int r = 0; r < A.rows; ++r) {
    int cnt = 0;
    for (int p = A.off[r]; p < A.off[r + 1]; ++p) cnt += (A.idx[p] >= c0 && A.idx[p] < c1);
    B.off[r + 1] = B.off[r] + cnt;
  }
  B.idx.resize(B.off[A.rows]);
  B.val.resize(B.off[A.rows]);
#pragma omp parallel for schedule(static)
  for (int r = 0; r < A.rows; ++r) {
    int q = B.off[r];
    for (int p = A.off[r]; p < A.off[r + 1]; ++p)
      if (A.idx[p] >= c0 && A.idx[p] < c1) {
        B.idx[q] = A.idx[p];
        B.val[q] = A.val[p];
        ++q;
      }
  }
  return B;
}

// round-1 production schedule: <= 256 nnz and <= max_rows rows per warp block
std::vector<int2> warp_blocks(const std::vector<int>& off, int max_rows)
{
  const int rows = (int)off.size() - 1;
  std::vector<int2> wd;
  int r = 0;
  while (r < rows) {
    const int lo = off[r];
    int r1       = r;
    if (off[r + 1] - lo > WARP_NNZ) r1 = r + 1;
    else
      while (r1 < rows && off[r1 + 1] - lo <= WARP_NNZ && (r1 - r) < max_rows) ++r1;
    wd.push_back(make_int2(r, lo));
    r = r1;
  }
  wd.push_back(make_int2(rows, off[rows]));
  return wd;
}

// Block-interleaved CSR: blocks of whole rows with <= 32*CH entries and <= MAXR rows; block b owns the slots
// [b*32*CH, (b+1)*32*CH); slot k*32 + l holds the block's entry CH*l + k; bit 31 of the index marks the last entry of a row;
// padding slots are {index 0, value 0}.  (Rows longer than 32*CH are not handled in the lab.)
struct bicsr_host_t {
  int n_blk = 0;
  std::vector<int> first_row;  // n_blk + 1
  std::vector<int> idx;
  std::vector<double> val;
};
bicsr_host_t make_bicsr(const csr_host_t& A, int CH, int max_rows)
{
  bicsr_host_t B;
  const int cap = 32 * CH;
  int r         = 0;
  while (r < A.rows) {
    const int lo = A.off[r];
    int r1       = r;
    if (A.off[r + 1] - lo > cap) {
      printf("row longer than a block: not supported in the lab\n");
      exit(1);
    }
    while (r1 < A.rows && A.off[r1 + 1] - lo <= cap && (r1 - r) < max_rows) ++r1;
    B.first_row.push_back(r);
    r = r1;
  }
  B.n_blk = (int)B.first_row.size();
  B.first_row.push_back(A.rows);
  B.idx.assign((size_t)B.n_blk * cap, 0x7fffffff);  // padding slot: no gather at all
  B.val.assign((size_t)B.n_blk * cap, 0.0);
#pragma omp parallel for schedule(static)
  for (int b = 0; b < B.n_blk; ++b) {
    const int r0 = B.first_row[b], r1 = B.first_row[b + 1];
    const int lo = A.off[r0];
    for (int rr = r0; rr < r1; ++rr)
      for (int p = A.off[rr]; p < A.off[rr + 1]; ++p) {
        const int q    = p - lo;
        const size_t s = (size_t)b * cap + (size_t)(q % CH) * 32 + q / CH;
        B.idx[s]       = A.idx[p] | (p == A.off[rr + 1] - 1 ? (int)0x80000000u : 0);
        B.val[s]       = A.val[p];
      }
  }
  return B;
}

// ------------------------------------------------------------------------------------------------ kernels
__global__ void k_reference(int rows, const int* off, const int* idx, const double* val, const double* x, double* y)
{
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int p = off[r]; p < off[r + 1]; ++p) s += val[p] * x[idx[p]];
    y[r] = s;
  }
}

template <int RPL>
__global__ void __launch_bounds__(WARP_THREADS, RPL == 1 ? 6 : 4) k_base(csr_warp_view_t A, const double* __restrict__ x,
                                                                        double* __restrict__ out)
{
  __shared__ double prod[WARP_PER_CTA][WARP_NNZ];
  struct payload_t {};
  auto pre_op = [&](int) { return payload_t{}; };
  auto row_op = [&](int i, double s, const payload_t&) { out[i] = s; };
  spmv_warp_rows<payload_t, RPL>(A, x, prod[threadIdx.x >> 5], pre_op, row_op, make_l2_policies(1).keep);
}

struct lab_bicsr_view_t {
  const int* first_row;
  const int* off;
  const int* idx;
  const double* val;
  int n_blk;
};

// GATHER: 0 = L1::no_allocate + L2 evict-last hint (production), 1 = plain read-only load
template <int GATHER>
__device__ __forceinline__ double lab_gather(const double* p, unsigned long long pol)
{
  if constexpr (GATHER == 0) return ld_l2(p, pol);
  else return __ldg(p);
}

template <int CH, int MINB, bool PREFETCH, int GATHER>
__global__ void __launch_bounds__(256, MINB) k_bicsr(lab_bicsr_view_t A, const double* __restrict__ x, double* __restrict__ out)
{
  __shared__ double rs_all[8][32 * CH];
  double* rsw                  = rs_all[threadIdx.x >> 5];
  const int lane               = threadIdx.x & 31;
  const int gwarp              = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int nwarps             = gridDim.x * 8;
  const unsigned long long pol = make_l2_policies(1).keep;
  constexpr unsigned FULL      = 0xffffffffu;
  int c[CH];
  if (PREFETCH && gwarp < A.n_blk) {
#pragma unroll
    for (int k = 0; k < CH; ++k) c[k] = ld_stream(A.idx + (size_t)gwarp * (32 * CH) + k * 32 + lane);
  }
  for (int b = gwarp; b < A.n_blk; b += nwarps) {
    const size_t base = (size_t)b * (32 * CH) + lane;
    const int r0 = __ldg(A.first_row + b), r1 = __ldg(A.first_row + b + 1);
    if (!PREFETCH) {
#pragma unroll
      for (int k = 0; k < CH; ++k) c[k] = ld_stream(A.idx + base + k * 32);
    }
    double a[CH];
#pragma unroll
    for (int k = 0; k < CH; ++k) a[k] = ld_stream(A.val + base + k * 32);
    double g[CH];
#pragma unroll
    for (int k = 0; k < CH; ++k) {
      const int col = c[k] & 0x7fffffff;
      g[k]          = col != 0x7fffffff ? lab_gather<GATHER>(x + col, pol) : 0.0;
    }
    // rows of the block (first 32 of them; more only when rows are short)
    const int lo = __ldg(A.off + r0);
    int e0 = 0, e1 = 0;
    if (r0 + lane < r1) {
      e0 = __ldg(A.off + r0 + lane);
      e1 = __ldg(A.off + r0 + lane + 1);
    }
    unsigned ends = 0;
#pragma unroll
    for (int k = 0; k < CH; ++k) ends |= (unsigned)(c[k] < 0) << k;
    if (PREFETCH && b + nwarps < A.n_blk) {
#pragma unroll
      for (int k = 0; k < CH; ++k) c[k] = ld_stream(A.idx + (size_t)(b + nwarps) * (32 * CH) + k * 32 + lane);
    }
    // chunk sums, left to right (branch-free: selects and predicated stores); the first row end of the chunk waits
    // for the carry of the previous lanes
    double s = 0.0, head = 0.0;
    const int kf = ends ? __ffs(ends) - 1 : -1;
#pragma unroll
    for (int k = 0; k < CH; ++k) {
      s += a[k] * g[k];
      const bool e = (ends >> k) & 1u;
      if (e && k != kf) rsw[k * 32 + lane] = s;
      head = (k == kf) ? s : head;
      s    = e ? 0.0 : s;
    }
    double T     = s;
    double carry = __shfl_up_sync(FULL, T, 1);
    if (lane == 0) carry = 0.0;
    unsigned pending = __ballot_sync(FULL, kf < 0);
    while (pending) {
      if (kf < 0) T = carry + s;
      carry = __shfl_up_sync(FULL, T, 1);
      if (lane == 0) carry = 0.0;
      pending &= pending << 1;
    }
    if (kf >= 0) rsw[kf * 32 + lane] = carry + head;
    __syncwarp();
    if (r0 + lane < r1) {
      double sum = 0.0;
      if (e1 > e0) {
        const int q = e1 - 1 - lo;
        sum         = rsw[(q % CH) * 32 + q / CH];
      }
      out[r0 + lane] = sum;
    }
    for (int r = r0 + 32 + lane; r < r1; r += 32) {
      const int f0 = __ldg(A.off + r), f1 = __ldg(A.off + r + 1);
      double sum = 0.0;
      if (f1 > f0) {
        const int q = f1 - 1 - lo;
        sum         = rsw[(q % CH) * 32 + q / CH];
      }
      out[r] = sum;
    }
    __syncwarp();
  }
}

// rowless ceilings ---------------------------------------------------------------------------------
template <int U, int GATHER>
__global__ void __launch_bounds__(256) k_gather(const int* __restrict__ idx, const double* __restrict__ x, size_t n, double* out)
{
  double acc                   = 0.0;
  const unsigned long long pol = make_l2_policies(1).keep;
  const size_t stride          = (size_t)gridDim.x * blockDim.x;
  size_t i                     = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  int c[U];
  bool have = i + (U - 1) * stride < n;
  if (have)
#pragma unroll
    for (int u = 0; u < U; ++u) c[u] = __ldcs(idx + i + u * stride);
  while (have) {
    double g[U];
#pragma unroll
    for (int u = 0; u < U; ++u) g[u] = lab_gather<GATHER>(x + (c[u] & 0x7fffffff), pol);
    i += U * stride;
    have = i + (U - 1) * stride < n;
    if (have)
#pragma unroll
      for (int u = 0; u < U; ++u) c[u] = __ldcs(idx + i + u * stride);
#pragma unroll
    for (int u = 0; u < U; ++u) acc += g[u];
  }
  if (acc == 1.2345e-300) *out = acc;
}
template <int U, int GATHER>
__global__ void __launch_bounds__(256) k_stream_gather(const int* __restrict__ idx, const double* __restrict__ val,
                                                        const double* __restrict__ x, size_t n, double* out)
{
  double acc                   = 0.0;
  const unsigned long long pol = make_l2_policies(1).keep;
  const size_t stride          = (size_t)gridDim.x * blockDim.x;
  size_t i                     = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  int c[U];
  bool have = i + (U - 1) * stride < n;
  if (have)
#pragma unroll
    for (int u = 0; u < U; ++u) c[u] = __ldcs(idx + i + u * stride);
  while (have) {
    double a[U], g[U];
#pragma unroll
    for (int u = 0; u < U; ++u) a[u] = __ldcs(val + i + u * stride);
#pragma unroll
    for (int u = 0; u < U; ++u) g[u] = lab_gather<GATHER>(x + (c[u] & 0x7fffffff), pol);
    i += U * stride;
    have = i + (U - 1) * stride < n;
    if (have)
#pragma unroll
      for (int u = 0; u < U; ++u) c[u] = __ldcs(idx + i + u * stride);
#pragma unroll
    for (int u = 0; u < U; ++u) acc += a[u] * g[u];
  }
  if (acc == 1.2345e-300) *out = acc;
}
__global__ void k_flush(double* p, size_t n)
{
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = 1.0;
}
// the same, every line tagged evict-last: what the L2 looks like in the solver, where x-bar and y' (2 x 80 MB at configs[3])
// are stored and gathered with the "keep" policy
__global__ void k_flush_keep(double* p, size_t n)
{
  const unsigned long long keep = make_l2_policies(1).keep;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) st_l2(p + i, 1.0, keep);
}

// ------------------------------------------------------------------------------------------------ harness
template <typename T>
T* to_dev(const std::vector<T>& h, size_t slack = 64)
{
  T* d;
  CK(cudaMalloc(&d, (h.size() + slack) * sizeof(T)));
  CK(cudaMemset(d, 0, (h.size() + slack) * sizeof(T)));
  if (!h.empty()) CK(cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
  return d;
}

// sequential sweep that pulls a vector into L2 (evict-last), see k_l2_warm in pdlp_kernels.cuh
__global__ void k_warm(const double* __restrict__ x, size_t count)
{
  unsigned long long keep;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(keep));
  double a, b, acc = 0.0;
  for (size_t i = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) * 2; i + 1 < count; i += (size_t)gridDim.x * blockDim.x * 2) {
    asm volatile("ld.global.L1::no_allocate.L2::cache_hint.v2.f64 {%0, %1}, [%2], %3;" : "=d"(a), "=d"(b) : "l"(x + i), "l"(keep));
    acc += a + b;
  }
  if (acc == 1.2345e-300) asm volatile("trap;");
}
static int g_mode               = 0;  // 0 hot (back-to-back repetitions), 1 cold (L2 flushed before every repetition), 2 cold, L2 full of stale evict-last lines
static double* g_flush   = nullptr;
static size_t g_flush_n  = 0;
static int g_sms         = 0;
static bool g_need_flush = false;

template <typename F>
double time_us(F launch, int reps = 9)
{
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  std::vector<float> t;
  for (int i = 0; i < reps + 3; ++i) {
    if (g_mode == 2) k_flush_keep<<<g_sms * 8, 256>>>(g_flush, g_flush_n / 2);  // 192 MB of stale evict-last lines
    else if (g_need_flush || g_mode) k_flush<<<g_sms * 8, 256>>>(g_flush, g_flush_n);
    cudaEventRecord(a);
    launch();
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms;
    cudaEventElapsedTime(&ms, a, b);
    if (i >= 3) t.push_back(ms * 1e3f);
  }
  CK(cudaGetLastError());
  cudaEventDestroy(a);
  cudaEventDestroy(b);
  std::sort(t.begin(), t.end());
  return t[t.size() / 2];
}

double check(const double* d_y, const std::vector<double>& ref)
{
  std::vector<double> y(ref.size());
  CK(cudaMemcpy(y.data(), d_y, ref.size() * sizeof(double), cudaMemcpyDeviceToHost));
  double worst = 0.0;
  for (size_t i = 0; i < ref.size(); ++i) {
    const double d = std::fabs(y[i] - ref[i]) / std::max(1.0, std::fabs(ref[i]));
    if (!(d <= worst)) worst = d;  // catches NaN
  }
  return worst;
}

struct case_dev_t {
  int rows, cols;
  size_t nnz;
  int *off, *idx;
  double *val, *x, *y;
  std::vector<double> ref;
};

template <int CH, int MINB, bool PREFETCH, int GATHER>
void run_bicsr(const char* label, const csr_host_t& A, const case_dev_t& d, const bicsr_host_t& B, const int* d_first,
               const int* d_idx, const double* d_val)
{
  int occ = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_bicsr<CH, MINB, PREFETCH, GATHER>, 256, 0));
  cudaFuncAttributes fa;
  CK(cudaFuncGetAttributes(&fa, k_bicsr<CH, MINB, PREFETCH, GATHER>));
  const int grid = std::max(1, std::min((B.n_blk + 7) / 8, g_sms * occ));
  lab_bicsr_view_t v{d_first, d.off, d_idx, d_val, B.n_blk};
  CK(cudaMemset(d.y, 0xff, (size_t)d.rows * sizeof(double)));
  k_bicsr<CH, MINB, PREFETCH, GATHER><<<grid, 256>>>(v, d.x, d.y);
  CK(cudaDeviceSynchronize());
  const double err = check(d.y, d.ref);
  double t[3];
  for (int mode = 0; mode < 3; ++mode) {
    g_mode = mode;
    t[mode] = time_us([&] { k_bicsr<CH, MINB, PREFETCH, GATHER><<<grid, 256>>>(v, d.x, d.y); });
  }
  g_mode = 0;
  const double us = t[0];
  const double bytes = 12.0 * d.nnz + 4.0 * (d.rows + 1) + 8.0 * (d.rows + d.cols);
  printf("  %-34s CH=%2d occ=%d regs=%3d grid=%5d : hot %8.1f us  cold %8.1f  cold(keep-polluted) %8.1f  | hot %6.1f Gnnz/s %6.0f GB/s alg  err %.1e%s\n", label, CH, occ,
         fa.numRegs, grid, us, t[1], t[2], d.nnz / us * 1e-3, bytes / us * 1e-3, err, err <= 1e-12 ? "" : "  WRONG");
  (void)A;
}

void run_case(const char* name, const csr_host_t& A, bool ceilings, int = 0)
{
  printf("== %s: %d x %d, nnz %zu (%.2f per row), gathered vector %.0f MB\n", name, A.rows, A.cols, A.nnz(),
         (double)A.nnz() / A.rows, A.cols * 8e-6);
  case_dev_t d;
  d.rows = A.rows;
  d.cols = A.cols;
  d.nnz  = A.nnz();
  d.off  = to_dev(A.off);
  d.idx  = to_dev(A.idx);
  d.val  = to_dev(A.val);
  std::vector<double> hx(A.cols);
  uint64_t s = 777;
  for (auto& v : hx) v = ((double)(splitmix(s) >> 11) / 9007199254740992.0) * 2.0 - 1.0;
  d.x = to_dev(hx);
  CK(cudaMalloc(&d.y, (size_t)A.rows * sizeof(double)));
  k_reference<<<g_sms * 8, 256>>>(A.rows, d.off, d.idx, d.val, d.x, d.y);
  CK(cudaDeviceSynchronize());
  d.ref.resize(A.rows);
  CK(cudaMemcpy(d.ref.data(), d.y, (size_t)A.rows * sizeof(double), cudaMemcpyDeviceToHost));
  // streams smaller than L2 would be served from it in a timing loop: flush between repetitions
  g_need_flush       = (12.0 * A.nnz() < 400e6);
  const double bytes = 12.0 * d.nnz + 4.0 * (d.rows + 1) + 8.0 * (d.rows + d.cols);

  // ---- round-1 production core
  for (int rpl : {1, 8}) {
    auto wd   = warp_blocks(A.off, 32 * rpl);
    int2* dwd = to_dev(wd);
    csr_warp_view_t v{d.off, d.idx, d.val, (int)wd.size() - 1, dwd};
    int occ = 0;
    if (rpl == 1) CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_base<1>, WARP_THREADS, 0));
    else CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_base<8>, WARP_THREADS, 0));
    const int grid = std::max(1, std::min((v.n_wb + 7) / 8, g_sms * occ));
    CK(cudaMemset(d.y, 0xff, (size_t)d.rows * sizeof(double)));
    auto launch = [&] {
      if (rpl == 1) k_base<1><<<grid, WARP_THREADS>>>(v, d.x, d.y);
      else k_base<8><<<grid, WARP_THREADS>>>(v, d.x, d.y);
    };
    launch();
    CK(cudaDeviceSynchronize());
    const double err = check(d.y, d.ref);
    double t[3];
    for (int mode = 0; mode < 3; ++mode) {
      g_mode  = mode;
      t[mode] = time_us(launch);
    }
    g_mode          = 0;
    const double us = t[0];
    printf("  %-34s RPL=%d occ=%d grid=%5d blocks=%8d : hot %8.1f us  cold %8.1f  cold(keep-polluted) %8.1f  | hot %6.1f Gnnz/s %6.0f GB/s alg  err %.1e%s\n", "base (round-1 core)",
           rpl, occ, grid, v.n_wb, us, t[1], t[2], d.nnz / us * 1e-3, bytes / us * 1e-3, err, err <= 1e-12 ? "" : "  WRONG");
    cudaFree(dwd);
  }
  // ---- the production kernels (pdlp_kernels.cuh) on the production format, built by the production fill kernel
  {
    pdhg_ctl_t hc{};
    hc.active = 1;
    pdhg_ctl_t* dctl;
    CK(cudaMalloc(&dctl, sizeof(hc)));
    CK(cudaMemcpy(dctl, &hc, sizeof(hc), cudaMemcpyHostToDevice));
    std::vector<int2> desc;
    for (int r = 0; r < A.rows;) {
      const int lo = A.off[r];
      int r1       = r;
      while (r1 < A.rows && A.off[r1 + 1] - lo <= BICSR_SLOTS && (r1 - r) < BICSR_MAX_ROWS) ++r1;
      if (r1 == r) { printf("long row: not in the lab\n"); exit(1); }
      desc.push_back(make_int2(r, r1));
      r = r1;
    }
    const int n_std = (int)desc.size();
    int2* d_desc    = to_dev(desc);
    unsigned short* d_slot;
    int* d_bidx;
    double* d_bval;
    CK(cudaMalloc(&d_slot, (size_t)A.rows * 2));
    CK(cudaMalloc(&d_bidx, (size_t)n_std * BICSR_SLOTS * 4));
    CK(cudaMalloc(&d_bval, (size_t)n_std * BICSR_SLOTS * 8));
    k_bicsr_fill<<<g_sms * 8, 256>>>(n_std, d_desc, d.off, d.idx, d.val, d_bidx, d_bval, d_slot);
    CK(cudaDeviceSynchronize());
    bicsr_view_t v{d_desc, d_slot, d_bidx, d_bval, n_std, n_std, d.off, d.idx, d.val};
    int occ = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_spmv, BICSR_THREADS, 0));
    const int grid = std::max(1, std::min((n_std + 7) / 8, g_sms * occ));
    CK(cudaMemset(d.y, 0xff, (size_t)d.rows * sizeof(double)));
    k_spmv<<<grid, BICSR_THREADS>>>(v, d.x, d.y);
    CK(cudaDeviceSynchronize());
    const double err = check(d.y, d.ref);
    for (int which = 0; which < 3; ++which) {
      auto launch = [&] {
        if (which == 0) k_spmv<<<grid, BICSR_THREADS>>>(v, d.x, d.y);
        else k_block_pass<<<grid, BICSR_THREADS>>>(dctl, v, d.x, d.x, 0, d.y, which == 1, nullptr, 0);
      };
      double t[3];
      for (int mode = 0; mode < 3; ++mode) {
        g_mode  = mode;
        t[mode] = time_us(launch);
      }
      g_mode = 0;
      printf("  %-34s occ=%d grid=%5d blocks=%8d : hot %8.1f us  cold %8.1f  cold(keep-polluted) %8.1f  | hot %6.1f Gnnz/s %6.0f GB/s alg  err %.1e%s\n",
             which == 0 ? "PRODUCTION k_spmv (bicsr)" : (which == 1 ? "PRODUCTION k_block_pass first=1" : "PRODUCTION k_block_pass first=0"),
             occ, grid, n_std, t[0], t[1], t[2], d.nnz / t[0] * 1e-3, bytes / t[0] * 1e-3, err, err <= 1e-12 ? "" : "  WRONG");
    }
    cudaFree(d_desc); cudaFree(d_slot); cudaFree(d_bidx); cudaFree(d_bval); cudaFree(dctl);
  }
  // ---- block-interleaved CSR
  for (int CH : {8, 16}) {
    bicsr_host_t B = make_bicsr(A, CH, 256);
    int* d_first   = to_dev(B.first_row);
    int* d_idx     = to_dev(B.idx);
    double* d_val  = to_dev(B.val);
    printf("  bicsr CH=%d: %d blocks, %.2f%% padding\n", CH, B.n_blk, 100.0 * ((double)B.n_blk * 32 * CH / A.nnz() - 1.0));
    if (CH == 8) {
      run_bicsr<8, 4, false, 0>("bicsr hint", A, d, B, d_first, d_idx, d_val);
      run_bicsr<8, 4, true, 0>("bicsr hint +prefetch", A, d, B, d_first, d_idx, d_val);
      run_bicsr<8, 4, false, 1>("bicsr ldg", A, d, B, d_first, d_idx, d_val);
      run_bicsr<8, 4, true, 1>("bicsr ldg +prefetch", A, d, B, d_first, d_idx, d_val);
      run_bicsr<8, 5, true, 0>("bicsr hint +prefetch minb5", A, d, B, d_first, d_idx, d_val);
      run_bicsr<8, 6, false, 0>("bicsr hint minb6", A, d, B, d_first, d_idx, d_val);
    } else {
      run_bicsr<16, 2, true, 0>("bicsr hint +prefetch", A, d, B, d_first, d_idx, d_val);
      run_bicsr<16, 3, false, 0>("bicsr hint minb3", A, d, B, d_first, d_idx, d_val);
    }
    cudaFree(d_first);
    cudaFree(d_idx);
    cudaFree(d_val);
  }
  // ---- rowless ceilings
  if (ceilings) {
    double* out;
    CK(cudaMalloc(&out, 8));
    for (int occ : {4, 8}) {
      const int grid = g_sms * occ;
      double us      = time_us([&] { k_gather<8, 0><<<grid, 256>>>(d.idx, d.x, d.nnz, out); });
      printf("  ceiling gather<8>  hint  grid %4d : %8.1f us  %6.1f Ggather/s\n", grid, us, d.nnz / us * 1e-3);
      us = time_us([&] { k_gather<16, 0><<<grid, 256>>>(d.idx, d.x, d.nnz, out); });
      printf("  ceiling gather<16> hint  grid %4d : %8.1f us  %6.1f Ggather/s\n", grid, us, d.nnz / us * 1e-3);
      us = time_us([&] { k_gather<16, 1><<<grid, 256>>>(d.idx, d.x, d.nnz, out); });
      printf("  ceiling gather<16> ldg   grid %4d : %8.1f us  %6.1f Ggather/s\n", grid, us, d.nnz / us * 1e-3);
      us = time_us([&] { k_stream_gather<8, 0><<<grid, 256>>>(d.idx, d.val, d.x, d.nnz, out); });
      printf("  ceiling stream+gather<8>  grid %4d : %8.1f us  %6.1f Gnnz/s  %6.0f GB/s (12 B/nnz)\n", grid, us, d.nnz / us * 1e-3,
             12.0 * d.nnz / us * 1e-3);
      us = time_us([&] { k_stream_gather<16, 0><<<grid, 256>>>(d.idx, d.val, d.x, d.nnz, out); });
      printf("  ceiling stream+gather<16> grid %4d : %8.1f us  %6.1f Gnnz/s  %6.0f GB/s (12 B/nnz)\n", grid, us, d.nnz / us * 1e-3,
             12.0 * d.nnz / us * 1e-3);
    }
    cudaFree(out);
  }
  cudaFree(d.off);
  cudaFree(d.idx);
  cudaFree(d.val);
  cudaFree(d.x);
  cudaFree(d.y);
  fflush(stdout);
}

int main(int argc, char** argv)
{
  const int big = argc > 1 ? atoi(argv[1]) : 10000000;
  const int sml = argc > 2 ? atoi(argv[2]) : 1000000;
  CK(cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, 0));
  g_flush_n = (size_t)48 << 20;  // 384 MB
  CK(cudaMalloc(&g_flush, g_flush_n * sizeof(double)));
  {
    csr_host_t A = make_fixed(sml, sml, 8, 1);
    run_case("configs[1] A (8 per row)", A, true);
    csr_host_t T = transpose(A);
    run_case("configs[1] A^T (Poisson 8)", T, false);
  }
  if (big > 0) {
    csr_host_t A = make_fixed(big, big, 8, 2);
    run_case("configs[3] A, unblocked", A, true);
    {
      csr_host_t B0 = column_block(A, 0, big / 2);
      run_case("configs[3] A, column block 0 of 2", B0, true, big / 2);
    }
    csr_host_t T = transpose(A);
    A            = csr_host_t{};
    run_case("configs[3] A^T, unblocked", T, false);
    {
      csr_host_t B0 = column_block(T, 0, big / 2);
      run_case("configs[3] A^T, column block 0 of 2", B0, false, big / 2);
    }
  }
  return 0;
}
