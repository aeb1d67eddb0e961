// Device CSR transpose (setup only, once per solve): A (rows x cols) -> A^T as CSR with row indices ascending inside
// each transposed row — the same ordering cusparseCsr2cscEx2 hands the reference
// (cpp/src/mip/problem/problem.cu:277-309 via raft::sparse::linalg::csr_transpose).
//
// Stable by construction: an LSD radix sort (cub::DeviceRadixSort, stable) of the entry ids by column index keeps
// entries of one column in their original row-major order, so the result is deterministic and identical to a
// sequential counting-sort transpose.  CUB is used here like the reference uses cuSPARSE: a library call in the
// one-time setup, not in the iteration loop.
#include "device_utils.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

namespace cuopt_b200 {

// SM count of the device the calling thread is bound to (a rank of a multi-GPU solve is not on device 0)
static int current_device_sms()
{
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

namespace {

__global__ void k_expand_rows_and_count(int rows, const int* __restrict__ off, const int* __restrict__ idx,
                                        int* __restrict__ entry_row, int* __restrict__ entry_id, int* __restrict__ col_count)
{
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < rows; r += gridDim.x * wpb) {
    for (int p = off[r] + lane; p < off[r + 1]; p += 32) {
      entry_row[p] = r;
      entry_id[p]  = p;
      atomicAdd(col_count + idx[p], 1);  // integer counts: order independent
    }
  }
}

__global__ void k_permute(int nnz, const int* __restrict__ sorted_entry, const int* __restrict__ entry_row,
                          const double* __restrict__ val, int* __restrict__ tidx, double* __restrict__ tval)
{
  const int stride = gridDim.x * blockDim.x;
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < nnz; q += stride) {
    const int e = sorted_entry[q];
    tidx[q]     = entry_row[e];
    tval[q]     = val[e];
  }
}

// ---- column-block split (gather blocking, DESIGN.md §5) ----
constexpr int MAX_COLUMN_BLOCKS = 16;
struct block_ptrs_t {
  int* off[MAX_COLUMN_BLOCKS];
  int* idx[MAX_COLUMN_BLOCKS];
  double* val[MAX_COLUMN_BLOCKS];
};
// counts[b * (rows + 1) + r] = entries of row r whose column lies in block b (slot rows stays 0: scan total)
__global__ void k_block_count(int rows, const int* __restrict__ off, const int* __restrict__ idx, int width, int n_blocks,
                              int* __restrict__ counts)
{
  const int stride = gridDim.x * blockDim.x;
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += stride) {
    int c[MAX_COLUMN_BLOCKS];
#pragma unroll
    for (int b = 0; b < MAX_COLUMN_BLOCKS; ++b) c[b] = 0;
    for (int p = off[r]; p < off[r + 1]; ++p) {
      const int b = idx[p] / width;
#pragma unroll
      for (int q = 0; q < MAX_COLUMN_BLOCKS; ++q)
        if (q == b) ++c[q];
    }
#pragma unroll
    for (int b = 0; b < MAX_COLUMN_BLOCKS; ++b)
      if (b < n_blocks) counts[(size_t)b * (rows + 1) + r] = c[b];
  }
}
// stable: the entries of a row keep their order inside each block
__global__ void k_block_fill(int rows, const int* __restrict__ off, const int* __restrict__ idx,
                             const double* __restrict__ val, int width, block_ptrs_t out)
{
  const int stride = gridDim.x * blockDim.x;
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += stride) {
    int pos[MAX_COLUMN_BLOCKS];
#pragma unroll
    for (int b = 0; b < MAX_COLUMN_BLOCKS; ++b) pos[b] = out.off[b] ? out.off[b][r] : 0;
    for (int p = off[r]; p < off[r + 1]; ++p) {
      const int j = idx[p], b = j / width;
      const double v = val[p];
#pragma unroll
      for (int q = 0; q < MAX_COLUMN_BLOCKS; ++q)
        if (q == b) {
          out.idx[q][pos[q]] = j;
          out.val[q][pos[q]] = v;
          ++pos[q];
        }
    }
  }
}

}  // namespace

// Splits a CSR matrix into n_blocks CSR matrices with the same rows: block b keeps the entries whose column lies in
// [b * width, (b + 1) * width), in their original order, with GLOBAL column indices.  Step 1 (this call) fills the
// row offsets blk_off[b] (rows + 1 ints each, caller-allocated) and returns the block sizes; the caller allocates
// idx / val and calls csr_split_columns_fill.
void csr_split_columns_offsets(int rows, const int* off, const int* idx, int width, int n_blocks, int* const* blk_off,
                               int* blk_nnz_host, cudaStream_t stream)
{
  if (n_blocks > MAX_COLUMN_BLOCKS) throw lp_error(error_type_t::RuntimeError, "too many column blocks");
  dvec<int> counts((size_t)n_blocks * (rows + 1));
  counts.zero(stream);
  const int sms = current_device_sms();
  const int grid = std::max(1, std::min((rows + 255) / 256, sms * 8));
  k_block_count<<<grid, 256, 0, stream>>>(rows, off, idx, width, n_blocks, counts.data());
  CUOPT_CUDA_TRY(cudaGetLastError());
  size_t tmp_bytes = 0;
  CUOPT_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, counts.data(), blk_off[0], rows + 1, stream));
  dvec<unsigned char> tmp(tmp_bytes + 16);
  for (int b = 0; b < n_blocks; ++b) {
    size_t bytes = tmp.size();
    CUOPT_CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp.data(), bytes, counts.data() + (size_t)b * (rows + 1), blk_off[b],
                                                  rows + 1, stream));
    CUOPT_CUDA_TRY(cudaMemcpyAsync(blk_nnz_host + b, blk_off[b] + rows, sizeof(int), cudaMemcpyDeviceToHost, stream));
  }
  CUOPT_CUDA_TRY(cudaStreamSynchronize(stream));
}

void csr_split_columns_fill(int rows, const int* off, const int* idx, const double* val, int width, int n_blocks,
                            int* const* blk_off, int* const* blk_idx, double* const* blk_val, cudaStream_t stream)
{
  block_ptrs_t out{};
  for (int b = 0; b < n_blocks; ++b) {
    out.off[b] = blk_off[b];
    out.idx[b] = blk_idx[b];
    out.val[b] = blk_val[b];
  }
  const int sms = current_device_sms();
  const int grid = std::max(1, std::min((rows + 255) / 256, sms * 8));
  k_block_fill<<<grid, 256, 0, stream>>>(rows, off, idx, val, width, out);
  CUOPT_CUDA_TRY(cudaGetLastError());
  CUOPT_CUDA_TRY(cudaStreamSynchronize(stream));
}

// ---- small CUB wrappers for the trust-region restart (trust_region.cuh): library calls once per major iteration ----
// keys_out ascending (doubles >= 0 or +inf), vals_out = the permutation that sorts them (stable)
void sort_keys_with_index(int count, const double* keys_in, double* keys_out, const int* vals_in, int* vals_out,
                          cudaStream_t stream)
{
  size_t bytes = 0;
  CUOPT_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, bytes, keys_in, keys_out, vals_in, vals_out, count, 0, 64, stream));
  dvec<unsigned char> tmp(bytes + 16);
  bytes = tmp.size();
  CUOPT_CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp.data(), bytes, keys_in, keys_out, vals_in, vals_out, count, 0, 64, stream));
  CUOPT_CUDA_TRY(cudaStreamSynchronize(stream));
}
void exclusive_sum_int(int count, const int* in, int* out, cudaStream_t stream)
{
  if (count <= 0) return;
  size_t bytes = 0;
  CUOPT_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, count, stream));
  dvec<unsigned char> tmp(bytes + 16);
  bytes = tmp.size();
  CUOPT_CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp.data(), bytes, in, out, count, stream));
  CUOPT_CUDA_TRY(cudaStreamSynchronize(stream));  // tmp goes out of scope
}

void inclusive_sum_in_place(int count, double* values, cudaStream_t stream)
{
  size_t bytes = 0;
  CUOPT_CUDA_TRY(cub::DeviceScan::InclusiveSum(nullptr, bytes, values, values, count, stream));
  dvec<unsigned char> tmp(bytes + 16);
  bytes = tmp.size();
  CUOPT_CUDA_TRY(cub::DeviceScan::InclusiveSum(tmp.data(), bytes, values, values, count, stream));
  CUOPT_CUDA_TRY(cudaStreamSynchronize(stream));
}

// toff must hold cols + 1 ints, tidx / tval nnz elements.  All pointers are device pointers.
void csr_transpose_device(int rows, int cols, int nnz, const int* off, const int* idx, const double* val, int* toff,
                          int* tidx, double* tval, cudaStream_t stream)
{
  dvec<int> entry_row(nnz), entry_id(nnz), keys_out(nnz), sorted_entry(nnz), col_count((size_t)cols + 1);
  col_count.zero(stream);
  const int sms = current_device_sms();
  k_expand_rows_and_count<<<std::max(1, std::min((rows + 7) / 8, sms * 16)), 256, 0, stream>>>(
    rows, off, idx, entry_row.data(), entry_id.data(), col_count.data());
  CUOPT_CUDA_TRY(cudaGetLastError());

  size_t tmp_scan = 0, tmp_sort = 0;
  CUOPT_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tmp_scan, col_count.data(), toff, cols + 1, stream));
  int end_bit = 1;
  while (end_bit < 31 && (1LL << end_bit) < (long long)cols) ++end_bit;
  CUOPT_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, idx, keys_out.data(), entry_id.data(),
                                                  sorted_entry.data(), nnz, 0, end_bit, stream));
  dvec<unsigned char> tmp(std::max(tmp_scan, tmp_sort) + 16);
  size_t bytes = tmp.size();
  CUOPT_CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp.data(), bytes, col_count.data(), toff, cols + 1, stream));
  bytes = tmp.size();
  CUOPT_CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp.data(), bytes, idx, keys_out.data(), entry_id.data(),
                                                  sorted_entry.data(), nnz, 0, end_bit, stream));
  k_permute<<<std::max(1, std::min((nnz + 255) / 256, sms * 8)), 256, 0, stream>>>(nnz, sorted_entry.data(),
                                                                                   entry_row.data(), val, tidx, tval);
  CUOPT_CUDA_TRY(cudaGetLastError());
  CUOPT_CUDA_TRY(cudaStreamSynchronize(stream));  // temporaries die with this scope
}

}  // namespace cuopt_b200
