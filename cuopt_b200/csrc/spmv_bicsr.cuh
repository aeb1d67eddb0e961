// Block-interleaved CSR ("BICSR"): the storage format and SpMV core of every sparse product of the solver (sm_90a).
//
// Layout.  The host cuts the rows of a CSR matrix into blocks of whole consecutive rows with at most 256 entries and at
// most 256 rows.  Block b owns the 256 slots [256 b, 256 b + 256) of the index / value arrays; slot 32 k + l holds the
// block's entry 8 l + k, so ONE coalesced load instruction k (lane l reads slot 32 k + l) hands lane l the k-th of its
// EIGHT CONSECUTIVE entries 8 l .. 8 l + 7.  Bit 31 of a stored column index marks the last entry of a row; unused slots
// hold {0x7fffffff, 0.0} and are never gathered.  A 2-byte table gives, per row, the slot of its last entry (0xffff: empty
// row).  Rows longer than a block stay in the plain CSR arrays and are handled by "long-row" blocks (one warp strides the
// row).  Storage overhead over CSR: the padding of the last, partly filled lane group of each block (0 % for 8 entries
// per row, 0.7-1.6 % for the Binomial / Poisson row lengths of the bench workloads) + 2 bytes per row.
//
// Kernel core (one warp per block, blocks dealt round robin):
//   1. 8 coalesced 4-byte + 8 coalesced 8-byte loads (evict-first) bring the block; the index loads of the warp's NEXT block
//      are issued before the arithmetic of this one, so its gathers can start the moment the loop comes around;
//   2. 8 independent gathers per lane (L1 no-allocate, L2 evict-last);
//   3. products never leave the registers: every lane adds its 8 consecutive products left to right, closing a partial sum
//      at every row end; the sum of a row that continues from earlier lanes is completed by a carry handed down with
//      __shfl_up (one round per additional lane a row spans, usually 0-2);
//   4. ONE double per row goes through shared memory — written to the slot of the row's last entry, read by the lane that
//      runs the row epilogue (lane r mod 32 of row r, so the epilogue's vector accesses are coalesced).
// Against the round-1 core (products parked in shared memory, one lane per row re-reading them) this removes ~80 % of the
// shared-memory wavefronts and every per-entry bank conflict from the L1TEX unit that also has to serve the gathers
// (scripts/spmv_lab.cu compares the two).
//
// Summation order.  Inside a lane: strictly left to right.  A row that spans lanes is (carry from the earlier lanes) +
// (this lane's left-to-right part).  Everything is a fixed function of the block cut, so results are bit-reproducible run
// to run; they differ in the last bits from a sequential row sum (parity tests: 1e-12 relative, tests/test_gpu_parity.py).
#pragma once

#include "device_utils.cuh"

namespace cuopt_b200 {

constexpr int BICSR_CH              = 8;              // consecutive entries per lane
constexpr int BICSR_SLOTS           = 32 * BICSR_CH;  // entries per block
constexpr int BICSR_MAX_ROWS        = 256;            // rows per block
constexpr int BICSR_THREADS         = 256;            // CTA size of the SpMV kernels
constexpr int BICSR_WARPS           = BICSR_THREADS / 32;
constexpr int BICSR_PAD             = 0x7fffffff;     // index of an unused slot
constexpr unsigned short BICSR_EMPTY = 0xffff;        // row_slot of a row without entries
constexpr int BICSR_MIN_CTAS        = 4;              // 64 registers: 8 idx + 8 next idx + 16 val + 16 gathered + payload
__host__ __device__ constexpr int bicsr_min_ctas(int npre) { return npre > 1 ? 3 : BICSR_MIN_CTAS; }  // two payload sets: 85

__host__ __device__ constexpr int bicsr_slot(int q) { return (q % BICSR_CH) * 32 + q / BICSR_CH; }

struct bicsr_view_t {
  const int2* desc;                // n_blk block descriptors {first row, one past the last row}; long-row blocks: {row, row + 1}
  const unsigned short* row_slot;  // per row: slot (inside its block) of the row's last entry, BICSR_EMPTY for an empty row
  const int* idx;                  // n_std * 256 column indices (bit 31: row end; BICSR_PAD: unused slot)
  const double* val;               // n_std * 256 values
  int n_std, n_blk;                // blocks [0, n_std) are interleaved blocks, [n_std, n_blk) long rows
  const int* off;                  // plain CSR of the same matrix: read by the long-row blocks only
  const int* cidx;
  const double* cval;
};

// Steps 3-4 of the core for one gathered vector: bit k of `ends` = entry k of this lane closes a row; the sum of every row
// that ends in this lane's chunk goes to rsw[slot of its last entry].
__device__ __forceinline__ void bicsr_block_row_sums(const double (&a)[BICSR_CH], const double (&g)[BICSR_CH], unsigned ends,
                                                     int lane, double* rsw)
{
  constexpr unsigned FULL = 0xffffffffu;
  // chunk sums, left to right, branch-free; the FIRST row end of the chunk still lacks what earlier lanes hold of that row
  double s = 0.0, head = 0.0;
  const int kf = ends ? __ffs(ends) - 1 : -1;
#pragma unroll
  for (int k = 0; k < BICSR_CH; ++k) {
    s = __dadd_rn(s, __dmul_rn(a[k], g[k]));  // product, then sum: no FMA contraction (the CPU oracle has none either)
    const bool e = (ends >> k) & 1u;
    if (e && k != kf) rsw[k * 32 + lane] = s;
    head = (k == kf) ? s : head;
    s    = e ? 0.0 : s;
  }
  // carry = what the lanes before this one hold of the row that is open at this lane's first entry.  A lane without any
  // row end passes its whole chunk on; runs of such lanes need one more shuffle round each.
  double tail  = s;
  double carry = __shfl_up_sync(FULL, tail, 1);
  if (lane == 0) carry = 0.0;
  unsigned pending = __ballot_sync(FULL, kf < 0);
  while (pending) {
    if (kf < 0) tail = carry + s;
    carry = __shfl_up_sync(FULL, tail, 1);
    if (lane == 0) carry = 0.0;
    pending &= pending << 1;
  }
  if (kf >= 0) rsw[kf * 32 + lane] = carry + head;
}

// Walks this warp's blocks.
//   pre_op(row)            -> payload P (vector operands of the row epilogue; issued before the matrix loads for the first
//                             32 rows of a block, so their latency hides behind the gathers)
//   row_op(row, sum, P)    exactly once per row of the matrix, by lane (row - first row of the block) mod 32
// rsw: this warp's BICSR_SLOTS doubles of shared memory.
// INIT: the row's result is P::init + (sum over this matrix's entries) — a running sum over the column blocks of a gather-
// blocked product (pdlp_kernels.cuh).
// NPRE: row groups (of 32 rows) per block whose payload is fetched ahead of the gathers: 1, or 2 for matrices with short
// rows, whose blocks hold ~64 rows (the column blocks of a gather-blocked matrix: 4 entries per row at configs[3]).
template <typename P, bool INIT = false, int NPRE = 1, typename PreOp, typename RowOp>
__device__ __forceinline__ void spmv_bicsr_rows(const bicsr_view_t& A,
                                                const double* __restrict__ x,
                                                double* rsw,
                                                PreOp& pre_op,
                                                RowOp& row_op,
                                                unsigned long long gather_policy)
{
  const int lane          = threadIdx.x & 31;
  const int gwarp         = blockIdx.x * BICSR_WARPS + (threadIdx.x >> 5);
  const int nwarps        = gridDim.x * BICSR_WARPS;
  int c[BICSR_CH];
  if (gwarp < A.n_std) {
#pragma unroll
    for (int k = 0; k < BICSR_CH; ++k) c[k] = ld_stream(A.idx + (size_t)gwarp * BICSR_SLOTS + k * 32 + lane);
  }
  for (int b = gwarp; b < A.n_std; b += nwarps) {
    const int2 d  = __ldg(A.desc + b);
    const int r0 = d.x, r1 = d.y;
    P pl[NPRE];
    unsigned short slot[NPRE];
#pragma unroll
    for (int q = 0; q < NPRE; ++q) {
      slot[q] = BICSR_EMPTY;
      if (r0 + lane + 32 * q < r1) {
        pl[q]   = pre_op(r0 + lane + 32 * q);
        slot[q] = __ldg(A.row_slot + r0 + lane + 32 * q);
      }
    }
    const size_t base = (size_t)b * BICSR_SLOTS + lane;
    double a[BICSR_CH], g[BICSR_CH];
#pragma unroll
    for (int k = 0; k < BICSR_CH; ++k) a[k] = ld_stream(A.val + base + k * 32);
#pragma unroll
    for (int k = 0; k < BICSR_CH; ++k) {
      const int col = c[k] & 0x7fffffff;
      g[k]          = col != BICSR_PAD ? ld_l2(x + col, gather_policy) : 0.0;
    }
    unsigned ends = 0;
#pragma unroll
    for (int k = 0; k < BICSR_CH; ++k) ends |= (unsigned)(c[k] < 0) << k;
    if (b + nwarps < A.n_std) {
#pragma unroll
      for (int k = 0; k < BICSR_CH; ++k) c[k] = ld_stream(A.idx + (size_t)(b + nwarps) * BICSR_SLOTS + k * 32 + lane);
    }
    bicsr_block_row_sums(a, g, ends, lane, rsw);
    __syncwarp();
#pragma unroll
    for (int q = 0; q < NPRE; ++q) {
      if (r0 + lane + 32 * q < r1) {
        double sum = slot[q] != BICSR_EMPTY ? rsw[slot[q]] : 0.0;
        if constexpr (INIT) sum = pl[q].init + sum;
        row_op(r0 + lane + 32 * q, sum, pl[q]);
      }
    }
    for (int r = r0 + 32 * NPRE + lane; r < r1; r += 32) {  // blocks of very short rows hold more rows still
      const P p2              = pre_op(r);
      const unsigned short s2 = __ldg(A.row_slot + r);
      double sum              = s2 != BICSR_EMPTY ? rsw[s2] : 0.0;
      if constexpr (INIT) sum = p2.init + sum;
      row_op(r, sum, p2);
    }
    __syncwarp();
  }
  // rows longer than a block: lanes stride over the row in the plain CSR arrays, fixed xor tree at the end
  for (int b = A.n_std + gwarp; b < A.n_blk; b += nwarps) {
    const int row = __ldg(A.desc + b).x;
    const int lo = __ldg(A.off + row), hi = __ldg(A.off + row + 1);
    P pl;
    if (lane == 0) pl = pre_op(row);
    double acc = 0.0;
    for (int e = lo + lane; e < hi; e += 32) acc += ld_stream(A.cval + e) * ld_l2(x + ld_stream(A.cidx + e), gather_policy);
    acc = warp_sum(acc);
    if (lane == 0) {
      if constexpr (INIT) acc = pl.init + acc;
      row_op(row, acc, pl);
    }
  }
}

// Two vectors through ONE stream of the matrix: row_op(row, (M u)_row, (M v)_row) exactly once per row, by the same lane as
// in spmv_bicsr_rows.  Each sum is formed exactly as spmv_bicsr_rows forms it.  rsw_u / rsw_v: BICSR_SLOTS doubles each.
// No payload is fetched ahead and the next block's indices are not prefetched: the 16 gathers of a block already keep the
// warp's loads in flight, and the registers go to the second set of gathered values.
template <typename RowOp>
__device__ __forceinline__ void spmv_bicsr_rows_pair(const bicsr_view_t& A,
                                                     const double* __restrict__ u,
                                                     const double* __restrict__ v,
                                                     double* rsw_u,
                                                     double* rsw_v,
                                                     RowOp& row_op,
                                                     unsigned long long gather_policy)
{
  const int lane   = threadIdx.x & 31;
  const int gwarp  = blockIdx.x * BICSR_WARPS + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * BICSR_WARPS;
  for (int b = gwarp; b < A.n_std; b += nwarps) {
    const int2 d      = __ldg(A.desc + b);
    const size_t base = (size_t)b * BICSR_SLOTS + lane;
    int c[BICSR_CH];
    double a[BICSR_CH], gu[BICSR_CH], gv[BICSR_CH];
#pragma unroll
    for (int k = 0; k < BICSR_CH; ++k) c[k] = ld_stream(A.idx + base + k * 32);
#pragma unroll
    for (int k = 0; k < BICSR_CH; ++k) a[k] = ld_stream(A.val + base + k * 32);
#pragma unroll
    for (int k = 0; k < BICSR_CH; ++k) {
      const int col = c[k] & 0x7fffffff;
      gu[k]         = col != BICSR_PAD ? ld_l2(u + col, gather_policy) : 0.0;
      gv[k]         = col != BICSR_PAD ? ld_l2(v + col, gather_policy) : 0.0;
    }
    unsigned ends = 0;
#pragma unroll
    for (int k = 0; k < BICSR_CH; ++k) ends |= (unsigned)(c[k] < 0) << k;
    bicsr_block_row_sums(a, gu, ends, lane, rsw_u);
    bicsr_block_row_sums(a, gv, ends, lane, rsw_v);
    __syncwarp();
    for (int r = d.x + lane; r < d.y; r += 32) {
      const unsigned short s = __ldg(A.row_slot + r);
      row_op(r, s != BICSR_EMPTY ? rsw_u[s] : 0.0, s != BICSR_EMPTY ? rsw_v[s] : 0.0);
    }
    __syncwarp();
  }
  for (int b = A.n_std + gwarp; b < A.n_blk; b += nwarps) {
    const int row = __ldg(A.desc + b).x;
    const int lo = __ldg(A.off + row), hi = __ldg(A.off + row + 1);
    double acc_u = 0.0, acc_v = 0.0;
    for (int e = lo + lane; e < hi; e += 32) {
      const double a = ld_stream(A.cval + e);
      const int col  = ld_stream(A.cidx + e);
      acc_u += a * ld_l2(u + col, gather_policy);
      acc_v += a * ld_l2(v + col, gather_policy);
    }
    acc_u = warp_sum(acc_u);
    acc_v = warp_sum(acc_v);
    if (lane == 0) row_op(row, acc_u, acc_v);
  }
}

// ---- device-side construction (one warp per interleaved block) ----------------------------------------------------------
// Fills the block's 256 slots from the plain CSR arrays (bval may be null: structure only) and the row_slot table.
__global__ void __launch_bounds__(256) k_bicsr_fill(int n_std,
                                                    const int2* __restrict__ desc,
                                                    const int* __restrict__ off,
                                                    const int* __restrict__ idx,
                                                    const double* __restrict__ val,
                                                    int* __restrict__ bidx,
                                                    double* __restrict__ bval,
                                                    unsigned short* __restrict__ row_slot)
{
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int b = blockIdx.x * wpb + (threadIdx.x >> 5); b < n_std; b += gridDim.x * wpb) {
    const int2 d      = desc[b];
    const int lo      = off[d.x];
    const size_t base = (size_t)b * BICSR_SLOTS;
    const int cnt = off[d.y] - lo;
    // slot-major: coalesced stores (the loads of one instruction are 8 entries apart); row ends are flagged afterwards
#pragma unroll
    for (int k = 0; k < BICSR_CH; ++k) {
      const int q                = BICSR_CH * lane + k;
      bidx[base + k * 32 + lane] = q < cnt ? idx[lo + q] : BICSR_PAD;
      if (bval) bval[base + k * 32 + lane] = q < cnt ? val[lo + q] : 0.0;
    }
    __syncwarp();
    for (int r = d.x + lane; r < d.y; r += 32) {
      const int p0 = off[r], p1 = off[r + 1];
      unsigned short slot = BICSR_EMPTY;
      if (p1 > p0) {
        slot = (unsigned short)bicsr_slot(p1 - 1 - lo);
        bidx[base + slot] |= (int)0x80000000u;  // each row flags its own last entry: no two lanes touch the same slot
      }
      row_slot[r] = slot;
    }
    __syncwarp();
  }
}
// Values only, onto an existing structure (the scaled copy of a matrix shares indices / descriptors with the original).
__global__ void __launch_bounds__(256) k_bicsr_fill_values(int n_std,
                                                           const int2* __restrict__ desc,
                                                           const int* __restrict__ off,
                                                           const double* __restrict__ val,
                                                           double* __restrict__ bval)
{
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int b = blockIdx.x * wpb + (threadIdx.x >> 5); b < n_std; b += gridDim.x * wpb) {
    const int2 d      = desc[b];
    const int lo      = off[d.x];
    const int cnt     = off[d.y] - lo;
    const size_t base = (size_t)b * BICSR_SLOTS;
    // slot-major: coalesced stores, the loads of one instruction are 8 entries apart
#pragma unroll
    for (int k = 0; k < BICSR_CH; ++k) {
      const int q                = BICSR_CH * lane + k;
      bval[base + k * 32 + lane] = q < cnt ? val[lo + q] : 0.0;
    }
  }
}

}  // namespace cuopt_b200
