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
// Compact form (column blocks of a gather-blocked product on one GPU, template parameter FMT of the kernels below).
//   BICSR_FMT_IDX3: an entry's column is stored RELATIVE TO THE FIRST COLUMN OF ITS COLUMN BLOCK (col0; the gathers read
//     x + col0) in three bytes: the low 16 bits in lo16, lane-major (lane l's entries 8 l .. 8 l + 7 are one 16-byte
//     word), and one 8-byte word hi8 per lane whose byte k holds the high 5 bits of its entry k, BICSR_HI_PAD (bit 6) for an
//     unused slot and BICSR_HI_END (bit 7) for the last entry of a row.  Needs a column block of at most 2^21 columns.
//   BICSR_FMT_MASK: instead of row_slot, 8 words per block whose bit i is set when row (first row + i) has entries in the
//     block.  The sum of a row goes to rsw[q], q = its ordinal among the block's non-empty rows, which the row sums find
//     from the ballots of the row ends and the epilogue from a prefix popcount of the mask.
// Both change where bytes come from, not what is added: the products and every summation order are those of FMT 0.
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

constexpr int BICSR_FMT_IDX3     = 1;        // three-byte block-local column indices (lo16 + hi8)
constexpr int BICSR_FMT_MASK     = 2;        // non-empty-row mask instead of row_slot
constexpr int BICSR_IDX3_MAX_WIDTH = 1 << 21;  // widest column block the three-byte indices can address
constexpr unsigned BICSR_HI_PAD  = 0x40u;
constexpr unsigned BICSR_HI_END  = 0x80u;

struct bicsr_view_t {
  const int2* desc;                // n_blk block descriptors {first row, one past the last row}; long-row blocks: {row, row + 1}
  const unsigned short* row_slot;  // per row: slot (inside its block) of the row's last entry, BICSR_EMPTY for an empty row
  const int* idx;                  // n_std * 256 column indices (bit 31: row end; BICSR_PAD: unused slot)
  const double* val;               // n_std * 256 values
  int n_std, n_blk;                // blocks [0, n_std) are interleaved blocks, [n_std, n_blk) long rows
  const int* off;                  // plain CSR of the same matrix: read by the long-row blocks only
  const int* cidx;
  const double* cval;
  const unsigned short* lo16;      // BICSR_FMT_IDX3: n_std * 256 low halves of the local columns
  const unsigned long long* hi8;   // BICSR_FMT_IDX3: n_std * 32 words of high bytes (one per lane)
  const unsigned* mask;            // BICSR_FMT_MASK: n_std * 8 words
  int col0;                        // BICSR_FMT_IDX3: first column of the column block
};

// Index words of one interleaved block, as the core keeps them between the load and the gathers.
template <int FMT>
struct bicsr_cols_t {
  int c[BICSR_CH];  // FMT 0: stored index (bit 31: row end)
};
template <>
struct bicsr_cols_t<BICSR_FMT_IDX3> {
  uint4 lo;
  unsigned long long hi;
};
template <>
struct bicsr_cols_t<BICSR_FMT_IDX3 | BICSR_FMT_MASK> : bicsr_cols_t<BICSR_FMT_IDX3> {};
template <>
struct bicsr_cols_t<BICSR_FMT_MASK> : bicsr_cols_t<0> {};

template <int FMT>
__device__ __forceinline__ void bicsr_load_cols(const bicsr_view_t& A, int b, int lane, bicsr_cols_t<FMT>& w)
{
  if constexpr ((FMT & BICSR_FMT_IDX3) != 0) {
    w.lo = __ldcs(reinterpret_cast<const uint4*>(A.lo16 + (size_t)b * BICSR_SLOTS) + lane);
    w.hi = __ldcs(A.hi8 + (size_t)b * 32 + lane);
  } else {
#pragma unroll
    for (int k = 0; k < BICSR_CH; ++k) w.c[k] = ld_stream(A.idx + (size_t)b * BICSR_SLOTS + k * 32 + lane);
  }
}
// column of entry k, relative to the gather pointer (-1: unused slot)
template <int FMT>
__device__ __forceinline__ int bicsr_col(const bicsr_cols_t<FMT>& w, int k)
{
  if constexpr ((FMT & BICSR_FMT_IDX3) != 0) {
    const unsigned lw = k < 2 ? w.lo.x : k < 4 ? w.lo.y : k < 6 ? w.lo.z : w.lo.w;
    const unsigned hb = (unsigned)(w.hi >> (8 * k)) & 0xffu;
    return (hb & BICSR_HI_PAD) ? -1 : (int)(((hb & 0x1fu) << 16) | ((lw >> (16 * (k & 1))) & 0xffffu));
  } else {
    const int col = w.c[k] & 0x7fffffff;
    return col != BICSR_PAD ? col : -1;
  }
}
// bit k: entry k closes a row
template <int FMT>
__device__ __forceinline__ unsigned bicsr_ends(const bicsr_cols_t<FMT>& w)
{
  unsigned ends = 0;
#pragma unroll
  for (int k = 0; k < BICSR_CH; ++k) {
    if constexpr ((FMT & BICSR_FMT_IDX3) != 0) ends |= (unsigned)((w.hi >> (8 * k + 7)) & 1u) << k;
    else ends |= (unsigned)(w.c[k] < 0) << k;
  }
  return ends;
}
template <int FMT>
__device__ __forceinline__ const double* bicsr_gather_base(const bicsr_view_t& A, const double* x)
{
  if constexpr ((FMT & BICSR_FMT_IDX3) != 0) return x + A.col0;
  else return x;
}

// Row epilogue lookup of BICSR_FMT_MASK: the block's mask word of row group q (mw: word `lane` of the block's mask in
// lanes 0-7) gives this lane's row its ordinal among the non-empty rows; base counts the non-empty rows of groups < q.
struct bicsr_mask_cursor_t {
  unsigned mw;
  int base;
  // -1: this lane's row of group q is empty in the block
  __device__ __forceinline__ int next(int q, int lane)
  {
    const unsigned m = __shfl_sync(0xffffffffu, mw, q);
    const int ord    = ((m >> lane) & 1u) ? base + __popc(m & ((1u << lane) - 1u)) : -1;
    base += __popc(m);
    return ord;
  }
};

// Row ends in the lanes before this one (BICSR_FMT_MASK): prefix popcount over the bits of the per-lane counts (<= 8: 4 ballots).
__device__ __forceinline__ int bicsr_ends_before(unsigned ends, int lane)
{
  const unsigned cnt = __popc(ends), lt = (1u << lane) - 1u;
  int before         = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) before += __popc(__ballot_sync(0xffffffffu, (cnt >> j) & 1u) & lt) << j;
  return before;
}

// Steps 3-4 of the core for one gathered vector: bit k of `ends` = entry k of this lane closes a row; the sum of every row
// that ends in this lane's chunk goes to rsw[slot of its last entry].  MASK (BICSR_FMT_MASK): to rsw[ordinal of the row
// among the block's row ends] instead; before = bicsr_ends_before(ends, lane).
template <bool MASK = false>
__device__ __forceinline__ void bicsr_block_row_sums(const double (&a)[BICSR_CH], const double (&g)[BICSR_CH], unsigned ends,
                                                     int lane, double* rsw, int before = 0)
{
  constexpr unsigned FULL = 0xffffffffu;
  // chunk sums, left to right, branch-free; the FIRST row end of the chunk still lacks what earlier lanes hold of that row
  double s = 0.0, head = 0.0;
  const int kf = ends ? __ffs(ends) - 1 : -1;
  int ord      = before;  // MASK: ordinal of the next row end
#pragma unroll
  for (int k = 0; k < BICSR_CH; ++k) {
    s = __dadd_rn(s, __dmul_rn(a[k], g[k]));  // product, then sum: no FMA contraction (the CPU oracle has none either)
    const bool e = (ends >> k) & 1u;
    if (e && k != kf) rsw[MASK ? ord : k * 32 + lane] = s;
    if constexpr (MASK) ord += e;
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
  if (kf >= 0) rsw[MASK ? before : kf * 32 + lane] = carry + head;
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
// FMT: storage form of the interleaved blocks (BICSR_FMT_* bits, 0 = plain).
template <typename P, bool INIT = false, int NPRE = 1, int FMT = 0, typename PreOp, typename RowOp>
__device__ __forceinline__ void spmv_bicsr_rows(const bicsr_view_t& A,
                                                const double* __restrict__ x,
                                                double* rsw,
                                                PreOp& pre_op,
                                                RowOp& row_op,
                                                unsigned long long gather_policy)
{
  constexpr bool MASK     = (FMT & BICSR_FMT_MASK) != 0;
  const int lane          = threadIdx.x & 31;
  const int gwarp         = blockIdx.x * BICSR_WARPS + (threadIdx.x >> 5);
  const int nwarps        = gridDim.x * BICSR_WARPS;
  const double* xg        = bicsr_gather_base<FMT>(A, x);
  bicsr_cols_t<FMT> c;
  if (gwarp < A.n_std) bicsr_load_cols<FMT>(A, gwarp, lane, c);
  for (int b = gwarp; b < A.n_std; b += nwarps) {
    const int2 d  = __ldg(A.desc + b);
    const int r0 = d.x, r1 = d.y;
    P pl[NPRE];
    unsigned short slot[NPRE];
    bicsr_mask_cursor_t mc{0u, 0};
#pragma unroll
    for (int q = 0; q < NPRE; ++q) {
      slot[q] = BICSR_EMPTY;
      if (r0 + lane + 32 * q < r1) {
        pl[q] = pre_op(r0 + lane + 32 * q);
        if constexpr (!MASK) slot[q] = __ldg(A.row_slot + r0 + lane + 32 * q);
      }
    }
    const size_t base = (size_t)b * BICSR_SLOTS + lane;
    double a[BICSR_CH], g[BICSR_CH];
#pragma unroll
    for (int k = 0; k < BICSR_CH; ++k) a[k] = ld_stream(A.val + base + k * 32);
#pragma unroll
    for (int k = 0; k < BICSR_CH; ++k) {
      const int col = bicsr_col<FMT>(c, k);
      g[k]          = col >= 0 ? ld_l2(xg + col, gather_policy) : 0.0;
    }
    if constexpr (MASK) mc.mw = lane < 8 ? __ldg(A.mask + (size_t)b * 8 + lane) : 0u;  // after the gathers: fewer live registers
    const unsigned ends = bicsr_ends<FMT>(c);
    if (b + nwarps < A.n_std) bicsr_load_cols<FMT>(A, b + nwarps, lane, c);
    bicsr_block_row_sums<MASK>(a, g, ends, lane, rsw, MASK ? bicsr_ends_before(ends, lane) : 0);
    __syncwarp();
#pragma unroll
    for (int q = 0; q < NPRE; ++q) {
      int src = slot[q] != BICSR_EMPTY ? (int)slot[q] : -1;
      if constexpr (MASK) src = mc.next(q, lane);
      if (r0 + lane + 32 * q < r1) {
        double sum = src >= 0 ? rsw[src] : 0.0;
        if constexpr (INIT) sum = pl[q].init + sum;
        row_op(r0 + lane + 32 * q, sum, pl[q]);
      }
    }
    for (int q = NPRE; 32 * q < r1 - r0; ++q) {  // blocks of very short rows hold more rows still
      const int r = r0 + 32 * q + lane;
      int src     = -1;
      if constexpr (MASK) src = mc.next(q, lane);
      if (r < r1) {
        const P p2 = pre_op(r);
        if constexpr (!MASK) {
          const unsigned short s2 = __ldg(A.row_slot + r);
          src                     = s2 != BICSR_EMPTY ? (int)s2 : -1;
        }
        double sum = src >= 0 ? rsw[src] : 0.0;
        if constexpr (INIT) sum = p2.init + sum;
        row_op(r, sum, p2);
      }
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
template <int FMT = 0, typename RowOp>
__device__ __forceinline__ void spmv_bicsr_rows_pair(const bicsr_view_t& A,
                                                     const double* __restrict__ u,
                                                     const double* __restrict__ v,
                                                     double* rsw_u,
                                                     double* rsw_v,
                                                     RowOp& row_op,
                                                     unsigned long long gather_policy)
{
  constexpr bool MASK = (FMT & BICSR_FMT_MASK) != 0;
  const int lane   = threadIdx.x & 31;
  const int gwarp  = blockIdx.x * BICSR_WARPS + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * BICSR_WARPS;
  const double* ug = bicsr_gather_base<FMT>(A, u);
  const double* vg = bicsr_gather_base<FMT>(A, v);
  for (int b = gwarp; b < A.n_std; b += nwarps) {
    const int2 d      = __ldg(A.desc + b);
    const size_t base = (size_t)b * BICSR_SLOTS + lane;
    bicsr_cols_t<FMT> c;
    double a[BICSR_CH], gu[BICSR_CH], gv[BICSR_CH];
    bicsr_load_cols<FMT>(A, b, lane, c);
    bicsr_mask_cursor_t mc{0u, 0};
#pragma unroll
    for (int k = 0; k < BICSR_CH; ++k) a[k] = ld_stream(A.val + base + k * 32);
#pragma unroll
    for (int k = 0; k < BICSR_CH; ++k) {
      const int col = bicsr_col<FMT>(c, k);
      gu[k]         = col >= 0 ? ld_l2(ug + col, gather_policy) : 0.0;
      gv[k]         = col >= 0 ? ld_l2(vg + col, gather_policy) : 0.0;
    }
    const unsigned ends = bicsr_ends<FMT>(c);
    const int before    = MASK ? bicsr_ends_before(ends, lane) : 0;
    bicsr_block_row_sums<MASK>(a, gu, ends, lane, rsw_u, before);
    bicsr_block_row_sums<MASK>(a, gv, ends, lane, rsw_v, before);
    if constexpr (MASK) mc.mw = lane < 8 ? __ldg(A.mask + (size_t)b * 8 + lane) : 0u;  // two sets of gathers hold the registers
    __syncwarp();
    for (int q = 0; 32 * q < d.y - d.x; ++q) {
      const int r = d.x + 32 * q + lane;
      int s       = -1;
      if constexpr (MASK) s = mc.next(q, lane);
      if (r < d.y) {
        if constexpr (!MASK) {
          const unsigned short s2 = __ldg(A.row_slot + r);
          s                       = s2 != BICSR_EMPTY ? (int)s2 : -1;
        }
        row_op(r, s >= 0 ? rsw_u[s] : 0.0, s >= 0 ? rsw_v[s] : 0.0);
      }
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

// Structure of a column block in a compact form, from its plain CSR (values: k_bicsr_fill; the plain idx / row_slot arrays
// stay for the parts of the form that are not compact).  Null outputs are not written: lo16 / hi8 (BICSR_FMT_IDX3, columns
// relative to col0), mask (BICSR_FMT_MASK).
__global__ void __launch_bounds__(BICSR_THREADS) k_bicsr_fill_structure(int n_std,
                                                                      const int2* __restrict__ desc,
                                                                      const int* __restrict__ off,
                                                                      const int* __restrict__ idx,
                                                                      int col0,
                                                                      unsigned short* __restrict__ lo16,
                                                                      unsigned long long* __restrict__ hi8,
                                                                      unsigned* __restrict__ mask)
{
  __shared__ unsigned char is_end[BICSR_WARPS][BICSR_SLOTS];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned char* e = is_end[w];
  for (int b = blockIdx.x * BICSR_WARPS + w; b < n_std; b += gridDim.x * BICSR_WARPS) {
    const int2 d      = desc[b];
    const int lo      = off[d.x];
    const int cnt     = off[d.y] - lo;
    const size_t base = (size_t)b * BICSR_SLOTS;
#pragma unroll
    for (int k = 0; k < BICSR_CH; ++k) e[BICSR_CH * lane + k] = 0;
    __syncwarp();
    for (int q = 0; q < BICSR_MAX_ROWS / 32; ++q) {  // warp-uniform: the ballot needs every lane
      const int r  = d.x + 32 * q + lane;
      const int p0 = r < d.y ? off[r] : 0, p1 = r < d.y ? off[r + 1] : 0;
      if (p1 > p0) e[p1 - 1 - lo] = 1;
      const unsigned word = __ballot_sync(0xffffffffu, p1 > p0);
      if (mask && lane == 0) mask[(size_t)b * 8 + q] = word;
    }
    __syncwarp();
    if (lo16) {
      unsigned lw[4] = {0u, 0u, 0u, 0u};
      unsigned long long hw = 0ull;
#pragma unroll
      for (int k = 0; k < BICSR_CH; ++k) {
        const int q = BICSR_CH * lane + k;
        unsigned hb = BICSR_HI_PAD;
        if (q < cnt) {
          const unsigned c = (unsigned)(idx[lo + q] - col0);
          lw[k / 2] |= (c & 0xffffu) << (16 * (k & 1));
          hb = (c >> 16) | (e[q] ? BICSR_HI_END : 0u);
        }
        hw |= (unsigned long long)hb << (8 * k);
      }
      reinterpret_cast<uint4*>(lo16 + base)[lane] = make_uint4(lw[0], lw[1], lw[2], lw[3]);
      hi8[(size_t)b * 32 + lane]                  = hw;
    }
    __syncwarp();
  }
}

}  // namespace cuopt_b200
