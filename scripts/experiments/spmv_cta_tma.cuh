// CTA-staged / warp-consumed CSR row blocks (sm_90a: TMA bulk copies + mbarrier): TMA takes the matrix stream off the L1TEX request path.
//
// ncu on the plain warp-synchronous kernels (spmv_warp.cuh) shows they execute in exactly
// l1tex__t_sectors / #SM cycles: ~1 global-load sector per clock per SM, of which 8.0 M are the unavoidable
// gathers, 3.0 M the (col,val) stream and ~1.4 M epilogue operands.  Here the (col,val,row-offset) slices of a
// GROUP of 8 consecutive warp blocks (<= 2048 nonzeros, one contiguous range) are fetched by ONE producer warp with
// three cp.async.bulk copies per group (bulk copies must be large: per-warp 1-2 KB copies ran at ~95 cycles per
// copy and made the kernels slower), land in shared memory through the TMA unit, and are consumed by
// 8 independent consumer warps, one warp block each, exactly as in spmv_warp.cuh: 8 gathers per lane, products
// parked in place (XOR-swizzled), left-to-right row sums, fused epilogue.  Synchronisation is by mbarriers only
// (full[stage]: producer -> consumers, transaction count; empty[stage]: 8 consumer arrivals -> producer); there is no
// __syncthreads in the loop, so consumer warps drift apart by up to one stage.
#pragma once

#include "spmv_pipeline.cuh"  // mbarrier / bulk-copy PTX
#include "spmv_warp.cuh"      // warp blocks, swizzle, csr_warp_view_t

namespace cuopt_b200 {

constexpr int CT_WARPS   = 8;                    // consumer warps per CTA
constexpr int CT_THREADS = (CT_WARPS + 1) * 32;  // + one producer warp
constexpr int CT_STAGES  = 2;
constexpr int CT_NNZ     = CT_WARPS * WARP_NNZ;  // 2048
constexpr int CT_ROWS    = CT_WARPS * 32;

struct __align__(16) ct_stage_t {
  double val[CT_NNZ + 4];  // window starts at (lo0 & ~1); a consumer overwrites ITS slice with products
  int idx[CT_NNZ + 8];     // window starts at (lo0 & ~3)
  int off[CT_ROWS + 8];    // window starts at (r00 & ~3)
};
struct __align__(16) ct_smem_t {
  ct_stage_t stage[CT_STAGES];
  uint64_t full[CT_STAGES];
  uint64_t empty[CT_STAGES];
};

// swizzle that never leaves [0, cnt): full groups of 8 are permuted, a trailing partial group stays in place
__device__ __forceinline__ int ct_swz(int e, int cnt) { return ((e | 7) < cnt) ? warp_swz(e) : e; }

// Direct (unstaged) processing of one warp block: long rows and groups that cannot be staged.
template <typename P, typename PreOp, typename RowOp>
__device__ __forceinline__ void ct_block_direct(const csr_warp_view_t& A, const double* __restrict__ x, int2 d0, int2 d1,
                                                double* scratch, PreOp& pre_op, RowOp& row_op)
{
  const int lane = threadIdx.x & 31;
  const int r0 = d0.x, lo = d0.y, r1 = d1.x, hi = d1.y;
  if (hi - lo > WARP_NNZ) {
    P pl;
    if (lane == 0) pl = pre_op(r0);
    double acc = 0.0;
    for (int e = lo + lane; e < hi; e += 32) acc += ld_stream(A.val + e) * __ldcg(x + ld_stream(A.idx + e));
    acc = warp_sum(acc);
    if (lane == 0) row_op(r0, acc, pl);
    return;
  }
  const int r = r0 + lane;
  int rs = 0, re = 0;
  P pl;
  if (r < r1) {
    rs = __ldg(A.off + r) - lo;
    re = __ldg(A.off + r + 1) - lo;
    pl = pre_op(r);
  }
  const int cnt = hi - lo;
#pragma unroll
  for (int k = 0; k < WARP_KN; ++k) {
    const int e = lane + 32 * k;
    if (e < cnt) scratch[ct_swz(e, cnt)] = ld_stream(A.val + lo + e) * __ldcg(x + ld_stream(A.idx + lo + e));
  }
  __syncwarp();
  if (r < r1) {
    double sum = 0.0;
    for (int p = rs; p < re; ++p) sum += scratch[ct_swz(p, cnt)];
    row_op(r, sum, pl);
  }
  __syncwarp();
}

// Whole-CTA pipeline.  Must be called by all CT_THREADS threads.
//   pre_op(row) -> payload P (issued before the wait on the stage); row_op(row, sum, P) once per row.
template <typename P, typename PreOp, typename RowOp>
__device__ __forceinline__ void spmv_cta_tma(const csr_warp_view_t& A,
                                             const double* __restrict__ x,
                                             ct_smem_t& sm,
                                             PreOp& pre_op,
                                             RowOp& row_op)
{
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    for (int s = 0; s < CT_STAGES; ++s) {
      mbar_init(&sm.full[s], 1);
      mbar_init(&sm.empty[s], CT_WARPS);
    }
    mbar_fence_init();
  }
  __syncthreads();
  const int n_groups = (A.n_wb + CT_WARPS - 1) / CT_WARPS;

  // group descriptors: lanes 0..8 of the calling warp load the 9 warp-block boundaries of group g
  auto load_group = [&](int g, int2& mine, bool& regular, int& lo0, int& r00, int& hi_last, int& r_last) {
    const int wb0 = g * CT_WARPS;
    const int j   = min(wb0 + min(lane, CT_WARPS), A.n_wb);
    mine          = __ldg(A.wdesc + j);
    const int nxt_lo = __shfl_down_sync(0xffffffffu, mine.y, 1);
    const bool too_long = (lane < CT_WARPS) && (nxt_lo - mine.y > WARP_NNZ);
    lo0     = __shfl_sync(0xffffffffu, mine.y, 0);
    r00     = __shfl_sync(0xffffffffu, mine.x, 0);
    hi_last = __shfl_sync(0xffffffffu, mine.y, CT_WARPS);
    r_last  = __shfl_sync(0xffffffffu, mine.x, CT_WARPS);
    regular = !__any_sync(0xffffffffu, too_long) && hi_last > lo0;
  };

  if (warp == CT_WARPS) {
    // ------------------------------------------------------------------ producer warp
    int it = 0;
    for (int g = blockIdx.x; g < n_groups; g += gridDim.x, ++it) {
      const int s = it % CT_STAGES;
      int2 mine;
      bool regular;
      int lo0, r00, hi_last, r_last;
      load_group(g, mine, regular, lo0, r00, hi_last, r_last);
      if (it >= CT_STAGES) mbar_wait(&sm.empty[s], (uint32_t)(((it / CT_STAGES) + 1) & 1));
      if (lane == 0) {
        if (!regular) {
          mbar_arrive(&sm.full[s]);
        } else {
          ct_stage_t* st = &sm.stage[s];
          const int lo_v = lo0 & ~1, lo_i = lo0 & ~3, r0_a = r00 & ~3;
          const uint32_t bv = (uint32_t)(((hi_last - lo_v) * 8 + 15) & ~15);
          const uint32_t bi = (uint32_t)(((hi_last - lo_i) * 4 + 15) & ~15);
          const uint32_t bo = (uint32_t)(((r_last + 1 - r0_a) * 4 + 15) & ~15);
          fence_proxy_async();
          mbar_arrive_expect_tx(&sm.full[s], bv + bi + bo);
          bulk_g2s(st->val, A.val + lo_v, bv, &sm.full[s]);
          bulk_g2s(st->idx, A.idx + lo_i, bi, &sm.full[s]);
          bulk_g2s(st->off, A.off + r0_a, bo, &sm.full[s]);
        }
      }
      __syncwarp();
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warps
  int it = 0;
  for (int g = blockIdx.x; g < n_groups; g += gridDim.x, ++it) {
    const int s    = it % CT_STAGES;
    ct_stage_t& st = sm.stage[s];
    int2 mine;
    bool regular;
    int lo0, r00, hi_last, r_last;
    load_group(g, mine, regular, lo0, r00, hi_last, r_last);
    const int2 d0 = make_int2(__shfl_sync(0xffffffffu, mine.x, warp), __shfl_sync(0xffffffffu, mine.y, warp));
    const int2 d1 = make_int2(__shfl_sync(0xffffffffu, mine.x, warp + 1), __shfl_sync(0xffffffffu, mine.y, warp + 1));
    const bool have = (g * CT_WARPS + warp) < A.n_wb;
    const int r0 = d0.x, lo = d0.y, r1 = d1.x, hi = d1.y;
    if (!regular) {
      mbar_wait(&sm.full[s], (uint32_t)((it / CT_STAGES) & 1));
      if (have) ct_block_direct<P>(A, x, d0, d1, st.val + warp * WARP_NNZ, pre_op, row_op);
    } else {
      const int r = r0 + lane;
      P pl;
      if (have && r < r1) pl = pre_op(r);
      mbar_wait(&sm.full[s], (uint32_t)((it / CT_STAGES) & 1));
      if (have) {
        const int cnt = hi - lo;
        const int di = lo - (lo0 & ~3), dv = lo - (lo0 & ~1), doff = r0 - (r00 & ~3);
        double gx[WARP_KN], a[WARP_KN];
#pragma unroll
        for (int k = 0; k < WARP_KN; ++k) {
          const int e = lane + 32 * k;
          if (e < cnt) gx[k] = __ldcg(x + st.idx[di + e]);
        }
#pragma unroll
        for (int k = 0; k < WARP_KN; ++k) {
          const int e = lane + 32 * k;
          if (e < cnt) a[k] = st.val[dv + e];
        }
        int rs = 0, re = 0;
        if (r < r1) {
          rs = st.off[doff + lane] - lo;
          re = st.off[doff + lane + 1] - lo;
        }
        __syncwarp();  // every lane holds its staged values: the slice may now take the products
#pragma unroll
        for (int k = 0; k < WARP_KN; ++k) {
          const int e = lane + 32 * k;
          if (e < cnt) st.val[dv + ct_swz(e, cnt)] = a[k] * gx[k];
        }
        __syncwarp();
        if (r < r1) {
          double sum = 0.0;
          for (int p = rs; p < re; p += 8) {
            double v[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = (p + j < re) ? st.val[dv + ct_swz(p + j, cnt)] : 0.0;
#pragma unroll
            for (int j = 0; j < 8; ++j) sum += v[j];
          }
          row_op(r, sum, pl);
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm.empty[s]);  // this warp is done with the stage
  }
}

}  // namespace cuopt_b200
