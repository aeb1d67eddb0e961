// Hand-written sm_90a kernels of the PDLP hot path.
//
// One PDHG attempt = three launches (K1 primal step, K2 A*xbar + dual step,
// K3 A^T*y' + interaction/movement reductions + step-size rule), replacing the
// reference's per-iteration sequence of 2 cusparseSpMV + 4 cub::DeviceTransform +
// 3 cublasDdot + 1 scalar kernel + host sync
// (cpp/src/linear_programming/pdhg.cu:73-216,
//  step_size_strategy/adaptive_step_size_strategy.cu:92-345,
//  restart_strategy/weighted_average_solution.cu:73-110).
// Accept/reject, the step-size update, the weighted-average accumulation and the
// x<->x' buffer swap all happen on the device (control block pdhg_ctl_t), so a
// whole batch of attempts runs without the host.
//
// SpMV scheme (spmv_bicsr.cuh): every matrix lives in block-interleaved CSR — blocks of whole rows with at most 256
// entries, stored so that one coalesced load hands each lane 8 CONSECUTIVE entries; ONE WARP streams a block (evict-first),
// gathers the vector (L1 no-allocate, L2 evict-last), adds its products in registers (left to right per lane, carries between
// lanes by shuffle) and passes one double per row through shared memory to the lane that runs the fused row epilogue; only
// __syncwarp, never __syncthreads.  Matrix bytes are read exactly once per pass; reductions use fixed-shape trees and a
// fixed grid, so results are bit-reproducible run to run.  For large LPs K2 / K3 are split by column blocks ("gather
// blocking", further down) with the row epilogue fused into the LAST block's pass; the sharded multi-GPU attempt and its
// NVLink peer transport follow the single-GPU kernels; the evaluation / infeasibility kernels are element-wise over
// products formed by k_spmv_pair (both iterates in one stream of the unscaled matrix, over its column blocks when blocked).  DESIGN.md §5 describes these choices and their measurements.
#pragma once

#include "device_utils.cuh"
#include "spmv_bicsr.cuh"

#include <math_constants.h>

namespace cuopt_b200 {

constexpr int EW_THREADS  = 256;  // element-wise kernels
static __device__ int g_l2_hints = 1;  // device_utils.cuh make_l2_policies; CUOPT_B200_L2_HINTS=0 clears it

// Device-resident control block: every scalar the PDHG loop reads or writes.
struct pdhg_ctl_t {
  double step_size, primal_weight, tau, sigma;
  double pending_weight;  // weight of the accepted-but-not-yet-averaged iterate
  double sum_weights;     // sum of averaging weights since the last restart
  double interaction, norm_dx2, norm_dy2;
  double reduction_exponent, growth_exponent, primal_smoothing, dual_smoothing;
  int parity;       // which of the two (x, y, A^T y) buffer sets is "current"
  int pending_avg;  // buffers[parity] hold an accepted iterate that still has to enter the running sums
  int active;       // 0 -> remaining launches of the batch are no-ops
  int valid;        // last attempt: 1 accepted, 0 rejected, -1 numerical error
  int k_pdhg;       // attempts with a sane movement (reference: d_total_pdhg_iterations_)
  int attempts;     // all attempts (reference: total_pdhg_iterations_ on the host)
  int accepted;     // accepted steps (reference: internal_solver_iterations_)
  int target;       // the batch stops once `accepted` reaches this
  int its_since_restart;
  unsigned ticket[4];
};

// Result of one termination evaluation (termination_strategy/convergence_information.cu).
struct eval_t {
  double l2_primal_residual, l2_dual_residual, primal_objective, dual_objective, gap, abs_objective, kkt;
  double l2_primal_variable, l2_dual_variable;
  int status;  // termination_status_t; 6 (NumericalError) == "keep going" as in termination_strategy.cu:186
  int pad;
  double linf_relative_primal_residual, linf_relative_dual_residual;  // per_constraint_residual only, else 0
};

struct eval_consts_t {
  double objective_scaling_factor, objective_offset;
  double abs_gap_tol, rel_gap_tol, abs_primal_tol, rel_primal_tol, abs_dual_tol, rel_dual_tol;
  double l2_norm_b, l2_norm_c;
  int reduced_cost_rule;  // 1: handle_some_primal_gradients_on_finite_bounds_as_residuals
  int per_constraint_residual;  // feasibility tests on linf(residual_i - rel * rhs_i) <= abs (termination_strategy.cu:141-166)
  double primal_infeasible_tol, dual_infeasible_tol;  // infeasibility detection (k_infeasibility_* below)
};

// Publish per-CTA partial sums and elect the last CTA to finish (returns true in every thread of
// that CTA).  `parts` is NQ x gridDim.x doubles; the elected CTA reads them back in a fixed order.
template <int NQ>
__device__ __forceinline__ bool publish_and_elect(const double (&local)[NQ], double* parts, unsigned* ticket, double* red)
{
  __shared__ bool is_last;
  double tot[NQ];
#pragma unroll
  for (int q = 0; q < NQ; ++q) tot[q] = block_reduce(local[q], red);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int q = 0; q < NQ; ++q) parts[q * gridDim.x + blockIdx.x] = tot[q];
    __threadfence();
    const unsigned t = atomicAdd(ticket, 1u);
    is_last          = (t == gridDim.x - 1);
    if (is_last) *ticket = 0u;
  }
  __syncthreads();
  if (is_last) __threadfence();
  return is_last;
}

// Sum `count` published partials (written by other CTAs) in a fixed order; result in all threads.
__device__ __forceinline__ double gather_partials(const double* parts, int count, double* red)
{
  double s = 0.0;
  for (int i = threadIdx.x; i < count; i += blockDim.x) s += __ldcg(parts + i);
  return block_reduce(s, red);
}

// Adaptive step-size rule with accept / reject, executed by ONE thread per attempt
// (adaptive_step_size_strategy.cu:92-188) plus the bookkeeping the reference does on the host in take_step
// (pdlp.cu:1188-1222): buffer swap, running-average weight, iteration counters.
__device__ __forceinline__ void pdhg_step_rule(pdhg_ctl_t* ctl, double interaction, double dx2, double dy2)
{
  pdhg_ctl_t s     = *ctl;
  s.interaction    = interaction;
  s.norm_dx2       = dx2;
  s.norm_dy2       = dy2;
  s.attempts += 1;
  const double pw       = s.primal_weight;
  const double movement = s.primal_smoothing * pw * dx2 + (s.dual_smoothing / pw) * dy2;
  bool accept;
  if (movement <= 0.0 || movement >= 1.0e100) {
    // numerical error (or exact convergence): the reference leaves the retry loop, still averages and
    // swaps, and lets the next major iteration decide (pdlp.cu:1193-1221, :780-789)
    s.valid = -1;
    accept  = true;
  } else {
    const double inter = fabs(interaction);
    s.k_pdhg += 1;
    const double kc    = (double)s.k_pdhg;
    const double limit = inter > 0.0 ? movement / inter : CUDART_INF;
    accept             = s.step_size <= limit;
    s.valid            = accept ? 1 : 0;
    const double c1    = (1.0 - pow(kc + 1.0, -s.reduction_exponent)) * limit;
    const double c2    = (1.0 + pow(kc + 1.0, -s.growth_exponent)) * s.step_size;
    s.step_size        = fmin(c1, c2);
    s.tau              = s.step_size / pw;
    s.sigma            = s.step_size * pw;
  }
  if (accept) {
    s.parity ^= 1;
    s.pending_avg    = 1;
    s.pending_weight = s.step_size;  // the already-updated step size (pdlp.cu:1216-1219)
    s.sum_weights += s.step_size;
    s.accepted += 1;
    s.its_since_restart += 1;
  } else {
    s.pending_avg = 0;
  }
  s.active    = (s.valid != -1 && s.accepted < s.target) ? 1 : 0;
  s.ticket[0] = 0u;
  *ctl        = s;
}

// ---- multi-GPU peer transport primitives (used by the column-sliced attempt further down) ----
constexpr int DIST_MAX_PEERS        = 8;
constexpr int DIST_FLAG_XBAR        = 0 * DIST_MAX_PEERS;  // flags[slot + g]: rank g's contribution has landed
constexpr int DIST_FLAG_Y           = 1 * DIST_MAX_PEERS;  // gather transport: first half of rank g's y' entries
constexpr int DIST_FLAG_SCALARS     = 2 * DIST_MAX_PEERS;
constexpr int DIST_FLAG_XBAR_B      = 3 * DIST_MAX_PEERS;  // gather transport: second half of rank g's xbar entries
constexpr int DIST_FLAG_Y_B         = 4 * DIST_MAX_PEERS;  // gather transport: second half of rank g's y' entries
constexpr int DIST_FLAG_COUNT       = 5 * DIST_MAX_PEERS;
constexpr long long DIST_SPIN_LIMIT = 20000000000LL;  // ~10 s of SM clocks, then trap instead of hanging the box
struct peer_ptrs_t {
  double* p[DIST_MAX_PEERS];
};
struct peer_flags_t {
  unsigned long long* p[DIST_MAX_PEERS];
};
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v)
{
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p)
{
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
// whole CTA: returns once flags[0..count) have all reached `epoch`
__device__ __forceinline__ void peer_wait(const unsigned long long* flags, int count, unsigned long long epoch)
{
  if ((int)threadIdx.x < count) {
    const long long t0 = clock64();
    while (ld_acquire_sys(flags + threadIdx.x) < epoch) {
      __nanosleep(64);
      if (clock64() - t0 > DIST_SPIN_LIMIT) __trap();
    }
  }
  __syncthreads();
}
// whole CTA, after its last peer store: the last CTA of the grid raises flag `index` on every rank
// index2 >= 0: a second flag raised together with the first (a producer that delivers both halves at once)
__device__ __forceinline__ void peer_signal_grid_done(unsigned* ticket, const peer_flags_t& flags, int world, int index,
                                                      unsigned long long epoch, int index2 = -1)
{
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x != 0) return;
  const unsigned t = atomicAdd(ticket, 1u);
  if (t != gridDim.x - 1) return;
  *ticket = 0u;
  __threadfence_system();
#pragma unroll
  for (int r = 0; r < DIST_MAX_PEERS; ++r)
    if (r < world) {
      st_release_sys(flags.p[r] + index, epoch);
      if (index2 >= 0) st_release_sys(flags.p[r] + index2, epoch);
    }
}

// =============================================================================================
// K1 — primal step.  x' = clamp(x - tau (c - A^T y), l, u), xbar = 2x' - x
// (pdhg.cu:137-158 + utils.cuh:81-95), fused with the primal half of the running-average update
// of the PREVIOUS accepted step (weighted_average_solution.cu:88-94).
// Algorithmic bytes per variable: read x, c, A^T y, l, u (+ sum_x r/w when pending) ; write x', xbar.
// =============================================================================================
__global__ void __launch_bounds__(EW_THREADS) k_primal_step(const pdhg_ctl_t* __restrict__ ctl,
                                                            int n,
                                                            double* __restrict__ xbuf0,
                                                            double* __restrict__ xbuf1,
                                                            const double* __restrict__ aty0,
                                                            const double* __restrict__ aty1,
                                                            const double* __restrict__ c,
                                                            const double* __restrict__ l,
                                                            const double* __restrict__ u,
                                                            double* __restrict__ sum_x,
                                                            double* __restrict__ xbar)
{
  if (!ctl->active) return;
  const int cur           = ctl->parity;
  const double* x         = cur ? xbuf1 : xbuf0;
  double* xn              = cur ? xbuf0 : xbuf1;
  const double* aty       = cur ? aty1 : aty0;
  const double tau        = ctl->tau;
  const bool pending      = ctl->pending_avg != 0;
  const double w          = ctl->pending_weight;
  const int stride        = gridDim.x * blockDim.x;
  const l2_policy_t pol   = make_l2_policies(g_l2_hints);
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
    const double xj = x[j];
    if (pending) sum_x[j] = sum_x[j] + w * xj;
    const double gradient = ld_stream(c + j) - aty[j];
    double next           = xj - (tau * gradient);
    next                  = fmax(fmin(next, ld_stream(u + j)), ld_stream(l + j));
    xn[j]                 = next;
    st_l2(xbar + j, next - xj + next, pol.keep);  // K2 gathers from xbar: keep it in L2
  }
}

// =============================================================================================
// K2 — A*xbar and dual step.  y' = max(ybar + sigma lc, min(ybar + sigma uc, 0)), ybar = y - sigma (A xbar)
// (pdhg.cu:73-117 + utils.cuh:98-112) + dual half of the running average + partial ||dy||^2.
// =============================================================================================
// INIT: the product continues the running sum t of the earlier column blocks (gather blocking: this is the LAST block's pass)
// BCAST (multi-GPU "gather" transport): y' of this rank's rows also goes to the packed y' buffer of every rank that reads
// the row (peer stores over NVLink, y_peers.p[r] = rank r's buffer) and the last CTA raises the y' flag.
// FMT: storage form of A (spmv_bicsr.cuh BICSR_FMT_*)
template <bool INIT, int NPRE, bool BCAST = false, int FMT = 0>
__global__ void __launch_bounds__(BICSR_THREADS, bicsr_min_ctas(NPRE)) k_dual_step(pdhg_ctl_t* __restrict__ ctl,
                                                                             bicsr_view_t A,
                                                                             const double* __restrict__ xbar,
                                                                             double* __restrict__ ybuf0,
                                                                             double* __restrict__ ybuf1,
                                                                             const double* __restrict__ lc,
                                                                             const double* __restrict__ uc,
                                                                             double* __restrict__ sum_y,
                                                                             double* __restrict__ part_dy2,
                                                                             const unsigned long long* xbar_flags,
                                                                             int n_xbar_flags,
                                                                             const double* __restrict__ t,
                                                                             peer_ptrs_t y_peers = peer_ptrs_t{},
                                                                             peer_flags_t flags = peer_flags_t{},
                                                                             int world = 1,
                                                                             int rank = 0,
                                                                             const int* __restrict__ send = nullptr,
                                                                             int send_stride = 0)
{
  if (!ctl->active) return;
  __shared__ double rows[BICSR_WARPS][BICSR_SLOTS];
  __shared__ double red[32];
  const unsigned long long epoch = (unsigned long long)ctl->attempts + 1ull;
  // multi-GPU peer transport: xbar slices arrive by NVLink stores of the other ranks' K1s (see k_primal_step_bcast)
  if (xbar_flags) peer_wait(xbar_flags, n_xbar_flags, (unsigned long long)ctl->attempts + 1ull);
  const int cur      = ctl->parity;
  const double* y    = cur ? ybuf1 : ybuf0;
  double* yn         = cur ? ybuf0 : ybuf1;
  const double sigma = ctl->sigma;
  const bool pending = ctl->pending_avg != 0;
  const double w     = ctl->pending_weight;
  double dy2         = 0.0;
  const l2_policy_t pol = make_l2_policies(g_l2_hints);
  struct payload_t {
    double y, lc, uc, sum, init;
  };
  auto pre_op = [&](int i) {
    payload_t p;
    p.y    = y[i];
    p.lc   = ld_stream(lc + i);
    p.uc   = ld_stream(uc + i);
    p.sum  = pending ? sum_y[i] : 0.0;
    p.init = INIT ? ld_l2(t + i, pol.stream) : 0.0;
    return p;
  };
  auto row_op = [&](int i, double s, const payload_t& p) {
    if (pending) sum_y[i] = p.sum + w * p.y;
    double next      = p.y - (sigma * s);
    const double low = next + sigma * p.lc;
    const double up  = next + sigma * p.uc;
    next             = fmax(low, fmin(up, 0.0));
    st_l2(yn + i, next, pol.keep);  // K3 gathers from y': keep it in L2
    if constexpr (BCAST) {  // send[r * send_stride + i]: where row i lives in rank r's packed y' (-1: rank r never reads it)
#pragma unroll
      for (int r = 0; r < DIST_MAX_PEERS; ++r)
        if (r < world) {
          const int d = __ldg(send + (size_t)r * send_stride + i);
          if (d >= 0) y_peers.p[r][d] = next;
        }
    }
    const double d   = next - p.y;
    dy2 += d * d;
  };
  spmv_bicsr_rows<payload_t, INIT, NPRE, FMT>(A, xbar, rows[threadIdx.x >> 5], pre_op, row_op, pol.keep);
  const double tot = block_reduce(dy2, red);
  if (threadIdx.x == 0) part_dy2[blockIdx.x] = tot;
  if constexpr (BCAST) peer_signal_grid_done(&ctl->ticket[2], flags, world, DIST_FLAG_Y + rank, epoch, DIST_FLAG_Y_B + rank);
}

// =============================================================================================
// K3 — A^T*y' with the interaction / movement reductions and, in the last CTA to finish, the
// adaptive step-size rule with accept/reject (adaptive_step_size_strategy.cu:92-188, 232-345).
// interaction = dx . (A^T y' - A^T y)  (the reference's SpMV-saving form, :267-277).
// =============================================================================================
// INIT: as in k_dual_step (the last column block's pass of a gather-blocked A^T y')
template <bool INIT, int NPRE, int FMT = 0>
__global__ void __launch_bounds__(BICSR_THREADS, bicsr_min_ctas(NPRE)) k_transpose_step(pdhg_ctl_t* __restrict__ ctl,
                                                                                  bicsr_view_t AT,
                                                                                  const double* __restrict__ ybuf0,
                                                                                  const double* __restrict__ ybuf1,
                                                                                  const double* __restrict__ xbuf0,
                                                                                  const double* __restrict__ xbuf1,
                                                                                  double* __restrict__ aty0,
                                                                                  double* __restrict__ aty1,
                                                                                  double* __restrict__ parts,  // 2 x gridDim.x
                                                                                  const double* __restrict__ part_dy2,
                                                                                  int n_part_dy2,
                                                                                  const double* __restrict__ t)
{
  if (!ctl->active) return;
  __shared__ double rows[BICSR_WARPS][BICSR_SLOTS];
  __shared__ double red[32];
  const int cur     = ctl->parity;
  const double* yn  = cur ? ybuf0 : ybuf1;  // candidate y'
  const double* x   = cur ? xbuf1 : xbuf0;
  const double* xn  = cur ? xbuf0 : xbuf1;
  const double* aty = cur ? aty1 : aty0;
  double* atyn      = cur ? aty0 : aty1;
  double acc[2]     = {0.0, 0.0};  // interaction, ||dx||^2
  const l2_policy_t pol = make_l2_policies(g_l2_hints);
  struct payload_t {
    double dx, aty, init;
  };
  auto pre_op = [&](int j) {
    payload_t p;
    p.dx   = ld_l2(xn + j, pol.stream) - ld_l2(x + j, pol.stream);
    p.aty  = ld_l2(aty + j, pol.stream);
    p.init = INIT ? ld_l2(t + j, pol.stream) : 0.0;
    return p;
  };
  auto row_op = [&](int j, double s, const payload_t& p) {
    st_l2(atyn + j, s, pol.stream);
    acc[0] += p.dx * (s - p.aty);
    acc[1] += p.dx * p.dx;
  };
  spmv_bicsr_rows<payload_t, INIT, NPRE, FMT>(AT, yn, rows[threadIdx.x >> 5], pre_op, row_op, pol.keep);

  if (!publish_and_elect<2>(acc, parts, &ctl->ticket[0], red)) return;
  const double interaction = gather_partials(parts, gridDim.x, red);
  const double dx2         = gather_partials(parts + gridDim.x, gridDim.x, red);
  const double dy2         = gather_partials(part_dy2, n_part_dy2, red);
  if (threadIdx.x != 0) return;

  pdhg_step_rule(ctl, interaction, dx2, dy2);
}

// Multi-GPU "gather" transport: rank g also owns ROWS J_g OF THE GLOBAL A^T (n_g x m, all constraint rows as columns), so
// A^T y' on its slice is a complete row sum over the all-gathered y' (yfull: every rank's K2 stores its rows there) —
// no partial products, no reduce-scatter, and per rank exactly 1/G of the single-GPU K3.  Row j is LOCAL to the slice
// (the x / A^T y pointers are offset by the slice start).  Tail: {interaction, ||dx||^2 of the slice, ||dy||^2 of this
// rank's rows} go to the scalar table of every rank; k_step_rule_gather follows.
template <bool INIT, int NPRE>
__global__ void __launch_bounds__(BICSR_THREADS, bicsr_min_ctas(NPRE)) k_transpose_step_slice(pdhg_ctl_t* __restrict__ ctl,
                                                                                        bicsr_view_t AT,
                                                                                        const double* __restrict__ yfull,
                                                                                        const double* __restrict__ xbuf0,
                                                                                        const double* __restrict__ xbuf1,
                                                                                        double* __restrict__ aty0,
                                                                                        double* __restrict__ aty1,
                                                                                        double* __restrict__ parts,
                                                                                        const double* __restrict__ part_dy2,
                                                                                        int n_part_dy2,
                                                                                        const double* __restrict__ t,
                                                                                        const unsigned long long* wait_flags,
                                                                                        int n_wait,
                                                                                        peer_ptrs_t scal_peers,
                                                                                        peer_flags_t flags,
                                                                                        int world,
                                                                                        int rank)
{
  if (!ctl->active) return;
  __shared__ double rows[BICSR_WARPS][BICSR_SLOTS];
  __shared__ double red[32];
  const unsigned long long epoch = (unsigned long long)ctl->attempts + 1ull;
  if (wait_flags) peer_wait(wait_flags, n_wait, epoch);
  const int cur     = ctl->parity;
  const double* x   = cur ? xbuf1 : xbuf0;
  const double* xn  = cur ? xbuf0 : xbuf1;
  const double* aty = cur ? aty1 : aty0;
  double* atyn      = cur ? aty0 : aty1;
  double acc[2]     = {0.0, 0.0};  // interaction, ||dx||^2
  const l2_policy_t pol = make_l2_policies(g_l2_hints);
  struct payload_t {
    double dx, aty, init;
  };
  auto pre_op = [&](int j) {
    payload_t p;
    p.dx   = ld_l2(xn + j, pol.stream) - ld_l2(x + j, pol.stream);
    p.aty  = ld_l2(aty + j, pol.stream);
    p.init = INIT ? ld_l2(t + j, pol.stream) : 0.0;
    return p;
  };
  auto row_op = [&](int j, double s, const payload_t& p) {
    st_l2(atyn + j, s, pol.stream);
    acc[0] += p.dx * (s - p.aty);
    acc[1] += p.dx * p.dx;
  };
  spmv_bicsr_rows<payload_t, INIT, NPRE>(AT, yfull, rows[threadIdx.x >> 5], pre_op, row_op, pol.keep);

  if (!publish_and_elect<2>(acc, parts, &ctl->ticket[0], red)) return;
  const double interaction = gather_partials(parts, gridDim.x, red);
  const double dx2         = gather_partials(parts + gridDim.x, gridDim.x, red);
  const double dy2         = gather_partials(part_dy2, n_part_dy2, red);
  if (threadIdx.x != 0) return;
#pragma unroll
  for (int r = 0; r < DIST_MAX_PEERS; ++r)
    if (r < world) {
      double* o = scal_peers.p[r];
      o[0]      = interaction;
      o[1]      = dx2;
      o[2]      = dy2;
    }
  __threadfence_system();
#pragma unroll
  for (int r = 0; r < DIST_MAX_PEERS; ++r)
    if (r < world) st_release_sys(flags.p[r] + DIST_FLAG_SCALARS + rank, epoch);
}

// Setup of that transport: the rows J_h of the global (scaled) A^T are assembled on rank h from the transposes A_g^T of the
// row blocks, read straight from the peers' memory (rank order = ascending global row index = the order a single-GPU
// transpose gives).  offs / idxs / vals: peer-mapped CSR arrays of every rank's A_g^T (n rows, m_g columns).
struct peer_csr_t {
  const int* off[DIST_MAX_PEERS];
  const int* idx[DIST_MAX_PEERS];
  const double* val[DIST_MAX_PEERS];
  int row0[DIST_MAX_PEERS];  // first global constraint row of every rank
};
__global__ void __launch_bounds__(EW_THREADS) k_slice_row_counts(int rows, int j0, peer_csr_t src, int world, int* __restrict__ cnt)
{
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j <= rows; j += stride) {
    int c = 0;
    if (j < rows) {
#pragma unroll
      for (int g = 0; g < DIST_MAX_PEERS; ++g)
        if (g < world) c += src.off[g][j0 + j + 1] - src.off[g][j0 + j];
    }
    cnt[j] = c;
  }
}
__global__ void __launch_bounds__(EW_THREADS) k_slice_fill(int rows, int j0, peer_csr_t src, int world,
                                                           const int* __restrict__ soff, int* __restrict__ sidx,
                                                           double* __restrict__ sval)
{
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < rows; j += stride) {
    int p = soff[j];
#pragma unroll
    for (int g = 0; g < DIST_MAX_PEERS; ++g)
      if (g < world) {
        const int lo = src.off[g][j0 + j], hi = src.off[g][j0 + j + 1];
        for (int e = lo; e < hi; ++e, ++p) {
          sidx[p] = src.idx[g][e] + src.row0[g];
          sval[p] = src.val[g][e];
        }
      }
  }
}

// Packed exchange of the gather transport: a rank reads only the entries of xbar (y') whose column (row) occurs in its rows
// of A (of A^T) — 1 - exp(-nnz_g / n) of them for uniformly random columns, 63 % at 8 ranks of configs[3] — so only those
// travel, into a buffer indexed by RANK AMONG THE NEEDED ENTRIES (ascending, so row entries stay sorted).
__global__ void __launch_bounds__(EW_THREADS) k_mark_indices(int nnz, const int* __restrict__ idx, int* __restrict__ flag)
{
  const int stride = gridDim.x * blockDim.x;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride) flag[idx[e]] = 1;
}
__global__ void __launch_bounds__(EW_THREADS) k_fill_int(int n, int* __restrict__ v, int value)
{
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) v[i] = value;
}
// Two halves.  The packed buffer of a rank holds first the needed entries that lie in the FIRST half of their owner's slice
// (slots [0, count A)), then, from slot W on, those of the second halves: the column blocks of the gather-blocked products
// are cut at W, so the pass over block 0 needs only the first halves — which the owners send first — and runs while the
// second halves are still on the wire.  owner h holds entries [start[h], start[h + 1]), its first half is the first half[h].
struct half_map_t {
  int start[DIST_MAX_PEERS + 1];
  int half[DIST_MAX_PEERS];
  int world;
};
__global__ void __launch_bounds__(EW_THREADS) k_half_flags(int n, const int* __restrict__ needed, half_map_t hm,
                                                           int* __restrict__ flag_a, int* __restrict__ flag_b)
{
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
    int h = 0;
#pragma unroll
    for (int r = 1; r < DIST_MAX_PEERS; ++r)
      if (r < hm.world && j >= hm.start[r]) h = r;
    const bool first = (j - hm.start[h]) < hm.half[h];
    const int need   = needed[j];
    flag_a[j]        = (need && first) ? 1 : 0;
    flag_b[j]        = (need && !first) ? 1 : 0;
  }
}
// pos[j] = slot of entry j in the packed buffer, -1 when it is not needed (scan_* = exclusive sums of flag_*)
__global__ void __launch_bounds__(EW_THREADS) k_packed_positions(int n, const int* __restrict__ flag_a, const int* __restrict__ scan_a,
                                                                 const int* __restrict__ flag_b, const int* __restrict__ scan_b,
                                                                 int second_half_base, int* __restrict__ pos)
{
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride)
    pos[j] = flag_a[j] ? scan_a[j] : flag_b[j] ? second_half_base + scan_b[j] : -1;
}
// sender side: list of the local entries a destination reads, ascending (flag = its slot table >= 0, scan = exclusive sum)
__global__ void __launch_bounds__(EW_THREADS) k_flag_nonnegative(int n, const int* __restrict__ v, int* __restrict__ flag)
{
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) flag[i] = v[i] >= 0 ? 1 : 0;
}
__global__ void __launch_bounds__(EW_THREADS) k_fill_list(int n, const int* __restrict__ flag, const int* __restrict__ scan,
                                                          int* __restrict__ list)
{
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    if (flag[i]) list[scan[i]] = i;
}

// The exchange itself, as its own kernel on the communication stream (it overlaps the first column-block pass of the
// consumer, see pdlp_solver.cu enqueue_gather_attempt): for every destination rank, its slots in DESTINATION order — thread k
// stores v[list[k]] into slot base + k, warps aligned to 256-byte segments of the destination, so the NVLink stores are
// full contiguous lines (stores issued in SOURCE order by the producing kernel hit every destination with ragged ~20-of-32
// lane runs, which use the link far less efficiently than full lines).  First halves of all
// destinations, flag A, second halves, flag B.  Destinations are visited starting after the sender's own rank.
constexpr int SEND_UNROLL = 8;
struct send_plan_t {
  int count_a[DIST_MAX_PEERS];  // entries of the first half that destination r reads
  int count[DIST_MAX_PEERS];    // all entries it reads (the list holds the first-half ones first)
};
__global__ void __launch_bounds__(EW_THREADS, 8) k_send_packed(const pdhg_ctl_t* __restrict__ ctl,
                                                               const double* __restrict__ v0,
                                                               const double* __restrict__ v1,
                                                               int pick_candidate,  // 1: v = parity ? v0 : v1 (the candidate y')
                                                               const int* __restrict__ list,  // [world][stride]
                                                               const int* __restrict__ slot,  // [world][stride]: slot of entry i at rank r
                                                               int stride,
                                                               send_plan_t plan,
                                                               peer_ptrs_t peers,
                                                               peer_flags_t flags,
                                                               int world,
                                                               int rank,
                                                               int flag_a,
                                                               int flag_b,
                                                               unsigned* __restrict__ tickets)
{
  if (!ctl->active) return;
  const unsigned long long epoch = (unsigned long long)ctl->attempts + 1ull;
  const double* v   = pick_candidate ? (ctl->parity ? v0 : v1) : v0;
  const int gstride = gridDim.x * blockDim.x;
  const int gtid    = blockIdx.x * blockDim.x + threadIdx.x;
  for (int part = 0; part < 2; ++part) {
    for (int d = 0; d < world; ++d) {
      int r = rank + 1 + d;
      if (r >= world) r -= world;
      int lo = 0, hi = 0;
      double* dst = peers.p[0];
#pragma unroll
      for (int q = 0; q < DIST_MAX_PEERS; ++q)
        if (q == r) {
          lo  = part ? plan.count_a[q] : 0;
          hi  = part ? plan.count[q] : plan.count_a[q];
          dst = peers.p[q];
        }
      if (hi <= lo) continue;
      const int* lst  = list + (size_t)r * stride;
      const int* slt  = slot + (size_t)r * stride;
      const int base  = __ldg(slt + __ldg(lst + lo));  // slots of a half are consecutive from here
      const int shift = base & 31;
      const int total = hi - lo + shift;
      // few CTAs (the SpMV kernels keep almost the whole GPU): SEND_UNROLL independent list -> value chains per thread
      for (int t0 = gtid; t0 < total; t0 += gstride * SEND_UNROLL) {
        int src[SEND_UNROLL];
        double val[SEND_UNROLL];
#pragma unroll
        for (int u = 0; u < SEND_UNROLL; ++u) {
          const int k = t0 + u * gstride - shift;
          src[u]      = (k >= 0 && k < hi - lo) ? __ldg(lst + lo + k) : -1;
        }
#pragma unroll
        for (int u = 0; u < SEND_UNROLL; ++u) val[u] = src[u] >= 0 ? v[src[u]] : 0.0;
#pragma unroll
        for (int u = 0; u < SEND_UNROLL; ++u)
          if (src[u] >= 0) dst[base + t0 + u * gstride - shift] = val[u];
      }
    }
    peer_signal_grid_done(tickets + part, flags, world, (part ? flag_b : flag_a) + rank, epoch);
    __syncthreads();
  }
}
__global__ void __launch_bounds__(EW_THREADS) k_remap_indices(int nnz, const int* __restrict__ idx_in, const int* __restrict__ pos,
                                                              int* __restrict__ idx_out)
{
  const int stride = gridDim.x * blockDim.x;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += stride) idx_out[e] = pos[idx_in[e]];
}

// ---------------------------------------------------------------------------------------------
// Row-sharded (multi-GPU) K3 of the NCCL transport.  Each rank owns a block of rows of A; A_g^T y'_g is a PARTIAL
// A^T y' over all n columns that the reduce-scatter sums over ranks into the slice owners (k_interaction_slice).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(BICSR_THREADS, BICSR_MIN_CTAS) k_transpose_partial(const pdhg_ctl_t* __restrict__ ctl,
                                                                                     bicsr_view_t AT,
                                                                                     const double* __restrict__ ybuf0,
                                                                                     const double* __restrict__ ybuf1,
                                                                                     double* __restrict__ buf)
{
  if (!ctl->active) return;
  __shared__ double rows[BICSR_WARPS][BICSR_SLOTS];
  const double* yn = ctl->parity ? ybuf0 : ybuf1;
  struct payload_t {};
  auto pre_op = [&](int) { return payload_t{}; };
  auto row_op = [&](int j, double s, const payload_t&) { buf[j] = s; };
  spmv_bicsr_rows<payload_t>(AT, yn, rows[threadIdx.x >> 5], pre_op, row_op, make_l2_policies(g_l2_hints).keep);
}
// buf[slot] = sum of `count` per-CTA partials (one CTA, fixed order)
__global__ void __launch_bounds__(EW_THREADS) k_sum_partials(const double* __restrict__ parts,
                                                             int count,
                                                             int n_quantities,
                                                             double* __restrict__ out)
{
  __shared__ double red[32];
  for (int q = 0; q < n_quantities; ++q) {
    double s = 0.0;
    for (int i = threadIdx.x; i < count; i += blockDim.x) s += parts[q * count + i];
    s = block_reduce(s, red);
    if (threadIdx.x == 0) out[q] = s;
  }
}

// ---------------------------------------------------------------------------------------------
// Column-sliced multi-GPU attempt (SURVEY §8e scheme (ii)): rank g owns rows R_g of A AND the slice
// J_g = [g*nslice, (g+1)*nslice) of every primal vector.  Two transports.
// gather (default): rank g also owns the rows J_g of the global A^T, so both products take all-gathered inputs and
// there are no partial products.  The producing kernels store what each rank reads into its packed buffers
// themselves (NVLink peer stores that overlap the work; flags replace the collectives, no NCCL in the loop):
//   K1s   primal step on J_g; xbar entries -> the ranks that read them   (k_primal_step_bcast)
//   K2    dual step on R_g over the packed xbar; y' entries -> the ranks that read them   (k_dual_step<..., true>)
//   K3s   A^T y' on J_g over the all-gathered y', interaction / movement partial sums   (k_transpose_step_slice)
//   rule  three scalars from every rank, summed in rank order -> identical accept/reject everywhere
// Flags are monotone epochs (= attempt number), written with st.release.sys by the last CTA of the producer
// after every CTA fenced its stores system-wide; consumers poll with ld.acquire.sys and read the payload
// with ld.global.cg (L2 is the coherence point for peer writes).
// nccl (selectable, and the fallback when the GPUs cannot map each other's memory): NCCL collectives between the kernels
//   K1s   primal step on J_g; xbar slice -> every rank           (all-gather)
//   K2    dual step on R_g (needs the full xbar)
//   K3p   partial A_g^T y'_g over all n columns -> slice owners  (reduce-scatter)
//   K3s   interaction / movement partial sums on J_g             (k_interaction_slice)
//   rule  three scalars from every rank, summed over the ranks   (all-reduce)
// ---------------------------------------------------------------------------------------------
// K1s with the xbar exchange fused in: pointers are already offset to this rank's slice; send[r * send_stride + j] = slot
// of x_j in rank r's packed xbar (xbar_peers.p[r]), -1 if rank r never reads it.
__global__ void __launch_bounds__(EW_THREADS) k_primal_step_bcast(pdhg_ctl_t* __restrict__ ctl,
                                                                  int nloc,
                                                                  double* __restrict__ xbuf0,
                                                                  double* __restrict__ xbuf1,
                                                                  const double* __restrict__ aty0,
                                                                  const double* __restrict__ aty1,
                                                                  const double* __restrict__ c,
                                                                  const double* __restrict__ l,
                                                                  const double* __restrict__ u,
                                                                  double* __restrict__ sum_x,
                                                                  peer_ptrs_t xbar_peers,
                                                                  peer_flags_t flags,
                                                                  int world,
                                                                  int rank,
                                                                  const int* __restrict__ send,
                                                                  int send_stride)
{
  if (!ctl->active) return;
  const unsigned long long epoch = (unsigned long long)ctl->attempts + 1ull;
  const int cur      = ctl->parity;
  const double* x    = cur ? xbuf1 : xbuf0;
  double* xn         = cur ? xbuf0 : xbuf1;
  const double* aty  = cur ? aty1 : aty0;
  const double tau   = ctl->tau;
  const bool pending = ctl->pending_avg != 0;
  const double w     = ctl->pending_weight;
  const int stride   = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nloc; j += stride) {
    const double xj = x[j];
    if (pending) sum_x[j] = sum_x[j] + w * xj;
    const double gradient = ld_stream(c + j) - aty[j];
    double next           = xj - (tau * gradient);
    next                  = fmax(fmin(next, ld_stream(u + j)), ld_stream(l + j));
    xn[j]                 = next;
    const double xb       = next - xj + next;
#pragma unroll
    for (int r = 0; r < DIST_MAX_PEERS; ++r)
      if (r < world) {
        const int d = __ldg(send + (size_t)r * send_stride + j);
        if (d >= 0) xbar_peers.p[r][d] = xb;
      }
  }
  peer_signal_grid_done(&ctl->ticket[1], flags, world, DIST_FLAG_XBAR + rank, epoch, DIST_FLAG_XBAR_B + rank);
}

// K3s (NCCL transport): A^T y' on this rank's slice = the reduce-scatter output src, then the slice's share of the
// interaction and ||dx||^2; the last CTA writes {interaction, ||dx||^2, ||dy||^2 of this rank's rows} to scal[0..3),
// which the all-reduce sums over the ranks before k_step_rule_gather.
__global__ void __launch_bounds__(EW_THREADS) k_interaction_slice(pdhg_ctl_t* __restrict__ ctl,
                                                                  int nloc,
                                                                  const double* __restrict__ src,
                                                                  const double* __restrict__ xbuf0,
                                                                  const double* __restrict__ xbuf1,
                                                                  double* __restrict__ aty0,
                                                                  double* __restrict__ aty1,
                                                                  double* __restrict__ parts,
                                                                  const double* __restrict__ part_dy2,
                                                                  int n_part_dy2,
                                                                  double* __restrict__ scal)
{
  if (!ctl->active) return;
  __shared__ double red[32];
  const int cur     = ctl->parity;
  const double* x   = cur ? xbuf1 : xbuf0;
  const double* xn  = cur ? xbuf0 : xbuf1;
  const double* aty = cur ? aty1 : aty0;
  double* atyn      = cur ? aty0 : aty1;
  double acc[2]     = {0.0, 0.0};
  const int stride  = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nloc; j += stride) {
    double s = 0.0;  // a sum from +0.0, not a copy: -0.0 becomes +0.0, and the iterates depend on the sign of a zero
    s += __ldcg(src + j);
    atyn[j]        = s;
    const double d = xn[j] - x[j];
    acc[0] += d * (s - aty[j]);
    acc[1] += d * d;
  }
  if (!publish_and_elect<2>(acc, parts, &ctl->ticket[0], red)) return;
  const double interaction = gather_partials(parts, gridDim.x, red);
  const double dx2         = gather_partials(parts + gridDim.x, gridDim.x, red);
  const double dy2         = gather_partials(part_dy2, n_part_dy2, red);
  if (threadIdx.x != 0) return;
  scal[0] = interaction;
  scal[1] = dx2;
  scal[2] = dy2;
}

// Step rule from the n_src scalar triples (rank order).  One warp.
__global__ void k_step_rule_gather(pdhg_ctl_t* __restrict__ ctl, const double* __restrict__ scal, int n_src,
                                   const unsigned long long* wait_flags)
{
  if (!ctl->active) return;
  if (wait_flags) peer_wait(wait_flags, n_src, (unsigned long long)ctl->attempts + 1ull);
  if (threadIdx.x != 0) return;
  double interaction = 0.0, dx2 = 0.0, dy2 = 0.0;
  for (int g = 0; g < n_src; ++g) {
    interaction += __ldcg(scal + 4 * g + 0);
    dx2 += __ldcg(scal + 4 * g + 1);
    dy2 += __ldcg(scal + 4 * g + 2);
  }
  pdhg_step_rule(ctl, interaction, dx2, dy2);
}

// ---------------------------------------------------------------------------------------------
// Gather blocking (large LPs).  When the vector an SpMV gathers from is much larger than what stays in L2 (80 MB at
// configs[3], against an L2 that also sees ~2 GB of streams per kernel), the fused kernels turn DRAM-bound well above
// their algorithmic bytes: every gathered double drags a 32-byte sector in from HBM.  The host then splits the matrix by COLUMN blocks whose slice of the gathered vector is L2-sized (csr_transpose.cu),
// and K2 / K3 become   (B - 1) x k_block_pass (t += A_b * x, payload-free)  +  the fused kernel on the LAST block with
// INIT = true (its row sums start from t, its row epilogue is the step's).  Rows keep their entry order inside and across
// blocks; the result is t_0 + t_1 + ... in block order.
// ---------------------------------------------------------------------------------------------
// t[r] = (first ? 0 : t[r]) + sum over the entries of row r in this column block.
//   pick_candidate = 0: x = x0;  1: x = the candidate dual y' = parity ? x0 : x1  (K3).
//   wait_flags: gather transport only, first pass of K2 / K3 (the other ranks' xbar / y' entries must have landed).
template <int FMT = 0>
__global__ void __launch_bounds__(BICSR_THREADS, BICSR_MIN_CTAS) k_block_pass(const pdhg_ctl_t* __restrict__ ctl,
                                                                              bicsr_view_t Ab,
                                                                              const double* __restrict__ x0,
                                                                              const double* __restrict__ x1,
                                                                              int pick_candidate,
                                                                              double* __restrict__ t,
                                                                              int first,
                                                                              const unsigned long long* wait_flags,
                                                                              int n_wait)
{
  if (!ctl->active) return;
  __shared__ double rows[BICSR_WARPS][BICSR_SLOTS];
  if (wait_flags) peer_wait(wait_flags, n_wait, (unsigned long long)ctl->attempts + 1ull);
  const double* x       = pick_candidate ? (ctl->parity ? x0 : x1) : x0;
  const l2_policy_t pol = make_l2_policies(g_l2_hints);
  struct payload_t {
    double init;
  };
  auto pre_op = [&](int r) {
    payload_t p;
    p.init = first ? 0.0 : ld_l2(t + r, pol.stream);
    return p;
  };
  auto row_op = [&](int r, double s, const payload_t&) { st_l2(t + r, s, pol.stream); };
  spmv_bicsr_rows<payload_t, true, 1, FMT>(Ab, x, rows[threadIdx.x >> 5], pre_op, row_op, pol.keep);
}

// Applies a still-pending running-average update (end of a batch, before averages are formed).
__global__ void __launch_bounds__(EW_THREADS) k_flush_average(const pdhg_ctl_t* __restrict__ ctl,
                                                              int n,
                                                              const double* __restrict__ xbuf0,
                                                              const double* __restrict__ xbuf1,
                                                              double* __restrict__ sum_x,
                                                              int m,
                                                              const double* __restrict__ ybuf0,
                                                              const double* __restrict__ ybuf1,
                                                              double* __restrict__ sum_y)
{
  if (!ctl->pending_avg) return;
  const int cur    = ctl->parity;
  const double* x  = cur ? xbuf1 : xbuf0;
  const double* y  = cur ? ybuf1 : ybuf0;
  const double w   = ctl->pending_weight;
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) sum_x[j] = sum_x[j] + w * x[j];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) sum_y[i] = sum_y[i] + w * y[i];
}
__global__ void k_clear_pending(pdhg_ctl_t* ctl) { ctl->pending_avg = 0; }
// take_step starts from set_valid_step_size(0) (pdlp.cu:1191): a batch that follows a zero-movement step tries again, so
// the iteration count keeps advancing and the next termination test can answer Optimal / NumericalError (pdlp.cu:780-789)
__global__ void k_begin_batch(pdhg_ctl_t* ctl, int steps)
{
  ctl->target = ctl->accepted + steps;
  ctl->valid  = 0;
  ctl->active = steps > 0 ? 1 : 0;
}

// Plain y = A x on the row-block scheme (A^T y after a restart to the average, pdhg.cu:120-134).
__global__ void __launch_bounds__(BICSR_THREADS, BICSR_MIN_CTAS) k_spmv(bicsr_view_t A,
                                                                        const double* __restrict__ x,
                                                                        double* __restrict__ out)
{
  __shared__ double rows[BICSR_WARPS][BICSR_SLOTS];
  struct payload_t {};
  auto pre_op = [&](int) { return payload_t{}; };
  auto row_op = [&](int i, double s, const payload_t&) { out[i] = s; };
  spmv_bicsr_rows<payload_t>(A, x, rows[threadIdx.x >> 5], pre_op, row_op, make_l2_policies(g_l2_hints).keep);
}

// Products of the termination evaluation, current and average iterate in ONE stream of the (unscaled) matrix:
//   out_u = M u, out_v = M v  (first),   out_u += M u, out_v += M v  (otherwise).
// A gather-blocked matrix runs one launch per column block, in block order (first = block 0): the sums of a row come out in
// the order of k_block_pass.  An unblocked matrix is one first pass, whose sums are exactly k_spmv's.
template <int FMT = 0>
__global__ void __launch_bounds__(BICSR_THREADS, BICSR_MIN_CTAS) k_spmv_pair(bicsr_view_t M,
                                                                             const double* __restrict__ u,
                                                                             const double* __restrict__ v,
                                                                             double* __restrict__ out_u,
                                                                             double* __restrict__ out_v,
                                                                             int first)
{
  __shared__ double rows[2][BICSR_WARPS][BICSR_SLOTS];
  auto row_op = [&](int r, double su, double sv) {
    out_u[r] = first ? su : out_u[r] + su;
    out_v[r] = first ? sv : out_v[r] + sv;
  };
  const int w = threadIdx.x >> 5;
  spmv_bicsr_rows_pair<FMT>(M, u, v, rows[0][w], rows[1][w], row_op, make_l2_policies(g_l2_hints).keep);
}

// =============================================================================================
// Termination evaluation on the UNSCALED problem, current and average iterate in ONE pass over A and
// one over A^T (convergence_information.cu:150-422, termination_strategy.cu:117-250).
// =============================================================================================
// utils.cuh:205-219
__device__ __forceinline__ double bound_value_product(double value, double lower, double upper)
{
  double bound = 0.0;
  if (value > 0.0) bound = lower;
  else if (value < 0.0) bound = upper;
  return isfinite(bound) ? value * bound : 0.0;
}

// Per-column part of the evaluation, for the current (v = 0) and the average (v = 1) iterate; s[v] = (A^T y_v)_j.
// acc layout: {||g - rc||^2, rc-part of the dual objective, c.x, ||x||^2} x {cur, avg}
__device__ __forceinline__ void eval_column(int j, const double (&s)[2], double cj, double lo, double hi,
                                            const double (&xv)[2], int reduced_cost_rule, double* __restrict__ rc_cur,
                                            double* __restrict__ rc_avg, double (&acc)[8])
{
  double* rcs[2] = {rc_cur, rc_avg};
#pragma unroll
  for (int v = 0; v < 2; ++v) {
    const double g     = cj - s[v];
    const double bound = g > 0.0 ? lo : hi;  // utils.cuh:196-202
    double rc;
    if (g == 0.0) rc = g;
    else if (reduced_cost_rule ? (fabs(xv[v] - bound) <= fabs(xv[v])) : isfinite(bound)) rc = g;  // :222-239
    else rc = 0.0;
    rcs[v][j]      = rc;
    const double r = g - rc;
    acc[v] += r * r;
    acc[2 + v] += bound_value_product(rc, lo, hi);
    acc[4 + v] += xv[v] * cj;
    acc[6 + v] += xv[v] * xv[v];
  }
}

// Final scalars of the evaluation, run by the last CTA of the column pass (all its threads enter).
// parts: 8 x gridDim.x column partials; parts_rows: 6 x n_parts_rows row partials
// ({viol^2, y-part of the dual objective, ||y||^2} x {cur, avg}).
// max of `count` published partials (all >= 0 or seeded with 0); result in all threads
__device__ __forceinline__ double gather_partials_max(const double* parts, int count, double* red)
{
  double s = 0.0;
  for (int i = threadIdx.x; i < count; i += blockDim.x) s = fmax(s, __ldcg(parts + i));
  return block_reduce<true>(s, red);
}

// max_cols: 2 x gridDim.x column maxima, max_rows: 2 x n_max_rows row maxima (per_constraint_residual), else nullptr
__device__ __forceinline__ void eval_finalize(pdhg_ctl_t* ctl, const double* parts, const double* parts_rows,
                                              int n_parts_rows, const eval_consts_t& k, eval_t* out, double* red,
                                              const double* max_cols = nullptr, const double* max_rows = nullptr,
                                              int n_max_rows = 0)
{
  double tot[14];
  for (int q = 0; q < 8; ++q) tot[q] = gather_partials(parts + q * gridDim.x, gridDim.x, red);
  for (int q = 0; q < 6; ++q) tot[8 + q] = gather_partials(parts_rows + q * n_parts_rows, n_parts_rows, red);
  double linf_p[2] = {0.0, 0.0}, linf_d[2] = {0.0, 0.0};
  if (k.per_constraint_residual && max_cols != nullptr && max_rows != nullptr) {
    for (int v = 0; v < 2; ++v) {
      linf_d[v] = gather_partials_max(max_cols + v * gridDim.x, gridDim.x, red);
      linf_p[v] = gather_partials_max(max_rows + v * n_max_rows, n_max_rows, red);
    }
  }
  if (threadIdx.x != 0) return;
  const double pw = ctl->primal_weight;
  for (int v = 0; v < 2; ++v) {
    eval_t e;
    e.l2_primal_residual = sqrt(tot[8 + v]);
    e.l2_dual_residual   = sqrt(tot[v]);
    double p             = tot[4 + v];
    double dobj          = tot[8 + 2 + v] + tot[2 + v];
    if (k.objective_scaling_factor != 1.0 || k.objective_offset != 0.0) {
      p    = k.objective_scaling_factor * p + k.objective_offset;
      dobj = k.objective_scaling_factor * dobj + k.objective_offset;
    }
    e.primal_objective   = p;
    e.dual_objective     = dobj;
    e.gap                = fabs(p - dobj);
    e.abs_objective      = fabs(p) + fabs(dobj);
    e.l2_primal_variable = sqrt(tot[6 + v]);
    e.l2_dual_variable   = sqrt(tot[8 + 4 + v]);
    // termination_strategy.cu:117-250 (l2 criteria)
    const bool gap_ok    = e.gap <= k.abs_gap_tol + k.rel_gap_tol * e.abs_objective;
    bool primal_ok = e.l2_primal_residual <= k.abs_primal_tol + k.rel_primal_tol * k.l2_norm_b;
    bool dual_ok   = e.l2_dual_residual <= k.abs_dual_tol + k.rel_dual_tol * k.l2_norm_c;
    e.linf_relative_primal_residual = linf_p[v];
    e.linf_relative_dual_residual   = linf_d[v];
    if (k.per_constraint_residual) {  // termination_strategy.cu:141-166: absolute tolerance only
      primal_ok = linf_p[v] <= k.abs_primal_tol;
      dual_ok   = linf_d[v] <= k.abs_dual_tol;
    }
    e.status             = (dual_ok && primal_ok && gap_ok) ? 1 : (primal_ok ? 7 : 6);
    // pdlp_restart_strategy.cu:367-380
    const double w2 = pw * pw;
    e.kkt = sqrt(w2 * e.l2_primal_residual * e.l2_primal_residual + e.l2_dual_residual * e.l2_dual_residual / w2 +
                 e.gap * e.gap);
    e.pad  = 0;
    out[v] = e;
  }
}

// Row math of the evaluation on precomputed products ax_cur = A x_cur, ax_avg = A x_avg (element-wise).
// parts layout: 6 x gridDim.x = {viol^2, y-part of dual objective, ||y||^2} x {cur, avg}
__global__ void __launch_bounds__(EW_THREADS) k_eval_rows_from_ax(int m,
                                                                  const double* __restrict__ ax_cur,
                                                                  const double* __restrict__ ax_avg,
                                                                  const double* __restrict__ y_cur,
                                                                  const double* __restrict__ y_avg,
                                                                  const double* __restrict__ lc,
                                                                  const double* __restrict__ uc,
                                                                  double* __restrict__ parts,
                                                                  double rel_primal_tol,
                                                                  double* __restrict__ parts_max)  // 2 x gridDim.x or null
{
  __shared__ double red[32];
  double acc[6]    = {0, 0, 0, 0, 0, 0};
  double mx[2]     = {0.0, 0.0};  // per_constraint_residual: max_i (violation_i - rel * b_i), seeded with 0
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
    const double lo = lc[i], hi = uc[i];
    const double s[2]  = {__ldcs(ax_cur + i), __ldcs(ax_avg + i)};
    const double yv[2] = {y_cur[i], y_avg[i]};
    // combine_finite_abs_bounds (utils.cuh:140-148)
    const double b = fmax(isfinite(lo) ? fabs(lo) : 0.0, isfinite(hi) ? fabs(hi) : 0.0);
#pragma unroll
    for (int v = 0; v < 2; ++v) {
      const double viol = s[v] < lo ? lo - s[v] : (s[v] > hi ? s[v] - hi : 0.0);  // utils.cuh:166-178
      acc[v] += viol * viol;
      acc[2 + v] += bound_value_product(yv[v], lo, hi);
      acc[4 + v] += yv[v] * yv[v];
      mx[v] = fmax(mx[v], viol - rel_primal_tol * b);
    }
  }
#pragma unroll
  for (int q = 0; q < 6; ++q) {
    const double t = block_reduce(acc[q], red);
    if (threadIdx.x == 0) parts[q * gridDim.x + blockIdx.x] = t;
  }
  if (parts_max != nullptr) {
#pragma unroll
    for (int v = 0; v < 2; ++v) {
      const double t = block_reduce<true>(mx[v], red);
      if (threadIdx.x == 0) parts_max[v * gridDim.x + blockIdx.x] = t;
    }
  }
}
// out[v] = max over `count` per-CTA maxima (one CTA); the row-sharded evaluation all-reduces them with MAX
__global__ void __launch_bounds__(EW_THREADS) k_max_partials(const double* __restrict__ parts, int count, int n_quantities,
                                                             double* __restrict__ out)
{
  __shared__ double red[32];
  for (int q = 0; q < n_quantities; ++q) {
    const double t = gather_partials_max(parts + q * count, count, red);
    if (threadIdx.x == 0) out[q] = t;
  }
}

// Column math of the evaluation on precomputed A^T y (current, average; all-reduced in the row-sharded mode) + final scalars.
// parts layout: 8 x gridDim.x = {||g - rc||^2, rc-part of dual objective, c.x, ||x||^2} x {cur, avg}
__global__ void __launch_bounds__(EW_THREADS) k_eval_cols_from_aty(pdhg_ctl_t* __restrict__ ctl,
                                                                   int n,
                                                                   const double* __restrict__ aty_cur,
                                                                   const double* __restrict__ aty_avg,
                                                                   const double* __restrict__ x_cur,
                                                                   const double* __restrict__ x_avg,
                                                                   const double* __restrict__ c,
                                                                   const double* __restrict__ l,
                                                                   const double* __restrict__ u,
                                                                   double* __restrict__ rc_cur,
                                                                   double* __restrict__ rc_avg,
                                                                   double* __restrict__ parts,
                                                                   const double* __restrict__ parts_rows,
                                                                   int n_parts_rows,
                                                                   eval_consts_t k,
                                                                   eval_t* __restrict__ out,
                                                                   double* __restrict__ parts_max,  // 2 x gridDim.x or null
                                                                   const double* __restrict__ max_rows,
                                                                   int n_max_rows)
{
  __shared__ double red[32];
  double acc[8]    = {0, 0, 0, 0, 0, 0, 0, 0};
  double mx[2]     = {0.0, 0.0};  // per_constraint_residual: max_j ((g - rc)_j - rel * c_j), signed (utils.cuh:392-404)
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
    const double s[2]  = {aty_cur[j], aty_avg[j]};
    const double xv[2] = {x_cur[j], x_avg[j]};
    const double cj    = c[j];
    eval_column(j, s, cj, l[j], u[j], xv, k.reduced_cost_rule, rc_cur, rc_avg, acc);
    if (parts_max != nullptr) {
      mx[0] = fmax(mx[0], ((cj - s[0]) - rc_cur[j]) - k.rel_dual_tol * cj);
      mx[1] = fmax(mx[1], ((cj - s[1]) - rc_avg[j]) - k.rel_dual_tol * cj);
    }
  }
  if (parts_max != nullptr) {  // published ahead of the ticket of publish_and_elect (its fence covers these stores)
#pragma unroll
    for (int v = 0; v < 2; ++v) {
      const double t = block_reduce<true>(mx[v], red);
      if (threadIdx.x == 0) parts_max[v * gridDim.x + blockIdx.x] = t;
    }
  }
  if (!publish_and_elect<8>(acc, parts, &ctl->ticket[1], red)) return;
  eval_finalize(ctl, parts, parts_rows, n_parts_rows, k, out, red, parts_max, max_rows, n_max_rows);
}

// ---------------------------------------------------------------------------------------------
// Infeasibility detection (termination_strategy/infeasibility_information.cu:183-223, termination_strategy.cu:229-250):
// the iterate itself is the ray estimate.  Two element-wise passes over the products the evaluation already formed
// (A x and A^T y for the current and the average iterate), launched only when `infeasibility_detection` is set; the
// last CTA of the column pass turns a "keep going" status of k_eval_cols_from_aty into 2 (PrimalInfeasible) or
// 3 (DualInfeasible).
// rows -> parts (6 x gridDim.x): max |violation(Ax; homogeneous bounds)|, max |y|, sum bound_value_product(y) x {cur, avg}
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(EW_THREADS) k_infeasibility_rows(int m,
                                                                   const double* __restrict__ ax_cur,
                                                                   const double* __restrict__ ax_avg,
                                                                   const double* __restrict__ y_cur,
                                                                   const double* __restrict__ y_avg,
                                                                   const double* __restrict__ lc,
                                                                   const double* __restrict__ uc,
                                                                   double* __restrict__ parts)
{
  __shared__ double red[32];
  double hres[2] = {0, 0}, yinf[2] = {0, 0}, dobj[2] = {0, 0};
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
    const double lo = lc[i], hi = uc[i];
    const double hl = isfinite(lo) ? 0.0 : lo, hu = isfinite(hi) ? 0.0 : hi;  // zero_if_is_finite, utils.cuh:256-263
    const double s[2]  = {ax_cur[i], ax_avg[i]};
    const double yv[2] = {y_cur[i], y_avg[i]};
#pragma unroll
    for (int v = 0; v < 2; ++v) {
      const double viol = s[v] < hl ? hl - s[v] : (s[v] > hu ? s[v] - hu : 0.0);
      hres[v] = fmax(hres[v], fabs(viol));
      yinf[v] = fmax(yinf[v], fabs(yv[v]));
      dobj[v] += bound_value_product(yv[v], lo, hi);
    }
  }
#pragma unroll
  for (int v = 0; v < 2; ++v) {
    const double a = block_reduce<true>(hres[v], red);
    const double b = block_reduce<true>(yinf[v], red);
    const double c = block_reduce(dobj[v], red);
    if (threadIdx.x == 0) {
      parts[(0 + v) * gridDim.x + blockIdx.x] = a;
      parts[(2 + v) * gridDim.x + blockIdx.x] = b;
      parts[(4 + v) * gridDim.x + blockIdx.x] = c;
    }
  }
}
// columns -> parts (12 x gridDim.x): max |x|, max bound violation of the ray, max |g - rc|, max |rc| (max), c.x,
// sum bound_value_product(rc) (sum), each x {cur, avg}; g = -A^T y.  Last CTA: compute_remaining_stats_kernel
// (:118-181) + the two tests.  stats_out (nullable; null in the solve) receives INFEAS_STATS doubles per iterate:
// xinf, max_viol, hres, c.x, yinf, rcinf, hdres, dobj, pobj, max_primal, hdres / scaling, dobj / scaling, and the status
// the tests give (2, 3 or 6), for cuOptB200SolverInfeasibilityStats.
constexpr int INFEAS_STATS = 13;
__global__ void __launch_bounds__(EW_THREADS) k_infeasibility_cols(pdhg_ctl_t* __restrict__ ctl,
                                                                   int n,
                                                                   const double* __restrict__ aty_cur,
                                                                   const double* __restrict__ aty_avg,
                                                                   const double* __restrict__ x_cur,
                                                                   const double* __restrict__ x_avg,
                                                                   const double* __restrict__ c,
                                                                   const double* __restrict__ l,
                                                                   const double* __restrict__ u,
                                                                   double* __restrict__ parts,
                                                                   const double* __restrict__ parts_rows,
                                                                   int n_parts_rows,
                                                                   eval_consts_t k,
                                                                   eval_t* __restrict__ out,
                                                                   double* __restrict__ stats_out)
{
  __shared__ double red[32];
  __shared__ bool is_last;
  double mx[8] = {0, 0, 0, 0, 0, 0, 0, 0};  // xinf, max_viol, hdres, rcinf  x {cur, avg}
  double sm[4] = {0, 0, 0, 0};              // c.x, dobj_rc            x {cur, avg}
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
    const double lo = l[j], hi = u[j], cj = c[j];
    const double s[2]  = {aty_cur[j], aty_avg[j]};
    const double xv[2] = {x_cur[j], x_avg[j]};
#pragma unroll
    for (int v = 0; v < 2; ++v) {
      mx[0 + v] = fmax(mx[0 + v], fabs(xv[v]));
      if (isfinite(lo)) mx[2 + v] = fmax(mx[2 + v], -xv[v]);  // utils.cuh:181-193
      if (isfinite(hi)) mx[2 + v] = fmax(mx[2 + v], xv[v]);
      const double g     = -s[v];
      const double bound = g > 0.0 ? lo : hi;
      double rc;
      if (g == 0.0) rc = g;
      else if (k.reduced_cost_rule ? (fabs(xv[v] - bound) <= fabs(xv[v])) : isfinite(bound)) rc = g;
      else rc = 0.0;
      mx[4 + v] = fmax(mx[4 + v], fabs(g - rc));
      mx[6 + v] = fmax(mx[6 + v], fabs(rc));
      sm[0 + v] += xv[v] * cj;
      sm[2 + v] += bound_value_product(rc, lo, hi);
    }
  }
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const double t = block_reduce<true>(mx[q], red);
    if (threadIdx.x == 0) parts[q * gridDim.x + blockIdx.x] = t;
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const double t = block_reduce(sm[q], red);
    if (threadIdx.x == 0) parts[(8 + q) * gridDim.x + blockIdx.x] = t;
  }
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned t = atomicAdd(&ctl->ticket[3], 1u);
    is_last          = (t == gridDim.x - 1);
    if (is_last) ctl->ticket[3] = 0u;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  double cmax[8], csum[4], rmax[4], rsum[2];
  for (int q = 0; q < 8; ++q) cmax[q] = gather_partials_max(parts + q * gridDim.x, gridDim.x, red);
  for (int q = 0; q < 4; ++q) csum[q] = gather_partials(parts + (8 + q) * gridDim.x, gridDim.x, red);
  for (int q = 0; q < 4; ++q) rmax[q] = gather_partials_max(parts_rows + q * n_parts_rows, n_parts_rows, red);
  for (int q = 0; q < 2; ++q) rsum[q] = gather_partials(parts_rows + (4 + q) * n_parts_rows, n_parts_rows, red);
  if (threadIdx.x != 0) return;
  for (int v = 0; v < 2; ++v) {
    if (out[v].status != 6) continue;  // Optimal / PrimalFeasible were decided first (termination_strategy.cu:141-227)
    const double xinf = cmax[0 + v], max_viol = cmax[2 + v], rcinf = cmax[6 + v];
    const double hres = rmax[0 + v], yinf = rmax[2 + v];
    double hdres = cmax[4 + v];
    double pobj  = xinf != 0.0 ? csum[0 + v] * (1.0 / xinf) : 0.0;
    double dobj  = rsum[v] + csum[2 + v];
    const double scaling = fmax(yinf, rcinf);
    if (scaling != 0.0) {
      hdres /= scaling;
      dobj /= scaling;
    } else {
      hdres = 0.0;
      dobj  = 0.0;
    }
    double max_primal;
    if (xinf > 0.0) {
      max_primal = fmax(hres, max_viol) / xinf;
    } else {
      max_primal = 0.0;
      pobj       = 0.0;
    }
    int status = 6;
    if (dobj > 0.0 && hdres / dobj <= k.primal_infeasible_tol) status = 2;
    else if (pobj < 0.0 && max_primal / -pobj <= k.dual_infeasible_tol) status = 3;
    if (status != 6) out[v].status = status;
    if (stats_out != nullptr) {
      const double s[INFEAS_STATS] = {xinf, max_viol, hres, csum[0 + v], yinf, rcinf, cmax[4 + v], rsum[v] + csum[2 + v],
                                      pobj, max_primal, hdres, dobj, (double)status};
      for (int q = 0; q < INFEAS_STATS; ++q) stats_out[v * INFEAS_STATS + q] = s[q];
    }
  }
}

// Averages + in-place unscaling ahead of the evaluation (pdlp.cu:1103-1136,
// weighted_average_solution.cu:114-142, initial_scaling.cu:456-484).
// mode 0: avg := current (k_internal <= 1); mode 1: avg := sum / sum_weights (0 when nothing was summed);
// mode 2: avg untouched (first major iteration of a warm-started solve, pdlp.cu:1100-1129)
__global__ void __launch_bounds__(EW_THREADS) k_average_and_unscale(const pdhg_ctl_t* __restrict__ ctl,
                                                                    int mode,
                                                                    int n,
                                                                    double* __restrict__ v,
                                                                    const double* __restrict__ sum_v,
                                                                    double* __restrict__ avg,
                                                                    const double* __restrict__ scale)
{
  const double sw  = ctl->sum_weights;
  const bool empty = ctl->its_since_restart == 0;
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
    const double vj = v[j];
    const double d  = scale[j];
    if (mode != 2) {
      const double a = mode == 0 ? vj : (empty ? 0.0 : sum_v[j] / sw);
      avg[j]         = a * d;
    }
    v[j] = vj * d;
  }
}
// x /= D with 0 for D == 0 (eltwiseDivideCheckZero; initial_scaling.cu:411-427)
__global__ void __launch_bounds__(EW_THREADS) k_scale_back(int n, double* __restrict__ v, const double* __restrict__ scale)
{
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
    const double d = scale[j];
    v[j]           = d == 0.0 ? 0.0 : v[j] / d;
  }
}

// Primal-weight update from the squared distances to the last restart point (pdlp_restart_strategy.cu:685-732).
__device__ __forceinline__ void update_primal_weight(pdhg_ctl_t* ctl, double dp2, double dd2, double smoothing)
{
  const double pd = sqrt(dp2), dd = sqrt(dd2);
  const double guard = 1.0e-10;
  if (pd < guard || pd >= 1.0 / guard || dd < guard || dd >= 1.0 / guard) return;
  const double lw    = smoothing * log(dd / pd) + (1.0 - smoothing) * log(ctl->primal_weight);
  const double pw    = exp(lw);
  ctl->primal_weight = pw;
  ctl->tau           = ctl->step_size / pw;
  ctl->sigma         = ctl->step_size * pw;
}
// row-sharded mode: distances[0] = primal (replicated), distances[1] = dual (all-reduced)
__global__ void k_update_primal_weight(pdhg_ctl_t* ctl, const double* distances, double smoothing)
{
  update_primal_weight(ctl, distances[0], distances[1], smoothing);
}

// Squared distance of the restart candidate to the last restart point for primal and dual
// (pdlp_restart_strategy.cu:753-801, 1681-1714: plain L2), then the primal-weight update, or — when `distances_out`
// is given (row-sharded mode, the dual part still has to be summed over ranks) — just the two sums.
__global__ void __launch_bounds__(EW_THREADS) k_restart_distance_and_weight(pdhg_ctl_t* __restrict__ ctl,
                                                                            int n,
                                                                            const double* __restrict__ cand_x,
                                                                            const double* __restrict__ last_x,
                                                                            int m,
                                                                            const double* __restrict__ cand_y,
                                                                            const double* __restrict__ last_y,
                                                                            double smoothing,
                                                                            double* __restrict__ parts,
                                                                            double* __restrict__ distances_out)
{
  __shared__ double red[32];
  double acc[2]    = {0.0, 0.0};
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
    const double d = last_x[j] - cand_x[j];
    acc[0] += d * d;
  }
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += stride) {
    const double d = last_y[i] - cand_y[i];
    acc[1] += d * d;
  }
  if (!publish_and_elect<2>(acc, parts, &ctl->ticket[2], red)) return;
  const double dp2 = gather_partials(parts, gridDim.x, red);
  const double dd2 = gather_partials(parts + gridDim.x, gridDim.x, red);
  if (threadIdx.x != 0) return;
  if (distances_out) {
    distances_out[0] = dp2;
    distances_out[1] = dd2;
    return;
  }
  update_primal_weight(ctl, dp2, dd2, smoothing);
}
__global__ void k_reset_after_restart(pdhg_ctl_t* ctl)
{
  ctl->sum_weights       = 0.0;
  ctl->its_since_restart = 0;
  ctl->pending_avg       = 0;
}

// =============================================================================================
// One-time setup kernels: diagonal scaling (initial_scaling.cu:95-408).  A group of W lanes per row; not hot.
// =============================================================================================
// mode 0: out[row] = max |(a * rs[row]) * cs[col]|        (Ruiz, :95-122)
// mode 1: out[row] = sum |(a * rs[row]) * cs[col]|^power  (Pock-Chambolle, :177-252)
// For A^T pass row_scale = variable scaling, col_scale = constraint scaling and `swap_assoc` keeps the
// reference's association (a * constraint_scale) * variable_scale.
// W lanes per row (W = 4, 8, 16 or 32, picked from the average row length: a warp per 8-entry row idles 24 lanes and took
// 3 ms per pass at configs[3], 22 passes per solve); fixed xor tree over the W lanes.
template <int W>
__global__ void __launch_bounds__(256) k_row_scaling_stat(int rows,
                                                          const int* __restrict__ off,
                                                          const int* __restrict__ idx,
                                                          const double* __restrict__ val,
                                                          const double* __restrict__ row_scale,
                                                          const double* __restrict__ col_scale,
                                                          int swap_assoc,
                                                          int mode,
                                                          double power,
                                                          double* __restrict__ out)
{
  const int sub    = threadIdx.x % W;
  const int gpb    = blockDim.x / W;  // row groups per CTA
  const int stride = gridDim.x * gpb;
  // all lanes of a warp run the same number of rounds (the shuffles below need the whole warp)
  const int rounds = (rows + stride - 1) / stride;
  for (int it = 0; it < rounds; ++it) {
    const int r     = it * stride + blockIdx.x * gpb + threadIdx.x / W;
    const bool live = r < rows;
    double acc      = 0.0;
    if (live) {
      const double rs = row_scale[r];
      const int hi    = off[r + 1];
      for (int p = off[r] + sub; p < hi; p += W) {
        const double cs = col_scale[idx[p]];
        const double a  = swap_assoc ? fabs((val[p] * cs) * rs) : fabs((val[p] * rs) * cs);
        if (mode == 0) acc = fmax(acc, a);
        else acc += pow(a, power);
      }
    }
#pragma unroll
    for (int o = W / 2; o > 0; o >>= 1) {
      const double other = __shfl_xor_sync(0xffffffffu, acc, o);
      acc                = mode == 0 ? fmax(acc, other) : acc + other;
    }
    if (live && sub == 0) out[r] = acc;
  }
}
// cum[i] = stat[i] > 0 ? cum[i] / sqrt(stat[i]) : cum[i]   (utils.cuh:123-129)
__global__ void k_apply_scaling_stat(int n, double* __restrict__ cum, const double* __restrict__ stat)
{
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
    const double s = stat[j];
    if (s > 0.0) cum[j] = cum[j] / sqrt(s);
  }
}
// val[p] = val[p] * row_scale[row] * col_scale[col]   (initial_scaling.cu:310-345; same expression for A and A^T)
template <int W>
__global__ void __launch_bounds__(256) k_scale_matrix(int rows,
                                                      const int* __restrict__ off,
                                                      const int* __restrict__ idx,
                                                      double* __restrict__ val,
                                                      const double* __restrict__ row_scale,
                                                      const double* __restrict__ col_scale)
{
  const int sub    = threadIdx.x % W;
  const int gpb    = blockDim.x / W;
  const int stride = gridDim.x * gpb;
  for (int r = blockIdx.x * gpb + threadIdx.x / W; r < rows; r += stride) {
    const double rs = row_scale[r];
    const int hi    = off[r + 1];
    for (int p = off[r] + sub; p < hi; p += W) val[p] = val[p] * rs * col_scale[idx[p]];
  }
}
// op 0: v *= s ; op 1: v = s == 0 ? 0 : v / s
__global__ void k_scale_vector(int n, double* __restrict__ v, const double* __restrict__ s, int op)
{
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
    const double d = s[j];
    v[j]           = op == 0 ? v[j] * d : (d == 0.0 ? 0.0 : v[j] / d);
  }
}
__global__ void k_fill(int n, double* __restrict__ v, double value)
{
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) v[j] = value;
}
__global__ void k_scale_constant(int n, double* __restrict__ v, double a)
{
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) v[j] *= a;
}
// *count += number of positions with lo > hi (problem validation on the device: the arrays are uploaded unchecked)
__global__ void k_count_crossed_bounds(int n, const double* __restrict__ lo, const double* __restrict__ hi, int* __restrict__ count)
{
  const int stride = gridDim.x * blockDim.x;
  int bad          = 0;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) bad += lo[j] > hi[j];
  if (bad) atomicAdd(count, bad);
}
__global__ void k_clamp(int n, double* __restrict__ v, const double* __restrict__ lo, const double* __restrict__ hi)
{
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) v[j] = fmin(fmax(v[j], lo[j]), hi[j]);
}

// Generic deterministic reductions for the setup phase.  kind 0: max |v| ; 1: sum v^2 * w ;
// 2: sum combine_finite_abs_bounds(lo, hi)^2 * w (utils.cuh:140-148).  Single-CTA finish via ticket.
__global__ void __launch_bounds__(EW_THREADS) k_setup_reduce(int kind,
                                                             int n,
                                                             const double* __restrict__ a,
                                                             const double* __restrict__ b,
                                                             double weight,
                                                             double* __restrict__ parts,
                                                             unsigned* __restrict__ ticket,
                                                             double* __restrict__ out)
{
  __shared__ double red[32];
  __shared__ bool is_last;
  double acc       = 0.0;
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
    if (kind == 0) {
      acc = fmax(acc, fabs(a[j]));
    } else if (kind == 1) {
      acc += a[j] * a[j] * weight;
    } else {
      double v = 0.0;
      if (isfinite(b[j])) v = fmax(v, fabs(b[j]));
      if (isfinite(a[j])) v = fmax(v, fabs(a[j]));
      acc += v * v * weight;
    }
  }
  const double t = kind == 0 ? block_reduce<true>(acc, red) : block_reduce<false>(acc, red);
  if (threadIdx.x == 0) {
    parts[blockIdx.x] = t;
    __threadfence();
    is_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    if (is_last) *ticket = 0u;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  double s = 0.0;
  for (int i = threadIdx.x; i < (int)gridDim.x; i += blockDim.x) s = kind == 0 ? fmax(s, __ldcg(parts + i)) : s + __ldcg(parts + i);
  s = kind == 0 ? block_reduce<true>(s, red) : block_reduce<false>(s, red);
  if (threadIdx.x == 0) *out = s;
}

}  // namespace cuopt_b200
