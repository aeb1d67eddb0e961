// Opt-in presolve on the device (settings.presolve) and the matching postsolve; see presolve.cuh and DESIGN.md §8.
//
// A round applies four rules, in this order, to the problem in minimisation form:
//   1. fixed column (l_j = u_j, finite): x_j = l_j is substituted into the row bounds and the column removed;
//   2. empty row (no live entry): infeasible when 0 lies outside [lc_i, uc_i] by more than the tolerance, else removed;
//   3. singleton row a x_j in [lc_i, uc_i]: the implied bounds tighten [l_j, u_j] and the row is removed; each side of a
//      column remembers the row that supplied it (ties: the smallest row index, the first met in A^T's ascending order);
//   4. empty column: x_j goes to the bound c_j favours (the projection of 0 when c_j = 0) and the column is removed; a
//      column whose favoured bound is infinite stays.
// An entry is live when its row and column are alive and its stored value is not zero.  Rounds repeat until one removes
// nothing.  Every kernel is deterministic: per-row and per-column sums run in a fixed lane order, counters are integers.
#include "presolve.cuh"

#include <cmath>
#include <cstdio>

namespace cuopt_b200 {

void csr_transpose_device(int rows, int cols, int nnz, const int* off, const int* idx, const double* val, int* toff,
                          int* tidx, double* tval, cudaStream_t stream);  // csr_transpose.cu
void exclusive_sum_int(int count, const int* in, int* out, cudaStream_t stream);

namespace {

// Each round can only enable reductions next to the ones it made (a fixed column can make a singleton row, a removed
// singleton row an empty column), so real models settle in a handful of rounds; the cap bounds the host round trips on an
// adversarial chain.  Reductions still available at the cap stay in the problem, which is always safe.
constexpr int PRESOLVE_MAX_ROUNDS = 32;

// per-round counters (the one block that comes back to the host)
enum { C_FIXED = 0, C_EMPTY_ROWS, C_SINGLETON_ROWS, C_EMPTY_COLS, C_INFEASIBLE, C_FREE_EMPTY_COLS, C_COUNT = 8 };

constexpr int PS_THREADS = 256;
constexpr int PS_WARPS   = PS_THREADS / 32;

__device__ __forceinline__ int warp_count(int v) { return (int)__reduce_add_sync(0xffffffffu, (unsigned)v); }

// rule 1: columns whose bounds meet become fixed in this round
__global__ void k_ps_fix_columns(int n, int round, const double* __restrict__ l, const double* __restrict__ u,
                                 unsigned char* __restrict__ col_alive, int* __restrict__ fixed_round,
                                 double* __restrict__ x_fix, int* __restrict__ cnt)
{
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
    if (!col_alive[j] || !(l[j] == u[j]) || !isfinite(l[j])) continue;
    col_alive[j]   = 0;
    fixed_round[j] = round;
    x_fix[j]       = l[j];
    atomicAdd(cnt + C_FIXED, 1);
  }
}

// one warp per alive row: shift the row bounds by the columns fixed in this round (row-wise product in CSR order), count
// the live entries, remember the single one of a singleton row, apply rule 2
__global__ void k_ps_rows(int m, int round, const int* __restrict__ off, const int* __restrict__ idx,
                          const double* __restrict__ val, const unsigned char* __restrict__ col_alive,
                          const int* __restrict__ fixed_round, const double* __restrict__ x_fix, double* __restrict__ lc,
                          double* __restrict__ uc, unsigned char* __restrict__ row_alive, int* __restrict__ row_cnt,
                          int* __restrict__ row_col, double tol, int* __restrict__ cnt)
{
  const int lane = threadIdx.x & 31;
  for (int i = blockIdx.x * PS_WARPS + (threadIdx.x >> 5); i < m; i += gridDim.x * PS_WARPS) {
    if (!row_alive[i]) continue;
    double shift = 0.0;
    int live = 0, col = -1;
    for (int p = off[i] + lane; p < off[i + 1]; p += 32) {
      const int j    = idx[p];
      const double a = val[p];
      if (fixed_round[j] == round) shift += a * x_fix[j];
      else if (col_alive[j] && a != 0.0) { ++live; col = j; }
    }
    shift                 = warp_sum(shift);
    const int total       = warp_count(live);
    const unsigned holder = __ballot_sync(0xffffffffu, live > 0);
    const int single      = total == 1 ? __shfl_sync(0xffffffffu, col, __ffs(holder) - 1) : -1;
    if (lane == 0) {
      double lo = lc[i], hi = uc[i];
      if (isfinite(lo)) lo -= shift;
      if (isfinite(hi)) hi -= shift;
      lc[i]      = lo;
      uc[i]      = hi;
      row_cnt[i] = total;
      row_col[i] = single;
      if (total == 0) {
        if (lo > tol || hi < -tol) cnt[C_INFEASIBLE] = 1;
        row_alive[i] = 0;
        atomicAdd(cnt + C_EMPTY_ROWS, 1);
      }
    }
  }
}

// rule 3, one thread per alive column scanning its row of A^T in ascending row order
__global__ void k_ps_singletons(int n, const int* __restrict__ toff, const int* __restrict__ tidx,
                                const double* __restrict__ tval, const unsigned char* __restrict__ col_alive,
                                unsigned char* __restrict__ row_alive, const int* __restrict__ row_cnt,
                                const int* __restrict__ row_col, const double* __restrict__ lc,
                                const double* __restrict__ uc, double* __restrict__ l, double* __restrict__ u,
                                int* __restrict__ src_lo, int* __restrict__ src_hi, double* __restrict__ a_lo,
                                double* __restrict__ a_hi, double tol, int* __restrict__ cnt)
{
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
    if (!col_alive[j]) continue;
    double lj = l[j], uj = u[j];
    int removed = 0;
    for (int p = toff[j]; p < toff[j + 1]; ++p) {
      const int i    = tidx[p];
      const double a = tval[p];
      // a row whose single live entry is (i, j) belongs to this thread alone
      if (a == 0.0 || row_col[i] != j || row_cnt[i] != 1 || !row_alive[i]) continue;
      const double lo = a > 0.0 ? lc[i] / a : uc[i] / a;
      const double hi = a > 0.0 ? uc[i] / a : lc[i] / a;
      if (lo > lj) { lj = lo; src_lo[j] = i; a_lo[j] = a; }
      if (hi < uj) { uj = hi; src_hi[j] = i; a_hi[j] = a; }
      row_alive[i] = 0;
      ++removed;
    }
    if (removed == 0) continue;
    if (lj > uj + tol) cnt[C_INFEASIBLE] = 1;
    else if (lj > uj) uj = lj;
    l[j] = lj;
    u[j] = uj;
    atomicAdd(cnt + C_SINGLETON_ROWS, removed);
  }
}

// rule 4, one warp per alive column
__global__ void k_ps_columns(int n, const int* __restrict__ toff, const int* __restrict__ tidx,
                             const double* __restrict__ tval, const unsigned char* __restrict__ row_alive,
                             unsigned char* __restrict__ col_alive, const double* __restrict__ c,
                             const double* __restrict__ l, const double* __restrict__ u, double* __restrict__ x_fix,
                             int* __restrict__ cnt)
{
  const int lane = threadIdx.x & 31;
  for (int j = blockIdx.x * PS_WARPS + (threadIdx.x >> 5); j < n; j += gridDim.x * PS_WARPS) {
    if (!col_alive[j]) continue;
    int live = 0;
    for (int p = toff[j] + lane; p < toff[j + 1]; p += 32) live += (row_alive[tidx[p]] && tval[p] != 0.0) ? 1 : 0;
    if (warp_count(live) != 0 || lane != 0) continue;
    const double cj = c[j];
    const double v  = cj > 0.0 ? l[j] : cj < 0.0 ? u[j] : fmin(fmax(0.0, l[j]), u[j]);
    if (isfinite(v)) {
      x_fix[j]     = v;
      col_alive[j] = 0;
      atomicAdd(cnt + C_EMPTY_COLS, 1);
    } else {
      atomicAdd(cnt + C_FREE_EMPTY_COLS, 1);
    }
  }
}

// sum of c_j x_fix_j over the removed columns: fixed-shape two-pass reduction
__global__ void k_ps_offset_partial(int n, const unsigned char* __restrict__ col_alive, const double* __restrict__ c,
                                    const double* __restrict__ x_fix, double* __restrict__ part)
{
  __shared__ double scratch[32];
  double s = 0.0;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x)
    if (!col_alive[j]) s += c[j] * x_fix[j];
  s = block_reduce(s, scratch);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}
__global__ void k_ps_offset_final(int parts, const double* __restrict__ part, double* __restrict__ out)
{
  __shared__ double scratch[32];
  double s = 0.0;
  for (int q = threadIdx.x; q < parts; q += blockDim.x) s += part[q];
  s = block_reduce(s, scratch);
  if (threadIdx.x == 0) *out = s;
}

__global__ void k_ps_flags(int count, const unsigned char* __restrict__ alive, int* __restrict__ out)
{
  const int stride = gridDim.x * blockDim.x;
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q <= count; q += stride) out[q] = q < count ? alive[q] : 0;
}
__global__ void k_ps_map(int count, const unsigned char* __restrict__ alive, const int* __restrict__ pos,
                         int* __restrict__ map)
{
  const int stride = gridDim.x * blockDim.x;
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < count; q += stride)
    if (alive[q]) map[pos[q]] = q;
}
// kept entries per kept row (slot m1 stays 0: the scan total)
__global__ void k_ps_kept_counts(int m, const int* __restrict__ off, const int* __restrict__ idx,
                                 const double* __restrict__ val, const unsigned char* __restrict__ row_alive,
                                 const unsigned char* __restrict__ col_alive, const int* __restrict__ row_new,
                                 int* __restrict__ counts)
{
  const int lane = threadIdx.x & 31;
  for (int i = blockIdx.x * PS_WARPS + (threadIdx.x >> 5); i < m; i += gridDim.x * PS_WARPS) {
    if (!row_alive[i]) continue;
    int k = 0;
    for (int p = off[i] + lane; p < off[i + 1]; p += 32) k += (col_alive[idx[p]] && val[p] != 0.0) ? 1 : 0;
    k = warp_count(k);
    if (lane == 0) counts[row_new[i]] = k;
  }
}
// copies the kept entries of the kept rows, in their order, with renumbered columns
__global__ void k_ps_compact(int m, const int* __restrict__ off, const int* __restrict__ idx,
                             const double* __restrict__ val, const unsigned char* __restrict__ row_alive,
                             const unsigned char* __restrict__ col_alive, const int* __restrict__ row_new,
                             const int* __restrict__ col_new, const int* __restrict__ new_off, int* __restrict__ new_idx,
                             double* __restrict__ new_val)
{
  const int lane = threadIdx.x & 31;
  for (int i = blockIdx.x * PS_WARPS + (threadIdx.x >> 5); i < m; i += gridDim.x * PS_WARPS) {
    if (!row_alive[i]) continue;
    int out = new_off[row_new[i]];
    for (int base = off[i]; base < off[i + 1]; base += 32) {
      const int p    = base + lane;
      int j          = 0;
      double a       = 0.0;
      bool keep      = false;
      if (p < off[i + 1]) {
        j    = idx[p];
        a    = val[p];
        keep = col_alive[j] && a != 0.0;
      }
      const unsigned b = __ballot_sync(0xffffffffu, keep);
      if (keep) {
        const int q = out + __popc(b & ((1u << lane) - 1u));
        new_idx[q]  = col_new[j];
        new_val[q]  = a;
      }
      out += __popc(b);
    }
  }
}
__global__ void k_ps_gather(int count, const int* __restrict__ map, const double* __restrict__ src, double* __restrict__ dst)
{
  const int stride = gridDim.x * blockDim.x;
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < count; q += stride) dst[q] = src[map[q]];
}

// ---- postsolve ----
__global__ void k_pst_scatter(int count, const unsigned char* __restrict__ alive, const int* __restrict__ pos,
                              const double* __restrict__ red, const double* __restrict__ removed_value,
                              double* __restrict__ full)
{
  const int stride = gridDim.x * blockDim.x;
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < count; q += stride)
    full[q] = alive[q] ? red[pos[q]] : (removed_value ? removed_value[q] : 0.0);
}
// r = c - A^T y, one warp per column of the original A
__global__ void k_pst_reduced_cost(int n, const int* __restrict__ toff, const int* __restrict__ tidx,
                                   const double* __restrict__ tval, const double* __restrict__ c,
                                   const double* __restrict__ y, double* __restrict__ r)
{
  const int lane = threadIdx.x & 31;
  for (int j = blockIdx.x * PS_WARPS + (threadIdx.x >> 5); j < n; j += gridDim.x * PS_WARPS) {
    double s = 0.0;
    for (int p = toff[j] + lane; p < toff[j + 1]; p += 32) s += tval[p] * y[tidx[p]];
    s = warp_sum(s);
    if (lane == 0) r[j] = c[j] - s;
  }
}
// the singleton row behind the active side of a column (from the sign of r0_j) takes the dual that zeroes r_j
__global__ void k_pst_singleton_duals(int n, const double* __restrict__ r0, const int* __restrict__ src_lo,
                                      const int* __restrict__ src_hi, const double* __restrict__ a_lo,
                                      const double* __restrict__ a_hi, double* __restrict__ y)
{
  const int stride = gridDim.x * blockDim.x;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
    const double r = r0[j];
    if (r > 0.0 && src_lo[j] >= 0) y[src_lo[j]] = r / a_lo[j];
    else if (r < 0.0 && src_hi[j] >= 0) y[src_hi[j]] = r / a_hi[j];
  }
}

int device_sms()
{
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}
int grid_threads(int count, int sms) { return std::max(1, std::min((count + PS_THREADS - 1) / PS_THREADS, sms * 8)); }
int grid_warps(int count, int sms) { return std::max(1, std::min((count + PS_WARPS - 1) / PS_WARPS, sms * 16)); }

struct event_timer_t {
  cudaEvent_t a = nullptr, b = nullptr;
  cudaStream_t s;
  explicit event_timer_t(cudaStream_t st) : s(st)
  {
    CUOPT_CUDA_TRY(cudaEventCreate(&a));
    CUOPT_CUDA_TRY(cudaEventCreate(&b));
    CUOPT_CUDA_TRY(cudaEventRecord(a, s));
  }
  double seconds()
  {
    CUOPT_CUDA_TRY(cudaEventRecord(b, s));
    CUOPT_CUDA_TRY(cudaEventSynchronize(b));
    float ms = 0.f;
    CUOPT_CUDA_TRY(cudaEventElapsedTime(&ms, a, b));
    return 1e-3 * ms;
  }
  ~event_timer_t()
  {
    if (a) cudaEventDestroy(a);
    if (b) cudaEventDestroy(b);
  }
};

}  // namespace

void presolve_device(int& m, int& n, dvec<int>& off, dvec<int>& idx, dvec<double>& val, dvec<double>& c, dvec<double>& l,
                     dvec<double>& u, dvec<double>& lc, dvec<double>& uc, double tol, presolve_state_t& ps,
                     cudaStream_t s, bool trace)
{
  event_timer_t timer(s);
  const int sms = device_sms();
  ps.m0 = m;
  ps.n0 = n;
  ps.nnz0 = (int)val.size();
  const int gm = grid_threads(m, sms), gn = grid_threads(n, sms);
  const int wm = grid_warps(m, sms), wn = grid_warps(n, sms);

  // original A^T, kept until postsolve
  ps.toff.resize((size_t)n + 1);
  ps.tidx.resize(ps.nnz0);
  ps.tval.resize(ps.nnz0);
  if (ps.nnz0 > 0)
    csr_transpose_device(m, n, ps.nnz0, off.data(), idx.data(), val.data(), ps.toff.data(), ps.tidx.data(),
                         ps.tval.data(), s);
  else
    ps.toff.zero(s);
  ps.c0.copy_from(c, s);
  ps.row_alive.resize(m);
  ps.col_alive.resize(n);
  if (m) CUOPT_CUDA_TRY(cudaMemsetAsync(ps.row_alive.data(), 1, m, s));
  if (n) CUOPT_CUDA_TRY(cudaMemsetAsync(ps.col_alive.data(), 1, n, s));
  dvec<int> fixed_round(n), row_cnt(m), row_col(m), cnt(C_COUNT);
  if (n) CUOPT_CUDA_TRY(cudaMemsetAsync(fixed_round.data(), 0xff, (size_t)n * sizeof(int), s));
  ps.x_fix.resize(n);
  ps.x_fix.zero(s);
  for (dvec<int>* v : {&ps.src_lo, &ps.src_hi}) {
    v->resize(n);
    if (n) CUOPT_CUDA_TRY(cudaMemsetAsync(v->data(), 0xff, (size_t)n * sizeof(int), s));
  }
  for (dvec<double>* v : {&ps.a_lo, &ps.a_hi}) {
    v->resize(n);
    v->zero(s);
  }

  presolve_stats_t& st = ps.stats;
  st                   = presolve_stats_t{};
  st.ran               = 1;
  st.original_m        = m;
  st.original_n        = n;
  st.original_nnz      = ps.nnz0;
  int h[C_COUNT]       = {};
  for (int round = 0; round < PRESOLVE_MAX_ROUNDS; ++round) {
    cnt.zero(s);
    k_ps_fix_columns<<<gn, PS_THREADS, 0, s>>>(n, round, l.data(), u.data(), ps.col_alive.data(), fixed_round.data(),
                                               ps.x_fix.data(), cnt.data());
    k_ps_rows<<<wm, PS_THREADS, 0, s>>>(m, round, off.data(), idx.data(), val.data(), ps.col_alive.data(),
                                        fixed_round.data(), ps.x_fix.data(), lc.data(), uc.data(), ps.row_alive.data(),
                                        row_cnt.data(), row_col.data(), tol, cnt.data());
    k_ps_singletons<<<gn, PS_THREADS, 0, s>>>(n, ps.toff.data(), ps.tidx.data(), ps.tval.data(), ps.col_alive.data(),
                                              ps.row_alive.data(), row_cnt.data(), row_col.data(), lc.data(), uc.data(),
                                              l.data(), u.data(), ps.src_lo.data(), ps.src_hi.data(), ps.a_lo.data(),
                                              ps.a_hi.data(), tol, cnt.data());
    k_ps_columns<<<wn, PS_THREADS, 0, s>>>(n, ps.toff.data(), ps.tidx.data(), ps.tval.data(), ps.row_alive.data(),
                                           ps.col_alive.data(), c.data(), l.data(), u.data(), ps.x_fix.data(), cnt.data());
    CUOPT_CUDA_TRY(cudaGetLastError());
    CUOPT_CUDA_TRY(cudaMemcpyAsync(h, cnt.data(), sizeof(h), cudaMemcpyDeviceToHost, s));
    CUOPT_CUDA_TRY(cudaStreamSynchronize(s));
    st.rounds += 1;
    st.fixed_columns += h[C_FIXED];
    st.empty_rows += h[C_EMPTY_ROWS];
    st.singleton_rows += h[C_SINGLETON_ROWS];
    st.empty_columns += h[C_EMPTY_COLS];
    const int removed = h[C_FIXED] + h[C_EMPTY_ROWS] + h[C_SINGLETON_ROWS] + h[C_EMPTY_COLS];
    if (trace)
      std::fprintf(stderr, "[cuopt-b200 trace] presolve round %d: %d fixed columns, %d empty rows, %d singleton rows, "
                   "%d empty columns\n", round, h[C_FIXED], h[C_EMPTY_ROWS], h[C_SINGLETON_ROWS], h[C_EMPTY_COLS]);
    if (h[C_INFEASIBLE]) {
      ps.verdict = termination_status_t::PrimalInfeasible;
      break;
    }
    if (removed == 0) break;
  }
  const int rows_left = m - st.empty_rows - st.singleton_rows;
  const int cols_left = n - st.fixed_columns - st.empty_columns;
  if (ps.verdict == termination_status_t::NoTermination && rows_left == 0)
    ps.verdict = cols_left == 0 ? termination_status_t::Optimal : termination_status_t::DualInfeasible;

  {  // objective offset of the removed columns
    const int parts = std::max(1, std::min((n + PS_THREADS - 1) / PS_THREADS, 1024));
    dvec<double> part(parts), out(1);
    k_ps_offset_partial<<<parts, PS_THREADS, 0, s>>>(n, ps.col_alive.data(), ps.c0.data(), ps.x_fix.data(), part.data());
    k_ps_offset_final<<<1, 1024, 0, s>>>(parts, part.data(), out.data());
    CUOPT_CUDA_TRY(cudaGetLastError());
    CUOPT_CUDA_TRY(cudaMemcpyAsync(&ps.offset, out.data(), sizeof(double), cudaMemcpyDeviceToHost, s));
    CUOPT_CUDA_TRY(cudaStreamSynchronize(s));
  }

  // row and column maps
  {
    dvec<int> flags((size_t)std::max(m, n) + 1);
    ps.row_new.resize((size_t)m + 1);
    ps.col_new.resize((size_t)n + 1);
    k_ps_flags<<<gm, PS_THREADS, 0, s>>>(m, ps.row_alive.data(), flags.data());
    exclusive_sum_int(m + 1, flags.data(), ps.row_new.data(), s);
    k_ps_flags<<<gn, PS_THREADS, 0, s>>>(n, ps.col_alive.data(), flags.data());
    exclusive_sum_int(n + 1, flags.data(), ps.col_new.data(), s);
    CUOPT_CUDA_TRY(cudaGetLastError());
  }
  CUOPT_CUDA_TRY(cudaMemcpyAsync(&ps.m1, ps.row_new.data() + m, sizeof(int), cudaMemcpyDeviceToHost, s));
  CUOPT_CUDA_TRY(cudaMemcpyAsync(&ps.n1, ps.col_new.data() + n, sizeof(int), cudaMemcpyDeviceToHost, s));
  CUOPT_CUDA_TRY(cudaStreamSynchronize(s));
  ps.row_map.resize(ps.m1);
  ps.col_map.resize(ps.n1);
  k_ps_map<<<gm, PS_THREADS, 0, s>>>(m, ps.row_alive.data(), ps.row_new.data(), ps.row_map.data());
  k_ps_map<<<gn, PS_THREADS, 0, s>>>(n, ps.col_alive.data(), ps.col_new.data(), ps.col_map.data());

  // reduced matrix
  dvec<int> counts((size_t)ps.m1 + 1), new_off((size_t)ps.m1 + 1);
  counts.zero(s);
  k_ps_kept_counts<<<wm, PS_THREADS, 0, s>>>(m, off.data(), idx.data(), val.data(), ps.row_alive.data(),
                                             ps.col_alive.data(), ps.row_new.data(), counts.data());
  CUOPT_CUDA_TRY(cudaGetLastError());
  exclusive_sum_int(ps.m1 + 1, counts.data(), new_off.data(), s);
  CUOPT_CUDA_TRY(cudaMemcpyAsync(&ps.nnz1, new_off.data() + ps.m1, sizeof(int), cudaMemcpyDeviceToHost, s));
  CUOPT_CUDA_TRY(cudaStreamSynchronize(s));
  dvec<int> new_idx(ps.nnz1);
  dvec<double> new_val(ps.nnz1);
  k_ps_compact<<<wm, PS_THREADS, 0, s>>>(m, off.data(), idx.data(), val.data(), ps.row_alive.data(), ps.col_alive.data(),
                                         ps.row_new.data(), ps.col_new.data(), new_off.data(), new_idx.data(),
                                         new_val.data());
  // reduced vectors
  auto gather = [&](dvec<double>& v, const dvec<int>& map, int count) {
    dvec<double> r(count);
    k_ps_gather<<<grid_threads(count, sms), PS_THREADS, 0, s>>>(count, map.data(), v.data(), r.data());
    v = std::move(r);  // the old array goes back to the block cache after a device synchronisation
  };
  gather(c, ps.col_map, ps.n1);
  gather(l, ps.col_map, ps.n1);
  gather(u, ps.col_map, ps.n1);
  gather(lc, ps.row_map, ps.m1);
  gather(uc, ps.row_map, ps.m1);
  CUOPT_CUDA_TRY(cudaGetLastError());
  off = std::move(new_off);  // the original A is freed here
  idx = std::move(new_idx);
  val = std::move(new_val);
  m   = ps.m1;
  n   = ps.n1;
  st.reduced_m        = ps.m1;
  st.reduced_n        = ps.n1;
  st.reduced_nnz      = ps.nnz1;
  st.presolve_seconds = timer.seconds();
}

void postsolve_device(const presolve_state_t& ps, const std::vector<double>& x_red, const std::vector<double>& y_red,
                      const std::vector<double>& rc_red, bool certificate, bool dual_ray, std::vector<double>& x,
                      std::vector<double>& y, std::vector<double>& rc, cudaStream_t s)
{
  const int sms = device_sms();
  const int m = ps.m0, n = ps.n0;
  dvec<double> xr(std::max<size_t>(x_red.size(), 1)), yr(std::max<size_t>(y_red.size(), 1));
  dvec<double> xf(n), yf(m), r(n);
  xr.zero(s);
  yr.zero(s);
  if (!x_red.empty()) CUOPT_CUDA_TRY(cudaMemcpyAsync(xr.data(), x_red.data(), x_red.size() * sizeof(double), cudaMemcpyHostToDevice, s));
  if (!y_red.empty()) CUOPT_CUDA_TRY(cudaMemcpyAsync(yr.data(), y_red.data(), y_red.size() * sizeof(double), cudaMemcpyHostToDevice, s));
  const int gm = grid_threads(m, sms), gn = grid_threads(n, sms);
  k_pst_scatter<<<gn, PS_THREADS, 0, s>>>(n, ps.col_alive.data(), ps.col_new.data(), xr.data(),
                                          certificate ? nullptr : ps.x_fix.data(), xf.data());
  k_pst_scatter<<<gm, PS_THREADS, 0, s>>>(m, ps.row_alive.data(), ps.row_new.data(), yr.data(), nullptr, yf.data());
  if (certificate) {
    dvec<double> rr(std::max<size_t>(rc_red.size(), 1));
    rr.zero(s);
    if (!rc_red.empty())
      CUOPT_CUDA_TRY(cudaMemcpyAsync(rr.data(), rc_red.data(), rc_red.size() * sizeof(double), cudaMemcpyHostToDevice, s));
    k_pst_scatter<<<gn, PS_THREADS, 0, s>>>(n, ps.col_alive.data(), ps.col_new.data(), rr.data(), nullptr, r.data());
    dvec<double> zero, r0;
    if (dual_ray) {
      // A bound a singleton row supplied is part of the reduced problem's ray objective; the row's dual carries it back
      // to the original problem (the optimal ending's rule, with the gradient r0 = -A^T y of the ray: zero cost)
      const int wn = grid_warps(n, sms);
      zero.resize(n);
      r0.resize(n);
      zero.zero(s);
      k_pst_reduced_cost<<<wn, PS_THREADS, 0, s>>>(n, ps.toff.data(), ps.tidx.data(), ps.tval.data(), zero.data(),
                                                   yf.data(), r0.data());
      k_pst_singleton_duals<<<gn, PS_THREADS, 0, s>>>(n, r0.data(), ps.src_lo.data(), ps.src_hi.data(), ps.a_lo.data(),
                                                      ps.a_hi.data(), yf.data());
    }
    CUOPT_CUDA_TRY(cudaStreamSynchronize(s));
  } else {
    const int wn = grid_warps(n, sms);
    k_pst_reduced_cost<<<wn, PS_THREADS, 0, s>>>(n, ps.toff.data(), ps.tidx.data(), ps.tval.data(), ps.c0.data(),
                                                 yf.data(), r.data());
    k_pst_singleton_duals<<<gn, PS_THREADS, 0, s>>>(n, r.data(), ps.src_lo.data(), ps.src_hi.data(), ps.a_lo.data(),
                                                    ps.a_hi.data(), yf.data());
    k_pst_reduced_cost<<<wn, PS_THREADS, 0, s>>>(n, ps.toff.data(), ps.tidx.data(), ps.tval.data(), ps.c0.data(),
                                                 yf.data(), r.data());
  }
  CUOPT_CUDA_TRY(cudaGetLastError());
  x.resize(n);
  y.resize(m);
  rc.resize(n);
  xf.download(x.data(), s);
  yf.download(y.data(), s);
  r.download(rc.data(), s);
  CUOPT_CUDA_TRY(cudaStreamSynchronize(s));
}

}  // namespace cuopt_b200
