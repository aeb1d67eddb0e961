// H100-native PDLP driver: device data layout, setup (transpose, diagonal scaling), the
// batched PDHG loop and the major-iteration logic (termination test + KKT restart).
//
// Control flow follows pdlp_solver_t::run_solver (cpp/src/linear_programming/pdlp.cu:984-1185)
// with these structural differences:
//   * the reference synchronises the host once per PDHG iteration to read the accept/reject flag
//     (adaptive_step_size_strategy.cu:228); here a whole batch of attempts (up to the next major
//     iteration) is enqueued as one CUDA graph and the device decides accept/reject itself;
//   * per major iteration the reference issues ~40 library calls and two device->host syncs; here it is
//     two element-wise launches, two fused SpMV launches evaluating the current AND the average iterate
//     in a single pass over A and A^T, and one sync.
// HBM layout (all fp64 / int32, one cudaMalloc each): A and A^T as CSR (scaled, hot) + their unscaled
// copies (termination only) + int4 row-block descriptors; 2x(x, y, A^T y) ping-pong buffers; xbar;
// running sums; averages; last-restart point; reduced costs; bound / cost vectors (scaled + unscaled).
#include "pdlp_solver.hpp"

#include "dist_comm.hpp"
#include "pdlp_kernels.cuh"
#include "trust_region.cuh"

#include <math_constants.h>
#include <nvtx3/nvToolsExt.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <atomic>
#include <map>
#include <mutex>
#include <thread>
#include <string>

namespace cuopt_b200 {

namespace {

// Block-interleaved storage of a matrix (spmv_bicsr.cuh): what every SpMV kernel reads.
struct bicsr_dev_t {
  int n_std = 0, n_blk = 0;
  dvec<int2> desc;
  dvec<unsigned short> row_slot;
  dvec<int> idx;
  dvec<double> val;
};

// A matrix on the device: plain CSR (setup kernels: scaling statistics, transpose, column split; long rows of the SpMV)
// + its block-interleaved form (all SpMV kernels).
struct csr_dev_t {
  int rows = 0, cols = 0, nnz = 0;
  dvec<int> off, idx;
  dvec<double> val;
  bicsr_dev_t bi;
  const csr_dev_t* structure = nullptr;  // scaled copies share offsets / indices / block structure with the original
  const int* off_ptr() const { return structure ? structure->off.data() : off.data(); }
  const int* idx_ptr() const { return structure ? structure->idx.data() : idx.data(); }
  const bicsr_dev_t& bi_structure() const { return structure ? structure->bi : bi; }
  int n_blk() const { return bi_structure().n_blk; }
  bicsr_view_t view() const
  {
    const bicsr_dev_t& s = bi_structure();
    return bicsr_view_t{s.desc.data(), s.row_slot.data(), s.idx.data(), bi.val.data(), s.n_std, s.n_blk,
                        off_ptr(),     idx_ptr(),         val.data()};
  }
  // same sparsity pattern, own values (device-to-device copy)
  void alias_structure_copy_values(const csr_dev_t& o, cudaStream_t s)
  {
    rows = o.rows; cols = o.cols; nnz = o.nnz;
    structure = &o;
    val.copy_from(o.val, s);
  }
};

// The greedy cut below is sequential in nature; at 10M rows and several matrices per solve it was ~0.5 s of host time.
// Rows are therefore cut in independent segments of SCHEDULE_SEGMENT rows (a block never spans a segment boundary) that
// worker threads process in parallel; the segment results are concatenated in order, so the cut is the same run to run
// and independent of the thread count.
constexpr int SCHEDULE_SEGMENT = 1 << 16;
template <typename T, typename F>
std::vector<T> cut_in_segments(int rows, F cut_segment)
{
  const int n_seg = std::max(1, (rows + SCHEDULE_SEGMENT - 1) / SCHEDULE_SEGMENT);
  std::vector<std::vector<T>> part(n_seg);
  const int n_thr = (int)std::max(1u, std::min<unsigned>({std::thread::hardware_concurrency(), 32u, (unsigned)n_seg}));
  std::atomic<int> next{0};
  auto work = [&]() {
    for (int sgm = next.fetch_add(1); sgm < n_seg; sgm = next.fetch_add(1))
      cut_segment(sgm * SCHEDULE_SEGMENT, std::min(rows, (sgm + 1) * SCHEDULE_SEGMENT), part[sgm]);
  };
  if (n_thr <= 1) {
    work();
  } else {
    std::vector<std::thread> pool;
    for (int t = 0; t < n_thr; ++t) pool.emplace_back(work);
    for (auto& t : pool) t.join();
  }
  size_t total = 0;
  for (auto& v : part) total += v.size();
  std::vector<T> all;
  all.reserve(total + 1);
  for (auto& v : part) all.insert(all.end(), v.begin(), v.end());
  return all;
}

// Cuts the rows into BICSR blocks (whole consecutive rows, <= 256 entries, <= 256 rows; a longer row is a long-row block)
// from HOST row offsets, uploads the descriptors and fills the interleaved arrays on the device from d's plain CSR.
template <typename VI>
void build_bicsr(csr_dev_t& d, const VI& off, cudaStream_t s, int sms)
{
  const int all_rows = (int)off.size() - 1;
  constexpr int LONG = (int)0x80000000u;
  std::vector<int2> cut = cut_in_segments<int2>(all_rows, [&](int r, int rows, std::vector<int2>& out) {
    while (r < rows) {
      const int lo = off[r];
      if (off[r + 1] - lo > BICSR_SLOTS) {
        out.push_back(make_int2(r | LONG, r + 1));
        ++r;
        continue;
      }
      int r1 = r;
      while (r1 < rows && off[r1 + 1] - lo <= BICSR_SLOTS && (r1 - r) < BICSR_MAX_ROWS) ++r1;
      out.push_back(make_int2(r, r1));
      r = r1;
    }
  });
  std::vector<int2> desc;
  desc.reserve(cut.size());
  for (const int2& c : cut)
    if (!(c.x & LONG)) desc.push_back(c);
  const int n_std = (int)desc.size();
  for (const int2& c : cut)
    if (c.x & LONG) desc.push_back(make_int2(c.x & ~LONG, c.y));
  bicsr_dev_t& b = d.bi;
  b.n_std        = n_std;
  b.n_blk        = (int)desc.size();
  b.desc.upload(desc, s);
  b.row_slot.resize((size_t)std::max(all_rows, 1));
  b.idx.resize((size_t)std::max(n_std, 1) * BICSR_SLOTS);
  b.val.resize((size_t)std::max(n_std, 1) * BICSR_SLOTS);
  if (all_rows > 0) CUOPT_CUDA_TRY(cudaMemsetAsync(b.row_slot.data(), 0xff, (size_t)all_rows * sizeof(unsigned short), s));
  if (n_std > 0) {
    const int grid = std::max(1, std::min((n_std + 7) / 8, sms * 8));
    k_bicsr_fill<<<grid, 256, 0, s>>>(n_std, b.desc.data(), d.off.data(), d.idx.data(), d.val.data(), b.idx.data(),
                                      b.val.data(), b.row_slot.data());
    CUOPT_CUDA_TRY(cudaGetLastError());
  }
}
// values of a copy that shares the structure of another matrix (after its plain values were scaled)
void fill_bicsr_values(csr_dev_t& d, cudaStream_t s, int sms)
{
  const bicsr_dev_t& st = d.bi_structure();
  d.bi.val.resize((size_t)std::max(st.n_std, 1) * BICSR_SLOTS);
  if (st.n_std > 0) {
    const int grid = std::max(1, std::min((st.n_std + 7) / 8, sms * 8));
    k_bicsr_fill_values<<<grid, 256, 0, s>>>(st.n_std, st.desc.data(), d.off_ptr(), d.val.data(), d.bi.val.data());
    CUOPT_CUDA_TRY(cudaGetLastError());
  }
}

template <typename VI, typename VD>
void upload_csr(csr_dev_t& d, int rows, int cols, const VI& off, const VI& idx, const VD& val, cudaStream_t s, int sms);

}  // namespace

void csr_transpose_device(int rows, int cols, int nnz, const int* off, const int* idx, const double* val, int* toff,
                          int* tidx, double* tval, cudaStream_t stream);  // csr_transpose.cu

void sort_keys_with_index(int count, const double* keys_in, double* keys_out, const int* vals_in, int* vals_out,
                          cudaStream_t stream);  // csr_transpose.cu (CUB)
void inclusive_sum_in_place(int count, double* values, cudaStream_t stream);
void exclusive_sum_int(int count, const int* in, int* out, cudaStream_t stream);
void csr_split_columns_offsets(int rows, const int* off, const int* idx, int width, int n_blocks, int* const* blk_off,
                               int* blk_nnz_host, cudaStream_t stream);  // csr_transpose.cu
void csr_split_columns_fill(int rows, const int* off, const int* idx, const double* val, int width, int n_blocks,
                            int* const* blk_off, int* const* blk_idx, double* const* blk_val, cudaStream_t stream);

namespace {

// A^T on the device (stable order, see csr_transpose.cu); only its row offsets come back to the host, to cut the schedules.
void transpose_to(csr_dev_t& t, const csr_dev_t& a, cudaStream_t s, int sms)
{
  t.rows = a.cols;
  t.cols = a.rows;
  t.nnz  = a.nnz;
  t.off.resize((size_t)t.rows + 1);
  t.idx.resize(t.nnz);
  t.val.resize(t.nnz);
  csr_transpose_device(a.rows, a.cols, a.nnz, a.off.data(), a.idx.data(), a.val.data(), t.off.data(), t.idx.data(),
                       t.val.data(), s);
  std::vector<int> toff((size_t)t.rows + 1);
  t.off.download(toff.data(), s);
  CUOPT_CUDA_TRY(cudaStreamSynchronize(s));
  build_bicsr(t, toff, s, sms);
}

int ew_grid(int n, int sms) { return std::max(1, std::min((n + EW_THREADS - 1) / EW_THREADS, sms * 8)); }

double now_seconds()
{
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// NVTX phase ranges (nsys / ncu timelines), named like the reference's raft::common::nvtx::range scopes where a phase is
// the same (pdlp.cu:541 "Check termination", pdlp_restart_strategy.cu:288 "run trust region restart", :656
// "compute_restart", convergence_information.cu:158 "compute_convergence_information", ...).  Header-only NVTX3: no cost
// without a profiler attached.
struct nvtx_range_t {
  explicit nvtx_range_t(const char* name) { nvtxRangePushA(name); }
  ~nvtx_range_t() { nvtxRangePop(); }
  nvtx_range_t(const nvtx_range_t&)            = delete;
  nvtx_range_t& operator=(const nvtx_range_t&) = delete;
};

// CUOPT_B200_TRACE=1: wall-clock of the setup phases on stderr (each mark synchronises the stream first)
struct phase_trace_t {
  bool on = false;
  double t = 0.0;
  cudaStream_t stream = nullptr;
  void start(cudaStream_t s)
  {
    const char* e = std::getenv("CUOPT_B200_TRACE");
    on            = e != nullptr && e[0] == '1';
    alloc_stats().on = on;
    stream        = s;
    t             = now_seconds();
  }
  void mark(const char* what)
  {
    if (!on) return;
    if (stream) cudaStreamSynchronize(stream);
    const double now = now_seconds();
    std::fprintf(stderr, "[cuopt-b200 trace] %-44s %8.1f ms\n", what, 1e3 * (now - t));
    t = now;
  }
};

// Host -> device copies of the problem arrays go through a process-wide ring of pinned staging buffers: worker threads copy
// the caller's pageable memory into a slot while the DMA engine drains the previous ones (a plain cudaMemcpy from pageable
// memory does the same internally, single-threaded, at ~10 GB/s; this reaches the PCIe rate).  One ring per device, allocated
// on first use and kept: page-locking 128 MB costs more than one upload.
class staged_uploader_t {
 public:
  static staged_uploader_t& get()  // one ring per device: its events belong to the device that was current at creation
  {
    static staged_uploader_t per_device[64];
    int dev = 0;
    cudaGetDevice(&dev);
    return per_device[dev & 63];
  }
  void upload(void* dst, const void* src, size_t bytes, cudaStream_t s)
  {
    if (bytes == 0) return;
    std::lock_guard<std::mutex> guard(mu_);
    if (!ensure() || bytes < SLOT / 4) {  // small arrays, or no pinned memory to be had: the plain path
      CUOPT_CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s));
      return;
    }
    const char* from = static_cast<const char*>(src);
    char* to         = static_cast<char*>(dst);
    for (size_t done = 0; done < bytes;) {
      const int k    = next_;
      next_          = (next_ + 1) % SLOTS;
      const size_t b = std::min(SLOT, bytes - done);
      CUOPT_CUDA_TRY(cudaEventSynchronize(free_[k]));  // the DMA that last read this slot has finished
      char* slot = buf_ + (size_t)k * SLOT;
      parallel_chunks(b, [slot, from, done](size_t lo, size_t hi) { std::memcpy(slot + lo, from + done + lo, hi - lo); },
                      size_t(2) << 20);
      CUOPT_CUDA_TRY(cudaMemcpyAsync(to + done, slot, b, cudaMemcpyHostToDevice, s));
      CUOPT_CUDA_TRY(cudaEventRecord(free_[k], s));
      done += b;
    }
  }

 private:
  static constexpr size_t SLOT = size_t(32) << 20;
  static constexpr int SLOTS   = 4;
  std::mutex mu_;
  char* buf_ = nullptr;
  bool tried_ = false;
  int next_ = 0;
  cudaEvent_t free_[SLOTS] = {};
  bool ensure()
  {
    if (tried_) return buf_ != nullptr;
    tried_ = true;
    if (cudaMallocHost(&buf_, SLOT * SLOTS) != cudaSuccess) {
      cudaGetLastError();
      buf_ = nullptr;
      return false;
    }
    for (auto& e : free_) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
    return true;
  }
};
template <typename T, typename V>
void upload_staged(dvec<T>& d, const V& h, cudaStream_t s)
{
  d.resize(h.size());
  staged_uploader_t::get().upload(d.data(), h.data(), h.size() * sizeof(T), s);
}
template <typename VI, typename VD>
void upload_csr(csr_dev_t& d, int rows, int cols, const VI& off, const VI& idx, const VD& val, cudaStream_t s, int sms)
{
  d.rows = rows;
  d.cols = cols;
  d.nnz  = (int)val.size();
  upload_staged(d.off, off, s);
  upload_staged(d.idx, idx, s);
  upload_staged(d.val, val, s);
  build_bicsr(d, off, s, sms);
}

// Gather blocking (pdlp_kernels.cuh): the largest slice of the gathered vector one column block may span, as a share of the
// device's L2.  Every extra block costs one more read and write of the row sums, so blocks stay as wide as the cache allows.
// configs[3] on an H100 80GB HBM3 (400 W power limit, 50 MB L2), PDLP iterations/s: 16 MB blocks (this fraction) 312,
// 24 MB 311, 40 MB 232, unblocked 184.
constexpr double GATHER_BLOCK_L2_FRACTION = 0.32;

}  // namespace

struct pdlp_solver_t::impl_t {
  // ---- problem ----
  int m = 0, n = 0, nnz = 0;
  bool maximize    = false;
  double obj_scale = 1.0, obj_offset = 0.0;
  pdlp_hyper_params_t hp;
  pdlp_settings_t st;
  cudaStream_t stream = nullptr;
  int sms             = 132;

  csr_dev_t A, AT, As, ATs;
  dvec<double> c, l, u, lc, uc, cs, ls, us, lcs, ucs, Dr, Dc;
  dvec<double> xbuf[2], ybuf[2], atybuf[2], xbar, sum_x, sum_y, x_avg, y_avg, x_lr, y_lr, rc_cur, rc_avg;
  dvec<double> part_dy2, part_k3, part_rows, part_cols, part_misc, scratch_n, scratch_m, d_scalar;
  dvec<double> dist_buf;  // row-sharded mode: partial A^T y' (+1 slot) / 2n for the evaluation, all-reduced in place
  const dist_context_t* dist = nullptr;
  bool sharded() const { return dist != nullptr && dist->world > 1; }
  // Transport of the sharded PDHG attempt (DESIGN.md §6): 0 = replicated primal side + one all-reduce (scheme (i)),
  // 1 = column slices + NCCL all-gather / reduce-scatter (scheme (ii)), 2 = column slices + NVLink peer stores
  // issued by the producing kernels (scheme (ii), no NCCL in the loop), 3 = "gather" (default): every rank also owns the
  // rows J_g of the global A^T, so BOTH products take all-gathered inputs (xbar from K1, y' from K2, by peer stores) and
  // there are no partial products at all.  CUOPT_B200_DIST_MODE=allreduce|nccl|p2p|gather.
  enum { DIST_ALLREDUCE = 0, DIST_NCCL_SLICES = 1, DIST_P2P = 2, DIST_GATHER = 3 };
  int dist_mode = DIST_ALLREDUCE;
  bool peer_transport() const { return dist_mode == DIST_P2P || dist_mode == DIST_GATHER; }
  // gather transport: global row offsets of the ranks, the all-gathered y', this rank's rows of the global scaled A^T
  int row0[DIST_MAX_PEERS + 1] = {};
  int m_total = 0;
  dvec<double> yfull, t_slice;
  void* yfull_peer[DIST_MAX_PEERS] = {};
  peer_ptrs_t p_yfull{};
  csr_dev_t ATslice;
  // packed exchange: Ahot = the scaled A_g with column indices renumbered to the entries of xbar this rank reads; sendX / sendY
  // = per destination rank, where each of MY xbar / y' entries lives in ITS packed buffer (-1: it never reads that entry)
  csr_dev_t Ahot;
  dvec<int> sendX, sendY;    // [world][stride]: slot of my entry i in rank r's packed buffer, -1 if r never reads it
  dvec<int> listX, listY;    // [world][stride]: my entries rank r reads, ascending (first-half entries first)
  send_plan_t planX{}, planY{};
  dvec<double> xloc;         // this rank's slice of xbar before it is sent
  int cntX = 0, cntY = 0;    // packed lengths (second half starts at half the length)
  bool dist_pack = true;     // CUOPT_B200_DIST_PACK=0: identity packing (everything travels), for comparison
  // How the packed entries travel.  "fused" (default): the producing kernels (K1, K2) issue the peer stores themselves, in
  // source order, overlapped with their own work.
  // "kernel" (CUOPT_B200_DIST_SEND=kernel): k_send_packed on a second stream, destination order (full 256-byte lines), halves
  // pipelined with the consumer's column blocks.  The SpMV kernels lose the CTA slots reserved for the send kernel, so it
  // only pays where the attempt is wire-bound (many ranks, ragged source-order stores); opt-in, speed not measured on H100.
  bool dist_send_kernel = false;
  cudaStream_t comm_stream = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  int grid_send = 1, send_slots = 0;  // SpMV CTA slots left to the send kernel (default: one per SM); CUOPT_B200_DIST_SEND_SLOTS
  const csr_dev_t& hot_A() const { return (dist != nullptr && dist->world > 1 && dist_mode == DIST_GATHER) ? Ahot : As; }
  // CUOPT_B200_DIST_TRACE=1: CUDA-event time of every kernel slot of the sharded attempt (waiting for the peers' flags
  // included), printed per rank when the solver goes away.  Turns the CUDA graphs off and synchronises once per attempt.
  bool dist_trace = false;
  cudaEvent_t tr_ev[6] = {};
  double tr_acc[5] = {};
  long tr_count = 0;
  void tr_tick(int i)
  {
    if (dist_trace) cudaEventRecord(tr_ev[i], stream);
  }
  void tr_close(int last)
  {
    if (!dist_trace) return;
    cudaEventSynchronize(tr_ev[last]);
    for (int i = 0; i < last; ++i) {
      float ms = 0.f;
      cudaEventElapsedTime(&ms, tr_ev[i], tr_ev[i + 1]);
      tr_acc[i] += ms;
    }
    ++tr_count;
  }
  int nslice = 0, n_pad = 0, slice_j0 = 0, slice_n = 0, grid_slice = 1;
  dvec<double> rs_buf, stage, scal;
  dvec<unsigned long long> d_flags;
  void* xbar_peer[DIST_MAX_PEERS]  = {};
  void* stage_peer[DIST_MAX_PEERS] = {};
  void* scal_peer[DIST_MAX_PEERS]  = {};
  void* flag_peer[DIST_MAX_PEERS]  = {};
  bool peers_open = false;
  peer_ptrs_t p_xbar{}, p_stage{}, p_scal{};
  peer_flags_t p_flags{};
  dvec<unsigned> d_ticket;
  dvec<pdhg_ctl_t> d_ctl;
  dvec<eval_t> d_eval;
  pdhg_ctl_t* h_ctl = nullptr;  // pinned mirrors
  eval_t* h_eval    = nullptr;
  double* h_scalar  = nullptr;
  int occ_spmv = 1;   // resident CTAs per SM of the SpMV kernels (64 registers, 16 KB of shared memory)
  int occ_spmv2 = 1;  // ... of the fused kernels that prefetch the payload of two row groups (85 registers)
  int npre_override = 0;  // experiment switch CUOPT_B200_SPMV_NPRE=1|2
  dvec<double> eval_m, eval_n;  // A x (current, average) and, on one GPU, A^T y (current, average)
  dvec<double> part_max;        // per_constraint_residual: per-CTA maxima, rows (2 x grid_m) then columns (2 x grid_n)
  dvec<double> part_infeas;     // infeasibility detection: rows (6 x grid_m) then columns (12 x grid_n)
  // trust-region restart (Methodical1): trust_region.cuh
  bool tr_enabled = false;
  double tr_gap_reduction_last_trial = 1.0;  // never initialised in the reference (pdlp_restart_strategy.cu:160); 1 as in PDLP.jl
  int grid_tr = 1;
  dvec<double> tr_aty, tr_ax, tr_grad, tr_dir, tr_thr, tr_thr_sorted, tr_A, tr_B, tr_parts, tr_scal;
  dvec<int> tr_iota, tr_perm;
  struct tr_gap_t {
    const double *px, *py;
    double pd = 0, dd = 0, dist = 0, lower = 0, upper = 0, ngap = 0;
  };
  // gather blocking (pdlp_kernels.cuh): the scaled A / A^T cut into column blocks whose slice of the gathered vector
  // is L2-sized; B == 1 (small LPs) keeps the fused kernels
  struct gather_blocks_t {
    int B = 1, width = 0;
    std::vector<csr_dev_t> blk;
    std::vector<int> grid;  // per block, for the schedule (wide or not) its pass uses
    bool on() const { return B > 1; }
  };
  gather_blocks_t blkA, blkAT, blkATslice;
  dvec<double> t_m, t_n;
  size_t gather_block_bytes = 0;  // set in build() from the device's L2 size (see there)
  int n_part_dy2 = 1;  // CTAs that publish ||dy||^2 partials: grid_k2 (fused K2) or grid_m (blocked K2 epilogue)
  int grid_k1 = 1, grid_k2 = 1, grid_k3 = 1, grid_n = 1, grid_m = 1, grid_misc = 1;
  std::map<int, cudaGraphExec_t> graphs;
  bool use_graphs = true;
  cudaEvent_t ev_a = nullptr, ev_b = nullptr;

  // ---- host-side loop state (names follow pdlp.cu / pdlp_restart_strategy.cu) ----
  int total_pdlp_iterations      = 0;
  bool initialised               = false;
  bool need_aty                  = true;   // first step, or first step after a restart to the average
  bool last_restart_was_average  = false;
  bool warm_started              = false;  // pdlp.cu:1074: the first major iteration keeps the given averages
  double last_candidate_kkt      = 0.0, last_restart_kkt = 0.0;
  double l2_norm_b = 0.0, l2_norm_c = 0.0;
  lp_solution_t sol;
  bool finished   = false;
  double t_start  = 0.0;
  long long launches = 0;

  // Peer mappings must be gone everywhere before any rank frees the memory behind them.  Collective when
  // `collective` (end of a solve: every rank gets here); the destructor alone can only close its own side.
  void close_peer_memory(bool collective)
  {
    if (!peers_open) return;
    cudaStreamSynchronize(stream);
    dist->close_peers(xbar_peer);
    dist->close_peers(stage_peer);
    dist->close_peers(scal_peer);
    dist->close_peers(flag_peer);
    dist->close_peers(yfull_peer);
    peers_open = false;
    if (collective) {
      dist->allreduce(d_scalar.data(), 1, true, stream);  // barrier
      cudaStreamSynchronize(stream);
    }
  }

  ~impl_t()
  {
    if (trace.on) {
      const alloc_stats_t& a = alloc_stats();
      std::fprintf(stderr, "[cuopt-b200 trace] so far in this process: %ld cudaMalloc %.1f ms (%.2f GB), %ld cudaFree %.1f ms\n",
                   a.n_malloc, 1e3 * a.malloc_s, a.bytes * 1e-9, a.n_free, 1e3 * a.free_s);
    }
    if (dist_trace && tr_count > 0)
      std::fprintf(stderr, "[cuopt-b200 dist trace] rank %d of %d, mode %d, %ld attempts: K1 %.1f us, K2 %.1f us, K3 %.1f us, rule %.1f us "
                   "(each slot includes the wait for the peers' flags)\n", dist->rank, dist->world, dist_mode, tr_count,
                   1e3 * tr_acc[0] / tr_count, 1e3 * tr_acc[1] / tr_count, 1e3 * tr_acc[2] / tr_count, 1e3 * tr_acc[3] / tr_count);
    for (auto& e : tr_ev) if (e) cudaEventDestroy(e);
    if (ev_fork) cudaEventDestroy(ev_fork);
    if (ev_join) cudaEventDestroy(ev_join);
    if (comm_stream) cudaStreamDestroy(comm_stream);
    close_peer_memory(false);
    for (auto& g : graphs) cudaGraphExecDestroy(g.second);
    if (ev_a) cudaEventDestroy(ev_a);
    if (ev_b) cudaEventDestroy(ev_b);
    if (h_ctl) cudaFreeHost(h_ctl);
    if (h_eval) cudaFreeHost(h_eval);
    if (h_scalar) cudaFreeHost(h_scalar);
    if (stream) cudaStreamDestroy(stream);
  }

  // one wave of resident CTAs, or fewer when the matrix has fewer blocks than that (8 warps = 8 blocks per CTA)
  int spmv_grid(const csr_dev_t& M, int npre = 1) const
  {
    // gather transport: a consumer may spin on flags the send kernel of THIS rank still has to raise, so that kernel must
    // always find room beside a full wave of SpMV CTAs: send_slots CTA slots stay free (wherever the scheduler leaves them: each
    // holds >= 16 K registers = 2 send CTAs of 256 threads x 28 registers, and the send grid is 2 x send_slots CTAs)
    const int reserve = (dist != nullptr && dist->world > 1 && dist_mode == DIST_GATHER && dist_send_kernel) ? send_slots : 0;
    const int wave    = std::max(1, sms * (npre > 1 ? occ_spmv2 : occ_spmv) - reserve);
    return std::max(1, std::min((M.n_blk() + BICSR_WARPS - 1) / BICSR_WARPS, wave));
  }
  // payload row groups the fused kernels fetch ahead (spmv_bicsr.cuh): 2 when the blocks hold clearly more than 32 rows
  int fused_npre(const csr_dev_t& M) const
  {
    if (npre_override) return npre_override > 1 ? 2 : 1;
    const bicsr_dev_t& b = M.bi_structure();
    return (b.n_std > 0 && (long long)M.rows > 40LL * b.n_std) ? 2 : 1;
  }

  void sync() { CUOPT_CUDA_TRY(cudaStreamSynchronize(stream)); }
  void check_launch() { CUOPT_CUDA_TRY(cudaGetLastError()); }

  // ------------------------------------------------------------------------------- construction
  phase_trace_t trace;
  void build(const lp_problem_t& p, const pdlp_settings_t& settings)
  {
    nvtx_range_t nvtx_scope("pdlp build: upload, transpose, block-interleaved matrices");
    trace.start(nullptr);
    p.check_representation();
    trace.mark("check_representation");
    st       = settings;
    hp       = pdlp_hyper_params_t::preset(settings.pdlp_solver_mode);
    m        = p.n_constraints;
    n        = p.n_variables;
    nnz      = p.nnz();
    maximize = p.maximize;
    if (m == 0 || nnz == 0) {
      // solve.cu:355-360: PDLP cannot run without constraints -> NumericalError solution
      throw lp_error(error_type_t::Success, "No constraints in the problem: PDLP can't be run");
    }
    int dev = 0;
    CUOPT_CUDA_TRY(cudaGetDevice(&dev));
    CUOPT_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    CUOPT_CUDA_TRY(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    CUOPT_CUDA_TRY(cudaEventCreate(&ev_a));
    CUOPT_CUDA_TRY(cudaEventCreate(&ev_b));
    CUOPT_CUDA_TRY(cudaMallocHost(&h_ctl, sizeof(pdhg_ctl_t)));
    CUOPT_CUDA_TRY(cudaMallocHost(&h_eval, 2 * sizeof(eval_t)));
    CUOPT_CUDA_TRY(cudaMallocHost(&h_scalar, 8 * sizeof(double)));
    if (const char* e = std::getenv("CUOPT_B200_NO_GRAPH")) use_graphs = !(e[0] == '1');
    if (const char* e = std::getenv("CUOPT_B200_L2_HINTS")) {  // experiment switch, default on (pdlp_kernels.cuh)
      const int on = e[0] != '0';
      CUOPT_CUDA_TRY(cudaMemcpyToSymbol(g_l2_hints, &on, sizeof(int)));
    }

    // problem_t construction semantics (mip/problem/problem.cu:55-93, problem_helpers.cuh:34-142): maximise => c <- -c,
    // default variable bounds [0, +inf), row senses -> two-sided bounds.  The caller's arrays go to the device as they are
    // (no host copies); negation, defaults and the bound checks run there.
    obj_scale  = p.objective_scaling_factor;
    obj_offset = p.objective_offset;
    if (maximize) obj_scale = -obj_scale;
    trace.stream = stream;
    trace.mark("stream + pinned control buffers");
    upload_csr(A, m, n, p.A_offsets, p.A_indices, p.A_values, stream, sms);
    trace.mark("upload A + BICSR(A)");
    transpose_to(AT, A, stream, sms);
    trace.mark("transpose + BICSR(A^T)");
    As.alias_structure_copy_values(A, stream);
    ATs.alias_structure_copy_values(AT, stream);
    const int gn = ew_grid(n, sms), gm = ew_grid(m, sms);
    upload_staged(c, p.objective_coefficients, stream);
    if (maximize) k_scale_constant<<<gn, EW_THREADS, 0, stream>>>(n, c.data(), -1.0);
    if (p.variable_lower_bounds.empty()) {
      l.resize(n);
      k_fill<<<gn, EW_THREADS, 0, stream>>>(n, l.data(), 0.0);
    } else {
      upload_staged(l, p.variable_lower_bounds, stream);
    }
    if (p.variable_upper_bounds.empty()) {
      u.resize(n);
      k_fill<<<gn, EW_THREADS, 0, stream>>>(n, u.data(), std::numeric_limits<double>::infinity());
    } else {
      upload_staged(u, p.variable_upper_bounds, stream);
    }
    if (!p.constraint_lower_bounds.empty()) {
      upload_staged(lc, p.constraint_lower_bounds, stream);
      upload_staged(uc, p.constraint_upper_bounds, stream);
    } else {
      hvec<double> hlc, huc;
      p.row_bounds(hlc, huc);
      upload_staged(lc, hlc, stream);
      upload_staged(uc, huc, stream);
      sync();  // hlc / huc go out of scope
    }
    {
      dvec<int> bad(2);
      bad.zero(stream);
      k_count_crossed_bounds<<<gn, EW_THREADS, 0, stream>>>(n, l.data(), u.data(), bad.data());
      k_count_crossed_bounds<<<gm, EW_THREADS, 0, stream>>>(m, lc.data(), uc.data(), bad.data() + 1);
      check_launch();
      int h_bad[2] = {0, 0};
      CUOPT_CUDA_TRY(cudaMemcpyAsync(h_bad, bad.data(), sizeof(h_bad), cudaMemcpyDeviceToHost, stream));
      sync();
      if (h_bad[0]) throw lp_error(error_type_t::ValidationError, "Variable lower bound above upper bound");
      if (h_bad[1]) throw lp_error(error_type_t::ValidationError, "Constraint lower bound above upper bound");
    }
    cs.copy_from(c, stream); ls.copy_from(l, stream); us.copy_from(u, stream); lcs.copy_from(lc, stream); ucs.copy_from(uc, stream);
    trace.mark("objective / bound vectors");

    // sharded: primal vectors that travel by all-gather are padded to world * nslice (the pad is never read as data)
    size_t pad = 0;
    if (sharded()) {
      if (dist->world > DIST_MAX_PEERS) throw lp_error(error_type_t::ValidationError, "at most 8 ranks per solve");
      nslice   = (((n + dist->world - 1) / dist->world) + 31) & ~31;
      n_pad    = nslice * dist->world;
      slice_j0 = std::min(n, dist->rank * nslice);
      slice_n  = std::max(0, std::min(nslice, n - slice_j0));
      pad      = (size_t)(n_pad - n);
    }
    for (int b = 0; b < 2; ++b) {
      xbuf[b].resize(n, pad); xbuf[b].zero(stream);
      ybuf[b].resize(m); ybuf[b].zero(stream);
      atybuf[b].resize(n, pad); atybuf[b].zero(stream);
    }
    // xbar doubles as the packed receive buffer of the gather transport: two halves, each rounded up to 32 slots
    xbar.resize(n, pad + (sharded() ? 64 * (size_t)dist->world + 64 : 0));
    xbar.zero(stream);
    sum_x.resize(n, pad);
    sum_x.zero(stream);
    for (dvec<double>* v : {&x_avg, &x_lr, &rc_cur, &rc_avg, &scratch_n}) { v->resize(n); v->zero(stream); }
    for (dvec<double>* v : {&sum_y, &y_avg, &y_lr, &scratch_m}) { v->resize(m); v->zero(stream); }
    Dr.resize(m);
    Dc.resize(n);

    // persistent grids: one wave of resident CTAs (the SpMV kernels all share the core's footprint; the fused K2 / K3
    // carry the largest payload, so their occupancy bounds the others')
    {
      int o2 = 1, o3 = 1;
      CUOPT_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o2, (const void*)k_dual_step<true, 1>, BICSR_THREADS, 0));
      CUOPT_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o3, (const void*)k_transpose_step<true, 1>, BICSR_THREADS, 0));
      occ_spmv = std::max(1, std::min(o2, o3));
      CUOPT_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o2, (const void*)k_dual_step<true, 2>, BICSR_THREADS, 0));
      CUOPT_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o3, (const void*)k_transpose_step<true, 2>, BICSR_THREADS, 0));
      occ_spmv2 = std::max(1, std::min(o2, o3));
      if (const char* e = std::getenv("CUOPT_B200_SPMV_NPRE")) npre_override = std::atoi(e);
    }
    grid_k2   = spmv_grid(As);
    grid_k3   = spmv_grid(ATs);
    grid_n    = ew_grid(n, sms);
    grid_m    = ew_grid(m, sms);
    grid_k1   = grid_n;
    grid_misc = ew_grid(std::max(n, m), sms);
    part_dy2.resize((size_t)std::max({grid_k2, grid_m, sms * 16}));
    n_part_dy2 = grid_k2;
    // size of the slice of the gathered vector one column block may span (0 = never block); bytes, for the tests too.
    // GATHER_BLOCK_L2_FRACTION of the L2: the slice shares the cache with the matrix streams and the row sums passing by
    {
      int l2 = 0;
      CUOPT_CUDA_TRY(cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, dev));
      gather_block_bytes = (size_t)((double)l2 * GATHER_BLOCK_L2_FRACTION);
    }
    if (const char* e = std::getenv("CUOPT_B200_GATHER_BLOCK_BYTES")) gather_block_bytes = (size_t)std::atoll(e);
    part_k3.resize(2 * (size_t)std::max({grid_k3, grid_n, sms * 16}));
    part_rows.resize(6 * (size_t)grid_m);
    if (hp.restart_strategy == 2) {
      tr_enabled = true;
      {
        if (sharded())
          throw lp_error(error_type_t::ValidationError, "Methodical1 is not available in multi-GPU solves");
        const size_t N = (size_t)n + m;
        grid_tr        = ew_grid((int)std::min<size_t>(N, 1u << 30), sms);
        tr_aty.resize(n); tr_ax.resize(m); tr_grad.resize(N); tr_dir.resize(N); tr_thr.resize(N); tr_thr_sorted.resize(N);
        tr_A.resize(N); tr_B.resize(N); tr_iota.resize(N); tr_perm.resize(N);
        tr_parts.resize(5 * (size_t)grid_tr);
        tr_scal.resize(TR_SCALARS);
        tr_scal.zero(stream);
      }
    }
    if (st.detect_infeasibility) {
      if (sharded())
        throw lp_error(error_type_t::ValidationError, "infeasibility_detection is not available in multi-GPU solves yet");
      part_infeas.resize(6 * (size_t)grid_m + 12 * (size_t)grid_n);
    }
    if (st.per_constraint_residual) part_max.resize(2 * (size_t)std::max(grid_m, grid_n) * 2);
    eval_m.resize(2 * (size_t)m);
    if (!sharded()) eval_n.resize(2 * (size_t)n);
    part_cols.resize(8 * (size_t)grid_n);
    part_misc.resize(2 * (size_t)std::max(grid_misc, ew_grid(nnz, sms)));
    d_scalar.resize(12);
    if (sharded()) setup_transport();
    d_ticket.resize(8);
    d_ticket.zero(stream);
    d_ctl.resize(1);
    d_ctl.zero(stream);
    d_eval.resize(2);
    d_eval.zero(stream);
    sync();
    trace.mark("vectors, grids, work buffers");
  }

  // sharded solve: pick the transport of the PDHG attempt and set up its buffers (collective)
  void setup_transport()
  {
    dist_buf.resize(2 * (size_t)std::max(n, n_pad) + 8);
    dist_buf.zero(stream);
    dist_mode = DIST_GATHER;
    if (const char* e = std::getenv("CUOPT_B200_DIST_MODE")) {
      const std::string v(e);
      if (v == "allreduce") dist_mode = DIST_ALLREDUCE;
      else if (v == "nccl") dist_mode = DIST_NCCL_SLICES;
      else if (v == "p2p") dist_mode = DIST_P2P;
      else if (v == "gather") dist_mode = DIST_GATHER;
      else throw lp_error(error_type_t::InvalidArgument, "CUOPT_B200_DIST_MODE must be allreduce, nccl, p2p or gather");
    }
    {  // global row offsets of the ranks (the row blocks are contiguous and in rank order)
      dvec<double> cnt((size_t)dist->world);
      cnt.zero(stream);
      const double mine = (double)m;
      CUOPT_CUDA_TRY(cudaMemcpyAsync(cnt.data() + dist->rank, &mine, sizeof(double), cudaMemcpyHostToDevice, stream));
      dist->allgather(cnt.data(), 1, stream);
      std::vector<double> h((size_t)dist->world);
      cnt.download(h.data(), stream);
      sync();
      long long tot = 0;
      for (int r = 0; r < dist->world; ++r) { row0[r] = (int)tot; tot += (long long)h[r]; }
      if (tot > 0x7fffffffLL) throw lp_error(error_type_t::ValidationError, "more than 2^31 - 1 constraint rows over all ranks");
      row0[dist->world] = m_total = (int)tot;
    }
    grid_slice = ew_grid(std::max(nslice, 1), sms);
    scal.resize(4 * DIST_MAX_PEERS);
    scal.zero(stream);
    if (dist_mode == DIST_NCCL_SLICES) { rs_buf.resize(nslice); rs_buf.zero(stream); }
    if (peer_transport()) {
      if (dist_mode == DIST_P2P) stage.resize((size_t)nslice * dist->world);
      else {
        stage.resize(32);
        yfull.resize((size_t)m_total + 64 * (size_t)dist->world + 64);
        yfull.zero(stream);
        xloc.resize((size_t)std::max(nslice, 32));
        xloc.zero(stream);
      }
      stage.zero(stream);
      d_flags.resize(DIST_FLAG_COUNT);
      d_flags.zero(stream);
      // every rank's buffers are zeroed (stream order) before its handles leave through the stream-ordered all-gather
      bool ok = dist->open_peers(xbar.data(), xbar_peer, stream);
      ok      = ok && dist->open_peers(stage.data(), stage_peer, stream);
      ok      = ok && dist->open_peers(scal.data(), scal_peer, stream);
      ok      = ok && dist->open_peers(d_flags.data(), flag_peer, stream);
      if (dist_mode == DIST_GATHER) ok = ok && dist->open_peers(yfull.data(), yfull_peer, stream);
      if (!ok) {  // unanimous (open_peers agrees across ranks): no peer access on this box -> NCCL transport
        dist->close_peers(xbar_peer); dist->close_peers(stage_peer); dist->close_peers(scal_peer);
        dist->close_peers(flag_peer); dist->close_peers(yfull_peer);
        dist_mode = DIST_NCCL_SLICES;
        rs_buf.resize(nslice);
        rs_buf.zero(stream);
      } else {
        peers_open = true;
        for (int r = 0; r < dist->world; ++r) {
          p_xbar.p[r]  = static_cast<double*>(xbar_peer[r]) + (dist_mode == DIST_GATHER ? 0 : slice_j0);
          p_stage.p[r] = static_cast<double*>(stage_peer[r]) + (size_t)dist->rank * nslice;
          p_scal.p[r]  = static_cast<double*>(scal_peer[r]) + 4 * dist->rank;
          p_flags.p[r] = static_cast<unsigned long long*>(flag_peer[r]);
          if (dist_mode == DIST_GATHER) p_yfull.p[r] = static_cast<double*>(yfull_peer[r]);
        }
      }
    }
    if (const char* e = std::getenv("CUOPT_B200_DIST_TRACE")) dist_trace = e[0] == '1';
    if (const char* e = std::getenv("CUOPT_B200_DIST_PACK")) dist_pack = e[0] != '0';
    if (const char* e = std::getenv("CUOPT_B200_DIST_SEND")) dist_send_kernel = std::string(e) == "kernel";
    if (dist_mode == DIST_GATHER) {
      CUOPT_CUDA_TRY(cudaStreamCreateWithFlags(&comm_stream, cudaStreamNonBlocking));
      CUOPT_CUDA_TRY(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
      CUOPT_CUDA_TRY(cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming));
      send_slots = sms;  // one slot per SM: far fewer send CTAs cannot keep the link busy
      if (const char* e = std::getenv("CUOPT_B200_DIST_SEND_SLOTS")) send_slots = std::max(1, std::min(std::atoi(e), sms));
      grid_send = 2 * send_slots;
    }
    if (dist_trace) {
      use_graphs = false;
      for (auto& e : tr_ev) CUOPT_CUDA_TRY(cudaEventCreate(&e));
    }
    if (!peer_transport()) {
      use_graphs  = false;  // NCCL calls between the kernels
      p_scal.p[0] = scal.data();
    }
  }

  // lanes per row of the setup kernels that walk plain CSR rows: the power of two at or above the average row length
  static int row_group_width(const csr_dev_t& M)
  {
    const double avg = M.rows > 0 ? (double)M.nnz / M.rows : 0.0;
    return avg <= 4.0 ? 4 : avg <= 8.0 ? 8 : avg <= 16.0 ? 16 : 32;
  }
  // deterministic setup reduction, result on the host
  // `across_ranks`: the reduced quantity lives on row-sharded data (rows of A, lc/uc), combine over ranks too
  double setup_reduce(int kind, int count, const double* a, const double* b, double weight, bool across_ranks = false)
  {
    const int g = ew_grid(count, sms);
    k_setup_reduce<<<g, EW_THREADS, 0, stream>>>(kind, count, a, b, weight, part_misc.data(), d_ticket.data(), d_scalar.data());
    check_launch();
    if (across_ranks && sharded()) dist->allreduce(d_scalar.data(), 1, kind == 0, stream);
    CUOPT_CUDA_TRY(cudaMemcpyAsync(h_scalar, d_scalar.data(), sizeof(double), cudaMemcpyDeviceToHost, stream));
    sync();
    return h_scalar[0];
  }

  // initial_scaling.cu:85-307
  void compute_scaling_vectors()
  {
    nvtx_range_t nvtx_scope("compute_scaling_vectors (Ruiz + Pock-Chambolle)");
    k_fill<<<grid_m, EW_THREADS, 0, stream>>>(m, Dr.data(), 1.0);
    k_fill<<<grid_n, EW_THREADS, 0, stream>>>(n, Dc.data(), 1.0);
    auto stat = [&](const csr_dev_t& M, const double* rs, const double* cs, int swap, int mode, double power, double* out) {
      const int w    = row_group_width(M);
      const int grid = std::max(1, std::min((int)(((long long)M.rows * w + 255) / 256), sms * 16));
#define CUOPT_STAT(W)                                                                                                   \
  k_row_scaling_stat<W><<<grid, 256, 0, stream>>>(M.rows, M.off.data(), M.idx.data(), M.val.data(), rs, cs, swap, mode, \
                                                  power, out)
      if (w == 4) CUOPT_STAT(4); else if (w == 8) CUOPT_STAT(8); else if (w == 16) CUOPT_STAT(16); else CUOPT_STAT(32);
#undef CUOPT_STAT
    };
    auto pass = [&](int mode, double pr, double pc) {
      // statistics of rows of A and of rows of A^T (columns of A), both with the OLD scaling vectors
      stat(A, Dr.data(), Dc.data(), 0, mode, pr, scratch_m.data());
      stat(AT, Dc.data(), Dr.data(), 1, mode, pc, scratch_n.data());
      // row-sharded: a column's statistic spans the row blocks of all ranks (max for Ruiz, sum for Pock-Chambolle)
      if (sharded()) dist->allreduce(scratch_n.data(), n, mode == 0, stream);
      k_apply_scaling_stat<<<grid_m, EW_THREADS, 0, stream>>>(m, Dr.data(), scratch_m.data());
      k_apply_scaling_stat<<<grid_n, EW_THREADS, 0, stream>>>(n, Dc.data(), scratch_n.data());
    };
    if (hp.do_ruiz_scaling)
      for (int it = 0; it < hp.default_l_inf_ruiz_iterations; ++it) pass(0, 0.0, 0.0);
    if (hp.do_pock_chambolle_scaling) {
      const double alpha = hp.default_alpha_pock_chambolle_rescaling;
      if (!(alpha >= 0.0 && alpha <= 2.0)) throw lp_error(error_type_t::ValidationError, "Invalid Pock-Chambolle alpha");
      pass(1, alpha, 2.0 - alpha);
    }
    check_launch();
  }

  // initial_scaling.cu:348-408
  void scale_problem()
  {
    nvtx_range_t nvtx_scope("scale_problem");
    auto scale = [&](csr_dev_t& M, const double* rs, const double* cs) {
      const int w    = row_group_width(M);
      const int grid = std::max(1, std::min((int)(((long long)M.rows * w + 255) / 256), sms * 16));
#define CUOPT_SCALE(W) k_scale_matrix<W><<<grid, 256, 0, stream>>>(M.rows, M.off_ptr(), M.idx_ptr(), M.val.data(), rs, cs)
      if (w == 4) CUOPT_SCALE(4); else if (w == 8) CUOPT_SCALE(8); else if (w == 16) CUOPT_SCALE(16); else CUOPT_SCALE(32);
#undef CUOPT_SCALE
    };
    scale(As, Dr.data(), Dc.data());
    scale(ATs, Dc.data(), Dr.data());
    k_scale_vector<<<grid_n, EW_THREADS, 0, stream>>>(n, cs.data(), Dc.data(), 0);
    k_scale_vector<<<grid_n, EW_THREADS, 0, stream>>>(n, ls.data(), Dc.data(), 1);
    k_scale_vector<<<grid_n, EW_THREADS, 0, stream>>>(n, us.data(), Dc.data(), 1);
    k_scale_vector<<<grid_m, EW_THREADS, 0, stream>>>(m, lcs.data(), Dr.data(), 0);
    k_scale_vector<<<grid_m, EW_THREADS, 0, stream>>>(m, ucs.data(), Dr.data(), 0);
    check_launch();
    // x = y = 0 at this point: scaling the (zero) iterates is a no-op
  }

  double initial_step_size(const csr_dev_t& M)  // pdlp.cu:1225-1258
  {
    const double mx = setup_reduce(0, M.nnz, M.val.data(), nullptr, 0.0, true);
    return mx == 0.0 ? 0.0 : hp.initial_step_size_scaling / mx;
  }
  double initial_primal_weight(const dvec<double>& cc, const dvec<double>& lo, const dvec<double>& hi)  // pdlp.cu:1261-1309
  {
    const double bn = std::sqrt(setup_reduce(2, m, lo.data(), hi.data(), hp.initial_primal_weight_b_scaling, true));
    const double cn = std::sqrt(setup_reduce(1, n, cc.data(), nullptr, hp.initial_primal_weight_c_scaling));
    return (bn > 0.0 && cn > 0.0) ? hp.primal_importance * (cn / bn) : hp.primal_importance;
  }

  void initialise()
  {
    if (initialised) return;
    nvtx_range_t nvtx_scope("pdlp initialise: scaling, initial step size / primal weight");
    const double t0 = now_seconds();
    // norms of the unscaled problem used by the relative tolerances (convergence_information.cu:74-82)
    trace.mark("(gap between build and initialise)");
    l2_norm_c = std::sqrt(setup_reduce(1, n, c.data(), nullptr, 1.0));
    l2_norm_b = std::sqrt(setup_reduce(2, m, lc.data(), uc.data(), 1.0, true));
    trace.mark("norms");
    compute_scaling_vectors();
    trace.mark("scaling vectors (Ruiz + Pock-Chambolle)");
    double step = 0.0, weight = 0.0;
    if (hp.compute_initial_step_size_before_scaling) step = initial_step_size(A);
    if (hp.compute_initial_primal_weight_before_scaling) weight = initial_primal_weight(c, lc, uc);
    scale_problem();
    fill_bicsr_values(As, stream, sms);
    fill_bicsr_values(ATs, stream, sms);
    trace.mark("scale problem + scaled BICSR values");
    if (sharded() && dist_mode == DIST_GATHER) {
      build_gather_transport();  // packed A_g, rows J_g of the global A^T; the hot loop never multiplies by A_g^T
    } else {
      build_gather_blocks(As, blkA, t_m);
      build_gather_blocks(ATs, blkAT, t_n);
    }
    trace.mark("gather blocks");
    n_part_dy2 = k2_grid();  // CTAs of the kernel that runs the dual row epilogue
    if (!hp.compute_initial_step_size_before_scaling) step = initial_step_size(As);
    if (!hp.compute_initial_primal_weight_before_scaling) weight = initial_primal_weight(cs, lcs, ucs);

    pdhg_ctl_t k{};
    k.step_size          = step;
    k.primal_weight      = weight;
    k.tau                = step / weight;  // adaptive_step_size_strategy.cu:348-366
    k.sigma              = step * weight;
    k.reduction_exponent = hp.reduction_exponent;
    k.growth_exponent    = hp.growth_exponent;
    k.primal_smoothing   = hp.primal_distance_smoothing;
    k.dual_smoothing     = hp.dual_distance_smoothing;
    *h_ctl               = k;
    if (st.warm_start && !st.warm_start->empty()) apply_warm_start(*st.warm_start);
    CUOPT_CUDA_TRY(cudaMemcpyAsync(d_ctl.data(), h_ctl, sizeof(k), cudaMemcpyHostToDevice, stream));
    if (hp.project_initial_primal) {  // pdlp.cu:1041-1056 (the unscaled average is clamped to the SCALED bounds there too)
      k_clamp<<<grid_n, EW_THREADS, 0, stream>>>(n, xbuf[0].data(), ls.data(), us.data());
      k_clamp<<<grid_n, EW_THREADS, 0, stream>>>(n, x_avg.data(), ls.data(), us.data());
    }
    check_launch();
    sync();
    trace.mark("initial step size / primal weight, control block");
    sol.stats.initial_step_size     = step;
    sol.stats.initial_primal_weight = weight;
    sol.stats.setup_seconds += now_seconds() - t0;
    initialised = true;
  }

  // pdlp.cu:131-181 + :1010-1038: continue a previous solve.  Called with *h_ctl holding the fresh-start scalars.
  void apply_warm_start(const pdlp_warm_start_t& w)
  {
    auto need = [&](const std::vector<double>& v, int size, const char* what) {
      if ((int)v.size() != size)
        throw lp_error(error_type_t::ValidationError, std::string("warm start: ") + what + " has the wrong size");
    };
    need(w.current_primal_solution, n, "current_primal_solution");
    need(w.current_dual_solution, m, "current_dual_solution");
    need(w.initial_primal_average, n, "initial_primal_average");
    need(w.initial_dual_average, m, "initial_dual_average");
    need(w.current_ATY, n, "current_ATY");
    need(w.sum_primal_solutions, n, "sum_primal_solutions");
    need(w.sum_dual_solutions, m, "sum_dual_solutions");
    need(w.last_restart_duality_gap_primal_solution, n, "last_restart_duality_gap_primal_solution");
    need(w.last_restart_duality_gap_dual_solution, m, "last_restart_duality_gap_dual_solution");
    auto put = [&](dvec<double>& d, const std::vector<double>& h) {
      if (!h.empty()) CUOPT_CUDA_TRY(cudaMemcpyAsync(d.data(), h.data(), h.size() * sizeof(double), cudaMemcpyHostToDevice, stream));
    };
    put(xbuf[0], w.current_primal_solution);  // unscaled on arrival; update_primal_dual_solutions scales it (:963)
    put(ybuf[0], w.current_dual_solution);
    k_scale_back<<<grid_n, EW_THREADS, 0, stream>>>(n, xbuf[0].data(), Dc.data());
    k_scale_back<<<grid_m, EW_THREADS, 0, stream>>>(m, ybuf[0].data(), Dr.data());
    put(x_avg, w.initial_primal_average);
    put(y_avg, w.initial_dual_average);
    put(atybuf[0], w.current_ATY);
    put(sum_x, w.sum_primal_solutions);
    put(sum_y, w.sum_dual_solutions);
    put(x_lr, w.last_restart_duality_gap_primal_solution);
    put(y_lr, w.last_restart_duality_gap_dual_solution);
    check_launch();
    sync();  // the host vectors may go away with the settings object
    pdhg_ctl_t& k       = *h_ctl;
    k.step_size         = w.initial_step_size;
    k.primal_weight     = w.initial_primal_weight;
    k.tau               = k.step_size / k.primal_weight;
    k.sigma             = k.step_size * k.primal_weight;
    k.k_pdhg            = w.total_pdhg_iterations;
    k.attempts          = w.total_pdhg_iterations;
    k.sum_weights       = w.sum_solution_weight;
    k.its_since_restart = w.iterations_since_last_restart;
    total_pdlp_iterations = w.total_pdlp_iterations;
    last_candidate_kkt    = w.last_candidate_kkt_score;
    last_restart_kkt      = w.last_restart_kkt_score;
    need_aty              = w.total_pdhg_iterations == 0;  // pdhg.cu:183: otherwise the given A^T y is the current one
    warm_started          = true;
  }

  // pdlp.cu:469-489, at the moment a solution is returned: current iterate and averages are unscaled, the rest scaled
  void capture_warm_start()
  {
    const int cur = h_ctl->parity;
    auto w        = std::make_shared<pdlp_warm_start_t>();
    auto get      = [&](std::vector<double>& h, const dvec<double>& d, int size) {
      h.resize(size);
      if (size) CUOPT_CUDA_TRY(cudaMemcpyAsync(h.data(), d.data(), (size_t)size * sizeof(double), cudaMemcpyDeviceToHost, stream));
    };
    get(w->current_primal_solution, xbuf[cur], n);
    get(w->current_dual_solution, ybuf[cur], m);
    get(w->initial_primal_average, x_avg, n);
    get(w->initial_dual_average, y_avg, m);
    get(w->current_ATY, atybuf[cur], n);
    get(w->sum_primal_solutions, sum_x, n);
    get(w->sum_dual_solutions, sum_y, m);
    get(w->last_restart_duality_gap_primal_solution, x_lr, n);
    get(w->last_restart_duality_gap_dual_solution, y_lr, m);
    sync();
    w->initial_primal_weight         = h_ctl->primal_weight;
    w->initial_step_size             = h_ctl->step_size;
    w->total_pdlp_iterations         = total_pdlp_iterations;
    w->total_pdhg_iterations         = h_ctl->attempts;
    w->last_candidate_kkt_score      = last_candidate_kkt;
    w->last_restart_kkt_score        = last_restart_kkt;
    w->sum_solution_weight           = h_ctl->sum_weights;
    w->iterations_since_last_restart = h_ctl->its_since_restart;
    sol.warm_start                   = w;
  }

  // Gather transport, setup (collective): this rank's rows J_g of the global scaled A^T, assembled from the scaled A_h^T of
  // every rank through peer reads (k_slice_row_counts / k_slice_fill) as plain CSR with GLOBAL row ids as column indices;
  // returns its host row offsets (build_gather_transport renumbers the columns and builds the BICSR form).
  std::vector<int> build_slice_transpose()
  {
    const int G = dist->world;
    void *offp[DIST_MAX_PEERS] = {}, *idxp[DIST_MAX_PEERS] = {}, *valp[DIST_MAX_PEERS] = {};
    bool ok = dist->open_peers(const_cast<int*>(ATs.off_ptr()), offp, stream);
    ok      = ok && dist->open_peers(const_cast<int*>(ATs.idx_ptr()), idxp, stream);
    ok      = ok && dist->open_peers(ATs.val.data(), valp, stream);
    if (!ok) throw lp_error(error_type_t::RuntimeError, "gather transport: peer mapping of the transposed row blocks failed");
    peer_csr_t src{};
    for (int r = 0; r < G; ++r) {
      src.off[r]  = static_cast<const int*>(offp[r]);
      src.idx[r]  = static_cast<const int*>(idxp[r]);
      src.val[r]  = static_cast<const double*>(valp[r]);
      src.row0[r] = row0[r];
    }
    ATslice      = csr_dev_t{};
    ATslice.rows = slice_n;
    ATslice.cols = m_total;
    dvec<int> cnt((size_t)slice_n + 1);
    ATslice.off.resize((size_t)slice_n + 1);
    const int g = ew_grid(slice_n + 1, sms);
    k_slice_row_counts<<<g, EW_THREADS, 0, stream>>>(slice_n, slice_j0, src, G, cnt.data());
    exclusive_sum_int(slice_n + 1, cnt.data(), ATslice.off.data(), stream);
    std::vector<int> hoff((size_t)slice_n + 1);
    ATslice.off.download(hoff.data(), stream);
    sync();
    ATslice.nnz = hoff[slice_n];
    ATslice.idx.resize((size_t)std::max(ATslice.nnz, 1));
    ATslice.val.resize((size_t)std::max(ATslice.nnz, 1));
    k_slice_fill<<<g, EW_THREADS, 0, stream>>>(slice_n, slice_j0, src, G, ATslice.off.data(), ATslice.idx.data(),
                                               ATslice.val.data());
    check_launch();
    sync();
    // nobody may touch / free its A_h^T while a peer still reads it: barrier, then unmap
    dist->allreduce(d_scalar.data(), 1, true, stream);
    sync();
    dist->close_peers(offp); dist->close_peers(idxp); dist->close_peers(valp);
    return hoff;
  }

  // Which of `count` entries occur among `nnz` indices -> pos[j] = slot in the packed buffer or -1 (every entry when packing
  // is off).  The needed entries of the first halves (hm) fill slots [0, W), those of the second halves [W, 2 W); returns W
  // (a multiple of 32).  pos has `padded` >= count entries (the pad is -1).
  int packed_positions(int count, int padded, int nnz, const int* idx, const half_map_t& hm, dvec<int>& pos)
  {
    const size_t len = (size_t)padded + 1;
    dvec<int> need(len), fa(len), fb(len), sa(len), sb(len);
    need.zero(stream);
    if (dist_pack) {
      if (nnz > 0) k_mark_indices<<<ew_grid(nnz, sms), EW_THREADS, 0, stream>>>(nnz, idx, need.data());
    } else if (count > 0) {
      k_fill_int<<<ew_grid(count, sms), EW_THREADS, 0, stream>>>(count, need.data(), 1);
    }
    k_half_flags<<<ew_grid((int)len, sms), EW_THREADS, 0, stream>>>((int)len, need.data(), hm, fa.data(), fb.data());
    exclusive_sum_int((int)len, fa.data(), sa.data(), stream);
    exclusive_sum_int((int)len, fb.data(), sb.data(), stream);
    int tot[2] = {0, 0};
    CUOPT_CUDA_TRY(cudaMemcpyAsync(&tot[0], sa.data() + padded, sizeof(int), cudaMemcpyDeviceToHost, stream));
    CUOPT_CUDA_TRY(cudaMemcpyAsync(&tot[1], sb.data() + padded, sizeof(int), cudaMemcpyDeviceToHost, stream));
    sync();
    const int W = (std::max({tot[0], tot[1], 1}) + 31) & ~31;
    pos.resize((size_t)std::max(padded, 1));
    if (padded > 0)
      k_packed_positions<<<ew_grid(padded, sms), EW_THREADS, 0, stream>>>(padded, fa.data(), sa.data(), fb.data(), sb.data(), W,
                                                                        pos.data());
    check_launch();
    sync();
    return W;
  }
  // Sender side: from the slot table of every destination (tbl[r * count + i]) the ascending list of my entries it reads and
  // how many of them lie below `half` (they are sent, and flagged, first).
  void build_send_lists(const dvec<int>& tbl, int count, int half, dvec<int>& list, send_plan_t& plan)
  {
    const int G = dist->world;
    plan        = send_plan_t{};
    list.resize((size_t)std::max(count, 1) * G);
    if (count <= 0) return;
    dvec<int> flag((size_t)count + 1), scan((size_t)count + 1);
    for (int r = 0; r < G; ++r) {
      flag.zero(stream);
      k_flag_nonnegative<<<ew_grid(count, sms), EW_THREADS, 0, stream>>>(count, tbl.data() + (size_t)r * count, flag.data());
      exclusive_sum_int(count + 1, flag.data(), scan.data(), stream);
      k_fill_list<<<ew_grid(count, sms), EW_THREADS, 0, stream>>>(count, flag.data(), scan.data(), list.data() + (size_t)r * count);
      CUOPT_CUDA_TRY(cudaMemcpyAsync(&plan.count_a[r], scan.data() + std::min(half, count), sizeof(int), cudaMemcpyDeviceToHost, stream));
      CUOPT_CUDA_TRY(cudaMemcpyAsync(&plan.count[r], scan.data() + count, sizeof(int), cudaMemcpyDeviceToHost, stream));
      check_launch();
      sync();
    }
  }
  // every rank's pos array (same length everywhere) -> mine[g * count + i] = peer g's pos[first + i]  (collective)
  void exchange_positions(dvec<int>& pos, int first, int count, dvec<int>& mine)
  {
    const int G = dist->world;
    void* peers[DIST_MAX_PEERS] = {};
    if (!dist->open_peers(pos.data(), peers, stream))
      throw lp_error(error_type_t::RuntimeError, "gather transport: peer mapping of the packing tables failed");
    mine.resize((size_t)std::max(count, 1) * G);
    for (int g = 0; g < G && count > 0; ++g)
      CUOPT_CUDA_TRY(cudaMemcpyAsync(mine.data() + (size_t)g * count, static_cast<const int*>(peers[g]) + first,
                                     (size_t)count * sizeof(int), cudaMemcpyDefault, stream));
    sync();
    dist->allreduce(d_scalar.data(), 1, true, stream);  // nobody frees its table while a peer still reads it
    sync();
    dist->close_peers(peers);
  }
  void build_gather_transport()
  {
    const int G = dist->world, rk = dist->rank;
    // xbar side: the columns this rank's rows of A touch; owner h holds columns [h nslice, (h + 1) nslice)
    half_map_t hx{}, hy{};
    hx.world = hy.world = G;
    for (int h = 0; h < G; ++h) {
      hx.start[h] = h * nslice;
      hx.half[h]  = nslice / 2;
      hy.start[h] = row0[h];
      hy.half[h]  = (row0[h + 1] - row0[h] + 1) / 2;
    }
    for (int h = G; h <= DIST_MAX_PEERS; ++h) { hx.start[h] = n_pad; hy.start[h] = m_total; }
    dvec<int> posX, posY;
    const int WX = packed_positions(n, n_pad, A.nnz, A.idx.data(), hx, posX);
    cntX         = 2 * WX;
    if ((size_t)cntX > (size_t)n_pad + 64 * (size_t)G + 64) throw lp_error(error_type_t::RuntimeError, "gather transport: packed xbar exceeds its buffer");
    Ahot      = csr_dev_t{};
    Ahot.rows = m;
    Ahot.cols = cntX;
    Ahot.nnz  = A.nnz;
    Ahot.off.copy_from(A.off, stream);
    Ahot.idx.resize((size_t)std::max(A.nnz, 1));
    if (A.nnz > 0) k_remap_indices<<<ew_grid(A.nnz, sms), EW_THREADS, 0, stream>>>(A.nnz, A.idx.data(), posX.data(), Ahot.idx.data());
    Ahot.val.copy_from(As.val, stream);
    trace.mark("  gather transport: packed A_g (positions, renumbered indices)");
    build_gather_blocks(Ahot, blkA, t_m, WX);  // block 0 = first halves, block 1 = second halves
    if (!blkA.on()) {
      std::vector<int> hoff((size_t)m + 1);
      A.off.download(hoff.data(), stream);
      sync();
      build_bicsr(Ahot, hoff, stream, sms);
    }
    trace.mark("  gather transport: column blocks of the packed A_g");
    exchange_positions(posX, rk * nslice, nslice, sendX);
    build_send_lists(sendX, nslice, hx.half[rk], listX, planX);
    trace.mark("  gather transport: xbar send tables and lists");
    // y' side: the constraint rows this rank's rows of the global A^T touch
    std::vector<int> hoff = build_slice_transpose();
    trace.mark("  gather transport: rows J_g of the global A^T from the peers");
    const int WY = packed_positions(m_total, m_total, ATslice.nnz, ATslice.idx.data(), hy, posY);
    cntY         = 2 * WY;
    if ((size_t)cntY > yfull.size()) throw lp_error(error_type_t::RuntimeError, "gather transport: packed y' exceeds its buffer");
    if (ATslice.nnz > 0)
      k_remap_indices<<<ew_grid(ATslice.nnz, sms), EW_THREADS, 0, stream>>>(ATslice.nnz, ATslice.idx.data(), posY.data(),
                                                                            ATslice.idx.data());
    ATslice.cols = cntY;
    trace.mark("  gather transport: packed A^T slice (positions, renumbered indices)");
    build_gather_blocks(ATslice, blkATslice, t_slice, WY);
    if (!blkATslice.on()) build_bicsr(ATslice, hoff, stream, sms);
    trace.mark("  gather transport: column blocks of the A^T slice");
    exchange_positions(posY, row0[rk], m, sendY);
    build_send_lists(sendY, m, hy.half[rk], listY, planY);
    trace.mark("  gather transport: y' send tables and lists");
    check_launch();
    sync();
  }

  // ------------------------------------------------------------------------------ PDHG batches
  // Cuts the scaled matrix M into column blocks (device, stable) when the vector it gathers from exceeds the block size.
  // forced_width > 0 (gather transport): exactly two blocks, cut at that column, whatever the size of the gathered vector
  void build_gather_blocks(const csr_dev_t& M, gather_blocks_t& g, dvec<double>& t, int forced_width = 0)
  {
    g = gather_blocks_t{};
    const size_t bytes = (size_t)M.cols * sizeof(double);
    int B              = 1;
    if (forced_width > 0) {
      if (M.nnz == 0 || M.rows == 0) return;
      g.width = forced_width;
      B       = 2;
    } else {
      if (gather_block_bytes == 0 || bytes <= gather_block_bytes + gather_block_bytes / 2 || M.nnz == 0) return;
      B       = (int)std::min<size_t>(16, (bytes + gather_block_bytes - 1) / gather_block_bytes);
      g.width = (((M.cols + B - 1) / B) + 31) & ~31;
      B       = (M.cols + g.width - 1) / g.width;
    }
    if (B <= 1) return;
    g.B = B;
    g.blk.resize(B);
    std::vector<int*> offs(B), idxs(B);
    std::vector<double*> vals(B);
    std::vector<int> nnz_b(B, 0);
    for (int b = 0; b < B; ++b) {
      g.blk[b].rows = M.rows;
      g.blk[b].cols = M.cols;
      g.blk[b].off.resize((size_t)M.rows + 1);
      offs[b] = g.blk[b].off.data();
    }
    csr_split_columns_offsets(M.rows, M.off_ptr(), M.idx_ptr(), g.width, B, offs.data(), nnz_b.data(), stream);
    for (int b = 0; b < B; ++b) {
      g.blk[b].nnz = nnz_b[b];
      g.blk[b].idx.resize((size_t)nnz_b[b]);
      g.blk[b].val.resize((size_t)nnz_b[b]);
      idxs[b] = g.blk[b].idx.data();
      vals[b] = g.blk[b].val.data();
    }
    csr_split_columns_fill(M.rows, M.off_ptr(), M.idx_ptr(), M.val.data(), g.width, B, offs.data(), idxs.data(), vals.data(),
                           stream);
    std::vector<int> hoff((size_t)M.rows + 1);
    g.grid.resize(B);
    for (int b = 0; b < B; ++b) {
      g.blk[b].off.download(hoff.data(), stream);
      sync();
      build_bicsr(g.blk[b], hoff, stream, sms);
      g.grid[b] = spmv_grid(g.blk[b]);
    }
    t.resize((size_t)M.rows);
    t.zero(stream);
  }
  // t (+)= M_b * x for the column blocks [0, count), in block order
  void launch_block_passes(const gather_blocks_t& g, int count, const double* x0, const double* x1, int pick_candidate,
                           double* t, const unsigned long long* wait_flags, int n_wait)
  {
    for (int b = 0; b < count; ++b) {
      const csr_dev_t& M = g.blk[b];
      k_block_pass<<<g.grid[b], BICSR_THREADS, 0, stream>>>(d_ctl.data(), M.view(), x0, x1, pick_candidate, t, b == 0,
                                                            b == 0 ? wait_flags : nullptr, n_wait);
    }
  }
  // K2: one fused kernel; with gather blocking (B - 1) payload-free passes over the first column blocks, then the fused kernel
  // on the last block continuing their running sum.  wait_flags: peer transport (xbar slices of the peers)
  // bcast: gather transport, the fused kernel also stores y' into every rank's all-gathered y' buffer
  // wait_flags_b (gather transport): the second halves' flags, awaited by the kernel of the LAST column block
  void enqueue_k2(const unsigned long long* wait_flags, int n_wait, bool bcast = false,
                  const unsigned long long* wait_flags_b = nullptr)
  {
    const bool blocked  = blkA.on();
    const csr_dev_t& L  = blocked ? blkA.blk[blkA.B - 1] : hot_A();
    const int npre      = fused_npre(L);
    const int grid      = spmv_grid(L, npre);
    const double* t     = blocked ? t_m.data() : nullptr;
    const unsigned long long* wf = wait_flags_b ? wait_flags_b : (blocked ? nullptr : wait_flags);
    if (blocked) launch_block_passes(blkA, blkA.B - 1, xbar.data(), xbar.data(), 0, t_m.data(), wait_flags, n_wait);
#define CUOPT_K2(INIT, NPRE)                                                                                             \
  k_dual_step<INIT, NPRE><<<grid, BICSR_THREADS, 0, stream>>>(d_ctl.data(), L.view(), xbar.data(), ybuf[0].data(),       \
                                                              ybuf[1].data(), lcs.data(), ucs.data(), sum_y.data(),      \
                                                              part_dy2.data(), wf, n_wait, t)
#define CUOPT_K2B(INIT, NPRE)                                                                                            \
  k_dual_step<INIT, NPRE, true><<<grid, BICSR_THREADS, 0, stream>>>(d_ctl.data(), L.view(), xbar.data(), ybuf[0].data(), \
                                                                    ybuf[1].data(), lcs.data(), ucs.data(), sum_y.data(), \
                                                                    part_dy2.data(), wf, n_wait, t, p_yfull, p_flags,     \
                                                                    dist->world, dist->rank, sendY.data(), m)
    if (bcast) {
      if (blocked) { if (npre > 1) CUOPT_K2B(true, 2); else CUOPT_K2B(true, 1); }
      else { if (npre > 1) CUOPT_K2B(false, 2); else CUOPT_K2B(false, 1); }
    } else if (blocked) { if (npre > 1) CUOPT_K2(true, 2); else CUOPT_K2(true, 1); }
    else { if (npre > 1) CUOPT_K2(false, 2); else CUOPT_K2(false, 1); }
#undef CUOPT_K2B
#undef CUOPT_K2
  }
  int k2_grid() const
  {
    const csr_dev_t& L = blkA.on() ? blkA.blk[blkA.B - 1] : hot_A();
    return spmv_grid(L, fused_npre(L));
  }
  // K3 on one GPU: same structure, the step rule runs in the last CTA of the fused kernel
  void enqueue_k3()
  {
    const bool blocked = blkAT.on();
    const csr_dev_t& L = blocked ? blkAT.blk[blkAT.B - 1] : ATs;
    const int npre     = npre_override > 1 ? 2 : 1;  // two payload sets pay in K2 only (fused_npre), not in this last pass
    const int grid     = spmv_grid(L, npre);
    const double* t    = blocked ? t_n.data() : nullptr;
    if (blocked) launch_block_passes(blkAT, blkAT.B - 1, ybuf[0].data(), ybuf[1].data(), 1, t_n.data(), nullptr, 0);
#define CUOPT_K3(INIT, NPRE)                                                                                              \
  k_transpose_step<INIT, NPRE><<<grid, BICSR_THREADS, 0, stream>>>(d_ctl.data(), L.view(), ybuf[0].data(), ybuf[1].data(), \
                                                                   xbuf[0].data(), xbuf[1].data(), atybuf[0].data(),      \
                                                                   atybuf[1].data(), part_k3.data(), part_dy2.data(),     \
                                                                   n_part_dy2, t)
    if (blocked) { if (npre > 1) CUOPT_K3(true, 2); else CUOPT_K3(true, 1); }
    else { if (npre > 1) CUOPT_K3(false, 2); else CUOPT_K3(false, 1); }
#undef CUOPT_K3
  }
  int kernels_per_attempt() const
  {
    const int k2 = blkA.on() ? blkA.B : 1;
    if (!sharded()) return 1 + k2 + (blkAT.on() ? blkAT.B : 1);
    if (dist_mode == DIST_GATHER) return 1 + k2 + (blkATslice.on() ? blkATslice.B : 1) + 1 + (dist_send_kernel ? 2 : 0);
    const int k3p = blkAT.on() ? blkAT.B + (dist_mode == DIST_P2P ? 1 : 0) : 1;
    return 1 + k2 + k3p + (dist_mode == DIST_ALLREDUCE ? 2 : 2);
  }

  // partial A_g^T y' of this rank into dist_buf (NCCL transports); wide blocks when the shard's transpose is very sparse
  void launch_transpose_partial()
  {
    if (blkAT.on()) {  // the passes accumulate straight into the collective's send buffer
      launch_block_passes(blkAT, blkAT.B, ybuf[0].data(), ybuf[1].data(), 1, dist_buf.data(), nullptr, 0);
      return;
    }
    k_transpose_partial<<<grid_k3, BICSR_THREADS, 0, stream>>>(d_ctl.data(), ATs.view(), ybuf[0].data(), ybuf[1].data(),
                                                               dist_buf.data());
  }
  // out = M v
  void launch_spmv(const csr_dev_t& M, const double* v, double* out)
  {
    k_spmv<<<spmv_grid(M), BICSR_THREADS, 0, stream>>>(M.view(), v, out);
  }

  // scheme (ii): this rank updates only its slice of the primal side (kernel comments in pdlp_kernels.cuh)
  void enqueue_sliced_attempt()
  {
    const int j0 = slice_j0, G = dist->world, rk = dist->rank;
    double *x0 = xbuf[0].data() + j0, *x1 = xbuf[1].data() + j0, *a0 = atybuf[0].data() + j0, *a1 = atybuf[1].data() + j0;
    if (dist_mode == DIST_GATHER) {
      const unsigned long long* fl = d_flags.data();
      tr_tick(0);
      if (dist_send_kernel) {
        // K1 on the slice, then the xbar exchange on the communication stream: first halves -> flag A, second halves -> flag B
        k_primal_step<<<grid_slice, EW_THREADS, 0, stream>>>(d_ctl.data(), slice_n, x0, x1, a0, a1, cs.data() + j0,
                                                             ls.data() + j0, us.data() + j0, sum_x.data() + j0, xloc.data());
        CUOPT_CUDA_TRY(cudaEventRecord(ev_fork, stream));
        CUOPT_CUDA_TRY(cudaStreamWaitEvent(comm_stream, ev_fork, 0));
        k_send_packed<<<grid_send, EW_THREADS, 0, comm_stream>>>(d_ctl.data(), xloc.data(), xloc.data(), 0, listX.data(),
                                                                 sendX.data(), nslice, planX, p_xbar, p_flags, G, rk,
                                                                 DIST_FLAG_XBAR, DIST_FLAG_XBAR_B, d_ticket.data() + 4);
      } else {
        k_primal_step_bcast<<<grid_slice, EW_THREADS, 0, stream>>>(d_ctl.data(), slice_n, x0, x1, a0, a1, cs.data() + j0,
                                                                   ls.data() + j0, us.data() + j0, sum_x.data() + j0, p_xbar,
                                                                   p_flags, G, rk, sendX.data(), nslice);
      }
      tr_tick(1);
      // K2: the pass over column block 0 (first halves) runs while the second halves are still on the wire
      enqueue_k2(fl + DIST_FLAG_XBAR, G, !dist_send_kernel, fl + DIST_FLAG_XBAR_B);
      tr_tick(2);
      if (dist_send_kernel) {
        CUOPT_CUDA_TRY(cudaEventRecord(ev_fork, stream));
        CUOPT_CUDA_TRY(cudaStreamWaitEvent(comm_stream, ev_fork, 0));
        k_send_packed<<<grid_send, EW_THREADS, 0, comm_stream>>>(d_ctl.data(), ybuf[0].data(), ybuf[1].data(), 1, listY.data(),
                                                                 sendY.data(), m, planY, p_yfull, p_flags, G, rk,
                                                                 DIST_FLAG_PARTIAL, DIST_FLAG_Y_B, d_ticket.data() + 4);
        CUOPT_CUDA_TRY(cudaEventRecord(ev_join, comm_stream));
      }
      // K3 on this rank's rows of the global A^T, gathering from the packed y'; its last CTA sends this rank's three scalars
      const bool blocked = blkATslice.on();
      const csr_dev_t& L = blocked ? blkATslice.blk[blkATslice.B - 1] : ATslice;
      const int grid     = spmv_grid(L, 1);
      if (blocked)
        launch_block_passes(blkATslice, blkATslice.B - 1, yfull.data(), yfull.data(), 0, t_slice.data(), fl + DIST_FLAG_PARTIAL, G);
#define CUOPT_K3S(INIT)                                                                                                     \
  k_transpose_step_slice<INIT, 1><<<grid, BICSR_THREADS, 0, stream>>>(                                                      \
    d_ctl.data(), L.view(), yfull.data(), x0, x1, a0, a1, part_k3.data(), part_dy2.data(), n_part_dy2,                      \
    blocked ? t_slice.data() : nullptr, fl + DIST_FLAG_Y_B, G, p_scal, p_flags, G, rk)
      if (blocked) CUOPT_K3S(true); else CUOPT_K3S(false);
#undef CUOPT_K3S
      tr_tick(3);
      k_step_rule_gather<<<1, 32, 0, stream>>>(d_ctl.data(), scal.data(), G, d_flags.data() + DIST_FLAG_SCALARS);
      if (dist_send_kernel) CUOPT_CUDA_TRY(cudaStreamWaitEvent(stream, ev_join, 0));  // the communication stream joins
      tr_tick(4);
      tr_close(4);
      return;
    }
    if (dist_mode == DIST_P2P) {
      tr_tick(0);
      k_primal_step_bcast<<<grid_slice, EW_THREADS, 0, stream>>>(d_ctl.data(), slice_n, x0, x1, a0, a1, cs.data() + j0,
                                                                 ls.data() + j0, us.data() + j0, sum_x.data() + j0, p_xbar,
                                                                 p_flags, G, rk);
      tr_tick(1);
      enqueue_k2(d_flags.data() + DIST_FLAG_XBAR, G);
      tr_tick(2);
      if (blkAT.on()) {
        launch_block_passes(blkAT, blkAT.B, ybuf[0].data(), ybuf[1].data(), 1, t_n.data(), nullptr, 0);
        k_scatter_partials<<<grid_n, EW_THREADS, 0, stream>>>(d_ctl.data(), n, t_n.data(), p_stage, nslice, p_flags, G, rk);
      } else
        k_transpose_partial_scatter<<<grid_k3, BICSR_THREADS, 0, stream>>>(d_ctl.data(), ATs.view(), ybuf[0].data(),
                                                                          ybuf[1].data(), p_stage, nslice, p_flags, G, rk);
      k_interaction_slice<<<grid_slice, EW_THREADS, 0, stream>>>(d_ctl.data(), slice_n, stage.data(), G, (size_t)nslice, x0, x1,
                                                                 a0, a1, part_k3.data(), part_dy2.data(), n_part_dy2,
                                                                 d_flags.data() + DIST_FLAG_PARTIAL, p_scal, p_flags, G, rk);
      tr_tick(3);
      k_step_rule_gather<<<1, 32, 0, stream>>>(d_ctl.data(), scal.data(), G, d_flags.data() + DIST_FLAG_SCALARS);
      tr_tick(4);
      tr_close(4);
      return;
    }
    k_primal_step<<<grid_slice, EW_THREADS, 0, stream>>>(d_ctl.data(), slice_n, x0, x1, a0, a1, cs.data() + j0,
                                                         ls.data() + j0, us.data() + j0, sum_x.data() + j0,
                                                         xbar.data() + j0);
    dist->allgather(xbar.data(), nslice, stream);
    enqueue_k2(nullptr, 0);
    launch_transpose_partial();
    dist->reduce_scatter(dist_buf.data(), rs_buf.data(), nslice, stream);
    peer_flags_t no_flags{};
    k_interaction_slice<<<grid_slice, EW_THREADS, 0, stream>>>(d_ctl.data(), slice_n, rs_buf.data(), 1, 0, x0, x1, a0, a1,
                                                               part_k3.data(), part_dy2.data(), n_part_dy2, nullptr, p_scal,
                                                               no_flags, 1, rk);
    dist->allreduce(scal.data(), 3, false, stream);
    k_step_rule_gather<<<1, 32, 0, stream>>>(d_ctl.data(), scal.data(), 1, nullptr);
  }

  void enqueue_attempt()
  {
    if (sharded() && dist_mode != DIST_ALLREDUCE) {
      enqueue_sliced_attempt();
      return;
    }
    k_primal_step<<<grid_k1, EW_THREADS, 0, stream>>>(d_ctl.data(), n, xbuf[0].data(), xbuf[1].data(), atybuf[0].data(),
                                                      atybuf[1].data(), cs.data(), ls.data(), us.data(), sum_x.data(),
                                                      xbar.data());
    enqueue_k2(nullptr, 0);
    if (!sharded()) {
      enqueue_k3();
      return;
    }
    // row-sharded: partial A_g^T y'_g and this rank's ||dy||^2 -> one all-reduce of n + 1 doubles -> K3b
    launch_transpose_partial();
    k_sum_partials<<<1, EW_THREADS, 0, stream>>>(d_ctl.data(), part_dy2.data(), n_part_dy2, 1, dist_buf.data() + n);
    dist->allreduce(dist_buf.data(), (size_t)n + 1, false, stream);
    k_interaction_step<<<grid_n, EW_THREADS, 0, stream>>>(d_ctl.data(), n, dist_buf.data(), xbuf[0].data(), xbuf[1].data(),
                                                          atybuf[0].data(), atybuf[1].data(), part_k3.data());
  }

  void launch_attempts(int count)
  {
    if (count <= 0) return;
    launches += (long long)kernels_per_attempt() * count;  // kernels; collectives are not counted
    if (!use_graphs || count == 1) {
      for (int i = 0; i < count; ++i) enqueue_attempt();
      check_launch();
      return;
    }
    auto it = graphs.find(count);
    if (it == graphs.end()) {
      cudaGraph_t g;
      CUOPT_CUDA_TRY(cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal));
      for (int i = 0; i < count; ++i) enqueue_attempt();
      CUOPT_CUDA_TRY(cudaStreamEndCapture(stream, &g));
      cudaGraphExec_t ge;
      CUOPT_CUDA_TRY(cudaGraphInstantiate(&ge, g, 0));
      cudaGraphDestroy(g);
      it = graphs.emplace(count, ge).first;
    }
    CUOPT_CUDA_TRY(cudaGraphLaunch(it->second, stream));
  }

  void fetch_ctl()
  {
    CUOPT_CUDA_TRY(cudaMemcpyAsync(h_ctl, d_ctl.data(), sizeof(pdhg_ctl_t), cudaMemcpyDeviceToHost, stream));
    sync();
  }

  // take_step x `steps` (pdlp.cu:1188-1222): returns when `steps` more steps were accepted or an error was flagged.
  void run_steps(int steps)
  {
    if (steps <= 0) return;
    nvtx_range_t nvtx_scope("take_step batch (PDHG attempts up to the next major iteration)");
    CUOPT_CUDA_TRY(cudaEventRecord(ev_a, stream));
    if (need_aty) {  // pdhg.cu:183-202
      const int cur = h_ctl->parity;
      launch_spmv(ATs, ybuf[cur].data(), atybuf[cur].data());
      if (sharded()) dist->allreduce(atybuf[cur].data(), n, false, stream);
      ++launches;
      need_aty = false;
    }
    k_begin_batch<<<1, 1, 0, stream>>>(d_ctl.data(), steps);
    const int target = h_ctl->accepted + steps;
    int todo         = steps;
    while (true) {
      // a couple of spare attempts cover the occasional rejected step without another round trip
      launch_attempts(todo + (todo >= 16 ? 2 : 0));
      const bool sliced = sharded() && dist_mode != DIST_ALLREDUCE;
      const int fj0 = sliced ? slice_j0 : 0, fn = sliced ? slice_n : n;
      k_flush_average<<<grid_misc, EW_THREADS, 0, stream>>>(d_ctl.data(), fn, xbuf[0].data() + fj0, xbuf[1].data() + fj0,
                                                            sum_x.data() + fj0, m, ybuf[0].data(), ybuf[1].data(),
                                                            sum_y.data());
      k_clear_pending<<<1, 1, 0, stream>>>(d_ctl.data());
      launches += 3;
      check_launch();
      fetch_ctl();
      if (h_ctl->valid == -1 || h_ctl->accepted >= target) break;
      todo = target - h_ctl->accepted;
    }
    if (sharded() && dist_mode != DIST_ALLREDUCE) {
      // back to the replicated representation the major-iteration code works on: every rank receives the other
      // slices of the current iterate, its A^T y and the running sum (3 all-gathers per batch of ~40 attempts)
      const int cur = h_ctl->parity;
      dist->allgather(xbuf[cur].data(), nslice, stream);
      dist->allgather(atybuf[cur].data(), nslice, stream);
      dist->allgather(sum_x.data(), nslice, stream);
    }
    CUOPT_CUDA_TRY(cudaEventRecord(ev_b, stream));
    CUOPT_CUDA_TRY(cudaEventSynchronize(ev_b));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev_a, ev_b);
    sol.stats.pdhg_loop_seconds += ms * 1e-3;
  }

  // ------------------------------------------------------------------------- major iteration
  eval_consts_t eval_consts() const
  {
    eval_consts_t k;
    k.objective_scaling_factor = obj_scale;
    k.objective_offset         = obj_offset;
    k.abs_gap_tol              = st.absolute_gap_tolerance;
    k.rel_gap_tol              = st.relative_gap_tolerance;
    k.abs_primal_tol           = st.absolute_primal_tolerance;
    k.rel_primal_tol           = st.relative_primal_tolerance;
    k.abs_dual_tol             = st.absolute_dual_tolerance;
    k.rel_dual_tol             = st.relative_dual_tolerance;
    k.l2_norm_b                = l2_norm_b;
    k.l2_norm_c                = l2_norm_c;
    k.reduced_cost_rule        = hp.handle_some_primal_gradients_on_finite_bounds_as_residuals ? 1 : 0;
    k.per_constraint_residual  = st.per_constraint_residual ? 1 : 0;
    k.primal_infeasible_tol    = st.primal_infeasible_tolerance;
    k.dual_infeasible_tol      = st.dual_infeasible_tolerance;
    return k;
  }

  // averages, in-place unscaling, evaluation of current and average (pdlp.cu:1103-1142 up to check_termination's inputs)
  void evaluate_iterates()
  {
    nvtx_range_t nvtx_scope("compute_convergence_information (current + average)");
    const int cur  = h_ctl->parity;
    // pdlp.cu:1100-1129: warm start given and no step taken yet => the averages handed in are used as they are
    const int mode = (warm_started && h_ctl->accepted == 0) ? 2 : (h_ctl->accepted <= 1) ? 0 : 1;
    k_average_and_unscale<<<grid_n, EW_THREADS, 0, stream>>>(d_ctl.data(), mode, n, xbuf[cur].data(), sum_x.data(),
                                                             x_avg.data(), Dc.data());
    k_average_and_unscale<<<grid_m, EW_THREADS, 0, stream>>>(d_ctl.data(), mode, m, ybuf[cur].data(), sum_y.data(),
                                                             y_avg.data(), Dr.data());
    launch_spmv(A, xbuf[cur].data(), eval_m.data());
    launch_spmv(A, x_avg.data(), eval_m.data() + m);
    k_eval_rows_from_ax<<<grid_m, EW_THREADS, 0, stream>>>(m, eval_m.data(), eval_m.data() + m, ybuf[cur].data(),
                                                           y_avg.data(), lc.data(), uc.data(), part_rows.data(),
                                                           st.relative_primal_tolerance,
                                                           st.per_constraint_residual ? part_max.data() : nullptr);
    const int n_rows_parts = grid_m;
    launches += 2;
    {
      // A^T y for both iterates, then the column math element-wise.  Row-sharded: the six row sums and both products
      // are partial and are combined over the ranks first.
      double* aty2            = sharded() ? dist_buf.data() : eval_n.data();
      const double* rows_src  = part_rows.data();
      int rows_count          = n_rows_parts;
      if (sharded()) {
        k_sum_partials<<<1, EW_THREADS, 0, stream>>>(nullptr, part_rows.data(), n_rows_parts, 6, d_scalar.data());
        dist->allreduce(d_scalar.data(), 6, false, stream);
        rows_src   = d_scalar.data();
        rows_count = 1;
      }
      launch_spmv(AT, ybuf[cur].data(), aty2);
      launch_spmv(AT, y_avg.data(), aty2 + n);
      if (sharded()) dist->allreduce(aty2, 2 * (size_t)n, false, stream);
      double* max_cols       = nullptr;
      const double* max_rows = nullptr;
      int max_rows_count     = 0;
      if (st.per_constraint_residual) {
        max_rows       = part_max.data();
        max_rows_count = grid_m;
        max_cols       = part_max.data() + 2 * (size_t)std::max(grid_m, grid_n);
        if (sharded()) {  // the row maxima of the other ranks' blocks
          k_max_partials<<<1, EW_THREADS, 0, stream>>>(part_max.data(), grid_m, 2, d_scalar.data() + 8);
          dist->allreduce(d_scalar.data() + 8, 2, true, stream);
          max_rows       = d_scalar.data() + 8;
          max_rows_count = 1;
        }
      }
      k_eval_cols_from_aty<<<grid_n, EW_THREADS, 0, stream>>>(d_ctl.data(), n, aty2, aty2 + n, xbuf[cur].data(), x_avg.data(),
                                                              c.data(), l.data(), u.data(), rc_cur.data(), rc_avg.data(),
                                                              part_cols.data(), rows_src, rows_count, eval_consts(),
                                                              d_eval.data(), max_cols, max_rows, max_rows_count);
      launches += 3;
      if (st.detect_infeasibility) {  // single GPU only (checked in build)
        double* rows_parts = part_infeas.data();
        double* cols_parts = part_infeas.data() + 6 * (size_t)grid_m;
        k_infeasibility_rows<<<grid_m, EW_THREADS, 0, stream>>>(m, eval_m.data(), eval_m.data() + m, ybuf[cur].data(),
                                                                y_avg.data(), lc.data(), uc.data(), rows_parts);
        k_infeasibility_cols<<<grid_n, EW_THREADS, 0, stream>>>(d_ctl.data(), n, aty2, aty2 + n, xbuf[cur].data(),
                                                                x_avg.data(), c.data(), l.data(), u.data(), cols_parts,
                                                                rows_parts, grid_m, eval_consts(), d_eval.data());
        launches += 2;
      }
    }
    launches += 4;
    check_launch();
    CUOPT_CUDA_TRY(cudaMemcpyAsync(h_eval, d_eval.data(), 2 * sizeof(eval_t), cudaMemcpyDeviceToHost, stream));
    sync();
  }

  void fill_solution(bool average, termination_status_t status)  // termination_strategy.cu:270-357
  {
    const int cur   = h_ctl->parity;
    const eval_t& e = h_eval[average ? 1 : 0];
    sol.primal.resize(n);
    sol.dual.resize(m);
    sol.reduced_cost.resize(n);
    (average ? x_avg : xbuf[cur]).download(sol.primal.data(), stream);
    (average ? y_avg : ybuf[cur]).download(sol.dual.data(), stream);
    (average ? rc_avg : rc_cur).download(sol.reduced_cost.data(), stream);
    fetch_ctl();
    sol.termination_status                    = status;
    sol.error_status                          = 0;
    lp_stats_t& s                             = sol.stats;
    s.number_of_steps_taken                   = h_ctl->accepted;
    s.total_number_of_attempted_steps         = h_ctl->attempts;
    s.l2_primal_residual                      = e.l2_primal_residual;
    s.l2_dual_residual                        = e.l2_dual_residual;
    s.l2_relative_primal_residual             = e.l2_primal_residual / (1.0 + l2_norm_b);
    s.l2_relative_dual_residual               = e.l2_dual_residual / (1.0 + l2_norm_c);
    s.primal_objective                        = e.primal_objective;
    s.dual_objective                          = e.dual_objective;
    s.gap                                     = e.gap;
    s.relative_gap                            = e.gap / (1.0 + std::fabs(e.primal_objective) + std::fabs(e.dual_objective));
    s.solved_by_pdlp                          = 1;
    s.final_step_size                         = h_ctl->step_size;
    s.final_primal_weight                     = h_ctl->primal_weight;
    s.kernel_launches                         = launches;
    if (st.capture_warm_start) capture_warm_start();
    finished                                  = true;
  }

  // ---- save_best_primal_so_far (pdlp.cu:333-463): the best of {current, average} by primal quality at every major
  // iteration that did not terminate, returned instead of the current iterate when a limit is hit (:265-331) ----
  struct quality_t {
    bool feasible    = false;
    double residual  = std::numeric_limits<double>::infinity();
    double objective = std::numeric_limits<double>::infinity();  // -inf when maximising
  };
  quality_t best_quality;
  bool have_best = false;
  dvec<double> best_x, best_y, best_rc;
  eval_t best_eval{};
  int best_accepted = 0, best_attempts = 0;
  bool first_is_better(const quality_t& a, const quality_t& b) const  // get_best_quality(current = a, other = b) == a
  {
    if (a.feasible && !b.feasible) return true;
    if (!a.feasible && b.feasible) return false;
    if (a.feasible && b.feasible) {
      const bool lower = a.objective < b.objective;
      return (!maximize && lower) || (maximize && !lower);
    }
    return a.residual < b.residual;
  }
  void record_best_primal_so_far()
  {
    if (!have_best && maximize) best_quality.objective = -std::numeric_limits<double>::infinity();
    const quality_t qc{h_eval[0].status == 7, h_eval[0].l2_primal_residual, h_eval[0].primal_objective};
    const quality_t qa{h_eval[1].status == 7, h_eval[1].l2_primal_residual, h_eval[1].primal_objective};
    const bool cur_wins   = first_is_better(qc, qa);
    const quality_t& cand = cur_wins ? qc : qa;
    if (!first_is_better(cand, best_quality)) return;
    best_quality  = cand;
    const int cur = h_ctl->parity;
    best_x.copy_from(cur_wins ? xbuf[cur] : x_avg, stream);  // unscaled at this point, like fill_solution's sources
    best_y.copy_from(cur_wins ? ybuf[cur] : y_avg, stream);
    best_rc.copy_from(cur_wins ? rc_cur : rc_avg, stream);
    best_eval     = h_eval[cur_wins ? 0 : 1];
    best_accepted = h_ctl->accepted;  // the reference fills the returned solution at record time (:441-447)
    best_attempts = h_ctl->attempts;
    have_best     = true;
  }
  bool fill_best_solution(termination_status_t status)
  {
    if (!(st.save_best_primal_so_far && have_best)) return false;
    sol.primal.resize(n);
    sol.dual.resize(m);
    sol.reduced_cost.resize(n);
    CUOPT_CUDA_TRY(cudaMemcpyAsync(sol.primal.data(), best_x.data(), (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, stream));
    CUOPT_CUDA_TRY(cudaMemcpyAsync(sol.dual.data(), best_y.data(), (size_t)m * sizeof(double), cudaMemcpyDeviceToHost, stream));
    CUOPT_CUDA_TRY(cudaMemcpyAsync(sol.reduced_cost.data(), best_rc.data(), (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, stream));
    fetch_ctl();
    const eval_t& e                   = best_eval;
    sol.termination_status            = status;
    sol.error_status                  = 0;
    lp_stats_t& s                     = sol.stats;
    s.number_of_steps_taken           = best_accepted;
    s.total_number_of_attempted_steps = best_attempts;
    s.l2_primal_residual              = e.l2_primal_residual;
    s.l2_dual_residual                = e.l2_dual_residual;
    s.l2_relative_primal_residual     = e.l2_primal_residual / (1.0 + l2_norm_b);
    s.l2_relative_dual_residual       = e.l2_dual_residual / (1.0 + l2_norm_c);
    s.primal_objective                = e.primal_objective;
    s.dual_objective                  = e.dual_objective;
    s.gap                             = e.gap;
    s.relative_gap                    = e.gap / (1.0 + std::fabs(e.primal_objective) + std::fabs(e.dual_objective));
    s.solved_by_pdlp                  = 1;
    s.final_step_size                 = h_ctl->step_size;
    s.final_primal_weight             = h_ctl->primal_weight;
    s.kernel_launches                 = launches;
    if (st.capture_warm_start) capture_warm_start();  // continuing after a limit is the main use of a warm start
    finished                          = true;
    return true;
  }

  bool check_limits()  // pdlp.cu:265-331
  {
    bool out_of_time = now_seconds() - t_start >= st.time_limit;
    if (sharded() && std::isfinite(st.time_limit)) {  // every rank must take the same branch: any rank over => all stop
      h_scalar[1] = out_of_time ? 1.0 : 0.0;
      CUOPT_CUDA_TRY(cudaMemcpyAsync(d_scalar.data() + 7, h_scalar + 1, sizeof(double), cudaMemcpyHostToDevice, stream));
      dist->allreduce(d_scalar.data() + 7, 1, true, stream);
      CUOPT_CUDA_TRY(cudaMemcpyAsync(h_scalar + 1, d_scalar.data() + 7, sizeof(double), cudaMemcpyDeviceToHost, stream));
      sync();
      out_of_time = h_scalar[1] > 0.5;
    }
    if (out_of_time) {
      if (!fill_best_solution(termination_status_t::TimeLimit)) fill_solution(false, termination_status_t::TimeLimit);
      return true;
    }
    if (h_ctl->accepted >= st.iteration_limit) {
      if (!fill_best_solution(termination_status_t::IterationLimit)) fill_solution(false, termination_status_t::IterationLimit);
      return true;
    }
    return false;
  }

  bool check_termination()  // pdlp.cu:538-802
  {
    nvtx_range_t nvtx_scope("Check termination");
    if (total_pdlp_iterations <= 1) return check_limits();
    const int sc = h_eval[0].status, sa = h_eval[1].status;
    if (st.first_primal_feasible) {  // :587-633
      if (sa == 7 && sc == 7) {
        fill_solution(!(h_eval[0].l2_primal_residual < h_eval[1].l2_primal_residual), termination_status_t::PrimalFeasible);
        return true;
      } else if (sc == 7) {
        fill_solution(false, termination_status_t::PrimalFeasible);
        return true;
      } else if (sa == 7) {
        fill_solution(true, termination_status_t::PrimalFeasible);
        return true;
      }
    }
    if (sa == 1 && sc == 1) {
      fill_solution(!(h_eval[0].kkt < h_eval[1].kkt), termination_status_t::Optimal);
      return true;
    }
    if (sa == 1) { fill_solution(true, termination_status_t::Optimal); return true; }
    if (sc == 1) { fill_solution(false, termination_status_t::Optimal); return true; }
    if (st.detect_infeasibility) {  // pdlp.cu:716-770: strict -> either iterate suffices, else both must agree
      const bool ic = sc == 2 || sc == 3, ia = sa == 2 || sa == 3;
      if (st.strict_infeasibility) {
        if (ic) { fill_solution(false, static_cast<termination_status_t>(sc)); return true; }
        if (ia) { fill_solution(true, static_cast<termination_status_t>(sa)); return true; }
      } else if (ic && sc == sa) {
        fill_solution(false, static_cast<termination_status_t>(sc));
        return true;
      }
    }
    if (h_ctl->valid == -1) {  // :780-789
      fetch_ctl();
      const lp_stats_t kept                      = sol.stats;  // setup / loop times, restarts, major iterations so far
      sol                                        = lp_solution_t{};
      sol.stats                                  = kept;
      sol.termination_status                     = termination_status_t::NumericalError;
      sol.stats.number_of_steps_taken            = h_ctl->accepted;
      sol.stats.total_number_of_attempted_steps  = h_ctl->attempts;
      sol.stats.kernel_launches                  = launches;
      finished                                   = true;
      return true;
    }
    if (st.save_best_primal_so_far) record_best_primal_so_far();  // pdlp.cu:790-796
    return check_limits();
  }

  // ---- trust-region restart (Methodical1): mirrors oracle_t::run_trust_region_restart ----
  double tr_weighted_distance(double pd, double dd) const  // pdlp_restart_strategy.cu:804-817
  {
    const double w = h_ctl->primal_weight;
    return std::sqrt(pd * hp.primal_distance_smoothing * w + dd * (hp.dual_distance_smoothing / w));
  }
  void tr_distances(tr_gap_t& g)  // :1681-1714
  {
    k_restart_distance_and_weight<<<grid_misc, EW_THREADS, 0, stream>>>(d_ctl.data(), n, g.px, x_lr.data(), m, g.py,
                                                                        y_lr.data(), hp.primal_weight_update_smoothing,
                                                                        part_misc.data(), d_scalar.data());
    CUOPT_CUDA_TRY(cudaMemcpyAsync(h_scalar, d_scalar.data(), 2 * sizeof(double), cudaMemcpyDeviceToHost, stream));
    sync();
    g.pd   = h_scalar[0];
    g.dd   = h_scalar[1];
    g.dist = tr_weighted_distance(g.pd, g.dd);
  }
  void tr_bound(tr_gap_t& g)  // bound_optimal_objective, :1034-1051
  {
    nvtx_range_t nvtx_scope("bound_optimal_objective");
    const int N = n + m;
    launch_spmv(ATs, g.py, tr_aty.data());
    launch_spmv(As, g.px, tr_ax.data());
    h_scalar[0] = g.dist;
    CUOPT_CUDA_TRY(cudaMemcpyAsync(tr_scal.data() + 5, h_scalar, sizeof(double), cudaMemcpyHostToDevice, stream));
    tr_problem_t P{n, m, g.px, g.py, tr_aty.data(), tr_ax.data(), cs.data(), ls.data(), us.data(), lcs.data(), ucs.data()};
    k_tr_prepare<<<grid_tr, EW_THREADS, 0, stream>>>(d_ctl.data(), P, tr_dir.data(), tr_thr.data(), tr_grad.data(),
                                                     tr_iota.data(), tr_parts.data(), tr_scal.data());
    CUOPT_CUDA_TRY(cudaMemcpyAsync(h_scalar, tr_scal.data() + 3, sizeof(double), cudaMemcpyDeviceToHost, stream));
    sync();
    const bool degenerate = g.dist == 0.0 || h_scalar[0] == 0.0;  // :1420-1431
    if (!degenerate) {
      sort_keys_with_index(N, tr_thr.data(), tr_thr_sorted.data(), tr_iota.data(), tr_perm.data(), stream);
      k_tr_weights<<<grid_tr, EW_THREADS, 0, stream>>>(d_ctl.data(), n, N, tr_thr_sorted.data(), tr_perm.data(),
                                                       tr_dir.data(), tr_A.data(), tr_B.data());
      inclusive_sum_in_place(N, tr_A.data(), stream);
      inclusive_sum_in_place(N, tr_B.data(), stream);
      k_tr_bisect<<<1, 1, 0, stream>>>(N, tr_thr_sorted.data(), tr_A.data(), tr_B.data(), tr_scal.data());
    }
    k_tr_bounds<<<grid_tr, EW_THREADS, 0, stream>>>(d_ctl.data(), P, tr_dir.data(), tr_grad.data(), degenerate ? 1 : 0,
                                                    tr_parts.data(), tr_scal.data());
    check_launch();
    CUOPT_CUDA_TRY(cudaMemcpyAsync(h_scalar, tr_scal.data() + 7, 2 * sizeof(double), cudaMemcpyDeviceToHost, stream));
    sync();
    g.lower = h_scalar[0];
    g.upper = h_scalar[1];
    launches += degenerate ? 4 : 6;
  }
  void trust_region_restart()  // pdlp_restart_strategy.cu:278-364
  {
    nvtx_range_t nvtx_scope("run trust region restart");
    if (h_ctl->its_since_restart == 0) return;
    const int cur = h_ctl->parity;
    bool restart  = should_do_artificial_restart(total_pdlp_iterations);
    tr_gap_t avg{x_avg.data(), y_avg.data()}, curg{xbuf[cur].data(), ybuf[cur].data()};
    tr_distances(avg);
    tr_distances(curg);
    tr_bound(avg);
    tr_bound(curg);
    avg.ngap  = (avg.upper - avg.lower) / avg.dist;
    curg.ngap = (curg.upper - curg.lower) / curg.dist;
    const bool to_avg = curg.ngap / curg.dist >= avg.ngap / avg.dist;  // pick_restart_candidate :842-873
    tr_gap_t& cand    = to_avg ? avg : curg;
    if (!restart) {  // should_do_adaptive_restart_normalized_duality_gap :903-937
      tr_gap_t last{x_lr.data(), y_lr.data()};
      last.pd   = cand.pd;
      last.dd   = cand.dd;
      last.dist = tr_weighted_distance(cand.pd, cand.dd);
      tr_bound(last);
      last.ngap          = (last.upper - last.lower) / last.dist;
      const double ratio = cand.ngap / last.ngap;
      if (ratio < hp.necessary_reduction_for_restart &&
          (ratio < hp.sufficient_reduction_for_restart || ratio > tr_gap_reduction_last_trial))
        restart = true;
      tr_gap_reduction_last_trial = ratio;
    }
    if (!restart) return;
    const bool use_avg = to_avg && !hp.never_restart_to_average;
    dvec<double>& cx   = to_avg ? x_avg : xbuf[cur];  // the candidate: new restart point and source of the weight update
    dvec<double>& cy   = to_avg ? y_avg : ybuf[cur];
    k_restart_distance_and_weight<<<grid_misc, EW_THREADS, 0, stream>>>(d_ctl.data(), n, cx.data(), x_lr.data(), m,
                                                                        cy.data(), y_lr.data(),
                                                                        hp.primal_weight_update_smoothing,
                                                                        part_misc.data(), nullptr);
    if (use_avg) {
      xbuf[cur].copy_from(x_avg, stream);
      ybuf[cur].copy_from(y_avg, stream);
      need_aty = true;
    }
    last_restart_was_average = use_avg;
    x_lr.copy_from(cx, stream);
    y_lr.copy_from(cy, stream);
    sum_x.zero(stream);
    sum_y.zero(stream);
    k_reset_after_restart<<<1, 1, 0, stream>>>(d_ctl.data());
    launches += 2;
    check_launch();
    sol.stats.n_restarts += 1;
    fetch_ctl();
  }

  bool should_do_artificial_restart(int total_iterations) const  // pdlp_restart_strategy.cu:940-961
  {
    return h_ctl->its_since_restart >= hp.default_artificial_restart_threshold * total_iterations;
  }

  void kkt_restart()  // pdlp_restart_strategy.cu:468-641
  {
    nvtx_range_t nvtx_scope("compute_restart");
    const int cur        = h_ctl->parity;
    const double kkt_cur = h_eval[0].kkt;
    if (h_ctl->its_since_restart == 0) {
      last_candidate_kkt = kkt_cur;
      last_restart_kkt   = kkt_cur;
      return;
    }
    const double kkt_avg = h_eval[1].kkt;
    const bool to_avg    = !(kkt_cur < kkt_avg);
    const double cand    = to_avg ? kkt_avg : kkt_cur;
    const bool decay     = cand < hp.sufficient_reduction_for_restart * last_restart_kkt ||
                       (cand < hp.necessary_reduction_for_restart * last_restart_kkt && cand > last_candidate_kkt);
    if (should_do_artificial_restart(total_pdlp_iterations) || decay) {
      const bool use_avg = to_avg && !hp.never_restart_to_average;
      dvec<double>& cx   = use_avg ? x_avg : xbuf[cur];
      dvec<double>& cy   = use_avg ? y_avg : ybuf[cur];
      k_restart_distance_and_weight<<<grid_misc, EW_THREADS, 0, stream>>>(
        d_ctl.data(), n, cx.data(), x_lr.data(), m, cy.data(), y_lr.data(), hp.primal_weight_update_smoothing,
        part_misc.data(), sharded() ? d_scalar.data() : nullptr);
      if (sharded()) {  // the dual distance is a sum over the row blocks of all ranks; the primal one is replicated
        dist->allreduce(d_scalar.data() + 1, 1, false, stream);
        k_update_primal_weight<<<1, 1, 0, stream>>>(d_ctl.data(), d_scalar.data(), hp.primal_weight_update_smoothing);
      }
      if (use_avg) {
        xbuf[cur].copy_from(x_avg, stream);
        ybuf[cur].copy_from(y_avg, stream);
        need_aty = true;
      }
      last_restart_was_average = use_avg;
      x_lr.copy_from(cx, stream);
      y_lr.copy_from(cy, stream);
      sum_x.zero(stream);
      sum_y.zero(stream);
      k_reset_after_restart<<<1, 1, 0, stream>>>(d_ctl.data());
      launches += 2;
      check_launch();
      last_restart_kkt = cand;
      sol.stats.n_restarts += 1;
      fetch_ctl();
    }
    last_candidate_kkt = cand;
  }

  // number of PDHG steps until the outer loop has to look at the iterate again
  int steps_until_next_check() const
  {
    const int k = total_pdlp_iterations;
    int t       = 1;
    while (true) {
      const int kk = k + t;
      if (((kk % hp.major_iteration == 0) && kk > 0) || kk <= hp.min_iteration_restart) break;
      if (hp.artificial_restart_in_main_loop &&
          (h_ctl->its_since_restart + t) >= hp.default_artificial_restart_threshold * kk)
        break;
      ++t;
    }
    return t;
  }

  // pdlp.cu:1081-1185.  budget < 0: run to termination; otherwise stop after `budget` accepted steps.
  bool outer_loop(int budget)
  {
    initialise();
    if (finished) return true;
    if (t_start == 0.0) t_start = now_seconds();
    while (true) {
      const int k          = total_pdlp_iterations;
      const bool is_major  = ((k % hp.major_iteration == 0) && k > 0) || (k <= hp.min_iteration_restart);
      const bool error     = h_ctl->valid == -1;
      const bool artificial = hp.artificial_restart_in_main_loop && should_do_artificial_restart(k);
      if (is_major || artificial || error) {
        CUOPT_CUDA_TRY(cudaEventRecord(ev_a, stream));
        sol.stats.n_major_iterations += 1;
        evaluate_iterates();
        if (check_termination()) return true;
        const int cur = h_ctl->parity;
        if (hp.rescale_for_restart) {  // pdlp.cu:1144-1149
          k_scale_back<<<grid_n, EW_THREADS, 0, stream>>>(n, x_avg.data(), Dc.data());
          k_scale_back<<<grid_m, EW_THREADS, 0, stream>>>(m, y_avg.data(), Dr.data());
          k_scale_back<<<grid_n, EW_THREADS, 0, stream>>>(n, xbuf[cur].data(), Dc.data());
          k_scale_back<<<grid_m, EW_THREADS, 0, stream>>>(m, ybuf[cur].data(), Dr.data());
          launches += 4;
        }
        if (hp.restart_strategy == 1) kkt_restart();
        else if (hp.restart_strategy == 2) {
          trust_region_restart();  // trust_region.cuh
        }
        if (!hp.rescale_for_restart) {  // pdlp.cu:1168-1175
          k_scale_back<<<grid_n, EW_THREADS, 0, stream>>>(n, xbuf[cur].data(), Dc.data());
          k_scale_back<<<grid_m, EW_THREADS, 0, stream>>>(m, ybuf[cur].data(), Dr.data());
          launches += 2;
        }
        check_launch();
        CUOPT_CUDA_TRY(cudaEventRecord(ev_b, stream));
        CUOPT_CUDA_TRY(cudaEventSynchronize(ev_b));
        float ms = 0.f;
        cudaEventElapsedTime(&ms, ev_a, ev_b);
        sol.stats.termination_seconds += ms * 1e-3;
      }
      if (budget == 0) return false;
      int steps = steps_until_next_check();
      if (budget > 0) steps = std::min(steps, budget);
      const int before = h_ctl->accepted;
      run_steps(steps);
      const int done = h_ctl->accepted - before;
      total_pdlp_iterations += done;
      if (budget > 0) budget -= done;
      if (h_ctl->valid == -1 && done < steps) {
        // the batch stopped on a numerical error: the reference's loop would now hit `error_occured`
      }
    }
  }
};

// ------------------------------------------------------------------------------------------------
pdlp_solver_t::pdlp_solver_t(const lp_problem_t& problem, const pdlp_settings_t& settings, dist_context_t* dist)
  : impl_(new impl_t)
{
  const double t0 = now_seconds();
  impl_->dist = dist;
  impl_->build(problem, settings);
  impl_->sol.stats.setup_seconds += now_seconds() - t0;
}
pdlp_solver_t::~pdlp_solver_t() = default;

void pdlp_solver_t::initialise() { impl_->initialise(); }
bool pdlp_solver_t::advance(int accepted_steps) { return impl_->outer_loop(accepted_steps); }
const lp_solution_t& pdlp_solver_t::solution() const { return impl_->sol; }

lp_solution_t pdlp_solver_t::run()
{
  impl_t& s        = *impl_;
  const double t0  = now_seconds();
  s.t_start        = t0;
  s.outer_loop(-1);
  s.close_peer_memory(true);
  s.sol.stats.solve_time = now_seconds() - t0;
  return s.sol;
}

double pdlp_solver_t::scalar(const std::string& name)
{
  impl_t& s = *impl_;
  s.fetch_ctl();
  const pdhg_ctl_t& k = *s.h_ctl;
  if (name == "step_size") return k.step_size;
  if (name == "primal_weight") return k.primal_weight;
  if (name == "tau") return k.tau;
  if (name == "sigma") return k.sigma;
  if (name == "sum_w") return k.sum_weights;
  if (name == "k_total") return s.total_pdlp_iterations;
  if (name == "k_pdhg") return k.attempts;
  if (name == "its_since_restart") return k.its_since_restart;
  if (name == "interaction") return k.interaction;
  if (name == "norm_dx2") return k.norm_dx2;
  if (name == "norm_dy2") return k.norm_dy2;
  if (name == "l2_norm_b") return s.l2_norm_b;
  if (name == "l2_norm_c") return s.l2_norm_c;
  if (name == "last_restart_kkt") return s.last_restart_kkt;
  if (name == "last_candidate_kkt") return s.last_candidate_kkt;
  if (name == "n_restarts") return s.sol.stats.n_restarts;
  if (name == "valid") return k.valid;
  return std::nan("");
}

std::vector<double> pdlp_solver_t::vector(const std::string& name)
{
  impl_t& s = *impl_;
  s.fetch_ctl();
  const int cur         = s.h_ctl->parity;
  const dvec<double>* v = nullptr;
  if (name == "x") v = &s.xbuf[cur];
  else if (name == "y") v = &s.ybuf[cur];
  else if (name == "aty") v = &s.atybuf[cur];
  else if (name == "x_next") v = &s.xbuf[cur ^ 1];
  else if (name == "y_next") v = &s.ybuf[cur ^ 1];
  else if (name == "aty_next") v = &s.atybuf[cur ^ 1];
  else if (name == "x_bar") v = &s.xbar;
  else if (name == "sum_x") v = &s.sum_x;
  else if (name == "sum_y") v = &s.sum_y;
  else if (name == "x_avg") v = &s.x_avg;
  else if (name == "y_avg") v = &s.y_avg;
  else if (name == "row_scaling") v = &s.Dr;
  else if (name == "col_scaling") v = &s.Dc;
  else if (name == "scaled_values") v = &s.As.val;
  else if (name == "scaled_values_t") v = &s.ATs.val;
  else if (name == "scaled_c") v = &s.cs;
  else if (name == "scaled_l") v = &s.ls;
  else if (name == "scaled_u") v = &s.us;
  else if (name == "scaled_lc") v = &s.lcs;
  else if (name == "scaled_uc") v = &s.ucs;
  else if (name == "x_last_restart") v = &s.x_lr;
  else if (name == "y_last_restart") v = &s.y_lr;
  if (!v) throw lp_error(error_type_t::InvalidArgument, "unknown vector " + name);
  std::vector<double> h(v->size());
  v->download(h.data(), s.stream);
  s.sync();
  return h;
}

kernel_profile_t pdlp_solver_t::profile_kernels(int warmup_steps, int reps)
{
  impl_t& s = *impl_;
  s.initialise();
  if (warmup_steps > 0) s.outer_loop(warmup_steps);
  kernel_profile_t out;
  out.reps = reps;
  out.grid_primal = s.grid_k1; out.grid_dual = s.grid_k2; out.grid_transpose = s.grid_k3;
  out.blocks_dual = s.blkA.B; out.blocks_transpose = s.blkAT.B;
  // SURVEY.md §8(d) per-kernel algorithmic bytes (gathers counted once per vector element)
  const double n = s.n, m = s.m, nz = s.nnz;
  out.bytes_primal_step    = 8.0 * (5 * n + 2 * n + 2 * n);                       // x,c,AtY,l,u | x',xbar | sum_x r/w
  out.bytes_dual_step      = 12.0 * nz + 4.0 * (m + 1) + 8.0 * (n + 3 * m + m + 2 * m);  // A | xbar gather, y,lc,uc | y' | sum_y r/w
  out.bytes_transpose_step = 12.0 * nz + 4.0 * (n + 1) + 8.0 * (m + n + 3 * n);   // A^T | y' gather | AtY' | x,x',AtY
  // make every attempt a "typical" one: previous step accepted (running-sum update fused in) and no batch end
  s.need_aty = false;
  k_begin_batch<<<1, 1, 0, s.stream>>>(s.d_ctl.data(), 1 << 30);
  std::vector<cudaEvent_t> ev(4);
  for (auto& e : ev) cudaEventCreate(&e);
  double acc[3] = {0, 0, 0};
  for (int r = 0; r < reps + 3; ++r) {
    cudaEventRecord(ev[0], s.stream);
    k_primal_step<<<s.grid_k1, EW_THREADS, 0, s.stream>>>(s.d_ctl.data(), s.n, s.xbuf[0].data(), s.xbuf[1].data(),
                                                          s.atybuf[0].data(), s.atybuf[1].data(), s.cs.data(), s.ls.data(),
                                                          s.us.data(), s.sum_x.data(), s.xbar.data());
    cudaEventRecord(ev[1], s.stream);
    s.enqueue_k2(nullptr, 0);  // fused kernel, or block passes + epilogue
    cudaEventRecord(ev[2], s.stream);
    s.enqueue_k3();
    cudaEventRecord(ev[3], s.stream);
    cudaEventSynchronize(ev[3]);
    if (r >= 3) {
      for (int q = 0; q < 3; ++q) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, ev[q], ev[q + 1]);
        acc[q] += ms;
      }
    }
  }
  s.check_launch();
  out.ms_primal_step    = acc[0] / reps;
  out.ms_dual_step      = acc[1] / reps;
  out.ms_transpose_step = acc[2] / reps;
  // whole attempts back to back (graph when enabled), no events in between
  cudaEventRecord(ev[0], s.stream);
  s.launch_attempts(reps);
  cudaEventRecord(ev[1], s.stream);
  cudaEventSynchronize(ev[1]);
  float ms = 0.f;
  cudaEventElapsedTime(&ms, ev[0], ev[1]);
  out.ms_iteration = ms / reps;
  // the sharded solve's payload-free partial product on this A^T (scratch output)
  {
    dvec<double> scratch((size_t)s.n);
    for (int r = 0; r < reps + 3; ++r) {
      if (r == 3) cudaEventRecord(ev[0], s.stream);
      k_transpose_partial<<<s.grid_k3, BICSR_THREADS, 0, s.stream>>>(s.d_ctl.data(), s.ATs.view(), s.ybuf[0].data(),
                                                                    s.ybuf[1].data(), scratch.data());
    }
    cudaEventRecord(ev[1], s.stream);
    cudaEventSynchronize(ev[1]);
    cudaEventElapsedTime(&ms, ev[0], ev[1]);
    out.ms_transpose_partial      = ms / reps;
    out.ms_transpose_partial_wide = 0.0;  // the wide schedule of round 1 is gone: one block format serves all densities
    s.check_launch();
  }
  for (auto& e : ev) cudaEventDestroy(e);
  s.sync();
  return out;
}

lp_solution_t solve_lp(const lp_problem_t& problem, const pdlp_settings_t& settings, dist_context_t* dist)
{
  lp_solution_t sol;
  try {
    pdlp_solver_t solver(problem, settings, dist);
    sol = solver.run();
  } catch (const lp_error& e) {
    if (e.type == error_type_t::Success) {  // "cannot run" cases the reference answers with a NumericalError solution
      sol.termination_status = termination_status_t::NumericalError;
      sol.error_status       = 0;
      sol.error_message      = e.what();
      return sol;
    }
    sol                    = lp_solution_t{};
    sol.termination_status = termination_status_t::NoTermination;
    sol.error_status       = (int)e.type;
    sol.error_message      = e.what();
  } catch (const std::bad_alloc&) {
    sol                    = lp_solution_t{};
    sol.error_status       = (int)error_type_t::RuntimeError;
    sol.error_message      = "Memory allocation failed";
  } catch (const std::exception& e) {
    sol                    = lp_solution_t{};
    sol.error_status       = (int)error_type_t::RuntimeError;
    sol.error_message      = e.what();
  }
  return sol;
}

}  // namespace cuopt_b200
