// The "kernel to beat" (BASELINE.md §4, SURVEY.md §2.2 K1/K2): the reference's PDHG attempt re-assembled from the
// library calls it makes, on the same synthetic matrices as bench.py's workloads, timed on the same GPU.
//
// Per attempt the reference issues (cpp/src/linear_programming/pdhg.cu:73-158,
// step_size_strategy/adaptive_step_size_strategy.cu:232-345, restart_strategy/weighted_average_solution.cu:73-110):
//   transform  primal projection        reads x, c, A^T y, l, u; writes x', dx, xbar          (cub::DeviceTransform)
//   cusparseSpMV(A, CSR_ALG2)            dual_gradient = A xbar                               (SpMV_preprocess done once)
//   transform  dual projection          reads y, A xbar, lc, uc; writes y', dy
//   cusparseSpMV(A^T, CSR_ALG2)          next A^T y
//   transform  next A^T y - A^T y
//   3 x cublasDdot (device pointer mode): interaction, |dx|^2, |dy|^2
//   scalar kernel (step-size rule), then a host synchronisation on the accept flag
//   2 x transform  running averages      sum_x += w x', sum_y += w y'
// The element-wise transforms are written here as plain grid-stride kernels (cub::DeviceTransform is a header-only
// element-wise launcher; both run at HBM speed), everything else IS the library code the reference runs.  The sequence is
// captured in one CUDA graph per attempt like the reference does; the per-attempt host synchronisation the reference
// needs is reported separately (with and without).
//
// nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -Xcompiler -fopenmp scripts/cusparse_pdhg.cu -lcusparse -lcublas -o scripts/_bin/cusparse_pdhg   (python -c "import __graft_entry__ as g; g.build_tools()")
#include <cublas_v2.h>
#include <cuda_runtime.h>
#include <cusparse.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x)                                                                   \
  do {                                                                          \
    cudaError_t e = (x);                                                        \
    if (e != cudaSuccess) {                                                     \
      printf("CUDA error %s at line %d\n", cudaGetErrorString(e), __LINE__);    \
      exit(1);                                                                  \
    }                                                                           \
  } while (0)
#define CS(x)                                                                   \
  do {                                                                          \
    cusparseStatus_t e = (x);                                                   \
    if (e != CUSPARSE_STATUS_SUCCESS) {                                         \
      printf("cuSPARSE error %d at line %d\n", (int)e, __LINE__);               \
      exit(1);                                                                  \
    }                                                                           \
  } while (0)
#define CB(x)                                                                   \
  do {                                                                          \
    cublasStatus_t e = (x);                                                     \
    if (e != CUBLAS_STATUS_SUCCESS) {                                           \
      printf("cuBLAS error %d at line %d\n", (int)e, __LINE__);                 \
      exit(1);                                                                  \
    }                                                                           \
  } while (0)

static inline uint64_t splitmix(uint64_t& s)
{
  uint64_t z = (s += 0x9e3779b97f4a7c15ull);
  z          = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z          = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}

struct csr_t {
  int rows, cols;
  std::vector<int> off, idx;
  std::vector<double> val;
};
csr_t make_fixed(int rows, int cols, int k, uint64_t seed)
{
  csr_t A{rows, cols};
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
csr_t transpose(const csr_t& A)
{
  csr_t T{A.cols, A.rows};
  T.off.assign((size_t)T.rows + 1, 0);
  T.idx.resize(A.idx.size());
  T.val.resize(A.idx.size());
  for (size_t p = 0; p < A.idx.size(); ++p) T.off[A.idx[p] + 1]++;
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
template <typename T>
T* to_dev(const std::vector<T>& h)
{
  T* d;
  CK(cudaMalloc(&d, std::max<size_t>(h.size(), 1) * sizeof(T)));
  CK(cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
  return d;
}
double* dev_fill(size_t n, double lo, double hi, uint64_t seed)
{
  std::vector<double> h(n);
  uint64_t s = seed;
  for (auto& v : h) v = lo + (hi - lo) * ((double)(splitmix(s) >> 11) / 9007199254740992.0);
  return to_dev(h);
}

// utils.cuh:81-95 / :98-112 as plain element-wise kernels
__global__ void k_primal_projection(int n, const double* x, const double* c, const double* aty, const double* l, const double* u,
                                    const double* tau, double* xn, double* dx, double* xbar)
{
  const double t = *tau;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    const double g    = c[j] - aty[j];
    const double next = fmax(fmin(x[j] - t * g, u[j]), l[j]);
    const double d    = next - x[j];
    xn[j]             = next;
    dx[j]             = d;
    xbar[j]           = next + d;
  }
}
__global__ void k_dual_projection(int m, const double* y, const double* ax, const double* lc, const double* uc, const double* sigma,
                                  double* yn, double* dy)
{
  const double s = *sigma;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
    const double next = y[i] - s * ax[i];
    const double v    = fmax(next + s * lc[i], fmin(next + s * uc[i], 0.0));
    yn[i]             = v;
    dy[i]             = v - y[i];
  }
}
__global__ void k_sub(int n, const double* a, const double* b, double* o)
{
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) o[j] = a[j] - b[j];
}
__global__ void k_axpy(int n, const double* w, const double* x, double* s)
{
  const double ww = *w;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) s[j] += ww * x[j];
}
// adaptive_step_size_strategy.cu:92-188 (one thread); step kept finite so the loop can run forever
__global__ void k_step_rule(const double* inter, const double* dx2, const double* dy2, double* step, double* tau, double* sigma, int* k)
{
  const double w        = 1.0;
  const double movement = 0.5 * w * *dx2 + (0.5 / w) * *dy2;
  const double limit    = fabs(*inter) > 0.0 ? movement / fabs(*inter) : 1e300;
  *k += 1;
  const double kc = (double)*k;
  double s        = fmin((1.0 - pow(kc + 1.0, -0.3)) * limit, (1.0 + pow(kc + 1.0, -0.6)) * *step);
  s               = fmin(fmax(s, 1e-3), 1e-1);
  *step           = s;
  *tau            = s / w;
  *sigma          = s * w;
}

struct spmv_t {
  cusparseSpMatDescr_t mat;
  cusparseDnVecDescr_t in, out;
  void* buffer;
};

int main(int argc, char** argv)
{
  std::vector<int> sizes;
  for (int i = 1; i < argc; ++i) sizes.push_back(atoi(argv[i]));
  if (sizes.empty()) sizes = {1000000, 10000000};
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  cudaStream_t stream, s1, s2;
  CK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&s1, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&s2, cudaStreamNonBlocking));
  cusparseHandle_t sp;
  cublasHandle_t bl;
  CS(cusparseCreate(&sp));
  CS(cusparseSetStream(sp, stream));
  CS(cusparseSetPointerMode(sp, CUSPARSE_POINTER_MODE_DEVICE));
  CB(cublasCreate(&bl));
  CB(cublasSetPointerMode(bl, CUBLAS_POINTER_MODE_DEVICE));
  int ver = 0;
  cusparseGetVersion(sp, &ver);
  printf("cuSPARSE %d\n", ver);

  for (int size : sizes) {
    const int m = size, n = size;
    csr_t A  = make_fixed(m, n, 8, 2);
    csr_t AT = transpose(A);
    const size_t nnz = A.idx.size();
    int *a_off = to_dev(A.off), *a_idx = to_dev(A.idx), *t_off = to_dev(AT.off), *t_idx = to_dev(AT.idx);
    double *a_val = to_dev(A.val), *t_val = to_dev(AT.val);
    double *x = dev_fill(n, 0, 1, 1), *xn = dev_fill(n, 0, 1, 2), *dx = dev_fill(n, 0, 0, 3), *xbar = dev_fill(n, 0, 1, 4);
    double *c = dev_fill(n, -1, 1, 5), *l = dev_fill(n, 0, 0, 6), *u = dev_fill(n, 5, 10, 7), *aty = dev_fill(n, -1, 1, 8);
    double *atyn = dev_fill(n, 0, 0, 9), *tmpn = dev_fill(n, 0, 0, 10), *sumx = dev_fill(n, 0, 0, 11);
    double *y = dev_fill(m, -1, 1, 12), *yn = dev_fill(m, 0, 0, 13), *dy = dev_fill(m, 0, 0, 14), *ax = dev_fill(m, 0, 0, 15);
    double *lc = dev_fill(m, -1, 0, 16), *uc = dev_fill(m, 0, 1, 17), *sumy = dev_fill(m, 0, 0, 18);
    double* scal = dev_fill(16, 0, 0, 19);  // 0 one, 1 zero, 2 tau, 3 sigma, 4 step, 5 inter, 6 dx2, 7 dy2
    {
      const double h[8] = {1.0, 0.0, 0.01, 0.01, 0.01, 0, 0, 0};
      CK(cudaMemcpy(scal, h, sizeof(h), cudaMemcpyHostToDevice));
    }
    int* d_k;
    CK(cudaMalloc(&d_k, 4));
    CK(cudaMemset(d_k, 0, 4));

    auto make_spmv = [&](int rows, int cols, int* off, int* idx, double* val, double* in, double* out) {
      spmv_t s;
      CS(cusparseCreateCsr(&s.mat, rows, cols, (int64_t)nnz, off, idx, val, CUSPARSE_INDEX_32I, CUSPARSE_INDEX_32I,
                           CUSPARSE_INDEX_BASE_ZERO, CUDA_R_64F));
      CS(cusparseCreateDnVec(&s.in, cols, in, CUDA_R_64F));
      CS(cusparseCreateDnVec(&s.out, rows, out, CUDA_R_64F));
      size_t bytes = 0;
      CS(cusparseSpMV_bufferSize(sp, CUSPARSE_OPERATION_NON_TRANSPOSE, scal + 0, s.mat, s.in, scal + 1, s.out, CUDA_R_64F,
                                 CUSPARSE_SPMV_CSR_ALG2, &bytes));
      CK(cudaMalloc(&s.buffer, std::max<size_t>(bytes, 8)));
      CS(cusparseSpMV_preprocess(sp, CUSPARSE_OPERATION_NON_TRANSPOSE, scal + 0, s.mat, s.in, scal + 1, s.out, CUDA_R_64F,
                                 CUSPARSE_SPMV_CSR_ALG2, s.buffer));
      printf("  SpMV %d x %d: ALG2 buffer %.1f MB\n", rows, cols, bytes * 1e-6);
      return s;
    };
    spmv_t sa  = make_spmv(m, n, a_off, a_idx, a_val, xbar, ax);
    spmv_t sat = make_spmv(n, m, t_off, t_idx, t_val, yn, atyn);
    auto spmv  = [&](spmv_t& s) {
      CS(cusparseSpMV(sp, CUSPARSE_OPERATION_NON_TRANSPOSE, scal + 0, s.mat, s.in, scal + 1, s.out, CUDA_R_64F,
                      CUSPARSE_SPMV_CSR_ALG2, s.buffer));
    };
    CK(cudaStreamSynchronize(stream));

    const int gn = std::min((n + 255) / 256, sms * 8), gm = std::min((m + 255) / 256, sms * 8);
    cudaEvent_t ev_fork, ev_j1, ev_j2, t0, t1;
    CK(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&ev_j1, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&ev_j2, cudaEventDisableTiming));
    CK(cudaEventCreate(&t0));
    CK(cudaEventCreate(&t1));
    auto attempt = [&]() {
      k_primal_projection<<<gn, 256, 0, stream>>>(n, x, c, aty, l, u, scal + 2, xn, dx, xbar);
      spmv(sa);
      k_dual_projection<<<gm, 256, 0, stream>>>(m, y, ax, lc, uc, scal + 3, yn, dy);
      CK(cudaEventRecord(ev_fork, stream));  // deltas_are_done_
      spmv(sat);
      k_sub<<<gn, 256, 0, stream>>>(n, atyn, aty, tmpn);
      CB(cublasSetStream(bl, stream));
      CB(cublasDdot(bl, n, tmpn, 1, dx, 1, scal + 5));
      CK(cudaStreamWaitEvent(s1, ev_fork, 0));
      CB(cublasSetStream(bl, s1));
      CB(cublasDdot(bl, n, dx, 1, dx, 1, scal + 6));
      CK(cudaEventRecord(ev_j1, s1));
      CK(cudaStreamWaitEvent(s2, ev_fork, 0));
      CB(cublasSetStream(bl, s2));
      CB(cublasDdot(bl, m, dy, 1, dy, 1, scal + 7));
      CK(cudaEventRecord(ev_j2, s2));
      CK(cudaStreamWaitEvent(stream, ev_j1, 0));
      CK(cudaStreamWaitEvent(stream, ev_j2, 0));
      k_step_rule<<<1, 1, 0, stream>>>(scal + 5, scal + 6, scal + 7, scal + 4, scal + 2, scal + 3, d_k);
      k_axpy<<<gn, 256, 0, stream>>>(n, scal + 4, xn, sumx);
      k_axpy<<<gm, 256, 0, stream>>>(m, scal + 4, yn, sumy);
    };
    // one CUDA graph per attempt (the reference: graph_prim_proj_gradient_dual + the step-size graph)
    cudaGraph_t g;
    cudaGraphExec_t ge;
    CK(cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal));
    attempt();
    CK(cudaStreamEndCapture(stream, &g));
    CK(cudaGraphInstantiate(&ge, g, 0));

    auto time_ms = [&](auto f, int reps) {
      for (int i = 0; i < 3; ++i) f();
      CK(cudaStreamSynchronize(stream));
      CK(cudaEventRecord(t0, stream));
      for (int i = 0; i < reps; ++i) f();
      CK(cudaEventRecord(t1, stream));
      CK(cudaEventSynchronize(t1));
      float ms;
      CK(cudaEventElapsedTime(&ms, t0, t1));
      return ms / reps;
    };
    const int reps      = size >= 5000000 ? 30 : 100;
    const double us_a   = 1e3 * time_ms([&] { spmv(sa); }, reps);
    const double us_at  = 1e3 * time_ms([&] { spmv(sat); }, reps);
    const double us_it  = 1e3 * time_ms([&] { CK(cudaGraphLaunch(ge, stream)); }, reps);
    const double us_its = 1e3 * time_ms([&] { CK(cudaGraphLaunch(ge, stream)); CK(cudaStreamSynchronize(stream)); }, reps);
    const double b_iter = 24.0 * nnz + 4.0 * (m + 1) + 4.0 * (n + 1) + 8.0 * (14.0 * n + 7.0 * m);
    printf("{\"comparator\": \"cusparse_pdhg\", \"m\": %d, \"n\": %d, \"nnz\": %zu, \"us_spmv_A\": %.1f, \"us_spmv_AT\": %.1f, "
           "\"us_attempt_graph\": %.1f, \"us_attempt_graph_with_host_sync\": %.1f, \"iterations_per_s\": %.1f, "
           "\"algorithmic_bytes_per_iteration\": %.0f, \"algorithmic_GBps\": %.1f}\n",
           m, n, nnz, us_a, us_at, us_it, us_its, 1e6 / us_its, b_iter, b_iter / us_its * 1e-3);
    fflush(stdout);
    for (void* p : {(void*)a_off, (void*)a_idx, (void*)t_off, (void*)t_idx, (void*)a_val, (void*)t_val, (void*)x, (void*)xn, (void*)dx,
                    (void*)xbar, (void*)c, (void*)l, (void*)u, (void*)aty, (void*)atyn, (void*)tmpn, (void*)sumx, (void*)y, (void*)yn,
                    (void*)dy, (void*)ax, (void*)lc, (void*)uc, (void*)sumy, (void*)scal, (void*)d_k, sa.buffer, sat.buffer})
      cudaFree(p);
    cudaGraphExecDestroy(ge);
    cudaGraphDestroy(g);
  }
  return 0;
}
