// Common infrastructure of libdftk_b200: context, error handling, device buffers, launch accounting.
#pragma once
#include <cuda_runtime.h>
#include <cublas_v2.h>
#include <cusolverDn.h>
#include <nccl.h>
#include <stdint.h>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>
#include "../../include/dftk_b200.h"
#include "fft_core.cuh"

namespace dftk {

struct Error : public std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

#define CUDA_CHECK(expr)                                                                         \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess)                                                                       \
      throw ::dftk::Error(DFTK_B200_ECUDA, std::string(#expr) + ": " + cudaGetErrorString(_e) +  \
                                               " (" + __FILE__ + ":" + std::to_string(__LINE__) + ")"); \
  } while (0)
#define CUBLAS_CHECK(expr)                                                                       \
  do {                                                                                           \
    cublasStatus_t _s = (expr);                                                                  \
    if (_s != CUBLAS_STATUS_SUCCESS)                                                             \
      throw ::dftk::Error(DFTK_B200_ECUDA, std::string(#expr) + ": cublas status " + std::to_string((int)_s)); \
  } while (0)
#define CUSOLVER_CHECK(expr)                                                                     \
  do {                                                                                           \
    cusolverStatus_t _s = (expr);                                                                \
    if (_s != CUSOLVER_STATUS_SUCCESS)                                                           \
      throw ::dftk::Error(DFTK_B200_ECUDA, std::string(#expr) + ": cusolver status " + std::to_string((int)_s)); \
  } while (0)
#define NCCL_CHECK(expr)                                                                         \
  do {                                                                                           \
    ncclResult_t _r = (expr);                                                                    \
    if (_r != ncclSuccess)                                                                       \
      throw ::dftk::Error(DFTK_B200_ENCCL, std::string(#expr) + ": " + ncclGetErrorString(_r));  \
  } while (0)
#define REQUIRE(cond, msg)                                              \
  do {                                                                  \
    if (!(cond)) throw ::dftk::Error(DFTK_B200_EINVAL, std::string(msg)); \
  } while (0)

// Growable device buffer (the library's scratch arena is a handful of these; they only ever grow).
template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;
  ~DevBuf() { release(); }
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  T* ensure(size_t n) {
    if (n > cap) {
      release();
      CUDA_CHECK(cudaMalloc((void**)&p, n * sizeof(T)));
      cap = n;
    }
    return p;
  }
  void upload(const T* host, size_t n, cudaStream_t s) {
    ensure(n);
    if (n) CUDA_CHECK(cudaMemcpyAsync(p, host, n * sizeof(T), cudaMemcpyDefault, s));
  }
};

}  // namespace dftk

struct dftk_b200_ctx {
  int device = 0;
  cudaStream_t stream = 0;
  cublasHandle_t cublas = nullptr;
  cusolverDnHandle_t cusolver = nullptr;
  cusolverDnParams_t solver_params = nullptr;
  std::vector<char> solver_host_work;
  ncclComm_t nccl = nullptr;
  int rank = 0, nranks = 1;
  int64_t launches = 0;
  int gemm_backend = 0;   // 0 (default) = own FP64 DMMA kernels; 4 = INT8 tensor cores (wgmma s8, TMA-fed; i8emu.cu / i8tc2.cu) for
                          // contractions of at least i8_min_rows rows, DMMA otherwise; 1 = cuBLAS (A/B comparison only); 2 = checker of
                          // the INT8 scheme (integer products on CUDA cores).  DMMA is the default because it is the faster of the two on
                          // an H100 SXM (700 W): LOBPCG iteration of the 128-atom Si cell (259 bands) 0.12 s vs 0.21 s, nonlocal products
                          // 9.8 ms vs 16.3 ms, equal eigenvalues to 2e-15
  int band_chunk = 0;     // 0 = auto
  int fft_engine = 0;     // 0 = register two-pass engine where a factor pair exists, 1 = generic Stockham (applies to grids created afterwards)
  int gemm_stages = 4;    // cp.async ring depth (2..4) of the DMMA GEMMs; one 8-warp CTA per SM at every depth (2, 3 and 4 time
                          // within noise of each other on an H100; scripts/gemm_probe.py compares them)
  int64_t i8_min_rows = 32768;   // gemm_backend 4: shortest contraction length that goes to the INT8 tensor-core path
  int z_pipeline = 0;     // fused z stage of the H apply: 0 = one tile per CTA (default), 1 = persistent cp.async-pipelined kernel
  int force_svd_fallback = 0;   // test hook: the next N ortho! calls behave as if safe_cholesky had given up
  int small_dense = 1;    // LOBPCG with <= 32 bands: fused small-matrix kernels (lobpcg_small.cuh); 0 = GEMM + cuSOLVER path
  dftk::DevBuf<int> small_counter;   // arrival counter of k_small_gram (kept at zero between launches)
  int sm_count = 132;
  int smem_optin = 227 * 1024;   // largest dynamic shared memory of one CTA (cudaDevAttrMaxSharedMemoryPerBlockOptin)
  std::string last_error;
  dftk::DevBuf<char> solver_work;
  dftk::DevBuf<int> dev_info;
  dftk::DevBuf<double> scal;     // small scalar scratch
  dftk::DevBuf<char> gemm_ws;    // split-K partials
  dftk::DevBuf<int> sym_i;       // symmetry tables (integer rotations)
  dftk::DevBuf<double> sym_d;    //                 (fractional translations)
  dftk::DevBuf<double> radial_part;   // per-split partial sums of the radial transform (setup.cu)
  dftk::DevBuf<char> stage_in, stage_out;  // host<->device staging for host-buffer calls
  // pipelined host staging (H2D of chunk k+1 || compute of chunk k || D2H of chunk k-1)
  cudaStream_t s_in = nullptr, s_out = nullptr;
  cudaEvent_t ev_in[2] = {nullptr, nullptr}, ev_comp[2] = {nullptr, nullptr}, ev_out[2] = {nullptr, nullptr};
  dftk::DevBuf<char> pipe_in[2], pipe_out[2];
  // batched small-matrix LOBPCG (lobpcg.cu): descriptor ring and per-round result gather, device + pinned host sides
  dftk::DevBuf<char> batch_ring;
  dftk::DevBuf<double> batch_gather;
  char* batch_ring_h = nullptr;
  double* batch_gather_h = nullptr;
  dftk::DevBuf<signed char> i8_tmp_planes;   // gemm_backend 4: planes of an operand prepared inside a generic zgemm call
  dftk::DevBuf<int> i8_tmp_exps;
  // second executor of the pipelined batched solves (two groups of k-blocks on two streams: while one group's round runs on
  // the GPU, the host records and issues the other group's): its own descriptor ring, gather buffer, Gram workspace, counters
  dftk::DevBuf<char> batch_ring2, batch_ws2;
  dftk::DevBuf<double> batch_gather2;
  dftk::DevBuf<int> small_counter2;
  char* batch_ring_h2 = nullptr;
  double* batch_gather_h2 = nullptr;
  cudaStream_t batch_streams[2] = {nullptr, nullptr};
  cudaEvent_t batch_events[2] = {nullptr, nullptr};
  cudaStream_t batch_user_stream = nullptr;   // the context's own stream while a pipelined batch has swapped ctx->stream
  bool batch_pipelined = false;
  int batch_pipeline = 0;     // option: 1 = two pipelined groups for batches of >= 8 k-blocks, 0 (default) = one group (one sync per
                              // round)
  double lobpcg_flops = 0.0;  // FP64-equivalent GEMM flops executed by the large-path LOBPCG solves (Gram, update, Cholesky-QR, nonlocal) since reset
  int64_t batch_rounds = 0;   // scheduler rounds (= host synchronisations) of the batched solves since creation / reset
  // direct minimisation (dm.cu): item descriptors, reduction partials and results, small matrices of all blocks
  dftk::DevBuf<char> dm_items;
  dftk::DevBuf<double> dm_ws, dm_out, dm_w, dm_stats;
  dftk::DevBuf<dftk::cplx> dm_C, dm_M, dm_V;
  dftk::DevBuf<char> tr_items;   // basis transfers (transfer.cu): descriptors of the pairs of one sphere remap
  // batched overlap products (overlap.cu): group and pair descriptors, chunk partials, the gathered block of the large path
  dftk::DevBuf<char> ov_items;
  dftk::DevBuf<dftk::cplx> ov_ws, ov_scratch;
  dftk::DevBuf<char> ldos_items;   // LDOS pass (ldos.cu): the density-row and weight-column pointers of every round
};

namespace dftk {
#define LAUNCH(ctx, kernel, grid, block, smem, ...)                     \
  do {                                                                  \
    kernel<<<(grid), (block), (smem), (ctx)->stream>>>(__VA_ARGS__);    \
    (ctx)->launches++;                                                  \
    CUDA_CHECK(cudaGetLastError());                                     \
  } while (0)

// The error boundary of every extern "C" entry point: an exception becomes its error code, and its message is kept for
// dftk_b200_last_error, per context and process-wide (the latter also answers calls that had no context).
int record_error(dftk_b200_ctx* ctx, int code, const std::string& msg);   // api.cu
#define API_BEGIN try {
#define API_END(ctx)                                                                                \
  }                                                                                                 \
  catch (const ::dftk::Error& e) { return ::dftk::record_error((ctx), e.code, e.what()); }           \
  catch (const std::exception& e) { return ::dftk::record_error((ctx), DFTK_B200_EINVAL, e.what()); } \
  catch (...) { return ::dftk::record_error((ctx), DFTK_B200_EINVAL, "unknown C++ exception"); }      \
  return DFTK_B200_OK;

inline bool is_device_ptr(const void* p) {
  cudaPointerAttributes a;
  cudaError_t e = cudaPointerGetAttributes(&a, p);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}
}  // namespace dftk
