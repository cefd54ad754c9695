// Common infrastructure of libdftk_b200: context, error handling, device buffers, launch accounting.
#pragma once
#include <cuda_runtime.h>
#include <cublas_v2.h>
#include <cusolverDn.h>
#include <nccl.h>
#include <stdint.h>
#include <algorithm>
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

// Descriptor ring: the launch data a call builds on the host (item structs, pointer lists, band weights) is copied into a
// pinned block and from there, in stream order, into a device block of the same size.  The rules that keep a descriptor
// intact until the kernels reading it have run:
//  - put() returns the device copy; it stays valid until the next rewind().
//  - rewind() is called only right after a synchronisation of the stream the puts went to (the end of a scheduler round,
//    the trailing synchronisation of a one-shot call).
//  - a put that does not fit behind the data already staged synchronises the stream, then rewinds;
//  - a put larger than the whole ring synchronises and grows the ring to fit (a put never fails for size);
//  - a call that puts several regions before the launches that read them first calls reserve() with their total (padded()
//    each), so that none of its puts wraps over an earlier one.
// Both blocks are created at first use (cudaMallocHost costs about a millisecond) and kept for the context's lifetime.
struct DescRing {
  char* host = nullptr;
  DevBuf<char> dev;
  size_t cap = 0, off = 0;
  ~DescRing() {
    if (host) cudaFreeHost(host);
  }
  static size_t padded(size_t bytes) { return (bytes + 255) & ~(size_t)255; }
  template <class T>
  static size_t padded(const std::vector<T>& v) { return padded(v.size() * sizeof(T)); }
  void reserve(size_t bytes, cudaStream_t s) {
    bytes = padded(bytes);
    if (off + bytes <= cap) return;
    if (cap) CUDA_CHECK(cudaStreamSynchronize(s));
    off = 0;
    if (bytes <= cap) return;
    if (host) CUDA_CHECK(cudaFreeHost(host));
    host = nullptr;
    cap = 0;
    const size_t n = std::max(bytes, (size_t)4 << 20);
    CUDA_CHECK(cudaMallocHost((void**)&host, n));
    dev.ensure(n);
    cap = n;
  }
  const void* put(const void* src, size_t bytes, cudaStream_t s) {
    reserve(bytes, s);
    char* d = dev.p + off;
    if (bytes) {
      memcpy(host + off, src, bytes);
      CUDA_CHECK(cudaMemcpyAsync(d, host + off, bytes, cudaMemcpyHostToDevice, s));
    }
    off += padded(bytes);
    return d;
  }
  template <class T>
  const T* put(const std::vector<T>& v, cudaStream_t s) {
    return (const T*)put(v.data(), v.size() * sizeof(T), s);
  }
  void rewind() { off = 0; }
};

// One executor slot of the batched small-matrix kernels (BatchExec, lobpcg.cu); slot 1 serves the second group of the
// pipelined scheduler, slot 0 everything else, including the descriptors of the one-shot multi-block calls.
struct BatchSlot {
  static constexpr size_t GATHER_CAP = (size_t)1 << 18;   // doubles of the per-round result gather
  DescRing ring;
  DevBuf<double> gather;
  double* gather_h = nullptr;    // pinned landing zone of the gather
  DevBuf<char> own_ws;
  DevBuf<char>* gram_ws;         // per-CTA partials of kb_gram: slot 0 shares the split-K workspace of the GEMMs
  DevBuf<int> counter;           // arrival counters of kb_gram (kept at zero between launches)
  cudaEvent_t ev = nullptr;      // end of the issued round
  explicit BatchSlot(DevBuf<char>* ws = nullptr) : gram_ws(ws ? ws : &own_ws) {}
  ~BatchSlot() {
    if (gather_h) cudaFreeHost(gather_h);
    if (ev) cudaEventDestroy(ev);
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
  dftk::DevBuf<signed char> i8_tmp_planes;   // gemm_backend 4: planes of an operand prepared inside a generic zgemm call
  dftk::DevBuf<int> i8_tmp_exps;
  // executor slots of the batched small-matrix kernels: slot 1 is the second group of the pipelined batched solves (two
  // groups of k-blocks on two streams: while one group's round runs on the GPU, the host records and issues the other's)
  dftk::BatchSlot slot[2]{dftk::BatchSlot(&gemm_ws), dftk::BatchSlot()};
  cudaStream_t batch_streams[2] = {nullptr, nullptr};
  cudaStream_t batch_user_stream = nullptr;   // the context's own stream while a pipelined batch has swapped ctx->stream
  bool batch_pipelined = false;
  int batch_pipeline = 0;     // option: 1 = two pipelined groups for batches of >= 8 k-blocks, 0 (default) = one group (one sync per
                              // round)
  double lobpcg_flops = 0.0;  // FP64-equivalent GEMM flops executed by the large-path LOBPCG solves (Gram, update, Cholesky-QR, nonlocal) since reset
  int64_t batch_rounds = 0;   // scheduler rounds (= host synchronisations) of the batched solves since creation / reset
  // direct minimisation (dm.cu): reduction partials and results, small matrices of all blocks
  dftk::DevBuf<double> dm_ws, dm_out, dm_w, dm_stats;
  dftk::DevBuf<dftk::cplx> dm_C, dm_M, dm_V;
  // batched overlap products (overlap.cu): chunk partials, the gathered block of the large path
  dftk::DevBuf<dftk::cplx> ov_ws, ov_scratch;
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
// `p` is device or managed memory, and device memory of the context's device; what: "<entry point>: <argument>"
inline void require_device(const dftk_b200_ctx* ctx, const void* p, const std::string& what) {
  cudaPointerAttributes a;
  const cudaError_t e = p ? cudaPointerGetAttributes(&a, p) : cudaErrorInvalidValue;
  if (e != cudaSuccess) cudaGetLastError();
  REQUIRE(e == cudaSuccess && (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged), what + " must be device memory");
  REQUIRE(a.type != cudaMemoryTypeDevice || a.device == ctx->device, what + " must be on the context's device");
}
}  // namespace dftk
