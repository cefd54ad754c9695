// Device operations of the direct minimisation of the Kohn-Sham energy (direct_minimization.py; reference seam
// src/scf/direct_minimization.jl): every entry point works on all (k, spin) blocks of a rank in one call.  Blocks of
// <= SMALL_MAX_N bands take the batched small-matrix kernels of the LOBPCG scheduler (a fixed number of launches whatever
// the block count); larger blocks take the DMMA ZGEMMs and cuSOLVER, one block after the other.
#include <algorithm>
#include <cmath>
#include "batch_exec.cuh"
#include "dm_core.cuh"

using namespace dftk;

namespace {

struct DmScaleItem { cplx* p; long long len; double s; };
struct DmTpaItem { const cplx* q; cplx* s; long long n_rows; int n_cols; const double* kin; const double* mk; double inv_w; };

__global__ void __launch_bounds__(DM_THREADS) k_dm_dot_partial(const DmDotItem* __restrict__ items, int n_chunks,
                                                             double* __restrict__ ws) {
  const DmDotItem it = items[blockIdx.y];
  __shared__ double red[DM_THREADS];
  red[threadIdx.x] = dm_chunk_partial(it, blockIdx.x, n_chunks, threadIdx.x);
  __syncthreads();
  for (int w = DM_THREADS / 2; w > 0; w >>= 1) {
    dm_tree_step(red, threadIdx.x, w);
    __syncthreads();
  }
  if (threadIdx.x == 0) ws[(long long)blockIdx.y * n_chunks + blockIdx.x] = red[0];
}

// one thread per pair: the items of pair p are [p * n_blocks, (p + 1) * n_blocks)
__global__ void k_dm_dot_final(const double* __restrict__ ws, int n_pairs, int n_blocks, int n_chunks, double* __restrict__ out) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n_pairs) out[p] = dm_final_sum(ws, p * n_blocks, n_blocks, n_chunks);
}

__global__ void __launch_bounds__(DM_THREADS) k_dm_scale(const DmScaleItem* __restrict__ items) {
  const DmScaleItem it = items[blockIdx.y];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < it.len; i += (long long)gridDim.x * blockDim.x) {
    cplx v = it.p[i];
    it.p[i] = make_double2(v.x * it.s, v.y * it.s);
  }
}

__global__ void __launch_bounds__(DM_THREADS) k_dm_tpa(const DmTpaItem* __restrict__ items) {
  const DmTpaItem it = items[blockIdx.y];
  const long long total = it.n_rows * it.n_cols;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long i = idx % it.n_rows, c = idx / it.n_rows;
    it.s[idx] = dm_tpa_entry(it.q[idx], it.kin ? it.kin[i] : 0.0, it.mk ? it.mk[c] : -1.0, it.inv_w);
  }
}

// small matrices of all blocks, n x n each, consecutive in memory; one CTA per block
__global__ void k_dm_herm(const cplx* __restrict__ C, cplx* __restrict__ M, int n) {
  const cplx* c = C + (size_t)blockIdx.x * n * n;
  cplx* m = M + (size_t)blockIdx.x * n * n;
  for (int e = threadIdx.x; e < n * n; e += blockDim.x) m[e] = dm_herm_entry(c, n, e % n, e / n);
}
// n <= SMALL_MAX_N: w^{-1/2} once into shared memory, then V diag(w^{-1/2}) V^H
__global__ void k_dm_invsqrt(const cplx* __restrict__ V, const double* __restrict__ w, cplx* __restrict__ S, int n) {
  __shared__ double f[SMALL_MAX_N];
  const cplx* v = V + (size_t)blockIdx.x * n * n;
  const double* ww = w + (size_t)blockIdx.x * n;
  cplx* s = S + (size_t)blockIdx.x * n * n;
  for (int l = threadIdx.x; l < n; l += blockDim.x) f[l] = 1.0 / sqrt(ww[l]);
  __syncthreads();
  for (int e = threadIdx.x; e < n * n; e += blockDim.x) s[e] = dm_invsqrt_entry(v, f, n, e % n, e / n);
}
// one block's A = diag(w^{-1/4}) V^H (coalesced writes; the GEMM then forms A^H A)
__global__ void k_dm_scaled_adjoint(const cplx* __restrict__ V, const double* __restrict__ w, cplx* __restrict__ A, int n) {
  const long long total = (long long)n * n;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x)
    A[e] = dm_scaled_adjoint_entry(V, w, n, (int)(e % n), (int)(e / n));
}

unsigned grid_for(dftk_b200_ctx* ctx, long long total) {
  long long g = (total + DM_THREADS - 1) / DM_THREADS;
  return (unsigned)std::max<long long>(1, std::min<long long>(g, (long long)ctx->sm_count * 16));
}

// the stream synchronisation every entry point ends with; the descriptors it staged are then no longer read
void finish(dftk_b200_ctx* ctx) {
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  ctx->slot[0].ring.rewind();
}

// Sum_pairs of Re<A, B> (or the fused update + dot) over all block items: two launches, one synchronisation.
void dots(dftk_b200_ctx* ctx, const std::vector<DmDotItem>& items, int n_pairs, int n_blocks, double* out_host) {
  long long max_len = 1;
  for (auto& it : items) max_len = std::max(max_len, it.len);
  const int n_chunks = (int)std::min<long long>(DM_MAX_CHUNKS, (max_len + DM_THREADS - 1) / DM_THREADS);
  double* ws = ctx->dm_ws.ensure((size_t)items.size() * n_chunks);
  double* out = ctx->dm_out.ensure(std::max(n_pairs, 1));
  LAUNCH(ctx, k_dm_dot_partial, dim3((unsigned)n_chunks, (unsigned)items.size()), DM_THREADS, 0,
         ctx->slot[0].ring.put(items, ctx->stream), n_chunks, ws);
  if (n_pairs > 0) {
    LAUNCH(ctx, k_dm_dot_final, (unsigned)((n_pairs + 63) / 64), 64, 0, (const double*)ws, n_pairs, n_blocks, n_chunks, out);
    CUDA_CHECK(cudaMemcpyAsync(out_host, out, n_pairs * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  }
  finish(ctx);
}

void heev_large(dftk_b200_ctx* ctx, cplx* A, int64_t n, double* w) {
  if (!ctx->solver_params) CUSOLVER_CHECK(cusolverDnCreateParams(&ctx->solver_params));
  size_t wd = 0, wh = 0;
  CUSOLVER_CHECK(cusolverDnXsyevd_bufferSize(ctx->cusolver, ctx->solver_params, CUSOLVER_EIG_MODE_VECTOR, CUBLAS_FILL_MODE_UPPER,
                                             n, CUDA_C_64F, A, n, CUDA_R_64F, w, CUDA_C_64F, &wd, &wh));
  char* wk = ctx->solver_work.ensure(wd + 16);
  if (ctx->solver_host_work.size() < wh + 16) ctx->solver_host_work.resize(wh + 16);
  int* dinfo = ctx->dev_info.ensure(4);
  CUSOLVER_CHECK(cusolverDnXsyevd(ctx->cusolver, ctx->solver_params, CUSOLVER_EIG_MODE_VECTOR, CUBLAS_FILL_MODE_UPPER, n,
                                  CUDA_C_64F, A, n, CUDA_R_64F, w, CUDA_C_64F, wk, wd, ctx->solver_host_work.data(), wh, dinfo));
  ctx->launches++;
  int info = 0;
  CUDA_CHECK(cudaMemcpyAsync(&info, dinfo, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  if (info != 0) throw Error(DFTK_B200_ENUM, "stiefel_retract: heevd failed, info=" + std::to_string(info));
}

// C_i = A_i^H B_i (nb x nb at C + i nb^2) for all blocks
void grams(dftk_b200_ctx* ctx, int n, dftk_b200_kblock* const* kbs, const cplx* const* A, const cplx* const* Bm, int nb, cplx* C) {
  if (nb <= SMALL_MAX_N) {
    std::vector<GramItem> v;
    for (int i = 0; i < n; ++i)
      v.push_back(single_gram_item(ctx, A[i], kbs[i]->n_pw, nb, Bm[i], kbs[i]->n_pw, nb, kbs[i]->n_pw, C + (size_t)i * nb * nb));
    BatchExec(ctx, ctx->slot[0]).gram_batch(v);
    finish(ctx);
    return;
  }
  for (int i = 0; i < n; ++i)
    zgemm(ctx, 2, nb, nb, kbs[i]->n_pw, make_double2(1.0, 0.0), A[i], kbs[i]->n_pw, Bm[i], kbs[i]->n_pw, make_double2(0.0, 0.0),
          C + (size_t)i * nb * nb, nb);
}
// out_i = alpha Y_i M_i + beta out_i
void times(dftk_b200_ctx* ctx, int n, dftk_b200_kblock* const* kbs, const cplx* const* Y, const cplx* M, int nb, cplx* const* out,
           double alpha, double beta) {
  if (nb <= SMALL_MAX_N) {
    std::vector<BtimesItem> v;
    for (int i = 0; i < n; ++i)
      v.push_back(single_btimes_item(Y[i], nb, M + (size_t)i * nb * nb, nb, out[i], kbs[i]->n_pw, alpha, beta));
    BatchExec(ctx, ctx->slot[0]).btimes_batch(v);
    finish(ctx);
    return;
  }
  for (int i = 0; i < n; ++i)
    zgemm(ctx, 0, kbs[i]->n_pw, nb, nb, make_double2(alpha, 0.0), Y[i], kbs[i]->n_pw, M + (size_t)i * nb * nb, nb,
          make_double2(beta, 0.0), out[i], kbs[i]->n_pw);
}

dftk_b200_ctx* ctx_of(int64_t n, dftk_b200_kblock* const* kbs) { return (n > 0 && kbs && kbs[0]) ? kbs[0]->grid->ctx : nullptr; }

void check_blocks(dftk_b200_ctx* ctx, int64_t n, dftk_b200_kblock* const* kbs, int64_t n_bands, const char* what) {
  REQUIRE(n >= 0 && (n == 0 || kbs) && n_bands >= 1, std::string(what) + ": bad argument");
  for (int64_t i = 0; i < n; ++i)
    REQUIRE(kbs[i] && kbs[i]->grid->ctx == ctx, std::string(what) + ": all blocks must belong to one context");
}
void check_orbitals(dftk_b200_ctx* ctx, int64_t n, const void* const* p, const char* what) {
  REQUIRE(p, std::string(what) + ": NULL block list");
  for (int64_t i = 0; i < n; ++i) require_device(ctx, p[i], std::string(what) + ": orbitals");
}

}  // namespace

extern "C" {

int dftk_b200_apply_h_multi(int64_t n_blocks, dftk_b200_kblock* const* kbs, const void* const* psi, void* const* out,
                            int64_t n_bands, const double* scale_host) {
  dftk_b200_ctx* ctx = ctx_of(n_blocks, kbs);
  API_BEGIN
  check_blocks(ctx, n_blocks, kbs, n_bands, "apply_h_multi");
  if (n_blocks == 0) return DFTK_B200_OK;
  check_orbitals(ctx, n_blocks, psi, "apply_h_multi");
  check_orbitals(ctx, n_blocks, (const void* const*)out, "apply_h_multi");
  std::vector<ApplyHItem> items;
  for (int64_t i = 0; i < n_blocks; ++i) items.push_back(ApplyHItem{kbs[i], (const cplx*)psi[i], (cplx*)out[i], (int)n_bands});
  BatchExec(ctx, ctx->slot[0]).apply_h_batch(items);
  finish(ctx);
  if (scale_host) {
    std::vector<DmScaleItem> v;
    long long mt = 1;
    for (int64_t i = 0; i < n_blocks; ++i) {
      v.push_back(DmScaleItem{(cplx*)out[i], (long long)kbs[i]->n_pw * n_bands, scale_host[i]});
      mt = std::max(mt, v.back().len);
    }
    LAUNCH(ctx, k_dm_scale, dim3(grid_for(ctx, mt), (unsigned)n_blocks), DM_THREADS, 0, ctx->slot[0].ring.put(v, ctx->stream));
    finish(ctx);
  }
  API_END(ctx)
}

int dftk_b200_stiefel_project_multi(int64_t n_blocks, dftk_b200_kblock* const* kbs, const void* const* X, void* const* G,
                                    int64_t n_bands) {
  dftk_b200_ctx* ctx = ctx_of(n_blocks, kbs);
  API_BEGIN
  check_blocks(ctx, n_blocks, kbs, n_bands, "stiefel_project_multi");
  if (n_blocks == 0) return DFTK_B200_OK;
  check_orbitals(ctx, n_blocks, X, "stiefel_project_multi");
  check_orbitals(ctx, n_blocks, (const void* const*)G, "stiefel_project_multi");
  const int nb = (int)n_bands, n = (int)n_blocks;
  cplx* C = ctx->dm_C.ensure((size_t)n * nb * nb);
  cplx* M = ctx->dm_M.ensure((size_t)n * nb * nb);
  grams(ctx, n, kbs, (const cplx* const*)X, (const cplx* const*)G, nb, C);        // X^H G
  LAUNCH(ctx, k_dm_herm, (unsigned)n, DM_THREADS, 0, (const cplx*)C, M, nb);          // (X^H G + G^H X) / 2
  times(ctx, n, kbs, (const cplx* const*)X, M, nb, (cplx* const*)G, -1.0, 1.0);       // G -= X M
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  API_END(ctx)
}

int dftk_b200_stiefel_retract_multi(int64_t n_blocks, dftk_b200_kblock* const* kbs, const void* const* Y, void* const* X_out,
                                    int64_t n_bands) {
  dftk_b200_ctx* ctx = ctx_of(n_blocks, kbs);
  API_BEGIN
  check_blocks(ctx, n_blocks, kbs, n_bands, "stiefel_retract_multi");
  if (n_blocks == 0) return DFTK_B200_OK;
  check_orbitals(ctx, n_blocks, Y, "stiefel_retract_multi");
  check_orbitals(ctx, n_blocks, (const void* const*)X_out, "stiefel_retract_multi");
  for (int64_t i = 0; i < n_blocks; ++i) REQUIRE(Y[i] != X_out[i], "stiefel_retract_multi: the output must not alias the input");
  const int nb = (int)n_bands, n = (int)n_blocks;
  cplx* C = ctx->dm_C.ensure((size_t)n * nb * nb);
  cplx* V = ctx->dm_V.ensure((size_t)n * nb * nb);
  cplx* S = ctx->dm_M.ensure((size_t)n * nb * nb);
  double* w = ctx->dm_w.ensure((size_t)n * nb);
  grams(ctx, n, kbs, (const cplx* const*)Y, (const cplx* const*)Y, nb, C);           // Y^H Y
  std::vector<double> w_h((size_t)n * nb);
  if (nb <= SMALL_MAX_N) {
    double* st = ctx->dm_stats.ensure((size_t)2 * n);
    std::vector<HeevItem> v;                                                            // eigenvectors overwrite C
    for (int i = 0; i < n; ++i)
      v.push_back(HeevItem{C + (size_t)i * nb * nb, nb, nb, w + (size_t)i * nb, V + (size_t)i * nb * nb, st + 2 * i, nullptr, 0});
    BatchExec(ctx, ctx->slot[0]).heev_batch(v);
    finish(ctx);
    std::vector<double> st_h((size_t)2 * n);
    CUDA_CHECK(cudaMemcpy(st_h.data(), st, st_h.size() * sizeof(double), cudaMemcpyDeviceToHost));
    for (int i = 0; i < n; ++i)
      if (!(st_h[2 * i] > 0.0))      // stats[0] = sweeps used, 0 when the Jacobi iteration did not converge
        throw Error(DFTK_B200_ENUM, "stiefel_retract: the Jacobi eigensolver of block " + std::to_string(i) +
                                        " did not converge (off-diagonal norm " + std::to_string(st_h[2 * i + 1]) + ")");
  } else {
    for (int i = 0; i < n; ++i) heev_large(ctx, C + (size_t)i * nb * nb, nb, w + (size_t)i * nb);
  }
  CUDA_CHECK(cudaMemcpy(w_h.data(), w, w_h.size() * sizeof(double), cudaMemcpyDeviceToHost));
  for (int i = 0; i < n; ++i)        // ascending: the smallest eigenvalue of each block leads
    REQUIRE(w_h[(size_t)i * nb] > 0.0 && std::isfinite(w_h[(size_t)i * nb + nb - 1]),
            "stiefel_retract: the Gram matrix of block " + std::to_string(i) + " is not positive definite (rank-deficient input)");
  if (nb <= SMALL_MAX_N) {
    LAUNCH(ctx, k_dm_invsqrt, (unsigned)n, DM_THREADS, 0, (const cplx*)C, (const double*)w, S, nb);   // (Y^H Y)^{-1/2}
  } else {
    for (int i = 0; i < n; ++i) {
      const size_t o = (size_t)i * nb * nb;
      LAUNCH(ctx, k_dm_scaled_adjoint, grid_for(ctx, (long long)nb * nb), DM_THREADS, 0, (const cplx*)(C + o),
             (const double*)(w + (size_t)i * nb), V + o, nb);
      zgemm(ctx, 2, nb, nb, nb, make_double2(1.0, 0.0), V + o, nb, V + o, nb, make_double2(0.0, 0.0), S + o, nb);
    }
  }
  times(ctx, n, kbs, (const cplx* const*)Y, S, nb, (cplx* const*)X_out, 1.0, 0.0);
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  API_END(ctx)
}

int dftk_b200_tpa_multi(int64_t n_blocks, dftk_b200_kblock* const* kbs, const void* const* X, const void* const* Q, void* const* S,
                        int64_t n_bands, const double* inv_w_host, int use_tpa, double* mean_kin) {
  dftk_b200_ctx* ctx = ctx_of(n_blocks, kbs);
  API_BEGIN
  check_blocks(ctx, n_blocks, kbs, n_bands, "tpa_multi");
  if (n_blocks == 0) return DFTK_B200_OK;
  if (use_tpa) require_device(ctx, mean_kin, "tpa_multi: mean_kin");
  const int n = (int)n_blocks, nb = (int)n_bands;
  if (use_tpa)
    for (int i = 0; i < n; ++i) REQUIRE(kbs[i]->has_kin, "tpa_multi: the TPA preconditioner needs a kinetic term");
  if (X && use_tpa) {     // precondprep!: mean_kin[n] = sum_G kin_G |x_Gn|^2
    check_orbitals(ctx, n_blocks, X, "tpa_multi");
    std::vector<KinDotsItem> v;
    for (int i = 0; i < n; ++i)
      v.push_back(KinDotsItem{(const cplx*)X[i], kbs[i]->n_pw, kbs[i]->n_pw, nb, kbs[i]->kin.p, mean_kin + (size_t)i * nb});
    BatchExec(ctx, ctx->slot[0]).kin_dots_batch(v);
    finish(ctx);
  }
  if (Q) {                // ldiv!
    check_orbitals(ctx, n_blocks, Q, "tpa_multi");
    check_orbitals(ctx, n_blocks, (const void* const*)S, "tpa_multi");
    REQUIRE(inv_w_host, "tpa_multi: NULL weights");
    std::vector<DmTpaItem> v;
    long long mt = 1;
    for (int i = 0; i < n; ++i) {
      v.push_back(DmTpaItem{(const cplx*)Q[i], (cplx*)S[i], kbs[i]->n_pw, nb, use_tpa ? kbs[i]->kin.p : nullptr,
                            use_tpa ? mean_kin + (size_t)i * nb : nullptr, inv_w_host[i]});
      mt = std::max(mt, (long long)kbs[i]->n_pw * nb);
    }
    LAUNCH(ctx, k_dm_tpa, dim3(grid_for(ctx, mt), (unsigned)n), DM_THREADS, 0, ctx->slot[0].ring.put(v, ctx->stream));
  }
  finish(ctx);
  API_END(ctx)
}

int dftk_b200_real_dots_multi(int64_t n_pairs, int64_t n_blocks, dftk_b200_kblock* const* kbs, const void* const* A,
                              const void* const* B, int64_t n_bands, double* out_host) {
  dftk_b200_ctx* ctx = ctx_of(n_blocks, kbs);
  API_BEGIN
  check_blocks(ctx, n_blocks, kbs, n_bands, "real_dots_multi");
  REQUIRE(n_pairs >= 1 && out_host, "real_dots_multi: bad argument");
  if (n_blocks == 0) {
    for (int64_t p = 0; p < n_pairs; ++p) out_host[p] = 0.0;
    return DFTK_B200_OK;
  }
  check_orbitals(ctx, n_pairs * n_blocks, A, "real_dots_multi");
  check_orbitals(ctx, n_pairs * n_blocks, B, "real_dots_multi");
  std::vector<DmDotItem> v;
  for (int64_t p = 0; p < n_pairs; ++p)
    for (int64_t i = 0; i < n_blocks; ++i) {
      const int64_t k = p * n_blocks + i;
      v.push_back(DmDotItem{(const cplx*)A[k], (const cplx*)B[k], nullptr, nullptr, 0.0, (long long)kbs[i]->n_pw * n_bands});
    }
  dots(ctx, v, (int)n_pairs, (int)n_blocks, out_host);
  API_END(ctx)
}

int dftk_b200_axpy_dot_multi(int64_t n_blocks, dftk_b200_kblock* const* kbs, void* const* Y, const void* const* X, double c,
                             const void* const* Z, int64_t n_bands, double* out_host) {
  dftk_b200_ctx* ctx = ctx_of(n_blocks, kbs);
  API_BEGIN
  check_blocks(ctx, n_blocks, kbs, n_bands, "axpy_dot_multi");
  if (out_host) *out_host = 0.0;
  if (n_blocks == 0) return DFTK_B200_OK;
  check_orbitals(ctx, n_blocks, (const void* const*)Y, "axpy_dot_multi");
  check_orbitals(ctx, n_blocks, X, "axpy_dot_multi");
  if (Z) {
    check_orbitals(ctx, n_blocks, Z, "axpy_dot_multi");
    REQUIRE(out_host, "axpy_dot_multi: NULL result");
  }
  std::vector<DmDotItem> v;
  for (int64_t i = 0; i < n_blocks; ++i)
    v.push_back(DmDotItem{Z ? (const cplx*)Z[i] : nullptr, (const cplx*)Y[i], (cplx*)Y[i], (const cplx*)X[i], c,
                          (long long)kbs[i]->n_pw * n_bands});
  dots(ctx, v, Z ? 1 : 0, (int)n_blocks, out_host);
  API_END(ctx)
}

}  // extern "C"
