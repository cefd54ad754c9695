// Batched overlap products with an indirect right operand (wannier.py; reference seam src/external/wannier_shared.jl
// overlap_Mmn_k_kpb and compute_amn_kpoint): C_p = A_p^H B_p[idx_p] for all pairs of one call.  Blocks of <= SMALL_MAX_N
// columns take the fused gather-product of overlap_core.cuh (two launches whatever the pair count); larger blocks gather
// B_p[idx_p] into one scratch block (the sphere-remap body of transfer_core.cuh) and take the DMMA ZGEMM, one pair at a time.
#include <algorithm>
#include "structs.cuh"
#include "lobpcg_small.cuh"
#include "transfer_core.cuh"
#include "overlap_core.cuh"

using namespace dftk;

namespace {

__global__ void __launch_bounds__(OV_THREADS) k_ov_partial(const OvGroup* __restrict__ groups, const OvPair* __restrict__ pairs,
                                                         int n_chunks, int n_a, int n_b, long long n_pairs, cplx* __restrict__ ws) {
  extern __shared__ __align__(16) unsigned char ov_smem[];
  ov_cta(groups[blockIdx.x], pairs, (int)blockIdx.y, n_chunks, n_a, n_b, OV_THREADS, n_pairs, ws, (cplx*)ov_smem);
}

__global__ void __launch_bounds__(OV_THREADS) k_ov_reduce(const cplx* __restrict__ ws, int n_chunks, long long n_pairs, int nab,
                                                        cplx* __restrict__ C) {
  const long long total = n_pairs * nab;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x)
    C[e] = ov_reduce_entry(ws, n_chunks, n_pairs, nab, e / nab, (int)(e % nab));
}

// dst[b, j] = B[b, idx[j]] for b < n_b, j < n_G (dst: n_b x n_G, row length n_G)
__global__ void __launch_bounds__(OV_THREADS) k_ov_gather(const cplx* __restrict__ B, long long ld_b, const long long* __restrict__ idx,
                                                        long long n_G, cplx* __restrict__ dst) {
  const cplx* src = B + (long long)blockIdx.y * ld_b;
  for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < n_G; j += (long long)gridDim.x * blockDim.x)
    dst[(long long)blockIdx.y * n_G + j] = tr_remap_value(src, idx[j], nullptr, j);
}

unsigned ov_grid(dftk_b200_ctx* ctx, long long total) {
  const long long g = (total + OV_THREADS - 1) / OV_THREADS;
  return (unsigned)std::max<long long>(1, std::min<long long>(g, (long long)ctx->sm_count * 32));
}

// one pair at a time: gather B_p[idx_p] (n_b x n_G) into scratch, then C_p = A_p^H gathered on the DMMA ZGEMM
void overlap_large(dftk_b200_ctx* ctx, int64_t n_pairs, int64_t n_a, int64_t n_b, const void* const* A, const int64_t* ld_a,
                   const int64_t* n_G, const void* const* B, const int64_t* ld_b, const int64_t* const* idx, cplx* Cd,
                   long long max_nG) {
  const long long nab = n_a * n_b;
  REQUIRE(n_b <= 65535, "overlap_multi: too many columns");
  for (int64_t p = 0; p < n_pairs; ++p) {
    cplx* Cp = Cd + p * nab;
    if (n_G[p] == 0) {
      CUDA_CHECK(cudaMemsetAsync(Cp, 0, nab * sizeof(cplx), ctx->stream));
      continue;
    }
    const cplx* Bp = (const cplx*)B[p];
    long long ldb = ld_b[p];
    if (idx && idx[p]) {
      cplx* scratch = ctx->ov_scratch.ensure((size_t)n_b * max_nG);
      LAUNCH(ctx, k_ov_gather, dim3(std::min<unsigned>(ov_grid(ctx, n_G[p]), 65535u), (unsigned)n_b), OV_THREADS, 0, Bp,
             (long long)ld_b[p], (const long long*)idx[p], (long long)n_G[p], scratch);
      Bp = scratch;
      ldb = n_G[p];
    }
    zgemm(ctx, 2, n_a, n_b, n_G[p], make_double2(1.0, 0.0), (const cplx*)A[p], ld_a[p], Bp, ldb, make_double2(0.0, 0.0), Cp, n_a);
  }
}

}  // namespace

extern "C" {

int dftk_b200_overlap_multi(dftk_b200_ctx* ctx, int64_t n_pairs, int64_t n_a, int64_t n_b, const void* const* A,
                            const int64_t* ld_a, const int64_t* n_G, const void* const* B, const int64_t* ld_b,
                            const int64_t* const* idx, void* C) {
  API_BEGIN
  REQUIRE(ctx && n_pairs >= 0 && n_a >= 1 && n_b >= 1, "overlap_multi: bad argument");
  if (n_pairs == 0) return DFTK_B200_OK;
  REQUIRE(A && ld_a && n_G && B && ld_b, "overlap_multi: NULL argument list");
  REQUIRE((long long)n_a * n_b <= (1LL << 30), "overlap_multi: blocks too large");
  require_device(ctx, C, "overlap_multi: arrays");
  long long max_nG = 0;
  for (int64_t p = 0; p < n_pairs; ++p) {
    const bool ident = !idx || !idx[p];
    REQUIRE(n_G[p] >= 0 && ld_a[p] >= n_G[p] && ld_b[p] >= 1 && (!ident || ld_b[p] >= n_G[p]), "overlap_multi: bad sizes");
    require_device(ctx, A[p], "overlap_multi: arrays");
    require_device(ctx, B[p], "overlap_multi: arrays");
    if (!ident && n_G[p] > 0) require_device(ctx, idx[p], "overlap_multi: arrays");
    max_nG = std::max<long long>(max_nG, n_G[p]);
  }
  const long long nab = n_a * n_b;
  cplx* Cd = (cplx*)C;
  if (std::max(n_a, n_b) > SMALL_MAX_N) {
    overlap_large(ctx, n_pairs, n_a, n_b, A, ld_a, n_G, B, ld_b, idx, Cd, max_nG);
    return DFTK_B200_OK;
  }
  // fused path: groups of consecutive pairs with the same A, a row split into chunks for enough CTAs, two launches
  std::vector<OvGroup> groups;
  std::vector<OvPair> pairs;
  for (int64_t p = 0; p < n_pairs; ++p) {
    pairs.push_back(OvPair{(const cplx*)B[p], (long long)ld_b[p], idx ? (const long long*)idx[p] : nullptr});
    if (!groups.empty() && groups.back().A == A[p] && groups.back().ld_a == ld_a[p] && groups.back().n_G == n_G[p])
      groups.back().count++;
    else
      groups.push_back(OvGroup{(const cplx*)A[p], (long long)ld_a[p], (long long)n_G[p], (int)p, 1});
  }
  const long long n_groups = (long long)groups.size();
  const long long want = (8LL * ctx->sm_count + n_groups - 1) / n_groups;
  const int n_chunks = (int)std::max<long long>(1, std::min<long long>({want, (max_nG + OV_ROWS - 1) / OV_ROWS, OV_MAX_CHUNKS}));
  REQUIRE(n_groups <= 0x7fffffffLL, "overlap_multi: too many pairs");
  DescRing& ring = ctx->slot[0].ring;
  ring.reserve(DescRing::padded(groups) + DescRing::padded(pairs), ctx->stream);
  const OvGroup* d_groups = ring.put(groups, ctx->stream);
  const OvPair* d_pairs = ring.put(pairs, ctx->stream);
  cplx* ws = ctx->ov_ws.ensure((size_t)n_chunks * n_pairs * nab);
  const size_t smem = (size_t)ov_smem_entries((int)n_a, (int)n_b) * sizeof(cplx);
  CUDA_CHECK(cudaFuncSetAttribute(k_ov_partial, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  LAUNCH(ctx, k_ov_partial, dim3((unsigned)n_groups, (unsigned)n_chunks), OV_THREADS, smem, d_groups, d_pairs, n_chunks, (int)n_a,
         (int)n_b, (long long)n_pairs, ws);
  LAUNCH(ctx, k_ov_reduce, ov_grid(ctx, n_pairs * nab), OV_THREADS, 0, (const cplx*)ws, n_chunks, (long long)n_pairs, (int)nab, Cd);
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  ring.rewind();
  API_END(ctx)
}

}  // extern "C"
