// Moving data between plane-wave bases (transfer.py; reference seams src/transfer.jl, src/symmetry.jl apply_symop,
// src/supercell.jl, src/interpolation.jl): the batched sphere remap with its table builder, the Fourier block copy between
// cubes and the periodic quadratic B-spline interpolation.  Kernel bodies are in transfer_core.cuh.
#include <algorithm>
#include "structs.cuh"
#include "transfer_core.cuh"

using namespace dftk;

namespace {

#define TR_THREADS 256
#define TR_BAND_GROUP 16   // bands per CTA of the remap: the table entry of a column is read once for this many rows

struct TrTableArgs { int M[9]; int delta[3]; double tau[3]; };
struct TrRemapItem {
  const cplx* src; cplx* dst; const long long* idx; const cplx* phase;
  long long ld_src, ld_dst, row_offset, n_dst, n_bands;
};

__global__ void __launch_bounds__(TR_THREADS) k_remap_tables(long long n, const long long* __restrict__ G, TrTableArgs a,
                                                           const long long* __restrict__ lookup, int nx, int ny, int nz,
                                                           long long* __restrict__ idx, cplx* __restrict__ phase) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) tr_table_entry(j, G, a.M, a.delta, a.tau, lookup, nx, ny, nz, idx, phase);
}

// blockIdx.y: pair; blockIdx.z: group of TR_BAND_GROUP bands; one thread per destination column j (coalesced writes).
__global__ void __launch_bounds__(TR_THREADS) k_sphere_remap(const TrRemapItem* __restrict__ items) {
  const TrRemapItem it = items[blockIdx.y];
  const long long b0 = (long long)blockIdx.z * TR_BAND_GROUP;
  const long long b1 = b0 + TR_BAND_GROUP < it.n_bands ? b0 + TR_BAND_GROUP : it.n_bands;
  for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < it.n_dst; j += (long long)gridDim.x * blockDim.x) {
    const long long i = it.idx[j];
#pragma unroll 4
    for (long long b = b0; b < b1; ++b)
      it.dst[(it.row_offset + b) * it.ld_dst + j] = tr_remap_value(it.src + b * it.ld_src, i, it.phase, j);
  }
}

__global__ void __launch_bounds__(TR_THREADS) k_block_copy(const cplx* __restrict__ in, int nxi, int nyi, int nzi,
                                                         cplx* __restrict__ out, int nxo, int nyo, int nzo) {
  const long long Ni = (long long)nxi * nyi * nzi, No = (long long)nxo * nyo * nzo;
  const cplx* src = in + blockIdx.y * Ni;
  cplx* dst = out + blockIdx.y * No;
  for (long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x; o < No; o += (long long)gridDim.x * blockDim.x)
    dst[o] = tr_block_copy_value(o, src, nxi, nyi, nzi, nxo, nyo, nzo);
}

__global__ void __launch_bounds__(TR_THREADS) k_bspline_prefilter(cplx* __restrict__ f, int nx, int ny, int nz, long long batch) {
  const long long N = (long long)nx * ny * nz;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (long long)gridDim.x * blockDim.x) {
    const double s = tr_bspline_prefilter_factor(i, nx, ny, nz);
    for (long long b = 0; b < batch; ++b) {
      const cplx v = f[b * N + i];
      f[b * N + i] = make_double2(s * v.x, s * v.y);
    }
  }
}

struct TrRep { int r[3]; };

__global__ void __launch_bounds__(TR_THREADS) k_bspline_eval(const double* __restrict__ f, int nx, int ny, int nz, TrRep rep,
                                                           double* __restrict__ out, int nxo, int nyo, int nzo, int direct) {
  const long long Ni = (long long)nx * ny * nz, No = (long long)nxo * nyo * nzo;
  const double* src = f + blockIdx.y * Ni;
  double* dst = out + blockIdx.y * No;
  for (long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x; o < No; o += (long long)gridDim.x * blockDim.x)
    dst[o] = tr_bspline_value(o, src, nx, ny, nz, rep.r, nxo, nyo, nzo, direct);
}

unsigned tr_grid(dftk_b200_ctx* ctx, long long total) {
  const long long g = (total + TR_THREADS - 1) / TR_THREADS;
  return (unsigned)std::max<long long>(1, std::min<long long>(g, (long long)ctx->sm_count * 32));
}

void check_cube(int nx, int ny, int nz, const char* what) {
  REQUIRE(nx >= 1 && ny >= 1 && nz >= 1, std::string(what) + ": cube sizes must be positive");
}

}  // namespace

extern "C" {

int dftk_b200_remap_tables(dftk_b200_ctx* ctx, int64_t n_G, const int64_t* G, const int32_t* M, const int32_t* delta,
                           const double* tau, const int64_t* lookup, int nx, int ny, int nz, int64_t* idx, void* phase) {
  API_BEGIN
  REQUIRE(ctx && n_G >= 0 && M && delta && (tau || !phase), "remap_tables: bad argument");
  check_cube(nx, ny, nz, "remap_tables");
  REQUIRE(!is_device_ptr(M) && !is_device_ptr(delta) && !(tau && is_device_ptr(tau)), "remap_tables: M, delta and tau are host arrays");
  if (n_G == 0) return DFTK_B200_OK;
  require_device(ctx, G, "remap_tables: arrays");
  require_device(ctx, lookup, "remap_tables: arrays");
  require_device(ctx, idx, "remap_tables: arrays");
  if (phase) require_device(ctx, phase, "remap_tables: arrays");
  TrTableArgs a;
  for (int i = 0; i < 9; ++i) a.M[i] = M[i];
  for (int i = 0; i < 3; ++i) {
    a.delta[i] = delta[i];
    a.tau[i] = tau ? tau[i] : 0.0;
  }
  LAUNCH(ctx, k_remap_tables, (unsigned)((n_G + TR_THREADS - 1) / TR_THREADS), TR_THREADS, 0, (long long)n_G,
         (const long long*)G, a, (const long long*)lookup, nx, ny, nz, (long long*)idx, (cplx*)phase);
  API_END(ctx)
}

int dftk_b200_sphere_remap(dftk_b200_ctx* ctx, int64_t n_pairs, const void* const* src, const int64_t* ld_src, void* const* dst,
                           const int64_t* ld_dst, const int64_t* row_offset, const int64_t* n_bands,
                           const int64_t* const* idx, const int64_t* n_dst, const void* const* phase) {
  API_BEGIN
  REQUIRE(ctx && n_pairs >= 0, "sphere_remap: bad argument");
  if (n_pairs == 0) return DFTK_B200_OK;
  REQUIRE(src && ld_src && dst && ld_dst && n_bands && idx && n_dst, "sphere_remap: NULL argument list");
  REQUIRE(n_pairs <= 65535, "sphere_remap: at most 65535 pairs per call");
  std::vector<TrRemapItem> items;
  long long max_dst = 1, max_bands = 1;
  for (int64_t p = 0; p < n_pairs; ++p) {
    REQUIRE(n_bands[p] >= 0 && n_dst[p] >= 0 && ld_dst[p] >= n_dst[p] && ld_src[p] >= 0 && (!row_offset || row_offset[p] >= 0),
            "sphere_remap: bad sizes");
    if (n_bands[p] == 0 || n_dst[p] == 0) continue;
    require_device(ctx, src[p], "sphere_remap: arrays");
    require_device(ctx, dst[p], "sphere_remap: arrays");
    require_device(ctx, idx[p], "sphere_remap: arrays");
    if (phase && phase[p]) require_device(ctx, phase[p], "sphere_remap: arrays");
    items.push_back(TrRemapItem{(const cplx*)src[p], (cplx*)dst[p], (const long long*)idx[p],
                                phase ? (const cplx*)phase[p] : nullptr, (long long)ld_src[p], (long long)ld_dst[p],
                                row_offset ? (long long)row_offset[p] : 0, (long long)n_dst[p], (long long)n_bands[p]});
    max_dst = std::max<long long>(max_dst, n_dst[p]);
    max_bands = std::max<long long>(max_bands, n_bands[p]);
  }
  if (items.empty()) return DFTK_B200_OK;
  const TrRemapItem* d = ctx->slot[0].ring.put(items, ctx->stream);
  const unsigned gx = (unsigned)std::min<long long>((max_dst + TR_THREADS - 1) / TR_THREADS, 65535);
  const unsigned gz = (unsigned)((max_bands + TR_BAND_GROUP - 1) / TR_BAND_GROUP);
  REQUIRE(gz <= 65535, "sphere_remap: too many bands");
  LAUNCH(ctx, k_sphere_remap, dim3(gx, (unsigned)items.size(), gz), TR_THREADS, 0, d);
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  ctx->slot[0].ring.rewind();
  API_END(ctx)
}

int dftk_b200_fourier_block_copy(dftk_b200_ctx* ctx, const void* in, int nx_in, int ny_in, int nz_in, void* out, int nx_out,
                                 int ny_out, int nz_out, int64_t batch) {
  API_BEGIN
  REQUIRE(ctx && batch >= 0 && batch <= 65535, "fourier_block_copy: bad argument");
  check_cube(nx_in, ny_in, nz_in, "fourier_block_copy");
  check_cube(nx_out, ny_out, nz_out, "fourier_block_copy");
  if (batch == 0) return DFTK_B200_OK;
  require_device(ctx, in, "fourier_block_copy: arrays");
  require_device(ctx, out, "fourier_block_copy: arrays");
  REQUIRE(in != out, "fourier_block_copy: in and out must not alias");
  const long long No = (long long)nx_out * ny_out * nz_out;
  LAUNCH(ctx, k_block_copy, dim3(tr_grid(ctx, No), (unsigned)batch), TR_THREADS, 0, (const cplx*)in, nx_in, ny_in, nz_in,
         (cplx*)out, nx_out, ny_out, nz_out);
  API_END(ctx)
}

int dftk_b200_bspline2_prefilter(dftk_b200_ctx* ctx, void* f, int nx, int ny, int nz, int64_t batch) {
  API_BEGIN
  REQUIRE(ctx && batch >= 0, "bspline2_prefilter: bad argument");
  check_cube(nx, ny, nz, "bspline2_prefilter");
  if (batch == 0) return DFTK_B200_OK;
  require_device(ctx, f, "bspline2_prefilter: arrays");
  LAUNCH(ctx, k_bspline_prefilter, tr_grid(ctx, (long long)nx * ny * nz), TR_THREADS, 0, (cplx*)f, nx, ny, nz, (long long)batch);
  API_END(ctx)
}

int dftk_b200_bspline2_evaluate(dftk_b200_ctx* ctx, const double* f, int nx, int ny, int nz, const int32_t* rep, double* out,
                                int nx_out, int ny_out, int nz_out, int64_t batch, int direct) {
  API_BEGIN
  REQUIRE(ctx && rep && batch >= 0 && batch <= 65535, "bspline2_evaluate: bad argument");
  REQUIRE(!is_device_ptr(rep) && rep[0] >= 1 && rep[1] >= 1 && rep[2] >= 1, "bspline2_evaluate: rep must be 3 positive host integers");
  check_cube(nx, ny, nz, "bspline2_evaluate");
  check_cube(nx_out, ny_out, nz_out, "bspline2_evaluate");
  if (direct)
    REQUIRE((long long)nx * rep[0] == nx_out && (long long)ny * rep[1] == ny_out && (long long)nz * rep[2] == nz_out,
            "bspline2_evaluate: direct sampling needs n_out = rep * n_in on every axis");
  if (batch == 0) return DFTK_B200_OK;
  require_device(ctx, f, "bspline2_evaluate: arrays");
  require_device(ctx, out, "bspline2_evaluate: arrays");
  REQUIRE((const void*)f != (const void*)out, "bspline2_evaluate: in and out must not alias");
  TrRep r{{rep[0], rep[1], rep[2]}};
  const long long No = (long long)nx_out * ny_out * nz_out;
  LAUNCH(ctx, k_bspline_eval, dim3(tr_grid(ctx, No), (unsigned)batch), TR_THREADS, 0, f, nx, ny, nz, r, out, nx_out, ny_out,
         nz_out, direct);
  API_END(ctx)
}

}  // extern "C"
