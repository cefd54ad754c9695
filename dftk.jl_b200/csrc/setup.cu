// Setup kernels next to the hot path (SURVEY §8f rank 4): the O(n_atoms x N) structure-factor work that dominates the
// time to the first SCF step of large cells.
//   * structure factors on the FFT cube (build_local_potential, src/terms/local.jl:108-138; guess_density,
//     src/density_methods.jl:103-181): out[G] = sum_a c_a exp(-2 pi i G.r_a), G from the cube index
//   * projector table of a k-block (build_projection_vectors, src/terms/nonlocal.jl:166-199):
//     P[(a, p), G] = exp(-2 pi i (G+k).r_a) ff[p, G]
//   * radial transforms of the numerical tables of a UPF pseudopotential (src/pseudo/PspUpf.jl, src/common/hankel.jl): the
//     projector, local-potential and core/valence density form factors at every distinct |q|
#include <algorithm>
#include "structs.cuh"

namespace dftk {

__device__ __forceinline__ int wrapped_index(int i, int n) { return i <= (n - 1) / 2 ? i : i - n; }   // src/fft.jl:24-31

// one thread per cube point, atoms staged through shared memory in tiles of 256
__global__ void __launch_bounds__(256)
k_structure_factor(int nx, int ny, int nz, int n_atoms, const double* __restrict__ pos, const double* __restrict__ coeff,
                   cplx* __restrict__ out) {
  __shared__ double sp[256 * 4];
  const int64_t N = (int64_t)nx * ny * nz;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = idx < N;
  const int ix = (int)(idx % nx), iy = (int)((idx / nx) % ny), iz = (int)(idx / ((int64_t)nx * ny));
  const double gx = wrapped_index(ix, nx), gy = wrapped_index(iy, ny), gz = wrapped_index(live ? iz : 0, nz);
  double re = 0.0, im = 0.0;
  for (int a0 = 0; a0 < n_atoms; a0 += 256) {
    const int na = min(256, n_atoms - a0);
    __syncthreads();
    if ((int)threadIdx.x < na) {
      sp[4 * threadIdx.x] = pos[3 * (a0 + threadIdx.x)];
      sp[4 * threadIdx.x + 1] = pos[3 * (a0 + threadIdx.x) + 1];
      sp[4 * threadIdx.x + 2] = pos[3 * (a0 + threadIdx.x) + 2];
      sp[4 * threadIdx.x + 3] = coeff ? coeff[a0 + threadIdx.x] : 1.0;
    }
    __syncthreads();
    if (live)
      for (int a = 0; a < na; ++a) {
        double s, c;
        sincospi(-2.0 * (gx * sp[4 * a] + gy * sp[4 * a + 1] + gz * sp[4 * a + 2]), &s, &c);
        re += sp[4 * a + 3] * c;
        im += sp[4 * a + 3] * s;
      }
  }
  if (live) out[idx] = make_double2(re, im);
}

// grid (ceil(n_pw/256), n_atoms): all n_rows projectors of one atom for 256 plane waves
__global__ void __launch_bounds__(256)
k_build_projectors(int64_t n_pw, const double* __restrict__ gpk, const double* __restrict__ pos, int n_rows,
                   const cplx* __restrict__ ff, cplx* __restrict__ P) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pw) return;
  const int a = blockIdx.y;
  double s, c;
  sincospi(-2.0 * (gpk[i] * pos[3 * a] + gpk[n_pw + i] * pos[3 * a + 1] + gpk[2 * n_pw + i] * pos[3 * a + 2]), &s, &c);
  for (int p = 0; p < n_rows; ++p) {
    const cplx f = ff[(int64_t)p * n_pw + i];
    P[((int64_t)a * n_rows + p) * n_pw + i] = make_double2(c * f.x - s * f.y, c * f.y + s * f.x);
  }
}

// ---------------------------------------------------------------- radial transforms of numerical pseudopotentials
// F[f, q] = 4π / q^l_f · Σ_i g_f[i] j_{l_f}(q r_i)  (the modified Hankel transform of src/common/hankel.jl; g_f = w_i r_i² f(r_i)
// with the quadrature weights folded in), and for q <= 10 eps the moment limit 4π/(2l+1)!! · Σ_i g_f[i] r_i^l (hankel.jl:26-33).
// One thread per q holds the accumulators of every function; r and g pass through shared memory in tiles, and one sincos per
// (q, r_i) serves all functions.  Blocks along y split the mesh; k_radial_finalize adds their partial sums in a fixed order.
constexpr int RT_THREADS = 128, RT_TILE = 128;
constexpr double RT_SMALL_Q = 10 * 2.220446049250313e-16;

// j_l(x) = x^l/(2l+1)!! Σ_k (-x²/2)^k / (k! (2l+3)(2l+5)···(2l+2k+1)); below x = 2 the closed forms lose digits to cancellation
__device__ __forceinline__ double jl_series(int l, double x2, double lead) {
  double t = 1.0, sum = 1.0;
#pragma unroll
  for (int k = 1; k <= 12; ++k) {
    t *= -0.5 * x2 / (double)(k * (2 * l + 2 * k + 1));
    sum += t;
  }
  return lead * sum;
}

template <int NF>
__global__ void __launch_bounds__(RT_THREADS)
k_radial_transform(int64_t n_r, int64_t chunk, const double* __restrict__ r, int n_f, const double* __restrict__ g, RadialL L,
                   int64_t n_q, const double* __restrict__ q, double* __restrict__ part) {
  __shared__ double sr[RT_TILE];
  __shared__ double sg[NF][RT_TILE];
  const int64_t iq = (int64_t)blockIdx.x * RT_THREADS + threadIdx.x;
  const bool live = iq < n_q;
  const double qv = live ? q[iq] : 1.0;
  const bool small = qv <= RT_SMALL_Q;
  double acc[NF];
#pragma unroll
  for (int f = 0; f < NF; ++f) acc[f] = 0.0;
  const int64_t i_begin = (int64_t)blockIdx.y * chunk, i_end = min(n_r, i_begin + chunk);
  for (int64_t i0 = i_begin; i0 < i_end; i0 += RT_TILE) {
    const int nt = (int)min((int64_t)RT_TILE, i_end - i0);
    __syncthreads();
    for (int j = threadIdx.x; j < RT_TILE; j += RT_THREADS) {
      sr[j] = j < nt ? r[i0 + j] : 0.0;
#pragma unroll
      for (int f = 0; f < NF; ++f) sg[f][j] = (f < n_f && j < nt) ? g[(int64_t)f * n_r + i0 + j] : 0.0;
    }
    __syncthreads();
    if (!live) continue;
    for (int j = 0; j < nt; ++j) {
      const double ri = sr[j];
      double b0, b1, b2, b3;
      if (small) {                       // r^l: the moments of the q -> 0 limit
        b0 = 1.0; b1 = ri; b2 = ri * ri; b3 = b2 * ri;
      } else {
        const double x = qv * ri;
        if (x < 2.0) {
          const double x2 = x * x;
          b0 = jl_series(0, x2, 1.0);
          b1 = L.lmax >= 1 ? jl_series(1, x2, x / 3) : 0.0;
          b2 = L.lmax >= 2 ? jl_series(2, x2, x2 / 15) : 0.0;
          b3 = L.lmax >= 3 ? jl_series(3, x2, x2 * x / 105) : 0.0;
        } else {                         // closed forms by upward recurrence (stable for l <= 3 < x + 2)
          double s, c;
          sincos(x, &s, &c);
          const double inv = 1.0 / x;
          b0 = s * inv;
          b1 = (b0 - c) * inv;
          b2 = 3.0 * b1 * inv - b0;
          b3 = 5.0 * b2 * inv - b1;
        }
      }
#pragma unroll
      for (int f = 0; f < NF; ++f) {
        const int l = L.l[f];
        acc[f] += sg[f][j] * (l == 0 ? b0 : l == 1 ? b1 : l == 2 ? b2 : b3);
      }
    }
  }
  if (!live) return;
#pragma unroll
  for (int f = 0; f < NF; ++f)
    if (f < n_f) part[((int64_t)blockIdx.y * n_f + f) * n_q + iq] = acc[f];
}

__global__ void k_radial_finalize(int n_split, int n_f, RadialL L, int64_t n_q, const double* __restrict__ q,
                                  const double* __restrict__ part, double* __restrict__ F) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)n_f * n_q) return;
  const int f = (int)(idx / n_q);
  const int64_t iq = idx % n_q;
  double s = 0.0;
  for (int k = 0; k < n_split; ++k) s += part[((int64_t)k * n_f + f) * n_q + iq];
  const int l = L.l[f];
  const double qv = q[iq];
  double den = 1.0;
  if (qv <= RT_SMALL_Q)
    den = l == 0 ? 1.0 : l == 1 ? 3.0 : l == 2 ? 15.0 : 105.0;     // (2l+1)!!
  else
    for (int k = 0; k < l; ++k) den *= qv;
  F[idx] = 4.0 * M_PI * s / den;
}

template <int NF>
static void launch_radial(dftk_b200_ctx* ctx, dim3 grid, int64_t n_r, int64_t chunk, const double* r, int n_f, const double* g,
                          const RadialL& L, int64_t n_q, const double* q, double* part) {
  LAUNCH(ctx, k_radial_transform<NF>, grid, RT_THREADS, 0, n_r, chunk, r, n_f, g, L, n_q, q, part);
}

void radial_transform(dftk_b200_ctx* ctx, int64_t n_r, const double* r, int n_f, const double* g, const int* l_host, int64_t n_q,
                      const double* q, double* F) {
  if (n_f == 0 || n_q == 0) return;
  const int64_t q_blocks = (n_q + RT_THREADS - 1) / RT_THREADS;
  REQUIRE(q_blocks <= 0x7fffffff, "radial_transform: too many q values");
  // split the mesh until about two blocks per SM are in flight; every split covers whole tiles
  const int64_t tiles = (n_r + RT_TILE - 1) / RT_TILE;
  const int64_t want = std::max<int64_t>(1, (2 * ctx->sm_count + q_blocks - 1) / q_blocks);
  const int64_t chunk = RT_TILE * ((tiles + std::min(tiles, want) - 1) / std::min(tiles, want));
  const int n_split = (int)((n_r + chunk - 1) / chunk);
  for (int f0 = 0; f0 < n_f; f0 += RADIAL_MAX_F) {
    const int nf = std::min(RADIAL_MAX_F, n_f - f0);
    RadialL L{};
    for (int f = 0; f < nf; ++f) {
      REQUIRE(l_host[f0 + f] >= 0 && l_host[f0 + f] <= 3, "radial_transform: l must be 0..3");
      L.l[f] = l_host[f0 + f];
      L.lmax = std::max(L.lmax, L.l[f]);
    }
    double* part = ctx->radial_part.ensure((size_t)n_split * nf * n_q);
    const dim3 grid((unsigned)q_blocks, (unsigned)n_split);
    const double* gf = g + (int64_t)f0 * n_r;
    if (nf == 1) launch_radial<1>(ctx, grid, n_r, chunk, r, nf, gf, L, n_q, q, part);
    else if (nf <= 4) launch_radial<4>(ctx, grid, n_r, chunk, r, nf, gf, L, n_q, q, part);
    else if (nf <= 8) launch_radial<8>(ctx, grid, n_r, chunk, r, nf, gf, L, n_q, q, part);
    else launch_radial<RADIAL_MAX_F>(ctx, grid, n_r, chunk, r, nf, gf, L, n_q, q, part);
    const int64_t n_out = (int64_t)nf * n_q;
    LAUNCH(ctx, k_radial_finalize, (unsigned)((n_out + 255) / 256), 256, 0, n_split, nf, L, n_q, q, (const double*)part,
           F + (int64_t)f0 * n_q);
  }
}

void structure_factor(dftk_b200_grid* g, int n_atoms, const double* pos_host, const double* coeff_host, cplx* out) {
  dftk_b200_ctx* ctx = g->ctx;
  double* d = ctx->sym_d.ensure((size_t)4 * n_atoms + 8);
  CUDA_CHECK(cudaMemcpyAsync(d, pos_host, (size_t)3 * n_atoms * sizeof(double), cudaMemcpyDefault, ctx->stream));
  if (coeff_host) CUDA_CHECK(cudaMemcpyAsync(d + 3 * n_atoms, coeff_host, (size_t)n_atoms * sizeof(double), cudaMemcpyDefault, ctx->stream));
  LAUNCH(ctx, k_structure_factor, (unsigned)((g->N + 255) / 256), 256, 0, g->nx, g->ny, g->nz, n_atoms, (const double*)d,
         coeff_host ? (const double*)(d + 3 * n_atoms) : (const double*)nullptr, out);
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));     // the host arrays may go away
}

void build_projectors(dftk_b200_ctx* ctx, int64_t n_pw, const double* gpk, int n_atoms, const double* pos_host, int n_rows,
                      const cplx* ff, cplx* P) {
  if (n_atoms == 0 || n_rows == 0) return;
  REQUIRE(n_atoms <= 65535, "build_projectors: too many atoms in one group");
  double* d = ctx->sym_d.ensure((size_t)3 * n_atoms + 8);
  CUDA_CHECK(cudaMemcpyAsync(d, pos_host, (size_t)3 * n_atoms * sizeof(double), cudaMemcpyDefault, ctx->stream));
  LAUNCH(ctx, k_build_projectors, dim3((unsigned)((n_pw + 255) / 256), (unsigned)n_atoms), 256, 0, n_pw, gpk, (const double*)d,
         n_rows, ff, P);
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
}

}  // namespace dftk
