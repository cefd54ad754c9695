// Force kernels next to the hot path (SURVEY §8f rank 4): local-potential forces (src/terms/local.jl:152-181) and
// nonlocal-projector forces (src/terms/nonlocal.jl:49-100).  Bodies live in forces_core.cuh.
#include "structs.cuh"
#include "forces_core.cuh"

namespace dftk {

// grid (blocks_per_atom, n_atoms); partial[(atom * gridDim.x + blockIdx.x) * 3 + α]
__global__ void __launch_bounds__(256)
k_local_forces(int nx, int ny, int nz, const cplx* w, const double* pos, double* partial) {
  const int atom = blockIdx.y;
  const double rx = pos[3 * atom], ry = pos[3 * atom + 1], rz = pos[3 * atom + 2];
  const int64_t N = (int64_t)nx * ny * nz;
  double acc[3] = {0.0, 0.0, 0.0};
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N; i += (int64_t)gridDim.x * blockDim.x)
    local_force_point(i, nx, ny, nz, w, rx, ry, rz, acc);
  __shared__ double red[3][8];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    double v = acc[a];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[a][threadIdx.x >> 5] = v;
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    double v = 0.0;
    for (int wv = 0; wv < 8; ++wv) v += red[threadIdx.x][wv];
    partial[((int64_t)atom * gridDim.x + blockIdx.x) * 3 + threadIdx.x] = v;
  }
}

// one thread per (atom, α): fixed-order sum of the block partials, F = -2π Σ
__global__ void k_local_forces_reduce(const double* partial, int n_atoms, int n_blocks, double* out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 3 * n_atoms) return;
  const int atom = t / 3, a = t % 3;
  double s = 0.0;
  for (int b = 0; b < n_blocks; ++b) s += partial[((int64_t)atom * n_blocks + b) * 3 + a];
  out[t] = -2.0 * FORCES_PI * s;
}

__global__ void __launch_bounds__(256)
k_scale_by_momentum(int64_t n_rows, int64_t nb, const double* gpk, const cplx* psi, int64_t ld, cplx* out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rows) return;
  scale_by_momentum_point(i, blockIdx.y, blockIdx.z, n_rows, nb, gpk, psi, ld, out);
}

__global__ void k_nonlocal_force_rows(int64_t np, int64_t nb, const cplx* dproj, const cplx* pa, const double* w,
                                      double* f) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= np) return;
  nonlocal_force_row(j, blockIdx.y, np, nb, dproj, pa, w, f);
}

// ---------------------------------------------------------------------------------------------- Ewald (ewald.jl:64-168)
// Energy and forces of point charges in a uniform background, q = 0: the O(n_atoms² n_R) real-space sum and the
// O(n_atoms n_G) reciprocal sum as one kernel each (one CTA per atom, fixed-order block reductions: deterministic), after
// the structure factor S(G) = Σ_j Z_j e^{2πi G·r_j} (one thread per G).
struct EwaldGeom {
  double lat[9];     // lattice vectors as columns, row-major storage lat[3*r + c]
  double recip[9];
  double eta, vol;
  int glim[3], rlim[3];
  int n_atoms;
};
__device__ __forceinline__ void ewald_block_sum4(double* v) {   // v[0..3] summed over the CTA (256 threads), result on thread 0
  __shared__ double red[4][8];
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    double x = v[a];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
    if ((threadIdx.x & 31) == 0) red[a][threadIdx.x >> 5] = x;
  }
  __syncthreads();
  if (threadIdx.x == 0)
    for (int a = 0; a < 4; ++a) {
      double x = 0.0;
      for (int w = 0; w < 8; ++w) x += red[a][w];
      v[a] = x;
    }
  __syncthreads();
}
// real space: out[4 i + 0] = Σ_{j,R}' Z_i Z_j erfc(η d)/d,  out[4 i + 1..3] = reduced-coordinate force on atom i
__global__ void __launch_bounds__(256)
k_ewald_real(EwaldGeom g, const double* __restrict__ Z, const double* __restrict__ pos, double* __restrict__ out) {
  const int i = blockIdx.x;
  const int nr0 = 2 * g.rlim[0] + 1, nr1 = 2 * g.rlim[1] + 1, nr2 = 2 * g.rlim[2] + 1;
  const long long nR = (long long)nr0 * nr1 * nr2, total = nR * g.n_atoms;
  const double pix = pos[3 * i], piy = pos[3 * i + 1], piz = pos[3 * i + 2], zi = Z[i];
  double acc[4] = {0.0, 0.0, 0.0, 0.0};     // energy, cartesian Σ dE/dist * Δr
  for (long long t = threadIdx.x; t < total; t += blockDim.x) {
    const int j = (int)(t / nR);
    const long long r = t % nR;
    const int r0 = (int)(r % nr0) - g.rlim[0], r1 = (int)((r / nr0) % nr1) - g.rlim[1], r2 = (int)(r / ((long long)nr0 * nr1)) - g.rlim[2];
    if (j == i && r0 == 0 && r1 == 0 && r2 == 0) continue;
    const double f0 = pix - pos[3 * j] - r0, f1 = piy - pos[3 * j + 1] - r1, f2 = piz - pos[3 * j + 2] - r2;   // Δr reduced
    const double dx = g.lat[0] * f0 + g.lat[1] * f1 + g.lat[2] * f2, dy = g.lat[3] * f0 + g.lat[4] * f1 + g.lat[5] * f2,
                 dz = g.lat[6] * f0 + g.lat[7] * f1 + g.lat[8] * f2;
    const double d2 = dx * dx + dy * dy + dz * dz, d = sqrt(d2);
    const double zz = zi * Z[j];
    const double e = zz * erfc(g.eta * d) / d;
    const double dE = (zz * g.eta * (-2.0 * exp(-g.eta * g.eta * d2) * 0.5641895835477563) - e) / d;   // 1/sqrt(pi)
    acc[0] += e;
    const double s = dE / d;
    acc[1] += s * dx;
    acc[2] += s * dy;
    acc[3] += s * dz;
  }
  ewald_block_sum4(acc);
  if (threadIdx.x == 0) {
    out[4 * i] = acc[0];
    // F_red = -(lattice' * cartesian sum)
    out[4 * i + 1] = -(g.lat[0] * acc[1] + g.lat[3] * acc[2] + g.lat[6] * acc[3]);
    out[4 * i + 2] = -(g.lat[1] * acc[1] + g.lat[4] * acc[2] + g.lat[7] * acc[3]);
    out[4 * i + 3] = -(g.lat[2] * acc[1] + g.lat[5] * acc[2] + g.lat[8] * acc[3]);
  }
}
// structure factor and damping per G (G = 0 excluded: damp = 0): sf[4 t] = cos sum, sin sum, damp, -
__global__ void __launch_bounds__(256)
k_ewald_structure(EwaldGeom g, const double* __restrict__ Z, const double* __restrict__ pos, double* __restrict__ sf) {
  const int n0 = 2 * g.glim[0] + 1, n1 = 2 * g.glim[1] + 1, n2 = 2 * g.glim[2] + 1;
  const long long nG = (long long)n0 * n1 * n2;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nG) return;
  const int g0 = (int)(t % n0) - g.glim[0], g1 = (int)((t / n0) % n1) - g.glim[1], g2 = (int)(t / ((long long)n0 * n1)) - g.glim[2];
  double cs = 0.0, sn = 0.0;
  for (int j = 0; j < g.n_atoms; ++j) {
    double s, c;
    sincospi(2.0 * (g0 * pos[3 * j] + g1 * pos[3 * j + 1] + g2 * pos[3 * j + 2]), &s, &c);
    cs += Z[j] * c;
    sn += Z[j] * s;
  }
  const double gx = g.recip[0] * g0 + g.recip[1] * g1 + g.recip[2] * g2, gy = g.recip[3] * g0 + g.recip[4] * g1 + g.recip[5] * g2,
               gz = g.recip[6] * g0 + g.recip[7] * g1 + g.recip[8] * g2;
  const double G2 = gx * gx + gy * gy + gz * gz;
  sf[4 * t] = cs;
  sf[4 * t + 1] = sn;
  sf[4 * t + 2] = (g0 == 0 && g1 == 0 && g2 == 0) ? 0.0 : exp(-G2 / (4.0 * g.eta * g.eta)) / G2;
  sf[4 * t + 3] = 0.0;
}
// reciprocal space: block 0..n_atoms-1: forces on atom i (out[4 i + 1..3]); block n_atoms: energy Σ_G |S|² damp (out[4 n_atoms])
__global__ void __launch_bounds__(256)
k_ewald_recip(EwaldGeom g, const double* __restrict__ Z, const double* __restrict__ pos, const double* __restrict__ sf,
              double* __restrict__ out) {
  const int i = blockIdx.x;
  const int n0 = 2 * g.glim[0] + 1, n1 = 2 * g.glim[1] + 1, n2 = 2 * g.glim[2] + 1;
  const long long nG = (long long)n0 * n1 * n2;
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  if (i == g.n_atoms) {
    for (long long t = threadIdx.x; t < nG; t += blockDim.x)
      acc[0] += (sf[4 * t] * sf[4 * t] + sf[4 * t + 1] * sf[4 * t + 1]) * sf[4 * t + 2];
  } else {
    const double p0 = pos[3 * i], p1 = pos[3 * i + 1], p2 = pos[3 * i + 2], zi = Z[i];
    for (long long t = threadIdx.x; t < nG; t += blockDim.x) {
      const int g0 = (int)(t % n0) - g.glim[0], g1 = (int)((t / n0) % n1) - g.glim[1], g2 = (int)(t / ((long long)n0 * n1)) - g.glim[2];
      double s, c;
      sincospi(2.0 * (g0 * p0 + g1 * p1 + g2 * p2), &s, &c);
      const double coeff = zi * 6.283185307179586 * (-sf[4 * t] * s + sf[4 * t + 1] * c) * sf[4 * t + 2];
      acc[1] -= coeff * g0;
      acc[2] -= coeff * g1;
      acc[3] -= coeff * g2;
    }
  }
  ewald_block_sum4(acc);
  if (threadIdx.x == 0) {
    out[4 * i] = acc[0];
    out[4 * i + 1] = acc[1];
    out[4 * i + 2] = acc[2];
    out[4 * i + 3] = acc[3];
  }
}

void ewald(dftk_b200_ctx* ctx, const double* lattice_colmajor, int n_atoms, const double* charges, const double* positions,
           double eta, const int* glims, const int* rlims, double* energy_host, double* forces_host) {
  EwaldGeom g;
  // lattice_colmajor[3*c + r] = component r of lattice vector c  ->  lat[3*r + c]
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) g.lat[3 * r + c] = lattice_colmajor[3 * c + r];
  // recip = 2π inv(lat)': recip[3*r + c] = 2π inv(lat)[c][r]
  const double* a = g.lat;
  const double det = a[0] * (a[4] * a[8] - a[5] * a[7]) - a[1] * (a[3] * a[8] - a[5] * a[6]) + a[2] * (a[3] * a[7] - a[4] * a[6]);
  REQUIRE(det != 0.0 && n_atoms >= 1 && eta > 0.0, "ewald: bad lattice / atoms / eta");
  double inv[9] = {(a[4] * a[8] - a[5] * a[7]) / det, (a[2] * a[7] - a[1] * a[8]) / det, (a[1] * a[5] - a[2] * a[4]) / det,
                   (a[5] * a[6] - a[3] * a[8]) / det, (a[0] * a[8] - a[2] * a[6]) / det, (a[2] * a[3] - a[0] * a[5]) / det,
                   (a[3] * a[7] - a[4] * a[6]) / det, (a[1] * a[6] - a[0] * a[7]) / det, (a[0] * a[4] - a[1] * a[3]) / det};
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) g.recip[3 * r + c] = 6.283185307179586 * inv[3 * c + r];
  g.eta = eta;
  g.vol = std::fabs(det);
  g.n_atoms = n_atoms;
  for (int q = 0; q < 3; ++q) {
    g.glim[q] = glims[q];
    g.rlim[q] = rlims[q];
    REQUIRE(glims[q] >= 0 && rlims[q] >= 0 && glims[q] < 2048 && rlims[q] < 2048, "ewald: bad summation limits");
  }
  const long long nG = (long long)(2 * g.glim[0] + 1) * (2 * g.glim[1] + 1) * (2 * g.glim[2] + 1);
  double* d = ctx->sym_d.ensure((size_t)4 * n_atoms + 4 * (n_atoms + 1) + 4 * (n_atoms + 1) + 4 * nG + 16);
  double* dZ = d;
  double* dpos = d + n_atoms;
  double* dreal = d + 4 * n_atoms;
  double* drec = dreal + 4 * (n_atoms + 1);
  double* dsf = drec + 4 * (n_atoms + 1);
  CUDA_CHECK(cudaMemcpyAsync(dZ, charges, n_atoms * sizeof(double), cudaMemcpyDefault, ctx->stream));
  CUDA_CHECK(cudaMemcpyAsync(dpos, positions, 3 * n_atoms * sizeof(double), cudaMemcpyDefault, ctx->stream));
  LAUNCH(ctx, k_ewald_real, (unsigned)n_atoms, 256, 0, g, (const double*)dZ, (const double*)dpos, dreal);
  LAUNCH(ctx, k_ewald_structure, (unsigned)((nG + 255) / 256), 256, 0, g, (const double*)dZ, (const double*)dpos, dsf);
  LAUNCH(ctx, k_ewald_recip, (unsigned)(n_atoms + 1), 256, 0, g, (const double*)dZ, (const double*)dpos, (const double*)dsf, drec);
  std::vector<double> hr(4 * (n_atoms + 1)), hk(4 * (n_atoms + 1));
  CUDA_CHECK(cudaMemcpyAsync(hr.data(), dreal, 4 * n_atoms * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_CHECK(cudaMemcpyAsync(hk.data(), drec, 4 * (n_atoms + 1) * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  double ztot = 0.0, z2 = 0.0, sum_real = 0.0;
  for (int i = 0; i < n_atoms; ++i) {
    ztot += charges[i];
    z2 += charges[i] * charges[i];
    sum_real += hr[4 * i];
  }
  const double pref = 4.0 * FORCES_PI / g.vol;
  const double sum_recip = (-(ztot * ztot) / (4.0 * eta * eta) + hk[4 * n_atoms]) * pref;
  sum_real += -2.0 * eta / std::sqrt(FORCES_PI) * z2;
  if (energy_host) *energy_host = (sum_recip + sum_real) / 2.0;
  if (forces_host)
    for (int i = 0; i < n_atoms; ++i)
      for (int c = 0; c < 3; ++c) forces_host[3 * i + c] = pref * hk[4 * i + 1 + c] + hr[4 * i + 1 + c];
}

void local_forces(dftk_b200_grid* g, const cplx* w, int n_atoms, const double* pos_host, double* out_host) {
  dftk_b200_ctx* ctx = g->ctx;
  if (n_atoms == 0) return;
  int n_blocks = std::max(1, (4 * ctx->sm_count + n_atoms - 1) / n_atoms);
  n_blocks = (int)std::min<int64_t>(n_blocks, (g->N + 255) / 256);
  double* d = ctx->sym_d.ensure((size_t)3 * n_atoms * (2 + n_blocks));
  double* d_pos = d;
  double* d_out = d + 3 * n_atoms;
  double* d_part = d + 6 * n_atoms;
  CUDA_CHECK(cudaMemcpyAsync(d_pos, pos_host, (size_t)3 * n_atoms * sizeof(double), cudaMemcpyDefault, ctx->stream));
  for (int a0 = 0; a0 < n_atoms; a0 += 65535) {     // gridDim.y limit
    const int na = std::min(65535, n_atoms - a0);
    LAUNCH(ctx, k_local_forces, dim3((unsigned)n_blocks, (unsigned)na), 256, 0, g->nx, g->ny, g->nz, w,
           (const double*)(d_pos + 3 * a0), d_part + (size_t)3 * a0 * n_blocks);
  }
  LAUNCH(ctx, k_local_forces_reduce, (unsigned)((3 * n_atoms + 127) / 128), 128, 0, (const double*)d_part, n_atoms,
         n_blocks, d_out);
  CUDA_CHECK(cudaMemcpyAsync(out_host, d_out, (size_t)3 * n_atoms * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
}

void kb_nonlocal_force_rows(dftk_b200_kblock* kb, const cplx* psi, const double* occ_w_host, int64_t n_bands,
                            const double* gpk, double* out_host) {
  dftk_b200_ctx* ctx = kb->grid->ctx;
  const int64_t np = kb->n_proj, n_pw = kb->n_pw;
  for (int64_t i = 0; i < 3 * np; ++i) out_host[i] = 0.0;
  if (np == 0 || n_bands == 0) return;
  REQUIRE(n_pw <= (int64_t)2147483647 * 256, "nonlocal forces: n_pw too large");
  // bands in chunks so that the three scaled copies of psi stay within 1 GiB of scratch
  const int64_t chunk = std::max<int64_t>(1, std::min<int64_t>(std::min<int64_t>(n_bands, 65535),
                                                               ((int64_t)1 << 30) / (3 * n_pw * (int64_t)sizeof(cplx))));
  cplx* scaled = kb->W1.ensure((size_t)3 * n_pw * chunk);
  cplx* proj = kb->proj.ensure((size_t)5 * np * chunk);     // P'psi | D P'psi | P'(p_α psi) α = 0..2
  cplx* dproj = proj + (size_t)np * chunk;
  cplx* pa = proj + (size_t)2 * np * chunk;
  DescRing& ring = ctx->slot[0].ring;
  const double* w_dev = (const double*)ring.put(occ_w_host, (size_t)n_bands * sizeof(double), ctx->stream);
  double* f = ctx->scal.ensure((size_t)3 * np + 8);
  CUDA_CHECK(cudaMemsetAsync(f, 0, (size_t)3 * np * sizeof(double), ctx->stream));
  const cplx one = make_double2(1.0, 0.0), zero = make_double2(0.0, 0.0);
  for (int64_t b0 = 0; b0 < n_bands; b0 += chunk) {
    const int64_t nb = std::min(chunk, n_bands - b0);
    const cplx* p = psi + (size_t)b0 * n_pw;
    LAUNCH(ctx, k_scale_by_momentum, dim3((unsigned)((n_pw + 255) / 256), (unsigned)nb, 3), 256, 0, n_pw, nb, gpk, p,
           n_pw, scaled);
    zgemm(ctx, 2, np, nb, n_pw, one, kb->P.p, n_pw, p, n_pw, zero, proj, np);
    zgemm(ctx, 0, np, nb, np, one, kb->Dc.p, np, proj, np, zero, dproj, np);
    zgemm(ctx, 2, np, 3 * nb, n_pw, one, kb->P.p, n_pw, scaled, n_pw, zero, pa, np);
    LAUNCH(ctx, k_nonlocal_force_rows, dim3((unsigned)((np + 127) / 128), 3), 128, 0, np, nb, (const cplx*)dproj,
           (const cplx*)pa, w_dev + b0, f);
  }
  CUDA_CHECK(cudaMemcpyAsync(out_host, f, (size_t)3 * np * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  ring.rewind();
}

}  // namespace dftk
