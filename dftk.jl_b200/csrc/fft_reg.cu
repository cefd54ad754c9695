// __global__ wrappers + dispatch table of the register two-pass FFT engine (fft_reg.cuh).
// Compiled several times with -DREG_GROUP=g (g = 0..REG_NGROUPS-1); each translation unit instantiates
// the factor pairs with (pair index % REG_NGROUPS) == g so that the build parallelises.
#include "structs.cuh"
#include "fft_reg.cuh"

#ifndef REG_GROUP
#define REG_GROUP 0
#endif
#ifndef REG_NGROUPS
#define REG_NGROUPS 1
#endif

namespace dftk {

extern __shared__ __align__(16) unsigned char dyn_smem_reg[];
#define REG_MAXT(A, B) (32 * ((A) > (B) ? (A) : (B)))

// XM: W1 layout, 0 = [col][x], 1 = [x][col] (fused y-z path)
template <int A, int B, int XM>
__global__ void __launch_bounds__(REG_MAXT(A, B))
kr_sphere_to_x(SphereTablesX T, const cplx* tw, const cplx* psi, int64_t ldpsi, cplx* W1, int L, int Lp) {
  reg_sphere_to_x<A, B, XM>(T, tw, psi, ldpsi, W1, L, Lp, (cplx*)dyn_smem_reg, Dim3i{(int)blockIdx.x, (int)blockIdx.y, 0});
}
template <int A, int B>
__global__ void __launch_bounds__(REG_MAXT(A, B))
kr_y_backward(SphereTablesX T, const cplx* tw, const cplx* W1, cplx* W2, int L, int Lp) {
  reg_y_backward<A, B>(T, tw, W1, W2, L, Lp, (cplx*)dyn_smem_reg, Dim3i{(int)blockIdx.x, (int)blockIdx.y, (int)blockIdx.z});
}
template <int A, int B>
__global__ void __launch_bounds__(REG_MAXT(A, B))
kr_z_apply(SphereTablesX T, const cplx* tw, cplx* W2, const double* V, int L, int Lp) {
  reg_z_apply_potential<A, B>(T, tw, W2, V, L, Lp, (cplx*)dyn_smem_reg, Dim3i{(int)blockIdx.x, (int)blockIdx.y, (int)blockIdx.z});
}
template <int A, int B>
__global__ void __launch_bounds__(REG_MAXT(A, B))
kr_z_apply_pipe(SphereTablesX T, const cplx* tw, cplx* W2, const double* V, int n_bands) {
  reg_z_apply_potential_pipe<A, B>(T, tw, W2, V, (cplx*)dyn_smem_reg, n_bands);
}
template <int A, int B>
__global__ void __launch_bounds__(REG_MAXT(A, B))
kr_z_to_cube(SphereTablesX T, const cplx* tw, const cplx* W2, cplx* cube, double scale, int L, int Lp) {
  reg_z_to_cube<A, B>(T, tw, W2, cube, scale, L, Lp, (cplx*)dyn_smem_reg, Dim3i{(int)blockIdx.x, (int)blockIdx.y, (int)blockIdx.z});
}
template <int A, int B>
__global__ void __launch_bounds__(REG_MAXT(A, B))
kr_z_from_cube(SphereTablesX T, const cplx* tw, const cplx* cube, cplx* W2, int L, int Lp) {
  reg_z_from_cube<A, B>(T, tw, cube, W2, L, Lp, (cplx*)dyn_smem_reg, Dim3i{(int)blockIdx.x, (int)blockIdx.y, (int)blockIdx.z});
}
template <int A, int B>
__global__ void __launch_bounds__(REG_MAXT(A, B))
kr_z_density(SphereTablesX T, const cplx* tw, const cplx* W2, const double* wts, int nb, double* rho, int L, int Lp) {
  reg_z_density<A, B>(T, tw, W2, wts, nb, rho, L, Lp, (cplx*)dyn_smem_reg, Dim3i{(int)blockIdx.x, (int)blockIdx.y, 0});
}
template <int A, int B>
__global__ void __launch_bounds__(REG_MAXT(A, B))
kr_y_forward(SphereTablesX T, const cplx* tw, const cplx* W2, cplx* W1, int L, int Lp) {
  reg_y_forward<A, B>(T, tw, W2, W1, L, Lp, (cplx*)dyn_smem_reg, Dim3i{(int)blockIdx.x, (int)blockIdx.y, (int)blockIdx.z});
}
template <int A, int B, int XM>
__global__ void __launch_bounds__(REG_MAXT(A, B))
kr_x_to_sphere(SphereTablesX T, const cplx* tw, const cplx* W1, cplx* out, int64_t ldout, double scale,
               const double* kin, const cplx* psi, int64_t ldpsi, int accumulate, int L, int Lp) {
  reg_x_to_sphere<A, B, XM>(T, tw, W1, out, ldout, scale, kin, psi, ldpsi, accumulate, L, Lp, (cplx*)dyn_smem_reg,
                        Dim3i{(int)blockIdx.x, (int)blockIdx.y, 0});
}
// fused y and z passes of the local H apply (ny == nz): persistent CTAs over the items (band, x line) of nb bands, item
// i = x * nb + band, so that the CTAs in flight share a few x lines and their Vt planes stay in L2.  No CTA barrier
// between items: a group goes on to the next item's y backward as soon as it has finished this one's y forward.
template <int A, int B>
__global__ void __launch_bounds__(RegYZ<A, B>::NT, 1)
kr_yz_apply(SphereTablesX T, const cplx* tw, cplx* W1t, const double* Vt, int nb) {
  const int n_items = nb * T.nx;
  for (int i = blockIdx.x; i < n_items; i += gridDim.x)
    reg_yz_apply<A, B>(T, tw, W1t, Vt, (cplx*)dyn_smem_reg, Dim3i{i / nb, 0, i % nb});
}

// ---- the same five H-apply stages for MANY k-blocks in one launch (batched small-matrix LOBPCG, lobpcg.cu): the band
//      index of the grid runs over the bands of all blocks; `bandmap[band] = {item, band within the item}`.  Blocks of
//      one basis share the FFT grid (same factor pair, same shared-memory size); only the pruning tables differ.
template <int A, int B>
__global__ void __launch_bounds__(REG_MAXT(A, B))
kr_sphere_to_x_multi(const FftMultiItem* __restrict__ items, const int2* __restrict__ bandmap, const cplx* tw, int L, int Lp) {
  const int2 bm = bandmap[blockIdx.y];
  const FftMultiItem& it = items[bm.x];
  if ((int)blockIdx.x * L >= it.T.n_cols) return;
  reg_sphere_to_x<A, B>(it.T, tw, it.psi, it.ldpsi, it.W1, L, Lp, (cplx*)dyn_smem_reg, Dim3i{(int)blockIdx.x, bm.y, 0});
}
template <int A, int B>
__global__ void __launch_bounds__(REG_MAXT(A, B))
kr_y_backward_multi(const FftMultiItem* __restrict__ items, const int2* __restrict__ bandmap, const cplx* tw, int L, int Lp) {
  const int2 bm = bandmap[blockIdx.z];
  const FftMultiItem& it = items[bm.x];
  if ((int)blockIdx.y >= it.T.n_zc) return;
  reg_y_backward<A, B>(it.T, tw, it.W1, it.W2, L, Lp, (cplx*)dyn_smem_reg, Dim3i{(int)blockIdx.x, (int)blockIdx.y, bm.y});
}
template <int A, int B>
__global__ void __launch_bounds__(REG_MAXT(A, B))
kr_z_apply_multi(const FftMultiItem* __restrict__ items, const int2* __restrict__ bandmap, const cplx* tw, int L, int Lp) {
  const int2 bm = bandmap[blockIdx.z];
  const FftMultiItem& it = items[bm.x];
  reg_z_apply_potential<A, B>(it.T, tw, it.W2, it.V, L, Lp, (cplx*)dyn_smem_reg, Dim3i{(int)blockIdx.x, (int)blockIdx.y, bm.y});
}
template <int A, int B>
__global__ void __launch_bounds__(REG_MAXT(A, B))
kr_y_forward_multi(const FftMultiItem* __restrict__ items, const int2* __restrict__ bandmap, const cplx* tw, int L, int Lp) {
  const int2 bm = bandmap[blockIdx.z];
  const FftMultiItem& it = items[bm.x];
  if ((int)blockIdx.y >= it.T.n_zc) return;
  reg_y_forward<A, B>(it.T, tw, it.W2, it.W1, L, Lp, (cplx*)dyn_smem_reg, Dim3i{(int)blockIdx.x, (int)blockIdx.y, bm.y});
}
template <int A, int B>
__global__ void __launch_bounds__(REG_MAXT(A, B))
kr_x_to_sphere_multi(const FftMultiItem* __restrict__ items, const int2* __restrict__ bandmap, const cplx* tw, int L, int Lp) {
  const int2 bm = bandmap[blockIdx.y];
  const FftMultiItem& it = items[bm.x];
  if ((int)blockIdx.x * L >= it.T.n_cols) return;
  reg_x_to_sphere<A, B>(it.T, tw, it.W1, it.out, it.ldout, 1.0, it.kin, it.psi, it.ldpsi, 0, L, Lp, (cplx*)dyn_smem_reg,
                        Dim3i{(int)blockIdx.x, bm.y, 0});
}

// density of all k-blocks of one spin channel: the CTA of a (y, x-tile) accumulates the bands of block after block
// (single writer per density element, fixed order: deterministic)
template <int A, int B>
__global__ void __launch_bounds__(REG_MAXT(A, B))
kr_z_density_multi(const FftMultiItem* __restrict__ items, int n_items, int spin, const cplx* tw, double* rho, int L, int Lp) {
  for (int i = 0; i < n_items; ++i) {
    const FftMultiItem& it = items[i];
    if ((int)(intptr_t)it.kin != spin) continue;
    reg_z_density<A, B>(it.T, tw, it.W2, it.wts, it.nb, rho, L, Lp, (cplx*)dyn_smem_reg, Dim3i{(int)blockIdx.x, (int)blockIdx.y, 0});
    __syncthreads();
  }
}

template <int A, int B>
static RegKernels make_entry() {
  RegKernels k;
  k.A = A;
  k.B = B;
  k.T = RegPair<A, B>::T;
  k.yz_threads = RegYZ<A, B>::NT;
  k.sphere_to_x = (const void*)kr_sphere_to_x<A, B, 0>;
  k.sphere_to_xt = (const void*)kr_sphere_to_x<A, B, 1>;
  k.y_backward = (const void*)kr_y_backward<A, B>;
  k.z_apply = (const void*)kr_z_apply<A, B>;
  k.z_apply_pipe = (const void*)kr_z_apply_pipe<A, B>;
  k.z_to_cube = (const void*)kr_z_to_cube<A, B>;
  k.z_from_cube = (const void*)kr_z_from_cube<A, B>;
  k.z_density = (const void*)kr_z_density<A, B>;
  k.y_forward = (const void*)kr_y_forward<A, B>;
  k.x_to_sphere = (const void*)kr_x_to_sphere<A, B, 0>;
  k.xt_to_sphere = (const void*)kr_x_to_sphere<A, B, 1>;
  k.yz_apply = (const void*)kr_yz_apply<A, B>;
  k.m_sphere_to_x = (const void*)kr_sphere_to_x_multi<A, B>;
  k.m_y_backward = (const void*)kr_y_backward_multi<A, B>;
  k.m_z_apply = (const void*)kr_z_apply_multi<A, B>;
  k.m_y_forward = (const void*)kr_y_forward_multi<A, B>;
  k.m_x_to_sphere = (const void*)kr_x_to_sphere_multi<A, B>;
  k.m_z_density = (const void*)kr_z_density_multi<A, B>;
  return k;
}

#define REG_CONCAT2(a, b) a##b
#define REG_CONCAT(a, b) REG_CONCAT2(a, b)
void REG_CONCAT(reg_register_group_, REG_GROUP)(std::vector<RegKernels>& out) {
  int idx = 0;
#define DFTK_X(a, b)                                          \
  if ((idx++ % REG_NGROUPS) == REG_GROUP) out.push_back(make_entry<a, b>());
  DFTK_REG_PAIRS(DFTK_X)
#undef DFTK_X
}

}  // namespace dftk
