// Host emulation of the FFT pipeline kernel bodies (TEST INFRASTRUCTURE ONLY, never loaded by the
// product).  Runs the same __host__ __device__ stage bodies as the CUDA kernels, block by block and
// "thread" by "thread", so the index logic can be validated against NumPy without a GPU.
#include <vector>
#include <cstring>
#include "../../dftk.jl_b200/csrc/fft_plan.h"
using namespace dftk;

static SphereTables view(const SphereTablesHost& H) {
  SphereTables T;
  T.nx = H.nx; T.ny = H.ny; T.nz = H.nz; T.n_pw = H.n_pw; T.n_cols = H.n_cols; T.cnt_max = H.cnt_max;
  T.n_zc = H.n_zc; T.col_start = H.col_start.data(); T.col_cnt = H.col_cnt.data();
  T.slot_ix = H.slot_ix.data(); T.slot_src = H.slot_src.data(); T.zlist = H.zlist.data();
  T.colmap = H.colmap.data();
  return T;
}
struct Emu {
  SphereTablesHost H; SphereTables T; FftPlan px, py, pz; std::vector<double> twx, twy, twz;
  int Lx, Ly, Lz; std::vector<cplx> W1, W2, sm;
  Emu(int nx, int ny, int nz, int64_t n_pw, const int64_t* mapping, int nb) {
    H = build_sphere_tables(nx, ny, nz, n_pw, mapping); T = view(H);
    px = make_plan(nx); py = make_plan(ny); pz = make_plan(nz);
    twx = make_twiddles(nx); twy = make_twiddles(ny); twz = make_twiddles(nz);
    Lx = choose_lines(nx); Ly = choose_lines(ny); Lz = choose_lines(nz);
    W1.resize((size_t)nb * H.n_cols * nx); W2.resize((size_t)nb * H.n_zc * ny * nx);
    size_t m = std::max(std::max(nx, ny), nz);
    sm.resize(3 * m * 17 + 64);
  }
  const cplx* tx() { return (const cplx*)twx.data(); }
  const cplx* ty() { return (const cplx*)twy.data(); }
  const cplx* tz() { return (const cplx*)twz.data(); }
  void to_planes(const cplx* psi, int nb) {
    int L = Lx, Lp = L | 1;
    for (int b = 0; b < nb; ++b) for (int bx = 0; bx < (T.n_cols + L - 1) / L; ++bx)
      stage_sphere_to_x(T, px, tx(), psi, T.n_pw, W1.data(), L, Lp, sm.data(), Dim3i{bx, b, 0});
    L = Ly; Lp = L | 1;
    for (int b = 0; b < nb; ++b) for (int z = 0; z < T.n_zc; ++z) for (int bx = 0; bx < (T.nx + L - 1) / L; ++bx)
      stage_y_backward(T, py, ty(), W1.data(), W2.data(), L, Lp, sm.data(), Dim3i{bx, z, b});
  }
  void from_planes(cplx* out, int nb, double scale, const double* kin, const cplx* psi, int acc) {
    int L = Ly, Lp = L | 1;
    for (int b = 0; b < nb; ++b) for (int z = 0; z < T.n_zc; ++z) for (int bx = 0; bx < (T.nx + L - 1) / L; ++bx)
      stage_y_forward(T, py, ty(), W2.data(), W1.data(), L, Lp, sm.data(), Dim3i{bx, z, b});
    L = Lx; Lp = L | 1;
    for (int b = 0; b < nb; ++b) for (int bx = 0; bx < (T.n_cols + L - 1) / L; ++bx)
      stage_x_to_sphere(T, px, tx(), W1.data(), out, T.n_pw, scale, kin, psi, T.n_pw, acc, L, Lp, sm.data(), Dim3i{bx, b, 0});
  }
};

extern "C" {
int emu_apply_local(int nx, int ny, int nz, int64_t n_pw, const int64_t* mapping, const double* psi,
                    int nb, const double* Vscaled, const double* kin, double* out) {
  Emu e(nx, ny, nz, n_pw, mapping, nb);
  e.to_planes((const cplx*)psi, nb);
  int L = e.Lz, Lp = L | 1;
  for (int b = 0; b < nb; ++b) for (int y = 0; y < ny; ++y) for (int bx = 0; bx < (nx + L - 1) / L; ++bx)
    stage_z_apply_potential(e.T, e.pz, e.tz(), e.W2.data(), Vscaled, L, Lp, e.sm.data(), Dim3i{bx, y, b});
  e.from_planes((cplx*)out, nb, 1.0, kin, (const cplx*)psi, 0);
  return 0;
}
int emu_sphere_to_real(int nx, int ny, int nz, int64_t n_pw, const int64_t* mapping, const double* psi,
                       int nb, double scale, double* cube) {
  Emu e(nx, ny, nz, n_pw, mapping, nb);
  e.to_planes((const cplx*)psi, nb);
  int L = e.Lz, Lp = L | 1;
  for (int b = 0; b < nb; ++b) for (int y = 0; y < ny; ++y) for (int bx = 0; bx < (nx + L - 1) / L; ++bx)
    stage_z_to_cube(e.T, e.pz, e.tz(), e.W2.data(), (cplx*)cube, scale, L, Lp, e.sm.data(), Dim3i{bx, y, b});
  return 0;
}
int emu_real_to_sphere(int nx, int ny, int nz, int64_t n_pw, const int64_t* mapping, const double* cube,
                       int nb, double scale, double* out) {
  Emu e(nx, ny, nz, n_pw, mapping, nb);
  int L = e.Lz, Lp = L | 1;
  for (int b = 0; b < nb; ++b) for (int y = 0; y < ny; ++y) for (int bx = 0; bx < (nx + L - 1) / L; ++bx)
    stage_z_from_cube(e.T, e.pz, e.tz(), (const cplx*)cube, e.W2.data(), L, Lp, e.sm.data(), Dim3i{bx, y, b});
  e.from_planes((cplx*)out, nb, scale, nullptr, nullptr, 0);
  return 0;
}
int emu_density(int nx, int ny, int nz, int64_t n_pw, const int64_t* mapping, const double* psi,
                int nb, const double* wts, double* rho) {
  Emu e(nx, ny, nz, n_pw, mapping, nb);
  e.to_planes((const cplx*)psi, nb);
  int L = e.Lz, Lp = L | 1;
  for (int y = 0; y < ny; ++y) for (int bx = 0; bx < (nx + L - 1) / L; ++bx)
    stage_z_density(e.T, e.pz, e.tz(), e.W2.data(), wts, nb, rho, L, Lp, e.sm.data(), Dim3i{bx, y, 0});
  return 0;
}
int emu_fft_cube(int nx, int ny, int nz, double* data, int sign, int batch) {
  FftPlan px = make_plan(nx), py = make_plan(ny), pz = make_plan(nz);
  auto twx = make_twiddles(nx), twy = make_twiddles(ny), twz = make_twiddles(nz);
  size_t m = std::max(std::max(nx, ny), nz);
  std::vector<cplx> sm(2 * m * 17 + 64);
  int L = choose_lines(nx), Lp = L | 1;
  int64_t nl = (int64_t)ny * nz;
  for (int b = 0; b < batch; ++b) for (int bx = 0; bx < (nl + L - 1) / L; ++bx)
    cube_pass_x((cplx*)data, nx, nl, px, (const cplx*)twx.data(), sign, L, Lp, sm.data(), Dim3i{bx, b, 0});
  L = choose_lines(ny); Lp = L | 1;
  for (int b = 0; b < batch; ++b) for (int z = 0; z < nz; ++z) for (int bx = 0; bx < (nx + L - 1) / L; ++bx)
    cube_pass_strided((cplx*)data, nx, ny, nx, (int64_t)nx * ny, (int64_t)nx * ny * nz, py, (const cplx*)twy.data(), sign, L, Lp, sm.data(), Dim3i{bx, z, b});
  L = choose_lines(nz); Lp = L | 1;
  for (int b = 0; b < batch; ++b) for (int y = 0; y < ny; ++y) for (int bx = 0; bx < (nx + L - 1) / L; ++bx)
    cube_pass_strided((cplx*)data, nx, nz, (int64_t)nx * ny, nx, (int64_t)nx * ny * nz, pz, (const cplx*)twz.data(), sign, L, Lp, sm.data(), Dim3i{bx, y, b});
  return 0;
}
}

// ------------------------------------------------------------------------------------------------
// Register two-pass engine (fft_reg.cuh) emulation: every factor pair of the device engine is instantiated on the host,
// so a pair added to DFTK_REG_PAIRS is emulated (and tested) without further edits.
// ------------------------------------------------------------------------------------------------
#include "../../dftk.jl_b200/csrc/fft_reg.cuh"
#define EMU_PAIRS(X) DFTK_REG_PAIRS(X)
static bool emu_pair(int n, int* A, int* B) {
  *A = 0;
#define PX(a, b) if (n == (a) * (b) && *A == 0) { *A = a; *B = b; }
  EMU_PAIRS(PX)
#undef PX
  return *A != 0;
}
#define DISPATCH(n, CALL)                                   \
  do {                                                      \
    int A_, B_;                                             \
    if (!emu_pair(n, &A_, &B_)) return -7;                  \
    bool done_ = false;                                     \
    EMU_PAIRS(CALL)                                         \
    if (!done_) return -8;                                  \
  } while (0)

static bool force_tables = false;
extern "C" void emur_force_tables(int f) { force_tables = f != 0; }
extern "C" int emur_ranges_ok(int nx, int ny, int nz, int64_t n_pw, const int64_t* mapping) {
  return build_sphere_tables(nx, ny, nz, n_pw, mapping).ranges_ok;
}
struct EmuR : Emu {
  SphereTablesX TX;
  EmuR(int nx, int ny, int nz, int64_t n_pw, const int64_t* mapping, int nb) : Emu(nx, ny, nz, n_pw, mapping, nb) {
    static_cast<SphereTables&>(TX) = T;
    TX.zc_of = H.zc_of.data();
    TX.ranges_ok = H.ranges_ok;
    TX.z_s0 = H.z_s0; TX.z_n0 = H.z_n0; TX.z_s1 = H.z_s1; TX.z_n1 = H.z_n1;
    TX.pl_s0 = H.pl_s0.data(); TX.pl_n0 = H.pl_n0.data(); TX.pl_s1 = H.pl_s1.data(); TX.pl_n1 = H.pl_n1.data();
    TX.pl_col0 = H.pl_col0.data();
    TX.cx_s0 = H.cx_s0.data(); TX.cx_n0 = H.cx_n0.data(); TX.cx_s1 = H.cx_s1.data(); TX.cx_n1 = H.cx_n1.data();
    sm.resize(4 * (size_t)std::max(std::max(nx, ny), nz) * 33 + 64);
  }
  static int Lof(int A, int B) { int T = A > B ? A : B; return T >= 12 ? 8 : (T >= 5 ? 16 : 32); }
  int to_planes(const cplx* psi, int nb) {
    if (!H.ranges_ok) return -9;   // the product falls back to the generic engine for such k-blocks
#define CX(a, b) if (A_ == a && B_ == b) { int L = Lof(a, b), Lp = L + 1; done_ = true; \
    for (int bb = 0; bb < nb; ++bb) for (int bx = 0; bx < (T.n_cols + L - 1) / L; ++bx) \
      reg_sphere_to_x<a, b>(TX, tx(), psi, T.n_pw, W1.data(), L, Lp, sm.data(), Dim3i{bx, bb, 0}); }
    DISPATCH(T.nx, CX);
#undef CX
#define CY(a, b) if (A_ == a && B_ == b) { int L = Lof(a, b), Lp = L + 1; done_ = true; \
    for (int bb = 0; bb < nb; ++bb) for (int z = 0; z < T.n_zc; ++z) for (int bx = 0; bx < (T.nx + L - 1) / L; ++bx) \
      reg_y_backward<a, b>(TX, ty(), W1.data(), W2.data(), L, Lp, sm.data(), Dim3i{bx, z, bb}); }
    DISPATCH(T.ny, CY);
#undef CY
    return 0;
  }
  int from_planes(cplx* out, int nb, double scale, const double* kin, const cplx* psi, int acc) {
#define CY(a, b) if (A_ == a && B_ == b) { int L = Lof(a, b), Lp = L + 1; done_ = true; \
    for (int bb = 0; bb < nb; ++bb) for (int z = 0; z < T.n_zc; ++z) for (int bx = 0; bx < (T.nx + L - 1) / L; ++bx) \
      reg_y_forward<a, b>(TX, ty(), W2.data(), W1.data(), L, Lp, sm.data(), Dim3i{bx, z, bb}); }
    DISPATCH(T.ny, CY);
#undef CY
#define CX(a, b) if (A_ == a && B_ == b) { int L = Lof(a, b), Lp = L + 1; done_ = true; \
    for (int bb = 0; bb < nb; ++bb) for (int bx = 0; bx < (T.n_cols + L - 1) / L; ++bx) \
      reg_x_to_sphere<a, b>(TX, tx(), W1.data(), out, T.n_pw, scale, kin, psi, T.n_pw, acc, L, Lp, sm.data(), Dim3i{bx, bb, 0}); }
    DISPATCH(T.nx, CX);
#undef CX
    return 0;
  }
};

extern "C" {
int emur_apply_local(int nx, int ny, int nz, int64_t n_pw, const int64_t* mapping, const double* psi, int nb,
                     const double* Vscaled, const double* kin, double* out) {
  EmuR e(nx, ny, nz, n_pw, mapping, nb);
  int rc = e.to_planes((const cplx*)psi, nb);
  if (rc) return rc;
#define CZ(a, b) if (A_ == a && B_ == b) { int L = EmuR::Lof(a, b), Lp = L + 1; done_ = true; \
  for (int bb = 0; bb < nb; ++bb) for (int y = 0; y < ny; ++y) for (int bx = 0; bx < (nx + L - 1) / L; ++bx) \
    reg_z_apply_potential<a, b>(e.TX, e.tz(), e.W2.data(), Vscaled, L, Lp, e.sm.data(), Dim3i{bx, y, bb}); }
  DISPATCH(nz, CZ);
#undef CZ
  return e.from_planes((cplx*)out, nb, 1.0, kin, (const cplx*)psi, 0);
}
int emur_sphere_to_real(int nx, int ny, int nz, int64_t n_pw, const int64_t* mapping, const double* psi, int nb,
                        double scale, double* cube) {
  EmuR e(nx, ny, nz, n_pw, mapping, nb);
  int rc = e.to_planes((const cplx*)psi, nb);
  if (rc) return rc;
#define CZ(a, b) if (A_ == a && B_ == b) { int L = EmuR::Lof(a, b), Lp = L + 1; done_ = true; \
  for (int bb = 0; bb < nb; ++bb) for (int y = 0; y < ny; ++y) for (int bx = 0; bx < (nx + L - 1) / L; ++bx) \
    reg_z_to_cube<a, b>(e.TX, e.tz(), e.W2.data(), (cplx*)cube, scale, L, Lp, e.sm.data(), Dim3i{bx, y, bb}); }
  DISPATCH(nz, CZ);
#undef CZ
  return 0;
}
int emur_real_to_sphere(int nx, int ny, int nz, int64_t n_pw, const int64_t* mapping, const double* cube, int nb,
                        double scale, double* out) {
  EmuR e(nx, ny, nz, n_pw, mapping, nb);
  if (!e.H.ranges_ok) return -9;
#define CZ(a, b) if (A_ == a && B_ == b) { int L = EmuR::Lof(a, b), Lp = L + 1; done_ = true; \
  for (int bb = 0; bb < nb; ++bb) for (int y = 0; y < ny; ++y) for (int bx = 0; bx < (nx + L - 1) / L; ++bx) \
    reg_z_from_cube<a, b>(e.TX, e.tz(), (const cplx*)cube, e.W2.data(), L, Lp, e.sm.data(), Dim3i{bx, y, bb}); }
  DISPATCH(nz, CZ);
#undef CZ
  return e.from_planes((cplx*)out, nb, scale, nullptr, nullptr, 0);
}
int emur_density(int nx, int ny, int nz, int64_t n_pw, const int64_t* mapping, const double* psi, int nb,
                 const double* wts, double* rho) {
  EmuR e(nx, ny, nz, n_pw, mapping, nb);
  int rc = e.to_planes((const cplx*)psi, nb);
  if (rc) return rc;
#define CZ(a, b) if (A_ == a && B_ == b) { int L = EmuR::Lof(a, b), Lp = L + 1; done_ = true; \
  for (int y = 0; y < ny; ++y) for (int bx = 0; bx < (nx + L - 1) / L; ++bx) \
    reg_z_density<a, b>(e.TX, e.tz(), e.W2.data(), wts, nb, rho, L, Lp, e.sm.data(), Dim3i{bx, y, 0}); }
  DISPATCH(nz, CZ);
#undef CZ
  return 0;
}
}

// ------------------------------------------------------------------------------------------------
// XC functionals and density symmetrisation (xc_core.cuh) on the host
// ------------------------------------------------------------------------------------------------
#include "../../dftk.jl_b200/csrc/xc_core.cuh"
extern "C" {
int emu_xc(int mask, int n_spin, int gga, int64_t N, const double* rho, const double* sigma, double* e, double* vrho,
           double* vsigma) {
  for (int64_t i = 0; i < N; ++i) {
    if (n_spin == 1 && !gga) xc_eval_range<1, false>(mask, i, N, rho, sigma, e, vrho, vsigma);
    else if (n_spin == 2 && !gga) xc_eval_range<2, false>(mask, i, N, rho, sigma, e, vrho, vsigma);
    else if (n_spin == 1 && gga) xc_eval_range<1, true>(mask, i, N, rho, sigma, e, vrho, vsigma);
    else if (n_spin == 2 && gga) xc_eval_range<2, true>(mask, i, N, rho, sigma, e, vrho, vsigma);
    else return -1;
  }
  return 0;
}
int emu_symmetrize(int nx, int ny, int nz, const double* in, double* out, int n_sym, const int* invS, const double* tau) {
  for (int64_t i = 0; i < (int64_t)nx * ny * nz; ++i)
    symmetrize_point(i, nx, ny, nz, (const cplx*)in, (cplx*)out, n_sym, invS, tau);
  return 0;
}
}

// ------------------------------------------------------------------------------------------------
// Force bodies (forces_core.cuh) on the host
// ------------------------------------------------------------------------------------------------
#include "../../dftk.jl_b200/csrc/forces_core.cuh"
extern "C" {
int emu_local_forces(int nx, int ny, int nz, const double* w, int n_atoms, const double* pos, double* out) {
  for (int a = 0; a < n_atoms; ++a) {
    double acc[3] = {0, 0, 0};
    for (int64_t i = 0; i < (int64_t)nx * ny * nz; ++i)
      local_force_point(i, nx, ny, nz, (const cplx*)w, pos[3 * a], pos[3 * a + 1], pos[3 * a + 2], acc);
    for (int c = 0; c < 3; ++c) out[3 * a + c] = -2.0 * FORCES_PI * acc[c];
  }
  return 0;
}
int emu_scale_by_momentum(int64_t n_rows, int64_t nb, const double* gpk, const double* psi, double* out) {
  for (int a = 0; a < 3; ++a)
    for (int64_t b = 0; b < nb; ++b)
      for (int64_t i = 0; i < n_rows; ++i)
        scale_by_momentum_point(i, b, a, n_rows, nb, gpk, (const cplx*)psi, n_rows, (cplx*)out);
  return 0;
}
int emu_nonlocal_force_rows(int64_t np, int64_t nb, const double* dproj, const double* pa, const double* w, double* f) {
  for (int a = 0; a < 3; ++a)
    for (int64_t j = 0; j < np; ++j) nonlocal_force_row(j, a, np, nb, (const cplx*)dproj, (const cplx*)pa, w, f);
  return 0;
}
}

// ------------------------------------------------------------------------------------------------
// Fused small-matrix LOBPCG bodies (lobpcg_small.cuh) on the host
// ------------------------------------------------------------------------------------------------
#include "../../dftk.jl_b200/csrc/lobpcg_small.cuh"
#include <vector>
static SmallMatList emu_list(int nblocks, const double* const* ptrs, const int64_t* lds, const int* cols) {
  SmallMatList L{};
  L.n = nblocks;
  int off = 0;
  for (int i = 0; i < 3; ++i) {
    L.start[i] = off;
    if (i < nblocks) {
      L.p[i] = (const cplx*)ptrs[i];
      L.ld[i] = lds[i];
      L.cols[i] = cols[i];
      off += cols[i];
    }
  }
  L.start[3] = off;
  for (int i = nblocks; i < 4; ++i) L.start[i] = off;
  return L;
}
extern "C" {
int emu_small_gram(int nA, const double* const* pA, const int64_t* ldA, const int* colsA, int nB, const double* const* pB,
                   const int64_t* ldB, const int* colsB, int64_t n_rows, int64_t rows_per_cta, int upper_only, double* C,
                   int64_t ldc) {
  SmallMatList A = emu_list(nA, pA, ldA, colsA), B = emu_list(nB, pB, ldB, colsB);
  const int ta = A.start[A.n], tb = B.start[B.n];
  const int n_ctas = (int)((n_rows + rows_per_cta - 1) / rows_per_cta);
  std::vector<cplx> ws((size_t)n_ctas * ta * tb), sm((size_t)SMALL_TR * (ta + tb));
  for (int c = 0; c < n_ctas; ++c) small_gram_cta(c, rows_per_cta, n_rows, A, B, upper_only, ws.data(), sm.data());
  small_gram_reduce(n_ctas, A, B, upper_only, ws.data(), (cplx*)C, ldc);
  return 0;
}
int emu_small_blocks_times(int nY, const double* const* pY, const int64_t* ldY, const int* colsY, const double* cm,
                           int ldcm, int ncols, double* out, int64_t ldo, int64_t n_rows, double alpha, double beta) {
  SmallMatList Y = emu_list(nY, pY, ldY, colsY);
  for (int64_t r = 0; r < n_rows; ++r) small_blocks_times_row(r, Y, (const cplx*)cm, ldcm, ncols, (cplx*)out, ldo, alpha, beta);
  return 0;
}
int emu_small_rmul(double* X, int64_t ld, int64_t n_rows, int n, const double* invR, int ldr) {
  for (int64_t r = 0; r < n_rows; ++r) small_rmul_row(r, (cplx*)X, ld, n, (const cplx*)invR, ldr);
  return 0;
}
int emu_small_heev(double* G, int64_t ldg, int n, double* w, double* stats) {
  std::vector<cplx> As((size_t)n * n), V((size_t)n * n), rot((size_t)n + 4);
  std::vector<double> red(SMALL_RED);
  std::vector<int> iw((size_t)n + 4);
  small_heev_cta((cplx*)G, ldg, n, w, As.data(), V.data(), rot.data(), red.data(), iw.data(), stats, nullptr, 0);
  return 0;
}
int emu_small_chol(const double* O, int64_t ldo, int n, double* invR, int64_t ldi, double* stats) {
  std::vector<cplx> As((size_t)SMALL_MAX_N * SMALL_MAX_N), Bs((size_t)SMALL_MAX_N * SMALL_MAX_N);
  std::vector<double> red(SMALL_RED);
  int flag[2] = {0, 0};
  small_chol_cta((const cplx*)O, ldo, n, (cplx*)invR, ldi, stats, As.data(), Bs.data(), red.data(), flag);
  return 0;
}
}

// ------------------------------------------------------------------------------------------------
// INT8-emulated FP64 GEMM bodies (i8emu_core.cuh) on the host
// ------------------------------------------------------------------------------------------------
#include "../../dftk.jl_b200/csrc/i8emu_core.cuh"
extern "C" {
// tables: q[n_mod], w[n_mod*4], P[4], returns operand bits
int emu_i8_tables(int n_mod, int64_t K, int* q, double* w, double* P) {
  I8Tables T = i8_make_tables(n_mod, K);
  for (int t = 0; t < n_mod; ++t) {
    q[t] = T.q[t];
    for (int j = 0; j < I8_LIMBS; ++j) w[t * I8_LIMBS + j] = T.w[t][j];
  }
  for (int j = 0; j < I8_LIMBS; ++j) P[j] = T.P[j];
  return T.bits;
}
// C (m x n complex, column-major) = A^H B for A (k x m), B (k x n) complex column-major, through int8 residues
int emu_i8_zgemm_cn(int n_mod, int64_t m, int64_t n, int64_t k, const double* A, const double* B, double* C) {
  I8Tables T = i8_make_tables(n_mod, 2 * k);
  const cplx* a = (const cplx*)A;
  const cplx* b = (const cplx*)B;
  std::vector<int> ea(m), eb(n);
  std::vector<signed char> ra((size_t)n_mod * 2 * m * k), rb((size_t)n_mod * 2 * n * k);
  for (int64_t i = 0; i < m; ++i) {
    double mx = 0.0;
    for (int64_t r = 0; r < k; ++r) mx = fmax(mx, fmax(fabs(a[r + k * i].x), fabs(a[r + k * i].y)));
    ea[i] = i8_scale_exponent(mx, T.bits);
    for (int64_t r = 0; r < k; ++r) i8_residues_entry(a[r + k * i], ea[i], n_mod, ra.data() + (r + k * i), (long long)m * k);
  }
  for (int64_t j = 0; j < n; ++j) {
    double mx = 0.0;
    for (int64_t r = 0; r < k; ++r) mx = fmax(mx, fmax(fabs(b[r + k * j].x), fabs(b[r + k * j].y)));
    eb[j] = i8_scale_exponent(mx, T.bits);
    for (int64_t r = 0; r < k; ++r) i8_residues_entry(b[r + k * j], eb[j], n_mod, rb.data() + (r + k * j), (long long)n * k);
  }
  cplx* c = (cplx*)C;
  for (int64_t j = 0; j < n; ++j)
    for (int64_t i = 0; i < m; ++i) {
      int rre[I8_MAX_MODULI], rim[I8_MAX_MODULI];
      for (int t = 0; t < n_mod; ++t)
        i8_dot_conj(ra.data() + (size_t)(2 * t) * m * k + k * i, ra.data() + (size_t)(2 * t + 1) * m * k + k * i,
                    rb.data() + (size_t)(2 * t) * n * k + k * j, rb.data() + (size_t)(2 * t + 1) * n * k + k * j, k,
                    i8_modulus(t), &rre[t], &rim[t]);
      c[i + m * j] = make_double2(ldexp(i8_crt(rre, T), -(ea[i] + eb[j])), ldexp(i8_crt(rim, T), -(ea[i] + eb[j])));
    }
  return T.bits;
}
}
extern "C" {
// C (m x n) = A B for A (m x k), B (k x n) complex column-major: scales per ROW of A and per column of B
int emu_i8_zgemm_nn(int n_mod, int64_t m, int64_t n, int64_t k, const double* A, const double* B, double* C) {
  I8Tables T = i8_make_tables(n_mod, 2 * k);
  const cplx* a = (const cplx*)A;
  const cplx* b = (const cplx*)B;
  std::vector<int> ea(m), eb(n);
  std::vector<signed char> ra((size_t)n_mod * 2 * m * k), rb((size_t)n_mod * 2 * n * k);   // A planes keep A's layout (m fastest)
  for (int64_t i = 0; i < m; ++i) {
    double mx = 0.0;
    for (int64_t r = 0; r < k; ++r) mx = fmax(mx, fmax(fabs(a[i + m * r].x), fabs(a[i + m * r].y)));
    ea[i] = i8_scale_exponent(mx, T.bits);
    for (int64_t r = 0; r < k; ++r) i8_residues_entry(a[i + m * r], ea[i], n_mod, ra.data() + (i + m * r), (long long)m * k);
  }
  for (int64_t j = 0; j < n; ++j) {
    double mx = 0.0;
    for (int64_t r = 0; r < k; ++r) mx = fmax(mx, fmax(fabs(b[r + k * j].x), fabs(b[r + k * j].y)));
    eb[j] = i8_scale_exponent(mx, T.bits);
    for (int64_t r = 0; r < k; ++r) i8_residues_entry(b[r + k * j], eb[j], n_mod, rb.data() + (r + k * j), (long long)n * k);
  }
  cplx* c = (cplx*)C;
  for (int64_t j = 0; j < n; ++j)
    for (int64_t i = 0; i < m; ++i) {
      int rre[I8_MAX_MODULI], rim[I8_MAX_MODULI];
      for (int t = 0; t < n_mod; ++t)
        i8_dot_plain(ra.data() + (size_t)(2 * t) * m * k + i, ra.data() + (size_t)(2 * t + 1) * m * k + i, m,
                     rb.data() + (size_t)(2 * t) * n * k + k * j, rb.data() + (size_t)(2 * t + 1) * n * k + k * j, 1, k,
                     i8_modulus(t), &rre[t], &rim[t]);
      c[i + m * j] = make_double2(ldexp(i8_crt(rre, T), -(ea[i] + eb[j])), ldexp(i8_crt(rim, T), -(ea[i] + eb[j])));
    }
  return T.bits;
}
}
extern "C" {
// residues of integer-valued doubles: division-free variant against the 64-bit integer remainder; returns #mismatches
int64_t emu_i8_residue_compare(int64_t n, const double* a) {
  int64_t bad = 0;
  for (int64_t i = 0; i < n; ++i)
    for (int t = 0; t < I8_MAX_MODULI; ++t) bad += i8_residue(a[i], i8_modulus(t)) != i8_residue_fast(a[i], i8_modulus(t));
  return bad;
}
}
