// Host emulation of the fused y-z path of the local H apply (TEST INFRASTRUCTURE ONLY): the x stages on the x-major W1
// and reg_yz_apply (fft_reg.cuh), run block by block and "thread" by "thread" on top of the emulator of emu.cu.
#include "emu.cu"

extern "C" {
// sphere -> x-major W1 [band][x][col], y-z per (band, x line), W1 -> sphere (+ kin psi) (+ out0 when given)
int emur_apply_local_yz(int nx, int ny, int nz, int64_t n_pw, const int64_t* mapping, const double* psi, int nb,
                        const double* Vt_scaled, const double* kin, const double* out0, double* out) {
  EmuR e(nx, ny, nz, n_pw, mapping, nb);
  if (!e.H.ranges_ok) return -9;
  if (ny != nz) return -10;
  const SphereTablesX& TX = e.TX;
  const int n_cols = e.T.n_cols;
#define CX(a, b) if (A_ == a && B_ == b) { int L = EmuR::Lof(a, b), Lp = L + 1; done_ = true; \
  for (int bb = 0; bb < nb; ++bb) for (int bx = 0; bx < (n_cols + L - 1) / L; ++bx) \
    reg_sphere_to_x<a, b, 1>(TX, e.tx(), (const cplx*)psi, n_pw, e.W1.data(), L, Lp, e.sm.data(), Dim3i{bx, bb, 0}); }
  DISPATCH(nx, CX);
#undef CX
#define CYZ(a, b) if (A_ == a && B_ == b) { done_ = true; \
  std::vector<cplx> sm(RegYZ<a, b>::smem(TX.n_zc) / sizeof(cplx)); \
  for (int bb = 0; bb < nb; ++bb) for (int x = 0; x < nx; ++x) \
    reg_yz_apply<a, b>(TX, e.ty(), e.W1.data(), Vt_scaled, sm.data(), Dim3i{x, 0, bb}); }
  DISPATCH(ny, CYZ);
#undef CYZ
  if (out0) std::memcpy(out, out0, sizeof(cplx) * (size_t)nb * n_pw);
  const int acc = out0 ? 1 : 0;
#define CX(a, b) if (A_ == a && B_ == b) { int L = EmuR::Lof(a, b), Lp = L + 1; done_ = true; \
  for (int bb = 0; bb < nb; ++bb) for (int bx = 0; bx < (n_cols + L - 1) / L; ++bx) \
    reg_x_to_sphere<a, b, 1>(TX, e.tx(), e.W1.data(), (cplx*)out, n_pw, 1.0, kin, (const cplx*)psi, n_pw, acc, L, Lp, \
                             e.sm.data(), Dim3i{bx, bb, 0}); }
  DISPATCH(nx, CX);
#undef CX
  return 0;
}
}
