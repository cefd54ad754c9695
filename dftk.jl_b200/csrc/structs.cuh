// Grid / k-block handle definitions shared by the translation units of libdftk_b200.
#pragma once
#include "common.cuh"
#include "fft_reg_fwd.cuh"
#include "fft_plan.h"

namespace dftk {
struct SphereTablesX;
// kernel entry points of the register two-pass engine for one factor pair (fft_reg.cu)
struct RegKernels {
  int A, B, T;
  int yz_threads;             // blockDim of yz_apply (RegYZ<A, B>::NT)
  const void *sphere_to_x, *y_backward, *z_apply, *z_to_cube, *z_from_cube, *z_density, *y_forward, *x_to_sphere;
  const void* z_apply_pipe;   // persistent, software-pipelined form of z_apply (cp.async staged input tiles)
  const void* yz_apply;       // fused y-z stage of the local H apply on an x-major W1 (ny == nz)
  const void *sphere_to_xt, *xt_to_sphere;   // the x stages on the x-major W1 of yz_apply
  const void *m_sphere_to_x, *m_y_backward, *m_z_apply, *m_y_forward, *m_x_to_sphere, *m_z_density;   // many k-blocks per launch
};
// one k-block's share of a batched H-apply launch (local + kinetic part)
struct FftMultiItem {
  SphereTablesX T;
  const cplx* psi;
  long long ldpsi;
  cplx *W1, *W2;
  const double* V;
  cplx* out;
  long long ldout;
  const double* kin;
  const double* wts;     // density accumulation: band weights of this block (device) and their number
  int nb;
};
const RegKernels* reg_kernels_for(int n);   // nullptr: use the generic Stockham engine
void reg_set_attributes(int smem_optin);
}  // namespace dftk

namespace dftk {
struct I8Operand {                  // an operand of C = A^H B converted to INT8 residue planes (i8emu.cu)
  const signed char* planes = nullptr;
  const int* exps = nullptr;
  int64_t cols = 0, k = 0, ldk = 0;
  int n_mod = 0;
};
}  // namespace dftk

struct dftk_b200_grid {
  dftk_b200_ctx* ctx;
  int nx, ny, nz;
  int64_t N;
  double omega;
  double ifft_norm, fft_norm;  // src/fft.jl:87-88
  dftk::FftPlan px, py, pz;
  dftk::DevBuf<double> twx, twy, twz;
  int Lx, Ly, Lz;
  const dftk::RegKernels *rx = nullptr, *ry = nullptr, *rz = nullptr;  // register engine per axis
  dftk::DevBuf<double> Vs[2];   // total local potential per spin (pre-scaled by 1/N), shared by the k-blocks that opt in
  dftk::DevBuf<double> Vts[2];  // the same as [x][y][z] (z contiguous) for the fused y-z stage, when the grid has one
  bool has_Vs[2] = {false, false};
};

struct dftk_b200_kblock {
  dftk_b200_grid* grid;
  int64_t n_pw, n_proj;
  int spin;
  double kweight;
  dftk::SphereTablesHost Th;
  dftk::SphereTablesX T;  // device view
  dftk::DevBuf<int> d_col_start, d_col_cnt, d_slot_ix, d_slot_src, d_zlist, d_colmap, d_zc_of, d_pl_s0, d_pl_n0, d_pl_s1, d_pl_n1, d_pl_col0, d_cx_s0, d_cx_n0, d_cx_s1,
      d_cx_n1;
  dftk::DevBuf<double> kin;       // n_pw (may be empty)
  bool has_kin = false;
  dftk::DevBuf<dftk::cplx> P;     // n_pw x n_nl(): the atomic projectors, then the orbital columns (kblock_set_orbitals)
  std::vector<double> D_host;     // n_proj x n_proj
  dftk::DevBuf<dftk::cplx> Dc;    // complex copy of D on the device (n_proj x n_proj)
  // Hubbard orbitals: n_orb more columns of P that every H apply carries in the same pair of projector products.
  // n_proj, Dc, the band energies and the force rows keep covering the atomic projectors only.
  int64_t n_orb = 0;
  dftk::DevBuf<dftk::cplx> Dh;    // n_nl() x n_nl() block-diagonal [D 0; 0 V] of the H apply (only when n_orb > 0)
  std::vector<int64_t> map_h;     // sphere mapping, kept to re-pair the fold when the projector table changes
  int64_t n_nl() const { return n_proj + n_orb; }
  const dftk::cplx* Dnl() const { return n_orb ? Dh.p : Dc.p; }
  dftk::DevBuf<signed char> i8_pool[8];  // gemm_backend 4: residue planes of the LOBPCG blocks (cache slots of a solve)
  dftk::DevBuf<int> i8_epool[8];
  dftk::I8Operand i8_Pop;                // prepared projector table (kept for the lifetime of the block)
  dftk::DevBuf<signed char> i8_psi_planes;   // planes of the orbitals entering P'psi (own buffer: the pool slots belong to LOBPCG's cache)
  dftk::DevBuf<int> i8_psi_exps;
  dftk::DevBuf<signed char> i8_planes;   // gemm_backend 4: cached INT8 residue planes of P (built at first use)
  dftk::DevBuf<int> i8_exps;
  dftk::DevBuf<dftk::cplx> PD;    // P Dnl (n_pw x n_nl), kept when n_nl is small: Hψ += (P D)(P'ψ) as two batched small products
  // time-reversal fold of the projector products (blas.cu, kb_setup_fold): set on blocks whose sphere is closed under
  // q -> -q and whose projectors satisfy P(-q) = conj(P(q)); n_half = 0 keeps the complex products
  int64_t n_half = 0;                   // |H|: one plane wave of each pair ±q
  dftk::DevBuf<int> fold_i, fold_p;     // H (ascending sphere indices) and the partner -q of each
  dftk::DevBuf<double> R;               // [Re P(H); Im P(H)]: 2 n_half x n_nl, column-major
  dftk::DevBuf<dftk::cplx> fold_ws;     // folded orbitals, then [a; b], for a chunk of bands (2 n_half x chunk)
  dftk::DevBuf<double> V;         // N, pre-scaled by 1/N (fft_norm*ifft_norm)
  bool has_V = false;
  int grid_V = -1;                // >= 0: use grid->Vs[grid_V] instead of the block's own copy
  const double* Vp() const { return grid_V >= 0 ? grid->Vs[grid_V].p : V.p; }
  dftk::DevBuf<double> Vt;        // V as [x][y][z], written beside V on grids with a fused y-z stage (grid_yz_fusable)
  const double* Vtp() const { return grid_V >= 0 ? grid->Vts[grid_V].p : Vt.p; }
  // scratch
  dftk::DevBuf<dftk::cplx> W1, W2;    // pruned intermediates for a chunk of bands
  dftk::DevBuf<dftk::cplx> ldos_cube; // LDOS pass (ldos.cu): the cubes of a chunk of bands, then their |ψ|²/Ω
  dftk::DevBuf<double> ldos_rho;
  dftk::DevBuf<dftk::cplx> proj;      // n_proj x n_bands (+ D*proj)
  dftk::DevBuf<dftk::cplx> lobpcg_ws; // big LOBPCG workspace
  dftk::DevBuf<dftk::cplx> small_ws;  // small dense LOBPCG workspace
  dftk::DevBuf<dftk::cplx> slab_x, slab_stage;   // slab-distributed solve (lobpcg_run_slab): this rank's rows of X, reassembly staging
  dftk::DevBuf<double> scal;          // per-block scalars of a LOBPCG solve (several blocks are solved side by side)
};

namespace dftk {
// fft.cu
int band_chunk_for(dftk_b200_kblock* kb, int64_t n_bands, bool with_W2 = true);
bool grid_yz_fusable(const dftk_b200_grid* g);
void fft_cube_inplace(dftk_b200_grid* g, cplx* data, int sign, int64_t batch);
void kb_sphere_to_planes(dftk_b200_kblock* kb, const cplx* psi, int64_t ldpsi, int nb);
void kb_planes_to_sphere(dftk_b200_kblock* kb, cplx* out, int64_t ldout, int nb, double scale,
                         const double* kin, const cplx* psi, int64_t ldpsi, int accumulate);
void kb_apply_local_kinetic(dftk_b200_kblock* kb, const cplx* psi, cplx* hpsi, int64_t n_bands,
                            bool with_local, bool with_kin, bool accumulate);
// the same for several k-blocks of ONE grid in five launches in total; returns false (nothing done) when the blocks do
// not qualify (different grids, generic FFT engine, missing potential / kinetic term): the caller then loops
bool kb_apply_local_kinetic_multi(int n, dftk_b200_kblock* const* kbs, const cplx* const* psi, cplx* const* hpsi,
                                  const int* n_bands, DescRing& ring);
void kb_sphere_to_real(dftk_b200_kblock* kb, const cplx* psi, cplx* cube, int64_t n_bands, double scale);
void kb_real_to_sphere(dftk_b200_kblock* kb, const cplx* cube, cplx* out, int64_t n_bands, double scale);
void kb_density_accumulate(dftk_b200_kblock* kb, const cplx* psi, const double* occ_w_host,
                           int64_t n_bands, double* rho);
// all k-blocks of a rank: stages A, B batched over the blocks, one accumulation launch per spin channel;
// rho: n_spin x N (device), occ_w_host: n x ld_w.  Returns false (nothing done) when the blocks do not qualify.
bool kb_density_accumulate_multi(int n, dftk_b200_kblock* const* kbs, const cplx* const* psi, const double* occ_w_host,
                                 int64_t ld_w, const int* n_bands, double* rho);
void fft_set_attributes();
// blas.cu
void zgemm(dftk_b200_ctx* ctx, int transA, int64_t m, int64_t n, int64_t k, cplx alpha, const cplx* A,
           int64_t lda, const cplx* B, int64_t ldb, cplx beta, cplx* C, int64_t ldc, bool upper_only = false);
// upper_only: transA == 2 -> only tiles on/above the diagonal are computed (Hermitian result);
//             transA == 0 -> B is upper triangular (trmm-like: half the flops)
void blas_set_attributes();
void kb_apply_nonlocal(dftk_b200_kblock* kb, const cplx* psi, cplx* hpsi, int64_t n_bands);
void kb_project(dftk_b200_kblock* kb, const cplx* psi, int64_t n_bands, cplx* proj);   // proj = P' psi (n_proj x n_bands)
// proj (nc x n_bands) = P[:, c0 : c0+nc]' psi, on the folded operands where the block has them
void kb_project_cols(dftk_b200_kblock* kb, int64_t c0, int64_t nc, const cplx* psi, int64_t n_bands, cplx* proj);
void kb_refresh_pd(dftk_b200_kblock* kb, int64_t c0);   // PD[:, c0:] = P Dnl[:, c0:] (PD is kept when n_nl <= 96)
bool sphere_mirror(int nx, int ny, int nz, int64_t n_pw, const int64_t* map, std::vector<int>& mir);
void kb_setup_fold(dftk_b200_kblock* kb, const int64_t* map_h);
void columnwise_dots(dftk_b200_ctx* ctx, const cplx* A, int64_t lda, const cplx* B, int64_t ldb,
                     int64_t n_rows, int64_t n_cols, cplx* out_dev);
void kin_dots(dftk_b200_ctx* ctx, const cplx* X, int64_t ldx, const double* kin, int64_t n_rows,
              int64_t n_cols, double* out_dev);
void scale_kin_add(dftk_b200_ctx* ctx, const cplx* psi, cplx* hpsi, const double* kin, int64_t n_rows,
                   int64_t n_cols, int accumulate);
// xc.cu
void xc_evaluate(dftk_b200_ctx* ctx, int mask, int n_spin, bool gga, int64_t N, const double* rho,
                 const double* sigma, double* e, double* vrho, double* vsigma);
void symmetrize_fourier(dftk_b200_grid* g, const cplx* in, cplx* out, int n_sym, const int* invS_host,
                        const double* tau_host);
// i8emu.cu (experimental, option gemm_backend = 2)
void zgemm_i8_cn(dftk_b200_ctx* ctx, int64_t m, int64_t n, int64_t k, const cplx* A, int64_t lda, const cplx* B, int64_t ldb,
                 cplx* C, int64_t ldc, bool tensor_cores, const signed char* ra_cached = nullptr, const int* ea_cached = nullptr);
void i8tc2_products(dftk_b200_ctx* ctx, const signed char* ra, const signed char* rb, int64_t m, int64_t n, int64_t ldk,
                    int n_mod, short* part, int* res, bool upper_only);
I8Operand i8_prepare(dftk_b200_ctx* ctx, const cplx* X, int64_t ld, int64_t cols, int64_t k, DevBuf<signed char>& store,
                     DevBuf<int>& estore);
void i8_gram(dftk_b200_ctx* ctx, const I8Operand& A, const I8Operand& B, cplx* C, int64_t ldc, bool upper_only);
// C (rows x n) = alpha sum_b A_b B[rows of b, :] + beta C from prepared tall operands (update-type products)
void i8_update(dftk_b200_ctx* ctx, int n_blocks, const I8Operand* A, const cplx* B, int64_t ldb, int64_t n, cplx* C, int64_t ldc,
               double alpha, double beta);
void i8tc2_products_nn(dftk_b200_ctx* ctx, int n_blocks, const signed char* const* ra, const int* kcols, const int* k_off,
                       int64_t ldm, const signed char* rb, int64_t ldkb, int64_t m, int64_t n, int n_mod, signed char* resid);
void i8tc2_set_attributes();
bool zgemm_i8_nn(dftk_b200_ctx* ctx, int64_t m, int64_t n, int64_t k, const cplx* A, int64_t lda, const cplx* B, int64_t ldb,
                 cplx* C, int64_t ldc, bool accumulate);
// forces.cu
void local_forces(dftk_b200_grid* g, const cplx* w, int n_atoms, const double* pos_host, double* out_host);
void kb_nonlocal_force_rows(dftk_b200_kblock* kb, const cplx* psi, const double* occ_w_host, int64_t n_bands,
                            const double* gpk, double* out_host);
void ewald(dftk_b200_ctx* ctx, const double* lattice_colmajor, int n_atoms, const double* charges, const double* positions,
           double eta, const int* glims, const int* rlims, double* energy_host, double* forces_host);
// setup.cu
void structure_factor(dftk_b200_grid* g, int n_atoms, const double* pos_host, const double* coeff_host, cplx* out);
void build_projectors(dftk_b200_ctx* ctx, int64_t n_pw, const double* gpk, int n_atoms, const double* pos_host, int n_rows,
                      const cplx* ff, cplx* P);
constexpr int RADIAL_MAX_F = 16;     // functions per launch of the radial transform (accumulators held in registers)
struct RadialL {                     // angular momenta of the functions of one launch, passed by value
  int l[RADIAL_MAX_F];
  int lmax;
};
void radial_transform(dftk_b200_ctx* ctx, int64_t n_r, const double* r, int n_f, const double* g, const int* l_host, int64_t n_q,
                      const double* q, double* F);
// lobpcg.cu
int lobpcg_run(dftk_b200_kblock* kb, cplx* X, int64_t M, double tol, int miniter, int maxiter,
               int64_t n_conv_check, bool use_prec, double* lambda_host, double* resid_host,
               int* n_iter, int64_t* n_matvec, int* converged);
int lobpcg_run_multi(int64_t n_blocks, dftk_b200_kblock* const* kbs, cplx* const* Xs, int64_t M, double tol, int miniter,
                     int maxiter, int64_t n_conv_check, bool use_prec, double* lambda_host, double* resid_host, int* n_iter,
                     int64_t* n_matvec, int* converged);
int lobpcg_run_slab(dftk_b200_kblock* kb, cplx* Xfull, int64_t M, double tol, int miniter, int maxiter, int64_t n_conv_check,
                    bool use_prec, double* lambda_host, double* resid_host, int* n_iter, int64_t* n_matvec, int* converged,
                    double* exchange_bytes);
void random_orbitals_multi(int64_t n_blocks, dftk_b200_kblock* const* kbs, cplx* const* Xs, int64_t M, uint64_t seed);
void band_energies_multi(int64_t n, dftk_b200_kblock* const* kbs, const cplx* const* psi, const int* n_bands, int64_t ld_out,
                         double* ekin_host, double* enl_host);
void orbital_occupation_multi(int64_t n, dftk_b200_kblock* const* kbs, const cplx* const* psi, const double* occ_w_host,
                              int64_t ld_w, const int* n_bands, cplx* n_out);
void tall_gram(dftk_b200_ctx* ctx, const cplx* A, int64_t lda, int nA, const cplx* B, int64_t ldb, int nB, int64_t n_rows,
               cplx* out_host);
void lobpcg_set_attributes();
}  // namespace dftk
