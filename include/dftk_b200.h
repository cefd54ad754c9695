/*
 * libdftk_b200 -- C ABI of the H100-native (sm_90a) plane-wave Kohn-Sham hot path.
 *
 * Drop-in boundary for the seam where DFTK.jl's ext/DFTKCUDAExt.jl + src/architecture.jl plug in
 * today (reference paths relative to the DFTK.jl tree).  Each entry point names the reference
 * function it replaces.  Conventions (SURVEY.md §8b):
 *   - all functions return 0 on success, a negative DFTK_B200_E* code on failure; the message of the
 *     last failure on a context is available from dftk_b200_last_error(); nothing throws.
 *   - column-major arrays, complex = interleaved double[2], indices 0-based (Julia glue subtracts 1
 *     once when it passes `kpt.mapping`).
 *   - "dev/host" pointers may be device or host memory (resolved through UVA); hot-path buffers
 *     (psi, hpsi, X, rho) are expected on the device -- host buffers are staged through H2D/D2H copies
 *     inside the call (this is what the end-to-end benchmark measures).
 *   - handles are opaque and not thread-safe; one context per GPU / rank; the caller owns psi/rho/V
 *     buffers, the library owns plans, scratch and its copies of mapping/kin/P/D.
 */
#ifndef DFTK_B200_H
#define DFTK_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dftk_b200_ctx dftk_b200_ctx;
typedef struct dftk_b200_grid dftk_b200_grid;
typedef struct dftk_b200_kblock dftk_b200_kblock;

#define DFTK_B200_OK 0
#define DFTK_B200_EINVAL (-1)   /* bad argument */
#define DFTK_B200_ECUDA (-2)    /* CUDA runtime / library failure */
#define DFTK_B200_ENUM (-3)     /* numerical failure (e.g. LOBPCG cannot keep vectors normalised) */
#define DFTK_B200_ENCCL (-4)    /* NCCL failure / communicator missing */

#define DFTK_B200_F64 0
#define DFTK_B200_I64 1

/* ---- context (replaces the `architecture=GPU(CuArray)` selection, src/architecture.jl:4-53;
 *      synchronize_device / memory_usage, ext/DFTKCUDAExt.jl:11-15) ---- */
int dftk_b200_ctx_create(int device, dftk_b200_ctx** out);
/* distributed variant: `nccl_unique_id` = 128 bytes from dftk_b200_nccl_unique_id on rank 0 */
int dftk_b200_ctx_create_dist(int device, const void* nccl_unique_id, int rank, int nranks,
                              dftk_b200_ctx** out);
int dftk_b200_nccl_unique_id(void* out128);
int dftk_b200_ctx_destroy(dftk_b200_ctx* ctx);
const char* dftk_b200_last_error(dftk_b200_ctx* ctx); /* ctx may be NULL: last global error */
/* Every kernel, copy and library call of this context is enqueued on ONE CUDA stream: the legacy default stream after
 * creation (ordered with the caller's default-stream work, which is what DFTK's GPU path uses), or the `cudaStream_t`
 * given here (e.g. CUDA.jl's task-local stream, `CUDA.stream().handle`).  Handles created from the context follow. */
int dftk_b200_ctx_set_stream(dftk_b200_ctx* ctx, void* cuda_stream);
int dftk_b200_sync(dftk_b200_ctx* ctx);
int dftk_b200_mem_info(dftk_b200_ctx* ctx, int64_t* free_bytes, int64_t* total_bytes);
/* number of kernel launches issued by this library on the context since creation / last reset */
int64_t dftk_b200_launch_count(dftk_b200_ctx* ctx, int reset);
/* number of scheduler rounds (= host synchronisations) of the batched LOBPCG solves since creation / last reset */
int64_t dftk_b200_sync_count(dftk_b200_ctx* ctx, int reset);
/* FP64-equivalent GEMM flops the large-path LOBPCG solves of this context have executed since the last reset: Gram-type products
 * (8 rows·m·n, half of it for the upper-triangle-only diagonal blocks), update-type products, the X R^-1 updates of ortho! and the
 * two projector products of every H apply -- the "sum actually executed" of SURVEY §8d.  Batched small-block solves are not counted. */
double dftk_b200_lobpcg_flops(dftk_b200_ctx* ctx, int reset);
/* tuning knobs: "gemm_backend" (0 = default: own FP64 DMMA kernels; 4 = the Gram-type and update-type products of
 * contractions with at least "i8_min_rows" (32768) rows on the INT8 tensor cores -- wgmma s8 fed by TMA, FP64-equivalent results
 * through INT8 residues + CRT -- and everything smaller on the DMMA kernels; 1 = cuBLAS, for A/B comparison and peak calibration
 * only; 2 = checker of the INT8 scheme: integer products on CUDA cores), "gemm_stages" (cp.async ring depth 2|3|4 of the DMMA kernels, default 4), "band_chunk" (bands per batched-FFT
 * launch, 0 = auto), "fft_engine" (0 = register two-pass engine where a factor pair exists, 1 = generic Stockham; applies to
 * grids created afterwards), "small_dense" (1 = batched small-matrix path for LOBPCG solves with <= 32 bands, 0 = the GEMM +
 * cuSOLVER sequence of the large path), "z_pipeline" (1 = persistent cp.async-pipelined fused z stage; default 0),
 * "batch_pipeline" (1 = batched solves of >= 8 k-blocks run as two groups on two streams so that one group's host work hides
 * behind the other's kernels; 0 = one group, one stream synchronisation per round; default 0),
 * "force_svd_fallback" (test hook) */
int dftk_b200_set_option(dftk_b200_ctx* ctx, const char* name, int64_t value);

/* ---- FFT grid (FFTGrid + build_fft_plans!, src/fft.jl:57-98,343-362) ---- */
int dftk_b200_grid_create(dftk_b200_ctx* ctx, int nx, int ny, int nz, double unit_cell_volume,
                          dftk_b200_grid** out);
int dftk_b200_grid_destroy(dftk_b200_grid* grid);
/* in-place unnormalised 3D C2C transform of `batch` cubes; direction -1 = forward (e^{-iGr}),
 * +1 = backward (ipFFT / ipBFFT of src/fft.jl:107,119,159,166) */
int dftk_b200_fft_cube(dftk_b200_grid* grid, void* data /*dev: complex[N*batch]*/, int direction,
                       int64_t batch);

/* ---- k-block = Kpoint + DftHamiltonianBlock data (src/Kpoint.jl:6-41,
 *      src/terms/Hamiltonian.jl:22-57, kinetic.jl:24-35, nonlocal.jl:9-28) ----
 * mapping: n_pw int64, 0-based linear cube index of each sphere coefficient (kpt.mapping - 1)
 * kin:     n_pw doubles, ½|k+G|² (FourierMultiplication multiplier); may be NULL (no kinetic term)
 * P:       n_pw × n_proj complex, column-major (NonlocalOperator.P); n_proj may be 0
 * D:       n_proj × n_proj real, column-major (NonlocalOperator.D, block diagonal) */
int dftk_b200_kblock_create(dftk_b200_grid* grid, int64_t n_pw, const int64_t* mapping,
                            const double* kin, int64_t n_proj, const void* P, const double* D,
                            int spin, double kweight, dftk_b200_kblock** out);
int dftk_b200_kblock_destroy(dftk_b200_kblock* kb);

/* ---- DFT+U orbitals (the NonlocalOperator(Φ_k, D[σ]) of TermHubbard, src/terms/hubbard.jl:103-184) ----
 * Attaches n_orb Hubbard orbital columns Phi (n_pw × n_orb complex, column-major, host or device) to the block: every H
 * apply then carries [P | Φ] with D = [D 0; 0 V] in ONE pair of projector products, on every path (complex and folded
 * DMMA products, batched small path while n_proj + n_orb <= 96, INT8 planes of gemm_backend 4).  V starts at zero.
 * n_orb = 0 removes the orbitals.  n_proj, the nonlocal band energies and dftk_b200_nonlocal_force_rows keep covering
 * the atomic projectors only.  The slab solver (dftk_b200_lobpcg_slab) rejects blocks with orbitals. */
int dftk_b200_kblock_set_orbitals(dftk_b200_kblock* kb, int64_t n_orb, const void* Phi /*n_pw×n_orb*/);
/* Plane waves of one ±q pair on which the block's projector products run when they take the time-reversal fold (Γ and
 * other k with 2k in the reciprocal lattice, and a table with P(-q) = conj P(q), orbital columns included); 0 when the
 * block runs the complex products. */
int dftk_b200_kblock_fold_size(dftk_b200_kblock* kb, int64_t* n_half);
/* Installs the orbital block V (n_orb × n_orb complex Hermitian, column-major, host or device; NULL = zero) of the
 * block's D and refreshes the derived tables on the device.  Called every SCF step; Φ is not re-uploaded. */
int dftk_b200_kblock_set_orbital_coefficients(dftk_b200_kblock* kb, const void* V /*n_orb×n_orb*/);
/* Occupation matrices of the orbitals (hubbard.jl:201-232 before its mpi_sum), all k-blocks of a rank in one call:
 * n_out[σ] += Σ_{blocks of spin σ} Σ_n w_n (Φ'ψ_n)(Φ'ψ_n)'.  psi[i]: n_pw × n_bands[i] device orbitals; occ_w_host:
 * n_blocks × ld_w band weights (k-weight × occupation / filled occupation); n_out: n_spin × n_orb × n_orb complex
 * column-major device array, accumulated.  Every block must carry the same n_orb.  Blocks of <= 32 bands and <= 96
 * orbitals share one batched projection launch; one synchronisation in all. */
int dftk_b200_orbital_occupation_multi(int64_t n_blocks, dftk_b200_kblock* const* kblocks, const void* const* psi,
                                       const double* occ_w_host, int64_t ld_w, const int32_t* n_bands, void* n_out);
/* total local potential on the real-space grid for this block's spin (sum of all
 * RealSpaceMultiplication operators, src/terms/operators.jl:213-222); N_fft doubles.  NULL = none */
int dftk_b200_kblock_set_potential(dftk_b200_kblock* kb, const double* V);

/* The same potential for all k-blocks of one spin channel: ONE pre-scaled copy per (grid, spin) instead of one per block
 * (all blocks of a spin share the term potentials, src/terms/Hamiltonian.jl:200-227).  A block opts in with
 * dftk_b200_kblock_use_grid_potential(kb, spin) (spin = -1: back to its own copy). */
int dftk_b200_grid_set_potential(dftk_b200_grid* grid, int spin, const double* V);
int dftk_b200_kblock_use_grid_potential(dftk_b200_kblock* kb, int spin);

/* Frees the scratch a k-block has grown (LOBPCG workspaces, INT8 residue-plane pools of the solver, FFT intermediates); the
 * operator data (kinetic energies, projectors and their prepared planes, potential) stays, and every later call re-grows what
 * it needs.  A 503-band solve at n_pw = 264 859 holds ≈ 60 GB of such scratch (no reference counterpart: Julia's GC does this). */
int dftk_b200_kblock_trim(dftk_b200_kblock* kb);

/* ---- sphere <-> real-space transforms (ifft!/fft! with Gvec_mapping, src/fft.jl:110-122,162-172) */
int dftk_b200_fft_sphere_to_real(dftk_b200_kblock* kb, const void* psi /*n_pw×n_bands*/,
                                 void* out_real /*N_fft×n_bands complex*/, int64_t n_bands,
                                 int normalize);
int dftk_b200_fft_real_to_sphere(dftk_b200_kblock* kb, const void* in_real /*N_fft×n_bands*/,
                                 void* out /*n_pw×n_bands*/, int64_t n_bands, int normalize);

/* ---- Hψ (LinearAlgebra.mul!(Hψ, ::DftHamiltonianBlock, ψ), src/terms/Hamiltonian.jl:137-192) ----
 * hpsi = FFT[V·IFFT[psi]] + kin·psi + P (D (P' psi)), all bands of the block in one batched pass. */
int dftk_b200_apply_h(dftk_b200_kblock* kb, const void* psi, void* hpsi, int64_t n_bands);
/* individual operators, `apply!(out, op, in)` semantics of src/terms/operators.jl (ACCUMULATE into hpsi
 * when accumulate != 0): parts bitmask 1 = local (RealSpaceMultiplication :71-78),
 * 2 = kinetic (FourierMultiplication :104-112), 4 = nonlocal (NonlocalOperator :119-129) */
int dftk_b200_apply_terms(dftk_b200_kblock* kb, const void* psi, void* hpsi, int64_t n_bands,
                          int parts, int accumulate);
/* per-band <psi|kin|psi> and <psi|P D P'|psi> (ene_ops, kinetic.jl:40-57, nonlocal.jl:31-47); host out */
int dftk_b200_band_energies(dftk_b200_kblock* kb, const void* psi, int64_t n_bands,
                            double* ekin_host, double* enl_host);

/* the same for all k-blocks of a rank in four launches and ONE synchronisation (blocks of <= 32 bands and <= 96 projectors);
 * ekin_host / enl_host: n_blocks × ld_out, either may be NULL */
int dftk_b200_band_energies_multi(int64_t n_blocks, dftk_b200_kblock* const* kblocks, const void* const* psi,
                                  const int32_t* n_bands, int64_t ld_out, double* ekin_host, double* enl_host);

/* ---- LOBPCG (lobpcg_hyper, src/eigen/diag_lobpcg_hyper.jl:5-18 -> LOBPCG,
 *      src/eigen/lobpcg_hyper_impl.jl:354-582, PreconditionerTPA src/eigen/preconditioners.jl:27-78) ----
 * X: n_pw × n_bands, in: guess, out: eigenvectors (device).  lambda/resid: host, n_bands each. */
int dftk_b200_lobpcg(dftk_b200_kblock* kb, void* X, int64_t n_bands, double tol, int miniter,
                     int maxiter, int64_t n_conv_check, int use_tpa_preconditioner,
                     double* lambda_host, double* resid_host, int* n_iter, int64_t* n_matvec,
                     int* converged);

/* All (k, spin) blocks of a rank at once (diagonalize_all_kblocks, src/eigen/diag.jl:9-65: the per-k eigenproblems are
 * independent).  Same algorithm and same results per block as dftk_b200_lobpcg; for blocks of <= 32 bands the solves advance
 * in lockstep and every operation of all blocks is ONE kernel launch (one host synchronisation per round instead of per
 * block) -- the launch-latency-bound regime of small cells with many k-points.  X[i]: n_pw_i × n_bands (device);
 * lambda_host / resid_host: n_blocks × n_bands (block-major); n_iter / n_matvec / converged: n_blocks each. */
int dftk_b200_lobpcg_multi(int64_t n_blocks, dftk_b200_kblock* const* kblocks, void* const* X, int64_t n_bands,
                           double tol, int miniter, int maxiter, int64_t n_conv_check, int use_tpa_preconditioner,
                           double* lambda_host, double* resid_host, int* n_iter, int64_t* n_matvec, int* converged);

/* ONE k-block solved by all ranks of a distributed context together (single-k multi-GPU; the reference cannot use more
 * than one process for one k-point, docs/src/tricks/parallelization.md:83-84).  Collective: every rank of the context calls
 * it with its own k-block handle of the SAME k-point and the same X (n_pw × n_bands, device, identical on all ranks).
 * The plane-wave rows of every tall block of lobpcg_hyper_impl.jl are cut into one slab per rank: Gram products, norms and
 * Rayleigh quotients are local products completed by ncclAllReduce, the small dense algebra (Cholesky, Rayleigh-Ritz) runs
 * replicated, and H is applied band-wise after a rows <-> bands exchange over NCCL point-to-point.  On return X holds the
 * eigenvectors on every rank; the other outputs are those of dftk_b200_lobpcg.  exchange_bytes (may be NULL): bytes this
 * rank sent in the rows <-> bands exchanges. */
int dftk_b200_lobpcg_slab(dftk_b200_kblock* kb, void* X, int64_t n_bands, double tol, int miniter, int maxiter,
                          int64_t n_conv_check, int use_tpa_preconditioner, double* lambda_host, double* resid_host,
                          int* n_iter, int64_t* n_matvec, int* converged, double* exchange_bytes);

/* Start vectors (random_orbitals, src/common/orbitals.jl:82-87: orthonormalised complex normal numbers) for several
 * k-blocks at once: X[i] (n_pw_i × n_bands, device) is filled and orthonormalised on the device. */
int dftk_b200_random_orbitals(int64_t n_blocks, dftk_b200_kblock* const* kblocks, void* const* X, int64_t n_bands,
                              uint64_t seed);

/* ---- density (compute_density inner loop, src/densities.jl:32-44):
 *      rho[:,:,:] += sum_n occ_w[n] |IFFT psi_n|² / Ω   with occ_w[n] = occupation·kweight (host) ---- */
int dftk_b200_density_accumulate(dftk_b200_kblock* kb, const void* psi, const double* occ_w_host,
                                 int64_t n_bands, double* rho /*dev: N_fft doubles of this spin*/);

/* compute_density's loop over the k-blocks of a rank in one call: rho (n_spin × N_fft, device) += contributions of all
 * blocks (each into the channel of its spin); occ_w_host: n_blocks × ld_w.  Blocks that share the grid's register FFT engine
 * are transformed together (two launches for all of them) and accumulated by one launch per spin channel. */
int dftk_b200_density_accumulate_multi(int64_t n_blocks, dftk_b200_kblock* const* kblocks, const void* const* psi,
                                       const double* occ_w_host, int64_t ld_w, const int32_t* n_bands, double* rho);

/* The LDOS at n_energies energies in one pass over the bands (compute_ldos, src/postprocess/dos.jl):
 *   ldos[j, σ, :] += Σ_blocks of spin σ Σ_n W[j, i, n] |IFFT psi_n|² / Ω
 * W (device): n_energies × n_blocks × ld_w doubles, W[(j n_blocks + i) ld_w + n] the weight of band n of block i at energy j
 * (k-point weight included); ldos (device): n_energies × n_spin × N_fft.  A band whose weight is zero at every energy is
 * neither transformed nor multiplied.  Each kept band is transformed once with the density pass's sphere -> cube FFT, staged
 * as |ψ|²/Ω in k-block scratch (released by kblock_trim), and multiplied into all energies by a real FP64 DMMA product;
 * fixed-order sums, so a rerun is bit-identical.  n_spin is the model's: a rank may hold blocks of one spin only. */
int dftk_b200_ldos_accumulate_multi(int64_t n_blocks, dftk_b200_kblock* const* kblocks, const void* const* psi,
                                    const int32_t* n_bands, int64_t n_energies, int64_t n_spin, const double* W /*dev*/,
                                    int64_t ld_w, double* ldos /*dev: n_energies × n_spin × N_fft*/);

/* ---- collectives (mpi_sum!/mpi_min/mpi_max over basis.comm_kpts, src/common/mpi.jl:19-31) ---- */
int dftk_b200_allreduce(dftk_b200_ctx* ctx, void* buf /*dev*/, int64_t count, int dtype,
                        int op /*0 sum, 1 min, 2 max*/);
int dftk_b200_allgather(dftk_b200_ctx* ctx, const void* send /*dev*/, void* recv /*dev*/,
                        int64_t count_per_rank, int dtype);

/* ---- SCF plumbing next to the hot path (SURVEY §8f rank 1) ----
 * Pointwise exchange-correlation (replaces the Libxc dispatch, ext/DFTKCUDAExt.jl:17-25, src/terms/xc.jl:104-113).
 * functional_mask: 1 lda_x | 2 lda_c_vwn | 4 lda_c_pw | 8 gga_x_pbe | 16 gga_c_pbe | 32 lda_xc_teter93 | 64 lda_c_pz |
 * 128 gga_x_pbe_sol | 256 gga_c_pbe_sol | 512 gga_x_pbe_r | 1024 gga_x_rpbe; a gga_* bit needs sigma.  Arrays are component-major
 * device doubles: rho[n_spin][n], sigma[1|3][n] (uu, ud, dd; GGA only), e[n] (energy per volume),
 * vrho[n_spin][n], vsigma[1|3][n] -- the quantities libxc returns as zk*rho, vrho, vsigma. */
int dftk_b200_xc_evaluate(dftk_b200_ctx* ctx, int functional_mask, int n_spin, int64_t n_points,
                          const double* rho, const double* sigma, double* e, double* vrho, double* vsigma);
/* accumulate_over_symmetries! + normalisation (src/symmetry.jl:282-327,340-357) on Fourier coefficients of the cube:
 * out[G] = 1/n_sym * sum_s exp(-2 pi i G.tau_s) in[S_s^-1 G]  (terms outside the FFT box dropped).
 * invS: n_sym row-major 3x3 integer matrices (host), tau: n_sym fractional translations (host). */
int dftk_b200_symmetrize_fourier(dftk_b200_grid* grid, const void* rho_fourier_in, void* rho_fourier_out,
                                 int n_sym, const int32_t* invS, const double* tau);

/* ---- Hellmann-Feynman forces (SURVEY §8f rank 4; compute_forces, src/postprocess/forces.jl:24-30) ----
 * Local term (forces_local, src/terms/local.jl:152-181): for every atom of one species,
 *   F_a,α = -Re( Σ_G -2πi G_α e^{-2πi G·r_a} w_G ),  w_G = conj(ρ_G) v_loc(|G|) / sqrt(Ω)  (device, N_fft complex),
 * positions: 3·n_atoms fractional coordinates (host), forces_host: 3·n_atoms reduced-coordinate forces. */
int dftk_b200_local_forces(dftk_b200_grid* grid, const void* w, int n_atoms, const double* positions,
                           double* forces_host);
/* Nonlocal term (compute_forces(::TermAtomicNonlocal), src/terms/nonlocal.jl:49-100) for one k-block: per projector
 * row j and direction α the contribution  -Σ_n occ_w[n] 2 Re <ψ_n| P D (dP_j/dR_α)† |ψ_n>  with
 * dP/dR_α = -2πi (G+k)_α P, obtained from four projections P†[ψ, p_x ψ, p_y ψ, p_z ψ] instead of the reference's
 * 3·n_atoms full-height GEMM pairs.  gpk: 3 × n_pw reduced G+k components, component-major (device);
 * rows_host: 3 × n_proj (α-major).  The caller sums the rows of each atom, allreduces over k and symmetrises. */
int dftk_b200_nonlocal_force_rows(dftk_b200_kblock* kb, const void* psi, const double* occ_w_host, int64_t n_bands,
                                  const double* gpk, double* rows_host);

/* Ewald energy and forces of the ionic point charges (energy_forces_ewald, src/terms/ewald.jl:64-168, q = 0): the real-space
 * and the reciprocal-space lattice sums as one kernel each.  lattice: 3×3 column-major (columns = lattice vectors), charges:
 * n_atoms, positions: 3·n_atoms fractional (all host); eta and the summation limits (|G_i| <= glims[i], |R_i| <= rlims[i]) are
 * the caller's (ewald.jl:86-104).  energy_host: 1 double (Hartree); forces_host: 3·n_atoms, reduced coordinates; either NULL. */
int dftk_b200_ewald(dftk_b200_ctx* ctx, const double* lattice, int n_atoms, const double* charges, const double* positions,
                    double eta, const int32_t* glims, const int32_t* rlims, double* energy_host, double* forces_host);

/* ---- setup kernels (SURVEY §8f rank 4): the O(n_atoms × N) structure-factor work before the first SCF step ----
 * out[G] = Σ_a c_a exp(-2πi G·r_a) on the whole FFT cube (G from the cube index, src/fft.jl:24-31): the atomic sums of
 * build_local_potential (src/terms/local.jl:108-138) and guess_density (src/density_methods.jl:103-181).
 * positions: 3·n_atoms fractional (host), coefficients: n_atoms (host) or NULL = 1, out: N_fft complex (device). */
int dftk_b200_structure_factor(dftk_b200_grid* grid, int n_atoms, const double* positions, const double* coefficients, void* out);
/* P[(a, p), G] = exp(-2πi (G+k)·r_a) · ff[p, G]: the projector table of one species for one k-block
 * (build_projection_vectors, src/terms/nonlocal.jl:166-199).  gpk: 3 × n_pw reduced G+k, component-major (device);
 * positions: 3·n_atoms (host); form_factors: n_rows × n_pw complex, row = projector (l, m, i) already divided by sqrt(Ω)
 * (device); P: (n_atoms·n_rows) × n_pw complex, i.e. the column-major n_pw × n_proj block of these atoms (device). */
int dftk_b200_build_projectors(dftk_b200_ctx* ctx, int64_t n_pw, const double* gpk, int n_atoms, const double* positions,
                               int n_rows, const void* form_factors, void* P);
/* Radial (modified Hankel) transforms of n_f functions tabulated on one radial mesh (the eval_psp_*_fourier methods of a
 * numerical UPF pseudopotential, src/pseudo/PspUpf.jl, src/common/hankel.jl):
 *   F[f, q] = 4π / q^l_f · Σ_i g[f, i] j_{l_f}(q r_i),   and for q <= 10·eps the limit 4π/(2l_f+1)!! · Σ_i g[f, i] r_i^l_f.
 * r: n_r mesh points (device); g: n_f × n_r row-major integrands r²f(r) times the quadrature weights, zero beyond the end of a
 * function (device); l: n_f angular momenta 0..3 (host); q: n_q values >= 0 (device); F: n_f × n_q row-major (device). */
int dftk_b200_radial_transform(dftk_b200_ctx* ctx, int64_t n_r, const double* r, int n_f, const double* g, const int32_t* l,
                               int64_t n_q, const double* q, double* F);

/* ---- small dense helpers used by the host driver (columnwise_dots, src/common/linalg.jl:2-15) ---- */
int dftk_b200_columnwise_dots(dftk_b200_ctx* ctx, const void* A, const void* B, int64_t n_rows,
                              int64_t n_cols, void* out_host /*complex[n_cols]*/);
/* out (n_cols_a × n_cols_b, HOST, column-major complex) = A' B for tall column-major device blocks with at most 96 columns
 * each: one fused launch.  With real vectors viewed as complex pairs the real part is the real Gram matrix -- the history
 * dot products of Anderson mixing (src/scf/anderson.jl:81-130) and of GMRES (LdosMixing, src/scf/mixing.jl:283). */
int dftk_b200_tall_gram(dftk_b200_ctx* ctx, const void* A, int64_t lda, int64_t n_cols_a, const void* B, int64_t ldb,
                        int64_t n_cols_b, int64_t n_rows, void* out_host);
/* C = alpha * op(A) * B + beta * C on complex128 column-major device arrays (own DMMA kernels);
 * transA: 0 = N, 2 = C (conjugate transpose) */
int dftk_b200_zgemm(dftk_b200_ctx* ctx, int transA, int64_t m, int64_t n, int64_t k,
                    const double* alpha2, const void* A, int64_t lda, const void* B, int64_t ldb,
                    const double* beta2, void* C, int64_t ldc);

/* ---- direct minimisation of the Kohn-Sham energy (src/scf/direct_minimization.jl).  Every call works on all listed
 * (k, spin) blocks of one context at once; block i holds n_bands orbitals of its k-block (n_pw_i x n_bands, column-major,
 * device).  Blocks of <= 32 bands take a fixed number of launches whatever their count.  Reductions are deterministic
 * (fixed-order two-stage sums, no floating-point atomics): identical inputs give bit-identical results. */
/* out[i] = scale[i] * H_i psi[i] (scale_host NULL: no scaling).  The scale is a separate elementwise pass over the outputs
 * after the H apply (one launch for all blocks), not folded into the H apply's own output write. */
int dftk_b200_apply_h_multi(int64_t n_blocks, dftk_b200_kblock* const* kblocks, const void* const* psi, void* const* out,
                            int64_t n_bands, const double* scale_host);
/* tangent projection onto the Stiefel manifold at X: G[i] -= X[i] (X[i]' G[i] + G[i]' X[i]) / 2 */
int dftk_b200_stiefel_project_multi(int64_t n_blocks, dftk_b200_kblock* const* kblocks, const void* const* X, void* const* G,
                                    int64_t n_bands);
/* polar retraction: X_out[i] = Y[i] (Y[i]' Y[i])^{-1/2}, from the eigendecomposition of the Gram matrix; X_out must not alias Y.
 * Returns DFTK_B200_ENUM when an eigensolve does not converge or a Gram matrix is not positive definite. */
int dftk_b200_stiefel_retract_multi(int64_t n_blocks, dftk_b200_kblock* const* kblocks, const void* const* Y, void* const* X_out,
                                    int64_t n_bands);
/* TPA preconditioner of the minimiser.  X non-NULL (precondprep!): mean_kin[i * n_bands + n] = sum_G kin_G |X[i]_Gn|^2.
 * Q non-NULL (ldiv!): S[i]_Gn = mean_kin[n] / (mean_kin[n] + kin_G) * Q[i]_Gn * inv_w[i].  use_tpa = 0: the identity,
 * S = Q * inv_w.  mean_kin: device, n_blocks x n_bands. */
int dftk_b200_tpa_multi(int64_t n_blocks, dftk_b200_kblock* const* kblocks, const void* const* X, const void* const* Q,
                        void* const* S, int64_t n_bands, const double* inv_w_host, int use_tpa, double* mean_kin);
/* out_host[p] = sum_i Re <A[p n_blocks + i], B[p n_blocks + i]> for p < n_pairs: two launches, one synchronisation */
int dftk_b200_real_dots_multi(int64_t n_pairs, int64_t n_blocks, dftk_b200_kblock* const* kblocks, const void* const* A,
                              const void* const* B, int64_t n_bands, double* out_host);
/* Y[i] += c X[i], then *out_host = sum_i Re <Z[i], Y[i]> in the same pass over memory (Z NULL: the update alone) */
int dftk_b200_axpy_dot_multi(int64_t n_blocks, dftk_b200_kblock* const* kblocks, void* const* Y, const void* const* X, double c,
                             const void* const* Z, int64_t n_bands, double* out_host);

/* ---- moving data between plane-wave bases (src/transfer.jl, apply_symop of src/symmetry.jl:229-270, src/supercell.jl,
 * src/interpolation.jl).  Orbital blocks are (n_bands, n_G) row-major complex128 device arrays (a band is a row); cubes are
 * linear with x fastest.  None of these calls reads the k-block or grid objects: they take plain device arrays. */
/* Tables of a sphere remap into a destination sphere of n_G integer vectors G (n_G x 3 int64, row-major, device):
 *   H_j = G_j + delta,  idx[j] = lookup[cube index of M H_j] (-1 when M H_j is outside the nx x ny x nz source cube),
 *   phase[j] = exp(-2 pi i H_j . tau)  (sincospi: rational tau with small denominators give exact +-1, +-i).
 * M: 3x3 row-major integers, delta: 3 integers, tau: 3 doubles (all host; tau may be NULL when phase is NULL).  lookup: the
 * source cube's nx*ny*nz int64 map cube index -> source row index, -1 outside the source sphere (device).  idx: n_G int64,
 * phase: n_G complex128 or NULL (device).  Users: transfer to an equivalent k-point (M = I, delta = the lattice vector between
 * the two k-points, tau = 0), apply_symop (M = S^-1, delta = the k shift that brings S k back to [-1/2, 1/2), tau), and
 * the unit cell -> supercell map (M = I on the supercell's integer coordinates of k+G). */
int dftk_b200_remap_tables(dftk_b200_ctx* ctx, int64_t n_G, const int64_t* G, const int32_t* M, const int32_t* delta,
                           const double* tau, const int64_t* lookup, int nx, int ny, int nz, int64_t* idx, void* phase);
/* Batched sphere remap, one launch for all n_pairs (source, destination) pairs (host arrays of n_pairs entries):
 *   dst[p][row_offset[p] + b, j] = phase[p][j] * src[p][b, idx[p][j]]   for b < n_bands[p], j < n_dst[p],
 * idx -1 giving 0 and a NULL phase (list or entry) giving 1.  ld_src / ld_dst: row lengths of the source and destination
 * blocks; row_offset NULL = 0 (several sources may fill disjoint row ranges of one destination).  Destinations must not
 * alias sources. */
int dftk_b200_sphere_remap(dftk_b200_ctx* ctx, int64_t n_pairs, const void* const* src, const int64_t* ld_src, void* const* dst,
                           const int64_t* ld_dst, const int64_t* row_offset, const int64_t* n_bands,
                           const int64_t* const* idx, const int64_t* n_dst, const void* const* phase);
/* Fourier block copy between cubes of different sizes (transfer_density; the blocks of transfer_mapping(basis_in, basis_out),
 * transfer.jl:10-31, including its placement of the unmatched component of even sizes); every other output entry is zero.
 * in: batch x (nx_in ny_in nz_in), out: batch x (nx_out ny_out nz_out), complex128 device. */
int dftk_b200_fourier_block_copy(dftk_b200_ctx* ctx, const void* in, int nx_in, int ny_in, int nz_in, void* out, int nx_out,
                                 int ny_out, int nz_out, int64_t batch);
/* Prefilter of the periodic quadratic B-spline (Interpolations.jl BSpline(Quadratic(Periodic(OnCell())))) on Fourier
 * coefficients, in place: f[b, m] /= prod_a (3/4 + cos(2 pi m_a / n_a) / 4)  (>= 1/8).  f: batch x N complex128 (device). */
int dftk_b200_bspline2_prefilter(dftk_b200_ctx* ctx, void* f, int nx, int ny, int nz, int64_t batch);
/* Evaluation of the periodic quadratic B-spline with coefficients f (batch x nx ny nz real, device) at the output points
 * (i/nx_out, j/ny_out, k/nz_out) of a cell spanning rep[a] input cells along axis a (rep: 3 host integers, 1 1 1 for the same
 * lattice): 27 taps per point, the tiling folded into the index arithmetic.  direct != 0 (needs n_out = rep * n_in on every
 * axis): f holds the samples themselves and out is their periodic tiling.  out: batch x (nx_out ny_out nz_out) real (device). */
int dftk_b200_bspline2_evaluate(dftk_b200_ctx* ctx, const double* f, int nx, int ny, int nz, const int32_t* rep, double* out,
                                int nx_out, int ny_out, int nz_out, int64_t batch, int direct);
/* Batched overlap products with an indirect right operand, one call for all n_pairs pairs (host arrays of n_pairs entries):
 *   C_p[m, n] = Σ_{j < n_G[p]} conj(A_p[m, j]) · B_p[n, idx_p[j]]   for m < n_a, n < n_b,
 * idx_p[j] = -1 contributing nothing and a NULL idx (list or entry) meaning idx_p[j] = j.  A_p: n_a rows of length ld_a[p]
 * (>= n_G[p]), B_p: n_b rows of length ld_b[p], complex128 (device), a band per row; idx_p: n_G[p] int64 (device), in range
 * [-1, ld_b[p]) by the caller's contract, as for sphere_remap.  C: n_pairs column-major n_a × n_b matrices (device).  The
 * Wannier90 overlaps M^{k,b} (A = ψ_k, B = ψ_{k+b}, idx from remap_tables with M = I and delta = G_shift) and projections A_k
 * (B = the projection table of k, idx NULL, src/external/wannier_shared.jl).  Up to 32 columns: a fused gather-product in two
 * launches whatever the pair count; consecutive pairs with the same A (pointer, ld_a, n_G) read A once; fixed-order sums, so a
 * rerun is bit-identical.  Larger blocks: per pair a gather into scratch and the DMMA ZGEMM. */
int dftk_b200_overlap_multi(dftk_b200_ctx* ctx, int64_t n_pairs, int64_t n_a, int64_t n_b, const void* const* A,
                            const int64_t* ld_a, const int64_t* n_G, const void* const* B, const int64_t* ld_b,
                            const int64_t* const* idx, void* C);

#ifdef __cplusplus
}
#endif
#endif
