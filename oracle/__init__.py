"""CPU oracle: a NumPy restatement of DFTK.jl's CPU algorithm for the plane-wave
Kohn-Sham SCF hot path (Hψ apply, LOBPCG, compute_density, SCF plumbing).

THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only `tests/`, `__graft_entry__.smoke()`
and the `cpu_baseline` / `--impl reference` legs of `bench.py` may import it.  The product
package (`dftk.jl_b200/`, importable as `dftk_b200`) never imports anything from here and
fails loudly if its CUDA library is missing.

Why a restatement: the reference is pure Julia and `julia` is not installed in the build
or measurement containers (no network), so the reference itself cannot be imported or
compiled.  Every function cites the reference file:line it follows (paths relative to
the DFTK.jl tree).  Parity pins (all checked in tests/test_oracle_golden.py):
  * test/PspHgh.jl:41-84           HGH local / projector Fourier values
  * test/energy_nuclear.jl:31,48   Ewald, psp correction (ABINIT numbers)
  * test/compute_fft_size.jl:6-12  FFT grid sizes
  * test/fourier_transforms.jl     FFT round trips / explicit DFT matrices
  * test/lobpcg.jl:13-22,63-103    free-electron, kinetic+local(+nonlocal) eigenvalues
  * test/energies_guess_density.jl:8-36   every energy term of LDA silicon to 5e-8
  * test/silicon_lda.jl:10-20      full SCF vs ABINIT eigenvalues / total energy
Third-party arithmetic restated from published formulas (not in the DFTK.jl tree):
libxc (lda_x, lda_c_vwn, lda_c_pw, gga_x_pbe, gga_c_pbe), pinned through the energy
values above; spglib is avoided (symmetries found by brute force over lattice isometries).
"""
