// Host emulation of the basis-transfer kernels (TEST INFRASTRUCTURE ONLY): the per-entry bodies of transfer_core.cuh run in a
// sequential loop over the entries each device thread computes in transfer.cu.
#include <cstdint>
#include "../../dftk.jl_b200/csrc/transfer_core.cuh"

using namespace dftk;

extern "C" {
// k_remap_tables: idx (n) and phase (n complex as (re, im) pairs, NULL: not written)
void emu_tr_tables(int64_t n, const int64_t* G, const int* M, const int* delta, const double* tau, const int64_t* lookup, int nx,
                   int ny, int nz, int64_t* idx, double* phase) {
  for (long long j = 0; j < n; ++j)
    tr_table_entry(j, (const long long*)G, M, delta, tau, (const long long*)lookup, nx, ny, nz, (long long*)idx, (cplx*)phase);
}
// k_sphere_remap for one pair
void emu_tr_remap(int64_t n_bands, const double* src, int64_t ld_src, double* dst, int64_t ld_dst, int64_t row_offset,
                  int64_t n_dst, const int64_t* idx, const double* phase) {
  for (long long j = 0; j < n_dst; ++j)
    for (long long b = 0; b < n_bands; ++b)
      ((cplx*)dst)[(row_offset + b) * ld_dst + j] = tr_remap_value((const cplx*)src + b * ld_src, idx[j], (const cplx*)phase, j);
}
// k_block_copy
void emu_tr_block_copy(const double* in, int nxi, int nyi, int nzi, double* out, int nxo, int nyo, int nzo, int64_t batch) {
  const long long Ni = (long long)nxi * nyi * nzi, No = (long long)nxo * nyo * nzo;
  for (long long b = 0; b < batch; ++b)
    for (long long o = 0; o < No; ++o)
      ((cplx*)out)[b * No + o] = tr_block_copy_value(o, (const cplx*)in + b * Ni, nxi, nyi, nzi, nxo, nyo, nzo);
}
// the factor k_bspline_prefilter multiplies each Fourier entry by
void emu_tr_prefilter_factor(int nx, int ny, int nz, double* out) {
  for (long long i = 0; i < (long long)nx * ny * nz; ++i) out[i] = tr_bspline_prefilter_factor(i, nx, ny, nz);
}
// k_bspline_eval for one spin channel
void emu_tr_bspline(const double* f, int nx, int ny, int nz, const int* rep, double* out, int nxo, int nyo, int nzo, int direct) {
  for (long long o = 0; o < (long long)nxo * nyo * nzo; ++o) out[o] = tr_bspline_value(o, f, nx, ny, nz, rep, nxo, nyo, nzo, direct);
}
}
