// Host emulation of the batched overlap product (TEST INFRASTRUCTURE ONLY): k_ov_partial and k_ov_reduce of overlap.cu run
// CTA by CTA on the bodies of overlap_core.cuh, with the device's CTA size and the pair grouping of dftk_b200_overlap_multi.
#include <cstdint>
#include <vector>
#include "../../dftk.jl_b200/csrc/overlap_core.cuh"

using namespace dftk;

extern "C" {
// C (n_pairs column-major n_a x n_b, (re, im) pairs) = A_p^H B_p[idx_p] for n_a, n_b <= 32 with n_chunks row chunks per group.
// A, B: (re, im) interleaved blocks; idx: list of n_G[p] int64 entries or NULL entries (identity), or a NULL list.
// Returns the number of groups (runs of consecutive pairs with the same A, ld_a and n_G).
int emu_overlap(int64_t n_pairs, int n_a, int n_b, const double* const* A, const int64_t* ld_a, const int64_t* n_G,
                const double* const* B, const int64_t* ld_b, const int64_t* const* idx, int n_chunks, double* C) {
  std::vector<OvGroup> groups;
  std::vector<OvPair> pairs;
  for (int64_t p = 0; p < n_pairs; ++p) {
    pairs.push_back(OvPair{(const cplx*)B[p], (long long)ld_b[p], idx ? (const long long*)idx[p] : nullptr});
    if (!groups.empty() && groups.back().A == (const cplx*)A[p] && groups.back().ld_a == ld_a[p] && groups.back().n_G == n_G[p])
      groups.back().count++;
    else
      groups.push_back(OvGroup{(const cplx*)A[p], (long long)ld_a[p], (long long)n_G[p], (int)p, 1});
  }
  const int nab = n_a * n_b;
  std::vector<cplx> ws((size_t)n_chunks * n_pairs * nab), sm((size_t)ov_smem_entries(n_a, n_b));
  for (const OvGroup& g : groups)
    for (int c = 0; c < n_chunks; ++c) ov_cta(g, pairs.data(), c, n_chunks, n_a, n_b, OV_THREADS, n_pairs, ws.data(), sm.data());
  for (long long e = 0; e < (long long)n_pairs * nab; ++e)
    ((cplx*)C)[e] = ov_reduce_entry(ws.data(), n_chunks, n_pairs, nab, e / nab, (int)(e % nab));
  return (int)groups.size();
}
}
