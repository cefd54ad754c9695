// Host emulation of the LDOS product (TEST INFRASTRUCTURE ONLY): k_ldos_product of ldos.cu runs CTA by CTA on the body of
// ldos_core.cuh, with the device's tiles and the MMA evaluated from the fragments of all 32 lanes of a warp.
#include <cstdint>
#include <vector>
#include "../../dftk.jl_b200/csrc/ldos_core.cuh"

using namespace dftk;

extern "C" {
// C[j ldc + r] += Σ_k D[k][r] W[k][j ldw] for r < M, j < n, k < K.  D, W: K pointers each (host).
void emu_ldos(int K, const double* const* D, const double* const* W, long long ldw, long long M, int n, double* C, long long ldc) {
  LdosProduct p{D, W, ldw, K, M, n, C, ldc};
  std::vector<double> sm(LD_SMEM_DOUBLES), acc(2 * 4 * LD_SLOTS * 4);
  for (long long bm = 0; bm < (M + LD_TM - 1) / LD_TM; ++bm)
    for (int bn = 0; bn < (n + LD_TN - 1) / LD_TN; ++bn) ldos_cta(p, bm, bn, sm.data(), acc.data());
}
}
