// Host emulation of the direct-minimisation reductions (TEST INFRASTRUCTURE ONLY): k_dm_dot_partial and k_dm_dot_final of
// dm.cu run CTA by CTA and thread by thread on the bodies of dm_core.cuh, with the device's grid geometry.
#include <algorithm>
#include <cstdint>
#include <vector>
#include "../../dftk.jl_b200/csrc/dm_core.cuh"

using namespace dftk;

extern "C" {
// For each block i: y_i += c x_i (x NULL: no update), then out = sum_i Re<z_i, y_i> (z NULL: no dot, out = 0).
// Arrays are interleaved (re, im) doubles of len[i] complex entries.  Returns the chunk count used.
int emu_dm_axpy_dot(int n_blocks, const int64_t* len, double* const* y, const double* const* x, const double* const* z, double c,
                    double* out) {
  std::vector<DmDotItem> items;
  long long max_len = 1;
  for (int i = 0; i < n_blocks; ++i) {
    items.push_back(DmDotItem{z ? (const cplx*)z[i] : nullptr, (const cplx*)y[i], (cplx*)y[i], x ? (const cplx*)x[i] : nullptr,
                              c, (long long)len[i]});
    max_len = std::max<long long>(max_len, len[i]);
  }
  const int n_chunks = (int)std::min<long long>(DM_MAX_CHUNKS, (max_len + DM_THREADS - 1) / DM_THREADS);
  std::vector<double> ws((size_t)n_blocks * n_chunks), red(DM_THREADS);
  for (int b = 0; b < n_blocks; ++b)
    for (int ch = 0; ch < n_chunks; ++ch) {
      for (int t = 0; t < DM_THREADS; ++t) red[t] = dm_chunk_partial(items[b], ch, n_chunks, t);
      for (int w = DM_THREADS / 2; w > 0; w >>= 1)
        for (int t = 0; t < DM_THREADS; ++t) dm_tree_step(red.data(), t, w);
      ws[(size_t)b * n_chunks + ch] = red[0];
    }
  *out = z ? dm_final_sum(ws.data(), 0, n_blocks, n_chunks) : 0.0;
  return n_chunks;
}
}
