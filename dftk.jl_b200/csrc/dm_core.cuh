// Kernel bodies of the direct minimisation (dm.cu): the tall-block vector operations of a Riemannian L-BFGS over all
// (k, spin) blocks of a rank.  Every reduction is deterministic: a fixed grid-stride split into chunks, a fixed-shape tree
// inside a chunk, and a sequential sum over (block, chunk) in index order; no floating-point atomics.  The line search
// takes discrete decisions on these sums, so identical inputs must give bit-identical results.
#pragma once
#include "fft_core.cuh"

namespace dftk {

#define DM_THREADS 256       // CTA size of the chunk kernels
#define DM_MAX_CHUNKS 1024   // chunks per block item (the grid's x extent)

// One block of one reduction: optionally y += c x first (x != nullptr), then Re<a, b> over len complex entries.
// a == nullptr: no dot product (the update alone).
struct DmDotItem {
  const cplx* a;
  const cplx* b;
  cplx* y;
  const cplx* x;
  double c;
  long long len;
};

// Per-thread partial of chunk `chunk` of `n_chunks`: entries chunk*T + t, stepping by n_chunks*T.
HD double dm_chunk_partial(const DmDotItem& it, int chunk, int n_chunks, int t) {
  double s = 0.0;
  for (long long i = (long long)chunk * DM_THREADS + t; i < it.len; i += (long long)n_chunks * DM_THREADS) {
    if (it.x) {
      const cplx u = it.x[i];
      cplx v = it.y[i];
      v.x += it.c * u.x;
      v.y += it.c * u.y;
      it.y[i] = v;
    }
    if (it.a) {
      const cplx p = it.a[i], q = it.b[i];
      s += p.x * q.x + p.y * q.y;
    }
  }
  return s;
}

// Fixed-shape tree over the DM_THREADS per-thread partials held in `red` (in place; result in red[0]).
HD void dm_tree_step(double* red, int t, int width) {
  if (t < width) red[t] += red[t + width];
}

// Sum over the items [first, first + n_items) of a pair and all their chunks, in index order.
HD double dm_final_sum(const double* ws, int first, int n_items, int n_chunks) {
  double s = 0.0;
  for (int i = first; i < first + n_items; ++i)
    for (int c = 0; c < n_chunks; ++c) s += ws[(long long)i * n_chunks + c];
  return s;
}

// TPA of one (row, band): s = mk / (mk + kin) q * inv_w   (preconditioners.jl:75-77, direct_minimization.jl:39-47);
// mk < 0 marks the identity preconditioner.
HD cplx dm_tpa_entry(cplx q, double kin, double mk, double inv_w) {
  const double f = (mk < 0.0 ? 1.0 : mk / (mk + kin)) * inv_w;
  return make_double2(f * q.x, f * q.y);
}

// Small n x n operations of the Stiefel projection and the polar retraction (column-major, leading dimension n).
// M = (C + C^H) / 2
HD cplx dm_herm_entry(const cplx* C, int n, int i, int j) {
  const cplx a = C[i + n * j], b = C[j + n * i];
  return make_double2(0.5 * (a.x + b.x), 0.5 * (a.y - b.y));
}
// S = V diag(f) V^H with f = w^{-1/2} precomputed
HD cplx dm_invsqrt_entry(const cplx* V, const double* f, int n, int i, int j) {
  double sx = 0.0, sy = 0.0;
  for (int l = 0; l < n; ++l) {
    const cplx a = V[i + n * l], b = V[j + n * l];     // a conj(b)
    sx += f[l] * (a.x * b.x + a.y * b.y);
    sy += f[l] * (a.y * b.x - a.x * b.y);
  }
  return make_double2(sx, sy);
}
// A = diag(w^{-1/4}) V^H, so that A^H A = V diag(w^{-1/2}) V^H (the large-block path takes that product on the GEMMs)
HD cplx dm_scaled_adjoint_entry(const cplx* V, const double* w, int n, int l, int j) {
  const double f = 1.0 / sqrt(sqrt(w[l]));
  const cplx v = V[j + n * l];
  return make_double2(f * v.x, -f * v.y);
}

}  // namespace dftk
