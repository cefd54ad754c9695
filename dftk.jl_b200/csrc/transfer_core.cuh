// Kernel bodies of the basis transfers (transfer.cu): index/phase tables of the sphere remap, the remap itself, the Fourier
// block copy between cubes of different sizes and the periodic quadratic B-spline.  Host-callable so that tests/hostemu can
// run them sequentially.  Cubes are linear with x fastest: index = ix + nx (iy + ny iz).
#pragma once
#include <math.h>
#include "fft_core.cuh"

namespace dftk {

// Cube index of the integer frequency (g0, g1, g2) on an (nx, ny, nz) cube, or -1 when it lies outside the FFT box
// (index_G_vectors, PlaneWaveBasis.jl:465-480).
HD long long tr_cube_index(long long g0, long long g1, long long g2, int nx, int ny, int nz) {
  const long long g[3] = {g0, g1, g2};
  const int n[3] = {nx, ny, nz};
  long long j[3];
  for (int a = 0; a < 3; ++a) {
    if (g[a] < -(n[a] / 2) || g[a] > (n[a] - 1) / 2) return -1;
    j[a] = g[a] < 0 ? g[a] + n[a] : g[a];
  }
  return j[0] + (long long)nx * (j[1] + (long long)ny * j[2]);
}

// Table entry j of a sphere remap: H = G_j + delta, idx = lookup[cube index of M H] (-1 outside the source cube or sphere),
// phase = exp(-2 pi i H.tau), computed with sincospi so that rational tau with small denominators give exact +-1, +-i.
// G: n x 3 row-major; M: 3 x 3 row-major.  phase may be NULL.
HD void tr_table_entry(long long j, const long long* G, const int* M, const int* delta, const double* tau,
                       const long long* lookup, int nx, int ny, int nz, long long* idx, cplx* phase) {
  const long long H[3] = {G[3 * j] + delta[0], G[3 * j + 1] + delta[1], G[3 * j + 2] + delta[2]};
  long long g[3];
  for (int a = 0; a < 3; ++a) g[a] = M[3 * a] * H[0] + M[3 * a + 1] * H[1] + M[3 * a + 2] * H[2];
  const long long c = tr_cube_index(g[0], g[1], g[2], nx, ny, nz);
  idx[j] = c < 0 ? -1 : lookup[c];
  if (phase) {
    double s, co;
    sincospi(-2.0 * ((double)H[0] * tau[0] + (double)H[1] * tau[1] + (double)H[2] * tau[2]), &s, &co);
    phase[j] = make_double2(co, s);
  }
}

// One entry of the remap dst[b, j] = phase[j] src[b, idx[j]] (idx < 0: 0; phase NULL: 1); src_row = &src[b, 0].
HD cplx tr_remap_value(const cplx* src_row, long long i, const cplx* phase, long long j) {
  if (i < 0) return make_double2(0.0, 0.0);
  const cplx v = src_row[i];
  if (!phase) return v;
  const cplx p = phase[j];
  return make_double2(p.x * v.x - p.y * v.y, p.x * v.y + p.y * v.x);
}

// Per axis, the source index of output index o in the Fourier block copy of transfer_mapping(basis_in, basis_out)
// (transfer.jl:10-31), or -1 when o is not matched.  Growing: the ceil(n_in/2) non-negative and floor(n_in/2) negative
// frequencies of the input keep their frequency (an even input's unmatched -n_in/2 lands on -n_in/2).  Shrinking: the output's
// ceil(n_out/2) leading and floor(n_out/2) trailing entries come from the input's leading and trailing ones.
HD int tr_block_axis(int o, int n_in, int n_out) {
  if (n_in <= n_out) {
    const int a = (n_in + 1) / 2, b = n_in / 2;
    if (o < a) return o;
    if (o >= n_out - b) return o - n_out + n_in;
    return -1;
  }
  const int a = (n_out + 1) / 2;
  return o < a ? o : o + n_in - n_out;
}

// Output entry `o` (linear, one cube) of the block copy from the (nxi, nyi, nzi) cube `in`.
HD cplx tr_block_copy_value(long long o, const cplx* in, int nxi, int nyi, int nzi, int nxo, int nyo, int nzo) {
  const int ox = (int)(o % nxo), oy = (int)((o / nxo) % nyo), oz = (int)(o / ((long long)nxo * nyo));
  const int ix = tr_block_axis(ox, nxi, nxo), iy = tr_block_axis(oy, nyi, nyo), iz = tr_block_axis(oz, nzi, nzo);
  if (ix < 0 || iy < 0 || iz < 0) return make_double2(0.0, 0.0);
  return in[ix + (long long)nxi * (iy + (long long)nyi * iz)];
}

// 1 / prod_a (3/4 + cos(2 pi m_a / n_a) / 4): the inverse symbol of the periodic quadratic B-spline's sampling at the nodes
// (1/8, 3/4, 1/8).  The symbol is at least 1/2 per axis, 1/8 over three axes, so the division is always safe.
HD double tr_bspline_prefilter_factor(long long i, int nx, int ny, int nz) {
  const int ix = (int)(i % nx), iy = (int)((i / nx) % ny), iz = (int)(i / ((long long)nx * ny));
  const int id[3] = {ix, iy, iz}, n[3] = {nx, ny, nz};
  double s = 1.0;
  for (int a = 0; a < 3; ++a) s *= 0.75 + 0.25 * cospi(2.0 * (double)id[a] / (double)n[a]);
  return 1.0 / s;
}

// Nearest node and the three weights of the quadratic B-spline at position i * num / den in units of the input grid
// (t = x - nearest in [-1/2, 1/2]: (1/2 - t)^2 / 2, 3/4 - t^2, (1/2 + t)^2 / 2 for nodes nearest - 1, nearest, nearest + 1).
HD long long tr_bspline_axis(long long i, long long num, long long den, double* w) {
  const long long p = i * num;
  const long long q = (2 * p + den) / (2 * den);     // round half up
  const double t = (double)(p - q * den) / (double)den;
  w[0] = 0.5 * (0.5 - t) * (0.5 - t);
  w[1] = 0.75 - t * t;
  w[2] = 0.5 * (0.5 + t) * (0.5 + t);
  return q;
}

HD int tr_wrap(long long j, int n) {
  const long long r = j % n;
  return (int)(r < 0 ? r + n : r);
}

// Output point o (linear on the (nxo, nyo, nzo) cube) of interpolate_density: the output point r = (ox/nxo, oy/nyo, oz/nzo)
// of the output cell, which spans rep[a] input cells along axis a, lies at r_a rep_a n_a in units of the periodic input grid
// (the tiled supercell is never formed).  direct != 0: the point falls on an input node on every axis (n_a rep_a == n_out_a);
// f is then sampled there.  Otherwise f holds the B-spline coefficients and the 27 taps are summed.
HD double tr_bspline_value(long long o, const double* f, int nx, int ny, int nz, const int* rep, int nxo, int nyo, int nzo,
                           int direct) {
  const long long oi[3] = {o % nxo, (o / nxo) % nyo, o / ((long long)nxo * nyo)};
  const int n[3] = {nx, ny, nz}, no[3] = {nxo, nyo, nzo};
  if (direct) {
    int j[3];
    for (int a = 0; a < 3; ++a) j[a] = tr_wrap(oi[a], n[a]);
    return f[j[0] + (long long)nx * (j[1] + (long long)ny * j[2])];
  }
  double w[3][3];
  long long q[3];
  for (int a = 0; a < 3; ++a) q[a] = tr_bspline_axis(oi[a], (long long)n[a] * rep[a], no[a], w[a]);
  double s = 0.0;
  for (int c = 0; c < 3; ++c) {
    const long long zoff = (long long)nx * ny * tr_wrap(q[2] + c - 1, nz);
    double sy = 0.0;
    for (int b = 0; b < 3; ++b) {
      const double* row = f + zoff + (long long)nx * tr_wrap(q[1] + b - 1, ny);
      double sx = 0.0;
      for (int a = 0; a < 3; ++a) sx += w[0][a] * row[tr_wrap(q[0] + a - 1, nx)];
      sy += w[1][b] * sx;
    }
    s += w[2][c] * sy;
  }
  return s;
}

}  // namespace dftk
