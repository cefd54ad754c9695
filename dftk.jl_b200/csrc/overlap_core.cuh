// Kernel bodies of the batched overlap product with an indirect right operand (overlap.cu; the Wannier90 overlap and
// projection matrices, reference seam src/external/wannier_shared.jl overlap_Mmn_k_kpb / compute_amn_kpoint):
//   C_p[m, n] = Σ_j conj(A_p[m, j]) B_p[n, idx_p[j]]     (idx_p[j] < 0: nothing; idx_p NULL: j itself)
// for blocks of at most SMALL_MAX_N columns.  A CTA owns one row chunk of one group of pairs that share their A: it holds
// OV_ROWS rows of A in shared memory and runs every pair of the group over them, so A is read once per group.  The B rows are
// gathered through idx into a shared tile (the gathered block is never materialised).  Every reduction has a fixed order: a
// thread sums its rows in ascending order, the row lanes of an output are added in lane order, the sub-chunks of a chunk in
// row order, and the chunks in index order by a second launch; no floating-point atomics, so a rerun is bit-identical.
// Host-callable: tests/hostemu runs the CTAs one after the other with TLOOP as a sequential loop (no register state is live
// across a TSYNC).
#pragma once
#include "fft_core.cuh"

namespace dftk {

#define OV_THREADS 256    // CTA size; n_a * ceil(n_b / 4) <= 32 * 8 output tiles fit one per thread
#define OV_ROWS 64        // rows of A held in shared memory at a time (a sub-chunk)
#define OV_TR 16          // rows of B gathered per shared tile
#define OV_MAX_CHUNKS 64  // row chunks per group at most: the partials need n_chunks * n_pairs * n_a * n_b entries

struct OvGroup {          // consecutive pairs [first, first + count) with the same A
  const cplx* A;
  long long ld_a, n_G;    // A: n_a rows (bands) of length ld_a; the product runs over j < n_G
  int first, count;
};
struct OvPair {
  const cplx* B;
  long long ld_b;
  const long long* idx;   // n_G entries of the group, or NULL (identity)
};

// dynamic shared memory of one CTA, in complex entries: A sub-chunk, B tile, per-thread accumulators (4 outputs each)
HD long long ov_smem_entries(int n_a, int n_b) { return (long long)OV_ROWS * n_a + (long long)OV_TR * n_b + 4LL * OV_THREADS; }

// CTA (group g, chunk `chunk` of n_chunks): writes ws[(chunk * n_pairs + p) * n_a n_b + i + n_a j] for every pair p of g.
HD void ov_cta(const OvGroup& g, const OvPair* __restrict__ pairs, int chunk, int n_chunks, int n_a, int n_b, int n_threads,
               long long n_pairs, cplx* __restrict__ ws, cplx* sm) {
  const int nab = n_a * n_b, n_tiles = n_a * ((n_b + 3) / 4), n_lanes = n_threads / n_tiles;
  const long long rpc = (g.n_G + n_chunks - 1) / n_chunks;
  const long long c0 = (long long)chunk * rpc, c1 = c0 + rpc < g.n_G ? c0 + rpc : g.n_G;
  cplx* As = sm;
  cplx* Bs = sm + (long long)OV_ROWS * n_a;
  cplx* acc = Bs + (long long)OV_TR * n_b;
  if (c0 >= c1) {                      // an empty chunk still owns its partials
    for (int q = 0; q < g.count; ++q) {
      cplx* out = ws + ((long long)chunk * n_pairs + g.first + q) * nab;
      TLOOP(o, nab) out[o] = make_double2(0.0, 0.0);
    }
    return;
  }
  for (long long s0 = c0; s0 < c1; s0 += OV_ROWS) {
    const int ns = (int)(c1 - s0 < OV_ROWS ? c1 - s0 : OV_ROWS);
    TSYNC();
    TLOOP(e, OV_ROWS * n_a) {
      const int r = e % OV_ROWS, i = e / OV_ROWS;
      As[r * n_a + i] = r < ns ? g.A[i * g.ld_a + s0 + r] : make_double2(0.0, 0.0);
    }
    for (int q = 0; q < g.count; ++q) {
      const OvPair pr = pairs[g.first + q];
      TSYNC();
      TLOOP(t, 4 * n_threads) acc[t] = make_double2(0.0, 0.0);
      for (int t0 = 0; t0 < ns; t0 += OV_TR) {
        const int nr = ns - t0 < OV_TR ? ns - t0 : OV_TR;
        TSYNC();
        TLOOP(e, OV_TR * n_b) {
          const int r = e % OV_TR, j = e / OV_TR;
          cplx v = make_double2(0.0, 0.0);
          if (r < nr) {
            const long long row = s0 + t0 + r;
            const long long src = pr.idx ? pr.idx[row] : row;
            if (src >= 0) v = pr.B[j * pr.ld_b + src];
          }
          Bs[r * n_b + j] = v;
        }
        TSYNC();
        // thread t: output tile t % n_tiles (row i, columns j0 .. j0 + 3 of C), rows lane, lane + n_lanes, ... of the tile
        TLOOP(t, n_threads) {
          const int tile = t % n_tiles, lane = t / n_tiles;
          if (lane < n_lanes) {
            const int i = tile % n_a, j0 = (tile / n_a) * 4;
            int jq[4];
            for (int c = 0; c < 4; ++c) jq[c] = j0 + c < n_b ? j0 + c : n_b - 1;   // clamped columns are dropped below
            double ax[4] = {0.0, 0.0, 0.0, 0.0}, ay[4] = {0.0, 0.0, 0.0, 0.0};
            for (int r = lane; r < nr; r += n_lanes) {
              const cplx a = As[(t0 + r) * n_a + i];
              const cplx* brow = Bs + r * n_b;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
              for (int c = 0; c < 4; ++c) {
                const cplx b = brow[jq[c]];
                ax[c] += a.x * b.x + a.y * b.y;     // conj(a) * b
                ay[c] += a.x * b.y - a.y * b.x;
              }
            }
            for (int c = 0; c < 4; ++c) {
              acc[4 * t + c].x += ax[c];
              acc[4 * t + c].y += ay[c];
            }
          }
        }
      }
      TSYNC();
      cplx* out = ws + ((long long)chunk * n_pairs + g.first + q) * nab;
      TLOOP(o, nab) {
        const int i = o % n_a, j = o / n_a, tile = i + n_a * (j / 4), c = j % 4;
        double sx = 0.0, sy = 0.0;
        for (int l = 0; l < n_lanes; ++l) {
          const cplx v = acc[4 * (l * n_tiles + tile) + c];
          sx += v.x;
          sy += v.y;
        }
        if (s0 == c0) {
          out[o] = make_double2(sx, sy);
        } else {
          out[o].x += sx;
          out[o].y += sy;
        }
      }
    }
  }
}

// C entry (pair p, o = i + n_a j): the chunk partials in index order.
HD cplx ov_reduce_entry(const cplx* __restrict__ ws, int n_chunks, long long n_pairs, int nab, long long p, int o) {
  double sx = 0.0, sy = 0.0;
  for (int c = 0; c < n_chunks; ++c) {
    const cplx v = ws[((long long)c * n_pairs + p) * nab + o];
    sx += v.x;
    sy += v.y;
  }
  return make_double2(sx, sy);
}

}  // namespace dftk
