// Register-resident two-pass ("four-step") 1D FFT stages of the pruned sphere<->cube pipeline.
//
// An axis of length n = A*B is transformed in two passes with ONE shared-memory exchange:
//   pass 1 (B threads per line, thread q holds the A elements q + B r):  Y[c] = DFT_A over r, times W_n^{qc}
//   exchange through shared memory S[c*B + q]
//   pass 2 (A threads per line, thread c holds S[c*B + q], q < B):       X[c + A d] = DFT_B over q
// The butterflies are generated straight-line code (fft_radix_gen.cuh).  Compared with the generic
// Stockham engine (fft_core.cuh, kept as the fallback for sizes without a factor pair) this moves 32 B per
// element per transform through shared memory instead of ~160 B and does no per-butterfly index division.
//
// Global memory goes straight to/from registers for the strided axes (y, z): consecutive threads are
// consecutive x (the contiguous dimension), so every access is a 16-lane * 16 B = 256 B segment.
// The contiguous axis (x) is transposed through shared memory on the way in/out.
//
// Bodies are __host__ __device__ with TLOOP/TSYNC like fft_core.cuh so tests/hostemu can run them.
// Contract on the device: blockDim.x == L * max(A, B); no register state is live across a TSYNC.
#pragma once
#include "fft_core.cuh"
#include "fft_reg_fwd.cuh"
#include "fft_radix_gen.cuh"

namespace dftk {

template <int A, int B>
struct RegPair {
  static constexpr int n = A * B;
  static constexpr int T = (A > B ? A : B);
  // lines per CTA: about 128 threads per CTA (more independent CTAs per SM overlap the load / exchange / store
  // phases better); compile-time so that every shared-memory offset folds into an immediate
  static constexpr int L = (T >= 12 ? 8 : (T >= 5 ? 16 : 32));
  static constexpr int Lp = L + 1;
};

// thread q (< B) holds x[r] = element q + B*r; writes twiddled DFT_A to S[(c*B + q)]
template <int A, int B, int S>
HD void pass1_store(const cplx* x, int q, int line, cplx* __restrict__ Sbuf, int Lp,
                    const cplx* __restrict__ tw) {
  cplx Y[A];
  dft_r<A, S>(x, Y);
#pragma unroll
  for (int c = 0; c < A; ++c) {
    cplx v = Y[c];
    if (c != 0 && q != 0) v = cmul(v, twiddle(tw, q * c, S));
    Sbuf[(c * B + q) * Lp + line] = v;
  }
}
// thread c (< A) loads S[(c*B + q)], q < B; X[d] = element c + A*d
template <int A, int B, int S>
HD void pass2_load(cplx* X, int c, int line, const cplx* __restrict__ Sbuf, int Lp) {
  cplx t[B];
#pragma unroll
  for (int q = 0; q < B; ++q) t[q] = Sbuf[(c * B + q) * Lp + line];
  dft_r<B, S>(t, X);
}

// ---------------------------------------------------------------------------------------------- z stages
// compute-only half of pass 1 (the caller stores Y[c] to S[(c*B + q)])
template <int A, int B, int S>
HD void pass1_compute(const cplx* x, int q, const cplx* __restrict__ tw, cplx* Y) {
  dft_r<A, S>(x, Y);
#pragma unroll
  for (int c = 1; c < A; ++c)
    if (q != 0) Y[c] = cmul(Y[c], twiddle(tw, q * c, S));
}

// On the device the two exchange buffers of the fused z stage alias (one buffer, an extra barrier between the
// last read and the first write), halving the shared-memory footprint; the host emulation keeps two buffers.
#if defined(__CUDA_ARCH__)
#define DFTK_Z_ALIAS 1
#else
#define DFTK_Z_ALIAS 0
#endif

template <int A, int B>
HD void reg_z_apply_potential(const SphereTablesX& T, const cplx* __restrict__ tw, cplx* __restrict__ W2,
                              const double* __restrict__ V, int L_rt, int Lp_rt, cplx* sm, Dim3i bid) {
  constexpr int n = A * B, TT = RegPair<A, B>::T, L = RegPair<A, B>::L, Lp = RegPair<A, B>::Lp;
  (void)L_rt;
  (void)Lp_rt;
  const int nx = T.nx, ny = T.ny;
  cplx* bufA = sm;
  cplx* bufB = DFTK_Z_ALIAS ? sm : sm + (size_t)n * Lp;
  const int x0 = bid.x * L, y = bid.y;
  cplx* w2 = W2 + (size_t)bid.z * T.n_zc * ny * nx;
  const uint64_t pol_keep = l2_policy_evict_last(), pol_stream = l2_policy_evict_first();
  TLOOP(t, L * TT) {
    const int line = t % L, p = t / L, x = x0 + line;
    if (p < B) {
      cplx v[A];
#pragma unroll
      for (int r = 0; r < A; ++r) {
        int zc = zc_index(T, p + B * r);
        v[r] = ld_pred_hint(w2 + (unsigned)(((zc < 0 ? 0 : zc) * ny + y) * nx + x), zc >= 0 && x < nx, pol_stream);
      }
      pass1_store<A, B, +1>(v, p, line, bufA, Lp, tw);
    }
  }
  TSYNC();
  TLOOP(t, L * TT) {
    const int line = t % L, p = t / L, x = x0 + line;
    cplx Y[B];
    if (p < A) {
      cplx X[B];
      pass2_load<A, B, +1>(X, p, line, bufA, Lp);
#pragma unroll
      for (int d = 0; d < B; ++d) {
        double vv = ld_pred_hint(V + (unsigned)(((p + A * d) * ny + y) * nx + x), x < nx, pol_keep);
        X[d] = cscale(X[d], vv);
      }
      // forward transform of the elements p + A*d: pass 1 with the roles of A and B swapped
      pass1_compute<B, A, -1>(X, p, tw, Y);
    }
#if DFTK_Z_ALIAS
    __syncthreads();   // every thread of the CTA runs this body exactly once (blockDim == L*TT)
#endif
    if (p < A) {
#pragma unroll
      for (int c = 0; c < B; ++c) bufB[(c * A + p) * Lp + line] = Y[c];
    }
  }
  TSYNC();
  TLOOP(t, L * TT) {
    const int line = t % L, p = t / L, x = x0 + line;
    if (p < B) {
      cplx X[A];
      pass2_load<B, A, -1>(X, p, line, bufB, Lp);
#pragma unroll
      for (int f = 0; f < A; ++f) {
        int zc = zc_index(T, p + B * f);
        st_pred_hint(w2 + (unsigned)(((zc < 0 ? 0 : zc) * ny + y) * nx + x), X[f], zc >= 0 && x < nx, pol_stream);
      }
    }
  }
}

#if defined(__CUDACC__)
// ---- software-pipelined form of the fused z stage (device only).  The plain kernel above is latency bound: one tile per
// CTA, 12 dependent-free global loads per thread, then nothing to do until they land (ncu: 24 % warps active, top stall
// long-scoreboard).  Here a CTA is persistent over tiles (x-tile, y, band) and the pruned input column block of tile i+1
// (n_zc rows of L complex numbers, 12 KB at 192^3) travels global -> shared with cp.async while the butterflies of tile i
// run; pass 1 then reads its A elements from shared memory.  V(r) (L2 resident, evict-last) and the stores are unchanged.
__device__ __forceinline__ void zp_cp_async16(void* smem, const void* gmem, bool pred) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  int sz = pred ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(sz));
}
template <int A, int B>
__device__ void reg_z_apply_potential_pipe(const SphereTablesX& T, const cplx* __restrict__ tw, cplx* __restrict__ W2,
                                           const double* __restrict__ V, cplx* sm, int n_bands) {
  constexpr int n = A * B, TT = RegPair<A, B>::T, L = RegPair<A, B>::L, Lp = RegPair<A, B>::Lp;
  const int nx = T.nx, ny = T.ny, n_zc = T.n_zc;
  const int n_xt = (nx + L - 1) / L;
  const long long n_tiles = (long long)n_xt * ny * n_bands;
  cplx* bufA = sm;                                // exchange buffer (both exchanges alias, as in the plain kernel)
  cplx* in0 = sm + (size_t)n * Lp;                // two staged input tiles [n_zc][L]
  cplx* in1 = in0 + (size_t)n_zc * L;
  const uint64_t pol_keep = l2_policy_evict_last(), pol_stream = l2_policy_evict_first();
  const int tid = threadIdx.x, line = tid % L, p = tid / L;
  auto stage = [&](long long tile, cplx* dst) {
    const int xt = (int)(tile % n_xt), y = (int)((tile / n_xt) % ny), band = (int)(tile / ((long long)n_xt * ny));
    const cplx* w2 = W2 + (size_t)band * n_zc * ny * nx;
    for (int c = tid; c < n_zc * L; c += L * TT) {
      const int zc = c / L, l = c % L, x = xt * L + l;
      zp_cp_async16(dst + c, w2 + (unsigned)((zc * ny + y) * nx + (x < nx ? x : 0)), x < nx);
    }
    asm volatile("cp.async.commit_group;\n" ::);
  };
  long long tile = blockIdx.x;
  if (tile < n_tiles) stage(tile, in0);
  int it = 0;
  for (; tile < n_tiles; tile += gridDim.x, ++it) {
    cplx* cur = (it & 1) ? in1 : in0;
    cplx* nxt = (it & 1) ? in0 : in1;
    const long long tn = tile + gridDim.x;
    if (tn < n_tiles) {
      stage(tn, nxt);
      asm volatile("cp.async.wait_group 1;\n" ::);
    } else {
      asm volatile("cp.async.wait_group 0;\n" ::);
    }
    __syncthreads();
    const int xt = (int)(tile % n_xt), y = (int)((tile / n_xt) % ny), band = (int)(tile / ((long long)n_xt * ny));
    const int x = xt * L + line;
    cplx* w2 = W2 + (size_t)band * n_zc * ny * nx;
    if (p < B) {
      cplx v[A];
#pragma unroll
      for (int r = 0; r < A; ++r) {
        const int zc = zc_index(T, p + B * r);
        v[r] = zc >= 0 ? cur[zc * L + line] : make_double2(0.0, 0.0);
      }
      pass1_store<A, B, +1>(v, p, line, bufA, Lp, tw);
    }
    __syncthreads();
    cplx Y[B];
    if (p < A) {
      cplx X[B];
      pass2_load<A, B, +1>(X, p, line, bufA, Lp);
#pragma unroll
      for (int d = 0; d < B; ++d) {
        double vv = ld_pred_hint(V + (unsigned)(((p + A * d) * ny + y) * nx + x), x < nx, pol_keep);
        X[d] = cscale(X[d], vv);
      }
      pass1_compute<B, A, -1>(X, p, tw, Y);
    }
    __syncthreads();
    if (p < A) {
#pragma unroll
      for (int c = 0; c < B; ++c) bufA[(c * A + p) * Lp + line] = Y[c];
    }
    __syncthreads();
    if (p < B) {
      cplx X[A];
      pass2_load<B, A, -1>(X, p, line, bufA, Lp);
#pragma unroll
      for (int f = 0; f < A; ++f) {
        const int zc = zc_index(T, p + B * f);
        st_pred_hint(w2 + (unsigned)(((zc < 0 ? 0 : zc) * ny + y) * nx + x), X[f], zc >= 0 && x < nx, pol_stream);
      }
    }
    __syncthreads();     // bufA and `cur` are free again (the next iteration stages into `cur`)
  }
}
#endif

template <int A, int B>
HD void reg_z_to_cube(const SphereTablesX& T, const cplx* __restrict__ tw, const cplx* __restrict__ W2,
                      cplx* __restrict__ cube, double scale, int L_rt, int Lp_rt, cplx* sm, Dim3i bid) {
  constexpr int n = A * B, TT = RegPair<A, B>::T, L = RegPair<A, B>::L, Lp = RegPair<A, B>::Lp;
  (void)L_rt;
  (void)Lp_rt;
  const int nx = T.nx, ny = T.ny;
  cplx* bufA = sm;
  const int x0 = bid.x * L, y = bid.y;
  const cplx* w2 = W2 + (size_t)bid.z * T.n_zc * ny * nx;
  cplx* out = cube + (size_t)bid.z * nx * ny * n;
  TLOOP(t, L * TT) {
    const int line = t % L, p = t / L, x = x0 + line;
    if (p < B) {
      cplx v[A];
#pragma unroll
      for (int r = 0; r < A; ++r) {
        int zc = zc_index(T, p + B * r);
        v[r] = ld_pred(w2 + (unsigned)(((zc < 0 ? 0 : zc) * ny + y) * nx + x), zc >= 0 && x < nx);
      }
      pass1_store<A, B, +1>(v, p, line, bufA, Lp, tw);
    }
  }
  TSYNC();
  TLOOP(t, L * TT) {
    const int line = t % L, p = t / L, x = x0 + line;
    if (p < A) {
      cplx X[B];
      pass2_load<A, B, +1>(X, p, line, bufA, Lp);
#pragma unroll
      for (int d = 0; d < B; ++d)
        st_pred(out + (unsigned)(((p + A * d) * ny + y) * nx + x), cscale(X[d], scale), x < nx);
    }
  }
}

template <int A, int B>
HD void reg_z_from_cube(const SphereTablesX& T, const cplx* __restrict__ tw, const cplx* __restrict__ cube,
                        cplx* __restrict__ W2, int L_rt, int Lp_rt, cplx* sm, Dim3i bid) {
  constexpr int n = A * B, TT = RegPair<A, B>::T, L = RegPair<A, B>::L, Lp = RegPair<A, B>::Lp;
  (void)L_rt;
  (void)Lp_rt;
  const int nx = T.nx, ny = T.ny;
  cplx* bufA = sm;
  const int x0 = bid.x * L, y = bid.y;
  const cplx* in = cube + (size_t)bid.z * nx * ny * n;
  cplx* w2 = W2 + (size_t)bid.z * T.n_zc * ny * nx;
  TLOOP(t, L * TT) {
    const int line = t % L, p = t / L, x = x0 + line;
    if (p < B) {
      cplx v[A];
#pragma unroll
      for (int r = 0; r < A; ++r)
        v[r] = ld_pred(in + (unsigned)(((p + B * r) * ny + y) * nx + x), x < nx);
      pass1_store<A, B, -1>(v, p, line, bufA, Lp, tw);
    }
  }
  TSYNC();
  TLOOP(t, L * TT) {
    const int line = t % L, p = t / L, x = x0 + line;
    if (p < A) {
      cplx X[B];
      pass2_load<A, B, -1>(X, p, line, bufA, Lp);
#pragma unroll
      for (int d = 0; d < B; ++d) {
        int zc = zc_index(T, p + A * d);
        st_pred(w2 + (unsigned)(((zc < 0 ? 0 : zc) * ny + y) * nx + x), X[d], zc >= 0 && x < nx);
      }
    }
  }
}

// density: acc (double[n*L] after the two complex buffers) is owned element-wise by the pass-2 threads
template <int A, int B>
HD void reg_z_density(const SphereTablesX& T, const cplx* __restrict__ tw, const cplx* __restrict__ W2,
                      const double* __restrict__ wts, int nb, double* __restrict__ rho, int L_rt, int Lp_rt,
                      cplx* sm, Dim3i bid) {
  constexpr int n = A * B, TT = RegPair<A, B>::T, L = RegPair<A, B>::L, Lp = RegPair<A, B>::Lp;
  (void)L_rt;
  (void)Lp_rt;
  const int nx = T.nx, ny = T.ny;
  cplx* bufA = sm;
  double* acc = (double*)(sm + 2 * (size_t)n * Lp);
  const int x0 = bid.x * L, y = bid.y;
  TLOOP(t, n * L) acc[t] = 0.0;
  for (int band = 0; band < nb; ++band) {
    const cplx* w2 = W2 + (size_t)band * T.n_zc * ny * nx;
    TSYNC();
    TLOOP(t, L * TT) {
      const int line = t % L, p = t / L, x = x0 + line;
      if (p < B) {
        cplx v[A];
#pragma unroll
        for (int r = 0; r < A; ++r) {
          int zc = zc_index(T, p + B * r);
          v[r] = ld_pred(w2 + (unsigned)(((zc < 0 ? 0 : zc) * ny + y) * nx + x), zc >= 0 && x < nx);
        }
        pass1_store<A, B, +1>(v, p, line, bufA, Lp, tw);
      }
    }
    TSYNC();
    const double w = wts[band];
    TLOOP(t, L * TT) {
      const int line = t % L, p = t / L;
      if (p < A) {
        cplx X[B];
        pass2_load<A, B, +1>(X, p, line, bufA, Lp);
#pragma unroll
        for (int d = 0; d < B; ++d) acc[(p + A * d) * L + line] += w * (X[d].x * X[d].x + X[d].y * X[d].y);
      }
    }
  }
  TSYNC();
  TLOOP(t, n * L) {
    const int line = t % L, iz = t / L, x = x0 + line;
    if (x < nx) rho[((size_t)iz * ny + y) * nx + x] += acc[t];
  }
}

// ---------------------------------------------------------------------------------------------- y stages
template <int A, int B>
HD void reg_y_backward(const SphereTablesX& T, const cplx* __restrict__ tw, const cplx* __restrict__ W1,
                       cplx* __restrict__ W2, int L_rt, int Lp_rt, cplx* sm, Dim3i bid) {
  constexpr int n = A * B, TT = RegPair<A, B>::T, L = RegPair<A, B>::L, Lp = RegPair<A, B>::Lp;
  (void)L_rt;
  (void)Lp_rt;
  const int nx = T.nx;
  cplx* bufA = sm;
  const int x0 = bid.x * L, izc = bid.y;
  const cplx* in = W1 + (size_t)bid.z * T.n_cols * nx;
  cplx* out = W2 + ((size_t)bid.z * T.n_zc + izc) * n * nx;
  const PlaneCols pc = plane_cols(T, izc);
  TLOOP(t, L * TT) {
    const int line = t % L, p = t / L, x = x0 + line;
    if (p < B) {
      cplx v[A];
#pragma unroll
      for (int r = 0; r < A; ++r) {
        int c = pc.col(p + B * r);
        v[r] = ld_pred(in + (unsigned)((c < 0 ? 0 : c) * nx + x), c >= 0 && x < nx);
      }
      pass1_store<A, B, +1>(v, p, line, bufA, Lp, tw);
    }
  }
  TSYNC();
  TLOOP(t, L * TT) {
    const int line = t % L, p = t / L, x = x0 + line;
    if (p < A) {
      cplx X[B];
      pass2_load<A, B, +1>(X, p, line, bufA, Lp);
#pragma unroll
      for (int d = 0; d < B; ++d)
        st_pred(out + (unsigned)((p + A * d) * nx + x), X[d], x < nx);
    }
  }
}

template <int A, int B>
HD void reg_y_forward(const SphereTablesX& T, const cplx* __restrict__ tw, const cplx* __restrict__ W2,
                      cplx* __restrict__ W1, int L_rt, int Lp_rt, cplx* sm, Dim3i bid) {
  constexpr int n = A * B, TT = RegPair<A, B>::T, L = RegPair<A, B>::L, Lp = RegPair<A, B>::Lp;
  (void)L_rt;
  (void)Lp_rt;
  const int nx = T.nx;
  cplx* bufA = sm;
  const int x0 = bid.x * L, izc = bid.y;
  const cplx* in = W2 + ((size_t)bid.z * T.n_zc + izc) * n * nx;
  cplx* out = W1 + (size_t)bid.z * T.n_cols * nx;
  const PlaneCols pc = plane_cols(T, izc);
  TLOOP(t, L * TT) {
    const int line = t % L, p = t / L, x = x0 + line;
    if (p < B) {
      cplx v[A];
#pragma unroll
      for (int r = 0; r < A; ++r)
        v[r] = ld_pred(in + (unsigned)((p + B * r) * nx + x), x < nx);
      pass1_store<A, B, -1>(v, p, line, bufA, Lp, tw);
    }
  }
  TSYNC();
  TLOOP(t, L * TT) {
    const int line = t % L, p = t / L, x = x0 + line;
    if (p < A) {
      cplx X[B];
      pass2_load<A, B, -1>(X, p, line, bufA, Lp);
#pragma unroll
      for (int d = 0; d < B; ++d) {
        int c = pc.col(p + A * d);
        st_pred(out + (unsigned)((c < 0 ? 0 : c) * nx + x), X[d], c >= 0 && x < nx);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------- fused y-z stage
// The y and z passes of the local H apply for one x line of one band (ny == nz, so both axes use the pair (A, B) and one
// twiddle table).  The whole pruned y-z intermediate of the line, S[zc][y] (n_zc * (n|1) complex numbers), stays in
// shared memory, so only the x-major W1 row W1t[band][x][0:n_cols] crosses global memory, once in and once out:
//   y backward: the sphere columns of GL planes at a time -> S rows
//   z apply:    GL y lines at a time: S[zc][y] -> inverse z transform -> * Vt(x, y, .) -> forward z transform -> S[zc][y]
//   y forward:  GL S rows at a time -> the sphere columns of the plane, back into W1t in place
// The CTA is G warp groups (GLOOP).  Group g owns a contiguous, balanced share of the planes (the same in both y passes)
// and of the y lines (z pass), GL lines of the exchange buffer E[line][n|1] (the y passes read or write S / W1t on the
// other side) and a named barrier, so the rounds of the groups overlap and only the two pass boundaries wait for the
// whole CTA.  The two exchanges of the z pass alias on the device as in reg_z_apply_potential, behind the group's barrier.
// GL = 8: the line is the fastest index of a group's threads, and 8 lines at the odd stride n|1 keep the 16-byte shared
// accesses of every quarter warp conflict-free.  Up to G = 3 groups use 24 of the LL = 25 exchange lines of smem() (at
// 150^3 with 71 planes the buffers take 231 936 of the H100's 232 448 bytes, one CTA per SM); fewer groups for T > 16,
// so that a CTA has at most 12 warps and a thread may keep 168 registers.
template <int A, int B>
struct RegYZ {
  static constexpr int n = A * B, T = RegPair<A, B>::T, LL = 25, Sy = n | 1;   // odd row stride: conflict-free columns
  static constexpr int GL = 8, GW = (GL * T + 31) / 32;                          // lines per round, warps per group
  static constexpr int G = (12 / GW < 3 ? 12 / GW : 3), GT = 32 * GW, NT = G * GT;   // groups, threads per group / CTA
  static_assert(G >= 1 && G * GL <= LL, "the groups' exchange lines must fit the buffer");
  static size_t smem(int n_zc) { return ((size_t)n_zc + (DFTK_Z_ALIAS ? 1 : 2) * LL) * Sy * sizeof(cplx); }
};

// One item (band bid.z, x line bid.x); blockDim == RegYZ<A, B>::NT.  A group touches only its own planes and exchange
// lines after the last CTA barrier, so the device kernel may start a group on its next item without one.
template <int A, int B>
HD void reg_yz_apply(const SphereTablesX& T, const cplx* __restrict__ tw, cplx* __restrict__ W1t,
                     const double* __restrict__ Vt, cplx* sm, Dim3i bid) {
  constexpr int n = A * B, LL = RegYZ<A, B>::LL, Sy = RegYZ<A, B>::Sy;
  constexpr int GL = RegYZ<A, B>::GL, G = RegYZ<A, B>::G, GT = RegYZ<A, B>::GT;
  const int n_zc = T.n_zc, x = bid.x;
  cplx* S = sm;
  cplx* row = W1t + ((size_t)bid.z * T.nx + x) * T.n_cols;
  const double* vx = Vt + (size_t)x * n * n;
  const uint64_t pol_keep = l2_policy_evict_last();
  // y backward: the group's planes zc0 .. zc0+GL-1
  GLOOP(g, G, GT) {
    cplx* E = sm + ((size_t)n_zc + g * GL) * Sy;
    const int zc1 = (g + 1) * n_zc / G;
    for (int zc0 = g * n_zc / G; zc0 < zc1; zc0 += GL) {
      GTLOOP(t, GT) {
        const int line = t % GL, p = t / GL, zc = zc0 + line;
        if (p < B && zc < zc1) {
          const PlaneCols pc = plane_cols(T, zc);
          cplx v[A];
#pragma unroll
          for (int r = 0; r < A; ++r) {
            int c = pc.col(p + B * r);
            v[r] = ld_pred(row + (c < 0 ? 0 : c), c >= 0);
          }
          pass1_store<A, B, +1>(v, p, 0, E + line * Sy, 1, tw);
        }
      }
      GSYNC(g, GT);
      GTLOOP(t, GT) {
        const int line = t % GL, p = t / GL, zc = zc0 + line;
        if (p < A && zc < zc1) {
          cplx X[B];
          pass2_load<A, B, +1>(X, p, 0, E + line * Sy, 1);
#pragma unroll
          for (int d = 0; d < B; ++d) S[zc * Sy + p + A * d] = X[d];
        }
      }
      GSYNC(g, GT);
    }
  }
  TSYNC();
  // z apply: the group's y lines y0 .. y0+GL-1 (S columns)
  GLOOP(g, G, GT) {
    cplx* E = sm + ((size_t)n_zc + g * GL) * Sy;
    cplx* E2 = DFTK_Z_ALIAS ? E : E + (size_t)LL * Sy;
    const int y1 = (g + 1) * n / G;
    for (int y0 = g * n / G; y0 < y1; y0 += GL) {
      GTLOOP(t, GT) {
        const int line = t % GL, p = t / GL, y = y0 + line;
        if (p < B && y < y1) {
          cplx v[A];
#pragma unroll
          for (int r = 0; r < A; ++r) {
            int zc = zc_index(T, p + B * r);
            v[r] = zc >= 0 ? S[zc * Sy + y] : make_double2(0.0, 0.0);
          }
          pass1_store<A, B, +1>(v, p, 0, E + line * Sy, 1, tw);
        }
      }
      GSYNC(g, GT);
      GTLOOP(t, GT) {
        const int line = t % GL, p = t / GL, y = y0 + line;
        cplx Y[B];
        if (p < A && y < y1) {
          cplx X[B];
          pass2_load<A, B, +1>(X, p, 0, E + line * Sy, 1);
#pragma unroll
          for (int d = 0; d < B; ++d) X[d] = cscale(X[d], ld_pred_hint(vx + y * n + p + A * d, true, pol_keep));
          pass1_compute<B, A, -1>(X, p, tw, Y);
        }
#if DFTK_Z_ALIAS
        GSYNC(g, GT);   // every thread of the group runs this body exactly once (GTLOOP on the device)
#endif
        if (p < A && y < y1) {
#pragma unroll
          for (int c = 0; c < B; ++c) E2[line * Sy + c * A + p] = Y[c];
        }
      }
      GSYNC(g, GT);
      GTLOOP(t, GT) {
        const int line = t % GL, p = t / GL, y = y0 + line;
        if (p < B && y < y1) {
          cplx X[A];
          pass2_load<B, A, -1>(X, p, 0, E2 + line * Sy, 1);
#pragma unroll
          for (int f = 0; f < A; ++f) {
            int zc = zc_index(T, p + B * f);
            if (zc >= 0) S[zc * Sy + y] = X[f];
          }
        }
      }
      GSYNC(g, GT);
    }
  }
  TSYNC();
  // y forward: the group's planes zc0 .. zc0+GL-1 (the same as in y backward), the sphere columns back to the W1t row
  GLOOP(g, G, GT) {
    cplx* E = sm + ((size_t)n_zc + g * GL) * Sy;
    const int zc1 = (g + 1) * n_zc / G;
    for (int zc0 = g * n_zc / G; zc0 < zc1; zc0 += GL) {
      GTLOOP(t, GT) {
        const int line = t % GL, p = t / GL, zc = zc0 + line;
        if (p < B && zc < zc1) {
          cplx v[A];
#pragma unroll
          for (int r = 0; r < A; ++r) v[r] = S[zc * Sy + p + B * r];
          pass1_store<A, B, -1>(v, p, 0, E + line * Sy, 1, tw);
        }
      }
      GSYNC(g, GT);
      GTLOOP(t, GT) {
        const int line = t % GL, p = t / GL, zc = zc0 + line;
        if (p < A && zc < zc1) {
          const PlaneCols pc = plane_cols(T, zc);
          cplx X[B];
          pass2_load<A, B, -1>(X, p, 0, E + line * Sy, 1);
#pragma unroll
          for (int d = 0; d < B; ++d) {
            int c = pc.col(p + A * d);
            st_pred(row + (c < 0 ? 0 : c), X[d], c >= 0);
          }
        }
      }
      GSYNC(g, GT);
    }
  }
}

// ---------------------------------------------------------------------------------------------- x stages
// (contiguous axis: coalesced transposing load/store through shared memory)
// Column descriptors of the CTA's L columns, staged in shared memory: {first slot, n0, s0, n1, s1}
HD void load_col_desc(const SphereTablesX& T, int c0, int L, int* cd) {
  TLOOP(t, L) {
    int c = c0 + t;
    bool ok = c < T.n_cols;
    cd[5 * t + 0] = ok ? T.col_start[c] : 0;
    cd[5 * t + 1] = ok ? T.cx_n0[c] : 0;
    cd[5 * t + 2] = ok ? T.cx_s0[c] : 0;
    cd[5 * t + 3] = ok ? T.cx_n1[c] : 0;
    cd[5 * t + 4] = ok ? T.cx_s1[c] : 0;
  }
}

// W1 of a band is [col][x] (XM == 0: the y / z stages read x-contiguous lines) or [x][col] (XM == 1: the fused y-z
// stage reads one x row).  The element order of the copy loops follows the layout, so consecutive threads always touch
// consecutive addresses (for [x][col]: the L columns of the tile, 8 * 16 B = 128 B at L = 8).
template <int n, int L, int XM>
HD void w1_index(int t, int& line, int& x) {
  line = XM ? t % L : t / n;
  x = XM ? t / L : t % n;
}
template <int n, int XM>
HD size_t w1_offset(int c, int x, int n_cols) {
  return XM ? (size_t)x * n_cols + c : (size_t)c * n + x;
}

template <int A, int B, int XM = 0>
HD void reg_sphere_to_x(const SphereTablesX& T, const cplx* __restrict__ tw, const cplx* __restrict__ psi,
                        int64_t ldpsi, cplx* __restrict__ W1, int L_rt, int Lp_rt, cplx* sm, Dim3i bid) {
  constexpr int n = A * B, TT = RegPair<A, B>::T, L = RegPair<A, B>::L, Lp = RegPair<A, B>::Lp;
  (void)L_rt;
  (void)Lp_rt;
  cplx* bufA = sm;
  cplx* bufB = sm + (size_t)n * Lp;
  int* cd = (int*)(sm + 2 * (size_t)n * Lp);
  const int c0 = bid.x * L;
  const int64_t band = bid.y;
  load_col_desc(T, c0, L, cd);
  TLOOPC(t, n * Lp, L * TT) bufA[t] = make_double2(0.0, 0.0);
  TSYNC();
  // gather: TT threads per column walk its sphere points (contiguous in psi)
  const cplx* pb = psi + band * ldpsi;
  TLOOPC(t, L * n, L * TT) {
    const int line = t / n, i = t % n;   // n is a compile-time constant
    const int n0 = cd[5 * line + 1], n1 = cd[5 * line + 3];
    if (i < n0 + n1) {
      const int ix = i < n0 ? cd[5 * line + 2] + i : cd[5 * line + 4] + (i - n0);
      bufA[ix * Lp + line] = pb[cd[5 * line] + i];
    }
  }
  TSYNC();
  TLOOP(t, L * TT) {
    const int line = t % L, p = t / L;
    if (p < B) {
      cplx v[A];
#pragma unroll
      for (int r = 0; r < A; ++r) v[r] = bufA[(p + B * r) * Lp + line];
      pass1_store<A, B, +1>(v, p, line, bufB, Lp, tw);
    }
  }
  TSYNC();
  TLOOP(t, L * TT) {
    const int line = t % L, p = t / L;
    if (p < A) {
      cplx X[B];
      pass2_load<A, B, +1>(X, p, line, bufB, Lp);
#pragma unroll
      for (int d = 0; d < B; ++d) bufA[(p + A * d) * Lp + line] = X[d];
    }
  }
  TSYNC();
  cplx* out = W1 + (size_t)band * T.n_cols * n;
  TLOOPC(t, L * n, L * TT) {
    int line, x;
    w1_index<n, L, XM>(t, line, x);
    const int c = c0 + line;
    if (c < T.n_cols) out[w1_offset<n, XM>(c, x, T.n_cols)] = bufA[x * Lp + line];
  }
}

template <int A, int B, int XM = 0>
HD void reg_x_to_sphere(const SphereTablesX& T, const cplx* __restrict__ tw, const cplx* __restrict__ W1,
                        cplx* __restrict__ out, int64_t ldout, double scale, const double* __restrict__ kin,
                        const cplx* __restrict__ psi, int64_t ldpsi, int accumulate, int L_rt, int Lp_rt, cplx* sm,
                        Dim3i bid) {
  constexpr int n = A * B, TT = RegPair<A, B>::T, L = RegPair<A, B>::L, Lp = RegPair<A, B>::Lp;
  (void)L_rt;
  (void)Lp_rt;
  cplx* bufA = sm;
  cplx* bufB = sm + (size_t)n * Lp;
  int* cd = (int*)(sm + 2 * (size_t)n * Lp);
  const int c0 = bid.x * L;
  const int64_t band = bid.y;
  const cplx* in = W1 + (size_t)band * T.n_cols * n;
  load_col_desc(T, c0, L, cd);
  TLOOPC(t, L * n, L * TT) {
    int line, x;
    w1_index<n, L, XM>(t, line, x);
    const int c = c0 + line;
    bufA[x * Lp + line] = (c < T.n_cols) ? in[w1_offset<n, XM>(c, x, T.n_cols)] : make_double2(0.0, 0.0);
  }
  TSYNC();
  TLOOP(t, L * TT) {
    const int line = t % L, p = t / L;
    if (p < B) {
      cplx v[A];
#pragma unroll
      for (int r = 0; r < A; ++r) v[r] = bufA[(p + B * r) * Lp + line];
      pass1_store<A, B, -1>(v, p, line, bufB, Lp, tw);
    }
  }
  TSYNC();
  TLOOP(t, L * TT) {
    const int line = t % L, p = t / L;
    if (p < A) {
      cplx X[B];
      pass2_load<A, B, -1>(X, p, line, bufB, Lp);
#pragma unroll
      for (int d = 0; d < B; ++d) bufA[(p + A * d) * Lp + line] = X[d];
    }
  }
  TSYNC();
  const cplx* pb = psi ? psi + band * ldpsi : nullptr;
  cplx* ob = out + band * ldout;
  TLOOPC(t, L * n, L * TT) {
    const int line = t / n, i = t % n;
    const int n0 = cd[5 * line + 1], n1 = cd[5 * line + 3];
    if (i < n0 + n1) {
      const int ix = i < n0 ? cd[5 * line + 2] + i : cd[5 * line + 4] + (i - n0);
      const int s = cd[5 * line] + i;
      cplx v = cscale(bufA[ix * Lp + line], scale);
      if (kin) {
        cplx pp = pb[s];
        double kk = kin[s];
        v.x += kk * pp.x;
        v.y += kk * pp.y;
      }
      if (accumulate) {
        cplx o = ob[s];
        v.x += o.x;
        v.y += o.y;
      }
      ob[s] = v;
    }
  }
}

}  // namespace dftk
