// Shared-memory batched 1D FFT engine and the pruned sphere<->cube pipeline stages.
//
// Every stage body is a __host__ __device__ function over (block index, "thread loop") so that the
// same index logic can be executed sequentially on the host by tests/hostemu (there is no GPU in the
// build container).  On the device TLOOP strides over the CTA's threads and TSYNC is __syncthreads().
//
// Data layout in shared memory: buf[idx * Lp + line], `line` = which of the L lines of the tile,
// Lp = L | 1 (odd pitch => 16-byte accesses are bank-conflict free both for line-major butterflies
// and for transposed loads).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#if defined(__CUDA_ARCH__)
#define TLOOP(t, n) for (int t = threadIdx.x; t < (n); t += blockDim.x)
#define TSYNC() __syncthreads()
#else
#define TLOOP(t, n) for (int t = 0; t < (n); ++t)
#define TSYNC() ((void)0)
#endif
// TLOOPC: thread loop with compile-time count and CTA size -> constant trip count, fully unrolled on the device
// (all global loads of the iterations are issued before the first use); TLOOPU: runtime count, unrolled by 4.
#if defined(__CUDA_ARCH__)
#define TLOOPC(t, n, nthr)                                                        \
  _Pragma("unroll") for (int i__ = 0; i__ < ((n) + (nthr)-1) / (nthr); ++i__)    \
      for (int t = (int)threadIdx.x + i__ * (nthr), once__ = 1; once__ && t < (n); once__ = 0)
#define TLOOPU(t, n) _Pragma("unroll 4") for (int t = threadIdx.x; t < (n); t += blockDim.x)
#else
#define TLOOPC(t, n, nthr) for (int t = 0; t < (n); ++t)
#define TLOOPU(t, n) for (int t = 0; t < (n); ++t)
#endif
// threadIdx.x read anew at every use: what a group thread derives from its index (twiddles, plane maps) is then recomputed
// per round instead of being hoisted out of a persistent kernel's item loop into registers for the whole kernel.
__device__ __forceinline__ int tid_volatile() {
  int t;
  asm volatile("mov.u32 %0, %%tid.x;" : "=r"(t));
  return t;
}
// Warp groups: a CTA of blockDim == G * GT threads split into G groups of GT (a multiple of 32) consecutive threads that
// work on disjoint data between CTA-wide barriers.  GLOOP(g, G, GT) runs its body for the thread's own group g on the
// device and for every group in turn on the host; GTLOOP(t, GT) is TLOOP over the group's threads; GSYNC(g, GT) is the
// group's named barrier 1 + g (barrier 0 is __syncthreads).  As for TSYNC, no register state is live across a GSYNC.
#if defined(__CUDA_ARCH__)
#define GLOOP(g, G, GT) for (int g = (int)threadIdx.x / (GT), gonce__ = 1; gonce__; gonce__ = 0)
#define GTLOOP(t, GT) for (int t = tid_volatile() % (GT), tonce__ = 1; tonce__; tonce__ = 0)
#define GSYNC(g, GT) asm volatile("bar.sync %0, %1;" ::"r"(1 + (g)), "r"(GT) : "memory")
#else
#define GLOOP(g, G, GT) for (int g = 0; g < (G); ++g)
#define GTLOOP(t, GT) for (int t = 0; t < (GT); ++t)
#define GSYNC(g, GT) ((void)(g))
#endif
#define HD __host__ __device__ __forceinline__

namespace dftk {

typedef double2 cplx;

HD cplx cmul(cplx a, cplx b) { return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
HD cplx cadd(cplx a, cplx b) { return make_double2(a.x + b.x, a.y + b.y); }
HD cplx csub(cplx a, cplx b) { return make_double2(a.x - b.x, a.y - b.y); }
HD cplx cscale(cplx a, double s) { return make_double2(a.x * s, a.y * s); }
// multiply by s*i (s = +-1)
HD cplx cmuli(cplx a, double s) { return make_double2(-s * a.y, s * a.x); }

#define DFTK_MAX_PASSES 12
struct FftPlan {
  int n;
  int npass;
  int radix[DFTK_MAX_PASSES];
};

// Twiddle table tw[m] = exp(-2 pi i m / n) (forward sign).  sign = -1 forward, +1 backward.
HD cplx twiddle(const cplx* __restrict__ tw, int m, int sign) {
  cplx w = tw[m];
  if (sign > 0) w.y = -w.y;
  return w;
}

// One Stockham autosort pass of radix R over L lines.
template <int R>
HD void butterfly(cplx* v, int sign) {
  const double s = (double)sign;
  if (R == 2) {
    cplx a = v[0], b = v[1];
    v[0] = cadd(a, b);
    v[1] = csub(a, b);
  } else if (R == 4) {
    cplx t0 = cadd(v[0], v[2]), t1 = csub(v[0], v[2]);
    cplx t2 = cadd(v[1], v[3]), t3 = cmuli(csub(v[1], v[3]), s);
    v[0] = cadd(t0, t2);
    v[2] = csub(t0, t2);
    v[1] = cadd(t1, t3);
    v[3] = csub(t1, t3);
  } else if (R == 3) {
    const double h = 0.86602540378443864676;  // sqrt(3)/2
    cplx t1 = cadd(v[1], v[2]);
    cplx m = make_double2(v[0].x - 0.5 * t1.x, v[0].y - 0.5 * t1.y);
    cplx d = cmuli(cscale(csub(v[1], v[2]), h), s);
    v[0] = cadd(v[0], t1);
    v[1] = cadd(m, d);
    v[2] = csub(m, d);
  } else if (R == 5) {
    const double c1 = 0.30901699437494742410, c2 = -0.80901699437494742410;
    const double s1 = 0.95105651629515357212, s2 = 0.58778525229247312917;
    cplx t1 = cadd(v[1], v[4]), t2 = cadd(v[2], v[3]);
    cplx t3 = csub(v[1], v[4]), t4 = csub(v[2], v[3]);
    cplx m1 = make_double2(v[0].x + c1 * t1.x + c2 * t2.x, v[0].y + c1 * t1.y + c2 * t2.y);
    cplx m2 = make_double2(v[0].x + c2 * t1.x + c1 * t2.x, v[0].y + c2 * t1.y + c1 * t2.y);
    cplx n1 = cmuli(make_double2(s1 * t3.x + s2 * t4.x, s1 * t3.y + s2 * t4.y), s);
    cplx n2 = cmuli(make_double2(s2 * t3.x - s1 * t4.x, s2 * t3.y - s1 * t4.y), s);
    v[0] = cadd(v[0], cadd(t1, t2));
    v[1] = cadd(m1, n1);
    v[4] = csub(m1, n1);
    v[2] = cadd(m2, n2);
    v[3] = csub(m2, n2);
  }
}

template <int R>
HD void stockham_pass(const cplx* __restrict__ in, cplx* __restrict__ out, int n, int Ns, int L,
                      int Lp, const cplx* __restrict__ tw, int sign) {
  const int nb = n / R;
  const int tstep = n / (Ns * R);
  TLOOP(t, nb * L) {
    int line = t % L, j = t / L;
    int k = j % Ns;
    cplx v[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      cplx x = in[(j + r * nb) * Lp + line];
      v[r] = (r == 0 || k == 0) ? x : cmul(x, twiddle(tw, r * k * tstep, sign));
    }
    butterfly<R>(v, sign);
    int j0 = (j / Ns) * Ns * R + k;
#pragma unroll
    for (int r = 0; r < R; ++r) out[(j0 + r * Ns) * Lp + line] = v[r];
  }
}

// Generic (any radix, O(R^2)) pass; only used for odd primes > 5.
HD void stockham_pass_generic(const cplx* __restrict__ in, cplx* __restrict__ out, int n, int R,
                              int Ns, int L, int Lp, const cplx* __restrict__ tw, int sign) {
  const int nb = n / R;
  const int tstep = n / (Ns * R);
  TLOOP(t, nb * L * R) {
    int line = t % L, jq = t / L;
    int j = jq % nb, q = jq / nb;
    int k = j % Ns;
    cplx acc = make_double2(0.0, 0.0);
    for (int r = 0; r < R; ++r) {
      cplx x = in[(j + r * nb) * Lp + line];
      // twiddle exp(s 2 pi i r k /(Ns R)) * exp(s 2 pi i r q / R)
      int m = (r * k * tstep + ((r * q) % R) * nb) % n;
      acc = cadd(acc, cmul(x, twiddle(tw, m, sign)));
    }
    int j0 = (j / Ns) * Ns * R + k;
    out[(j0 + q * Ns) * Lp + line] = acc;
  }
}

// Transform L lines of length plan.n held in `a` (layout [idx][Lp]); `b` is scratch of the same size.
// Returns the buffer holding the result.  All threads of the CTA must call it.
HD cplx* fft_lines(cplx* a, cplx* b, const FftPlan& plan, const cplx* __restrict__ tw, int L, int Lp,
                   int sign) {
  int Ns = 1;
  const int n = plan.n;
  for (int p = 0; p < plan.npass; ++p) {
    int R = plan.radix[p];
    TSYNC();
    switch (R) {
      case 2: stockham_pass<2>(a, b, n, Ns, L, Lp, tw, sign); break;
      case 3: stockham_pass<3>(a, b, n, Ns, L, Lp, tw, sign); break;
      case 4: stockham_pass<4>(a, b, n, Ns, L, Lp, tw, sign); break;
      case 5: stockham_pass<5>(a, b, n, Ns, L, Lp, tw, sign); break;
      default: stockham_pass_generic(a, b, n, R, Ns, L, Lp, tw, sign); break;
    }
    cplx* t = a;
    a = b;
    b = t;
    Ns *= R;
  }
  TSYNC();
  return a;
}

// ------------------------------------------------------------------------------------------------
// Pruned sphere <-> cube pipeline.  Axis order x (contiguous) -> y -> z on the way to real space.
//   W1[b][col][x]      : after the x pass; col enumerates the (y,z) columns that hold sphere points
//   W2[b][izc][y][x]   : after the y pass; izc enumerates the z planes that hold sphere points
// ------------------------------------------------------------------------------------------------
struct SphereTables {
  int nx, ny, nz;
  int64_t n_pw;
  int n_cols;     // number of non-empty (y,z) columns
  int cnt_max;    // max sphere points in one column
  int n_zc;       // number of non-empty z planes
  const int* col_start;  // [n_cols] first slot of the column (slots are column-sorted sphere points)
  const int* col_cnt;    // [n_cols]
  const int* slot_ix;    // [n_pw] x index (wrapped, 0..nx-1) of the slot
  const int* slot_src;   // [n_pw] index into psi of the slot (identity for ascending mappings)
  const int* zlist;      // [n_zc] wrapped z index of plane izc
  const int* colmap;     // [n_zc*ny] column id of (izc, iy) or -1
};

struct Dim3i {
  int x, y, z;
};

// Stage A: gather sphere -> x lines, backward FFT along x, write W1.  grid (ceil(n_cols/L), nb)
HD void stage_sphere_to_x(const SphereTables& T, const FftPlan& px, const cplx* twx,
                          const cplx* __restrict__ psi, int64_t ldpsi, cplx* __restrict__ W1, int L,
                          int Lp, cplx* sm, Dim3i bid) {
  const int nx = T.nx;
  cplx* a = sm;
  cplx* b = sm + (size_t)nx * Lp;
  const int c0 = bid.x * L;
  const int64_t band = bid.y;
  TLOOP(t, nx * Lp) a[t] = make_double2(0.0, 0.0);
  TSYNC();
  TLOOP(t, L * T.cnt_max) {
    int line = t / T.cnt_max, i = t % T.cnt_max;
    int c = c0 + line;
    if (c < T.n_cols && i < T.col_cnt[c]) {
      int s = T.col_start[c] + i;
      a[T.slot_ix[s] * Lp + line] = psi[band * ldpsi + T.slot_src[s]];
    }
  }
  cplx* r = fft_lines(a, b, px, twx, L, Lp, +1);
  cplx* out = W1 + (size_t)band * T.n_cols * nx;
  TLOOP(t, L * nx) {
    int line = t / nx, x = t % nx;
    int c = c0 + line;
    if (c < T.n_cols) out[(size_t)c * nx + x] = r[x * Lp + line];
  }
}

// Stage B: backward FFT along y.  grid (ceil(nx/L), n_zc, nb)
HD void stage_y_backward(const SphereTables& T, const FftPlan& py, const cplx* twy,
                         const cplx* __restrict__ W1, cplx* __restrict__ W2, int L, int Lp, cplx* sm,
                         Dim3i bid) {
  const int nx = T.nx, ny = T.ny;
  cplx* a = sm;
  cplx* b = sm + (size_t)ny * Lp;
  const int x0 = bid.x * L, izc = bid.y;
  const int64_t band = bid.z;
  const cplx* in = W1 + (size_t)band * T.n_cols * nx;
  TLOOP(t, ny * L) {
    int line = t % L, iy = t / L;
    int x = x0 + line;
    int c = T.colmap[izc * ny + iy];
    cplx v = make_double2(0.0, 0.0);
    if (c >= 0 && x < nx) v = in[(size_t)c * nx + x];
    a[iy * Lp + line] = v;
  }
  cplx* r = fft_lines(a, b, py, twy, L, Lp, +1);
  cplx* out = W2 + ((size_t)band * T.n_zc + izc) * ny * nx;
  TLOOP(t, ny * L) {
    int line = t % L, iy = t / L;
    int x = x0 + line;
    if (x < nx) out[(size_t)iy * nx + x] = r[iy * Lp + line];
  }
}

// Load the z lines of tile (x0.., y) from W2 (zero padded) into a.  Helper for the z stages.
HD void load_z_lines(const SphereTables& T, const cplx* __restrict__ W2band, int y, int x0, int L,
                     int Lp, cplx* a) {
  const int nx = T.nx, ny = T.ny, nz = T.nz;
  TLOOP(t, nz * Lp) a[t] = make_double2(0.0, 0.0);
  TSYNC();
  TLOOP(t, T.n_zc * L) {
    int line = t % L, izc = t / L;
    int x = x0 + line;
    if (x < nx) a[T.zlist[izc] * Lp + line] = W2band[((size_t)izc * ny + y) * nx + x];
  }
}

// Stage C (Hψ): backward FFT along z, multiply by V, forward FFT along z, store pruned in place.
// grid (ceil(nx/L), ny, nb).  V is pre-scaled by 1/N_fft.
HD void stage_z_apply_potential(const SphereTables& T, const FftPlan& pz, const cplx* twz,
                                cplx* __restrict__ W2, const double* __restrict__ V, int L, int Lp,
                                cplx* sm, Dim3i bid) {
  const int nx = T.nx, ny = T.ny, nz = T.nz;
  cplx* a = sm;
  cplx* b = sm + (size_t)nz * Lp;
  const int x0 = bid.x * L, y = bid.y;
  const int64_t band = bid.z;
  cplx* w2 = W2 + (size_t)band * T.n_zc * ny * nx;
  load_z_lines(T, w2, y, x0, L, Lp, a);
  cplx* r = fft_lines(a, b, pz, twz, L, Lp, +1);
  cplx* o = (r == a) ? b : a;
  TLOOP(t, nz * L) {
    int line = t % L, iz = t / L;
    int x = x0 + line;
    double v = (x < nx) ? V[((size_t)iz * ny + y) * nx + x] : 0.0;
    r[iz * Lp + line] = cscale(r[iz * Lp + line], v);
  }
  cplx* f = fft_lines(r, o, pz, twz, L, Lp, -1);
  TLOOP(t, T.n_zc * L) {
    int line = t % L, izc = t / L;
    int x = x0 + line;
    if (x < nx) w2[((size_t)izc * ny + y) * nx + x] = f[T.zlist[izc] * Lp + line];
  }
}

// Stage C (sphere_to_real): backward z FFT and write the full cube.  out[b][z][y][x] *= scale
HD void stage_z_to_cube(const SphereTables& T, const FftPlan& pz, const cplx* twz,
                        const cplx* __restrict__ W2, cplx* __restrict__ cube, double scale, int L,
                        int Lp, cplx* sm, Dim3i bid) {
  const int nx = T.nx, ny = T.ny, nz = T.nz;
  cplx* a = sm;
  cplx* b = sm + (size_t)nz * Lp;
  const int x0 = bid.x * L, y = bid.y;
  const int64_t band = bid.z;
  load_z_lines(T, W2 + (size_t)band * T.n_zc * ny * nx, y, x0, L, Lp, a);
  cplx* r = fft_lines(a, b, pz, twz, L, Lp, +1);
  cplx* out = cube + (size_t)band * nx * ny * nz;
  TLOOP(t, nz * L) {
    int line = t % L, iz = t / L;
    int x = x0 + line;
    if (x < nx) out[((size_t)iz * ny + y) * nx + x] = cscale(r[iz * Lp + line], scale);
  }
}

// Stage C (real_to_sphere): read the full cube, forward z FFT, store pruned W2.
HD void stage_z_from_cube(const SphereTables& T, const FftPlan& pz, const cplx* twz,
                          const cplx* __restrict__ cube, cplx* __restrict__ W2, int L, int Lp,
                          cplx* sm, Dim3i bid) {
  const int nx = T.nx, ny = T.ny, nz = T.nz;
  cplx* a = sm;
  cplx* b = sm + (size_t)nz * Lp;
  const int x0 = bid.x * L, y = bid.y;
  const int64_t band = bid.z;
  const cplx* in = cube + (size_t)band * nx * ny * nz;
  TLOOP(t, nz * L) {
    int line = t % L, iz = t / L;
    int x = x0 + line;
    a[iz * Lp + line] = (x < nx) ? in[((size_t)iz * ny + y) * nx + x] : make_double2(0.0, 0.0);
  }
  cplx* f = fft_lines(a, b, pz, twz, L, Lp, -1);
  cplx* w2 = W2 + (size_t)band * T.n_zc * ny * nx;
  TLOOP(t, T.n_zc * L) {
    int line = t % L, izc = t / L;
    int x = x0 + line;
    if (x < nx) w2[((size_t)izc * ny + y) * nx + x] = f[T.zlist[izc] * Lp + line];
  }
}

// Stage C (density): for every band of the chunk: backward z FFT, acc += w_b |psi(r)|^2; then
// rho[z][y][x] += acc.  grid (ceil(nx/L), ny); acc is a double[nz*L] region after the two cplx buffers.
HD void stage_z_density(const SphereTables& T, const FftPlan& pz, const cplx* twz,
                        const cplx* __restrict__ W2, const double* __restrict__ wts, int nb,
                        double* __restrict__ rho, int L, int Lp, cplx* sm, Dim3i bid) {
  const int nx = T.nx, ny = T.ny, nz = T.nz;
  cplx* a = sm;
  cplx* b = sm + (size_t)nz * Lp;
  double* acc = (double*)(sm + 2 * (size_t)nz * Lp);
  const int x0 = bid.x * L, y = bid.y;
  TLOOP(t, nz * L) acc[t] = 0.0;
  for (int band = 0; band < nb; ++band) {
    TSYNC();
    load_z_lines(T, W2 + (size_t)band * T.n_zc * ny * nx, y, x0, L, Lp, a);
    cplx* r = fft_lines(a, b, pz, twz, L, Lp, +1);
    const double w = wts[band];
    TLOOP(t, nz * L) {
      int line = t % L, iz = t / L;
      cplx v = r[iz * Lp + line];
      acc[t] += w * (v.x * v.x + v.y * v.y);
    }
  }
  TSYNC();
  TLOOP(t, nz * L) {
    int line = t % L, iz = t / L;
    int x = x0 + line;
    if (x < nx) rho[((size_t)iz * ny + y) * nx + x] += acc[t];
  }
}

// Stage D: forward FFT along y, keep only the rows that belong to sphere columns.
HD void stage_y_forward(const SphereTables& T, const FftPlan& py, const cplx* twy,
                        const cplx* __restrict__ W2, cplx* __restrict__ W1, int L, int Lp, cplx* sm,
                        Dim3i bid) {
  const int nx = T.nx, ny = T.ny;
  cplx* a = sm;
  cplx* b = sm + (size_t)ny * Lp;
  const int x0 = bid.x * L, izc = bid.y;
  const int64_t band = bid.z;
  const cplx* in = W2 + ((size_t)band * T.n_zc + izc) * ny * nx;
  TLOOP(t, ny * L) {
    int line = t % L, iy = t / L;
    int x = x0 + line;
    a[iy * Lp + line] = (x < nx) ? in[(size_t)iy * nx + x] : make_double2(0.0, 0.0);
  }
  cplx* r = fft_lines(a, b, py, twy, L, Lp, -1);
  cplx* out = W1 + (size_t)band * T.n_cols * nx;
  TLOOP(t, ny * L) {
    int line = t % L, iy = t / L;
    int x = x0 + line;
    int c = T.colmap[izc * ny + iy];
    if (c >= 0 && x < nx) out[(size_t)c * nx + x] = r[iy * Lp + line];
  }
}

// Stage E: forward FFT along x, gather the sphere coefficients.
//   out[src] = (accumulate ? out[src] : 0) + scale * val + (kin ? kin[src] * psi[src] : 0)
HD void stage_x_to_sphere(const SphereTables& T, const FftPlan& px, const cplx* twx,
                          const cplx* __restrict__ W1, cplx* __restrict__ out, int64_t ldout,
                          double scale, const double* __restrict__ kin, const cplx* __restrict__ psi,
                          int64_t ldpsi, int accumulate, int L, int Lp, cplx* sm, Dim3i bid) {
  const int nx = T.nx;
  cplx* a = sm;
  cplx* b = sm + (size_t)nx * Lp;
  const int c0 = bid.x * L;
  const int64_t band = bid.y;
  const cplx* in = W1 + (size_t)band * T.n_cols * nx;
  TLOOP(t, L * nx) {
    int line = t / nx, x = t % nx;
    int c = c0 + line;
    a[x * Lp + line] = (c < T.n_cols) ? in[(size_t)c * nx + x] : make_double2(0.0, 0.0);
  }
  cplx* r = fft_lines(a, b, px, twx, L, Lp, -1);
  TLOOP(t, L * T.cnt_max) {
    int line = t / T.cnt_max, i = t % T.cnt_max;
    int c = c0 + line;
    if (c < T.n_cols && i < T.col_cnt[c]) {
      int s = T.col_start[c] + i;
      int src = T.slot_src[s];
      cplx v = cscale(r[T.slot_ix[s] * Lp + line], scale);
      if (kin) {
        cplx p = psi[band * ldpsi + src];
        double kk = kin[src];
        v.x += kk * p.x;
        v.y += kk * p.y;
      }
      cplx* o = out + band * ldout + src;
      if (accumulate) {
        v.x += o->x;
        v.y += o->y;
      }
      *o = v;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Plain (unpruned) in-place cube passes for densities / potentials (Hartree, XC, symmetrisation).
// ------------------------------------------------------------------------------------------------
// x axis: lines are contiguous.  grid (ceil(n_lines/L), batch), n_lines = ny*nz
HD void cube_pass_x(cplx* __restrict__ data, int nx, int64_t n_lines, const FftPlan& px,
                    const cplx* twx, int sign, int L, int Lp, cplx* sm, Dim3i bid) {
  cplx* a = sm;
  cplx* b = sm + (size_t)nx * Lp;
  const int64_t l0 = (int64_t)bid.x * L;
  cplx* d = data + (size_t)bid.y * n_lines * nx;
  TLOOP(t, L * nx) {
    int line = t / nx, x = t % nx;
    a[x * Lp + line] = (l0 + line < n_lines) ? d[(size_t)(l0 + line) * nx + x] : make_double2(0.0, 0.0);
  }
  cplx* r = fft_lines(a, b, px, twx, L, Lp, sign);
  TLOOP(t, L * nx) {
    int line = t / nx, x = t % nx;
    if (l0 + line < n_lines) d[(size_t)(l0 + line) * nx + x] = r[x * Lp + line];
  }
}

// strided axis: element (i, o, x) at data[i*stride_line + o*stride_outer + x].
// grid (ceil(nx/L), n_outer, batch)
HD void cube_pass_strided(cplx* __restrict__ data, int nx, int n, int64_t stride_line,
                          int64_t stride_outer, int64_t cube_size, const FftPlan& p, const cplx* tw,
                          int sign, int L, int Lp, cplx* sm, Dim3i bid) {
  cplx* a = sm;
  cplx* b = sm + (size_t)n * Lp;
  const int x0 = bid.x * L;
  cplx* d = data + (size_t)bid.z * cube_size + (size_t)bid.y * stride_outer;
  TLOOP(t, n * L) {
    int line = t % L, i = t / L;
    int x = x0 + line;
    a[i * Lp + line] = (x < nx) ? d[(size_t)i * stride_line + x] : make_double2(0.0, 0.0);
  }
  cplx* r = fft_lines(a, b, p, tw, L, Lp, sign);
  TLOOP(t, n * L) {
    int line = t % L, i = t / L;
    int x = x0 + line;
    if (x < nx) d[(size_t)i * stride_line + x] = r[i * Lp + line];
  }
}

}  // namespace dftk
