// Batched kernels of the small-matrix LOBPCG path: every launch serves one operation of MANY independent (k, spin)
// blocks (blockIdx.y = item), so that the 29-84 small eigenproblems of BASELINE configs C1/C2/C4/C5 share launches
// and host synchronisations instead of paying them one k-block at a time (reference seam: the independent per-k solves
// of src/eigen/diag.jl:16-52).  The per-item work is the single-problem body: lobpcg_small.cuh for the small dense
// algebra, item_body below for the elementwise and reduction operations, which the direct solver path launches for one
// item through k_item.  Item descriptors (batch_exec.cuh) live in a device-side ring that the host fills per launch.
#pragma once
#include "batch_exec.cuh"

namespace dftk {

extern __shared__ __align__(16) unsigned char batch_dyn_smem[];

__global__ void __launch_bounds__(256) kb_gram(const GramItem* __restrict__ items) {
  const GramItem& it = items[blockIdx.y];
  if ((int)blockIdx.x >= it.n_ctas) return;
  small_gram_cta((int)blockIdx.x, it.rows_per_cta, it.n_rows, it.A, it.B, it.upper_only, it.ws, (cplx*)batch_dyn_smem);
  __shared__ int is_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(it.counter, 1u) == (unsigned)it.n_ctas - 1;
  __syncthreads();
  if (is_last) {
    __threadfence();
    small_gram_reduce(it.n_ctas, it.A, it.B, it.upper_only, it.ws, it.C, it.ldc);
    if (threadIdx.x == 0) *it.counter = 0;
  }
}

__global__ void __launch_bounds__(SMALL_RED) kb_chol(const CholItem* __restrict__ items) {
  const CholItem it = items[blockIdx.x];
  __shared__ cplx As[SMALL_MAX_N * SMALL_MAX_N], Bs[SMALL_MAX_N * SMALL_MAX_N];
  __shared__ double red[SMALL_RED];
  __shared__ int flag[2];
  small_chol_cta(it.O, it.ldo, it.n, it.invR, it.ldi, it.stats, As, Bs, red, flag);
}

__global__ void __launch_bounds__(128) kb_rmul(const RmulItem* __restrict__ items) {
  const RmulItem it = items[blockIdx.y];
  if ((long long)blockIdx.x * blockDim.x >= it.n_rows) return;
  cplx* rs = (cplx*)batch_dyn_smem;
  for (int e = threadIdx.x; e < it.n * it.n; e += blockDim.x) rs[e] = it.invR[e % it.n + it.ldr * (e / it.n)];
  __syncthreads();
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < it.n_rows) small_rmul_row(r, it.X, it.ld, it.n, rs, it.n);
}

__global__ void __launch_bounds__(128) kb_btimes(const BtimesItem* __restrict__ items) {
  const BtimesItem& it = items[blockIdx.y];
  if ((long long)blockIdx.x * blockDim.x >= it.n_rows) return;
  cplx* cs = (cplx*)batch_dyn_smem;
  const int ny = it.Y.start[it.Y.n];
  for (int e = threadIdx.x; e < ny * it.ncols; e += blockDim.x) cs[e] = it.cm[e % ny + it.ldcm * (e / ny)];
  __syncthreads();
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < it.n_rows) small_blocks_times_row(r, it.Y, cs, ny, it.ncols, it.out, it.ldo, it.alpha, it.beta);
}

// dynamic smem: n*n cplx (A) + 2*(n/2+1) cplx (rotations) + SMALL_RED doubles + 2*(n/2+1) ints
__global__ void __launch_bounds__(SMALL_RED) kb_heev(const HeevItem* __restrict__ items) {
  const HeevItem it = items[blockIdx.x];
  const int half = ((it.n + 1) & ~1) / 2;
  cplx* As = (cplx*)batch_dyn_smem;
  cplx* rot = As + (size_t)it.n * it.n;
  double* red = (double*)(rot + 2 * (half + 1));
  int* iw = (int*)(red + SMALL_RED);
  small_heev_cta(it.G, it.ldg, it.n, it.w, As, it.V, rot, red, iw, it.stats, it.lam_out, it.n_keep);
}

// block reduction helper: sums a and b over the CTA (blockDim multiple of 32, <= 1024); results valid on thread 0
__device__ __forceinline__ void block_sum2(double& a, double& b) {
  __shared__ double ra[32], rb[32];
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_down_sync(0xffffffffu, a, o);
    b += __shfl_down_sync(0xffffffffu, b, o);
  }
  if ((threadIdx.x & 31) == 0) {
    ra[threadIdx.x >> 5] = a;
    rb[threadIdx.x >> 5] = b;
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    const int nw = blockDim.x >> 5;
    a = (int)threadIdx.x < nw ? ra[threadIdx.x] : 0.0;
    b = (int)threadIdx.x < nw ? rb[threadIdx.x] : 0.0;
    for (int o = 16; o > 0; o >>= 1) {
      a += __shfl_down_sync(0xffffffffu, a, o);
      b += __shfl_down_sync(0xffffffffu, b, o);
    }
  }
}

// compute_λ of the start vectors: lam = real(<x|Ax> / <x|x>)   (lobpcg_hyper_impl.jl:341-344)
__global__ void __launch_bounds__(256) kb_lambda(const LambdaItem* __restrict__ items) {
  const LambdaItem it = items[blockIdx.y];
  const int col = blockIdx.x;
  if (col >= it.n_cols) return;
  const cplx* x = it.X + it.ld * col;
  const cplx* ax = it.AX + it.ld * col;
  double nre = 0.0, nim = 0.0, d = 0.0, dz = 0.0;
  for (long long i = threadIdx.x; i < it.n_rows; i += blockDim.x) {
    const cplx a = x[i], b = ax[i];
    nre += a.x * b.x + a.y * b.y;
    nim += a.x * b.y - a.y * b.x;
    d += a.x * a.x + a.y * a.y;
  }
  block_sum2(nre, nim);
  __syncthreads();
  block_sum2(d, dz);
  if (threadIdx.x == 0) it.lam[col] = nre / d;    // <x|x> is real: the complex division keeps the real part only
}

// ---- The block operations shared by both solver paths.  Each has ONE per-item body, run by two entry shapes: the batched
//      kb_* kernel (items[blockIdx.y], or items[blockIdx.x] for one-CTA items, from the descriptor ring) and k_item (a single
//      item passed by value as the kernel parameter: the direct path, no descriptor upload).  The elementwise bodies loop
//      with a grid stride; a direct launch of one thread per element runs one iteration per thread.

// R = AX - X lam; norms = ||R||; meankin = <X|kin|X>  (one CTA per column; lobpcg_hyper_impl.jl:443-445 + precondprep!)
// squared: norms = ||R||^2 of this rank's rows (slab solves: summed over the ranks, then square-rooted)
__device__ __forceinline__ void item_body(const ResidualItem& it) {
  const int col = blockIdx.x;
  if (col >= it.n_cols) return;
  const cplx* ax = it.AX + it.ld * col;
  const cplx* x = it.X + it.ld * col;
  cplx* r = it.R + it.ld * col;
  const double l = it.lam[col];
  double s = 0.0, mk = 0.0;
  for (long long i = threadIdx.x; i < it.n_rows; i += blockDim.x) {
    const cplx a = ax[i], b = x[i];
    const cplx v = make_double2(a.x - l * b.x, a.y - l * b.y);
    r[i] = v;
    s += v.x * v.x + v.y * v.y;
    if (it.kin) mk += it.kin[i] * (b.x * b.x + b.y * b.y);
  }
  block_sum2(s, mk);
  if (threadIdx.x == 0) {
    it.norms[col] = it.squared ? s : sqrt(s);
    it.meankin[col] = mk;
  }
}

// R[:,n] *= mk_n / (mk_n + kin)    (ldiv!(::PreconditionerTPA), src/gpu/linalg.jl:29-36)
__device__ __forceinline__ void item_body(const PrecondItem& it) {
  const long long total = it.n_rows * it.n_cols;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long i = idx % it.n_rows, c = idx / it.n_rows;
    const double mk = it.meankin[c];
    const double f = mk / (mk + it.kin[i]);
    cplx v = it.R[i + it.ld * c];
    it.R[i + it.ld * c] = make_double2(v.x * f, v.y * f);
  }
}

// norms = ||X[:,n]|| (||X[:,n]||^2 when `squared`, as for the residual); one CTA per column
__device__ __forceinline__ void item_body(const ColnormItem& it) {
  const int col = blockIdx.x;
  if (col >= it.n_cols) return;
  const cplx* x = it.X + it.ld * col;
  double s = 0.0, z = 0.0;
  for (long long i = threadIdx.x; i < it.n_rows; i += blockDim.x) {
    const cplx v = x[i];
    s += v.x * v.x + v.y * v.y;
  }
  block_sum2(s, z);
  if (threadIdx.x == 0) it.norms[col] = it.squared ? s : sqrt(s);
}

__device__ __forceinline__ void item_body(const ScaleItem& it) {
  const long long total = it.n_rows * it.n_cols;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long i = idx % it.n_rows, c = idx / it.n_rows;
    const double f = 1.0 / it.norms[c];
    cplx v = it.X[i + it.ld * c];
    it.X[i + it.ld * c] = make_double2(v.x * f, v.y * f);
  }
}

// strided 2D copy (dst and src column-major with different leading dimensions)
__device__ __forceinline__ void item_body(const Copy2dItem& it) {
  const long long total = it.n_rows * it.n_cols;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const long long i = idx % it.n_rows, c = idx / it.n_rows;
    it.dst[i + it.ldd * c] = it.src ? it.src[i + it.lds * c] : make_double2(0.0, 0.0);
  }
}

// cP = cX[:, c0:] - e,  e[c0 + c, c] = 1 for c < lenXn   (lobpcg_hyper_impl.jl:495-503)
__device__ __forceinline__ void item_body(const MakecpItem& it) {
  const int total = it.n_rows * it.n_cols;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int i = idx % it.n_rows, c = idx / it.n_rows;
    const int cc = c + it.c0;
    cplx v = it.cX[i + it.ld * cc];
    if (cc < it.lenXn && i == it.c0 + cc) v.x -= 1.0;
    it.cP[i + it.ld * c] = v;
  }
}

// stats[0] = max |diag|, stats[1] = sum |offdiag|^2, stats[2] = #nan/inf, stats[3] = sum |all|^2   (one CTA, <= 1024 threads)
__device__ __forceinline__ void item_body(const StatsItem& it) {
  double md = 0.0, so = 0.0, bad = 0.0, sa = 0.0;
  for (int idx = threadIdx.x; idx < it.n_rows * it.n_cols; idx += blockDim.x) {
    const int i = idx % it.n_rows, j = idx / it.n_rows;
    const cplx v = it.A[i + it.ld * j];
    const double a2 = v.x * v.x + v.y * v.y;
    if (!isfinite(a2)) bad += 1.0;
    sa += a2;
    if (i == j) md = fmax(md, sqrt(a2));
    else so += a2;
  }
  __shared__ double r0[32];
  for (int o = 16; o > 0; o >>= 1) md = fmax(md, __shfl_down_sync(0xffffffffu, md, o));
  if ((threadIdx.x & 31) == 0) r0[threadIdx.x >> 5] = md;
  __syncthreads();
  block_sum2(so, bad);
  __syncthreads();
  double z = 0.0;
  block_sum2(sa, z);
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) md = fmax(md, r0[w]);
    it.stats[0] = md;
    it.stats[1] = so;
    it.stats[2] = bad;
    it.stats[3] = sa;
  }
}

// counter-based normal random numbers (random start vectors, drop_small!'s re-randomisation; statistically plain):
// x[i] from the SplitMix64 finaliser of the counters seed + 2i and seed + 2i + 1
__device__ __forceinline__ unsigned long long counter_hash(unsigned long long x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__device__ __forceinline__ void item_body(const RandnItem& it) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < it.n_rows; i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long a = counter_hash(it.seed + 2 * (unsigned long long)i), b = counter_hash(it.seed + 2 * (unsigned long long)i + 1);
    const double u1 = ((a >> 11) + 1.0) * (1.0 / 9007199254740993.0);
    const double u2 = (b >> 11) * (1.0 / 9007199254740992.0);
    const double r = sqrt(-2.0 * log(u1));
    it.x[i] = make_double2(r * cospi(2.0 * u2) * 0.70710678118654752, r * sinpi(2.0 * u2) * 0.70710678118654752);
  }
}

template <class Item>
__global__ void k_item(const Item it) { item_body(it); }

// the item is read in place: a copy would hold `squared` in a register through the loop (48 instead of 40 registers)
__global__ void __launch_bounds__(256) kb_residual(const ResidualItem* __restrict__ items) { item_body(items[blockIdx.y]); }
__global__ void __launch_bounds__(256) kb_precondition(const PrecondItem* __restrict__ items) {
  const PrecondItem it = items[blockIdx.y];
  item_body(it);
}
__global__ void __launch_bounds__(256) kb_col_norms(const ColnormItem* __restrict__ items) {
  const ColnormItem it = items[blockIdx.y];
  item_body(it);
}
__global__ void __launch_bounds__(256) kb_scale_cols_inv(const ScaleItem* __restrict__ items) {
  const ScaleItem it = items[blockIdx.y];
  item_body(it);
}
__global__ void __launch_bounds__(256) kb_copy2d(const Copy2dItem* __restrict__ items) {
  const Copy2dItem it = items[blockIdx.y];
  item_body(it);
}
__global__ void __launch_bounds__(256) kb_make_cP(const MakecpItem* __restrict__ items) {
  const MakecpItem it = items[blockIdx.y];
  item_body(it);
}
__global__ void __launch_bounds__(256) kb_matrix_stats(const StatsItem* __restrict__ items) {   // one CTA per item
  const StatsItem it = items[blockIdx.x];
  item_body(it);
}
__global__ void __launch_bounds__(256) kb_randn_col(const RandnItem* __restrict__ items) {
  const RandnItem it = items[blockIdx.y];
  item_body(it);
}

// <x_n|kin|x_n> per band (ene_ops(::TermKinetic), src/terms/kinetic.jl:40-57); one CTA per (band, item)
__global__ void __launch_bounds__(256) kb_kin_dots(const KinDotsItem* __restrict__ items) {
  const KinDotsItem it = items[blockIdx.y];
  const int col = blockIdx.x;
  if (col >= it.n_cols) return;
  const cplx* x = it.X + it.ld * col;
  double s = 0.0, z = 0.0;
  for (long long i = threadIdx.x; i < it.n_rows; i += blockDim.x) {
    const cplx v = x[i];
    s += it.kin[i] * (v.x * v.x + v.y * v.y);
  }
  block_sum2(s, z);
  if (threadIdx.x == 0) it.out[col] = s;
}
// <psi_n|P D P'|psi_n> = Re sum_ij conj(proj_in) D_ij proj_jn per band (ene_ops(::TermAtomicNonlocal), nonlocal.jl:31-47)
__global__ void __launch_bounds__(64) kb_nl_energy(const NlEnergyItem* __restrict__ items) {
  const NlEnergyItem it = items[blockIdx.x];
  for (int b = threadIdx.x; b < it.nb; b += blockDim.x) {
    const cplx* p = it.proj + (long long)it.np * b;
    double e = 0.0;
    for (int j = 0; j < it.np; ++j) {
      const cplx pj = p[j];
      double sx = 0.0, sy = 0.0;               // (D p)_... accumulated as conj(p_i) D_ij, D real symmetric stored complex
      for (int i = 0; i < it.np; ++i) {
        const double d = it.D[i + (long long)it.np * j].x;
        sx += d * p[i].x;
        sy += d * p[i].y;
      }
      e += sx * pj.x + sy * pj.y;
    }
    it.out[b] = e;
  }
}

// collect the small per-item results of a round into one contiguous buffer (one D2H copy per round instead of one per item)
__global__ void __launch_bounds__(64) kb_gather(const GatherItem* __restrict__ items, double* __restrict__ out) {
  const GatherItem it = items[blockIdx.x];
  for (int i = threadIdx.x; i < it.n; i += blockDim.x) out[it.offset + i] = it.src[i];
}

}  // namespace dftk
