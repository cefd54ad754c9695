// Dense complex128 kernels of the hot path:
//   * zgemm_cn : C(m x n) = alpha * A^H B + beta * C, A: K x m, B: K x n, K = N_pw huge  ("Gram" type:
//                P'psi, X'AX blocks, BY'X)                      -- src/terms/operators.jl:127,
//                src/eigen/lobpcg_hyper_impl.jl:90-113,216-221,277
//   * zgemm_nn : C(K x n) = alpha * A(K x m) B(m x n) + beta * C              ("update" type:
//                Hpsi += P (D P'psi), new_X = Y cX, X -= Y (BY'X), X = X invR) -- lobpcg_hyper_impl.jl:124-137
// Both are real FP64 tensor-core GEMMs on the interleaved complex storage, built on mma.sync.m16n8k16.f64
// (DMMA.16x8x16, 2048 MACs per warp instruction; Hopper's wgmma has no f64 form).  With A~ the real (2K x m) view of A
// (rows re,im,re,im,...),
//   Re(A^H B) = A~^T B~,   Im(A^H B) = A~^T (J B~),   (J b)[2k] = b[2k+1], (J b)[2k+1] = -b[2k]
// and for the update C~ = A^ B~ with A^[:,2i] = A~[:,i], A^[:,2i+1] = J' A~[:,i].
// The contraction index of an MMA may be permuted as long as both operands agree: the four k slots a lane holds
// (t, t+4, t+8, t+12 with t = lane % 4) are mapped to the real indices 4t .. 4t+3, i.e. two whole complex numbers.
// Fragments then load with LDS.128 and the J-images are formed in registers (a swap and a sign), so no operand is
// ever materialised twice.  Tiles are staged with cp.async in a STAGES-deep ring (ctx->gemm_stages).
#include "structs.cuh"

namespace dftk {

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool pred) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  int sz = pred ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}
// c += a b: A 16 x 16 (rows g, g+8 for a[even], a[odd]; k slot i/2), B 16 x 8 (k slot i, column g), C 16 x 8
// (c[0..1]: row g, columns 2t, 2t+1; c[2..3]: row g+8), g = lane / 4, t = lane % 4
__device__ __forceinline__ void dmma16(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
  asm("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
      "{%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
      : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}
// sign flip with an integer XOR (ALU pipe, keeps the FP64 pipe free)
__device__ __forceinline__ double neg(double x) {
  return __hiloint2double(__double2hiint(x) ^ (int)0x80000000, __double2loint(x));
}
__device__ __forceinline__ double2 lds128(const double* p) { return *(const double2*)p; }
// number of MMA tiles of `size` rows (at most `cap`) needed to cover `rem` remaining outputs
__device__ __forceinline__ int mma_tiles(int64_t rem, int size, int cap) {
  return rem <= 0 ? 0 : rem >= (int64_t)size * cap ? cap : (int)((rem + size - 1) / size);
}

#define GEMM_THREADS 256    // 8 warps, one CTA per SM (the accumulators and fragments take ~200 registers per thread)
#define BKC 16              // complex k per stage (32 real: two k16 MMA steps)
#define LDK (2 * BKC + 2)   // doubles per k-major smem row; LDK % 4 == 2 => the LDS.128 fragment loads of a quarter warp
                            // (rows g, g+1; doubles 4t .. 4t+3) hit eight distinct 16-byte bank groups

// ------------------------------------------------------------------------------------------------
// Gram kernel.  CTA tile: 64 (i) x 96 (j) complex outputs; warp w owns i in 32 (w & 1) + [0, 32), j in 24 (w >> 1) +
// [0, 24).  96 columns cover the 259 bands of the benchmark cell in 3 tiles (11 % padding).  Partial sums over the
// K-slice [k_begin, k_end) are written to ws[split][m x n]; k_reduce_partials applies alpha/beta.
// ------------------------------------------------------------------------------------------------
#define GT_M 64
#define GT_N 96
template <int STAGES>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
k_zgemm_cn(const cplx* __restrict__ A, int64_t lda, const cplx* __restrict__ B, int64_t ldb,
           cplx* __restrict__ ws, int64_t m, int64_t n, int64_t K, int64_t k_per_split, int upper_only) {
  // Hermitian results (X'X, X'AX): tiles strictly below the diagonal are never read by the callers
  if (upper_only && (int64_t)blockIdx.x * GT_M >= (int64_t)blockIdx.y * GT_N + GT_N) return;
  extern __shared__ __align__(16) double smem_d[];
  double* As = smem_d;                              // [STAGES][GT_M][LDK]
  double* Bs = smem_d + STAGES * GT_M * LDK;        // [STAGES][GT_N][LDK]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t i0 = (int64_t)blockIdx.x * GT_M, j0 = (int64_t)blockIdx.y * GT_N;
  const int64_t kb = (int64_t)blockIdx.z * k_per_split;
  const int64_t ke = min(K, kb + k_per_split);
  const int nkt = (int)((ke - kb + BKC - 1) / BKC);
  const int wi = (warp & 1) * 32, wj = (warp >> 1) * 24;

  // Per-thread copy plan (fixed across k tiles): element e = tid + 256 r -> column tid/16 + 16 r, k tid%16.
  const int lkk = tid & (BKC - 1), lcol = tid >> 4;
  const cplx* pA = A + kb + lkk + lda * (i0 + lcol);
  const cplx* pB = B + kb + lkk + ldb * (j0 + lcol);
  unsigned okA = 0, okB = 0;   // column-in-range masks
#pragma unroll
  for (int r = 0; r < GT_M / 16; ++r) okA |= (i0 + lcol + 16 * r < m) ? (1u << r) : 0u;
#pragma unroll
  for (int r = 0; r < GT_N / 16; ++r) okB |= (j0 + lcol + 16 * r < n) ? (1u << r) : 0u;
  auto load_tile = [&](int kt, int slot) {
    const int64_t koff = (int64_t)kt * BKC;
    const bool rowok = kb + koff + lkk < ke;
    double* da = As + ((size_t)slot * GT_M + lcol) * LDK + 2 * lkk;
    double* db = Bs + ((size_t)slot * GT_N + lcol) * LDK + 2 * lkk;
#pragma unroll
    for (int r = 0; r < GT_M / 16; ++r) {
      bool ok = rowok && ((okA >> r) & 1u);
      cp_async16(da + (size_t)16 * r * LDK, ok ? (pA + koff + (int64_t)16 * r * lda) : A, ok);
    }
#pragma unroll
    for (int r = 0; r < GT_N / 16; ++r) {
      bool ok = rowok && ((okB >> r) & 1u);
      cp_async16(db + (size_t)16 * r * LDK, ok ? (pB + koff + (int64_t)16 * r * ldb) : B, ok);
    }
  };

  double cr[2][3][4], ci[2][3][4];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b)
#pragma unroll
      for (int e = 0; e < 4; ++e) cr[a][b][e] = ci[a][b][e] = 0.0;

  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < nkt) load_tile(s, s);
    cp_async_commit();
  }
  const int g = lane >> 2, t = lane & 3;
  // MMA tiles of this warp that hold outputs (warp-uniform): narrow products skip the MMAs on padding
  const int na = mma_tiles(m - i0 - wi, 16, 2), nb = mma_tiles(n - j0 - wj, 8, 3);
  for (int kt = 0; kt < nkt; ++kt) {
    cp_async_wait<STAGES - 2>();
    __syncthreads();
    {
      int nxt = kt + STAGES - 1;
      if (nxt < nkt) load_tile(nxt, nxt % STAGES);
      cp_async_commit();
    }
    const double* as = As + (size_t)(kt % STAGES) * GT_M * LDK + 4 * t;
    const double* bs = Bs + (size_t)(kt % STAGES) * GT_N * LDK + 4 * t;
#pragma unroll
    for (int ks = 0; ks < BKC / 8; ++ks) {
      double af[2][8];
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        const double* p = as + (wi + 16 * a + g) * LDK + 16 * ks;
        const double2 x0 = lds128(p), x1 = lds128(p + 2), y0 = lds128(p + 8 * LDK), y1 = lds128(p + 8 * LDK + 2);
        af[a][0] = x0.x; af[a][1] = y0.x; af[a][2] = x0.y; af[a][3] = y0.y;
        af[a][4] = x1.x; af[a][5] = y1.x; af[a][6] = x1.y; af[a][7] = y1.y;
      }
#pragma unroll
      for (int b = 0; b < 3; ++b) {
        const double* p = bs + (wj + 8 * b + g) * LDK + 16 * ks;
        const double2 v0 = lds128(p), v1 = lds128(p + 2);
        const double bf[4] = {v0.x, v0.y, v1.x, v1.y};
        const double bh[4] = {v0.y, neg(v0.x), v1.y, neg(v1.x)};   // J-image
#pragma unroll
        for (int a = 0; a < 2; ++a) {
          if (a < na && b < nb) {
            dmma16(cr[a][b], af[a], bf);
            dmma16(ci[a][b], af[a], bh);
          }
        }
      }
    }
  }
  cp_async_wait<0>();
  cplx* out = ws + (size_t)blockIdx.z * m * n;
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        int64_t gi = i0 + wi + 16 * a + g + 8 * (e >> 1);
        int64_t gj = j0 + wj + 8 * b + 2 * t + (e & 1);
        if (gi < m && gj < n) out[gi + m * gj] = make_double2(cr[a][b][e], ci[a][b][e]);
      }
}

__global__ void k_reduce_partials(const cplx* __restrict__ ws, int nsplit, int64_t m, int64_t n,
                                  cplx alpha, cplx beta, cplx* __restrict__ C, int64_t ldc) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= m * n) return;
  int64_t i = idx % m, j = idx / m;
  double sx = 0.0, sy = 0.0;
  for (int s = 0; s < nsplit; ++s) {
    cplx v = ws[(size_t)s * m * n + idx];
    sx += v.x;
    sy += v.y;
  }
  cplx r = cmul(alpha, make_double2(sx, sy));
  if (beta.x != 0.0 || beta.y != 0.0) r = cadd(r, cmul(beta, C[i + ldc * j]));
  C[i + ldc * j] = r;
}

// ------------------------------------------------------------------------------------------------
// Update kernel.  CTA tile: 64 complex rows x 96 columns; warp w owns rows 32 (w & 1) + [0, 32), columns 24 (w >> 1) +
// [0, 24).  An MMA covers 8 complex rows: its rows g and g+8 are the real and imaginary parts of complex row g, so a
// lane holds whole complex outputs and the epilogue needs no shuffles.
// ------------------------------------------------------------------------------------------------
#define UT_M 64                 // complex rows
#define UT_N 96
#define LDA_U (2 * UT_M + 2)    // doubles per inner-index row of the A tile; LDA_U % 8 == 2 => conflict-free LDS.128
template <int STAGES>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
k_zgemm_nn(const cplx* __restrict__ A, int64_t lda, const cplx* __restrict__ B, int64_t ldb,
           cplx* __restrict__ C, int64_t ldc, int64_t Krows, int64_t n, int64_t m, cplx alpha, cplx beta,
           int b_upper) {
  extern __shared__ __align__(16) double smem_d[];
  double* As = smem_d;                              // [STAGES][BKC][LDA_U]
  double* Bs = smem_d + STAGES * BKC * LDA_U;       // [STAGES][UT_N][LDK]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // blockIdx.x = column tile (fastest): CTAs sharing one A row panel run together and hit it in L2
  const int64_t r0 = (int64_t)blockIdx.y * UT_M, j0 = (int64_t)blockIdx.x * UT_N;
  // B upper triangular (X * inv(R), rmul! with an UpperTriangular): rows i > j of column j are zero
  const int64_t m_eff = b_upper ? min(m, j0 + UT_N) : m;
  const int nkt = (int)((m_eff + BKC - 1) / BKC);
  const int wr = (warp & 1) * 32, wj = (warp >> 1) * 24;

  // Per-thread copy plan: A tile element e = tid + 256 r -> inner index e/64 = tid/64 + 4 r, row e%64 = tid%64;
  //                       B tile element e = tid + 256 r -> column tid/16 + 16 r, inner index tid%16.
  const int arow = tid & (UT_M - 1), aii = tid >> 6;
  const int bii = tid & (BKC - 1), bcol = tid >> 4;
  const bool arow_ok = r0 + arow < Krows;
  const cplx* pA = A + (r0 + arow) + lda * aii;
  const cplx* pB = B + bii + ldb * (j0 + bcol);
  unsigned okB = 0;
#pragma unroll
  for (int r = 0; r < UT_N / 16; ++r) okB |= (j0 + bcol + 16 * r < n) ? (1u << r) : 0u;
  auto load_tile = [&](int kt, int slot) {
    const int64_t i0 = (int64_t)kt * BKC;
    double* da = As + ((size_t)slot * BKC + aii) * LDA_U + 2 * arow;
    double* db = Bs + ((size_t)slot * UT_N + bcol) * LDK + 2 * bii;
#pragma unroll
    for (int r = 0; r < BKC / 4; ++r) {
      bool ok = arow_ok && (i0 + aii + 4 * r < m_eff);
      cp_async16(da + (size_t)4 * r * LDA_U, ok ? (pA + (i0 + 4 * r) * lda) : A, ok);
    }
    const bool iiok = i0 + bii < m_eff;
#pragma unroll
    for (int r = 0; r < UT_N / 16; ++r) {
      bool ok = iiok && ((okB >> r) & 1u);
      cp_async16(db + (size_t)16 * r * LDK, ok ? (pB + i0 + (int64_t)16 * r * ldb) : B, ok);
    }
  };

  double acc[4][3][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[a][b][e] = 0.0;

  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < nkt) load_tile(s, s);
    cp_async_commit();
  }
  const int g = lane >> 2, t = lane & 3;
  // MMA tiles of this warp that hold outputs (warp-uniform): narrow products skip the MMAs on padding
  const int na = mma_tiles(Krows - r0 - wr, 8, 4), nb = mma_tiles(n - j0 - wj, 8, 3);
  for (int kt = 0; kt < nkt; ++kt) {
    cp_async_wait<STAGES - 2>();
    __syncthreads();
    {
      int nxt = kt + STAGES - 1;
      if (nxt < nkt) load_tile(nxt, nxt % STAGES);
      cp_async_commit();
    }
    const double* as = As + (size_t)(kt % STAGES) * BKC * LDA_U + 2 * t * LDA_U + 2 * (wr + g);
    const double* bs = Bs + (size_t)(kt % STAGES) * UT_N * LDK + 4 * t;
#pragma unroll
    for (int ks = 0; ks < BKC / 8; ++ks) {
      // k slots 4t .. 4t+3 = (inner 2t, re), (2t, im), (2t+1, re), (2t+1, im); rows g / g+8 = Re / Im of the output row:
      //   Re row: Ar Br - Ai Bi,   Im row: Ai Br + Ar Bi
      double bf[3][4];
#pragma unroll
      for (int b = 0; b < 3; ++b) {
        const double* p = bs + (wj + 8 * b + g) * LDK + 16 * ks;
        const double2 v0 = lds128(p), v1 = lds128(p + 2);
        bf[b][0] = v0.x; bf[b][1] = v0.y; bf[b][2] = v1.x; bf[b][3] = v1.y;
      }
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        const double* p = as + 8 * ks * LDA_U + 16 * a;
        const double2 z0 = lds128(p), z1 = lds128(p + LDA_U);
        const double af[8] = {z0.x, z0.y, neg(z0.y), z0.x, z1.x, z1.y, neg(z1.y), z1.x};
#pragma unroll
        for (int b = 0; b < 3; ++b)
          if (a < na && b < nb) dmma16(acc[a][b], af, bf[b]);
      }
    }
  }
  cp_async_wait<0>();
  const bool has_beta = (beta.x != 0.0 || beta.y != 0.0);
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int64_t grow = r0 + wr + 8 * a + g;
        const int64_t gj = j0 + wj + 8 * b + 2 * t + e;
        if (grow < Krows && gj < n) {
          cplx o = cmul(alpha, make_double2(acc[a][b][e], acc[a][b][2 + e]));
          if (has_beta) o = cadd(o, cmul(beta, C[grow + ldc * gj]));
          C[grow + ldc * gj] = o;
        }
      }
}

// ------------------------------------------------------------------------------------------------
// Real-A forms of the two products, for the time-reversal fold of the nonlocal apply (kb_apply_nonlocal_folded).  A is
// real (R = [Pr; Pi], K' x m column-major), B and C are complex.  An MMA k step covers 16 complex k: A supplies 16 real
// k, and each lane's four complex B values give a real and an imaginary B fragment, so one A fragment feeds two MMAs
// (Re and Im of the result).  Per complex k that is half the DMMA work of k_zgemm_cn / k_zgemm_nn.
// ------------------------------------------------------------------------------------------------
#define RBK 32            // complex k per stage of the real-A kernels (two k16 MMA steps)
#define RLDK (2 * RBK + 2) // doubles per k-major row of the Gram's B tile; RLDK % 4 == 2 => conflict-free LDS.128 (as LDK)
#define LDR (RBK + 2)      // doubles per k-major row of the Gram's real A tile; LDR % 4 == 2 likewise
// Position of complex k in a k-major B row of the real-A Gram: lanes t = 0..3 of a quarter warp read complex
// 16 ks + 4t + s, which would put t and t + 2 on one 16-byte bank group; XOR-ing 2 where bit 3 is set spreads them.
__device__ __forceinline__ int bswz(int k) { return k ^ ((k >> 2) & 2); }

// Gram, real A: ws[split] (m x n) = A^T B over the K-slice of the split.  Same tiles, warp layout, copy ring and
// split-K as k_zgemm_cn; K, lda and the split length must be even (a 16-byte copy holds two real k).  Lane (g, t)
// takes k 4t .. 4t+3 of the stage in its four k slots, for A and B alike.
template <int STAGES>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
k_rgemm_cn(const double* __restrict__ A, int64_t lda, const cplx* __restrict__ B, int64_t ldb,
           cplx* __restrict__ ws, int64_t m, int64_t n, int64_t K, int64_t k_per_split) {
  extern __shared__ __align__(16) double smem_d[];
  double* As = smem_d;                              // [STAGES][GT_M][LDR]
  double* Bs = smem_d + STAGES * GT_M * LDR;        // [STAGES][GT_N][RLDK], complex k at bswz(k)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t i0 = (int64_t)blockIdx.x * GT_M, j0 = (int64_t)blockIdx.y * GT_N;
  const int64_t kb = (int64_t)blockIdx.z * k_per_split;
  const int64_t ke = min(K, kb + k_per_split);
  const int nkt = (int)((ke - kb + RBK - 1) / RBK);
  const int wi = (warp & 1) * 32, wj = (warp >> 1) * 24;

  // Per-thread copy plan: A element (two reals) e = tid + 256 r -> column tid/16 + 16 r, k 2 (tid%16);
  //                       B element e = tid + 256 r -> column tid/32 + 8 r, complex k tid%32.
  const int akk = 2 * (tid & 15), acol = tid >> 4;
  const int lkk = tid & (RBK - 1), lcol = tid >> 5;
  const double* pA = A + kb + akk + lda * (i0 + acol);
  const cplx* pB = B + kb + lkk + ldb * (j0 + lcol);
  unsigned okA = 0, okB = 0;
#pragma unroll
  for (int r = 0; r < GT_M / 16; ++r) okA |= (i0 + acol + 16 * r < m) ? (1u << r) : 0u;
#pragma unroll
  for (int r = 0; r < GT_N / 8; ++r) okB |= (j0 + lcol + 8 * r < n) ? (1u << r) : 0u;
  auto load_tile = [&](int kt, int slot) {
    const int64_t koff = (int64_t)kt * RBK;
    const bool aok = kb + koff + akk < ke;
    const bool rowok = kb + koff + lkk < ke;
    double* da = As + ((size_t)slot * GT_M + acol) * LDR + akk;
    double* db = Bs + ((size_t)slot * GT_N + lcol) * RLDK + 2 * bswz(lkk);
#pragma unroll
    for (int r = 0; r < GT_M / 16; ++r) {
      bool ok = aok && ((okA >> r) & 1u);
      cp_async16(da + (size_t)16 * r * LDR, ok ? (pA + koff + (int64_t)16 * r * lda) : A, ok);
    }
#pragma unroll
    for (int r = 0; r < GT_N / 8; ++r) {
      bool ok = rowok && ((okB >> r) & 1u);
      cp_async16(db + (size_t)8 * r * RLDK, ok ? (pB + koff + (int64_t)8 * r * ldb) : B, ok);
    }
  };

  double cr[2][3][4], ci[2][3][4];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b)
#pragma unroll
      for (int e = 0; e < 4; ++e) cr[a][b][e] = ci[a][b][e] = 0.0;

  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < nkt) load_tile(s, s);
    cp_async_commit();
  }
  const int g = lane >> 2, t = lane & 3;
  const int na = mma_tiles(m - i0 - wi, 16, 2), nb = mma_tiles(n - j0 - wj, 8, 3);
  for (int kt = 0; kt < nkt; ++kt) {
    cp_async_wait<STAGES - 2>();
    __syncthreads();
    {
      int nxt = kt + STAGES - 1;
      if (nxt < nkt) load_tile(nxt, nxt % STAGES);
      cp_async_commit();
    }
    const double* as = As + (size_t)(kt % STAGES) * GT_M * LDR + 4 * t;
    const double* bs = Bs + (size_t)(kt % STAGES) * GT_N * RLDK;
#pragma unroll
    for (int ks = 0; ks < RBK / 16; ++ks) {
    double af[2][8];
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const double* p = as + (wi + 16 * a + g) * LDR + 16 * ks;
      const double2 x0 = lds128(p), x1 = lds128(p + 2), y0 = lds128(p + 8 * LDR), y1 = lds128(p + 8 * LDR + 2);
      af[a][0] = x0.x; af[a][1] = y0.x; af[a][2] = x0.y; af[a][3] = y0.y;
      af[a][4] = x1.x; af[a][5] = y1.x; af[a][6] = x1.y; af[a][7] = y1.y;
    }
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      const double* p = bs + (wj + 8 * b + g) * RLDK;
      double br[4], bi[4];
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        const double2 v = lds128(p + 2 * bswz(16 * ks + 4 * t + s));
        br[s] = v.x;
        bi[s] = v.y;
      }
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        if (a < na && b < nb) {
          dmma16(cr[a][b], af[a], br);
          dmma16(ci[a][b], af[a], bi);
        }
      }
    }
    }
  }
  cp_async_wait<0>();
  cplx* out = ws + (size_t)blockIdx.z * m * n;
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        int64_t gi = i0 + wi + 16 * a + g + 8 * (e >> 1);
        int64_t gj = j0 + wj + 8 * b + 2 * t + (e & 1);
        if (gi < m && gj < n) out[gi + m * gj] = make_double2(cr[a][b][e], ci[a][b][e]);
      }
}

// Update, real A: C (Krows x n) = A (Krows x m, real) B (m x n).  CTA tile 64 rows x 96 columns, warp w owns rows
// 32 (w & 1) + [0, 32), columns 24 (w >> 1) + [0, 24).  Lane (g, t) takes inner index t + 4s in k slot s; MMA rows g and
// g + 8 are the output rows 2g and 2g + 1 of its 16-row block, so one LDS.128 of the row-major A tile loads both.
// Krows and lda must be even.
#define LDRU (UT_M + 4)       // doubles per inner-index row of the real A tile; LDRU / 2 % 8 == 2 => conflict-free LDS.128
#define LDBU (2 * RBK + 8)    // doubles per column of the B tile;              LDBU / 2 % 8 == 4 => conflict-free LDS.128
template <int STAGES>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
k_rgemm_nn(const double* __restrict__ A, int64_t lda, const cplx* __restrict__ B, int64_t ldb,
           cplx* __restrict__ C, int64_t ldc, int64_t Krows, int64_t n, int64_t m) {
  extern __shared__ __align__(16) double smem_d[];
  double* As = smem_d;                              // [STAGES][RBK][LDRU]
  double* Bs = smem_d + STAGES * RBK * LDRU;        // [STAGES][UT_N][LDBU]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t r0 = (int64_t)blockIdx.y * UT_M, j0 = (int64_t)blockIdx.x * UT_N;
  const int nkt = (int)((m + RBK - 1) / RBK);
  const int wr = (warp & 1) * 32, wj = (warp >> 1) * 24;

  // Per-thread copy plan: A element (two reals) e = tid + 256 r -> inner index tid/32 + 8 r, rows 2 (tid%32);
  //                       B element e = tid + 256 r -> column tid/32 + 8 r, inner index tid%32.
  const int arow = 2 * (tid & 31), aii = tid >> 5;
  const int bii = tid & (RBK - 1), bcol = tid >> 5;
  const bool arow_ok = r0 + arow < Krows;
  const double* pA = A + (r0 + arow) + lda * aii;
  const cplx* pB = B + bii + ldb * (j0 + bcol);
  unsigned okB = 0;
#pragma unroll
  for (int r = 0; r < UT_N / 8; ++r) okB |= (j0 + bcol + 8 * r < n) ? (1u << r) : 0u;
  auto load_tile = [&](int kt, int slot) {
    const int64_t i0 = (int64_t)kt * RBK;
    double* da = As + ((size_t)slot * RBK + aii) * LDRU + arow;
    double* db = Bs + ((size_t)slot * UT_N + bcol) * LDBU + 2 * bii;
#pragma unroll
    for (int r = 0; r < RBK / 8; ++r) {
      bool ok = arow_ok && (i0 + aii + 8 * r < m);
      cp_async16(da + (size_t)8 * r * LDRU, ok ? (pA + (i0 + 8 * r) * lda) : A, ok);
    }
    const bool iiok = i0 + bii < m;
#pragma unroll
    for (int r = 0; r < UT_N / 8; ++r) {
      bool ok = iiok && ((okB >> r) & 1u);
      cp_async16(db + (size_t)8 * r * LDBU, ok ? (pB + i0 + (int64_t)8 * r * ldb) : B, ok);
    }
  };

  double ar[2][3][4], ai[2][3][4];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b)
#pragma unroll
      for (int e = 0; e < 4; ++e) ar[a][b][e] = ai[a][b][e] = 0.0;

  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < nkt) load_tile(s, s);
    cp_async_commit();
  }
  const int g = lane >> 2, t = lane & 3;
  const int na = mma_tiles(Krows - r0 - wr, 16, 2), nb = mma_tiles(n - j0 - wj, 8, 3);
  for (int kt = 0; kt < nkt; ++kt) {
    cp_async_wait<STAGES - 2>();
    __syncthreads();
    {
      int nxt = kt + STAGES - 1;
      if (nxt < nkt) load_tile(nxt, nxt % STAGES);
      cp_async_commit();
    }
    const double* as = As + (size_t)(kt % STAGES) * RBK * LDRU + t * LDRU + wr + 2 * g;
    const double* bs = Bs + (size_t)(kt % STAGES) * UT_N * LDBU + 2 * t;
#pragma unroll
    for (int ks = 0; ks < RBK / 16; ++ks) {
    double af[2][8];
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        const double2 v = lds128(as + (16 * ks + 4 * s) * LDRU + 16 * a);
        af[a][2 * s] = v.x;
        af[a][2 * s + 1] = v.y;
      }
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      const double* p = bs + (wj + 8 * b + g) * LDBU;
      double br[4], bi[4];
#pragma unroll
      for (int s = 0; s < 4; ++s) {
        const double2 v = lds128(p + 32 * ks + 8 * s);
        br[s] = v.x;
        bi[s] = v.y;
      }
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        if (a < na && b < nb) {
          dmma16(ar[a][b], af[a], br);
          dmma16(ai[a][b], af[a], bi);
        }
      }
    }
    }
  }
  cp_async_wait<0>();
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int64_t row = r0 + wr + 16 * a + 2 * g + (e >> 1);
        const int64_t gj = j0 + wj + 8 * b + 2 * t + (e & 1);
        if (row < Krows && gj < n) C[row + ldc * gj] = make_double2(ar[a][b][e], ai[a][b][e]);
      }
}

static size_t smem_cn(int st) { return (size_t)st * (GT_M + GT_N) * LDK * sizeof(double); }
static size_t smem_nn(int st) { return (size_t)st * (BKC * LDA_U + UT_N * LDK) * sizeof(double); }
// a 32-deep stage of the real-A kernels takes 68 / 73 KB: they run at most three stages (gemm_stages 4 runs 3)
static size_t smem_rcn(int st) { return (size_t)st * (GT_M * LDR + GT_N * RLDK) * sizeof(double); }
static size_t smem_rnn(int st) { return (size_t)st * (RBK * LDRU + UT_N * LDBU) * sizeof(double); }

// ---------------------------------------------------------------- elementwise / reduction kernels
__global__ void k_columnwise_dots(const cplx* __restrict__ A, int64_t lda, const cplx* __restrict__ B,
                                  int64_t ldb, int64_t n_rows, cplx* __restrict__ out) {
  // one CTA per column, deterministic tree reduction
  const int64_t col = blockIdx.x;
  const cplx* a = A + lda * col;
  const cplx* b = B + ldb * col;
  double sx = 0.0, sy = 0.0;
  for (int64_t i = threadIdx.x; i < n_rows; i += blockDim.x) {
    cplx x = a[i], y = b[i];
    sx += x.x * y.x + x.y * y.y;   // conj(a) * b
    sy += x.x * y.y - x.y * y.x;
  }
  __shared__ double rx[32], ry[32];
  for (int o = 16; o > 0; o >>= 1) {
    sx += __shfl_down_sync(0xffffffffu, sx, o);
    sy += __shfl_down_sync(0xffffffffu, sy, o);
  }
  if ((threadIdx.x & 31) == 0) {
    rx[threadIdx.x >> 5] = sx;
    ry[threadIdx.x >> 5] = sy;
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    int nw = blockDim.x >> 5;
    sx = threadIdx.x < nw ? rx[threadIdx.x] : 0.0;
    sy = threadIdx.x < nw ? ry[threadIdx.x] : 0.0;
    for (int o = 16; o > 0; o >>= 1) {
      sx += __shfl_down_sync(0xffffffffu, sx, o);
      sy += __shfl_down_sync(0xffffffffu, sy, o);
    }
    if (threadIdx.x == 0) out[col] = make_double2(sx, sy);
  }
}

__global__ void k_kin_dots(const cplx* __restrict__ X, int64_t ldx, const double* __restrict__ kin,
                           int64_t n_rows, double* __restrict__ out) {
  const int64_t col = blockIdx.x;
  const cplx* x = X + ldx * col;
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n_rows; i += blockDim.x) {
    cplx v = x[i];
    s += kin[i] * (v.x * v.x + v.y * v.y);
  }
  __shared__ double r[32];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) r[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    int nw = blockDim.x >> 5;
    s = threadIdx.x < nw ? r[threadIdx.x] : 0.0;
    for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) out[col] = s;
  }
}

__global__ void k_scale_kin_add(const cplx* __restrict__ psi, cplx* __restrict__ hpsi,
                                const double* __restrict__ kin, int64_t n_rows, int64_t total,
                                int accumulate) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  cplx v = make_double2(0.0, 0.0);
  if (kin) {
    double k = kin[idx % n_rows];
    cplx p = psi[idx];
    v = make_double2(k * p.x, k * p.y);
  }
  if (accumulate) v = cadd(v, hpsi[idx]);
  hpsi[idx] = v;
}

void blas_set_attributes() {
  CUDA_CHECK(cudaFuncSetAttribute(k_zgemm_cn<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cn(2)));
  CUDA_CHECK(cudaFuncSetAttribute(k_zgemm_nn<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_nn(2)));
  CUDA_CHECK(cudaFuncSetAttribute(k_zgemm_cn<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cn(3)));
  CUDA_CHECK(cudaFuncSetAttribute(k_zgemm_nn<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_nn(3)));
  CUDA_CHECK(cudaFuncSetAttribute(k_zgemm_cn<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cn(4)));
  CUDA_CHECK(cudaFuncSetAttribute(k_zgemm_nn<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_nn(4)));
  CUDA_CHECK(cudaFuncSetAttribute(k_rgemm_cn<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_rcn(2)));
  CUDA_CHECK(cudaFuncSetAttribute(k_rgemm_nn<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_rnn(2)));
  CUDA_CHECK(cudaFuncSetAttribute(k_rgemm_cn<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_rcn(3)));
  CUDA_CHECK(cudaFuncSetAttribute(k_rgemm_nn<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_rnn(3)));
}

void columnwise_dots(dftk_b200_ctx* ctx, const cplx* A, int64_t lda, const cplx* B, int64_t ldb,
                     int64_t n_rows, int64_t n_cols, cplx* out_dev) {
  if (n_cols == 0) return;
  LAUNCH(ctx, k_columnwise_dots, (unsigned)n_cols, 256, 0, A, lda, B, ldb, n_rows, out_dev);
}
void kin_dots(dftk_b200_ctx* ctx, const cplx* X, int64_t ldx, const double* kin, int64_t n_rows,
              int64_t n_cols, double* out_dev) {
  if (n_cols == 0) return;
  LAUNCH(ctx, k_kin_dots, (unsigned)n_cols, 256, 0, X, ldx, kin, n_rows, out_dev);
}
void scale_kin_add(dftk_b200_ctx* ctx, const cplx* psi, cplx* hpsi, const double* kin, int64_t n_rows,
                   int64_t n_cols, int accumulate) {
  int64_t total = n_rows * n_cols;
  if (total == 0) return;
  if (!kin && accumulate) return;
  LAUNCH(ctx, k_scale_kin_add, (unsigned)((total + 255) / 256), 256, 0, psi, hpsi, kin, n_rows, total,
         accumulate);
}

// Split-K of a Gram product over `tiles` output tiles that do work: one CTA per SM is resident, so the CTA count should
// fill whole waves of sm_count, keeping >= 8 stages per split; the mild per-split penalty stands for the pipeline fill
// and the reduce pass.  Returns the number of splits and their length (a multiple of BKC) in *kps.
static int64_t gram_splits(const dftk_b200_ctx* ctx, int64_t tiles, int64_t k, int64_t* kps) {
  const int64_t slots = ctx->sm_count;
  const int64_t max_split = std::min<int64_t>(64, (k + 8 * BKC - 1) / (8 * BKC));
  int64_t nsplit = 1;
  double best = -1.0;
  for (int64_t sp = 1; sp <= max_split; ++sp) {
    const int64_t total = tiles * sp;
    const double eff = (double)total / (double)(((total + slots - 1) / slots) * slots) - 0.002 * sp;
    if (eff > best) {
      best = eff;
      nsplit = sp;
    }
  }
  int64_t len = (k + nsplit - 1) / nsplit;
  len = ((len + BKC - 1) / BKC) * BKC;
  *kps = len;
  return (k + len - 1) / len;
}

// C = alpha op(A) B + beta C.  transA: 0 = N (A: m x k... see header), 2 = C.
//   transA == 2: A is (k x m), B is (k x n), C is (m x n)        [Gram type, k large]
//   transA == 0: A is (m x k), B is (k x n), C is (m x n)        [update type, m large]
void zgemm(dftk_b200_ctx* ctx, int transA, int64_t m, int64_t n, int64_t k, cplx alpha, const cplx* A,
           int64_t lda, const cplx* B, int64_t ldb, cplx beta, cplx* C, int64_t ldc, bool upper_only) {
  if (m == 0 || n == 0) return;
  REQUIRE(transA == 0 || transA == 2, "zgemm: transA must be 0 (N) or 2 (C)");
  if (ctx->gemm_backend == 1) {
    cuDoubleComplex a = make_cuDoubleComplex(alpha.x, alpha.y), b = make_cuDoubleComplex(beta.x, beta.y);
    CUBLAS_CHECK(cublasZgemm(ctx->cublas, transA == 2 ? CUBLAS_OP_C : CUBLAS_OP_N, CUBLAS_OP_N, (int)m,
                             (int)n, (int)k, &a, (const cuDoubleComplex*)A, (int)lda,
                             (const cuDoubleComplex*)B, (int)ldb, &b, (cuDoubleComplex*)C, (int)ldc));
    ctx->launches++;
    return;
  }
  if ((ctx->gemm_backend == 2 || (ctx->gemm_backend == 4 && k >= ctx->i8_min_rows && m >= 32 && n >= 32)) && transA == 2 && k > 0 && alpha.x == 1.0 && alpha.y == 0.0 && beta.x == 0.0 && beta.y == 0.0) {
    // FP64 by INT8 residues + CRT (i8emu.cu): integer products on the tensor cores (4) or the CUDA-core reference pipeline (2)
    zgemm_i8_cn(ctx, m, n, k, A, lda, B, ldb, C, ldc, ctx->gemm_backend == 4);
    return;
  }
  if (ctx->gemm_backend == 4 && transA == 0 && m >= ctx->i8_min_rows && k >= 32 && n >= 16 && alpha.y == 0.0 && beta.y == 0.0 && !upper_only) {
    // update-type product on the INT8 tensor cores: A prepared here (callers with reusable operands use i8_update directly)
    const I8Operand opA = i8_prepare(ctx, A, lda, k, m, ctx->i8_tmp_planes, ctx->i8_tmp_exps);
    i8_update(ctx, 1, &opA, B, ldb, n, C, ldc, alpha.x, beta.x);
    return;
  }
  if (ctx->gemm_backend == 2 && transA == 0 && k > 0 && alpha.x == 1.0 && alpha.y == 0.0 && beta.y == 0.0 &&
      (beta.x == 0.0 || beta.x == 1.0) && !upper_only) {
    if (zgemm_i8_nn(ctx, m, n, k, A, lda, B, ldb, C, ldc, beta.x == 1.0)) return;     // too large: DMMA kernel below
  }
  if (k == 0) {
    // C = beta C
    LAUNCH(ctx, k_reduce_partials, (unsigned)((m * n + 255) / 256), 256, 0, (const cplx*)nullptr, 0, m, n,
           alpha, beta, C, ldc);
    return;
  }
  const int st = ctx->gemm_stages;
  if (transA == 2) {
    // tiles that do work (Hermitian Grams skip the tiles strictly below the diagonal)
    const int64_t mt = (m + GT_M - 1) / GT_M, nt = (n + GT_N - 1) / GT_N;
    const bool upper = upper_only && m == n;
    int64_t tiles = 0;
    for (int64_t bj = 0; bj < nt; ++bj) tiles += upper ? std::min(mt, ((bj + 1) * GT_N + GT_M - 1) / GT_M) : mt;
    int64_t kps = 0;
    const int64_t nsplit = gram_splits(ctx, tiles, k, &kps);
    cplx* ws = (cplx*)ctx->gemm_ws.ensure((size_t)nsplit * m * n * sizeof(cplx));
    dim3 grid((unsigned)mt, (unsigned)nt, (unsigned)nsplit);
    const int uo = upper ? 1 : 0;
    if (st == 2) LAUNCH(ctx, k_zgemm_cn<2>, grid, GEMM_THREADS, smem_cn(2), A, lda, B, ldb, ws, m, n, k, kps, uo);
    else if (st == 3) LAUNCH(ctx, k_zgemm_cn<3>, grid, GEMM_THREADS, smem_cn(3), A, lda, B, ldb, ws, m, n, k, kps, uo);
    else LAUNCH(ctx, k_zgemm_cn<4>, grid, GEMM_THREADS, smem_cn(4), A, lda, B, ldb, ws, m, n, k, kps, uo);
    LAUNCH(ctx, k_reduce_partials, (unsigned)((m * n + 255) / 256), 256, 0, (const cplx*)ws, (int)nsplit, m,
           n, alpha, beta, C, ldc);
  } else {
    REQUIRE((m + UT_M - 1) / UT_M <= 65535, "zgemm: more than 4.19M rows are not supported by the update kernel grid");
    dim3 grid((unsigned)((n + UT_N - 1) / UT_N), (unsigned)((m + UT_M - 1) / UT_M));
    const int bu = (upper_only && k == n) ? 1 : 0;
    if (st == 2) LAUNCH(ctx, k_zgemm_nn<2>, grid, GEMM_THREADS, smem_nn(2), A, lda, B, ldb, C, ldc, m, n, k, alpha, beta, bu);
    else if (st == 3) LAUNCH(ctx, k_zgemm_nn<3>, grid, GEMM_THREADS, smem_nn(3), A, lda, B, ldb, C, ldc, m, n, k, alpha, beta, bu);
    else LAUNCH(ctx, k_zgemm_nn<4>, grid, GEMM_THREADS, smem_nn(4), A, lda, B, ldb, C, ldc, m, n, k, alpha, beta, bu);
  }
}

// ---------------------------------------------------------------- time-reversal fold of the projector products
// On a k-block whose sphere is closed under q -> -q (q = k + G; Γ and the other k with 2k in the reciprocal lattice),
// the projectors satisfy P(-q) = conj(P(q)).  With a half set H holding one member q of each pair and P = Pr + i Pi:
//   P'psi = sum_{q in H} Pr(q) s(q) + Pi(q) u(q),   s = psi(q) + psi(-q),   u = i (psi(-q) - psi(q))
//   P c   : Hpsi(q) += a + i b,  Hpsi(-q) += a - i b,   [a; b] = R c,  R = [Pr(H); Pi(H)]  (real, K' = 2|H| rows)
// (at q = -q: s = psi(q), u = 0 and Hpsi(q) += a).  Both products become real-A products of half the DMMA work.

// Sphere point paired with each sphere point by G -> -G - m, m = 2k read off the sphere's bounding box (the sphere of
// k + G is symmetric about -k).  False when that reflection does not map the sphere onto itself.
bool sphere_mirror(int nx, int ny, int nz, int64_t n_pw, const int64_t* map, std::vector<int>& mir) {
  const int64_t N = (int64_t)nx * ny * nz;
  const int n[3] = {nx, ny, nz};
  std::vector<int> G((size_t)3 * n_pw);
  int lo[3] = {1 << 30, 1 << 30, 1 << 30}, hi[3] = {-(1 << 30), -(1 << 30), -(1 << 30)};
  for (int64_t i = 0; i < n_pw; ++i) {
    int64_t lin = map[i];
    for (int d = 0; d < 3; ++d) {
      const int c = (int)(lin % n[d]);
      lin /= n[d];
      const int g = c <= (n[d] - 1) / 2 ? c : c - n[d];   // G_axis: [0 .. (n-1)/2, -n/2 .. -1]
      G[3 * i + d] = g;
      lo[d] = std::min(lo[d], g);
      hi[d] = std::max(hi[d], g);
    }
  }
  std::vector<int> slot(N, -1);
  for (int64_t i = 0; i < n_pw; ++i) slot[map[i]] = (int)i;
  mir.assign(n_pw, -1);
  for (int64_t i = 0; i < n_pw; ++i) {
    int64_t lin = 0;
    for (int d = 2; d >= 0; --d) {
      const int g = -G[3 * i + d] + lo[d] + hi[d];   // -G - m with m = -(lo + hi)
      lin = lin * n[d] + ((g % n[d]) + n[d]) % n[d];
    }
    mir[i] = slot[lin];
    if (mir[i] < 0) return false;
  }
  for (int64_t i = 0; i < n_pw; ++i)
    if (mir[mir[i]] != i) return false;
  return true;
}

__global__ void k_fold_check(const cplx* __restrict__ P, int64_t ldp, const int* __restrict__ hi,
                             const int* __restrict__ hp, int64_t nh, int64_t np, unsigned long long* __restrict__ out) {
  // out[0] = max |P(-q) - conj(P(q))|, out[1] = max |P| (non-negative doubles order like their bit patterns)
  double dmax = 0.0, pmax = 0.0;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < nh * np; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t h = idx % nh, j = idx / nh;
    const cplx a = P[hi[h] + ldp * j], b = P[hp[h] + ldp * j];
    dmax = fmax(dmax, hypot(b.x - a.x, b.y + a.y));
    pmax = fmax(pmax, fmax(hypot(a.x, a.y), hypot(b.x, b.y)));
  }
  for (int o = 16; o > 0; o >>= 1) {
    dmax = fmax(dmax, __shfl_down_sync(0xffffffffu, dmax, o));
    pmax = fmax(pmax, __shfl_down_sync(0xffffffffu, pmax, o));
  }
  if ((threadIdx.x & 31) == 0) {
    atomicMax(out, (unsigned long long)__double_as_longlong(dmax));
    atomicMax(out + 1, (unsigned long long)__double_as_longlong(pmax));
  }
}

// R (K' x np, column-major) = [Pr(H); Pi(H)]
__global__ void k_fold_projectors(const cplx* __restrict__ P, int64_t ldp, const int* __restrict__ hi, int64_t nh,
                                  int64_t np, double* __restrict__ R) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nh * np) return;
  const int64_t h = idx % nh, j = idx / nh;
  const cplx a = P[hi[h] + ldp * j];
  R[h + 2 * nh * j] = a.x;
  R[nh + h + 2 * nh * j] = a.y;
}

// F[:, j] = [s; u] of band j
__global__ void k_fold(const cplx* __restrict__ psi, int64_t ldpsi, const int* __restrict__ hi,
                       const int* __restrict__ hp, int64_t nh, int64_t nb, cplx* __restrict__ F, int64_t ldf) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nh * nb) return;
  const int64_t h = idx % nh, j = idx / nh;
  const int i = hi[h], p = hp[h];
  const cplx a = psi[i + ldpsi * j];
  cplx s = a, u = make_double2(0.0, 0.0);
  if (p != i) {
    const cplx b = psi[p + ldpsi * j];
    s = cadd(a, b);
    u = make_double2(a.y - b.y, b.x - a.x);   // i (b - a)
  }
  F[h + ldf * j] = s;
  F[nh + h + ldf * j] = u;
}

// hpsi(q) += a + i b, hpsi(-q) += a - i b from Y[:, j] = [a; b]
__global__ void k_unfold_acc(const cplx* __restrict__ Y, int64_t ldy, const int* __restrict__ hi,
                             const int* __restrict__ hp, int64_t nh, int64_t nb, cplx* __restrict__ hpsi, int64_t ldh) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nh * nb) return;
  const int64_t h = idx % nh, j = idx / nh;
  const int i = hi[h], p = hp[h];
  const cplx a = Y[h + ldy * j];
  cplx* o = hpsi + ldh * j;
  if (p == i) {
    o[i] = cadd(o[i], a);
    return;
  }
  const cplx b = Y[nh + h + ldy * j];
  o[i] = cadd(o[i], make_double2(a.x - b.y, a.y + b.x));
  o[p] = cadd(o[p], make_double2(a.x + b.y, a.y - b.x));
}

// Pairs the sphere and checks the projector table (atomic projectors and orbital columns) of a k-block; on success keeps
// H, the partners and R so that kb_apply_nonlocal and the band energies take the folded path.  Any other block keeps the
// complex products.  Called again whenever the table changes (kblock_set_orbitals).
void kb_setup_fold(dftk_b200_kblock* kb, const int64_t* map_h) {
  kb->n_half = 0;
  kb->fold_i.release();
  kb->fold_p.release();
  kb->R.release();
  if (kb->n_nl() == 0) return;
  dftk_b200_ctx* ctx = kb->grid->ctx;
  const dftk_b200_grid* g = kb->grid;
  std::vector<int> mir;
  if (!sphere_mirror(g->nx, g->ny, g->nz, kb->n_pw, map_h, mir)) return;
  std::vector<int> hi, hp;
  for (int64_t i = 0; i < kb->n_pw; ++i)
    if (i <= mir[i]) {
      hi.push_back((int)i);
      hp.push_back(mir[i]);
    }
  const int64_t nh = (int64_t)hi.size(), np = kb->n_nl();
  cudaStream_t s = ctx->stream;
  kb->fold_i.upload(hi.data(), nh, s);
  kb->fold_p.upload(hp.data(), nh, s);
  unsigned long long* d = (unsigned long long*)ctx->scal.ensure(8);
  CUDA_CHECK(cudaMemsetAsync(d, 0, 2 * sizeof(unsigned long long), s));
  LAUNCH(ctx, k_fold_check, (unsigned)(4 * ctx->sm_count), 256, 0, (const cplx*)kb->P.p, kb->n_pw,
         (const int*)kb->fold_i.p, (const int*)kb->fold_p.p, nh, np, d);
  unsigned long long r[2];
  CUDA_CHECK(cudaMemcpyAsync(r, d, sizeof(r), cudaMemcpyDeviceToHost, s));
  CUDA_CHECK(cudaStreamSynchronize(s));
  double dev, pmax;
  std::memcpy(&dev, &r[0], sizeof(double));
  std::memcpy(&pmax, &r[1], sizeof(double));
  if (!(dev <= 1e-12 * pmax)) {
    kb->fold_i.release();
    kb->fold_p.release();
    return;
  }
  kb->R.ensure((size_t)2 * nh * np);
  LAUNCH(ctx, k_fold_projectors, (unsigned)((nh * np + 255) / 256), 256, 0, (const cplx*)kb->P.p, kb->n_pw,
         (const int*)kb->fold_i.p, nh, np, kb->R.p);
  kb->n_half = nh;
}

// widest band chunk of the folded products: bounds the folded-orbital scratch (K' x chunk) for wide LOBPCG blocks
#define FOLD_MAX_COLS 384
static int64_t fold_chunk(int64_t n_bands) {
  const int64_t c = (n_bands + FOLD_MAX_COLS - 1) / FOLD_MAX_COLS;
  return (n_bands + c - 1) / c;
}

// C (m x n, ldc) = A^T B with A real (K x m), B complex (K x n); K, lda even
static void rgemm_cn(dftk_b200_ctx* ctx, int64_t m, int64_t n, int64_t K, const double* A, int64_t lda, const cplx* B,
                     int64_t ldb, cplx* C, int64_t ldc) {
  const int64_t mt = (m + GT_M - 1) / GT_M, nt = (n + GT_N - 1) / GT_N;
  int64_t kps = 0;
  const int64_t nsplit = gram_splits(ctx, mt * nt, K, &kps);
  cplx* ws = (cplx*)ctx->gemm_ws.ensure((size_t)nsplit * m * n * sizeof(cplx));
  dim3 grid((unsigned)mt, (unsigned)nt, (unsigned)nsplit);
  if (ctx->gemm_stages == 2) LAUNCH(ctx, k_rgemm_cn<2>, grid, GEMM_THREADS, smem_rcn(2), A, lda, B, ldb, ws, m, n, K, kps);
  else LAUNCH(ctx, k_rgemm_cn<3>, grid, GEMM_THREADS, smem_rcn(3), A, lda, B, ldb, ws, m, n, K, kps);
  LAUNCH(ctx, k_reduce_partials, (unsigned)((m * n + 255) / 256), 256, 0, (const cplx*)ws, (int)nsplit, m, n,
         make_double2(1.0, 0.0), make_double2(0.0, 0.0), C, ldc);
}

// C (Krows x n, ldc) = A B with A real (Krows x m), B complex (m x n); Krows, lda even
static void rgemm_nn(dftk_b200_ctx* ctx, int64_t Krows, int64_t n, int64_t m, const double* A, int64_t lda,
                     const cplx* B, int64_t ldb, cplx* C, int64_t ldc) {
  REQUIRE((Krows + UT_M - 1) / UT_M <= 65535, "rgemm_nn: more than 4.19M rows are not supported by the update kernel grid");
  dim3 grid((unsigned)((n + UT_N - 1) / UT_N), (unsigned)((Krows + UT_M - 1) / UT_M));
  if (ctx->gemm_stages == 2) LAUNCH(ctx, k_rgemm_nn<2>, grid, GEMM_THREADS, smem_rnn(2), A, lda, B, ldb, C, ldc, Krows, n, m);
  else LAUNCH(ctx, k_rgemm_nn<3>, grid, GEMM_THREADS, smem_rnn(3), A, lda, B, ldb, C, ldc, Krows, n, m);
}

static bool kb_folds(const dftk_b200_kblock* kb) { return kb->n_half > 0 && kb->grid->ctx->gemm_backend == 0; }

// proj (nc x n_bands) = P[:, c0 : c0+nc]' psi
void kb_project_cols(dftk_b200_kblock* kb, int64_t c0, int64_t nc, const cplx* psi, int64_t n_bands, cplx* proj) {
  dftk_b200_ctx* ctx = kb->grid->ctx;
  const int64_t nh = kb->n_half, kf = 2 * nh;
  if (!kb_folds(kb)) {
    zgemm(ctx, 2, nc, n_bands, kb->n_pw, make_double2(1, 0), kb->P.p + kb->n_pw * c0, kb->n_pw, psi, kb->n_pw,
          make_double2(0, 0), proj, nc);
    return;
  }
  const int64_t w0 = fold_chunk(n_bands);
  cplx* F = kb->fold_ws.ensure((size_t)kf * w0);
  for (int64_t j0 = 0; j0 < n_bands; j0 += w0) {
    const int64_t w = std::min(w0, n_bands - j0);
    LAUNCH(ctx, k_fold, (unsigned)((nh * w + 255) / 256), 256, 0, psi + kb->n_pw * j0, kb->n_pw,
           (const int*)kb->fold_i.p, (const int*)kb->fold_p.p, nh, w, F, kf);
    rgemm_cn(ctx, nc, w, kf, kb->R.p + kf * c0, kf, F, kf, proj + nc * j0, nc);
  }
}

// proj (n_proj x n_bands) = P' psi over the atomic projectors
void kb_project(dftk_b200_kblock* kb, const cplx* psi, int64_t n_bands, cplx* proj) {
  kb_project_cols(kb, 0, kb->n_proj, psi, n_bands, proj);
}

// PD[:, c0:] = P Dnl[:, c0:]; Dnl is block diagonal, so columns from a block boundary on only need those rows of Dnl
void kb_refresh_pd(dftk_b200_kblock* kb, int64_t c0) {
  const int64_t n = kb->n_nl();
  if (!kb->PD.p || c0 >= n) return;
  zgemm(kb->grid->ctx, 0, kb->n_pw, n - c0, n - c0, make_double2(1, 0), kb->P.p + kb->n_pw * c0, kb->n_pw,
        kb->Dnl() + c0 + n * c0, n, make_double2(0, 0), kb->PD.p + kb->n_pw * c0, kb->n_pw);
}

// the nonlocal apply on the folded operands, one band chunk at a time; the update writes [a; b] over the folded orbitals
static void kb_apply_nonlocal_folded(dftk_b200_kblock* kb, const cplx* psi, cplx* hpsi, int64_t n_bands) {
  dftk_b200_ctx* ctx = kb->grid->ctx;
  const int64_t np = kb->n_nl(), nh = kb->n_half, kf = 2 * nh;
  const int64_t nc = fold_chunk(n_bands);
  cplx* F = kb->fold_ws.ensure((size_t)kf * nc);
  cplx* proj = kb->proj.ensure((size_t)2 * np * nc);
  cplx* dproj = proj + (size_t)np * nc;
  for (int64_t j0 = 0; j0 < n_bands; j0 += nc) {
    const int64_t w = std::min(nc, n_bands - j0);
    const unsigned blocks = (unsigned)((nh * w + 255) / 256);
    LAUNCH(ctx, k_fold, blocks, 256, 0, psi + kb->n_pw * j0, kb->n_pw, (const int*)kb->fold_i.p,
           (const int*)kb->fold_p.p, nh, w, F, kf);
    rgemm_cn(ctx, np, w, kf, kb->R.p, kf, F, kf, proj, np);
    zgemm(ctx, 0, np, w, np, make_double2(1, 0), kb->Dnl(), np, proj, np, make_double2(0, 0), dproj, np);
    rgemm_nn(ctx, kf, w, np, kb->R.p, kf, dproj, np, F, kf);
    LAUNCH(ctx, k_unfold_acc, blocks, 256, 0, (const cplx*)F, kf, (const int*)kb->fold_i.p, (const int*)kb->fold_p.p,
           nh, w, hpsi + kb->n_pw * j0, kb->n_pw);
  }
}

// hpsi += P (D (P' psi))      (apply!(::NonlocalOperator), src/terms/operators.jl:126-128); with Hubbard orbitals
// attached P = [P | Φ] and D = [D 0; 0 V], so the orbital term rides in the same pair of products
void kb_apply_nonlocal(dftk_b200_kblock* kb, const cplx* psi, cplx* hpsi, int64_t n_bands) {
  if (kb->n_nl() == 0 || n_bands == 0) return;
  if (kb_folds(kb)) {
    kb_apply_nonlocal_folded(kb, psi, hpsi, n_bands);
    return;
  }
  dftk_b200_ctx* ctx = kb->grid->ctx;
  const int64_t np = kb->n_nl();
  cplx* proj = kb->proj.ensure((size_t)2 * np * n_bands);
  cplx* dproj = proj + (size_t)np * n_bands;
  const cplx one = make_double2(1.0, 0.0), zero = make_double2(0.0, 0.0);
  if (ctx->gemm_backend == 4 && np >= 64 && n_bands >= 32 && kb->n_pw >= ctx->i8_min_rows) {
    // both projector products on the INT8 tensor cores (wgmma s8, TMA-fed; i8emu.cu / i8tc2.cu): the residue
    // planes of P are prepared once per k-block and serve P'psi (K-major operand) and P (D P'psi) (MN-major operand)
    if (!kb->i8_Pop.planes) kb->i8_Pop = i8_prepare(ctx, kb->P.p, kb->n_pw, np, kb->n_pw, kb->i8_planes, kb->i8_exps);
    const I8Operand op_psi = i8_prepare(ctx, psi, kb->n_pw, n_bands, kb->n_pw, kb->i8_psi_planes, kb->i8_psi_exps);
    i8_gram(ctx, kb->i8_Pop, op_psi, proj, np, false);
    zgemm(ctx, 0, np, n_bands, np, one, kb->Dnl(), np, proj, np, zero, dproj, np);
    i8_update(ctx, 1, &kb->i8_Pop, dproj, np, n_bands, hpsi, kb->n_pw, 1.0, 1.0);
    return;
  }
  zgemm(ctx, 2, np, n_bands, kb->n_pw, one, kb->P.p, kb->n_pw, psi, kb->n_pw, zero, proj, np);
  zgemm(ctx, 0, np, n_bands, np, one, kb->Dnl(), np, proj, np, zero, dproj, np);
  zgemm(ctx, 0, kb->n_pw, n_bands, np, one, kb->P.p, kb->n_pw, dproj, np, one, hpsi, kb->n_pw);
}

}  // namespace dftk
