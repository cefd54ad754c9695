// Dense complex128 kernels of the hot path:
//   * zgemm_cn : C(m x n) = alpha * A^H B + beta * C, A: K x m, B: K x n, K = N_pw huge  ("Gram" type:
//                P'psi, X'AX blocks, BY'X)                      -- src/terms/operators.jl:127,
//                src/eigen/lobpcg_hyper_impl.jl:90-113,216-221,277
//   * zgemm_nn : C(K x n) = alpha * A(K x m) B(m x n) + beta * C              ("update" type:
//                Hpsi += P (D P'psi), new_X = Y cX, X -= Y (BY'X), X = X invR) -- lobpcg_hyper_impl.jl:124-137
// Both are real FP64 tensor-core GEMMs (mma.sync.m8n8k4.f64 = DMMA) on the interleaved complex
// storage: with A~ the real (2K x m) view of A (rows re,im,re,im,...),
//   Re(A^H B) = A~^T B~,   Im(A^H B) = A~^T (J B~),   (J b)[2k] = b[2k+1], (J b)[2k+1] = -b[2k]
// and for the update C~ = A^ B~ with A^[:,2i] = A~[:,i], A^[:,2i+1] = J' A~[:,i].
// The J-images are formed while loading MMA fragments from shared memory (index ^1 and a sign), so no
// operand is ever materialised twice.  Tiles are staged with cp.async in a 3-stage ring.
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
__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

#define GEMM_THREADS 128
#define BKC 16              // complex k per stage (32 real)
#define LDK (2 * BKC + 4)   // doubles per k-major smem row; LDK % 16 == 4 => conflict-free fragments

// ------------------------------------------------------------------------------------------------
// Gram kernel.  CTA tile: 64 (i) x 32 (j) complex outputs; warp w owns i in [16w... no: rows 32*(w&1)..,
// cols 16*(w>>1)..  => 4 warps = 2 x 2.  Partial sums over the K-slice [k_begin, k_end) are written to
// ws[split][m x n]; reduce_partials applies alpha/beta.
// ------------------------------------------------------------------------------------------------
#define GT_M 64
#define GT_N 32
template <int GEMM_STAGES>
__global__ void __launch_bounds__(GEMM_THREADS)
k_zgemm_cn(const cplx* __restrict__ A, int64_t lda, const cplx* __restrict__ B, int64_t ldb,
           cplx* __restrict__ ws, int64_t m, int64_t n, int64_t K, int64_t k_per_split, int upper_only) {
  // Hermitian results (X'X, X'AX): tiles strictly below the diagonal are never read by the callers
  if (upper_only && (int64_t)blockIdx.x * GT_M >= (int64_t)blockIdx.y * GT_N + GT_N) return;
  extern __shared__ __align__(16) double smem_d[];
  double* As = smem_d;                                   // [STAGES][GT_M][LDK]
  double* Bs = smem_d + GEMM_STAGES * GT_M * LDK;        // [STAGES][GT_N][LDK]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t i0 = (int64_t)blockIdx.x * GT_M, j0 = (int64_t)blockIdx.y * GT_N;
  const int64_t kb = (int64_t)blockIdx.z * k_per_split;
  const int64_t ke = min(K, kb + k_per_split);
  const int nkt = (int)((ke - kb + BKC - 1) / BKC);
  const int wi = (warp & 1) * 32, wj = (warp >> 1) * 16;

  // Per-thread copy plan (fixed across k tiles): element e = tid + 128 i -> column tid/16 + 8 i, row tid%16.
  const int lkk = tid & (BKC - 1), lcol = tid >> 4;
  const cplx* pA = A + kb + lkk + lda * (i0 + lcol);
  const cplx* pB = B + kb + lkk + ldb * (j0 + lcol);
  unsigned okA = 0, okB = 0;   // column-in-range masks
#pragma unroll
  for (int i = 0; i < GT_M / 8; ++i) okA |= (i0 + lcol + 8 * i < m) ? (1u << i) : 0u;
#pragma unroll
  for (int i = 0; i < GT_N / 8; ++i) okB |= (j0 + lcol + 8 * i < n) ? (1u << i) : 0u;
  auto load_tile = [&](int kt, int slot) {
    const int64_t koff = (int64_t)kt * BKC;
    const bool rowok = kb + koff + lkk < ke;
    double* da = As + ((size_t)slot * GT_M + lcol) * LDK + 2 * lkk;
    double* db = Bs + ((size_t)slot * GT_N + lcol) * LDK + 2 * lkk;
#pragma unroll
    for (int i = 0; i < GT_M / 8; ++i) {
      bool ok = rowok && ((okA >> i) & 1u);
      cp_async16(da + (size_t)8 * i * LDK, ok ? (pA + koff + (int64_t)8 * i * lda) : A, ok);
    }
#pragma unroll
    for (int i = 0; i < GT_N / 8; ++i) {
      bool ok = rowok && ((okB >> i) & 1u);
      cp_async16(db + (size_t)8 * i * LDK, ok ? (pB + koff + (int64_t)8 * i * ldb) : B, ok);
    }
  };

  double cr[4][2][2], ci[4][2][2];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 2; ++b) cr[a][b][0] = cr[a][b][1] = ci[a][b][0] = ci[a][b][1] = 0.0;

  for (int s = 0; s < GEMM_STAGES - 1; ++s) {
    if (s < nkt) load_tile(s, s);
    cp_async_commit();
  }
  const int fr = lane >> 2, fk = lane & 3;
  const int sgnmask = (lane & 1) ? (int)0x80000000 : 0;   // J-image sign, applied with an integer XOR (ALU pipe)
  for (int kt = 0; kt < nkt; ++kt) {
    cp_async_wait<GEMM_STAGES - 2>();
    __syncthreads();
    {
      int nxt = kt + GEMM_STAGES - 1;
      if (nxt < nkt) load_tile(nxt, nxt % GEMM_STAGES);
      cp_async_commit();
    }
    const double* as = As + (size_t)(kt % GEMM_STAGES) * GT_M * LDK;
    const double* bs = Bs + (size_t)(kt % GEMM_STAGES) * GT_N * LDK;
#pragma unroll
    for (int s4 = 0; s4 < 2 * BKC / 4; ++s4) {
      double af[4], bf[2], bh[2];
#pragma unroll
      for (int a = 0; a < 4; ++a) af[a] = as[(wi + 8 * a + fr) * LDK + 4 * s4 + fk];
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const double* row = bs + (wj + 8 * b + fr) * LDK + 4 * s4;
        bf[b] = row[fk];
        double t = row[fk ^ 1];
        bh[b] = __hiloint2double(__double2hiint(t) ^ sgnmask, __double2loint(t));
      }
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          dmma(cr[a][b][0], cr[a][b][1], af[a], bf[b]);
          dmma(ci[a][b][0], ci[a][b][1], af[a], bh[b]);
        }
    }
  }
  cp_async_wait<0>();
  cplx* out = ws + (size_t)blockIdx.z * m * n;
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 2; ++b)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        int64_t gi = i0 + wi + 8 * a + fr;
        int64_t gj = j0 + wj + 8 * b + 2 * fk + e;
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
// Update kernel.  CTA tile: 64 complex rows (128 real) x 32 columns; warp w owns real rows 32w..32w+31.
// ------------------------------------------------------------------------------------------------
#define UT_M 64                 // complex rows
#define UT_N 32
#define LDA_U (2 * UT_M + 4)    // doubles per inner-index row of the A tile (132 % 16 == 4)
template <int GEMM_STAGES>
__global__ void __launch_bounds__(GEMM_THREADS)
k_zgemm_nn(const cplx* __restrict__ A, int64_t lda, const cplx* __restrict__ B, int64_t ldb,
           cplx* __restrict__ C, int64_t ldc, int64_t Krows, int64_t n, int64_t m, cplx alpha, cplx beta,
           int b_upper) {
  extern __shared__ __align__(16) double smem_d[];
  double* As = smem_d;                                   // [STAGES][BKC][LDA_U]
  double* Bs = smem_d + GEMM_STAGES * BKC * LDA_U;       // [STAGES][UT_N][LDK]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // blockIdx.x = column tile (fastest): CTAs sharing one A row panel run together and hit it in L2
  const int64_t r0 = (int64_t)blockIdx.y * UT_M, j0 = (int64_t)blockIdx.x * UT_N;
  // B upper triangular (X * inv(R), rmul! with an UpperTriangular): rows i > j of column j are zero
  const int64_t m_eff = b_upper ? min(m, j0 + UT_N) : m;
  const int nkt = (int)((m_eff + BKC - 1) / BKC);

  // Per-thread copy plan: A tile element e = tid + 128 i -> inner index e/64 = tid/64 + 2 i, row e%64 = tid%64;
  //                       B tile element e = tid + 128 i -> column tid/16 + 8 i, inner index tid%16.
  const int arow = tid & (UT_M - 1), aii = tid >> 6;
  const int bii = tid & (BKC - 1), bcol = tid >> 4;
  const bool arow_ok = r0 + arow < Krows;
  const cplx* pA = A + (r0 + arow) + lda * aii;
  const cplx* pB = B + bii + ldb * (j0 + bcol);
  unsigned okB = 0;
#pragma unroll
  for (int i = 0; i < UT_N / 8; ++i) okB |= (j0 + bcol + 8 * i < n) ? (1u << i) : 0u;
  auto load_tile = [&](int kt, int slot) {
    const int64_t i0 = (int64_t)kt * BKC;
    double* da = As + ((size_t)slot * BKC + aii) * LDA_U + 2 * arow;
    double* db = Bs + ((size_t)slot * UT_N + bcol) * LDK + 2 * bii;
#pragma unroll
    for (int i = 0; i < BKC / 2; ++i) {
      bool ok = arow_ok && (i0 + aii + 2 * i < m_eff);
      cp_async16(da + (size_t)2 * i * LDA_U, ok ? (pA + (i0 + 2 * i) * lda) : A, ok);
    }
    const bool iiok = i0 + bii < m_eff;
#pragma unroll
    for (int i = 0; i < UT_N / 8; ++i) {
      bool ok = iiok && ((okB >> i) & 1u);
      cp_async16(db + (size_t)8 * i * LDK, ok ? (pB + i0 + (int64_t)8 * i * ldb) : B, ok);
    }
  };

  double acc[4][4][2];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b][0] = acc[a][b][1] = 0.0;

  for (int s = 0; s < GEMM_STAGES - 1; ++s) {
    if (s < nkt) load_tile(s, s);
    cp_async_commit();
  }
  const int fr = lane >> 2, fk = lane & 3;
  const int wr = warp * 32;
  for (int kt = 0; kt < nkt; ++kt) {
    cp_async_wait<GEMM_STAGES - 2>();
    __syncthreads();
    {
      int nxt = kt + GEMM_STAGES - 1;
      if (nxt < nkt) load_tile(nxt, nxt % GEMM_STAGES);
      cp_async_commit();
    }
    const double* as = As + (size_t)(kt % GEMM_STAGES) * BKC * LDA_U;
    const double* bs = Bs + (size_t)(kt % GEMM_STAGES) * UT_N * LDK;
#pragma unroll
    for (int s4 = 0; s4 < 2 * BKC / 4; ++s4) {
      double af[4], bf[4];
      const int ii = 2 * s4 + (fk >> 1);
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        int R = wr + 8 * a + fr;  // real row inside the tile
        // A^[R][2i] = A~[R][i];  A^[R][2i+1] = (R odd) ? A~[R-1][i] : -A~[R+1][i]
        double v = as[ii * LDA_U + ((fk & 1) ? (R ^ 1) : R)];
        af[a] = ((fk & 1) && !(R & 1)) ? __hiloint2double(__double2hiint(v) ^ (int)0x80000000, __double2loint(v)) : v;
      }
#pragma unroll
      for (int b = 0; b < 4; ++b) bf[b] = bs[(8 * b + fr) * LDK + 4 * s4 + fk];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) dmma(acc[a][b][0], acc[a][b][1], af[a], bf[b]);
    }
  }
  cp_async_wait<0>();
  const bool has_beta = (beta.x != 0.0 || beta.y != 0.0);
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        int R = wr + 8 * a + fr;
        double v = acc[a][b][e];
        double partner = __shfl_xor_sync(0xffffffffu, v, 4);  // other component of the same complex entry
        int64_t grow = r0 + (R >> 1);
        int64_t gj = j0 + 8 * b + 2 * fk + e;
        double o;
        if (R & 1) o = alpha.x * v + alpha.y * partner;   // imaginary part: ar*im + ai*re
        else o = alpha.x * v - alpha.y * partner;         // real part:      ar*re - ai*im
        if (grow < Krows && gj < n) {
          double* cp = (double*)(C + grow + ldc * gj);
          if (has_beta) {
            double2 c = *(const double2*)cp;
            o += (R & 1) ? (beta.x * c.y + beta.y * c.x) : (beta.x * c.x - beta.y * c.y);
          }
          cp[R & 1] = o;
        }
      }
}

static size_t smem_cn(int st) { return (size_t)st * (GT_M + GT_N) * LDK * sizeof(double); }
static size_t smem_nn(int st) { return (size_t)st * (BKC * LDA_U + UT_N * LDK) * sizeof(double); }

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
  if (transA == 2) {
    int64_t tiles = ((m + GT_M - 1) / GT_M) * ((n + GT_N - 1) / GT_N);
    // split K so that the CTA count fills whole waves (3 resident CTAs per SM) at least twice over
    const int64_t slots = (ctx->gemm_stages == 3 ? 2 : 4) * (int64_t)ctx->sm_count;   // resident CTAs
    int64_t max_split = std::min<int64_t>(64, (k + 8 * BKC - 1) / (8 * BKC));
    int64_t nsplit = 1;
    double best = -1.0;
    for (int64_t sp = 1; sp <= max_split; ++sp) {
      int64_t total = tiles * sp;
      double eff = (double)total / (double)(((total + slots - 1) / slots) * slots);
      if (total < 2 * slots) eff *= 0.5 + 0.25 * (double)total / (double)slots;   // prefer >= 2 waves
      eff -= 0.002 * sp;                                                          // mild penalty: reduce pass
      if (eff > best) {
        best = eff;
        nsplit = sp;
      }
    }
    int64_t kps = (k + nsplit - 1) / nsplit;
    kps = ((kps + BKC - 1) / BKC) * BKC;
    nsplit = (k + kps - 1) / kps;
    cplx* ws = (cplx*)ctx->gemm_ws.ensure((size_t)nsplit * m * n * sizeof(cplx));
    dim3 grid((unsigned)((m + GT_M - 1) / GT_M), (unsigned)((n + GT_N - 1) / GT_N), (unsigned)nsplit);
    if (ctx->gemm_stages == 3)
      LAUNCH(ctx, k_zgemm_cn<3>, grid, GEMM_THREADS, smem_cn(3), A, lda, B, ldb, ws, m, n, k, kps,
             (upper_only && m == n) ? 1 : 0);
    else
      LAUNCH(ctx, k_zgemm_cn<2>, grid, GEMM_THREADS, smem_cn(2), A, lda, B, ldb, ws, m, n, k, kps,
             (upper_only && m == n) ? 1 : 0);
    LAUNCH(ctx, k_reduce_partials, (unsigned)((m * n + 255) / 256), 256, 0, (const cplx*)ws, (int)nsplit, m,
           n, alpha, beta, C, ldc);
  } else {
    REQUIRE((m + UT_M - 1) / UT_M <= 65535, "zgemm: more than 4.19M rows are not supported by the update kernel grid");
    dim3 grid((unsigned)((n + UT_N - 1) / UT_N), (unsigned)((m + UT_M - 1) / UT_M));
    if (ctx->gemm_stages == 3)
      LAUNCH(ctx, k_zgemm_nn<3>, grid, GEMM_THREADS, smem_nn(3), A, lda, B, ldb, C, ldc, m, n, k, alpha, beta,
             (upper_only && k == n) ? 1 : 0);
    else
      LAUNCH(ctx, k_zgemm_nn<2>, grid, GEMM_THREADS, smem_nn(2), A, lda, B, ldb, C, ldc, m, n, k, alpha, beta,
             (upper_only && k == n) ? 1 : 0);
  }
}

// hpsi += P (D (P' psi))      (apply!(::NonlocalOperator), src/terms/operators.jl:126-128)
void kb_apply_nonlocal(dftk_b200_kblock* kb, const cplx* psi, cplx* hpsi, int64_t n_bands) {
  if (kb->n_proj == 0 || n_bands == 0) return;
  dftk_b200_ctx* ctx = kb->grid->ctx;
  const int64_t np = kb->n_proj;
  cplx* proj = kb->proj.ensure((size_t)2 * np * n_bands);
  cplx* dproj = proj + (size_t)np * n_bands;
  const cplx one = make_double2(1.0, 0.0), zero = make_double2(0.0, 0.0);
  if (ctx->gemm_backend == 4 && np >= 64 && n_bands >= 32 && kb->n_pw >= ctx->i8_min_rows) {
    // both projector products on the INT8 tensor cores (wgmma s8, TMA-fed; i8emu.cu / i8tc2.cu): the residue
    // planes of P are prepared once per k-block and serve P'psi (K-major operand) and P (D P'psi) (MN-major operand)
    if (!kb->i8_Pop.planes) kb->i8_Pop = i8_prepare(ctx, kb->P.p, kb->n_pw, np, kb->n_pw, kb->i8_planes, kb->i8_exps);
    const I8Operand op_psi = i8_prepare(ctx, psi, kb->n_pw, n_bands, kb->n_pw, kb->i8_psi_planes, kb->i8_psi_exps);
    i8_gram(ctx, kb->i8_Pop, op_psi, proj, np, false);
    zgemm(ctx, 0, np, n_bands, np, one, kb->Dc.p, np, proj, np, zero, dproj, np);
    i8_update(ctx, 1, &kb->i8_Pop, dproj, np, n_bands, hpsi, kb->n_pw, 1.0, 1.0);
    return;
  }
  zgemm(ctx, 2, np, n_bands, kb->n_pw, one, kb->P.p, kb->n_pw, psi, kb->n_pw, zero, proj, np);
  zgemm(ctx, 0, np, n_bands, np, one, kb->Dc.p, np, proj, np, zero, dproj, np);
  zgemm(ctx, 0, kb->n_pw, n_bands, np, one, kb->P.p, kb->n_pw, dproj, np, one, hpsi, kb->n_pw);
}

}  // namespace dftk
