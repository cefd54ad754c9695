// Reference device pipeline of the INT8-emulated FP64 complex GEMM (i8emu_core.cuh): column scales -> int8 residue planes
// -> per-modulus integer dot products -> CRT.  The integer products of option gemm_backend = 2 are plain CUDA-core loops
// (the checker); gemm_backend = 4 runs them on the tensor cores (i8tc2.cu).
#include "structs.cuh"
#include "i8emu_core.cuh"

namespace dftk {

// e[col] = scale exponent of column col (largest |re|, |im| over the rows); one CTA per column
__global__ void __launch_bounds__(256)
k_i8_col_exponent(const cplx* __restrict__ X, int64_t ld, int64_t n_rows, int bits, int* __restrict__ e) {
  const int64_t col = blockIdx.x;
  double mx = 0.0;
  for (int64_t r = threadIdx.x; r < n_rows; r += blockDim.x) {
    const cplx v = X[r + ld * col];
    mx = fmax(mx, fmax(fabs(v.x), fabs(v.y)));
  }
  __shared__ double red[8];
  for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_down_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) mx = fmax(mx, red[w]);
    e[col] = i8_scale_exponent(mx, bits);
  }
}

// planes[(2 t + part)][col][row] (row fastest: K-major per column), plane stride = n_cols * n_rows
__global__ void __launch_bounds__(256)
k_i8_residues(const cplx* __restrict__ X, int64_t ld, int64_t n_rows, int64_t n_cols, const int* __restrict__ e, int n_mod,
              signed char* __restrict__ planes) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t col = blockIdx.y;
  if (r >= n_rows) return;
  i8_residues_entry(X[r + ld * col], e[col], n_mod, planes + (r + n_rows * col), (long long)n_rows * n_cols);
}

// same with a padded leading dimension (tensor-core path: rows 16-byte aligned, K padded with zeros to the stage size)
__global__ void __launch_bounds__(256)
k_i8_residues_ld(const cplx* __restrict__ X, int64_t ld, int64_t n_rows, int64_t n_cols, int64_t ldk, const int* __restrict__ e,
                 int n_mod, signed char* __restrict__ planes) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t col = blockIdx.y;
  if (r >= n_rows) return;
  i8_residues_entry(X[r + ld * col], e[col], n_mod, planes + (r + ldk * col), (long long)ldk * n_cols);
}

// The same planes four K entries per thread: the rounded operand a' (at most 55 bits + sign) is split into three 20-bit
// limbs once, every residue is then a few 32-bit integer operations (limb * (2^20k mod p) summed, one remainder by a
// constant) instead of six FP64 operations, and the four int8 residues of a plane leave as one 32-bit store (a warp writes
// 128 contiguous bytes per plane instead of 32).  ldk % 4 == 0; rows [n_rows, ldk) of a column are zero padding.
__device__ __forceinline__ void i8_limbs(double a, int& l0, int& l1, int& l2) {
  long long v = (long long)a;                     // |a'| < 2^56: exact
  const long long s = v >> 63;                    // limbs of |v| with the sign folded into each (C remainder semantics)
  long long u = (v ^ s) - s;
  const int sg = (int)(1 | s);
  l0 = sg * (int)(u & 0xFFFFF);
  l1 = sg * (int)((u >> 20) & 0xFFFFF);
  l2 = sg * (int)(u >> 40);
}
__global__ void __launch_bounds__(256)
k_i8_residues_ld4(const cplx* __restrict__ X, int64_t ld, int64_t n_rows, int64_t n_cols, int64_t ldk, const int* __restrict__ e,
                  int n_mod, signed char* __restrict__ planes) {
  const int64_t r4 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const int64_t col = blockIdx.y;
  if (r4 >= ldk) return;
  const int ex = e[col];
  int lr[4][3], li[4][3];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    cplx x = make_double2(0.0, 0.0);
    if (r4 + q < n_rows) x = X[r4 + q + ld * col];
    i8_limbs(rint(ldexp(x.x, ex)), lr[q][0], lr[q][1], lr[q][2]);
    i8_limbs(rint(ldexp(x.y, ex)), li[q][0], li[q][1], li[q][2]);
  }
  const long long plane_stride = (long long)ldk * n_cols;
  signed char* out = planes + (r4 + ldk * col);
#pragma unroll
  for (int t = 0; t < I8_MAX_MODULI; ++t) {          // unrolled: p, c1, c2 are compile-time constants (no integer division)
    if (t >= n_mod) break;
    const int p = i8_modulus(t);
    const int c1 = (1 << 20) % p, c2 = (int)((1ll << 40) % p);
    unsigned wr = 0, wi = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      // |l0 + l1 c1 + l2 c2| < 2^20 + 2^28 + 2^24: int32
      const int rr = i8_sym(lr[q][0] + lr[q][1] * c1 + lr[q][2] * c2, p);
      const int ri = i8_sym(li[q][0] + li[q][1] * c1 + li[q][2] * c2, p);
      wr |= (unsigned)(rr & 0xFF) << (8 * q);
      wi |= (unsigned)(ri & 0xFF) << (8 * q);
    }
    *reinterpret_cast<unsigned*>(out + (long long)(2 * t) * plane_stride) = wr;
    *reinterpret_cast<unsigned*>(out + (long long)(2 * t + 1) * plane_stride) = wi;
  }
}

// one warp per (i, j, t): residues of conj(a_i) . b_j modulo p_t;  res[(2 t + part)][j][i]
__global__ void __launch_bounds__(256)
k_i8_dot_ref(const signed char* __restrict__ ra, const signed char* __restrict__ rb, int64_t m, int64_t n, int64_t k,
             int n_mod, int* __restrict__ res) {
  const int lane = threadIdx.x & 31;
  const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (w >= m * n * n_mod) return;
  const int64_t i = w % m, j = (w / m) % n;
  const int t = (int)(w / (m * n));
  const int p = i8_modulus(t);
  const signed char* ar = ra + (size_t)(2 * t) * m * k + k * i;
  const signed char* ai = ra + (size_t)(2 * t + 1) * m * k + k * i;
  const signed char* br = rb + (size_t)(2 * t) * n * k + k * j;
  const signed char* bi = rb + (size_t)(2 * t + 1) * n * k + k * j;
  int sre = 0, sim = 0;
  for (int64_t k0 = 0; k0 < k; k0 += 32 * (int64_t)I8_K_CHUNK) {       // per lane at most I8_K_CHUNK terms per int32 sum
    const int64_t k1 = k0 + 32 * (int64_t)I8_K_CHUNK < k ? k0 + 32 * (int64_t)I8_K_CHUNK : k;
    int x1 = 0, x2 = 0, x3 = 0, x4 = 0;
    for (int64_t q = k0 + lane; q < k1; q += 32) {
      const int a0 = ar[q], a1 = ai[q], b0 = br[q], b1 = bi[q];
      x1 += a0 * b0;
      x2 += a1 * b1;
      x3 += a0 * b1;
      x4 += a1 * b0;
    }
    sre = (sre + x1 % p + x2 % p) % p;
    sim = (sim + x3 % p - x4 % p) % p;
  }
  for (int o = 16; o > 0; o >>= 1) {                                     // |partial| < p: the warp sum stays below 32 p
    sre += __shfl_down_sync(0xffffffffu, sre, o);
    sim += __shfl_down_sync(0xffffffffu, sim, o);
  }
  if (lane == 0) {
    res[((size_t)(2 * t) * n + j) * m + i] = i8_sym(sre, p);
    res[((size_t)(2 * t + 1) * n + j) * m + i] = i8_sym(sim, p);
  }
}

__global__ void __launch_bounds__(128)
k_i8_crt(const int* __restrict__ res, int64_t m, int64_t n, I8Tables T, const int* __restrict__ ea, const int* __restrict__ eb,
         cplx* __restrict__ C, int64_t ldc, int accumulate) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= m * n) return;
  const int64_t i = idx % m, j = idx / m;
  int rre[I8_MAX_MODULI], rim[I8_MAX_MODULI];
#pragma unroll
  for (int t = 0; t < I8_MAX_MODULI; ++t) {
    rre[t] = rim[t] = 0;
    if (t < T.n_mod) {
      rre[t] = res[((size_t)(2 * t) * n + j) * m + i];
      rim[t] = res[((size_t)(2 * t + 1) * n + j) * m + i];
    }
  }
  const int sh = -(ea[i] + eb[j]);
  cplx v = make_double2(ldexp(i8_crt(rre, T), sh), ldexp(i8_crt(rim, T), sh));
  if (accumulate) {
    const cplx o = C[i + ldc * j];
    v.x += o.x;
    v.y += o.y;
  }
  C[i + ldc * j] = v;
}

// ---- update-type products C (m x n) (+)= A B, A: m x k (rows scaled), B: k x n (columns scaled) ----
// e[row] = scale exponent of row `row` of A (largest |re|, |im| over the k columns)
__global__ void __launch_bounds__(256)
k_i8_row_exponent(const cplx* __restrict__ A, int64_t lda, int64_t m, int64_t k, int bits, int* __restrict__ e) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  double mx = 0.0;
  for (int64_t c = 0; c < k; ++c) {
    const cplx v = A[i + lda * c];
    mx = fmax(mx, fmax(fabs(v.x), fabs(v.y)));
  }
  e[i] = i8_scale_exponent(mx, bits);
}
// planes[(2 t + part)][c][i] (i fastest, like A itself), plane stride = m * k
__global__ void __launch_bounds__(256)
k_i8_residues_rows(const cplx* __restrict__ A, int64_t lda, int64_t m, int64_t k, const int* __restrict__ e, int n_mod,
                   signed char* __restrict__ planes) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t c = blockIdx.y;
  if (i >= m) return;
  i8_residues_entry(A[i + lda * c], e[i], n_mod, planes + (i + m * c), (long long)m * k);
}
// one thread per (i, j, t);  res[(2 t + part)][j][i]
__global__ void __launch_bounds__(256)
k_i8_dot_plain_ref(const signed char* __restrict__ ra, const signed char* __restrict__ rb, int64_t m, int64_t n, int64_t k,
                   int n_mod, int* __restrict__ res) {
  const int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= m * n * n_mod) return;
  const int64_t i = w % m, j = (w / m) % n;
  const int t = (int)(w / (m * n));
  int re, im;
  i8_dot_plain(ra + (size_t)(2 * t) * m * k + i, ra + (size_t)(2 * t + 1) * m * k + i, m,
               rb + (size_t)(2 * t) * n * k + k * j, rb + (size_t)(2 * t + 1) * n * k + k * j, 1, k, i8_modulus(t), &re, &im);
  res[((size_t)(2 * t) * n + j) * m + i] = re;
  res[((size_t)(2 * t + 1) * n + j) * m + i] = im;
}

// number of moduli for FP64-level accuracy at contraction length K (55 bits per operand, scripts/ozaki_study.py)
static I8Tables tables_for(int64_t K) {
  for (int n = 8; n <= I8_MAX_MODULI; ++n) {
    I8Tables T = i8_make_tables(n, K);
    if (T.bits >= 55) return T;
  }
  return i8_make_tables(I8_MAX_MODULI, K);
}

// C (m x n) = A^H B,  A: k x m, B: k x n (column-major, complex).  tensor_cores: integer products by k_i8_gemm_tc (i8tc.cu)
// ---- prepared operands: an operand (a block of columns along the contraction index) is converted ONCE and then enters any
//      number of products C = A^H B (the block Gram matrices of LOBPCG reuse every block three times)
I8Operand i8_prepare(dftk_b200_ctx* ctx, const cplx* X, int64_t ld, int64_t cols, int64_t k, DevBuf<signed char>& store,
                     DevBuf<int>& estore) {
  I8Operand op;
  const I8Tables T = tables_for(2 * k);
  op.cols = cols;
  op.k = k;
  op.ldk = (k + 127) / 128 * 128;
  op.n_mod = T.n_mod;
  signed char* r = store.ensure(2 * (size_t)T.n_mod * cols * op.ldk + 16);
  r += (16 - ((uintptr_t)r & 15)) & 15;
  int* e = estore.ensure((size_t)cols);
  LAUNCH(ctx, k_i8_col_exponent, (unsigned)cols, 256, 0, X, ld, k, T.bits, e);
  LAUNCH(ctx, k_i8_residues_ld4, dim3((unsigned)((op.ldk / 4 + 255) / 256), (unsigned)cols), 256, 0, X, ld, k, cols, op.ldk, (const int*)e,
         T.n_mod, r);
  op.planes = r;
  op.exps = e;
  return op;
}
// C (A.cols x B.cols, leading dimension ldc) = A^H B from prepared operands: TMA-fed wgmma s8 products, chunk sums, CRT.
// upper_only: tiles strictly below the diagonal are skipped (their entries of C are unspecified), as in the DMMA kernel.
void i8_gram(dftk_b200_ctx* ctx, const I8Operand& A, const I8Operand& B, cplx* C, int64_t ldc, bool upper_only) {
  REQUIRE(A.k == B.k && A.ldk == B.ldk && A.n_mod == B.n_mod, "i8_gram: operands prepared for different contraction lengths");
  const int64_t m = A.cols, n = B.cols;
  if (m == 0 || n == 0) return;
  const I8Tables T = tables_for(2 * A.k);
  const int n_chunks = (int)((A.ldk + I8_K_CHUNK - 1) / I8_K_CHUNK);
  const size_t n_res = 2 * (size_t)T.n_mod * m * n;
  char* ws = (char*)ctx->gemm_ws.ensure(n_res * sizeof(int) + n_res * n_chunks * sizeof(short) + 256);
  int* res = (int*)ws;
  short* part = (short*)(res + n_res);
  i8tc2_products(ctx, A.planes, B.planes, m, n, A.ldk, T.n_mod, part, res, upper_only);
  LAUNCH(ctx, k_i8_crt, (unsigned)((m * n + 127) / 128), 128, 0, (const int*)res, m, n, T, A.exps, B.exps, C, ldc, 0);
}

// ---- update-type products from prepared tall operands:  C (m x n) = alpha sum_b A_b B[rows of b, :] + beta C.
// A_b's planes hold a'[G,k] = round(A[G,k] 2^{e_k}) with one scale per COLUMN k (as prepared for the Gram products); the scale
// moves into the small matrix, B~[k,j] = B[k,j] 2^{-e_k}, whose columns get their own scales f_j:  C = 2^{-f_j} sum a' b'
// exactly.  (Errors: the two operand roundings, relative to the column maxima of A and of B~ -- a norm-wise bound like the
// FP64 GEMM's, not a component-wise one.)
struct I8BBlocks {
  int n_blocks;
  int k0[3];        // first row of block b in B
  int kc[3];        // its number of rows (= columns of A_b)
  int pad0[3];      // first padded contraction index of block b in the planes (multiple of 128)
  const int* exps[3];
};
// f[j]: scale exponent of column j of B~ (one CTA per column)
__global__ void __launch_bounds__(256)
k_i8_bscale_exponent(const cplx* __restrict__ B, int64_t ldb, I8BBlocks bl, int bits, int* __restrict__ f) {
  const int64_t j = blockIdx.x;
  double mx = 0.0;
  for (int b = 0; b < bl.n_blocks; ++b)
    for (int k = threadIdx.x; k < bl.kc[b]; k += blockDim.x) {
      const cplx v = B[bl.k0[b] + k + ldb * j];
      mx = fmax(mx, ldexp(fmax(fabs(v.x), fabs(v.y)), -bl.exps[b][k]));
    }
  __shared__ double red[8];
  for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_down_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) mx = fmax(mx, red[w]);
    f[j] = i8_scale_exponent(mx, bits);
  }
}
// planes[(2 t + part)][j][ldkb]: residues of round(B[k,j] 2^{f_j - e_k}) at the padded contraction index, zeros in the padding
__global__ void __launch_bounds__(256)
k_i8_bscale_residues(const cplx* __restrict__ B, int64_t ldb, int64_t n, I8BBlocks bl, int64_t ldkb, const int* __restrict__ f,
                     int n_mod, signed char* __restrict__ planes) {
  const int64_t kp = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t j = blockIdx.y;
  if (kp >= ldkb) return;
  cplx x = make_double2(0.0, 0.0);
  int e = 0;
  for (int b = 0; b < bl.n_blocks; ++b)
    if (kp >= bl.pad0[b] && kp < bl.pad0[b] + bl.kc[b]) {
      const int k = (int)(kp - bl.pad0[b]);
      x = B[bl.k0[b] + k + ldb * j];
      e = f[j] - bl.exps[b][k];
    }
  i8_residues_entry(x, e, n_mod, planes + (kp + ldkb * j), (long long)ldkb * n);
}
// C[G, j] = alpha 2^{-f_j} CRT(residues) + beta C[G, j];  resid: int8 [(2 t + part)][j][ldm].  Four consecutive rows per thread:
// one 32-bit load per residue plane, 64 contiguous bytes of C.
__global__ void __launch_bounds__(128)
k_i8_crt_nn(const signed char* __restrict__ resid, int64_t m, int64_t n, int64_t ldm, I8Tables T, const int* __restrict__ f,
            cplx* __restrict__ C, int64_t ldc, double alpha, double beta) {
  const int64_t i4 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const int64_t j = blockIdx.y;
  if (i4 >= m) return;
  unsigned wre[I8_MAX_MODULI], wim[I8_MAX_MODULI];
#pragma unroll
  for (int t = 0; t < I8_MAX_MODULI; ++t) {          // unrolled: the residue words stay in registers
    wre[t] = wim[t] = 0;
    if (t < T.n_mod) {
      wre[t] = *reinterpret_cast<const unsigned*>(resid + ((size_t)(2 * t) * n + j) * ldm + i4);        // ldm % 128 == 0: aligned
      wim[t] = *reinterpret_cast<const unsigned*>(resid + ((size_t)(2 * t + 1) * n + j) * ldm + i4);
    }
  }
  const int sh = -f[j];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    if (i4 + q >= m) break;
    int rre[I8_MAX_MODULI], rim[I8_MAX_MODULI];
#pragma unroll
    for (int t = 0; t < I8_MAX_MODULI; ++t) {
      rre[t] = (int)(signed char)((wre[t] >> (8 * q)) & 0xFF);
      rim[t] = (int)(signed char)((wim[t] >> (8 * q)) & 0xFF);
    }
    cplx v = make_double2(alpha * ldexp(i8_crt(rre, T), sh), alpha * ldexp(i8_crt(rim, T), sh));
    if (beta != 0.0) {
      const cplx o = C[i4 + q + ldc * j];
      v.x += beta * o.x;
      v.y += beta * o.y;
    }
    C[i4 + q + ldc * j] = v;
  }
}

void i8_update(dftk_b200_ctx* ctx, int n_blocks, const I8Operand* A, const cplx* B, int64_t ldb, int64_t n, cplx* C, int64_t ldc,
               double alpha, double beta) {
  REQUIRE(n_blocks >= 1 && n_blocks <= 3 && n >= 1, "i8_update: 1..3 blocks");
  const int64_t m = A[0].k, ldm = A[0].ldk;       // the operands' contraction length is the output's row count
  const I8Tables T = tables_for(2 * m);
  I8BBlocks bl{};
  bl.n_blocks = n_blocks;
  int k0 = 0, pad = 0;
  int kcols[3], k_off[3];
  const signed char* ra[3];
  for (int b = 0; b < n_blocks; ++b) {
    REQUIRE(A[b].k == m && A[b].ldk == ldm && A[b].n_mod == T.n_mod, "i8_update: blocks prepared differently");
    bl.k0[b] = k0;
    bl.kc[b] = (int)A[b].cols;
    bl.pad0[b] = pad;
    bl.exps[b] = A[b].exps;
    kcols[b] = (int)A[b].cols;
    k_off[b] = pad;
    ra[b] = A[b].planes;
    k0 += (int)A[b].cols;
    pad += (int)((A[b].cols + 127) / 128 * 128);
  }
  const int64_t ldkb = pad;
  // K 2^(2 bits) <= P / 4 holds a fortiori: the tables were sized for the (much longer) contraction of the Gram products
  const size_t plane_b = (size_t)n * ldkb;
  const size_t bytes = (size_t)n * sizeof(int) + 64 + 2 * (size_t)T.n_mod * plane_b + 64 + 2 * (size_t)T.n_mod * n * ldm + 64;
  char* ws = (char*)ctx->gemm_ws.ensure(bytes);
  int* f = (int*)ws;
  signed char* rb = (signed char*)(f + n);
  rb += (16 - ((uintptr_t)rb & 15)) & 15;
  signed char* resid = rb + 2 * (size_t)T.n_mod * plane_b;
  resid += (16 - ((uintptr_t)resid & 15)) & 15;
  LAUNCH(ctx, k_i8_bscale_exponent, (unsigned)n, 256, 0, B, ldb, bl, T.bits, f);
  LAUNCH(ctx, k_i8_bscale_residues, dim3((unsigned)((ldkb + 255) / 256), (unsigned)n), 256, 0, B, ldb, n, bl, ldkb, (const int*)f,
         T.n_mod, rb);
  i8tc2_products_nn(ctx, n_blocks, ra, kcols, k_off, ldm, rb, ldkb, m, n, T.n_mod, resid);
  LAUNCH(ctx, k_i8_crt_nn, dim3((unsigned)((m + 511) / 512), (unsigned)n), 128, 0, (const signed char*)resid, m, n, ldm, T, (const int*)f,
         C, ldc, alpha, beta);
}

void zgemm_i8_cn(dftk_b200_ctx* ctx, int64_t m, int64_t n, int64_t k, const cplx* A, int64_t lda, const cplx* B, int64_t ldb,
                 cplx* C, int64_t ldc, bool tensor_cores, const signed char* ra_cached, const int* ea_cached) {
  if (m == 0 || n == 0) return;
  REQUIRE(k >= 1 && m <= 65535 && n <= 65535, "zgemm_i8: unsupported shape");
  const I8Tables T = tables_for(2 * k);
  const int64_t ldk = tensor_cores ? (k + 127) / 128 * 128 : k;
  const int n_chunks = (int)((ldk + I8_K_CHUNK - 1) / I8_K_CHUNK);
  const size_t plane_a = (size_t)m * ldk, plane_b = (size_t)n * ldk;
  const size_t n_res = 2 * (size_t)T.n_mod * m * n;
  const bool cached = ra_cached != nullptr && tensor_cores;
  const size_t bytes = (size_t)(m + n) * sizeof(int) + 64 + n_res * sizeof(int) + 2 * (size_t)T.n_mod * ((cached ? 0 : plane_a) + plane_b) + 256 +
                       (tensor_cores ? n_res * n_chunks * sizeof(short) : 0);
  char* ws = (char*)ctx->gemm_ws.ensure(bytes);
  int* ea = (int*)ws;
  int* eb = ea + m;
  int* res = eb + n;
  signed char* ra = (signed char*)(res + n_res);
  ra += (16 - ((uintptr_t)ra & 15)) & 15;                       // cp.async / TMA need 16-byte aligned rows
  signed char* rb = ra + (cached ? 0 : 2 * (size_t)T.n_mod * plane_a);
  short* part = (short*)(rb + 2 * (size_t)T.n_mod * plane_b);
  if (cached) {
    ra = const_cast<signed char*>(ra_cached);
    ea = const_cast<int*>(ea_cached);
  } else {
    LAUNCH(ctx, k_i8_col_exponent, (unsigned)m, 256, 0, A, lda, k, T.bits, ea);
  }
  LAUNCH(ctx, k_i8_col_exponent, (unsigned)n, 256, 0, B, ldb, k, T.bits, eb);
  if (tensor_cores) {
    // (the four-per-thread kernel writes the zero K padding itself)
    if (!cached)
      LAUNCH(ctx, k_i8_residues_ld4, dim3((unsigned)((ldk / 4 + 255) / 256), (unsigned)m), 256, 0, A, lda, k, m, ldk, (const int*)ea,
             T.n_mod, ra);
    LAUNCH(ctx, k_i8_residues_ld4, dim3((unsigned)((ldk / 4 + 255) / 256), (unsigned)n), 256, 0, B, ldb, k, n, ldk, (const int*)eb,
           T.n_mod, rb);
    i8tc2_products(ctx, ra, rb, m, n, ldk, T.n_mod, part, res, false);
  } else {
    LAUNCH(ctx, k_i8_residues, dim3((unsigned)((k + 255) / 256), (unsigned)m), 256, 0, A, lda, k, m, (const int*)ea, T.n_mod, ra);
    LAUNCH(ctx, k_i8_residues, dim3((unsigned)((k + 255) / 256), (unsigned)n), 256, 0, B, ldb, k, n, (const int*)eb, T.n_mod, rb);
    const int64_t warps = m * n * T.n_mod;
    LAUNCH(ctx, k_i8_dot_ref, (unsigned)((warps * 32 + 255) / 256), 256, 0, (const signed char*)ra, (const signed char*)rb, m, n,
           k, T.n_mod, res);
  }
  LAUNCH(ctx, k_i8_crt, (unsigned)((m * n + 127) / 128), 128, 0, (const int*)res, m, n, T, (const int*)ea, (const int*)eb, C, ldc, 0);
}

// C (m x n) = A B (+ C if accumulate): reference pipeline only (integer products on CUDA cores); returns false when the
// residue planes would not fit the workspace budget (the caller then uses the DMMA kernel)
bool zgemm_i8_nn(dftk_b200_ctx* ctx, int64_t m, int64_t n, int64_t k, const cplx* A, int64_t lda, const cplx* B, int64_t ldb,
                 cplx* C, int64_t ldc, bool accumulate) {
  if (m == 0 || n == 0 || k == 0) return true;
  const I8Tables T = tables_for(2 * k);
  const size_t n_res = 2 * (size_t)T.n_mod * m * n;
  const size_t bytes = (size_t)(m + n) * sizeof(int) + 64 + n_res * sizeof(int) + 2 * (size_t)T.n_mod * (size_t)k * (m + n) + 64;
  if (bytes > ((size_t)8 << 30) || k > 65535 || m * n * T.n_mod > (int64_t)1 << 40) return false;
  char* ws = (char*)ctx->gemm_ws.ensure(bytes);
  int* ea = (int*)ws;
  int* eb = ea + m;
  int* res = eb + n;
  signed char* ra = (signed char*)(res + n_res);
  signed char* rb = ra + 2 * (size_t)T.n_mod * m * k;
  LAUNCH(ctx, k_i8_row_exponent, (unsigned)((m + 255) / 256), 256, 0, A, lda, m, k, T.bits, ea);
  LAUNCH(ctx, k_i8_col_exponent, (unsigned)n, 256, 0, B, ldb, k, T.bits, eb);
  LAUNCH(ctx, k_i8_residues_rows, dim3((unsigned)((m + 255) / 256), (unsigned)k), 256, 0, A, lda, m, k, (const int*)ea, T.n_mod, ra);
  LAUNCH(ctx, k_i8_residues, dim3((unsigned)((k + 255) / 256), (unsigned)n), 256, 0, B, ldb, k, n, (const int*)eb, T.n_mod, rb);
  const int64_t threads = m * n * T.n_mod;
  LAUNCH(ctx, k_i8_dot_plain_ref, (unsigned)((threads + 255) / 256), 256, 0, (const signed char*)ra, (const signed char*)rb, m, n,
         k, T.n_mod, res);
  LAUNCH(ctx, k_i8_crt, (unsigned)((m * n + 127) / 128), 128, 0, (const int*)res, m, n, T, (const int*)ea, (const int*)eb, C, ldc,
         accumulate ? 1 : 0);
  return true;
}

}  // namespace dftk
