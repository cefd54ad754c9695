// Tensor-core kernels of the INT8-residue GEMM emulation (option gemm_backend = 4, i8emu_core.cuh): for one modulus they form
// the four integer products
//     X1 = Ar^T Br,  X2 = Ai^T Bi,  X3 = Ar^T Bi,  X4 = Ai^T Br          (s8 x s8 -> s32, Hopper `wgmma.mma_async ... .s32.s8.s8`)
// of the residue planes and write their residues modulo p.
//
// Operand tiles travel global -> shared by TMA (`cp.async.bulk.tensor.2d`, 128-byte swizzle) into a ring of stages guarded
// by mbarriers (full: TMA transaction bytes, empty: one arrival per consumer thread).  Two consumer warpgroups own 64 output
// rows each and keep the four accumulators in registers; one producer warp issues the copies.  A consumer keeps one wgmma
// group in flight (wait_group 1) and releases a stage once the group that read it has completed.
//
// Shared-memory descriptor (sm_90 GMMA descriptor, K-major, SWIZZLE_128B): start address, LBO unused (one swizzle atom covers
// the 32-byte K extent of one instruction), SBO = 1024 B between 8-row groups, layout type 1.  Rows are 128 bytes of K; a
// K = 32 step advances the start address by 32 bytes.  Tile bases are 1024-byte aligned (the swizzle XORs address bits
// [4,7) with bits [7,10)).  wgmma takes 8-bit operands K-major only, so the update-type kernel transposes its MN-major tall
// operand in shared memory before the MMAs.
#include <cuda.h>
#include <algorithm>
#include <string>
#include "structs.cuh"
#include "i8emu_core.cuh"

namespace dftk {

constexpr int T2_M = 128;        // output rows per tile: two warpgroups x 64
constexpr int T2_N = 64;         // output columns per tile (4 accumulators x 32 registers per thread)
constexpr int T2_BK = 128;       // K bytes per stage = one swizzle row
constexpr int T2_STAGES = 4;
constexpr int T2_A_BYTES = T2_M * T2_BK;                         // 16 KB
constexpr int T2_B_BYTES = T2_N * T2_BK;                         // 8 KB
constexpr int T2_STAGE_BYTES = 2 * T2_A_BYTES + 2 * T2_B_BYTES;  // Ar, Ai, Br, Bi
constexpr int T2_SMEM = T2_STAGES * T2_STAGE_BYTES + 1024;       // + alignment slack
constexpr int T2_THREADS = 288;                                  // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int T2_CONSUMERS = 256;

__device__ __forceinline__ uint32_t t2_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void t2_mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(t2_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void t2_mbar_arrive(uint64_t* bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" :: "r"(t2_smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void t2_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" :: "r"(t2_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void t2_mbar_wait(uint64_t* bar, uint32_t parity) {
  const long long t0 = clock64();              // bounded: a protocol error traps after ~2 s instead of hanging the GPU
  for (;;) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P1;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P1;\n\t}\n"
        : "=r"(ok) : "r"(t2_smem_u32(bar)), "r"(parity) : "memory");
    if (ok) return;
    if (clock64() - t0 > 4000000000ll) __trap();
  }
}
__device__ __forceinline__ void t2_tma_load(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      :: "r"(t2_smem_u32(smem_dst)), "l"(map), "r"(c0), "r"(c1), "r"(t2_smem_u32(bar)) : "memory");
}
// K-major SWIZZLE_128B operand descriptor (LBO = 16 B, unused; SBO = 1024 B; layout type 1 = 128-byte swizzle)
__device__ __forceinline__ uint64_t t2_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
__device__ __forceinline__ void t2_wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void t2_wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void t2_wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void t2_wgmma_wait1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }
// d (64 x 64 s32, warpgroup fragment) += A (64 x 32 s8) B (32 x 64 s8), both from shared memory
__device__ __forceinline__ void t2_mma(int (&d)[32], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]),
        "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]),
        "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]),
        "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
      : "l"(da), "l"(db));
}
// accumulator fragment of m64nNk32: register r of thread (warp w of the warpgroup, lane l) holds row w*16 + l/4 + 8*((r/2)%2)
// and column (r/4)*8 + 2*(l%4) + r%2
__device__ __forceinline__ int t2_frag_row(int r, int wq, int lane) { return wq * 16 + (lane >> 2) + 8 * ((r >> 1) & 1); }
__device__ __forceinline__ int t2_frag_col(int r, int lane) { return (r >> 2) * 8 + 2 * (lane & 3) + (r & 1); }

// tensor maps: 2-D views [rows_total][ldk] of the residue planes of A (2 n_mod m rows, box 128 rows) and B (2 n_mod n rows,
// box 64 rows), 128 bytes of K per box.  grid (m tiles, n tiles, n_mod * n_chunks).  part[(chunk)][(2 t + part)][j][i] int16.
__global__ void __launch_bounds__(T2_THREADS, 1)
k_i8_gemm_tc2(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, int64_t m, int64_t n,
              int64_t ldk, int n_mod, int n_chunks, int64_t chunk_len, short* __restrict__ part, int upper_only) {
  // Hermitian results (X'X, X'AX): tiles strictly below the diagonal are never read by the callers
  if (upper_only && (int64_t)blockIdx.x * T2_M >= (int64_t)blockIdx.y * T2_N + T2_N) return;
  extern __shared__ unsigned char t2_raw[];
  unsigned char* sm = (unsigned char*)(((uintptr_t)t2_raw + 1023) & ~(uintptr_t)1023);
  __shared__ __align__(8) uint64_t full_bar[T2_STAGES], empty_bar[T2_STAGES];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int t = blockIdx.z % n_mod, chunk = blockIdx.z / n_mod;
  const int64_t i0 = (int64_t)blockIdx.x * T2_M, j0 = (int64_t)blockIdx.y * T2_N;
  const int64_t k_begin = (int64_t)chunk * chunk_len;
  const int64_t k_end = k_begin + chunk_len < ldk ? k_begin + chunk_len : ldk;
  const int n_iters = (int)((k_end - k_begin) / T2_BK);           // chunk_len and ldk are multiples of T2_BK

  if (tid == 0) {
    for (int s = 0; s < T2_STAGES; ++s) {
      t2_mbar_init(&full_bar[s], 1);                 // one arrive.expect_tx by the producer lane (+ the TMA transaction bytes)
      t2_mbar_init(&empty_bar[s], T2_CONSUMERS);     // every consumer thread once its MMAs of the stage have completed
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    // ---------------- TMA producer
    if (lane == 0) {
      const int row_ar = (int)((int64_t)(2 * t) * m + i0), row_ai = (int)((int64_t)(2 * t + 1) * m + i0);
      const int row_br = (int)((int64_t)(2 * t) * n + j0), row_bi = (int)((int64_t)(2 * t + 1) * n + j0);
      for (int it = 0; it < n_iters; ++it) {
        const int s = it % T2_STAGES;
        if (it >= T2_STAGES) t2_mbar_wait(&empty_bar[s], (uint32_t)((it / T2_STAGES - 1) & 1));
        unsigned char* stage = sm + (size_t)s * T2_STAGE_BYTES;
        const int kc = (int)(k_begin + (int64_t)it * T2_BK);
        t2_mbar_expect_tx(&full_bar[s], (uint32_t)T2_STAGE_BYTES);
        t2_tma_load(stage, &map_a, kc, row_ar, &full_bar[s]);
        t2_tma_load(stage + T2_A_BYTES, &map_a, kc, row_ai, &full_bar[s]);
        t2_tma_load(stage + 2 * T2_A_BYTES, &map_b, kc, row_br, &full_bar[s]);
        t2_tma_load(stage + 2 * T2_A_BYTES + T2_B_BYTES, &map_b, kc, row_bi, &full_bar[s]);
      }
    }
    return;
  }
  // ---------------- consumers: warpgroup g = rows [64 g, 64 g + 64) of the tile
  const int g = warp >> 2, wq = warp & 3;
  int x1[32], x2[32], x3[32], x4[32];
#pragma unroll
  for (int r = 0; r < 32; ++r) x1[r] = x2[r] = x3[r] = x4[r] = 0;
  for (int it = 0; it < n_iters; ++it) {
    const int s = it % T2_STAGES;
    t2_mbar_wait(&full_bar[s], (uint32_t)((it / T2_STAGES) & 1));
    const uint32_t base = t2_smem_u32(sm + (size_t)s * T2_STAGE_BYTES);
    const uint32_t ar = base + g * (64 * T2_BK), ai = ar + T2_A_BYTES;
    const uint32_t br = base + 2 * T2_A_BYTES, bi = br + T2_B_BYTES;
    t2_wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < T2_BK / 32; ++kk) {
      const uint32_t ko = (uint32_t)kk * 32u;
      t2_mma(x1, t2_desc(ar + ko), t2_desc(br + ko));
      t2_mma(x2, t2_desc(ai + ko), t2_desc(bi + ko));
      t2_mma(x3, t2_desc(ar + ko), t2_desc(bi + ko));
      t2_mma(x4, t2_desc(ai + ko), t2_desc(br + ko));
    }
    t2_wgmma_commit();
    t2_wgmma_wait1();                                                    // the group of it - 1 has completed
    if (it > 0) t2_mbar_arrive(&empty_bar[(it - 1) % T2_STAGES]);        // its stage is free
  }
  t2_wgmma_wait0();
  // ---------------- epilogue: residues modulo p of this K chunk as int16
  const int p = i8_modulus(t);
  const unsigned long long magic = i8_barrett_magic(p);
  short* out_re = part + (((size_t)chunk * 2 * n_mod + 2 * t) * n) * m;
  short* out_im = part + (((size_t)chunk * 2 * n_mod + 2 * t + 1) * n) * m;
#pragma unroll
  for (int r = 0; r < 32; ++r) {
    const int64_t i = i0 + g * 64 + t2_frag_row(r, wq, lane), j = j0 + t2_frag_col(r, lane);
    if (i < m && j < n) {
      // |x| <= 2^16 x 2^14: reduce each accumulator first (the sum of two would overflow int32)
      const int re = i8_reduce_sym(i8_reduce_sym(x1[r] >> 4, p, magic) * 16 + (x1[r] & 15) +
                                   i8_reduce_sym(x2[r] >> 4, p, magic) * 16 + (x2[r] & 15), p, magic);
      const int im = i8_reduce_sym(i8_reduce_sym(x3[r] >> 4, p, magic) * 16 + (x3[r] & 15) -
                                   i8_reduce_sym(x4[r] >> 4, p, magic) * 16 - (x4[r] & 15), p, magic);
      out_re[(size_t)j * m + i] = (short)re;
      out_im[(size_t)j * m + i] = (short)im;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------------
// Update-type products  C (m x n) = sum over blocks  A_b (m x K_b) B_b (K_b x n)  (LazyHcat * matrix of LOBPCG, P (D P'psi)):
// the tall operand A_b arrives in its stored orientation -- its residue planes [plane][column k][row G] are the ones the Gram
// products already prepared (G contiguous) -- and the small matrix B as K-major planes [plane][j][k].  Complex product
// without conjugation: re = X1 - X2, im = X3 + X4.  All blocks accumulate in registers (|sum| <= 1536 x 2^14: no int32
// overflow); the epilogue writes the symmetric residues as int8.
// The product is formed transposed, D[j, G] = sum_k B~[k, j] A[G, k]: the small matrix is the wgmma "A" operand (64 rows j
// per warpgroup), the tall operand the "B" operand (64 columns G).  Its stage holds the MN-major box [128 k][64 G]; the
// consumer threads transpose it into the K-major swizzled layout [64 G][128 k] (4 x 4 byte blocks through byte permutes)
// before the MMAs read it.  grid (n tiles, m tiles, n_mod): the n tiles of one G tile are neighbours in launch order and
// share the A tile in L2.
struct T2NnBlocks {
  int n_blocks;
  int kcols[3];      // columns of A_b = rows of its planes
  int n_iters[3];    // ceil(kcols / 128)
  int k_off[3];      // first (padded) contraction index of the block in B's planes (multiple of 128)
};

constexpr int NN_STAGES = 3;
constexpr int NN_S_BYTES = T2_M * T2_BK;                           // small matrix: 128 rows j x 128 k (16 KB)
constexpr int NN_T_BYTES = T2_BK * T2_N;                           // tall operand: 128 k x 64 G (8 KB), both orientations
constexpr int NN_STAGE_BYTES = 2 * NN_S_BYTES + 2 * NN_T_BYTES;   // Sr, Si, Tr, Ti (MN-major)
constexpr int NN_TT_BUFS = 3;                                      // transposed [Tr | Ti] tiles (one MMA group in flight)
constexpr int NN_SMEM = NN_STAGES * NN_STAGE_BYTES + NN_TT_BUFS * 2 * NN_T_BYTES + 1024;

// [128 k][64 G] (row-major) -> [64 G][128 k] in the 128-byte swizzle; 256 consumer threads, both parts
__device__ __forceinline__ void t2_transpose(const unsigned char* src, unsigned char* dst, int tid) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int b = tid + T2_CONSUMERS * q;              // 1024 blocks of 4 x 4 bytes: part, 32 k blocks, 16 G blocks
    const int part = b >> 9, kb = (b >> 4) & 31, gb = b & 15;
    const unsigned char* s = src + part * NN_T_BYTES + (4 * kb) * T2_N + 4 * gb;
    const uint32_t w0 = *reinterpret_cast<const uint32_t*>(s);
    const uint32_t w1 = *reinterpret_cast<const uint32_t*>(s + T2_N);
    const uint32_t w2 = *reinterpret_cast<const uint32_t*>(s + 2 * T2_N);
    const uint32_t w3 = *reinterpret_cast<const uint32_t*>(s + 3 * T2_N);
    const uint32_t t0 = __byte_perm(w0, w1, 0x5140), t1 = __byte_perm(w2, w3, 0x5140);
    const uint32_t t2 = __byte_perm(w0, w1, 0x7362), t3 = __byte_perm(w2, w3, 0x7362);
    const uint32_t o[4] = {__byte_perm(t0, t1, 0x5410), __byte_perm(t0, t1, 0x7632), __byte_perm(t2, t3, 0x5410),
                           __byte_perm(t2, t3, 0x7632)};
    unsigned char* d = dst + part * NN_T_BYTES;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int G = 4 * gb + c;                        // o[c]: k = 4 kb .. 4 kb + 3 of column G
      *reinterpret_cast<uint32_t*>(d + G * T2_BK + ((((kb >> 2) ^ (G & 7)) << 4) | ((4 * kb) & 15))) = o[c];
    }
  }
}

__global__ void __launch_bounds__(T2_THREADS, 1)
k_i8_gemm_tc2_nn(const __grid_constant__ CUtensorMap map_a0, const __grid_constant__ CUtensorMap map_a1,
                 const __grid_constant__ CUtensorMap map_a2, const __grid_constant__ CUtensorMap map_b, T2NnBlocks blocks,
                 int64_t m, int64_t n, int n_mod, signed char* __restrict__ resid, int64_t ldm) {
  extern __shared__ unsigned char t2_raw[];
  unsigned char* sm = (unsigned char*)(((uintptr_t)t2_raw + 1023) & ~(uintptr_t)1023);
  unsigned char* tt = sm + NN_STAGES * NN_STAGE_BYTES;               // transposed tall tiles, NN_TT_BUFS buffers
  __shared__ __align__(8) uint64_t full_bar[NN_STAGES], empty_bar[NN_STAGES];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int t = blockIdx.z;
  const int64_t j0 = (int64_t)blockIdx.x * T2_M, i0 = (int64_t)blockIdx.y * T2_N;      // j: MMA rows, G: MMA columns
  int total_iters = 0;
  for (int b = 0; b < blocks.n_blocks; ++b) total_iters += blocks.n_iters[b];

  if (tid == 0) {
    for (int s = 0; s < NN_STAGES; ++s) {
      t2_mbar_init(&full_bar[s], 1);
      t2_mbar_init(&empty_bar[s], T2_CONSUMERS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      const int row_br = (int)((int64_t)(2 * t) * n + j0), row_bi = (int)((int64_t)(2 * t + 1) * n + j0);
      int it = 0;
      for (int b = 0; b < blocks.n_blocks; ++b) {
        const CUtensorMap* ma = b == 0 ? &map_a0 : (b == 1 ? &map_a1 : &map_a2);
        const int kc = blocks.kcols[b];
        for (int q = 0; q < blocks.n_iters[b]; ++q, ++it) {
          const int s = it % NN_STAGES;
          if (it >= NN_STAGES) t2_mbar_wait(&empty_bar[s], (uint32_t)((it / NN_STAGES - 1) & 1));
          unsigned char* stage = sm + (size_t)s * NN_STAGE_BYTES;
          t2_mbar_expect_tx(&full_bar[s], (uint32_t)NN_STAGE_BYTES);
          // small matrix: 128 rows j x 128 bytes of k; tall operand: 128 contraction rows (plane rows k) x 64 bytes of G
          t2_tma_load(stage, &map_b, blocks.k_off[b] + q * T2_BK, row_br, &full_bar[s]);
          t2_tma_load(stage + NN_S_BYTES, &map_b, blocks.k_off[b] + q * T2_BK, row_bi, &full_bar[s]);
          t2_tma_load(stage + 2 * NN_S_BYTES, ma, (int)i0, (2 * t) * kc + q * T2_BK, &full_bar[s]);
          t2_tma_load(stage + 2 * NN_S_BYTES + NN_T_BYTES, ma, (int)i0, (2 * t + 1) * kc + q * T2_BK, &full_bar[s]);
        }
      }
    }
    return;
  }
  const int g = warp >> 2, wq = warp & 3;
  int x1[32], x2[32], x3[32], x4[32];
#pragma unroll
  for (int r = 0; r < 32; ++r) x1[r] = x2[r] = x3[r] = x4[r] = 0;
  for (int it = 0; it < total_iters; ++it) {
    const int s = it % NN_STAGES;
    t2_mbar_wait(&full_bar[s], (uint32_t)((it / NN_STAGES) & 1));
    unsigned char* stage = sm + (size_t)s * NN_STAGE_BYTES;
    unsigned char* tb = tt + (it % NN_TT_BUFS) * 2 * NN_T_BYTES;
    // buffer it % 3 was last read by the MMAs of iteration it - 3; every consumer waited for them (wait_group 1 at the end of
    // iteration it - 2) before it arrived at the barrier of iteration it - 1
    t2_transpose(stage + 2 * NN_S_BYTES, tb, tid);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy stores -> visible to wgmma
    asm volatile("bar.sync 1, %0;" :: "n"(T2_CONSUMERS) : "memory");
    const uint32_t sr = t2_smem_u32(stage) + g * (64 * T2_BK), si = sr + NN_S_BYTES;
    const uint32_t tr = t2_smem_u32(tb), ti = tr + NN_T_BYTES;
    t2_wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < T2_BK / 32; ++kk) {
      const uint32_t ko = (uint32_t)kk * 32u;
      t2_mma(x1, t2_desc(sr + ko), t2_desc(tr + ko));      // X1 = Sr Tr
      t2_mma(x2, t2_desc(si + ko), t2_desc(ti + ko));      // X2 = Si Ti
      t2_mma(x3, t2_desc(si + ko), t2_desc(tr + ko));      // X3 = Si Tr   (tall re x small im)
      t2_mma(x4, t2_desc(sr + ko), t2_desc(ti + ko));      // X4 = Sr Ti   (tall im x small re)
    }
    t2_wgmma_commit();
    t2_wgmma_wait1();
    if (it > 0) t2_mbar_arrive(&empty_bar[(it - 1) % NN_STAGES]);
  }
  t2_wgmma_wait0();
  // ---------------- epilogue: pairs of consecutive G of one row j leave as 16-bit stores
  const int p = i8_modulus(t);
  const unsigned long long magic = i8_barrett_magic(p);
#pragma unroll
  for (int r = 0; r < 32; r += 2) {
    const int64_t j = j0 + g * 64 + t2_frag_row(r, wq, lane), G = i0 + t2_frag_col(r, lane);
    if (j < n) {
      // |x| <= 1536 x 2^14 < 2^25: sums and differences of two accumulators stay below 2^26
      uint32_t wre = 0, wim = 0;
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        wre |= (uint32_t)(i8_reduce_sym(x1[r + q] - x2[r + q], p, magic) & 0xFF) << (8 * q);
        wim |= (uint32_t)(i8_reduce_sym(x3[r + q] + x4[r + q], p, magic) & 0xFF) << (8 * q);
      }
      *reinterpret_cast<uint16_t*>(resid + ((size_t)(2 * t) * n + j) * ldm + G) = (uint16_t)wre;
      *reinterpret_cast<uint16_t*>(resid + ((size_t)(2 * t + 1) * n + j) * ldm + G) = (uint16_t)wim;
    }
  }
}

__global__ void k_i8_sum_chunks2(const short* __restrict__ part, int n_chunks, int n_mod, int64_t mn, int* __restrict__ res) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= 2 * (int64_t)n_mod * mn) return;
  const int t = (int)(idx / (2 * mn));
  const int p = i8_modulus(t);
  int s = 0;
  for (int c = 0; c < n_chunks; ++c) s = (s + part[(size_t)c * 2 * n_mod * mn + idx]) % p;
  res[idx] = i8_sym(s, p);
}

void i8tc2_set_attributes() {
  CUDA_CHECK(cudaFuncSetAttribute(k_i8_gemm_tc2, cudaFuncAttributeMaxDynamicSharedMemorySize, T2_SMEM));
  CUDA_CHECK(cudaFuncSetAttribute(k_i8_gemm_tc2_nn, cudaFuncAttributeMaxDynamicSharedMemorySize, NN_SMEM));
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
    REQUIRE(p != nullptr && q == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled is not available in this driver");
    fn = (EncodeTiledFn)p;
  }
  return fn;
}
// 2-D view [rows_total][ld] of int8 planes; box = box_cols bytes x box_rows rows
static CUtensorMap plane_map(const signed char* base, int64_t rows_total, int64_t ld, int box_cols, int box_rows,
                             CUtensorMapSwizzle swizzle) {
  CUtensorMap map;
  const cuuint64_t gdim[2] = {(cuuint64_t)ld, (cuuint64_t)rows_total};
  const cuuint64_t gstride[1] = {(cuuint64_t)ld};                    // bytes between rows
  const cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
  const cuuint32_t estride[2] = {1, 1};
  const CUresult r = encode_tiled()(&map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, (void*)base, gdim, gstride, box, estride,
                                    CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw Error(DFTK_B200_ECUDA, "cuTensorMapEncodeTiled failed: " + std::to_string((int)r));
  return map;
}

// integer stage of the update-type product: blocks of prepared tall operands (planes [plane][col][ldm], ldm = padded rows) against
// the planes of the small matrix rb ([plane][j][ldkb], contraction index padded per block); resid: int8 [(2 t + part)][j][ldm]
void i8tc2_products_nn(dftk_b200_ctx* ctx, int n_blocks, const signed char* const* ra, const int* kcols, const int* k_off,
                       int64_t ldm, const signed char* rb, int64_t ldkb, int64_t m, int64_t n, int n_mod, signed char* resid) {
  REQUIRE(n_blocks >= 1 && n_blocks <= 3, "i8tc2_nn: 1..3 blocks");
  T2NnBlocks bl{};
  bl.n_blocks = n_blocks;
  CUtensorMap maps[3];
  for (int b = 0; b < n_blocks; ++b) {
    REQUIRE(((uintptr_t)ra[b] & 15) == 0 && ldm % T2_BK == 0 && k_off[b] % T2_BK == 0, "i8tc2_nn: alignment");
    bl.kcols[b] = kcols[b];
    bl.n_iters[b] = (kcols[b] + T2_BK - 1) / T2_BK;
    bl.k_off[b] = k_off[b];
    maps[b] = plane_map(ra[b], 2 * (int64_t)n_mod * kcols[b], ldm, T2_N, T2_BK, CU_TENSOR_MAP_SWIZZLE_NONE);
  }
  for (int b = n_blocks; b < 3; ++b) maps[b] = maps[0];
  const CUtensorMap map_b = plane_map(rb, 2 * (int64_t)n_mod * n, ldkb, T2_BK, T2_M, CU_TENSOR_MAP_SWIZZLE_128B);
  const int64_t m_tiles = (m + T2_N - 1) / T2_N;
  REQUIRE(m_tiles <= 65535, "i8tc2_nn: too many row tiles");
  dim3 grid((unsigned)((n + T2_M - 1) / T2_M), (unsigned)m_tiles, (unsigned)n_mod);
  LAUNCH(ctx, k_i8_gemm_tc2_nn, grid, T2_THREADS, NN_SMEM, maps[0], maps[1], maps[2], map_b, bl, m, n, n_mod, resid, ldm);
}

// integer stage of C = A^H B on the tensor cores, TMA-fed; ra / rb: padded residue planes (16-byte aligned, ldk % 128 == 0)
void i8tc2_products(dftk_b200_ctx* ctx, const signed char* ra, const signed char* rb, int64_t m, int64_t n, int64_t ldk,
                    int n_mod, short* part, int* res, bool upper_only) {
  REQUIRE(ldk % T2_BK == 0 && ((uintptr_t)ra & 15) == 0 && ((uintptr_t)rb & 15) == 0, "i8tc2: planes must be 16-byte aligned, ldk % 128 == 0");
  REQUIRE(2 * (int64_t)n_mod * std::max(m, n) < 2147483647, "i8tc2: too many plane rows");
  const int64_t chunk_len = I8_K_CHUNK;                         // multiple of T2_BK
  const int n_chunks = (int)((ldk + chunk_len - 1) / chunk_len);
  const CUtensorMap map_a = plane_map(ra, 2 * (int64_t)n_mod * m, ldk, T2_BK, T2_M, CU_TENSOR_MAP_SWIZZLE_128B);
  const CUtensorMap map_b = plane_map(rb, 2 * (int64_t)n_mod * n, ldk, T2_BK, T2_N, CU_TENSOR_MAP_SWIZZLE_128B);
  dim3 grid((unsigned)((m + T2_M - 1) / T2_M), (unsigned)((n + T2_N - 1) / T2_N), (unsigned)(n_mod * n_chunks));
  LAUNCH(ctx, k_i8_gemm_tc2, grid, T2_THREADS, T2_SMEM, map_a, map_b, m, n, ldk, n_mod, n_chunks, chunk_len, part, upper_only ? 1 : 0);
  const int64_t tot = 2 * (int64_t)n_mod * m * n;
  LAUNCH(ctx, k_i8_sum_chunks2, (unsigned)((tot + 255) / 256), 256, 0, (const short*)part, n_chunks, n_mod, m * n, res);
}

}  // namespace dftk
