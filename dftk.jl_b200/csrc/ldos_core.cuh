// Kernel body of the LDOS product of many energies (ldos.cu; reference seam src/postprocess/dos.jl compute_ldos):
//   C[j ldc + r] += Σ_k D_k[r] W_k[j ldw]
// with D_k the staged band density |ψ_k(r)|²/Ω of band k of the round (N doubles) and W_k[j ldw] its weight at energy j.
// A real × real FP64 product on the DMMA pipe (mma.sync.m16n8k16.f64): rows r are the MMA's M, energies j its N and the
// bands of the round its K.  A CTA owns an LD_TM × LD_TN tile of C and runs all K of the round over it, so every output is
// read and written once per round and its sum has a fixed order (no atomics: a rerun is bit-identical).
// Host-callable: tests/hostemu runs the CTAs one after the other.  On the host a warp's 32 lanes are looped over and the
// MMA is evaluated from the fragments of all lanes; the accumulators of every thread of the CTA then live in `acc`
// (LD_SLOTS = LD_THREADS of them), where on the device each thread holds its own in registers (LD_SLOTS = 1).
#pragma once
#include "fft_core.cuh"

namespace dftk {

#define LD_THREADS 256           // 8 warps: 4 along r x 2 along j
#define LD_TM 128                // rows r per CTA tile (each warp 32: two MMA tiles of 16)
#define LD_TN 64                 // energies per CTA tile (each warp 32: four MMA tiles of 8)
#define LD_BK 32                 // bands per k step (two MMA k16)
#define LD_LDA (LD_TM + 8)       // doubles per band row of the D tile; % 16 == 8 => a fragment load takes two wavefronts
#define LD_LDB (LD_TN + 8)       // doubles per band row of the W tile; likewise
#define LD_SMEM_DOUBLES (LD_BK * (LD_LDA + LD_LDB))

#ifdef __CUDA_ARCH__
#define LD_SLOTS 1
#define LD_LN 1
#define LD_WARPS(w) for (int w = (int)threadIdx.x >> 5, wonce__ = 1; wonce__; wonce__ = 0)
#define LD_LANES(l) for (int l = (int)threadIdx.x & 31, lonce__ = 1; lonce__; lonce__ = 0)
#define LD_SLOT(w, l) 0
#define LD_LS(l) 0
#else
#define LD_SLOTS LD_THREADS
#define LD_LN 32
#define LD_WARPS(w) for (int w = 0; w < LD_THREADS / 32; ++w)
#define LD_LANES(l) for (int l = 0; l < 32; ++l)
#define LD_SLOT(w, l) ((w) * 32 + (l))
#define LD_LS(l) (l)
#endif

struct LdosProduct {
  const double* const* D;   // K band densities of the round (N doubles each)
  const double* const* W;   // K weight columns: energy j of band k at W[k][j * ldw]
  long long ldw;
  int K;
  long long M;              // rows: the grid points N
  int n;                    // energies
  double* C;                // C[j * ldc + r]
  long long ldc;
};

// accumulator e of MMA tile (a, b) of thread slot s
#define LD_ACC(acc, a, b, s) ((acc) + ((((a) * 4 + (b)) * LD_SLOTS + (s)) * 4))

// c += a b for one warp: A 16 x 16 (a[i]: row g + 8 (i & 1), k t + 4 (i >> 1)), B 16 x 8 (b[i]: k t + 4 i, column g),
// C 16 x 8 (c[e]: row g + 8 (e >> 1), column 2 t + (e & 1)), g = lane / 4, t = lane % 4.  c points at the lane-0 slot of the
// warp: one slot on the device, 32 consecutive ones on the host.
HD void ld_mma16(double* c, const double (*a)[8], const double (*b)[4]) {
#ifdef __CUDA_ARCH__
  asm("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
      "{%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
      : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
      : "d"(a[0][0]), "d"(a[0][1]), "d"(a[0][2]), "d"(a[0][3]), "d"(a[0][4]), "d"(a[0][5]), "d"(a[0][6]), "d"(a[0][7]),
        "d"(b[0][0]), "d"(b[0][1]), "d"(b[0][2]), "d"(b[0][3]));
#else
  double A[16][16], B[16][8];
  for (int l = 0; l < 32; ++l) {
    const int g = l >> 2, t = l & 3;
    for (int i = 0; i < 8; ++i) A[g + 8 * (i & 1)][t + 4 * (i >> 1)] = a[l][i];
    for (int i = 0; i < 4; ++i) B[t + 4 * i][g] = b[l][i];
  }
  for (int l = 0; l < 32; ++l) {
    const int g = l >> 2, t = l & 3;
    for (int e = 0; e < 4; ++e) {
      const int row = g + 8 * (e >> 1), col = 2 * t + (e & 1);
      double s = c[4 * l + e];
      for (int k = 0; k < 16; ++k) s = fma(A[row][k], B[k][col], s);
      c[4 * l + e] = s;
    }
  }
#endif
}

// number of MMA tiles of `size` (at most `cap`) needed to cover `rem` remaining outputs
HD int ld_tiles(long long rem, int size, int cap) {
  return rem <= 0 ? 0 : rem >= (long long)size * cap ? cap : (int)((rem + size - 1) / size);
}

// CTA (bm, bn): rows [bm LD_TM, +LD_TM), energies [bn LD_TN, +LD_TN).  sm: LD_SMEM_DOUBLES; acc: 2 x 4 x LD_SLOTS x 4.
HD void ldos_cta(const LdosProduct& p, long long bm, int bn, double* sm, double* acc) {
  double* As = sm;                       // [LD_BK][LD_LDA]: D tile, band-major
  double* Bs = sm + LD_BK * LD_LDA;      // [LD_BK][LD_LDB]: W tile, band-major
  const long long r0 = bm * LD_TM;
  const int j0 = bn * LD_TN;
  LD_WARPS(w) LD_LANES(l) {
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b)
#pragma unroll
        for (int e = 0; e < 4; ++e) LD_ACC(acc, a, b, LD_SLOT(w, l))[e] = 0.0;
  }
  for (int k0 = 0; k0 < p.K; k0 += LD_BK) {
    TSYNC();
    TLOOP(e, LD_BK * LD_TM) {
      const int k = e / LD_TM, r = e % LD_TM;
      As[k * LD_LDA + r] = (k0 + k < p.K && r0 + r < p.M) ? p.D[k0 + k][r0 + r] : 0.0;
    }
    TLOOP(e, LD_BK * LD_TN) {
      const int k = e / LD_TN, j = e % LD_TN;
      Bs[k * LD_LDB + j] = (k0 + k < p.K && j0 + j < p.n) ? p.W[k0 + k][(long long)(j0 + j) * p.ldw] : 0.0;
    }
    TSYNC();
    LD_WARPS(w) {
      const int wr = (w & 3) * 32, wj = (w >> 2) * 32;
      // MMA tiles of this warp that hold outputs (warp-uniform): narrow energy ranges skip the MMAs on padding
      const int na = ld_tiles(p.M - r0 - wr, 16, 2), nb = ld_tiles((long long)p.n - j0 - wj, 8, 4);
      if (na > 0 && nb > 0) {
#pragma unroll
        for (int ks = 0; ks < LD_BK / 16; ++ks) {
          double af[2][LD_LN][8], bf[4][LD_LN][4];
          LD_LANES(l) {
            const int g = l >> 2, t = l & 3;
#pragma unroll
            for (int a = 0; a < 2; ++a)
#pragma unroll
              for (int i = 0; i < 8; ++i)
                af[a][LD_LS(l)][i] = As[(16 * ks + t + 4 * (i >> 1)) * LD_LDA + wr + 16 * a + g + 8 * (i & 1)];
#pragma unroll
            for (int b = 0; b < 4; ++b)
#pragma unroll
              for (int i = 0; i < 4; ++i) bf[b][LD_LS(l)][i] = Bs[(16 * ks + t + 4 * i) * LD_LDB + wj + 8 * b + g];
          }
#pragma unroll
          for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b)
              if (a < na && b < nb) ld_mma16(LD_ACC(acc, a, b, LD_SLOT(w, 0)), af[a], bf[b]);
        }
      }
    }
  }
  LD_WARPS(w) LD_LANES(l) {
    const int g = l >> 2, t = l & 3, wr = (w & 3) * 32, wj = (w >> 2) * 32;
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const long long r = r0 + wr + 16 * a + g + 8 * (e >> 1);
          const int j = j0 + wj + 8 * b + 2 * t + (e & 1);
          if (r < p.M && j < p.n) p.C[(long long)j * p.ldc + r] += LD_ACC(acc, a, b, LD_SLOT(w, l))[e];
        }
  }
}

}  // namespace dftk
