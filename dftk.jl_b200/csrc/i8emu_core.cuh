// FP64 complex GEMM emulated with INT8 products and INT32 accumulation: the GEMM-shaped half of H psi -- P' psi,
// P (D P' psi), the LOBPCG Gram/update products -- moves from the FP64 DMMA pipe onto the INT8 tensor cores (Hopper
// `wgmma ... .s32.s8.s8` multiplies s8 x s8 into s32 register accumulators, i8tc2.cu).  scripts/ozaki_study.py holds the
// numerics study that selected the scheme.
//
// Scheme (integer modular technique, Ozaki / Uchino / Imamura 2025):
//   1. every column of an operand (a vector along the contraction index) gets a power-of-two scale 2^e such that
//      a' = round(a 2^e) is an integer of at most `bits` bits, with  K 2^(2 bits) <= P / 4,  P = prod of the moduli;
//   2. a' is reduced modulo N pairwise coprime moduli p_t <= 256 to symmetric residues in [-128, 127]  (int8 planes);
//   3. per modulus the residues are multiplied exactly: int8 x int8 products, int32 accumulation over at most 2^17 terms,
//      partial sums reduced mod p_t;
//   4. the Chinese remainder theorem recombines the N residues of every output element into the exact integer
//      C' = sum a' b'  (|C'| <= P/4), evaluated with 40-bit limbs held in FP64 (all limb operations are exact);
//   5. C = C' 2^-(e_a + e_b).
// The only errors are the roundings of step 1: with N = 16 (55 bits per operand at K = 8.5k) the result is as accurate as
// an FP64 GEMM; N = 17 covers K = 2 x 264 859.
// Bodies are __host__ __device__ (host emulation in tests/hostemu).
#pragma once
#include <math.h>
#include <stdint.h>
#include "fft_core.cuh"

namespace dftk {

#define I8_MAX_MODULI 20
#define I8_LIMBS 4          // 40-bit limbs: covers P < 2^160
#define I8_K_CHUNK 65536    // int32 accumulation: 2^16 x 128 x 128 = 2^30

// pairwise coprime, all <= 256 (256 = 2^8, 255 = 3 5 17, 253 = 11 23, 251, 247 = 13 19, 241, 239, 233, 229, 227, 223, 217 = 7 31, ...)
HD int i8_modulus(int t) {
  const int p[I8_MAX_MODULI] = {256, 255, 253, 251, 247, 241, 239, 233, 229, 227, 223, 217, 211, 199, 197, 193, 191, 181, 179, 173};
  return p[t];
}

struct I8Tables {
  int n_mod;
  int bits;                              // operand budget for the contraction length the tables were built for
  int q[I8_MAX_MODULI];                  // (P / p_t)^-1 mod p_t
  double w[I8_MAX_MODULI][I8_LIMBS];     // P / p_t in 40-bit limbs (little endian)
  double P[I8_LIMBS];                    // P in 40-bit limbs
  double P_top;                          // P as a double (rounded) for the quotient estimate
};

// symmetric residue of an integer-valued double (|a| < 2^62) modulo p, in [-(p/2), (p-1)/2] (256 -> [-128, 127])
HD int i8_residue(double a, int p) {
  long long v = (long long)a;
  int r = (int)(v % p);                  // C semantics: sign of the dividend
  if (r > (p - 1) / 2) r -= p;
  if (r < -(p / 2)) r += p;
  return r;
}
// the same residue with six FP64 operations instead of a 64-bit integer division: a - p rint(a / p) evaluated with FMAs
// (both remainders are small integers, hence exact); a is an integer-valued double with at most 53 significant bits
HD int i8_residue_fast(double a, int p) {
  const double dp = (double)p, ip = 1.0 / dp;
  const double r0 = fma(-dp, rint(a * ip), a);       // |r0| <= p (1/2 + 2^-52 |a| / p ... ) : a few hundred at most
  double r = fma(-dp, rint(r0 * ip), r0);            // in [-p/2, p/2]
  if (r > (double)((p - 1) / 2)) r -= dp;            // even p: +p/2 -> -p/2
  if (r < -(double)(p / 2)) r += dp;
  return (int)r;
}
// Barrett reduction of |s| < 2^27 modulo p in [173, 256] to the symmetric representative: no integer division.
// magic = ceil(2^36 / p), precomputed once per thread for the modulus of its CTA.
HD unsigned long long i8_barrett_magic(int p) { return ((1ull << 36) + (unsigned long long)p - 1) / (unsigned long long)p; }
HD int i8_reduce_sym(int s, int p, unsigned long long magic) {
  const unsigned long long u = (unsigned long long)((long long)s + ((long long)p << 19));   // >= 0, < 2^28
  const unsigned long long q = (u * magic) >> 36;
  int r = (int)(u - q * (unsigned long long)p);                  // in [-p, p): the rounded-up magic may overshoot by one
  if (r < 0) r += p;
  if (r > (p - 1) / 2) r -= p;
  return r;
}
HD int i8_sym(int r, int p) {            // symmetric representative of any int
  r %= p;
  if (r > (p - 1) / 2) r -= p;
  if (r < -(p / 2)) r += p;
  return r;
}

// scale exponent for a column with largest magnitude amax: trunc(a 2^e) has at most `bits` bits
HD int i8_scale_exponent(double amax, int bits) {
  if (!(amax > 0.0)) return 0;
  int ex;
  frexp(amax, &ex);                      // amax = f 2^ex, f in [0.5, 1)
  return bits - ex;                      // |a| 2^e < 2^bits
}

// residues of one complex entry: out[(t * 2 + part) * plane_stride] for part = 0 (re), 1 (im)
HD void i8_residues_entry(cplx x, int e, int n_mod, signed char* __restrict__ out, long long plane_stride) {
  // round to nearest: unbiased operand errors (truncation would bias e.g. the diagonal of a Gram matrix low)
  const double ar = rint(ldexp(x.x, e)), ai = rint(ldexp(x.y, e));
  for (int t = 0; t < n_mod; ++t) {
    const int p = i8_modulus(t);
    out[(long long)(2 * t) * plane_stride] = (signed char)i8_residue_fast(ar, p);
    out[(long long)(2 * t + 1) * plane_stride] = (signed char)i8_residue_fast(ai, p);
  }
}

// reference int8 dot products of the four real combinations for one (row of A^H, column of B), one modulus:
// returns (Ar.Br + Ai.Bi) mod p and (Ar.Bi - Ai.Br) mod p  == Re / Im of conj(a) . b;  K split so that int32 never overflows
HD void i8_dot_conj(const signed char* __restrict__ ar, const signed char* __restrict__ ai,
                    const signed char* __restrict__ br, const signed char* __restrict__ bi, long long K, int p, int* re, int* im) {
  int sre = 0, sim = 0;
  for (long long k0 = 0; k0 < K; k0 += I8_K_CHUNK) {
    const long long k1 = k0 + I8_K_CHUNK < K ? k0 + I8_K_CHUNK : K;
    int x1 = 0, x2 = 0, x3 = 0, x4 = 0;
    for (long long k = k0; k < k1; ++k) {
      x1 += (int)ar[k] * (int)br[k];
      x2 += (int)ai[k] * (int)bi[k];
      x3 += (int)ar[k] * (int)bi[k];
      x4 += (int)ai[k] * (int)br[k];
    }
    sre = (sre + x1 % p + x2 % p) % p;
    sim = (sim + x3 % p - x4 % p) % p;
  }
  *re = i8_sym(sre, p);
  *im = i8_sym(sim, p);
}

// same for a . b without conjugation (update-type products C = A B: rows of A against columns of B), strided operands:
// returns (Ar.Br - Ai.Bi) mod p and (Ar.Bi + Ai.Br) mod p
HD void i8_dot_plain(const signed char* __restrict__ ar, const signed char* __restrict__ ai, long long sa,
                     const signed char* __restrict__ br, const signed char* __restrict__ bi, long long sb, long long K, int p,
                     int* re, int* im) {
  int sre = 0, sim = 0;
  for (long long k0 = 0; k0 < K; k0 += I8_K_CHUNK) {
    const long long k1 = k0 + I8_K_CHUNK < K ? k0 + I8_K_CHUNK : K;
    int x1 = 0, x2 = 0, x3 = 0, x4 = 0;
    for (long long k = k0; k < k1; ++k) {
      x1 += (int)ar[k * sa] * (int)br[k * sb];
      x2 += (int)ai[k * sa] * (int)bi[k * sb];
      x3 += (int)ar[k * sa] * (int)bi[k * sb];
      x4 += (int)ai[k * sa] * (int)br[k * sb];
    }
    sre = (sre + x1 % p - x2 % p) % p;
    sim = (sim + x3 % p + x4 % p) % p;
  }
  *re = i8_sym(sre, p);
  *im = i8_sym(sim, p);
}

// CRT: residues r[t] (any representatives) of the integer C' (|C'| <= P/4)  ->  C' as a double (faithfully rounded)
HD double i8_crt(const int* __restrict__ r, const I8Tables& T) {
  const double B40 = 1099511627776.0;    // 2^40
  double S[I8_LIMBS + 1];
  for (int j = 0; j <= I8_LIMBS; ++j) S[j] = 0.0;
  // fully unrolled over the table of moduli: every p is a compile-time constant, so the remainders are multiply-shift
  // sequences instead of integer divisions
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (int t = 0; t < I8_MAX_MODULI; ++t) {
    if (t < T.n_mod) {
      const int p = i8_modulus(t);
      const int s = i8_sym(i8_sym(r[t], p) * T.q[t], p);          // |s| <= 128
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
      for (int j = 0; j < I8_LIMBS; ++j) S[j] += (double)s * T.w[t][j];   // |S_j| <= 20 * 128 * 2^40 < 2^52: exact
    }
  }
  // quotient estimate (|Q| <= 20 * 128 / 2; the FP64 Horner value is accurate to 2^-50 |V| << P / 4)
  double top = 0.0;
  for (int j = I8_LIMBS - 1; j >= 0; --j) top = top * B40 + S[j];
  const double Q = rint(top / T.P_top);
  for (int j = 0; j < I8_LIMBS; ++j) S[j] -= Q * T.P[j];         // exact: |Q P_j| < 2^51
  // carry normalisation to |limb| <= 2^39, then sum from the top (the leading limbs cancel exactly when |C'| << P)
  for (int j = 0; j < I8_LIMBS; ++j) {
    const double c = rint(S[j] / B40);
    S[j] -= c * B40;
    S[j + 1] += c;
  }
  double v = S[I8_LIMBS];
  for (int j = I8_LIMBS - 1; j >= 0; --j) v = v * B40 + S[j];
  return v;
}

}  // namespace dftk

// ------------------------------------------------------------------ host-only: table construction (small bigint)
#include <vector>
namespace dftk {
struct I8Big {                            // little-endian base 2^32
  std::vector<uint32_t> d;
  static I8Big one() { I8Big b; b.d = {1u}; return b; }
  void mul_small(uint32_t m) {
    uint64_t c = 0;
    for (auto& x : d) { uint64_t v = (uint64_t)x * m + c; x = (uint32_t)v; c = v >> 32; }
    if (c) d.push_back((uint32_t)c);
  }
  uint32_t divmod_small(uint32_t m) {     // in place, returns remainder
    uint64_t r = 0;
    for (size_t i = d.size(); i-- > 0;) { uint64_t v = (r << 32) | d[i]; d[i] = (uint32_t)(v / m); r = v % m; }
    while (d.size() > 1 && d.back() == 0) d.pop_back();
    return (uint32_t)r;
  }
  uint32_t mod_small(uint32_t m) const { I8Big c = *this; return c.divmod_small(m); }
  int bit_length() const {
    int n = (int)d.size() * 32;
    uint32_t top = d.back();
    for (int b = 31; b >= 0 && !((top >> b) & 1u); --b) --n;
    return n;
  }
  void limbs40(double* out, int n) const {
    for (int j = 0; j < n; ++j) {
      double v = 0.0;
      for (int b = 39; b >= 0; --b) {
        const int bit = 40 * j + b;
        const uint32_t w = (size_t)(bit / 32) < d.size() ? d[bit / 32] : 0u;
        v = 2.0 * v + (double)((w >> (bit % 32)) & 1u);
      }
      out[j] = v;
    }
  }
};

// number of moduli needed so that a contraction of length K with `bits` bits per operand fits: K 2^(2 bits) <= P / 4
inline I8Tables i8_make_tables(int n_mod, long long K) {
  I8Tables T{};
  T.n_mod = n_mod;
  I8Big P = I8Big::one();
  for (int t = 0; t < n_mod; ++t) P.mul_small((uint32_t)i8_modulus(t));
  int kbits = 0;
  while (((long long)1 << kbits) < K) ++kbits;
  T.bits = (P.bit_length() - 1 - 2 - kbits) / 2;       // 2^(bitlen-1) <= P
  if (T.bits > 61) T.bits = 61;
  P.limbs40(T.P, I8_LIMBS);
  T.P_top = 0.0;
  for (int j = I8_LIMBS - 1; j >= 0; --j) T.P_top = T.P_top * 1099511627776.0 + T.P[j];
  for (int t = 0; t < n_mod; ++t) {
    const uint32_t p = (uint32_t)i8_modulus(t);
    I8Big W = P;
    W.divmod_small(p);
    W.limbs40(T.w[t], I8_LIMBS);
    const uint32_t wm = W.mod_small(p);
    int inv = 0;
    for (uint32_t c = 1; c < p; ++c)
      if ((uint64_t)c * wm % p == 1) { inv = (int)c; break; }
    T.q[t] = inv;
  }
  return T;
}
}  // namespace dftk
