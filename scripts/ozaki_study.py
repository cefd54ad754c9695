"""Numerics study (CPU, NumPy): emulating the FP64 complex GEMMs of the nonlocal projector P'psi with INT8 products and
INT32 accumulation -- the arithmetic of the INT8 tensor-core MMAs (`wgmma` s8 -> s32 on sm_90a) -- so that the GEMM-shaped
half of H psi can move from the FP64 DMMA pipe to the INT8 tensor cores.  Two error-free schemes:

  I.  slicing (Ozaki 2012 / ozIMMU): row-scaled operands are cut into s slices of `bits` bits; all slice pairs with
      i + j < s are multiplied exactly in integers: s(s+1)/2 int8 GEMMs.
  II. modular (Ozaki-Uchino-Imamura 2025): operands are scaled to integer matrices, reduced modulo N pairwise coprime
      moduli <= 256, multiplied modulo each (N int8 GEMMs) and recombined by the Chinese remainder theorem.

Inputs are the real projector table P and orbitals of the oracle's silicon blocks (structure-factor phases, Gaussian
form factors, decaying orbital coefficients), i.e. the dynamic ranges the product sees.  Reference: exact rational
arithmetic on the FP64 inputs (Python integers).  Prints the relative error max|C - C_exact| / max|C_exact| next to
that of a plain FP64 GEMM, and the number of int8 GEMMs each setting costs.
"""
import math
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np


def real_form(Ac, Bc):
    """C = A^H B (complex) as one real GEMM: [Ar Ai]^T-style stacking; returns real A (2k x 2m... ) operands
    At (M x K) and B (K x N) with K = 2k such that At @ B = [Re C | Im C] blocks."""
    # C = (Ar - i Ai)^T (Br + i Bi) = (Ar^T Br + Ai^T Bi) + i (Ar^T Bi - Ai^T Br)
    Ar, Ai, Br, Bi = Ac.real, Ac.imag, Bc.real, Bc.imag
    At = np.concatenate([Ar.T, Ai.T], axis=1)                       # m x 2k
    B_re = np.concatenate([Br, Bi], axis=0)                         # 2k x n  -> Re C
    B_im = np.concatenate([Bi, -Br], axis=0)                        # 2k x n  -> Im C
    return At, np.concatenate([B_re, B_im], axis=1)                 # m x 2k, 2k x 2n


def exact_product(At, B):
    """Exact At @ B for FP64 inputs via Python integers (every double is m * 2^e)."""
    ma, ea = np.frexp(At)
    mb, eb = np.frexp(B)
    Ea, Eb = int(ea.min()) - 53, int(eb.min()) - 53
    Ia = np.vectorize(lambda m, e: int(m * 2 ** 53) << int(e - 53 - Ea), otypes=[object])(ma, ea)
    Ib = np.vectorize(lambda m, e: int(m * 2 ** 53) << int(e - 53 - Eb), otypes=[object])(mb, eb)
    C = Ia.dot(Ib)
    return C, Ea + Eb      # value = C * 2^(Ea+Eb)


def scheme_slices(At, B, s, bits):
    """Scheme I.  Rows of At / columns of B share one power-of-two scale; slice q holds bits [q*bits, (q+1)*bits)."""
    sa = 2.0 ** np.ceil(np.log2(np.abs(At).max(axis=1, keepdims=True)))      # |a| / sa < 1
    sb = 2.0 ** np.ceil(np.log2(np.abs(B).max(axis=0, keepdims=True)))
    ra, rb = At / sa, B / sb
    As, Bs = [], []
    for q in range(s):
        w = 2.0 ** (bits * (q + 1))
        ia, ib = np.trunc(ra * w), np.trunc(rb * w)                          # |i| < 2^bits
        As.append(ia.astype(np.int64))
        Bs.append(ib.astype(np.int64))
        ra, rb = ra - ia / w, rb - ib / w
    assert max(np.abs(a).max() for a in As) <= 2 ** bits and At.shape[1] * 4 ** bits < 2 ** 31
    C = np.zeros((At.shape[0], B.shape[1]))
    n_gemm = 0
    for i in range(s - 1, -1, -1):                                           # small terms first
        for j in range(s - 1 - i, -1, -1):
            C += (As[i] @ Bs[j]).astype(np.float64) * 2.0 ** (-bits * (i + j + 2))   # int32-exact accumulation
            n_gemm += 1
    return C * sa * sb, n_gemm


MODULI = [256, 255, 253, 251, 247, 241, 239, 233, 229, 227, 223, 217, 211, 199, 197, 193, 191, 181, 179, 173]


def scheme_modular(At, B, n_mod):
    """Scheme II.  Integer operands A' = round(mu A), B' = round(B nu) with k max|a'| max|b'| < P/2; residues in
    [-128, 127]; int32 accumulation over chunks of k <= 2^17; CRT recombination (Python integers here -- the device
    version uses 40-bit FP64 pieces, exact as well)."""
    p = MODULI[:n_mod]
    assert all(math.gcd(a, b) == 1 for i, a in enumerate(p) for b in p[i + 1:])
    P = math.prod(p)
    k = At.shape[1]
    budget = math.floor(math.log2(P // 2 // k) / 2)                           # bits per operand
    mu = 2.0 ** (budget - np.ceil(np.log2(np.abs(At).max(axis=1, keepdims=True))))
    nu = 2.0 ** (budget - np.ceil(np.log2(np.abs(B).max(axis=0, keepdims=True))))
    Ai, Bi = np.rint(At * mu), np.rint(B * nu)                                # exact integers held in FP64
    res = []
    for pt in p:
        a = np.fmod(Ai, pt); a = np.where(a > pt // 2 - (pt % 2 == 0), a - pt, a); a = np.where(a < -(pt // 2), a + pt, a)
        b = np.fmod(Bi, pt); b = np.where(b > pt // 2 - (pt % 2 == 0), b - pt, b); b = np.where(b < -(pt // 2), b + pt, b)
        a, b = a.astype(np.int64), b.astype(np.int64)
        assert a.min() >= -128 and a.max() <= 127 and b.min() >= -128 and b.max() <= 127
        c = np.zeros((At.shape[0], B.shape[1]), dtype=np.int64)
        for k0 in range(0, k, 1 << 17):
            part = a[:, k0:k0 + (1 << 17)] @ b[k0:k0 + (1 << 17)]
            assert np.abs(part).max() < 2 ** 31
            c = (c + part % pt) % pt
        res.append(c)
    # CRT: C' = sum_t r_t * (P/p_t) * inv(P/p_t mod p_t)  (mod P), symmetric representative
    Cp = np.zeros(res[0].shape, dtype=object)
    for pt, c in zip(p, res):
        W = P // pt
        q = pow(W % pt, -1, pt)
        Cp = Cp + np.vectorize(lambda x: (int(x) * q % pt) * W, otypes=[object])(c)
    Cp = np.vectorize(lambda x: ((x + P // 2) % P) - P // 2, otypes=[object])(Cp)
    C = np.vectorize(float, otypes=[float])(Cp) / mu / nu
    return C, n_mod, budget


def main():
    from oracle.basis import Element, Model, PlaneWaveBasis
    from oracle.terms import Terms, energy_hamiltonian, guess_density
    sys.argv = ["bench.py"]
    import bench
    rep = int(os.environ.get("REP", 2))
    lat, pos = bench.supercell(rep)
    m = Model(lat, [Element("Si")] * len(pos), pos, symmetries=False, terms=("Kinetic", "AtomicLocal", "AtomicNonlocal"))
    b = PlaneWaveBasis(m, float(os.environ.get("ECUT", 12)), kcoords=[[0, 0, 0]], kweights=[1.0])
    t = Terms(b)
    Pmat = t.PD[0][0]
    rng = np.random.default_rng(0)
    nb = 12
    psi = rng.standard_normal((Pmat.shape[0], nb)) + 1j * rng.standard_normal((Pmat.shape[0], nb))
    # orbital-like decay: weight by 1/(1 + kin)^2, then orthonormalise (what LOBPCG iterates look like)
    psi *= (1.0 / (1.0 + t.kin[0]) ** 2)[:, None]
    psi, _ = np.linalg.qr(psi)
    mcols = min(Pmat.shape[1], 24)
    At, B = real_form(Pmat[:, :mcols], psi)
    print(f"k = 2 n_pw = {At.shape[1]}, m = {At.shape[0]}, n = {B.shape[1]};  dynamic range of P rows "
          f"{np.abs(At).max() / np.abs(At[At != 0]).min():.1e}, of psi columns {np.abs(B).max() / np.abs(B[B != 0]).min():.1e}")
    t0 = time.time()
    Cx, ex = exact_product(At, B)
    Cref = np.array([[math.ldexp(int(c), ex) if abs(int(c)).bit_length() < 1000 else 0.0 for c in row] for row in Cx])
    print(f"exact reference in {time.time() - t0:.1f} s; max |C| = {np.abs(Cref).max():.3e}")
    scale = np.abs(Cref).max()
    print(f"{'plain FP64 GEMM (numpy)':44s} rel err {np.abs(At @ B - Cref).max() / scale:.2e}")
    for bits, s in ((6, 7), (6, 8), (6, 9), (6, 10), (6, 11)):
        C, ng = scheme_slices(At, B, s, bits)
        print(f"{'I  slices: ' + str(s) + ' x ' + str(bits) + ' bits':44s} rel err {np.abs(C - Cref).max() / scale:.2e}   int8 GEMMs {ng}")
    for nm in (12, 13, 14, 15, 16, 17, 18):
        C, ng, budget = scheme_modular(At, B, nm)
        print(f"{'II modular: ' + str(nm) + ' moduli (' + str(budget) + ' bits/operand)':44s} rel err {np.abs(C - Cref).max() / scale:.2e}   int8 GEMMs {ng}")


if __name__ == "__main__":
    main()
