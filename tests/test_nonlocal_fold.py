"""Time-reversal fold of the nonlocal projector products (blas.cu, kb_setup_fold / kb_apply_nonlocal_folded), checked
in NumPy on the oracle's projectors of Si2.

On a k-block whose sphere {q = k + G : |q|^2 / 2 <= Ecut} is closed under q -> -q (Γ and the other k with 2k in the
reciprocal lattice) the projectors satisfy P(-q) = conj(P(q)), and with a half set H (one q of each pair) and
R = [Re P(H); Im P(H)]:
    P'psi = R^T [s; u],  s = psi(q) + psi(-q),  u = i (psi(-q) - psi(q))     (s = psi(q), u = 0 where q = -q)
    P c   : [a; b] = R c,  Hpsi(q) += a + i b,  Hpsi(-q) += a - i b            (Hpsi(q) += a where q = -q)
The mirror map here follows the same rule as the library's sphere_mirror: G -> -G - m, m read off the bounding box."""
import numpy as np
import pytest

from oracle.basis import Element, Model, PlaneWaveBasis, G_axis
from oracle.terms import Terms, energy_hamiltonian, guess_density
from silicon import LATTICE, POSITIONS

KS = {"gamma": (0.0, 0.0, 0.0), "trim": (0.5, 0.0, 0.0), "generic": (0.1, -0.2, 0.3)}


@pytest.fixture(scope="module")
def blocks():
    m = Model(LATTICE, [Element("Si")] * 2, POSITIONS, functionals=("lda_x", "lda_c_vwn"), symmetries=False)
    b = PlaneWaveBasis(m, 15, fft_size=(27, 27, 27), kcoords=list(KS.values()), kweights=[1 / 3] * 3)
    _, ham = energy_hamiltonian(b, Terms(b), None, None, guess_density(b))
    return dict(zip(KS, ham)), b.fft_size


def sphere_mirror(fft_size, mapping):
    """Partner index of every sphere point under G -> -G - m, or None when that is not an involution of the sphere."""
    n = np.array(fft_size)
    lin = np.asarray(mapping)
    idx = np.stack([lin % n[0], (lin // n[0]) % n[1], lin // (n[0] * n[1])], axis=1)
    G = np.stack([G_axis(n[d])[idx[:, d]] for d in range(3)], axis=1)
    m = -(G.min(axis=0) + G.max(axis=0))
    Gm = -G - m
    c = Gm % n
    lin_m = c[:, 0] + n[0] * (c[:, 1] + n[1] * c[:, 2])
    slot = np.full(int(np.prod(n)), -1)
    slot[lin] = np.arange(len(lin))
    mir = slot[lin_m]
    if (mir < 0).any() or (mir[mir] != np.arange(len(lin))).any():
        return None
    return mir


def fold_products(P, mir, psi, c):
    """(P'psi, P c) through the folded real products."""
    H = np.nonzero(np.arange(len(mir)) <= mir)[0]
    p = mir[H]
    own = p == H
    R = np.concatenate([P[H].real, P[H].imag])                        # K' x n_proj
    s = psi[H] + np.where(own[:, None], 0, psi[p])
    u = np.where(own[:, None], 0, 1j * (psi[p] - psi[H]))
    gram = R.T @ np.concatenate([s, u])
    ab = R @ c
    a, b = ab[:len(H)], ab[len(H):]
    out = np.zeros((len(mir), c.shape[1]), dtype=complex)
    out[H] += np.where(own[:, None], a, a + 1j * b)
    out[p[~own]] += a[~own] - 1j * b[~own]
    return gram, out


@pytest.mark.parametrize("name", ["gamma", "trim"])
def test_fold_matches_complex_products(blocks, name):
    ham, fft_size = blocks
    blk = ham[name]
    P, D = blk.PD
    mir = sphere_mirror(fft_size, blk.kpt.mapping)
    assert mir is not None
    assert (mir[mir] == np.arange(len(mir))).all()
    # q(mir) = -q, so P(mir(q)) = conj(P(q))
    q = blk.kpt.G_vectors + blk.kpt.coordinate
    np.testing.assert_array_equal(q[mir], -q)
    assert np.abs(P[mir] - P.conj()).max() <= 1e-14 * np.abs(P).max()
    if name == "gamma":
        assert (mir == np.arange(len(mir))).sum() == 1                # G = 0 is its own partner
    rng = np.random.default_rng(0)
    nb = 5
    psi = rng.standard_normal((len(mir), nb)) + 1j * rng.standard_normal((len(mir), nb))
    c = rng.standard_normal((P.shape[1], nb)) + 1j * rng.standard_normal((P.shape[1], nb))
    gram, upd = fold_products(P, mir, psi, c)
    ref_gram, ref_upd = P.conj().T @ psi, P @ c
    assert np.abs(gram - ref_gram).max() <= 1e-14 * np.abs(ref_gram).max()
    assert np.abs(upd - ref_upd).max() <= 1e-14 * np.abs(ref_upd).max()
    # the whole nonlocal apply
    _, nl = fold_products(P, mir, psi, D @ fold_products(P, mir, psi, c)[0])
    ref = P @ (D @ (P.conj().T @ psi))
    assert np.abs(nl - ref).max() <= 1e-14 * np.abs(ref).max()


def test_generic_k_is_rejected(blocks):
    ham, fft_size = blocks
    assert sphere_mirror(fft_size, ham["generic"].kpt.mapping) is None


def test_random_projectors_fail_the_symmetry_check(blocks):
    ham, fft_size = blocks
    blk = ham["gamma"]
    mir = sphere_mirror(fft_size, blk.kpt.mapping)
    rng = np.random.default_rng(1)
    P = rng.standard_normal(blk.PD[0].shape) + 1j * rng.standard_normal(blk.PD[0].shape)
    assert np.abs(P[mir] - P.conj()).max() > 1e-12 * np.abs(P).max()
