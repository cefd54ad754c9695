"""Host emulation (tests/hostemu/emu_overlap.cu) of the batched overlap product of the Wannier interface (overlap_core.cuh):
C_p = A_p^H B_p[idx_p] over ragged row counts, n_a != n_b, -1 entries in idx and several pairs sharing one A, against NumPy;
two runs are bit-identical."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu_overlap") / "libemu_overlap.so")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-Wno-deprecated-gpu-targets",
                           "-o", so, os.path.join(HERE, "hostemu", "emu_overlap.cu")])
    lib = ctypes.CDLL(so)
    lib.emu_overlap.restype = ctypes.c_int
    return lib


def _run(lib, n_a, n_b, A, nG, B, idx, n_chunks):
    n = len(A)
    P = ctypes.c_void_p * n
    arr = lambda v: np.ascontiguousarray(v, dtype=np.int64)
    ld_a, ld_b, n_G = arr([a.shape[1] for a in A]), arr([b.shape[1] for b in B]), arr(nG)
    C = np.zeros((n, n_b, n_a), dtype=np.complex128)          # column-major n_a x n_b per pair
    idx_list = None if idx is None else P(*[None if i is None else i.ctypes.data for i in idx])
    groups = lib.emu_overlap(ctypes.c_int64(n), n_a, n_b, P(*[a.ctypes.data for a in A]), ld_a.ctypes.data_as(ctypes.c_void_p),
                             n_G.ctypes.data_as(ctypes.c_void_p), P(*[b.ctypes.data for b in B]),
                             ld_b.ctypes.data_as(ctypes.c_void_p), idx_list, n_chunks, C.ctypes.data_as(ctypes.c_void_p))
    return np.transpose(C, (0, 2, 1)), groups


def _reference(A, nG, B, idx):
    out = []
    for a, g, b, ix in zip(A, nG, B, idx if idx is not None else [None] * len(A)):
        if ix is None:
            ix = np.arange(g)
        bg = np.where(ix[None, :] >= 0, b[:, np.clip(ix, 0, None)], 0)
        out.append(a[:, :g].conj() @ bg.T)
    return out


def _block(rng, rows, cols):
    return np.ascontiguousarray(rng.standard_normal((rows, cols)) + 1j * rng.standard_normal((rows, cols)))


@pytest.mark.parametrize("n_a,n_b,n_chunks", [(4, 7, 1), (12, 12, 3), (32, 5, 2), (1, 32, 7), (32, 32, 4)])
def test_overlap_matches_numpy(emu, n_a, n_b, n_chunks):
    """Ragged n_G (1 .. 5000), row padding beyond n_G, -1 entries, an identity pair, and runs of pairs sharing their A."""
    rng = np.random.default_rng(n_a * 100 + n_b)
    sizes = [1, 5000, 63, 700, 129]
    As = [_block(rng, n_a, g + 3) for g in sizes]
    A, nG, B, idx = [], [], [], []
    for ia, (a, g) in enumerate(zip(As, sizes)):
        for q in range(3 if ia % 2 == 0 else 1):          # groups of 3, 1, 3, 1, 3 pairs
            ldb = g + int(rng.integers(0, 50))
            b = _block(rng, n_b, ldb)
            if ia == 3 and q == 0:
                ix = None                                  # identity
            else:
                ix = rng.integers(0, ldb, g).astype(np.int64)
                ix[rng.random(g) < 0.2] = -1
            A.append(a)
            nG.append(g)
            B.append(b)
            idx.append(ix)
    C, groups = _run(emu, n_a, n_b, A, nG, B, idx, n_chunks)
    assert groups == len(sizes)
    for c, r in zip(C, _reference(A, nG, B, idx)):
        np.testing.assert_allclose(c, r, rtol=0, atol=1e-13 * max(np.abs(r).max(), 1e-300))
    C2, _ = _run(emu, n_a, n_b, A, nG, B, idx, n_chunks)
    assert np.array_equal(np.ascontiguousarray(C).view(np.float64), np.ascontiguousarray(C2).view(np.float64))


def test_identity_list_and_empty_chunks(emu):
    """A NULL idx list is the identity; more chunks than rows leaves empty chunks that contribute zero."""
    rng = np.random.default_rng(3)
    A, B = [_block(rng, 6, 10)], [_block(rng, 9, 12)]
    C, _ = _run(emu, 6, 9, A, [10], B, None, 16)
    np.testing.assert_allclose(C[0], A[0].conj() @ B[0][:, :10].T, rtol=0, atol=1e-14)
    C, _ = _run(emu, 6, 9, A, [0], B, None, 2)
    assert not C.any()


def test_chunking_changes_only_rounding(emu):
    """The chunk count is the device's choice (it depends on the SM count); other counts agree to rounding."""
    rng = np.random.default_rng(11)
    A, B = [_block(rng, 12, 3000)] * 8, [_block(rng, 12, 3100) for _ in range(8)]
    idx = [rng.integers(-1, 3100, 3000).astype(np.int64) for _ in range(8)]
    ref = _reference(A, [3000] * 8, B, idx)
    for n_chunks in (1, 5, 47):
        C, groups = _run(emu, 12, 12, A, [3000] * 8, B, idx, n_chunks)
        assert groups == 1
        for c, r in zip(C, ref):
            np.testing.assert_allclose(c, r, rtol=0, atol=1e-13 * np.abs(r).max())
