"""Host emulation (tests/hostemu/emu_ldos.cu) of the LDOS product of many energies (ldos_core.cuh):
C[:, j] += Σ_k D_k W_k[j] against NumPy, on shapes that are not multiples of the tiles (energies, rows and bands), with
bands gathered from several blocks of one weight array and an output row stride of two spin channels."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu_ldos") / "libemu_ldos.so")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-Wno-deprecated-gpu-targets",
                           "-o", so, os.path.join(HERE, "hostemu", "emu_ldos.cu")])
    lib = ctypes.CDLL(so)
    lib.emu_ldos.restype = None
    lib.emu_ldos.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_longlong,
                             ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong]
    return lib


def _run(lib, D_rows, W, cols, C, n_spin, spin):
    """D_rows: K arrays of M doubles; W: (n_e, n_cols) array, band k uses column cols[k]; C: (n_e, n_spin, M)."""
    K = len(D_rows)
    n_e, ldw = W.shape
    M = C.shape[2]
    P = ctypes.c_void_p * max(K, 1)
    Dp = P(*[d.ctypes.data for d in D_rows])
    Wp = P(*[W.ctypes.data + 8 * c for c in cols])
    lib.emu_ldos(K, Dp, Wp, ldw, M, n_e, C.ctypes.data + 8 * spin * M, n_spin * M)


@pytest.mark.parametrize("n_e", [1, 7, 1000])
@pytest.mark.parametrize("K", [1, 13, 64])
def test_ldos_product_matches_numpy(emu, n_e, K):
    rng = np.random.default_rng(1000 * K + n_e)
    M = 517                                   # 4 row tiles of 128, the last one partial
    n_spin, spin = 2, 1
    # bands from three blocks of one weight array (n_e, 3, ld_w): the columns of a round are not contiguous
    ld_w = 40
    W = rng.standard_normal((n_e, 3 * ld_w))
    cols = [(k % 3) * ld_w + (k * 7) % ld_w for k in range(K)]
    D = [np.ascontiguousarray(rng.random(M)) for _ in range(K)]
    C0 = rng.standard_normal((n_e, n_spin, M))
    C = C0.copy()
    _run(emu, D, W, cols, C, n_spin, spin)
    ref = C0.copy()
    ref[:, spin, :] += W[:, cols] @ np.stack(D)
    np.testing.assert_array_equal(C[:, 0, :], C0[:, 0, :])          # the other spin channel is untouched
    scale = np.abs(W[:, cols]) @ np.abs(np.stack(D)) + np.abs(C0[:, spin, :])
    assert np.max(np.abs(C[:, spin, :] - ref[:, spin, :]) / scale) < 1e-13
    C2 = C0.copy()
    _run(emu, D, W, cols, C2, n_spin, spin)
    assert np.array_equal(C, C2)


def test_zero_bands_leave_output(emu):
    rng = np.random.default_rng(5)
    C0 = rng.standard_normal((3, 1, 129))
    C = C0.copy()
    _run(emu, [], np.zeros((3, 4)), [], C, 1, 0)
    assert np.array_equal(C, C0)
