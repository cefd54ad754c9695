"""Host emulation (tests/hostemu/emu_dm.cu) of the deterministic reductions of the direct minimisation (dm_core.cuh): the
fused update y += c x followed by Re<z, y>, over blocks of ragged sizes, against NumPy and against the fixed summation
order written out in Python."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
THREADS, MAX_CHUNKS = 256, 1024


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu_dm") / "libemu_dm.so")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-Wno-deprecated-gpu-targets",
                           "-o", so, os.path.join(HERE, "hostemu", "emu_dm.cu")])
    lib = ctypes.CDLL(so)
    lib.emu_dm_axpy_dot.restype = ctypes.c_int
    return lib


def _run(lib, ys, xs, zs, c):
    n = len(ys)
    P = ctypes.c_void_p * n
    lens = np.array([y.size for y in ys], dtype=np.int64)
    ptr = lambda arrs: None if arrs is None else P(*[a.ctypes.data for a in arrs])
    out = ctypes.c_double()
    chunks = lib.emu_dm_axpy_dot(n, lens.ctypes.data_as(ctypes.c_void_p), ptr(ys), ptr(xs), ptr(zs), ctypes.c_double(c),
                                 ctypes.byref(out))
    return out.value, chunks


def _blocks(rng, sizes):
    return [(rng.standard_normal(s) + 1j * rng.standard_normal(s)).astype(np.complex128) for s in sizes]


@pytest.mark.parametrize("sizes", [[7], [300, 1, 257, 4096], [5000, 120, 260 * 1024 + 3]])
def test_axpy_dot_matches_numpy(emu, sizes):
    rng = np.random.default_rng(len(sizes))
    ys, xs, zs = _blocks(rng, sizes), _blocks(rng, sizes), _blocks(rng, sizes)
    y_ref = [y + 0.37 * x for y, x in zip(ys, xs)]
    d_ref = sum(float(np.real(np.vdot(z, y))) for z, y in zip(zs, y_ref))
    d, chunks = _run(emu, ys, xs, zs, 0.37)
    assert chunks == min(MAX_CHUNKS, -(-max(sizes) // THREADS))
    for y, r in zip(ys, y_ref):
        np.testing.assert_allclose(y, r, rtol=0, atol=1e-15 * np.abs(r).max())
    assert d == pytest.approx(d_ref, rel=1e-12)


def test_dot_alone_and_update_alone(emu):
    rng = np.random.default_rng(5)
    a, b = _blocks(rng, [1000, 33]), _blocks(rng, [1000, 33])
    b0 = [t.copy() for t in b]
    d, _ = _run(emu, b, None, a, 0.0)
    assert all(np.array_equal(t, t0) for t, t0 in zip(b, b0))
    assert d == pytest.approx(sum(float(np.real(np.vdot(x, y))) for x, y in zip(a, b)), rel=1e-13)
    d, _ = _run(emu, b, a, None, -1.0)
    assert d == 0.0
    for t, t0, x in zip(b, b0, a):
        np.testing.assert_allclose(t, t0 - x, atol=1e-15)


def test_reduction_order_is_fixed(emu):
    """Bit for bit the order of the device: per thread a strided sum, a pairwise tree over the CTA, then blocks and chunks
    in index order."""
    rng = np.random.default_rng(9)
    sizes = [700, 1300]
    zs, ys = _blocks(rng, sizes), _blocks(rng, sizes)
    d, chunks = _run(emu, ys, None, zs, 0.0)
    assert chunks == 6
    total = 0.0
    for z, y in zip(zs, ys):
        for ch in range(chunks):
            red = []
            for t in range(THREADS):
                s = 0.0
                for i in range(ch * THREADS + t, len(y), chunks * THREADS):
                    s += float(z[i].real) * float(y[i].real) + float(z[i].imag) * float(y[i].imag)
                red.append(s)
            w = THREADS // 2
            while w:
                for t in range(w):
                    red[t] += red[t + w]
                w //= 2
            total += red[0]
    assert d == total
    assert _run(emu, ys, None, zs, 0.0)[0] == d
