"""Host emulation (tests/hostemu/emu_yz.cu) of the fused y-z stage of the local H apply (reg_yz_apply, fft_reg.cuh) with
the x stages on the x-major W1 layout, for every factor pair of the register engine on (18, n, n) boxes, against the
direct DFT of fft_reference.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import fft_reference as fr

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "hostemu", "libhostemu_yz.so")
NX = 18


@pytest.fixture(scope="module")
def emu():
    src = os.path.join(HERE, "hostemu", "emu_yz.cu")
    csrc = os.path.join(HERE, "..", "dftk.jl_b200", "csrc")
    deps = [src, os.path.join(HERE, "hostemu", "emu.cu")] + [os.path.join(csrc, f) for f in os.listdir(csrc)
                                                             if f.endswith((".cuh", ".h"))]
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC",
                               "-Wno-deprecated-gpu-targets", "-o", SO, src])
    return ctypes.CDLL(SO)


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _run(lib, shape, mapping, psi, V, kin, out0):
    nx, ny, nz = shape
    N = nx * ny * nz
    Vt = np.ascontiguousarray(V.reshape(nz, ny, nx).transpose(2, 1, 0) / N)      # [x][y][z], scaled by 1/N
    out = np.full_like(psi, np.nan)
    rc = lib.emur_apply_local_yz(nx, ny, nz, ctypes.c_int64(mapping.size), _p(mapping), _p(psi), psi.shape[0], _p(Vt),
                                 _p(kin) if kin is not None else None, _p(out0) if out0 is not None else None, _p(out))
    assert rc == 0
    return out


@pytest.mark.parametrize("frac", [fr.HALF, fr.FULL, 0], ids=["half", "full", "point"])
@pytest.mark.parametrize("n", [a * b for a, b in fr.reg_pairs()])
def test_emulated_yz_fused_every_pair(emu, n, frac):
    shape = (NX, n, n)
    N = NX * n * n
    mapping = fr.ellipsoid_mapping(shape, frac)
    assert frac != fr.FULL or mapping.size == N
    assert emu.emur_ranges_ok(NX, n, n, ctypes.c_int64(mapping.size), _p(mapping)) == 1
    rng = np.random.default_rng(n)
    nb = 2
    psi = rng.standard_normal((nb, mapping.size)) + 1j * rng.standard_normal((nb, mapping.size))
    V = rng.standard_normal(N) + 0.5              # nonzero mean: the one-point result is mean(V) psi
    kin = rng.random(mapping.size)
    out0 = rng.standard_normal((nb, mapping.size)) + 1j * rng.standard_normal((nb, mapping.size))
    loc = fr.local_apply(psi, mapping, shape, V)

    def check(got, ref):
        assert np.abs(got - ref).max() <= 1e-13 * np.abs(ref).max()
    check(_run(emu, shape, mapping, psi, V, None, None), loc)
    check(_run(emu, shape, mapping, psi, V, kin, None), loc + kin * psi)
    check(_run(emu, shape, mapping, psi, V, kin, out0), out0 + loc + kin * psi)
