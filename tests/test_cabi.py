"""CPU-side checks of the drop-in boundary: the shared library loads without a GPU, exports exactly the
symbols include/dftk_b200.h declares, and fails loudly (no CPU fallback) when there is no device."""
import ctypes
import os
import re
import subprocess
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    return g.build()


def _header_functions():
    text = open(os.path.join(ROOT, "include", "dftk_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(dftk_b200_[a-z_0-9]+)\s*\(", text)))


def test_header_symbols_exported(built):
    from dftk_b200 import _lib
    L = _lib.lib()
    names = _header_functions()
    assert len(names) >= 25
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/dftk_b200.h but not exported"
    assert sorted(_lib.SIGNATURES) == names, "ctypes signature table out of sync with the header"
    out = subprocess.check_output(["nm", "-D", "--defined-only", built], text=True)
    exported = sorted(set(re.findall(r"\bT (dftk_b200_[a-z_0-9]+)", out)))
    assert exported == names


def test_no_cpu_fallback(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from dftk_b200 import _lib
    L = _lib.lib()
    h = ctypes.c_void_p()
    rc = L.dftk_b200_ctx_create(0, ctypes.byref(h))
    assert rc < 0 and not h.value
    assert L.dftk_b200_last_error(None)
    import dftk_b200
    with pytest.raises(RuntimeError):
        dftk_b200.Context(0)


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "dftk.jl_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f
                assert "oracle/" not in src, f


def test_sm90a_code_and_dmma_in_library(built):
    out = subprocess.run(["cuobjdump", "-lelf", built], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    sass = subprocess.run(["cuobjdump", "-sass", "-fun", "_ZN4dftk10k_zgemm_cnILi2EEEvPK7double2lS3_lPS1_lllli", built],
                          capture_output=True, text=True).stdout
    assert "DMMA" in sass and "LDGSTS" in sass      # FP64 tensor-core MMA fed by cp.async staging
    # INT8 residue products: warpgroup MMAs (wgmma s8) fed by TMA
    sass = subprocess.run(["cuobjdump", "-sass", built], capture_output=True, text=True).stdout
    assert "IGMMA" in sass and "UTMALDG" in sass
    # register two-pass FFT stage for 192-point axes (the 192^3 grid of the 250-atom Si cell) is in the library
    elf = subprocess.run(["cuobjdump", "-elf", built], capture_output=True, text=True).stdout
    assert "kr_z_applyILi12ELi16E" in elf


def _build_c_smoke(built, tmpdir):
    exe = os.path.join(tmpdir, "c_smoke")
    libdir = os.path.dirname(built)
    subprocess.check_call(["gcc", "-O1", "-Wall", os.path.join(ROOT, "tests", "c_smoke.c"), "-I", os.path.join(ROOT, "include"),
                           "-L", libdir, "-l:libdftk_b200.so", f"-Wl,-rpath,{libdir}", "-lm", "-o", exe])
    return exe


def test_c_program_links_against_the_library(built, tmp_path):
    """A plain-C consumer (tests/c_smoke.c: no CUDA headers, no Python) compiles against include/dftk_b200.h and links the
    shared library; without a GPU it must report that and exit with the skip code, not crash."""
    import torch
    exe = _build_c_smoke(built, str(tmp_path))
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    if torch.cuda.is_available():
        assert r.returncode == 0, r.stdout + r.stderr
    else:
        assert r.returncode == 77 and "no sm_90 device" in r.stderr, (r.returncode, r.stderr)


@pytest.mark.gpu
def test_c_program_runs_h_apply_on_gpu(built, tmp_path):
    exe = _build_c_smoke(built, str(tmp_path))
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "max |H psi - (c + kin) psi|" in r.stdout
