"""Build libdftk_b200.so in-tree for sm_90a (nvcc cross-compiles without a GPU)."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
SOURCES = ["fft.cu", "blas.cu", "lobpcg.cu", "api.cu", "xc.cu", "forces.cu", "setup.cu", "i8emu.cu", "i8tc2.cu", "dm.cu",
           "transfer.cu", "overlap.cu", "ldos.cu"]
REG_NGROUPS = 4
HEADERS = ["common.cuh", "structs.cuh", "fft_core.cuh", "fft_plan.h", "fft_reg.cuh", "fft_reg_fwd.cuh", "fft_reg.cu",
           "fft_radix_gen.cuh", "xc_core.cuh", "forces_core.cuh", "lobpcg_small.cuh", "lobpcg_batch.cuh", "i8emu_core.cuh", "dm_core.cuh", "transfer_core.cuh",
           "overlap_core.cuh", "ldos_core.cuh", "batch_exec.cuh",
           os.path.join("..", "..", "include", "dftk_b200.h")]
LIB = os.path.join(HERE, "..", "libdftk_b200.so")


def _nccl_dirs():
    import importlib.util
    spec = importlib.util.find_spec("nvidia.nccl")
    if spec and spec.submodule_search_locations:
        base = list(spec.submodule_search_locations)[0]
        return os.path.join(base, "include"), os.path.join(base, "lib")
    return "/usr/include", "/usr/lib/x86_64-linux-gnu"


def build(force=False, verbose=False):
    inc, libdir = _nccl_dirs()
    deps = [os.path.join(HERE, f) for f in SOURCES + HEADERS]
    newest = max(os.path.getmtime(d) for d in deps)
    lib = os.path.abspath(LIB)
    if not force and os.path.exists(lib) and os.path.getmtime(lib) >= newest:
        return lib
    flags = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
             "-Xcompiler", "-fPIC", "-I", inc, "-Wno-deprecated-gpu-targets"]
    if verbose:
        flags += ["-Xptxas", "-v"]
    objs = []

    def cc(src):
        extra = []
        if isinstance(src, tuple):           # (source, group) for the register-engine instantiation units
            src, grp = src
            obj = os.path.join(HERE, f"fft_reg_g{grp}.o")
            extra = [f"-DREG_GROUP={grp}", f"-DREG_NGROUPS={REG_NGROUPS}"]
        else:
            obj = os.path.join(HERE, src.replace(".cu", ".o"))
        cmd = ["nvcc"] + flags + extra + ["-c", os.path.join(HERE, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stderr}")
        if verbose:
            print(r.stderr)
        return obj

    with ThreadPoolExecutor(8) as ex:
        objs = list(ex.map(cc, SOURCES + [("fft_reg.cu", g) for g in range(REG_NGROUPS)]))
    nccl_so = os.path.join(libdir, "libnccl.so.2")
    link = ["g++", "-shared", "-o", lib] + objs + ["-L/usr/local/cuda/lib64", "-lcublas", "-lcusolver",
                                                    "-lcudart", f"-Wl,-rpath,{libdir}",
                                                    "-Wl,-rpath,/usr/local/cuda/lib64"]
    link += [f"-L{libdir}", "-l:libnccl.so.2"] if os.path.exists(nccl_so) else ["-lnccl"]
    r = subprocess.run(link, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stderr)
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
