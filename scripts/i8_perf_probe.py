"""Development probe: the INT8-residue emulation of C = A^H B (gemm_backend 4: wgmma s8 integer products)
against the FP64 DMMA kernel (backend 0) and cuBLAS (backend 1) at the C3 nonlocal shape  P^H psi
(K = 264 859, m = n_proj = 1250, n = 503 bands) and at the Gram shape (m = n = 1509)."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import dftk_b200

dev = torch.device("cuda:0")
ctx = dftk_b200.Context(0)
K = int(os.environ.get("K", 264859))
g = torch.Generator(device=dev).manual_seed(0)
res = {}


def timeit(fn, n=3, warm=1):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return min(ts)


SHAPES = (("nonlocal_PHpsi", 1250, 503),) if os.environ.get("ONLY_NONLOCAL") else (("nonlocal_PHpsi", 1250, 503), ("gram", 1509, 1509))
BACKENDS = tuple(int(b) for b in os.environ.get("BACKENDS", "0,1,4").split(","))
for name, m, n in SHAPES:
    decay = torch.exp(-torch.linspace(0, 20, K, dtype=torch.float64, device=dev))
    A = torch.view_as_complex(torch.randn(m, K, 2, generator=g, device=dev, dtype=torch.float64)) * decay.sqrt() / np.sqrt(K)
    B = torch.view_as_complex(torch.randn(n, K, 2, generator=g, device=dev, dtype=torch.float64)) * decay
    ref = torch.zeros((n, m), dtype=torch.complex128, device=dev)
    ctx.set_option("gemm_backend", 0)
    ctx.zgemm("C", A, B, ref)
    fl = 8.0 * K * m * n
    for backend in BACKENDS:
        ctx.set_option("gemm_backend", backend)
        C = torch.zeros_like(ref)
        try:
            t = timeit(lambda: ctx.zgemm("C", A, B, C), n=int(os.environ.get("REPS", 3)))
            err = float((C - ref).abs().max() / ref.abs().max())
            res[f"{name}_backend{backend}"] = dict(ms=t, TFLOPs_equiv=fl / t / 1e9, max_err_rel_to_max=err)
        except Exception as e:
            res[f"{name}_backend{backend}"] = dict(error=repr(e))
        finally:
            ctx.set_option("gemm_backend", 4)
        print(name, backend, res[f"{name}_backend{backend}"], flush=True)
    del A, B, ref, C
    torch.cuda.empty_cache()
os.makedirs("gpurun_out", exist_ok=True)
json.dump(res, open("gpurun_out/i8_perf_probe.json", "w"), indent=1)

# ---- the nonlocal term of a k-block (P' psi with cached residue planes of P under backend 4; P (D P'psi) stays on the DMMA kernel)
if os.environ.get("NONLOCAL_APPLY", "1") == "1":
    m, n = 1250, 503
    g = torch.Generator(device=dev).manual_seed(1)
    P = torch.view_as_complex(torch.randn(m, K, 2, generator=g, device=dev, dtype=torch.float64)) / np.sqrt(K)
    grid = dftk_b200.FFTGrid(ctx, (192, 192, 192), 1000.0)
    mapping = np.arange(K, dtype=np.int64)
    kb = dftk_b200.KBlock(grid, mapping, kin=np.ones(K), P=P, D=np.diag(np.linspace(0.5, 1.5, m)))
    psi = torch.view_as_complex(torch.randn(n, K, 2, generator=g, device=dev, dtype=torch.float64))
    outs = {}
    for backend in (0, 4):
        ctx.set_option("gemm_backend", backend)
        out = torch.zeros_like(psi)
        t = timeit(lambda: kb.apply_terms(psi, 4, out=out), n=3)
        outs[backend] = out.clone()
        res[f"nonlocal_apply_backend{backend}"] = dict(ms=t, TFLOPs_equiv=16.0 * K * m * n / t / 1e9)
        print("nonlocal apply", backend, res[f"nonlocal_apply_backend{backend}"], flush=True)
    ctx.set_option("gemm_backend", 4)
    print("nonlocal apply: max |difference| backend 4 vs 0:", float((outs[4] - outs[0]).abs().max() / outs[0].abs().max()))
    json.dump(res, open("gpurun_out/i8_perf_probe.json", "w"), indent=1)
