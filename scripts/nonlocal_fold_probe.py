"""Development probe: the folded nonlocal apply Hpsi += P D P'psi at the benchmark shape (Γ block of the 128-atom Si
cell, 259 bands), kernel by kernel, against the complex products.

    python scripts/nonlocal_fold_probe.py [--rep 4] [--ecut 30] [--m 259] [--reps 10] [--out FILE.json]

Three forms of the same operator run in one process:
  folded   the block as the library builds it (Γ: fold, real-A Gram, reduce, D, real-A update, unfold)
  complex  the same block created with P e^{iπ/4}: P D P' is unchanged, but P(-q) = conj(P(q)) no longer holds, so the
           block keeps the complex DMMA products (k_zgemm_cn, k_zgemm_nn)
  cublas   gemm_backend 1 (cuBLAS ZGEMM) on the folded block
Per-kernel times come from torch.profiler in a separate pass; bytes and flops are what each step must move and compute.
The package is imported from PYTHONPATH first, so pointing PYTHONPATH at another checkout times that checkout."""
import argparse
import json
import os
import subprocess
import sys

sys.path.append(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import dftk_b200 as dftk  # noqa: E402

A_SI = 10.26 / 2
STEPS = ("k_fold", "k_rgemm_cn", "k_reduce_partials", "k_zgemm_nn", "k_rgemm_nn", "k_unfold_acc")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "nvidia-smi unavailable"


def timeit(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rep", type=int, default=4)
    ap.add_argument("--ecut", type=float, default=30.0)
    ap.add_argument("--m", type=int, default=259)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    lat = args.rep * np.array([[0, A_SI, A_SI], [A_SI, 0, A_SI], [A_SI, A_SI, 0]])
    r = args.rep
    pos = [(b + np.array([i, j, k])) / r for i in range(r) for j in range(r) for k in range(r)
           for b in (np.ones(3) / 8, -np.ones(3) / 8)]
    Si = dftk.ElementPsp("Si")
    model = dftk.model_DFT(lat, [Si] * len(pos), pos, functionals=dftk.LDA(), symmetries=False)
    basis = dftk.PlaneWaveBasis(model, Ecut=args.ecut, kgrid=dftk.ExplicitKpoints([[0.0, 0.0, 0.0]]))
    _, ham = dftk.energy_hamiltonian(basis, None, None, rho=dftk.guess_density(basis))
    kb = ham[0].bind()
    ctx = kb.ctx
    op = basis.term("AtomicNonlocal").ops[0]
    D = op.D.cpu().numpy() if torch.is_tensor(op.D) else np.asarray(op.D)
    kb_c = dftk.KBlock(basis.fft_grid, basis.kpoints[0].mapping.cpu().numpy(), P=op.P * complex(np.exp(0.25j * np.pi)), D=D)
    npw, npj, M = kb.n_pw, kb.n_proj, args.m
    kf = npw + 1 if npw % 2 else npw          # K' = 2 |H|; at Γ, G = 0 is its own partner
    g = torch.Generator(device=ctx.device).manual_seed(0)
    psi = torch.view_as_complex(torch.randn(M, npw, 2, generator=g, device=ctx.device, dtype=torch.float64))
    hpsi = torch.zeros_like(psi)

    def apply(block):
        return lambda: block.apply_terms(psi, 4, out=hpsi, accumulate=True)

    res = dict(gpu=gpu_info(), shape=dict(n_pw=npw, n_proj=npj, M=M, K_folded=kf), library=os.path.abspath(dftk.__file__))
    res["folded_ms"] = timeit(apply(kb), args.reps)
    res["complex_ms"] = timeit(apply(kb_c), args.reps)
    ctx.set_option("gemm_backend", 1)
    res["cublas_ms"] = timeit(apply(kb), args.reps)
    ctx.set_option("gemm_backend", 0)
    res["folded_over_complex"] = res["folded_ms"] / res["complex_ms"]
    res["folded_over_cublas"] = res["folded_ms"] / res["cublas_ms"]

    # one pass under the profiler: per-kernel device time of the folded apply
    fn = apply(kb)
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            fn()
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        for s in STEPS:
            if f"::{s}(" in e.key or f"::{s}<" in e.key:
                per[s] = per.get(s, 0.0) + e.device_time_total / 1e3 / args.reps
    need = {
        "k_fold": dict(bytes=16.0 * M * (npw + kf)),
        "k_rgemm_cn": dict(flop=4.0 * kf * npj * M, bytes=8.0 * kf * npj + 16.0 * kf * M),
        "k_reduce_partials": dict(),
        "k_zgemm_nn": dict(flop=8.0 * npj * npj * M),
        "k_rgemm_nn": dict(flop=4.0 * kf * npj * M, bytes=8.0 * kf * npj + 16.0 * kf * M),
        "k_unfold_acc": dict(bytes=16.0 * M * (kf + 2 * npw)),
    }
    steps = {}
    for s in STEPS:
        ms = per.get(s)
        row = dict(ms=None if ms is None else round(ms, 4), **need[s])
        if ms:
            if "flop" in need[s]:
                row["TFLOPs"] = round(need[s]["flop"] / ms / 1e9, 2)
            if "bytes" in need[s]:
                row["GBs"] = round(need[s]["bytes"] / ms / 1e6, 1)
        steps[s] = row
    res["steps"] = steps
    bw = [steps[s]["ms"] or 0.0 for s in ("k_fold", "k_unfold_acc")]
    res["fold_unfold_share_of_folded"] = sum(bw) / res["folded_ms"]
    res["device_memory_MB"] = dict(R=8.0 * kf * npj / 2**20, fold_ws=16.0 * kf * M / 2**20)
    print(json.dumps(res, indent=1), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
