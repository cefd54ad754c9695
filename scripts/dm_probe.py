"""Time direct_minimization against the SCF on the device, and the fused two-loop pass against memory bandwidth.

For C2 (Si2 LDA, Ecut 30, 8x8x8 k-grid: many small blocks) and the benchmark's Si128 Γ cell (Ecut 30, 256 occupied
bands): the wall time per DM iteration (after the first, which carries one-time set-up) next to the time of one SCF step,
and the library launches per DM iteration.  On Si128: the time of dftk_b200_axpy_dot_multi (y += c x, then Re<z, y>,
the memory-bound core of the two-loop recursion) with CUDA events, against its byte count at the H100 SXM's 3.35 TB/s.
The card's name and power limit are read in the same run.

    python scripts/dm_probe.py [--iters 4] [--reps 20] [--skip-si128] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import dftk_b200 as dftk  # noqa: E402
from dftk_b200 import device as dev  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--iters", type=int, default=4)
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--skip-si128", action="store_true")
ap.add_argument("--out", default=None)
args = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("dm_probe: no CUDA device")

A_SI = 5.131570667152971
HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def silicon(rep):
    lat = rep * np.array([[0, A_SI, A_SI], [A_SI, 0, A_SI], [A_SI, A_SI, 0]])
    pos = [(b + np.array([i, j, k])) / rep for i in range(rep) for j in range(rep) for k in range(rep)
           for b in (np.ones(3) / 8, -np.ones(3) / 8)]
    Si = dftk.ElementPsp("Si")
    return dftk.model_DFT(lat, [Si] * len(pos), pos, functionals=dftk.LDA())


def measure(name, basis, scf_steps):
    ctx = basis.architecture.ctx
    out = dict(case=name, n_blocks=len(basis.kpoints), fft_size=list(basis.fft_size), n_G_max=max(k.n_G for k in basis.kpoints))
    steps = []
    dftk.self_consistent_field(basis, maxiter=scf_steps, callback=lambda info: steps.append(info["time_step"]))
    out["scf_step_s"] = steps[1:]
    stamps = []

    def cb(info):
        torch.cuda.synchronize()
        stamps.append((time.perf_counter(), ctx.launch_count()))
    never = lambda info: False
    torch.cuda.synchronize()
    dftk.direct_minimization(basis, maxiter=args.iters + 1, is_converged=never, callback=cb, seed=1)
    dt = [b[0] - a[0] for a, b in zip(stamps, stamps[1:])]
    dl = [b[1] - a[1] for a, b in zip(stamps, stamps[1:])]
    out["dm_iteration_s"] = dt
    out["dm_launches_per_iteration"] = dl
    print(f"{name}: {out['n_blocks']} blocks, fft {out['fft_size']}; SCF step {np.median(steps[1:]):.3f} s; "
          f"DM iteration {np.median(dt):.3f} s ({', '.join(f'{t:.3f}' for t in dt)}); launches per DM iteration {dl}",
          flush=True)
    return out


info = card()
print(f"card: {info}", flush=True)
results = []
model = silicon(1)
results.append(measure("C2 Si2 Ecut 30 k 8x8x8", dftk.PlaneWaveBasis(model, Ecut=30, kgrid=(8, 8, 8)), 4))
if not args.skip_si128:
    basis = dftk.PlaneWaveBasis(silicon(4), Ecut=30, kgrid=(1, 1, 1))
    results.append(measure("Si128 Gamma Ecut 30", basis, 3))
    kbs = basis.kblocks
    nb = 256
    Y, X, Z = (dev.random_orbitals_multi(kbs, nb, s) for s in (1, 2, 3))
    for _ in range(3):
        dev.axpy_dot_multi(kbs, Y, X, 1e-3, Z)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(args.reps):
        dev.axpy_dot_multi(kbs, Y, X, 1e-3, Z)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / args.reps
    nbytes = 4 * Y[0].numel() * 16            # read x, y, z, write y
    bound_ms = nbytes / HBM_BYTES_PER_S * 1e3
    results.append(dict(case="axpy_dot Si128", bytes=nbytes, ms=ms, bound_ms=bound_ms))
    print(f"fused two-loop pass (Si128, {nb} bands x {Y[0].shape[1]} G): {ms:.3f} ms per call, {nbytes / 1e9:.2f} GB, "
          f"{nbytes / ms / 1e6:.0f} GB/s = {bound_ms / ms:.0%} of 3.35 TB/s (includes the host synchronisation)", flush=True)
if args.out:
    with open(args.out, "w") as fh:
        json.dump(dict(card=info, results=results), fh, indent=1)
