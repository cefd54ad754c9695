"""Time dftk_b200_xc_evaluate on a 150^3 grid (3.375 M points, the benchmark's grid) with CUDA events, once per
functional set (LDA, PBE, PBEsol, Teter-Pade) and spin count, after a warm-up.  The card's name and power limit are
read in the same run and printed with the times.

    python scripts/xc_probe.py [--reps 20] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import dftk_b200  # noqa: E402
from dftk_b200 import xc as pxc  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=150)
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--out", default=None)
args = ap.parse_args()

if not torch.cuda.is_available():
    sys.exit("xc_probe: no CUDA device")
SETS = {"LDA": dftk_b200.LDA(), "PBE": dftk_b200.PBE(), "PBEsol": dftk_b200.PBEsol(), "Teter93": ["lda_xc_teter93"]}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def fields(n_spin, N, seed=0):
    """A positive density with a spread of magnitudes and polarisations, and a gradient at reduced gradient 0-3."""
    rng = np.random.default_rng(seed)
    n = 10.0 ** rng.uniform(-4, 0.5, N)
    z = rng.uniform(-0.9, 0.9, N)
    s = rng.uniform(0, 3, N)
    sig = s * s * 4 * (3 * np.pi ** 2) ** (2 / 3) * n ** (8 / 3)
    if n_spin == 1:
        rho, sigma = n[None], sig[None]
    else:
        rho = np.array([n * (1 + z) / 2, n * (1 - z) / 2])
        sigma = np.array([sig * (1 + z) ** 2 / 4, sig * (1 - z * z) / 4, sig * (1 - z) ** 2 / 4])
    return (torch.tensor(rho, device="cuda").contiguous(), torch.tensor(sigma, device="cuda").contiguous())


ctx = dftk_b200.Context(0)
N = args.n ** 3
info = card()
print(f"card: {info}")
results = []
for n_spin in (1, 2):
    rho, sigma = fields(n_spin, N)
    for name, funs in SETS.items():
        gga = any(f.startswith("gga") for f in funs)
        sg = sigma if gga else None
        for _ in range(3):
            pxc.evaluate(ctx, funs, rho, sg)
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.reps):
            pxc.evaluate(ctx, funs, rho, sg)
        t1.record()
        torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / args.reps
        results.append(dict(set=name, n_spin=n_spin, points=N, ms=ms, gpoints_per_s=N / ms / 1e6))
        print(f"{name:8s} n_spin {n_spin}: {ms:7.3f} ms per call ({N / ms / 1e6:6.2f} Gpoints/s)")
if args.out:
    with open(args.out, "w") as fh:
        json.dump(dict(card=info, results=results), fh, indent=1)
