"""Per-kernel times of the local + kinetic H apply at the benchmark shape (128-atom Si cell, Γ sphere at Ecut = 30 Ha,
150^3 grid, 259 bands), with the bytes each kernel must move per band computed from the shapes and the bandwidth that
implies.  On this shape the library runs the fused y-z path (kr_sphere_to_x, kr_yz_apply, kr_x_to_sphere); a library
without it runs the five-stage path through the W2 intermediate.  `--tree DIR` imports dftk_b200 from another checkout,
e.g. a build of an earlier commit, so that both paths can be timed by the same script.

    python scripts/yz_probe.py [--tree DIR] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ap = argparse.ArgumentParser()
ap.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--bands", type=int, default=259)
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--out", default=None)
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.tree))

import torch  # noqa: E402
import dftk_b200  # noqa: E402

n, M = 150, args.bands
A = 10.26 / 2
lattice = 4 * np.array([[0, A, A], [A, 0, A], [A, A, 0]])
recip = 2 * np.pi * np.linalg.inv(lattice).T
g = np.where(np.arange(n) <= (n - 1) // 2, np.arange(n), np.arange(n) - n)
gz, gy, gx = np.meshgrid(g, g, g, indexing="ij")
G = np.stack([gx, gy, gz], -1) @ recip.T
kin_all = ((G ** 2).sum(-1) / 2).reshape(-1)
mapping = np.flatnonzero(kin_all <= 30.0).astype(np.int64)
n_pw = mapping.size
n_cols = np.unique(mapping // n).size
n_zc = np.unique(mapping // (n * n)).size

dev = torch.device("cuda:0")
ctx = dftk_b200.Context(0)
grid = dftk_b200.FFTGrid(ctx, (n, n, n), abs(np.linalg.det(lattice)))
kb = dftk_b200.KBlock(grid, mapping, kin=kin_all[mapping])
gen = torch.Generator(device=dev).manual_seed(0)
kb.set_potential(torch.randn(n ** 3, generator=gen, device=dev, dtype=torch.float64))
psi = torch.view_as_complex(torch.randn(M, n_pw, 2, generator=gen, device=dev, dtype=torch.float64))
out = torch.empty_like(psi)

for _ in range(3):
    kb.apply_terms(psi, 3, out=out)
torch.cuda.synchronize()
ts = []
for _ in range(args.reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    kb.apply_terms(psi, 3, out=out)
    b.record()
    torch.cuda.synchronize()
    ts.append(a.elapsed_time(b))

from torch.profiler import ProfilerActivity, profile  # noqa: E402
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(args.reps):
        kb.apply_terms(psi, 3, out=out)
    torch.cuda.synchronize()
per_kernel = {}
for e in prof.key_averages():
    if e.device_type.name == "CUDA" and e.count:
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        per_kernel[e.key] = per_kernel.get(e.key, 0.0) + t / 1e3 / args.reps      # ms per apply

# bytes each kernel must move per band (the potential is left out: it is re-read by every band from L2)
c16, W1, W2 = 16, 16 * n_cols * n, 16 * n_zc * n * n
traffic = {"kr_sphere_to_x": c16 * n_pw + W1, "kr_y_backward": W1 + W2, "kr_z_apply": 2 * W2, "kr_y_forward": W2 + W1,
           "kr_yz_apply": 2 * W1, "kr_x_to_sphere": W1 + 3 * c16 * n_pw}
rows = []
for name, ms in sorted(per_kernel.items(), key=lambda kv: -kv[1]):
    short = next((k for k in traffic if k + "<" in name or name.endswith(k)), None)
    rec = dict(kernel=name[:90], ms_per_apply=round(ms, 4))
    if short:
        rec["bytes_per_band"] = traffic[short]
        rec["GB_per_s"] = round(traffic[short] * M / (ms * 1e-3) / 1e9, 1)
    rows.append(rec)
try:
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
except OSError:
    gpu = torch.cuda.get_device_name(0)
res = dict(gpu=gpu, tree=os.path.abspath(args.tree), n_pw=n_pw, n_cols=n_cols, n_zc=n_zc, bands=M,
           ms_local_kin_apply=dict(min=min(ts), median=float(np.median(ts)), max=max(ts)),
           MB_per_band=dict(W1=W1 / 1e6, W2=W2 / 1e6, psi=c16 * n_pw / 1e6), kernels=rows)
print(json.dumps(res, indent=1))
if args.out:
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
