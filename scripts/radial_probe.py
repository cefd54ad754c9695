"""Time the UPF form-factor build: every radial transform a basis needs (the projectors at each k-point's |G+k|, the
local potential and the core density on the FFT cube) with the device kernel (dftk_b200_radial_transform) and with the
host oracle (NumPy + scipy.special.spherical_jn) on the same distinct |q| values.  Shape: Al₄ fcc (cubic cell) with
Al_m.upf, Ecut 40, 12³ Monkhorst-Pack grid.  Prints one JSON line; writes nothing.

    python scripts/radial_probe.py [--reps 3]
"""
import argparse
import json
import lzma
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import dftk_b200 as dftk                                     # noqa: E402
from oracle import psp_upf                                   # noqa: E402


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = "unknown"
    return name, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--kgrid", type=int, default=12)
    ap.add_argument("--Ecut", type=float, default=40)
    args = ap.parse_args()
    path = os.path.join(ROOT, "tests", "golden", "upf", "Al_m.upf.xz")
    with lzma.open(path, "rt") as fh:
        psp = dftk.parse_upf(fh.read(), identifier="Al_m.upf")
    opsp = psp_upf.load(path)
    a = 7.65
    pos = [[0, 0, 0], [0, 0.5, 0.5], [0.5, 0, 0.5], [0.5, 0.5, 0]]
    Al = dftk.ElementPsp("Al", psp=psp)
    model = dftk.model_DFT(a * np.eye(3), [Al] * 4, pos, functionals=dftk.PBE(), temperature=0.01)
    basis = dftk.PlaneWaveBasis(model, Ecut=args.Ecut, kgrid=(args.kgrid,) * 3)
    qs = [basis.Gplusk_vectors_cart(k).norm(dim=1).contiguous() for k in basis.kpoints]
    cube = basis.G_vectors_cart.norm(dim=1).contiguous()

    def device_build():
        out = []
        for q in qs:
            out.append(psp.radial_transform("proj", q))
        out.append(psp.eval_psp_local_fourier(cube))
        out.append(psp.eval_psp_core_density_fourier(cube))
        return out

    device_build()                                            # warm-up: tables on the device, kernels loaded
    torch.cuda.synchronize()
    t_dev = []
    for _ in range(args.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        dev = device_build()
        e1.record()
        torch.cuda.synchronize()
        t_dev.append(e0.elapsed_time(e1) / 1e3)

    # host oracle on the same distinct values, with the same gather
    qs_h = [q.cpu().numpy() for q in qs]
    cube_h = cube.cpu().numpy()
    t0 = time.perf_counter()
    host = []
    for q in qs_h:
        u, inv = np.unique(q, return_inverse=True)
        rows = [opsp.eval_projector_fourier(i, l, u)[inv] for l in range(opsp.lmax + 1)
                for i in range(1, opsp.n_proj_radial(l) + 1)]
        host.append(np.array(rows))
    u, inv = np.unique(cube_h, return_inverse=True)
    host.append(opsp.eval_local_fourier(u)[inv])
    host.append(opsp.eval_core_density_fourier(u)[inv])
    t_host = time.perf_counter() - t0

    err = max(float(np.abs(d.cpu().numpy() - h).max() / np.abs(h).max()) for d, h in zip(dev, host))
    name, power = gpu_info()
    n_q = sum(len(torch.unique(q)) for q in qs) + len(torch.unique(cube))
    res = dict(gpu=name, power_limit=power, n_kpoints=len(qs), n_pw_max=max(len(q) for q in qs), fft_size=basis.fft_size,
               distinct_q=n_q, n_functions=sum(len(fl) for fl in psp.r2_projs) + 2,
               device_s=min(t_dev), device_s_all=t_dev, host_oracle_s=t_host, speedup=t_host / min(t_dev),
               max_rel_diff=err)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
