"""Timing of the LDOS at many energies on one GPU: compute_ldos over an energy array (one pass over the bands,
dftk_b200_ldos_accumulate_multi) against one compute_ldos call per energy (a full density pass each, what a plot of the
LDOS costs without it), alternated in the same run on the same card:

  si2     the examples/dos.jl shape: Si₂, LDA, Ecut 15, 4³ k-grid, Fermi-Dirac T = 5e-3, SCF to 1e-8, 1000 energies over the
          band range
  si128   the Γ block of the Si₁₂₈ supercell (4³ cells), Ecut 30, 259 bands, 100 energies over the band range.  Orbitals are
          seeded random orthonormal blocks and the eigenvalues evenly spaced: the cost does not depend on their values.

Times are host clocks around calls that end in a device synchronise (best of the alternated repeats).  The FP64 rate of the
product kernel (k_ldos_product) comes from a separate torch.profiler run: 2·N·n_ε·n_kept flop over its summed kernel time,
against the H100 SXM data-sheet FP64 tensor-core figure of 67 TFLOP/s.  The card's name and power limit are printed beside
the numbers.  `--out PATH` also writes the result as JSON."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import dftk_b200 as dftk  # noqa: E402
from dftk_b200.dos import dos_weights  # noqa: E402
from silicon import LATTICE, POSITIONS  # noqa: E402

PEAK_FP64_TC = 67e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                     text=True).strip()
    except Exception:
        pl = "unknown"
    return name, pl


def wall(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t, out


def setup(name):
    Si = dftk.ElementPsp("Si")
    if name == "si2":
        model = dftk.model_DFT(LATTICE, [Si, Si], POSITIONS, functionals=dftk.LDA(), temperature=5e-3)
        basis = dftk.PlaneWaveBasis(model, Ecut=15, kgrid=(4, 4, 4))
        res = dftk.self_consistent_field(basis, tol=1e-8)
        return basis, res["eigenvalues"], res["psi"], 1000
    rep = 4
    pos = [(np.asarray(p) + np.array([i, j, k])) / rep for i in range(rep) for j in range(rep) for k in range(rep)
           for p in POSITIONS]
    model = dftk.model_DFT(rep * LATTICE, [Si] * len(pos), pos, functionals=dftk.LDA(), temperature=5e-3, symmetries=False)
    basis = dftk.PlaneWaveBasis(model, Ecut=30, kgrid=(1, 1, 1))
    gen = torch.Generator(device=basis.architecture.device)
    gen.manual_seed(1234)
    psi = [dftk.random_orbitals(basis, basis.kpoints[0], 259, gen).contiguous()]
    return basis, [np.linspace(-0.2, 0.5, 259)], psi, 100


def case(name, repeats):
    basis, eig, psi, n_e = setup(name)
    e = np.concatenate(eig)
    εs = np.linspace(e.min(), e.max(), n_e)
    one_pass = lambda: dftk.compute_ldos(εs, basis, eig, psi)
    loop = lambda: torch.stack([dftk.compute_ldos(float(ε), basis, eig, psi) for ε in εs])
    one_pass(), loop()                                      # warm-up: scratch, plans, module loads
    t_one, t_loop = [], []
    for _ in range(repeats):                                # alternated
        t, a = wall(one_pass)
        t_one.append(t)
        t, b = wall(loop)
        t_loop.append(t)
    rel = float((a - b).abs().max() / b.abs().max())
    del a, b
    # product kernel time and FP64 rate, profiler on, in a run of its own
    W = dos_weights(basis, eig, εs, basis.model.smearing, basis.model.temperature)
    thr = np.finfo(float).eps
    n_kept = sum(int(np.any(np.abs(w[:, :p.shape[0]]) >= thr, axis=0).sum()) for w, p in zip(W, psi))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        one_pass()
        torch.cuda.synchronize()
    k_us = sum(ev.device_time_total for ev in prof.key_averages() if "k_ldos_product" in ev.key)
    flop = 2.0 * basis.N * n_e * n_kept
    rate = flop / (k_us * 1e-6) if k_us else float("nan")
    return dict(case=name, fft_size=list(basis.fft_size), N=basis.N, n_blocks=len(basis.kpoints),
                n_bands=[int(p.shape[0]) for p in psi][:4], n_kept_bands=n_kept, n_energies=n_e,
                one_pass_s=min(t_one), density_loop_s=min(t_loop), speedup=min(t_loop) / min(t_one),
                one_pass_all_s=t_one, density_loop_all_s=t_loop, max_rel_diff=rel,
                product_kernel_ms=k_us / 1e3, product_tflops=rate / 1e12, product_share_of_67=rate / PEAK_FP64_TC)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="si2,si128")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dos_probe needs a CUDA device")
    name, pl = card()
    rows = []
    for c in args.cases.split(","):
        r = case(c, args.repeats)
        r.update(card=name, power_limit=pl)
        print(json.dumps(r), flush=True)
        rows.append(r)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(rows, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
