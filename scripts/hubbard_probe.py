"""DFT+U cost on the benchmark's Si128 Γ cell (Si 4x4x4 supercell, 128 atoms, Ecut 30 Ha, 259 bands) with
Si.pbe-hgh.upf and U on 3P: 384 orbital columns beside the 640 atomic projector columns.

Times, with CUDA events after warm-up: a full-block Hψ with and without the orbital columns on the folded (Γ) and the
complex (k = [0.1, 0.1, 0.1]) products, the Löwdin setup of the orbital table, and one dftk_b200_orbital_occupation_multi.
Prints one JSON line, and writes it to OUT/hubbard_probe.json with --out OUT.

    python scripts/hubbard_probe.py [--rep 4] [--Ecut 30] [--steps 5] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np
import torch

import dftk_b200 as dftk
from upf_data import product_psp

A_SI = 5.131570667152971


def supercell(rep):
    lat = rep * np.array([[0, A_SI, A_SI], [A_SI, 0, A_SI], [A_SI, A_SI, 0]])
    pos = [(b + np.array([i, j, k])) / rep for i in range(rep) for j in range(rep) for k in range(rep)
           for b in (np.ones(3) / 8, -np.ones(3) / 8)]
    return lat, pos


def event_time(fn, steps, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rep", type=int, default=4)
    ap.add_argument("--Ecut", type=float, default=30.0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    lat, pos = supercell(args.rep)
    Si = dftk.ElementPsp("Si", product_psp("Si.pbe-hgh.upf"))
    n_atoms = len(pos)
    M = 2 * n_atoms + 3
    model = dftk.model_DFT(lat, [Si] * n_atoms, pos, functionals=dftk.LDA(), symmetries=False)
    basis = dftk.PlaneWaveBasis(model, Ecut=args.Ecut, kgrid=dftk.ExplicitKpoints([[0, 0, 0], [0.1, 0.1, 0.1]]))
    ctx = basis.architecture.ctx
    # the Löwdin setup of the complete orbital table (radial transform, build_projectors, S = Φ'Φ, eigh, Φ S^-1/2)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    hub = dftk.Hubbard((dftk.OrbitalManifold("Si", "3P"), 0.1))
    term = dftk.TermHubbard(basis, hub)      # the orbitals are attached to the k-blocks below, one block at a time
    torch.cuda.synchronize()
    t_setup = time.perf_counter() - t0
    n_orb = term.n_orb
    rho = dftk.guess_density(basis)
    n0 = [np.zeros((1, n_atoms, n_atoms, 3, 3), dtype=complex)]
    for i in range(n_atoms):
        n0[0][0, i, i] = np.diag([0.3, 0.4, 0.5])
    D, _ = term.coefficients(basis, n0)
    _, ham = dftk.energy_hamiltonian(basis, None, None, rho=rho)
    out = dict(gpu=gpu, n_atoms=n_atoms, bands=M, Ecut=args.Ecut, n_proj=int(basis.kblocks[0].n_proj), n_orb=n_orb,
               lowdin_setup_s=t_setup)
    g = torch.Generator(device=ctx.device).manual_seed(0)
    for ik, name in ((0, "folded_gamma"), (1, "complex_k")):
        kb = ham[ik].bind()
        psi = torch.randn((M, kb.n_pw), dtype=torch.complex128, device=ctx.device, generator=g)
        res = torch.empty_like(psi)
        kb.set_orbitals(None)
        t_without = event_time(lambda: kb.apply_h(psi, res), args.steps)
        nl_without = event_time(lambda: kb.apply_terms(psi, 4, res), args.steps)
        kb.set_orbitals(term.P_vec[ik])
        kb.set_orbital_coefficients(D[0])
        t_with = event_time(lambda: kb.apply_h(psi, res), args.steps)
        nl_with = event_time(lambda: kb.apply_terms(psi, 4, res), args.steps)
        out[name] = dict(n_pw=kb.n_pw, hpsi_without_s=t_without, hpsi_with_s=t_with, nonlocal_without_s=nl_without,
                         nonlocal_with_s=nl_with, nonlocal_ratio=nl_with / nl_without)
        if ik == 0:
            w = [np.full(M, 1.0)]
            out["orbital_occupation_multi_s"] = event_time(
                lambda: dftk.device.orbital_occupation_multi([kb], [psi], w, 1, n_orb), args.steps)
        kb.set_orbitals(None)
        del psi, res
        torch.cuda.empty_cache()
    s = json.dumps(out)
    print(s)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "hubbard_probe.json"), "w") as fh:
            fh.write(s + "\n")


if __name__ == "__main__":
    main()
