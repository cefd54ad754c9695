"""Generates tests/golden/baseline_configs.json: converged SCF results of the CPU oracle (the restatement of the
reference's algorithm, pinned in tests/test_oracle_golden.py) for the BASELINE configurations at their FULL sizes:
  C1  Si2 LDA  Ecut 15  k 4x4x4          C2  Si2 LDA  Ecut 30  k 8x8x8
  C4  Al4 PBE  Ecut 40  k 12x12x12  T = 0.01 Ha Fermi-Dirac, Kerker mixing (SURVEY §8d)
  C5  Fe bcc PBE collinear spin  Ecut 45  k 8x8x8  T = 0.01 Ha, Kerker mixing
The GPU suite and bench.py compare the product's energies / eigenvalues / Fermi levels with these numbers at the
BASELINE tolerances (1e-8 Ha/atom, 1e-6 Ha).  CPU only, NumPy; usage:  python scripts/make_golden_configs.py [C1 C2 C4 C5]
Existing entries of the JSON are kept unless regenerated."""
import json
import os
import sys
import time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from oracle.basis import Element, Model, PlaneWaveBasis
from oracle import scf as oscf

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "baseline_configs.json")
A_SI = 5.131570667152971      # test/testcases.jl:12 (a = 10.263141334305942 bohr / 2)


def config(name):
    if name in ("C1", "C2"):
        lat = np.array([[0, A_SI, A_SI], [A_SI, 0, A_SI], [A_SI, A_SI, 0]])
        m = Model(lat, [Element("Si")] * 2, [np.ones(3) / 8, -np.ones(3) / 8], functionals=("lda_x", "lda_c_pw"))
        return m, dict(Ecut=15, kgrid=(4, 4, 4)) if name == "C1" else dict(Ecut=30, kgrid=(8, 8, 8)), "simple", 1e-10
    if name == "C4":
        a = 7.65339
        pos = [[0, 0, 0], [0, 0.5, 0.5], [0.5, 0, 0.5], [0.5, 0.5, 0]]
        m = Model(a * np.eye(3), [Element("Al", functional="pbe")] * 4, pos, functionals=("gga_x_pbe", "gga_c_pbe"),
                  temperature=0.01)
        return m, dict(Ecut=40, kgrid=(12, 12, 12)), "kerker", 1e-10
    if name == "C5":
        lat = 2.71176 * np.array([[-1, 1, 1], [1, -1, 1], [1, 1, -1]], dtype=float)
        m = Model(lat, [Element("Fe", functional="pbe")], [[0, 0, 0]], functionals=("gga_x_pbe", "gga_c_pbe"),
                  temperature=0.01, magnetic_moments=[4.0])
        return m, dict(Ecut=45, kgrid=(8, 8, 8)), "kerker", 1e-10
    raise KeyError(name)


def main():
    names = sys.argv[1:] or ["C1", "C2", "C5", "C4"]
    data = json.load(open(OUT)) if os.path.exists(OUT) else {}
    for name in names:
        m, bk, mixing, tol = config(name)
        t0 = time.time()
        b = PlaneWaveBasis(m, **bk)
        res = oscf.self_consistent_field(b, tol=tol, mixing=mixing)
        nk = len(b.kpoints)
        entry = dict(Ecut=bk["Ecut"], kgrid=list(bk["kgrid"]), fft_size=list(b.fft_size), n_blocks=nk, n_atoms=len(m.atoms),
                     temperature=m.temperature, mixing=mixing, tol=tol, converged=bool(res["converged"]), n_iter=res["n_iter"],
                     energies={k: float(v) for k, v in res["energies"].items()},
                     eF=float(res["eF"]),
                     kcoords=[k.coordinate.tolist() for k in b.kpoints], spins=[int(k.spin) for k in b.kpoints],
                     kweights=[float(w) for w in b.kweights],
                     n_bands_compared=int(min(len(e) for e in res["eigenvalues"])) - 3,
                     eigenvalues=[np.asarray(e).tolist() for e in res["eigenvalues"]],
                     rho_l2=float(np.linalg.norm(res["rho"]) * np.sqrt(b.dvol)),
                     oracle_seconds=time.time() - t0, host_cores=os.cpu_count())
        if m.magnetic_moments is not None and len(getattr(m, "magnetic_moments", ())) and res["rho"].shape[0] == 2:
            entry["magnetisation"] = float((res["rho"][0] - res["rho"][1]).sum() * b.dvol)
        data[name] = entry
        json.dump(data, open(OUT, "w"), indent=1)
        rho_path = OUT.replace("baseline_configs.json", "baseline_rho.npz")      # converged densities (density L2 parity, 1e-7)
        rhos = dict(np.load(rho_path)) if os.path.exists(rho_path) else {}
        rhos[name] = res["rho"]
        np.savez_compressed(rho_path, **rhos)
        print(name, "E =", entry["energies"]["total"], "eF =", entry["eF"], "n_iter", entry["n_iter"], f"{entry['oracle_seconds']:.1f} s",
              flush=True)


if __name__ == "__main__":
    main()
