"""Development probe: section timing of one LOBPCG solve at the benchmark shape (DFTK_B200_PROFILE=1)."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["DFTK_B200_PROFILE"] = "1"
import numpy as np
import torch
sys.argv = ["bench.py"]
import bench
import dftk_b200 as dftk

lat, pos = bench.supercell(int(os.environ.get("REP", 4)))
Si = dftk.ElementPsp("Si")
model = dftk.model_DFT(lat, [Si] * len(pos), pos, functionals=dftk.LDA(), symmetries=False)
basis = dftk.PlaneWaveBasis(model, Ecut=30.0, kgrid=dftk.ExplicitKpoints([[0, 0, 0]]))
_, ham = dftk.energy_hamiltonian(basis, None, None, rho=dftk.guess_density(basis))
kb = ham[0].bind()
M = bench.n_bands_for(len(pos))
X0 = dftk.random_orbitals(basis, basis.kpoints[0], M)
ctx = basis.architecture.ctx
lams = {}
for backend in [int(b) for b in os.environ.get("BACKENDS", "0").split(",")]:
    ctx.set_option("gemm_backend", backend)
    X = X0.clone()
    kb.lobpcg(X.clone(), tol=1.0, maxiter=1, n_conv_check=M - 3)      # warm workspaces / cached planes
    torch.cuda.synchronize()
    t = time.perf_counter()
    res = kb.lobpcg(X, tol=float(os.environ.get("TOL", 0.025)), maxiter=int(os.environ.get("MAXITER", 8)), n_conv_check=M - 3)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t
    lams[backend] = res["λ"]
    print("gemm_backend", backend, "lobpcg", dt, "s", res["n_iter"], "iterations ->", dt / max(1, res["n_iter"]), "s/iteration", res["n_matvec"],
          res["converged"], "max resid", float(np.max(res["residual_norms"][:M - 3])), flush=True)
ctx.set_option("gemm_backend", 0)
if len(lams) > 1:
    ks = sorted(lams)
    print("max |eigenvalue difference| between backends", ks, ":", float(np.abs(lams[ks[0]] - lams[ks[-1]]).max()))
