"""Run with torch.distributed.run on >= 2 GPUs: a Γ-only silicon supercell with the BlowupCHV kinetic table, solved by
all ranks together (plane-wave slabs in the eigensolver, which read the slab rows of the k-block's kinetic table) against
a single-GPU solve of the same Hamiltonian.  Prints one line `SLAB_BLOWUP_RESULT {json}` on rank 0."""
import os
import sys
import json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
import dftk_b200 as dftk

a, rep = 5.131570667152971, 2
unit = np.array([[0, a, a], [a, 0, a], [a, a, 0]])
Si = dftk.ElementPsp("Si")
pos = [(np.asarray(p) + np.array([i, j, k])) / rep for i in range(rep) for j in range(rep) for k in range(rep)
       for p in (np.ones(3) / 8, -np.ones(3) / 8)]
model = dftk.model_DFT(rep * unit, [Si] * len(pos), pos, functionals=dftk.LDA(), symmetries=False,
                       kinetic_blowup=dftk.BlowupCHV())
comm = dftk.KpointComm.from_torch_distributed()
basis = dftk.PlaneWaveBasis(model, Ecut=10, kgrid=(1, 1, 1), comm_slab=comm)
ham = dftk.energy_hamiltonian(basis, None, None, rho=dftk.guess_density(basis))[1]
gen = torch.Generator(device=basis.architecture.device)
gen.manual_seed(1234)
X0 = dftk.random_orbitals(basis, basis.kpoints[0], 40, gen)
r_slab = ham[0].bind().lobpcg_slab(X0.clone(), tol=1e-8, maxiter=200)
r_one = ham[0].bind().lobpcg(X0.clone(), tol=1e-8, maxiter=200)
res = dftk.self_consistent_field(basis, tol=1e-9)
if rank == 0:
    basis1 = dftk.PlaneWaveBasis(model, Ecut=10, kgrid=(1, 1, 1), fft_size=basis.fft_size, architecture=dftk.B200(local))
    ref = dftk.self_consistent_field(basis1, tol=1e-9)
    print("SLAB_BLOWUP_RESULT " + json.dumps(dict(
        lobpcg_dlambda=float(np.abs(r_slab["λ"] - r_one["λ"]).max()),
        converged=[bool(r_slab["converged"]), bool(r_one["converged"]), bool(res["converged"])],
        dE=abs(res["energies"].total - ref["energies"].total), n_atoms=len(pos))), flush=True)
dist.barrier()
dist.destroy_process_group()
