"""torchrun worker: the (k, spin)-sharded SCF of a DFT+U model (Si2 with Si.pbe-hgh.upf, U on 3P, collinear spin, 3x3x3
k-points) must reproduce the single-GPU SCF in energy and Hubbard occupation.  The per-rank partial of the occupation
travels behind the density in the step's packed allreduce.  Launched by tests/test_gpu_hubbard.py when two GPUs are
visible, or standalone:
  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 scripts/hubbard_multi_gpu_check.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
import torch.distributed as dist

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
import dftk_b200 as dftk
from upf_data import product_psp

a = 5.131570667152971
lat = np.array([[0, a, a], [a, 0, a], [a, a, 0]])
Si = dftk.ElementPsp("Si", product_psp("Si.pbe-hgh.upf"))
hub = dftk.Hubbard((dftk.OrbitalManifold("Si", "3P"), 0.3))
model = dftk.model_DFT(lat, [Si, Si], [np.ones(3) / 8, -np.ones(3) / 8], functionals=dftk.LDA(), temperature=0.01,
                       smearing="Gaussian", magnetic_moments=[1.0, 1.0], extra_terms=[hub])
Ecut, kgrid, tol = 10, (3, 3, 3), 1e-10
comm = dftk.KpointComm.from_torch_distributed()
basis = dftk.PlaneWaveBasis(model, Ecut=Ecut, kgrid=kgrid, comm_kpts=comm)
assert basis.architecture.device.index == local
res = dftk.self_consistent_field(basis, tol=tol, seed=1)
if rank == 0:
    basis1 = dftk.PlaneWaveBasis(model, Ecut=Ecut, kgrid=kgrid, architecture=dftk.B200(local))
    ref = dftk.self_consistent_field(basis1, tol=tol, seed=1)
    out = dict(world=world, dE=abs(res["energies"].total - ref["energies"].total),
               dn=float(np.abs(res["hubbard_n"][0] - ref["hubbard_n"][0]).max()),
               E_hubbard=res["energies"]["Hubbard"], converged=[bool(res["converged"]), bool(ref["converged"])],
               nk_local=len(basis.kpoints), nk_total=len(basis1.kpoints))
    print("MULTIGPU_RESULT " + json.dumps(out), flush=True)
dist.barrier()
dist.destroy_process_group()
