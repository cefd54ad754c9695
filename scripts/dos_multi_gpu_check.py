"""torchrun worker: the densities of states of a (k, spin)-sharded SCF of spin-polarised iron (one rank per GPU; the blocks of
one spin may all sit on one rank) must reproduce those of the single-GPU SCF.  Launched by tests/test_gpu_dos.py:
  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 scripts/dos_multi_gpu_check.py
Prints DOS_MULTIGPU {json} on rank 0: the largest differences of LDOS, DOS and PDOS, relative to their largest values.
Both SCFs converge to 1e-10, so the results agree to the SCF tolerance, not to rounding."""
import json
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
import dftk_b200 as dftk

lat = 2.71176 * np.array([[-1, 1, 1], [1, -1, 1], [1, 1, -1]], dtype=float)
Fe = dftk.ElementPsp("Fe", functional="pbe")
model = dftk.model_DFT(lat, [Fe], [np.zeros(3)], functionals=dftk.PBE(), temperature=0.01, magnetic_moments=[4.0])
Ecut, kgrid, tol = 15, (2, 2, 2), 1e-10


def densities(res, εs):
    ldos = dftk.compute_ldos(εs, res["basis"], res["eigenvalues"], res["psi"]).cpu().numpy()
    dos = dftk.compute_dos(εs, res["basis"], res["eigenvalues"])
    pdos = dftk.compute_pdos(εs, res["basis"], res["psi"], res["eigenvalues"]).pdos
    return ldos, dos, pdos


comm = dftk.KpointComm.from_torch_distributed()
basis = dftk.PlaneWaveBasis(model, Ecut=Ecut, kgrid=kgrid, comm_kpts=comm)
res = dftk.self_consistent_field(basis, tol=tol, mixing=dftk.KerkerMixing())
εs = np.linspace(min(np.min(e) for e in res["eigenvalues_global"]), max(np.max(e) for e in res["eigenvalues_global"]), 31)
sharded = densities(res, εs)
if rank == 0:
    basis1 = dftk.PlaneWaveBasis(model, Ecut=Ecut, kgrid=kgrid, architecture=dftk.B200(local))
    ref = dftk.self_consistent_field(basis1, tol=tol, mixing=dftk.KerkerMixing())
    one = densities(ref, εs)
    rel = lambda a, b: float(np.abs(a - b).max() / np.abs(b).max())
    out = dict(world=world, nk_local=len(basis.kpoints), nk_total=len(basis1.kpoints),
               spins_local=sorted({k.spin for k in basis.kpoints}), ldos=rel(sharded[0], one[0]), dos=rel(sharded[1], one[1]),
               pdos=rel(sharded[2], one[2]))
    print("DOS_MULTIGPU " + json.dumps(out), flush=True)
dist.barrier()
dist.destroy_process_group()
