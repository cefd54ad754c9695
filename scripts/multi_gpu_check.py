"""torchrun worker: (k, spin)-sharded SCF (one rank per GPU; per step one NCCL allgather of eigenvalues and one
allreduce of the density + packed energy sums) must reproduce the single-GPU SCF.  Launched by tests/test_gpu_multi.py,
by __graft_entry__.smoke() when >= 2 GPUs are visible, and usable standalone:
  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 scripts/multi_gpu_check.py
CASE=si (default; TEMPERATURE=0|0.01) or CASE=fe (collinear spin: spin x k blocks flattened over the ranks), or CASE=slab:
ONE k-point (Γ-only 3x3x3 Si supercell, 54 atoms, 111 bands) solved by all ranks together -- plane-wave slabs in the
eigensolver (dftk_b200_lobpcg_slab), band shares in compute_density -- against the single-GPU SCF."""
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

case = os.environ.get("CASE", "si")
temperature = float(os.environ.get("TEMPERATURE", "0.0"))
if case == "slab":
    a = 5.131570667152971
    rep3, Ecut, fft = 3, 12, 72
    unit = np.array([[0, a, a], [a, 0, a], [a, a, 0]])
    Si = dftk.ElementPsp("Si")
    pos = [(np.asarray(p) + np.array([i, j, k])) / rep3 for i in range(rep3) for j in range(rep3) for k in range(rep3)
           for p in (np.ones(3) / 8, -np.ones(3) / 8)]
    model = dftk.model_DFT(rep3 * unit, [Si] * len(pos), pos, functionals=dftk.LDA(), symmetries=False)
    comm = dftk.KpointComm.from_torch_distributed()
    i8_rows = int(os.environ.get("I8_MIN_ROWS", "32768"))
    basis = dftk.PlaneWaveBasis(model, Ecut=Ecut, kgrid=(1, 1, 1), fft_size=(fft,) * 3, comm_slab=comm)
    assert basis.architecture.device.index == local and len(basis.kpoints) == 1
    # I8_MIN_ROWS selects the INT8 tensor-core path (gemm_backend 4) for contractions of at least that many rows
    i8_backend = 4 if "I8_MIN_ROWS" in os.environ else 0
    basis.architecture.ctx.set_option("gemm_backend", i8_backend)
    basis.architecture.ctx.set_option("i8_min_rows", i8_rows)
    # eigensolver alone first: same start vectors, slab solve vs this rank's own single-GPU solve of the same block
    ham = dftk.energy_hamiltonian(basis, None, None, rho=dftk.guess_density(basis))[1]
    gen = torch.Generator(device=basis.architecture.device)
    gen.manual_seed(1234)
    X0 = dftk.random_orbitals(basis, basis.kpoints[0], 60, gen)
    r_slab = ham[0].bind().lobpcg_slab(X0.clone(), tol=1e-8, maxiter=200)
    r_one = ham[0].bind().lobpcg(X0.clone(), tol=1e-8, maxiter=200)
    HX = ham[0].mul(r_slab["X"])
    resid = float((HX - torch.as_tensor(r_slab["λ"], device=HX.device)[:, None] * r_slab["X"]).norm(dim=1).max())
    ortho = float((r_slab["X"].conj() @ r_slab["X"].T - torch.eye(60, device=HX.device)).abs().max())
    xs = r_slab["X"].contiguous()
    xg = [torch.empty_like(xs) for _ in range(world)]
    dist.all_gather(xg, xs)
    x_same = max(float((g - xs).abs().max()) for g in xg)
    c0 = comm.n_collectives
    res = dftk.self_consistent_field(basis, tol=1e-9)
    out = None
    if rank == 0:
        basis1 = dftk.PlaneWaveBasis(model, Ecut=Ecut, kgrid=(1, 1, 1), fft_size=(fft,) * 3, architecture=dftk.B200(local))
        basis1.architecture.ctx.set_option("gemm_backend", i8_backend)
        basis1.architecture.ctx.set_option("i8_min_rows", i8_rows)
        ref = dftk.self_consistent_field(basis1, tol=1e-9)
        nocc = 4 * len(pos) // 2
        out = dict(world=world, case=case, n_atoms=len(pos), n_pw=int(basis.kpoints[0].n_G),
                   lobpcg_dlambda=float(np.abs(r_slab["λ"] - r_one["λ"]).max()), lobpcg_resid=resid, lobpcg_ortho=ortho,
                   lobpcg_iters=[r_slab["n_iter"], r_one["n_iter"]], lobpcg_converged=[r_slab["converged"], r_one["converged"]],
                   x_identical_on_ranks=x_same, exchange_MB=r_slab["exchange_bytes"] / 1e6,
                   dE=abs(res["energies"].total - ref["energies"].total), E=res["energies"].total,
                   deig=float(np.abs(res["eigenvalues"][0][:nocc] - ref["eigenvalues"][0][:nocc]).max()),
                   drho=float((res["rho"] - ref["rho"]).norm()) * np.sqrt(basis.dvol),
                   n_iter=res["n_iter"], n_iter_ref=ref["n_iter"], converged=bool(res["converged"]),
                   collectives_per_step=(comm.n_collectives - c0) / res["n_iter"])
        print("MULTIGPU_RESULT " + json.dumps(out), flush=True)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0)
if case == "si":
    a = 5.131570667152971
    lat = np.array([[0, a, a], [a, 0, a], [a, a, 0]])
    Si = dftk.ElementPsp("Si")
    model = dftk.model_DFT(lat, [Si, Si], [np.ones(3) / 8, -np.ones(3) / 8], functionals=dftk.LDA(), temperature=temperature)
    Ecut, kgrid, tol = 10, (3, 3, 3), 1e-9
else:
    a = 2.71176
    lat = a * np.array([[-1, 1, 1], [1, -1, 1], [1, 1, -1]], dtype=float)
    Fe = dftk.ElementPsp("Fe", functional="pbe")
    model = dftk.model_DFT(lat, [Fe], [np.zeros(3)], functionals=dftk.PBE(), temperature=0.01, magnetic_moments=[4.0])
    Ecut, kgrid, tol = 15, (3, 3, 3), 1e-8
    temperature = 0.01
mixing = dftk.KerkerMixing() if temperature > 0 else None
comm = dftk.KpointComm.from_torch_distributed()
# default architecture: must land on this rank's GPU (LOCAL_RANK), not on cuda:0
basis = dftk.PlaneWaveBasis(model, Ecut=Ecut, kgrid=kgrid, comm_kpts=comm)
assert basis.architecture.device.index == local
c0 = comm.n_collectives
res = dftk.self_consistent_field(basis, tol=tol, mixing=mixing)
coll_per_step = (comm.n_collectives - c0) / res["n_iter"]
out = None
if rank == 0:
    arch1 = dftk.B200(local)
    basis1 = dftk.PlaneWaveBasis(model, Ecut=Ecut, kgrid=kgrid, architecture=arch1)
    ref = dftk.self_consistent_field(basis1, tol=tol, mixing=mixing)
    nocc = 4 if case == "si" else 8
    deig = max(np.abs(np.array(res["eigenvalues_global"][b][:nocc]) - ref["eigenvalues"][b][:nocc]).max()
               for b in range(len(basis1.kpoints)))
    drho = float((res["rho"] - ref["rho"]).norm()) * np.sqrt(basis.dvol)
    out = dict(world=world, case=case, dE=abs(res["energies"].total - ref["energies"].total), deig=float(deig), drho=drho,
               E=res["energies"].total, n_iter=res["n_iter"], n_iter_ref=ref["n_iter"], eF=res["eF"], eF_ref=ref["eF"],
               nk_local=len(basis.kpoints), nk_total=len(basis1.kpoints), n_spin=model.n_spin_components,
               spins_local=sorted({k.spin for k in basis.kpoints}), collectives_per_step=coll_per_step,
               n_atoms=len(model.atoms))
    print("MULTIGPU_RESULT " + json.dumps(out), flush=True)
dist.barrier()
dist.destroy_process_group()
