"""Architecture selector, the seam of src/architecture.jl:4-53 / ext/DFTKCUDAExt.jl.

`PlaneWaveBasis(model; architecture=B200())` places every hot-path array on the GPU and routes the
Hamiltonian apply, LOBPCG and compute_density through libdftk_b200.  There is no CPU architecture in
this package: the reference's own CPU path is the baseline we are compared with, not something we ship.
"""
import torch
from .device import Context


class AbstractArchitecture:
    pass


class CPU(AbstractArchitecture):
    def __init__(self):
        raise NotImplementedError("dftk_b200 is a GPU back end only; use DFTK.jl itself for CPU runs")


class B200(AbstractArchitecture):
    """GPU{B200Array} analogue.  One instance per process (= per GPU / rank)."""
    _contexts = {}

    def __init__(self, device=None, comm=None):
        if device is None:
            # one process per GPU: a multi-rank run must not pile every rank onto cuda:0
            if comm is not None and comm.nranks > 1:
                import os
                device = int(os.environ["LOCAL_RANK"]) if "LOCAL_RANK" in os.environ else torch.cuda.current_device()
            else:
                device = 0
        self.device_index = device
        self.comm = comm  # a dftk_b200.parallel.KpointComm or None
        dist = comm is not None and comm.nranks > 1
        key = (device, comm.rank, comm.nranks, comm.nccl_id) if dist else (device, 0, 1, None)
        if key not in B200._contexts:
            if dist:
                if comm.nccl_id is None:
                    raise ValueError("multi-rank KpointComm without an NCCL id (use KpointComm.from_torch_distributed())")
                B200._contexts[key] = Context(device, comm.nccl_id, comm.rank, comm.nranks)
            else:
                B200._contexts[key] = Context(device)
        self.ctx = B200._contexts[key]
        self.device = self.ctx.device
        if dist:
            comm.attach(self.ctx)

    # to_device / to_cpu / synchronize_device / memory_usage  (architecture.jl:18-48)
    def to_device(self, x):
        return x.to(self.device) if isinstance(x, torch.Tensor) else torch.as_tensor(x, device=self.device)

    @staticmethod
    def to_cpu(x):
        return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else x

    def synchronize_device(self):
        self.ctx.sync()

    def memory_usage(self):
        free, total = self.ctx.mem_info()
        return dict(used=total - free, total=total)
