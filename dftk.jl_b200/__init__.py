"""dftk_b200: H100-native (sm_90a) plane-wave Kohn-Sham SCF hot path behind DFTK.jl's operator API.

The package directory is `dftk.jl_b200/`; import it as `dftk_b200` (see dftk_b200.py at the repo root).
Names follow the reference (Model, PlaneWaveBasis, self_consistent_field, HamiltonianBlock, ...).
"""
import os as _os


def effective_cpus():
    """CPUs this process may actually use: min(affinity mask, cgroup v2/v1 CPU quota, os.cpu_count())."""
    n = _os.cpu_count() or 1
    try:
        n = min(n, len(_os.sched_getaffinity(0)))
    except Exception:
        pass
    try:
        q, p = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = min(n, max(1, int(int(q) / int(p))))
    except Exception:
        try:
            q = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            p = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if q > 0:
                n = min(n, max(1, q // p))
        except Exception:
            pass
    return n


# cuSOLVER's legacy dense routines have OpenMP host stages: an unset OMP_NUM_THREADS means one thread per *visible*
# core, which oversubscribes containers with a CPU quota by 8x (measured: Zheevd 10x slower; the Rayleigh-Ritz of
# LOBPCG now uses cusolverDnXsyevd, which does not depend on these settings, but potrf/trtri and NumPy still do).
# Spinning OpenMP workers (the libgomp default) fight the CUDA-synchronising host thread for a quota-limited CPU
# budget: measured 0.03 s (passive) vs 0.25-3.7 s (active) per 1509x1509 heevd.
_os.environ.setdefault("OMP_WAIT_POLICY", "passive")
if "OMP_NUM_THREADS" not in _os.environ:
    _os.environ["OMP_NUM_THREADS"] = str(max(1, min(16, effective_cpus() // max(1, int(_os.environ.get("LOCAL_WORLD_SIZE", "1"))))))


def _limit_openmp_team():
    """The variables above are read when libgomp is loaded -- which `import torch` already does (through libcusolver).
    If that happened before this package was imported, at least cap the team size through the runtime API (the wait
    policy cannot be changed any more: import dftk_b200, or set OMP_WAIT_POLICY=passive, before torch for large
    eigenproblems)."""
    try:
        import ctypes
        g = ctypes.CDLL("libgomp.so.1")
        want = int(_os.environ["OMP_NUM_THREADS"].split(",")[0])
        if g.omp_get_max_threads() > want:
            g.omp_set_num_threads(want)
    except Exception:
        pass


_limit_openmp_team()

from . import _lib
from ._lib import DftkB200Error, LIB_PATH
from .device import Context, FFTGrid, KBlock
from .architecture import B200, CPU
from .pseudo import PspHgh, PspUpf, ElementPsp, load_psp, parse_hgh, parse_upf
from .model import Model, model_DFT, model_atomic, LDA, PBE, PBEsol, SymOp, symmetry_operations
from .parallel import KpointComm, split_evenly
from .basis import PlaneWaveBasis, MonkhorstPack, ExplicitKpoints, Kpoint, compute_fft_size
from .terms import (guess_density, Kinetic, BlowupIdentity, BlowupCHV, BlowupAbinit, smearing_occupation,
                    smearing_entropy, occupation_derivative)
from .hamiltonian import Hamiltonian, DftHamiltonianBlock, energy_hamiltonian, energy, Energies
from .eigen import lobpcg_hyper, diagonalize_all_kblocks, random_orbitals
from .occupation import compute_occupation, FermiBisection, FermiTwoStage, default_fermialg
from .densities import compute_density, symmetrize_rho
from .forces import (compute_forces, compute_forces_cart, symmetrize_forces, energy_forces_ewald,
                     energy_forces_ewald_device)
from .hubbard import (OrbitalManifold, Hubbard, TermHubbard, atomic_orbital_projectors, atomic_orbital_projections,
                      compute_hubbard_n, symmetrize_hubbard_n, wigner_d_matrix, resolve_hubbard_manifold)
from .scf import (self_consistent_field, next_density, AdaptiveBands, FixedBands, AdaptiveDiagtol,
                  ScfConvergenceDensity, ScfConvergenceEnergy, SimpleMixing, KerkerMixing, LdosMixing,
                  AndersonAcceleration, ScfDefaultCallback)
from .direct_minimization import direct_minimization, select_occupied_orbitals
from .transfer import (transfer_mapping, transfer_blochwave_kpt, transfer_blochwave, transfer_density, interpolate_density,
                       apply_symop, unfold_bz, create_supercell, cell_to_supercell)
from .wannier import (GaussianWannierProjection, HydrogenicWannierProjection, default_wannier_centers, overlap_Mmn_k_kpb,
                      compute_amn_kpoint, write_w90_win, read_w90_nnkp, write_w90_eig, write_w90_unk, write_w90_mmn,
                      write_w90_amn, write_wannier90_files, run_wannier90)
from .dos import compute_dos, compute_ldos, compute_pdos, sum_pdos, PdosResult
