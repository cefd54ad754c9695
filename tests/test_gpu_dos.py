"""GPU tests of the densities of states (dos.py over dftk_b200_ldos_accumulate_multi): the LDOS of many energies from one
pass over the bands against a loop of single-energy density passes with the same weights, for every smearing and on a
spin-polarised metal; the single-energy case against the LdosMixing form; the sum rule against compute_dos; the PDOS
against the restatement of dos.jl, and Σ_p PDOS <= DOS where the weights are non-negative; two sharded ranks."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import dos_oracle as oracle
from silicon import LATTICE, POSITIONS
from upf_data import product_psp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = ["FermiDirac", "Gaussian", "MarzariVanderbilt", ("MethfesselPaxton", 1), ("MethfesselPaxton", 2)]
EPS = np.finfo(float).eps


@pytest.fixture(scope="module")
def si():
    """Si₂, symmetry-reduced 4³ k-grid, Gaussian smearing; a UPF pseudopotential, which carries the atomic orbitals of the
    PDOS."""
    import dftk_b200 as dftk
    Si = dftk.ElementPsp("Si", product_psp("Si.pbe-hgh.upf"))
    model = dftk.model_DFT(LATTICE, [Si, Si], POSITIONS, functionals=dftk.LDA(), temperature=5e-3, smearing="Gaussian")
    basis = dftk.PlaneWaveBasis(model, Ecut=10, kgrid=(4, 4, 4))
    assert len(basis.kpoints) < 64 and len(basis.symmetries) > 1
    return dftk.self_consistent_field(basis, tol=1e-8)


@pytest.fixture(scope="module")
def fe():
    import dftk_b200 as dftk
    Fe = dftk.ElementPsp("Fe", functional="pbe")
    lat = 2.71176 * np.array([[-1, 1, 1], [1, -1, 1], [1, 1, -1]], dtype=float)
    model = dftk.model_DFT(lat, [Fe], [[0, 0, 0]], functionals=dftk.PBE(), temperature=0.01, magnetic_moments=[4.0])
    basis = dftk.PlaneWaveBasis(model, Ecut=15, kgrid=(2, 2, 2))
    return dftk.self_consistent_field(basis, tol=1e-6)


def _energies(res, n):
    e = np.concatenate([np.asarray(x) for x in res["eigenvalues"]])
    return np.linspace(e.min() - 0.02, e.max() + 0.02, n)


def _density_loop(dftk, res, εs, kind, T):
    """One compute_density pass per energy, with the weights of the restatement (screened as compute_ldos screens)."""
    basis, filled = res["basis"], res["basis"].model.filled_occupation
    out = []
    for ε in εs:
        w = [np.array([oracle.ldos_weight(x, ε, filled, kind, T) for x in e[:p.shape[0]]])
             for e, p in zip(res["eigenvalues"], res["psi"])]
        out.append(dftk.compute_density(basis, res["psi"], w, occupation_threshold=EPS))
    return torch.stack(out)


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


@pytest.mark.parametrize("kind", KINDS, ids=str)
def test_many_energies_equal_density_loop(si, kind):
    import dftk_b200 as dftk
    εs = _energies(si, 9)
    T = 0.01
    ldos = dftk.compute_ldos(εs, si["basis"], si["eigenvalues"], si["psi"], smearing=kind, temperature=T)
    assert ldos.shape == (len(εs), 1, si["basis"].N)
    ref = _density_loop(dftk, si, εs, kind, T)
    assert _rel(ldos, ref) < 1e-12
    again = dftk.compute_ldos(εs, si["basis"], si["eigenvalues"], si["psi"], smearing=kind, temperature=T)
    assert torch.equal(ldos, again)                     # fixed-order sums: a rerun is bit-identical


def test_spin_polarised_iron(fe):
    import dftk_b200 as dftk
    εs = _energies(fe, 6)
    ldos = dftk.compute_ldos(εs, fe["basis"], fe["eigenvalues"], fe["psi"])
    assert ldos.shape == (len(εs), 2, fe["basis"].N)
    ref = _density_loop(dftk, fe, εs, fe["basis"].model.smearing, fe["basis"].model.temperature)
    assert _rel(ldos, ref) < 1e-12
    dos = dftk.compute_dos(εs, fe["basis"], fe["eigenvalues"])
    integral = (ldos.sum(dim=2) * fe["basis"].dvol).cpu().numpy()
    assert np.abs(integral - dos).max() < 1e-10 * max(1.0, np.abs(dos).max())
    assert np.abs(dos[:, 0] - dos[:, 1]).max() > 1e-3        # the two spin channels differ


def test_single_energy_equals_ldos_mixing_form(si):
    import dftk_b200 as dftk
    basis, T = si["basis"], 0.01
    old = dftk.compute_ldos(basis, si["eF"], si["eigenvalues"], si["psi"], temperature=T)
    one = dftk.compute_ldos(np.array([si["eF"]]), basis, si["eigenvalues"], si["psi"], smearing="Gaussian", temperature=T)
    assert _rel(one[0], old) < 1e-13
    scalar = dftk.compute_ldos(si, smearing="Gaussian", temperature=T)       # scfres form, ε = εF, one density pass
    assert scalar.shape == (1, basis.N) and _rel(scalar, old) < 1e-13


def test_sum_rule(si):
    import dftk_b200 as dftk
    εs = _energies(si, 40)
    for kind in ("Gaussian", ("MethfesselPaxton", 1)):
        ldos = dftk.compute_ldos(εs, si["basis"], si["eigenvalues"], si["psi"], smearing=kind)
        dos = dftk.compute_dos(εs, si["basis"], si["eigenvalues"], smearing=kind)
        integral = (ldos.sum(dim=2) * si["basis"].dvol).cpu().numpy()
        assert np.abs(integral - dos).max() < 1e-10 * max(1.0, np.abs(dos).max())


def test_pdos_matches_oracle_and_is_bounded_by_dos(si):
    import dftk_b200 as dftk
    basis = si["basis"]
    εs = _energies(si, 25)
    proj, labels = dftk.atomic_orbital_projections(basis, si["psi"])
    spins = [k.spin for k in basis.kpoints]
    for kind in ("FermiDirac", "Gaussian", ("MethfesselPaxton", 2)):
        res = dftk.compute_pdos(εs, basis, si["psi"], si["eigenvalues"], smearing=kind)
        assert res.pdos.shape == (len(εs), len(labels), 1) and len(res.projector_labels) == len(labels)
        ref = oracle.compute_pdos(εs, spins, basis.kweights, si["eigenvalues"], proj, 1, basis.model.filled_occupation, kind,
                                  basis.model.temperature)
        assert np.abs(res.pdos - ref).max() < 1e-12 * np.abs(ref).max()
        if kind in ("FermiDirac", "Gaussian"):      # non-negative weights, orthonormal projectors
            dos = dftk.compute_dos(εs, basis, si["eigenvalues"], smearing=kind)
            assert np.all(res.pdos.sum(axis=1) <= dos * (1 + 1e-12) + 1e-12)
            s = dftk.sum_pdos(res, [lambda o: True])
            np.testing.assert_allclose(s, res.pdos.sum(axis=1), rtol=1e-14)


def test_two_ranks_match_one_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29537",
                        os.path.join(ROOT, "scripts", "dos_multi_gpu_check.py")], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    out = json.loads([l for l in r.stdout.splitlines() if l.startswith("DOS_MULTIGPU ")][-1][len("DOS_MULTIGPU "):])
    assert out["nk_local"] < out["nk_total"]
    assert out["ldos"] < 1e-6 and out["dos"] < 1e-6 and out["pdos"] < 1e-6, out      # two SCFs converged to 1e-10
