"""Model / model_DFT / model_atomic (host-side mirror of src/Model.jl:128-219 and
src/standard_models.jl:45-134).  Pure setup: small NumPy arrays only."""
import itertools
import math
import numpy as np

SYMMETRY_TOLERANCE = 1e-5


class SymOp:
    """src/SymOp.jl: x -> W x + w in reduced coordinates; reciprocal S = W', tau = -W^-1 w."""

    def __init__(self, W, w):
        self.W = np.array(np.rint(W), dtype=np.int64)
        self.w = np.array(w, dtype=float)
        self.S = self.W.T.copy()
        self.tau = -np.linalg.solve(self.W.astype(float), self.w)

    def isone(self):
        return np.array_equal(self.W, np.eye(3, dtype=np.int64)) and not np.any(np.abs(self.w) > 1e-12)


def symmetry_operations(lattice, labels, positions, tol=SYMMETRY_TOLERANCE):
    """Space-group operations of the decorated lattice by exhaustive search over unimodular integer
    matrices (replaces the spglib call of src/symmetry.jl:91-120; spglib is not available here)."""
    metric = lattice.T @ lattice
    scale = np.max(np.abs(metric))
    pos = [np.asarray(p, dtype=float) for p in positions]
    rots = []
    for e in itertools.product((-1, 0, 1), repeat=9):
        W = np.array(e, dtype=np.int64).reshape(3, 3)
        if abs(round(float(np.linalg.det(W)))) == 1 and np.allclose(W.T @ metric @ W, metric, atol=tol * scale):
            rots.append(W)
    ops = []

    def same(a, b):
        d = a - b
        return np.max(np.abs(d - np.round(d))) < tol

    for W in rots:
        seen = []
        for j, pj in enumerate(pos):
            if labels[j] != labels[0]:
                continue
            w = pj - W @ pos[0]
            w -= np.round(w)
            if any(same(w, s) for s in seen):
                continue
            if all(any(labels[a] == labels[b] and same(W @ pa + w, pb) for b, pb in enumerate(pos))
                   for a, pa in enumerate(pos)):
                seen.append(w)
                ops.append(SymOp(W, np.where(np.abs(w) < tol, 0.0, w)))
    ops.sort(key=lambda o: not o.isone())
    return ops


def LDA():
    return ["lda_x", "lda_c_pw"]       # standard_models.jl:220


def PBE():
    return ["gga_x_pbe", "gga_c_pbe"]  # standard_models.jl:224


def PBEsol():
    return ["gga_x_pbe_sol", "gga_c_pbe_sol"]  # standard_models.jl:234


def _check_smearing(smearing):
    """Smearing.jl: "None", "FermiDirac", "Gaussian", "MarzariVanderbilt" or ("MethfesselPaxton", order >= 0)."""
    if isinstance(smearing, (tuple, list)) and len(smearing) == 2 and smearing[0] == "MethfesselPaxton":
        order = smearing[1]
        if isinstance(order, (bool, np.bool_)) or not isinstance(order, (int, np.integer)) or order < 0:
            raise ValueError(f"Methfessel-Paxton order must be a non-negative integer, got {order!r}")
        return ("MethfesselPaxton", int(order))
    if isinstance(smearing, str) and smearing in ("None", "FermiDirac", "Gaussian", "MarzariVanderbilt"):
        return smearing
    raise NotImplementedError(f"smearing {smearing!r}: only 'None', 'FermiDirac', 'Gaussian', 'MarzariVanderbilt' and "
                              "('MethfesselPaxton', order) are supported")


class Model:
    def __init__(self, lattice, atoms=(), positions=(), *, model_name="custom", n_electrons=None,
                 magnetic_moments=(), terms=("Kinetic",), functionals=(), temperature=0.0, smearing=None,
                 spin_polarization=None, symmetries=True):
        self.model_name = model_name
        self.lattice = np.array(lattice, dtype=float)
        if len(atoms) != len(positions):
            raise ValueError("Length of atoms and positions vectors need to agree.")
        if not terms:
            raise ValueError("Model without terms not supported.")
        self.atoms = list(atoms)
        self.positions = [np.array(p, dtype=float) for p in positions]
        self.recip_lattice = 2 * math.pi * np.linalg.inv(self.lattice.T)
        self.inv_lattice = np.linalg.inv(self.lattice)
        self.unit_cell_volume = abs(float(np.linalg.det(self.lattice)))
        self.n_electrons = int(sum(a.n_elec_valence() for a in self.atoms)) if n_electrons is None else int(n_electrons)
        if self.n_electrons < 0:
            raise ValueError("n_electrons should be non-negative.")
        if temperature < 0:
            raise ValueError("temperature must be non-negative")
        self.temperature = float(temperature)
        self.smearing = _check_smearing(smearing or ("FermiDirac" if temperature > 0 else "None"))
        self.magnetic_moments = [float(m) for m in magnetic_moments]
        if self.magnetic_moments and len(self.magnetic_moments) != len(self.atoms):
            raise ValueError("Length of atoms and magnetic_moments vectors need to agree.")
        if spin_polarization is None:
            spin_polarization = "collinear" if any(m != 0 for m in self.magnetic_moments) or self.magnetic_moments else "none"
        if spin_polarization not in ("none", "collinear", "spinless"):
            raise ValueError("Only :none, :collinear and :spinless allowed for spin_polarization")
        self.spin_polarization = spin_polarization
        self.n_spin_components = 2 if spin_polarization == "collinear" else 1
        self.term_types = list(terms)          # names, or term objects such as Hubbard(...) (called with the basis)
        self.term_names = [t if isinstance(t, str) else t.name for t in self.term_types]
        self.functionals = list(functionals)
        groups = {}
        for i, a in enumerate(self.atoms):
            groups.setdefault(a, []).append(i)
        self.atom_groups = list(groups.values())
        if symmetries is True:
            labels = [(a.symbol, a.psp.identifier, round(self.magnetic_moments[i], 6) if self.magnetic_moments else 0)
                      for i, a in enumerate(self.atoms)]
            self.symmetries = (symmetry_operations(self.lattice, labels, self.positions)
                               if self.atoms else [SymOp(np.eye(3), np.zeros(3))])
        elif symmetries is False:
            self.symmetries = [SymOp(np.eye(3), np.zeros(3))]
        else:
            self.symmetries = list(symmetries)

    @property
    def filled_occupation(self):      # Model.jl:352-360
        return 2 if self.spin_polarization == "none" else 1


def model_atomic(lattice, atoms, positions, *, extra_terms=(), kinetic_blowup=None, **kwargs):
    """standard_models.jl:45-60; `kinetic_blowup` (BlowupCHV(), BlowupAbinit(...)) smooths the kinetic energy near Ecut."""
    from .terms import Kinetic
    kinetic = "Kinetic" if kinetic_blowup is None else Kinetic(blowup=kinetic_blowup)
    terms = [kinetic, "AtomicLocal", "AtomicNonlocal", "Ewald", "PspCorrection", *extra_terms]
    if kwargs.get("temperature", 0) != 0:
        terms.append("Entropy")
    kwargs.setdefault("model_name", "atomic")
    return Model(lattice, atoms, positions, terms=terms, **kwargs)


def model_DFT(lattice, atoms, positions, *, functionals, extra_terms=(), **kwargs):
    """standard_models.jl:116-134: atomic model + Hartree + Xc(functionals) + extra_terms (e.g. Hubbard(...))."""
    return model_atomic(lattice, atoms, positions, extra_terms=("Hartree", "Xc", *extra_terms), functionals=functionals,
                        model_name="DFT", **kwargs)
