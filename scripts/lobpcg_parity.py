"""Output parity of the device LOBPCG between two builds: seeded solves on the batched small path and on the direct path,
written out so that the results of two builds can be compared call for call.

  python scripts/lobpcg_parity.py OUT_DIR          # writes OUT_DIR/parity.json
  python scripts/lobpcg_parity.py --compare A B    # compares two parity.json files, exit code 1 on a mismatch

Every case records λ, the residual norms, n_iter, n_matvec, a checksum of the orbitals (sha256 of the bytes and the
Frobenius norm) and the launches and host synchronisations of the call.  The comparison expects the small path to be
bit-for-bit identical, and on the direct path equal n_iter and n_matvec, λ within 1e-12 relative, and orbitals equal up
to the same tolerance; launch and sync counts must be equal everywhere.  The direct path may differ in the last bits
because `matrix_stats` there may sum across warps in another order; its outputs only steer conditioning thresholds.
"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np

A_SI = 10.26 / 2
OPTION_DEFAULTS = dict(small_dense=1, gemm_backend=0, i8_min_rows=32768, force_svd_fallback=0)


def _si_basis(dftk, rep, Ecut, kgrid):
    lat = rep * np.array([[0, A_SI, A_SI], [A_SI, 0, A_SI], [A_SI, A_SI, 0]])
    pos = [(b + np.array([i, j, k])) / rep for i in range(rep) for j in range(rep) for k in range(rep)
           for b in (np.ones(3) / 8, -np.ones(3) / 8)]
    Si = dftk.ElementPsp("Si")
    model = dftk.model_DFT(lat, [Si] * len(pos), pos, functionals=["lda_x", "lda_c_vwn"], symmetries=kgrid != (1, 1, 1))
    kg = dftk.ExplicitKpoints([[0, 0, 0]]) if kgrid == (1, 1, 1) else kgrid
    basis = dftk.PlaneWaveBasis(model, Ecut=Ecut, kgrid=kg)
    _, ham = dftk.energy_hamiltonian(basis, None, None, rho=dftk.guess_density(basis))
    for h in ham:
        h.bind()
    return basis, [h.kblock for h in ham]


def _orbitals(Xs):
    h = hashlib.sha256()
    norm2 = 0.0
    for X in Xs:
        a = X.cpu().numpy()
        h.update(np.ascontiguousarray(a).tobytes())
        norm2 += float(np.vdot(a, a).real)
    return dict(sha256=h.hexdigest(), norm=norm2 ** 0.5, data=[X.cpu().numpy() for X in Xs])


def _case(ctx, fn, **options):
    for k, v in options.items():
        ctx.set_option(k, v)
    try:
        ctx.sync()
        ctx.launch_count(reset=True)
        ctx.sync_count(reset=True)
        out = fn()
        ctx.sync()
        out.update(launches=ctx.launch_count(), syncs=ctx.sync_count())
    finally:
        for k in options:
            ctx.set_option(k, OPTION_DEFAULTS[k])
    return out


def _solves(results, Xs):
    out = dict(lam=[[float(v) for v in r["λ"]] for r in results], resid=[[float(v) for v in r["residual_norms"]] for r in results],
               n_iter=[r["n_iter"] for r in results], n_matvec=[r["n_matvec"] for r in results])
    out.update(_orbitals(Xs))
    return out


def run(out_dir):
    import torch
    import dftk_b200 as dftk
    from dftk_b200 import device as dev

    os.makedirs(out_dir, exist_ok=True)
    cases = {}
    # C2-like: Si2 on a 3x3x3 k-grid, 8 bands per block
    basis, kbs = _si_basis(dftk, 1, 15.0, (3, 3, 3))
    ctx = basis.architecture.ctx

    def multi_small():
        Xs = dev.random_orbitals_multi(kbs, 8, 1)
        res = dev.lobpcg_multi(kbs, Xs, tol=1e-9, maxiter=100)
        return _solves(res, Xs)
    cases["lobpcg_multi_small"] = _case(ctx, multi_small)

    def random_orbitals(nb, seed):
        def f():
            return _orbitals(dev.random_orbitals_multi(kbs, nb, seed))
        return f
    cases["random_orbitals_small"] = _case(ctx, random_orbitals(8, 3))
    cases["random_orbitals_direct_nb8"] = _case(ctx, random_orbitals(8, 3), small_dense=0)
    cases["random_orbitals_direct_nb40"] = _case(ctx, random_orbitals(40, 5))

    def band_energies():
        Xs = dev.random_orbitals_multi(kbs, 8, 7)
        ek, en = dev.band_energies_multi(kbs, Xs)
        return dict(ekin=[[float(v) for v in e] for e in ek], enl=[[float(v) for v in e] for e in en])
    cases["band_energies_multi"] = _case(ctx, band_energies)

    def single(nb, seed, **kw):
        def f():
            X = dev.random_orbitals_multi(kbs[:1], nb, seed)[0]
            return _solves([kbs[0].lobpcg(X, **kw)], [X])
        return f
    # the SVD fallback of ortho! runs the direct forms inside a batched solve
    cases["lobpcg_small_svd_fallback"] = _case(ctx, single(8, 9, tol=1e-9, maxiter=100), force_svd_fallback=1)
    cases["lobpcg_direct_svd_fallback"] = _case(ctx, single(8, 9, tol=1e-9, maxiter=100), small_dense=0, force_svd_fallback=1)

    # Si16 at Gamma, 40 bands: the direct path (GEMMs + cuSOLVER), with the DMMA GEMMs and with the INT8 tensor cores
    basis16, kbs16 = _si_basis(dftk, 2, 20.0, (1, 1, 1))
    ctx16 = basis16.architecture.ctx
    kb = kbs16[0]

    def direct(M):
        def f():
            X = dev.random_orbitals_multi([kb], M, 11)[0]
            return _solves([kb.lobpcg(X, tol=1e-8, maxiter=60, n_conv_check=M - 4)], [X])
        return f
    cases["lobpcg_direct_be0"] = _case(ctx16, direct(40), small_dense=0, gemm_backend=0)
    cases["lobpcg_direct_be4"] = _case(ctx16, direct(40), small_dense=0, gemm_backend=4, i8_min_rows=1024)
    cases["lobpcg_direct_nb24_be0"] = _case(ctx16, direct(24), small_dense=0, gemm_backend=0)
    cases["lobpcg_small_nb24"] = _case(ctx16, direct(24))

    arrays = {}
    for name, c in cases.items():
        for i, a in enumerate(c.pop("data", [])):
            arrays[f"{name}.{i}"] = a
    np.savez(os.path.join(out_dir, "orbitals.npz"), **arrays)
    with open(os.path.join(out_dir, "parity.json"), "w") as f:
        json.dump(dict(device=torch.cuda.get_device_name(0), cases=cases), f, indent=1)
    print(json.dumps({k: dict(n_iter=v.get("n_iter"), launches=v["launches"], syncs=v["syncs"]) for k, v in cases.items()}))


def compare(dir_a, dir_b):
    A = json.load(open(os.path.join(dir_a, "parity.json")))["cases"]
    B = json.load(open(os.path.join(dir_b, "parity.json")))["cases"]
    XA, XB = np.load(os.path.join(dir_a, "orbitals.npz")), np.load(os.path.join(dir_b, "orbitals.npz"))
    ok = True
    for name in A:
        a, b = A[name], B[name]
        exact = a == b and all(np.array_equal(XA[k], XB[k]) for k in XA.files if k.startswith(name + "."))
        direct = "direct" in name
        line = dict(case=name, bitwise=exact, launches=(a["launches"], b["launches"]), syncs=(a["syncs"], b["syncs"]))
        good = a["launches"] == b["launches"] and a["syncs"] == b["syncs"]
        if "lam" in a:
            la, lb = np.array(a["lam"]), np.array(b["lam"])
            line["lam_rel"] = float(np.abs(la - lb).max() / np.abs(la).max())
            line["n_iter"] = (a["n_iter"], b["n_iter"])
            good = good and a["n_iter"] == b["n_iter"] and a["n_matvec"] == b["n_matvec"]
        if direct:
            xs = [k for k in XA.files if k.startswith(name + ".")]
            line["X_rel"] = max((float(np.abs(XA[k] - XB[k]).max() / np.abs(XA[k]).max()) for k in xs), default=0.0)
            good = good and line.get("lam_rel", 0.0) <= 1e-12
        else:
            good = good and exact
        line["ok"] = bool(good)
        ok = ok and good
        print(json.dumps(line))
    return ok


if __name__ == "__main__":
    if sys.argv[1] == "--compare":
        sys.exit(0 if compare(sys.argv[2], sys.argv[3]) else 1)
    run(sys.argv[1])
