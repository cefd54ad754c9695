"""Timing of the Wannier90 overlap products M^{k,b} = ψ_k^H ψ_{k+b}[idx] (dftk_b200_overlap_multi) on one GPU, each against
the formulation "gather every pair into a copy (sphere_remap), then one GEMM per pair" in the same run on the same card:

  c2     Si2, Ecut 30, the unfolded 8³ k-grid (512 k-points), 12 bands, the first shell of 8 b-vectors: 4096 pairs (fused path)
  si128  the Γ block of the Si128 supercell (4³ cells), Ecut 30, 259 bands, its 8 G-shift neighbours (large path)

Orbitals are seeded random blocks on the spheres (the product does not depend on their values).  Times are CUDA events over
repeated calls after a warm-up; the algorithmic bytes are 16·n_G·n_bands·(1 + nntot) per k-point for the blocks plus
8·n_G·nntot for the index tables.  The card's name and power limit are printed beside the numbers.  `--out PATH` also writes
the result as JSON."""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import dftk_b200 as dftk  # noqa: E402
from dftk_b200.transfer import remap_tables, sphere_remap  # noqa: E402
from dftk_b200.wannier import overlap_multi  # noqa: E402
import wannier_oracle as W  # noqa: E402
from silicon import LATTICE  # noqa: E402

I3 = np.eye(3, dtype=np.int32)


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3 / reps


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                     text=True).strip()
    except Exception:
        pl = "unknown"
    return name, pl


def spheres(recip, Ecut, kcoords, dev):
    """G vectors (n_G, 3) of each k-sphere, a cube holding every sphere and its neighbours' shifts, and the per-k lookup
    cube index -> sphere row (-1 outside)."""
    kc = np.asarray(kcoords, dtype=float)
    gmax = math.sqrt(2 * Ecut)
    nmax = [int(math.ceil(gmax * np.linalg.norm(np.linalg.inv(recip)[a]))) + 2 for a in range(3)]
    n = [2 * m + 1 for m in nmax]
    axes = [torch.tensor([i if i <= m else i - nn for i in range(nn)], device=dev) for m, nn in zip(nmax, n)]
    Z, Y, X = torch.meshgrid(axes[2], axes[1], axes[0], indexing="ij")
    G = torch.stack([X.reshape(-1), Y.reshape(-1), Z.reshape(-1)], dim=1)
    rec = torch.as_tensor(recip, device=dev)
    out = []
    for k in kc:
        p = (G.to(torch.float64) + torch.as_tensor(k, device=dev)) @ rec.T
        mapping = torch.nonzero((p * p).sum(dim=1) / 2 <= Ecut).reshape(-1)
        lk = torch.full((G.shape[0],), -1, dtype=torch.int64, device=dev)
        lk[mapping] = torch.arange(mapping.numel(), device=dev)
        out.append((G[mapping].contiguous(), lk))
    return out, tuple(n)


def random_blocks(sph, n_bands, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return [torch.randn((n_bands, G.shape[0]), dtype=torch.complex128, device=dev, generator=g) for G, _ in sph]


def case(name, recip, Ecut, kcoords, kgrid, n_bands, reps):
    dev = torch.device("cuda:0")
    ctx = dftk.B200().ctx
    sph, fft_size = spheres(recip, Ecut, kcoords, dev)
    psi = random_blocks(sph, n_bands, dev, 7)
    nntot, nnkpts, _, _ = W.nnkp_list(kcoords, recip, kgrid)
    pairs = []
    for ik, ikb, Gs in nnkpts:
        idx, _ = remap_tables(ctx, sph[ik][0], I3, np.asarray(Gs), sph[ikb][1], fft_size)
        pairs.append((psi[ik], psi[ikb], idx, sph[ik][0].shape[0]))
    fused = lambda: overlap_multi(ctx, n_bands, n_bands, pairs)
    gathered = [torch.empty((n_bands, p[3]), dtype=torch.complex128, device=dev) for p in pairs]
    C_ref = torch.empty((len(pairs), n_bands, n_bands), dtype=torch.complex128, device=dev)

    def remap_gemm():
        sphere_remap(ctx, [(B, g, idx, None, 0) for (_, B, idx, _), g in zip(pairs, gathered)])
        for p, ((A, _, _, _), g) in enumerate(zip(pairs, gathered)):
            ctx.zgemm("C", A, g, C_ref[p])

    M = fused()
    remap_gemm()
    diff = float((M - C_ref.transpose(1, 2)).abs().max() / C_ref.abs().max())
    t_fused = min(timed(fused, reps) for _ in range(3))
    t_ref = min(timed(remap_gemm, reps) for _ in range(3))
    n_G = [G.shape[0] for G, _ in sph]
    nbytes = sum(16 * g * n_bands * (1 + nntot) + 8 * g * nntot for g in n_G)
    return dict(case=name, n_k=len(kcoords), n_pairs=len(pairs), n_bands=n_bands, mean_n_G=float(np.mean(n_G)),
                path="fused" if n_bands <= 32 else "large", bytes=nbytes, fused_s=t_fused, remap_gemm_s=t_ref,
                fused_GBps=nbytes / t_fused / 1e9, remap_gemm_GBps=nbytes / t_ref / 1e9, speedup=t_ref / t_fused,
                max_rel_diff=diff)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("wannier_probe needs a GPU")
    name, pl = card()
    recip = 2 * np.pi * np.linalg.inv(LATTICE).T
    kgrid = (8, 8, 8)
    kc = [(np.array([i, j, k]) / 8) - (np.array([i, j, k]) / 8 >= 0.5) for k in range(8) for j in range(8) for i in range(8)]
    rows = [case("c2", recip, 30.0, kc, kgrid, 12, args.reps)]
    recip_sc = recip / 4
    rows.append(case("si128", recip_sc, 30.0, [np.zeros(3)], (1, 1, 1), 259, max(2, args.reps // 5)))
    for r in rows:
        r.update(card=name, power_limit=pl)
        print(f"{r['case']:6s} {r['path']:5s} pairs {r['n_pairs']:5d} bands {r['n_bands']:3d} n_G {r['mean_n_G']:9.0f}  "
              f"fused {r['fused_s'] * 1e3:8.3f} ms ({r['fused_GBps']:7.1f} GB/s)  remap+GEMM {r['remap_gemm_s'] * 1e3:8.3f} ms "
              f"({r['remap_gemm_GBps']:7.1f} GB/s)  x{r['speedup']:.2f}  diff {r['max_rel_diff']:.1e}  [{name}, {pl}]")
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
