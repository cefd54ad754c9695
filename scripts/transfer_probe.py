"""Timing of the basis-transfer kernels on one GPU: the batched sphere remap on a block the size of the Γ block of the Si128
supercell (259 bands x 135 491 plane waves, complex128: 0.56 GB read and 0.56 GB written), as one pair and as the same
bytes split into 8 pairs, and interpolate_density from 150^3 to 192^3 and to 96^3 (FFT prefilter + 27-tap evaluation).
Bandwidth is (bytes read + bytes written) / time with CUDA events, against the H100 SXM data-sheet 3.35 TB/s; the card's
name and power limit are printed beside the numbers.  `--out PATH` also writes the result as JSON to PATH."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import dftk_b200 as dftk  # noqa: E402
from dftk_b200.transfer import sphere_remap, _ctx_of  # noqa: E402

PEAK = 3.35e12


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    ctx = _ctx_of(torch.zeros(1, device=dev))
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    nb, n = 259, 135491
    g = torch.Generator(device=dev).manual_seed(0)
    src = torch.randn((nb, n), dtype=torch.complex128, device=dev, generator=g)
    dst = torch.empty_like(src)
    perm = torch.randperm(n, device=dev, generator=g)
    ident = torch.arange(n, device=dev)
    phase = torch.exp(1j * torch.rand(n, dtype=torch.float64, device=dev, generator=g))
    res = dict(gpu=gpu)
    moved = 2 * src.numel() * 16 + nb // 16 * n * 8
    for name, idx, ph in [("remap_identity", ident, None), ("remap_permuted", perm, None), ("remap_phase", perm, phase)]:
        t = timed(lambda: sphere_remap(ctx, [(src, dst, idx, ph, 0)]), 20)
        res[name] = dict(seconds=t, GBps=moved / t / 1e9, share_of_peak=moved / t / PEAK)
    assert torch.allclose(dst, src[:, perm] * phase, rtol=0, atol=1e-15 * src.abs().max().item())
    rows = nb // 8
    pairs = [(src[i * rows:(i + 1) * rows].contiguous(), torch.empty((rows, n), dtype=src.dtype, device=dev), perm, None, 0)
             for i in range(8)]
    t = timed(lambda: sphere_remap(ctx, pairs), 20)
    moved8 = 8 * (2 * rows * n * 16)
    res["remap_8_pairs"] = dict(seconds=t, GBps=moved8 / t / 1e9, share_of_peak=moved8 / t / PEAK)
    rho = torch.rand((1, 150, 150, 150), dtype=torch.float64, device=dev, generator=g)
    for grid in [(192, 192, 192), (96, 96, 96)]:
        t = timed(lambda: dftk.interpolate_density(rho, grid), 10)
        res[f"interpolate_150_to_{grid[0]}"] = dict(seconds=t)
    print(json.dumps(res, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
