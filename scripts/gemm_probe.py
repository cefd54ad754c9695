"""Development probe: the FP64 GEMMs of the H apply and of LOBPCG at the benchmark shape, own DMMA kernels vs cuBLAS,
and the FP64 tensor-core throughput of the three mma.sync f64 shapes in a register-resident loop.

    python scripts/gemm_probe.py [--npw 135491] [--nproj 640] [--m 259] [--stages 2,3,4] [--out FILE.json]

Defaults are the 128-atom Si cell of bench.py.  The package is imported from PYTHONPATH first, so pointing PYTHONPATH
at another checkout times that checkout's kernels with this probe."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

sys.path.append(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import dftk_b200  # noqa: E402

DMMA_SRC = r"""
#include <cuda_runtime.h>
// ITER dependent steps on NACC independent accumulators per warp; operands never leave registers
template <int SHAPE>
__global__ void k_dmma(double* out, double seed, int iters) {
  constexpr int NACC = 8;
  double a[8], b[4], c[NACC][4];
  for (int i = 0; i < 8; ++i) a[i] = seed * (threadIdx.x + i);
  for (int i = 0; i < 4; ++i) b[i] = seed * (threadIdx.x - i);
  for (int j = 0; j < NACC; ++j) c[j][0] = c[j][1] = c[j][2] = c[j][3] = 0.0;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int j = 0; j < NACC; ++j) {
      if (SHAPE == 4)
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                     : "+d"(c[j][0]), "+d"(c[j][1]) : "d"(a[0]), "d"(b[0]));
      else if (SHAPE == 8)
        asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+d"(c[j][0]), "+d"(c[j][1]), "+d"(c[j][2]), "+d"(c[j][3])
                     : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
      else
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};"
                     : "+d"(c[j][0]), "+d"(c[j][1]), "+d"(c[j][2]), "+d"(c[j][3])
                     : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                       "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
    }
  }
  double s = 0.0;
  for (int j = 0; j < NACC; ++j) s += c[j][0] + c[j][1] + c[j][2] + c[j][3];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
// FLOP/s of SHAPE (4, 8, 16 = k of m8n8k4, m16n8k8, m16n8k16) over `blocks` CTAs of `threads` threads
extern "C" double dmma_tflops(int shape, int blocks, int threads, int iters) {
  double* out;
  cudaMalloc(&out, sizeof(double) * blocks * threads);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  auto run = [&](int n) {
    if (shape == 4) k_dmma<4><<<blocks, threads>>>(out, 1e-3, n);
    else if (shape == 8) k_dmma<8><<<blocks, threads>>>(out, 1e-3, n);
    else k_dmma<16><<<blocks, threads>>>(out, 1e-3, n);
  };
  run(iters / 10);
  cudaEventRecord(e0);
  run(iters);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  cudaFree(out);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  if (cudaGetLastError() != cudaSuccess) return -1.0;
  const double macs_per_mma = shape == 4 ? 256.0 : 128.0 * shape;
  return 2.0 * macs_per_mma * 8 * (double)iters * blocks * (threads / 32) / (ms * 1e-3) / 1e12;
}
"""


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "nvidia-smi unavailable"


def timeit(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return min(ts)


def dmma_ceiling(sm_count):
    with tempfile.TemporaryDirectory() as d:
        src, so = os.path.join(d, "dmma.cu"), os.path.join(d, "dmma.so")
        open(src, "w").write(DMMA_SRC)
        subprocess.check_call(["nvcc", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-Xcompiler", "-fPIC",
                               "-o", so, src])
        L = ctypes.CDLL(so)
        L.dmma_tflops.restype = ctypes.c_double
        res = {}
        for shape, iters in ((4, 800000), (8, 200000), (16, 100000)):   # ~0.1-0.4 s per run: long enough for sustained clocks
            for warps in (4, 8, 16):
                res[f"m{'8n8k4' if shape == 4 else f'16n8k{shape}'}_{warps}warps_per_sm"] = \
                    L.dmma_tflops(shape, sm_count, 32 * warps, iters)
        return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--npw", type=int, default=135491)
    ap.add_argument("--nproj", type=int, default=640)
    ap.add_argument("--m", type=int, default=259)
    ap.add_argument("--stages", default="2,3,4", help="gemm_stages values to time for the own kernels")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-dmma", action="store_true", help="skip the mma.sync throughput loop")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    ctx = dftk_b200.Context(0)
    dev = ctx.device
    npw, nproj, M = args.npw, args.nproj, args.m
    g = torch.Generator(device=dev).manual_seed(0)

    def rnd(*shape):
        return torch.view_as_complex(torch.randn(*shape, 2, generator=g, device=dev, dtype=torch.float64))

    P, psi, D = rnd(nproj, npw), rnd(M, npw), rnd(nproj, nproj)
    proj, dproj, hpsi = rnd(M, nproj), rnd(M, nproj), rnd(M, npw)
    Y = rnd(3 * M, npw)
    G = torch.empty(3 * M, 3 * M, dtype=torch.complex128, device=dev)
    cX = rnd(M, 3 * M)
    # name: (call, FP64 flop)
    cases = {
        "nonlocal_gram_C": (lambda: ctx.zgemm("C", P, psi, proj), 8.0 * npw * nproj * M),
        "nonlocal_D": (lambda: ctx.zgemm("N", D, proj, dproj), 8.0 * nproj * nproj * M),
        "nonlocal_update_N_beta1": (lambda: ctx.zgemm("N", P, dproj, hpsi, 1.0, 1.0), 8.0 * npw * nproj * M),
        "lobpcg_gram_3Mx3M": (lambda: ctx.zgemm("C", Y, Y, G), 8.0 * npw * 9 * M * M),
        "lobpcg_update_Kx3M_3MxM": (lambda: ctx.zgemm("N", Y, cX, psi), 8.0 * npw * 3 * M * M),
    }
    res = dict(gpu=gpu_info(), sm_count=torch.cuda.get_device_properties(0).multi_processor_count,
               shape=dict(npw=npw, nproj=nproj, M=M), library=os.path.abspath(dftk_b200.__file__))
    configs = [(f"own_stages{s}", 0, int(s)) for s in args.stages.split(",")] + [("cublas", 1, 2)]
    for name, backend, stages in configs:
        ctx.set_option("gemm_backend", backend)
        ctx.set_option("gemm_stages", stages)
        row = {}
        for case, (fn, fl) in cases.items():
            ms = timeit(fn, args.reps)
            row[case] = dict(ms=round(ms, 4), TFLOPs=round(fl / ms / 1e9, 2))
        row["nonlocal_total_ms"] = round(sum(row[c]["ms"] for c in ("nonlocal_gram_C", "nonlocal_D", "nonlocal_update_N_beta1")), 4)
        res[name] = row
        print(name, json.dumps(row), flush=True)
    ctx.set_option("gemm_backend", 0)
    if not args.no_dmma:
        res["dmma_ceiling_TFLOPs"] = dmma_ceiling(res["sm_count"])
        print("dmma", json.dumps(res["dmma_ceiling_TFLOPs"]), flush=True)
    print(json.dumps(res), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
