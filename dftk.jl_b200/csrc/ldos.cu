// LDOS of many energies from one pass over the bands (dos.py; reference seam src/postprocess/dos.jl compute_ldos):
//   ldos[j, spin, :] += Σ_kn W[j, k, n] |ψ_kn(r)|² / Ω
// |ψ_kn(r)|² does not depend on the energy, so every kept band is transformed once (the sphere -> cube inverse FFT of the
// density pass), staged as |ψ|²/Ω in k-block scratch, and multiplied into all energies at once by the real × real DMMA
// product of ldos_core.cuh.  A round takes the next chunk of every block of one spin, so the output is read and written
// once per round and not once per block.
#include <algorithm>
#include "structs.cuh"
#include "ldos_core.cuh"

using namespace dftk;

namespace {

// two CTAs per SM (<= 128 registers): while one waits at a barrier for its tiles, the other runs its MMAs
__global__ void __launch_bounds__(LD_THREADS, 2) k_ldos_product(LdosProduct p) {
  extern __shared__ __align__(16) double sm[];
  double acc[2 * 4 * LD_SLOTS * 4];
  ldos_cta(p, blockIdx.x, (int)blockIdx.y, sm, acc);
}

// rho[e] = nrm |cube[e]|² over nb bands of N points
__global__ void k_ldos_abs2(const cplx* __restrict__ cube, long long total, double nrm, double* __restrict__ rho) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const cplx v = cube[e];
    rho[e] = nrm * (v.x * v.x + v.y * v.y);
  }
}

struct Piece {      // bands [b0, b0 + nb) of block i, all kept
  int i;
  int b0, nb;
};

}  // namespace

extern "C" {

int dftk_b200_ldos_accumulate_multi(int64_t n_blocks, dftk_b200_kblock* const* kbs, const void* const* psi, const int32_t* n_bands,
                                    int64_t n_energies, int64_t n_spin, const double* W, int64_t ld_w, double* ldos) {
  dftk_b200_ctx* ctx = (n_blocks > 0 && kbs && kbs[0]) ? kbs[0]->grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(n_blocks >= 0 && (n_blocks == 0 || (kbs && psi && n_bands && W && ldos)), "ldos_accumulate_multi: bad argument");
  if (n_blocks == 0 || n_energies == 0) return DFTK_B200_OK;
  REQUIRE(n_energies > 0 && n_energies <= 65535 * (int64_t)LD_TN && (n_spin == 1 || n_spin == 2) && ld_w > 0,
          "ldos_accumulate_multi: bad energy count, spin count or ld_w");
  dftk_b200_grid* g = kbs[0]->grid;
  for (int64_t i = 0; i < n_blocks; ++i) {
    REQUIRE(kbs[i] && kbs[i]->grid == g && kbs[i]->spin >= 0 && kbs[i]->spin < n_spin && n_bands[i] >= 0 && n_bands[i] <= ld_w,
            "ldos_accumulate_multi: the blocks must share one grid, with spins below n_spin and n_bands <= ld_w");
    if (n_bands[i] > 0) require_device(ctx, psi[i], "ldos_accumulate_multi: orbitals");
  }
  require_device(ctx, W, "ldos_accumulate_multi: W");
  require_device(ctx, ldos, "ldos_accumulate_multi: ldos");
  // screening: a band with a zero weight at every energy is neither transformed nor multiplied
  const int64_t ldw_e = n_blocks * ld_w;           // W[j * ldw_e + i * ld_w + n]
  std::vector<double> Wh((size_t)n_energies * ldw_e);
  CUDA_CHECK(cudaMemcpyAsync(Wh.data(), W, Wh.size() * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  std::vector<std::vector<Piece>> queue(n_blocks);     // kept runs of each block, cut into FFT chunks
  size_t total = 0;
  for (int64_t i = 0; i < n_blocks; ++i) {
    const int nbi = n_bands[i];
    if (nbi == 0) continue;
    std::vector<char> keep(nbi, 0);
    for (int64_t j = 0; j < n_energies; ++j)
      for (int n = 0; n < nbi; ++n) keep[n] |= Wh[(size_t)j * ldw_e + i * ld_w + n] != 0.0;
    const int chunk = band_chunk_for(kbs[i], nbi);
    for (int n = 0; n < nbi;) {
      if (!keep[n]) {
        ++n;
        continue;
      }
      int e = n;
      while (e < nbi && keep[e] && e - n < chunk) ++e;
      queue[i].push_back(Piece{(int)i, n, e - n});
      total += e - n;
      n = e;
    }
  }
  if (total == 0) return DFTK_B200_OK;
  // rounds: per spin, the next piece of every block of that spin; their pointer lists all go up in one copy
  std::vector<std::vector<Piece>> rounds;
  std::vector<int> round_spin;
  for (int spin = 0; spin < n_spin; ++spin) {
    std::vector<size_t> next(n_blocks, 0);
    for (;;) {
      std::vector<Piece> r;
      for (int64_t i = 0; i < n_blocks; ++i)
        if (kbs[i]->spin == spin && next[i] < queue[i].size()) r.push_back(queue[i][next[i]++]);
      if (r.empty()) break;
      rounds.push_back(r);
      round_spin.push_back(spin);
    }
  }
  std::vector<const double*> ptrs(2 * total);        // per round: its K density rows, then its K weight columns
  std::vector<size_t> round_off(rounds.size());
  size_t o = 0;
  for (size_t q = 0; q < rounds.size(); ++q) {
    round_off[q] = o;
    size_t K = 0;
    for (const Piece& pc : rounds[q]) K += pc.nb;
    size_t k = 0;
    for (const Piece& pc : rounds[q]) {
      dftk_b200_kblock* kb = kbs[pc.i];
      kb->ldos_rho.ensure((size_t)band_chunk_for(kb, n_bands[pc.i]) * g->N);
      for (int b = 0; b < pc.nb; ++b, ++k) {
        ptrs[o + k] = kb->ldos_rho.p + (size_t)b * g->N;
        ptrs[o + K + k] = W + pc.i * ld_w + pc.b0 + b;
      }
    }
    o += 2 * K;
  }
  const double* const* d_ptrs = ctx->slot[0].ring.put(ptrs, ctx->stream);
  const double nrm = g->ifft_norm * g->ifft_norm;
  const size_t smem = LD_SMEM_DOUBLES * sizeof(double);      // 53 KB: above the default limit of 48 KB
  CUDA_CHECK(cudaFuncSetAttribute(k_ldos_product, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  for (size_t q = 0; q < rounds.size(); ++q) {
    int K = 0;
    for (const Piece& pc : rounds[q]) {
      dftk_b200_kblock* kb = kbs[pc.i];
      cplx* cube = kb->ldos_cube.ensure((size_t)band_chunk_for(kb, n_bands[pc.i]) * g->N);
      kb_sphere_to_real(kb, (const cplx*)psi[pc.i] + (size_t)pc.b0 * kb->n_pw, cube, pc.nb, 1.0);
      const long long n_el = (long long)pc.nb * g->N;
      const unsigned grid = (unsigned)std::min<long long>((n_el + 255) / 256, (long long)ctx->sm_count * 16);
      LAUNCH(ctx, k_ldos_abs2, grid, 256, 0, (const cplx*)cube, n_el, nrm, kb->ldos_rho.p);
      K += pc.nb;
    }
    LdosProduct p;
    p.D = d_ptrs + round_off[q];
    p.W = d_ptrs + round_off[q] + K;
    p.ldw = ldw_e;
    p.K = K;
    p.M = g->N;
    p.n = (int)n_energies;
    p.C = ldos + (size_t)round_spin[q] * g->N;
    p.ldc = n_spin * g->N;
    LAUNCH(ctx, k_ldos_product, dim3((unsigned)((g->N + LD_TM - 1) / LD_TM), (unsigned)((n_energies + LD_TN - 1) / LD_TN)),
           LD_THREADS, smem, p);
  }
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  ctx->slot[0].ring.rewind();
  API_END(ctx)
}

}  // extern "C"
