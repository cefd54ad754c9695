// CUDA kernels (thin __global__ wrappers over the stage bodies of fft_core.cuh) and host drivers of
// the batched, pruned sphere<->cube FFT pipeline.  Reference semantics: src/fft.jl:106-172 (ifft!/fft!
// with Gvec_mapping) and the "local" part of mul!(::DftHamiltonianBlock), src/terms/Hamiltonian.jl:152-163.
#include "structs.cuh"

namespace dftk {

#define FFT_THREADS 256
extern __shared__ __align__(16) unsigned char dyn_smem[];

__global__ void __launch_bounds__(FFT_THREADS)
k_sphere_to_x(SphereTables T, FftPlan px, const cplx* twx, const cplx* psi, int64_t ldpsi, cplx* W1,
              int L, int Lp) {
  stage_sphere_to_x(T, px, twx, psi, ldpsi, W1, L, Lp, (cplx*)dyn_smem,
                    Dim3i{(int)blockIdx.x, (int)blockIdx.y, 0});
}
__global__ void __launch_bounds__(FFT_THREADS)
k_y_backward(SphereTables T, FftPlan py, const cplx* twy, const cplx* W1, cplx* W2, int L, int Lp) {
  stage_y_backward(T, py, twy, W1, W2, L, Lp, (cplx*)dyn_smem,
                   Dim3i{(int)blockIdx.x, (int)blockIdx.y, (int)blockIdx.z});
}
__global__ void __launch_bounds__(FFT_THREADS)
k_z_apply_potential(SphereTables T, FftPlan pz, const cplx* twz, cplx* W2, const double* V, int L,
                    int Lp) {
  stage_z_apply_potential(T, pz, twz, W2, V, L, Lp, (cplx*)dyn_smem,
                          Dim3i{(int)blockIdx.x, (int)blockIdx.y, (int)blockIdx.z});
}
__global__ void __launch_bounds__(FFT_THREADS)
k_z_to_cube(SphereTables T, FftPlan pz, const cplx* twz, const cplx* W2, cplx* cube, double scale,
            int L, int Lp) {
  stage_z_to_cube(T, pz, twz, W2, cube, scale, L, Lp, (cplx*)dyn_smem,
                  Dim3i{(int)blockIdx.x, (int)blockIdx.y, (int)blockIdx.z});
}
__global__ void __launch_bounds__(FFT_THREADS)
k_z_from_cube(SphereTables T, FftPlan pz, const cplx* twz, const cplx* cube, cplx* W2, int L, int Lp) {
  stage_z_from_cube(T, pz, twz, cube, W2, L, Lp, (cplx*)dyn_smem,
                    Dim3i{(int)blockIdx.x, (int)blockIdx.y, (int)blockIdx.z});
}
__global__ void __launch_bounds__(FFT_THREADS)
k_z_density(SphereTables T, FftPlan pz, const cplx* twz, const cplx* W2, const double* wts, int nb,
            double* rho, int L, int Lp) {
  stage_z_density(T, pz, twz, W2, wts, nb, rho, L, Lp, (cplx*)dyn_smem,
                  Dim3i{(int)blockIdx.x, (int)blockIdx.y, 0});
}
__global__ void __launch_bounds__(FFT_THREADS)
k_y_forward(SphereTables T, FftPlan py, const cplx* twy, const cplx* W2, cplx* W1, int L, int Lp) {
  stage_y_forward(T, py, twy, W2, W1, L, Lp, (cplx*)dyn_smem,
                  Dim3i{(int)blockIdx.x, (int)blockIdx.y, (int)blockIdx.z});
}
__global__ void __launch_bounds__(FFT_THREADS)
k_x_to_sphere(SphereTables T, FftPlan px, const cplx* twx, const cplx* W1, cplx* out, int64_t ldout,
              double scale, const double* kin, const cplx* psi, int64_t ldpsi, int accumulate, int L,
              int Lp) {
  stage_x_to_sphere(T, px, twx, W1, out, ldout, scale, kin, psi, ldpsi, accumulate, L, Lp,
                    (cplx*)dyn_smem, Dim3i{(int)blockIdx.x, (int)blockIdx.y, 0});
}
__global__ void __launch_bounds__(FFT_THREADS)
k_cube_pass_x(cplx* data, int nx, int64_t n_lines, FftPlan px, const cplx* twx, int sign, int L, int Lp) {
  cube_pass_x(data, nx, n_lines, px, twx, sign, L, Lp, (cplx*)dyn_smem,
              Dim3i{(int)blockIdx.x, (int)blockIdx.y, 0});
}
__global__ void __launch_bounds__(FFT_THREADS)
k_cube_pass_strided(cplx* data, int nx, int n, int64_t stride_line, int64_t stride_outer,
                    int64_t cube_size, FftPlan p, const cplx* tw, int sign, int L, int Lp) {
  cube_pass_strided(data, nx, n, stride_line, stride_outer, cube_size, p, tw, sign, L, Lp,
                    (cplx*)dyn_smem, Dim3i{(int)blockIdx.x, (int)blockIdx.y, (int)blockIdx.z});
}

static const int kMaxSmem = 200 * 1024;

void fft_set_attributes() {
#define SETATTR(k) CUDA_CHECK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem))
  SETATTR(k_sphere_to_x);
  SETATTR(k_y_backward);
  SETATTR(k_z_apply_potential);
  SETATTR(k_z_to_cube);
  SETATTR(k_z_from_cube);
  SETATTR(k_z_density);
  SETATTR(k_y_forward);
  SETATTR(k_x_to_sphere);
  SETATTR(k_cube_pass_x);
  SETATTR(k_cube_pass_strided);
#undef SETATTR
}

static inline size_t smem_for(int n, int L) { return 2 * (size_t)n * (L | 1) * sizeof(cplx); }

// ---- register two-pass engine registry (fft_reg.cu, compiled in REG_NGROUPS translation units)
void reg_register_group_0(std::vector<RegKernels>&);
void reg_register_group_1(std::vector<RegKernels>&);
void reg_register_group_2(std::vector<RegKernels>&);
void reg_register_group_3(std::vector<RegKernels>&);
static std::vector<RegKernels>& reg_table() {
  static std::vector<RegKernels> tab = [] {
    std::vector<RegKernels> t;
    reg_register_group_0(t);
    reg_register_group_1(t);
    reg_register_group_2(t);
    reg_register_group_3(t);
    return t;
  }();
  return tab;
}
const RegKernels* reg_kernels_for(int n) {
  int A, B;
  reg_pair_for(n, &A, &B);
  if (A == 0) return nullptr;
  for (const RegKernels& k : reg_table())
    if (k.A == A && k.B == B) return &k;
  return nullptr;
}
void reg_set_attributes(int smem_optin) {
  for (const RegKernels& k : reg_table()) {
    for (const void* f : {k.sphere_to_x, k.y_backward, k.z_apply, k.z_to_cube, k.z_from_cube, k.z_density,
                          k.y_forward, k.x_to_sphere, k.sphere_to_xt, k.xt_to_sphere, k.z_apply_pipe, k.m_sphere_to_x, k.m_y_backward, k.m_z_apply, k.m_y_forward,
                          k.m_x_to_sphere, k.m_z_density})
      CUDA_CHECK(cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
    // the fused y-z stage keeps a whole y-z intermediate per CTA: it may use all the shared memory of an SM
    CUDA_CHECK(cudaFuncSetAttribute(k.yz_apply, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin));
  }
}
// must match RegPair<A,B>::L (fft_reg.cuh)
static inline int reg_L(const RegKernels* k) { return k->T >= 12 ? 8 : (k->T >= 5 ? 16 : 32); }
static inline size_t reg_smem(const RegKernels* k) { return 2 * (size_t)k->A * k->B * (reg_L(k) + 1) * sizeof(cplx); }
// must match RegYZ<A,B>::smem on the device (fft_reg.cuh): S[n_zc][n|1] and one exchange buffer of kYzLines lines
static const int kYzLines = 25;
static inline size_t yz_smem(int n, int n_zc) { return ((size_t)n_zc + kYzLines) * (n | 1) * sizeof(cplx); }

// The local H apply runs its y and z passes in one kernel per (band, x line) (kr_yz_apply) when y and z share a factor
// pair of the register engine and the line's y-z intermediate fits in one CTA's shared memory.  The grid part of the
// condition also decides whether the potential gets its [x][y][z] copy.
bool grid_yz_fusable(const dftk_b200_grid* g) { return g->rx && g->ry && g->rz && g->ny == g->nz; }
static bool kb_yz_fused(const dftk_b200_kblock* kb) {
  const dftk_b200_grid* g = kb->grid;
  return grid_yz_fusable(g) && kb->T.ranges_ok && yz_smem(g->ny, kb->Th.n_zc) <= (size_t)g->ctx->smem_optin;
}
static void launch_ptr(dftk_b200_ctx* ctx, const void* f, dim3 grid, int threads, size_t smem, void** args) {
  CUDA_CHECK(cudaLaunchKernel(f, grid, dim3(threads), args, smem, ctx->stream));
  ctx->launches++;
}
static inline unsigned cdiv(int64_t a, int64_t b) { return (unsigned)((a + b - 1) / b); }

// CUDA limits gridDim.y/z to 65535: fine for every axis length the engine supports.
void fft_cube_inplace(dftk_b200_grid* g, cplx* data, int sign, int64_t batch) {
  dftk_b200_ctx* ctx = g->ctx;
  const int nx = g->nx, ny = g->ny, nz = g->nz;
  REQUIRE(batch <= 65535, "fft_cube: batch too large");
  {
    int L = g->Lx, Lp = L | 1;
    int64_t nl = (int64_t)ny * nz;
    LAUNCH(ctx, k_cube_pass_x, dim3(cdiv(nl, L), (unsigned)batch), FFT_THREADS, smem_for(nx, L),
           data, nx, nl, g->px, (const cplx*)g->twx.p, sign, L, Lp);
  }
  if (ny > 1) {
    int L = g->Ly, Lp = L | 1;
    LAUNCH(ctx, k_cube_pass_strided, dim3(cdiv(nx, L), nz, (unsigned)batch), FFT_THREADS,
           smem_for(ny, L), data, nx, ny, (int64_t)nx, (int64_t)nx * ny, g->N, g->py,
           (const cplx*)g->twy.p, sign, L, Lp);
  }
  if (nz > 1) {
    int L = g->Lz, Lp = L | 1;
    LAUNCH(ctx, k_cube_pass_strided, dim3(cdiv(nx, L), ny, (unsigned)batch), FFT_THREADS,
           smem_for(nz, L), data, nx, nz, (int64_t)nx * ny, (int64_t)nx, g->N, g->pz,
           (const cplx*)g->twz.p, sign, L, Lp);
  }
}

int band_chunk_for(dftk_b200_kblock* kb, int64_t n_bands, bool with_W2) {
  dftk_b200_grid* g = kb->grid;
  int64_t chunk = g->ctx->band_chunk;
  if (chunk <= 0) {
    // enough CTAs to fill the machine several times over, bounded scratch (<= ~4 GiB)
    size_t per_band = ((size_t)kb->Th.n_cols * g->nx + (with_W2 ? (size_t)kb->Th.n_zc * g->ny * g->nx : 0)) * sizeof(cplx);
    chunk = (int64_t)((size_t)4 << 30) / (int64_t)(per_band ? per_band : 1);
    if (chunk > 64) chunk = 64;
    if (chunk < 1) chunk = 1;
  }
  if (chunk > n_bands) chunk = n_bands;
  if (chunk > 65535) chunk = 65535;
  return (int)chunk;
}

static void ensure_scratch(dftk_b200_kblock* kb, int nb) {
  dftk_b200_grid* g = kb->grid;
  kb->W1.ensure((size_t)nb * kb->Th.n_cols * g->nx);
  kb->W2.ensure((size_t)nb * kb->Th.n_zc * g->ny * g->nx);
}

void kb_sphere_to_planes(dftk_b200_kblock* kb, const cplx* psi, int64_t ldpsi, int nb) {
  dftk_b200_grid* g = kb->grid;
  dftk_b200_ctx* ctx = g->ctx;
  ensure_scratch(kb, nb);
  if ((g->rx && kb->T.ranges_ok)) {
    int L = reg_L(g->rx), Lp = L + 1;
    const cplx* tw = (const cplx*)g->twx.p;
    cplx* W1 = kb->W1.p;
    void* args[] = {&kb->T, &tw, &psi, &ldpsi, &W1, &L, &Lp};
    launch_ptr(ctx, g->rx->sphere_to_x, dim3(cdiv(kb->T.n_cols, L), nb), L * g->rx->T, reg_smem(g->rx) + 5 * L * sizeof(int), args);
  } else {
    int L = g->Lx, Lp = L | 1;
    LAUNCH(ctx, k_sphere_to_x, dim3(cdiv(kb->T.n_cols, L), nb), FFT_THREADS, smem_for(g->nx, L), kb->T,
           g->px, (const cplx*)g->twx.p, psi, ldpsi, kb->W1.p, L, Lp);
  }
  if ((g->ry && kb->T.ranges_ok)) {
    int L = reg_L(g->ry), Lp = L + 1;
    const cplx* tw = (const cplx*)g->twy.p;
    const cplx* W1 = kb->W1.p;
    cplx* W2 = kb->W2.p;
    void* args[] = {&kb->T, &tw, &W1, &W2, &L, &Lp};
    launch_ptr(ctx, g->ry->y_backward, dim3(cdiv(g->nx, L), kb->T.n_zc, nb), L * g->ry->T, reg_smem(g->ry), args);
  } else {
    int L = g->Ly, Lp = L | 1;
    LAUNCH(ctx, k_y_backward, dim3(cdiv(g->nx, L), kb->T.n_zc, nb), FFT_THREADS, smem_for(g->ny, L),
           kb->T, g->py, (const cplx*)g->twy.p, (const cplx*)kb->W1.p, kb->W2.p, L, Lp);
  }
}

void kb_planes_to_sphere(dftk_b200_kblock* kb, cplx* out, int64_t ldout, int nb, double scale,
                         const double* kin, const cplx* psi, int64_t ldpsi, int accumulate) {
  dftk_b200_grid* g = kb->grid;
  dftk_b200_ctx* ctx = g->ctx;
  if ((g->ry && kb->T.ranges_ok)) {
    int L = reg_L(g->ry), Lp = L + 1;
    const cplx* tw = (const cplx*)g->twy.p;
    const cplx* W2 = kb->W2.p;
    cplx* W1 = kb->W1.p;
    void* args[] = {&kb->T, &tw, &W2, &W1, &L, &Lp};
    launch_ptr(ctx, g->ry->y_forward, dim3(cdiv(g->nx, L), kb->T.n_zc, nb), L * g->ry->T, reg_smem(g->ry), args);
  } else {
    int L = g->Ly, Lp = L | 1;
    LAUNCH(ctx, k_y_forward, dim3(cdiv(g->nx, L), kb->T.n_zc, nb), FFT_THREADS, smem_for(g->ny, L),
           kb->T, g->py, (const cplx*)g->twy.p, (const cplx*)kb->W2.p, kb->W1.p, L, Lp);
  }
  if ((g->rx && kb->T.ranges_ok)) {
    int L = reg_L(g->rx), Lp = L + 1;
    const cplx* tw = (const cplx*)g->twx.p;
    const cplx* W1 = kb->W1.p;
    void* args[] = {&kb->T, &tw, &W1, &out, &ldout, &scale, &kin, &psi, &ldpsi, &accumulate, &L, &Lp};
    launch_ptr(ctx, g->rx->x_to_sphere, dim3(cdiv(kb->T.n_cols, L), nb), L * g->rx->T, reg_smem(g->rx) + 5 * L * sizeof(int), args);
  } else {
    int L = g->Lx, Lp = L | 1;
    LAUNCH(ctx, k_x_to_sphere, dim3(cdiv(kb->T.n_cols, L), nb), FFT_THREADS, smem_for(g->nx, L), kb->T,
           g->px, (const cplx*)g->twx.p, (const cplx*)kb->W1.p, out, ldout, scale, kin, psi, ldpsi,
           accumulate, L, Lp);
  }
}

// hpsi (+)= FFT[V IFFT psi] (+ kin psi), batched over bands in chunks.
void kb_apply_local_kinetic(dftk_b200_kblock* kb, const cplx* psi, cplx* hpsi, int64_t n_bands,
                            bool with_local, bool with_kin, bool accumulate) {
  dftk_b200_grid* g = kb->grid;
  dftk_b200_ctx* ctx = g->ctx;
  if (n_bands == 0) return;
  if (!with_local) {
    scale_kin_add(ctx, psi, hpsi, with_kin ? kb->kin.p : nullptr, kb->n_pw, n_bands, accumulate);
    return;
  }
  REQUIRE(kb->has_V, "apply_h: local potential not set (dftk_b200_kblock_set_potential)");
  const bool fused = kb_yz_fused(kb);
  const int chunk = band_chunk_for(kb, n_bands, !fused);
  for (int64_t b0 = 0; b0 < n_bands; b0 += chunk) {
    int nb = (int)std::min<int64_t>(chunk, n_bands - b0);
    const cplx* p = psi + b0 * kb->n_pw;
    if (fused) {
      // x-major W1 [band][x][col]: sphere -> x lines, y-z in shared memory per x line, x lines -> sphere
      kb->W1.ensure((size_t)nb * kb->Th.n_cols * g->nx);
      int L = reg_L(g->rx), Lp = L + 1;
      const size_t sm_x = reg_smem(g->rx) + 5 * L * sizeof(int);
      const cplx* twx = (const cplx*)g->twx.p;
      const cplx* twy = (const cplx*)g->twy.p;
      cplx* W1 = kb->W1.p;
      int64_t ld = kb->n_pw;
      void* a1[] = {&kb->T, &twx, &p, &ld, &W1, &L, &Lp};
      launch_ptr(ctx, g->rx->sphere_to_xt, dim3(cdiv(kb->T.n_cols, L), nb), L * g->rx->T, sm_x, a1);
      const double* Vt = kb->Vtp();
      void* a2[] = {&kb->T, &twy, &W1, &Vt, &nb};
      // persistent: as many CTAs as are resident at once (one per SM at the larger grids), each loops over items
      const size_t sm_yz = yz_smem(g->ny, kb->T.n_zc);
      int per_sm = 1;
      CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, g->ry->yz_apply, g->ry->yz_threads, sm_yz));
      const unsigned yz_ctas = (unsigned)std::min<int64_t>((int64_t)nb * g->nx, (int64_t)std::max(per_sm, 1) * ctx->sm_count);
      launch_ptr(ctx, g->ry->yz_apply, dim3(yz_ctas), g->ry->yz_threads, sm_yz, a2);
      cplx* out = hpsi + b0 * kb->n_pw;
      double scale = 1.0;
      const double* kin = with_kin ? kb->kin.p : nullptr;
      int acc = accumulate ? 1 : 0;
      void* a3[] = {&kb->T, &twx, &W1, &out, &ld, &scale, &kin, &p, &ld, &acc, &L, &Lp};
      launch_ptr(ctx, g->rx->xt_to_sphere, dim3(cdiv(kb->T.n_cols, L), nb), L * g->rx->T, sm_x, a3);
      continue;
    }
    kb_sphere_to_planes(kb, p, kb->n_pw, nb);
    if ((g->rz && kb->T.ranges_ok)) {
      int L = reg_L(g->rz), Lp = L + 1;
      const cplx* tw = (const cplx*)g->twz.p;
      cplx* W2 = kb->W2.p;
      const double* V = kb->Vp();
      void* args[] = {&kb->T, &tw, &W2, &V, &L, &Lp};
      const size_t sm_pipe = reg_smem(g->rz) / 2 + 2 * (size_t)kb->T.n_zc * L * sizeof(cplx);
      const int64_t n_tiles = (int64_t)cdiv(g->nx, L) * g->ny * nb;
      if (ctx->z_pipeline && sm_pipe <= 100 * 1024 && n_tiles >= 2 * (int64_t)ctx->sm_count) {
        // persistent CTAs (as many as fit an SM by shared memory, at most 4), each loops over tiles with the next tile's
        // input in flight (cp.async) while the current one is transformed
        int per_sm = (int)std::min<size_t>(4, (size_t)(220 * 1024) / sm_pipe);
        unsigned grid = (unsigned)std::min<int64_t>(n_tiles, (int64_t)per_sm * ctx->sm_count);
        void* pargs[] = {&kb->T, &tw, &W2, &V, &nb};
        launch_ptr(ctx, g->rz->z_apply_pipe, dim3(grid), L * g->rz->T, sm_pipe, pargs);
      } else {
        // single (aliased) exchange buffer on the device, cf. DFTK_Z_ALIAS in fft_reg.cuh
        launch_ptr(ctx, g->rz->z_apply, dim3(cdiv(g->nx, L), g->ny, nb), L * g->rz->T, reg_smem(g->rz) / 2, args);
      }
    } else {
      int L = g->Lz, Lp = L | 1;
      LAUNCH(ctx, k_z_apply_potential, dim3(cdiv(g->nx, L), g->ny, nb), FFT_THREADS, smem_for(g->nz, L),
             kb->T, g->pz, (const cplx*)g->twz.p, kb->W2.p, (const double*)kb->Vp(), L, Lp);
    }
    kb_planes_to_sphere(kb, hpsi + b0 * kb->n_pw, kb->n_pw, nb, 1.0, with_kin ? kb->kin.p : nullptr, p,
                        kb->n_pw, accumulate ? 1 : 0);
  }
}

bool kb_apply_local_kinetic_multi(int n, dftk_b200_kblock* const* kbs, const cplx* const* psi, cplx* const* hpsi,
                                  const int* n_bands, DescRing& ring) {
  if (n <= 0) return true;
  dftk_b200_grid* g = kbs[0]->grid;
  dftk_b200_ctx* ctx = g->ctx;
  if (!(g->rx && g->ry && g->rz)) return false;
  int total = 0, max_cols = 0, max_zc = 0;
  for (int i = 0; i < n; ++i) {
    dftk_b200_kblock* kb = kbs[i];
    if (kb->grid != g || !kb->T.ranges_ok || !kb->has_V || !kb->has_kin || n_bands[i] <= 0) return false;
    // whole band blocks in one chunk (the small problems this path serves have <= 32 bands)
    if (band_chunk_for(kb, n_bands[i]) < n_bands[i]) return false;
    total += n_bands[i];
    max_cols = std::max(max_cols, kb->T.n_cols);
    max_zc = std::max(max_zc, kb->T.n_zc);
  }
  if (total > 65535) return false;
  std::vector<FftMultiItem> items(n);
  std::vector<int2> bandmap(total);
  int b = 0;
  for (int i = 0; i < n; ++i) {
    dftk_b200_kblock* kb = kbs[i];
    ensure_scratch(kb, n_bands[i]);
    FftMultiItem& it = items[i];
    it.T = kb->T;
    it.psi = psi[i];
    it.ldpsi = kb->n_pw;
    it.W1 = kb->W1.p;
    it.W2 = kb->W2.p;
    it.V = kb->Vp();
    it.wts = nullptr;
    it.nb = n_bands[i];
    it.out = hpsi[i];
    it.ldout = kb->n_pw;
    it.kin = kb->kin.p;
    for (int l = 0; l < n_bands[i]; ++l) bandmap[b++] = make_int2(i, l);
  }
  ring.reserve(DescRing::padded(items) + DescRing::padded(bandmap), ctx->stream);
  const FftMultiItem* d_items = ring.put(items, ctx->stream);
  const int2* d_map = ring.put(bandmap, ctx->stream);
  {
    int L = reg_L(g->rx), Lp = L + 1;
    const cplx* tw = (const cplx*)g->twx.p;
    void* args[] = {&d_items, &d_map, &tw, &L, &Lp};
    launch_ptr(ctx, g->rx->m_sphere_to_x, dim3(cdiv(max_cols, L), total), L * g->rx->T, reg_smem(g->rx) + 5 * L * sizeof(int), args);
  }
  {
    int L = reg_L(g->ry), Lp = L + 1;
    const cplx* tw = (const cplx*)g->twy.p;
    void* args[] = {&d_items, &d_map, &tw, &L, &Lp};
    launch_ptr(ctx, g->ry->m_y_backward, dim3(cdiv(g->nx, L), max_zc, total), L * g->ry->T, reg_smem(g->ry), args);
  }
  {
    int L = reg_L(g->rz), Lp = L + 1;
    const cplx* tw = (const cplx*)g->twz.p;
    void* args[] = {&d_items, &d_map, &tw, &L, &Lp};
    launch_ptr(ctx, g->rz->m_z_apply, dim3(cdiv(g->nx, L), g->ny, total), L * g->rz->T, reg_smem(g->rz) / 2, args);
  }
  {
    int L = reg_L(g->ry), Lp = L + 1;
    const cplx* tw = (const cplx*)g->twy.p;
    void* args[] = {&d_items, &d_map, &tw, &L, &Lp};
    launch_ptr(ctx, g->ry->m_y_forward, dim3(cdiv(g->nx, L), max_zc, total), L * g->ry->T, reg_smem(g->ry), args);
  }
  {
    int L = reg_L(g->rx), Lp = L + 1;
    const cplx* tw = (const cplx*)g->twx.p;
    void* args[] = {&d_items, &d_map, &tw, &L, &Lp};
    launch_ptr(ctx, g->rx->m_x_to_sphere, dim3(cdiv(max_cols, L), total), L * g->rx->T, reg_smem(g->rx) + 5 * L * sizeof(int), args);
  }
  return true;
}

bool kb_density_accumulate_multi(int n, dftk_b200_kblock* const* kbs, const cplx* const* psi, const double* occ_w_host,
                                 int64_t ld_w, const int* n_bands, double* rho) {
  if (n <= 0) return true;
  dftk_b200_grid* g = kbs[0]->grid;
  dftk_b200_ctx* ctx = g->ctx;
  if (!(g->rx && g->ry && g->rz)) return false;
  int total = 0, max_cols = 0, max_zc = 0;
  for (int i = 0; i < n; ++i) {
    dftk_b200_kblock* kb = kbs[i];
    if (kb->grid != g || !kb->T.ranges_ok || kb->spin < 0 || kb->spin > 1) return false;
    if (n_bands[i] > 0 && band_chunk_for(kb, n_bands[i]) < n_bands[i]) return false;
    total += n_bands[i];
    max_cols = std::max(max_cols, kb->T.n_cols);
    max_zc = std::max(max_zc, kb->T.n_zc);
  }
  if (total == 0) return true;
  if (total > 65535) return false;
  // device copies: weights (scaled by ifft_norm^2), items, band map -- staged through the context's descriptor ring
  std::vector<double> w;
  std::vector<FftMultiItem> items;
  std::vector<int2> bandmap;
  const double nrm = g->ifft_norm * g->ifft_norm;
  for (int i = 0; i < n; ++i) {
    dftk_b200_kblock* kb = kbs[i];
    if (n_bands[i] <= 0) continue;
    ensure_scratch(kb, n_bands[i]);
    FftMultiItem it{};
    it.T = kb->T;
    it.psi = psi[i];
    it.ldpsi = kb->n_pw;
    it.W1 = kb->W1.p;
    it.W2 = kb->W2.p;
    it.nb = n_bands[i];
    it.V = nullptr;
    it.out = nullptr;
    it.kin = (const double*)(intptr_t)kb->spin;      // spin channel of the block rides in an unused pointer slot
    for (int l = 0; l < n_bands[i]; ++l) {
      w.push_back(occ_w_host[(size_t)i * ld_w + l] * nrm);
      bandmap.push_back(make_int2((int)items.size(), l));
    }
    items.push_back(it);
  }
  DescRing& ring = ctx->slot[0].ring;
  ring.reserve(DescRing::padded(w) + DescRing::padded(items) + DescRing::padded(bandmap), ctx->stream);
  const double* d_w = ring.put(w, ctx->stream);
  for (auto& it : items) {
    it.wts = d_w;
    d_w += it.nb;
  }
  const FftMultiItem* c_items = ring.put(items, ctx->stream);
  const int2* c_map = ring.put(bandmap, ctx->stream);
  {
    int L = reg_L(g->rx), Lp = L + 1;
    const cplx* tw = (const cplx*)g->twx.p;
    void* args[] = {&c_items, &c_map, &tw, &L, &Lp};
    launch_ptr(ctx, g->rx->m_sphere_to_x, dim3(cdiv(max_cols, L), total), L * g->rx->T, reg_smem(g->rx) + 5 * L * sizeof(int), args);
  }
  {
    int L = reg_L(g->ry), Lp = L + 1;
    const cplx* tw = (const cplx*)g->twy.p;
    void* args[] = {&c_items, &c_map, &tw, &L, &Lp};
    launch_ptr(ctx, g->ry->m_y_backward, dim3(cdiv(g->nx, L), max_zc, total), L * g->ry->T, reg_smem(g->ry), args);
  }
  int n_items = (int)items.size();
  for (int spin = 0; spin < 2; ++spin) {
    bool any = false;
    for (auto& it : items) any = any || (int)(intptr_t)it.kin == spin;
    if (!any) continue;
    int L = reg_L(g->rz), Lp = L + 1;
    const cplx* tw = (const cplx*)g->twz.p;
    double* r = rho + (size_t)spin * g->N;
    size_t sm = reg_smem(g->rz) + (size_t)g->nz * L * sizeof(double);
    void* args[] = {&c_items, &n_items, &spin, &tw, &r, &L, &Lp};
    launch_ptr(ctx, g->rz->m_z_density, dim3(cdiv(g->nx, L), g->ny), L * g->rz->T, sm, args);
  }
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  ring.rewind();
  return true;
}

void kb_sphere_to_real(dftk_b200_kblock* kb, const cplx* psi, cplx* cube, int64_t n_bands, double scale) {
  dftk_b200_grid* g = kb->grid;
  dftk_b200_ctx* ctx = g->ctx;
  const int chunk = band_chunk_for(kb, n_bands);
  for (int64_t b0 = 0; b0 < n_bands; b0 += chunk) {
    int nb = (int)std::min<int64_t>(chunk, n_bands - b0);
    kb_sphere_to_planes(kb, psi + b0 * kb->n_pw, kb->n_pw, nb);
    if ((g->rz && kb->T.ranges_ok)) {
      int L = reg_L(g->rz), Lp = L + 1;
      const cplx* tw = (const cplx*)g->twz.p;
      const cplx* W2 = kb->W2.p;
      cplx* cb = cube + b0 * g->N;
      void* args[] = {&kb->T, &tw, &W2, &cb, &scale, &L, &Lp};
      launch_ptr(ctx, g->rz->z_to_cube, dim3(cdiv(g->nx, L), g->ny, nb), L * g->rz->T, reg_smem(g->rz), args);
    } else {
      int L = g->Lz, Lp = L | 1;
      LAUNCH(ctx, k_z_to_cube, dim3(cdiv(g->nx, L), g->ny, nb), FFT_THREADS, smem_for(g->nz, L), kb->T,
             g->pz, (const cplx*)g->twz.p, (const cplx*)kb->W2.p, cube + b0 * g->N, scale, L, Lp);
    }
  }
}

void kb_real_to_sphere(dftk_b200_kblock* kb, const cplx* cube, cplx* out, int64_t n_bands, double scale) {
  dftk_b200_grid* g = kb->grid;
  dftk_b200_ctx* ctx = g->ctx;
  const int chunk = band_chunk_for(kb, n_bands);
  for (int64_t b0 = 0; b0 < n_bands; b0 += chunk) {
    int nb = (int)std::min<int64_t>(chunk, n_bands - b0);
    ensure_scratch(kb, nb);
    if ((g->rz && kb->T.ranges_ok)) {
      int L = reg_L(g->rz), Lp = L + 1;
      const cplx* tw = (const cplx*)g->twz.p;
      const cplx* cb = cube + b0 * g->N;
      cplx* W2 = kb->W2.p;
      void* args[] = {&kb->T, &tw, &cb, &W2, &L, &Lp};
      launch_ptr(ctx, g->rz->z_from_cube, dim3(cdiv(g->nx, L), g->ny, nb), L * g->rz->T, reg_smem(g->rz), args);
    } else {
      int L = g->Lz, Lp = L | 1;
      LAUNCH(ctx, k_z_from_cube, dim3(cdiv(g->nx, L), g->ny, nb), FFT_THREADS, smem_for(g->nz, L), kb->T,
             g->pz, (const cplx*)g->twz.p, cube + b0 * g->N, kb->W2.p, L, Lp);
    }
    kb_planes_to_sphere(kb, out + b0 * kb->n_pw, kb->n_pw, nb, scale, nullptr, nullptr, 0, 0);
  }
}

// rho += sum_n occ_w[n] |IFFT psi_n|^2 * ifft_norm^2      (src/densities.jl:38-41)
void kb_density_accumulate(dftk_b200_kblock* kb, const cplx* psi, const double* occ_w_host,
                           int64_t n_bands, double* rho) {
  dftk_b200_grid* g = kb->grid;
  dftk_b200_ctx* ctx = g->ctx;
  if (n_bands == 0) return;
  std::vector<double> w(n_bands);
  for (int64_t i = 0; i < n_bands; ++i) w[i] = occ_w_host[i] * g->ifft_norm * g->ifft_norm;
  DescRing& ring = ctx->slot[0].ring;
  const double* w_dev = ring.put(w, ctx->stream);
  const int chunk = band_chunk_for(kb, n_bands);
  for (int64_t b0 = 0; b0 < n_bands; b0 += chunk) {
    int nb = (int)std::min<int64_t>(chunk, n_bands - b0);
    kb_sphere_to_planes(kb, psi + b0 * kb->n_pw, kb->n_pw, nb);
    if ((g->rz && kb->T.ranges_ok)) {
      int L = reg_L(g->rz), Lp = L + 1;
      const cplx* tw = (const cplx*)g->twz.p;
      const cplx* W2 = kb->W2.p;
      const double* wp = w_dev + b0;
      size_t sm = reg_smem(g->rz) + (size_t)g->nz * L * sizeof(double);
      void* args[] = {&kb->T, &tw, &W2, &wp, &nb, &rho, &L, &Lp};
      launch_ptr(ctx, g->rz->z_density, dim3(cdiv(g->nx, L), g->ny), L * g->rz->T, sm, args);
    } else {
      int L = g->Lz, Lp = L | 1;
      size_t sm = smem_for(g->nz, L) + (size_t)g->nz * L * sizeof(double);
      LAUNCH(ctx, k_z_density, dim3(cdiv(g->nx, L), g->ny), FFT_THREADS, sm, kb->T, g->pz,
             (const cplx*)g->twz.p, (const cplx*)kb->W2.p, w_dev + b0, nb, rho, L, Lp);
    }
  }
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  ring.rewind();
}

}  // namespace dftk
