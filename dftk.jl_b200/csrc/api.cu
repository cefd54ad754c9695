// extern "C" entry points of libdftk_b200 (see include/dftk_b200.h for the contract).
#include <mutex>
#include "structs.cuh"
#include "xc_core.cuh"

using namespace dftk;

static std::string g_last_error;
static std::mutex g_err_mutex;

int dftk::record_error(dftk_b200_ctx* ctx, int code, const std::string& msg) {
  {
    std::lock_guard<std::mutex> lk(g_err_mutex);
    g_last_error = msg;
  }
  if (ctx) ctx->last_error = msg;
  return code;
}

// Stage a (possibly host) input buffer onto the device.  Returns a device pointer.
static const void* stage_in(dftk_b200_ctx* ctx, const void* p, size_t bytes, DevBuf<char>& buf) {
  if (is_device_ptr(p)) return p;
  buf.ensure(bytes);
  CUDA_CHECK(cudaMemcpyAsync(buf.p, p, bytes, cudaMemcpyHostToDevice, ctx->stream));
  return buf.p;
}

// Runs `fn(dev_in, dev_out)` with psi-like input/outputs that may live on the host.
template <class F>
static void with_staging(dftk_b200_ctx* ctx, const void* in, size_t in_bytes, void* out, size_t out_bytes,
                         bool out_is_inout, F fn) {
  const void* din = stage_in(ctx, in, in_bytes, ctx->stage_in);
  if (is_device_ptr(out)) {
    fn(din, out);
    return;
  }
  ctx->stage_out.ensure(out_bytes);
  if (out_is_inout) CUDA_CHECK(cudaMemcpyAsync(ctx->stage_out.p, out, out_bytes, cudaMemcpyHostToDevice, ctx->stream));
  fn(din, (void*)ctx->stage_out.p);
  CUDA_CHECK(cudaMemcpyAsync(out, ctx->stage_out.p, out_bytes, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
}

// Host-resident psi/hpsi: overlap the PCIe copies with the kernels in chunks of bands (double buffered).
static void apply_terms_host_pipelined(dftk_b200_kblock* kb, const cplx* psi_h, cplx* hpsi_h, int64_t n_bands,
                                       bool loc, bool kinp, bool nl) {
  dftk_b200_ctx* ctx = kb->grid->ctx;
  if (!ctx->s_in) {
    CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->s_in, cudaStreamNonBlocking));
    CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->s_out, cudaStreamNonBlocking));
    for (int i = 0; i < 2; ++i) {
      CUDA_CHECK(cudaEventCreateWithFlags(&ctx->ev_in[i], cudaEventDisableTiming));
      CUDA_CHECK(cudaEventCreateWithFlags(&ctx->ev_comp[i], cudaEventDisableTiming));
      CUDA_CHECK(cudaEventCreateWithFlags(&ctx->ev_out[i], cudaEventDisableTiming));
    }
  }
  const int64_t chunk = std::min<int64_t>(n_bands, 128);
  const size_t cbytes = (size_t)chunk * kb->n_pw * sizeof(cplx);
  for (int i = 0; i < 2; ++i) {
    ctx->pipe_in[i].ensure(cbytes);
    ctx->pipe_out[i].ensure(cbytes);
  }
  int it = 0;
  for (int64_t b0 = 0; b0 < n_bands; b0 += chunk, ++it) {
    const int buf = it & 1;
    const int64_t nb = std::min<int64_t>(chunk, n_bands - b0);
    const size_t bytes = (size_t)nb * kb->n_pw * sizeof(cplx);
    cplx* din = (cplx*)ctx->pipe_in[buf].p;
    cplx* dout = (cplx*)ctx->pipe_out[buf].p;
    // the input buffer may be overwritten once the compute that read it (two chunks ago) has finished
    if (it >= 2) CUDA_CHECK(cudaStreamWaitEvent(ctx->s_in, ctx->ev_comp[buf], 0));
    CUDA_CHECK(cudaMemcpyAsync(din, psi_h + b0 * kb->n_pw, bytes, cudaMemcpyHostToDevice, ctx->s_in));
    CUDA_CHECK(cudaEventRecord(ctx->ev_in[buf], ctx->s_in));
    CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->ev_in[buf], 0));
    if (it >= 2) CUDA_CHECK(cudaStreamWaitEvent(ctx->stream, ctx->ev_out[buf], 0));   // output buffer drained
    if (loc || kinp) kb_apply_local_kinetic(kb, din, dout, nb, loc, kinp, false);
    else CUDA_CHECK(cudaMemsetAsync(dout, 0, bytes, ctx->stream));
    if (nl) kb_apply_nonlocal(kb, din, dout, nb);
    CUDA_CHECK(cudaEventRecord(ctx->ev_comp[buf], ctx->stream));
    CUDA_CHECK(cudaStreamWaitEvent(ctx->s_out, ctx->ev_comp[buf], 0));
    CUDA_CHECK(cudaMemcpyAsync(hpsi_h + b0 * kb->n_pw, dout, bytes, cudaMemcpyDeviceToHost, ctx->s_out));
    CUDA_CHECK(cudaEventRecord(ctx->ev_out[buf], ctx->s_out));
  }
  CUDA_CHECK(cudaStreamSynchronize(ctx->s_out));
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
}

extern "C" {

const char* dftk_b200_last_error(dftk_b200_ctx* ctx) {
  if (ctx) return ctx->last_error.c_str();
  return g_last_error.c_str();
}

static int ctx_create_common(int device, dftk_b200_ctx** out) {
  REQUIRE(out != nullptr, "ctx_create: out is NULL");
  int ndev = 0;
  CUDA_CHECK(cudaGetDeviceCount(&ndev));
  REQUIRE(device >= 0 && device < ndev, "ctx_create: no such CUDA device (the product path has no CPU fallback)");
  CUDA_CHECK(cudaSetDevice(device));
  cudaDeviceProp prop;
  CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
  REQUIRE(prop.major == 9 && prop.minor == 0, "libdftk_b200 is built for sm_90a (Hopper) only");
  dftk_b200_ctx* c = new dftk_b200_ctx();
  c->device = device;
  c->sm_count = prop.multiProcessorCount;
  CUDA_CHECK(cudaDeviceGetAttribute(&c->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  c->stream = 0;  // legacy default stream: ordered with the caller's default-stream work
  CUBLAS_CHECK(cublasCreate(&c->cublas));
  CUBLAS_CHECK(cublasSetStream(c->cublas, c->stream));
  CUSOLVER_CHECK(cusolverDnCreate(&c->cusolver));
  CUSOLVER_CHECK(cusolverDnSetStream(c->cusolver, c->stream));
  fft_set_attributes();
  reg_set_attributes(c->smem_optin);
  blas_set_attributes();
  i8tc2_set_attributes();
  lobpcg_set_attributes();
  *out = c;
  return 0;
}

int dftk_b200_ctx_create(int device, dftk_b200_ctx** out) {
  API_BEGIN
  ctx_create_common(device, out);
  API_END(nullptr)
}

int dftk_b200_nccl_unique_id(void* out128) {
  API_BEGIN
  REQUIRE(out128 != nullptr, "nccl_unique_id: out is NULL");
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId size");
  ncclUniqueId id;
  NCCL_CHECK(ncclGetUniqueId(&id));
  memcpy(out128, &id, 128);
  API_END(nullptr)
}

int dftk_b200_ctx_create_dist(int device, const void* nccl_unique_id, int rank, int nranks,
                              dftk_b200_ctx** out) {
  API_BEGIN
  REQUIRE(nccl_unique_id != nullptr && nranks >= 1 && rank >= 0 && rank < nranks, "ctx_create_dist: bad arguments");
  ctx_create_common(device, out);
  ncclUniqueId id;
  memcpy(&id, nccl_unique_id, 128);
  (*out)->rank = rank;
  (*out)->nranks = nranks;
  NCCL_CHECK(ncclCommInitRank(&(*out)->nccl, nranks, id, rank));
  API_END(nullptr)
}

int dftk_b200_ctx_destroy(dftk_b200_ctx* ctx) {
  if (!ctx) return DFTK_B200_OK;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  if (ctx->s_in) {
    cudaStreamDestroy(ctx->s_in);
    cudaStreamDestroy(ctx->s_out);
    for (int i = 0; i < 2; ++i) {
      cudaEventDestroy(ctx->ev_in[i]);
      cudaEventDestroy(ctx->ev_comp[i]);
      cudaEventDestroy(ctx->ev_out[i]);
    }
  }
  for (int i = 0; i < 2; ++i)
    if (ctx->batch_streams[i]) cudaStreamDestroy(ctx->batch_streams[i]);
  if (ctx->nccl) ncclCommDestroy(ctx->nccl);
  if (ctx->cublas) cublasDestroy(ctx->cublas);
  if (ctx->solver_params) cusolverDnDestroyParams(ctx->solver_params);
  if (ctx->cusolver) cusolverDnDestroy(ctx->cusolver);
  delete ctx;
  return DFTK_B200_OK;
}

int dftk_b200_sync(dftk_b200_ctx* ctx) {
  API_BEGIN
  REQUIRE(ctx, "sync: ctx is NULL");
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  API_END(ctx)
}

int dftk_b200_ctx_set_stream(dftk_b200_ctx* ctx, void* cuda_stream) {
  API_BEGIN
  REQUIRE(ctx, "ctx_set_stream: ctx is NULL");
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));        // nothing of ours may still be in flight on the old stream
  ctx->stream = (cudaStream_t)cuda_stream;
  CUBLAS_CHECK(cublasSetStream(ctx->cublas, ctx->stream));
  CUSOLVER_CHECK(cusolverDnSetStream(ctx->cusolver, ctx->stream));
  API_END(ctx)
}

int dftk_b200_mem_info(dftk_b200_ctx* ctx, int64_t* free_bytes, int64_t* total_bytes) {
  API_BEGIN
  size_t f = 0, t = 0;
  CUDA_CHECK(cudaMemGetInfo(&f, &t));
  if (free_bytes) *free_bytes = (int64_t)f;
  if (total_bytes) *total_bytes = (int64_t)t;
  API_END(ctx)
}

int64_t dftk_b200_launch_count(dftk_b200_ctx* ctx, int reset) {
  if (!ctx) return -1;
  int64_t v = ctx->launches;
  if (reset) ctx->launches = 0;
  return v;
}

double dftk_b200_lobpcg_flops(dftk_b200_ctx* ctx, int reset) {
  if (!ctx) return -1.0;
  const double v = ctx->lobpcg_flops;
  if (reset) ctx->lobpcg_flops = 0.0;
  return v;
}

int64_t dftk_b200_sync_count(dftk_b200_ctx* ctx, int reset) {
  if (!ctx) return -1;
  int64_t v = ctx->batch_rounds;
  if (reset) ctx->batch_rounds = 0;
  return v;
}

int dftk_b200_set_option(dftk_b200_ctx* ctx, const char* name, int64_t value) {
  API_BEGIN
  REQUIRE(ctx && name, "set_option: NULL argument");
  std::string n(name);
  if (n == "gemm_backend") {
    REQUIRE(value == 0 || value == 1 || value == 2 || value == 4, "set_option: gemm_backend must be 0, 1, 2 or 4");
    ctx->gemm_backend = (int)value;
  }
  else if (n == "band_chunk") ctx->band_chunk = (int)value;
  else if (n == "gemm_stages") ctx->gemm_stages = (int)std::min<int64_t>(4, std::max<int64_t>(2, value));
  else if (n == "small_dense") ctx->small_dense = (int)value;
  else if (n == "i8_min_rows") ctx->i8_min_rows = value;
  else if (n == "z_pipeline") ctx->z_pipeline = (int)value;
  else if (n == "batch_pipeline") ctx->batch_pipeline = (int)value;
  else if (n == "force_svd_fallback") ctx->force_svd_fallback = (int)value;
  else if (n == "fft_engine") ctx->fft_engine = (int)value;  // 0 = register two-pass where available, 1 = generic
  else throw Error(DFTK_B200_EINVAL, "set_option: unknown option " + n);
  API_END(ctx)
}

// ------------------------------------------------------------------ grid
int dftk_b200_grid_create(dftk_b200_ctx* ctx, int nx, int ny, int nz, double unit_cell_volume,
                          dftk_b200_grid** out) {
  API_BEGIN
  REQUIRE(ctx && out, "grid_create: NULL argument");
  REQUIRE(nx >= 1 && ny >= 1 && nz >= 1 && unit_cell_volume > 0, "grid_create: bad size / volume");
  REQUIRE(ny <= 65535 && nz <= 65535, "grid_create: axis too long");
  dftk_b200_grid* g = new dftk_b200_grid();
  g->ctx = ctx;
  g->nx = nx;
  g->ny = ny;
  g->nz = nz;
  g->N = (int64_t)nx * ny * nz;
  g->omega = unit_cell_volume;
  g->ifft_norm = 1.0 / std::sqrt(unit_cell_volume);          // src/fft.jl:87
  g->fft_norm = std::sqrt(unit_cell_volume) / (double)g->N;  // src/fft.jl:88
  try {
    g->px = make_plan(nx);
    g->py = make_plan(ny);
    g->pz = make_plan(nz);
    g->Lx = choose_lines(nx);
    g->Ly = choose_lines(ny);
    g->Lz = choose_lines(nz);
    if (ctx->fft_engine == 0) {
      g->rx = reg_kernels_for(nx);
      g->ry = reg_kernels_for(ny);
      g->rz = reg_kernels_for(nz);
    }
    auto tx = make_twiddles(nx), ty = make_twiddles(ny), tz = make_twiddles(nz);
    g->twx.upload(tx.data(), tx.size(), ctx->stream);
    g->twy.upload(ty.data(), ty.size(), ctx->stream);
    g->twz.upload(tz.data(), tz.size(), ctx->stream);
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  } catch (...) {
    delete g;
    throw;
  }
  *out = g;
  API_END(ctx)
}

int dftk_b200_grid_destroy(dftk_b200_grid* grid) {
  delete grid;
  return DFTK_B200_OK;
}

int dftk_b200_fft_cube(dftk_b200_grid* grid, void* data, int direction, int64_t batch) {
  dftk_b200_ctx* ctx = grid ? grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(grid && data, "fft_cube: NULL argument");
  REQUIRE(direction == 1 || direction == -1, "fft_cube: direction must be +1 (backward) or -1 (forward)");
  size_t bytes = (size_t)grid->N * batch * sizeof(cplx);
  if (is_device_ptr(data)) {
    fft_cube_inplace(grid, (cplx*)data, direction, batch);
  } else {
    cplx* d = (cplx*)stage_in(ctx, data, bytes, ctx->stage_in);
    fft_cube_inplace(grid, d, direction, batch);
    CUDA_CHECK(cudaMemcpyAsync(data, d, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  }
  API_END(ctx)
}

// ------------------------------------------------------------------ k-block
int dftk_b200_kblock_create(dftk_b200_grid* grid, int64_t n_pw, const int64_t* mapping,
                            const double* kin, int64_t n_proj, const void* P, const double* D, int spin,
                            double kweight, dftk_b200_kblock** out) {
  dftk_b200_ctx* ctx = grid ? grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(grid && mapping && out, "kblock_create: NULL argument");
  REQUIRE(n_pw >= 1 && n_pw <= grid->N, "kblock_create: n_pw out of range");
  REQUIRE(n_proj >= 0 && (n_proj == 0 || (P && D)), "kblock_create: projectors missing");
  std::vector<int64_t> map_h(n_pw);
  CUDA_CHECK(cudaMemcpy(map_h.data(), mapping, n_pw * sizeof(int64_t), cudaMemcpyDefault));
  dftk_b200_kblock* kb = new dftk_b200_kblock();
  try {
    kb->grid = grid;
    kb->n_pw = n_pw;
    kb->n_proj = n_proj;
    kb->spin = spin;
    kb->kweight = kweight;
    kb->Th = build_sphere_tables(grid->nx, grid->ny, grid->nz, n_pw, map_h.data());
    kb->map_h = map_h;
    const SphereTablesHost& H = kb->Th;
    cudaStream_t s = ctx->stream;
    kb->d_col_start.upload(H.col_start.data(), H.col_start.size(), s);
    kb->d_col_cnt.upload(H.col_cnt.data(), H.col_cnt.size(), s);
    kb->d_slot_ix.upload(H.slot_ix.data(), H.slot_ix.size(), s);
    kb->d_slot_src.upload(H.slot_src.data(), H.slot_src.size(), s);
    kb->d_zlist.upload(H.zlist.data(), H.zlist.size(), s);
    kb->d_colmap.upload(H.colmap.data(), H.colmap.size(), s);
    kb->d_zc_of.upload(H.zc_of.data(), H.zc_of.size(), s);
    kb->d_pl_s0.upload(H.pl_s0.data(), H.pl_s0.size(), s);
    kb->d_pl_n0.upload(H.pl_n0.data(), H.pl_n0.size(), s);
    kb->d_pl_s1.upload(H.pl_s1.data(), H.pl_s1.size(), s);
    kb->d_pl_n1.upload(H.pl_n1.data(), H.pl_n1.size(), s);
    kb->d_pl_col0.upload(H.pl_col0.data(), H.pl_col0.size(), s);
    kb->d_cx_s0.upload(H.cx_s0.data(), H.cx_s0.size(), s);
    kb->d_cx_n0.upload(H.cx_n0.data(), H.cx_n0.size(), s);
    kb->d_cx_s1.upload(H.cx_s1.data(), H.cx_s1.size(), s);
    kb->d_cx_n1.upload(H.cx_n1.data(), H.cx_n1.size(), s);
    SphereTablesX& T = kb->T;
    T.nx = H.nx; T.ny = H.ny; T.nz = H.nz; T.n_pw = n_pw; T.n_cols = H.n_cols; T.cnt_max = H.cnt_max;
    T.n_zc = H.n_zc; T.col_start = kb->d_col_start.p; T.col_cnt = kb->d_col_cnt.p;
    T.slot_ix = kb->d_slot_ix.p; T.slot_src = kb->d_slot_src.p; T.zlist = kb->d_zlist.p;
    T.colmap = kb->d_colmap.p;
    T.zc_of = kb->d_zc_of.p;
    T.ranges_ok = H.ranges_ok; T.z_s0 = H.z_s0; T.z_n0 = H.z_n0; T.z_s1 = H.z_s1; T.z_n1 = H.z_n1;
    T.pl_s0 = kb->d_pl_s0.p; T.pl_n0 = kb->d_pl_n0.p; T.pl_s1 = kb->d_pl_s1.p; T.pl_n1 = kb->d_pl_n1.p;
    T.pl_col0 = kb->d_pl_col0.p;
    T.cx_s0 = kb->d_cx_s0.p; T.cx_n0 = kb->d_cx_n0.p; T.cx_s1 = kb->d_cx_s1.p; T.cx_n1 = kb->d_cx_n1.p;
    if (kin) {
      kb->kin.ensure(n_pw);
      CUDA_CHECK(cudaMemcpyAsync(kb->kin.p, kin, n_pw * sizeof(double), cudaMemcpyDefault, s));
      kb->has_kin = true;
    }
    if (n_proj > 0) {
      kb->P.ensure((size_t)n_pw * n_proj);
      CUDA_CHECK(cudaMemcpyAsync(kb->P.p, P, (size_t)n_pw * n_proj * sizeof(cplx), cudaMemcpyDefault, s));
      kb->D_host.resize((size_t)n_proj * n_proj);
      CUDA_CHECK(cudaMemcpy(kb->D_host.data(), D, (size_t)n_proj * n_proj * sizeof(double), cudaMemcpyDefault));
      std::vector<double> dc(2 * (size_t)n_proj * n_proj, 0.0);
      for (size_t i = 0; i < (size_t)n_proj * n_proj; ++i) dc[2 * i] = kb->D_host[i];
      kb->Dc.ensure((size_t)n_proj * n_proj);
      CUDA_CHECK(cudaMemcpyAsync(kb->Dc.p, dc.data(), dc.size() * sizeof(double), cudaMemcpyHostToDevice, s));
      if (n_proj <= 96) {      // SMALL_MAX_COLS of the batched small-matrix path (lobpcg_small.cuh)
        kb->PD.ensure((size_t)n_pw * n_proj);
        zgemm(ctx, 0, n_pw, n_proj, n_proj, make_double2(1, 0), kb->P.p, n_pw, kb->Dc.p, n_proj, make_double2(0, 0), kb->PD.p, n_pw);
      }
      kb_setup_fold(kb, map_h.data());
    }
    CUDA_CHECK(cudaStreamSynchronize(s));
  } catch (...) {
    delete kb;
    throw;
  }
  *out = kb;
  API_END(ctx)
}

int dftk_b200_kblock_destroy(dftk_b200_kblock* kb) {
  delete kb;
  return DFTK_B200_OK;
}

int dftk_b200_kblock_set_orbitals(dftk_b200_kblock* kb, int64_t n_orb, const void* Phi) {
  dftk_b200_ctx* ctx = kb ? kb->grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(kb && n_orb >= 0 && (n_orb == 0 || Phi), "kblock_set_orbitals: bad argument");
  const int64_t n_pw = kb->n_pw, np = kb->n_proj, n = np + n_orb;
  cudaStream_t s = ctx->stream;
  CUDA_CHECK(cudaStreamSynchronize(s));
  {
    // the new table [P | Φ]; the old one is freed when `old` leaves this scope (after the stream has drained)
    DevBuf<cplx> old;
    std::swap(old.p, kb->P.p);
    std::swap(old.cap, kb->P.cap);
    if (n > 0) {
      kb->P.ensure((size_t)n_pw * n);
      if (np) CUDA_CHECK(cudaMemcpyAsync(kb->P.p, old.p, (size_t)n_pw * np * sizeof(cplx), cudaMemcpyDeviceToDevice, s));
      if (n_orb)
        CUDA_CHECK(cudaMemcpyAsync(kb->P.p + n_pw * np, Phi, (size_t)n_pw * n_orb * sizeof(cplx), cudaMemcpyDefault, s));
    }
    kb->n_orb = n_orb;
    if (n_orb) {
      // D of the H apply: [D 0; 0 V] with V = 0 until kblock_set_orbital_coefficients
      kb->Dh.ensure((size_t)n * n);
      CUDA_CHECK(cudaMemsetAsync(kb->Dh.p, 0, (size_t)n * n * sizeof(cplx), s));
      if (np)
        CUDA_CHECK(cudaMemcpy2DAsync(kb->Dh.p, n * sizeof(cplx), kb->Dc.p, np * sizeof(cplx), np * sizeof(cplx), np,
                                     cudaMemcpyDeviceToDevice, s));
    } else {
      kb->Dh.release();
    }
    if (n > 0 && n <= 96) {      // SMALL_MAX_COLS of the batched small-matrix path (lobpcg_small.cuh)
      kb->PD.ensure((size_t)n_pw * n);
      kb_refresh_pd(kb, 0);
    } else {
      kb->PD.release();
    }
    // the INT8 planes of gemm_backend 4 describe the old table: prepared again at first use
    kb->i8_Pop = I8Operand{};
    // Löwdin keeps Φ(-q) = conj Φ(q) at time-reversal-invariant k (S is real there); checked like the projectors
    kb_setup_fold(kb, kb->map_h.data());
    CUDA_CHECK(cudaStreamSynchronize(s));
  }
  API_END(ctx)
}

int dftk_b200_kblock_fold_size(dftk_b200_kblock* kb, int64_t* n_half) {
  dftk_b200_ctx* ctx = kb ? kb->grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(kb && n_half, "kblock_fold_size: NULL argument");
  *n_half = kb->n_half;
  API_END(ctx)
}

int dftk_b200_kblock_set_orbital_coefficients(dftk_b200_kblock* kb, const void* V) {
  dftk_b200_ctx* ctx = kb ? kb->grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(kb, "kblock_set_orbital_coefficients: kblock is NULL");
  REQUIRE(kb->n_orb > 0, "kblock_set_orbital_coefficients: the k-block has no orbitals (kblock_set_orbitals)");
  const int64_t np = kb->n_proj, no = kb->n_orb, n = np + no;
  cudaStream_t s = ctx->stream;
  cplx* blk = kb->Dh.p + np + n * np;
  if (V)
    CUDA_CHECK(cudaMemcpy2DAsync(blk, n * sizeof(cplx), V, no * sizeof(cplx), no * sizeof(cplx), no, cudaMemcpyDefault, s));
  else
    CUDA_CHECK(cudaMemset2DAsync(blk, n * sizeof(cplx), 0, no * sizeof(cplx), no));
  kb_refresh_pd(kb, np);
  CUDA_CHECK(cudaStreamSynchronize(s));
  API_END(ctx)
}

int dftk_b200_orbital_occupation_multi(int64_t n_blocks, dftk_b200_kblock* const* kbs, const void* const* psi,
                                       const double* occ_w_host, int64_t ld_w, const int32_t* n_bands, void* n_out) {
  dftk_b200_ctx* ctx = (n_blocks > 0 && kbs && kbs[0]) ? kbs[0]->grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(n_blocks >= 0 && (n_blocks == 0 || (kbs && psi && occ_w_host && n_bands && n_out)),
          "orbital_occupation_multi: bad argument");
  if (n_blocks == 0) return DFTK_B200_OK;
  require_device(ctx, n_out, "orbital_occupation_multi: n_out");
  for (int64_t i = 0; i < n_blocks; ++i) {
    REQUIRE(kbs[i], "orbital_occupation_multi: NULL k-block");
    require_device(ctx, psi[i], "orbital_occupation_multi: orbitals");
  }
  orbital_occupation_multi(n_blocks, kbs, (const cplx* const*)psi, occ_w_host, ld_w, (const int*)n_bands, (cplx*)n_out);
  API_END(ctx)
}

__global__ void k_scale_copy(double* dst, const double* src, double f, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[i] * f;
}

// Vt[x][y][z] = f V[z][y][x]: one (z, x) tile transpose per y, coalesced on both sides
__global__ void k_scale_transpose_xz(double* __restrict__ dst, const double* __restrict__ src, double f, int nx, int ny, int nz) {
  __shared__ double tile[32][33];
  const int y = blockIdx.z, x0 = blockIdx.x * 32, z0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int z = z0 + i, x = x0 + threadIdx.x;
    if (z < nz && x < nx) tile[i][threadIdx.x] = src[((size_t)z * ny + y) * nx + x];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int x = x0 + i, z = z0 + threadIdx.x;
    if (x < nx && z < nz) dst[((size_t)x * ny + y) * nz + z] = tile[threadIdx.x][i] * f;
  }
}

// the scaled potential of a k-block or grid, and on grids with a fused y-z stage its [x][y][z] copy
static void install_potential(dftk_b200_grid* g, const double* d, dftk::DevBuf<double>& V, dftk::DevBuf<double>& Vt) {
  dftk_b200_ctx* ctx = g->ctx;
  const int64_t N = g->N;
  const double f = g->fft_norm * g->ifft_norm;
  V.ensure(N);
  // pre-scale by fft_normalization * ifft_normalization = 1/N (src/terms/Hamiltonian.jl:152-153)
  LAUNCH(ctx, k_scale_copy, (unsigned)((N + 255) / 256), 256, 0, V.p, d, f, N);
  if (grid_yz_fusable(g)) {
    Vt.ensure(N);
    LAUNCH(ctx, k_scale_transpose_xz, dim3((g->nx + 31) / 32, (g->nz + 31) / 32, g->ny), dim3(32, 8), 0, Vt.p, d, f, g->nx,
           g->ny, g->nz);
  }
}

int dftk_b200_kblock_set_potential(dftk_b200_kblock* kb, const double* V) {
  dftk_b200_ctx* ctx = kb ? kb->grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(kb, "set_potential: kblock is NULL");
  kb->grid_V = -1;
  if (!V) {
    kb->has_V = false;
    return DFTK_B200_OK;
  }
  const int64_t N = kb->grid->N;
  const double* d = (const double*)stage_in(ctx, V, N * sizeof(double), ctx->stage_in);
  install_potential(kb->grid, d, kb->V, kb->Vt);
  kb->has_V = true;
  API_END(ctx)
}

int dftk_b200_grid_set_potential(dftk_b200_grid* grid, int spin, const double* V) {
  dftk_b200_ctx* ctx = grid ? grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(grid && (spin == 0 || spin == 1), "grid_set_potential: bad argument");
  if (!V) {
    grid->has_Vs[spin] = false;
    return DFTK_B200_OK;
  }
  const int64_t N = grid->N;
  const double* d = (const double*)stage_in(ctx, V, N * sizeof(double), ctx->stage_in);
  install_potential(grid, d, grid->Vs[spin], grid->Vts[spin]);
  grid->has_Vs[spin] = true;
  API_END(ctx)
}

int dftk_b200_kblock_trim(dftk_b200_kblock* kb) {
  dftk_b200_ctx* ctx = kb ? kb->grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(kb, "kblock_trim: NULL k-block");
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  kb->lobpcg_ws.release();
  kb->small_ws.release();
  kb->slab_x.release();
  kb->slab_stage.release();
  kb->i8_psi_planes.release();
  kb->i8_psi_exps.release();
  for (int i = 0; i < 8; ++i) {
    kb->i8_pool[i].release();
    kb->i8_epool[i].release();
  }
  kb->W1.release();
  kb->W2.release();
  kb->ldos_cube.release();
  kb->ldos_rho.release();
  kb->proj.release();
  kb->fold_ws.release();
  API_END(ctx)
}

int dftk_b200_kblock_use_grid_potential(dftk_b200_kblock* kb, int spin) {
  dftk_b200_ctx* ctx = kb ? kb->grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(kb && spin >= -1 && spin <= 1, "kblock_use_grid_potential: bad argument");
  if (spin < 0) {
    kb->grid_V = -1;
    kb->has_V = kb->V.p != nullptr;
    return DFTK_B200_OK;
  }
  REQUIRE(kb->grid->has_Vs[spin], "kblock_use_grid_potential: dftk_b200_grid_set_potential was not called for this spin");
  kb->grid_V = spin;
  kb->has_V = true;
  API_END(ctx)
}

int dftk_b200_fft_sphere_to_real(dftk_b200_kblock* kb, const void* psi, void* out_real, int64_t n_bands,
                                 int normalize) {
  dftk_b200_ctx* ctx = kb ? kb->grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(kb && psi && out_real && n_bands >= 0, "fft_sphere_to_real: bad argument");
  with_staging(ctx, psi, (size_t)kb->n_pw * n_bands * sizeof(cplx), out_real,
               (size_t)kb->grid->N * n_bands * sizeof(cplx), false, [&](const void* i, void* o) {
                 kb_sphere_to_real(kb, (const cplx*)i, (cplx*)o, n_bands, normalize ? kb->grid->ifft_norm : 1.0);
               });
  API_END(ctx)
}

int dftk_b200_fft_real_to_sphere(dftk_b200_kblock* kb, const void* in_real, void* out, int64_t n_bands,
                                 int normalize) {
  dftk_b200_ctx* ctx = kb ? kb->grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(kb && in_real && out && n_bands >= 0, "fft_real_to_sphere: bad argument");
  with_staging(ctx, in_real, (size_t)kb->grid->N * n_bands * sizeof(cplx), out,
               (size_t)kb->n_pw * n_bands * sizeof(cplx), false, [&](const void* i, void* o) {
                 kb_real_to_sphere(kb, (const cplx*)i, (cplx*)o, n_bands, normalize ? kb->grid->fft_norm : 1.0);
               });
  API_END(ctx)
}

int dftk_b200_apply_terms(dftk_b200_kblock* kb, const void* psi, void* hpsi, int64_t n_bands, int parts,
                          int accumulate) {
  dftk_b200_ctx* ctx = kb ? kb->grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(kb && psi && hpsi && n_bands >= 0, "apply: bad argument");
  REQUIRE(psi != hpsi, "apply: psi and hpsi must not alias");
  const bool loc = parts & 1, kinp = parts & 2, nl = parts & 4;
  REQUIRE(!kinp || kb->has_kin, "apply: kinetic energies were not given to kblock_create");
  size_t bytes = (size_t)kb->n_pw * n_bands * sizeof(cplx);
  if (!accumulate && n_bands > 0 && !is_device_ptr(psi) && !is_device_ptr(hpsi)) {
    apply_terms_host_pipelined(kb, (const cplx*)psi, (cplx*)hpsi, n_bands, loc, kinp, nl);
    return DFTK_B200_OK;
  }
  with_staging(ctx, psi, bytes, hpsi, bytes, accumulate != 0, [&](const void* i, void* o) {
    if (loc || kinp) kb_apply_local_kinetic(kb, (const cplx*)i, (cplx*)o, n_bands, loc, kinp, accumulate != 0);
    else if (!accumulate) CUDA_CHECK(cudaMemsetAsync(o, 0, bytes, ctx->stream));
    if (nl) kb_apply_nonlocal(kb, (const cplx*)i, (cplx*)o, n_bands);
  });
  API_END(ctx)
}

int dftk_b200_apply_h(dftk_b200_kblock* kb, const void* psi, void* hpsi, int64_t n_bands) {
  if (!kb) return record_error(nullptr, DFTK_B200_EINVAL, "apply_h: kblock is NULL");
  int parts = (kb->has_V ? 1 : 0) | (kb->has_kin ? 2 : 0) | (kb->n_nl() > 0 ? 4 : 0);
  return dftk_b200_apply_terms(kb, psi, hpsi, n_bands, parts, 0);
}

__global__ void k_nonlocal_band_energy(const cplx* proj, const cplx* dproj, int64_t np, int64_t nb,
                                       double* out) {
  // one thread per band: sum_i real(conj(proj) * dproj)
  int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nb) return;
  double s = 0.0;
  for (int64_t i = 0; i < np; ++i) {
    cplx a = proj[i + np * b], d = dproj[i + np * b];
    s += a.x * d.x + a.y * d.y;
  }
  out[b] = s;
}

int dftk_b200_band_energies(dftk_b200_kblock* kb, const void* psi, int64_t n_bands, double* ekin_host,
                            double* enl_host) {
  dftk_b200_ctx* ctx = kb ? kb->grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(kb && psi && n_bands >= 0, "band_energies: bad argument");
  if (n_bands == 0) return DFTK_B200_OK;
  const cplx* d = (const cplx*)stage_in(ctx, psi, (size_t)kb->n_pw * n_bands * sizeof(cplx), ctx->stage_in);
  double* sc = ctx->scal.ensure(2 * n_bands + 8);
  if (ekin_host) {
    REQUIRE(kb->has_kin, "band_energies: no kinetic term");
    kin_dots(ctx, d, kb->n_pw, kb->kin.p, kb->n_pw, n_bands, sc);
    CUDA_CHECK(cudaMemcpyAsync(ekin_host, sc, n_bands * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  }
  if (enl_host) {
    if (kb->n_proj == 0) {
      CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
      for (int64_t i = 0; i < n_bands; ++i) enl_host[i] = 0.0;
    } else {
      const int64_t np = kb->n_proj;
      cplx* proj = kb->proj.ensure((size_t)2 * np * n_bands);
      cplx* dproj = proj + (size_t)np * n_bands;
      const cplx one = make_double2(1, 0), zero = make_double2(0, 0);
      kb_project(kb, d, n_bands, proj);
      zgemm(ctx, 0, np, n_bands, np, one, kb->Dc.p, np, proj, np, zero, dproj, np);
      LAUNCH(ctx, k_nonlocal_band_energy, (unsigned)((n_bands + 63) / 64), 64, 0, (const cplx*)proj,
             (const cplx*)dproj, np, n_bands, sc + n_bands);
      CUDA_CHECK(cudaMemcpyAsync(enl_host, sc + n_bands, n_bands * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    }
  }
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  API_END(ctx)
}

int dftk_b200_band_energies_multi(int64_t n_blocks, dftk_b200_kblock* const* kbs, const void* const* psi, const int32_t* n_bands,
                                  int64_t ld_out, double* ekin_host, double* enl_host) {
  dftk_b200_ctx* ctx = (n_blocks > 0 && kbs && kbs[0]) ? kbs[0]->grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(n_blocks >= 0 && (n_blocks == 0 || (kbs && psi && n_bands)), "band_energies_multi: bad argument");
  for (int64_t i = 0; i < n_blocks; ++i) {
    REQUIRE(kbs[i], "band_energies_multi: NULL k-block");
    require_device(ctx, psi[i], "band_energies_multi: orbitals");
  }
  band_energies_multi(n_blocks, kbs, (const cplx* const*)psi, (const int*)n_bands, ld_out, ekin_host, enl_host);
  API_END(ctx)
}

int dftk_b200_density_accumulate_multi(int64_t n_blocks, dftk_b200_kblock* const* kbs, const void* const* psi,
                                       const double* occ_w_host, int64_t ld_w, const int32_t* n_bands, double* rho) {
  dftk_b200_ctx* ctx = (n_blocks > 0 && kbs && kbs[0]) ? kbs[0]->grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(n_blocks >= 0 && (n_blocks == 0 || (kbs && psi && n_bands && occ_w_host && rho)), "density_accumulate_multi: bad argument");
  if (n_blocks == 0) return DFTK_B200_OK;
  require_device(ctx, rho, "density_accumulate_multi: rho");
  for (int64_t i = 0; i < n_blocks; ++i) {
    REQUIRE(kbs[i] && n_bands[i] >= 0 && n_bands[i] <= ld_w, "density_accumulate_multi: bad block");
    require_device(ctx, psi[i], "density_accumulate_multi: orbitals");
  }
  if (!kb_density_accumulate_multi((int)n_blocks, kbs, (const cplx* const*)psi, occ_w_host, ld_w, (const int*)n_bands, rho))
    for (int64_t i = 0; i < n_blocks; ++i)       // blocks that do not qualify for the batched kernels: one after the other
      if (n_bands[i] > 0)
        kb_density_accumulate(kbs[i], (const cplx*)psi[i], occ_w_host + i * ld_w, n_bands[i], rho + (size_t)kbs[i]->spin * kbs[i]->grid->N);
  API_END(ctx)
}

int dftk_b200_lobpcg(dftk_b200_kblock* kb, void* X, int64_t n_bands, double tol, int miniter, int maxiter,
                     int64_t n_conv_check, int use_tpa_preconditioner, double* lambda_host,
                     double* resid_host, int* n_iter, int64_t* n_matvec, int* converged) {
  dftk_b200_ctx* ctx = kb ? kb->grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(kb && X && lambda_host && resid_host && n_iter && n_matvec && converged, "lobpcg: NULL argument");
  REQUIRE(maxiter >= 0 && miniter >= 0, "lobpcg: bad iteration limits");
  size_t bytes = (size_t)kb->n_pw * n_bands * sizeof(cplx);
  if (is_device_ptr(X)) {
    lobpcg_run(kb, (cplx*)X, n_bands, tol, miniter, maxiter, n_conv_check, use_tpa_preconditioner != 0,
               lambda_host, resid_host, n_iter, n_matvec, converged);
  } else {
    ctx->stage_out.ensure(bytes);
    CUDA_CHECK(cudaMemcpyAsync(ctx->stage_out.p, X, bytes, cudaMemcpyHostToDevice, ctx->stream));
    lobpcg_run(kb, (cplx*)ctx->stage_out.p, n_bands, tol, miniter, maxiter, n_conv_check,
               use_tpa_preconditioner != 0, lambda_host, resid_host, n_iter, n_matvec, converged);
    CUDA_CHECK(cudaMemcpyAsync(X, ctx->stage_out.p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  }
  API_END(ctx)
}

int dftk_b200_lobpcg_multi(int64_t n_blocks, dftk_b200_kblock* const* kbs, void* const* X, int64_t n_bands, double tol,
                           int miniter, int maxiter, int64_t n_conv_check, int use_tpa_preconditioner,
                           double* lambda_host, double* resid_host, int* n_iter, int64_t* n_matvec, int* converged) {
  dftk_b200_ctx* ctx = (n_blocks > 0 && kbs && kbs[0]) ? kbs[0]->grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(n_blocks >= 0, "lobpcg_multi: negative block count");
  if (n_blocks == 0) return DFTK_B200_OK;
  REQUIRE(kbs && X && lambda_host && resid_host && n_iter && n_matvec && converged, "lobpcg_multi: NULL argument");
  REQUIRE(maxiter >= 0 && miniter >= 0, "lobpcg_multi: bad iteration limits");
  for (int64_t i = 0; i < n_blocks; ++i) {
    REQUIRE(kbs[i], "lobpcg_multi: NULL k-block");
    require_device(ctx, X[i], "lobpcg_multi: orbitals");
  }
  lobpcg_run_multi(n_blocks, kbs, (cplx* const*)X, n_bands, tol, miniter, maxiter, n_conv_check, use_tpa_preconditioner != 0,
                   lambda_host, resid_host, n_iter, n_matvec, converged);
  API_END(ctx)
}

int dftk_b200_lobpcg_slab(dftk_b200_kblock* kb, void* X, int64_t n_bands, double tol, int miniter, int maxiter,
                          int64_t n_conv_check, int use_tpa_preconditioner, double* lambda_host, double* resid_host,
                          int* n_iter, int64_t* n_matvec, int* converged, double* exchange_bytes) {
  dftk_b200_ctx* ctx = kb ? kb->grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(kb && X && lambda_host && resid_host && n_iter && n_matvec && converged, "lobpcg_slab: NULL argument");
  REQUIRE(maxiter >= 0 && miniter >= 0, "lobpcg_slab: bad iteration limits");
  REQUIRE(is_device_ptr(X), "lobpcg_slab: orbitals must be device memory");
  lobpcg_run_slab(kb, (cplx*)X, n_bands, tol, miniter, maxiter, n_conv_check, use_tpa_preconditioner != 0, lambda_host,
                  resid_host, n_iter, n_matvec, converged, exchange_bytes);
  API_END(ctx)
}

int dftk_b200_random_orbitals(int64_t n_blocks, dftk_b200_kblock* const* kbs, void* const* X, int64_t n_bands, uint64_t seed) {
  dftk_b200_ctx* ctx = (n_blocks > 0 && kbs && kbs[0]) ? kbs[0]->grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(n_blocks >= 0 && (n_blocks == 0 || (kbs && X)) && n_bands >= 1, "random_orbitals: bad argument");
  for (int64_t i = 0; i < n_blocks; ++i) {
    REQUIRE(kbs[i], "random_orbitals: NULL k-block");
    require_device(ctx, X[i], "random_orbitals: orbitals");
  }
  random_orbitals_multi(n_blocks, kbs, (cplx* const*)X, n_bands, seed);
  API_END(ctx)
}

int dftk_b200_density_accumulate(dftk_b200_kblock* kb, const void* psi, const double* occ_w_host,
                                 int64_t n_bands, double* rho) {
  dftk_b200_ctx* ctx = kb ? kb->grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(kb && psi && occ_w_host && rho && n_bands >= 0, "density_accumulate: bad argument");
  const cplx* d = (const cplx*)stage_in(ctx, psi, (size_t)kb->n_pw * n_bands * sizeof(cplx), ctx->stage_in);
  if (is_device_ptr(rho)) {
    kb_density_accumulate(kb, d, occ_w_host, n_bands, rho);
  } else {
    size_t bytes = (size_t)kb->grid->N * sizeof(double);
    ctx->stage_out.ensure(bytes);
    CUDA_CHECK(cudaMemcpyAsync(ctx->stage_out.p, rho, bytes, cudaMemcpyHostToDevice, ctx->stream));
    kb_density_accumulate(kb, d, occ_w_host, n_bands, (double*)ctx->stage_out.p);
    CUDA_CHECK(cudaMemcpyAsync(rho, ctx->stage_out.p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  }
  API_END(ctx)
}

// ------------------------------------------------------------------ collectives
static ncclDataType_t nccl_type(int dtype) {
  if (dtype == DFTK_B200_F64) return ncclFloat64;
  if (dtype == DFTK_B200_I64) return ncclInt64;
  throw Error(DFTK_B200_EINVAL, "collective: unknown dtype");
}

int dftk_b200_allreduce(dftk_b200_ctx* ctx, void* buf, int64_t count, int dtype, int op) {
  API_BEGIN
  REQUIRE(ctx && buf && count >= 0, "allreduce: bad argument");
  if (ctx->nranks == 1) return DFTK_B200_OK;
  REQUIRE(ctx->nccl, "allreduce: context has no communicator (use ctx_create_dist)");
  REQUIRE(is_device_ptr(buf), "allreduce: buffer must be device memory");
  ncclRedOp_t o = op == 0 ? ncclSum : (op == 1 ? ncclMin : ncclMax);
  NCCL_CHECK(ncclAllReduce(buf, buf, (size_t)count, nccl_type(dtype), o, ctx->nccl, ctx->stream));
  ctx->launches++;
  API_END(ctx)
}

int dftk_b200_allgather(dftk_b200_ctx* ctx, const void* send, void* recv, int64_t count_per_rank, int dtype) {
  API_BEGIN
  REQUIRE(ctx && send && recv && count_per_rank >= 0, "allgather: bad argument");
  if (ctx->nranks == 1) {
    if (send != recv)
      CUDA_CHECK(cudaMemcpyAsync(recv, send, (size_t)count_per_rank * 8, cudaMemcpyDefault, ctx->stream));
    return DFTK_B200_OK;
  }
  REQUIRE(ctx->nccl, "allgather: context has no communicator (use ctx_create_dist)");
  NCCL_CHECK(ncclAllGather(send, recv, (size_t)count_per_rank, nccl_type(dtype), ctx->nccl, ctx->stream));
  ctx->launches++;
  API_END(ctx)
}

// ------------------------------------------------------------------ SCF plumbing next to the hot path
int dftk_b200_xc_evaluate(dftk_b200_ctx* ctx, int functional_mask, int n_spin, int64_t n_points, const double* rho,
                          const double* sigma, double* e, double* vrho, double* vsigma) {
  API_BEGIN
  REQUIRE(ctx && rho && e && vrho && n_points >= 0, "xc_evaluate: NULL argument");
  const bool gga = (functional_mask & XC_GGA_BITS) != 0;
  REQUIRE(!gga || (sigma && vsigma), "xc_evaluate: GGA functionals need sigma and vsigma");
  REQUIRE((functional_mask & ~XC_VALID_BITS) == 0 && functional_mask != 0, "xc_evaluate: unknown functional bits");
  REQUIRE(is_device_ptr(rho) && is_device_ptr(e) && is_device_ptr(vrho), "xc_evaluate: arrays must be device memory");
  xc_evaluate(ctx, functional_mask, n_spin, gga, n_points, rho, sigma, e, vrho, vsigma);
  API_END(ctx)
}

int dftk_b200_symmetrize_fourier(dftk_b200_grid* grid, const void* rho_fourier_in, void* rho_fourier_out,
                                 int n_sym, const int32_t* invS, const double* tau) {
  dftk_b200_ctx* ctx = grid ? grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(grid && rho_fourier_in && rho_fourier_out && invS && tau && n_sym >= 1, "symmetrize_fourier: bad argument");
  REQUIRE(rho_fourier_in != rho_fourier_out, "symmetrize_fourier: in and out must not alias");
  REQUIRE(is_device_ptr(rho_fourier_in) && is_device_ptr(rho_fourier_out), "symmetrize_fourier: arrays must be device memory");
  symmetrize_fourier(grid, (const cplx*)rho_fourier_in, (cplx*)rho_fourier_out, n_sym, (const int*)invS, tau);
  API_END(ctx)
}

// ------------------------------------------------------------------ forces
int dftk_b200_local_forces(dftk_b200_grid* grid, const void* w, int n_atoms, const double* positions,
                           double* forces_host) {
  dftk_b200_ctx* ctx = grid ? grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(grid && w && n_atoms >= 0 && (n_atoms == 0 || (positions && forces_host)), "local_forces: bad argument");
  REQUIRE(is_device_ptr(w), "local_forces: w must be device memory");
  REQUIRE(!is_device_ptr(forces_host), "local_forces: forces are returned in host memory");
  local_forces(grid, (const cplx*)w, n_atoms, positions, forces_host);
  API_END(ctx)
}

int dftk_b200_ewald(dftk_b200_ctx* ctx, const double* lattice, int n_atoms, const double* charges, const double* positions,
                    double eta, const int32_t* glims, const int32_t* rlims, double* energy_host, double* forces_host) {
  API_BEGIN
  REQUIRE(ctx && lattice && charges && positions && glims && rlims && n_atoms >= 1, "ewald: bad argument");
  REQUIRE(!is_device_ptr(lattice) && !is_device_ptr(charges) && !is_device_ptr(positions), "ewald: inputs are host arrays");
  ewald(ctx, lattice, n_atoms, charges, positions, eta, (const int*)glims, (const int*)rlims, energy_host, forces_host);
  API_END(ctx)
}

int dftk_b200_nonlocal_force_rows(dftk_b200_kblock* kb, const void* psi, const double* occ_w_host, int64_t n_bands,
                                  const double* gpk, double* rows_host) {
  dftk_b200_ctx* ctx = kb ? kb->grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(kb && psi && occ_w_host && gpk && rows_host && n_bands >= 0, "nonlocal_force_rows: bad argument");
  REQUIRE(is_device_ptr(gpk), "nonlocal_force_rows: gpk must be device memory");
  const cplx* d = (const cplx*)stage_in(ctx, psi, (size_t)kb->n_pw * n_bands * sizeof(cplx), ctx->stage_in);
  kb_nonlocal_force_rows(kb, d, occ_w_host, n_bands, gpk, rows_host);
  API_END(ctx)
}

// ------------------------------------------------------------------ setup kernels
int dftk_b200_structure_factor(dftk_b200_grid* grid, int n_atoms, const double* positions, const double* coefficients, void* out) {
  dftk_b200_ctx* ctx = grid ? grid->ctx : nullptr;
  API_BEGIN
  REQUIRE(grid && positions && out && n_atoms >= 1, "structure_factor: bad argument");
  REQUIRE(is_device_ptr(out) && !is_device_ptr(positions), "structure_factor: positions on the host, result on the device");
  structure_factor(grid, n_atoms, positions, coefficients, (cplx*)out);
  API_END(ctx)
}

int dftk_b200_build_projectors(dftk_b200_ctx* ctx, int64_t n_pw, const double* gpk, int n_atoms, const double* positions,
                               int n_rows, const void* form_factors, void* P) {
  API_BEGIN
  REQUIRE(ctx && gpk && positions && form_factors && P && n_pw >= 1 && n_atoms >= 0 && n_rows >= 0, "build_projectors: bad argument");
  REQUIRE(is_device_ptr(gpk) && is_device_ptr(form_factors) && is_device_ptr(P) && !is_device_ptr(positions),
          "build_projectors: gpk / form factors / P on the device, positions on the host");
  build_projectors(ctx, n_pw, gpk, n_atoms, positions, n_rows, (const cplx*)form_factors, (cplx*)P);
  API_END(ctx)
}

int dftk_b200_radial_transform(dftk_b200_ctx* ctx, int64_t n_r, const double* r, int n_f, const double* g, const int32_t* l,
                               int64_t n_q, const double* q, double* F) {
  API_BEGIN
  REQUIRE(ctx && n_r >= 1 && n_f >= 0 && n_q >= 0 && (n_f == 0 || n_q == 0 || (r && g && l && q && F)),
          "radial_transform: bad argument");
  if (n_f > 0 && n_q > 0) {
    REQUIRE(is_device_ptr(r) && is_device_ptr(g) && is_device_ptr(q) && is_device_ptr(F) && !is_device_ptr(l),
            "radial_transform: r, g, q and F on the device, l on the host");
    radial_transform(ctx, n_r, r, n_f, g, (const int*)l, n_q, q, F);
  }
  API_END(ctx)
}

// ------------------------------------------------------------------ dense helpers
int dftk_b200_columnwise_dots(dftk_b200_ctx* ctx, const void* A, const void* B, int64_t n_rows,
                              int64_t n_cols, void* out_host) {
  API_BEGIN
  REQUIRE(ctx && A && B && out_host, "columnwise_dots: NULL argument");
  REQUIRE(is_device_ptr(A) && is_device_ptr(B), "columnwise_dots: inputs must be device memory");
  cplx* o = (cplx*)ctx->scal.ensure(2 * n_cols + 8);
  columnwise_dots(ctx, (const cplx*)A, n_rows, (const cplx*)B, n_rows, n_rows, n_cols, o);
  CUDA_CHECK(cudaMemcpyAsync(out_host, o, n_cols * sizeof(cplx), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  API_END(ctx)
}

int dftk_b200_tall_gram(dftk_b200_ctx* ctx, const void* A, int64_t lda, int64_t n_cols_a, const void* B, int64_t ldb,
                        int64_t n_cols_b, int64_t n_rows, void* out_host) {
  API_BEGIN
  REQUIRE(ctx && A && B && out_host && n_rows >= 1, "tall_gram: bad argument");
  REQUIRE(is_device_ptr(A) && is_device_ptr(B) && !is_device_ptr(out_host), "tall_gram: A, B on the device, result on the host");
  tall_gram(ctx, (const cplx*)A, lda, (int)n_cols_a, (const cplx*)B, ldb, (int)n_cols_b, n_rows, (cplx*)out_host);
  API_END(ctx)
}

int dftk_b200_zgemm(dftk_b200_ctx* ctx, int transA, int64_t m, int64_t n, int64_t k, const double* alpha2,
                    const void* A, int64_t lda, const void* B, int64_t ldb, const double* beta2, void* C,
                    int64_t ldc) {
  API_BEGIN
  REQUIRE(ctx && A && B && C && alpha2 && beta2, "zgemm: NULL argument");
  REQUIRE(is_device_ptr(A) && is_device_ptr(B) && is_device_ptr(C), "zgemm: operands must be device memory");
  zgemm(ctx, transA, m, n, k, make_double2(alpha2[0], alpha2[1]), (const cplx*)A, lda, (const cplx*)B, ldb,
        make_double2(beta2[0], beta2[1]), (cplx*)C, ldc);
  API_END(ctx)
}

}  // extern "C"
