// LOBPCG block eigensolver on the device.  Restates the algorithm of the reference's
// src/eigen/lobpcg_hyper_impl.jl:354-582 (LOBPCG with B = I), :141-171 (rayleigh_ritz), :216-261
// (ortho!), :271-323 (ortho!(X,Y,BY)), :190-210 (safe_cholesky), :264-268 (drop_small!) and the TPA
// preconditioner of src/eigen/preconditioners.jl:27-78, with Julia's active-block views expressed as
// column offsets.  All N_pw-sized work is GEMMs (blas.cu) or fused elementwise kernels (lobpcg_batch.cuh); the small
// dense factorisations (<= 3M x 3M) use cuSOLVER (heevd / potrf / trtri), as SURVEY.md §7 allows.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <numeric>
#include "structs.cuh"
#include <ucontext.h>
#include <functional>
#include <memory>
#include "lobpcg_batch.cuh"

namespace dftk {

static const double EPS = DBL_EPSILON;

struct Mat {
  cplx* p;
  int64_t ld, rows, cols;
  Mat cols_from(int64_t c0) const { return Mat{p + ld * c0, ld, rows, cols - c0}; }
  Mat cols_range(int64_t c0, int64_t nc) const { return Mat{p + ld * c0, ld, rows, nc}; }
};

// ------------------------------------------------------------------ small kernels of the direct path only
__global__ void k_sqrt_n(double* __restrict__ v, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) v[i] = sqrt(v[i]);
}
// Hermitian(upper): mirror the strictly upper triangle into the lower one, make the diagonal real
__global__ void k_hermitize_upper(cplx* __restrict__ A, int64_t ld, int64_t n) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * n) return;
  int64_t i = idx % n, j = idx / n;
  if (i > j) {
    cplx v = A[j + ld * i];
    A[i + ld * j] = make_double2(v.x, -v.y);
  } else if (i == j) {
    A[i + ld * j].y = 0.0;
  }
}
__global__ void k_zero_lower(cplx* __restrict__ A, int64_t ld, int64_t n) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * n) return;
  int64_t i = idx % n, j = idx / n;
  if (i > j) A[i + ld * j] = make_double2(0.0, 0.0);
}
__global__ void k_add_diag(cplx* __restrict__ A, int64_t ld, int64_t n, double shift) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) A[i + ld * i].x += shift;
}
__global__ void k_compute_lambda(const cplx* __restrict__ num, const cplx* __restrict__ den,
                                 double* __restrict__ lam, int64_t n) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  // real((x'Ax)/(x'x)) with complex division, compute_λ (:341-344)
  cplx a = num[i], b = den[i];
  double d = b.x * b.x + b.y * b.y;
  lam[i] = (a.x * b.x + a.y * b.y) / d;
}

static inline unsigned nblk(int64_t n) { return (unsigned)((n + 255) / 256); }

// Optional section timing (env DFTK_B200_PROFILE=1): stream-synchronising wall clock per LOBPCG section.
struct SectionProf {
  bool on;
  cudaStream_t st;
  std::vector<std::pair<std::string, double>> acc;
  double t0 = 0;
  std::string cur;
  static double now() {
    timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return ts.tv_sec + 1e-9 * ts.tv_nsec;
  }
  void begin(const char* name) {
    if (!on) return;
    end();
    cudaStreamSynchronize(st);
    cur = name;
    t0 = now();
  }
  void end() {
    if (!on || cur.empty()) return;
    cudaStreamSynchronize(st);
    double dt = now() - t0;
    for (auto& a : acc)
      if (a.first == cur) {
        a.second += dt;
        cur.clear();
        return;
      }
    acc.push_back({cur, dt});
    cur.clear();
  }
  // DFTK_B200_PROFILE=2: accumulate over all solves of the process, print once at exit (small systems: hundreds of solves)
  struct Global {
    std::vector<std::pair<std::string, double>> acc;
    long iters = 0, solves = 0;
    ~Global() {
      if (acc.empty()) return;
      double tot = 0;
      for (auto& a : acc) tot += a.second;
      fprintf(stderr, "[dftk_b200 lobpcg profile, all solves] %ld solves, %ld iterations, %.3f s in sections\n", solves, iters, tot);
      for (auto& a : acc) fprintf(stderr, "  %-22s %9.3f s  %5.1f %%\n", a.first.c_str(), a.second, 100 * a.second / tot);
    }
  };
  static Global& global() {
    static Global g;
    return g;
  }
  bool aggregate = false;
  void report(int niter) {
    if (!on) return;
    end();
    if (aggregate) {
      Global& g = global();
      g.iters += niter;
      g.solves++;
      for (auto& a : acc) {
        bool found = false;
        for (auto& b : g.acc)
          if (b.first == a.first) {
            b.second += a.second;
            found = true;
          }
        if (!found) g.acc.push_back(a);
      }
      return;
    }
    double tot = 0;
    for (auto& a : acc) tot += a.second;
    fprintf(stderr, "[dftk_b200 lobpcg profile] %d iterations, %.3f s in sections\n", niter, tot);
    for (auto& a : acc) fprintf(stderr, "  %-22s %9.3f s  %5.1f %%\n", a.first.c_str(), a.second, 100 * a.second / tot);
  }
};


// ------------------------------------------------------------------ deferred operations of the batched small path
// A solve with <= SMALL_MAX_N bands never launches anything itself: it records operations, and the scheduler below
// merges the same operation of all k-blocks in flight into ONE launch (lobpcg_batch.cuh).  Each solve runs as a
// coroutine (ucontext) that yields where the algorithm needs a value on the host.
enum OpType {
  OP_GRAM = 0, OP_CHOL, OP_RMUL, OP_BTIMES, OP_HEEV, OP_RESIDUAL, OP_PRECOND, OP_COLNORMS, OP_SCALE, OP_COPY2D, OP_MAKECP,
  OP_STATS, OP_RANDN, OP_LAMBDA, OP_APPLYH, OP_D2H, OP_NTYPES
};
struct D2HItem { const double* src; int n; double* host_dst; };
struct Op {
  int type;
  union U {
    GramItem gram; CholItem chol; RmulItem rmul; BtimesItem btimes; HeevItem heev; ResidualItem residual; PrecondItem precond;
    ColnormItem colnorm; ScaleItem scale; Copy2dItem copy2d; MakecpItem makecp; StatsItem stats; RandnItem randn;
    LambdaItem lambda; ApplyHItem applyh; D2HItem d2h;
    U() {}
  } u;
  Op() : type(-1) {}
};

struct Coro {
  ucontext_t uc;
  std::unique_ptr<char[]> stack;
  size_t stack_size = 0;
  std::function<void()> body;
  bool finished = false, waiting_align = false, failed = false;
  int err_code = 0;
  std::string err;
  std::vector<Op> ops;
  size_t cursor = 0;
};
static thread_local Coro* g_coro = nullptr;
static thread_local ucontext_t* g_main_uc = nullptr;

static void coro_entry() {
  Coro* c = g_coro;
  try {
    c->body();
  } catch (const Error& e) {
    c->failed = true;
    c->err_code = e.code;
    c->err = e.what();
  } catch (const std::exception& e) {
    c->failed = true;
    c->err_code = DFTK_B200_EINVAL;
    c->err = e.what();
  } catch (...) {
    c->failed = true;
    c->err_code = DFTK_B200_EINVAL;
    c->err = "unknown exception in a LOBPCG solve";
  }
  c->finished = true;
  swapcontext(&c->uc, g_main_uc);
}
static inline void coro_yield(Coro* c) { swapcontext(&c->uc, g_main_uc); }

static void small_gram_geometry(dftk_b200_ctx* ctx, int64_t rows, int* n_ctas_out, long long* rpc_out) {
  int64_t n_ctas = std::max<int64_t>(1, std::min<int64_t>((rows + 127) / 128, 2 * (int64_t)ctx->sm_count));
  int64_t rpc = (rows + n_ctas - 1) / n_ctas;
  rpc = (rpc + SMALL_TR - 1) / SMALL_TR * SMALL_TR;
  n_ctas = std::max<int64_t>(1, (rows + rpc - 1) / rpc);
  *n_ctas_out = (int)n_ctas;
  *rpc_out = rpc;
}
GramItem single_gram_item(dftk_b200_ctx* ctx, const cplx* A, int64_t lda, int nA, const cplx* B, int64_t ldb, int nB,
                          int64_t n_rows, cplx* C) {
  GramItem g{};
  g.A.n = g.B.n = 1;
  g.A.p[0] = A; g.A.ld[0] = lda; g.A.cols[0] = nA;
  g.B.p[0] = B; g.B.ld[0] = ldb; g.B.cols[0] = nB;
  for (int q = 1; q < 4; ++q) { g.A.start[q] = nA; g.B.start[q] = nB; }
  g.n_rows = n_rows;
  small_gram_geometry(ctx, n_rows, &g.n_ctas, &g.rows_per_cta);
  g.upper_only = 0;
  g.C = C;
  g.ldc = nA;
  return g;
}
BtimesItem single_btimes_item(const cplx* Y, int nY, const cplx* c, int ncols, cplx* out, int64_t n_rows, double alpha,
                              double beta) {
  BtimesItem b{};
  b.Y.n = 1;
  b.Y.p[0] = Y; b.Y.ld[0] = n_rows; b.Y.cols[0] = nY;
  for (int q = 1; q < 4; ++q) b.Y.start[q] = nY;
  b.cm = c; b.ldcm = nY; b.ncols = ncols;
  b.out = out; b.ldo = n_rows; b.n_rows = n_rows; b.alpha = alpha; b.beta = beta;
  return b;
}

BatchExec::BatchExec(dftk_b200_ctx* c, BatchSlot& s) : ctx(c), slot(s) {
  // pinned staging is created once per slot (cudaMallocHost costs about a millisecond)
  if (!slot.gather_h) CUDA_CHECK(cudaMallocHost((void**)&slot.gather_h, BatchSlot::GATHER_CAP * sizeof(double)));
  slot.gather.ensure(BatchSlot::GATHER_CAP);
  if (!slot.ev) CUDA_CHECK(cudaEventCreateWithFlags(&slot.ev, cudaEventDisableTiming));
}
void BatchExec::reset_counters(size_t n) {
  slot.counter.ensure(std::max<size_t>(n, 256));
  CUDA_CHECK(cudaMemsetAsync(slot.counter.p, 0, slot.counter.cap * sizeof(int), ctx->stream));
}

void BatchExec::gram_batch(std::vector<GramItem>& v) {
  // per-item partial workspaces and arrival counters
  size_t ws_total = 0;
  int max_ctas = 1;
  size_t smem = 0;
  for (auto& it : v) {
    const int nA = it.A.start[it.A.n], nB = it.B.start[it.B.n];
    ws_total += (size_t)it.n_ctas * nA * nB;
    max_ctas = std::max(max_ctas, it.n_ctas);
    smem = std::max(smem, (size_t)SMALL_TR * (nA + nB) * sizeof(cplx));
  }
  cplx* ws = (cplx*)slot.gram_ws->ensure(ws_total * sizeof(cplx));
  if (slot.counter.cap < v.size()) reset_counters(v.size());
  size_t off = 0;
  for (size_t i = 0; i < v.size(); ++i) {
    const int nA = v[i].A.start[v[i].A.n], nB = v[i].B.start[v[i].B.n];
    v[i].ws = ws + off;
    v[i].counter = (unsigned*)slot.counter.p + i;
    off += (size_t)v[i].n_ctas * nA * nB;
  }
  const GramItem* d = upload(v);
  LAUNCH(ctx, kb_gram, dim3((unsigned)max_ctas, (unsigned)v.size()), 256, smem, d);
}
void BatchExec::btimes_batch(const std::vector<BtimesItem>& v) {
  long long max_rows = 1;
  size_t smem = 0;
  for (auto& it : v) {
    max_rows = std::max(max_rows, it.n_rows);
    smem = std::max(smem, (size_t)it.Y.start[it.Y.n] * it.ncols * sizeof(cplx));
  }
  const BtimesItem* d = upload(v);
  LAUNCH(ctx, kb_btimes, dim3((unsigned)((max_rows + 127) / 128), (unsigned)v.size()), 128, smem, d);
}
void BatchExec::heev_batch(const std::vector<HeevItem>& v) {
  size_t smem = 0;
  for (auto& it : v) {
    const size_t half = ((it.n + 1) & ~1) / 2;
    smem = std::max(smem, (size_t)it.n * it.n * sizeof(cplx) + 2 * (half + 1) * sizeof(cplx) + SMALL_RED * sizeof(double) +
                              2 * (half + 1) * sizeof(int) + 16);
  }
  LAUNCH(ctx, kb_heev, (unsigned)v.size(), SMALL_RED, smem, upload(v));
}
void BatchExec::kin_dots_batch(const std::vector<KinDotsItem>& v) {
  int mc = 1;
  for (auto& it : v) mc = std::max(mc, it.n_cols);
  LAUNCH(ctx, kb_kin_dots, dim3((unsigned)mc, (unsigned)v.size()), 256, 0, upload(v));
}
// local + kinetic part: the k-block's own batched FFT pipeline; nonlocal part P (D P'psi) as two batched small products
// over all items (projector counts of the small configurations are <= 20)
void BatchExec::apply_h_batch(const std::vector<ApplyHItem>& v) {
  {
    // local + kinetic part of all k-blocks in five launches when they share the grid's register FFT engine
    std::vector<dftk_b200_kblock*> kbs;
    std::vector<const cplx*> in;
    std::vector<cplx*> out;
    std::vector<int> nb;
    for (const ApplyHItem& a : v) {
      kbs.push_back(a.kb); in.push_back(a.in); out.push_back(a.out); nb.push_back(a.ncols);
    }
    if (!kb_apply_local_kinetic_multi((int)kbs.size(), kbs.data(), in.data(), out.data(), nb.data(), slot.ring))
      for (const ApplyHItem& a : v) kb_apply_local_kinetic(a.kb, a.in, a.out, a.ncols, a.kb->has_V, a.kb->has_kin, false);
  }
  std::vector<GramItem> g;
  std::vector<BtimesItem> b;
  for (const ApplyHItem& a : v) {
    dftk_b200_kblock* kb = a.kb;
    if (kb->n_nl() == 0) continue;
    if (kb->n_nl() > SMALL_MAX_COLS || a.ncols > SMALL_MAX_N || !kb->PD.p) {
      kb_apply_nonlocal(kb, a.in, a.out, a.ncols);
      continue;
    }
    cplx* proj = kb->proj.ensure((size_t)2 * kb->n_nl() * SMALL_MAX_N);
    const int nl = (int)kb->n_nl();
    g.push_back(single_gram_item(ctx, kb->P.p, kb->n_pw, nl, a.in, kb->n_pw, a.ncols, kb->n_pw, proj));
    b.push_back(single_btimes_item(kb->PD.p, nl, proj, a.ncols, a.out, kb->n_pw, 1.0, 1.0));
  }
  if (!g.empty()) {
    gram_batch(g);
    btimes_batch(b);
  }
}

void BatchExec::launch(int type, const std::vector<Op*>& ops) {
  const unsigned n = (unsigned)ops.size();
  switch (type) {
    case OP_GRAM: {
      auto v = collect<GramItem>(ops, [](Op* o) { return o->u.gram; });
      gram_batch(v);
      break;
    }
    case OP_CHOL: {
      auto v = collect<CholItem>(ops, [](Op* o) { return o->u.chol; });
      LAUNCH(ctx, kb_chol, n, SMALL_RED, 0, upload(v));
      break;
    }
    case OP_RMUL: {
      auto v = collect<RmulItem>(ops, [](Op* o) { return o->u.rmul; });
      long long max_rows = 1;
      size_t smem = 0;
      for (auto& it : v) {
        max_rows = std::max(max_rows, it.n_rows);
        smem = std::max(smem, (size_t)it.n * it.n * sizeof(cplx));
      }
      LAUNCH(ctx, kb_rmul, dim3((unsigned)((max_rows + 127) / 128), n), 128, smem, upload(v));
      break;
    }
    case OP_BTIMES: btimes_batch(collect<BtimesItem>(ops, [](Op* o) { return o->u.btimes; })); break;
    case OP_HEEV: heev_batch(collect<HeevItem>(ops, [](Op* o) { return o->u.heev; })); break;
    case OP_RESIDUAL: {
      auto v = collect<ResidualItem>(ops, [](Op* o) { return o->u.residual; });
      int mc = 1;
      for (auto& it : v) mc = std::max(mc, it.n_cols);
      LAUNCH(ctx, kb_residual, dim3((unsigned)mc, n), 256, 0, upload(v));
      break;
    }
    case OP_LAMBDA: {
      auto v = collect<LambdaItem>(ops, [](Op* o) { return o->u.lambda; });
      int mc = 1;
      for (auto& it : v) mc = std::max(mc, it.n_cols);
      LAUNCH(ctx, kb_lambda, dim3((unsigned)mc, n), 256, 0, upload(v));
      break;
    }
    case OP_COLNORMS: {
      auto v = collect<ColnormItem>(ops, [](Op* o) { return o->u.colnorm; });
      int mc = 1;
      for (auto& it : v) mc = std::max(mc, it.n_cols);
      LAUNCH(ctx, kb_col_norms, dim3((unsigned)mc, n), 256, 0, upload(v));
      break;
    }
    case OP_PRECOND: {
      auto v = collect<PrecondItem>(ops, [](Op* o) { return o->u.precond; });
      long long mt = 1;
      for (auto& it : v) mt = std::max(mt, it.n_rows * it.n_cols);
      LAUNCH(ctx, kb_precondition, dim3(gx_for(mt), n), 256, 0, upload(v));
      break;
    }
    case OP_SCALE: {
      auto v = collect<ScaleItem>(ops, [](Op* o) { return o->u.scale; });
      long long mt = 1;
      for (auto& it : v) mt = std::max(mt, it.n_rows * it.n_cols);
      LAUNCH(ctx, kb_scale_cols_inv, dim3(gx_for(mt), n), 256, 0, upload(v));
      break;
    }
    case OP_COPY2D: {
      auto v = collect<Copy2dItem>(ops, [](Op* o) { return o->u.copy2d; });
      long long mt = 1;
      for (auto& it : v) mt = std::max(mt, it.n_rows * it.n_cols);
      LAUNCH(ctx, kb_copy2d, dim3(gx_for(mt), n), 256, 0, upload(v));
      break;
    }
    case OP_MAKECP: {
      auto v = collect<MakecpItem>(ops, [](Op* o) { return o->u.makecp; });
      long long mt = 1;
      for (auto& it : v) mt = std::max(mt, (long long)it.n_rows * it.n_cols);
      LAUNCH(ctx, kb_make_cP, dim3(gx_for(mt), n), 256, 0, upload(v));
      break;
    }
    case OP_STATS: {
      auto v = collect<StatsItem>(ops, [](Op* o) { return o->u.stats; });
      LAUNCH(ctx, kb_matrix_stats, n, 256, 0, upload(v));
      break;
    }
    case OP_RANDN: {
      auto v = collect<RandnItem>(ops, [](Op* o) { return o->u.randn; });
      long long mt = 1;
      for (auto& it : v) mt = std::max(mt, it.n_rows);
      LAUNCH(ctx, kb_randn_col, dim3(gx_for(mt), n), 256, 0, upload(v));
      break;
    }
    case OP_APPLYH: apply_h_batch(collect<ApplyHItem>(ops, [](Op* o) { return o->u.applyh; })); break;
    case OP_D2H: {
      std::vector<GatherItem> v;
      for (Op* o : ops) {
        const D2HItem& d = o->u.d2h;
        REQUIRE(gather_used + d.n <= BatchSlot::GATHER_CAP, "batched LOBPCG: gather buffer too small");
        v.push_back(GatherItem{d.src, d.n, (int)gather_used});
        scatter.push_back({d.host_dst, {gather_used, d.n}});
        gather_used += d.n;
      }
      LAUNCH(ctx, kb_gather, n, 64, 0, upload(v), slot.gather.p);
      break;
    }
    default: throw Error(DFTK_B200_EINVAL, "batched LOBPCG: unknown operation");
  }
}
void BatchExec::issue(std::vector<Coro*>& coros) {
  bool any = false;
  for (auto& c : coros) any = any || c->cursor < c->ops.size();
  if (!any) return;
  rounds++;
  std::vector<Op*> batch;
  while (true) {
    // count the operation types at the cursors; run the rarest one first so that solves that are an operation behind
    // (a retry, a re-randomised column) catch up with the pack
    int count[OP_NTYPES] = {0};
    for (auto& c : coros)
      if (c->cursor < c->ops.size()) count[c->ops[c->cursor].type]++;
    int best = -1;
    for (int t = 0; t < OP_NTYPES; ++t)
      if (count[t] > 0 && (best < 0 || count[t] < count[best])) best = t;
    if (best < 0) break;
    batch.clear();
    for (auto& c : coros)
      if (c->cursor < c->ops.size() && c->ops[c->cursor].type == best) batch.push_back(&c->ops[c->cursor++]);
    launch(best, batch);
  }
  if (gather_used)
    CUDA_CHECK(cudaMemcpyAsync(slot.gather_h, slot.gather.p, gather_used * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_CHECK(cudaEventRecord(slot.ev, ctx->stream));
  in_flight = true;
}
void BatchExec::complete(std::vector<Coro*>& coros) {
  if (!in_flight) return;
  CUDA_CHECK(cudaEventSynchronize(slot.ev));
  in_flight = false;
  for (auto& s : scatter) memcpy(s.first, slot.gather_h + s.second.first, s.second.second * sizeof(double));
  scatter.clear();
  gather_used = 0;
  slot.ring.rewind();
  for (auto& c : coros) {
    c->ops.clear();
    c->cursor = 0;
  }
}

// ------------------------------------------------------------------ solver object
struct SolveArgs {
  cplx* X;
  double tol;
  int miniter, maxiter;
  int64_t n_conv_check;
  double* lambda_host;
  double* resid_host;
  int* n_iter;
  int64_t* n_matvec;
  int* converged;
};

struct Lobpcg {
  dftk_b200_kblock* kb;
  dftk_b200_ctx* ctx;
  int64_t N, M;
  bool use_prec;
  uint64_t rng_counter = 0x5EEDull;
  // device scalars / small vectors
  double *d_lam, *d_norms, *d_meankin, *d_stats, *d_w;
  cplx* d_cdots;
  // small dense scratch (leading dimension S3 = 3M)
  int64_t S3;
  cplx *G, *cX, *cP, *Ochol, *invR, *BYX, *tmpS;
  // big scratch
  cplx *AX, *R, *AR, *P, *AP, *nX, *nAX, *nR, *nP, *nAP;
  cplx* tmpN;  // N x M
  // batched small-matrix path (M <= SMALL_MAX_N): operations are recorded on `co` and launched by BatchExec
  bool small = false;
  Coro* co = nullptr;
  int64_t ldBYX = 0;
  int64_t n_chol_total = 0;

  // ---- INT8 tensor-core path of the large solves (gemm_backend 4): residue planes of the N_pw-sized blocks, prepared once
  //      and reused by every Gram and update product until the block's data changes (`touch`)
  struct PlaneEntry {
    const cplx* p = nullptr;
    int64_t ld = 0, cols = 0;
    I8Operand op;
    uint64_t stamp = 0;
    bool valid = false;
  };
  static constexpr int N_PLANE_SLOTS = 8;
  PlaneEntry planes[N_PLANE_SLOTS];
  uint64_t plane_clock = 0;
  // ---- plane-wave slabs of ONE k-block over the ranks of the context (single-k multi-GPU, SURVEY §8 f3): every tall
  //      block holds the rows [row0, row0 + N) of the n_pw coefficients.  Gram products, norms and dots are completed by an
  //      NCCL allreduce on the solve's stream, the small dense algebra runs replicated on identical data, and H is applied
  //      band-wise after a rows <-> bands exchange (grouped ncclSend/ncclRecv) -- `apply_h_slab` below.
  bool slab = false;
  int64_t Nfull = 0, row0 = 0;
  std::vector<int64_t> row_off;            // first row of every rank (+ end)
  cplx *slab_in = nullptr, *slab_out = nullptr, *slab_stage = nullptr;
  int64_t slab_exchange_bytes = 0;
  bool slab_timing = false;                // DFTK_B200_PROFILE: synchronising wall clock of the exchange / apply phases
  double slab_t_exchange = 0, slab_t_apply = 0;
  const double* kinp() const { return kb->kin.p + row0; }
  void reduce(void* dev, size_t n_doubles) {
    if (!slab || n_doubles == 0) return;
    NCCL_CHECK(ncclAllReduce(dev, dev, n_doubles, ncclFloat64, ncclSum, ctx->nccl, ctx->stream));
  }
  // tall blocks are distributed, the small dense matrices (at most 3M < N rows) are replicated
  bool is_dist(int64_t rows) const { return slab && rows == N; }
  void reduce_block(cplx* C, int64_t ldc, int64_t rows, int64_t cols) {
    if (!slab || rows == 0 || cols == 0) return;
    reduce(C, (size_t)(2 * (ldc * (cols - 1) + rows)));
  }
  void apply_h_slab(Mat in, Mat out);

  double flops = 0.0;      // GEMM flops executed by this solve (large path), added to ctx->lobpcg_flops at the end
  bool use_i8(int64_t rows) const { return !small && ctx->gemm_backend == 4 && rows >= ctx->i8_min_rows; }
  I8Operand planes_for(const Mat& X) {
    for (auto& e : planes)
      if (e.valid && e.p == X.p && e.ld == X.ld && e.cols == X.cols) {
        e.stamp = ++plane_clock;
        return e.op;
      }
    int slot = 0;
    for (int i = 0; i < N_PLANE_SLOTS; ++i) {
      if (!planes[i].valid) { slot = i; break; }
      if (planes[i].stamp < planes[slot].stamp) slot = i;
    }
    PlaneEntry& e = planes[slot];
    e.op = i8_prepare(ctx, X.p, X.ld, X.cols, X.rows, kb->i8_pool[slot], kb->i8_epool[slot]);
    e.p = X.p; e.ld = X.ld; e.cols = X.cols; e.valid = true; e.stamp = ++plane_clock;
    return e.op;
  }
  // the n complex numbers from p on are about to be (or have been) overwritten: planes of overlapping blocks are stale
  void touch(const cplx* p, int64_t n) {
    if (small || ctx->gemm_backend != 4) return;
    for (auto& e : planes)
      if (e.valid && p < e.p + e.ld * e.cols && e.p < p + n) e.valid = false;
  }
  void touch(const Mat& X) { touch(X.p, X.ld * X.cols); }

  Op& newop(int type) {
    co->ops.emplace_back();
    Op& o = co->ops.back();
    o.type = type;
    return o;
  }
  // host <- device doubles; the solve continues once the value is there
  void get(void* host, const void* dev, size_t bytes) {
    if (small) {
      Op& o = newop(OP_D2H);
      o.u.d2h = D2HItem{(const double*)dev, (int)(bytes / sizeof(double)), (double*)host};
      coro_yield(co);
      return;
    }
    // slab solves: what steers the iteration on the host is taken from rank 0, so that all ranks take the same branches
    // even if their replicated small dense results differed in the last bit
    if (slab) NCCL_CHECK(ncclBroadcast(dev, (void*)dev, bytes / sizeof(double), ncclFloat64, 0, ctx->nccl, ctx->stream));
    CUDA_CHECK(cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  }
  // solves of one batch meet here so that the same operations of all of them share launches again after a divergence
  void align() {
    if (!small) return;
    co->waiting_align = true;
    coro_yield(co);
  }

  static SmallMatList mklist(const std::vector<Mat>& v) {
    SmallMatList L{};
    REQUIRE(v.size() >= 1 && v.size() <= 3, "small path: block list too long");
    L.n = (int)v.size();
    int off = 0;
    for (int i = 0; i < 3; ++i) {
      L.start[i] = off;
      if (i < L.n) {
        L.p[i] = v[i].p;
        L.ld[i] = v[i].ld;
        L.cols[i] = (int)v[i].cols;
        off += (int)v[i].cols;
      } else {
        L.p[i] = nullptr;
        L.ld[i] = 0;
        L.cols[i] = 0;
      }
    }
    L.start[3] = off;
    for (int i = L.n; i < 4; ++i) L.start[i] = off;
    REQUIRE(off <= SMALL_MAX_COLS, "small path: too many columns");
    return L;
  }
  void small_gram(const std::vector<Mat>& A, const std::vector<Mat>& B, cplx* C, int64_t ldc, bool upper_only) {
    GramItem g{};
    g.A = mklist(A);
    g.B = mklist(B);
    if (g.A.start[g.A.n] == 0 || g.B.start[g.B.n] == 0) return;
    g.n_rows = A[0].rows;
    small_gram_geometry(ctx, g.n_rows, &g.n_ctas, &g.rows_per_cta);
    g.upper_only = upper_only ? 1 : 0;
    g.C = C;
    g.ldc = ldc;
    newop(OP_GRAM).u.gram = g;
  }
  void small_blocks_times(const std::vector<Mat>& Y, const cplx* c, int64_t ldc, int64_t ncols, Mat out, double alpha,
                          double beta) {
    if (ncols == 0 || out.rows == 0) return;
    REQUIRE(ncols <= SMALL_MAX_N, "small path: too many output columns");
    BtimesItem b{};
    b.Y = mklist(Y);
    b.cm = c; b.ldcm = ldc; b.ncols = (int)ncols; b.out = out.p; b.ldo = out.ld; b.n_rows = out.rows; b.alpha = alpha; b.beta = beta;
    newop(OP_BTIMES).u.btimes = b;
  }

  // One block operation of lobpcg_batch.cuh: recorded for the batched launch on the small path, launched on its own
  // otherwise (k_item on grid x block threads, the item passed as the kernel parameter)
  template <class Item>
  void block_op(int type, Item Op::U::*slot, const Item& it, unsigned grid, unsigned block = 256) {
    if (small) {
      newop(type).u.*slot = it;
      return;
    }
    LAUNCH(ctx, k_item<Item>, grid, block, 0, it);
  }

  void copy2d(Mat dst, Mat src) {
    if (src.rows == 0 || src.cols == 0) return;
    touch(dst.p, dst.ld * src.cols);
    block_op(OP_COPY2D, &Op::U::copy2d, Copy2dItem{dst.p, dst.ld, src.p, src.ld, src.rows, (int)src.cols}, nblk(src.rows * src.cols));
  }
  // contiguous device copy / zero fill of `n` complex numbers
  void copy_flat(cplx* dst, const cplx* src, int64_t n) {
    if (n <= 0) return;
    if (small) {
      newop(OP_COPY2D).u.copy2d = Copy2dItem{dst, n, src, n, n, 1};
      return;
    }
    touch(dst, n);
    if (src) CUDA_CHECK(cudaMemcpyAsync(dst, src, (size_t)n * sizeof(cplx), cudaMemcpyDeviceToDevice, ctx->stream));
    else CUDA_CHECK(cudaMemsetAsync(dst, 0, (size_t)n * sizeof(cplx), ctx->stream));
  }
  void col_norms(Mat X, double* out) {
    if (X.cols == 0) return;
    const bool dist = is_dist(X.rows);     // slab rows: squared norms, summed over the ranks
    block_op(OP_COLNORMS, &Op::U::colnorm, ColnormItem{X.p, X.ld, X.rows, (int)X.cols, dist, out}, (unsigned)X.cols);
    if (dist) {
      reduce(out, (size_t)X.cols);
      LAUNCH(ctx, k_sqrt_n, nblk(X.cols), 256, 0, out, X.cols);
    }
  }
  void scale_cols_inv(Mat X, const double* norms) {
    if (X.cols == 0) return;
    touch(X);
    block_op(OP_SCALE, &Op::U::scale, ScaleItem{X.p, X.ld, X.rows, (int)X.cols, norms}, nblk(X.rows * X.cols));
  }
  void matrix_stats(const cplx* A, int64_t ld, int64_t r, int64_t c, double* out) {
    block_op(OP_STATS, &Op::U::stats, StatsItem{A, ld, (int)r, (int)c, out}, 1, 1024);
  }
  void randn_col(cplx* x, int64_t n_rows, uint64_t seed) {
    touch(x, n_rows);
    const uint64_t s = seed + (is_dist(n_rows) ? 2 * (uint64_t)row0 : 0);   // slabs: one global random column
    block_op(OP_RANDN, &Op::U::randn, RandnItem{x, n_rows, s}, nblk(n_rows));
  }
  void stats(const cplx* A, int64_t ld, int64_t r, int64_t c, double* out4) {
    matrix_stats(A, ld, r, c, d_stats);
    get(out4, d_stats, 4 * sizeof(double));
  }
  double normest(const cplx* A, int64_t ld, int64_t n) {
    double s[4];
    stats(A, ld, n, n, s);
    return s[0] + std::sqrt(s[1]);
  }

  // C = op(A)' * B accumulated over block lists (LazyHcat products, :90-137)
  void gram(const std::vector<Mat>& A, const std::vector<Mat>& B, cplx* C, int64_t ldc, bool upper_only) {
    if (small) return small_gram(A, B, C, ldc, upper_only);
    if (!A.empty() && use_i8(A[0].rows)) {
      // INT8 tensor cores (wgmma s8, TMA-fed; i8emu.cu / i8tc2.cu): every distinct block is converted to residue
      // planes once and enters all its block products
      bool ok = A.size() + B.size() <= N_PLANE_SLOTS;
      for (auto& a : A) ok = ok && a.cols >= 32;
      for (auto& b : B) ok = ok && b.cols >= 32;
      if (ok) {
        std::vector<I8Operand> opA(A.size()), opB(B.size());
        for (size_t ia = 0; ia < A.size(); ++ia) opA[ia] = planes_for(A[ia]);
        for (size_t ib = 0; ib < B.size(); ++ib) opB[ib] = planes_for(B[ib]);
        int64_t oc = 0;
        for (size_t ib = 0; ib < B.size(); ++ib) {
          int64_t orow = 0;
          for (size_t ia = 0; ia < A.size(); ++ia) {
            if (!(upper_only && ib < ia)) {
              i8_gram(ctx, opA[ia], opB[ib], C + orow + ldc * oc, ldc, upper_only && ia == ib);
              flops += 8.0 * (double)A[ia].rows * A[ia].cols * B[ib].cols * ((upper_only && ia == ib) ? 0.5 : 1.0);
            }
            orow += A[ia].cols;
          }
          oc += B[ib].cols;
        }
        if (is_dist(A[0].rows)) reduce_block(C, ldc, orow_total(A), oc);
        return;
      }
    }
    const cplx one = make_double2(1, 0), zero = make_double2(0, 0);
    int64_t oc = 0;
    for (size_t ib = 0; ib < B.size(); ++ib) {
      int64_t orow = 0;
      for (size_t ia = 0; ia < A.size(); ++ia) {
        if (!(upper_only && ib < ia)) {
          zgemm(ctx, 2, A[ia].cols, B[ib].cols, A[ia].rows, one, A[ia].p, A[ia].ld, B[ib].p, B[ib].ld,
                zero, C + orow + ldc * oc, ldc, /*upper tiles only on diagonal blocks*/ upper_only && ia == ib);
          flops += 8.0 * (double)A[ia].rows * A[ia].cols * B[ib].cols * ((upper_only && ia == ib) ? 0.5 : 1.0);
        }
        orow += A[ia].cols;
      }
      oc += B[ib].cols;
    }
    if (!A.empty() && is_dist(A[0].rows)) reduce_block(C, ldc, orow_total(A), oc);
  }
  static int64_t orow_total(const std::vector<Mat>& A) {
    int64_t n = 0;
    for (auto& a : A) n += a.cols;
    return n;
  }
  // out (=|+=) alpha * [Y blocks] * c     (mul!(res, ::LazyHcat, B, α, β), :124-132)
  void blocks_times(const std::vector<Mat>& Y, const cplx* c, int64_t ldc, int64_t ncols, Mat out,
                    double alpha, double beta) {
    if (small) return small_blocks_times(Y, c, ldc, ncols, out, alpha, beta);
    for (auto& y : Y) flops += 8.0 * (double)out.rows * y.cols * ncols;
    if (!Y.empty() && use_i8(Y[0].rows) && Y.size() <= 3 && ncols >= 16) {
      bool ok = true;
      for (auto& y : Y) ok = ok && y.cols >= 32;
      if (ok) {
        I8Operand ops[3];
        for (size_t i = 0; i < Y.size(); ++i) ops[i] = planes_for(Y[i]);
        i8_update(ctx, (int)Y.size(), ops, c, ldc, ncols, out.p, out.ld, alpha, beta);
        touch(out.p, out.ld * ncols);
        return;
      }
    }
    touch(out.p, out.ld * ncols);
    int64_t off = 0;
    for (size_t i = 0; i < Y.size(); ++i) {
      zgemm(ctx, 0, Y[i].rows, ncols, Y[i].cols, make_double2(alpha, 0), Y[i].p, Y[i].ld, c + off, ldc,
            make_double2(i == 0 ? beta : 1.0, 0), out.p, out.ld);
      off += Y[i].cols;
    }
  }

  // SVD fallback of ortho! (only reachable when five shifted Cholesky factorisations fail); defined below
  void ortho_svd_fallback(Mat X, cplx* tmp, int64_t ldtmp);

  // ortho!(X) :216-261.  X: rows x n (in place).  `tmp` must hold rows x n.  Returns the growth factor.
  double ortho(Mat X, cplx* tmp, int64_t ldtmp) {
    const int64_t n = X.cols;
    if (n == 0) return 1.0;
    double growth = 1.0;
    int fallbacks = 0;
    if (small) {
      // gram -> fused safe_cholesky/inverse/normest (one CTA) -> one host sync -> X *= invR
      for (;;) {
        gram({X}, {X}, Ochol, S3, true);
        newop(OP_CHOL).u.chol = CholItem{Ochol, (long long)S3, (int)n, invR, (long long)S3, d_stats};
        double s[4];
        get(s, d_stats, 4 * sizeof(double));
        int nchol = (int)s[0];
        if (ctx->force_svd_fallback > 0) {
          ctx->force_svd_fallback--;
          nchol = 0;
        }
        if (nchol == 0) {      // safe_cholesky gave up (:226-231): SVD fallback, then a regular pass polishes the result
          if (++fallbacks > 3) throw Error(DFTK_B200_ENUM, "ortho!: cannot orthogonalise the block even after the SVD fallback");
          ortho_svd_fallback(X, tmp, ldtmp);
          growth = 1.0;
          continue;
        }
        newop(OP_RMUL).u.rmul = RmulItem{X.p, (long long)X.ld, (long long)X.rows, (int)n, invR, (long long)S3};
        const double norminvR = s[1];
        growth *= norminvR;
        const double condR = s[2] * norminvR;
        const double est = EPS * condR * condR;
        n_chol_total += nchol;
        if (nchol == 1 && est < 2 * EPS) break;
      }
      return growth;
    }
    for (;;) {
      gram({X}, {X}, Ochol, S3, true);
      LAUNCH(ctx, k_hermitize_upper, nblk(n * n), 256, 0, Ochol, S3, n);
      // safe_cholesky :190-210
      int nchol = 0;
      double alpha = 100.0;
      bool ok = false;
      double onorm = -1.0;
      while (nchol < 5) {
        nchol++;
        copy2d(Mat{invR, S3, n, n}, Mat{Ochol, S3, n, n});  // factor a copy (invR doubles as R storage)
        int info = potrf_upper(invR, n);
        if (info == 0) {
          // R = upper factor; keep R in tmpS, invert in invR
          LAUNCH(ctx, k_zero_lower, nblk(n * n), 256, 0, invR, S3, n);
          copy2d(Mat{tmpS, S3, n, n}, Mat{invR, S3, n, n});
          int info2 = trtri_upper(invR, n);
          double s[4];
          stats(invR, S3, n, n, s);
          if (info2 == 0 && s[2] == 0.0) {
            ok = true;
            break;
          }
        }
        if (onorm < 0) {
          double s[4];
          stats(Ochol, S3, n, n, s);
          onorm = std::sqrt(s[3]);
        }
        LAUNCH(ctx, k_add_diag, nblk(n), 256, 0, Ochol, S3, n, alpha * EPS * onorm);
        // note: the reference recomputes norm(O) of the shifted matrix; the difference is O(eps)
        alpha *= 10;
      }
      if (ctx->force_svd_fallback > 0) {
        ctx->force_svd_fallback--;
        ok = false;
      }
      if (!ok) {
        if (++fallbacks > 3) throw Error(DFTK_B200_ENUM, "ortho!: cannot orthogonalise the block even after the SVD fallback");
        ortho_svd_fallback(X, tmp, ldtmp);
        growth = 1.0;
        continue;
      }
      // X <- X * invR   (rmul!(X, invR))
      flops += 8.0 * (double)X.rows * n * n * 0.5;      // invR is upper triangular
      if (use_i8(X.rows) && n >= 32) {
        const I8Operand opX = planes_for(X);        // prepared for the Gram product above
        touch(tmp, ldtmp * n);
        i8_update(ctx, 1, &opX, invR, S3, n, tmp, ldtmp, 1.0, 0.0);
      } else {
        touch(tmp, ldtmp * n);
        zgemm(ctx, 0, X.rows, n, n, make_double2(1, 0), X.p, X.ld, invR, S3, make_double2(0, 0), tmp, ldtmp,
              /*invR is upper triangular*/ true);
      }
      copy2d(X, Mat{tmp, ldtmp, X.rows, n});
      double norminvR = normest(invR, S3, n);
      growth *= norminvR;
      double condR = normest(tmpS, S3, n) * norminvR;
      double est = EPS * condR * condR;
      n_chol_total += nchol;
      if (nchol == 1 && est < 2 * EPS) break;
    }
    return growth;
  }

  int potrf_upper(cplx* A, int64_t n) {
    int lwork = 0;
    CUSOLVER_CHECK(cusolverDnZpotrf_bufferSize(ctx->cusolver, CUBLAS_FILL_MODE_UPPER, (int)n,
                                               (cuDoubleComplex*)A, (int)S3, &lwork));
    char* w = ctx->solver_work.ensure((size_t)lwork * sizeof(cuDoubleComplex) + 16);
    int* dinfo = ctx->dev_info.ensure(4);
    CUSOLVER_CHECK(cusolverDnZpotrf(ctx->cusolver, CUBLAS_FILL_MODE_UPPER, (int)n, (cuDoubleComplex*)A,
                                    (int)S3, (cuDoubleComplex*)w, lwork, dinfo));
    ctx->launches++;
    int info = 0;
    CUDA_CHECK(cudaMemcpyAsync(&info, dinfo, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    return info;
  }
  int trtri_upper(cplx* A, int64_t n) {
    size_t wd = 0, wh = 0;
    CUSOLVER_CHECK(cusolverDnXtrtri_bufferSize(ctx->cusolver, CUBLAS_FILL_MODE_UPPER, CUBLAS_DIAG_NON_UNIT,
                                               n, CUDA_C_64F, A, S3, &wd, &wh));
    char* w = ctx->solver_work.ensure(wd + 16);
    std::vector<char> hw(wh + 16);
    int* dinfo = ctx->dev_info.ensure(4);
    CUSOLVER_CHECK(cusolverDnXtrtri(ctx->cusolver, CUBLAS_FILL_MODE_UPPER, CUBLAS_DIAG_NON_UNIT, n,
                                    CUDA_C_64F, A, S3, w, wd, hw.data(), wh, dinfo));
    ctx->launches++;
    int info = 0;
    CUDA_CHECK(cudaMemcpyAsync(&info, dinfo, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    return info;
  }
  // eigen(Hermitian(A)) upper triangle, leading dimension S3; eigenvectors overwrite A, eigenvalues -> d_w (ascending)
  // lam_out / n_keep (batched path only): the n_keep lowest eigenvalues are also written to lam_out
  void heev(cplx* A, int64_t n, double* lam_out = nullptr, int n_keep = 0) {
    if (small) {
      // one-CTA Jacobi per k-block (lobpcg_small.cuh): no library call, no host synchronisation; tmpS holds V
      newop(OP_HEEV).u.heev = HeevItem{A, (long long)S3, (int)n, d_w, tmpS, d_stats + 4, lam_out, n_keep};
      return;
    }
    // 64-bit generic API: unlike the legacy cusolverDnZheevd it has no OpenMP host stage whose speed depends on the
    // process' OMP_* environment (measured: 26 ms for n = 1509 under every setting vs 30-700 ms for Zheevd)
    if (!ctx->solver_params) CUSOLVER_CHECK(cusolverDnCreateParams(&ctx->solver_params));
    size_t wd = 0, wh = 0;
    CUSOLVER_CHECK(cusolverDnXsyevd_bufferSize(ctx->cusolver, ctx->solver_params, CUSOLVER_EIG_MODE_VECTOR,
                                               CUBLAS_FILL_MODE_UPPER, n, CUDA_C_64F, A, S3, CUDA_R_64F, d_w, CUDA_C_64F,
                                               &wd, &wh));
    char* w = ctx->solver_work.ensure(wd + 16);
    if (ctx->solver_host_work.size() < wh + 16) ctx->solver_host_work.resize(wh + 16);
    int* dinfo = ctx->dev_info.ensure(4);
    CUSOLVER_CHECK(cusolverDnXsyevd(ctx->cusolver, ctx->solver_params, CUSOLVER_EIG_MODE_VECTOR, CUBLAS_FILL_MODE_UPPER, n,
                                    CUDA_C_64F, A, S3, CUDA_R_64F, d_w, CUDA_C_64F, w, wd, ctx->solver_host_work.data(), wh,
                                    dinfo));
    ctx->launches++;
    int info = 0;
    CUDA_CHECK(cudaMemcpyAsync(&info, dinfo, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    if (info != 0) throw Error(DFTK_B200_ENUM, "rayleigh_ritz: heevd failed, info=" + std::to_string(info));
  }

  // ortho!(X, Y, BY=Y) :271-323.  X: rows x n in place; Y: block list with the same row count.
  void ortho_against(Mat X, const std::vector<Mat>& Y, cplx* tmp, int64_t ldtmp) {
    const int64_t n = X.cols;
    if (n == 0) return;
    const double tol = 2 * EPS;
    int64_t ny = 0;
    for (auto& y : Y) ny += y.cols;
    REQUIRE(ny <= ldBYX, "ortho_against: workspace too small");
    col_norms(X, d_norms);
    scale_cols_inv(X, d_norms);
    std::vector<double> norms(n);
    for (int niter = 1;; ++niter) {
      gram(Y, {X}, BYX, ldBYX, false);
      blocks_times(Y, BYX, ldBYX, n, X, -1.0, 1.0);  // X -= Y * BY'X
      // drop_small! :264-268
      col_norms(X, d_norms);
      // ||BY'X|| is needed below; it does not depend on the re-randomisation, so both results share one host sync
      matrix_stats(BYX, ldBYX, ny, n, d_stats);
      const size_t span = (size_t)(d_stats - d_norms) + 4;
      std::vector<double> both(span);
      get(both.data(), d_norms, span * sizeof(double));
      std::copy(both.begin(), both.begin() + n, norms.begin());
      const double* s = both.data() + (d_stats - d_norms);
      for (int64_t c = 0; c < n; ++c) {
        if (norms[c] <= tol) {
          Mat xc = X.cols_range(c, 1);
          rng_counter += 0x100000000ull;
          randn_col(xc.p, X.rows, rng_counter);
          // X[:,c] -= Y (BY' X[:,c])
          gram(Y, {xc}, tmpS, S3, false);
          blocks_times(Y, tmpS, S3, 1, xc, -1.0, 1.0);
        }
      }
      if (std::sqrt(s[3]) < tol && niter > 1) break;
      double growth = ortho(X, tmp, ldtmp);
      if (growth * EPS < tol) break;
      if (niter > 10) {
        // :307-314 "Ortho(X, Y) is failing badly, falling back to SVD": X <- U V' and return
        ortho_svd_fallback(X, tmp, ldtmp);
        ortho(X, tmp, ldtmp);
        break;
      }
    }
  }

  void prepare(SolveArgs& a);
  void body(SolveArgs& a);
};

// ---- SVD fallback of ortho! (lobpcg_hyper_impl.jl:226-231, :307-314): X <- U V' for X = U S V'.
// Through the eigendecomposition of the Gram matrix, X'X = V S² V': the columns of X V are S_l u_l.  Directions whose
// singular value is below sqrt(eps) S_max cannot be recovered from the Gram matrix (LAPACK's U is arbitrary there, too):
// they are replaced by random vectors projected against the recovered ones.  The caller runs a regular Cholesky pass
// afterwards, which removes what rounding left (the block is well conditioned by then).
__global__ void k_conj_transpose(const cplx* __restrict__ A, int64_t lda, cplx* __restrict__ B, int64_t ldb, int n) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * n) return;
  const int i = idx % n, j = idx / n;
  const cplx v = A[j + lda * i];
  B[i + ldb * j] = make_double2(v.x, -v.y);
}
void Lobpcg::ortho_svd_fallback(Mat X, cplx* tmp, int64_t ldtmp) {
  const int64_t n = X.cols;
  if (n == 0) return;
  if (small) {
    // everything this solve has recorded so far must have run: read something back (yields to the scheduler)
    double dummy[4];
    get(dummy, d_stats, 4 * sizeof(double));
  }
  // a rare recovery path, executed synchronously with the direct (immediate-launch) forms even inside a batched solve
  const bool was_small = small;
  small = false;
  // inside a pipelined batch the other group may be in flight and ctx->stream is this group's stream: the direct forms use the
  // context's workspaces and its cuBLAS / cuSOLVER handles (bound to the context's own stream), so everything is drained first
  // and the recovery runs on the context's own stream
  cudaStream_t group_stream = ctx->stream;
  if (was_small && ctx->batch_pipelined) {
    CUDA_CHECK(cudaDeviceSynchronize());
    ctx->stream = ctx->batch_user_stream;
  }
  try {
    const cplx one = make_double2(1, 0), zero = make_double2(0, 0);
    gram({X}, {X}, Ochol, S3, true);
    LAUNCH(ctx, k_hermitize_upper, nblk(n * n), 256, 0, Ochol, S3, n);
    heev(Ochol, n);                                                   // V in Ochol (columns), S² in d_w, ascending
    zgemm(ctx, 0, X.rows, n, n, one, X.p, X.ld, Ochol, S3, zero, tmp, ldtmp);   // T = X V
    Mat T{tmp, ldtmp, X.rows, n};
    std::vector<double> nrm(n);
    col_norms(T, d_norms);
    get(nrm.data(), d_norms, n * sizeof(double));
    double smax = 0.0;
    for (double v : nrm) smax = std::max(smax, v);
    REQUIRE(std::isfinite(smax) && smax > 0.0, "ortho!: SVD fallback on a zero or non-finite block");
    std::vector<int64_t> good, bad;
    for (int64_t c = 0; c < n; ++c) (nrm[c] > std::sqrt(EPS) * smax ? good : bad).push_back(c);
    scale_cols_inv(T, d_norms);                                       // u_l = X v_l / S_l (the lost ones are rewritten below)
    for (int64_t c : bad) {
      Mat tc = T.cols_range(c, 1);
      rng_counter += 0x100000000ull;
      randn_col(tc.p, X.rows, rng_counter);
      for (int pass = 0; pass < 2; ++pass)                            // project against all other columns, twice
        for (int64_t o = 0; o < n; ++o) {
          if (o == c || (std::find(bad.begin(), bad.end(), o) != bad.end() && o > c)) continue;
          Mat to = T.cols_range(o, 1);
          gram({to}, {tc}, tmpS, S3, false);
          zgemm(ctx, 0, X.rows, 1, 1, make_double2(-1, 0), to.p, to.ld, tmpS, S3, one, tc.p, tc.ld);
        }
      col_norms(tc, d_norms);
      scale_cols_inv(tc, d_norms);
    }
    LAUNCH(ctx, k_conj_transpose, nblk(n * n), 256, 0, (const cplx*)Ochol, S3, invR, S3, (int)n);   // V'
    zgemm(ctx, 0, X.rows, n, n, one, tmp, ldtmp, invR, S3, zero, X.p, X.ld);                          // X = U V'
    touch(X);
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  } catch (...) {
    small = was_small;
    ctx->stream = group_stream;
    throw;
  }
  small = was_small;
  ctx->stream = group_stream;
}

// H on a block of slab-distributed columns: rows <-> bands exchange, band-wise apply with the k-block's own kernels, and back.
// Rank r applies H to the columns [c_r, c_r+1) of the block (split evenly); what it sends to rank q -- its rows of q's
// columns -- is one contiguous piece of the column-major slab, what it receives is placed by a strided copy.
static inline int64_t split_start(int64_t n, int parts, int i) { return (n / parts) * i + std::min<int64_t>(i, n % parts); }
void Lobpcg::apply_h_slab(Mat in, Mat out) {
  const int R = ctx->nranks, me = ctx->rank;
  const int64_t nc = in.cols;
  REQUIRE(in.ld == N && out.ld == N, "slab apply: unexpected leading dimension");
  auto c0 = [&](int r) { return split_start(nc, R, r); };
  const int64_t my_c0 = c0(me), my_nc = c0(me + 1) - my_c0;
  double t0 = 0;
  auto tick = [&]() {
    if (!slab_timing) return 0.0;
    cudaStreamSynchronize(ctx->stream);
    const double t = SectionProf::now(), dt = t - t0;
    t0 = t;
    return dt;
  };
  tick();
  // rows -> bands
  NCCL_CHECK(ncclGroupStart());
  for (int r = 0; r < R; ++r) {
    const int64_t ncr = c0(r + 1) - c0(r), nr = row_off[r + 1] - row_off[r];
    if (ncr > 0) NCCL_CHECK(ncclSend(in.p + N * c0(r), (size_t)(2 * N * ncr), ncclFloat64, r, ctx->nccl, ctx->stream));
    if (my_nc > 0) NCCL_CHECK(ncclRecv(slab_stage + row_off[r] * my_nc, (size_t)(2 * nr * my_nc), ncclFloat64, r, ctx->nccl, ctx->stream));
  }
  NCCL_CHECK(ncclGroupEnd());
  slab_exchange_bytes += 16 * (N * (nc - my_nc) + (Nfull - N) * my_nc);   // sent by this rank, both directions
  slab_t_exchange += tick();
  if (my_nc > 0) {
    for (int r = 0; r < R; ++r) {
      const int64_t nr = row_off[r + 1] - row_off[r];
      copy2d(Mat{slab_in + row_off[r], Nfull, nr, my_nc}, Mat{slab_stage + row_off[r] * my_nc, nr, nr, my_nc});
    }
    kb_apply_local_kinetic(kb, slab_in, slab_out, my_nc, kb->has_V, kb->has_kin, false);
    kb_apply_nonlocal(kb, slab_in, slab_out, my_nc);
    for (int r = 0; r < R; ++r) {
      const int64_t nr = row_off[r + 1] - row_off[r];
      copy2d(Mat{slab_stage + row_off[r] * my_nc, nr, nr, my_nc}, Mat{slab_out + row_off[r], Nfull, nr, my_nc});
    }
  }
  slab_t_apply += tick();
  // bands -> rows
  NCCL_CHECK(ncclGroupStart());
  for (int r = 0; r < R; ++r) {
    const int64_t ncr = c0(r + 1) - c0(r), nr = row_off[r + 1] - row_off[r];
    if (my_nc > 0) NCCL_CHECK(ncclSend(slab_stage + row_off[r] * my_nc, (size_t)(2 * nr * my_nc), ncclFloat64, r, ctx->nccl, ctx->stream));
    if (ncr > 0) NCCL_CHECK(ncclRecv(out.p + N * c0(r), (size_t)(2 * N * ncr), ncclFloat64, r, ctx->nccl, ctx->stream));
  }
  NCCL_CHECK(ncclGroupEnd());
  slab_t_exchange += tick();
}

void Lobpcg::prepare(SolveArgs& a) {
  (void)a;
  S3 = 3 * M;
  ldBYX = 2 * M > S3 ? 2 * M : S3;
  const int64_t slab_cols = slab ? (M + ctx->nranks - 1) / ctx->nranks : 0;
  cplx* big = kb->lobpcg_ws.ensure((size_t)11 * N * M + (size_t)3 * Nfull * slab_cols);
  if (slab) {
    slab_in = big + 11 * N * M;
    slab_out = slab_in + Nfull * slab_cols;
    slab_stage = slab_out + Nfull * slab_cols;
  }
  AX = big; R = big + N * M; AR = big + 2 * N * M; P = big + 3 * N * M; AP = big + 4 * N * M;
  nX = big + 5 * N * M; nAX = big + 6 * N * M; nR = big + 7 * N * M; nP = big + 8 * N * M; nAP = big + 9 * N * M;
  tmpN = big + 10 * N * M;
  size_t small_elems = (size_t)S3 * S3 * 4 + (size_t)S3 * M * 2 + (size_t)ldBYX * M + 4 * M + 64;
  cplx* sm = kb->small_ws.ensure(small_elems);
  G = sm;
  Ochol = sm + S3 * S3;
  invR = sm + 2 * S3 * S3;
  tmpS = sm + 3 * S3 * S3;
  cX = sm + 4 * S3 * S3;
  cP = cX + S3 * M;
  BYX = cP + S3 * M;
  d_cdots = BYX + ldBYX * M;
  double* dsc = kb->scal.ensure(4 * M + 3 * S3 + 64);     // per k-block: batched solves run side by side
  d_lam = dsc;
  d_norms = dsc + M;
  d_meankin = dsc + 2 * M;
  d_w = dsc + 3 * M;
  d_stats = dsc + 3 * M + 3 * S3;       // [0..4) matrix stats / Cholesky stats, [4..8) Jacobi stats
}

void Lobpcg::body(SolveArgs& a) {
  cplx* Xio = a.X;
  const double tol = a.tol;
  const int miniter = a.miniter, maxiter = a.maxiter;
  int64_t n_conv_check = a.n_conv_check;
  if (n_conv_check <= 0 || n_conv_check > M) n_conv_check = M;

  SectionProf prof;
  prof.on = !small && getenv("DFTK_B200_PROFILE") != nullptr;
  prof.aggregate = prof.on && atoi(getenv("DFTK_B200_PROFILE")) == 2;
  prof.st = ctx->stream;
  slab_timing = slab && prof.on;

  Mat X{Xio, N, N, M};
  auto mat = [&](cplx* p) { return Mat{p, N, N, M}; };
  auto applyH = [&](Mat in, Mat out) {
    // A*X: full H apply on a block of columns (mul!(AX, A, X), :379,416)
    if (in.cols == 0) return;
    if (small) {
      newop(OP_APPLYH).u.applyh = ApplyHItem{kb, in.p, out.p, (int)in.cols};
      return;
    }
    touch(out);
    flops += 16.0 * (double)(slab ? Nfull : N) * kb->n_nl() * (slab ? (double)in.cols / ctx->nranks : (double)in.cols);
    if (slab) return apply_h_slab(in, out);
    kb_apply_local_kinetic(kb, in.p, out.p, in.cols, kb->has_V, kb->has_kin, false);
    kb_apply_nonlocal(kb, in.p, out.p, in.cols);
  };
  auto copycols = [&](cplx* dst, const cplx* src, int64_t c0, int64_t nc) { copy_flat(dst + N * c0, src + N * c0, N * nc); };

  std::vector<double> resid_hist((size_t)M * (maxiter + 1), 0.0);
  auto RH = [&](int64_t i, int it) -> double& { return resid_hist[(size_t)it * M + i]; };

  // X = ortho!(copy(X)) :370
  prof.begin("ortho(X0)");
  ortho(X, tmpN, N);
  align();
  prof.begin("H*X");
  int64_t n_matvec = M;
  applyH(X, mat(AX));
  prof.begin("misc");
  copy_flat(R, nullptr, 4 * N * M);      // R, AR, P, AP
  copy_flat(nR, nullptr, 3 * N * M);     // nR, nP, nAP
  copycols(nX, Xio, 0, M);
  copycols(nAX, AX, 0, M);
  // λ = compute_λ(X, AX, X)
  if (small) {
    newop(OP_LAMBDA).u.lambda = LambdaItem{Xio, AX, N, N, (int)M, d_lam};
  } else {
    columnwise_dots(ctx, Xio, N, AX, N, N, M, d_cdots);
    columnwise_dots(ctx, Xio, N, Xio, N, N, M, d_cdots + M);
    reduce(d_cdots, (size_t)(4 * M));
    LAUNCH(ctx, k_compute_lambda, nblk(M), 256, 0, (const cplx*)d_cdots, (const cplx*)(d_cdots + M), d_lam, M);
  }

  int64_t nlocked = 0, a0 = 0;
  int niter = 0;
  std::vector<double> norms(M + 8), lam_h(M);
  int64_t ncolsY = 0;
  int final_iter = maxiter;
  while (true) {
    const int64_t Ma = M - a0;
    std::vector<Mat> Y, AY;
    if (niter > 0) {
      align();
      prof.begin("H*R");
      applyH(mat(R).cols_from(a0), mat(AR).cols_from(a0));
      n_matvec += Ma;
      Y = {X.cols_from(a0), mat(R).cols_from(a0)};
      AY = {mat(AX).cols_from(a0), mat(AR).cols_from(a0)};
      if (niter > 1) {
        Y.push_back(mat(P).cols_from(a0));
        AY.push_back(mat(AP).cols_from(a0));
      }
      ncolsY = (int64_t)Y.size() * Ma;
      // rayleigh_ritz :141-171
      prof.begin("RR gram Y'AY");
      gram(Y, AY, G, S3, true);
      prof.begin("RR heevd");
      // only the block upper triangle of G is written; the eigensolver reads the upper triangle only
      heev(G, ncolsY, d_lam + a0, (int)Ma);
      prof.begin("X,AX = Y cX");
      // cX = vectors[:, 1:Ma], λ = values[1:Ma]
      copy2d(Mat{cX, S3, ncolsY, Ma}, Mat{G, S3, ncolsY, Ma});
      if (!small) CUDA_CHECK(cudaMemcpyAsync(d_lam + a0, d_w, Ma * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
      blocks_times(Y, cX, S3, Ma, mat(nX).cols_from(a0), 1.0, 0.0);
      blocks_times(AY, cX, S3, Ma, mat(nAX).cols_from(a0), 1.0, 0.0);
    }
    prof.begin("residual+precond");
    // residuals :443-445 (+ precondprep! :452-457 fused)
    touch(nR + N * a0, N * Ma);
    block_op(OP_RESIDUAL, &Op::U::residual, ResidualItem{nAX + N * a0, nX + N * a0, d_lam + a0, nR + N * a0, N, N, (int)Ma, slab,
                                                         use_prec ? kinp() : nullptr, d_norms, d_meankin}, (unsigned)Ma);
    if (slab) {
      reduce(d_norms, (size_t)(M + Ma));          // [d_norms, d_norms + M) and the Ma entries of d_meankin behind it
      LAUNCH(ctx, k_sqrt_n, nblk(Ma), 256, 0, d_norms, Ma);
    }
    {
      // one read-back: the residual norms and, on the small path, the status of the Jacobi eigensolver of this Rayleigh-Ritz step
      const size_t jacobi = (size_t)(d_stats - d_norms) + 4;
      std::vector<double> back(small ? jacobi + 4 : (size_t)Ma);
      get(back.data(), d_norms, back.size() * sizeof(double));
      std::copy(back.begin(), back.begin() + Ma, norms.begin());
      if (small && niter > 0 && back[jacobi] == 0.0) throw Error(DFTK_B200_ENUM, "rayleigh_ritz: Jacobi eigensolver did not converge");
    }
    for (int64_t i = 0; i < Ma; ++i) RH(a0 + i, niter) = norms[i];
    if (use_prec) {
      touch(nR + N * a0, N * Ma);
      block_op(OP_PRECOND, &Op::U::precond, PrecondItem{nR + N * a0, N, N, (int)Ma, kinp(), d_meankin}, nblk(N * Ma));
    }

    const int64_t prev_nlocked = nlocked;
    if (niter >= miniter) {
      for (int64_t i = nlocked; i < M; ++i) {
        if (RH(i, niter) < tol) nlocked++;
        else break;
      }
    }
    if (nlocked >= n_conv_check) {
      copycols(Xio, nX, a0, Ma);
      copycols(AX, nAX, a0, Ma);
      final_iter = niter;
      break;
    }
    const int64_t newly = nlocked - prev_nlocked;

    if (niter > 0) {
      const int64_t lenXn = Ma - newly;
      prof.begin("cP ortho");
      // cP = (cX - e)[:, newly:Ma]; ortho!(cP, cX, cX)
      block_op(OP_MAKECP, &Op::U::makecp, MakecpItem{cP, cX, S3, (int)ncolsY, (int)lenXn, (int)newly, (int)lenXn},
               nblk(ncolsY * lenXn));
      ortho_against(Mat{cP, S3, ncolsY, lenXn}, {Mat{cX, S3, ncolsY, Ma}}, G, S3);
      prof.begin("P,AP = Y cP");
      blocks_times(Y, cP, S3, lenXn, mat(nP).cols_from(a0 + newly), 1.0, 0.0);
      blocks_times(AY, cP, S3, lenXn, mat(nAP).cols_from(a0 + newly), 1.0, 0.0);
    }
    prof.begin("copies+check");
    copycols(Xio, nX, a0, Ma);
    copycols(AX, nAX, a0, Ma);
    copycols(R, nR, a0, Ma);
    // sanity check :531-535
    {
      col_norms(Mat{Xio + N * a0, N, N, Ma}, d_norms);
      get(norms.data(), d_norms, Ma * sizeof(double));
      for (int64_t i = 0; i < Ma; ++i)
        if (!(std::fabs(norms[i] * norms[i] - 1.0) < std::sqrt(EPS)))
          throw Error(DFTK_B200_ENUM, "LOBPCG is badly failing to keep the vectors normalized; this should never happen");
    }
    a0 += newly;
    std::vector<Mat> Z = {X};
    if (niter > 0) {
      copycols(P, nP, a0, M - a0);
      copycols(AP, nAP, a0, M - a0);
      Z.push_back(mat(P).cols_from(a0));
    }
    prof.begin("ortho R vs (X,P)");
    ortho_against(mat(R).cols_from(a0), Z, tmpN, N);
    prof.end();

    if (niter >= maxiter) break;
    niter++;
  }
  prof.report(niter);
  if (slab_timing)
    fprintf(stderr, "[dftk_b200 slab rank %d] H applies: exchange %.3f s (%.2f GB sent), band-wise apply incl. staging copies %.3f s\n",
            ctx->rank, slab_t_exchange, slab_exchange_bytes / 1e9, slab_t_apply);
  // final_retval :325-338
  get(lam_h.data(), d_lam, M * sizeof(double));
  std::vector<int64_t> perm(M);
  std::iota(perm.begin(), perm.end(), 0);
  bool sorted = std::is_sorted(lam_h.begin(), lam_h.end());
  if (!sorted) {
    std::stable_sort(perm.begin(), perm.end(), [&](int64_t p, int64_t q) { return lam_h[p] < lam_h[q]; });
    // permute X columns through tmpN
    for (int64_t c = 0; c < M; ++c) copy_flat(tmpN + N * c, Xio + N * perm[c], N);
    copy_flat(Xio, tmpN, N * M);
  }
  double maxres = 0.0;
  for (int64_t c = 0; c < M; ++c) {
    a.lambda_host[c] = lam_h[perm[c]];
    a.resid_host[c] = RH(perm[c], final_iter);
    if (c < n_conv_check) maxres = std::max(maxres, a.resid_host[c]);
  }
  *a.n_iter = final_iter;
  *a.n_matvec = n_matvec;
  *a.converged = maxres < tol ? 1 : 0;
  if (!small) {
    ctx->lobpcg_flops += flops;
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  }
}

// Batched execution: one coroutine per k-block runs `bodies[i]` (which records operations on L[i].co); BatchExec merges
// the recorded operations of all blocks into shared launches, one stream synchronisation per round.
static void run_batched(dftk_b200_ctx* ctx, std::vector<Lobpcg>& L, std::vector<std::function<void()>>& bodies) {
  const int64_t n_blocks = (int64_t)L.size();
  // Two pipelined groups when the batch is large enough: each group has its own stream and executor, and while the GPU runs
  // one group's round the host resumes the other group's solves, records and issues their next round -- the host work and the
  // synchronisation bubble of a round hide behind the other group's kernels (and small kernels of the two streams overlap).
  bool pipelined = ctx->batch_pipeline != 0 && n_blocks >= 8;
  for (auto& l : L)      // blocks whose nonlocal term would take the large (context-workspace) path stay in one group
    pipelined = pipelined && (l.kb->n_nl() == 0 || (l.kb->n_nl() <= SMALL_MAX_COLS && l.kb->PD.p != nullptr));
  const int G = pipelined ? 2 : 1;
  cudaStream_t user = ctx->stream;
  if (pipelined) {
    for (int g = 0; g < 2; ++g)
      if (!ctx->batch_streams[g]) CUDA_CHECK(cudaStreamCreateWithFlags(&ctx->batch_streams[g], cudaStreamNonBlocking));
    CUDA_CHECK(cudaStreamSynchronize(user));     // the inputs are ready before the groups start on their own streams
  }
  std::vector<std::unique_ptr<Coro>> coros;
  ucontext_t main_uc;
  ucontext_t* saved_main = g_main_uc;
  Coro* saved_coro = g_coro;
  g_main_uc = &main_uc;
  for (int64_t i = 0; i < n_blocks; ++i) {
    coros.emplace_back(new Coro());
    Coro* c = coros.back().get();
    c->stack_size = (size_t)1 << 20;
    c->stack.reset(new char[c->stack_size]);       // not value-initialised: pages are touched only as deep as the solve goes
    L[i].co = c;
    c->body = bodies[i];
    getcontext(&c->uc);
    c->uc.uc_stack.ss_sp = c->stack.get();
    c->uc.uc_stack.ss_size = c->stack_size;
    c->uc.uc_link = nullptr;
    makecontext(&c->uc, (void (*)())coro_entry, 0);
  }
  std::vector<Coro*> members[2];
  for (int64_t i = 0; i < n_blocks; ++i) members[i % G].push_back(coros[i].get());   // interleaved: similar work per group
  std::unique_ptr<BatchExec> exec[2];
  for (int g = 0; g < G; ++g) exec[g].reset(new BatchExec(ctx, ctx->slot[g]));
  auto stream_of = [&](int g) { return pipelined ? ctx->batch_streams[g] : user; };
  std::string first_err;
  int first_code = 0;
  auto restore = [&]() {
    ctx->stream = user;
    ctx->batch_pipelined = false;
    g_main_uc = saved_main;
    g_coro = saved_coro;
  };
  // resume the runnable solves of a group until each needs a value from the device, then enqueue what they recorded
  auto advance = [&](int g) {
    ctx->stream = stream_of(g);
    for (Coro* c : members[g]) {
      if (c->finished || c->waiting_align) continue;
      g_coro = c;
      swapcontext(&main_uc, &c->uc);
      if (c->failed && first_err.empty()) {
        first_err = c->err;
        first_code = c->err_code;
      }
    }
    if (first_err.empty()) exec[g]->issue(members[g]);
    ctx->stream = user;
  };
  try {
    ctx->batch_user_stream = user;
    ctx->batch_pipelined = pipelined;
    for (int g = 0; g < G; ++g) {
      ctx->stream = stream_of(g);
      exec[g]->reset_counters((size_t)members[g].size());
      ctx->stream = user;
    }
    bool done[2] = {false, G == 1};
    for (int g = 0; g < G && first_err.empty(); ++g) advance(g);
    while (first_err.empty() && !(done[0] && done[1])) {
      for (int g = 0; g < G && first_err.empty(); ++g) {
        if (done[g]) continue;
        ctx->stream = stream_of(g);
        exec[g]->complete(members[g]);
        ctx->stream = user;
        bool all_done = true, all_waiting = true;
        for (Coro* c : members[g]) {
          if (c->finished) continue;
          all_done = false;
          if (!c->waiting_align) all_waiting = false;
        }
        if (all_done) {
          done[g] = true;
          continue;
        }
        if (all_waiting)
          for (Coro* c : members[g]) c->waiting_align = false;
        advance(g);
      }
    }
  } catch (...) {
    restore();
    cudaDeviceSynchronize();
    throw;
  }
  restore();
  for (auto& l : L) l.co = nullptr;
  for (int g = 0; g < G; ++g) ctx->batch_rounds += exec[g]->rounds;
  if (!first_err.empty()) {
    cudaDeviceSynchronize();
    throw Error(first_code, first_err);
  }
  if (pipelined)
    for (int g = 0; g < 2; ++g) CUDA_CHECK(cudaStreamSynchronize(ctx->batch_streams[g]));
}

static void init_solver(Lobpcg& L, dftk_b200_kblock* kb, int64_t M, bool use_prec) {
  dftk_b200_ctx* ctx = kb->grid->ctx;
  const int64_t N = kb->n_pw;
  REQUIRE(M >= 1, "lobpcg: n_bands must be >= 1");
  REQUIRE(N > 3 * M, "The eigenproblem is too small, and the iterative eigensolver will fail; increase "
                     "the number of degrees of freedom, or use a dense eigensolver.");
  L.kb = kb;
  L.ctx = ctx;
  L.N = N;
  L.M = M;
  L.use_prec = use_prec && kb->has_kin;
  L.small = M <= SMALL_MAX_N && ctx->small_dense != 0;
}

// All k-blocks of a rank in lockstep (diagonalize_all_kblocks, src/eigen/diag.jl:16-52: independent eigenproblems).
int lobpcg_run_multi(int64_t n_blocks, dftk_b200_kblock* const* kbs, cplx* const* Xs, int64_t M, double tol, int miniter,
                     int maxiter, int64_t n_conv_check, bool use_prec, double* lambda_host, double* resid_host, int* n_iter,
                     int64_t* n_matvec, int* converged) {
  if (n_blocks <= 0) return 0;
  dftk_b200_ctx* ctx = kbs[0]->grid->ctx;
  std::vector<Lobpcg> L(n_blocks);
  std::vector<SolveArgs> A(n_blocks);
  for (int64_t i = 0; i < n_blocks; ++i) {
    REQUIRE(kbs[i] && Xs[i], "lobpcg: NULL k-block or orbital pointer");
    REQUIRE(kbs[i]->grid->ctx == ctx, "lobpcg: all k-blocks of a batch must belong to one context");
    init_solver(L[i], kbs[i], M, use_prec);
    A[i] = SolveArgs{Xs[i], tol, miniter, maxiter, n_conv_check, lambda_host + i * M, resid_host + i * M, n_iter + i,
                     n_matvec + i, converged + i};
    L[i].prepare(A[i]);
  }
  for (int64_t i = 0; i < n_blocks; ++i)
    for (int64_t j = 0; j < i; ++j) REQUIRE(kbs[i] != kbs[j], "lobpcg: a k-block appears twice in one batch");
  if (!L[0].small) {
    for (int64_t i = 0; i < n_blocks; ++i) L[i].body(A[i]);
    return 0;
  }
  std::vector<std::function<void()>> bodies;
  for (int64_t i = 0; i < n_blocks; ++i) {
    Lobpcg* Lp = &L[i];
    SolveArgs* Ap = &A[i];
    bodies.push_back([Lp, Ap]() { Lp->body(*Ap); });
  }
  run_batched(ctx, L, bodies);
  return 0;
}

// random_orbitals (src/common/orbitals.jl:82-87: ortho_qr(randn)) for several k-blocks at once: counter-based normal
// numbers, then the solver's own ortho! (Cholesky-QR with its retries) -- same span, orthonormal to 2 eps.
void random_orbitals_multi(int64_t n_blocks, dftk_b200_kblock* const* kbs, cplx* const* Xs, int64_t M, uint64_t seed) {
  if (n_blocks <= 0) return;
  dftk_b200_ctx* ctx = kbs[0]->grid->ctx;
  std::vector<Lobpcg> L(n_blocks);
  std::vector<SolveArgs> A(n_blocks);
  for (int64_t i = 0; i < n_blocks; ++i) {
    REQUIRE(kbs[i] && Xs[i] && kbs[i]->grid->ctx == ctx, "random_orbitals: bad k-block / orbital pointer");
    init_solver(L[i], kbs[i], M, false);
    A[i] = SolveArgs{Xs[i], 0, 0, 0, 0, nullptr, nullptr, nullptr, nullptr, nullptr};
    L[i].prepare(A[i]);
    const uint64_t s = seed * 0x9E3779B97F4A7C15ull + ((uint64_t)i << 40);
    for (int64_t c = 0; c < M; ++c) {
      const RandnItem col{Xs[i] + L[i].N * c, L[i].N, s + ((uint64_t)c << 24) * 2654435761ull};
      LAUNCH(ctx, k_item<RandnItem>, nblk(L[i].N), 256, 0, col);
    }
  }
  if (!L[0].small) {
    for (int64_t i = 0; i < n_blocks; ++i) L[i].ortho(Mat{Xs[i], L[i].N, L[i].N, M}, L[i].tmpN, L[i].N);
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    return;
  }
  std::vector<std::function<void()>> bodies;
  for (int64_t i = 0; i < n_blocks; ++i) {
    Lobpcg* Lp = &L[i];
    cplx* X = Xs[i];
    bodies.push_back([Lp, X, M]() { Lp->ortho(Mat{X, Lp->N, Lp->N, M}, Lp->tmpN, Lp->N); });
  }
  run_batched(ctx, L, bodies);
}

// Per-band kinetic and nonlocal energies of ALL k-blocks of a rank in four launches and one synchronisation
// (dftk_b200_band_energies does the same for one block): ekin / enl are n x ld_out host arrays.
void band_energies_multi(int64_t n, dftk_b200_kblock* const* kbs, const cplx* const* psi, const int* n_bands, int64_t ld_out,
                         double* ekin_host, double* enl_host) {
  if (n <= 0) return;
  dftk_b200_ctx* ctx = kbs[0]->grid->ctx;
  BatchExec exec(ctx, ctx->slot[0]);
  std::vector<KinDotsItem> kd;
  std::vector<GramItem> gr;
  std::vector<NlEnergyItem> ne;
  std::vector<GatherItem> ga;
  size_t used = 0;
  std::vector<std::pair<double*, std::pair<size_t, int>>> scatter;
  for (int64_t i = 0; i < n; ++i) {
    dftk_b200_kblock* kb = kbs[i];
    const int nb = n_bands[i];
    REQUIRE(kb && kb->grid->ctx == ctx && nb >= 0 && nb <= ld_out, "band_energies_multi: bad block");
    if (nb == 0) continue;
    REQUIRE(nb <= SMALL_MAX_N && kb->n_proj <= SMALL_MAX_COLS, "band_energies_multi: block too large for the batched path");
    double* sc = kb->scal.ensure(2 * SMALL_MAX_N + 8);
    if (ekin_host) {
      REQUIRE(kb->has_kin, "band_energies: no kinetic term");
      kd.push_back(KinDotsItem{psi[i], (long long)kb->n_pw, (long long)kb->n_pw, nb, kb->kin.p, sc});
      ga.push_back(GatherItem{sc, nb, (int)used});
      scatter.push_back({ekin_host + i * ld_out, {used, nb}});
      used += nb;
    }
    if (enl_host) {
      if (kb->n_proj == 0) {
        for (int b = 0; b < nb; ++b) enl_host[i * ld_out + b] = 0.0;
      } else {
        cplx* proj = kb->proj.ensure((size_t)2 * kb->n_proj * SMALL_MAX_N);
        gr.push_back(single_gram_item(ctx, kb->P.p, kb->n_pw, (int)kb->n_proj, psi[i], kb->n_pw, nb, kb->n_pw, proj));
        ne.push_back(NlEnergyItem{proj, kb->Dc.p, (int)kb->n_proj, nb, sc + SMALL_MAX_N});
        ga.push_back(GatherItem{sc + SMALL_MAX_N, nb, (int)used});
        scatter.push_back({enl_host + i * ld_out, {used, nb}});
        used += nb;
      }
    }
  }
  REQUIRE(used <= BatchSlot::GATHER_CAP, "band_energies_multi: gather buffer too small");
  BatchSlot& slot = ctx->slot[0];
  if (!kd.empty()) exec.kin_dots_batch(kd);
  if (!gr.empty()) {
    exec.gram_batch(gr);
    LAUNCH(ctx, kb_nl_energy, (unsigned)ne.size(), 64, 0, exec.upload(ne));
  }
  if (!ga.empty()) {
    LAUNCH(ctx, kb_gather, (unsigned)ga.size(), 64, 0, exec.upload(ga), slot.gather.p);
    CUDA_CHECK(cudaMemcpyAsync(slot.gather_h, slot.gather.p, used * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  }
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  slot.ring.rewind();
  for (auto& sct : scatter) memcpy(sct.first, slot.gather_h + sct.second.first, sct.second.second * sizeof(double));
}

struct OrbOccItem { const cplx* a; int nb, spin; const double* w; };

// n[s](i, j) += Σ_blocks of spin s Σ_b w_b a_ib conj(a_jb): one thread per output entry, the blocks and bands summed in
// a fixed order (the result does not depend on scheduling)
__global__ void k_orbital_occupation(const OrbOccItem* __restrict__ items, int n_items, int n_orb, int n_spin,
                                     cplx* __restrict__ n_out) {
  const int64_t nn = (int64_t)n_orb * n_orb;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_spin * nn) return;
  const int s = (int)(idx / nn), i = (int)(idx % nn % n_orb), j = (int)(idx % nn / n_orb);
  double re = 0.0, im = 0.0;
  for (int t = 0; t < n_items; ++t) {
    const OrbOccItem it = items[t];
    if (it.spin != s) continue;
    for (int b = 0; b < it.nb; ++b) {
      const cplx x = it.a[i + (int64_t)n_orb * b], y = it.a[j + (int64_t)n_orb * b];
      const double w = it.w[b];
      re += w * (x.x * y.x + x.y * y.y);
      im += w * (x.y * y.x - x.x * y.y);
    }
  }
  n_out[idx] = make_double2(n_out[idx].x + re, n_out[idx].y + im);
}

// Occupation matrices of the Hubbard orbitals over ALL k-blocks of a rank (hubbard.jl:201-232 before its mpi_sum):
// a = Φ' ψ per block, then the weighted Hermitian update into the block's spin channel.  Blocks of <= 32 bands and
// <= 96 orbitals share one batched projection launch; larger ones project with the block's own GEMMs (folded where it
// folds).  One launch for the update and one synchronisation in all.
void orbital_occupation_multi(int64_t n, dftk_b200_kblock* const* kbs, const cplx* const* psi, const double* occ_w_host,
                              int64_t ld_w, const int* n_bands, cplx* n_out) {
  if (n <= 0) return;
  dftk_b200_ctx* ctx = kbs[0]->grid->ctx;
  const int64_t n_orb = kbs[0]->n_orb;
  REQUIRE(n_orb > 0, "orbital_occupation_multi: the k-blocks have no orbitals (kblock_set_orbitals)");
  BatchExec exec(ctx, ctx->slot[0]);
  // the weights are read by the last launch: the ring takes them and the descriptors of both launches without wrapping
  DescRing& ring = ctx->slot[0].ring;
  const size_t w_bytes = (size_t)n * ld_w * sizeof(double);
  ring.reserve(DescRing::padded(w_bytes) + DescRing::padded(n * sizeof(GramItem)) + DescRing::padded(n * sizeof(OrbOccItem)),
               ctx->stream);
  const double* w_dev = (const double*)ring.put(occ_w_host, w_bytes, ctx->stream);
  std::vector<GramItem> gr;
  std::vector<OrbOccItem> items;
  int n_spin = 1;
  for (int64_t i = 0; i < n; ++i) {
    dftk_b200_kblock* kb = kbs[i];
    const int nb = n_bands[i];
    REQUIRE(kb && kb->grid->ctx == ctx && kb->n_orb == n_orb && nb >= 0 && nb <= ld_w,
            "orbital_occupation_multi: bad block (all blocks need the same number of orbitals)");
    if (nb == 0) continue;
    n_spin = std::max(n_spin, kb->spin + 1);
    cplx* a = kb->proj.ensure((size_t)n_orb * std::max(nb, SMALL_MAX_N));
    if (nb <= SMALL_MAX_N && n_orb <= SMALL_MAX_COLS) {
      gr.push_back(single_gram_item(ctx, kb->P.p + kb->n_pw * kb->n_proj, kb->n_pw, (int)n_orb, psi[i], kb->n_pw, nb, kb->n_pw, a));
    } else {
      kb_project_cols(kb, kb->n_proj, n_orb, psi[i], nb, a);
    }
    items.push_back(OrbOccItem{a, nb, kb->spin, w_dev + i * ld_w});
  }
  if (!gr.empty()) exec.gram_batch(gr);
  if (!items.empty()) {
    const int64_t total = n_spin * n_orb * n_orb;
    LAUNCH(ctx, k_orbital_occupation, (unsigned)((total + 255) / 256), 256, 0, exec.upload(items), (int)items.size(),
           (int)n_orb, n_spin, n_out);
  }
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  ring.rewind();
}

// C (nA x nB, host, column-major) = A' B for tall column-major blocks (n_rows >> nA, nB <= SMALL_MAX_COLS): one fused launch
// (CTA partials + last-CTA reduction, lobpcg_small.cuh).  Used by the host driver for the history dot products of Anderson
// mixing (src/scf/anderson.jl:81-130) instead of a QR factorisation of the N_fft x m history matrix.
void tall_gram(dftk_b200_ctx* ctx, const cplx* A, int64_t lda, int nA, const cplx* B, int64_t ldb, int nB, int64_t n_rows,
               cplx* out_host) {
  REQUIRE(nA >= 1 && nB >= 1 && nA <= SMALL_MAX_COLS && nB <= SMALL_MAX_COLS, "tall_gram: 1 <= columns <= 96");
  BatchExec exec(ctx, ctx->slot[0]);
  cplx* C = (cplx*)ctx->slot[0].gather.p;       // >= 96 x 96 complex fit the gather buffer
  std::vector<GramItem> v{single_gram_item(ctx, A, lda, nA, B, ldb, nB, n_rows, C)};
  exec.gram_batch(v);
  CUDA_CHECK(cudaMemcpyAsync(out_host, C, (size_t)nA * nB * sizeof(cplx), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  ctx->slot[0].ring.rewind();
}

// One k-block solved by all ranks of the context together (single-k multi-GPU): X (n_pw x M, identical on every rank on
// entry) is cut into row slabs, the slab solve runs (Lobpcg with slab = true), and the converged slabs are put together
// again on every rank by one broadcast per rank.
int lobpcg_run_slab(dftk_b200_kblock* kb, cplx* Xfull, int64_t M, double tol, int miniter, int maxiter, int64_t n_conv_check,
                    bool use_prec, double* lambda_host, double* resid_host, int* n_iter, int64_t* n_matvec, int* converged,
                    double* exchange_bytes) {
  dftk_b200_ctx* ctx = kb->grid->ctx;
  REQUIRE(ctx->nccl != nullptr, "lobpcg_slab: the context has no communicator (use ctx_create_dist)");
  REQUIRE(kb->n_orb == 0, "lobpcg_slab: k-blocks with Hubbard orbitals (kblock_set_orbitals) are not supported by the slab solver");
  const int R = ctx->nranks, me = ctx->rank;
  const int64_t Nf = kb->n_pw;
  Lobpcg L;
  init_solver(L, kb, M, use_prec);
  L.small = false;
  L.slab = true;
  L.Nfull = Nf;
  L.row_off.resize(R + 1);
  for (int r = 0; r <= R; ++r) L.row_off[r] = split_start(Nf, R, r);
  L.row0 = L.row_off[me];
  L.N = L.row_off[me + 1] - L.row_off[me];
  REQUIRE(split_start(Nf, R, R) - split_start(Nf, R, R - 1) > 3 * M,
          "lobpcg_slab: every rank needs more than 3 n_bands plane-wave rows");
  SolveArgs A{nullptr, tol, miniter, maxiter, n_conv_check, lambda_host, resid_host, n_iter, n_matvec, converged};
  L.prepare(A);
  // the slab of X lives behind the solver's workspace
  cplx* Xloc = kb->slab_x.ensure((size_t)L.N * M);
  L.copy2d(Mat{Xloc, L.N, L.N, M}, Mat{Xfull + L.row0, Nf, L.N, M});
  A.X = Xloc;
  L.body(A);
  // reassemble: the staging area (Nfull x ceil(M/R) x 3 complex numbers behind the workspace) takes one rank's slab at a time
  int64_t max_rows = 0;
  for (int r = 0; r < R; ++r) max_rows = std::max(max_rows, L.row_off[r + 1] - L.row_off[r]);
  cplx* stage = kb->slab_stage.ensure((size_t)max_rows * M);
  for (int r = 0; r < R; ++r) {
    const int64_t nr = L.row_off[r + 1] - L.row_off[r];
    NCCL_CHECK(ncclBroadcast(Xloc, stage, (size_t)(2 * nr * M), ncclFloat64, r, ctx->nccl, ctx->stream));
    L.copy2d(Mat{Xfull + L.row_off[r], Nf, nr, M}, Mat{stage, nr, nr, M});
  }
  CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
  if (exchange_bytes) *exchange_bytes = (double)L.slab_exchange_bytes;
  return 0;
}

void lobpcg_set_attributes() {
  const int big = 200 * 1024;
  CUDA_CHECK(cudaFuncSetAttribute(kb_heev, cudaFuncAttributeMaxDynamicSharedMemorySize, big));
  CUDA_CHECK(cudaFuncSetAttribute(kb_btimes, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
  CUDA_CHECK(cudaFuncSetAttribute(kb_gram, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
}

int lobpcg_run(dftk_b200_kblock* kb, cplx* Xio, int64_t M, double tol, int miniter, int maxiter,
               int64_t n_conv_check, bool use_prec, double* lambda_host, double* resid_host, int* n_iter_out,
               int64_t* n_matvec_out, int* converged_out) {
  return lobpcg_run_multi(1, &kb, &Xio, M, tol, miniter, maxiter, n_conv_check, use_prec, lambda_host, resid_host,
                          n_iter_out, n_matvec_out, converged_out);
}

}  // namespace dftk
