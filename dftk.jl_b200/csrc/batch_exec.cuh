// The executor of the batched small-matrix kernels (lobpcg_batch.cuh; defined in lobpcg.cu): the item descriptors of
// every batched operation, and BatchExec, which stages them in a slot's descriptor ring and launches each operation for
// all items at once.  The LOBPCG scheduler records operations and has them launched a round at a time; the one-shot
// multi-block calls (band energies, Hubbard occupations, direct minimisation) call the per-operation methods directly.
#pragma once
#include "structs.cuh"
#include "lobpcg_small.cuh"

namespace dftk {

struct GramItem {
  SmallMatList A, B;
  long long rows_per_cta, n_rows;
  int n_ctas, upper_only;
  cplx* ws;            // n_ctas x (nA nB) partials of this item
  cplx* C;
  long long ldc;
  unsigned* counter;   // arrival counter of this item (zero between launches)
};
struct CholItem { const cplx* O; long long ldo; int n; cplx* invR; long long ldi; double* stats; };
struct RmulItem { cplx* X; long long ld, n_rows; int n; const cplx* invR; long long ldr; };
struct BtimesItem { SmallMatList Y; const cplx* cm; long long ldcm; int ncols; cplx* out; long long ldo, n_rows; double alpha, beta; };
struct HeevItem { cplx* G; long long ldg; int n; double* w; cplx* V; double* stats; double* lam_out; int n_keep; };
struct ResidualItem { const cplx* AX; const cplx* X; const double* lam; cplx* R; long long ld, n_rows; int n_cols, squared; const double* kin; double* norms; double* meankin; };
struct PrecondItem { cplx* R; long long ld, n_rows; int n_cols; const double* kin; const double* meankin; };
struct ColnormItem { const cplx* X; long long ld, n_rows; int n_cols, squared; double* norms; };
struct ScaleItem { cplx* X; long long ld, n_rows; int n_cols; const double* norms; };
struct Copy2dItem { cplx* dst; long long ldd; const cplx* src; long long lds, n_rows; int n_cols; };   // src == nullptr: zero fill
struct MakecpItem { cplx* cP; const cplx* cX; long long ld; int n_rows, n_cols, c0, lenXn; };
struct StatsItem { const cplx* A; long long ld; int n_rows, n_cols; double* stats; };
struct RandnItem { cplx* x; long long n_rows; unsigned long long seed; };
struct LambdaItem { const cplx* X; const cplx* AX; long long ld, n_rows; int n_cols; double* lam; };
struct GatherItem { const double* src; int n; int offset; };
struct KinDotsItem { const cplx* X; long long ld, n_rows; int n_cols; const double* kin; double* out; };
struct NlEnergyItem { const cplx* proj; const cplx* D; int np, nb; double* out; };

struct ApplyHItem { dftk_b200_kblock* kb; const cplx* in; cplx* out; int ncols; };

// C = A' B of single tall blocks, with the CTA geometry of the batched kernel
GramItem single_gram_item(dftk_b200_ctx* ctx, const cplx* A, int64_t lda, int nA, const cplx* B, int64_t ldb, int nB,
                          int64_t n_rows, cplx* C);
// out = alpha Y c + beta out of a single tall block Y (n_rows x nY, like out of leading dimension n_rows; c is nY x ncols,
// packed)
BtimesItem single_btimes_item(const cplx* Y, int nY, const cplx* c, int ncols, cplx* out, int64_t n_rows, double alpha,
                              double beta);

struct Op;
struct Coro;

// Launches the recorded operations: the same operation of several solves becomes one launch.  The descriptors go through
// the slot's ring, which complete() rewinds after the round's synchronisation; a one-shot caller rewinds it after its own.
struct BatchExec {
  dftk_b200_ctx* ctx;
  BatchSlot& slot;
  std::vector<std::pair<double*, std::pair<size_t, int>>> scatter;   // host_dst <- gather_h[offset .. offset+n)
  size_t gather_used = 0;
  int64_t rounds = 0;
  bool in_flight = false;

  BatchExec(dftk_b200_ctx* c, BatchSlot& s);
  BatchExec(const BatchExec&) = delete;
  BatchExec& operator=(const BatchExec&) = delete;
  // arrival counters of kb_gram, zeroed (also recovers from an aborted solve)
  void reset_counters(size_t n);
  template <class T>
  const T* upload(const std::vector<T>& items) {
    return slot.ring.put(items, ctx->stream);
  }
  template <class T, class F>
  std::vector<T> collect(const std::vector<Op*>& ops, F get) {
    std::vector<T> v;
    v.reserve(ops.size());
    for (Op* o : ops) v.push_back(get(o));
    return v;
  }
  unsigned gx_for(long long total) const {
    long long g = (total + 255) / 256;
    return (unsigned)std::max<long long>(1, std::min<long long>(g, (long long)ctx->sm_count * 32));
  }

  // one operation over all items (apply_h_batch: the local and kinetic part as the batched FFT pipeline, the nonlocal part
  // as one Gram and one update launch)
  void gram_batch(std::vector<GramItem>& v);
  void btimes_batch(const std::vector<BtimesItem>& v);
  void heev_batch(const std::vector<HeevItem>& v);
  void kin_dots_batch(const std::vector<KinDotsItem>& v);
  void apply_h_batch(const std::vector<ApplyHItem>& v);
  void launch(int type, const std::vector<Op*>& ops);
  // enqueue everything recorded by the solves since the last round (launches + the round's result gather) on ctx->stream
  void issue(std::vector<Coro*>& coros);
  // wait for the issued round, hand the gathered values to the solves
  void complete(std::vector<Coro*>& coros);
};

}  // namespace dftk
