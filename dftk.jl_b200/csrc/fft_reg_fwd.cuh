// SphereTablesX: device view of the pruning tables incl. the inverse z-plane map (register engine).
#pragma once
#include "fft_core.cuh"
namespace dftk {
struct SphereTablesX : SphereTables {
  const int* zc_of;  // [nz] plane index of wrapped z, or -1
  // range form (see SphereTablesHost); ranges_ok == 0 => fall back to zc_of / colmap lookups
  int ranges_ok, z_s0, z_n0, z_s1, z_n1;
  const int *pl_s0, *pl_n0, *pl_s1, *pl_n1, *pl_col0;
  const int *cx_s0, *cx_n0, *cx_s1, *cx_n1;   // per-column x ranges (slot order)
};
// plane index of wrapped z (or -1): pure arithmetic on the range form (no dependent global load).  The host only
// selects the register engine for k-blocks whose tables have the range form (always true for a k-point sphere).
HD int zc_index(const SphereTablesX& T, int iz) {
  unsigned a = (unsigned)(iz - T.z_s0), b = (unsigned)(iz - T.z_s1);
  return a < (unsigned)T.z_n0 ? (int)a : (b < (unsigned)T.z_n1 ? T.z_n0 + (int)b : -1);
}
struct PlaneCols {
  int s0, n0, s1, n1, col0;
  HD int col(int iy) const {
    unsigned a = (unsigned)(iy - s0), b = (unsigned)(iy - s1);
    return a < (unsigned)n0 ? col0 + (int)a : (b < (unsigned)n1 ? col0 + n0 + (int)b : -1);
  }
};
HD PlaneCols plane_cols(const SphereTablesX& T, int izc) {
  PlaneCols p;
  p.s0 = T.pl_s0[izc]; p.n0 = T.pl_n0[izc]; p.s1 = T.pl_s1[izc]; p.n1 = T.pl_n1[izc]; p.col0 = T.pl_col0[izc];
  return p;
}
// Branch-free predicated global accesses (a plain `cond ? *p : 0` compiles to a divergent-branch region per
// element, which serialises the loads of the unrolled butterflies).
HD cplx ld_pred(const cplx* p, bool ok) {
#if defined(__CUDA_ARCH__)
  double x, y;
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.s32 q, %3, 0;\n\tmov.f64 %0, 0d0000000000000000;\n\t"
               "mov.f64 %1, 0d0000000000000000;\n\t@q ld.global.v2.f64 {%0, %1}, [%2];\n\t}"
               : "=d"(x), "=d"(y) : "l"(p), "r"((int)ok));
  return make_double2(x, y);
#else
  return ok ? *p : make_double2(0.0, 0.0);
#endif
}
// L2 eviction policies: the potential V(r) (N_fft doubles, re-read by every band) should stay resident in the
// 50 MB L2 of the H100 while the per-band pruned intermediates stream through it once.
HD uint64_t l2_policy_evict_last() {
#if defined(__CUDA_ARCH__)
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
#else
  return 0;
#endif
}
HD uint64_t l2_policy_evict_first() {
#if defined(__CUDA_ARCH__)
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
#else
  return 0;
#endif
}
HD double ld_pred_hint(const double* p, bool ok, uint64_t pol) {
#if defined(__CUDA_ARCH__)
  double x;
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.s32 q, %2, 0;\n\tmov.f64 %0, 0d0000000000000000;\n\t"
               "@q ld.global.L2::cache_hint.f64 %0, [%1], %3;\n\t}" : "=d"(x) : "l"(p), "r"((int)ok), "l"(pol));
  return x;
#else
  (void)pol;
  return ok ? *p : 0.0;
#endif
}
HD cplx ld_pred_hint(const cplx* p, bool ok, uint64_t pol) {
#if defined(__CUDA_ARCH__)
  double x, y;
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.s32 q, %3, 0;\n\tmov.f64 %0, 0d0000000000000000;\n\t"
               "mov.f64 %1, 0d0000000000000000;\n\t@q ld.global.L2::cache_hint.v2.f64 {%0, %1}, [%2], %4;\n\t}"
               : "=d"(x), "=d"(y) : "l"(p), "r"((int)ok), "l"(pol));
  return make_double2(x, y);
#else
  (void)pol;
  return ok ? *p : make_double2(0.0, 0.0);
#endif
}
HD void st_pred_hint(cplx* p, cplx v, bool ok, uint64_t pol) {
#if defined(__CUDA_ARCH__)
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.s32 q, %3, 0;\n\t@q st.global.L2::cache_hint.v2.f64 [%0], {%1, %2}, %4;\n\t}"
               :: "l"(p), "d"(v.x), "d"(v.y), "r"((int)ok), "l"(pol) : "memory");
#else
  (void)pol;
  if (ok) *p = v;
#endif
}
HD double ld_pred(const double* p, bool ok) {
#if defined(__CUDA_ARCH__)
  double x;
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.s32 q, %2, 0;\n\tmov.f64 %0, 0d0000000000000000;\n\t"
               "@q ld.global.f64 %0, [%1];\n\t}" : "=d"(x) : "l"(p), "r"((int)ok));
  return x;
#else
  return ok ? *p : 0.0;
#endif
}
HD void st_pred(cplx* p, cplx v, bool ok) {
#if defined(__CUDA_ARCH__)
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.s32 q, %3, 0;\n\t@q st.global.v2.f64 [%0], {%1, %2};\n\t}"
               :: "l"(p), "d"(v.x), "d"(v.y), "r"((int)ok) : "memory");
#else
  if (ok) *p = v;
#endif
}
}  // namespace dftk
