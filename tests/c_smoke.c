/* Plain-C consumer of libdftk_b200.so (no CUDA headers, no Python): what a foreign-language binding does.
 * grid -> k-block -> H apply on HOST buffers (the library stages them), with a constant local potential c and a
 * kinetic term: (H psi)(G) = (c + kin(G)) psi(G) exactly, so the result is checked against a closed form.
 * Build: gcc tests/c_smoke.c -Iinclude -Ldftk.jl_b200 -l:libdftk_b200.so -Wl,-rpath,$PWD/dftk.jl_b200 -lm -o c_smoke
 * Exit codes: 0 ok, 77 no usable GPU (skip), 1 failure. */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include "dftk_b200.h"

#define CHECK(call)                                                                                   \
  do {                                                                                                \
    int rc_ = (call);                                                                                 \
    if (rc_ != 0) {                                                                                   \
      fprintf(stderr, "%s failed: %d: %s\n", #call, rc_, dftk_b200_last_error(ctx));                  \
      return 1;                                                                                       \
    }                                                                                                 \
  } while (0)

int main(void) {
  dftk_b200_ctx* ctx = NULL;
  if (dftk_b200_ctx_create(0, &ctx) != 0) {
    fprintf(stderr, "no sm_90 device: %s\n", dftk_b200_last_error(NULL));
    return 77;
  }
  const int n = 12;                       /* 12^3 cube, sphere = |G|^2 <= 16 in integer units */
  dftk_b200_grid* grid = NULL;
  CHECK(dftk_b200_grid_create(ctx, n, n, n, 100.0, &grid));
  int64_t* mapping = malloc(sizeof(int64_t) * n * n * n);
  double* kin = malloc(sizeof(double) * n * n * n);
  int64_t n_pw = 0;
  for (int z = 0; z < n; ++z)
    for (int y = 0; y < n; ++y)
      for (int x = 0; x < n; ++x) {
        int gx = x <= (n - 1) / 2 ? x : x - n, gy = y <= (n - 1) / 2 ? y : y - n, gz = z <= (n - 1) / 2 ? z : z - n;
        int g2 = gx * gx + gy * gy + gz * gz;
        if (g2 <= 16) {
          mapping[n_pw] = x + n * (y + (int64_t)n * z);   /* ascending, 0-based */
          kin[n_pw] = 0.5 * 0.3 * g2;
          n_pw++;
        }
      }
  dftk_b200_kblock* kb = NULL;
  CHECK(dftk_b200_kblock_create(grid, n_pw, mapping, kin, 0, NULL, NULL, 0, 1.0, &kb));
  const double c = -0.7;
  double* V = malloc(sizeof(double) * n * n * n);
  for (int i = 0; i < n * n * n; ++i) V[i] = c;
  CHECK(dftk_b200_kblock_set_potential(kb, V));
  const int nb = 3;
  double* psi = malloc(sizeof(double) * 2 * n_pw * nb);
  double* hpsi = malloc(sizeof(double) * 2 * n_pw * nb);
  for (int64_t i = 0; i < 2 * n_pw * nb; ++i) psi[i] = sin(0.37 * (double)i) + 0.1;
  CHECK(dftk_b200_apply_h(kb, psi, hpsi, nb));
  double err = 0.0;
  for (int b = 0; b < nb; ++b)
    for (int64_t i = 0; i < n_pw; ++i)
      for (int p = 0; p < 2; ++p) {
        double want = (c + kin[i]) * psi[2 * (i + n_pw * b) + p];
        double d = fabs(hpsi[2 * (i + n_pw * b) + p] - want);
        if (d > err) err = d;
      }
  printf("c_smoke: n_pw = %lld, max |H psi - (c + kin) psi| = %.3e, launches = %lld\n", (long long)n_pw, err,
         (long long)dftk_b200_launch_count(ctx, 0));
  dftk_b200_kblock_destroy(kb);
  dftk_b200_grid_destroy(grid);
  dftk_b200_ctx_destroy(ctx);
  return err < 1e-12 ? 0 : 1;
}
