/*
 * krylov_oracle.c -- TEST INFRASTRUCTURE ONLY.  CPU restatement of the
 * Krylov.jl solvers (see krylov_oracle_impl.h for the per-function
 * reference citations and the parity-pinning status): every solver family's
 * header, instantiated in Float64 and Float32.  Built by oracle/Makefile into
 * oracle/libkrylov_oracle.so; loaded by oracle/oracle.py.
 * The product library (krylov.jl_b200/) never links, loads or calls this.
 */
#include <math.h>
#include <float.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

int oracle_dot_mode = 0;
void oracle_set_dot_mode(int m) { oracle_dot_mode = m; }
int oracle_precond_block = 0;
void oracle_set_precond_block(int bs) { oracle_precond_block = bs; }

/* ---- Float64 instantiation ---- */
#define REAL double
#define SUF(name) name##_f64
#define SQRT sqrt
#define FABS fabs
#define COPYSIGN copysign
#define POW pow
#define EPS DBL_EPSILON
#define FLTMAX_OF DBL_MAX
#include "krylov_oracle_impl.h"
#include "krylov_oracle_siblings.h"
#include "krylov_oracle_block.h"
#include "krylov_oracle_lsq.h"
#include "krylov_oracle_cgls.h"
#include "krylov_oracle_lslq.h"
#include "krylov_oracle_biorth.h"
#include "krylov_oracle_ares.h"
#include "krylov_oracle_adjoint.h"
#include "krylov_oracle_leastnorm.h"
#include "krylov_oracle_lnlq.h"
#include "krylov_oracle_cgne.h"
#include "krylov_oracle_processes.h"
#include "krylov_oracle_solve.h"
#undef REAL
#undef SUF
#undef SQRT
#undef FABS
#undef COPYSIGN
#undef POW
#undef EPS
#undef FLTMAX_OF

/* ---- Float32 instantiation ---- */
#define REAL float
#define SUF(name) name##_f32
#define SQRT sqrtf
#define FABS fabsf
#define COPYSIGN copysignf
#define POW powf
#define EPS FLT_EPSILON
#define FLTMAX_OF FLT_MAX
#include "krylov_oracle_impl.h"
#include "krylov_oracle_siblings.h"
#include "krylov_oracle_block.h"
#include "krylov_oracle_lsq.h"
#include "krylov_oracle_cgls.h"
#include "krylov_oracle_lslq.h"
#include "krylov_oracle_biorth.h"
#include "krylov_oracle_ares.h"
#include "krylov_oracle_adjoint.h"
#include "krylov_oracle_leastnorm.h"
#include "krylov_oracle_lnlq.h"
#include "krylov_oracle_cgne.h"
#include "krylov_oracle_processes.h"
#include "krylov_oracle_solve.h"


/* ---------------------------------------------------------------------------
 * CPU timing legs of bench.py (cpu_baseline / --impl reference).  Runs `iters`
 * iterations of the cg.jl:195-268 loop body (M = I, no stopping test, atol =
 * rtol = 0 semantics) and returns the wall time in seconds.
 *   threads == 1 : the faithful sequential port (SparseArrays' mul! is single
 *                  threaded, docs/src/tips.md:38).
 *   threads  > 1 : "generous" variant -- row-parallel SpMV and OpenMP BLAS-1 on
 *                  all requested host threads (what a multithreaded BLAS plus a
 *                  threaded mul! would give the reference).
 * ------------------------------------------------------------------------- */
#include <omp.h>
double oracle_cg_timed_f64(int n, const int *rowptr, const int *colind, const double *val, const double *b,
                           int iters, int threads, double *x_out, double *rnorm_out, double *hist_out /* iters+1 or NULL */) {
  double *x = calloc(n, sizeof(double)), *r = malloc(sizeof(double) * n), *p = malloc(sizeof(double) * n),
         *Ap = malloc(sizeof(double) * n);
  if (threads < 1) threads = 1;
  omp_set_num_threads(threads);
  double gamma = 0;
#pragma omp parallel for reduction(+ : gamma) schedule(static)
  for (int i = 0; i < n; i++) { r[i] = b[i]; p[i] = b[i]; gamma += b[i] * b[i]; }
  if (hist_out) hist_out[0] = sqrt(gamma);
  double t0 = omp_get_wtime();
  for (int it = 0; it < iters; it++) {
    double pAp = 0;
#pragma omp parallel for reduction(+ : pAp) schedule(static)
    for (int i = 0; i < n; i++) {
      double acc = 0;
      for (int k = rowptr[i]; k < rowptr[i + 1]; k++) acc += val[k] * p[colind[k]];
      Ap[i] = acc;
      pAp += p[i] * acc;
    }
    double alpha = gamma / pAp, gamma_next = 0;
#pragma omp parallel for reduction(+ : gamma_next) schedule(static)
    for (int i = 0; i < n; i++) {
      x[i] += alpha * p[i];
      r[i] -= alpha * Ap[i];
      gamma_next += r[i] * r[i];
    }
    double beta = gamma_next / gamma;
    gamma = gamma_next;
    if (hist_out) hist_out[it + 1] = sqrt(gamma);
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n; i++) p[i] = r[i] + beta * p[i];
  }
  double t1 = omp_get_wtime();
  if (x_out) memcpy(x_out, x, sizeof(double) * n);
  if (rnorm_out) *rnorm_out = sqrt(gamma);
  free(x); free(r); free(p); free(Ap);
  return t1 - t0;
}

int oracle_abi_version(void) { return 5; }
