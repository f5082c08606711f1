/*
 * krylov_oracle_impl.h -- TEST INFRASTRUCTURE ONLY (see oracle/README.md).
 *
 * CPU restatement of the Krylov.jl inner-iteration path, included twice by
 * krylov_oracle.c (REAL = double, REAL = float).  Plain sequential loops, no
 * FMA contraction (-ffp-contract=off), SpMV accumulates each row in ascending
 * column order (what SparseArrays' CSC mul! does for every y[i]).
 *
 * Every function cites the reference file:line it follows (paths relative to
 * the Krylov.jl tree @ v0.10.8).  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may use this code.
 *
 * PARITY STATUS: the scalar helpers (sym_givens, roots_quadratic, to_boundary)
 * and the solver end states are pinned against the reference's own known-answer
 * tests (tests/test_oracle_kat.py).  Per-iteration residual histories and exact
 * iteration counts on the benchmark configs are NOT pinned by any reference
 * test and Julia is not available here: for those, "parity unpinned".
 */

#ifndef REAL
#error "define REAL, SUF() and the math macros before including"
#endif

/* ---- operators: CSR (int32, 0-based) and optional diagonal preconditioners ---- */

typedef struct {
  int n;
  const int *rowptr;
  const int *colind;
  const REAL *val;
} SUF(csr);

/* kmul!(y, A, x) -> mul!(y, A, x)  (src/krylov_utils.jl:305).  Row i sums its
 * terms left to right in ascending column order, product rounded before the add. */
static void SUF(spmv)(const SUF(csr) *A, const REAL *x, REAL *y) {
  for (int i = 0; i < A->n; i++) {
    REAL acc = (REAL)0;
    for (int k = A->rowptr[i]; k < A->rowptr[i + 1]; k++) {
      REAL prod = A->val[k] * x[A->colind[k]];
      acc = acc + prod;
    }
    y[i] = acc;
  }
}

/* BLAS-1 wrappers, src/krylov_utils.jl:309-347 (sequential restatement). */
/* Test knob (oracle_set_dot_mode): 0 = the restatement's sequential sum in REAL; 1 = the same terms accumulated in
 * double and rounded once.  Float32 parity tests run both and take the gap between the two histories as the
 * measured sensitivity of the iteration to the rounding of its dot products (tests/test_gpu_solvers.py).
 * 2 = the order of the device's reductions at one CTA of 256 threads (n <= 256; NaN beyond): term i is thread i's
 * partial (REAL)0 + x[i]*y[i], each warp of 32 lanes folds in halves (lane l += lane l+16, +8, +4, +2, +1: what
 * warp_sum's xor butterfly leaves in lane 0), and the 8 warp sums, padded to 32 with zeros, fold the same way
 * (block_sum).  With it the oracle and the GPU must agree bit for bit (tests/test_gpu_exact_small.py). */
extern int oracle_dot_mode;
static REAL SUF(fold32)(REAL *v) {
  for (int s = 16; s > 0; s >>= 1)
    for (int l = 0; l < s; l++) v[l] = v[l] + v[l + s];
  return v[0];
}
static REAL SUF(kdot)(int n, const REAL *x, const REAL *y) {
  if (oracle_dot_mode == 1) {
    double s = 0.0;
    for (int i = 0; i < n; i++) { double p = (double)x[i] * (double)y[i]; s = s + p; }
    return (REAL)s;
  }
  if (oracle_dot_mode == 2) {
    if (n > 256) return (REAL)NAN;
    REAL lane[256], warp[32];
    for (int i = 0; i < 256; i++) { REAL p = i < n ? x[i] * y[i] : (REAL)0; lane[i] = (REAL)0 + p; }
    for (int w = 0; w < 32; w++) warp[w] = w < 8 ? SUF(fold32)(lane + 32 * w) : (REAL)0;
    return SUF(fold32)(warp);
  }
  REAL s = (REAL)0;
  for (int i = 0; i < n; i++) { REAL p = x[i] * y[i]; s = s + p; }
  return s;
}
static REAL SUF(knorm)(int n, const REAL *x) { return SQRT(SUF(kdot)(n, x, x)); }
static void SUF(kscal)(int n, REAL s, REAL *x) { for (int i = 0; i < n; i++) x[i] = s * x[i]; }
/* The norm of a solver's window of error estimates: a few scalars the product keeps on the host and sums there in
 * order, so a plain sequential sum whatever the dot mode. */
static REAL SUF(err_norm)(int w, const REAL *e) {
  REAL s = 0;
  for (int i = 0; i < w; i++) s += e[i] * e[i];
  return SQRT(s);
}
/* kdiv!(n,x,s) = kscal!(n, one/s, x)  (krylov_utils.jl:325) */
static void SUF(kdiv)(int n, REAL *x, REAL s) { SUF(kscal)(n, (REAL)1 / s, x); }
static void SUF(kcopy)(int n, REAL *y, const REAL *x) { memcpy(y, x, sizeof(REAL) * (size_t)n); }
/* kdivcopy!(n,y,x,s): y .= x ./ s  (krylov_utils.jl:334) -- a true division */
static void SUF(kdivcopy)(int n, REAL *y, const REAL *x, REAL s) { for (int i = 0; i < n; i++) y[i] = x[i] / s; }
static void SUF(kaxpy)(int n, REAL s, const REAL *x, REAL *y) {
  for (int i = 0; i < n; i++) { REAL p = s * x[i]; y[i] = y[i] + p; }
}
static void SUF(kaxpby)(int n, REAL s, const REAL *x, REAL t, REAL *y) {
  for (int i = 0; i < n; i++) { REAL a = s * x[i]; REAL b = t * y[i]; y[i] = a + b; }
}
static void SUF(kfill)(int n, REAL *x, REAL v) { for (int i = 0; i < n; i++) x[i] = v; }

/* mulorldiv!(y, P, x, ldiv) for P = Diagonal(d)  (krylov_utils.jl:307).
 * Test knob (oracle_set_precond_block(bs), bs >= 2): `d` then holds ceil(n/bs) dense bs x bs row-major diagonal
 * blocks (block-Jacobi, docs/src/preconditioners.md:33): mul! is the block product, ldiv! a dense solve per block
 * (Gaussian elimination with partial pivoting). */
extern int oracle_precond_block;
static void SUF(bdiagmul)(int n, int bs, REAL *y, const REAL *B, const REAL *x, int ldiv) {
  for (int r0 = 0; r0 < n; r0 += bs) {
    const int rows = (n - r0 < bs) ? n - r0 : bs;
    const REAL *Bk = B + (size_t)(r0 / bs) * bs * bs;
    if (!ldiv) {
      for (int i = 0; i < rows; i++) {
        REAL acc = (REAL)0;
        for (int j = 0; j < rows; j++) { REAL p = Bk[i * bs + j] * x[r0 + j]; acc = acc + p; }
        y[r0 + i] = acc;
      }
    } else {
      REAL a[8][9];
      for (int i = 0; i < rows; i++) { for (int j = 0; j < rows; j++) a[i][j] = Bk[i * bs + j]; a[i][rows] = x[r0 + i]; }
      for (int c = 0; c < rows; c++) {
        int piv = c;
        for (int i = c + 1; i < rows; i++) if (FABS(a[i][c]) > FABS(a[piv][c])) piv = i;
        if (piv != c) for (int j = 0; j <= rows; j++) { REAL t = a[c][j]; a[c][j] = a[piv][j]; a[piv][j] = t; }
        for (int i = c + 1; i < rows; i++) {
          REAL f = a[i][c] / a[c][c];
          for (int j = c; j <= rows; j++) a[i][j] = a[i][j] - f * a[c][j];
        }
      }
      for (int i = rows - 1; i >= 0; i--) {
        REAL s = a[i][rows];
        for (int j = i + 1; j < rows; j++) s = s - a[i][j] * y[r0 + j];
        y[r0 + i] = s / a[i][i];
      }
    }
  }
}
static void SUF(diagmul)(int n, REAL *y, const REAL *d, const REAL *x, int ldiv) {
  if (oracle_precond_block >= 2) { SUF(bdiagmul)(n, oracle_precond_block, y, d, x, ldiv); return; }
  if (ldiv) for (int i = 0; i < n; i++) y[i] = x[i] / d[i];
  else      for (int i = 0; i < n; i++) y[i] = d[i] * x[i];
}

/* ---- scalar helpers ---- */

/* sym_givens(a, b), real case: src/krylov_utils.jl:21-51 */
void SUF(oracle_sym_givens)(REAL a, REAL b, REAL *c, REAL *s, REAL *rho) {
  REAL sa = (REAL)((a > 0) - (a < 0)), sb = (REAL)((b > 0) - (b < 0));
  if (b == (REAL)0) {
    *c = sa + (REAL)(a == (REAL)0);
    *s = (REAL)0;
    *rho = FABS(a);
  } else if (a == (REAL)0) {
    *c = (REAL)0;
    *s = sb;
    *rho = FABS(b);
  } else if (FABS(b) > FABS(a)) {
    REAL t = a / b;
    *s = sb / SQRT((REAL)1 + t * t);
    *c = *s * t;
    *rho = b / *s;
  } else {
    REAL t = b / a;
    *c = sa / SQRT((REAL)1 + t * t);
    *s = *c * t;
    *rho = a / *c;
  }
}

/* roots_quadratic(q2, q1, q0; nitref): src/krylov_utils.jl:110-152.
 * Returns 0, or 1 where the reference raises ("doesn't have real roots"). */
int SUF(oracle_roots_quadratic)(REAL q2, REAL q1, REAL q0, int nitref, REAL *r1, REAL *r2) {
  REAL root1, root2;
  if (q2 == (REAL)0) {
    REAL root;
    if (q1 == (REAL)0) {
      if (q0 != (REAL)0) return 1;
      root = (REAL)0;
    } else {
      root = -q0 / q1;
    }
    *r1 = root; *r2 = root;
    return 0;
  }
  REAL rhs = SQRT(EPS) * q1 * q1;
  if (FABS(q0 * q2) > rhs) {
    REAL rho = q1 * q1 - 4 * q2 * q0;
    if (rho < 0) return 1;
    REAL d = -(q1 + COPYSIGN(SQRT(rho), q1)) / 2;
    root1 = d / q2;
    root2 = q0 / d;
  } else {
    root1 = -q1 / q2;
    root2 = (REAL)0;
  }
  for (int it = 0; it < nitref; it++) {
    REAL q = (q2 * root1 + q1) * root1 + q0;
    REAL dq = 2 * q2 * root1 + q1;
    if (dq == (REAL)0) continue;
    root1 = root1 - q / dq;
  }
  for (int it = 0; it < nitref; it++) {
    REAL q = (q2 * root2 + q1) * root2 + q0;
    REAL dq = 2 * q2 * root2 + q1;
    if (dq == (REAL)0) continue;
    root2 = root2 - q / dq;
  }
  *r1 = root1; *r2 = root2;
  return 0;
}

/* to_boundary(n, x, d, z, radius; flip, xNorm2, dNorm2, M, ldiv): src/krylov_utils.jl:375-402.
 * Mdiag == NULL means M === I.  Returns 0, or an error code where the reference raises:
 * 1 radius<=0, 2 zero direction, 3 outside the trust region, 4 no real roots. */
int SUF(oracle_to_boundary)(int n, const REAL *x, const REAL *d, REAL *z, REAL radius, int flip,
                            REAL xNorm2, REAL dNorm2, const REAL *Mdiag, int ldiv,
                            REAL *s1, REAL *s2) {
  if (!(radius > 0)) return 1;
  REAL rxd;
  if (Mdiag == NULL) {
    rxd = SUF(kdot)(n, x, d);
    if (dNorm2 == (REAL)0) dNorm2 = SUF(kdot)(n, d, d);
    if (xNorm2 == (REAL)0) xNorm2 = SUF(kdot)(n, x, x);
  } else {
    SUF(diagmul)(n, z, Mdiag, x, ldiv);
    rxd = SUF(kdot)(n, z, d);
    xNorm2 = SUF(kdot)(n, z, x);
    SUF(diagmul)(n, z, Mdiag, d, ldiv);
    dNorm2 = SUF(kdot)(n, z, d);
  }
  if (dNorm2 == (REAL)0) return 2;
  if (flip) rxd = -rxd;
  REAL radius2 = radius * radius;
  if (!(xNorm2 <= radius2)) return 3;
  if (SUF(oracle_roots_quadratic)(dNorm2, 2 * rxd, xNorm2 - radius2, 1, s1, s2)) return 4;
  return 0;
}

/* ---- solver result record (SimpleStats, src/krylov_stats.jl:24-36) ---- */
#ifndef ORACLE_STATS_DEFINED
#define ORACLE_STATS_DEFINED
typedef struct {
  int niter;
  int solved;
  int inconsistent;
  int indefinite;
  int npcCount;
  int nres;        /* entries written to residuals[] */
  int nAres;       /* entries written to Aresiduals[] / Acond[] (MINRES) */
  int error;       /* 0, or >0 where the reference would raise error(...) */
  char status[96];
} oracle_stats;

static void set_status(oracle_stats *st, const char *s) {
  strncpy(st->status, s, sizeof(st->status) - 1);
  st->status[sizeof(st->status) - 1] = 0;
}

/* Per-iteration callback of the solvers that take one (NULL: none): returns nonzero to stop. */
typedef int (*oracle_iter_cb)(int iter, void *user);

/* The keyword arguments of every solver; each reads the fields its reference signature has.  Scalars stay double
 * here and each body rounds them to REAL where the reference converts them. */
typedef struct {
  double atol, rtol, etol, axtol, btol, utol, utolx, utoly; /* NaN -> sqrt(eps(T)) */
  double conlim;                /* NaN -> 1/sqrt(eps(T)) */
  double artol;                 /* MINARES' Artol: NaN -> sqrt(eps(T)) */
  double lambda, sigma, radius;
  double gamma;                 /* CR: NaN -> sqrt(eps(T)) */
  int itmax;                    /* 0 -> the family's default (2n square, m + n rectangular) */
  int history;
  int window;                   /* 0 -> 5 */
  int memory;                   /* 0 -> 20 (5 for block_gmres) */
  int restart, reorthogonalization, linesearch;
  int ldiv;                     /* preconditioners applied with ldiv! instead of mul! */
  int check_curvature;          /* CG-Lanczos */
  int transfer_to_lsqr, transfer_to_craig;
  int transfer;                 /* BiLQ / BiLQR: transfer_to_bicg; TriLQR: transfer_to_usymcg */
  double timemax;               /* seconds; < 0: no limit */
  oracle_iter_cb callback;
  void *cb_user;
  int hist_cap;                 /* capacity of the history arrays */
} oracle_options;
/* Wall clock in seconds, for timemax. */
static double oracle_now(void) { struct timespec ts; timespec_get(&ts, TIME_UTC); return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec; }
#endif

/* One solve's operands: A is m x n (square solvers: m = n); At, Aᵀ as its own CSR, is NULL for the solvers that
 * do not apply it.  b, c, x0, y0 and the diagonals M, N are NULL where not given. */
typedef struct {
  int m, n;
  const int *rowptr, *colind;
  const REAL *val;
  const int *trowptr, *tcolind;
  const REAL *tval;
  const REAL *b, *c, *x0, *y0, *M, *N;
} SUF(problem);

/* One solve's results.  A NULL history is not written; residuals counts its entries in stats.nres, Aresiduals and
 * Acond in stats.nAres, every other history in its own n_ field (counts may exceed options.hist_cap, the entries
 * stored). */
typedef struct {
  REAL *x, *y;
  REAL *residuals, *Aresiduals, *Acond;
  REAL *err_lbnds, *err_ubnds_lq, *err_ubnds_cg, *error_bnd_x, *error_bnd_y, *residuals_dual;
  int n_err_lbnds, n_err_ubnds_lq, n_err_ubnds_cg, n_error_bnd_x, n_error_bnd_y, n_residuals_dual;
  REAL *npc_dir;
  REAL Anorm;
  int error_with_bnd, solved_primal, solved_dual;
} SUF(outputs);

#define PUSH(arr, cnt, v) do { if ((arr) && (cnt) < o->hist_cap) (arr)[(cnt)] = (v); (cnt)++; } while (0)

static REAL SUF(tol)(double t) { return isnan(t) ? SQRT(EPS) : (REAL)t; }

/* =========================== cg!  (src/cg.jl:120-291) =========================== */
/* Mdiag: NULL => M === I, else M = Diagonal(Mdiag).  x0: NULL => no warm start.
 * npc_dir: optional output (length n) when linesearch || radius > 0. */
static int SUF(cg)(int variant, const SUF(problem) *P, const oracle_options *o, SUF(outputs) *out, oracle_stats *st) {
  const int n = P->n;
  const REAL *b = P->b, *x0 = P->x0, *Mdiag = P->M;
  REAL *x = out->x, *residuals = out->residuals, *npc_dir_out = out->npc_dir;
  SUF(csr) A = {n, P->rowptr, P->colind, P->val};
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  REAL radius = (REAL)o->radius;
  int linesearch = o->linesearch, history = o->history, ldiv = o->ldiv;
  int warm_start = (x0 != NULL);
  if (linesearch && radius > 0) { st->error = 1; return 1; }     /* cg.jl:130 */
  if (warm_start && linesearch) { st->error = 2; return 2; }     /* cg.jl:131 */
  int MisI = (Mdiag == NULL);
  REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol);
  int itmax = o->itmax;

  REAL *r = malloc(sizeof(REAL) * n), *p = malloc(sizeof(REAL) * n), *Ap = malloc(sizeof(REAL) * n);
  REAL *zbuf = MisI ? NULL : malloc(sizeof(REAL) * n);
  REAL *npc_dir = (linesearch || radius > 0) ? malloc(sizeof(REAL) * n) : NULL;
  REAL *z = MisI ? r : zbuf;                                      /* cg.jl:148 */
  int rc = 0;

  SUF(kfill)(n, x, 0);                                            /* cg.jl:153 */
  if (warm_start) {                                               /* cg.jl:154-156 */
    SUF(spmv)(&A, x0, r);
    SUF(kaxpby)(n, 1, b, -1, r);
  } else {
    SUF(kcopy)(n, r, b);
  }
  if (!MisI) SUF(diagmul)(n, z, Mdiag, r, ldiv);
  SUF(kcopy)(n, p, z);
  REAL gamma = SUF(kdot)(n, r, z);                                /* cg.jl:162 */
  if (!(gamma >= 0)) { st->error = 3; rc = 3; goto done; }
  REAL rNorm = SQRT(gamma);
  if (history) PUSH(residuals, st->nres, rNorm);
  if (gamma == 0) {                                               /* cg.jl:166-174 */
    st->niter = 0; st->solved = 1; st->inconsistent = 0;
    set_status(st, "x is a zero-residual solution");
    if (warm_start) SUF(kaxpy)(n, 1, x0, x);
    goto done;
  }
  int iter = 0;
  if (itmax == 0) itmax = 2 * n;
  REAL pAp = 0, pNorm2 = gamma;
  REAL eps_ = atol + rtol * rNorm;                                /* cg.jl:181 */
  int solved = rNorm <= eps_, tired = iter >= itmax;
  int inconsistent = 0, on_boundary = 0, zero_curvature = 0;

  while (!(solved || tired || zero_curvature)) {                  /* cg.jl:195 */
    SUF(spmv)(&A, p, Ap);
    pAp = SUF(kdot)(n, p, Ap);
    if ((pAp <= EPS * pNorm2) && (radius == 0)) {                 /* cg.jl:198-210 */
      if (FABS(pAp) <= EPS * pNorm2) { zero_curvature = 1; inconsistent = !linesearch; }
      if (linesearch) {
        if (iter == 0) SUF(kcopy)(n, x, p);
        SUF(kcopy)(n, npc_dir, p);
        st->npcCount = 1; st->indefinite = 1; solved = 1;
      }
    }
    if (zero_curvature || solved) continue;
    REAL alpha = gamma / pAp, sigma;
    if (radius == 0) {
      sigma = alpha;
    } else {                                                      /* cg.jl:218-222 */
      REAL s1, s2; int e;
      if (MisI) e = SUF(oracle_to_boundary)(n, x, p, z, radius, 0, 0, pNorm2, NULL, 0, &s1, &s2);
      else      e = SUF(oracle_to_boundary)(n, x, p, z, radius, 0, 0, 0, Mdiag, !ldiv, &s1, &s2);
      if (e) { st->error = 10 + e; rc = st->error; goto done; }
      sigma = s1 > s2 ? s1 : s2;
    }
    if ((radius > 0) && ((pAp <= 0) || (alpha > sigma))) {        /* cg.jl:229-237 */
      alpha = sigma;
      if (pAp <= 0) { SUF(kcopy)(n, npc_dir, p); st->npcCount = 1; st->indefinite = 1; }
      on_boundary = 1;
    }
    SUF(kaxpy)(n, alpha, p, x);                                   /* cg.jl:239-240 */
    SUF(kaxpy)(n, -alpha, Ap, r);
    if (!MisI) SUF(diagmul)(n, z, Mdiag, r, ldiv);
    REAL gamma_next = SUF(kdot)(n, r, z);
    if (!(gamma_next >= 0)) { st->error = 3; rc = 3; goto done; }
    rNorm = SQRT(gamma_next);
    if (history) PUSH(residuals, st->nres, rNorm);
    int resid_decrease_mach = (rNorm + (REAL)1 <= (REAL)1);
    int resid_decrease_lim = rNorm <= eps_;
    solved = resid_decrease_lim || resid_decrease_mach || on_boundary;
    if (!solved) {                                                /* cg.jl:255-260 */
      REAL beta = gamma_next / gamma;
      pNorm2 = gamma_next + beta * beta * pNorm2;
      gamma = gamma_next;
      SUF(kaxpby)(n, 1, z, beta, p);
    }
    iter = iter + 1;
    tired = iter >= itmax;
  }
  if (solved && on_boundary) set_status(st, "on trust-region boundary");       /* cg.jl:272-278 */
  if (solved && st->indefinite) set_status(st, "nonpositive curvature");
  if (solved && !strcmp(st->status, "unknown")) set_status(st, "solution good enough given atol and rtol");
  if (zero_curvature) set_status(st, "zero curvature detected");
  if (tired) set_status(st, "maximum number of iterations exceeded");
  if (warm_start) SUF(kaxpy)(n, 1, x0, x);
  st->niter = iter; st->solved = solved; st->inconsistent = inconsistent;
done:
  if (npc_dir && npc_dir_out) SUF(kcopy)(n, npc_dir_out, npc_dir);
  free(r); free(p); free(Ap); free(zbuf); free(npc_dir);
  return rc;
}

/* ======================== bicgstab!  (src/bicgstab.jl:125-277) ======================== */
static int SUF(bicgstab)(int variant, const SUF(problem) *P, const oracle_options *o, SUF(outputs) *out, oracle_stats *st) {
  const int n = P->n;
  const REAL *b = P->b, *c_in = P->c, *x0 = P->x0, *Mdiag = P->M, *Ndiag = P->N;
  REAL *x = out->x, *residuals = out->residuals;
  SUF(csr) A = {n, P->rowptr, P->colind, P->val};
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  int history = o->history, ldiv = o->ldiv, warm_start = (x0 != NULL);
  int MisI = (Mdiag == NULL), NisI = (Ndiag == NULL);
  const REAL *c = c_in ? c_in : b;                                /* c = b default, bicgstab.jl:105 */
  REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol);
  int itmax = o->itmax;
  size_t nb = sizeof(REAL) * (size_t)n;
  REAL *r = malloc(nb), *p = malloc(nb), *v = malloc(nb), *s = malloc(nb), *qd = malloc(nb);
  REAL *tbuf = MisI ? NULL : malloc(nb), *yz = NisI ? NULL : malloc(nb);
  REAL *q = qd, *d = qd;                                          /* bicgstab.jl:153-157 */
  REAL *t = MisI ? d : tbuf;
  REAL *y = NisI ? p : yz;
  REAL *z = NisI ? s : yz;
  REAL *r0 = MisI ? r : qd;

  if (warm_start) { SUF(spmv)(&A, x0, r0); SUF(kaxpby)(n, 1, b, -1, r0); }
  else SUF(kcopy)(n, r0, b);
  SUF(kfill)(n, x, 0); SUF(kfill)(n, s, 0); SUF(kfill)(n, v, 0);
  if (!MisI) SUF(diagmul)(n, r, Mdiag, r0, ldiv);
  SUF(kcopy)(n, p, r);
  REAL alpha = 1, omega = 1, rho = 1;
  REAL rNorm = SUF(knorm)(n, r);
  if (history) PUSH(residuals, st->nres, rNorm);
  if (rNorm == 0) {
    st->niter = 0; st->solved = 1; st->inconsistent = 0;
    set_status(st, "x is a zero-residual solution");
    if (warm_start) SUF(kaxpy)(n, 1, x0, x);
    goto done;
  }
  int iter = 0;
  if (itmax == 0) itmax = 2 * n;
  REAL eps_ = atol + rtol * rNorm;
  REAL next_rho = SUF(kdot)(n, c, r);                             /* bicgstab.jl:196 */
  if (next_rho == 0) {
    st->niter = 0; st->solved = 0; st->inconsistent = 0;
    set_status(st, "Breakdown b\xe1\xb4\xb4" "c = 0");                      /* "Breakdown bᴴc = 0" */
    if (warm_start) SUF(kaxpy)(n, 1, x0, x);
    goto done;
  }
  int solved = rNorm <= eps_, tired = iter >= itmax, breakdown = 0;
  while (!(solved || tired || breakdown)) {                       /* bicgstab.jl:215 */
    iter = iter + 1;
    rho = next_rho;
    if (!NisI) SUF(diagmul)(n, y, Ndiag, p, ldiv);
    SUF(spmv)(&A, y, q);
    if (MisI) SUF(kcopy)(n, v, q); else SUF(diagmul)(n, v, Mdiag, q, ldiv);   /* :222 unguarded */
    alpha = rho / SUF(kdot)(n, c, v);
    SUF(kcopy)(n, s, r);
    SUF(kaxpy)(n, -alpha, v, s);
    SUF(kaxpy)(n, alpha, y, x);
    if (!NisI) SUF(diagmul)(n, z, Ndiag, s, ldiv);
    SUF(spmv)(&A, z, d);
    if (!MisI) SUF(diagmul)(n, t, Mdiag, d, ldiv);
    { REAL ts = SUF(kdot)(n, t, s); REAL tt = SUF(kdot)(n, t, t); omega = ts / tt; }
    SUF(kaxpy)(n, omega, z, x);
    SUF(kcopy)(n, r, s);
    SUF(kaxpy)(n, -omega, t, r);
    next_rho = SUF(kdot)(n, c, r);
    REAL beta = (next_rho / rho) * (alpha / omega);
    SUF(kaxpy)(n, -omega, v, p);
    SUF(kaxpby)(n, 1, r, beta, p);
    rNorm = SUF(knorm)(n, r);
    if (history) PUSH(residuals, st->nres, rNorm);
    int resid_decrease_mach = (rNorm + (REAL)1 <= (REAL)1);
    solved = (rNorm <= eps_) || resid_decrease_mach;
    tired = iter >= itmax;
    breakdown = (alpha == 0 || isnan(alpha));
  }
  if (tired) set_status(st, "maximum number of iterations exceeded");
  if (breakdown) set_status(st, "breakdown \xce\xb1\xe2\x82\x96 == 0");           /* "breakdown αₖ == 0" */
  if (solved) set_status(st, "solution good enough given atol and rtol");
  if (warm_start) SUF(kaxpy)(n, 1, x0, x);
  st->niter = iter; st->solved = solved; st->inconsistent = 0;
done:
  free(r); free(p); free(v); free(s); free(qd); free(tbuf); free(yz);
  return 0;
}

/* ========================== gmres!  (src/gmres.jl:121-384) ========================== */
static int SUF(gmres)(int variant, const SUF(problem) *P, const oracle_options *o, SUF(outputs) *out, oracle_stats *st) {
  const int n = P->n;
  const REAL *b = P->b, *x0 = P->x0, *Mdiag = P->M, *Ndiag = P->N;
  REAL *x = out->x, *residuals = out->residuals;
  SUF(csr) A = {n, P->rowptr, P->colind, P->val};
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  int history = o->history, ldiv = o->ldiv, warm_start = (x0 != NULL);
  int restart = o->restart, reorth = o->reorthogonalization;
  int MisI = (Mdiag == NULL), NisI = (Ndiag == NULL);
  REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol);
  int itmax = o->itmax;
  int mem = o->memory == 0 ? 20 : o->memory;
  if (mem > n) mem = n;                                           /* krylov_workspaces.jl:2900 */
  size_t nb = sizeof(REAL) * (size_t)n;
  REAL *w = malloc(nb);
  REAL *qbuf = MisI ? NULL : malloc(nb), *pbuf = NisI ? NULL : malloc(nb);
  REAL *dx = (restart || warm_start) ? calloc(n, sizeof(REAL)) : NULL;
  if (warm_start) SUF(kcopy)(n, dx, x0);
  int vcap = mem, scap = mem, rcap = mem * (mem + 1) / 2, zcap = mem;
  REAL **V = malloc(sizeof(REAL *) * vcap);
  for (int i = 0; i < vcap; i++) V[i] = malloc(nb);
  REAL *cc = malloc(sizeof(REAL) * scap), *ss = malloc(sizeof(REAL) * scap);
  REAL *zz = malloc(sizeof(REAL) * zcap), *R = malloc(sizeof(REAL) * rcap);
  int clen = mem, rlen = rcap, vlen = mem, zlen = mem;            /* Julia vector lengths */
  REAL *q = MisI ? w : qbuf, *r0 = MisI ? w : qbuf;               /* gmres.jl:150-151 */
  REAL *xr = restart ? dx : x;                                    /* gmres.jl:152 */

  SUF(kfill)(n, x, 0);
  if (warm_start) {                                               /* gmres.jl:158-161 */
    SUF(spmv)(&A, dx, w);
    SUF(kaxpby)(n, 1, b, -1, w);
    if (restart) SUF(kaxpy)(n, 1, dx, x);
  } else {
    SUF(kcopy)(n, w, b);
  }
  if (!MisI) SUF(diagmul)(n, r0, Mdiag, w, ldiv);
  REAL beta = SUF(knorm)(n, r0);
  REAL rNorm = beta;
  if (history) PUSH(residuals, st->nres, beta);
  REAL eps_ = atol + rtol * rNorm;
  if (beta == 0) {
    st->niter = 0; st->solved = 1; st->inconsistent = 0;
    set_status(st, "x is a zero-residual solution");
    if (warm_start) SUF(kaxpy)(n, 1, x0, x);   /* note: with restart x already holds dx; reference adds again (gmres.jl:178) */
    goto done;
  }
  mem = clen;
  int npass = 0, iter = 0, inner_iter = 0;
  if (itmax == 0) itmax = 2 * n;
  int inner_itmax = itmax;
  REAL btol = POW(EPS, (REAL)0.75);                               /* gmres.jl:195 */
  int breakdown = 0, inconsistent = 0, solved = rNorm <= eps_, tired = iter >= itmax;
  int inner_tired = inner_iter >= inner_itmax;
  (void)inner_tired;

  while (!(solved || tired || breakdown)) {                       /* gmres.jl:207 */
    int nr = 0;
    for (int i = 0; i < mem; i++) SUF(kfill)(n, V[i], 0);        /* only the first `mem` (=length(c) at entry) */
    for (int i = 0; i < clen; i++) { ss[i] = 0; cc[i] = 0; }
    for (int i = 0; i < rlen; i++) R[i] = 0;
    for (int i = 0; i < zlen; i++) zz[i] = 0;
    if (restart) {
      SUF(kfill)(n, xr, 0);
      if (npass >= 1) {
        SUF(spmv)(&A, x, w);
        SUF(kaxpby)(n, 1, b, -1, w);
        if (!MisI) SUF(diagmul)(n, r0, Mdiag, w, ldiv);
      }
    }
    beta = SUF(knorm)(n, r0);
    zz[0] = beta;
    SUF(kdivcopy)(n, V[0], r0, rNorm);                            /* gmres.jl:231 divides by rNorm */
    npass = npass + 1;
    inner_iter = 0;
    inner_tired = 0;
    while (!(solved || inner_tired || breakdown)) {               /* gmres.jl:237 */
      inner_iter = inner_iter + 1;
      if (!restart && (inner_iter > mem)) {                       /* gmres.jl:244-252 */
        int newr = rlen + inner_iter;
        if (newr > rcap) { rcap = 2 * newr; R = realloc(R, sizeof(REAL) * rcap); }
        for (int i = rlen; i < newr; i++) R[i] = 0;
        rlen = newr;
        if (clen + 1 > scap) { scap = 2 * (clen + 1); cc = realloc(cc, sizeof(REAL) * scap); ss = realloc(ss, sizeof(REAL) * scap); }
        ss[clen] = 0; cc[clen] = 0; clen++;
      }
      REAL *pv = V[inner_iter - 1];
      REAL *p = NisI ? pv : pbuf;
      if (!NisI) SUF(diagmul)(n, p, Ndiag, pv, ldiv);
      SUF(spmv)(&A, p, w);
      if (!MisI) SUF(diagmul)(n, q, Mdiag, w, ldiv);
      for (int i = 0; i < inner_iter; i++) {                      /* MGS, gmres.jl:259-262 */
        R[nr + i] = SUF(kdot)(n, V[i], q);
        SUF(kaxpy)(n, -R[nr + i], V[i], q);
      }
      if (reorth) {
        for (int i = 0; i < inner_iter; i++) {
          REAL Htmp = SUF(kdot)(n, V[i], q);
          R[nr + i] += Htmp;
          SUF(kaxpy)(n, -Htmp, V[i], q);
        }
      }
      REAL Hbis = SUF(knorm)(n, q);
      for (int i = 0; i < inner_iter - 1; i++) {                  /* gmres.jl:280-284 */
        REAL Rtmp = cc[i] * R[nr + i] + ss[i] * R[nr + i + 1];
        R[nr + i + 1] = ss[i] * R[nr + i] - cc[i] * R[nr + i + 1];
        R[nr + i] = Rtmp;
      }
      SUF(oracle_sym_givens)(R[nr + inner_iter - 1], Hbis, &cc[inner_iter - 1], &ss[inner_iter - 1], &R[nr + inner_iter - 1]);
      REAL zeta_next = ss[inner_iter - 1] * zz[inner_iter - 1];
      zz[inner_iter - 1] = cc[inner_iter - 1] * zz[inner_iter - 1];
      rNorm = FABS(zeta_next);
      if (history) PUSH(residuals, st->nres, rNorm);
      nr = nr + inner_iter;
      int resid_decrease_mach = (rNorm + (REAL)1 <= (REAL)1);
      breakdown = Hbis <= btol;
      solved = (rNorm <= eps_) || resid_decrease_mach;
      {
        int lim = restart ? (mem < inner_itmax ? mem : inner_itmax) : inner_itmax;
        inner_tired = inner_iter >= lim;
      }
      if (!(solved || inner_tired || breakdown)) {                /* gmres.jl:318-327 */
        if (!restart && (inner_iter >= mem)) {
          if (vlen + 1 > vcap) { vcap = 2 * (vlen + 1); V = realloc(V, sizeof(REAL *) * vcap); }
          V[vlen++] = malloc(nb);
          if (zlen + 1 > zcap) { zcap = 2 * (zlen + 1); zz = realloc(zz, sizeof(REAL) * zcap); }
          zz[zlen++] = 0;
        }
        SUF(kdivcopy)(n, V[inner_iter], q, Hbis);
        zz[inner_iter] = zeta_next;
      }
    }
    REAL *y = zz;                                                 /* gmres.jl:331-345 */
    for (int i = inner_iter; i >= 1; i--) {
      int pos = nr + i - inner_iter;                              /* 1-based */
      for (int j = inner_iter; j >= i + 1; j--) {
        y[i - 1] = y[i - 1] - R[pos - 1] * y[j - 1];
        pos = pos - j + 1;
      }
      if (FABS(R[pos - 1]) <= btol) { y[i - 1] = 0; inconsistent = 1; }
      else y[i - 1] = y[i - 1] / R[pos - 1];
    }
    for (int i = 0; i < inner_iter; i++) SUF(kaxpy)(n, y[i], V[i], xr);
    if (!NisI) { SUF(kcopy)(n, pbuf, xr); SUF(diagmul)(n, xr, Ndiag, pbuf, ldiv); }
    if (restart) SUF(kaxpy)(n, 1, xr, x);
    inner_itmax = inner_itmax - inner_iter;
    iter = iter + inner_iter;
    tired = iter >= itmax;
  }
  if (tired) set_status(st, "maximum number of iterations exceeded");
  if (solved) set_status(st, "solution good enough given atol and rtol");
  if (inconsistent) set_status(st, "found approximate least-squares solution");
  if (warm_start && !restart) SUF(kaxpy)(n, 1, x0, x);
  st->niter = iter; st->solved = solved; st->inconsistent = inconsistent;
done:
  for (int i = 0; i < vlen; i++) free(V[i]);
  free(V); free(cc); free(ss); free(zz); free(R); free(w); free(qbuf); free(pbuf); free(dx);
  return 0;
}

/* ========================== minres!  (src/minres.jl:164-485) ========================== */
static int SUF(minres)(int variant, const SUF(problem) *P, const oracle_options *o, SUF(outputs) *out, oracle_stats *st) {
  const int n = P->n;
  const REAL *b = P->b, *x0 = P->x0, *Mdiag = P->M;
  REAL *x = out->x, *residuals = out->residuals, *Aresiduals = out->Aresiduals, *Aconds = out->Acond;
  REAL *npc_dir_out = out->npc_dir;
  SUF(csr) A = {n, P->rowptr, P->colind, P->val};
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  int history = o->history, ldiv = o->ldiv, warm_start = (x0 != NULL), linesearch = o->linesearch;
  if (warm_start && linesearch) { st->error = 2; return 2; }      /* minres.jl:174 */
  int MisI = (Mdiag == NULL);
  REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol);
  REAL etol = SUF(tol)(o->etol);
  REAL conlim = isnan(o->conlim) ? (REAL)1 / SQRT(EPS) : (REAL)o->conlim;
  REAL lambda = (REAL)o->lambda;
  int itmax = o->itmax;
  int window = o->window == 0 ? 5 : o->window;
  size_t nb = sizeof(REAL) * (size_t)n;
  REAL *r1 = malloc(nb), *r2 = malloc(nb), *w1 = malloc(nb), *w2 = malloc(nb), *y = malloc(nb);
  REAL *vbuf = MisI ? NULL : malloc(nb);
  REAL *npc_dir = linesearch ? malloc(nb) : NULL;
  REAL *err_vec = calloc(window, sizeof(REAL));
  REAL *v = MisI ? r2 : vbuf;                                     /* minres.jl:193 */
  REAL epsM = EPS;
  REAL ctol = conlim > 0 ? (REAL)1 / conlim : (REAL)0;
  int rc = 0;
  int nAc = 0;

  SUF(kfill)(n, x, 0);
  if (warm_start) {
    SUF(spmv)(&A, x0, r1);
    if (lambda != 0) SUF(kaxpy)(n, lambda, x0, r1);
    SUF(kaxpby)(n, 1, b, -1, r1);
  } else {
    SUF(kcopy)(n, r1, b);
  }
  SUF(kcopy)(n, r2, r1);
  if (!MisI) SUF(diagmul)(n, v, Mdiag, r1, ldiv);
  if (linesearch) SUF(kcopy)(n, npc_dir, v);
  REAL beta1 = SUF(kdot)(n, r1, v);
  if (beta1 < 0) { st->error = 4; rc = 4; goto done; }
  if (beta1 == 0) {                                               /* minres.jl:220-231 */
    st->niter = 1; st->solved = 1; st->inconsistent = 0;
    set_status(st, "x is a zero-residual solution");
    if (history) { PUSH(residuals, st->nres, beta1); PUSH(Aresiduals, st->nAres, 0); PUSH(Aconds, nAc, 0); }
    if (warm_start) SUF(kaxpy)(n, 1, x0, x);
    goto done;
  }
  beta1 = SQRT(beta1);
  REAL beta = beta1, oldbeta = 0, deltabar = 0, eps_rot = 0, rNorm = beta1;
  if (history) PUSH(residuals, st->nres, beta1);
  REAL phibar = beta1, rhs1 = beta1, rhs2 = 0, gmax = 0, gmin = (REAL)INFINITY;
  REAL cs = -1, sn = 0;
  SUF(kfill)(n, w1, 0); SUF(kfill)(n, w2, 0);
  REAL ANorm2 = 0, ANorm = 0, Acond = 0, ArNorm = 0, xNorm = 0;
  if (history) PUSH(Aconds, nAc, Acond);
  if (history) PUSH(Aresiduals, st->nAres, ArNorm);
  REAL xENorm2 = 0, err_lbnd = 0;
  int iter = 0;
  if (itmax == 0) itmax = 2 * n;
  REAL eps_ = atol + rtol * beta1;                                /* minres.jl:269 */
  int solved = 0, solved_mach = 0, solved_lim = 0, tired = iter >= itmax;
  int ill_cond = 0, ill_cond_mach = 0, ill_cond_lim = 0;
  int zero_resid = (rNorm <= eps_), zero_resid_mach = zero_resid, zero_resid_lim = zero_resid;
  int fwd_err = 0;
  (void)zero_resid_mach; (void)zero_resid_lim; (void)solved_mach; (void)solved_lim; (void)xNorm; (void)rhs1;
  REAL delta_w = 0, beta_w = 0, zeta_k = 0, zeta_km1 = 0;
  REAL *wa = w1, *wb = w2;                                        /* @kswap! swaps bindings */

  while (!(solved || tired || ill_cond)) {                        /* minres.jl:285 */
    iter = iter + 1;
    SUF(spmv)(&A, v, y);
    if (lambda != 0) SUF(kaxpy)(n, lambda, v, y);
    SUF(kdiv)(n, y, beta);
    if (iter >= 2) SUF(kaxpy)(n, -beta / oldbeta, r1, y);
    REAL alpha = SUF(kdot)(n, v, y) / beta;
    SUF(kaxpy)(n, -alpha / beta, r2, y);
    REAL delta = cs * deltabar + sn * alpha;
    REAL *w;
    if (iter == 1) {
      w = wb;
      SUF(kdivcopy)(n, w, v, beta);
    } else {
      w = wa;
      if (iter >= 3) SUF(kscal)(n, -eps_rot, w);
      SUF(kaxpy)(n, -delta, wb, w);
      SUF(kaxpy)(n, (REAL)1 / beta, v, w);
    }
    SUF(kcopy)(n, r1, r2);
    SUF(kcopy)(n, r2, y);
    if (!MisI) SUF(diagmul)(n, v, Mdiag, r2, ldiv);
    oldbeta = beta;
    beta = SUF(kdot)(n, r2, v);
    if (beta < 0) { st->error = 4; rc = 4; goto done; }
    beta = SQRT(beta);
    ANorm2 = ANorm2 + alpha * alpha + oldbeta * oldbeta + beta * beta;
    REAL gbar = sn * deltabar - cs * alpha;
    eps_rot = sn * beta;
    deltabar = -cs * beta;
    REAL root = SQRT(gbar * gbar + deltabar * deltabar);
    ArNorm = phibar * root;
    if (history) PUSH(Aresiduals, st->nAres, ArNorm);
    REAL gamma = SQRT(gbar * gbar + beta * beta);
    gamma = gamma > epsM ? gamma : epsM;
    SUF(kdiv)(n, w, gamma);
    if (linesearch) {                                             /* minres.jl:336-373 */
      REAL cg_ = cs * gbar;
      if (iter > 1) {
        zeta_km1 = zeta_k;
        zeta_k = -cg_ * (rNorm * rNorm);
        beta_w = (zeta_km1 != 0) ? zeta_k / zeta_km1 : zeta_k;
        delta_w = zeta_k + beta_w * beta_w * delta_w;
      }
      if (cg_ >= 0) {
        st->solved = 1; st->npcCount = 1;
        if (iter == 1) SUF(kcopy)(n, x, b);
        else if (delta_w < 0) st->npcCount = 2;
        st->niter = iter; st->inconsistent = 0;
        set_status(st, "nonpositive curvature");
        st->indefinite = 1;
        goto done;
      }
    }
    cs = gbar / gamma;
    sn = beta / gamma;
    REAL phi = cs * phibar;
    phibar = sn * phibar;
    if (linesearch) {
      SUF(kscal)(n, sn * sn, npc_dir);
      SUF(kaxpy)(n, -phibar * cs / beta, v, npc_dir);
    }
    SUF(kaxpy)(n, phi, w, x);
    xENorm2 = xENorm2 + phi * phi;
    if (iter >= 2) { REAL *tmp = wa; wa = wb; wb = tmp; }
    err_vec[iter % window] = phi;
    if (iter >= window) err_lbnd = SUF(err_norm)(window, err_vec);
    gmax = gmax > gamma ? gmax : gamma;
    gmin = gmin < gamma ? gmin : gamma;
    REAL zeta = rhs1 / gamma;
    rhs1 = rhs2 - delta * zeta;
    rhs2 = -eps_rot * zeta;
    ANorm = SQRT(ANorm2);
    xNorm = SUF(knorm)(n, x);
    rNorm = phibar;
    REAL test1 = rNorm / (ANorm * xNorm);
    REAL test2 = root / ANorm;
    if (history) PUSH(residuals, st->nres, rNorm);
    Acond = gmax / gmin;
    if (history) PUSH(Aconds, nAc, Acond);
    if (iter == 1 && beta / beta1 <= 10 * epsM) {                 /* minres.jl:425-435 */
      st->niter = 1; st->solved = 1; st->inconsistent = 1;
      set_status(st, "x is a minimum least-squares solution");
      if (warm_start) SUF(kaxpy)(n, 1, x0, x);
      goto done;
    }
    ill_cond_mach = ((REAL)1 + (REAL)1 / Acond <= (REAL)1);
    solved_mach = ((REAL)1 + test2 <= (REAL)1);
    zero_resid_mach = ((REAL)1 + test1 <= (REAL)1);
    int resid_decrease_mach = (rNorm + (REAL)1 <= (REAL)1);
    tired = iter >= itmax;
    ill_cond_lim = ((REAL)1 / Acond <= ctol);
    solved_lim = (test2 <= eps_);
    zero_resid_lim = MisI && (test1 <= EPS);
    int resid_decrease_lim = (rNorm <= eps_);
    if (iter >= window) fwd_err = err_lbnd <= etol * SQRT(xENorm2);
    zero_resid = zero_resid_mach || zero_resid_lim;
    int resid_decrease = resid_decrease_mach || resid_decrease_lim;
    ill_cond = ill_cond_mach || ill_cond_lim;
    solved = solved_mach || solved_lim || zero_resid || fwd_err || resid_decrease;
  }
  if (tired) set_status(st, "maximum number of iterations exceeded");           /* minres.jl:465-472 */
  if (ill_cond_mach) set_status(st, "condition number seems too large for this machine");
  if (ill_cond_lim) set_status(st, "condition number exceeds tolerance");
  if (solved) set_status(st, "found approximate minimum least-squares solution");
  if (zero_resid) set_status(st, "found approximate zero-residual solution");
  if (fwd_err) set_status(st, "truncated forward error small enough");
  if (warm_start) SUF(kaxpy)(n, 1, x0, x);
  st->niter = iter; st->solved = solved; st->inconsistent = !zero_resid;
done:
  if (npc_dir && npc_dir_out) SUF(kcopy)(n, npc_dir_out, npc_dir);
  free(r1); free(r2); free(w1); free(w2); free(y); free(vbuf); free(npc_dir); free(err_vec);
  return rc;
}

/* y = A x, exported for bit-exact SpMV parity tests. */
void SUF(oracle_spmv)(int n, const int *rowptr, const int *colind, const REAL *val, const REAL *x, REAL *y) {
  SUF(csr) A = {n, rowptr, colind, val};
  SUF(spmv)(&A, x, y);
}
REAL SUF(oracle_dot)(int n, const REAL *x, const REAL *y) { return SUF(kdot)(n, x, y); }

#undef PUSH
