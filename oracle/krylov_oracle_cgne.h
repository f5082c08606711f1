/*
 * krylov_oracle_cgne.h -- TEST INFRASTRUCTURE ONLY (same status as krylov_oracle_impl.h, which must be included first).
 * Restatement of cgne! (src/cgne.jl:134-252) and crmr! (src/crmr.jl:132-244), CG and CR on A A^T y = b with
 * x = A^T y: the least-norm solution of A x = b on an m x n CSR matrix.  Written from the algorithm on the BLAS-1
 * wrappers of krylov_oracle_impl.h, instantiated by krylov_oracle.c and loaded by oracle/cgne_oracle.py.  A^T is
 * passed as its own CSR (n rows, ascending row indices of A in each row).  N (m entries, on the residual space) is a
 * diagonal or NULL; lambda >= 0 regularizes through the m-vector s.
 * Parity pinning: tests/test_oracle_cgne_crmr.py (the reference's assertions of test/test_cgne.jl and
 * test/test_crmr.jl) and tests/golden/oracle_cgne_crmr.json (frozen histories).
 */
#define PUSH(arr, cnt, v) do { if ((arr) && (cnt) < o->hist_cap) (arr)[(cnt)] = (v); (cnt)++; } while (0)

/* cgne! (src/cgne.jl:134-252).  res: ||b||, then sqrt(<r, z>) after every iteration. */
static int SUF(cgne)(int variant, const SUF(problem) *P, const oracle_options *o, SUF(outputs) *out, oracle_stats *st) {
  const int m = P->m, n = P->n;
  const REAL *b = P->b, *Ndiag = P->N;
  REAL *x = out->x, *res = out->residuals;
  SUF(csr) A = {m, P->rowptr, P->colind, P->val}, At = {n, P->trowptr, P->tcolind, P->tval};
  const double start = oracle_now();
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  const int history = o->history, ldiv = o->ldiv, NisI = Ndiag == NULL;
  const REAL lambda = (REAL)o->lambda;
  const REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol);
  int itmax = o->itmax > 0 ? o->itmax : m + n;
  size_t nbm = sizeof(REAL) * (size_t)(m > 0 ? m : 1), nbn = sizeof(REAL) * (size_t)(n > 0 ? n : 1);
  REAL *r = malloc(nbm), *q = malloc(nbm), *s = malloc(nbm), *zb = NisI ? NULL : malloc(nbm);
  REAL *p = malloc(nbn), *Atz = malloc(nbn);
  REAL *z = NisI ? r : zb;

  SUF(kfill)(n, x, 0);
  SUF(kcopy)(m, r, b);                                          /* r ← b */
  if (!NisI) SUF(diagmul)(m, z, Ndiag, r, ldiv);
  REAL rNorm = SUF(knorm)(m, r);
  if (history) PUSH(res, st->nres, rNorm);
  if (rNorm == 0) {
    st->niter = 0; st->solved = 1; st->inconsistent = 0;
    set_status(st, "x is a zero-residual solution");
    goto done;
  }
  if (lambda > 0) SUF(kcopy)(m, s, r);                          /* s ← r */
  SUF(spmv)(&At, z, p);
  REAL pNorm = SUF(knorm)(n, p);                                /* ‖p‖ detects an inconsistent system */
  REAL gamma = SUF(kdot)(m, r, z);
  int iter = 0;
  const REAL eps_c = atol + rtol * rNorm, eps_i = atol + rtol * pNorm;
  int solved = rNorm <= eps_c, inconsistent = (rNorm > 100 * eps_c) && (pNorm <= eps_i), tired = iter >= itmax;
  int user_exit = 0, overtimed = 0;
  while (!(solved || inconsistent || tired || user_exit || overtimed)) {
    SUF(spmv)(&A, p, q);
    if (lambda > 0) SUF(kaxpy)(m, lambda, s, q);
    REAL delta = SUF(kdot)(n, p, p);
    if (lambda > 0) delta += lambda * SUF(kdot)(m, s, s);
    const REAL alpha = gamma / delta;
    SUF(kaxpy)(n, alpha, p, x);
    SUF(kaxpy)(m, -alpha, q, r);
    if (!NisI) SUF(diagmul)(m, z, Ndiag, r, ldiv);
    const REAL gamma_next = SUF(kdot)(m, r, z);
    const REAL beta = gamma_next / gamma;
    SUF(spmv)(&At, z, Atz);
    SUF(kaxpby)(n, 1, Atz, beta, p);                            /* p = Aᵀz + β p */
    pNorm = SUF(knorm)(n, p);
    if (lambda > 0) SUF(kaxpby)(m, 1, r, beta, s);              /* s = r + β s */
    gamma = gamma_next;
    rNorm = SQRT(gamma_next);
    if (history) PUSH(res, st->nres, rNorm);
    iter = iter + 1;
    const int resid_decrease_mach = rNorm + (REAL)1 <= (REAL)1;
    user_exit = o->callback ? o->callback(iter, o->cb_user) != 0 : 0;
    const int resid_decrease_lim = rNorm <= eps_c;
    solved = resid_decrease_lim || resid_decrease_mach;
    inconsistent = (rNorm > 100 * eps_c) && (pNorm <= eps_i);
    tired = iter >= itmax;
    overtimed = o->timemax >= 0 && oracle_now() - start > o->timemax;
  }
  {
    const char *sx = "unknown";
    if (tired) sx = "maximum number of iterations exceeded";
    if (inconsistent) sx = "system probably inconsistent";
    if (solved) sx = "solution good enough given atol and rtol";
    if (user_exit) sx = "user-requested exit";
    if (overtimed) sx = "time limit exceeded";
    set_status(st, sx);
  }
  st->niter = iter; st->solved = solved; st->inconsistent = inconsistent;
done:
  free(r); free(q); free(s); free(zb); free(p); free(Atz);
  return 0;
}

/* crmr! (src/crmr.jl:132-244).  res: ||r|| (r = N (b - A x)); ares: ||A^T r|| (+ λ ||r||² under the root). */
static int SUF(crmr)(int variant, const SUF(problem) *P, const oracle_options *o, SUF(outputs) *out, oracle_stats *st) {
  const int m = P->m, n = P->n;
  const REAL *b = P->b, *Ndiag = P->N;
  REAL *x = out->x, *res = out->residuals, *ares = out->Aresiduals;
  SUF(csr) A = {m, P->rowptr, P->colind, P->val}, At = {n, P->trowptr, P->tcolind, P->tval};
  const double start = oracle_now();
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  const int history = o->history, ldiv = o->ldiv, NisI = Ndiag == NULL;
  const REAL lambda = (REAL)o->lambda;
  const REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol);
  int itmax = o->itmax > 0 ? o->itmax : m + n;
  size_t nbm = sizeof(REAL) * (size_t)(m > 0 ? m : 1), nbn = sizeof(REAL) * (size_t)(n > 0 ? n : 1);
  REAL *r = malloc(nbm), *q = malloc(nbm), *s = malloc(nbm), *Nqb = NisI ? NULL : malloc(nbm);
  REAL *p = malloc(nbn), *Atr = malloc(nbn);
  REAL *Nq = NisI ? q : Nqb;

  SUF(kfill)(n, x, 0);
  if (NisI) SUF(kcopy)(m, r, b);                                /* r = N b */
  else SUF(diagmul)(m, r, Ndiag, b, ldiv);
  const REAL bNorm = SUF(knorm)(m, r);
  REAL rNorm = bNorm;
  if (history) PUSH(res, st->nres, rNorm);
  if (bNorm == 0) {
    st->niter = 0; st->solved = 1; st->inconsistent = 0;
    set_status(st, "x is a zero-residual solution");
    if (history) PUSH(ares, st->nAres, (REAL)0);
    goto done;
  }
  if (lambda > 0) SUF(kcopy)(m, s, r);                          /* s ← r */
  SUF(spmv)(&At, r, Atr);
  SUF(kcopy)(n, p, Atr);                                        /* p ← Aᵀr */
  REAL gamma = SUF(kdot)(n, Atr, Atr);
  if (lambda > 0) gamma += lambda * rNorm * rNorm;
  int iter = 0;
  REAL ArNorm = SQRT(gamma);
  if (history) PUSH(ares, st->nAres, ArNorm);
  const REAL eps_c = atol + rtol * rNorm, eps_i = atol + rtol * ArNorm;
  int solved = rNorm <= eps_c, inconsistent = (rNorm > 100 * eps_c) && (ArNorm <= eps_i), tired = iter >= itmax;
  int user_exit = 0, overtimed = 0;
  while (!(solved || inconsistent || tired || user_exit || overtimed)) {
    SUF(spmv)(&A, p, q);
    if (lambda > 0) SUF(kaxpy)(m, lambda, s, q);                /* q = q + λ s */
    if (!NisI) SUF(diagmul)(m, Nq, Ndiag, q, ldiv);
    const REAL alpha = gamma / SUF(kdot)(m, q, Nq);             /* qᵀ N q */
    SUF(kaxpy)(n, alpha, p, x);
    SUF(kaxpy)(m, -alpha, Nq, r);
    rNorm = SUF(knorm)(m, r);
    SUF(spmv)(&At, r, Atr);
    REAL gamma_next = SUF(kdot)(n, Atr, Atr);
    if (lambda > 0) gamma_next += lambda * rNorm * rNorm;
    const REAL beta = gamma_next / gamma;
    SUF(kaxpby)(n, 1, Atr, beta, p);                            /* p = Aᵀr + β p */
    if (lambda > 0) SUF(kaxpby)(m, 1, r, beta, s);              /* s = r + β s */
    gamma = gamma_next;
    ArNorm = SQRT(gamma);
    if (history) { PUSH(res, st->nres, rNorm); PUSH(ares, st->nAres, ArNorm); }
    iter = iter + 1;
    user_exit = o->callback ? o->callback(iter, o->cb_user) != 0 : 0;
    solved = rNorm <= eps_c;
    inconsistent = (rNorm > 100 * eps_c) && (ArNorm <= eps_i);
    tired = iter >= itmax;
    overtimed = o->timemax >= 0 && oracle_now() - start > o->timemax;
  }
  {
    const char *sx = "unknown";
    if (tired) sx = "maximum number of iterations exceeded";
    if (solved) sx = "solution good enough given atol and rtol";
    if (inconsistent) sx = "system probably inconsistent but least squares/norm solution found";
    if (user_exit) sx = "user-requested exit";
    if (overtimed) sx = "time limit exceeded";
    set_status(st, sx);
  }
  st->niter = iter; st->solved = solved; st->inconsistent = inconsistent;
done:
  free(r); free(q); free(s); free(Nqb); free(p); free(Atr);
  return 0;
}
