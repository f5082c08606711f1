/*
 * krylov_oracle_cgls.h -- TEST INFRASTRUCTURE ONLY (same status as krylov_oracle_impl.h; include it and
 * krylov_oracle_lsq.h first, instantiated by krylov_oracle.c).  Literal restatements of the least-squares solvers
 * on the normal equations, on an m x n CSR matrix:
 *   cgls!  src/cgls.jl:129-243
 *   crls!  src/crls.jl:120-268
 * A v sums each row in ascending column order; A^T u sums each column in ascending row order of A (spmv_t of
 * krylov_oracle_lsq.h).  M (m entries, acting on the residual space) is a diagonal or NULL.
 * Parity pinning: the reference's own assertions of test/test_cgls.jl and test/test_crls.jl (tests/test_oracle_cgls.py).
 */
#define PUSH(arr, cnt, v) do { if ((arr) && (cnt) < o->hist_cap) (arr)[(cnt)] = (v); (cnt)++; } while (0)

/* variant 0: cgls!, 1: crls!.  Returns 0, or where the reference raises: 10 + to_boundary's error code. */
static int SUF(cgls)(int variant, const SUF(problem) *P, const oracle_options *o, SUF(outputs) *out, oracle_stats *st) {
  const int crls = variant, m = P->m, n = P->n;
  const int *rowptr = P->rowptr, *colind = P->colind;
  const REAL *val = P->val, *b = P->b, *Mdiag = P->M;
  REAL *x = out->x, *residuals = out->residuals, *Aresiduals = out->Aresiduals;
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  int history = o->history, ldiv = o->ldiv, rc = 0;
  int MisI = (Mdiag == NULL);
  REAL lambda = (REAL)o->lambda, radius = (REAL)o->radius;
  REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol);
  size_t mb = sizeof(REAL) * (size_t)(m > 0 ? m : 1), nb = sizeof(REAL) * (size_t)(n > 0 ? n : 1);
  REAL *r = malloc(mb), *qm = malloc(mb), *Ap = malloc(mb), *s_m = malloc(mb), *Mbuf = MisI ? NULL : malloc(mb);
  REAL *p = malloc(nb), *s_n = malloc(nb), *Ar = malloc(nb), *q_n = malloc(nb), *z = malloc(nb);
  int iter = 0, itmax = o->itmax != 0 ? o->itmax : m + n;
  int solved = 0, tired = 0, on_boundary = 0, psd = 0;

  SUF(kfill)(n, x, 0);
  SUF(kcopy)(m, r, b);
  REAL bNorm = SUF(knorm)(m, r);
  if (!crls) {
    /* ---------------------------- cgls.jl:155-226 ---------------------------- */
    REAL *s = s_n, *q = qm;
    REAL *Mr = MisI ? r : Mbuf, *Mq = MisI ? q : Mbuf;
    if (bNorm == 0) {
      st->niter = 0; st->solved = 1; st->inconsistent = 0;
      set_status(st, "x is a zero-residual solution");
      if (history) { PUSH(residuals, st->nres, 0); PUSH(Aresiduals, st->nAres, 0); }
      goto done;
    }
    if (!MisI) SUF(diagmul)(m, Mr, Mdiag, r, ldiv);
    SUF(spmv_t)(m, n, rowptr, colind, val, Mr, s);
    SUF(kcopy)(n, p, s);
    REAL gamma = SUF(kdot)(n, s, s);
    REAL rNorm = bNorm, ArNorm = SQRT(gamma);
    if (history) { PUSH(residuals, st->nres, rNorm); PUSH(Aresiduals, st->nAres, ArNorm); }
    REAL eps = atol + rtol * ArNorm;
    solved = ArNorm <= eps;
    tired = iter >= itmax;
    while (!(solved || tired)) {
      SUF(spmv_rect)(m, rowptr, colind, val, p, q);
      if (!MisI) SUF(diagmul)(m, Mq, Mdiag, q, ldiv);
      REAL delta = SUF(kdot)(m, q, Mq);
      if (lambda > 0) delta += lambda * SUF(kdot)(n, p, p);
      REAL alpha = gamma / delta;
      if (radius > 0) {
        REAL t1, t2;
        int e = SUF(oracle_to_boundary)(n, x, p, z, radius, 0, 0, 0, NULL, 0, &t1, &t2);
        if (e) { rc = 10 + e; goto done; }
        REAL sigma = t1 > t2 ? t1 : t2;
        if (alpha > sigma) { alpha = sigma; on_boundary = 1; }
      }
      SUF(kaxpy)(n, alpha, p, x);
      SUF(kaxpy)(m, -alpha, q, r);
      if (!MisI) SUF(diagmul)(m, Mr, Mdiag, r, ldiv);
      SUF(spmv_t)(m, n, rowptr, colind, val, Mr, s);
      if (lambda > 0) SUF(kaxpy)(n, -lambda, x, s);
      REAL gamma_next = SUF(kdot)(n, s, s);
      REAL beta = gamma_next / gamma;
      SUF(kaxpby)(n, 1, s, beta, p);
      gamma = gamma_next;
      rNorm = SUF(knorm)(m, r);
      ArNorm = SQRT(gamma);
      if (history) { PUSH(residuals, st->nres, rNorm); PUSH(Aresiduals, st->nAres, ArNorm); }
      iter = iter + 1;
      solved = (ArNorm <= eps) || on_boundary;
      tired = iter >= itmax;
    }
  } else {
    /* ---------------------------- crls.jl:151-250 ---------------------------- */
    REAL *s = s_m, *q = q_n, *pp = p;
    REAL *Ms = MisI ? s : Mbuf, *Mr = MisI ? r : Mbuf, *MAp = MisI ? Ap : Mbuf;
    REAL rNorm = bNorm;
    if (history) PUSH(residuals, st->nres, rNorm);
    if (bNorm == 0) {
      st->niter = 0; st->solved = 1; st->inconsistent = 0;
      set_status(st, "x is a zero-residual solution");
      if (history) PUSH(Aresiduals, st->nAres, 0);
      goto done;
    }
    if (!MisI) SUF(diagmul)(m, Mr, Mdiag, r, ldiv);
    SUF(spmv_t)(m, n, rowptr, colind, val, Mr, Ar);
    SUF(spmv_rect)(m, rowptr, colind, val, Ar, s);
    if (!MisI) SUF(diagmul)(m, Ms, Mdiag, s, ldiv);
    SUF(kcopy)(n, pp, Ar);
    SUF(kcopy)(m, Ap, s);
    SUF(spmv_t)(m, n, rowptr, colind, val, Ms, q);
    if (lambda > 0) SUF(kaxpy)(n, lambda, pp, q);
    REAL gamma = SUF(kdot)(m, s, Ms);
    REAL ArNorm = SUF(knorm)(n, Ar);
    if (lambda > 0) gamma += lambda * ArNorm * ArNorm;
    if (history) PUSH(Aresiduals, st->nAres, ArNorm);
    REAL eps = atol + rtol * ArNorm;
    solved = ArNorm <= eps;
    tired = iter >= itmax;
    while (!(solved || tired)) {
      REAL qNorm2 = SUF(kdot)(n, q, q);
      REAL alpha = gamma / qNorm2;
      if (radius > 0) {
        REAL pNorm = SUF(knorm)(n, pp), t1, t2;
        int e;
        if (SUF(kdot)(m, Ap, Ap) <= eps * SQRT(qNorm2) * pNorm) {
          psd = 1;
          pp = Ar;
          REAL pNorm2 = ArNorm * ArNorm;
          SUF(spmv_t)(m, n, rowptr, colind, val, s, q);
          e = SUF(oracle_to_boundary)(n, x, pp, z, radius, 0, 0, pNorm2, NULL, 0, &t1, &t2);
          if (e) { rc = 10 + e; goto done; }
          REAL tmax = t1 > t2 ? t1 : t2, a1 = ArNorm * ArNorm / gamma;
          alpha = a1 < tmax ? a1 : tmax;
        } else {
          REAL pNorm2 = pNorm * pNorm;
          e = SUF(oracle_to_boundary)(n, x, pp, z, radius, 0, 0, pNorm2, NULL, 0, &t1, &t2);
          if (e) { rc = 10 + e; goto done; }
          REAL sigma = t1 > t2 ? t1 : t2;
          if (alpha >= sigma) { alpha = sigma; on_boundary = 1; }
        }
      }
      SUF(kaxpy)(n, alpha, pp, x);
      SUF(kaxpy)(n, -alpha, q, Ar);
      ArNorm = SUF(knorm)(n, Ar);
      solved = psd || on_boundary;
      if (solved) continue;
      SUF(kaxpy)(m, -alpha, Ap, r);
      SUF(spmv_rect)(m, rowptr, colind, val, Ar, s);
      if (!MisI) SUF(diagmul)(m, Ms, Mdiag, s, ldiv);
      REAL gamma_next = SUF(kdot)(m, s, Ms);
      if (lambda > 0) gamma_next += lambda * ArNorm * ArNorm;
      REAL beta = gamma_next / gamma;
      SUF(kaxpby)(n, 1, Ar, beta, pp);
      SUF(kaxpby)(m, 1, s, beta, Ap);
      if (!MisI) SUF(diagmul)(m, MAp, Mdiag, Ap, ldiv);
      SUF(spmv_t)(m, n, rowptr, colind, val, MAp, q);
      if (lambda > 0) SUF(kaxpy)(n, lambda, pp, q);
      gamma = gamma_next;
      if (lambda > 0) rNorm = SQRT(SUF(kdot)(m, r, r) + lambda * SUF(kdot)(n, x, x));
      else rNorm = SUF(knorm)(m, r);
      if (history) { PUSH(residuals, st->nres, rNorm); PUSH(Aresiduals, st->nAres, ArNorm); }
      iter = iter + 1;
      solved = (ArNorm <= eps) || on_boundary;
      tired = iter >= itmax;
    }
  }
  if (tired) set_status(st, "maximum number of iterations exceeded");
  if (solved) set_status(st, "solution good enough given atol and rtol");
  if (psd) set_status(st, "zero-curvature encountered");
  if (on_boundary) set_status(st, "on trust-region boundary");
  st->niter = iter; st->solved = solved; st->inconsistent = 0;
done:
  free(r); free(qm); free(Ap); free(s_m); free(Mbuf); free(p); free(s_n); free(Ar); free(q_n); free(z);
  return rc;
}

#undef PUSH
