/*
 * krylov_oracle_leastnorm.h -- TEST INFRASTRUCTURE ONLY (same status as krylov_oracle_impl.h, which must be included
 * first).  Restatement of the least-norm solvers, min ||x|| subject to A x = b with x = A^T y, on an m x n CSR matrix:
 *   craig!    src/craig.jl:174-405   (CG on A A^T y = b)
 *   craigmr!  src/craigmr.jl:161-396 (MINRES on A A^T y = b)
 * written from the algorithm on the BLAS-1 wrappers of krylov_oracle_impl.h, instantiated by krylov_oracle.c
 * and loaded by oracle/leastnorm_oracle.py.  A^T is passed as its own CSR (n rows, ascending row indices of A in each
 * row).  M (m entries) and N (n entries) are diagonals or NULL.
 * Parity pinning: tests/test_oracle_leastnorm.py (the reference's assertions of test/test_craig.jl and
 * test/test_craigmr.jl) and tests/golden/oracle_leastnorm.json (frozen histories).
 */
#define PUSH(arr, cnt, v) do { if ((arr) && (cnt) < o->hist_cap) (arr)[(cnt)] = (v); (cnt)++; } while (0)

static REAL SUF(ln_knorm_ell)(int n, const REAL *x, const REAL *y) {   /* knorm_elliptic (krylov_utils.jl:319) */
  return x == y ? SUF(knorm)(n, x) : SQRT(SUF(kdot)(n, x, y));
}

/* variant 0: craig!, 1: craigmr!.  The callback (NULL: none) returns nonzero to stop; timemax < 0 means no limit. */
static int SUF(leastnorm)(int variant, const SUF(problem) *P, const oracle_options *o, SUF(outputs) *out, oracle_stats *st) {
  const int mr = variant, m = P->m, n = P->n;
  const REAL *b = P->b, *Mdiag = P->M, *Ndiag = P->N;
  REAL *x = out->x, *y = out->y, *res = out->residuals, *ares = out->Aresiduals;
  SUF(csr) A = {m, P->rowptr, P->colind, P->val}, At = {n, P->trowptr, P->tcolind, P->tval};
  const double start = oracle_now();
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  const int history = o->history, ldiv = o->ldiv, MisI = Mdiag == NULL, NisI = Ndiag == NULL;
  const REAL lambda = (REAL)o->lambda;
  const REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol);
  int itmax = o->itmax > 0 ? o->itmax : m + n;
  size_t nbm = sizeof(REAL) * (size_t)(m > 0 ? m : 1), nbn = sizeof(REAL) * (size_t)(n > 0 ? n : 1);
  REAL *Mu = malloc(nbm), *Av = malloc(nbm), *w = malloc(nbm), *ub = MisI ? NULL : malloc(nbm), *wbar = malloc(nbm);
  REAL *Nv = malloc(nbn), *Atu = malloc(nbn), *vb = NisI ? NULL : malloc(nbn), *aux = malloc(nbn), *d = malloc(nbn);
  REAL *u = MisI ? Mu : ub, *v = NisI ? Nv : vb;
  int iter = 0, solved = 0, inconsistent = 0, tired = 0, user_exit = 0, overtimed = 0;

  SUF(kfill)(n, x, 0);
  SUF(kfill)(m, y, 0);
  SUF(kcopy)(m, Mu, b);
  if (!MisI) SUF(diagmul)(m, u, Mdiag, Mu, ldiv);
  REAL beta = SUF(ln_knorm_ell)(m, u, Mu);

  if (!mr) {
    /* ---------------- craig! ---------------- */
    const REAL conlim = isnan(o->conlim) ? (REAL)1 / SQRT(EPS) : (REAL)o->conlim;
    const REAL btol = SUF(tol)(o->btol);
    REAL *w2 = aux;
    const REAL beta1 = beta;
    REAL rNorm = beta1;
    if (history) PUSH(res, st->nres, rNorm);
    if (beta1 == 0) {
      st->niter = 0; st->solved = 1; st->inconsistent = 0;
      set_status(st, "x is a zero-residual solution");
      goto done;
    }
    const REAL beta1_2 = beta1 * beta1;
    REAL theta = beta1, xi = -1, delta = lambda, rho_prev = 1;
    SUF(kdiv)(m, u, beta1);
    if (!MisI) SUF(kdiv)(m, Mu, beta1);
    SUF(kfill)(n, Nv, 0);
    SUF(kfill)(m, w, 0);
    if (lambda > 0) SUF(kfill)(n, w2, 0);
    REAL Anorm2 = 0, Anorm = 0, Dnorm2 = 0, Acond = 0, xNorm2 = 0, xNorm = 0;
    const REAL eps_c = atol + rtol * rNorm;
    const REAL ctol = conlim > 0 ? (REAL)1 / conlim : (REAL)0;
    REAL bkwerr = 1;
    int solved_lim = bkwerr <= btol, solved_mach = (REAL)1 + bkwerr <= (REAL)1, solved_resid_tol = rNorm <= eps_c;
    int solved_resid_lim = rNorm <= btol + atol * Anorm * xNorm / beta1;
    int ill_cond = 0, ill_cond_mach = 0, ill_cond_lim = 0;
    solved = solved_mach || solved_lim || solved_resid_tol || solved_resid_lim;
    tired = iter >= itmax;
    while (!(solved || inconsistent || ill_cond || tired || user_exit || overtimed)) {
      SUF(spmv)(&At, u, Atu);                                   /* αNv = Aᵀu - βNv */
      SUF(kaxpby)(n, 1, Atu, -beta, Nv);
      if (!NisI) SUF(diagmul)(n, v, Ndiag, Nv, ldiv);
      REAL alpha = SUF(ln_knorm_ell)(n, v, Nv);
      if (alpha == 0) { inconsistent = 1; continue; }
      SUF(kdiv)(n, v, alpha);
      if (!NisI) SUF(kdiv)(n, Nv, alpha);
      Anorm2 += alpha * alpha + lambda * lambda;
      REAL c1 = 1, s1 = 0, rho;
      if (lambda > 0) SUF(oracle_sym_givens)(alpha, delta, &c1, &s1, &rho);
      else rho = alpha;
      xi = -theta / rho * xi;
      if (lambda > 0) {
        SUF(kaxpy)(n, xi * c1, v, x);
        SUF(kaxpy)(n, xi * s1, w2, x);
        SUF(kaxpby)(n, s1, v, -c1, w2);
      } else {
        SUF(kaxpy)(n, xi, v, x);
      }
      SUF(kaxpby)(m, 1, u, -theta / rho_prev, w);              /* recur y */
      SUF(kaxpy)(m, xi / rho, w, y);
      Dnorm2 += SUF(knorm)(m, w);                               /* a norm, not its square: as the reference has it */
      SUF(spmv)(&A, v, Av);                                     /* βMu = A v - αMu */
      SUF(kaxpby)(m, 1, Av, -alpha, Mu);
      if (!MisI) SUF(diagmul)(m, u, Mdiag, Mu, ldiv);
      beta = SUF(ln_knorm_ell)(m, u, Mu);
      if (beta != 0) {
        SUF(kdiv)(m, u, beta);
        if (!MisI) SUF(kdiv)(m, Mu, beta);
      }
      if (lambda > 0) {
        theta = beta * c1;
        REAL gamma = beta * s1, c2, s2;
        SUF(oracle_sym_givens)(lambda, gamma, &c2, &s2, &delta);
        SUF(kscal)(n, s2, w2);
      } else {
        theta = beta;
      }
      Anorm2 += beta * beta;
      Anorm = SQRT(Anorm2);
      Acond = Anorm * SQRT(Dnorm2);
      xNorm2 += xi * xi;
      xNorm = SQRT(xNorm2);
      rNorm = beta * FABS(xi);
      if (lambda > 0) rNorm *= FABS(c1);
      if (history) PUSH(res, st->nres, rNorm);
      iter = iter + 1;
      bkwerr = rNorm / SQRT(beta1_2 + Anorm2 * xNorm2);
      rho_prev = rho;
      solved_lim = bkwerr <= btol;
      solved_mach = (REAL)1 + bkwerr <= (REAL)1;
      solved_resid_tol = rNorm <= eps_c;
      solved_resid_lim = rNorm <= btol + atol * Anorm * xNorm / beta1;
      solved = solved_mach || solved_lim || solved_resid_tol || solved_resid_lim;
      ill_cond_mach = (REAL)1 + (REAL)1 / Acond <= (REAL)1;
      ill_cond_lim = (REAL)1 / Acond <= ctol;
      ill_cond = ill_cond_mach || ill_cond_lim;
      user_exit = o->callback ? o->callback(iter, o->cb_user) != 0 : 0;
      inconsistent = 0;
      tired = iter >= itmax;
      overtimed = o->timemax >= 0 && oracle_now() - start > o->timemax;
    }
    if (lambda > 0 && o->transfer_to_lsqr) {
      xi *= -theta / delta;
      SUF(kaxpy)(n, xi, w2, x);
    }
    const char *s = "unknown";
    if (tired) s = "maximum number of iterations exceeded";
    if (solved) s = "solution good enough for the tolerances given";
    if (ill_cond_mach) s = "condition number seems too large for this machine";
    if (ill_cond_lim) s = "condition number exceeds tolerance";
    if (inconsistent) s = "system may be inconsistent";
    if (user_exit) s = "user-requested exit";
    if (overtimed) s = "time limit exceeded";
    set_status(st, s);
  } else {
    /* ---------------- craigmr! ---------------- */
    REAL *q = aux;
    if (beta == 0) {
      st->niter = 0; st->solved = 1; st->inconsistent = 0;
      if (history) { PUSH(res, st->nres, beta); PUSH(ares, st->nAres, 0); }
      set_status(st, "x is a zero-residual solution");
      goto done;
    }
    SUF(kdiv)(m, u, beta);
    if (!MisI) SUF(kdiv)(m, Mu, beta);
    SUF(spmv)(&At, u, Atu);
    SUF(kcopy)(n, Nv, Atu);
    if (!NisI) SUF(diagmul)(n, v, Ndiag, Nv, ldiv);
    REAL alpha = SUF(ln_knorm_ell)(n, v, Nv);
    REAL Anorm2 = alpha * alpha;
    if (alpha == 0) {
      st->niter = 0; st->solved = 1; st->inconsistent = 0;
      if (history) { PUSH(res, st->nres, beta); PUSH(ares, st->nAres, 0); }
      set_status(st, "x is a minimum least-squares solution");
      goto done;
    }
    SUF(kdiv)(n, v, alpha);
    if (!NisI) SUF(kdiv)(n, Nv, alpha);
    const REAL lambdak = lambda;
    REAL cpk = 1, spk = 1, cdk = 1, sdk = 1, alphahat;
    if (lambda > 0) SUF(kcopy)(n, q, v);
    if (lambda > 0) {
      SUF(oracle_sym_givens)(alpha, lambdak, &cpk, &spk, &alphahat);
      SUF(kscal)(n, spk, q);
    } else {
      alphahat = alpha;
    }
    REAL zetabar = beta, rhobar = alphahat, theta = 0;
    REAL rNorm = zetabar, ArNorm = alpha;
    if (history) { PUSH(res, st->nres, rNorm); PUSH(ares, st->nAres, ArNorm); }
    const REAL eps_c = atol + rtol * rNorm, eps_i = atol + rtol * ArNorm;
    SUF(kdivcopy)(m, wbar, u, alphahat);
    SUF(kfill)(m, w, 0);
    SUF(kfill)(n, d, 0);
    solved = rNorm <= eps_c;
    inconsistent = (rNorm > 100 * eps_c) && (ArNorm <= eps_i);
    tired = iter >= itmax;
    while (!(solved || inconsistent || tired || user_exit || overtimed)) {
      iter = iter + 1;
      SUF(spmv)(&A, v, Av);                                     /* βMu = A v - αMu */
      SUF(kaxpby)(m, 1, Av, -alpha, Mu);
      if (!MisI) SUF(diagmul)(m, u, Mdiag, Mu, ldiv);
      beta = SUF(ln_knorm_ell)(m, u, Mu);
      if (beta != 0) {
        SUF(kdiv)(m, u, beta);
        if (!MisI) SUF(kdiv)(m, Mu, beta);
      }
      Anorm2 = Anorm2 + beta * beta;
      REAL betahat, lambda_aux = 0;
      if (lambda > 0) { betahat = cpk * beta; lambda_aux = spk * beta; }
      else betahat = beta;
      REAL c, s, rho;
      SUF(oracle_sym_givens)(rhobar, betahat, &c, &s, &rho);
      const REAL zeta = c * zetabar;
      zetabar = s * zetabar;
      rNorm = FABS(zetabar);
      if (history) PUSH(res, st->nres, rNorm);
      SUF(kaxpby)(m, (REAL)1 / rho, wbar, -theta / rho, w);     /* w = (w̄ - θ w) / ρ */
      SUF(kaxpy)(m, zeta, w, y);
      if (lambda > 0) {
        if (iter == 1) {
          SUF(kaxpy)(n, cpk / rho, v, d);
        } else {
          SUF(kaxpby)(n, cpk / rho, v, -theta / rho, d);
          SUF(kaxpy)(n, spk / rho, q, d);
          SUF(kaxpby)(n, spk, v, -cpk, q);
        }
      } else {
        if (iter == 1) SUF(kdivcopy)(n, d, v, rho);
        else SUF(kaxpby)(n, (REAL)1 / rho, v, -theta / rho, d);
      }
      SUF(kaxpy)(n, zeta, d, x);
      SUF(spmv)(&At, u, Atu);                                   /* αNv = Aᵀu - βNv */
      SUF(kaxpby)(n, 1, Atu, -beta, Nv);
      if (!NisI) SUF(diagmul)(n, v, Ndiag, Nv, ldiv);
      alpha = SUF(ln_knorm_ell)(n, v, Nv);
      Anorm2 = Anorm2 + alpha * alpha;
      ArNorm = alpha * beta * FABS(zeta / rho);
      if (history) PUSH(ares, st->nAres, ArNorm);
      if (lambda > 0) {
        REAL lambdak1;
        SUF(oracle_sym_givens)(lambda, lambda_aux, &cdk, &sdk, &lambdak1);
        SUF(kscal)(n, sdk, q);
        SUF(oracle_sym_givens)(alpha, lambdak1, &cpk, &spk, &alphahat);
      } else {
        alphahat = alpha;
      }
      if (alpha != 0) {
        SUF(kdiv)(n, v, alpha);
        if (!NisI) SUF(kdiv)(n, Nv, alpha);
        SUF(kaxpby)(m, (REAL)1 / alphahat, u, -betahat / alphahat, wbar);
      }
      theta = s * alphahat;
      rhobar = -c * alphahat;
      user_exit = o->callback ? o->callback(iter, o->cb_user) != 0 : 0;
      solved = rNorm <= eps_c;
      inconsistent = (rNorm > 100 * eps_c) && (ArNorm <= eps_i);
      tired = iter >= itmax;
      overtimed = o->timemax >= 0 && oracle_now() - start > o->timemax;
    }
    const char *sts = "unknown";
    if (tired) sts = "maximum number of iterations exceeded";
    if (solved) sts = "found approximate minimum-norm solution";
    if (!tired && !solved) sts = "found approximate minimum least-squares solution";
    if (user_exit) sts = "user-requested exit";
    if (overtimed) sts = "time limit exceeded";
    set_status(st, sts);
    (void)cdk;
  }
  st->niter = iter; st->solved = solved; st->inconsistent = inconsistent;
done:
  free(Mu); free(Av); free(w); free(ub); free(wbar); free(Nv); free(Atu); free(vb); free(aux); free(d);
  return 0;
}

#undef PUSH
