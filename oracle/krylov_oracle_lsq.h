/*
 * krylov_oracle_lsq.h -- TEST INFRASTRUCTURE ONLY (same status as krylov_oracle_impl.h, which must be included
 * first; instantiated by krylov_oracle_lsq.c).  Literal restatements of the least-squares solvers on an m x n CSR matrix:
 *   lsqr!  src/lsqr.jl:174-440
 *   lsmr!  src/lsmr.jl:178-455
 * A v sums each row in ascending column order; A^T u sums each column in ascending row order of A (what a
 * sequential A' * u over the CSC storage of A does).  M (m entries) and N (n entries) are diagonals or NULL.
 * Parity pinning: the reference's own assertions of test/test_lsqr.jl and test/test_lsmr.jl (tests/test_oracle_lsq.py).
 */
#ifndef ORACLE_LSQ_OPTS_DEFINED
#define ORACLE_LSQ_OPTS_DEFINED
typedef struct {
  double atol, rtol;            /* NaN -> sqrt(eps(T)) */
  double etol, axtol, btol;     /* NaN -> sqrt(eps(T)) */
  double conlim;                /* NaN -> 1/sqrt(eps(T)) */
  double lambda, radius;
  int itmax;                    /* 0 -> m + n */
  int history;
  int window;                   /* 0 -> 5 */
  int ldiv;
  int hist_cap;
} oracle_lsq_opts;
#endif

#define PUSH(arr, cnt, v) do { if ((arr) && (cnt) < o->hist_cap) (arr)[(cnt)] = (v); (cnt)++; } while (0)

/* y = A^T x for an m x n CSR A: column sums in ascending row order */
static void SUF(spmv_t)(int m, int n, const int *rowptr, const int *colind, const REAL *val, const REAL *x, REAL *y) {
  for (int j = 0; j < n; j++) y[j] = (REAL)0;
  for (int i = 0; i < m; i++)
    for (int k = rowptr[i]; k < rowptr[i + 1]; k++) { REAL p = val[k] * x[i]; y[colind[k]] = y[colind[k]] + p; }
}
static void SUF(spmv_rect)(int m, const int *rowptr, const int *colind, const REAL *val, const REAL *x, REAL *y) {
  SUF(csr) A = {m, rowptr, colind, val};
  SUF(spmv)(&A, x, y);
}
/* knorm_elliptic(n, x, y) (krylov_utils.jl:319) */
static REAL SUF(knorm_ell)(int n, const REAL *x, const REAL *y) {
  return x == y ? SUF(knorm)(n, x) : SQRT(SUF(kdot)(n, x, y));
}
static REAL SUF(err_norm)(int w, const REAL *e) {
  REAL s = 0;
  for (int i = 0; i < w; i++) s += e[i] * e[i];
  return SQRT(s);
}

/* lsmr = 0: lsqr!, 1: lsmr!.  Returns 0, or where the reference raises: 10 + to_boundary's error code. */
int SUF(oracle_lsq)(int lsmr, int m, int n, const int *rowptr, const int *colind, const REAL *val, const REAL *b,
                    const REAL *Mdiag, const REAL *Ndiag, const oracle_lsq_opts *o, REAL *x, REAL *residuals,
                    REAL *Aresiduals, REAL *Anorm_out, oracle_stats *st) {
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  int history = o->history, ldiv = o->ldiv, rc = 0;
  int MisI = (Mdiag == NULL), NisI = (Ndiag == NULL);
  REAL lambda = (REAL)o->lambda, lambda2 = lambda * lambda, radius = (REAL)o->radius;
  REAL conlim = isnan(o->conlim) ? (REAL)1 / SQRT(EPS) : (REAL)o->conlim;
  REAL ctol = conlim > 0 ? (REAL)1 / conlim : (REAL)0;
  REAL etol = SUF(tol)(o->etol), axtol = SUF(tol)(o->axtol), btol = SUF(tol)(o->btol);
  REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol);
  int window = o->window > 0 ? o->window : 5;
  size_t mb = sizeof(REAL) * (size_t)(m > 0 ? m : 1), nb = sizeof(REAL) * (size_t)(n > 0 ? n : 1);
  REAL *Mu = malloc(mb), *Av = malloc(mb), *uu = MisI ? NULL : malloc(mb);
  REAL *Nv = malloc(nb), *Atu = malloc(nb), *vv = NisI ? NULL : malloc(nb), *w = malloc(nb), *hbar = malloc(nb), *z = malloc(nb);
  REAL *err_vec = calloc((size_t)window, sizeof(REAL));
  REAL *u = MisI ? Mu : uu, *v = NisI ? Nv : vv;
  REAL *h = w;                                          /* LSMR's h uses the storage of LSQR's w */
  *Anorm_out = (REAL)0;

  SUF(kfill)(n, x, 0);
  SUF(kcopy)(m, Mu, b);
  if (!MisI) SUF(diagmul)(m, u, Mdiag, Mu, ldiv);
  REAL beta1 = SUF(knorm_ell)(m, u, Mu);
  if (beta1 == 0) {
    st->niter = 0; st->solved = 1; st->inconsistent = 0;
    set_status(st, "x is a zero-residual solution");
    if (history) { PUSH(residuals, st->nres, 0); PUSH(Aresiduals, st->nAres, 0); }
    goto done;
  }
  REAL beta = beta1;
  SUF(kdiv)(m, u, beta1);
  if (!MisI) SUF(kdiv)(m, Mu, beta1);
  SUF(spmv_t)(m, n, rowptr, colind, val, u, Atu);
  SUF(kcopy)(n, Nv, Atu);
  if (!NisI) SUF(diagmul)(n, v, Ndiag, Nv, ldiv);
  int iter = 0;
  int itmax = o->itmax != 0 ? o->itmax : m + n;
  int solved = 0, tired = 0, ill_cond = 0, ill_cond_mach = 0, ill_cond_lim = 0, zero_resid = 0, fwd_err = 0, on_boundary = 0;
  REAL xENorm2 = 0, err_lbnd = 0;

  if (!lsmr) {
    /* ---------------------------- lsqr.jl:235-419 ---------------------------- */
    REAL Anorm2 = SUF(kdot)(n, v, Nv), Anorm = SQRT(Anorm2), alpha = Anorm;
    REAL Acond = 0, xNorm = 0, xNorm2 = 0, dNorm2 = 0, c2 = -1, s2 = 0, zz = 0;
    REAL rNorm = beta1, res2 = 0;
    if (history) PUSH(residuals, st->nres, rNorm);
    REAL ArNorm = alpha * beta, ArNorm0 = ArNorm;
    if (history) PUSH(Aresiduals, st->nAres, ArNorm);
    if (alpha == 0) {
      st->niter = 0; st->solved = 1; st->inconsistent = 0;
      set_status(st, "x is a minimum least-squares solution");
      goto done;
    }
    SUF(kdiv)(n, v, alpha);
    if (!NisI) SUF(kdiv)(n, Nv, alpha);
    SUF(kcopy)(n, w, v);
    REAL phibar = beta1, rhobar = alpha;
    solved = (ArNorm / (Anorm * rNorm) <= axtol) | ((REAL)1 + ArNorm / (Anorm * rNorm) <= (REAL)1);
    tired = iter >= itmax;
    zero_resid = ((REAL)1 + rNorm / beta1 <= (REAL)1) | (rNorm / beta1 <= axtol);
    while (!(solved || tired || ill_cond)) {
      iter = iter + 1;
      SUF(spmv_rect)(m, rowptr, colind, val, v, Av);
      SUF(kaxpby)(m, 1, Av, -alpha, Mu);
      if (!MisI) SUF(diagmul)(m, u, Mdiag, Mu, ldiv);
      beta = SUF(knorm_ell)(m, u, Mu);
      if (beta != 0) {
        SUF(kdiv)(m, u, beta);
        if (!MisI) SUF(kdiv)(m, Mu, beta);
        Anorm2 = Anorm2 + alpha * alpha + beta * beta;
        if (lambda > 0) Anorm2 += lambda2;
        SUF(spmv_t)(m, n, rowptr, colind, val, u, Atu);
        SUF(kaxpby)(n, 1, Atu, -beta, Nv);
        if (!NisI) SUF(diagmul)(n, v, Ndiag, Nv, ldiv);
        alpha = SUF(knorm_ell)(n, v, Nv);
        if (alpha != 0) { SUF(kdiv)(n, v, alpha); if (!NisI) SUF(kdiv)(n, Nv, alpha); }
      }
      REAL c1, s1, rhobar1, cs, sn, rho;
      SUF(oracle_sym_givens)(rhobar, lambda, &c1, &s1, &rhobar1);
      REAL psi = s1 * phibar;
      phibar = c1 * phibar;
      SUF(oracle_sym_givens)(rhobar1, beta, &cs, &sn, &rho);
      REAL phi = cs * phibar;
      phibar = sn * phibar;
      xENorm2 = xENorm2 + phi * phi;
      err_vec[iter % window] = phi;
      if (iter >= window) err_lbnd = SUF(err_norm)(window, err_vec);
      REAL tau = sn * phi, theta = sn * alpha;
      rhobar = -cs * alpha;
      dNorm2 += SUF(kdot)(n, w, w) / (rho * rho);
      REAL sigma = phi / rho;
      if (radius > 0) {
        REAL t1, t2;
        int e = SUF(oracle_to_boundary)(n, x, w, z, radius, 0, 0, 0, NULL, 0, &t1, &t2);
        if (e) { rc = 10 + e; goto done; }
        REAL tmax = t1 > t2 ? t1 : t2, tmin = t1 < t2 ? t1 : t2;
        on_boundary = sigma > tmax || sigma < tmin;
        sigma = sigma > 0 ? (sigma < tmax ? sigma : tmax) : (sigma > tmin ? sigma : tmin);
      }
      SUF(kaxpy)(n, sigma, w, x);
      SUF(kaxpby)(n, 1, v, -theta / rho, w);
      REAL delta = s2 * rho, gammabar = -c2 * rho, rhs = phi - delta * zz, zbar = rhs / gammabar, gamma;
      xNorm = SQRT(xNorm2 + zbar * zbar);
      SUF(oracle_sym_givens)(gammabar, theta, &c2, &s2, &gamma);
      zz = rhs / gamma;
      xNorm2 += zz * zz;
      Anorm = SQRT(Anorm2);
      Acond = Anorm * SQRT(dNorm2);
      REAL res1 = phibar * phibar;
      res2 += psi * psi;
      rNorm = SQRT(res1 + res2);
      ArNorm = alpha * FABS(tau);
      if (history) PUSH(Aresiduals, st->nAres, ArNorm);
      if (history) PUSH(residuals, st->nres, rNorm);
      REAL test1 = rNorm / beta1, test2 = ArNorm / (Anorm * rNorm), test3 = (REAL)1 / Acond;
      REAL t1 = test1 / ((REAL)1 + Anorm * xNorm / beta1);
      REAL rNormtol = btol + axtol * Anorm * xNorm / beta1;
      ill_cond_mach = ((REAL)1 + test3 <= (REAL)1);
      int solved_mach = ((REAL)1 + test2 <= (REAL)1), zero_resid_mach = ((REAL)1 + t1 <= (REAL)1);
      tired = iter >= itmax;
      ill_cond_lim = (test3 <= ctol);
      int solved_lim = (test2 <= axtol), solved_opt = ArNorm <= atol + rtol * ArNorm0, zero_resid_lim = (test1 <= rNormtol);
      if (iter >= window) fwd_err = err_lbnd <= etol * SQRT(xENorm2);
      ill_cond = ill_cond_mach || ill_cond_lim;
      zero_resid = zero_resid_mach || zero_resid_lim;
      solved = solved_mach || solved_lim || solved_opt || zero_resid || fwd_err || on_boundary;
    }
  } else {
    /* ---------------------------- lsmr.jl:238-429 ---------------------------- */
    REAL alpha = SUF(knorm_ell)(n, v, Nv);
    REAL zetabar = alpha * beta, alphabar = alpha, rho = 1, rhobar = 1, cbar = 1, sbar = 0;
    REAL betadd = beta, betad = 0, rhodold = 1, tautildeold = 0, thetatilde = 0, zeta = 0, d = 0;
    REAL Anorm2 = alpha * alpha, maxrbar = 0;
    REAL minrbar = (REAL)1.0e+100 < FLTMAX_OF ? (REAL)1.0e+100 : FLTMAX_OF;
    REAL Acond, Anorm = SQRT(Anorm2), xNorm = 0;
    REAL rNorm = beta;
    if (history) PUSH(residuals, st->nres, rNorm);
    REAL ArNorm = alpha * beta, ArNorm0 = ArNorm;
    if (history) PUSH(Aresiduals, st->nAres, ArNorm);
    if (alpha == 0) {
      st->niter = 0; st->solved = 1; st->inconsistent = 0;
      set_status(st, "x is a minimum least-squares solution");
      *Anorm_out = Anorm;
      goto done;
    }
    SUF(kdiv)(n, v, alpha);
    if (!NisI) SUF(kdiv)(n, Nv, alpha);
    SUF(kcopy)(n, h, v);
    SUF(kfill)(n, hbar, 0);
    solved = (rNorm <= axtol);
    tired = iter >= itmax;
    while (!(solved || tired || ill_cond)) {
      iter = iter + 1;
      SUF(spmv_rect)(m, rowptr, colind, val, v, Av);
      SUF(kaxpby)(m, 1, Av, -alpha, Mu);
      if (!MisI) SUF(diagmul)(m, u, Mdiag, Mu, ldiv);
      beta = SUF(knorm_ell)(m, u, Mu);
      if (beta != 0) {
        SUF(kdiv)(m, u, beta);
        if (!MisI) SUF(kdiv)(m, Mu, beta);
        SUF(spmv_t)(m, n, rowptr, colind, val, u, Atu);
        SUF(kaxpby)(n, 1, Atu, -beta, Nv);
        if (!NisI) SUF(diagmul)(n, v, Ndiag, Nv, ldiv);
        alpha = SUF(knorm_ell)(n, v, Nv);
        if (alpha != 0) { SUF(kdiv)(n, v, alpha); if (!NisI) SUF(kdiv)(n, Nv, alpha); }
      }
      REAL chat, shat, alphahat, cs, sn;
      SUF(oracle_sym_givens)(alphabar, lambda, &chat, &shat, &alphahat);
      REAL rhoold = rho;
      SUF(oracle_sym_givens)(alphahat, beta, &cs, &sn, &rho);
      REAL thetanew = sn * alpha;
      alphabar = cs * alpha;
      REAL rhobarold = rhobar, zetaold = zeta, thetabar = sbar * rho, rhotemp = cbar * rho;
      SUF(oracle_sym_givens)(rhotemp, thetanew, &cbar, &sbar, &rhobar);
      zeta = cbar * zetabar;
      zetabar = -sbar * zetabar;
      xENorm2 = xENorm2 + zeta * zeta;
      err_vec[iter % window] = zeta;
      if (iter >= window) err_lbnd = SUF(err_norm)(window, err_vec);
      REAL delta = thetabar * rho / (rhoold * rhobarold);
      SUF(kaxpby)(n, 1, h, -delta, hbar);
      REAL sigma = zeta / (rho * rhobar);
      if (radius > 0) {
        REAL t1, t2;
        int e = SUF(oracle_to_boundary)(n, x, hbar, z, radius, 0, 0, 0, NULL, 0, &t1, &t2);
        if (e) { rc = 10 + e; goto done; }
        REAL tmax = t1 > t2 ? t1 : t2, tmin = t1 < t2 ? t1 : t2;
        on_boundary = sigma > tmax || sigma < tmin;
        sigma = sigma > 0 ? (sigma < tmax ? sigma : tmax) : (sigma > tmin ? sigma : tmin);
      }
      SUF(kaxpy)(n, sigma, hbar, x);
      SUF(kaxpby)(n, 1, v, -thetanew / rho, h);
      REAL betaacute = chat * betadd, betacheck = -shat * betadd, betahat = cs * betaacute;
      betadd = -sn * betaacute;
      REAL thetatildeold = thetatilde, ctildeold, stildeold, rhotildeold;
      SUF(oracle_sym_givens)(rhodold, thetabar, &ctildeold, &stildeold, &rhotildeold);
      thetatilde = stildeold * rhobar;
      rhodold = ctildeold * rhobar;
      betad = -stildeold * betad + ctildeold * betahat;
      tautildeold = (zetaold - thetatildeold * tautildeold) / rhotildeold;
      REAL taud = (zeta - thetatilde * tautildeold) / rhodold;
      d = d + betacheck * betacheck;
      rNorm = SQRT(d + (betad - taud) * (betad - taud) + betadd * betadd);
      if (history) PUSH(residuals, st->nres, rNorm);
      Anorm2 += beta * beta;
      Anorm = SQRT(Anorm2);
      Anorm2 += alpha * alpha;
      maxrbar = maxrbar > rhobarold ? maxrbar : rhobarold;
      if (iter > 1) minrbar = minrbar < rhobarold ? minrbar : rhobarold;
      Acond = (maxrbar > rhotemp ? maxrbar : rhotemp) / (minrbar < rhotemp ? minrbar : rhotemp);
      ArNorm = FABS(zetabar);
      if (history) PUSH(Aresiduals, st->nAres, ArNorm);
      xNorm = SUF(knorm)(n, x);
      REAL test1 = rNorm / beta1, test2 = ArNorm / (Anorm * rNorm), test3 = (REAL)1 / Acond;
      REAL t1 = test1 / ((REAL)1 + Anorm * xNorm / beta1);
      REAL rNormtol = btol + axtol * Anorm * xNorm / beta1;
      ill_cond_mach = ((REAL)1 + test3 <= (REAL)1);
      int solved_mach = ((REAL)1 + test2 <= (REAL)1), zero_resid_mach = ((REAL)1 + t1 <= (REAL)1);
      tired = iter >= itmax;
      ill_cond_lim = (test3 <= ctol);
      int solved_lim = (test2 <= axtol), solved_opt = ArNorm <= atol + rtol * ArNorm0, zero_resid_lim = (test1 <= rNormtol);
      if (iter >= window) fwd_err = err_lbnd <= etol * SQRT(xENorm2);
      ill_cond = ill_cond_mach || ill_cond_lim;
      zero_resid = zero_resid_mach || zero_resid_lim;
      solved = solved_mach || solved_lim || solved_opt || zero_resid || fwd_err || on_boundary;
    }
    *Anorm_out = Anorm;
  }
  if (tired) set_status(st, "maximum number of iterations exceeded");
  if (ill_cond_mach) set_status(st, "condition number seems too large for this machine");
  if (ill_cond_lim) set_status(st, "condition number exceeds tolerance");
  if (solved) set_status(st, "found approximate minimum least-squares solution");
  if (zero_resid) set_status(st, "found approximate zero-residual solution");
  if (fwd_err) set_status(st, "truncated forward error small enough");
  if (on_boundary) set_status(st, "on trust-region boundary");
  st->niter = iter; st->solved = solved; st->inconsistent = !zero_resid;
done:
  free(Mu); free(Av); free(uu); free(Nv); free(Atu); free(vv); free(w); free(hbar); free(z); free(err_vec);
  return rc;
}

#undef PUSH
