/*
 * krylov_oracle_lslq.h -- TEST INFRASTRUCTURE ONLY (same status as krylov_oracle_impl.h; include it and
 * krylov_oracle_lsq.h first, instantiated by krylov_oracle.c).  Literal restatement of lslq! (src/lslq.jl:201-520)
 * on an m x n CSR matrix, with the products of krylov_oracle_lsq.h (A^T u in ascending row order of A).  M (m entries)
 * and N (n entries) are diagonals or NULL.
 * Parity pinning: the reference's own assertions of test/test_lslq.jl (tests/test_oracle_cgls.py).
 */
#define PUSH(arr, cnt, v) do { if ((arr) && (cnt) < o->hist_cap) (arr)[(cnt)] = (v); (cnt)++; } while (0)

/* Writes the histories residuals, Aresiduals, err_lbnds, err_ubnds_lq and err_ubnds_cg, and error_with_bnd. */
static int SUF(lslq)(int variant, const SUF(problem) *P, const oracle_options *o, SUF(outputs) *out, oracle_stats *st) {
  const int m = P->m, n = P->n;
  const int *rowptr = P->rowptr, *colind = P->colind;
  const REAL *val = P->val, *b = P->b, *Mdiag = P->M, *Ndiag = P->N;
  REAL *x = out->x;
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  out->n_err_lbnds = out->n_err_ubnds_lq = out->n_err_ubnds_cg = 0;
  int *error_with_bnd = &out->error_with_bnd;
  *error_with_bnd = 0;
  int history = o->history, ldiv = o->ldiv;
  int MisI = (Mdiag == NULL), NisI = (Ndiag == NULL);
  REAL lambda = (REAL)o->lambda, lambda2 = lambda * lambda, sigma = (REAL)o->sigma;
  REAL conlim = isnan(o->conlim) ? (REAL)1 / SQRT(EPS) : (REAL)o->conlim;
  REAL ctol = conlim > 0 ? (REAL)1 / conlim : (REAL)0;
  REAL etol = SUF(tol)(o->etol), utol = SUF(tol)(o->utol);
  REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol);
  int window = o->window > 0 ? o->window : 5;
  size_t mb = sizeof(REAL) * (size_t)(m > 0 ? m : 1), nb = sizeof(REAL) * (size_t)(n > 0 ? n : 1);
  REAL *Mu = malloc(mb), *Av = malloc(mb), *uu = MisI ? NULL : malloc(mb);
  REAL *Nv = malloc(nb), *Atu = malloc(nb), *vv = NisI ? NULL : malloc(nb), *wbar = malloc(nb);
  REAL *err_vec = calloc((size_t)window, sizeof(REAL));
  REAL *u = MisI ? Mu : uu, *v = NisI ? Nv : vv;

  SUF(kfill)(n, x, 0);
  SUF(kcopy)(m, Mu, b);
  if (!MisI) SUF(diagmul)(m, u, Mdiag, Mu, ldiv);
  REAL beta1 = SUF(knorm_ell)(m, u, Mu);
  if (beta1 == 0) {
    st->niter = 0; st->solved = 1; st->inconsistent = 0;
    if (history) { PUSH(out->residuals, st->nres, 0); PUSH(out->Aresiduals, st->nAres, 0); }
    set_status(st, "x is a zero-residual solution");
    goto done;
  }
  REAL beta = beta1;
  SUF(kdiv)(m, u, beta1);
  if (!MisI) SUF(kdiv)(m, Mu, beta1);
  SUF(spmv_t)(m, n, rowptr, colind, val, u, Atu);
  SUF(kcopy)(n, Nv, Atu);
  if (!NisI) SUF(diagmul)(n, v, Ndiag, Nv, ldiv);
  REAL alpha = SUF(knorm_ell)(n, v, Nv);
  if (alpha == 0) {
    st->niter = 0; st->solved = 1; st->inconsistent = 0;
    if (history) { PUSH(out->residuals, st->nres, beta1); PUSH(out->Aresiduals, st->nAres, 0); }
    set_status(st, "x is a minimum least-squares solution");
    goto done;
  }
  SUF(kdiv)(n, v, alpha);
  if (!NisI) SUF(kdiv)(n, Nv, alpha);
  {
    REAL Anorm = alpha, Anorm2 = alpha * alpha;
    REAL sigmax = 0, sigmin = (REAL)INFINITY, Acond = 0;
    REAL xlqNorm = 0, xlqNorm2 = 0, xcgNorm2 = 0;
    SUF(kcopy)(n, wbar, v);
    REAL err_lbnd = 0;
    int complex_error_bnd = 0;
    REAL alphaL = alpha, betaL = beta, rhobar = -sigma, gammabar = alpha, psi = beta1;
    REAL c = -1, s = 0, delta = -1, tau = alpha * beta1, zeta = 0, zetabar = 0, zetatilde = 0, csig = -1;
    REAL rNorm = beta1, ArNorm = alpha * beta;
    if (history) { PUSH(out->residuals, st->nres, rNorm); PUSH(out->Aresiduals, st->nAres, ArNorm); }
    int iter = 0, itmax = o->itmax != 0 ? o->itmax : m + n;
    REAL eps = atol + rtol * beta1;
    int solved = rNorm <= eps, tired = iter >= itmax, ill_cond = 0, ill_cond_mach = 0, ill_cond_lim = 0;
    int zero_resid = 0, fwd_err_lbnd = 0, fwd_err_ubnd = 0;
    while (!(solved || tired || ill_cond)) {
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
        alphaL = alpha;
        betaL = beta;
        if (lambda != 0) {
          REAL cL, sL;
          SUF(oracle_sym_givens)(beta, lambda, &cL, &sL, &betaL);
          alphaL = cL * alpha;
          lambda = SQRT(lambda2 + (sL * alpha) * (sL * alpha));
        }
        Anorm2 = Anorm2 + alphaL * alphaL + betaL * betaL;
        Anorm = SQRT(Anorm2);
      }
      REAL cp, sp, gamma;
      SUF(oracle_sym_givens)(gammabar, betaL, &cp, &sp, &gamma);
      tau = -tau * delta / gamma;
      delta = sp * alphaL;
      gammabar = -cp * alphaL;
      REAL omega = 0;
      if (sigma > 0 && !complex_error_bnd) {
        REAL mubar = -csig * gamma, ssig, rho;
        SUF(oracle_sym_givens)(rhobar, gamma, &csig, &ssig, &rho);
        rhobar = ssig * mubar + csig * sigma;
        mubar = -csig * delta;
        REAL h = delta * csig / rhobar;
        REAL disc = sigma * (sigma - delta * h);
        if (disc < 0) complex_error_bnd = 1; else omega = SQRT(disc);
        SUF(oracle_sym_givens)(rhobar, delta, &csig, &ssig, &rho);
        rhobar = ssig * mubar + csig * sigma;
      }
      REAL epsbar = -gamma * c, eta = gamma * s, epsl;
      SUF(oracle_sym_givens)(epsbar, delta, &c, &s, &epsl);
      REAL ae = FABS(epsbar);
      sigmax = sigmax > epsl ? sigmax : epsl; sigmax = sigmax > ae ? sigmax : ae;
      sigmin = sigmin < epsl ? sigmin : epsl; sigmin = sigmin < ae ? sigmin : ae;
      Acond = sigmax / sigmin;
      REAL zetaold = zeta;
      zeta = (tau - zeta * eta) / epsl;
      zetabar = zeta / c;
      REAL ra = psi * cp - zetaold * eta, rb = psi * sp;
      rNorm = SQRT(ra * ra + rb * rb);
      if (history) PUSH(out->residuals, st->nres, rNorm);
      REAL aa = gamma * epsl * zeta, ab = delta * eta * zetaold;
      ArNorm = SQRT(aa * aa + ab * ab);
      if (history) PUSH(out->Aresiduals, st->nAres, ArNorm);
      psi = psi * sp;
      xcgNorm2 = xlqNorm2 + zetabar * zetabar;
      if (sigma > 0 && iter > 0 && !complex_error_bnd) {
        REAL disc = zetatilde * zetatilde - zetabar * zetabar;
        if (disc < 0) complex_error_bnd = 1;
        else {
          REAL ub = SQRT(disc);
          if (history) PUSH(out->err_ubnds_cg, out->n_err_ubnds_cg, ub);
          fwd_err_ubnd = ub <= utol * SQRT(xcgNorm2);
        }
      }
      REAL test1 = rNorm, test2 = ArNorm / (Anorm * rNorm), test3 = (REAL)1 / Acond;
      REAL t1 = test1 / ((REAL)1 + Anorm * xlqNorm);
      SUF(kaxpy)(n, c * zeta, wbar, x);
      SUF(kaxpy)(n, s * zeta, v, x);
      SUF(kaxpby)(n, -c, v, s, wbar);
      xlqNorm2 += zeta * zeta;
      xlqNorm = SQRT(xlqNorm2);
      err_vec[iter % window] = zeta;
      if (iter >= window) {
        err_lbnd = SUF(err_norm)(window, err_vec);
        if (history) PUSH(out->err_lbnds, out->n_err_lbnds, err_lbnd);
        fwd_err_lbnd = err_lbnd <= etol * xlqNorm;
      }
      if (sigma > 0 && !complex_error_bnd) {
        REAL etatilde = omega * s, epstilde = -omega * c, tautilde = -tau * delta / omega;
        zetatilde = (tautilde - zeta * etatilde) / epstilde;
        if (history) PUSH(out->err_ubnds_lq, out->n_err_ubnds_lq, FABS(zetatilde));
      }
      ill_cond_mach = ((REAL)1 + test3 <= (REAL)1);
      int solved_mach = ((REAL)1 + test2 <= (REAL)1), zero_resid_mach = ((REAL)1 + t1 <= (REAL)1);
      tired = iter >= itmax;
      ill_cond_lim = (test3 <= ctol);
      int solved_lim = (test2 <= atol), zero_resid_lim = (test1 <= eps);
      ill_cond = ill_cond_mach || ill_cond_lim;
      zero_resid = zero_resid_mach || zero_resid_lim;
      solved = solved_mach || solved_lim || zero_resid || fwd_err_lbnd || fwd_err_ubnd;
      iter = iter + 1;
    }
    if (o->transfer_to_lsqr) SUF(kaxpy)(n, zetabar, wbar, x);
    if (tired) set_status(st, "maximum number of iterations exceeded");
    if (ill_cond_mach) set_status(st, "condition number seems too large for this machine");
    if (ill_cond_lim) set_status(st, "condition number exceeds tolerance");
    if (solved) set_status(st, "found approximate minimum least-squares solution");
    if (zero_resid) set_status(st, "found approximate zero-residual solution");
    if (fwd_err_lbnd) set_status(st, "forward error lower bound small enough");
    if (fwd_err_ubnd) set_status(st, "forward error upper bound small enough");
    st->niter = iter; st->solved = solved; st->inconsistent = !zero_resid;
    *error_with_bnd = complex_error_bnd;
    (void)err_lbnd; (void)ill_cond_mach;
  }
done:
  free(Mu); free(Av); free(uu); free(Nv); free(Atu); free(vv); free(wbar); free(err_vec);
  return 0;
}

#undef PUSH
