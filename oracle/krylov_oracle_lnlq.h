/*
 * krylov_oracle_lnlq.h -- TEST INFRASTRUCTURE ONLY (same status as krylov_oracle_impl.h, which must be included first).
 * Restatement of lnlq! (src/lnlq.jl:168-568), SYMMLQ on A A^T y = b with x = A^T y: the least-norm solution of
 * A x = b on an m x n CSR matrix, with the sigma-based upper bounds on ||x - x*|| and ||y - y*||.  Written from the
 * algorithm on the BLAS-1 wrappers of krylov_oracle_impl.h, instantiated by krylov_oracle.c and loaded by
 * oracle/lnlq_oracle.py.  A^T is passed as its own CSR (n rows, ascending row indices of A in each row).  M (m entries)
 * and N (n entries) are diagonals or NULL.
 * Parity pinning: tests/test_oracle_lnlq.py (the reference's assertions of test/test_lnlq.jl) and
 * tests/golden/oracle_lnlq.json (frozen histories).
 */
#define PUSH(arr, cnt, v) do { if ((arr) && (cnt) < o->hist_cap) (arr)[(cnt)] = (v); (cnt)++; } while (0)

static REAL SUF(lnlq_knorm_ell)(int n, const REAL *x, const REAL *y) {   /* knorm_elliptic (krylov_utils.jl:319) */
  return x == y ? SUF(knorm)(n, x) : SQRT(SUF(kdot)(n, x, y));
}

/* lnlq! (src/lnlq.jl:168-568).  Writes the histories residuals, error_bnd_x and error_bnd_y, and error_with_bnd.
 * `iter` is incremented before the loop and at the end of every pass: niter = passes + 1. */
static int SUF(lnlq)(int variant, const SUF(problem) *P, const oracle_options *o, SUF(outputs) *out, oracle_stats *st) {
  const int m = P->m, n = P->n;
  const REAL *b = P->b, *Mdiag = P->M, *Ndiag = P->N;
  REAL *x = out->x, *y = out->y, *res = out->residuals, *errx = out->error_bnd_x, *erry = out->error_bnd_y;
  SUF(csr) A = {m, P->rowptr, P->colind, P->val}, At = {n, P->trowptr, P->tcolind, P->tval};
  const double start = oracle_now();
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  out->n_error_bnd_x = out->n_error_bnd_y = out->error_with_bnd = 0;
  const int history = o->history, ldiv = o->ldiv, MisI = Mdiag == NULL, NisI = Ndiag == NULL;
  const int transfer = o->transfer_to_craig;
  const REAL lambda = (REAL)o->lambda, sigma = (REAL)o->sigma;
  const REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol), utolx = SUF(tol)(o->utolx), utoly = SUF(tol)(o->utoly);
  const int itmax = o->itmax > 0 ? o->itmax : m + n;
  size_t nbm = sizeof(REAL) * (size_t)(m > 0 ? m : 1), nbn = sizeof(REAL) * (size_t)(n > 0 ? n : 1);
  REAL *Mu = malloc(nbm), *Av = malloc(nbm), *wbar = malloc(nbm), *ub = MisI ? NULL : malloc(nbm);
  REAL *Nv = malloc(nbn), *Atu = malloc(nbn), *vb = NisI ? NULL : malloc(nbn), *q = malloc(nbn);
  REAL *u = MisI ? Mu : ub, *v = NisI ? Nv : vb;
  const REAL sigma_est = SQRT(sigma * sigma + lambda * lambda);
  int complex_error_bnd = 0, iter = 0;
  int solved_lq = 0, solved_cg = 0, tired = 0, user_exit = 0, overtimed = 0;

  SUF(kfill)(n, x, 0);
  SUF(kfill)(m, y, 0);
  const REAL bNorm = SUF(knorm)(m, b);
  if (bNorm == 0) {
    st->niter = 0; st->solved = 1;
    if (history) PUSH(res, st->nres, bNorm);
    set_status(st, "x is a zero-residual solution");
    goto done;
  }
  if (history) PUSH(res, st->nres, bNorm);
  const REAL eps_c = atol + rtol * bNorm;
  iter = iter + 1;

  SUF(kcopy)(m, Mu, b);                                         /* β₁Mu₁ = b */
  if (!MisI) SUF(diagmul)(m, u, Mdiag, Mu, ldiv);
  REAL beta = SUF(lnlq_knorm_ell)(m, u, Mu);
  if (beta != 0) {
    SUF(kdiv)(m, u, beta);
    if (!MisI) SUF(kdiv)(m, Mu, beta);
  }
  SUF(spmv)(&At, u, Atu);                                       /* α₁Nv₁ = Aᵀu₁ */
  SUF(kcopy)(n, Nv, Atu);
  if (!NisI) SUF(diagmul)(n, v, Ndiag, Nv, ldiv);
  REAL alpha = SUF(lnlq_knorm_ell)(n, v, Nv);
  if (alpha != 0) {
    SUF(kdiv)(n, v, alpha);
    if (!NisI) SUF(kdiv)(n, Nv, alpha);
  }
  SUF(kcopy)(m, wbar, u);                                       /* w̄₁ = u₁ */
  REAL sk = 0, zeta_km1 = 0, etak = 0, cpk = 1, spk = 1, alphahat;
  if (lambda > 0) SUF(kcopy)(n, q, v);
  if (lambda > 0) {
    SUF(oracle_sym_givens)(alpha, lambda, &cpk, &spk, &alphahat);
    SUF(kscal)(n, spk, q);
  } else {
    alphahat = alpha;
  }
  REAL epsbar = alphahat, tau = beta / alphahat;
  REAL zetabar = tau / epsbar, thetak = tau;
  REAL err_x = 0, err_y = 0, tautilde = 0, rhobar = 0, csig = 0;
  if (sigma_est > 0) {
    tautilde = beta / sigma_est;
    const REAL zetatilde = tautilde / sigma_est;
    err_x = tautilde;
    err_y = zetatilde;
    solved_lq = err_x <= utolx || err_y <= utoly;
    if (history) { PUSH(errx, out->n_error_bnd_x, err_x); PUSH(erry, out->n_error_bnd_y, err_y); }
    rhobar = -sigma_est;
    csig = -1;
  }

  while (!(solved_lq || solved_cg || tired || user_exit || overtimed)) {
    if (lambda > 0) {
      SUF(kaxpy)(n, tau * cpk, v, x);
      if (iter >= 2) {
        SUF(kaxpy)(n, tau * spk, q, x);
        SUF(kaxpby)(n, spk, v, -cpk, q);
      }
    } else {
      SUF(kaxpy)(n, tau, v, x);
    }
    SUF(spmv)(&A, v, Av);                                       /* βMu = A v - αMu */
    SUF(kaxpby)(m, 1, Av, -alpha, Mu);
    if (!MisI) SUF(diagmul)(m, u, Mdiag, Mu, ldiv);
    const REAL beta_next = SUF(lnlq_knorm_ell)(m, u, Mu);
    if (beta_next != 0) {
      SUF(kdiv)(m, u, beta_next);
      if (!MisI) SUF(kdiv)(m, Mu, beta_next);
    }
    SUF(spmv)(&At, u, Atu);                                     /* αNv = Aᵀu - βNv */
    SUF(kaxpby)(n, 1, Atu, -beta_next, Nv);
    if (!NisI) SUF(diagmul)(n, v, Ndiag, Nv, ldiv);
    const REAL alpha_next = SUF(lnlq_knorm_ell)(n, v, Nv);
    if (alpha_next != 0) {
      SUF(kdiv)(n, v, alpha_next);
      if (!NisI) SUF(kdiv)(n, Nv, alpha_next);
    }
    REAL betahat, alphahat_next, cp_next = cpk, sp_next = spk;
    if (lambda > 0) {
      betahat = cpk * beta_next;
      const REAL theta_reg = spk * beta_next;
      REAL cdk, sdk, lambda_next;
      SUF(oracle_sym_givens)(lambda, theta_reg, &cdk, &sdk, &lambda_next);
      SUF(kscal)(n, sdk, q);
      SUF(oracle_sym_givens)(alpha_next, lambda_next, &cp_next, &sp_next, &alphahat_next);
    } else {
      betahat = beta_next;
      alphahat_next = alpha_next;
    }
    REAL omega = 0;
    if (sigma_est > 0 && !complex_error_bnd) {
      REAL mubar = -csig * alphahat;
      REAL rho = SQRT(rhobar * rhobar + alphahat * alphahat);
      csig = rhobar / rho;
      REAL ssig = alphahat / rho;
      rhobar = ssig * mubar + csig * sigma_est;
      mubar = -csig * betahat;
      const REAL theta = betahat * csig / rhobar;
      const REAL omega_disc = sigma_est * sigma_est - sigma_est * betahat * theta;
      if (omega_disc < 0) {
        complex_error_bnd = 1;
      } else {
        omega = SQRT(omega_disc);
        tautilde = -tau * betahat / omega;
      }
      rho = SQRT(rhobar * rhobar + betahat * betahat);
      csig = rhobar / rho;
      ssig = betahat / rho;
      rhobar = ssig * mubar + csig * sigma_est;
    }
    const REAL tau_next = -betahat * tau / alphahat_next;
    REAL c_next, s_next, epsk;
    SUF(oracle_sym_givens)(epsbar, betahat, &c_next, &s_next, &epsk);
    const REAL eta_next = alphahat_next * s_next;
    const REAL epsbar_next = -alphahat_next * c_next;
    const REAL zetak = thetak / epsk;
    const REAL theta_next = tau_next - eta_next * zetak;
    const REAL zetabar_next = theta_next / epsbar_next;
    SUF(kaxpy)(m, zetak * c_next, wbar, y);                     /* y += ζₖ wₖ */
    SUF(kaxpy)(m, zetak * s_next, u, y);
    SUF(kaxpby)(m, -c_next, u, s_next, wbar);                   /* w̄ₖ₊₁ */
    if (sigma_est > 0 && !complex_error_bnd) {
      if (transfer) {
        const REAL disc_x = tautilde * tautilde - tau_next * tau_next;
        if (disc_x < 0) complex_error_bnd = 1; else err_x = SQRT(disc_x);
      } else {
        const REAL d = tau_next - eta_next * zetak;
        const REAL disc_xL = tautilde * tautilde - tau_next * tau_next + d * d;
        if (disc_xL < 0) complex_error_bnd = 1; else err_x = SQRT(disc_xL);
      }
      const REAL etatilde = omega * s_next, epstilde = -omega * c_next;
      const REAL zetatilde = (tautilde - etatilde * zetak) / epstilde;
      if (transfer) {
        const REAL disc_y = zetatilde * zetatilde - zetabar_next * zetabar_next;
        if (disc_y < 0) complex_error_bnd = 1; else err_y = SQRT(disc_y);
      } else {
        err_y = FABS(zetatilde);
      }
      if (history) { PUSH(errx, out->n_error_bnd_x, err_x); PUSH(erry, out->n_error_bnd_y, err_y); }
    }
    REAL rNorm_lq;
    if (iter == 1) {
      rNorm_lq = bNorm;
    } else {
      const REAL ra = epsbar * zetabar, rb = betahat * sk * zeta_km1;
      rNorm_lq = FABS(alphahat) * SQRT(ra * ra + rb * rb);
    }
    if (history) PUSH(res, st->nres, rNorm_lq);
    const REAL rNorm_cg = transfer ? FABS(betahat * tau) : 0;
    user_exit = o->callback ? o->callback(iter, o->cb_user) != 0 : 0;
    tired = iter >= itmax;
    solved_lq = rNorm_lq <= eps_c;
    solved_cg = transfer && (FABS(zetabar) > EPS) && (rNorm_cg <= eps_c);
    if (sigma_est > 0) {
      solved_lq = solved_lq || err_x <= utolx || err_y <= utoly;
      solved_cg = transfer && (solved_cg || err_x <= utolx || err_y <= utoly);
    }
    overtimed = o->timemax >= 0 && oracle_now() - start > o->timemax;
    sk = s_next;
    alpha = alpha_next;
    alphahat = alphahat_next;
    etak = eta_next;
    thetak = theta_next;
    epsbar = epsbar_next;
    tau = tau_next;
    zeta_km1 = zetak;
    zetabar = zetabar_next;
    if (lambda > 0) { cpk = cp_next; spk = sp_next; }
    iter = iter + 1;
  }
  (void)beta;
  if (solved_cg && zetabar > EPS) {                             /* the CRAIG point: a signed test */
    if (lambda > 0) {
      SUF(kaxpy)(n, tau * cpk, v, x);
      if (iter >= 2) SUF(kaxpy)(n, tau * spk, q, x);
    } else {
      SUF(kaxpy)(n, tau, v, x);
    }
    SUF(kaxpy)(m, zetabar, wbar, y);
  } else {
    if (lambda > 0) {
      SUF(kaxpy)(n, etak * zeta_km1 * cpk, v, x);
      if (iter >= 2) SUF(kaxpy)(n, etak * zeta_km1 * spk, q, x);
    } else {
      SUF(kaxpy)(n, etak * zeta_km1, v, x);
    }
  }
  {
    const char *s = "unknown";
    if (tired) s = "maximum number of iterations exceeded";
    if (solved_lq) s = "solutions (xᴸ, yᴸ) good enough for the tolerances given";
    if (solved_cg) s = "solutions (xᶜ, yᶜ) good enough for the tolerances given";
    if (user_exit) s = "user-requested exit";
    if (overtimed) s = "time limit exceeded";
    set_status(st, s);
  }
  st->niter = iter; st->solved = solved_lq || solved_cg; st->inconsistent = 0;
  out->error_with_bnd = complex_error_bnd;
done:
  free(Mu); free(Av); free(wbar); free(ub); free(Nv); free(Atu); free(vb); free(q);
  return 0;
}


#undef PUSH
