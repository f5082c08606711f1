/*
 * krylov_oracle_ares.h -- TEST INFRASTRUCTURE ONLY (same status as krylov_oracle_impl.h, which must be included
 * first).  Literal restatement of car! (src/car.jl:108-256) and minares! (src/minares.jl:113-595) for real element
 * types, built with the BLAS-1 wrappers of krylov_oracle_impl.h into libkrylov_oracle_ares.so by ares.mk and loaded by
 * oracle/ares_oracle.py.  Parity pinning: tests/test_oracle_car_minares.py (the reference's assertions of
 * test/test_car.jl and test/test_minares.jl) and tests/golden/oracle_car_minares.json (frozen histories).
 * Both solvers minimize ||A r_k|| over the same Krylov space: CAR through CG-like short recurrences, MINARES through
 * the symmetric Lanczos process.  The callback (NULL: none) returns nonzero to stop; timemax < 0 means no limit.
 */
#define PUSH(arr, cnt, v) do { if ((arr) && (cnt) < o->hist_cap) (arr)[(cnt)] = (v); (cnt)++; } while (0)
#ifndef ORACLE_ARES_DEFINED
#define ORACLE_ARES_DEFINED
#include <time.h>
typedef int (*oracle_iter_cb)(int iter, void *user);
static double oracle_now(void) { struct timespec ts; timespec_get(&ts, TIME_UTC); return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec; }
#endif

/* ============ car!  (src/car.jl:108-256) ============
 * Mdiag: NULL => M === I (then Mu aliases u), else M = Diagonal(Mdiag) applied with mul! or ldiv!. */
int SUF(oracle_car)(int n, const int *rowptr, const int *colind, const REAL *val, const REAL *b, const REAL *x0,
                    const REAL *Mdiag, double timemax, oracle_iter_cb callback, void *cb_user, const oracle_opts *o,
                    REAL *x, REAL *residuals, REAL *Aresiduals, oracle_stats *st) {
  SUF(csr) A = {n, rowptr, colind, val};
  const double start = oracle_now();
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  int history = o->history, ldiv = o->ldiv, warm_start = (x0 != NULL), MisI = (Mdiag == NULL);
  REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol);
  int itmax = o->itmax;
  size_t nb = sizeof(REAL) * (size_t)n;
  REAL *r = malloc(nb), *p = malloc(nb), *s = malloc(nb), *q = malloc(nb), *t = malloc(nb), *u = malloc(nb);
  REAL *Mu = MisI ? u : malloc(nb);

  SUF(kfill)(n, x, 0);
  if (warm_start) { SUF(spmv)(&A, x0, r); SUF(kaxpby)(n, 1, b, -1, r); }
  else SUF(kcopy)(n, r, b);
  if (MisI) SUF(kcopy)(n, p, r);                                 /* p₀ = r₀ = M(b - Ax₀) */
  else { SUF(diagmul)(n, p, Mdiag, r, ldiv); SUF(kcopy)(n, r, p); }
  SUF(spmv)(&A, r, s);                                           /* s₀ = Ar₀ */
  if (MisI) SUF(kcopy)(n, q, s);                                 /* q₀ = MAp₀ and s₀ = MAr₀ */
  else { SUF(diagmul)(n, q, Mdiag, s, ldiv); SUF(kcopy)(n, s, q); }
  SUF(spmv)(&A, s, t);                                           /* t₀ = As₀ */
  SUF(kcopy)(n, u, t);                                           /* u₀ = Aq₀ */
  REAL rho = SUF(kdot)(n, t, s);                                 /* ρ₀ = ⟨t₀ , s₀⟩ */
  REAL rNorm = SUF(knorm)(n, r);
  if (history) PUSH(residuals, st->nres, rNorm);
  REAL ArNorm = MisI ? SUF(knorm)(n, s) : SQRT(SUF(kdot)(n, r, u));   /* knorm_elliptic(n, r, u) */
  if (history) PUSH(Aresiduals, st->nAres, ArNorm);
  if (rNorm == 0) {
    st->niter = 0; st->solved = 1; st->inconsistent = 0;
    set_status(st, "x is a zero-residual solution");
    if (warm_start) SUF(kaxpy)(n, 1, x0, x);
    goto done;
  }
  int iter = 0;
  if (itmax == 0) itmax = 2 * n;
  REAL eps_ = atol + rtol * rNorm;
  int solved = rNorm <= eps_, tired = iter >= itmax, user_exit = 0, overtimed = 0;
  while (!(solved || tired || user_exit || overtimed)) {
    if (!MisI) SUF(diagmul)(n, Mu, Mdiag, u, ldiv);
    REAL alpha = rho / SUF(kdot)(n, u, Mu);                      /* αₖ = ρₖ / ⟨uₖ, Muₖ⟩ */
    SUF(kaxpy)(n, alpha, p, x);
    SUF(kaxpy)(n, -alpha, q, r);
    SUF(kaxpy)(n, -alpha, Mu, s);
    rNorm = SUF(knorm)(n, r);
    if (history) PUSH(residuals, st->nres, rNorm);
    int resid_decrease_mach = (rNorm + (REAL)1 <= (REAL)1);
    solved = (rNorm <= eps_) || resid_decrease_mach;
    if (!solved) {
      SUF(spmv)(&A, s, t);                                       /* tₖ₊₁ = A * sₖ₊₁ */
      REAL rho_next = SUF(kdot)(n, t, s);
      REAL beta = rho_next / rho;
      rho = rho_next;
      SUF(kaxpby)(n, 1, r, beta, p);
      SUF(kaxpby)(n, 1, s, beta, q);
      SUF(kaxpby)(n, 1, t, beta, u);
      ArNorm = MisI ? SUF(knorm)(n, s) : SQRT(SUF(kdot)(n, r, u));
      if (history) PUSH(Aresiduals, st->nAres, ArNorm);
    }
    iter++;
    tired = iter >= itmax;
    user_exit = callback ? (callback(iter, cb_user) != 0) : 0;
    overtimed = timemax >= 0 && oracle_now() - start > timemax;
  }
  if (solved) set_status(st, "solution good enough given atol and rtol");
  if (tired) set_status(st, "maximum number of iterations exceeded");
  if (user_exit) set_status(st, "user-requested exit");
  if (overtimed) set_status(st, "time limit exceeded");
  if (warm_start) SUF(kaxpy)(n, 1, x0, x);
  st->niter = iter; st->solved = solved; st->inconsistent = 0;
done:
  free(r); free(p); free(s); free(q); free(t); free(u);
  if (!MisI) free(Mu);
  return 0;
}

/* ============ minares!  (src/minares.jl:113-595), M = I ============
 * o->lambda is the shift λ; artol is the kwarg Artol (NaN -> sqrt(eps)).  The reference refuses any M != I.
 * vₖ / vₖ₊₁, wₖ₋₂ / wₖ₋₁ and dₖ₋₂ / dₖ₋₁ are swapped as @kswap! does. */
int SUF(oracle_minares)(int n, const int *rowptr, const int *colind, const REAL *val, const REAL *b, const REAL *x0,
                        double artol, double timemax, oracle_iter_cb callback, void *cb_user, const oracle_opts *o,
                        REAL *x, REAL *residuals, REAL *Aresiduals, oracle_stats *st) {
  SUF(csr) A = {n, rowptr, colind, val};
  const double start = oracle_now();
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  int history = o->history, warm_start = (x0 != NULL);
  REAL lambda = (REAL)o->lambda;
  REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol), Artol = SUF(tol)(artol);
  int itmax = o->itmax;
  size_t nb = sizeof(REAL) * (size_t)n;
  REAL *vk = malloc(nb), *vk1 = malloc(nb), *wk2 = malloc(nb), *wk1 = malloc(nb), *dk2 = malloc(nb), *dk1 = malloc(nb);
  REAL *q = malloc(nb), *tmp;
  int iter = 0;
  if (itmax == 0) itmax = 2 * n;

  SUF(kfill)(n, x, 0);
  if (warm_start) {                                              /* β₁v₁ = r₀ */
    SUF(spmv)(&A, x0, vk);
    if (lambda != 0) SUF(kaxpy)(n, lambda, x0, vk);
    SUF(kaxpby)(n, 1, b, -1, vk);
  } else {
    SUF(kcopy)(n, vk, b);
  }
  REAL betak = SUF(knorm)(n, vk);
  if (betak != 0) SUF(kdiv)(n, vk, betak);
  REAL beta1 = betak;
  SUF(spmv)(&A, vk, vk1);                                        /* β₂v₂ = (A + λI)v₁ - α₁v₁ */
  if (lambda != 0) SUF(kaxpy)(n, lambda, vk, vk1);
  REAL alphak = SUF(kdot)(n, vk, vk1);
  SUF(kaxpy)(n, -alphak, vk, vk1);
  REAL betak1 = SUF(knorm)(n, vk1);
  if (betak1 != 0) SUF(kdiv)(n, vk1, betak1);

  REAL xik1 = 0, tauk2 = 0, tauk1 = 0, tauk = 0, thetabark2 = 0, psibisk2 = 0, psibark1 = 0;
  REAL pik2 = 0, pik1 = 0, pik = 0, chibark = 0, zetabisk = 0, zetabark1 = 0, gammabark = 0, lambdabark = 0, gammak1 = 0;
  REAL ct4 = 0, st4 = 0, ct3 = 0, st3 = 0, ct2 = 0, st2 = 0, ct1 = 0, st1 = 0, ct0 = 0, st0 = 0;   /* c̃₂ₖ₋₄ ... c̃₂ₖ */
  SUF(kfill)(n, wk2, 0);
  SUF(kfill)(n, wk1, 0);
  SUF(kfill)(n, dk2, 0);
  SUF(kfill)(n, dk1, 0);
  REAL b1a1 = betak * alphak, b1b2 = betak * betak1;             /* β₁α₁, β₁β₂ */
  REAL epsk2 = 0, epsk1 = 0;
  long long ell = (long long)itmax + 2;

  REAL rNorm = beta1;
  REAL eps_ = atol + rtol * rNorm;
  if (history) PUSH(residuals, st->nres, rNorm);
  REAL ArNorm = SQRT(b1a1 * b1a1 + b1b2 * b1b2);
  REAL kappa = atol + Artol * ArNorm;
  if (history) PUSH(Aresiduals, st->nAres, ArNorm);
  if (rNorm == 0) {
    st->niter = 0; st->solved = 1; st->inconsistent = 0;
    set_status(st, "x is a zero-residual solution");
    if (warm_start) SUF(kaxpy)(n, 1, x0, x);
    goto done;
  }
  const double btol = pow((double)EPS, 0.75);                    /* eps(T)^(3/4): a Float64 in the reference */
  int solved = (rNorm <= eps_) || (ArNorm <= kappa), breakdown = 0, tired = iter >= itmax, user_exit = 0, overtimed = 0;
  while (!(solved || tired || breakdown || user_exit || overtimed)) {
    iter++;
    long long k = iter;
    if (iter == 1) { lambdabark = alphak; gammabark = betak1; }
    REAL ck, sk, lambdak;
    SUF(oracle_sym_givens)(lambdabark, betak1, &ck, &sk, &lambdak);

    REAL *wk = NULL;
    if (iter == 1) { wk = wk1; SUF(kdivcopy)(n, wk, vk, lambdak); }
    if (iter == 2) { wk = wk2; SUF(kaxpy)(n, -gammak1, wk1, wk); SUF(kaxpy)(n, 1, vk, wk); SUF(kdiv)(n, wk, lambdak); }
    if (iter >= 3) {
      SUF(kscal)(n, -epsk2, wk2);
      wk = wk2; SUF(kaxpy)(n, -gammak1, wk1, wk); SUF(kaxpy)(n, 1, vk, wk); SUF(kdiv)(n, wk, lambdak);
    }

    REAL alphak1 = 0, betak2 = 0;
    if (k <= ell - 1) {
      SUF(spmv)(&A, vk1, q);
      SUF(kaxpby)(n, 1, q, -betak1, vk);
      if (lambda != 0) SUF(kaxpy)(n, lambda, vk1, vk);
      alphak1 = SUF(kdot)(n, vk, vk1);
      SUF(kaxpy)(n, -alphak1, vk1, vk);
      betak2 = SUF(knorm)(n, vk);
      if ((double)betak2 <= btol) ell = k + 1;
      else SUF(kdiv)(n, vk, betak2);
    }

    REAL epsk = 0, gammabark1 = 0, gammak = 0, lambdabark1 = 0;
    if (k <= ell - 2) { epsk = sk * betak2; gammabark1 = -ck * betak2; }
    if (k <= ell - 1) { gammak = ck * gammabark + sk * alphak1; lambdabark1 = sk * gammabark - ck * alphak1; }

    REAL rhok2 = 0, lambdahatk = 0, phibark1 = 0, mubark = 0, phik1 = 0, gammahatk = 0, mubisk = 0, muk = 0;
    if (iter >= 3) { rhok2 = st4 * lambdak; lambdahatk = -ct4 * lambdak; }
    if (iter == 2) lambdahatk = lambdak;
    if (iter >= 2) {
      phibark1 = st3 * lambdahatk;
      mubark = -ct3 * lambdahatk;
      if (k <= ell - 1) { phik1 = ct2 * phibark1 + st2 * gammak; gammahatk = st2 * phibark1 - ct2 * gammak; }
      else phik1 = phibark1;
    }
    if (iter == 1) { mubark = lambdak; gammahatk = gammak; }
    if (k <= ell - 1) SUF(oracle_sym_givens)(mubark, gammahatk, &ct1, &st1, &mubisk);
    else mubisk = mubark;
    if (k <= ell - 2) SUF(oracle_sym_givens)(mubisk, epsk, &ct0, &st0, &muk);
    else muk = mubisk;

    if (iter == 1) { zetabisk = b1a1; zetabark1 = b1b2; }
    REAL zetaringk, zetabisk1 = 0, zetak, zetabark2 = 0;
    if (k <= ell - 1) { zetaringk = ct1 * zetabisk + st1 * zetabark1; zetabisk1 = st1 * zetabisk - ct1 * zetabark1; }
    else zetaringk = zetabisk;
    if (k <= ell - 2) { zetak = ct0 * zetaringk; zetabark2 = st0 * zetaringk; }
    else zetak = zetaringk;

    REAL *dk = NULL;
    if (iter == 1) { dk = dk1; SUF(kdivcopy)(n, dk, wk, muk); }
    if (iter == 2) { dk = dk2; SUF(kaxpy)(n, -phik1, dk1, dk); SUF(kaxpy)(n, 1, wk, dk); SUF(kdiv)(n, dk, muk); }
    if (iter >= 3) {
      SUF(kscal)(n, -rhok2, dk2);
      dk = dk2; SUF(kaxpy)(n, -phik1, dk1, dk); SUF(kaxpy)(n, 1, wk, dk); SUF(kdiv)(n, dk, muk);
    }
    SUF(kaxpy)(n, zetak, dk, x);

    if (k <= ell - 2) ArNorm = SQRT(zetabisk1 * zetabisk1 + zetabark2 * zetabark2);
    if (k == ell - 1) ArNorm = FABS(zetabisk1);
    if (k == ell) ArNorm = 0;
    if (history) PUSH(Aresiduals, st->nAres, ArNorm);

    REAL psibark = 0, ch3 = 0, sh3 = 0, psibisk1 = 0, thetabark1 = 0, ch4 = 0, sh4 = 0, psik2 = 0, thetak2 = 0, deltak = 0;
    REAL omegak2 = 0, etak = 0;
    if (iter == 1) {
      psibark = muk;
    } else if (iter == 2) {
      SUF(oracle_sym_givens)(psibark1, phik1, &ch3, &sh3, &psibisk1);
      thetabark1 = sh3 * muk;
      psibark = -ch3 * muk;
    } else {
      SUF(oracle_sym_givens)(psibisk2, rhok2, &ch4, &sh4, &psik2);
      thetak2 = ch4 * thetabark2 + sh4 * phik1;
      deltak = sh4 * thetabark2 - ch4 * phik1;
      omegak2 = sh4 * muk;
      etak = -ch4 * muk;
      SUF(oracle_sym_givens)(psibark1, deltak, &ch3, &sh3, &psibisk1);
      thetabark1 = sh3 * etak;
      psibark = -ch3 * etak;
    }

    REAL xik = 0;
    if (iter == 1) {
      tauk = zetak / psibark;
    } else if (iter == 2) {
      tauk1 = tauk;
      tauk1 = tauk1 * psibark1 / psibisk1;
      xik = zetak;
      tauk = (xik - thetabark1 * tauk1) / psibark;
    } else {
      tauk2 = tauk1;
      tauk2 = tauk2 * psibisk2 / psik2;
      tauk1 = (xik1 - thetak2 * tauk2) / psibisk1;
      xik = zetak - omegak2 * tauk2;
      tauk = (xik - thetabark1 * tauk1) / psibark;
    }

    if (iter == 1) chibark = beta1;
    REAL chik = ck * chibark, chibark1 = sk * chibark;
    if (iter == 1) {
      pik = chik;
    } else if (iter == 2) {
      REAL piaux1 = pik1;
      pik1 = ch3 * piaux1 + sh3 * chik;
      pik = sh3 * piaux1 - ch3 * chik;
    } else {
      REAL piaux2 = pik2;
      pik2 = ch4 * piaux2 + sh4 * chik;
      pik = sh4 * piaux2 - ch4 * chik;
      REAL piaux1 = pik1;
      pik1 = ch3 * piaux1 + sh3 * pik;
      pik = sh3 * piaux1 - ch3 * pik;
    }
    REAL pik_1 = chibark1;                                       /* πₖ₊₁ */
    if (iter == 1) rNorm = SQRT((pik - tauk) * (pik - tauk) + pik_1 * pik_1);
    else rNorm = SQRT((pik1 - tauk1) * (pik1 - tauk1) + (pik - tauk) * (pik - tauk) + pik_1 * pik_1);
    if (history) PUSH(residuals, st->nres, rNorm);

    breakdown = (double)betak1 <= btol;
    solved = (rNorm <= eps_) || (ArNorm <= kappa);
    tired = iter >= itmax;
    overtimed = timemax >= 0 && oracle_now() - start > timemax;
    user_exit = callback ? (callback(iter, cb_user) != 0) : 0;

    tmp = vk; vk = vk1; vk1 = tmp;
    if (iter >= 2) {
      tmp = wk2; wk2 = wk1; wk1 = tmp;
      tmp = dk2; dk2 = dk1; dk1 = tmp;
      epsk2 = epsk1; ct4 = ct2; st4 = st2; xik1 = xik; psibisk2 = psibisk1; thetabark2 = thetabark1; pik2 = pik1;
    }
    ct3 = ct1; st3 = st1; ct2 = ct0; st2 = st0;
    betak = betak1; chibark = chibark1; psibark1 = psibark; pik1 = pik;
    if (k <= ell - 1) { alphak = alphak1; betak1 = betak2; gammak1 = gammak; lambdabark = lambdabark1; zetabisk = zetabisk1; }
    if (k <= ell - 2) { epsk1 = epsk; gammabark = gammabark1; zetabark1 = zetabark2; }
  }
  (void)betak;
  if (solved) set_status(st, "solution good enough given atol, rtol and Artol");
  if (tired) set_status(st, "maximum number of iterations exceeded");
  if (user_exit) set_status(st, "user-requested exit");
  if (overtimed) set_status(st, "time limit exceeded");
  if (warm_start) SUF(kaxpy)(n, 1, x0, x);
  st->niter = iter; st->solved = solved; st->inconsistent = 0;
done:
  free(vk); free(vk1); free(wk2); free(wk1); free(dk2); free(dk1); free(q);
  return 0;
}
#undef PUSH
