/*
 * krylov_oracle_biorth.h -- TEST INFRASTRUCTURE ONLY (same status as krylov_oracle_impl.h, which must be included
 * first).  Literal restatement of bilq! (src/bilq.jl:118-407) and qmr! (src/qmr.jl:124-405), built with the BLAS-1
 * wrappers of krylov_oracle_impl.h into libkrylov_oracle_biorth.so by biorth.mk and loaded by oracle/biorth_oracle.py.
 * Parity pinning: tests/test_oracle_bilq_qmr.py (the reference's assertions of test/test_bilq.jl and test/test_qmr.jl)
 * and tests/golden/oracle_bilq_qmr.json (frozen histories).
 */
#define PUSH(arr, cnt, v) do { if ((arr) && (cnt) < o->hist_cap) (arr)[(cnt)] = (v); (cnt)++; } while (0)

/* ============ bilq!  (src/bilq.jl:118-407) and qmr!  (src/qmr.jl:124-405) ============
 * Both run the same Lanczos biorthogonalization (bilq.jl:226-255 = qmr.jl:230-258); they differ in the factorization
 * of the tridiagonal kept on the host and in the direction / solution update.  qmr != 0 selects QMR.  A^T is passed
 * as its own CSR (rows ascending in each column of A: the order of the reference's adjoint product).  The callback
 * (NULL: none) returns nonzero to stop; timemax < 0 means no limit.  Unlike the reference, v / u / w are copied and
 * swapped exactly as written (kcopy!, @kswap!). */
#ifndef ORACLE_BIORTH_DEFINED
#define ORACLE_BIORTH_DEFINED
#include <time.h>
typedef int (*oracle_iter_cb)(int iter, void *user);
static double oracle_now(void) { struct timespec ts; timespec_get(&ts, TIME_UTC); return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec; }
#endif
int SUF(oracle_biorth)(int qmr, int n, const int *rowptr, const int *colind, const REAL *val,
                       const int *trowptr, const int *tcolind, const REAL *tval,
                       const REAL *b, const REAL *c_in, const REAL *x0, const REAL *Mdiag, const REAL *Ndiag,
                       int transfer_to_bicg, double timemax, oracle_iter_cb callback, void *cb_user,
                       const oracle_opts *o, REAL *x, REAL *residuals, oracle_stats *st) {
  SUF(csr) A = {n, rowptr, colind, val}, At = {n, trowptr, tcolind, tval};
  const double start = oracle_now();
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  int history = o->history, ldiv = o->ldiv, warm_start = (x0 != NULL);
  int MisI = (Mdiag == NULL), NisI = (Ndiag == NULL);
  const REAL *c = c_in ? c_in : b;                                /* kwarg c = b */
  REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol);
  int itmax = o->itmax;
  size_t nb = sizeof(REAL) * (size_t)n;
  REAL *uprev = malloc(nb), *uk = malloc(nb), *q = malloc(nb), *vprev = malloc(nb), *vk = malloc(nb), *p = malloc(nb);
  REAL *w2 = malloc(nb), *w1 = qmr ? malloc(nb) : NULL;          /* QMR: w_{k-2}, w_{k-1}; BiLQ: d̅ (in w2) */
  REAL *dbar = w2;
  REAL *tb = MisI ? NULL : malloc(nb), *sb = NisI ? NULL : malloc(nb);
  const REAL *r0 = warm_start ? q : b;                            /* bilq.jl:152-161 */
  REAL *Mu = MisI ? uk : tb, *t = MisI ? q : tb, *Nv = NisI ? vk : sb, *s = NisI ? p : sb;
  if (warm_start) { SUF(spmv)(&A, x0, q); SUF(kaxpby)(n, 1, b, -1, q); }
  if (!MisI) { SUF(diagmul)(n, tb, Mdiag, r0, ldiv); r0 = tb; }
  SUF(kfill)(n, x, 0);
  REAL bNorm = SUF(knorm)(n, r0);
  if (history) PUSH(residuals, st->nres, bNorm);
  if (bNorm == 0) {
    st->niter = 0; st->solved = 1; st->inconsistent = 0;
    set_status(st, "x is a zero-residual solution");
    if (warm_start) SUF(kaxpy)(n, 1, x0, x);
    goto done;
  }
  int iter = 0;
  if (itmax == 0) itmax = 2 * n;
  REAL cb = SUF(kdot)(n, c, r0);                                  /* ⟨c,r₀⟩ */
  if (cb == 0) {
    st->niter = 0; st->solved = 0; st->inconsistent = 0;
    set_status(st, "Breakdown b\xe1\xb4\xb4" "c = 0");
    if (warm_start) SUF(kaxpy)(n, 1, x0, x);
    goto done;
  }
  REAL eps_ = atol + rtol * bNorm;
  REAL betak = SQRT(FABS(cb));
  REAL gammak = cb / betak;
  SUF(kfill)(n, vprev, 0);
  SUF(kfill)(n, uprev, 0);
  SUF(kdivcopy)(n, vk, r0, betak);
  SUF(kdivcopy)(n, uk, c, gammak);
  /* QMR state (qmr.jl:215-220) */
  REAL ck2 = 0, ck1 = 0, ck = 0, sk2 = 0, sk1 = 0, sk = 0, zetabar = betak, tau = 0;
  /* BiLQ state (bilq.jl:209-215) */
  REAL zeta1 = 0, eta1 = 0, etak = 0, zeta2 = 0, dbar1 = 0, dbark = 0, norm_vk = 0, rNorm_cg = 0;
  if (qmr) {
    SUF(kfill)(n, w2, 0);
    SUF(kfill)(n, w1, 0);
    tau = SUF(kdot)(n, vk, vk);
  } else {
    ck1 = ck = -1;
    SUF(kfill)(n, dbar, 0);
    zetabar = 0;
    norm_vk = bNorm / betak;
  }
  int solved = bNorm <= eps_, solved_cg = 0, breakdown = 0, tired = iter >= itmax, user_exit = 0, overtimed = 0;
  while (!(solved || solved_cg || tired || breakdown || user_exit || overtimed)) {
    iter = iter + 1;
    /* Lanczos biorthogonalization (bilq.jl:234-254, qmr.jl:238-258) */
    if (!NisI) SUF(diagmul)(n, Nv, Ndiag, vk, ldiv);
    SUF(spmv)(&A, Nv, t);
    if (!MisI) SUF(diagmul)(n, q, Mdiag, t, ldiv);
    if (!MisI) SUF(diagmul)(n, Mu, Mdiag, uk, ldiv);
    SUF(spmv)(&At, Mu, s);
    if (!NisI) SUF(diagmul)(n, p, Ndiag, s, ldiv);
    SUF(kaxpy)(n, -gammak, vprev, q);
    SUF(kaxpy)(n, -betak, uprev, p);
    REAL alphak = SUF(kdot)(n, uk, q);
    SUF(kaxpy)(n, -alphak, vk, q);
    SUF(kaxpy)(n, -alphak, uk, p);
    REAL pq = SUF(kdot)(n, p, q);
    REAL betak1 = SQRT(FABS(pq));
    REAL gammak1 = pq / betak1;
    REAL rNorm;
    if (qmr) {
      /* QR factorization of T_{k+1,k} (qmr.jl:275-312) */
      REAL epsk2 = 0, lbar1 = 0, l1 = 0, dbk = 0, deltak;
      if (iter >= 3) { epsk2 = sk2 * gammak; lbar1 = -ck2 * gammak; }
      if (iter >= 2) {
        if (iter == 2) lbar1 = gammak;
        l1 = ck1 * lbar1 + sk1 * alphak;
        dbk = sk1 * lbar1 - ck1 * alphak;
        sk2 = sk1; ck2 = ck1;
      }
      if (iter == 1) dbk = alphak;
      SUF(oracle_sym_givens)(dbk, betak1, &ck, &sk, &deltak);
      REAL zetak = ck * zetabar;
      REAL zetabar1 = sk * zetabar;
      sk1 = sk; ck1 = ck;
      /* w_k (qmr.jl:316-334) and x (:338) */
      REAL *wk = w1;
      if (iter == 1) { wk = w1; SUF(kdivcopy)(n, wk, vk, deltak); }
      if (iter == 2) { wk = w2; SUF(kaxpy)(n, -l1, w1, wk); SUF(kaxpy)(n, 1, vk, wk); SUF(kdiv)(n, wk, deltak); }
      if (iter >= 3) {
        SUF(kscal)(n, -epsk2, w2);
        wk = w2;
        SUF(kaxpy)(n, -l1, w1, wk); SUF(kaxpy)(n, 1, vk, wk); SUF(kdiv)(n, wk, deltak);
      }
      SUF(kaxpy)(n, zetak, wk, x);
      SUF(kcopy)(n, vprev, vk);
      SUF(kcopy)(n, uprev, uk);
      if (pq != 0) { SUF(kdivcopy)(n, vk, q, betak1); SUF(kdivcopy)(n, uk, p, gammak1); }
      REAL tau1 = tau + SUF(kdot)(n, vk, vk);
      rNorm = FABS(zetabar1) * SQRT(tau1);
      if (history) PUSH(residuals, st->nres, rNorm);
      if (iter >= 2) { REAL *tmp = w2; w2 = w1; w1 = tmp; }
      zetabar = zetabar1; betak = betak1; gammak = gammak1; tau = tau1;
      int resid_decrease_mach = (rNorm + (REAL)1 <= (REAL)1);
      if (callback) user_exit = callback(iter, cb_user) != 0;
      solved = (rNorm <= eps_) || resid_decrease_mach;
      tired = iter >= itmax;
      breakdown = !solved && (pq == 0);
    } else {
      /* LQ factorization of T_k (bilq.jl:265-285) */
      REAL delta1 = 0, l1 = 0, epsk2 = 0;
      if (iter == 1) {
        dbark = alphak;
      } else if (iter == 2) {
        SUF(oracle_sym_givens)(dbar1, gammak, &ck, &sk, &delta1);
        l1 = ck * betak + sk * alphak;
        dbark = sk * betak - ck * alphak;
      } else {
        SUF(oracle_sym_givens)(dbar1, gammak, &ck, &sk, &delta1);
        epsk2 = sk1 * betak;
        l1 = -ck1 * ck * betak + sk * alphak;
        dbark = -ck1 * sk * betak - ck * alphak;
      }
      /* ζ_{k-1}, η_k (bilq.jl:289-305) */
      if (iter == 1) etak = betak;
      if (iter == 2) { zeta1 = eta1 / delta1; etak = -l1 * zeta1; }
      if (iter >= 3) { zeta2 = zeta1; zeta1 = eta1 / delta1; etak = -epsk2 * zeta2 - l1 * zeta1; }
      /* directions and x (bilq.jl:310-322) */
      if (iter == 1) {
        SUF(kcopy)(n, dbar, vk);
      } else {
        SUF(kaxpy)(n, zeta1 * ck, dbar, x);
        SUF(kaxpy)(n, zeta1 * sk, vk, x);
        SUF(kaxpby)(n, -ck, vk, sk, dbar);
      }
      SUF(kcopy)(n, vprev, vk);
      SUF(kcopy)(n, uprev, uk);
      if (pq != 0) { SUF(kdivcopy)(n, vk, q, betak1); SUF(kdivcopy)(n, uk, p, gammak1); }
      REAL vv1 = SUF(kdot)(n, vprev, vk);
      REAL norm_vk1 = SUF(knorm)(n, vk);
      if (iter == 1) {
        rNorm = bNorm;
      } else {                                                    /* bilq.jl:342-345 */
        REAL mu = betak * (sk1 * zeta2 - ck1 * ck * zeta1) + alphak * sk * zeta1;
        REAL om = betak1 * sk * zeta1;
        REAL th = mu * om * vv1;
        rNorm = SQRT((mu * mu) * (norm_vk * norm_vk) + (om * om) * (norm_vk1 * norm_vk1) + 2 * th);
      }
      if (history) PUSH(residuals, st->nres, rNorm);
      int bicg_ok = transfer_to_bicg && (FABS(dbark) > EPS);
      if (bicg_ok) {                                              /* bilq.jl:351-355 */
        zetabar = etak / dbark;
        REAL rho = betak1 * (sk * zeta1 - ck * zetabar);
        rNorm_cg = FABS(rho) * norm_vk1;
      }
      sk1 = sk; ck1 = ck; eta1 = etak; gammak = gammak1; betak = betak1; dbar1 = dbark; norm_vk = norm_vk1;
      if (callback) user_exit = callback(iter, cb_user) != 0;
      solved = rNorm <= eps_;
      solved_cg = bicg_ok && (rNorm_cg <= eps_);
      tired = iter >= itmax;
      breakdown = !solved && !solved_cg && (pq == 0);
    }
    overtimed = timemax >= 0 && (oracle_now() - start) > timemax;
  }
  if (solved_cg) SUF(kaxpy)(n, zetabar, dbar, x);                 /* BiCG point (bilq.jl:380-382) */
  if (tired) set_status(st, "maximum number of iterations exceeded");
  if (breakdown) set_status(st, "Breakdown \xe2\x9f\xa8u\xe2\x82\x96\xe2\x82\x8a\xe2\x82\x81,v\xe2\x82\x96\xe2\x82\x8a\xe2\x82\x81\xe2\x9f\xa9 = 0");
  if (solved) set_status(st, qmr ? "solution good enough given atol and rtol" : "solution x\xe1\xb4\xb8 good enough given atol and rtol");
  if (solved_cg) set_status(st, "solution x\xe1\xb6\x9c good enough given atol and rtol");
  if (user_exit) set_status(st, "user-requested exit");
  if (overtimed) set_status(st, "time limit exceeded");
  if (!NisI) { SUF(kcopy)(n, sb, x); SUF(diagmul)(n, x, Ndiag, sb, ldiv); }
  if (warm_start) SUF(kaxpy)(n, 1, x0, x);
  st->niter = iter; st->solved = solved || solved_cg; st->inconsistent = 0;
done:
  free(uprev); free(uk); free(q); free(vprev); free(vk); free(p); free(w1); free(w2); free(tb); free(sb);
  return 0;
}


#undef PUSH
