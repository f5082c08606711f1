/*
 * krylov_oracle_adjoint.h -- TEST INFRASTRUCTURE ONLY (same status as krylov_oracle_impl.h, which must be included
 * first).  Literal restatement of bilqr! (src/bilqr.jl:115-484) and trilqr! (src/trilqr.jl:114-461) on the BLAS-1
 * wrappers of krylov_oracle_impl.h, instantiated by krylov_oracle_adjoint.c and loaded by oracle/adjoint_oracle.py.
 * Parity pinning: tests/test_oracle_adjoint.py (the reference's assertions of test/test_bilqr.jl and
 * test/test_trilqr.jl) and tests/golden/oracle_adjoint.json (frozen histories).
 */
#define PUSH(arr, cnt, v) do { if ((arr) && (cnt) < o->hist_cap) (arr)[(cnt)] = (v); (cnt)++; } while (0)

/* ============ bilqr! (src/bilqr.jl:115-484) and trilqr! (src/trilqr.jl:114-461) ============
 * tri != 0 selects TriLQR: A is m x n, b and y have m entries, c and x have n (BiLQR: m == n).  A^T is passed as its own
 * CSR (n rows, ascending row indices of A in each row).  x0 / y0: NULL (no warm start) or Δx / Δy.  The callback
 * (NULL: none) returns nonzero to stop; timemax < 0 means no limit.  Vectors are copied and swapped as written (kcopy!,
 * @kswap!).  Stats: solved = solved_primal && solved_dual; the dual solution goes to y, its history to sres. */
int SUF(oracle_adjoint)(int tri, int m, int n, const int *rowptr, const int *colind, const REAL *val,
                        const int *trowptr, const int *tcolind, const REAL *tval,
                        const REAL *b, const REAL *c, const REAL *x0, const REAL *y0,
                        int transfer, double timemax, oracle_iter_cb callback, void *cb_user,
                        const oracle_opts *o, REAL *x, REAL *t, REAL *rres, REAL *sres, int *nsres,
                        int *solved_primal_out, int *solved_dual_out, oracle_stats *st) {
  SUF(csr) A = {m, rowptr, colind, val}, At = {n, trowptr, tcolind, tval};
  const double start = oracle_now();
  memset(st, 0, sizeof(*st));
  *nsres = 0;
  set_status(st, "unknown");
  int history = o->history, warm_start = (x0 != NULL);
  REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol);
  int itmax = o->itmax;
  size_t nbm = sizeof(REAL) * (size_t)m, nbn = sizeof(REAL) * (size_t)n;
  /* v-space (m): v, q, w; u-space (n): u, p, d̅ */
  REAL *uprev = malloc(nbn), *uk = malloc(nbn), *p = malloc(nbn), *dbar = malloc(nbn);
  REAL *vprev = malloc(nbm), *vk = malloc(nbm), *q = malloc(nbm), *wk3 = malloc(nbm), *wk2 = malloc(nbm);
  const REAL *r0 = warm_start ? q : b, *s0 = warm_start ? p : c;
  if (warm_start) {
    SUF(spmv)(&A, x0, q); SUF(kaxpby)(m, 1, b, -1, q);
    SUF(spmv)(&At, y0, p); SUF(kaxpby)(n, 1, c, -1, p);
  }
  SUF(kfill)(n, x, 0);
  REAL bNorm = SUF(knorm)(m, r0);
  SUF(kfill)(m, t, 0);
  REAL cNorm = SUF(knorm)(n, s0);
  int iter = 0;
  if (itmax == 0) itmax = tri ? m + n : 2 * n;
  if (history) { PUSH(rres, st->nres, bNorm); PUSH(sres, *nsres, cNorm); }
  REAL epsL = atol + rtol * bNorm, epsQ = atol + rtol * cNorm;
  REAL xi = 0;
  int solved_lq = bNorm == 0, solved_lq_tol = 0, solved_lq_mach = 0;
  int solved_cg = 0, solved_cg_tol = 0, solved_cg_mach = 0;
  int solved_primal = solved_lq || solved_cg;
  int solved_qr_tol = 0, solved_qr_mach = 0, inconsistent = 0;
  int solved_dual = cNorm == 0;
  int tired = 0, breakdown = 0, user_exit = 0, overtimed = 0;
  REAL betak, gammak;
  if (tri) {
    betak = SUF(knorm)(m, r0);                                    /* trilqr.jl:172-173 */
    gammak = SUF(knorm)(n, s0);
  } else {
    REAL cb = SUF(kdot)(n, s0, r0);                               /* bilqr.jl:173-184 */
    if (cb == 0) {
      st->niter = 0;
      set_status(st, "Breakdown b\xe1\xb4\xb4" "c = 0");
      if (warm_start) { SUF(kaxpy)(n, 1, x0, x); SUF(kaxpy)(m, 1, y0, t); }
      *solved_primal_out = 0; *solved_dual_out = 0; st->solved = 0;
      goto done;
    }
    betak = SQRT(FABS(cb));
    gammak = cb / betak;
  }
  SUF(kfill)(m, vprev, 0);
  SUF(kfill)(n, uprev, 0);
  SUF(kdivcopy)(m, vk, r0, betak);
  SUF(kdivcopy)(n, uk, s0, gammak);
  REAL ck1 = -1, ck = -1, sk1 = 0, sk = 0;
  SUF(kfill)(n, dbar, 0);
  REAL zeta1 = 0, zetabar = 0, zeta2 = 0, etak = 0, eta1 = 0, dbar1 = 0, dbark = 0;
  REAL psibar1 = 0, psi1 = 0, psibar = 0;
  REAL norm_vk = bNorm / betak;
  REAL eps3 = 0, lam2 = 0;
  SUF(kfill)(m, wk3, 0);
  SUF(kfill)(m, wk2, 0);
  REAL tau = 0, rNorm_lq = 0, rNorm_cg = 0, sNorm = 0;
  tired = iter >= itmax;
  while (!((solved_primal && solved_dual) || tired || breakdown || user_exit || overtimed)) {
    iter = iter + 1;
    REAL alphak, betak1, gammak1, pq = 0;
    if (tri) {                                                    /* trilqr.jl:210-224 */
      SUF(spmv)(&A, uk, q);
      SUF(spmv)(&At, vk, p);
      if (iter >= 2) { SUF(kaxpy)(m, -gammak, vprev, q); SUF(kaxpy)(n, -betak, uprev, p); }
      alphak = SUF(kdot)(m, vk, q);
      SUF(kaxpy)(m, -alphak, vk, q);
      SUF(kaxpy)(n, -alphak, uk, p);
      betak1 = SUF(knorm)(m, q);
      gammak1 = SUF(knorm)(n, p);
    } else {                                                      /* bilqr.jl:227-240 */
      SUF(spmv)(&A, vk, q);
      SUF(spmv)(&At, uk, p);
      SUF(kaxpy)(n, -gammak, vprev, q);
      SUF(kaxpy)(n, -betak, uprev, p);
      alphak = SUF(kdot)(n, uk, q);
      SUF(kaxpy)(n, -alphak, vk, q);
      SUF(kaxpy)(n, -alphak, uk, p);
      pq = SUF(kdot)(n, p, q);
      betak1 = SQRT(FABS(pq));
      gammak1 = pq / betak1;
    }
    /* LQ factorization of T_k (bilqr.jl:251-271, trilqr.jl:235-255) */
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
    if (!solved_primal) {                                         /* bilqr.jl:273-348, trilqr.jl:257-324 */
      if (iter == 1) etak = betak;
      if (iter == 2) { eta1 = etak; zeta1 = eta1 / delta1; etak = -l1 * zeta1; }
      if (iter >= 3) { zeta2 = zeta1; eta1 = etak; zeta1 = eta1 / delta1; etak = -epsk2 * zeta2 - l1 * zeta1; }
      const REAL *a = tri ? uk : vk;
      if (iter == 1) {
        SUF(kcopy)(n, dbar, a);
      } else {
        SUF(kaxpy)(n, zeta1 * ck, dbar, x);
        SUF(kaxpy)(n, zeta1 * sk, a, x);
        SUF(kaxpby)(n, -ck, a, sk, dbar);
      }
      REAL norm_vk1 = 0;
      if (tri) {
        if (iter == 1) rNorm_lq = bNorm;
        else {
          REAL mu = betak * (sk1 * zeta2 - ck1 * ck * zeta1) + alphak * sk * zeta1;
          REAL om = betak1 * sk * zeta1;
          rNorm_lq = SQRT(mu * mu + om * om);
        }
      } else {
        REAL vv1 = SUF(kdot)(n, vk, q) / betak1;
        norm_vk1 = SUF(knorm)(n, q) / betak1;
        if (iter == 1) rNorm_lq = bNorm;
        else {
          REAL mu = betak * (sk1 * zeta2 - ck1 * ck * zeta1) + alphak * sk * zeta1;
          REAL om = betak1 * sk * zeta1;
          REAL th = mu * om * vv1;
          rNorm_lq = SQRT((mu * mu) * (norm_vk * norm_vk) + (om * om) * (norm_vk1 * norm_vk1) + 2 * th);
        }
        norm_vk = norm_vk1;
      }
      if (history) PUSH(rres, st->nres, rNorm_lq);
      int cg_ok = transfer && (FABS(dbark) > EPS);
      if (cg_ok) {
        zetabar = etak / dbark;
        REAL rho = betak1 * (sk * zeta1 - ck * zetabar);
        rNorm_cg = tri ? FABS(rho) : FABS(rho) * norm_vk1;
      }
      solved_lq_tol = rNorm_lq <= epsL;
      solved_lq_mach = rNorm_lq + (REAL)1 <= (REAL)1;
      solved_lq = solved_lq_tol || solved_lq_mach;
      solved_cg_tol = cg_ok && (rNorm_cg <= epsL);
      solved_cg_mach = cg_ok && (rNorm_cg + (REAL)1 <= (REAL)1);
      solved_cg = solved_cg_tol || solved_cg_mach;
      solved_primal = solved_lq || solved_cg;
    }
    if (!solved_dual) {                                           /* bilqr.jl:350-408, trilqr.jl:326-386 */
      if (iter == 1) psibar = gammak;
      else { psi1 = ck * psibar1; psibar = sk * psibar1; }
      const REAL *src = tri ? vprev : uprev;
      REAL *wk1 = NULL;
      if (iter == 2) { wk1 = wk2; SUF(kdivcopy)(m, wk1, src, delta1); }
      if (iter == 3) {
        wk1 = wk3;
        SUF(kaxpy)(m, 1, src, wk1); SUF(kaxpy)(m, -lam2, wk2, wk1); SUF(kdiv)(m, wk1, delta1);
      }
      if (iter >= 4) {
        SUF(kscal)(m, -eps3, wk3);
        wk1 = wk3;
        SUF(kaxpy)(m, 1, src, wk1); SUF(kaxpy)(m, -lam2, wk2, wk1); SUF(kdiv)(m, wk1, delta1);
      }
      if (iter >= 3) { REAL *tmp = wk3; wk3 = wk2; wk2 = tmp; }
      if (iter >= 2) SUF(kaxpy)(m, psi1, wk1, t);
      psibar1 = psibar;
      REAL AsNorm = 0;
      if (tri) {
        sNorm = FABS(psibar);
        AsNorm = FABS(psibar) * SQRT(dbark * dbark + (ck * betak1) * (ck * betak1));
        if (iter == 1) xi = atol + rtol * AsNorm;
      } else {
        tau = tau + SUF(kdot)(n, uk, uk);
        sNorm = FABS(psibar) * SQRT(tau);
      }
      if (history) PUSH(sres, *nsres, sNorm);
      solved_qr_tol = sNorm <= epsQ;
      solved_qr_mach = sNorm + (REAL)1 <= (REAL)1;
      inconsistent = tri && AsNorm <= xi;
      solved_dual = solved_qr_tol || solved_qr_mach || inconsistent;
    }
    SUF(kcopy)(m, vprev, vk);
    SUF(kcopy)(n, uprev, uk);
    if (tri) {
      if (betak1 != 0) SUF(kdivcopy)(m, vk, q, betak1);
      if (gammak1 != 0) SUF(kdivcopy)(n, uk, p, gammak1);
    } else if (pq != 0) {
      SUF(kdivcopy)(n, vk, q, betak1);
      SUF(kdivcopy)(n, uk, p, gammak1);
    }
    if (iter >= 3) eps3 = epsk2;
    if (iter >= 2) lam2 = l1;
    dbar1 = dbark; ck1 = ck; sk1 = sk; gammak = gammak1; betak = betak1;
    if (callback) user_exit = callback(iter, cb_user) != 0;
    tired = iter >= itmax;
    breakdown = !tri && !solved_lq && !solved_cg && (pq == 0);
    overtimed = timemax >= 0 && (oracle_now() - start) > timemax;
  }
  if (solved_cg) SUF(kaxpy)(n, zetabar, dbar, x);
  if (tired) set_status(st, "maximum number of iterations exceeded");
  if (breakdown) set_status(st, "Breakdown \xe2\x9f\xa8u\xe2\x82\x96\xe2\x82\x8a\xe2\x82\x81,v\xe2\x82\x96\xe2\x82\x8a\xe2\x82\x81\xe2\x9f\xa9 = 0");
  if (solved_lq_tol && !solved_dual) set_status(st, "Only the primal solution x\xe1\xb4\xb8 is good enough given atol and rtol");
  if (solved_cg_tol && !solved_dual) set_status(st, "Only the primal solution x\xe1\xb6\x9c is good enough given atol and rtol");
  if (!solved_primal && solved_qr_tol) set_status(st, "Only the dual solution t is good enough given atol and rtol");
  if (solved_lq_tol && solved_qr_tol) set_status(st, "Both primal and dual solutions (x\xe1\xb4\xb8, t) are good enough given atol and rtol");
  if (solved_cg_tol && solved_qr_tol) set_status(st, "Both primal and dual solutions (x\xe1\xb6\x9c, t) are good enough given atol and rtol");
  if (solved_lq_mach && !solved_dual) set_status(st, "Only found approximate zero-residual primal solution x\xe1\xb4\xb8");
  if (solved_cg_mach && !solved_dual) set_status(st, "Only found approximate zero-residual primal solution x\xe1\xb6\x9c");
  if (!solved_primal && solved_qr_mach) set_status(st, "Only found approximate zero-residual dual solution t");
  if (solved_lq_mach && solved_qr_mach) set_status(st, "Found approximate zero-residual primal and dual solutions (x\xe1\xb4\xb8, t)");
  if (solved_cg_mach && solved_qr_mach) set_status(st, "Found approximate zero-residual primal and dual solutions (x\xe1\xb6\x9c, t)");
  if (solved_lq_mach && solved_qr_tol)
    set_status(st, "Found approximate zero-residual primal solutions x\xe1\xb4\xb8 and a dual solution t good enough given atol and rtol");
  if (solved_cg_mach && solved_qr_tol)
    set_status(st, "Found approximate zero-residual primal solutions x\xe1\xb6\x9c and a dual solution t good enough given atol and rtol");
  if (solved_lq_tol && solved_qr_mach)
    set_status(st, "Found a primal solution x\xe1\xb4\xb8 good enough given atol and rtol and an approximate zero-residual dual solutions t");
  if (solved_cg_tol && solved_qr_mach)
    set_status(st, "Found a primal solution x\xe1\xb6\x9c good enough given atol and rtol and an approximate zero-residual dual solutions t");
  if (user_exit) set_status(st, "user-requested exit");
  if (overtimed) set_status(st, "time limit exceeded");
  if (warm_start) { SUF(kaxpy)(n, 1, x0, x); SUF(kaxpy)(m, 1, y0, t); }
  st->niter = iter; st->solved = solved_primal && solved_dual; st->inconsistent = 0;
  *solved_primal_out = solved_primal; *solved_dual_out = solved_dual;
done:
  free(uprev); free(uk); free(p); free(dbar); free(vprev); free(vk); free(q); free(wk3); free(wk2);
  return 0;
}

#undef PUSH
