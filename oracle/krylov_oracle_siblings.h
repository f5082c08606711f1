/*
 * krylov_oracle_siblings.h -- TEST INFRASTRUCTURE ONLY (same status as
 * krylov_oracle_impl.h, which must be included first).
 *
 * Sibling solvers of SURVEY.md section 8(f)-3: they reuse the hot-path kernels
 * unchanged, so the product runs them through the same primitives.  Literal
 * restatements, one statement per reference line:
 *   cgs!         src/cgs.jl:125-282
 *   cg_lanczos!  src/cg_lanczos.jl:110-264
 *   fom!         src/fom.jl:121-368
 *   fgmres!      src/fgmres.jl:128-388
 *   dqgmres!     src/dqgmres.jl:121-335
 *   diom!        src/diom.jl:121-332
 *   cr!          src/cr.jl:128-478  (trust region and linesearch included)
 * Parity pinning: checked against the properties the reference's own tests
 * assert (test/test_cgs.jl, test_cg_lanczos.jl, test_fom.jl, test_fgmres.jl:
 * residual <= atol + rtol*||b||, stats.solved, status strings) in
 * tests/test_oracle_kat.py; no Julia runtime exists here to compare iterates,
 * so iterate-level parity is "unpinned" exactly as for the four main solvers.
 */
#define PUSH(arr, cnt, v) do { if ((arr) && (cnt) < o->hist_cap) (arr)[(cnt)] = (v); (cnt)++; } while (0)

/* ============================ cgs!  (src/cgs.jl:125-282) ============================ */
static int SUF(cgs)(int variant, const SUF(problem) *P, const oracle_options *o, SUF(outputs) *out, oracle_stats *st) {
  const int n = P->n;
  const REAL *b = P->b, *c_in = P->c, *x0 = P->x0, *Mdiag = P->M, *Ndiag = P->N;
  REAL *x = out->x, *residuals = out->residuals;
  SUF(csr) A = {n, P->rowptr, P->colind, P->val};
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  int history = o->history, ldiv = o->ldiv, warm_start = (x0 != NULL);
  int MisI = (Mdiag == NULL), NisI = (Ndiag == NULL);
  const REAL *c = c_in ? c_in : b;                                /* cgs.jl:105 */
  REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol);
  int itmax = o->itmax;
  size_t nb = sizeof(REAL) * (size_t)n;
  REAL *r = malloc(nb), *u = malloc(nb), *p = malloc(nb), *q = malloc(nb), *ts = malloc(nb);
  REAL *vw = MisI ? NULL : malloc(nb), *yz = NisI ? NULL : malloc(nb);
  REAL *t = ts, *s = ts;                                          /* cgs.jl:150-155 */
  REAL *v = MisI ? t : vw, *w = MisI ? s : vw;
  REAL *y = NisI ? p : yz, *z = NisI ? u : yz;
  REAL *r0 = MisI ? r : ts;

  if (warm_start) { SUF(spmv)(&A, x0, r0); SUF(kaxpby)(n, 1, b, -1, r0); }
  else SUF(kcopy)(n, r0, b);
  SUF(kfill)(n, x, 0);
  if (!MisI) SUF(diagmul)(n, r, Mdiag, r0, ldiv);
  REAL rNorm = SUF(knorm)(n, r);
  if (history) PUSH(residuals, st->nres, rNorm);
  if (rNorm == 0) {
    st->niter = 0; st->solved = 1; st->inconsistent = 0;
    set_status(st, "x is a zero-residual solution");
    if (warm_start) SUF(kaxpy)(n, 1, x0, x);
    goto done;
  }
  REAL rho = SUF(kdot)(n, c, r);                                  /* cgs.jl:181 */
  if (rho == 0) {
    st->niter = 0; st->solved = 0; st->inconsistent = 0;
    set_status(st, "Breakdown b\xe1\xb4\xb4" "c = 0");
    if (warm_start) SUF(kaxpy)(n, 1, x0, x);
    goto done;
  }
  int iter = 0;
  if (itmax == 0) itmax = 2 * n;
  REAL eps_ = atol + rtol * rNorm;
  SUF(kcopy)(n, u, r);
  SUF(kcopy)(n, p, r);
  SUF(kfill)(n, q, 0);
  int solved = rNorm <= eps_, tired = iter >= itmax, breakdown = 0;
  while (!(solved || tired || breakdown)) {                       /* cgs.jl:210-252 */
    if (!NisI) SUF(diagmul)(n, y, Ndiag, p, ldiv);
    SUF(spmv)(&A, y, t);
    if (!MisI) SUF(diagmul)(n, v, Mdiag, t, ldiv);
    REAL sigma = SUF(kdot)(n, c, v);
    REAL alpha = rho / sigma;
    SUF(kcopy)(n, q, u);
    SUF(kaxpy)(n, -alpha, v, q);
    SUF(kaxpy)(n, 1, q, u);
    if (!NisI) SUF(diagmul)(n, z, Ndiag, u, ldiv);
    SUF(kaxpy)(n, alpha, z, x);
    SUF(spmv)(&A, z, s);
    if (!MisI) SUF(diagmul)(n, w, Mdiag, s, ldiv);
    SUF(kaxpy)(n, -alpha, w, r);
    REAL rho_next = SUF(kdot)(n, c, r);
    REAL beta = rho_next / rho;
    SUF(kcopy)(n, u, r);
    SUF(kaxpy)(n, beta, q, u);
    SUF(kaxpby)(n, 1, q, beta, p);
    SUF(kaxpby)(n, 1, u, beta, p);
    rho = rho_next;
    iter = iter + 1;
    rNorm = SUF(knorm)(n, r);
    if (history) PUSH(residuals, st->nres, rNorm);
    int resid_decrease_mach = (rNorm + (REAL)1 <= (REAL)1);
    solved = (rNorm <= eps_) || resid_decrease_mach;
    tired = iter >= itmax;
    breakdown = (alpha == 0 || isnan(alpha));
  }
  if (tired) set_status(st, "maximum number of iterations exceeded");
  if (breakdown) set_status(st, "breakdown \xce\xb1\xe2\x82\x96 == 0");
  if (solved) set_status(st, "solution good enough given atol and rtol");
  if (warm_start) SUF(kaxpy)(n, 1, x0, x);
  st->niter = iter; st->solved = solved; st->inconsistent = 0;
done:
  free(r); free(u); free(p); free(q); free(ts); free(vw); free(yz);
  return 0;
}

/* ======================= cg_lanczos!  (src/cg_lanczos.jl:110-264) ======================= */
/* LanczosStats: residuals, indefinite, Anorm (returned through out->Anorm), Acond stays NaN. */
static int SUF(cg_lanczos)(int variant, const SUF(problem) *P, const oracle_options *o, SUF(outputs) *out, oracle_stats *st) {
  const int n = P->n, check_curvature = o->check_curvature;
  const REAL *b = P->b, *x0 = P->x0, *Mdiag = P->M;
  REAL *x = out->x, *residuals = out->residuals, *Anorm = &out->Anorm;
  SUF(csr) A = {n, P->rowptr, P->colind, P->val};
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  int history = o->history, ldiv = o->ldiv, warm_start = (x0 != NULL);
  int MisI = (Mdiag == NULL);
  REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol);
  int itmax = o->itmax;
  size_t nb = sizeof(REAL) * (size_t)n;
  REAL *Mv = malloc(nb), *Mv_prev = malloc(nb), *p = malloc(nb), *Mv_next = malloc(nb);
  REAL *vbuf = MisI ? NULL : malloc(nb);
  REAL *v = MisI ? Mv : vbuf;                                     /* cg_lanczos.jl:138 */
  *Anorm = (REAL)NAN;

  SUF(kfill)(n, x, 0);
  if (warm_start) { SUF(spmv)(&A, x0, Mv); SUF(kaxpby)(n, 1, b, -1, Mv); }
  else SUF(kcopy)(n, Mv, b);
  if (!MisI) SUF(diagmul)(n, v, Mdiag, Mv, ldiv);
  REAL beta = (v == Mv) ? SUF(knorm)(n, v) : SQRT(SUF(kdot)(n, v, Mv));   /* knorm_elliptic, krylov_utils.jl:319 */
  REAL sigma = beta;
  REAL rNorm = sigma;
  if (history) PUSH(residuals, st->nres, rNorm);
  if (beta == 0) {
    st->niter = 0; st->solved = 1; *Anorm = 0; st->indefinite = 0;
    set_status(st, "x is a zero-residual solution");
    if (warm_start) SUF(kaxpy)(n, 1, x0, x);
    goto done;
  }
  SUF(kcopy)(n, p, v);
  SUF(kdiv)(n, v, beta);
  if (!MisI) SUF(kdiv)(n, Mv, beta);
  SUF(kcopy)(n, Mv_prev, Mv);
  int iter = 0;
  if (itmax == 0) itmax = 2 * n;
  REAL omega = 0, gamma = 1, Anorm2 = 0, beta_prev = 0;
  REAL eps_ = atol + rtol * rNorm;
  int indefinite = 0, solved = rNorm <= eps_, tired = iter >= itmax;
  while (!(solved || tired || (check_curvature && indefinite))) { /* cg_lanczos.jl:190-236 */
    SUF(spmv)(&A, v, Mv_next);
    REAL delta = SUF(kdot)(n, v, Mv_next);
    gamma = (REAL)1 / (delta - omega / gamma);
    indefinite |= (gamma <= 0);
    if (check_curvature && indefinite) continue;
    SUF(kaxpy)(n, -delta, Mv, Mv_next);
    if (iter > 0) {
      SUF(kaxpy)(n, -beta, Mv_prev, Mv_next);
      SUF(kcopy)(n, Mv_prev, Mv);
    }
    SUF(kcopy)(n, Mv, Mv_next);
    if (!MisI) SUF(diagmul)(n, v, Mdiag, Mv, ldiv);
    beta = (v == Mv) ? SUF(knorm)(n, v) : SQRT(SUF(kdot)(n, v, Mv));
    SUF(kdiv)(n, v, beta);
    if (!MisI) SUF(kdiv)(n, Mv, beta);
    Anorm2 += beta_prev * beta_prev + beta * beta + delta * delta;
    beta_prev = beta;
    SUF(kaxpy)(n, gamma, p, x);
    omega = beta * gamma;
    sigma = -omega * sigma;
    omega = omega * omega;
    SUF(kaxpby)(n, sigma, v, omega, p);
    rNorm = FABS(sigma);
    if (history) PUSH(residuals, st->nres, rNorm);
    iter = iter + 1;
    int resid_decrease_mach = (rNorm + (REAL)1 <= (REAL)1);
    solved = (rNorm <= eps_) || resid_decrease_mach;
    tired = iter >= itmax;
  }
  if (tired) set_status(st, "maximum number of iterations exceeded");
  if (check_curvature && indefinite) set_status(st, "negative curvature");
  if (solved) set_status(st, "solution good enough given atol and rtol");
  if (warm_start) SUF(kaxpy)(n, 1, x0, x);
  st->niter = iter; st->solved = solved; *Anorm = SQRT(Anorm2); st->indefinite = indefinite;
done:
  free(Mv); free(Mv_prev); free(p); free(Mv_next); free(vbuf);
  return 0;
}

/* ============================ fom!  (src/fom.jl:121-368) ============================ */
static int SUF(fom)(int variant, const SUF(problem) *P, const oracle_options *o, SUF(outputs) *out, oracle_stats *st) {
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
  if (mem > n) mem = n;                                           /* krylov_workspaces.jl:3067 */
  size_t nb = sizeof(REAL) * (size_t)n;
  REAL *w = malloc(nb);
  REAL *qbuf = MisI ? NULL : malloc(nb), *pbuf = NisI ? NULL : malloc(nb);
  REAL *dx = (restart || warm_start) ? calloc(n, sizeof(REAL)) : NULL;
  if (warm_start) SUF(kcopy)(n, dx, x0);
  int vcap = mem, lcap = mem, ucap = mem * (mem + 1) / 2;
  REAL **V = malloc(sizeof(REAL *) * vcap);
  for (int i = 0; i < vcap; i++) V[i] = malloc(nb);
  REAL *l = malloc(sizeof(REAL) * lcap), *zz = malloc(sizeof(REAL) * lcap), *U = malloc(sizeof(REAL) * ucap);
  int llen = mem, ulen = ucap, vlen = mem;                        /* Julia vector lengths (l and z grow together) */
  REAL *q = MisI ? w : qbuf, *r0 = MisI ? w : qbuf;               /* fom.jl:150-152 */
  REAL *xr = restart ? dx : x;

  SUF(kfill)(n, x, 0);
  if (warm_start) {
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
    if (warm_start) SUF(kaxpy)(n, 1, x0, x);
    goto done;
  }
  mem = llen;                                                     /* fom.jl:183 */
  int npass = 0, iter = 0, inner_iter = 0;
  if (itmax == 0) itmax = 2 * n;
  int inner_itmax = itmax;
  REAL btol = POW(EPS, (REAL)0.75);
  int breakdown = 0, solved = rNorm <= eps_, tired = iter >= itmax, inner_tired;

  while (!(solved || tired || breakdown)) {                       /* fom.jl:207 */
    int nr = 0;
    for (int i = 0; i < mem; i++) SUF(kfill)(n, V[i], 0);
    for (int i = 0; i < llen; i++) { l[i] = 0; zz[i] = 0; }
    for (int i = 0; i < ulen; i++) U[i] = 0;
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
    SUF(kdivcopy)(n, V[0], r0, rNorm);                            /* fom.jl:231 */
    npass = npass + 1;
    inner_iter = 0;
    inner_tired = 0;
    while (!(solved || inner_tired || breakdown)) {               /* fom.jl:237 */
      inner_iter = inner_iter + 1;
      if (!restart && (inner_iter > mem)) {                       /* fom.jl:243-251 */
        int newu = ulen + inner_iter;
        if (newu > ucap) { ucap = 2 * newu; U = realloc(U, sizeof(REAL) * ucap); }
        for (int i = ulen; i < newu; i++) U[i] = 0;
        ulen = newu;
        if (llen + 1 > lcap) { lcap = 2 * (llen + 1); l = realloc(l, sizeof(REAL) * lcap); zz = realloc(zz, sizeof(REAL) * lcap); }
        l[llen] = 0; zz[llen] = 0; llen++;
      }
      REAL *pv = V[inner_iter - 1];
      REAL *p = NisI ? pv : pbuf;
      if (!NisI) SUF(diagmul)(n, p, Ndiag, pv, ldiv);
      SUF(spmv)(&A, p, w);
      if (!MisI) SUF(diagmul)(n, q, Mdiag, w, ldiv);
      for (int i = 0; i < inner_iter; i++) {
        U[nr + i] = SUF(kdot)(n, V[i], q);
        SUF(kaxpy)(n, -U[nr + i], V[i], q);
      }
      if (reorth) {
        for (int i = 0; i < inner_iter; i++) {
          REAL Htmp = SUF(kdot)(n, V[i], q);
          U[nr + i] += Htmp;
          SUF(kaxpy)(n, -Htmp, V[i], q);
        }
      }
      REAL Hbis = SUF(knorm)(n, q);
      if (inner_iter >= 2) {                                      /* LU update, fom.jl:274-281 */
        for (int i = 2; i <= inner_iter; i++) U[nr + i - 1] = U[nr + i - 1] - l[i - 2] * U[nr + i - 2];
        zz[inner_iter - 1] = -l[inner_iter - 2] * zz[inner_iter - 2];
      }
      l[inner_iter - 1] = Hbis / U[nr + inner_iter - 1];
      rNorm = Hbis * FABS(zz[inner_iter - 1] / U[nr + inner_iter - 1]);
      if (history) PUSH(residuals, st->nres, rNorm);
      nr = nr + inner_iter;
      int resid_decrease_mach = (rNorm + (REAL)1 <= (REAL)1);
      breakdown = Hbis <= btol;
      solved = (rNorm <= eps_) || resid_decrease_mach;
      {
        int lim = restart ? (mem < inner_itmax ? mem : inner_itmax) : inner_itmax;
        inner_tired = inner_iter >= lim;
      }
      if (!(solved || inner_tired || breakdown)) {
        if (!restart && (inner_iter >= mem)) {
          if (vlen + 1 > vcap) { vcap = 2 * (vlen + 1); V = realloc(V, sizeof(REAL *) * vcap); }
          V[vlen++] = malloc(nb);
        }
        SUF(kdivcopy)(n, V[inner_iter], q, Hbis);
      }
    }
    REAL *y = zz;                                                 /* fom.jl:322-331 */
    for (int i = inner_iter; i >= 1; i--) {
      int pos = nr + i - inner_iter;
      for (int j = inner_iter; j >= i + 1; j--) {
        y[i - 1] = y[i - 1] - U[pos - 1] * y[j - 1];
        pos = pos - j + 1;
      }
      y[i - 1] = y[i - 1] / U[pos - 1];
    }
    for (int i = 0; i < inner_iter; i++) SUF(kaxpy)(n, y[i], V[i], xr);
    if (!NisI) { SUF(kcopy)(n, pbuf, xr); SUF(diagmul)(n, xr, Ndiag, pbuf, ldiv); }
    if (restart) SUF(kaxpy)(n, 1, xr, x);
    inner_itmax = inner_itmax - inner_iter;
    iter = iter + inner_iter;
    tired = iter >= itmax;
  }
  if (tired) set_status(st, "maximum number of iterations exceeded");
  if (breakdown) set_status(st, "inconsistent linear system");
  if (solved) set_status(st, "solution good enough given atol and rtol");
  if (warm_start && !restart) SUF(kaxpy)(n, 1, x0, x);
  st->niter = iter; st->solved = solved; st->inconsistent = !solved && breakdown;
done:
  for (int i = 0; i < vlen; i++) free(V[i]);
  free(V); free(l); free(zz); free(U); free(w); free(qbuf); free(pbuf); free(dx);
  return 0;
}

/* ========================== fgmres!  (src/fgmres.jl:128-388) ========================== */
/* Ndiag == NULL: N === I, and Z[k] <- V[k] by the unconditional mulorldiv! (fgmres.jl:262). */
static int SUF(fgmres)(int variant, const SUF(problem) *P, const oracle_options *o, SUF(outputs) *out, oracle_stats *st) {
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
  if (mem > n) mem = n;                                           /* krylov_workspaces.jl:2985 */
  size_t nb = sizeof(REAL) * (size_t)n;
  REAL *w = malloc(nb);
  REAL *qbuf = MisI ? NULL : malloc(nb);
  REAL *dx = (restart || warm_start) ? calloc(n, sizeof(REAL)) : NULL;
  if (warm_start) SUF(kcopy)(n, dx, x0);
  int vcap = mem, zvcap = mem, scap = mem, rcap = mem * (mem + 1) / 2, zcap = mem;
  REAL **V = malloc(sizeof(REAL *) * vcap), **Z = malloc(sizeof(REAL *) * zvcap);
  for (int i = 0; i < vcap; i++) { V[i] = malloc(nb); Z[i] = malloc(nb); }
  REAL *cc = malloc(sizeof(REAL) * scap), *ss = malloc(sizeof(REAL) * scap);
  REAL *zz = malloc(sizeof(REAL) * zcap), *R = malloc(sizeof(REAL) * rcap);
  int clen = mem, rlen = rcap, vlen = mem, zvlen = mem, zlen = mem;
  REAL *q = MisI ? w : qbuf, *r0 = MisI ? w : qbuf;
  REAL *xr = restart ? dx : x;

  SUF(kfill)(n, x, 0);
  if (warm_start) {
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
    if (warm_start) SUF(kaxpy)(n, 1, x0, x);
    goto done;
  }
  mem = clen;
  int npass = 0, iter = 0, inner_iter = 0;
  if (itmax == 0) itmax = 2 * n;
  int inner_itmax = itmax;
  REAL btol = POW(EPS, (REAL)0.75);
  int breakdown = 0, inconsistent = 0, solved = rNorm <= eps_, tired = iter >= itmax, inner_tired;

  while (!(solved || tired || breakdown)) {
    int nr = 0;
    for (int i = 0; i < mem; i++) { SUF(kfill)(n, V[i], 0); SUF(kfill)(n, Z[i], 0); }
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
    SUF(kdivcopy)(n, V[0], r0, rNorm);
    npass = npass + 1;
    inner_iter = 0;
    inner_tired = 0;
    while (!(solved || inner_tired || breakdown)) {
      inner_iter = inner_iter + 1;
      if (!restart && (inner_iter > mem)) {                       /* fgmres.jl:250-259 */
        int newr = rlen + inner_iter;
        if (newr > rcap) { rcap = 2 * newr; R = realloc(R, sizeof(REAL) * rcap); }
        for (int i = rlen; i < newr; i++) R[i] = 0;
        rlen = newr;
        if (clen + 1 > scap) { scap = 2 * (clen + 1); cc = realloc(cc, sizeof(REAL) * scap); ss = realloc(ss, sizeof(REAL) * scap); }
        ss[clen] = 0; cc[clen] = 0; clen++;
        if (zvlen + 1 > zvcap) { zvcap = 2 * (zvlen + 1); Z = realloc(Z, sizeof(REAL *) * zvcap); }
        Z[zvlen++] = malloc(nb);
      }
      REAL *zk = Z[inner_iter - 1];
      if (NisI) SUF(kcopy)(n, zk, V[inner_iter - 1]);             /* mul!(z, I, v) */
      else SUF(diagmul)(n, zk, Ndiag, V[inner_iter - 1], ldiv);
      SUF(spmv)(&A, zk, w);
      if (!MisI) SUF(diagmul)(n, q, Mdiag, w, ldiv);
      for (int i = 0; i < inner_iter; i++) {
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
      for (int i = 0; i < inner_iter - 1; i++) {
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
      if (!(solved || inner_tired || breakdown)) {
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
    REAL *y = zz;
    for (int i = inner_iter; i >= 1; i--) {
      int pos = nr + i - inner_iter;
      for (int j = inner_iter; j >= i + 1; j--) {
        y[i - 1] = y[i - 1] - R[pos - 1] * y[j - 1];
        pos = pos - j + 1;
      }
      if (FABS(R[pos - 1]) <= btol) { y[i - 1] = 0; inconsistent = 1; }
      else y[i - 1] = y[i - 1] / R[pos - 1];
    }
    for (int i = 0; i < inner_iter; i++) SUF(kaxpy)(n, y[i], Z[i], xr);   /* fgmres.jl:355-357 */
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
  for (int i = 0; i < zvlen; i++) free(Z[i]);
  free(V); free(Z); free(cc); free(ss); free(zz); free(R); free(w); free(qbuf); free(dx);
  return 0;
}

/* ========================== dqgmres!  (src/dqgmres.jl:121-335) ========================== */
static int SUF(dqgmres)(int variant, const SUF(problem) *prob, const oracle_options *o, SUF(outputs) *out, oracle_stats *st) {
  const int n = prob->n;
  const REAL *b = prob->b, *x0 = prob->x0, *Mdiag = prob->M, *Ndiag = prob->N;
  REAL *x = out->x, *residuals = out->residuals;
  SUF(csr) A = {n, prob->rowptr, prob->colind, prob->val};
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  int history = o->history, ldiv = o->ldiv, warm_start = (x0 != NULL), reorth = o->reorthogonalization;
  int MisI = (Mdiag == NULL), NisI = (Ndiag == NULL);
  REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol);
  int itmax = o->itmax;
  int mem = o->memory == 0 ? 20 : o->memory;
  if (mem > n) mem = n;                                           /* krylov_workspaces.jl:834 */
  size_t nb = sizeof(REAL) * (size_t)n;
  REAL *t = malloc(nb), *wbuf = MisI ? NULL : malloc(nb), *zbuf = NisI ? NULL : malloc(nb);
  REAL **P = malloc(sizeof(REAL *) * mem), **V = malloc(sizeof(REAL *) * mem);
  for (int i = 0; i < mem; i++) { P[i] = malloc(nb); V[i] = malloc(nb); }
  REAL *c = calloc(mem, sizeof(REAL)), *s = calloc(mem, sizeof(REAL)), *H = calloc(mem + 1, sizeof(REAL));
  REAL *w = MisI ? t : wbuf, *r0 = MisI ? t : wbuf;

  SUF(kfill)(n, x, 0);
  if (warm_start) { SUF(spmv)(&A, x0, t); SUF(kaxpby)(n, 1, b, -1, t); }
  else SUF(kcopy)(n, t, b);
  if (!MisI) SUF(diagmul)(n, r0, Mdiag, t, ldiv);
  REAL rNorm = SUF(knorm)(n, r0);
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
  for (int i = 0; i < mem; i++) { SUF(kfill)(n, V[i], 0); SUF(kfill)(n, P[i], 0); }
  REAL gamma_k = rNorm;
  SUF(kdivcopy)(n, V[0], r0, rNorm);
  int solved = rNorm <= eps_, tired = iter >= itmax;
  while (!(solved || tired)) {
    iter = iter + 1;
    int pos = (iter - 1) % mem + 1, next_pos = iter % mem + 1;    /* 1-based like the reference */
    REAL *z = NisI ? V[pos - 1] : zbuf;
    if (!NisI) SUF(diagmul)(n, z, Ndiag, V[pos - 1], ldiv);
    SUF(spmv)(&A, z, t);
    if (!MisI) SUF(diagmul)(n, w, Mdiag, t, ldiv);
    int lo = iter - mem + 1 > 1 ? iter - mem + 1 : 1;
    for (int i = lo; i <= iter; i++) {                            /* incomplete orthogonalization */
      int ipos = (i - 1) % mem + 1, diag = iter - i + 1;
      H[diag - 1] = SUF(kdot)(n, w, V[ipos - 1]);
      SUF(kaxpy)(n, -H[diag - 1], V[ipos - 1], w);
    }
    if (reorth) {
      for (int i = lo; i <= iter; i++) {
        int ipos = (i - 1) % mem + 1, diag = iter - i + 1;
        REAL Htmp = SUF(kdot)(n, w, V[ipos - 1]);
        H[diag - 1] += Htmp;
        SUF(kaxpy)(n, -Htmp, V[ipos - 1], w);
      }
    }
    REAL Haux = SUF(knorm)(n, w);
    if (Haux != 0) SUF(kdivcopy)(n, V[next_pos - 1], w, Haux);
    if (iter >= mem + 2) H[mem] = 0;                              /* H[mem+1] = 0 */
    int lo2 = iter - mem > 1 ? iter - mem : 1;
    for (int i = lo2; i <= iter - 1; i++) {                       /* previous rotations */
      int irot = (i - 1) % mem + 1, diag = iter - i, next_diag = diag + 1;
      REAL Htmp = c[irot - 1] * H[next_diag - 1] + s[irot - 1] * H[diag - 1];
      H[diag - 1] = s[irot - 1] * H[next_diag - 1] - c[irot - 1] * H[diag - 1];
      H[next_diag - 1] = Htmp;
    }
    SUF(oracle_sym_givens)(H[0], Haux, &c[pos - 1], &s[pos - 1], &H[0]);
    REAL gamma_next = s[pos - 1] * gamma_k;
    gamma_k = c[pos - 1] * gamma_k;
    for (int i = lo2; i <= iter - 1; i++) {                       /* direction p_k */
      int ipos = (i - 1) % mem + 1, diag = iter - i + 1;
      if (ipos == pos) SUF(kscal)(n, -H[diag - 1], P[pos - 1]);
      else SUF(kaxpy)(n, -H[diag - 1], P[ipos - 1], P[pos - 1]);
    }
    SUF(kaxpy)(n, 1, z, P[pos - 1]);
    SUF(kdiv)(n, P[pos - 1], H[0]);
    SUF(kaxpy)(n, gamma_k, P[pos - 1], x);
    rNorm = FABS(gamma_next);
    if (history) PUSH(residuals, st->nres, rNorm);
    gamma_k = gamma_next;
    int resid_decrease_mach = (rNorm + (REAL)1 <= (REAL)1);
    solved = (rNorm <= eps_) || resid_decrease_mach;
    tired = iter >= itmax;
  }
  if (solved) set_status(st, "solution good enough given atol and rtol");      /* dqgmres.jl:319-320: this order */
  if (tired) set_status(st, "maximum number of iterations exceeded");
  if (warm_start) SUF(kaxpy)(n, 1, x0, x);
  st->niter = iter; st->solved = solved; st->inconsistent = 0;
done:
  for (int i = 0; i < mem; i++) { free(P[i]); free(V[i]); }
  free(P); free(V); free(c); free(s); free(H); free(t); free(wbuf); free(zbuf);
  return 0;
}

/* ============================ diom!  (src/diom.jl:121-332) ============================ */
static int SUF(diom)(int variant, const SUF(problem) *prob, const oracle_options *o, SUF(outputs) *out, oracle_stats *st) {
  const int n = prob->n;
  const REAL *b = prob->b, *x0 = prob->x0, *Mdiag = prob->M, *Ndiag = prob->N;
  REAL *x = out->x, *residuals = out->residuals;
  SUF(csr) A = {n, prob->rowptr, prob->colind, prob->val};
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  int history = o->history, ldiv = o->ldiv, warm_start = (x0 != NULL), reorth = o->reorthogonalization;
  int MisI = (Mdiag == NULL), NisI = (Ndiag == NULL);
  REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol);
  int itmax = o->itmax;
  int mem = o->memory == 0 ? 20 : o->memory;
  if (mem > n) mem = n;                                           /* krylov_workspaces.jl:916 */
  if (mem < 2) { st->error = 20; set_status(st, "memory must be at least 2"); return 20; }   /* mod(., mem-1) */
  size_t nb = sizeof(REAL) * (size_t)n;
  REAL *t = malloc(nb), *wbuf = MisI ? NULL : malloc(nb), *zbuf = NisI ? NULL : malloc(nb);
  REAL **P = malloc(sizeof(REAL *) * (mem - 1)), **V = malloc(sizeof(REAL *) * mem);
  for (int i = 0; i < mem - 1; i++) P[i] = malloc(nb);
  for (int i = 0; i < mem; i++) V[i] = malloc(nb);
  REAL *L = calloc(mem - 1, sizeof(REAL)), *H = calloc(mem, sizeof(REAL));
  REAL *w = MisI ? t : wbuf, *r0 = MisI ? t : wbuf;

  SUF(kfill)(n, x, 0);
  if (warm_start) { SUF(spmv)(&A, x0, t); SUF(kaxpby)(n, 1, b, -1, t); }
  else SUF(kcopy)(n, t, b);
  if (!MisI) SUF(diagmul)(n, r0, Mdiag, t, ldiv);
  REAL rNorm = SUF(knorm)(n, r0);
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
  for (int i = 0; i < mem; i++) SUF(kfill)(n, V[i], 0);
  for (int i = 0; i < mem - 1; i++) SUF(kfill)(n, P[i], 0);
  REAL xi = rNorm;
  SUF(kdivcopy)(n, V[0], r0, rNorm);
  int solved = rNorm <= eps_, tired = iter >= itmax;
  while (!(solved || tired)) {
    iter = iter + 1;
    int pos = (iter - 1) % mem + 1, next_pos = iter % mem + 1;
    REAL *z = NisI ? V[pos - 1] : zbuf;
    if (!NisI) SUF(diagmul)(n, z, Ndiag, V[pos - 1], ldiv);
    SUF(spmv)(&A, z, t);
    if (!MisI) SUF(diagmul)(n, w, Mdiag, t, ldiv);
    int lo = iter - mem + 1 > 1 ? iter - mem + 1 : 1;
    for (int i = lo; i <= iter; i++) {
      int ipos = (i - 1) % mem + 1, diag = iter - i + 1;
      H[diag - 1] = SUF(kdot)(n, w, V[ipos - 1]);
      SUF(kaxpy)(n, -H[diag - 1], V[ipos - 1], w);
    }
    if (reorth) {
      for (int i = lo; i <= iter; i++) {
        int ipos = (i - 1) % mem + 1, diag = iter - i + 1;
        REAL Htmp = SUF(kdot)(n, w, V[ipos - 1]);
        H[diag - 1] += Htmp;
        SUF(kaxpy)(n, -Htmp, V[ipos - 1], w);
      }
    }
    REAL Haux = SUF(knorm)(n, w);
    if (Haux != 0) SUF(kdivcopy)(n, V[next_pos - 1], w, Haux);
    if (iter >= 2) {                                              /* LU of the band Hessenberg, diom.jl:262-272 */
      int lo3 = iter - mem + 2 > 2 ? iter - mem + 2 : 2;
      for (int i = lo3; i <= iter; i++) {
        int lpos = (i - 1) % (mem - 1) + 1, diag = iter - i + 1, next_diag = diag + 1;
        H[diag - 1] = H[diag - 1] - L[lpos - 1] * H[next_diag - 1];
        if (i == iter) xi = -L[lpos - 1] * xi;
      }
    }
    int next_lpos = iter % (mem - 1) + 1;
    L[next_lpos - 1] = Haux / H[0];
    int ppos = (iter - 1) % (mem - 1) + 1;
    for (int i = lo; i <= iter - 1; i++) {
      int ipos = (i - 1) % (mem - 1) + 1, diag = iter - i + 1;
      if (ipos == ppos) SUF(kscal)(n, -H[diag - 1], P[ppos - 1]);
      else SUF(kaxpy)(n, -H[diag - 1], P[ipos - 1], P[ppos - 1]);
    }
    SUF(kaxpy)(n, 1, z, P[ppos - 1]);
    SUF(kdiv)(n, P[ppos - 1], H[0]);
    SUF(kaxpy)(n, xi, P[ppos - 1], x);
    rNorm = Haux * FABS(xi / H[0]);
    if (history) PUSH(residuals, st->nres, rNorm);
    int resid_decrease_mach = (rNorm + (REAL)1 <= (REAL)1);
    solved = (rNorm <= eps_) || resid_decrease_mach;
    tired = iter >= itmax;
  }
  if (tired) set_status(st, "maximum number of iterations exceeded");
  if (solved) set_status(st, "solution good enough given atol and rtol");
  if (warm_start) SUF(kaxpy)(n, 1, x0, x);
  st->niter = iter; st->solved = solved; st->inconsistent = 0;
done:
  for (int i = 0; i < mem - 1; i++) free(P[i]);
  for (int i = 0; i < mem; i++) free(V[i]);
  free(P); free(V); free(L); free(H); free(t); free(wbuf); free(zbuf);
  return 0;
}

/* ============================== cr!  (src/cr.jl:128-478) ============================== */
/* o->gamma: NaN -> sqrt(eps(T)).  npc_dir: output (length n) when linesearch || radius > 0.
 * Aresiduals receives ||A r|| like stats.Aresiduals.  st->error: 1 linesearch&&radius>0, 2 warm_start&&linesearch,
 * 5 "Indefinite system and no trust region", 10+e to_boundary errors. */
static int SUF(cr)(int variant, const SUF(problem) *P, const oracle_options *o, SUF(outputs) *out, oracle_stats *st) {
  const int n = P->n;
  const REAL *b = P->b, *x0 = P->x0, *Mdiag = P->M;
  REAL *x = out->x, *residuals = out->residuals, *Aresiduals = out->Aresiduals, *npc_dir = out->npc_dir;
  SUF(csr) A = {n, P->rowptr, P->colind, P->val};
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  int history = o->history, ldiv = o->ldiv, warm_start = (x0 != NULL), linesearch = o->linesearch;
  REAL radius = (REAL)o->radius;
  REAL gam = isnan(o->gamma) ? SQRT(EPS) : (REAL)o->gamma;
  int MisI = (Mdiag == NULL);
  REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol);
  int itmax = o->itmax;
  int rc = 0;
  if (linesearch && radius > 0) { st->error = 1; return 1; }
  if (warm_start && linesearch) { st->error = 2; return 2; }
  size_t nb = sizeof(REAL) * (size_t)n;
  REAL *r = malloc(nb), *pbuf = malloc(nb), *qbuf = malloc(nb), *Ar = malloc(nb), *Mqbuf = MisI ? NULL : malloc(nb);
  REAL *p = pbuf, *q = qbuf;                                      /* rebound to r / Ar by the trust-region logic */
  REAL *Mq = MisI ? q : Mqbuf;

  SUF(kfill)(n, x, 0);
  if (warm_start) { SUF(spmv)(&A, x0, p); SUF(kaxpby)(n, 1, b, -1, p); }
  else SUF(kcopy)(n, p, b);
  if (MisI) SUF(kcopy)(n, r, p); else SUF(diagmul)(n, r, Mdiag, p, ldiv);
  REAL rNorm = SQRT(SUF(kdot)(n, r, p));                          /* knorm_elliptic(n, r, p): r !== p */
  if (history) PUSH(residuals, st->nres, rNorm);
  if (rNorm == 0) {
    st->niter = 0; st->solved = 1; st->inconsistent = 0;
    set_status(st, "x is a zero-residual solution");
    if (history) PUSH(Aresiduals, st->nAres, 0);
    if (warm_start) SUF(kaxpy)(n, 1, x0, x);
    goto done;
  }
  SUF(spmv)(&A, r, Ar);
  REAL rho = SUF(kdot)(n, r, Ar);
  if (rho == 0) {
    st->niter = 0; st->solved = 1; st->inconsistent = 0;
    set_status(st, "b is a zero-curvature direction");
    if (history) PUSH(Aresiduals, st->nAres, 0);
    if (linesearch || radius > 0) {
      SUF(kcopy)(n, x, p);
      SUF(kcopy)(n, npc_dir, p);
      st->npcCount = 1; st->indefinite = 1;
    }
    goto done;
  }
  SUF(kcopy)(n, p, r);
  SUF(kcopy)(n, q, Ar);
  int iter = 0;
  if (itmax == 0) itmax = 2 * n;
  REAL rNorm2 = rNorm * rNorm, pNorm = rNorm, pNorm2 = rNorm2, pr = rNorm2, abspr = pr, pAp = rho, abspAp = FABS(pAp);
  REAL xNorm = 0;
  REAL ArNorm = SUF(knorm)(n, Ar);
  if (history) PUSH(Aresiduals, st->nAres, ArNorm);
  REAL eps_ = atol + rtol * rNorm;
  int descent = pr > 0, solved = rNorm <= eps_, tired = iter >= itmax, on_boundary = 0, npcurv = 0;
  REAL sqeps = SQRT(EPS);

  while (!(solved || tired)) {
    REAL alpha = 0;
    if (linesearch) {
      int p_curv = pAp <= gam * pNorm * pNorm, r_curv = rho <= gam * rNorm * rNorm;
      if (p_curv || r_curv) {                                     /* cr.jl:233-262 */
        npcurv = 1;
        st->solved = 1; st->niter = iter; st->inconsistent = 0;
        set_status(st, "nonpositive curvature");
        st->indefinite = 1;
        if (iter == 0) {
          SUF(kcopy)(n, npc_dir, p);
          SUF(kcopy)(n, x, p);
          st->npcCount = 1;
        } else {
          if (r_curv) { SUF(kcopy)(n, npc_dir, r); st->npcCount += 1; }
          if (p_curv) { st->npcCount += 1; if (!r_curv) SUF(kcopy)(n, npc_dir, p); }
        }
        goto done;
      }
    } else if (pAp <= 0 && radius == 0) {
      st->error = 5; rc = 5; goto done;
    }
    if (!MisI) SUF(diagmul)(n, Mq, Mdiag, q, ldiv);
    if (radius > 0) {                                             /* cr.jl:268-373 */
      REAL xNorm2 = xNorm * xNorm, s1, s2, t1, t2, tr;
      int e = SUF(oracle_to_boundary)(n, x, p, Mq, radius, 0, xNorm2, pNorm2, NULL, 0, &s1, &s2);
      if (e) { st->error = 10 + e; rc = st->error; goto done; }
      t1 = s1 > s2 ? s1 : s2; t2 = s1 < s2 ? s1 : s2;
      e = SUF(oracle_to_boundary)(n, x, r, Mq, radius, 0, xNorm2, rNorm2, NULL, 0, &s1, &s2);
      if (e) { st->error = 10 + e; rc = st->error; goto done; }
      tr = s1 > s2 ? s1 : s2;
      if (abspAp <= gam * pNorm * SUF(knorm)(n, q)) {             /* p'Ap ~ 0 */
        npcurv = 1; st->indefinite = 1; st->npcCount = 1;
        SUF(kcopy)(n, npc_dir, p);
        if (abspr <= gam * pNorm * rNorm) {                       /* p'r ~ 0: p := r */
          p = r; q = Ar;
          if (rho > 0) alpha = tr < rNorm2 / rho ? tr : rNorm2 / rho;
          else { alpha = tr; if (iter > 0) { st->npcCount = 2; SUF(kcopy)(n, npc_dir, r); } }
        } else {
          alpha = descent ? t1 : t2;
          if (rho > 0) tr = tr < rNorm2 / rho ? tr : rNorm2 / rho;
          REAL Delta = -alpha * pr + tr * rNorm2 - tr * tr * rho / 2;
          if (Delta > 0) { p = r; q = Ar; alpha = tr; }
        }
      } else if (pAp > 0 && rho > 0) {
        alpha = rho / SUF(kdot)(n, q, Mq);
        if (alpha >= t1) { alpha = t1; on_boundary = 1; }
      } else if (pAp > 0 && rho < 0) {
        npcurv = 1; st->indefinite = 1; st->npcCount = 1;
        SUF(kcopy)(n, npc_dir, r);
        alpha = descent ? (t1 < pr / pAp ? t1 : pr / pAp) : (t2 > pr / pAp ? t2 : pr / pAp);
        REAL Delta = -alpha * pr + tr * rNorm2 + (alpha * alpha * pAp - tr * tr * rho) / 2;
        if (Delta > 0) { p = r; q = Ar; alpha = tr; }
      } else if (pAp < 0 && rho > 0) {
        npcurv = 1; st->indefinite = 1; st->npcCount = 1;
        SUF(kcopy)(n, npc_dir, p);
        alpha = descent ? t1 : t2;
        tr = tr < rNorm2 / rho ? tr : rNorm2 / rho;
        REAL Delta = -alpha * pr + tr * rNorm2 + (alpha * alpha * pAp - tr * tr * rho) / 2;
        if (Delta > 0) { p = r; q = Ar; alpha = tr; }
      } else if (pAp < 0 && rho < 0) {
        npcurv = 1; st->indefinite = 1; st->npcCount = 2;
        SUF(kcopy)(n, npc_dir, r);
        alpha = descent ? t1 : t2;
        REAL Delta = -alpha * pr + tr * rNorm2 + (alpha * alpha * pAp - tr * tr * rho) / 2;
        if (Delta > 0) { p = r; q = Ar; alpha = tr; }
      }
    } else if (radius == 0) {
      alpha = rho / SUF(kdot)(n, q, Mq);
    }
    SUF(kaxpy)(n, alpha, p, x);
    xNorm = SUF(knorm)(n, x);
    if (radius > 0) {                                             /* xNorm ≈ radius > 0  (isapprox, rtol = sqrt(eps)) */
      REAL mx = FABS(xNorm) > FABS(radius) ? FABS(xNorm) : FABS(radius);
      if (FABS(xNorm - radius) <= sqeps * mx) on_boundary = 1;
    }
    SUF(kaxpy)(n, -alpha, Mq, r);
    if (MisI) { rNorm2 = SUF(kdot)(n, r, r); rNorm = SQRT(rNorm2); }
    else {
      REAL omega = SQRT(alpha) * SQRT(rho);
      rNorm = SQRT(FABS(rNorm + omega)) * SQRT(FABS(rNorm - omega));
      rNorm2 = rNorm * rNorm;
    }
    if (history) PUSH(residuals, st->nres, rNorm);
    SUF(spmv)(&A, r, Ar);
    ArNorm = SUF(knorm)(n, Ar);
    if (history) PUSH(Aresiduals, st->nAres, ArNorm);
    iter = iter + 1;
    int resid_decrease_mach = (rNorm + (REAL)1 <= (REAL)1);
    int resid_decrease = (rNorm <= eps_) || resid_decrease_mach;
    solved = resid_decrease || npcurv || on_boundary;
    tired = iter >= itmax;
    if (solved || tired) continue;
    REAL rhobar = rho;
    rho = SUF(kdot)(n, r, Ar);
    REAL beta = rho / rhobar;
    SUF(kaxpby)(n, 1, r, beta, p);
    SUF(kaxpby)(n, 1, Ar, beta, q);
    pNorm2 = rNorm2 + 2 * beta * pr - 2 * beta * alpha * pAp + beta * beta * pNorm2;
    if (pNorm2 > sqeps) pNorm = SQRT(pNorm2);
    else if (FABS(pNorm2) <= sqeps) pNorm = 0;
    else {
      st->niter = iter; st->solved = solved; st->inconsistent = 0;
      set_status(st, "solver encountered numerical issues");
      if (warm_start) SUF(kaxpy)(n, 1, x0, x);
      goto done;
    }
    pr = rNorm2 + beta * pr - beta * alpha * pAp;
    abspr = FABS(pr);
    pAp = rho + beta * beta * pAp;
    abspAp = FABS(pAp);
    descent = pr > 0;
  }
  if (tired) set_status(st, "maximum number of iterations exceeded");
  if (solved) set_status(st, "solution good enough given atol and rtol");
  if (npcurv) set_status(st, "nonpositive curvature");
  if (on_boundary) set_status(st, "on trust-region boundary");
  if (warm_start) SUF(kaxpy)(n, 1, x0, x);
  st->niter = iter; st->solved = solved; st->inconsistent = 0;
done:
  free(r); free(pbuf); free(qbuf); free(Ar); free(Mqbuf);
  return rc;
}

#undef PUSH
