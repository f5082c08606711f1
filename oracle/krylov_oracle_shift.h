/*
 * krylov_oracle_shift.h -- TEST INFRASTRUCTURE ONLY (include after krylov_oracle_impl.h).
 *
 *   cg_lanczos_shift!    src/cg_lanczos_shift.jl:206-268   (A + σᵢ I) xᵢ = b,       i = 1 … p
 *   cgls_lanczos_shift!  src/cgls_lanczos_shift.jl:206-260 (AᵀA + σᵢ I) xᵢ = Aᵀb,  i = 1 … p
 *
 * One Lanczos process for all p systems; the per-shift recurrences in the reference's order: δ̂ᵢ, γᵢ (and, for CG,
 * `indefinite`) for every shift, then not_cv, then ωᵢ, σᵢ, xᵢ, pᵢ and rNormsᵢ for the active shifts only, a history
 * entry for the shifts active in that iteration, then not_cv again.  X (the solutions) is column-major n x p, the
 * histories are hist_cap entries per shift.  They have their own entry (they return p solutions), like block_gmres.
 *
 * Parity pinning: tests/test_oracle_shift.py restates test/test_cg_lanczos_shift.jl and
 * test/test_cgls_lanczos_shift.jl (each xᵢ against a direct solve, the `indefinite` flags, b = 0, M, callback).
 */
#define PUSH_SHIFT(i, v) do { if (hist && hist_len[i] < o->hist_cap) hist[(size_t)(i) * o->hist_cap + hist_len[i]] = (v); hist_len[i]++; } while (0)

/* variant 0: cg_lanczos_shift (square A, M: a diagonal or, with the precond_block knob, block-Jacobi; NULL = I);
 * variant 1: cgls_lanczos_shift (A m x n with Aᵀ in P->t*; M must be NULL: returns 1, st->error = 1). */
static int SUF(lanczos_shift)(int variant, const SUF(problem) *P, const REAL *shifts, int nshifts, const oracle_options *o,
                              REAL *X, REAL *hist, int *hist_len, int *indefinite, oracle_stats *st) {
  const int cgls = variant == 1, m = P->m, n = P->n, p = nshifts;
  const REAL *b = P->b, *Mdiag = P->M;
  SUF(csr) A = {m, P->rowptr, P->colind, P->val};
  SUF(csr) At = {n, P->trowptr, P->tcolind, P->tval};
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  for (int i = 0; i < p; i++) { hist_len[i] = 0; indefinite[i] = 0; }
  if (cgls && Mdiag) { st->error = 1; set_status(st, "Preconditioner `M` is not supported."); return 1; }
  const double t0 = oracle_now();
  const int history = o->history, ldiv = o->ldiv, check_curvature = cgls ? 0 : o->check_curvature;
  const int MisI = (Mdiag == NULL);
  REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol);
  int itmax = o->itmax;
  size_t nb = sizeof(REAL) * (size_t)n, mb = sizeof(REAL) * (size_t)m;
  /* CG: Mv, Mv_prev, Mv_next (v aliases Mv when M = I).  CGLS: v (n) and u_prev, u, u_next (m). */
  REAL *Mv = malloc(nb), *Mv_prev = cgls ? NULL : malloc(nb), *Mv_next = cgls ? NULL : malloc(nb);
  REAL *vbuf = MisI ? NULL : malloc(nb);
  REAL *u_prev = cgls ? malloc(mb) : NULL, *u = cgls ? malloc(mb) : NULL, *u_next = cgls ? malloc(mb) : NULL;
  REAL *v = MisI ? Mv : vbuf;
  REAL *Pd = malloc(nb * (size_t)p);
  REAL *sigma = malloc(sizeof(REAL) * p), *dhat = malloc(sizeof(REAL) * p), *omega = malloc(sizeof(REAL) * p);
  REAL *gamma = malloc(sizeof(REAL) * p), *rNorms = malloc(sizeof(REAL) * p);
  int *converged = malloc(sizeof(int) * p), *not_cv = malloc(sizeof(int) * p);
  REAL beta;

  for (int i = 0; i < p; i++) SUF(kfill)(n, X + (size_t)i * n, 0);
  if (cgls) {
    SUF(kcopy)(m, u, b);
    SUF(kfill)(m, u_prev, 0);
    SUF(spmv)(&At, u, v);
    beta = SUF(knorm)(n, v);
  } else {
    SUF(kcopy)(n, Mv, b);
    if (!MisI) SUF(diagmul)(n, v, Mdiag, Mv, ldiv);
    beta = MisI ? SUF(knorm)(n, v) : SQRT(SUF(kdot)(n, v, Mv));      /* knorm_elliptic */
  }
  for (int i = 0; i < p; i++) rNorms[i] = beta;
  if (history) for (int i = 0; i < p; i++) PUSH_SHIFT(i, rNorms[i]);
  if (beta == 0) {
    st->niter = 0; st->solved = 1;
    set_status(st, "x is a zero-residual solution");
    goto done;
  }
  for (int i = 0; i < p; i++) SUF(kcopy)(n, Pd + (size_t)i * n, v);
  SUF(kdiv)(n, v, beta);
  if (cgls) SUF(kdiv)(m, u, beta);
  else {
    if (!MisI) SUF(kdiv)(n, Mv, beta);
    SUF(kcopy)(n, Mv_prev, Mv);
  }
  REAL rho = 1;
  for (int i = 0; i < p; i++) { sigma[i] = beta; dhat[i] = 0; omega[i] = 0; gamma[i] = 1; }
  REAL eps_ = atol + rtol * beta;
  for (int i = 0; i < p; i++) { converged[i] = rNorms[i] <= eps_; not_cv[i] = !converged[i]; }
  int iter = 0;
  if (itmax == 0) itmax = cgls ? m + n : 2 * n;
  int solved = 1;
  for (int i = 0; i < p; i++) if (not_cv[i]) solved = 0;
  int tired = iter >= itmax, user_exit = 0, overtimed = 0;

  while (!(solved || tired || user_exit || overtimed)) {
    REAL delta;
    if (cgls) {                                                   /* cgls_lanczos_shift.jl:209-219 */
      SUF(spmv)(&A, v, u_next);
      delta = SUF(kdot)(m, u_next, u_next);
      SUF(kaxpy)(m, -delta, u, u_next);
      SUF(kaxpy)(m, -beta, u_prev, u_next);
      SUF(spmv)(&At, u_next, v);
      beta = SUF(knorm)(n, v);
      SUF(kdiv)(n, v, beta);
      SUF(kdiv)(m, u_next, beta);
      SUF(kcopy)(m, u_prev, u);
      SUF(kcopy)(m, u, u_next);
    } else {                                                      /* cg_lanczos_shift.jl:209-222 */
      SUF(spmv)(&A, v, Mv_next);
      delta = SUF(kdot)(n, v, Mv_next);
      SUF(kaxpy)(n, -delta, Mv, Mv_next);
      if (iter > 0) {
        SUF(kaxpy)(n, -beta, Mv_prev, Mv_next);
        SUF(kcopy)(n, Mv_prev, Mv);
      }
      SUF(kcopy)(n, Mv, Mv_next);
      if (!MisI) SUF(diagmul)(n, v, Mdiag, Mv, ldiv);
      beta = MisI ? SUF(knorm)(n, v) : SQRT(SUF(kdot)(n, v, Mv));
      SUF(kdiv)(n, v, beta);
      if (!MisI) SUF(kdiv)(n, Mv, beta);
      if (!MisI) rho = SUF(kdot)(n, v, v);
    }
    for (int i = 0; i < p; i++) {
      dhat[i] = delta + rho * shifts[i];
      gamma[i] = (REAL)1 / (dhat[i] - omega[i] / gamma[i]);
    }
    if (!cgls) for (int i = 0; i < p; i++) indefinite[i] |= gamma[i] <= 0;
    for (int i = 0; i < p; i++) {
      not_cv[i] = check_curvature ? !(converged[i] || indefinite[i]) : !converged[i];
      if (not_cv[i]) {
        REAL *xi = X + (size_t)i * n, *pi = Pd + (size_t)i * n;
        SUF(kaxpy)(n, gamma[i], pi, xi);
        omega[i] = beta * gamma[i];
        sigma[i] = sigma[i] * -omega[i];
        omega[i] = omega[i] * omega[i];
        SUF(kaxpby)(n, sigma[i], v, omega[i], pi);
        rNorms[i] = FABS(sigma[i]);
        converged[i] = rNorms[i] <= eps_;
      }
    }
    if (history) for (int i = 0; i < p; i++) if (not_cv[i]) PUSH_SHIFT(i, rNorms[i]);
    for (int i = 0; i < p; i++) not_cv[i] = check_curvature ? !(converged[i] || indefinite[i]) : !converged[i];
    iter = iter + 1;
    if (o->callback) user_exit = o->callback(iter, o->cb_user) != 0;
    solved = 1;
    for (int i = 0; i < p; i++) if (not_cv[i]) solved = 0;
    tired = iter >= itmax;
    overtimed = o->timemax >= 0 && oracle_now() - t0 > o->timemax;
  }
  if (tired) set_status(st, "maximum number of iterations exceeded");
  if (solved) set_status(st, "solution good enough given atol and rtol");
  if (user_exit) set_status(st, "user-requested exit");
  if (overtimed) set_status(st, "time limit exceeded");
  st->niter = iter; st->solved = solved;
done:
  free(Mv); free(Mv_prev); free(Mv_next); free(vbuf); free(u_prev); free(u); free(u_next); free(Pd);
  free(sigma); free(dhat); free(omega); free(gamma); free(rNorms); free(converged); free(not_cv);
  return 0;
}

/* The one entry of both shift solvers: name "cg_lanczos_shift" or "cgls_lanczos_shift"; -1 for another name. */
int SUF(oracle_lanczos_shift)(const char *name, const SUF(problem) *P, const REAL *shifts, int nshifts,
                              const oracle_options *o, REAL *X, REAL *hist, int *hist_len, int *indefinite,
                              oracle_stats *st) {
  const int variant = !strcmp(name, "cg_lanczos_shift") ? 0 : !strcmp(name, "cgls_lanczos_shift") ? 1 : -1;
  if (variant < 0) return -1;
  return SUF(lanczos_shift)(variant, P, shifts, nshifts, o, X, hist, hist_len, indefinite, st);
}
#undef PUSH_SHIFT
