/*
 * krylov_oracle_block.h -- TEST INFRASTRUCTURE ONLY (include after krylov_oracle_impl.h).
 *
 * block_gmres!  (src/block_gmres.jl:110-359) restated for real element types, with the LAPACK calls of
 * src/block_krylov_utils.jl:192-208 (geqrf / orgqr / ormqr) restated as their unblocked reference algorithms
 * (dgeqr2 + dlarfg, dorg2r, dorm2r -- what LAPACK runs for panels of <= 128 columns, where dgeqrf does not block).
 * Panels are column-major n x p like Julia matrices.
 *
 * Parity pinning: the only functional reference test of block_gmres is interfaces/test/C/test_block.c (tridiagonal
 * system, ||X - Xtrue|| < 1e-6), which tests/test_oracle_kat.py restates; iterate-level parity is unpinned.
 */
#define PUSH(arr, cnt, v) do { if ((arr) && (cnt) < o->hist_cap) (arr)[(cnt)] = (v); (cnt)++; } while (0)

/* ---- small dense kernels, column-major with leading dimension ld ---- */
/* Householder reflector (dlarfg): on exit *alpha = beta, x = v(2:n), returns tau. */
static REAL SUF(larfg)(int n, REAL *alpha, REAL *x) {
  if (n <= 1) return 0;
  REAL xnorm = 0;
  for (int i = 0; i < n - 1; i++) xnorm += x[i] * x[i];
  xnorm = SQRT(xnorm);
  if (xnorm == 0) return 0;
  REAL a = *alpha;
  REAL beta = -COPYSIGN(SQRT(a * a + xnorm * xnorm), a);
  REAL tau = (beta - a) / beta;
  REAL scal = (REAL)1 / (a - beta);
  for (int i = 0; i < n - 1; i++) x[i] *= scal;
  *alpha = beta;
  return tau;
}
/* QR factorization A = Q R of an m x k panel (dgeqr2): R in the upper triangle, reflectors below, tau[k]. */
static void SUF(geqr2)(int m, int k, REAL *A, int ld, REAL *tau) {
  for (int j = 0; j < k && j < m; j++) {
    tau[j] = SUF(larfg)(m - j, &A[j + (size_t)j * ld], &A[(j + 1 < m ? j + 1 : j) + (size_t)j * ld]);
    if (j + 1 < k) {                                              /* apply H_j to A(j:m, j+1:k) from the left */
      REAL ajj = A[j + (size_t)j * ld];
      A[j + (size_t)j * ld] = 1;
      for (int c = j + 1; c < k; c++) {
        REAL w = 0;
        for (int i = j; i < m; i++) w += A[i + (size_t)j * ld] * A[i + (size_t)c * ld];
        w *= tau[j];
        for (int i = j; i < m; i++) A[i + (size_t)c * ld] -= w * A[i + (size_t)j * ld];
      }
      A[j + (size_t)j * ld] = ajj;
    }
  }
}
/* Form the m x k matrix Q with orthonormal columns from the reflectors (dorg2r). */
static void SUF(org2r)(int m, int k, REAL *A, int ld, const REAL *tau) {
  for (int j = k - 1; j >= 0; j--) {
    if (j + 1 < k) {                                              /* apply H_j to A(j:m, j+1:k) */
      A[j + (size_t)j * ld] = 1;
      for (int c = j + 1; c < k; c++) {
        REAL w = 0;
        for (int i = j; i < m; i++) w += A[i + (size_t)j * ld] * A[i + (size_t)c * ld];
        w *= tau[j];
        for (int i = j; i < m; i++) A[i + (size_t)c * ld] -= w * A[i + (size_t)j * ld];
      }
    }
    for (int i = j + 1; i < m; i++) A[i + (size_t)j * ld] = -tau[j] * A[i + (size_t)j * ld];
    A[j + (size_t)j * ld] = (REAL)1 - tau[j];
    for (int i = 0; i < j; i++) A[i + (size_t)j * ld] = 0;
  }
}
/* C <- Q^T C with Q = H_1 ... H_k held as reflectors in A (dorm2r, side 'L', trans 'T'); C is m x nc. */
static void SUF(orm2r_lt)(int m, int nc, int k, REAL *A, int lda, const REAL *tau, REAL *Cm, int ldc) {
  for (int j = 0; j < k; j++) {
    REAL ajj = A[j + (size_t)j * lda];
    A[j + (size_t)j * lda] = 1;
    for (int c = 0; c < nc; c++) {
      REAL w = 0;
      for (int i = j; i < m; i++) w += A[i + (size_t)j * lda] * Cm[i + (size_t)c * ldc];
      w *= tau[j];
      for (int i = j; i < m; i++) Cm[i + (size_t)c * ldc] -= w * A[i + (size_t)j * lda];
    }
    A[j + (size_t)j * lda] = ajj;
  }
}
/* householder!(Q, R, tau; compact) (src/block_krylov_utils.jl:201-208): R is k x k, zero-filled then upper triangle */
static void SUF(householder)(int m, int k, REAL *Q, REAL *R, REAL *tau, int compact) {
  for (int i = 0; i < k * k; i++) R[i] = 0;
  SUF(geqr2)(m, k, Q, m, tau);
  for (int j = 0; j < k; j++) for (int i = 0; i <= j; i++) R[i + j * k] = Q[i + (size_t)j * m];
  if (!compact) SUF(org2r)(m, k, Q, m, tau);
}
void SUF(oracle_householder)(int m, int k, REAL *Q, REAL *R, REAL *tau, int compact) { SUF(householder)(m, k, Q, R, tau, compact); }

static void SUF(spmm)(const SUF(csr) *A, int p, const REAL *X, REAL *Y) {
  for (int c = 0; c < p; c++) SUF(spmv)(A, X + (size_t)c * A->n, Y + (size_t)c * A->n);
}
static void SUF(diagmul_panel)(int n, int p, REAL *Y, const REAL *d, const REAL *X, int ldiv) {
  for (int c = 0; c < p; c++) SUF(diagmul)(n, Y + (size_t)c * n, d, X + (size_t)c * n, ldiv);
}
/* C(pxp) = V^T Q */
static void SUF(panel_tn)(int n, int p, const REAL *V, const REAL *Q, REAL *Cm) {
  for (int j = 0; j < p; j++)
    for (int i = 0; i < p; i++) Cm[i + j * p] = SUF(kdot)(n, V + (size_t)i * n, Q + (size_t)j * n);
}
/* Q = beta Q + alpha V S   (V n x p, S p x p) */
static void SUF(panel_nn)(int n, int p, REAL alpha, const REAL *V, const REAL *S, REAL beta, REAL *Q) {
  for (int j = 0; j < p; j++) {
    REAL *qj = Q + (size_t)j * n;
    for (int r = 0; r < n; r++) {
      REAL acc = 0;
      for (int i = 0; i < p; i++) acc += V[r + (size_t)i * n] * S[i + j * p];
      qj[r] = beta * qj[r] + alpha * acc;
    }
  }
}

/* ====================== block_gmres!  (src/block_gmres.jl:110-359) ====================== */
/* B, X0, X: n x p column-major.  memory: 0 -> 5 (block_gmres.jl:99), clipped to div(n,p). */
int SUF(oracle_block_gmres)(int n, int p, const int *rowptr, const int *colind, const REAL *val,
                            const REAL *B, const REAL *X0, const REAL *Mdiag, const REAL *Ndiag,
                            const oracle_options *o, REAL *X, REAL *residuals, oracle_stats *st) {
  SUF(csr) A = {n, rowptr, colind, val};
  memset(st, 0, sizeof(*st));
  set_status(st, "unknown");
  int history = o->history, ldiv = o->ldiv, warm_start = (X0 != NULL);
  int restart = o->restart, reorth = o->reorthogonalization;
  int MisI = (Mdiag == NULL), NisI = (Ndiag == NULL);
  REAL atol = SUF(tol)(o->atol), rtol = SUF(tol)(o->rtol);
  int itmax = o->itmax;
  int mem = o->memory == 0 ? 5 : o->memory;
  if (mem > n / p) mem = n / p;                                   /* block_krylov_workspaces.jl:138 */
  size_t np = (size_t)n * p, nb = sizeof(REAL) * np, pp = (size_t)p * p;
  REAL *W = malloc(nb), *Qbuf = MisI ? NULL : malloc(nb), *Pbuf = NisI ? NULL : malloc(nb);
  REAL *dX = (restart || warm_start) ? calloc(np, sizeof(REAL)) : NULL;
  if (warm_start) memcpy(dX, X0, nb);
  REAL *Cm = malloc(sizeof(REAL) * pp), *D = malloc(sizeof(REAL) * 2 * pp);
  int vlen = mem, rlen = mem * (mem + 1) / 2, hlen = mem, zlen = mem;
  int vcap = vlen, rcap = rlen, hcap = hlen, zcap = zlen;
  REAL **V = malloc(sizeof(REAL *) * vcap), **Z = malloc(sizeof(REAL *) * zcap);
  REAL **R = malloc(sizeof(REAL *) * rcap), **H = malloc(sizeof(REAL *) * hcap), **tau = malloc(sizeof(REAL *) * hcap);
  for (int i = 0; i < vlen; i++) V[i] = malloc(nb);
  for (int i = 0; i < zlen; i++) Z[i] = malloc(sizeof(REAL) * pp);
  for (int i = 0; i < rlen; i++) R[i] = malloc(sizeof(REAL) * pp);
  for (int i = 0; i < hlen; i++) { H[i] = malloc(sizeof(REAL) * 2 * pp); tau[i] = malloc(sizeof(REAL) * p); }
  REAL *Q = MisI ? W : Qbuf, *R0 = MisI ? W : Qbuf;
  REAL *Xr = restart ? dX : X;
  REAL *D1 = D, *D2 = D + p;                                       /* views of the 2p x p matrix D (ld = 2p) */
  int ldd = 2 * p;

  SUF(kfill)((int)np, X, 0);
  if (warm_start) {
    SUF(spmm)(&A, p, dX, W);
    for (size_t i = 0; i < np; i++) W[i] = B[i] - W[i];
    if (restart) for (size_t i = 0; i < np; i++) X[i] += dX[i];
  } else {
    memcpy(W, B, nb);
  }
  if (!MisI) SUF(diagmul_panel)(n, p, R0, Mdiag, W, ldiv);
  REAL RNorm = SUF(knorm)((int)np, R0);                           /* Frobenius norm */
  if (history) PUSH(residuals, st->nres, RNorm);
  REAL eps_ = atol + rtol * RNorm;
  mem = vlen;
  int npass = 0, iter = 0, inner_iter = 0;
  if (itmax == 0) itmax = 2 * (n / p);
  int inner_itmax = itmax;
  int solved = RNorm <= eps_, tired = iter >= itmax, inner_tired;

  while (!(solved || tired)) {
    int nr = 0;
    for (int i = 0; i < mem; i++) SUF(kfill)((int)np, V[i], 0);
    for (int i = 0; i < rlen; i++) for (size_t k = 0; k < pp; k++) R[i][k] = 0;
    for (int i = 0; i < zlen; i++) for (size_t k = 0; k < pp; k++) Z[i][k] = 0;
    if (restart) {
      SUF(kfill)((int)np, Xr, 0);
      if (npass >= 1) {
        SUF(spmm)(&A, p, X, W);
        for (size_t i = 0; i < np; i++) W[i] = B[i] - W[i];
        if (!MisI) SUF(diagmul_panel)(n, p, R0, Mdiag, W, ldiv);
      }
    }
    memcpy(V[0], R0, nb);
    SUF(householder)(n, p, V[0], Z[0], tau[0], 0);                /* Gamma and V_1 */
    npass = npass + 1;
    inner_iter = 0;
    inner_tired = 0;
    while (!(solved || inner_tired)) {
      inner_iter = inner_iter + 1;
      if (!restart && (inner_iter > mem)) {                       /* block_gmres.jl:231-239 */
        if (rlen + inner_iter > rcap) { rcap = 2 * (rlen + inner_iter); R = realloc(R, sizeof(REAL *) * rcap); }
        for (int i = 0; i < inner_iter; i++) R[rlen++] = calloc(pp, sizeof(REAL));
        if (hlen + 1 > hcap) { hcap = 2 * (hlen + 1); H = realloc(H, sizeof(REAL *) * hcap); tau = realloc(tau, sizeof(REAL *) * hcap); }
        H[hlen] = calloc(2 * pp, sizeof(REAL)); tau[hlen] = calloc(p, sizeof(REAL)); hlen++;
      }
      REAL *Vk = V[inner_iter - 1];
      REAL *P = NisI ? Vk : Pbuf;
      if (!NisI) SUF(diagmul_panel)(n, p, P, Ndiag, Vk, ldiv);
      SUF(spmm)(&A, p, P, W);
      if (!MisI) SUF(diagmul_panel)(n, p, Q, Mdiag, W, ldiv);
      for (int i = 0; i < inner_iter; i++) {                      /* block MGS */
        SUF(panel_tn)(n, p, V[i], Q, R[nr + i]);
        SUF(panel_nn)(n, p, -1, V[i], R[nr + i], 1, Q);
      }
      if (reorth) {
        for (int i = 0; i < inner_iter; i++) {
          SUF(panel_tn)(n, p, V[i], Q, Cm);
          SUF(panel_nn)(n, p, -1, V[i], Cm, 1, Q);
          for (size_t k = 0; k < pp; k++) R[nr + i][k] += Cm[k];
        }
      }
      SUF(householder)(n, p, Q, Cm, tau[inner_iter - 1], 0);      /* V_{k+1} in Q, Psi_{k+1,k} in C */
      for (int i = 0; i < inner_iter - 1; i++) {                  /* previous reflections, :268-274 */
        for (int c = 0; c < p; c++) for (int r = 0; r < p; r++) { D1[r + c * ldd] = R[nr + i][r + c * p]; D2[r + c * ldd] = R[nr + i + 1][r + c * p]; }
        SUF(orm2r_lt)(2 * p, p, p, H[i], 2 * p, tau[i], D, ldd);
        for (int c = 0; c < p; c++) for (int r = 0; r < p; r++) { R[nr + i][r + c * p] = D1[r + c * ldd]; R[nr + i + 1][r + c * p] = D2[r + c * ldd]; }
      }
      REAL *Hk = H[inner_iter - 1];
      for (int c = 0; c < p; c++) for (int r = 0; r < p; r++) { Hk[r + c * 2 * p] = R[nr + inner_iter - 1][r + c * p]; Hk[p + r + c * 2 * p] = Cm[r + c * p]; }
      SUF(householder)(2 * p, p, Hk, R[nr + inner_iter - 1], tau[inner_iter - 1], 1);
      for (int c = 0; c < p; c++) for (int r = 0; r < p; r++) { D1[r + c * ldd] = Z[inner_iter - 1][r + c * p]; D2[r + c * ldd] = 0; }
      SUF(orm2r_lt)(2 * p, p, p, Hk, 2 * p, tau[inner_iter - 1], D, ldd);
      for (int c = 0; c < p; c++) for (int r = 0; r < p; r++) Z[inner_iter - 1][r + c * p] = D1[r + c * ldd];
      for (int c = 0; c < p; c++) for (int r = 0; r < p; r++) Cm[r + c * p] = D2[r + c * ldd];
      RNorm = SUF(knorm)((int)pp, Cm);
      if (history) PUSH(residuals, st->nres, RNorm);
      nr = nr + inner_iter;
      solved = RNorm <= eps_;
      {
        int lim = restart ? (mem < inner_itmax ? mem : inner_itmax) : inner_itmax;
        inner_tired = inner_iter >= lim;
      }
      if (!(solved || inner_tired)) {
        if (!restart && (inner_iter >= mem)) {
          if (vlen + 1 > vcap) { vcap = 2 * (vlen + 1); V = realloc(V, sizeof(REAL *) * vcap); }
          V[vlen++] = malloc(nb);
          if (zlen + 1 > zcap) { zcap = 2 * (zlen + 1); Z = realloc(Z, sizeof(REAL *) * zcap); }
          Z[zlen++] = calloc(pp, sizeof(REAL));
        }
        memcpy(V[inner_iter], Q, nb);
        for (int c = 0; c < p; c++) for (int r = 0; r < p; r++) Z[inner_iter][r + c * p] = D2[r + c * ldd];
      }
    }
    REAL **Y = Z;                                                 /* block back substitution, :316-324 */
    for (int i = inner_iter; i >= 1; i--) {
      int pos = nr + i - inner_iter;
      for (int j = inner_iter; j >= i + 1; j--) {
        for (int c = 0; c < p; c++)                               /* Y_i <- Y_i - Psi_ij Y_j */
          for (int r = 0; r < p; r++) {
            REAL acc = 0;
            for (int k = 0; k < p; k++) acc += R[pos - 1][r + k * p] * Y[j - 1][k + c * p];
            Y[i - 1][r + c * p] -= acc;
          }
        pos = pos - j + 1;
      }
      for (int c = 0; c < p; c++)                                 /* ldiv!(UpperTriangular(R[pos]), Y_i) */
        for (int r = p - 1; r >= 0; r--) {
          REAL acc = Y[i - 1][r + c * p];
          for (int k = r + 1; k < p; k++) acc -= R[pos - 1][r + k * p] * Y[i - 1][k + c * p];
          Y[i - 1][r + c * p] = acc / R[pos - 1][r + r * p];
        }
    }
    for (int i = 0; i < inner_iter; i++) SUF(panel_nn)(n, p, 1, V[i], Y[i], 1, Xr);
    if (!NisI) { memcpy(Pbuf, Xr, nb); SUF(diagmul_panel)(n, p, Xr, Ndiag, Pbuf, ldiv); }
    if (restart) for (size_t i = 0; i < np; i++) X[i] += Xr[i];
    inner_itmax = inner_itmax - inner_iter;
    iter = iter + inner_iter;
    tired = iter >= itmax;
  }
  if (tired) set_status(st, "maximum number of iterations exceeded");
  if (solved) set_status(st, "solution good enough given atol and rtol");
  if (warm_start && !restart) for (size_t i = 0; i < np; i++) X[i] += dX[i];
  st->niter = iter; st->solved = solved;
  for (int i = 0; i < vlen; i++) free(V[i]);
  for (int i = 0; i < zlen; i++) free(Z[i]);
  for (int i = 0; i < rlen; i++) free(R[i]);
  for (int i = 0; i < hlen; i++) { free(H[i]); free(tau[i]); }
  free(V); free(Z); free(R); free(H); free(tau); free(W); free(Qbuf); free(Pbuf); free(dX); free(Cm); free(D);
  return 0;
}
#undef PUSH
