/*
 * krylov_oracle_processes.h -- TEST INFRASTRUCTURE ONLY (same status as krylov_oracle_impl.h, which must be included
 * first).  Restatement of the Krylov processes of src/krylov_processes.jl (hermitian_lanczos, arnoldi, golub_kahan,
 * nonhermitian_lanczos, saunders_simon_yip), real case, written from the algorithms on the BLAS-1 wrappers of
 * krylov_oracle_impl.h.  Instantiated by krylov_oracle.c and loaded by oracle/processes_oracle.py.
 * V and U are column-major with leading dimension = the vector's length.  T, Th and L are the nzval arrays of the
 * reference's SparseMatrixCSC outputs (zeroed here first, like zeros(R, ...)); H is dense (k+1) x k column-major.
 * A^T is passed as its own CSR.  Return value: 0, or the breakdown kind (1-based, in the order the reference checks)
 * with *brk_iter set, at the first exact breakdown when allow_breakdown is 0 (the process stops there, as the reference
 * raises).  With allow_breakdown the column is zero-filled (kfill!) and the process goes on.  Where the reference
 * leaves V[:,1] and U[:,1] undefined (nonhermitian_lanczos with c'b == 0), they are zero-filled.
 * Parity pinning: tests/test_oracle_processes.py and tests/golden/oracle_processes.json.
 */
#define COL(M, ld, j) ((M) + (size_t)(ld) * (size_t)((j) - 1))   /* column j, 1-based */
#define BREAK(kind, it) do { if (!allow_breakdown) { *brk_iter = (it); return (kind); } } while (0)

/* hermitian_lanczos (src/krylov_processes.jl:28-103) */
int SUF(oracle_hermitian_lanczos)(int n, const int *rowptr, const int *colind, const REAL *val, const REAL *b, int k,
                                  int allow_breakdown, int reorthogonalization, REAL *V, REAL *beta, REAL *nzval, int *brk_iter) {
  SUF(csr) A = {n, rowptr, colind, val};
  SUF(kfill)(3 * k - 1, nzval, 0);
  *beta = 0;
  int pa = 0;                                   /* 0-based position of αᵢ in nzval */
  for (int i = 1; i <= k; i++) {
    REAL *vi = COL(V, n, i), *q = COL(V, n, i + 1);
    if (i == 1) {
      *beta = SUF(knorm)(n, b);
      if (*beta == 0) { BREAK(1, 0); SUF(kfill)(n, vi, 0); }
      else SUF(kdivcopy)(n, vi, b, *beta);
    }
    SUF(spmv)(&A, vi, q);
    if (i >= 2) {
      REAL *vprev = COL(V, n, i - 1);
      REAL bi = nzval[pa - 2];
      nzval[pa - 1] = bi;
      SUF(kaxpy)(n, -bi, vprev, q);
    }
    REAL alpha = SUF(kdot)(n, vi, q);
    SUF(kaxpy)(n, -alpha, vi, q);
    if (reorthogonalization) {
      if (i >= 2) {
        REAL *vprev = COL(V, n, i - 1);
        REAL btmp = SUF(kdot)(n, vprev, q);
        nzval[pa - 2] = nzval[pa - 2] + btmp;
        nzval[pa - 1] = nzval[pa - 1] + btmp;
        SUF(kaxpy)(n, -btmp, vprev, q);
      }
      REAL atmp = SUF(kdot)(n, vi, q);
      alpha = alpha + atmp;
      SUF(kaxpy)(n, -atmp, vi, q);
    }
    nzval[pa] = alpha;
    REAL bnext = SUF(knorm)(n, q);
    if (bnext == 0) { BREAK(2, i); SUF(kfill)(n, q, 0); }
    else SUF(kdivcopy)(n, q, q, bnext);
    nzval[pa + 1] = bnext;
    pa += 3;
  }
  return 0;
}

/* arnoldi (src/krylov_processes.jl:250-296), modified Gram-Schmidt */
int SUF(oracle_arnoldi)(int n, const int *rowptr, const int *colind, const REAL *val, const REAL *b, int k, int allow_breakdown,
                        int reorthogonalization, REAL *V, REAL *beta, REAL *H, int *brk_iter) {
  SUF(csr) A = {n, rowptr, colind, val};
  const size_t hk = (size_t)k + 1;
  SUF(kfill)((int)(hk * (size_t)k), H, 0);
  *beta = 0;
  for (int j = 1; j <= k; j++) {
    REAL *vj = COL(V, n, j), *q = COL(V, n, j + 1);
    if (j == 1) {
      *beta = SUF(knorm)(n, b);
      if (*beta == 0) { BREAK(1, 0); SUF(kfill)(n, vj, 0); }
      else SUF(kdivcopy)(n, vj, b, *beta);
    }
    SUF(spmv)(&A, vj, q);
    for (int i = 1; i <= j; i++) {
      REAL *hij = &H[(size_t)(i - 1) + (size_t)(j - 1) * hk];
      *hij = SUF(kdot)(n, COL(V, n, i), q);
      SUF(kaxpy)(n, -*hij, COL(V, n, i), q);
    }
    if (reorthogonalization) {
      for (int i = 1; i <= j; i++) {
        REAL *hij = &H[(size_t)(i - 1) + (size_t)(j - 1) * hk];
        REAL htmp = SUF(kdot)(n, COL(V, n, i), q);
        SUF(kaxpy)(n, -htmp, COL(V, n, i), q);
        *hij = *hij + htmp;
      }
    }
    REAL *hnext = &H[(size_t)j + (size_t)(j - 1) * hk];
    *hnext = SUF(knorm)(n, q);
    if (*hnext == 0) { BREAK(2, j); SUF(kfill)(n, q, 0); }
    else SUF(kdivcopy)(n, q, q, *hnext);
  }
  return 0;
}

/* golub_kahan (src/krylov_processes.jl:323-402): A is m x n, b has m entries; V is n x (k+1), U m x (k+1) */
int SUF(oracle_golub_kahan)(int m, int n, const int *rowptr, const int *colind, const REAL *val, const int *trowptr,
                            const int *tcolind, const REAL *tval, const REAL *b, int k, int allow_breakdown, REAL *V, REAL *U,
                            REAL *beta, REAL *nzval, int *brk_iter) {
  SUF(csr) A = {m, rowptr, colind, val}, At = {n, trowptr, tcolind, tval};
  SUF(kfill)(2 * k + 1, nzval, 0);
  *beta = 0;
  int pa = 0;
  for (int i = 1; i <= k; i++) {
    REAL *ui = COL(U, m, i), *vi = COL(V, n, i), *q = COL(U, m, i + 1), *p = COL(V, n, i + 1);
    if (i == 1) {
      *beta = SUF(knorm)(m, b);
      if (*beta == 0) { BREAK(1, 0); SUF(kfill)(m, ui, 0); }
      else SUF(kdivcopy)(m, ui, b, *beta);
      SUF(spmv)(&At, ui, vi);                                       /* wᵢ = vᵢ */
      REAL a1 = SUF(knorm)(n, vi);
      if (a1 == 0) { BREAK(2, 0); SUF(kfill)(n, vi, 0); }
      else SUF(kdivcopy)(n, vi, vi, a1);
      nzval[pa] = a1;
    }
    SUF(spmv)(&A, vi, q);
    REAL alpha = nzval[pa];
    SUF(kaxpy)(m, -alpha, ui, q);
    REAL bnext = SUF(knorm)(m, q);
    if (bnext == 0) { BREAK(3, i); SUF(kfill)(m, q, 0); }
    else SUF(kdivcopy)(m, q, q, bnext);
    SUF(spmv)(&At, q, p);
    SUF(kaxpy)(n, -bnext, vi, p);
    REAL anext = SUF(knorm)(n, p);
    if (anext == 0) { BREAK(4, i); SUF(kfill)(n, p, 0); }
    else SUF(kdivcopy)(n, p, p, anext);
    nzval[pa + 1] = bnext;
    nzval[pa + 2] = anext;
    pa += 2;
  }
  return 0;
}

/* nonhermitian_lanczos (src/krylov_processes.jl:133-224): square A, b and c of length n */
int SUF(oracle_nonhermitian_lanczos)(int n, const int *rowptr, const int *colind, const REAL *val, const int *trowptr,
                                     const int *tcolind, const REAL *tval, const REAL *b, const REAL *c, int k,
                                     int allow_breakdown, REAL *V, REAL *U, REAL *beta, REAL *gamma, REAL *T, REAL *Th,
                                     int *brk_iter) {
  SUF(csr) A = {n, rowptr, colind, val}, At = {n, trowptr, tcolind, tval};
  SUF(kfill)(3 * k - 1, T, 0);
  SUF(kfill)(3 * k - 1, Th, 0);
  *beta = 0; *gamma = 0;
  int pa = 0;
  for (int i = 1; i <= k; i++) {
    REAL *vi = COL(V, n, i), *ui = COL(U, n, i), *q = COL(V, n, i + 1), *p = COL(U, n, i + 1);
    if (i == 1) {
      REAL cb = SUF(kdot)(n, c, b);
      if (cb == 0) {
        BREAK(1, 0);
        SUF(kfill)(n, q, 0); SUF(kfill)(n, p, 0);
        SUF(kfill)(n, vi, 0); SUF(kfill)(n, ui, 0);                 /* undefined in the reference */
      } else {
        *beta = SQRT(FABS(cb));
        *gamma = cb / *beta;
        SUF(kdivcopy)(n, vi, b, *beta);
        SUF(kdivcopy)(n, ui, c, *gamma);
      }
    }
    SUF(spmv)(&A, vi, q);
    SUF(spmv)(&At, ui, p);
    if (i >= 2) {
      REAL bi = T[pa - 2], gi = T[pa - 1];
      SUF(kaxpy)(n, -gi, COL(V, n, i - 1), q);
      SUF(kaxpy)(n, -bi, COL(U, n, i - 1), p);
    }
    REAL alpha = SUF(kdot)(n, ui, q);
    T[pa] = alpha;
    Th[pa] = alpha;
    SUF(kaxpy)(n, -alpha, vi, q);
    SUF(kaxpy)(n, -alpha, ui, p);
    REAL pq = SUF(kdot)(n, p, q), bnext, gnext;
    if (pq == 0) {
      BREAK(2, i);
      bnext = 0; gnext = 0;
      SUF(kfill)(n, q, 0); SUF(kfill)(n, p, 0);
    } else {
      bnext = SQRT(FABS(pq));
      gnext = pq / bnext;
      SUF(kdivcopy)(n, q, q, bnext);
      SUF(kdivcopy)(n, p, p, gnext);
    }
    T[pa + 1] = bnext;
    Th[pa + 1] = gnext;
    if (i <= k - 1) { T[pa + 2] = gnext; Th[pa + 2] = bnext; }
    pa += 3;
  }
  return 0;
}

/* saunders_simon_yip (src/krylov_processes.jl:431-524): A is m x n, b has m entries, c n; V is m x (k+1), U n x (k+1) */
int SUF(oracle_saunders_simon_yip)(int m, int n, const int *rowptr, const int *colind, const REAL *val, const int *trowptr,
                                   const int *tcolind, const REAL *tval, const REAL *b, const REAL *c, int k,
                                   int allow_breakdown, REAL *V, REAL *U, REAL *beta, REAL *gamma, REAL *T, REAL *Th,
                                   int *brk_iter) {
  SUF(csr) A = {m, rowptr, colind, val}, At = {n, trowptr, tcolind, tval};
  SUF(kfill)(3 * k - 1, T, 0);
  SUF(kfill)(3 * k - 1, Th, 0);
  *beta = 0; *gamma = 0;
  int pa = 0;
  for (int i = 1; i <= k; i++) {
    REAL *vi = COL(V, m, i), *ui = COL(U, n, i), *q = COL(V, m, i + 1), *p = COL(U, n, i + 1);
    if (i == 1) {
      *beta = SUF(knorm)(m, b);
      if (*beta == 0) { BREAK(1, 0); SUF(kfill)(m, vi, 0); }
      else SUF(kdivcopy)(m, vi, b, *beta);
      *gamma = SUF(knorm)(n, c);
      if (*gamma == 0) { BREAK(2, 0); SUF(kfill)(n, ui, 0); }
      else SUF(kdivcopy)(n, ui, c, *gamma);
    }
    SUF(spmv)(&A, ui, q);
    SUF(spmv)(&At, vi, p);
    if (i >= 2) {
      REAL bi = T[pa - 2], gi = T[pa - 1];
      SUF(kaxpy)(m, -gi, COL(V, m, i - 1), q);
      SUF(kaxpy)(n, -bi, COL(U, n, i - 1), p);
    }
    REAL alpha = SUF(kdot)(m, vi, q);
    T[pa] = alpha;
    Th[pa] = alpha;
    SUF(kaxpy)(m, -alpha, vi, q);
    SUF(kaxpy)(n, -alpha, ui, p);
    REAL bnext = SUF(knorm)(m, q);
    if (bnext == 0) { BREAK(3, i); SUF(kfill)(m, q, 0); }
    else SUF(kdivcopy)(m, q, q, bnext);
    REAL gnext = SUF(knorm)(n, p);
    if (gnext == 0) { BREAK(4, i); SUF(kfill)(n, p, 0); }
    else SUF(kdivcopy)(n, p, p, gnext);
    T[pa + 1] = bnext;
    Th[pa + 1] = gnext;
    if (i <= k - 1) { T[pa + 2] = gnext; Th[pa + 2] = bnext; }
    pa += 3;
  }
  return 0;
}

#undef COL
#undef BREAK
