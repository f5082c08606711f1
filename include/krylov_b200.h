/*
 * krylov_b200.h -- C ABI of libkrylov_b200.so, the H100 (sm_90a) drop-in for
 * the inner-iteration path of Krylov.jl's cg!/gmres!/bicgstab!/minres!.
 *
 * PART 1 is binary-compatible with the reference's libkrylov
 * (interfaces/include/krylov.h @ Krylov.jl v0.10.8): same symbol names, same
 * struct layouts (interfaces/src/c_enums.jl:30-62), same enum values
 * (interfaces/scripts/solver_table.jl:5-42), same return-code conventions
 * (docs/src/interfaces/reference.md:144-170).  A C/Fortran program written
 * against krylov.h links against this library unchanged.
 *
 * PART 2 is additive: the CUDA device id, a device-resident CSR operator (so
 * the SpMV can be fused with the BLAS-1 work instead of crossing back into a
 * host callback once per product), statistics the reference keeps in
 * SimpleStats, and the flat per-primitive entry points a Julia `ccall` shim
 * binds (krylov.jl_b200/julia/KrylovB200.jl).
 *
 * Where vectors live: every workspace vector lives in HBM and every vector
 * operation runs on the GPU.  `device` only says where the CALLER's buffers
 * are: KRYLOV_CPU  -> b, c, x0, x and the matvec callbacks use host pointers
 * (the library stages them); KRYLOV_CUDA -> they are device pointers.
 * There is no CPU compute path: without a usable GPU, create returns -1.
 */
#ifndef KRYLOV_B200_H
#define KRYLOV_B200_H

#ifdef __cplusplus
extern "C" {
#endif

/* ======================= PART 1: the libkrylov ABI ======================= */

#ifndef KRYLOV_H /* allow inclusion next to the reference header */

#define KRYLOV_VERSION_MAJOR 0
#define KRYLOV_VERSION_MINOR 10
#define KRYLOV_VERSION_PATCH 8

/* element type of every vector (krylov.h:37-42) */
typedef enum { KRYLOV_FLOAT32 = 0, KRYLOV_FLOAT64 = 1, KRYLOV_COMPLEX32 = 2, KRYLOV_COMPLEX64 = 3 } KrylovDataType;

/* krylov.h:44-46 has KRYLOV_CPU only; KRYLOV_CUDA is this library's addition */
typedef enum { KRYLOV_CPU = 0, KRYLOV_CUDA = 1 } KrylovDeviceType;

/* positional, frozen (krylov.h:48-83).  Implemented here: CG, MINRES, GMRES, BICGSTAB (the hot path), the
 * siblings CR, DIOM, DQGMRES, FOM, FGMRES, CGS that run on the same kernels, CAR and MINARES on a symmetric operator
 * (CAR takes M, MINARES the shift `lambda` and no preconditioner; neither takes N), BILQ and QMR on a square operator and
 * its adjoint (matvec_At with matvec_A, or the transpose of an attached CSR operator; `c` is accepted, default b), the
 * adjoint pairs A x = b, A^T y = c of BILQR (square A) and TRILQR (A m x n: b and y have m entries, c and x have n),
 * which require c, take no preconditioner and return y through krylov_get_y, and the least-squares solvers LSQR, LSMR,
 * LSLQ, CGLS and CRLS on an m x n operator (b has m entries, x has n; matvec_A maps n -> m and matvec_At m -> n, or a
 * CSR operator of m rows and n columns is attached), and the least-norm solvers CRAIG, CRAIGMR and LNLQ on the same m x n
 * operators (min ||x|| subject to A x = b; x = A^T y, and y, m entries, is returned through krylov_get_y; `c` is
 * ignored), and the least-norm solvers CGNE and CRMR on the same operators, which return x only (krylov_get_y returns
 * -2), take `lambda` and one preconditioner, N, on the m-dimensional residual space (a solve given matvec_M or an M
 * diagonal is refused); every other value returns -2. */
typedef enum {
  KRYLOV_CG = 0, KRYLOV_CR = 1, KRYLOV_SYMMLQ = 2, KRYLOV_MINRES = 3, KRYLOV_MINRES_QLP = 4, KRYLOV_DIOM = 5,
  KRYLOV_DQGMRES = 6, KRYLOV_FOM = 7, KRYLOV_GMRES = 8, KRYLOV_FGMRES = 9, KRYLOV_BICGSTAB = 10, KRYLOV_CGS = 11,
  KRYLOV_BILQ = 12, KRYLOV_QMR = 13, KRYLOV_USYMLQ = 14, KRYLOV_USYMQR = 15, KRYLOV_TRICG = 16, KRYLOV_TRIMR = 17,
  KRYLOV_TRILQR = 18, KRYLOV_BILQR = 19, KRYLOV_LSLQ = 20, KRYLOV_LSQR = 21, KRYLOV_LSMR = 22, KRYLOV_USYMLQR = 23,
  KRYLOV_CGLS = 24, KRYLOV_CRLS = 25, KRYLOV_CGNE = 26, KRYLOV_CRMR = 27, KRYLOV_CRAIG = 28, KRYLOV_CRAIGMR = 29,
  KRYLOV_LNLQ = 30, KRYLOV_GPMR = 31, KRYLOV_CAR = 32, KRYLOV_MINARES = 33
} KrylovSolverType;

typedef enum { KRYLOV_BLOCK_GMRES = 0, KRYLOV_BLOCK_MINRES = 1 } KrylovBlockSolverType;

/* y = A x, y = A^H x, or y = M^-1 x.  The library owns x and y; they are
 * valid only during the call (reference.md:57-61). */
typedef void (*KrylovMatvec)(const void *x, void *y, void *userdata);
typedef void (*KrylovBlockMatvec)(const void *X, void *Y, int p, void *userdata);

/* construction-time options; 0 = solver default (memory 20, window 5) */
typedef struct {
  int memory;
  int window;
} KrylovWorkspaceOptions;

/* solve-time options; NaN / 0 = solver default (c_stores.jl:255-260) */
typedef struct {
  double atol;
  double rtol;
  int itmax;
  int verbose;
  double lambda;
  double tau;
  double nu;
  double timemax;
  double radius;
  int restart;
  int reorthogonalization;
  int linesearch;
} KrylovOptions;

#endif /* KRYLOV_H */

/* 0 ok | -1 error (message on stderr, *ws_out untouched) | -2 unknown/unsupported (solver, dtype) */
int krylov_workspace_create(KrylovSolverType solver, int m, int n, KrylovDataType dtype, KrylovDeviceType device,
                            const KrylovWorkspaceOptions *wopts, void **ws_out);
KrylovWorkspaceOptions krylov_default_workspace_options(void);
KrylovOptions krylov_default_options(void);
void krylov_get_version(int *major, int *minor, int *patch);
/* 0 ok | -1 error.  matvec_A may be NULL once a CSR operator is attached (part 2). */
int krylov_solve(void *ws, KrylovMatvec matvec_A, KrylovMatvec matvec_At, KrylovMatvec matvec_M, KrylovMatvec matvec_N,
                 const void *b, const void *c, void *userdata, const KrylovOptions *opts);
int krylov_get_x(void *ws, void *x, int n);
int krylov_get_y(void *ws, void *y, int m); /* BILQR, TRILQR, CRAIG, CRAIGMR, LNLQ: y (m entries); -2: single-solution solver */
int krylov_is_solved(void *ws);             /* 1 | 0 | -1 */
int krylov_niter(void *ws);
double krylov_elapsed_time(void *ws);
int krylov_warm_start(void *ws, const void *x0, int n);
/* BILQR, TRILQR: x0 (n entries) and y0 (m entries), -1 when the lengths differ; -2: single-solution solver.
 * krylov_warm_start on a BILQR / TRILQR workspace returns -1. */
int krylov_warm_start2(void *ws, const void *x0, const void *y0, int nx, int ny);
int krylov_workspace_free(void *ws); /* 0 | 1 if the handle is unknown (double free is safe) */

/* Block solvers (krylov.h:250-285): KRYLOV_BLOCK_GMRES is implemented (p <= 32, Float32 / Float64; the tall-skinny
 * panel products of Float64 p = 8 / 16 / 32 run on the FP64 tensor cores); KRYLOV_BLOCK_MINRES answers -2. */
int krylov_block_workspace_create(KrylovBlockSolverType solver, int m, int n, int p, KrylovDataType dtype,
                                  KrylovDeviceType device, const KrylovWorkspaceOptions *wopts, void **ws_out);
int krylov_block_solve(void *ws, KrylovBlockMatvec matvec_A, KrylovBlockMatvec matvec_M, KrylovBlockMatvec matvec_N,
                       const void *B, void *userdata, const KrylovOptions *opts);
int krylov_block_get_X(void *ws, void *X, int n, int p);
int krylov_block_is_solved(void *ws);
int krylov_block_niter(void *ws);
double krylov_block_elapsed_time(void *ws);
int krylov_block_warm_start(void *ws, const void *x0, int n, int p);
int krylov_block_workspace_free(void *ws);
/* Number of panel QR factorizations of this block workspace that left the fast path: a Gram matrix that is not
 * numerically positive definite (rank-deficient block of right-hand sides or Krylov block) makes CholQR2 impossible,
 * and that ONE panel is then factorized by LAPACK's Householder algorithm run as 4p passes of the panel kernels
 * (still on the device).  0 on well-posed blocks. */
long long krylov_b200_block_qr_fallbacks(void *ws);

/* ===================== PART 2: GPU-path additions (additive) ===================== */

/* Number of usable CUDA devices (0 when there is no GPU / no driver). */
int krylov_b200_device_count(void);
/* Device used by subsequently created workspaces (default: current device). */
int krylov_b200_set_device(int device);
/* Last error message of the calling thread ("" if none). */
const char *krylov_b200_last_error(void);

/* Attach a CSR matrix as the operator A of `ws`: replaces mul!(y, A, x) at
 * cg.jl:196, gmres.jl:257, bicgstab.jl:221,228, minres.jl:289.
 *   rowptr[n+1], colind[nnz], values[nnz] (element type = workspace dtype);
 *   least-squares and least-norm (CRAIG, CRAIGMR, LNLQ, CGNE, CRMR) workspaces: n is the number of rows (the workspace's m) and the
 *   columns are the workspace's n;
 *   TriLQR workspaces: n is the number of rows (the workspace's m) and the columns are the workspace's n;
 *   least-squares, least-norm, BiLQ, QMR, BiLQR and TriLQR workspaces: the library forms A^T once (host-side) on the first solve and keeps it
 *   until the operator changes;
 *   index_base 0|1, index_bytes 4|8 (Julia's SparseMatrixCSC{T,Int64} passes
 *   1 and 8 -- for a symmetric matrix its CSC arrays ARE the CSR arrays);
 *   location 0 = host arrays, 1 = device arrays.
 * The library keeps its own int32 / 0-based device copy. */
int krylov_b200_set_operator_csr(void *ws, int n, long long nnz, const void *rowptr, const void *colind,
                                 const void *values, int index_base, int index_bytes, int location);
/* Share the CSR operator already attached to `src` (no copy). */
int krylov_b200_share_operator(void *ws, void *src);
/* Attach a CSR object made by kb200_csr_create (not owned: keep it alive while `ws` uses it). */
int krylov_b200_attach_csr(void *ws, void *csr);
/* Diagonal preconditioner: which = 0 -> M, 1 -> N; d[n] holds the diagonal of
 * the operator the solver applies (P^-1 with the default ldiv=false). NULL detaches.
 * LSQR / LSMR / LSLQ / CRAIG / CRAIGMR / LNLQ: M acts on the data space (d[m]), N on the solution space (d[n]).  CGLS / CRLS: M acts on the
 * residual space (d[m]); they take no N (a solve with N attached or matvec_N given is refused).  CGNE / CRMR: N acts on
 * the residual space (d[m]); they take no M (a solve with M attached or matvec_M given is refused). */
int krylov_b200_set_preconditioner_diag(void *ws, int which, const void *d, int location);
/* Block-Jacobi preconditioner (docs/src/preconditioners.md:33,159): which = 0 -> M, 1 -> N; blocks[ceil(n/bs)][bs][bs]
 * (row-major dense diagonal blocks, 2 <= bs <= 8, element type = workspace dtype; a last block of n % bs rows uses
 * its leading part) of the operator the solver applies (P^-1 with the default ldiv = false; with ldiv = true the
 * blocks are P and their inverses, formed once here, are applied).  cg! with M block-diagonal runs the persistent
 * fused kernel (z = M r formed block by block in the r-update phase); every other solver applies it as one extra
 * kernel per product.  A diagonal set with krylov_b200_set_preconditioner_diag takes precedence.  NULL detaches.
 * A singular block is accepted (ldiv = false applies the blocks as given), but a solve with ldiv = true then returns
 * -1 and names the first singular block in krylov_b200_last_error, as the reference's factorization raises. */
int krylov_b200_set_preconditioner_blockdiag(void *ws, int which, int bs, const void *blocks, int location);

/* cg_lanczos! (src/cg_lanczos.jl) has no slot in the reference's KrylovSolverType; this value selects it in
 * krylov_workspace_create.  Options: M, check_curvature (KrylovB200Options), the common tolerances. */
#define KRYLOV_B200_CG_LANCZOS 100

/* ---- shift solvers: one Lanczos process for p shifted systems, p solutions ----
 * cg_lanczos_shift! (src/cg_lanczos_shift.jl): (A + σᵢ I) xᵢ = b, A square (symmetric), M on the n-space;
 * cgls_lanczos_shift! (src/cgls_lanczos_shift.jl): (AᵀA + σᵢ I) xᵢ = Aᵀb, A m x n (b: m entries, xᵢ: n), no M.
 * They have no slot in the reference's KrylovSolverType; these values select them in
 * krylov_b200_shift_workspace_create (-2 for another solver or a complex dtype, -1 for nshifts <= 0 or, for
 * CG-Lanczos-shift, m != n).  The handle is a third kind: krylov_b200_set_operator_csr, _attach_csr,
 * _share_operator, _set_preconditioner_diag / _blockdiag (M only: which = 1 is refused; CGLS-Lanczos-shift refuses any M
 * at solve time),
 * _set_options (history, ldiv, fused, callback, check_curvature), _get_stats, _launch_count and _stream accept it;
 * krylov_solve, krylov_get_x, krylov_get_y, the warm starts and row partitioning refuse it (-1, last_error).
 * krylov_b200_shift_solve: matvec_A (and matvec_At for CGLS-Lanczos-shift) may be NULL once a CSR operator is
 * attached; shifts[nshifts] (host doubles, rounded to the dtype).  Options: atol, rtol, itmax (0: 2n, or m + n for
 * CGLS-Lanczos-shift), timemax, verbose of KrylovOptions.  `shift` arguments are 0-based.
 * krylov_b200_shift_get_x copies x_shift (n entries) to host or device memory, following the workspace's device.
 * krylov_b200_shift_get_stats: any pointer may be NULL; status gets at most status_cap - 1 characters;
 * indefinite[nshifts] (CG-Lanczos-shift: γᵢ ≤ 0 met; 0 for CGLS-Lanczos-shift) and history_len[nshifts].
 * krylov_b200_shift_get_history copies shift's residual history (<= cap entries) and returns the count, or -1. */
#define KRYLOV_B200_CG_LANCZOS_SHIFT 101
#define KRYLOV_B200_CGLS_LANCZOS_SHIFT 102
int krylov_b200_shift_workspace_create(int solver, int m, int n, int nshifts, KrylovDataType dtype, KrylovDeviceType device,
                                       void **ws_out);
int krylov_b200_shift_workspace_free(void *ws); /* 0 | 1 if the handle is unknown */
int krylov_b200_shift_solve(void *ws, KrylovMatvec matvec_A, KrylovMatvec matvec_At, KrylovMatvec matvec_M, const void *b,
                            const double *shifts, void *userdata, const KrylovOptions *opts);
int krylov_b200_shift_get_x(void *ws, int shift, void *x, int n);
int krylov_b200_shift_get_stats(void *ws, int *niter, int *solved, double *timer, char *status, int status_cap,
                                int *indefinite, int *history_len);
int krylov_b200_shift_get_history(void *ws, int shift, double *out, int cap);

/* Extra solve-time switches not present in KrylovOptions. */
typedef struct {
  int history;        /* 1: record residual history (kwarg `history`)              */
  int ldiv;           /* 1: preconditioners are applied with ldiv! (kwarg `ldiv`)   */
  double etol;        /* MINRES; LNLQ: kwarg `utoly`; NaN -> sqrt(eps)                 */
  double conlim;      /* MINRES; NaN -> 1/sqrt(eps)                                 */
  int fused;          /* 1 (default): fused kernels when eligible (CG: one persistent cooperative launch per
                       * batch of iterations); 2: fused CG as two launches per iteration; 0: primitives */
  int batch;          /* fused CG: iterations enqueued per host poll; 0 -> default  */
  int (*callback)(void *ws, void *user); /* kwarg `callback`; nonzero return = stop */
  void *callback_user;
  int time_kernels;   /* fused CG: time the two phases of the iteration (see krylov_b200_get_kernel_times) */
  int check_curvature; /* CG-Lanczos: kwarg `check_curvature` (src/cg_lanczos.jl:94)                            */
  double cr_gamma;     /* CR: kwarg `γ` (src/cr.jl:112); NaN -> sqrt(eps)                                        */
  double axtol;        /* LSQR, LSMR: kwarg `axtol` (src/lsqr.jl:152); MINARES: kwarg `Artol`, the relative
                          tolerance on ||A r|| (src/minares.jl:99); NaN -> sqrt(eps)                                  */
  double btol;         /* LSQR, LSMR, LSLQ, CRAIG: kwarg `btol`; NaN -> sqrt(eps)                                 */
  double sigma;        /* LSLQ: kwarg `σ` (src/lslq.jl:178), Gauss-Radau error bounds when > 0; LNLQ: kwarg `σ`      */
  double utol;         /* LSLQ: kwarg `utol`; LNLQ: kwarg `utolx`; NaN -> sqrt(eps)                                  */
  int transfer_to_lsqr; /* LSLQ, CRAIG (acts when lambda > 0): 1 -> return the LSQR point (kwarg `transfer_to_lsqr`)  */
  int transfer_to_bicg; /* BiLQ, BiLQR: 1 (default) -> return the BiCG point when it converges first (kwarg `transfer_to_bicg`);
                          TriLQR: its kwarg `transfer_to_usymcg` (the USYMCG point), in the same field.
                          LNLQ: its kwarg `transfer_to_craig` (the CRAIG point), default 1 as the reference's `true`   */
} KrylovB200Options;
KrylovB200Options krylov_b200_default_options(void);
int krylov_b200_set_options(void *ws, const KrylovB200Options *opts);

/* SimpleStats (src/krylov_stats.jl:24-36) */
typedef struct {
  int niter;
  int solved;
  int inconsistent;
  int indefinite;
  int npcCount;
  int nresiduals;
  int nAresiduals;
  int nAcond;
  double allocation_timer;
  double timer;
  char status[96];
  double Anorm;       /* LanczosStats.Anorm (cg_lanczos!); NaN for the other solvers */
  int error_with_bnd;  /* LSLQStats (src/krylov_stats.jl:352-365), LNLQStats: the error bounds became complex */
  int nerr_lbnds;      /* LSLQ history lengths (krylov_b200_get_history which = 3, 4, 5); LNLQ: error_bnd_x and
                          error_bnd_y in nerr_lbnds / nerr_ubnds_lq (which = 3, 4)                              */
  int nerr_ubnds_lq;
  int nerr_ubnds_cg;
  int solved_primal;   /* AdjointStats (src/krylov_stats.jl:263-280) of BiLQR / TriLQR; `solved` = solved_primal && solved_dual */
  int solved_dual;
  int nresiduals_dual; /* length of residuals_dual (krylov_b200_get_history which = 6); residuals_primal is which = 0 */
} KrylovB200Stats;
int krylov_b200_get_stats(void *ws, KrylovB200Stats *out);
/* which: 0 residuals, 1 Aresiduals, 2 Acond; LSLQ: 3 err_lbnds, 4 err_ubnds_lq, 5 err_ubnds_cg; LNLQ: 3 error_bnd_x,
 * 4 error_bnd_y; BiLQR / TriLQR:
 * 0 residuals_primal, 6 residuals_dual.
 * Returns the number copied (<= cap) or -1. */
int krylov_b200_get_history(void *ws, int which, double *out, int cap);
/* Device pointer of a workspace vector by its reference field name
 * ("x","r","p","Ap","z","npc_dir","v","s","qd","r1","r2","w1","w2","y","w","dx","V1".."Vk"; LNLQ: "x", "Nv", "Aᴴu", "y", "w̄", "Mu", "Av", "u", "v", "q"; CRAIG / CRAIGMR: "y", "Nv",
 * "Mu", "Av", "Aᴴu", "u", "v", "w", CRAIG "w2", CRAIGMR "d", "w̄" and "q"; BiLQR / TriLQR: "y", "d̅",
 * "wₖ₋₃", "wₖ₋₂", "uₖ₋₁", "uₖ", "vₖ₋₁", "vₖ", "q", "p", "Δx", "Δy"; CGNE: "x", "p", "Aᴴz", "r", "q", "s", "z";
 * CRMR: "x", "p", "Aᴴr", "r", "q", "s", "Nq".  The fused CGNE path does not write "q" or "Aᴴz": they hold what the
 * last primitive-path solve left). */
int krylov_b200_get_vector(void *ws, const char *name, void **dev_ptr);
/* Average durations (ms) of the fused kernels measured with CUDA events on the workspace stream during the
 * last solve run with time_kernels = 1: out[0] = K1 (SpMV + p update + <p,Ap>), out[1] = K2 (x, r update + <r,r>),
 * out[2] = number of timed iterations. */
int krylov_b200_get_kernel_times(void *ws, double *out3);
/* Kernels launched so far through this workspace's stream. */
long long krylov_b200_launch_count(void *ws);
/* The CUDA stream (cudaStream_t) all of this workspace's work is ordered on.  It is a private NON-BLOCKING stream:
 * nothing orders it against the caller's streams implicitly.  STREAM CONTRACT for device-pointer inputs (KRYLOV_CUDA
 * workspaces: b, c, x0; location = 1 arrays of krylov_b200_set_operator_csr / set_preconditioner_diag): the data
 * must be complete when the call is made, OR the producer must be ordered before this stream with
 * krylov_b200_wait_stream (or cudaStreamWaitEvent on krylov_b200_stream(ws)).  Outputs need no care: every solve
 * returns after synchronising its stream. */
void *krylov_b200_stream(void *ws);
/* Make the workspace's stream wait for everything enqueued so far on `producer_stream` (a cudaStream_t; NULL = the
 * legacy default stream): records an event there and waits for it on krylov_b200_stream(ws).  Returns 0 / -1. */
int krylov_b200_wait_stream(void *ws, void *producer_stream);

/* ---- row-partitioned solves: one process per GPU, one workspace per process ----
 * The workspace is created with n = number of LOCAL rows; its CSR operator has
 * n rows and n + nhalo columns: column j < n is local, column n + h is the halo
 * entry h, owned by rank halo_rank[h] at offset halo_off[h] of that rank's local
 * vectors.  Peers' vectors are mapped with CUDA IPC: every rank calls dist_init,
 * dist_export (fills krylov_b200_dist_handle_bytes() bytes), the caller gathers
 * the blobs of all ranks in rank order (e.g. torch.distributed.all_gather) and
 * passes the concatenation to dist_import.  Afterwards krylov_solve on a CG
 * workspace runs the fused path with in-kernel NVLink halo loads and in-kernel
 * all-reduces of the dot products (csrc/dist.cuh).  All ranks must call
 * krylov_solve with the same options. */
int krylov_b200_dist_handle_bytes(void);
int krylov_b200_dist_init(void *ws, int rank, int world, int nhalo, const int *halo_rank, const int *halo_off);
/* Optional push mode (after dist_init, any time before the first solve): `ranges4` holds nranges (<= 4) quadruples
 * (first local row, count, peer rank, first slot in the peer's halo) describing which contiguous blocks of this
 * rank's rows each peer needs; nhalo_all[world] = every rank's halo length.  The producing kernels then store
 * those entries directly into the peers' halo buffers and nobody issues fine-grained P2P loads. */
int krylov_b200_dist_set_push(void *ws, int nranges, const int *ranges4, const int *nhalo_all);
/* Send list of the general x-halo exchange that precedes every y = A x of a distributed workspace (all four
 * solvers): entry e sends local row rows[e] to slot slots[e] of rank peers[e]'s halo.  nhalo_all[world] = every
 * rank's halo length, nglobal = global number of rows.  Call after dist_init and before dist_export/import. */
int krylov_b200_dist_set_sendlist(void *ws, int nsend, const int *rows, const int *peers, const int *slots,
                                  const int *nhalo_all, long long nglobal);
int krylov_b200_dist_export(void *ws, void *handles_out);
int krylov_b200_dist_import(void *ws, const void *all_handles);

/* ---- flat primitives: the k* wrappers of src/krylov_utils.jl:305-349 ----
 * dtype selects float/double; all pointers are device pointers; scalars by
 * value as double; results by pointer.  `ctx` comes from kb200_ctx_create. */
void *kb200_ctx_create(int device);
void kb200_ctx_destroy(void *ctx);
int kb200_sync(void *ctx);
void *kb200_alloc(long long bytes);
int kb200_free(void *p);
/* copies are complete when these return (the device data may be used on any stream right after kb200_h2d) */
int kb200_h2d(void *dst, const void *src, long long bytes);
int kb200_d2h(void *dst, const void *src, long long bytes);
int kb200_dot(void *ctx, int dtype, int n, const void *x, const void *y, double *result);
int kb200_nrm2(void *ctx, int dtype, int n, const void *x, double *result);
int kb200_axpy(void *ctx, int dtype, int n, double s, const void *x, void *y);
int kb200_axpby(void *ctx, int dtype, int n, double s, const void *x, double t, void *y);
int kb200_scal(void *ctx, int dtype, int n, double s, void *x);
int kb200_copy(void *ctx, int dtype, int n, void *y, const void *x);
int kb200_scalcopy(void *ctx, int dtype, int n, void *y, double s, const void *x);
int kb200_divcopy(void *ctx, int dtype, int n, void *y, const void *x, double s);
int kb200_fill(void *ctx, int dtype, int n, void *x, double v);
/* The fused primitives of the solvers' unfused path, for testing them directly.  dot2: *r1 = <a, b> and
 * *r2 = <u, v> in one pass (bicgstab's omega).  cg_prologue: x = 0, r = p = b and *gamma = <b, b> in one pass (cg with
 * x0 = 0 and M = I).  diagmul: y = d .* x, or y = x ./ d when ldiv is non-zero (a diagonal preconditioner). */
int kb200_dot2(void *ctx, int dtype, int n, const void *a, const void *b, const void *u, const void *v, double *r1,
               double *r2);
int kb200_cg_prologue(void *ctx, int dtype, int n, const void *b, void *x, void *r, void *p, double *gamma);
int kb200_diagmul(void *ctx, int dtype, int n, void *y, const void *d, const void *x, int ldiv);
/* The block-Jacobi kernels behind krylov_b200_set_preconditioner_blockdiag, on ceil(n / bs) dense bs x bs row-major
 * blocks (2 <= bs <= 8; a last block of n % bs rows uses its leading part).  blockdiag_mul: y = blockdiag(B_k) x,
 * each row summed left to right with every product rounded.  blockdiag_invert: inv[k] = B_k^-1 (Gauss-Jordan with
 * partial pivoting; the padding of the last block is zero); a singular block gets a zero inverse and sets *singular
 * (a device int) to 1, which is never cleared here. */
int kb200_blockdiag_mul(void *ctx, int dtype, int n, int bs, const void *blocks, const void *x, void *y);
int kb200_blockdiag_invert(void *ctx, int dtype, int n, int bs, const void *blocks, void *inv, int *singular);
/* CSR operator objects for the flat API (same arguments as set_operator_csr). */
void *kb200_csr_create(void *ctx, int dtype, int n, long long nnz, const void *rowptr, const void *colind,
                       const void *values, int index_base, int index_bytes, int location);
/* m x n CSR object (rectangular operators of LSQR / LSMR): rowptr[m+1], column indices < n. */
void *kb200_csr_create_rect(void *ctx, int dtype, int m, int n, long long nnz, const void *rowptr, const void *colind,
                            const void *values, int index_base, int index_bytes, int location);
void kb200_csr_destroy(void *csr);
/* Data formats either side of the path (SURVEY.md 8f-4).  kb200_csr_read_mtx: Matrix Market `matrix coordinate
 * {real|integer|pattern} {general|symmetric|skew-symmetric}` (what benchmark/benchmarks.jl:23-33 reads through
 * MatrixMarket.jl), duplicates summed, symmetric storage expanded; NULL on error (krylov_b200_last_error).
 * kb200_csr_transpose: a new object holding A^T (= A^H for the real types here, docs/src/matrix_free.md:36-44). */
void *kb200_csr_read_mtx(void *ctx, const char *path, int dtype);
void *kb200_csr_transpose(void *ctx, void *csr);
int kb200_csr_info(void *csr, int *n, long long *nnz);
/* rows, columns and nonzeros of a CSR object (square or rectangular); any pointer may be NULL */
int kb200_csr_shape(void *csr, int *m, int *n, long long *nnz);
/* rowptr[n+1], colind[nnz] (0-based int32), values[nnz] in the object's dtype; any pointer may be NULL */
int kb200_csr_download(void *ctx, void *csr, int *rowptr, int *colind, void *values);
/* Host-side pieces, callable without a GPU (they make no CUDA call): the Matrix Market parser behind
 * kb200_csr_read_mtx (pass NULL arrays to query n / nnz first) and the small dense algebra of the block path --
 * LAPACK-style Householder QR (householder!, src/block_krylov_utils.jl:201-208: Q m x k column-major in/out, R k x k,
 * compact = 1 keeps the reflectors), the Cholesky factor / inverse of a Gram matrix (1: not positive definite
 * enough for CholQR2), and the Householder-sign reconstruction from the top p x p block of an orthonormal factor. */
int kb200_mtx_read(const char *path, int *n, long long *nnz, int *rowptr, int *colind, double *values);
int kb200_host_householder(int m, int k, double *Q, double *R, double *tau, int compact);
int kb200_host_cholqr_factors(int p, const double *G, double *R, double *Rinv);
int kb200_host_householder_signs(int p, const double *top, double *s);
/* y = A x (x has the object's n columns, y its m rows).  variant: 0 auto, 1 row-per-thread LDG kernel, 2 TMA-staged kernel,
 * 3 the constant-coefficient encoding (forced only; -1 and last_error when the operator is not encoded, see kb200_csr_dict). */
int kb200_spmv_csr(void *ctx, void *csr, const void *x, void *y, int variant);
/* W = A X on row-major n x p device panels (the SpMM of block_gmres).  variant: 0 auto (what block_gmres runs),
 * 1 p-threads-per-row kernel, 2 TMA-staged (p in {2,4,8,16,32} and a fitting tile plan, else -1 and last_error).
 * Synchronises before returning. */
int kb200_spmm_csr(void *ctx, void *csr, int p, const void *X, void *Y, int variant);
/* One panel operation of a block workspace on device pointers, which may point into larger allocations (the
 * Householder fallback of the panel QR runs them on row ranges).  op 0: G = L^T Out (L = Next, or Out when Next is
 * NULL); 1: Out = beta Out + alpha In S; 2: op 1 then op 0 in one pass.  S, G: p x p column-major, device.
 * 1 <= rows <= the workspace's n.  path 0: the solver's own dispatch; 1 DMMA (Float64, p in {8,16,32}); 2 SIMT;
 * 3 SIMT with prefetch; 4 SIMT alternative lanes-per-row (p in {8,16}); 5 tiled generic (any p).  Unavailable
 * combinations return -1.  Synchronises before returning. */
int krylov_b200_block_panel_op(void *ws, int op, int path, int rows, double alpha, const void *In, const void *S,
                               double beta, void *Out, const void *Next, void *G);
/* staging plan of a CSR object: out[0]=ntiles out[1]=tile_cap out[2]=max_row out[3]=tma_ok out[4]=stages out[5]=grid out[6]=smem_bytes */
int kb200_csr_plan(void *csr, long long *out7);
/* constant-coefficient encoding of a square CSR object (every entry one of <= 8 (column - row, value) pairs, stored as one
 * mask byte per row; built when the operator is created unless KB200_CSR_DICT=0): 1 if encoded (*npairs = number of
 * pairs), 0 if not (*npairs = 0), -1 on a NULL object.  Fused CG runs its persistent kernel on the encoding. */
int kb200_csr_dict(void *csr, int *npairs);
/* Kernels launched so far through a flat-API context (kb200_ctx_create); -1 for NULL. */
long long kb200_ctx_launch_count(void *ctx);

/* ---- Krylov processes (src/krylov_processes.jl): the basis and the projected matrix of k steps ----
 * csr: the operator A (m x n; square for the Lanczos processes and Arnoldi).  csrT: A^T as a CSR object (n x m), or
 * NULL to have the call form it with kb200_csr_transpose and free it afterwards.  b (and c): device vectors in dtype,
 * which must be the CSR object's.  V, U: caller-allocated device outputs, column-major, k+1 columns, leading dimension
 * = the vector's length.  beta, gamma: host scalars; T, TH, L: host arrays of the reference's SparseMatrixCSC nzval
 * (3k-1 entries for T and TH, 2k+1 for L); H: host, dense (k+1) x k column-major.  flags: bit 0 allow_breakdown, bit 1
 * reorthogonalization (hermitian_lanczos: local, arnoldi: full; ignored by the others).
 * All k steps are enqueued on the context's stream with the coefficients kept on the device; the call reads them back
 * once and returns after synchronising the stream.  With csrT = NULL the call first forms A^T through the host (the
 * operator is copied down, transposed and uploaded again), so pass csrT to repeat calls on one operator at one
 * read-back each.  The coefficient block and scratch vectors are kept in the context between calls (grown on demand).  0 on success; -1 with krylov_b200_last_error on an exact breakdown
 * without allow_breakdown (the reference's message), k < 1, a shape or dtype mismatch, or a row-partitioned context;
 * -2 for a complex dtype.  With allow_breakdown, the column after a breakdown is zero, as kfill! leaves it; when
 * nonhermitian_lanczos meets c^T b == 0 its first columns V[:,1], U[:,1] are zero too (the reference leaves them
 * undefined). */
int kb200_hermitian_lanczos(void *ctx, void *csr, int k, int dtype, const void *b, void *V, double *beta, double *T, int flags);
int kb200_arnoldi(void *ctx, void *csr, int k, int dtype, const void *b, void *V, double *beta, double *H, int flags);
int kb200_golub_kahan(void *ctx, void *csr, void *csrT, int k, int dtype, const void *b, void *V, void *U, double *beta, double *L,
                      int flags);
int kb200_nonhermitian_lanczos(void *ctx, void *csr, void *csrT, int k, int dtype, const void *b, const void *c, void *V, void *U,
                               double *beta, double *gamma, double *T, double *TH, int flags);
int kb200_saunders_simon_yip(void *ctx, void *csr, void *csrT, int k, int dtype, const void *b, const void *c, void *V, void *U,
                             double *beta, double *gamma, double *T, double *TH, int flags);

#ifdef __cplusplus
}
#endif
#endif /* KRYLOV_B200_H */
