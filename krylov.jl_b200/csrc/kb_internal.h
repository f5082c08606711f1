// kb_internal.h -- internal C++ interfaces of libkrylov_b200.
//
// Layering (mirrors Krylov.jl's L1..L3, SURVEY.md section 1):
//   Ctx           one CUDA stream + reduction scratch + pinned scalar mailbox
//   blas1.cu      k* primitives on device vectors   (src/krylov_utils.jl:309-349)
//   spmv.cu       CSR operator: plain and TMA-staged SpMV (kmul!, krylov_utils.jl:305)
//   cg_fused.cu   two-launch CG iteration               (src/cg.jl:195-268)
//   fused_phases.cu  fused iteration phases of every solver family with a fused path except cg!, and their scalar
//                 read-back (one state struct per family in the workspace's device block)
//   solvers.cu    host control flow of cg!/bicgstab!/minres! and the one Arnoldi driver of gmres!/fom!/fgmres!
//   siblings.cu   cgs!, cg_lanczos!, dqgmres!, diom!, cr!, car!, minares! on the same kernels (SURVEY.md 8f-3)
//   solver_common.h  host helpers of the drivers, among them SolveRun: the callback / clock / exit protocol
//   block.cu      block_gmres! on row-major device panels (8f-2; block.h)
//   biorth.cu     host control flow of bilq!/qmr! (one Lanczos biorthogonalization driver; A and A^T)
//   adjoint.cu    host control flow of bilqr!/trilqr! (adjoint system pairs A x = b, A^T y = c; two solutions)
//   lsq.cu        host control flow of lsqr!/lsmr!/lslq!/cgls!/crls! and of the least-norm craig!/craigmr!/lnlq!/cgne!/crmr! on rectangular
//                 operators (primitive and fused paths)
//   mtx.cu        Matrix Market ingestion, transposed operator (8f-4; mtx.h)
//   capi.cu       the C ABI (include/krylov_b200.h)
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

#include "common.cuh"
#include "dist.cuh"

namespace kb {

// ---------------------------------------------------------------------------
// Execution context: everything a solve needs besides its vectors.
// ---------------------------------------------------------------------------
struct Ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  void* partials = nullptr;      // kMaxPartials * 4 doubles of reduction scratch
  unsigned* tickets = nullptr;   // 8 tickets (zero-initialised, self re-arming)
  void* dscal = nullptr;         // 16 device scalars (doubles) written by reductions: slot 0 the dots of blas1.cu,
                                 // slot 1 the SpMV's, slot 15 k_dist_sum (the fused passes use ws.fused_state)
  void* hscal = nullptr;         // pinned mirror of dscal
  long long launches = 0;        // kernels launched through this context (bench: gpu_launches)
  void* proc_scratch = nullptr;  // the Krylov processes' coefficient block and scratch vectors (processes.cu), kept
  size_t proc_scratch_bytes = 0; // from one call to the next and grown on demand; freed by destroy()
  DistComm* dcomm = nullptr;     // device-resident communicator of a row-partitioned solve (nullptr: single GPU)
  DistExchange* dex = nullptr;   // host-side plan of the general x-halo exchange (nullptr: single GPU)

  void init(int dev);
  void destroy();
  void sync() { KB_CUDA(cudaStreamSynchronize(stream)); }
};

template <class T> T* dev_alloc(size_t n);                // cudaMalloc, n elements (+ 64 B pad)
void dev_free(void* p);

// ---------------------------------------------------------------------------
// BLAS-1 on device vectors.  Scalars that solvers consume on the host are
// returned by value (one pinned read-back + stream sync), exactly like the
// reference's kdot/knorm; the *_dev variants leave the result in ctx.dscal[slot].
// ---------------------------------------------------------------------------
template <class T> T    k_dot(Ctx& c, int n, const T* x, const T* y);
template <class T> T    k_nrm2(Ctx& c, int n, const T* x);
template <class T> T    k_cg_prologue(Ctx& c, int n, const T* b, T* x, T* r, T* p);   // x = 0, r = p = b, returns <b, b>
template <class T> void k_dot2(Ctx& c, int n, const T* a, const T* b, const T* u, const T* v, T* r1, T* r2);
template <class T> void k_dot_dev(Ctx& c, int n, const T* x, const T* y, int slot);
template <class T> void k_axpy(Ctx& c, int n, T s, const T* x, T* y);                 // y += s x
template <class T> void k_axpby(Ctx& c, int n, T s, const T* x, T t, T* y);           // y = s x + t y
template <class T> void k_scal(Ctx& c, int n, T s, T* x);                             // x *= s
template <class T> void k_copy(Ctx& c, int n, T* y, const T* x);                      // y = x
template <class T> void k_scalcopy(Ctx& c, int n, T* y, T s, const T* x);             // y = s x
template <class T> void k_divcopy(Ctx& c, int n, T* y, const T* x, T s);              // y = x / s
template <class T> void k_fill(Ctx& c, int n, T* x, T v);
template <class T> void k_diagmul(Ctx& c, int n, T* y, const T* d, const T* x, bool ldiv);  // y = d.*x or x./d
template <class T> void k_blockdiag_mul(Ctx& c, int n, int bs, const T* blocks, const T* x, T* y);   // y = blockdiag(B_k) x
template <class T> void k_blockdiag_invert(Ctx& c, int n, int bs, const T* blocks, T* inv, int* singular);  // per-block inverse
// row-partitioned solves (no-ops on a single GPU)
double k_dist_sum(Ctx& c, double v);                                   // sum of a host scalar over all ranks
void dist_agree_on_exit(Ctx& c, bool& user_exit, bool& overtimed);     // OR the exit flags over the ranks
void dist_check_alive(Ctx& c);                                         // throws once a reduction has timed out
// A NaN scalar read back on a row-partitioned workspace may be the mark of a dead communicator (every reduction
// returns NaN from then on): raise at once instead of iterating on NaNs until itmax.
inline void dist_nan_guard(Ctx& c, double v) { if (c.dcomm && v != v) dist_check_alive(c); }

// ---------------------------------------------------------------------------
// CSR operator resident in HBM (int32 indices, 0-based, columns ascending).
// n rows; ncols columns (= n for square operators, the only kind the square solvers take).
// ---------------------------------------------------------------------------
constexpr int kTileRows = 256;   // rows per TMA-staged tile (= consumer threads per CTA)

template <class T>
struct Csr {
  int n = 0;
  int ncols = 0;
  long long nnz = 0;
  int* rowptr = nullptr;    // n+1 (+ pad)
  int* colind = nullptr;    // nnz (+ pad)
  T* val = nullptr;         // nnz (+ pad)
  // TMA staging plan (filled by plan()):
  int ntiles = 0;
  int tile_cap = 0;         // max nnz of any kTileRows-row tile
  int max_row = 0;          // longest row
  int max_col = -1;         // largest column index (validated against the number of columns when a solve starts)
  bool tma_ok = false;      // tile fits the shared-memory stage budget
  int stages = 0;           // pipeline depth chosen for tile_cap
  size_t smem_bytes = 0;    // dynamic smem of the staged kernels
  int grid = 0;             // persistent grid (multiple of the SM count)
  int ctas_per_sm = 0;      // resident CTAs per SM the ring was sized for
};

// Constant-coefficient encoding of a square CSR operator (DESIGN.md §2).  When every stored entry is one of at most
// kDictSlots (column - row, value) pairs, the pairs form an operator-wide dictionary sorted by offset (then by the
// value's bits) and each row is one byte: bit u set <=> the row holds pair u.  Because the columns of a row ascend,
// so do its offsets: the bit order is the summation order and the encoded row sums are bit-identical to the CSR ones.
// Kept OUT of Csr<T> (whose parameter block the existing kernels share) and passed by value to the kernels that
// read it, so offsets and values sit in the parameter bank.
constexpr int kDictSlots = 8;
template <class T>
struct CsrDict {
  int n = 0;
  int npairs = 0;                       // 0: not encoded (the operator keeps the CSR path only)
  int off[kDictSlots] = {};             // column - row of pair u, ascending
  T val[kDictSlots] = {};
  unsigned char* mask = nullptr;        // n bytes (device), allocated with the operator
};

// ncols < 0: square (ncols = n).  dict != nullptr: try to encode the operator (csr_plan).
template <class T> void csr_upload(Ctx& c, Csr<T>& A, int n, long long nnz, const void* rowptr, const void* colind,
                                   const T* val, int index_base, int index_bytes, bool on_device, int ncols = -1,
                                   CsrDict<T>* dict = nullptr);
template <class T> void csr_free(Csr<T>& A);
template <class T> void csr_dict_free(CsrDict<T>& D);
// dict != nullptr: also build the encoding when the operator qualifies (KB200_CSR_DICT=0 disables it)
template <class T> void csr_plan(Ctx& c, Csr<T>& A, CsrDict<T>* dict = nullptr);
// y = A x.  variant: 0 auto (TMA-staged when the plan allows), 1 force row-per-thread LDG, 2 force TMA-staged
template <class T> void k_spmv(Ctx& c, const Csr<T>& A, const T* x, T* y, int variant = 0);
// y = A x through the encoded rows (kb200_spmv_csr variant 3); throws when the operator is not encoded
template <class T> void k_spmv_dict(Ctx& c, const CsrDict<T>& D, const T* x, T* y);
// Row-partitioned operators: send this rank's boundary entries of x to the peers' halo buffers and meet in the
// in-kernel barrier (no-op on a single GPU).  Every y = A x on a distributed workspace is preceded by one.
template <class T> void k_halo_exchange(Ctx& c, const T* x);

// ---------------------------------------------------------------------------
// Operators as the solvers see them (A, M, N of the reference's kwargs).
// ---------------------------------------------------------------------------
typedef void (*MatvecFn)(const void* x, void* y, void* userdata);

template <class T>
struct LinOp {
  enum Kind { NONE, CSR, DIAG, BDIAG, HOST_CB, DEV_CB } kind = NONE;
  const Csr<T>* csr = nullptr;
  const CsrDict<T>* dict = nullptr;   // CSR: its constant-coefficient encoding, if any (the persistent CG kernel reads it)
  const T* diag = nullptr;      // DIAG: y = diag .* x (or x ./ diag with ldiv)
  const T* blocks = nullptr;     // BDIAG: dense bs x bs diagonal blocks, row-major, ceil(n / bs) of them (block-Jacobi)
  const T* blocks_inv = nullptr; //        their inverses (ldiv = true applies these)
  int bs = 0;
  MatvecFn fn = nullptr;         // callbacks: host pointers (HOST_CB) or device pointers (DEV_CB)
  void* userdata = nullptr;
  T* hx = nullptr;               // pinned staging for HOST_CB
  T* hy = nullptr;
  int n = 0;                     // length of y (and of x unless nin is set)
  int nin = 0;                   // HOST_CB of a rectangular operator: length of x (0: n)
  bool is_identity() const { return kind == NONE; }
};
template <class T> void op_apply(Ctx& c, const LinOp<T>& op, const T* x, T* y, bool ldiv = false);

// ---------------------------------------------------------------------------
// Solver options / statistics (kwargs of cg!/gmres!/bicgstab!/minres!;
// SimpleStats, src/krylov_stats.jl:24-36).
// ---------------------------------------------------------------------------
struct SolveOpts {
  double atol = -1, rtol = -1;      // <0 => sqrt(eps(T))
  int itmax = 0;                    // 0 => 2n
  double timemax = 1.0 / 0.0;
  int verbose = 0;
  bool history = false;
  double radius = 0;                // CG
  bool linesearch = false;          // CG, MINRES
  double lambda = 0;                // MINRES, LSQR, LSMR
  double etol = -1, conlim = -1;    // MINRES, LSQR, LSMR (<0 => defaults)
  double axtol = -1, btol = -1;     // LSQR, LSMR (<0 => sqrt(eps(T))); btol: LSLQ too
  double sigma = 0, utol = -1;      // LSLQ: σ (Gauss-Radau bounds when > 0), utol (<0 => sqrt(eps(T)))
  bool transfer_to_lsqr = false;    // LSLQ
  bool transfer_to_bicg = true;     // BiLQ, BiLQR
  bool transfer_to_usymcg = true;   // TriLQR
  bool restart = false;             // GMRES, FOM, FGMRES
  bool reorthogonalization = false; // GMRES, FOM, FGMRES
  bool check_curvature = false;     // CG-Lanczos
  double cr_gamma = -1;             // CR: kwarg γ (<0 => sqrt(eps(T)))
  bool ldiv = false;
  int (*callback)(void* ws, void* user) = nullptr;   // returns nonzero => user-requested exit
  void* callback_user = nullptr;
  int fused = 1;                    // 0 => force the generic primitive path
  int batch = 0;                    // fused CG: iterations enqueued per host poll (0 => default)
  int time_kernels = 0;             // fused CG: bracket the first launches of K1/K2 with CUDA events
  int persist = 1;                  // fused CG: 0 => keep the two-launch kernels instead of the persistent one
};

struct Stats {
  int niter = 0;
  bool solved = false, inconsistent = false, indefinite = false;
  int npcCount = 0;
  std::vector<double> residuals, Aresiduals, Acond;
  double allocation_timer = 0, timer = 0;
  double Anorm = NAN;                  // LanczosStats (cg_lanczos!)
  bool error_with_bnd = false;         // LSLQStats (lslq!)
  std::vector<double> err_lbnds, err_ubnds_lq, err_ubnds_cg;
  bool solved_primal = false, solved_dual = false;   // AdjointStats (bilqr!, trilqr!): residuals holds residuals_primal
  std::vector<double> residuals_dual;
  std::vector<std::vector<double>> shift_residuals;  // LanczosShiftStats (cg_lanczos_shift!, cgls_lanczos_shift!):
  std::vector<unsigned char> shift_indefinite;       // one history and one flag per shift
  std::string status = "unknown";
  void reset() {
    residuals.clear(); Aresiduals.clear(); Acond.clear(); indefinite = false; npcCount = 0;
    err_lbnds.clear(); err_ubnds_lq.clear(); err_ubnds_cg.clear(); error_with_bnd = false;
    residuals_dual.clear(); solved_primal = false; solved_dual = false;
  }
};

// values of KrylovSolverType (interfaces/include/krylov.h:48-83); cg_lanczos has no slot in the reference's C enum
enum SolverKind { S_CG = 0, S_CR = 1, S_MINRES = 3, S_DIOM = 5, S_DQGMRES = 6, S_FOM = 7, S_GMRES = 8, S_FGMRES = 9, S_BICGSTAB = 10,
                  S_CGS = 11, S_BILQ = 12, S_QMR = 13, S_TRILQR = 18, S_BILQR = 19, S_LSLQ = 20, S_LSQR = 21, S_LSMR = 22, S_CGLS = 24, S_CRLS = 25,
                  S_CGNE = 26, S_CRMR = 27, S_CRAIG = 28, S_CRAIGMR = 29, S_LNLQ = 30, S_CAR = 32, S_MINARES = 33, S_CG_LANCZOS = 100,
                  S_CG_LANCZOS_SHIFT = 101, S_CGLS_LANCZOS_SHIFT = 102 };   // the shift solvers: their own handle kind
// The interface facts of each solver the C ABI serves, one row per SolverKind (capi.cu reads them; ws_create `rect`).
enum PrecondUse : unsigned char {
  P_ON_N,        // takes the preconditioner on the n-dimensional space (the square solvers: n = m)
  P_ON_M,        // takes it on the m-dimensional space
  P_IGNORED,     // accepted and not applied, as the reference's C layer does
  P_REFUSED      // refused with the row's text
};
struct PrecondSlot { PrecondUse use; const char* refusal; };
enum BdiagRule : unsigned char { BD_TAKES, BD_REFUSED_AT_ATTACH, BD_REFUSED_AT_SOLVE };
enum CRule : unsigned char {
  C_NONE,            // c is ignored
  C_OPTIONAL_M,      // c has m entries; nullptr: c = b
  C_REQUIRED_N       // the adjoint system A^T y = c: c has n entries (and A^T, cached, max(m, n) rows)
};
enum WarmRule : unsigned char { WARM_X0, WARM_X0_Y0, WARM_NONE };
// the KrylovOptions fields that reach SolveOpts
enum OptField : unsigned { O_RADIUS = 1, O_LINESEARCH = 2, O_LAMBDA = 4, O_RESTART = 8, O_REORTH = 16 };
struct SolverInfo {
  const char* name;
  bool rect;                 // A is m x n (b has m entries, x n); else m == n
  bool adjoint;              // applies A^T: matvec_At, or the cached transpose of the CSR operator
  PrecondSlot M, N;
  BdiagRule bdiag;           // block-Jacobi M / N
  const char* bdiag_refusal;
  CRule c;
  int nsol;                  // 2: krylov_get_y returns y (m entries)
  WarmRule warm;
  const char* dist;          // nullptr: row-partitioned solves are available; else the refusal of krylov_b200_dist_init
  unsigned opts;             // OptField bits
};

constexpr PrecondSlot kOnN{P_ON_N, nullptr}, kOnM{P_ON_M, nullptr}, kIgnored{P_IGNORED, nullptr};
constexpr const char* kLsqBdiag =
    "not available on least-squares (LSQR, LSMR, CGLS, CRLS) or least-norm (CRAIG, CRAIGMR, LNLQ, CGNE, CRMR) workspaces";
constexpr const char* kLsqDist = "row-partitioned least-squares (LSQR, LSMR, CGLS, CRLS) and least-norm (CRAIG, CRAIGMR, "
                                 "LNLQ, CGNE, CRMR) solves are not available";
constexpr PrecondSlot kNoNLs{P_REFUSED, "cgls and crls take no right preconditioner N (M acts on the m-dimensional residual space)"};
constexpr PrecondSlot kNoNCar{P_REFUSED, "car and minares take no right preconditioner N (matvec_N): only M, and for minares none"};
constexpr const char* kCarDist = "row-partitioned CAR / MINARES solves are not available";
constexpr const char* kBiorthBdiag = "bilq and qmr apply M^H and N^H: block-Jacobi preconditioners are not available for them";
constexpr const char* kBiorthDist = "row-partitioned BiLQ / QMR solves are not available";
constexpr const char* kAdjointDist = "row-partitioned BiLQR / TriLQR solves are not available";
constexpr const char* kNoPBilqr = "bilqr takes no preconditioner (matvec_M, matvec_N or an attached M / N)";
constexpr const char* kNoPTrilqr = "trilqr takes no preconditioner (matvec_M, matvec_N or an attached M / N)";
constexpr const char* kNoMCgne = "cgne takes no preconditioner M: N (on the m-dimensional residual space) is its only preconditioner";
constexpr const char* kNoMCrmr = "crmr takes no preconditioner M: N (on the m-dimensional residual space) is its only preconditioner";

// Indexed by SolverKind; the last row is S_CG_LANCZOS.  Rows without a name: ids the library does not serve.
inline constexpr SolverInfo kSolvers[] = {
  // name, rect, adjoint, M, N, bdiag, bdiag_refusal, c, nsol, warm, dist, opts
  {"cg",         false, false, kOnN,    kIgnored, BD_TAKES, nullptr, C_NONE, 1, WARM_X0, nullptr, O_RADIUS | O_LINESEARCH},
  {"cr",         false, false, kOnN,    kIgnored, BD_TAKES, nullptr, C_NONE, 1, WARM_X0, nullptr, O_RADIUS | O_LINESEARCH},
  {},                                                                                                  // 2 SYMMLQ
  {"minres",     false, false, kOnN,    kIgnored, BD_TAKES, nullptr, C_NONE, 1, WARM_X0, nullptr, O_LAMBDA | O_LINESEARCH},
  {},                                                                                                  // 4 MINRES-QLP
  {"diom",       false, false, kOnN,    kOnN,     BD_TAKES, nullptr, C_NONE, 1, WARM_X0, nullptr, O_REORTH},
  {"dqgmres",    false, false, kOnN,    kOnN,     BD_TAKES, nullptr, C_NONE, 1, WARM_X0, nullptr, O_REORTH},
  {"fom",        false, false, kOnN,    kOnN,     BD_TAKES, nullptr, C_NONE, 1, WARM_X0, nullptr, O_RESTART | O_REORTH},
  {"gmres",      false, false, kOnN,    kOnN,     BD_TAKES, nullptr, C_NONE, 1, WARM_X0, nullptr, O_RESTART | O_REORTH},
  {"fgmres",     false, false, kOnN,    kOnN,     BD_TAKES, nullptr, C_NONE, 1, WARM_X0, nullptr, O_RESTART | O_REORTH},
  // BiCGSTAB, CGS, BiLQ and QMR accept c when given; the reference's C layer never forwards it (c = b)
  {"bicgstab",   false, false, kOnN,    kOnN,     BD_TAKES, nullptr, C_OPTIONAL_M, 1, WARM_X0, nullptr, 0},
  {"cgs",        false, false, kOnN,    kOnN,     BD_TAKES, nullptr, C_OPTIONAL_M, 1, WARM_X0, nullptr, 0},
  // A^T of a row block needs the column halo of A, not its row halo
  {"bilq",       false, true,  kOnN,    kOnN,     BD_REFUSED_AT_SOLVE, kBiorthBdiag, C_OPTIONAL_M, 1, WARM_X0, kBiorthDist, 0},
  {"qmr",        false, true,  kOnN,    kOnN,     BD_REFUSED_AT_SOLVE, kBiorthBdiag, C_OPTIONAL_M, 1, WARM_X0, kBiorthDist, 0},
  {}, {}, {}, {},                                                                                      // 14-17 USYMLQ, USYMQR, TriCG, TriMR
  {"trilqr",     true,  true,  {P_REFUSED, kNoPTrilqr}, {P_REFUSED, kNoPTrilqr}, BD_REFUSED_AT_SOLVE, kNoPTrilqr,
                 C_REQUIRED_N, 2, WARM_X0_Y0, kAdjointDist, 0},
  {"bilqr",      false, true,  {P_REFUSED, kNoPBilqr}, {P_REFUSED, kNoPBilqr}, BD_REFUSED_AT_SOLVE, kNoPBilqr,
                 C_REQUIRED_N, 2, WARM_X0_Y0, kAdjointDist, 0},
  {"lslq",       true,  true,  kOnM,    kOnN,     BD_REFUSED_AT_ATTACH, kLsqBdiag, C_NONE, 1, WARM_NONE, kLsqDist, O_LAMBDA},
  {"lsqr",       true,  true,  kOnM,    kOnN,     BD_REFUSED_AT_ATTACH, kLsqBdiag, C_NONE, 1, WARM_NONE, kLsqDist, O_LAMBDA | O_RADIUS},
  {"lsmr",       true,  true,  kOnM,    kOnN,     BD_REFUSED_AT_ATTACH, kLsqBdiag, C_NONE, 1, WARM_NONE, kLsqDist, O_LAMBDA | O_RADIUS},
  {},                                                                                                  // 23 USYMLQR
  // the reference's C layer drops N for CGLS / CRLS; a caller passing one expects it to act, so it is refused
  {"cgls",       true,  true,  kOnM,    kNoNLs,   BD_REFUSED_AT_ATTACH, kLsqBdiag, C_NONE, 1, WARM_NONE, kLsqDist, O_LAMBDA | O_RADIUS},
  {"crls",       true,  true,  kOnM,    kNoNLs,   BD_REFUSED_AT_ATTACH, kLsqBdiag, C_NONE, 1, WARM_NONE, kLsqDist, O_LAMBDA | O_RADIUS},
  // CGNE / CRMR: CG and CR on A A^T y = b with x = A^T y; the C layer drops M in the same way, N (on the m-dimensional
  // residual space) is their only preconditioner
  {"cgne",       true,  true,  {P_REFUSED, kNoMCgne}, kOnM, BD_REFUSED_AT_ATTACH, kLsqBdiag, C_NONE, 1, WARM_NONE, kLsqDist, O_LAMBDA},
  {"crmr",       true,  true,  {P_REFUSED, kNoMCrmr}, kOnM, BD_REFUSED_AT_ATTACH, kLsqBdiag, C_NONE, 1, WARM_NONE, kLsqDist, O_LAMBDA},
  // the least-norm solvers: min ||x|| subject to A x = b, x = A^T y; they return the multipliers y too
  {"craig",      true,  true,  kOnM,    kOnN,     BD_REFUSED_AT_ATTACH, kLsqBdiag, C_NONE, 2, WARM_NONE, kLsqDist, O_LAMBDA},
  {"craigmr",    true,  true,  kOnM,    kOnN,     BD_REFUSED_AT_ATTACH, kLsqBdiag, C_NONE, 2, WARM_NONE, kLsqDist, O_LAMBDA},
  {"lnlq",       true,  true,  kOnM,    kOnN,     BD_REFUSED_AT_ATTACH, kLsqBdiag, C_NONE, 2, WARM_NONE, kLsqDist, O_LAMBDA},
  {},                                                                                                  // 31 GPMR
  // the reference's C layer drops N for CAR and MINARES; it is refused as for CGLS.  MINARES's driver refuses M.
  {"car",        false, false, kOnN,    kNoNCar,  BD_TAKES, nullptr, C_NONE, 1, WARM_X0, kCarDist, 0},
  {"minares",    false, false, kOnN,    kNoNCar,  BD_TAKES, nullptr, C_NONE, 1, WARM_X0, kCarDist, O_LAMBDA},
  {"cg_lanczos", false, false, kOnN,    kIgnored, BD_TAKES, nullptr, C_NONE, 1, WARM_X0, nullptr, 0},
};
constexpr int kSolverRows = sizeof(kSolvers) / sizeof(kSolvers[0]);
static_assert(kSolverRows == S_MINARES + 2, "one row per id up to S_MINARES, then S_CG_LANCZOS");
// the row of `kind`, nullptr for ids the library does not serve
inline const SolverInfo* solver_info(int kind) {
  if (kind == S_CG_LANCZOS) return &kSolvers[kSolverRows - 1];
  return kind >= 0 && kind < kSolverRows - 1 && kSolvers[kind].name ? &kSolvers[kind] : nullptr;
}
// entries of an attached diagonal: a refused or ignored M has m, N n
inline int precond_len(const SolverInfo& s, int which, int m, int n) {
  const PrecondUse u = which == 0 ? s.M.use : s.N.use;
  return u == P_ON_M || (u != P_ON_N && which == 0) ? m : n;
}

// One workspace per (solver, dtype): owns every device vector of the solver
// (src/krylov_workspaces.jl; SURVEY.md appendix B for fields and aliasing).
template <class T>
struct Workspace {
  SolverKind kind;
  int m = 0, n = 0;
  Ctx ctx;
  Stats stats;
  bool warm_start = false;
  // device vectors (nullptr == Julia's length-0 vector)
  T *x = nullptr, *dx = nullptr;
  T *r = nullptr, *p = nullptr, *Ap = nullptr, *z = nullptr, *npc_dir = nullptr;      // CG
  T *p2 = nullptr;                                                                   // CG fused: second p buffer
  T *v = nullptr, *s = nullptr, *qd = nullptr, *t = nullptr, *yz = nullptr;           // BiCGSTAB (+ r, p)
  T *r1 = nullptr, *r2 = nullptr, *w1 = nullptr, *w2 = nullptr, *y = nullptr, *vv = nullptr;  // MINRES
  T *w = nullptr, *q = nullptr, *pp = nullptr;                                        // GMRES / FOM / FGMRES (+ V)
  T *u = nullptr, *ts = nullptr, *vw = nullptr;                                       // CGS (+ r, p, q, yz)
  T *Mv = nullptr, *Mv_prev = nullptr, *Mv_next = nullptr;                            // CG-Lanczos (+ p, vv)
  T *Nv = nullptr, *Mu = nullptr, *Av = nullptr, *Atu = nullptr;                     // LSQR / LSMR (+ w, u, v; Mu, Av, u: m)
  T *h = nullptr, *hbar = nullptr;                                                   // LSMR
  T *u_prev = nullptr, *v_prev = nullptr;                                             // BiLQ / QMR (+ u, v, q, p; w1, w2 / w)
  T *dy = nullptr;                     // BiLQR / TriLQR: Δy of a warm start (+ x, y = t, u, v, u_prev, v_prev, q, p,
                                       // w = d̅, w1 = w_{k-3}, w2 = w_{k-2}; TriLQR: v-space vectors have m entries)
  T *d1 = nullptr, *d2 = nullptr;      // MINARES: d_{k-1}, d_{k-2} (+ v = v_k, vv = v_{k+1}, w1 = w_{k-1}, w2 = w_{k-2}, q)
                                       // CAR: r, p, s, q, t, u (+ Mu, lazy)
                                       // CRAIG: x, Nv, Atu (n), y, w, Mu, Av (m) (+ u, v, w2: lazy)
                                       // CRAIGMR: d in d1, w̄ in w1 (+ x, Nv, Atu, y, w, Mu, Av; u, v, q: lazy)
                                       // LNLQ: w̄ in w (+ x, Nv, y, Mu; Atu, Av, u, v, q: lazy)
  T *Ar = nullptr, *Mr = nullptr;      // CGLS: Mr (m, lazy; Mq aliases it) (+ x, p, s: n; r, q: m)
                                       // CRLS: Ar (n), Ms in Mr (m, lazy) (+ x, p, q: n; r, Ap, s: m)
                                       // CGNE: Aᴴz in Ar (+ x, p: n; r, q: m; s, z: m, lazy)
                                       // CRMR: Aᴴr in Ar, Nq in z (m, lazy) (+ x, p: n; r, q: m; s: m, lazy)
  T *Xs = nullptr, *Ps = nullptr;      // shift solvers: x_i and p_i, column-major n x nshifts blocks
  T *u_next = nullptr;                 // CGLS-Lanczos-shift (+ v: n; u_prev, u: m)
  int nshifts = 0;
  std::vector<T*> V;
  std::vector<T*> Z;                   // FGMRES: Z[k] = N_k V[k];  DQGMRES / DIOM: the direction stack P
  std::vector<T> c, sgiv, zg, R;       // GMRES host-side Givens data
  std::vector<T> err_vec;              // MINRES, LSQR, LSMR window
  int memory = 20, window = 5;
  int inner_iter = 0;
  const T* mdiag_fused = nullptr;      // diagonal of M for the fused phases (set per solve; nullptr: M = I)
  double k1_ms = 0, k2_ms = 0;         // average event-timed duration of the fused kernels (time_kernels)
  int timed_pairs = 0;
  void* fused_state = nullptr;         // device scalar block of the fused paths (4 KB; CG: cg_fused.cu's layout, else
                                       // one state struct per family at its start, fused_phases.cu)
  void* fused_host = nullptr;          // pinned mirror: CG's layout, else two copies of the state struct (seed, read-back)
  cudaEvent_t fused_ev[2] = {nullptr, nullptr};   // fused CG: one event per read-back slot
  unsigned long long fused_seq = 0;               // persistent CG: sequence number of the last launch (host-polled report)
  T* bbuf = nullptr;                   // device copies of host b / c for the C ABI
  T* cbuf = nullptr;
  // row-partitioned (multi-GPU) state; world == 1 means single GPU
  struct Dist {
    int rank = 0, world = 1;
    HaloMap halo{0, 0, nullptr, nullptr};      // device arrays
    void* mailbox = nullptr;                    // local mailbox allocation (values + flags)
    T* bufA_peer[kMaxRanks] = {};               // every rank's `p` allocation (as created)
    T* bufB_peer[kMaxRanks] = {};               // every rank's `p2` allocation
    T* r_peer[kMaxRanks] = {};
    std::vector<void*> opened;                  // cudaIpcOpenMemHandle results to close
    bool swapped = false;                       // ws.p currently points at the bufB allocation
    T* halo_buf = nullptr;                      // local halo buffers [r | p(bufA) | p(bufB)], nhalo entries each
    T* halo_buf_peer[kMaxRanks] = {};           // every rank's halo_buf
    int nhalo_peer[kMaxRanks] = {};             // every rank's halo length (section stride inside its halo_buf)
    void* dummy[3] = {nullptr, nullptr, nullptr};  // placeholder IPC exports of the non-CG solvers
    T* xhalo = nullptr;                         // general x-halo buffer (2 sections) of k_halo_exchange
    T* xhalo_peer[kMaxRanks] = {};
    int nsend = 0;                              // send list of the general exchange (device arrays)
    int* send_row = nullptr; int* send_peer = nullptr; int* send_slot = nullptr;
    long long nglobal = 0;                      // global number of rows (default itmax = 2 n)
    int npush = 0;                              // > 0: push mode (contiguous send ranges), else pull mode
    int* tile_order = nullptr;                  // persistent CG: interior tiles first, halo tiles last (device)
    const void* tile_order_for = nullptr;       // ... built for this operator
    int tile_order_n = 0;
    int tile_order_interior = 0;                // number of tiles without halo columns (they come first)
    PushRange push[kMaxPushRanges];
  } dist;
};

template <class T> Workspace<T>* ws_create(SolverKind kind, int m, int n, int memory, int window, int device);
template <class T> void ws_destroy(Workspace<T>* ws);
template <class T> void ws_warm_start(Workspace<T>* ws, const T* x0_dev);

// Solver drivers (device pointers for b, c).  Throw std::runtime_error where
// the reference calls error(...).
template <class T> void cg_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const SolveOpts& o);
template <class T> void bicgstab_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const T* c, const LinOp<T>& M, const LinOp<T>& N, const SolveOpts& o);
template <class T> void minres_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const SolveOpts& o);
// one Arnoldi driver (solvers.cu)
template <class T> void gmres_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const LinOp<T>& N, const SolveOpts& o);
template <class T> void fom_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const LinOp<T>& N, const SolveOpts& o);
template <class T> void fgmres_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const LinOp<T>& N, const SolveOpts& o);
// Sibling solvers on the same kernels (siblings.cu; SURVEY.md 8f-3)
template <class T> void cgs_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const T* c, const LinOp<T>& M, const LinOp<T>& N, const SolveOpts& o);
template <class T> void cg_lanczos_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const SolveOpts& o);
template <class T> void dqgmres_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const LinOp<T>& N, const SolveOpts& o);
template <class T> void diom_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const LinOp<T>& N, const SolveOpts& o);
template <class T> void cr_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const SolveOpts& o);
template <class T> void car_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const SolveOpts& o);
// minares! takes no preconditioner (the reference refuses M != I); o.lambda shifts A, o.axtol holds its Artol
template <class T> void minares_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const SolveOpts& o);
// The shift solvers (shift.cu): one Lanczos process for the p systems (A + σᵢ I) xᵢ = b (CG-Lanczos-shift, M on
// the n-space) or (AᵀA + σᵢ I) xᵢ = Aᵀb (CGLS-Lanczos-shift, no M; At: A^T as a CSR operator or a callback m -> n).
// Their workspace holds X and P (n x nshifts) besides the Lanczos vectors; stats.shift_* the per-shift results.
template <class T> Workspace<T>* shift_ws_create(SolverKind kind, int m, int n, int nshifts, int device);
template <class T> void cg_lanczos_shift_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const T* shifts,
                                               const LinOp<T>& M, const SolveOpts& o);
template <class T> void cgls_lanczos_shift_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b,
                                                 const T* shifts, const SolveOpts& o);
// Least squares on an m x n operator (lsq.cu).  At: the adjoint (a CSR operator holding A^T, or a callback m -> n).
template <class T> void lsqr_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& M,
                                   const LinOp<T>& N, const SolveOpts& o);
template <class T> void lsmr_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& M,
                                   const LinOp<T>& N, const SolveOpts& o);
template <class T> void lslq_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& M,
                                   const LinOp<T>& N, const SolveOpts& o);
// Least norm (lsq.cu): min ||x|| subject to A x = b, x = A^T y; M acts on the m-space, N on the n-space.
template <class T> void craig_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& M,
                                    const LinOp<T>& N, const SolveOpts& o);
template <class T> void craigmr_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& M,
                                      const LinOp<T>& N, const SolveOpts& o);
template <class T> void lnlq_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& M,
                                   const LinOp<T>& N, const SolveOpts& o);
// CGNE / CRMR: N (m x m) acts on the residual space; they take no M.
template <class T> void cgne_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& N,
                                   const SolveOpts& o);
template <class T> void crmr_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& N,
                                   const SolveOpts& o);
// CGLS / CRLS: M (m x m) acts on the residual space; they take no N.
template <class T> void cgls_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& M,
                                   const SolveOpts& o);
template <class T> void crls_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& M,
                                   const SolveOpts& o);

// Fused CG (cg_fused.cu).  cg_fused_plan decides once whether and how a solve runs fused: fused == false sends it
// to the generic primitive path (still on the GPU); otherwise the plan holds everything cg_fused_loop launches.
template <class T> struct CgState;
template <class T> struct CgPeers;
template <class T> struct CgPersistArgs;
struct GridBar;
template <class T>
struct CgFusedPlan {
  typedef void (*K1Fn)(Csr<T>, const T*, const T*, T*, T*, CgState<T>*, T*, unsigned*, DistComm*, CgPeers<T>, T*);
  typedef void (*K2Fn)(int, T*, T*, const T*, const T*, CgState<T>*, T*, unsigned*, DistComm*, const T*, PushPlan<T>);
  typedef void (*KpFn)(Csr<T>, CgPersistArgs<T>, CgState<T>*, T*, GridBar*, DistComm*);
  typedef void (*KdFn)(CsrDict<T>, CgPersistArgs<T>, CgState<T>*, T*, GridBar*);
  bool fused = false;
  bool persist = false;         // one cooperative launch per batch of iterations; false: K1 + K2 per iteration
  bool single_step = false;     // callback, verbose or timemax: x is current and the stream idle after every iteration
  bool xup = false;             // x += alpha p rides in the next K1 / phase A (else in K2)
  int batch = 1;                // iterations per launch / host poll
  const Csr<T>* A = nullptr;
  const T* mdiag = nullptr;     // Jacobi M (nullptr: none)
  const T* mblocks = nullptr;   // block-Jacobi M: dense mbs x mbs diagonal blocks, row-major (nullptr: none)
  int mbs = 0;
  K1Fn k1 = nullptr;            // two-launch kernels and their launch shapes
  K2Fn k2 = nullptr;
  int k1_grid = 0, k1_block = 0, k2_grid = 0;
  size_t k1_smem = 0;
  KpFn kp = nullptr;            // persistent kernel on CSR ...
  KdFn kd = nullptr;            // ... or on the operator's encoding `dict` (nullptr: CSR)
  const CsrDict<T>* dict = nullptr;
  int pgrid = 0;
};
struct CgFusedExit { int iter; bool solved, tired, zero_curvature, inconsistent, user_exit, overtimed; };
template <class T> CgFusedPlan<T> cg_fused_plan(const Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& M, const SolveOpts& o);
template <class T> CgFusedExit cg_fused_loop(Workspace<T>& ws, const CgFusedPlan<T>& plan, const SolveOpts& o, T gamma0, T eps_tol,
                                             int itmax, double start_time);
template <class T> void cg_dist_push_r(Workspace<T>& ws);
template <class T> void cg_fused_prepare(Workspace<T>& ws);   // p2 and the read-back events (ws_create)
// the 4 KB device block ws.fused_state and its pinned mirror ws.fused_host, zeroed (ws_create, every kind)
template <class T> void fused_block_alloc(Workspace<T>& ws);
constexpr size_t kFusedBlockBytes = 4096;

// Fused iteration phases of BiCGSTAB / MINRES / GMRES (fused_phases.cu); eligible when A is a CSR operator,
// M = N = I (and for GMRES no reorthogonalization).
template <class T> void bicgstab_fused_iteration(Workspace<T>& ws, const Csr<T>& A, const T* cvec, bool first, T rho_in, T* alpha,
                                                 T* omega, T* next_rho, T* rNorm);
template <class T> void minres_fused_lanczos(Workspace<T>& ws, const Csr<T>& A, int iter, T lambda, T beta, T oldbeta, T cs, T sn,
                                             T deltabar, T eps_rot, T* w, T* alpha, T* beta2);
template <class T> T minres_fused_update(Workspace<T>& ws, T* w, T gamma, T phi);
// xin: vector the operator is applied to (default V[k]; FGMRES passes Z[k])
template <class T> void gmres_fused_arnoldi(Workspace<T>& ws, const Csr<T>& A, int k, T* h_out, T* Hbis, const T* xin = nullptr);
template <class T> void fused_multi_axpy(Workspace<T>& ws, T* xr, int k, const T* y, T* const* vecs);
// sibling solvers (fused_phases.cu): grouped passes with host-side scalars
template <class T> void fused_orth_chain(Workspace<T>& ws, const Csr<T>& A, const T* xin, T* q, const T* const* vecs, int cnt, T* h_out, T* Hbis);
template <class T> void trunc_fused_direction(Workspace<T>& ws, T* pp, int cnt, T* const* pvecs, const T* coefs, const T* z, T h0, T step);
template <class T> T cgs_fused_sigma(Workspace<T>& ws, const Csr<T>& A, const T* cvec);
template <class T> void cgs_fused_update(Workspace<T>& ws, const Csr<T>& A, const T* cvec, T alpha, T* rho_next, T* rr);
template <class T> void cgs_fused_directions(Workspace<T>& ws, T beta);
template <class T> T lanczos_fused_delta(Workspace<T>& ws, const Csr<T>& A);
template <class T> T lanczos_fused_recur(Workspace<T>& ws, T delta, T beta, bool later);
template <class T> void lanczos_fused_update(Workspace<T>& ws, T beta, T gamma, T sigma, T omega);
// Shift solvers (fused_phases.cu).  The shift update of cnt active shifts (columns x[i], p[i] and their scalars), in
// ceil(cnt / kShiftPass) streaming passes over n; `scale`: the first pass sets v = v / beta first.
constexpr int kShiftPass = 16;
template <class T> void shift_fused_update(Workspace<T>& ws, T* v, bool scale, T beta, int cnt, T* const* x, T* const* p,
                                           const T* gamma, const T* sigma, const T* omega);
// CGLS-Lanczos-shift, M = I, A and A^T CSR operators: u_next = A v, returns <u_next, u_next> (one read-back) ...
template <class T> T shift_gk_delta(Workspace<T>& ws, const Csr<T>& A);
// ... then u_k = s_u ũ_k, u_next -= delta u_k + beta u_prev, u_prev = u_k over m, and v = A^T u_next; returns <v, v>.
template <class T> T shift_gk_next(Workspace<T>& ws, const Csr<T>& At, T s_u, T delta, T beta);
template <class T> void cr_fused_step(Workspace<T>& ws, const Csr<T>& A, T alpha, T* xx, T* rr, T* ArAr, T* rAr);
template <class T> T cr_fused_directions(Workspace<T>& ws, T beta);
// CAR (fused_phases.cu), M = I.  C1: x += alpha p ; r -= alpha q ; s -= alpha u, one read-back of ||r||^2, ||s||^2.
template <class T> void car_fused_step(Workspace<T>& ws, T alpha, T* rr, T* ss);
// C2: t = A s, rho_next = <t, s> and beta = rho_next / rho on the device; C3: p = r + beta p ; q = s + beta q ;
// u = t + beta u, <u, u>.  One read-back of {rho_next, <u, u>}.
template <class T> void car_fused_directions(Workspace<T>& ws, const Csr<T>& A, T rho, T* rho_next, T* uu);
// MINARES (fused_phases.cu).  M1: w_k from v_k, w_{k-1}, w_{k-2} (into wk: w_{k-1}'s buffer at iteration 1, w_{k-2}'s
// after); with `lanczos`, M1 is the SpMV on v_{k+1} that also forms v_k = A v_{k+1} - beta v_k (+ shift v_{k+1}) and
// alpha = <v_k, v_{k+1}> on the device, and M2 v_k -= alpha v_{k+1} with ||v_k||^2: one read-back of {alpha, ||v_k||^2}.
// Without `lanczos` (past the early-termination point) M1 is a streaming pass with the w update only.
template <class T> void minares_fused_lanczos(Workspace<T>& ws, const Csr<T>& A, bool lanczos, int iter, T* vk, const T* vk1,
                                              T* wk, const T* w1, T eps2, T gamma1, T lam, T beta1, T shift, T* alpha, T* vv);
// M3: v_k /= beta (scale), d_k from w_k, d_{k-1}, d_{k-2} (into dk, as for w), x += zeta d_k.
template <class T> void minares_fused_update(Workspace<T>& ws, int iter, T* vk, bool scale, T beta, T* dk, const T* d1,
                                             const T* wk, T rho2, T phi1, T mu, T zeta);
int gmres_fused_max();
// LSQR / LSMR (fused_phases.cu), M = N = I, A and A^T CSR operators, no trust region.  Golub-Kahan step: P1 (SpMV on A
// with Mu <- A v - alpha Mu and ||Mu||^2) and P2 (SpMV on A^T with Nv <- A^T u - beta Nv, ||Nv||^2 and, for LSQR,
// <w, w>), then one read-back of {beta, alpha, <w, w>}.  `init`: first iteration, sets the device scalars from the host.
template <class T> void lsq_fused_bidiag(Workspace<T>& ws, const Csr<T>& A, const Csr<T>& At, bool init, T alpha, bool want_ww,
                                         T* beta, T* alpha_out, T* ww);
// P3.  LSQR: v = Nv / alpha (scale_v), x += sigma w, w = v - tau w.  LSMR (lsmr = true, w = h):
// v = Nv / alpha (scale_v), hbar = h - delta hbar, x += sigma hbar, h = v - tau h; returns ||x|| (LSMR only).
template <class T> T lsq_fused_update(Workspace<T>& ws, bool lsmr, bool scale_v, T inv_alpha, T sigma, T tau, T delta);
// LSLQ's update after P1 / P2 (w = w̄): v = Nv / alpha (scale_v), x += (c zeta) w̄, x += (s zeta) v, w̄ = -c v + s w̄.
template <class T> void lslq_fused_update(Workspace<T>& ws, bool scale_v, T inv_alpha, T czeta, T szeta, T c, T s);
// CRAIG (fused_phases.cu), lambda = 0, M = N = I, A and A^T CSR operators; Mu and Nv stay unscaled (s_u = 1/beta and
// s_v = 1/alpha are applied by their readers).  C1: SpMV on A^T gathering u with x += xi v (the previous iteration's
// update, pending when xup), Nv = A^T u - beta v; returns alpha (one read-back).  `init`: first iteration.
template <class T> T craig_fused_p1(Workspace<T>& ws, const Csr<T>& At, bool init, T beta, T s_v, bool xup, T xi);
// C2: SpMV on A gathering v with w = u + tw w, y += ty w, Mu = A v - alpha u; one read-back of beta and <w, w>.
template <class T> void craig_fused_p2(Workspace<T>& ws, const Csr<T>& A, T s_u, T alpha, T tw, T ty, T* beta, T* ww);
// the pending x += xi v (before a callback and after the last iteration)
template <class T> void craig_fused_flush(Workspace<T>& ws, T xi, T s_v);
// CRAIGMR (fused_phases.cu), same conditions.  R1: SpMV on A gathering v, Mu = A v - alpha u; returns beta.
template <class T> T craigmr_fused_p1(Workspace<T>& ws, const Csr<T>& A, bool init, T s_u, T alpha);
// R2: SpMV on A^T gathering u, d = v / rho (first) or (1/rho) v + tr d, x += zeta d, Nv = A^T u - beta v; R3 over m:
// w = (1/rho) w̄ + tr w, y += zeta w and, when alpha != 0, w̄ = (1/alpha) u - (beta/alpha) w̄.  Returns alpha.
template <class T> T craigmr_fused_p23(Workspace<T>& ws, const Csr<T>& At, bool first, T s_u, T s_v, T beta, T rho, T inv_rho,
                                       T tr, T zeta);
// LNLQ (fused_phases.cu), same conditions and the same pending factors.  L1: SpMV on A gathering v; first the previous
// pass's update (when yup: y += yc w̄, y += ys u, w̄ = wc u + ws w̄ with u = Mu s_u), then Mu = A v - alpha u; returns
// beta.  `init`: first pass (u_1 and v_1 stored scaled).
template <class T>
T lnlq_fused_l1(Workspace<T>& ws, const Csr<T>& A, bool init, T s_u, T alpha, bool yup, T yc, T ys, T wc, T wsn);
// L2: SpMV on A^T gathering u, x += tau v (v = Nv s_v), Nv = A^T u - beta v; returns alpha.
template <class T> T lnlq_fused_l2(Workspace<T>& ws, const Csr<T>& At, T s_v, T beta, T tau);
// the pending y / w̄ update over m (before a callback and after the last pass), and the terminal x += a v
template <class T> void lnlq_fused_flush(Workspace<T>& ws, T s_u, T yc, T ys, T wc, T wsn);
template <class T> void lnlq_fused_xup(Workspace<T>& ws, T a, T s_v);
// One CGLS iteration, M = I, no trust region, 4 launches: K1 q = A p (alpha on the device), K2 r -= alpha q, K3 s = A^T r
// with x += alpha p and s -= lambda x, K4 p = s + beta p.  One read-back: <r, r> and gamma = <s, s>.
// `init`: first iteration, sets gamma (and <p, p> = gamma) on the device from the host.
template <class T> void cgls_fused_iteration(Workspace<T>& ws, const Csr<T>& A, const Csr<T>& At, bool init, T gamma, T lambda,
                                             T* rr, T* gamma_out);
// One CRLS iteration, M = I, no trust region, 4 launches: L1 x += alpha p, Ar -= alpha q; L2 s = A Ar with r -= alpha Ap
// (gamma, beta on the device); L3 Ap = s + beta Ap; L4 q = A^T Ap with p = Ar + beta p, q += lambda p (next alpha).
// One read-back: <Ar, Ar>, <x, x>, <r, r> and gamma.  `init`: first iteration, sets alpha and gamma from the host.
template <class T> void crls_fused_iteration(Workspace<T>& ws, const Csr<T>& A, const Csr<T>& At, bool init, T alpha, T gamma,
                                             T lambda, T* ArAr, T* xx, T* rr, T* gamma_out);
// One CGNE iteration, N = I, lambda = 0, 2 launches: E1 (SpMV on A gathering p) r -= alpha (A p), with gamma and beta on
// the device; E2 (SpMV on A^T gathering r) x += alpha p, p = A^T r + beta p, delta = <p, p> and the next alpha on the
// device.  One read-back: gamma and delta.  `init`: first iteration, sets gamma and alpha = gamma / delta from the host.
template <class T> void cgne_fused_iteration(Workspace<T>& ws, const Csr<T>& A, const Csr<T>& At, bool init, T gamma, T delta,
                                             T* gamma_out, T* delta_out);
// One CRMR iteration, N = I, lambda = 0, 4 launches: R1 q = A p (alpha on the device), R2 r -= alpha q, R3 Aᴴr = A^T r
// with x += alpha p (gamma, beta on the device), R4 p = Aᴴr + beta p.  One read-back: <r, r> and gamma.
// `init`: first iteration, sets gamma on the device from the host.
template <class T> void crmr_fused_iteration(Workspace<T>& ws, const Csr<T>& A, const Csr<T>& At, bool init, T gamma, T* rr,
                                             T* gamma_out);
// BiLQ / QMR (fused_phases.cu), M = N = I, A and A^T CSR operators.  One Lanczos biorthogonalization step: B1 (SpMV on A
// gathering v: q = A v - gamma v_prev, alpha = <u, q> on the device) and B2 (SpMV on A^T gathering u: p = A^T u -
// beta u_prev - alpha u, q -= alpha v, <p, q>), then one read-back of {alpha, <p, q>}.
template <class T> void biorth_fused_lanczos(Workspace<T>& ws, const Csr<T>& A, const Csr<T>& At, T beta, T gamma, T* alpha, T* pq);
// QMR's update pass: w_k (into wk; w1 = w_{k-1}), x += zeta w_k, v_prev = q / beta1 and u_prev = p / gamma1 (keep: copies of
// v and u); returns ||v_prev||^2.  The caller then swaps v / v_prev and u / u_prev.
template <class T> T qmr_fused_update(Workspace<T>& ws, T* wk, const T* w1, int iter, T eps2, T lambda, T delta, T zeta, T beta1,
                                      T gamma1, bool keep);
// BiLQ's update pass (d̅ in ws.w): d̅ = v when first, else x += czeta d̅ + szeta v, d̅ = -c v + s d̅; the next v, u as for QMR;
// returns <v, v_next> and ||v_next||^2.
template <class T> void bilq_fused_update(Workspace<T>& ws, bool first, T czeta, T szeta, T c, T s, T beta1, T gamma1, bool keep,
                                          T* vv1, T* v1v1);
// BiLQR (fused_phases.cu): the update pass after B1 / B2.  Primal half (primal): d̅ = v when iter == 1, else
// x += czeta d̅ + szeta v, d̅ = -c v + s d̅, and <v, q>, ||q||^2.  Dual half (dual): w_{k-1} from u_{k-1} into wk (iter >= 2,
// as bilqr.jl:363-381; w3 = w_{k-3}, w2 = w_{k-2}), y += psi w_{k-1}, and ||u_{k+1}||^2.  Then v_{k+1} = q / beta1 and
// u_{k+1} = p / gamma1 into the buffers of v_{k-1}, u_{k-1} (keep: copies of v, u).  out: {<v, q>, ||q||^2, ||u_{k+1}||^2}.
template <class T> void bilqr_fused_update(Workspace<T>& ws, bool primal, bool dual, int iter, T czeta, T szeta, T c, T s,
                                           T* wk, const T* w2, T eps3, T lam2, T delta1, T psi1, T beta1, T gamma1, bool keep,
                                           T* out3);
// TriLQR (fused_phases.cu), A (m x n) and At (A^T, max(m, n) rows: rows beyond n are empty) CSR operators.  One SSY step:
// T1 (SpMV on A gathering u: q = A u - gamma v_prev, alpha = <v, q> on the device) and T2 (SpMV on A^T gathering v:
// p = A^T v - beta u_prev - alpha u, q -= alpha v over all m rows, ||p||^2 and ||q||^2), then one read-back of
// {alpha, ||q||^2, ||p||^2}.  `first`: iteration 1 (no gamma / beta terms).
template <class T> void trilqr_fused_ssy(Workspace<T>& ws, const Csr<T>& A, const Csr<T>& At, bool first, T beta, T gamma,
                                         T* alpha, T* qq, T* pp);
// TriLQR's update pass over max(m, n): primal half on the n-space (d̅ = u or x += czeta d̅ + szeta u, d̅ = -c u + s d̅),
// dual half on the m-space (w_{k-1} from v_{k-1}, y += psi w_{k-1}), then v_{k+1} = q / beta1 (beta1 != 0) and
// u_{k+1} = p / gamma1 (gamma1 != 0) into the buffers of v_{k-1}, u_{k-1}, else copies of v, u.  No read-back.
template <class T> void trilqr_fused_update(Workspace<T>& ws, bool primal, bool dual, int iter, T czeta, T szeta, T c, T s,
                                            T* wk, const T* w2, T eps3, T lam2, T delta1, T psi1, T beta1, T gamma1);
// bilqr! / trilqr! (adjoint.cu): A with its adjoint At (a CSR operator holding A^T, or a callback); b, c required.
template <class T> void bilqr_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const T* c,
                                    const SolveOpts& o);
template <class T> void trilqr_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const T* c,
                                     const SolveOpts& o);
template <class T> void ws_warm_start2(Workspace<T>* ws, const T* x0_dev, const T* y0_dev);
// bilq! / qmr! (biorth.cu): square A with its adjoint At (a CSR operator holding A^T, or a callback); c = nullptr: c = b.
template <class T> void bilq_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const T* c,
                                   const LinOp<T>& M, const LinOp<T>& N, const SolveOpts& o);
template <class T> void qmr_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const T* c,
                                  const LinOp<T>& M, const LinOp<T>& N, const SolveOpts& o);

// ---------------------------------------------------------------------------
// Krylov processes (src/krylov_processes.jl): drivers in processes.cu, passes in fused_phases.cu.  A call enqueues
// every pass of its k steps back to back; the coefficients live in a per-call device block laid out like the
// reference's nzval, the passes read their scalars from it, and the host reads the block back once at the end.
// ---------------------------------------------------------------------------
template <class T> struct ProcHead {       // start of the per-call device block
  int brk_kind, brk_iter;                  // first exact breakdown (kind 0: none), recorded in stream order
  T one, tmp;                              // 1 (the divisor of a stored column) and a reorthogonalization coefficient
  T beta1, gamma1;                         // β₁ and γ₁ (γ₁ᴴ) of the two-sided processes
};

template <class T> __device__ __forceinline__ T proc_div(T x, T s) { return s == T(0) ? T(0) : div_rn(x, s); }

// Gather of an SpMV that applies a pending division: x[j] / *scale_src, 0 when the divisor is 0 (kdivcopy! on a
// column that kfill! zeroes after a breakdown).  gather_for_cta (spmv_tiles.cuh) loads the divisor once per CTA.
template <class T> struct ProcXDiv {
  const T* __restrict__ x;
  const T* scale_src;
  T scale;
  __device__ __forceinline__ T operator()(int j) const { return proc_div(__ldg(&x[j]), scale); }
};

// SpMV epilogue of every process.  For its own row: own = src / *src_s stored in vout (the column the pending
// division produces, never the gathered one); q = acc - *s1 w1 - *s2 w2 (a null w stands for own, a null s skips the
// term); qout = q; with src2: own2 = src2 / *src2_s stored in vout2; with r: r -= *rs rx.  Accumulates one dot:
// dot 0 <own, q>, 1 <q, q>, 2 <own2, q>, 3 <y, q>, 4 <q, r>.
template <class T> struct ProcEpi {
  const T* src; const T* src_s; T* vout;
  const T* src2; const T* src2_s; T* vout2;
  const T* w1; const T* s1;
  const T* w2; const T* s2;
  T* qout;
  T* r; const T* rx; const T* rs;
  const T* y;
  int dot;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    const T own = src ? proc_div(src[row], *src_s) : T(0);
    if (vout) vout[row] = own;
    T q = acc;
    if (s1) q = add_rn(q, mul_rn(-*s1, w1 ? w1[row] : own));
    if (s2) q = add_rn(q, mul_rn(-*s2, w2 ? w2[row] : own));
    qout[row] = q;
    T own2 = T(0);
    if (src2) { own2 = proc_div(src2[row], *src2_s); vout2[row] = own2; }
    T rv = T(0);
    if (r) { rv = add_rn(r[row], mul_rn(-*rs, rx[row])); r[row] = rv; }
    const T a = dot == 0 ? own : dot == 1 ? q : dot == 2 ? own2 : dot == 3 ? y[row] : rv;
    d[0] += a * q;
  }
};

// Streaming pass: q -= *s x (x null: q is only read), then <y, q> (y null: <q, q>).
template <class T> struct ProcUpdBody {
  T* q; const T* x; const T* s; const T* y;
  __device__ __forceinline__ void operator()(int i, T* d) const {
    T v = q[i];
    if (x) { v = add_rn(v, mul_rn(-*s, x[i])); q[i] = v; }
    d[0] += (y ? y[i] : v) * v;
  }
};

// Final normalisation: out1 = src1 / *s1 over n1 entries and out2 = src2 / *s2 over n2 (0 when the divisor is 0).
template <class T> struct ProcDivBody {
  T* out1; const T* src1; const T* s1; int n1;
  T* out2; const T* src2; const T* s2; int n2;
  __device__ __forceinline__ void operator()(int i, T*) const {
    if (i < n1) out1[i] = proc_div(src1[i], *s1);
    if (out2 && i < n2) out2[i] = proc_div(src2[i], *s2);
  }
};

// What the CTA that completes a pass's reduction does with the total t (one thread, in stream order).
//   SET:    dst[0..3] = t; then *copy_dst = *copy_src (Lanczos: Tᵢ₋₁.ᵢ = Tᵢ.ᵢ₋₁).
//   NORM:   v = sqrt(t) into dst[0..3]; v == 0 records breakdown (kind, iter).
//   ACC:    *tmp = t; dst[k] += t (reorthogonalization).
//   BIORTH: t = pᴴq (or cᴴb); 0 records breakdown and gives β = γ = 0, else β = sqrt(|t|), γ = t / β;
//           dst[0] = β, dst[1] = γ, dst[2] = γ, dst[3] = β.
template <class T> struct ProcFin {
  enum { SET, NORM, ACC, BIORTH };
  ProcHead<T>* h;
  T* dst[4];
  const T* copy_src; T* copy_dst;
  int mode, kind, iter;
  __device__ void operator()(const T* tot) const {
    T v = tot[0], w = v;
    if (mode == NORM) { v = w = sqrt_rn(tot[0]); }
    if (mode == ACC) h->tmp = v;
    if (mode == BIORTH) {
      if (v == T(0)) { v = w = T(0); }
      else { const T b = sqrt_rn(fabs(tot[0])); w = div_rn(tot[0], b); v = b; }
    }
    if ((mode == NORM || mode == BIORTH) && v == T(0) && h->brk_kind == 0) { h->brk_kind = kind; h->brk_iter = iter; }
    for (int k = 0; k < 4; k++) {
      if (!dst[k]) continue;
      const T val = (mode == BIORTH && (k == 1 || k == 2)) ? w : v;
      *dst[k] = mode == ACC ? add_rn(*dst[k], val) : val;
    }
    if (copy_dst) *copy_dst = *copy_src;
  }
};

// The launches (fused_phases.cu): an SpMV on A whose gather divides by a device scalar, a streaming update / dot pass
// and the final normalisation pass.
template <class T> void proc_spmv(Ctx& c, const Csr<T>& A, const T* x, const T* x_s, const ProcEpi<T>& epi, const ProcFin<T>& fin);
template <class T> void proc_stream(Ctx& c, int n, const ProcUpdBody<T>& body, const ProcFin<T>& fin);
template <class T> void proc_divide(Ctx& c, const ProcDivBody<T>& body);

// The processes (processes.cu).  V / U: caller's device outputs, column-major with leading dimension = the vector's
// length.  coef (and coefH): host outputs in the reference's nzval order (dense column-major (k+1) x k for H).
// Exact breakdown without allow_breakdown throws the reference's message.  flags: bit 0 allow_breakdown, bit 1
// reorthogonalization.
template <class T> void hermitian_lanczos_run(Ctx& c, const Csr<T>& A, int k, const T* b, T* V, double* beta, double* coef, int flags);
template <class T> void arnoldi_run(Ctx& c, const Csr<T>& A, int k, const T* b, T* V, double* beta, double* H, int flags);
template <class T> void golub_kahan_run(Ctx& c, const Csr<T>& A, const Csr<T>& At, int k, const T* b, T* V, T* U, double* beta,
                                        double* coef, int flags);
template <class T> void nonhermitian_lanczos_run(Ctx& c, const Csr<T>& A, const Csr<T>& At, int k, const T* b, const T* cv, T* V,
                                                 T* U, double* beta, double* gamma, double* coefT, double* coefTH, int flags);
template <class T> void saunders_simon_yip_run(Ctx& c, const Csr<T>& A, const Csr<T>& At, int k, const T* b, const T* cv, T* V,
                                               T* U, double* beta, double* gamma, double* coefT, double* coefTH, int flags);

double now_seconds();

}  // namespace kb
