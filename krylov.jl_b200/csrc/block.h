// block.h -- block Krylov workspace and operator types (block.cu, capi.cu).
#pragma once
#include <vector>

#include "kb_internal.h"

namespace kb {

typedef void (*BlockMatvecFn)(const void* X, void* Y, int p, void* userdata);

template <class T>
struct BlockOp {
  enum Kind { NONE, CSR, DIAG, HOST_CB, DEV_CB } kind = NONE;
  const Csr<T>* csr = nullptr;
  const T* diag = nullptr;
  BlockMatvecFn fn = nullptr;
  void* userdata = nullptr;
  bool is_identity() const { return kind == NONE; }
};

// BlockGmresWorkspace (src/block_krylov_workspaces.jl:108-163).  Device panels are row-major n x p; the small
// blocks Z, R, H, tau, C, D live on the host, column-major, exactly the reference's fields.
template <class T>
struct BlockWorkspace {
  int m = 0, n = 0, p = 0;
  Ctx ctx;
  Stats stats;
  bool warm_start = false;
  int memory = 5;
  T *X = nullptr, *dX = nullptr, *W = nullptr, *P = nullptr, *Q = nullptr;
  std::vector<T*> V;
  std::vector<std::vector<T>> Z, R, H, tau;
  std::vector<T> C, D;
  // scratch
  T *Bbuf = nullptr, *tmp = nullptr, *tmp2 = nullptr;   // staged right-hand side; transposition / callback panels
  T *part = nullptr;                                    // grid x p^2 partial Gram matrices
  T *dG = nullptr, *dS = nullptr;                       // device p x p: last Gram matrix, matrix being applied
  std::vector<T*> dPsi;                                 // device p x p blocks of the current Arnoldi column
  T* hsmall = nullptr;                                  // pinned host staging (p x p blocks): [Gram | top of Q | slots...]
  size_t hsmall_cap = 0;
  T *hX = nullptr, *hY = nullptr;                       // pinned panels for host block callbacks
  int grid = 1;                                         // tiled generic kernels
  int fast_grid = 1;                                    // register-resident kernels (p = 2, 4, 8, 16, 32)
  // panel-kernel choice: set from the environment by block_ws_create (A/B runs, sweeps), overridden for one call by
  // block_panel_op
  bool generic_kernels = false;                         // KB200_BLOCK_GENERIC: the tiled any-p kernels only
  int mma_mode = 1;                                     // KB200_BLOCK_MMA: 0 no DMMA, 16 DMMA for p = 16 / 32 only
  bool fast_prefetch = false;                           // KB200_FAST_PREFETCH: software-pipelined SIMT row loads
  bool fast_alt_tpr = false;                            // KB200_FAST_TPR: second lanes-per-row shape of p = 8 / 16
  long long qr_fallbacks = 0;
};

template <class T> BlockWorkspace<T>* block_ws_create(int m, int n, int p, int memory, int device);
template <class T> void block_ws_destroy(BlockWorkspace<T>* ws);
// B, X0: device panels in the reference's column-major layout (n x p); the solution is read with block_get_X
template <class T> void block_gmres_solve(BlockWorkspace<T>& ws, const BlockOp<T>& A, const T* B_colmajor, const BlockOp<T>& M,
                                          const BlockOp<T>& N, const SolveOpts& o);
template <class T> void block_warm_start(BlockWorkspace<T>& ws, const T* X0_colmajor_dev);
template <class T> void block_get_X(BlockWorkspace<T>& ws, T* X_colmajor_dev);
// Single kernels of the solver, for tests (kb200_spmm_csr, krylov_b200_block_panel_op in krylov_b200.h).  Both
// synchronise before returning and throw on a combination that has no kernel.
template <class T> void block_spmm(Ctx& c, const Csr<T>& A, int p, const T* X, T* Y, int variant);
template <class T> void block_panel_op(BlockWorkspace<T>& ws, int op, int path, int rows, T alpha, const T* In, const T* S, T beta,
                                       T* Out, const T* Next, T* G);

}  // namespace kb
