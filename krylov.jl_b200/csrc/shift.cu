// shift.cu -- the shift solvers: cg_lanczos_shift! (src/cg_lanczos_shift.jl:120-294) and cgls_lanczos_shift!
// (src/cgls_lanczos_shift.jl:117-286).  One Lanczos process serves all p shifted systems; the per-shift scalar
// recurrences run on the host in T in the reference's order, and the p updates of x_i and p_i are one streaming pass
// per kShiftPass active shifts (fused_phases.cu: shift_fused_update), or the primitive kaxpy! / kaxpby! per shift with
// fused = 0.  The Lanczos half is CG-Lanczos's grouped passes (CSR operator, M = I) or CGLS-Lanczos-shift's SpMV
// epilogues on A and its cached A^T; otherwise the primitives of blas1.cu / spmv.cu.
#include <algorithm>
#include <cstring>

#include "solver_common.h"

namespace kb {

template <class T> Workspace<T>* shift_ws_create(SolverKind kind, int m, int n, int nshifts, int device) {
  const double t0 = now_seconds();
  if (kind != S_CG_LANCZOS_SHIFT && kind != S_CGLS_LANCZOS_SHIFT) throw std::runtime_error("not a shift solver");
  if (kind == S_CG_LANCZOS_SHIFT && m != n) throw std::runtime_error("System must be square");
  if (nshifts <= 0) throw std::runtime_error("nshifts must be positive");
  Workspace<T>* ws = new Workspace<T>();
  try {
    ws->kind = kind; ws->m = m; ws->n = n; ws->nshifts = nshifts;
    ws->ctx.init(device);
    fused_block_alloc<T>(*ws);
    auto A = [&](int len) { return dev_alloc<T>((size_t)len); };
    ws->Xs = dev_alloc<T>((size_t)n * nshifts);
    ws->Ps = dev_alloc<T>((size_t)n * nshifts);
    if (kind == S_CG_LANCZOS_SHIFT) {          // CgLanczosShiftWorkspace (krylov_workspaces.jl:616-660; v: by the solve)
      ws->Mv = A(n); ws->Mv_prev = A(n); ws->Mv_next = A(n);
    } else {                                   // CglsLanczosShiftWorkspace: v (n), u_prev, u, u_next (m)
      ws->v = A(n); ws->u_prev = A(m); ws->u = A(m); ws->u_next = A(m);
    }
  } catch (...) {
    ws_destroy(ws);
    throw;
  }
  ws->stats.allocation_timer = now_seconds() - t0;
  return ws;
}

// The per-shift half of both solvers (cg_lanczos_shift.jl:227-262, cgls_lanczos_shift.jl:222-254), on the host.
template <class T> struct ShiftSet {
  Workspace<T>& ws;
  const int p;
  const bool check_curvature, track_indefinite;
  std::vector<T> shift, sigma, omega, gamma, rNorms;
  std::vector<unsigned char> converged, not_cv, indefinite;
  std::vector<T*> xs, ps;                      // the columns and scalars of this iteration's active shifts
  std::vector<T> ga, sa, oa;
  T eps_tol = 0;
  ShiftSet(Workspace<T>& w, const T* shifts, bool cc, bool track)
      : ws(w), p(w.nshifts), check_curvature(cc), track_indefinite(track), shift(shifts, shifts + w.nshifts),
        sigma(p), omega(p), gamma(p), rNorms(p), converged(p), not_cv(p), indefinite(p, 0) {}
  T* x(int i) { return ws.Xs + (size_t)i * ws.n; }
  T* pv(int i) { return ws.Ps + (size_t)i * ws.n; }
  void start(T beta, T eps) {
    eps_tol = eps;
    for (int i = 0; i < p; i++) {
      sigma[i] = beta; omega[i] = 0; gamma[i] = 1;
      converged[i] = rNorms[i] <= eps_tol; not_cv[i] = !converged[i];
    }
  }
  bool active(int i) const { return check_curvature ? !(converged[i] || indefinite[i]) : !converged[i]; }
  bool solved() const { for (int i = 0; i < p; i++) if (not_cv[i]) return false; return true; }
  // One iteration: gamma for every shift, then the active shifts' updates.  scale: v still holds beta v.
  void step(T* v, T delta, T rho, T beta, bool scale, bool fused, bool history) {
    for (int i = 0; i < p; i++) {
      const T dhat = delta + rho * shift[i];
      gamma[i] = T(1) / (dhat - omega[i] / gamma[i]);
    }
    if (track_indefinite) for (int i = 0; i < p; i++) indefinite[i] |= gamma[i] <= 0;
    xs.clear(); ps.clear(); ga.clear(); sa.clear(); oa.clear();
    for (int i = 0; i < p; i++) {
      not_cv[i] = active(i);
      if (!not_cv[i]) continue;
      omega[i] = beta * gamma[i];
      sigma[i] = sigma[i] * -omega[i];
      omega[i] = omega[i] * omega[i];
      xs.push_back(x(i)); ps.push_back(pv(i)); ga.push_back(gamma[i]); sa.push_back(sigma[i]); oa.push_back(omega[i]);
      rNorms[i] = std::fabs(sigma[i]);
      converged[i] = rNorms[i] <= eps_tol;
    }
    const int cnt = (int)xs.size();
    if (fused) {
      shift_fused_update<T>(ws, v, scale, beta, cnt, xs.data(), ps.data(), ga.data(), sa.data(), oa.data());
    } else {
      if (scale) k_scal<T>(ws.ctx, ws.n, T(1) / beta, v);
      for (int k = 0; k < cnt; k++) {
        k_axpy<T>(ws.ctx, ws.n, ga[k], ps[k], xs[k]);
        k_axpby<T>(ws.ctx, ws.n, sa[k], v, oa[k], ps[k]);
      }
    }
    if (history)
      for (int i = 0; i < p; i++) if (not_cv[i]) ws.stats.shift_residuals[i].push_back(rNorms[i]);
    for (int i = 0; i < p; i++) not_cv[i] = active(i);
  }
  void display(int iter, int verbose, double t) const {
    if (!kdisplay(iter, verbose)) return;
    printf("%5d", iter);
    for (int i = 0; i < p; i++) printf("  %8.1e", (double)rNorms[i]);
    printf("  %.2fs\n", t);
  }
};

// Common prologue: x_i = 0, and the stats reset to one empty history per shift.
template <class T> static void shift_reset(Workspace<T>& ws) {
  ws.stats.reset();
  ws.stats.shift_residuals.assign(ws.nshifts, {});
  ws.stats.shift_indefinite.assign(ws.nshifts, 0);
  for (int i = 0; i < ws.nshifts; i++) k_fill<T>(ws.ctx, ws.n, ws.Xs + (size_t)i * ws.n, T(0));
}

template <class T> static std::string shift_status(bool tired, bool solved, bool user_exit, bool overtimed) {
  std::string status = "unknown";
  if (tired) status = "maximum number of iterations exceeded";
  if (solved) status = "solution good enough given atol and rtol";
  if (user_exit) status = "user-requested exit";
  if (overtimed) status = "time limit exceeded";
  return status;
}

// ===========================================================================
// cg_lanczos_shift!  (src/cg_lanczos_shift.jl:120-294)
// ===========================================================================
template <class T>
void cg_lanczos_shift_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const T* shifts, const LinOp<T>& M,
                            const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int n = ws.n, p = ws.nshifts;
  const bool history = o.history, ldiv = o.ldiv;
  if (o.verbose > 0) printf("CG-LANCZOS-SHIFT: system of %d equations in %d variables with %d shifts\n", n, n, p);
  const bool MisI = M.is_identity();
  allocate_if(!MisI, ws, ws.vv);
  T *Mv = ws.Mv, *Mv_prev = ws.Mv_prev, *Mv_next = ws.Mv_next;
  T* v = MisI ? Mv : ws.vv;
  auto norm_elliptic = [&]() { return MisI ? k_nrm2<T>(c, n, v) : (T)std::sqrt(k_dot<T>(c, n, v, Mv)); };
  ShiftSet<T> sh(ws, shifts, o.check_curvature, true);
  shift_reset(ws);

  k_copy<T>(c, n, Mv, b);
  if (!MisI) op_apply(c, M, Mv, v, ldiv);
  T beta = norm_elliptic();
  std::fill(sh.rNorms.begin(), sh.rNorms.end(), beta);
  if (history) for (int i = 0; i < p; i++) ws.stats.shift_residuals[i].push_back(beta);
  if (beta == 0) { run.finish(0, true, false, "x is a zero-residual solution"); return; }
  for (int i = 0; i < p; i++) k_copy<T>(c, n, sh.pv(i), v);
  k_scal<T>(c, n, T(1) / beta, v);
  if (!MisI) k_scal<T>(c, n, T(1) / beta, Mv);
  k_copy<T>(c, n, Mv_prev, Mv);
  T rho = 1;
  sh.start(beta, tol_of<T>(o.atol) + tol_of<T>(o.rtol) * beta);
  int iter = 0;
  const int itmax = default_itmax(ws, o.itmax);
  sh.display(iter, o.verbose, run.elapsed());
  bool solved = sh.solved(), tired = iter >= itmax, user_exit = false, overtimed = false;

  // CSR operator, M = I: CG-Lanczos's two grouped passes, then the shift update (which also scales v): 2 + ceil(active /
  // kShiftPass) launches and 2 read-backs per iteration
  const bool fusedL = o.fused && A.kind == LinOp<T>::CSR && MisI;
  while (!(solved || tired || user_exit || overtimed)) {
    T delta;
    if (fusedL) {
      delta = lanczos_fused_delta<T>(ws, *A.csr);
      beta = lanczos_fused_recur<T>(ws, delta, beta, iter > 0);
    } else {
      op_apply(c, A, v, Mv_next);
      delta = k_dot<T>(c, n, v, Mv_next);
      k_axpy<T>(c, n, -delta, Mv, Mv_next);
      if (iter > 0) {
        k_axpy<T>(c, n, -beta, Mv_prev, Mv_next);
        k_copy<T>(c, n, Mv_prev, Mv);
      }
      k_copy<T>(c, n, Mv, Mv_next);
      if (!MisI) op_apply(c, M, Mv, v, ldiv);
      beta = norm_elliptic();
      k_scal<T>(c, n, T(1) / beta, v);
      if (!MisI) k_scal<T>(c, n, T(1) / beta, Mv);
      if (!MisI) rho = k_dot<T>(c, n, v, v);
    }
    sh.step(v, delta, rho, beta, fusedL, o.fused != 0, history);
    iter = iter + 1;
    sh.display(iter, o.verbose, run.elapsed());
    run.poll(iter, user_exit, overtimed);
    solved = sh.solved();
    tired = iter >= itmax;
  }
  if (o.verbose > 0) printf("\n");
  ws.stats.shift_indefinite = sh.indefinite;
  run.finish(iter, solved, false, shift_status<T>(tired, solved, user_exit, overtimed));
}

// ===========================================================================
// cgls_lanczos_shift!  (src/cgls_lanczos_shift.jl:117-286), M = I
// ===========================================================================
template <class T>
void cgls_lanczos_shift_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const T* shifts,
                              const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int m = ws.m, n = ws.n, p = ws.nshifts;
  const bool history = o.history;
  if (o.verbose > 0) printf("CGLS-LANCZOS-SHIFT: system of %d equations in %d variables with %d shifts\n", m, n, p);
  T* v = ws.v;
  ShiftSet<T> sh(ws, shifts, false, false);
  shift_reset(ws);

  k_copy<T>(c, m, ws.u, b);
  k_fill<T>(c, m, ws.u_prev, T(0));
  op_apply(c, At, ws.u, v);
  T beta = k_nrm2<T>(c, n, v);
  std::fill(sh.rNorms.begin(), sh.rNorms.end(), beta);
  if (history) for (int i = 0; i < p; i++) ws.stats.shift_residuals[i].push_back(beta);
  if (beta == 0) { run.finish(0, true, false, "x is a zero-residual solution"); return; }
  for (int i = 0; i < p; i++) k_copy<T>(c, n, sh.pv(i), v);
  k_scal<T>(c, n, T(1) / beta, v);
  // the fused passes keep u unscaled and apply s_u = 1 / beta where they read it; the primitive path scales it here
  const bool fusedG = o.fused && A.kind == LinOp<T>::CSR && At.kind == LinOp<T>::CSR;
  T s_u = T(1) / beta;
  if (!fusedG) k_scal<T>(c, m, s_u, ws.u);
  sh.start(beta, tol_of<T>(o.atol) + tol_of<T>(o.rtol) * beta);
  int iter = 0;
  const long long mn = (long long)m + n;
  const int itmax = o.itmax != 0 ? o.itmax : (int)std::min(mn, 2147483647LL);
  sh.display(iter, o.verbose, run.elapsed());
  bool solved = sh.solved(), tired = iter >= itmax, user_exit = false, overtimed = false;

  // CSR operators: u_next = A v (+ delta), the u pass, v = A^T u_next (+ ||v||^2), then the shift update (which also
  // scales v): 3 + ceil(active / kShiftPass) launches and 2 read-backs per iteration
  while (!(solved || tired || user_exit || overtimed)) {
    T delta;
    if (fusedG) {
      delta = shift_gk_delta<T>(ws, *A.csr);
      beta = std::sqrt(shift_gk_next<T>(ws, *At.csr, s_u, delta, beta));
      std::swap(ws.u, ws.u_next);             // u <- u_next (unscaled), u_prev <- u (written by the u pass)
      s_u = T(1) / beta;
    } else {
      op_apply(c, A, v, ws.u_next);
      delta = k_dot<T>(c, m, ws.u_next, ws.u_next);
      k_axpy<T>(c, m, -delta, ws.u, ws.u_next);
      k_axpy<T>(c, m, -beta, ws.u_prev, ws.u_next);
      op_apply(c, At, ws.u_next, v);
      beta = k_nrm2<T>(c, n, v);
      k_scal<T>(c, n, T(1) / beta, v);
      k_scal<T>(c, m, T(1) / beta, ws.u_next);
      k_copy<T>(c, m, ws.u_prev, ws.u);
      k_copy<T>(c, m, ws.u, ws.u_next);
    }
    sh.step(v, delta, T(1), beta, fusedG, o.fused != 0, history);
    iter = iter + 1;
    sh.display(iter, o.verbose, run.elapsed());
    run.poll(iter, user_exit, overtimed);
    solved = sh.solved();
    tired = iter >= itmax;
  }
  if (o.verbose > 0) printf("\n");
  run.finish(iter, solved, false, shift_status<T>(tired, solved, user_exit, overtimed));
}

#define INST(T)                                                                                                        \
  template Workspace<T>* shift_ws_create<T>(SolverKind, int, int, int, int);                                          \
  template void cg_lanczos_shift_solve<T>(Workspace<T>&, const LinOp<T>&, const T*, const T*, const LinOp<T>&,         \
                                          const SolveOpts&);                                                           \
  template void cgls_lanczos_shift_solve<T>(Workspace<T>&, const LinOp<T>&, const LinOp<T>&, const T*, const T*,      \
                                            const SolveOpts&);
INST(double)
INST(float)
#undef INST

}  // namespace kb
