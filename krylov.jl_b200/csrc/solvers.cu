// solvers.cu -- host control flow of cg!, bicgstab!, minres! and of the one
// Arnoldi driver behind gmres!, fom! and fgmres!, on device vectors.  Each
// driver keeps the reference's scalar recurrences, stopping tests, status
// strings and aliasing rules (files cited per function); every vector operation
// is a kernel from blas1.cu / spmv.cu / fused_phases.cu, nothing is computed on
// the host except O(1)/O(k^2) scalar work the reference also does on the host.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>

#include "solver_common.h"

namespace kb {

// ---------------------------------------------------------------------------
// Workspaces  (src/krylov_workspaces.jl: CgWorkspace :236-291, MinresWorkspace
// :77-141, BicgstabWorkspace :1568-1629, GmresWorkspace :2857-2924)
// ---------------------------------------------------------------------------
template <class T> Workspace<T>* ws_create(SolverKind kind, int m, int n, int memory, int window, int device) {
  const double t0 = now_seconds();
  const SolverInfo* info = solver_info(kind);
  if (m != n && !(info && info->rect)) throw std::runtime_error("System must be square");
  Workspace<T>* ws = new Workspace<T>();
  try {
    ws->kind = kind; ws->m = m; ws->n = n;
    ws->ctx.init(device);
    fused_block_alloc<T>(*ws);
    auto A = [&]() { return dev_alloc<T>((size_t)n); };
    ws->x = A();
    switch (kind) {
      case S_CG: ws->r = A(); ws->p = A(); ws->Ap = A(); cg_fused_prepare<T>(*ws); break;
      case S_BICGSTAB: ws->r = A(); ws->p = A(); ws->v = A(); ws->s = A(); ws->qd = A(); break;
      case S_MINRES:
        ws->r1 = A(); ws->r2 = A(); ws->w1 = A(); ws->w2 = A(); ws->y = A();
        ws->window = window > 0 ? window : 5;
        ws->err_vec.assign(ws->window, T(0));
        break;
      case S_GMRES: case S_FGMRES: case S_FOM: {     // FgmresWorkspace :2983-3003, FomWorkspace :3065-3084
        ws->w = A();
        int mem = memory > 0 ? memory : 20;
        if (mem > m) mem = m;                       // krylov_workspaces.jl:2900
        ws->memory = mem;
        for (int i = 0; i < mem; i++) ws->V.push_back(A());
        if (kind == S_FGMRES) for (int i = 0; i < mem; i++) ws->Z.push_back(A());
        // host-side small arrays: GMRES/FGMRES c, s, z, R; FOM l (sgiv), z (zg), U (R)
        ws->c.assign(mem, T(0)); ws->sgiv.assign(mem, T(0)); ws->zg.assign(mem, T(0));
        ws->R.assign((size_t)mem * (mem + 1) / 2, T(0));
        break;
      }
      case S_CGS: ws->r = A(); ws->u = A(); ws->p = A(); ws->q = A(); ws->ts = A(); break;          // CgsWorkspace :1527-1545
      case S_CR: ws->r = A(); ws->p = A(); ws->q = A(); ws->Ap = A(); break;                        // CrWorkspace :343-360 (Ar == Ap)
      case S_DQGMRES: case S_DIOM: {                // DqgmresWorkspace :832-852, DiomWorkspace :914-933
        ws->t = A();
        int mem = memory > 0 ? memory : 20;
        if (mem > m) mem = m;
        if (kind == S_DIOM && mem < 2) throw std::runtime_error("diom needs memory >= 2");
        ws->memory = mem;
        const int np_ = kind == S_DIOM ? mem - 1 : mem;
        for (int i = 0; i < mem; i++) ws->V.push_back(A());
        for (int i = 0; i < np_; i++) ws->Z.push_back(A());                       // P
        ws->c.assign(mem, T(0));
        ws->sgiv.assign(kind == S_DIOM ? mem - 1 : mem, T(0));                    // s / L
        ws->R.assign(kind == S_DIOM ? mem : mem + 1, T(0));                       // H
        break;
      }
      case S_CG_LANCZOS: ws->Mv = A(); ws->Mv_prev = A(); ws->p = A(); ws->Mv_next = A(); break;    // CgLanczosWorkspace :575-591
      case S_LSQR: case S_LSMR: case S_LSLQ:        // Lsqr / Lsmr / LslqWorkspace: Av, Aᴴu, u, v are allocated by the solve
        ws->Nv = A(); ws->Mu = dev_alloc<T>((size_t)m);
        if (kind != S_LSMR) ws->w = A(); else { ws->h = A(); ws->hbar = A(); }     // LSLQ: w̄ in w
        ws->window = window > 0 ? window : 5;
        ws->err_vec.assign(ws->window, T(0));
        break;
      case S_CGLS:                                  // CglsWorkspace :1916-1944 (Mr is allocated by the solve)
        ws->p = A(); ws->s = A(); ws->r = dev_alloc<T>((size_t)m); ws->q = dev_alloc<T>((size_t)m);
        break;
      case S_CRLS:                                  // CrlsWorkspace :2100-2131 (Ms is allocated by the solve)
        ws->p = A(); ws->Ar = A(); ws->q = A();
        ws->r = dev_alloc<T>((size_t)m); ws->Ap = dev_alloc<T>((size_t)m); ws->s = dev_alloc<T>((size_t)m);
        break;
      case S_BILQ: case S_QMR:                      // BilqWorkspace / QmrWorkspace (t, s are allocated by the solve)
        ws->u_prev = A(); ws->u = A(); ws->q = A(); ws->v_prev = A(); ws->v = A(); ws->p = A();
        if (kind == S_QMR) { ws->w1 = A(); ws->w2 = A(); } else { ws->w = A(); }   // w_{k-2}, w_{k-1} / d̅
        break;
      case S_BILQR: case S_TRILQR: {                // BilqrWorkspace / TrilqrWorkspace (Δx, Δy by warm_start2)
        // TriLQR: x, d̅, u_{k-1}, u_k, p live in the n-space and y, v_{k-1}, v_k, q, w_{k-3}, w_{k-2} in the m-space.  p
        // has max(m, n) entries: the cached A^T has that many rows (the fused T2 pass covers every row of q with them).
        auto Am = [&]() { return dev_alloc<T>((size_t)m); };
        ws->u_prev = A(); ws->u = A(); ws->w = A(); ws->p = dev_alloc<T>((size_t)std::max(m, n));
        ws->v_prev = Am(); ws->v = Am(); ws->q = Am(); ws->y = Am(); ws->w1 = Am(); ws->w2 = Am();
        break;
      }
      case S_CGNE: case S_CRMR:                     // CgneWorkspace / CrmrWorkspace: Aᴴz / Aᴴr in Ar (s, z / Nq: by the solve)
        ws->p = A(); ws->Ar = A(); ws->r = dev_alloc<T>((size_t)m); ws->q = dev_alloc<T>((size_t)m);
        break;
      case S_CRAIG: case S_CRAIGMR: {               // CraigWorkspace / CraigmrWorkspace (Av, Aᴴu, u, v, w2 / q: by the solve)
        auto Am = [&]() { return dev_alloc<T>((size_t)m); };
        ws->Nv = A(); ws->Mu = Am(); ws->y = Am(); ws->w = Am();
        if (kind == S_CRAIGMR) { ws->d1 = A(); ws->w1 = Am(); }   // d, w̄
        break;
      }
      case S_LNLQ: {                                // LnlqWorkspace: w̄ in w (Av, Aᴴu, u, v, q: by the solve)
        auto Am = [&]() { return dev_alloc<T>((size_t)m); };
        ws->Nv = A(); ws->Mu = Am(); ws->y = Am(); ws->w = Am();
        break;
      }
      case S_CAR:                                   // CarWorkspace (Mu is allocated by the solve)
        ws->r = A(); ws->p = A(); ws->s = A(); ws->q = A(); ws->t = A(); ws->u = A();
        break;
      case S_MINARES:                               // MinaresWorkspace: v_k, v_{k+1}, w_{k-2}, w_{k-1}, d_{k-2}, d_{k-1}, q
        ws->v = A(); ws->vv = A(); ws->w2 = A(); ws->w1 = A(); ws->d2 = A(); ws->d1 = A(); ws->q = A();
        break;
      default: throw std::runtime_error("unsupported solver");
    }
  } catch (...) {
    ws_destroy(ws);
    throw;
  }
  ws->stats.allocation_timer = now_seconds() - t0;
  return ws;
}

template <class T> void ws_destroy(Workspace<T>* ws) {
  if (!ws) return;
  if (ws->ctx.stream) cudaStreamSynchronize(ws->ctx.stream);
  T* vecs[] = {ws->x, ws->dx, ws->r, ws->p, ws->Ap, ws->z, ws->npc_dir, ws->p2, ws->v, ws->s, ws->qd, ws->t, ws->yz,
               ws->r1, ws->r2, ws->w1, ws->w2, ws->y, ws->vv, ws->w, ws->q, ws->pp, ws->bbuf, ws->cbuf,
               ws->u, ws->ts, ws->vw, ws->Mv, ws->Mv_prev, ws->Mv_next, ws->Nv, ws->Mu, ws->Av, ws->Atu, ws->h, ws->hbar,
               ws->Ar, ws->Mr, ws->u_prev, ws->v_prev, ws->d1, ws->d2, ws->dy, ws->Xs, ws->Ps, ws->u_next};
  for (T* p : vecs) dev_free(p);
  for (T* p : ws->V) dev_free(p);
  for (T* p : ws->Z) dev_free(p);
  if (ws->fused_state) cudaFree(ws->fused_state);
  if (ws->fused_host) cudaFreeHost(ws->fused_host);
  for (auto& e : ws->fused_ev) if (e) cudaEventDestroy(e);
  if (ws->dist.tile_order) cudaFree(ws->dist.tile_order);
  for (void* p : ws->dist.opened) cudaIpcCloseMemHandle(p);
  if (ws->dist.mailbox) cudaFree(ws->dist.mailbox);
  dev_free(ws->dist.halo_buf);
  dev_free(ws->dist.xhalo);
  for (void* d : ws->dist.dummy) if (d) cudaFree(d);
  if (ws->dist.send_row) cudaFree(ws->dist.send_row);
  if (ws->dist.send_peer) cudaFree(ws->dist.send_peer);
  if (ws->dist.send_slot) cudaFree(ws->dist.send_slot);
  delete ws->ctx.dex; ws->ctx.dex = nullptr;
  if (ws->dist.halo.src_rank) cudaFree((void*)ws->dist.halo.src_rank);
  if (ws->dist.halo.src_off) cudaFree((void*)ws->dist.halo.src_off);
  if (ws->ctx.dcomm) cudaFree(ws->ctx.dcomm);
  ws->ctx.destroy();
  delete ws;
}

// warm_start! (src/workspace_accessors.jl:193-200)
template <class T> void ws_warm_start(Workspace<T>* ws, const T* x0_dev) {
  allocate_if(true, *ws, ws->dx);
  k_copy<T>(ws->ctx, ws->n, ws->dx, x0_dev);
  ws->warm_start = true;
}

// ===========================================================================
// cg!  (src/cg.jl:120-291)
// ===========================================================================
template <class T>
void cg_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int n = ws.n;
  const T radius = (T)o.radius;
  const bool linesearch = o.linesearch, history = o.history, ldiv = o.ldiv;
  if (linesearch && radius > 0) throw std::runtime_error("`linesearch` set to `true` but trust-region radius > 0");
  if (ws.warm_start && linesearch) throw std::runtime_error("warm_start and linesearch cannot be used together");
  if (o.verbose > 0) printf("CG: system of %d equations in %d variables\n", n, n);
  const bool MisI = M.is_identity();
  allocate_if(!MisI, ws, ws.z);
  allocate_if(linesearch || radius > 0, ws, ws.npc_dir);
  T *dx = ws.dx, *x = ws.x, *r = ws.r, *Ap = ws.Ap;
  Stats& stats = ws.stats;
  const bool warm_start = ws.warm_start;
  stats.reset();
  T* z = MisI ? r : ws.z;                                    // cg.jl:148

  T gamma;
  if (!warm_start && MisI && ws.dist.npush == 0) {
    gamma = k_cg_prologue<T>(c, n, b, x, r, ws.p);          // x = 0, r = b, p = z = r, gamma = <r, z> in one pass
  } else {
    k_fill<T>(c, n, x, T(0));
    if (warm_start) {
      op_apply(c, A, dx, r);
      k_axpby<T>(c, n, T(1), b, T(-1), r);
    } else {
      k_copy<T>(c, n, r, b);
    }
    cg_dist_push_r<T>(ws);                                  // row-partitioned push mode: neighbours' halo copy of r_0
    if (!MisI) op_apply(c, M, r, z, ldiv);
    k_copy<T>(c, n, ws.p, z);
    gamma = k_dot<T>(c, n, r, z);
  }
  if (!(gamma >= 0)) throw std::runtime_error("The linear operator `A` or the preconditioner `M` is not symmetric positive definite.");
  T rNorm = std::sqrt(gamma);
  if (history) stats.residuals.push_back(rNorm);
  if (gamma == 0) { run.finish(0, true, false, "x is a zero-residual solution"); return; }
  int iter = 0;
  int itmax = default_itmax(ws, o.itmax);
  T pAp = 0, pNorm2 = gamma;
  const T eps_tol = tol_of<T>(o.atol) + tol_of<T>(o.rtol) * rNorm;     // cg.jl:181
  if (o.verbose > 0) printf("%5s  %7s  %8s  %8s  %8s  %5s\n", "k", "‖r‖", "pAp", "α", "σ", "timer");
  if (kdisplay(iter, o.verbose)) printf("%5d  %7.1e", iter, (double)rNorm);
  bool solved = rNorm <= eps_tol, tired = iter >= itmax;
  bool inconsistent = false, on_boundary = false, zero_curvature = false, user_exit = false, overtimed = false;
  std::string status = "unknown";

  const CgFusedPlan<T> plan = (solved || tired) ? CgFusedPlan<T>() : cg_fused_plan<T>(ws, A, M, o);
  if (plan.fused) {
    const CgFusedExit e = cg_fused_loop<T>(ws, plan, o, gamma, eps_tol, itmax, run.start);
    iter = e.iter;
    solved = e.solved; tired = e.tired; zero_curvature = e.zero_curvature; inconsistent = e.inconsistent;
    user_exit = e.user_exit; overtimed = e.overtimed;
  } else {
    T* p = ws.p;
    while (!(solved || tired || zero_curvature || user_exit || overtimed)) {
      op_apply(c, A, p, Ap);
      pAp = k_dot<T>(c, n, p, Ap);
      if ((pAp <= eps_of<T>() * pNorm2) && (radius == 0)) {
        if (std::fabs(pAp) <= eps_of<T>() * pNorm2) { zero_curvature = true; inconsistent = !linesearch; }
        if (linesearch) {
          if (iter == 0) k_copy<T>(c, n, x, p);
          k_copy<T>(c, n, ws.npc_dir, p);
          stats.npcCount = 1; stats.indefinite = true; solved = true;
        }
      }
      if (zero_curvature || solved) continue;
      T alpha = gamma / pAp, sigma;
      if (radius == 0) {
        sigma = alpha;
      } else {
        T s1, s2;
        int e = MisI ? to_boundary<T>(c, n, x, p, z, radius, pNorm2, M, false, &s1, &s2)
                     : to_boundary<T>(c, n, x, p, z, radius, T(0), M, !ldiv, &s1, &s2);
        if (e == 2) throw std::runtime_error("zero direction");
        if (e == 3) throw std::runtime_error("outside of the trust region");
        if (e) throw std::runtime_error("The quadratic `q` doesn't have real roots.");
        sigma = s1 > s2 ? s1 : s2;
      }
      if (kdisplay(iter, o.verbose))
        printf("  %8.1e  %8.1e  %8.1e  %.2fs\n", (double)pAp, (double)alpha, (double)sigma, run.elapsed());
      if ((radius > 0) && ((pAp <= 0) || (alpha > sigma))) {
        alpha = sigma;
        if (pAp <= 0) { k_copy<T>(c, n, ws.npc_dir, p); stats.npcCount = 1; stats.indefinite = true; }
        on_boundary = true;
      }
      k_axpy<T>(c, n, alpha, p, x);
      k_axpy<T>(c, n, -alpha, Ap, r);
      if (!MisI) op_apply(c, M, r, z, ldiv);
      T gamma_next = k_dot<T>(c, n, r, z);
      if (!(gamma_next >= 0)) throw std::runtime_error("The linear operator `A` or the preconditioner `M` is not symmetric positive definite.");
      rNorm = std::sqrt(gamma_next);
      if (history) stats.residuals.push_back(rNorm);
      const bool resid_decrease_mach = (rNorm + T(1) <= T(1));
      const bool resid_decrease_lim = rNorm <= eps_tol;
      solved = resid_decrease_lim || resid_decrease_mach || on_boundary;
      if (!solved) {
        const T beta = gamma_next / gamma;
        pNorm2 = gamma_next + beta * beta * pNorm2;
        gamma = gamma_next;
        k_axpby<T>(c, n, T(1), z, beta, p);
      }
      iter = iter + 1;
      tired = iter >= itmax;
      run.poll(iter, user_exit, overtimed);
      if (kdisplay(iter, o.verbose)) printf("%5d  %7.1e", iter, (double)rNorm);
    }
  }
  if (o.verbose > 0) printf("\n\n");
  if (solved && on_boundary) status = "on trust-region boundary";
  if (solved && stats.indefinite) status = "nonpositive curvature";
  if (solved && status == "unknown") status = "solution good enough given atol and rtol";
  if (zero_curvature) status = "zero curvature detected";
  if (tired) status = "maximum number of iterations exceeded";
  if (user_exit) status = "user-requested exit";
  if (overtimed) status = "time limit exceeded";
  run.finish(iter, solved, inconsistent, status);
}

// ===========================================================================
// bicgstab!  (src/bicgstab.jl:125-277)
// ===========================================================================
template <class T>
void bicgstab_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const T* c_in, const LinOp<T>& M, const LinOp<T>& N,
                    const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int n = ws.n;
  const bool history = o.history, ldiv = o.ldiv;
  if (o.verbose > 0) printf("BICGSTAB: system of size %d\n", n);
  const bool MisI = M.is_identity(), NisI = N.is_identity();
  allocate_if(!MisI, ws, ws.t);
  allocate_if(!NisI, ws, ws.yz);
  T *dx = ws.dx, *x = ws.x, *r = ws.r, *p = ws.p, *v = ws.v, *s = ws.s;
  Stats& stats = ws.stats;
  const bool warm_start = ws.warm_start;
  stats.reset();
  T* q = ws.qd; T* d = ws.qd;                                // bicgstab.jl:153-157
  T* t = MisI ? d : ws.t;
  T* y = NisI ? p : ws.yz;
  T* z = NisI ? s : ws.yz;
  T* r0 = MisI ? r : ws.qd;
  const T* cvec = c_in ? c_in : b;

  if (warm_start) { op_apply(c, A, dx, r0); k_axpby<T>(c, n, T(1), b, T(-1), r0); }
  else k_copy<T>(c, n, r0, b);
  k_fill<T>(c, n, x, T(0)); k_fill<T>(c, n, s, T(0)); k_fill<T>(c, n, v, T(0));
  if (!MisI) op_apply(c, M, r0, r, ldiv);
  k_copy<T>(c, n, p, r);
  T alpha = 1, omega = 1, rho = 1;
  T rNorm = k_nrm2<T>(c, n, r);
  if (history) stats.residuals.push_back(rNorm);
  if (rNorm == 0) { run.finish(0, true, false, "x is a zero-residual solution"); return; }
  int iter = 0;
  const int itmax = default_itmax(ws, o.itmax);
  const T eps_tol = tol_of<T>(o.atol) + tol_of<T>(o.rtol) * rNorm;
  if (o.verbose > 0) printf("%5s  %7s  %8s  %8s  %5s\n", "k", "‖rₖ‖", "|αₖ|", "|ωₖ|", "timer");
  if (kdisplay(iter, o.verbose)) printf("%5d  %7.1e  %8.1e  %8.1e  %.2fs\n", iter, (double)rNorm, 1.0, 1.0, run.elapsed());
  T next_rho = k_dot<T>(c, n, cvec, r);
  if (next_rho == 0) { run.finish(0, false, false, "Breakdown bᴴc = 0"); return; }
  bool solved = rNorm <= eps_tol, tired = iter >= itmax, breakdown = false, user_exit = false, overtimed = false;
  std::string status = "unknown";
  const bool fusedB = o.fused && A.kind == LinOp<T>::CSR && NisI && (MisI || (M.kind == LinOp<T>::DIAG && !ldiv));
  ws.mdiag_fused = (fusedB && !MisI) ? M.diag : nullptr;     // Jacobi M rides in the SpMV epilogues

  while (!(solved || tired || breakdown || user_exit || overtimed)) {
    iter = iter + 1;
    rho = next_rho;
    if (fusedB) {
      // 5 launches, scalars chained on the device, one read-back (fused_phases.cu)
      bicgstab_fused_iteration<T>(ws, *A.csr, cvec, iter == 1, rho, &alpha, &omega, &next_rho, &rNorm);
    } else {
    if (!NisI) op_apply(c, N, p, y, ldiv);
    op_apply(c, A, y, q);
    if (MisI) k_copy<T>(c, n, v, q); else op_apply(c, M, q, v, ldiv);    // bicgstab.jl:222 (unguarded mulorldiv!)
    alpha = rho / k_dot<T>(c, n, cvec, v);
    k_copy<T>(c, n, s, r);
    k_axpy<T>(c, n, -alpha, v, s);
    k_axpy<T>(c, n, alpha, y, x);
    if (!NisI) op_apply(c, N, s, z, ldiv);
    op_apply(c, A, z, d);
    if (!MisI) op_apply(c, M, d, t, ldiv);
    { T ts, tt; k_dot2<T>(c, n, t, s, t, t, &ts, &tt); omega = ts / tt; }
    k_axpy<T>(c, n, omega, z, x);
    k_copy<T>(c, n, r, s);
    k_axpy<T>(c, n, -omega, t, r);
    next_rho = k_dot<T>(c, n, cvec, r);
    const T beta = (next_rho / rho) * (alpha / omega);
    k_axpy<T>(c, n, -omega, v, p);
    k_axpby<T>(c, n, T(1), r, beta, p);
    rNorm = k_nrm2<T>(c, n, r);
    }
    if (history) stats.residuals.push_back(rNorm);
    const bool resid_decrease_mach = (rNorm + T(1) <= T(1));
    run.poll(iter, user_exit, overtimed);
    solved = (rNorm <= eps_tol) || resid_decrease_mach;
    tired = iter >= itmax;
    breakdown = (alpha == 0 || std::isnan(alpha));
    if (kdisplay(iter, o.verbose))
      printf("%5d  %7.1e  %8.1e  %8.1e  %.2fs\n", iter, (double)rNorm, (double)std::fabs(alpha), (double)std::fabs(omega), run.elapsed());
  }
  if (o.verbose > 0) printf("\n");
  if (tired) status = "maximum number of iterations exceeded";
  if (breakdown) status = "breakdown αₖ == 0";
  if (solved) status = "solution good enough given atol and rtol";
  if (user_exit) status = "user-requested exit";
  if (overtimed) status = "time limit exceeded";
  run.finish(iter, solved, false, status);
}

// ---------------------------------------------------------------------------
// gmres!, fom! and fgmres! are one driver: the restart cycle, MGS with optional reorthogonalization, the fused
// Arnoldi step, memory growth, the back substitution and the x update are shared.  They differ in the small
// factorization of H kept on the host (Givens QR: GMRES, FGMRES; LU without pivoting: FOM) and in where the right
// preconditioner lives (FGMRES stores Z[k] = N_k V[k]; GMRES and FOM apply N through pp).  The differences are marked.
//   gmres!   src/gmres.jl:121-384
//   fom!     src/fom.jl:121-368
//   fgmres!  src/fgmres.jl:128-388
// ---------------------------------------------------------------------------
enum class Arnoldi { GMRES, FOM, FGMRES };

template <class T, Arnoldi K>
static void arnoldi_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const LinOp<T>& N, const SolveOpts& o) {
  constexpr bool QR = K != Arnoldi::FOM;          // Givens QR of H (else LU)
  constexpr bool FLEX = K == Arnoldi::FGMRES;     // right preconditioner kept in Z[k]
  SolveRun<T> run(ws, o);
  Ctx& cx = ws.ctx;
  const int n = ws.n;
  const bool history = o.history, ldiv = o.ldiv, restart = o.restart, reorth = o.reorthogonalization;
  if (o.verbose > 0) printf("%s: system of size %d\n", K == Arnoldi::GMRES ? "GMRES" : FLEX ? "FGMRES" : "FOM", n);
  const bool MisI = M.is_identity(), NisI = N.is_identity();
  allocate_if(!MisI, ws, ws.q);
  if (!FLEX) allocate_if(!NisI, ws, ws.pp);
  allocate_if(restart, ws, ws.dx);
  T *dx = ws.dx, *x = ws.x, *w = ws.w;
  std::vector<T*>& V = ws.V;
  std::vector<T*>& Z = ws.Z;
  // QR: c, s (sgiv), z (zg), R.   FOM: l (sgiv), z (zg), U (R); c is unused.
  std::vector<T>&c = ws.c, &s = ws.sgiv, &z = ws.zg, &R = ws.R;
  std::vector<T>& l = ws.sgiv;
  Stats& stats = ws.stats;
  const bool warm_start = ws.warm_start;
  stats.reset();
  T* q = MisI ? w : ws.q;                                     // gmres.jl:150-152
  T* r0 = MisI ? w : ws.q;
  T* xr = restart ? dx : x;

  k_fill<T>(cx, n, x, T(0));
  if (warm_start) {
    op_apply(cx, A, dx, w);
    k_axpby<T>(cx, n, T(1), b, T(-1), w);
    if (restart) k_axpy<T>(cx, n, T(1), dx, x);
  } else {
    k_copy<T>(cx, n, w, b);
  }
  if (!MisI) op_apply(cx, M, w, r0, ldiv);
  T beta = k_nrm2<T>(cx, n, r0);
  T rNorm = beta;
  if (history) stats.residuals.push_back(beta);
  const T eps_tol = tol_of<T>(o.atol) + tol_of<T>(o.rtol) * rNorm;
  if (beta == 0) { run.finish(0, true, false, "x is a zero-residual solution"); return; }
  const int mem = (int)s.size();                              // length(c) / length(l)
  int npass = 0, iter = 0, inner_iter = 0;
  const int itmax = default_itmax(ws, o.itmax);
  int inner_itmax = itmax;
  if (o.verbose > 0) printf("%5s  %5s  %7s  %7s  %5s\n", "pass", "k", "‖rₖ‖", "hₖ₊₁.ₖ", "timer");
  if (kdisplay(iter, o.verbose)) printf("%5d  %5d  %7.1e  %7s  %.2fs\n", npass, iter, (double)rNorm, "✗ ✗ ✗ ✗", run.elapsed());
  const T btol = std::pow(eps_of<T>(), T(0.75));              // gmres.jl:195
  // the fused Arnoldi step folds a left diagonal M into the SpMV epilogue; GMRES and FOM need N = I (FGMRES
  // materialises Z[k])
  const bool fusedA = o.fused && A.kind == LinOp<T>::CSR && !reorth && (FLEX || NisI) &&
                      (MisI || (M.kind == LinOp<T>::DIAG && !ldiv));
  ws.mdiag_fused = (fusedA && !MisI) ? M.diag : nullptr;
  bool breakdown = false, inconsistent = false, solved = rNorm <= eps_tol, tired = iter >= itmax;
  bool inner_tired = inner_iter >= inner_itmax, user_exit = false, overtimed = false;
  std::string status = "unknown";

  while (!(solved || tired || breakdown || user_exit || overtimed)) {
    int nr = 0;
    // The reference zero-fills V (and Z) every cycle.  GMRES and FGMRES read only entries they wrote first (V[1] by
    // kdivcopy!, V[k+1] at the end of step k), so the fill is kept only where callbacks could see unused columns.
    // FOM does read a zero V[k+1] after a user exit or timeout (its inner loop does not test them, fom.jl:237), so
    // FOM always fills.
    if (!restart || !QR) for (int i = 0; i < mem; i++) { k_fill<T>(cx, n, V[i], T(0)); if (FLEX) k_fill<T>(cx, n, Z[i], T(0)); }
    std::fill(s.begin(), s.end(), T(0));
    if (QR) std::fill(c.begin(), c.end(), T(0));
    std::fill(R.begin(), R.end(), T(0));
    std::fill(z.begin(), z.end(), T(0));
    if (restart) {
      k_fill<T>(cx, n, xr, T(0));
      if (npass >= 1) {
        op_apply(cx, A, x, w);
        k_axpby<T>(cx, n, T(1), b, T(-1), w);
        if (!MisI) op_apply(cx, M, w, r0, ldiv);
      }
    }
    beta = k_nrm2<T>(cx, n, r0);
    z[0] = beta;
    k_divcopy<T>(cx, n, V[0], r0, rNorm);                     // gmres.jl:231 (divides by rNorm)
    npass = npass + 1;
    ws.inner_iter = 0;
    inner_tired = false;

    // fom.jl:237 tests only solved/inner_tired/breakdown; gmres! and fgmres! (fgmres.jl:243) also the user exit and the timer
    while (!(solved || inner_tired || breakdown || (QR && (user_exit || overtimed)))) {
      ws.inner_iter = ws.inner_iter + 1;
      inner_iter = ws.inner_iter;
      if (!restart && (inner_iter > mem)) {                   // gmres.jl:244-252
        const double t0 = now_seconds();
        for (int i = 0; i < inner_iter; i++) R.push_back(T(0));
        s.push_back(T(0));                                    // s / FOM l
        if (QR) c.push_back(T(0));
        if (FLEX) Z.push_back(dev_alloc<T>((size_t)n));
        if (!QR) z.push_back(T(0));                           // fom.jl:249 grows z here, gmres.jl / fgmres.jl with V
        stats.allocation_timer += now_seconds() - t0;
      }
      if (!QR && inner_iter > (int)V.size()) {
        // FOM past `memory` after a user exit or timeout: its inner loop runs one more step (fom.jl:237), on a
        // V[k] the previous step did not form.  Give it the zero column it has within `memory`.
        V.push_back(dev_alloc<T>((size_t)n));
        k_fill<T>(cx, n, V.back(), T(0));
      }
      T* vk = V[inner_iter - 1];
      T* p;
      if (FLEX) {                                             // z_k <- N_k v_k, unconditional (fgmres.jl:262)
        p = Z[inner_iter - 1];
        if (NisI) k_copy<T>(cx, n, p, vk); else op_apply(cx, N, vk, p, ldiv);
      } else {
        p = NisI ? vk : ws.pp;
        if (!NisI) op_apply(cx, N, vk, p, ldiv);
      }
      T Hbis;
      if (fusedA && inner_iter <= gmres_fused_max()) {
        // 1 + k launches: SpMV fused with the first MGS dot, then one launch per MGS step that applies
        // q -= h_i v_i and accumulates the next dot (or ||q||^2); one read-back of the whole R column.
        gmres_fused_arnoldi<T>(ws, *A.csr, inner_iter, &R[nr], &Hbis, p);
      } else {
        op_apply(cx, A, p, w);
        if (!MisI) op_apply(cx, M, w, q, ldiv);
        for (int i = 0; i < inner_iter; i++) {                // MGS, gmres.jl:259-262
          R[nr + i] = k_dot<T>(cx, n, V[i], q);
          k_axpy<T>(cx, n, -R[nr + i], V[i], q);
        }
        if (reorth) {
          for (int i = 0; i < inner_iter; i++) {
            const T Htmp = k_dot<T>(cx, n, V[i], q);
            R[nr + i] += Htmp;
            k_axpy<T>(cx, n, -Htmp, V[i], q);
          }
        }
        Hbis = k_nrm2<T>(cx, n, q);
      }
      T zeta_next = 0;
      if (QR) {                                               // Givens QR of H, gmres.jl:280-284 / fgmres.jl:285-303
        for (int i = 0; i < inner_iter - 1; i++) {
          const T Rtmp = c[i] * R[nr + i] + s[i] * R[nr + i + 1];
          R[nr + i + 1] = s[i] * R[nr + i] - c[i] * R[nr + i + 1];
          R[nr + i] = Rtmp;
        }
        sym_givens<T>(R[nr + inner_iter - 1], Hbis, &c[inner_iter - 1], &s[inner_iter - 1], &R[nr + inner_iter - 1]);
        zeta_next = s[inner_iter - 1] * z[inner_iter - 1];
        z[inner_iter - 1] = c[inner_iter - 1] * z[inner_iter - 1];
        rNorm = std::fabs(zeta_next);
      } else {                                                // LU of H without pivoting, fom.jl:274-288
        if (inner_iter >= 2) {
          for (int i = 2; i <= inner_iter; i++) R[nr + i - 1] = R[nr + i - 1] - l[i - 2] * R[nr + i - 2];
          z[inner_iter - 1] = -l[inner_iter - 2] * z[inner_iter - 2];
        }
        l[inner_iter - 1] = Hbis / R[nr + inner_iter - 1];
        rNorm = Hbis * std::fabs(z[inner_iter - 1] / R[nr + inner_iter - 1]);
      }
      if (history) stats.residuals.push_back(rNorm);
      nr = nr + inner_iter;
      const bool resid_decrease_mach = (rNorm + T(1) <= T(1));
      run.poll(iter + inner_iter, user_exit, overtimed);
      const bool resid_decrease_lim = rNorm <= eps_tol;
      breakdown = Hbis <= btol;
      solved = resid_decrease_lim || resid_decrease_mach;
      inner_tired = restart ? inner_iter >= std::min(mem, inner_itmax) : inner_iter >= inner_itmax;
      if (kdisplay(iter + inner_iter, o.verbose))
        printf("%5d  %5d  %7.1e  %7.1e  %.2fs\n", npass, iter + inner_iter, (double)rNorm, (double)Hbis, run.elapsed());
      if (!(solved || inner_tired || breakdown || user_exit || overtimed)) {   // gmres.jl:318-327
        if (!restart && (inner_iter >= mem)) {
          const double t0 = now_seconds();
          V.push_back(dev_alloc<T>((size_t)n));
          if (QR) z.push_back(T(0));
          stats.allocation_timer += now_seconds() - t0;
        }
        k_divcopy<T>(cx, n, V[inner_iter], q, Hbis);
        if (QR) z[inner_iter] = zeta_next;
      }
    }
    std::vector<T>& y = z;                                    // back substitution, gmres.jl:331-345 / fom.jl:322-331
    for (int i = inner_iter; i >= 1; i--) {
      int pos = nr + i - inner_iter;                          // 1-based
      for (int j = inner_iter; j >= i + 1; j--) {
        y[i - 1] = y[i - 1] - R[pos - 1] * y[j - 1];
        pos = pos - j + 1;
      }
      if (QR && std::fabs(R[pos - 1]) <= btol) { y[i - 1] = T(0); inconsistent = true; }
      else y[i - 1] = y[i - 1] / R[pos - 1];
    }
    T* const* basis = FLEX ? Z.data() : V.data();             // x_k = Z_k y_k (FGMRES) or N V_k y_k (GMRES, FOM)
    if (fusedA) fused_multi_axpy<T>(ws, xr, inner_iter, y.data(), basis);   // same sums, same order, one pass per 8 vectors
    else for (int i = 0; i < inner_iter; i++) k_axpy<T>(cx, n, y[i], basis[i], xr);
    if (!FLEX && !NisI) { k_copy<T>(cx, n, ws.pp, xr); op_apply(cx, N, ws.pp, xr, ldiv); }
    if (restart) k_axpy<T>(cx, n, T(1), xr, x);
    inner_itmax = inner_itmax - inner_iter;
    iter = iter + inner_iter;
    tired = iter >= itmax;
    run.poll(iter, user_exit, overtimed, false);             // the clock only: the callback ran in the inner loop
  }
  if (o.verbose > 0) printf("\n");
  if (tired) status = "maximum number of iterations exceeded";
  if (!QR && breakdown) status = "inconsistent linear system";
  if (solved) status = "solution good enough given atol and rtol";
  if (QR && inconsistent) status = "found approximate least-squares solution";
  if (user_exit) status = "user-requested exit";
  if (overtimed) status = "time limit exceeded";
  run.finish(iter, solved, QR ? inconsistent : (!solved && breakdown), status, !restart);
}

template <class T>
void gmres_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const LinOp<T>& N, const SolveOpts& o) {
  arnoldi_solve<T, Arnoldi::GMRES>(ws, A, b, M, N, o);
}
template <class T>
void fom_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const LinOp<T>& N, const SolveOpts& o) {
  arnoldi_solve<T, Arnoldi::FOM>(ws, A, b, M, N, o);
}
template <class T>
void fgmres_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const LinOp<T>& N, const SolveOpts& o) {
  arnoldi_solve<T, Arnoldi::FGMRES>(ws, A, b, M, N, o);
}

// ===========================================================================
// minres!  (src/minres.jl:164-485)
// ===========================================================================
template <class T>
void minres_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int n = ws.n;
  const bool history = o.history, ldiv = o.ldiv, linesearch = o.linesearch;
  if (o.verbose > 0) printf("MINRES: system of size %d\n", n);
  if (ws.warm_start && linesearch) throw std::runtime_error("warm_start and linesearch cannot be used together");
  const bool MisI = M.is_identity();
  allocate_if(!MisI, ws, ws.vv);
  allocate_if(linesearch, ws, ws.npc_dir);
  T *dx = ws.dx, *x = ws.x, *r1 = ws.r1, *r2 = ws.r2, *y = ws.y;
  std::vector<T>& err_vec = ws.err_vec;
  Stats& stats = ws.stats;
  const bool warm_start = ws.warm_start;
  stats.reset();
  T* v = MisI ? r2 : ws.vv;                                   // minres.jl:193
  T* npc_dir = ws.npc_dir;
  const T epsM = eps_of<T>();
  const T conlim = o.conlim < 0 ? T(1) / std::sqrt(eps_of<T>()) : (T)o.conlim;
  const T ctol = conlim > 0 ? T(1) / conlim : T(0);
  const T etol = tol_of<T>(o.etol), rtol = tol_of<T>(o.rtol), atol = tol_of<T>(o.atol);
  const T lambda = (T)o.lambda;
  (void)rtol;

  k_fill<T>(c, n, x, T(0));
  if (warm_start) {
    op_apply(c, A, dx, r1);
    if (lambda != 0) k_axpy<T>(c, n, lambda, dx, r1);
    k_axpby<T>(c, n, T(1), b, T(-1), r1);
  } else {
    k_copy<T>(c, n, r1, b);
  }
  k_copy<T>(c, n, r2, r1);
  if (!MisI) op_apply(c, M, r1, v, ldiv);
  if (linesearch) k_copy<T>(c, n, npc_dir, v);
  T beta1 = k_dot<T>(c, n, r1, v);
  if (beta1 < 0) throw std::runtime_error("Preconditioner is not positive definite");
  if (beta1 == 0) {                                           // minres.jl:220-231
    if (history) { stats.residuals.push_back(beta1); stats.Aresiduals.push_back(0); stats.Acond.push_back(0); }
    run.finish(1, true, false, "x is a zero-residual solution");
    return;
  }
  beta1 = std::sqrt(beta1);
  T beta = beta1, oldbeta = 0, deltabar = 0, eps_rot = 0, rNorm = beta1;
  if (history) stats.residuals.push_back(beta1);
  T phibar = beta1, rhs1 = beta1, rhs2 = 0, gmax = 0, gmin = std::numeric_limits<T>::infinity();
  T cs = -1, sn = 0;
  k_fill<T>(c, n, ws.w1, T(0));
  k_fill<T>(c, n, ws.w2, T(0));
  T ANorm2 = 0, ANorm = 0, Acond = 0, ArNorm = 0, xNorm = 0;
  if (history) stats.Acond.push_back(Acond);
  if (history) stats.Aresiduals.push_back(ArNorm);
  T xENorm2 = 0, err_lbnd = 0;
  const int window = (int)err_vec.size();
  std::fill(err_vec.begin(), err_vec.end(), T(0));
  int iter = 0;
  const int itmax = default_itmax(ws, o.itmax);
  if (o.verbose > 0)
    printf("%5s  %7s  %7s  %7s  %8s  %8s  %7s  %7s  %7s  %7s  %5s\n", "k", "‖r‖", "‖Aᴴr‖", "β", "cos", "sin", "‖A‖", "κ(A)", "test1", "test2", "timer");
  const T eps_tol = atol + tol_of<T>(o.rtol) * beta1;        // minres.jl:269
  bool solved = false, solved_mach = false, solved_lim = false, tired = iter >= itmax;
  bool ill_cond = false, ill_cond_mach = false, ill_cond_lim = false;
  bool zero_resid = (rNorm <= eps_tol), zero_resid_mach = zero_resid, zero_resid_lim = zero_resid;
  bool fwd_err = false, user_exit = false, overtimed = false;
  stats.indefinite = false;
  T delta_w = 0, beta_w = 0, zeta_k = 0, zeta_km1 = 0;
  std::string status = "unknown";
  const bool fusedM = o.fused && A.kind == LinOp<T>::CSR && !linesearch && (MisI || (M.kind == LinOp<T>::DIAG && !ldiv));
  ws.mdiag_fused = (fusedM && !MisI) ? M.diag : nullptr;

  while (!(solved || tired || ill_cond || user_exit || overtimed)) {
    iter = iter + 1;
    T alpha, delta;
    T* w;
    if (fusedM) {
      // 2 launches + 1 read-back: SpMV with the y recurrence and <v,y>; then y -= (alpha/beta) r2, the w update
      // and <y,y>; r1/r2/y rotate by pointer instead of the two copies (fused_phases.cu)
      w = (iter == 1) ? ws.w2 : ws.w1;
      T beta2;
      minres_fused_lanczos<T>(ws, *A.csr, iter, lambda, beta, oldbeta, cs, sn, deltabar, eps_rot, w, &alpha, &beta2);
      r1 = ws.r1; r2 = ws.r2; y = ws.y; v = MisI ? r2 : ws.vv;
      delta = cs * deltabar + sn * alpha;
      oldbeta = beta;
      beta = beta2;
    } else {
    op_apply(c, A, v, y);
    if (lambda != 0) k_axpy<T>(c, n, lambda, v, y);
    k_scal<T>(c, n, T(1) / beta, y);                          // kdiv!(n, y, β)
    if (iter >= 2) k_axpy<T>(c, n, -beta / oldbeta, r1, y);
    alpha = k_dot<T>(c, n, v, y) / beta;
    k_axpy<T>(c, n, -alpha / beta, r2, y);
    delta = cs * deltabar + sn * alpha;
    if (iter == 1) {
      w = ws.w2;
      k_divcopy<T>(c, n, w, v, beta);
    } else {
      w = ws.w1;
      if (iter >= 3) k_scal<T>(c, n, -eps_rot, w);
      k_axpy<T>(c, n, -delta, ws.w2, w);
      k_axpy<T>(c, n, T(1) / beta, v, w);
    }
    k_copy<T>(c, n, r1, r2);
    k_copy<T>(c, n, r2, y);
    if (!MisI) op_apply(c, M, r2, v, ldiv);
    oldbeta = beta;
    beta = k_dot<T>(c, n, r2, v);
    }
    if (beta < 0) throw std::runtime_error("Preconditioner is not positive definite");
    beta = std::sqrt(beta);
    ANorm2 = ANorm2 + alpha * alpha + oldbeta * oldbeta + beta * beta;
    const T gbar = sn * deltabar - cs * alpha;
    eps_rot = sn * beta;
    deltabar = -cs * beta;
    const T root = std::sqrt(gbar * gbar + deltabar * deltabar);
    ArNorm = phibar * root;
    if (history) stats.Aresiduals.push_back(ArNorm);
    T gamma = std::sqrt(gbar * gbar + beta * beta);
    gamma = gamma > epsM ? gamma : epsM;
    if (!fusedM) k_scal<T>(c, n, T(1) / gamma, w);            // kdiv!(n, w, γ)  (fused: folded into the x update below)
    if (linesearch) {                                         // minres.jl:336-373
      const T cg_ = cs * gbar;
      if (iter > 1) {
        zeta_km1 = zeta_k;
        zeta_k = -cg_ * (rNorm * rNorm);
        beta_w = (zeta_km1 != 0) ? zeta_k / zeta_km1 : zeta_k;
        delta_w = zeta_k + beta_w * beta_w * delta_w;
      }
      if (cg_ >= 0) {
        if (o.verbose > 0) printf("nonpositive curvature detected:  cs * γbar = %e\n", (double)cg_);
        stats.npcCount = 1;
        // (the reference's `w1 = w` only rebinds a local name)
        if (iter == 1) k_copy<T>(c, n, x, b);
        else if (delta_w < 0) stats.npcCount = 2;
        stats.indefinite = true;
        run.finish(iter, true, false, "nonpositive curvature", false);
        return;
      }
    }
    cs = gbar / gamma;
    sn = beta / gamma;
    const T phi = cs * phibar;
    phibar = sn * phibar;
    if (linesearch) {
      k_scal<T>(c, n, sn * sn, npc_dir);
      k_axpy<T>(c, n, -phibar * cs / beta, v, npc_dir);
    }
    T xNorm_fused = 0;
    if (fusedM) xNorm_fused = minres_fused_update<T>(ws, w, gamma, phi);   // w /= γ ; x += ϕ w ; ‖x‖ in one pass
    else k_axpy<T>(c, n, phi, w, x);
    xENorm2 = xENorm2 + phi * phi;
    if (iter >= 2) { T* tmp = ws.w1; ws.w1 = ws.w2; ws.w2 = tmp; }   // @kswap!(w1, w2)
    err_vec[iter % window] = phi;
    if (iter >= window) {
      T ssq = 0;
      for (int i = 0; i < window; i++) ssq += err_vec[i] * err_vec[i];
      err_lbnd = std::sqrt(ssq);
    }
    gmax = gmax > gamma ? gmax : gamma;
    gmin = gmin < gamma ? gmin : gamma;
    const T zeta = rhs1 / gamma;
    rhs1 = rhs2 - delta * zeta;
    rhs2 = -eps_rot * zeta;
    ANorm = std::sqrt(ANorm2);
    xNorm = fusedM ? xNorm_fused : k_nrm2<T>(c, n, x);
    rNorm = phibar;
    const T test1 = rNorm / (ANorm * xNorm);
    const T test2 = root / ANorm;
    if (history) stats.residuals.push_back(rNorm);
    Acond = gmax / gmin;
    if (history) stats.Acond.push_back(Acond);
    if (kdisplay(iter, o.verbose))
      printf("%5d  %7.1e  %7.1e  %7.1e  %8.1e  %8.1e  %7.1e  %7.1e  %7.1e  %7.1e  %.2fs\n", iter, (double)rNorm, (double)ArNorm,
             (double)beta, (double)cs, (double)sn, (double)ANorm, (double)Acond, (double)test1, (double)test2, run.elapsed());
    if (iter == 1 && beta / beta1 <= 10 * epsM) {             // minres.jl:425-435
      run.finish(1, true, true, "x is a minimum least-squares solution");
      return;
    }
    ill_cond_mach = (T(1) + T(1) / Acond <= T(1));
    solved_mach = (T(1) + test2 <= T(1));
    zero_resid_mach = (T(1) + test1 <= T(1));
    const bool resid_decrease_mach = (rNorm + T(1) <= T(1));
    tired = iter >= itmax;
    ill_cond_lim = (T(1) / Acond <= ctol);
    solved_lim = (test2 <= eps_tol);
    zero_resid_lim = MisI && (test1 <= eps_of<T>());
    const bool resid_decrease_lim = (rNorm <= eps_tol);
    if (iter >= window) fwd_err = err_lbnd <= etol * std::sqrt(xENorm2);
    run.poll(iter, user_exit, overtimed);
    zero_resid = zero_resid_mach || zero_resid_lim;
    const bool resid_decrease = resid_decrease_mach || resid_decrease_lim;
    ill_cond = ill_cond_mach || ill_cond_lim;
    solved = solved_mach || solved_lim || zero_resid || fwd_err || resid_decrease;
  }
  if (o.verbose > 0) printf("\n");
  if (tired) status = "maximum number of iterations exceeded";
  if (ill_cond_mach) status = "condition number seems too large for this machine";
  if (ill_cond_lim) status = "condition number exceeds tolerance";
  if (solved) status = "found approximate minimum least-squares solution";
  if (zero_resid) status = "found approximate zero-residual solution";
  if (fwd_err) status = "truncated forward error small enough";
  if (user_exit) status = "user-requested exit";
  if (overtimed) status = "time limit exceeded";
  run.finish(iter, solved, !zero_resid, status);
}

#define INST(T)                                                                                                   \
  template Workspace<T>* ws_create<T>(SolverKind, int, int, int, int, int);                                       \
  template void ws_destroy<T>(Workspace<T>*);                                                                     \
  template void ws_warm_start<T>(Workspace<T>*, const T*);                                                        \
  template void cg_solve<T>(Workspace<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const SolveOpts&);          \
  template void gmres_solve<T>(Workspace<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const LinOp<T>&, const SolveOpts&); \
  template void fom_solve<T>(Workspace<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const LinOp<T>&, const SolveOpts&); \
  template void fgmres_solve<T>(Workspace<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const LinOp<T>&, const SolveOpts&); \
  template void bicgstab_solve<T>(Workspace<T>&, const LinOp<T>&, const T*, const T*, const LinOp<T>&, const LinOp<T>&, const SolveOpts&); \
  template void minres_solve<T>(Workspace<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const SolveOpts&);
INST(double)
INST(float)
#undef INST

}  // namespace kb
