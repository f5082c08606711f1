// siblings.cu -- sibling solvers that run on the hot-path kernels unchanged
// (SURVEY.md section 8f-3): cgs!, cg_lanczos!, dqgmres!, diom!, cr!.  Same rules
// as solvers.cu: the reference's host control flow statement by statement (files
// cited per function), every vector operation a kernel from blas1.cu / spmv.cu
// / fused_phases.cu.  fom! and fgmres! run on GMRES's Arnoldi driver in solvers.cu.
#include <cstring>

#include "solver_common.h"

namespace kb {

// ===========================================================================
// cgs!  (src/cgs.jl:125-282)
// ===========================================================================
template <class T>
void cgs_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const T* c_in, const LinOp<T>& M, const LinOp<T>& N,
               const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int n = ws.n;
  const bool history = o.history, ldiv = o.ldiv;
  if (o.verbose > 0) printf("CGS: system of size %d\n", n);
  const bool MisI = M.is_identity(), NisI = N.is_identity();
  allocate_if(!MisI, ws, ws.vw);
  allocate_if(!NisI, ws, ws.yz);
  T *dx = ws.dx, *x = ws.x, *r = ws.r, *u = ws.u, *p = ws.p, *q = ws.q;
  Stats& stats = ws.stats;
  const bool warm_start = ws.warm_start;
  stats.reset();
  T* t = ws.ts; T* s = ws.ts;                                 // cgs.jl:150-155
  T* v = MisI ? t : ws.vw;
  T* w = MisI ? s : ws.vw;
  T* y = NisI ? p : ws.yz;
  T* z = NisI ? u : ws.yz;
  T* r0 = MisI ? r : ws.ts;
  const T* cvec = c_in ? c_in : b;

  if (warm_start) { op_apply(c, A, dx, r0); k_axpby<T>(c, n, T(1), b, T(-1), r0); }
  else k_copy<T>(c, n, r0, b);
  k_fill<T>(c, n, x, T(0));
  if (!MisI) op_apply(c, M, r0, r, ldiv);
  T rNorm = k_nrm2<T>(c, n, r);
  if (history) stats.residuals.push_back(rNorm);
  if (rNorm == 0) { run.finish(0, true, false, "x is a zero-residual solution"); return; }
  T rho = k_dot<T>(c, n, cvec, r);
  if (rho == 0) { run.finish(0, false, false, "Breakdown bᴴc = 0"); return; }
  int iter = 0;
  const int itmax = default_itmax(ws, o.itmax);
  const T eps_tol = tol_of<T>(o.atol) + tol_of<T>(o.rtol) * rNorm;
  if (o.verbose > 0) printf("%5s  %7s  %5s\n", "k", "‖rₖ‖", "timer");
  if (kdisplay(iter, o.verbose)) printf("%5d  %7.1e  %.2fs\n", iter, (double)rNorm, run.elapsed());
  k_copy<T>(c, n, u, r);
  k_copy<T>(c, n, p, r);
  k_fill<T>(c, n, q, T(0));
  bool solved = rNorm <= eps_tol, tired = iter >= itmax, breakdown = false, user_exit = false, overtimed = false;
  std::string status = "unknown";

  // grouped passes (fused_phases.cu): 4 launches and 2 read-backs per iteration instead of 12 and 3
  const bool fusedS = o.fused && A.kind == LinOp<T>::CSR && MisI && NisI;
  while (!(solved || tired || breakdown || user_exit || overtimed)) {
    T alpha, rho_next;
    if (fusedS) {
      const T sigma = cgs_fused_sigma<T>(ws, *A.csr, cvec);
      alpha = rho / sigma;
      T rr;
      cgs_fused_update<T>(ws, *A.csr, cvec, alpha, &rho_next, &rr);
      const T beta = rho_next / rho;
      cgs_fused_directions<T>(ws, beta);
      rho = rho_next;
      iter = iter + 1;
      rNorm = std::sqrt(rr);
    } else {
      if (!NisI) op_apply(c, N, p, y, ldiv);
      op_apply(c, A, y, t);
      if (!MisI) op_apply(c, M, t, v, ldiv);
      const T sigma = k_dot<T>(c, n, cvec, v);
      alpha = rho / sigma;
      k_copy<T>(c, n, q, u);
      k_axpy<T>(c, n, -alpha, v, q);
      k_axpy<T>(c, n, T(1), q, u);
      if (!NisI) op_apply(c, N, u, z, ldiv);
      k_axpy<T>(c, n, alpha, z, x);
      op_apply(c, A, z, s);
      if (!MisI) op_apply(c, M, s, w, ldiv);
      k_axpy<T>(c, n, -alpha, w, r);
      rho_next = k_dot<T>(c, n, cvec, r);
      const T beta = rho_next / rho;
      k_copy<T>(c, n, u, r);
      k_axpy<T>(c, n, beta, q, u);
      k_axpby<T>(c, n, T(1), q, beta, p);
      k_axpby<T>(c, n, T(1), u, beta, p);
      rho = rho_next;
      iter = iter + 1;
      rNorm = k_nrm2<T>(c, n, r);
    }
    if (history) stats.residuals.push_back(rNorm);
    const bool resid_decrease_mach = (rNorm + T(1) <= T(1));
    run.poll(iter, user_exit, overtimed);
    solved = (rNorm <= eps_tol) || resid_decrease_mach;
    tired = iter >= itmax;
    breakdown = (alpha == 0 || std::isnan(alpha));
    if (kdisplay(iter, o.verbose)) printf("%5d  %7.1e  %.2fs\n", iter, (double)rNorm, run.elapsed());
  }
  if (o.verbose > 0) printf("\n");
  if (tired) status = "maximum number of iterations exceeded";
  if (breakdown) status = "breakdown αₖ == 0";
  if (solved) status = "solution good enough given atol and rtol";
  if (user_exit) status = "user-requested exit";
  if (overtimed) status = "time limit exceeded";
  run.finish(iter, solved, false, status);
}

// ===========================================================================
// cg_lanczos!  (src/cg_lanczos.jl:110-264)
// ===========================================================================
template <class T>
void cg_lanczos_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int n = ws.n;
  const bool history = o.history, ldiv = o.ldiv, check_curvature = o.check_curvature;
  if (o.verbose > 0) printf("CG-LANCZOS: system of %d equations in %d variables\n", n, n);
  const bool MisI = M.is_identity();
  allocate_if(!MisI, ws, ws.vv);
  T *dx = ws.dx, *x = ws.x, *Mv = ws.Mv, *Mv_prev = ws.Mv_prev, *p = ws.p, *Mv_next = ws.Mv_next;
  Stats& stats = ws.stats;
  const bool warm_start = ws.warm_start;
  stats.reset();
  stats.Anorm = NAN;
  T* v = MisI ? Mv : ws.vv;                                   // cg_lanczos.jl:138
  // knorm_elliptic (src/krylov_utils.jl:319): ||v|| when v === Mv, else sqrt(<v, Mv>)
  auto norm_elliptic = [&]() { return MisI ? k_nrm2<T>(c, n, v) : (T)std::sqrt(k_dot<T>(c, n, v, Mv)); };

  k_fill<T>(c, n, x, T(0));
  if (warm_start) { op_apply(c, A, dx, Mv); k_axpby<T>(c, n, T(1), b, T(-1), Mv); }
  else k_copy<T>(c, n, Mv, b);
  if (!MisI) op_apply(c, M, Mv, v, ldiv);
  T beta = norm_elliptic();
  T sigma = beta;
  T rNorm = sigma;
  if (history) stats.residuals.push_back(rNorm);
  if (beta == 0) {
    stats.Anorm = 0; stats.indefinite = false;
    run.finish(0, true, false, "x is a zero-residual solution");
    return;
  }
  k_copy<T>(c, n, p, v);
  k_scal<T>(c, n, T(1) / beta, v);                            // kdiv!(n, v, β)
  if (!MisI) k_scal<T>(c, n, T(1) / beta, Mv);
  k_copy<T>(c, n, Mv_prev, Mv);
  int iter = 0;
  const int itmax = default_itmax(ws, o.itmax);
  T omega = 0, gamma = 1, Anorm2 = 0, beta_prev = 0;
  const T eps_tol = tol_of<T>(o.atol) + tol_of<T>(o.rtol) * rNorm;
  if (o.verbose > 0) printf("%5s  %7s  %5s\n", "k", "‖rₖ‖", "timer");
  if (kdisplay(iter, o.verbose)) printf("%5d  %7.1e  %.2fs\n", iter, (double)rNorm, run.elapsed());
  bool indefinite = false, solved = rNorm <= eps_tol, tired = iter >= itmax, user_exit = false, overtimed = false;
  std::string status = "unknown";

  while (!(solved || tired || (check_curvature && indefinite) || user_exit || overtimed)) {
    // grouped passes (fused_phases.cu; M = I so v === Mv): 3 launches per iteration instead of 8
    const bool fusedL = o.fused && A.kind == LinOp<T>::CSR && MisI;
    const T delta = fusedL ? lanczos_fused_delta<T>(ws, *A.csr) : (op_apply(c, A, v, Mv_next), k_dot<T>(c, n, v, Mv_next));
    gamma = T(1) / (delta - omega / gamma);
    indefinite = indefinite || (gamma <= 0);
    if (check_curvature && indefinite) continue;
    if (fusedL) {
      beta = lanczos_fused_recur<T>(ws, delta, beta, iter > 0);
    } else {
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
    }
    Anorm2 += beta_prev * beta_prev + beta * beta + delta * delta;
    beta_prev = beta;
    if (!fusedL) k_axpy<T>(c, n, gamma, p, x);
    omega = beta * gamma;
    sigma = -omega * sigma;
    omega = omega * omega;
    if (fusedL) lanczos_fused_update<T>(ws, beta, gamma, sigma, omega);
    else k_axpby<T>(c, n, sigma, v, omega, p);
    rNorm = std::fabs(sigma);
    if (history) stats.residuals.push_back(rNorm);
    iter = iter + 1;
    if (kdisplay(iter, o.verbose)) printf("%5d  %7.1e  %.2fs\n", iter, (double)rNorm, run.elapsed());
    const bool resid_decrease_mach = (rNorm + T(1) <= T(1));
    run.poll(iter, user_exit, overtimed);
    solved = (rNorm <= eps_tol) || resid_decrease_mach;
    tired = iter >= itmax;
  }
  if (o.verbose > 0) printf("\n");
  if (tired) status = "maximum number of iterations exceeded";
  if (check_curvature && indefinite) status = "negative curvature";
  if (solved) status = "solution good enough given atol and rtol";
  if (user_exit) status = "user-requested exit";
  if (overtimed) status = "time limit exceeded";
  stats.Anorm = std::sqrt(Anorm2); stats.indefinite = indefinite;
  run.finish(iter, solved, false, status);
}

// ---------------------------------------------------------------------------
// dqgmres! (src/dqgmres.jl:121-335) and diom! (src/diom.jl:121-332): the truncated
// (incomplete orthogonalization) variants; circular stacks V, P of `memory` vectors.
// One driver: QR by Givens rotations (DQGMRES) or LU without pivoting (DIOM) of the
// band Hessenberg matrix, kept on the host.  Indices are 1-based like the reference.
//   workspace fields: t (ws.t), z (ws.yz), w (ws.vw), V, P (ws.Z), c, s / L (ws.sgiv), H (ws.R)
// ---------------------------------------------------------------------------
template <class T, bool QR>
static void truncated_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const LinOp<T>& N, const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& cx = ws.ctx;
  const int n = ws.n;
  const bool history = o.history, ldiv = o.ldiv, reorth = o.reorthogonalization;
  if (o.verbose > 0) printf("%s: system of size %d\n", QR ? "DQGMRES" : "DIOM", n);
  const bool MisI = M.is_identity(), NisI = N.is_identity();
  allocate_if(!MisI, ws, ws.vw);
  allocate_if(!NisI, ws, ws.yz);
  T *dx = ws.dx, *x = ws.x, *t = ws.t;
  std::vector<T*>&P = ws.Z, &V = ws.V;
  std::vector<T>&c = ws.c, &s = ws.sgiv, &H = ws.R;
  std::vector<T>& L = ws.sgiv;
  Stats& stats = ws.stats;
  const bool warm_start = ws.warm_start;
  stats.reset();
  T* w = MisI ? t : ws.vw;
  T* r0 = MisI ? t : ws.vw;

  k_fill<T>(cx, n, x, T(0));
  if (warm_start) { op_apply(cx, A, dx, t); k_axpby<T>(cx, n, T(1), b, T(-1), t); }
  else k_copy<T>(cx, n, t, b);
  if (!MisI) op_apply(cx, M, t, r0, ldiv);
  T rNorm = k_nrm2<T>(cx, n, r0);
  if (history) stats.residuals.push_back(rNorm);
  if (rNorm == 0) { run.finish(0, true, false, "x is a zero-residual solution"); return; }
  int iter = 0;
  const int itmax = default_itmax(ws, o.itmax);
  const T eps_tol = tol_of<T>(o.atol) + tol_of<T>(o.rtol) * rNorm;
  if (o.verbose > 0) printf("%5s  %7s  %5s\n", "k", "‖rₖ‖", "timer");
  if (kdisplay(iter, o.verbose)) printf("%5d  %7.1e  %.2fs\n", iter, (double)rNorm, run.elapsed());
  const int mem = (int)V.size();
  for (int i = 0; i < mem; i++) k_fill<T>(cx, n, V[i], T(0));
  for (size_t i = 0; i < P.size(); i++) k_fill<T>(cx, n, P[i], T(0));
  std::fill(H.begin(), H.end(), T(0));
  std::fill(s.begin(), s.end(), T(0));          // DQGMRES sines / DIOM pivots L
  if (QR) std::fill(c.begin(), c.end(), T(0));
  T gamma_k = rNorm;                            // DQGMRES: last component of g_k;  DIOM: xi
  k_divcopy<T>(cx, n, V[0], r0, rNorm);
  bool solved = rNorm <= eps_tol, tired = iter >= itmax, user_exit = false, overtimed = false;
  std::string status = "unknown";

  // grouped passes (fused_phases.cu): window + 3 launches and one read-back per iteration instead of 2 window + 6
  constexpr int kMaxWindow = 120;
  const bool fusedT = o.fused && A.kind == LinOp<T>::CSR && MisI && NisI && !reorth && mem <= kMaxWindow && mem <= gmres_fused_max();
  ws.mdiag_fused = nullptr;
  T* dvec[kMaxWindow]; T dcoef[kMaxWindow];
  while (!(solved || tired || user_exit || overtimed)) {
    iter = iter + 1;
    int ndir = 0;
    const int pos = (iter - 1) % mem + 1, next_pos = iter % mem + 1;
    T* z = NisI ? V[pos - 1] : ws.yz;
    const int lo = std::max(1, iter - mem + 1);
    T Haux;
    if (fusedT) {
      // SpMV + incomplete orthogonalization as ONE chain of passes (fused_phases.cu: fused_orth_chain): the dot
      // product with the next basis vector rides in the pass that subtracts the current one; one read-back
      const T* vecs[kMaxWindow]; T hbuf[kMaxWindow];
      const int cnt = iter - lo + 1;
      for (int i = lo; i <= iter; i++) vecs[i - lo] = V[(i - 1) % mem];
      fused_orth_chain<T>(ws, *A.csr, z, w, vecs, cnt, hbuf, &Haux);
      for (int i = lo; i <= iter; i++) H[iter - i] = hbuf[i - lo];
    } else {
      if (!NisI) op_apply(cx, N, V[pos - 1], z, ldiv);
      op_apply(cx, A, z, t);
      if (!MisI) op_apply(cx, M, t, w, ldiv);
      for (int i = lo; i <= iter; i++) {          // incomplete orthogonalization
        const int ipos = (i - 1) % mem + 1, diag = iter - i + 1;
        H[diag - 1] = k_dot<T>(cx, n, w, V[ipos - 1]);
        k_axpy<T>(cx, n, -H[diag - 1], V[ipos - 1], w);
    }
    if (reorth) {
      for (int i = lo; i <= iter; i++) {
        const int ipos = (i - 1) % mem + 1, diag = iter - i + 1;
        const T Htmp = k_dot<T>(cx, n, w, V[ipos - 1]);
        H[diag - 1] += Htmp;
        k_axpy<T>(cx, n, -Htmp, V[ipos - 1], w);
      }
    }
    Haux = k_nrm2<T>(cx, n, w);
    }
    if (Haux != 0) k_divcopy<T>(cx, n, V[next_pos - 1], w, Haux);
    int ppos;                                   // position of p_k in the circular stack P
    T step;                                     // x += step * p_k
    if (QR) {                                   // dqgmres.jl:268-289
      if (iter >= mem + 2) H[mem] = T(0);
      const int lo2 = std::max(1, iter - mem);
      for (int i = lo2; i <= iter - 1; i++) {
        const int irot = (i - 1) % mem + 1, diag = iter - i, next_diag = diag + 1;
        const T Htmp = c[irot - 1] * H[next_diag - 1] + s[irot - 1] * H[diag - 1];
        H[diag - 1] = s[irot - 1] * H[next_diag - 1] - c[irot - 1] * H[diag - 1];
        H[next_diag - 1] = Htmp;
      }
      sym_givens<T>(H[0], Haux, &c[pos - 1], &s[pos - 1], &H[0]);
      const T gamma_next = s[pos - 1] * gamma_k;
      gamma_k = c[pos - 1] * gamma_k;
      ppos = pos;
      for (int i = lo2; i <= iter - 1; i++) {
        const int ipos = (i - 1) % mem + 1, diag = iter - i + 1;
        if (fusedT) { dvec[ndir] = P[ipos - 1]; dcoef[ndir++] = -H[diag - 1]; }
        else if (ipos == ppos) k_scal<T>(cx, n, -H[diag - 1], P[ppos - 1]);
        else k_axpy<T>(cx, n, -H[diag - 1], P[ipos - 1], P[ppos - 1]);
      }
      step = gamma_k;
      rNorm = std::fabs(gamma_next);
      gamma_k = gamma_next;
    } else {                                    // diom.jl:262-289
      if (iter >= 2) {
        for (int i = std::max(2, iter - mem + 2); i <= iter; i++) {
          const int lpos = (i - 1) % (mem - 1) + 1, diag = iter - i + 1, next_diag = diag + 1;
          H[diag - 1] = H[diag - 1] - L[lpos - 1] * H[next_diag - 1];
          if (i == iter) gamma_k = -L[lpos - 1] * gamma_k;
        }
      }
      const int next_lpos = iter % (mem - 1) + 1;
      L[next_lpos - 1] = Haux / H[0];
      ppos = (iter - 1) % (mem - 1) + 1;
      for (int i = lo; i <= iter - 1; i++) {
        const int ipos = (i - 1) % (mem - 1) + 1, diag = iter - i + 1;
        if (fusedT) { dvec[ndir] = P[ipos - 1]; dcoef[ndir++] = -H[diag - 1]; }
        else if (ipos == ppos) k_scal<T>(cx, n, -H[diag - 1], P[ppos - 1]);
        else k_axpy<T>(cx, n, -H[diag - 1], P[ipos - 1], P[ppos - 1]);
      }
      step = gamma_k;
      rNorm = Haux * std::fabs(gamma_k / H[0]);
    }
    if (fusedT) {
      // the whole direction update + x update in one pass per 8 stack vectors (trunc_fused_direction)
      trunc_fused_direction<T>(ws, P[ppos - 1], ndir, dvec, dcoef, z, H[0], step);
    } else {
      k_axpy<T>(cx, n, T(1), z, P[ppos - 1]);
      k_scal<T>(cx, n, T(1) / H[0], P[ppos - 1]);   // kdiv!(n, P[pos], H[1])
      k_axpy<T>(cx, n, step, P[ppos - 1], x);
    }
    if (history) stats.residuals.push_back(rNorm);
    const bool resid_decrease_mach = (rNorm + T(1) <= T(1));
    run.poll(iter, user_exit, overtimed);
    solved = (rNorm <= eps_tol) || resid_decrease_mach;
    tired = iter >= itmax;
    if (kdisplay(iter, o.verbose)) printf("%5d  %7.1e  %.2fs\n", iter, (double)rNorm, run.elapsed());
  }
  if (o.verbose > 0) printf("\n");
  if (QR) {                                     // dqgmres.jl:319-322 assigns in this order (tired overrides solved)
    if (solved) status = "solution good enough given atol and rtol";
    if (tired) status = "maximum number of iterations exceeded";
  } else {
    if (tired) status = "maximum number of iterations exceeded";
    if (solved) status = "solution good enough given atol and rtol";
  }
  if (user_exit) status = "user-requested exit";
  if (overtimed) status = "time limit exceeded";
  run.finish(iter, solved, false, status);
}

template <class T>
void dqgmres_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const LinOp<T>& N, const SolveOpts& o) {
  truncated_solve<T, true>(ws, A, b, M, N, o);
}
template <class T>
void diom_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const LinOp<T>& N, const SolveOpts& o) {
  truncated_solve<T, false>(ws, A, b, M, N, o);
}

// ===========================================================================
// cr!  (src/cr.jl:128-478), trust region and linesearch included
//   workspace fields: r, p, q, Ar (ws.Ap), Mq (ws.z), npc_dir
// ===========================================================================
// to_boundary(n, x, d, z, radius; flip = false, xNorm2, dNorm2) with M = I (src/krylov_utils.jl:375-402)
template <class T>
static void cr_to_boundary(Ctx& c, int n, const T* x, const T* d, T radius, T xNorm2, T dNorm2, T* lo, T* hi) {
  if (!(radius > 0)) throw std::runtime_error("radius must be positive");
  const T rxd = k_dot<T>(c, n, x, d);
  if (dNorm2 == T(0)) dNorm2 = k_dot<T>(c, n, d, d);
  if (xNorm2 == T(0)) xNorm2 = k_dot<T>(c, n, x, x);
  if (dNorm2 == T(0)) throw std::runtime_error("zero direction");
  const T radius2 = radius * radius;
  if (!(xNorm2 <= radius2)) throw std::runtime_error("outside of the trust region");
  T s1, s2;
  if (roots_quadratic<T>(dNorm2, 2 * rxd, xNorm2 - radius2, 1, &s1, &s2)) throw std::runtime_error("negative discriminant");
  *hi = std::max(s1, s2); *lo = std::min(s1, s2);
}

template <class T>
void cr_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int n = ws.n;
  const bool history = o.history, ldiv = o.ldiv, linesearch = o.linesearch;
  const T radius = (T)o.radius;
  const T gam = o.cr_gamma < 0 ? std::sqrt(eps_of<T>()) : (T)o.cr_gamma;
  if (linesearch && radius > 0) throw std::runtime_error("'linesearch' set to 'true' but radius > 0");
  if (o.verbose > 0) printf("CR: system of %d equations in %d variables\n", n, n);
  if (ws.warm_start && linesearch) throw std::runtime_error("warm_start and linesearch cannot be used together");
  const bool MisI = M.is_identity();
  allocate_if(!MisI, ws, ws.z);
  allocate_if(linesearch || radius > 0, ws, ws.npc_dir);
  T *dx = ws.dx, *x = ws.x, *r = ws.r, *p = ws.p, *q = ws.q, *Ar = ws.Ap;
  Stats& stats = ws.stats;
  const bool warm_start = ws.warm_start;
  stats.reset();
  T* Mq = MisI ? q : ws.z;
  T* npc_dir = ws.npc_dir;

  k_fill<T>(c, n, x, T(0));
  if (warm_start) { op_apply(c, A, dx, p); k_axpby<T>(c, n, T(1), b, T(-1), p); }
  else k_copy<T>(c, n, p, b);
  if (MisI) k_copy<T>(c, n, r, p); else op_apply(c, M, p, r, ldiv);
  T rNorm = std::sqrt(k_dot<T>(c, n, r, p));                  // knorm_elliptic(n, r, p)
  if (history) stats.residuals.push_back(rNorm);
  if (rNorm == 0) {
    if (history) stats.Aresiduals.push_back(0);
    run.finish(0, true, false, "x is a zero-residual solution");
    return;
  }
  op_apply(c, A, r, Ar);
  T rho = k_dot<T>(c, n, r, Ar);
  if (rho == 0) {
    if (history) stats.Aresiduals.push_back(0);
    if (linesearch || radius > 0) {
      k_copy<T>(c, n, x, p);
      k_copy<T>(c, n, npc_dir, p);
      stats.npcCount = 1; stats.indefinite = true;
    }
    run.finish(0, true, false, "b is a zero-curvature direction", false);
    return;
  }
  k_copy<T>(c, n, p, r);
  k_copy<T>(c, n, q, Ar);
  T mquad = 0;                                                // quadratic model (verbose only)
  int iter = 0;
  const int itmax = default_itmax(ws, o.itmax);
  T rNorm2 = rNorm * rNorm, pNorm = rNorm, pNorm2 = rNorm2, pr = rNorm2, abspr = pr, pAp = rho, abspAp = std::fabs(pAp);
  T xNorm = 0;
  T ArNorm = k_nrm2<T>(c, n, Ar);
  if (history) stats.Aresiduals.push_back(ArNorm);
  const T eps_tol = tol_of<T>(o.atol) + tol_of<T>(o.rtol) * rNorm;
  if (o.verbose > 0) printf("%5s  %8s  %8s  %8s  %5s\n", "k", "‖x‖", "‖r‖", "quad", "timer");
  if (kdisplay(iter, o.verbose)) printf("%5d  %8.1e  %8.1e  %8.1e  %.2fs\n", iter, (double)xNorm, (double)rNorm, (double)mquad, run.elapsed());
  bool descent = pr > 0, solved = rNorm <= eps_tol, tired = iter >= itmax, on_boundary = false, npcurv = false;
  bool user_exit = false, overtimed = false;
  // grouped passes (no trust region, no linesearch, M = I): 3 launches and 2 read-backs per iteration instead of 9 and 5
  const bool fusedC = o.fused && A.kind == LinOp<T>::CSR && MisI && radius == 0 && !linesearch;
  T qq = 0;
  bool have_qq = false;
  std::string status = "unknown";
  const T sqeps = std::sqrt(eps_of<T>());

  while (!(solved || tired || user_exit || overtimed)) {
    T alpha = 0;
    if (linesearch) {
      const bool p_curv = pAp <= gam * pNorm * pNorm, r_curv = rho <= gam * rNorm * rNorm;
      if (p_curv || r_curv) {                                 // cr.jl:233-262
        npcurv = true;
        if (o.verbose > 0) printf("nonpositive curvature detected: pᴴAp = %8.1e and rᴴAr = %8.1e\n", (double)pAp, (double)rho);
        stats.indefinite = true;
        if (iter == 0) {
          k_copy<T>(c, n, npc_dir, p);
          k_copy<T>(c, n, x, p);
          stats.npcCount = 1;
        } else {
          if (r_curv) { k_copy<T>(c, n, npc_dir, r); stats.npcCount += 1; }
          if (p_curv) { stats.npcCount += 1; if (!r_curv) k_copy<T>(c, n, npc_dir, p); }
        }
        run.finish(iter, true, false, "nonpositive curvature", false);
        return;
      }
    } else if (pAp <= 0 && radius == 0) {
      throw std::runtime_error("Indefinite system and no trust region");
    }
    if (!MisI) op_apply(c, M, q, Mq, ldiv);
    if (radius > 0) {                                         // cr.jl:268-373
      const T xNorm2 = xNorm * xNorm;
      T t1, t2, tr, tlo;
      cr_to_boundary<T>(c, n, x, p, radius, xNorm2, pNorm2, &t2, &t1);
      cr_to_boundary<T>(c, n, x, r, radius, xNorm2, rNorm2, &tlo, &tr);
      if (abspAp <= gam * pNorm * k_nrm2<T>(c, n, q)) {       // pᴴAp ≃ 0
        npcurv = true; stats.indefinite = true; stats.npcCount = 1;
        k_copy<T>(c, n, npc_dir, p);
        if (abspr <= gam * pNorm * rNorm) {                   // pᴴr ≃ 0: p := r
          p = r; q = Ar;
          if (rho > 0) alpha = std::min(tr, rNorm2 / rho);
          else { alpha = tr; if (iter > 0) { stats.npcCount = 2; k_copy<T>(c, n, npc_dir, r); } }
        } else {
          alpha = descent ? t1 : t2;
          if (rho > 0) tr = std::min(tr, rNorm2 / rho);
          const T Delta = -alpha * pr + tr * rNorm2 - tr * tr * rho / 2;
          if (Delta > 0) { p = r; q = Ar; alpha = tr; }
        }
      } else if (pAp > 0 && rho > 0) {
        alpha = rho / k_dot<T>(c, n, q, Mq);
        if (alpha >= t1) { alpha = t1; on_boundary = true; }
      } else if (pAp > 0 && rho < 0) {
        npcurv = true; stats.indefinite = true; stats.npcCount = 1;
        k_copy<T>(c, n, npc_dir, r);
        alpha = descent ? std::min(t1, pr / pAp) : std::max(t2, pr / pAp);
        const T Delta = -alpha * pr + tr * rNorm2 + (alpha * alpha * pAp - tr * tr * rho) / 2;
        if (Delta > 0) { p = r; q = Ar; alpha = tr; }
      } else if (pAp < 0 && rho > 0) {
        npcurv = true; stats.indefinite = true; stats.npcCount = 1;
        k_copy<T>(c, n, npc_dir, p);
        alpha = descent ? t1 : t2;
        tr = std::min(tr, rNorm2 / rho);
        const T Delta = -alpha * pr + tr * rNorm2 + (alpha * alpha * pAp - tr * tr * rho) / 2;
        if (Delta > 0) { p = r; q = Ar; alpha = tr; }
      } else if (pAp < 0 && rho < 0) {
        npcurv = true; stats.indefinite = true; stats.npcCount = 2;
        k_copy<T>(c, n, npc_dir, r);
        alpha = descent ? t1 : t2;
        const T Delta = -alpha * pr + tr * rNorm2 + (alpha * alpha * pAp - tr * tr * rho) / 2;
        if (Delta > 0) { p = r; q = Ar; alpha = tr; }
      }
      // (when the branches above rebind p := r, q := Ar, `Mq` keeps naming the ORIGINAL q array, as in the reference
      //  where Mq was bound once at cr.jl:155; the rebinding always ends the solve in this iteration)
    } else if (radius == 0) {
      alpha = rho / (fusedC && have_qq ? qq : k_dot<T>(c, n, q, Mq));
    }
    T rAr_fused = 0;
    if (fusedC) {
      // grouped passes (fused_phases.cu): x, r updates with ||x||, ||r||; then Ar = A r with ||Ar||, <r, Ar>
      T xx, ArAr;
      cr_fused_step<T>(ws, *A.csr, alpha, &xx, &rNorm2, &ArAr, &rAr_fused);
      xNorm = std::sqrt(xx); rNorm = std::sqrt(rNorm2); ArNorm = std::sqrt(ArAr);
      if (history) { stats.residuals.push_back(rNorm); stats.Aresiduals.push_back(ArNorm); }
    } else {
      k_axpy<T>(c, n, alpha, p, x);
      xNorm = k_nrm2<T>(c, n, x);
      if (radius > 0 && std::fabs(xNorm - radius) <= sqeps * std::max(std::fabs(xNorm), std::fabs(radius))) on_boundary = true;   // xNorm ≈ radius
      k_axpy<T>(c, n, -alpha, Mq, r);
      if (MisI) { rNorm2 = k_dot<T>(c, n, r, r); rNorm = std::sqrt(rNorm2); }
      else {
        const T omega = std::sqrt(alpha) * std::sqrt(rho);
        rNorm = std::sqrt(std::fabs(rNorm + omega)) * std::sqrt(std::fabs(rNorm - omega));
        rNorm2 = rNorm * rNorm;
    }
    if (history) stats.residuals.push_back(rNorm);
    op_apply(c, A, r, Ar);
    ArNorm = k_nrm2<T>(c, n, Ar);
    if (history) stats.Aresiduals.push_back(ArNorm);
    }
    iter = iter + 1;
    if (kdisplay(iter, o.verbose)) {
      mquad = mquad - alpha * pr + alpha * alpha * pAp / 2;
      printf("%5d  %8.1e  %8.1e  %8.1e  %.2fs\n", iter, (double)xNorm, (double)rNorm, (double)mquad, run.elapsed());
    }
    const bool resid_decrease_mach = (rNorm + T(1) <= T(1));
    run.poll(iter, user_exit, overtimed);
    const bool resid_decrease = (rNorm <= eps_tol) || resid_decrease_mach;
    solved = resid_decrease || npcurv || on_boundary;
    tired = iter >= itmax;
    if (solved || tired || user_exit || overtimed) continue;
    const T rhobar = rho;
    rho = fusedC ? rAr_fused : k_dot<T>(c, n, r, Ar);
    const T beta = rho / rhobar;
    if (fusedC) { qq = cr_fused_directions<T>(ws, beta); have_qq = true; }   // p, q updates + ||q||^2 for the next alpha
    else {
      k_axpby<T>(c, n, T(1), r, beta, p);
      k_axpby<T>(c, n, T(1), Ar, beta, q);
    }
    pNorm2 = rNorm2 + 2 * beta * pr - 2 * beta * alpha * pAp + beta * beta * pNorm2;
    if (pNorm2 > sqeps) pNorm = std::sqrt(pNorm2);
    else if (std::fabs(pNorm2) <= sqeps) pNorm = T(0);
    else { run.finish(iter, solved, false, "solver encountered numerical issues"); return; }
    pr = rNorm2 + beta * pr - beta * alpha * pAp;
    abspr = std::fabs(pr);
    pAp = rho + beta * beta * pAp;
    abspAp = std::fabs(pAp);
    descent = pr > 0;
  }
  if (o.verbose > 0) printf("\n");
  if (tired) status = "maximum number of iterations exceeded";
  if (solved) status = "solution good enough given atol and rtol";
  if (user_exit) status = "user-requested exit";
  if (overtimed) status = "time limit exceeded";
  if (npcurv) status = "nonpositive curvature";
  if (on_boundary) status = "on trust-region boundary";
  run.finish(iter, solved, false, status);
}

// ===========================================================================
// car!  (src/car.jl:108-256)
//   workspace fields: r, p, s, q, t, u, Mu (lazy; Mu === u when M = I)
// ===========================================================================
template <class T>
void car_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int n = ws.n;
  const bool history = o.history, ldiv = o.ldiv;
  if (o.verbose > 0) printf("CAR: system of %d equations in %d variables\n", n, n);
  const bool MisI = M.is_identity();
  allocate_if(!MisI, ws, ws.Mu);
  T *dx = ws.dx, *x = ws.x, *r = ws.r, *p = ws.p, *s = ws.s, *q = ws.q, *t = ws.t, *u = ws.u;
  T* Mu = MisI ? u : ws.Mu;
  Stats& stats = ws.stats;
  const bool warm_start = ws.warm_start;
  stats.reset();

  k_fill<T>(c, n, x, T(0));
  if (warm_start) { op_apply(c, A, dx, r); k_axpby<T>(c, n, T(1), b, T(-1), r); }
  else k_copy<T>(c, n, r, b);
  if (MisI) k_copy<T>(c, n, p, r);                            // p₀ = r₀ = M(b - Ax₀)
  else { op_apply(c, M, r, p, ldiv); k_copy<T>(c, n, r, p); }
  op_apply(c, A, r, s);                                       // s₀ = Ar₀
  if (MisI) k_copy<T>(c, n, q, s);                            // q₀ = MAp₀ and s₀ = MAr₀
  else { op_apply(c, M, s, q, ldiv); k_copy<T>(c, n, s, q); }
  op_apply(c, A, s, t);                                       // t₀ = As₀
  k_copy<T>(c, n, u, t);                                      // u₀ = Aq₀
  T rho = k_dot<T>(c, n, t, s);                               // ρ₀ = ⟨t₀ , s₀⟩
  T rNorm = k_nrm2<T>(c, n, r);
  if (history) stats.residuals.push_back(rNorm);
  T ArNorm = MisI ? k_nrm2<T>(c, n, s) : std::sqrt(k_dot<T>(c, n, r, u));   // knorm_elliptic(n, r, u)
  if (history) stats.Aresiduals.push_back(ArNorm);
  if (rNorm == 0) {
    run.finish(0, true, false, "x is a zero-residual solution");
    return;
  }
  int iter = 0;
  const int itmax = default_itmax(ws, o.itmax);
  const T eps_tol = tol_of<T>(o.atol) + tol_of<T>(o.rtol) * rNorm;
  if (o.verbose > 0) printf("%5s  %7s  %7s  %7s  %7s  %5s\n", "k", "‖rₖ‖", "‖Arₖ‖", "α", "β", "timer");
  if (kdisplay(iter, o.verbose)) printf("%5d  %7.1e  %7.1e  %7s  %7s  %.2fs\n", iter, (double)rNorm, (double)ArNorm, "✗ ✗ ✗ ✗", "✗ ✗ ✗ ✗", run.elapsed());
  bool solved = rNorm <= eps_tol, tired = iter >= itmax, user_exit = false, overtimed = false;
  // grouped passes (M = I, CSR operator): 3 launches and 2 read-backs per iteration instead of 11 and 4
  const bool fusedC = o.fused && A.kind == LinOp<T>::CSR && MisI;
  T uu = 0;
  bool have_uu = false;

  while (!(solved || tired || user_exit || overtimed)) {
    if (!MisI) op_apply(c, M, u, Mu, ldiv);
    const T alpha = rho / (have_uu ? uu : k_dot<T>(c, n, u, Mu));   // αₖ = ρₖ / ⟨uₖ, Muₖ⟩
    T beta = 0, ss = 0;
    if (fusedC) {
      T rr;
      car_fused_step<T>(ws, alpha, &rr, &ss);
      rNorm = std::sqrt(rr);
    } else {
      k_axpy<T>(c, n, alpha, p, x);                           // xₖ₊₁ = xₖ + αₖ * pₖ
      k_axpy<T>(c, n, -alpha, q, r);                          // rₖ₊₁ = rₖ - αₖ * qₖ
      k_axpy<T>(c, n, -alpha, Mu, s);                         // sₖ₊₁ = sₖ - αₖ * Muₖ
      rNorm = k_nrm2<T>(c, n, r);
    }
    if (history) stats.residuals.push_back(rNorm);
    const bool resid_decrease_mach = (rNorm + T(1) <= T(1));
    solved = rNorm <= eps_tol || resid_decrease_mach;
    if (!solved) {
      if (fusedC) {                                           // C2 + C3; ‖Arₖ‖ = ‖sₖ₊₁‖ from C1
        T rho_next;
        car_fused_directions<T>(ws, *A.csr, rho, &rho_next, &uu);
        have_uu = true;
        beta = rho_next / rho;
        rho = rho_next;
        ArNorm = std::sqrt(ss);
      } else {
        op_apply(c, A, s, t);                                 // tₖ₊₁ = A * sₖ₊₁
        const T rho_next = k_dot<T>(c, n, t, s);              // ρₖ₊₁ = ⟨tₖ₊₁ , sₖ₊₁⟩
        beta = rho_next / rho;                                // βₖ = ρₖ₊₁ / ρₖ
        rho = rho_next;
        k_axpby<T>(c, n, T(1), r, beta, p);                   // pₖ₊₁ = rₖ₊₁ + βₖ * pₖ
        k_axpby<T>(c, n, T(1), s, beta, q);                   // qₖ₊₁ = sₖ₊₁ + βₖ * qₖ
        k_axpby<T>(c, n, T(1), t, beta, u);                   // uₖ₊₁ = tₖ₊₁ + βₖ * uₖ
        ArNorm = MisI ? k_nrm2<T>(c, n, s) : std::sqrt(k_dot<T>(c, n, r, u));
      }
      if (history) stats.Aresiduals.push_back(ArNorm);
    }
    iter = iter + 1;
    tired = iter >= itmax;
    run.poll(iter, user_exit, overtimed);
    if (kdisplay(iter, o.verbose) && !solved)
      printf("%5d  %7.1e  %7.1e  %7.1e  %7.1e  %.2fs\n", iter, (double)rNorm, (double)ArNorm, (double)alpha, (double)beta, run.elapsed());
    if (kdisplay(iter, o.verbose) && solved)
      printf("%5d  %7.1e  %7s  %7.1e  %7s  %.2fs\n", iter, (double)rNorm, "✗ ✗ ✗ ✗", (double)alpha, "✗ ✗ ✗ ✗", run.elapsed());
  }
  if (o.verbose > 0) printf("\n");
  std::string status = "unknown";
  if (solved) status = "solution good enough given atol and rtol";
  if (tired) status = "maximum number of iterations exceeded";
  if (user_exit) status = "user-requested exit";
  if (overtimed) status = "time limit exceeded";
  run.finish(iter, solved, false, status);
}

// ===========================================================================
// minares!  (src/minares.jl:113-595), M = I (the reference refuses any other M)
//   workspace fields: vₖ (v), vₖ₊₁ (vv), wₖ₋₂ (w2), wₖ₋₁ (w1), dₖ₋₂ (d2), dₖ₋₁ (d1), q; the pairs rotate by pointer
//   (@kswap!).  Every rotation runs on the host; the fused path (CSR operator) groups the vector work of an
//   iteration into M1 (the SpMV with the w update), M2 and M3, with one read-back.
// ===========================================================================
template <class T>
void minares_solve(Workspace<T>& ws, const LinOp<T>& A, const T* b, const LinOp<T>& M, const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int n = ws.n;
  const bool history = o.history;
  const T lambda = (T)o.lambda;
  if (o.verbose > 0) printf("MINARES: system of size %d\n", n);
  if (!M.is_identity()) throw std::runtime_error("Preconditioners are not yet supported");
  T *dx = ws.dx, *x = ws.x, *q = ws.q;
  T *vk = ws.v, *vk1 = ws.vv, *wk2 = ws.w2, *wk1 = ws.w1, *dk2 = ws.d2, *dk1 = ws.d1;
  Stats& stats = ws.stats;
  const bool warm_start = ws.warm_start;
  stats.reset();
  int iter = 0;
  const int itmax = default_itmax(ws, o.itmax);
  const bool fusedM = o.fused && A.kind == LinOp<T>::CSR;

  k_fill<T>(c, n, x, T(0));
  if (warm_start) {                                           // β₁v₁ = r₀ = b - (A + λI)x₀
    op_apply(c, A, dx, vk);
    if (lambda != 0) k_axpy<T>(c, n, lambda, dx, vk);
    k_axpby<T>(c, n, T(1), b, T(-1), vk);
  } else {
    k_copy<T>(c, n, vk, b);
  }
  T betak = k_nrm2<T>(c, n, vk);
  if (betak != 0) k_scal<T>(c, n, T(1) / betak, vk);          // kdiv!
  const T beta1 = betak;
  op_apply(c, A, vk, vk1);                                    // β₂v₂ = (A + λI)v₁ - α₁v₁
  if (lambda != 0) k_axpy<T>(c, n, lambda, vk, vk1);
  T alphak = k_dot<T>(c, n, vk, vk1);
  k_axpy<T>(c, n, -alphak, vk, vk1);
  T betak1 = k_nrm2<T>(c, n, vk1);
  if (betak1 != 0) k_scal<T>(c, n, T(1) / betak1, vk1);

  T xik1 = 0;
  T tauk2 = 0, tauk1 = 0, tauk = 0;
  T thetabark2 = 0;
  T psibisk2 = 0, psibark1 = 0;
  T pik2 = 0, pik1 = 0, pik = 0;
  T chibark = 0;
  T zetabisk = 0, zetabark1 = 0, gammabark = 0;
  T lambdabark = 0, gammak1 = 0;
  T ct4 = 0, st4 = 0, ct3 = 0, st3 = 0, ct2 = 0, st2 = 0, ct1 = 0, st1 = 0, ct0 = 0, st0 = 0;   // c̃₂ₖ₋₄ ... c̃₂ₖ
  k_fill<T>(c, n, wk2, T(0));
  k_fill<T>(c, n, wk1, T(0));
  k_fill<T>(c, n, dk2, T(0));
  k_fill<T>(c, n, dk1, T(0));
  const T b1a1 = betak * alphak;                              // β₁α₁, β₁β₂: zₖ's first entries
  const T b1b2 = betak * betak1;
  T epsk2 = 0, epsk1 = 0;
  long long ell = (long long)itmax + 2;

  T rNorm = beta1;
  const T eps_tol = tol_of<T>(o.atol) + tol_of<T>(o.rtol) * rNorm;
  if (history) stats.residuals.push_back(rNorm);
  T ArNorm = std::sqrt(b1a1 * b1a1 + b1b2 * b1b2);
  const T kappa = tol_of<T>(o.atol) + tol_of<T>(o.axtol) * ArNorm;
  if (history) stats.Aresiduals.push_back(ArNorm);
  if (rNorm == 0) {
    run.finish(0, true, false, "x is a zero-residual solution");
    return;
  }
  if (o.verbose > 0) printf("%5s  %7s  %7s  %7s  %8s  %5s\n", "k", "‖rₖ‖", "‖Arₖ‖", "βₖ₊₁", "ζₖ", "timer");
  if (kdisplay(iter, o.verbose)) printf("%5d  %7.1e  %7.1e  %7.1e  %8s  %.2fs\n", iter, (double)rNorm, (double)ArNorm, (double)beta1, " ✗ ✗ ✗ ✗", run.elapsed());
  const double btol = std::pow((double)eps_of<T>(), 3.0 / 4.0);   // eps(T)^(3/4) is a Float64 in the reference

  bool solved = (rNorm <= eps_tol) || (ArNorm <= kappa), breakdown = false, tired = iter >= itmax;
  bool user_exit = false, overtimed = false;
  while (!(solved || tired || breakdown || user_exit || overtimed)) {
    iter = iter + 1;
    const long long k = iter;
    if (iter == 1) { lambdabark = alphak; gammabark = betak1; }
    T ck, sk, lambdak;
    sym_givens<T>(lambdabark, betak1, &ck, &sk, &lambdak);   // Qₖ.ₖ₊₁

    // wₖ, the last column of Wₖ = Vₖ(Rₖ)⁻¹, then the Lanczos step βₖ₊₂vₖ₊₂ = (A + λI)vₖ₊₁ - αₖ₊₁vₖ₊₁ - βₖ₊₁vₖ
    T* wk = iter == 1 ? wk1 : wk2;
    T alphak1 = 0, betak2 = 0;
    bool scale_v = false;
    if (fusedM) {
      T vv = 0;
      minares_fused_lanczos<T>(ws, *A.csr, k <= ell - 1, iter, vk, vk1, wk, wk1, epsk2, gammak1, lambdak, betak1, lambda,
                               &alphak1, &vv);
      if (k <= ell - 1) betak2 = std::sqrt(vv);
    } else {
      if (iter == 1) {
        k_divcopy<T>(c, n, wk, vk, lambdak);
      } else {
        if (iter >= 3) k_scal<T>(c, n, -epsk2, wk2);
        k_axpy<T>(c, n, -gammak1, wk1, wk);
        k_axpy<T>(c, n, T(1), vk, wk);
        k_scal<T>(c, n, T(1) / lambdak, wk);                  // kdiv!
      }
      if (k <= ell - 1) {
        op_apply(c, A, vk1, q);                               // q ← Avₖ₊₁
        k_axpby<T>(c, n, T(1), q, -betak1, vk);               // vₖ ← Avₖ₊₁ - βₖ₊₁vₖ
        if (lambda != 0) k_axpy<T>(c, n, lambda, vk1, vk);
        alphak1 = k_dot<T>(c, n, vk, vk1);
        k_axpy<T>(c, n, -alphak1, vk1, vk);
        betak2 = k_nrm2<T>(c, n, vk);
      }
    }
    if (k <= ell - 1) {
      if ((double)betak2 <= btol) ell = k + 1;                // early termination
      else scale_v = true;
      if (!fusedM && scale_v) k_scal<T>(c, n, T(1) / betak2, vk);
    }

    T epsk = 0, gammabark1 = 0, gammak = 0, lambdabark1 = 0;
    if (k <= ell - 2) { epsk = sk * betak2; gammabark1 = -ck * betak2; }
    if (k <= ell - 1) { gammak = ck * gammabark + sk * alphak1; lambdabark1 = sk * gammabark - ck * alphak1; }

    // QR factorization of Nₖ = Q̃ₖ [Uₖ; 0]
    T rhok2 = 0, lambdahatk = 0, phibark1 = 0, mubark = 0, phik1 = 0, gammahatk = 0, mubisk = 0, muk = 0;
    if (iter >= 3) { rhok2 = st4 * lambdak; lambdahatk = -ct4 * lambdak; }
    if (iter == 2) lambdahatk = lambdak;
    if (iter >= 2) {
      phibark1 = st3 * lambdahatk;
      mubark = -ct3 * lambdahatk;
      if (k <= ell - 1) { phik1 = ct2 * phibark1 + st2 * gammak; gammahatk = st2 * phibark1 - ct2 * gammak; }
      else phik1 = phibark1;
    }
    if (iter == 1) { mubark = lambdak; gammahatk = gammak; }
    if (k <= ell - 1) sym_givens<T>(mubark, gammahatk, &ct1, &st1, &mubisk);
    else mubisk = mubark;
    if (k <= ell - 2) sym_givens<T>(mubisk, epsk, &ct0, &st0, &muk);
    else muk = mubisk;

    // zₖ = (Q̃ₖ)ᵀ(β₁α₁e₁ + β₁β₂e₂)
    if (iter == 1) { zetabisk = b1a1; zetabark1 = b1b2; }
    T zetaringk, zetabisk1 = 0, zetak, zetabark2 = 0;
    if (k <= ell - 1) { zetaringk = ct1 * zetabisk + st1 * zetabark1; zetabisk1 = st1 * zetabisk - ct1 * zetabark1; }
    else zetaringk = zetabisk;
    if (k <= ell - 2) { zetak = ct0 * zetaringk; zetabark2 = st0 * zetaringk; }
    else zetak = zetaringk;

    // dₖ, the last column of Dₖ = Wₖ(Uₖ)⁻¹, and x = x₋₁ + ζₖdₖ (v_k's scaling rides in the same pass when fused)
    T* dk = iter == 1 ? dk1 : dk2;
    if (fusedM) {
      minares_fused_update<T>(ws, iter, vk, scale_v, betak2, dk, dk1, wk, rhok2, phik1, muk, zetak);
    } else {
      if (iter == 1) {
        k_divcopy<T>(c, n, dk, wk, muk);
      } else {
        if (iter >= 3) k_scal<T>(c, n, -rhok2, dk2);
        k_axpy<T>(c, n, -phik1, dk1, dk);
        k_axpy<T>(c, n, T(1), wk, dk);
        k_scal<T>(c, n, T(1) / muk, dk);                      // kdiv!
      }
      k_axpy<T>(c, n, zetak, dk, x);
    }

    if (k <= ell - 2) ArNorm = std::sqrt(zetabisk1 * zetabisk1 + zetabark2 * zetabark2);
    if (k == ell - 1) ArNorm = std::fabs(zetabisk1);
    if (k == ell) ArNorm = T(0);
    if (history) stats.Aresiduals.push_back(ArNorm);

    // LQ factorization Uₖ = L̂ₖP̂ₖ
    T psibark = 0, ch3 = 0, sh3 = 0, psibisk1 = 0, thetabark1 = 0, ch4 = 0, sh4 = 0, psik2 = 0, thetak2 = 0, deltak = 0;
    T omegak2 = 0, etak = 0;
    if (iter == 1) {
      psibark = muk;
    } else if (iter == 2) {
      sym_givens<T>(psibark1, phik1, &ch3, &sh3, &psibisk1);
      thetabark1 = sh3 * muk;
      psibark = -ch3 * muk;
    } else {
      sym_givens<T>(psibisk2, rhok2, &ch4, &sh4, &psik2);
      thetak2 = ch4 * thetabark2 + sh4 * phik1;
      deltak = sh4 * thetabark2 - ch4 * phik1;
      omegak2 = sh4 * muk;
      etak = -ch4 * muk;
      sym_givens<T>(psibark1, deltak, &ch3, &sh3, &psibisk1);
      thetabark1 = sh3 * etak;
      psibark = -ch3 * etak;
    }

    // L̂ₖtₖ = zₖ
    T xik = 0;
    if (iter == 1) {
      tauk = zetak / psibark;
    } else if (iter == 2) {
      tauk1 = tauk;
      tauk1 = tauk1 * psibark1 / psibisk1;
      xik = zetak;
      tauk = (xik - thetabark1 * tauk1) / psibark;
    } else {
      tauk2 = tauk1;
      tauk2 = tauk2 * psibisk2 / psik2;
      tauk1 = (xik1 - thetak2 * tauk2) / psibisk1;
      xik = zetak - omegak2 * tauk2;
      tauk = (xik - thetabark1 * tauk1) / psibark;
    }

    // (Qₖ)ᵀβ₁e₁ = (χ₁, ..., χₖ, χbarₖ₊₁)
    if (iter == 1) chibark = beta1;
    const T chik = ck * chibark;
    const T chibark1 = sk * chibark;

    // pₖ₊₁ = [P̂ₖ 0; 0 1](Qₖ)ᵀβ₁e₁
    if (iter == 1) {
      pik = chik;
    } else if (iter == 2) {
      const T piaux1 = pik1;
      pik1 = ch3 * piaux1 + sh3 * chik;
      pik = sh3 * piaux1 - ch3 * chik;
    } else {
      const T piaux2 = pik2;
      pik2 = ch4 * piaux2 + sh4 * chik;
      pik = sh4 * piaux2 - ch4 * chik;
      const T piaux1 = pik1;
      pik1 = ch3 * piaux1 + sh3 * pik;
      pik = sh3 * piaux1 - ch3 * pik;
    }
    const T pik_1 = chibark1;                                 // πₖ₊₁

    if (iter == 1) rNorm = std::sqrt((pik - tauk) * (pik - tauk) + pik_1 * pik_1);
    else rNorm = std::sqrt((pik1 - tauk1) * (pik1 - tauk1) + (pik - tauk) * (pik - tauk) + pik_1 * pik_1);
    if (history) stats.residuals.push_back(rNorm);

    breakdown = (double)betak1 <= btol;
    solved = (rNorm <= eps_tol) || (ArNorm <= kappa);
    tired = iter >= itmax;
    run.poll(iter, user_exit, overtimed);

    std::swap(vk, vk1);
    if (iter >= 2) {
      std::swap(wk2, wk1);
      std::swap(dk2, dk1);
      epsk2 = epsk1;
      ct4 = ct2; st4 = st2;
      xik1 = xik;
      psibisk2 = psibisk1;
      thetabark2 = thetabark1;
      pik2 = pik1;
    }
    ct3 = ct1; st3 = st1;
    ct2 = ct0; st2 = st0;
    betak = betak1;
    chibark = chibark1;
    psibark1 = psibark;
    pik1 = pik;
    if (k <= ell - 1) {
      alphak = alphak1;
      betak1 = betak2;
      gammak1 = gammak;
      lambdabark = lambdabark1;
      zetabisk = zetabisk1;
    }
    if (k <= ell - 2) {
      epsk1 = epsk;
      gammabark = gammabark1;
      zetabark1 = zetabark2;
    }
    if (kdisplay(iter, o.verbose)) printf("%5d  %7.1e  %7.1e  %7.1e  %8.1e  %.2fs\n", iter, (double)rNorm, (double)ArNorm, (double)betak, (double)zetak, run.elapsed());
  }
  if (o.verbose > 0) printf("\n");
  std::string status = "unknown";                             // a breakdown alone leaves it so
  if (solved) status = "solution good enough given atol, rtol and Artol";
  if (tired) status = "maximum number of iterations exceeded";
  if (user_exit) status = "user-requested exit";
  if (overtimed) status = "time limit exceeded";
  run.finish(iter, solved, false, status);
}

#define INST(T)                                                                                                          \
  template void car_solve<T>(Workspace<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const SolveOpts&);             \
  template void minares_solve<T>(Workspace<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const SolveOpts&);         \
  template void cgs_solve<T>(Workspace<T>&, const LinOp<T>&, const T*, const T*, const LinOp<T>&, const LinOp<T>&, const SolveOpts&); \
  template void cg_lanczos_solve<T>(Workspace<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const SolveOpts&);        \
  template void dqgmres_solve<T>(Workspace<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const LinOp<T>&, const SolveOpts&); \
  template void diom_solve<T>(Workspace<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const LinOp<T>&, const SolveOpts&); \
  template void cr_solve<T>(Workspace<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const SolveOpts&);
INST(double)
INST(float)
#undef INST

}  // namespace kb
