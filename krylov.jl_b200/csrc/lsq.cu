// lsq.cu -- host control flow of lsqr! (src/lsqr.jl:174-440) and lsmr! (src/lsmr.jl:178-455) on an m x n operator.
// Both run the Golub-Kahan bidiagonalization: one product with A and one with A^H per iteration.  The primitive path
// restates the reference line by line over blas1.cu / spmv.cu (11 launches per LSQR iteration, 12 per LSMR one).  When
// A is a CSR operator, M = N = I and there is no trust region, the fused path runs the same iteration as 3 launches
// (fused_phases.cu: P1 on A, P2 on A^T, P3 over n) and one read-back (LSMR: two, its tests need ||x|| after P3).  The
// scalar recurrences, stopping tests and status strings run on the host, unchanged.
// lslq! (src/lslq.jl:201-520) runs the same Golub-Kahan step (fused: LSQR's P1 / P2 and its own update pass).
// cgls! (src/cgls.jl:129-243) and crls! (src/crls.jl:120-268) run the normal-equations recurrences on the same operator
// pair: 8 / 11 launches per iteration on the primitives, 4 fused ones (fused_phases.cu) and one read-back when A is a
// CSR operator, M = I and there is no trust region.  cgne! and crmr! run them on A Aᴴ y = b, x = Aᴴ y: 2 and 4 fused
// launches per iteration and one read-back when A is a CSR operator, N = I and λ = 0.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <limits>

#include "solver_common.h"

namespace kb {

namespace {

// knorm_elliptic(n, x, y) (src/krylov_utils.jl:319)
template <class T> T knorm_elliptic(Ctx& c, int n, const T* x, const T* y) {
  return x == y ? k_nrm2<T>(c, n, x) : std::sqrt(k_dot<T>(c, n, x, y));
}

template <class T> T err_window_norm(const std::vector<T>& e) {   // knorm(window, err_vec)
  T ssq = 0;
  for (T v : e) ssq += v * v;
  return std::sqrt(ssq);
}

// to_boundary(n, x, d, z, radius; dNorm2) with M = I, raising where the reference raises
template <class T> void boundary_roots(Ctx& c, int n, const T* x, const T* d, T radius, T dNorm2, T* t1, T* t2) {
  LinOp<T> I;
  const int e = to_boundary<T>(c, n, x, d, nullptr, radius, dNorm2, I, false, t1, t2);
  if (e == 2) throw std::runtime_error("zero direction");
  if (e == 3) throw std::runtime_error("outside of the trust region");
  if (e) throw std::runtime_error("The quadratic `q` doesn't have real roots.");
}

// Step to the trust-region boundary along d (lsqr.jl:355-358, lsmr.jl:358-361): returns the clipped sigma.
template <class T> T clip_to_boundary(Ctx& c, int n, const T* x, const T* d, T radius, T sigma, bool& on_boundary) {
  T t1, t2;
  boundary_roots<T>(c, n, x, d, radius, T(0), &t1, &t2);
  const T tmax = std::max(t1, t2), tmin = std::min(t1, t2);
  on_boundary = sigma > tmax || sigma < tmin;
  return sigma > 0 ? std::min(sigma, tmax) : std::max(sigma, tmin);
}

struct Setup {
  bool MisI, NisI, fused;
};

// Common prologue: argument checks, lazily allocated vectors, x = 0, Mu = b, u = M Mu, beta_1.
template <class T>
Setup lsq_prologue(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& M, const LinOp<T>& N,
                   const SolveOpts& o, T* beta1) {
  Ctx& c = ws.ctx;
  const int m = ws.m, n = ws.n;
  Setup s;
  s.MisI = M.is_identity(); s.NisI = N.is_identity();
  s.fused = o.fused && A.kind == LinOp<T>::CSR && At.kind == LinOp<T>::CSR && s.MisI && s.NisI && !(o.radius > 0);
  allocate_if(true, ws, ws.Mu, m);                // u, Mu and Av have m entries
  allocate_if(true, ws, ws.Nv);
  allocate_if(!s.MisI, ws, ws.u, m);
  allocate_if(!s.NisI, ws, ws.v);
  allocate_if(!s.fused, ws, ws.Av, m);
  allocate_if(!s.fused, ws, ws.Atu);
  ws.stats.reset();
  ws.stats.Anorm = NAN;
  k_fill<T>(c, n, ws.x, T(0));
  k_copy<T>(c, m, ws.Mu, b);
  T* u = s.MisI ? ws.Mu : ws.u;
  if (!s.MisI) op_apply(c, M, ws.Mu, u, o.ldiv);
  *beta1 = m > 0 ? knorm_elliptic<T>(c, m, u, ws.Mu) : T(0);
  return s;
}

// Golub-Kahan start: u /= beta_1, Nv = A^H u, v = N Nv (lsqr.jl:230-234).
template <class T> void lsq_start(Workspace<T>& ws, const Setup& s, const LinOp<T>& At, const LinOp<T>& N, bool ldiv, T beta1) {
  Ctx& c = ws.ctx;
  const int m = ws.m, n = ws.n;
  T* u = s.MisI ? ws.Mu : ws.u;
  k_scal<T>(c, m, T(1) / beta1, u);
  if (!s.MisI) k_scal<T>(c, m, T(1) / beta1, ws.Mu);
  if (s.fused) {
    op_apply(c, At, u, ws.Nv);                  // kmul!(Aᴴu, Aᴴ, u) ; kcopy!(n, Nv, Aᴴu) without the copy
  } else {
    op_apply(c, At, u, ws.Atu);
    k_copy<T>(c, n, ws.Nv, ws.Atu);
  }
  if (!s.NisI) op_apply(c, N, ws.Nv, ws.v, ldiv);
}

// One Golub-Kahan step on the primitives (lsqr.jl:299-318): returns the new beta; alpha is updated when beta != 0.
// `on_beta` runs between the two products (LSQR's Anorm update).
template <class T, class OnBeta>
T lsq_bidiag_step(Workspace<T>& ws, const Setup& s, const LinOp<T>& A, const LinOp<T>& At, const LinOp<T>& M, const LinOp<T>& N,
                  bool ldiv, T& alpha, OnBeta on_beta) {
  Ctx& c = ws.ctx;
  const int m = ws.m, n = ws.n;
  T* u = s.MisI ? ws.Mu : ws.u;
  T* v = s.NisI ? ws.Nv : ws.v;
  op_apply(c, A, v, ws.Av);
  k_axpby<T>(c, m, T(1), ws.Av, -alpha, ws.Mu);
  if (!s.MisI) op_apply(c, M, ws.Mu, u, ldiv);
  const T beta = knorm_elliptic<T>(c, m, u, ws.Mu);
  if (beta != 0) {
    k_scal<T>(c, m, T(1) / beta, u);
    if (!s.MisI) k_scal<T>(c, m, T(1) / beta, ws.Mu);
    on_beta(beta);
    op_apply(c, At, u, ws.Atu);
    k_axpby<T>(c, n, T(1), ws.Atu, -beta, ws.Nv);
    if (!s.NisI) op_apply(c, N, ws.Nv, v, ldiv);
    alpha = knorm_elliptic<T>(c, n, v, ws.Nv);
    if (alpha != 0) {
      k_scal<T>(c, n, T(1) / alpha, v);
      if (!s.NisI) k_scal<T>(c, n, T(1) / alpha, ws.Nv);
    }
  }
  return beta;
}

struct Exit {
  bool solved = false, tired = false, ill_cond = false, ill_cond_mach = false, ill_cond_lim = false;
  bool zero_resid = false, fwd_err = false, on_boundary = false, user_exit = false, overtimed = false;
  const char* status() const {   // termination status, in the reference's order of precedence (lsqr.jl:423-431)
    const char* st = "unknown";
    if (tired) st = "maximum number of iterations exceeded";
    if (ill_cond_mach) st = "condition number seems too large for this machine";
    if (ill_cond_lim) st = "condition number exceeds tolerance";
    if (solved) st = "found approximate minimum least-squares solution";
    if (zero_resid) st = "found approximate zero-residual solution";
    if (fwd_err) st = "truncated forward error small enough";
    if (on_boundary) st = "on trust-region boundary";
    if (user_exit) st = "user-requested exit";
    if (overtimed) st = "time limit exceeded";
    return st;
  }
};

template <class T> int ls_itmax(const Workspace<T>& ws, int itmax) {
  if (itmax != 0) return itmax;
  const long long mn = (long long)ws.m + ws.n;
  return mn > 2147483647LL ? 2147483647 : (int)mn;
}

}  // namespace

// ===========================================================================
// lsqr!  (src/lsqr.jl:174-440)
// ===========================================================================
template <class T>
void lsqr_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& M, const LinOp<T>& N,
                const SolveOpts& o) {
  // LSQR / LSMR workspaces refuse warm starts and row partitioning, so run.finish never adds dx and the cross-rank
  // OR in run.poll is a no-op for them; they share the protocol for its callback / clock / sync order.
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int m = ws.m, n = ws.n;
  const bool history = o.history, ldiv = o.ldiv;
  if (o.verbose > 0) printf("LSQR: system of %d equations in %d variables\n", m, n);
  const T lambda = (T)o.lambda, lambda2 = lambda * lambda;
  const T conlim = o.conlim < 0 ? T(1) / std::sqrt(eps_of<T>()) : (T)o.conlim;
  const T ctol = conlim > 0 ? T(1) / conlim : T(0);
  const T etol = tol_of<T>(o.etol), axtol = tol_of<T>(o.axtol), btol = tol_of<T>(o.btol);
  const T atol = tol_of<T>(o.atol), rtol = tol_of<T>(o.rtol), radius = (T)o.radius;
  Stats& stats = ws.stats;
  std::vector<T>& err_vec = ws.err_vec;

  T beta1;
  const Setup s = lsq_prologue<T>(ws, A, At, b, M, N, o, &beta1);
  if (beta1 == 0) {
    run.finish(0, true, false, "x is a zero-residual solution");
    if (history) { stats.residuals.push_back(0); stats.Aresiduals.push_back(0); }
    return;
  }
  T beta = beta1;
  lsq_start<T>(ws, s, At, N, ldiv, beta1);
  T* v = s.NisI ? ws.Nv : ws.v;
  T Anorm2 = k_dot<T>(c, n, v, ws.Nv);
  T Anorm = std::sqrt(Anorm2);
  T alpha = Anorm;
  T Acond = 0, xNorm = 0, xNorm2 = 0, dNorm2 = 0, c2 = -1, s2 = 0, z = 0;
  T xENorm2 = 0, err_lbnd = 0;
  const int window = (int)err_vec.size();
  std::fill(err_vec.begin(), err_vec.end(), T(0));
  int iter = 0;
  const int itmax = ls_itmax(ws, o.itmax);
  if (o.verbose > 0) {
    printf("%5s  %7s  %7s  %7s  %7s  %7s  %7s  %7s  %7s  %5s\n", "k", "α", "β", "‖r‖", "‖Aᴴr‖", "compat", "backwrd", "‖A‖", "κ(A)", "timer");
    printf("%5d  %7.1e  %7.1e  %7.1e  %7.1e  %7.1e  %7.1e  %7.1e  %7.1e  %.2fs\n", iter, (double)beta1, (double)alpha, (double)beta1,
           (double)alpha, 0.0, 1.0, (double)Anorm, (double)Acond, run.elapsed());
  }
  T rNorm = beta1, r1Norm = rNorm, r2Norm = rNorm, res2 = 0;
  (void)r1Norm;
  if (history) stats.residuals.push_back(r2Norm);
  T ArNorm = alpha * beta;
  const T ArNorm0 = ArNorm;
  if (history) stats.Aresiduals.push_back(ArNorm);
  if (alpha == 0) {                                          // Aᴴb = 0: x = 0 is a minimum least-squares solution
    run.finish(0, true, false, "x is a minimum least-squares solution");
    return;
  }
  k_scal<T>(c, n, T(1) / alpha, v);
  if (!s.NisI) k_scal<T>(c, n, T(1) / alpha, ws.Nv);
  k_copy<T>(c, n, ws.w, v);

  T phibar = beta1, rhobar = alpha;
  Exit ex;
  const bool solved_lim0 = ArNorm / (Anorm * rNorm) <= axtol;
  const bool solved_mach0 = T(1) + ArNorm / (Anorm * rNorm) <= T(1);
  ex.solved = solved_mach0 || solved_lim0;
  ex.tired = iter >= itmax;
  ex.zero_resid = (T(1) + rNorm / beta1 <= T(1)) || (rNorm / beta1 <= axtol);

  while (!(ex.solved || ex.tired || ex.ill_cond || ex.user_exit || ex.overtimed)) {
    iter = iter + 1;
    T ww = 0;
    bool scale_v = false;
    if (s.fused) {
      // P1 + P2 and one read-back of {beta, alpha, <w, w>}; v /= alpha is applied by P3
      T alpha_new;
      lsq_fused_bidiag<T>(ws, *A.csr, *At.csr, iter == 1, alpha, true, &beta, &alpha_new, &ww);
      if (beta != 0) {
        Anorm2 = Anorm2 + alpha * alpha + beta * beta;       // = ‖B_{k-1}‖²
        if (lambda > 0) Anorm2 += lambda2;
        alpha = alpha_new;
        scale_v = alpha != 0;
      }
    } else {
      beta = lsq_bidiag_step<T>(ws, s, A, At, M, N, ldiv, alpha, [&](T bt) {
        Anorm2 = Anorm2 + alpha * alpha + bt * bt;
        if (lambda > 0) Anorm2 += lambda2;
      });
    }

    // 1. Eliminate the regularization parameter.
    T c1, s1, rhobar1;
    sym_givens<T>(rhobar, lambda, &c1, &s1, &rhobar1);
    const T psi = s1 * phibar;
    phibar = c1 * phibar;
    // 2. Eliminate beta.
    T cs, sn, rho;
    sym_givens<T>(rhobar1, beta, &cs, &sn, &rho);
    const T phi = cs * phibar;
    phibar = sn * phibar;

    xENorm2 = xENorm2 + phi * phi;
    err_vec[iter % window] = phi;
    if (iter >= window) err_lbnd = err_window_norm(err_vec);

    const T tau = sn * phi;
    const T theta = sn * alpha;
    rhobar = -cs * alpha;
    if (!s.fused) ww = k_dot<T>(c, n, ws.w, ws.w);
    dNorm2 += ww / (rho * rho);

    T sigma = phi / rho;
    if (radius > 0) sigma = clip_to_boundary<T>(c, n, ws.x, ws.w, radius, sigma, ex.on_boundary);

    if (s.fused) {
      lsq_fused_update<T>(ws, false, scale_v, T(1) / alpha, sigma, theta / rho, T(0));
    } else {
      k_axpy<T>(c, n, sigma, ws.w, ws.x);                       // x = x + ϕ / ρ * w
      k_axpby<T>(c, n, T(1), v, -theta / rho, ws.w);            // w = v - θ / ρ * w
    }

    // plane rotation on the right: estimate of ‖x‖
    const T delta = s2 * rho;
    const T gammabar = -c2 * rho;
    const T rhs = phi - delta * z;
    const T zbar = rhs / gammabar;
    xNorm = std::sqrt(xNorm2 + zbar * zbar);
    T gamma;
    sym_givens<T>(gammabar, theta, &c2, &s2, &gamma);
    z = rhs / gamma;
    xNorm2 += z * z;

    Anorm = std::sqrt(Anorm2);
    Acond = Anorm * std::sqrt(dNorm2);
    const T res1 = phibar * phibar;
    res2 += psi * psi;
    rNorm = std::sqrt(res1 + res2);

    ArNorm = alpha * std::fabs(tau);
    if (history) stats.Aresiduals.push_back(ArNorm);

    const T r1sq = rNorm * rNorm - lambda2 * xNorm2;
    r1Norm = std::sqrt(std::fabs(r1sq));
    if (r1sq < 0) r1Norm = -r1Norm;
    r2Norm = rNorm;
    if (history) stats.residuals.push_back(r2Norm);

    const T test1 = rNorm / beta1;
    const T test2 = ArNorm / (Anorm * rNorm);
    const T test3 = T(1) / Acond;
    const T t1 = test1 / (T(1) + Anorm * xNorm / beta1);
    const T rNormtol = btol + axtol * Anorm * xNorm / beta1;
    if (kdisplay(iter, o.verbose))
      printf("%5d  %7.1e  %7.1e  %7.1e  %7.1e  %7.1e  %7.1e  %7.1e  %7.1e  %.2fs\n", iter, (double)alpha, (double)beta, (double)rNorm,
             (double)ArNorm, (double)test1, (double)test2, (double)Anorm, (double)Acond, run.elapsed());

    ex.ill_cond_mach = (T(1) + test3 <= T(1));
    const bool solved_mach = (T(1) + test2 <= T(1));
    const bool zero_resid_mach = (T(1) + t1 <= T(1));
    run.poll(iter, ex.user_exit, ex.overtimed);
    ex.tired = iter >= itmax;
    ex.ill_cond_lim = (test3 <= ctol);
    const bool solved_lim = (test2 <= axtol);
    const bool solved_opt = ArNorm <= atol + rtol * ArNorm0;
    const bool zero_resid_lim = (test1 <= rNormtol);
    if (iter >= window) ex.fwd_err = err_lbnd <= etol * std::sqrt(xENorm2);
    ex.ill_cond = ex.ill_cond_mach || ex.ill_cond_lim;
    ex.zero_resid = zero_resid_mach || zero_resid_lim;
    ex.solved = solved_mach || solved_lim || solved_opt || ex.zero_resid || ex.fwd_err || ex.on_boundary;
  }
  if (o.verbose > 0) printf("\n");
  run.finish(iter, ex.solved, !ex.zero_resid, ex.status());
}

// ===========================================================================
// lsmr!  (src/lsmr.jl:178-455)
// ===========================================================================
template <class T>
void lsmr_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& M, const LinOp<T>& N,
                const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int m = ws.m, n = ws.n;
  const bool history = o.history, ldiv = o.ldiv;
  if (o.verbose > 0) printf("LSMR: system of %d equations in %d variables\n", m, n);
  const T lambda = (T)o.lambda;
  const T conlim = o.conlim < 0 ? T(1) / std::sqrt(eps_of<T>()) : (T)o.conlim;
  const T ctol = conlim > 0 ? T(1) / conlim : T(0);
  const T etol = tol_of<T>(o.etol), axtol = tol_of<T>(o.axtol), btol = tol_of<T>(o.btol);
  const T atol = tol_of<T>(o.atol), rtol = tol_of<T>(o.rtol), radius = (T)o.radius;
  Stats& stats = ws.stats;
  std::vector<T>& err_vec = ws.err_vec;

  T beta1;
  const Setup s = lsq_prologue<T>(ws, A, At, b, M, N, o, &beta1);
  if (beta1 == 0) {
    run.finish(0, true, false, "x is a zero-residual solution");
    if (history) { stats.residuals.push_back(0); stats.Aresiduals.push_back(0); }
    return;
  }
  T beta = beta1;
  lsq_start<T>(ws, s, At, N, ldiv, beta1);
  T* v = s.NisI ? ws.Nv : ws.v;
  T alpha = knorm_elliptic<T>(c, n, v, ws.Nv);

  T zetabar = alpha * beta, alphabar = alpha, rho = 1, rhobar = 1, cbar = 1, sbar = 0;
  T betadd = beta, betad = 0, rhodold = 1, tautildeold = 0, thetatilde = 0, zeta = 0, d = 0;
  T Anorm2 = alpha * alpha, maxrbar = 0;
  T minrbar = std::min(std::numeric_limits<T>::max(), (T)1.0e+100);
  T Acond = maxrbar / minrbar, Anorm = std::sqrt(Anorm2), xNorm = 0;
  T rNorm = beta;
  if (history) stats.residuals.push_back(rNorm);
  T ArNorm = alpha * beta;
  const T ArNorm0 = ArNorm;
  if (history) stats.Aresiduals.push_back(ArNorm);
  T xENorm2 = 0, err_lbnd = 0;
  const int window = (int)err_vec.size();
  std::fill(err_vec.begin(), err_vec.end(), T(0));
  int iter = 0;
  const int itmax = ls_itmax(ws, o.itmax);
  if (o.verbose > 0) {
    printf("%5s  %7s  %7s  %7s  %7s  %8s  %8s  %7s  %5s\n", "k", "‖r‖", "‖Aᴴr‖", "β", "α", "cos", "sin", "‖A‖²", "timer");
    printf("%5d  %7.1e  %7.1e  %7.1e  %7.1e  %8.1e  %8.1e  %7.1e  %.2fs\n", iter, (double)beta1, (double)alpha, (double)beta1,
           (double)alpha, 0.0, 1.0, (double)Anorm2, run.elapsed());
  }
  if (alpha == 0) {                                          // Aᴴb = 0: x = 0 is a minimum least-squares solution
    run.finish(0, true, false, "x is a minimum least-squares solution");
    stats.Anorm = Anorm;
    return;
  }
  k_scal<T>(c, n, T(1) / alpha, v);
  if (!s.NisI) k_scal<T>(c, n, T(1) / alpha, ws.Nv);
  k_copy<T>(c, n, ws.h, v);
  k_fill<T>(c, n, ws.hbar, T(0));

  Exit ex;
  ex.solved = (rNorm <= axtol);
  ex.tired = iter >= itmax;

  while (!(ex.solved || ex.tired || ex.ill_cond || ex.user_exit || ex.overtimed)) {
    iter = iter + 1;
    bool scale_v = false;
    if (s.fused) {
      T alpha_new, unused;
      lsq_fused_bidiag<T>(ws, *A.csr, *At.csr, iter == 1, alpha, false, &beta, &alpha_new, &unused);
      if (beta != 0) { alpha = alpha_new; scale_v = alpha != 0; }
    } else {
      beta = lsq_bidiag_step<T>(ws, s, A, At, M, N, ldiv, alpha, [](T) {});
    }

    // Continue QR factorization
    T chat, shat, alphahat;
    sym_givens<T>(alphabar, lambda, &chat, &shat, &alphahat);
    const T rhoold = rho;
    T cs, sn;
    sym_givens<T>(alphahat, beta, &cs, &sn, &rho);
    const T thetanew = sn * alpha;
    alphabar = cs * alpha;

    const T rhobarold = rhobar;
    const T zetaold = zeta;
    const T thetabar = sbar * rho;
    const T rhotemp = cbar * rho;
    sym_givens<T>(rhotemp, thetanew, &cbar, &sbar, &rhobar);
    zeta = cbar * zetabar;
    zetabar = -sbar * zetabar;

    xENorm2 = xENorm2 + zeta * zeta;
    err_vec[iter % window] = zeta;
    if (iter >= window) err_lbnd = err_window_norm(err_vec);

    // Update h, hbar and x.
    const T delta = thetabar * rho / (rhoold * rhobarold);   // δₖ = θbarₖ * ρₖ / (ρₖ₋₁ * ρbarₖ₋₁)
    T sigma = zeta / (rho * rhobar);
    if (s.fused) {
      xNorm = lsq_fused_update<T>(ws, true, scale_v, T(1) / alpha, sigma, thetanew / rho, delta);
    } else {
      k_axpby<T>(c, n, T(1), ws.h, -delta, ws.hbar);            // ĥₖ = hₖ - δₖ * ĥₖ₋₁
      if (radius > 0) sigma = clip_to_boundary<T>(c, n, ws.x, ws.hbar, radius, sigma, ex.on_boundary);
      k_axpy<T>(c, n, sigma, ws.hbar, ws.x);                    // xₖ = xₖ₋₁ + σₖ * ĥₖ
      k_axpby<T>(c, n, T(1), v, -thetanew / rho, ws.h);         // hₖ₊₁ = vₖ₊₁ - (θₖ₊₁/ρₖ) * hₖ
    }

    // Estimate ‖r‖.
    const T betaacute = chat * betadd;
    const T betacheck = -shat * betadd;
    const T betahat = cs * betaacute;
    betadd = -sn * betaacute;
    const T thetatildeold = thetatilde;
    T ctildeold, stildeold, rhotildeold;
    sym_givens<T>(rhodold, thetabar, &ctildeold, &stildeold, &rhotildeold);
    thetatilde = stildeold * rhobar;
    rhodold = ctildeold * rhobar;
    betad = -stildeold * betad + ctildeold * betahat;
    tautildeold = (zetaold - thetatildeold * tautildeold) / rhotildeold;
    const T taud = (zeta - thetatilde * tautildeold) / rhodold;
    d = d + betacheck * betacheck;
    rNorm = std::sqrt(d + (betad - taud) * (betad - taud) + betadd * betadd);
    if (history) stats.residuals.push_back(rNorm);

    // Estimate ‖A‖.
    Anorm2 += beta * beta;
    Anorm = std::sqrt(Anorm2);
    Anorm2 += alpha * alpha;

    // Estimate cond(A).
    maxrbar = std::max(maxrbar, rhobarold);
    if (iter > 1) minrbar = std::min(minrbar, rhobarold);
    Acond = std::max(maxrbar, rhotemp) / std::min(minrbar, rhotemp);

    // Test for convergence.
    ArNorm = std::fabs(zetabar);
    if (history) stats.Aresiduals.push_back(ArNorm);
    if (!s.fused) xNorm = k_nrm2<T>(c, n, ws.x);

    const T test1 = rNorm / beta1;
    const T test2 = ArNorm / (Anorm * rNorm);
    const T test3 = T(1) / Acond;
    const T t1 = test1 / (T(1) + Anorm * xNorm / beta1);
    const T rNormtol = btol + axtol * Anorm * xNorm / beta1;
    if (kdisplay(iter, o.verbose))
      printf("%5d  %7.1e  %7.1e  %7.1e  %7.1e  %8.1e  %8.1e  %7.1e  %.2fs\n", iter, (double)rNorm, (double)ArNorm, (double)beta,
             (double)alpha, (double)cs, (double)sn, (double)Anorm2, run.elapsed());

    ex.ill_cond_mach = (T(1) + test3 <= T(1));
    const bool solved_mach = (T(1) + test2 <= T(1));
    const bool zero_resid_mach = (T(1) + t1 <= T(1));
    run.poll(iter, ex.user_exit, ex.overtimed);
    ex.tired = iter >= itmax;
    ex.ill_cond_lim = (test3 <= ctol);
    const bool solved_lim = (test2 <= axtol);
    const bool solved_opt = ArNorm <= atol + rtol * ArNorm0;
    const bool zero_resid_lim = (test1 <= rNormtol);
    if (iter >= window) ex.fwd_err = err_lbnd <= etol * std::sqrt(xENorm2);
    ex.ill_cond = ex.ill_cond_mach || ex.ill_cond_lim;
    ex.zero_resid = zero_resid_mach || zero_resid_lim;
    ex.solved = solved_mach || solved_lim || solved_opt || ex.zero_resid || ex.fwd_err || ex.on_boundary;
  }
  if (o.verbose > 0) printf("\n");
  stats.Anorm = Anorm;
  run.finish(iter, ex.solved, !ex.zero_resid, ex.status());
}

// ===========================================================================
// lslq!  (src/lslq.jl:201-520).  Unlike LSQR, `iter` is incremented at the END of the body, so the forward-error
// window, the `tired` test and the CG-bound guard see the count from before the increment; λ is overwritten by the
// regularization rotation while λ² keeps its initial value.
// ===========================================================================
template <class T>
void lslq_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& M, const LinOp<T>& N,
                const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int m = ws.m, n = ws.n;
  const bool history = o.history, ldiv = o.ldiv;
  if (o.verbose > 0) printf("LSLQ: system of %d equations in %d variables\n", m, n);
  T lambda = (T)o.lambda;
  const T lambda2 = lambda * lambda;
  const T sigma = (T)o.sigma;
  const T conlim = o.conlim < 0 ? T(1) / std::sqrt(eps_of<T>()) : (T)o.conlim;
  const T ctol = conlim > 0 ? T(1) / conlim : T(0);
  const T etol = tol_of<T>(o.etol), utol = tol_of<T>(o.utol), btol = tol_of<T>(o.btol);
  const T atol = tol_of<T>(o.atol), rtol = tol_of<T>(o.rtol);
  Stats& stats = ws.stats;
  std::vector<T>& err_vec = ws.err_vec;
  (void)btol;                                                   // lslq.jl computes `tol` from btol and never reads it

  T beta1;
  const Setup s = lsq_prologue<T>(ws, A, At, b, M, N, o, &beta1);
  if (beta1 == 0) {
    run.finish(0, true, false, "x is a zero-residual solution");
    stats.error_with_bnd = false;
    if (history) { stats.residuals.push_back(0); stats.Aresiduals.push_back(0); }
    return;
  }
  T beta = beta1;
  lsq_start<T>(ws, s, At, N, ldiv, beta1);
  T* v = s.NisI ? ws.Nv : ws.v;
  T alpha = knorm_elliptic<T>(c, n, v, ws.Nv);
  if (alpha == 0) {                                             // Aᴴb = 0: x = 0 is a minimum least-squares solution
    run.finish(0, true, false, "x is a minimum least-squares solution");
    stats.error_with_bnd = false;
    if (history) { stats.residuals.push_back(beta1); stats.Aresiduals.push_back(0); }
    return;
  }
  k_scal<T>(c, n, T(1) / alpha, v);
  if (!s.NisI) k_scal<T>(c, n, T(1) / alpha, ws.Nv);

  T Anorm2 = alpha * alpha, Anorm = alpha;
  T sigmax = 0, sigmin = std::numeric_limits<T>::infinity(), Acond = 0;
  T xlqNorm = 0, xlqNorm2 = 0, xcgNorm2 = 0;
  k_copy<T>(c, n, ws.w, v);                                     // w̄₁ = v₁
  T err_lbnd = 0;
  const int window = (int)err_vec.size();
  std::fill(err_vec.begin(), err_vec.end(), T(0));
  bool complex_error_bnd = false;

  T alphaL = alpha, betaL = beta, rhobar = -sigma, gammabar = alpha, psi = beta1;
  T cc = -1, ss = 0, delta = -1, tau = alpha * beta1, zeta = 0, zetabar = 0, zetatilde = 0, csig = -1;
  T rNorm = beta1;
  if (history) stats.residuals.push_back(rNorm);
  T ArNorm = alpha * beta;
  if (history) stats.Aresiduals.push_back(ArNorm);
  int iter = 0;
  const int itmax = ls_itmax(ws, o.itmax);
  if (o.verbose > 0) {
    printf("%5s  %7s  %7s  %7s  %7s  %8s  %8s  %7s  %7s  %7s  %5s\n", "k", "‖r‖", "‖Aᴴr‖", "β", "α", "cos", "sin", "‖A‖²", "κ(A)",
           "‖xL‖", "timer");
    printf("%5d  %7.1e  %7.1e  %7.1e  %7.1e  %8.1e  %8.1e  %7.1e  %7.1e  %7.1e  %.2fs\n", iter, (double)rNorm, (double)ArNorm,
           (double)beta, (double)alpha, (double)cc, (double)ss, (double)Anorm2, (double)Acond, (double)xlqNorm, run.elapsed());
  }

  const T eps = atol + rtol * beta1;
  bool solved = rNorm <= eps, tired = iter >= itmax, ill_cond = false, ill_cond_mach = false, ill_cond_lim = false;
  bool zero_resid = false, fwd_err_lbnd = false, fwd_err_ubnd = false, user_exit = false, overtimed = false;

  while (!(solved || tired || ill_cond || user_exit || overtimed)) {
    // Golub-Kahan step: βₖ₊₁Muₖ₊₁ = Avₖ - αₖMuₖ, αₖ₊₁Nvₖ₊₁ = Aᴴuₖ₊₁ - βₖ₊₁Nvₖ
    bool scale_v = false;
    if (s.fused) {                                              // P1 + P2 and one read-back; v /= alpha is applied below
      T alpha_new, unused;
      lsq_fused_bidiag<T>(ws, *A.csr, *At.csr, iter == 0, alpha, false, &beta, &alpha_new, &unused);
      if (beta != 0) { alpha = alpha_new; scale_v = alpha != 0; }
    } else {
      beta = lsq_bidiag_step<T>(ws, s, A, At, M, N, ldiv, alpha, [](T) {});
    }
    if (beta != 0) {
      alphaL = alpha;                                           // rotate out the regularization term if present
      betaL = beta;
      if (lambda != 0) {
        T cL, sL;
        sym_givens<T>(beta, lambda, &cL, &sL, &betaL);
        alphaL = cL * alpha;
        lambda = std::sqrt(lambda2 + (sL * alpha) * (sL * alpha));   // the rotation updates the next λ
      }
      Anorm2 = Anorm2 + alphaL * alphaL + betaL * betaL;      // = ‖Lₖ‖²
      Anorm = std::sqrt(Anorm2);
    }

    // Continue the QR factorization of Bₖ
    T cp, sp, gamma;
    sym_givens<T>(gammabar, betaL, &cp, &sp, &gamma);
    tau = -tau * delta / gamma;
    delta = sp * alphaL;
    gammabar = -cp * alphaL;

    T omega = 0;
    if (sigma > 0 && !complex_error_bnd) {                      // QR factorization for the error estimate
      T mubar = -csig * gamma, ssig, rho;
      sym_givens<T>(rhobar, gamma, &csig, &ssig, &rho);
      rhobar = ssig * mubar + csig * sigma;
      mubar = -csig * delta;
      const T h = delta * csig / rhobar;                        // eigenvector component and Gauss-Radau parameter
      const T disc = sigma * (sigma - delta * h);
      if (disc < 0) complex_error_bnd = true; else omega = std::sqrt(disc);
      sym_givens<T>(rhobar, delta, &csig, &ssig, &rho);
      rhobar = ssig * mubar + csig * sigma;
    }

    // Continue the LQ factorization of Rₖ
    const T epsbar = -gamma * cc;
    const T eta = gamma * ss;
    T epsl;
    sym_givens<T>(epsbar, delta, &cc, &ss, &epsl);
    sigmax = std::max(sigmax, std::max(epsl, std::fabs(epsbar)));
    sigmin = std::min(sigmin, std::min(epsl, std::fabs(epsbar)));
    Acond = sigmax / sigmin;

    const T zetaold = zeta;
    zeta = (tau - zeta * eta) / epsl;
    zetabar = zeta / cc;

    const T ra = psi * cp - zetaold * eta, rb = psi * sp;
    rNorm = std::sqrt(ra * ra + rb * rb);
    if (history) stats.residuals.push_back(rNorm);
    const T aa = gamma * epsl * zeta, ab = delta * eta * zetaold;
    ArNorm = std::sqrt(aa * aa + ab * ab);
    if (history) stats.Aresiduals.push_back(ArNorm);
    psi = psi * sp;
    xcgNorm2 = xlqNorm2 + zetabar * zetabar;

    if (sigma > 0 && iter > 0 && !complex_error_bnd) {
      const T disc = zetatilde * zetatilde - zetabar * zetabar;
      if (disc < 0) {
        complex_error_bnd = true;
      } else {
        const T err_ubnd_cg = std::sqrt(disc);
        if (history) stats.err_ubnds_cg.push_back(err_ubnd_cg);
        fwd_err_ubnd = err_ubnd_cg <= utol * std::sqrt(xcgNorm2);
      }
    }

    const T test1 = rNorm;
    const T test2 = ArNorm / (Anorm * rNorm);
    const T test3 = T(1) / Acond;
    const T t1 = test1 / (T(1) + Anorm * xlqNorm);

    // update the LSLQ point and w̄
    if (s.fused) {
      lslq_fused_update<T>(ws, scale_v, T(1) / alpha, cc * zeta, ss * zeta, cc, ss);
    } else {
      k_axpy<T>(c, n, cc * zeta, ws.w, ws.x);
      k_axpy<T>(c, n, ss * zeta, v, ws.x);
      k_axpby<T>(c, n, -cc, v, ss, ws.w);
    }
    xlqNorm2 += zeta * zeta;
    xlqNorm = std::sqrt(xlqNorm2);

    err_vec[iter % window] = zeta;                              // iter: the count before this iteration
    if (iter >= window) {
      err_lbnd = err_window_norm(err_vec);
      if (history) stats.err_lbnds.push_back(err_lbnd);
      fwd_err_lbnd = err_lbnd <= etol * xlqNorm;
    }

    if (sigma > 0 && !complex_error_bnd) {                      // LQ forward-error upper bound
      const T etatilde = omega * ss;
      const T epstilde = -omega * cc;
      const T tautilde = -tau * delta / omega;
      zetatilde = (tautilde - zeta * etatilde) / epstilde;
      if (history) stats.err_ubnds_lq.push_back(std::fabs(zetatilde));
    }

    ill_cond_mach = (T(1) + test3 <= T(1));
    const bool solved_mach = (T(1) + test2 <= T(1));
    const bool zero_resid_mach = (T(1) + t1 <= T(1));
    run.poll(iter + 1, user_exit, overtimed);                    // callback, then the clock
    tired = iter >= itmax;
    ill_cond_lim = (test3 <= ctol);
    const bool solved_lim = (test2 <= atol);                    // atol, as lslq.jl has it
    const bool zero_resid_lim = (test1 <= eps);
    ill_cond = ill_cond_mach || ill_cond_lim;
    zero_resid = zero_resid_mach || zero_resid_lim;
    solved = solved_mach || solved_lim || zero_resid || fwd_err_lbnd || fwd_err_ubnd;
    iter = iter + 1;
    if (kdisplay(iter, o.verbose))
      printf("%5d  %7.1e  %7.1e  %7.1e  %7.1e  %8.1e  %8.1e  %7.1e  %7.1e  %7.1e  %.2fs\n", iter, (double)rNorm, (double)ArNorm,
             (double)beta, (double)alpha, (double)cc, (double)ss, (double)Anorm, (double)Acond, (double)xlqNorm, run.elapsed());
  }
  if (o.verbose > 0) printf("\n");
  if (o.transfer_to_lsqr) k_axpy<T>(c, n, zetabar, ws.w, ws.x);   // the LSQR point

  const char* st = "unknown";
  if (tired) st = "maximum number of iterations exceeded";
  if (ill_cond_mach) st = "condition number seems too large for this machine";
  if (ill_cond_lim) st = "condition number exceeds tolerance";
  if (solved) st = "found approximate minimum least-squares solution";
  if (zero_resid) st = "found approximate zero-residual solution";
  if (fwd_err_lbnd) st = "forward error lower bound small enough";
  if (fwd_err_ubnd) st = "forward error upper bound small enough";
  if (user_exit) st = "user-requested exit";
  if (overtimed) st = "time limit exceeded";
  stats.error_with_bnd = complex_error_bnd;
  run.finish(iter, solved, !zero_resid, st);
}

// ===========================================================================
// cgls!  (src/cgls.jl:129-243).  M acts on the m-dimensional residual space; Mq aliases the Mr buffer when M != I.
// ===========================================================================
template <class T>
void cgls_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& M, const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int m = ws.m, n = ws.n;
  const bool history = o.history, ldiv = o.ldiv;
  if (o.verbose > 0) printf("CGLS: system of %d equations in %d variables\n", m, n);
  const bool MisI = M.is_identity();
  const T lambda = (T)o.lambda, radius = (T)o.radius;
  const T atol = tol_of<T>(o.atol), rtol = tol_of<T>(o.rtol);
  const bool fused = o.fused && A.kind == LinOp<T>::CSR && At.kind == LinOp<T>::CSR && MisI && !(radius > 0);
  Stats& stats = ws.stats;
  allocate_if(!MisI, ws, ws.Mr, m);
  stats.reset();
  T* Mr = MisI ? ws.r : ws.Mr;
  T* Mq = MisI ? ws.q : ws.Mr;

  k_fill<T>(c, n, ws.x, T(0));
  k_copy<T>(c, m, ws.r, b);
  const T bNorm = k_nrm2<T>(c, m, ws.r);
  if (bNorm == 0) {
    run.finish(0, true, false, "x is a zero-residual solution");
    if (history) { stats.residuals.push_back(0); stats.Aresiduals.push_back(0); }
    return;
  }
  if (!MisI) op_apply(c, M, ws.r, Mr, ldiv);
  op_apply(c, At, Mr, ws.s);
  k_copy<T>(c, n, ws.p, ws.s);
  T gamma = k_dot<T>(c, n, ws.s, ws.s);
  int iter = 0;
  const int itmax = ls_itmax(ws, o.itmax);

  T rNorm = bNorm, ArNorm = std::sqrt(gamma);
  if (history) { stats.residuals.push_back(rNorm); stats.Aresiduals.push_back(ArNorm); }
  const T eps = atol + rtol * ArNorm;
  if (o.verbose > 0) printf("%5s  %8s  %8s  %5s\n", "k", "‖Aᴴr‖", "‖r‖", "timer");
  if (kdisplay(iter, o.verbose)) printf("%5d  %8.2e  %8.2e  %.2fs\n", iter, (double)ArNorm, (double)rNorm, run.elapsed());

  bool on_boundary = false, solved = ArNorm <= eps, tired = iter >= itmax, user_exit = false, overtimed = false;
  while (!(solved || tired || user_exit || overtimed)) {
    if (fused) {
      T rr;
      cgls_fused_iteration<T>(ws, *A.csr, *At.csr, iter == 0, gamma, lambda, &rr, &gamma);
      rNorm = std::sqrt(rr);
    } else {
      op_apply(c, A, ws.p, ws.q);
      if (!MisI) op_apply(c, M, ws.q, Mq, ldiv);
      T delta = k_dot<T>(c, m, ws.q, Mq);                       // δ = qᴴMq
      if (lambda > 0) delta += lambda * k_dot<T>(c, n, ws.p, ws.p);
      T alpha = gamma / delta;
      if (radius > 0) {                                         // step to the boundary (in the Euclidean norm)
        T t1, t2;
        boundary_roots<T>(c, n, ws.x, ws.p, radius, T(0), &t1, &t2);
        const T sigma = std::max(t1, t2);
        if (alpha > sigma) { alpha = sigma; on_boundary = true; }
      }
      k_axpy<T>(c, n, alpha, ws.p, ws.x);
      k_axpy<T>(c, m, -alpha, ws.q, ws.r);
      if (!MisI) op_apply(c, M, ws.r, Mr, ldiv);
      op_apply(c, At, Mr, ws.s);
      if (lambda > 0) k_axpy<T>(c, n, -lambda, ws.x, ws.s);    // s = Aᴴr - λx, with the updated x
      const T gamma_next = k_dot<T>(c, n, ws.s, ws.s);
      const T beta = gamma_next / gamma;
      k_axpby<T>(c, n, T(1), ws.s, beta, ws.p);
      gamma = gamma_next;
      rNorm = k_nrm2<T>(c, m, ws.r);
    }
    ArNorm = std::sqrt(gamma);
    if (history) { stats.residuals.push_back(rNorm); stats.Aresiduals.push_back(ArNorm); }
    iter = iter + 1;
    if (kdisplay(iter, o.verbose)) printf("%5d  %8.2e  %8.2e  %.2fs\n", iter, (double)ArNorm, (double)rNorm, run.elapsed());
    run.poll(iter, user_exit, overtimed);
    solved = (ArNorm <= eps) || on_boundary;
    tired = iter >= itmax;
  }
  if (o.verbose > 0) printf("\n");
  const char* st = "unknown";
  if (tired) st = "maximum number of iterations exceeded";
  if (solved) st = "solution good enough given atol and rtol";
  if (on_boundary) st = "on trust-region boundary";
  if (user_exit) st = "user-requested exit";
  if (overtimed) st = "time limit exceeded";
  run.finish(iter, solved, false, st);
}

// ===========================================================================
// crls!  (src/crls.jl:120-268).  M acts on the m-dimensional residual space: Ms, Mr and MAp share one buffer.
// ===========================================================================
template <class T>
void crls_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& M, const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int m = ws.m, n = ws.n;
  const bool history = o.history, ldiv = o.ldiv;
  if (o.verbose > 0) printf("CRLS: system of %d equations in %d variables\n", m, n);
  const bool MisI = M.is_identity();
  const T lambda = (T)o.lambda, radius = (T)o.radius;
  const T atol = tol_of<T>(o.atol), rtol = tol_of<T>(o.rtol);
  const bool fused = o.fused && A.kind == LinOp<T>::CSR && At.kind == LinOp<T>::CSR && MisI && !(radius > 0);
  Stats& stats = ws.stats;
  allocate_if(!MisI, ws, ws.Mr, m);
  stats.reset();
  T* Ms = MisI ? ws.s : ws.Mr;
  T* Mr = MisI ? ws.r : ws.Mr;
  T* MAp = MisI ? ws.Ap : ws.Mr;

  k_fill<T>(c, n, ws.x, T(0));
  k_copy<T>(c, m, ws.r, b);
  const T bNorm = k_nrm2<T>(c, m, ws.r);
  T rNorm = bNorm;
  if (history) stats.residuals.push_back(rNorm);
  if (bNorm == 0) {
    run.finish(0, true, false, "x is a zero-residual solution");
    if (history) stats.Aresiduals.push_back(0);
    return;
  }
  if (!MisI) op_apply(c, M, ws.r, Mr, ldiv);
  op_apply(c, At, Mr, ws.Ar);
  op_apply(c, A, ws.Ar, ws.s);
  if (!MisI) op_apply(c, M, ws.s, Ms, ldiv);
  k_copy<T>(c, n, ws.p, ws.Ar);
  k_copy<T>(c, m, ws.Ap, ws.s);
  op_apply(c, At, Ms, ws.q);
  if (lambda > 0) k_axpy<T>(c, n, lambda, ws.p, ws.q);        // q = q + λ p
  T gamma = k_dot<T>(c, m, ws.s, Ms);
  int iter = 0;
  const int itmax = ls_itmax(ws, o.itmax);

  T ArNorm = k_nrm2<T>(c, n, ws.Ar);
  if (lambda > 0) gamma += lambda * ArNorm * ArNorm;
  if (history) stats.Aresiduals.push_back(ArNorm);
  const T eps = atol + rtol * ArNorm;
  if (o.verbose > 0) printf("%5s  %8s  %8s  %5s\n", "k", "‖Aᴴr‖", "‖r‖", "timer");
  if (kdisplay(iter, o.verbose)) printf("%5d  %8.2e  %8.2e  %.2fs\n", iter, (double)ArNorm, (double)rNorm, run.elapsed());

  bool on_boundary = false, solved = ArNorm <= eps, tired = iter >= itmax, psd = false, user_exit = false, overtimed = false;
  T* p = ws.p;                                                  // rebound to Ar by the zero-curvature branch
  while (!(solved || tired || user_exit || overtimed)) {
    if (fused) {
      T ArAr, xx, rr;
      const T alpha0 = iter == 0 ? gamma / k_dot<T>(c, n, ws.q, ws.q) : T(0);   // later alphas stay on the device
      crls_fused_iteration<T>(ws, *A.csr, *At.csr, iter == 0, alpha0, gamma, lambda, &ArAr, &xx, &rr, &gamma);
      ArNorm = std::sqrt(ArAr);
      rNorm = lambda > 0 ? std::sqrt(rr + lambda * xx) : std::sqrt(rr);
    } else {
      const T qNorm2 = k_dot<T>(c, n, ws.q, ws.q);
      T alpha = gamma / qNorm2;
      if (radius > 0) {                                         // α > 0 in CRLS
        const T pNorm = k_nrm2<T>(c, n, p);
        T t1, t2;
        if (k_dot<T>(c, m, ws.Ap, ws.Ap) <= eps * std::sqrt(qNorm2) * pNorm) {   // the quadratic is constant along p
          psd = true;
          p = ws.Ar;                                            // p = Aᴴr
          const T pNorm2 = ArNorm * ArNorm;
          op_apply(c, At, ws.s, ws.q);
          boundary_roots<T>(c, n, ws.x, p, radius, pNorm2, &t1, &t2);
          alpha = std::min(ArNorm * ArNorm / gamma, std::max(t1, t2));
        } else {
          const T pNorm2 = pNorm * pNorm;
          boundary_roots<T>(c, n, ws.x, p, radius, pNorm2, &t1, &t2);
          const T sigma = std::max(t1, t2);
          if (alpha >= sigma) { alpha = sigma; on_boundary = true; }
        }
      }
      k_axpy<T>(c, n, alpha, p, ws.x);
      k_axpy<T>(c, n, -alpha, ws.q, ws.Ar);
      ArNorm = k_nrm2<T>(c, n, ws.Ar);
      solved = psd || on_boundary;
      if (solved) continue;                                     // leaves the loop: no iteration count, history or callback
      k_axpy<T>(c, m, -alpha, ws.Ap, ws.r);
      op_apply(c, A, ws.Ar, ws.s);
      if (!MisI) op_apply(c, M, ws.s, Ms, ldiv);
      T gamma_next = k_dot<T>(c, m, ws.s, Ms);
      if (lambda > 0) gamma_next += lambda * ArNorm * ArNorm;
      const T beta = gamma_next / gamma;
      k_axpby<T>(c, n, T(1), ws.Ar, beta, p);
      k_axpby<T>(c, m, T(1), ws.s, beta, ws.Ap);
      if (!MisI) op_apply(c, M, ws.Ap, MAp, ldiv);
      op_apply(c, At, MAp, ws.q);
      if (lambda > 0) k_axpy<T>(c, n, lambda, p, ws.q);
      gamma = gamma_next;
      rNorm = lambda > 0 ? std::sqrt(k_dot<T>(c, m, ws.r, ws.r) + lambda * k_dot<T>(c, n, ws.x, ws.x)) : k_nrm2<T>(c, m, ws.r);
    }
    if (history) { stats.residuals.push_back(rNorm); stats.Aresiduals.push_back(ArNorm); }
    iter = iter + 1;
    if (kdisplay(iter, o.verbose)) printf("%5d  %8.2e  %8.2e  %.2fs\n", iter, (double)ArNorm, (double)rNorm, run.elapsed());
    run.poll(iter, user_exit, overtimed);
    solved = (ArNorm <= eps) || on_boundary;
    tired = iter >= itmax;
  }
  if (o.verbose > 0) printf("\n");
  const char* st = "unknown";
  if (tired) st = "maximum number of iterations exceeded";
  if (solved) st = "solution good enough given atol and rtol";
  if (psd) st = "zero-curvature encountered";
  if (on_boundary) st = "on trust-region boundary";
  if (user_exit) st = "user-requested exit";
  if (overtimed) st = "time limit exceeded";
  run.finish(iter, solved, false, st);
}

// ===========================================================================
// craig!  (src/craig.jl:174-405): CG on A Aᴴ y = b, x = Aᴴ y.  The Golub-Kahan products run in the opposite order from
// LSQR's: Aᴴu first, then A v.  Fused (λ = 0, M = N = I, CSR A and Aᴴ): C1 on Aᴴ, then C2 on A, one read-back each;
// x += ξ v rides in the next C1 and is flushed before a callback and after the last iteration.
// ===========================================================================
template <class T>
void craig_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& M, const LinOp<T>& N,
                 const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int m = ws.m, n = ws.n;
  const bool history = o.history, ldiv = o.ldiv;
  if (o.verbose > 0) printf("CRAIG: system of %d equations in %d variables\n", m, n);
  const T lambda = (T)o.lambda;
  const T conlim = o.conlim < 0 ? T(1) / std::sqrt(eps_of<T>()) : (T)o.conlim;
  const T btol = tol_of<T>(o.btol), atol = tol_of<T>(o.atol), rtol = tol_of<T>(o.rtol);
  Stats& stats = ws.stats;

  T beta1;
  Setup s = lsq_prologue<T>(ws, A, At, b, M, N, o, &beta1);
  s.fused = s.fused && lambda == 0;                             // the fused passes carry no regularization
  allocate_if(!s.fused, ws, ws.Av, m);
  allocate_if(!s.fused, ws, ws.Atu);
  allocate_if(lambda > 0, ws, ws.w2);
  T* u = s.MisI ? ws.Mu : ws.u;
  T* v = s.NisI ? ws.Nv : ws.v;
  k_fill<T>(c, m, ws.y, T(0));
  T rNorm = beta1;
  if (history) stats.residuals.push_back(rNorm);
  if (beta1 == 0) {
    run.finish(0, true, false, "x is a zero-residual solution");
    return;
  }
  const T beta1_2 = beta1 * beta1;
  T beta = beta1, theta = beta1, xi = T(-1), delta = lambda, rho_prev = T(1);

  k_scal<T>(c, m, T(1) / beta1, u);                            // β₁Mu₁ = b
  if (!s.MisI) k_scal<T>(c, m, T(1) / beta1, ws.Mu);
  k_fill<T>(c, n, ws.Nv, T(0));
  k_fill<T>(c, m, ws.w, T(0));
  if (lambda > 0) k_fill<T>(c, n, ws.w2, T(0));

  T Anorm2 = 0, Anorm = 0, Dnorm2 = 0, Acond = 0, xNorm2 = 0, xNorm = 0;
  int iter = 0;
  const int itmax = ls_itmax(ws, o.itmax);
  const T eps_c = atol + rtol * rNorm;
  const T ctol = conlim > 0 ? T(1) / conlim : T(0);
  if (o.verbose > 0) printf("%5s  %8s  %8s  %8s  %8s  %8s  %7s  %5s\n", "k", "‖r‖", "‖x‖", "‖A‖", "κ(A)", "α", "β", "timer");
  if (kdisplay(iter, o.verbose))
    printf("%5d  %8.2e  %8.2e  %8.2e  %8.2e  %8s  %7s  %.2fs\n", iter, (double)rNorm, (double)xNorm, (double)Anorm, (double)Acond,
           " ✗ ✗ ✗ ✗", "✗ ✗ ✗ ✗", run.elapsed());

  T bkwerr = 1;
  bool solved_lim = bkwerr <= btol, solved_mach = T(1) + bkwerr <= T(1), solved_resid_tol = rNorm <= eps_c;
  bool solved_resid_lim = rNorm <= btol + atol * Anorm * xNorm / beta1;
  bool solved = solved_mach || solved_lim || solved_resid_tol || solved_resid_lim;
  bool ill_cond = false, ill_cond_mach = false, ill_cond_lim = false, inconsistent = false;
  bool tired = iter >= itmax, user_exit = false, overtimed = false;
  // fused: the x update of the last completed iteration waits for the next C1 (factor s_v = 1/α of that iteration)
  // fused: s_u = 1/β and s_v = 1/α of the stored Mu and Nv (1 while they hold u₁ and v₀ = 0)
  bool xpend = false;
  T xi_pend = 0, s_u = 1, s_v = 1;

  while (!(solved || inconsistent || ill_cond || tired || user_exit || overtimed)) {
    // 1. αₖ₊₁Nvₖ₊₁ = Aᴴuₖ₊₁ - βₖ₊₁Nvₖ
    T alpha;
    if (s.fused) {
      alpha = craig_fused_p1<T>(ws, *At.csr, iter == 0 && !xpend, beta, s_v, xpend, xi_pend);
      xpend = false;
    } else {
      op_apply(c, At, u, ws.Atu);
      k_axpby<T>(c, n, T(1), ws.Atu, -beta, ws.Nv);
      if (!s.NisI) op_apply(c, N, ws.Nv, v, ldiv);
      alpha = knorm_elliptic<T>(c, n, v, ws.Nv);
    }
    if (alpha == 0) {
      inconsistent = true;
      continue;
    }
    if (s.fused) {
      s_v = T(1) / alpha;                                       // kdiv!(n, v, α), applied by v's readers
    } else {
      k_scal<T>(c, n, T(1) / alpha, v);
      if (!s.NisI) k_scal<T>(c, n, T(1) / alpha, ws.Nv);
    }

    Anorm2 += alpha * alpha + lambda * lambda;
    T c1 = 1, s1 = 0, rho;
    if (lambda > 0) sym_givens<T>(alpha, delta, &c1, &s1, &rho);
    else rho = alpha;
    xi = -theta / rho * xi;

    if (lambda > 0) {
      // w1 = c₁ v + s₁ w2 ; w2 = s₁ v - c₁ w2 ; x = x + ξ w1
      k_axpy<T>(c, n, xi * c1, v, ws.x);
      k_axpy<T>(c, n, xi * s1, ws.w2, ws.x);
      k_axpby<T>(c, n, s1, v, -c1, ws.w2);
    } else if (s.fused) {
      xpend = true; xi_pend = xi;
    } else {
      k_axpy<T>(c, n, xi, v, ws.x);
    }

    // Recur y, then 2. βₖ₊₁Muₖ₊₁ = Avₖ - αₖMuₖ
    if (s.fused) {
      T ww;
      craig_fused_p2<T>(ws, *A.csr, s_u, alpha, -theta / rho_prev, xi / rho, &beta, &ww);
      s_u = beta == 0 ? T(1) : T(1) / beta;                     // kdiv!(m, u, β), applied by u's readers
      Dnorm2 += std::sqrt(ww);
    } else {
      k_axpby<T>(c, m, T(1), u, -theta / rho_prev, ws.w);      // w = u - θ/ρ_prev * w
      k_axpy<T>(c, m, xi / rho, ws.w, ws.y);                    // y = y + ξ/ρ * w
      Dnorm2 += k_nrm2<T>(c, m, ws.w);                          // knorm(m, w): a norm, as the reference has it
      op_apply(c, A, v, ws.Av);
      k_axpby<T>(c, m, T(1), ws.Av, -alpha, ws.Mu);
      if (!s.MisI) op_apply(c, M, ws.Mu, u, ldiv);
      beta = knorm_elliptic<T>(c, m, u, ws.Mu);
      if (beta != 0) {
        k_scal<T>(c, m, T(1) / beta, u);
        if (!s.MisI) k_scal<T>(c, m, T(1) / beta, ws.Mu);
      }
    }

    // Finish the updates from the first Givens rotation.
    T gamma = 0;
    if (lambda > 0) {
      theta = beta * c1;
      gamma = beta * s1;
      T c2, s2;
      sym_givens<T>(lambda, gamma, &c2, &s2, &delta);
      k_scal<T>(c, n, s2, ws.w2);
    } else {
      theta = beta;
    }

    Anorm2 += beta * beta;
    Anorm = std::sqrt(Anorm2);
    Acond = Anorm * std::sqrt(Dnorm2);
    xNorm2 += xi * xi;
    xNorm = std::sqrt(xNorm2);
    rNorm = beta * std::fabs(xi);                               // r = - β ξ u
    if (lambda > 0) rNorm *= std::fabs(c1);                     // r = - c₁ β ξ u when λ > 0
    if (history) stats.residuals.push_back(rNorm);
    iter = iter + 1;
    bkwerr = rNorm / std::sqrt(beta1_2 + Anorm2 * xNorm2);
    rho_prev = rho;
    if (kdisplay(iter, o.verbose))
      printf("%5d  %8.2e  %8.2e  %8.2e  %8.2e  %8.1e  %7.1e  %.2fs\n", iter, (double)rNorm, (double)xNorm, (double)Anorm,
             (double)Acond, (double)alpha, (double)beta, run.elapsed());

    solved_lim = bkwerr <= btol;
    solved_mach = T(1) + bkwerr <= T(1);
    solved_resid_tol = rNorm <= eps_c;
    solved_resid_lim = rNorm <= btol + atol * Anorm * xNorm / beta1;
    solved = solved_mach || solved_lim || solved_resid_tol || solved_resid_lim;
    ill_cond_mach = T(1) + T(1) / Acond <= T(1);
    ill_cond_lim = T(1) / Acond <= ctol;
    ill_cond = ill_cond_mach || ill_cond_lim;
    if (xpend && o.callback) {                                  // the callback reads x
      craig_fused_flush<T>(ws, xi_pend, s_v);
      xpend = false;
    }
    run.poll(iter, user_exit, overtimed);
    inconsistent = false;
    tired = iter >= itmax;
  }
  if (xpend) craig_fused_flush<T>(ws, xi_pend, s_v);
  if (o.verbose > 0) printf("\n");

  if (lambda > 0 && o.transfer_to_lsqr) {                       // the LSQR point
    xi *= -theta / delta;
    k_axpy<T>(c, n, xi, ws.w2, ws.x);
  }

  const char* st = "unknown";
  if (tired) st = "maximum number of iterations exceeded";
  if (solved) st = "solution good enough for the tolerances given";
  if (ill_cond_mach) st = "condition number seems too large for this machine";
  if (ill_cond_lim) st = "condition number exceeds tolerance";
  if (inconsistent) st = "system may be inconsistent";
  if (user_exit) st = "user-requested exit";
  if (overtimed) st = "time limit exceeded";
  run.finish(iter, solved, inconsistent, st);
}

// ===========================================================================
// craigmr!  (src/craigmr.jl:161-396): MINRES on A Aᴴ y = b, x = Aᴴ y.  Fused (λ = 0, M = N = I, CSR A and Aᴴ): R1 on A,
// read β, the Givens step on the host, then R2 on Aᴴ and R3 over m, read α: 3 launches and 2 read-backs.
// ===========================================================================
template <class T>
void craigmr_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& M, const LinOp<T>& N,
                   const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int m = ws.m, n = ws.n;
  const bool history = o.history, ldiv = o.ldiv;
  if (o.verbose > 0) printf("CRAIGMR: system of %d equations in %d variables\n", m, n);
  const T lambda = (T)o.lambda;
  const T atol = tol_of<T>(o.atol), rtol = tol_of<T>(o.rtol);
  Stats& stats = ws.stats;

  T beta;
  Setup s = lsq_prologue<T>(ws, A, At, b, M, N, o, &beta);
  s.fused = s.fused && lambda == 0;                             // the fused passes carry no regularization
  allocate_if(!s.fused, ws, ws.Av, m);
  allocate_if(!s.fused, ws, ws.Atu);
  allocate_if(lambda > 0, ws, ws.q);
  T* u = s.MisI ? ws.Mu : ws.u;
  T* v = s.NisI ? ws.Nv : ws.v;
  k_fill<T>(c, m, ws.y, T(0));
  if (beta == 0) {
    run.finish(0, true, false, "x is a zero-residual solution");
    if (history) { stats.residuals.push_back(beta); stats.Aresiduals.push_back(0); }
    return;
  }
  lsq_start<T>(ws, s, At, N, ldiv, beta);                       // u /= β₁, Nv = Aᴴu, v = N Nv
  T alpha = knorm_elliptic<T>(c, n, v, ws.Nv);
  T Anorm2 = alpha * alpha;
  int iter = 0;
  const int itmax = ls_itmax(ws, o.itmax);
  if (o.verbose > 0) printf("%5s  %7s  %7s  %7s  %7s  %8s  %8s  %7s  %5s\n", "k", "‖r‖", "‖Aᴴr‖", "β", "α", "cos", "sin", "‖A‖²", "timer");
  if (kdisplay(iter, o.verbose))
    printf("%5d  %7.1e  %7.1e  %7.1e  %7.1e  %8.1e  %8.1e  %7.1e  %.2fs\n", iter, (double)beta, (double)alpha, (double)beta,
           (double)alpha, 0.0, 1.0, (double)Anorm2, run.elapsed());
  if (alpha == 0) {                                             // Aᴴb = 0: x = 0 is a minimum least-squares solution
    run.finish(0, true, false, "x is a minimum least-squares solution");
    if (history) { stats.residuals.push_back(beta); stats.Aresiduals.push_back(0); }
    return;
  }
  k_scal<T>(c, n, T(1) / alpha, v);
  if (!s.NisI) k_scal<T>(c, n, T(1) / alpha, ws.Nv);

  // Regularization
  const T lambdak = lambda;                                     // λ₁ = λ
  T cpk = 1, spk = 1, cdk = 1, sdk = 1, alphahat;
  if (lambda > 0) k_copy<T>(c, n, ws.q, v);                     // q₀ = 0 by definition
  if (lambda > 0) {
    sym_givens<T>(alpha, lambdak, &cpk, &spk, &alphahat);
    k_scal<T>(c, n, spk, ws.q);                                 // q̄₁ = sp₁ v₁
  } else {
    alphahat = alpha;
  }
  (void)cdk;

  T zetabar = beta, rhobar = alphahat, theta = 0;
  T rNorm = zetabar;
  if (history) stats.residuals.push_back(rNorm);
  T ArNorm = alpha;
  if (history) stats.Aresiduals.push_back(ArNorm);
  const T eps_c = atol + rtol * rNorm;
  const T eps_i = atol + rtol * ArNorm;
  k_divcopy<T>(c, m, ws.w1, u, alphahat);                       // w̄ = u / α̂
  k_fill<T>(c, m, ws.w, T(0));
  k_fill<T>(c, n, ws.d1, T(0));

  bool solved = rNorm <= eps_c;
  bool inconsistent = (rNorm > 100 * eps_c) && (ArNorm <= eps_i);
  bool tired = iter >= itmax, user_exit = false, overtimed = false;
  T s_u = 1, s_v = 1;                                           // fused: 1/β and 1/α of the stored Mu and Nv (u₁, v₁ are scaled)

  while (!(solved || inconsistent || tired || user_exit || overtimed)) {
    iter = iter + 1;
    // 1. βₖ₊₁Muₖ₊₁ = Avₖ - αₖMuₖ
    if (s.fused) {
      beta = craigmr_fused_p1<T>(ws, *A.csr, iter == 1, s_u, alpha);
    } else {
      op_apply(c, A, v, ws.Av);
      k_axpby<T>(c, m, T(1), ws.Av, -alpha, ws.Mu);
      if (!s.MisI) op_apply(c, M, ws.Mu, u, ldiv);
      beta = knorm_elliptic<T>(c, m, u, ws.Mu);
      if (beta != 0) {
        k_scal<T>(c, m, T(1) / beta, u);
        if (!s.MisI) k_scal<T>(c, m, T(1) / beta, ws.Mu);
      }
    }
    Anorm2 = Anorm2 + beta * beta;                              // = ‖B_{k-1}‖²

    T betahat, lambda_aux = 0;
    if (lambda > 0) {
      betahat = cpk * beta;
      lambda_aux = spk * beta;
    } else {
      betahat = beta;
    }

    // Continue QR factorization
    T cs, sn, rho;
    sym_givens<T>(rhobar, betahat, &cs, &sn, &rho);
    const T zeta = cs * zetabar;
    zetabar = sn * zetabar;
    rNorm = std::fabs(zetabar);
    if (history) stats.residuals.push_back(rNorm);

    if (s.fused) {
      s_u = beta == 0 ? T(1) : T(1) / beta;
      alpha = craigmr_fused_p23<T>(ws, *At.csr, iter == 1, s_u, s_v, beta, rho, T(1) / rho, -theta / rho, zeta);
      s_v = alpha == 0 ? T(1) : T(1) / alpha;
    } else {
      k_axpby<T>(c, m, T(1) / rho, ws.w1, -theta / rho, ws.w); // w = (w̄ - θ w) / ρ
      k_axpy<T>(c, m, zeta, ws.w, ws.y);                        // y = y + ζ w
      if (lambda > 0) {                                         // DₖRₖ = V̅ₖ with v̅ₖ = cpₖvₖ + spₖqₖ₋₁
        if (iter == 1) {
          k_axpy<T>(c, n, cpk / rho, v, ws.d1);
        } else {
          k_axpby<T>(c, n, cpk / rho, v, -theta / rho, ws.d1);
          k_axpy<T>(c, n, spk / rho, ws.q, ws.d1);
          k_axpby<T>(c, n, spk, v, -cpk, ws.q);                 // q̄ₖ ← spₖ vₖ - cpₖ qₖ₋₁
        }
      } else {                                                  // DₖRₖ = Vₖ
        if (iter == 1) k_divcopy<T>(c, n, ws.d1, v, rho);
        else k_axpby<T>(c, n, T(1) / rho, v, -theta / rho, ws.d1);
      }
      k_axpy<T>(c, n, zeta, ws.d1, ws.x);                       // xₖ = Dₖzₖ
      // 2. αₖ₊₁Nvₖ₊₁ = Aᴴuₖ₊₁ - βₖ₊₁Nvₖ
      op_apply(c, At, u, ws.Atu);
      k_axpby<T>(c, n, T(1), ws.Atu, -beta, ws.Nv);
      if (!s.NisI) op_apply(c, N, ws.Nv, v, ldiv);
      alpha = knorm_elliptic<T>(c, n, v, ws.Nv);
    }
    Anorm2 = Anorm2 + alpha * alpha;                            // = ‖Lₖ‖
    ArNorm = alpha * beta * std::fabs(zeta / rho);
    if (history) stats.Aresiduals.push_back(ArNorm);
    if (kdisplay(iter, o.verbose))
      printf("%5d  %7.1e  %7.1e  %7.1e  %7.1e  %8.1e  %8.1e  %7.1e  %.2fs\n", iter, (double)rNorm, (double)ArNorm, (double)beta,
             (double)alpha, (double)cs, (double)sn, (double)Anorm2, run.elapsed());

    if (lambda > 0) {
      T lambdak1;
      sym_givens<T>(lambda, lambda_aux, &cdk, &sdk, &lambdak1);
      k_scal<T>(c, n, sdk, ws.q);                               // qₖ ← sdₖ q̄ₖ
      sym_givens<T>(alpha, lambdak1, &cpk, &spk, &alphahat);
    } else {
      alphahat = alpha;
    }
    if (alpha != 0 && !s.fused) {                               // fused: R3 updated w̄ and v's readers apply 1/α
      k_scal<T>(c, n, T(1) / alpha, v);
      if (!s.NisI) k_scal<T>(c, n, T(1) / alpha, ws.Nv);
      k_axpby<T>(c, m, T(1) / alphahat, u, -betahat / alphahat, ws.w1);   // w̄ = (u - β̂ w̄) / α̂
    }
    theta = sn * alphahat;
    rhobar = -cs * alphahat;

    run.poll(iter, user_exit, overtimed);
    solved = rNorm <= eps_c;
    inconsistent = (rNorm > 100 * eps_c) && (ArNorm <= eps_i);
    tired = iter >= itmax;
  }
  if (o.verbose > 0) printf("\n");

  const char* st = "unknown";
  if (tired) st = "maximum number of iterations exceeded";
  if (solved) st = "found approximate minimum-norm solution";
  if (!tired && !solved) st = "found approximate minimum least-squares solution";
  if (user_exit) st = "user-requested exit";
  if (overtimed) st = "time limit exceeded";
  run.finish(iter, solved, inconsistent, st);
}

// ===========================================================================
// lnlq!  (src/lnlq.jl:168-568): SYMMLQ on A Aᴴ y = b, x = Aᴴ y.  `iter` is incremented once before the loop and once
// at the end of each pass, so niter = passes + 1.  σ-based upper bounds on ‖x - x*‖ (stats.err_lbnds) and ‖y - y*‖
// (stats.err_ubnds_lq) when √(σ² + λ²) > 0.  Fused (λ = 0, M = N = I, CSR A and Aᴴ): L1 on A, read β, then L2 on Aᴴ,
// read α; the y / w̄ update of a pass rides in the next L1 and is flushed before a callback and after the last pass.
// ===========================================================================
template <class T>
void lnlq_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& M, const LinOp<T>& N,
                const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int m = ws.m, n = ws.n;
  const bool history = o.history, ldiv = o.ldiv, transfer_to_craig = o.transfer_to_bicg;
  if (o.verbose > 0) printf("LNLQ: system of %d equations in %d variables\n", m, n);
  const T lambda = (T)o.lambda, sigma = (T)o.sigma;
  const T utolx = tol_of<T>(o.utol), utoly = tol_of<T>(o.etol), atol = tol_of<T>(o.atol), rtol = tol_of<T>(o.rtol);
  const T eps = eps_of<T>();
  Stats& stats = ws.stats;
  std::vector<double>& xNorms = stats.err_lbnds;                // error_bnd_x
  std::vector<double>& yNorms = stats.err_ubnds_lq;             // error_bnd_y

  T beta;
  Setup s = lsq_prologue<T>(ws, A, At, b, M, N, o, &beta);      // x = 0, Mu = b, u = M⁻¹Mu, β₁ = ‖u‖_M
  s.fused = s.fused && lambda == 0;                             // the fused passes carry no regularization
  allocate_if(!s.fused, ws, ws.Av, m);
  allocate_if(!s.fused, ws, ws.Atu);
  allocate_if(lambda > 0, ws, ws.q);
  T* u = s.MisI ? ws.Mu : ws.u;
  T* v = s.NisI ? ws.Nv : ws.v;
  T* wbar = ws.w;
  const T sigma_est = std::sqrt(sigma * sigma + lambda * lambda);
  bool complex_error_bnd = false;
  k_fill<T>(c, m, ws.y, T(0));

  const T bNorm = s.MisI ? beta : (m > 0 ? k_nrm2<T>(c, m, b) : T(0));   // M = I: β₁ is knorm(m, b)
  if (bNorm == 0) {
    run.finish(0, true, false, "x is a zero-residual solution");
    stats.error_with_bnd = false;
    if (history) stats.residuals.push_back(bNorm);
    return;
  }
  if (history) stats.residuals.push_back(bNorm);
  const T eps_c = atol + rtol * bNorm;
  int iter = 0;
  const int itmax = ls_itmax(ws, o.itmax);
  if (o.verbose > 0) printf("%5s  %7s  %5s\n", "k", "‖rₖ‖", "timer");
  if (kdisplay(iter, o.verbose)) printf("%5d  %7.1e  %.2fs\n", iter, (double)bNorm, run.elapsed());
  iter = iter + 1;

  // β₁Mu₁ = b ; α₁Nv₁ = Aᴴu₁
  if (beta != 0) {
    k_scal<T>(c, m, T(1) / beta, u);
    if (!s.MisI) k_scal<T>(c, m, T(1) / beta, ws.Mu);
  }
  if (s.fused) {
    op_apply(c, At, u, ws.Nv);                                  // kmul!(Aᴴu, Aᴴ, u) ; kcopy!(n, Nv, Aᴴu) without the copy
  } else {
    op_apply(c, At, u, ws.Atu);
    k_copy<T>(c, n, ws.Nv, ws.Atu);
  }
  if (!s.NisI) op_apply(c, N, ws.Nv, v, ldiv);
  T alpha = knorm_elliptic<T>(c, n, v, ws.Nv);
  if (alpha != 0) {
    k_scal<T>(c, n, T(1) / alpha, v);
    if (!s.NisI) k_scal<T>(c, n, T(1) / alpha, ws.Nv);
  }
  k_copy<T>(c, m, wbar, u);                                     // w̄₁ = u₁

  T sk = 0, zeta_km1 = 0, etak = 0;
  T cpk = 1, spk = 1;                                           // Givens rotation that zeroes out λₖ
  if (lambda > 0) k_copy<T>(c, n, ws.q, v);                     // q₀ = 0 by definition
  T alphahat;
  if (lambda > 0) {
    sym_givens<T>(alpha, lambda, &cpk, &spk, &alphahat);
    k_scal<T>(c, n, spk, ws.q);                                 // q̄₁ = sp₁ v₁
  } else {
    alphahat = alpha;
  }
  T epsbar = alphahat;
  T tau = beta / alphahat;                                      // τ₁ = β₁ / α̂₁
  T zetabar = tau / epsbar;
  T thetak = tau;

  bool solved_lq = false, solved_cg = false, tired = false, user_exit = false, overtimed = false;
  T err_x = 0, err_y = 0, tautilde = 0, rhobar = 0, csig = 0;
  if (sigma_est > 0) {
    tautilde = beta / sigma_est;
    const T zetatilde = tautilde / sigma_est;
    err_x = tautilde;
    err_y = zetatilde;
    solved_lq = err_x <= utolx || err_y <= utoly;
    if (history) { xNorms.push_back(err_x); yNorms.push_back(err_y); }
    rhobar = -sigma_est;
    csig = -1;
  }
  // fused: s_u = 1/β and s_v = 1/α of the stored Mu and Nv (1 while they hold u₁ and v₁, scaled above); the y / w̄
  // update of the last pass waits for the next L1 with its coefficients ζc, ζs, -c, s
  T s_u = 1, s_v = 1;
  bool ypend = false;
  T yc = 0, ys = 0, wc = 0, wsn = 0;

  while (!(solved_lq || solved_cg || tired || user_exit || overtimed)) {
    // (xᵃᵘˣ)ₖ ← (xᵃᵘˣ)ₖ₋₁ + τₖ v̄ₖ  (fused: in L2, before Nv is overwritten)
    if (lambda > 0) {
      k_axpy<T>(c, n, tau * cpk, v, ws.x);
      if (iter >= 2) {
        k_axpy<T>(c, n, tau * spk, ws.q, ws.x);
        k_axpby<T>(c, n, spk, v, -cpk, ws.q);                   // q̄ₖ ← spₖ vₖ - cpₖ qₖ₋₁
      }
    } else if (!s.fused) {
      k_axpy<T>(c, n, tau, v, ws.x);
    }

    // βₖ₊₁Muₖ₊₁ = Avₖ - αₖMuₖ ; αₖ₊₁Nvₖ₊₁ = Aᴴuₖ₊₁ - βₖ₊₁Nvₖ
    T beta_next, alpha_next;
    if (s.fused) {
      beta_next = lnlq_fused_l1<T>(ws, *A.csr, iter == 1, s_u, alpha, ypend, yc, ys, wc, wsn);
      ypend = false;
      const T s_v_old = s_v;
      s_u = beta_next == 0 ? T(1) : T(1) / beta_next;           // kdiv!(m, u, β), applied by u's readers
      alpha_next = lnlq_fused_l2<T>(ws, *At.csr, s_v_old, beta_next, tau);
      s_v = alpha_next == 0 ? T(1) : T(1) / alpha_next;         // kdiv!(n, v, α), applied by v's readers
    } else {
      op_apply(c, A, v, ws.Av);
      k_axpby<T>(c, m, T(1), ws.Av, -alpha, ws.Mu);
      if (!s.MisI) op_apply(c, M, ws.Mu, u, ldiv);
      beta_next = knorm_elliptic<T>(c, m, u, ws.Mu);
      if (beta_next != 0) {
        k_scal<T>(c, m, T(1) / beta_next, u);
        if (!s.MisI) k_scal<T>(c, m, T(1) / beta_next, ws.Mu);
      }
      op_apply(c, At, u, ws.Atu);
      k_axpby<T>(c, n, T(1), ws.Atu, -beta_next, ws.Nv);
      if (!s.NisI) op_apply(c, N, ws.Nv, v, ldiv);
      alpha_next = knorm_elliptic<T>(c, n, v, ws.Nv);
      if (alpha_next != 0) {
        k_scal<T>(c, n, T(1) / alpha_next, v);
        if (!s.NisI) k_scal<T>(c, n, T(1) / alpha_next, ws.Nv);
      }
    }

    // Continue the regularization.
    T betahat, alphahat_next, cp_next = cpk, sp_next = spk;
    if (lambda > 0) {
      betahat = cpk * beta_next;
      const T theta_reg = spk * beta_next;
      T cdk, sdk, lambda_next;
      sym_givens<T>(lambda, theta_reg, &cdk, &sdk, &lambda_next);
      k_scal<T>(c, n, sdk, ws.q);                               // qₖ ← sdₖ q̄ₖ
      sym_givens<T>(alpha_next, lambda_next, &cp_next, &sp_next, &alphahat_next);
    } else {
      betahat = beta_next;
      alphahat_next = alpha_next;
    }

    T omega = 0;
    if (sigma_est > 0 && !complex_error_bnd) {                  // QR factorization for the Gauss-Radau estimate
      T mubar = -csig * alphahat;
      T rho = std::sqrt(rhobar * rhobar + alphahat * alphahat);
      csig = rhobar / rho;
      T ssig = alphahat / rho;
      rhobar = ssig * mubar + csig * sigma_est;
      mubar = -csig * betahat;
      const T theta = betahat * csig / rhobar;
      const T omega_disc = sigma_est * sigma_est - sigma_est * betahat * theta;
      if (omega_disc < 0) {
        complex_error_bnd = true;
      } else {
        omega = std::sqrt(omega_disc);
        tautilde = -tau * betahat / omega;
      }
      rho = std::sqrt(rhobar * rhobar + betahat * betahat);
      csig = rhobar / rho;
      ssig = betahat / rho;
      rhobar = ssig * mubar + csig * sigma_est;
    }

    // Lₖ₊₁tₖ₊₁ = β₁e₁, the LQ factorization of (Lₖ₊₁)ᴴ and M̅ₖ₊₁z̅ₖ₊₁ = tₖ₊₁
    const T tau_next = -betahat * tau / alphahat_next;
    T c_next, s_next, epsk;
    sym_givens<T>(epsbar, betahat, &c_next, &s_next, &epsk);
    const T eta_next = alphahat_next * s_next;
    const T epsbar_next = -alphahat_next * c_next;
    const T zetak = thetak / epsk;
    const T theta_next = tau_next - eta_next * zetak;
    const T zetabar_next = theta_next / epsbar_next;

    // (yᴸ)ₖ₊₁ ← (yᴸ)ₖ + ζₖ wₖ with wₖ = cₖ₊₁ w̄ₖ + sₖ₊₁ uₖ₊₁ ; w̄ₖ₊₁ = sₖ₊₁ w̄ₖ - cₖ₊₁ uₖ₊₁
    if (s.fused) {
      ypend = true;
      yc = zetak * c_next; ys = zetak * s_next; wc = -c_next; wsn = s_next;
    } else {
      k_axpy<T>(c, m, zetak * c_next, wbar, ws.y);
      k_axpy<T>(c, m, zetak * s_next, u, ws.y);
      k_axpby<T>(c, m, -c_next, u, s_next, wbar);
    }

    if (sigma_est > 0 && !complex_error_bnd) {
      if (transfer_to_craig) {
        const T disc_x = tautilde * tautilde - tau_next * tau_next;
        if (disc_x < 0) complex_error_bnd = true; else err_x = std::sqrt(disc_x);
      } else {
        const T d = tau_next - eta_next * zetak;
        const T disc_xL = tautilde * tautilde - tau_next * tau_next + d * d;
        if (disc_xL < 0) complex_error_bnd = true; else err_x = std::sqrt(disc_xL);
      }
      const T etatilde = omega * s_next;
      const T epstilde = -omega * c_next;
      const T zetatilde = (tautilde - etatilde * zetak) / epstilde;
      if (transfer_to_craig) {
        const T disc_y = zetatilde * zetatilde - zetabar_next * zetabar_next;
        if (disc_y < 0) complex_error_bnd = true; else err_y = std::sqrt(disc_y);
      } else {
        err_y = std::fabs(zetatilde);
      }
      if (history) { xNorms.push_back(err_x); yNorms.push_back(err_y); }
    }

    // ‖(rᴸ)ₖ‖ = |α̂ₖ| √(|ϵ̄ₖζ̄ₖ|² + |β̂ₖ₊₁sₖζₖ₋₁|²) ; the first pass reports ‖b‖ again
    T rNorm_lq;
    if (iter == 1) {
      rNorm_lq = bNorm;
    } else {
      const T ra = epsbar * zetabar, rb = betahat * sk * zeta_km1;
      rNorm_lq = std::fabs(alphahat) * std::sqrt(ra * ra + rb * rb);
    }
    if (history) stats.residuals.push_back(rNorm_lq);
    const T rNorm_cg = transfer_to_craig ? std::fabs(betahat * tau) : T(0);   // ‖(rᶜ)ₖ‖ = |β̂ₖ₊₁τₖ|

    if (ypend && o.callback) {                                  // the callback reads y
      lnlq_fused_flush<T>(ws, s_u, yc, ys, wc, wsn);
      ypend = false;
    }
    run.poll(iter, user_exit, overtimed);
    tired = iter >= itmax;
    solved_lq = rNorm_lq <= eps_c;
    solved_cg = transfer_to_craig && (std::fabs(zetabar) > eps) && (rNorm_cg <= eps_c);
    if (sigma_est > 0) {
      solved_lq = solved_lq || err_x <= utolx || err_y <= utoly;
      solved_cg = transfer_to_craig && (solved_cg || err_x <= utolx || err_y <= utoly);
    }
    if (kdisplay(iter, o.verbose)) printf("%5d  %7.1e  %.2fs\n", iter, (double)rNorm_lq, run.elapsed());

    sk = s_next;
    alpha = alpha_next;
    alphahat = alphahat_next;
    etak = eta_next;
    thetak = theta_next;
    epsbar = epsbar_next;
    tau = tau_next;
    zeta_km1 = zetak;
    zetabar = zetabar_next;
    if (lambda > 0) { cpk = cp_next; spk = sp_next; }
    iter = iter + 1;
  }
  if (o.verbose > 0) printf("\n");
  if (ypend) lnlq_fused_flush<T>(ws, s_u, yc, ys, wc, wsn);

  // The CRAIG point (signed test on ζ̄, unlike the loop's) or the LNLQ point
  const bool craig_point = solved_cg && (zetabar > eps);
  const T xcoef = craig_point ? tau : etak * zeta_km1;
  if (lambda > 0) {
    k_axpy<T>(c, n, xcoef * cpk, v, ws.x);
    if (iter >= 2) k_axpy<T>(c, n, xcoef * spk, ws.q, ws.x);
  } else if (s.fused) {
    lnlq_fused_xup<T>(ws, xcoef, s_v);
  } else {
    k_axpy<T>(c, n, xcoef, v, ws.x);
  }
  if (craig_point) k_axpy<T>(c, m, zetabar, wbar, ws.y);        // (yᶜ)ₖ ← (yᴸ)ₖ₋₁ + ζ̄ₖ w̄ₖ

  const char* st = "unknown";
  if (tired) st = "maximum number of iterations exceeded";
  if (solved_lq) st = "solutions (xᴸ, yᴸ) good enough for the tolerances given";
  if (solved_cg) st = "solutions (xᶜ, yᶜ) good enough for the tolerances given";
  if (user_exit) st = "user-requested exit";
  if (overtimed) st = "time limit exceeded";
  stats.error_with_bnd = complex_error_bnd;
  run.finish(iter, solved_lq || solved_cg, false, st);
}

// ===========================================================================
// cgne!  (src/cgne.jl:134-252): CG on A Aᴴ y = b, x = Aᴴ y (Craig's method).  N acts on the m-dimensional residual
// space: z = N r.  The first history entry is ‖b‖, every later one √⟨r, z⟩.  Fused (N = I, λ = 0, CSR A and Aᴴ): E1 on
// A, E2 on Aᴴ, one read-back of {γ, δ}; q and Aᴴz are not stored, x is current after every iteration.
// ===========================================================================
template <class T>
void cgne_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& N, const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int m = ws.m, n = ws.n;
  const bool history = o.history, ldiv = o.ldiv;
  if (o.verbose > 0) printf("CGNE: system of %d equations in %d variables\n", m, n);
  const bool NisI = N.is_identity();
  const T lambda = (T)o.lambda;
  const T atol = tol_of<T>(o.atol), rtol = tol_of<T>(o.rtol);
  const bool fused = o.fused && A.kind == LinOp<T>::CSR && At.kind == LinOp<T>::CSR && NisI && lambda == 0;
  Stats& stats = ws.stats;
  allocate_if(!NisI, ws, ws.z, m);
  allocate_if(lambda > 0, ws, ws.s, m);
  stats.reset();
  T* z = NisI ? ws.r : ws.z;

  k_fill<T>(c, n, ws.x, T(0));
  k_copy<T>(c, m, ws.r, b);                                     // r ← b
  if (!NisI) op_apply(c, N, ws.r, z, ldiv);
  T rNorm = k_nrm2<T>(c, m, ws.r);
  if (history) stats.residuals.push_back(rNorm);
  if (rNorm == 0) {
    run.finish(0, true, false, "x is a zero-residual solution");
    return;
  }
  if (lambda > 0) k_copy<T>(c, m, ws.s, ws.r);                  // s ← r
  op_apply(c, At, z, ws.p);
  T pNorm = k_nrm2<T>(c, n, ws.p);                              // ‖p‖ detects an inconsistent system
  T gamma = k_dot<T>(c, m, ws.r, z);
  int iter = 0;
  const int itmax = ls_itmax(ws, o.itmax);

  const T eps_c = atol + rtol * rNorm;                          // consistent systems
  const T eps_i = atol + rtol * pNorm;                          // inconsistent systems
  if (o.verbose > 0) printf("%5s  %8s  %5s\n", "k", "‖r‖", "timer");
  if (kdisplay(iter, o.verbose)) printf("%5d  %8.2e  %.2fs\n", iter, (double)rNorm, run.elapsed());

  bool solved = rNorm <= eps_c, inconsistent = (rNorm > 100 * eps_c) && (pNorm <= eps_i), tired = iter >= itmax;
  bool user_exit = false, overtimed = false;
  const T delta0 = fused && !(solved || inconsistent || tired) ? k_dot<T>(c, n, ws.p, ws.p) : T(0);
  while (!(solved || inconsistent || tired || user_exit || overtimed)) {
    if (fused) {
      T pp;
      cgne_fused_iteration<T>(ws, *A.csr, *At.csr, iter == 0, gamma, delta0, &gamma, &pp);
      pNorm = std::sqrt(pp);
      rNorm = std::sqrt(gamma);
    } else {
      op_apply(c, A, ws.p, ws.q);
      if (lambda > 0) k_axpy<T>(c, m, lambda, ws.s, ws.q);
      T delta = k_dot<T>(c, n, ws.p, ws.p);
      if (lambda > 0) delta += lambda * k_dot<T>(c, m, ws.s, ws.s);
      const T alpha = gamma / delta;
      k_axpy<T>(c, n, alpha, ws.p, ws.x);
      k_axpy<T>(c, m, -alpha, ws.q, ws.r);
      if (!NisI) op_apply(c, N, ws.r, z, ldiv);
      const T gamma_next = k_dot<T>(c, m, ws.r, z);
      const T beta = gamma_next / gamma;
      op_apply(c, At, z, ws.Ar);                                // Aᴴz
      k_axpby<T>(c, n, T(1), ws.Ar, beta, ws.p);                // p = Aᴴz + β p
      pNorm = k_nrm2<T>(c, n, ws.p);
      if (lambda > 0) k_axpby<T>(c, m, T(1), ws.r, beta, ws.s); // s = r + β s
      gamma = gamma_next;
      rNorm = std::sqrt(gamma_next);
    }
    if (history) stats.residuals.push_back(rNorm);
    iter = iter + 1;
    if (kdisplay(iter, o.verbose)) printf("%5d  %8.2e  %.2fs\n", iter, (double)rNorm, run.elapsed());
    const bool resid_decrease_mach = rNorm + T(1) <= T(1);
    run.poll(iter, user_exit, overtimed);
    const bool resid_decrease_lim = rNorm <= eps_c;
    solved = resid_decrease_lim || resid_decrease_mach;
    inconsistent = (rNorm > 100 * eps_c) && (pNorm <= eps_i);
    tired = iter >= itmax;
  }
  if (o.verbose > 0) printf("\n");
  const char* st = "unknown";
  if (tired) st = "maximum number of iterations exceeded";
  if (inconsistent) st = "system probably inconsistent";
  if (solved) st = "solution good enough given atol and rtol";
  if (user_exit) st = "user-requested exit";
  if (overtimed) st = "time limit exceeded";
  run.finish(iter, solved, inconsistent, st);
}

// ===========================================================================
// crmr!  (src/crmr.jl:132-244): CR on A Aᴴ y = b, x = Aᴴ y.  N acts on the m-dimensional residual space: r = N b and
// Nq = N q.  Fused (N = I, λ = 0, CSR A and Aᴴ): R1 on A, R2 over m, R3 on Aᴴ, R4 over n, one read-back of
// {‖r‖², γ}; x is current after every iteration.
// ===========================================================================
template <class T>
void crmr_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const LinOp<T>& N, const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int m = ws.m, n = ws.n;
  const bool history = o.history, ldiv = o.ldiv;
  if (o.verbose > 0) printf("CRMR: system of %d equations in %d variables\n", m, n);
  const bool NisI = N.is_identity();
  const T lambda = (T)o.lambda;
  const T atol = tol_of<T>(o.atol), rtol = tol_of<T>(o.rtol);
  const bool fused = o.fused && A.kind == LinOp<T>::CSR && At.kind == LinOp<T>::CSR && NisI && lambda == 0;
  Stats& stats = ws.stats;
  allocate_if(!NisI, ws, ws.z, m);
  allocate_if(lambda > 0, ws, ws.s, m);
  stats.reset();
  T* Nq = NisI ? ws.q : ws.z;

  k_fill<T>(c, n, ws.x, T(0));
  if (NisI) k_copy<T>(c, m, ws.r, b);                           // r = N b
  else op_apply(c, N, b, ws.r, ldiv);
  const T bNorm = k_nrm2<T>(c, m, ws.r);
  T rNorm = bNorm;
  if (history) stats.residuals.push_back(rNorm);
  if (bNorm == 0) {
    run.finish(0, true, false, "x is a zero-residual solution");
    if (history) stats.Aresiduals.push_back(0);
    return;
  }
  if (lambda > 0) k_copy<T>(c, m, ws.s, ws.r);                  // s ← r
  op_apply(c, At, ws.r, ws.Ar);
  k_copy<T>(c, n, ws.p, ws.Ar);                                 // p ← Aᴴr
  T gamma = k_dot<T>(c, n, ws.Ar, ws.Ar);
  if (lambda > 0) gamma += lambda * rNorm * rNorm;
  int iter = 0;
  const int itmax = ls_itmax(ws, o.itmax);

  T ArNorm = std::sqrt(gamma);
  if (history) stats.Aresiduals.push_back(ArNorm);
  const T eps_c = atol + rtol * rNorm;                          // consistent systems
  const T eps_i = atol + rtol * ArNorm;                         // inconsistent systems
  if (o.verbose > 0) printf("%5s  %8s  %8s  %5s\n", "k", "‖Aᴴr‖", "‖r‖", "timer");
  if (kdisplay(iter, o.verbose)) printf("%5d  %8.2e  %8.2e  %.2fs\n", iter, (double)ArNorm, (double)rNorm, run.elapsed());

  bool solved = rNorm <= eps_c, inconsistent = (rNorm > 100 * eps_c) && (ArNorm <= eps_i), tired = iter >= itmax;
  bool user_exit = false, overtimed = false;
  while (!(solved || inconsistent || tired || user_exit || overtimed)) {
    if (fused) {
      T rr;
      crmr_fused_iteration<T>(ws, *A.csr, *At.csr, iter == 0, gamma, &rr, &gamma);
      rNorm = std::sqrt(rr);
    } else {
      op_apply(c, A, ws.p, ws.q);
      if (lambda > 0) k_axpy<T>(c, m, lambda, ws.s, ws.q);     // q = q + λ s
      if (!NisI) op_apply(c, N, ws.q, Nq, ldiv);
      const T alpha = gamma / k_dot<T>(c, m, ws.q, Nq);        // qᴴ N q
      k_axpy<T>(c, n, alpha, ws.p, ws.x);
      k_axpy<T>(c, m, -alpha, Nq, ws.r);
      rNorm = k_nrm2<T>(c, m, ws.r);
      op_apply(c, At, ws.r, ws.Ar);
      T gamma_next = k_dot<T>(c, n, ws.Ar, ws.Ar);
      if (lambda > 0) gamma_next += lambda * rNorm * rNorm;
      const T beta = gamma_next / gamma;
      k_axpby<T>(c, n, T(1), ws.Ar, beta, ws.p);                // p = Aᴴr + β p
      if (lambda > 0) k_axpby<T>(c, m, T(1), ws.r, beta, ws.s); // s = r + β s
      gamma = gamma_next;
    }
    ArNorm = std::sqrt(gamma);
    if (history) { stats.residuals.push_back(rNorm); stats.Aresiduals.push_back(ArNorm); }
    iter = iter + 1;
    if (kdisplay(iter, o.verbose)) printf("%5d  %8.2e  %8.2e  %.2fs\n", iter, (double)ArNorm, (double)rNorm, run.elapsed());
    run.poll(iter, user_exit, overtimed);
    solved = rNorm <= eps_c;
    inconsistent = (rNorm > 100 * eps_c) && (ArNorm <= eps_i);
    tired = iter >= itmax;
  }
  if (o.verbose > 0) printf("\n");
  const char* st = "unknown";
  if (tired) st = "maximum number of iterations exceeded";
  if (solved) st = "solution good enough given atol and rtol";
  if (inconsistent) st = "system probably inconsistent but least squares/norm solution found";
  if (user_exit) st = "user-requested exit";
  if (overtimed) st = "time limit exceeded";
  run.finish(iter, solved, inconsistent, st);
}

#define INST(T)                                                                                                         \
  template void cgne_solve<T>(Workspace<T>&, const LinOp<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const SolveOpts&); \
  template void crmr_solve<T>(Workspace<T>&, const LinOp<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const SolveOpts&); \
  template void lnlq_solve<T>(Workspace<T>&, const LinOp<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const LinOp<T>&, \
                              const SolveOpts&);                                                                        \
  template void craig_solve<T>(Workspace<T>&, const LinOp<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const LinOp<T>&, \
                               const SolveOpts&);                                                                       \
  template void craigmr_solve<T>(Workspace<T>&, const LinOp<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const LinOp<T>&, \
                                 const SolveOpts&);                                                                     \
  template void lslq_solve<T>(Workspace<T>&, const LinOp<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const LinOp<T>&, \
                              const SolveOpts&);                                                                        \
  template void cgls_solve<T>(Workspace<T>&, const LinOp<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const SolveOpts&); \
  template void crls_solve<T>(Workspace<T>&, const LinOp<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const SolveOpts&); \
  template void lsqr_solve<T>(Workspace<T>&, const LinOp<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const LinOp<T>&, \
                              const SolveOpts&);                                                                        \
  template void lsmr_solve<T>(Workspace<T>&, const LinOp<T>&, const LinOp<T>&, const T*, const LinOp<T>&, const LinOp<T>&, \
                              const SolveOpts&);
INST(double)
INST(float)
#undef INST

}  // namespace kb
