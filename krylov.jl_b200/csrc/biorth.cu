// biorth.cu -- host control flow of bilq! (src/bilq.jl:118-407) and qmr! (src/qmr.jl:124-405) on a square operator.
// Both run the same Lanczos biorthogonalization (one product with A and one with A^H per iteration) and differ only in
// the small factorization kept on the host -- BiLQ an LQ factorization of T_k, QMR a QR factorization of T_{k+1,k} --
// and in their direction / solution update.  One driver serves both.  The primitive path restates the reference line
// by line over blas1.cu / spmv.cu.  When A is a CSR operator with its cached A^T and M = N = I, the fused path runs an
// iteration as 3 launches (fused_phases.cu: B1 on A, B2 on A^T, one update pass over n) and 2 read-backs.  The scalar
// recurrences, stopping tests and status strings run on the host, unchanged.  v_{k-1} / v_k and u_{k-1} / u_k rotate by
// pointer instead of kcopy!: the next vector is written into the buffer of the previous one.
#include <cmath>
#include <cstdio>
#include <utility>

#include "biorth_lq.h"
#include "solver_common.h"

namespace kb {

namespace {

// QR factorization of T_{k+1,k} by Givens reflections and the update of z̄ (qmr.jl:275-312)
template <class T> struct QmrQR {
  T c2 = 0, c1 = 0, s2 = 0, s1 = 0;          // c_{k-2}, c_{k-1}, s_{k-2}, s_{k-1}
  T zetabar = 0, tau = 0;                    // last component of z̄_k; running sum of ||v_i||^2
  T eps2 = 0, lambda = 0, delta = 0, zeta = 0, zetabar1 = 0;   // this iteration's ϵ_{k-2}, λ_{k-1}, δ_k, ζ_k, ζ̄_{k+1}
  void step(int iter, T alpha, T gamma, T beta1) {
    T lbar = 0, dbar = 0;
    if (iter >= 3) { eps2 = s2 * gamma; lbar = -c2 * gamma; }
    if (iter >= 2) {
      if (iter == 2) lbar = gamma;
      lambda = c1 * lbar + s1 * alpha;
      dbar = s1 * lbar - c1 * alpha;
      s2 = s1; c2 = c1;
    }
    if (iter == 1) dbar = alpha;
    T c, s;
    sym_givens<T>(dbar, beta1, &c, &s, &delta);
    zeta = c * zetabar;
    zetabar1 = s * zetabar;
    s1 = s; c1 = c;
  }
};

// v_{k+1} = q / beta_{k+1} and u_{k+1} = p / gamma_{k+1} into the buffers of v_{k-1}, u_{k-1} (pq = 0: v_k and u_k are
// kept, bilq.jl:325-331), then the rotation.
template <class T> void next_vectors(Workspace<T>& ws, bool keep, T beta1, T gamma1) {
  Ctx& c = ws.ctx;
  if (keep) {
    k_copy<T>(c, ws.n, ws.v_prev, ws.v);
    k_copy<T>(c, ws.n, ws.u_prev, ws.u);
  } else {
    k_divcopy<T>(c, ws.n, ws.v_prev, ws.q, beta1);
    k_divcopy<T>(c, ws.n, ws.u_prev, ws.p, gamma1);
  }
}
template <class T> void rotate(Workspace<T>& ws) { std::swap(ws.v, ws.v_prev); std::swap(ws.u, ws.u_prev); }

template <class T>
void biorth_solve(bool qmr, Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const T* c_in,
                  const LinOp<T>& M, const LinOp<T>& N, const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int n = ws.n;
  const bool history = o.history, ldiv = o.ldiv;
  if (o.verbose > 0) printf("%s: system of size %d\n", qmr ? "QMR" : "BILQ", n);
  const bool MisI = M.is_identity(), NisI = N.is_identity();
  const bool fused = o.fused && A.kind == LinOp<T>::CSR && At.kind == LinOp<T>::CSR && MisI && NisI && ws.dist.world == 1;
  const T atol = tol_of<T>(o.atol), rtol = tol_of<T>(o.rtol);
  Stats& stats = ws.stats;
  allocate_if(!MisI, ws, ws.t);
  allocate_if(!NisI, ws, ws.s);
  stats.reset();
  const T* cvec = c_in ? c_in : b;                 // kwarg c = b
  const T* r0 = run.warm_start ? ws.q : b;
  if (run.warm_start) {
    op_apply(c, A, ws.dx, ws.q);
    k_axpby<T>(c, n, T(1), b, T(-1), ws.q);
  }
  if (!MisI) { op_apply(c, M, r0, ws.t, ldiv); r0 = ws.t; }
  k_fill<T>(c, n, ws.x, T(0));
  const T bNorm = k_nrm2<T>(c, n, r0);
  if (history) stats.residuals.push_back(bNorm);
  if (bNorm == 0) { run.finish(0, true, false, "x is a zero-residual solution"); return; }
  int iter = 0;
  const int itmax = default_itmax(ws, o.itmax);
  const T cb = k_dot<T>(c, n, cvec, r0);           // ⟨c, r₀⟩
  if (cb == 0) { run.finish(0, false, false, "Breakdown bᴴc = 0"); return; }
  const T eps = atol + rtol * bNorm;
  if (o.verbose > 0) printf("%5s  %8s  %7s  %5s\n", "k", "αₖ", "‖rₖ‖", "timer");
  if (kdisplay(iter, o.verbose)) printf("%5d  %8.1e  %7.1e  %.2fs\n", iter, (double)cb, (double)bNorm, run.elapsed());

  T beta = std::sqrt(std::fabs(cb)), gamma = cb / beta;
  k_fill<T>(c, n, ws.v_prev, T(0));
  k_fill<T>(c, n, ws.u_prev, T(0));
  k_divcopy<T>(c, n, ws.v, r0, beta);
  k_divcopy<T>(c, n, ws.u, cvec, gamma);
  QmrQR<T> qr;
  BilqLQ<T> lq;
  T* wk2 = ws.w1;                                  // QMR: w_{k-2}, w_{k-1} (swapped by pointer, qmr.jl:357-359)
  T* wk1 = ws.w2;
  if (qmr) {
    k_fill<T>(c, n, wk2, T(0));
    k_fill<T>(c, n, wk1, T(0));
    qr.zetabar = beta;
    qr.tau = k_dot<T>(c, n, ws.v, ws.v);
  } else {
    k_fill<T>(c, n, ws.w, T(0));                   // d̅
    lq.norm_v = bNorm / beta;
  }

  bool solved = bNorm <= eps, solved_cg = false, breakdown = false, tired = iter >= itmax, user_exit = false,
       overtimed = false;
  T rNorm_cg = 0;
  while (!(solved || solved_cg || tired || breakdown || user_exit || overtimed)) {
    iter = iter + 1;
    // Lanczos biorthogonalization (bilq.jl:234-254, qmr.jl:238-258)
    T alpha, pq;
    if (fused) {
      biorth_fused_lanczos<T>(ws, *A.csr, *At.csr, beta, gamma, &alpha, &pq);
    } else {
      T* Nv = NisI ? ws.v : ws.s;
      T* t = MisI ? ws.q : ws.t;
      T* Mu = MisI ? ws.u : ws.t;
      T* s = NisI ? ws.p : ws.s;
      if (!NisI) op_apply(c, N, ws.v, Nv, ldiv);
      op_apply(c, A, Nv, t);
      if (!MisI) op_apply(c, M, t, ws.q, ldiv);
      if (!MisI) op_apply(c, M, ws.u, Mu, ldiv);   // Mᴴ = M: diagonal preconditioners, or self-adjoint callbacks
      op_apply(c, At, Mu, s);
      if (!NisI) op_apply(c, N, s, ws.p, ldiv);
      k_axpy<T>(c, n, -gamma, ws.v_prev, ws.q);
      k_axpy<T>(c, n, -beta, ws.u_prev, ws.p);
      alpha = k_dot<T>(c, n, ws.u, ws.q);
      k_axpy<T>(c, n, -alpha, ws.v, ws.q);
      k_axpy<T>(c, n, -alpha, ws.u, ws.p);
      pq = k_dot<T>(c, n, ws.p, ws.q);
    }
    const T beta1 = std::sqrt(std::fabs(pq)), gamma1 = pq / beta1;
    const bool keep = pq == T(0);
    T rNorm;
    if (qmr) {
      qr.step(iter, alpha, gamma, beta1);
      T* wk = iter == 1 ? wk1 : wk2;               // w_k overwrites w_{k-1} (k = 1) or w_{k-2}
      T vv;
      if (fused) {
        vv = qmr_fused_update<T>(ws, wk, wk1, iter, qr.eps2, qr.lambda, qr.delta, qr.zeta, beta1, gamma1, keep);
      } else {
        if (iter == 1) {
          k_divcopy<T>(c, n, wk, ws.v, qr.delta);
        } else {
          if (iter >= 3) k_scal<T>(c, n, -qr.eps2, wk);
          k_axpy<T>(c, n, -qr.lambda, wk1, wk);
          k_axpy<T>(c, n, T(1), ws.v, wk);
          k_scal<T>(c, n, T(1) / qr.delta, wk);
        }
        k_axpy<T>(c, n, qr.zeta, wk, ws.x);
        next_vectors<T>(ws, keep, beta1, gamma1);
        vv = k_dot<T>(c, n, ws.v_prev, ws.v_prev);
      }
      rotate(ws);
      const T tau1 = qr.tau + vv;                  // τ_{k+1} = τ_k + ||v_{k+1}||²
      rNorm = std::fabs(qr.zetabar1) * std::sqrt(tau1);
      if (iter >= 2) std::swap(wk2, wk1);
      qr.zetabar = qr.zetabar1;
      qr.tau = tau1;
    } else {
      lq.step(iter, alpha, beta, gamma);
      T vv1, norm_v1;
      if (fused) {
        T v1v1;
        bilq_fused_update<T>(ws, iter == 1, lq.zeta1 * lq.c, lq.zeta1 * lq.s, lq.c, lq.s, beta1, gamma1, keep, &vv1, &v1v1);
        norm_v1 = std::sqrt(v1v1);
        rotate(ws);
      } else {
        if (iter == 1) {
          k_copy<T>(c, n, ws.w, ws.v);                                  // d̅₁ = v₁
        } else {
          k_axpy<T>(c, n, lq.zeta1 * lq.c, ws.w, ws.x);
          k_axpy<T>(c, n, lq.zeta1 * lq.s, ws.v, ws.x);
          k_axpby<T>(c, n, -lq.c, ws.v, lq.s, ws.w);
        }
        next_vectors<T>(ws, keep, beta1, gamma1);
        rotate(ws);
        vv1 = k_dot<T>(c, n, ws.v_prev, ws.v);      // ⟨v_k, v_{k+1}⟩
        norm_v1 = k_nrm2<T>(c, n, ws.v);
      }
      rNorm = lq.residual(iter, bNorm, alpha, beta, beta1, vv1, norm_v1);
      const bool bicg = o.transfer_to_bicg && std::fabs(lq.dbar) > eps_of<T>();
      if (bicg) {                                   // BiCG residual norm (bilq.jl:351-355)
        lq.zetabar = lq.eta / lq.dbar;
        const T rho = beta1 * (lq.s * lq.zeta1 - lq.c * lq.zetabar);
        rNorm_cg = std::fabs(rho) * norm_v1;
      }
      lq.s1 = lq.s; lq.c1 = lq.c; lq.eta1 = lq.eta; lq.dbar1 = lq.dbar; lq.norm_v = norm_v1;
      solved_cg = bicg && rNorm_cg <= eps;
    }
    if (history) stats.residuals.push_back(rNorm);
    gamma = gamma1;
    beta = beta1;
    run.poll(iter, user_exit, overtimed);
    solved = rNorm <= eps || (qmr && rNorm + T(1) <= T(1));
    tired = iter >= itmax;
    breakdown = !solved && !solved_cg && pq == T(0);
    if (kdisplay(iter, o.verbose)) printf("%5d  %8.1e  %7.1e  %.2fs\n", iter, (double)alpha, (double)rNorm, run.elapsed());
  }
  if (o.verbose > 0) printf("\n");
  if (solved_cg) k_axpy<T>(c, n, lq.zetabar, ws.w, ws.x);   // BiCG point x + ζ̄ d̅ (bilq.jl:380-382)
  const char* st = "unknown";
  if (tired) st = "maximum number of iterations exceeded";
  if (breakdown) st = "Breakdown ⟨uₖ₊₁,vₖ₊₁⟩ = 0";
  if (solved) st = qmr ? "solution good enough given atol and rtol" : "solution xᴸ good enough given atol and rtol";
  if (solved_cg) st = "solution xᶜ good enough given atol and rtol";
  if (user_exit) st = "user-requested exit";
  if (overtimed) st = "time limit exceeded";
  if (!NisI) {
    k_copy<T>(c, n, ws.s, ws.x);
    op_apply(c, N, ws.s, ws.x, ldiv);
  }
  run.finish(iter, solved || solved_cg, false, st);
}

}  // namespace

template <class T>
void bilq_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const T* c, const LinOp<T>& M,
                const LinOp<T>& N, const SolveOpts& o) {
  biorth_solve<T>(false, ws, A, At, b, c, M, N, o);
}

template <class T>
void qmr_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const T* c, const LinOp<T>& M,
               const LinOp<T>& N, const SolveOpts& o) {
  biorth_solve<T>(true, ws, A, At, b, c, M, N, o);
}

#define INST(T)                                                                                                        \
  template void bilq_solve<T>(Workspace<T>&, const LinOp<T>&, const LinOp<T>&, const T*, const T*, const LinOp<T>&,    \
                              const LinOp<T>&, const SolveOpts&);                                                      \
  template void qmr_solve<T>(Workspace<T>&, const LinOp<T>&, const LinOp<T>&, const T*, const T*, const LinOp<T>&,     \
                             const LinOp<T>&, const SolveOpts&);
INST(double)
INST(float)
#undef INST

}  // namespace kb
