// adjoint.cu -- host control flow of bilqr! (src/bilqr.jl:115-484) and trilqr! (src/trilqr.jl:114-461): one primal
// system A x = b and its adjoint A^T y = c, solved together from one Krylov process.  BiLQR (square A) runs the Lanczos
// biorthogonalization of bilq!, TriLQR (A m x n) the Saunders-Simon-Yip tridiagonalization; both factor the tridiagonal
// T_k = L̅_k Q_k (BilqLQ, biorth_lq.h) and run BiLQ's / USYMLQ's recurrence on the primal half and a QMR-type recurrence
// on the dual half.  One driver serves both: they differ in the process step and in the residual estimates.
//
// The x update stops once the primal half is solved and the y update once the dual half is; the process runs until
// both are.  The primitive path restates the reference line by line over blas1.cu / spmv.cu.  When A is a CSR operator
// with its cached A^T (and the workspace is not row-partitioned), the fused path runs an iteration as 3 launches
// (fused_phases.cu: BiLQR B1, B2, U; TriLQR T1, T2, U) with 2 read-backs (BiLQR) or 1 (TriLQR).  v_{k-1} / v_k and
// u_{k-1} / u_k rotate by pointer: the next vector is written into the buffer of the previous one.
#include <cmath>
#include <cstdio>
#include <utility>

#include "biorth_lq.h"
#include "solver_common.h"

namespace kb {

namespace {

template <class T>
void adjoint_solve(bool tri, Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const T* cvec,
                   const SolveOpts& o) {
  SolveRun<T> run(ws, o);
  Ctx& c = ws.ctx;
  const int m = ws.m, n = ws.n;                    // BiLQR: m == n.  TriLQR: b, y, v, q, w have m entries; c, x, u, p, d̅ n
  const bool history = o.history;
  const bool fused = o.fused && A.kind == LinOp<T>::CSR && At.kind == LinOp<T>::CSR && ws.dist.world == 1;
  const bool transfer = tri ? o.transfer_to_usymcg : o.transfer_to_bicg;
  if (o.verbose > 0) {
    if (tri) {
      printf("TRILQR: primal system of %d equations in %d variables\n", m, n);
      printf("TRILQR: dual system of %d equations in %d variables\n", n, m);
    } else {
      printf("BILQR: systems of size %d\n", n);
    }
  }
  const T atol = tol_of<T>(o.atol), rtol = tol_of<T>(o.rtol);
  Stats& stats = ws.stats;
  stats.reset();
  const bool warm_start = run.warm_start;
  const T* r0 = warm_start ? ws.q : b;             // r₀ = b - A Δx, s₀ = c - Aᵀ Δy
  const T* s0 = warm_start ? ws.p : cvec;
  if (warm_start) {
    op_apply(c, A, ws.dx, ws.q);
    k_axpby<T>(c, m, T(1), b, T(-1), ws.q);
    op_apply(c, At, ws.dy, ws.p);
    k_axpby<T>(c, n, T(1), cvec, T(-1), ws.p);
  }
  k_fill<T>(c, n, ws.x, T(0));
  const T bNorm = k_nrm2<T>(c, m, r0);
  k_fill<T>(c, m, ws.y, T(0));
  const T cNorm = k_nrm2<T>(c, n, s0);
  int iter = 0;
  const long long itmax_ll = o.itmax != 0 ? (long long)o.itmax : tri ? (long long)m + n : 2LL * n;
  const int itmax = itmax_ll > 2147483647LL ? 2147483647 : (int)itmax_ll;
  if (history) { stats.residuals.push_back(bNorm); stats.residuals_dual.push_back(cNorm); }
  const T epsL = atol + rtol * bNorm, epsQ = atol + rtol * cNorm;
  if (o.verbose > 0) printf("%5s  %7s  %7s  %5s\n", "k", "‖rₖ‖", "‖sₖ‖", "timer");
  if (kdisplay(iter, o.verbose)) printf("%5d  %7.1e  %7.1e  %.2fs\n", iter, (double)bNorm, (double)cNorm, run.elapsed());

  // the end of every exit: y += Δy, then x += Δx and the statistics (SolveRun::finish)
  auto finish = [&](bool solved_primal, bool solved_dual, const char* st) {
    if (warm_start) k_axpy<T>(c, m, T(1), ws.dy, ws.y);
    run.finish(iter, solved_primal && solved_dual, false, st);
    stats.solved_primal = solved_primal;
    stats.solved_dual = solved_dual;
  };

  T beta, gamma;
  if (tri) {
    beta = bNorm;                                  // β₁ = ‖r₀‖, γ₁ = ‖s₀‖
    gamma = cNorm;
  } else {
    const T cb = k_dot<T>(c, n, s0, r0);           // ⟨s₀,r₀⟩
    if (cb == 0) { finish(false, false, "Breakdown bᴴc = 0"); return; }
    beta = std::sqrt(std::fabs(cb));
    gamma = cb / beta;
  }
  // v₀ = u₀ = 0, d̅ = w_{k-3} = w_{k-2} = 0.  The fused passes never read d̅, w_{k-3} or w_{k-2} before writing them
  // (they use the zero w_{k-3} of iteration 3 as a constant), nor, in TriLQR, v₀ and u₀ (T1 / T2 skip those terms at
  // iteration 1): those fills are the primitive path's only.
  if (!fused || !tri) {
    k_fill<T>(c, m, ws.v_prev, T(0));
    k_fill<T>(c, n, ws.u_prev, T(0));
  }
  k_divcopy<T>(c, m, ws.v, r0, beta);
  k_divcopy<T>(c, n, ws.u, s0, gamma);
  BilqLQ<T> lq;
  lq.norm_v = bNorm / beta;                        // BiLQR: ‖v_k‖
  T psibar1 = 0, psibar = 0, psi1 = 0;             // ψ̄_{k-1}, ψ̄_k, ψ_{k-1}
  T eps3 = 0, lam2 = 0;                            // ϵ_{k-3}, λ_{k-2}
  T* wk3 = ws.w1;                                  // w_{k-3}, w_{k-2} (swapped by pointer)
  T* wk2 = ws.w2;
  if (!fused) {
    k_fill<T>(c, n, ws.w, T(0));
    k_fill<T>(c, m, wk3, T(0));
    k_fill<T>(c, m, wk2, T(0));
  }
  T tau = 0, xi = 0;                               // BiLQR: τ_k; TriLQR: ξ
  T uu = (fused && !tri) ? k_dot<T>(c, n, ws.u, ws.u) : T(0);   // fused BiLQR: ‖u_k‖², formed by the previous pass

  bool solved_lq = bNorm == 0, solved_lq_tol = false, solved_lq_mach = false;
  bool solved_cg = false, solved_cg_tol = false, solved_cg_mach = false;
  bool solved_primal = solved_lq || solved_cg;
  bool solved_qr_tol = false, solved_qr_mach = false, inconsistent = false;
  bool solved_dual = cNorm == 0;
  bool tired = iter >= itmax, breakdown = false, user_exit = false, overtimed = false;
  T rNorm_lq = 0, rNorm_cg = 0, sNorm = 0;
  while (!((solved_primal && solved_dual) || tired || breakdown || user_exit || overtimed)) {
    iter = iter + 1;
    // the process step: q and p, αₖ, βₖ₊₁ and γₖ₊₁
    T alpha, beta1, gamma1, pq = 0;
    if (tri) {                                     // SSY tridiagonalization (trilqr.jl:210-224)
      if (fused) {
        T qq, pp;
        trilqr_fused_ssy<T>(ws, *A.csr, *At.csr, iter == 1, beta, gamma, &alpha, &qq, &pp);
        beta1 = std::sqrt(qq);
        gamma1 = std::sqrt(pp);
      } else {
        op_apply(c, A, ws.u, ws.q);
        op_apply(c, At, ws.v, ws.p);
        if (iter >= 2) {
          k_axpy<T>(c, m, -gamma, ws.v_prev, ws.q);
          k_axpy<T>(c, n, -beta, ws.u_prev, ws.p);
        }
        alpha = k_dot<T>(c, m, ws.v, ws.q);
        k_axpy<T>(c, m, -alpha, ws.v, ws.q);
        k_axpy<T>(c, n, -alpha, ws.u, ws.p);
        beta1 = k_nrm2<T>(c, m, ws.q);
        gamma1 = k_nrm2<T>(c, n, ws.p);
      }
    } else {                                       // Lanczos biorthogonalization (bilqr.jl:227-240)
      if (fused) {
        biorth_fused_lanczos<T>(ws, *A.csr, *At.csr, beta, gamma, &alpha, &pq);
      } else {
        op_apply(c, A, ws.v, ws.q);
        op_apply(c, At, ws.u, ws.p);
        k_axpy<T>(c, n, -gamma, ws.v_prev, ws.q);
        k_axpy<T>(c, n, -beta, ws.u_prev, ws.p);
        alpha = k_dot<T>(c, n, ws.u, ws.q);
        k_axpy<T>(c, n, -alpha, ws.v, ws.q);
        k_axpy<T>(c, n, -alpha, ws.u, ws.p);
        pq = k_dot<T>(c, n, ws.p, ws.q);
      }
      beta1 = std::sqrt(std::fabs(pq));
      gamma1 = pq / beta1;
    }

    lq.factor(iter, alpha, beta, gamma);           // T_k = L̅_k Q_k
    const bool primal = !solved_primal, dual = !solved_dual;   // the halves this iteration updates
    if (primal) lq.solve(iter, beta);              // ζ_{k-1}, η_k
    if (dual) {                                    // ψ_{k-1}, ψ̄_k: the last components of h̅_k = Q_k γ₁ e₁
      if (iter == 1) psibar = gamma;
      else { psi1 = lq.c * psibar1; psibar = lq.s * psibar1; }
    }
    T* wk = dual && iter >= 2 ? (iter == 2 ? wk2 : wk3) : nullptr;   // w_{k-1}'s buffer
    const T czeta = lq.zeta1 * lq.c, szeta = lq.zeta1 * lq.s;
    T vq = 0, norm_v1 = 0;                         // BiLQR: ⟨v_k, q⟩ and ‖v_{k+1}‖
    if (fused) {
      if (tri) {
        trilqr_fused_update<T>(ws, primal, dual, iter, czeta, szeta, lq.c, lq.s, wk, wk2, eps3, lam2, lq.delta1, psi1, beta1, gamma1);
      } else {
        T out[3];
        bilqr_fused_update<T>(ws, primal, dual, iter, czeta, szeta, lq.c, lq.s, wk, wk2, eps3, lam2, lq.delta1, psi1, beta1, gamma1,
                              pq == T(0), out);
        vq = out[0];
        norm_v1 = std::sqrt(out[1]) / beta1;
        if (dual) tau = tau + uu;                  // τ_k = τ_{k-1} + ‖u_k‖²
        uu = out[2];                               // ‖u_{k+1}‖²
      }
    } else {
      const T* a = tri ? ws.u : ws.v;              // the primal directions d̅ live in the space of x
      if (primal) {
        if (iter == 1) {
          k_copy<T>(c, n, ws.w, a);                // d̅₁ = v₁ (BiLQR), u₁ (TriLQR)
        } else {
          k_axpy<T>(c, n, czeta, ws.w, ws.x);
          k_axpy<T>(c, n, szeta, a, ws.x);
          k_axpby<T>(c, n, -lq.c, a, lq.s, ws.w);
        }
        if (!tri) {
          vq = k_dot<T>(c, n, ws.v, ws.q);
          norm_v1 = k_nrm2<T>(c, n, ws.q) / beta1;
        }
      }
      if (dual) {
        const T* src = tri ? ws.v_prev : ws.u_prev;   // w_{k-1} = (src - λ̄ₖ₋₂ wₖ₋₂ - ϵ̄ₖ₋₃ wₖ₋₃) / δ̄ₖ₋₁
        if (iter == 2) k_divcopy<T>(c, m, wk, src, lq.delta1);
        if (iter >= 3) {
          if (iter >= 4) k_scal<T>(c, m, -eps3, wk3);
          k_axpy<T>(c, m, T(1), src, wk);
          k_axpy<T>(c, m, -lam2, wk2, wk);
          k_scal<T>(c, m, T(1) / lq.delta1, wk);
        }
        if (iter >= 2) k_axpy<T>(c, m, psi1, wk, ws.y);
        if (!tri) tau = tau + k_dot<T>(c, n, ws.u, ws.u);
      }
      // v_{k+1}, u_{k+1} into the buffers of v_{k-1}, u_{k-1}; kept (copies of v_k, u_k) where the reference keeps them
      if (tri ? beta1 != T(0) : pq != T(0)) k_divcopy<T>(c, m, ws.v_prev, ws.q, beta1);
      else k_copy<T>(c, m, ws.v_prev, ws.v);
      if (tri ? gamma1 != T(0) : pq != T(0)) k_divcopy<T>(c, n, ws.u_prev, ws.p, gamma1);
      else k_copy<T>(c, n, ws.u_prev, ws.u);
    }
    std::swap(ws.v, ws.v_prev);
    std::swap(ws.u, ws.u_prev);
    if (dual && iter >= 3) std::swap(wk3, wk2);

    if (primal) {                                  // bilqr.jl:313-347, trilqr.jl:297-323
      if (tri) {
        rNorm_lq = bNorm;
        if (iter >= 2) {
          const T mu = lq.mu(alpha, beta), om = lq.omega(beta1);
          rNorm_lq = std::sqrt(mu * mu + om * om);
        }
      } else {
        rNorm_lq = lq.residual(iter, bNorm, alpha, beta, beta1, vq / beta1, norm_v1);
        lq.norm_v = norm_v1;
      }
      if (history) stats.residuals.push_back(rNorm_lq);
      const bool cg_ok = transfer && std::fabs(lq.dbar) > eps_of<T>();
      if (cg_ok) {                                 // BiCG / USYMCG residual norm
        lq.zetabar = lq.eta / lq.dbar;
        const T rho = beta1 * (lq.s * lq.zeta1 - lq.c * lq.zetabar);
        rNorm_cg = tri ? std::fabs(rho) : std::fabs(rho) * norm_v1;
      }
      solved_lq_tol = rNorm_lq <= epsL;
      solved_lq_mach = rNorm_lq + T(1) <= T(1);
      solved_lq = solved_lq_tol || solved_lq_mach;
      solved_cg_tol = cg_ok && rNorm_cg <= epsL;
      solved_cg_mach = cg_ok && rNorm_cg + T(1) <= T(1);
      solved_cg = solved_cg_tol || solved_cg_mach;
      solved_primal = solved_lq || solved_cg;
    }
    if (dual) {                                    // bilqr.jl:394-407, trilqr.jl:370-385
      psibar1 = psibar;
      T AsNorm = 0;
      if (tri) {
        sNorm = std::fabs(psibar);                 // ‖s_{k-1}‖ = |ψ̄_k|, ‖A s_{k-1}‖ = |ψ̄_k| √(|δ̄_k|² + |c_k β_{k+1}|²)
        const T cb1 = lq.c * beta1;
        AsNorm = std::fabs(psibar) * std::sqrt(lq.dbar * lq.dbar + cb1 * cb1);
        if (iter == 1) xi = atol + rtol * AsNorm;
      } else {
        sNorm = std::fabs(psibar) * std::sqrt(tau);   // ‖s_{k-1}‖ ≤ |ψ̄_k| √τ_k
      }
      if (history) stats.residuals_dual.push_back(sNorm);
      solved_qr_tol = sNorm <= epsQ;
      solved_qr_mach = sNorm + T(1) <= T(1);
      inconsistent = tri && AsNorm <= xi;
      solved_dual = solved_qr_tol || solved_qr_mach || inconsistent;
    }

    if (iter >= 3) eps3 = lq.eps2;
    if (iter >= 2) lam2 = lq.lambda;
    lq.dbar1 = lq.dbar; lq.c1 = lq.c; lq.s1 = lq.s; lq.eta1 = lq.eta;
    gamma = gamma1;
    beta = beta1;
    run.poll(iter, user_exit, overtimed);
    tired = iter >= itmax;
    breakdown = !tri && !solved_lq && !solved_cg && pq == T(0);
    if (kdisplay(iter, o.verbose)) {
      if (solved_primal && !solved_dual) printf("%5d  %7s  %7.1e  %.2fs\n", iter, "✗ ✗ ✗ ✗", (double)sNorm, run.elapsed());
      if (!solved_primal && solved_dual) printf("%5d  %7.1e  %7s  %.2fs\n", iter, (double)rNorm_lq, "✗ ✗ ✗ ✗", run.elapsed());
      if (!solved_primal && !solved_dual) printf("%5d  %7.1e  %7.1e  %.2fs\n", iter, (double)rNorm_lq, (double)sNorm, run.elapsed());
    }
  }
  if (o.verbose > 0) printf("\n");
  if (solved_cg) k_axpy<T>(c, n, lq.zetabar, ws.w, ws.x);   // BiCG / USYMCG point x + ζ̄ d̅

  // the termination status, word for word (bilqr.jl:451-469, trilqr.jl:429-446)
  const char* st = "unknown";
  if (tired) st = "maximum number of iterations exceeded";
  if (breakdown) st = "Breakdown ⟨uₖ₊₁,vₖ₊₁⟩ = 0";
  if (solved_lq_tol && !solved_dual) st = "Only the primal solution xᴸ is good enough given atol and rtol";
  if (solved_cg_tol && !solved_dual) st = "Only the primal solution xᶜ is good enough given atol and rtol";
  if (!solved_primal && solved_qr_tol) st = "Only the dual solution t is good enough given atol and rtol";
  if (solved_lq_tol && solved_qr_tol) st = "Both primal and dual solutions (xᴸ, t) are good enough given atol and rtol";
  if (solved_cg_tol && solved_qr_tol) st = "Both primal and dual solutions (xᶜ, t) are good enough given atol and rtol";
  if (solved_lq_mach && !solved_dual) st = "Only found approximate zero-residual primal solution xᴸ";
  if (solved_cg_mach && !solved_dual) st = "Only found approximate zero-residual primal solution xᶜ";
  if (!solved_primal && solved_qr_mach) st = "Only found approximate zero-residual dual solution t";
  if (solved_lq_mach && solved_qr_mach) st = "Found approximate zero-residual primal and dual solutions (xᴸ, t)";
  if (solved_cg_mach && solved_qr_mach) st = "Found approximate zero-residual primal and dual solutions (xᶜ, t)";
  if (solved_lq_mach && solved_qr_tol)
    st = "Found approximate zero-residual primal solutions xᴸ and a dual solution t good enough given atol and rtol";
  if (solved_cg_mach && solved_qr_tol)
    st = "Found approximate zero-residual primal solutions xᶜ and a dual solution t good enough given atol and rtol";
  if (solved_lq_tol && solved_qr_mach)
    st = "Found a primal solution xᴸ good enough given atol and rtol and an approximate zero-residual dual solutions t";
  if (solved_cg_tol && solved_qr_mach)
    st = "Found a primal solution xᶜ good enough given atol and rtol and an approximate zero-residual dual solutions t";
  if (user_exit) st = "user-requested exit";
  if (overtimed) st = "time limit exceeded";
  finish(solved_primal, solved_dual, st);
}

}  // namespace

template <class T>
void bilqr_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const T* c, const SolveOpts& o) {
  adjoint_solve<T>(false, ws, A, At, b, c, o);
}

template <class T>
void trilqr_solve(Workspace<T>& ws, const LinOp<T>& A, const LinOp<T>& At, const T* b, const T* c, const SolveOpts& o) {
  adjoint_solve<T>(true, ws, A, At, b, c, o);
}

// warm_start!(workspace, x0, y0) (src/workspace_accessors.jl): Δx (n entries) and Δy (m entries)
template <class T> void ws_warm_start2(Workspace<T>* ws, const T* x0_dev, const T* y0_dev) {
  allocate_if(true, *ws, ws->dx, ws->n);
  allocate_if(true, *ws, ws->dy, ws->m);
  k_copy<T>(ws->ctx, ws->n, ws->dx, x0_dev);
  k_copy<T>(ws->ctx, ws->m, ws->dy, y0_dev);
  ws->warm_start = true;
}

#define INST(T)                                                                                                        \
  template void bilqr_solve<T>(Workspace<T>&, const LinOp<T>&, const LinOp<T>&, const T*, const T*, const SolveOpts&); \
  template void trilqr_solve<T>(Workspace<T>&, const LinOp<T>&, const LinOp<T>&, const T*, const T*, const SolveOpts&); \
  template void ws_warm_start2<T>(Workspace<T>*, const T*, const T*);
INST(double)
INST(float)
#undef INST

}  // namespace kb
