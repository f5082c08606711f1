// biorth_lq.h -- the LQ factorization of the tridiagonal T_k = L̅_k Q_k kept on the host by bilq! (bilq.jl:265-305),
// bilqr! (bilqr.jl:251-294) and trilqr! (trilqr.jl:235-278).  The three solvers factor T_k the same way; they differ in
// the process that builds it (Lanczos biorthogonalization or SSY tridiagonalization) and in what they do with it.
#pragma once
#include <cmath>

#include "solver_common.h"

namespace kb {

template <class T> struct BilqLQ {
  T c1 = -1, c = -1, s1 = 0, s = 0;          // c_{k-1}, c_k, s_{k-1}, s_k
  T zeta2 = 0, zeta1 = 0, zetabar = 0;       // ζ_{k-2}, ζ_{k-1}, ζ̄_k
  T eta1 = 0, eta = 0, dbar1 = 0, dbar = 0;  // η_{k-1}, η_k, δ̄_{k-1}, δ̄_k
  T norm_v = 0;                              // ||v_k||
  T delta1 = 0, lambda = 0, eps2 = 0;        // this iteration's δ_{k-1}, λ_{k-1}, ϵ_{k-2} (0 where not formed)
  // T_k = L̅_k Q_k: the Givens rotation (c_k, s_k) and the last row of L̅_k
  void factor(int iter, T alpha, T beta, T gamma) {
    delta1 = 0; lambda = 0; eps2 = 0;
    if (iter == 1) {
      dbar = alpha;
    } else if (iter == 2) {
      sym_givens<T>(dbar1, gamma, &c, &s, &delta1);
      lambda = c * beta + s * alpha;
      dbar = s * beta - c * alpha;
    } else {
      sym_givens<T>(dbar1, gamma, &c, &s, &delta1);
      eps2 = s1 * beta;
      lambda = -c1 * c * beta + s * alpha;
      dbar = -c1 * s * beta - c * alpha;
    }
  }
  // ζ_{k-1} and η_k: forward substitution for z̄_k = L̅_k⁻¹ β₁ e₁
  void solve(int iter, T beta) {
    if (iter == 1) eta = beta;
    if (iter == 2) { zeta1 = eta1 / delta1; eta = -lambda * zeta1; }
    if (iter >= 3) { zeta2 = zeta1; zeta1 = eta1 / delta1; eta = -eps2 * zeta2 - lambda * zeta1; }
  }
  void step(int iter, T alpha, T beta, T gamma) { factor(iter, alpha, beta, gamma); solve(iter, beta); }
  // μ_k and ω_k of the LQ point's residual r_k = μ_k v_k + ω_k v_{k+1} (bilq.jl:342-343; iter >= 2)
  T mu(T alpha, T beta) const { return beta * (s1 * zeta2 - c1 * c * zeta1) + alpha * s * zeta1; }
  T omega(T beta1) const { return beta1 * s * zeta1; }
  // ||r_k|| of the LQ point (bilq.jl:339-346); vv1 = <v_k, v_{k+1}>
  T residual(int iter, T bNorm, T alpha, T beta, T beta1, T vv1, T norm_v1) const {
    if (iter == 1) return bNorm;
    const T mu_ = mu(alpha, beta);
    const T om = omega(beta1);
    const T th = mu_ * om * vv1;
    return std::sqrt((mu_ * mu_) * (norm_v * norm_v) + (om * om) * (norm_v1 * norm_v1) + 2 * th);
  }
};

}  // namespace kb
