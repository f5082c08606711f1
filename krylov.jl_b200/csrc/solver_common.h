// solver_common.h -- small host helpers shared by the solver drivers (solvers.cu, siblings.cu, lsq.cu).
#pragma once
#include <cmath>
#include <limits>
#include <string>

#include "kb_internal.h"

namespace kb {

template <class T> static inline T eps_of() { return std::numeric_limits<T>::epsilon(); }
template <class T> static inline T tol_of(double t) { return t < 0 ? std::sqrt(eps_of<T>()) : (T)t; }

// allocate_if (src/krylov_utils.jl:281-288); len < 0: ws.n entries (LSQR / LSMR also hold vectors of m entries)
template <class T> static inline void allocate_if(bool cond, Workspace<T>& ws, T*& v, int len = -1) {
  const double t0 = now_seconds();
  if (cond && !v) v = dev_alloc<T>((size_t)(len < 0 ? ws.n : len));
  ws.stats.allocation_timer += now_seconds() - t0;
}

// Row-partitioned solves: exit decisions taken from a per-rank clock or callback are OR-ed over the ranks (one extra
// tiny launch per iteration, only when a callback or a finite timemax is in play).
template <class T> static inline void agree_exit(Workspace<T>& ws, const SolveOpts& o, bool& user_exit, bool& overtimed) {
  if (ws.dist.world > 1 && (o.callback != nullptr || o.timemax < 1e300)) dist_agree_on_exit(ws.ctx, user_exit, overtimed);
}

// The library's exit protocol, shared by every single right-hand-side driver.  Constructed at driver entry: it takes
// the start time and the warm-start flag there.
template <class T> struct SolveRun {
  Workspace<T>& ws;
  const SolveOpts& o;
  const double start;
  const bool warm_start;
  SolveRun(Workspace<T>& ws_, const SolveOpts& o_) : ws(ws_), o(o_), start(now_seconds()), warm_start(ws_.warm_start) {}
  double elapsed() const { return now_seconds() - start; }
  // End of an iteration: the callback (when one is set and `callback` is true) sees a synchronized stream and
  // stats.niter = niter; the clock is read after it; a row-partitioned solve ORs both flags over the ranks.
  void poll(int niter, bool& user_exit, bool& overtimed, bool callback = true) {
    if (callback && o.callback) { ws.ctx.sync(); ws.stats.niter = niter; user_exit = o.callback(&ws, o.callback_user) != 0; }
    overtimed = elapsed() > o.timemax;
    agree_exit(ws, o, user_exit, overtimed);
  }
  // End of the solve: x += dx when warm-started (unless add_dx is false), one sync, then the statistics.
  void finish(int niter, bool solved, bool inconsistent, const std::string& status, bool add_dx = true) {
    if (warm_start && add_dx) k_axpy<T>(ws.ctx, ws.n, T(1), ws.dx, ws.x);
    ws.warm_start = false;
    ws.ctx.sync();
    Stats& st = ws.stats;
    st.niter = niter; st.solved = solved; st.inconsistent = inconsistent;
    st.timer = elapsed();
    st.status = status;
  }
};

static inline bool kdisplay(int iter, int verbose) { return verbose > 0 && iter % verbose == 0; }

// default itmax = 2n of the GLOBAL system (row-partitioned workspaces hold a slice)
template <class T> static inline int default_itmax(const Workspace<T>& ws, int itmax) {
  if (itmax != 0) return itmax;
  const long long two_n = 2LL * (ws.dist.world > 1 ? ws.dist.nglobal : (long long)ws.n);
  return two_n > 2147483647LL ? 2147483647 : (int)two_n;
}

// sym_givens, real case (src/krylov_utils.jl:21-51)
template <class T> static inline void sym_givens(T a, T b, T* c, T* s, T* rho) {
  const T sa = (T)((a > 0) - (a < 0)), sb = (T)((b > 0) - (b < 0));
  if (b == T(0)) { *c = sa + (T)(a == T(0)); *s = T(0); *rho = std::fabs(a); }
  else if (a == T(0)) { *c = T(0); *s = sb; *rho = std::fabs(b); }
  else if (std::fabs(b) > std::fabs(a)) {
    const T t = a / b;
    *s = sb / std::sqrt(T(1) + t * t); *c = *s * t; *rho = b / *s;
  } else {
    const T t = b / a;
    *c = sa / std::sqrt(T(1) + t * t); *s = *c * t; *rho = a / *c;
  }
}

// roots_quadratic (src/krylov_utils.jl:110-152); returns nonzero where the reference raises.
template <class T> static inline int roots_quadratic(T q2, T q1, T q0, int nitref, T* r1, T* r2) {
  T root1, root2;
  if (q2 == T(0)) {
    T root;
    if (q1 == T(0)) { if (q0 != T(0)) return 1; root = T(0); }
    else root = -q0 / q1;
    *r1 = root; *r2 = root;
    return 0;
  }
  const T rhs = std::sqrt(eps_of<T>()) * q1 * q1;
  if (std::fabs(q0 * q2) > rhs) {
    const T rho = q1 * q1 - 4 * q2 * q0;
    if (rho < 0) return 1;
    const T d = -(q1 + std::copysign(std::sqrt(rho), q1)) / 2;
    root1 = d / q2; root2 = q0 / d;
  } else {
    root1 = -q1 / q2; root2 = T(0);
  }
  for (int it = 0; it < nitref; it++) {
    const T q = (q2 * root1 + q1) * root1 + q0, dq = 2 * q2 * root1 + q1;
    if (dq == T(0)) continue;
    root1 = root1 - q / dq;
  }
  for (int it = 0; it < nitref; it++) {
    const T q = (q2 * root2 + q1) * root2 + q0, dq = 2 * q2 * root2 + q1;
    if (dq == T(0)) continue;
    root2 = root2 - q / dq;
  }
  *r1 = root1; *r2 = root2;
  return 0;
}

// to_boundary (src/krylov_utils.jl:375-402)
template <class T>
static inline int to_boundary(Ctx& c, int n, const T* x, const T* d, T* z, T radius, T dNorm2, const LinOp<T>& M, bool ldiv, T* s1, T* s2) {
  if (!(radius > 0)) return 1;
  T rxd, xNorm2 = 0;
  if (M.is_identity()) {
    rxd = k_dot<T>(c, n, x, d);
    if (dNorm2 == T(0)) dNorm2 = k_dot<T>(c, n, d, d);
    xNorm2 = k_dot<T>(c, n, x, x);
  } else {
    op_apply(c, M, x, z, ldiv);
    rxd = k_dot<T>(c, n, z, d);
    xNorm2 = k_dot<T>(c, n, z, x);
    op_apply(c, M, d, z, ldiv);
    dNorm2 = k_dot<T>(c, n, z, d);
  }
  if (dNorm2 == T(0)) return 2;
  const T radius2 = radius * radius;
  if (!(xNorm2 <= radius2)) return 3;
  if (roots_quadratic<T>(dNorm2, 2 * rxd, xNorm2 - radius2, 1, s1, s2)) return 4;
  return 0;
}

}  // namespace kb
