// fused_phases.cu -- fused iteration phases of every solver family with a fused path except CG (cg_fused.cu)
// (SURVEY.md section 8a phase structures).  Each phase is ONE launch: an SpMV or a streaming pass whose epilogue applies
// the adjacent axpy/axpby/scal updates and accumulates the dot products the next scalar needs; the CTA that finishes
// the grid reduction stores them, or the scalar derived from them, in the family's state struct on the device.  The
// phases of one iteration chain through that struct, and the host reads it back (StateBlock) to run the reference's
// stopping logic unchanged.
//
// Arithmetic is the reference's, operation by operation (non-contracted mul/add in the same order as the
// kaxpy!/kaxpby!/kscal! sequence it replaces), so these paths produce the same vectors as the primitive path given the
// same scalars; tests assert that equality.
#include "kb_internal.h"
#include "spmv_tiles.cuh"

namespace kb {

// ---------------------------------------------------------------------------
// generic launchers
// ---------------------------------------------------------------------------
template <class T, int K, class Epi, class Fin, class G>
__global__ void __launch_bounds__(kTileThreads, 3) spmv_epi_tma(Csr<T> A, G xg, Epi epi, Fin fin, T* part,
                                                             unsigned* ticket, DistComm* dc) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ T sm[32];
  T d[K];
#pragma unroll
  for (int k = 0; k < K; k++) d[k] = T(0);
  spmv_tiles_run<T>(
      A, smem, gather_for_cta(xg), NoRowBegin(), [&](int row, T acc, int) { epi(row, acc, d); });
  T mine[K], tot[K];
#pragma unroll
  for (int k = 0; k < K; k++) mine[k] = block_sum(d[k], sm);
  if (grid_sum_last<T, K>(mine, part, ticket, sm, tot) && threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < K; k++) tot[k] = dist_reduce(dc, tot[k]);     // row-partitioned: sum over ranks
    fin(tot);
  }
}

template <class T, int K, class Epi, class Fin, class G>
__global__ void __launch_bounds__(kBlock) spmv_epi_rows(Csr<T> A, G xg, Epi epi, Fin fin, T* part,
                                                        unsigned* ticket, DistComm* dc) {
  __shared__ T sm[32];
  T d[K];
#pragma unroll
  for (int k = 0; k < K; k++) d[k] = T(0);
  const G g = gather_for_cta(xg);
  const int stride = gridDim.x * blockDim.x;
  for (int row = blockIdx.x * blockDim.x + threadIdx.x; row < A.n; row += stride) {
    const int kb = A.rowptr[row], ke = A.rowptr[row + 1];
    T acc = T(0);
    for (int k = kb; k < ke; k++) acc = add_rn(acc, mul_rn(A.val[k], g(A.colind[k])));
    epi(row, acc, d);
  }
  T mine[K], tot[K];
#pragma unroll
  for (int k = 0; k < K; k++) mine[k] = block_sum(d[k], sm);
  if (grid_sum_last<T, K>(mine, part, ticket, sm, tot) && threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < K; k++) tot[k] = dist_reduce(dc, tot[k]);
    fin(tot);
  }
}

template <class T, int K, class Body, class Fin>
__global__ void __launch_bounds__(kBlock) stream_epi(int n, Body body, Fin fin, T* part, unsigned* ticket, DistComm* dc) {
  __shared__ T sm[32];
  T d[K > 0 ? K : 1];
#pragma unroll
  for (int k = 0; k < (K > 0 ? K : 1); k++) d[k] = T(0);
  const int stride = gridDim.x * blockDim.x;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + stride < n; i += 2 * stride) {      // two independent elements per trip
    body(i, d);
    body(i + stride, d);
  }
  if (i < n) body(i, d);
  if (K > 0) {
    T mine[K > 0 ? K : 1], tot[K > 0 ? K : 1];
#pragma unroll
    for (int k = 0; k < K; k++) mine[k] = block_sum(d[k], sm);
    if (grid_sum_last<T, (K > 0 ? K : 1)>(mine, part, ticket, sm, tot) && threadIdx.x == 0) {
#pragma unroll
      for (int k = 0; k < K; k++) tot[k] = dist_reduce(dc, tot[k]);
      fin(tot);
    }
  }
}

struct NoFin {
  template <class T> __device__ void operator()(const T*) const {}
};

template <class T, int K, class Epi, class Fin, class G>
static void launch_spmv_epi_g(Ctx& c, const Csr<T>& A, G xg, Epi epi, Fin fin) {
  unsigned* ticket = c.tickets + 4;       // the SpMV passes' grid reduction ticket (the streaming passes take 5)
  if (A.tma_ok) {
    ensure_dyn_smem((const void*)spmv_epi_tma<T, K, Epi, Fin, G>, 220 * 1024);
    int occ = 0;          // persistent grid = what is really co-resident (never more than one wave)
    KB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, spmv_epi_tma<T, K, Epi, Fin, G>, kTileThreads, A.smem_bytes));
    if (occ < 1) throw std::runtime_error("spmv_epi_tma does not fit on an SM with the planned shared-memory ring");
    const int grid = std::min(std::min(occ, A.ctas_per_sm) * sm_count(), std::max(1, A.ntiles));
    spmv_epi_tma<T, K, Epi, Fin, G><<<grid, kTileThreads, A.smem_bytes, c.stream>>>(A, xg, epi, fin, (T*)c.partials, ticket, c.dcomm);
  } else {
    spmv_epi_rows<T, K, Epi, Fin, G><<<stream_grid(A.n, 1, 8), kBlock, 0, c.stream>>>(A, xg, epi, fin, (T*)c.partials, ticket, c.dcomm);
  }
  KB_CUDA(cudaGetLastError());
  c.launches++;
}

template <class T, int K, class Epi, class Fin>
static void launch_spmv_epi(Ctx& c, const Csr<T>& A, const T* x, Epi epi, Fin fin) {
  if (A.n <= 0) return;
  if (c.dex) {                               // row-partitioned operator: exchange the halo of x, gather [local | halo]
    k_halo_exchange<T>(c, x);
    launch_spmv_epi_g<T, K, Epi, Fin, XGather<T>>(c, A, xgather_of<T>(c, x), epi, fin);
  } else {
    launch_spmv_epi_g<T, K, Epi, Fin, XPlain<T>>(c, A, XPlain<T>{x}, epi, fin);
  }
}

template <class T, int K, class Body, class Fin>
static void launch_stream(Ctx& c, int n, Body body, Fin fin) {
  if (n <= 0) return;
  stream_epi<T, K, Body, Fin><<<stream_grid(n, 2, 8), kBlock, 0, c.stream>>>(n, body, fin, (T*)c.partials, c.tickets + 5, c.dcomm);
  KB_CUDA(cudaGetLastError());
  c.launches++;
}

// Every scalar the host needs from a family's passes is written by their Fin into the family's state struct S<T>,
// which sits at the start of the workspace's device block (ws.fused_state), next to the values the passes carry from
// one launch to the next.  The pinned mirror (ws.fused_host) holds two copies of S<T>: slot 0 stages a seed, slot 1
// receives the read-back.  post() and wait() are apart because some passes are queued behind the copy and must stay
// queued before the host blocks.
template <template <class> class S, class T> struct StateBlock {
  typedef S<T> St;
  static_assert(2 * sizeof(St) <= kFusedBlockBytes, "the state struct and its two host slots must fit the block");
  Ctx& c;
  St* dev;
  St* host;
  size_t posted = 0;
  explicit StateBlock(Workspace<T>& ws) : c(ws.ctx), dev((St*)ws.fused_state), host((St*)ws.fused_host) {}
  void seed(const St& s) {                  // host slot 0 -> device
    host[0] = s;
    KB_CUDA(cudaMemcpyAsync(dev, host, sizeof(St), cudaMemcpyHostToDevice, c.stream));
  }
  void post(size_t bytes = sizeof(St)) {    // device -> host slot 1, queued on the stream
    KB_CUDA(cudaMemcpyAsync(host + 1, dev, bytes, cudaMemcpyDeviceToHost, c.stream));
    posted = bytes;
  }
  const St& wait() {                        // slot 1 once the stream has drained; every posted word passes the guard
    c.sync();
    const T* w = reinterpret_cast<const T*>(host + 1);
    for (size_t i = 0; i < posted / sizeof(T); i++) dist_nan_guard(c, (double)w[i]);
    return host[1];
  }
  const St& read() { post(); return wait(); }
};

// ===========================================================================
// BiCGSTAB  (src/bicgstab.jl:215-256, N = I, M = I or a diagonal applied by multiplication)
// ===========================================================================
template <class T> struct BicgState { T rho, alpha, omega, beta, next_rho, rNorm, cv, ts, tt, cr, rr; };

template <class T> struct BicgK1Epi {   // v = M (A p) ; <c, v>          (bicgstab.jl:221-223; m: diagonal of M or null)
  T* v; const T* c; const T* m;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    if (m) acc = mul_rn(__ldg(&m[row]), acc);
    v[row] = acc; d[0] += __ldg(&c[row]) * acc;
  }
};
template <class T> struct BicgK1Fin {   // alpha = rho / <c, v>          (bicgstab.jl:223)
  BicgState<T>* s;
  __device__ void operator()(const T* tot) const { s->cv = tot[0]; s->alpha = div_rn(s->rho, tot[0]); }
};
template <class T> struct BicgK2Body {  // s = r - alpha v               (bicgstab.jl:224-225)
  const T* r; const T* v; T* sv; const BicgState<T>* s;
  __device__ __forceinline__ void operator()(int i, T*) const { sv[i] = add_rn(r[i], mul_rn(-s->alpha, v[i])); }
};
template <class T> struct BicgK3Epi {   // t = M (A s) ; <t,s>, <t,t>     (bicgstab.jl:228-230)
  T* t; const T* sv; const T* m;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    if (m) acc = mul_rn(__ldg(&m[row]), acc);
    t[row] = acc; d[0] += acc * __ldg(&sv[row]); d[1] += acc * acc;
  }
};
template <class T> struct BicgK3Fin {   // omega = <t,s>/<t,t>           (bicgstab.jl:230)
  BicgState<T>* s;
  __device__ void operator()(const T* tot) const { s->ts = tot[0]; s->tt = tot[1]; s->omega = div_rn(tot[0], tot[1]); }
};
template <class T> struct BicgK4Body {  // x += alpha p ; x += omega s ; r = s - omega t ; <c,r>, <r,r>   (:226,231-234,240)
  T* x; const T* p; const T* sv; const T* t; const T* c; T* r; const BicgState<T>* s;
  __device__ __forceinline__ void operator()(int i, T* d) const {
    const T si = sv[i];
    x[i] = add_rn(add_rn(x[i], mul_rn(s->alpha, p[i])), mul_rn(s->omega, si));
    const T rn = add_rn(si, mul_rn(-s->omega, t[i]));
    r[i] = rn;
    d[0] += c[i] * rn;
    d[1] += rn * rn;
  }
};
template <class T> struct BicgK4Fin {   // next_rho, beta = (next_rho/rho)(alpha/omega), rNorm   (:234-235,240)
  BicgState<T>* s;
  __device__ void operator()(const T* tot) const {
    s->cr = tot[0]; s->rr = tot[1];
    s->next_rho = tot[0];
    s->beta = mul_rn(div_rn(tot[0], s->rho), div_rn(s->alpha, s->omega));
    s->rNorm = sqrt_rn(tot[1]);
    s->rho = tot[0];                       // loop top of the next iteration: rho = next_rho (:218)
  }
};
template <class T> struct BicgK5Body {  // p -= omega v ; p = r + beta p   (bicgstab.jl:236-237)
  T* p; const T* r; const T* v; const BicgState<T>* s;
  __device__ __forceinline__ void operator()(int i, T*) const {
    p[i] = add_rn(r[i], mul_rn(s->beta, add_rn(p[i], mul_rn(-s->omega, v[i]))));
  }
};

// One fused BiCGSTAB iteration.  In: next_rho of the previous iteration (host value, written to the device
// block at iteration 1 only).  Out (host): alpha, omega, next_rho, rNorm -- one read-back.
template <class T>
void bicgstab_fused_iteration(Workspace<T>& ws, const Csr<T>& A, const T* cvec, bool first, T rho_in, T* alpha, T* omega,
                              T* next_rho, T* rNorm) {
  Ctx& c = ws.ctx;
  const int n = ws.n;
  StateBlock<BicgState, T> sb(ws);
  BicgState<T>* S = sb.dev;
  if (first) {
    BicgState<T> s{};
    s.rho = rho_in;
    sb.seed(s);
  }
  const T* m = ws.mdiag_fused;          // left diagonal preconditioner fused into the two SpMV epilogues
  T* t = m ? ws.t : ws.qd;              // t == d == qd when M = I  (bicgstab.jl:153-154)
  launch_spmv_epi<T, 1>(c, A, ws.p, BicgK1Epi<T>{ws.v, cvec, m}, BicgK1Fin<T>{S});
  launch_stream<T, 0>(c, n, BicgK2Body<T>{ws.r, ws.v, ws.s, S}, NoFin());
  launch_spmv_epi<T, 2>(c, A, ws.s, BicgK3Epi<T>{t, ws.s, m}, BicgK3Fin<T>{S});
  launch_stream<T, 2>(c, n, BicgK4Body<T>{ws.x, ws.p, ws.s, t, cvec, ws.r, S}, BicgK4Fin<T>{S});
  sb.post();                            // scalars of this iteration
  launch_stream<T, 0>(c, n, BicgK5Body<T>{ws.p, ws.r, ws.v, S}, NoFin());
  const BicgState<T>& h = sb.wait();
  *alpha = h.alpha; *omega = h.omega; *next_rho = h.next_rho; *rNorm = h.rNorm;
}

// ===========================================================================
// MINRES  (src/minres.jl:285-333,389-409, M = I or a diagonal applied by multiplication)
// ===========================================================================
template <class T> struct MinresState { T vy, alpha, beta2, xx; };

template <class T> struct MinresK1Epi {  // y = (A v [+ lambda v]) / beta [- (beta/oldbeta) r1] ; <v, y>   (:289-294)
  T* y; const T* v; const T* r1; T lambda, inv_beta, c1; int iter;     // v == r2 when M = I, else v = M r2
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    const T vr = __ldg(&v[row]);
    T t = acc;
    if (lambda != T(0)) t = add_rn(t, mul_rn(lambda, vr));
    t = mul_rn(inv_beta, t);
    if (iter >= 2) t = add_rn(t, mul_rn(c1, __ldg(&r1[row])));
    y[row] = t;
    d[0] += vr * t;
  }
};
template <class T> struct MinresK1Fin {  // alpha = <v,y> / beta
  MinresState<T>* s; T beta;
  __device__ void operator()(const T* tot) const { s->vy = tot[0]; s->alpha = div_rn(tot[0], beta); }
};
template <class T> struct MinresK2Body { // y -= (alpha/beta) r2 ; w update (:295-307) ; v = M y ; <y,v> (:311-313, r2 <- y)
  T* y; const T* r2; T* w; const T* w2; const MinresState<T>* s;
  T beta, inv_beta, cs, sn, deltabar, eps; int iter;
  T* v; const T* m;                                         // M = I: v == nullptr (v aliases r2)
  __device__ __forceinline__ void operator()(int i, T* d) const {
    const T alpha = s->alpha;
    const T r2i = r2[i];
    const T vi = m ? v[i] : r2i;                            // v_k, value BEFORE v <- M y
    const T yn = add_rn(y[i], mul_rn(div_rn(-alpha, beta), r2i));
    y[i] = yn;
    if (m) {
      const T vn = mul_rn(m[i], yn);                        // v_{k+1} = M r2_{k+1}
      v[i] = vn;
      d[0] += yn * vn;
    } else {
      d[0] += yn * yn;
    }
    if (iter == 1) {
      w[i] = div_rn(vi, beta);                              // kdivcopy!(n, w, v, beta), w == w2
    } else {
      const T delta = add_rn(mul_rn(cs, deltabar), mul_rn(sn, alpha));
      T wv = w[i];                                          // w == w1
      if (iter >= 3) wv = mul_rn(-eps, wv);
      wv = add_rn(wv, mul_rn(-delta, w2[i]));
      wv = add_rn(wv, mul_rn(inv_beta, vi));
      w[i] = wv;
    }
  }
};
template <class T> struct MinresK2Fin {
  MinresState<T>* s;
  __device__ void operator()(const T* tot) const { s->beta2 = tot[0]; }
};
template <class T> struct MinresK3Body { // w /= gamma ; x += phi w ; <x,x>   (:333,389,409)
  T* w; T* x; T inv_gamma, phi;
  __device__ __forceinline__ void operator()(int i, T* d) const {
    const T wv = mul_rn(inv_gamma, w[i]);
    w[i] = wv;
    const T xn = add_rn(x[i], mul_rn(phi, wv));
    x[i] = xn;
    d[0] += xn * xn;
  }
};
template <class T> struct MinresK3Fin {
  MinresState<T>* s;
  __device__ void operator()(const T* tot) const { s->xx = tot[0]; }
};

// Phase A of a fused MINRES iteration: Lanczos step.  Rotates r1/r2/y by pointer (the reference copies).
// Returns alpha and beta_new^2 = <r2,r2>.
template <class T>
void minres_fused_lanczos(Workspace<T>& ws, const Csr<T>& A, int iter, T lambda, T beta, T oldbeta, T cs, T sn, T deltabar,
                          T eps_rot, T* w, T* alpha, T* beta2) {
  Ctx& c = ws.ctx;
  const int n = ws.n;
  StateBlock<MinresState, T> sb(ws);
  MinresState<T>* S = sb.dev;
  const T inv_beta = T(1) / beta;
  const T c1 = iter >= 2 ? -beta / oldbeta : T(0);
  const T* m = ws.mdiag_fused;
  T* v = m ? ws.vv : ws.r2;                                 // minres.jl:193
  launch_spmv_epi<T, 1>(c, A, v, MinresK1Epi<T>{ws.y, v, ws.r1, lambda, inv_beta, c1, iter}, MinresK1Fin<T>{S, beta});
  launch_stream<T, 1>(c, n, MinresK2Body<T>{ws.y, ws.r2, w, ws.w2, S, beta, inv_beta, cs, sn, deltabar, eps_rot, iter,
                                            m ? ws.vv : nullptr, m},
                      MinresK2Fin<T>{S});
  const MinresState<T>& h = sb.read();
  *alpha = h.alpha; *beta2 = h.beta2;
  T* old_r1 = ws.r1;          // r1 <- r2 ; r2 <- y   (minres.jl:309-310) by rotating the bindings
  ws.r1 = ws.r2; ws.r2 = ws.y; ws.y = old_r1;
}

// Phase B: w /= gamma ; x += phi w ; returns ||x||.
template <class T>
T minres_fused_update(Workspace<T>& ws, T* w, T gamma, T phi) {
  StateBlock<MinresState, T> sb(ws);
  launch_stream<T, 1>(ws.ctx, ws.n, MinresK3Body<T>{w, ws.x, T(1) / gamma, phi}, MinresK3Fin<T>{sb.dev});
  return std::sqrt(sb.read().xx);
}

// ===========================================================================
// GMRES  (src/gmres.jl:255-262,274, N = I, M = I or a diagonal applied by multiplication, no reorthogonalization)
// ===========================================================================
constexpr int kGmresMaxFused = 120;    // h[] slots in the state block
template <class T> struct GmresState { T hbis2; T h[kGmresMaxFused]; };

template <class T> struct GmresSpmvEpi {  // q = M (A v_k) ; h_1 = <v_1, q>   (gmres.jl:256-260; m: diagonal of M or null)
  T* w; const T* v1; const T* m;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    if (m) acc = mul_rn(__ldg(&m[row]), acc);
    w[row] = acc; d[0] += __ldg(&v1[row]) * acc;
  }
};
template <class T> struct GmresHFin {
  GmresState<T>* s; int slot;            // slot < 0: ||q||^2
  __device__ void operator()(const T* tot) const { if (slot >= 0) s->h[slot] = tot[0]; else s->hbis2 = tot[0]; }
};
template <class T> struct GmresMgsBody {  // q -= h_i v_i ; then <v_{i+1}, q> or <q, q>   (gmres.jl:259-262,274)
  T* q; const T* vi; const T* vnext; const GmresState<T>* s; int i;
  __device__ __forceinline__ void operator()(int j, T* d) const {
    const T qn = add_rn(q[j], mul_rn(-s->h[i], vi[j]));
    q[j] = qn;
    d[0] += (vnext ? vnext[j] : qn) * qn;
  }
};

// q = M (A xin), modified Gram-Schmidt of q against vecs[0..cnt-1] IN THAT ORDER, one launch per vector with the next
// dot product (or ||q||^2 after the last one) accumulated in the same pass; returns h[0..cnt-1] and ||q||.
// gmres! / fom! / fgmres! pass V[1..k]; dqgmres! / diom! the live window of their circular stack.
template <class T>
void fused_orth_chain(Workspace<T>& ws, const Csr<T>& A, const T* xin, T* q, const T* const* vecs, int cnt, T* h_out, T* Hbis) {
  Ctx& c = ws.ctx;
  const int n = ws.n;
  StateBlock<GmresState, T> sb(ws);
  GmresState<T>* S = sb.dev;
  const T* m = ws.mdiag_fused;
  launch_spmv_epi<T, 1>(c, A, xin, GmresSpmvEpi<T>{q, vecs[0], m}, GmresHFin<T>{S, 0});
  for (int i = 0; i < cnt; i++) {
    const T* vnext = (i + 1 < cnt) ? vecs[i + 1] : nullptr;
    launch_stream<T, 1>(c, n, GmresMgsBody<T>{q, vecs[i], vnext, S, i}, GmresHFin<T>{S, (i + 1 < cnt) ? i + 1 : -1});
  }
  sb.post(sizeof(T) * (size_t)(cnt + 1));                   // hbis2 and h[0..cnt-1]
  const GmresState<T>& h = sb.wait();
  for (int i = 0; i < cnt; i++) h_out[i] = h.h[i];
  *Hbis = std::sqrt(h.hbis2);
}

// Arnoldi step k (1-based inner_iter): w = A V[k]; MGS against V[1..k]; returns h[0..k-1] and Hbis.
template <class T>
void gmres_fused_arnoldi(Workspace<T>& ws, const Csr<T>& A, int k, T* h_out, T* Hbis, const T* xin) {
  T* q = ws.mdiag_fused ? ws.q : ws.w;                      // q == w when M = I (gmres.jl:150)
  fused_orth_chain<T>(ws, A, xin ? xin : ws.V[k - 1], q, ws.V.data(), k, h_out, Hbis);
}

// xr += sum_i y_i V[i], accumulated in index order in one pass (gmres.jl:348-350)
template <class T, int NV> struct MultiAxpyBody {
  T* xr; const T* v[NV]; T y[NV]; int cnt;
  __device__ __forceinline__ void operator()(int j, T*) const {
    T acc = xr[j];
#pragma unroll
    for (int i = 0; i < NV; i++) if (i < cnt) acc = add_rn(acc, mul_rn(y[i], v[i][j]));
    xr[j] = acc;
  }
};
template <class T>
void fused_multi_axpy(Workspace<T>& ws, T* xr, int k, const T* y, T* const* vecs) {
  constexpr int NV = 8;
  for (int base = 0; base < k; base += NV) {
    MultiAxpyBody<T, NV> body;
    body.xr = xr; body.cnt = std::min(NV, k - base);
    for (int i = 0; i < NV; i++) { body.v[i] = vecs[std::min(base + i, k - 1)]; body.y[i] = (base + i < k) ? y[base + i] : T(0); }
    launch_stream<T, 0>(ws.ctx, ws.n, body, NoFin());
  }
}

// ===========================================================================
// Sibling solvers (SURVEY.md 8f-3), M = N = I, CSR operator: the vector operations of one iteration are grouped into
// the fewest passes the data dependencies allow.  The scalars stay on the HOST (these loops run the reference's
// control flow unchanged and read each group of dot products back once), so unlike the four path solvers nothing
// chains through device memory; what is saved is launches, vector passes and read-backs:
//   dqgmres! / diom!  2 k + 6 launches, 2 k + 2 read-backs per iteration  ->  k + 3 launches, 1 read-back (k = window)
//   cgs!              12 launches, 3 read-backs                           ->  4 launches, 2 read-backs
//   cg_lanczos!        8 launches, 2 read-backs                           ->  3 launches, 2 read-backs
//   cr!                9 launches, 5 read-backs                           ->  3 launches, 2 read-backs
// Every element update repeats the k* sequence it replaces operation by operation (non-contracted), so vectors are
// bit-identical to the primitive path given the same scalars.
// ===========================================================================
// ---- dqgmres! / diom!: direction update (dqgmres.jl:279-289, diom.jl:279-289) in one pass per 8 stack vectors ----
//   for every live i: P[ppos] = -H_i P[ppos] (same slot) or P[ppos] -= H_i P[ipos];  then P[ppos] += z; P[ppos] /= H_1;
//   x += step P[ppos]
template <class T, int NV> struct TruncPBody {
  T* pp; const T* pv[NV]; T coef[NV]; int same[NV]; int cnt; int last; const T* z; T inv_h0; T step; T* x;
  __device__ __forceinline__ void operator()(int j, T*) const {
    T acc = pp[j];
#pragma unroll
    for (int i = 0; i < NV; i++)
      if (i < cnt) acc = same[i] ? mul_rn(coef[i], acc) : add_rn(acc, mul_rn(coef[i], pv[i][j]));
    if (last) {
      acc = add_rn(acc, z[j]);                    // kaxpy!(n, one, z, p)
      acc = mul_rn(inv_h0, acc);                  // kdiv!(n, p, H[1]) = kscal!(n, 1 / H[1], p)
      x[j] = add_rn(x[j], mul_rn(step, acc));
    }
    pp[j] = acc;
  }
};
template <class T>
void trunc_fused_direction(Workspace<T>& ws, T* pp, int cnt, T* const* pvecs, const T* coefs, const T* z, T h0, T step) {
  constexpr int NV = 8;
  int base = 0;
  do {
    TruncPBody<T, NV> body;
    body.pp = pp; body.cnt = std::max(0, std::min(NV, cnt - base)); body.z = z; body.inv_h0 = T(1) / h0; body.step = step; body.x = ws.x;
    body.last = (base + NV >= cnt) ? 1 : 0;
    for (int i = 0; i < NV; i++) {
      const int k = std::min(base + i, std::max(cnt - 1, 0));
      body.pv[i] = cnt > 0 ? pvecs[k] : pp; body.coef[i] = (cnt > 0 && base + i < cnt) ? coefs[base + i] : T(0);
      body.same[i] = (cnt > 0 && pvecs[k] == pp) ? 1 : 0;
    }
    launch_stream<T, 0>(ws.ctx, ws.n, body, NoFin());
    base += NV;
  } while (base < cnt);
}

// ---- cgs! (src/cgs.jl:196-239) ----
template <class T> struct CgsState { T sigma, rho_next, rr; };

template <class T> struct CgsK1Epi {               // t = A p ; sigma = <c, t>
  T* t; const T* cv;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const { t[row] = acc; d[0] += __ldg(&cv[row]) * acc; }
};
template <class T> struct CgsK2Body {              // q = u - alpha v ; u += q ; x += alpha u
  T* q; T* u; const T* v; T* x; T alpha;
  __device__ __forceinline__ void operator()(int j, T*) const {
    const T qn = add_rn(u[j], mul_rn(-alpha, v[j]));
    q[j] = qn;
    const T un = add_rn(u[j], qn);
    u[j] = un;
    x[j] = add_rn(x[j], mul_rn(alpha, un));
  }
};
template <class T> struct CgsK3Epi {               // s = A u ; r -= alpha s ; <c, r>, <r, r>
  T* s; T* r; const T* cv; T alpha;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    s[row] = acc;
    const T rn = add_rn(r[row], mul_rn(-alpha, acc));
    r[row] = rn;
    d[0] += __ldg(&cv[row]) * rn; d[1] += rn * rn;
  }
};
template <class T> struct CgsK1Fin { CgsState<T>* s; __device__ void operator()(const T* tot) const { s->sigma = tot[0]; } };
template <class T> struct CgsK3Fin { CgsState<T>* s; __device__ void operator()(const T* tot) const { s->rho_next = tot[0]; s->rr = tot[1]; } };
template <class T> struct CgsK4Body {              // u = r + beta q ; p = u + beta (q + beta p)
  T* u; T* p; const T* r; const T* q; T beta;
  __device__ __forceinline__ void operator()(int j, T*) const {
    const T un = add_rn(r[j], mul_rn(beta, q[j]));
    u[j] = un;
    const T p1 = add_rn(q[j], mul_rn(beta, p[j]));
    p[j] = add_rn(un, mul_rn(beta, p1));
  }
};
template <class T> T cgs_fused_sigma(Workspace<T>& ws, const Csr<T>& A, const T* cvec) {
  StateBlock<CgsState, T> sb(ws);
  launch_spmv_epi<T, 1>(ws.ctx, A, ws.p, CgsK1Epi<T>{ws.ts, cvec}, CgsK1Fin<T>{sb.dev});
  return sb.read().sigma;
}
template <class T> void cgs_fused_update(Workspace<T>& ws, const Csr<T>& A, const T* cvec, T alpha, T* rho_next, T* rr) {
  Ctx& c = ws.ctx;
  StateBlock<CgsState, T> sb(ws);
  launch_stream<T, 0>(c, ws.n, CgsK2Body<T>{ws.q, ws.u, ws.ts, ws.x, alpha}, NoFin());
  launch_spmv_epi<T, 2>(c, A, ws.u, CgsK3Epi<T>{ws.ts, ws.r, cvec, alpha}, CgsK3Fin<T>{sb.dev});
  const CgsState<T>& h = sb.read();
  *rho_next = h.rho_next; *rr = h.rr;
}
template <class T> void cgs_fused_directions(Workspace<T>& ws, T beta) {
  launch_stream<T, 0>(ws.ctx, ws.n, CgsK4Body<T>{ws.u, ws.p, ws.r, ws.q, beta}, NoFin());
}

// ---- cg_lanczos! (src/cg_lanczos.jl:186-216), M = I so v === Mv ----
template <class T> struct LanState { T delta, mm; };

template <class T> struct LanK1Epi {               // Mv_next = A v ; delta = <v, Mv_next>
  T* mvn; const T* v;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const { mvn[row] = acc; d[0] += __ldg(&v[row]) * acc; }
};
template <class T> struct LanK2Body {              // Mv_next -= delta Mv (- beta Mv_prev) ; Mv_prev = Mv ; Mv = Mv_next ; ||Mv||^2
  T* mvn; T* mv; T* mvp; T delta; T beta; int later;
  __device__ __forceinline__ void operator()(int j, T* d) const {
    T m = add_rn(mvn[j], mul_rn(-delta, mv[j]));
    if (later) { m = add_rn(m, mul_rn(-beta, mvp[j])); mvp[j] = mv[j]; }
    mvn[j] = m; mv[j] = m;
    d[0] += m * m;
  }
};
template <class T> struct LanK1Fin { LanState<T>* s; __device__ void operator()(const T* tot) const { s->delta = tot[0]; } };
template <class T> struct LanK2Fin { LanState<T>* s; __device__ void operator()(const T* tot) const { s->mm = tot[0]; } };
template <class T> struct LanK3Body {              // v /= beta ; x += gamma p ; p = sigma v + omega p
  T* v; T* x; T* p; T inv_beta; T gamma; T sigma; T omega;
  __device__ __forceinline__ void operator()(int j, T*) const {
    const T vn = mul_rn(inv_beta, v[j]);
    v[j] = vn;
    x[j] = add_rn(x[j], mul_rn(gamma, p[j]));
    p[j] = add_rn(mul_rn(sigma, vn), mul_rn(omega, p[j]));
  }
};
template <class T> T lanczos_fused_delta(Workspace<T>& ws, const Csr<T>& A) {
  StateBlock<LanState, T> sb(ws);
  launch_spmv_epi<T, 1>(ws.ctx, A, ws.Mv, LanK1Epi<T>{ws.Mv_next, ws.Mv}, LanK1Fin<T>{sb.dev});
  return sb.read().delta;
}
template <class T> T lanczos_fused_recur(Workspace<T>& ws, T delta, T beta, bool later) {
  StateBlock<LanState, T> sb(ws);
  launch_stream<T, 1>(ws.ctx, ws.n, LanK2Body<T>{ws.Mv_next, ws.Mv, ws.Mv_prev, delta, beta, later ? 1 : 0}, LanK2Fin<T>{sb.dev});
  return std::sqrt(sb.read().mm);
}
template <class T> void lanczos_fused_update(Workspace<T>& ws, T beta, T gamma, T sigma, T omega) {
  launch_stream<T, 0>(ws.ctx, ws.n, LanK3Body<T>{ws.Mv, ws.x, ws.p, T(1) / beta, gamma, sigma, omega}, NoFin());
}

// ---- cr! (src/cr.jl:375-445), M = I, no trust region, no linesearch ----
template <class T> struct CrState { T xx, rr, ArAr, rAr, qq; };

template <class T> struct CrK1Body {               // x += alpha p ; r -= alpha q ; ||x||^2, ||r||^2
  T* x; T* r; const T* p; const T* q; T alpha;
  __device__ __forceinline__ void operator()(int j, T* d) const {
    const T xn = add_rn(x[j], mul_rn(alpha, p[j]));
    x[j] = xn;
    const T rn = add_rn(r[j], mul_rn(-alpha, q[j]));
    r[j] = rn;
    d[0] += xn * xn; d[1] += rn * rn;
  }
};
template <class T> struct CrK2Epi {                // Ar = A r ; ||Ar||^2, <r, Ar>
  T* Ar; const T* r;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const { Ar[row] = acc; d[0] += acc * acc; d[1] += __ldg(&r[row]) * acc; }
};
template <class T> struct CrK3Body {               // p = r + beta p ; q = Ar + beta q ; ||q||^2 (the next alpha's denominator)
  T* p; T* q; const T* r; const T* Ar; T beta;
  __device__ __forceinline__ void operator()(int j, T* d) const {
    p[j] = add_rn(r[j], mul_rn(beta, p[j]));
    const T qn = add_rn(Ar[j], mul_rn(beta, q[j]));
    q[j] = qn;
    d[0] += qn * qn;
  }
};
template <class T> struct CrK1Fin { CrState<T>* s; __device__ void operator()(const T* tot) const { s->xx = tot[0]; s->rr = tot[1]; } };
template <class T> struct CrK2Fin { CrState<T>* s; __device__ void operator()(const T* tot) const { s->ArAr = tot[0]; s->rAr = tot[1]; } };
template <class T> struct CrK3Fin { CrState<T>* s; __device__ void operator()(const T* tot) const { s->qq = tot[0]; } };
template <class T> void cr_fused_step(Workspace<T>& ws, const Csr<T>& A, T alpha, T* xx, T* rr, T* ArAr, T* rAr) {
  Ctx& c = ws.ctx;
  StateBlock<CrState, T> sb(ws);
  launch_stream<T, 2>(c, ws.n, CrK1Body<T>{ws.x, ws.r, ws.p, ws.q, alpha}, CrK1Fin<T>{sb.dev});
  launch_spmv_epi<T, 2>(c, A, ws.r, CrK2Epi<T>{ws.Ap, ws.r}, CrK2Fin<T>{sb.dev});
  const CrState<T>& h = sb.read();
  *xx = h.xx; *rr = h.rr; *ArAr = h.ArAr; *rAr = h.rAr;
}
template <class T> T cr_fused_directions(Workspace<T>& ws, T beta) {
  StateBlock<CrState, T> sb(ws);
  launch_stream<T, 1>(ws.ctx, ws.n, CrK3Body<T>{ws.p, ws.q, ws.r, ws.Ap, beta}, CrK3Fin<T>{sb.dev});
  return sb.read().qq;
}

// ===========================================================================
// LSQR / LSMR  (src/lsqr.jl:297-317,361-362, src/lsmr.jl:309-328,352-365, M = N = I, no trust region)
// kdiv!(u, beta) = kscal!(1/beta, u) is left pending: Mu stays unscaled in memory and both of its readers apply
// s_u = 1/beta (the scaled gather of P2 and the Mu read of the next P1), which are the two roundings the reference
// performs.  v === Nv is scaled in place by P3, as kdiv!(v, alpha) does.
// ===========================================================================
template <class T> struct LsqState { T alpha, beta, s_u, ww, xx; };   // alpha, s_u: carried from one pass to the next

template <class T> struct LsqP1Epi {      // Mu = A v - alpha (Mu s_u) ; ||Mu||^2   (kaxpby!(m, one, Av, -alpha, Mu))
  T* mu; const LsqState<T>* s;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    const T u = mul_rn(mu[row], s->s_u);
    const T nm = add_rn(mul_rn(T(1), acc), mul_rn(-s->alpha, u));
    mu[row] = nm;
    d[0] += nm * nm;
  }
};
template <class T> struct LsqP1Fin {      // beta = ||Mu|| ; s_u = 1/beta (1 when beta = 0: kdiv! is skipped)
  LsqState<T>* s;
  __device__ void operator()(const T* tot) const {
    const T beta = sqrt_rn(tot[0]);
    s->beta = beta;
    s->s_u = beta == T(0) ? T(1) : div_rn(T(1), beta);
  }
};
template <class T, bool WW> struct LsqP2Epi {   // Nv = A^T u - beta Nv ; ||Nv||^2 ; LSQR: <w, w> of the old w
  T* nv; const T* w; const LsqState<T>* s;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    if (WW) { const T wr = w[row]; d[1] += wr * wr; }
    if (s->beta == T(0)) return;                  // beta = 0: the reference skips this product (lsqr.jl:303)
    const T nn = add_rn(mul_rn(T(1), acc), mul_rn(-s->beta, nv[row]));
    nv[row] = nn;
    d[0] += nn * nn;
  }
};
template <class T, int K> struct LsqP2Fin {
  LsqState<T>* s;
  __device__ void operator()(const T* tot) const {
    if (K > 1) s->ww = tot[K - 1];
    if (s->beta != T(0)) s->alpha = sqrt_rn(tot[0]);
  }
};
template <class T> struct LsqrP3Body {    // v = Nv / alpha ; x += sigma w ; w = v - tau w   (lsqr.jl:315,361-362)
  T* v; T* x; T* w; T inv_alpha, sigma, tau; int scale_v;
  __device__ __forceinline__ void operator()(int i, T*) const {
    T vi = v[i];
    if (scale_v) { vi = mul_rn(inv_alpha, vi); v[i] = vi; }
    const T wi = w[i];
    x[i] = add_rn(x[i], mul_rn(sigma, wi));
    w[i] = add_rn(mul_rn(T(1), vi), mul_rn(-tau, wi));
  }
};
template <class T> struct LsmrP3Body {    // v = Nv / alpha ; hbar = h - delta hbar ; x += sigma hbar ; h = v - tau h ; ||x||^2
  T* v; T* x; T* h; T* hbar; T inv_alpha, sigma, tau, delta; int scale_v;   // (lsmr.jl:325,352,364-365,399)
  __device__ __forceinline__ void operator()(int i, T* d) const {
    T vi = v[i];
    if (scale_v) { vi = mul_rn(inv_alpha, vi); v[i] = vi; }
    const T hi = h[i];
    const T hb = add_rn(mul_rn(T(1), hi), mul_rn(-delta, hbar[i]));
    hbar[i] = hb;
    const T xn = add_rn(x[i], mul_rn(sigma, hb));
    x[i] = xn;
    h[i] = add_rn(mul_rn(T(1), vi), mul_rn(-tau, hi));
    d[0] += xn * xn;
  }
};
template <class T> struct LsmrP3Fin { LsqState<T>* s; __device__ void operator()(const T* tot) const { s->xx = tot[0]; } };

template <class T>
void lsq_fused_bidiag(Workspace<T>& ws, const Csr<T>& A, const Csr<T>& At, bool init, T alpha, bool want_ww, T* beta, T* alpha_out,
                      T* ww) {
  Ctx& c = ws.ctx;
  StateBlock<LsqState, T> sb(ws);
  LsqState<T>* S = sb.dev;
  if (init) {                     // Mu holds u_1 already scaled (the initialisation runs on the primitives)
    LsqState<T> s{};
    s.alpha = alpha; s.s_u = T(1);
    sb.seed(s);
  }
  launch_spmv_epi_g<T, 1>(c, A, XPlain<T>{ws.Nv}, LsqP1Epi<T>{ws.Mu, S}, LsqP1Fin<T>{S});
  const XScaled<T> ug{ws.Mu, &S->s_u, T(1)};
  if (want_ww) launch_spmv_epi_g<T, 2>(c, At, ug, LsqP2Epi<T, true>{ws.Nv, ws.w, S}, LsqP2Fin<T, 2>{S});
  else launch_spmv_epi_g<T, 1>(c, At, ug, LsqP2Epi<T, false>{ws.Nv, ws.w, S}, LsqP2Fin<T, 1>{S});
  const LsqState<T>& h = sb.read();
  *beta = h.beta; *alpha_out = h.alpha; *ww = h.ww;
}

template <class T> T lsq_fused_update(Workspace<T>& ws, bool lsmr, bool scale_v, T inv_alpha, T sigma, T tau, T delta) {
  Ctx& c = ws.ctx;
  if (!lsmr) {
    launch_stream<T, 0>(c, ws.n, LsqrP3Body<T>{ws.Nv, ws.x, ws.w, inv_alpha, sigma, tau, scale_v ? 1 : 0}, NoFin());
    return T(0);
  }
  StateBlock<LsqState, T> sb(ws);
  launch_stream<T, 1>(c, ws.n, LsmrP3Body<T>{ws.Nv, ws.x, ws.h, ws.hbar, inv_alpha, sigma, tau, delta, scale_v ? 1 : 0},
                      LsmrP3Fin<T>{sb.dev});
  return std::sqrt(sb.read().xx);
}

// LSLQ (src/lslq.jl:302-320,411-416): after LSQR's P1 / P2 (want_ww = false), one pass over n:
//   v = Nv / alpha ; x += (c zeta) w̄ ; x += (s zeta) v ; w̄ = -c v + s w̄
template <class T> struct LslqUpdateBody {
  T* v; T* x; T* wbar; T inv_alpha, czeta, szeta, c, s; int scale_v;
  __device__ __forceinline__ void operator()(int i, T*) const {
    T vi = v[i];
    if (scale_v) { vi = mul_rn(inv_alpha, vi); v[i] = vi; }
    const T wi = wbar[i];
    x[i] = add_rn(add_rn(x[i], mul_rn(czeta, wi)), mul_rn(szeta, vi));
    wbar[i] = add_rn(mul_rn(-c, vi), mul_rn(s, wi));
  }
};
template <class T> void lslq_fused_update(Workspace<T>& ws, bool scale_v, T inv_alpha, T czeta, T szeta, T c, T s) {
  launch_stream<T, 0>(ws.ctx, ws.n, LslqUpdateBody<T>{ws.Nv, ws.x, ws.w, inv_alpha, czeta, szeta, c, s, scale_v ? 1 : 0},
                      NoFin());
}

// ===========================================================================
// CGLS  (src/cgls.jl:192-219, M = I, no trust region)
// The scalars chain through the device block: K1's Fin derives alpha, K3's Fin gamma and beta, K4's Fin <p, p> (the
// next delta's lambda term).  The host reads {<r, r>, gamma} once, after K3; K4 is already queued behind the copy.
// ===========================================================================
template <class T> struct CglsState { T gamma, alpha, beta, pp, rr; };

template <class T> struct CglsK1Epi {     // q = A p ; <q, q>                       (cgls.jl:193,195)
  T* q;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const { q[row] = acc; d[0] += acc * acc; }
};
template <class T> struct CglsK1Fin {     // delta (+ lambda <p, p>) ; alpha = gamma / delta   (cgls.jl:195-197)
  CglsState<T>* s; T lambda;
  __device__ void operator()(const T* tot) const {
    T delta = tot[0];
    if (lambda > T(0)) delta = add_rn(delta, mul_rn(lambda, s->pp));
    s->alpha = div_rn(s->gamma, delta);
  }
};
template <class T> struct CglsK2Body {    // r -= alpha q ; <r, r>                  (cgls.jl:207,215)
  T* r; const T* q; const CglsState<T>* s;
  __device__ __forceinline__ void operator()(int i, T* d) const {
    const T rn = add_rn(r[i], mul_rn(-s->alpha, q[i]));
    r[i] = rn;
    d[0] += rn * rn;
  }
};
template <class T> struct CglsK2Fin {
  CglsState<T>* s;
  __device__ void operator()(const T* tot) const { s->rr = tot[0]; }
};
template <class T> struct CglsK3Epi {     // x += alpha p ; s = A^T r (- lambda x) ; <s, s>   (cgls.jl:206,209-211)
  T* x; const T* p; T* sv; const CglsState<T>* s; T lambda;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    const T xn = add_rn(x[row], mul_rn(s->alpha, p[row]));
    x[row] = xn;
    T sn = acc;
    if (lambda > T(0)) sn = add_rn(sn, mul_rn(-lambda, xn));
    sv[row] = sn;
    d[0] += sn * sn;
  }
};
template <class T> struct CglsK3Fin {     // beta = gamma_next / gamma ; gamma = gamma_next   (cgls.jl:212,214)
  CglsState<T>* s;
  __device__ void operator()(const T* tot) const { s->beta = div_rn(tot[0], s->gamma); s->gamma = tot[0]; }
};
template <class T> struct CglsK4Body {    // p = s + beta p ; <p, p>                (cgls.jl:213)
  T* p; const T* sv; const CglsState<T>* s;
  __device__ __forceinline__ void operator()(int i, T* d) const {
    const T pn = add_rn(mul_rn(T(1), sv[i]), mul_rn(s->beta, p[i]));
    p[i] = pn;
    d[0] += pn * pn;
  }
};
template <class T> struct CglsK4Fin {
  CglsState<T>* s;
  __device__ void operator()(const T* tot) const { s->pp = tot[0]; }
};

template <class T>
void cgls_fused_iteration(Workspace<T>& ws, const Csr<T>& A, const Csr<T>& At, bool init, T gamma, T lambda, T* rr, T* gamma_out) {
  Ctx& c = ws.ctx;
  StateBlock<CglsState, T> sb(ws);
  CglsState<T>* S = sb.dev;
  if (init) {                     // p = s, so <p, p> is the gamma the host computed
    CglsState<T> s{};
    s.gamma = gamma; s.pp = gamma;
    sb.seed(s);
  }
  launch_spmv_epi_g<T, 1>(c, A, XPlain<T>{ws.p}, CglsK1Epi<T>{ws.q}, CglsK1Fin<T>{S, lambda});
  launch_stream<T, 1>(c, ws.m, CglsK2Body<T>{ws.r, ws.q, S}, CglsK2Fin<T>{S});
  launch_spmv_epi_g<T, 1>(c, At, XPlain<T>{ws.r}, CglsK3Epi<T>{ws.x, ws.p, ws.s, S, lambda}, CglsK3Fin<T>{S});
  sb.post();
  launch_stream<T, 1>(c, ws.n, CglsK4Body<T>{ws.p, ws.s, S}, CglsK4Fin<T>{S});
  const CglsState<T>& h = sb.wait();
  *rr = h.rr; *gamma_out = h.gamma;
}

// ===========================================================================
// CRLS  (src/crls.jl:194-240, M = I, no trust region)
// L4's Fin derives the next alpha, L2's Fin gamma and beta; the host reads {<Ar, Ar>, <x, x>, <r, r>, gamma} once,
// after L2; L3 and L4 are already queued behind the copy.
// ===========================================================================
template <class T> struct CrlsState { T gamma, alpha, beta, ArAr, xx, rr; };

template <class T> struct CrlsL1Body {    // x += alpha p ; Ar -= alpha q ; <Ar, Ar>, <x, x>   (crls.jl:217-219,237)
  T* x; T* Ar; const T* p; const T* q; const CrlsState<T>* s;
  __device__ __forceinline__ void operator()(int j, T* d) const {
    const T alpha = s->alpha;
    const T xn = add_rn(x[j], mul_rn(alpha, p[j]));
    x[j] = xn;
    const T an = add_rn(Ar[j], mul_rn(-alpha, q[j]));
    Ar[j] = an;
    d[0] += an * an; d[1] += xn * xn;
  }
};
template <class T> struct CrlsL1Fin {
  CrlsState<T>* s;
  __device__ void operator()(const T* tot) const { s->ArAr = tot[0]; s->xx = tot[1]; }
};
template <class T> struct CrlsL2Epi {     // r -= alpha Ap ; s = A Ar ; <s, s>, <r, r>   (crls.jl:222-225)
  T* r; const T* Ap; T* sv; const CrlsState<T>* s;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    const T rn = add_rn(r[row], mul_rn(-s->alpha, Ap[row]));
    r[row] = rn;
    sv[row] = acc;
    d[0] += acc * acc; d[1] += rn * rn;
  }
};
template <class T> struct CrlsL2Fin {     // gamma_next (+ lambda ||Ar||^2) ; beta = gamma_next / gamma   (crls.jl:225-227,235)
  CrlsState<T>* s; T lambda;
  __device__ void operator()(const T* tot) const {
    T g = tot[0];
    if (lambda > T(0)) { const T an = sqrt_rn(s->ArAr); g = add_rn(g, mul_rn(mul_rn(lambda, an), an)); }
    s->beta = div_rn(g, s->gamma);
    s->gamma = g;
    s->rr = tot[1];
  }
};
template <class T> struct CrlsL3Body {    // Ap = s + beta Ap                       (crls.jl:230)
  T* Ap; const T* sv; const CrlsState<T>* s;
  __device__ __forceinline__ void operator()(int i, T*) const { Ap[i] = add_rn(mul_rn(T(1), sv[i]), mul_rn(s->beta, Ap[i])); }
};
template <class T> struct CrlsL4Epi {     // p = Ar + beta p ; q = A^T Ap (+ lambda p) ; <q, q>   (crls.jl:229,232-233,194)
  T* p; const T* Ar; T* q; const CrlsState<T>* s; T lambda;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    const T pn = add_rn(mul_rn(T(1), Ar[row]), mul_rn(s->beta, p[row]));
    p[row] = pn;
    T qn = acc;
    if (lambda > T(0)) qn = add_rn(qn, mul_rn(lambda, pn));
    q[row] = qn;
    d[0] += qn * qn;
  }
};
template <class T> struct CrlsL4Fin {     // alpha = gamma / <q, q>                 (crls.jl:195)
  CrlsState<T>* s;
  __device__ void operator()(const T* tot) const { s->alpha = div_rn(s->gamma, tot[0]); }
};

template <class T>
void crls_fused_iteration(Workspace<T>& ws, const Csr<T>& A, const Csr<T>& At, bool init, T alpha, T gamma, T lambda, T* ArAr,
                          T* xx, T* rr, T* gamma_out) {
  Ctx& c = ws.ctx;
  StateBlock<CrlsState, T> sb(ws);
  CrlsState<T>* S = sb.dev;
  if (init) {
    CrlsState<T> s{};
    s.alpha = alpha; s.gamma = gamma;
    sb.seed(s);
  }
  launch_stream<T, 2>(c, ws.n, CrlsL1Body<T>{ws.x, ws.Ar, ws.p, ws.q, S}, CrlsL1Fin<T>{S});
  launch_spmv_epi_g<T, 2>(c, A, XPlain<T>{ws.Ar}, CrlsL2Epi<T>{ws.r, ws.Ap, ws.s, S}, CrlsL2Fin<T>{S, lambda});
  sb.post();
  launch_stream<T, 0>(c, ws.m, CrlsL3Body<T>{ws.Ap, ws.s, S}, NoFin());
  launch_spmv_epi_g<T, 1>(c, At, XPlain<T>{ws.Ap}, CrlsL4Epi<T>{ws.p, ws.Ar, ws.q, S, lambda}, CrlsL4Fin<T>{S});
  const CrlsState<T>& h = sb.wait();
  *ArAr = h.ArAr; *xx = h.xx; *rr = h.rr; *gamma_out = h.gamma;
}

// ===========================================================================
// BiLQ / QMR  (src/bilq.jl:234-254,310-335, src/qmr.jl:238-258,314-350, M = N = I)
// One Lanczos biorthogonalization step is two SpMV launches: B1's Fin leaves alpha in the device block, B2 reads it and
// its Fin stores <p, q>; the host reads {alpha, <p, q>} once, runs the factorization, and one streaming pass U applies
// the direction / solution update and forms v_{k+1}, u_{k+1} in the buffers of v_{k-1}, u_{k-1} (the caller rotates
// the pointers).  When <p, q> = 0 the reference keeps v_k and u_k: U then copies them instead of dividing.
// ===========================================================================
template <class T> struct BiorthState { T alpha, pq, vv1, v1v1; };   // alpha: B1 -> B2; vv1, v1v1: the update pass

template <class T> struct BiorthB1Epi {   // q = A v - gamma v_{k-1} ; <u, q>          (bilq.jl:236,244,247)
  T* q; const T* vprev; const T* u; T gamma;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    const T qn = add_rn(acc, mul_rn(-gamma, vprev[row]));
    q[row] = qn;
    d[0] += u[row] * qn;
  }
};
template <class T> struct BiorthB1Fin {
  BiorthState<T>* s;
  __device__ void operator()(const T* tot) const { s->alpha = tot[0]; }
};
template <class T> struct BiorthB2Epi {   // p = A^T u - beta u_{k-1} - alpha u ; q -= alpha v ; <p, q>   (:241,245,249-252)
  T* p; T* q; const T* uprev; const T* u; const T* v; const BiorthState<T>* s; T beta;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    const T alpha = s->alpha;
    const T pn = add_rn(add_rn(acc, mul_rn(-beta, uprev[row])), mul_rn(-alpha, u[row]));
    const T qn = add_rn(q[row], mul_rn(-alpha, v[row]));
    p[row] = pn;
    q[row] = qn;
    d[0] += pn * qn;
  }
};
template <class T> struct BiorthB2Fin {
  BiorthState<T>* s;
  __device__ void operator()(const T* tot) const { s->pq = tot[0]; }
};
// v_{k+1} = q / beta_{k+1}, u_{k+1} = p / gamma_{k+1} into the rotated buffers (kdivcopy!: true divisions)
template <class T> struct BiorthNext {
  T* vnext; T* unext; const T* q; const T* p; const T* v; const T* u; T beta1, gamma1; int keep;
  __device__ __forceinline__ T operator()(int i) const {
    if (keep) { unext[i] = u[i]; return vnext[i] = v[i]; }
    unext[i] = div_rn(p[i], gamma1);
    return vnext[i] = div_rn(q[i], beta1);
  }
};
// QMR (qmr.jl:316-350): w_k = (v - lambda w_{k-1} - eps w_{k-2}) / delta in the kscal!/kaxpy!/kdiv! order (first
// iteration: w_1 = v / delta into w_{k-1}); x += zeta w_k; the next v, u; ||v_{k+1}||^2 (tau).
template <class T, bool FIRST> struct BiorthQmrBody {   // FIRST: iteration 1 (its own instantiation: no spill)
  T* wk; const T* w1; T* x; const T* v; BiorthNext<T> nx; T eps2, lambda, inv_delta, delta, zeta; int iter;
  __device__ __forceinline__ void operator()(int i, T* d) const {
    const T vi = v[i];
    T w;
    if (FIRST) {
      w = div_rn(vi, delta);
    } else {
      w = wk[i];
      if (iter >= 3) w = mul_rn(-eps2, w);
      w = add_rn(w, mul_rn(-lambda, w1[i]));
      w = add_rn(w, mul_rn(T(1), vi));
      w = mul_rn(inv_delta, w);
    }
    wk[i] = w;
    x[i] = add_rn(x[i], mul_rn(zeta, w));
    const T vn = nx(i);
    d[0] += vn * vn;
  }
};
// BiLQ (bilq.jl:310-335): d̅ = v on the first iteration, else x += (zeta c) d̅, x += (zeta s) v, d̅ = -c v + s d̅;
// the next v, u; <v_k, v_{k+1}> and ||v_{k+1}||^2.
template <class T> struct BiorthBilqBody {
  T* dbar; T* x; const T* v; BiorthNext<T> nx; T czeta, szeta, c, s; int first;
  __device__ __forceinline__ void operator()(int i, T* d) const {
    const T vi = v[i];
    if (first) {
      dbar[i] = vi;
    } else {
      const T di = dbar[i];
      x[i] = add_rn(add_rn(x[i], mul_rn(czeta, di)), mul_rn(szeta, vi));
      dbar[i] = add_rn(mul_rn(-c, vi), mul_rn(s, di));
    }
    const T vn = nx(i);
    d[0] += vi * vn; d[1] += vn * vn;
  }
};

template <class T> struct BiorthQmrFin { BiorthState<T>* s; __device__ void operator()(const T* tot) const { s->v1v1 = tot[0]; } };
template <class T> struct BiorthBilqFin {
  BiorthState<T>* s;
  __device__ void operator()(const T* tot) const { s->vv1 = tot[0]; s->v1v1 = tot[1]; }
};

template <class T>
void biorth_fused_lanczos(Workspace<T>& ws, const Csr<T>& A, const Csr<T>& At, T beta, T gamma, T* alpha, T* pq) {
  Ctx& c = ws.ctx;
  StateBlock<BiorthState, T> sb(ws);
  BiorthState<T>* S = sb.dev;
  launch_spmv_epi_g<T, 1>(c, A, XPlain<T>{ws.v}, BiorthB1Epi<T>{ws.q, ws.v_prev, ws.u, gamma}, BiorthB1Fin<T>{S});
  launch_spmv_epi_g<T, 1>(c, At, XPlain<T>{ws.u}, BiorthB2Epi<T>{ws.p, ws.q, ws.u_prev, ws.u, ws.v, S, beta},
                          BiorthB2Fin<T>{S});
  const BiorthState<T>& h = sb.read();
  *alpha = h.alpha; *pq = h.pq;
}

template <class T>
T qmr_fused_update(Workspace<T>& ws, T* wk, const T* w1, int iter, T eps2, T lambda, T delta, T zeta, T beta1, T gamma1,
                   bool keep) {
  Ctx& c = ws.ctx;
  StateBlock<BiorthState, T> sb(ws);
  const BiorthNext<T> nx{ws.v_prev, ws.u_prev, ws.q, ws.p, ws.v, ws.u, beta1, gamma1, keep ? 1 : 0};
  if (iter == 1)
    launch_stream<T, 1>(c, ws.n, BiorthQmrBody<T, true>{wk, w1, ws.x, ws.v, nx, eps2, lambda, T(1) / delta, delta, zeta, iter},
                        BiorthQmrFin<T>{sb.dev});
  else
    launch_stream<T, 1>(c, ws.n, BiorthQmrBody<T, false>{wk, w1, ws.x, ws.v, nx, eps2, lambda, T(1) / delta, delta, zeta, iter},
                        BiorthQmrFin<T>{sb.dev});
  return sb.read().v1v1;
}

template <class T>
void bilq_fused_update(Workspace<T>& ws, bool first, T czeta, T szeta, T cs, T sn, T beta1, T gamma1, bool keep, T* vv1,
                       T* v1v1) {
  StateBlock<BiorthState, T> sb(ws);
  const BiorthNext<T> nx{ws.v_prev, ws.u_prev, ws.q, ws.p, ws.v, ws.u, beta1, gamma1, keep ? 1 : 0};
  launch_stream<T, 2>(ws.ctx, ws.n, BiorthBilqBody<T>{ws.w, ws.x, ws.v, nx, czeta, szeta, cs, sn, first ? 1 : 0},
                      BiorthBilqFin<T>{sb.dev});
  const BiorthState<T>& h = sb.read();
  *vv1 = h.vv1; *v1v1 = h.v1v1;
}

// ===========================================================================
// CAR  (src/car.jl:187-214, M = I: Mu === u)
// C1 updates x, r, s and returns ||r||^2, ||s||^2 (the host decides `solved` from ||r||); when not solved, C2 (SpMV on s)
// leaves rho_next = <t, s> and beta = rho_next / rho in the device block, C3 reads beta and updates the directions,
// and the host reads {rho_next, <u, u>} once and re-derives beta with the same division.
// ===========================================================================
template <class T> struct CarState { T rho_next, beta, uu, rr, ss; };   // beta: C2 -> C3

template <class T> struct CarC1Body {     // x += alpha p ; r -= alpha q ; s -= alpha u ; ||r||^2, ||s||^2   (car.jl:189-191)
  T* x; T* r; T* s; const T* p; const T* q; const T* u; T alpha;
  __device__ __forceinline__ void operator()(int j, T* d) const {
    x[j] = add_rn(x[j], mul_rn(alpha, p[j]));
    const T rn = add_rn(r[j], mul_rn(-alpha, q[j]));
    r[j] = rn;
    const T sn = add_rn(s[j], mul_rn(-alpha, u[j]));
    s[j] = sn;
    d[0] += rn * rn; d[1] += sn * sn;
  }
};
template <class T> struct CarC1Fin { CarState<T>* st; __device__ void operator()(const T* tot) const { st->rr = tot[0]; st->ss = tot[1]; } };
template <class T> struct CarC2Epi {      // t = A s ; <t, s>                       (car.jl:203-204)
  T* t; const T* s;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const { t[row] = acc; d[0] += acc * __ldg(&s[row]); }
};
template <class T> struct CarC2Fin {      // rho_next ; beta = rho_next / rho        (car.jl:205)
  CarState<T>* st; T rho;
  __device__ void operator()(const T* tot) const { st->rho_next = tot[0]; st->beta = div_rn(tot[0], rho); }
};
template <class T> struct CarC3Body {     // p = r + beta p ; q = s + beta q ; u = t + beta u ; <u, u>   (car.jl:207-209)
  T* p; T* q; T* u; const T* r; const T* s; const T* t; const CarState<T>* st;
  __device__ __forceinline__ void operator()(int j, T* d) const {
    const T beta = st->beta;
    p[j] = add_rn(mul_rn(T(1), r[j]), mul_rn(beta, p[j]));
    q[j] = add_rn(mul_rn(T(1), s[j]), mul_rn(beta, q[j]));
    const T un = add_rn(mul_rn(T(1), t[j]), mul_rn(beta, u[j]));
    u[j] = un;
    d[0] += un * un;
  }
};
template <class T> struct CarC3Fin {
  CarState<T>* st;
  __device__ void operator()(const T* tot) const { st->uu = tot[0]; }
};

template <class T> void car_fused_step(Workspace<T>& ws, T alpha, T* rr, T* ss) {
  StateBlock<CarState, T> sb(ws);
  launch_stream<T, 2>(ws.ctx, ws.n, CarC1Body<T>{ws.x, ws.r, ws.s, ws.p, ws.q, ws.u, alpha}, CarC1Fin<T>{sb.dev});
  const CarState<T>& h = sb.read();
  *rr = h.rr; *ss = h.ss;
}
template <class T> void car_fused_directions(Workspace<T>& ws, const Csr<T>& A, T rho, T* rho_next, T* uu) {
  Ctx& c = ws.ctx;
  StateBlock<CarState, T> sb(ws);
  CarState<T>* S = sb.dev;
  launch_spmv_epi<T, 1>(c, A, ws.s, CarC2Epi<T>{ws.t, ws.s}, CarC2Fin<T>{S, rho});
  launch_stream<T, 1>(c, ws.n, CarC3Body<T>{ws.p, ws.q, ws.u, ws.r, ws.s, ws.t, S}, CarC3Fin<T>{S});
  const CarState<T>& h = sb.read();
  *rho_next = h.rho_next; *uu = h.uu;
}

// ===========================================================================
// MINARES  (src/minares.jl:283-321,450-471)
// M1's Fin leaves alpha_{k+1} in the device block and M2 reads it; the host reads {alpha, ||v_k||^2} once, runs every
// rotation unchanged, and M3 applies the scaling of v_k, the d recurrence and the solution update.  w_k and d_k are
// formed in the buffers of w_{k-1} / d_{k-1} at iteration 1 and of w_{k-2} / d_{k-2} after (the caller rotates them).
// ===========================================================================
template <class T> struct MinaresState { T alpha, vv; };

// w_k = v_k / lam (iteration 1, kdivcopy!), else (v_k - gamma1 w_{k-1} - eps2 w_{k-2}) / lam in the
// kscal!/kaxpy!/kaxpy!/kdiv! order   (minares.jl:283-302)
template <class T> struct MinaresW {
  T* wk; const T* w1; T eps2, gamma1, lam, inv_lam; int iter;
  __device__ __forceinline__ void operator()(int i, T vi) const {
    T w;
    if (iter == 1) {
      w = div_rn(vi, lam);
    } else {
      w = wk[i];
      if (iter >= 3) w = mul_rn(-eps2, w);
      w = add_rn(w, mul_rn(-gamma1, w1[i]));
      w = add_rn(w, mul_rn(T(1), vi));
      w = mul_rn(inv_lam, w);
    }
    wk[i] = w;
  }
};
template <class T> struct MinaresM1Epi {  // w_k ; v_k = A v_{k+1} - beta v_k (+ shift v_{k+1}) ; <v_k, v_{k+1}>   (:307-311)
  MinaresW<T> w; T* vk; const T* vk1; T beta1, shift; int shifted;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    const T vi = vk[row];
    w(row, vi);
    T vn = add_rn(mul_rn(T(1), acc), mul_rn(-beta1, vi));
    const T v1 = __ldg(&vk1[row]);
    if (shifted) vn = add_rn(vn, mul_rn(shift, v1));
    vk[row] = vn;
    d[0] += vn * v1;
  }
};
template <class T> struct MinaresM1Fin {
  MinaresState<T>* st;
  __device__ void operator()(const T* tot) const { st->alpha = tot[0]; }
};
template <class T> struct MinaresWBody {  // w_k only: no product once the Lanczos process has terminated
  MinaresW<T> w; const T* vk;
  __device__ __forceinline__ void operator()(int j, T*) const { w(j, vk[j]); }
};
template <class T> struct MinaresM2Body { // v_k -= alpha v_{k+1} ; ||v_k||^2        (minares.jl:312-313)
  T* vk; const T* vk1; const MinaresState<T>* st;
  __device__ __forceinline__ void operator()(int j, T* d) const {
    const T vn = add_rn(vk[j], mul_rn(-st->alpha, vk1[j]));
    vk[j] = vn;
    d[0] += vn * vn;
  }
};
template <class T> struct MinaresM2Fin {
  MinaresState<T>* st;
  __device__ void operator()(const T* tot) const { st->vv = tot[0]; }
};
// v_k /= beta (kdiv!) ; d_k = w_k / mu (iteration 1, kdivcopy!), else (w_k - phi1 d_{k-1} - rho2 d_{k-2}) / mu ;
// x += zeta d_k   (minares.jl:319,450-471)
template <class T> struct MinaresM3Body {
  T* vk; T* dk; const T* d1; const T* wk; T* x; T inv_beta, rho2, phi1, mu, inv_mu, zeta; int scale, iter;
  __device__ __forceinline__ void operator()(int j, T*) const {
    if (scale) vk[j] = mul_rn(inv_beta, vk[j]);
    T dd;
    if (iter == 1) {
      dd = div_rn(wk[j], mu);
    } else {
      dd = dk[j];
      if (iter >= 3) dd = mul_rn(-rho2, dd);
      dd = add_rn(dd, mul_rn(-phi1, d1[j]));
      dd = add_rn(dd, mul_rn(T(1), wk[j]));
      dd = mul_rn(inv_mu, dd);
    }
    dk[j] = dd;
    x[j] = add_rn(x[j], mul_rn(zeta, dd));
  }
};

template <class T>
void minares_fused_lanczos(Workspace<T>& ws, const Csr<T>& A, bool lanczos, int iter, T* vk, const T* vk1, T* wk, const T* w1,
                           T eps2, T gamma1, T lam, T beta1, T shift, T* alpha, T* vv) {
  Ctx& c = ws.ctx;
  const MinaresW<T> w{wk, w1, eps2, gamma1, lam, T(1) / lam, iter};
  if (!lanczos) {
    launch_stream<T, 0>(c, ws.n, MinaresWBody<T>{w, vk}, NoFin());
    return;
  }
  StateBlock<MinaresState, T> sb(ws);
  MinaresState<T>* S = sb.dev;
  launch_spmv_epi<T, 1>(c, A, vk1, MinaresM1Epi<T>{w, vk, vk1, beta1, shift, shift != T(0) ? 1 : 0}, MinaresM1Fin<T>{S});
  launch_stream<T, 1>(c, ws.n, MinaresM2Body<T>{vk, vk1, S}, MinaresM2Fin<T>{S});
  const MinaresState<T>& h = sb.read();
  *alpha = h.alpha; *vv = h.vv;
}

template <class T>
void minares_fused_update(Workspace<T>& ws, int iter, T* vk, bool scale, T beta, T* dk, const T* d1, const T* wk, T rho2,
                          T phi1, T mu, T zeta) {
  launch_stream<T, 0>(ws.ctx, ws.n,
                      MinaresM3Body<T>{vk, dk, d1, wk, ws.x, scale ? T(1) / beta : T(1), rho2, phi1, mu, T(1) / mu, zeta,
                                       scale ? 1 : 0, iter},
                      NoFin());
}

// ===========================================================================
// BiLQR / TriLQR  (src/bilqr.jl:227-418, src/trilqr.jl:210-397; adjoint pairs A x = b, A^T y = c)
// BiLQR runs BiLQ's B1 / B2 unchanged and one update pass U over n.  TriLQR's SSY step is T1 (SpMV on A, alpha on the
// device) and T2 (SpMV on A^T, which also finishes q over all m rows: beta_{k+1} = ||q|| is needed before U), then one
// update pass over max(m, n).  U carries the primal half (x, d̅), the dual half (w_{k-1}, y) and the next v, u; a half
// that has converged gets an instantiation without its vectors.
// ===========================================================================
template <class T> struct AdjointState { T alpha, qq, pp, vq, uu; };   // alpha: T1 -> T2; qq: ||q||^2 of T2 or of U

// Dual direction and solution (bilqr.jl:363-392, trilqr.jl:339-368), iteration >= 2: w_{k-1} = src / delta at iteration
// 2 (kdivcopy!), else (w_{k-3} + src - lam2 w_{k-2}) / delta with w_{k-3} first scaled by -eps3 from iteration 4 on, in
// the kscal!/kaxpy!/kaxpy!/kdiv! order; y += psi w_{k-1}.  wk is the buffer of w_{k-2} at iteration 2, of w_{k-3} after.
// w_{k-3} is still the reference's zero vector at iteration 3: it is not read then, so the fused path needs no fill.
template <class T> struct AdjointW {
  T* wk; const T* w2; T* y; T eps3, lam2, delta, inv_delta, psi; int iter;
  __device__ __forceinline__ void operator()(int i, T src) const {
    T w;
    if (iter == 2) {
      w = div_rn(src, delta);
    } else {
      w = iter >= 4 ? mul_rn(-eps3, wk[i]) : T(0);
      w = add_rn(w, mul_rn(T(1), src));
      w = add_rn(w, mul_rn(-lam2, w2[i]));
      w = mul_rn(inv_delta, w);
    }
    wk[i] = w;
    y[i] = add_rn(y[i], mul_rn(psi, w));
  }
};
// Primal direction and solution (bilqr.jl:299-311, trilqr.jl:283-295): d̅ = a at iteration 1, else x += (zeta c) d̅,
// x += (zeta s) a, d̅ = -c a + s d̅ (a = v_k for BiLQR, u_k for TriLQR).
template <class T> struct AdjointD {
  T* dbar; T* x; T czeta, szeta, c, s; int iter;
  __device__ __forceinline__ void operator()(int i, T a) const {
    if (iter == 1) {
      dbar[i] = a;
    } else {
      const T di = dbar[i];
      x[i] = add_rn(add_rn(x[i], mul_rn(czeta, di)), mul_rn(szeta, a));
      dbar[i] = add_rn(mul_rn(-c, a), mul_rn(s, di));
    }
  }
};

// The next v and u are written into the buffers of v_{k-1} and u_{k-1}, and the dual direction reads one of those
// same buffers (u_{k-1} in BiLQR, v_{k-1} in TriLQR).  So every element of it is read, by the thread that then
// overwrites it, before the next vector is stored: each body below calls the dual update first.
template <class T, bool PRIMAL, bool DUAL> struct AdjointBilqrBody {
  AdjointD<T> dd; AdjointW<T> w; const T* v; const T* q; const T* p; const T* u; T* vnext; T* unext; T beta1, gamma1; int keep;
  __device__ __forceinline__ void operator()(int i, T* d) const {
    if (DUAL && w.iter >= 2) w(i, unext[i]);          // u_{k-1}, read before u_{k+1} overwrites it
    const T qi = q[i];
    if (PRIMAL) {
      const T vi = v[i];
      dd(i, vi);
      d[0] += vi * qi; d[1] += qi * qi;
    }
    vnext[i] = keep ? v[i] : div_rn(qi, beta1);
    const T un = keep ? u[i] : div_rn(p[i], gamma1);
    unext[i] = un;
    if (DUAL) d[2] += un * un;
  }
};
template <class T> struct AdjointBilqrFin {
  AdjointState<T>* s;
  __device__ void operator()(const T* tot) const { s->vq = tot[0]; s->qq = tot[1]; s->uu = tot[2]; }
};
template <class T, bool PRIMAL, bool DUAL> struct AdjointTrilqrBody {
  AdjointD<T> dd; AdjointW<T> w; const T* v; const T* q; const T* p; const T* u; T* vnext; T* unext; T beta1, gamma1;
  int m, n;
  __device__ __forceinline__ void operator()(int i, T*) const {
    if (i < m) {
      if (DUAL && w.iter >= 2) w(i, vnext[i]);        // v_{k-1}, read before v_{k+1} overwrites it
      vnext[i] = beta1 != T(0) ? div_rn(q[i], beta1) : v[i];
    }
    if (i < n) {
      const T ui = u[i];
      if (PRIMAL) dd(i, ui);
      unext[i] = gamma1 != T(0) ? div_rn(p[i], gamma1) : ui;
    }
  }
};
template <class T> struct AdjointT1Epi {   // q = A u - gamma v_{k-1} ; <v, q>           (trilqr.jl:210,214,218)
  T* q; const T* vprev; const T* v; T gamma; int first;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    const T qn = first ? acc : add_rn(acc, mul_rn(-gamma, vprev[row]));
    q[row] = qn;
    d[0] += v[row] * qn;
  }
};
template <class T> struct AdjointT1Fin {
  AdjointState<T>* s;
  __device__ void operator()(const T* tot) const { s->alpha = tot[0]; }
};
// p = A^T v - beta u_{k-1} - alpha u (rows < n) ; q -= alpha v (rows < m) ; ||q||^2, ||p||^2   (trilqr.jl:211,215,220-224)
template <class T> struct AdjointT2Epi {
  T* p; T* q; const T* uprev; const T* u; const T* v; const AdjointState<T>* s; T beta; int m, n, first;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    const T alpha = s->alpha;
    if (row < n) {
      T pn = first ? acc : add_rn(acc, mul_rn(-beta, uprev[row]));
      pn = add_rn(pn, mul_rn(-alpha, u[row]));
      p[row] = pn;
      d[1] += pn * pn;
    }
    if (row < m) {
      const T qn = add_rn(q[row], mul_rn(-alpha, v[row]));
      q[row] = qn;
      d[0] += qn * qn;
    }
  }
};
template <class T> struct AdjointT2Fin {
  AdjointState<T>* s;
  __device__ void operator()(const T* tot) const { s->qq = tot[0]; s->pp = tot[1]; }
};

template <class T>
void bilqr_fused_update(Workspace<T>& ws, bool primal, bool dual, int iter, T czeta, T szeta, T cs, T sn, T* wk, const T* w2,
                        T eps3, T lam2, T delta1, T psi1, T beta1, T gamma1, bool keep, T* out3) {
  Ctx& c = ws.ctx;
  const AdjointD<T> dd{ws.w, ws.x, czeta, szeta, cs, sn, iter};
  const AdjointW<T> w{wk, w2, ws.y, eps3, lam2, delta1, T(1) / delta1, psi1, iter};
  StateBlock<AdjointState, T> sb(ws);
  const AdjointBilqrFin<T> fin{sb.dev};
  const int k = keep ? 1 : 0;
  if (primal && dual)
    launch_stream<T, 3>(c, ws.n, AdjointBilqrBody<T, true, true>{dd, w, ws.v, ws.q, ws.p, ws.u, ws.v_prev, ws.u_prev, beta1, gamma1, k}, fin);
  else if (primal)
    launch_stream<T, 3>(c, ws.n, AdjointBilqrBody<T, true, false>{dd, w, ws.v, ws.q, ws.p, ws.u, ws.v_prev, ws.u_prev, beta1, gamma1, k}, fin);
  else
    launch_stream<T, 3>(c, ws.n, AdjointBilqrBody<T, false, true>{dd, w, ws.v, ws.q, ws.p, ws.u, ws.v_prev, ws.u_prev, beta1, gamma1, k}, fin);
  const AdjointState<T>& h = sb.read();
  out3[0] = h.vq; out3[1] = h.qq; out3[2] = h.uu;
}

template <class T>
void trilqr_fused_ssy(Workspace<T>& ws, const Csr<T>& A, const Csr<T>& At, bool first, T beta, T gamma, T* alpha, T* qq, T* pp) {
  Ctx& c = ws.ctx;
  StateBlock<AdjointState, T> sb(ws);
  AdjointState<T>* S = sb.dev;
  const int f = first ? 1 : 0;
  launch_spmv_epi_g<T, 1>(c, A, XPlain<T>{ws.u}, AdjointT1Epi<T>{ws.q, ws.v_prev, ws.v, gamma, f}, AdjointT1Fin<T>{S});
  launch_spmv_epi_g<T, 2>(c, At, XPlain<T>{ws.v}, AdjointT2Epi<T>{ws.p, ws.q, ws.u_prev, ws.u, ws.v, S, beta, ws.m, ws.n, f},
                          AdjointT2Fin<T>{S});
  const AdjointState<T>& h = sb.read();
  *alpha = h.alpha; *qq = h.qq; *pp = h.pp;
}

template <class T>
void trilqr_fused_update(Workspace<T>& ws, bool primal, bool dual, int iter, T czeta, T szeta, T cs, T sn, T* wk, const T* w2,
                         T eps3, T lam2, T delta1, T psi1, T beta1, T gamma1) {
  Ctx& c = ws.ctx;
  const AdjointD<T> dd{ws.w, ws.x, czeta, szeta, cs, sn, iter};
  const AdjointW<T> w{wk, w2, ws.y, eps3, lam2, delta1, T(1) / delta1, psi1, iter};
  const int len = std::max(ws.m, ws.n);
  if (primal && dual)
    launch_stream<T, 0>(c, len, AdjointTrilqrBody<T, true, true>{dd, w, ws.v, ws.q, ws.p, ws.u, ws.v_prev, ws.u_prev, beta1, gamma1,
                                                                 ws.m, ws.n}, NoFin());
  else if (primal)
    launch_stream<T, 0>(c, len, AdjointTrilqrBody<T, true, false>{dd, w, ws.v, ws.q, ws.p, ws.u, ws.v_prev, ws.u_prev, beta1, gamma1,
                                                                  ws.m, ws.n}, NoFin());
  else
    launch_stream<T, 0>(c, len, AdjointTrilqrBody<T, false, true>{dd, w, ws.v, ws.q, ws.p, ws.u, ws.v_prev, ws.u_prev, beta1, gamma1,
                                                                  ws.m, ws.n}, NoFin());
}

// ===========================================================================
// CRAIG / CRAIGMR  (src/craig.jl:276-379, src/craigmr.jl:280-379; lambda = 0, M = N = I)
// As for LSQR, kdiv!(u, beta) and kdiv!(v, alpha) are left pending: Mu and Nv stay unscaled in memory and every reader
// applies s_u = 1/beta or s_v = 1/alpha (1 when the reference skips the division), which is the rounding kdiv! does.
// The SpMV gathers take the factor from the device block (written by the Fin of the pass that produced the norm); the
// epilogues take it by value from the host, which computed the same quotient from the same read-back.
// ===========================================================================
template <class T> struct CraigState { T s_u, s_v, alpha, beta, ww, ia, mba; };

template <class T> struct CraigNormFin {     // tot[0] = ||z||^2 -> s = ||z|| ; inverse = 1/s (1 when s = 0)
  T* out; T* inv;
  __device__ void operator()(const T* tot) const {
    const T s = sqrt_rn(tot[0]);
    *out = s;
    *inv = s == T(0) ? T(1) : div_rn(T(1), s);
  }
};
// CRAIG C1 on A^T, gathering u: x += xi v (the previous iteration's, pending) ; Nv = A^T u - beta v ; ||Nv||^2
template <class T> struct CraigP1Epi {
  T* nv; T* x; T beta, s_v, xi; int xup;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    const T v = mul_rn(nv[row], s_v);
    if (xup) x[row] = add_rn(x[row], mul_rn(xi, v));
    const T nn = add_rn(mul_rn(T(1), acc), mul_rn(-beta, v));
    nv[row] = nn;
    d[0] += nn * nn;
  }
};
// CRAIG C2 on A, gathering v: w = u + tw w ; y += ty w ; ||w||^2 ; Mu = A v - alpha u ; ||Mu||^2
template <class T> struct CraigP2Epi {
  T* mu; T* w; T* y; T s_u, alpha, tw, ty;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    const T u = mul_rn(mu[row], s_u);
    const T wn = add_rn(mul_rn(T(1), u), mul_rn(tw, w[row]));
    w[row] = wn;
    y[row] = add_rn(y[row], mul_rn(ty, wn));
    d[1] += wn * wn;
    const T nm = add_rn(mul_rn(T(1), acc), mul_rn(-alpha, u));
    mu[row] = nm;
    d[0] += nm * nm;
  }
};
template <class T> struct CraigP2Fin {
  CraigState<T>* s;
  __device__ void operator()(const T* tot) const {
    CraigNormFin<T>{&s->beta, &s->s_u}(tot);
    s->ww = tot[1];
  }
};
template <class T> struct CraigFlushBody {   // x += xi v, v = Nv s_v
  T* x; const T* nv; T xi, s_v;
  __device__ __forceinline__ void operator()(int i, T*) const { x[i] = add_rn(x[i], mul_rn(xi, mul_rn(nv[i], s_v))); }
};

template <class T> T craig_fused_p1(Workspace<T>& ws, const Csr<T>& At, bool init, T beta, T s_v, bool xup, T xi) {
  StateBlock<CraigState, T> sb(ws);
  CraigState<T>* S = sb.dev;
  if (init) {                     // u_1 and v_0 = 0 are stored scaled: both factors start at 1
    CraigState<T> s{};
    s.s_u = T(1); s.s_v = T(1);
    sb.seed(s);
  }
  launch_spmv_epi_g<T, 1>(ws.ctx, At, XScaled<T>{ws.Mu, &S->s_u, T(1)}, CraigP1Epi<T>{ws.Nv, ws.x, beta, s_v, xi, xup ? 1 : 0},
                          CraigNormFin<T>{&S->alpha, &S->s_v});
  return sb.read().alpha;
}
template <class T> void craig_fused_p2(Workspace<T>& ws, const Csr<T>& A, T s_u, T alpha, T tw, T ty, T* beta, T* ww) {
  StateBlock<CraigState, T> sb(ws);
  CraigState<T>* S = sb.dev;
  launch_spmv_epi_g<T, 2>(ws.ctx, A, XScaled<T>{ws.Nv, &S->s_v, T(1)}, CraigP2Epi<T>{ws.Mu, ws.w, ws.y, s_u, alpha, tw, ty},
                          CraigP2Fin<T>{S});
  const CraigState<T>& h = sb.read();
  *beta = h.beta; *ww = h.ww;
}
template <class T> void craig_fused_flush(Workspace<T>& ws, T xi, T s_v) {
  launch_stream<T, 0>(ws.ctx, ws.n, CraigFlushBody<T>{ws.x, ws.Nv, xi, s_v}, NoFin());
}

// CRAIGMR R1 on A, gathering v: Mu = A v - alpha u ; ||Mu||^2
template <class T> struct CraigmrP1Epi {
  T* mu; T s_u, alpha;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    const T nm = add_rn(mul_rn(T(1), acc), mul_rn(-alpha, mul_rn(mu[row], s_u)));
    mu[row] = nm;
    d[0] += nm * nm;
  }
};
// CRAIGMR R2 on A^T, gathering u: d = v / rho (first) or d = (1/rho) v + tr d ; x += zeta d ; Nv = A^T u - beta v ; ||Nv||^2
template <class T> struct CraigmrP2Epi {
  T* nv; T* dd; T* x; T s_v, rho, inv_rho, tr, zeta, beta; int first;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    const T v = mul_rn(nv[row], s_v);
    const T dn = first ? div_rn(v, rho) : add_rn(mul_rn(inv_rho, v), mul_rn(tr, dd[row]));
    dd[row] = dn;
    x[row] = add_rn(x[row], mul_rn(zeta, dn));
    const T nn = add_rn(mul_rn(T(1), acc), mul_rn(-beta, v));
    nv[row] = nn;
    d[0] += nn * nn;
  }
};
template <class T> struct CraigmrP2Fin {     // alpha, s_v and the coefficients of the w̄ update: 1/alpha, -beta/alpha
  CraigState<T>* s;
  __device__ void operator()(const T* tot) const {
    CraigNormFin<T>{&s->alpha, &s->s_v}(tot);
    if (s->alpha != T(0)) { s->ia = div_rn(T(1), s->alpha); s->mba = div_rn(-s->beta, s->alpha); }
  }
};
// CRAIGMR R3 over m: w = (1/rho) w̄ + tr w ; y += zeta w ; alpha != 0: w̄ = (1/alpha) u - (beta/alpha) w̄
template <class T> struct CraigmrP3Body {
  T* w; T* y; T* wbar; const T* mu; const CraigState<T>* s; T s_u, inv_rho, tr, zeta;
  __device__ __forceinline__ void operator()(int i, T*) const {
    const T wb = wbar[i];
    const T wn = add_rn(mul_rn(inv_rho, wb), mul_rn(tr, w[i]));
    w[i] = wn;
    y[i] = add_rn(y[i], mul_rn(zeta, wn));
    if (s->alpha != T(0)) wbar[i] = add_rn(mul_rn(s->ia, mul_rn(mu[i], s_u)), mul_rn(s->mba, wb));
  }
};

template <class T> T craigmr_fused_p1(Workspace<T>& ws, const Csr<T>& A, bool init, T s_u, T alpha) {
  StateBlock<CraigState, T> sb(ws);
  CraigState<T>* S = sb.dev;
  if (init) {
    CraigState<T> s{};
    s.s_u = T(1); s.s_v = T(1);
    sb.seed(s);
  }
  launch_spmv_epi_g<T, 1>(ws.ctx, A, XScaled<T>{ws.Nv, &S->s_v, T(1)}, CraigmrP1Epi<T>{ws.Mu, s_u, alpha},
                          CraigNormFin<T>{&S->beta, &S->s_u});
  return sb.read().beta;
}
template <class T>
T craigmr_fused_p23(Workspace<T>& ws, const Csr<T>& At, bool first, T s_u, T s_v, T beta, T rho, T inv_rho, T tr, T zeta) {
  StateBlock<CraigState, T> sb(ws);
  CraigState<T>* S = sb.dev;
  launch_spmv_epi_g<T, 1>(ws.ctx, At, XScaled<T>{ws.Mu, &S->s_u, T(1)},
                          CraigmrP2Epi<T>{ws.Nv, ws.d1, ws.x, s_v, rho, inv_rho, tr, zeta, beta, first ? 1 : 0}, CraigmrP2Fin<T>{S});
  launch_stream<T, 0>(ws.ctx, ws.m, CraigmrP3Body<T>{ws.w, ws.y, ws.w1, ws.Mu, S, s_u, inv_rho, tr, zeta}, NoFin());
  return sb.read().alpha;
}

// ===========================================================================
// LNLQ  (src/lnlq.jl:326-552; lambda = 0, M = N = I)
// The products run in LSQR's order, A v then A^T u, with kdiv!(u, beta) and kdiv!(v, alpha) pending as in CRAIG.  The
// y / w̄ update of a pass needs u_{k+1}, so it rides in the next L1, which reads u before overwriting Mu.
// ===========================================================================
template <class T> struct LnlqState { T s_u, s_v, alpha, beta; };

template <class T> struct LnlqNormFin {      // tot[0] = ||z||^2 -> s = ||z|| ; inverse = 1/s (1 when s = 0)
  T* out; T* inv;
  __device__ void operator()(const T* tot) const {
    const T s = sqrt_rn(tot[0]);
    *out = s;
    *inv = s == T(0) ? T(1) : div_rn(T(1), s);
  }
};
// y += yc w̄ ; y += ys u ; w̄ = wc u + ws w̄   (kaxpy!, kaxpy!, kaxpby!: lnlq.jl:449-453)
template <class T> __device__ __forceinline__ void lnlq_y_update(T* y, T* wbar, int i, T u, T yc, T ys, T wc, T ws) {
  const T wb = wbar[i];
  y[i] = add_rn(add_rn(y[i], mul_rn(yc, wb)), mul_rn(ys, u));
  wbar[i] = add_rn(mul_rn(wc, u), mul_rn(ws, wb));
}
// L1 on A, gathering v: the previous pass's y / w̄ update (pending when yup), then Mu = A v - alpha u ; ||Mu||^2
template <class T> struct LnlqL1Epi {
  T* mu; T* y; T* wbar; T s_u, alpha, yc, ys, wc, ws; int yup;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    const T u = mul_rn(mu[row], s_u);
    if (yup) lnlq_y_update(y, wbar, row, u, yc, ys, wc, ws);
    const T nm = add_rn(mul_rn(T(1), acc), mul_rn(-alpha, u));
    mu[row] = nm;
    d[0] += nm * nm;
  }
};
// L2 on A^T, gathering u: x += tau v ; Nv = A^T u - beta v ; ||Nv||^2
template <class T> struct LnlqL2Epi {
  T* nv; T* x; T s_v, beta, tau;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    const T v = mul_rn(nv[row], s_v);
    x[row] = add_rn(x[row], mul_rn(tau, v));
    const T nn = add_rn(mul_rn(T(1), acc), mul_rn(-beta, v));
    nv[row] = nn;
    d[0] += nn * nn;
  }
};
template <class T> struct LnlqFlushBody {    // the pending y / w̄ update over m, u = Mu s_u
  T* y; T* wbar; const T* mu; T s_u, yc, ys, wc, ws;
  __device__ __forceinline__ void operator()(int i, T*) const { lnlq_y_update(y, wbar, i, mul_rn(mu[i], s_u), yc, ys, wc, ws); }
};
template <class T> struct LnlqXBody {        // x += a v, v = Nv s_v
  T* x; const T* nv; T a, s_v;
  __device__ __forceinline__ void operator()(int i, T*) const { x[i] = add_rn(x[i], mul_rn(a, mul_rn(nv[i], s_v))); }
};

template <class T>
T lnlq_fused_l1(Workspace<T>& ws, const Csr<T>& A, bool init, T s_u, T alpha, bool yup, T yc, T ys, T wc, T wsn) {
  StateBlock<LnlqState, T> sb(ws);
  LnlqState<T>* S = sb.dev;
  if (init) {                     // u_1 and v_1 are stored scaled: both factors start at 1
    LnlqState<T> s{};
    s.s_u = T(1); s.s_v = T(1);
    sb.seed(s);
  }
  launch_spmv_epi_g<T, 1>(ws.ctx, A, XScaled<T>{ws.Nv, &S->s_v, T(1)},
                          LnlqL1Epi<T>{ws.Mu, ws.y, ws.w, s_u, alpha, yc, ys, wc, wsn, yup ? 1 : 0},
                          LnlqNormFin<T>{&S->beta, &S->s_u});
  return sb.read().beta;
}
template <class T> T lnlq_fused_l2(Workspace<T>& ws, const Csr<T>& At, T s_v, T beta, T tau) {
  StateBlock<LnlqState, T> sb(ws);
  LnlqState<T>* S = sb.dev;
  launch_spmv_epi_g<T, 1>(ws.ctx, At, XScaled<T>{ws.Mu, &S->s_u, T(1)}, LnlqL2Epi<T>{ws.Nv, ws.x, s_v, beta, tau},
                          LnlqNormFin<T>{&S->alpha, &S->s_v});
  return sb.read().alpha;
}
template <class T> void lnlq_fused_flush(Workspace<T>& ws, T s_u, T yc, T ys, T wc, T wsn) {
  launch_stream<T, 0>(ws.ctx, ws.m, LnlqFlushBody<T>{ws.y, ws.w, ws.Mu, s_u, yc, ys, wc, wsn}, NoFin());
}
template <class T> void lnlq_fused_xup(Workspace<T>& ws, T a, T s_v) {
  launch_stream<T, 0>(ws.ctx, ws.n, LnlqXBody<T>{ws.x, ws.Nv, a, s_v}, NoFin());
}

// ===========================================================================
// CGNE  (src/cgne.jl:201-235; N = I, lambda = 0)
// CG on A A^T y = b with x = A^T y.  E1's Fin derives gamma_next and beta, E2's Fin delta = <p, p> and the next alpha
// (cgne.jl:204-206 at the start of the next iteration).  q = A p and Aᴴz = A^T r are consumed in the epilogues and not
// stored.  The host reads {gamma, delta} once, after E2.  No Fin writes a field its own pass's epilogue reads: E1 hands
// alpha to E2 in `ax`.
// ===========================================================================
template <class T> struct CgneState { T gamma, delta, alpha, ax, beta; };

template <class T> struct CgneE1Epi {     // q = A p ; r -= alpha q ; <r, r>            (cgne.jl:202,208,210)
  T* r; const CgneState<T>* s;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    const T rn = add_rn(r[row], mul_rn(-s->alpha, acc));
    r[row] = rn;
    d[0] += rn * rn;
  }
};
template <class T> struct CgneE1Fin {     // beta = gamma_next / gamma ; gamma = gamma_next   (cgne.jl:211,218)
  CgneState<T>* s;
  __device__ void operator()(const T* tot) const {
    s->ax = s->alpha;
    s->beta = div_rn(tot[0], s->gamma);
    s->gamma = tot[0];
  }
};
template <class T> struct CgneE2Epi {     // x += alpha p ; p = A^T r + beta p ; <p, p>   (cgne.jl:207,212-214)
  T* x; T* p; const CgneState<T>* s;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    const T pv = p[row];
    x[row] = add_rn(x[row], mul_rn(s->ax, pv));
    const T pn = add_rn(mul_rn(T(1), acc), mul_rn(s->beta, pv));
    p[row] = pn;
    d[0] += pn * pn;
  }
};
template <class T> struct CgneE2Fin {     // delta = <p, p> ; alpha = gamma / delta          (cgne.jl:204,206)
  CgneState<T>* s;
  __device__ void operator()(const T* tot) const { s->delta = tot[0]; s->alpha = div_rn(s->gamma, tot[0]); }
};

template <class T>
void cgne_fused_iteration(Workspace<T>& ws, const Csr<T>& A, const Csr<T>& At, bool init, T gamma, T delta, T* gamma_out,
                          T* delta_out) {
  Ctx& c = ws.ctx;
  StateBlock<CgneState, T> sb(ws);
  CgneState<T>* S = sb.dev;
  if (init) {
    CgneState<T> s{};
    s.gamma = gamma; s.delta = delta; s.alpha = gamma / delta;
    sb.seed(s);
  }
  launch_spmv_epi_g<T, 1>(c, A, XPlain<T>{ws.p}, CgneE1Epi<T>{ws.r, S}, CgneE1Fin<T>{S});
  launch_spmv_epi_g<T, 1>(c, At, XPlain<T>{ws.r}, CgneE2Epi<T>{ws.x, ws.p, S}, CgneE2Fin<T>{S});
  const CgneState<T>& h = sb.read();
  *gamma_out = h.gamma; *delta_out = h.delta;
}

// ===========================================================================
// CRMR  (src/crmr.jl:197-227; N = I, lambda = 0)
// CR on A A^T y = b with x = A^T y, CGLS's pass structure with the roles of the spaces swapped: R1's Fin derives alpha,
// R3's Fin gamma and beta.  The host reads {<r, r>, gamma} once, after R3; R4 is already queued behind the copy.
// ===========================================================================
template <class T> struct CrmrState { T gamma, alpha, beta, rr; };

template <class T> struct CrmrR1Epi {     // q = A p ; <q, q>                          (crmr.jl:198,201)
  T* q;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const { q[row] = acc; d[0] += acc * acc; }
};
template <class T> struct CrmrR1Fin {     // alpha = gamma / <q, q>                    (crmr.jl:201)
  CrmrState<T>* s;
  __device__ void operator()(const T* tot) const { s->alpha = div_rn(s->gamma, tot[0]); }
};
template <class T> struct CrmrR2Body {    // r -= alpha q ; <r, r>                     (crmr.jl:203-204)
  T* r; const T* q; const CrmrState<T>* s;
  __device__ __forceinline__ void operator()(int i, T* d) const {
    const T rn = add_rn(r[i], mul_rn(-s->alpha, q[i]));
    r[i] = rn;
    d[0] += rn * rn;
  }
};
template <class T> struct CrmrR2Fin {
  CrmrState<T>* s;
  __device__ void operator()(const T* tot) const { s->rr = tot[0]; }
};
template <class T> struct CrmrR3Epi {     // x += alpha p ; Aᴴr = A^T r ; <Aᴴr, Aᴴr>   (crmr.jl:202,205-206)
  T* x; const T* p; T* ar; const CrmrState<T>* s;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const {
    x[row] = add_rn(x[row], mul_rn(s->alpha, p[row]));
    ar[row] = acc;
    d[0] += acc * acc;
  }
};
template <class T> struct CrmrR3Fin {     // beta = gamma_next / gamma ; gamma = gamma_next   (crmr.jl:208,215)
  CrmrState<T>* s;
  __device__ void operator()(const T* tot) const { s->beta = div_rn(tot[0], s->gamma); s->gamma = tot[0]; }
};
template <class T> struct CrmrR4Body {    // p = Aᴴr + beta p                          (crmr.jl:210)
  T* p; const T* ar; const CrmrState<T>* s;
  __device__ __forceinline__ void operator()(int i, T*) const { p[i] = add_rn(mul_rn(T(1), ar[i]), mul_rn(s->beta, p[i])); }
};

template <class T>
void crmr_fused_iteration(Workspace<T>& ws, const Csr<T>& A, const Csr<T>& At, bool init, T gamma, T* rr, T* gamma_out) {
  Ctx& c = ws.ctx;
  StateBlock<CrmrState, T> sb(ws);
  CrmrState<T>* S = sb.dev;
  if (init) {
    CrmrState<T> s{};
    s.gamma = gamma;
    sb.seed(s);
  }
  launch_spmv_epi_g<T, 1>(c, A, XPlain<T>{ws.p}, CrmrR1Epi<T>{ws.q}, CrmrR1Fin<T>{S});
  launch_stream<T, 1>(c, ws.m, CrmrR2Body<T>{ws.r, ws.q, S}, CrmrR2Fin<T>{S});
  launch_spmv_epi_g<T, 1>(c, At, XPlain<T>{ws.r}, CrmrR3Epi<T>{ws.x, ws.p, ws.Ar, S}, CrmrR3Fin<T>{S});
  sb.post();
  launch_stream<T, 0>(c, ws.n, CrmrR4Body<T>{ws.p, ws.Ar, S}, NoFin());
  const CrmrState<T>& h = sb.wait();
  *rr = h.rr; *gamma_out = h.gamma;
}

// ===========================================================================
// Krylov processes  (src/krylov_processes.jl; drivers in processes.cu, functors Proc* in kb_internal.h)
// ===========================================================================
// No read-back here: every scalar a pass needs is in the call's device block, and the driver reads it once at the end.
template <class T> void proc_spmv(Ctx& c, const Csr<T>& A, const T* x, const T* x_s, const ProcEpi<T>& epi, const ProcFin<T>& fin) {
  if (A.n <= 0) return;
  launch_spmv_epi_g<T, 1>(c, A, ProcXDiv<T>{x, x_s, T(0)}, epi, fin);
}
template <class T> void proc_stream(Ctx& c, int n, const ProcUpdBody<T>& body, const ProcFin<T>& fin) {
  launch_stream<T, 1>(c, n, body, fin);
}
template <class T> void proc_divide(Ctx& c, const ProcDivBody<T>& body) {
  launch_stream<T, 0>(c, std::max(body.n1, body.out2 ? body.n2 : 0), body, NoFin());
}

// ===========================================================================
// CG-Lanczos-shift and CGLS-Lanczos-shift  (src/cg_lanczos_shift.jl:206-268, src/cgls_lanczos_shift.jl:206-260)
// ===========================================================================
// The shift update both solvers share, for up to kShiftPass active shifts per launch: v is read once (the first launch
// of an iteration may scale it by 1/beta and store it back, kdiv!(n, v, β)), then for every shift i of the launch
// x_i += gamma_i p_i ; p_i = sigma_i v + omega_i p_i: the reference's kaxpy! and kaxpby!, operation by operation.  The
// columns and scalars of the launch's shifts travel by value, so converged shifts cost no bytes.
template <class T> struct ShiftUpdBody {
  T* v; T inv_beta; int scale; int cnt;
  T* x[kShiftPass]; T* p[kShiftPass];
  T gamma[kShiftPass], sigma[kShiftPass], omega[kShiftPass];
  __device__ __forceinline__ void operator()(int j, T*) const {
    T vj = v[j];
    if (scale) { vj = mul_rn(inv_beta, vj); v[j] = vj; }
#pragma unroll
    for (int i = 0; i < kShiftPass; i++) {
      if (i < cnt) {
        const T pi = p[i][j];
        x[i][j] = add_rn(x[i][j], mul_rn(gamma[i], pi));
        p[i][j] = add_rn(mul_rn(sigma[i], vj), mul_rn(omega[i], pi));
      }
    }
  }
};
template <class T>
void shift_fused_update(Workspace<T>& ws, T* v, bool scale, T beta, int cnt, T* const* x, T* const* p, const T* gamma,
                        const T* sigma, const T* omega) {
  // with no active shift a requested scaling still runs (a pass over v alone), so v leaves every iteration scaled
  for (int base = 0; base < cnt || (base == 0 && scale); base += kShiftPass) {
    ShiftUpdBody<T> body{};
    body.v = v; body.inv_beta = T(1) / beta; body.scale = (scale && base == 0) ? 1 : 0;
    body.cnt = std::min(kShiftPass, cnt - base);
    for (int i = 0; i < kShiftPass; i++) {
      const bool live = base + i < cnt;
      const int k = live ? base + i : std::max(cnt - 1, 0);
      body.x[i] = cnt > 0 ? x[k] : v; body.p[i] = cnt > 0 ? p[k] : v;     // not read unless live
      body.gamma[i] = live ? gamma[k] : T(0); body.sigma[i] = live ? sigma[k] : T(0); body.omega[i] = live ? omega[k] : T(0);
    }
    launch_stream<T, 0>(ws.ctx, ws.n, body, NoFin());
  }
}

// The Golub-Kahan-like half of CGLS-Lanczos-shift, M = I, A and A^T CSR operators.  The u vectors stay unscaled until
// read: ws.u holds ũ_k = β_k u_k, and the u pass forms u_k = (1/β_k) ũ_k, the reference's kdiv!(m, u_next, β) of the
// previous iteration, with the same product.
template <class T> struct ShiftGkState { T uu, vv; };
template <class T> struct ShiftGkAvEpi {           // u_next = A v ; <u_next, u_next>
  T* un;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const { un[row] = acc; d[0] += acc * acc; }
};
template <class T> struct ShiftGkUBody {           // u_k = s_u ũ_k ; u_next -= delta u_k ; u_next -= beta u_prev ; u_prev = u_k
  T* un; const T* ut; T* up; T s_u; T delta; T beta;
  __device__ __forceinline__ void operator()(int j, T*) const {
    const T uk = mul_rn(s_u, ut[j]);
    T t = add_rn(un[j], mul_rn(-delta, uk));
    t = add_rn(t, mul_rn(-beta, up[j]));
    un[j] = t;
    up[j] = uk;
  }
};
template <class T> struct ShiftGkAtuEpi {          // v = A^T u_next ; <v, v>
  T* v;
  __device__ __forceinline__ void operator()(int row, T acc, T* d) const { v[row] = acc; d[0] += acc * acc; }
};
template <class T> struct ShiftGkFin {
  T* dst;
  __device__ void operator()(const T* tot) const { *dst = tot[0]; }
};
template <class T> T shift_gk_delta(Workspace<T>& ws, const Csr<T>& A) {
  StateBlock<ShiftGkState, T> sb(ws);
  launch_spmv_epi<T, 1>(ws.ctx, A, ws.v, ShiftGkAvEpi<T>{ws.u_next}, ShiftGkFin<T>{&sb.dev->uu});
  return sb.read().uu;
}
template <class T> T shift_gk_next(Workspace<T>& ws, const Csr<T>& At, T s_u, T delta, T beta) {
  StateBlock<ShiftGkState, T> sb(ws);
  launch_stream<T, 0>(ws.ctx, ws.m, ShiftGkUBody<T>{ws.u_next, ws.u, ws.u_prev, s_u, delta, beta}, NoFin());
  launch_spmv_epi<T, 1>(ws.ctx, At, ws.u_next, ShiftGkAtuEpi<T>{ws.v}, ShiftGkFin<T>{&sb.dev->vv});
  return sb.read().vv;
}

int gmres_fused_max() { return kGmresMaxFused; }

#define INST(T)                                                                                                      \
  template void bicgstab_fused_iteration<T>(Workspace<T>&, const Csr<T>&, const T*, bool, T, T*, T*, T*, T*);         \
  template void minres_fused_lanczos<T>(Workspace<T>&, const Csr<T>&, int, T, T, T, T, T, T, T, T*, T*, T*);          \
  template T minres_fused_update<T>(Workspace<T>&, T*, T, T);                                                        \
  template void gmres_fused_arnoldi<T>(Workspace<T>&, const Csr<T>&, int, T*, T*, const T*);                         \
  template void fused_orth_chain<T>(Workspace<T>&, const Csr<T>&, const T*, T*, const T* const*, int, T*, T*);       \
  template void trunc_fused_direction<T>(Workspace<T>&, T*, int, T* const*, const T*, const T*, T, T);               \
  template T cgs_fused_sigma<T>(Workspace<T>&, const Csr<T>&, const T*);                                             \
  template void cgs_fused_update<T>(Workspace<T>&, const Csr<T>&, const T*, T, T*, T*);                              \
  template void cgs_fused_directions<T>(Workspace<T>&, T);                                                           \
  template T lanczos_fused_delta<T>(Workspace<T>&, const Csr<T>&);                                                   \
  template T lanczos_fused_recur<T>(Workspace<T>&, T, T, bool);                                                      \
  template void lanczos_fused_update<T>(Workspace<T>&, T, T, T, T);                                                  \
  template void cr_fused_step<T>(Workspace<T>&, const Csr<T>&, T, T*, T*, T*, T*);                                   \
  template T cr_fused_directions<T>(Workspace<T>&, T);                                                               \
  template void fused_multi_axpy<T>(Workspace<T>&, T*, int, const T*, T* const*);                                    \
  template void lsq_fused_bidiag<T>(Workspace<T>&, const Csr<T>&, const Csr<T>&, bool, T, bool, T*, T*, T*);        \
  template T lsq_fused_update<T>(Workspace<T>&, bool, bool, T, T, T, T);                                             \
  template void lslq_fused_update<T>(Workspace<T>&, bool, T, T, T, T, T);                                          \
  template void cgls_fused_iteration<T>(Workspace<T>&, const Csr<T>&, const Csr<T>&, bool, T, T, T*, T*);            \
  template void crls_fused_iteration<T>(Workspace<T>&, const Csr<T>&, const Csr<T>&, bool, T, T, T, T*, T*, T*, T*);   \
  template void biorth_fused_lanczos<T>(Workspace<T>&, const Csr<T>&, const Csr<T>&, T, T, T*, T*);                  \
  template T qmr_fused_update<T>(Workspace<T>&, T*, const T*, int, T, T, T, T, T, T, bool);                          \
  template void bilq_fused_update<T>(Workspace<T>&, bool, T, T, T, T, T, T, bool, T*, T*);                           \
  template void car_fused_step<T>(Workspace<T>&, T, T*, T*);                                                         \
  template void car_fused_directions<T>(Workspace<T>&, const Csr<T>&, T, T*, T*);                                    \
  template void minares_fused_lanczos<T>(Workspace<T>&, const Csr<T>&, bool, int, T*, const T*, T*, const T*, T, T, T, T, T, \
                                         T*, T*);                                                                    \
  template void minares_fused_update<T>(Workspace<T>&, int, T*, bool, T, T*, const T*, const T*, T, T, T, T);       \
  template void bilqr_fused_update<T>(Workspace<T>&, bool, bool, int, T, T, T, T, T*, const T*, T, T, T, T, T, T, bool, T*); \
  template void trilqr_fused_ssy<T>(Workspace<T>&, const Csr<T>&, const Csr<T>&, bool, T, T, T*, T*, T*);             \
  template void trilqr_fused_update<T>(Workspace<T>&, bool, bool, int, T, T, T, T, T*, const T*, T, T, T, T, T, T); \
  template T craig_fused_p1<T>(Workspace<T>&, const Csr<T>&, bool, T, T, bool, T);                                 \
  template void craig_fused_p2<T>(Workspace<T>&, const Csr<T>&, T, T, T, T, T*, T*);                              \
  template void craig_fused_flush<T>(Workspace<T>&, T, T);                                                         \
  template T craigmr_fused_p1<T>(Workspace<T>&, const Csr<T>&, bool, T, T);                                         \
  template T craigmr_fused_p23<T>(Workspace<T>&, const Csr<T>&, bool, T, T, T, T, T, T, T);                        \
  template T lnlq_fused_l1<T>(Workspace<T>&, const Csr<T>&, bool, T, T, bool, T, T, T, T);                          \
  template T lnlq_fused_l2<T>(Workspace<T>&, const Csr<T>&, T, T, T);                                               \
  template void lnlq_fused_flush<T>(Workspace<T>&, T, T, T, T, T);                                                  \
  template void lnlq_fused_xup<T>(Workspace<T>&, T, T);                                                           \
  template void cgne_fused_iteration<T>(Workspace<T>&, const Csr<T>&, const Csr<T>&, bool, T, T, T*, T*);          \
  template void crmr_fused_iteration<T>(Workspace<T>&, const Csr<T>&, const Csr<T>&, bool, T, T*, T*);          \
  template void proc_spmv<T>(Ctx&, const Csr<T>&, const T*, const T*, const ProcEpi<T>&, const ProcFin<T>&);       \
  template void proc_stream<T>(Ctx&, int, const ProcUpdBody<T>&, const ProcFin<T>&);                                \
  template void proc_divide<T>(Ctx&, const ProcDivBody<T>&);                                                         \
  template void shift_fused_update<T>(Workspace<T>&, T*, bool, T, int, T* const*, T* const*, const T*, const T*, const T*); \
  template T shift_gk_delta<T>(Workspace<T>&, const Csr<T>&);                                                        \
  template T shift_gk_next<T>(Workspace<T>&, const Csr<T>&, T, T, T);
INST(double)
INST(float)
#undef INST

}  // namespace kb
