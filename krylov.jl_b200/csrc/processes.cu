// processes.cu -- the Krylov processes of src/krylov_processes.jl on CSR operators: hermitian_lanczos, arnoldi,
// golub_kahan, nonhermitian_lanczos and saunders_simon_yip (DESIGN.md §3i).
//
// A process has no stopping test, so a call enqueues all k steps back to back and synchronises once.  Every
// coefficient goes from one pass to the next in the call's device block (ProcHead, then the nzval arrays), where the
// fins write them and the gathers and epilogues read them.  Each normalisation kdivcopy!(v, q, β) stays pending: the
// next SpMV gathers q / β (ProcXDiv) and its epilogue stores the divided column for its own rows, so the column is
// never rewritten and no launch stores into the vector it gathers.  Arithmetic is the reference's, operation by
// operation (kb_internal.h: ProcEpi, ProcUpdBody); the first exact breakdown is recorded on the device and raised
// here, after the one read-back, with the reference's message.
#include <cstring>
#include <initializer_list>
#include <stdexcept>

#include "kb_internal.h"

namespace kb {

namespace {

constexpr int kAllowBreakdown = 1, kReorth = 2;

// The per-call device block (head + coefficients) and the scratch vectors, carved from the context's process buffer
// (Ctx::proc_scratch, grown when a call needs more and kept for the next call), and the one read-back.
template <class T> struct ProcCall {
  static constexpr size_t kAlign = 256;
  Ctx& c;
  size_t ncoef, head_bytes, bytes;
  char* dev = nullptr;
  std::vector<char> host;
  std::vector<T*> vecs;
  ProcHead<T>* h;
  T* coef;
  static size_t up(size_t b) { return (b + kAlign - 1) & ~(kAlign - 1); }
  ProcCall(Ctx& ctx, size_t nc, std::initializer_list<size_t> lens) : c(ctx), ncoef(nc) {
    head_bytes = (sizeof(ProcHead<T>) + 15) & ~size_t(15);
    bytes = head_bytes + nc * sizeof(T);
    size_t total = up(bytes);
    for (size_t n : lens) total += up(n * sizeof(T));
    if (c.proc_scratch_bytes < total) {         // cudaFree waits for the device: only when the buffer grows
      dev_free(c.proc_scratch);
      c.proc_scratch = nullptr;
      c.proc_scratch_bytes = 0;
      c.proc_scratch = dev_alloc<char>(total);
      c.proc_scratch_bytes = total;
    }
    dev = static_cast<char*>(c.proc_scratch);
    size_t off = up(bytes);
    for (size_t n : lens) { vecs.push_back(reinterpret_cast<T*>(dev + off)); off += up(n * sizeof(T)); }
    h = reinterpret_cast<ProcHead<T>*>(dev);
    coef = reinterpret_cast<T*>(dev + head_bytes);
    host.assign(bytes, 0);                      // zero coefficients, as the reference's zeros(R, ...)
    ProcHead<T> h0{};
    h0.one = T(1);
    std::memcpy(host.data(), &h0, sizeof(h0));
    KB_CUDA(cudaMemcpyAsync(dev, host.data(), bytes, cudaMemcpyHostToDevice, c.stream));
  }
  // the one device-to-host copy of the call
  const ProcHead<T>& read() {
    KB_CUDA(cudaMemcpyAsync(host.data(), dev, bytes, cudaMemcpyDeviceToHost, c.stream));
    c.sync();
    return *reinterpret_cast<const ProcHead<T>*>(host.data());
  }
  T coef_host(size_t i) const { T v; std::memcpy(&v, host.data() + head_bytes + i * sizeof(T), sizeof(T)); return v; }
  void coefs_out(double* out, size_t off, size_t cnt) const { for (size_t i = 0; i < cnt; i++) out[i] = (double)coef_host(off + i); }
  ProcFin<T> fin(int mode, T* d0, T* d1 = nullptr, T* d2 = nullptr, T* d3 = nullptr, int kind = 0, int iter = 0) const {
    ProcFin<T> f{};
    f.h = h; f.dst[0] = d0; f.dst[1] = d1; f.dst[2] = d2; f.dst[3] = d3;
    f.mode = mode; f.kind = kind; f.iter = iter;
    return f;
  }
  // ‖x‖ (or <x, y>) of an input vector into *dst
  void norm_of(int n, const T* x, const T* y, int mode, T* d0, T* d1, int kind) {
    ProcUpdBody<T> body{const_cast<T*>(x), nullptr, nullptr, y};   // no update: x is only read
    proc_stream<T>(c, n, body, fin(mode, d0, d1, nullptr, nullptr, kind, 0));
  }
};

template <class T> ProcEpi<T> epi() { ProcEpi<T> e{}; return e; }

void check_k(int k) { if (k < 1) throw std::runtime_error("k must be at least 1 (got " + std::to_string(k) + ")"); }

// The reference's error for breakdown kind `kind` (1-based into msgs) at iteration `iter`.
[[noreturn]] void breakdown(const char* const* msgs, int kind, int iter) {
  std::string m = msgs[kind - 1];
  const size_t at = m.find("%d");
  if (at != std::string::npos) m.replace(at, 2, std::to_string(iter));
  throw std::runtime_error(m);
}

template <class T> T* col(T* V, size_t ld, int j) { return V + ld * (size_t)(j - 1); }   // column j (1-based)

}  // namespace

// hermitian_lanczos (krylov_processes.jl:28-103).  Per step: L1 SpMV q = A v_i - β_i v_{i-1} with α_i = <v_i, q>;
// L2 q -= α_i v_i with β_{i+1} = ‖q‖.  Local reorthogonalization adds one pass per term it removes.
template <class T> void hermitian_lanczos_run(Ctx& c, const Csr<T>& A, int k, const T* b, T* V, double* beta, double* coef, int flags) {
  static const char* const msgs[] = {"Exact breakdown β₁ == 0.", "Exact breakdown βᵢ₊₁ == 0 at iteration i = %d."};
  check_k(k);
  const int n = A.n;
  const size_t ld = (size_t)n;
  ProcCall<T> P(c, 3 * (size_t)k - 1, {ld, ld});
  T* Q[2] = {P.vecs[0], P.vecs[1]};
  T* nz = P.coef;
  P.norm_of(n, b, nullptr, ProcFin<T>::NORM, &P.h->beta1, nullptr, 1);
  for (int i = 1; i <= k; i++) {
    const size_t pa = 3 * (size_t)(i - 1);          // position of αᵢ in nzval (0-based)
    T* q = Q[i % 2];
    const T* src = i == 1 ? b : Q[(i - 1) % 2];
    const T* div = i == 1 ? &P.h->beta1 : &nz[pa - 2];
    T* vi = col(V, ld, i);
    ProcEpi<T> e = epi<T>();
    e.src = src; e.src_s = div; e.vout = vi; e.qout = q; e.dot = 0;
    ProcFin<T> f = P.fin(ProcFin<T>::SET, &nz[pa]);
    if (i >= 2) {
      e.w1 = col(V, ld, i - 1); e.s1 = &nz[pa - 2];
      f.copy_src = &nz[pa - 2]; f.copy_dst = &nz[pa - 1];   // Tᵢ₋₁.ᵢ = βᵢ
    }
    proc_spmv<T>(c, A, src, div, e, f);
    if (flags & kReorth) {
      if (i >= 2) {
        proc_stream<T>(c, n, ProcUpdBody<T>{q, vi, &nz[pa], col(V, ld, i - 1)}, P.fin(ProcFin<T>::ACC, &nz[pa - 2], &nz[pa - 1]));
        proc_stream<T>(c, n, ProcUpdBody<T>{q, col(V, ld, i - 1), &P.h->tmp, vi}, P.fin(ProcFin<T>::ACC, &nz[pa]));
      } else {
        proc_stream<T>(c, n, ProcUpdBody<T>{q, vi, &nz[pa], vi}, P.fin(ProcFin<T>::ACC, &nz[pa]));
      }
      proc_stream<T>(c, n, ProcUpdBody<T>{q, vi, &P.h->tmp, nullptr}, P.fin(ProcFin<T>::NORM, &nz[pa + 1], nullptr, nullptr, nullptr, 2, i));
    } else {
      proc_stream<T>(c, n, ProcUpdBody<T>{q, vi, &nz[pa], nullptr}, P.fin(ProcFin<T>::NORM, &nz[pa + 1], nullptr, nullptr, nullptr, 2, i));
    }
  }
  const size_t plast = 3 * (size_t)(k - 1);
  proc_divide<T>(c, ProcDivBody<T>{col(V, ld, k + 1), Q[k % 2], &nz[plast + 1], n, nullptr, nullptr, nullptr, 0});
  const ProcHead<T>& h = P.read();
  if (h.brk_kind && !(flags & kAllowBreakdown)) breakdown(msgs, h.brk_kind, h.brk_iter);
  *beta = (double)h.beta1;
  P.coefs_out(coef, 0, P.ncoef);
}

// arnoldi (krylov_processes.jl:250-296), modified Gram-Schmidt.  Step j: A1 SpMV q = A v_j with H₁.ⱼ = <v_1, q>, then
// for i = 2..j a pass q -= Hᵢ₋₁.ⱼ vᵢ₋₁ with Hᵢ.ⱼ = <v_i, q>, and q -= Hⱼ.ⱼ v_j with Hⱼ₊₁.ⱼ = ‖q‖: j + 1 launches
// (full reorthogonalization: j more).
template <class T> void arnoldi_run(Ctx& c, const Csr<T>& A, int k, const T* b, T* V, double* beta, double* Hout, int flags) {
  static const char* const msgs[] = {"Exact breakdown β == 0.", "Exact breakdown Hᵢ₊₁.ᵢ == 0 at iteration i = %d."};
  check_k(k);
  const int n = A.n;
  const size_t ld = (size_t)n, hk = (size_t)k + 1;
  ProcCall<T> P(c, hk * (size_t)k, {ld, ld});
  T* Q[2] = {P.vecs[0], P.vecs[1]};
  auto H = [&](int i, int j) { return P.coef + (size_t)(i - 1) + (size_t)(j - 1) * hk; };
  P.norm_of(n, b, nullptr, ProcFin<T>::NORM, &P.h->beta1, nullptr, 1);
  for (int j = 1; j <= k; j++) {
    T* q = Q[j % 2];
    const T* src = j == 1 ? b : Q[(j - 1) % 2];
    const T* div = j == 1 ? &P.h->beta1 : H(j, j - 1);
    ProcEpi<T> e = epi<T>();
    e.src = src; e.src_s = div; e.vout = col(V, ld, j); e.qout = q;
    e.dot = j == 1 ? 0 : 3; e.y = col(V, ld, 1);
    proc_spmv<T>(c, A, src, div, e, P.fin(ProcFin<T>::SET, H(1, j)));
    for (int i = 2; i <= j; i++)
      proc_stream<T>(c, n, ProcUpdBody<T>{q, col(V, ld, i - 1), H(i - 1, j), col(V, ld, i)}, P.fin(ProcFin<T>::SET, H(i, j)));
    const T* last = H(j, j);
    if (flags & kReorth) {
      proc_stream<T>(c, n, ProcUpdBody<T>{q, col(V, ld, j), last, col(V, ld, 1)}, P.fin(ProcFin<T>::ACC, H(1, j)));
      for (int i = 2; i <= j; i++)
        proc_stream<T>(c, n, ProcUpdBody<T>{q, col(V, ld, i - 1), &P.h->tmp, col(V, ld, i)}, P.fin(ProcFin<T>::ACC, H(i, j)));
      last = &P.h->tmp;
    }
    proc_stream<T>(c, n, ProcUpdBody<T>{q, col(V, ld, j), last, nullptr},
                   P.fin(ProcFin<T>::NORM, H(j + 1, j), nullptr, nullptr, nullptr, 2, j));
  }
  proc_divide<T>(c, ProcDivBody<T>{col(V, ld, k + 1), Q[k % 2], H(k + 1, k), n, nullptr, nullptr, nullptr, 0});
  const ProcHead<T>& h = P.read();
  if (h.brk_kind && !(flags & kAllowBreakdown)) breakdown(msgs, h.brk_kind, h.brk_iter);
  *beta = (double)h.beta1;
  P.coefs_out(Hout, 0, P.ncoef);
}

// golub_kahan (krylov_processes.jl:323-402), A m x n with At = Aᵀ.  Set-up: β₁ = ‖b‖, then an SpMV on Aᵀ gathering
// b / β₁ for α₁.  Step i: G1 SpMV on A gathering p / αᵢ (v_i) stores u_i = q / βᵢ and forms q = A v_i - αᵢ u_i with
// βᵢ₊₁ = ‖q‖; G2 SpMV on Aᵀ gathering q / βᵢ₊₁ (u_{i+1}) stores v_i = p / αᵢ and forms p = Aᵀu_{i+1} - βᵢ₊₁ v_i with
// αᵢ₊₁ = ‖p‖.  The two SpMVs gather different spaces, so q and p need no second buffer.
template <class T> void golub_kahan_run(Ctx& c, const Csr<T>& A, const Csr<T>& At, int k, const T* b, T* V, T* U, double* beta,
                                        double* coef, int flags) {
  static const char* const msgs[] = {"Exact breakdown β₁ == 0.", "Exact breakdown α₁ == 0.",
                                     "Exact breakdown βᵢ₊₁ == 0 at iteration i = %d.", "Exact breakdown αᵢ₊₁ == 0 at iteration i = %d."};
  check_k(k);
  const int m = A.n, n = A.ncols;
  ProcCall<T> P(c, 2 * (size_t)k + 1, {(size_t)m, (size_t)n});
  T* q = P.vecs[0];
  T* p = P.vecs[1];
  T* nz = P.coef;
  P.norm_of(m, b, nullptr, ProcFin<T>::NORM, &P.h->beta1, nullptr, 1);
  {
    ProcEpi<T> e = epi<T>();
    e.qout = p; e.dot = 1;
    proc_spmv<T>(c, At, b, &P.h->beta1, e, P.fin(ProcFin<T>::NORM, &nz[0], nullptr, nullptr, nullptr, 2, 0));
  }
  for (int i = 1; i <= k; i++) {
    const size_t pa = 2 * (size_t)(i - 1);
    ProcEpi<T> e1 = epi<T>();
    e1.src = i == 1 ? b : q; e1.src_s = i == 1 ? &P.h->beta1 : &nz[pa - 1]; e1.vout = col(U, (size_t)m, i);
    e1.s1 = &nz[pa]; e1.qout = q; e1.dot = 1;
    proc_spmv<T>(c, A, p, &nz[pa], e1, P.fin(ProcFin<T>::NORM, &nz[pa + 1], nullptr, nullptr, nullptr, 3, i));
    ProcEpi<T> e2 = epi<T>();
    e2.src = p; e2.src_s = &nz[pa]; e2.vout = col(V, (size_t)n, i);
    e2.s1 = &nz[pa + 1]; e2.qout = p; e2.dot = 1;
    proc_spmv<T>(c, At, q, &nz[pa + 1], e2, P.fin(ProcFin<T>::NORM, &nz[pa + 2], nullptr, nullptr, nullptr, 4, i));
  }
  const size_t plast = 2 * (size_t)(k - 1);
  proc_divide<T>(c, ProcDivBody<T>{col(U, (size_t)m, k + 1), q, &nz[plast + 1], m, col(V, (size_t)n, k + 1), p, &nz[plast + 2], n});
  const ProcHead<T>& h = P.read();
  if (h.brk_kind && !(flags & kAllowBreakdown)) breakdown(msgs, h.brk_kind, h.brk_iter);
  *beta = (double)h.beta1;
  P.coefs_out(coef, 0, P.ncoef);
}

// nonhermitian_lanczos (krylov_processes.jl:133-224), square A with At = Aᵀ.  Step i: N1 SpMV on A gathering
// q / βᵢ (v_i) stores v_i and u_i = p / γᵢ, forms q = A v_i - γᵢ v_{i-1} and αᵢ = <u_i, q>; N2 SpMV on Aᵀ gathering
// the stored u_i forms p = Aᵀu_i - βᵢ u_{i-1} - αᵢ u_i and q -= αᵢ v_i with pᴴq, from which βᵢ₊₁ and γᵢ₊₁ follow on
// the device.  q, which N1 gathers while it writes the next one, alternates between two buffers.
template <class T> void nonhermitian_lanczos_run(Ctx& c, const Csr<T>& A, const Csr<T>& At, int k, const T* b, const T* cv, T* V,
                                                 T* U, double* beta, double* gamma, double* coefT, double* coefTH, int flags) {
  static const char* const msgs[] = {"Exact breakdown β₁γ₁ == 0.", "Exact breakdown βᵢ₊₁γᵢ₊₁ == 0 at iteration i = %d."};
  check_k(k);
  const int n = A.n;
  const size_t ld = (size_t)n, nc = 3 * (size_t)k - 1;
  ProcCall<T> P(c, 2 * nc, {ld, ld, ld});
  T* Q[2] = {P.vecs[0], P.vecs[1]};
  T* p = P.vecs[2];
  T* Tn = P.coef;
  T* Th = P.coef + nc;
  P.norm_of(n, cv, b, ProcFin<T>::BIORTH, &P.h->beta1, &P.h->gamma1, 1);   // cᴴb
  for (int i = 1; i <= k; i++) {
    const size_t pa = 3 * (size_t)(i - 1);
    T* q = Q[i % 2];
    const T* srcv = i == 1 ? b : Q[(i - 1) % 2];
    const T* divv = i == 1 ? &P.h->beta1 : &Tn[pa - 2];
    T* vi = col(V, ld, i);
    T* ui = col(U, ld, i);
    ProcEpi<T> e1 = epi<T>();
    e1.src = srcv; e1.src_s = divv; e1.vout = vi; e1.qout = q;
    e1.src2 = i == 1 ? cv : p; e1.src2_s = i == 1 ? &P.h->gamma1 : &Th[pa - 2]; e1.vout2 = ui; e1.dot = 2;
    if (i >= 2) { e1.w1 = col(V, ld, i - 1); e1.s1 = &Tn[pa - 1]; }
    proc_spmv<T>(c, A, srcv, divv, e1, P.fin(ProcFin<T>::SET, &Tn[pa], &Th[pa]));
    ProcEpi<T> e2 = epi<T>();
    if (i >= 2) { e2.w1 = col(U, ld, i - 1); e2.s1 = &Tn[pa - 2]; }
    e2.w2 = ui; e2.s2 = &Tn[pa]; e2.qout = p;
    e2.r = q; e2.rx = vi; e2.rs = &Tn[pa]; e2.dot = 4;
    const bool inner = i <= k - 1;
    proc_spmv<T>(c, At, ui, &P.h->one, e2,
                 P.fin(ProcFin<T>::BIORTH, &Tn[pa + 1], &Th[pa + 1], inner ? &Tn[pa + 2] : nullptr, inner ? &Th[pa + 2] : nullptr, 2, i));
  }
  const size_t plast = 3 * (size_t)(k - 1);
  proc_divide<T>(c, ProcDivBody<T>{col(V, ld, k + 1), Q[k % 2], &Tn[plast + 1], n, col(U, ld, k + 1), p, &Th[plast + 1], n});
  const ProcHead<T>& h = P.read();
  if (h.brk_kind && !(flags & kAllowBreakdown)) breakdown(msgs, h.brk_kind, h.brk_iter);
  *beta = (double)h.beta1;
  *gamma = (double)h.gamma1;
  P.coefs_out(coefT, 0, nc);
  P.coefs_out(coefTH, nc, nc);
}

// saunders_simon_yip (krylov_processes.jl:431-524), A m x n with At = Aᵀ.  Step i: S1 SpMV on A gathering p / γᵢ (u_i)
// stores v_i = q / βᵢ and forms q = A u_i - γᵢ v_{i-1} with αᵢ = <v_i, q>; S3 q -= αᵢ v_i with βᵢ₊₁ = ‖q‖ (over m);
// S2 SpMV on Aᵀ gathering the stored v_i stores u_i = p / γᵢ and forms p = Aᵀv_i - βᵢ u_{i-1} - αᵢ u_i with
// γᵢ₊₁ = ‖p‖.  S3 runs before S2 so that the breakdowns are met in the reference's order.
template <class T> void saunders_simon_yip_run(Ctx& c, const Csr<T>& A, const Csr<T>& At, int k, const T* b, const T* cv, T* V,
                                               T* U, double* beta, double* gamma, double* coefT, double* coefTH, int flags) {
  static const char* const msgs[] = {"Exact breakdown β₁ == 0.", "Exact breakdown γ₁ᴴ == 0.",
                                     "Exact breakdown βᵢ₊₁ == 0 at iteration i = %d.", "Exact breakdown γᵢ₊₁ == 0 at iteration i = %d."};
  check_k(k);
  const int m = A.n, n = A.ncols;
  const size_t nc = 3 * (size_t)k - 1;
  ProcCall<T> P(c, 2 * nc, {(size_t)m, (size_t)n});
  T* q = P.vecs[0];
  T* p = P.vecs[1];
  T* Tn = P.coef;
  T* Th = P.coef + nc;
  P.norm_of(m, b, nullptr, ProcFin<T>::NORM, &P.h->beta1, nullptr, 1);
  P.norm_of(n, cv, nullptr, ProcFin<T>::NORM, &P.h->gamma1, nullptr, 2);
  for (int i = 1; i <= k; i++) {
    const size_t pa = 3 * (size_t)(i - 1);
    const bool inner = i <= k - 1;
    T* vi = col(V, (size_t)m, i);
    const T* srcu = i == 1 ? cv : p;
    const T* divu = i == 1 ? &P.h->gamma1 : &Th[pa - 2];
    ProcEpi<T> e1 = epi<T>();
    e1.src = i == 1 ? b : q; e1.src_s = i == 1 ? &P.h->beta1 : &Tn[pa - 2]; e1.vout = vi; e1.qout = q; e1.dot = 0;
    if (i >= 2) { e1.w1 = col(V, (size_t)m, i - 1); e1.s1 = &Tn[pa - 1]; }
    proc_spmv<T>(c, A, srcu, divu, e1, P.fin(ProcFin<T>::SET, &Tn[pa], &Th[pa]));
    proc_stream<T>(c, m, ProcUpdBody<T>{q, vi, &Tn[pa], nullptr},
                   P.fin(ProcFin<T>::NORM, &Tn[pa + 1], inner ? &Th[pa + 2] : nullptr, nullptr, nullptr, 3, i));
    ProcEpi<T> e2 = epi<T>();
    e2.src = srcu; e2.src_s = divu; e2.vout = col(U, (size_t)n, i);
    if (i >= 2) { e2.w1 = col(U, (size_t)n, i - 1); e2.s1 = &Tn[pa - 2]; }
    e2.s2 = &Tn[pa]; e2.qout = p; e2.dot = 1;
    proc_spmv<T>(c, At, vi, &P.h->one, e2,
                 P.fin(ProcFin<T>::NORM, &Th[pa + 1], inner ? &Tn[pa + 2] : nullptr, nullptr, nullptr, 4, i));
  }
  const size_t plast = 3 * (size_t)(k - 1);
  proc_divide<T>(c, ProcDivBody<T>{col(V, (size_t)m, k + 1), q, &Tn[plast + 1], m, col(U, (size_t)n, k + 1), p, &Th[plast + 1], n});
  const ProcHead<T>& h = P.read();
  if (h.brk_kind && !(flags & kAllowBreakdown)) breakdown(msgs, h.brk_kind, h.brk_iter);
  *beta = (double)h.beta1;
  *gamma = (double)h.gamma1;
  P.coefs_out(coefT, 0, nc);
  P.coefs_out(coefTH, nc, nc);
}

#define INST(T)                                                                                                         \
  template void hermitian_lanczos_run<T>(Ctx&, const Csr<T>&, int, const T*, T*, double*, double*, int);                \
  template void arnoldi_run<T>(Ctx&, const Csr<T>&, int, const T*, T*, double*, double*, int);                          \
  template void golub_kahan_run<T>(Ctx&, const Csr<T>&, const Csr<T>&, int, const T*, T*, T*, double*, double*, int);    \
  template void nonhermitian_lanczos_run<T>(Ctx&, const Csr<T>&, const Csr<T>&, int, const T*, const T*, T*, T*, double*, \
                                            double*, double*, double*, int);                                           \
  template void saunders_simon_yip_run<T>(Ctx&, const Csr<T>&, const Csr<T>&, int, const T*, const T*, T*, T*, double*,  \
                                          double*, double*, double*, int);
INST(double)
INST(float)
#undef INST

}  // namespace kb
