// blas1.cu -- device implementations of Krylov.jl's vector primitives
// (src/krylov_utils.jl:309-349): kdot/kdotr, knorm, kscal!, kdiv!, kcopy!,
// kscalcopy!, kdivcopy!, kaxpy!, kaxpby!, kfill!.
//
// All kernels are HBM-bound streaming passes: grid = whole CTAs per SM,
// grid-stride loops with 4 independent elements in flight per thread.
// Element updates use non-contracted mul/add so they agree bit-for-bit with
// the reference's `y[i] += s*x[i]` (Julia does not fuse); reductions are
// deterministic two-stage tree sums finalised by the last CTA on the device.
#include <cmath>
#include <limits>
#include <mutex>
#include <set>
#include <utility>

#include "kb_internal.h"

#include <chrono>

namespace kb {

void ensure_dyn_smem(const void* func, int bytes) {
  static std::mutex mu;
  static std::set<std::pair<const void*, int>> done;
  int dev = 0;
  KB_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lk(mu);
  if (done.count({func, dev})) return;
  KB_CUDA(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  done.insert({func, dev});
}

double now_seconds() {
  using namespace std::chrono;
  return duration_cast<duration<double>>(steady_clock::now().time_since_epoch()).count();
}

// ---------------------------------------------------------------------------
void Ctx::init(int dev) {
  device = dev;
  KB_CUDA(cudaSetDevice(dev));
  KB_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  own_stream = true;
  KB_CUDA(cudaMalloc(&partials, sizeof(double) * kMaxPartials * 4));
  KB_CUDA(cudaMalloc((void**)&tickets, sizeof(unsigned) * 8));
  KB_CUDA(cudaMemset(tickets, 0, sizeof(unsigned) * 8));
  KB_CUDA(cudaMalloc(&dscal, sizeof(double) * 16));
  KB_CUDA(cudaMemset(dscal, 0, sizeof(double) * 16));
  KB_CUDA(cudaHostAlloc(&hscal, sizeof(double) * 16, cudaHostAllocDefault));
}

void Ctx::destroy() {
  if (partials) cudaFree(partials);
  if (tickets) cudaFree(tickets);
  if (dscal) cudaFree(dscal);
  if (hscal) cudaFreeHost(hscal);
  if (proc_scratch) cudaFree(proc_scratch);
  if (own_stream && stream) cudaStreamDestroy(stream);
  partials = nullptr; tickets = nullptr; dscal = nullptr; hscal = nullptr; stream = nullptr;
  proc_scratch = nullptr; proc_scratch_bytes = 0;
}

template <class T> T* dev_alloc(size_t n) {
  void* p = nullptr;
  KB_CUDA(cudaMalloc(&p, n * sizeof(T) + 64));   // 64 B tail pad: TMA tiles may over-read up to 16 B
  return (T*)p;
}
void dev_free(void* p) { if (p) cudaFree(p); }
template double* dev_alloc<double>(size_t);
template float* dev_alloc<float>(size_t);
template int* dev_alloc<int>(size_t);
template char* dev_alloc<char>(size_t);

// ---------------------------------------------------------------------------
// Elementwise kernels
// ---------------------------------------------------------------------------
enum EwOp { EW_AXPY, EW_AXPBY, EW_SCAL, EW_COPY, EW_SCALCOPY, EW_DIVCOPY, EW_FILL, EW_DIAGMUL, EW_DIAGDIV };

// The grid-stride loops here count in unsigned 32-bit: n <= INT_MAX and stride <= kMaxPartials * kBlock = 2^19, so
// i + 3 * stride and every step stay below n + 4 * stride < 2^32.  In int they overflow once n is within 4 strides
// of INT_MAX (an 8 GiB Float32 vector fits on one GPU).  A negative n counts as 0 (un), as it did in int: the
// reductions still launch one CTA for n <= 0 to write their result.
template <class T, int OP>
__global__ void __launch_bounds__(kBlock) ew_kernel(int n, T s, T t, const T* x, const T* d, T* y) {
  const unsigned stride = gridDim.x * blockDim.x, un = n > 0 ? n : 0;
  unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  // 4 independent elements per trip keep enough loads in flight per thread.
  for (; i + 3 * stride < un; i += 4 * stride) {
    T xv[4], yv[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const unsigned j = i + u * stride;
      if (OP != EW_FILL && OP != EW_SCAL) xv[u] = x[j];
      if (OP == EW_AXPY || OP == EW_AXPBY || OP == EW_SCAL) yv[u] = y[j];
      if (OP == EW_DIAGMUL || OP == EW_DIAGDIV) yv[u] = d[j];
    }
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const unsigned j = i + u * stride;
      T r;
      if (OP == EW_AXPY) r = add_rn(yv[u], mul_rn(s, xv[u]));
      else if (OP == EW_AXPBY) r = add_rn(mul_rn(s, xv[u]), mul_rn(t, yv[u]));
      else if (OP == EW_SCAL) r = mul_rn(s, yv[u]);
      else if (OP == EW_COPY) r = xv[u];
      else if (OP == EW_SCALCOPY) r = mul_rn(s, xv[u]);
      else if (OP == EW_DIVCOPY) r = div_rn(xv[u], s);
      else if (OP == EW_FILL) r = s;
      else if (OP == EW_DIAGMUL) r = mul_rn(yv[u], xv[u]);
      else r = div_rn(xv[u], yv[u]);
      y[j] = r;
    }
  }
  for (; i < un; i += stride) {
    T r;
    if (OP == EW_AXPY) r = add_rn(y[i], mul_rn(s, x[i]));
    else if (OP == EW_AXPBY) r = add_rn(mul_rn(s, x[i]), mul_rn(t, y[i]));
    else if (OP == EW_SCAL) r = mul_rn(s, y[i]);
    else if (OP == EW_COPY) r = x[i];
    else if (OP == EW_SCALCOPY) r = mul_rn(s, x[i]);
    else if (OP == EW_DIVCOPY) r = div_rn(x[i], s);
    else if (OP == EW_FILL) r = s;
    else if (OP == EW_DIAGMUL) r = mul_rn(d[i], x[i]);
    else r = div_rn(x[i], d[i]);
    y[i] = r;
  }
}

template <class T, int OP>
static void ew_launch(Ctx& c, int n, T s, T t, const T* x, const T* d, T* y) {
  if (n <= 0) return;
  const int grid = stream_grid(n, 4, 8);
  ew_kernel<T, OP><<<grid, kBlock, 0, c.stream>>>(n, s, t, x, d, y);
  KB_CUDA(cudaGetLastError());
  c.launches++;
}

template <class T> void k_axpy(Ctx& c, int n, T s, const T* x, T* y) { ew_launch<T, EW_AXPY>(c, n, s, T(0), x, nullptr, y); }
template <class T> void k_axpby(Ctx& c, int n, T s, const T* x, T t, T* y) { ew_launch<T, EW_AXPBY>(c, n, s, t, x, nullptr, y); }
template <class T> void k_scal(Ctx& c, int n, T s, T* x) { ew_launch<T, EW_SCAL>(c, n, s, T(0), nullptr, nullptr, x); }
template <class T> void k_copy(Ctx& c, int n, T* y, const T* x) {
  if (n > 0 && y != x) KB_CUDA(cudaMemcpyAsync(y, x, sizeof(T) * (size_t)n, cudaMemcpyDeviceToDevice, c.stream));
}
template <class T> void k_scalcopy(Ctx& c, int n, T* y, T s, const T* x) { ew_launch<T, EW_SCALCOPY>(c, n, s, T(0), x, nullptr, y); }
template <class T> void k_divcopy(Ctx& c, int n, T* y, const T* x, T s) { ew_launch<T, EW_DIVCOPY>(c, n, s, T(0), x, nullptr, y); }
template <class T> void k_fill(Ctx& c, int n, T* x, T v) {
  if (n <= 0) return;
  if (v == T(0) && !std::signbit(v)) { KB_CUDA(cudaMemsetAsync(x, 0, sizeof(T) * (size_t)n, c.stream)); return; }   // -0.0 is not all-zero bits
  ew_launch<T, EW_FILL>(c, n, v, T(0), nullptr, nullptr, x);
}
template <class T> void k_diagmul(Ctx& c, int n, T* y, const T* d, const T* x, bool ldiv) {
  if (ldiv) ew_launch<T, EW_DIAGDIV>(c, n, T(0), T(0), x, d, y);
  else ew_launch<T, EW_DIAGMUL>(c, n, T(0), T(0), x, d, y);
}

// ---------------------------------------------------------------------------
// Block-Jacobi: y = blockdiag(B_0, B_1, ...) x with dense bs x bs blocks (row-major), bs in 2..8
// (docs/src/preconditioners.md:33 -- the operator handed to the solver is P^-1; SURVEY.md 8f-1).
// One thread per block; the row sums run left to right, non-contracted, like every k* primitive.
// ---------------------------------------------------------------------------
template <class T>
__global__ void __launch_bounds__(kBlock) blockdiag_mul_kernel(int n, int bs, const T* __restrict__ B, const T* __restrict__ x, T* __restrict__ y) {
  const int nb = (n + bs - 1) / bs;
  for (int blk = blockIdx.x * blockDim.x + threadIdx.x; blk < nb; blk += gridDim.x * blockDim.x) {
    const int r0 = blk * bs, rows = min(bs, n - r0);
    const T* Bk = B + (size_t)blk * bs * bs;
    T xv[8];
    for (int j = 0; j < rows; j++) xv[j] = x[r0 + j];
    for (int i = 0; i < rows; i++) {
      T acc = T(0);
      for (int j = 0; j < rows; j++) acc = add_rn(acc, mul_rn(Bk[i * bs + j], xv[j]));
      y[r0 + i] = acc;
    }
  }
}
template <class T> void k_blockdiag_mul(Ctx& c, int n, int bs, const T* blocks, const T* x, T* y) {
  if (n <= 0) return;
  blockdiag_mul_kernel<T><<<stream_grid((n + bs - 1) / bs, 1, 8), kBlock, 0, c.stream>>>(n, bs, blocks, x, y);
  KB_CUDA(cudaGetLastError());
  c.launches++;
}

// inverse of every diagonal block (Gauss-Jordan with partial pivoting, one thread per block): ldiv = true with a
// block-diagonal P applies these
template <class T>
__global__ void __launch_bounds__(kBlock) blockdiag_invert_kernel(int n, int bs, const T* __restrict__ B, T* __restrict__ Inv, int* singular) {
  const int nb = (n + bs - 1) / bs;
  for (int blk = blockIdx.x * blockDim.x + threadIdx.x; blk < nb; blk += gridDim.x * blockDim.x) {
    const int rows = min(bs, n - blk * bs);
    T a[8][16];
    for (int i = 0; i < rows; i++)
      for (int j = 0; j < rows; j++) { a[i][j] = B[(size_t)blk * bs * bs + i * bs + j]; a[i][rows + j] = i == j ? T(1) : T(0); }
    bool bad = false;
    for (int col = 0; col < rows; col++) {
      int piv = col;
      for (int i = col + 1; i < rows; i++) if (fabs(a[i][col]) > fabs(a[piv][col])) piv = i;
      if (a[piv][col] == T(0)) { bad = true; break; }
      if (piv != col) for (int j = 0; j < 2 * rows; j++) { const T t = a[col][j]; a[col][j] = a[piv][j]; a[piv][j] = t; }
      const T d = T(1) / a[col][col];
      for (int j = 0; j < 2 * rows; j++) a[col][j] *= d;
      for (int i = 0; i < rows; i++) {
        if (i == col) continue;
        const T f = a[i][col];
        for (int j = 0; j < 2 * rows; j++) a[i][j] -= f * a[col][j];
      }
    }
    if (bad) atomicExch(singular, 1);
    for (int i = 0; i < bs; i++)
      for (int j = 0; j < bs; j++) Inv[(size_t)blk * bs * bs + i * bs + j] = (!bad && i < rows && j < rows) ? a[i][rows + j] : T(0);
  }
}
template <class T> void k_blockdiag_invert(Ctx& c, int n, int bs, const T* blocks, T* inv, int* singular) {
  if (n <= 0) return;
  blockdiag_invert_kernel<T><<<stream_grid((n + bs - 1) / bs, 1, 4), kBlock, 0, c.stream>>>(n, bs, blocks, inv, singular);
  KB_CUDA(cudaGetLastError());
  c.launches++;
}

// ---------------------------------------------------------------------------
// Reductions
// ---------------------------------------------------------------------------
// DOT_SUM: out[k] = <a, b> (k = 0) and <u, v> (k = 1 when K = 2).  The two modes of k_nrm2 read only a:
// DOT_NRM2 sums a_i^2 and also leaves max|a_i| in out[1]; DOT_NRM2_SCALED sums (a_i 2^-e)^2, where 2^e <= max|a_i| < 2^(e+1)
// is taken from that out[1], and returns 2^e sqrt(sum).  do_sqrt: out[k] = sqrt(sum) instead of the sum.
enum DotMode { DOT_SUM, DOT_NRM2, DOT_NRM2_SCALED };

__device__ __forceinline__ double scale2(double v, int e) { return scalbn(v, e); }   // v 2^e, one rounding
__device__ __forceinline__ float scale2(float v, int e) { return scalbnf(v, e); }
__device__ __forceinline__ int exponent_of(double v) { return ilogb(v); }
__device__ __forceinline__ int exponent_of(float v) { return ilogbf(v); }

// Like block_sum, for the maximum (NaNs are ignored: fmax).  All threads of the CTA must call; valid in thread 0.
template <class T>
__device__ __forceinline__ T block_max(T v, T* smem) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  if (lane == 0) smem[w] = v;
  __syncthreads();
  T r = T(0);
  if (w == 0) {
    r = lane < nw ? smem[lane] : T(0);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r = fmax(r, __shfl_xor_sync(0xffffffffu, r, o));
  }
  __syncthreads();
  return r;
}

template <class T, int K, int MODE = DOT_SUM>
__global__ void __launch_bounds__(kBlock) dot_kernel(int n, const T* __restrict__ a, const T* __restrict__ b,
                                                     const T* __restrict__ u, const T* __restrict__ v, T* part,
                                                     unsigned* ticket, T* out, int do_sqrt, DistComm* dc) {
  static_assert(MODE == DOT_SUM || K == 1, "the nrm2 modes reduce one vector");
  __shared__ T sm[32];
  const unsigned stride = gridDim.x * blockDim.x, un = n > 0 ? n : 0;   // unsigned: see ew_kernel
  const int sh = MODE == DOT_NRM2_SCALED ? -exponent_of(out[1]) : 0;
  T acc[K], mx = T(0);
#pragma unroll
  for (int k = 0; k < K; k++) acc[k] = T(0);
  unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + 3 * stride < un; i += 4 * stride) {
    T av[4], bv[4], uv[4], vv[4];
#pragma unroll
    for (int q = 0; q < 4; q++) {
      av[q] = a[i + q * stride];
      if (MODE == DOT_NRM2_SCALED) av[q] = scale2(av[q], sh);
      bv[q] = MODE == DOT_SUM ? b[i + q * stride] : av[q];
      if (K > 1) { uv[q] = u[i + q * stride]; vv[q] = v[i + q * stride]; }
    }
#pragma unroll
    for (int q = 0; q < 4; q++) {
      acc[0] += av[q] * bv[q];
      if (K > 1) acc[K - 1] += uv[q] * vv[q];
      if (MODE == DOT_NRM2) mx = fmax(mx, fabs(av[q]));
    }
  }
  for (; i < un; i += stride) {
    if (MODE == DOT_SUM) acc[0] += a[i] * b[i];
    else {
      const T ai = MODE == DOT_NRM2_SCALED ? scale2(a[i], sh) : a[i];
      acc[0] += ai * ai;
      if (MODE == DOT_NRM2) mx = fmax(mx, fabs(ai));
    }
    if (K > 1) acc[K - 1] += u[i] * v[i];
  }
  T mine[K], tot[K];
#pragma unroll
  for (int k = 0; k < K; k++) {
    mine[k] = block_sum(acc[k], sm);
  }
  if (MODE == DOT_NRM2) {
    const T m = block_max(mx, sm);
    if (threadIdx.x == 0) part[gridDim.x + blockIdx.x] = m;   // after the sums' partials; grid_sum_last's fence covers it
  }
  if (grid_sum_last<T, K>(mine, part, ticket, sm, tot)) {
    T gmax = T(0);
    if (MODE == DOT_NRM2) {
      for (int j = threadIdx.x; j < (int)gridDim.x; j += blockDim.x) gmax = fmax(gmax, __ldcg(&part[gridDim.x + j]));
      gmax = block_max(gmax, sm);
    }
    if (threadIdx.x == 0) {
#pragma unroll
      for (int k = 0; k < K; k++) {
        const T g = dist_reduce(dc, tot[k]);       // row-partitioned solve: sum over ranks
        const T r = do_sqrt ? sqrt_rn(g) : g;
        out[k] = MODE == DOT_NRM2_SCALED ? scale2(r, -sh) : r;
      }
      if (MODE == DOT_NRM2) out[1] = gmax;
    }
  }
}

template <class T>
static T* slot_ptr(Ctx& c, int slot) { return reinterpret_cast<T*>(reinterpret_cast<double*>(c.dscal) + slot); }

template <class T>
static void dot_launch(Ctx& c, int n, const T* a, const T* b, int slot, int do_sqrt) {
  const int grid = n > 0 ? stream_grid(n, 4, 4) : 1;
  dot_kernel<T, 1><<<grid, kBlock, 0, c.stream>>>(n, a, b, nullptr, nullptr, (T*)c.partials, c.tickets, slot_ptr<T>(c, slot), do_sqrt, c.dcomm);
  KB_CUDA(cudaGetLastError());
  c.launches++;
}

template <class T>
static T read_slot(Ctx& c, int slot) {
  KB_CUDA(cudaMemcpyAsync(reinterpret_cast<double*>(c.hscal) + slot, reinterpret_cast<double*>(c.dscal) + slot,
                          sizeof(double), cudaMemcpyDeviceToHost, c.stream));
  c.sync();
  const T v = *reinterpret_cast<T*>(reinterpret_cast<double*>(c.hscal) + slot);
  dist_nan_guard(c, (double)v);
  return v;
}

template <class T> void k_dot_dev(Ctx& c, int n, const T* x, const T* y, int slot) { dot_launch<T>(c, n, x, y, slot, 0); }
template <class T> T k_dot(Ctx& c, int n, const T* x, const T* y) {
  dot_launch<T>(c, n, x, y, 0, 0);
  return read_slot<T>(c, 0);
}
template <class T, int MODE>
static void nrm2_launch(Ctx& c, int n, const T* x) {
  const int grid = n > 0 ? stream_grid(n, 4, 4) : 1;
  dot_kernel<T, 1, MODE><<<grid, kBlock, 0, c.stream>>>(n, x, x, nullptr, nullptr, (T*)c.partials, c.tickets, slot_ptr<T>(c, 0), 1, nullptr);
  KB_CUDA(cudaGetLastError());
  c.launches++;
}

// knorm = BLAS nrm2 (src/krylov_utils.jl:316): finite and accurate whenever ||x|| itself is.  One pass forms
// sqrt(sum x_i^2) and max|x_i|; the result stands unless the sum overflowed (Inf while max|x_i| is finite) or is so
// small that squares below the normal range may have moved it.  In that case one more pass sums the squares of x
// scaled by a power of two that brings max|x_i| into [1, 2), and scales the root back.
//
// Threshold: a rounding whose result is below realmin (the smallest normal number, 2^emin) errs by at most half the
// subnormal spacing, 2^(emin - p) = realmin * eps / 2 (p = 53 / 24 bits).  The sum makes fewer than n such roundings,
// so they move it by less than n * realmin * eps / 2, which is at most one ulp of the sum (ulp(S) > S * eps / 2)
// whenever S >= n * realmin.  Hence: rescale when sqrt(S) < sqrt(n * realmin).  A zero vector (max|x_i| = 0) never
// does, so it still costs one launch; nor does a NaN, which the first pass already returns.
//
// A row-partitioned solve (c.dcomm) keeps the plain sqrt(sum x_i^2): every rank sees the same reduced sum, but a
// rescaled pass would need a max over the ranks as well.
template <class T> T k_nrm2(Ctx& c, int n, const T* x) {
  if (c.dcomm) {
    dot_launch<T>(c, n, x, x, 0, 1);
    return read_slot<T>(c, 0);
  }
  nrm2_launch<T, DOT_NRM2>(c, n, x);
  KB_CUDA(cudaMemcpyAsync(c.hscal, c.dscal, 2 * sizeof(double), cudaMemcpyDeviceToHost, c.stream));
  c.sync();
  const T nrm = reinterpret_cast<T*>(c.hscal)[0], xmax = reinterpret_cast<T*>(c.hscal)[1];
  const T small = (T)std::sqrt((double)n * (double)std::numeric_limits<T>::min());
  const bool overflowed = std::isinf(nrm) && std::isfinite(xmax);
  const bool underflowed = xmax > T(0) && nrm < small;
  if (!overflowed && !underflowed) return nrm;
  nrm2_launch<T, DOT_NRM2_SCALED>(c, n, x);
  return read_slot<T>(c, 0);
}
template <class T> void k_dot2(Ctx& c, int n, const T* a, const T* b, const T* u, const T* v, T* r1, T* r2) {
  const int grid = n > 0 ? stream_grid(n, 4, 4) : 1;
  // two adjacent T outputs live in slot 0 (out[0], out[1])
  dot_kernel<T, 2><<<grid, kBlock, 0, c.stream>>>(n, a, b, u, v, (T*)c.partials, c.tickets, slot_ptr<T>(c, 0), 0, c.dcomm);
  KB_CUDA(cudaGetLastError());
  c.launches++;
  KB_CUDA(cudaMemcpyAsync(c.hscal, c.dscal, 2 * sizeof(double), cudaMemcpyDeviceToHost, c.stream));
  c.sync();
  *r1 = reinterpret_cast<T*>(c.hscal)[0];
  *r2 = reinterpret_cast<T*>(c.hscal)[1];
  dist_nan_guard(c, (double)*r1 + (double)*r2);
}

// ---------------------------------------------------------------------------
// Row-partitioned solves: host-visible pieces of the communicator
// ---------------------------------------------------------------------------
__global__ void dist_sum_kernel(DistComm* dc, double v, double* out) {
  const double r = dist_allreduce_sum_warp<double>(dc, v);
  if (threadIdx.x == 0) *out = r;
}

// Sum of one host scalar over all ranks (every rank must call it the same number of times).
double k_dist_sum(Ctx& c, double v) {
  if (!c.dcomm) return v;
  dist_sum_kernel<<<1, 32, 0, c.stream>>>(c.dcomm, v, reinterpret_cast<double*>(c.dscal) + 15);
  KB_CUDA(cudaGetLastError());
  c.launches++;
  return read_slot<double>(c, 15);
}

// Every rank of a row-partitioned solve must take the SAME exit decision: a rank that stops on its own callback
// result or wall clock leaves its peers spinning in the next reduction.  Flags are OR-ed over the ranks.
void dist_agree_on_exit(Ctx& c, bool& user_exit, bool& overtimed) {
  if (!c.dcomm) return;
  const double s = k_dist_sum(c, (user_exit ? 1.0 : 0.0) + (overtimed ? 1024.0 : 0.0));
  if (!(s == s)) return;                        // dead communicator: dist_check_alive raises
  const long long code = (long long)s;
  user_exit = (code % 1024) > 0;
  overtimed = (code / 1024) > 0;
}

// A reduction that timed out kills the communicator (dist.cuh); every later reduction returns NaN at once.
// The drivers call this before and after each solve and raise instead of handing NaNs to the caller.
void dist_check_alive(Ctx& c) {
  if (!c.dcomm) return;
  int err = 0;
  KB_CUDA(cudaMemcpyAsync(&err, &c.dcomm->error, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
  c.sync();
  if (err) throw std::runtime_error("cross-GPU reduction timed out: a peer rank stopped participating; the communicator of this "
                                    "workspace is dead (free the workspace on every rank and create it again)");
}

// cg! prologue for x0 = 0 and M = I (cg.jl:150-162): x = 0, r = b, p = r, gamma = <r, r> in ONE pass instead of
// fill + copy + copy + dot (the per-solve fixed cost matters once several GPUs share a short solve).
template <class T>
__global__ void __launch_bounds__(kBlock) cg_prologue_kernel(int n, const T* __restrict__ b, T* __restrict__ x, T* __restrict__ r,
                                                             T* __restrict__ p, T* part, unsigned* ticket, T* out, DistComm* dc) {
  __shared__ T sm[32];
  T acc = T(0);
  const unsigned stride = gridDim.x * blockDim.x, un = n > 0 ? n : 0;   // unsigned: see ew_kernel
  unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + 3 * stride < un; i += 4 * stride) {    // 4 loads in flight per thread, summed in the same order as one by one
    T v[4];
#pragma unroll
    for (int q = 0; q < 4; q++) v[q] = b[i + q * stride];
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const unsigned j = i + q * stride;
      x[j] = T(0); r[j] = v[q]; p[j] = v[q];
      acc += v[q] * v[q];
    }
  }
  for (; i < un; i += stride) {
    const T v = b[i];
    x[i] = T(0); r[i] = v; p[i] = v;
    acc += v * v;
  }
  T mine[1] = {block_sum(acc, sm)}, tot[1];
  if (grid_sum_last<T, 1>(mine, part, ticket, sm, tot) && threadIdx.x == 0) out[0] = dist_reduce(dc, tot[0]);
}
template <class T> T k_cg_prologue(Ctx& c, int n, const T* b, T* x, T* r, T* p) {
  const int grid = n > 0 ? stream_grid(n, 4, 4) : 1;
  cg_prologue_kernel<T><<<grid, kBlock, 0, c.stream>>>(n, b, x, r, p, (T*)c.partials, c.tickets, slot_ptr<T>(c, 0), c.dcomm);
  KB_CUDA(cudaGetLastError());
  c.launches++;
  return read_slot<T>(c, 0);
}

#define INST(T)                                                                        \
  template T k_dot<T>(Ctx&, int, const T*, const T*);                                  \
  template T k_cg_prologue<T>(Ctx&, int, const T*, T*, T*, T*);                        \
  template T k_nrm2<T>(Ctx&, int, const T*);                                           \
  template void k_dot2<T>(Ctx&, int, const T*, const T*, const T*, const T*, T*, T*);  \
  template void k_dot_dev<T>(Ctx&, int, const T*, const T*, int);                      \
  template void k_axpy<T>(Ctx&, int, T, const T*, T*);                                 \
  template void k_axpby<T>(Ctx&, int, T, const T*, T, T*);                             \
  template void k_scal<T>(Ctx&, int, T, T*);                                           \
  template void k_copy<T>(Ctx&, int, T*, const T*);                                    \
  template void k_scalcopy<T>(Ctx&, int, T*, T, const T*);                             \
  template void k_divcopy<T>(Ctx&, int, T*, const T*, T);                              \
  template void k_fill<T>(Ctx&, int, T*, T);                                           \
  template void k_diagmul<T>(Ctx&, int, T*, const T*, const T*, bool);                 \
  template void k_blockdiag_mul<T>(Ctx&, int, int, const T*, const T*, T*);            \
  template void k_blockdiag_invert<T>(Ctx&, int, int, const T*, T*, int*);
INST(double)
INST(float)
#undef INST

}  // namespace kb
