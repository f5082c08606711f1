// block.cu -- block_gmres! on device panels (SURVEY.md section 8f-2; src/block_gmres.jl:110-359).
//
// Data layout: every n x p block (X, B, W, V[k], ...) is a ROW-MAJOR panel in HBM (row r = p contiguous values),
// not the reference's column-major matrix: the sparse product then gathers one contiguous p-vector per nonzero and
// reads A once for all p right-hand sides, and the tall-skinny products stream both panels once.  B and X are
// transposed on the way in / out (the C ABI keeps the reference's column-major blocks).
//
// Kernels (p/8 flop per byte in the tall-skinny products: HBM-bound for p <= 8, FP64/issue-bound from p = 16 on):
//   spmm_tma_kernel<P>      W = A P on the TMA-staged tile pipeline of the SpMV, P lanes per row (P = 2..32);
//   spmm_rows_kernel        the same for any p: p threads per row, plain loads
//   panel_fast_kernel<P,..> register-resident tall-skinny products for P = 2, 4, 8, 16, 32:
//                             product   G = V^T Q (p x p, deterministic "last block finalises" reduction)
//                             update    Q = beta Q + alpha V S  (S p x p read from device memory: the Gram-Schmidt
//                                       chain never visits the host)
//                             fused     update followed by the next product in the same pass over the panels
//   panel_tn / panel_nn / panel_nn_tn_kernel   the same three operations for any p, 4 x 4 register-blocked on
//                             shared-memory tiles with an odd row stride
//   rows_diag_kernel        P = diag(d) V (Jacobi M / N);  relayout_kernel: column-major block <-> panel
// The panel QR of the reference (LAPACK geqrf + orgqr, src/block_krylov_utils.jl:201-208) is CholQR2 on the
// device (two Gram matrices, two p x p Cholesky factorizations on the host) followed by the reconstruction of
// the Householder signs from the top p x p block of Q (Ballard et al., "Reconstructing Householder vectors
// from tall-skinny QR", 2014), so V[k] and the R factors equal LAPACK's, not only up to column signs.  A Gram
// matrix that is not numerically positive definite (rank-deficient block) falls back to LAPACK's Householder
// algorithm, also on the device (panel_qr).
// Everything p x p (the Hessenberg QR, the block back substitution) stays on the host like the reference's.
#include <cstring>

#include "solver_common.h"
#include "block.h"
#include "dense_small.h"
#include "spmv_tiles.cuh"

namespace kb {

constexpr int kMaxBlockP = 32;
constexpr int kPanelTileElems = 2048;   // capacity of one staged panel tile (16 KB of doubles)

// ---------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------
template <class T> struct Vec2 { T x, y; };
template <class T> __device__ __forceinline__ Vec2<T> ld2(const T* p) {
  return *reinterpret_cast<const Vec2<T>*>(p);   // p is 2-element aligned (P even, 256-byte aligned panels)
}
// Layout conversion between the ABI's column-major n x p blocks and the row-major panels: one thread per panel row,
// so the column-major side is accessed coalesced across threads and the panel side as contiguous p-vectors.
template <class T, bool TO_PANEL>
__global__ void __launch_bounds__(kBlock) relayout_kernel(int n, int p, const T* __restrict__ in, T* __restrict__ out) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
    for (int c = 0; c < p; c++) {
      if (TO_PANEL) out[(size_t)r * p + c] = in[(size_t)c * n + r];
      else out[(size_t)c * n + r] = in[(size_t)r * p + c];
    }
  }
}

// W = A P, generic: p threads per row (any p, any row length)
template <class T>
__global__ void __launch_bounds__(kBlock) spmm_rows_kernel(Csr<T> A, int p, const T* __restrict__ X, T* __restrict__ Y) {
  const long long total = (long long)A.n * p;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int row = (int)(i / p), c = (int)(i % p);
    const int kb = A.rowptr[row], ke = A.rowptr[row + 1];
    T acc = T(0);
    for (int k = kb; k < ke; k++) acc = add_rn(acc, mul_rn(A.val[k], __ldg(&X[(size_t)A.colind[k] * p + c])));
    Y[i] = acc;
  }
}

// W = A P on the TMA-staged tile pipeline of the SpMV (spmv_tiles.cuh: same producer, same shared-memory ring):
// P lanes share a row (see the consumer loop).  Row sums accumulate in ascending column order, non-contracted, like
// the SpMV.
template <class T, int P>
__global__ void __launch_bounds__(kTileThreads, 3) spmm_tma_kernel(Csr<T> A, const T* __restrict__ X, T* __restrict__ Y) {
  extern __shared__ __align__(128) unsigned char smem[];
  const TileLayout<T> L{A.tile_cap};
  const int S = A.stages;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);
  uint64_t* empty = full + S;
  unsigned char* ring = smem + 128;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int VA = 16 / sizeof(T);
  if (tid == 0) {
    for (int s = 0; s < S; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], kConsumerWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (warp == kConsumerWarps) {
    if (lane == 0) tile_producer<T>(A, L, S, ring, full, empty);
    return;
  }
  int it = 0;
  for (int t = blockIdx.x; t < A.ntiles; t += gridDim.x, it++) {
    const int s = it % S;
    mbar_wait(&full[s], (it / S) & 1);
    const unsigned char* st = ring + (size_t)s * L.stage_bytes();
    const int* rp = reinterpret_cast<const int*>(st);
    const T* vs = reinterpret_cast<const T*>(st + L.rp_bytes());
    const int* cs = reinterpret_cast<const int*>(st + L.rp_bytes() + L.val_bytes());
    {
      // P lanes per row: the P lanes of a row read the same staged (value, column) pair (broadcast) and one contiguous
      // P-vector of the panel (coalesced); a warp covers 32 / P rows per step and its 32 tile rows in P steps.
      const int k0 = rp[0];
      const T* vrow = vs - (k0 & ~(VA - 1));
      const int* crow = cs - (k0 & ~3);
      constexpr int RPW = 32 / P;
      const int rsub = lane / P, c = lane % P;
      // RU rows per trip with independent accumulators, D nonzeros of each row per batch: RU * D gathers of the
      // panel in flight per lane (a row-at-a-time loop leaves one row's 7 gathers in flight and the warp idles on
      // their latency 32 times per tile at P = 32).  Indices are clamped into the row and the sums selected, so the
      // batch is straight-line code (spmv_tiles.cuh); every row still accumulates in ascending column order.
      constexpr int RU = P >= 4 ? 4 : P, D = 4;
#pragma unroll 1
      for (int step = 0; step < P; step += RU) {
        int kb[RU], ke[RU];
        T acc[RU];
        int kmax = 0;
#pragma unroll
        for (int u = 0; u < RU; u++) {
          const int lr = warp * 32 + (step + u) * RPW + rsub;    // row inside the tile
          kb[u] = rp[lr]; ke[u] = rp[lr + 1];
          acc[u] = T(0);
          kmax = max(kmax, ke[u] - kb[u]);
        }
        kmax = __reduce_max_sync(0xffffffffu, kmax);               // uniform trip count for the warp
        for (int kk = 0; kk < kmax; kk += D) {
          T xv[RU][D];
#pragma unroll
          for (int u = 0; u < RU; u++)
#pragma unroll
            for (int d = 0; d < D; d++) {
              const int idx = max(kb[u], min(kb[u] + kk + d, ke[u] - 1));
              // an EMPTY row (also the rows past n of the last tile) has no slot of its own: whatever sits at
              // `idx` in shared memory is not a column index -- gather row 0 of the panel instead (value ignored)
              const int cc = crow[idx];
              xv[u][d] = __ldg(&X[(size_t)(kb[u] < ke[u] ? cc : 0) * P + c]);
            }
          asm volatile("" ::: "memory");
#pragma unroll
          for (int u = 0; u < RU; u++)
#pragma unroll
            for (int d = 0; d < D; d++) {
              const int idx = max(kb[u], min(kb[u] + kk + d, ke[u] - 1));
              const T nx = add_rn(acc[u], mul_rn(vrow[idx], xv[u][d]));
              acc[u] = (kb[u] + kk + d < ke[u]) ? nx : acc[u];
            }
        }
#pragma unroll
        for (int u = 0; u < RU; u++) {
          const int grow = t * kTileRows + warp * 32 + (step + u) * RPW + rsub;
          if (grow < A.n) Y[(size_t)grow * P + c] = acc[u];
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);
  }
}

template <class T>
__global__ void __launch_bounds__(kBlock) rows_diag_kernel(long long total, int p, const T* __restrict__ d, const T* __restrict__ in,
                                                          T* __restrict__ out, int ldiv) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const T dv = d[i / p];
    out[i] = ldiv ? div_rn(in[i], dv) : mul_rn(dv, in[i]);
  }
}

// ---- tiles ------------------------------------------------------------------------------------------------------
// A tile of `rows` panel rows is staged in shared memory with an ODD row stride ps = p | 1 (bank-conflict-free
// when consecutive lanes read consecutive rows).  Both tall-skinny products are register-blocked 4 x 4: 16 FMAs per
// 8 shared-memory loads, which is what keeps them HBM-bound up to p = 16 (fp64 FMA issue is the limit at p = 32).
__host__ __device__ inline int panel_stride(int p) { return p | 1; }
__host__ __device__ inline int panel_tile_rows(int p) { return kPanelTileElems / panel_stride(p); }

template <class T>
__device__ __forceinline__ void load_tile(T* dstS, const T* __restrict__ src, int rows, int p, int ps) {
  for (int e = threadIdx.x; e < rows * p; e += kBlock) {
    const int r = e / p, c = e - r * p;
    dstS[r * ps + c] = src[e];
  }
}

// G(i,j) = sum_r L[r][i] Rt[r][j], column-major p x p.  Thread = (4 x 4 block of G, row group): the block index
// varies fastest across lanes, group g takes rows g, g + ngroups, ... of every staged tile.
template <class T>
struct PairAcc {
  T acc[4][4];
  int nbi, nb, ngroups, bi, bj, group;
  bool active;
  __device__ __forceinline__ void init(int p) {
    nbi = (p + 3) >> 2;
    nb = nbi * nbi;                               // <= 64 for p <= 32
    ngroups = kBlock / nb;
    const int tid = threadIdx.x;
    active = tid < ngroups * nb;
    const int blk = tid % nb;
    group = tid / nb;
    bi = (blk % nbi) * 4;
    bj = (blk / nbi) * 4;
#pragma unroll
    for (int a = 0; a < 4; a++)
#pragma unroll
      for (int b = 0; b < 4; b++) acc[a][b] = T(0);
  }
  __device__ __forceinline__ void tile(int p, int ps, int rows, const T* Ls, const T* Rs) {
    if (!active) return;
    for (int r = group; r < rows; r += ngroups) {
      T l[4], q[4];
#pragma unroll
      for (int a = 0; a < 4; a++) {
        l[a] = bi + a < p ? Ls[r * ps + bi + a] : T(0);
        q[a] = bj + a < p ? Rs[r * ps + bj + a] : T(0);
      }
#pragma unroll
      for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++) acc[a][b] += l[a] * q[b];
    }
  }
  // combine the row groups of this CTA (fixed order) through `scratch` (>= 256 * 16 entries, may alias the tiles),
  // then the CTAs ("last block finalises", fixed order) -> G
  __device__ __forceinline__ void finish(int p, T* scratch, T* part, unsigned* ticket, T* G) {
    __shared__ bool is_last;
    const int tid = threadIdx.x;
    const int pp = p * p;
    __syncthreads();                              // tiles are dead from here on
    if (active) {
#pragma unroll
      for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++) scratch[tid * 16 + a * 4 + b] = acc[a][b];
    }
    __syncthreads();
    for (int pair = tid; pair < pp; pair += kBlock) {
      const int i = pair % p, j = pair / p;
      const int blk = (i >> 2) + (j >> 2) * nbi, off = (i & 3) * 4 + (j & 3);
      T s = T(0);
      for (int g = 0; g < ngroups; g++) s += scratch[(g * nb + blk) * 16 + off];
      part[(size_t)blockIdx.x * pp + pair] = s;
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) {
      const unsigned t = atomicAdd(ticket, 1u);
      is_last = (t == gridDim.x - 1);
      if (is_last) *ticket = 0u;
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    for (int pair = tid; pair < pp; pair += kBlock) {
      T s = T(0);
      for (int b = 0; b < (int)gridDim.x; b++) s += __ldcg(&part[(size_t)b * pp + pair]);
      G[pair] = s;
    }
  }
};

// Out tile <- beta * Out + alpha * In * S for one staged tile, 4 rows x 4 columns per thread.  Consecutive lanes take
// consecutive rows (odd stride: conflict-free) and the same column block (S loads broadcast).  Results go to global
// memory and, when OsNew != nullptr, into that shared tile (for a following product).
template <class T>
__device__ __forceinline__ void nn_tile(int p, int ps, int rows, T alpha, const T* Is, const T* Ss, T beta, const T* OsOld, T* OsNew,
                                        T* OutG) {
  const int R4 = (rows + 3) >> 2;                 // rows are handled as r, r + R4, r + 2 R4, r + 3 R4
  const int ncq = (p + 3) >> 2;
  for (int item = threadIdx.x; item < R4 * ncq; item += kBlock) {
    const int rq = item % R4, cq = (item / R4) * 4;
    T acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; a++)
#pragma unroll
      for (int b = 0; b < 4; b++) acc[a][b] = T(0);
    for (int i = 0; i < p; i++) {
      T in[4], sv[4];
#pragma unroll
      for (int a = 0; a < 4; a++) {
        const int r = rq + a * R4;
        in[a] = r < rows ? Is[r * ps + i] : T(0);
        sv[a] = cq + a < p ? Ss[i + (cq + a) * p] : T(0);
      }
#pragma unroll
      for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++) acc[a][b] = fma(in[a], sv[b], acc[a][b]);
    }
#pragma unroll
    for (int a = 0; a < 4; a++) {
      const int r = rq + a * R4;
      if (r >= rows) continue;
#pragma unroll
      for (int b = 0; b < 4; b++) {
        const int cidx = cq + b;
        if (cidx >= p) continue;
        const T v = beta == T(0) ? mul_rn(alpha, acc[a][b]) : add_rn(mul_rn(beta, OsOld[r * ps + cidx]), mul_rn(alpha, acc[a][b]));
        if (OsNew) OsNew[r * ps + cidx] = v;
        OutG[(size_t)r * p + cidx] = v;
      }
    }
  }
}

template <class T>
__global__ void __launch_bounds__(kBlock) panel_tn_kernel(int n, int p, const T* __restrict__ V, const T* __restrict__ Q,
                                                         T* part, unsigned* ticket, T* G) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int ps = panel_stride(p), trows = panel_tile_rows(p);
  T* Vs = reinterpret_cast<T*>(smem_raw);         // 2 tiles of kPanelTileElems; reused as the 4096-entry scratch
  T* Qs = Vs + kPanelTileElems;
  PairAcc<T> pa;
  pa.init(p);
  const int ntiles = (n + trows - 1) / trows;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int r0 = tile * trows;
    const int rows = min(trows, n - r0);
    __syncthreads();
    load_tile(Vs, V + (size_t)r0 * p, rows, p, ps);
    load_tile(Qs, Q + (size_t)r0 * p, rows, p, ps);
    __syncthreads();
    pa.tile(p, ps, rows, Vs, Qs);
  }
  pa.finish(p, Vs, part, ticket, G);
}

// Fused update + next product (one pass over the panels instead of two):
//   Out[r][:] = beta Out[r][:] + alpha In[r][:] S        then        G = Next^T Out   (Next == nullptr: Out^T Out)
// Block Gram-Schmidt:  Q -= V_i Psi_i and Psi_{i+1} = V_{i+1}^T Q (or the Gram matrix Q^T Q of the panel QR after
// the last block).  Panel QR pass 1:  Q <- Q R1^-1 and the second Gram matrix.  Out may alias In.
template <class T>
__global__ void __launch_bounds__(kBlock) panel_nn_tn_kernel(int n, int p, T alpha, const T* In, const T* __restrict__ S, T beta,
                                                            T* Out, const T* Next, T* part, unsigned* ticket, T* G) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int ps = panel_stride(p), trows = panel_tile_rows(p);
  T* Is = reinterpret_cast<T*>(smem_raw);         // 3 tiles + S
  T* Os = Is + kPanelTileElems;
  T* Ns = Os + kPanelTileElems;
  T* Ss = Ns + kPanelTileElems;
  const int tid = threadIdx.x;
  for (int e = tid; e < p * p; e += kBlock) Ss[e] = S[e];
  PairAcc<T> pa;
  pa.init(p);
  const int ntiles = (n + trows - 1) / trows;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int r0 = tile * trows;
    const int rows = min(trows, n - r0);
    __syncthreads();
    load_tile(Is, In + (size_t)r0 * p, rows, p, ps);
    if (beta != T(0)) load_tile(Os, (const T*)Out + (size_t)r0 * p, rows, p, ps);
    if (Next) load_tile(Ns, Next + (size_t)r0 * p, rows, p, ps);
    __syncthreads();
    nn_tile<T>(p, ps, rows, alpha, Is, Ss, beta, Os, Os, Out + (size_t)r0 * p);
    __syncthreads();
    pa.tile(p, ps, rows, Next ? Ns : Os, Os);
  }
  pa.finish(p, Is, part, ticket, G);             // Is + Os = 4096 entries of scratch
}

// Out[r][j] = beta * Out[r][j] + alpha * sum_i In[r][i] S(i,j);  S column-major p x p in device memory.
// In is staged per tile, so Out may alias In (the in-place Q <- Q S of the panel QR).
template <class T>
__global__ void __launch_bounds__(kBlock) panel_nn_kernel(int n, int p, T alpha, const T* In, const T* __restrict__ S, T beta, T* Out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int ps = panel_stride(p), trows = panel_tile_rows(p);
  T* Is = reinterpret_cast<T*>(smem_raw);
  T* Os = Is + kPanelTileElems;
  T* Ss = Os + kPanelTileElems;
  const int tid = threadIdx.x;
  for (int e = tid; e < p * p; e += kBlock) Ss[e] = S[e];
  const int ntiles = (n + trows - 1) / trows;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int r0 = tile * trows;
    const int rows = min(trows, n - r0);
    __syncthreads();
    load_tile(Is, In + (size_t)r0 * p, rows, p, ps);
    if (beta != T(0)) load_tile(Os, (const T*)Out + (size_t)r0 * p, rows, p, ps);
    __syncthreads();
    nn_tile<T>(p, ps, rows, alpha, Is, Ss, beta, Os, (T*)nullptr, Out + (size_t)r0 * p);
  }
}

// ---- register-resident fast path for P in {2, 4, 8, 16, 32} -------------------------------------------------------
// No shared-memory tiles: TPR adjacent lanes share one panel row (1, 1, 2, 8, 16 for P = 2..32, chosen by the sweep
// profiles/sweep_block.py), each owning a slab of
// C = P/TPR columns of the updated row and a P x C slab (<= 64 accumulators) of the Gram-type product; operands stream from
// global memory as 16-byte vectors, every panel element is loaded by exactly one lane (its slab owner) and the TPR
// lanes of a row exchange slabs by warp shuffle.  ~190 instructions per row at P = 8 against 256 B of HBM traffic:
// bandwidth-bound, unlike the tiled generic kernels.
//   UPDATE: Out[r][:] = beta Out[r][:] + alpha In[r][:] S         GRAM: G = Next^T Out  (Next == nullptr: Out^T Out)

template <class T, int P, int TPR, bool UPDATE, bool GRAM, bool PREFETCH>
__global__ void __launch_bounds__(kBlock, (P * P / TPR <= 32 ? 2 : 1)) panel_fast_kernel(int n, T alpha, const T* In, const T* __restrict__ S,
                                                                                     T beta, T* Out, const T* Next, T* part,
                                                                                     unsigned* ticket, T* G) {
  constexpr int C = P / TPR;
  static_assert(P % 2 == 0 && C >= 2 && TPR <= 32, "fast path block sizes");
  __shared__ __align__(16) T Ss[UPDATE ? P * P : 2];   // Ss[i * P + j] = S(i, j): the slab of row i is contiguous
  __shared__ __align__(16) T Gs[GRAM ? P * P : 2];
  __shared__ bool is_last;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int slab = tid % TPR, c0 = slab * C;
  if (UPDATE) {
    for (int e = tid; e < P * P; e += kBlock) Ss[(e % P) * P + e / P] = S[e];     // column-major S -> row-major Ss
    __syncthreads();
  }
  T acc[GRAM ? P : 1][C];
  if (GRAM) {
#pragma unroll
    for (int i = 0; i < P; i++)
#pragma unroll
      for (int j = 0; j < C; j++) acc[i][j] = T(0);
  }
  const int rows_per_pass = gridDim.x * (kBlock / TPR);
  const int first = blockIdx.x * (kBlock / TPR) + tid / TPR;
  const int passes = (n + rows_per_pass - 1) / rows_per_pass;        // uniform trip count: shuffles stay convergent
  const int lane0 = lane - slab;                   // first of the TPR lanes that share a row
  const bool need_out = !UPDATE || beta != T(0);
  // this lane's slabs of one panel row: every panel element is loaded by exactly one lane, as 16-byte vectors
  struct Slabs { T in[C], out[C], nx[C]; bool valid; size_t base; };
  auto load_row = [&](int it, Slabs& r) {
    const int row = first + it * rows_per_pass;
    r.valid = row < n;
    r.base = (size_t)(r.valid ? row : 0) * P;
#pragma unroll
    for (int j = 0; j < C; j += 2) {
      Vec2<T> z; z.x = T(0); z.y = T(0);
      Vec2<T> vi = z, vo = z, vn = z;
      if (r.valid) {
        if (UPDATE) vi = ld2(In + r.base + c0 + j);
        if (need_out) vo = ld2(Out + r.base + c0 + j);
        if (GRAM && Next) vn = ld2(Next + r.base + c0 + j);
      }
      r.in[j] = vi.x; r.in[j + 1] = vi.y;
      r.out[j] = vo.x; r.out[j + 1] = vo.y;
      r.nx[j] = vn.x; r.nx[j + 1] = vn.y;
    }
  };
  Slabs cur;
  load_row(0, cur);
  for (int it = 0; it < passes; it++) {
    Slabs nxt;
    if (PREFETCH && it + 1 < passes) load_row(it + 1, nxt);      // next row's loads in flight during this row's math
    T outv[C];
    if (UPDATE) {
      // the other slabs of the In row arrive by shuffle from the lanes that hold them, in ascending column order
      // (the order of the row-times-matrix sum)
      T a[C];
#pragma unroll
      for (int j = 0; j < C; j++) a[j] = T(0);
#pragma unroll
      for (int k = 0; k < TPR; k++) {
#pragma unroll
        for (int jj = 0; jj < C; jj++) {
          const T in = TPR == 1 ? cur.in[jj] : __shfl_sync(0xffffffffu, cur.in[jj], lane0 + k);
          const int i = k * C + jj;
#pragma unroll
          for (int j = 0; j < C; j++) a[j] = fma(in, Ss[i * P + c0 + j], a[j]);     // contracted: this is a GEMM, not a k* primitive
        }
      }
#pragma unroll
      for (int j = 0; j < C; j++) outv[j] = beta != T(0) ? fma(alpha, a[j], mul_rn(beta, cur.out[j])) : mul_rn(alpha, a[j]);
      if (cur.valid) {                             // Out may alias In: each lane rewrites exactly the slab it read
#pragma unroll
        for (int j = 0; j < C; j += 2) {
          Vec2<T> o; o.x = outv[j]; o.y = outv[j + 1];
          *reinterpret_cast<Vec2<T>*>(Out + cur.base + c0 + j) = o;
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < C; j++) outv[j] = cur.out[j];
    }
    if (GRAM) {
#pragma unroll
      for (int k = 0; k < TPR; k++) {
#pragma unroll
        for (int jj = 0; jj < C; jj++) {
          const T mine = Next ? cur.nx[jj] : outv[jj];         // this lane's slab of the left operand row
          const T l = TPR == 1 ? mine : __shfl_sync(0xffffffffu, mine, lane0 + k);
#pragma unroll
          for (int j = 0; j < C; j++) acc[k * C + jj][j] += l * outv[j];
        }
      }
    }
    if (PREFETCH) cur = nxt;
    else if (it + 1 < passes) load_row(it + 1, cur);
  }
  if (!GRAM) return;
  // rows of this warp (lanes with the same slab), then the warps in order, then the CTAs in order
#pragma unroll
  for (int i = 0; i < P; i++)
#pragma unroll
    for (int j = 0; j < C; j++) {
      T v = acc[i][j];
      for (int off = TPR; off < 32; off <<= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
      acc[i][j] = v;
    }
  for (int e = tid; e < P * P; e += kBlock) Gs[e] = T(0);
  __syncthreads();
  for (int w = 0; w < kBlock / 32; w++) {
    if (warp == w && lane < TPR) {
#pragma unroll
      for (int i = 0; i < P; i++)
#pragma unroll
        for (int j = 0; j < C; j++) Gs[i + (c0 + j) * P] += acc[i][j];
    }
    __syncthreads();
  }
  for (int e = tid; e < P * P; e += kBlock) part[(size_t)blockIdx.x * (P * P) + e] = Gs[e];
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const unsigned t = atomicAdd(ticket, 1u);
    is_last = (t == gridDim.x - 1);
    if (is_last) *ticket = 0u;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  for (int pair = tid; pair < P * P; pair += kBlock) {
    T s = T(0);
    for (int b = 0; b < (int)gridDim.x; b++) s += __ldcg(&part[(size_t)b * (P * P) + pair]);
    G[pair] = s;
  }
}


// ---- tensor-core path for Float64, P in {8, 16, 32}: mma.sync.m8n8k4.f64 (SASS DMMA) ------------------------------
// Same two operations as panel_fast_kernel (UPDATE: Out = beta Out + alpha In S;  GRAM: G = Next^T Out), one warp
// per tile of 8 panel rows, no shuffles and no shared-memory tiles: every operand is loaded straight into the
// fragment layout of the instruction, and the two products are oriented so that the OUTPUT fragment of the update
// is, register for register, the INPUT fragment of the Gram product:
//   update, transposed:  Out_tile^T (P x 8) = S^T (P x P) . In_tile^T (P x 8)
//       A (8 x 4, row)  = S^T block   lane (a, b) holds S(i = kslot, j = 8 mb + a)        -- constant, staged in smem
//       B (4 x 8, col)  = In_tile^T   lane (a, b) holds In[row a][kslot]                   -- 16-byte loads
//       D (8 x 8)       = lane (a, b) holds Out[row 2b + e][col 8 mb + a], e = 0, 1
//   Gram:  G (P x P) += L_tile^T (P x 8) . Out_tile (8 x P),  L = Next (or Out itself)
//       A (8 x 4, row)  = L^T block   lane (a, b) holds L[row 2b + e][col 8 ib + a]       -- the D layout above
//       B (4 x 8, col)  = Out block   lane (a, b) holds Out[row 2b + e][col 8 jb + a]     -- the D registers themselves
//       the two k-steps e = 0 / 1 cover rows {0,2,4,6} / {1,3,5,7}: the reduction index may be permuted freely.
// with a = lane >> 2, b = lane & 3 and kslot(ks, b) = 8 (ks / 2) + 2 b + (ks & 1) (again a permutation of the
// reduction index, chosen so that one 16-byte load feeds two k-steps).  256 FMAs per instruction instead of 32:
// the issue slots that bound the SIMT kernels at P >= 16 are freed, the kernels go
// back to being HBM-bound.  Float32 panels keep the SIMT path.
__device__ __forceinline__ void dmma_884(double& d0, double& d1, double a, double b, double c0, double c1) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%4, %5};"
               : "=d"(d0), "=d"(d1)
               : "d"(a), "d"(b), "d"(c0), "d"(c1));
}

constexpr int kMmaWarps = 8;

template <int P, bool UPDATE, bool GRAM>
__global__ void __launch_bounds__(kMmaWarps * 32, (P <= 16 ? 3 : 2))
panel_mma_kernel(int n, double alpha, const double* In, const double* __restrict__ S, double beta, double* Out, const double* Next,
                 double* part, unsigned* ticket, double* G) {
  constexpr int NB = P / 8;           // 8-column blocks of a panel row
  constexpr int KS = P / 4;           // k-steps of the update
  __shared__ double Sf[UPDATE ? KS * NB * 32 : 1];     // S^T fragments: [ks][mb][lane]
  __shared__ double Gs[GRAM ? P * P : 1];
  __shared__ bool is_last;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int a = lane >> 2, b = lane & 3;
  if (UPDATE) {
    for (int idx = tid; idx < KS * NB * 32; idx += kMmaWarps * 32) {
      const int ks = idx / (NB * 32), mb = (idx / 32) % NB, l = idx % 32;
      const int i = 8 * (ks >> 1) + 2 * (l & 3) + (ks & 1), j = 8 * mb + (l >> 2);
      Sf[idx] = S[i + (size_t)j * P];                   // S is column-major: S(i, j)
    }
    __syncthreads();
  }
  double acc[GRAM ? NB : 1][GRAM ? NB : 1][2];
  if (GRAM) {
#pragma unroll
    for (int i = 0; i < NB; i++)
#pragma unroll
      for (int j = 0; j < NB; j++) acc[i][j][0] = acc[i][j][1] = 0.0;
  }
  const bool need_old = !UPDATE || beta != 0.0;
  const int ntiles = (n + 7) >> 3;
  for (int tile = blockIdx.x * kMmaWarps + warp; tile < ntiles; tile += gridDim.x * kMmaWarps) {
    const int row0 = tile << 3;
    // ---- loads (all issued before any use) ----
    double inx[UPDATE ? NB : 1], iny[UPDATE ? NB : 1];            // In[row0 + a][8 q + 2 b], [.. + 1]
    double old[NB][2], nx[GRAM ? NB : 1][2];
    const int rin = row0 + a;
    // Next feeds only the Gram product.  Its loads are issued with the others, so that their latency hides behind
    // the update, except in the fused P = 32 kernel: held across the update there they push it past the
    // 128-register budget of two CTAs per SM on sm_90a (spills), so they follow the update's DMMA chain instead.
    constexpr bool kLateNext = UPDATE && P >= 32;
    auto load_next = [&]() {
#pragma unroll
      for (int e = 0; e < 2; e++) {
        const int r = row0 + 2 * b + e;
#pragma unroll
        for (int mb = 0; mb < NB; mb++) nx[mb][e] = (Next != nullptr && r < n) ? Next[(size_t)r * P + 8 * mb + a] : 0.0;
      }
    };
    if (UPDATE) {
#pragma unroll
      for (int q = 0; q < NB; q++) {
        Vec2<double> v; v.x = 0.0; v.y = 0.0;
        if (rin < n) v = ld2(In + (size_t)rin * P + 8 * q + 2 * b);
        inx[q] = v.x; iny[q] = v.y;
      }
    }
#pragma unroll
    for (int e = 0; e < 2; e++) {
      const int r = row0 + 2 * b + e;
      const bool ok = r < n;
#pragma unroll
      for (int mb = 0; mb < NB; mb++) {
        old[mb][e] = (need_old && ok) ? Out[(size_t)r * P + 8 * mb + a] : 0.0;
        if (GRAM && !kLateNext) nx[mb][e] = (Next != nullptr && ok) ? Next[(size_t)r * P + 8 * mb + a] : 0.0;
      }
    }
    // ---- update: D[mb] = sum_ks S^T frag x In frag ----
    double o[NB][2];
    if (UPDATE) {
      // k-step outermost: the NB accumulator chains (one per 8-column block) are independent, so consecutive DMMAs
      // never wait for each other's result (a per-block loop issues KS dependent DMMAs back to back)
      double cacc[NB][2];
#pragma unroll
      for (int mb = 0; mb < NB; mb++) cacc[mb][0] = cacc[mb][1] = 0.0;
#pragma unroll
      for (int ks = 0; ks < KS; ks++) {
        const double bfrag = (ks & 1) ? iny[ks >> 1] : inx[ks >> 1];
#pragma unroll
        for (int mb = 0; mb < NB; mb++)
          dmma_884(cacc[mb][0], cacc[mb][1], Sf[(ks * NB + mb) * 32 + lane], bfrag, cacc[mb][0], cacc[mb][1]);
      }
      if (GRAM && kLateNext) load_next();
#pragma unroll
      for (int mb = 0; mb < NB; mb++) {
        o[mb][0] = beta != 0.0 ? fma(alpha, cacc[mb][0], beta * old[mb][0]) : alpha * cacc[mb][0];
        o[mb][1] = beta != 0.0 ? fma(alpha, cacc[mb][1], beta * old[mb][1]) : alpha * cacc[mb][1];
      }
#pragma unroll
      for (int e = 0; e < 2; e++) {
        const int r = row0 + 2 * b + e;
        if (r < n) {
#pragma unroll
          for (int mb = 0; mb < NB; mb++) Out[(size_t)r * P + 8 * mb + a] = o[mb][e];
        }
      }
    } else {
#pragma unroll
      for (int mb = 0; mb < NB; mb++) { o[mb][0] = old[mb][0]; o[mb][1] = old[mb][1]; }
    }
    // ---- Gram: acc[ib][jb] += L^T frag x Out frag (rows past n contribute zeros) ----
    if (GRAM) {
#pragma unroll
      for (int e = 0; e < 2; e++)             // k-step outermost: NB * NB independent accumulators per step
#pragma unroll
        for (int ib = 0; ib < NB; ib++)
#pragma unroll
          for (int jb = 0; jb < NB; jb++)
            dmma_884(acc[ib][jb][0], acc[ib][jb][1], Next != nullptr ? nx[ib][e] : o[ib][e], o[jb][e], acc[ib][jb][0], acc[ib][jb][1]);
    }
  }
  if (!GRAM) return;
  // deterministic reduction: warps of the CTA in order, then the CTAs in order (last CTA finalises)
  for (int e = tid; e < P * P; e += kMmaWarps * 32) Gs[e] = 0.0;
  __syncthreads();
  for (int w = 0; w < kMmaWarps; w++) {
    if (warp == w) {
#pragma unroll
      for (int ib = 0; ib < NB; ib++)
#pragma unroll
        for (int jb = 0; jb < NB; jb++)
#pragma unroll
          for (int e = 0; e < 2; e++) Gs[(8 * ib + a) + (size_t)(8 * jb + 2 * b + e) * P] += acc[ib][jb][e];
    }
    __syncthreads();
  }
  for (int e = tid; e < P * P; e += kMmaWarps * 32) part[(size_t)blockIdx.x * (P * P) + e] = Gs[e];
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const unsigned t = atomicAdd(ticket, 1u);
    is_last = (t == gridDim.x - 1);
    if (is_last) *ticket = 0u;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  for (int pair = tid; pair < P * P; pair += kMmaWarps * 32) {
    double s = 0.0;
    for (int bk = 0; bk < (int)gridDim.x; bk++) s += __ldcg(&part[(size_t)bk * (P * P) + pair]);
    G[pair] = s;
  }
}

// ---------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------
template <class T> static int panel_grid(int n, int p) {
  const int trows = panel_tile_rows(p);
  const int ntiles = (n + trows - 1) / trows;
  return std::max(1, std::min(ntiles, sm_count() * 4));
}
// k_transpose(rows, cols): `in` is rows x cols row-major, `out` cols x rows row-major.  Only two shapes occur:
// (p, n) = column-major block -> panel, and (n, p) = panel -> column-major block.
template <class T> static void k_transpose(Ctx& c, int rows, int cols, const T* in, T* out) {
  if ((long long)rows * cols <= 0) return;
  const bool to_panel = rows <= cols;          // p <= 32 < n on this path (n >= p is checked at creation)
  const int n = to_panel ? cols : rows, p = to_panel ? rows : cols;
  if (to_panel) relayout_kernel<T, true><<<stream_grid(n, 1, 8), kBlock, 0, c.stream>>>(n, p, in, out);
  else relayout_kernel<T, false><<<stream_grid(n, 1, 8), kBlock, 0, c.stream>>>(n, p, in, out);
  KB_CUDA(cudaGetLastError()); c.launches++;
}
template <class T, int P> static void launch_spmm_tma(Ctx& c, const Csr<T>& A, const T* X, T* Y) {
  ensure_dyn_smem((const void*)spmm_tma_kernel<T, P>, 220 * 1024);
  int occ = 0;
  KB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, spmm_tma_kernel<T, P>, kTileThreads, A.smem_bytes));
  if (occ < 1) throw std::runtime_error("spmm_tma_kernel does not fit on an SM with the planned shared-memory ring");
  const int grid = std::min(std::min(occ, A.ctas_per_sm) * sm_count(), std::max(1, A.ntiles));
  spmm_tma_kernel<T, P><<<grid, kTileThreads, A.smem_bytes, c.stream>>>(A, X, Y);
}
// variant: 0 auto (what block_gmres runs), 1 the p-threads-per-row kernel, 2 TMA-staged (throws when p has no
// specialization or the tile plan does not fit)
template <class T> static void k_spmm(Ctx& c, const Csr<T>& A, int p, const T* X, T* Y, int variant = 0) {
  if (variant < 0 || variant > 2) throw std::runtime_error("SpMM variant must be 0, 1 or 2");
  if (variant == 2 && !A.tma_ok) throw std::runtime_error("TMA-staged SpMM requested but the tile plan does not fit shared memory");
  if (A.n <= 0) return;
  static const char* spmm_env = getenv("KB200_SPMM");          // "rows": force the generic kernel (A/B runs)
  const bool auto_tma = variant == 0 && A.tma_ok && !getenv("KB200_BLOCK_GENERIC") && !(spmm_env && !strcmp(spmm_env, "rows"));
  if (variant == 2 || auto_tma) {
    bool done = true;
    switch (p) {
      case 2: launch_spmm_tma<T, 2>(c, A, X, Y); break;
      case 4: launch_spmm_tma<T, 4>(c, A, X, Y); break;
      case 8: launch_spmm_tma<T, 8>(c, A, X, Y); break;
      case 16: launch_spmm_tma<T, 16>(c, A, X, Y); break;
      case 32: launch_spmm_tma<T, 32>(c, A, X, Y); break;
      default: done = false;
    }
    if (done) { KB_CUDA(cudaGetLastError()); c.launches++; return; }
    if (variant == 2) throw std::runtime_error("TMA-staged SpMM exists for p = 2, 4, 8, 16, 32 only");
  }
  spmm_rows_kernel<T><<<stream_grid((long long)A.n * p, 1, 8), kBlock, 0, c.stream>>>(A, p, X, Y);
  KB_CUDA(cudaGetLastError()); c.launches++;
}
template <class T> static void k_rows_diag(Ctx& c, int n, int p, const T* d, const T* in, T* out, bool ldiv) {
  rows_diag_kernel<T><<<stream_grid((long long)n * p, 1, 8), kBlock, 0, c.stream>>>((long long)n * p, p, d, in, out, ldiv ? 1 : 0);
  KB_CUDA(cudaGetLastError()); c.launches++;
}
// tensor-core dispatch (Float64, p = 8 / 16 / 32).  ws.mma_mode (KB200_BLOCK_MMA) 0 keeps the SIMT kernels (A/B
// runs, tests), 16 only p = 16 / 32 (p = 8 stays on the SIMT kernel)
template <class T, bool UPDATE, bool GRAM>
static bool launch_mma(BlockWorkspace<T>&, T, const T*, const T*, T, T*, const T*, T*, int) { return false; }
template <bool UPDATE, bool GRAM>
static bool launch_mma_f64(BlockWorkspace<double>& ws, double alpha, const double* In, const double* S, double beta, double* Out,
                           const double* Next, double* G, int rows) {
  Ctx& c = ws.ctx;
  const int mode = ws.mma_mode;
  if (mode == 0) return false;
  const int p = ws.p;
  if (!(p == 16 || p == 32 || (p == 8 && mode != 16))) return false;
  const int ntiles = (rows + 7) / 8;
  const int per_sm = p <= 16 ? 3 : 2;
  const int grid = std::max(1, std::min(sm_count() * per_sm, (ntiles + kMmaWarps - 1) / kMmaWarps));
  switch (p) {
    case 8: panel_mma_kernel<8, UPDATE, GRAM><<<grid, kMmaWarps * 32, 0, c.stream>>>(rows, alpha, In, S, beta, Out, Next, ws.part, c.tickets + 6, G); break;
    case 16: panel_mma_kernel<16, UPDATE, GRAM><<<grid, kMmaWarps * 32, 0, c.stream>>>(rows, alpha, In, S, beta, Out, Next, ws.part, c.tickets + 6, G); break;
    default: panel_mma_kernel<32, UPDATE, GRAM><<<grid, kMmaWarps * 32, 0, c.stream>>>(rows, alpha, In, S, beta, Out, Next, ws.part, c.tickets + 6, G); break;
  }
  KB_CUDA(cudaGetLastError()); c.launches++;
  return true;
}
template <> bool launch_mma<double, true, true>(BlockWorkspace<double>& ws, double al, const double* In, const double* S, double be, double* Out, const double* Nx, double* G, int rows) { return launch_mma_f64<true, true>(ws, al, In, S, be, Out, Nx, G, rows); }
template <> bool launch_mma<double, true, false>(BlockWorkspace<double>& ws, double al, const double* In, const double* S, double be, double* Out, const double* Nx, double* G, int rows) { return launch_mma_f64<true, false>(ws, al, In, S, be, Out, Nx, G, rows); }
template <> bool launch_mma<double, false, true>(BlockWorkspace<double>& ws, double al, const double* In, const double* S, double be, double* Out, const double* Nx, double* G, int rows) { return launch_mma_f64<false, true>(ws, al, In, S, be, Out, Nx, G, rows); }

// fast-path dispatch: true when p has a register-resident specialization
template <class T, bool UPDATE, bool GRAM>
static bool launch_fast(BlockWorkspace<T>& ws, T alpha, const T* In, const T* S, T beta, T* Out, const T* Next, T* G, int rows) {
  Ctx& c = ws.ctx;
  if (ws.generic_kernels) return false;
  if (launch_mma<T, UPDATE, GRAM>(ws, alpha, In, S, beta, Out, Next, G, rows)) return true;
  const int grid = ws.fast_grid;
  // the second lanes-per-row shape of P = 8 / 16 (sweeps, profiles/sweep_block.py) and software-pipelined row loads
  const bool alt = ws.fast_alt_tpr;
  const bool prefetch = ws.fast_prefetch;
#define KB_FAST(PV, TV)                                                                                                   \
  do {                                                                                                                    \
    if (prefetch)                                                                                                         \
      panel_fast_kernel<T, PV, TV, UPDATE, GRAM, true><<<grid, kBlock, 0, c.stream>>>(rows, alpha, In, S, beta, Out, Next, \
                                                                                      ws.part, c.tickets + 6, G);         \
    else                                                                                                                  \
      panel_fast_kernel<T, PV, TV, UPDATE, GRAM, false><<<grid, kBlock, 0, c.stream>>>(rows, alpha, In, S, beta, Out, Next, \
                                                                                       ws.part, c.tickets + 6, G);        \
  } while (0)
  switch (ws.p) {
    case 2: KB_FAST(2, 1); break;
    case 4: KB_FAST(4, 1); break;
    case 8: if (alt) KB_FAST(8, 4); else KB_FAST(8, 2); break;
    case 16: if (alt) KB_FAST(16, 4); else KB_FAST(16, 8); break;
    case 32: KB_FAST(32, 16); break;
    default: return false;
  }
#undef KB_FAST
  KB_CUDA(cudaGetLastError()); c.launches++;
  return true;
}

// `rows` < 0: the whole panel (ws.n rows); otherwise the first `rows` rows starting at the given pointers
template <class T> static void k_panel_tn(BlockWorkspace<T>& ws, const T* V, const T* Q, T* G, int rows = -1) {
  Ctx& c = ws.ctx;
  const int p = ws.p;
  if (rows < 0) rows = ws.n;
  if (launch_fast<T, false, true>(ws, T(0), (const T*)nullptr, (const T*)nullptr, T(0), const_cast<T*>(Q), V == Q ? (const T*)nullptr : V, G, rows)) return;
  const size_t smem = sizeof(T) * ((size_t)2 * kPanelTileElems);
  panel_tn_kernel<T><<<ws.grid, kBlock, smem, c.stream>>>(rows, p, V, Q, ws.part, c.tickets + 6, G);
  KB_CUDA(cudaGetLastError()); c.launches++;
}
template <class T> static void k_panel_nn_tn(BlockWorkspace<T>& ws, T alpha, const T* In, const T* S, T beta, T* Out, const T* Next, T* G,
                                             int rows = -1) {
  Ctx& c = ws.ctx;
  const int p = ws.p;
  if (rows < 0) rows = ws.n;
  if (launch_fast<T, true, true>(ws, alpha, In, S, beta, Out, Next, G, rows)) return;
  const size_t smem = sizeof(T) * ((size_t)3 * kPanelTileElems + (size_t)p * p);
  ensure_dyn_smem((const void*)panel_nn_tn_kernel<T>, 96 * 1024);
  panel_nn_tn_kernel<T><<<ws.grid, kBlock, smem, c.stream>>>(rows, p, alpha, In, S, beta, Out, Next, ws.part, c.tickets + 6, G);
  KB_CUDA(cudaGetLastError()); c.launches++;
}
template <class T> static void k_panel_nn(BlockWorkspace<T>& ws, T alpha, const T* In, const T* S, T beta, T* Out, int rows = -1) {
  Ctx& c = ws.ctx;
  const int p = ws.p;
  if (rows < 0) rows = ws.n;
  if (launch_fast<T, true, false>(ws, alpha, In, S, beta, Out, (const T*)nullptr, (T*)nullptr, rows)) return;
  const size_t smem = sizeof(T) * ((size_t)2 * kPanelTileElems + (size_t)p * p);
  panel_nn_kernel<T><<<ws.grid, kBlock, smem, c.stream>>>(rows, p, alpha, In, S, beta, Out);
  KB_CUDA(cudaGetLastError()); c.launches++;
}
// block operator application: CSR (SpMM), diagonal, or a user block callback on host / device panels (column-major)
template <class T> static void block_apply(BlockWorkspace<T>& ws, const BlockOp<T>& op, const T* X, T* Y, bool ldiv) {
  Ctx& c = ws.ctx;
  const int n = ws.n, p = ws.p;
  switch (op.kind) {
    case BlockOp<T>::CSR: k_spmm<T>(c, *op.csr, p, X, Y); break;
    case BlockOp<T>::DIAG: k_rows_diag<T>(c, n, p, op.diag, X, Y, ldiv); break;
    case BlockOp<T>::HOST_CB: {
      // the callback sees the reference's column-major blocks in host memory (krylov.h:105-107)
      k_transpose<T>(c, n, p, X, ws.tmp);
      KB_CUDA(cudaMemcpyAsync(ws.hX, ws.tmp, sizeof(T) * (size_t)n * p, cudaMemcpyDeviceToHost, c.stream));
      c.sync();
      op.fn(ws.hX, ws.hY, p, op.userdata);
      KB_CUDA(cudaMemcpyAsync(ws.tmp, ws.hY, sizeof(T) * (size_t)n * p, cudaMemcpyHostToDevice, c.stream));
      k_transpose<T>(c, p, n, ws.tmp, Y);
      break;
    }
    case BlockOp<T>::DEV_CB: {
      k_transpose<T>(c, n, p, X, ws.tmp);
      c.sync();
      op.fn(ws.tmp, ws.tmp2, p, op.userdata);
      KB_CUDA(cudaDeviceSynchronize());
      k_transpose<T>(c, p, n, ws.tmp2, Y);
      break;
    }
    default: throw std::runtime_error("block operator missing");
  }
}

// householder!(Q, R, tau) with compact = false on an n x p device panel: dst <- orthonormal factor (dst may be Q),
// Rout <- p x p R.  Q is used as scratch.  gram_ready: Q^T Q is already in the pinned G block (the fused
// Gram-Schmidt chain produced it and the caller synchronised).
// Pinned layout of ws.hsmall: [G | top p rows of Q | Tinv pass 0 | Tinv pass 1 | slots...].
template <class T> static void panel_qr(BlockWorkspace<T>& ws, T* Q, T* Rout, T* dst, bool gram_ready) {
  Ctx& c = ws.ctx;
  const int n = ws.n, p = ws.p, pp = p * p;
  T* hG = ws.hsmall;
  T* hTop = ws.hsmall + pp;
  T* hT[2] = {ws.hsmall + 2 * pp, ws.hsmall + 3 * pp};
  std::vector<T> R1(pp), R2(pp), tmp(pp), sgn(p);
  int failed_pass = -1;
  if (!gram_ready) {
    k_panel_tn<T>(ws, Q, Q, ws.dG);
    KB_CUDA(cudaMemcpyAsync(hG, ws.dG, sizeof(T) * pp, cudaMemcpyDeviceToHost, c.stream));
    c.sync();
  }
  // pass 0: Q <- Q R1^-1, fused with the Gram matrix of the result
  const bool force_householder = getenv("KB200_QR_FORCE_HOUSEHOLDER") != nullptr;   // tests: exercise the slow path on full-rank panels
  if (!force_householder && dense::cholesky_upper<T>(p, hG, R1.data())) {
    dense::inv_upper<T>(p, R1.data(), hT[0]);
    KB_CUDA(cudaMemcpyAsync(ws.dS, hT[0], sizeof(T) * pp, cudaMemcpyHostToDevice, c.stream));
    k_panel_nn_tn<T>(ws, T(1), Q, ws.dS, T(0), Q, (const T*)nullptr, ws.dG);
    KB_CUDA(cudaMemcpyAsync(hG, ws.dG, sizeof(T) * pp, cudaMemcpyDeviceToHost, c.stream));
    KB_CUDA(cudaMemcpyAsync(hTop, Q, sizeof(T) * pp, cudaMemcpyDeviceToHost, c.stream));   // first p rows (row-major panel)
    c.sync();
    // pass 1: dst <- Q R2^-1 S with S the Householder signs
    if (dense::cholesky_upper<T>(p, hG, R2.data())) {
      T* Tinv = hT[1];
      dense::inv_upper<T>(p, R2.data(), Tinv);
      std::vector<T> W(pp);                      // top block of the final orthonormal factor
      for (int r = 0; r < p; r++)
        for (int j = 0; j < p; j++) {
          T sacc = 0;
          for (int i = 0; i < p; i++) sacc += hTop[r * p + i] * Tinv[i + j * p];
          W[r + j * p] = sacc;
        }
      dense::householder_signs<T>(p, W.data(), sgn.data());
      for (int j = 0; j < p; j++) for (int i = 0; i < p; i++) Tinv[i + j * p] *= sgn[j];
      KB_CUDA(cudaMemcpyAsync(ws.dS, Tinv, sizeof(T) * pp, cudaMemcpyHostToDevice, c.stream));
      k_panel_nn<T>(ws, T(1), Q, ws.dS, T(0), dst);
      dense::matmul<T>(p, R2.data(), R1.data(), tmp.data());               // R = S R2 R1
      for (int j = 0; j < p; j++) for (int i = 0; i < p; i++) Rout[i + j * p] = i <= j ? sgn[i] * tmp[i + j * p] : T(0);
      return;
    }
    failed_pass = 1;
  } else {
    failed_pass = 0;
  }
  // rank-deficient (or too ill-conditioned) block: LAPACK's Householder algorithm (dgeqr2 + dorg2r), still on the
  // device.  Column j of the panel below row j IS the reflector direction, so applying H_j to the rows below j is a
  // right-multiplication of those rows by an elementary p x p matrix (panel_nn on a row range); the inner products
  // it needs are row j of the Gram matrix of the rows below j (panel_tn on the same range); only row j itself --
  // p numbers -- is patched from the host.  4p passes over the panel instead of 4: a fallback, counted.
  ws.qr_fallbacks++;
  std::vector<T> tau(p, T(0)), E(pp), Rh(pp, T(0));
  T* hE = hT[0];                                  // pinned staging: elementary matrix, patched row
  T* hRow = hT[1];
  auto gram_below = [&](int j) {                  // hG <- Gram of rows j+1.., hTop <- rows 0..p-1 (after a sync)
    const int below = n - (j + 1);
    if (below > 0) {
      k_panel_tn<T>(ws, Q + (size_t)(j + 1) * p, Q + (size_t)(j + 1) * p, ws.dG, below);
      KB_CUDA(cudaMemcpyAsync(hG, ws.dG, sizeof(T) * pp, cudaMemcpyDeviceToHost, c.stream));
    }
    KB_CUDA(cudaMemcpyAsync(hTop, Q, sizeof(T) * pp, cudaMemcpyDeviceToHost, c.stream));
    c.sync();
    if (below <= 0) for (int i = 0; i < pp; i++) hG[i] = T(0);
  };
  auto apply_below = [&](int j, const std::vector<T>& Em, const T* row, int ncopy) {
    // rows below j <- rows * Em ; row(s) 0..: ncopy leading entries of hTop-sized `row` buffer written back
    const int below = n - (j + 1);
    std::memcpy(hE, Em.data(), sizeof(T) * pp);
    if (below > 0) {
      KB_CUDA(cudaMemcpyAsync(ws.dS, hE, sizeof(T) * pp, cudaMemcpyHostToDevice, c.stream));
      k_panel_nn<T>(ws, T(1), Q + (size_t)(j + 1) * p, ws.dS, T(0), Q + (size_t)(j + 1) * p, below);
    }
    KB_CUDA(cudaMemcpyAsync(Q, row, sizeof(T) * (size_t)ncopy, cudaMemcpyHostToDevice, c.stream));
    c.sync();
  };
  for (int j = 0; j < p; j++) {                   // dgeqr2: reflectors H_0 .. H_{p-1}
    gram_below(j);
    const T alpha_j = hTop[j * p + j], xn2 = hG[j + j * p];      // hTop is row-major (rows of the panel)
    if (xn2 == T(0)) { tau[j] = T(0); continue; }
    const T beta_j = -std::copysign(std::sqrt(alpha_j * alpha_j + xn2), alpha_j);
    tau[j] = (beta_j - alpha_j) / beta_j;
    const T scal = T(1) / (alpha_j - beta_j);
    for (int i = 0; i < pp; i++) E[i] = T(0);
    for (int i = 0; i < p; i++) E[i + i * p] = T(1);
    E[j + j * p] = scal;
    std::memcpy(hRow, hTop, sizeof(T) * pp);
    for (int k = j + 1; k < p; k++) {
      const T vTa = hTop[j * p + k] + scal * hG[j + k * p];       // v^T A_k, v = [1; scal * A(j+1:, j)]
      E[j + k * p] = -tau[j] * vTa * scal;
      hRow[j * p + k] = hTop[j * p + k] - tau[j] * vTa;
    }
    hRow[j * p + j] = beta_j;
    apply_below(j, E, hRow, (j + 1) * p);
  }
  gram_below(p - 1);                              // refresh hTop: R is its upper triangle
  for (int jc = 0; jc < p; jc++) for (int i = 0; i <= jc; i++) Rh[i + jc * p] = hTop[i * p + jc];
  for (int j = p - 1; j >= 0; j--) {              // dorg2r: accumulate Q = H_0 ... H_{p-1} [I; 0]
    gram_below(j);
    for (int i = 0; i < pp; i++) E[i] = T(0);
    for (int i = 0; i < p; i++) E[i + i * p] = T(1);
    std::memcpy(hRow, hTop, sizeof(T) * pp);
    for (int k = j + 1; k < p; k++) {
      const T w = hTop[j * p + k] + hG[j + k * p];               // v^T A_k with v_j = 1
      E[j + k * p] = -tau[j] * w;
      hRow[j * p + k] = hTop[j * p + k] - tau[j] * w;
    }
    E[j + j * p] = -tau[j];
    hRow[j * p + j] = T(1) - tau[j];
    for (int i = 0; i < j; i++) hRow[i * p + j] = T(0);
    apply_below(j, E, hRow, (j + 1) * p);
  }
  if (dst != Q) k_copy<T>(c, n * p, dst, Q);
  c.sync();
  if (failed_pass == 1) { dense::matmul<T>(p, Rh.data(), R1.data(), tmp.data()); Rh = tmp; }   // Q was already Q R1^-1
  for (int i = 0; i < pp; i++) Rout[i] = Rh[i];
}

// ---------------------------------------------------------------------------
// workspace
// ---------------------------------------------------------------------------
template <class T> static void ensure_small(BlockWorkspace<T>& ws, int nblocks) {
  // device Psi blocks and pinned slots for `nblocks` p x p blocks (+4 pinned blocks for the panel QR)
  const size_t pp = (size_t)ws.p * ws.p;
  while ((int)ws.dPsi.size() < nblocks) {
    T* d = nullptr;
    KB_CUDA(cudaMalloc(&d, sizeof(T) * pp));
    ws.dPsi.push_back(d);
  }
  const size_t need = (size_t)(nblocks + 4) * pp;
  if (need > ws.hsmall_cap) {
    ws.ctx.sync();
    if (ws.hsmall) KB_CUDA(cudaFreeHost(ws.hsmall));
    ws.hsmall_cap = 2 * need;
    KB_CUDA(cudaHostAlloc(&ws.hsmall, sizeof(T) * ws.hsmall_cap, cudaHostAllocDefault));
  }
}
template <class T> static T* slot(BlockWorkspace<T>& ws, int i) { return ws.hsmall + (size_t)(4 + i) * ws.p * ws.p; }

template <class T> BlockWorkspace<T>* block_ws_create(int m, int n, int p, int memory, int device) {
  const double t0 = now_seconds();
  if (m != n) throw std::runtime_error("System must be square");
  if (p < 1 || p > kMaxBlockP) throw std::runtime_error("block size p must be in 1..32 on the GPU path");
  if (n < p) throw std::runtime_error("block size exceeds the number of rows");
  BlockWorkspace<T>* ws = new BlockWorkspace<T>();
  try {
    ws->m = m; ws->n = n; ws->p = p;
    ws->ctx.init(device);
    int mem = memory > 0 ? memory : 5;                          // block_gmres.jl:99
    if (mem > n / p) mem = n / p;                               // block_krylov_workspaces.jl:138
    ws->memory = mem;
    const size_t np = (size_t)n * p, pp = (size_t)p * p;
    ws->X = dev_alloc<T>(np); ws->W = dev_alloc<T>(np);
    ws->tmp = dev_alloc<T>(np);
    for (int i = 0; i < mem; i++) ws->V.push_back(dev_alloc<T>(np));
    ws->Z.assign(mem, std::vector<T>(pp)); ws->R.assign((size_t)mem * (mem + 1) / 2, std::vector<T>(pp));
    ws->H.assign(mem, std::vector<T>(2 * pp)); ws->tau.assign(mem, std::vector<T>(p));
    ws->C.assign(pp, T(0)); ws->D.assign(2 * pp, T(0));
    ws->grid = panel_grid<T>(n, p);
    ws->fast_grid = std::max(1, std::min(sm_count() * 2, (int)(((long long)n + kBlock - 1) / kBlock)));
    ws->generic_kernels = getenv("KB200_BLOCK_GENERIC") != nullptr;     // tests: force the tiled any-p kernels
    const char* mma_env = getenv("KB200_BLOCK_MMA");
    ws->mma_mode = mma_env ? atoi(mma_env) : 1;
    ws->fast_prefetch = getenv("KB200_FAST_PREFETCH") != nullptr;
    ws->fast_alt_tpr = getenv("KB200_FAST_TPR") != nullptr;
    // partial Gram matrices: one p x p block per CTA of whichever panel kernel runs (tiled, register-resident, or the
    // tensor-core kernels with up to 3 CTAs of 8 warps per SM, one 8-row tile per warp)
    const int mma_grid = std::max(1, std::min(sm_count() * 3, (int)((((long long)n + 7) / 8 + kMmaWarps - 1) / kMmaWarps)));
    ws->part = dev_alloc<T>((size_t)std::max(std::max(ws->grid, ws->fast_grid), mma_grid) * pp);
    KB_CUDA(cudaMalloc(&ws->dG, sizeof(T) * pp));
    KB_CUDA(cudaMalloc(&ws->dS, sizeof(T) * pp));
    ensure_small(*ws, mem + 1);
  } catch (...) {
    block_ws_destroy(ws);
    throw;
  }
  ws->stats.allocation_timer = now_seconds() - t0;
  return ws;
}

template <class T> void block_ws_destroy(BlockWorkspace<T>* ws) {
  if (!ws) return;
  if (ws->ctx.stream) cudaStreamSynchronize(ws->ctx.stream);
  T* vecs[] = {ws->X, ws->dX, ws->W, ws->P, ws->Q, ws->Bbuf, ws->tmp, ws->tmp2, ws->part};
  for (T* v : vecs) dev_free(v);
  for (T* v : ws->V) dev_free(v);
  for (T* d : ws->dPsi) cudaFree(d);
  if (ws->dG) cudaFree(ws->dG);
  if (ws->dS) cudaFree(ws->dS);
  if (ws->hsmall) cudaFreeHost(ws->hsmall);
  if (ws->hX) cudaFreeHost(ws->hX);
  if (ws->hY) cudaFreeHost(ws->hY);
  ws->ctx.destroy();
  delete ws;
}

template <class T> static void alloc_panel_if(bool cond, BlockWorkspace<T>& ws, T*& v) {
  const double t0 = now_seconds();
  if (cond && !v) v = dev_alloc<T>((size_t)ws.n * ws.p);
  ws.stats.allocation_timer += now_seconds() - t0;
}

template <class T> void block_warm_start(BlockWorkspace<T>& ws, const T* X0_colmajor_dev) {
  alloc_panel_if(true, ws, ws.dX);
  k_transpose<T>(ws.ctx, ws.p, ws.n, X0_colmajor_dev, ws.dX);
  ws.ctx.sync();
  ws.warm_start = true;
}

template <class T> void block_get_X(BlockWorkspace<T>& ws, T* X_colmajor_dev) {
  k_transpose<T>(ws.ctx, ws.n, ws.p, ws.X, X_colmajor_dev);
  ws.ctx.sync();
}

template <class T> void block_spmm(Ctx& c, const Csr<T>& A, int p, const T* X, T* Y, int variant) {
  if (p < 1 || p > kMaxBlockP) throw std::runtime_error("block size p must be in 1..32");
  k_spmm<T>(c, A, p, X, Y, variant);
  c.sync();
}

// One panel operation through the solver's own launchers.  path 0 keeps the workspace's dispatch; the others set
// the dispatch fields for this call only: 1 DMMA, 2 SIMT, 3 SIMT with prefetch, 4 SIMT with the alternative
// lanes-per-row shape, 5 tiled.
template <class T>
void block_panel_op(BlockWorkspace<T>& ws, int op, int path, int rows, T alpha, const T* In, const T* S, T beta, T* Out, const T* Next,
                    T* G) {
  const int p = ws.p;
  const bool simt_p = p == 2 || p == 4 || p == 8 || p == 16 || p == 32;
  bool ok = path == 0 || path == 5;
  if (path == 1) ok = sizeof(T) == sizeof(double) && (p == 8 || p == 16 || p == 32);
  if (path == 2 || path == 3) ok = simt_p;
  if (path == 4) ok = p == 8 || p == 16;
  if (!ok) throw std::runtime_error("no panel kernel for this path, dtype and block size");
  if (op < 0 || op > 2) throw std::runtime_error("op must be 0, 1 or 2");
  if (rows < 1 || rows > ws.n) throw std::runtime_error("rows must be in 1..n of the workspace");
  if (!Out || (op != 1 && !G) || (op != 0 && (!In || !S))) throw std::runtime_error("missing operand");
  const bool generic = ws.generic_kernels, prefetch = ws.fast_prefetch, alt = ws.fast_alt_tpr;
  const int mma = ws.mma_mode;
  if (path != 0) {
    ws.generic_kernels = path == 5;
    ws.mma_mode = path == 1 ? 1 : 0;
    ws.fast_prefetch = path == 3;
    ws.fast_alt_tpr = path == 4;
  }
  auto restore = [&]() { ws.generic_kernels = generic; ws.fast_prefetch = prefetch; ws.fast_alt_tpr = alt; ws.mma_mode = mma; };
  try {
    if (op == 0) k_panel_tn<T>(ws, Next ? Next : Out, Out, G, rows);
    else if (op == 1) k_panel_nn<T>(ws, alpha, In, S, beta, Out, rows);
    else k_panel_nn_tn<T>(ws, alpha, In, S, beta, Out, Next, G, rows);
    ws.ctx.sync();
  } catch (...) {
    restore();
    throw;
  }
  restore();
}

// ===========================================================================
// block_gmres!  (src/block_gmres.jl:110-359)
// ===========================================================================
template <class T>
void block_gmres_solve(BlockWorkspace<T>& ws, const BlockOp<T>& A, const T* B_colmajor, const BlockOp<T>& M, const BlockOp<T>& N,
                       const SolveOpts& o) {
  const double start_time = now_seconds();
  Ctx& cx = ws.ctx;
  const int n = ws.n, p = ws.p;
  const int np = n * p;                        // panels are addressed as vectors of length n p by the BLAS-1 kernels
  if ((long long)n * p > 2147483647LL) throw std::runtime_error("n * p exceeds the 32-bit panel index");
  const size_t pp = (size_t)p * p;
  const bool history = o.history, ldiv = o.ldiv, restart = o.restart, reorth = o.reorthogonalization;
  if (o.verbose > 0) printf("BLOCK-GMRES: system of size %d with %d right-hand sides\n", n, p);
  const bool MisI = M.is_identity(), NisI = N.is_identity();
  alloc_panel_if(!MisI, ws, ws.Q);
  alloc_panel_if(!NisI, ws, ws.P);
  alloc_panel_if(restart, ws, ws.dX);
  alloc_panel_if(true, ws, ws.Bbuf);
  if (A.kind == BlockOp<T>::DEV_CB || M.kind == BlockOp<T>::DEV_CB || N.kind == BlockOp<T>::DEV_CB) alloc_panel_if(true, ws, ws.tmp2);
  if (A.kind == BlockOp<T>::HOST_CB || M.kind == BlockOp<T>::HOST_CB || N.kind == BlockOp<T>::HOST_CB) {
    if (!ws.hX) KB_CUDA(cudaHostAlloc(&ws.hX, sizeof(T) * (size_t)np, cudaHostAllocDefault));
    if (!ws.hY) KB_CUDA(cudaHostAlloc(&ws.hY, sizeof(T) * (size_t)np, cudaHostAllocDefault));
  }
  T *dX = ws.dX, *X = ws.X, *W = ws.W;
  std::vector<T*>& V = ws.V;
  std::vector<std::vector<T>>&Z = ws.Z, &R = ws.R, &H = ws.H, &tau = ws.tau;
  std::vector<T>&C = ws.C, &D = ws.D;
  Stats& stats = ws.stats;
  const bool warm_start = ws.warm_start;
  stats.reset();
  T* Q = MisI ? W : ws.Q;
  T* R0 = MisI ? W : ws.Q;
  T* Xr = restart ? dX : X;
  T* B = ws.Bbuf;
  const int ldd = 2 * p;
  T* D1 = D.data(); T* D2 = D.data() + p;      // D1 = D[1:p,:], D2 = D[p+1:2p,:]
  auto frob = [&](const std::vector<T>& Mx) { T s = 0; for (T v : Mx) s += v * v; return (T)std::sqrt(s); };

  k_transpose<T>(cx, p, n, B_colmajor, B);     // B as a row-major panel
  k_fill<T>(cx, np, X, T(0));
  if (warm_start) {
    block_apply(ws, A, dX, W, false);
    k_axpby<T>(cx, np, T(1), B, T(-1), W);     // W = B - W
    if (restart) k_axpy<T>(cx, np, T(1), dX, X);
  } else {
    k_copy<T>(cx, np, W, B);
  }
  if (!MisI) block_apply(ws, M, W, R0, ldiv);
  T RNorm = k_nrm2<T>(cx, np, R0);             // Frobenius norm
  if (history) stats.residuals.push_back(RNorm);
  const T eps_tol = tol_of<T>(o.atol) + tol_of<T>(o.rtol) * RNorm;
  const int mem = (int)V.size();
  int npass = 0, iter = 0, inner_iter = 0;
  const int itmax = o.itmax == 0 ? 2 * (n / p) : o.itmax;
  int inner_itmax = itmax;
  if (o.verbose > 0) printf("%5s  %5s  %7s  %5s\n", "pass", "k", "‖Rₖ‖", "timer");
  if (kdisplay(iter, o.verbose)) printf("%5d  %5d  %7.1e  %.2fs\n", npass, iter, (double)RNorm, now_seconds() - start_time);
  bool solved = RNorm <= eps_tol, tired = iter >= itmax, inner_tired = inner_iter >= inner_itmax;
  bool user_exit = false, overtimed = false;
  std::string status = "unknown";

  while (!(solved || tired || user_exit || overtimed)) {
    int nr = 0;
    // (the reference zero-fills V every cycle; every block read below is written first)
    for (auto& Psi : R) std::fill(Psi.begin(), Psi.end(), T(0));
    for (auto& blk : Z) std::fill(blk.begin(), blk.end(), T(0));
    if (restart) {
      k_fill<T>(cx, np, Xr, T(0));
      if (npass >= 1) {
        block_apply(ws, A, X, W, false);
        k_axpby<T>(cx, np, T(1), B, T(-1), W);
        if (!MisI) block_apply(ws, M, W, R0, ldiv);
      }
    }
    panel_qr<T>(ws, R0, Z[0].data(), V[0], false);   // copyto!(V[1], R0); householder!: Gamma (Z[1]) and V_1
    npass = npass + 1;
    inner_iter = 0;
    inner_tired = false;

    while (!(solved || inner_tired || user_exit || overtimed)) {
      inner_iter = inner_iter + 1;
      if (!restart && (inner_iter > mem)) {     // block_gmres.jl:231-239
        const double t0 = now_seconds();
        for (int i = 0; i < inner_iter; i++) R.push_back(std::vector<T>(pp, T(0)));
        H.push_back(std::vector<T>(2 * pp, T(0)));
        tau.push_back(std::vector<T>(p, T(0)));
        stats.allocation_timer += now_seconds() - t0;
      }
      ensure_small(ws, inner_iter + 1);
      T* Vk = V[inner_iter - 1];
      T* P = NisI ? Vk : ws.P;
      if (!NisI) block_apply(ws, N, Vk, P, ldiv);
      block_apply(ws, A, P, W, false);
      if (!MisI) block_apply(ws, M, W, Q, ldiv);
      // block modified Gram-Schmidt.  The Psi blocks stay on the device between the product that makes them and the
      // update that consumes them; each update Q -= V_i Psi_i also forms the next product (Psi_{i+1} = V_{i+1}^T Q,
      // or the Gram matrix Q^T Q the panel QR starts from) in the same pass; host copies arrive after one sync.
      T* dst = inner_iter < (int)V.size() ? V[inner_iter] : Q;      // where V_{k+1} goes (no separate copy)
      if (!reorth) {
        k_panel_tn<T>(ws, V[0], Q, ws.dPsi[0]);
        for (int i = 0; i < inner_iter; i++) {
          const bool last = i + 1 == inner_iter;
          k_panel_nn_tn<T>(ws, T(-1), V[i], ws.dPsi[i], T(1), Q, last ? (const T*)nullptr : V[i + 1], last ? ws.dG : ws.dPsi[i + 1]);
          KB_CUDA(cudaMemcpyAsync(slot(ws, i), ws.dPsi[i], sizeof(T) * pp, cudaMemcpyDeviceToHost, cx.stream));
        }
        KB_CUDA(cudaMemcpyAsync(ws.hsmall, ws.dG, sizeof(T) * pp, cudaMemcpyDeviceToHost, cx.stream));
        cx.sync();
        for (int i = 0; i < inner_iter; i++) std::memcpy(R[nr + i].data(), slot(ws, i), sizeof(T) * pp);
        panel_qr<T>(ws, Q, C.data(), dst, true);  // V_{k+1} in dst, Psi_{k+1,k} in C
      } else {
        for (int pass = 0; pass < 2; pass++) {    // second pass: reorthogonalization, block_gmres.jl:250-256
          for (int i = 0; i < inner_iter; i++) {
            k_panel_tn<T>(ws, V[i], Q, ws.dPsi[i]);
            k_panel_nn<T>(ws, T(-1), V[i], ws.dPsi[i], T(1), Q);
            KB_CUDA(cudaMemcpyAsync(slot(ws, i), ws.dPsi[i], sizeof(T) * pp, cudaMemcpyDeviceToHost, cx.stream));
          }
          cx.sync();
          for (int i = 0; i < inner_iter; i++) {
            const T* t = slot(ws, i);
            if (pass == 0) std::memcpy(R[nr + i].data(), t, sizeof(T) * pp);
            else for (size_t k = 0; k < pp; k++) R[nr + i][k] += t[k];
          }
        }
        panel_qr<T>(ws, Q, C.data(), dst, false);
      }
      for (int i = 0; i < inner_iter - 1; i++) {  // previous reflections, block_gmres.jl:268-274
        for (int c = 0; c < p; c++) for (int r = 0; r < p; r++) { D1[r + c * ldd] = R[nr + i][r + c * p]; D2[r + c * ldd] = R[nr + i + 1][r + c * p]; }
        dense::orm2r_lt<T>(2 * p, p, p, H[i].data(), 2 * p, tau[i].data(), D.data(), ldd);
        for (int c = 0; c < p; c++) for (int r = 0; r < p; r++) { R[nr + i][r + c * p] = D1[r + c * ldd]; R[nr + i + 1][r + c * p] = D2[r + c * ldd]; }
      }
      std::vector<T>& Hk = H[inner_iter - 1];
      for (int c = 0; c < p; c++) for (int r = 0; r < p; r++) { Hk[r + c * 2 * p] = R[nr + inner_iter - 1][r + c * p]; Hk[p + r + c * 2 * p] = C[r + c * p]; }
      dense::householder_compact<T>(2 * p, p, Hk.data(), R[nr + inner_iter - 1].data(), tau[inner_iter - 1].data());
      for (int c = 0; c < p; c++) for (int r = 0; r < p; r++) { D1[r + c * ldd] = Z[inner_iter - 1][r + c * p]; D2[r + c * ldd] = T(0); }
      dense::orm2r_lt<T>(2 * p, p, p, Hk.data(), 2 * p, tau[inner_iter - 1].data(), D.data(), ldd);
      for (int c = 0; c < p; c++) for (int r = 0; r < p; r++) Z[inner_iter - 1][r + c * p] = D1[r + c * ldd];
      for (int c = 0; c < p; c++) for (int r = 0; r < p; r++) C[r + c * p] = D2[r + c * ldd];
      RNorm = frob(C);
      if (history) stats.residuals.push_back(RNorm);
      nr = nr + inner_iter;
      if (o.callback) { cx.sync(); stats.niter = iter + inner_iter; user_exit = o.callback(&ws, o.callback_user) != 0; }
      solved = RNorm <= eps_tol;
      inner_tired = restart ? inner_iter >= std::min(mem, inner_itmax) : inner_iter >= inner_itmax;
      overtimed = (now_seconds() - start_time) > o.timemax;
      if (kdisplay(iter + inner_iter, o.verbose)) printf("%5d  %5d  %7.1e  %.2fs\n", npass, iter + inner_iter, (double)RNorm, now_seconds() - start_time);
      if (!(solved || inner_tired || user_exit || overtimed)) {
        if (!restart && (inner_iter >= mem)) {
          const double t0 = now_seconds();
          V.push_back(dev_alloc<T>((size_t)np));
          Z.push_back(std::vector<T>(pp, T(0)));
          stats.allocation_timer += now_seconds() - t0;
        }
        if (dst != V[inner_iter]) k_copy<T>(cx, np, V[inner_iter], Q);     // only when V grew just now (copyto!(V[k+1], Q))
        for (int c = 0; c < p; c++) for (int r = 0; r < p; r++) Z[inner_iter][r + c * p] = D2[r + c * ldd];
      }
    }
    std::vector<std::vector<T>>& Y = Z;         // block back substitution, block_gmres.jl:316-324
    for (int i = inner_iter; i >= 1; i--) {
      int pos = nr + i - inner_iter;
      for (int j = inner_iter; j >= i + 1; j--) {
        for (int c = 0; c < p; c++)
          for (int r = 0; r < p; r++) {
            T acc = 0;
            for (int k = 0; k < p; k++) acc += R[pos - 1][r + k * p] * Y[j - 1][k + c * p];
            Y[i - 1][r + c * p] -= acc;
          }
        pos = pos - j + 1;
      }
      for (int c = 0; c < p; c++)
        for (int r = p - 1; r >= 0; r--) {
          T acc = Y[i - 1][r + c * p];
          for (int k = r + 1; k < p; k++) acc -= R[pos - 1][r + k * p] * Y[i - 1][k + c * p];
          Y[i - 1][r + c * p] = acc / R[pos - 1][r + r * p];
        }
    }
    ensure_small(ws, inner_iter + 1);
    for (int i = 0; i < inner_iter; i++) {      // X_r += V_i Y_i
      std::memcpy(slot(ws, i), Y[i].data(), sizeof(T) * pp);
      KB_CUDA(cudaMemcpyAsync(ws.dPsi[i], slot(ws, i), sizeof(T) * pp, cudaMemcpyHostToDevice, cx.stream));
      k_panel_nn<T>(ws, T(1), V[i], ws.dPsi[i], T(1), Xr);
    }
    if (!NisI) { k_copy<T>(cx, np, ws.P, Xr); block_apply(ws, N, ws.P, Xr, ldiv); }
    if (restart) k_axpy<T>(cx, np, T(1), Xr, X);
    cx.sync();
    inner_itmax = inner_itmax - inner_iter;
    iter = iter + inner_iter;
    tired = iter >= itmax;
    overtimed = (now_seconds() - start_time) > o.timemax;
  }
  if (o.verbose > 0) printf("\n");
  if (tired) status = "maximum number of iterations exceeded";
  if (solved) status = "solution good enough given atol and rtol";
  if (overtimed) status = "time limit exceeded";
  if (user_exit) status = "user-requested exit";
  if (warm_start && !restart) k_axpy<T>(cx, np, T(1), dX, X);
  ws.warm_start = false;
  cx.sync();
  stats.niter = iter; stats.solved = solved;
  stats.timer = now_seconds() - start_time;
  stats.status = status;
}

#define INST(T)                                                                                                  \
  template BlockWorkspace<T>* block_ws_create<T>(int, int, int, int, int);                                       \
  template void block_ws_destroy<T>(BlockWorkspace<T>*);                                                         \
  template void block_gmres_solve<T>(BlockWorkspace<T>&, const BlockOp<T>&, const T*, const BlockOp<T>&, const BlockOp<T>&, const SolveOpts&); \
  template void block_warm_start<T>(BlockWorkspace<T>&, const T*);                                               \
  template void block_get_X<T>(BlockWorkspace<T>&, T*);                                                          \
  template void block_spmm<T>(Ctx&, const Csr<T>&, int, const T*, T*, int);                                      \
  template void block_panel_op<T>(BlockWorkspace<T>&, int, int, int, T, const T*, const T*, T, T*, const T*, T*);
INST(double)
INST(float)
#undef INST

}  // namespace kb
