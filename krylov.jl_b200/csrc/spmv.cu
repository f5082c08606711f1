// spmv.cu -- the CSR operator: upload/normalisation, staging plan, and the
// y = A x kernels that stand in for `kmul!(y, A, x)` = mul!(y, A, x)
// (src/krylov_utils.jl:305; call sites cg.jl:196, gmres.jl:257,
// bicgstab.jl:221,228, minres.jl:289).
#include "kb_internal.h"
#include "spmv_tiles.cuh"

#include <algorithm>
#include <cstring>
#include <vector>

namespace kb {

// ---------------------------------------------------------------------------
// Upload: accept the caller's (rowptr, colind, val) with 0/1-based, 32/64-bit
// indices on host or device; store int32 0-based in padded device arrays.
// The bijection (shift by index_base, narrow to int32) keeps every
// (row, col, val) triplet of the input -- "bit-exact integer indexing".
// ---------------------------------------------------------------------------
template <class I>
__global__ void index_convert_kernel(long long cnt, const I* __restrict__ in, int* __restrict__ out, int base, int* bad) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < cnt; i += stride) {
    long long v = (long long)in[i] - base;
    if (v < 0 || v > 2147483647LL) atomicExch(bad, 1);
    out[i] = (int)v;
  }
}

__global__ void fill_int_kernel(int cnt, int* out, int v) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < cnt) out[i] = v;
}

template <class T>
void csr_upload(Ctx& c, Csr<T>& A, int n, long long nnz, const void* rowptr, const void* colind, const T* val,
                int index_base, int index_bytes, bool on_device, int ncols, CsrDict<T>* dict) {
  if (ncols < 0) ncols = n;
  if (n < 0 || nnz < 0 || nnz > 2147483647LL - 64) throw std::runtime_error("CSR operator: n/nnz out of int32 range");
  if (index_bytes != 4 && index_bytes != 8) throw std::runtime_error("CSR operator: index_bytes must be 4 or 8");
  if (index_base != 0 && index_base != 1) throw std::runtime_error("CSR operator: index_base must be 0 or 1");
  csr_free(A);
  A.n = n; A.ncols = ncols; A.nnz = nnz;
  const size_t rp_len = (size_t)n + 1, rp_pad = kTileRows + 16;
  A.rowptr = dev_alloc<int>(rp_len + rp_pad);
  A.colind = dev_alloc<int>((size_t)nnz + 16);
  A.val = dev_alloc<T>((size_t)nnz + 16);
  const cudaMemcpyKind kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  KB_CUDA(cudaMemcpyAsync(A.val, val, sizeof(T) * (size_t)nnz, kind, c.stream));
  KB_CUDA(cudaMemsetAsync(A.val + nnz, 0, sizeof(T) * 16, c.stream));
  KB_CUDA(cudaMemsetAsync(A.colind + nnz, 0, sizeof(int) * 16, c.stream));
  int* bad = nullptr;
  KB_CUDA(cudaMalloc((void**)&bad, sizeof(int)));
  KB_CUDA(cudaMemsetAsync(bad, 0, sizeof(int), c.stream));
  void* tmp_rp = nullptr; void* tmp_ci = nullptr;
  if (index_bytes == 4 && index_base == 0) {
    KB_CUDA(cudaMemcpyAsync(A.rowptr, rowptr, sizeof(int) * rp_len, kind, c.stream));
    KB_CUDA(cudaMemcpyAsync(A.colind, colind, sizeof(int) * (size_t)nnz, kind, c.stream));
  } else {
    const void* drp = rowptr; const void* dci = colind;
    if (!on_device) {
      KB_CUDA(cudaMalloc(&tmp_rp, (size_t)index_bytes * rp_len));
      KB_CUDA(cudaMalloc(&tmp_ci, (size_t)index_bytes * (size_t)(nnz ? nnz : 1)));
      KB_CUDA(cudaMemcpyAsync(tmp_rp, rowptr, (size_t)index_bytes * rp_len, cudaMemcpyHostToDevice, c.stream));
      KB_CUDA(cudaMemcpyAsync(tmp_ci, colind, (size_t)index_bytes * (size_t)nnz, cudaMemcpyHostToDevice, c.stream));
      drp = tmp_rp; dci = tmp_ci;
    }
    const int g = sm_count() * 8;
    if (index_bytes == 8) {
      index_convert_kernel<long long><<<g, 256, 0, c.stream>>>((long long)rp_len, (const long long*)drp, A.rowptr, index_base, bad);
      index_convert_kernel<long long><<<g, 256, 0, c.stream>>>(nnz, (const long long*)dci, A.colind, index_base, bad);
    } else {
      index_convert_kernel<int><<<g, 256, 0, c.stream>>>((long long)rp_len, (const int*)drp, A.rowptr, index_base, bad);
      index_convert_kernel<int><<<g, 256, 0, c.stream>>>(nnz, (const int*)dci, A.colind, index_base, bad);
    }
    KB_CUDA(cudaGetLastError());
  }
  // rows past n (read by the last tile's row-pointer slice) are empty
  fill_int_kernel<<<((int)rp_pad + 255) / 256, 256, 0, c.stream>>>((int)rp_pad, A.rowptr + rp_len, (int)nnz);
  KB_CUDA(cudaGetLastError());
  int hbad = 0;
  KB_CUDA(cudaMemcpyAsync(&hbad, bad, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
  c.sync();
  cudaFree(bad);
  if (tmp_rp) cudaFree(tmp_rp);
  if (tmp_ci) cudaFree(tmp_ci);
  if (hbad) { csr_free(A); throw std::runtime_error("CSR operator: index outside int32 range after rebasing"); }
  try { csr_plan(c, A, dict); } catch (...) { csr_free(A); if (dict) csr_dict_free(*dict); throw; }
}

template <class T> void csr_free(Csr<T>& A) {
  dev_free(A.rowptr); dev_free(A.colind); dev_free(A.val);
  A = Csr<T>();
}

template <class T> void csr_dict_free(CsrDict<T>& D) {
  dev_free(D.mask);
  D = CsrDict<T>();
}

// ---------------------------------------------------------------------------
// Constant-coefficient encoding (CsrDict).  Deterministic, lock-free, bounded: round q finds the LOWEST-index
// nonzero whose (column - row, value bits) pair is not yet in the dictionary (atomicMin), one thread then locates
// its row by bisection of the row pointers, and the host appends the pair.  At most kDictSlots + 1 rounds: a
// (kDictSlots + 1)-th pair means the operator does not qualify.  Values compare by their bits, so 0.0 and -0.0 are
// different pairs and stored zeros stay.  A last pass writes one mask byte per row.
// ---------------------------------------------------------------------------
__device__ __host__ inline unsigned long long val_bits(double v) { unsigned long long b; memcpy(&b, &v, 8); return b; }
__device__ __host__ inline unsigned long long val_bits(float v) { unsigned b; memcpy(&b, &v, 4); return b; }

struct DictKeys { int npairs; int off[kDictSlots]; unsigned long long bits[kDictSlots]; };
template <class T> struct DictProbe { int k, off; T val; };

__device__ __forceinline__ int dict_slot(const DictKeys& K, int off, unsigned long long bits) {
  int s = -1;
  for (int u = 0; u < K.npairs; u++) s = (K.off[u] == off && K.bits[u] == bits) ? u : s;
  return s;
}

template <class T>
__global__ void dict_find_kernel(int n, const int* __restrict__ rowptr, const int* __restrict__ colind, const T* __restrict__ val,
                                 DictKeys K, DictProbe<T>* probe) {
  int best = 2147483647;
  const int stride = gridDim.x * blockDim.x;
  for (int row = blockIdx.x * blockDim.x + threadIdx.x; row < n; row += stride) {
    const int kb = rowptr[row], ke = rowptr[row + 1];
    for (int k = kb; k < ke && k < best; k++)
      if (dict_slot(K, colind[k] - row, val_bits(val[k])) < 0) { best = k; break; }
  }
  for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
  if ((threadIdx.x & 31) == 0 && best != 2147483647) atomicMin(&probe->k, best);
}

template <class T>
__global__ void dict_pair_kernel(int n, const int* __restrict__ rowptr, const int* __restrict__ colind, const T* __restrict__ val,
                                 DictProbe<T>* probe) {
  const int k = probe->k;
  if (k == 2147483647) return;
  int lo = 0, hi = n - 1;                  // the row of nonzero k: the last row whose first nonzero is <= k
  while (lo < hi) {
    const int mid = lo + (hi - lo + 1) / 2;
    if (rowptr[mid] <= k) lo = mid; else hi = mid - 1;
  }
  probe->off = colind[k] - lo;
  probe->val = val[k];
}

template <class T>
__global__ void dict_mask_kernel(int n, const int* __restrict__ rowptr, const int* __restrict__ colind, const T* __restrict__ val,
                                 DictKeys K, unsigned char* __restrict__ mask) {
  const int stride = gridDim.x * blockDim.x;
  for (int row = blockIdx.x * blockDim.x + threadIdx.x; row < n; row += stride) {
    unsigned m = 0;
    for (int k = rowptr[row]; k < rowptr[row + 1]; k++) m |= 1u << dict_slot(K, colind[k] - row, val_bits(val[k]));
    mask[row] = (unsigned char)m;
  }
}

template <class T> static void csr_dict_build(Ctx& c, const Csr<T>& A, CsrDict<T>& D) {
  DictKeys K;
  memset(&K, 0, sizeof(K));
  T hval[kDictSlots] = {};
  DictProbe<T>* dprobe = nullptr;
  KB_CUDA(cudaMalloc((void**)&dprobe, sizeof(DictProbe<T>)));
  const int g = sm_count() * 8;
  bool fits = true;
  for (;;) {
    DictProbe<T> h;
    memset(&h, 0, sizeof(h));
    h.k = 2147483647;
    KB_CUDA(cudaMemcpyAsync(dprobe, &h, sizeof(h), cudaMemcpyHostToDevice, c.stream));
    dict_find_kernel<T><<<g, 256, 0, c.stream>>>(A.n, A.rowptr, A.colind, A.val, K, dprobe);
    dict_pair_kernel<T><<<1, 1, 0, c.stream>>>(A.n, A.rowptr, A.colind, A.val, dprobe);
    KB_CUDA(cudaGetLastError());
    KB_CUDA(cudaMemcpyAsync(&h, dprobe, sizeof(h), cudaMemcpyDeviceToHost, c.stream));
    c.sync();
    if (h.k == 2147483647) break;                        // every nonzero is one of the K.npairs pairs
    if (K.npairs == kDictSlots) { fits = false; break; }
    K.off[K.npairs] = h.off; K.bits[K.npairs] = val_bits(h.val); hval[K.npairs] = h.val;
    K.npairs++;
  }
  if (fits && K.npairs > 0) {
    // sort by offset, then by value bits: a row's bits then come in ascending column order
    int ord[kDictSlots];
    for (int u = 0; u < K.npairs; u++) ord[u] = u;
    std::sort(ord, ord + K.npairs, [&](int a, int b) { return K.off[a] != K.off[b] ? K.off[a] < K.off[b] : K.bits[a] < K.bits[b]; });
    DictKeys S = K;
    for (int u = 0; u < K.npairs; u++) { S.off[u] = K.off[ord[u]]; S.bits[u] = K.bits[ord[u]]; D.off[u] = S.off[u]; D.val[u] = hval[ord[u]]; }
    KB_CUDA(cudaMalloc((void**)&D.mask, (size_t)A.n));
    dict_mask_kernel<T><<<g, 256, 0, c.stream>>>(A.n, A.rowptr, A.colind, A.val, S, D.mask);
    KB_CUDA(cudaGetLastError());
    c.sync();
    D.n = A.n;
    D.npairs = K.npairs;
  }
  cudaFree(dprobe);
}

// ---------------------------------------------------------------------------
// Staging plan: largest tile (nnz of kTileRows consecutive rows) and longest
// row decide whether the TMA ring fits, how deep it is, and the grid.
// ---------------------------------------------------------------------------
__global__ void plan_kernel(int n, int ncols, int ntiles, const int* __restrict__ rowptr,
                            int* out /* [0]=tile_cap [1]=max_row [2]=unsorted [3]=rowptr not monotone [4]=max col [5]=negative col */,
                            const int* __restrict__ colind, long long nnz) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int stride = gridDim.x * blockDim.x;
  int cap = 0, mr = 0, uns = 0, bad = 0, mc = -1, neg = 0;
  for (int i = t; i < n; i += stride) {
    const int kb = rowptr[i], ke = rowptr[i + 1];
    // validation (a malformed matrix must be an error, not an out-of-bounds read in the SpMV): row pointers
    // non-decreasing and inside [0, nnz] -- only then are the column indices of the row looked at
    if (kb > ke || kb < 0 || (long long)ke > nnz) { bad = 1; continue; }
    mr = max(mr, ke - kb);
    for (int k = kb; k < ke; k++) { const int cj = colind[k]; mc = max(mc, cj); neg |= cj < 0; }
    // halo columns (index >= ncols, row-partitioned operators) keep their global position in the row: skip them
    for (int k = kb + 1; k < ke; k++) uns |= (colind[k] <= colind[k - 1]) && colind[k] < ncols && colind[k - 1] < ncols;
  }
  if (bad) atomicExch(&out[3], 1);
  __syncthreads();
  for (int i = t; i < ntiles; i += stride) {
    const int r0 = i * kTileRows, r1 = min(r0 + kTileRows, n);
    cap = max(cap, rowptr[r1] - rowptr[r0]);
  }
  atomicMax(&out[0], cap);
  atomicMax(&out[1], mr);
  atomicMax(&out[4], mc);
  if (uns) atomicExch(&out[2], 1);
  if (neg) atomicExch(&out[5], 1);
}

template <class T> void csr_plan(Ctx& c, Csr<T>& A, CsrDict<T>* dict) {
  if (dict) csr_dict_free(*dict);
  A.ntiles = (A.n + kTileRows - 1) / kTileRows;
  int* dout = nullptr;
  KB_CUDA(cudaMalloc((void**)&dout, 6 * sizeof(int)));
  KB_CUDA(cudaMemsetAsync(dout, 0, 6 * sizeof(int), c.stream));
  int h[6] = {0, 0, 0, 0, -1, 0};
  int ends[2] = {0, (int)A.nnz};
  if (A.n > 0) {
    KB_CUDA(cudaMemcpyAsync(dout + 4, &h[4], sizeof(int), cudaMemcpyHostToDevice, c.stream));
    plan_kernel<<<sm_count() * 4, 256, 0, c.stream>>>(A.n, A.ncols, A.ntiles, A.rowptr, dout, A.colind, A.nnz);
    KB_CUDA(cudaGetLastError());
    KB_CUDA(cudaMemcpyAsync(&ends[0], A.rowptr, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
    KB_CUDA(cudaMemcpyAsync(&ends[1], A.rowptr + A.n, sizeof(int), cudaMemcpyDeviceToHost, c.stream));
  }
  KB_CUDA(cudaMemcpyAsync(h, dout, sizeof(h), cudaMemcpyDeviceToHost, c.stream));
  c.sync();
  cudaFree(dout);
  // the reference would throw a BoundsError on such input; here it must not reach the kernels
  if (ends[0] != 0 || (long long)ends[1] != A.nnz || h[3])
    throw std::runtime_error("CSR operator: row pointers must start at 0 (after rebasing), be non-decreasing and end at nnz");
  if (h[5]) throw std::runtime_error("CSR operator: negative column index (after rebasing)");
  A.max_col = h[4];
  if (h[2]) fprintf(stderr, "[krylov_b200] warning: CSR column indices are not strictly ascending within rows; "
                            "results remain correct but are no longer bit-comparable to SparseArrays' order\n");
  A.tile_cap = h[0];
  A.max_row = h[1];
  // Ring sizing: prefer 2 CTAs/SM (<= 110 KB each) with up to 4 stages; fall
  // back to 1 CTA/SM (<= 220 KB) with >= 2 stages; otherwise no TMA staging.
  TileLayout<T> L{A.tile_cap};
  const size_t two_cta = 110 * 1024, one_cta = 220 * 1024;
  A.tma_ok = false;
  int per_sm = 2;
  // tuning overrides (profiles/sweep_k1.py): KB200_STAGES, KB200_CTAS_PER_SM.  A forced ring gets the per-CTA ceiling
  // of the default rule for the same CTAs per SM (and never more than the 220 KB every staged launcher opts in to);
  // one that does not fit falls through to the default choice.
  const char* es = getenv("KB200_STAGES");
  const char* ec = getenv("KB200_CTAS_PER_SM");
  if (es && ec) {
    const int s = atoi(es), cps = atoi(ec);
    if (s >= 1 && s <= 8 && cps >= 1 && cps <= 8) {
      const size_t per_cta = cps == 1 ? one_cta : cps == 2 ? two_cta : 226 * 1024 / cps;
      if (L.total_bytes(s) <= per_cta) { A.tma_ok = true; A.stages = s; per_sm = cps; }
    }
  }
  // default: 3 CTAs/SM x 2 stages when it fits (profiles/sweep_k1.py sweeps the alternatives): the gather latency
  // wants 27 warps/SM, and a shallower ring leaves more of the SM's 228 KB to L1 for the gathered vectors.
  if (!A.tma_ok && L.total_bytes(2) * 3 <= 226 * 1024) { A.tma_ok = true; A.stages = 2; per_sm = 3; }
  for (int s = 4; s >= 2 && !A.tma_ok; s--)
    if (L.total_bytes(s) <= two_cta) { A.tma_ok = true; A.stages = s; per_sm = 2; }
  for (int s = 4; s >= 2 && !A.tma_ok; s--)
    if (L.total_bytes(s) <= one_cta) { A.tma_ok = true; A.stages = s; per_sm = 1; }
  if (A.tma_ok) {
    A.smem_bytes = L.total_bytes(A.stages);
    int g = sm_count() * per_sm;
    A.grid = g < A.ntiles ? g : (A.ntiles > 0 ? A.ntiles : 1);
    A.ctas_per_sm = per_sm;
  } else {
    A.stages = 0; A.smem_bytes = 0; A.grid = 0;
  }
  // Constant-coefficient encoding: square operators whose rows ascend strictly and that have no halo columns.
  // KB200_CSR_DICT=0 keeps the CSR path alone (A/B measurements, tests); read at every plan.
  const char* ed = getenv("KB200_CSR_DICT");
  if (dict && !(ed && atoi(ed) == 0) && A.n > 0 && A.ncols == A.n && A.max_col < A.n && !h[2]) csr_dict_build<T>(c, A, *dict);
}

// ---------------------------------------------------------------------------
// Kernels
// ---------------------------------------------------------------------------
// Row-per-thread LDG kernel: always valid (any row length), used when the
// staging plan does not fit and as an independent check of the staged kernel.
template <class T, bool DOT, class G>
__global__ void __launch_bounds__(kBlock) spmv_rows_kernel(Csr<T> A, G xg, T* __restrict__ y, T* part,
                                                           unsigned* ticket, T* out) {
  __shared__ T sm[32];
  T dacc = T(0);
  const int stride = gridDim.x * blockDim.x;
  for (int row = blockIdx.x * blockDim.x + threadIdx.x; row < A.n; row += stride) {
    const int kb = A.rowptr[row], ke = A.rowptr[row + 1];
    T acc = T(0);
    for (int k = kb; k < ke; k++) acc = add_rn(acc, mul_rn(A.val[k], xg(A.colind[k])));
    y[row] = acc;
    if (DOT) dacc += __ldg(&xg.x[row]) * acc;
  }
  if (DOT) {
    T mine[1] = {block_sum(dacc, sm)}, tot[1];
    if (grid_sum_last<T, 1>(mine, part, ticket, sm, tot) && threadIdx.x == 0) out[0] = tot[0];
  }
}

template <class T, bool DOT, class G>
__global__ void __launch_bounds__(kTileThreads, 3) spmv_tma_kernel(Csr<T> A, G xg, T* __restrict__ y, T* part,
                                                                unsigned* ticket, T* out) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ T sm[32];
  T dacc = T(0);
  spmv_tiles_run<T>(
      A, smem, xg, [&](int row) { return DOT ? __ldg(&xg.x[row]) : T(0); },
      [&](int row, T acc, T xr) {
        y[row] = acc;
        if (DOT) dacc += xr * acc;
      });
  if (DOT) {
    T mine[1] = {block_sum(dacc, sm)}, tot[1];
    if (grid_sum_last<T, 1>(mine, part, ticket, sm, tot) && threadIdx.x == 0) out[0] = tot[0];
  }
}

template <class T, bool DOT, class G>
static void spmv_launch_g(Ctx& c, const Csr<T>& A, G xg, T* y, int slot, int variant) {
  T* out = reinterpret_cast<T*>(reinterpret_cast<double*>(c.dscal) + slot);
  const bool staged = variant == 2 || (variant == 0 && A.tma_ok);
  if (staged) {
    if (!A.tma_ok) throw std::runtime_error("TMA-staged SpMV requested but the tile plan does not fit shared memory");
    ensure_dyn_smem((const void*)spmv_tma_kernel<T, DOT, G>, 220 * 1024);
    int occ = 0;   // persistent grid = what is really co-resident (never more than one wave)
    KB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, spmv_tma_kernel<T, DOT, G>, kTileThreads, A.smem_bytes));
    if (occ < 1) throw std::runtime_error("spmv_tma_kernel does not fit on an SM with the planned shared-memory ring");
    const int grid = std::min(std::min(occ, A.ctas_per_sm) * sm_count(), std::max(1, A.ntiles));
    spmv_tma_kernel<T, DOT, G><<<grid, kTileThreads, A.smem_bytes, c.stream>>>(A, xg, y, (T*)c.partials, c.tickets + 1, out);
  } else {
    const int grid = stream_grid(A.n, 1, 8);
    spmv_rows_kernel<T, DOT, G><<<grid, kBlock, 0, c.stream>>>(A, xg, y, (T*)c.partials, c.tickets + 1, out);
  }
  KB_CUDA(cudaGetLastError());
  c.launches++;
}

template <class T, bool DOT>
static void spmv_launch(Ctx& c, const Csr<T>& A, const T* x, T* y, int slot, int variant) {
  if (A.n <= 0) return;
  if (c.dex) spmv_launch_g<T, DOT, XGather<T>>(c, A, xgather_of<T>(c, x), y, slot, variant);   // row-partitioned: [local | halo]
  else spmv_launch_g<T, DOT, XPlain<T>>(c, A, XPlain<T>{x}, y, slot, variant);
}

template <class T> void k_spmv(Ctx& c, const Csr<T>& A, const T* x, T* y, int variant) { spmv_launch<T, false>(c, A, x, y, 1, variant); }

// y = A x through the encoded rows, one row per thread (the row arithmetic of cg_persist_dict on its own)
template <class T>
__global__ void __launch_bounds__(kBlock) spmv_dict_kernel(CsrDict<T> D, const T* __restrict__ x, T* __restrict__ y) {
  const int stride = gridDim.x * blockDim.x;
  for (int row = blockIdx.x * blockDim.x + threadIdx.x; row < D.n; row += stride)
    y[row] = dict_row_sum<T>(D, row, __ldg(&D.mask[row]), XPlain<T>{x}, [](T v) { return v; });
}

template <class T> void k_spmv_dict(Ctx& c, const CsrDict<T>& D, const T* x, T* y) {
  if (D.npairs <= 0 || !D.mask) throw std::runtime_error("the operator carries no constant-coefficient encoding");
  spmv_dict_kernel<T><<<stream_grid(D.n, 1, 8), kBlock, 0, c.stream>>>(D, x, y);
  KB_CUDA(cudaGetLastError());
  c.launches++;
}

// ---------------------------------------------------------------------------
// General x-halo exchange of row-partitioned operators (dist.cuh: DistExchange)
// ---------------------------------------------------------------------------
template <class T> struct ExchangeDst { T* p[kMaxRanks]; };

template <class T>
__global__ void __launch_bounds__(kBlock) halo_exchange_kernel(const T* __restrict__ x, int nsend, const int* __restrict__ row,
                                                               const int* __restrict__ peer, const int* __restrict__ slot,
                                                               ExchangeDst<T> dst, unsigned* ticket, DistComm* dc) {
  __shared__ bool is_last;
  const int stride = gridDim.x * blockDim.x;
  bool sent = false;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < nsend; e += stride) {
    dst.p[peer[e]][slot[e]] = x[row[e]];
    sent = true;
  }
  if (sent) __threadfence_system();        // my stores are visible to the peers before the barrier below
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned t = atomicAdd(ticket, 1u);
    is_last = (t == gridDim.x - 1);
    if (is_last) *ticket = 0u;
  }
  __syncthreads();
  // the last CTA of this rank enters the cross-GPU barrier: when it returns, every rank has finished pushing
  if (is_last && threadIdx.x == 0) dist_allreduce_sum(dc, 0.0);
}

template <class T> void k_halo_exchange(Ctx& c, const T* x) {
  if (!c.dex) return;
  DistExchange& d = *c.dex;
  ExchangeDst<T> dst;
  const size_t par = (size_t)(d.count & 1);
  for (int k = 0; k < kMaxRanks; k++)
    dst.p[k] = d.xhalo_peer[k] ? reinterpret_cast<T*>(d.xhalo_peer[k]) + par * (size_t)d.nhalo_peer[k] : nullptr;
  const int grid = d.nsend > 0 ? std::min(sm_count(), (d.nsend + kBlock - 1) / kBlock) : 1;
  halo_exchange_kernel<T><<<grid, kBlock, 0, c.stream>>>(x, d.nsend, d.send_row, d.send_peer, d.send_slot, dst, c.tickets + 6, c.dcomm);
  KB_CUDA(cudaGetLastError());
  c.launches++;
  d.count++;
}

// ---------------------------------------------------------------------------
// Operator application (A, M, N as the solvers see them)
// ---------------------------------------------------------------------------
template <class T> void op_apply(Ctx& c, const LinOp<T>& op, const T* x, T* y, bool ldiv) {
  switch (op.kind) {
    case LinOp<T>::CSR:
      k_halo_exchange<T>(c, x);            // row-partitioned operators only; no-op on a single GPU
      k_spmv<T>(c, *op.csr, x, y, 0);
      break;
    case LinOp<T>::DIAG: k_diagmul<T>(c, op.n, y, op.diag, x, ldiv); break;
    case LinOp<T>::BDIAG: k_blockdiag_mul<T>(c, op.n, op.bs, ldiv ? op.blocks_inv : op.blocks, x, y); break;
    case LinOp<T>::DEV_CB:
      c.sync();                       // the callback may use its own stream
      op.fn(x, y, op.userdata);
      KB_CUDA(cudaDeviceSynchronize());
      break;
    case LinOp<T>::HOST_CB:
      // reference: ccall(op.fptr, ..., x, y, userdata) on host pointers
      // (interfaces/src/c_operator.jl:35-42); here x/y live in HBM, so stage.
      KB_CUDA(cudaMemcpyAsync(op.hx, x, sizeof(T) * (size_t)(op.nin ? op.nin : op.n), cudaMemcpyDeviceToHost, c.stream));
      c.sync();
      op.fn(op.hx, op.hy, op.userdata);
      KB_CUDA(cudaMemcpyAsync(y, op.hy, sizeof(T) * (size_t)op.n, cudaMemcpyHostToDevice, c.stream));
      break;
    case LinOp<T>::NONE: k_copy<T>(c, op.n, y, x); break;
  }
}

#define INST(T)                                                                                                  \
  template void csr_upload<T>(Ctx&, Csr<T>&, int, long long, const void*, const void*, const T*, int, int, bool, int, \
                              CsrDict<T>*);                                                                      \
  template void csr_free<T>(Csr<T>&);                                                                            \
  template void csr_dict_free<T>(CsrDict<T>&);                                                                   \
  template void csr_plan<T>(Ctx&, Csr<T>&, CsrDict<T>*);                                                         \
  template void k_spmv<T>(Ctx&, const Csr<T>&, const T*, T*, int);                                               \
  template void k_spmv_dict<T>(Ctx&, const CsrDict<T>&, const T*, T*);                                           \
  template void k_halo_exchange<T>(Ctx&, const T*);                                                              \
  template void op_apply<T>(Ctx&, const LinOp<T>&, const T*, T*, bool);
INST(double)
INST(float)
#undef INST

}  // namespace kb
