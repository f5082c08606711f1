// mtx.cu -- the data formats either side of the path (SURVEY.md section 8f-4): Matrix Market ingestion (the
// reference's benchmarks read SuiteSparse .mtx files through MatrixMarket.jl, benchmark/benchmarks.jl:23-33,
// benchmark/gpu.jl:26-35) and the transposed operator A^T (= A^H for the real types of this path,
// docs/src/matrix_free.md:36-44).  Host-side conversions; the result is an ordinary CSR operator in HBM.
#include <algorithm>
#include <cctype>
#include <cstdio>
#include <cstring>
#include <numeric>
#include <string>
#include <vector>

#include "mtx.h"

namespace kb {

namespace {
std::string lower(std::string s) {
  for (char& ch : s) ch = (char)std::tolower((unsigned char)ch);
  return s;
}
}  // namespace

// Triplets (0-based) -> CSR with ascending columns and duplicates summed (what SparseArrays.sparse(I, J, V) does).
void coo_to_csr(int n, const std::vector<int>& I, const std::vector<int>& J, const std::vector<double>& V, HostCsr& out) {
  const size_t nz = I.size();
  std::vector<long long> cnt((size_t)n + 1, 0);
  for (size_t k = 0; k < nz; k++) cnt[(size_t)I[k] + 1]++;
  for (int i = 0; i < n; i++) cnt[(size_t)i + 1] += cnt[i];
  std::vector<int> cj(nz);
  std::vector<double> cv(nz);
  {
    std::vector<long long> pos(cnt.begin(), cnt.end() - 1);
    for (size_t k = 0; k < nz; k++) { const long long q = pos[I[k]]++; cj[q] = J[k]; cv[q] = V[k]; }
  }
  out.n = n; out.ncols = n;
  out.rowptr.assign((size_t)n + 1, 0);
  out.colind.clear(); out.val.clear();
  out.colind.reserve(nz); out.val.reserve(nz);
  std::vector<int> perm;
  for (int i = 0; i < n; i++) {
    const long long b = cnt[i], e = cnt[(size_t)i + 1];
    perm.resize((size_t)(e - b));
    std::iota(perm.begin(), perm.end(), 0);
    std::stable_sort(perm.begin(), perm.end(), [&](int a, int c) { return cj[b + a] < cj[b + c]; });   // stable: duplicates keep file order
    for (size_t t = 0; t < perm.size(); t++) {
      const int col = cj[b + perm[t]];
      const double v = cv[b + perm[t]];
      if (!out.colind.empty() && (long long)out.colind.size() > out.rowptr[i] && out.colind.back() == col) out.val.back() += v;
      else { out.colind.push_back(col); out.val.push_back(v); }
    }
    out.rowptr[(size_t)i + 1] = (long long)out.colind.size();
  }
}

// Matrix Market exchange format, `matrix coordinate {real|integer|pattern} {general|symmetric|skew-symmetric}`.
void read_matrix_market(const char* path, HostCsr& out) {
  FILE* f = fopen(path, "r");
  if (!f) throw std::runtime_error(std::string("cannot open ") + path);
  struct Closer { FILE* f; ~Closer() { fclose(f); } } closer{f};
  std::vector<char> line(1 << 16);
  if (!fgets(line.data(), (int)line.size(), f)) throw std::runtime_error("empty Matrix Market file");
  char banner[64], object[64], format[64], field[64], symmetry[64];
  if (sscanf(line.data(), "%63s %63s %63s %63s %63s", banner, object, format, field, symmetry) != 5 || lower(banner) != "%%matrixmarket")
    throw std::runtime_error("not a Matrix Market file (missing %%MatrixMarket banner)");
  const std::string obj = lower(object), fmt = lower(format), fld = lower(field), sym = lower(symmetry);
  if (obj != "matrix" || fmt != "coordinate") throw std::runtime_error("only `matrix coordinate` files are supported");
  if (fld != "real" && fld != "integer" && fld != "pattern") throw std::runtime_error("field `" + fld + "` is outside the real path");
  if (sym != "general" && sym != "symmetric" && sym != "skew-symmetric") throw std::runtime_error("symmetry `" + sym + "` is not supported");
  long long M = 0, N = 0, L = 0;
  for (;;) {
    if (!fgets(line.data(), (int)line.size(), f)) throw std::runtime_error("missing size line");
    const char* s = line.data();
    while (*s == ' ' || *s == '\t') s++;
    if (*s == '%' || *s == '\n' || *s == '\r' || *s == 0) continue;
    if (sscanf(s, "%lld %lld %lld", &M, &N, &L) != 3) throw std::runtime_error("bad size line");
    break;
  }
  if (M != N) throw std::runtime_error("System must be square");
  if (M > 2147483647LL - 1024) throw std::runtime_error("dimension exceeds the int32 index range");
  std::vector<int> I, J;
  std::vector<double> V;
  const bool mirror = sym != "general";
  I.reserve((size_t)(mirror ? 2 * L : L)); J.reserve(I.capacity()); V.reserve(I.capacity());
  for (long long k = 0; k < L; k++) {
    long long i, j;
    double v = 1.0;
    int got;
    if (fld == "pattern") got = fscanf(f, "%lld %lld", &i, &j) == 2 ? 3 : 0;
    else got = fscanf(f, "%lld %lld %lf", &i, &j, &v);
    if (got != 3) throw std::runtime_error("truncated entry list");
    if (i < 1 || i > M || j < 1 || j > N) throw std::runtime_error("entry index out of range");
    I.push_back((int)(i - 1)); J.push_back((int)(j - 1)); V.push_back(v);
    if (mirror && i != j) { I.push_back((int)(j - 1)); J.push_back((int)(i - 1)); V.push_back(sym == "skew-symmetric" ? -v : v); }
  }
  coo_to_csr((int)M, I, J, V, out);
}

// out = A^T, m x n -> n x m.  Rows of A are scattered in ascending order, so every row of A^T lists its columns (the
// rows of A) in ascending order and A^T u sums in ascending row order of A, as a sequential A' * u does.
void transpose_csr(const HostCsr& A, HostCsr& out) {
  const int m = A.n, n = A.ncols;
  const size_t nz = A.colind.size();
  for (size_t k = 0; k < nz; k++)
    if (A.colind[k] < 0 || A.colind[k] >= n) throw std::runtime_error("transpose: column index outside the operator's columns");
  out.n = n; out.ncols = m;
  out.rowptr.assign((size_t)n + 1, 0);
  for (size_t k = 0; k < nz; k++) out.rowptr[(size_t)A.colind[k] + 1]++;
  for (int i = 0; i < n; i++) out.rowptr[(size_t)i + 1] += out.rowptr[i];
  out.colind.resize(nz); out.val.resize(nz);
  std::vector<long long> pos(out.rowptr.begin(), out.rowptr.end() - 1);
  for (int i = 0; i < m; i++)
    for (long long k = A.rowptr[i]; k < A.rowptr[(size_t)i + 1]; k++) {
      const long long q = pos[A.colind[k]]++;
      out.colind[q] = i; out.val[q] = A.val[k];
    }
}

template <class T> void csr_from_host(Ctx& c, Csr<T>& dst, const HostCsr& h) {
  std::vector<T> v(h.val.begin(), h.val.end());
  csr_upload<T>(c, dst, h.n, (long long)h.colind.size(), h.rowptr.data(), h.colind.data(), v.data(), 0, 8, false, h.ncols);
}

template <class T> void csr_to_host(Ctx& c, const Csr<T>& A, HostCsr& h) {
  h.n = A.n; h.ncols = A.ncols;
  std::vector<int> rp((size_t)A.n + 1), ci((size_t)A.nnz);
  std::vector<T> v((size_t)A.nnz);
  KB_CUDA(cudaMemcpyAsync(rp.data(), A.rowptr, sizeof(int) * rp.size(), cudaMemcpyDeviceToHost, c.stream));
  if (A.nnz) {
    KB_CUDA(cudaMemcpyAsync(ci.data(), A.colind, sizeof(int) * ci.size(), cudaMemcpyDeviceToHost, c.stream));
    KB_CUDA(cudaMemcpyAsync(v.data(), A.val, sizeof(T) * v.size(), cudaMemcpyDeviceToHost, c.stream));
  }
  c.sync();
  h.rowptr.assign(rp.begin(), rp.end());
  h.colind.assign(ci.begin(), ci.end());
  h.val.assign(v.begin(), v.end());
}

template void csr_from_host<double>(Ctx&, Csr<double>&, const HostCsr&);
template void csr_from_host<float>(Ctx&, Csr<float>&, const HostCsr&);
template void csr_to_host<double>(Ctx&, const Csr<double>&, HostCsr&);
template void csr_to_host<float>(Ctx&, const Csr<float>&, HostCsr&);

}  // namespace kb
