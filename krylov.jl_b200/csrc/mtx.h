// mtx.h -- host-side CSR container, Matrix Market reader and transposition (mtx.cu).
#pragma once
#include <vector>

#include "kb_internal.h"

namespace kb {

struct HostCsr {
  int n = 0;
  int ncols = 0;                   // columns (= n for square matrices)
  std::vector<long long> rowptr;   // n + 1, 0-based (64-bit: csr_upload narrows with a range check)
  std::vector<long long> colind;   // stored wide for the same upload path
  std::vector<double> val;
};

void coo_to_csr(int n, const std::vector<int>& I, const std::vector<int>& J, const std::vector<double>& V, HostCsr& out);
void read_matrix_market(const char* path, HostCsr& out);
void transpose_csr(const HostCsr& A, HostCsr& out);   // m x n -> n x m
template <class T> void csr_from_host(Ctx& c, Csr<T>& dst, const HostCsr& h);
template <class T> void csr_to_host(Ctx& c, const Csr<T>& A, HostCsr& h);

}  // namespace kb
