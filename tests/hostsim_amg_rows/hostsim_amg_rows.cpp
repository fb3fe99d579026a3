// tests/hostsim_amg_rows/hostsim_amg_rows.cpp -- TEST INFRASTRUCTURE ONLY (never linked into libb200krylov.so).
//
// The row functions of the device AMG setup (csrc/amg_setup_core.h) run serially on the CPU, each next to amg_core.h's
// serial setup for comparison: hostsim_amg_aggregate_rows assembles the aggregates from the pass-1 decision rule as
// amg_setup.cu does, hostsim_amg_spgemm_rows forms C = A B row by row.  tests/hostsim_amg/hostsim_amg.cpp is compiled in
// unchanged (its CSR view, export conventions and copy_csr); only these exports are added.
#include "../hostsim_amg/hostsim_amg.cpp"
#include "../../iterativesolvers.jl_b200/csrc/amg_setup_core.h"

namespace {
b200::AmgCsr to_amg(const hostsim_csr *A) {
  b200::AmgCsr h;
  h.m = A->m;
  h.n = A->n;
  const int64_t nnz = A->rowptr[A->m];
  h.rowptr.assign(A->rowptr, A->rowptr + A->m + 1);
  h.colind.assign(A->colind, A->colind + nnz);
  h.vals.assign((const double *)A->vals, (const double *)A->vals + nnz);
  return h;
}
struct Rows32 {   // an AmgCsr as the int32-offset view of the row functions
  std::vector<int> rp;
  b200::AmgRows r;
  explicit Rows32(const b200::AmgCsr &M) : rp(M.rowptr.begin(), M.rowptr.end()) {
    r = b200::AmgRows{rp.data(), M.colind.data(), M.vals.empty() ? nullptr : M.vals.data()};
  }
};
}  // namespace

// The aggregates of A's strength pattern (theta) twice: agg_ref by amg_aggregate, agg by the device's steps (pass 1 as
// the rounds of amg_pass1_decide, ids by a scan over the roots, pass 2 per row from the pass-1 result, pass 3 serially).
// Returns amg_aggregate's count; *naggs = the other; *rounds = pass 1's rounds; *pass3 = rows pass 3 started or joined.
EXPORT int hostsim_amg_aggregate_rows(const hostsim_csr *A, double theta, int32_t *agg_ref, int32_t *agg, int *naggs,
                                      int *rounds, int *pass3) {
  const b200::AmgCsr h = to_amg(A);
  std::vector<double> d;
  b200::amg_diagonal(h, &d);
  b200::AmgCsr S = b200::amg_strength(h, d, theta);
  S.vals.assign(S.colind.size(), 0.0);   // amg_transpose moves values too
  const b200::AmgCsr St = b200::amg_transpose(S);
  std::vector<int> ref;
  const int nref = b200::amg_aggregate(S, &ref);
  memcpy(agg_ref, ref.data(), sizeof(int) * ref.size());
  const Rows32 s(S), t(St);
  const int n = (int)S.m, kFree = -2;
  std::vector<int> state, x1((size_t)n, kFree), x((size_t)n);
  *rounds = b200::amg_pass1_rounds(s.r, t.r, n, &state);
  int next = 0;
  for (int i = 0; i < n; ++i)   // the scan over the root flags gives ids in row order
    if (state[(size_t)i] == b200::AMG_ROOT) {
      x1[(size_t)i] = next;
      for (int p = s.rp[(size_t)i]; p < s.rp[(size_t)i + 1]; ++p) x1[(size_t)S.colind[(size_t)p]] = next;
      ++next;
    }
  for (int i = 0; i < n; ++i)
    if (x1[(size_t)i] == kFree && s.rp[(size_t)i] == s.rp[(size_t)i + 1]) x1[(size_t)i] = -1;
  for (int i = 0; i < n; ++i) {
    int a = x1[(size_t)i];
    if (a == kFree)
      for (int p = s.rp[(size_t)i]; p < s.rp[(size_t)i + 1]; ++p)
        if (x1[(size_t)S.colind[(size_t)p]] >= 0) {
          a = x1[(size_t)S.colind[(size_t)p]];
          break;
        }
    x[(size_t)i] = a;
  }
  *pass3 = 0;
  for (int i = 0; i < n; ++i) {
    if (x[(size_t)i] != kFree) continue;
    x[(size_t)i] = next;
    ++*pass3;
    for (int p = s.rp[(size_t)i]; p < s.rp[(size_t)i + 1]; ++p)
      if (x[(size_t)S.colind[(size_t)p]] == kFree) {
        x[(size_t)S.colind[(size_t)p]] = next;
        ++*pass3;
      }
    ++next;
  }
  memcpy(agg, x.data(), sizeof(int) * x.size());
  *naggs = next;
  return nref;
}

// C = A B row by row through amg_spgemm_row_serial (table of `cap` slots) into (rowptr, colind, vals), and by
// amg_spgemm into the *_ref arrays (capacity: the caller's bound on nnz(C)).  Returns nnz(C) by amg_spgemm, -1 when a row
// overflowed the table, -2 when the two patterns differ in size.
EXPORT int64_t hostsim_amg_spgemm_rows(const hostsim_csr *A, const hostsim_csr *B, int cap, int64_t *rowptr,
                                       int32_t *colind, double *vals, int64_t *rowptr_ref, int32_t *colind_ref,
                                       double *vals_ref) {
  const b200::AmgCsr a = to_amg(A), b = to_amg(B);
  const Rows32 ra(a), rb(b);
  std::vector<int> ci;
  std::vector<double> v;
  rowptr[0] = 0;
  for (int64_t i = 0; i < a.m; ++i) {
    const int u = b200::amg_spgemm_row_serial(ra.r, rb.r, i, cap, &ci, &v);
    if (u < 0) return -1;
    memcpy(colind + rowptr[i], ci.data(), sizeof(int) * (size_t)u);
    memcpy(vals + rowptr[i], v.data(), sizeof(double) * (size_t)u);
    rowptr[i + 1] = rowptr[i] + u;
  }
  const b200::AmgCsr C = b200::amg_spgemm(a, b);
  if (C.nnz() != rowptr[a.m]) return -2;
  copy_csr(C, rowptr_ref, colind_ref, vals_ref);
  return C.nnz();
}
