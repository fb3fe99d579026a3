// tests/hostsim_amg/hostsim_amg.cpp -- TEST INFRASTRUCTURE ONLY (never linked into libb200krylov.so).
//
// The smoothed-aggregation setup of csrc/amg_core.h (the code the library runs on the host) and its serial V-cycle, on the
// CPU.  hostsim.cpp is compiled in unchanged (its CSR view and export conventions); only the AMG exports are added.
// A hierarchy is an opaque handle: hostsim_amg_setup builds it from an fp64 CSR (ascending columns), the accessors copy
// a level out, hostsim_amg_vcycle applies one V-cycle in Float64 (is_f64 = 1) or Float32 (0).
// Setup statuses: 0 ok; 1 zero or missing diagonal entry; 2 singular coarsest level; 3 coarsest level too large
// (level and row in bad[0], bad[1]).
#include "../hostsim/hostsim.cpp"
#include "../../iterativesolvers.jl_b200/csrc/amg_core.h"

namespace {
struct HostAmg {
  b200::AmgOptions opts;
  std::vector<b200::AmgLevel> levels;
};
}  // namespace

EXPORT int hostsim_amg_setup(const hostsim_csr *A, double theta, int max_levels, int max_coarse, int presweeps,
                             int postsweeps, int64_t *bad, void **out) {
  b200::AmgCsr h;
  h.m = A->m;
  h.n = A->n;
  const int64_t nnz = A->rowptr[A->m];
  h.rowptr.assign(A->rowptr, A->rowptr + A->m + 1);
  h.colind.assign(A->colind, A->colind + nnz);
  h.vals.assign((const double *)A->vals, (const double *)A->vals + nnz);
  HostAmg *H = new HostAmg();
  H->opts = b200::AmgOptions{theta, max_levels, max_coarse, presweeps, postsweeps};
  b200::AmgTimes tm;
  const b200::AmgStatus st = b200::amg_setup(std::move(h), H->opts, &H->levels, &tm, [] { return 0.0; });
  *out = nullptr;
  if (st.code != b200::AMG_OK) {
    bad[0] = st.level;
    bad[1] = st.row;
    delete H;
    return st.code;
  }
  *out = H;
  return 0;
}

EXPORT int hostsim_amg_levels(const void *h) { return (int)((const HostAmg *)h)->levels.size(); }

// sizes[0..3] = rows of A_l, nonzeros of A_l, columns of P_l (0 on the coarsest level), nonzeros of P_l
EXPORT void hostsim_amg_level_sizes(const void *h, int l, int64_t *sizes) {
  const b200::AmgLevel &L = ((const HostAmg *)h)->levels[(size_t)l];
  sizes[0] = L.A.m;
  sizes[1] = L.A.nnz();
  sizes[2] = L.P.n * (L.P.m > 0);
  sizes[3] = L.P.m > 0 ? L.P.nnz() : 0;
}

static void copy_csr(const b200::AmgCsr &M, int64_t *rowptr, int32_t *colind, double *vals) {
  if (rowptr) memcpy(rowptr, M.rowptr.data(), sizeof(int64_t) * M.rowptr.size());
  if (colind) memcpy(colind, M.colind.data(), sizeof(int32_t) * M.colind.size());
  if (vals) memcpy(vals, M.vals.data(), sizeof(double) * M.vals.size());
}

// level l: A_l, P_l (not on the coarsest level), aggregates and smoother weights (not on the coarsest level), and the
// coarse inverse (coarsest level only, row-major); any pointer may be NULL
EXPORT void hostsim_amg_level_get(const void *h, int l, int64_t *a_rowptr, int32_t *a_colind, double *a_vals,
                                  int64_t *p_rowptr, int32_t *p_colind, double *p_vals, int32_t *agg, double *w,
                                  double *inv) {
  const b200::AmgLevel &L = ((const HostAmg *)h)->levels[(size_t)l];
  copy_csr(L.A, a_rowptr, a_colind, a_vals);
  if (L.P.m > 0) copy_csr(L.P, p_rowptr, p_colind, p_vals);
  if (agg && !L.agg.empty()) memcpy(agg, L.agg.data(), sizeof(int32_t) * L.agg.size());
  if (w && !L.w.empty()) memcpy(w, L.w.data(), sizeof(double) * L.w.size());
  if (inv && !L.inv.empty()) memcpy(inv, L.inv.data(), sizeof(double) * L.inv.size());
}

// x = one V-cycle applied to b (x must not alias b)
EXPORT void hostsim_amg_vcycle(const void *h, int is_f64, const void *b, void *x) {
  const HostAmg *H = (const HostAmg *)h;
  if (is_f64) b200::amg_vcycle_serial<double>(H->levels, H->opts, 0, (const double *)b, (double *)x);
  else b200::amg_vcycle_serial<float>(H->levels, H->opts, 0, (const float *)b, (float *)x);
}

EXPORT void hostsim_amg_free(void *h) { delete (HostAmg *)h; }
