// tests/hostsim_ilu/hostsim_ilu.cpp -- TEST INFRASTRUCTURE ONLY (never linked into libb200krylov.so).
//
// The ILU(0) preconditioner of csrc/ilu_core.h on the CPU: the same row functions the GPU kernels run (factor row,
// forward row, backward row) driven serially over the same chunk schedules, with a `wait` that accepts only rows of
// EARLIER chunks -- so every run also checks that the schedule orders each row after its dependencies.  hostsim.cpp is
// compiled in unchanged (its CSR view and export conventions); only the ILU exports are added.  is_f64 = 1: Float64,
// 0: Float32.  Statuses: 0 ok; 1 = a dependency was not in an earlier chunk (*bad = the row); 2 = zero pivot (*bad = the
// smallest such row); 3 = missing or zero diagonal entry of A (*bad = the row).
#include "../hostsim/hostsim.cpp"
#include "../../iterativesolvers.jl_b200/csrc/ilu_core.h"

namespace {

template <typename T>
int ilu_factor_impl(const hostsim_csr *A, T *f, int64_t *bad, int *levels_f, int *levels_b) {
  std::vector<int> dpos;
  b200::IluSchedule fw, bw;
  const int64_t sing = b200::ilu_analyse<T, int64_t>(A->m, A->rowptr, A->colind, (const T *)A->vals, &dpos, &fw, &bw);
  if (sing) {
    *bad = sing - 1;
    return 3;
  }
  *levels_f = fw.levels;
  *levels_b = bw.levels;
  memcpy(f, A->vals, sizeof(T) * (size_t)A->rowptr[A->m]);
  const b200::IluView<T, int64_t> v{A->rowptr, A->colind, dpos.data(), f};
  return b200::ilu_run_serial(fw, A->m, [&](int64_t i, auto &wait) { return b200::ilu_factor_row(v, i, wait); }, bad);
}

template <typename T>
int ilu_ldiv_impl(const hostsim_csr *A, const T *f, const T *x, T *y, int64_t *bad) {
  std::vector<int> dpos;
  b200::IluSchedule fw, bw;
  const int64_t sing = b200::ilu_analyse<T, int64_t>(A->m, A->rowptr, A->colind, (const T *)A->vals, &dpos, &fw, &bw);
  if (sing) {
    *bad = sing - 1;
    return 3;
  }
  const b200::IluView<T, int64_t> v{A->rowptr, A->colind, dpos.data(), (T *)f};
  int st = b200::ilu_run_serial(fw, A->m, [&](int64_t i, auto &wait) { return b200::ilu_forward_row(v, i, x, y, wait); },
                                bad);
  if (st) return st;
  return b200::ilu_run_serial(bw, A->m, [&](int64_t i, auto &wait) { return b200::ilu_backward_row(v, i, y, y, wait); },
                              bad);
}

}  // namespace

// the ILU(0) factor of A (values in A's CSR order) into f
EXPORT int hostsim_ilu0_factor(int is_f64, const hostsim_csr *A, void *f, int64_t *bad, int *levels_f, int *levels_b) {
  return is_f64 ? ilu_factor_impl<double>(A, (double *)f, bad, levels_f, levels_b)
                : ilu_factor_impl<float>(A, (float *)f, bad, levels_f, levels_b);
}

// y = U \ (L \ x) with the factor values f (A's pattern); x may be y
EXPORT int hostsim_ilu0_ldiv(int is_f64, const hostsim_csr *A, const void *f, const void *x, void *y, int64_t *bad) {
  return is_f64 ? ilu_ldiv_impl<double>(A, (const double *)f, (const double *)x, (double *)y, bad)
                : ilu_ldiv_impl<float>(A, (const float *)f, (const float *)x, (float *)y, bad);
}

// the chunk schedule of the forward (backward = 0) or backward (1) sweep: rows (n) and cptr (chunks + 1, at most n + 1);
// returns the number of chunks, or -1 for a missing or zero diagonal entry
EXPORT int64_t hostsim_ilu0_chunks(const hostsim_csr *A, int backward, int32_t *rows, int32_t *cptr) {
  std::vector<int> dpos;
  b200::IluSchedule fw, bw;
  if (b200::ilu_analyse<double, int64_t>(A->m, A->rowptr, A->colind, (const double *)A->vals, &dpos, &fw, &bw)) return -1;
  const b200::IluSchedule &s = backward ? bw : fw;
  memcpy(rows, s.rows.data(), sizeof(int) * s.rows.size());
  memcpy(cptr, s.cptr.data(), sizeof(int) * s.cptr.size());
  return s.chunks();
}
