// tests/hostsim_complex/hostsim_complex.cpp -- TEST INFRASTRUCTURE ONLY (never linked into libb200krylov.so).
//
// The complex instantiations (ComplexF64 / ComplexF32) of the cg! and gmres! fused-pass engines (csrc/cg_core.h,
// csrc/gmres_core.h) on the serial CPU backend of tests/hostsim.  The backend is not restated: hostsim.cpp is compiled
// into this library as it stands, so the complex runs go through the very pass loop (row order, split finish, poisoned
// scratch) that the real runs of tests/hostsim use; only the operator application is the complex product.  Vectors and
// matrix values are interleaved (re, im); is_f64 = 1 selects ComplexF64, 0 ComplexF32.
#include "../hostsim/hostsim.cpp"

namespace {

struct ComplexBackend : HostBackend {
  // y = A x with complex values, rounded as the engines' complex arithmetic rounds (csrc/complex.h)
  template <typename T>
  static void spmv(const HostCsr *A, const void *x, void *y) {
    const T *v = (const T *)A->vals, *xx = (const T *)x;
    T *yy = (T *)y;
    for (int64_t i = 0; i < A->m; ++i) {
      T t = (T)0;
      for (int64_t k = A->rowptr[i]; k < A->rowptr[i + 1]; ++k) t = t + v[k] * xx[A->colind[k]];
      yy[i] = t;
    }
  }
  int apply(const Op *A, const void *x, void *y) {
    ++applies;
    if (A->is_f64) spmv<b200::cplx<double>>(A, x, y);
    else spmv<b200::cplx<float>>(A, x, y);
    return 0;
  }
};

}  // namespace

EXPORT int hostsim_cg_c(int is_f64, const hostsim_csr *A, const hostsim_csr *Pl, const void *diag, void *x, const void *b,
                        double abstol, double reltol, int64_t maxiter, int initially_zero, int check_every,
                        int64_t hist_cap, double *hist, int order, int split, hostsim_out *out) {
  typedef b200::cplx<double> Z;
  typedef b200::cplx<float> C;
  ComplexBackend be;
  be.order = order;
  be.split = split;
  HostCsr a = mk(A, is_f64), p;
  if (Pl) p = mk(Pl, is_f64);
  b200::CgpOutcome o;
  memset(&o, 0, sizeof(o));
  int st = is_f64 ? b200::cgp_run<Z>(be, &a, Pl ? &p : nullptr, (const Z *)diag, A->m, A->n, (Z *)x, (const Z *)b, abstol,
                                     reltol, maxiter, initially_zero, check_every, hist_cap, hist, &o)
                  : b200::cgp_run<C>(be, &a, Pl ? &p : nullptr, (const C *)diag, A->m, A->n, (C *)x, (const C *)b, abstol,
                                     reltol, maxiter, initially_zero, check_every, hist_cap, hist, &o);
  out->iters = o.iters; out->mvps = o.mvps; out->mtvps = 0; out->n_hist = o.n_hist;
  out->resnorm = o.residual; out->tol = o.tol; out->converged = o.converged; out->breakdown = o.breakdown;
  out->passes = be.passes; out->applies = be.applies;
  return st;
}

EXPORT int hostsim_gmres_c(int is_f64, const hostsim_csr *A, const hostsim_csr *Pl, const hostsim_csr *Pr,
                           const void *pl_diag, const void *pr_diag, void *x, const void *b, double abstol, double reltol,
                           int restart, int64_t maxiter, int initially_zero, int orth_meth, int64_t hist_cap, double *hist,
                           int order, int split, hostsim_out *out) {
  typedef b200::cplx<double> Z;
  typedef b200::cplx<float> C;
  ComplexBackend be;
  be.order = order;
  be.split = split;
  HostCsr a = mk(A, is_f64), pl, pr;
  if (Pl) pl = mk(Pl, is_f64);
  if (Pr) pr = mk(Pr, is_f64);
  b200::GmresOutcome o;
  memset(&o, 0, sizeof(o));
  int st = is_f64 ? b200::gmres_run<Z>(be, &a, Pl ? &pl : nullptr, Pr ? &pr : nullptr, (const Z *)pl_diag,
                                       (const Z *)pr_diag, A->m, A->n, (Z *)x, (const Z *)b, abstol, reltol, restart,
                                       maxiter, initially_zero, orth_meth, hist_cap, hist, &o)
                  : b200::gmres_run<C>(be, &a, Pl ? &pl : nullptr, Pr ? &pr : nullptr, (const C *)pl_diag,
                                       (const C *)pr_diag, A->m, A->n, (C *)x, (const C *)b, abstol, reltol, restart,
                                       maxiter, initially_zero, orth_meth, hist_cap, hist, &o);
  out->iters = o.iters; out->mvps = o.mvps; out->mtvps = 0; out->n_hist = o.n_hist;
  out->resnorm = o.residual; out->tol = o.tol; out->converged = o.converged; out->breakdown = o.breakdown;
  out->passes = be.passes; out->applies = be.applies;
  return st;
}

// the complex least-squares solve of the GMRES engine (ldiv!(FastHessenberg(H), rhs), src/hessenberg.jl:15-46) on a given
// (m+1) x m column-major ComplexF64 H with leading dimension ldh and an rhs of m+1 values, both mutated in place
EXPORT void hostsim_hessenberg_c(double *H, int ldh, int m, double *rhs) {
  b200::gm_hessenberg_solve_c((b200::cplx<double> *)H, ldh, m, (b200::cplx<double> *)rhs);
}
