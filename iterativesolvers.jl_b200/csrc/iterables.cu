// iterables.cu -- the resumable forms of gmres!, minres! and bicgstabl!: gmres_iterable! (reference src/gmres.jl:108-136),
// minres_iterable! (src/minres.jl:39-89), bicgstabl_iterator! (src/bicgstabl.jl:27-73) -- "the iterator is the solver"
// of docs/src/iterators.md.  An iterable owns its scratch (basis vectors, recurrence scalars: everything the fused-pass
// engines of gmres_core.h / minres_core.h / bicgstabl_core.h keep in device memory), so solves on the same context may
// run between two b200_iter_next calls.  x and b stay the caller's device vectors, as in the reference.
#include "linop.cuh"
#include "bicgstabl_core.h"
#include "cg_core.h"
#include "gmres_core.h"
#include "minres_core.h"

using namespace b200;

namespace {
constexpr int64_t kIterWindow = 4096;   // residuals recorded per b200_iter_next call (as b200_cg_iter_next)
enum { IT_GMRES = 1, IT_MINRES = 2, IT_BICGSTABL = 3, IT_CG = 4 };
}  // namespace

struct b200_iter {
  int kind = 0, dtype = B200_F64;
  b200_ctx *ctx = nullptr;
  int64_t n = 0, n_global = 0;
  b200_linop a_fn{}, pl_fn{}, pr_fn{};          // copies of the caller's callback descriptors
  CudaOp A, Pl, Pr;
  const void *pl_diag = nullptr, *pr_diag = nullptr;
  void *x = nullptr;
  const void *b = nullptr, *shadow = nullptr;
  void *ws = nullptr;
  int restart = 0, orth = 0, l = 0;
  int64_t mv = 0;                               // products so far (gmres: counted on the host; minres: the initial one)
};

namespace {

int set_operator(b200_iter *it, b200_ctx *ctx, const b200_csr *A, const b200_linop *Aop) {
  B200_REQUIRE((A != nullptr) != (Aop != nullptr), "exactly one of the CSR operator and the callback operator must be given");
  it->ctx = ctx;
  if (A) {
    B200_REQUIRE(A->ctx == ctx, "operator belongs to another context");
    B200_REQUIRE(is_square(A), "this solver needs a square operator");
    it->A = CudaOp{A, nullptr};
    it->dtype = A->dtype;
    it->n = A->m_local;
    it->n_global = A->n_global;
  } else {
    B200_TRY(check_linop(Aop, "A"));
    B200_REQUIRE(Aop->m_global == Aop->n_global && Aop->m_local == Aop->n_local, "this solver needs a square operator");
    it->a_fn = *Aop;
    it->A = CudaOp{nullptr, &it->a_fn};
    it->dtype = Aop->dtype;
    it->n = Aop->m_local;
    it->n_global = Aop->n_global;
  }
  return B200_OK;
}

int set_precond(b200_iter *it, const b200_precond &P, const char *what, b200_linop *slot, CudaOp *op, const void **diag) {
  *op = CudaOp{};
  *diag = nullptr;
  if (P.kind == B200_PREC_IDENTITY) return B200_OK;
  B200_REQUIRE((P.kind == B200_PREC_JACOBI || P.kind == B200_PREC_CALLBACK) && P.diag, "unsupported preconditioner %s", what);
  if (P.kind == B200_PREC_JACOBI) {
    *diag = P.diag;
    return B200_OK;
  }
  const b200_linop *fn = (const b200_linop *)P.diag;
  B200_TRY(check_linop(fn, what));
  B200_REQUIRE(fn->dtype == it->dtype && fn->m_local == it->n && fn->n_local == it->n,
               "%s must act on vectors of the operator's local length", what);
  *slot = *fn;
  *op = CudaOp{nullptr, slot};
  return B200_OK;
}

int alloc_ws(b200_iter *it, size_t bytes) {
  B200_CUDA(cudaSetDevice(it->ctx->device));
  if (cudaMalloc(&it->ws, bytes) != cudaSuccess) {
    set_error("iterable: cudaMalloc(%zu) failed", bytes);
    return B200_ERR_ALLOC;
  }
  return B200_OK;
}

template <typename T>
GmresOps<T, CudaBackend> gm_ops(const b200_iter *it) {
  return GmresOps<T, CudaBackend>{&it->A, it->Pl.fn ? &it->Pl : nullptr, it->Pr.fn ? &it->Pr : nullptr,
                                  (const T *)it->pl_diag, (const T *)it->pr_diag};
}

void fill_result(b200_result *res, int64_t iters, int64_t mvps, int converged, int done, double tol, double residual,
                 int64_t n_hist) {
  if (!res) return;
  res->iters = iters;
  res->mvps = mvps;
  res->isconverged = converged;
  res->status = done ? 1 : 0;          // 1 once done() holds (as b200_cg_iter_next)
  res->tol = tol;
  res->residual = residual;
  res->n_resnorm = n_hist;
}

template <typename T>
int next_impl(b200_iter *it, int64_t k, b200_result *res, double *resnorm_host, int64_t cap) {
  CudaBackend be{it->ctx};
  const int64_t want = resnorm_host ? std::min(cap, kIterWindow) : 0;
  std::vector<double> window((size_t)kIterWindow);
  int st;
  if (it->kind == IT_GMRES) {
    const GmresLayout<T> L = gmres_layout<T>(it->ws, it->n, it->restart, kIterWindow);
    const GmresOps<T, CudaBackend> op = gm_ops<T>(it);
    if ((st = gmres_reset_window(be, L.s))) return st;
    if (k > 0 && (st = gmres_advance<T, CudaBackend>(be, op, L, it->n, (T *)it->x, (const T *)it->b, it->orth, k, &it->mv)))
      return st;
    GmresOutcome o;
    memset(&o, 0, sizeof(o));
    if ((st = gmres_collect<T, CudaBackend>(be, L, it->mv, window.data(), &o))) return st;
    const int64_t nh = std::min(o.n_hist, want);
    for (int64_t i = 0; i < nh; ++i) resnorm_host[i] = window[(size_t)i];
    fill_result(res, o.iters, o.mvps, o.converged, o.done, o.tol, o.residual, nh);
    return o.breakdown ? B200_ERR_BREAKDOWN : B200_OK;
  }
  if (it->kind == IT_MINRES) {
    const MinresLayout<T> L = minres_layout<T>(it->ws, it->n, kIterWindow);
    if ((st = minres_reset_window(be, L.s))) return st;
    if (k > 0 && (st = minres_advance<T, CudaBackend>(be, &it->A, L, it->n, (T *)it->x, k, 0))) return st;
    MinresOutcome o;
    memset(&o, 0, sizeof(o));
    if ((st = minres_collect<T, CudaBackend>(be, L, it->mv, window.data(), &o))) return st;
    const int64_t nh = std::min(o.n_hist, want);
    for (int64_t i = 0; i < nh; ++i) resnorm_host[i] = window[(size_t)i];
    fill_result(res, o.iters, o.mvps, o.converged, o.done, o.tol, o.residual, nh);
    return o.breakdown ? B200_ERR_BREAKDOWN : B200_OK;
  }
  if (it->kind == IT_CG) {
    const CgpLayout<T> L = cgp_layout<T>(it->ws, it->n, kIterWindow);
    if ((st = cgp_reset_window(be, L.s))) return st;
    if (k > 0 && (st = cgp_advance<T, CudaBackend>(be, &it->A, it->Pl.fn ? &it->Pl : nullptr, (const T *)it->pl_diag, L, it->n,
                                                  (T *)it->x, k, 0)))
      return st;
    CgpOutcome o;
    memset(&o, 0, sizeof(o));
    if ((st = cgp_collect<T, CudaBackend>(be, L, it->mv, window.data(), &o))) return st;
    const int64_t nh = std::min(o.n_hist, want);
    for (int64_t i = 0; i < nh; ++i) resnorm_host[i] = window[(size_t)i];
    fill_result(res, o.iters, o.mvps, o.converged, o.done, o.tol, o.residual, nh);
    return o.breakdown ? B200_ERR_BREAKDOWN : B200_OK;
  }
  const BcgLayout<T> L = bicgstabl_layout<T>(it->ws, it->n, it->l, kIterWindow);
  if ((st = bicgstabl_reset_window(be, L.s))) return st;
  if (k > 0 && (st = bicgstabl_advance<T, CudaBackend>(be, &it->A, it->Pl.fn ? &it->Pl : nullptr, (const T *)it->pl_diag, L,
                                                      it->n, (T *)it->x, (const T *)it->shadow, it->l, k, 0)))
    return st;
  BcgOutcome o;
  memset(&o, 0, sizeof(o));
  if ((st = bicgstabl_collect<T, CudaBackend>(be, L, window.data(), &o))) return st;
  const int64_t nh = std::min(o.n_hist, want);
  for (int64_t i = 0; i < nh; ++i) resnorm_host[i] = window[(size_t)i];
  fill_result(res, o.iters, o.mvps, o.converged, o.done, o.tol, o.residual, nh);
  if (o.singular) {
    set_error("SingularException in the BiCGStab(l) MR step (reference src/bicgstabl.jl:123)");
    return B200_ERR_BREAKDOWN;
  }
  return o.breakdown ? B200_ERR_BREAKDOWN : B200_OK;
}

}  // namespace

extern "C" {

int b200_gmres_iter_create(b200_ctx *ctx, const b200_csr *A, const b200_linop *Aop, void *x_dev, const void *b_dev,
                           const b200_gmres_opts *opts, b200_iter **out) {
  B200_TRY(real_only(A, "b200_gmres_iter_create"));
  B200_TRY(real_only(Aop ? Aop->dtype : B200_F64, "b200_gmres_iter_create"));
  B200_REQUIRE(ctx && x_dev && b_dev && opts && out, "NULL argument");
  std::unique_ptr<b200_iter> it(new b200_iter());
  it->kind = IT_GMRES;
  B200_TRY(set_operator(it.get(), ctx, A, Aop));
  B200_TRY(set_precond(it.get(), opts->Pl, "Pl", &it->pl_fn, &it->Pl, &it->pl_diag));
  B200_TRY(set_precond(it.get(), opts->Pr, "Pr", &it->pr_fn, &it->Pr, &it->pr_diag));
  it->restart = opts->restart > 0 ? opts->restart : (int)std::min<int64_t>(20, it->n_global);   // src/gmres.jl:188
  B200_REQUIRE(it->restart <= kGmMaxRestart, "restart=%d: this version supports restart <= %d", it->restart, kGmMaxRestart);
  B200_REQUIRE(opts->orth_meth >= B200_ORTH_MGS && opts->orth_meth <= B200_ORTH_DGKS, "unknown orth_meth %d", opts->orth_meth);
  it->orth = opts->orth_meth;
  it->x = x_dev;
  it->b = b_dev;
  const bool f64 = it->dtype == B200_F64;
  B200_TRY(alloc_ws(it.get(), f64 ? gmres_ws_bytes<double>(it->n, it->restart, kIterWindow)
                                  : gmres_ws_bytes<float>(it->n, it->restart, kIterWindow)));
  CudaBackend be{ctx};
  int st;
  if (f64) {
    const GmresLayout<double> L = gmres_layout<double>(it->ws, it->n, it->restart, kIterWindow);
    st = gmres_setup<double, CudaBackend>(be, gm_ops<double>(it.get()), L, it->n, it->n_global, (double *)x_dev,
                                          (const double *)b_dev, opts->abstol, opts->reltol, it->restart, opts->maxiter,
                                          opts->initially_zero, &it->mv);
  } else {
    const GmresLayout<float> L = gmres_layout<float>(it->ws, it->n, it->restart, kIterWindow);
    st = gmres_setup<float, CudaBackend>(be, gm_ops<float>(it.get()), L, it->n, it->n_global, (float *)x_dev,
                                         (const float *)b_dev, opts->abstol, opts->reltol, it->restart, opts->maxiter,
                                         opts->initially_zero, &it->mv);
  }
  if (st != B200_OK) {
    b200_iter_destroy(it.release());
    return st;
  }
  *out = it.release();
  return B200_OK;
}

int b200_minres_iter_create(b200_ctx *ctx, const b200_csr *A, const b200_linop *Aop, void *x_dev, const void *b_dev,
                            const b200_minres_opts *opts, b200_iter **out) {
  B200_TRY(real_only(A, "b200_minres_iter_create"));
  B200_TRY(real_only(Aop ? Aop->dtype : B200_F64, "b200_minres_iter_create"));
  B200_REQUIRE(ctx && x_dev && b_dev && opts && out, "NULL argument");
  std::unique_ptr<b200_iter> it(new b200_iter());
  it->kind = IT_MINRES;
  B200_TRY(set_operator(it.get(), ctx, A, Aop));
  it->x = x_dev;
  it->b = b_dev;
  const bool f64 = it->dtype == B200_F64;
  B200_TRY(alloc_ws(it.get(), f64 ? minres_ws_bytes<double>(it->n, kIterWindow) : minres_ws_bytes<float>(it->n, kIterWindow)));
  CudaBackend be{ctx};
  int st;
  if (f64)
    st = minres_setup<double, CudaBackend>(be, &it->A, minres_layout<double>(it->ws, it->n, kIterWindow), it->n, it->n_global,
                                           (double *)x_dev, (const double *)b_dev, opts->abstol, opts->reltol, opts->maxiter,
                                           opts->initially_zero, opts->skew_hermitian, &it->mv);
  else
    st = minres_setup<float, CudaBackend>(be, &it->A, minres_layout<float>(it->ws, it->n, kIterWindow), it->n, it->n_global,
                                          (float *)x_dev, (const float *)b_dev, opts->abstol, opts->reltol, opts->maxiter,
                                          opts->initially_zero, opts->skew_hermitian, &it->mv);
  if (st != B200_OK) {
    b200_iter_destroy(it.release());
    return st;
  }
  *out = it.release();
  return B200_OK;
}

int b200_bicgstabl_iter_create(b200_ctx *ctx, const b200_csr *A, const b200_linop *Aop, void *x_dev, const void *b_dev,
                               const b200_bicgstabl_opts *opts, b200_iter **out) {
  B200_TRY(real_only(A, "b200_bicgstabl_iter_create"));
  B200_TRY(real_only(Aop ? Aop->dtype : B200_F64, "b200_bicgstabl_iter_create"));
  B200_REQUIRE(ctx && x_dev && b_dev && opts && out, "NULL argument");
  B200_REQUIRE(opts->l >= 1 && opts->l <= kBcMaxL, "bicgstabl!: l=%d not in 1..%d", opts->l, kBcMaxL);
  B200_REQUIRE(opts->r_shadow, "r_shadow (device vector) is required: the reference draws rand(T, n) "
                               "(src/bicgstabl.jl:38), the host passes the draw");
  std::unique_ptr<b200_iter> it(new b200_iter());
  it->kind = IT_BICGSTABL;
  B200_TRY(set_operator(it.get(), ctx, A, Aop));
  B200_TRY(set_precond(it.get(), opts->Pl, "Pl", &it->pl_fn, &it->Pl, &it->pl_diag));
  it->l = opts->l;
  it->x = x_dev;
  it->b = b_dev;
  it->shadow = opts->r_shadow;
  const bool f64 = it->dtype == B200_F64;
  B200_TRY(alloc_ws(it.get(), f64 ? bicgstabl_ws_bytes<double>(it->n, it->l, kIterWindow)
                                  : bicgstabl_ws_bytes<float>(it->n, it->l, kIterWindow)));
  CudaBackend be{ctx};
  const CudaOp *pl = it->Pl.fn ? &it->Pl : nullptr;
  int st;
  if (f64)
    st = bicgstabl_setup<double, CudaBackend>(be, &it->A, pl, (const double *)it->pl_diag,
                                              bicgstabl_layout<double>(it->ws, it->n, it->l, kIterWindow), it->n,
                                              it->n_global, (double *)x_dev, (const double *)b_dev, it->l, opts->abstol,
                                              opts->reltol, opts->max_mv_products, opts->initial_zero);
  else
    st = bicgstabl_setup<float, CudaBackend>(be, &it->A, pl, (const float *)it->pl_diag,
                                             bicgstabl_layout<float>(it->ws, it->n, it->l, kIterWindow), it->n, it->n_global,
                                             (float *)x_dev, (const float *)b_dev, it->l, opts->abstol, opts->reltol,
                                             opts->max_mv_products, opts->initial_zero);
  if (st != B200_OK) {
    b200_iter_destroy(it.release());
    return st;
  }
  *out = it.release();
  return B200_OK;
}

// cg_iterator!(x, A, b, Pl; ...) for a callback operator and / or a callback preconditioner (reference src/cg.jl:120-155);
// the CSR + Identity / Jacobi form is b200_cg_iter_create (tuned engine, caller-owned state vectors).
int b200_cg_iter_create_op(b200_ctx *ctx, const b200_csr *A, const b200_linop *Aop, void *x_dev, const void *b_dev,
                           const b200_cg_opts *opts, b200_iter **out) {
  B200_TRY(real_only(A, "b200_cg_iter_create_op"));
  B200_TRY(real_only(Aop ? Aop->dtype : B200_F64, "b200_cg_iter_create_op"));
  B200_REQUIRE(ctx && x_dev && b_dev && opts && out, "NULL argument");
  B200_REQUIRE(!opts->fixed_iterations && !opts->variant, "fixed_iterations / variant are not available on this path");
  std::unique_ptr<b200_iter> it(new b200_iter());
  it->kind = IT_CG;
  B200_TRY(set_operator(it.get(), ctx, A, Aop));
  B200_TRY(set_precond(it.get(), opts->Pl, "Pl", &it->pl_fn, &it->Pl, &it->pl_diag));
  it->x = x_dev;
  it->b = b_dev;
  const bool f64 = it->dtype == B200_F64;
  B200_TRY(alloc_ws(it.get(), f64 ? cgp_ws_bytes<double>(it->n, kIterWindow) : cgp_ws_bytes<float>(it->n, kIterWindow)));
  CudaBackend be{ctx};
  const bool precond = it->Pl.fn != nullptr || it->pl_diag != nullptr;
  int st;
  if (f64)
    st = cgp_setup<double, CudaBackend>(be, &it->A, precond, cgp_layout<double>(it->ws, it->n, kIterWindow), it->n,
                                        it->n_global, (double *)x_dev, (const double *)b_dev, opts->abstol, opts->reltol,
                                        opts->maxiter, opts->initially_zero, &it->mv);
  else
    st = cgp_setup<float, CudaBackend>(be, &it->A, precond, cgp_layout<float>(it->ws, it->n, kIterWindow), it->n,
                                       it->n_global, (float *)x_dev, (const float *)b_dev, opts->abstol, opts->reltol,
                                       opts->maxiter, opts->initially_zero, &it->mv);
  if (st != B200_OK) {
    b200_iter_destroy(it.release());
    return st;
  }
  *out = it.release();
  return B200_OK;
}

int b200_iter_next(b200_iter *it, int64_t k, b200_result *res, double *resnorm_host, int64_t resnorm_cap) {
  B200_REQUIRE(it && it->ctx && it->ws, "NULL argument");
  B200_REQUIRE(k >= 0, "k must be >= 0 (0 reports the state without iterating)");
  B200_CUDA(cudaSetDevice(it->ctx->device));
  return it->dtype == B200_F64 ? next_impl<double>(it, k, res, resnorm_host, resnorm_cap)
                               : next_impl<float>(it, k, res, resnorm_host, resnorm_cap);
}

int b200_iter_destroy(b200_iter *it) {
  if (!it) return B200_OK;
  if (it->ctx) {
    cudaSetDevice(it->ctx->device);
    cudaStreamSynchronize(it->ctx->stream);
  }
  if (it->ws) cudaFree(it->ws);
  delete it;
  return B200_OK;
}

}  // extern "C"
