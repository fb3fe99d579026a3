// minres_bicgstabl_op.cu -- minres! and bicgstabl! for general (callback) operators, bicgstabl! with a callback
// preconditioner: the fused-pass engines of minres_core.h / bicgstabl_core.h on the CUDA backend.  b200_csr operators
// (with Identity / Jacobi) take the specialised engines of minres.cu / bicgstabl.cu; b200_bicgstabl_solve forwards here
// when its preconditioner is a callback.
#include "linop.cuh"
#include "bicgstabl_core.h"
#include "minres_core.h"

using namespace b200;

namespace b200 {

int bicgstabl_general(b200_ctx *ctx, const CudaOp &A, int dtype, int64_t n, int64_t n_global, void *x_dev,
                      const void *b_dev, const b200_bicgstabl_opts *opts, b200_result *res, double *resnorm_host,
                      int64_t resnorm_cap) {
  B200_REQUIRE(opts->l >= 1 && opts->l <= kBcMaxL, "bicgstabl!: l=%d not in 1..%d", opts->l, kBcMaxL);
  B200_REQUIRE(opts->r_shadow, "r_shadow (device vector) is required: the reference draws rand(T, n) "
                               "(src/bicgstabl.jl:38), the host passes the draw");
  const b200_linop *plf = nullptr;
  const void *diag = nullptr;
  if (opts->Pl.kind == B200_PREC_JACOBI) {
    B200_REQUIRE(opts->Pl.diag, "Jacobi preconditioner without a diagonal");
    diag = opts->Pl.diag;
  } else if (opts->Pl.kind == B200_PREC_CALLBACK) {
    plf = (const b200_linop *)opts->Pl.diag;
    B200_TRY(check_linop(plf, "Pl"));
    B200_REQUIRE(plf->dtype == dtype && plf->m_local == n && plf->n_local == n,
                 "Pl must act on vectors of the operator's local length");
  } else {
    B200_REQUIRE(opts->Pl.kind == B200_PREC_IDENTITY, "unsupported preconditioner");
  }
  B200_CUDA(cudaSetDevice(ctx->device));
  CudaBackend be{ctx};
  CudaOp pl{nullptr, plf};
  BcgOutcome o;
  memset(&o, 0, sizeof(o));
  const int st =
      dtype == B200_F64
          ? bicgstabl_run<double>(be, &A, plf ? &pl : nullptr, (const double *)diag, n, n_global, (double *)x_dev,
                                  (const double *)b_dev, (const double *)opts->r_shadow, opts->l, opts->abstol, opts->reltol,
                                  opts->max_mv_products, opts->initial_zero, 0, resnorm_cap, resnorm_host, &o)
          : bicgstabl_run<float>(be, &A, plf ? &pl : nullptr, (const float *)diag, n, n_global, (float *)x_dev,
                                 (const float *)b_dev, (const float *)opts->r_shadow, opts->l, opts->abstol, opts->reltol,
                                 opts->max_mv_products, opts->initial_zero, 0, resnorm_cap, resnorm_host, &o);
  if (st != B200_OK) return st;
  if (res) {
    res->iters = o.iters;
    res->mvps = o.mvps;
    res->isconverged = o.converged;
    res->status = (o.breakdown || o.singular) ? B200_ERR_BREAKDOWN : 0;
    res->tol = o.tol;
    res->residual = o.residual;
    res->n_resnorm = o.n_hist;
  }
  if (o.singular) {
    set_error("SingularException in the BiCGStab(l) MR step (reference src/bicgstabl.jl:123)");
    return B200_ERR_BREAKDOWN;
  }
  return B200_OK;
}

}  // namespace b200

extern "C" {

int b200_bicgstabl_solve_op(b200_ctx *ctx, const b200_linop *A, void *x_dev, const void *b_dev,
                            const b200_bicgstabl_opts *opts, b200_result *res, double *resnorm_host, int64_t resnorm_cap) {
  B200_TRY(real_only(A ? A->dtype : B200_F64, "b200_bicgstabl_solve_op"));
  B200_REQUIRE(ctx && x_dev && b_dev && opts, "NULL argument");
  B200_TRY(check_linop(A, "A"));
  B200_REQUIRE(A->m_global == A->n_global && A->m_local == A->n_local, "bicgstabl! needs a square operator");
  return bicgstabl_general(ctx, CudaOp{nullptr, A}, A->dtype, A->m_local, A->n_global, x_dev, b_dev, opts, res,
                           resnorm_host, resnorm_cap);
}

int b200_minres_solve_op(b200_ctx *ctx, const b200_linop *A, void *x_dev, const void *b_dev, const b200_minres_opts *opts,
                         b200_result *res, double *resnorm_host, int64_t resnorm_cap) {
  B200_TRY(real_only(A ? A->dtype : B200_F64, "b200_minres_solve_op"));
  B200_REQUIRE(ctx && x_dev && b_dev && opts, "NULL argument");
  B200_TRY(check_linop(A, "A"));
  B200_REQUIRE(A->m_global == A->n_global && A->m_local == A->n_local, "minres! needs a square operator");
  B200_CUDA(cudaSetDevice(ctx->device));
  CudaBackend be{ctx};
  CudaOp a{nullptr, A};
  MinresOutcome o;
  memset(&o, 0, sizeof(o));
  const int64_t n = A->m_local;
  const int st = A->dtype == B200_F64
                     ? minres_run<double>(be, &a, n, A->n_global, (double *)x_dev, (const double *)b_dev, opts->abstol,
                                          opts->reltol, opts->maxiter, opts->initially_zero, opts->skew_hermitian, 0,
                                          resnorm_cap, resnorm_host, &o)
                     : minres_run<float>(be, &a, n, A->n_global, (float *)x_dev, (const float *)b_dev, opts->abstol,
                                         opts->reltol, opts->maxiter, opts->initially_zero, opts->skew_hermitian, 0,
                                         resnorm_cap, resnorm_host, &o);
  if (st != B200_OK) return st;
  if (res) {
    res->iters = o.iters;
    res->mvps = o.mvps;
    res->isconverged = o.converged;
    res->status = o.breakdown ? B200_ERR_BREAKDOWN : 0;
    res->tol = o.tol;
    res->residual = o.residual;
    res->n_resnorm = o.n_hist;
  }
  return B200_OK;
}

}  // extern "C"
