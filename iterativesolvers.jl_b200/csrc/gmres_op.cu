// gmres_op.cu -- gmres!(x, A, b; Pl, Pr, ...) for general (callback) operators and preconditioners: the fused-pass engine
// of gmres_core.h on the CUDA backend.  b200_csr operators with Identity / Jacobi on both sides take the specialised
// engine of gmres.cu; b200_gmres_solve forwards here when one of its preconditioners is a callback.
#include "linop.cuh"
#include "gmres_core.h"

using namespace b200;

namespace b200 {

// one side of the preconditioning: callback, Jacobi diagonal or Identity
static int side(const b200_precond &P, const char *what, int dtype, int64_t n, const b200_linop **fn, const void **diag) {
  *fn = nullptr;
  *diag = nullptr;
  if (P.kind == B200_PREC_IDENTITY) return B200_OK;
  B200_REQUIRE((P.kind == B200_PREC_JACOBI || P.kind == B200_PREC_CALLBACK) && P.diag, "unsupported preconditioner %s", what);
  if (P.kind == B200_PREC_JACOBI) {
    *diag = P.diag;
    return B200_OK;
  }
  *fn = (const b200_linop *)P.diag;
  B200_TRY(check_linop_complex(*fn, what));
  B200_REQUIRE((*fn)->dtype == dtype && (*fn)->m_local == n && (*fn)->n_local == n,
               "%s must act on vectors of the operator's local length", what);
  return B200_OK;
}

int gmres_general(b200_ctx *ctx, const CudaOp &A, int dtype, int64_t n, int64_t n_global, void *x_dev, const void *b_dev,
                  const b200_gmres_opts *opts, b200_result *res, double *resnorm_host, int64_t resnorm_cap) {
  const b200_linop *plf, *prf;
  const void *pld, *prd;
  if (is_complex_dtype(dtype) && ctx->world > 1) {
    set_error("gmres!: %s operators are single-GPU in this version", dtype_name(dtype));
    return B200_ERR_UNSUPPORTED;
  }
  B200_TRY(side(opts->Pl, "Pl", dtype, n, &plf, &pld));
  B200_TRY(side(opts->Pr, "Pr", dtype, n, &prf, &prd));
  const int restart = opts->restart > 0 ? opts->restart : (int)std::min<int64_t>(20, n_global);   // src/gmres.jl:188
  B200_REQUIRE(restart <= kGmMaxRestart, "restart=%d: this version supports restart <= %d", restart, kGmMaxRestart);
  B200_REQUIRE(opts->orth_meth >= B200_ORTH_MGS && opts->orth_meth <= B200_ORTH_DGKS, "unknown orth_meth %d", opts->orth_meth);
  static_assert(B200_ORTH_MGS == GM_ORTH_MGS && B200_ORTH_CGS == GM_ORTH_CGS && B200_ORTH_DGKS == GM_ORTH_DGKS, "orth codes");
  B200_CUDA(cudaSetDevice(ctx->device));
  CudaBackend be{ctx};
  CudaOp pl{nullptr, plf}, pr{nullptr, prf};
  GmresOutcome o;
  memset(&o, 0, sizeof(o));
  int st;
  if (dtype == B200_CF64)
    st = gmres_run<cplx<double>>(be, &A, plf ? &pl : nullptr, prf ? &pr : nullptr, (const cplx<double> *)pld,
                                 (const cplx<double> *)prd, n, n_global, (cplx<double> *)x_dev, (const cplx<double> *)b_dev,
                                 opts->abstol, opts->reltol, restart, opts->maxiter, opts->initially_zero, opts->orth_meth,
                                 resnorm_cap, resnorm_host, &o);
  else if (dtype == B200_CF32)
    st = gmres_run<cplx<float>>(be, &A, plf ? &pl : nullptr, prf ? &pr : nullptr, (const cplx<float> *)pld,
                                (const cplx<float> *)prd, n, n_global, (cplx<float> *)x_dev, (const cplx<float> *)b_dev,
                                opts->abstol, opts->reltol, restart, opts->maxiter, opts->initially_zero, opts->orth_meth,
                                resnorm_cap, resnorm_host, &o);
  else
    st =
      dtype == B200_F64
          ? gmres_run<double>(be, &A, plf ? &pl : nullptr, prf ? &pr : nullptr, (const double *)pld, (const double *)prd, n,
                              n_global, (double *)x_dev, (const double *)b_dev, opts->abstol, opts->reltol, restart,
                              opts->maxiter, opts->initially_zero, opts->orth_meth, resnorm_cap, resnorm_host, &o)
          : gmres_run<float>(be, &A, plf ? &pl : nullptr, prf ? &pr : nullptr, (const float *)pld, (const float *)prd, n,
                             n_global, (float *)x_dev, (const float *)b_dev, opts->abstol, opts->reltol, restart,
                             opts->maxiter, opts->initially_zero, opts->orth_meth, resnorm_cap, resnorm_host, &o);
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

}  // namespace b200

extern "C" {

int b200_gmres_solve_op(b200_ctx *ctx, const b200_linop *A, void *x_dev, const void *b_dev, const b200_gmres_opts *opts,
                        b200_result *res, double *resnorm_host, int64_t resnorm_cap) {
  B200_REQUIRE(ctx && x_dev && b_dev && opts, "NULL argument");
  B200_TRY(check_linop_complex(A, "A"));
  B200_REQUIRE(A->m_global == A->n_global && A->m_local == A->n_local, "gmres! needs a square operator");
  return gmres_general(ctx, CudaOp{nullptr, A}, A->dtype, A->m_local, A->n_global, x_dev, b_dev, opts, res, resnorm_host,
                       resnorm_cap);
}

}  // extern "C"
