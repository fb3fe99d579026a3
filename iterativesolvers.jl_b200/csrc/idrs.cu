// idrs.cu -- idrs!(x, A, b; s, Pl, ...) of reference src/idrs.jl:49-64 on the GPU: the fused-pass engine of
// idrs_core.h instantiated with the CUDA backend (pass.cuh).  The s x s system (M, f, c, omega) is solved inside the
// scalar sections of the passes; the host only polls the done flag.
#include "linop.cuh"
#include "idrs_core.h"

using namespace b200;

namespace {

int idrs_dispatch(b200_ctx *ctx, const CudaOp &A, int dtype, int64_t n, int64_t n_global, void *x_dev,
                  const void *b_dev, const b200_idrs_opts *opts, b200_result *res, double *resnorm_host,
                  int64_t resnorm_cap) {
  B200_REQUIRE(opts->s >= 1 && opts->s <= kIdrsMaxS, "shadow space dimension s must be in [1, %d]", kIdrsMaxS);
  B200_REQUIRE(opts->P && opts->ldp >= n, "P (n x s shadow vectors, device) is required: the reference draws "
                                          "rand!(copy(C)) (src/idrs.jl:132), the host passes the draw");
  B200_REQUIRE(opts->Pl.kind == B200_PREC_IDENTITY ||
                   ((opts->Pl.kind == B200_PREC_JACOBI || opts->Pl.kind == B200_PREC_CALLBACK) && opts->Pl.diag),
               "unsupported preconditioner");
  const b200_linop *plfn = opts->Pl.kind == B200_PREC_CALLBACK ? (const b200_linop *)opts->Pl.diag : nullptr;
  if (plfn) {
    B200_TRY(check_linop(plfn, "Pl"));
    B200_REQUIRE(plfn->dtype == dtype && plfn->m_local == n && plfn->n_local == n,
                 "Pl must act on vectors of the operator's local length");
  }
  B200_CUDA(cudaSetDevice(ctx->device));
  CudaBackend be{ctx};
  IdrsOutcome o;
  memset(&o, 0, sizeof(o));
  const void *diag = opts->Pl.kind == B200_PREC_JACOBI ? opts->Pl.diag : nullptr;
  CudaOp plop{nullptr, plfn};
  const CudaOp *plp = plfn ? &plop : nullptr;
  const int st =
      dtype == B200_F64
          ? idrs_run<double>(be, &A, n, n_global, (double *)x_dev, (const double *)b_dev, opts->s,
                             (const double *)opts->P, opts->ldp, (const double *)diag, opts->abstol, opts->reltol,
                             opts->maxiter, opts->smoothing, opts->check_every, resnorm_cap, resnorm_host, &o, plp)
          : idrs_run<float>(be, &A, n, n_global, (float *)x_dev, (const float *)b_dev, opts->s, (const float *)opts->P,
                            opts->ldp, (const float *)diag, opts->abstol, opts->reltol, opts->maxiter, opts->smoothing,
                            opts->check_every, resnorm_cap, resnorm_host, &o, plp);
  if (st != B200_OK) return st;
  if (res) {
    res->iters = o.iters;
    res->mvps = o.iters;                 // nextiter!(it.log, mvps=1) per step  src/idrs.jl:267
    res->isconverged = o.converged;      // 0 <= normR < tol  src/idrs.jl:168
    res->status = o.breakdown ? B200_ERR_BREAKDOWN : 0;
    res->tol = o.tol;
    res->residual = o.normR;
    res->n_resnorm = o.n_hist;
  }
  return B200_OK;
}

}  // namespace

extern "C" {

int b200_idrs_solve(b200_ctx *ctx, const b200_csr *A, void *x_dev, const void *b_dev, const b200_idrs_opts *opts,
                    b200_result *res, double *resnorm_host, int64_t resnorm_cap) {
  B200_TRY(real_only(A, "b200_idrs_solve"));
  B200_REQUIRE(ctx && A && x_dev && b_dev && opts, "NULL argument");
  B200_REQUIRE(A->ctx == ctx, "operator belongs to another context");
  B200_REQUIRE(is_square(A), "idrs! needs a square operator (got %lld x %lld)", (long long)A->m_global,
               (long long)A->n_global);
  return idrs_dispatch(ctx, CudaOp{A, nullptr}, A->dtype, A->m_local, A->n_global, x_dev, b_dev, opts, res,
                       resnorm_host, resnorm_cap);
}

int b200_idrs_solve_op(b200_ctx *ctx, const b200_linop *A, void *x_dev, const void *b_dev, const b200_idrs_opts *opts,
                       b200_result *res, double *resnorm_host, int64_t resnorm_cap) {
  B200_TRY(real_only(A ? A->dtype : B200_F64, "b200_idrs_solve_op"));
  B200_REQUIRE(ctx && x_dev && b_dev && opts, "NULL argument");
  B200_TRY(check_linop(A, "A"));
  B200_REQUIRE(A->m_global == A->n_global && A->m_local == A->n_local, "idrs! needs a square operator");
  return idrs_dispatch(ctx, CudaOp{nullptr, A}, A->dtype, A->m_local, A->n_global, x_dev, b_dev, opts, res,
                       resnorm_host, resnorm_cap);
}

}  // extern "C"
