// qmr.cu -- qmr!(x, A, b; ...) of reference src/qmr.jl:262-297 on the GPU: the fused-pass engine of qmr_core.h
// instantiated with the CUDA backend (pass.cuh).  Six launches per iteration besides the two operator applications;
// every scalar of the two-sided Lanczos process and of the QMR rotations stays in device memory (QmrScal).
// The operator pair (A, adjoint(A)) is either two b200_csr handles or two b200_linop callbacks.
#include "pass.cuh"
#include "qmr_core.h"

using namespace b200;

namespace {

int qmr_dispatch(b200_ctx *ctx, const CudaOp &A, const CudaOp &At, int dtype, int64_t n, int64_t n_global, void *x_dev,
                 const void *b_dev, const b200_qmr_opts *opts, b200_result *res, double *resnorm_host,
                 int64_t resnorm_cap) {
  B200_CUDA(cudaSetDevice(ctx->device));
  CudaBackend be{ctx};
  QmrOutcome o;
  memset(&o, 0, sizeof(o));
  const int st = dtype == B200_F64
                     ? qmr_run<double>(be, &A, &At, n, n_global, (double *)x_dev, (const double *)b_dev, opts->abstol,
                                       opts->reltol, opts->maxiter, opts->initially_zero, opts->check_every,
                                       resnorm_cap, resnorm_host, &o)
                     : qmr_run<float>(be, &A, &At, n, n_global, (float *)x_dev, (const float *)b_dev, opts->abstol,
                                      opts->reltol, opts->maxiter, opts->initially_zero, opts->check_every,
                                      resnorm_cap, resnorm_host, &o);
  if (st != B200_OK) return st;
  if (res) {
    res->iters = o.iters;
    res->mvps = o.mvps + o.mtvps;       // products with A and with A' (the reference's history counts neither)
    res->isconverged = o.converged;
    res->status = o.breakdown ? B200_ERR_BREAKDOWN : 0;
    res->tol = o.tol;
    res->residual = o.resnorm;
    res->n_resnorm = o.n_hist;
  }
  return B200_OK;
}

}  // namespace

namespace b200 {
// argument check of a b200_linop with the complex element types allowed (cg! and gmres! on single-GPU contexts)
int check_linop_complex(const b200_linop *A, const char *what) {
  B200_REQUIRE(A, "%s is NULL", what);
  B200_REQUIRE(A->apply, "%s: apply callback is NULL", what);
  B200_REQUIRE(A->dtype >= B200_F64 && A->dtype <= B200_CF32, "%s: bad dtype", what);
  B200_REQUIRE(A->m_local >= 0 && A->n_local >= 0 && A->m_global >= A->m_local && A->n_global >= A->n_local,
               "%s: bad dimensions", what);
  return B200_OK;
}
// argument check shared by the *_op entry points (linop.cuh): real element types only
int check_linop(const b200_linop *A, const char *what) {
  B200_REQUIRE(A, "%s is NULL", what);
  B200_TRY(real_only(A->dtype, what));
  return check_linop_complex(A, what);
}
}  // namespace b200

extern "C" {

int b200_qmr_solve(b200_ctx *ctx, const b200_csr *A, const b200_csr *At, void *x_dev, const void *b_dev,
                   const b200_qmr_opts *opts, b200_result *res, double *resnorm_host, int64_t resnorm_cap) {
  B200_TRY(real_only(A, "b200_qmr_solve"));
  B200_TRY(real_only(At, "b200_qmr_solve"));
  B200_REQUIRE(ctx && A && At && x_dev && b_dev && opts, "NULL argument");
  B200_REQUIRE(A->ctx == ctx && At->ctx == ctx, "operator belongs to another context");
  B200_REQUIRE(is_square(A), "qmr! needs a square operator (got %lld x %lld)", (long long)A->m_global,
               (long long)A->n_global);
  B200_REQUIRE(At->dtype == A->dtype && At->m_local == A->m_local && At->n_global == A->n_global &&
                   At->row_begin == A->row_begin,
               "At must be the adjoint of A with the same row partition");
  return qmr_dispatch(ctx, CudaOp{A, nullptr}, CudaOp{At, nullptr}, A->dtype, A->m_local, A->n_global, x_dev, b_dev,
                      opts, res, resnorm_host, resnorm_cap);
}

int b200_qmr_solve_op(b200_ctx *ctx, const b200_linop *A, const b200_linop *At, void *x_dev, const void *b_dev,
                      const b200_qmr_opts *opts, b200_result *res, double *resnorm_host, int64_t resnorm_cap) {
  B200_TRY(real_only(A ? A->dtype : B200_F64, "b200_qmr_solve_op"));
  B200_TRY(real_only(At ? At->dtype : B200_F64, "b200_qmr_solve_op"));
  B200_REQUIRE(ctx && x_dev && b_dev && opts, "NULL argument");
  B200_TRY(check_linop(A, "A"));
  B200_TRY(check_linop(At, "At"));
  B200_REQUIRE(A->m_global == A->n_global && A->m_local == A->n_local, "qmr! needs a square operator");
  B200_REQUIRE(At->dtype == A->dtype && At->m_local == A->m_local && At->n_local == A->n_local,
               "At must be the adjoint of A with the same partition");
  return qmr_dispatch(ctx, CudaOp{nullptr, A}, CudaOp{nullptr, At}, A->dtype, A->m_local, A->n_global, x_dev, b_dev,
                      opts, res, resnorm_host, resnorm_cap);
}

}  // extern "C"
