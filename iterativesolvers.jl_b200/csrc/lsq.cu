// lsq.cu -- lsqr!(x, A, b; ...) (reference src/lsqr.jl:66-77) and lsmr!(x, A, b; ...) (reference src/lsmr.jl:67-82) on
// the GPU: the fused-pass engines of lsqr_core.h / lsmr_core.h instantiated with the CUDA backend (pass.cuh).
// Four vector launches per iteration besides the two SpMVs; every scalar of the Golub-Kahan process, of the plane
// rotations and of the stopping rules stays in device memory.  A may be rectangular (single-GPU contexts).
#include "linop.cuh"
#include "lsmr_core.h"
#include "lsqr_core.h"

using namespace b200;

namespace {

int check_ls_args(b200_ctx *ctx, const b200_csr *A, const b200_csr *At, const void *x, const void *b,
                  const b200_lsq_opts *o) {
  B200_REQUIRE(ctx && A && At && x && b && o, "NULL argument");
  B200_REQUIRE(A->ctx == ctx && At->ctx == ctx, "operator belongs to another context");
  B200_REQUIRE(At->dtype == A->dtype, "A and At differ in element type");
  if (ctx->world == 1) {
    B200_REQUIRE(At->m_global == A->n_global && At->n_global == A->m_global, "At must be n x m for an m x n operator A");
  } else {
    B200_REQUIRE(is_square(A) && is_square(At) && At->m_local == A->m_local && At->row_begin == A->row_begin,
                 "multi-GPU contexts: A square, At its adjoint with the same row partition");
  }
  return B200_OK;
}

void fill_result(b200_lsq_result *r, int64_t iters, int64_t mvps, int64_t mtvps, int converged, int istop,
                 int64_t n_hist, int64_t stride, double atol, double btol, double ctol) {
  if (!r) return;
  r->iters = iters;
  r->mvps = mvps;
  r->mtvps = mtvps;
  r->isconverged = converged;
  r->istop = istop;
  r->status = 0;
  r->reserved = 0;
  r->n_hist = n_hist;
  r->hist_stride = stride;
  r->atol = atol;
  r->btol = btol;
  r->ctol = ctol;
}

template <bool LSMR>
int lsq_dispatch(b200_ctx *ctx, const CudaOp &A, const CudaOp &At, int dtype, int64_t m, int64_t n, int64_t m_global,
                 int64_t n_global, void *x_dev, const void *b_dev, const b200_lsq_opts *opts, b200_lsq_result *res,
                 double *hist_host, int64_t hist_cap) {
  B200_CUDA(cudaSetDevice(ctx->device));
  CudaBackend be{ctx};
  int64_t maxiter = opts->maxiter;
  if (maxiter < 0) maxiter = std::max(m_global, n_global);                  // maximum(size(A))  src/lsqr.jl:67, src/lsmr.jl:68
  if constexpr (LSMR) {
    LsmrOutcome o;
    memset(&o, 0, sizeof(o));
    const int st = dtype == B200_F64
                       ? lsmr_run<double>(be, &A, &At, m, n, (double *)x_dev, (const double *)b_dev, opts->damp,
                                          opts->atol, opts->btol, opts->conlim, maxiter, opts->check_every, hist_cap,
                                          hist_host, &o)
                       : lsmr_run<float>(be, &A, &At, m, n, (float *)x_dev, (const float *)b_dev, opts->damp,
                                         opts->atol, opts->btol, opts->conlim, maxiter, opts->check_every, hist_cap,
                                         hist_host, &o);
    if (st != B200_OK) return st;
    fill_result(res, o.iters, o.mvps, o.mtvps, o.converged, o.istop, o.n_hist, o.hist_stride, o.atol, o.btol, o.ctol);
    return B200_OK;
  } else {
    LsqrOutcome o;
    memset(&o, 0, sizeof(o));
    const int st = dtype == B200_F64
                       ? lsqr_run<double>(be, &A, &At, m, n, (double *)x_dev, (const double *)b_dev, opts->damp,
                                          opts->atol, opts->btol, opts->conlim, maxiter, opts->check_every, hist_cap,
                                          hist_host, &o)
                       : lsqr_run<float>(be, &A, &At, m, n, (float *)x_dev, (const float *)b_dev, opts->damp,
                                         opts->atol, opts->btol, opts->conlim, maxiter, opts->check_every, hist_cap,
                                         hist_host, &o);
    if (st != B200_OK) return st;
    fill_result(res, o.iters, o.mvps, o.mtvps, o.converged, o.istop, o.n_hist, o.hist_stride, o.atol, o.btol, o.ctol);
    if (o.bad_x) {
      set_error("Initial guess for x must be finite");                      // src/lsqr.jl:102-104
      if (res) res->status = B200_ERR_INVALID;
      return B200_ERR_INVALID;
    }
    return B200_OK;
  }
}

int check_ls_op_args(b200_ctx *ctx, const b200_linop *A, const b200_linop *At, const void *x, const void *b,
                     const b200_lsq_opts *o) {
  B200_REQUIRE(ctx && x && b && o, "NULL argument");
  B200_TRY(check_linop(A, "A"));
  B200_TRY(check_linop(At, "At"));
  B200_REQUIRE(At->dtype == A->dtype && At->m_local == A->n_local && At->n_local == A->m_local,
               "At must map the range of A back to its domain (n x m for an m x n operator A)");
  return B200_OK;
}

}  // namespace

extern "C" {

int b200_lsqr_solve(b200_ctx *ctx, const b200_csr *A, const b200_csr *At, void *x_dev, const void *b_dev,
                    const b200_lsq_opts *opts, b200_lsq_result *res, double *hist_host, int64_t hist_cap) {
  B200_TRY(real_only(A, "b200_lsqr_solve"));
  B200_TRY(real_only(At, "b200_lsqr_solve"));
  B200_TRY(check_ls_args(ctx, A, At, x_dev, b_dev, opts));
  return lsq_dispatch<false>(ctx, CudaOp{A, nullptr}, CudaOp{At, nullptr}, A->dtype, A->m_local, At->m_local,
                             A->m_global, A->n_global, x_dev, b_dev, opts, res, hist_host, hist_cap);
}

int b200_lsmr_solve(b200_ctx *ctx, const b200_csr *A, const b200_csr *At, void *x_dev, const void *b_dev,
                    const b200_lsq_opts *opts, b200_lsq_result *res, double *hist_host, int64_t hist_cap) {
  B200_TRY(real_only(A, "b200_lsmr_solve"));
  B200_TRY(real_only(At, "b200_lsmr_solve"));
  B200_TRY(check_ls_args(ctx, A, At, x_dev, b_dev, opts));
  return lsq_dispatch<true>(ctx, CudaOp{A, nullptr}, CudaOp{At, nullptr}, A->dtype, A->m_local, At->m_local,
                            A->m_global, A->n_global, x_dev, b_dev, opts, res, hist_host, hist_cap);
}

int b200_lsqr_solve_op(b200_ctx *ctx, const b200_linop *A, const b200_linop *At, void *x_dev, const void *b_dev,
                       const b200_lsq_opts *opts, b200_lsq_result *res, double *hist_host, int64_t hist_cap) {
  B200_TRY(real_only(A ? A->dtype : B200_F64, "b200_lsqr_solve_op"));
  B200_TRY(real_only(At ? At->dtype : B200_F64, "b200_lsqr_solve_op"));
  B200_TRY(check_ls_op_args(ctx, A, At, x_dev, b_dev, opts));
  return lsq_dispatch<false>(ctx, CudaOp{nullptr, A}, CudaOp{nullptr, At}, A->dtype, A->m_local, A->n_local,
                             A->m_global, A->n_global, x_dev, b_dev, opts, res, hist_host, hist_cap);
}

int b200_lsmr_solve_op(b200_ctx *ctx, const b200_linop *A, const b200_linop *At, void *x_dev, const void *b_dev,
                       const b200_lsq_opts *opts, b200_lsq_result *res, double *hist_host, int64_t hist_cap) {
  B200_TRY(real_only(A ? A->dtype : B200_F64, "b200_lsmr_solve_op"));
  B200_TRY(real_only(At ? At->dtype : B200_F64, "b200_lsmr_solve_op"));
  B200_TRY(check_ls_op_args(ctx, A, At, x_dev, b_dev, opts));
  return lsq_dispatch<true>(ctx, CudaOp{nullptr, A}, CudaOp{nullptr, At}, A->dtype, A->m_local, A->n_local,
                            A->m_global, A->n_global, x_dev, b_dev, opts, res, hist_host, hist_cap);
}

}  // extern "C"
