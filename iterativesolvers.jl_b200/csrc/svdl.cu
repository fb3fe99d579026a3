// svdl.cu -- svdl(A; nsv, k, j, tol, reltol, maxiter, method = :ritz, vecs, dolock, v0) of reference src/svdl.jl:157-247
// on the GPU: the fused-pass engine of svdl_core.h on the CUDA backend (pass.cuh).  The Lanczos bases live on the
// device, the k x k projected problem is solved on the host once per outer iteration (as in the reference).
#include "linop.cuh"
#include "svdl_core.h"

using namespace b200;

namespace {

int svdl_dispatch(b200_ctx *ctx, const CudaOp &A, const CudaOp &At, int dtype, int64_t m, int64_t n, int64_t m_global,
                  int64_t n_global, const void *v0_dev, const b200_svdl_opts *o, b200_svdl_result *res,
                  double *sigma_host, void *U_dev, int64_t ldu, void *V_dev, int64_t ldv, double *hist_ritz,
                  double *hist_resnorm, int32_t *hist_conv, double *hist_betas, double *B_host) {
  B200_REQUIRE(o->method == 0 || o->method == 1, "Unknown restart method %d (0 = :ritz, 1 = :harmonic; src/svdl.jl:193-200)",
               o->method);
  B200_REQUIRE(!(o->method == 1 && o->dolock), "dolock needs the broken-arrow form of L.B, i.e. method = :ritz "
                                               "(src/svdl.jl:214-221 touches L.B.av)");
  const int nsv = o->nsv > 0 ? o->nsv : 6;                                   // nsv::Int = 6        :158
  const int k = o->k > 0 ? o->k : 2 * nsv;                                   // k::Int = 2nsv       :158
  const int j = o->j > 0 ? o->j : nsv;                                       // j::Int = l          :178
  B200_REQUIRE(k > 1, "svdl: k must exceed 1 (reference src/svdl.jl:183)");
  B200_REQUIRE(k <= kSvdlMaxK, "svdl: k = %d Lanczos vectors exceed the limit %d", k, kSvdlMaxK);
  B200_REQUIRE(nsv <= k && j >= 1 && j < k && nsv <= j + (k - j), "svdl: need nsv <= k and 1 <= j < k (nsv=%d k=%d j=%d)",
               nsv, k, j);
  B200_REQUIRE(k <= std::min(m_global, n_global), "svdl: k = %d exceeds min(size(A)) = %lld", k,
               (long long)std::min(m_global, n_global));
  B200_REQUIRE((!U_dev || ldu >= m) && (!V_dev || ldv >= n), "leading dimensions too small");
  const double sq = 1.4901161193847656e-08;                                  // sqrt(eps()) -- a Float64 literal :158, :179
  const double tol = o->tol < 0 ? sq : o->tol;
  const double reltol = o->reltol < 0 ? sq : o->reltol;
  const int64_t maxiter = o->maxiter < 0 ? std::min(m_global, n_global) : o->maxiter;   // :159
  B200_CUDA(cudaSetDevice(ctx->device));
  CudaBackend be{ctx};
  SvdlOutcome out;
  memset(&out, 0, sizeof(out));
  static_assert(sizeof(int32_t) == sizeof(int), "hist_conv is int32");
  const int st =
      dtype == B200_F64
          ? svdl_run<double>(be, &A, &At, m, n, (const double *)v0_dev, nsv, k, j, tol, reltol, maxiter, o->dolock,
                             sigma_host, (double *)U_dev, ldu, (double *)V_dev, ldv, hist_ritz, hist_resnorm,
                             (int *)hist_conv, hist_betas, B_host, &out, o->method)
          : svdl_run<float>(be, &A, &At, m, n, (const float *)v0_dev, nsv, k, j, tol, reltol, maxiter, o->dolock,
                            sigma_host, (float *)U_dev, ldu, (float *)V_dev, ldv, hist_ritz, hist_resnorm,
                            (int *)hist_conv, hist_betas, B_host, &out, o->method);
  if (st != B200_OK) return st;
  if (res) {
    res->iters = out.iters;
    res->mvps = out.mvps;
    res->mtvps = out.mtvps;
    res->isconverged = out.converged;
    res->k = out.kdim;
    res->beta = out.beta;
    res->tol = tol;
  }
  return B200_OK;
}

}  // namespace

extern "C" {

int b200_svdl(b200_ctx *ctx, const b200_csr *A, const b200_csr *At, const void *v0_dev, const b200_svdl_opts *opts,
              b200_svdl_result *res, double *sigma_host, void *U_dev, int64_t ldu, void *V_dev, int64_t ldv,
              double *hist_ritz, double *hist_resnorm, int32_t *hist_conv, double *hist_betas, double *B_host) {
  B200_TRY(real_only(A, "b200_svdl"));
  B200_TRY(real_only(At, "b200_svdl"));
  B200_REQUIRE(ctx && A && At && v0_dev && opts && sigma_host, "NULL argument");
  B200_REQUIRE(A->ctx == ctx && At->ctx == ctx && At->dtype == A->dtype, "operators must share context and element type");
  if (ctx->world == 1) {
    B200_REQUIRE(At->m_global == A->n_global && At->n_global == A->m_global, "At must be n x m for an m x n operator A");
  } else {
    B200_REQUIRE(is_square(A) && is_square(At) && At->m_local == A->m_local && At->row_begin == A->row_begin,
                 "multi-GPU contexts: A square, At its adjoint with the same row partition");
  }
  return svdl_dispatch(ctx, CudaOp{A, nullptr}, CudaOp{At, nullptr}, A->dtype, A->m_local, At->m_local, A->m_global,
                       A->n_global, v0_dev, opts, res, sigma_host, U_dev, ldu, V_dev, ldv, hist_ritz, hist_resnorm,
                       hist_conv, hist_betas, B_host);
}

int b200_svdl_op(b200_ctx *ctx, const b200_linop *A, const b200_linop *At, const void *v0_dev,
                 const b200_svdl_opts *opts, b200_svdl_result *res, double *sigma_host, void *U_dev, int64_t ldu,
                 void *V_dev, int64_t ldv, double *hist_ritz, double *hist_resnorm, int32_t *hist_conv,
                 double *hist_betas, double *B_host) {
  B200_TRY(real_only(A ? A->dtype : B200_F64, "b200_svdl_op"));
  B200_TRY(real_only(At ? At->dtype : B200_F64, "b200_svdl_op"));
  B200_REQUIRE(ctx && v0_dev && opts && sigma_host, "NULL argument");
  B200_TRY(check_linop(A, "A"));
  B200_TRY(check_linop(At, "At"));
  B200_REQUIRE(At->dtype == A->dtype && At->m_local == A->n_local && At->n_local == A->m_local,
               "At must map the range of A back to its domain");
  return svdl_dispatch(ctx, CudaOp{nullptr, A}, CudaOp{nullptr, At}, A->dtype, A->m_local, A->n_local, A->m_global,
                       A->n_global, v0_dev, opts, res, sigma_host, U_dev, ldu, V_dev, ldv, hist_ritz, hist_resnorm,
                       hist_conv, hist_betas, B_host);
}

}  // extern "C"
