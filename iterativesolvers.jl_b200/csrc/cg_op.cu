// cg_op.cu -- cg!(x, A, b; Pl, ...) and chebyshev!(x, A, b, lmin, lmax; Pl, ...) for general (callback) operators and
// preconditioners, and the power method powm! / invpowm!: the fused-pass engines of cg_core.h / chebyshev_core.h /
// powm_core.h on the CUDA backend.  b200_csr operators with Identity / Jacobi take the specialised engine of cg.cu.
#include "linop.cuh"
#include "cg_core.h"
#include "chebyshev_core.h"
#include "powm_core.h"

using namespace b200;

namespace b200 {

// cg! on a CSR or callback operator (cg_core.h).  Pl: the preconditioner callback given as an argument, or NULL: then
// opts->Pl decides (Identity, Jacobi, or B200_PREC_CALLBACK with the descriptor in opts->Pl.diag).
int cg_general(b200_ctx *ctx, const CudaOp &A, int dtype, int64_t n, int64_t n_global, const b200_linop *Pl, void *x_dev,
               const void *b_dev, const b200_cg_opts *opts, b200_result *res, double *resnorm_host, int64_t resnorm_cap) {
  if (!Pl && opts->Pl.kind == B200_PREC_CALLBACK) Pl = (const b200_linop *)opts->Pl.diag;
  if (is_complex_dtype(dtype) && ctx->world > 1) {
    set_error("cg!: %s operators are single-GPU in this version", dtype_name(dtype));
    return B200_ERR_UNSUPPORTED;
  }
  if (Pl) {
    B200_TRY(check_linop_complex(Pl, "Pl"));
    B200_REQUIRE(Pl->dtype == dtype && Pl->m_local == n && Pl->n_local == n,
                 "Pl must act on vectors of the operator's local length");
  } else {
    B200_REQUIRE(opts->Pl.kind == B200_PREC_IDENTITY || (opts->Pl.kind == B200_PREC_JACOBI && opts->Pl.diag),
                 "unsupported preconditioner");
  }
  B200_REQUIRE(!opts->fixed_iterations && !opts->variant, "fixed_iterations / variant are not available on this path");
  B200_CUDA(cudaSetDevice(ctx->device));
  CudaBackend be{ctx};
  CudaOp p{nullptr, Pl};
  const void *diag = (!Pl && opts->Pl.kind == B200_PREC_JACOBI) ? opts->Pl.diag : nullptr;
  CgpOutcome o;
  memset(&o, 0, sizeof(o));
  int st;
  if (dtype == B200_CF64)
    st = cgp_run<cplx<double>>(be, &A, Pl ? &p : nullptr, (const cplx<double> *)diag, n, n_global, (cplx<double> *)x_dev,
                               (const cplx<double> *)b_dev, opts->abstol, opts->reltol, opts->maxiter, opts->initially_zero,
                               opts->check_every, resnorm_cap, resnorm_host, &o);
  else if (dtype == B200_CF32)
    st = cgp_run<cplx<float>>(be, &A, Pl ? &p : nullptr, (const cplx<float> *)diag, n, n_global, (cplx<float> *)x_dev,
                              (const cplx<float> *)b_dev, opts->abstol, opts->reltol, opts->maxiter, opts->initially_zero,
                              opts->check_every, resnorm_cap, resnorm_host, &o);
  else
    st = dtype == B200_F64
                     ? cgp_run<double>(be, &A, Pl ? &p : nullptr, (const double *)diag, n, n_global, (double *)x_dev,
                                       (const double *)b_dev, opts->abstol, opts->reltol, opts->maxiter,
                                       opts->initially_zero, opts->check_every, resnorm_cap, resnorm_host, &o)
                     : cgp_run<float>(be, &A, Pl ? &p : nullptr, (const float *)diag, n, n_global, (float *)x_dev,
                                      (const float *)b_dev, opts->abstol, opts->reltol, opts->maxiter,
                                      opts->initially_zero, opts->check_every, resnorm_cap, resnorm_host, &o);
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

// chebyshev! on a CSR or callback operator with Identity / Jacobi / callback preconditioner (chebyshev_core.h)
int chebyshev_general(b200_ctx *ctx, const CudaOp &A, int dtype, int64_t n, int64_t n_global, void *x_dev,
                      const void *b_dev, double lmin, double lmax, const b200_cg_opts *opts, b200_result *res,
                      double *resnorm_host, int64_t resnorm_cap) {
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
  B200_REQUIRE(!opts->fixed_iterations && !opts->variant, "fixed_iterations / variant are not available on this path");
  B200_CUDA(cudaSetDevice(ctx->device));
  CudaBackend be{ctx};
  CudaOp pl{nullptr, plf};
  ChebOutcome o;
  memset(&o, 0, sizeof(o));
  const int st =
      dtype == B200_F64
          ? chebyshev_run<double>(be, &A, plf ? &pl : nullptr, (const double *)diag, n, n_global, (double *)x_dev,
                                  (const double *)b_dev, lmin, lmax, opts->abstol, opts->reltol, opts->maxiter,
                                  opts->initially_zero, opts->check_every, resnorm_cap, resnorm_host, &o)
          : chebyshev_run<float>(be, &A, plf ? &pl : nullptr, (const float *)diag, n, n_global, (float *)x_dev,
                                 (const float *)b_dev, lmin, lmax, opts->abstol, opts->reltol, opts->maxiter,
                                 opts->initially_zero, opts->check_every, resnorm_cap, resnorm_host, &o);
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

int b200_chebyshev_solve_op(b200_ctx *ctx, const b200_linop *A, void *x_dev, const void *b_dev, double lambda_min,
                            double lambda_max, const b200_cg_opts *opts, b200_result *res, double *resnorm_host,
                            int64_t resnorm_cap) {
  B200_TRY(real_only(A ? A->dtype : B200_F64, "b200_chebyshev_solve_op"));
  B200_REQUIRE(ctx && x_dev && b_dev && opts, "NULL argument");
  B200_TRY(check_linop(A, "A"));
  B200_REQUIRE(A->m_global == A->n_global && A->m_local == A->n_local, "chebyshev! needs a square operator");
  return chebyshev_general(ctx, CudaOp{nullptr, A}, A->dtype, A->m_local, A->n_global, x_dev, b_dev, lambda_min,
                           lambda_max, opts, res, resnorm_host, resnorm_cap);
}

int b200_cg_solve_op(b200_ctx *ctx, const b200_linop *A, const b200_linop *Pl, void *x_dev, const void *b_dev,
                     const b200_cg_opts *opts, b200_result *res, double *resnorm_host, int64_t resnorm_cap) {
  B200_REQUIRE(ctx && x_dev && b_dev && opts, "NULL argument");
  B200_TRY(check_linop_complex(A, "A"));
  B200_REQUIRE(A->m_global == A->n_global && A->m_local == A->n_local, "cg! needs a square operator");
  return cg_general(ctx, CudaOp{nullptr, A}, A->dtype, A->m_local, A->n_global, Pl, x_dev, b_dev, opts, res, resnorm_host,
                    resnorm_cap);
}

// powm!(B, x; shift, inverse, tol, maxiter) / invpowm! (reference src/simple.jl:118-151, :186): exactly one of A (device CSR)
// and Aop (callback: e.g. the action of inv(A - shift I) for inverse iteration) is non-NULL.
int b200_powm(b200_ctx *ctx, const b200_csr *A, const b200_linop *Aop, void *x_dev, const b200_powm_opts *opts,
              b200_result *res, double *lambda_out, double *resnorm_host, int64_t resnorm_cap) {
  B200_TRY(real_only(A, "b200_powm"));
  B200_TRY(real_only(Aop ? Aop->dtype : B200_F64, "b200_powm"));
  B200_REQUIRE(ctx && x_dev && opts, "NULL argument");
  B200_REQUIRE((A != nullptr) != (Aop != nullptr), "exactly one of the CSR operator and the callback operator must be given");
  CudaOp op;
  int dtype;
  int64_t n, n_global;
  if (A) {
    B200_REQUIRE(A->ctx == ctx, "operator belongs to another context");
    B200_REQUIRE(is_square(A), "powm! needs a square operator");
    op = CudaOp{A, nullptr};
    dtype = A->dtype;
    n = A->m_local;
    n_global = A->n_global;
  } else {
    B200_TRY(check_linop(Aop, "B"));
    B200_REQUIRE(Aop->m_global == Aop->n_global && Aop->m_local == Aop->n_local, "powm! needs a square operator");
    op = CudaOp{nullptr, Aop};
    dtype = Aop->dtype;
    n = Aop->m_local;
    n_global = Aop->n_global;
  }
  B200_CUDA(cudaSetDevice(ctx->device));
  CudaBackend be{ctx};
  PowmOutcome o;
  memset(&o, 0, sizeof(o));
  const int st = dtype == B200_F64 ? powm_run<double>(be, &op, n, n_global, (double *)x_dev, opts->tol, opts->maxiter,
                                                      opts->check_every, resnorm_cap, resnorm_host, &o)
                                   : powm_run<float>(be, &op, n, n_global, (float *)x_dev, opts->tol, opts->maxiter,
                                                     opts->check_every, resnorm_cap, resnorm_host, &o);
  if (st != B200_OK) return st;
  if (lambda_out) *lambda_out = opts->shift + (opts->inverse ? 1.0 / o.theta : o.theta);   // transform_eigenvalue :51
  if (res) {
    res->iters = o.iters;
    res->mvps = o.iters;                 // nextiter!(history, mvps = 1) :133
    res->isconverged = o.converged;
    res->status = o.breakdown ? B200_ERR_BREAKDOWN : 0;
    res->tol = o.tol;
    res->residual = o.residual;
    res->n_resnorm = o.n_hist;
  }
  return B200_OK;
}

}  // extern "C"
