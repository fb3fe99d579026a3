// lobpcg_general.cu -- the general form of lobpcg on the GPU (lobpcg_general_core.h on the CUDA backend): generalized
// problem A x = lambda B x, callback operators / preconditioner, constraint in the B inner product.  The standard
// problem on a b200_csr with Identity / Jacobi stays on the tuned engine of lobpcg.cu.
#include "linop.cuh"
#include "lobpcg_constraint.cuh"
#include "lobpcg_general_core.h"

using namespace b200;

namespace {

int csr_apply_thunk(void *user, const void *x, void *y, void *) {
  const b200_csr *A = (const b200_csr *)user;
  return b200::spmv(A->ctx, A, x, y);
}

}  // namespace

extern "C" {

int b200_csr_as_linop(const b200_csr *A, b200_linop *out) {
  B200_REQUIRE(A && out, "NULL argument");
  out->apply = csr_apply_thunk;
  out->user = (void *)A;
  out->m_local = A->m_local;
  out->n_local = A->ctx->world == 1 ? A->n_global : A->m_local;
  out->n_global = A->n_global;
  out->m_global = A->m_global;
  out->dtype = A->dtype;
  out->reserved = 0;
  return B200_OK;
}

int b200_lobpcg_solve_op(b200_ctx *ctx, const b200_linop *A, const b200_linop *B, void *X_dev, int64_t ldx,
                         const b200_lobpcg_opts *opts, const b200_lobpcg_constraint *C, b200_lobpcg_result *res,
                         double *lambda_host, double *resnorm_host) {
  B200_TRY(real_only(A ? A->dtype : B200_F64, "b200_lobpcg_solve_op"));
  B200_TRY(real_only(B ? B->dtype : B200_F64, "b200_lobpcg_solve_op"));
  B200_REQUIRE(ctx && X_dev && opts, "NULL argument");
  B200_TRY(check_linop(A, "A"));
  B200_REQUIRE(A->m_global == A->n_global && A->m_local == A->n_local, "lobpcg needs a square operator");
  if (B) {
    B200_TRY(check_linop(B, "B"));
    B200_REQUIRE(B->dtype == A->dtype && B->m_local == A->m_local && B->n_local == A->n_local && B->n_global == A->n_global,
                 "B must have the shape, partition and element type of A");
  }
  const int64_t n = A->m_local;
  const int sizeX = opts->blocksize;
  B200_REQUIRE(sizeX >= 1 && sizeX <= kConBlock, "lobpcg: block size %d not in 1..%d", sizeX, kConBlock);
  B200_REQUIRE(ldx >= n, "lobpcg: leading dimension of X too small");
  B200_REQUIRE(sizeX <= A->n_global, "X column dimension exceeds the row dimension");               // src/lobpcg.jl:833
  B200_REQUIRE(3 * (int64_t)sizeX <= A->n_global, "The LOBPCG algorithms is not stable to use when the matrix size is "
               "less than 3 times the block size. Please use a dense solver instead.");             // :834
  const b200_linop *pfn = nullptr;
  const void *jac = nullptr;
  if (opts->P.kind == B200_PREC_JACOBI) {
    B200_REQUIRE(opts->P.diag, "Jacobi preconditioner without a diagonal");
    jac = opts->P.diag;
  } else if (opts->P.kind == B200_PREC_CALLBACK) {
    pfn = (const b200_linop *)opts->P.diag;
    B200_TRY(check_linop(pfn, "P"));
    B200_REQUIRE(pfn->dtype == A->dtype && pfn->m_local == n && pfn->n_local == n, "P must act on the operator's vectors");
  } else {
    B200_REQUIRE(opts->P.kind == B200_PREC_IDENTITY, "unsupported preconditioner");
  }
  if (C) {
    B200_REQUIRE(C->ctx == ctx && C->dtype == A->dtype && C->n == n, "the constraint does not match the operator");
    B200_REQUIRE((C->BY != nullptr) == (B != nullptr) || (C->nc == 0 && !C->BY),
                 "generalized problems need a constraint built with b200_lobpcg_constraint_create_b (and vice versa)");
  }
  B200_CUDA(cudaSetDevice(ctx->device));
  CudaBackend be{ctx};
  CudaOp a{nullptr, A}, b{nullptr, B}, p{nullptr, pfn};
  LobpcgGenOutcome o;
  memset(&o, 0, sizeof(o));
  const int nc = C ? C->nc : 0;
  const void *Y = C ? C->Y : nullptr;
  const void *BY = C ? (C->BY ? C->BY : C->Y) : nullptr;
  const int64_t ldy = C ? C->ld : 0;
  const double *U = C ? C->U.data() : nullptr;
  const int st =
      A->dtype == B200_F64
          ? lobpcg_general_run<double>(be, &a, B ? &b : nullptr, pfn ? &p : nullptr, (const double *)jac, (const double *)Y,
                                       (const double *)BY, ldy, nc, U, (double *)X_dev, ldx, sizeX, n, opts->largest,
                                       opts->tol, opts->maxiter, opts->fixed_iterations, lambda_host, resnorm_host, &o,
                                       opts->trace_resnorm, opts->trace_ritz, opts->trace_cap)
          : lobpcg_general_run<float>(be, &a, B ? &b : nullptr, pfn ? &p : nullptr, (const float *)jac, (const float *)Y,
                                      (const float *)BY, ldy, nc, U, (float *)X_dev, ldx, sizeX, n, opts->largest,
                                      opts->tol, opts->maxiter, opts->fixed_iterations, lambda_host, resnorm_host, &o,
                                      opts->trace_resnorm, opts->trace_ritz, opts->trace_cap);
  if (st != B200_OK) return st;
  if (res) {
    res->iterations = o.iterations;
    res->converged = o.converged;
    res->status = o.status ? B200_ERR_BREAKDOWN : 0;
  }
  if (o.status) {
    set_error(o.status == 1 ? "PosDefException: CholQR Gram matrix is not positive definite (reference src/lobpcg.jl:380)"
                            : "PosDefException in the Rayleigh-Ritz problem (gramB not positive definite)");
    return B200_ERR_BREAKDOWN;
  }
  return B200_OK;
}

// Constraint(Y, B, X) for the generalized problem (reference src/lobpcg.jl:161-186): BY = B*Y is kept next to Y and
// the factor is that of Y' BY.
int b200_lobpcg_constraint_create_b(b200_ctx *ctx, const b200_linop *B, int64_t n_local, const void *Y_dev, int64_t ldy,
                                    int nc, int capacity, int dtype, b200_lobpcg_constraint **out) {
  B200_TRY(real_only(B ? B->dtype : B200_F64, "b200_lobpcg_constraint_create_b"));
  B200_TRY(real_only(dtype, "b200_lobpcg_constraint_create_b"));
  B200_REQUIRE(ctx && out && B && nc >= 0 && (nc == 0 || (Y_dev && ldy >= n_local)), "bad arguments");
  B200_TRY(check_linop(B, "B"));
  B200_REQUIRE(B->dtype == dtype && B->m_local == n_local && B->n_local == n_local, "B does not match the constraint");
  b200_lobpcg_constraint *c = nullptr;
  B200_TRY(b200_lobpcg_constraint_create(ctx, n_local, nullptr, n_local, 0, std::max(std::max(nc, capacity), 1), dtype,
                                         &c));                                                  // storage only
  c->Bfn = *B;
  const size_t vs = dtype_size(dtype);
  auto fail = [&](int s) {
    b200_lobpcg_constraint_destroy(c);
    return s;
  };
  if (cudaMalloc(&c->BY, vs * (size_t)c->ld * c->cap) != cudaSuccess) {
    set_error("constraint: cudaMalloc failed");
    return fail(B200_ERR_ALLOC);
  }
  if (n_local > 0 && nc > 0 &&
      cudaMemcpy2DAsync(c->Y, vs * c->ld, Y_dev, vs * ldy, vs * n_local, nc, cudaMemcpyDeviceToDevice, ctx->stream) !=
          cudaSuccess) {
    set_error("constraint: copy of Y failed");
    return fail(B200_ERR_CUDA);
  }
  c->nc = nc;
  CudaBackend be{ctx};
  CudaOp bop{nullptr, B};
  for (int j = 0; j < nc; ++j) {                                                                // mul!(BY, B, Y) :167
    const int st = be.apply(&bop, (char *)c->Y + vs * (size_t)c->ld * j, (char *)c->BY + vs * (size_t)c->ld * j);
    if (st) return fail(st);
  }
  c->U.assign((size_t)nc * nc, 0.0);
  for (int c0 = 0; c0 < nc; c0 += kConBlock) {                                                  // gramYBY = Y' BY :178
    const int bs = std::min(kConBlock, nc - c0);
    const int st = dtype == B200_F64
                       ? constraint_gram<double>(be, (const double *)c->Y, c->ld, nc, (const double *)c->BY + c->ld * c0, 1,
                                                 c->ld, bs, n_local, c->g_dev, c->g_host.data())
                       : constraint_gram<float>(be, (const float *)c->Y, c->ld, nc, (const float *)c->BY + c->ld * c0, 1,
                                                c->ld, bs, n_local, c->g_dev, c->g_host.data());
    if (st) return fail(st);
    for (int k = 0; k < nc; ++k)
      for (int j = 0; j < bs; ++j) c->U[k + (size_t)(c0 + j) * nc] = c->g_host[(size_t)k * kConBlock + j];
  }
  if (con_cholesky_upper(c->U.data(), nc)) {
    set_error("PosDefException: the constraint's Gram matrix Y'BY is not positive definite (reference src/lobpcg.jl:182)");
    return fail(B200_ERR_BREAKDOWN);
  }
  *out = c;
  return B200_OK;
}

}  // extern "C"
