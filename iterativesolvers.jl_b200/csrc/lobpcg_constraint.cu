// lobpcg_constraint.cu -- C ABI of the LOBPCG Constraint (reference src/lobpcg.jl:144-224; the `C` keyword of
// lobpcg, :829, and the deflation basis the nev > blocksize driver grows batch by batch, :925-962).
#include "lobpcg_constraint.cuh"
#include "lobpcg_constraint_core.h"
#include "pass.cuh"

using namespace b200;

namespace {

template <typename T>
int factor_impl(b200_lobpcg_constraint *c) {
  CudaBackend be{c->ctx};
  c->U.assign((size_t)c->nc * c->nc, 0.0);
  const int st = constraint_factor<T>(be, (const T *)c->Y, c->ld, c->nc, c->n, c->g_dev, c->g_host.data(), c->U.data());
  if (st == -1) {
    set_error("PosDefException: the constraint's Gram matrix Y'Y is not positive definite (reference src/lobpcg.jl:182)");
    return B200_ERR_BREAKDOWN;
  }
  return st;
}

}  // namespace

namespace b200 {

int constraint_apply_block(b200_ctx *ctx, const b200_lobpcg_constraint *c, void *X, int64_t rs, int64_t cs, int bs) {
  B200_REQUIRE(c && c->ctx == ctx, "constraint belongs to another context");
  B200_REQUIRE(bs >= 0 && bs <= kConBlock, "block of %d columns (max %d)", bs, kConBlock);
  CudaBackend be{ctx};
  auto *cm = const_cast<b200_lobpcg_constraint *>(c);   // scratch buffers only
  return c->dtype == B200_F64
             ? constraint_apply<double>(be, (const double *)c->Y, c->ld, c->nc, c->U.data(), (double *)X, rs, cs, bs,
                                        c->n, cm->g_dev, cm->g_host.data())
             : constraint_apply<float>(be, (const float *)c->Y, c->ld, c->nc, c->U.data(), (float *)X, rs, cs, bs, c->n,
                                       cm->g_dev, cm->g_host.data());
}

}  // namespace b200

extern "C" {

int b200_lobpcg_constraint_create(b200_ctx *ctx, int64_t n_local, const void *Y_dev, int64_t ldy, int nc, int capacity,
                                  int dtype, b200_lobpcg_constraint **out) {
  B200_TRY(real_only(dtype, "b200_lobpcg_constraint_create"));
  B200_REQUIRE(ctx && out && n_local >= 0 && nc >= 0 && (nc == 0 || (Y_dev && ldy >= n_local)), "bad arguments");
  B200_REQUIRE(dtype == B200_F64 || dtype == B200_F32, "bad dtype");
  B200_CUDA(cudaSetDevice(ctx->device));
  auto *c = new b200_lobpcg_constraint();
  c->ctx = ctx;
  c->dtype = dtype;
  c->n = n_local;
  c->nc = nc;
  c->cap = std::max(std::max(capacity, nc), 1);
  const size_t vs = dtype_size(dtype);
  c->ld = (int64_t)(align_up(vs * (size_t)std::max<int64_t>(n_local, 1), 256) / vs);
  auto fail = [&](int s) {
    b200_lobpcg_constraint_destroy(c);
    return s;
  };
  if (cudaMalloc(&c->Y, vs * (size_t)c->ld * c->cap) != cudaSuccess ||
      cudaMalloc((void **)&c->g_dev, sizeof(double) * (size_t)c->cap * kConBlock) != cudaSuccess) {
    set_error("constraint: cudaMalloc failed");
    return fail(B200_ERR_ALLOC);
  }
  c->g_host.assign((size_t)c->cap * kConBlock, 0.0);
  if (nc > 0 && n_local > 0) {
    cudaError_t e = cudaMemcpy2DAsync(c->Y, vs * c->ld, Y_dev, vs * ldy, vs * n_local, nc, cudaMemcpyDeviceToDevice,
                                      ctx->stream);
    if (e != cudaSuccess) {
      set_error("constraint: copy of Y failed: %s", cudaGetErrorString(e));
      return fail(B200_ERR_CUDA);
    }
  }
  const int st = dtype == B200_F64 ? factor_impl<double>(c) : factor_impl<float>(c);
  if (st != B200_OK) return fail(st);
  *out = c;
  return B200_OK;
}

int b200_lobpcg_constraint_append(b200_ctx *ctx, b200_lobpcg_constraint *c, const void *X_dev, int64_t ldx, int k) {
  B200_REQUIRE(ctx && c && c->ctx == ctx && k >= 0 && (k == 0 || (X_dev && ldx >= c->n)), "bad arguments");
  B200_REQUIRE(c->nc + k <= c->cap, "constraint capacity %d exceeded (%d + %d columns)", c->cap, c->nc, k);
  if (k == 0) return B200_OK;
  B200_CUDA(cudaSetDevice(ctx->device));
  const size_t vs = dtype_size(c->dtype);
  if (c->n > 0)
    B200_CUDA(cudaMemcpy2DAsync((char *)c->Y + vs * (size_t)c->ld * c->nc, vs * c->ld, X_dev, vs * ldx, vs * c->n, k,
                                cudaMemcpyDeviceToDevice, ctx->stream));
  if (c->BY) {                                          // generalized problem: BY[:, new] = B * X  (update!(c, X, BX) :188-206)
    CudaBackend be{ctx};
    CudaOp bop{nullptr, &c->Bfn};
    for (int j = 0; j < k; ++j)
      B200_TRY(be.apply(&bop, (char *)c->Y + vs * (size_t)c->ld * (c->nc + j), (char *)c->BY + vs * (size_t)c->ld * (c->nc + j)));
  }
  // update! (reference src/lobpcg.jl:188-206): the factor is extended by an identity block -- the appended columns
  // are orthonormal Ritz vectors, orthogonal to the old Y by construction
  const int nc0 = c->nc, nc1 = c->nc + k;
  std::vector<double> U((size_t)nc1 * nc1, 0.0);
  for (int j = 0; j < nc0; ++j)
    for (int i = 0; i <= j; ++i) U[i + (size_t)j * nc1] = c->U[i + (size_t)j * nc0];
  for (int j = nc0; j < nc1; ++j) U[j + (size_t)j * nc1] = 1.0;
  c->U.swap(U);
  c->nc = nc1;
  return B200_OK;
}

int b200_lobpcg_constraint_apply(b200_ctx *ctx, const b200_lobpcg_constraint *c, void *X_dev, int64_t ldx, int bs) {
  B200_REQUIRE(ctx && c && X_dev && ldx >= c->n && bs >= 0, "bad arguments");
  B200_REQUIRE(!c->BY, "b200_lobpcg_constraint_apply: standard-problem constraints only");
  B200_CUDA(cudaSetDevice(ctx->device));
  const size_t vs = dtype_size(c->dtype);
  for (int j0 = 0; j0 < bs; j0 += kConBlock) {         // blocks wider than 16 columns: 16 at a time
    const int w = std::min(kConBlock, bs - j0);
    B200_TRY(constraint_apply_block(ctx, c, (char *)X_dev + vs * (size_t)ldx * j0, 1, ldx, w));
  }
  return B200_OK;
}

int b200_lobpcg_constraint_info(const b200_lobpcg_constraint *c, int *nc, int *capacity) {
  B200_REQUIRE(c, "NULL argument");
  if (nc) *nc = c->nc;
  if (capacity) *capacity = c->cap;
  return B200_OK;
}

int b200_lobpcg_constraint_destroy(b200_lobpcg_constraint *c) {
  if (!c) return B200_OK;
  if (c->ctx) {
    cudaSetDevice(c->ctx->device);
    cudaStreamSynchronize(c->ctx->stream);
  }
  cudaFree(c->Y);
  cudaFree(c->BY);
  cudaFree(c->g_dev);
  delete c;
  return B200_OK;
}

}  // extern "C"
