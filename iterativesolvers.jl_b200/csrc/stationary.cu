// stationary.cu -- jacobi!, gauss_seidel!, sor!, ssor! on a device CSR operator (reference src/stationary_sparse.jl): the
// level-scheduled sweeps of stationary_core.h on the CUDA backend.  The host analysis of the sparsity pattern (diagonal
// positions, dependency levels: the reference's DiagonalIndices and the order its column sweeps impose) is done on the
// first call and kept with the operator; a call then runs exactly `maxiter` iterations, one kernel per dependency level.
#include <memory>

#include "pass.cuh"
#include "stationary_core.h"

using namespace b200;

namespace {

struct DevInts {
  int *p = nullptr;
  ~DevInts() { if (p) cudaFree(p); }
  int upload(const std::vector<int> &h, cudaStream_t st) {
    if (h.empty()) return B200_OK;
    if (cudaMalloc((void **)&p, sizeof(int) * h.size()) != cudaSuccess) {
      set_error("stationary: cudaMalloc failed");
      return B200_ERR_ALLOC;
    }
    B200_CUDA(cudaMemcpyAsync(p, h.data(), sizeof(int) * h.size(), cudaMemcpyHostToDevice, st));
    return B200_OK;
  }
};

// the analysis of one operator (what the reference's DiagonalIndices and the order of its column sweeps encode), built on
// first use and kept with the operator: level sets of both sweep directions, on the host and on the device
struct StPlan {
  StLevels lv;
  DevInts dpos, rows_f, rows_b;
  int64_t singular = 0;            // row + 1 of a zero / missing diagonal entry
};
void st_plan_free(void *p) { delete (StPlan *)p; }

template <typename T>
int stationary_plan(b200_ctx *ctx, const b200_csr *A, const StPlan **out) {
  if (A->st_plan) {
    *out = (const StPlan *)A->st_plan;
    return B200_OK;
  }
  const int64_t n = A->m_local;
  std::vector<int> rowptr((size_t)n + 1), colind((size_t)A->nnz);
  std::vector<T> vals((size_t)A->nnz);
  B200_CUDA(cudaMemcpyAsync(rowptr.data(), A->rowptr, sizeof(int) * (size_t)(n + 1), cudaMemcpyDeviceToHost, ctx->stream));
  B200_CUDA(cudaMemcpyAsync(colind.data(), A->colind, sizeof(int) * (size_t)A->nnz, cudaMemcpyDeviceToHost, ctx->stream));
  B200_CUDA(cudaMemcpyAsync(vals.data(), A->vals, sizeof(T) * (size_t)A->nnz, cudaMemcpyDeviceToHost, ctx->stream));
  B200_CUDA(cudaStreamSynchronize(ctx->stream));
  for (int64_t i = 0; i < n; ++i)
    for (int p = rowptr[(size_t)i] + 1; p < rowptr[(size_t)i + 1]; ++p)
      B200_REQUIRE(colind[(size_t)p - 1] < colind[(size_t)p], "stationary methods need rows with ascending column indices "
                   "(row %lld)", (long long)i);
  std::unique_ptr<StPlan> plan(new StPlan());
  plan->singular = stationary_analyse<T, int>(n, rowptr.data(), colind.data(), vals.data(), true, true, &plan->lv);
  if (!plan->singular) {
    B200_TRY(plan->dpos.upload(plan->lv.dpos, ctx->stream));
    B200_TRY(plan->rows_f.upload(plan->lv.rows_f, ctx->stream));
    B200_TRY(plan->rows_b.upload(plan->lv.rows_b, ctx->stream));
    B200_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  A->st_plan = plan.release();
  A->st_plan_free = st_plan_free;
  *out = (const StPlan *)A->st_plan;
  return B200_OK;
}

template <typename T>
int stationary_impl(b200_ctx *ctx, const b200_csr *A, T *x, const T *b, int method, double omega, int64_t maxiter) {
  const StPlan *plan = nullptr;
  B200_TRY(stationary_plan<T>(ctx, A, &plan));
  if (plan->singular) {
    set_error("SingularException(%lld): zero or missing diagonal entry (reference src/stationary_sparse.jl:19)",
              (long long)plan->singular);
    return B200_ERR_BREAKDOWN;
  }
  CudaBackend be{ctx};
  const CsrView<T, int> view{A->m_local, A->rowptr, A->colind, (const T *)A->vals};
  return stationary_run<T, int>(be, view, plan->lv, plan->dpos.p, plan->rows_f.p, plan->rows_b.p, x, b, method, omega,
                                maxiter);
}

}  // namespace

extern "C" {

int b200_stationary(b200_ctx *ctx, const b200_csr *A, void *x_dev, const void *b_dev, int method, double omega,
                    int64_t maxiter) {
  B200_TRY(real_only(A, "b200_stationary"));
  B200_REQUIRE(ctx && A && x_dev && b_dev, "NULL argument");
  B200_REQUIRE(A->ctx == ctx, "operator belongs to another context");
  B200_REQUIRE(ctx->world == 1, "the stationary methods sweep the whole matrix in order: single-GPU contexts only");
  B200_REQUIRE(is_square(A), "this solver needs a square operator");
  if (A->rowptr64) {
    set_error("b200_stationary: the sweeps' analysis holds int32 row offsets; an operator with 8-byte row offsets "
              "(nnz >= 2^31, or built with \"rowptr64\" = 1) is not supported");
    return B200_ERR_UNSUPPORTED;
  }
  const int base = method & ~B200_STATIONARY_DENSE_ARITHMETIC;
  B200_REQUIRE(base >= B200_STATIONARY_JACOBI && base <= B200_STATIONARY_SSOR, "unknown stationary method %d", method);
  static_assert(B200_STATIONARY_JACOBI == ST_JACOBI && B200_STATIONARY_GAUSS_SEIDEL == ST_GAUSS_SEIDEL &&
                B200_STATIONARY_SOR == ST_SOR && B200_STATIONARY_SSOR == ST_SSOR &&
                B200_STATIONARY_DENSE_ARITHMETIC == ST_DENSE_ARITHMETIC, "method codes");
  B200_CUDA(cudaSetDevice(ctx->device));
  return A->dtype == B200_F64 ? stationary_impl<double>(ctx, A, (double *)x_dev, (const double *)b_dev, method, omega, maxiter)
                              : stationary_impl<float>(ctx, A, (float *)x_dev, (const float *)b_dev, method, omega, maxiter);
}

}  // extern "C"
