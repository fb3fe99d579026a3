// blas1.cuh -- internal (no-argument-check) vector primitives used by the solver engines.
#pragma once
#include <math.h>

#include "common.cuh"

struct b200_csr;

namespace b200 {
int spmv(b200_ctx *ctx, const b200_csr *A, const void *x, void *y);  // halo exchange + y = A x
int spmv_gated(b200_ctx *ctx, const b200_csr *A, const void *x, void *y, const int *gate, int gate_mask);   // world == 1
int dot_dev(b200_ctx *ctx, int64_t n, const void *x, const void *y, int dtype, double *out_dev);
int dotc_dev(b200_ctx *ctx, int64_t n, const void *x, const void *y, int dtype, double *out_dev);   // complex: 2 doubles
int allreduce_sum_dev(b200_ctx *ctx, double *buf_dev, int count);
int read_scalars(b200_ctx *ctx, const double *src_dev, int count, double *dst_host);
int axpby(b200_ctx *ctx, int64_t n, double a, const void *x, double b, void *y, int dtype);
int scal(b200_ctx *ctx, int64_t n, double a, void *x, int dtype);
int fill(b200_ctx *ctx, int64_t n, double a, void *x, int dtype);
int copy(b200_ctx *ctx, int64_t n, const void *x, void *y, int dtype);
int jacobi_ldiv(b200_ctx *ctx, int64_t n, const void *d, const void *x, void *y, int dtype);

// RAII-less scratch helper for the engines
struct DevBuf {
  void *p = nullptr;
  int alloc(size_t bytes) {
    cudaError_t e = cudaMalloc(&p, bytes ? bytes : 16);
    if (e != cudaSuccess) {
      set_error("cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
      p = nullptr;
      return B200_ERR_ALLOC;
    }
    return B200_OK;
  }
  ~DevBuf() {
    if (p) cudaFree(p);
  }
};
}  // namespace b200
