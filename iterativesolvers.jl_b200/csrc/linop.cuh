// linop.cuh -- shared helpers of the *_op (callback operator) entry points.
#pragma once
#include "pass.cuh"

namespace b200 {
int check_linop(const b200_linop *A, const char *what);           // qmr.cu; real element types only
int check_linop_complex(const b200_linop *A, const char *what);   // qmr.cu; also ComplexF64 / ComplexF32 (cg_op, gmres_op)
// the general (fused-pass) engines behind both the *_solve_op entry points and the b200_csr entry points when one of
// their preconditioners is a callback
int gmres_general(b200_ctx *ctx, const CudaOp &A, int dtype, int64_t n, int64_t n_global, void *x_dev, const void *b_dev,
                  const b200_gmres_opts *opts, b200_result *res, double *resnorm_host, int64_t resnorm_cap);   // gmres_op.cu
int bicgstabl_general(b200_ctx *ctx, const CudaOp &A, int dtype, int64_t n, int64_t n_global, void *x_dev,
                      const void *b_dev, const b200_bicgstabl_opts *opts, b200_result *res, double *resnorm_host,
                      int64_t resnorm_cap);                                                                     // minres_bicgstabl_op.cu
int chebyshev_general(b200_ctx *ctx, const CudaOp &A, int dtype, int64_t n, int64_t n_global, void *x_dev,
                      const void *b_dev, double lmin, double lmax, const b200_cg_opts *opts, b200_result *res,
                      double *resnorm_host, int64_t resnorm_cap);                                               // cg_op.cu
int cg_general(b200_ctx *ctx, const CudaOp &A, int dtype, int64_t n, int64_t n_global, const b200_linop *Pl, void *x_dev,
               const void *b_dev, const b200_cg_opts *opts, b200_result *res, double *resnorm_host, int64_t resnorm_cap);   // cg_op.cu
}
