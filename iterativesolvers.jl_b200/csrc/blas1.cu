// blas1.cu -- dot / nrm2 / axpby / scal / copy / fill / Jacobi ldiv! on device vectors.
// All are single-pass streaming kernels (grid = multiple of the SM count, 128-bit accesses when the
// pointers allow it); reductions are deterministic (fixed slot order, last-block finish).
#include "blas1.cuh"

using namespace b200;

namespace {

constexpr int kThreads = 256;

template <typename T>
__global__ void __launch_bounds__(kThreads) k_dot(const T *__restrict__ x, const T *__restrict__ y, int64_t n,
                                                  double *partials, unsigned int *ticket, double *out) {
  __shared__ double smem[kThreads / 32];
  double acc = 0.0;
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads)
    acc += (double)x[i] * (double)y[i];
  acc = block_sum<kThreads>(acc, smem);
  double total;
  if (grid_reduce_finish<kThreads>(acc, partials, ticket, smem, &total)) {
    if (threadIdx.x == 0) out[0] = total;
  }
}

// sum conj(x_i) y_i of complex vectors: the two sums (re, im) reduced like k_dot's one (per-block slots 2b, 2b+1 in a fixed
// order, the last block to arrive sums them with the fixed block tree)
template <typename R>
__global__ void __launch_bounds__(kThreads) k_dotc(const cplx<R> *__restrict__ x, const cplx<R> *__restrict__ y, int64_t n,
                                                   double *partials, unsigned int *ticket, double *out) {
  __shared__ double smem[kThreads / 32];
  __shared__ bool is_last;
  double re = 0.0, im = 0.0;
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    const cplx<R> a = x[i], b = y[i];
    re += (double)a.re * (double)b.re + (double)a.im * (double)b.im;
    im += (double)a.re * (double)b.im - (double)a.im * (double)b.re;
  }
  re = block_sum<kThreads>(re, smem);
  im = block_sum<kThreads>(im, smem);
  if (threadIdx.x == 0) {
    partials[2 * blockIdx.x] = re;
    partials[2 * blockIdx.x + 1] = im;
    __threadfence();
    is_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  double a = 0.0, b = 0.0;
  for (unsigned int i = threadIdx.x; i < gridDim.x; i += kThreads) {
    a += __ldcg(&partials[2 * i]);
    b += __ldcg(&partials[2 * i + 1]);
  }
  a = block_sum<kThreads>(a, smem);
  b = block_sum<kThreads>(b, smem);
  if (threadIdx.x == 0) {
    out[0] = a;
    out[1] = b;
    *ticket = 0u;   // re-arm for the next reduction on this stream
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) k_axpby(double a, const T *__restrict__ x, double b, T *__restrict__ y,
                                                    int64_t n) {
  const T ta = (T)a, tb = (T)b;
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    if (b == 0.0) y[i] = ta * x[i];
    else y[i] = ta * x[i] + tb * y[i];
  }
}
template <typename T>
__global__ void __launch_bounds__(kThreads) k_scal(double a, T *__restrict__ x, int64_t n) {
  const T ta = (T)a;
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads)
    x[i] = ta * x[i];
}
template <typename T>
__global__ void __launch_bounds__(kThreads) k_fill(double a, T *__restrict__ x, int64_t n) {
  const T ta = (T)a;
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads)
    x[i] = ta;
}
template <typename T>
__global__ void __launch_bounds__(kThreads) k_jacobi(const T *__restrict__ d, const T *x, T *y, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads)
    y[i] = x[i] / d[i];
}

int grid1(const b200_ctx *ctx, int64_t n) { return stream_grid(ctx, n, kThreads * 4, 8); }

}  // namespace

namespace b200 {

// device-resident dot: result (local part) in out_dev[0]; multi-GPU callers allreduce afterwards
int dot_dev(b200_ctx *ctx, int64_t n, const void *x, const void *y, int dtype, double *out_dev) {
  const int g = grid1(ctx, n);
  if (dtype == B200_F64)
    k_dot<double><<<g, kThreads, 0, ctx->stream>>>((const double *)x, (const double *)y, n, ctx->red.partials, ctx->red.ticket, out_dev);
  else
    k_dot<float><<<g, kThreads, 0, ctx->stream>>>((const float *)x, (const float *)y, n, ctx->red.partials, ctx->red.ticket, out_dev);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

// device-resident dotc of complex vectors: (re, im) of the local part in out_dev[0..1]
int dotc_dev(b200_ctx *ctx, int64_t n, const void *x, const void *y, int dtype, double *out_dev) {
  const int g = grid1(ctx, n);
  if (dtype == B200_CF64)
    k_dotc<double><<<g, kThreads, 0, ctx->stream>>>((const cplx<double> *)x, (const cplx<double> *)y, n, ctx->red.partials, ctx->red.ticket, out_dev);
  else
    k_dotc<float><<<g, kThreads, 0, ctx->stream>>>((const cplx<float> *)x, (const cplx<float> *)y, n, ctx->red.partials, ctx->red.ticket, out_dev);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

int allreduce_sum_dev(b200_ctx *ctx, double *buf_dev, int count) {
  if (ctx->world > 1) B200_NCCL(ncclAllReduce(buf_dev, buf_dev, count, ncclDouble, ncclSum, ctx->comm, ctx->stream));
  return B200_OK;
}

int read_scalars(b200_ctx *ctx, const double *src_dev, int count, double *dst_host) {
  B200_CUDA(cudaMemcpyAsync(ctx->h_scalars, src_dev, sizeof(double) * count, cudaMemcpyDeviceToHost, ctx->stream));
  B200_CUDA(cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < count; ++i) dst_host[i] = ctx->h_scalars[i];
  return B200_OK;
}

int axpby(b200_ctx *ctx, int64_t n, double a, const void *x, double b, void *y, int dtype) {
  if (n == 0) return B200_OK;
  if (is_complex_dtype(dtype)) {   // real scalars: the 2n real components of a complex vector are updated alike
    n *= 2;
    dtype = dtype == B200_CF64 ? B200_F64 : B200_F32;
  }
  const int g = grid1(ctx, n);
  if (dtype == B200_F64) k_axpby<double><<<g, kThreads, 0, ctx->stream>>>(a, (const double *)x, b, (double *)y, n);
  else k_axpby<float><<<g, kThreads, 0, ctx->stream>>>(a, (const float *)x, b, (float *)y, n);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}
int scal(b200_ctx *ctx, int64_t n, double a, void *x, int dtype) {
  if (n == 0) return B200_OK;
  if (is_complex_dtype(dtype)) {
    n *= 2;
    dtype = dtype == B200_CF64 ? B200_F64 : B200_F32;
  }
  const int g = grid1(ctx, n);
  if (dtype == B200_F64) k_scal<double><<<g, kThreads, 0, ctx->stream>>>(a, (double *)x, n);
  else k_scal<float><<<g, kThreads, 0, ctx->stream>>>(a, (float *)x, n);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}
int fill(b200_ctx *ctx, int64_t n, double a, void *x, int dtype) {
  if (n == 0) return B200_OK;
  const int g = grid1(ctx, n);
  if (dtype == B200_CF64) k_fill<cplx<double>><<<g, kThreads, 0, ctx->stream>>>(a, (cplx<double> *)x, n);   // (a, 0)
  else if (dtype == B200_CF32) k_fill<cplx<float>><<<g, kThreads, 0, ctx->stream>>>(a, (cplx<float> *)x, n);
  else if (dtype == B200_F64) k_fill<double><<<g, kThreads, 0, ctx->stream>>>(a, (double *)x, n);
  else k_fill<float><<<g, kThreads, 0, ctx->stream>>>(a, (float *)x, n);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}
int copy(b200_ctx *ctx, int64_t n, const void *x, void *y, int dtype) {
  if (n == 0 || x == y) return B200_OK;
  B200_CUDA(cudaMemcpyAsync(y, x, dtype_size(dtype) * n, cudaMemcpyDeviceToDevice, ctx->stream));
  return B200_OK;
}
int jacobi_ldiv(b200_ctx *ctx, int64_t n, const void *d, const void *x, void *y, int dtype) {
  if (n == 0) return B200_OK;
  const int g = grid1(ctx, n);
  if (dtype == B200_CF64)   // complex (Smith) division
    k_jacobi<cplx<double>><<<g, kThreads, 0, ctx->stream>>>((const cplx<double> *)d, (const cplx<double> *)x, (cplx<double> *)y, n);
  else if (dtype == B200_CF32)
    k_jacobi<cplx<float>><<<g, kThreads, 0, ctx->stream>>>((const cplx<float> *)d, (const cplx<float> *)x, (cplx<float> *)y, n);
  else if (dtype == B200_F64) k_jacobi<double><<<g, kThreads, 0, ctx->stream>>>((const double *)d, (const double *)x, (double *)y, n);
  else k_jacobi<float><<<g, kThreads, 0, ctx->stream>>>((const float *)d, (const float *)x, (float *)y, n);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

}  // namespace b200

extern "C" {

int b200_dot(b200_ctx *ctx, int64_t n, const void *x_dev, const void *y_dev, int dtype, double *result) {
  B200_REQUIRE(ctx && result && n >= 0 && (n == 0 || (x_dev && y_dev)), "bad arguments");
  if (is_complex_dtype(dtype)) {
    set_error("b200_dot: %s vectors need a conjugating dot product: use b200_dotc", dtype_name(dtype));
    return B200_ERR_UNSUPPORTED;
  }
  B200_TRY(dot_dev(ctx, n, x_dev, y_dev, dtype, ctx->d_scalars));
  B200_TRY(allreduce_sum_dev(ctx, ctx->d_scalars, 1));
  return read_scalars(ctx, ctx->d_scalars, 1, result);
}
int b200_dotc(b200_ctx *ctx, int64_t n, const void *x_dev, const void *y_dev, int dtype, double result[2]) {
  B200_REQUIRE(ctx && result && n >= 0 && (n == 0 || (x_dev && y_dev)), "bad arguments");
  B200_REQUIRE(dtype >= B200_F64 && dtype <= B200_CF32, "bad dtype");
  if (!is_complex_dtype(dtype)) {
    result[1] = 0.0;
    return b200_dot(ctx, n, x_dev, y_dev, dtype, result);
  }
  B200_TRY(dotc_dev(ctx, n, x_dev, y_dev, dtype, ctx->d_scalars));
  B200_TRY(allreduce_sum_dev(ctx, ctx->d_scalars, 2));
  return read_scalars(ctx, ctx->d_scalars, 2, result);
}
int b200_nrm2(b200_ctx *ctx, int64_t n, const void *x_dev, int dtype, double *result) {
  B200_REQUIRE(ctx && result && n >= 0 && (n == 0 || x_dev), "bad arguments");
  if (is_complex_dtype(dtype)) {   // sum |x_i|^2 = the real part of dotc(x, x)
    B200_TRY(dotc_dev(ctx, n, x_dev, x_dev, dtype, ctx->d_scalars));
    B200_TRY(allreduce_sum_dev(ctx, ctx->d_scalars, 1));
    B200_TRY(read_scalars(ctx, ctx->d_scalars, 1, result));
    *result = sqrt(*result);
    return B200_OK;
  }
  B200_TRY(dot_dev(ctx, n, x_dev, x_dev, dtype, ctx->d_scalars));
  B200_TRY(allreduce_sum_dev(ctx, ctx->d_scalars, 1));
  B200_TRY(read_scalars(ctx, ctx->d_scalars, 1, result));
  *result = sqrt(*result);
  return B200_OK;
}
int b200_axpby(b200_ctx *ctx, int64_t n, double a, const void *x_dev, double b, void *y_dev, int dtype) {
  B200_REQUIRE(ctx && n >= 0 && (n == 0 || (x_dev && y_dev)), "bad arguments");
  return axpby(ctx, n, a, x_dev, b, y_dev, dtype);
}
int b200_scal(b200_ctx *ctx, int64_t n, double a, void *x_dev, int dtype) {
  B200_REQUIRE(ctx && n >= 0 && (n == 0 || x_dev), "bad arguments");
  return scal(ctx, n, a, x_dev, dtype);
}
int b200_copy(b200_ctx *ctx, int64_t n, const void *x_dev, void *y_dev, int dtype) {
  B200_REQUIRE(ctx && n >= 0 && (n == 0 || (x_dev && y_dev)), "bad arguments");
  return copy(ctx, n, x_dev, y_dev, dtype);
}
int b200_fill(b200_ctx *ctx, int64_t n, double a, void *x_dev, int dtype) {
  B200_REQUIRE(ctx && n >= 0 && (n == 0 || x_dev), "bad arguments");
  return fill(ctx, n, a, x_dev, dtype);
}
int b200_jacobi_ldiv(b200_ctx *ctx, int64_t n, const void *diag_dev, const void *x_dev, void *y_dev, int dtype) {
  B200_REQUIRE(ctx && n >= 0 && (n == 0 || (diag_dev && x_dev && y_dev)), "bad arguments");
  return jacobi_ldiv(ctx, n, diag_dev, x_dev, y_dev, dtype);
}

}  // extern "C"
