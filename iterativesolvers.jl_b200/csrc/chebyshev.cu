// chebyshev.cu -- chebyshev!(x, A, b, lmin, lmax; ...) of reference src/chebyshev.jl:131-160 (iterate :29-57,
// chebyshev_iterable! :59-92).  SURVEY.md section 8(f) item 2: the same kernels as CG with ONE global
// reduction per step (the residual norm) -- alpha and beta depend only on the iteration number and the
// spectral bounds, so the host passes them as kernel arguments.
//
// The reference's recurrence is reproduced literally, including its two oddities (src/chebyshev.jl:39-46):
// the branch `iteration == 1` is taken on the SECOND call (iteration starts at 0), and the general branch
// computes `u .= c .+ beta .* c` (c, not u).
//   K1  c = Pl \ r ; u = c  or  u = c + beta*c          (Identity: c = r is not materialised)
//   K2  c = A*u                                          (TMA-streamed SpMV, spmv.cu)
//   K3  x += alpha*u ; r -= alpha*c ; ||r||^2 -> residual, history, done
#include "blas1.cuh"
#include "csr.cuh"
#include "linop.cuh"

using namespace b200;

namespace {

constexpr int kThreads = 256;

struct ChebScal {
  double resnorm, tol, abstol, reltol, sum;
  long long iter, maxiter, hist_cap;
  int done, breakdown;
};

__device__ __forceinline__ void cheb_after_norm(ChebScal *s, double rr, double *hist, bool init) {
  const double res = sqrt(rr);
  s->resnorm = res;
  if (!(res == res)) s->breakdown = 1;
  if (init) {
    s->tol = fmax(s->reltol * res, s->abstol);                              // :86-87
    s->iter = 0;
  } else {
    if (hist && s->iter < s->hist_cap) hist[s->iter] = res;
    s->iter += 1;
  }
  s->done = (s->iter >= s->maxiter) || (res <= s->tol) || s->breakdown;     // done() :27
}

__global__ void k_cheb_scalar(ChebScal *s, double *hist, int init) {
  if (!init && s->done) return;
  cheb_after_norm(s, s->sum, hist, init != 0);
}

// init: r = b - c (or b); u = 0; ||r||^2        (:73-86)
template <typename T>
__global__ void __launch_bounds__(kThreads) k_cheb_init(const T *__restrict__ b, const T *__restrict__ c, int has_c,
                                                        T *__restrict__ r, T *__restrict__ u, int64_t n,
                                                        ChebScal *s, double *partials, unsigned int *ticket,
                                                        int single) {
  __shared__ double smem[kThreads / 32];
  double acc = 0.0;
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    T ri = b[i];
    if (has_c) ri = ri - c[i];
    r[i] = ri;
    u[i] = (T)0;
    acc += (double)ri * (double)ri;
  }
  acc = block_sum<kThreads>(acc, smem);
  double total;
  if (grid_reduce_finish<kThreads>(acc, partials, ticket, smem, &total) && threadIdx.x == 0) {
    if (single) cheb_after_norm(s, total, nullptr, true);
    else s->sum = total;
  }
}

// K1: c = Pl \ r (Jacobi or Identity) ; u = c (copy) or u = c + beta*c      (:37-46)
template <typename T>
__global__ void __launch_bounds__(kThreads) k_cheb_update_u(const T *__restrict__ r, const T *__restrict__ d,
                                                            T *__restrict__ u, int64_t n, double beta, int copy,
                                                            const ChebScal *__restrict__ s) {
  if (s->done) return;
  const T tb = (T)beta;
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    T ci = r[i];
    if (d) ci = ci / d[i];
    u[i] = copy ? ci : ci + tb * ci;
  }
}

// K3: x += alpha*u ; r -= alpha*c ; ||r||^2      (:51-54)
template <typename T>
__global__ void __launch_bounds__(kThreads) k_cheb_update_xr(T *__restrict__ x, T *__restrict__ r,
                                                             const T *__restrict__ u, const T *__restrict__ c,
                                                             int64_t n, double alpha, ChebScal *s, double *hist,
                                                             double *partials, unsigned int *ticket, int single) {
  if (s->done) return;
  __shared__ double smem[kThreads / 32];
  const T ta = (T)alpha;
  double acc = 0.0;
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    x[i] = x[i] + ta * u[i];
    const T ri = r[i] - ta * c[i];
    r[i] = ri;
    acc += (double)ri * (double)ri;
  }
  acc = block_sum<kThreads>(acc, smem);
  double total;
  if (grid_reduce_finish<kThreads>(acc, partials, ticket, smem, &total) && threadIdx.x == 0) {
    if (single) cheb_after_norm(s, total, hist, false);
    else s->sum = total;
  }
}

template <typename T>
int chebyshev_impl(b200_ctx *ctx, const b200_csr *A, T *x, const T *b, double lmin, double lmax,
                   const b200_cg_opts *o, b200_result *res, double *resnorm_host, int64_t resnorm_cap) {
  cudaStream_t st = ctx->stream;
  const int64_t n = A->m_local;
  const double eps = sizeof(T) == 8 ? 2.220446049250313e-16 : 1.1920928955078125e-07;
  const double reltol = o->reltol < 0 ? sqrt(eps) : o->reltol;
  const int64_t maxiter = o->maxiter < 0 ? A->n_global : o->maxiter;
  const int64_t hist_cap = resnorm_host ? std::min<int64_t>(resnorm_cap, maxiter) : 0;
  const T *jac = o->Pl.kind == B200_PREC_JACOBI ? (const T *)o->Pl.diag : nullptr;
  const int single = ctx->world == 1;
  const double l_avg = (lmax + lmin) / 2, l_diff = (lmax - lmin) / 2;       // :65-66

  const size_t vec_bytes = align_up(sizeof(T) * (size_t)std::max<int64_t>(n, 1), 256);
  const size_t hist_bytes = align_up(sizeof(double) * (size_t)std::max<int64_t>(hist_cap, 1), 256);
  void *ws = nullptr;
  B200_TRY(ws_get(ctx, 3 * vec_bytes + 256 + hist_bytes, &ws));
  char *p = (char *)ws;
  T *u = (T *)p; p += vec_bytes;
  T *r = (T *)p; p += vec_bytes;
  T *c = (T *)p; p += vec_bytes;
  ChebScal *s = (ChebScal *)p; p += 256;
  double *hist = hist_cap ? (double *)p : nullptr;
  ChebScal h;
  memset(&h, 0, sizeof(h));
  h.abstol = o->abstol;
  h.reltol = reltol;
  h.maxiter = maxiter;
  h.hist_cap = hist_cap;
  B200_CUDA(cudaMemcpyAsync(s, &h, sizeof(h), cudaMemcpyHostToDevice, st));
  const int gv = stream_grid(ctx, n, kThreads * 2, 8);

  auto after = [&](int init) -> int {
    if (single) return B200_OK;
    B200_TRY(allreduce_sum_dev(ctx, &s->sum, 1));
    k_cheb_scalar<<<1, 1, 0, st>>>(s, hist, init);
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
  };

  int64_t mv_products = 0;
  if (!o->initially_zero) {                                                  // :78-82
    mv_products = 1;
    B200_TRY(spmv(ctx, A, x, c));
  }
  k_cheb_init<T><<<gv, kThreads, 0, st>>>(b, c, o->initially_zero ? 0 : 1, r, u, n, s, ctx->red.partials,
                                           ctx->red.ticket, single);
  B200_LAUNCH_CHECK(ctx);
  B200_TRY(after(1));

  double alpha = 0.0;                                                        // zero(real(T)) :89
  int64_t iteration = 0;
  int *h_done = ctx->h_flags;
  const int check_every = o->check_every > 0 ? o->check_every : 32;
  for (;;) {
    B200_CUDA(cudaMemcpyAsync(h_done, &s->done, sizeof(int), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    if (*h_done || iteration >= maxiter) break;
    const int64_t batch = std::min<int64_t>(check_every, maxiter - iteration);
    for (int64_t q = 0; q < batch; ++q, ++iteration) {
      double beta = 0.0;
      int copy = 0;
      if (iteration == 1) {                                                  // :39-41
        alpha = 2.0 / l_avg;
        copy = 1;
      } else {                                                               // :42-46
        beta = (l_diff * alpha / 2) * (l_diff * alpha / 2);
        alpha = 1.0 / (l_avg - beta);
      }
      if (sizeof(T) == 4) {  // the reference keeps alpha in real(T)
        alpha = (double)(float)alpha;
        beta = (double)(float)beta;
      }
      {
        ProfScope prof(ctx, 2);
        k_cheb_update_u<T><<<gv, kThreads, 0, st>>>(r, jac, u, n, beta, copy, s);
      }
      B200_LAUNCH_CHECK(ctx);
      {
        ProfScope prof(ctx, 0);
        B200_TRY(spmv(ctx, A, u, c));                                        // :48 (runs also past `done`: harmless)
      }
      {
        ProfScope prof(ctx, 1);
        k_cheb_update_xr<T><<<gv, kThreads, 0, st>>>(x, r, u, c, n, alpha, s, hist, ctx->red.partials,
                                                     ctx->red.ticket, single);
      }
      B200_LAUNCH_CHECK(ctx);
      B200_TRY(after(0));
    }
  }
  B200_CUDA(cudaMemcpyAsync(&h, s, sizeof(h), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  if (res) {
    res->iters = h.iter;
    res->mvps = mv_products + h.iter;                                        // :49, :151
    res->isconverged = h.resnorm <= h.tol;
    res->status = h.breakdown ? B200_ERR_BREAKDOWN : 0;
    res->tol = h.tol;
    res->residual = h.resnorm;
    res->n_resnorm = std::min<int64_t>(h.iter, hist_cap);
  }
  if (hist_cap && h.iter > 0) {
    B200_CUDA(cudaMemcpyAsync(resnorm_host, hist, sizeof(double) * std::min<int64_t>(h.iter, hist_cap),
                              cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
  }
  return B200_OK;
}

}  // namespace

extern "C" {

int b200_chebyshev_solve(b200_ctx *ctx, const b200_csr *A, void *x_dev, const void *b_dev, double lambda_min,
                         double lambda_max, const b200_cg_opts *opts, b200_result *res, double *resnorm_host,
                         int64_t resnorm_cap) {
  B200_TRY(real_only(A, "b200_chebyshev_solve"));
  B200_REQUIRE(ctx && A && x_dev && b_dev && opts, "NULL argument");
  B200_REQUIRE(A->ctx == ctx, "operator belongs to another context");
  B200_REQUIRE(is_square(A), "this solver needs a square operator (got %lld x %lld)", (long long)A->m_global,
               (long long)A->n_global);
  if (opts->Pl.kind == B200_PREC_CALLBACK)                                       // ldiv! by callback: the general engine
    return chebyshev_general(ctx, CudaOp{A, nullptr}, A->dtype, A->m_local, A->n_global, x_dev, b_dev, lambda_min,
                             lambda_max, opts, res, resnorm_host, resnorm_cap);
  B200_REQUIRE(opts->Pl.kind == B200_PREC_IDENTITY || (opts->Pl.kind == B200_PREC_JACOBI && opts->Pl.diag),
               "unsupported preconditioner");
  B200_CUDA(cudaSetDevice(ctx->device));
  return A->dtype == B200_F64 ? chebyshev_impl<double>(ctx, A, (double *)x_dev, (const double *)b_dev, lambda_min,
                                                       lambda_max, opts, res, resnorm_host, resnorm_cap)
                              : chebyshev_impl<float>(ctx, A, (float *)x_dev, (const float *)b_dev, lambda_min,
                                                      lambda_max, opts, res, resnorm_host, resnorm_cap);
}

}  // extern "C"
