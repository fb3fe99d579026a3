// bicgstabl.cu -- bicgstabl!(x, A, b, l; ...) of reference src/bicgstabl.jl:181-219
// (bicgstabl_iterator! :27-73, iterate :79-134).
//
// rs, us: n_local x (l+1) column-major blocks on the device.  Scalars (rho, sigma, alpha, beta,
// omega, gamma, M) live in device memory; the host only reads the residual once per outer
// iteration (2l SpMVs) to evaluate done() (:77).  Fusions:
//   * us[:,1:j] = rs[:,1:j] - beta*us[:,1:j]                         one launch for the j columns (:93)
//   * rs[:,1:j] -= alpha*us[:,2:j+1]  and  x += alpha*us[:,1]        one launch (:103,:111)
//   * M = rs'rs                                                       ONE pass over rs for all
//     (l+1)(l+2)/2 dots (:120)
//   * the three MR gemv updates + the residual norm                  one launch (:126-131)
// The (l x l) LU solve (:123-124, partial pivoting as lu!) runs in a one-thread kernel.
#include "blas1.cuh"
#include "spmv.cuh"
#include "linop.cuh"

using namespace b200;

namespace {

constexpr int kThreads = 256;
constexpr int LMAX = 8;                       // (LMAX+1)(LMAX+2)/2 = 45 <= kMaxReduceWidth
constexpr int NPAIR = (LMAX + 1) * (LMAX + 2) / 2;

struct BcScal {
  double rho, sigma, alpha, beta, omega;
  double residual, tol, abstol, reltol;
  double sum;                 // dot in flight
  double gram[NPAIR];         // upper triangle of rs'rs, (p,q) p<=q at index p*(2L+1-p)/2 + (q-p), L = l+1
  double gamma[LMAX];
  long long mv_products, max_mv, iters, hist_cap;
  int l, singular, breakdown, pad;
};

enum { BC_INIT = 1, BC_RHO = 2, BC_SIGMA = 3, BC_END = 4 };

__global__ void k_bc_scalar(int kind, BcScal *s, double *hist) {
  const double v = s->sum;
  switch (kind) {
    case BC_INIT:                                                       // :60-66
      s->residual = sqrt(v);
      s->tol = fmax(s->reltol * s->residual, s->abstol);
      s->omega = 1.0;
      s->sigma = 1.0;
      break;
    case BC_RHO:                                                        // :89-90
      s->rho = v;
      s->beta = v / s->sigma;
      break;
    case BC_SIGMA:                                                      // :100-101
      s->sigma = v;
      s->alpha = s->rho / v;
      break;
    case BC_END:                                                        // :115,:131
      s->mv_products += 2 * s->l;
      s->residual = sqrt(v);
      if (!(s->residual == s->residual)) s->breakdown = 1;
      if (hist && s->iters < s->hist_cap) hist[s->iters] = s->residual;
      s->iters += 1;
      break;
  }
}
__global__ void k_bc_begin(BcScal *s) { s->sigma = -s->omega * s->sigma; }    // :85

// MR part scalars: gamma = M[L,L] \ M[L,1] with lu! (partial pivoting)  (:120-124, :130)
__global__ void k_bc_mr_solve(BcScal *s) {
  const int l = s->l, L = l + 1;
  double M[LMAX + 1][LMAX + 1];
  for (int p = 0; p < L; ++p)
    for (int q = p; q < L; ++q) {
      const double v = s->gram[p * (2 * (LMAX + 1) + 1 - p) / 2 + (q - p)];
      M[p][q] = v;
      M[q][p] = v;
    }
  double a[LMAX][LMAX], rhs[LMAX];
  for (int i = 0; i < l; ++i) {
    rhs[i] = M[i + 1][0];
    for (int j = 0; j < l; ++j) a[i][j] = M[i + 1][j + 1];
  }
  int singular = 0;
  for (int k = 0; k < l; ++k) {
    int piv = k;
    double best = fabs(a[k][k]);
    for (int i = k + 1; i < l; ++i)
      if (fabs(a[i][k]) > best) { best = fabs(a[i][k]); piv = i; }
    if (best == 0.0 || !(best == best)) { singular = 1; break; }
    if (piv != k) {
      for (int j = 0; j < l; ++j) { const double t = a[k][j]; a[k][j] = a[piv][j]; a[piv][j] = t; }
      const double t = rhs[k]; rhs[k] = rhs[piv]; rhs[piv] = t;
    }
    for (int i = k + 1; i < l; ++i) {
      const double f = a[i][k] / a[k][k];
      for (int j = k; j < l; ++j) a[i][j] -= f * a[k][j];
      rhs[i] -= f * rhs[k];
    }
  }
  if (!singular) {
    for (int i = l - 1; i >= 0; --i) {
      double acc = rhs[i];
      for (int j = i + 1; j < l; ++j) acc -= a[i][j] * s->gamma[j];
      s->gamma[i] = acc / a[i][i];
    }
    s->omega = s->gamma[l - 1];                                         // :130
  }
  s->singular = singular;
}

// us[:,0:j) = rs[:,0:j) - beta*us[:,0:j)
template <typename T>
__global__ void __launch_bounds__(kThreads) k_bc_update_u(const T *__restrict__ rs, T *__restrict__ us, int64_t n,
                                                          int j, const BcScal *__restrict__ s) {
  const T beta = (T)s->beta;
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads)
    for (int c = 0; c < j; ++c) us[i + c * n] = rs[i + c * n] - beta * us[i + c * n];
}

// rs[:,0:j) -= alpha*us[:,1:j+1) ; x += alpha*us[:,0]
template <typename T>
__global__ void __launch_bounds__(kThreads) k_bc_update_r(T *__restrict__ rs, const T *__restrict__ us,
                                                          T *__restrict__ x, int64_t n, int j,
                                                          const BcScal *__restrict__ s) {
  const T alpha = (T)s->alpha;
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    for (int c = 0; c < j; ++c) rs[i + c * n] = rs[i + c * n] - alpha * us[i + (c + 1) * n];
    x[i] = x[i] + alpha * us[i];
  }
}

// upper triangle of rs'rs in one pass.  LC = compile-time column count (l + 1 for the common l, LMAX + 1 with
// zero-padded columns otherwise): the generic 9-column version carries 45 fp64 accumulators at 128 registers; l = 2
// needs 6.
// Output slots keep the static (p,q) numbering over LMAX+1 columns that k_bc_mr_solve reads.
__host__ __device__ constexpr int pair_slot(int p, int q) { return p * (2 * (LMAX + 1) + 1 - p) / 2 + (q - p); }

template <typename T, int LC>
__global__ void __launch_bounds__(kThreads) k_bc_gram(const T *__restrict__ rs, int64_t n, int L, double *partials,
                                                      unsigned int *ticket, double *__restrict__ out) {
  constexpr int NPL = LC * (LC + 1) / 2;
  __shared__ double smem[kThreads / 32][NPL];
  __shared__ bool is_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double acc[NPL];
#pragma unroll
  for (int p = 0; p < NPL; ++p) acc[p] = 0.0;
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
    double r[LC];
#pragma unroll
    for (int c = 0; c < LC; ++c) r[c] = c < L ? (double)rs[i + c * n] : 0.0;
    int k = 0;
#pragma unroll
    for (int p = 0; p < LC; ++p)
#pragma unroll
      for (int q = p; q < LC; ++q, ++k) acc[k] += r[p] * r[q];
  }
#pragma unroll
  for (int p = 0; p < NPL; ++p) {
    const double v = warp_sum(acc[p]);
    if (lane == 0) smem[warp][p] = v;
  }
  __syncthreads();
  if (threadIdx.x < NPL) {
    double sacc = 0.0;
    for (int wv = 0; wv < kThreads / 32; ++wv) sacc += smem[wv][threadIdx.x];
    partials[(size_t)blockIdx.x * kMaxReduceWidth + threadIdx.x] = sacc;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    is_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  if (threadIdx.x < NPAIR) out[threadIdx.x] = 0.0;      // pairs with a column >= LC
  __syncthreads();
  // warp w finishes pairs w, w + 8, ...: its lanes stride over the block slots (fixed order per lane, fixed shuffle tree:
  // deterministic), instead of NPL threads walking all slots one after the other
  for (int pr = warp; pr < NPL; pr += kThreads / 32) {
    double sacc = 0.0;
    for (unsigned int b = lane; b < gridDim.x; b += 32) sacc += __ldcg(&partials[(size_t)b * kMaxReduceWidth + pr]);
    sacc = warp_sum(sacc);
    if (lane == 0) {
      int p = 0, k = pr;                                  // local pair index -> (p, q)
      while (k >= LC - p) { k -= LC - p; ++p; }
      out[pair_slot(p, p + k)] = sacc;
    }
  }
  if (threadIdx.x == 0) *ticket = 0u;
}

// us[:,0] -= us[:,1:L) g ; x += rs[:,0:l) g ; rs[:,0] -= rs[:,1:L) g ; sum rs[:,0]^2   (:126-131)
// LCOL = compile-time l (0: runtime loops).  All 2l + 3 loads of a row are issued before the arithmetic.
template <typename T, int LCOL>
__global__ void __launch_bounds__(kThreads) k_bc_mr_update(T *__restrict__ rs, T *__restrict__ us, T *__restrict__ x,
                                                           int64_t n, int l, BcScal *s, double *partials,
                                                           unsigned int *ticket) {
  __shared__ double smem[kThreads / 32];
  double acc = 0.0;
  if constexpr (LCOL > 0) {
    T g[LCOL];
#pragma unroll
    for (int c = 0; c < LCOL; ++c) g[c] = (T)s->gamma[c];
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
      T r[LCOL + 1], u[LCOL + 1];
#pragma unroll
      for (int c = 0; c <= LCOL; ++c) {
        r[c] = rs[i + c * n];
        u[c] = us[i + c * n];
      }
      T u0 = u[0], xi = x[i], r0 = r[0];
#pragma unroll
      for (int c = 0; c < LCOL; ++c) {
        u0 -= u[c + 1] * g[c];
        xi += r[c] * g[c];
        r0 -= r[c + 1] * g[c];
      }
      us[i] = u0;
      x[i] = xi;
      rs[i] = r0;
      acc += (double)r0 * (double)r0;
    }
  } else {
    T g[LMAX];
    for (int c = 0; c < LMAX; ++c) g[c] = c < l ? (T)s->gamma[c] : (T)0;
    for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
      T r[LMAX + 1];
      for (int c = 0; c <= l; ++c) r[c] = rs[i + c * n];
      T u0 = us[i], xi = x[i], r0 = r[0];
      for (int c = 0; c < l; ++c) {
        u0 -= us[i + (c + 1) * n] * g[c];
        xi += r[c] * g[c];
        r0 -= r[c + 1] * g[c];
      }
      us[i] = u0;
      x[i] = xi;
      rs[i] = r0;
      acc += (double)r0 * (double)r0;
    }
  }
  acc = block_sum<kThreads>(acc, smem);
  double total;
  if (grid_reduce_finish<kThreads>(acc, partials, ticket, smem, &total) && threadIdx.x == 0) s->sum = total;
}

template <typename T>
int bicgstabl_impl(b200_ctx *ctx, const b200_csr *A, T *x, const T *b, const b200_bicgstabl_opts *o, b200_result *res,
                   double *resnorm_host, int64_t resnorm_cap) {
  cudaStream_t st = ctx->stream;
  const int64_t n = A->m_local;
  const int dt = dtype_of<T>::value;
  const double eps = sizeof(T) == 8 ? 2.220446049250313e-16 : 1.1920928955078125e-07;
  const double reltol = o->reltol < 0 ? sqrt(eps) : o->reltol;
  const int64_t max_mv = o->max_mv_products < 0 ? A->n_global : o->max_mv_products;
  const int l = o->l > 0 ? o->l : 2;
  B200_REQUIRE(l <= LMAX, "bicgstabl: l=%d exceeds the supported maximum %d", l, LMAX);
  const T *jac = o->Pl.kind == B200_PREC_JACOBI ? (const T *)o->Pl.diag : nullptr;
  const T *r_shadow = (const T *)o->r_shadow;
  const int64_t hist_cap = resnorm_host ? std::min<int64_t>(resnorm_cap, max_mv) : 0;

  const size_t blk = align_up(sizeof(T) * (size_t)std::max<int64_t>(n, 1) * (l + 1), 256);
  const size_t hist_bytes = align_up(sizeof(double) * (size_t)std::max<int64_t>(hist_cap, 1), 256);
  void *ws = nullptr;
  B200_TRY(ws_get(ctx, 2 * blk + 1024 + hist_bytes, &ws));
  char *p = (char *)ws;
  T *rs = (T *)p; p += blk;
  T *us = (T *)p; p += blk;
  BcScal *s = (BcScal *)p; p += 1024;
  static_assert(sizeof(BcScal) <= 1024, "BcScal too large");
  double *hist = hist_cap ? (double *)p : nullptr;

  BcScal h;
  memset(&h, 0, sizeof(h));
  h.abstol = o->abstol;
  h.reltol = reltol;
  h.max_mv = max_mv;
  h.hist_cap = hist_cap;
  h.l = l;
  h.omega = h.sigma = 1.0;
  B200_CUDA(cudaMemcpyAsync(s, &h, sizeof(h), cudaMemcpyHostToDevice, st));
  B200_CUDA(cudaMemsetAsync(us, 0, sizeof(T) * (size_t)n * (l + 1), st));        // us = zeros(T, n, l+1) :40
  const int gv = stream_grid(ctx, n, kThreads * 2, 8);

  auto scalar = [&](int kind) -> int {
    B200_TRY(allreduce_sum_dev(ctx, &s->sum, 1));
    k_bc_scalar<<<1, 1, 0, st>>>(kind, s, hist);
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
  };
  auto apply = [&](const T *src, T *dst) -> int {                                // dst = Pl \ (A src)
    {
      ProfScope prof(ctx, 0);
      B200_TRY(spmv(ctx, A, src, dst));
    }
    if (jac) B200_TRY(jacobi_ldiv(ctx, n, jac, dst, dst, dt));
    return B200_OK;
  };

  // bicgstabl_iterator! (:27-73)
  int64_t mv0 = 0;
  if (o->initial_zero) {
    B200_TRY(copy(ctx, n, b, rs, dt));                                           // :47
  } else {
    B200_TRY(spmv(ctx, A, x, rs));                                               // :49
    B200_TRY(axpby(ctx, n, 1.0, b, -1.0, rs, dt));                               // residual .= b .- residual :50
    mv0 = 1;
  }
  if (jac) B200_TRY(jacobi_ldiv(ctx, n, jac, rs, rs, dt));                       // :55
  B200_TRY(dot_dev(ctx, n, rs, rs, dt, &s->sum));                                // :60
  B200_TRY(scalar(BC_INIT));
  h.mv_products = mv0;
  B200_CUDA(cudaMemcpyAsync(&s->mv_products, &h.mv_products, sizeof(long long), cudaMemcpyHostToDevice, st));

  int status = B200_OK;
  for (;;) {
    B200_CUDA(cudaMemcpyAsync(&h, s, sizeof(h), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    if (h.singular) { status = B200_ERR_BREAKDOWN; set_error("SingularException in the BiCGStab(l) MR step"); break; }
    if (h.mv_products >= max_mv || h.residual <= h.tol || h.breakdown) break;    // done() :77
    k_bc_begin<<<1, 1, 0, st>>>(s);                                              // :85
    B200_LAUNCH_CHECK(ctx);
    for (int j = 1; j <= l; ++j) {                                               // :88
      B200_TRY(dot_dev(ctx, n, r_shadow, rs + (int64_t)(j - 1) * n, dt, &s->sum));  // :89
      B200_TRY(scalar(BC_RHO));
      k_bc_update_u<T><<<gv, kThreads, 0, st>>>(rs, us, n, j, s);                // :93
      B200_LAUNCH_CHECK(ctx);
      B200_TRY(apply(us + (int64_t)(j - 1) * n, us + (int64_t)j * n));           // :97-98
      B200_TRY(dot_dev(ctx, n, r_shadow, us + (int64_t)j * n, dt, &s->sum));     // :100
      B200_TRY(scalar(BC_SIGMA));
      k_bc_update_r<T><<<gv, kThreads, 0, st>>>(rs, us, x, n, j, s);             // :103, :111
      B200_LAUNCH_CHECK(ctx);
      B200_TRY(apply(rs + (int64_t)(j - 1) * n, rs + (int64_t)j * n));           // :107-108
    }
    {
      ProfScope prof(ctx, 1);
      switch (l) {                                                               // rs' rs  :120
        case 1: k_bc_gram<T, 2><<<gv, kThreads, 0, st>>>(rs, n, 2, ctx->red.partials, ctx->red.ticket, s->gram); break;
        case 2: k_bc_gram<T, 3><<<gv, kThreads, 0, st>>>(rs, n, 3, ctx->red.partials, ctx->red.ticket, s->gram); break;
        case 4: k_bc_gram<T, 5><<<gv, kThreads, 0, st>>>(rs, n, 5, ctx->red.partials, ctx->red.ticket, s->gram); break;
        default:
          k_bc_gram<T, LMAX + 1><<<gv, kThreads, 0, st>>>(rs, n, l + 1, ctx->red.partials, ctx->red.ticket, s->gram);
      }
    }
    B200_LAUNCH_CHECK(ctx);
    B200_TRY(allreduce_sum_dev(ctx, s->gram, NPAIR));
    k_bc_mr_solve<<<1, 1, 0, st>>>(s);                                           // :123-124
    B200_LAUNCH_CHECK(ctx);
    {
      ProfScope prof(ctx, 1);
      switch (l) {                                                               // :126-131
        case 1: k_bc_mr_update<T, 1><<<gv, kThreads, 0, st>>>(rs, us, x, n, l, s, ctx->red.partials, ctx->red.ticket); break;
        case 2: k_bc_mr_update<T, 2><<<gv, kThreads, 0, st>>>(rs, us, x, n, l, s, ctx->red.partials, ctx->red.ticket); break;
        case 4: k_bc_mr_update<T, 4><<<gv, kThreads, 0, st>>>(rs, us, x, n, l, s, ctx->red.partials, ctx->red.ticket); break;
        default: k_bc_mr_update<T, 0><<<gv, kThreads, 0, st>>>(rs, us, x, n, l, s, ctx->red.partials, ctx->red.ticket);
      }
    }
    B200_LAUNCH_CHECK(ctx);
    B200_TRY(scalar(BC_END));
  }
  if (res) {
    res->iters = h.iters;
    res->mvps = h.mv_products;                                                   // history.mvps = iterable.mv_products :207
    res->isconverged = h.residual <= h.tol;
    res->status = h.breakdown ? B200_ERR_BREAKDOWN : 0;
    res->tol = h.tol;
    res->residual = h.residual;
    res->n_resnorm = std::min<int64_t>(h.iters, hist_cap);
  }
  if (hist_cap && h.iters > 0) {
    B200_CUDA(cudaMemcpyAsync(resnorm_host, hist, sizeof(double) * std::min<int64_t>(h.iters, hist_cap),
                              cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
  }
  return status;
}

}  // namespace

extern "C" {

int b200_bicgstabl_solve(b200_ctx *ctx, const b200_csr *A, void *x_dev, const void *b_dev,
                         const b200_bicgstabl_opts *opts, b200_result *res, double *resnorm_host,
                         int64_t resnorm_cap) {
  B200_TRY(real_only(A, "b200_bicgstabl_solve"));
  B200_REQUIRE(ctx && A && x_dev && b_dev && opts && opts->r_shadow, "NULL argument (r_shadow is required)");
  B200_REQUIRE(A->ctx == ctx, "operator belongs to another context");
  B200_REQUIRE(is_square(A), "this solver needs a square operator (got %lld x %lld)", (long long)A->m_global,
               (long long)A->n_global);
  if (opts->Pl.kind == B200_PREC_CALLBACK)                                       // ldiv! by callback: the general engine
    return bicgstabl_general(ctx, CudaOp{A, nullptr}, A->dtype, A->m_local, A->n_global, x_dev, b_dev, opts, res,
                             resnorm_host, resnorm_cap);
  B200_REQUIRE(opts->Pl.kind == B200_PREC_IDENTITY || (opts->Pl.kind == B200_PREC_JACOBI && opts->Pl.diag),
               "unsupported preconditioner Pl");
  B200_CUDA(cudaSetDevice(ctx->device));
  return A->dtype == B200_F64 ? bicgstabl_impl<double>(ctx, A, (double *)x_dev, (const double *)b_dev, opts, res,
                                                       resnorm_host, resnorm_cap)
                              : bicgstabl_impl<float>(ctx, A, (float *)x_dev, (const float *)b_dev, opts, res,
                                                      resnorm_host, resnorm_cap);
}

}  // extern "C"
