// amg.cu -- the smoothed-aggregation AMG preconditioner on one GPU (DESIGN section 23).  The setup runs on the host
// (amg_core.h, fp64) and uploads each level as an ordinary operator, so every level gets finish_operator's analysis: the
// fine level of a stencil keeps its band description and value tables.  ldiv! is one V-cycle from a zero initial guess
// (AlgebraicMultigrid.jl's aspreconditioner), every SpMV of it one launch_spmv_fused with an epilogue of this file:
//   SmoothEpi    y = x + w .* (b - A x)       weighted-Jacobi sweep, w = omega_s ./ diag(A) per level, ping-pong buffers
//   ResidualEpi  r = b - A x
//   AddEpi       y = x + P e (prolongation), or y = R r with no addend (restriction)
// plus two small kernels: the first pre-sweep from x = 0 (x = w .* b, no SpMV) and the coarsest level's dense GEMV.
// A level above the coarsest costs presweeps + postsweeps SpMVs with A (the first pre-sweep is the vector pass, the
// residual one SpMV; with presweeps = 0 the residual is b itself), one with R and one with P.
//
// Buffers: everything the apply touches is owned by the handle (ldiv! runs inside a solver's preconditioner callback,
// where the context's workspace belongs to the solver).  x == y works: on the finest level only the last step writes y,
// and it reads b = x at its own row only; a one-level hierarchy copies x first.  No atomics: results are the same bits
// run to run.
#include <chrono>
#include <memory>

#include "amg_core.h"
#include "csr.cuh"
#include "spmv_launch.cuh"

using namespace b200;

namespace {

constexpr int kAmgThreads = 256;

template <typename T>
struct SmoothEpi {
  const T *x, *w, *b;
  T *y;
  __device__ __forceinline__ bool begin() const { return true; }
  __device__ __forceinline__ T pre(int64_t row) const { return __ldg(b + row); }
  __device__ __forceinline__ void operator()(int64_t row, T v, T bi) { y[row] = x[row] + __ldg(w + row) * (bi - v); }
  template <int THREADS>
  __device__ __forceinline__ void end(double *) const {}
  __device__ static constexpr bool rev() { return false; }
};

template <typename T>
struct ResidualEpi {
  const T *b;
  T *r;
  __device__ __forceinline__ bool begin() const { return true; }
  __device__ __forceinline__ T pre(int64_t row) const { return __ldg(b + row); }
  __device__ __forceinline__ void operator()(int64_t row, T v, T bi) { r[row] = bi - v; }
  template <int THREADS>
  __device__ __forceinline__ void end(double *) const {}
  __device__ static constexpr bool rev() { return false; }
};

template <typename T>
struct AddEpi {
  const T *x;   // nullptr: y = A e
  T *y;
  __device__ __forceinline__ bool begin() const { return true; }
  __device__ __forceinline__ T pre(int64_t row) const { return x ? x[row] : (T)0; }
  __device__ __forceinline__ void operator()(int64_t row, T v, T xi) { y[row] = xi + v; }
  template <int THREADS>
  __device__ __forceinline__ void end(double *) const {}
  __device__ static constexpr bool rev() { return false; }
};

// the first pre-sweep from x = 0: x = w .* b
template <typename T>
__global__ void __launch_bounds__(kAmgThreads) k_amg_scale(int64_t n, const T *__restrict__ w, const T *__restrict__ b,
                                                           T *__restrict__ x) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    x[i] = w[i] * b[i];
}

// the coarsest level: x = C b, C dense n x n row-major; one warp per row, lanes over the columns, a fixed shuffle tree
template <typename T>
__global__ void __launch_bounds__(kAmgThreads) k_amg_gemv(int n, const T *__restrict__ C, const T *__restrict__ b,
                                                          T *__restrict__ x) {
  const int lane = threadIdx.x & 31;
  for (int i = blockIdx.x * (kAmgThreads / 32) + threadIdx.x / 32; i < n; i += gridDim.x * (kAmgThreads / 32)) {
    const T *row = C + (int64_t)i * n;
    T acc = (T)0;
    for (int j = lane; j < n; j += 32) acc += row[j] * b[j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) x[i] = acc;
  }
}

struct DevLevel {
  const b200_csr *A = nullptr;   // level 0: the caller's operator; coarser levels: owned
  b200_csr *P = nullptr, *R = nullptr;
  int64_t n = 0;
  void *w = nullptr, *b = nullptr, *x = nullptr, *u0 = nullptr, *u1 = nullptr, *inv = nullptr;
  std::vector<int> agg;
};

}  // namespace

struct b200_amg {
  b200_ctx *ctx = nullptr;
  int dtype = B200_F64;
  AmgOptions opts;
  std::vector<DevLevel> lev;
  std::vector<int64_t> nnz_P;
  double seconds[5] = {0, 0, 0, 0, 0};   // download, aggregation, P, RAP + coarse inverse, upload
  ~b200_amg() {
    if (ctx) {
      cudaSetDevice(ctx->device);
      cudaStreamSynchronize(ctx->stream);
    }
    for (size_t l = 0; l < lev.size(); ++l) {
      DevLevel &L = lev[l];
      if (l > 0 && L.A) b200_csr_destroy(const_cast<b200_csr *>(L.A));
      if (L.P) b200_csr_destroy(L.P);
      if (L.R) b200_csr_destroy(L.R);
      for (void *p : {L.w, L.b, L.x, L.u0, L.u1, L.inv})
        if (p) cudaFree(p);
    }
  }
};

namespace {

int dev_alloc(void **p, size_t bytes) {
  if (cudaMalloc(p, bytes ? bytes : 16) != cudaSuccess) {
    *p = nullptr;
    set_error("b200_amg_create: cudaMalloc(%zu) failed", bytes);
    return B200_ERR_ALLOC;
  }
  return B200_OK;
}

template <typename T>
int upload_vec(void **p, const std::vector<double> &h, cudaStream_t st) {
  std::vector<T> t(h.begin(), h.end());
  B200_TRY(dev_alloc(p, sizeof(T) * t.size()));
  if (!t.empty()) B200_CUDA(cudaMemcpyAsync(*p, t.data(), sizeof(T) * t.size(), cudaMemcpyHostToDevice, st));
  B200_CUDA(cudaStreamSynchronize(st));   // t is a temporary
  return B200_OK;
}

// a host level matrix as a device operator: square ones through the CSR slab constructor, rectangular ones (P) as the
// CSC whose arrays are those of P' (both finish_operator'd); values rounded to T
template <typename T>
int upload_csr(b200_ctx *ctx, const AmgCsr &M, b200_csr **out) {
  const int dtype = sizeof(T) == 8 ? B200_F64 : B200_F32;
  if (M.m == M.n) {
    std::vector<T> v(M.vals.begin(), M.vals.end());
    std::vector<int64_t> ci(M.colind.begin(), M.colind.end());
    return b200_csr_from_csr_slab(ctx, M.n, 0, M.m, M.rowptr.data(), ci.data(), v.data(), 8, dtype, 0, nullptr, out);
  }
  const AmgCsr Mt = amg_transpose(M);
  std::vector<T> vt(Mt.vals.begin(), Mt.vals.end());
  std::vector<int64_t> ri(Mt.colind.begin(), Mt.colind.end());
  return b200_csr_from_csc(ctx, M.m, M.n, Mt.rowptr.data(), ri.data(), vt.data(), 8, dtype, 0, out);
}

double now_s() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

template <typename T>
int amg_create(b200_ctx *ctx, const b200_csr *A, const AmgOptions &o, b200_amg **out) {
  const int64_t n = A->m_local, nnz = A->nnz;
  cudaStream_t st = ctx->stream;
  std::unique_ptr<b200_amg> H(new b200_amg());
  H->ctx = ctx;
  H->dtype = A->dtype;
  H->opts = o;
  double t0 = now_s();
  AmgCsr h;
  h.m = h.n = n;
  {
    std::vector<int> rowptr((size_t)n + 1);
    std::vector<T> vals((size_t)nnz);
    h.colind.resize((size_t)nnz);
    B200_CUDA(cudaMemcpyAsync(rowptr.data(), A->rowptr, sizeof(int) * (size_t)(n + 1), cudaMemcpyDeviceToHost, st));
    if (nnz) {
      B200_CUDA(cudaMemcpyAsync(h.colind.data(), A->colind, sizeof(int) * (size_t)nnz, cudaMemcpyDeviceToHost, st));
      B200_CUDA(cudaMemcpyAsync(vals.data(), A->vals, sizeof(T) * (size_t)nnz, cudaMemcpyDeviceToHost, st));
    }
    B200_CUDA(cudaStreamSynchronize(st));
    h.rowptr.assign(rowptr.begin(), rowptr.end());
    h.vals.assign(vals.begin(), vals.end());
  }
  for (int64_t i = 0; i < n; ++i)
    for (int64_t p = h.rowptr[(size_t)i] + 1; p < h.rowptr[(size_t)i + 1]; ++p)
      B200_REQUIRE(h.colind[(size_t)p - 1] < h.colind[(size_t)p], "AMG needs rows with ascending column indices (row %lld)",
                   (long long)i);
  double t1 = now_s();
  H->seconds[0] = t1 - t0;
  std::vector<AmgLevel> levels;
  AmgTimes tm;
  const AmgStatus s = amg_setup(std::move(h), o, &levels, &tm, now_s);
  if (s.code == AMG_ZERO_DIAGONAL) {
    set_error("smoothed aggregation: zero or missing diagonal entry in row %lld (0-based) of level %d", (long long)s.row,
              s.level);
    return B200_ERR_BREAKDOWN;
  }
  if (s.code == AMG_ZERO_PIVOT) {
    set_error("smoothed aggregation: the coarsest level (level %d) is singular: zero pivot in column %lld (0-based)",
              s.level, (long long)s.row);
    return B200_ERR_BREAKDOWN;
  }
  if (s.code == AMG_TOO_LARGE) {
    set_error("smoothed aggregation: the coarsest level (level %d) has %lld rows, more than the %d its dense inverse "
              "allows; raise max_levels or lower max_coarse",
              s.level, (long long)s.row, kAmgMaxCoarsest);
    return B200_ERR_INVALID;
  }
  H->seconds[1] = tm.aggregation;
  H->seconds[2] = tm.prolongator;
  H->seconds[3] = tm.rap;
  t0 = now_s();
  H->lev.resize(levels.size());
  const size_t vs = sizeof(T);
  for (size_t l = 0; l < levels.size(); ++l) {
    AmgLevel &hl = levels[l];
    DevLevel &L = H->lev[l];
    L.n = hl.A.m;
    if (l == 0) {
      L.A = A;
    } else {
      b200_csr *Al = nullptr;
      B200_TRY(upload_csr<T>(ctx, hl.A, &Al));
      L.A = Al;
    }
    if (l + 1 < levels.size()) {
      B200_TRY(upload_csr<T>(ctx, hl.P, &L.P));
      B200_TRY(b200_csr_transpose(ctx, L.P, &L.R));
      B200_TRY(upload_vec<T>(&L.w, hl.w, st));
      L.agg = std::move(hl.agg);
      H->nnz_P.push_back(hl.P.nnz());
      B200_TRY(dev_alloc(&L.u0, vs * (size_t)L.n));
      B200_TRY(dev_alloc(&L.u1, vs * (size_t)L.n));
    } else {
      B200_TRY(upload_vec<T>(&L.inv, hl.inv, st));
      if (l == 0) B200_TRY(dev_alloc(&L.u0, vs * (size_t)L.n));   // the copy of x when x == y
    }
    if (l > 0) {
      B200_TRY(dev_alloc(&L.b, vs * (size_t)L.n));
      B200_TRY(dev_alloc(&L.x, vs * (size_t)L.n));
    }
  }
  B200_CUDA(cudaStreamSynchronize(st));
  H->seconds[4] = now_s() - t0;
  *out = H.release();
  return B200_OK;
}

template <typename T>
int launch_scale(b200_ctx *ctx, int64_t n, const void *w, const void *b, void *x) {
  k_amg_scale<T><<<stream_grid(ctx, n, kAmgThreads, 8), kAmgThreads, 0, ctx->stream>>>(n, (const T *)w, (const T *)b,
                                                                                       (T *)x);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

// one V-cycle on level l: x = V_l(b); x is written by the level's last step only
template <typename T>
int vcycle(b200_amg *H, size_t l, const T *b, T *x) {
  b200_ctx *ctx = H->ctx;
  DevLevel &L = H->lev[l];
  if (l + 1 == H->lev.size()) {
    const int n = (int)L.n;
    k_amg_gemv<T><<<stream_grid(ctx, n, kAmgThreads / 32, 8), kAmgThreads, 0, ctx->stream>>>(n, (const T *)L.inv, b, x);
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
  }
  const AmgOptions &o = H->opts;
  T *u0 = (T *)L.u0, *u1 = (T *)L.u1;
  auto other = [&](const T *p) { return p == u0 ? u1 : u0; };
  const T *w = (const T *)L.w;
  T *cur = nullptr;   // nullptr: x = 0
  for (int s = 0; s < o.presweeps; ++s) {
    T *dst = other(cur);
    if (!cur) B200_TRY(launch_scale<T>(ctx, L.n, w, b, dst));
    else B200_TRY(launch_spmv_fused<T>(ctx, L.A, cur, false, SmoothEpi<T>{cur, w, b, dst}, false));
    cur = dst;
  }
  const T *r = b;
  if (cur) {
    T *dst = other(cur);
    B200_TRY(launch_spmv_fused<T>(ctx, L.A, cur, false, ResidualEpi<T>{b, dst}, false));
    r = dst;
  }
  DevLevel &C = H->lev[l + 1];
  B200_TRY(launch_spmv_fused<T>(ctx, L.R, r, false, AddEpi<T>{nullptr, (T *)C.b}, false));
  B200_TRY(vcycle<T>(H, l + 1, (const T *)C.b, (T *)C.x));
  T *dst = o.postsweeps == 0 ? x : (cur ? cur : u0);   // in place on cur: P reads e only
  B200_TRY(launch_spmv_fused<T>(ctx, L.P, C.x, false, AddEpi<T>{cur, dst}, false));
  cur = dst;
  for (int s = 0; s < o.postsweeps; ++s) {
    dst = s + 1 == o.postsweeps ? x : other(cur);
    B200_TRY(launch_spmv_fused<T>(ctx, L.A, cur, false, SmoothEpi<T>{cur, w, b, dst}, false));
    cur = dst;
  }
  return B200_OK;
}

int amg_ldiv(b200_amg *H, const void *x, void *y) {
  b200_ctx *ctx = H->ctx;
  if (H->lev.size() == 1 && x == y) {   // the dense GEMV reads all of b while it writes x
    B200_CUDA(cudaMemcpyAsync(H->lev[0].u0, x, dtype_size(H->dtype) * (size_t)H->lev[0].n, cudaMemcpyDeviceToDevice,
                              ctx->stream));
    x = H->lev[0].u0;
  }
  if (H->dtype == B200_F64) return vcycle<double>(H, 0, (const double *)x, (double *)y);
  return vcycle<float>(H, 0, (const float *)x, (float *)y);
}

int amg_apply_thunk(void *user, const void *x, void *y, void *) { return amg_ldiv((b200_amg *)user, x, y); }

}  // namespace

extern "C" {

int b200_amg_create(b200_ctx *ctx, const b200_csr *A, const b200_amg_opts *opts, b200_amg **out) {
  B200_REQUIRE(ctx && A && out, "NULL argument");
  *out = nullptr;
  B200_TRY(real_only(A, "b200_amg_create"));
  B200_REQUIRE(A->ctx == ctx, "operator belongs to another context");
  if (A->rowptr64) {
    set_error("b200_amg_create: the setup holds int32 row offsets; an operator with 8-byte row offsets (nnz >= 2^31, or "
              "built with \"rowptr64\" = 1) is not supported");
    return B200_ERR_UNSUPPORTED;
  }
  B200_REQUIRE(ctx->world == 1, "smoothed aggregation builds the whole hierarchy on one GPU: single-GPU contexts only");
  B200_REQUIRE(is_square(A), "smoothed aggregation needs a square operator");
  AmgOptions o;
  if (opts) {
    o.theta = opts->theta;
    o.max_levels = opts->max_levels;
    o.max_coarse = opts->max_coarse;
    o.presweeps = opts->presweeps;
    o.postsweeps = opts->postsweeps;
  }
  B200_REQUIRE(o.theta >= 0.0, "smoothed aggregation: theta = %g must be >= 0", o.theta);
  B200_REQUIRE(o.max_levels >= 1, "smoothed aggregation: max_levels = %d must be >= 1", o.max_levels);
  B200_REQUIRE(o.max_coarse >= 1, "smoothed aggregation: max_coarse = %d must be >= 1", o.max_coarse);
  B200_REQUIRE(o.presweeps >= 0 && o.postsweeps >= 0, "smoothed aggregation: presweeps = %d and postsweeps = %d must be >= 0",
               o.presweeps, o.postsweeps);
  B200_CUDA(cudaSetDevice(ctx->device));
  return A->dtype == B200_F64 ? amg_create<double>(ctx, A, o, out) : amg_create<float>(ctx, A, o, out);
}

int b200_amg_ldiv(b200_ctx *ctx, b200_amg *P, const void *x_dev, void *y_dev) {
  B200_REQUIRE(ctx && P && x_dev && y_dev, "NULL argument");
  B200_REQUIRE(P->ctx == ctx, "preconditioner belongs to another context");
  B200_CUDA(cudaSetDevice(ctx->device));
  return amg_ldiv(P, x_dev, y_dev);
}

int b200_amg_as_linop(b200_amg *P, b200_linop *out) {
  B200_REQUIRE(P && out, "NULL argument");
  out->apply = amg_apply_thunk;
  out->user = (void *)P;
  out->m_local = out->n_local = out->n_global = out->m_global = P->lev[0].n;
  out->dtype = P->dtype;
  out->reserved = 0;
  return B200_OK;
}

int b200_amg_info(const b200_amg *P, int *levels, int64_t *rows, int64_t *nnz, int cap, double *setup_seconds) {
  B200_REQUIRE(P, "NULL argument");
  if (levels) *levels = (int)P->lev.size();
  for (int l = 0; l < cap && l < (int)P->lev.size(); ++l) {
    if (rows) rows[l] = P->lev[(size_t)l].n;
    if (nnz) nnz[l] = P->lev[(size_t)l].A->nnz;
  }
  if (setup_seconds)
    for (int k = 0; k < 5; ++k) setup_seconds[k] = P->seconds[k];
  return B200_OK;
}

int b200_amg_download_level(const b200_amg *P, int level, const b200_csr **A, const b200_csr **Pl, int32_t *agg,
                            void *coarse_inv) {
  B200_REQUIRE(P, "NULL argument");
  B200_REQUIRE(level >= 0 && level < (int)P->lev.size(), "level %d out of range [0, %d)", level, (int)P->lev.size());
  const DevLevel &L = P->lev[(size_t)level];
  const bool coarsest = level + 1 == (int)P->lev.size();
  if (A) *A = L.A;
  if (Pl) *Pl = L.P;
  if (agg && !coarsest) memcpy(agg, L.agg.data(), sizeof(int32_t) * L.agg.size());
  if (coarse_inv && coarsest) {
    B200_CUDA(cudaSetDevice(P->ctx->device));
    B200_CUDA(cudaMemcpyAsync(coarse_inv, L.inv, dtype_size(P->dtype) * (size_t)(L.n * L.n), cudaMemcpyDeviceToHost,
                              P->ctx->stream));
    B200_CUDA(cudaStreamSynchronize(P->ctx->stream));
  }
  return B200_OK;
}

int b200_amg_destroy(b200_amg *P) {
  delete P;
  return B200_OK;
}

}  // extern "C"
