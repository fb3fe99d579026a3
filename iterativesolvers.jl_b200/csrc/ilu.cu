// ilu.cu -- the ILU(0) preconditioner on one GPU (ilu_core.h): the factorization and each of the two triangular solves of
// ldiv! are ONE persistent launch each, scheduled through a chunk list (DESIGN section 22).
//
//   Schedule   the host analysis (stationary_analyse: diagonal positions, forward / backward dependency levels) is cut into
//              chunks of up to 32 consecutive rows of one level, in level order.  A warp claims chunks in order through an
//              atomic ticket (not blockIdx), one lane per row.  A chunk depends only on chunks of earlier levels, i.e. on
//              chunks that running warps have already claimed, so the launch cannot deadlock whatever the grid size.
//   Handshake  a lane waits for each dependency's ready flag with an acquire load, then reads its value; it publishes its
//              own value, then its flag with a release store.  Flags are one epoch word per row: every launch uses a fresh
//              epoch, so no reset pass is needed; the flags are cleared only when the epoch counter wraps.  The ticket is
//              never reset either: a launch of W warps over C chunks takes exactly C + W tickets, and the next launch
//              starts counting where this one ended.
//   Bounded    a spin gives up after kIluSpinLimit polls and raises the handle's error word (pinned host memory) instead of
//              hanging; the next ldiv / download reports it.  Cannot happen with a valid schedule.
//   Buffers    everything the apply touches is owned by the handle: ldiv! runs inside a solver's preconditioner callback,
//              where the context's workspace belongs to the calling solver.
#include <memory>

#include "csr.cuh"
#include "ilu_core.h"

using namespace b200;

namespace {

constexpr int kIluThreads = 128;
constexpr int kIluBlocksPerSm = 2;   // 8 resident warps per SM
constexpr unsigned long long kIluSpinLimit = 1ull << 26;
enum { K_FACTOR = 0, K_FORWARD = 1, K_BACKWARD = 2 };

__device__ __forceinline__ unsigned ld_acquire_gpu_u32(const unsigned *p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu_u32(unsigned *p, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// wait(j) of the row functions: bounded spin on row j's flag, with a short sleep between polls (spinning lanes would
// otherwise flood L2 with acquire loads and slow down the lanes they wait for)
struct DevWait {
  const unsigned *flags;
  unsigned epoch;
  __device__ __forceinline__ bool operator()(int j) const {
    unsigned long long spins = 0;
    while (ld_acquire_gpu_u32(&flags[j]) != epoch) {
      if (++spins > kIluSpinLimit) return false;
      __nanosleep(64);
    }
    return true;
  }
};

struct SweepArgs {
  const int *rows, *cptr;              // the chunk schedule of the sweep
  long long nchunks;
  unsigned *flags;
  unsigned epoch;
  unsigned long long *ticket, base;    // chunk c = ticket - base
  unsigned long long *pivot;           // factorization: smallest zero-pivot row + 1 (atomicMin)
  unsigned long long *err;             // pinned host word: row + 1 of a spin that timed out
};

template <typename T, int KIND>
__global__ void __launch_bounds__(kIluThreads) k_ilu_sweep(const IluView<T, int> v, const SweepArgs a, const T *x, T *y) {
  const int lane = threadIdx.x & 31;
  DevWait wait{a.flags, a.epoch};
  for (;;) {
    unsigned long long t = 0;
    if (lane == 0) t = atomicAdd(a.ticket, 1ull);
    t = __shfl_sync(0xffffffffu, t, 0);
    const unsigned long long c = t - a.base;
    if (c >= (unsigned long long)a.nchunks) return;
    const int b = __ldg(&a.cptr[c]), e = __ldg(&a.cptr[c + 1]);
    if (b + lane < e) {
      const int i = __ldg(&a.rows[b + lane]);
      int st;
      if constexpr (KIND == K_FACTOR) st = ilu_factor_row(v, i, wait);
      else if constexpr (KIND == K_FORWARD) st = ilu_forward_row(v, i, x, y, wait);
      else st = ilu_backward_row(v, i, (const T *)x, y, wait);
      if (st == ILU_ZERO_PIVOT) atomicMin(a.pivot, (unsigned long long)i + 1ull);
      else if (st == ILU_NOT_READY) *(volatile unsigned long long *)a.err = (unsigned long long)i + 1ull;
      st_release_gpu_u32(&a.flags[i], a.epoch);   // published even after a failure: the dependants do not spin too
    }
  }
}

template <typename T>
struct DevArray {
  T *p = nullptr;
  ~DevArray() { if (p) cudaFree(p); }
  int alloc(size_t count) {
    if (cudaMalloc((void **)&p, sizeof(T) * (count ? count : 1)) != cudaSuccess) {
      set_error("b200_ilu0_create: cudaMalloc failed");
      return B200_ERR_ALLOC;
    }
    return B200_OK;
  }
  int upload(const std::vector<T> &h, cudaStream_t st) {
    B200_TRY(alloc(h.size()));
    if (!h.empty()) B200_CUDA(cudaMemcpyAsync(p, h.data(), sizeof(T) * h.size(), cudaMemcpyHostToDevice, st));
    return B200_OK;
  }
};

}  // namespace

struct b200_ilu0 {
  b200_ctx *ctx = nullptr;
  const b200_csr *A = nullptr;     // the factor reuses A's rowptr / colind: A must outlive the handle
  int dtype = B200_F64;
  int64_t n = 0, nnz = 0, nnz_lower = 0;
  int levels_f = 0, levels_b = 0;
  int64_t chunks_f = 0, chunks_b = 0;
  DevArray<char> f;                 // factor values, A's CSR order
  DevArray<int> dpos, rows_f, cptr_f, rows_b, cptr_b;
  DevArray<unsigned> flags;
  DevArray<unsigned long long> ticket, pivot;
  unsigned long long ticket_base = 0;
  unsigned epoch = 0;
  unsigned long long *err = nullptr;   // pinned, device-mapped
  ~b200_ilu0() {
    if (ctx) {
      cudaSetDevice(ctx->device);
      cudaStreamSynchronize(ctx->stream);
    }
    if (err) cudaFreeHost(err);
  }
};

namespace {

// blocks per launch: at most kIluBlocksPerSm per SM (any grid is deadlock-free; more resident warps keep more levels in
// flight but poll more and measured slower on H100: DESIGN section 22), at most one warp per chunk
int sweep_blocks(const b200_ctx *ctx, int64_t nchunks) {
  const int64_t warps_per_block = kIluThreads / 32;
  const int64_t need = (nchunks + warps_per_block - 1) / warps_per_block;
  return (int)std::max<int64_t>(1, std::min<int64_t>(need, (int64_t)ctx->sm_count * kIluBlocksPerSm));
}

int check_err(const b200_ilu0 *P) {
  const unsigned long long e = *(volatile unsigned long long *)P->err;
  if (e) {
    set_error("ILU(0): a dependency wait timed out at row %llu (0-based): the factor is unusable", e - 1ull);
    return B200_ERR_CUDA;
  }
  return B200_OK;
}

template <typename T, int KIND>
int sweep(b200_ilu0 *P, const void *x, void *y, cudaStream_t st) {
  const bool fwd = KIND != K_BACKWARD;
  const int64_t nchunks = fwd ? P->chunks_f : P->chunks_b;
  if (nchunks <= 0) return B200_OK;
  if (P->epoch == 0xffffffffu) {                      // the epoch wraps: clear the flags once
    B200_CUDA(cudaMemsetAsync(P->flags.p, 0, sizeof(unsigned) * (size_t)P->n, st));
    P->epoch = 0;
  }
  P->epoch += 1;
  SweepArgs a{fwd ? P->rows_f.p : P->rows_b.p, fwd ? P->cptr_f.p : P->cptr_b.p, (long long)nchunks, P->flags.p,
              P->epoch, P->ticket.p, P->ticket_base, P->pivot.p, P->err};
  const IluView<T, int> v{P->A->rowptr, P->A->colind, P->dpos.p, (T *)P->f.p};
  const int blocks = sweep_blocks(P->ctx, nchunks);
  k_ilu_sweep<T, KIND><<<blocks, kIluThreads, 0, st>>>(v, a, (const T *)x, (T *)y);
  B200_LAUNCH_CHECK(P->ctx);
  P->ticket_base += (unsigned long long)nchunks + (unsigned long long)blocks * (kIluThreads / 32);
  return B200_OK;
}

// ldiv!(y, P, x): forward solve x -> y, backward solve in place on y (both in-place safe, so x == y works)
int ilu_ldiv(b200_ilu0 *P, const void *x, void *y, cudaStream_t st) {
  B200_TRY(check_err(P));
  if (P->dtype == B200_F64) {
    B200_TRY((sweep<double, K_FORWARD>(P, x, y, st)));
    return sweep<double, K_BACKWARD>(P, y, y, st);
  }
  B200_TRY((sweep<float, K_FORWARD>(P, x, y, st)));
  return sweep<float, K_BACKWARD>(P, y, y, st);
}

int ilu_apply_thunk(void *user, const void *x, void *y, void *stream) {
  b200_ilu0 *P = (b200_ilu0 *)user;
  return ilu_ldiv(P, x, y, (cudaStream_t)stream);
}

template <typename T>
int ilu_create(b200_ctx *ctx, const b200_csr *A, b200_ilu0 **out) {
  const int64_t n = A->m_local, nnz = A->nnz;
  cudaStream_t st = ctx->stream;
  std::vector<int> rowptr((size_t)n + 1), colind((size_t)nnz);
  std::vector<T> vals((size_t)nnz);
  B200_CUDA(cudaMemcpyAsync(rowptr.data(), A->rowptr, sizeof(int) * (size_t)(n + 1), cudaMemcpyDeviceToHost, st));
  if (nnz) {
    B200_CUDA(cudaMemcpyAsync(colind.data(), A->colind, sizeof(int) * (size_t)nnz, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaMemcpyAsync(vals.data(), A->vals, sizeof(T) * (size_t)nnz, cudaMemcpyDeviceToHost, st));
  }
  B200_CUDA(cudaStreamSynchronize(st));
  for (int64_t i = 0; i < n; ++i)
    for (int p = rowptr[(size_t)i] + 1; p < rowptr[(size_t)i + 1]; ++p)
      B200_REQUIRE(colind[(size_t)p - 1] < colind[(size_t)p], "ILU(0) needs rows with ascending column indices (row %lld)",
                   (long long)i);
  std::vector<int> dpos;
  IluSchedule fw, bw;
  const int64_t singular = ilu_analyse<T, int>(n, rowptr.data(), colind.data(), vals.data(), &dpos, &fw, &bw);
  if (singular) {
    set_error("ILU(0): zero or missing diagonal entry in row %lld (0-based)", (long long)(singular - 1));
    return B200_ERR_BREAKDOWN;
  }
  std::unique_ptr<b200_ilu0> P(new b200_ilu0());
  P->ctx = ctx;
  P->A = A;
  P->dtype = A->dtype;
  P->n = n;
  P->nnz = nnz;
  for (int64_t i = 0; i < n; ++i) P->nnz_lower += dpos[(size_t)i];
  P->levels_f = fw.levels;
  P->levels_b = bw.levels;
  P->chunks_f = fw.chunks();
  P->chunks_b = bw.chunks();
  B200_TRY(P->f.alloc(sizeof(T) * (size_t)nnz));
  if (nnz) B200_CUDA(cudaMemcpyAsync(P->f.p, A->vals, sizeof(T) * (size_t)nnz, cudaMemcpyDeviceToDevice, st));
  B200_TRY(P->dpos.upload(dpos, st));
  B200_TRY(P->rows_f.upload(fw.rows, st));
  B200_TRY(P->cptr_f.upload(fw.cptr, st));
  B200_TRY(P->rows_b.upload(bw.rows, st));
  B200_TRY(P->cptr_b.upload(bw.cptr, st));
  B200_TRY(P->flags.alloc((size_t)n));
  B200_CUDA(cudaMemsetAsync(P->flags.p, 0, sizeof(unsigned) * (size_t)n, st));
  B200_TRY(P->ticket.alloc(1));
  B200_CUDA(cudaMemsetAsync(P->ticket.p, 0, sizeof(unsigned long long), st));
  B200_TRY(P->pivot.alloc(1));
  B200_CUDA(cudaMemsetAsync(P->pivot.p, 0xff, sizeof(unsigned long long), st));
  if (cudaHostAlloc((void **)&P->err, sizeof(unsigned long long), cudaHostAllocMapped) != cudaSuccess) {
    P->err = nullptr;
    set_error("b200_ilu0_create: cudaHostAlloc failed");
    return B200_ERR_ALLOC;
  }
  *P->err = 0;
  B200_TRY((sweep<T, K_FACTOR>(P.get(), nullptr, nullptr, st)));
  unsigned long long pivot = 0;
  B200_CUDA(cudaMemcpyAsync(&pivot, P->pivot.p, sizeof(pivot), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  B200_TRY(check_err(P.get()));
  if (pivot != ~0ull) {
    set_error("ILU(0): zero pivot u_ii in row %llu (0-based)", pivot - 1ull);
    return B200_ERR_BREAKDOWN;
  }
  *out = P.release();
  return B200_OK;
}

}  // namespace

extern "C" {

int b200_ilu0_create(b200_ctx *ctx, const b200_csr *A, b200_ilu0 **out) {
  B200_REQUIRE(ctx && A && out, "NULL argument");
  *out = nullptr;
  B200_TRY(real_only(A, "b200_ilu0_create"));
  B200_REQUIRE(A->ctx == ctx, "operator belongs to another context");
  if (A->rowptr64) {
    set_error("b200_ilu0_create: the factor's analysis holds int32 row offsets; an operator with 8-byte row offsets "
              "(nnz >= 2^31, or built with \"rowptr64\" = 1) is not supported");
    return B200_ERR_UNSUPPORTED;
  }
  B200_REQUIRE(ctx->world == 1, "ILU(0) factors the whole matrix in order: single-GPU contexts only");
  B200_REQUIRE(is_square(A), "ILU(0) needs a square operator");
  B200_CUDA(cudaSetDevice(ctx->device));
  return A->dtype == B200_F64 ? ilu_create<double>(ctx, A, out) : ilu_create<float>(ctx, A, out);
}

int b200_ilu0_ldiv(b200_ctx *ctx, b200_ilu0 *P, const void *x_dev, void *y_dev) {
  B200_REQUIRE(ctx && P && x_dev && y_dev, "NULL argument");
  B200_REQUIRE(P->ctx == ctx, "preconditioner belongs to another context");
  B200_CUDA(cudaSetDevice(ctx->device));
  return ilu_ldiv(P, x_dev, y_dev, ctx->stream);
}

int b200_ilu0_as_linop(b200_ilu0 *P, b200_linop *out) {
  B200_REQUIRE(P && out, "NULL argument");
  out->apply = ilu_apply_thunk;
  out->user = (void *)P;
  out->m_local = out->n_local = out->n_global = out->m_global = P->n;
  out->dtype = P->dtype;
  out->reserved = 0;
  return B200_OK;
}

int b200_ilu0_download(const b200_ilu0 *P, void *vals_host) {
  B200_REQUIRE(P && vals_host, "NULL argument");
  B200_CUDA(cudaSetDevice(P->ctx->device));
  if (P->nnz)
    B200_CUDA(cudaMemcpyAsync(vals_host, P->f.p, dtype_size(P->dtype) * (size_t)P->nnz, cudaMemcpyDeviceToHost,
                              P->ctx->stream));
  B200_CUDA(cudaStreamSynchronize(P->ctx->stream));
  return check_err(P);
}

int b200_ilu0_info(const b200_ilu0 *P, int *levels_forward, int *levels_backward, int64_t *nnz_lower,
                   int64_t *nnz_upper) {
  B200_REQUIRE(P, "NULL argument");
  if (levels_forward) *levels_forward = P->levels_f;
  if (levels_backward) *levels_backward = P->levels_b;
  if (nnz_lower) *nnz_lower = P->nnz_lower;
  if (nnz_upper) *nnz_upper = P->nnz - P->nnz_lower - P->n;
  return B200_OK;
}

int b200_ilu0_destroy(b200_ilu0 *P) {
  delete P;
  return B200_OK;
}

}  // extern "C"
