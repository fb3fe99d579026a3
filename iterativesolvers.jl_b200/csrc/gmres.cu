// gmres.cu -- orthogonalize_and_normalize! (reference src/orthogonalize.jl), FastHessenberg ldiv!
// (src/hessenberg.jl) and the restarted GMRES engine (src/gmres.jl:57-304).
//
// Data layout: the Arnoldi basis V is n_local x (restart+1), column-major, device-resident (the
// reference hard-codes a host Matrix, src/gmres.jl:5-15; "drop-in" therefore means the whole iterate
// runs here).  H ((restart+1) x restart) and the null-vector residual recurrence are O(restart^2)
// scalars: they live on the host, as in the reference, except for the Givens least-squares solve
// which runs in a single-warp kernel so that y never leaves the device.
//
// Fused classical Gram-Schmidt (CGS / DGKS), 2 launches + 1 scale instead of 2k+3 BLAS calls:
//   k_block_dots : h = V' w        -- all k dots in ONE pass over V and w   ((k+1) n-passes)
//   k_block_axpy : w -= V h ; ||w||^2 fused                                  ((k+2) n-passes)
//   k_scale_dev  : w *= inv(nrm)                                             (2 n-passes)
// Algorithmic bytes per CGS step k: (2k+5) * n * V (SURVEY.md section 8d).
#include <cooperative_groups.h>

#include "blas1.cuh"
#include "spmv.cuh"
#include "linop.cuh"
#include "gmres_core.h"

using namespace b200;

namespace {

constexpr int kThreads = 256;
constexpr int JB = 8;  // columns of V per register block

// VEC consecutive rows per thread: VEC = 2 uses 128-bit (fp64) / 64-bit (fp32) accesses.  Scalar versions of both
// orthogonalisation kernels are latency-bound: wider accesses and explicitly independent column loads double the bytes
// in flight per thread.
template <typename T, int VEC>
__device__ __forceinline__ void ldv(const T *p, T (&v)[VEC]) {
  if constexpr (VEC == 1) v[0] = *p;
  else if constexpr (sizeof(T) == 8) {
    const double2 t = *reinterpret_cast<const double2 *>(p);
    v[0] = t.x; v[1] = t.y;
  } else {
    const float2 t = *reinterpret_cast<const float2 *>(p);
    v[0] = t.x; v[1] = t.y;
  }
}
template <typename T, int VEC>
__device__ __forceinline__ void stv(T *p, const T (&v)[VEC]) {
  if constexpr (VEC == 1) *p = v[0];
  else if constexpr (sizeof(T) == 8) *reinterpret_cast<double2 *>(p) = make_double2(v[0], v[1]);
  else *reinterpret_cast<float2 *>(p) = make_float2(v[0], v[1]);
}

// h[j0+j] = sum_i V[i, j0+j] * w[i]  for all j < k.  Partials: partials[block * kMaxReduceWidth + j].
template <typename T, int VEC>
__global__ void __launch_bounds__(kThreads) k_block_dots(const T *__restrict__ V, int64_t ld, int k,
                                                         const T *__restrict__ w, int64_t n, double *partials,
                                                         unsigned int *ticket, double *__restrict__ out) {
  __shared__ double smem[kThreads / 32][JB];
  __shared__ bool is_last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t nv = n / VEC;   // VEC == 2 is only launched when n is even
  for (int j0 = 0; j0 < k; j0 += JB) {
    const int jn = min(JB, k - j0);
    double acc[JB];
#pragma unroll
    for (int j = 0; j < JB; ++j) acc[j] = 0.0;
    for (int64_t iv = blockIdx.x * (int64_t)kThreads + threadIdx.x; iv < nv; iv += (int64_t)gridDim.x * kThreads) {
      const int64_t i = iv * VEC;
      T wv[VEC], vv[JB][VEC];
      ldv<T, VEC>(w + i, wv);
#pragma unroll
      for (int j = 0; j < JB; ++j)
        if (j < jn) ldv<T, VEC>(V + i + (int64_t)(j0 + j) * ld, vv[j]);
#pragma unroll
      for (int j = 0; j < JB; ++j)
        if (j < jn) {
#pragma unroll
          for (int e = 0; e < VEC; ++e) acc[j] += (double)vv[j][e] * (double)wv[e];
        }
    }
#pragma unroll
    for (int j = 0; j < JB; ++j) acc[j] = warp_sum(acc[j]);
    if (lane == 0) {
#pragma unroll
      for (int j = 0; j < JB; ++j) smem[warp][j] = acc[j];
    }
    __syncthreads();
    if (threadIdx.x < jn) {
      double s = 0.0;
      for (int wv = 0; wv < kThreads / 32; ++wv) s += smem[wv][threadIdx.x];
      partials[(size_t)blockIdx.x * kMaxReduceWidth + j0 + threadIdx.x] = s;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    __threadfence();
    is_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  for (int j = warp; j < k; j += kThreads / 32) {     // warp per column, lanes stride over the block slots (deterministic)
    double s = 0.0;
    for (unsigned int b = lane; b < gridDim.x; b += 32) s += __ldcg(&partials[(size_t)b * kMaxReduceWidth + j]);
    s = warp_sum(s);
    if (lane == 0) out[j] = s;
  }
  if (threadIdx.x == 0) *ticket = 0u;
}

// out[i] = base[i] + sign * sum_j V[i,j] * y[j] ; optionally sum of out[i]^2 -> nrm2_out[0]
template <typename T, bool WITH_NORM, int VEC>
__global__ void __launch_bounds__(kThreads) k_block_axpy(const T *__restrict__ V, int64_t ld, int k,
                                                         const double *__restrict__ y, double sign,
                                                         const T *base, T *out, int64_t n, double *partials,
                                                         unsigned int *ticket, double *nrm2_out) {
  __shared__ T sy[kMaxReduceWidth];
  __shared__ double smem[kThreads / 32];
  for (int j = threadIdx.x; j < k; j += kThreads) sy[j] = (T)(sign * y[j]);
  __syncthreads();
  double acc = 0.0;
  const int64_t nv = n / VEC;
  for (int64_t iv = blockIdx.x * (int64_t)kThreads + threadIdx.x; iv < nv; iv += (int64_t)gridDim.x * kThreads) {
    const int64_t i = iv * VEC;
    T t[VEC];
    ldv<T, VEC>(base + i, t);
    int j = 0;
    for (; j + JB <= k; j += JB) {       // JB independent column loads in flight, then the ordered accumulation
      T vv[JB][VEC];
#pragma unroll
      for (int u = 0; u < JB; ++u) ldv<T, VEC>(V + i + (int64_t)(j + u) * ld, vv[u]);
#pragma unroll
      for (int u = 0; u < JB; ++u) {
#pragma unroll
        for (int e = 0; e < VEC; ++e) t[e] += sy[j + u] * vv[u][e];
      }
    }
    if (j < k) {
      T vv[JB][VEC];
#pragma unroll
      for (int u = 0; u < JB; ++u)
        if (j + u < k) ldv<T, VEC>(V + i + (int64_t)(j + u) * ld, vv[u]);
#pragma unroll
      for (int u = 0; u < JB; ++u)
        if (j + u < k) {
#pragma unroll
          for (int e = 0; e < VEC; ++e) t[e] += sy[j + u] * vv[u][e];
        }
    }
    stv<T, VEC>(out + i, t);
    if (WITH_NORM) {
#pragma unroll
      for (int e = 0; e < VEC; ++e) acc += (double)t[e] * (double)t[e];
    }
  }
  if (WITH_NORM) {
    acc = block_sum<kThreads>(acc, smem);
    double total;
    if (grid_reduce_finish<kThreads>(acc, partials, ticket, smem, &total) && threadIdx.x == 0) nrm2_out[0] = total;
  }
}

// w .*= inv(nrm), nrm = sqrt(*nrm2) read from the device (no host round trip)
template <typename T>
__global__ void __launch_bounds__(kThreads) k_scale_dev(T *__restrict__ w, int64_t n,
                                                        const double *__restrict__ nrm2) {
  const T inv = (T)1 / (T)sqrt(nrm2[0]);
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads)
    w[i] = w[i] * inv;
}

__global__ void k_add_small(double *h, const double *c, int k) {
  for (int j = threadIdx.x; j < k; j += blockDim.x) h[j] += c[j];
}

// LinearAlgebra.givensAlgorithm(f, g) for reals (LAPACK dlartg convention as in Julia's stdlib)
__device__ __forceinline__ void givens(double f, double g, double &c, double &s, double &r) {
  if (g == 0.0) { c = 1.0; s = 0.0; r = f; return; }
  if (f == 0.0) { c = 0.0; s = 1.0; r = g; return; }
  r = hypot(f, g);
  c = f / r;
  s = g / r;
  if (fabs(f) > fabs(g) && c < 0.0) { c = -c; s = -s; r = -r; }
}

// ldiv!(FastHessenberg(H), rhs): one warp; lanes run over the columns j of each rotation.  H and rhs are NOT
// __restrict__: lanes read what other lanes wrote across __syncwarp(), and a restrict-qualified pointer lets the
// compiler forward a lane's own earlier store past the barrier (stale rhs entries in the back substitution).
__global__ void k_hessenberg_ldiv(double *H, int ldh, int m, double *rhs) {
  const int lane = threadIdx.x;
  for (int i = 0; i < m; ++i) {                                   // src/hessenberg.jl:24
    double c, s, r;
    givens(H[i + i * ldh], H[i + 1 + i * ldh], c, s, r);          // :25
    __syncwarp();
    for (int j = i + 1 + lane; j < m; j += 32) {                  // :31-35
      const double a = H[i + j * ldh], b = H[i + 1 + j * ldh];
      H[i + j * ldh] = c * a + s * b;
      H[i + 1 + j * ldh] = -s * a + c * b;
    }
    if (lane == 0) {
      H[i + i * ldh] = c * H[i + i * ldh] + s * H[i + 1 + i * ldh];  // :28
      const double a = rhs[i], b = rhs[i + 1];                    // :38-40
      rhs[i] = c * a + s * b;
      rhs[i + 1] = -s * a + c * b;
    }
    __syncwarp();
  }
  // UpperTriangular solve (:44-45), column-oriented back substitution
  for (int j = m - 1; j >= 0; --j) {
    if (lane == 0) rhs[j] = rhs[j] / H[j + j * ldh];
    __syncwarp();
    const double xj = rhs[j];
    for (int i = lane; i < j; i += 32) rhs[i] -= H[i + j * ldh] * xj;
    __syncwarp();
  }
}


// ------------------------------------------------------------------------------------------------
// orthogonalize_and_normalize!(V[:, 1:k], w, h, ClassicalGramSchmidt() / DGKS()) in ONE cooperative launch
// (reference src/orthogonalize.jl:41-51, :13-39) and, for the GMRES engine, the scalar part of the inner iteration
// (src/gmres.jl:68-104: H column, null-vector residual recurrence, stopping test, Givens least-squares solve at the end
// of a cycle) in its finishing thread.  Every scalar lives in the device GmScal (gmres_core.h), so the host neither
// reads nor decides anything between the launches of a restart cycle:
//
//   phase 1  h = V' w: block partial sums of the k dots                                  grid.sync
//   phase 2  block j sums column j of the partials in a fixed order -> dst[j]            grid.sync
//   phase 3  w -= V dst, block partial of ||w||^2                                        grid.sync
//   phase 4  block 0: ||w||; DGKS: projection size and the re-orthogonalisation test (:20-33); when no further round
//            is needed and do_step: gm_step                                              grid.sync
//   (DGKS: back to phase 1 with dst = correction while nrm < eta * projection_size)
//   phase 5  w *= inv(nrm)
//
// Every thread sweeps the same rows in phases 1, 3 and 5.  HBM traffic is that of the three separate kernels
// ((2k+5) n V, SURVEY 8d); what goes away are two launches, the allreduce placeholders and the host round trip.
// `gate_mask`: the launch is a no-op when (s->flags & gate_mask) != 0 -- GMRES enqueues a whole restart cycle ahead of
// the device-side stopping test.
namespace cgx = cooperative_groups;

// the scalar sections run in ONE thread: kept out of line so that their locals do not set the register count (and with it
// the occupancy) of the streaming phases
__device__ __noinline__ void orth_scalar_section(GmScal *s, int k, int dgks, int round, int do_step, double nrm2) {
  s->nrm2 = nrm2;
  s->nrm = sqrt(nrm2);
  s->k = k;
  if (dgks) {
    if (round == 0) gm_dgks_first(s);      // projection_size = norm(h); nrm < eta * projection_size ?  :20-26
    else gm_dgks_next(s);                  // h .+= correction; projection_size = norm(correction)    :28-31
  } else {
    s->reorth = 0;
  }
  if (!s->reorth && do_step) gm_step(s);   // src/gmres.jl:68-104
}

template <typename T, int VEC>
__global__ void __launch_bounds__(kThreads, 2) k_orth_fused(const T *__restrict__ V, int64_t ld, int k, T *w, int64_t n,
                                                         int dgks, double *partials, GmScal *s, int do_step,
                                                         int gate_mask) {
  if (s->flags & gate_mask) return;             // uniform over the grid: nobody reaches a grid.sync
  cgx::grid_group grid = cgx::this_grid();
  __shared__ double smem[kThreads / 32][JB];
  __shared__ double sred[kThreads / 32];
  __shared__ T sy[kMaxReduceWidth];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t nv = n / VEC;                   // VEC == 2 is only launched when n is even
  double *dst = s->h;
  for (int round = 0;; ++round) {
    // ---- phase 1: dots (register block of JB columns, as k_block_dots)
    for (int j0 = 0; j0 < k; j0 += JB) {
      const int jn = min(JB, k - j0);
      double acc[JB];
#pragma unroll
      for (int j = 0; j < JB; ++j) acc[j] = 0.0;
      for (int64_t iv = blockIdx.x * (int64_t)kThreads + threadIdx.x; iv < nv; iv += (int64_t)gridDim.x * kThreads) {
        const int64_t i = iv * VEC;
        T wv[VEC], vv[JB][VEC];
        ldv<T, VEC>(w + i, wv);
#pragma unroll
        for (int j = 0; j < JB; ++j)
          if (j < jn) ldv<T, VEC>(V + i + (int64_t)(j0 + j) * ld, vv[j]);
#pragma unroll
        for (int j = 0; j < JB; ++j)
          if (j < jn) {
#pragma unroll
            for (int e = 0; e < VEC; ++e) acc[j] += (double)vv[j][e] * (double)wv[e];
          }
      }
#pragma unroll
      for (int j = 0; j < JB; ++j) acc[j] = warp_sum(acc[j]);
      if (lane == 0) {
#pragma unroll
        for (int j = 0; j < JB; ++j) smem[warp][j] = acc[j];
      }
      __syncthreads();
      if (threadIdx.x < jn) {
        double t = 0.0;
        for (int wv = 0; wv < kThreads / 32; ++wv) t += smem[wv][threadIdx.x];
        partials[(size_t)blockIdx.x * kMaxReduceWidth + j0 + threadIdx.x] = t;
      }
      __syncthreads();
    }
    __threadfence();
    grid.sync();
    // ---- phase 2: column j of the partials, summed by block j in slot order (deterministic)
    for (int j = blockIdx.x; j < k; j += gridDim.x) {
      double a = 0.0;
      for (unsigned int b = threadIdx.x; b < gridDim.x; b += kThreads) a += __ldcg(&partials[(size_t)b * kMaxReduceWidth + j]);
      a = block_sum<kThreads>(a, sred);
      if (threadIdx.x == 0) dst[j] = a;
    }
    __threadfence();
    grid.sync();
    // ---- phase 3: w -= V dst ; ||w||^2
    for (int j = threadIdx.x; j < k; j += kThreads) sy[j] = (T)(-__ldcg(&dst[j]));
    __syncthreads();
    double nacc = 0.0;
    for (int64_t iv = blockIdx.x * (int64_t)kThreads + threadIdx.x; iv < nv; iv += (int64_t)gridDim.x * kThreads) {
      const int64_t i = iv * VEC;
      T t[VEC];
      ldv<T, VEC>(w + i, t);
      int j = 0;
      for (; j + JB <= k; j += JB) {
        T vv[JB][VEC];
#pragma unroll
        for (int u = 0; u < JB; ++u) ldv<T, VEC>(V + i + (int64_t)(j + u) * ld, vv[u]);
#pragma unroll
        for (int u = 0; u < JB; ++u) {
#pragma unroll
          for (int e = 0; e < VEC; ++e) t[e] += sy[j + u] * vv[u][e];
        }
      }
      if (j < k) {
        T vv[JB][VEC];
#pragma unroll
        for (int u = 0; u < JB; ++u)
          if (j + u < k) ldv<T, VEC>(V + i + (int64_t)(j + u) * ld, vv[u]);
#pragma unroll
        for (int u = 0; u < JB; ++u)
          if (j + u < k) {
#pragma unroll
            for (int e = 0; e < VEC; ++e) t[e] += sy[j + u] * vv[u][e];
          }
      }
      stv<T, VEC>(w + i, t);
#pragma unroll
      for (int e = 0; e < VEC; ++e) nacc += (double)t[e] * (double)t[e];
    }
    nacc = block_sum<kThreads>(nacc, sred);
    if (threadIdx.x == 0) partials[(size_t)blockIdx.x * kMaxReduceWidth] = nacc;
    __threadfence();
    grid.sync();
    // ---- phase 4: the norm and everything scalar
    if (blockIdx.x == 0) {
      double a = 0.0;
      for (unsigned int b = threadIdx.x; b < gridDim.x; b += kThreads) a += __ldcg(&partials[(size_t)b * kMaxReduceWidth]);
      a = block_sum<kThreads>(a, sred);
      if (threadIdx.x == 0) {
        orth_scalar_section(s, k, dgks, round, do_step, a);
        __threadfence();
      }
    }
    grid.sync();
    if (!*(volatile int *)&s->reorth) break;
    dst = s->corr;
  }
  // ---- phase 5: w .*= inv(nrm)  (:36 / :48); nrm == 0 (lucky breakdown) gives the reference's NaNs
  const T inv = (T)1 / (T)(*(volatile double *)&s->nrm);
  for (int64_t iv = blockIdx.x * (int64_t)kThreads + threadIdx.x; iv < nv; iv += (int64_t)gridDim.x * kThreads) {
    const int64_t i = iv * VEC;
    T t[VEC];
    ldv<T, VEC>(w + i, t);
#pragma unroll
    for (int e = 0; e < VEC; ++e) t[e] = t[e] * inv;
    stv<T, VEC>(w + i, t);
  }
}

__global__ void k_gm_set_beta(GmScal *s, const double *sumsq, int clear_mask) {
  gm_set_beta(s, sumsq[0]);
  s->flags &= ~clear_mask;
}

int gridv(const b200_ctx *ctx, int64_t n) { return stream_grid(ctx, n, kThreads * 2, 8); }

// grid = one full wave of the kernel's real occupancy (grid-stride loops: a partial last wave is pure tail)
template <typename K>
int grid_one_wave(const b200_ctx *ctx, K kernel, int64_t n) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, 0) != cudaSuccess || per_sm < 1)
    per_sm = 2;
  return stream_grid(ctx, n, kThreads * 2, per_sm);
}

// two rows per thread when every column start stays 2*sizeof(T)-aligned
template <typename T>
bool can_vec2(int64_t n, int64_t ld, std::initializer_list<const void *> ptrs) {
  if ((n & 1) || (ld & 1)) return false;
  for (const void *p : ptrs)
    if (reinterpret_cast<uintptr_t>(p) % (2 * sizeof(T))) return false;
  return true;
}

template <typename T>
int block_dots(b200_ctx *ctx, const T *V, int64_t ld, int k, const T *w, int64_t n, double *out_dev) {
  const bool v2 = can_vec2<T>(n, ld, {V, w});
  // chunks of at most kMaxReduceWidth columns
  for (int j0 = 0; j0 < k; j0 += kMaxReduceWidth) {
    const int kk = std::min(kMaxReduceWidth, k - j0);
    ProfScope prof(ctx, 1);
    auto kern = v2 ? k_block_dots<T, 2> : k_block_dots<T, 1>;
    kern<<<grid_one_wave(ctx, kern, n), kThreads, 0, ctx->stream>>>(V + (int64_t)j0 * ld, ld, kk, w, n,
                                                                    ctx->red.partials, ctx->red.ticket, out_dev + j0);
    ctx->launches++;
  }
  B200_CUDA(cudaPeekAtLastError());
  return allreduce_sum_dev(ctx, out_dev, k);
}

template <typename T>
int block_axpy(b200_ctx *ctx, const T *V, int64_t ld, int k, const double *y_dev, double sign, const T *base, T *out,
               int64_t n, double *nrm2_dev) {
  for (int j0 = 0; j0 < k || j0 == 0; j0 += kMaxReduceWidth) {
    const int kk = std::min(kMaxReduceWidth, k - j0);
    const bool last = j0 + kMaxReduceWidth >= k;
    const T *src = j0 == 0 ? base : out;
    ProfScope prof(ctx, 1);
    const bool v2 = can_vec2<T>(n, ld, {V, src, out});
    const T *Vj = V + (int64_t)j0 * ld;
    if (last && nrm2_dev) {
      auto kern = v2 ? k_block_axpy<T, true, 2> : k_block_axpy<T, true, 1>;
      kern<<<grid_one_wave(ctx, kern, n), kThreads, 0, ctx->stream>>>(Vj, ld, kk, y_dev + j0, sign, src, out, n,
                                                                      ctx->red.partials, ctx->red.ticket, nrm2_dev);
    } else {
      auto kern = v2 ? k_block_axpy<T, false, 2> : k_block_axpy<T, false, 1>;
      kern<<<grid_one_wave(ctx, kern, n), kThreads, 0, ctx->stream>>>(Vj, ld, kk, y_dev + j0, sign, src, out, n,
                                                                      nullptr, nullptr, nullptr);
    }
    ctx->launches++;
    if (last) break;
  }
  B200_CUDA(cudaPeekAtLastError());
  if (nrm2_dev) B200_TRY(allreduce_sum_dev(ctx, nrm2_dev, 1));
  return B200_OK;
}

template <typename T>
int scale_dev(b200_ctx *ctx, T *w, int64_t n, const double *nrm2_dev) {
  ProfScope prof(ctx, 2);
  k_scale_dev<T><<<gridv(ctx, n), kThreads, 0, ctx->stream>>>(w, n, nrm2_dev);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

// one cooperative launch of k_orth_fused (single-GPU contexts, CGS / DGKS, 1 <= k <= 64)
template <typename T>
int orth_fused_launch(b200_ctx *ctx, const T *V, int64_t ld, int k, T *w, int64_t n, int dgks, GmScal *s, int do_step,
                      int gate_mask) {
  const bool v2 = can_vec2<T>(n, ld, {V, w});
  auto kern = v2 ? k_orth_fused<T, 2> : k_orth_fused<T, 1>;
  static int occ[2][64];                                   // blocks per SM of the two instantiations, per device
  int &per_sm = occ[v2 ? 1 : 0][ctx->device & 63];
  if (per_sm == 0) {
    int q = 0;
    B200_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&q, kern, kThreads, 0));
    per_sm = q < 1 ? 1 : q;
  }
  const int grid = stream_grid(ctx, n, kThreads * 2, per_sm);   // <= sm_count * per_sm: all blocks co-resident (grid.sync)
  double *partials = ctx->red.partials;
  void *args[] = {(void *)&V, (void *)&ld, (void *)&k, (void *)&w, (void *)&n, (void *)&dgks, (void *)&partials, (void *)&s,
                  (void *)&do_step, (void *)&gate_mask};
  ProfScope prof(ctx, 1);
  B200_CUDA(cudaLaunchCooperativeKernel((const void *)kern, dim3(grid), dim3(kThreads), args, 0, ctx->stream));
  ctx->launches++;
  return B200_OK;
}

// orthogonalize_and_normalize!(V[:,1:k], w, h, method): h_host (k doubles) out, returns nrm.
// Scratch: ctx->d_scalars[0..63] = h, [64..127] = correction, [200] = ||w||^2
template <typename T>
int orth_impl(b200_ctx *ctx, int64_t n, const T *V, int64_t ld, int k, T *w, double *h_host, int method,
              double *nrm_out) {
  double *d_h = ctx->d_scalars, *d_c = ctx->d_scalars + 64, *d_n = ctx->d_scalars + 200;
  B200_REQUIRE(k >= 0 && k <= 64, "orthogonalize_and_normalize!: k=%d exceeds 64 basis vectors", k);
  double nrm2 = 0.0;
  if (ctx->world == 1 && method != B200_ORTH_MGS && k >= 1 && ctx->opt_orth_fused) {
    // one cooperative launch; h, the correction rounds and the norm stay in a device GmScal until they are read back
    if (!ctx->orth_scal) B200_CUDA(cudaMalloc(&ctx->orth_scal, sizeof(GmScal)));
    GmScal *s = (GmScal *)ctx->orth_scal;
    B200_CUDA(cudaMemsetAsync(&s->flags, 0, sizeof(int), ctx->stream));
    B200_TRY(orth_fused_launch<T>(ctx, V, ld, k, w, n, method == B200_ORTH_DGKS ? 1 : 0, s, 0, 0));
    B200_CUDA(cudaMemcpyAsync(ctx->h_scalars, s->h, sizeof(double) * k, cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA(cudaMemcpyAsync(ctx->h_scalars + 64, &s->nrm, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA(cudaStreamSynchronize(ctx->stream));
    for (int j = 0; j < k; ++j) h_host[j] = ctx->h_scalars[j];
    *nrm_out = ctx->h_scalars[64];
    return B200_OK;
  }
  if (method == B200_ORTH_MGS) {
    // reference src/orthogonalize.jl:67-79: k sequential (dot ; axpy) pairs
    for (int i = 0; i < k; ++i) {
      B200_TRY(block_dots<T>(ctx, V + (int64_t)i * ld, ld, 1, w, n, d_h + i));                       // :71
      B200_TRY(block_axpy<T>(ctx, V + (int64_t)i * ld, ld, 1, d_h + i, -1.0, w, w, n, i == k - 1 ? d_n : nullptr));  // :72
    }
    if (k == 0) {
      B200_TRY(dot_dev(ctx, n, w, w, dtype_of<T>::value, d_n));
      B200_TRY(allreduce_sum_dev(ctx, d_n, 1));
    }
    B200_CUDA(cudaMemcpyAsync(ctx->h_scalars, d_h, sizeof(double) * std::max(k, 1), cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA(cudaMemcpyAsync(ctx->h_scalars + 64, d_n, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA(cudaStreamSynchronize(ctx->stream));
    for (int j = 0; j < k; ++j) h_host[j] = ctx->h_scalars[j];
    nrm2 = ctx->h_scalars[64];
  } else {
    if (k > 0) {
      B200_TRY(block_dots<T>(ctx, V, ld, k, w, n, d_h));                       // mul!(h, V', w)         :15/:43
      B200_TRY(block_axpy<T>(ctx, V, ld, k, d_h, -1.0, w, w, n, d_n));         // mul!(w, V, h, -1, 1)   :16/:44 + norm :17/:45
    } else {
      B200_TRY(dot_dev(ctx, n, w, w, dtype_of<T>::value, d_n));
      B200_TRY(allreduce_sum_dev(ctx, d_n, 1));
    }
    B200_CUDA(cudaMemcpyAsync(ctx->h_scalars, d_h, sizeof(double) * std::max(k, 1), cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA(cudaMemcpyAsync(ctx->h_scalars + 64, d_n, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA(cudaStreamSynchronize(ctx->stream));
    for (int j = 0; j < k; ++j) h_host[j] = ctx->h_scalars[j];
    nrm2 = ctx->h_scalars[64];
    if (method == B200_ORTH_DGKS && k > 0) {
      const double eta = 1.0 / sqrt(2.0);                                      // :20
      double proj = 0.0;
      for (int j = 0; j < k; ++j) proj += h_host[j] * h_host[j];
      proj = sqrt(proj);                                                       // :22
      int guard = 0;
      while (sqrt(nrm2) < eta * proj && guard++ < 8) {                          // :26
        B200_TRY(block_dots<T>(ctx, V, ld, k, w, n, d_c));                     // correction = V' w     :27
        B200_TRY(block_axpy<T>(ctx, V, ld, k, d_c, -1.0, w, w, n, d_n));       // w -= V correction     :30, norm :32
        k_add_small<<<1, 64, 0, ctx->stream>>>(d_h, d_c, k);                   // h .+= correction      :31
        ctx->launches++;
        B200_CUDA(cudaMemcpyAsync(ctx->h_scalars, d_c, sizeof(double) * k, cudaMemcpyDeviceToHost, ctx->stream));
        B200_CUDA(cudaMemcpyAsync(ctx->h_scalars + 64, d_n, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
        B200_CUDA(cudaStreamSynchronize(ctx->stream));
        proj = 0.0;
        for (int j = 0; j < k; ++j) {
          proj += ctx->h_scalars[j] * ctx->h_scalars[j];
          h_host[j] += ctx->h_scalars[j];
        }
        proj = sqrt(proj);                                                     // :28
        nrm2 = ctx->h_scalars[64];
      }
    }
  }
  B200_TRY(scale_dev<T>(ctx, w, n, d_n));                                      // w .*= inv(nrm)  :36/:48/:76
  *nrm_out = sqrt(nrm2);
  return B200_OK;
}

// ------------------------------------------------------------------------------------------------
// GMRES engine
// ------------------------------------------------------------------------------------------------
template <typename T>
struct Gmres {
  b200_ctx *ctx;
  const b200_csr *A;
  int64_t n;
  int restart;
  T *V;       // n x (restart+1)
  T *Ax;      // work vector
  T *x;
  const T *b;
  const T *pl, *pr;  // Jacobi diagonals or NULL
  std::vector<double> H, nullvec;  // host, column-major (restart+1) x restart
  double *d_H, *d_rhs;             // device copies for the LS solve
  int ldh;

  T *col(int j) { return V + (int64_t)j * n; }

  // init! (src/gmres.jl:235-255): V[:,1] = Pl \ (b - A x); returns beta and normalises
  int init(bool initially_zero, double *beta) {
    const int dt = dtype_of<T>::value;
    T *v0 = col(0);
    B200_TRY(copy(ctx, n, b, v0, dt));                                   // :241
    if (!initially_zero) {
      B200_TRY(spmv(ctx, A, x, Ax));                                     // :245
      B200_TRY(axpby(ctx, n, -1.0, Ax, 1.0, v0, dt));                    // :246
    }
    if (pl) B200_TRY(jacobi_ldiv(ctx, n, pl, v0, v0, dt));               // :249
    double *d_n = ctx->d_scalars + 200;
    B200_TRY(dot_dev(ctx, n, v0, v0, dt, d_n));                          // :252
    B200_TRY(allreduce_sum_dev(ctx, d_n, 1));
    B200_TRY(scale_dev<T>(ctx, v0, n, d_n));                             // :253
    double nn;
    B200_TRY(read_scalars(ctx, d_n, 1, &nn));
    *beta = sqrt(nn);
    return B200_OK;
  }

  // expand! (src/gmres.jl:285-304)
  int expand(int k) {  // k is 1-based as in the reference: V[:,k+1] = Pl \ (A (Pr \ V[:,k]))
    const int dt = dtype_of<T>::value;
    T *next = col(k), *cur = col(k - 1);
    if (!pr) {
      {
        ProfScope prof(ctx, 0);
        B200_TRY(spmv(ctx, A, cur, next));                               // :287/:293
      }
      if (pl) B200_TRY(jacobi_ldiv(ctx, n, pl, next, next, dt));         // :294
    } else {
      B200_TRY(jacobi_ldiv(ctx, n, pr, cur, next, dt));                  // :300
      B200_TRY(spmv(ctx, A, next, Ax));                                  // :301
      B200_TRY(copy(ctx, n, Ax, next, dt));                              // :302
      if (pl) B200_TRY(jacobi_ldiv(ctx, n, pl, next, next, dt));         // :303
    }
    return B200_OK;
  }

  // solve_least_squares! + update_solution! (src/gmres.jl:262-283), k as in the reference (k-1 columns)
  int solve_and_update(int k, double beta) {
    const int m = k - 1;
    if (m <= 0) return B200_OK;
    std::vector<double> rhs(k, 0.0);
    rhs[0] = beta;                                                        // :265
    B200_CUDA(cudaMemcpyAsync(d_H, H.data(), sizeof(double) * ldh * restart, cudaMemcpyHostToDevice, ctx->stream));
    B200_CUDA(cudaMemcpyAsync(d_rhs, rhs.data(), sizeof(double) * k, cudaMemcpyHostToDevice, ctx->stream));
    k_hessenberg_ldiv<<<1, 32, 0, ctx->stream>>>(d_H, ldh, m, d_rhs);     // :267-268
    B200_LAUNCH_CHECK(ctx);
    // the reference's ldiv! mutates arnoldi.H in place; mirror that on the host copy
    B200_CUDA(cudaMemcpyAsync(H.data(), d_H, sizeof(double) * ldh * restart, cudaMemcpyDeviceToHost, ctx->stream));
    if (!pr) {
      B200_TRY(block_axpy<T>(ctx, V, n, m, d_rhs, 1.0, x, x, n, nullptr));    // x += V[:,1:k-1] y   :275
    } else {
      B200_TRY(fill(ctx, n, 0.0, Ax, dtype_of<T>::value));
      B200_TRY(block_axpy<T>(ctx, V, n, m, d_rhs, 1.0, Ax, Ax, n, nullptr));  // :280
      B200_TRY(jacobi_ldiv(ctx, n, pr, Ax, Ax, dtype_of<T>::value));          // :281
      B200_TRY(axpby(ctx, n, 1.0, Ax, 1.0, x, dtype_of<T>::value));           // :282
    }
    B200_CUDA(cudaStreamSynchronize(ctx->stream));
    return B200_OK;
  }
};

template <typename T>
int gmres_impl(b200_ctx *ctx, const b200_csr *A, T *x, const T *b, const b200_gmres_opts *o, b200_result *res,
               double *resnorm_host, int64_t resnorm_cap) {
  const int64_t n = A->m_local;
  const double eps = sizeof(T) == 8 ? 2.220446049250313e-16 : 1.1920928955078125e-07;
  const double reltol = o->reltol < 0 ? sqrt(eps) : o->reltol;
  const int64_t maxiter = o->maxiter < 0 ? A->n_global : o->maxiter;
  const int restart = o->restart > 0 ? o->restart : (int)std::min<int64_t>(20, A->n_global);
  B200_REQUIRE(restart <= 64, "restart=%d: this version supports restart <= 64", restart);
  const int method = o->orth_meth;

  Gmres<T> g;
  g.ctx = ctx;
  g.A = A;
  g.n = n;
  g.restart = restart;
  g.x = x;
  g.b = b;
  g.pl = o->Pl.kind == B200_PREC_JACOBI ? (const T *)o->Pl.diag : nullptr;
  g.pr = o->Pr.kind == B200_PREC_JACOBI ? (const T *)o->Pr.diag : nullptr;
  g.ldh = restart + 1;
  g.H.assign((size_t)g.ldh * restart, 0.0);                               // zeros(T, order+1, order) :14
  g.nullvec.assign(restart + 1, 1.0);                                     // ones(T, order+1)         :27
  const size_t vec_bytes = align_up(sizeof(T) * (size_t)std::max<int64_t>(n, 1), 256);
  void *ws = nullptr;
  B200_TRY(ws_get(ctx, vec_bytes * (restart + 2) + 65536, &ws));
  g.V = (T *)ws;
  // columns must be contiguous with leading dimension n (not the padded size)
  g.Ax = (T *)((char *)ws + align_up(sizeof(T) * (size_t)n * (restart + 1), 256));
  g.d_H = (double *)((char *)g.Ax + vec_bytes);
  g.d_rhs = g.d_H + (size_t)g.ldh * restart;
  B200_REQUIRE((char *)(g.d_rhs + g.ldh) <= (char *)ws + ctx->ws_bytes, "internal: GMRES workspace too small");
  B200_CUDA(cudaMemsetAsync(g.V, 0, sizeof(T) * (size_t)n * (restart + 1), ctx->stream));  // zeros(T, n, order+1) :13

  // gmres_iterable! (src/gmres.jl:108-136)
  int64_t mv_products = o->initially_zero ? 1 : 0;                        // :122 (sic)
  double current, accumulator = 1.0, beta_res;
  B200_TRY(g.init(o->initially_zero != 0, &current));                     // :126
  beta_res = current;                                                     // init_residual! :257-260
  const double tol = std::max(reltol * current, o->abstol);               // :129
  double beta = current;                                                  // g.beta  :133
  int k = 1;
  int64_t iteration = 0, n_hist = 0;
  bool breakdown = false;
  auto done = [&](int64_t it) { return it >= maxiter || current <= tol; };  // :55
  std::vector<double> h(restart + 1);

  while (!done(iteration)) {                                              // :59
    B200_TRY(g.expand(k));                                                // :63
    mv_products += 1;                                                     // :65
    double nrm = 0.0;
    B200_TRY(orth_impl<T>(ctx, n, g.V, n, k, g.col(k), h.data(), method, &nrm));  // :68-73
    for (int j = 0; j < k; ++j) g.H[j + (size_t)(k - 1) * g.ldh] = h[j];
    g.H[k + (size_t)(k - 1) * g.ldh] = nrm;
    // update_residual! (:224-233)
    if (nrm == 0.0) {
      current = 0.0;
    } else {
      double d = 0.0;
      for (int j = 0; j < k; ++j) d += g.nullvec[j] * g.H[j + (size_t)(k - 1) * g.ldh];
      g.nullvec[k] = -(d / nrm);
      accumulator += g.nullvec[k] * g.nullvec[k];
      current = beta_res / sqrt(accumulator);
    }
    if (!(current == current)) breakdown = true;
    k += 1;                                                               // :78
    if (k == restart + 1 || done(iteration + 1)) {                        // :82
      B200_TRY(g.solve_and_update(k, beta));                              // :85-88
      k = 1;                                                              // :90
      if (!done(iteration)) {                                             // :93 (sic)
        B200_TRY(g.init(false, &beta));                                   // :96
        accumulator = 1.0;                                                // :99 (current is NOT reset)
        beta_res = beta;
        mv_products += 1;                                                 // :101
      }
    }
    iteration += 1;
    if (resnorm_host && n_hist < resnorm_cap) resnorm_host[n_hist++] = current;  // push!(:resnorm) :211
    if (breakdown) break;
  }
  if (res) {
    res->iters = iteration;
    res->mvps = mv_products;                                              // history.mvps = iterable.mv_products :210
    res->isconverged = current <= tol;                                    // :218
    res->status = breakdown ? B200_ERR_BREAKDOWN : 0;
    res->tol = tol;
    res->residual = current;
    res->n_resnorm = n_hist;
  }
  return B200_OK;
}


// ------------------------------------------------------------------------------------------------
// gmres! with a device-resident restart cycle (single GPU, CGS / DGKS): H, the null-vector residual recurrence, the
// stopping test and the Givens least-squares solve live in a device GmScal (gmres_core.h: gm_step is the scalar part
// of src/gmres.jl:68-104, run by the finishing thread of k_orth_fused).  The host enqueues expand! + orthogonalize for
// the whole cycle -- launches behind the point where the cycle closes (restart reached, converged, maxiter) are no-ops
// gated on s->flags -- and synchronises ONCE per cycle to learn how many columns the solution update takes.
// ------------------------------------------------------------------------------------------------
template <typename T>
int gmres_impl_fused(b200_ctx *ctx, const b200_csr *A, T *x, const T *b, const b200_gmres_opts *o, b200_result *res,
                     double *resnorm_host, int64_t resnorm_cap) {
  const int64_t n = A->m_local;
  const int dt = dtype_of<T>::value;
  const double eps = sizeof(T) == 8 ? 2.220446049250313e-16 : 1.1920928955078125e-07;
  const double reltol = o->reltol < 0 ? sqrt(eps) : o->reltol;
  const int64_t maxiter = o->maxiter < 0 ? A->n_global : o->maxiter;
  const int restart = o->restart > 0 ? o->restart : (int)std::min<int64_t>(20, A->n_global);
  B200_REQUIRE(restart <= kGmMaxRestart, "restart=%d: this version supports restart <= 64", restart);
  const int dgks = o->orth_meth == B200_ORTH_DGKS ? 1 : 0;
  const T *pl = o->Pl.kind == B200_PREC_JACOBI ? (const T *)o->Pl.diag : nullptr;
  const T *pr = o->Pr.kind == B200_PREC_JACOBI ? (const T *)o->Pr.diag : nullptr;
  const int64_t hist_cap = resnorm_host ? std::min<int64_t>(resnorm_cap, maxiter) : 0;   // reserve!(history, :resnorm, maxiter) :198

  const size_t vec_bytes = align_up(sizeof(T) * (size_t)std::max<int64_t>(n, 1), 256);
  const size_t v_bytes = align_up(sizeof(T) * (size_t)std::max<int64_t>(n, 1) * (restart + 1), 256);
  const size_t s_bytes = align_up(sizeof(GmScal), 256);
  void *ws = nullptr;
  B200_TRY(ws_get(ctx, v_bytes + vec_bytes + s_bytes + align_up(sizeof(double) * (size_t)std::max<int64_t>(hist_cap, 1), 256), &ws));
  T *V = (T *)ws;                                            // n x (restart+1), leading dimension n
  T *Ax = (T *)((char *)ws + v_bytes);
  GmScal *s = (GmScal *)((char *)Ax + vec_bytes);
  double *d_hist = (double *)((char *)s + s_bytes);
  double *d_n = ctx->d_scalars + 200;
  auto col = [&](int j) { return V + (int64_t)j * n; };
  {
    std::unique_ptr<GmScal> h(new GmScal);
    memset(h.get(), 0, sizeof(GmScal));
    for (int i = 0; i < kGmLdh; ++i) h->nullvec[i] = 1.0;                 // ones(T, order+1) :27
    h->accumulator = h->current = h->beta_res = h->beta = 1.0;
    h->abstol = o->abstol;
    h->reltol = reltol;
    h->maxiter = maxiter;
    h->hist = hist_cap > 0 ? d_hist : nullptr;
    h->hist_cap = hist_cap;
    h->k = 1;
    h->restart = restart;
    h->first = 1;
    B200_CUDA(cudaMemcpyAsync(s, h.get(), sizeof(GmScal), cudaMemcpyHostToDevice, ctx->stream));
    B200_CUDA(cudaStreamSynchronize(ctx->stream));                        // h goes out of scope
  }
  B200_CUDA(cudaMemsetAsync(V, 0, sizeof(T) * (size_t)n * (restart + 1), ctx->stream));   // zeros(T, n, order+1) :13

  // init! (:235-255) with beta, tol and the first stopping test formed on the device
  auto init = [&](bool zero, int clear_mask) -> int {
    T *v0 = col(0);
    B200_TRY(copy(ctx, n, b, v0, dt));                                   // :241
    if (!zero) {
      B200_TRY(spmv(ctx, A, x, Ax));                                     // :245
      B200_TRY(axpby(ctx, n, -1.0, Ax, 1.0, v0, dt));                    // :246
    }
    if (pl) B200_TRY(jacobi_ldiv(ctx, n, pl, v0, v0, dt));               // :249
    B200_TRY(dot_dev(ctx, n, v0, v0, dt, d_n));                          // :252
    k_gm_set_beta<<<1, 1, 0, ctx->stream>>>(s, d_n, clear_mask);         // :126-133 / :96-99
    ctx->launches++;
    B200_TRY(scale_dev<T>(ctx, v0, n, d_n));                             // :253
    return B200_OK;
  };
  const int kGate = GM_FIN | GM_DONE;
  // expand! (:285-304); k 1-based: V[:, k+1] = Pl \ (A (Pr \ V[:, k])).  The product is gated, the cheap vector passes are not
  auto expand = [&](int k) -> int {
    T *next = col(k), *cur = col(k - 1);
    if (!pr) {
      {
        ProfScope prof(ctx, 0);
        B200_TRY(spmv_gated(ctx, A, cur, next, &s->flags, kGate));       // :287/:293
        ctx->launches++;
      }
      if (pl) B200_TRY(jacobi_ldiv(ctx, n, pl, next, next, dt));         // :294
    } else {
      B200_TRY(jacobi_ldiv(ctx, n, pr, cur, next, dt));                  // :300
      B200_TRY(spmv_gated(ctx, A, next, Ax, &s->flags, kGate));          // :301
      ctx->launches++;
      B200_TRY(copy(ctx, n, Ax, next, dt));                              // :302
      if (pl) B200_TRY(jacobi_ldiv(ctx, n, pl, next, next, dt));         // :303
    }
    return B200_OK;
  };
  struct Tail { double current, tol; long long iteration, n_hist; int k, m, flags; } t;
  auto read_tail = [&]() -> int {
    // the scalars the host steers by; one small copy each, one synchronisation
    B200_CUDA(cudaMemcpyAsync(&ctx->h_scalars[0], &s->current, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA(cudaMemcpyAsync(&ctx->h_scalars[1], &s->tol, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA(cudaMemcpyAsync(&ctx->h_scalars[2], &s->iteration, sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA(cudaMemcpyAsync(&ctx->h_scalars[3], &s->n_hist, sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA(cudaMemcpyAsync(&ctx->h_scalars[4], &s->k, 4 * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));   // k, restart, m, flags
    B200_CUDA(cudaStreamSynchronize(ctx->stream));
    t.current = ctx->h_scalars[0];
    t.tol = ctx->h_scalars[1];
    memcpy(&t.iteration, &ctx->h_scalars[2], sizeof(long long));
    memcpy(&t.n_hist, &ctx->h_scalars[3], sizeof(long long));
    int q[4];
    memcpy(q, &ctx->h_scalars[4], sizeof(q));
    t.k = q[0];
    t.m = q[2];
    t.flags = q[3];
    return B200_OK;
  };

  int64_t mv_products = o->initially_zero ? 1 : 0;                        // :122 (sic)
  B200_TRY(init(o->initially_zero != 0, 0));                              // :126
  B200_TRY(read_tail());
  while (!(t.flags & GM_DONE)) {                                          // :59
    const int64_t before = t.iteration;
    const int64_t left = maxiter - t.iteration;
    const int kc = (int)std::min<int64_t>(restart, left);                 // the cycle closes at the latest after kc steps
    for (int k = 1; k <= kc; ++k) {
      B200_TRY(expand(k));                                                // :63
      B200_TRY(orth_fused_launch<T>(ctx, V, n, k, col(k), n, dgks, s, 1, kGate));   // :68-73 + the scalar part of the step
    }
    B200_TRY(read_tail());
    mv_products += t.iteration - before;                                  // :65, for the steps that really ran
    B200_REQUIRE(t.flags & (GM_FIN | GM_DONE), "internal: GMRES cycle did not close (flags=%d)", t.flags);
    if (t.flags & GM_FIN) {
      const int m = t.m;                                                  // update_solution! :273-283 with y = s->rhs
      if (m > 0) {
        if (!pr) {
          B200_TRY(block_axpy<T>(ctx, V, n, m, s->rhs, 1.0, x, x, n, nullptr));       // :275
        } else {
          B200_TRY(fill(ctx, n, 0.0, Ax, dt));
          B200_TRY(block_axpy<T>(ctx, V, n, m, s->rhs, 1.0, Ax, Ax, n, nullptr));     // :280
          B200_TRY(jacobi_ldiv(ctx, n, pr, Ax, Ax, dt));                               // :281
          B200_TRY(axpby(ctx, n, 1.0, Ax, 1.0, x, dt));                                // :282
        }
      }
      if (t.flags & GM_REINIT) {                                          // :93 (sic: tested with the old iteration count)
        B200_TRY(init(false, GM_FIN | GM_REINIT));                        // :96-99
        mv_products += 1;                                                 // :101
      }
    }
    if (t.flags & GM_BREAKDOWN) break;
  }
  B200_CUDA(cudaStreamSynchronize(ctx->stream));
  const int64_t n_hist = std::min<int64_t>(t.n_hist, hist_cap);
  if (resnorm_host && n_hist > 0) {
    B200_CUDA(cudaMemcpyAsync(resnorm_host, d_hist, sizeof(double) * (size_t)n_hist, cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  if (res) {
    res->iters = t.iteration;
    res->mvps = mv_products;                                              // history.mvps = iterable.mv_products :210
    res->isconverged = t.current <= t.tol;                                // :218
    res->status = (t.flags & GM_BREAKDOWN) ? B200_ERR_BREAKDOWN : 0;
    res->tol = t.tol;
    res->residual = t.current;
    res->n_resnorm = n_hist;
  }
  return B200_OK;
}

}  // namespace

extern "C" {

int b200_orthogonalize_and_normalize(b200_ctx *ctx, int64_t n_local, const void *V_dev, int64_t ldv, int k, void *w_dev,
                                     double *h_host, int method, int dtype, double *nrm) {
  B200_TRY(real_only(dtype, "b200_orthogonalize_and_normalize"));
  B200_REQUIRE(ctx && w_dev && nrm && (k == 0 || (V_dev && h_host)), "NULL argument");
  B200_REQUIRE(ldv >= n_local && n_local >= 0, "bad leading dimension");
  B200_REQUIRE(method == B200_ORTH_MGS || method == B200_ORTH_CGS || method == B200_ORTH_DGKS, "bad orth_meth");
  B200_CUDA(cudaSetDevice(ctx->device));
  return dtype == B200_F64 ? orth_impl<double>(ctx, n_local, (const double *)V_dev, ldv, k, (double *)w_dev, h_host, method, nrm)
                           : orth_impl<float>(ctx, n_local, (const float *)V_dev, ldv, k, (float *)w_dev, h_host, method, nrm);
}

int b200_hessenberg_ldiv(b200_ctx *ctx, double *H_dev, int ldh, int m, double *rhs_dev) {
  B200_REQUIRE(ctx && H_dev && rhs_dev && m >= 0 && ldh >= m + 1, "bad arguments");
  if (m == 0) return B200_OK;
  k_hessenberg_ldiv<<<1, 32, 0, ctx->stream>>>(H_dev, ldh, m, rhs_dev);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

int b200_gmres_solve(b200_ctx *ctx, const b200_csr *A, void *x_dev, const void *b_dev, const b200_gmres_opts *opts,
                     b200_result *res, double *resnorm_host, int64_t resnorm_cap) {
  B200_REQUIRE(ctx && A && x_dev && b_dev && opts, "NULL argument");
  B200_REQUIRE(A->ctx == ctx, "operator belongs to another context");
  B200_REQUIRE(is_square(A), "this solver needs a square operator (got %lld x %lld)", (long long)A->m_global,
               (long long)A->n_global);
  // ldiv! callbacks, or a complex operator (the engine below is real-only): the general engine
  if (opts->Pl.kind == B200_PREC_CALLBACK || opts->Pr.kind == B200_PREC_CALLBACK || is_complex_dtype(A->dtype))
    return gmres_general(ctx, CudaOp{A, nullptr}, A->dtype, A->m_local, A->n_global, x_dev, b_dev, opts, res, resnorm_host,
                         resnorm_cap);
  B200_REQUIRE(opts->Pl.kind == B200_PREC_IDENTITY || (opts->Pl.kind == B200_PREC_JACOBI && opts->Pl.diag),
               "unsupported preconditioner Pl");
  B200_REQUIRE(opts->Pr.kind == B200_PREC_IDENTITY || (opts->Pr.kind == B200_PREC_JACOBI && opts->Pr.diag),
               "unsupported preconditioner Pr");
  B200_CUDA(cudaSetDevice(ctx->device));
  if (ctx->world == 1 && ctx->opt_orth_fused && opts->orth_meth != B200_ORTH_MGS && A->m_local > 0)
    return A->dtype == B200_F64
               ? gmres_impl_fused<double>(ctx, A, (double *)x_dev, (const double *)b_dev, opts, res, resnorm_host, resnorm_cap)
               : gmres_impl_fused<float>(ctx, A, (float *)x_dev, (const float *)b_dev, opts, res, resnorm_host, resnorm_cap);
  return A->dtype == B200_F64
             ? gmres_impl<double>(ctx, A, (double *)x_dev, (const double *)b_dev, opts, res, resnorm_host, resnorm_cap)
             : gmres_impl<float>(ctx, A, (float *)x_dev, (const float *)b_dev, opts, res, resnorm_host, resnorm_cap);
}

}  // extern "C"
