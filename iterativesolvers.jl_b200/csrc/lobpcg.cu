// lobpcg.cu -- lobpcg(A, largest, X0; P, tol, maxiter) of reference src/lobpcg.jl:787-839, 865-893 and
// the step functor :692-749, for the standard problem (B = nothing) without constraint -- the path of
// BASELINE.json configs[4] (block = 16, fp32, 3-D Laplacian).
//
// Layout: the caller's X is n x bs column-major (the reference's layout).  Inside the engine every block
// (X, AX, R, AR, P, AP) is ROW-major, n rows x 16 values (zero-padded beyond bs): one row = 64 B (fp32) /
// 128 B (fp64) contiguous.  That makes the SpMM gather one aligned 64-byte read per nonzero, turns every
// block operand of the dense kernels into a plain contiguous stream, and lets the Gram kernel pull its
// operands with TMA bulk copies.  X is transposed in at the start and out at the end (2 passes per solve).
//
// Per step (it >= 3), all HBM-bound:
//   CholQR(R)  : k_gram (R'R) -> host Cholesky (fp64) -> k_rdiv (the reference's column sweeps of rdiv!
//                :345-355, done per row in registers)                                        (:365-393)
//   AR = A*R   : k_spmm_rm, A streamed ONCE for the 16 columns (the CPU path re-reads A per column) (:124-131)
//   CholQR(P)  : same, AP updated in the same launch                                          (:733)
//   Gram blocks: X'[AR R AP P], R'[AR P], AR'P, P'AP -- 4 launches of k_gram: a producer warp streams the
//                row chunks of the operands into a shared-memory ring with cp.async.bulk + mbarriers, 256
//                consumer threads accumulate 4x4 register tiles (16 row groups x 16 tiles)      (:586-605)
//   Rayleigh-Ritz: (3bs x 3bs) generalized symmetric eigenproblem on the host in fp64 (dense_small.h) (:607-627)
//   update     : ONE launch computes P = R Vr + P Vp, X = X Vx + P, the same for AP/AX, the residual
//                block R = AX - X diag(lambda) and its column norms                            (:629-690, :533-547)
// Soft locking (activeMask, :549-562) gathers the active columns into scratch blocks; with a full mask the
// active blocks alias R/P/AP (no copies).
// The contractions are fp32/fp64 FMA on CUDA cores: at bs = 16 they are HBM-bound (4 flop/byte) and TF32
// tensor cores would cost the fp32 eigenvalue parity.
#include "lobpcg_constraint.cuh"
#include "blas1.cuh"
#include "dense_small.h"
#include "spmv_stream.cuh"
#include "lobpcg_gram_wgmma.cuh"

using namespace b200;

namespace {

constexpr int kThreads = 256;
constexpr int BS = 16;             // padded block width
constexpr int RC = 128;            // rows per Gram chunk
constexpr int GSTAGES = 4;
constexpr int kGramConsumers = 2 * kThreads;      // two consumer groups of 256 threads
constexpr int kGramThreads = kGramConsumers + 32; // + producer warp

// 4 consecutive values from shared memory as one (fp32) or two (fp64) 128-bit loads
template <typename T>
__device__ __forceinline__ void lds4(const T *p, T (&v)[4]) {
  if constexpr (sizeof(T) == 4) {
    const float4 t = *reinterpret_cast<const float4 *>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  } else {
    const double2 a = reinterpret_cast<const double2 *>(p)[0], b = reinterpret_cast<const double2 *>(p)[1];
    v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
  }
}

template <typename T>
__device__ __forceinline__ void st4(T *p, const T (&v)[4]) {
  if constexpr (sizeof(T) == 4) {
    *reinterpret_cast<float4 *>(p) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
    reinterpret_cast<double2 *>(p)[0] = make_double2(v[0], v[1]);
    reinterpret_cast<double2 *>(p)[1] = make_double2(v[2], v[3]);
  }
}

template <typename T>
__device__ __forceinline__ void load_row(const T *__restrict__ p, T (&v)[BS]) {
  if constexpr (sizeof(T) == 4) {
    const float4 *q = reinterpret_cast<const float4 *>(p);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float4 t = q[i];
      v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
    }
  } else {
    const double2 *q = reinterpret_cast<const double2 *>(p);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const double2 t = q[i];
      v[2 * i] = t.x; v[2 * i + 1] = t.y;
    }
  }
}
template <typename T>
__device__ __forceinline__ void store_row(T *__restrict__ p, const T (&v)[BS]) {
  if constexpr (sizeof(T) == 4) {
    float4 *q = reinterpret_cast<float4 *>(p);
#pragma unroll
    for (int i = 0; i < 4; ++i) q[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
  } else {
    double2 *q = reinterpret_cast<double2 *>(p);
#pragma unroll
    for (int i = 0; i < 8; ++i) q[i] = make_double2(v[2 * i], v[2 * i + 1]);
  }
}

// column-major n x bs (ld = n)  <->  row-major n x 16
template <typename T>
__global__ void __launch_bounds__(kThreads) k_to_rowmajor(const T *__restrict__ cm, T *__restrict__ rm, int64_t n,
                                                          int bs) {
  for (int64_t r = blockIdx.x * (int64_t)kThreads + threadIdx.x; r < n; r += (int64_t)gridDim.x * kThreads) {
    T v[BS];
#pragma unroll
    for (int j = 0; j < BS; ++j) v[j] = j < bs ? cm[r + (int64_t)j * n] : (T)0;
    store_row<T>(rm + r * BS, v);
  }
}
template <typename T>
__global__ void __launch_bounds__(kThreads) k_to_colmajor(const T *__restrict__ rm, T *__restrict__ cm, int64_t n,
                                                          int bs) {
  for (int64_t r = blockIdx.x * (int64_t)kThreads + threadIdx.x; r < n; r += (int64_t)gridDim.x * kThreads) {
    T v[BS];
    load_row<T>(rm + r * BS, v);
#pragma unroll
    for (int j = 0; j < BS; ++j)
      if (j < bs) cm[r + (int64_t)j * n] = v[j];
  }
}

// multi-GPU: rows idx[k] of a row-major block -> contiguous send buffer (4 lanes per row)
template <typename T>
__global__ void __launch_bounds__(kThreads) k_pack_rows(const int *__restrict__ idx, const T *__restrict__ X,
                                                        int64_t nrows, T *__restrict__ out) {
  const int sub = threadIdx.x & 3;
  for (int64_t k = (blockIdx.x * (int64_t)kThreads + threadIdx.x) >> 2; k < nrows;
       k += ((int64_t)gridDim.x * kThreads) >> 2) {
    T v[4];
    lds4<T>(X + (int64_t)idx[k] * BS + 4 * sub, v);
    st4<T>(out + k * BS + 4 * sub, v);
  }
}

// Y = A X on row-major blocks: 4 lanes per row, each lane owns 4 of the 16 columns, so every nonzero is one
// coalesced 64-byte (fp32) read of the X row.
// k_spmm_rm has an overload per row-offset width (int, int64_t; spmv_launch.cuh says why overloads).
template <typename T, typename I>
__device__ __forceinline__ void spmm_rm_rows(const I *__restrict__ rowptr, const int *__restrict__ colind,
                                             const T *__restrict__ vals, const T *__restrict__ X,
                                             const T *__restrict__ Xhalo, int64_t m, T *__restrict__ Y) {
  const int sub = threadIdx.x & 3;
  const int rib = threadIdx.x >> 2;
  const uint64_t pol = policy_evict_first();
  for (int64_t base = (int64_t)blockIdx.x * (kThreads / 4); base < m; base += (int64_t)gridDim.x * (kThreads / 4)) {
    const int64_t row = base + rib;
    if (row >= m) continue;
    const I b = __ldg(rowptr + row), e = __ldg(rowptr + row + 1);
    T acc[4] = {(T)0, (T)0, (T)0, (T)0};
    // four nonzeros per round: their column indices, then their four X rows are in flight together (the one-by-one loop
    // chains index load -> gather -> FMA per nonzero and is latency-bound); the products are added
    // in the row's storage order, as before
    for (I k = b; k < e; k += 4) {
      int c[4];
      T a[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const I kk = k + u < e ? k + u : e - 1;
        c[u] = ld_stream<int>(colind + kk, pol);
        a[u] = ld_stream<T>(vals + kk, pol);
        if (k + u >= e) a[u] = (T)0;
      }
      T t[4][4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        // local extended index: [0, m) own rows, [m, m + n_halo) rows received from the neighbours
        const T *xr = (c[u] < m ? X + (int64_t)c[u] * BS : Xhalo + (int64_t)(c[u] - m) * BS) + 4 * sub;
        if constexpr (sizeof(T) == 4) {
          const float4 v = __ldg(reinterpret_cast<const float4 *>(xr));
          t[u][0] = v.x; t[u][1] = v.y; t[u][2] = v.z; t[u][3] = v.w;
        } else {
          const double2 v0 = __ldg(reinterpret_cast<const double2 *>(xr));
          const double2 v1 = __ldg(reinterpret_cast<const double2 *>(xr) + 1);
          t[u][0] = v0.x; t[u][1] = v0.y; t[u][2] = v1.x; t[u][3] = v1.y;
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (k + u < e) {
#pragma unroll
          for (int q = 0; q < 4; ++q) acc[q] += a[u] * t[u][q];
        }
      }
    }
    T *yr = Y + row * BS + 4 * sub;
    if constexpr (sizeof(T) == 4) *reinterpret_cast<float4 *>(yr) = make_float4(acc[0], acc[1], acc[2], acc[3]);
    else {
      reinterpret_cast<double2 *>(yr)[0] = make_double2(acc[0], acc[1]);
      reinterpret_cast<double2 *>(yr)[1] = make_double2(acc[2], acc[3]);
    }
  }
}
template <typename T>
__global__ void __launch_bounds__(kThreads) k_spmm_rm(const int *__restrict__ rowptr, const int *__restrict__ colind,
                                                      const T *__restrict__ vals, const T *__restrict__ X,
                                                      const T *__restrict__ Xhalo, int64_t m, T *__restrict__ Y) {
  spmm_rm_rows(rowptr, colind, vals, X, Xhalo, m, Y);
}
template <typename T>
__global__ void __launch_bounds__(kThreads) k_spmm_rm(const int64_t *__restrict__ rowptr, const int *__restrict__ colind,
                                                      const T *__restrict__ vals, const T *__restrict__ X,
                                                      const T *__restrict__ Xhalo, int64_t m, T *__restrict__ Y) {
  spmm_rm_rows(rowptr, colind, vals, X, Xhalo, m, Y);
}

// ---------------------------------------------------------------------------------------------------------
// G_b = L' * R_b  (b < NR), all blocks row-major n x 16.  TMA-fed: see file header.
// ---------------------------------------------------------------------------------------------------------
template <typename T, int NR>
struct GramSmem {
  alignas(128) T buf[GSTAGES][1 + NR][RC * BS];
  alignas(8) unsigned long long full[GSTAGES];
  alignas(8) unsigned long long empty[GSTAGES];
};

template <typename T, int NR>
__global__ void __launch_bounds__(kGramThreads, 1)
    k_gram(const T *__restrict__ L, const T *__restrict__ R0, const T *__restrict__ R1, const T *__restrict__ R2,
           const T *__restrict__ R3, int same0 /* R0 is L itself: stream it once */, int64_t n, double *partials,
           unsigned int *ticket, double *__restrict__ out) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  GramSmem<T, NR> *sm = reinterpret_cast<GramSmem<T, NR> *>(smem_raw);
  __shared__ bool is_last;
  const T *Rp[4] = {R0, R1, R2, R3};
  const int tid = threadIdx.x;
  const int64_t nchunks = (n + RC - 1) / RC;
  if (tid == 0) {
    for (int s = 0; s < GSTAGES; ++s) {
      mbar_init(&sm->full[s], 1);
      mbar_init(&sm->empty[s], kThreads / 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // consumers: two groups of 256 threads work on alternate chunks (first ncu capture with one group:
  // issue 43 %, 9 warps resident -> dependency-bound); inside a group 16 row groups x 16 (4x4) tiles.
  const int grp = tid / kThreads;               // 0, 1 (consumers), 2 (producer warp)
  const int lt = tid % kThreads;
  const int g = lt >> 4;                        // row group 0..15 inside the consumer group
  const int ti = (lt & 15) >> 2, tj = lt & 3;
  // accumulators in the operand precision over the thread's whole run (<= n/(132*32) rows per thread on an H100: fp32
  // rounding stays ~1e-6 relative per partial); the cross-thread and cross-CTA sums are fp64
  T acc[NR][4][4];
#pragma unroll
  for (int b = 0; b < NR; ++b)
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[b][a][c] = (T)0;

  if (tid >= kGramConsumers) {
    if (tid == kGramConsumers) {                // producer
      const uint64_t pol = policy_evict_first();
      int it = 0;
      for (int64_t c = blockIdx.x; c < nchunks; c += gridDim.x, ++it) {
        const int s = it % GSTAGES;
        const uint32_t ph = (uint32_t)((it / GSTAGES) & 1);
        mbar_wait(&sm->empty[s], ph ^ 1u);
        const int64_t r0 = c * RC;
        const int rows = (int)((n - r0 < RC) ? (n - r0) : RC);
        const uint32_t bytes = (uint32_t)rows * BS * (uint32_t)sizeof(T);
        mbar_expect_tx(&sm->full[s], bytes * (1 + NR - (same0 ? 1 : 0)));
        bulk_g2s(sm->buf[s][0], L + r0 * BS, bytes, &sm->full[s], pol);
#pragma unroll
        for (int b = 0; b < NR; ++b)
          if (!(same0 && b == 0)) bulk_g2s(sm->buf[s][1 + b], Rp[b] + r0 * BS, bytes, &sm->full[s], pol);
      }
    }
  } else {
    for (int64_t k = grp;; k += 2) {
      const int64_t c = (int64_t)blockIdx.x + k * gridDim.x;
      if (c >= nchunks) break;
      const int s = (int)(k % GSTAGES);
      const uint32_t ph = (uint32_t)((k / GSTAGES) & 1);
      const int64_t r0 = c * RC;
      const int rows = (int)((n - r0 < RC) ? (n - r0) : RC);
      mbar_wait(&sm->full[s], ph);
#pragma unroll 2
      for (int q = 0; q < RC / 16; ++q) {
        const int r = g + 16 * q;
        if (r < rows) {
          T l[4];
          lds4<T>(&sm->buf[s][0][r * BS + 4 * ti], l);
#pragma unroll
          for (int b = 0; b < NR; ++b) {
            T rv[4];
            lds4<T>(&sm->buf[s][(same0 && b == 0) ? 0 : 1 + b][r * BS + 4 * tj], rv);
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
              for (int cc = 0; cc < 4; ++cc) acc[b][a][cc] += l[a] * rv[cc];
          }
        }
      }
      __syncwarp();
      if ((tid & 31) == 0) mbar_arrive(&sm->empty[s]);
    }
  }
  __syncthreads();   // all TMA data consumed: the ring memory is reused for the cross-group reduction
  double(*red)[256] = reinterpret_cast<double(*)[256]>(smem_raw);
  static_assert(sizeof(GramSmem<T, NR>) >= sizeof(double) * 32 * 256, "reduction scratch does not fit");
  for (int b = 0; b < NR; ++b) {
    if (tid < kGramConsumers) {
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int c = 0; c < 4; ++c) red[grp * 16 + g][(4 * ti + a) * 16 + 4 * tj + c] = (double)acc[b][a][c];
    }
    __syncthreads();
    if (tid < kThreads) {
      double s = 0.0;
      for (int gg = 0; gg < 32; ++gg) s += red[gg][tid];
      partials[((size_t)blockIdx.x * NR + b) * 256 + tid] = s;
    }
    __syncthreads();
  }
  if (tid == 0) {
    __threadfence();
    is_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  if (tid < kThreads) {
    for (int b = 0; b < NR; ++b) {
      double s = 0.0;
      for (unsigned int blk = 0; blk < gridDim.x; ++blk) s += __ldcg(&partials[((size_t)blk * NR + b) * 256 + tid]);
      out[b * 256 + tid] = s;      // out[b][i*16 + j] = G_b[i][j]
    }
  }
  if (tid == 0) *ticket = 0u;
}

// rdiv!(A, U::UpperTriangular) row by row (reference src/lobpcg.jl:345-355), up to 2 blocks per launch
template <typename T>
__global__ void __launch_bounds__(kThreads, 4) k_rdiv(T *__restrict__ X0, T *__restrict__ X1, int nblk, int bs,
                                                   int64_t n, const T *__restrict__ Ufac /* bs x bs col-major */) {
  __shared__ T U[BS][BS];
  for (int q = threadIdx.x; q < BS * BS; q += kThreads) {
    const int i = q % BS, j = q / BS;
    U[i][j] = (i < bs && j < bs) ? Ufac[i + j * bs] : (T)(i == j);
  }
  __syncthreads();
  for (int64_t r = blockIdx.x * (int64_t)kThreads + threadIdx.x; r < n; r += (int64_t)gridDim.x * kThreads) {
    for (int blk = 0; blk < nblk; ++blk) {
      T *X = (blk == 0 ? X0 : X1) + r * BS;
      T a[BS];
      load_row<T>(X, a);
      a[0] = a[0] / U[0][0];                                         // :347
#pragma unroll
      for (int i = 1; i < BS; ++i) {
        if (i < bs) {
#pragma unroll
          for (int j = 0; j < i; ++j) a[i] = a[i] - a[j] * U[j][i];   // :350
          a[i] = a[i] / U[i][i];                                      // :352
        }
      }
      store_row<T>(X, a);
    }
  }
}

// ---- quad layout for the dense row-block kernels ---------------------------------------------------------------
// A warp works on 8 consecutive rows at a time: lanes 4q..4q+3 form the quad of row q and lane c of the quad owns
// columns 4c..4c+3, so every global load/store instruction of the warp covers 8 x 64 B contiguous bytes (fp32).
// (A row per thread issues 32 sectors per request and is L1/LSU-bound); the other three chunks of a row come from the
// quad by shuffle.
template <typename T>
__device__ __forceinline__ void quad_gather(const T (&mine)[4], T (&row)[BS]) {
#pragma unroll
  for (int cc = 0; cc < 4; ++cc) {
#pragma unroll
    for (int e = 0; e < 4; ++e) row[4 * cc + e] = __shfl_sync(0xffffffffu, mine[e], cc, 4);
  }
}
// o0[e] += sum_i r0[i] * V[i][4c+e], o1 likewise for a second row (the V loads are shared by the two rows)
template <typename T>
__device__ __forceinline__ void rows2_times_vchunk(const T (&r0)[BS], const T (&r1)[BS], int nin, const T (*V)[BS],
                                                   int c, T (&o0)[4], T (&o1)[4]) {
#pragma unroll
  for (int i = 0; i < BS; ++i) {
    if (i < nin) {
      T v[4];
      lds4<T>(&V[i][4 * c], v);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        o0[e] += r0[i] * v[e];
        o1[e] += r1[i] * v[e];
      }
    }
  }
}

struct UpdateArgs {
  void *X, *AX, *P, *AP, *R;          // in/out blocks
  const void *aR, *aAR, *aP, *aAP;    // active blocks, bs1 / bs2 columns used
  int sizeX, bs1, bs2;
  int64_t n;
};

// update_X_P! (:629-690) + residuals! (:533-547).  Vbuf: Vx | Vr | Vp as 16x16 row-major [i][j] (zero padded),
// lambda: 16.  Two launches (the fused single kernel needed 228 registers):
//   PHASE 0: P = aR Vr + aP Vp ; X = X Vx + P                                  (reads 3 blocks, writes 2)
//   PHASE 1: AP = aAR Vr + aAP Vp ; AX = AX Vx + AP ; R = AX - X diag(lambda) ; column norms of R
//                                                                               (reads 4 blocks, writes 3)
// Quad layout, two rows (q and q+8 of a 16-row group) per thread.
template <typename T, int PHASE>
__global__ void __launch_bounds__(kThreads) k_update(UpdateArgs a, const T *__restrict__ Vbuf,
                                                        const T *__restrict__ lambda, double *partials,
                                                        unsigned int *ticket, double *__restrict__ norms2) {
  __shared__ __align__(16) T Vx[BS][BS], Vr[BS][BS], Vp[BS][BS];
  __shared__ T lam[BS];
  __shared__ double smem[kThreads / 32][BS];
  __shared__ bool is_last;
  for (int q = threadIdx.x; q < BS * BS; q += kThreads) {
    (&Vx[0][0])[q] = Vbuf[q];
    (&Vr[0][0])[q] = Vbuf[256 + q];
    (&Vp[0][0])[q] = Vbuf[512 + q];
  }
  if (threadIdx.x < BS) lam[threadIdx.x] = threadIdx.x < a.sizeX ? lambda[threadIdx.x] : (T)0;
  __syncthreads();
  // PHASE 0 works on the blocks themselves, PHASE 1 on their A-images
  T *Xb = (T *)(PHASE == 0 ? a.X : a.AX), *Pb = (T *)(PHASE == 0 ? a.P : a.AP), *R = (T *)a.R;
  const T *Xnew = (const T *)a.X;
  const T *aRb = (const T *)(PHASE == 0 ? a.aR : a.aAR), *aPb = (const T *)(PHASE == 0 ? a.aP : a.aAP);
  const int64_t n = a.n;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c = lane & 3, q = lane >> 2;
  const bool has1 = a.bs1 > 0, has2 = a.bs2 > 0;
  double nrm[4] = {0.0, 0.0, 0.0, 0.0};
  const int64_t warps_total = (int64_t)gridDim.x * (kThreads / 32);
  for (int64_t base = ((int64_t)blockIdx.x * (kThreads / 32) + warp) * 16; base < n; base += warps_total * 16) {
    const int64_t r0 = base + q, r1 = base + 8 + q;
    const bool ok0 = r0 < n, ok1 = r1 < n;
    const int64_t o0 = (ok0 ? r0 : 0) * BS + 4 * c, o1 = (ok1 ? r1 : 0) * BS + 4 * c;   // clamped: shuffles need all lanes
    T x0[4], x1[4], p0[4], p1[4], q0[4], q1[4];
    // all chunk loads first (up to 6 x 128-bit loads in flight per thread), then the shuffles and FMAs
    if (has1) { lds4<T>(aRb + o0, p0); lds4<T>(aRb + o1, p1); }
    if (has2) { lds4<T>(aPb + o0, q0); lds4<T>(aPb + o1, q1); }
    lds4<T>(Xb + o0, x0);
    lds4<T>(Xb + o1, x1);
    T pn0[4] = {(T)0, (T)0, (T)0, (T)0}, pn1[4] = {(T)0, (T)0, (T)0, (T)0};
    T xn0[4] = {(T)0, (T)0, (T)0, (T)0}, xn1[4] = {(T)0, (T)0, (T)0, (T)0};
    T w0[BS], w1[BS];
    if (has1) {
      quad_gather<T>(p0, w0);
      quad_gather<T>(p1, w1);
      rows2_times_vchunk<T>(w0, w1, a.bs1, Vr, c, pn0, pn1);
    }
    if (has2) {                                                             // + aP Vp  (:652-658)
      quad_gather<T>(q0, w0);
      quad_gather<T>(q1, w1);
      rows2_times_vchunk<T>(w0, w1, a.bs2, Vp, c, pn0, pn1);
    }
    quad_gather<T>(x0, w0);
    quad_gather<T>(x1, w1);
    rows2_times_vchunk<T>(w0, w1, a.sizeX, Vx, c, xn0, xn1);
    if (has1) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {                                         // tempX .+ P  (:675)
        xn0[e] = xn0[e] + pn0[e];
        xn1[e] = xn1[e] + pn1[e];
      }
      if (ok0) st4<T>(Pb + o0, pn0);
      if (ok1) st4<T>(Pb + o1, pn1);
    }
    if (ok0) st4<T>(Xb + o0, xn0);
    if (ok1) st4<T>(Xb + o1, xn1);
    if constexpr (PHASE == 1) {
      // residuals!: R = AX - X * Diagonal(lambda)  (:535-536) and column norms (:538-545); X is already updated
      lds4<T>(Xnew + o0, x0);
      lds4<T>(Xnew + o1, x1);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int j = 4 * c + e;
        const T res0 = (j < a.sizeX && ok0) ? xn0[e] - x0[e] * lam[j] : (T)0;
        const T res1 = (j < a.sizeX && ok1) ? xn1[e] - x1[e] * lam[j] : (T)0;
        pn0[e] = res0;
        pn1[e] = res1;
        nrm[e] += (double)res0 * (double)res0 + (double)res1 * (double)res1;
      }
      if (ok0) st4<T>(R + o0, pn0);
      if (ok1) st4<T>(R + o1, pn1);
    }
  }
  if constexpr (PHASE == 0) return;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    double v = nrm[e];
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 16);
    if (lane < 4) smem[warp][4 * lane + e] = v;
  }
  __syncthreads();
  if (threadIdx.x < BS) {
    double s = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) s += smem[w][threadIdx.x];
    partials[(size_t)blockIdx.x * kMaxReduceWidth + threadIdx.x] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    is_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  for (int j = warp; j < BS; j += kThreads / 32) {    // warp per column, lanes stride over the block slots (deterministic)
    double s = 0.0;
    for (unsigned int b = lane; b < gridDim.x; b += 32) s += __ldcg(&partials[(size_t)b * kMaxReduceWidth + j]);
    s = warp_sum(s);
    if (lane == 0) norms2[j] = s;
  }
  if (threadIdx.x == 0) *ticket = 0u;
}

// ---------------------------------------------------------------------------------------------------------
// fp32 blocks on the tensor pipe ("3xTF32": a = a_hi + a_lo in TF32, a*b ~ a_lo*b_hi + a_hi*b_lo + a_hi*b_hi,
// fp32 accumulate; products are exact, the dropped a_lo*b_lo term is 2^-22 relative).  The SIMT versions of the
// update and of the Rayleigh-Ritz Gram products are bound by shared-memory operand traffic / FMA issue, not by
// HBM (LSU and issue bound); as m16n8k8 MMAs the same arithmetic is ~6 % of the tensor pipe and the kernels
// become bandwidth-bound.  These are tall-skinny products (K or N = 16): one warp-level mma.sync per 16 rows is
// the natural tile.
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void split_tf32(float x, uint32_t &hi, uint32_t &lo) {
  hi = to_tf32(x);
  lo = to_tf32(x - __uint_as_float(hi));
}
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_3xtf32(float (&d)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4],
                                           uint32_t bh0, uint32_t bh1, uint32_t bl0, uint32_t bl1) {
  mma_tf32(d, al, bh0, bh1);   // small terms first
  mma_tf32(d, ah, bl0, bl1);
  mma_tf32(d, ah, bh0, bh1);
}

// B operand (16x16 coefficient matrix V, shared memory) as loop-invariant register fragments.  With lane = 4g + t
// the two k8 halves p of a 16-wide K use the column permutation  logical k = t (t+4)  <->  physical 4t+2p (+1),
// so that the A fragment is exactly the lane's own 16-byte chunk of the row (quad layout, coalesced).
struct BFrag {
  uint32_t h[2][2][2], l[2][2][2];   // [p][n-tile][b0/b1]
};
__device__ __forceinline__ void load_bfrag(const float (*V)[BS], int g, int t, BFrag &f) {
#pragma unroll
  for (int p = 0; p < 2; ++p)
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int h = 0; h < 2; ++h) split_tf32(V[4 * t + 2 * p + h][8 * nt + g], f.h[p][nt][h], f.l[p][nt][h]);
}
// acc[nt] += [x0 ; x1] * V   (x0: row g, x1: row g+8, both the lane's columns 4t..4t+3; columns >= nin are skipped)
// acc[nt] = {(g, 8nt+2t), (g, 8nt+2t+1), (g+8, 8nt+2t), (g+8, 8nt+2t+1)}
__device__ __forceinline__ void chunk_mma(const float (&x0)[4], const float (&x1)[4], int nin, int t, const BFrag &f,
                                          float (&acc)[2][4]) {
#pragma unroll
  for (int p = 0; p < 2; ++p) {
    const bool on0 = 4 * t + 2 * p < nin, on1 = 4 * t + 2 * p + 1 < nin;
    uint32_t ah[4], al[4];
    split_tf32(on0 ? x0[2 * p] : 0.f, ah[0], al[0]);
    split_tf32(on0 ? x1[2 * p] : 0.f, ah[1], al[1]);
    split_tf32(on1 ? x0[2 * p + 1] : 0.f, ah[2], al[2]);
    split_tf32(on1 ? x1[2 * p + 1] : 0.f, ah[3], al[3]);
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
      mma_3xtf32(acc[nt], ah, al, f.h[p][nt][0], f.h[p][nt][1], f.l[p][nt][0], f.l[p][nt][1]);
  }
}

// k_update for fp32 blocks on the tensor pipe; same phases, same memory behaviour as k_update<float, PHASE>.
template <int PHASE>
__global__ void __launch_bounds__(kThreads, 2) k_update_tc(UpdateArgs a, const float *__restrict__ Vbuf,
                                                            const float *__restrict__ lambda, double *partials,
                                                            unsigned int *ticket, double *__restrict__ norms2) {
  __shared__ float V3[3][BS][BS];
  __shared__ float lam[BS];
  __shared__ double smem[kThreads / 32][BS];
  __shared__ bool is_last;
  for (int q = threadIdx.x; q < 3 * BS * BS; q += kThreads) (&V3[0][0][0])[q] = Vbuf[q];
  if (threadIdx.x < BS) lam[threadIdx.x] = threadIdx.x < a.sizeX ? lambda[threadIdx.x] : 0.f;
  __syncthreads();
  float *Xb = (float *)(PHASE == 0 ? a.X : a.AX), *Pb = (float *)(PHASE == 0 ? a.P : a.AP), *R = (float *)a.R;
  const float *Xnew = (const float *)a.X;
  const float *aRb = (const float *)(PHASE == 0 ? a.aR : a.aAR), *aPb = (const float *)(PHASE == 0 ? a.aP : a.aAP);
  const int64_t n = a.n;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int t = lane & 3, g = lane >> 2;
  const bool has1 = a.bs1 > 0, has2 = a.bs2 > 0;
  BFrag fx, fr, fp;
  load_bfrag(V3[0], g, t, fx);
  if (has1) load_bfrag(V3[1], g, t, fr);
  if (has2) load_bfrag(V3[2], g, t, fp);
  double nrm[4] = {0.0, 0.0, 0.0, 0.0};   // columns 2t, 2t+1, 8+2t, 8+2t+1
  const int64_t warps_total = (int64_t)gridDim.x * (kThreads / 32);
  for (int64_t base = ((int64_t)blockIdx.x * (kThreads / 32) + warp) * 16; base < n; base += warps_total * 16) {
    const int64_t r0 = base + g, r1 = base + 8 + g;
    const bool ok0 = r0 < n, ok1 = r1 < n;
    const int64_t b0 = (ok0 ? r0 : 0) * BS, b1 = (ok1 ? r1 : 0) * BS;   // clamped: the MMAs need all lanes
    float x0[4], x1[4], p0[4], p1[4], q0[4], q1[4];
    if (has1) { lds4<float>(aRb + b0 + 4 * t, p0); lds4<float>(aRb + b1 + 4 * t, p1); }
    if (has2) { lds4<float>(aPb + b0 + 4 * t, q0); lds4<float>(aPb + b1 + 4 * t, q1); }
    lds4<float>(Xb + b0 + 4 * t, x0);
    lds4<float>(Xb + b1 + 4 * t, x1);
    float2 xw[2][2];
    if constexpr (PHASE == 1) {
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        xw[nt][0] = *reinterpret_cast<const float2 *>(Xnew + b0 + 8 * nt + 2 * t);
        xw[nt][1] = *reinterpret_cast<const float2 *>(Xnew + b1 + 8 * nt + 2 * t);
      }
    }
    float pn[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}}, xn[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
    if (has1) chunk_mma(p0, p1, a.bs1, t, fr, pn);
    if (has2) chunk_mma(q0, q1, a.bs2, t, fp, pn);                          // + aP Vp  (:652-658)
    chunk_mma(x0, x1, a.sizeX, t, fx, xn);
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      const int col = 8 * nt + 2 * t;
      if (has1) {
#pragma unroll
        for (int e = 0; e < 4; ++e) xn[nt][e] = xn[nt][e] + pn[nt][e];      // tempX .+ P  (:675)
        if (ok0) *reinterpret_cast<float2 *>(Pb + b0 + col) = make_float2(pn[nt][0], pn[nt][1]);
        if (ok1) *reinterpret_cast<float2 *>(Pb + b1 + col) = make_float2(pn[nt][2], pn[nt][3]);
      }
      if (ok0) *reinterpret_cast<float2 *>(Xb + b0 + col) = make_float2(xn[nt][0], xn[nt][1]);
      if (ok1) *reinterpret_cast<float2 *>(Xb + b1 + col) = make_float2(xn[nt][2], xn[nt][3]);
      if constexpr (PHASE == 1) {
        // residuals!: R = AX - X * Diagonal(lambda)  (:535-536) and column norms (:538-545); X is already updated
        const bool c0 = col < a.sizeX, c1 = col + 1 < a.sizeX;
        const float l0 = lam[col], l1 = lam[col + 1];
        const float ra = (c0 && ok0) ? xn[nt][0] - xw[nt][0].x * l0 : 0.f;
        const float rb = (c1 && ok0) ? xn[nt][1] - xw[nt][0].y * l1 : 0.f;
        const float rc = (c0 && ok1) ? xn[nt][2] - xw[nt][1].x * l0 : 0.f;
        const float rd = (c1 && ok1) ? xn[nt][3] - xw[nt][1].y * l1 : 0.f;
        nrm[2 * nt] += (double)ra * (double)ra + (double)rc * (double)rc;
        nrm[2 * nt + 1] += (double)rb * (double)rb + (double)rd * (double)rd;
        if (ok0) *reinterpret_cast<float2 *>(R + b0 + col) = make_float2(ra, rb);
        if (ok1) *reinterpret_cast<float2 *>(R + b1 + col) = make_float2(rc, rd);
      }
    }
  }
  if constexpr (PHASE == 0) return;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    double v = nrm[e];
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 16);
    if (lane < 4) smem[warp][8 * (e >> 1) + 2 * lane + (e & 1)] = v;
  }
  __syncthreads();
  if (threadIdx.x < BS) {
    double s = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) s += smem[w][threadIdx.x];
    partials[(size_t)blockIdx.x * kMaxReduceWidth + threadIdx.x] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    is_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  for (int j = warp; j < BS; j += kThreads / 32) {    // warp per column, lanes stride over the block slots (deterministic)
    double s = 0.0;
    for (unsigned int b = lane; b < gridDim.x; b += 32) s += __ldcg(&partials[(size_t)b * kMaxReduceWidth + j]);
    s = warp_sum(s);
    if (lane == 0) norms2[j] = s;
  }
  if (threadIdx.x == 0) *ticket = 0u;
}

// All Gram blocks of one Rayleigh-Ritz step in ONE pass over the blocks (reference src/lobpcg.jl:262-271 computes
// them as eight separate mul! calls; the SIMT path above needs five launches that stream 13 blocks):
//   MODE 1: blocks X, R, AR        -> X'AR, X'R, R'AR                                (3 products, no P yet)
//   MODE 2: blocks X, R, AR, P, AP -> X'AR, X'R, R'AR, X'AP, X'P, R'P, AR'P, P'AP    (8 products)
//   MODE 0: one block B -> B'B  (the CholQR Gram matrix, :378)
// out[p*256 + i*16 + j] = G_p[i][j].  TMA ring as k_gram; each consumer warp turns 8 staged rows into one k8 step:
// the lane's two 64-bit shared loads (rows k0+t, k0+t+4, columns 2g, 2g+1) are at once the A fragment of the block
// as a left factor (m = g <-> column 2g, m = g+8 <-> column 2g+1) and its B fragments as a right factor
// (n-tile nt, n = g <-> column 2g+nt) -- conflict-free, no transposition.
constexpr int kRrRows = 128;
constexpr int rr_blocks(int mode) { return mode == 2 ? 5 : (mode == 1 ? 3 : 1); }
constexpr int rr_stages(int mode) { return mode == 2 ? 3 : (mode == 1 ? 4 : 8); }   // 120 / 96 / 64 KB in flight
constexpr int kRrConsumerWarps = 16;
constexpr int kRrThreads = kRrConsumerWarps * 32 + 32;
template <int MODE>
struct RrSmem {
  alignas(128) float buf[rr_stages(MODE)][rr_blocks(MODE)][kRrRows * BS];
  alignas(8) unsigned long long full[rr_stages(MODE)];
  alignas(8) unsigned long long empty[rr_stages(MODE)];
};
struct RrArgs {
  const float *blk[5];   // X, R, AR, P, AP
  int64_t n;
};

template <int MODE>
__global__ void __launch_bounds__(kRrThreads, 1) k_gram_rr_tc(RrArgs a, double *partials, unsigned int *ticket,
                                                              double *__restrict__ out) {
  constexpr bool WITH_P = MODE == 2;
  constexpr int NB = rr_blocks(MODE);
  constexpr int NP = MODE == 2 ? 8 : (MODE == 1 ? 3 : 1);
  constexpr int kRrStages = rr_stages(MODE);
  // (left, right) block of each product; block order X=0, R=1, AR=2, P=3, AP=4
  constexpr int kL[8] = {0, 0, 1, 0, 0, 1, 2, 3};
  constexpr int kR[8] = {MODE == 0 ? 0 : 2, 1, 2, 4, 3, 3, 3, 4};
  extern __shared__ __align__(128) unsigned char smem_raw[];
  RrSmem<MODE> *sm = reinterpret_cast<RrSmem<MODE> *>(smem_raw);
  __shared__ bool is_last;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int t = lane & 3, g = lane >> 2;
  const int64_t n = a.n;
  const int64_t nchunks = (n + kRrRows - 1) / kRrRows;
  if (tid == 0) {
    for (int s = 0; s < kRrStages; ++s) {
      mbar_init(&sm->full[s], 1);
      mbar_init(&sm->empty[s], kRrConsumerWarps);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // WITH_P: warps 0-7 own products 0-3, warps 8-15 products 4-7 (32 accumulator registers per lane instead of 64),
  // each over 16 of the chunk's 128 rows; without P all 16 warps own the three products over 8 rows each.
  constexpr int NPW = WITH_P ? 4 : NP;
  constexpr int kSteps = WITH_P ? 2 : 1;
  const int half = WITH_P ? (warp >> 3) & 1 : 0;
  const int wrow = (WITH_P ? (warp & 7) : warp) * 8 * kSteps;
  float acc[NPW][2][4];
#pragma unroll
  for (int p = 0; p < NPW; ++p)
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[p][nt][e] = 0.f;
  float acc_small[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};   // MODE 0: the three small product terms
  // MODE 0 / 1 (the first Rayleigh-Ritz step and CholQR, on the default path too): the MMA accumulator is added to
  // `tot` with ordinary fp32 adds after every chunk.  The tensor core's fp32 accumulate truncates, so a chain that
  // grows with the rows per warp biases the diagonals of the Gram matrices (see lobpcg_gram_wgmma.cuh).
  constexpr int NTOT = WITH_P ? 1 : NPW;
  float tot[NTOT][2][4];
#pragma unroll
  for (int p = 0; p < NTOT; ++p)
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) tot[p][nt][e] = 0.f;

  if (warp == kRrConsumerWarps) {
    if (lane == 0) {                                   // producer
      const uint64_t pol = policy_evict_first();
      int it = 0;
      for (int64_t c = blockIdx.x; c < nchunks; c += gridDim.x, ++it) {
        const int s = it % kRrStages;
        const uint32_t ph = (uint32_t)((it / kRrStages) & 1);
        mbar_wait(&sm->empty[s], ph ^ 1u);
        const int64_t r0 = c * kRrRows;
        const int rows = (int)((n - r0 < kRrRows) ? (n - r0) : kRrRows);
        const uint32_t bytes = (uint32_t)rows * BS * (uint32_t)sizeof(float);
        mbar_expect_tx(&sm->full[s], bytes * NB);
#pragma unroll
        for (int b = 0; b < NB; ++b) bulk_g2s(sm->buf[s][b], a.blk[b] + r0 * BS, bytes, &sm->full[s], pol);
      }
    }
  } else {
    int it = 0;
    for (int64_t c = blockIdx.x; c < nchunks; c += gridDim.x, ++it) {
      const int s = it % kRrStages;
      const uint32_t ph = (uint32_t)((it / kRrStages) & 1);
      const int64_t r0 = c * kRrRows;
      const int rows = (int)((n - r0 < kRrRows) ? (n - r0) : kRrRows);
      mbar_wait(&sm->full[s], ph);
#pragma unroll
      for (int step = 0; step < kSteps; ++step) {
        const int k0 = wrow + 8 * step;
        const bool v0 = k0 + t < rows, v1 = k0 + t + 4 < rows;
        uint32_t fh[NB][4], fl[NB][4];                  // {row k0+t: col 2g, 2g+1 ; row k0+t+4: col 2g, 2g+1}
        float raw0[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int b = 0; b < NB; ++b) {
          const float2 u = *reinterpret_cast<const float2 *>(&sm->buf[s][b][(k0 + t) * BS + 2 * g]);
          const float2 w = *reinterpret_cast<const float2 *>(&sm->buf[s][b][(k0 + t + 4) * BS + 2 * g]);
          if (MODE == 0 && b == 0) { raw0[0] = u.x; raw0[1] = u.y; raw0[2] = w.x; raw0[3] = w.y; }
          split_tf32(v0 ? u.x : 0.f, fh[b][0], fl[b][0]);
          split_tf32(v0 ? u.y : 0.f, fh[b][1], fl[b][1]);
          split_tf32(v1 ? w.x : 0.f, fh[b][2], fl[b][2]);
          split_tf32(v1 ? w.y : 0.f, fh[b][3], fl[b][3]);
        }
        if (step == kSteps - 1) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&sm->empty[s]);    // operands are in registers: release the stage early
        }
        if constexpr (MODE == 0) {
          // CholQR squares the condition number of the block, so B'B gets fp32-exact products: a third TF32 term
          // (11 + 11 + 2 mantissa bits represent an fp32 value exactly) and the six products above 2^-33.
          uint32_t fm[4], fs[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float x = (e < 2 ? v0 : v1) ? raw0[e] : 0.f;
            const float r1 = x - __uint_as_float(fh[0][e]);
            fm[e] = to_tf32(r1);                                   // == fl[0][e]
            fs[e] = to_tf32(r1 - __uint_as_float(fm[e]));
          }
          // two independent accumulator chains per n-tile (small terms / leading terms), interleaved over nt
#pragma unroll
          for (int nt = 0; nt < 2; ++nt) mma_tf32(acc_small[nt], fs, fh[0][nt], fh[0][2 + nt]);
#pragma unroll
          for (int nt = 0; nt < 2; ++nt) mma_tf32(acc[0][nt], fm, fh[0][nt], fh[0][2 + nt]);
#pragma unroll
          for (int nt = 0; nt < 2; ++nt) mma_tf32(acc_small[nt], fh[0], fs[nt], fs[2 + nt]);
#pragma unroll
          for (int nt = 0; nt < 2; ++nt) mma_tf32(acc[0][nt], fh[0], fm[nt], fm[2 + nt]);
#pragma unroll
          for (int nt = 0; nt < 2; ++nt) mma_tf32(acc_small[nt], fm, fm[nt], fm[2 + nt]);
#pragma unroll
          for (int nt = 0; nt < 2; ++nt) mma_tf32(acc[0][nt], fh[0], fh[0][nt], fh[0][2 + nt]);
        } else if (half == 0) {
          // term by term over all (product, n-tile) accumulators: consecutive MMAs are independent
#pragma unroll
          for (int term = 0; term < 3; ++term)
#pragma unroll
            for (int q = 0; q < NPW; ++q) {
              const int lb = kL[q], rb = kR[q];
#pragma unroll
              for (int nt = 0; nt < 2; ++nt) {
                if (term == 0) mma_tf32(acc[q][nt], fl[lb], fh[rb][nt], fh[rb][2 + nt]);       // small terms first
                else if (term == 1) mma_tf32(acc[q][nt], fh[lb], fl[rb][nt], fl[rb][2 + nt]);
                else mma_tf32(acc[q][nt], fh[lb], fh[rb][nt], fh[rb][2 + nt]);
              }
            }
        } else if constexpr (WITH_P) {
#pragma unroll
          for (int term = 0; term < 3; ++term)
#pragma unroll
            for (int q = 0; q < NPW; ++q) {
              const int lb = kL[4 + q], rb = kR[4 + q];
#pragma unroll
              for (int nt = 0; nt < 2; ++nt) {
                if (term == 0) mma_tf32(acc[q][nt], fl[lb], fh[rb][nt], fh[rb][2 + nt]);
                else if (term == 1) mma_tf32(acc[q][nt], fh[lb], fl[rb][nt], fl[rb][2 + nt]);
                else mma_tf32(acc[q][nt], fh[lb], fh[rb][nt], fh[rb][2 + nt]);
              }
            }
        }
      }
      if constexpr (!WITH_P) {
#pragma unroll
        for (int p = 0; p < NPW; ++p)
#pragma unroll
          for (int nt = 0; nt < 2; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              tot[p][nt][e] += acc[p][nt][e];
              acc[p][nt][e] = 0.f;
            }
      }
    }
    if constexpr (!WITH_P) {
#pragma unroll
      for (int p = 0; p < NPW; ++p)
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[p][nt][e] = tot[p][nt][e];
    }
  }
  if constexpr (MODE == 0) {
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[0][nt][e] += acc_small[nt][e];
  }
  __syncthreads();   // all TMA data consumed: the ring memory is reused for the cross-warp reduction
  double(*red)[256] = reinterpret_cast<double(*)[256]>(smem_raw);
  static_assert(sizeof(RrSmem<MODE>) >= sizeof(double) * kRrConsumerWarps * 256, "reduction scratch does not fit");
  constexpr int kOwners = WITH_P ? 8 : kRrConsumerWarps;   // warps that hold a partial of a given product
  for (int q = 0; q < NPW; ++q) {
    // round q publishes product q (warps of half 0) and, with P, product 4+q (half 1) side by side
    if (warp < kRrConsumerWarps) {
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int i = 2 * g + (e >> 1);               // m = g (+8)  <-> column 2g (+1) of the left block
          const int j = 2 * (2 * t + (e & 1)) + nt;     // n = 2t (+1) <-> column 2n + nt of the right block
          red[warp][i * 16 + j] = (double)acc[q][nt][e];
        }
    }
    __syncthreads();
    if (tid < 256 * (WITH_P ? 2 : 1)) {
      const int h = tid >> 8, el = tid & 255;
      double s = 0.0;
      for (int w = 0; w < kOwners; ++w) s += red[h * 8 + w][el];
      partials[((size_t)blockIdx.x * NP + 4 * h + q) * 256 + el] = s;
    }
    __syncthreads();
  }
  if (tid == 0) {
    __threadfence();
    is_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  if (tid < 256) {
    for (int p = 0; p < NP; ++p) {
      double s = 0.0;
      for (unsigned int blk = 0; blk < gridDim.x; ++blk) s += __ldcg(&partials[((size_t)blk * NP + p) * 256 + tid]);
      out[p * 256 + tid] = s;
    }
  }
  if (tid == 0) *ticket = 0u;
}

// dst[:, k] = src[:, idx[k]] for k < bs, zero beyond  (update_active! :557-562)
template <typename T>
__global__ void __launch_bounds__(kThreads) k_gather_cols(T *__restrict__ dst, const T *__restrict__ src, int64_t n,
                                                          int bs, const int *__restrict__ idx) {
  __shared__ int sidx[BS];
  if (threadIdx.x < BS) sidx[threadIdx.x] = threadIdx.x < bs ? idx[threadIdx.x] : -1;
  __syncthreads();
  for (int64_t r = blockIdx.x * (int64_t)kThreads + threadIdx.x; r < n; r += (int64_t)gridDim.x * kThreads) {
    T in[BS], out[BS];
    load_row<T>(src + r * BS, in);
#pragma unroll
    for (int k = 0; k < BS; ++k) {
      T v = (T)0;
#pragma unroll
      for (int j = 0; j < BS; ++j)
        if (sidx[k] == j) v = in[j];
      out[k] = v;
    }
    store_row<T>(dst + r * BS, out);
  }
}

// precond!(R[:,1:bs]) with a Jacobi M: R[:,j] ./= d  (:236-242)
template <typename T>
__global__ void __launch_bounds__(kThreads) k_block_jacobi(T *__restrict__ X, int64_t n, const T *__restrict__ d) {
  for (int64_t r = blockIdx.x * (int64_t)kThreads + threadIdx.x; r < n; r += (int64_t)gridDim.x * kThreads) {
    T v[BS];
    load_row<T>(X + r * BS, v);
    const T di = d[r];
#pragma unroll
    for (int j = 0; j < BS; ++j) v[j] = v[j] / di;
    store_row<T>(X + r * BS, v);
  }
}

template <typename T>
struct Lobpcg {
  b200_ctx *ctx;
  const b200_csr *A;
  int64_t n;
  int sizeX;
  T *X, *AX, *R, *AR, *P, *AP, *gR, *gP, *gAP;   // row-major blocks; g*: gather scratch (first partial mask)
  double *gram_partials, *d_gram;                // device Gram output: 4 * 256 doubles
  T *d_small;                                    // V (3*256) + lambda (16) + U (256)
  int *d_idx;
  DevBuf scratch;
  // multi-GPU: packed boundary rows out / halo rows in (rows x 16), carved from the context workspace: a cudaMalloc / cudaFree
  // pair per solve costs tens of milliseconds once peer mappings exist (measured: 40 instead of 150 steps/s on 2 GPUs)
  struct { void *p = nullptr; } send_blk, halo_blk;
  int grid_gram, grid_vec, grid_spmm;

  template <int NR>
  int gram_launch(const T *L, const T *const *Rb) {
    const size_t smem = sizeof(GramSmem<T, NR>);
    B200_SMEM_ATTR_ONCE(ctx, smem, k_gram<T, NR>);
    k_gram<T, NR><<<grid_gram, kGramThreads, smem, ctx->stream>>>(L, Rb[0], Rb[NR > 1 ? 1 : 0], Rb[NR > 2 ? 2 : 0],
                                                                  Rb[NR > 3 ? 3 : 0], Rb[0] == L ? 1 : 0, n,
                                                                  gram_partials, ctx->red.ticket, d_gram);
    return B200_OK;
  }

  int gram(const T *L, const T *const *Rb, int nr, double *host_out /* nr*256 */) {
    {
      ProfScope prof(ctx, 1);
      if (nr == 1) B200_TRY(gram_launch<1>(L, Rb));
      else B200_TRY(gram_launch<2>(L, Rb));
    }
    B200_LAUNCH_CHECK(ctx);
    B200_TRY(allreduce_sum_dev(ctx, d_gram, 256 * nr));   // row slabs: global Gram = sum of the slabs' Grams
    B200_CUDA(cudaMemcpyAsync(host_out, d_gram, sizeof(double) * 256 * nr, cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA(cudaStreamSynchronize(ctx->stream));
    return B200_OK;
  }

  // fp32 blocks go through the tensor-pipe kernels unless the option "lobpcg_mma" is 0
  bool use_tc() const { return sizeof(T) == 4 && ctx->opt_lobpcg_mma != 0; }

  int gram_rr(bool with_p, const T *X_, const T *R_, const T *AR_, const T *P_, const T *AP_, double *host_out) {
    if constexpr (sizeof(T) == 4) {
      RrArgs ra;
      ra.blk[0] = X_; ra.blk[1] = R_; ra.blk[2] = AR_;
      ra.blk[3] = with_p ? P_ : X_; ra.blk[4] = with_p ? AP_ : X_;
      ra.n = n;
      B200_SMEM_ATTR_ONCE(ctx, sizeof(RrSmem<2>), k_gram_rr_tc<2>);
      B200_SMEM_ATTR_ONCE(ctx, sizeof(RrSmem<1>), k_gram_rr_tc<1>);
      {
        ProfScope prof(ctx, 1);
        if (with_p && ctx->opt_lobpcg_mma == 1) {
          // steady state: the eight products on wgmma (lobpcg_gram_wgmma.cuh); same output format
          WgArgs wa;
          for (int b = 0; b < 5; ++b) wa.blk[b] = ra.blk[b];
          wa.n = n;
          B200_SMEM_ATTR_ONCE(ctx, sizeof(WgSmem), k_gram_wgmma);
          k_gram_wgmma<<<grid_gram, kWgThreads, sizeof(WgSmem), ctx->stream>>>(wa, gram_partials, ctx->red.ticket, d_gram);
        } else if (with_p)
          k_gram_rr_tc<2><<<grid_gram, kRrThreads, sizeof(RrSmem<2>), ctx->stream>>>(ra, gram_partials,
                                                                                     ctx->red.ticket, d_gram);
        else
          k_gram_rr_tc<1><<<grid_gram, kRrThreads, sizeof(RrSmem<1>), ctx->stream>>>(ra, gram_partials,
                                                                                     ctx->red.ticket, d_gram);
      }
      B200_LAUNCH_CHECK(ctx);
      B200_TRY(allreduce_sum_dev(ctx, d_gram, 256 * (with_p ? 8 : 3)));
      B200_CUDA(cudaMemcpyAsync(host_out, d_gram, sizeof(double) * 256 * (with_p ? 8 : 3), cudaMemcpyDeviceToHost,
                                ctx->stream));
      B200_CUDA(cudaStreamSynchronize(ctx->stream));
      return B200_OK;
    } else {
      (void)with_p; (void)X_; (void)R_; (void)AR_; (void)P_; (void)AP_; (void)host_out;
      B200_REQUIRE(false, "gram_rr: fp32 only");
    }
  }

  // G = B' B on the tensor pipe (fp32 blocks)
  int gram_self(const T *B_, double *host_out) {
    if constexpr (sizeof(T) == 4) {
      RrArgs ra;
      for (int b = 0; b < 5; ++b) ra.blk[b] = B_;
      ra.n = n;
      B200_SMEM_ATTR_ONCE(ctx, sizeof(RrSmem<0>), k_gram_rr_tc<0>);
      {
        ProfScope prof(ctx, 1);
        k_gram_rr_tc<0><<<grid_gram, kRrThreads, sizeof(RrSmem<0>), ctx->stream>>>(ra, gram_partials, ctx->red.ticket,
                                                                                   d_gram);
      }
      B200_LAUNCH_CHECK(ctx);
      B200_TRY(allreduce_sum_dev(ctx, d_gram, 256));
      B200_CUDA(cudaMemcpyAsync(host_out, d_gram, sizeof(double) * 256, cudaMemcpyDeviceToHost, ctx->stream));
      B200_CUDA(cudaStreamSynchronize(ctx->stream));
      return B200_OK;
    } else {
      (void)B_; (void)host_out;
      B200_REQUIRE(false, "gram_self: fp32 only");
    }
  }

  // CholQR (:365-393): blk is orthonormalised, ablk (its A-block) follows if given
  int cholqr(T *blk, T *ablk, int bs) {
    double G[256];
    if (use_tc()) {
      B200_TRY(gram_self(blk, G));
    } else {
      const T *rb[1] = {blk};
      B200_TRY(gram(blk, rb, 1, G));
    }
    std::vector<double> U((size_t)bs * bs);
    for (int i = 0; i < bs; ++i)
      for (int j = 0; j < bs; ++j) U[i + (size_t)j * bs] = i <= j ? G[i * 16 + j] : G[j * 16 + i];  // Hermitian(gram): upper
    if (dense::cholesky_upper(U.data(), bs, bs)) {
      set_error("PosDefException: CholQR Gram matrix is not positive definite (reference src/lobpcg.jl:380)");
      return B200_ERR_BREAKDOWN;
    }
    std::vector<T> Ut((size_t)bs * bs);
    for (size_t q = 0; q < Ut.size(); ++q) Ut[q] = (T)U[q];
    T *dU = d_small + 3 * 256 + 16;
    B200_CUDA(cudaMemcpyAsync(dU, Ut.data(), sizeof(T) * Ut.size(), cudaMemcpyHostToDevice, ctx->stream));
    {
      ProfScope prof(ctx, 2);
      k_rdiv<T><<<grid_vec, kThreads, 0, ctx->stream>>>(blk, ablk, ablk ? 2 : 1, bs, n, dU);
    }
    B200_LAUNCH_CHECK(ctx);
    B200_CUDA(cudaStreamSynchronize(ctx->stream));   // Ut is a host temporary
    return B200_OK;
  }

  // multi-GPU: the rows of Xin the neighbours' SpMM needs (the operator's send lists) -> their halo blocks
  int halo_block(const T *Xin) {
    if (ctx->world == 1 || (A->n_send == 0 && A->n_halo == 0)) return B200_OK;
    cudaStream_t st = ctx->stream;
    if (A->n_send) {
      k_pack_rows<T><<<stream_grid(ctx, A->n_send, kThreads / 4, 8), kThreads, 0, st>>>(A->send_idx, Xin, A->n_send,
                                                                                       (T *)send_blk.p);
      B200_LAUNCH_CHECK(ctx);
    }
    const ncclDataType_t nt = sizeof(T) == 8 ? ncclDouble : ncclFloat;
    B200_NCCL(ncclGroupStart());
    for (int p = 0; p < ctx->world; ++p) {
      if (p == ctx->rank) continue;
      if (A->send_count[p])
        B200_NCCL(ncclSend((const T *)send_blk.p + (size_t)BS * A->send_offset[p], (size_t)BS * A->send_count[p], nt, p,
                           ctx->comm, st));
      if (A->recv_count[p])
        B200_NCCL(ncclRecv((T *)halo_blk.p + (size_t)BS * A->recv_offset[p], (size_t)BS * A->recv_count[p], nt, p,
                           ctx->comm, st));
    }
    B200_NCCL(ncclGroupEnd());
    return B200_OK;
  }

  int spmm(const T *Xin, T *Yout) {
    B200_TRY(halo_block(Xin));
    ProfScope prof(ctx, 0);
    with_rowptr(A, [&](auto rowptr) {
      k_spmm_rm<T><<<grid_spmm, kThreads, 0, ctx->stream>>>(rowptr, A->colind, (const T *)A->vals, Xin,
                                                            (const T *)halo_blk.p, n, Yout);
      return 0;
    });
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
  }
};

template <typename T>
int lobpcg_impl(b200_ctx *ctx, const b200_csr *A, T *Xcm, int64_t ldx, const b200_lobpcg_opts *o,
                const b200_lobpcg_constraint *C, b200_lobpcg_result *res, double *lambda_host, double *resnorm_host) {
  cudaStream_t st = ctx->stream;
  const int64_t n = A->m_local;
  const int sizeX = o->blocksize;
  B200_REQUIRE(sizeX >= 1 && sizeX <= BS, "lobpcg: block size %d not in 1..%d", sizeX, BS);
  B200_REQUIRE(ldx == n, "lobpcg: X must be n x blocksize with leading dimension n");
  B200_REQUIRE(sizeX <= A->n_global, "X column dimension exceeds the row dimension");              // :833
  B200_REQUIRE(3 * (int64_t)sizeX <= A->n_global, "The LOBPCG algorithms is not stable to use when the matrix size is less "
               "than 3 times the block size. Please use a dense solver instead.");                 // :834
  const double eps = sizeof(T) == 8 ? 2.220446049250313e-16 : 1.1920928955078125e-07;
  const double tol = o->tol < 0 ? pow(eps, 0.3) : o->tol;                                           // :751
  const int64_t maxiter = o->maxiter < 0 ? 200 : o->maxiter;
  const T *jac = o->P.kind == B200_PREC_JACOBI ? (const T *)o->P.diag : nullptr;

  Lobpcg<T> L;
  L.ctx = ctx;
  L.A = A;
  L.n = n;
  L.sizeX = sizeX;
  L.grid_gram = (int)std::min<int64_t>(ctx->sm_count, (n + RC - 1) / RC);
  L.grid_vec = stream_grid(ctx, n, kThreads, 4);
  L.grid_spmm = stream_grid(ctx, n, kThreads / 4, 8);
  const size_t blk_bytes = align_up(sizeof(T) * (size_t)n * BS, 256);
  const size_t small_bytes = align_up(sizeof(T) * (3 * 256 + 16 + 256), 256);
  const size_t gram_bytes = sizeof(double) * ((size_t)L.grid_gram * 8 * 256 + 8 * 256 + 64);
  const size_t send_bytes = ctx->world > 1 ? align_up(sizeof(T) * BS * (size_t)std::max<int64_t>(A->n_send, 1), 256) : 0;
  const size_t halo_bytes = ctx->world > 1 ? align_up(sizeof(T) * BS * (size_t)std::max<int64_t>(A->n_halo, 1), 256) : 0;
  void *ws = nullptr;
  B200_TRY(ws_get(ctx, 6 * blk_bytes + small_bytes + align_up(gram_bytes, 256) + send_bytes + halo_bytes + 1024, &ws));
  char *p = (char *)ws;
  L.X = (T *)p; p += blk_bytes;
  L.AX = (T *)p; p += blk_bytes;
  L.R = (T *)p; p += blk_bytes;
  L.AR = (T *)p; p += blk_bytes;
  L.P = (T *)p; p += blk_bytes;
  L.AP = (T *)p; p += blk_bytes;
  L.d_small = (T *)p; p += small_bytes;
  L.gram_partials = (double *)p; p += sizeof(double) * (size_t)L.grid_gram * 8 * 256;
  L.d_gram = (double *)p; p += sizeof(double) * 8 * 256;
  double *d_norms = (double *)p; p += sizeof(double) * 64;
  L.d_idx = (int *)p;
  L.gR = L.gP = L.gAP = nullptr;
  if (ctx->world > 1) {
    char *q = (char *)ws + 6 * blk_bytes + small_bytes + align_up(gram_bytes, 256) + 256;
    L.send_blk.p = q;
    L.halo_blk.p = q + send_bytes;
  }
  k_to_rowmajor<T><<<L.grid_vec, kThreads, 0, st>>>(Xcm, L.X, n, sizeX);
  B200_LAUNCH_CHECK(ctx);
  if (C) B200_TRY(constraint_apply_block(ctx, C, L.X, BS, 1, sizeX));   // iterator.constr!(X, temp) :868 / :875

  std::vector<double> ritz(3 * sizeX, 0.0), residuals(sizeX, NAN);                                  // :473-477
  std::vector<char> mask(sizeX, 1);
  int bs = sizeX;
  int64_t iteration = 1;
  int status = B200_OK;

  auto upload_v_and_update = [&](const std::vector<double> &Z, int sub, const std::vector<int> &perm, int bs1,
                                 int bs2, const T *aR, const T *aAR, const T *aP, const T *aAP) -> int {
    // V[1:sub, 1:sizeX] = eigenvectors of the selected Ritz values (:625); split into x / r / p parts
    std::vector<T> Vb(3 * 256 + 16, (T)0);
    for (int j = 0; j < sizeX; ++j) {
      const double *z = &Z[(size_t)perm[j] * sub];
      for (int i = 0; i < sizeX; ++i) Vb[i * 16 + j] = (T)z[i];
      for (int i = 0; i < bs1; ++i) Vb[256 + i * 16 + j] = (T)z[sizeX + i];
      for (int i = 0; i < bs2; ++i) Vb[512 + i * 16 + j] = (T)z[sizeX + bs1 + i];
      Vb[768 + j] = (T)ritz[j];
    }
    B200_CUDA(cudaMemcpyAsync(L.d_small, Vb.data(), sizeof(T) * Vb.size(), cudaMemcpyHostToDevice, st));
    UpdateArgs ua;
    ua.X = L.X; ua.AX = L.AX; ua.P = L.P; ua.AP = L.AP; ua.R = L.R;
    ua.aR = aR; ua.aAR = aAR; ua.aP = aP; ua.aAP = aAP;
    ua.sizeX = sizeX; ua.bs1 = bs1; ua.bs2 = bs2; ua.n = n;
    {
      ProfScope prof(ctx, 3);
      if constexpr (sizeof(T) == 4) {
        if (L.use_tc()) {
          const int gtc = stream_grid(ctx, n, kThreads / 2, 2);
          k_update_tc<0><<<gtc, kThreads, 0, st>>>(ua, L.d_small, L.d_small + 768, nullptr, nullptr, nullptr);
          k_update_tc<1><<<gtc, kThreads, 0, st>>>(ua, L.d_small, L.d_small + 768, ctx->red.partials, ctx->red.ticket, d_norms);
        } else {
          k_update<T, 0><<<L.grid_vec, kThreads, 0, st>>>(ua, L.d_small, L.d_small + 768, nullptr, nullptr, nullptr);
          k_update<T, 1><<<L.grid_vec, kThreads, 0, st>>>(ua, L.d_small, L.d_small + 768, ctx->red.partials, ctx->red.ticket, d_norms);
        }
      } else {
        k_update<T, 0><<<L.grid_vec, kThreads, 0, st>>>(ua, L.d_small, L.d_small + 768, nullptr, nullptr, nullptr);
        k_update<T, 1><<<L.grid_vec, kThreads, 0, st>>>(ua, L.d_small, L.d_small + 768, ctx->red.partials, ctx->red.ticket, d_norms);
      }
      ctx->launches++;   // two launches: the second is counted by B200_LAUNCH_CHECK below
    }
    B200_LAUNCH_CHECK(ctx);
    B200_TRY(allreduce_sum_dev(ctx, d_norms, BS));
    double nn[BS];
    B200_CUDA(cudaMemcpyAsync(nn, d_norms, sizeof(double) * BS, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    for (int j = 0; j < sizeX; ++j) residuals[j] = sqrt(nn[j]);                                     // :545
    return B200_OK;
  };
  auto select = [&](const std::vector<double> &w, int sub, std::vector<int> &perm) {               // :623-624
    perm.resize(sub);
    for (int i = 0; i < sub; ++i) perm[i] = i;
    if (o->largest) std::stable_sort(perm.begin(), perm.end(), [&](int a, int b) { return w[a] > w[b]; });
    for (int j = 0; j < sizeX; ++j) ritz[j] = w[perm[j]];
  };

  while (iteration <= maxiter) {                                                                    // :880
    if (iteration == 1) {                                                                           // :695-703
      status = L.cholqr(L.X, nullptr, sizeX);                                                       // ortho_AB_mul_X! :524-532
      if (status) break;
      B200_TRY(L.spmm(L.X, L.AX));
      double G[256];
      const T *rb[1] = {L.AX};
      B200_TRY(L.gram(L.X, rb, 1, G));                                                              // XAX :262
      std::vector<double> Am((size_t)sizeX * sizeX), w, Z;
      for (int i = 0; i < sizeX; ++i)
        for (int j = 0; j < sizeX; ++j) Am[i + (size_t)j * sizeX] = i <= j ? G[i * 16 + j] : G[j * 16 + i];
      if (dense::sym_eig(Am, sizeX, w, Z)) { status = B200_ERR_BREAKDOWN; set_error("eigen! did not converge"); break; }
      std::vector<int> perm;
      select(w, sizeX, perm);
      B200_TRY(upload_v_and_update(Z, sizeX, perm, 0, 0, nullptr, nullptr, nullptr, nullptr));      // update_X_P!(0,0)
    } else {
      const bool full = bs == sizeX;
      const bool with_p = iteration > 2;
      T *aR = L.R, *aP = L.P, *aAP = L.AP;
      if (!full) {                                                                                  // update_active! :557-562
        if (!L.gR) {
          B200_TRY(L.scratch.alloc(3 * blk_bytes));
          L.gR = (T *)L.scratch.p;
          L.gP = (T *)((char *)L.scratch.p + blk_bytes);
          L.gAP = (T *)((char *)L.scratch.p + 2 * blk_bytes);
        }
        int idx[BS], k = 0;
        for (int j = 0; j < sizeX; ++j)
          if (mask[j]) idx[k++] = j;
        B200_CUDA(cudaMemcpyAsync(L.d_idx, idx, sizeof(int) * bs, cudaMemcpyHostToDevice, st));
        k_gather_cols<T><<<L.grid_vec, kThreads, 0, st>>>(L.gR, L.R, n, bs, L.d_idx);
        if (with_p) {
          k_gather_cols<T><<<L.grid_vec, kThreads, 0, st>>>(L.gP, L.P, n, bs, L.d_idx);
          k_gather_cols<T><<<L.grid_vec, kThreads, 0, st>>>(L.gAP, L.AP, n, bs, L.d_idx);
        }
        B200_LAUNCH_CHECK(ctx);
        B200_CUDA(cudaStreamSynchronize(st));
        aR = L.gR; aP = L.gP; aAP = L.gAP;
      }
      if (jac) {                                                                                    // precond_constr! :564-569
        k_block_jacobi<T><<<L.grid_vec, kThreads, 0, st>>>(aR, n, jac);
        B200_LAUNCH_CHECK(ctx);
      }
      if (C) B200_TRY(constraint_apply_block(ctx, C, aR, BS, 1, bs));                               // constr!(R[:,1:bs]) :567
      status = L.cholqr(aR, nullptr, bs);                                                           // :524-532
      if (status) break;
      B200_TRY(L.spmm(aR, L.AR));
      if (with_p) {
        status = L.cholqr(aP, aAP, bs);                                                             // :733
        if (status) break;
      }
      const int n1 = sizeX, n2 = bs, n3 = with_p ? bs : 0, sub = n1 + n2 + n3;
      std::vector<double> gA((size_t)sub * sub, 0.0), gB((size_t)sub * sub, 0.0);
      auto setA = [&](int i, int j, double v) { gA[i + (size_t)j * sub] = v; gA[j + (size_t)i * sub] = v; };
      auto setB = [&](int i, int j, double v) { gB[i + (size_t)j * sub] = v; gB[j + (size_t)i * sub] = v; };
      for (int i = 0; i < n1; ++i) setA(i, i, ritz[i]);                                             // Diagonal(lambda) :289
      for (int i = 0; i < sub; ++i) setB(i, i, 1.0);                                                // I! :315,322,331
      // Gram blocks, slot p at G + 256 p:  0 X'AR  1 X'R  2 R'AR  3 X'AP  4 X'P  5 R'P  6 AR'P  7 P'AP
      double G[8 * 256];
      if (L.use_tc()) {
        B200_TRY(L.gram_rr(with_p, L.X, aR, L.AR, aP, aAP, G));                                     // one pass
      } else {
        {             // X' [AR, R]  (and X' [AP, P]): two right blocks per launch keeps the 4x4 tiles in registers
          const T *rb[2] = {L.AR, aR};
          B200_TRY(L.gram(L.X, rb, 2, G));
          if (with_p) {
            const T *rb2[2] = {aAP, aP};
            B200_TRY(L.gram(L.X, rb2, 2, G + 3 * 256));
          }
        }
        double G2[2 * 256];
        if (with_p) {   // R' [AR, P]
          const T *rb[2] = {L.AR, aP};
          B200_TRY(L.gram(aR, rb, 2, G2));
          memcpy(G + 2 * 256, G2, sizeof(double) * 256);
          memcpy(G + 5 * 256, G2 + 256, sizeof(double) * 256);
          const T *rb1[1] = {aP};
          B200_TRY(L.gram(L.AR, rb1, 1, G + 6 * 256));                                              // AR' P
          const T *rb2[1] = {aAP};
          B200_TRY(L.gram(aP, rb2, 1, G + 7 * 256));                                                // P' AP
        } else {
          const T *rb[1] = {L.AR};
          B200_TRY(L.gram(aR, rb, 1, G + 2 * 256));
        }
      }
      for (int i = 0; i < n1; ++i)
        for (int j = 0; j < n2; ++j) {
          setA(i, n1 + j, G[i * 16 + j]);                                                           // XAR :265
          setB(i, n1 + j, G[256 + i * 16 + j]);                                                     // XBR :270
          if (with_p) {
            setA(i, n1 + n2 + j, G[3 * 256 + i * 16 + j]);                                          // XAP :264
            setB(i, n1 + n2 + j, G[4 * 256 + i * 16 + j]);                                          // XBP :269
          }
        }
      for (int i = 0; i < n2; ++i)
        for (int j = i; j < n2; ++j) setA(n1 + i, n1 + j, G[2 * 256 + i * 16 + j]);                 // RAR :266 (upper triangle)
      if (with_p) {
        for (int i = 0; i < n2; ++i)
          for (int j = 0; j < n3; ++j) {
            setB(n1 + i, n1 + n2 + j, G[5 * 256 + i * 16 + j]);                                     // RBP :271
            setA(n1 + i, n1 + n2 + j, G[6 * 256 + i * 16 + j]);                                     // RAP :267
          }
        for (int i = 0; i < n3; ++i)
          for (int j = i; j < n3; ++j) setA(n1 + n2 + i, n1 + n2 + j, G[7 * 256 + i * 16 + j]);     // PAP :268
      }
      std::vector<double> w, Z;
      const int info = dense::sym_eig_generalized(gA, gB, sub, w, Z);                               // :622
      if (info) {
        status = B200_ERR_BREAKDOWN;
        set_error("PosDefException in the Rayleigh-Ritz problem (gramB not positive definite, info=%d)", info);
        break;
      }
      std::vector<int> perm;
      select(w, sub, perm);
      B200_TRY(upload_v_and_update(Z, sub, perm, n2, n3, aR, L.AR, aP, aAP));
    }
    if (iteration - 1 < o->trace_cap) {                            // log = true: LOBPCGState(iteration, residuals, ritz_values) :744-745
      for (int j = 0; j < sizeX; ++j) {
        if (o->trace_resnorm) o->trace_resnorm[(iteration - 1) * sizeX + j] = residuals[j];
        if (o->trace_ritz) o->trace_ritz[(iteration - 1) * sizeX + j] = ritz[j];
      }
    }
    bs = 0;                                                                                         // update_mask! :549-555
    for (int j = 0; j < sizeX; ++j) {
      mask[j] = o->fixed_iterations ? 1 : (residuals[j] > tol);
      bs += mask[j];
    }
    if (bs == 0) break;                                                                             // :885
    iteration += 1;                                                                                 // :886
  }
  k_to_colmajor<T><<<L.grid_vec, kThreads, 0, st>>>(L.X, Xcm, n, sizeX);
  B200_LAUNCH_CHECK(ctx);
  bool conv = true;
  for (int j = 0; j < sizeX; ++j) {
    if (lambda_host) lambda_host[j] = ritz[j];
    if (resnorm_host) resnorm_host[j] = residuals[j];
    conv = conv && (residuals[j] <= tol);
  }
  if (res) {
    res->iterations = iteration;                                                                    // :890
    res->converged = conv;
    res->status = status;
  }
  B200_CUDA(cudaStreamSynchronize(st));
  return status;
}

}  // namespace

extern "C" {

int b200_lobpcg_solve(b200_ctx *ctx, const b200_csr *A, void *X_dev, int64_t ldx, const b200_lobpcg_opts *opts,
                      b200_lobpcg_result *res, double *lambda_host, double *resnorm_host) {
  B200_TRY(real_only(A, "b200_lobpcg_solve"));
  B200_REQUIRE(ctx && A && X_dev && opts, "NULL argument");
  B200_REQUIRE(A->ctx == ctx, "operator belongs to another context");
  B200_REQUIRE(is_square(A), "this solver needs a square operator (got %lld x %lld)", (long long)A->m_global,
               (long long)A->n_global);
  B200_REQUIRE(opts->P.kind == B200_PREC_IDENTITY || (opts->P.kind == B200_PREC_JACOBI && opts->P.diag),
               "unsupported preconditioner P (this engine takes Identity or Jacobi)");
  B200_CUDA(cudaSetDevice(ctx->device));
  return A->dtype == B200_F64
             ? lobpcg_impl<double>(ctx, A, (double *)X_dev, ldx, opts, nullptr, res, lambda_host, resnorm_host)
             : lobpcg_impl<float>(ctx, A, (float *)X_dev, ldx, opts, nullptr, res, lambda_host, resnorm_host);
}

int b200_lobpcg_solve_constrained(b200_ctx *ctx, const b200_csr *A, void *X_dev, int64_t ldx,
                                  const b200_lobpcg_opts *opts, const b200_lobpcg_constraint *C,
                                  b200_lobpcg_result *res, double *lambda_host, double *resnorm_host) {
  B200_TRY(real_only(A, "b200_lobpcg_solve_constrained"));
  B200_REQUIRE(ctx && A && X_dev && opts, "NULL argument");
  B200_REQUIRE(A->ctx == ctx, "operator belongs to another context");
  B200_REQUIRE(is_square(A), "this solver needs a square operator (got %lld x %lld)", (long long)A->m_global,
               (long long)A->n_global);
  B200_REQUIRE(opts->P.kind == B200_PREC_IDENTITY || (opts->P.kind == B200_PREC_JACOBI && opts->P.diag),
               "unsupported preconditioner P (this engine takes Identity or Jacobi)");
  if (C) {
    B200_REQUIRE(C->ctx == ctx && C->dtype == A->dtype && C->n == A->m_local,
                 "the constraint does not match the operator (context, eltype or local rows)");
    B200_REQUIRE(!C->BY, "a generalized-problem constraint needs b200_lobpcg_solve_op");
  }
  B200_CUDA(cudaSetDevice(ctx->device));
  return A->dtype == B200_F64
             ? lobpcg_impl<double>(ctx, A, (double *)X_dev, ldx, opts, C, res, lambda_host, resnorm_host)
             : lobpcg_impl<float>(ctx, A, (float *)X_dev, ldx, opts, C, res, lambda_host, resnorm_host);
}

/* TEST HOOK (tests/test_gpu_lobpcg.py): the eight Rayleigh-Ritz Gram products of five row-major n x 16 fp32 blocks
 * (X, R, AR, P, AP: device pointers) through one of the engine's kernels -- variant 1: wgmma (k_gram_wgmma),
 * variant 2: legacy mma.sync (k_gram_rr_tc<2>).  out_host: 8 x 256 doubles, out[p * 256 + i * 16 + j]. */
int b200_debug_lobpcg_gram_rr(b200_ctx *ctx, const void *const *blk_dev, int64_t n, int variant, double *out_host) {
  B200_REQUIRE(ctx && blk_dev && out_host && n >= 0 && (variant == 1 || variant == 2 || (variant > 100 && variant < 1000)),
               "bad arguments");
  B200_CUDA(cudaSetDevice(ctx->device));
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(ctx->sm_count, (n + RC - 1) / RC));
  DevBuf part, outd;
  B200_TRY(part.alloc(sizeof(double) * (size_t)grid * 8 * 256));
  B200_TRY(outd.alloc(sizeof(double) * 8 * 256));
  if (variant != 2) {
    WgArgs wa;
    for (int b = 0; b < 5; ++b) wa.blk[b] = (const float *)blk_dev[b];
    wa.n = n;
    if (variant > 100) wa.drain = variant - 100;    // variant 100 + d: wgmma kernel with d stages per accumulator hand-over
    B200_SMEM_ATTR_ONCE(ctx, sizeof(WgSmem), k_gram_wgmma);
    k_gram_wgmma<<<grid, kWgThreads, sizeof(WgSmem), ctx->stream>>>(wa, (double *)part.p, ctx->red.ticket, (double *)outd.p);
  } else {
    RrArgs ra;
    for (int b = 0; b < 5; ++b) ra.blk[b] = (const float *)blk_dev[b];
    ra.n = n;
    B200_SMEM_ATTR_ONCE(ctx, sizeof(RrSmem<2>), k_gram_rr_tc<2>);
    k_gram_rr_tc<2><<<grid, kRrThreads, sizeof(RrSmem<2>), ctx->stream>>>(ra, (double *)part.p, ctx->red.ticket, (double *)outd.p);
  }
  B200_LAUNCH_CHECK(ctx);
  B200_CUDA(cudaMemcpyAsync(out_host, outd.p, sizeof(double) * 8 * 256, cudaMemcpyDeviceToHost, ctx->stream));
  B200_CUDA(cudaStreamSynchronize(ctx->stream));
  return B200_OK;
}

int b200_dense_sygv_host(int n, const double *A, const double *B, double *w, double *Z) {
  B200_REQUIRE(n >= 1 && n <= 64 && A && w && Z, "bad arguments");
  std::vector<double> Am(A, A + (size_t)n * n), wv, Zv;
  int info;
  if (B) {
    std::vector<double> Bm(B, B + (size_t)n * n);
    info = dense::sym_eig_generalized(Am, Bm, n, wv, Zv);
  } else {
    info = dense::sym_eig(Am, n, wv, Zv);
  }
  if (info) {
    set_error("dense symmetric eigen-solver failed (info=%d)", info);
    return B200_ERR_BREAKDOWN;
  }
  memcpy(w, wv.data(), sizeof(double) * n);
  memcpy(Z, Zv.data(), sizeof(double) * (size_t)n * n);
  return B200_OK;
}

}  // extern "C"
