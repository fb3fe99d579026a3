// spmv.cuh -- CSR SpMV building blocks shared by the solver kernels.
//
// Layout in HBM: rowptr I (m+1; I = int, or int64_t for operators of 2^31 or more nonzeros, csr.cuh), colind int32
// (nnz, local extended index), vals T (nnz), all contiguous in row order => a contiguous chunk of rows is a contiguous
// chunk of the colind/vals streams (12 B/nnz in fp64, read exactly once per SpMV); x is gathered through L1/L2.
//
// Algorithmic bytes per SpMV (SURVEY.md section 8d): nnz*(V+4) + (m+1)*sizeof(I) + 2*m*V.
#pragma once
#include <type_traits>

#include "csr.cuh"

namespace b200 {

#ifdef __CUDACC__

// lanes-per-row selection: smallest power of two >= average row length, in [2, 32]
inline int pick_lpr(double avg_row_nnz) {
  int l = 2;
  while (l < 32 && l < avg_row_nnz) l <<= 1;
  return l;
}

// f(std::integral_constant<int, L>{}) for the compile-time lanes per row L == lpr, a power of two in [MIN, 32] (anything
// else takes 32).  MIN keeps lane counts that no operator is given out of the instantiated kernels.
template <int MIN, typename F>
inline auto with_lpr(int lpr, F &&f) {
  if constexpr (MIN < 32) {
    if (lpr != MIN) return with_lpr<2 * MIN>(lpr, static_cast<F &&>(f));
  }
  return f(std::integral_constant<int, MIN>{});
}

// x gather from the extended vector: own slab or halo buffer
template <typename T>
struct XView {
  const T *__restrict__ x;     // own rows [0, m)
  const T *__restrict__ halo;  // halo values, already shifted by -m (halo_shifted[col] valid for col >= m)
  int m;
  __device__ __forceinline__ T operator()(int col) const { return col < m ? __ldg(x + col) : __ldg(halo + col); }
};
template <typename T>
inline XView<T> make_xview(const b200_csr *A, const void *x_dev, bool peer_halo = false) {
  XView<T> v;
  v.x = (const T *)x_dev;
  const void *h = peer_halo ? A->halo_peer : A->halo;   // which halo buffer the preceding exchange filled
  v.halo = h ? (const T *)h - A->m_local : (const T *)x_dev;
  v.m = (int)A->m_local;
  return v;
}

// One sub-warp of LPR lanes computes (A x)[row]; result valid in all LPR lanes.
template <typename T, int LPR, typename XV, typename I>
__device__ __forceinline__ T row_dot(const I *__restrict__ rowptr, const int *__restrict__ colind,
                                     const T *__restrict__ vals, const XV &xv, int64_t row, int sub) {
  const I b = __ldg(rowptr + row), e = __ldg(rowptr + row + 1);
  const uint64_t pol = policy_evict_first();
  T acc = (T)0;
  for (I k = b + sub; k < e; k += LPR) {
    const int c = ld_stream<int>(colind + k, pol);
    const T a = ld_stream<T>(vals + k, pol);
    acc += a * xv(c);
  }
#pragma unroll
  for (int o = LPR >> 1; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o, LPR);
  return acc;
}

constexpr int kRowsThreads = 256;   // block size of the sub-warp form

// Sub-warp (LPR lanes) per row over all rows; blocks stride the rows in interleaved chunks so that all resident blocks
// work on neighbouring rows (keeps the x planes of a stencil matrix in L2).  The epilogue contract is the streamed
// bodies' (spmv_stream.cuh): the lane that owns a row result calls epi.pre(row) and then epi(row, value, pre).
template <typename T, int LPR, typename XV, typename Epi, typename I>
__device__ __forceinline__ void spmv_rows(const I *__restrict__ rowptr, const int *__restrict__ colind,
                                          const T *__restrict__ vals, const XV &xv, int64_t m, Epi &epi) {
  constexpr int ROWS = kRowsThreads / LPR;
  const int sub = threadIdx.x % LPR;
  const int rib = threadIdx.x / LPR;
  for (int64_t base = (int64_t)blockIdx.x * ROWS; base < m; base += (int64_t)gridDim.x * ROWS) {
    const int64_t row = base + rib;
    const bool own = row < m && sub == 0;
    const T pre = own ? epi.pre(row) : (T)0;
    const T v = row_dot<T, LPR>(rowptr, colind, vals, xv, row < m ? row : (m - 1), sub);
    if (own) epi(row, v, pre);
  }
}

#endif  // __CUDACC__

}  // namespace b200
