// spmv_launch.cuh -- the three SpMV kernels and the one launch path shared by mul! (b200_spmv), cg!'s K2 and MINRES' Ka.
//
// A caller differs from the others only in its epilogue, a struct passed to the kernel by value:
//   bool begin()                         all threads, before the body; false = the whole block returns (block-uniform)
//   T pre(int64_t row)                   the epilogue's own per-row operand, requested ahead of the row's gathers
//   void operator()(int64_t row, T v, T pre)   once per row, by the thread that owns the row result v = (A x)[row]
//   template <int THREADS> void end(double *red)   all threads, after the body; red: THREADS / 32 doubles of shared memory
//   bool rev()                           the streamed forms sweep the tiles from the last to the first (constexpr false
//                                        where a caller never reverses, which keeps the sweep arithmetic out of its kernels)
// Which of the three forms serves an operator is decided here alone (launch_spmv_fused).
//
// Every kernel comes as two overloads, for int and for int64_t row offsets (csr.cuh), sharing one body.  Overloads rather
// than a template parameter keep the symbols of the 4-byte kernels, which profiles and ptxas reports are keyed on.
#pragma once
#include "spmv_stream.cuh"

namespace b200 {

#ifdef __CUDACC__

template <typename T, int LPR, typename I, typename XV, typename Epi>
__device__ __forceinline__ void spmv_rows_kernel(const I *__restrict__ rowptr, const int *__restrict__ colind,
                                                 const T *__restrict__ vals, const XV &xv, int64_t m, Epi &epi) {
  if (!epi.begin()) return;
  __shared__ double red[kRowsThreads / 32];
  spmv_rows<T, LPR>(rowptr, colind, vals, xv, m, epi);
  epi.template end<kRowsThreads>(red);
}

template <typename T, int LPR, typename Epi>
__global__ void __launch_bounds__(kRowsThreads) k_spmv_rows(const int *__restrict__ rowptr, const int *__restrict__ colind,
                                                            const T *__restrict__ vals, XView<T> xv, int64_t m, Epi epi) {
  spmv_rows_kernel<T, LPR>(rowptr, colind, vals, xv, m, epi);
}
template <typename T, int LPR, typename Epi>
__global__ void __launch_bounds__(kRowsThreads) k_spmv_rows(const int64_t *__restrict__ rowptr, const int *__restrict__ colind,
                                                            const T *__restrict__ vals, XView<T> xv, int64_t m, Epi epi) {
  spmv_rows_kernel<T, LPR>(rowptr, colind, vals, xv, m, epi);
}

// Complex operators (single-GPU, sub-warp form only): x is the whole operand (no halo); VEC = one vector __ldg per
// gathered element, chosen by the launcher only when x is aligned to 2 sizeof(R), else two scalar loads.
template <typename R, bool VEC>
struct XViewC {
  const cplx<R> *__restrict__ x;
  __device__ __forceinline__ cplx<R> operator()(int col) const {
    if constexpr (VEC) {
      return __ldg(x + col);
    } else {
      const R *p = reinterpret_cast<const R *>(x + col);
      return cplx<R>(__ldg(p), __ldg(p + 1));
    }
  }
};

template <typename R, int LPR, bool VEC, typename Epi>
__global__ void __launch_bounds__(kRowsThreads) k_spmv_rows_cplx(const int *__restrict__ rowptr, const int *__restrict__ colind,
                                                                 const cplx<R> *__restrict__ vals, XViewC<R, VEC> xv,
                                                                 int64_t m, Epi epi) {
  spmv_rows_kernel<cplx<R>, LPR>(rowptr, colind, vals, xv, m, epi);
}
template <typename R, int LPR, bool VEC, typename Epi>
__global__ void __launch_bounds__(kRowsThreads) k_spmv_rows_cplx(const int64_t *__restrict__ rowptr, const int *__restrict__ colind,
                                                                 const cplx<R> *__restrict__ vals, XViewC<R, VEC> xv,
                                                                 int64_t m, Epi epi) {
  spmv_rows_kernel<cplx<R>, LPR>(rowptr, colind, vals, xv, m, epi);
}

template <typename T, int LPR, typename I, typename Epi>
__device__ __forceinline__ void spmv_csr_stream_kernel(const I *__restrict__ rowptr, const int *__restrict__ colind,
                                                       const T *__restrict__ vals, const XView<T> &xv, int64_t m, Epi &epi) {
  if (!epi.begin()) return;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ double red[kStreamThreads / 32];
  spmv_stream_tiles<T, LPR>(rowptr, colind, vals, xv, m, epi, reinterpret_cast<StreamSmem<T, I> *>(smem_raw), epi.rev());
  epi.template end<kStreamThreads>(red);
}

template <typename T, int LPR, typename Epi>
__global__ void __launch_bounds__(kStreamThreads, kStreamCtasPerSm)
    k_spmv_csr_stream(const int *__restrict__ rowptr, const int *__restrict__ colind, const T *__restrict__ vals,
                      XView<T> xv, int64_t m, Epi epi) {
  spmv_csr_stream_kernel<T, LPR>(rowptr, colind, vals, xv, m, epi);
}
template <typename T, int LPR, typename Epi>
__global__ void __launch_bounds__(kStreamThreads, kStreamCtasPerSm)
    k_spmv_csr_stream(const int64_t *__restrict__ rowptr, const int *__restrict__ colind, const T *__restrict__ vals,
                      XView<T> xv, int64_t m, Epi epi) {
  spmv_csr_stream_kernel<T, LPR>(rowptr, colind, vals, xv, m, epi);
}

template <typename T, bool VF, typename BA, typename Epi>
__device__ __forceinline__ void spmv_band_stream_kernel(const BA &ba, const T *__restrict__ vals, const T *__restrict__ x,
                                                        int64_t nx, int64_t m, Epi &epi) {
  if (!epi.begin()) return;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ double red[kStreamThreads / 32];
  spmv_band_tiles<T, VF>(ba, vals, x, nx, m, epi, reinterpret_cast<BandSmem<T, VF> *>(smem_raw), epi.rev());
  epi.template end<kStreamThreads>(red);
}

template <typename T, typename Epi>
__global__ void __launch_bounds__(kStreamThreads, kStreamCtasPerSm)
    k_spmv_band_stream(BandArgs ba, const T *__restrict__ vals, const T *__restrict__ x, int64_t nx, int64_t m, Epi epi) {
  spmv_band_stream_kernel<T, false>(ba, vals, x, nx, m, epi);
}
template <typename T, typename Epi>
__global__ void __launch_bounds__(kStreamThreads, kStreamCtasPerSm)
    k_spmv_band_stream(BandArgs64 ba, const T *__restrict__ vals, const T *__restrict__ x, int64_t nx, int64_t m, Epi epi) {
  spmv_band_stream_kernel<T, false>(ba, vals, x, nx, m, epi);
}
// value-free form: every tile of the operator is uniform (BandStage, VF)
template <typename T, typename Epi>
__global__ void __launch_bounds__(kStreamThreads, kStreamCtasPerSm)
    k_spmv_band_stream_vf(BandArgs ba, const T *__restrict__ vals, const T *__restrict__ x, int64_t nx, int64_t m, Epi epi) {
  spmv_band_stream_kernel<T, true>(ba, vals, x, nx, m, epi);
}
template <typename T, typename Epi>
__global__ void __launch_bounds__(kStreamThreads, kStreamCtasPerSm)
    k_spmv_band_stream_vf(BandArgs64 ba, const T *__restrict__ vals, const T *__restrict__ x, int64_t nx, int64_t m, Epi epi) {
  spmv_band_stream_kernel<T, true>(ba, vals, x, nx, m, epi);
}

// One launch of (A x)[row] -> epi over the local rows, in the form the operator and the option "spmv_kernel" select: the
// band stream, the CSR stream, or the sub-warp form.  x is the operand of the local rows; peer_halo: the preceding halo
// exchange filled A->halo_peer instead of A->halo.  chained: programmatic dependent launch (an epilogue that allows it
// calls pdl_wait() in begin()).  Launches even when the operator has no local rows, so that a fused reduction in the
// epilogue completes.
template <typename T, typename I, typename Epi>
int launch_spmv_form(b200_ctx *ctx, const b200_csr *A, const I *rowptr, const void *x, bool peer_halo, const Epi &epi,
                     bool chained) {
  const T *vals = (const T *)A->vals;
  const int64_t m = A->m_local;
  if constexpr (is_cplx<T>::value) {
    // complex operators have neither a band description nor CSR-stream tiles (finish_operator): always the sub-warp form,
    // whatever "spmv_kernel" asks for.  vals are library-allocated (aligned); x may be a caller's view at any element offset.
    typedef typename real_of<T>::type R;
    const bool vec = ((uintptr_t)x % sizeof(T)) == 0;
    B200_TRY(with_lpr<2>(pick_lpr(A->avg_row_nnz), [&](auto lpr) -> int {
      constexpr int L = decltype(lpr)::value;
      const dim3 grid(stream_grid(ctx, m, kRowsThreads / L, 8));
      void (*k_vec)(const I *, const int *, const T *, XViewC<R, true>, int64_t, Epi) = k_spmv_rows_cplx<R, L, true, Epi>;
      void (*k_sca)(const I *, const int *, const T *, XViewC<R, false>, int64_t, Epi) = k_spmv_rows_cplx<R, L, false, Epi>;
      if (vec)
        B200_CUDA(launch_chained(chained, k_vec, grid, dim3(kRowsThreads), 0, ctx->stream, rowptr, A->colind, vals,
                                 XViewC<R, true>{(const T *)x}, m, epi));
      else
        B200_CUDA(launch_chained(chained, k_sca, grid, dim3(kRowsThreads), 0, ctx->stream, rowptr, A->colind, vals,
                                 XViewC<R, false>{(const T *)x}, m, epi));
      return B200_OK;
    }));
  } else if (use_band(ctx, A, x)) {
    // band descriptions exist on single-GPU contexts only: x is the whole operand, n_global entries (== m for the
    // square operators of the solvers)
    typedef typename std::conditional<sizeof(I) == 8, BandArgs64, BandArgs>::type BA;
    const void *tab = ctx->opt_band_values ? A->band_val : nullptr;   // null: every tile streams its vals
    const BA ba{A->band_hdr, A->band_mask, tab};
    const dim3 grid(stream_grid_size(ctx, A));
    if (tab && A->band_uniform == (m + kBandTileRows - 1) / kBandTileRows) {
      void (*k)(BA, const T *, const T *, int64_t, int64_t, Epi) = k_spmv_band_stream_vf<T, Epi>;
      const size_t smem = sizeof(BandSmem<T, true>);
      B200_SMEM_ATTR_ONCE(ctx, smem, k);
      B200_CUDA(launch_chained(chained, k, grid, dim3(kStreamThreads), smem, ctx->stream, ba, vals, (const T *)x,
                               A->n_global, m, epi));
    } else {
      void (*k)(BA, const T *, const T *, int64_t, int64_t, Epi) = k_spmv_band_stream<T, Epi>;
      const size_t smem = sizeof(BandSmem<T>);
      B200_SMEM_ATTR_ONCE(ctx, smem, k);
      B200_CUDA(launch_chained(chained, k, grid, dim3(kStreamThreads), smem, ctx->stream, ba, vals, (const T *)x,
                               A->n_global, m, epi));
    }
  } else if (use_stream(ctx, A)) {
    const XView<T> xv = make_xview<T>(A, x, peer_halo);
    const size_t smem = sizeof(StreamSmem<T, I>);
    B200_TRY(with_lpr<1>(A->stream_lpr, [&](auto lpr) -> int {
      constexpr int L = decltype(lpr)::value;
      void (*k)(const I *, const int *, const T *, XView<T>, int64_t, Epi) = k_spmv_csr_stream<T, L, Epi>;
      B200_SMEM_ATTR_ONCE(ctx, smem, k);
      B200_CUDA(launch_chained(chained, k, dim3(stream_grid_size(ctx, A)), dim3(kStreamThreads), smem, ctx->stream,
                               rowptr, A->colind, vals, xv, m, epi));
      return B200_OK;
    }));
  } else {
    const XView<T> xv = make_xview<T>(A, x, peer_halo);
    B200_TRY(with_lpr<2>(pick_lpr(A->avg_row_nnz), [&](auto lpr) -> int {
      constexpr int L = decltype(lpr)::value;
      void (*k)(const I *, const int *, const T *, XView<T>, int64_t, Epi) = k_spmv_rows<T, L, Epi>;
      B200_CUDA(launch_chained(chained, k, dim3(stream_grid(ctx, m, kRowsThreads / L, 8)), dim3(kRowsThreads), 0,
                               ctx->stream, rowptr, A->colind, vals, xv, m, epi));
      return B200_OK;
    }));
  }
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}
template <typename T, typename Epi>
int launch_spmv_fused(b200_ctx *ctx, const b200_csr *A, const void *x, bool peer_halo, const Epi &epi, bool chained) {
  return with_rowptr(A, [&](auto rowptr) { return launch_spmv_form<T>(ctx, A, rowptr, x, peer_halo, epi, chained); });
}

#endif  // __CUDACC__

}  // namespace b200
