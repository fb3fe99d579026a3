// csr.cu -- building the device operator: SparseMatrixCSC -> CSR (device transpose), CSR row slabs, the on-device
// laplace_matrix generator, halo plans and the halo exchange.
//
// Row offsets are int32, or int64 for single-GPU operators of INT32_MAX or more nonzeros (csr.cuh).  Every kernel that
// reads or writes them has an overload per width around one shared body (spmv_launch.cuh says why overloads).
#include <algorithm>
#include <cub/cub.cuh>

#include "csr.cuh"

using namespace b200;

// ------------------------------------------------------------------------------------------
// halo plan (pure host code)
// ------------------------------------------------------------------------------------------
void b200_halo_plan::rebuild_concat() {
  halo_sorted.clear();
  recv_offset.assign(world + 1, 0);
  for (int o = 0; o < world; ++o) {
    recv_offset[o] = (int64_t)halo_sorted.size();
    halo_sorted.insert(halo_sorted.end(), recv_cols[o].begin(), recv_cols[o].end());
  }
  recv_offset[world] = (int64_t)halo_sorted.size();
}

static int plan_owner(const b200_halo_plan *p, int64_t col) {
  // row_offsets ascending; owner = last r with row_offsets[r] <= col
  auto it = std::upper_bound(p->row_offsets.begin(), p->row_offsets.end(), col);
  return (int)(it - p->row_offsets.begin()) - 1;
}

static void plan_finish_scan(b200_halo_plan *p, std::vector<int64_t> &cols) {
  std::sort(cols.begin(), cols.end());
  cols.erase(std::unique(cols.begin(), cols.end()), cols.end());
  for (auto &v : p->recv_cols) v.clear();
  for (int64_t c : cols) p->recv_cols[plan_owner(p, c)].push_back(c);
  p->rebuild_concat();
}

extern "C" {

int b200_halo_plan_create(int rank, int world, const int64_t *row_offsets, b200_halo_plan **out) {
  B200_REQUIRE(out && row_offsets && world >= 1 && rank >= 0 && rank < world, "bad arguments");
  for (int r = 0; r < world; ++r)
    B200_REQUIRE(row_offsets[r] <= row_offsets[r + 1], "row_offsets must be non-decreasing");
  auto *p = new b200_halo_plan();
  p->rank = rank;
  p->world = world;
  p->row_offsets.assign(row_offsets, row_offsets + world + 1);
  p->recv_cols.resize(world);
  p->send_cols.resize(world);
  p->rebuild_concat();
  *out = p;
  return B200_OK;
}

int b200_halo_plan_scan(b200_halo_plan *p, int64_t m_local, const void *rowptr, const void *colind, int idx_bytes,
                        int base) {
  B200_REQUIRE(p && rowptr && (idx_bytes == 4 || idx_bytes == 8), "bad arguments");
  const int64_t lo = p->row_offsets[p->rank], hi = p->row_offsets[p->rank + 1];
  B200_REQUIRE(hi - lo == m_local, "m_local does not match the plan's slab");
  const int64_t n_global = p->row_offsets[p->world];
  int64_t nnz = idx_bytes == 8 ? ((const int64_t *)rowptr)[m_local] - ((const int64_t *)rowptr)[0]
                               : (int64_t)((const int32_t *)rowptr)[m_local] - ((const int32_t *)rowptr)[0];
  std::vector<int64_t> cols;
  for (int64_t k = 0; k < nnz; ++k) {
    int64_t c = (idx_bytes == 8 ? ((const int64_t *)colind)[k] : (int64_t)((const int32_t *)colind)[k]) - base;
    B200_REQUIRE(c >= 0 && c < n_global, "column index %lld out of range", (long long)c);
    if (c < lo || c >= hi) {
      // cheap de-dup of runs; full de-dup after the sort
      if (cols.empty() || cols.back() != c) cols.push_back(c);
    }
  }
  plan_finish_scan(p, cols);
  return B200_OK;
}

int b200_halo_plan_scan_laplacian(b200_halo_plan *p, int64_t N, int dims) {
  B200_REQUIRE(p && N >= 1 && dims >= 1 && dims <= 6, "bad arguments");
  int64_t n = 1, stride[8];
  for (int d = 0; d < dims; ++d) {
    stride[d] = n;
    n *= N;
  }
  B200_REQUIRE(n == p->row_offsets[p->world], "N^dims != n_global of the plan");
  const int64_t lo = p->row_offsets[p->rank], hi = p->row_offsets[p->rank + 1];
  std::vector<int64_t> cols;
  for (int d = 0; d < dims; ++d) {
    const int64_t s = stride[d];
    // rows whose -s neighbour falls below the slab: r in [lo, min(lo+s, hi)); +s above: r in [max(hi-s,lo), hi)
    for (int64_t r = lo; r < std::min(lo + s, hi); ++r)
      if ((r / s) % N > 0 && r - s < lo) cols.push_back(r - s);
    for (int64_t r = std::max(hi - s, lo); r < hi; ++r)
      if ((r / s) % N < N - 1 && r + s >= hi) cols.push_back(r + s);
  }
  plan_finish_scan(p, cols);
  return B200_OK;
}

int64_t b200_halo_plan_recv_count(const b200_halo_plan *p, int owner) {
  if (!p || owner < 0 || owner >= p->world) return -1;
  return (int64_t)p->recv_cols[owner].size();
}
int b200_halo_plan_recv_cols(const b200_halo_plan *p, int owner, int64_t *cols_out) {
  B200_REQUIRE(p && owner >= 0 && owner < p->world, "bad arguments");
  if (!p->recv_cols[owner].empty()) {
    B200_REQUIRE(cols_out, "cols_out is NULL");
    memcpy(cols_out, p->recv_cols[owner].data(), sizeof(int64_t) * p->recv_cols[owner].size());
  }
  return B200_OK;
}
int b200_halo_plan_set_send(b200_halo_plan *p, int peer, const int64_t *cols, int64_t count) {
  B200_REQUIRE(p && peer >= 0 && peer < p->world && count >= 0 && (count == 0 || cols), "bad arguments");
  const int64_t lo = p->row_offsets[p->rank], hi = p->row_offsets[p->rank + 1];
  for (int64_t i = 0; i < count; ++i)
    B200_REQUIRE(cols[i] >= lo && cols[i] < hi, "peer %d asks for row %lld that rank %d does not own", peer,
                 (long long)cols[i], p->rank);
  p->send_cols[peer].assign(cols, cols + count);
  return B200_OK;
}
int64_t b200_halo_plan_send_count(const b200_halo_plan *p, int peer) {
  if (!p || peer < 0 || peer >= p->world) return -1;
  return (int64_t)p->send_cols[peer].size();
}
int b200_halo_plan_send_range(const b200_halo_plan *p, int peer, int64_t *lo_local) {
  if (!p || peer < 0 || peer >= p->world) return -1;
  const std::vector<int64_t> &c = p->send_cols[peer];
  if (c.empty()) return 0;
  for (size_t k = 1; k < c.size(); ++k)
    if (c[k] != c[0] + (int64_t)k) return 0;
  if (lo_local) *lo_local = c[0] - p->row_offsets[p->rank];
  return 1;
}
int64_t b200_halo_plan_n_halo(const b200_halo_plan *p) { return p ? (int64_t)p->halo_sorted.size() : -1; }
int64_t b200_halo_plan_local_index(const b200_halo_plan *p, int64_t c) {
  if (!p) return -1;
  const int64_t lo = p->row_offsets[p->rank], hi = p->row_offsets[p->rank + 1];
  if (c >= lo && c < hi) return c - lo;
  auto it = std::lower_bound(p->halo_sorted.begin(), p->halo_sorted.end(), c);
  if (it == p->halo_sorted.end() || *it != c) return -1;
  return (hi - lo) + (int64_t)(it - p->halo_sorted.begin());
}
int b200_halo_plan_destroy(b200_halo_plan *p) {
  delete p;
  return B200_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------
// device kernels for construction
// ------------------------------------------------------------------------------------------
namespace {

__device__ __forceinline__ void count_one(int *c) { atomicAdd(c, 1); }
__device__ __forceinline__ void count_one(int64_t *c) { atomicAdd((unsigned long long *)c, 1ull); }

template <typename I, typename P>
__device__ __forceinline__ void count_rows(const I *__restrict__ rowval, int64_t nnz, int base, int64_t m,
                                           P *__restrict__ cnt, int *__restrict__ err) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < nnz; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = (int64_t)rowval[k] - base;
    if (r < 0 || r >= m) {
      *err = 1;
      continue;
    }
    count_one(&cnt[r]);
  }
}
template <typename I>
__global__ void k_count_rows(const I *__restrict__ rowval, int64_t nnz, int base, int64_t m, int *__restrict__ cnt,
                             int *__restrict__ err) {
  count_rows(rowval, nnz, base, m, cnt, err);
}
template <typename I>
__global__ void k_count_rows(const I *__restrict__ rowval, int64_t nnz, int base, int64_t m, int64_t *__restrict__ cnt,
                             int *__restrict__ err) {
  count_rows(rowval, nnz, base, m, cnt, err);
}

// expand colptr into a per-nonzero column id and the row key used by the stable sort
template <typename IC, typename IR>
__device__ __forceinline__ void expand_cols(const IC *__restrict__ colptr, int64_t n, int base,
                                            const IR *__restrict__ rowval, unsigned int *__restrict__ key_row,
                                            int *__restrict__ col_of) {
  // one warp per column (columns are short); lanes stride the column's entries
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t j = warp; j < n; j += nwarps) {
    const int64_t b = (int64_t)colptr[j] - base, e = (int64_t)colptr[j + 1] - base;
    for (int64_t k = b + lane; k < e; k += 32) {
      col_of[k] = (int)j;
      key_row[k] = (unsigned int)((int64_t)rowval[k] - base);
    }
  }
}
template <typename I>
__global__ void k_expand_cols(const I *__restrict__ colptr, int64_t n, int base, const I *__restrict__ rowval,
                              unsigned int *__restrict__ key_row, int *__restrict__ col_of) {
  expand_cols(colptr, n, base, rowval, key_row, col_of);
}
// the CSC of the adjoint of an operator with 8-byte row offsets: int64 colptr, int32 rowval
__global__ void k_expand_cols(const int64_t *__restrict__ colptr, int64_t n, int base, const int *__restrict__ rowval,
                              unsigned int *__restrict__ key_row, int *__restrict__ col_of) {
  expand_cols(colptr, n, base, rowval, key_row, col_of);
}

// perm: int, or int64_t when the operator has 8-byte row offsets (positions up to nnz)
template <typename T, typename TI, typename P>
__device__ __forceinline__ void gather_vals(const P *__restrict__ perm, const TI *__restrict__ nz_in, int64_t nnz,
                                            T *__restrict__ vals) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < nnz; k += (int64_t)gridDim.x * blockDim.x)
    vals[k] = (T)nz_in[perm[k]];
}
template <typename T, typename TI>
__global__ void k_gather_vals(const int *__restrict__ perm, const TI *__restrict__ nz_in, int64_t nnz,
                              T *__restrict__ vals) {
  gather_vals(perm, nz_in, nnz, vals);
}
template <typename T, typename TI>
__global__ void k_gather_vals(const int64_t *__restrict__ perm, const TI *__restrict__ nz_in, int64_t nnz,
                              T *__restrict__ vals) {
  gather_vals(perm, nz_in, nnz, vals);
}
template <typename P>
__device__ __forceinline__ void gather_int(const P *__restrict__ perm, const int *__restrict__ in, int64_t nnz,
                                           int *__restrict__ out) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < nnz; k += (int64_t)gridDim.x * blockDim.x)
    out[k] = in[perm[k]];
}
__global__ void k_gather_int(const int *__restrict__ perm, const int *__restrict__ in, int64_t nnz,
                             int *__restrict__ out) {
  gather_int(perm, in, nnz, out);
}
__global__ void k_gather_int(const int64_t *__restrict__ perm, const int *__restrict__ in, int64_t nnz,
                             int *__restrict__ out) {
  gather_int(perm, in, nnz, out);
}
__global__ void k_iota(int *p, int64_t n) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x)
    p[k] = (int)k;
}
__global__ void k_iota(int64_t *p, int64_t n) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x)
    p[k] = k;
}

// CSR slab: global column -> local extended index (binary search of the sorted halo list)
template <typename I>
__global__ void k_remap_cols(const I *__restrict__ col_in, int64_t nnz, int base, int64_t lo, int64_t hi,
                             const int64_t *__restrict__ halo_sorted, int64_t n_halo, int *__restrict__ col_out,
                             int *__restrict__ err) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < nnz; k += (int64_t)gridDim.x * blockDim.x) {
    const int64_t c = (int64_t)col_in[k] - base;
    if (c >= lo && c < hi) {
      col_out[k] = (int)(c - lo);
    } else {
      int64_t a = 0, b = n_halo;
      while (a < b) {
        const int64_t mid = (a + b) >> 1;
        if (halo_sorted[mid] < c) a = mid + 1; else b = mid;
      }
      if (a >= n_halo || halo_sorted[a] != c) {
        *err = 2;
        col_out[k] = 0;
      } else {
        col_out[k] = (int)((hi - lo) + a);
      }
    }
  }
}

template <typename I, typename P>
__device__ __forceinline__ void rowptr_convert(const I *__restrict__ in, int64_t m, P *__restrict__ out) {
  const I first = in[0];
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k <= m; k += (int64_t)gridDim.x * blockDim.x)
    out[k] = (P)(in[k] - first);
}
template <typename I>
__global__ void k_rowptr_convert(const I *__restrict__ in, int64_t m, int *__restrict__ out) {
  rowptr_convert(in, m, out);
}
template <typename I>
__global__ void k_rowptr_convert(const I *__restrict__ in, int64_t m, int64_t *__restrict__ out) {
  rowptr_convert(in, m, out);
}

template <typename T, typename TI>
__global__ void k_convert_vals(const TI *__restrict__ in, int64_t nnz, T *__restrict__ out) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < nnz; k += (int64_t)gridDim.x * blockDim.x)
    out[k] = (T)in[k];
}

// laplace_matrix(T,N,dims) on device: count pass and fill pass, one thread per local row
struct LapGeom {
  int64_t N;
  int dims;
  int64_t stride[6];
};
template <typename P>
__device__ __forceinline__ void lap_count(LapGeom g, int64_t row_begin, int64_t m, P *__restrict__ cnt) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t q = row_begin + i, rem = q;
    int c = 1;
    for (int d = 0; d < g.dims; ++d) {
      const int64_t x = rem % g.N;
      rem /= g.N;
      c += (x > 0) + (x < g.N - 1);
    }
    cnt[i] = c;
  }
}
__global__ void k_lap_count(LapGeom g, int64_t row_begin, int64_t m, int *__restrict__ cnt) {
  lap_count(g, row_begin, m, cnt);
}
__global__ void k_lap_count(LapGeom g, int64_t row_begin, int64_t m, int64_t *__restrict__ cnt) {
  lap_count(g, row_begin, m, cnt);
}
template <typename T, typename I>
__device__ __forceinline__ void lap_fill(LapGeom g, int64_t row_begin, int64_t m, const I *__restrict__ rowptr,
                                         const int64_t *__restrict__ halo_sorted, int64_t n_halo,
                                         int *__restrict__ colind, T *__restrict__ vals) {
  const int64_t lo = row_begin, hi = row_begin + m;
  auto local = [&](int64_t c) -> int {
    if (c >= lo && c < hi) return (int)(c - lo);
    int64_t a = 0, b = n_halo;
    while (a < b) {
      const int64_t mid = (a + b) >> 1;
      if (halo_sorted[mid] < c) a = mid + 1; else b = mid;
    }
    return (int)(m + a);
  };
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t q = row_begin + i;
    int64_t coord[6], rem = q;
    for (int d = 0; d < g.dims; ++d) {
      coord[d] = rem % g.N;
      rem /= g.N;
    }
    I k = rowptr[i];
    for (int d = g.dims - 1; d >= 0; --d)
      if (coord[d] > 0) {
        colind[k] = local(q - g.stride[d]);
        vals[k] = (T)-1;
        ++k;
      }
    colind[k] = (int)i;
    vals[k] = (T)(2 * g.dims);
    ++k;
    for (int d = 0; d < g.dims; ++d)
      if (coord[d] < g.N - 1) {
        colind[k] = local(q + g.stride[d]);
        vals[k] = (T)-1;
        ++k;
      }
  }
}
template <typename T>
__global__ void k_lap_fill(LapGeom g, int64_t row_begin, int64_t m, const int *__restrict__ rowptr,
                           const int64_t *__restrict__ halo_sorted, int64_t n_halo, int *__restrict__ colind,
                           T *__restrict__ vals) {
  lap_fill(g, row_begin, m, rowptr, halo_sorted, n_halo, colind, vals);
}
template <typename T>
__global__ void k_lap_fill(LapGeom g, int64_t row_begin, int64_t m, const int64_t *__restrict__ rowptr,
                           const int64_t *__restrict__ halo_sorted, int64_t n_halo, int *__restrict__ colind,
                           T *__restrict__ vals) {
  lap_fill(g, row_begin, m, rowptr, halo_sorted, n_halo, colind, vals);
}

template <typename T, typename I>
__device__ __forceinline__ void diag_rows(const I *__restrict__ rowptr, const int *__restrict__ colind,
                                          const T *__restrict__ vals, int64_t m, T *__restrict__ diag) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
    T d = (T)0;
    for (I k = rowptr[i]; k < rowptr[i + 1]; ++k)
      if (colind[k] == (int)i) d += vals[k];
    diag[i] = d;
  }
}
template <typename T>
__global__ void k_diag(const int *__restrict__ rowptr, const int *__restrict__ colind, const T *__restrict__ vals,
                       int64_t m, T *__restrict__ diag) {
  diag_rows(rowptr, colind, vals, m, diag);
}
template <typename T>
__global__ void k_diag(const int64_t *__restrict__ rowptr, const int *__restrict__ colind, const T *__restrict__ vals,
                       int64_t m, T *__restrict__ diag) {
  diag_rows(rowptr, colind, vals, m, diag);
}

// row lengths are < 2^31 (columns are int32) at either offset width
template <typename I>
__device__ __forceinline__ void row_stats(const I *__restrict__ rowptr, int64_t m, int *__restrict__ max_len) {
  int local = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x)
    local = max(local, (int)(rowptr[i + 1] - rowptr[i]));
  for (int o = 16; o > 0; o >>= 1) local = max(local, __shfl_xor_sync(0xffffffffu, local, o));
  if ((threadIdx.x & 31) == 0) atomicMax(max_len, local);
}
__global__ void k_row_stats(const int *__restrict__ rowptr, int64_t m, int *__restrict__ max_len) {
  row_stats(rowptr, m, max_len);
}
__global__ void k_row_stats(const int64_t *__restrict__ rowptr, int64_t m, int *__restrict__ max_len) {
  row_stats(rowptr, m, max_len);
}

// max over uniform tiles of R rows of the tile's nonzero count, clamped to INT_MAX (only counts <= 4096 matter)
template <typename I>
__device__ __forceinline__ void tile_max(const I *__restrict__ rowptr, int64_t m, int R, int *__restrict__ out) {
  const int64_t ntiles = (m + R - 1) / R;
  int local = 0;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < ntiles; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r0 = t * R, r1 = (r0 + R < m) ? r0 + R : m;
    const I c = rowptr[r1] - rowptr[r0];
    if constexpr (sizeof(I) == 8) local = max(local, (int)(c < INT_MAX ? c : INT_MAX));
    else local = max(local, c);
  }
  for (int o = 16; o > 0; o >>= 1) local = max(local, __shfl_xor_sync(0xffffffffu, local, o));
  if ((threadIdx.x & 31) == 0) atomicMax(out, local);
}
__global__ void k_tile_max(const int *__restrict__ rowptr, int64_t m, int R, int *__restrict__ out) {
  tile_max(rowptr, m, R, out);
}
__global__ void k_tile_max(const int64_t *__restrict__ rowptr, int64_t m, int R, int *__restrict__ out) {
  tile_max(rowptr, m, R, out);
}

// Band description (csr.cuh, spmv_stream.cuh): one block per tile of R = kBandTileRows rows, two rows per thread (r0+lt,
// r0+lt+R/2).  The tile's distinct offsets come out in ascending order from rounds of "smallest offset above the previous
// one" (a block minimum); each round also sets that offset's bit in the masks of the rows that have it.  A ninth offset,
// a row of more than 8 nonzeros or a row whose columns do not strictly ascend sets *bad: the operator keeps the CSR stream.
constexpr int kBandBuildThreads = kBandTileRows / 2;
template <typename I>
__device__ __forceinline__ void band_build(const I *__restrict__ rowptr, const int *__restrict__ colind, int64_t m,
                                           b200_band_tile *__restrict__ hdr, uint8_t *__restrict__ mask, int *bad) {
  constexpr int R = kBandTileRows, H = kBandBuildThreads;
  static_assert(2 * H == R, "two rows per thread");
  __shared__ int red[2][H / 32];
  const int lt = threadIdx.x, lane = lt & 31, wid = lt >> 5;
  const int64_t ntiles = (m + R - 1) / R;
  for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int64_t r0 = t * R;
    int d[2][8];   // the rows' offsets, INT_MAX where absent
    bool fail = false;
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int64_t r = r0 + lt + q * H;
      I b = 0, e = 0;
      if (r < m) {
        b = rowptr[r];
        e = rowptr[r + 1];
      }
      fail |= e - b > 8;
      int prev = -1;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const bool on = j < e - b;
        const int c = on ? colind[b + j] : 0;
        fail |= on && c <= prev;
        prev = c;
        d[q][j] = on ? c - (int)r : INT_MAX;
      }
    }
    // uniform exit once any block has found the operator ineligible
    if (__syncthreads_or(fail || (lt == 0 && *(volatile int *)bad))) {
      if (fail) atomicExch(bad, 1);
      return;
    }
    uint32_t mk[2] = {0u, 0u};
    int last = INT_MIN, nb = 0;
    for (int rd = 0;; ++rd) {
      int v = INT_MAX;
#pragma unroll
      for (int q = 0; q < 2; ++q)
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (d[q][j] > last && d[q][j] < v) v = d[q][j];
      v = __reduce_min_sync(0xffffffffu, v);
      if (lane == 0) red[rd & 1][wid] = v;   // double-buffered: the next round's writes cannot race this round's reads
      __syncthreads();
      int o = red[rd & 1][0];
#pragma unroll
      for (int w = 1; w < H / 32; ++w) o = min(o, red[rd & 1][w]);
      if (o == INT_MAX) break;
      if (rd == 8) {   // a ninth distinct offset
        if (lt == 0) atomicExch(bad, 1);
        return;
      }
#pragma unroll
      for (int q = 0; q < 2; ++q)
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (d[q][j] == o) mk[q] |= 1u << rd;
      if (lt == 0) hdr[t].off[rd] = o;
      last = o;
      nb = rd + 1;
    }
#pragma unroll
    for (int q = 0; q < 2; ++q) mask[r0 + lt + q * H] = (uint8_t)mk[q];   // 0 for the rows past m of the last tile
    if (lt < 8 && lt >= nb) hdr[t].off[lt] = 0;
    if (lt == 0) {
      const I k0 = rowptr[r0];
      hdr[t].nb = nb;
      hdr[t].k0 = (int)k0;
      hdr[t].k1 = (int)rowptr[r0 + R < m ? r0 + R : m];
      for (int p = 0; p < 5; ++p) hdr[t].pad[p] = 0;
      if constexpr (sizeof(I) == 8) hdr[t].pad[0] = (int)(k0 >> 32);   // the header layout (csr.cuh)
    }
  }
}
__global__ void __launch_bounds__(kBandBuildThreads)
    k_band_build(const int *__restrict__ rowptr, const int *__restrict__ colind, int64_t m,
                 b200_band_tile *__restrict__ hdr, uint8_t *__restrict__ mask, int *bad) {
  band_build(rowptr, colind, m, hdr, mask, bad);
}
__global__ void __launch_bounds__(kBandBuildThreads)
    k_band_build(const int64_t *__restrict__ rowptr, const int *__restrict__ colind, int64_t m,
                 b200_band_tile *__restrict__ hdr, uint8_t *__restrict__ mask, int *bad) {
  band_build(rowptr, colind, m, hdr, mask, bad);
}

// Value tables of an accepted band description (csr.cuh): one block per tile, the rows of band_build.  The i-th nonzero of
// a row has the i-th set bit of the row's mask, so every nonzero knows its offset slot j.  A block-wide minimum and maximum
// of the values' bit patterns per slot decide whether the tile is uniform (equal for every slot j < nb): bit patterns, not
// ==, so that -0.0 and +0.0 or two NaN payloads are never merged.  A uniform tile gets its values in val[t*8 + j] (0 for
// j >= nb) and pad[1] = 1; cnt[0] counts the uniform tiles and cnt[1] their nonzeros.
template <typename T, typename I>
__global__ void __launch_bounds__(kBandBuildThreads)
    k_band_values(const I *__restrict__ rowptr, const T *__restrict__ vals, int64_t m, const uint8_t *__restrict__ mask,
                  b200_band_tile *__restrict__ hdr, T *__restrict__ val, unsigned long long *__restrict__ cnt) {
  typedef typename std::conditional<sizeof(T) == 8, unsigned long long, unsigned int>::type U;
  constexpr int R = kBandTileRows, H = kBandBuildThreads, NB = 8;
  __shared__ U red_lo[H / 32][NB], red_hi[H / 32][NB];
  const U *__restrict__ bits = reinterpret_cast<const U *>(vals);
  const int lt = threadIdx.x, lane = lt & 31, wid = lt >> 5;
  const int64_t ntiles = (m + R - 1) / R;
  for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int64_t r0 = t * R;
    U lo[NB], hi[NB];
#pragma unroll
    for (int j = 0; j < NB; ++j) {
      lo[j] = ~(U)0;
      hi[j] = 0;
    }
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int64_t r = r0 + lt + q * H;
      if (r < m) {
        I k = rowptr[r];
        const uint32_t mk = mask[r];
#pragma unroll
        for (int j = 0; j < NB; ++j)
          if ((mk >> j) & 1u) {
            const U b = bits[k++];
            lo[j] = b < lo[j] ? b : lo[j];
            hi[j] = b > hi[j] ? b : hi[j];
          }
      }
    }
#pragma unroll
    for (int j = 0; j < NB; ++j)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const U l = __shfl_xor_sync(0xffffffffu, lo[j], o), h = __shfl_xor_sync(0xffffffffu, hi[j], o);
        lo[j] = l < lo[j] ? l : lo[j];
        hi[j] = h > hi[j] ? h : hi[j];
      }
    if (lane == 0)
#pragma unroll
      for (int j = 0; j < NB; ++j) {
        red_lo[wid][j] = lo[j];
        red_hi[wid][j] = hi[j];
      }
    __syncthreads();
    if (wid == 0) {
      const int nb = hdr[t].nb;
      U l = ~(U)0, h = 0;
      if (lane < NB)
#pragma unroll
        for (int w = 0; w < H / 32; ++w) {
          l = red_lo[w][lane] < l ? red_lo[w][lane] : l;
          h = red_hi[w][lane] > h ? red_hi[w][lane] : h;
        }
      // every offset of the header occurs in some row of the tile, so l <= h for j < nb
      const bool uniform = __all_sync(0xffffffffu, lane >= nb || l == h);
      if (uniform && lane < NB) reinterpret_cast<U *>(val)[t * NB + lane] = lane < nb ? l : (U)0;
      if (lane == 0) {
        hdr[t].pad[1] = uniform ? 1 : 0;
        if (uniform) {
          atomicAdd(cnt, 1ull);
          atomicAdd(cnt + 1, (unsigned long long)(rowptr[r0 + R < m ? r0 + R : m] - rowptr[r0]));
        }
      }
    }
    __syncthreads();   // red_lo / red_hi are rewritten for the next tile
  }
}

template <typename T>
__global__ void k_pack(const int *__restrict__ idx, const T *__restrict__ x, int64_t n, T *__restrict__ out) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x)
    out[k] = x[idx[k]];
}

int grid_for(const b200_ctx *ctx, int64_t n, int threads = 256) {
  int64_t g = (n + threads - 1) / threads;
  int64_t cap = (int64_t)ctx->sm_count * 8;
  if (g < 1) g = 1;
  return (int)(g < cap ? g : cap);
}

int finish_operator(b200_ctx *ctx, b200_csr *A, const b200_halo_plan *plan) {
  // row statistics for kernel selection
  int *d_max = (int *)ctx->d_scalars;  // reuse scratch (int view)
  B200_CUDA(cudaMemsetAsync(d_max, 0, sizeof(int), ctx->stream));
  if (A->m_local > 0) {
    with_rowptr(A, [&](auto rp) {
      k_row_stats<<<grid_for(ctx, A->m_local), 256, 0, ctx->stream>>>(rp, A->m_local, d_max);
      return 0;
    });
    B200_LAUNCH_CHECK(ctx);
  }
  B200_CUDA(cudaMemcpyAsync(ctx->h_flags, d_max, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  B200_CUDA(cudaStreamSynchronize(ctx->stream));
  A->max_row_nnz = ctx->h_flags[0];
  A->avg_row_nnz = A->m_local ? (double)A->nnz / (double)A->m_local : 0.0;
  // TMA-streamed kernel (spmv_stream.cuh): smallest lanes-per-row whose 512/LPR-row tiles hold <= 4096 nonzeros.
  // Complex operators always take the sub-warp form: a ComplexF64 stage would not fit (DESIGN.md, complex element types)
  A->stream_lpr = 0;
  if (A->m_local > 0 && !is_complex_dtype(A->dtype)) {
    for (int l = 0; l < 6; ++l) {
      B200_CUDA(cudaMemsetAsync(d_max + 1 + l, 0, sizeof(int), ctx->stream));
      with_rowptr(A, [&](auto rp) {
        k_tile_max<<<grid_for(ctx, (A->m_local + 15) / 16), 256, 0, ctx->stream>>>(rp, A->m_local, 512 >> l, d_max + 1 + l);
        return 0;
      });
      B200_LAUNCH_CHECK(ctx);
    }
    B200_CUDA(cudaMemcpyAsync(ctx->h_flags, d_max + 1, sizeof(int) * 6, cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA(cudaStreamSynchronize(ctx->stream));
    for (int l = 0; l < 6; ++l)
      if (ctx->h_flags[l] <= 4096) {
        A->stream_lpr = 1 << l;
        break;
      }
  }
  // band description (csr.cuh): single GPU, and only worth a pass when no row has more than 8 nonzeros and the CSR
  // stream runs with one lane per row
  A->band_ok = false;
  if (ctx->world == 1 && A->stream_lpr == 1 && A->max_row_nnz <= 8) {   // never for complex operators (stream_lpr == 0)
    const int64_t ntiles = (A->m_local + kBandTileRows - 1) / kBandTileRows;
    B200_CUDA(cudaMalloc(&A->band_hdr, sizeof(b200_band_tile) * ntiles));
    B200_CUDA(cudaMalloc(&A->band_mask, (size_t)kBandTileRows * ntiles));
    int *d_bad = d_max + 7;
    B200_CUDA(cudaMemsetAsync(d_bad, 0, sizeof(int), ctx->stream));
    with_rowptr(A, [&](auto rp) {
      k_band_build<<<grid_for(ctx, ntiles, 1), kBandBuildThreads, 0, ctx->stream>>>(rp, A->colind, A->m_local,
                                                                                     A->band_hdr, A->band_mask, d_bad);
      return 0;
    });
    B200_LAUNCH_CHECK(ctx);
    B200_CUDA(cudaMemcpyAsync(ctx->h_flags, d_bad, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    B200_CUDA(cudaStreamSynchronize(ctx->stream));
    A->band_ok = ctx->h_flags[0] == 0;
    if (!A->band_ok) {
      cudaFree(A->band_hdr);
      cudaFree(A->band_mask);
      A->band_hdr = nullptr;
      A->band_mask = nullptr;
    } else {
      // value tables of the uniform tiles (csr.cuh); kept only when some tile is uniform
      B200_CUDA(cudaMalloc(&A->band_val, (size_t)8 * dtype_size(A->dtype) * ntiles));
      unsigned long long *d_cnt = reinterpret_cast<unsigned long long *>(ctx->d_scalars + 4);
      B200_CUDA(cudaMemsetAsync(d_cnt, 0, 2 * sizeof(unsigned long long), ctx->stream));
      with_rowptr(A, [&](auto rp) {
        const int grid = grid_for(ctx, ntiles, 1);
        if (A->dtype == B200_F64)
          k_band_values<<<grid, kBandBuildThreads, 0, ctx->stream>>>(rp, (const double *)A->vals, A->m_local, A->band_mask,
                                                                     A->band_hdr, (double *)A->band_val, d_cnt);
        else
          k_band_values<<<grid, kBandBuildThreads, 0, ctx->stream>>>(rp, (const float *)A->vals, A->m_local, A->band_mask,
                                                                     A->band_hdr, (float *)A->band_val, d_cnt);
        return 0;
      });
      B200_LAUNCH_CHECK(ctx);
      B200_CUDA(cudaMemcpyAsync(ctx->h_scalars, d_cnt, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
      B200_CUDA(cudaStreamSynchronize(ctx->stream));
      unsigned long long h_cnt[2];
      memcpy(h_cnt, ctx->h_scalars, sizeof(h_cnt));
      A->band_uniform = (int64_t)h_cnt[0];
      A->band_uniform_nnz = (int64_t)h_cnt[1];
      if (A->band_uniform == 0) {
        cudaFree(A->band_val);
        A->band_val = nullptr;
      }
    }
  }
  B200_CUDA(cudaMemsetAsync(d_max, 0, sizeof(double) * 8, ctx->stream));
  // halo exchange lists
  const int W = ctx->world;
  A->send_count.assign(W, 0);
  A->send_offset.assign(W + 1, 0);
  A->recv_count.assign(W, 0);
  A->recv_offset.assign(W + 1, 0);
  if (plan && W > 1) {
    std::vector<int> send_idx;
    for (int p = 0; p < W; ++p) {
      A->send_offset[p] = (int64_t)send_idx.size();
      A->send_count[p] = (int64_t)plan->send_cols[p].size();
      for (int64_t c : plan->send_cols[p]) send_idx.push_back((int)(c - A->row_begin));
      A->recv_count[p] = (int64_t)plan->recv_cols[p].size();
      A->recv_offset[p] = plan->recv_offset[p];
    }
    A->send_offset[W] = (int64_t)send_idx.size();
    A->recv_offset[W] = plan->recv_offset[W];
    A->send_range_lo.assign(W, -1);
    for (int p = 0; p < W; ++p) {
      if (b200_halo_plan_send_range(plan, p, nullptr) == 1) A->send_range_lo[p] = plan->send_cols[p][0] - A->row_begin;
    }
    A->n_send = (int64_t)send_idx.size();
    const size_t vs = dtype_size(A->dtype);
    if (A->n_send) {
      B200_CUDA(cudaMalloc(&A->send_idx, sizeof(int) * A->n_send));
      B200_CUDA(cudaMemcpyAsync(A->send_idx, send_idx.data(), sizeof(int) * A->n_send, cudaMemcpyHostToDevice,
                                ctx->stream));
      B200_CUDA(cudaMalloc(&A->send_buf, vs * A->n_send));
    }
    if (A->n_halo) B200_CUDA(cudaMalloc(&A->halo, vs * A->n_halo));
    B200_CUDA(cudaStreamSynchronize(ctx->stream));
    // peer-memory path: my halo segment lives in my comm buffer; learn where my values go in each peer's segment
    A->peer_halo = false;
    A->peer_dst_offset.assign(W, 0);
    {
      std::vector<long long> mine(W + 1), all((size_t)W * (W + 1));
      for (int p = 0; p <= W; ++p) mine[p] = A->recv_offset[p];
      long long *d_all = nullptr;
      B200_CUDA(cudaMalloc(&d_all, sizeof(long long) * all.size()));
      B200_CUDA(cudaMemcpy(d_all + (size_t)ctx->rank * (W + 1), mine.data(), sizeof(long long) * (W + 1), cudaMemcpyHostToDevice));
      B200_NCCL(ncclAllGather(d_all + (size_t)ctx->rank * (W + 1), d_all, W + 1, ncclInt64, ctx->comm, ctx->stream));
      B200_CUDA(cudaStreamSynchronize(ctx->stream));
      B200_CUDA(cudaMemcpy(all.data(), d_all, sizeof(long long) * all.size(), cudaMemcpyDeviceToHost));
      cudaFree(d_all);
      bool fits = true;
      for (int p = 0; p < W; ++p) {
        A->peer_dst_offset[p] = all[(size_t)p * (W + 1) + ctx->rank];          // peer p's recv_offset[me]
        fits = fits && (size_t)all[(size_t)p * (W + 1) + W] * vs + kPeerHeaderBytes <= kPeerBufferBytes;
      }
      A->recv_mask = A->send_mask = 0;
      for (int p = 0; p < W; ++p) {
        if (A->recv_count[p]) A->recv_mask |= 1u << p;
        if (A->send_count[p]) A->send_mask |= 1u << p;
      }
      if (ctx->peer_ok && fits) {
        A->peer_halo = true;
        A->halo_peer = (char *)ctx->peer_local + kPeerHeaderBytes;
      }
    }
  }
  return B200_OK;
}

// the operator's row-offset array of width P (csr.cuh)
inline int *&rowptr_slot(b200_csr *A, int *) { return A->rowptr; }
inline int64_t *&rowptr_slot(b200_csr *A, int64_t *) { return A->rowptr64; }

// 8-byte row offsets: single-GPU operators of INT32_MAX or more nonzeros, or every single-GPU operator when the
// context's "rowptr64" is 1
bool wants_rowptr64(const b200_ctx *ctx, int64_t nnz) {
  return ctx->world == 1 && (ctx->opt_rowptr64 == 1 || nnz >= (int64_t)INT32_MAX);
}

int check_dist_args(b200_ctx *ctx, int64_t n_global, int64_t row_begin, int64_t m_local, const b200_halo_plan *plan) {
  B200_REQUIRE(ctx, "ctx is NULL");
  B200_REQUIRE(m_local >= 0 && row_begin >= 0 && row_begin + m_local <= n_global, "bad slab");
  if (ctx->world > 1) {
    B200_REQUIRE(plan, "multi-GPU context needs a halo plan");
    B200_REQUIRE(plan->world == ctx->world && plan->rank == ctx->rank, "plan/context rank mismatch");
    B200_REQUIRE(plan->row_offsets[ctx->rank] == row_begin && plan->row_offsets[ctx->rank + 1] == row_begin + m_local,
                 "slab does not match the plan");
  } else {
    B200_REQUIRE(row_begin == 0 && m_local == n_global, "single-GPU operator must own all rows");
  }
  B200_REQUIRE(m_local + (plan ? (int64_t)plan->halo_sorted.size() : 0) < (int64_t)INT32_MAX,
               "local rows + halo must fit int32");
  return B200_OK;
}

}  // namespace

// ------------------------------------------------------------------------------------------
// C ABI: operator construction
// ------------------------------------------------------------------------------------------
// P: the row offsets built (int, or int64_t: then the permutation is int64_t too and cub counts items in int64_t);
// IC, IR: the CSC's colptr and rowval (int32_t or int64_t; the adjoint of an 8-byte operator has int64 colptr and
// int32 rowval).
template <typename P, typename IC, typename IR, typename TI, typename T>
static int csr_from_csc_impl(b200_ctx *ctx, int64_t m, int64_t n, const IC *colptr, const IR *rowval, const TI *nzval,
                             int base, int64_t nnz, cudaMemcpyKind src_kind, b200_csr *A) {
  // colptr/rowval/nzval: host arrays (src_kind = cudaMemcpyHostToDevice; nnz = colptr[n] - base read by the caller)
  // or device arrays (cudaMemcpyDeviceToDevice: b200_csr_transpose feeds the CSR arrays of A as the CSC of A')
  typedef typename std::conditional<sizeof(P) == 8, int64_t, int>::type N;   // cub's num_items
  cudaStream_t st = ctx->stream;
  if (sizeof(P) == 4) B200_REQUIRE(nnz >= 0 && nnz < (int64_t)INT32_MAX, "nnz=%lld does not fit int32 CSR", (long long)nnz);
  B200_REQUIRE(nnz >= 0, "nnz=%lld", (long long)nnz);
  A->nnz = nnz;
  IC *d_colptr = nullptr;
  IR *d_rowval = nullptr;
  TI *d_nz = nullptr;
  unsigned int *key_in = nullptr, *key_out = nullptr;
  int *col_of = nullptr, *d_err = nullptr;
  P *perm_in = nullptr, *perm_out = nullptr;
  P *&rowptr = rowptr_slot(A, (P *)nullptr);
  void *d_tmp = nullptr;
  size_t tmp_bytes = 0, tmp2 = 0;
  int status = B200_OK;
  auto cleanup = [&]() {
    cudaFree(d_colptr); cudaFree(d_rowval); cudaFree(d_nz); cudaFree(key_in); cudaFree(key_out);
    cudaFree(col_of); cudaFree(perm_in); cudaFree(perm_out); cudaFree(d_err); cudaFree(d_tmp);
  };
#define CK(call)                          \
  do {                                    \
    cudaError_t _e = (call);              \
    if (_e != cudaSuccess) {              \
      set_error("%s:%d %s in `%s`", __FILE__, __LINE__, cudaGetErrorString(_e), #call); \
      cleanup();                          \
      return B200_ERR_CUDA;               \
    }                                     \
  } while (0)
  CK(cudaMalloc(&d_colptr, sizeof(IC) * (n + 1)));
  CK(cudaMalloc(&d_rowval, sizeof(IR) * (nnz ? nnz : 1)));
  CK(cudaMalloc(&d_nz, sizeof(TI) * (nnz ? nnz : 1)));
  CK(cudaMalloc(&d_err, sizeof(int)));
  CK(cudaMemsetAsync(d_err, 0, sizeof(int), st));
  CK(cudaMemcpyAsync(d_colptr, colptr, sizeof(IC) * (n + 1), src_kind, st));
  CK(cudaMemcpyAsync(d_rowval, rowval, sizeof(IR) * nnz, src_kind, st));
  CK(cudaMemcpyAsync(d_nz, nzval, sizeof(TI) * nnz, src_kind, st));
  CK(cudaMalloc(&rowptr, sizeof(P) * (m + kRowptrPad)));
  CK(cudaMalloc(&A->colind, sizeof(int) * (nnz + kNnzPad)));
  CK(cudaMalloc(&A->vals, sizeof(T) * (nnz + kNnzPad)));
  // rowptr: histogram of row ids, exclusive scan
  CK(cudaMemsetAsync(rowptr, 0, sizeof(P) * (m + kRowptrPad), st));
  if (nnz) {
    k_count_rows<IR><<<grid_for(ctx, nnz), 256, 0, st>>>(d_rowval, nnz, base, m, rowptr, d_err);
    ctx->launches++;
  }
  CK(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, rowptr, rowptr, (N)(m + 1), st));
  // stable radix sort of (row key, original position): orders by (row, column) because the CSC
  // arrays are column-major with ascending rows inside a column
  int end_bit = 1;
  while (end_bit < 32 && (1ull << end_bit) < (unsigned long long)(m > 1 ? m : 2)) ++end_bit;
  CK(cudaMalloc(&key_in, sizeof(unsigned int) * (nnz ? nnz : 1)));
  CK(cudaMalloc(&key_out, sizeof(unsigned int) * (nnz ? nnz : 1)));
  CK(cudaMalloc(&col_of, sizeof(int) * (nnz + kNnzPad)));
  CK(cudaMalloc(&perm_in, sizeof(P) * (nnz + kNnzPad)));
  CK(cudaMalloc(&perm_out, sizeof(P) * (nnz + kNnzPad)));
  CK(cub::DeviceRadixSort::SortPairs(nullptr, tmp2, key_in, key_out, perm_in, perm_out, (N)nnz, 0, end_bit, st));
  tmp_bytes = std::max(tmp_bytes, tmp2);
  CK(cudaMalloc(&d_tmp, tmp_bytes ? tmp_bytes : 16));
  CK(cub::DeviceScan::ExclusiveSum(d_tmp, tmp_bytes, rowptr, rowptr, (N)(m + 1), st));
  ctx->launches++;
  if (nnz) {
    k_expand_cols<<<grid_for(ctx, n * 32), 256, 0, st>>>(d_colptr, n, base, d_rowval, key_in, col_of);
    k_iota<<<grid_for(ctx, nnz), 256, 0, st>>>(perm_in, nnz);
    CK(cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, key_in, key_out, perm_in, perm_out, (N)nnz, 0, end_bit, st));
    k_gather_int<<<grid_for(ctx, nnz), 256, 0, st>>>(perm_out, col_of, nnz, A->colind);
    k_gather_vals<T, TI><<<grid_for(ctx, nnz), 256, 0, st>>>(perm_out, d_nz, nnz, (T *)A->vals);
    ctx->launches += 5;
  }
  CK(cudaMemcpyAsync(ctx->h_flags, d_err, sizeof(int), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  CK(cudaGetLastError());
  if (ctx->h_flags[0]) {
    set_error("row index out of range in SparseMatrixCSC arrays");
    status = B200_ERR_INVALID;
  }
#undef CK
  cleanup();
  return status;
}

// the levels of the device AMG setup (amg_setup.cu): copies of device CSR arrays with fp64 values rounded to dtype
int b200::csr_from_device_f64(b200_ctx *ctx, int64_t m, int64_t n, int64_t nnz, const int *rowptr, const int *colind,
                              const double *vals, int dtype, b200_csr **out) {
  B200_REQUIRE(dtype == B200_F64 || dtype == B200_F32, "bad dtype");
  B200_REQUIRE(nnz >= 0 && nnz < (int64_t)INT32_MAX, "nnz=%lld does not fit int32 CSR", (long long)nnz);
  cudaStream_t st = ctx->stream;
  auto *A = new b200_csr();
  A->ctx = ctx;
  A->dtype = dtype;
  A->m_local = A->m_global = m;
  A->n_global = n;
  A->nnz = nnz;
  auto fail = [&](int s) {
    b200_csr_destroy(A);
    return s;
  };
#define CK(call)                                                                        \
  do {                                                                                  \
    cudaError_t _e = (call);                                                            \
    if (_e != cudaSuccess) {                                                            \
      set_error("%s:%d %s in `%s`", __FILE__, __LINE__, cudaGetErrorString(_e), #call); \
      return fail(B200_ERR_CUDA);                                                       \
    }                                                                                   \
  } while (0)
  CK(cudaMalloc(&A->rowptr, sizeof(int) * (m + kRowptrPad)));
  CK(cudaMalloc(&A->colind, sizeof(int) * (nnz + kNnzPad)));
  CK(cudaMalloc(&A->vals, dtype_size(dtype) * (nnz + kNnzPad)));
  CK(cudaMemsetAsync(A->rowptr, 0, sizeof(int) * (m + kRowptrPad), st));
  CK(cudaMemcpyAsync(A->rowptr, rowptr, sizeof(int) * (m + 1), cudaMemcpyDeviceToDevice, st));
  if (nnz) {
    CK(cudaMemcpyAsync(A->colind, colind, sizeof(int) * nnz, cudaMemcpyDeviceToDevice, st));
    if (dtype == B200_F64) CK(cudaMemcpyAsync(A->vals, vals, sizeof(double) * nnz, cudaMemcpyDeviceToDevice, st));
    else k_convert_vals<float, double><<<grid_for(ctx, nnz), 256, 0, st>>>(vals, nnz, (float *)A->vals);
    ctx->launches++;
  }
  CK(cudaGetLastError());
#undef CK
  const int s = finish_operator(ctx, A, nullptr);
  if (s != B200_OK) return fail(s);
  *out = A;
  return B200_OK;
}

extern "C" {

int b200_csr_from_csc(b200_ctx *ctx, int64_t m, int64_t n, const void *colptr, const void *rowval, const void *nzval,
                      int idx_bytes, int dtype, int base, b200_csr **out) {
  B200_REQUIRE(ctx && out && colptr && (idx_bytes == 4 || idx_bytes == 8), "bad arguments");
  B200_REQUIRE(dtype == B200_F64 || dtype == B200_F32 || dtype == B200_CF64 || dtype == B200_CF32, "bad dtype");
  B200_REQUIRE(ctx->world == 1, "b200_csr_from_csc is single-GPU; use b200_csr_from_csr_slab on multi-GPU contexts");
  B200_REQUIRE(m >= 0 && n >= 0 && m < INT32_MAX && n < INT32_MAX, "dimensions must fit int32");
  // rectangular operators are accepted (lsqr!/lsmr!); the square-system solvers check is_square(A) themselves
  B200_CUDA(cudaSetDevice(ctx->device));
  auto *A = new b200_csr();
  A->ctx = ctx;
  A->dtype = dtype;
  A->m_local = m;
  A->m_global = m;
  A->n_global = n;
  const int64_t nnz = (idx_bytes == 8 ? (int64_t)((const int64_t *)colptr)[n] : (int64_t)((const int32_t *)colptr)[n]) - base;
  // the upload / sort / gather pipeline at the index width of the arrays, the element type and the row-offset width
  auto conv = [&](auto idx, auto elt) -> int {
    typedef decltype(idx) I;
    typedef decltype(elt) T;
    const I *cp = (const I *)colptr, *rv = (const I *)rowval;
    if (wants_rowptr64(ctx, nnz))
      return csr_from_csc_impl<int64_t, I, I, T, T>(ctx, m, n, cp, rv, (const T *)nzval, base, nnz, cudaMemcpyHostToDevice, A);
    return csr_from_csc_impl<int, I, I, T, T>(ctx, m, n, cp, rv, (const T *)nzval, base, nnz, cudaMemcpyHostToDevice, A);
  };
  auto by_dtype = [&](auto idx) -> int {
    switch (dtype) {
      case B200_F64: return conv(idx, double());
      case B200_F32: return conv(idx, float());
      case B200_CF64: return conv(idx, cplx<double>());
      default: return conv(idx, cplx<float>());
    }
  };
  int s = idx_bytes == 8 ? by_dtype(int64_t()) : by_dtype(int32_t());
  if (s == B200_OK) s = finish_operator(ctx, A, nullptr);
  if (s != B200_OK) {
    b200_csr_destroy(A);
    return s;
  }
  *out = A;
  return B200_OK;
}

/* adjoint(A) as an operator of its own (reference: LanczosDecomp stores `adjoint(A)`, src/qmr.jl:54; lsqr src/lsqr.jl:128,
 * lsmr src/lsmr.jl:117): the device CSR arrays of A are the CSC arrays of A', so the CSC->CSR conversion above builds
 * the CSR of A' without leaving the GPU.  Real element types: adjoint == transpose. */
int b200_csr_transpose(b200_ctx *ctx, const b200_csr *A, b200_csr **out) {
  B200_TRY(real_only(A, "b200_csr_transpose"));
  B200_REQUIRE(ctx && A && out, "NULL argument");
  B200_REQUIRE(A->ctx == ctx, "operator belongs to another context");
  B200_REQUIRE(ctx->world == 1, "b200_csr_transpose is single-GPU; on multi-GPU contexts build the adjoint from its own "
                                "row slabs with b200_csr_from_csr_slab");
  B200_CUDA(cudaSetDevice(ctx->device));
  auto *At = new b200_csr();
  At->ctx = ctx;
  At->dtype = A->dtype;
  At->m_local = A->n_global;
  At->m_global = A->n_global;
  At->n_global = A->m_local;
  const cudaMemcpyKind d2d = cudaMemcpyDeviceToDevice;
  // the adjoint keeps A's row-offset width (A's offsets are the colptr of the CSC of A')
  int s = with_rowptr(A, [&](auto rp) -> int {
    typedef typename std::remove_const<typename std::remove_pointer<decltype(rp)>::type>::type P;
    return A->dtype == B200_F64
               ? csr_from_csc_impl<P, P, int, double, double>(ctx, At->m_local, At->n_global, rp, A->colind,
                                                              (const double *)A->vals, 0, A->nnz, d2d, At)
               : csr_from_csc_impl<P, P, int, float, float>(ctx, At->m_local, At->n_global, rp, A->colind,
                                                            (const float *)A->vals, 0, A->nnz, d2d, At);
  });
  if (s == B200_OK) s = finish_operator(ctx, At, nullptr);
  if (s != B200_OK) {
    b200_csr_destroy(At);
    return s;
  }
  *out = At;
  return B200_OK;
}

int b200_csr_from_csr_slab(b200_ctx *ctx, int64_t n_global, int64_t row_begin, int64_t m_local, const void *rowptr,
                           const void *colind, const void *vals, int idx_bytes, int dtype, int base,
                           const b200_halo_plan *plan, b200_csr **out) {
  B200_TRY(real_only(dtype, "b200_csr_from_csr_slab"));
  B200_REQUIRE(out && rowptr && (idx_bytes == 4 || idx_bytes == 8), "bad arguments");
  B200_REQUIRE(dtype == B200_F64 || dtype == B200_F32, "bad dtype");
  B200_TRY(check_dist_args(ctx, n_global, row_begin, m_local, plan));
  B200_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const int64_t nnz = idx_bytes == 8 ? ((const int64_t *)rowptr)[m_local] - ((const int64_t *)rowptr)[0]
                                     : (int64_t)((const int32_t *)rowptr)[m_local] - ((const int32_t *)rowptr)[0];
  const bool wide = wants_rowptr64(ctx, nnz);   // multi-GPU slabs keep int32 row offsets
  B200_REQUIRE(nnz >= 0 && (wide || nnz < (int64_t)INT32_MAX), "local nnz must fit int32");
  auto *A = new b200_csr();
  A->ctx = ctx;
  A->dtype = dtype;
  A->m_local = m_local;
  A->m_global = n_global;   // row-partitioned operators are square
  A->n_global = n_global;
  A->row_begin = row_begin;
  A->nnz = nnz;
  A->n_halo = plan ? (int64_t)plan->halo_sorted.size() : 0;
  const size_t vs = dtype_size(dtype);
  void *d_rp = nullptr, *d_ci = nullptr;
  int64_t *d_halo = nullptr;
  int *d_err = nullptr;
  int status = B200_OK;
  auto fail = [&](int s) {
    cudaFree(d_rp); cudaFree(d_ci); cudaFree(d_halo); cudaFree(d_err);
    b200_csr_destroy(A);
    return s;
  };
#define CK(call)                                                                        \
  do {                                                                                  \
    cudaError_t _e = (call);                                                            \
    if (_e != cudaSuccess) {                                                            \
      set_error("%s:%d %s in `%s`", __FILE__, __LINE__, cudaGetErrorString(_e), #call); \
      return fail(B200_ERR_CUDA);                                                       \
    }                                                                                   \
  } while (0)
  if (wide) {
    CK(cudaMalloc(&A->rowptr64, sizeof(int64_t) * (m_local + kRowptrPad)));
    CK(cudaMemsetAsync(A->rowptr64, 0, sizeof(int64_t) * (m_local + kRowptrPad), st));
  } else {
    CK(cudaMalloc(&A->rowptr, sizeof(int) * (m_local + kRowptrPad)));
    CK(cudaMemsetAsync(A->rowptr, 0, sizeof(int) * (m_local + kRowptrPad), st));
  }
  CK(cudaMalloc(&A->colind, sizeof(int) * (nnz + kNnzPad)));
  CK(cudaMalloc(&A->vals, vs * (nnz + kNnzPad)));
  CK(cudaMalloc(&d_rp, (size_t)idx_bytes * (m_local + 1)));
  CK(cudaMalloc(&d_ci, (size_t)idx_bytes * (nnz ? nnz : 1)));
  CK(cudaMalloc(&d_halo, sizeof(int64_t) * (A->n_halo ? A->n_halo : 1)));
  CK(cudaMalloc(&d_err, sizeof(int)));
  CK(cudaMemsetAsync(d_err, 0, sizeof(int), st));
  CK(cudaMemcpyAsync(d_rp, rowptr, (size_t)idx_bytes * (m_local + 1), cudaMemcpyHostToDevice, st));
  if (nnz) {
    CK(cudaMemcpyAsync(d_ci, colind, (size_t)idx_bytes * nnz, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(A->vals, vals, vs * nnz, cudaMemcpyHostToDevice, st));
  }
  if (A->n_halo)
    CK(cudaMemcpyAsync(d_halo, plan->halo_sorted.data(), sizeof(int64_t) * A->n_halo, cudaMemcpyHostToDevice, st));
  const int64_t lo = row_begin, hi = row_begin + m_local;
  if (idx_bytes == 8) {
    if (wide) k_rowptr_convert<int64_t><<<grid_for(ctx, m_local + 1), 256, 0, st>>>((const int64_t *)d_rp, m_local, A->rowptr64);
    else k_rowptr_convert<int64_t><<<grid_for(ctx, m_local + 1), 256, 0, st>>>((const int64_t *)d_rp, m_local, A->rowptr);
    if (nnz) k_remap_cols<int64_t><<<grid_for(ctx, nnz), 256, 0, st>>>((const int64_t *)d_ci, nnz, base, lo, hi, d_halo, A->n_halo, A->colind, d_err);
  } else {
    if (wide) k_rowptr_convert<int32_t><<<grid_for(ctx, m_local + 1), 256, 0, st>>>((const int32_t *)d_rp, m_local, A->rowptr64);
    else k_rowptr_convert<int32_t><<<grid_for(ctx, m_local + 1), 256, 0, st>>>((const int32_t *)d_rp, m_local, A->rowptr);
    if (nnz) k_remap_cols<int32_t><<<grid_for(ctx, nnz), 256, 0, st>>>((const int32_t *)d_ci, nnz, base, lo, hi, d_halo, A->n_halo, A->colind, d_err);
  }
  ctx->launches += 2;
  CK(cudaMemcpyAsync(ctx->h_flags, d_err, sizeof(int), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  CK(cudaGetLastError());
#undef CK
  if (ctx->h_flags[0]) {
    set_error("column index not owned and not in the halo plan");
    return fail(B200_ERR_INVALID);
  }
  cudaFree(d_rp); cudaFree(d_ci); cudaFree(d_halo); cudaFree(d_err);
  status = finish_operator(ctx, A, plan);
  if (status != B200_OK) {
    b200_csr_destroy(A);
    return status;
  }
  *out = A;
  return B200_OK;
}

int b200_csr_laplacian(b200_ctx *ctx, int64_t N, int dims, int dtype, int64_t row_begin, int64_t m_local,
                       const b200_halo_plan *plan, b200_csr **out) {
  B200_TRY(real_only(dtype, "b200_csr_laplacian"));
  B200_REQUIRE(out && N >= 1 && dims >= 1 && dims <= 6, "bad arguments");
  B200_REQUIRE(dtype == B200_F64 || dtype == B200_F32, "bad dtype");
  LapGeom g;
  g.N = N;
  g.dims = dims;
  int64_t n = 1;
  for (int d = 0; d < dims; ++d) {
    g.stride[d] = n;
    n *= N;
  }
  B200_TRY(check_dist_args(ctx, n, row_begin, m_local, plan));
  B200_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  auto *A = new b200_csr();
  A->ctx = ctx;
  A->dtype = dtype;
  A->m_local = m_local;
  A->m_global = n;
  A->n_global = n;
  A->row_begin = row_begin;
  A->n_halo = plan ? (int64_t)plan->halo_sorted.size() : 0;
  // nnz of the whole operator: n diagonal entries and 2 (N-1) N^(dims-1) off-diagonal ones per dimension; only a
  // single-GPU operator (all rows) can take 8-byte row offsets
  int64_t nnz_all = n;
  for (int d = 0; d < dims; ++d) nnz_all += 2 * (N - 1) * (n / N);
  const bool wide = wants_rowptr64(ctx, nnz_all);
  int64_t *d_halo = nullptr;
  void *d_tmp = nullptr;
  size_t tmp_bytes = 0;
  auto fail = [&](int s) {
    cudaFree(d_halo); cudaFree(d_tmp);
    b200_csr_destroy(A);
    return s;
  };
#define CK(call)                                                                        \
  do {                                                                                  \
    cudaError_t _e = (call);                                                            \
    if (_e != cudaSuccess) {                                                            \
      set_error("%s:%d %s in `%s`", __FILE__, __LINE__, cudaGetErrorString(_e), #call); \
      return fail(B200_ERR_CUDA);                                                       \
    }                                                                                   \
  } while (0)
  CK(cudaMalloc(&d_halo, sizeof(int64_t) * (A->n_halo ? A->n_halo : 1)));
  if (A->n_halo)
    CK(cudaMemcpyAsync(d_halo, plan->halo_sorted.data(), sizeof(int64_t) * A->n_halo, cudaMemcpyHostToDevice, st));
  // counts, exclusive scan, fill through the offsets, at the operator's row-offset width P
  auto build = [&](auto *rp) -> int {
    typedef typename std::remove_pointer<decltype(rp)>::type P;
    typedef typename std::conditional<sizeof(P) == 8, int64_t, int>::type NI;   // cub's num_items
    P *&rowptr = rowptr_slot(A, rp);
    CK(cudaMalloc(&rowptr, sizeof(P) * (m_local + kRowptrPad)));
    CK(cudaMemsetAsync(rowptr, 0, sizeof(P) * (m_local + kRowptrPad), st));
    if (m_local) k_lap_count<<<grid_for(ctx, m_local), 256, 0, st>>>(g, row_begin, m_local, rowptr);
    CK(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, rowptr, rowptr, (NI)(m_local + 1), st));
    CK(cudaMalloc(&d_tmp, tmp_bytes ? tmp_bytes : 16));
    CK(cub::DeviceScan::ExclusiveSum(d_tmp, tmp_bytes, rowptr, rowptr, (NI)(m_local + 1), st));
    P nnz_local = 0;
    CK(cudaMemcpyAsync(&nnz_local, rowptr + m_local, sizeof(P), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    A->nnz = nnz_local;
    const size_t vs = dtype_size(dtype);
    CK(cudaMalloc(&A->colind, sizeof(int) * (A->nnz + kNnzPad)));
    CK(cudaMalloc(&A->vals, vs * (A->nnz + kNnzPad)));
    if (m_local) {
      if (dtype == B200_F64)
        k_lap_fill<double><<<grid_for(ctx, m_local), 256, 0, st>>>(g, row_begin, m_local, rowptr, d_halo, A->n_halo, A->colind, (double *)A->vals);
      else
        k_lap_fill<float><<<grid_for(ctx, m_local), 256, 0, st>>>(g, row_begin, m_local, rowptr, d_halo, A->n_halo, A->colind, (float *)A->vals);
    }
    return B200_OK;
  };
  if (wide) B200_TRY(build((int64_t *)nullptr));
  else B200_TRY(build((int *)nullptr));
  ctx->launches += 3;
  CK(cudaStreamSynchronize(st));
  CK(cudaGetLastError());
#undef CK
  cudaFree(d_halo); cudaFree(d_tmp);
  int status = finish_operator(ctx, A, plan);
  if (status != B200_OK) {
    b200_csr_destroy(A);
    return status;
  }
  *out = A;
  return B200_OK;
}

int b200_csr_destroy(b200_csr *A) {
  if (!A) return B200_OK;
  if (A->ctx) {
    cudaSetDevice(A->ctx->device);
    cudaStreamSynchronize(A->ctx->stream);
  }
  cudaFree(A->rowptr);
  cudaFree(A->rowptr64);
  cudaFree(A->colind);
  cudaFree(A->vals);
  cudaFree(A->send_idx);
  cudaFree(A->send_buf);
  cudaFree(A->halo);
  cudaFree(A->band_hdr);
  cudaFree(A->band_mask);
  cudaFree(A->band_val);
  if (A->st_plan && A->st_plan_free) A->st_plan_free(A->st_plan);
  delete A;
  return B200_OK;
}

int b200_csr_info(const b200_csr *A, int64_t *m_local, int64_t *n_global, int64_t *nnz_local, int *dtype,
                  int64_t *row_begin, int64_t *n_halo) {
  B200_REQUIRE(A, "A is NULL");
  if (m_local) *m_local = A->m_local;
  if (n_global) *n_global = A->n_global;
  if (nnz_local) *nnz_local = A->nnz;
  if (dtype) *dtype = A->dtype;
  if (row_begin) *row_begin = A->row_begin;
  if (n_halo) *n_halo = A->n_halo;
  return B200_OK;
}

int b200_csr_stream_kind(const b200_csr *A, int *kind, int64_t *structure_bytes) {
  B200_REQUIRE(A, "A is NULL");
  const int64_t ntiles = (A->m_local + kBandTileRows - 1) / kBandTileRows;
  int k;
  int64_t bytes;
  if (A->band_ok) {
    k = 3;
    bytes = ntiles * (int64_t)(sizeof(b200_band_tile) + kBandTileRows);
  } else {
    k = A->stream_lpr > 0 ? 2 : 1;
    bytes = 4 * A->nnz + (A->rowptr64 ? 8 : 4) * (A->m_local + 1);
  }
  if (kind) *kind = k;
  if (structure_bytes) *structure_bytes = bytes;
  return B200_OK;
}

int b200_csr_band_values(const b200_csr *A, int64_t *uniform_tiles, int64_t *value_bytes) {
  B200_REQUIRE(A, "A is NULL");
  const int64_t V = (int64_t)dtype_size(A->dtype);
  if (uniform_tiles) *uniform_tiles = A->band_uniform;
  if (value_bytes) *value_bytes = V * (A->nnz - A->band_uniform_nnz + 8 * A->band_uniform);
  return B200_OK;
}

int b200_csr_diag(b200_ctx *ctx, const b200_csr *A, void *diag_dev) {
  B200_REQUIRE(ctx && A && diag_dev, "NULL argument");
  if (A->m_local == 0) return B200_OK;
  const int grid = grid_for(ctx, A->m_local);
  with_rowptr(A, [&](auto rp) {
    if (A->dtype == B200_CF64)
      k_diag<cplx<double>><<<grid, 256, 0, ctx->stream>>>(rp, A->colind, (const cplx<double> *)A->vals, A->m_local, (cplx<double> *)diag_dev);
    else if (A->dtype == B200_CF32)
      k_diag<cplx<float>><<<grid, 256, 0, ctx->stream>>>(rp, A->colind, (const cplx<float> *)A->vals, A->m_local, (cplx<float> *)diag_dev);
    else if (A->dtype == B200_F64)
      k_diag<double><<<grid, 256, 0, ctx->stream>>>(rp, A->colind, (const double *)A->vals, A->m_local, (double *)diag_dev);
    else
      k_diag<float><<<grid, 256, 0, ctx->stream>>>(rp, A->colind, (const float *)A->vals, A->m_local, (float *)diag_dev);
    return 0;
  });
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

int b200_csr_download(b200_ctx *ctx, const b200_csr *A, int32_t *rowptr, int32_t *colind, void *vals) {
  B200_REQUIRE(ctx && A, "NULL argument");
  if (A->rowptr64) {
    set_error("b200_csr_download: the operator has 8-byte row offsets (nnz >= 2^31, or built with \"rowptr64\" = 1); "
              "use b200_csr_download64");
    return B200_ERR_UNSUPPORTED;
  }
  if (rowptr) B200_CUDA(cudaMemcpyAsync(rowptr, A->rowptr, sizeof(int) * (A->m_local + 1), cudaMemcpyDeviceToHost, ctx->stream));
  if (colind && A->nnz) B200_CUDA(cudaMemcpyAsync(colind, A->colind, sizeof(int) * A->nnz, cudaMemcpyDeviceToHost, ctx->stream));
  if (vals && A->nnz) B200_CUDA(cudaMemcpyAsync(vals, A->vals, dtype_size(A->dtype) * A->nnz, cudaMemcpyDeviceToHost, ctx->stream));
  B200_CUDA(cudaStreamSynchronize(ctx->stream));
  return B200_OK;
}

int b200_csr_download64(b200_ctx *ctx, const b200_csr *A, int64_t *rowptr, int32_t *colind, void *vals) {
  B200_REQUIRE(ctx && A, "NULL argument");
  std::vector<int> narrow;
  if (rowptr && A->rowptr64) {
    B200_CUDA(cudaMemcpyAsync(rowptr, A->rowptr64, sizeof(int64_t) * (A->m_local + 1), cudaMemcpyDeviceToHost, ctx->stream));
  } else if (rowptr) {
    narrow.resize((size_t)A->m_local + 1);
    B200_CUDA(cudaMemcpyAsync(narrow.data(), A->rowptr, sizeof(int) * (A->m_local + 1), cudaMemcpyDeviceToHost, ctx->stream));
  }
  if (colind && A->nnz) B200_CUDA(cudaMemcpyAsync(colind, A->colind, sizeof(int) * A->nnz, cudaMemcpyDeviceToHost, ctx->stream));
  if (vals && A->nnz) B200_CUDA(cudaMemcpyAsync(vals, A->vals, dtype_size(A->dtype) * A->nnz, cudaMemcpyDeviceToHost, ctx->stream));
  B200_CUDA(cudaStreamSynchronize(ctx->stream));
  for (size_t i = 0; i < narrow.size(); ++i) rowptr[i] = narrow[i];
  return B200_OK;
}

int b200_csr_index_bytes(const b200_csr *A, int *bytes) {
  B200_REQUIRE(A && bytes, "NULL argument");
  *bytes = A->rowptr64 ? 8 : 4;
  return B200_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------
// halo push over NVLink peer memory (peer.cuh): x[send_idx[k]] -> the peer's halo segment, then flags
// ------------------------------------------------------------------------------------------
namespace {
struct PushArgs {
  int world, rank;
  long long start[kPeerMaxWorld + 1];   // send_offset per peer
  void *dst[kPeerMaxWorld];             // peer halo segment + my offset inside it
  unsigned int send_mask;
};
template <typename T>
__global__ void __launch_bounds__(256) k_halo_push(PushArgs a, const int *__restrict__ idx, const T *__restrict__ x,
                                                   PeerView pv, unsigned long long seq, unsigned int *ticket,
                                                   const int *__restrict__ done_flag) {
  pdl_wait();
  if (done_flag && *done_flag) return;
  const long long n = a.start[a.world];
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < n; k += (long long)gridDim.x * blockDim.x) {
    int p = 0;
    while (k >= a.start[p + 1]) ++p;
    ((T *)a.dst[p])[k - a.start[p]] = x[idx[k]];      // store to mapped peer memory (NVLink)
  }
  pdl_launch_dependents();
  __threadfence_system();
  __shared__ bool is_last;
  __syncthreads();
  if (threadIdx.x == 0) is_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!is_last) return;
  if (threadIdx.x == 0) {
    __threadfence_system();
    for (int p = 0; p < a.world; ++p)
      if ((a.send_mask >> p) & 1u) st_release_sys(&pv.hdr[p]->halo_flag[a.rank], seq);
    *ticket = 0u;
  }
}
}  // namespace

int b200::halo_push(b200_ctx *ctx, const b200_csr *A, const void *x_dev, unsigned long long seq,
                    const int *done_flag) {
  if (A->send_mask == 0) return B200_OK;
  PushArgs a;
  a.world = ctx->world;
  a.rank = ctx->rank;
  a.send_mask = A->send_mask;
  const size_t vs = dtype_size(A->dtype);
  for (int p = 0; p <= ctx->world; ++p) a.start[p] = A->send_offset[p];
  for (int p = 0; p < ctx->world; ++p)
    a.dst[p] = (char *)ctx->peer_ptr[p] + kPeerHeaderBytes + vs * (size_t)A->peer_dst_offset[p];
  const int grid = std::max(1, std::min(ctx->sm_count, (int)((A->n_send + 1023) / 1024)));
  unsigned int *ticket = ctx->red.ticket + 1;   // own counter: must not interfere with a reduction in flight
  if (A->dtype == B200_F64)
    B200_CUDA(launch_chained(ctx->opt_pdl != 0, k_halo_push<double>, dim3(grid), dim3(256), 0, ctx->stream, a,
                             (const int *)A->send_idx, (const double *)x_dev, ctx->peer_view, seq, ticket, done_flag));
  else
    B200_CUDA(launch_chained(ctx->opt_pdl != 0, k_halo_push<float>, dim3(grid), dim3(256), 0, ctx->stream, a,
                             (const int *)A->send_idx, (const float *)x_dev, ctx->peer_view, seq, ticket, done_flag));
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

// ------------------------------------------------------------------------------------------
// halo exchange: pack boundary values, grouped ncclSend/ncclRecv with every peer that shares rows
// ------------------------------------------------------------------------------------------
int b200::halo_exchange(b200_ctx *ctx, const b200_csr *A, const void *x_dev) {
  if (ctx->world == 1 || (A->n_send == 0 && A->n_halo == 0)) return B200_OK;
  cudaStream_t st = ctx->stream;
  const size_t vs = dtype_size(A->dtype);
  if (A->n_send) {
    if (A->dtype == B200_F64)
      k_pack<double><<<grid_for(ctx, A->n_send), 256, 0, st>>>(A->send_idx, (const double *)x_dev, A->n_send, (double *)A->send_buf);
    else
      k_pack<float><<<grid_for(ctx, A->n_send), 256, 0, st>>>(A->send_idx, (const float *)x_dev, A->n_send, (float *)A->send_buf);
    B200_LAUNCH_CHECK(ctx);
  }
  const ncclDataType_t nt = A->dtype == B200_F64 ? ncclDouble : ncclFloat;
  B200_NCCL(ncclGroupStart());
  for (int p = 0; p < ctx->world; ++p) {
    if (p == ctx->rank) continue;
    if (A->send_count[p])
      B200_NCCL(ncclSend((const char *)A->send_buf + vs * A->send_offset[p], (size_t)A->send_count[p], nt, p, ctx->comm, st));
    if (A->recv_count[p])
      B200_NCCL(ncclRecv((char *)A->halo + vs * A->recv_offset[p], (size_t)A->recv_count[p], nt, p, ctx->comm, st));
  }
  B200_NCCL(ncclGroupEnd());
  return B200_OK;
}
