// csr.cuh -- the device operator (CSR with int32 column indices and int32 or int64 row offsets, row slab) and the
// host halo plan.
#pragma once
#include "common.cuh"

struct b200_halo_plan {
  int rank = 0, world = 1;
  std::vector<int64_t> row_offsets;                // world+1
  std::vector<std::vector<int64_t>> recv_cols;     // [owner] -> sorted global columns needed from owner
  std::vector<std::vector<int64_t>> send_cols;     // [peer]  -> my global rows the peer needs
  std::vector<int64_t> halo_sorted;                // concatenation of recv_cols (globally ascending)
  std::vector<int64_t> recv_offset;                // world+1 prefix over owners into halo_sorted
  void rebuild_concat();
};

namespace b200 {
// slack behind the CSR arrays so that the 16-byte-granular TMA bulk copies of the last tile stay
// inside the allocations (spmv_stream.cuh)
constexpr int64_t kRowptrPad = 520;
constexpr int64_t kNnzPad = 16;
constexpr int kBandTileRows = 512;   // rows per tile of the band description (spmv_stream.cuh)
}  // namespace b200
using b200::kNnzPad;
using b200::kRowptrPad;

// Per-tile header of the band description.  Tile t covers rows [t*R, min(t*R+R, m)), R = kBandTileRows; its nonzeros are
// vals[k0, k1) (= rowptr[r0], rowptr[r1]) in row order, and within a row in ascending offset order.  Operators with
// 8-byte row offsets store the low 32 bits of both bounds in k0, k1 and the high 32 bits of the first in pad[0]: a tile
// holds fewer than 2^32 nonzeros, so k1 = k0 + (uint32_t)(k1_lo - k0_lo).  pad[0] is 0 for 4-byte operators.
// pad[1] is 1 when the tile is uniform: for every offset j < nb, all of the tile's nonzeros with offset j have the same bit
// pattern, stored as band_val[t * 8 + j] (b200_csr); the band stream then reads those 8 values instead of vals[k0, k1).
// pad[2..4] are 0.  As int4s: {off[0..3]}, {off[4..7]}, {nb, k0, k1, pad[0]}, {pad[1], pad[2], pad[3], pad[4]}.
struct alignas(16) b200_band_tile {
  int off[8];   // the tile's distinct offsets col - row, ascending; entries >= nb are 0
  int nb;       // number of offsets
  int k0, k1;
  int pad[5];
};
static_assert(sizeof(b200_band_tile) == 64, "band tile header is 64 bytes");

struct b200_csr {
  b200_ctx *ctx = nullptr;
  int stream_lpr = 0;      // lanes per row of the TMA-streamed kernel; 0 = tiles do not fit, use the sub-warp kernel
  int dtype = B200_F64;
  int64_t m_local = 0, n_global = 0, row_begin = 0, nnz = 0, n_halo = 0;
  int64_t m_global = 0;    // size(A,1); != n_global only for single-GPU rectangular operators (lsqr!/lsmr!)
  // row offsets, m_local+1 (+ kRowptrPad): exactly one of the two is allocated.  Single-GPU operators with nnz >=
  // INT32_MAX (or built on a context with "rowptr64" = 1) get rowptr64, every other operator rowptr.
  int *rowptr = nullptr;
  int64_t *rowptr64 = nullptr;
  int *colind = nullptr;   // nnz; local extended index: [0,m_local) own, [m_local,m_local+n_halo) halo
  void *vals = nullptr;    // nnz
  int max_row_nnz = 0;
  double avg_row_nnz = 0.0;
  // band description (single GPU, every 512-row tile has <= 8 distinct offsets col - row, columns strictly ascending
  // in every row): the structure of the operator without colind/rowptr, consumed by the band-streamed SpMV
  // (spmv_stream.cuh).  vals stay the CSR's own array.
  bool band_ok = false;
  struct b200_band_tile *band_hdr = nullptr;  // one 64-byte header per tile
  uint8_t *band_mask = nullptr;               // one byte per row (padded to whole tiles): bit j = the row has offset j
  // value tables of the uniform tiles (header pad[1] == 1): 8 values of the element type per tile, indexed by tile; kept
  // only when band_uniform > 0.  band_uniform_nnz: the nonzeros those tiles hold
  void *band_val = nullptr;
  int64_t band_uniform = 0, band_uniform_nnz = 0;
  // halo exchange state (world > 1)
  std::vector<int64_t> send_count, send_offset, recv_count, recv_offset;  // per peer
  int64_t n_send = 0;
  int *send_idx = nullptr;   // device: local row index to pack, grouped by peer
  void *send_buf = nullptr;  // device: n_send values
  void *halo = nullptr;      // device: n_halo values (recv buffer == halo part of the extended vector), NCCL path
  // peer-memory path (peer.cuh): the halo segment lives in this rank's comm buffer, neighbours store into it
  bool peer_halo = false;
  void *halo_peer = nullptr;               // = ctx->peer_local + kPeerHeaderBytes
  std::vector<int64_t> peer_dst_offset;    // [peer] element offset of MY values inside the peer's halo segment
  std::vector<int64_t> send_range_lo;      // [peer] first local row when the rows sent to `peer` are ONE ascending contiguous range
                                           // (slabs of banded operators), -1 otherwise
  unsigned int recv_mask = 0, send_mask = 0;
  // lazily built analysis of the stationary sweeps (stationary.cu): diagonal positions and dependency levels; the
  // operator is immutable, so the plan stays valid for its lifetime
  mutable void *st_plan = nullptr;
  mutable void (*st_plan_free)(void *) = nullptr;
};

namespace b200 {
// packs x[send_idx] and exchanges with the peers; after return (stream-ordered) A->halo is valid
int halo_exchange(b200_ctx *ctx, const b200_csr *A, const void *x_dev);
// peer-memory variant: stores x[send_idx] into the neighbours' halo segments and raises halo flag `seq`
// (skipped on the device when *done_flag != 0); consumers wait with peer_wait_halo(.., A->recv_mask, seq)
int halo_push(b200_ctx *ctx, const b200_csr *A, const void *x_dev, unsigned long long seq, const int *done_flag);
inline bool is_square(const b200_csr *A) { return A->m_global == A->n_global; }
// f(rowptr) with the operator's row offsets at their own width (const int * or const int64_t *)
template <typename F>
inline auto with_rowptr(const b200_csr *A, F &&f) {
  return A->rowptr64 ? f((const int64_t *)A->rowptr64) : f((const int *)A->rowptr);
}
// real_only (common.cuh) for an operator argument (NULL is left to the entry point's own argument check)
inline int real_only(const b200_csr *A, const char *entry) { return A ? real_only(A->dtype, entry) : B200_OK; }
inline bool use_peer(const b200_ctx *ctx, const b200_csr *A) {
  return ctx->world > 1 && ctx->peer_ok && A->peer_halo && ctx->opt_comm != 1;
}
// a single-GPU m x n operator from device CSR arrays (int32 row offsets, ascending columns, fp64 values rounded to
// dtype), the arrays copied; the levels of the device AMG setup (amg_setup.cu)
int csr_from_device_f64(b200_ctx *ctx, int64_t m, int64_t n, int64_t nnz, const int *rowptr, const int *colind,
                        const double *vals, int dtype, b200_csr **out);
}  // namespace b200
