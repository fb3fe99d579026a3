// spmv_stream.cuh -- the TMA-streamed CSR SpMV body shared by b200_spmv and the fused solver kernels.
//
// Why: with ~7 nonzeros per row a "warp(-slice) per row" kernel is latency-bound: every row costs a
// dependent chain rowptr -> (colind, vals) -> x[col] with one row in flight per lane group
// (latency-bound, far below the HBM bandwidth).  Here the matrix is consumed as what it is in
// HBM -- three contiguous streams -- and only the x gather stays a per-thread load:
//
//   * rows are cut into uniform tiles of R = 512/LPR rows; the nonzeros of a tile are one contiguous
//     range of vals/colind, the row pointers one contiguous range of rowptr;
//   * a producer warp (one elected lane) moves the three ranges of the next tiles into a 4-stage
//     shared-memory ring with cp.async.bulk (the TMA engine; SASS: UBLKCP); completion is tracked by
//     mbarriers (full[stage]: expect_tx bytes; empty[stage]: one arrive per consumer warp of the group
//     that owns the tile).  The copies carry an L2 evict-first policy so the 12 B/nnz stream does not
//     evict x from L2;
//   * consumers read rowptr/colind/vals from shared memory (no dependent global loads) and issue all x
//     gathers of their rows back to back; x comes from L1/L2;
//   * the x gather of a row ends in a DRAM miss roughly once per row (first touch of the leading stencil
//     plane), so a tile's consumer latency is a loaded DRAM round trip (~2500 clk): the first streamed
//     version (one tile in consumer flight per CTA, 512 rows per SM) was bound by exactly that --
//     ncu: DRAM 65 %, L2 44 %, issue 40 %, "long scoreboard" the top stall.  Therefore the 16 consumer
//     warps form TWO groups that work on alternate tiles concurrently and every thread owns TWO rows:
//     1024 rows (7168 gathers) in flight per SM while two more tiles are landing;
//   * the grid is persistent: 1 CTA per SM, tiles interleaved across CTAs (k-th tile of CTA b is
//     b + k*gridDim) so that all resident CTAs sweep neighbouring rows and the x planes stay in L2.
//
// LPR (lanes per row) = 1 for matrices whose tiles of 512 rows hold <= 4096 nonzeros (the 5/7-point
// stencils), 2/4/../32 for denser rows; operators whose 16-row tiles exceed 4096 nonzeros fall back to
// the sub-warp kernel (spmv.cuh).  With LPR == 1 and fp64 the row sum is accumulated left to right
// with separate multiply and add, i.e. bit-identical to SparseArrays' CSC scatter for a matrix given
// with sorted columns.
//
// Operators with a band description (csr.cuh: <= 8 distinct offsets col - row per 512-row tile) take the second body
// below, spmv_band_tiles: the same tiles and thread mapping, but the producer stages per-tile masks and contiguous
// x bands instead of colind/rowptr, so a tile costs 8 B/nonzero + 1 B/row + 64 B of HBM structure and the consumers
// no longer gather x from L1/L2 at all.
#pragma once
#include "spmv.cuh"

namespace b200 {

constexpr int kStreamGroupThreads = 256;                  // consumer threads per group (8 warps)
constexpr int kStreamGroups = 2;                          // groups working on alternate tiles
constexpr int kStreamConsumers = kStreamGroupThreads * kStreamGroups;
constexpr int kStreamThreads = kStreamConsumers + 32;     // + producer warp
constexpr int kStreamTileRows = 512;                      // rows per tile at LPR == 1 (2 per thread)
constexpr int kStreamNnzCap = 4096;                       // nonzeros per tile
constexpr int kStreamStages = 4;
constexpr int kStreamCtasPerSm = 1;

// I: the operator's row offsets (csr.cuh), staged at their own width.  8-byte offsets add 2 KB per stage: in fp64 a
// stage is 53,504 B instead of 51,328 B, and the 4 stages still fit the 227 KB of shared memory.
template <typename T, typename I = int>
struct alignas(128) StreamStage {
  T val[kStreamNnzCap + 8];
  int col[kStreamNnzCap + 8];
  I rp[kStreamTileRows + 8];
};
template <typename T, typename I = int>
struct StreamSmem {
  StreamStage<T, I> stage[kStreamStages];
  alignas(8) unsigned long long full[kStreamStages];
  alignas(8) unsigned long long empty[kStreamStages];
};

#ifdef __CUDACC__

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// TMA 1-D bulk copy global -> shared, completion counted in bytes on an mbarrier, L2 cache policy
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes,
                                         unsigned long long *bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
      ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}

// Runs over all tiles of this CTA.  `epi(row, value)` is called once per row by the lane that owns
// the row result.  Must be called by all kStreamThreads threads of the block.
template <typename T, int LPR, typename XV, typename Epi, typename I>
__device__ __forceinline__ void spmv_stream_tiles(const I *__restrict__ rowptr, const int *__restrict__ colind,
                                                  const T *__restrict__ vals, const XV &xv, int64_t m, Epi &epi,
                                                  StreamSmem<T, I> *sm, bool rev = false) {
  constexpr int R = kStreamTileRows / LPR;          // rows per tile
  constexpr int SLOTS = kStreamGroupThreads / LPR;  // row slots per group; each slot owns rows s and s+SLOTS
  const int tid = threadIdx.x;
  const int64_t ntiles = (m + R - 1) / R;
  // `rev`: sweep the tiles from the last to the first.  Consecutive kernels of a solver alternate the sweep
  // direction so that each one starts on the rows the previous kernel touched last (still in L2).
  auto phys = [&](int64_t seq) -> int64_t { return rev ? ntiles - 1 - seq : seq; };
  if (tid == 0) {
    for (int s = 0; s < kStreamStages; ++s) {
      mbar_init(&sm->full[s], 1);
      mbar_init(&sm->empty[s], kStreamGroupThreads / 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (tid >= kStreamConsumers) {
    // ------------------------------------------------------------ producer warp
    if (tid == kStreamConsumers) {
      const uint64_t pol_stream = policy_evict_first();
      int64_t t = blockIdx.x;
      // bounds of the next tile are fetched one iteration ahead (off the critical path)
      I k0 = 0, k1 = 0;
      if (t < ntiles) {
        const int64_t r0 = phys(t) * R, r1 = (r0 + R < m) ? (r0 + R) : m;
        k0 = __ldg(rowptr + r0);
        k1 = __ldg(rowptr + r1);
      }
      for (int it = 0; t < ntiles; ++it) {
        const int s = it % kStreamStages;
        const uint32_t ph = (uint32_t)((it / kStreamStages) & 1);
        const int64_t r0 = phys(t) * R;
        const int64_t tn = t + gridDim.x;
        I nk0 = 0, nk1 = 0;
        if (tn < ntiles) {
          const int64_t nr0 = phys(tn) * R, nr1 = (nr0 + R < m) ? (nr0 + R) : m;
          nk0 = __ldg(rowptr + nr0);
          nk1 = __ldg(rowptr + nr1);
        }
        mbar_wait(&sm->empty[s], ph ^ 1u);
        const I k0a = k0 & ~(I)3;
        const uint32_t cnt = (uint32_t)(((k1 - k0a) + 3) & ~3);
        const uint32_t b_val = cnt * (uint32_t)sizeof(T), b_col = cnt * 4u, b_rp = (uint32_t)(R + 4) * (uint32_t)sizeof(I);
        StreamStage<T, I> *st = &sm->stage[s];
        mbar_expect_tx(&sm->full[s], b_val + b_col + b_rp);
        bulk_g2s(st->rp, rowptr + r0, b_rp, &sm->full[s], pol_stream);
        bulk_g2s(st->col, colind + k0a, b_col, &sm->full[s], pol_stream);
        bulk_g2s(st->val, vals + k0a, b_val, &sm->full[s], pol_stream);
        t = tn;
        k0 = nk0;
        k1 = nk1;
      }
    }
  } else {
    // ------------------------------------------------------------ consumers: group g takes tiles k = g, g+2, ...
    const int grp = tid / kStreamGroupThreads;
    const int lt = tid % kStreamGroupThreads;
    const int sub = lt % LPR, slot = lt / LPR;
    for (int64_t k = grp;; k += kStreamGroups) {
      const int64_t t = (int64_t)blockIdx.x + k * gridDim.x;
      if (t >= ntiles) break;
      const int s = (int)(k % kStreamStages);
      const uint32_t ph = (uint32_t)((k / kStreamStages) & 1);
      const int64_t r0 = phys(t) * R;
      mbar_wait(&sm->full[s], ph);
      const StreamStage<T, I> *st = &sm->stage[s];
      const I k0a = st->rp[0] & ~(I)3;
      int b[2], e[2];
      bool valid[2];
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int rib = slot + q * SLOTS;
        valid[q] = r0 + rib < m;
        b[q] = valid[q] ? (int)(st->rp[rib] - k0a) : 0;   // tile-relative: a tile holds <= kStreamNnzCap nonzeros
        e[q] = valid[q] ? (int)(st->rp[rib + 1] - k0a) : 0;
      }
      T acc[2] = {(T)0, (T)0};
      // the epilogue's own per-row operand (e.g. MINRES' v_prev[row]) is requested BEFORE the gathers so that its
      // DRAM latency overlaps theirs; loaded after them it doubled the time a tile occupies its stage
      T pre[2] = {(T)0, (T)0};
      if (sub == 0) {
        if (valid[0]) pre[0] = epi.pre(r0 + slot);
        if (valid[1]) pre[1] = epi.pre(r0 + slot + SLOTS);
      }
      if constexpr (LPR == 1) {
        // 2 rows x up to 8 gathers in flight; left-to-right, unfused multiply-add (see header comment)
        int kk0 = b[0], kk1 = b[1];
        while (kk0 < e[0] || kk1 < e[1]) {
          T xa[2][8];   // the gathers; vals are re-read from shared memory at multiply time (registers)
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const bool on0 = kk0 + j < e[0], on1 = kk1 + j < e[1];
            const int c0 = on0 ? st->col[kk0 + j] : 0;
            const int c1 = on1 ? st->col[kk1 + j] : 0;
            xa[0][j] = on0 ? xv(c0) : (T)0;
            xa[1][j] = on1 ? xv(c1) : (T)0;
          }
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            if (kk0 + j < e[0]) {
              if constexpr (sizeof(T) == 8) acc[0] = __dadd_rn(acc[0], __dmul_rn(st->val[kk0 + j], xa[0][j]));
              else acc[0] = __fadd_rn(acc[0], __fmul_rn(st->val[kk0 + j], xa[0][j]));
            }
            if (kk1 + j < e[1]) {
              if constexpr (sizeof(T) == 8) acc[1] = __dadd_rn(acc[1], __dmul_rn(st->val[kk1 + j], xa[1][j]));
              else acc[1] = __fadd_rn(acc[1], __fmul_rn(st->val[kk1 + j], xa[1][j]));
            }
          }
          kk0 += 8;
          kk1 += 8;
        }
      } else {
        int kk0 = b[0] + sub, kk1 = b[1] + sub;
        while (kk0 < e[0] || kk1 < e[1]) {
          T xa[2][4], va[2][4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const bool on0 = kk0 + j * LPR < e[0], on1 = kk1 + j * LPR < e[1];
            const int c0 = on0 ? st->col[kk0 + j * LPR] : 0;
            const int c1 = on1 ? st->col[kk1 + j * LPR] : 0;
            va[0][j] = on0 ? st->val[kk0 + j * LPR] : (T)0;
            va[1][j] = on1 ? st->val[kk1 + j * LPR] : (T)0;
            xa[0][j] = on0 ? xv(c0) : (T)0;
            xa[1][j] = on1 ? xv(c1) : (T)0;
          }
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            acc[0] += va[0][j] * xa[0][j];
            acc[1] += va[1][j] * xa[1][j];
          }
          kk0 += 4 * LPR;
          kk1 += 4 * LPR;
        }
#pragma unroll
        for (int o = LPR >> 1; o > 0; o >>= 1) {
          acc[0] += __shfl_xor_sync(0xffffffffu, acc[0], o, LPR);
          acc[1] += __shfl_xor_sync(0xffffffffu, acc[1], o, LPR);
        }
      }
      if (sub == 0) {
        if (valid[0]) epi(r0 + slot, acc[0], pre[0]);
        if (valid[1]) epi(r0 + slot + SLOTS, acc[1], pre[1]);
      }
      __syncwarp();
      if ((tid & 31) == 0) mbar_arrive(&sm->empty[s]);
    }
  }
}

#endif  // __CUDACC__

// ------------------------------------------------------------------------------------------------
// Band-streamed form (operators with A->band_ok, csr.cuh): the structure of a tile of 512 rows is its <= 8 distinct
// offsets d_j = col - row (the tile header, read by the producer one tile ahead) and one mask byte per row (bit j: the
// row has offset d_j).  Every x operand of the tile then lies in the band x[r0+d_j, r0+d_j+rows), so the producer
// bulk-copies, per stage: the tile's vals (evict-first, as above), its masks, and one x band per offset (default L2
// policy: the bands are the L2 reuse the sweep order relies on).  Consumers touch only shared memory: a row's first
// nonzero in the stage is the prefix popcount of the masks before it (one scan per group and tile), and the row sum is
// taken over the set mask bits in ascending j = ascending column, left to right with unfused multiply and add --
// bit-identical to the CSR stream.  Per SpMV this reads vals, 1 B/row of masks and 64 B/tile of headers instead of
// 4 B/nonzero of colind and 4 B/row of rowptr.  A uniform tile (csr.cuh: every offset holds one value) replaces its vals
// by its 8-value table, so an operator whose tiles are all uniform (constant-coefficient stencils) reads no vals at all.
// ------------------------------------------------------------------------------------------------
constexpr int kBandMax = 8;      // offsets per tile
constexpr int kBandStages = 3;     // 3 x 66 KB (fp64) of the 227 KB of shared memory
constexpr int kBandStagesVF = 6;   // value-free stages (every tile uniform): 6 x 33 KB (fp64)
// the same tiles, rows per thread and CTA interleave as spmv_stream_tiles<T, 1>: every row result and every epilogue
// partial sum (cg!'s dot(u, c)) is formed by the same thread in the same order, so the two forms are bit-identical
static_assert(kBandTileRows == kStreamTileRows, "band tiles are the LPR == 1 stream tiles");

// VF (value-free): every tile of the operator is uniform, so no stage ever receives vals; without the val region a stage
// is half the size and the ring twice as deep, which keeps twice as many tiles' x bands landing per SM
template <typename T, bool VF = false>
struct alignas(128) BandStage {
  T val[VF ? 16 / sizeof(T) : kStreamNnzCap + 8];   // VF: a 16-byte stub, never read
  // band j holds x[bs_j, be_j): bs_j rounded down and be_j up to 16 bytes, so at most R + 2*(16/sizeof(T) - 1) entries
  T xb[kBandMax][kStreamTileRows + 32 / sizeof(T)];
  uint8_t mask[kStreamTileRows];
  alignas(16) T tv[kBandMax];   // a uniform tile's value per offset (its value table), copied instead of val
};
template <typename T, bool VF = false>
struct BandSmem {
  static constexpr int S = VF ? kBandStagesVF : kBandStages;
  BandStage<T, VF> stage[S];
  // written by the producer with ordinary stores before it arrives on full[s] (never a bulk-copy target):
  // band[s][j] = {index in xb[j] of row 0's operand, entries copied, bs_j, 0}; kofs[s] = first nonzero - first copied;
  // uni[s] = 1: the stage holds the tile's value table in tv instead of its vals
  int4 band[S][kBandMax];
  int kofs[S];
  int uni[S];
  int fill[S];   // number of the last fill the producer started on each stage (-1: none yet)
  int scan[kStreamGroups][2][kStreamGroupThreads / 32];
  alignas(8) unsigned long long full[S];
  alignas(8) unsigned long long empty[S];
};

// tab: the value tables of the uniform tiles (b200_csr::band_val, kBandMax values of the element type per tile), or null:
// every tile streams its vals (the operator has no uniform tile, or the context option "band_values" is 0)
struct BandArgs {
  const b200_band_tile *hdr;
  const uint8_t *mask;
  const void *tab;
};
// the same description of an operator with 8-byte row offsets: tile bounds k0, k1 are 64-bit (b200_band_tile)
struct BandArgs64 {
  const b200_band_tile *hdr;
  const uint8_t *mask;
  const void *tab;
};

#ifdef __CUDACC__

__device__ __forceinline__ int ld_acquire_shared(const int *p) {
  int v;
  asm volatile("ld.acquire.cta.shared::cta.b32 %0, [%1];" : "=r"(v) : "r"(smem_u32(p)) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_shared(int *p, int v) {
  asm volatile("st.release.cta.shared::cta.b32 [%0], %1;" ::"r"(smem_u32(p)), "r"(v) : "memory");
}

__device__ __forceinline__ void bulk_g2s_plain(void *dst_smem, const void *src_gmem, uint32_t bytes,
                                               unsigned long long *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// Same contract as spmv_stream_tiles (LPR == 1): `x` (nx entries, 16-byte aligned) is the operand, m the rows.  VF: every
// tile of the operator is uniform and ba.tab is not null (BandStage).
template <typename T, bool VF, typename Epi, typename BA>
__device__ __forceinline__ void spmv_band_tiles(const BA ba, const T *__restrict__ vals, const T *__restrict__ x,
                                                int64_t nx, int64_t m, Epi &epi, BandSmem<T, VF> *sm, bool rev = false) {
  constexpr int R = kStreamTileRows;
  constexpr int SLOTS = kStreamGroupThreads;
  constexpr int AL = 16 / (int)sizeof(T);   // elements per 16 bytes
  constexpr int S = BandSmem<T, VF>::S;     // stages
  const int tid = threadIdx.x;
  const int64_t ntiles = (m + R - 1) / R;
  auto phys = [&](int64_t seq) -> int64_t { return rev ? ntiles - 1 - seq : seq; };
  if (tid == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&sm->full[s], 1);
      mbar_init(&sm->empty[s], kStreamGroupThreads / 32);
      sm->fill[s] = -1;
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (tid >= kStreamConsumers) {
    // ------------------------------------------------------------ producer warp
    if (tid == kStreamConsumers) {
      const uint64_t pol_stream = policy_evict_first();
      const int64_t nxa = nx & ~(int64_t)(AL - 1);   // bands never copy past the last whole 16 bytes of x
      int64_t t = blockIdx.x;
      // the header of the next tile is fetched one iteration ahead (off the critical path)
      int4 h0 = make_int4(0, 0, 0, 0), h1 = h0, h2 = h0, h3 = h0;
      if (t < ntiles) {
        const int4 *p = reinterpret_cast<const int4 *>(ba.hdr + phys(t));
        h0 = __ldg(p);
        h1 = __ldg(p + 1);
        h2 = __ldg(p + 2);
        h3 = __ldg(p + 3);
      }
      for (int it = 0; t < ntiles; ++it) {
        const int s = it % S;
        const uint32_t ph = (uint32_t)((it / S) & 1);
        const int64_t r0 = phys(t) * R;
        const int64_t rows = (r0 + R < m) ? R : m - r0;
        const int64_t tn = t + gridDim.x;
        int4 n0 = make_int4(0, 0, 0, 0), n1 = n0, n2 = n0, n3 = n0;
        if (tn < ntiles) {
          const int4 *p = reinterpret_cast<const int4 *>(ba.hdr + phys(tn));
          n0 = __ldg(p);
          n1 = __ldg(p + 1);
          n2 = __ldg(p + 2);
          n3 = __ldg(p + 3);
        }
        const int off[kBandMax] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
        constexpr bool K64 = std::is_same<BA, BandArgs64>::value;
        typedef typename std::conditional<K64, int64_t, int>::type K;
        const int nb = h2.x;
        K k0, k1;
        if constexpr (K64) {
          k0 = (int64_t)(((uint64_t)(uint32_t)h2.w << 32) | (uint32_t)h2.y);
          k1 = k0 + (uint32_t)(h2.z - h2.y);
        } else {
          k0 = h2.y;
          k1 = h2.z;
        }
        // a uniform tile (header pad[1]) copies its value table instead of its vals
        const bool uni = VF || (ba.tab != nullptr && h3.x != 0);
        mbar_wait(&sm->empty[s], ph ^ 1u);
        const K k0a = k0 & ~(K)3;
        const uint32_t b_val = uni ? 0u : (uint32_t)(((k1 - k0a) + 3) & ~3) * (uint32_t)sizeof(T);
        const uint32_t b_tab = uni ? (uint32_t)(kBandMax * sizeof(T)) : 0u;
        uint32_t total = b_val + b_tab + (uint32_t)R;
        int64_t bsj[kBandMax];
        uint32_t bb[kBandMax];
#pragma unroll
        for (int j = 0; j < kBandMax; ++j) {
          int4 e = make_int4(0, 0, 0, 0);
          bsj[j] = 0;
          bb[j] = 0;
          if (j < nb) {
            // clamp the band to [0, nx); masks guarantee no row of the tile reads outside it
            const int64_t lo = r0 + off[j] > 0 ? r0 + off[j] : 0;
            const int64_t hi = r0 + off[j] + rows < nx ? r0 + off[j] + rows : nx;
            const int64_t bs = lo & ~(int64_t)(AL - 1);
            const int64_t be_up = (hi + AL - 1) & ~(int64_t)(AL - 1);
            const int64_t be = be_up < nxa ? be_up : nxa;
            const int64_t cnt = be > bs ? be - bs : 0;
            e = make_int4((int)(r0 + off[j] - bs), (int)cnt, (int)bs, 0);
            bsj[j] = bs;
            bb[j] = (uint32_t)cnt * (uint32_t)sizeof(T);
            total += bb[j];
          }
          sm->band[s][j] = e;
        }
        sm->kofs[s] = (int)(k0 - k0a);
        sm->uni[s] = uni ? 1 : 0;
        st_release_shared(&sm->fill[s], it / S);   // see the consumers' wait
        BandStage<T, VF> *st = &sm->stage[s];
        mbar_expect_tx(&sm->full[s], total);   // releases the ordinary stores above together with the arrival
        bulk_g2s(st->mask, ba.mask + r0, (uint32_t)R, &sm->full[s], pol_stream);
        if (uni)
          bulk_g2s(st->tv, static_cast<const T *>(ba.tab) + phys(t) * kBandMax, b_tab, &sm->full[s], pol_stream);
        else if constexpr (!VF)
          bulk_g2s(st->val, vals + k0a, b_val, &sm->full[s], pol_stream);
#pragma unroll
        for (int j = 0; j < kBandMax; ++j)
          if (bb[j]) bulk_g2s_plain(st->xb[j], x + bsj[j], bb[j], &sm->full[s]);
        t = tn;
        h0 = n0;
        h1 = n1;
        h2 = n2;
        h3 = n3;
      }
    }
  } else {
    // ------------------------------------------------------------ consumers: group g takes tiles k = g, g+2, ...
    const int grp = tid / kStreamGroupThreads;
    const int slot = tid % kStreamGroupThreads;
    const int lane = tid & 31, wig = slot >> 5;   // warp in group
    // the epilogue's own per-row operands (e.g. cg!'s u[row]) are loaded one tile of the group ahead, so that their
    // latency overlaps the current tile instead of stalling its epilogue; the kernel does not write what they read
    auto pre_of = [&](int64_t kk, T (&p)[2]) {
      const int64_t tt = (int64_t)blockIdx.x + kk * gridDim.x;
      const int64_t row = tt < ntiles ? phys(tt) * R + slot : m;
      p[0] = row < m ? epi.pre(row) : (T)0;
      p[1] = row + SLOTS < m ? epi.pre(row + SLOTS) : (T)0;
    };
    T pre_next[2];
    pre_of(grp, pre_next);
    int nscan = 0;
    for (int64_t k = grp;; k += kStreamGroups) {
      const int64_t t = (int64_t)blockIdx.x + k * gridDim.x;
      if (t >= ntiles) break;
      const int s = (int)(k % S);
      const uint32_t ph = (uint32_t)((k / S) & 1);
      const int64_t r0 = phys(t) * R;
      const bool valid0 = r0 + slot < m, valid1 = r0 + slot + SLOTS < m;
      const T pre[2] = {pre_next[0], pre_next[1]};
      pre_of(k + kStreamGroups, pre_next);
      // With 3 stages and 2 groups, consecutive fills of a stage belong to DIFFERENT groups (tile k - 3 is the other
      // group's), so this group can reach its wait for fill n = k/3 of stage s while fill n - 1 is still landing.  The
      // parity of fill n is that of fill n - 2, long complete, so a parity wait alone would return at once: the group
      // would read a stage that is still being written and arrive on the wrong phase of empty[s], desynchronising the
      // ring until it hangs.  The producer therefore publishes the number of the fill it has started on each stage;
      // once that is n, fill n - 1 has been consumed (the producer waited for it) and fill n + 1 cannot start before
      // this group releases the stage, so the parity wait refers to fill n alone.  (With the 6 value-free stages a stage
      // stays with one group; the same wait is kept, so the ring's correctness does not rest on the stage count.)
      const int fill_no = (int)(k / S);
      while (ld_acquire_shared(&sm->fill[s]) != fill_no) __nanosleep(32);
      mbar_wait(&sm->full[s], ph);
      const BandStage<T, VF> *st = &sm->stage[s];
      const uint32_t mk0 = st->mask[slot], mk1 = st->mask[slot + SLOTS];   // 0 past the last row
      T acc[2] = {(T)0, (T)0};
      // left-to-right, unfused multiply-add in ascending column order (see the comment above).  The branch is uniform
      // across the block; a uniform tile's value of offset j is the same bit pattern as every vals entry it stands for
      if (VF || sm->uni[s]) {
#pragma unroll
        for (int j = 0; j < kBandMax; ++j) {
          const int4 bj = sm->band[s][j];
          const T vj = st->tv[j];
          if ((mk0 >> j) & 1u) {
            const int p = slot + bj.x;
            const T xj = p < bj.y ? st->xb[j][p] : __ldg(x + ((int64_t)bj.z + p));
            if constexpr (sizeof(T) == 8) acc[0] = __dadd_rn(acc[0], __dmul_rn(vj, xj));
            else acc[0] = __fadd_rn(acc[0], __fmul_rn(vj, xj));
          }
          if ((mk1 >> j) & 1u) {
            const int p = slot + SLOTS + bj.x;
            const T xj = p < bj.y ? st->xb[j][p] : __ldg(x + ((int64_t)bj.z + p));
            if constexpr (sizeof(T) == 8) acc[1] = __dadd_rn(acc[1], __dmul_rn(vj, xj));
            else acc[1] = __fadd_rn(acc[1], __fmul_rn(vj, xj));
          }
        }
      } else {
        // row starts: exclusive prefix of the popcounts over the group, both rows' counts packed in one int
        const int own = __popc(mk0) | (__popc(mk1) << 16);
        int inc = own;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int v = __shfl_up_sync(0xffffffffu, inc, o);
          if (lane >= o) inc += v;
        }
        // the two scan buffers alternate per scan the group takes (uniform tiles take none), so a buffer is rewritten
        // only after a bar.sync that follows every read of its previous contents
        int *scan = sm->scan[grp][nscan++ & 1];
        if (lane == 31) scan[wig] = inc;
        asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "r"(kStreamGroupThreads) : "memory");
        int before = 0, all = 0;
#pragma unroll
        for (int w = 0; w < kStreamGroupThreads / 32; ++w) {
          const int v = scan[w];
          if (w < wig) before += v;
          all += v;
        }
        const int excl = before + inc - own;
        const int kofs = sm->kofs[s];
        int kk0 = kofs + (excl & 0xffff);
        int kk1 = kofs + (all & 0xffff) + (excl >> 16);
#pragma unroll
        for (int j = 0; j < kBandMax; ++j) {
          const int4 bj = sm->band[s][j];
          if ((mk0 >> j) & 1u) {
            const int p = slot + bj.x;
            const T xj = p < bj.y ? st->xb[j][p] : __ldg(x + ((int64_t)bj.z + p));
            if constexpr (sizeof(T) == 8) acc[0] = __dadd_rn(acc[0], __dmul_rn(st->val[kk0], xj));
            else acc[0] = __fadd_rn(acc[0], __fmul_rn(st->val[kk0], xj));
            ++kk0;
          }
          if ((mk1 >> j) & 1u) {
            const int p = slot + SLOTS + bj.x;
            const T xj = p < bj.y ? st->xb[j][p] : __ldg(x + ((int64_t)bj.z + p));
            if constexpr (sizeof(T) == 8) acc[1] = __dadd_rn(acc[1], __dmul_rn(st->val[kk1], xj));
            else acc[1] = __fadd_rn(acc[1], __fmul_rn(st->val[kk1], xj));
            ++kk1;
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm->empty[s]);   // the stage is no longer read; the epilogue touches global memory only
      if (valid0) epi(r0 + slot, acc[0], pre[0]);
      if (valid1) epi(r0 + slot + SLOTS, acc[1], pre[1]);
    }
  }
}

#endif  // __CUDACC__

// true if the TMA-streamed kernel serves this operator (tiles fit, not overridden by the option)
inline bool use_stream(const b200_ctx *ctx, const b200_csr *A) {
  return A->stream_lpr > 0 && ctx->opt_spmv_kernel != 1;
}
// true if the band-streamed form serves y = A x: the operator has a band description, the option is auto (0) or
// band (3), and x is 16-byte aligned (bulk copies; user vectors may be offset views)
inline bool use_band(const b200_ctx *ctx, const b200_csr *A, const void *x) {
  return A->band_ok && (ctx->opt_spmv_kernel == 0 || ctx->opt_spmv_kernel == 3) && ((uintptr_t)x & 15u) == 0;
}
inline int stream_grid_size(const b200_ctx *ctx, const b200_csr *A) {
  const int R = kStreamTileRows / A->stream_lpr;
  const int64_t ntiles = (A->m_local + R - 1) / R;
  const int64_t cap = (int64_t)ctx->sm_count * kStreamCtasPerSm;
  return (int)(ntiles < cap ? ntiles : cap);
}

}  // namespace b200
