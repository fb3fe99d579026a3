// amg_setup.cu -- the setup of smoothed aggregation on the device (DESIGN section 23), bit for bit amg_core.h's
// amg_setup (which stays the serial reference of the CPU tests).  All setup arithmetic is fp64 whatever A's element
// type, every product, sum and difference rounded on its own (__dmul_rn / __dadd_rn / __dsub_rn through mul_rn / add_rn
// / sub_rn: no contraction into FMA); division and sqrt are IEEE-rounded.  Per level:
//   checks       the first row (in row order) whose diagonal entry is missing or zero: an atomicMin over the rows
//   strength     a count pass and a fill pass per row (column order kept); S' by a stable radix sort by column
//   aggregation  pass 1 as the lexicographically-first MIS (amg_setup_core.h) in one launch: blocks take tickets in
//                row order and each row polls its smaller conflicting rows until it is decided (bounded polls; a row
//                still undecided makes the host launch again, so no launch can wait forever); ids by a scan over the
//                root flags; pass 2 per row; pass 3 by one thread over the compacted list of rows still free
//   T, B_c       members sorted stably by aggregate, one thread per aggregate sums them in row order
//   rho, w       a max over the rows' sums in column order (an integer atomicMax on the non-negative doubles' bits)
//   P            A T by the SpGEMM below, merged with T row by row as amg_prolongator, exact zeros dropped
//   R, A_c       R = P' (stable radix sort), A_c = R (A P) by the SpGEMM below
//   coarsest     downloaded and inverted on the host (amg_dense_inverse), at most kAmgMaxCoarsest rows
// SpGEMM (amg_setup_core.h's row functions): one warp per row accumulates in a shared-memory table of up to kSgCap
// slots; rows whose distinct columns overflow it are redone one warp per row on global-memory tables, in batches of at
// most kSgGlobalSlots slots (24 bytes each: 96 MB whatever n).  A count pass sizes the rows, a fill pass writes them.
// Level operators are built from the device arrays (csr_from_device_f64), values rounded to T.
#include <chrono>
#include <climits>
#include <cub/cub.cuh>

#include "amg_setup.cuh"
#include "amg_setup_core.h"

using namespace b200;

namespace {

constexpr int kThreads = 256;
constexpr int kSgWarps = 4, kSgCap = 512;          // on-chip SpGEMM: warps per block, table slots per warp
constexpr int64_t kSgGlobalSlots = 1 << 22;        // global-memory SpGEMM: table slots per batch
constexpr int kSgGlobalMinCap = 2 * kSgCap;
constexpr int kPass1Polls = 1 << 12;               // polls of one row per pass-1 launch
constexpr int kFree = -2;

double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

template <typename X>
struct Buf {   // a device array freed with its owner
  X *p = nullptr;
  Buf() = default;
  Buf(const Buf &) = delete;
  Buf &operator=(const Buf &) = delete;
  ~Buf() { cudaFree(p); }
  void reset() {
    cudaFree(p);
    p = nullptr;
  }
  int alloc(int64_t count) {
    reset();
    const size_t bytes = sizeof(X) * (size_t)(count > 0 ? count : 1);
    if (cudaMalloc(&p, bytes) != cudaSuccess) {
      p = nullptr;
      cudaGetLastError();
      set_error("b200_amg_create: cudaMalloc(%zu) failed", bytes);
      return B200_ERR_ALLOC;
    }
    return B200_OK;
  }
  void swap(Buf &o) { std::swap(p, o.p); }
};

struct DCsr {   // an owned fp64 CSR with int32 row offsets
  int64_t m = 0, n = 0, nnz = 0;
  Buf<int> rp, ci;
  Buf<double> v;
  AmgRows rows() const { return AmgRows{rp.p, ci.p, v.p}; }
  void reset() {
    rp.reset();
    ci.reset();
    v.reset();
    m = n = nnz = 0;
  }
  void swap(DCsr &o) {
    std::swap(m, o.m);
    std::swap(n, o.n);
    std::swap(nnz, o.nnz);
    rp.swap(o.rp);
    ci.swap(o.ci);
    v.swap(o.v);
  }
};

int grid(const b200_ctx *ctx, int64_t n) { return stream_grid(ctx, n, kThreads, 8); }

#define GRID_STRIDE(i, n) for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < (n); i += (int64_t)gridDim.x * blockDim.x)

template <typename X>
__global__ void k_fill(X *p, int64_t n, X v) {
  GRID_STRIDE(i, n) p[i] = v;
}

template <typename TI>
__global__ void k_to_f64(const TI *__restrict__ in, int64_t n, double *__restrict__ out) {
  GRID_STRIDE(i, n) out[i] = (double)in[i];
}

// bad[0]: the first row whose columns are not ascending (when `sorted` is checked); bad[1]: the first row whose diagonal
// entry is missing or zero; d = the diagonal (amg_diagonal)
__global__ void k_checks(AmgRows A, int64_t n, int sorted, int *bad, double *d) {
  GRID_STRIDE(i, n) {
    double di = 0.0;
    for (int p = A.rp[i]; p < A.rp[i + 1]; ++p) {
      if (sorted && p > A.rp[i] && A.ci[p - 1] >= A.ci[p]) atomicMin(bad, (int)i);
      if (A.ci[p] == i) di = A.v[p];
    }
    d[i] = di;
    if (di == 0.0) atomicMin(bad + 1, (int)i);
  }
}

__device__ __forceinline__ bool strong(const AmgRows &A, const double *d, double theta, int64_t i, int p) {
  const int j = A.ci[p];
  return j != i && fabs(A.v[p]) >= mul_rn(theta, sqrt(fabs(mul_rn(d[i], d[j]))));
}

// SymmetricStrength(theta): count pass (rp == nullptr: cnt[i] = row length) or fill pass
__global__ void k_strength(AmgRows A, const double *__restrict__ d, int64_t n, double theta, int *cnt, const int *rp,
                           int *ci) {
  GRID_STRIDE(i, n) {
    int c = 0;
    for (int p = A.rp[i]; p < A.rp[i + 1]; ++p)
      if (strong(A, d, theta, i, p)) {
        if (rp) ci[rp[i] + c] = A.ci[p];
        ++c;
      }
    if (!rp) cnt[i] = c;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// transpose: counts per column, a stable radix sort of the positions by column (rows stay ascending)
__global__ void k_col_count(const int *__restrict__ ci, int64_t nnz, int *cnt) {
  GRID_STRIDE(p, nnz) atomicAdd(cnt + ci[p], 1);
}
__global__ void k_row_ids(const int *__restrict__ rp, int64_t m, int *rows) {
  GRID_STRIDE(i, m) for (int p = rp[i]; p < rp[i + 1]; ++p) rows[p] = (int)i;
}
__global__ void k_iota(int *p, int64_t n) {
  GRID_STRIDE(i, n) p[i] = (int)i;
}
__global__ void k_transpose_gather(const int *__restrict__ perm, const int *__restrict__ rows,
                                   const double *__restrict__ v, int64_t nnz, int *ci, double *vo) {
  GRID_STRIDE(q, nnz) {
    ci[q] = rows[perm[q]];
    if (v) vo[q] = v[perm[q]];
  }
}

int end_bit_for(int64_t n) {
  int b = 1;
  while (b < 32 && (1ll << b) < (n > 1 ? n : 2)) ++b;
  return b;
}

// in place exclusive scan of p[0, count)
template <typename X>
int scan(b200_ctx *ctx, X *p, int64_t count) {
  size_t bytes = 0;
  B200_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, p, p, (int)count, ctx->stream));
  Buf<char> tmp;
  B200_TRY(tmp.alloc((int64_t)bytes));
  B200_CUDA(cub::DeviceScan::ExclusiveSum(tmp.p, bytes, p, p, (int)count, ctx->stream));
  ctx->launches++;
  return B200_OK;
}

// stable sort of (key, value) int pairs by key's low end_bit bits
int sort_pairs(b200_ctx *ctx, const unsigned *kin, unsigned *kout, const int *vin, int *vout, int64_t count, int end_bit) {
  size_t bytes = 0;
  B200_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, bytes, kin, kout, vin, vout, (int)count, 0, end_bit, ctx->stream));
  Buf<char> tmp;
  B200_TRY(tmp.alloc((int64_t)bytes));
  B200_CUDA(cub::DeviceRadixSort::SortPairs(tmp.p, bytes, kin, kout, vin, vout, (int)count, 0, end_bit, ctx->stream));
  ctx->launches++;
  return B200_OK;
}

// M' (m x n, nnz entries; values when M.v is set)
int transpose(b200_ctx *ctx, const AmgRows &M, int64_t m, int64_t n, int64_t nnz, DCsr *out) {
  cudaStream_t st = ctx->stream;
  out->m = n;
  out->n = m;
  out->nnz = nnz;
  B200_TRY(out->rp.alloc(n + 1));
  B200_TRY(out->ci.alloc(nnz));
  if (M.v) B200_TRY(out->v.alloc(nnz));
  B200_CUDA(cudaMemsetAsync(out->rp.p, 0, sizeof(int) * (size_t)(n + 1), st));
  if (nnz) {
    k_col_count<<<grid(ctx, nnz), kThreads, 0, st>>>(M.ci, nnz, out->rp.p);
    B200_LAUNCH_CHECK(ctx);
  }
  B200_TRY(scan(ctx, out->rp.p, n + 1));
  if (!nnz) return B200_OK;
  Buf<int> rows, pin, pout;
  Buf<unsigned> kout;
  B200_TRY(rows.alloc(nnz));
  B200_TRY(pin.alloc(nnz));
  B200_TRY(pout.alloc(nnz));
  B200_TRY(kout.alloc(nnz));
  k_row_ids<<<grid(ctx, m), kThreads, 0, st>>>(M.rp, m, rows.p);
  B200_LAUNCH_CHECK(ctx);
  k_iota<<<grid(ctx, nnz), kThreads, 0, st>>>(pin.p, nnz);
  B200_LAUNCH_CHECK(ctx);
  B200_TRY(sort_pairs(ctx, (const unsigned *)M.ci, kout.p, pin.p, pout.p, nnz, end_bit_for(n)));
  k_transpose_gather<<<grid(ctx, nnz), kThreads, 0, st>>>(pout.p, rows.p, M.v, nnz, out->ci.p, out->v.p);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// aggregation
__global__ void k_pass1_init(AmgRows S, int64_t n, int *state) {
  GRID_STRIDE(i, n) state[i] = amg_pass1_initial(S, (int)i);
}

// one thread per row, blocks in ticket order: every row a thread waits for is smaller, so it belongs to a block that
// took an earlier ticket and is running or done.  A row still undecided after kPass1Polls polls raises *left.
__global__ void __launch_bounds__(kThreads) k_pass1(AmgRows S, AmgRows St, int64_t n, int *state, unsigned *ticket,
                                                    int *left) {
  __shared__ unsigned blk;
  if (threadIdx.x == 0) blk = atomicAdd(ticket, 1u);
  __syncthreads();
  const int64_t i = (int64_t)blk * kThreads + threadIdx.x;
  if (i >= n) return;
  volatile int *vs = state;
  if (vs[i] != AMG_UNDECIDED) return;
  for (int t = 0; t < kPass1Polls; ++t) {
    const int s = amg_pass1_decide(S, St, (int)i, [&](int r) { return vs[r]; });
    if (s != AMG_UNDECIDED) {
      vs[i] = s;
      __threadfence();
      return;
    }
    __nanosleep(64);
  }
  *left = 1;
}

__global__ void k_root_flags(const int *__restrict__ state, int64_t n, int *f) {
  GRID_STRIDE(i, n) f[i] = state[i] == AMG_ROOT;
}

// a root's aggregate: itself and its strong row (disjoint for distinct roots)
__global__ void k_root_scatter(AmgRows S, const int *__restrict__ state, const int *__restrict__ id, int64_t n, int *x) {
  GRID_STRIDE(i, n) if (state[i] == AMG_ROOT) {
    x[i] = id[i];
    for (int p = S.rp[i]; p < S.rp[i + 1]; ++p) x[S.ci[p]] = id[i];
  }
}

__global__ void k_isolated(AmgRows S, int64_t n, int *x) {
  GRID_STRIDE(i, n) if (x[i] == kFree && S.rp[i] == S.rp[i + 1]) x[i] = -1;
}

// pass 2: a free row joins the pass-1 aggregate of its first strong neighbour (column order) that has one
__global__ void k_pass2(AmgRows S, int64_t n, const int *__restrict__ x1, int *x2) {
  GRID_STRIDE(i, n) {
    int a = x1[i];
    if (a == kFree)
      for (int p = S.rp[i]; p < S.rp[i + 1]; ++p)
        if (x1[S.ci[p]] >= 0) {
          a = x1[S.ci[p]];
          break;
        }
    x2[i] = a;
  }
}

__global__ void k_free_flags(const int *__restrict__ x, int64_t n, uint8_t *f) {
  GRID_STRIDE(i, n) f[i] = x[i] == kFree;
}

// pass 3, serial in row order over the rows still free after pass 2; *next: the number of aggregates, in and out
__global__ void k_pass3(AmgRows S, const int *__restrict__ rows, const int *__restrict__ count, int *x, int *next) {
  int a = *next;
  for (int r = 0; r < *count; ++r) {
    const int i = rows[r];
    if (x[i] != kFree) continue;
    x[i] = a;
    for (int p = S.rp[i]; p < S.rp[i + 1]; ++p)
      if (x[S.ci[p]] == kFree) x[S.ci[p]] = a;
    ++a;
  }
  *next = a;
}

// ---------------------------------------------------------------------------------------------------------------------
// T, B_c, rho, w, the P merge
__global__ void k_agg_keys(const int *__restrict__ x, int64_t n, unsigned *key, int *cnt) {
  GRID_STRIDE(i, n) {
    key[i] = (unsigned)(x[i] + 1);   // isolated rows first
    if (x[i] >= 0) atomicAdd(cnt + x[i], 1);
  }
}

// B_c[a] = sqrt(sum of B[i]^2 over the members in row order); members of a: sorted[n - aptr[naggs] + aptr[a] ...]
__global__ void k_bc(const int *__restrict__ aptr, const int *__restrict__ sorted, const double *__restrict__ B,
                     int64_t naggs, int64_t n, double *Bc) {
  GRID_STRIDE(a, naggs) {
    const int64_t off = n - aptr[naggs];
    double s = 0.0;
    for (int64_t p = off + aptr[a]; p < off + aptr[a + 1]; ++p) {
      const double b = B[sorted[p]];
      s = add_rn(s, mul_rn(b, b));
    }
    Bc[a] = sqrt(s);
  }
}

__global__ void k_t_flags(const int *__restrict__ x, int64_t n, int *f) {
  GRID_STRIDE(i, n) f[i] = x[i] >= 0;
}
__global__ void k_t_fill(const int *__restrict__ x, const double *__restrict__ B, const double *__restrict__ Bc,
                         const int *__restrict__ trp, int64_t n, int *tci, double *tv) {
  GRID_STRIDE(i, n) if (x[i] >= 0) {
    tci[trp[i]] = x[i];
    tv[trp[i]] = B[i] / Bc[x[i]];
  }
}

__global__ void k_rho(AmgRows A, const double *__restrict__ d, int64_t n, unsigned long long *rho) {
  GRID_STRIDE(i, n) {
    double s = 0.0;
    for (int p = A.rp[i]; p < A.rp[i + 1]; ++p) s = add_rn(s, fabs(A.v[p]));
    const double r = s / fabs(d[i]);
    if (r > 0.0) atomicMax(rho, (unsigned long long)__double_as_longlong(r));   // bits order like non-negative doubles
  }
}

template <typename T>
__global__ void k_weights(const double *__restrict__ d, double c, int64_t n, T *w) {
  GRID_STRIDE(i, n) w[i] = (T)(c / d[i]);
}

// P = T - c D^-1 (A T), row by row as amg_prolongator: count pass (prp == nullptr) or fill pass
__global__ void k_p_merge(AmgRows T, AmgRows AT, const double *__restrict__ d, double c, int64_t n, int64_t *cnt,
                          const int *prp, int *pci, double *pv) {
  GRID_STRIDE(i, n) {
    int p = T.rp[i], q = AT.rp[i];
    const int p1 = T.rp[i + 1], q1 = AT.rp[i + 1];
    const double s = 1.0 / d[i];
    int k = 0;
    while (p < p1 || q < q1) {
      const int jp = p < p1 ? T.ci[p] : INT_MAX, jq = q < q1 ? AT.ci[q] : INT_MAX;
      const int j = jp < jq ? jp : jq;
      const double t = jp == j ? T.v[p++] : 0.0;
      const double v = jq == j ? sub_rn(t, mul_rn(c, mul_rn(AT.v[q++], s))) : t;
      if (v != 0.0) {
        if (prp) {
          pci[prp[i] + k] = j;
          pv[prp[i] + k] = v;
        }
        ++k;
      }
    }
    if (!prp) cnt[i] = k;
  }
}

__global__ void k_rowptr32(const int64_t *__restrict__ in, int64_t n, int *out) {
  GRID_STRIDE(i, n + 1) out[i] = (int)in[i];
}

// ---------------------------------------------------------------------------------------------------------------------
// SpGEMM
struct WarpSync {
  __device__ bool operator()(bool ok) const {
    __syncwarp();
    return __all_sync(0xffffffffu, ok);
  }
};

// one warp per row on a shared-memory table of up to kSgCap slots (sized to the row's product count).  Count pass
// (FILL false): cnt[i] = the row's length, over[i] = 1 when the table overflowed.  Fill pass: rows with over[i] skipped.
template <bool FILL>
__global__ void __launch_bounds__(kSgWarps * 32) k_spgemm_chip(AmgRows A, AmgRows B, int64_t m, int64_t *cnt,
                                                               uint8_t *over, const int *crp, int *cci, double *cv) {
  __shared__ int keys[kSgWarps][kSgCap], lc[kSgWarps][kSgCap];
  __shared__ double acc[kSgWarps][kSgCap], lv[kSgWarps][kSgCap];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int s = lane; s < kSgCap; s += 32) {
    keys[w][s] = -1;
    acc[w][s] = 0.0;
  }
  __syncwarp();
  for (int64_t i = blockIdx.x * (int64_t)kSgWarps + w; i < m; i += (int64_t)gridDim.x * kSgWarps) {
    if (FILL && over[i]) continue;
    long long prod = 0;
    for (int p = A.rp[i] + lane; p < A.rp[i + 1]; p += 32) prod += B.rp[A.ci[p] + 1] - B.rp[A.ci[p]];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) prod += __shfl_xor_sync(0xffffffffu, prod, o);
    int cap = 32;
    while (cap < kSgCap && cap < 2 * prod) cap <<= 1;
    if (!amg_spgemm_accumulate(A, B, i, keys[w], acc[w], cap, lane, 32, WarpSync())) {
      for (int s = lane; s < cap; s += 32) {
        keys[w][s] = -1;
        acc[w][s] = 0.0;
      }
      if (!FILL && lane == 0) over[i] = 1;
      __syncwarp();
      continue;
    }
    const int u = amg_table_compact(keys[w], acc[w], cap, lane, 32, lc[w], lv[w]);
    __syncwarp();
    if (FILL) amg_spgemm_emit(lc[w], lv[w], u, lane, 32, cci + crp[i], cv + crp[i]);
    else if (lane == 0) cnt[i] = u;
    __syncwarp();
  }
}

__global__ void k_prod_count(AmgRows A, AmgRows B, const int *__restrict__ rows, int64_t nrows, int64_t *prod) {
  GRID_STRIDE(r, nrows) {
    const int i = rows[r];
    int64_t s = 0;
    for (int p = A.rp[i]; p < A.rp[i + 1]; ++p) s += B.rp[A.ci[p] + 1] - B.rp[A.ci[p]];
    prod[r] = s;
  }
}

// the rows that overflowed the on-chip table, one warp per row on its own slots [slot0[r], slot0[r+1]) of global tables
// (keys -1 and acc 0 on entry, left so)
template <bool FILL>
__global__ void __launch_bounds__(kThreads) k_spgemm_global(AmgRows A, AmgRows B, const int *__restrict__ rows,
                                                            const int64_t *__restrict__ slot0, int64_t nrows, int *keys,
                                                            double *acc, int *lc, double *lv, int64_t *cnt,
                                                            const int *crp, int *cci, double *cv, int *fail) {
  const int lane = threadIdx.x & 31;
  for (int64_t r = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; r < nrows;
       r += ((int64_t)gridDim.x * blockDim.x) >> 5) {
    const int i = rows[r];
    const int64_t b = slot0[r];
    const int cap = (int)(slot0[r + 1] - b);
    if (!amg_spgemm_accumulate(A, B, i, keys + b, acc + b, cap, lane, 32, WarpSync())) {   // cannot happen: cap >= 2 u
      if (lane == 0) *fail = 1;
      continue;
    }
    const int u = amg_table_compact(keys + b, acc + b, cap, lane, 32, lc + b, lv + b);
    __syncwarp();
    if (FILL) amg_spgemm_emit(lc + b, lv + b, u, lane, 32, cci + crp[i], cv + crp[i]);
    else if (lane == 0) cnt[i] = u;
    __syncwarp();
  }
}

// C = A B (A: m rows; B: ncols columns), Gustavson's order (amg_setup_core.h)
int spgemm(b200_ctx *ctx, const AmgRows &A, int64_t m, const AmgRows &B, int64_t ncols, DCsr *C) {
  cudaStream_t st = ctx->stream;
  C->m = m;
  C->n = ncols;
  Buf<int64_t> cnt;
  Buf<uint8_t> over;
  B200_TRY(cnt.alloc(m + 1));
  B200_TRY(over.alloc(m));
  B200_CUDA(cudaMemsetAsync(cnt.p, 0, sizeof(int64_t) * (size_t)(m + 1), st));
  B200_CUDA(cudaMemsetAsync(over.p, 0, (size_t)(m > 0 ? m : 1), st));
  const int chip_grid = stream_grid(ctx, m, kSgWarps, 4);
  if (m) {
    k_spgemm_chip<false><<<chip_grid, kSgWarps * 32, 0, st>>>(A, B, m, cnt.p, over.p, nullptr, nullptr, nullptr);
    B200_LAUNCH_CHECK(ctx);
  }
  // the rows that overflowed, in row order
  Buf<int> list, nsel;
  B200_TRY(list.alloc(m));
  B200_TRY(nsel.alloc(1));
  {
    size_t bytes = 0;
    cub::CountingInputIterator<int> it(0);
    B200_CUDA(cub::DeviceSelect::Flagged(nullptr, bytes, it, over.p, list.p, nsel.p, (int)m, st));
    Buf<char> tmp;
    B200_TRY(tmp.alloc((int64_t)bytes));
    B200_CUDA(cub::DeviceSelect::Flagged(tmp.p, bytes, it, over.p, list.p, nsel.p, (int)m, st));
    ctx->launches++;
  }
  int h_nsel = 0;
  B200_CUDA(cudaMemcpyAsync(&h_nsel, nsel.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  // their tables: 2 x min(products, ncols) slots rounded up to a power of two, in batches of at most kSgGlobalSlots
  std::vector<int64_t> slot0;             // per overflowed row, offsets restarting at 0 in each batch
  std::vector<int64_t> batch{0};          // batch b: overflowed rows [batch[b], batch[b+1])
  Buf<int64_t> d_slot0;
  Buf<int> gkeys, glc, fail;
  Buf<double> gacc, glv;
  if (h_nsel) {
    Buf<int64_t> prod;
    B200_TRY(prod.alloc(h_nsel));
    k_prod_count<<<grid(ctx, h_nsel), kThreads, 0, st>>>(A, B, list.p, h_nsel, prod.p);
    B200_LAUNCH_CHECK(ctx);
    std::vector<int64_t> hp((size_t)h_nsel);
    B200_CUDA(cudaMemcpyAsync(hp.data(), prod.p, sizeof(int64_t) * (size_t)h_nsel, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    // slot0: per batch, the starts of its rows' slots followed by the batch's end, so batch b's row r (overall index)
    // finds its slots at slot0[r + b] .. slot0[r + b + 1]
    int64_t used = 0, most = 0;
    for (int r = 0; r < h_nsel; ++r) {
      const int64_t u = std::min(hp[(size_t)r], ncols);
      int64_t cap = kSgGlobalMinCap;
      while (cap < 2 * u) cap <<= 1;
      if (cap > kSgGlobalSlots) {
        set_error("smoothed aggregation: a row of a Galerkin product has %lld distinct columns, more than the %lld "
                  "the setup's SpGEMM holds",
                  (long long)u, (long long)(kSgGlobalSlots / 2));
        return B200_ERR_UNSUPPORTED;
      }
      if (used + cap > kSgGlobalSlots) {
        slot0.push_back(used);
        batch.push_back(r);
        used = 0;
      }
      slot0.push_back(used);
      used += cap;
      most = std::max(most, used);
    }
    slot0.push_back(used);
    batch.push_back(h_nsel);
    B200_TRY(d_slot0.alloc((int64_t)slot0.size()));
    B200_CUDA(cudaMemcpyAsync(d_slot0.p, slot0.data(), sizeof(int64_t) * slot0.size(), cudaMemcpyHostToDevice, st));
    B200_TRY(gkeys.alloc(most));
    B200_TRY(glc.alloc(most));
    B200_TRY(gacc.alloc(most));
    B200_TRY(glv.alloc(most));
    B200_TRY(fail.alloc(1));
    B200_CUDA(cudaMemsetAsync(gkeys.p, 0xff, sizeof(int) * (size_t)most, st));
    B200_CUDA(cudaMemsetAsync(gacc.p, 0, sizeof(double) * (size_t)most, st));
    B200_CUDA(cudaMemsetAsync(fail.p, 0, sizeof(int), st));
  }
  auto run_global = [&](bool fill) -> int {
    for (size_t b = 0; b + 1 < batch.size(); ++b) {
      const int64_t r0 = batch[b], nr = batch[b + 1] - r0;
      const int g = stream_grid(ctx, nr, kThreads / 32, 8);
      const int64_t *s0 = d_slot0.p + r0 + (int64_t)b;   // this batch's starts and its end
      if (fill)
        k_spgemm_global<true><<<g, kThreads, 0, st>>>(A, B, list.p + r0, s0, nr, gkeys.p, gacc.p, glc.p, glv.p, nullptr,
                                                       C->rp.p, C->ci.p, C->v.p, fail.p);
      else
        k_spgemm_global<false><<<g, kThreads, 0, st>>>(A, B, list.p + r0, s0, nr, gkeys.p, gacc.p, glc.p, glv.p, cnt.p,
                                                        nullptr, nullptr, nullptr, fail.p);
      B200_LAUNCH_CHECK(ctx);
    }
    return B200_OK;
  };
  B200_TRY(run_global(false));
  B200_TRY(scan(ctx, cnt.p, m + 1));
  int64_t nnz = 0;
  B200_CUDA(cudaMemcpyAsync(&nnz, cnt.p + m, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  if (nnz >= (int64_t)INT32_MAX) {
    set_error("smoothed aggregation: a level of the hierarchy has %lld nonzeros; the setup holds int32 row offsets",
              (long long)nnz);
    return B200_ERR_UNSUPPORTED;
  }
  C->nnz = nnz;
  B200_TRY(C->rp.alloc(m + 1));
  B200_TRY(C->ci.alloc(nnz));
  B200_TRY(C->v.alloc(nnz));
  k_rowptr32<<<grid(ctx, m + 1), kThreads, 0, st>>>(cnt.p, m, C->rp.p);
  B200_LAUNCH_CHECK(ctx);
  if (m) {
    k_spgemm_chip<true><<<chip_grid, kSgWarps * 32, 0, st>>>(A, B, m, nullptr, over.p, C->rp.p, C->ci.p, C->v.p);
    B200_LAUNCH_CHECK(ctx);
  }
  B200_TRY(run_global(true));
  if (h_nsel) {
    int h_fail = 0;
    B200_CUDA(cudaMemcpyAsync(&h_fail, fail.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    B200_REQUIRE(!h_fail, "smoothed aggregation: internal error: a global SpGEMM table overflowed");
  }
  return B200_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// one level
struct LevelState {
  int64_t n = 0, nnz = 0;
  AmgRows A{};     // level 0: the caller's arrays (values converted to fp64 for Float32); else `own`
  DCsr own;
  Buf<double> vals64, d, B;
};

int download_csr(b200_ctx *ctx, const LevelState &L, AmgCsr *h) {
  cudaStream_t st = ctx->stream;
  h->m = h->n = L.n;
  std::vector<int> rp((size_t)L.n + 1);
  h->colind.resize((size_t)L.nnz);
  h->vals.resize((size_t)L.nnz);
  B200_CUDA(cudaMemcpyAsync(rp.data(), L.A.rp, sizeof(int) * (size_t)(L.n + 1), cudaMemcpyDeviceToHost, st));
  if (L.nnz) {
    B200_CUDA(cudaMemcpyAsync(h->colind.data(), L.A.ci, sizeof(int) * (size_t)L.nnz, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaMemcpyAsync(h->vals.data(), L.A.v, sizeof(double) * (size_t)L.nnz, cudaMemcpyDeviceToHost, st));
  }
  B200_CUDA(cudaStreamSynchronize(st));
  h->rowptr.assign(rp.begin(), rp.end());
  return B200_OK;
}

template <typename T>
int upload_inv(b200_ctx *ctx, const std::vector<double> &h, void **out) {
  std::vector<T> t(h.begin(), h.end());
  if (cudaMalloc(out, sizeof(T) * (t.size() ? t.size() : 1)) != cudaSuccess) {
    *out = nullptr;
    cudaGetLastError();
    set_error("b200_amg_create: cudaMalloc(%zu) failed", sizeof(T) * t.size());
    return B200_ERR_ALLOC;
  }
  if (!t.empty())
    B200_CUDA(cudaMemcpyAsync(*out, t.data(), sizeof(T) * t.size(), cudaMemcpyHostToDevice, ctx->stream));
  B200_CUDA(cudaStreamSynchronize(ctx->stream));
  return B200_OK;
}

// the diagonal of level L into L.d; 0 or row + 1 of the first row whose diagonal entry is missing or zero (and, when
// `sorted`, *unsorted = row + 1 of the first row whose columns are not ascending)
int check_level(b200_ctx *ctx, LevelState &L, bool sorted, int64_t *unsorted, int64_t *bad_diag) {
  cudaStream_t st = ctx->stream;
  Buf<int> bad;
  B200_TRY(bad.alloc(2));
  B200_TRY(L.d.alloc(L.n));
  k_fill<int><<<1, 32, 0, st>>>(bad.p, 2, INT_MAX);
  B200_LAUNCH_CHECK(ctx);
  k_checks<<<grid(ctx, L.n), kThreads, 0, st>>>(L.A, L.n, sorted ? 1 : 0, bad.p, L.d.p);
  B200_LAUNCH_CHECK(ctx);
  int h[2];
  B200_CUDA(cudaMemcpyAsync(h, bad.p, sizeof(h), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  if (unsorted) *unsorted = h[0] == INT_MAX ? 0 : (int64_t)h[0] + 1;
  *bad_diag = h[1] == INT_MAX ? 0 : (int64_t)h[1] + 1;
  return B200_OK;
}

int zero_diagonal(int level, int64_t row) {
  set_error("smoothed aggregation: zero or missing diagonal entry in row %lld (0-based) of level %d", (long long)row,
            level);
  return B200_ERR_BREAKDOWN;
}

// strength and the three passes: *x = the aggregates, *naggs their number, *pass1 the launches pass 1 took
int aggregate(b200_ctx *ctx, const LevelState &L, double theta, DCsr *S, Buf<int> *x, int64_t *naggs, int *pass1) {
  cudaStream_t st = ctx->stream;
  const int64_t n = L.n;
  S->m = S->n = n;
  B200_TRY(S->rp.alloc(n + 1));
  B200_CUDA(cudaMemsetAsync(S->rp.p, 0, sizeof(int) * (size_t)(n + 1), st));
  k_strength<<<grid(ctx, n), kThreads, 0, st>>>(L.A, L.d.p, n, theta, S->rp.p, nullptr, nullptr);
  B200_LAUNCH_CHECK(ctx);
  B200_TRY(scan(ctx, S->rp.p, n + 1));
  int snnz = 0;
  B200_CUDA(cudaMemcpyAsync(&snnz, S->rp.p + n, sizeof(int), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  S->nnz = snnz;
  B200_TRY(S->ci.alloc(snnz));
  k_strength<<<grid(ctx, n), kThreads, 0, st>>>(L.A, L.d.p, n, theta, nullptr, S->rp.p, S->ci.p);
  B200_LAUNCH_CHECK(ctx);
  DCsr St;
  B200_TRY(transpose(ctx, S->rows(), n, n, snnz, &St));
  // pass 1
  Buf<int> state, id, misc;
  Buf<unsigned> ticket;
  B200_TRY(state.alloc(n));
  B200_TRY(id.alloc(n + 1));
  B200_TRY(misc.alloc(2));   // [0]: rows left undecided; [1]: the number of aggregates
  B200_TRY(ticket.alloc(1));
  k_pass1_init<<<grid(ctx, n), kThreads, 0, st>>>(S->rows(), n, state.p);
  B200_LAUNCH_CHECK(ctx);
  *pass1 = 0;
  for (int left = 1; left && n; ++*pass1) {
    B200_CUDA(cudaMemsetAsync(ticket.p, 0, sizeof(unsigned), st));
    B200_CUDA(cudaMemsetAsync(misc.p, 0, sizeof(int), st));
    k_pass1<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, st>>>(S->rows(), St.rows(), n, state.p, ticket.p,
                                                                            misc.p);
    B200_LAUNCH_CHECK(ctx);
    B200_CUDA(cudaMemcpyAsync(&left, misc.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
  }
  St.reset();
  B200_CUDA(cudaMemsetAsync(id.p + n, 0, sizeof(int), st));
  k_root_flags<<<grid(ctx, n), kThreads, 0, st>>>(state.p, n, id.p);
  B200_LAUNCH_CHECK(ctx);
  B200_TRY(scan(ctx, id.p, n + 1));
  Buf<int> x1;
  B200_TRY(x1.alloc(n));
  B200_TRY(x->alloc(n));
  k_fill<int><<<grid(ctx, n), kThreads, 0, st>>>(x1.p, n, kFree);
  B200_LAUNCH_CHECK(ctx);
  k_root_scatter<<<grid(ctx, n), kThreads, 0, st>>>(S->rows(), state.p, id.p, n, x1.p);
  B200_LAUNCH_CHECK(ctx);
  k_isolated<<<grid(ctx, n), kThreads, 0, st>>>(S->rows(), n, x1.p);
  B200_LAUNCH_CHECK(ctx);
  // pass 2, pass 3
  k_pass2<<<grid(ctx, n), kThreads, 0, st>>>(S->rows(), n, x1.p, x->p);
  B200_LAUNCH_CHECK(ctx);
  Buf<uint8_t> flags;
  B200_TRY(flags.alloc(n));
  k_free_flags<<<grid(ctx, n), kThreads, 0, st>>>(x->p, n, flags.p);
  B200_LAUNCH_CHECK(ctx);
  {
    size_t bytes = 0;
    cub::CountingInputIterator<int> it(0);
    B200_CUDA(cub::DeviceSelect::Flagged(nullptr, bytes, it, flags.p, x1.p, misc.p, (int)n, st));
    Buf<char> tmp;
    B200_TRY(tmp.alloc((int64_t)bytes));
    B200_CUDA(cub::DeviceSelect::Flagged(tmp.p, bytes, it, flags.p, x1.p, misc.p, (int)n, st));   // x1: the free rows
    ctx->launches++;
  }
  B200_CUDA(cudaMemcpyAsync(misc.p + 1, id.p + n, sizeof(int), cudaMemcpyDeviceToDevice, st));
  k_pass3<<<1, 1, 0, st>>>(S->rows(), x1.p, misc.p, x->p, misc.p + 1);
  B200_LAUNCH_CHECK(ctx);
  int h = 0;
  B200_CUDA(cudaMemcpyAsync(&h, misc.p + 1, sizeof(int), cudaMemcpyDeviceToHost, st));
  B200_CUDA(cudaStreamSynchronize(st));
  *naggs = h;
  return B200_OK;
}

}  // namespace

namespace b200 {

template <typename T>
int amg_device_setup(b200_ctx *ctx, const b200_csr *A0, const AmgOptions &o, std::vector<AmgDevLevel> *levels,
                     std::vector<int64_t> *nnz_P, double *seconds) {
  cudaStream_t st = ctx->stream;
  const int dtype = sizeof(T) == 8 ? B200_F64 : B200_F32;
  for (int k = 0; k < 5; ++k) seconds[k] = 0.0;
  double t0 = now_s();
  LevelState L;
  L.n = A0->m_local;
  L.nnz = A0->nnz;
  if (sizeof(T) == 8) {
    L.A = AmgRows{A0->rowptr, A0->colind, (const double *)A0->vals};
  } else {
    B200_TRY(L.vals64.alloc(L.nnz));
    k_to_f64<float><<<grid(ctx, L.nnz), kThreads, 0, st>>>((const float *)A0->vals, L.nnz, L.vals64.p);
    B200_LAUNCH_CHECK(ctx);
    L.A = AmgRows{A0->rowptr, A0->colind, L.vals64.p};
  }
  int64_t unsorted = 0, bad = 0;
  B200_TRY(check_level(ctx, L, true, &unsorted, &bad));
  B200_REQUIRE(!unsorted, "AMG needs rows with ascending column indices (row %lld)", (long long)(unsorted - 1));
  if (bad) return zero_diagonal(0, bad - 1);
  B200_TRY(L.B.alloc(L.n));
  k_fill<double><<<grid(ctx, L.n), kThreads, 0, st>>>(L.B.p, L.n, 1.0);
  B200_LAUNCH_CHECK(ctx);
  B200_CUDA(cudaStreamSynchronize(st));
  seconds[0] = now_s() - t0;
  auto build_A = [&](AmgDevLevel &D, int l) -> int {   // level l's operator (l > 0)
    const double ta = now_s();
    b200_csr *Al = nullptr;
    B200_TRY(csr_from_device_f64(ctx, L.n, L.n, L.nnz, L.A.rp, L.A.ci, L.A.v, dtype, &Al));
    D.A = Al;
    seconds[4] += now_s() - ta;
    return B200_OK;
  };
  while (L.n > o.max_coarse && (int)levels->size() + 1 < o.max_levels) {
    const int l = (int)levels->size();
    t0 = now_s();
    if (l > 0) {
      B200_TRY(check_level(ctx, L, false, nullptr, &bad));
      if (bad) return zero_diagonal(l, bad - 1);
    }
    DCsr S;
    Buf<int> x;
    int64_t naggs = 0;
    int pass1 = 0;
    B200_TRY(aggregate(ctx, L, o.theta, &S, &x, &naggs, &pass1));
    S.reset();
    double t1 = now_s();
    seconds[1] += t1 - t0;
    if (naggs == 0) break;   // every row isolated: this level is the coarsest
    const int64_t n = L.n;
    // T and B_c
    DCsr Tm;
    Buf<double> Bc;
    {
      Buf<unsigned> key, kout;
      Buf<int> rows, sorted;
      Tm.m = n;
      Tm.n = naggs;
      B200_TRY(Tm.rp.alloc(n + 1));
      B200_TRY(Bc.alloc(naggs));
      B200_TRY(key.alloc(n));
      B200_TRY(kout.alloc(n));
      B200_TRY(rows.alloc(n));
      B200_TRY(sorted.alloc(n));
      B200_CUDA(cudaMemsetAsync(Tm.rp.p, 0, sizeof(int) * (size_t)(n + 1), st));
      k_agg_keys<<<grid(ctx, n), kThreads, 0, st>>>(x.p, n, key.p, Tm.rp.p);   // Tm.rp: members per aggregate
      B200_LAUNCH_CHECK(ctx);
      B200_TRY(scan(ctx, Tm.rp.p, naggs + 1));
      k_iota<<<grid(ctx, n), kThreads, 0, st>>>(rows.p, n);
      B200_LAUNCH_CHECK(ctx);
      B200_TRY(sort_pairs(ctx, key.p, kout.p, rows.p, sorted.p, n, end_bit_for(naggs + 1)));
      k_bc<<<grid(ctx, naggs), kThreads, 0, st>>>(Tm.rp.p, sorted.p, L.B.p, naggs, n, Bc.p);
      B200_LAUNCH_CHECK(ctx);
      B200_CUDA(cudaMemsetAsync(Tm.rp.p + n, 0, sizeof(int), st));
      k_t_flags<<<grid(ctx, n), kThreads, 0, st>>>(x.p, n, Tm.rp.p);
      B200_LAUNCH_CHECK(ctx);
      B200_TRY(scan(ctx, Tm.rp.p, n + 1));
      int tnnz = 0;
      B200_CUDA(cudaMemcpyAsync(&tnnz, Tm.rp.p + n, sizeof(int), cudaMemcpyDeviceToHost, st));
      B200_CUDA(cudaStreamSynchronize(st));
      Tm.nnz = tnnz;
      B200_TRY(Tm.ci.alloc(tnnz));
      B200_TRY(Tm.v.alloc(tnnz));
      k_t_fill<<<grid(ctx, n), kThreads, 0, st>>>(x.p, L.B.p, Bc.p, Tm.rp.p, n, Tm.ci.p, Tm.v.p);
      B200_LAUNCH_CHECK(ctx);
    }
    // rho, w, P
    Buf<unsigned long long> rbits;
    B200_TRY(rbits.alloc(1));
    B200_CUDA(cudaMemsetAsync(rbits.p, 0, sizeof(unsigned long long), st));
    k_rho<<<grid(ctx, n), kThreads, 0, st>>>(L.A, L.d.p, n, rbits.p);
    B200_LAUNCH_CHECK(ctx);
    unsigned long long hb = 0;
    B200_CUDA(cudaMemcpyAsync(&hb, rbits.p, sizeof(hb), cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    double rho;
    memcpy(&rho, &hb, sizeof(rho));
    const double c = (4.0 / 3.0) / rho;
    levels->emplace_back();
    AmgDevLevel &D = levels->back();
    D.n = n;
    D.pass1_launches = pass1;
    {
      void *w = nullptr;
      if (cudaMalloc(&w, sizeof(T) * (size_t)(n > 0 ? n : 1)) != cudaSuccess) {
        cudaGetLastError();
        set_error("b200_amg_create: cudaMalloc(%zu) failed", sizeof(T) * (size_t)n);
        return B200_ERR_ALLOC;
      }
      D.w = w;
    }
    k_weights<T><<<grid(ctx, n), kThreads, 0, st>>>(L.d.p, c, n, (T *)D.w);
    B200_LAUNCH_CHECK(ctx);
    DCsr P;
    {
      DCsr AT;
      B200_TRY(spgemm(ctx, L.A, n, Tm.rows(), naggs, &AT));
      Buf<int64_t> cnt;
      B200_TRY(cnt.alloc(n + 1));
      B200_CUDA(cudaMemsetAsync(cnt.p + n, 0, sizeof(int64_t), st));
      k_p_merge<<<grid(ctx, n), kThreads, 0, st>>>(Tm.rows(), AT.rows(), L.d.p, c, n, cnt.p, nullptr, nullptr, nullptr);
      B200_LAUNCH_CHECK(ctx);
      B200_TRY(scan(ctx, cnt.p, n + 1));
      int64_t pnnz = 0;
      B200_CUDA(cudaMemcpyAsync(&pnnz, cnt.p + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
      B200_CUDA(cudaStreamSynchronize(st));
      P.m = n;
      P.n = naggs;
      P.nnz = pnnz;
      B200_TRY(P.rp.alloc(n + 1));
      B200_TRY(P.ci.alloc(pnnz));
      B200_TRY(P.v.alloc(pnnz));
      k_rowptr32<<<grid(ctx, n + 1), kThreads, 0, st>>>(cnt.p, n, P.rp.p);
      B200_LAUNCH_CHECK(ctx);
      k_p_merge<<<grid(ctx, n), kThreads, 0, st>>>(Tm.rows(), AT.rows(), L.d.p, c, n, nullptr, P.rp.p, P.ci.p, P.v.p);
      B200_LAUNCH_CHECK(ctx);
      B200_CUDA(cudaStreamSynchronize(st));
    }
    Tm.reset();
    t0 = now_s();
    seconds[2] += t0 - t1;
    // R = P', A_c = R (A P)
    DCsr Ac;
    {
      DCsr R, AP;
      B200_TRY(transpose(ctx, P.rows(), n, naggs, P.nnz, &R));
      B200_TRY(spgemm(ctx, L.A, n, P.rows(), naggs, &AP));
      B200_TRY(spgemm(ctx, R.rows(), naggs, AP.rows(), naggs, &Ac));
      B200_CUDA(cudaStreamSynchronize(st));
    }
    t1 = now_s();
    seconds[3] += t1 - t0;
    // the level's operators and aggregates
    if (l > 0) B200_TRY(build_A(D, l));
    B200_TRY(csr_from_device_f64(ctx, n, naggs, P.nnz, P.rp.p, P.ci.p, P.v.p, dtype, &D.P));
    B200_TRY(b200_csr_transpose(ctx, D.P, &D.R));
    nnz_P->push_back(P.nnz);
    D.agg.resize((size_t)n);
    B200_CUDA(cudaMemcpyAsync(D.agg.data(), x.p, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, st));
    B200_CUDA(cudaStreamSynchronize(st));
    seconds[4] += now_s() - t1;
    // the next level
    L.own.swap(Ac);
    L.vals64.reset();
    L.n = naggs;
    L.nnz = L.own.nnz;
    L.A = L.own.rows();
    L.B.swap(Bc);
  }
  // the coarsest level
  t0 = now_s();
  const int lc = (int)levels->size();
  if (L.n > kAmgMaxCoarsest) {
    set_error("smoothed aggregation: the coarsest level (level %d) has %lld rows, more than the %d its dense inverse "
              "allows; raise max_levels or lower max_coarse",
              lc, (long long)L.n, kAmgMaxCoarsest);
    return B200_ERR_INVALID;
  }
  AmgCsr h;
  B200_TRY(download_csr(ctx, L, &h));
  std::vector<double> inv;
  if (const int64_t zp = amg_dense_inverse(h, &inv)) {
    set_error("smoothed aggregation: the coarsest level (level %d) is singular: zero pivot in column %lld (0-based)", lc,
              (long long)(zp - 1));
    return B200_ERR_BREAKDOWN;
  }
  levels->emplace_back();
  AmgDevLevel &D = levels->back();
  D.n = L.n;
  B200_TRY(upload_inv<T>(ctx, inv, &D.inv));
  seconds[3] += now_s() - t0;
  if (lc > 0) B200_TRY(build_A(D, lc));
  return B200_OK;
}

template int amg_device_setup<double>(b200_ctx *, const b200_csr *, const AmgOptions &, std::vector<AmgDevLevel> *,
                                      std::vector<int64_t> *, double *);
template int amg_device_setup<float>(b200_ctx *, const b200_csr *, const AmgOptions &, std::vector<AmgDevLevel> *,
                                     std::vector<int64_t> *, double *);

}  // namespace b200
