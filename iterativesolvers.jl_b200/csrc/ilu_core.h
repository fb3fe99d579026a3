// ilu_core.h -- zero-fill incomplete LU, ILU(0) (Saad, Iterative Methods for Sparse Linear Systems, 2nd ed., Algorithm
// 10.4, IKJ order), the preconditioner the reference's docs/src/preconditioning.md points to (IncompleteLU.jl).  Beyond
// SURVEY section 8; single GPU, real element types.
//
// The factor keeps A's sparsity pattern: L (unit diagonal, not stored) and U share one value array in A's CSR order, so
// the factor reuses A's rowptr / colind.  Three row functions, each written once for the host and the device:
//   factor row i     for each k < i in row i, ascending:  a_ik <- a_ik / a_kk;
//                                                         a_ij <- a_ij - a_ik a_kj  for every j > k in rows i AND k
//   forward row i    y_i <- x_i - sum_{j < i, ascending} l_ij y_j
//   backward row i   z_i <- (y_i - sum_{j > i, ascending} u_ij z_j) / u_ii
// Every product and difference is rounded on its own (mul_rn / sub_rn of complex.h: no contraction on the device; the
// host test build uses -ffp-contract=off), so the serial host run and the GPU give the same bits.
//
// Row i of the factorization and of the forward solve waits for the rows of its strictly lower part; row i of the
// backward solve for the rows of its strictly upper part: the dependency graphs of the forward and backward sweeps of
// the stationary methods, whose level analysis (stationary_analyse) is reused.  The levels are cut into chunks of up to
// 32 consecutive rows of one level (one warp, one lane per row, on the device: ilu.cu).  A row function gets a `wait`
// functor that it calls with each dependency before reading that row's value; wait returns false when the value never
// became ready (the device's bounded spin, or a dependency outside the earlier chunks in the host's checked run).
#pragma once
#include <algorithm>
#include <vector>

#include "stationary_core.h"

namespace b200 {

constexpr int kIluChunkRows = 32;

enum { ILU_OK = 0, ILU_NOT_READY = 1, ILU_ZERO_PIVOT = 2 };

// the factor: A's pattern (rows with ascending column indices), dpos[i] = position of the diagonal within row i, f = the
// factor values in A's CSR order (strictly lower part: L without its unit diagonal; the rest: U)
template <typename T, typename RP>
struct IluView {
  const RP *rowptr;
  const int *colind;
  const int *dpos;
  T *f;
};

// one row of ILU(0) in IKJ order, in place on f; ILU_ZERO_PIVOT when u_ii ends up zero
template <typename T, typename RP, typename W>
B200_HD int ilu_factor_row(const IluView<T, RP> &v, int64_t i, W &wait) {
  const RP r0 = v.rowptr[i], r1 = v.rowptr[i + 1], d = r0 + v.dpos[i];
  for (RP p = r0; p < d; ++p) {
    const int k = v.colind[p];
    if (!wait(k)) return ILU_NOT_READY;
    const RP kd = v.rowptr[k] + v.dpos[k], k1 = v.rowptr[k + 1];
    const T lik = v.f[p] / v.f[kd];
    v.f[p] = lik;
    // merge the part of row i right of k with the part of row k right of its diagonal (both ascending)
    RP q = kd + 1;
    for (RP s = p + 1; s < r1 && q < k1; ++s) {
      const int j = v.colind[s];
      while (q < k1 && v.colind[q] < j) ++q;
      if (q < k1 && v.colind[q] == j) v.f[s] = sub_rn(v.f[s], mul_rn(lik, v.f[q]));
    }
  }
  return v.f[d] == (T)0 ? ILU_ZERO_PIVOT : ILU_OK;
}

// y_i = x_i - sum_{j<i} l_ij y_j.  x may be y (row i reads x_i before anything writes y_i, and no other row reads x_i)
template <typename T, typename RP, typename W>
B200_HD int ilu_forward_row(const IluView<T, RP> &v, int64_t i, const T *x, T *y, W &wait) {
  const RP r0 = v.rowptr[i], d = r0 + v.dpos[i];
  T acc = x[i];
  for (RP p = r0; p < d; ++p) {
    const int j = v.colind[p];
    if (!wait(j)) return ILU_NOT_READY;
    acc = sub_rn(acc, mul_rn(v.f[p], y[j]));
  }
  y[i] = acc;
  return ILU_OK;
}

// z_i = (y_i - sum_{j>i} u_ij z_j) / u_ii.  y may be z (same argument as above)
template <typename T, typename RP, typename W>
B200_HD int ilu_backward_row(const IluView<T, RP> &v, int64_t i, const T *y, T *z, W &wait) {
  const RP d = v.rowptr[i] + v.dpos[i], r1 = v.rowptr[i + 1];
  T acc = y[i];
  for (RP p = d + 1; p < r1; ++p) {
    const int j = v.colind[p];
    if (!wait(j)) return ILU_NOT_READY;
    acc = sub_rn(acc, mul_rn(v.f[p], z[j]));
  }
  z[i] = acc / v.f[d];
  return ILU_OK;
}

// The chunk schedule of one sweep: chunk c owns rows[cptr[c] .. cptr[c+1]), up to kIluChunkRows consecutive rows of one
// level; chunks are in level order, so every dependency of a chunk's rows lies in an earlier chunk.
struct IluSchedule {
  std::vector<int> rows;
  std::vector<int> cptr;
  int levels = 0;
  int64_t chunks() const { return (int64_t)cptr.size() - 1; }
};
inline void ilu_chunks(const std::vector<int> &rows, const std::vector<int64_t> &lptr, IluSchedule *out) {
  out->rows = rows;
  out->levels = (int)lptr.size() - 1;
  out->cptr.assign(1, 0);
  for (size_t l = 0; l + 1 < lptr.size(); ++l)
    for (int64_t b = lptr[l]; b < lptr[l + 1]; b += kIluChunkRows)
      out->cptr.push_back((int)std::min<int64_t>(b + kIluChunkRows, lptr[l + 1]));
}

// The host analysis of A: diagonal positions and the forward / backward chunk schedules.  Returns 0, or row + 1 of the
// first row with a missing or zero diagonal entry (stationary_analyse).
template <typename T, typename RP>
int64_t ilu_analyse(int64_t n, const RP *rowptr, const int *colind, const T *vals, std::vector<int> *dpos,
                    IluSchedule *fwd, IluSchedule *bwd) {
  StLevels lv;
  const int64_t singular = stationary_analyse<T, RP>(n, rowptr, colind, vals, true, true, &lv);
  if (singular) return singular;
  ilu_chunks(lv.rows_f, lv.lptr_f, fwd);
  ilu_chunks(lv.rows_b, lv.lptr_b, bwd);
  *dpos = std::move(lv.dpos);
  return 0;
}

// Serial run of a sweep over its chunk schedule: row(i, wait) for the rows of each chunk in turn; a row's value counts as
// ready only once its whole chunk is done, so a dependency inside the same or a later chunk is reported (ILU_NOT_READY,
// *bad = that row) instead of read.  A zero pivot does not stop the sweep, as on the device: every row is factored and
// *bad = the smallest row with a zero pivot (the first one in row order; rows before it are exact).
template <typename F>
int ilu_run_serial(const IluSchedule &s, int64_t n, F &&row, int64_t *bad) {
  std::vector<char> ready((size_t)n, 0);
  auto wait = [&](int j) { return ready[(size_t)j] != 0; };
  int status = ILU_OK;
  for (int64_t c = 0; c < s.chunks(); ++c) {
    for (int p = s.cptr[(size_t)c]; p < s.cptr[(size_t)c + 1]; ++p) {
      const int i = s.rows[(size_t)p];
      const int st = row((int64_t)i, wait);
      if (st == ILU_NOT_READY) {
        *bad = i;
        return st;
      }
      if (st == ILU_ZERO_PIVOT && (status == ILU_OK || i < *bad)) {
        status = st;
        *bad = i;
      }
    }
    for (int p = s.cptr[(size_t)c]; p < s.cptr[(size_t)c + 1]; ++p) ready[(size_t)s.rows[(size_t)p]] = 1;
  }
  return status;
}

}  // namespace b200
