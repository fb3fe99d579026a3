// amg_core.h -- the setup of the smoothed-aggregation AMG preconditioner (DESIGN section 23) and a serial V-cycle,
// host C++ only.  amg_setup is the serial reference: the library builds the same hierarchy, bit for bit, on the device
// (amg_setup.cu) and calls only amg_dense_inverse from here, for the coarsest level; the CPU tests (tests/hostsim_amg)
// run amg_setup and the serial V-cycle.  Beyond SURVEY section 8; single GPU, real element types.
//
// The setup is AlgebraicMultigrid.jl's / pyamg's smoothed_aggregation with one candidate (B = ones), in fp64:
//   strength      SymmetricStrength(theta): off-diagonal a_ij is strong when |a_ij| >= theta sqrt(|a_ii a_jj|)
//   aggregation   the three passes of standard_aggregation, in row order; ids in creation order; a row with no strong
//                 off-diagonal neighbour is isolated (aggregate -1, zero row of T)
//   T             fit_candidates: T[i, J] = B[i] / ||B|_J||, coarse candidate B_c[J] = ||B|_J||
//   P             JacobiProlongation(4/3): P = (I - (4/3) / rho D^-1 A) T, rho = max_i sum_j |a_ij| / |a_ii| (Gershgorin;
//                 AMG.jl / pyamg estimate rho with randomised Arnoldi: the deterministic bound is deviation 1)
//   R, A_c        R = P', A_c = R (A P) (Gustavson SpGEMM, columns ascending in every row)
//   coarsest      the explicit inverse, Gauss-Jordan with partial pivoting (AMG.jl's default coarse solver is Pinv)
// Sums that cancel to exactly 0 are dropped from the patterns of P and A_c, as scipy's sparse products do.  The smoother is
// weighted Jacobi, omega_s = (4/3) / rho per level (deviation 2: AMG.jl / pyamg use Gauss-Seidel, which on the GPU is the
// same level-scheduled chain that makes ILU(0) slow).
#pragma once
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <vector>

namespace b200 {

constexpr int kAmgMaxCoarsest = 4096;   // rows of the coarsest level, whose dense inverse the device applies

struct AmgCsr {   // host CSR, fp64, 0-based, columns strictly ascending in every row
  int64_t m = 0, n = 0;
  std::vector<int64_t> rowptr{0};
  std::vector<int> colind;
  std::vector<double> vals;
  int64_t nnz() const { return rowptr.back(); }
};

struct AmgOptions {
  double theta = 0.0;
  int max_levels = 10, max_coarse = 10, presweeps = 1, postsweeps = 1;
};

struct AmgLevel {
  AmgCsr A;
  AmgCsr P, R;               // empty on the coarsest level
  std::vector<int> agg;      // aggregate of every row, -1 = isolated (not on the coarsest level)
  std::vector<double> w;     // smoother weights omega_s / a_ii (not on the coarsest level)
  std::vector<double> inv;   // coarsest level only: A^-1, row-major
};

enum { AMG_OK = 0, AMG_ZERO_DIAGONAL = 1, AMG_ZERO_PIVOT = 2, AMG_TOO_LARGE = 3 };

struct AmgStatus {
  int code = AMG_OK;
  int level = 0;     // the level of a zero diagonal / pivot
  int64_t row = 0;   // its row (0-based)
};

// the diagonal of A; 0 or row + 1 of the first row whose diagonal entry is missing or zero
inline int64_t amg_diagonal(const AmgCsr &A, std::vector<double> *d) {
  d->assign((size_t)A.m, 0.0);
  for (int64_t i = 0; i < A.m; ++i) {
    for (int64_t p = A.rowptr[(size_t)i]; p < A.rowptr[(size_t)i + 1]; ++p)
      if (A.colind[(size_t)p] == i) (*d)[(size_t)i] = A.vals[(size_t)p];
    if ((*d)[(size_t)i] == 0.0) return i + 1;
  }
  return 0;
}

// the strong off-diagonal pattern of A (SymmetricStrength(theta)); vals unused
inline AmgCsr amg_strength(const AmgCsr &A, const std::vector<double> &d, double theta) {
  AmgCsr S;
  S.m = A.m;
  S.n = A.n;
  S.rowptr.assign((size_t)A.m + 1, 0);
  for (int64_t i = 0; i < A.m; ++i) {
    for (int64_t p = A.rowptr[(size_t)i]; p < A.rowptr[(size_t)i + 1]; ++p) {
      const int j = A.colind[(size_t)p];
      if (j != i && std::fabs(A.vals[(size_t)p]) >= theta * std::sqrt(std::fabs(d[(size_t)i] * d[(size_t)j])))
        S.colind.push_back(j);
    }
    S.rowptr[(size_t)i + 1] = (int64_t)S.colind.size();
  }
  return S;
}

// standard_aggregation's three passes over the strong pattern S (no diagonal entries); returns the number of aggregates
inline int amg_aggregate(const AmgCsr &S, std::vector<int> *agg) {
  const int64_t n = S.m;
  const int kFree = -2, kIsolated = -1;
  std::vector<int> &x = *agg;
  x.assign((size_t)n, kFree);
  int next = 0;
  auto nbrs = [&](int64_t i, auto &&f) {
    for (int64_t p = S.rowptr[(size_t)i]; p < S.rowptr[(size_t)i + 1]; ++p)
      if (!f(S.colind[(size_t)p])) return false;
    return true;
  };
  // pass 1: a free node none of whose strong neighbours is taken starts an aggregate with all of them
  for (int64_t i = 0; i < n; ++i) {
    if (x[(size_t)i] != kFree) continue;
    if (S.rowptr[(size_t)i] == S.rowptr[(size_t)i + 1]) {
      x[(size_t)i] = kIsolated;
      continue;
    }
    if (!nbrs(i, [&](int j) { return x[(size_t)j] == kFree; })) continue;
    x[(size_t)i] = next;
    nbrs(i, [&](int j) { x[(size_t)j] = next; return true; });
    ++next;
  }
  // pass 2: a free node joins the pass-1 aggregate of its first strong neighbour (column order) that has one; nodes
  // joining in this pass do not pass their aggregate on
  std::vector<int> joined((size_t)n, kFree);
  for (int64_t i = 0; i < n; ++i) {
    if (x[(size_t)i] != kFree) continue;
    nbrs(i, [&](int j) {
      const int a = x[(size_t)j];
      if (a >= 0) {
        joined[(size_t)i] = a;
        return false;
      }
      return true;
    });
  }
  for (int64_t i = 0; i < n; ++i)
    if (joined[(size_t)i] != kFree) x[(size_t)i] = joined[(size_t)i];
  // pass 3: a node still free starts an aggregate with its still-free strong neighbours
  for (int64_t i = 0; i < n; ++i) {
    if (x[(size_t)i] != kFree) continue;
    x[(size_t)i] = next;
    nbrs(i, [&](int j) {
      if (x[(size_t)j] == kFree) x[(size_t)j] = next;
      return true;
    });
    ++next;
  }
  return next;
}

// fit_candidates with one candidate: T (n x naggs, one entry per aggregated row) and the coarse candidate Bc
inline AmgCsr amg_tentative(const std::vector<int> &agg, int naggs, const std::vector<double> &B, std::vector<double> *Bc) {
  const int64_t n = (int64_t)agg.size();
  Bc->assign((size_t)naggs, 0.0);
  for (int64_t i = 0; i < n; ++i)
    if (agg[(size_t)i] >= 0) (*Bc)[(size_t)agg[(size_t)i]] += B[(size_t)i] * B[(size_t)i];
  for (double &v : *Bc) v = std::sqrt(v);
  AmgCsr T;
  T.m = n;
  T.n = naggs;
  T.rowptr.assign((size_t)n + 1, 0);
  for (int64_t i = 0; i < n; ++i) {
    const int a = agg[(size_t)i];
    if (a >= 0) {
      T.colind.push_back(a);
      T.vals.push_back(B[(size_t)i] / (*Bc)[(size_t)a]);
    }
    T.rowptr[(size_t)i + 1] = (int64_t)T.colind.size();
  }
  return T;
}

// Gustavson's C = A B: each row accumulated in a dense scratch row, columns sorted ascending, exact zeros dropped
inline AmgCsr amg_spgemm(const AmgCsr &A, const AmgCsr &B) {
  AmgCsr C;
  C.m = A.m;
  C.n = B.n;
  C.rowptr.assign((size_t)A.m + 1, 0);
  std::vector<double> acc((size_t)B.n, 0.0);
  std::vector<char> used((size_t)B.n, 0);
  std::vector<int> cols;
  for (int64_t i = 0; i < A.m; ++i) {
    cols.clear();
    for (int64_t p = A.rowptr[(size_t)i]; p < A.rowptr[(size_t)i + 1]; ++p) {
      const int k = A.colind[(size_t)p];
      const double a = A.vals[(size_t)p];
      for (int64_t q = B.rowptr[(size_t)k]; q < B.rowptr[(size_t)k + 1]; ++q) {
        const int j = B.colind[(size_t)q];
        if (!used[(size_t)j]) {
          used[(size_t)j] = 1;
          cols.push_back(j);
        }
        acc[(size_t)j] += a * B.vals[(size_t)q];
      }
    }
    std::sort(cols.begin(), cols.end());
    for (int j : cols) {
      if (acc[(size_t)j] != 0.0) {
        C.colind.push_back(j);
        C.vals.push_back(acc[(size_t)j]);
      }
      acc[(size_t)j] = 0.0;
      used[(size_t)j] = 0;
    }
    C.rowptr[(size_t)i + 1] = (int64_t)C.colind.size();
  }
  return C;
}

inline AmgCsr amg_transpose(const AmgCsr &A) {
  AmgCsr T;
  T.m = A.n;
  T.n = A.m;
  T.rowptr.assign((size_t)A.n + 1, 0);
  for (int64_t p = 0; p < A.nnz(); ++p) ++T.rowptr[(size_t)A.colind[(size_t)p] + 1];
  for (int64_t j = 0; j < A.n; ++j) T.rowptr[(size_t)j + 1] += T.rowptr[(size_t)j];
  T.colind.resize((size_t)A.nnz());
  T.vals.resize((size_t)A.nnz());
  std::vector<int64_t> next(T.rowptr.begin(), T.rowptr.end() - 1);
  for (int64_t i = 0; i < A.m; ++i)   // rows ascending: the columns of T come out ascending
    for (int64_t p = A.rowptr[(size_t)i]; p < A.rowptr[(size_t)i + 1]; ++p) {
      const int64_t q = next[(size_t)A.colind[(size_t)p]]++;
      T.colind[(size_t)q] = (int)i;
      T.vals[(size_t)q] = A.vals[(size_t)p];
    }
  return T;
}

// P = T - ((4/3) / rho) D^-1 (A T): row i of T merged with the scaled row i of A T, exact zeros dropped
inline AmgCsr amg_prolongator(const AmgCsr &A, const std::vector<double> &d, const AmgCsr &T, double rho) {
  const double c = (4.0 / 3.0) / rho;
  const AmgCsr AT = amg_spgemm(A, T);
  AmgCsr P;
  P.m = T.m;
  P.n = T.n;
  P.rowptr.assign((size_t)T.m + 1, 0);
  for (int64_t i = 0; i < T.m; ++i) {
    int64_t p = T.rowptr[(size_t)i], q = AT.rowptr[(size_t)i];
    const int64_t p1 = T.rowptr[(size_t)i + 1], q1 = AT.rowptr[(size_t)i + 1];
    const double s = 1.0 / d[(size_t)i];
    while (p < p1 || q < q1) {
      const int jp = p < p1 ? T.colind[(size_t)p] : INT32_MAX, jq = q < q1 ? AT.colind[(size_t)q] : INT32_MAX;
      const int j = std::min(jp, jq);
      const double t = jp == j ? T.vals[(size_t)p++] : 0.0;
      const double v = jq == j ? t - c * (AT.vals[(size_t)q++] * s) : t;
      if (v != 0.0) {
        P.colind.push_back(j);
        P.vals.push_back(v);
      }
    }
    P.rowptr[(size_t)i + 1] = (int64_t)P.colind.size();
  }
  return P;
}

// max_i sum_j |a_ij| / |a_ii|: the Gershgorin bound on the spectral radius of D^-1 A
inline double amg_rho(const AmgCsr &A, const std::vector<double> &d) {
  double rho = 0.0;
  for (int64_t i = 0; i < A.m; ++i) {
    double s = 0.0;
    for (int64_t p = A.rowptr[(size_t)i]; p < A.rowptr[(size_t)i + 1]; ++p) s += std::fabs(A.vals[(size_t)p]);
    rho = std::max(rho, s / std::fabs(d[(size_t)i]));
  }
  return rho;
}

// the inverse of the dense n x n matrix of A by Gauss-Jordan elimination with partial pivoting (row-major); 0, or
// column + 1 of the first zero pivot
inline int64_t amg_dense_inverse(const AmgCsr &A, std::vector<double> *inv) {
  const int64_t n = A.m;
  std::vector<double> M((size_t)(n * n), 0.0);
  inv->assign((size_t)(n * n), 0.0);
  for (int64_t i = 0; i < n; ++i) {
    for (int64_t p = A.rowptr[(size_t)i]; p < A.rowptr[(size_t)i + 1]; ++p) M[(size_t)(i * n + A.colind[(size_t)p])] = A.vals[(size_t)p];
    (*inv)[(size_t)(i * n + i)] = 1.0;
  }
  std::vector<double> &X = *inv;
  for (int64_t k = 0; k < n; ++k) {
    int64_t piv = k;
    for (int64_t i = k + 1; i < n; ++i)
      if (std::fabs(M[(size_t)(i * n + k)]) > std::fabs(M[(size_t)(piv * n + k)])) piv = i;
    if (M[(size_t)(piv * n + k)] == 0.0) return k + 1;
    if (piv != k)
      for (int64_t j = 0; j < n; ++j) {
        std::swap(M[(size_t)(k * n + j)], M[(size_t)(piv * n + j)]);
        std::swap(X[(size_t)(k * n + j)], X[(size_t)(piv * n + j)]);
      }
    const double s = 1.0 / M[(size_t)(k * n + k)];
    for (int64_t j = 0; j < n; ++j) {
      M[(size_t)(k * n + j)] *= s;
      X[(size_t)(k * n + j)] *= s;
    }
    for (int64_t i = 0; i < n; ++i) {
      if (i == k) continue;
      const double f = M[(size_t)(i * n + k)];
      if (f == 0.0) continue;
      for (int64_t j = 0; j < n; ++j) {
        M[(size_t)(i * n + j)] -= f * M[(size_t)(k * n + j)];
        X[(size_t)(i * n + j)] -= f * X[(size_t)(k * n + j)];
      }
    }
  }
  return 0;
}

// seconds spent in the phases of the setup (the library adds the download and the upload)
struct AmgTimes {
  double aggregation = 0.0, prolongator = 0.0, rap = 0.0;
};

// The hierarchy of A (levels.back() is the coarsest).  `clock` returns seconds (any origin).
template <typename Clock>
AmgStatus amg_setup(AmgCsr A, const AmgOptions &o, std::vector<AmgLevel> *levels, AmgTimes *times, Clock &&clock) {
  AmgStatus st;
  levels->clear();
  std::vector<double> B((size_t)A.m, 1.0), d;
  if (const int64_t bad = amg_diagonal(A, &d)) {
    st.code = AMG_ZERO_DIAGONAL;
    st.row = bad - 1;
    return st;
  }
  while (A.m > o.max_coarse && (int)levels->size() + 1 < o.max_levels) {
    if (const int64_t bad = amg_diagonal(A, &d)) {
      st = AmgStatus{AMG_ZERO_DIAGONAL, (int)levels->size(), bad - 1};
      return st;
    }
    double t0 = clock();
    AmgLevel L;
    const int naggs = amg_aggregate(amg_strength(A, d, o.theta), &L.agg);
    double t1 = clock();
    times->aggregation += t1 - t0;
    if (naggs == 0) break;   // every row isolated: nothing to coarsen, this level is the coarsest
    std::vector<double> Bc;
    const AmgCsr T = amg_tentative(L.agg, naggs, B, &Bc);
    const double rho = amg_rho(A, d);
    L.P = amg_prolongator(A, d, T, rho);
    L.w.resize((size_t)A.m);
    for (int64_t i = 0; i < A.m; ++i) L.w[(size_t)i] = ((4.0 / 3.0) / rho) / d[(size_t)i];
    t0 = clock();
    times->prolongator += t0 - t1;
    L.R = amg_transpose(L.P);
    AmgCsr Ac = amg_spgemm(L.R, amg_spgemm(A, L.P));
    times->rap += clock() - t0;
    L.A = std::move(A);
    levels->push_back(std::move(L));
    A = std::move(Ac);
    B = std::move(Bc);
  }
  const double t0 = clock();
  AmgLevel L;
  if (A.m > kAmgMaxCoarsest) {
    st = AmgStatus{AMG_TOO_LARGE, (int)levels->size(), A.m};
    return st;
  }
  if (const int64_t bad = amg_dense_inverse(A, &L.inv)) {
    st = AmgStatus{AMG_ZERO_PIVOT, (int)levels->size(), bad - 1};
    return st;
  }
  times->rap += clock() - t0;
  L.A = std::move(A);
  levels->push_back(std::move(L));
  return st;
}

// ---------------------------------------------------------------------------------------------------------------------
// The serial V-cycle (aspreconditioner: one cycle from a zero initial guess) in the element type T, on the fp64 levels
// rounded to T as the device stores them.  Each step is the device's: x = w b (first pre-sweep), x <- x + w (b - A x),
// r = b - A x, b_c = R r, recursion, x <- x + P x_c, post-sweeps; the coarsest level is x = A^-1 b.
template <typename T>
void amg_spmv_serial(const AmgCsr &A, const T *x, T *y) {
  for (int64_t i = 0; i < A.m; ++i) {
    T acc = (T)0;
    for (int64_t p = A.rowptr[(size_t)i]; p < A.rowptr[(size_t)i + 1]; ++p)
      acc += (T)A.vals[(size_t)p] * x[A.colind[(size_t)p]];
    y[i] = acc;
  }
}

template <typename T>
void amg_vcycle_serial(const std::vector<AmgLevel> &lev, const AmgOptions &o, size_t l, const T *b, T *x) {
  const AmgLevel &L = lev[l];
  const int64_t n = L.A.m;
  if (l + 1 == lev.size()) {
    for (int64_t i = 0; i < n; ++i) {
      T acc = (T)0;
      for (int64_t j = 0; j < n; ++j) acc += (T)L.inv[(size_t)(i * n + j)] * b[j];
      x[i] = acc;
    }
    return;
  }
  std::vector<T> w((size_t)n), Ax((size_t)n), r((size_t)n);
  for (int64_t i = 0; i < n; ++i) w[(size_t)i] = (T)L.w[(size_t)i];
  std::fill(x, x + n, (T)0);
  auto sweep = [&]() {
    amg_spmv_serial(L.A, x, Ax.data());
    for (int64_t i = 0; i < n; ++i) x[i] = x[i] + w[(size_t)i] * (b[i] - Ax[(size_t)i]);
  };
  for (int s = 0; s < o.presweeps; ++s) {
    if (s == 0)
      for (int64_t i = 0; i < n; ++i) x[i] = w[(size_t)i] * b[i];
    else
      sweep();
  }
  amg_spmv_serial(L.A, x, Ax.data());
  for (int64_t i = 0; i < n; ++i) r[(size_t)i] = b[i] - Ax[(size_t)i];
  const int64_t nc = L.P.n;
  std::vector<T> bc((size_t)nc), xc((size_t)nc), Pe((size_t)n);
  amg_spmv_serial(L.R, r.data(), bc.data());
  amg_vcycle_serial(lev, o, l + 1, bc.data(), xc.data());
  amg_spmv_serial(L.P, xc.data(), Pe.data());
  for (int64_t i = 0; i < n; ++i) x[i] = x[i] + Pe[(size_t)i];
  for (int s = 0; s < o.postsweeps; ++s) sweep();
}

}  // namespace b200
