// amg_setup_core.h -- the row functions of the device setup of smoothed aggregation (amg_setup.cu, DESIGN section 23),
// each written once for the host and the device so that the CPU tests (tests/hostsim_amg_rows) run them serially and compare
// them with amg_core.h's serial setup bit for bit.
//
//   pass 1 of the aggregation   amg_pass1_decide: the lexicographically-first maximal independent set of the candidates
//                               under the conflict relation r ~ i  <=>  r in S(i), or i in S(r), or S(r) and S(i) meet
//                               (S S', not S' S).  A candidate is a row with a non-empty strong row and no strong
//                               neighbour j < i whose own strong row is empty.  The roots are amg_aggregate's pass-1
//                               roots, and a root's aggregate is itself plus S(r).
//   SpGEMM row i of C = A B     amg_spgemm_accumulate / amg_table_compact / amg_spgemm_emit: Gustavson's order, as
//                               amg_spgemm: for each output (i, j) the products a_ik b_kj added in ascending k, starting
//                               from +0.0, into an open-addressing table; then exact zeros dropped and the columns
//                               written ascending.  The lanes of one row split each row k of B (distinct columns, so no
//                               two lanes touch one slot in a step); `sync` separates the k steps.
// Every product and sum is rounded on its own (mul_rn / add_rn of complex.h; the host test build has -ffp-contract=off).
#pragma once
#include <stdint.h>

#include <vector>

#include "complex.h"

namespace b200 {

enum { AMG_UNDECIDED = 0, AMG_ROOT = 1, AMG_NOT_ROOT = 2 };

struct AmgRows {   // a CSR view with int32 row offsets
  const int *rp;
  const int *ci;
  const double *v;   // may be NULL for a pattern
};

// The pass-1 state of undecided candidate i from the states of its smaller conflicting rows (st(r) reads row r's state):
// AMG_NOT_ROOT once one of them is a root, AMG_ROOT once all of them are decided non-roots, else AMG_UNDECIDED.
// S: the strong pattern; St: its transpose.
template <typename State>
B200_HD int amg_pass1_decide(const AmgRows &S, const AmgRows &St, int i, State &&st) {
  bool waiting = false;
  auto look = [&](int r) {   // true: r is a smaller root
    if (r >= i) return false;
    const int s = st(r);
    if (s == AMG_ROOT) return true;
    if (s == AMG_UNDECIDED) waiting = true;
    return false;
  };
  for (int p = S.rp[i]; p < S.rp[i + 1]; ++p) {
    const int j = S.ci[p];
    if (look(j)) return AMG_NOT_ROOT;   // r in S(i)
    for (int q = St.rp[j]; q < St.rp[j + 1]; ++q)
      if (look(St.ci[q])) return AMG_NOT_ROOT;   // j in S(r): S(r) and S(i) meet
  }
  for (int p = St.rp[i]; p < St.rp[i + 1]; ++p)
    if (look(St.ci[p])) return AMG_NOT_ROOT;   // i in S(r)
  return waiting ? AMG_UNDECIDED : AMG_ROOT;
}

// the initial pass-1 state of row i: AMG_UNDECIDED for a candidate, AMG_NOT_ROOT otherwise
B200_HD int amg_pass1_initial(const AmgRows &S, int i) {
  if (S.rp[i] == S.rp[i + 1]) return AMG_NOT_ROOT;
  for (int p = S.rp[i]; p < S.rp[i + 1]; ++p) {
    const int j = S.ci[p];
    if (j < i && S.rp[j] == S.rp[j + 1]) return AMG_NOT_ROOT;
  }
  return AMG_UNDECIDED;
}

B200_HD int amg_cas(int *p, int expect, int v) {
#ifdef __CUDA_ARCH__
  return atomicCAS(p, expect, v);
#else
  const int old = *p;
  if (old == expect) *p = v;
  return old;
#endif
}

// the slot of column j in keys[0, cap) (cap a power of two, -1 = empty), inserted if missing; -1 when the table is full
B200_HD int amg_table_insert(int *keys, int cap, int j) {
  unsigned h = ((unsigned)j * 2654435761u) & (unsigned)(cap - 1);
  for (int t = 0; t < cap; ++t) {
    const int old = amg_cas(keys + h, -1, j);
    if (old == -1 || old == j) return (int)h;
    h = (h + 1) & (unsigned)(cap - 1);
  }
  return -1;
}

// The products of row i of A B into the table (keys -1 and acc +0.0 on entry).  sync(ok) ends a k step and returns
// whether every lane's inserts fit so far; returns false once the table overflowed (the row is then incomplete).
template <typename Sync>
B200_HD bool amg_spgemm_accumulate(const AmgRows &A, const AmgRows &B, int64_t i, int *keys, double *acc, int cap,
                                   int lane, int nlanes, Sync &&sync) {
  for (int p = A.rp[i]; p < A.rp[i + 1]; ++p) {
    const int k = A.ci[p];
    const double a = A.v[p];
    bool ok = true;
    for (int q = B.rp[k] + lane; q < B.rp[k + 1]; q += nlanes) {
      const int s = amg_table_insert(keys, cap, B.ci[q]);
      if (s < 0) ok = false;
      else acc[s] = add_rn(acc[s], mul_rn(a, B.v[q]));
    }
    if (!sync(ok)) return false;
  }
  return true;
}

// Moves the table's nonzero sums to (lc, lv) in some order and empties the table; returns their number.  On the device
// the 32 lanes of a warp run it together (nlanes == 32, cap a multiple of 32).
B200_HD int amg_table_compact(int *keys, double *acc, int cap, int lane, int nlanes, int *lc, double *lv) {
  int u = 0;
  for (int s0 = 0; s0 < cap; s0 += nlanes) {
    const int s = s0 + lane;
    const bool keep = s < cap && keys[s] >= 0 && acc[s] != 0.0;
#ifdef __CUDA_ARCH__
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    const int pos = u + __popc(m & ((1u << lane) - 1u));
    u += __popc(m);
#else
    const int pos = u;
    u += keep;
#endif
    if (keep) {
      lc[pos] = keys[s];
      lv[pos] = acc[s];
    }
    if (s < cap) {
      keys[s] = -1;
      acc[s] = 0.0;
    }
  }
  return u;
}

// Writes the u compacted entries with their columns ascending (each entry's rank is the number of smaller columns)
B200_HD void amg_spgemm_emit(const int *lc, const double *lv, int u, int lane, int nlanes, int *ci, double *v) {
  for (int e = lane; e < u; e += nlanes) {
    const int j = lc[e];
    int r = 0;
    for (int f = 0; f < u; ++f) r += lc[f] < j;
    ci[r] = j;
    v[r] = lv[e];
  }
}

// Serial runs for the CPU tests.  Pass 1 in rounds (every undecided candidate re-decided from the previous round's
// states) to the fixpoint; returns the roots' flags and the number of rounds.
inline int amg_pass1_rounds(const AmgRows &S, const AmgRows &St, int n, std::vector<int> *state) {
  state->assign((size_t)n, AMG_NOT_ROOT);
  for (int i = 0; i < n; ++i) (*state)[(size_t)i] = amg_pass1_initial(S, i);
  std::vector<int> next;
  int rounds = 0;
  for (bool busy = true; busy;) {
    busy = false;
    next = *state;
    for (int i = 0; i < n; ++i)
      if ((*state)[(size_t)i] == AMG_UNDECIDED) {
        next[(size_t)i] = amg_pass1_decide(S, St, i, [&](int r) { return (*state)[(size_t)r]; });
        busy = busy || next[(size_t)i] == AMG_UNDECIDED;
      }
    state->swap(next);
    ++rounds;
  }
  return rounds;
}

// one row of C = A B on one lane with a table of cap slots; returns the row's length, or -1 when the table overflowed
inline int amg_spgemm_row_serial(const AmgRows &A, const AmgRows &B, int64_t i, int cap, std::vector<int> *ci,
                                 std::vector<double> *v) {
  std::vector<int> keys((size_t)cap, -1), lc((size_t)cap);
  std::vector<double> acc((size_t)cap, 0.0), lv((size_t)cap);
  if (!amg_spgemm_accumulate(A, B, i, keys.data(), acc.data(), cap, 0, 1, [](bool ok) { return ok; })) return -1;
  const int u = amg_table_compact(keys.data(), acc.data(), cap, 0, 1, lc.data(), lv.data());
  ci->resize((size_t)u);
  v->resize((size_t)u);
  amg_spgemm_emit(lc.data(), lv.data(), u, 0, 1, ci->data(), v->data());
  return u;
}

}  // namespace b200
