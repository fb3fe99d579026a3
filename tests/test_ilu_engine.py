"""The ILU(0) preconditioner (csrc/ilu_core.h), checked without a GPU.

tests/hostsim_ilu runs the row functions the GPU kernels run (factor row, forward row, backward row) serially over the
same chunk schedules, with a dependency check in place of the device's wait.  They are compared bit for bit with the plain
numpy restatement below (IKJ ILU(0), Saad Algorithm 10.4; the solves sum in ascending column order and round every step,
as the row functions do), in Float64 and Float32.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
_ILIB = None


def ilib():
    """the ILU(0) row functions on the serial backend (tests/hostsim_ilu, built with make)"""
    global _ILIB
    if _ILIB is None:
        d = os.path.join(HERE, "hostsim_ilu")
        subprocess.run(["make", "-s", "-C", d], check=True)
        _ILIB = C.CDLL(os.path.join(d, "libhostsim_ilu.so"))
        _ILIB.hostsim_ilu0_chunks.restype = C.c_int64
    return _ILIB


class _Csr(C.Structure):
    _fields_ = [("m", C.c_int64), ("n", C.c_int64), ("rowptr", C.c_void_p), ("colind", C.c_void_p),
                ("vals", C.c_void_p)]


class Csr:
    """0-based CSR (int64 row offsets, int32 columns, ascending in every row) kept alive for the C calls"""

    def __init__(self, A, dtype):
        A = sp.csr_matrix(A)
        A.sort_indices()
        self.shape = A.shape
        self.rowptr = np.ascontiguousarray(A.indptr, dtype=np.int64)
        self.colind = np.ascontiguousarray(A.indices, dtype=np.int32)
        self.vals = np.ascontiguousarray(A.data, dtype=dtype)
        self.c = _Csr(A.shape[0], A.shape[1], self.rowptr.ctypes.data, self.colind.ctypes.data, self.vals.ctypes.data)


def sim_factor(M: Csr):
    """(status, bad row, factor values, forward levels, backward levels) from the serial backend"""
    f = np.empty_like(M.vals)
    bad, lf, lb = C.c_int64(-1), C.c_int(0), C.c_int(0)
    st = ilib().hostsim_ilu0_factor(C.c_int(M.vals.dtype == np.float64), C.byref(M.c), C.c_void_p(f.ctypes.data),
                                    C.byref(bad), C.byref(lf), C.byref(lb))
    return st, bad.value, f, lf.value, lb.value


def sim_ldiv(M: Csr, f, x, y=None):
    """y = U \\ (L \\ x) on the serial backend (y = None: in place on a copy of x)"""
    x = np.ascontiguousarray(x, dtype=M.vals.dtype)
    y = x.copy() if y is None else y
    bad = C.c_int64(-1)
    st = ilib().hostsim_ilu0_ldiv(C.c_int(M.vals.dtype == np.float64), C.byref(M.c), C.c_void_p(f.ctypes.data),
                                  C.c_void_p(x.ctypes.data), C.c_void_p(y.ctypes.data), C.byref(bad))
    assert st == 0, (st, bad.value)
    return y


def sim_chunks(M: Csr, backward):
    n = M.shape[0]
    rows = np.empty(n, dtype=np.int32)
    cptr = np.empty(n + 1, dtype=np.int32)
    nc = ilib().hostsim_ilu0_chunks(C.byref(M.c), C.c_int(int(backward)), C.c_void_p(rows.ctypes.data),
                                    C.c_void_p(cptr.ctypes.data))
    assert nc >= 0
    return rows, cptr[: nc + 1]


# ------------------------------------------------------------------------------------------------------------------
# numpy restatement
# ------------------------------------------------------------------------------------------------------------------
class NumpyILU0:
    """ILU(0) of a CSR matrix (ascending columns) in IKJ order, and its two triangular solves.  Every operation is a
    numpy operation in the matrix's dtype (one rounding each, no fused multiply-add).  `ldiv` / `ldiv3` make it a
    preconditioner for the oracle's solvers (ldiv!(P, x) / ldiv!(y, P, x))."""

    def __init__(self, A, dtype):
        A = sp.csr_matrix(A)
        A.sort_indices()
        self.n = A.shape[0]
        self.rowptr = A.indptr.astype(np.int64)
        self.colind = A.indices.astype(np.int64)
        T = np.dtype(dtype)
        f = A.data.astype(T)
        rp, ci, n = self.rowptr, self.colind, self.n
        dpos = np.full(n, -1, dtype=np.int64)
        for i in range(n):
            hit = np.nonzero(ci[rp[i]:rp[i + 1]] == i)[0]
            if hit.size == 0 or f[rp[i] + hit[0]] == 0:
                raise np.linalg.LinAlgError(f"zero or missing diagonal entry in row {i}")
            dpos[i] = rp[i] + hit[0]
        self.d = dpos
        pivot = None
        for i in range(n):                                       # IKJ, Saad Algorithm 10.4
            cols_i = {int(ci[s]): s for s in range(rp[i], rp[i + 1])}
            for p in range(rp[i], dpos[i]):
                k = int(ci[p])
                f[p] = f[p] / f[dpos[k]]
                for q in range(dpos[k] + 1, rp[k + 1]):
                    s = cols_i.get(int(ci[q]))
                    if s is not None and s > p:
                        f[s] = f[s] - f[p] * f[q]
            if f[dpos[i]] == 0 and pivot is None:
                pivot = i
        if pivot is not None:
            raise np.linalg.LinAlgError(f"zero pivot in row {pivot}")
        self.f = f
        self._lev_f = self._levels(lambda i: range(rp[i], dpos[i]), range(n))
        self._lev_b = self._levels(lambda i: range(dpos[i] + 1, rp[i + 1]), range(n - 1, -1, -1))

    def _levels(self, deps, order):
        """per dependency level: (rows, [(selection of rows, positions of their t-th dependency), t = 0, 1, ...])"""
        lev = np.zeros(self.n, dtype=np.int64)
        for i in order:
            ps = deps(i)
            lev[i] = 1 + max(lev[self.colind[p]] for p in ps) if len(ps) else 0
        out = []
        for l in range(int(lev.max()) + 1 if self.n else 0):
            rows = np.nonzero(lev == l)[0]
            first = np.array([deps(i).start for i in rows], dtype=np.int64)
            cnt = np.array([len(deps(i)) for i in rows], dtype=np.int64)
            steps = []
            for t in range(int(cnt.max()) if rows.size else 0):
                sel = np.nonzero(cnt > t)[0]
                steps.append((sel, first[sel] + t))
            out.append((rows, steps))
        return out

    @property
    def levels(self):
        return len(self._lev_f), len(self._lev_b)

    def solve(self, x):
        f, ci = self.f, self.colind
        y = np.array(x, dtype=f.dtype, copy=True)
        for rows, steps in self._lev_f:                       # y_i = x_i - sum_{j<i, ascending} l_ij y_j
            acc = y[rows]
            for sel, pos in steps:
                acc[sel] = acc[sel] - f[pos] * y[ci[pos]]
            y[rows] = acc
        for rows, steps in self._lev_b:                       # z_i = (y_i - sum_{j>i, ascending} u_ij z_j) / u_ii
            acc = y[rows]
            for sel, pos in steps:
                acc[sel] = acc[sel] - f[pos] * y[ci[pos]]
            y[rows] = acc / f[self.d[rows]]
        return y

    def ldiv(self, x):
        x[...] = self.solve(x)
        return x

    def ldiv3(self, y, x):
        y[...] = self.solve(x)
        return y


# ------------------------------------------------------------------------------------------------------------------
# matrices
# ------------------------------------------------------------------------------------------------------------------
def random_nonsymmetric(n, density, seed):
    rng = np.random.default_rng(seed)
    R = sp.random(n, n, density=density, random_state=rng, format="csr")
    R.data = rng.standard_normal(R.nnz)
    A = (R + sp.diags(np.full(n, 4.0 + n * density))).tocsr()
    A.sort_indices()
    return A


def no_lower_rows(n=40, seed=7):
    """rows 0, 5, 10, ... have no strictly lower part; the others couple to a few earlier and later rows"""
    rng = np.random.default_rng(seed)
    A = random_nonsymmetric(n, 0.1, seed).tolil()
    for i in range(0, n, 5):
        A[i, :i] = 0
    A = A.tocsr()
    A.eliminate_zeros()
    A.sort_indices()
    A.data += rng.uniform(0.0, 0.1, A.nnz)
    return A


MATRICES = {
    "laplace2d_9": lambda: O.laplace_matrix_scipy(np.float64, 9, 2),
    "laplace3d_6": lambda: O.laplace_matrix_scipy(np.float64, 6, 3),
    "advection_12": lambda: O.advection_dominated(12)[0],
    "random_nonsym_300": lambda: random_nonsymmetric(300, 0.02, 11),
    "n1": lambda: sp.csr_matrix(np.array([[3.0]])),
    "no_lower_rows": no_lower_rows,
}


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", sorted(MATRICES))
def test_factor_and_solves_bit_for_bit(name, dtype):
    A = MATRICES[name]()
    M = Csr(A, dtype)
    st, bad, f, lf, lb = sim_factor(M)
    assert st == 0, (st, bad)
    ref = NumpyILU0(A, dtype)
    assert f.tobytes() == ref.f.tobytes()
    assert (lf, lb) == ref.levels
    rng = np.random.default_rng(5)
    x = rng.standard_normal(A.shape[0]).astype(dtype)
    y = sim_ldiv(M, f, x, np.empty_like(x))
    assert y.tobytes() == ref.solve(x).tobytes()
    assert sim_ldiv(M, f, x).tobytes() == y.tobytes()              # in place
    # the factor really is ILU(0): L U agrees with A on A's pattern (exact arithmetic up to rounding)
    if dtype == np.float64:
        F = sp.csr_matrix((f, M.colind, M.rowptr), shape=A.shape)
        L = sp.tril(F, -1) + sp.identity(A.shape[0])
        U = sp.triu(F)
        LU = (L @ U).tocsr()
        Ac = sp.csr_matrix(A)
        r, c = Ac.nonzero()
        assert np.allclose(np.asarray(LU[r, c]).ravel(), np.asarray(Ac[r, c]).ravel(), rtol=1e-12, atol=1e-12 * abs(Ac).max())


def test_laplace_levels_are_3N_minus_2():
    N = 7
    M = Csr(O.laplace_matrix_scipy(np.float64, N, 3), np.float64)
    st, _, _, lf, lb = sim_factor(M)
    assert st == 0 and lf == lb == 3 * N - 2


@pytest.mark.parametrize("name", sorted(MATRICES))
def test_chunk_list(name):
    A = sp.csr_matrix(MATRICES[name]())
    A.sort_indices()
    M = Csr(A, np.float64)
    n = A.shape[0]
    for backward in (0, 1):
        rows, cptr = sim_chunks(M, backward)
        assert sorted(rows.tolist()) == list(range(n))
        assert cptr[0] == 0 and cptr[-1] == n and np.all(np.diff(cptr) >= 1) and np.all(np.diff(cptr) <= 32)
        chunk_of = np.empty(n, dtype=np.int64)
        for c in range(len(cptr) - 1):
            chunk_of[rows[cptr[c]:cptr[c + 1]]] = c
        lev = np.zeros(n, dtype=np.int64)
        order = range(n - 1, -1, -1) if backward else range(n)
        for i in order:
            cols = A.indices[A.indptr[i]:A.indptr[i + 1]]
            deps = cols[cols > i] if backward else cols[cols < i]
            lev[i] = 1 + lev[deps].max() if deps.size else 0
            assert np.all(chunk_of[deps] < chunk_of[i]), (backward, i)          # every dependency in an earlier chunk
        for c in range(len(cptr) - 1):
            assert np.unique(lev[rows[cptr[c]:cptr[c + 1]]]).size == 1             # a chunk lies in one level
        assert np.all(np.diff(lev[rows]) >= 0)                                     # chunks in level order


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_zero_pivot_is_refused_with_its_row(dtype):
    # row 2: u_22 = 1 - (1/1) * 1 = 0 although a_22 != 0; rows 0, 1 are fine
    A = sp.csr_matrix(np.array([[2.0, 0.0, 1.0], [0.0, 1.0, 0.0], [2.0, 0.0, 1.0]]))
    st, bad, _, _, _ = sim_factor(Csr(A, dtype))
    assert (st, bad) == (2, 2)
    with pytest.raises(np.linalg.LinAlgError, match="zero pivot in row 2"):
        NumpyILU0(A, dtype)


def test_missing_or_zero_diagonal_is_refused_with_its_row():
    A = sp.csr_matrix(np.array([[2.0, 1.0, 0.0], [1.0, 0.0, 1.0], [0.0, 1.0, 2.0]]))   # row 1 has no diagonal entry
    st, bad, _, _, _ = sim_factor(Csr(A, np.float64))
    assert (st, bad) == (3, 1)
    B = sp.csr_matrix(np.array([[2.0, 1.0], [1.0, 1.0]]))
    B.data[3] = 0.0                                                                  # explicit zero a_11
    st, bad, _, _, _ = sim_factor(Csr(B, np.float64))
    assert (st, bad) == (3, 1)
