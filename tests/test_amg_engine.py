"""The smoothed-aggregation AMG preconditioner (csrc/amg_core.h), checked without a GPU.

tests/hostsim_amg runs the setup the library runs on the host, and the serial V-cycle, on the CPU.  They are compared
with the plain numpy / scipy restatement below (AlgebraicMultigrid.jl's / pyamg's smoothed_aggregation with B = ones,
SymmetricStrength, standard aggregation, fit_candidates, JacobiProlongation(4/3) with the Gershgorin bound for rho,
R = P', A_c = R A P, the coarsest level's explicit inverse; weighted-Jacobi V-cycle): identical aggregates, level sizes
and patterns, P, A_c and the coarse inverse within 1e-14 relative.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import oracle as O
from test_ilu_engine import Csr, random_nonsymmetric

HERE = os.path.dirname(os.path.abspath(__file__))
_ALIB = None


def alib():
    """the AMG setup and serial V-cycle on the serial backend (tests/hostsim_amg, built with make)"""
    global _ALIB
    if _ALIB is None:
        d = os.path.join(HERE, "hostsim_amg")
        subprocess.run(["make", "-s", "-C", d], check=True)
        _ALIB = C.CDLL(os.path.join(d, "libhostsim_amg.so"))
        _ALIB.hostsim_amg_setup.argtypes = [C.c_void_p, C.c_double, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                            C.c_void_p]
        _ALIB.hostsim_amg_levels.argtypes = [C.c_void_p]
        _ALIB.hostsim_amg_level_sizes.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        _ALIB.hostsim_amg_level_get.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 9
        _ALIB.hostsim_amg_vcycle.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        _ALIB.hostsim_amg_free.argtypes = [C.c_void_p]
    return _ALIB


def _p(a):
    return None if a is None else a.ctypes.data


class SimAMG:
    """a hierarchy built by the library's setup code on the CPU"""

    def __init__(self, A, theta=0.0, max_levels=10, max_coarse=10, presweeps=1, postsweeps=1):
        self.M = Csr(A, np.float64)
        self.n = self.M.shape[0]
        bad = np.zeros(2, dtype=np.int64)
        h = C.c_void_p()
        self.status = alib().hostsim_amg_setup(C.byref(self.M.c), theta, max_levels, max_coarse, presweeps, postsweeps,
                                               _p(bad), C.byref(h))
        self.bad = (int(bad[0]), int(bad[1]))
        self._h = h

    def __del__(self):
        if getattr(self, "_h", None) and self._h.value:
            alib().hostsim_amg_free(self._h)

    def levels(self):
        out = []
        nl = alib().hostsim_amg_levels(self._h)
        for l in range(nl):
            s = np.zeros(4, dtype=np.int64)
            alib().hostsim_amg_level_sizes(self._h, l, _p(s))
            n, nnz, nc, pnnz = (int(v) for v in s)
            coarsest = l + 1 == nl
            arp, aci, av = np.empty(n + 1, np.int64), np.empty(nnz, np.int32), np.empty(nnz)
            prp, pci, pv = np.empty(n + 1, np.int64), np.empty(pnnz, np.int32), np.empty(pnnz)
            agg, w = np.empty(n, np.int32), np.empty(n)
            inv = np.empty((n, n)) if coarsest else None
            alib().hostsim_amg_level_get(self._h, l, _p(arp), _p(aci), _p(av), _p(prp), _p(pci), _p(pv), _p(agg), _p(w),
                                         _p(inv))
            out.append({"A": sp.csr_matrix((av, aci, arp), shape=(n, n)),
                        "P": None if coarsest else sp.csr_matrix((pv, pci, prp), shape=(n, nc)),
                        "agg": None if coarsest else agg, "w": None if coarsest else w, "inv": inv})
        return out

    def vcycle(self, b, dtype=np.float64):
        b = np.ascontiguousarray(b, dtype=dtype)
        x = np.empty_like(b)
        alib().hostsim_amg_vcycle(self._h, int(dtype == np.float64), _p(b), _p(x))
        return x

    # ldiv!(P, x) / ldiv!(y, P, x) for the oracle's solvers
    def ldiv(self, x):
        x[...] = self.vcycle(x)
        return x

    def ldiv3(self, y, x):
        y[...] = self.vcycle(x)
        return y


# ------------------------------------------------------------------------------------------------------------------
# numpy / scipy restatement
# ------------------------------------------------------------------------------------------------------------------
def np_strength(A, theta):
    """SymmetricStrength(theta): the strong off-diagonal entries |a_ij| >= theta sqrt(|a_ii a_jj|), as a pattern"""
    C_ = sp.coo_matrix(A)
    d = A.diagonal()
    keep = (C_.row != C_.col) & (np.abs(C_.data) >= theta * np.sqrt(np.abs(d[C_.row] * d[C_.col])))
    S = sp.csr_matrix((np.ones(keep.sum()), (C_.row[keep], C_.col[keep])), shape=A.shape)
    S.sort_indices()
    return S


def np_aggregate(S):
    """standard_aggregation (pyamg / AlgebraicMultigrid.jl), in row order: returns (aggregate of each row, -1 =
    isolated; number of aggregates)"""
    n = S.shape[0]
    FREE = -2
    x = np.full(n, FREE, dtype=np.int64)
    nb = [S.indices[S.indptr[i]:S.indptr[i + 1]] for i in range(n)]
    nxt = 0
    for i in range(n):                                       # pass 1
        if x[i] != FREE:
            continue
        if len(nb[i]) == 0:
            x[i] = -1
        elif np.all(x[nb[i]] == FREE):
            x[i] = nxt
            x[nb[i]] = nxt
            nxt += 1
    join = x.copy()
    for i in range(n):                                       # pass 2: first aggregated strong neighbour
        if x[i] == FREE:
            for j in nb[i]:
                if x[j] >= 0:
                    join[i] = x[j]
                    break
    x = join
    for i in range(n):                                       # pass 3
        if x[i] == FREE:
            x[i] = nxt
            x[nb[i][x[nb[i]] == FREE]] = nxt
            nxt += 1
    return x, nxt


class NumpySA:
    """The hierarchy and the V-cycle, in numpy / scipy.  Levels: dicts with A, P, R, agg, w (the smoother weights
    omega_s / a_ii) and, on the coarsest level, inv."""

    def __init__(self, A, theta=0.0, max_levels=10, max_coarse=10, presweeps=1, postsweeps=1):
        A = sp.csr_matrix(A, dtype=np.float64)
        A.sort_indices()
        self.pre, self.post = presweeps, postsweeps
        self.levels = []
        B = np.ones(A.shape[0])
        while A.shape[0] > max_coarse and len(self.levels) + 1 < max_levels:
            n = A.shape[0]
            d = A.diagonal()
            agg, na = np_aggregate(np_strength(A, theta))
            if na == 0:
                break
            rows = np.nonzero(agg >= 0)[0]
            Bc = np.sqrt(np.bincount(agg[rows], weights=B[rows] ** 2, minlength=na))
            T = sp.csr_matrix((B[rows] / Bc[agg[rows]], (rows, agg[rows])), shape=(n, na))
            rho = np.max(np.asarray(abs(A).sum(axis=1)).ravel() / np.abs(d))
            P = (T - (4.0 / 3.0 / rho) * (sp.diags(1.0 / d) @ (A @ T))).tocsr()
            P.eliminate_zeros()
            P.sort_indices()
            R = P.T.tocsr()
            R.sort_indices()
            self.levels.append({"A": A, "P": P, "R": R, "agg": agg, "w": (4.0 / 3.0 / rho) / d})
            A = (R @ (A @ P)).tocsr()
            A.eliminate_zeros()
            A.sort_indices()
            B = Bc
        self.levels.append({"A": A, "P": None, "agg": None, "inv": np.linalg.inv(A.toarray())})

    def vcycle(self, b, dtype=np.float64, l=0):
        L = self.levels[l]
        if L["P"] is None:
            return L["inv"].astype(dtype) @ b
        A, w = L["A"].astype(dtype), L["w"].astype(dtype)
        x = np.zeros_like(b)
        for s in range(self.pre):
            x = w * b if s == 0 else x + w * (b - A @ x)
        r = b - A @ x
        x = x + L["P"].astype(dtype) @ self.vcycle(L["R"].astype(dtype) @ r, dtype, l + 1)
        for _ in range(self.post):
            x = x + w * (b - A @ x)
        return x

    def ldiv(self, x):
        x[...] = self.vcycle(x)
        return x

    def ldiv3(self, y, x):
        y[...] = self.vcycle(x)
        return y


# ------------------------------------------------------------------------------------------------------------------
# matrices
# ------------------------------------------------------------------------------------------------------------------
def isolated_rows(N=12):
    """the 2-D Laplacian with rows (and columns) 0, 7, 14, ... cut down to their diagonal: isolated nodes"""
    A = O.laplace_matrix_scipy(np.float64, N, 2).tolil()
    for i in range(0, N * N, 7):
        d = A[i, i]
        A[i, :] = 0
        A[:, i] = 0
        A[i, i] = d
    A = A.tocsr()
    A.eliminate_zeros()
    return A


def anisotropic(N=16, eps=1e-3):
    """-u_xx - eps u_yy: with theta = 0.25 the eps-couplings are weak and dropped from the strength pattern"""
    T = sp.diags([-np.ones(N - 1), 2 * np.ones(N), -np.ones(N - 1)], [-1, 0, 1])
    I = sp.identity(N)
    return (sp.kron(I, T) + eps * sp.kron(T, I)).tocsr()


MATRICES = {
    "laplace2d_20": (lambda: O.laplace_matrix_scipy(np.float64, 20, 2), {}),
    "laplace3d_10": (lambda: O.laplace_matrix_scipy(np.float64, 10, 3), {}),
    "advection_12": (lambda: O.advection_dominated(12)[0], {}),
    "isolated_rows": (isolated_rows, {}),
    "anisotropic_theta": (anisotropic, {"theta": 0.25}),
    "random_nonsym_300": (lambda: random_nonsymmetric(300, 0.02, 11), {}),
    "n1": (lambda: sp.csr_matrix(np.array([[3.0]])), {}),
    "small_le_max_coarse": (lambda: O.laplace_matrix_scipy(np.float64, 3, 2), {}),
    "two_levels_max": (lambda: O.laplace_matrix_scipy(np.float64, 8, 2), {"max_levels": 2}),
}


def _rel(a, b):
    a, b = np.asarray(a), np.asarray(b)
    scale = max(np.max(np.abs(b)), 1e-300) if b.size else 1.0
    return float(np.max(np.abs(a - b)) / scale) if b.size else 0.0


def compare_hierarchies(got, ref, tol=1e-14):
    """got: levels as from SimAMG.levels() / SmoothedAggregationPrec.levels(); ref: a NumpySA"""
    assert len(got) == len(ref.levels)
    for l, (g, r) in enumerate(zip(got, ref.levels)):
        for key in ("A", "P"):
            if r[key] is None:
                assert g[key] is None
                continue
            G, Rm = sp.csr_matrix(g[key]), r[key]
            assert G.shape == Rm.shape, (l, key)
            assert np.array_equal(G.indptr, Rm.indptr) and np.array_equal(G.indices, Rm.indices), (l, key)
            assert _rel(G.data, Rm.data) <= tol, (l, key, _rel(G.data, Rm.data))
        if r["agg"] is None:
            assert g["agg"] is None and _rel(g["inv"], r["inv"]) <= tol, l
        else:
            assert np.array_equal(g["agg"], r["agg"]), l


@pytest.mark.parametrize("name", sorted(MATRICES))
def test_hierarchy_matches_the_restatement(name):
    make, kw = MATRICES[name]
    A = make()
    sim = SimAMG(A, **kw)
    assert sim.status == 0, (sim.status, sim.bad)
    ref = NumpySA(A, **kw)
    got = sim.levels()
    compare_hierarchies(got, ref)
    for g, r in zip(got[:-1], ref.levels[:-1]):
        assert _rel(g["w"], r["w"]) <= 1e-15
    rng = np.random.default_rng(5)
    b = rng.standard_normal(A.shape[0])
    assert _rel(sim.vcycle(b), ref.vcycle(b)) <= 1e-13
    b32 = b.astype(np.float32)
    assert _rel(sim.vcycle(b32, np.float32), ref.vcycle(b32, np.float32)) <= 1e-5


def test_laplace_3d_coarsens_about_8x_per_level():
    sim = SimAMG(O.laplace_matrix_scipy(np.float64, 24, 3))
    rows = [L["A"].shape[0] for L in sim.levels()]
    assert rows[0] == 24 ** 3 and rows[-1] <= 10
    assert all(4 <= a / b for a, b in zip(rows[:-2], rows[1:-1])), rows


def test_aggregates_of_a_1d_laplacian():
    # pass 1: {0,1} from node 0, {2,3,4} from node 3, {5,6} from node 6; nothing is left for passes 2 and 3
    A = O.laplace_matrix_scipy(np.float64, 7, 1)
    lv = SimAMG(A, max_coarse=1).levels()
    assert lv[0]["agg"].tolist() == [0, 0, 1, 1, 1, 2, 2]


def test_passes_two_and_three():
    # node 0 is isolated (no strong off-diagonal); node 3 (pass 1) takes {3, 4}; node 5's only strong neighbour 4 is
    # taken, so pass 2 puts it into that aggregate; nodes 1 and 2 see only each other and the isolated node 0, so pass 1
    # skips them and pass 3 makes {1, 2}
    A = sp.csr_matrix(np.array([[4.0, 0, 0, 0, 0, 0],
                                [-1, 4, -1, 0, 0, 0],
                                [-1, 0, 4, 0, 0, 0],
                                [0, 0, 0, 4, -1, 0],
                                [0, 0, 0, -1, 4, 0],
                                [0, 0, 0, 0, -1, 4]]))
    agg_np, na = np_aggregate(np_strength(A, 0.0))
    assert agg_np.tolist() == [-1, 1, 1, 0, 0, 0] and na == 2
    lv = SimAMG(A, max_coarse=1).levels()
    assert lv[0]["agg"].tolist() == [-1, 1, 1, 0, 0, 0]
    compare_hierarchies(lv, NumpySA(A, max_coarse=1))


@pytest.mark.parametrize("name", ["laplace2d_20", "laplace3d_7", "isolated_rows"])
def test_vcycle_is_symmetric_positive_definite(name):
    A = {"laplace2d_20": lambda: O.laplace_matrix_scipy(np.float64, 20, 2),
         "laplace3d_7": lambda: O.laplace_matrix_scipy(np.float64, 7, 3), "isolated_rows": isolated_rows}[name]()
    n = A.shape[0]
    assert n <= 500
    sim = SimAMG(A)
    M = np.column_stack([sim.vcycle(e) for e in np.eye(n)])
    assert np.linalg.norm(M - M.T) <= 1e-12 * np.linalg.norm(M)
    assert np.linalg.eigvalsh((M + M.T) / 2).min() > 0


def test_exact_solve_when_n_is_at_most_max_coarse():
    A = O.laplace_matrix_scipy(np.float64, 3, 2)
    sim = SimAMG(A)
    assert len(sim.levels()) == 1
    b = np.random.default_rng(2).standard_normal(9)
    assert np.linalg.norm(A @ sim.vcycle(b) - b) <= 1e-14 * np.linalg.norm(b)


@pytest.mark.parametrize("N, expected", [(16, 14), (32, 16)])
def test_pcg_iterations_match_the_prototype(N, expected):
    A = O.laplace_matrix_scipy(np.float64, N, 3)
    b = np.random.default_rng(1).standard_normal(A.shape[0])
    sim = SimAMG(A)
    _, h = O.cg_(np.zeros(A.shape[0]), O.CSC.from_scipy(A), b, Pl=sim, log=True, initially_zero=True)
    assert h.isconverged and abs(h.niters - expected) <= 1, h.niters


def test_refusals():
    zero_diag = sp.csr_matrix(np.array([[2.0, -1, 0], [-1, 0, -1], [0, -1, 2]]))
    sim = SimAMG(zero_diag, max_coarse=1)
    assert (sim.status, sim.bad) == (1, (0, 1))
    big = O.laplace_matrix_scipy(np.float64, 70, 2)                        # 4900 rows, one level
    sim = SimAMG(big, max_levels=1)
    assert (sim.status, sim.bad) == (3, (0, 4900))
    singular = sp.csr_matrix(np.array([[1.0, 1.0], [1.0, 1.0]]))
    sim = SimAMG(singular)
    assert (sim.status, sim.bad) == (2, (0, 1))
