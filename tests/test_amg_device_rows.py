"""The row functions of the device AMG setup (csrc/amg_setup_core.h), checked without a GPU.

tests/hostsim_amg_rows runs them serially: pass 1 of the aggregation as the rounds of amg_pass1_decide to their fixpoint
(the lexicographically-first maximal independent set of the candidates under S S'), followed by the device's ids,
pass 2 and pass 3; and the per-row SpGEMM (open-addressing table, products in ascending k, exact zeros dropped, columns
ascending).  The aggregates must equal amg_aggregate's and the products amg_spgemm's, bit for bit.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import oracle as O
from test_amg_engine import SimAMG, anisotropic, isolated_rows
from test_ilu_engine import Csr, random_nonsymmetric

HERE = os.path.dirname(os.path.abspath(__file__))
_RLIB = None


def _lib():
    """the row functions on the serial backend (tests/hostsim_amg_rows, built with make)"""
    global _RLIB
    if _RLIB is not None:
        return _RLIB
    d = os.path.join(HERE, "hostsim_amg_rows")
    subprocess.run(["make", "-s", "-C", d], check=True)
    L = C.CDLL(os.path.join(d, "libhostsim_amg_rows.so"))
    L.hostsim_amg_aggregate_rows.argtypes = [C.c_void_p, C.c_double] + [C.c_void_p] * 5
    L.hostsim_amg_aggregate_rows.restype = C.c_int
    L.hostsim_amg_spgemm_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 6
    L.hostsim_amg_spgemm_rows.restype = C.c_int64
    _RLIB = L
    return L


def aggregate_both(A, theta):
    M = Csr(A, np.float64)
    n = A.shape[0]
    ref, got = np.empty(n, np.int32), np.empty(n, np.int32)
    na, rounds, p3 = C.c_int(), C.c_int(), C.c_int()
    nref = _lib().hostsim_amg_aggregate_rows(C.byref(M.c), theta, ref.ctypes.data, got.ctypes.data, C.byref(na),
                                             C.byref(rounds), C.byref(p3))
    return nref, ref, na.value, got, rounds.value, p3.value


def with_isolated(A, every):
    """A with rows and columns 0, every, 2 every, ... cut down to their diagonal"""
    A = sp.lil_matrix(A)
    for i in range(0, A.shape[0], every):
        d = A[i, i]
        A[i, :] = 0
        A[:, i] = 0
        A[i, i] = d
    A = A.tocsr()
    A.eliminate_zeros()
    return A


def random_pattern(n, density, seed):
    """a non-symmetric pattern with a few empty strong rows: random off-diagonal entries, some rows off-diagonal-free"""
    rng = np.random.default_rng(seed)
    A = random_nonsymmetric(n, density, seed).tolil()
    for i in rng.choice(n, n // 25, replace=False):
        d = A[i, i]
        A[i, :] = 0
        A[i, i] = d
    A = A.tocsr()
    A.eliminate_zeros()
    return A


CASES = ([("random", n, dens, seed, theta) for seed in range(16) for (n, dens) in ((60, 0.05), (300, 0.01), (300, 0.03))
          for theta in (0.0, 0.3)])


@pytest.mark.parametrize("kind, n, dens, seed, theta", CASES)
def test_aggregates_equal_amg_aggregate(kind, n, dens, seed, theta):
    A = random_pattern(n, dens, seed)
    nref, ref, na, got, rounds, _ = aggregate_both(A, theta)
    assert na == nref and np.array_equal(got, ref), (nref, na)
    assert rounds >= 1


def test_random_patterns_reach_pass_three_and_isolated_nodes():
    reached, isolated = 0, 0
    for seed, n, dens, theta in [(s, 300, 0.01, t) for s in range(16) for t in (0.0, 0.3)]:
        nref, ref, na, got, _, p3 = aggregate_both(random_pattern(n, dens, seed), theta)
        assert np.array_equal(got, ref)
        reached += p3 > 0
        isolated += int((ref == -1).any())
    assert reached >= 3 and isolated >= 3, (reached, isolated)


@pytest.mark.parametrize("name", ["laplace3d_12", "laplace2d_30", "isolated_rows", "anisotropic_theta",
                                  "advection_12", "with_isolated"])
def test_aggregates_of_the_engine_matrices(name):
    A, theta = {"laplace3d_12": (lambda: O.laplace_matrix_scipy(np.float64, 12, 3), 0.0),
                "laplace2d_30": (lambda: O.laplace_matrix_scipy(np.float64, 30, 2), 0.0),
                "isolated_rows": (isolated_rows, 0.0),
                "anisotropic_theta": (anisotropic, 0.25),
                "advection_12": (lambda: O.advection_dominated(12)[0], 0.0),
                "with_isolated": (lambda: with_isolated(random_nonsymmetric(200, 0.03, 5), 9), 0.1)}[name]
    A = A() if callable(A) else A
    nref, ref, na, got, rounds, _ = aggregate_both(A, theta)
    assert na == nref and np.array_equal(got, ref)


def test_pass_one_rounds_on_the_laplacian():
    # the rounds of the fixpoint grow about linearly with N on natural-order N^3 Laplacians
    r16 = aggregate_both(O.laplace_matrix_scipy(np.float64, 16, 3), 0.0)[4]
    assert 40 <= r16 <= 100, r16


def spgemm_both(A, B, cap):
    A, B = sp.csr_matrix(A), sp.csr_matrix(B)
    Ma, Mb = Csr(A, np.float64), Csr(B, np.float64)
    bound = int(((abs(A) > 0).astype(np.int64) @ (abs(B) > 0).astype(np.int64)).nnz) + 1
    m = A.shape[0]
    rp, ci, v = np.empty(m + 1, np.int64), np.empty(bound, np.int32), np.empty(bound)
    rpr, cir, vr = np.empty(m + 1, np.int64), np.empty(bound, np.int32), np.empty(bound)
    nnz = _lib().hostsim_amg_spgemm_rows(C.byref(Ma.c), C.byref(Mb.c), cap, rp.ctypes.data, ci.ctypes.data,
                                         v.ctypes.data, rpr.ctypes.data, cir.ctypes.data, vr.ctypes.data)
    assert nnz >= 0, nnz
    return (rp, ci[:nnz], v[:nnz]), (rpr, cir[:nnz], vr[:nnz])


def _same(got, ref):
    for g, r in zip(got, ref):
        assert g.tobytes() == r.tobytes()


def _cap(B):
    cap = 32
    while cap < 2 * B.shape[1]:
        cap *= 2
    return cap


@pytest.mark.parametrize("seed", range(12))
def test_spgemm_rows_equal_amg_spgemm_with_cancellation(seed):
    # small integer values: many sums cancel to exactly zero, and -0.0 products appear
    rng = np.random.default_rng(seed)
    m, k, n = 80, 70, 50
    A = sp.random(m, k, density=0.08, random_state=rng, format="csr")
    B = sp.random(k, n, density=0.1, random_state=rng, format="csr")
    A.data = rng.choice([-2.0, -1.0, 1.0, 2.0, -0.0], A.nnz)
    B.data = rng.choice([-1.0, 1.0, 0.5], B.nnz)
    A.sort_indices()
    B.sort_indices()
    got, ref = spgemm_both(A, B, _cap(B))
    _same(got, ref)


@pytest.mark.parametrize("seed", range(12))
def test_spgemm_rows_equal_amg_spgemm_on_random_reals(seed):
    rng = np.random.default_rng(100 + seed)
    A = random_nonsymmetric(150, 0.04, seed)
    B = sp.random(150, 90, density=0.05, random_state=rng, format="csr")
    B.data = rng.standard_normal(B.nnz)
    B.sort_indices()
    got, ref = spgemm_both(A, B, _cap(B))
    _same(got, ref)


@pytest.mark.parametrize("name", ["laplace3d_10", "random_nonsym_300", "advection_12"])
def test_spgemm_rows_equal_amg_spgemm_on_the_galerkin_products(name):
    from test_amg_engine import MATRICES
    make, kw = MATRICES[name]
    lv = SimAMG(make(), **kw).levels()
    for L in lv[:-1]:
        A, P = L["A"], L["P"]
        got, ref = spgemm_both(A, P, _cap(P))
        _same(got, ref)
        AP = sp.csr_matrix((ref[2], ref[1], ref[0]), shape=(A.shape[0], P.shape[1]))
        R = P.T.tocsr()
        R.sort_indices()
        got, ref = spgemm_both(R, AP, _cap(AP))
        _same(got, ref)


def test_spgemm_row_reports_a_full_table():
    A = sp.csr_matrix(np.ones((1, 40)))
    B = sp.identity(40, format="csr")
    Ma, Mb = Csr(A, np.float64), Csr(B, np.float64)
    buf = [np.empty(41, np.int64), np.empty(41, np.int32), np.empty(41)] * 2
    assert _lib().hostsim_amg_spgemm_rows(C.byref(Ma.c), C.byref(Mb.c), 32, *(b.ctypes.data for b in buf)) == -1
