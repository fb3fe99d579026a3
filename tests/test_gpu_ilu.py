"""The ILU(0) preconditioner on the GPU (csrc/ilu.cu): one persistent launch for the factorization and one per triangular
solve, scheduled through a chunk list with per-row ready flags.

  - the factor values and ldiv! are bit-identical to the serial evaluation of the same row functions (tests/hostsim_ilu)
    and to the numpy restatement of tests/test_ilu_engine.py, run to run and in place;
  - cg!, gmres! (Pl and Pr; MGS, CGS, DGKS), bicgstabl!(2) and idrs!(4) with ILU0Prec against the oracle's solvers given
    the numpy ILU(0): equal iteration counts, histories and x within 1e-10;
  - ILU(0)-PCG needs fewer iterations than Jacobi-PCG on the 64^3 Laplacian;
  - the refusals of b200_ilu0_create, each before any data is touched.
"""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import oracle as O
from test_ilu_engine import MATRICES, Csr, NumpyILU0, sim_factor, sim_ldiv

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def isb():
    import iterativesolvers_jl_b200 as m
    return m


def _csr(A):
    A = sp.csr_matrix(A)
    A.sort_indices()
    return A


GPU_MATRICES = dict(MATRICES)
GPU_MATRICES["laplace3d_64"] = lambda: O.laplace_matrix_scipy(np.float64, 64, 3)
GPU_MATRICES["advection_24"] = lambda: O.advection_dominated(24)[0]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", sorted(GPU_MATRICES))
def test_factor_and_ldiv_bit_identical_to_the_serial_run(isb, name, dtype):
    A = _csr(GPU_MATRICES[name]())
    M = Csr(A, dtype)
    st, bad, f_ref, lf, lb = sim_factor(M)
    assert st == 0, (st, bad)
    Ad = isb.B200CSR.from_scipy(A.astype(dtype))
    P = isb.ILU0Prec(Ad)
    assert P.values().tobytes() == f_ref.tobytes()
    assert P.levels == (lf, lb)
    rng = np.random.default_rng(3)
    x = rng.standard_normal(A.shape[0]).astype(dtype)
    y_ref = sim_ldiv(M, f_ref, x, np.empty_like(x))
    xd = isb.DeviceArray.from_numpy(Ad.ctx, x)
    yd = isb.DeviceArray(Ad.ctx, A.shape[0], dtype)
    P.ldiv_(yd, xd)
    y1 = yd.numpy()
    assert y1.tobytes() == y_ref.tobytes()
    P.ldiv_(yd, xd)                                            # a second apply: fresh epoch, same bits
    assert yd.numpy().tobytes() == y1.tobytes()
    P.ldiv_(xd, xd)                                            # ldiv!(P, x) in place
    assert xd.numpy().tobytes() == y1.tobytes()
    assert np.array_equal(xd.numpy(), y1)
    if A.shape[0] <= 2000:                                     # the numpy restatement (its factor loop is Python)
        ref = NumpyILU0(A, dtype)
        assert ref.f.tobytes() == f_ref.tobytes() and ref.solve(x).tobytes() == y1.tobytes()
    L, U = P.factors()
    F = sp.csr_matrix((f_ref, M.colind, M.rowptr), shape=A.shape)
    assert (L - (sp.tril(F, -1) + sp.identity(A.shape[0]))).count_nonzero() == 0
    assert (U - sp.triu(F)).count_nonzero() == 0


def _check(h, ho, x, xo, tol=1e-10):
    assert h.niters == ho.niters and h.isconverged == ho.isconverged, (h.niters, ho.niters)
    ro = np.asarray(ho["resnorm"])
    r = np.asarray(h["resnorm"])
    assert r.shape == ro.shape
    assert np.max(np.abs(r - ro)) <= tol * ro[0]
    assert np.linalg.norm(x - xo) <= tol * np.linalg.norm(xo)


def test_cg_with_ilu0_matches_the_oracle(isb):
    A = _csr(O.laplace_matrix_scipy(np.float64, 48, 3))
    b = np.random.default_rng(1).standard_normal(A.shape[0])
    b /= np.linalg.norm(b)
    P = isb.ILU0Prec(isb.B200CSR.from_scipy(A))
    x, h = isb.cg(P.A, b, Pl=P, log=True)
    xo, ho = O.cg_(np.zeros(A.shape[0]), O.CSC.from_scipy(A), b, Pl=NumpyILU0(A, np.float64), log=True,
                   initially_zero=True)
    assert h.isconverged
    _check(h, ho, x, xo)


@pytest.fixture(scope="module")
def advection(isb):
    A, b = O.advection_dominated(24)
    A = _csr(A)
    Ad = isb.B200CSR.from_scipy(A)
    return A, b, Ad, isb.ILU0Prec(Ad), NumpyILU0(A, np.float64), O.CSC.from_scipy(A)


@pytest.mark.parametrize("side", ["Pl", "Pr"])
@pytest.mark.parametrize("orth", ["mgs", "cgs", "dgks"])
def test_gmres_with_ilu0_matches_the_oracle(isb, advection, side, orth):
    A, b, Ad, P, Pn, Ao = advection
    x, h = isb.gmres(Ad, b, restart=20, orth_meth=orth, log=True, **{side: P})
    xo, ho = O.gmres_(np.zeros(A.shape[0]), Ao, b, restart=20, orth_meth=orth, log=True, initially_zero=True,
                      **{side: Pn})
    assert h.isconverged
    _check(h, ho, x, xo)


def test_bicgstabl_with_ilu0_matches_the_oracle(isb, advection):
    A, b, Ad, P, Pn, Ao = advection
    rs = np.random.default_rng(2).random(A.shape[0])
    x, h = isb.bicgstabl(Ad, b, 2, Pl=P, r_shadow=rs, log=True)
    xo, ho = O.bicgstabl_(np.zeros(A.shape[0]), Ao, b, 2, Pl=Pn, r_shadow=rs.copy(), log=True, initial_zero=True)
    assert h.isconverged
    _check(h, ho, x, xo)


def test_idrs_with_ilu0_matches_the_oracle(isb, advection):
    A, b, Ad, P, Pn, Ao = advection
    s = 4
    Pm = np.asfortranarray(np.random.default_rng(4).random((A.shape[0], s)))
    x, h = isb.idrs(Ad, b, s=s, Pl=P, P=Pm, log=True)
    xo, ho = O.idrs_(np.zeros(A.shape[0]), Ao, b, s=s, Pl=Pn, P=[Pm[:, j].copy() for j in range(s)], log=True)
    assert h.isconverged
    _check(h, ho, x, xo)


def test_ilu0_beats_jacobi_in_iterations_on_the_64_cube(isb):
    A = isb.B200CSR.laplacian(64, 3, np.float64)
    b = np.random.default_rng(6).standard_normal(A.m_local)
    _, hj = isb.cg(A, b, Pl=isb.JacobiPrec(A.diag()), log=True)
    P = isb.ILU0Prec(A)
    _, hi = isb.cg(A, b, Pl=P, log=True)
    assert hj.isconverged and hi.isconverged
    assert hi.niters < hj.niters, (hi.niters, hj.niters)


def _create(isb, A):
    h = C.c_void_p()
    st = isb.lib().b200_ilu0_create(A.ctx._h, A._h, C.byref(h))
    return st, isb.lib().b200_last_error().decode(), h


def _refused(isb, A, status, *words):
    before = A.download()
    st, msg, h = _create(isb, A)
    assert st == status, (st, msg)
    assert not h.value
    for w in words:
        assert w in msg, msg
    after = A.download()
    for u, v in zip(before, after):
        assert u.tobytes() == v.tobytes()                      # nothing touched


def test_refusals(isb):
    lap = O.laplace_matrix_scipy(np.float64, 5, 2)
    _refused(isb, isb.B200CSR.from_scipy(lap.astype(np.complex128)), -6, "b200_ilu0_create", "ComplexF64")
    _refused(isb, isb.B200CSR.from_scipy(lap.astype(np.complex64)), -6, "ComplexF32")
    ctx8 = isb.Context(0)
    ctx8.set_option("rowptr64", 1)
    A8 = isb.B200CSR.from_scipy(lap, ctx=ctx8)
    assert A8.index_bytes == 8
    _refused(isb, A8, -6, "8-byte")
    rect = sp.random(6, 8, 0.4, random_state=1, format="csr") + sp.eye(6, 8)
    _refused(isb, isb.B200CSR.from_scipy(rect), -1, "square")
    pivot = sp.csr_matrix(np.array([[2.0, 0.0, 1.0], [0.0, 1.0, 0.0], [2.0, 0.0, 1.0]]))
    _refused(isb, isb.B200CSR.from_scipy(pivot), -5, "zero pivot", "row 2")
    missing = sp.csr_matrix(np.array([[2.0, 1.0, 0.0], [1.0, 0.0, 1.0], [0.0, 1.0, 2.0]]))
    _refused(isb, isb.B200CSR.from_scipy(missing), -5, "row 1")
    with pytest.raises(isb.B200Error, match="zero pivot u_ii in row 2"):
        isb.ILU0Prec(isb.B200CSR.from_scipy(pivot))
