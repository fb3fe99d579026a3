"""GPU tests of the complex element types (ComplexF64 / ComplexF32): the complex CSR operator and its SpMV, the BLAS-1
calls, cg! and gmres! (general engines, csrc/cg_core.h and csrc/gmres_core.h), and the entry points that reject
complex data with B200_ERR_UNSUPPORTED.

The oracles are scipy's products, numpy, oracle.gmres_ and the complex cg! restatement of tests/test_complex_engines.py.
"""
import ctypes as C
import math

import numpy as np
import pytest
import scipy.linalg as sla
import scipy.sparse as sp

from oracle import oracle as O
from test_complex_engines import cg_oracle_c, crand

pytestmark = pytest.mark.gpu
UNSUPPORTED = -6


@pytest.fixture(scope="module")
def isb():
    import iterativesolvers_jl_b200 as m
    m.default_context()
    return m


def lib(isb):
    from iterativesolvers_jl_b200 import _lib
    return _lib.lib()


def set_spmv_kernel(isb, ctx, v):
    assert lib(isb).b200_ctx_set_option(ctx._h, b"spmv_kernel", v) == 0


def laplace3d(N):
    T = sp.diags([-np.ones(N - 1), 2 * np.ones(N), -np.ones(N - 1)], [-1, 0, 1])
    I = sp.identity(N)
    return (sp.kron(sp.kron(I, I), T) + sp.kron(sp.kron(I, T), I) + sp.kron(sp.kron(T, I), I)).tocsr()


def hpd3d(N):
    """A = L + I + i S: L the 3-D Laplacian, S the real antisymmetric central difference in x with coefficient 1/4;
    Hermitian positive definite, every eigenvalue >= 1/2."""
    D = sp.diags([-np.ones(N - 1), np.ones(N - 1)], [-1, 1]) * 0.25
    S = sp.kron(sp.identity(N * N), D)
    return (laplace3d(N) + sp.identity(N ** 3) + 1j * S).tocsr()


def helmholtz3d(N, k2=0.5, sigma=0.5):
    """the shifted Helmholtz operator -Laplace - k^2 I + i sigma I."""
    return (laplace3d(N) - k2 * sp.identity(N ** 3) + 1j * sigma * sp.identity(N ** 3)).tocsr()


def random_complex(rng, m, n, lens, dt):
    rows, cols = [], []
    for i, L in enumerate(lens):
        c = rng.choice(n, size=min(L, n), replace=False)
        rows += [i] * len(c)
        cols += list(c)
    v = rng.standard_normal(len(rows)) + 1j * rng.standard_normal(len(rows))
    return sp.csr_matrix((v.astype(dt), (rows, cols)), shape=(m, n))


def offset_view(isb, ctx, data, dt):
    """a device vector view that starts half an element past an element boundary: 8 bytes for ComplexF64 (numpy's
    complex128 alignment), 4 for ComplexF32; the SpMV must take its scalar-load instantiation"""
    n = data.shape[0]
    owner = isb.DeviceArray(ctx, n + 2, dt)
    ptr = owner.ptr + np.dtype(dt).itemsize // 2       # library allocations are 256-byte aligned
    v = isb.DeviceArray.view(ctx, ptr, n, dt)
    v.upload(data)
    return owner, v


# ------------------------------------------------------------------------------------------------ SpMV
CASES = [("rows_1_300", 1500, 1500), ("empty_rows", 700, 700), ("n1", 1, 1), ("wide", 400, 1300)]


@pytest.mark.parametrize("dt,tol", [(np.complex128, 1e-14), (np.complex64, 1e-5)])
@pytest.mark.parametrize("case,m,n", CASES)
def test_spmv_against_scipy(isb, dt, tol, case, m, n):
    rng = np.random.default_rng([c for c, _, _ in CASES].index(case) + 100)
    if case == "rows_1_300":
        lens = rng.integers(1, 301, size=m)                             # every lanes-per-row from 2 to 32
    elif case == "empty_rows":
        lens = np.where(rng.random(m) < 0.3, 0, rng.integers(1, 12, size=m))
    else:
        lens = rng.integers(1, 40, size=m) if m > 1 else [1]
    A = random_complex(rng, m, n, lens, dt)
    ctx = isb.default_context()
    Ad = isb.B200CSR.from_scipy(A)
    assert Ad.dtype == np.dtype(dt)
    kind = C.c_int()
    assert lib(isb).b200_csr_stream_kind(Ad._h, C.byref(kind), None) == 0 and kind.value == 1
    x = crand(rng, n, dt) - (0.5 + 0.5j)
    want = A.astype(np.complex128) @ x.astype(np.complex128)
    scale = abs(A).astype(np.float64) @ np.abs(x).astype(np.float64)
    scale[scale == 0] = 1.0
    ys = []
    for k in range(4):                                                  # spmv_kernel 0..3: the sub-warp form each time
        set_spmv_kernel(isb, ctx, k)
        ys.append(Ad @ x)
    set_spmv_kernel(isb, ctx, 0)
    for y in ys[1:]:
        assert np.array_equal(y, ys[0])
    assert float(np.max(np.abs(ys[0] - want) / scale)) <= tol
    # x and y views half an element off: the scalar-load instantiation, bit-identical values
    xo, xv = offset_view(isb, ctx, x, dt)
    yo, yv = offset_view(isb, ctx, np.zeros(m, dt), dt)
    Ad.mul_(yv, xv)
    assert np.array_equal(yv.numpy(), ys[0])
    # the operator round-trips and its diagonal is diag(A)
    rp, ci, vals = Ad.download()
    assert np.array_equal(sp.csr_matrix((vals, ci, rp), shape=(m, n)).toarray(), A.toarray())
    if m == n:
        assert np.array_equal(Ad.diag().numpy(), A.diagonal())


@pytest.mark.parametrize("dt,tol", [(np.complex128, 1e-13), (np.complex64, 1e-5)])
def test_blas1(isb, dt, tol):
    ctx = isb.default_context()
    L = lib(isb)
    code = 2 if dt == np.complex128 else 3
    rng = np.random.default_rng(5)
    n = 100003
    x, y, d = crand(rng, n, dt), crand(rng, n, dt), crand(rng, n, dt) + 1
    xd, yd, dd = (isb.DeviceArray.from_numpy(ctx, a) for a in (x, y, d))
    res = (C.c_double * 2)()
    assert L.b200_dotc(ctx._h, n, xd._p, yd._p, code, res) == 0
    want = np.vdot(x.astype(np.complex128), y.astype(np.complex128))
    assert abs(complex(res[0], res[1]) - want) / abs(want) <= tol
    r = C.c_double()
    assert L.b200_nrm2(ctx._h, n, xd._p, code, C.byref(r)) == 0
    assert abs(r.value - np.linalg.norm(x.astype(np.complex128))) / r.value <= tol
    assert L.b200_dot(ctx._h, n, xd._p, yd._p, code, C.byref(r)) == UNSUPPORTED
    assert b"b200_dotc" in L.b200_last_error()
    zd = isb.DeviceArray(ctx, n, dt)
    assert L.b200_jacobi_ldiv(ctx._h, n, dd._p, xd._p, zd._p, code) == 0
    np.testing.assert_allclose(zd.numpy(), x / d, rtol=10 * np.finfo(np.zeros(1, dt).real.dtype).eps)
    assert L.b200_axpby(ctx._h, n, 2.0, xd._p, -0.5, yd._p, code) == 0
    np.testing.assert_allclose(yd.numpy(), 2 * x - 0.5 * y, rtol=tol * 10)
    assert L.b200_scal(ctx._h, n, 3.0, xd._p, code) == 0
    np.testing.assert_allclose(xd.numpy(), 3 * x, rtol=tol * 10)
    assert L.b200_copy(ctx._h, n, xd._p, zd._p, code) == 0
    assert np.array_equal(zd.numpy(), xd.numpy())
    assert L.b200_fill(ctx._h, n, 1.5, zd._p, code) == 0
    assert np.all(zd.numpy() == 1.5 + 0j)


# ------------------------------------------------------------------------------------------------ cg!
def _jacobi_fn(isb, ctx, d):
    dd = isb.DeviceArray.from_numpy(ctx, d)
    jp = isb.JacobiPrec(dd)
    return isb.FunctionPrec(d.shape[0], d.dtype, lambda y, x: jp.ldiv_(y, x), ctx)


@pytest.mark.parametrize("prec", ["identity", "jacobi", "callback"])
@pytest.mark.parametrize("op", ["csr", "linop"])
@pytest.mark.parametrize("dt", [np.complex128, np.complex64])
def test_cg_against_oracle(isb, prec, op, dt):
    A = hpd3d(32)
    n = A.shape[0]
    ctx = isb.default_context()
    b = crand(np.random.default_rng(17), n)
    d = A.diagonal()
    Ad = isb.B200CSR.from_scipy(A.astype(dt))
    Aop = Ad if op == "csr" else isb.B200LinearOperator((n, n), dt, lambda y, x: Ad.mul_(y, x), ctx=ctx)
    Pl = {"identity": None, "jacobi": isb.JacobiPrec(d.astype(dt), ctx), "callback": _jacobi_fn(isb, ctx, d.astype(dt))}[prec]
    reltol = 1e-8 if dt == np.complex128 else 1e-4
    x, h = isb.cg(Aop, b.astype(dt), Pl=Pl, log=True, reltol=reltol)
    xo, ho = cg_oracle_c(np.zeros(n, np.complex128), A, b, diag=None if prec == "identity" else d, reltol=reltol,
                         initially_zero=True)
    if dt == np.complex128:
        assert h.niters == ho["iters"] and h.isconverged
        assert float(np.max(np.abs(h["resnorm"] - ho["resnorm"]))) / np.linalg.norm(b) <= 1e-10
        assert np.linalg.norm(x - xo) / np.linalg.norm(xo) <= 1e-10
    else:                                   # ComplexF32 vectors, fp64 scalars: within 3 iterations, x to 1e-3
        assert abs(h.niters - ho["iters"]) <= 3 and h.isconverged
        assert np.linalg.norm(x - xo) / np.linalg.norm(xo) <= 1e-3


# ------------------------------------------------------------------------------------------------ gmres!
@pytest.mark.parametrize("meth", ["mgs", "cgs", "dgks"])
def test_gmres_against_oracle(isb, meth):
    A = helmholtz3d(24)
    n = A.shape[0]
    b = crand(np.random.default_rng(23), n)
    Ad = isb.B200CSR.from_scipy(A)
    x, h = isb.gmres(Ad, b, restart=20, maxiter=60, orth_meth=meth, log=True)
    xo, ho = O.gmres_(np.zeros(n, np.complex128), A, b, restart=20, maxiter=60, log=True, initially_zero=True,
                      orth_meth=meth)
    hist_o = np.asarray(ho["resnorm"])
    assert h.iters == ho.iters and h.mvps == ho.mvps
    assert float(np.max(np.abs(h["resnorm"] - hist_o))) / hist_o[0] <= 1e-10
    assert np.linalg.norm(x - xo) / np.linalg.norm(xo) <= 1e-10


def test_gmres_reference_cases_lu_callbacks(isb):
    """test/gmres.jl:16-34 for ComplexF64 with the exact LU preconditioner as a Python ldiv! callback."""
    ctx = isb.default_context()
    rng = np.random.default_rng(1234321)
    n = 10
    A = crand(rng, (n, n)) + np.eye(n)
    b = crand(rng, n)
    lu = sla.lu_factor(A)
    F = isb.FunctionPrec(n, np.complex128, lambda y, x: y.upload(sla.lu_solve(lu, x.numpy())), ctx)
    Ad = isb.B200CSR.from_scipy(sp.csc_matrix(A))
    reltol = math.sqrt(np.finfo(np.float64).eps)
    x, h = isb.gmres(Ad, b, log=True, restart=3, maxiter=10, reltol=reltol)
    assert np.all(np.diff(h["resnorm"]) <= 0.0)
    x, h = isb.gmres(Ad, b, Pl=F, maxiter=1, restart=1, reltol=reltol, log=True)
    assert h.isconverged and np.linalg.norm(sla.lu_solve(lu, A @ x - b)) / np.linalg.norm(b) <= reltol
    x, h = isb.gmres(Ad, b, Pr=F, maxiter=1, restart=1, reltol=reltol, log=True)
    assert h.isconverged and np.linalg.norm(A @ x - b) / np.linalg.norm(b) <= reltol


def test_gmres30_cycle_128(isb):
    """one GMRES(30) cycle (CGS) on the 128^3 shifted Helmholtz operator against the live oracle."""
    A = helmholtz3d(128)
    n = A.shape[0]
    b = crand(np.random.default_rng(29), n)
    Ad = isb.B200CSR.from_scipy(A)
    x, h = isb.gmres(Ad, b, restart=30, maxiter=30, orth_meth="cgs", log=True)
    xo, ho = O.gmres_(np.zeros(n, np.complex128), A, b, restart=30, maxiter=30, log=True, initially_zero=True,
                      orth_meth="cgs")
    hist_o = np.asarray(ho["resnorm"])
    assert h.iters == ho.iters == 30
    assert float(np.max(np.abs(h["resnorm"] - hist_o))) / hist_o[0] <= 1e-10
    assert np.linalg.norm(x - xo) / np.linalg.norm(xo) <= 1e-10


# ------------------------------------------------------------------------------------------------ real data as complex
def test_real_data_as_complex(isb):
    """given real data, the complex solvers agree with the real general engines to 1e-13, imaginary parts exactly 0."""
    ctx = isb.default_context()
    L = laplace3d(16) + 0.1 * sp.identity(16 ** 3)
    N = (laplace3d(16) + sp.diags([np.full(16 ** 3 - 1, 0.4)], [1]) - 0.3 * sp.identity(16 ** 3)).tocsr()
    b = np.random.default_rng(31).random(16 ** 3)
    for A, solve in ((L, "cg"), (N, "gmres")):
        Ar = isb.B200CSR.from_scipy(A)
        Ac = isb.B200CSR.from_scipy(A.astype(np.complex128))
        fn = getattr(isb, solve)
        kw = dict(log=True) if solve == "cg" else dict(log=True, restart=20, maxiter=100, orth_meth="dgks")
        # the real general engine: the operator through the callback interface
        xr, hr = fn(isb.B200LinearOperator.from_csr(Ar), b, **kw)
        xc, hc = fn(Ac, b.astype(np.complex128), **kw)
        assert hr.iters == hc.iters
        assert np.all(xc.imag == 0)
        assert np.linalg.norm(xc.real - xr) / np.linalg.norm(xr) <= 1e-13
        assert float(np.max(np.abs(hc["resnorm"] - hr["resnorm"]))) / np.linalg.norm(b) <= 1e-13   # relative to r0


# ------------------------------------------------------------------------------------------------ rejections
REJECT = [  # entry point, {argument index: role}; every other argument is NULL / 0
    ("b200_minres_solve", {1: "A", 2: "x", 3: "b"}), ("b200_bicgstabl_solve", {1: "A", 2: "x", 3: "b"}),
    ("b200_chebyshev_solve", {1: "A", 2: "x", 3: "b"}), ("b200_idrs_solve", {1: "A", 2: "x", 3: "b"}),
    ("b200_qmr_solve", {1: "A", 2: "A", 3: "x", 4: "b"}), ("b200_lsqr_solve", {1: "A", 2: "A", 3: "x", 4: "b"}),
    ("b200_lsmr_solve", {1: "A", 2: "A", 3: "x", 4: "b"}), ("b200_lobpcg_solve", {1: "A", 2: "x"}),
    ("b200_lobpcg_solve_constrained", {1: "A", 2: "x"}), ("b200_svdl", {1: "A", 2: "A", 3: "x"}),
    ("b200_powm", {1: "A", 3: "x"}), ("b200_stationary", {1: "A", 2: "x", 3: "b"}),
    ("b200_cg_iter_create", {1: "A", 2: "x", 3: "b"}), ("b200_gmres_iter_create", {1: "A", 3: "x", 4: "b"}),
    ("b200_minres_iter_create", {1: "A", 3: "x", 4: "b"}), ("b200_bicgstabl_iter_create", {1: "A", 3: "x", 4: "b"}),
    ("b200_cg_iter_create_op", {1: "A", 3: "x", 4: "b"}), ("b200_spmm", {1: "A", 2: "x", 4: "b"}),
    ("b200_csr_transpose", {1: "A"}),
    ("b200_minres_solve_op", {1: "op", 2: "x", 3: "b"}), ("b200_bicgstabl_solve_op", {1: "op", 2: "x", 3: "b"}),
    ("b200_chebyshev_solve_op", {1: "op", 2: "x", 3: "b"}), ("b200_idrs_solve_op", {1: "op", 2: "x", 3: "b"}),
    ("b200_qmr_solve_op", {1: "op", 2: "op", 3: "x", 4: "b"}), ("b200_lsqr_solve_op", {1: "op", 2: "op", 3: "x", 4: "b"}),
    ("b200_lsmr_solve_op", {1: "op", 2: "op", 3: "x", 4: "b"}), ("b200_lobpcg_solve_op", {1: "op", 3: "x"}),
    ("b200_svdl_op", {1: "op", 2: "op", 3: "x"}), ("b200_powm", {2: "op", 3: "x"}),
    ("b200_gmres_iter_create", {2: "op", 3: "x", 4: "b"}), ("b200_cg_iter_create_op", {2: "op", 3: "x", 4: "b"}),
    ("b200_orthogonalize_and_normalize", {2: "x", 5: "b", 8: "code"}),
    ("b200_lobpcg_constraint_create", {2: "x", 6: "code"}), ("b200_csr_laplacian", {3: "code"}),
    ("b200_csr_from_csr_slab", {8: "code"}),
]


@pytest.mark.parametrize("fn,roles", REJECT, ids=[f"{f}-{sorted(set(r.values()))[0]}" for f, r in REJECT])
def test_rejections(isb, fn, roles):
    ctx = isb.default_context()
    n = 64
    A = sp.identity(n, format="csr", dtype=np.complex128) * (2 + 1j)
    Ad = isb.B200CSR.from_scipy(A)
    op = isb.B200LinearOperator.from_csr(Ad)
    x0 = crand(np.random.default_rng(1), n)
    xd = isb.DeviceArray.from_numpy(ctx, x0)
    bd = isb.DeviceArray.from_numpy(ctx, x0)
    f = getattr(lib(isb), fn)
    args = []
    for i, t in enumerate(f.argtypes):
        role = "ctx" if i == 0 else roles.get(i)
        if role == "ctx":
            args.append(ctx._h)
        elif role == "A":
            args.append(Ad._h)
        elif role == "op":
            args.append(C.byref(op._c))
        elif role == "x":
            args.append(xd._p)
        elif role == "b":
            args.append(bd._p)
        elif role == "code":
            args.append(2)
        elif t in (C.c_int, C.c_int64, C.c_int32):
            args.append(1)
        elif t is C.c_double:
            args.append(0.0)
        else:
            args.append(None)
    assert f(*args) == UNSUPPORTED, lib(isb).b200_last_error()
    assert b"Complex" in lib(isb).b200_last_error()
    assert np.array_equal(xd.numpy(), x0)
