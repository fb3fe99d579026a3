"""Complex element types (ComplexF64 / ComplexF32) of the cg! and gmres! engines, checked without a GPU.

The fused-pass engines (csrc/cg_core.h, csrc/gmres_core.h) run on the serial CPU backend of tests/hostsim with their
complex instantiations (tests/hostsim_complex), and are compared with
  - the reference's own complex test cases (test/cg.jl:27-50, test/gmres.jl:16-57 and :75-99),
  - the oracle (oracle.gmres_ handles complex inputs; complex cg! is restated below with np.vdot, src/cg.jl:43-100),
  - the real engine on real data given as complex values, which must agree bit for bit (hostsim builds with
    -ffp-contract=off; multiplying by a zero imaginary part and Smith-dividing by one are exact; the complex
    givensAlgorithm differs from the real one only by exact sign flips of both rotated rows).
"""
import ctypes as C
import json
import math
import os
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
ORTH = {"mgs": 0, "cgs": 1, "dgks": 2}
_CLIB = None


def clib():
    """the complex instantiations of the engines on the serial backend (tests/hostsim_complex, built with make)"""
    global _CLIB
    if _CLIB is None:
        d = os.path.join(HERE, "hostsim_complex")
        subprocess.run(["make", "-s", "-C", d], check=True)
        _CLIB = C.CDLL(os.path.join(d, "libhostsim_complex.so"))
    return _CLIB


@pytest.fixture(scope="module")
def sim():
    from hostsim import sim as s
    s.lib()
    return s


def _vp(a):
    return C.c_void_p(a.ctypes.data) if a is not None else None


def cg_c(sim, x, A, b, *, Pl=None, diag=None, abstol=0.0, reltol=-1.0, maxiter=-1, initially_zero=False, order=0,
         split=0):
    """the complex instantiation of the cg engine on the serial backend (Pl: a matrix whose product is Pl \\ x)."""
    dt = x.dtype
    Ac = sim.Csr(A, dt)
    Pc = sim.Csr(Pl, dt) if Pl is not None else None
    b = np.ascontiguousarray(b, dtype=dt)
    d = None if diag is None else np.ascontiguousarray(diag, dtype=dt)
    cap = (maxiter if maxiter >= 0 else A.shape[1]) + 1
    hist = np.zeros(cap)
    out = sim._Out()
    st = clib().hostsim_cg_c(C.c_int(dt == np.complex128), C.byref(Ac.c), C.byref(Pc.c) if Pc else None, _vp(d),
                             _vp(x), _vp(b), C.c_double(abstol), C.c_double(reltol), C.c_int64(maxiter),
                             C.c_int(initially_zero), C.c_int(0), C.c_int64(cap), _vp(hist), C.c_int(order),
                             C.c_int(split), C.byref(out))
    assert st == 0, st
    return x, sim._outcome(out, hist)


def gmres_c(sim, x, A, b, *, Pl=None, Pr=None, pl_diag=None, pr_diag=None, abstol=0.0, reltol=-1.0, restart=-1,
            maxiter=-1, initially_zero=False, orth_meth="mgs", order=0, split=0):
    """the complex instantiation of the gmres engine on the serial backend."""
    dt = x.dtype
    Ac = sim.Csr(A, dt)
    Plc = sim.Csr(Pl, dt) if Pl is not None else None
    Prc = sim.Csr(Pr, dt) if Pr is not None else None
    b = np.ascontiguousarray(b, dtype=dt)
    dl = None if pl_diag is None else np.ascontiguousarray(pl_diag, dtype=dt)
    dr = None if pr_diag is None else np.ascontiguousarray(pr_diag, dtype=dt)
    cap = maxiter if maxiter >= 0 else A.shape[1]
    hist = np.zeros(max(cap, 1))
    out = sim._Out()
    st = clib().hostsim_gmres_c(C.c_int(dt == np.complex128), C.byref(Ac.c), C.byref(Plc.c) if Plc else None,
                                C.byref(Prc.c) if Prc else None, _vp(dl), _vp(dr), _vp(x), _vp(b),
                                C.c_double(abstol), C.c_double(reltol), C.c_int(restart), C.c_int64(maxiter),
                                C.c_int(initially_zero), C.c_int(ORTH[orth_meth]), C.c_int64(cap), _vp(hist),
                                C.c_int(order), C.c_int(split), C.byref(out))
    assert st == 0, st
    return x, sim._outcome(out, hist)


def cg_oracle_c(x, A, b, *, Pl=None, diag=None, abstol=0.0, reltol=None, maxiter=None, initially_zero=False):
    """cg!(x, A, b; Pl, ...) of reference src/cg.jl:43-100, 120-155, 209-242 for complex element types: dot(u, c) is
    np.vdot(u, c) = sum conj(u) c; alpha, rho and beta are complex, the residual real.  Pl: a matrix M with
    ldiv!(c, Pl, r) = M \\ r; diag: Jacobi diagonal."""
    A = sp.csr_matrix(A)
    n = A.shape[0]
    if reltol is None:
        reltol = math.sqrt(np.finfo(x.real.dtype).eps)
    if maxiter is None:
        maxiter = n
    u = np.zeros_like(x)
    r = b.astype(x.dtype, copy=True)
    mvps = 0
    if not initially_zero:
        mvps = 1
        r -= A @ x
    residual = float(np.linalg.norm(r))
    tol = max(reltol * residual, abstol)
    prev_residual, rho = 1.0, 1.0 + 0j
    precond = Pl is not None or diag is not None
    hist, it = [], 0
    while not (it >= maxiter or residual <= tol):                      # :36
        if precond:
            c = np.linalg.solve(Pl, r) if Pl is not None else r / diag  # :79
            rho_prev, rho = rho, np.vdot(c, r)                          # :81-82
            u[...] = c + (rho / rho_prev) * u                           # :85-86
            c = A @ u                                                   # :89
            alpha = rho / np.vdot(u, c)                                 # :90
        else:
            u[...] = r + (residual ** 2 / prev_residual ** 2) * u       # :50-51
            c = A @ u                                                   # :54
            alpha = residual ** 2 / np.vdot(u, c)                       # :55
        x += alpha * u
        r -= alpha * c
        prev_residual = residual
        residual = float(np.linalg.norm(r))
        hist.append(residual)
        it += 1
    return x, dict(iters=it, mvps=mvps + it, resnorm=np.array(hist), converged=residual <= tol)


# ------------------------------------------------------------------------------------------------ operators
def laplace2d(N):
    T = sp.diags([-np.ones(N - 1), 2 * np.ones(N), -np.ones(N - 1)], [-1, 0, 1])
    I = sp.identity(N)
    return (sp.kron(I, T) + sp.kron(T, I)).tocsr()


def hpd_operator(N=12):
    """L + I + i S: L the 2-D Laplacian, S the real antisymmetric central difference in x with coefficient 1/4
    (i S is Hermitian, so the operator is Hermitian positive definite with every eigenvalue >= 1/2)."""
    L = laplace2d(N)
    D = sp.diags([-np.ones(N - 1), np.ones(N - 1)], [-1, 1]) * 0.25
    S = sp.kron(sp.identity(N), D)
    return (L + sp.identity(N * N) + 1j * S).tocsr()


def helmholtz_operator(N=10, k2=0.5, sigma=0.5):
    """the shifted Helmholtz operator -Laplace - k^2 I + i sigma I with a convection term: complex, non-Hermitian."""
    L = laplace2d(N)
    D = sp.diags([-np.ones(N - 1), np.ones(N - 1)], [-1, 1]) * 0.3
    C_ = sp.kron(sp.identity(N), D)
    return (L - k2 * sp.identity(N * N) + 1j * sigma * sp.identity(N * N) + C_).tocsr()


def crand(rng, shape, dt=np.complex128):
    return (rng.random(shape) + 1j * rng.random(shape)).astype(dt)


# ------------------------------------------------------------------------------------------------ reference cases
@pytest.mark.parametrize("dt", [np.complex64, np.complex128])
def test_reference_cg_small_full_system(sim, dt):
    """test/cg.jl:27-50 on the engine: A = A'A + I, convergence, exact start, Cholesky Pl, zero right-hand side."""
    rng = np.random.default_rng(1234321)
    n = 10
    A = crand(rng, (n, n), dt)
    A = (A.conj().T @ A + np.eye(n)).astype(dt)
    b = crand(rng, n, dt)
    reltol = math.sqrt(np.finfo(np.zeros(1, dt).real.dtype).eps)
    x, o = cg_c(sim, np.zeros(n, dt), sp.csr_matrix(A), b, reltol=reltol, maxiter=2 * n, initially_zero=True)
    assert np.linalg.norm(A @ x - b) / np.linalg.norm(b) <= reltol and o.converged
    eps = np.finfo(np.zeros(1, dt).real.dtype).eps
    x0 = np.linalg.solve(A.astype(np.complex128), b.astype(np.complex128)).astype(dt)
    x, o = cg_c(sim, x0.copy(), sp.csr_matrix(A), b, abstol=2 * n * eps, reltol=0.0)
    assert o.iters <= 1 and o.mvps <= 2
    Pinv = np.linalg.inv(A.astype(np.complex128)).astype(dt)          # Pl = cholesky(A): ldiv! is the exact inverse
    x, o = cg_c(sim, np.zeros(n, dt), sp.csr_matrix(A), b, Pl=sp.csr_matrix(Pinv), initially_zero=True)
    assert o.iters <= 2 and o.mvps <= 2
    x, o = cg_c(sim, np.zeros(n, dt), sp.csr_matrix(A), np.zeros(n, dt), initially_zero=True)
    assert np.all(x == 0) and o.iters == 0


@pytest.mark.parametrize("dt", [np.complex64, np.complex128])
def test_reference_gmres_small_full_system(sim, dt):
    """test/gmres.jl:16-34: non-increasing history, exact left and right preconditioners."""
    rng = np.random.default_rng(1234321)
    n = 10
    A = (crand(rng, (n, n), dt) + np.eye(n)).astype(dt)
    b = crand(rng, n, dt)
    Finv = sp.csr_matrix(np.linalg.inv(A.astype(np.complex128)).astype(dt))
    reltol = math.sqrt(np.finfo(np.zeros(1, dt).real.dtype).eps)
    for meth in ORTH:
        x, o = gmres_c(sim, np.zeros(n, dt), sp.csr_matrix(A), b, restart=3, maxiter=10, reltol=reltol,
                       initially_zero=True, orth_meth=meth)
        assert np.all(np.diff(o.hist) <= 0.0)
        x, o = gmres_c(sim, np.zeros(n, dt), sp.csr_matrix(A), b, Pl=Finv, maxiter=1, restart=1, reltol=reltol,
                       initially_zero=True, orth_meth=meth)
        assert o.converged
        assert np.linalg.norm(Finv @ (A @ x - b)) / np.linalg.norm(b) <= reltol
        x, o = gmres_c(sim, np.zeros(n, dt), sp.csr_matrix(A), b, Pr=Finv, maxiter=1, restart=1, reltol=reltol,
                       initially_zero=True, orth_meth=meth)
        assert o.converged
        assert np.linalg.norm(A @ x - b) / np.linalg.norm(b) <= reltol


@pytest.mark.parametrize("dt", [np.complex64, np.complex128])
def test_reference_gmres_termination(sim, dt):
    """test/gmres.jl:75-99: a small initial residual needs 2..n iterations with the default tolerance and none
    with an absolute tolerance above it."""
    A = np.array([[2, -1, 0], [-1, 2, -1], [0, -1, 2]], dtype=dt)
    n = 3
    b = np.ones(n, dt)
    x0 = np.linalg.solve(A, b).astype(dt)
    pert = (10 * math.sqrt(np.finfo(np.zeros(1, dt).real.dtype).eps) * np.array([(-1) ** i for i in range(1, n + 1)])).astype(dt)
    x, o = gmres_c(sim, (x0 + pert).astype(dt), sp.csr_matrix(A), b)
    assert 2 <= o.iters <= n
    x = (x0 + pert).astype(dt)
    r0 = float(np.linalg.norm(A @ x - b))
    x, o = gmres_c(sim, x, sp.csr_matrix(A), b, abstol=2 * r0, reltol=0.0)
    assert o.iters == 0


# ------------------------------------------------------------------------------------------------ against the oracle
def _cg_precs(A):
    d = A.diagonal()
    M = sp.diags([np.full(A.shape[0] - 1, -0.5), d, np.full(A.shape[0] - 1, -0.5)], [-1, 0, 1]).toarray().astype(np.complex128)
    return {"identity": {}, "jacobi": {"diag": d}, "callback": {"Pl": M}}


@pytest.mark.parametrize("prec", ["identity", "jacobi", "callback"])
@pytest.mark.parametrize("order,split", [(0, 0), (1, 0), (0, 1)])
def test_cg_engine_matches_oracle(sim, prec, order, split):
    A = hpd_operator(12)
    n = A.shape[0]
    rng = np.random.default_rng(7)
    b = crand(rng, n)
    kw = _cg_precs(A)[prec]
    xo, ho = cg_oracle_c(np.zeros(n, np.complex128), A, b, **kw, initially_zero=True)
    skw = {"diag": kw["diag"]} if "diag" in kw else ({"Pl": sp.csr_matrix(np.linalg.inv(kw["Pl"]))} if "Pl" in kw else {})
    x, o = cg_c(sim, np.zeros(n, np.complex128), A, b, **skw, initially_zero=True, order=order, split=split)
    assert o.iters == ho["iters"] and o.mvps == ho["mvps"] and o.converged
    r0 = np.linalg.norm(b)
    assert float(np.max(np.abs(o.hist - ho["resnorm"]))) / r0 <= 1e-11
    assert np.linalg.norm(x - xo) / np.linalg.norm(xo) <= 1e-11


@pytest.mark.parametrize("meth", ["mgs", "cgs", "dgks"])
@pytest.mark.parametrize("restart", [5, 20])
@pytest.mark.parametrize("pl", ["identity", "jacobi", "callback"])
@pytest.mark.parametrize("pr", ["identity", "jacobi", "callback"])
def test_gmres_engine_matches_oracle(sim, meth, restart, pl, pr):
    A = helmholtz_operator(10)
    n = A.shape[0]
    rng = np.random.default_rng(11)
    b = crand(rng, n)
    d = A.diagonal()
    M = sp.diags([np.full(n - 1, 0.3 - 0.1j), d, np.full(n - 1, -0.2j)], [-1, 0, 1]).toarray()
    oracle_prec = {"identity": None, "jacobi": O.JacobiPrec(d), "callback": O.MatrixPrec(M)}
    sim_kw = {}
    for side, p in (("l", pl), ("r", pr)):
        if p == "jacobi":
            sim_kw["p%s_diag" % side] = d
        elif p == "callback":
            sim_kw["P" + side] = sp.csr_matrix(np.linalg.inv(M))
    maxiter = 60
    xo, ho = O.gmres_(np.zeros(n, np.complex128), A, b, Pl=oracle_prec[pl], Pr=oracle_prec[pr], restart=restart,
                      maxiter=maxiter, log=True, initially_zero=True, orth_meth=meth)
    order = 1 if (pl, pr) == ("jacobi", "callback") else 0
    x, o = gmres_c(sim, np.zeros(n, np.complex128), A, b, restart=restart, maxiter=maxiter, initially_zero=True,
                   orth_meth=meth, order=order, **sim_kw)
    hist_o = np.asarray(ho["resnorm"])
    assert o.iters == ho.iters and o.mvps == ho.mvps
    assert float(np.max(np.abs(o.hist - hist_o))) / hist_o[0] <= 1e-13 if hist_o.size else True
    assert np.linalg.norm(x - xo) / np.linalg.norm(xo) <= 1e-13


def test_complexf32_engines_stated_tolerance(sim):
    """ComplexF32 vectors with fp64 scalars: the solution agrees with the fp64 oracle's to 1e-4 relative."""
    A = hpd_operator(10)
    n = A.shape[0]
    b = crand(np.random.default_rng(3), n)
    xo, _ = cg_oracle_c(np.zeros(n, np.complex128), A, b, reltol=1e-6, initially_zero=True)
    x, o = cg_c(sim, np.zeros(n, np.complex64), A, b, reltol=1e-6, initially_zero=True)
    assert o.converged and np.linalg.norm(x - xo) / np.linalg.norm(xo) <= 1e-4
    H = helmholtz_operator(8)
    b = crand(np.random.default_rng(4), H.shape[0])
    xo, _ = O.gmres_(np.zeros(H.shape[0], np.complex128), H, b, restart=20, maxiter=200, reltol=1e-6, log=True,
                     initially_zero=True, orth_meth="dgks")
    x, o = gmres_c(sim, np.zeros(H.shape[0], np.complex64), H, b, restart=20, maxiter=200, reltol=1e-6,
                   initially_zero=True, orth_meth="dgks")
    assert o.converged and np.linalg.norm(x - xo) / np.linalg.norm(xo) <= 1e-4


def test_hessenberg_h2_fixture(sim):
    """the engine's complex least-squares solve on the reference's complex Hessenberg fixture H2
    (test/hessenberg.jl:18-26) matches oracle.hessenberg_ldiv."""
    with open(os.path.join(GOLDEN, "hessenberg_fixtures.json")) as f:
        g = json.load(f)
    H2 = np.array(g["H2_re"], dtype=np.float64) + 1j * np.array(g["H2_im"], dtype=np.float64)
    m = H2.shape[1]
    rhs = np.zeros(m + 1, np.complex128)
    rhs[0] = 1
    want = O.hessenberg_ldiv(H2.copy(), rhs.copy())
    H = np.asfortranarray(H2.copy())
    got = rhs.copy()
    clib().hostsim_hessenberg_c(C.c_void_p(H.ctypes.data), C.c_int(m + 1), C.c_int(m), C.c_void_p(got.ctypes.data))
    assert float(np.max(np.abs(got - want))) / float(np.max(np.abs(want))) <= 1e-14


# ------------------------------------------------------------------------------------------------ real data as complex
def _real_ops():
    L = laplace2d(10)
    A = (L + 0.1 * sp.identity(100)).tocsr()
    Anon = (L + sp.diags([np.full(99, 0.4)], [1]) - 0.3 * sp.identity(100)).tocsr()
    return A, Anon


@pytest.mark.parametrize("prec", ["identity", "jacobi", "callback"])
def test_cg_real_data_as_complex_bitwise(sim, prec):
    A, _ = _real_ops()
    n = A.shape[0]
    b = np.random.default_rng(5).random(n)
    kw = {"identity": {}, "jacobi": {"diag": A.diagonal()},
          "callback": {"Pl": sp.csr_matrix(np.linalg.inv(sp.diags([np.full(n - 1, -0.5), A.diagonal(), np.full(n - 1, -0.5)], [-1, 0, 1]).toarray()))}}[prec]
    xr, orr = sim.cg_(np.zeros(n), A, b, initially_zero=True, **kw)
    ckw = {k: (v.astype(np.complex128) if isinstance(v, np.ndarray) else v.astype(np.complex128)) for k, v in kw.items()}
    xc, oc = cg_c(sim, np.zeros(n, np.complex128), A.astype(np.complex128), b.astype(np.complex128), initially_zero=True, **ckw)
    assert (oc.iters, oc.mvps, oc.converged) == (orr.iters, orr.mvps, orr.converged)
    assert np.array_equal(oc.hist, orr.hist)
    assert np.array_equal(xc.real, xr) and np.all(xc.imag == 0)


@pytest.mark.parametrize("meth", ["mgs", "cgs", "dgks"])
@pytest.mark.parametrize("restart", [5, 20])
@pytest.mark.parametrize("precs", [("identity", "identity"), ("jacobi", "callback"), ("callback", "jacobi")])
def test_gmres_real_data_as_complex_bitwise(sim, meth, restart, precs):
    _, A = _real_ops()
    n = A.shape[0]
    b = np.random.default_rng(6).random(n)
    d = A.diagonal()
    Minv = np.linalg.inv(sp.diags([np.full(n - 1, 0.3), d, np.full(n - 1, -0.2)], [-1, 0, 1]).toarray())
    kw = {}
    for side, p in zip("lr", precs):
        if p == "jacobi":
            kw["p%s_diag" % side] = d
        elif p == "callback":
            kw["P" + side] = sp.csr_matrix(Minv)
    xr, orr = sim.gmres_(np.zeros(n), A, b, restart=restart, maxiter=80, initially_zero=True, orth_meth=meth, **kw)
    ckw = {k: v.astype(np.complex128) for k, v in kw.items()}
    xc, oc = gmres_c(sim, np.zeros(n, np.complex128), A.astype(np.complex128), b.astype(np.complex128), restart=restart,
                     maxiter=80, initially_zero=True, orth_meth=meth, **ckw)
    assert (oc.iters, oc.mvps, oc.converged) == (orr.iters, orr.mvps, orr.converged)
    assert np.array_equal(oc.hist, orr.hist)
    assert np.array_equal(xc.real, xr) and np.all(xc.imag == 0)
