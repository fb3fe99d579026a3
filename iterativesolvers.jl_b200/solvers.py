"""Solver entry points with the reference's names, keywords, defaults and return shapes.

    cg!(x, A, b; kw...)  ->  cg_(x, A, b, **kw)        (Python has no `!`)
    cg(A, b; kw...)      ->  cg(A, b, **kw)

`A` is a B200CSR; `x`, `b` are either host numpy arrays (copied to the GPU and back inside the call:
the end-to-end path) or device arrays (DeviceArray / contiguous torch CUDA tensors, zero-copy).
`x` is updated in place and returned as the same object (reference src/cg.jl:241).
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass

import numpy as np

from . import _lib
from ._lib import B200Error, check, lib
from .device import DeviceArray, as_device_ptr, dtype_code, is_device
from .history import ConvergenceHistory
from .operators import B200CSR, B200LinearOperator, FunctionPrec, Identity, precond_to_c


def _eps(dtype):
    return float(np.finfo(np.dtype(dtype)).eps)


def _check_operator(A, linop_ok=False):
    if isinstance(A, B200CSR) or (linop_ok and isinstance(A, B200LinearOperator)):
        return
    raise TypeError("the device path needs a B200CSR operator (B200CSR.from_scipy / from_csc_arrays)"
                    + (" or a B200LinearOperator" if linop_ok else ""))


def _is_linop(A):
    return isinstance(A, B200LinearOperator)


def _call_op(fn, ops, *args):
    """call a *_op entry point; re-raise an exception a Python callback stored while C frames were on the stack."""
    status = fn(*args)
    for o in ops:
        if o is not None:
            o.raise_pending()
    return status


class _Staged:
    """host<->device staging of the (x, b) pair of a solve call."""

    def __init__(self, A: B200CSR, x, b):
        self.host = not is_device(x)
        self.x, self.b = x, b
        if self.host:
            if is_device(b):
                raise TypeError("x and b must both be host arrays or both be device arrays")
            if not (isinstance(x, np.ndarray) and x.dtype == A.dtype):
                raise TypeError(f"x must be a numpy array of eltype {A.dtype} (got {getattr(x, 'dtype', type(x))})")
            self.xd = DeviceArray.from_numpy(A.ctx, x)
            self.bd = DeviceArray.from_numpy(A.ctx, np.asarray(b, dtype=A.dtype))
        else:
            self.xd, self.bd = x, b
        if self._len(self.xd) != A.m_local or self._len(self.bd) != A.m_local:
            raise ValueError("dimension mismatch between A, x and b")

    @staticmethod
    def _len(v):
        return v.shape[0]

    def finish(self):
        if self.host:
            self.x[...] = self.xd.numpy().reshape(self.x.shape)
        return self.x


def _history(res: _lib.Result, resnorm, abstol, reltol, log, restart=None):
    h = ConvergenceHistory(restart=restart)
    h["abstol"], h["reltol"] = abstol, reltol
    h.isconverged = bool(res.isconverged)
    if log:
        h.mvps, h.iters = int(res.mvps), int(res.iters)
        h["resnorm"] = resnorm[: res.n_resnorm].copy()
        h["tol"] = res.tol
    return h


# ------------------------------------------------------------------------------------------------
# CG  (reference src/cg.jl:162, 209-242)
# ------------------------------------------------------------------------------------------------
def cg_(x, A, b, *, abstol=0.0, reltol=None, maxiter=None, log=False, verbose=False, Pl=None,
        initially_zero=False, statevars=None, check_every=0, _fixed_iterations=False):
    """cg!(x, A, b; abstol, reltol, maxiter, log, statevars, verbose, Pl, initially_zero).
    With `statevars` (CGStateVariables of three device vectors) the solve runs through the iterator form of the
    engine on the caller's u, r, c -- exactly `cg_iterator!(...; statevars)` driven to done() (src/cg.jl:224-236)."""
    _check_operator(A, linop_ok=True)
    if reltol is None:
        reltol = math.sqrt(_eps(A.dtype))                     # src/cg.jl:211
    if maxiter is None:
        maxiter = A.size(2)                                   # src/cg.jl:212
    if _is_linop(A) or isinstance(Pl, FunctionPrec):
        # general operator / preconditioner: the pass-based engine (csrc/cg_core.h) with device callbacks
        if statevars is not None or _fixed_iterations:
            raise TypeError("statevars / _fixed_iterations are only available for B200CSR operators")
        op = A if _is_linop(A) else B200LinearOperator.from_csr(A)
        pl = Pl.op if isinstance(Pl, FunctionPrec) else None
        opts = _lib.CgOpts(abstol, reltol, int(maxiter), int(bool(initially_zero)), int(check_every),
                           precond_to_c(None if pl is not None else Pl, A), 0, 0)
        res = _lib.Result()
        cap = int(maxiter) + 1 if log else 0
        resnorm = np.zeros(max(cap, 1), dtype=np.float64)
        st = _Staged(A, x, b)
        check(_call_op(lib().b200_cg_solve_op, (op, pl), A.ctx._h, C.byref(op._c), C.byref(pl._c) if pl else None,
                       as_device_ptr(st.xd), as_device_ptr(st.bd), C.byref(opts), C.byref(res),
                       resnorm.ctypes.data_as(C.c_void_p) if log else None, cap))
        st.finish()
        cg_.last_result = res
        return (x, _history(res, resnorm, abstol, reltol, log)) if log else x
    if statevars is not None:
        it = cg_iterator_(x, A, b, abstol=abstol, reltol=reltol, maxiter=maxiter, statevars=statevars, Pl=Pl,
                          initially_zero=initially_zero)
        resnorm = []
        while not it.done:
            resnorm.extend(it.step(4096))
        res = it.result
        it.close()
        cg_.last_result = res
        h = ConvergenceHistory()
        h["abstol"], h["reltol"] = abstol, reltol
        h.isconverged = bool(res.isconverged)
        if log:
            h.mvps, h.iters = int(res.mvps), int(res.iters)
            h["resnorm"] = np.array(resnorm, dtype=np.float64)
            h["tol"] = res.tol
        return (x, h) if log else x
    opts = _lib.CgOpts(abstol, reltol, int(maxiter), int(bool(initially_zero)), int(check_every),
                       precond_to_c(Pl, A), int(bool(_fixed_iterations)), 0)
    res = _lib.Result()
    cap = int(maxiter) + 1 if log else 0                      # reserve!(history, :resnorm, maxiter+1)  :221
    resnorm = np.zeros(max(cap, 1), dtype=np.float64)
    rp = resnorm.ctypes.data_as(C.c_void_p) if log else None
    if not is_device(x) and isinstance(x, np.ndarray) and x.ndim == 1 and x.flags.c_contiguous and x.dtype == A.dtype:
        bh = np.ascontiguousarray(b, dtype=A.dtype)
        if bh.shape != x.shape or x.shape[0] != A.m_local:
            raise ValueError("dimension mismatch between A, x and b")
        check(lib().b200_cg_solve_host(A.ctx._h, A._h, x.ctypes.data_as(C.c_void_p), bh.ctypes.data_as(C.c_void_p),
                                       C.byref(opts), C.byref(res), rp, cap))
    else:
        st = _Staged(A, x, b)
        check(lib().b200_cg_solve(A.ctx._h, A._h, as_device_ptr(st.xd), as_device_ptr(st.bd), C.byref(opts),
                                  C.byref(res), rp, cap))
        st.finish()
    if verbose:
        for i, r in enumerate(resnorm[: res.n_resnorm]):
            print(f"{i + 1:3d}\t{r:1.2e}")
        print()
    cg_.last_result = res
    return (x, _history(res, resnorm, abstol, reltol, log)) if log else x


class CGStateVariables:
    """CGStateVariables(u, r, c) -- reference src/cg.jl:114-118: three vectors similar to x that hold the
    intermediate results of the iteration; here three DeviceArrays of the operator's eltype and local length."""

    def __init__(self, u, r, c):
        for v in (u, r, c):
            if not is_device(v):
                raise TypeError("CGStateVariables holds device vectors (DeviceArray)")
        self.u, self.r, self.c = u, r, c


class CGIterable:
    """The object `cg_iterator!` returns (CGIterable / PCGIterable, reference src/cg.jl:5-30): iterating it yields
    the residual norm after each step (src/cg.jl:65, :99) and leaves x updated in place; `step(k)` performs up to k
    steps in one call (one launch batch, one host synchronisation)."""

    def __init__(self, x, A, b, opts, statevars):
        self._A, self._x = A, x
        self._st = _Staged(A, x, b)
        self._sv = statevars                                   # keep the state vectors alive
        sv = statevars
        self._h = C.c_void_p()
        check(lib().b200_cg_iter_create(A.ctx._h, A._h, as_device_ptr(self._st.xd), as_device_ptr(self._st.bd),
                                        C.byref(opts), as_device_ptr(sv.u) if sv else None,
                                        as_device_ptr(sv.r) if sv else None, as_device_ptr(sv.c) if sv else None,
                                        C.byref(self._h)))
        self.result = _lib.Result()
        self._buf = np.zeros(4096, dtype=np.float64)
        self.step(0)                                           # residual / tol of the initial state

    # -- reference field names -------------------------------------------------------------------
    @property
    def residual(self):
        return float(self.result.residual)

    @property
    def tol(self):
        return float(self.result.tol)

    @property
    def iteration(self):
        return int(self.result.iters)

    @property
    def mv_products(self):
        return int(self.result.mvps)

    @property
    def converged(self):                                       # converged(it)  src/cg.jl:32-34
        return bool(self.result.isconverged)

    @property
    def done(self):                                            # done(it, iteration)  src/cg.jl:36
        return self.result.status == 1

    @property
    def x(self):
        return self._x

    def step(self, k=1):
        """up to k calls of iterate(it); returns the residual norms of the steps performed."""
        if self._h is None:
            raise RuntimeError("iterator is closed")
        k = int(k)
        out = []
        while True:
            kk = min(k, 4096)
            check(lib().b200_cg_iter_next(self._h, kk, C.byref(self.result), self._buf.ctypes.data_as(C.c_void_p), 4096))
            out.extend(self._buf[: self.result.n_resnorm].tolist())
            k -= kk
            if k <= 0 or self.done:
                break
        self._st.finish()                                      # host x: copy the completed iterate back
        return out

    def __iter__(self):
        return self

    def __next__(self):
        if self.done:
            raise StopIteration
        r = self.step(1)
        if not r:
            raise StopIteration
        return r[0]

    def close(self):
        if self._h is not None:
            lib().b200_cg_iter_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def cg_iterator_(x, A, b, *, abstol=0.0, reltol=None, maxiter=None, statevars=None, Pl=None, initially_zero=False):
    """cg_iterator!(x, A, b, Pl = Identity(); abstol, reltol, maxiter, statevars, initially_zero)
    -- reference src/cg.jl:120-155.  A B200CSR with Identity / JacobiPrec gives the tuned iterator (optionally on the
    caller's CGStateVariables); a B200LinearOperator or a FunctionPrec gives the general one (a KrylovIterable)."""
    _check_operator(A, linop_ok=True)
    if reltol is None:
        reltol = math.sqrt(_eps(A.dtype))
    if maxiter is None:
        maxiter = A.size(2)
    opts = _lib.CgOpts(abstol, reltol, int(maxiter), int(bool(initially_zero)), 0, precond_to_c(Pl, A), 0, 0)
    if _is_linop(A) or isinstance(Pl, FunctionPrec):
        if statevars is not None:
            raise B200Error("statevars are taken by the tuned iterator only (B200CSR with Identity / JacobiPrec)")
        keep = [A] + ([Pl] if Pl is not None else []) + ([Pl.op] if isinstance(Pl, FunctionPrec) else [])
        return KrylovIterable(lib().b200_cg_iter_create_op, x, A, b, opts, keep)
    return CGIterable(x, A, b, opts, statevars)


def cg(A, b, **kw):
    """cg(A, b; kw...) = cg!(zerox(A, b), A, b; initially_zero = true, kw...)  (src/cg.jl:162)."""
    _check_operator(A, linop_ok=True)
    if is_device(b):
        x = DeviceArray.zeros(A.ctx, A.m_local, A.dtype)
    else:
        x = np.zeros(A.m_local, dtype=A.dtype)
    return cg_(x, A, b, initially_zero=True, **kw)


# ------------------------------------------------------------------------------------------------
# Chebyshev iteration  (reference src/chebyshev.jl:117-160)
# ------------------------------------------------------------------------------------------------
def chebyshev_(x, A, b, lmin, lmax, *, abstol=0.0, reltol=None, Pl=None, maxiter=None, log=False, verbose=False,
               initially_zero=False):
    """chebyshev!(x, A, b, λmin, λmax; abstol, reltol, Pl, maxiter, log, verbose, initially_zero).
    A: B200CSR or B200LinearOperator; Pl: Identity, JacobiPrec or FunctionPrec (callbacks: the general engine)."""
    _check_operator(A, linop_ok=True)
    if reltol is None:
        reltol = math.sqrt(_eps(A.dtype))
    if maxiter is None:
        maxiter = A.size(2)
    opts = _lib.CgOpts(abstol, reltol, int(maxiter), int(bool(initially_zero)), 0, precond_to_c(Pl, A), 0, 0)
    res = _lib.Result()
    cap = int(maxiter)                                          # reserve!(history, :resnorm, maxiter)  :144
    resnorm = np.zeros(max(cap, 1), dtype=np.float64)
    st = _Staged(A, x, b)
    cbs = (Pl.op,) if isinstance(Pl, FunctionPrec) else ()
    if _is_linop(A):
        check(_call_op(lib().b200_chebyshev_solve_op, (A,) + cbs, A.ctx._h, C.byref(A._c), as_device_ptr(st.xd),
                       as_device_ptr(st.bd), float(lmin), float(lmax), C.byref(opts), C.byref(res),
                       resnorm.ctypes.data_as(C.c_void_p), cap))
    else:
        check(_call_op(lib().b200_chebyshev_solve, cbs, A.ctx._h, A._h, as_device_ptr(st.xd), as_device_ptr(st.bd),
                       float(lmin), float(lmax), C.byref(opts), C.byref(res), resnorm.ctypes.data_as(C.c_void_p), cap))
    st.finish()
    if verbose:
        print("=== chebyshev ===\niter\tresnorm")
        for i, r in enumerate(resnorm[: res.n_resnorm], start=1):
            print(f"{i:3d}\t{r:1.2e}")
        print()
    h = _history(res, resnorm, abstol, reltol, True)            # mvps / setconv are always recorded (:146-155)
    return (x, h) if log else x


def chebyshev(A, b, lmin, lmax, **kw):
    _check_operator(A, linop_ok=True)
    x = DeviceArray.zeros(A.ctx, A.m_local, A.dtype) if is_device(b) else np.zeros(A.m_local, dtype=A.dtype)
    return chebyshev_(x, A, b, lmin, lmax, initially_zero=True, **kw)


# ------------------------------------------------------------------------------------------------
# GMRES  (reference src/gmres.jl:143, 184-222)
# ------------------------------------------------------------------------------------------------
_ORTH = {"mgs": _lib.ORTH_MGS, "cgs": _lib.ORTH_CGS, "dgks": _lib.ORTH_DGKS,
         "ModifiedGramSchmidt": _lib.ORTH_MGS, "ClassicalGramSchmidt": _lib.ORTH_CGS, "DGKS": _lib.ORTH_DGKS}


def gmres_(x, A, b, *, Pl=None, Pr=None, abstol=0.0, reltol=None, restart=None, maxiter=None, log=False,
           initially_zero=False, verbose=False, orth_meth="mgs"):
    """gmres!(x, A, b; Pl, Pr, abstol, reltol, restart, maxiter, log, initially_zero, verbose, orth_meth).
    A: B200CSR or B200LinearOperator (`mul!` by callback); Pl / Pr: Identity, JacobiPrec or FunctionPrec (`ldiv!` by
    callback).  A B200CSR with Identity / Jacobi runs the tuned engine, everything else the general one."""
    _check_operator(A, linop_ok=True)
    if reltol is None:
        reltol = math.sqrt(_eps(A.dtype))
    if restart is None:
        restart = min(20, A.size(2))                          # src/gmres.jl:189
    if maxiter is None:
        maxiter = A.size(2)
    opts = _lib.GmresOpts(abstol, reltol, int(maxiter), int(restart), int(bool(initially_zero)), _ORTH[orth_meth], 0,
                          precond_to_c(Pl, A), precond_to_c(Pr, A))
    res = _lib.Result()
    cap = int(maxiter) if log else 0                          # reserve!(history, :resnorm, maxiter)  :198
    resnorm = np.zeros(max(cap, 1), dtype=np.float64)
    st = _Staged(A, x, b)
    rp = resnorm.ctypes.data_as(C.c_void_p) if log else None
    cbs = tuple(P.op for P in (Pl, Pr) if isinstance(P, FunctionPrec))
    if _is_linop(A):
        check(_call_op(lib().b200_gmres_solve_op, (A,) + cbs, A.ctx._h, C.byref(A._c), as_device_ptr(st.xd),
                       as_device_ptr(st.bd), C.byref(opts), C.byref(res), rp, cap))
    else:
        check(_call_op(lib().b200_gmres_solve, cbs, A.ctx._h, A._h, as_device_ptr(st.xd), as_device_ptr(st.bd),
                       C.byref(opts), C.byref(res), rp, cap))
    st.finish()
    if verbose:
        print("=== gmres ===\nrest\titer\tresnorm")
        for i, r in enumerate(resnorm[: res.n_resnorm], start=1):
            print(f"{1 + (i - 1) // restart:3d}\t{1 + (i - 1) % restart:3d}\t{r:1.2e}")
        print()
    h = _history(res, resnorm, abstol, reltol, log, restart=restart)   # setconv always (src/gmres.jl:218)
    return (x, h) if log else x


def gmres(A, b, **kw):
    _check_operator(A, linop_ok=True)
    x = DeviceArray.zeros(A.ctx, A.m_local, A.dtype) if is_device(b) else np.zeros(A.m_local, dtype=A.dtype)
    return gmres_(x, A, b, initially_zero=True, **kw)


# ------------------------------------------------------------------------------------------------
# MINRES  (reference src/minres.jl:200-244)
# ------------------------------------------------------------------------------------------------
def minres_(x, A, b, *, skew_hermitian=False, verbose=False, log=False, abstol=0.0, reltol=None, maxiter=None,
            initially_zero=False):
    """minres!(x, A, b; skew_hermitian, verbose, log, abstol, reltol, maxiter, initially_zero) -- reference
    src/minres.jl:200-207.  A: B200CSR (tuned engine) or B200LinearOperator (`mul!` by callback: general engine)."""
    _check_operator(A, linop_ok=True)
    if reltol is None:
        reltol = math.sqrt(_eps(A.dtype))
    if maxiter is None:
        maxiter = A.size(2)
    opts = _lib.MinresOpts(abstol, reltol, int(maxiter), int(bool(initially_zero)), int(bool(skew_hermitian)))
    res = _lib.Result()
    cap = int(maxiter) if log else 0
    resnorm = np.zeros(max(cap, 1), dtype=np.float64)
    st = _Staged(A, x, b)
    rp = resnorm.ctypes.data_as(C.c_void_p) if log else None
    if _is_linop(A):
        check(_call_op(lib().b200_minres_solve_op, (A,), A.ctx._h, C.byref(A._c), as_device_ptr(st.xd),
                       as_device_ptr(st.bd), C.byref(opts), C.byref(res), rp, cap))
    else:
        check(lib().b200_minres_solve(A.ctx._h, A._h, as_device_ptr(st.xd), as_device_ptr(st.bd), C.byref(opts),
                                      C.byref(res), rp, cap))
    st.finish()
    if verbose:
        for i, r in enumerate(resnorm[: res.n_resnorm], start=1):
            print(f"{i:3d}\t{r:1.2e}")
        print()
    return (x, _history(res, resnorm, abstol, reltol, log)) if log else x


def minres(A, b, **kw):
    _check_operator(A, linop_ok=True)
    x = DeviceArray.zeros(A.ctx, A.m_local, A.dtype) if is_device(b) else np.zeros(A.m_local, dtype=A.dtype)
    return minres_(x, A, b, initially_zero=True, **kw)


# ------------------------------------------------------------------------------------------------
# BiCGStab(l)  (reference src/bicgstabl.jl:143, 181-219)
# ------------------------------------------------------------------------------------------------
def bicgstabl_(x, A, b, l=2, *, abstol=0.0, reltol=None, max_mv_products=None, log=False, verbose=False, Pl=None,
               initial_zero=False, r_shadow=None, rng=None):
    """bicgstabl!(x, A, b, l; ...).  The reference draws r_shadow = rand(T, n) (src/bicgstabl.jl:38);
    here the draw happens on the host (numpy Generator `rng`) unless `r_shadow` is given.
    A: B200CSR or B200LinearOperator; Pl: Identity, JacobiPrec or FunctionPrec (`ldiv!` by callback).  A B200CSR with
    Identity / Jacobi runs the tuned engine, everything else the general one (l <= 8)."""
    _check_operator(A, linop_ok=True)
    if reltol is None:
        reltol = math.sqrt(_eps(A.dtype))
    if max_mv_products is None:
        max_mv_products = A.size(2)
    if r_shadow is None:
        rng = rng or np.random.default_rng()
        r_shadow = rng.random(A.m_local).astype(A.dtype)
    rs = r_shadow if is_device(r_shadow) else DeviceArray.from_numpy(A.ctx, np.asarray(r_shadow, dtype=A.dtype))
    opts = _lib.BicgstablOpts(abstol, reltol, int(max_mv_products), int(l), int(bool(initial_zero)),
                              precond_to_c(Pl, A), as_device_ptr(rs))
    res = _lib.Result()
    cap = int(max_mv_products) if log else 0                  # src/bicgstabl.jl:194
    resnorm = np.zeros(max(cap, 1), dtype=np.float64)
    st = _Staged(A, x, b)
    rp = resnorm.ctypes.data_as(C.c_void_p) if log else None
    cbs = (Pl.op,) if isinstance(Pl, FunctionPrec) else ()
    if _is_linop(A):
        status = _call_op(lib().b200_bicgstabl_solve_op, (A,) + cbs, A.ctx._h, C.byref(A._c), as_device_ptr(st.xd),
                          as_device_ptr(st.bd), C.byref(opts), C.byref(res), rp, cap)
    else:
        status = _call_op(lib().b200_bicgstabl_solve, cbs, A.ctx._h, A._h, as_device_ptr(st.xd), as_device_ptr(st.bd),
                          C.byref(opts), C.byref(res), rp, cap)
    if status == _lib.ERR_BREAKDOWN:
        raise np.linalg.LinAlgError("SingularException in BiCGStab(l) MR step (reference src/bicgstabl.jl:123)")
    check(status)
    st.finish()
    if verbose:
        for i, r in enumerate(resnorm[: res.n_resnorm], start=1):
            print(f"{i:3d}\t{r:1.2e}")
        print()
    return (x, _history(res, resnorm, abstol, reltol, log)) if log else x


def bicgstabl(A, b, l=2, **kw):
    _check_operator(A, linop_ok=True)
    x = DeviceArray.zeros(A.ctx, A.m_local, A.dtype) if is_device(b) else np.zeros(A.m_local, dtype=A.dtype)
    return bicgstabl_(x, A, b, l, initial_zero=True, **kw)


# ------------------------------------------------------------------------------------------------
# Stationary methods  (reference src/stationary_sparse.jl)
# ------------------------------------------------------------------------------------------------
def _stationary_operator(A, method=None):
    """B200CSR as is; a dense matrix (numpy 2-D: the AbstractMatrix methods of reference src/stationary.jl) or a scipy sparse
    matrix is uploaded as CSR.  For a dense matrix the engine is asked for the arithmetic of the reference's dense methods
    (B200_STATIONARY_DENSE_ARITHMETIC): Jacobi and Gauss-Seidel (:48-70, :108-127) are the sparse operations on the stored
    entries (a zero entry contributes 0 * x_j = 0); dense SOR / SSOR (:167-186, :227-258) write the relaxation as
    x += w (t / a_ii - x); the backward half of the dense SSOR reads both triangles with the forward half's values
    (:247-258 subtract A[row, col] * x[col] before x[col] is updated) -- a different iteration from the sparse SSOR, and
    reproduced as such.  A full matrix has n dependency levels of one row each: a convenience, not a fast path."""
    if isinstance(A, B200CSR):
        return A
    if isinstance(A, B200LinearOperator):
        raise TypeError("the stationary methods need the matrix itself (its diagonal and triangles), not a callback operator")
    import scipy.sparse as sp
    if sp.issparse(A) or (isinstance(A, np.ndarray) and A.ndim == 2):
        return B200CSR.from_scipy(sp.csc_matrix(A))
    raise TypeError("the stationary methods take a B200CSR, a scipy sparse matrix or a dense numpy matrix")


def _stationary_prepare(A):
    """the operator for a stationary method; remembers that it came from a dense matrix (the AbstractMatrix methods of
    src/stationary.jl use slightly different arithmetic than the SparseMatrixCSC ones)."""
    dense = isinstance(A, np.ndarray) or getattr(A, "_dense_arithmetic", False)
    A = _stationary_operator(A)
    if dense:
        A._dense_arithmetic = True
    return A


def _stationary(method, x, A, b, omega, maxiter):
    A = _stationary_prepare(A)
    dense = getattr(A, "_dense_arithmetic", False)
    st = _Staged(A, x, b)
    status = lib().b200_stationary(A.ctx._h, A._h, as_device_ptr(st.xd), as_device_ptr(st.bd),
                                   method | (16 if dense else 0), float(omega), int(maxiter))
    if status == _lib.ERR_BREAKDOWN:
        raise np.linalg.LinAlgError("SingularException: zero or missing diagonal entry "
                                    "(reference src/stationary_sparse.jl:19)")
    check(status)
    return st.finish()


def _zerox(A, b):
    return DeviceArray.zeros(A.ctx, A.m_local, A.dtype) if is_device(b) else np.zeros(A.m_local, dtype=A.dtype)


def jacobi_(x, A, b, *, maxiter=10):
    """jacobi!(x, A::SparseMatrixCSC, b; maxiter = 10) -> x -- reference src/stationary_sparse.jl:233-237."""
    return _stationary(0, x, A, b, 1.0, maxiter)


def gauss_seidel_(x, A, b, *, maxiter=10):
    """gauss_seidel!(x, A::SparseMatrixCSC, b; maxiter = 10) -> x -- reference src/stationary_sparse.jl:280-284."""
    return _stationary(1, x, A, b, 1.0, maxiter)


def sor_(x, A, b, omega, *, maxiter=10):
    """sor!(x, A::SparseMatrixCSC, b, ω; maxiter = 10) -> x -- reference src/stationary_sparse.jl:344-348."""
    return _stationary(2, x, A, b, omega, maxiter)


def ssor_(x, A, b, omega, *, maxiter=10):
    """ssor!(x, A::SparseMatrixCSC, b, ω; maxiter = 10) -> x -- reference src/stationary_sparse.jl:420-424."""
    return _stationary(3, x, A, b, omega, maxiter)


def jacobi(A, b, **kw):
    A = _stationary_prepare(A)
    return jacobi_(_zerox(A, b), A, b, **kw)                   # jacobi!(zerox(A, b), A, b; kwargs...)  src/stationary.jl:19


def gauss_seidel(A, b, **kw):
    A = _stationary_prepare(A)
    return gauss_seidel_(_zerox(A, b), A, b, **kw)             # src/stationary.jl:79


def sor(A, b, omega, **kw):
    A = _stationary_prepare(A)
    return sor_(_zerox(A, b), A, b, omega, **kw)               # src/stationary.jl:136-137


def ssor(A, b, omega, **kw):
    A = _stationary_prepare(A)
    return ssor_(_zerox(A, b), A, b, omega, **kw)              # src/stationary.jl:195-196


# ------------------------------------------------------------------------------------------------
# Power method and inverse iteration  (reference src/simple.jl)
# ------------------------------------------------------------------------------------------------
def powm_(B, x, *, tol=None, maxiter=None, shift=0.0, inverse=False, log=False, verbose=False, check_every=0):
    """powm!(B, x; shift, inverse, tol, maxiter, log, verbose) -> λ, x[, history] -- reference src/simple.jl:118-151.
    B: B200CSR or B200LinearOperator (for shift-and-invert: the action of inv(A - shift I), :83-88); x: normalised start
    vector (host or device), overwritten by the eigenvector approximation."""
    _check_operator(B, linop_ok=True)
    if tol is None:
        tol = float(_eps(B.dtype)) * B.size(2) ** 3            # :119
    if maxiter is None:
        maxiter = B.size(1)                                    # :120
    host = not is_device(x)
    if host and not (isinstance(x, np.ndarray) and x.dtype == B.dtype):
        raise TypeError(f"x must be a numpy array of eltype {B.dtype}")
    xd = DeviceArray.from_numpy(B.ctx, x) if host else x
    if xd.shape[0] != B.m_local:
        raise ValueError("dimension mismatch between B and x")
    opts = _lib.PowmOpts(float(tol), int(maxiter), float(shift), int(bool(inverse)), int(check_every))
    res, lam = _lib.Result(), C.c_double()
    cap = int(maxiter) + 1                                     # done() lets iteration == maxiter through, :27
    resnorm = np.zeros(cap, dtype=np.float64)
    a_csr = None if _is_linop(B) else B._h
    a_op = C.byref(B._c) if _is_linop(B) else None
    check(_call_op(lib().b200_powm, (B,) if _is_linop(B) else (), B.ctx._h, a_csr, a_op, as_device_ptr(xd), C.byref(opts),
                   C.byref(res), C.byref(lam), resnorm.ctypes.data_as(C.c_void_p), cap))
    if host:
        x[...] = xd.numpy()
    if verbose:
        print("=== powm ===\niter\tresnorm")
        for i, r in enumerate(resnorm[: res.n_resnorm], start=1):
            print(f"{i:3d}\t{r:1.2e}")
        print()
    lam_T = B.dtype.type(lam.value)
    if not log:
        return lam_T, x
    h = ConvergenceHistory()
    h["tol"] = float(res.tol)
    h.isconverged, h.mvps, h.iters = bool(res.isconverged), int(res.mvps), int(res.iters)
    h["resnorm"] = resnorm[: res.n_resnorm].copy()
    return lam_T, x, h


def powm(B, *, rng=None, **kw):
    """powm(B; kwargs...) = powm!(B, x0; kwargs...) with a random unit start vector -- src/simple.jl:63-67 (the reference
    draws a complex vector; element types are real here)."""
    _check_operator(B, linop_ok=True)
    rng = rng or np.random.default_rng()
    x0 = rng.random(B.m_local).astype(B.dtype)
    x0 /= np.linalg.norm(x0)
    return powm_(B, x0, **kw)


def invpowm_(B, x, **kw):
    """invpowm!(B, x0; shift, kwargs...) = powm!(B, x0; inverse = true, kwargs...) -- src/simple.jl:186."""
    return powm_(B, x, inverse=True, **kw)


def invpowm(B, *, rng=None, **kw):
    """invpowm(B; shift, kwargs...) -- src/simple.jl:172-176."""
    return powm(B, rng=rng, inverse=True, **kw)


# ------------------------------------------------------------------------------------------------
# The resumable forms: gmres_iterable!, minres_iterable!, bicgstabl_iterator!  (docs/src/iterators.md)
# ------------------------------------------------------------------------------------------------
class KrylovIterable:
    """What gmres_iterable! (reference src/gmres.jl:108-136), minres_iterable! (src/minres.jl:39-89) and
    bicgstabl_iterator! (src/bicgstabl.jl:27-73) return: iterating yields the residual norm after each iterate() and
    leaves x updated in place; `step(k)` performs up to k iterations in one call.  The object owns its device scratch
    (other solves may run on the context in between); x, b (and the preconditioners / callbacks) are kept alive here."""

    def __init__(self, create, x, A, b, opts, keep):
        self._A, self._x, self._keep = A, x, keep
        self._st = _Staged(A, x, b)
        self._cbs = tuple(o for o in keep if isinstance(o, B200LinearOperator))
        self._h = C.c_void_p()
        a_csr = None if _is_linop(A) else A._h
        a_op = C.byref(A._c) if _is_linop(A) else None
        check(_call_op(create, self._cbs, A.ctx._h, a_csr, a_op, as_device_ptr(self._st.xd), as_device_ptr(self._st.bd),
                       C.byref(opts), C.byref(self._h)))
        self._opts = opts
        self.result = _lib.Result()
        self._buf = np.zeros(4096, dtype=np.float64)
        self.step(0)                                           # residual / tol of the initial state

    residual = property(lambda self: float(self.result.residual))
    tol = property(lambda self: float(self.result.tol))
    iteration = property(lambda self: int(self.result.iters))
    mv_products = property(lambda self: int(self.result.mvps))
    converged = property(lambda self: bool(self.result.isconverged))       # converged(it)
    done = property(lambda self: self.result.status == 1)                 # done(it, iteration)
    x = property(lambda self: self._x)

    def step(self, k=1):
        """up to k calls of iterate(it); returns the residual norms of the iterations performed."""
        if self._h is None:
            raise RuntimeError("iterator is closed")
        k = int(k)
        out = []
        while True:
            kk = min(k, 4096)
            status = _call_op(lib().b200_iter_next, self._cbs, self._h, kk, C.byref(self.result),
                              self._buf.ctypes.data_as(C.c_void_p), 4096)
            if status == _lib.ERR_BREAKDOWN:
                raise np.linalg.LinAlgError("breakdown in the iteration (SingularException of the BiCGStab(l) MR step, "
                                            "reference src/bicgstabl.jl:123, or a NaN residual)")
            check(status)
            out.extend(self._buf[: self.result.n_resnorm].tolist())
            k -= kk
            if k <= 0 or self.done:
                break
        self._st.finish()                                      # host x: copy the completed iterate back
        return out

    def __iter__(self):
        return self

    def __next__(self):
        if self.done:
            raise StopIteration
        r = self.step(1)
        if not r:
            raise StopIteration
        return r[0]

    def close(self):
        if self._h is not None:
            lib().b200_iter_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def gmres_iterable_(x, A, b, *, Pl=None, Pr=None, abstol=0.0, reltol=None, restart=None, maxiter=None,
                    initially_zero=False, orth_meth="mgs"):
    """gmres_iterable!(x, A, b; Pl, Pr, abstol, reltol, restart, maxiter, initially_zero, orth_meth) -- reference
    src/gmres.jl:108-136; one step = one inner iteration (iterate :57-106)."""
    _check_operator(A, linop_ok=True)
    if reltol is None:
        reltol = math.sqrt(_eps(A.dtype))
    if restart is None:
        restart = min(20, A.size(2))
    if maxiter is None:
        maxiter = A.size(2)
    opts = _lib.GmresOpts(abstol, reltol, int(maxiter), int(restart), int(bool(initially_zero)), _ORTH[orth_meth], 0,
                          precond_to_c(Pl, A), precond_to_c(Pr, A))
    keep = [P for P in (Pl, Pr) if P is not None] + [P.op for P in (Pl, Pr) if isinstance(P, FunctionPrec)] + [A]
    return KrylovIterable(lib().b200_gmres_iter_create, x, A, b, opts, keep)


def minres_iterable_(x, A, b, *, skew_hermitian=False, abstol=0.0, reltol=None, maxiter=None, initially_zero=False):
    """minres_iterable!(x, A, b; initially_zero, skew_hermitian, abstol, reltol, maxiter) -- reference src/minres.jl:39-89."""
    _check_operator(A, linop_ok=True)
    if reltol is None:
        reltol = math.sqrt(_eps(A.dtype))
    if maxiter is None:
        maxiter = A.size(2)
    opts = _lib.MinresOpts(abstol, reltol, int(maxiter), int(bool(initially_zero)), int(bool(skew_hermitian)))
    return KrylovIterable(lib().b200_minres_iter_create, x, A, b, opts, [A])


def minres_iterable(A, b, **kw):
    """minres_iterable(A, b; kwargs...) = minres_iterable!(zerox(A, b), A, b; initially_zero = true, kwargs...)
    -- reference src/minres.jl:27-37."""
    _check_operator(A, linop_ok=True)
    x = DeviceArray.zeros(A.ctx, A.m_local, A.dtype) if is_device(b) else np.zeros(A.m_local, dtype=A.dtype)
    return minres_iterable_(x, A, b, initially_zero=True, **kw)


def bicgstabl_iterator(A, b, l=2, **kw):
    """bicgstabl_iterator(A, b, l; kwargs...) = bicgstabl_iterator!(zerox(A, b), A, b, l; initial_zero = true, kwargs...)
    -- reference src/bicgstabl.jl:24-25."""
    _check_operator(A, linop_ok=True)
    x = DeviceArray.zeros(A.ctx, A.m_local, A.dtype) if is_device(b) else np.zeros(A.m_local, dtype=A.dtype)
    return bicgstabl_iterator_(x, A, b, l, initial_zero=True, **kw)


def bicgstabl_iterator_(x, A, b, l=2, *, Pl=None, max_mv_products=None, abstol=0.0, reltol=None, initial_zero=False,
                        r_shadow=None, rng=None):
    """bicgstabl_iterator!(x, A, b, l; Pl, max_mv_products, abstol, reltol, initial_zero) -- reference
    src/bicgstabl.jl:27-73; one step = one outer iteration (2 l products, iterate :79-134)."""
    _check_operator(A, linop_ok=True)
    if reltol is None:
        reltol = math.sqrt(_eps(A.dtype))
    if max_mv_products is None:
        max_mv_products = A.size(2)
    if r_shadow is None:
        rng = rng or np.random.default_rng()
        r_shadow = rng.random(A.m_local).astype(A.dtype)       # rand(T, n) :38
    rs = r_shadow if is_device(r_shadow) else DeviceArray.from_numpy(A.ctx, np.asarray(r_shadow, dtype=A.dtype))
    opts = _lib.BicgstablOpts(abstol, reltol, int(max_mv_products), int(l), int(bool(initial_zero)), precond_to_c(Pl, A),
                              as_device_ptr(rs))
    keep = [rs, A] + ([Pl] if Pl is not None else []) + ([Pl.op] if isinstance(Pl, FunctionPrec) else [])
    return KrylovIterable(lib().b200_bicgstabl_iter_create, x, A, b, opts, keep)


# ------------------------------------------------------------------------------------------------
# SURVEY.md section 8(f) item 4: the solvers that need A' (QMR, LSQR, LSMR) and IDR(s)
# ------------------------------------------------------------------------------------------------
class _StagedRect:
    """host<->device staging for an m x n operator: x has n entries, b has m."""

    def __init__(self, A: B200CSR, x, b):
        m = A.m_local
        n = A.n_local if isinstance(A, B200LinearOperator) else (A.n_global if A.ctx.world == 1 else A.m_local)
        self.host = not is_device(x)
        self.x = x
        if self.host:
            if is_device(b):
                raise TypeError("x and b must both be host arrays or both be device arrays")
            if not (isinstance(x, np.ndarray) and x.dtype == A.dtype):
                raise TypeError(f"x must be a numpy array of eltype {A.dtype} (got {getattr(x, 'dtype', type(x))})")
            self.xd = DeviceArray.from_numpy(A.ctx, x)
            self.bd = DeviceArray.from_numpy(A.ctx, np.asarray(b, dtype=A.dtype))
        else:
            self.xd, self.bd = x, b
        if self.xd.shape[0] != n:
            raise ValueError(f"x should be of length {n}")                   # src/lsqr.jl:99
        if self.bd.shape[0] != m:
            raise ValueError(f"b should be of length {m}")                   # src/lsqr.jl:100

    def finish(self):
        if self.host:
            self.x[...] = self.xd.numpy().reshape(self.x.shape)
        return self.x


def qmr_(x, A, b, *, abstol=0.0, reltol=None, maxiter=None, lookahead=False, log=False, initially_zero=False,
         verbose=False, check_every=0):
    """qmr!(x, A, b; abstol, reltol, maxiter, lookahead, log, initially_zero, verbose) -- reference src/qmr.jl:262-297.
    `lookahead` is accepted and ignored, as in the reference (it is never forwarded, src/qmr.jl:279-280)."""
    _check_operator(A, linop_ok=True)
    if reltol is None:
        reltol = math.sqrt(_eps(A.dtype))                     # src/qmr.jl:267
    if maxiter is None:
        maxiter = A.size(2)                                   # src/qmr.jl:268
    opts = _lib.QmrOpts(abstol, reltol, int(maxiter), int(bool(initially_zero)), int(check_every))
    res = _lib.Result()
    cap = int(maxiter) if log else 0                          # reserve!(history, :resnorm, maxiter)  :277
    resnorm = np.zeros(max(cap, 1), dtype=np.float64)
    st = _Staged(A, x, b)
    rp = resnorm.ctypes.data_as(C.c_void_p) if log else None
    if _is_linop(A):
        At = A.adjoint()
        check(_call_op(lib().b200_qmr_solve_op, (A, At), A.ctx._h, C.byref(A._c), C.byref(At._c), as_device_ptr(st.xd),
                       as_device_ptr(st.bd), C.byref(opts), C.byref(res), rp, cap))
    else:
        check(lib().b200_qmr_solve(A.ctx._h, A._h, A.adjoint()._h, as_device_ptr(st.xd), as_device_ptr(st.bd),
                                   C.byref(opts), C.byref(res), rp, cap))
    st.finish()
    if verbose:
        print("=== qmr ===\niter\tresnorm")
        for i, r in enumerate(resnorm[: res.n_resnorm], start=1):
            print(f"{i:3d}\t{r:1.2e}")
        print()
    qmr_.last_result = res
    h = _history(res, resnorm, abstol, reltol, log)
    h.isconverged = bool(res.isconverged) if log else False  # setconv only when log (src/qmr.jl:293)
    h.mvps = 0                                                # nextiter!(history) without mvps (src/qmr.jl:285)
    return (x, h) if log else x


def qmr(A, b, **kw):
    """qmr(A, b; kwargs...) = qmr!(zerox(A, b), A, b; initially_zero = true, kwargs...) -- src/qmr.jl:222."""
    _check_operator(A, linop_ok=True)
    x = DeviceArray.zeros(A.ctx, A.m_local, A.dtype) if is_device(b) else np.zeros(A.m_local, dtype=A.dtype)
    return qmr_(x, A, b, initially_zero=True, **kw)


def _lsq(fn, first_key, x, A, b, damp, atol, btol, conlim, maxiter, log, verbose, check_every, name):
    _check_operator(A, linop_ok=True)
    if maxiter is None:
        maxiter = max(A.shape)                                # maximum(size(A))  src/lsqr.jl:67, src/lsmr.jl:68
    opts = _lib.LsqOpts(float(damp), float(atol), float(btol), float(conlim), int(maxiter), int(check_every), 0)
    res = _lib.LsqResult()
    cap = int(maxiter)                                        # reserve!(history, [...], maxiter)  src/lsqr.jl:73
    hist = np.zeros(4 * max(cap, 1), dtype=np.float64)
    st = _StagedRect(A, x, b)
    if _is_linop(A):
        At = A.adjoint()
        status = _call_op(getattr(lib(), f"b200_{name}_solve_op"), (A, At), A.ctx._h, C.byref(A._c), C.byref(At._c),
                          as_device_ptr(st.xd), as_device_ptr(st.bd), C.byref(opts), C.byref(res),
                          hist.ctypes.data_as(C.c_void_p), cap)
    else:
        status = fn(A.ctx._h, A._h, A.adjoint()._h, as_device_ptr(st.xd), as_device_ptr(st.bd), C.byref(opts),
                    C.byref(res), hist.ctypes.data_as(C.c_void_p), cap)
    if status == _lib.ERR_INVALID and res.status == _lib.ERR_INVALID:
        raise ValueError("Initial guess for x must be finite")            # src/lsqr.jl:102-104
    check(status)
    st.finish()
    h = ConvergenceHistory()
    h["atol"], h["btol"], h["ctol"] = res.atol, res.btol, res.ctol       # src/lsqr.jl:118-120
    h.isconverged = bool(res.isconverged)
    h.iters, h.mvps, h.mtvps = int(res.iters), int(res.mvps), int(res.mtvps)
    h["istop"] = int(res.istop)
    sd, k = int(res.hist_stride), int(res.n_hist)
    for i, key in enumerate((first_key, "anorm", "rnorm", "cnorm")):
        if key is not None:
            h[key] = hist[i * sd: i * sd + k].copy()
    if verbose:
        print(f"=== {name} ===")
        for i in range(k):
            print(f"{i + 1:3d}\t{h['anorm'][i]:1.2e}\t{h['cnorm'][i]:1.2e}\t{h['rnorm'][i]:1.2e}")
        print()
    return (x, h) if log else x


def lsqr_(x, A, b, *, damp=0.0, atol=None, btol=None, conlim=None, maxiter=None, log=False, verbose=False,
          check_every=0):
    """lsqr!(x, A, b; damp, atol, btol, conlim, maxiter, verbose, log) -- reference src/lsqr.jl:66-77, 90-275.
    A may be rectangular (m x n): x has n entries, b has m."""
    s = math.sqrt(_eps(A.dtype)) if isinstance(A, (B200CSR, B200LinearOperator)) else 0.0
    atol = s if atol is None else atol                        # src/lsqr.jl:91
    btol = s if btol is None else btol
    conlim = (1.0 / s if s else 0.0) if conlim is None else conlim        # src/lsqr.jl:92
    return _lsq(lib().b200_lsqr_solve, "resnorm", x, A, b, damp, atol, btol, conlim, maxiter, log, verbose,
                check_every, "lsqr")


def lsqr(A, b, **kw):
    """lsqr(A, b; kwargs...) = lsqr!(zerox(A, b), A, b; kwargs...) -- src/lsqr.jl:8."""
    _check_operator(A, linop_ok=True)
    n = A.n_local if _is_linop(A) else (A.shape[1] if A.ctx.world == 1 else A.m_local)
    x = DeviceArray.zeros(A.ctx, n, A.dtype) if is_device(b) else np.zeros(n, dtype=A.dtype)
    return lsqr_(x, A, b, **kw)


def lsmr_(x, A, b, *, atol=1e-6, btol=1e-6, conlim=1e8, maxiter=None, lam=0.0, log=False, verbose=False,
          check_every=0):
    """lsmr!(x, A, b; atol, btol, conlim, maxiter, λ, verbose, log) -- reference src/lsmr.jl:67-82, 88-287
    (`λ` is spelled `lam`).  The work vectors v, h, hbar of src/lsmr.jl:78 are device scratch of the engine."""
    return _lsq(lib().b200_lsmr_solve, None, x, A, b, lam, atol, btol, conlim, maxiter, log, verbose, check_every,
                "lsmr")


def lsmr(A, b, **kw):
    """lsmr(A, b; kwargs...) = lsmr!(zerox(A, b), A, b; kwargs...) -- src/lsmr.jl:10."""
    _check_operator(A, linop_ok=True)
    n = A.n_local if _is_linop(A) else (A.shape[1] if A.ctx.world == 1 else A.m_local)
    x = DeviceArray.zeros(A.ctx, n, A.dtype) if is_device(b) else np.zeros(n, dtype=A.dtype)
    return lsmr_(x, A, b, **kw)


def idrs_(x, A, b, *, s=8, Pl=None, abstol=0.0, reltol=None, maxiter=None, log=False, smoothing=False, verbose=False,
          P=None, rng=None, check_every=0):
    """idrs!(x, A, b; s, Pl, abstol, reltol, maxiter, log, smoothing, verbose) -- reference src/idrs.jl:49-64.
    The reference draws the shadow space with rand!(copy(C)) (src/idrs.jl:132); here the draw happens on the host
    (numpy Generator `rng`) unless `P` (n x s) is given."""
    _check_operator(A, linop_ok=True)
    if reltol is None:
        reltol = math.sqrt(_eps(A.dtype))                     # src/idrs.jl:53
    if maxiter is None:
        maxiter = A.size(2)                                   # src/idrs.jl:54
    if P is None:
        rng = rng or np.random.default_rng()
        P = np.asfortranarray(rng.random((A.m_local, int(s))).astype(A.dtype))
    Pd = P if is_device(P) else DeviceArray.from_numpy(A.ctx, np.asfortranarray(P, dtype=A.dtype))
    if Pd.shape[0] != A.m_local or Pd.shape[1] != int(s):
        raise ValueError("P must be n x s")
    opts = _lib.IdrsOpts(abstol, reltol, int(maxiter), int(s), int(bool(smoothing)), precond_to_c(Pl, A),
                         as_device_ptr(Pd), int(Pd.shape[0]), int(check_every), 0)
    res = _lib.Result()
    cap = int(maxiter) if log else 0                          # reserve!(history, :resnorm, maxiter)  :60
    resnorm = np.zeros(max(cap, 1), dtype=np.float64)
    st = _Staged(A, x, b)
    rp = resnorm.ctypes.data_as(C.c_void_p) if log else None
    plop = Pl.op if isinstance(Pl, FunctionPrec) else None      # ldiv!(Pl, V) by callback (B200_PREC_CALLBACK)
    if _is_linop(A):
        check(_call_op(lib().b200_idrs_solve_op, (A, plop), A.ctx._h, C.byref(A._c), as_device_ptr(st.xd),
                       as_device_ptr(st.bd), C.byref(opts), C.byref(res), rp, cap))
    else:
        check(_call_op(lib().b200_idrs_solve, (plop,), A.ctx._h, A._h, as_device_ptr(st.xd), as_device_ptr(st.bd),
                       C.byref(opts), C.byref(res), rp, cap))
    st.finish()
    if verbose:
        print("=== idrs ===\niter\tstep\tresnorm")
        for i, r in enumerate(resnorm[: res.n_resnorm], start=1):
            print(f"{i:3d}\t{1 + (i - 1) % (int(s) + 1):3d}\t{r:1.2e}")
        print()
    idrs_.last_result = res
    return (x, _history(res, resnorm, abstol, reltol, log)) if log else x


def idrs(A, b, **kw):
    """idrs(A, b; kwargs...) = idrs!(zerox(A, b), A, b; kwargs...) -- src/idrs.jl:11."""
    _check_operator(A, linop_ok=True)
    x = DeviceArray.zeros(A.ctx, A.m_local, A.dtype) if is_device(b) else np.zeros(A.m_local, dtype=A.dtype)
    return idrs_(x, A, b, **kw)


# ------------------------------------------------------------------------------------------------
# LOBPCG  (reference src/lobpcg.jl:787-839, 865-893)
# ------------------------------------------------------------------------------------------------
@dataclass
class LOBPCGResults:
    """reference src/lobpcg.jl:56-65."""
    lam: np.ndarray            # λ
    X: object
    tolerance: float
    residual_norms: np.ndarray
    iterations: int
    maxiter: int
    converged: bool
    trace: list


def _linop_struct(op):
    """(b200_linop struct, python callback operator or None) of a B200CSR (applied by the library itself, no Python in
    the loop: b200_csr_as_linop) or of a B200LinearOperator."""
    if isinstance(op, B200LinearOperator):
        return op._c, op
    s = _lib.LinOp()
    check(lib().b200_csr_as_linop(op._h, C.byref(s)))
    return s, None


class LobpcgConstraint:
    """Constraint(Y, nothing, X) -- reference src/lobpcg.jl:144-224 (standard problem): a basis Y (n x nc, host array
    or DeviceArray; copied) the Ritz vectors are kept orthogonal to.  `capacity` columns are reserved for `append`
    (update!, :188-206)."""

    def __init__(self, ctx, n, dtype, Y=None, capacity=0, B=None):
        self.ctx, self.n, self.dtype = ctx, int(n), np.dtype(dtype)
        self._h = C.c_void_p()
        self.generalized = B is not None
        nc = 0 if Y is None else int(Y.shape[1])
        Yd = None
        if nc:
            Yd = Y if is_device(Y) else DeviceArray.from_numpy(ctx, np.asfortranarray(Y, dtype=self.dtype))
            if Yd.shape[0] != self.n:
                raise ValueError("the constraint must have as many rows as the operator")
        code = dtype_code(self.dtype)
        if B is not None:                                      # Constraint(Y, B, X) with BY = B*Y  src/lobpcg.jl:161-186
            bs, bop = _linop_struct(B)
            self._keep, self._bop = (bs, B), bop               # append applies B again (update!, :188-206)
            check(_call_op(lib().b200_lobpcg_constraint_create_b, (bop,), ctx._h, C.byref(bs), self.n,
                           as_device_ptr(Yd) if nc else None, self.n, nc, int(max(capacity, nc)), code, C.byref(self._h)))
        else:
            check(lib().b200_lobpcg_constraint_create(ctx._h, self.n, as_device_ptr(Yd) if nc else None, self.n, nc,
                                                      int(max(capacity, nc)), code, C.byref(self._h)))

    @property
    def ncols(self):
        k, cap = C.c_int(), C.c_int()
        check(lib().b200_lobpcg_constraint_info(self._h, C.byref(k), C.byref(cap)))
        return k.value

    def append(self, Xd: DeviceArray, k=None):
        """update!(constraint, X[:, 1:k], ...): the first k columns of the device block Xd join the basis."""
        k = Xd.shape[1] if k is None else int(k)
        check(_call_op(lib().b200_lobpcg_constraint_append, (getattr(self, "_bop", None),), self.ctx._h, self._h,
                       as_device_ptr(Xd), Xd.shape[0], k))

    def apply_(self, Xd: DeviceArray):
        """constr!(X, temp): X <- X - Y (Y'Y \\ Y'X), in place on a device block."""
        bs = Xd.shape[1] if len(Xd.shape) == 2 else 1
        check(lib().b200_lobpcg_constraint_apply(self.ctx._h, self._h, as_device_ptr(Xd), Xd.shape[0], bs))
        return Xd

    def close(self):
        if self._h:
            lib().b200_lobpcg_constraint_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _lobpcg_block(A, largest, Xd, P, constraint, tol, maxiter, not_zeros, rng, fixed, B=None, trace=None):
    """lobpcg!(iterator; ...) -- reference src/lobpcg.jl:865-893 on the device block Xd (overwritten).  `trace`: a list
    that receives (iteration, residual_norms, ritz_values) per iteration (log = true, :881-884)."""
    n, bs = Xd.shape
    if not not_zeros and not fixed:                            # :869-876 (the constraint itself is applied by the engine)
        nrm = C.c_double()
        for j in range(bs):                                    # all(x -> x == 0, X[:, j])  <=>  ||X[:, j]|| == 0
            col = Xd.column(j)
            check(lib().b200_nrm2(A.ctx._h, n, col._p, col.code, C.byref(nrm)))
            if nrm.value == 0.0:
                rng = rng or np.random.default_rng()
                col.upload(rng.random(n).astype(A.dtype))      # X[:, j] .= rand.() :872
    opts = _lib.LobpcgOpts(float(tol), int(maxiter), int(bool(largest)), int(bs), precond_to_c(P, A), int(bool(fixed)), 0)
    if trace is not None:
        tr_r, tr_l = np.zeros((max(int(maxiter), 1), bs)), np.zeros((max(int(maxiter), 1), bs))
        opts.trace_resnorm, opts.trace_ritz, opts.trace_cap = tr_r.ctypes.data, tr_l.ctypes.data, int(maxiter)
    res = _lib.LobpcgResult()
    lam = np.zeros(bs, dtype=np.float64)
    rn = np.zeros(bs, dtype=np.float64)
    if B is not None or _is_linop(A) or isinstance(P, FunctionPrec):
        # the general engine (csrc/lobpcg_general_core.h): generalized problem, callback operators / preconditioner
        a_s, a_op = _linop_struct(A)
        b_s, b_op = _linop_struct(B) if B is not None else (None, None)
        p_op = P.op if isinstance(P, FunctionPrec) else None
        status = _call_op(lib().b200_lobpcg_solve_op, (a_op, b_op, p_op), A.ctx._h, C.byref(a_s),
                          C.byref(b_s) if b_s is not None else None, as_device_ptr(Xd), n, C.byref(opts),
                          constraint._h if constraint is not None else None, C.byref(res),
                          lam.ctypes.data_as(C.c_void_p), rn.ctypes.data_as(C.c_void_p))
    elif constraint is None:
        status = lib().b200_lobpcg_solve(A.ctx._h, A._h, as_device_ptr(Xd), n, C.byref(opts), C.byref(res),
                                         lam.ctypes.data_as(C.c_void_p), rn.ctypes.data_as(C.c_void_p))
    else:
        status = lib().b200_lobpcg_solve_constrained(A.ctx._h, A._h, as_device_ptr(Xd), n, C.byref(opts), constraint._h,
                                                     C.byref(res), lam.ctypes.data_as(C.c_void_p),
                                                     rn.ctypes.data_as(C.c_void_p))
    if status == _lib.ERR_BREAKDOWN:
        raise np.linalg.LinAlgError("PosDefException in CholQR (reference src/lobpcg.jl:380)")
    check(status)
    if trace is not None:                                      # LOBPCGState(iteration, residual_norms, ritz_values) :744-745
        for i in range(min(int(res.iterations), int(maxiter))):
            trace.append((i + 1, tr_r[i].astype(A.dtype), tr_l[i].astype(A.dtype)))
    return lam, rn, res


def lobpcg(A, largest: bool, X0, nev=None, *, B=None, P=None, C_=None, tol=None, maxiter=200, log=False,
           not_zeros=False, rng=None, _fixed_iterations=False, **kw):
    """lobpcg(A, [B,] largest, X0; P, C, tol, maxiter, not_zeros) -> LOBPCGResults   reference src/lobpcg.jl:824-839
    lobpcg(A, [B,] largest, nev::Int; ...)   (X0 = rand(n, nev), not_zeros = true)   :787-792
    lobpcg(A, [B,] largest, X0, nev; ...)  (batches of size(X0, 2) with deflation)    :925-962
    `B=` (a B200CSR or B200LinearOperator) selects the generalized problem A x = λ B x; A may be a
    B200LinearOperator and P a FunctionPrec (callbacks): those three go through the general engine, the standard problem
    on a B200CSR with Identity / JacobiPrec through the tuned one.  The constraint is the keyword `C` (spelled `C=`
    here; `C_` is accepted as well): an n x nc host array / DeviceArray, or a LobpcgConstraint.  X0: n x blocksize,
    host (numpy, any order) or DeviceArray (column-major)."""
    Cc = kw.pop("C", C_)
    if kw:
        raise TypeError(f"unexpected keyword arguments {sorted(kw)}")
    _check_operator(A, linop_ok=True)
    if B is not None:
        _check_operator(B, linop_ok=True)
    if tol is None:
        tol = _eps(A.dtype) ** 0.3                             # default_tolerance  src/lobpcg.jl:751
    if isinstance(X0, (int, np.integer)):                      # lobpcg(A, largest, nev) :790-792
        rng = rng or np.random.default_rng()
        X0 = rng.random((A.m_local, int(X0))).astype(A.dtype)
        not_zeros = True
    host = not is_device(X0)
    Xd = DeviceArray.from_numpy(A.ctx, np.asarray(X0, dtype=A.dtype)) if host else X0
    n, bs = Xd.shape
    if n != A.m_local:
        raise ValueError("X0 has the wrong number of rows")
    if nev is not None and int(nev) > A.n_global:
        raise B200Error("Number of eigenvectors desired exceeds the row dimension.")          # :933
    if n < 3 * bs:
        # src/lobpcg.jl:834: throw("... not stable to use when the matrix size is less than 3 times the block size ...")
        raise B200Error("The order of the matrix must be at least 3 times the block size")
    if nev is None:
        con = Cc if isinstance(Cc, LobpcgConstraint) or Cc is None else LobpcgConstraint(A.ctx, n, A.dtype, Cc, B=B)
        trace = [] if log else None
        lam, rn, res = _lobpcg_block(A, largest, Xd, P, con, tol, maxiter, not_zeros, rng, _fixed_iterations, B=B,
                                     trace=trace)
        X = Xd.numpy() if host else Xd
        return LOBPCGResults(lam.astype(A.dtype), X, float(tol), rn.astype(A.dtype), int(res.iterations), int(maxiter),
                             bool(res.converged), trace or [])
    # ---- nev > blocksize driver :928-962
    nev = int(nev)
    rng = rng or np.random.default_rng()
    sizeX = min(nev, bs)                                       # :936
    if sizeX < bs:                                             # X = X0[:, 1:sizeX] :937
        Xd = DeviceArray.from_numpy(A.ctx, np.asfortranarray(Xd.numpy()[:, :sizeX]))
    elif not host:
        Xd = DeviceArray.from_numpy(A.ctx, Xd.numpy())         # X0 is not overwritten by this form
    sizeC = 0 if Cc is None else int(Cc.shape[1])
    con = LobpcgConstraint(A.ctx, n, A.dtype, Cc, capacity=sizeC + (nev // sizeX) * sizeX, B=B)  # :501-508, :519
    lam_all = np.zeros(nev, dtype=A.dtype)
    rn_all = np.zeros(nev, dtype=A.dtype)
    X_all = np.zeros((n, nev), dtype=A.dtype, order="F")
    iterations, conv = [], np.zeros(nev, dtype=bool)

    traces = []                                                # results.trace: one LOBPCGTrace per batch :74, :88

    def run(nz):
        tr = [] if log else None
        lam, rn, res = _lobpcg_block(A, largest, Xd, P, con, tol, maxiter, nz, rng, False, B=B, trace=tr)
        if log:
            traces.append(tr)
        return lam, rn, res, Xd.numpy()

    def append(r, n1, n2):                                     # append! :79-91
        lam, rn, res, Xh = r
        lam_all[n1:n1 + n2] = lam[-n2:]
        rn_all[n1:n1 + n2] = rn[-n2:]
        X_all[:, n1:n1 + n2] = Xh[:, -n2:]
        iterations.append(int(res.iterations))
        conv[n1:n1 + n2] = bool(res.converged)

    r = run(not_zeros)                                         # :941
    append(r, 0, sizeX)
    converged_x = sizeX
    while converged_x < nev:                                   # :944
        Xh = r[3]
        if nev - converged_x < sizeX:                          # :945-952
            cutoff = sizeX - (nev - converged_x)
            con.append(Xd, cutoff)                             # update!(constr!, X[:, 1:cutoff], ...)
            Xh[:, :sizeX - cutoff] = Xh[:, cutoff:sizeX].copy()
            Xh[:, cutoff:sizeX] = rng.random((n, sizeX - cutoff)).astype(A.dtype)
            Xd.upload(Xh)
            r = run(True)
            append(r, converged_x, sizeX - cutoff)
            converged_x += sizeX - cutoff
        else:                                                  # :953-959
            con.append(Xd)
            Xd.upload(rng.random((n, sizeX)).astype(A.dtype))
            r = run(True)
            append(r, converged_x, sizeX)
            converged_x += sizeX
    con.close()
    return LOBPCGResults(lam_all, X_all, float(tol), rn_all, iterations, int(maxiter), conv, traces)


class LOBPCGIterator:
    """LOBPCGIterator(A, B, largest, X, P = nothing, C = nothing) -- reference src/lobpcg.jl:450-493: the operators, the
    block X the iteration overwrites, the preconditioner and the constraint (built once: Constraint(C, B, X), :452).  The
    reference preallocates every block here; on the device the context scratch plays that role, so this object only ties the
    pieces together for `lobpcg_(iterator; ...)`.  X: n x blocksize host array (updated in place) or DeviceArray."""

    def __init__(self, A, B, largest: bool, X, P=None, C_=None, **kw):
        Cc = kw.pop("C", C_)
        if kw:
            raise TypeError(f"unexpected keyword arguments {sorted(kw)}")
        _check_operator(A, linop_ok=True)
        if B is not None:
            _check_operator(B, linop_ok=True)
        self.A, self.B, self.largest, self.P = A, B, bool(largest), P
        self.X = X
        n, bs = X.shape
        if n != A.m_local:
            raise ValueError("X has the wrong number of rows")
        if n < 3 * bs:
            raise B200Error("The order of the matrix must be at least 3 times the block size")       # src/lobpcg.jl:834
        self.constraint = (Cc if isinstance(Cc, LobpcgConstraint) or Cc is None
                           else LobpcgConstraint(A.ctx, n, A.dtype, Cc, B=B))
        self.iteration = 0
        self.trace = []


def lobpcg_(iterator: LOBPCGIterator, *, log=False, maxiter=200, not_zeros=False, tol=None, rng=None):
    """lobpcg!(iterator::LOBPCGIterator; log, maxiter, not_zeros, tol) -> LOBPCGResults -- reference src/lobpcg.jl:865-893.
    Overwrites iterator.X with the Ritz vectors (as the reference overwrites iterator.XBlocks.block)."""
    it = iterator
    A = it.A
    if tol is None:
        tol = _eps(A.dtype) ** 0.3                             # default_tolerance :751
    host = not is_device(it.X)
    Xd = DeviceArray.from_numpy(A.ctx, np.asarray(it.X, dtype=A.dtype)) if host else it.X
    trace = [] if log else None
    lam, rn, res = _lobpcg_block(A, it.largest, Xd, it.P, it.constraint, tol, maxiter, not_zeros, rng, False, B=it.B,
                                 trace=trace)
    if host:
        it.X[...] = Xd.numpy()
    it.iteration = int(res.iterations)
    it.trace = trace or []
    return LOBPCGResults(lam.astype(A.dtype), it.X, float(tol), rn.astype(A.dtype), int(res.iterations), int(maxiter),
                         bool(res.converged), it.trace)


# ------------------------------------------------------------------------------------------------
# svdl  (reference src/svdl.jl:157-247)
# ------------------------------------------------------------------------------------------------
@dataclass
class PartialFactorization:
    """what svdl returns as `L` (reference src/svdl.jl:76-84): here the projected matrix B (k x k, dense) and beta;
    the Lanczos bases P, Q stay on the device inside the engine."""
    B: np.ndarray
    beta: float


@dataclass
class SVD:
    """LinearAlgebra.SVD(leftvecs, values, rightvecs) as svdl builds it (src/svdl.jl:243-246): U m x nsv, S, Vt nsv x n
    (empty blocks for the sides `vecs` did not ask for)."""
    U: np.ndarray
    S: np.ndarray
    Vt: np.ndarray


def svdl(A, *, nsv=6, k=None, tol=None, maxiter=None, method="ritz", log=False, v0=None, j=None, reltol=None,
         vecs="none", dolock=False, verbose=False, rng=None):
    """svdl(A; nsv, k, tol, maxiter, method, log, v0, j, reltol, vecs, dolock) -> Σ, L[, history]
    (reference src/svdl.jl:157-247).  A: B200CSR (m x n, single GPU) or a B200LinearOperator with adjoint_mul.
    v0: starting vector in the domain of A (host or device); default randn normalised (src/svdl.jl:178)."""
    _check_operator(A, linop_ok=True)
    if method not in ("ritz", "harmonic"):
        raise ValueError(f"Unknown restart method {method}")              # ArgumentError  src/svdl.jl:199
    if vecs not in ("none", "left", "right", "both"):
        raise ValueError(f"vecs = {vecs!r}")
    m, n = A.m_local, (A.n_local if _is_linop(A) else (A.n_global if A.ctx.world == 1 else A.m_local))
    sq = math.sqrt(np.finfo(np.float64).eps)                              # sqrt(eps()): Float64 literal  :158, :179
    tol = sq if tol is None else tol
    reltol = sq if reltol is None else reltol
    k = 2 * nsv if k is None else int(k)                                  # :158
    j = nsv if j is None else int(j)                                      # :178
    maxiter = min(A.shape) if maxiter is None else int(maxiter)           # :159
    if v0 is None:
        rng = rng or np.random.default_rng()
        v0 = rng.standard_normal(n).astype(A.dtype)
        v0 /= np.linalg.norm(v0)
    v0d = v0 if is_device(v0) else DeviceArray.from_numpy(A.ctx, np.asarray(v0, dtype=A.dtype))
    if v0d.shape[0] != n:
        raise ValueError("v0 must have as many entries as A has columns")
    want_u, want_v = vecs in ("left", "both"), vecs in ("right", "both")
    Ud = DeviceArray(A.ctx, (m, nsv), A.dtype) if want_u else None
    Vd = DeviceArray(A.ctx, (n, nsv), A.dtype) if want_v else None
    opts = _lib.SvdlOpts(int(nsv), k, j, 1 if method == "harmonic" else 0, maxiter, float(tol), float(reltol),
                         int(bool(dolock)), 0)
    res = _lib.SvdlResult()
    sigma = np.zeros(nsv)
    mi = max(maxiter, 1)
    ritz, resn = np.zeros((mi, k)), np.zeros((mi, nsv))
    conv, betas, Bk = np.zeros((mi, nsv), dtype=np.int32), np.zeros(mi), np.zeros((k, k), order="F")
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    common = (as_device_ptr(v0d), C.byref(opts), C.byref(res), vp(sigma), as_device_ptr(Ud) if want_u else None, m,
              as_device_ptr(Vd) if want_v else None, n, vp(ritz), vp(resn), vp(conv), vp(betas), vp(Bk))
    if _is_linop(A):
        At = A.adjoint()
        check(_call_op(lib().b200_svdl_op, (A, At), A.ctx._h, C.byref(A._c), C.byref(At._c), *common))
    else:
        check(lib().b200_svdl(A.ctx._h, A._h, A.adjoint()._h, *common))
    it = int(res.iters)
    values = sigma.astype(A.dtype)
    L = PartialFactorization(Bk, float(res.beta))
    if vecs == "none":
        X = values                                                        # :243-244
    else:
        U = Ud.numpy() if want_u else np.zeros((m, 0), dtype=A.dtype)     # :230-235
        Vt = Vd.numpy().T.copy() if want_v else np.zeros((0, n), dtype=A.dtype)   # :236-241
        X = SVD(U, values, Vt)
    if verbose:
        for i in range(it):
            print(f"Iteration {i + 1}: beta = {betas[i]:1.3e}, converged {int(conv[i].sum())}/{nsv}")
    if not log:
        return X, L
    h = ConvergenceHistory()
    h["tol"] = float(res.tol)                                             # :164
    h.isconverged = bool(res.isconverged)
    h.iters, h.mvps, h.mtvps = it, int(res.mvps), int(res.mtvps)
    h["ritz"], h["resnorm"] = ritz[:it].copy(), resn[:it].copy()          # :209, :348
    h["conv"], h["betas"] = conv[:it].astype(bool), betas[:it].copy()     # :208, :211
    return X, L, h


# ------------------------------------------------------------------------------------------------
# L1 helpers exposed for tests / drop-in use
# ------------------------------------------------------------------------------------------------
def orthogonalize_and_normalize_(V: DeviceArray, w: DeviceArray, h: np.ndarray, method="mgs", k=None):
    """orthogonalize_and_normalize!(V[:, 1:k], w, h, method) -> nrm  (reference src/orthogonalize.jl)."""
    k = V.shape[1] if k is None else k
    nrm = C.c_double()
    hh = np.zeros(k, dtype=np.float64)
    check(lib().b200_orthogonalize_and_normalize(V.ctx._h, V.shape[0], V._p, V.shape[0], k, w._p,
                                                 hh.ctypes.data_as(C.c_void_p), _ORTH[method], V.code, C.byref(nrm)))
    h[:k] = hh
    return float(nrm.value)


def hessenberg_ldiv_(H: DeviceArray, rhs: DeviceArray):
    """ldiv!(FastHessenberg(H), rhs)  (reference src/hessenberg.jl:15-46); H (m+1) x m fp64 on device."""
    check(lib().b200_hessenberg_ldiv(H.ctx._h, H._p, H.shape[0], H.shape[1], rhs._p))
    return rhs
