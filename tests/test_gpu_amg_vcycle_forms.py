"""The AMG V-cycle (csrc/amg.cu) on every SpMV form and for sweep counts other than one pre- and one post-sweep.

Every smoothing, residual, restriction and prolongation step of the V-cycle is one launch_spmv_fused with an epilogue of
amg.cu, in the form the level's operator and the context option "spmv_kernel" select (1 sub-warp per row, 2 CSR stream,
3 band stream, 0 automatic).  The band stream sums every row in the CSR stream's order, so forms 0, 2 and 3 give the same
bits; the sub-warp form sums in another order and agrees with the serial V-cycle (tests/hostsim_amg) to rounding.

The sweep counts exercise the V-cycle's buffer rotation: no pre-sweep (the residual is b), no post-sweep (the
prolongation writes x), several sweeps of each (u0 / u1 ping-pong), ldiv!(P, x) in place, and a one-level hierarchy (the
dense coarse solve on a copy of x).
"""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import oracle as O
from test_amg_engine import NumpySA, SimAMG, _rel
from test_gpu_amg import _check

pytestmark = pytest.mark.gpu
SEED = 20261016
AUTO, SUBWARP, CSR, BAND = 0, 1, 2, 3
TOL = {np.float64: 1e-12, np.float32: 1e-5}


@pytest.fixture(scope="module")
def isb():
    import iterativesolvers_jl_b200 as m
    return m


@pytest.fixture(scope="module")
def ctx(isb):
    # a context of this module's own: a forced form or band_values = 0 left behind by a failing test reaches no other
    return isb.Context(0)


def long_row_spd(n, per_row, rng):
    """Symmetric, strictly diagonally dominant (so SPD) n x n matrix with about per_row + 1 nonzeros per row."""
    M = sp.random(n, n, density=per_row / (2 * n), random_state=rng, format="csr")
    M = M + M.T
    M = M + sp.diags(np.asarray(abs(M).sum(axis=1)).ravel() + 0.05)
    M = M.tocsr()
    M.sort_indices()
    return M


def stream_kind(isb, h):
    kind, nbytes = C.c_int(), C.c_int64()
    assert isb.lib().b200_csr_stream_kind(h, C.byref(kind), C.byref(nbytes)) == 0
    return kind.value


def level_kinds(isb, P):
    """per level, the form b200_csr_stream_kind reports for (A_l, P_l); P_l is None on the coarsest level"""
    out = []
    for l in range(len(P.level_rows)):
        ha, hp = C.c_void_p(), C.c_void_p()
        assert isb.lib().b200_amg_download_level(P._h, l, C.byref(ha), C.byref(hp), None, None) == 0
        out.append((stream_kind(isb, ha), stream_kind(isb, hp) if hp.value else None))
    return out


_MATS = {}


def matrix(name):
    """(scipy CSR in fp64, the form the fine level takes automatically)"""
    if name not in _MATS:
        if name == "laplace3d_64":
            M, kind = O.laplace_matrix_scipy(np.float64, 64, 3), BAND
        elif name == "laplace3d_32":
            M, kind = O.laplace_matrix_scipy(np.float64, 32, 3), BAND
        elif name == "long_rows":
            M = long_row_spd(20000, 20, np.random.default_rng(SEED))
            rp = M.indptr
            assert np.max(rp[512::512] - rp[:-512:512]) > 4096   # 512-row tiles overflow the stream at one lane per row
            kind = CSR
        else:
            M, kind = O.laplace_matrix_scipy(np.float64, 20, 2), None   # 400 rows: one level with max_levels = 1
        M = sp.csr_matrix(M)
        M.sort_indices()
        _MATS[name] = (M, kind)
    return _MATS[name]


def with_options(ctx, fn, **opts):
    old = {k: ctx.get_option(k) for k in opts}
    try:
        for k, v in opts.items():
            ctx.set_option(k, v)
        return fn()
    finally:
        for k, v in old.items():
            ctx.set_option(k, v)


def ldiv(isb, ctx, P, x):
    xd = isb.DeviceArray.from_numpy(ctx, x)
    yd = isb.DeviceArray(ctx, x.shape[0], x.dtype)
    P.ldiv_(yd, xd)
    return yd.numpy()


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", ["laplace3d_64", "long_rows"])
def test_vcycle_is_the_same_on_every_spmv_form(isb, ctx, name, dtype):
    M, fine_kind = matrix(name)
    A = isb.B200CSR.from_scipy(M.astype(dtype), ctx=ctx)
    P = isb.SmoothedAggregationPrec(A)
    kinds = level_kinds(isb, P)
    print(f"{name} {np.dtype(dtype).name}: rows per level {P.level_rows}, (A_l, P_l) forms {kinds}")
    assert kinds[0][0] == fine_kind
    sim = SimAMG(M)
    assert sim.status == 0
    x = np.random.default_rng(5).standard_normal(M.shape[0]).astype(dtype)
    y_ref = sim.vcycle(x, dtype)
    out = {}
    for bv in (1, 0):
        for form in (AUTO, SUBWARP, CSR, BAND):
            def run():
                y = ldiv(isb, ctx, P, x)
                assert ldiv(isb, ctx, P, x).tobytes() == y.tobytes(), (bv, form)   # run to run
                return y
            out[bv, form] = with_options(ctx, run, spmv_kernel=form, band_values=bv)
    for (bv, form), y in out.items():
        assert _rel(y, y_ref) <= TOL[dtype], (bv, form, _rel(y, y_ref))
        if form != SUBWARP:
            # the band stream forms each row sum in the CSR stream's order, with or without value tables
            assert y.tobytes() == out[1, AUTO].tobytes(), (bv, form)
    assert out[0, SUBWARP].tobytes() == out[1, SUBWARP].tobytes()


SWEEPS = [(0, 0), (0, 1), (1, 0), (1, 1), (2, 1), (1, 2), (3, 3)]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("pre, post", SWEEPS)
@pytest.mark.parametrize("name", ["laplace3d_32", "long_rows", "one_level"])
def test_vcycle_sweep_counts_match_the_serial_vcycle(isb, ctx, name, pre, post, dtype):
    M, _ = matrix(name)
    kw = dict(presweeps=pre, postsweeps=post)
    if name == "one_level":
        kw["max_levels"] = 1
    A = isb.B200CSR.from_scipy(M.astype(dtype), ctx=ctx)
    P = isb.SmoothedAggregationPrec(A, **kw)
    assert (len(P.level_rows) == 1) == (name == "one_level"), P.level_rows
    sim = SimAMG(M, **kw)
    assert sim.status == 0
    x = np.random.default_rng(7).standard_normal(M.shape[0]).astype(dtype)
    y_ref = sim.vcycle(x, dtype)
    xd = isb.DeviceArray.from_numpy(ctx, x)
    yd = isb.DeviceArray(ctx, M.shape[0], dtype)
    P.ldiv_(yd, xd)
    y = yd.numpy()
    assert _rel(y, y_ref) <= TOL[dtype], _rel(y, y_ref)
    P.ldiv_(xd, xd)                                            # ldiv!(P, x)
    assert xd.numpy().tobytes() == y.tobytes()
    if name != "one_level" and (pre, post) != (1, 1):
        # the counts change the result: a V-cycle that ran the default sweeps instead would fail the comparison above
        y11 = SimAMG(M).vcycle(x, dtype)
        assert _rel(y, y11) > 100 * TOL[dtype]


def test_cg_with_two_sweeps_each_matches_the_oracle(isb, ctx):
    # presweeps = postsweeps = 2 keeps the V-cycle symmetric, as cg! needs: equal iteration counts and histories
    A, _ = matrix("laplace3d_32")
    b = np.random.default_rng(1).standard_normal(A.shape[0])
    b /= np.linalg.norm(b)
    Ad = isb.B200CSR.from_scipy(A, ctx=ctx)
    P = isb.SmoothedAggregationPrec(Ad, presweeps=2, postsweeps=2)
    x, h = isb.cg(Ad, b, Pl=P, log=True)
    xo, ho = O.cg_(np.zeros(A.shape[0]), O.CSC.from_scipy(A), b, Pl=NumpySA(A, presweeps=2, postsweeps=2), log=True,
                   initially_zero=True)
    assert h.isconverged
    _check(h, ho, x, xo)
