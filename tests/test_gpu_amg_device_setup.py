"""The smoothed-aggregation hierarchy built on the device (csrc/amg_setup.cu) against the serial setup of
csrc/amg_core.h (tests/hostsim_amg), byte for byte: every level's A and P (row offsets, columns and values rounded to
the element type), the aggregates and the coarsest level's inverse, in Float64 and Float32.  Also the refusals of
b200_amg_create with their codes and messages.
"""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import oracle as O
from test_amg_engine import MATRICES, SimAMG

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def isb():
    import iterativesolvers_jl_b200 as m
    return m


def arrow(N=80, eps=1e-3):
    """the 2-D Laplacian plus a dense first row and column of weak couplings: row 0 of A T, A P and R A P has more
    distinct columns than the on-chip SpGEMM table holds, and so do the rows of A P that reach column 0"""
    A = O.laplace_matrix_scipy(np.float64, N, 2).tolil()
    n = N * N
    for j in range(1, n):
        if A[0, j] == 0:
            A[0, j] = -eps
            A[j, 0] = -eps
    A[0, 0] = 4.0 + n * eps
    return A.tocsr()


DEVICE_MATRICES = dict(MATRICES)
DEVICE_MATRICES["laplace3d_64"] = (lambda: O.laplace_matrix_scipy(np.float64, 64, 3), {})
DEVICE_MATRICES["laplace3d_128"] = (lambda: O.laplace_matrix_scipy(np.float64, 128, 3), {})
DEVICE_MATRICES["advection_24"] = (lambda: O.advection_dominated(24)[0], {})
DEVICE_MATRICES["arrow_theta"] = (arrow, {"theta": 0.25})


def _same_csr(G, R, dtype, what):
    G = sp.csr_matrix(G)
    assert G.shape == R.shape, what
    assert np.array_equal(G.indptr.astype(np.int64), R.indptr.astype(np.int64)), what
    assert np.array_equal(G.indices.astype(np.int32), R.indices.astype(np.int32)), what
    assert G.data.astype(dtype).tobytes() == R.data.astype(dtype).tobytes(), what


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", sorted(DEVICE_MATRICES))
def test_device_hierarchy_is_the_serial_setups_bit_for_bit(isb, name, dtype):
    make, kw = DEVICE_MATRICES[name]
    A = sp.csr_matrix(make()).astype(dtype)
    A.sort_indices()
    sim = SimAMG(A.astype(np.float64), **kw)                      # the setup runs in fp64 on A's values
    assert sim.status == 0, (sim.status, sim.bad)
    ref = sim.levels()
    P = isb.SmoothedAggregationPrec(isb.B200CSR.from_scipy(A), **kw)
    got = P.levels()
    assert len(got) == len(ref)
    for l, (g, r) in enumerate(zip(got, ref)):
        _same_csr(g["A"], r["A"], dtype, ("A", l))
        if r["P"] is None:
            assert g["P"] is None and g["agg"] is None
            assert g["inv"].astype(dtype).tobytes() == r["inv"].astype(dtype).tobytes(), ("inv", l)
        else:
            _same_csr(g["P"], r["P"], dtype, ("P", l))
            assert np.array_equal(g["agg"], r["agg"]), ("agg", l)
    assert set(P.setup_seconds) == {"download", "aggregation", "prolongator", "rap", "upload"}


def test_arrow_rows_overflow_the_on_chip_table():
    A = arrow()
    L = SimAMG(A, theta=0.25).levels()
    AP = L[0]["A"] @ L[0]["P"]
    assert (np.diff(AP.indptr) > 512).sum() > 1
    RAP = L[0]["P"].T @ AP
    assert np.diff(RAP.indptr).max() > 512


def _create(isb, A, **kw):
    o = dict(theta=0.0, max_levels=10, max_coarse=10, presweeps=1, postsweeps=1)
    o.update(kw)
    opts = isb._lib.AmgOpts(o["theta"], o["max_levels"], o["max_coarse"], o["presweeps"], o["postsweeps"])
    h = C.c_void_p()
    st = isb.lib().b200_amg_create(A.ctx._h, A._h, C.byref(opts), C.byref(h))
    return st, isb.lib().b200_last_error().decode(), h


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_refusals_keep_their_codes_and_messages(isb, dtype):
    # a row whose columns are not ascending (row 2), checked before the diagonal (row 1 is zero)
    rowptr = np.array([0, 2, 4, 6], dtype=np.int32)
    colind = np.array([0, 1, 0, 2, 2, 1], dtype=np.int32)
    vals = np.array([2, -1, -1, 0, 2, -1], dtype=dtype)
    st, msg, h = _create(isb, isb.B200CSR.from_csr_slab(rowptr, colind, vals, 3))
    assert (st, msg) == (-1, "AMG needs rows with ascending column indices (row 2)") and not h.value
    zero = sp.csr_matrix(np.array([[2.0, -1, 0], [-1, 0, -1], [0, -1, 2]], dtype=dtype))
    st, msg, h = _create(isb, isb.B200CSR.from_scipy(zero), max_coarse=1)
    assert (st, msg) == (-5, "smoothed aggregation: zero or missing diagonal entry in row 1 (0-based) of level 0")
    st, msg, h = _create(isb, isb.B200CSR.from_scipy(zero))          # checked even when A is the coarsest level
    assert (st, msg) == (-5, "smoothed aggregation: zero or missing diagonal entry in row 1 (0-based) of level 0")
    big = isb.B200CSR.from_scipy(O.laplace_matrix_scipy(np.float64, 70, 2).astype(dtype))
    st, msg, h = _create(isb, big, max_levels=1)
    assert (st, msg) == (-1, "smoothed aggregation: the coarsest level (level 0) has 4900 rows, more than the 4096 its "
                             "dense inverse allows; raise max_levels or lower max_coarse")
    singular = sp.csr_matrix(np.array([[1.0, 1.0], [1.0, 1.0]], dtype=dtype))
    st, msg, h = _create(isb, isb.B200CSR.from_scipy(singular))
    assert (st, msg) == (-5, "smoothed aggregation: the coarsest level (level 0) is singular: zero pivot in column 1 "
                             "(0-based)")
