"""The band-streamed SpMV (spmv_stream.cuh, spmv_kernel 0 / 3) against the CSR stream (spmv_kernel 2).

Operators whose 512-row tiles have at most 8 distinct offsets col - row are streamed as per-tile offsets, one mask byte
per row and staged x bands.  The row sums are taken in the same order with the same unfused operations, so every result
here is compared bit for bit: with the CSR stream, with the oracle's CSC scatter, and through cg! and minres!.
"""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu
SEED = 20261015
BAND, CSR = 3, 2


@pytest.fixture(scope="module")
def isb():
    import iterativesolvers_jl_b200 as m
    m.default_context()
    return m


def stream_kind(isb, A):
    kind, nbytes = C.c_int(), C.c_int64()
    assert isb.lib().b200_csr_stream_kind(A._h, C.byref(kind), C.byref(nbytes)) == 0
    return kind.value, nbytes.value


def with_kernel(isb, mode, fn):
    L, ctx = isb.lib(), isb.default_context()
    assert L.b200_ctx_set_option(ctx._h, b"spmv_kernel", mode) == 0
    try:
        return fn()
    finally:
        L.b200_ctx_set_option(ctx._h, b"spmv_kernel", 0)


def band_and_csr(isb, A, x):
    """A @ x with auto selection, with the band stream forced, and with the CSR stream."""
    return A @ x, with_kernel(isb, BAND, lambda: A @ x), with_kernel(isb, CSR, lambda: A @ x)


def check_band_kind(isb, A):
    kind, nbytes = stream_kind(isb, A)
    assert kind == BAND
    assert nbytes == ((A.m_local + 511) // 512) * 576   # 64-byte header + one mask byte per row, per 512-row tile


@pytest.mark.parametrize("N,dims", [(20, 3), (72, 3), (300, 2)])
def test_laplacian_band_equals_csr_and_oracle(isb, oracle, N, dims):
    rng = np.random.default_rng(SEED)
    O = oracle.laplace_matrix(np.float64, N, dims, base=1)
    A = isb.B200CSR.from_csc_arrays(O.colptr, O.rowval, O.nzval, O.shape, base=1)
    check_band_kind(isb, A)
    x = rng.standard_normal(O.n)
    y0, y3, y2 = band_and_csr(isb, A, x)
    yo = oracle.csc_spmv(O, x)
    assert np.array_equal(y2, yo)
    assert np.array_equal(y0, yo) and np.array_equal(y3, yo)


def test_advection_band_equals_csr_and_oracle(isb, oracle):
    rng = np.random.default_rng(SEED)
    M, _ = oracle.advection_dominated(30, 1000.0)
    O = oracle.CSC.from_scipy(M, base=1)
    A = isb.B200CSR.from_csc_arrays(O.colptr, O.rowval, O.nzval, O.shape, base=1)
    check_band_kind(isb, A)
    x = rng.standard_normal(O.n)
    y0, y3, y2 = band_and_csr(isb, A, x)
    yo = oracle.csc_spmv(O, x)
    assert np.array_equal(y2, yo) and np.array_equal(y0, yo) and np.array_equal(y3, yo)


def test_fp32_band_bitwise_equals_csr(isb, oracle):
    rng = np.random.default_rng(SEED)
    for N, dims in ((20, 3), (257, 2)):
        O = oracle.laplace_matrix(np.float32, N, dims, base=1)
        A = isb.B200CSR.from_csc_arrays(O.colptr, O.rowval, O.nzval, O.shape, base=1)
        check_band_kind(isb, A)
        x = rng.standard_normal(O.n).astype(np.float32)
        y0, y3, y2 = band_and_csr(isb, A, x)
        assert np.array_equal(y0, y2) and np.array_equal(y3, y2)


def random_banded(rng, m, n, noff, keep=0.8, empty_rows=0.05):
    """m x n matrix on <= noff random diagonals, with both corner diagonals when they exist, random missing entries and
    empty rows; sorted CSC."""
    lo, hi = -(m - 1), n - 1
    offs = {lo, hi} if noff >= 2 else {0}
    while len(offs) < min(noff, hi - lo + 1):
        offs.add(int(rng.integers(lo, hi + 1)))
    rows, cols = [], []
    for d in sorted(offs):
        r = np.arange(max(0, -d), min(m, n - d))
        rows.append(r)
        cols.append(r + d)
    rows, cols = np.concatenate(rows), np.concatenate(cols)
    keep_mask = rng.random(rows.size) < keep
    dead = rng.random(m) < empty_rows
    keep_mask &= ~dead[rows]
    if not keep_mask.any():
        keep_mask[0] = True
    rows, cols = rows[keep_mask], cols[keep_mask]
    vals = rng.standard_normal(rows.size)
    M = sp.csc_matrix((vals, (rows, cols)), shape=(m, n))
    M.sort_indices()
    return M


@pytest.mark.parametrize("n", [1, 7, 511, 512, 513, 4099, 300001])
def test_random_banded_matrices(isb, oracle, n):
    rng = np.random.default_rng(SEED + n)
    for noff in (1, 3, 8):
        M = random_banded(rng, n, n, noff)
        O = oracle.CSC.from_scipy(M, base=0)
        A = isb.B200CSR.from_scipy(M)
        check_band_kind(isb, A)
        x = rng.standard_normal(n)
        y0, y3, y2 = band_and_csr(isb, A, x)
        yo = oracle.csc_spmv(O, x)
        assert np.array_equal(y2, yo)
        assert np.array_equal(y0, yo) and np.array_equal(y3, yo)


@pytest.mark.parametrize("m,n", [(700, 1101), (1101, 700), (513, 4099)])
def test_rectangular_banded_matrices(isb, oracle, m, n):
    rng = np.random.default_rng(SEED + m + n)
    M = random_banded(rng, m, n, 8)
    O = oracle.CSC.from_scipy(M, base=0)
    A = isb.B200CSR.from_scipy(M)
    check_band_kind(isb, A)
    x = rng.standard_normal(n)
    y0, y3, y2 = band_and_csr(isb, A, x)
    yo = oracle.csc_spmv(O, x)
    assert np.array_equal(y2, yo) and np.array_equal(y0, yo) and np.array_equal(y3, yo)


def test_nine_offsets_in_one_tile_keeps_the_csr_stream(isb, oracle):
    rng = np.random.default_rng(SEED)
    n = 2000
    offs = [-300, -40, -1, 0, 1, 40, 300]
    M = sp.diags([rng.standard_normal(n - abs(d)) for d in offs], offs, shape=(n, n)).tolil()
    for r in range(600, 700):               # rows 600..699 get two more offsets
        M[r, r + 101] = 1.5
        M[r, r - 103] = -0.5
    M = M.tocsc()
    M.sort_indices()
    O = oracle.CSC.from_scipy(M, base=0)
    A = isb.B200CSR.from_scipy(M)
    kind, nbytes = stream_kind(isb, A)
    assert kind == CSR and nbytes == 4 * M.nnz + 4 * (n + 1)
    x = rng.standard_normal(n)
    y0, y3, y2 = band_and_csr(isb, A, x)
    yo = oracle.csc_spmv(O, x)
    assert np.array_equal(y0, yo) and np.array_equal(y3, yo) and np.array_equal(y2, yo)


def test_nonfinite_x_outside_the_referenced_columns(isb, oracle):
    """Bands copy x entries no row references; absent entries are skipped, never multiplied by zero."""
    rng = np.random.default_rng(SEED)
    n = 5000
    M = random_banded(rng, n, n, 5, keep=1.0, empty_rows=0.0).tolil()
    holes = rng.choice(n, size=60, replace=False)
    M[:, holes] = 0.0
    M = M.tocsc()
    M.eliminate_zeros()
    M.sort_indices()
    O = oracle.CSC.from_scipy(M, base=0)
    A = isb.B200CSR.from_scipy(M)
    check_band_kind(isb, A)
    x = rng.standard_normal(n)
    x[holes[::2]] = np.inf
    x[holes[1::2]] = np.nan
    y0, y3, y2 = band_and_csr(isb, A, x)
    assert np.all(np.isfinite(y2))
    np.testing.assert_array_equal(y0, y2)
    np.testing.assert_array_equal(y3, y2)
    np.testing.assert_array_equal(y2, oracle.csc_spmv(O, x))


def test_misaligned_x_view_takes_the_csr_stream(isb, oracle):
    """x 8 bytes past a 16-byte boundary cannot be bulk-copied: the launch takes the CSR stream and the result is the same."""
    rng = np.random.default_rng(SEED)
    ctx = isb.default_context()
    O = oracle.laplace_matrix(np.float64, 20, 3, base=1)
    A = isb.B200CSR.from_csc_arrays(O.colptr, O.rowval, O.nzval, O.shape, base=1)
    check_band_kind(isb, A)
    x = rng.standard_normal(O.n)
    buf = isb.DeviceArray.from_numpy(ctx, np.concatenate([[0.0], x]))
    assert buf.ptr % 16 == 0
    xv = isb.DeviceArray.view(ctx, buf.ptr + 8, O.n, np.float64)
    y = isb.DeviceArray.zeros(ctx, O.n)
    for mode in (0, BAND):
        with_kernel(isb, mode, lambda: A.mul_(y, xv))
        assert np.array_equal(y.numpy(), oracle.csc_spmv(O, x))


def test_cg_and_minres_band_bitwise_equal_csr(isb):
    L, ctx = isb.lib(), isb.default_context()
    rng = np.random.default_rng(SEED)
    A = isb.B200CSR.laplacian(72, 3)
    check_band_kind(isb, A)
    b = rng.standard_normal(A.m_local)
    b /= np.linalg.norm(b)
    assert L.b200_ctx_set_option(ctx._h, b"cg_persistent", 0) == 0
    try:
        out = {mode: with_kernel(isb, mode, lambda: isb.cg(A, b, log=True, maxiter=300)) for mode in (0, CSR)}
    finally:
        L.b200_ctx_set_option(ctx._h, b"cg_persistent", 1)
    (x0, h0), (x2, h2) = out[0], out[CSR]
    assert h0.niters == h2.niters > 50
    assert np.array_equal(h0["resnorm"], h2["resnorm"]) and np.array_equal(x0, x2)
    out = {mode: with_kernel(isb, mode, lambda: isb.minres(A, b, log=True, maxiter=120)) for mode in (BAND, CSR)}
    (x3, h3), (x2, h2) = out[BAND], out[CSR]
    assert len(h2["resnorm"]) > 50
    assert np.array_equal(h3["resnorm"], h2["resnorm"]) and np.array_equal(x3, x2)
