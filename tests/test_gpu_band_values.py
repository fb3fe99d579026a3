"""Value tables of the band stream (csr.cu k_band_values, spmv_stream.cuh): a 512-row band tile in which every offset
holds one single value (the same bit pattern) is streamed as its 8 values instead of its vals.

The row sums multiply the same numbers in the same order, so every result here is compared bit for bit: context option
"band_values" 1 against 0, against the CSR stream and against the oracle's CSC scatter, and through cg!, minres! and
gmres!.  The number of uniform tiles is checked against a numpy restatement of the rule.
"""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu
SEED = 20261016
BAND, CSR = 3, 2
R = 512


@pytest.fixture(scope="module")
def isb():
    import iterativesolvers_jl_b200 as m
    m.default_context()
    return m


def with_options(ctx, opts, fn):
    old = {k: ctx.get_option(k) for k in opts}
    for k, v in opts.items():
        ctx.set_option(k, v)
    try:
        return fn()
    finally:
        for k, v in old.items():
            ctx.set_option(k, v)


def stream_kind(isb, A):
    kind, nbytes = C.c_int(), C.c_int64()
    assert isb.lib().b200_csr_stream_kind(A._h, C.byref(kind), C.byref(nbytes)) == 0
    return kind.value, nbytes.value


def uniform_rule(A):
    """(uniform tiles, value bytes) of the downloaded CSR: a tile is uniform when, per offset col - row, all of its
    nonzeros have the same bit pattern."""
    rowptr, colind, vals = A.download()
    rowptr = rowptr.astype(np.int64)
    m, V = A.m_local, vals.dtype.itemsize
    ntiles = (m + R - 1) // R
    rows = np.repeat(np.arange(m, dtype=np.int64), np.diff(rowptr))
    bits = vals.view(np.uint64 if V == 8 else np.uint32)
    tile, off = rows // R, colind.astype(np.int64) - rows
    order = np.lexsort((bits, off, tile))
    tile, off, bits = tile[order], off[order], bits[order]
    start = np.ones(tile.size, bool)
    start[1:] = (tile[1:] != tile[:-1]) | (off[1:] != off[:-1])
    first = np.flatnonzero(start)
    last = np.append(first[1:], tile.size) - 1
    mixed_tiles = np.unique(tile[first[bits[first] != bits[last]]])
    uniform = np.ones(ntiles, bool)
    uniform[mixed_tiles] = False
    tile_nnz = rowptr[np.minimum(np.arange(1, ntiles + 1) * R, m)] - rowptr[np.arange(ntiles) * R]
    return int(uniform.sum()), V * int(8 * uniform.sum() + tile_nnz[~uniform].sum()), uniform


def check_spmv(isb, A, x, O=None, oracle=None):
    """A x with band_values 1 and 0 and with the CSR stream, bitwise equal (and to the oracle's scatter when given)."""
    ctx = A.ctx
    y1 = with_options(ctx, {"band_values": 1}, lambda: A @ x)
    y0 = with_options(ctx, {"band_values": 0}, lambda: A @ x)
    y2 = with_options(ctx, {"spmv_kernel": CSR}, lambda: A @ x)
    assert np.array_equal(y1.view(np.uint8), y0.view(np.uint8))
    assert np.array_equal(y1.view(np.uint8), y2.view(np.uint8))
    if O is not None:
        assert np.array_equal(y1, oracle.csc_spmv(O, x))


def check_counts(A, expect_all=None):
    u, vb = A.band_values
    ru, rvb, uniform = uniform_rule(A)
    assert (u, vb) == (ru, rvb)
    if expect_all is not None:
        assert (u == uniform.size) == expect_all
    return uniform


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("N,dims", [(1, 2), (511, 2), (512, 2), (513, 2), (1, 3), (9, 3), (72, 3)])
def test_laplacian_every_tile_uniform(isb, oracle, N, dims, dtype):
    rng = np.random.default_rng(SEED + N + dims)
    O = oracle.laplace_matrix(dtype, N, dims, base=1)
    for A in (isb.B200CSR.from_csc_arrays(O.colptr, O.rowval, O.nzval, O.shape, base=1),
              isb.B200CSR.laplacian(N, dims, dtype)):
        assert stream_kind(isb, A)[0] == BAND
        check_counts(A, expect_all=True)
        ntiles = (A.m_local + R - 1) // R
        assert A.band_values == (ntiles, ntiles * 8 * np.dtype(dtype).itemsize)
        x = rng.standard_normal(O.n).astype(dtype)
        check_spmv(isb, A, x, O if dtype == np.float64 else None, oracle)


def test_advection_every_tile_uniform(isb, oracle):
    rng = np.random.default_rng(SEED)
    M, _ = oracle.advection_dominated(30, 1000.0)
    O = oracle.CSC.from_scipy(M, base=1)
    A = isb.B200CSR.from_csc_arrays(O.colptr, O.rowval, O.nzval, O.shape, base=1)
    assert stream_kind(isb, A)[0] == BAND
    check_counts(A, expect_all=True)
    check_spmv(isb, A, rng.standard_normal(O.n), O, oracle)


@pytest.mark.parametrize("row", [3 * R, 4 * R - 1, 7950])
def test_one_ulp_makes_exactly_one_tile_stream_its_values(isb, oracle, row):
    """20^3 = 8000 rows: 15 full tiles and a partial one (rows 7680..7999).  One diagonal entry moved by 1 ulp, in a
    tile's first row, its last row, or the partial tile."""
    rng = np.random.default_rng(SEED + row)
    M = oracle.laplace_matrix_scipy(np.float64, 20, 3).tocsr()
    M.sort_indices()
    k = M.indptr[row] + int(np.flatnonzero(M.indices[M.indptr[row]:M.indptr[row + 1]] == row)[0])
    M.data[k] = np.nextafter(M.data[k], np.inf)
    M = M.tocsc()
    O = oracle.CSC.from_scipy(M, base=0)
    A = isb.B200CSR.from_scipy(M)
    uniform = check_counts(A)
    assert np.flatnonzero(~uniform).tolist() == [row // R]
    check_spmv(isb, A, rng.standard_normal(M.shape[0]), O, oracle)


def test_signed_zeros_are_not_merged(isb, oracle):
    n = 2 * R
    d = np.arange(n)
    up = d[:-1]
    vals_up = np.where(up % 2 == 0, 0.0, -0.0)   # +0.0 and -0.0 on offset +1 of both tiles
    vals_up[R:] = 0.0                             # the second tile holds +0.0 only
    rows = np.concatenate([d, up])
    cols = np.concatenate([d, up + 1])
    vals = np.concatenate([np.full(n, 2.0), vals_up])
    M = sp.csc_matrix((vals, (rows, cols)), shape=(n, n))
    M.sort_indices()
    assert M.nnz == rows.size   # explicit zeros are kept
    A = isb.B200CSR.from_scipy(M)
    assert stream_kind(isb, A)[0] == BAND
    uniform = check_counts(A)
    assert uniform.tolist() == [False, True]
    x = np.random.default_rng(SEED).standard_normal(n)
    x[::3] = 0.0
    check_spmv(isb, A, x, oracle.CSC.from_scipy(M, base=0), oracle)


@pytest.mark.parametrize("n", [513, 4099, 100003])
def test_random_banded_follows_the_rule(isb, oracle, n):
    """random values: only slots holding a single nonzero can be uniform, so few tiles (if any) are."""
    rng = np.random.default_rng(SEED + n)
    for noff in (1, 3, 8):
        offs = sorted({0} | {int(v) for v in rng.integers(-n + 1, n, size=noff - 1)})
        M = sp.diags([rng.standard_normal(n - abs(o)) for o in offs], offs, shape=(n, n), format="csc")
        M.sort_indices()
        A = isb.B200CSR.from_scipy(M)
        assert stream_kind(isb, A)[0] == BAND
        check_counts(A)
        check_spmv(isb, A, rng.standard_normal(n), oracle.CSC.from_scipy(M, base=0), oracle)


def test_eight_byte_row_offsets(isb, oracle):
    rng = np.random.default_rng(SEED)
    ctx = isb.Context(0)
    ctx.set_option("rowptr64", 1)
    O = oracle.laplace_matrix(np.float64, 40, 3, base=1)
    A = isb.B200CSR.from_csc_arrays(O.colptr, O.rowval, O.nzval, O.shape, base=1, ctx=ctx)
    assert A.index_bytes == 8 and stream_kind(isb, A)[0] == BAND
    check_counts(A, expect_all=True)
    check_spmv(isb, A, rng.standard_normal(O.n), O, oracle)
    M = oracle.laplace_matrix_scipy(np.float64, 40, 3).tocsr()
    M.sort_indices()
    k = M.indptr[5 * R + 7]
    M.data[k] = np.nextafter(M.data[k], -np.inf)
    M = M.tocsc()
    M.sort_indices()
    B = isb.B200CSR.from_scipy(M, ctx=ctx)
    assert B.index_bytes == 8
    uniform = check_counts(B)
    assert np.flatnonzero(~uniform).tolist() == [5]
    check_spmv(isb, B, rng.standard_normal(O.n), oracle.CSC.from_scipy(M, base=0), oracle)


def test_misaligned_x_view_takes_the_csr_stream(isb, oracle):
    rng = np.random.default_rng(SEED)
    ctx = isb.default_context()
    O = oracle.laplace_matrix(np.float64, 20, 3, base=1)
    A = isb.B200CSR.from_csc_arrays(O.colptr, O.rowval, O.nzval, O.shape, base=1)
    x = rng.standard_normal(O.n)
    buf = isb.DeviceArray.from_numpy(ctx, np.concatenate([[0.0], x]))
    xv = isb.DeviceArray.view(ctx, buf.ptr + 8, O.n, np.float64)
    y = isb.DeviceArray.zeros(ctx, O.n)
    for bv in (1, 0):
        with_options(ctx, {"band_values": bv}, lambda: A.mul_(y, xv))
        assert np.array_equal(y.numpy(), oracle.csc_spmv(O, x))


def test_solvers_bitwise_equal_with_and_without_tables(isb):
    ctx = isb.default_context()
    rng = np.random.default_rng(SEED)
    A = isb.B200CSR.laplacian(72, 3)
    assert A.band_values[0] == (A.m_local + R - 1) // R
    b = rng.standard_normal(A.m_local)
    b /= np.linalg.norm(b)
    runs = {
        "cg": lambda: isb.cg(A, b, log=True, maxiter=300),
        "minres": lambda: isb.minres(A, b, log=True, maxiter=120),
        "gmres": lambda: isb.gmres(A, b, log=True, restart=20, maxiter=60),
    }
    for name, run in runs.items():
        out = {bv: with_options(ctx, {"band_values": bv, "cg_persistent": 0}, run) for bv in (1, 0)}
        (x1, h1), (x0, h0) = out[1], out[0]
        assert len(h1["resnorm"]) > 20, name
        assert np.array_equal(h1["resnorm"], h0["resnorm"]), name
        assert np.array_equal(x1, x0), name


def test_value_bytes_query(isb, oracle):
    # all uniform
    A = isb.B200CSR.laplacian(16, 3)
    ntiles = (A.m_local + R - 1) // R
    assert A.band_values == (ntiles, 64 * ntiles)
    # mixed: tile 2 holds one changed value
    M = oracle.laplace_matrix_scipy(np.float64, 16, 3).tocsr()
    M.sort_indices()
    M.data[M.indptr[2 * R + 5] + 1] *= 3.0
    B = isb.B200CSR.from_scipy(M)
    tile_nnz = M.indptr[3 * R] - M.indptr[2 * R]
    assert B.band_values == (ntiles - 1, 64 * (ntiles - 1) + 8 * tile_nnz)
    # CSR stream: every value is read
    n = 2000
    offs = [-300, -40, -1, 0, 1, 40, 300]
    C9 = sp.diags([np.ones(n - abs(d)) for d in offs], offs, shape=(n, n)).tolil()
    for r in range(600, 700):
        C9[r, r + 101] = 1.5
        C9[r, r - 103] = -0.5
    C9 = C9.tocsc()
    D = isb.B200CSR.from_scipy(C9)
    assert stream_kind(isb, D)[0] == CSR
    assert D.band_values == (0, 8 * C9.nnz)
