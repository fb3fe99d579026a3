"""cg!'s K2 (c = A u fused with dot(u, c)) and minres!'s Ka (Lanczos update fused with dot(v_curr, v_next)) in each SpMV
form: sub-warp per row (spmv_kernel 1), CSR stream (2) and band stream (3).

The sub-warp form sums a row in another order than the streams, so its residual histories agree to rounding only; the
band stream forms every row sum and partial dot in the CSR stream's order, so those two agree bit for bit.  The long-row
operator's 512-row tiles exceed the stream's 4096 nonzeros, so its CSR stream runs with several lanes per row.
"""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu
SEED = 20261015
SUBWARP, CSR, BAND = 1, 2, 3


@pytest.fixture(scope="module")
def isb():
    import iterativesolvers_jl_b200 as m
    L, ctx = m.lib(), m.default_context()
    assert L.b200_ctx_set_option(ctx._h, b"cg_persistent", 0) == 0   # small operators would run k_cg_persistent instead
    yield m
    L.b200_ctx_set_option(ctx._h, b"cg_persistent", 1)


def stream_kind(isb, A):
    kind, nbytes = C.c_int(), C.c_int64()
    assert isb.lib().b200_csr_stream_kind(A._h, C.byref(kind), C.byref(nbytes)) == 0
    return kind.value


def with_kernel(isb, mode, fn):
    L, ctx = isb.lib(), isb.default_context()
    assert L.b200_ctx_set_option(ctx._h, b"spmv_kernel", mode) == 0
    try:
        return fn()
    finally:
        L.b200_ctx_set_option(ctx._h, b"spmv_kernel", 0)


def long_row_spd(n, per_row, rng):
    """Symmetric, strictly diagonally dominant (so SPD) n x n matrix with about per_row + 1 nonzeros per row."""
    M = sp.random(n, n, density=per_row / (2 * n), random_state=rng, format="csr")
    M = M + M.T
    M = M + sp.diags(np.asarray(abs(M).sum(axis=1)).ravel() + 0.05)
    M = M.tocsc()
    M.sort_indices()
    return M


def operator(isb, name, rng):
    if name == "laplace72":
        A = isb.B200CSR.laplacian(72, 3)
        assert stream_kind(isb, A) == BAND
        return A
    M = long_row_spd(20000, 20, rng)
    rp = M.tocsr().indptr
    assert np.max(rp[512::512] - rp[:-512:512]) > 4096   # 512-row tiles overflow the stream at one lane per row
    A = isb.B200CSR.from_scipy(M)
    assert stream_kind(isb, A) == CSR
    return A


@pytest.mark.parametrize("solver,maxiter", [("cg", 120), ("minres", 120)])
@pytest.mark.parametrize("name", ["laplace72", "long_rows"])
def test_fused_spmv_forms_agree(isb, name, solver, maxiter):
    rng = np.random.default_rng(SEED)
    A = operator(isb, name, rng)
    b = rng.standard_normal(A.m_local)
    b /= np.linalg.norm(b)
    run = getattr(isb, solver)
    out = {mode: with_kernel(isb, mode, lambda: run(A, b, log=True, maxiter=maxiter)) for mode in (SUBWARP, CSR, BAND)}
    (x1, h1), (x2, h2), (x3, h3) = out[SUBWARP], out[CSR], out[BAND]
    assert len(h2["resnorm"]) > 20
    assert len(h1["resnorm"]) == len(h2["resnorm"])
    np.testing.assert_allclose(h1["resnorm"], h2["resnorm"], rtol=1e-9, atol=0)
    assert np.array_equal(h3["resnorm"], h2["resnorm"]) and np.array_equal(x3, x2)
