"""cg! with the kernels of an iteration chained by programmatic dependent launch (context option "pdl" = 1).

With "pdl" = 1, cg.cu launches k_pcg_precond, k_cg_update_u, the K2 SpMV (CgDotEpi) and k_cg_update_r with
launch_chained: each kernel's blocks may start before the previous kernel has finished, and wait in pdl_wait() before
they touch its results.  The arithmetic is the same, so the run must be the same bits as with "pdl" = 0: residual
history, x and iteration count.  "cg_persistent" = 0 throughout: the operators up to 2^18 rows would otherwise run the
whole loop in k_cg_persistent, which is not chained.

A host read of the done flag between two iterations ends the chain there, so K3 -> K1 of plain CG is chained only when
check_every > 1.  That link once lost the last iteration's x update: K1 took its CgScal as const __restrict__, and the
compiler loaded s->done through the read-only path ahead of pdl_wait(), so the K1 behind the converging iteration saw
done = 0, updated x and u, and k_cg_flush_x then added alpha times the wrong u (residual history unchanged, x off in
the last bits).

Covered: CG and Jacobi PCG, each SpMV form (1 sub-warp, 2 CSR stream, 3 band stream) on the 72^3 Laplacian (band) and on
a long-row operator (CSR stream with several lanes per row), Float64 and Float32, a nonzero initial guess, runs stopped
by maxiter and by convergence, host checks of the done flag after every iteration and after every 32, and an operator
with 8-byte row offsets.  The partitioned CG's chained k_halo_push is not covered: tests/dist_worker.py sets no context
option but "comm".
"""
import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu
SEED = 20261016
SUBWARP, CSR, BAND = 1, 2, 3


@pytest.fixture(scope="module")
def isb():
    import iterativesolvers_jl_b200 as m
    return m


@pytest.fixture(scope="module")
def ctx(isb):
    # this module's own context, so that "pdl" = 1 or a forced form never reaches another test
    c = isb.Context(0)
    c.set_option("cg_persistent", 0)
    return c


def long_row_spd(n, per_row, rng):
    """Symmetric, strictly diagonally dominant (so SPD) n x n matrix with about per_row + 1 nonzeros per row."""
    M = sp.random(n, n, density=per_row / (2 * n), random_state=rng, format="csr")
    M = M + M.T
    M = M + sp.diags(np.asarray(abs(M).sum(axis=1)).ravel() + 0.05)
    return M.tocsc()


_OPS = {}


def operator(isb, ctx, name, dtype):
    key = (name, np.dtype(dtype).name)
    if key not in _OPS:
        if name == "laplace72":
            A = isb.B200CSR.laplacian(72, 3, dtype, ctx=ctx)
        else:
            M = long_row_spd(20000, 20, np.random.default_rng(SEED)).astype(dtype)
            rp = M.tocsr().indptr
            assert np.max(rp[512::512] - rp[:-512:512]) > 4096   # the CSR stream runs with several lanes per row
            A = isb.B200CSR.from_scipy(M, ctx=ctx)
        _OPS[key] = A
    return _OPS[key]


def both(isb, ctx, A, b, x0, **kw):
    """cg! with "pdl" 0 and 1: ((x, history) for 0, (x, history) for 1)"""
    out = []
    for pdl in (0, 1):
        ctx.set_option("pdl", pdl)
        try:
            x = x0.copy()
            out.append(isb.cg_(x, A, b, log=True, **kw))
        finally:
            ctx.set_option("pdl", 0)
    return out


def same(r0, r1):
    (x0, h0), (x1, h1) = r0, r1
    assert (h1.niters, h1.isconverged) == (h0.niters, h0.isconverged)
    assert np.asarray(h1["resnorm"]).tobytes() == np.asarray(h0["resnorm"]).tobytes()
    assert x1.tobytes() == x0.tobytes()


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("prec", ["none", "jacobi"])
@pytest.mark.parametrize("form", [SUBWARP, CSR, BAND])
@pytest.mark.parametrize("name", ["laplace72", "long_rows"])
def test_pdl_chain_gives_the_same_bits(isb, ctx, name, form, prec, dtype):
    A = operator(isb, ctx, name, dtype)
    rng = np.random.default_rng(SEED + form)
    b = rng.standard_normal(A.m_local).astype(dtype)
    x0 = (0.1 * rng.standard_normal(A.m_local)).astype(dtype)
    Pl = isb.JacobiPrec(A.diag()) if prec == "jacobi" else None
    ctx.set_option("spmv_kernel", form)
    try:
        # stopped by maxiter, the done flag read after every iteration, from a nonzero guess
        r0, r1 = both(isb, ctx, A, b, x0, Pl=Pl, maxiter=5, check_every=1)
        same(r0, r1)
        assert r0[1].niters == 5 and not r0[1].isconverged
        # stopped by convergence, the flag read after every 32 iterations (the long-row operator converges within the
        # first 32, so the chained launches behind its stop run as no-ops), from zero
        r0, r1 = both(isb, ctx, A, b, np.zeros_like(x0), Pl=Pl, initially_zero=True, check_every=32)
        same(r0, r1)
        assert r0[1].isconverged and r0[1].niters > 5, r0[1].niters
    finally:
        ctx.set_option("spmv_kernel", 0)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_pdl_chain_with_8_byte_row_offsets(isb, dtype):
    c = isb.Context(0)
    c.set_option("rowptr64", 1)
    c.set_option("cg_persistent", 0)
    A = isb.B200CSR.laplacian(48, 3, dtype, ctx=c)
    assert A.index_bytes == 8
    rng = np.random.default_rng(SEED)
    b = rng.standard_normal(A.m_local).astype(dtype)
    x0 = (0.1 * rng.standard_normal(A.m_local)).astype(dtype)
    for Pl in (None, isb.JacobiPrec(A.diag())):
        r0, r1 = both(isb, c, A, b, x0, Pl=Pl, check_every=7)
        same(r0, r1)
        assert r0[1].isconverged
