"""Operators with 8-byte row offsets (b200_csr_index_bytes == 8).

Small matrices are built twice, on a context with "rowptr64" = 0 (4-byte offsets) and on one with "rowptr64" = 1
(8-byte offsets, forced): the two run the same forms in the same order, so every product, residual history and
solution must agree bit for bit.  One real operator above 2^31 nonzeros (the 7-point Laplacian at 680^3) is checked
against the same stencil evaluated with torch, when the GPU has the memory for it.
"""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu
SEED = 20261015
SUBWARP, CSR, BAND = 1, 2, 3
ERR_UNSUPPORTED = -6


@pytest.fixture(scope="module")
def isb():
    import iterativesolvers_jl_b200 as m
    return m


@pytest.fixture(scope="module")
def ctxs(isb):
    # kept open for the process: an operator still referenced (e.g. by a failed test's traceback) must not outlive its
    # context
    out = {}
    for bytes_, opt in ((4, 0), (8, 1)):
        c = isb.Context(0)
        c.set_option("rowptr64", opt)
        c.set_option("cg_persistent", 0)   # the 4-byte operator would run k_cg_persistent, the 8-byte one cannot
        out[bytes_] = c
    return out


def laplace3(N):
    T = sp.diags([-np.ones(N - 1), 2 * np.ones(N), -np.ones(N - 1)], [-1, 0, 1])
    I = sp.identity(N)
    return (sp.kron(sp.kron(I, I), T) + sp.kron(sp.kron(I, T), I) + sp.kron(sp.kron(T, I), I)).tocsc()


def long_row_spd(n, per_row, rng):
    M = sp.random(n, n, density=per_row / (2 * n), random_state=rng, format="csr")
    M = M + M.T
    M = M + sp.diags(np.asarray(abs(M).sum(axis=1)).ravel() + 0.05)
    return M.tocsc()


def random_nonsym(n, per_row, rng):
    """non-symmetric, diagonally dominant; 16-row tiles exceed the CSR stream's 4096 nonzeros (sub-warp form)."""
    M = sp.random(n, n, density=per_row / n, random_state=rng, format="csr")
    M = M + sp.diags(np.asarray(abs(M).sum(axis=1)).ravel() + 1.0)
    return M.tocsc()


MATRICES = {"laplace72": BAND, "long_rows": CSR, "random": SUBWARP}


@pytest.fixture(scope="module")
def mats():
    rng = np.random.default_rng(SEED)
    out = {"laplace72": laplace3(72), "long_rows": long_row_spd(20000, 20, rng), "random": random_nonsym(3000, 300, rng)}
    for M in out.values():
        M.sort_indices()
    return out


def build(isb, ctxs, M, nbytes, dtype=np.float64):
    M = M.astype(dtype)
    A = isb.B200CSR.from_scipy(M, ctx=ctxs[nbytes])
    assert A.index_bytes == nbytes
    return A


def stream_kind(isb, A):
    kind, nbytes = C.c_int(), C.c_int64()
    assert isb.lib().b200_csr_stream_kind(A._h, C.byref(kind), C.byref(nbytes)) == 0
    return kind.value, nbytes.value


def pair(isb, ctxs, mats, name, dtype=np.float64):
    return build(isb, ctxs, mats[name], 4, dtype), build(isb, ctxs, mats[name], 8, dtype)


@pytest.mark.parametrize("name", list(MATRICES))
def test_forms_and_structure_bytes(isb, ctxs, mats, name):
    A4, A8 = pair(isb, ctxs, mats, name)
    (k4, b4), (k8, b8) = stream_kind(isb, A4), stream_kind(isb, A8)
    assert k4 == k8 == MATRICES[name]
    if k4 == BAND:
        assert b8 == b4
    else:   # 4 more bytes per row offset
        assert b8 == b4 + 4 * (A4.m_local + 1)


@pytest.mark.parametrize("dtype", [np.float64, np.float32, np.complex128, np.complex64])
@pytest.mark.parametrize("kernel", [0, 1, 2, 3])
@pytest.mark.parametrize("name", list(MATRICES))
def test_mul_bitwise(isb, ctxs, mats, name, kernel, dtype):
    M = mats[name]
    if np.iscomplexobj(np.empty(0, dtype)):
        M = M + 1j * sp.csc_matrix((np.sin(np.arange(M.nnz)), M.indices, M.indptr), shape=M.shape)
        M.sort_indices()
    rng = np.random.default_rng(SEED)
    x = rng.standard_normal(M.shape[1]).astype(dtype)
    if np.iscomplexobj(x):
        x = x + 1j * rng.standard_normal(M.shape[1]).astype(dtype)
    ys = {}
    for nb in (4, 8):
        A = build(isb, ctxs, M, nb, dtype)
        ctxs[nb].set_option("spmv_kernel", kernel)
        try:
            ys[nb] = A @ x
        finally:
            ctxs[nb].set_option("spmv_kernel", 0)
    assert np.array_equal(ys[4], ys[8])
    ref = (M.astype(np.complex128 if np.iscomplexobj(x) else np.float64) @ x.astype(np.complex128 if np.iscomplexobj(x) else np.float64))
    tol = 1e-12 if dtype in (np.float64, np.complex128) else 1e-4
    assert np.max(np.abs(ys[8] - ref)) <= tol * np.max(np.abs(ref))


def _same(h4, h8):
    assert (h4.iters, h4.mvps, h4.mtvps) == (h8.iters, h8.mvps, h8.mtvps)
    assert h4.data.keys() == h8.data.keys()
    for k in h4.data:
        assert np.array_equal(np.asarray(h4[k]), np.asarray(h8[k])), k


def _rhs(n):
    b = np.random.default_rng(SEED).standard_normal(n)
    return b / np.linalg.norm(b)


def _gershgorin(M):
    return float(np.max(np.asarray(abs(M).sum(axis=1)).ravel()))


SOLVERS = {
    "cg": (lambda isb, A, b, M: isb.cg(A, b, log=True, maxiter=40), True),
    "cg_jacobi": (lambda isb, A, b, M: isb.cg(A, b, log=True, maxiter=40, Pl=isb.JacobiPrec(A.diag())), True),
    "gmres_mgs": (lambda isb, A, b, M: isb.gmres(A, b, log=True, maxiter=40, restart=15, orth_meth="mgs"), False),
    "gmres_cgs": (lambda isb, A, b, M: isb.gmres(A, b, log=True, maxiter=40, restart=15, orth_meth="cgs"), False),
    "gmres_dgks": (lambda isb, A, b, M: isb.gmres(A, b, log=True, maxiter=40, restart=15, orth_meth="dgks"), False),
    "minres": (lambda isb, A, b, M: isb.minres(A, b, log=True, maxiter=40), True),
    "bicgstabl2": (lambda isb, A, b, M: isb.bicgstabl(A, b, 2, log=True, max_mv_products=60,
                                                      rng=np.random.default_rng(SEED)), False),
    "bicgstabl4": (lambda isb, A, b, M: isb.bicgstabl(A, b, 4, log=True, max_mv_products=60,
                                                      rng=np.random.default_rng(SEED)), False),
    "chebyshev": (lambda isb, A, b, M: isb.chebyshev(A, b, 1e-2, _gershgorin(M), log=True, maxiter=40), True),
    "idrs": (lambda isb, A, b, M: isb.idrs(A, b, log=True, maxiter=40, rng=np.random.default_rng(SEED)), False),
    "qmr": (lambda isb, A, b, M: isb.qmr(A, b, log=True, maxiter=40), False),
    "lsqr": (lambda isb, A, b, M: isb.lsqr(A, b, log=True, maxiter=40), False),
    "lsmr": (lambda isb, A, b, M: isb.lsmr(A, b, log=True, maxiter=40), False),
}


@pytest.mark.parametrize("solver", list(SOLVERS))
@pytest.mark.parametrize("name", list(MATRICES))
def test_solvers_bitwise(isb, ctxs, mats, name, solver):
    run, spd_only = SOLVERS[solver]
    if spd_only and name == "random":
        pytest.skip("needs a symmetric positive definite operator")
    A4, A8 = pair(isb, ctxs, mats, name)
    b = _rhs(A4.m_local)
    x4, h4 = run(isb, A4, b, mats[name])
    x8, h8 = run(isb, A8, b, mats[name])
    assert h4.iters > 0
    _same(h4, h8)
    assert np.array_equal(x4, x8)


@pytest.mark.parametrize("name", ["laplace72", "long_rows"])
def test_lobpcg_fp32_block16(isb, ctxs, mats, name):
    A4, A8 = pair(isb, ctxs, mats, name, np.float32)
    X0 = np.random.default_rng(SEED).random((A4.m_local, 16)).astype(np.float32)
    r4 = isb.lobpcg(A4, False, X0, maxiter=6, _fixed_iterations=True)
    r8 = isb.lobpcg(A8, False, X0, maxiter=6, _fixed_iterations=True)
    assert r4.iterations == r8.iterations
    assert np.array_equal(r4.lam, r8.lam)


def test_transpose_and_download(isb, ctxs, mats):
    M = mats["random"]
    A8 = build(isb, ctxs, M, 8)
    rp, ci, v = A8.download()
    R = M.tocsr()
    assert rp.dtype == np.int64
    assert np.array_equal(rp, R.indptr) and np.array_equal(ci, R.indices) and np.array_equal(v, R.data)
    At = A8.adjoint()
    assert At.index_bytes == 8
    rp, ci, v = At.download()
    Rt = M.conj().T.tocsr()
    Rt.sort_indices()
    assert np.array_equal(rp, Rt.indptr) and np.array_equal(ci, Rt.indices) and np.array_equal(v, Rt.data)
    # the 4-byte operator downloads through the same 64-bit entry
    rp4, ci4, v4 = build(isb, ctxs, M, 4).download()
    assert rp4.dtype == np.int32 and np.array_equal(rp4, R.indptr)


def test_laplacian_and_slab_constructors(isb, ctxs):
    A = isb.B200CSR.laplacian(20, 3, ctx=ctxs[8])
    assert A.index_bytes == 8 and stream_kind(isb, A)[0] == BAND
    R = laplace3(20).tocsr()
    rp, ci, v = A.download()
    assert np.array_equal(rp, R.indptr) and np.array_equal(ci, R.indices) and np.array_equal(v, R.data)
    S = isb.B200CSR.from_csr_slab(R.indptr.astype(np.int64), R.indices.astype(np.int64), R.data, R.shape[0],
                                  ctx=ctxs[8])
    assert S.index_bytes == 8
    x = np.random.default_rng(SEED).standard_normal(R.shape[0])
    assert np.array_equal(S @ x, isb.B200CSR.laplacian(20, 3, ctx=ctxs[4]) @ x)
    d = A.diag().numpy()
    assert np.array_equal(d, np.full(R.shape[0], 6.0))


def test_rejections_leave_data_unchanged(isb, ctxs, mats):
    M = mats["laplace72"]
    A8 = build(isb, ctxs, M, 8)
    L, ctx = isb.lib(), ctxs[8]
    x0 = np.arange(A8.m_local, dtype=np.float64)
    x = isb.DeviceArray.from_numpy(ctx, x0)
    b = isb.DeviceArray.from_numpy(ctx, np.ones(A8.m_local))
    assert L.b200_stationary(ctx._h, A8._h, x._p, b._p, 1, 1.0, 3) == ERR_UNSUPPORTED
    assert b"8-byte row offsets" in L.b200_last_error()
    assert np.array_equal(x.numpy(), x0)
    rp = np.full(A8.m_local + 1, -7, dtype=np.int32)
    ci = np.full(A8.nnz, -7, dtype=np.int32)
    v = np.full(A8.nnz, -7.0)
    assert L.b200_csr_download(ctx._h, A8._h, rp.ctypes.data_as(C.c_void_p), ci.ctypes.data_as(C.c_void_p),
                               v.ctypes.data_as(C.c_void_p)) == ERR_UNSUPPORTED
    assert b"b200_csr_download64" in L.b200_last_error()
    assert np.all(rp == -7) and np.all(ci == -7) and np.all(v == -7.0)


# ------------------------------------------------------------------------------------------ 2^31 nonzeros
N_BIG = 680
NNZ_BIG = 2_198_249_600


def stencil(torch, x, N):
    """y = laplace_matrix(T, N, 3) x on a flat vector; row q = i0 + N i1 + N^2 i2."""
    X = x.view(N, N, N)
    Y = 6 * X
    for d in range(3):
        Y.narrow(d, 1, N - 1).sub_(X.narrow(d, 0, N - 1))
        Y.narrow(d, 0, N - 1).sub_(X.narrow(d, 1, N - 1))
    return Y.view(-1)


def test_laplacian_680_above_2_31_nonzeros(isb):
    torch = pytest.importorskip("torch")
    n = N_BIG ** 3
    free, _ = torch.cuda.mem_get_info(0)
    # operator (8 B offsets + 4 B columns + values) and about six vectors (cg!'s four, torch's x, y and a temporary)
    need = {np.float64: NNZ_BIG * 12 + n * 8 + 7 * n * 8, np.float32: NNZ_BIG * 8 + n * 8 + 7 * n * 4}
    dtype = next((t for t in (np.float64, np.float32) if need[t] < free * 0.95), None)
    if dtype is None:
        pytest.skip(f"laplace_matrix(680, 3) needs {need[np.float32] / 2**30:.1f} GiB of free device memory (Float32), "
                    f"{free / 2**30:.1f} GiB are free")
    ctx = isb.default_context()   # "rowptr64" = 0: the width follows from nnz
    A = isb.B200CSR.laplacian(N_BIG, 3, dtype=dtype, ctx=ctx)
    try:
        assert A.nnz == NNZ_BIG and A.index_bytes == 8 and A.m_local == n
        assert stream_kind(isb, A)[0] == BAND
        tdt = torch.float64 if dtype == np.float64 else torch.float32
        g = torch.Generator(device="cuda:0").manual_seed(SEED)
        x = torch.rand(n, dtype=tdt, device="cuda:0", generator=g)
        y = torch.empty_like(x)
        torch.cuda.synchronize()
        A.mul_(y, x)
        ctx.sync()
        yr = stencil(torch, x, N_BIG)
        err = float((y - yr).abs().max()) / float(yr.abs().max())
        assert err <= (1e-14 if dtype == np.float64 else 1e-5), err
        del yr
        # five cg! iterations against the same recurrence in torch, x0 = 0
        b = x / torch.linalg.vector_norm(x)
        del x, y
        torch.cuda.synchronize()
        xs, h = isb.cg(A, b, log=True, maxiter=5)
        ctx.sync()
        del xs
        r = b.clone()
        u = torch.zeros_like(b)
        rho_prev, ref = 1.0, []
        for k in range(5):
            rho = float(torch.dot(r, r))
            u = r + (rho / rho_prev if k else 0.0) * u
            c = stencil(torch, u, N_BIG)
            alpha = rho / float(torch.dot(u, c))
            r -= alpha * c
            rho_prev = rho
            ref.append(float(torch.linalg.vector_norm(r)))
            del c
        got = np.asarray(h["resnorm"])[:5]
        rel = np.max(np.abs(got - np.asarray(ref)) / np.asarray(ref))
        assert rel <= (1e-10 if dtype == np.float64 else 1e-4), (got, ref)
    finally:
        A.close()
