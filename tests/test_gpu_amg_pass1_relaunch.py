"""Pass 1 of the device AMG aggregation (csrc/amg_setup.cu) relaunched: the 1-D Laplacian of 2^18 rows makes pass 1 a
chain of about 2n/3 rounds (tests/test_amg_pass1_chain.py), longer than one k_pass1 launch decides, so its setup takes
the relaunch path: rows decided in an earlier launch return at once, the others carry on from the states left behind.
The hierarchy must still be the serial setup's byte for byte (csrc/amg_core.h, tests/hostsim_amg), in Float64 and
Float32, at theta 0 and 0.25; the pass-1 launch counts of the hierarchy show that the relaunch happened.
"""
import numpy as np
import pytest
import scipy.sparse as sp

from test_amg_engine import SimAMG
from test_gpu_amg_device_setup import _same_csr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def isb():
    import iterativesolvers_jl_b200 as m
    return m


def laplace1d(n):
    return sp.diags([-np.ones(n - 1), 2 * np.ones(n), -np.ones(n - 1)], [-1, 0, 1], format="csr")


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("theta", [0.0, 0.25])
def test_a_relaunched_pass_one_gives_the_serial_hierarchy(isb, theta, dtype):
    A = laplace1d(1 << 18).astype(dtype)
    A.sort_indices()
    sim = SimAMG(A.astype(np.float64), theta=theta)
    assert sim.status == 0, (sim.status, sim.bad)
    ref = sim.levels()
    ctx = isb.Context(0)
    Ad = isb.B200CSR.from_scipy(A, ctx=ctx)
    before = ctx.launch_count()
    P = isb.SmoothedAggregationPrec(Ad, theta=theta)
    launches = ctx.launch_count() - before
    rows = P.level_rows
    assert len(rows) == 10 and rows[-1] <= 4096, rows     # max_levels is what ends the coarsening
    p1 = P.pass1_launches
    print(f"theta {theta} {np.dtype(dtype).name}: pass-1 launches per level {p1}, setup launches {launches}, rows {rows}")
    assert p1[-1] == 0 and all(k >= 1 for k in p1[:-1]), p1
    assert p1[0] > 1, p1                                  # one launch per level would give [1, 1, ..., 1, 0]
    assert launches > sum(p1), (launches, p1)             # the pass-1 launches are among the context's launches
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
    assert got[0]["agg"][:7].tolist() == [0, 0, 1, 1, 1, 2, 2]
