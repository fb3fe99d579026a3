"""How long a chain pass 1 of the device AMG aggregation (csrc/amg_setup.cu, k_pass1) can form, checked without a GPU.

A row of k_pass1 polls its smaller conflicting rows at most kPass1Polls = 4096 times per launch; a row still undecided
then makes the setup launch pass 1 again.  pass_one_depth below counts the rounds of amg_pass1_rounds (the serial
rounds of amg_pass1_decide to their fixpoint, tests/hostsim_amg_rows) in one sweep over the rows, checked against the
serial rounds, so that the depth of a 2^18-row chain can be counted in a test: the 1-D Laplacian of 2^18 rows needs far
more rounds than one launch's polls cover, which is why tests/test_gpu_amg_pass1_relaunch.py sees pass 1 relaunched.
"""
import numpy as np
import pytest
import scipy.sparse as sp

from oracle import oracle as O
from test_amg_device_rows import aggregate_both, random_pattern
from test_amg_engine import anisotropic, np_strength


def laplace1d(n):
    return sp.diags([-np.ones(n - 1), 2 * np.ones(n), -np.ones(n - 1)], [-1, 0, 1], format="csr")


def pass_one_depth(A, theta):
    """The rounds amg_pass1_rounds takes, from one sweep in row order instead of a sweep per round: a row decided by
    amg_pass1_initial is decided in round 0; any other row i, whose smaller conflicting rows (r < i with r in S(i), i in
    S(r), or S(r) meeting S(i)) are all decided by then, becomes a non-root in the round after its earliest-decided
    smaller conflicting root, or a root in the round after the last of them is decided."""
    S = np_strength(sp.csr_matrix(A, dtype=np.float64), theta)
    P = (S != 0).astype(np.int64)
    Cf = sp.tril(P + P.T + P @ P.T, k=-1, format="csr")
    srp, sci = S.indptr.tolist(), S.indices.tolist()
    crp, cci = Cf.indptr.tolist(), Cf.indices.tolist()
    n = A.shape[0]
    depth, root = [0] * n, [False] * n
    for i in range(n):
        if srp[i] == srp[i + 1] or any(j < i and srp[j] == srp[j + 1] for j in sci[srp[i]:srp[i + 1]]):
            continue                                                     # amg_pass1_initial: a non-root
        conf = cci[crp[i]:crp[i + 1]]
        roots = [depth[r] for r in conf if root[r]]
        if roots:
            depth[i] = 1 + min(roots)
        else:
            root[i] = True
            depth[i] = 1 + max((depth[r] for r in conf), default=0)
    return max(1, max(depth, default=0))


@pytest.mark.parametrize("name", ["laplace1d_300", "laplace1d_3001", "laplace2d_30", "laplace3d_12", "anisotropic_theta",
                                  "random_300"])
def test_pass_one_depth_counts_the_serial_rounds(name):
    A, theta = {"laplace1d_300": (lambda: laplace1d(300), 0.0), "laplace1d_3001": (lambda: laplace1d(3001), 0.0),
                "laplace2d_30": (lambda: O.laplace_matrix_scipy(np.float64, 30, 2), 0.0),
                "laplace3d_12": (lambda: O.laplace_matrix_scipy(np.float64, 12, 3), 0.0),
                "anisotropic_theta": (anisotropic, 0.25),
                "random_300": (lambda: random_pattern(300, 0.03, 4), 0.3)}[name]
    A = A()
    rounds = aggregate_both(A, theta)[4]
    assert pass_one_depth(A, theta) == rounds, rounds


def test_a_1d_laplacian_chains_pass_one_beyond_one_launchs_poll_budget():
    # On the 1-D Laplacian row 3k becomes a root only after rows 3k-2 and 3k-1 are non-roots, and they only after row
    # 3k-3 is a root: roots 0, 3, 6, ... are decided in rounds 1, 3, 5, ..., so pass 1 needs about 2n/3 rounds.  A row of
    # k_pass1 polls at most kPass1Polls = 4096 times per launch, and a poll advances the chain by about one round unless
    # polls of different rows happen to overlap it, so at n = 2^18 the device setup has to launch pass 1 again.
    assert aggregate_both(laplace1d(3001), 0.0)[4] == 2001
    depth = pass_one_depth(laplace1d(1 << 18), 0.0)
    assert depth == (2 * (1 << 18) + 2) // 3, depth
    assert depth > 32 * 4096
