"""The set-criterion matcher's solver (trackformer_b200/csrc/lsa_core.h, what csrc/lsa.cu's kernels run) against
scipy.optimize.linear_sum_assignment, on the CPU: the g++ host build of the same routine
(tests/host_build/lsa_host.cpp), one problem at a time in lsa_kernel's layout -- cost[query][target], every target
assigned a distinct query."""
import ctypes

import numpy as np
import pytest
from scipy.optimize import linear_sum_assignment

import host_twin


@pytest.fixture(scope="module")
def host_lsa(tmp_path_factory):
    lib = host_twin.build("lsa_host", tmp_path_factory.mktemp("lsa"))
    vp, i32 = ctypes.c_void_p, ctypes.c_int
    lib.tfb200_lsa_host.argtypes = [vp, i32, i32, vp]
    lib.tfb200_lsa_host.restype = i32

    def solve(cost):
        """(status, queries sorted ascending, their targets) -- linear_sum_assignment's (row_ind, col_ind) order."""
        cost = np.ascontiguousarray(cost, dtype=np.float32)
        q, t = cost.shape
        query = np.full(t, -1, dtype=np.int32)
        status = lib.tfb200_lsa_host(cost.ctypes.data, q, t, query.ctypes.data)
        order = np.argsort(query, kind="stable")
        return status, query[order], order
    return solve


# the shapes of test_lsa_gpu.py (one problem per (Q, targets)), and one of the wide solver's
@pytest.mark.parametrize("Q,T", [(300, 20), (300, 7), (50, 50), (50, 1), (50, 13), (900, 128), (900, 200), (17, 3),
                                 (17, 17), (17, 5), (7000, 150)])
def test_continuous_costs_match_scipy(host_lsa, Q, T):
    cost = (np.random.default_rng(Q * 1000 + T).standard_normal((Q, T)) * 3).astype(np.float32)
    status, rows, cols = host_lsa(cost)
    assert status == 0
    ref_rows, ref_cols = linear_sum_assignment(cost.astype(np.float64))
    assert np.array_equal(rows, ref_rows)
    assert np.array_equal(cols, ref_cols)


@pytest.mark.parametrize("Q,T,levels", [(30, 30, 3), (300, 20, 4), (60, 45, 2)])
def test_integer_costs_with_ties_reach_scipys_optimum(host_lsa, Q, T, levels):
    """Many equally optimal assignments: the total is scipy's; which of them is chosen may differ (scipy's column
    scan is not in index order)."""
    cost = np.random.default_rng(Q + T + levels).integers(0, levels, (Q, T)).astype(np.float32)
    status, rows, cols = host_lsa(cost)
    assert status == 0
    assert len(set(rows.tolist())) == T and sorted(cols.tolist()) == list(range(T))
    ref_rows, ref_cols = linear_sum_assignment(cost.astype(np.float64))
    assert cost[rows, cols].sum(dtype=np.float64) == cost[ref_rows, ref_cols].sum(dtype=np.float64)


def test_infeasible_problem_is_reported(host_lsa):
    cost = np.random.default_rng(5).standard_normal((40, 6)).astype(np.float32)
    cost[:, 4] = np.inf                       # target 4 reaches no query at a finite cost
    status, _, _ = host_lsa(cost)
    assert status == 2
