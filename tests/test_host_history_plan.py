"""
Correction pairs of the L-BFGS history in pinned host memory, host side (no GPU): the split byte count
evc_fit_workspace_split_bytes reports and the planner (engine.plan_fit_memory) that moves the fewest pairs to the
host only when even one sequence chunk does not fit the device with every pair on it.
"""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from evcouplings_b200 import _lib  # noqa: E402

try:
    _lib.load()
    HAVE_LIB = True
except _lib.EngineUnavailableError:
    HAVE_LIB = False

pytestmark = pytest.mark.skipif(not HAVE_LIB, reason="libevcplm.so not built")

SM = 132
AMPLE_HOST = 10 ** 13


def _ru(v, m):
    return -(-v // m) * m


def _fit_bytes(N, L, q, gap_code, m, chunk, k):
    """Device bytes of a planned fit: the handle at that chunk plus the reserve with k pairs on the host."""
    from evcouplings_b200.engine import fit_workspace_bytes, num_params, seq_chunk_reserve_bytes, tc_bytes
    n = num_params(L, q)
    reserve = seq_chunk_reserve_bytes(L, q, m) - fit_workspace_bytes(n, m, 0)[0] + fit_workspace_bytes(n, m, k)[0]
    return tc_bytes(N, L, q, gap_code, chunk, SM) + reserve


def test_existing_planner_shapes_keep_every_pair_on_the_device():
    from evcouplings_b200.engine import plan_fit_memory, plan_seq_chunk
    shapes = [(50000, 200, 21, -1, 6, 79e9), (2000000, 200, 21, -1, 6, 79e9), (500000, 500, 21, -1, 6, 79e9),
              (500000, 500, 21, -1, 6, 60e9)]
    shapes += [(300000, 150, 20, 20, 6, b) for b in (3e9, 6e9, 9e9)]
    for N, L, q, gap, m, free in shapes:
        assert plan_fit_memory(N, L, q, gap, m, SM, free, AMPLE_HOST) == \
            (plan_seq_chunk(N, L, q, gap, m, SM, free), 0), (N, L, free)
    # with no host memory at all, too: the host is only asked for when the device cannot hold the pairs
    assert plan_fit_memory(50000, 200, 21, -1, 6, SM, 79e9, 0) == (0, 0)


def test_L2000_plans_with_host_pairs():
    from evcouplings_b200.engine import fit_workspace_bytes, num_params, plan_fit_memory
    N, L, q, m, free = 100000, 2000, 21, 6, 79e9
    chunk, k = plan_fit_memory(N, L, q, -1, m, SM, free, AMPLE_HOST)
    assert 0 < k <= m
    assert chunk % 768 == 0 and 0 < chunk < N
    host = fit_workspace_bytes(num_params(L, q), m, k)[1]
    assert _fit_bytes(N, L, q, -1, m, chunk, k) <= free
    assert host <= AMPLE_HOST
    # the largest chunk under the budget with that k
    assert _fit_bytes(N, L, q, -1, m, chunk + 768, k) > free


def test_host_pairs_are_minimal():
    from evcouplings_b200.engine import plan_fit_memory
    for N, free in ((100000, 79e9), (20000, 79e9), (20000, 70e9), (20000, 60e9)):
        _chunk, k = plan_fit_memory(N, 2000, 21, -1, 6, SM, free, AMPLE_HOST)
        assert k >= 1
        assert _fit_bytes(N, 2000, 21, -1, 6, 768, k) <= free
        assert _fit_bytes(N, 2000, 21, -1, 6, 768, k - 1) > free, (N, free, k)
    # less device memory needs more host pairs
    assert plan_fit_memory(20000, 2000, 21, -1, 6, SM, 60e9, AMPLE_HOST)[1] > \
        plan_fit_memory(20000, 2000, 21, -1, 6, SM, 79e9, AMPLE_HOST)[1]


def test_too_little_host_memory_raises_with_both_byte_counts():
    from evcouplings_b200.engine import (HOST_FIT_BYTES_PER_PARAM, DeviceMemoryError, HostMemoryError,
                                         fit_workspace_bytes, num_params, plan_fit_memory)
    N, L, q, m, free = 100000, 2000, 21, 6, 79e9
    _chunk, k = plan_fit_memory(N, L, q, -1, m, SM, free, AMPLE_HOST)
    host_need = fit_workspace_bytes(num_params(L, q), m, k)[1]
    with pytest.raises(HostMemoryError) as ei:
        plan_fit_memory(N, L, q, -1, m, SM, free, host_need - 1)
    msg = str(ei.value)
    dev_need = _fit_bytes(N, L, q, -1, m, 768, k)
    total = host_need + HOST_FIT_BYTES_PER_PARAM * num_params(L, q)
    for v in (dev_need, int(free), host_need, total, host_need - 1):
        assert str(v) in msg, (v, msg)
    assert isinstance(ei.value, DeviceMemoryError)          # run_plmc turns both into ResourceError
    # the device too small even with every pair on the host
    with pytest.raises(DeviceMemoryError) as ei:
        plan_fit_memory(N, L, q, -1, m, SM, 40e9, AMPLE_HOST)
    msg = str(ei.value)
    assert str(_fit_bytes(N, L, q, -1, m, 768, m)) in msg and str(int(40e9)) in msg
    assert str(fit_workspace_bytes(num_params(L, q), m, m)[1]) in msg and str(AMPLE_HOST) in msg


def test_host_budget_counts_the_fits_own_host_arrays():
    """The pinned pairs alone fitting the budget is not enough: run_plmc also holds the float64 pair counts and
    frequencies, the start point and the result (24 bytes per parameter) while the pairs are pinned."""
    from evcouplings_b200.engine import (HOST_FIT_BYTES_PER_PARAM, HostMemoryError, fit_workspace_bytes, num_params,
                                         plan_fit_memory)
    N, L, q, m, free = 768, 2700, 21, 6, 79e9           # near the ceiling: every pair on the host
    n = num_params(L, q)
    _chunk, k = plan_fit_memory(N, L, q, -1, m, SM, free, AMPLE_HOST)
    assert k == m
    pairs = fit_workspace_bytes(n, m, k)[1]
    own = HOST_FIT_BYTES_PER_PARAM * n
    assert own > 30e9 and pairs > 70e9
    for budget in (pairs, pairs + own - 1):             # covers the pairs, not the pairs plus counts and x0
        with pytest.raises(HostMemoryError) as ei:
            plan_fit_memory(N, L, q, -1, m, SM, free, budget)
        assert str(pairs + own) in str(ei.value) and str(budget) in str(ei.value)
    assert plan_fit_memory(N, L, q, -1, m, SM, free, pairs + own)[1] == m
    # forced pairs are checked against the same budget; k = 0 needs no host memory
    with pytest.raises(HostMemoryError):
        plan_fit_memory(6000, 60, 21, -1, 6, SM, free, fit_workspace_bytes(num_params(60, 21), 6, 2)[1],
                        host_pairs=2)
    assert plan_fit_memory(6000, 60, 21, -1, 6, SM, free, 0, host_pairs=0) == (0, 0)


def test_forced_host_pairs():
    from evcouplings_b200.engine import plan_fit_memory
    assert plan_fit_memory(6000, 60, 21, -1, 6, SM, 79e9, AMPLE_HOST, host_pairs=6) == (0, 6)
    assert plan_fit_memory(6000, 60, 21, -1, 6, SM, 79e9, AMPLE_HOST, host_pairs=0) == (0, 0)
    with pytest.raises(ValueError):
        plan_fit_memory(6000, 60, 21, -1, 6, SM, 79e9, AMPLE_HOST, host_pairs=7)


def test_split_bytes_match_the_device_workspace():
    from evcouplings_b200.engine import fit_workspace_bytes
    lib = _lib.load()
    for n, m in ((1000, 6), (881601000, 6), (54321, 1), (54321, 32)):
        vec = _ru(n + 4, 64) * 4
        assert fit_workspace_bytes(n, m, 0) == (lib.evc_fit_workspace_bytes(n, m), 0)
        for k in range(1, m + 1):
            dev, host = fit_workspace_bytes(n, m, k)
            assert dev == lib.evc_fit_workspace_bytes(n, m) - 2 * k * vec
            assert host == 2 * k * vec
    for args in ((0, 6, 0), (1000, 0, 0), (1000, 6, 7), (1000, 6, -1), (1000, 33, 0)):
        with pytest.raises(_lib.EngineError):
            fit_workspace_bytes(*args)


def test_host_budget_shares_MemAvailable(tmp_path):
    from evcouplings_b200.engine import HOST_HISTORY_MARGIN_BYTES, host_history_budget_bytes
    mi = tmp_path / "meminfo"
    mi.write_text("MemTotal:       1000000000 kB\nMemFree:        10 kB\nMemAvailable:   100000000 kB\n")
    avail = 100000000 * 1024
    assert host_history_budget_bytes(1, str(mi)) == avail - HOST_HISTORY_MARGIN_BYTES
    assert host_history_budget_bytes(4, str(mi)) == (avail - HOST_HISTORY_MARGIN_BYTES) // 4
    mi.write_text("MemAvailable:   1024 kB\n")
    assert host_history_budget_bytes(1, str(mi)) == 0
