"""
Sequence chunks of the tensor-core path, host side (no GPU): the byte count evc_plm_tc_bytes reports and the
planner that picks the chunk size from the free device memory (engine.plan_seq_chunk).
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


def _ru(v, m):
    return -(-v // m) * m


def _expected_whole_shard_bytes(N, L, q, ksplit):
    """The buffers of evc_plm_create + set_forward(1), restated from their shapes (one chunk)."""
    lq = L * q
    S = q if q % 2 else q + 1
    Mp, Np, Kw, Kp = _ru(lq, 128), _ru(lq, 192), _ru(lq, 64), _ru(N, 64)
    nt = -(-N // 256)
    return dict(
        codes=N * L, msa4=_ru(L, 4) // 4 * _ru(N, 32) * 4, wts=4 * N,
        X=_ru(N, 384) * Kw * 2,                 # one-hot, forward
        Xt=Mp * Kp * 2,                         # one-hot, backward
        Zt=Mp * _ru(N, 192) * 4,                # logits
        Rt=2 * Np * Kp * 2,                     # residuals hi + lo
        Gd=ksplit * Mp * Np * 4,                # backward planes
        Wt=2 * Mp * Kw * 2,                     # couplings hi + lo
        parts=L * nt * S * 4 + L * nt * 8,      # g_h and fx partials
    )


def test_tc_bytes_whole_shard_matches_buffer_shapes():
    from evcouplings_b200.engine import tc_bytes
    N, L, q = 50000, 200, 21                    # bench config 2: 2 K slices on 132 SMs
    parts = _expected_whole_shard_bytes(N, L, q, ksplit=2)
    assert tc_bytes(N, L, q, -1, 0, SM) == sum(parts.values())
    assert tc_bytes(N, L, q, -1, N, SM) == tc_bytes(N, L, q, -1, 0, SM)          # chunk >= N: one chunk
    assert tc_bytes(N, L, q, -1, 10 ** 9, SM) == tc_bytes(N, L, q, -1, 0, SM)
    # X is allocated with N rounded up to 384 rows (50304 x 4224 bf16 = 425 MB), Zt with N rounded up to 192
    assert round(parts["X"] / 1e6) == 425 and round(parts["Zt"] / 1e6) == 847
    # q = 20 with ignored gaps: the gap code is not a state of X
    p20 = _expected_whole_shard_bytes(3000, 64, 20, ksplit=1)
    got = tc_bytes(3000, 64, 20, 20, 0, SM)
    rest = sum(p20.values()) - p20["Gd"]        # the K-slice count (1-4) depends on the SM count
    assert (got - rest) % p20["Gd"] == 0 and 1 <= (got - rest) // p20["Gd"] <= 4


def test_tc_bytes_monotone_in_chunk():
    from evcouplings_b200.engine import tc_bytes
    N, L, q = 200000, 120, 21
    prev = 0
    for c in range(768, N + 768 * 8, 768 * 7):
        b = tc_bytes(N, L, q, -1, c, SM)
        assert b >= prev, c
        prev = b
    assert tc_bytes(N, L, q, -1, 768, SM) < tc_bytes(N, L, q, -1, 0, SM)
    # the chunk is rounded up to a multiple of 768
    assert tc_bytes(N, L, q, -1, 1, SM) == tc_bytes(N, L, q, -1, 768, SM)
    assert tc_bytes(N, L, q, -1, 769, SM) == tc_bytes(N, L, q, -1, 1536, SM)


def test_tc_bytes_rejects_bad_arguments():
    from evcouplings_b200.engine import tc_bytes
    for args in ((0, 10, 21, -1, 0, SM), (100, 1, 21, -1, 0, SM), (100, 10, 7, -1, 0, SM),
                 (100, 10, 21, 5, 0, SM), (100, 10, 21, -1, -1, SM), (100, 10, 21, -1, 0, 0)):
        with pytest.raises(_lib.EngineError):
            tc_bytes(*args)


def test_planner_whole_shard_when_it_fits():
    from evcouplings_b200.engine import plan_seq_chunk
    assert plan_seq_chunk(50000, 200, 21, -1, 6, SM, 79e9) == 0


def test_planner_chunks_large_alignments():
    from evcouplings_b200.engine import plan_seq_chunk, seq_chunk_reserve_bytes, tc_bytes
    # 2M x 200: about 103 GB unchunked
    c = plan_seq_chunk(2000000, 200, 21, -1, 6, SM, 79e9)
    assert c > 0 and c % 768 == 0 and c < 2000000
    assert tc_bytes(2000000, 200, 21, -1, c, SM) + seq_chunk_reserve_bytes(200, 21, 6) <= 79e9
    # 500k x 500 needs about 70 GB whole: whole shard with 79 GB free, chunks with 60 GB free
    need = tc_bytes(500000, 500, 21, -1, 0, SM) + seq_chunk_reserve_bytes(500, 21, 6)
    assert need < 79e9 and plan_seq_chunk(500000, 500, 21, -1, 6, SM, 79e9) == 0
    c = plan_seq_chunk(500000, 500, 21, -1, 6, SM, 60e9)
    assert c > 0 and c % 768 == 0


def test_planner_picks_largest_chunk_under_budget():
    from evcouplings_b200.engine import plan_seq_chunk, seq_chunk_reserve_bytes, tc_bytes
    N, L, q, m = 300000, 150, 20, 6
    reserve = seq_chunk_reserve_bytes(L, q, m)
    for budget in (3e9, 6e9, 9e9):          # the whole shard needs about 12 GB
        c = plan_seq_chunk(N, L, q, q, m, SM, budget)
        assert c % 768 == 0 and 0 < c < N
        assert tc_bytes(N, L, q, q, c, SM) + reserve <= budget
        assert tc_bytes(N, L, q, q, c + 768, SM) + reserve > budget
    # a budget exactly at the whole-shard need is whole shard; one byte less is chunked
    whole = tc_bytes(N, L, q, q, 0, SM) + reserve
    assert plan_seq_chunk(N, L, q, q, m, SM, whole) == 0
    assert plan_seq_chunk(N, L, q, q, m, SM, whole - 1) > 0


def test_planner_raises_when_L_part_does_not_fit():
    from evcouplings_b200.engine import DeviceMemoryError, plan_seq_chunk, seq_chunk_reserve_bytes, tc_bytes
    with pytest.raises(DeviceMemoryError) as ei:
        plan_seq_chunk(100000, 2000, 21, -1, 6, SM, 79e9)
    need = tc_bytes(100000, 2000, 21, -1, 768, SM) + seq_chunk_reserve_bytes(2000, 21, 6)
    msg = str(ei.value)
    assert str(need) in msg and str(int(79e9)) in msg


def test_fit_workspace_bytes():
    lib = _lib.load()
    n, m = 1000, 6
    vec = _ru(n + 4, 64) * 4
    got = lib.evc_fit_workspace_bytes(n, m)
    assert (5 + 2 * m) * vec <= got < (5 + 2 * m) * vec + 65536
    assert lib.evc_fit_workspace_bytes(n, 8) - got == 4 * vec


def test_seq_chunk_count():
    from evcouplings_b200.engine import seq_chunk_count
    assert seq_chunk_count(6000, 0) == 1
    assert seq_chunk_count(6000, 768) == 8
    assert seq_chunk_count(6000, 2304) == 3
    assert seq_chunk_count(6000, 3072) == 2
    assert seq_chunk_count(6000, 6144) == 1
    assert seq_chunk_count(6000, 1000) == 4          # rounded up to 1536
