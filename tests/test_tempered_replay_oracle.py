"""The fp32 replay of replica exchange (oracle/tempered_replay.TemperedReplay), CPU side: a generated trajectory
replays clean, the replay's energies are the lane-and-butterfly sums, and each planted mistake of a tempered kernel
is caught."""
import numpy as np
import pytest

from oracle import potts_sampler as ps, tempered_replay as sr


def model(L=20, q=5, seed=3):
    """Non-dyadic fields and couplings strong enough that swaps are neither always nor never accepted."""
    rng = np.random.default_rng(seed)
    h = (rng.normal(0, 0.7, (L, q)) * 1.013).astype(np.float32)
    J = (rng.normal(0, 0.25, (L * (L - 1) // 2, q, q)) * 1.007).astype(np.float32)
    return h, J


LADDER = np.float32([0.3, 0.55, 0.8, 1.0])


def generate(mutation=None, n=4 * 32, interval=2):
    h, J = model()
    g = sr.TemperedReplay(h, J, seed=7, n_chains=n, chain_offset=8, ladder=LADDER, swap_interval=interval,
                          mutation=mutation)
    start = g.s.copy()
    for k in (9, 1, 24, 6):                        # 40 sweeps across the refresh at t = 32, calls split mid-interval
        g.temper(k)
    r = sr.replay_tempered_calls(sr.TemperedReplay(h, J, seed=7, n_chains=n, chain_offset=8, ladder=LADDER,
                                          swap_interval=interval, init=start), g.calls)
    return g, r


def test_generated_trajectory_replays_clean():
    g, r = generate()
    assert r.clean(), (r.violations[:2], r.swap_violations[:2], r.energy_mismatch[:1])
    assert r.decisions == 20 * 32 * 2 - 10 * 32 and r.swap_ties == 0       # rounds alternate 2 and 1 pairs
    assert np.array_equal(r.accepted, g.accepted) and np.array_equal(r.trips, g.trips)
    assert 0 < r.accepted.sum() < r.attempted.sum()
    assert r.checked_share() > 0.99


def test_energy_is_the_lane_sum_of_the_float64_energy():
    h, J = model()
    r = sr.TemperedReplay(h, J, seed=7, n_chains=8, ladder=LADDER)
    r.temper(3)
    exact = ps.energies(h, J, r.s)
    assert np.abs(r.energies() - exact).max() <= 1e-4 * np.abs(exact).max()
    d = np.random.default_rng(0).normal(size=(5, 77))
    assert np.allclose(sr.lane_sum(d), d.sum(axis=1), rtol=1e-13)


@pytest.mark.parametrize("mutation", sr.TEMPER_MUTATIONS)
def test_planted_mistake_is_caught(mutation):
    g, r = generate(mutation)
    print("%s: %d energy mismatches, %d swap violations (first %s), %d draw violations" %
          (mutation, len(r.energy_mismatch), r.n_swap_violations, r.swap_violations[:1], r.n_violations))
    assert not r.clean()
    if mutation == "energy_site_order":
        assert r.energy_mismatch
    else:
        assert r.n_swap_violations > 0


def test_whole_ladders_only():
    h, J = model()
    with pytest.raises(ValueError):
        sr.TemperedReplay(h, J, n_chains=10, ladder=LADDER)
    with pytest.raises(ValueError):
        sr.TemperedReplay(h, J, n_chains=8, chain_offset=2, ladder=LADDER)
