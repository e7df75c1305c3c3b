"""Replica exchange, CPU side: the float64 restatement (oracle/tempering.py) against the plain sampler's, the exact
rung distributions by enumeration (plain and conditional with masks), the Curie-Weiss Potts model's modes, planted
mistakes and the argument checks of the Python and command-line interfaces."""
import ctypes
import io

import numpy as np
import pytest

from evcouplings_b200 import model_ops, sample_cli
from oracle import conditional_sampler as cs, potts_sampler as ps, tempering as tp
from test_potts_sampler_oracle import distribution_bounds, small_model

# The Curie-Weiss Potts model of the mode tests (CPU and device), fixed here: q = 3, L = 16, K = 1/2 (dyadic, so the
# device's fields are exact).  At beta = 1 (beta K L = 8, far in the ordered phase) a plain chain started in mode 0
# stays there; the geometric ladder from 1/8 (disordered) to 1 crosses the transition near beta K L = 4 ln 2.
CW = dict(L=16, q=3, K=0.5)
CW_LADDER = dict(beta_min=0.125, beta_max=1.0, R=8)
CW_PLAIN_SWEEPS = 1000
CW_CPU = dict(ladders=400, sweeps=600)


def check_against(idx, p):
    """TV and chi^2 of the state indices ``idx`` against the exact distribution p, within distribution_bounds."""
    n = len(idx)
    freq = np.bincount(idx, minlength=len(p)) / n
    tv = 0.5 * np.abs(freq - p).sum()
    ok = p > 0
    x2 = n * (((freq - p) ** 2)[ok] / p[ok]).sum()
    tv_max, x2_max = distribution_bounds(p[ok], n)
    assert tv <= tv_max and x2 <= x2_max, (tv, tv_max, x2, x2_max)
    assert freq[~ok].sum() == 0
    return tv, x2


def test_equal_betas_are_the_plain_sampler_draw_for_draw():
    h, J = small_model(5, 4, 3)
    R, G, beta = 4, 50, 0.75
    plain = ps.Sampler(h, J, seed=9, n_chains=G * R, chain_offset=8)
    base = ps.Sampler(h, J, seed=9, n_chains=G * R, chain_offset=8)
    T = tp.Tempered(base, [beta] * R, 3, seed=9, ladder_offset=2)
    a = plain.run(40, beta)
    b = T.run(17) + T.run(23)                     # split between swap rounds and across the refresh at t = 32
    assert a == b and np.array_equal(plain.codes(), base.codes())
    assert T.attempted.sum() > 0 and np.array_equal(T.accepted, T.attempted)      # Delta = 0: every swap accepted


def test_swap_counter_is_not_a_chain_stream():
    # the swap key is the chain key of 2^63 + g, an index no chain reaches
    k = tp.swap_key(5, np.arange(4))
    assert not np.isin(k, ps.chain_key(5, np.arange(0, 4096))).any()
    u = tp.swap_uniform(k, 3, 1, 8)
    assert np.all((u > 0) & (u < 1))


def test_swap_rounds_and_parity():
    assert tp.swap_rounds(0, 7, 3) == [(3, 0), (6, 1)]
    assert tp.swap_rounds(5, 2, 3) == [(6, 1)]
    h, J = small_model(3, 2, 1)
    T = tp.Tempered(ps.Sampler(h, J, seed=1, n_chains=5 * 4), [0.1, 0.2, 0.4, 0.8, 1.0], 2, seed=1)
    T.run(8)
    assert [n for n, _ in T.decisions] == [0, 1, 2, 3]
    for n, acc in T.decisions:                    # only pairs of the round's parity are tried
        assert not acc[:, [k for k in range(4) if k % 2 != n % 2]].any()
    assert np.array_equal(T.attempted, [2 * 4, 2 * 4, 2 * 4, 2 * 4])


@pytest.mark.parametrize("L,q", [(4, 3), (3, 5)])
def test_rungs_match_enumeration(L, q):
    h, J = small_model(L, q, 10 * L + q)
    ladder = np.array([0.25, 0.5, 0.75, 1.0], dtype=np.float32)
    R, G = len(ladder), 12000
    T = tp.Tempered(ps.Sampler(h, J, seed=4, n_chains=G * R), ladder, 1, seed=4)
    T.run(40)
    for k in range(R):
        check_against(ps.state_index(T.rung_codes(k), q), ps.exact_distribution(h, J, float(ladder[k]), L, q))
    assert np.all(T.accepted > 0) and np.all(T.accepted < T.attempted)


def test_conditional_rungs_match_enumeration_with_masks():
    L, q = 6, 3
    h, J = small_model(L, q, 63)
    free = np.array([1, 3, 4])
    allowed = np.array([0b111, 0b101, 0b011])
    ladder = np.array([0.5, 1.0, 1.5], dtype=np.float32)
    R, G = len(ladder), 12000
    ctx = np.random.default_rng(2).integers(0, q, L)
    init = np.repeat(ctx[None], G * R, axis=0)
    base = cs.ConditionalSampler.from_model(h, J, 6, G * R, free, allowed, init)
    T = tp.Tempered(base, ladder, 2, seed=6)
    T.run(40)
    for k in range(R):
        codes = T.rung_codes(k).astype(np.int64)
        assert np.array_equal(codes[:, cs.clamped_sites(L, free)], init[:G, cs.clamped_sites(L, free)])
        p = cs.exact_conditional(h, J, float(ladder[k]), free, ctx, allowed)
        check_against(ps.state_index(codes[:, free], q), p)


def curie_weiss_ladder():
    return model_ops.geometric_ladder(CW_LADDER["beta_min"], CW_LADDER["beta_max"], CW_LADDER["R"])


def test_curie_weiss_plain_chains_stay_in_their_mode():
    L, q, K = CW["L"], CW["q"], CW["K"]
    h, J = tp.curie_weiss_model(L, q, K)
    n = 2000
    s = ps.Sampler(h, J, seed=1, n_chains=n, init=np.zeros((n, L), dtype=np.int64))
    s.run(CW_PLAIN_SWEEPS, 1.0)
    assert (tp.mode_of(s.codes(), q) == 0).mean() >= 0.99
    assert np.allclose(tp.curie_weiss_mode_probabilities(L, q, K, 1.0), 1.0 / q, atol=1e-12)


def test_curie_weiss_ladder_reaches_every_mode():
    L, q, K = CW["L"], CW["q"], CW["K"]
    h, J = tp.curie_weiss_model(L, q, K)
    ladder = curie_weiss_ladder()
    R, G = len(ladder), CW_CPU["ladders"]
    base = ps.Sampler(h, J, seed=2, n_chains=G * R, init=np.zeros((G * R, L), dtype=np.int64))
    T = tp.Tempered(base, ladder, 1, seed=2)
    T.run(CW_CPU["sweeps"])
    p = tp.curie_weiss_mode_probabilities(L, q, K, float(ladder[-1]))
    freq = np.bincount(tp.mode_of(T.rung_codes(R - 1), q), minlength=q) / G
    assert np.abs(freq - p).max() <= tp.mode_bound(p, G), (freq, p)
    assert T.trips.sum() > 0


def test_exact_curie_weiss_distribution_by_enumeration():
    L, q, K, beta = 5, 3, 0.5, 0.8
    h, J = tp.curie_weiss_model(L, q, K)
    p = ps.exact_distribution(h, J, beta, L, q)
    states = np.array(np.unravel_index(np.arange(q ** L), (q,) * L)).T
    mode = tp.mode_of(states, q)
    assert np.allclose([p[mode == a].sum() for a in range(q)], tp.curie_weiss_mode_probabilities(L, q, K, beta),
                       rtol=1e-12)


@pytest.mark.parametrize("mutation", ["energy_site_order", "delta_sign", "swap_states", "round_parity"])
def test_planted_mistakes_change_the_trajectory(mutation):
    h, J = small_model(6, 4, 5)
    ladder = np.array([0.2, 0.45, 0.7, 1.0], dtype=np.float32)
    R, G = len(ladder), 64
    runs = []
    for m in (None, mutation):
        base = ps.Sampler(h, J, seed=3, n_chains=G * R)
        T = tp.Tempered(base, ladder, 1, seed=3, mutation=m)
        T.run(6)
        runs.append((T, base.codes(), np.concatenate([a for _, a in T.decisions])))
    (good, gc, gd), (bad, bc, bd) = runs
    if mutation == "energy_site_order":
        # the device's energies are compared within swap_margin: fp32 sums in site order are far outside
        margin = tp.swap_margin(6, ps.z_bound(h, J, 6, 4), 1.0)
        assert np.abs(good.energies() - bad.energies()).max() > 1e3 * margin
    else:
        assert not (np.array_equal(gc, bc) and np.array_equal(gd, bd) and np.array_equal(good.rung, bad.rung))


def test_ladder_checks():
    assert np.array_equal(model_ops.check_ladder([0, 0.5, 1.0]), np.float32([0, 0.5, 1.0]))
    for bad in ([1.0], [0.5, 0.5], [1.0, 0.5], [-0.1, 1.0], [0.0, np.inf], [[0.1, 0.2]], [1.0, 1.0 + 1e-9]):
        with pytest.raises(ValueError):
            model_ops.check_ladder(bad)
    with pytest.raises(ValueError):
        model_ops.check_ladder([0.1, 0.2], swap_interval=0)
    g = model_ops.geometric_ladder(0.5, 2.0, 3)
    assert g.dtype == np.float32 and np.array_equal(g, np.float32([0.5, 1.0, 2.0]))
    for lo, hi, R in ((0.0, 1.0, 4), (1.0, 1.0, 4), (1.0, 0.5, 4), (0.5, 1.0, 1), (1.0, 1.0 + 1e-7, 8)):
        with pytest.raises(ValueError):
            model_ops.geometric_ladder(lo, hi, R)
    with pytest.raises(ValueError):
        model_ops.sample_codes(None, 4, 1, return_statistics=True)


def test_cli_tempering_arguments():
    base = ["m.model", "-n", "3", "--sweeps", "5", "-o", "o.a2m"]
    o = sample_cli.parse_args(base + ["--tempering", "3", "--beta-min", "0.5", "--beta", "2"])
    assert np.array_equal(o["ladder"], np.float32([0.5, 1.0, 2.0])) and o["swap_interval"] == 1
    o = sample_cli.parse_args(base + ["--ladder", "0,0.5,1", "--swap-interval", "4"])
    assert np.array_equal(o["ladder"], np.float32([0, 0.5, 1])) and o["swap_interval"] == 4
    assert "ladder" not in sample_cli.parse_args(base)
    text = sample_cli.format_swap_statistics(np.float32([0.5, 1.0]), model_ops._swap_summary([10], [4], [1, 2]))
    assert "accepted 4 of 10 (0.4000)" in text and "round trips: 3 in all, 1.5000 per ladder" in text


@pytest.mark.parametrize("extra", [["--tempering", "4"], ["--beta-min", "0.5"], ["--tempering", "1", "--beta-min", "0.5"],
                                   ["--tempering", "4", "--beta-min", "0"], ["--tempering", "4", "--beta-min", "2"],
                                   ["--ladder", "1,0.5"], ["--ladder", "0.5"], ["--ladder", "x,1"],
                                   ["--ladder", "0.5,1", "--tempering", "2", "--beta-min", "0.5"],
                                   ["--swap-interval", "2"], ["--ladder", "0.5,1", "--swap-interval", "0"]])
def test_cli_refuses_bad_ladders_before_device_work(tmp_path, extra):
    err = io.StringIO()
    rc = sample_cli.main([str(tmp_path / "none.model"), "-n", "2", "--sweeps", "1", "-o", str(tmp_path / "o.a2m")] +
                         extra, stderr=err)
    assert rc == 2 and err.getvalue().startswith("evcplm-sample: ")
    assert not (tmp_path / "o.a2m").exists()


def test_library_checks_ladder_arguments_without_a_device():
    from evcouplings_b200 import _lib
    lib = _lib.load()
    b = np.float32([0.5, 1.0])
    vp = ctypes.c_void_p
    assert lib.evc_sampler_set_ladder(None, b.ctypes.data_as(vp), 2, 1) == 1
    assert b"null" in lib.evc_last_error()
    assert lib.evc_sampler_temper(None, 1, None, None, None) == 1
    assert lib.evc_sampler_ladder_state(None, None, None, None, None) == 1


def test_ladder_chains_with_different_contexts_are_refused():
    free = np.array([1, 2, 4])
    ctx = np.zeros((6, 5), dtype=np.uint8)
    ctx[:, free] = np.arange(18).reshape(6, 3) % 3                 # free sites may differ
    model_ops.check_ladder_contexts(ctx, free, 3)
    ctx[4, 3] = 1                                                  # a clamped site of chain 4, ladder 1
    with pytest.raises(ValueError, match="ladder 1 .chains 3..5. have different contexts"):
        model_ops.check_ladder_contexts(ctx, free, 3)
    with pytest.raises(ValueError, match="ladder 2"):
        model_ops.check_ladder_contexts(ctx, free, 2)
