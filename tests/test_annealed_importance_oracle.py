"""Annealed importance sampling on the CPU: the exact log partition functions (enumeration, disjoint pairs, transfer
matrices) against each other, the float64 restatement of evc_sampler_anneal (oracle/ais.py) against them, and the
constants the device tests (tests/test_gpu_annealed_importance.py) gate on: the standard-error multiple, the chain
counts and schedules, and the share of chain-sweeps each draw-for-draw check compares.  Also the evcplm-logz command
line's and the library's argument refusals, and log_probabilities refusing symbols outside the model's states.  No
device is touched."""
import ctypes
import io
import math

import numpy as np
import pytest

from evcouplings_b200 import logz_cli, model_ops, synthetic
from oracle import ais, potts_sampler as ps
from test_potts_sampler_oracle import small_model
from test_sampler_geometry_oracle import CTA2, CTA13, chains_per_cta, clean_after, cta2_model, cta13_model, dense_J

# An estimate of log Z passes when it lies within N_SIGMA of its own delta-method standard errors of the exact value.
# Over 18 restated runs on the enumeration models (2048 and 4096 chains, K = 16 and 64, three seeds, both directions
# and the reverse from exact samples) the largest deviation was 2.9 standard errors; 5 leaves a tail of about 6e-7
# per check for a normal estimate.
N_SIGMA = 5.0
# the enumeration models of the sampler tests, restated here with ENUM_CHAINS chains; the device runs DEVICE_CHAINS
ENUM_MODELS = [(4, 3), (3, 5)]
ENUM_CHAINS, ENUM_K, ENUM_SEED = 4096, 64, 21
ENUM_DEVICE_CHAINS = 131072

# Draw for draw: n chains, one sweep at beta = 0 (t = 0) and K annealed sweeps (t = 1..K, across the refresh at
# t = 32), one call per sweep.  The least share of chain-sweeps compared (clean so far) that the restatement alone
# reaches for each case (test_draw_comparison_power prints it).
DRAW_CASES = [(12, 2), (12, 21), (12, 32), (64, 2), (64, 21), (64, 32)]
DRAW = dict(n=2048, K=32, seed=77)
# The restatement compares 0.999, 0.949, 0.889, 0.992, 0.669 and 0.478 of them, in DRAW_CASES order.
DRAW_POWER = {(12, 2): 0.95, (12, 21): 0.90, (12, 32): 0.85, (64, 2): 0.95, (64, 21): 0.60, (64, 32): 0.43}

# Geometry: the sampler's CTA13 and CTA2 cases (test_sampler_geometry_oracle), one sweep at beta = 0 and then the first
# GEOMETRY_SWEEPS - 1 sweeps of the linear schedule of GEOMETRY_K temperatures, across the refresh at t = 32.
GEOMETRY_K, GEOMETRY_SWEEPS = 64, 40
# The restatement compares 0.397 (CTA13, 43 chains clean past t = 32) and 0.393 (CTA2, 16 chains).
GEOMETRY_POWER = dict(CTA13=0.35, CTA2=0.35)

# Exact answers at production size: log_partition with these arguments on a planted model of disjoint pairs and on
# nearest-neighbour chains, whose log Z is exact (PRODUCTION_MODELS).
PRODUCTION = dict(n_chains=4096, temperatures=256, burn_in=256, seed=5)


def production_model(name):
    if name == "planted_L200_q21":
        return synthetic.planted_potts_model(200, 21, 20, 5)
    if name == "chain_L200_q21":
        return synthetic.chain_potts_model(200, 21, 6)
    if name == "chain_L200_q32":
        return synthetic.chain_potts_model(200, 32, 7, alphabet=(synthetic.ALPHABET + "BJOUXZ12345")[:32])
    raise KeyError(name)


PRODUCTION_MODELS = ["planted_L200_q21", "chain_L200_q21", "chain_L200_q32"]


def exact_log_z(model):
    if "contacts" in model:
        return ais.log_z_disjoint_pairs(model["h"], model["J"], model["contacts"])
    return ais.log_z_chain(model["h"], model["J"])


def within(estimate, exact, stderr):
    return abs(estimate - exact) <= N_SIGMA * stderr


# ---- shared by the draw-for-draw checks here and on the device -----------------------------------------------------

def draw_model(L, q, seed):
    """Fields N(0, 0.5) and couplings N(0, 0.05) as multiples of 2^-10: Z is exact on the device."""
    rng = np.random.default_rng(seed)
    h = np.round(rng.normal(0, 0.5, (L, q)) * 1024) / 1024
    J = np.round(rng.normal(0, 0.05, (L * (L - 1) // 2, q, q)) * 1024) / 1024
    return h.astype(np.float32), J.astype(np.float32)


def draw_margin(h, J):
    """The annealed near-tie margin of a dyadic model for any beta in [0, 1] (z_error = 0)."""
    L, q = h.shape
    assert ps.z_error_bound(h, J, L, q, bits=10) == 0.0
    return ais.annealed_near_tie_margin(q, 0.0, 1.0, ps.z_bound(h, J, L, q))


def sweep_schedules(K, sweeps=None):
    """One schedule per call: [0, 0] (the sweep at beta = 0), then [beta_{k-1}, beta_k] of linear_schedule(K)."""
    b = ais.linear_schedule(K)
    return [np.zeros(2, dtype=np.float32)] + [b[k - 1:k + 1] for k in range(1, (sweeps or K + 1))]


def geometry_restatement(name):
    case = dict(CTA13=CTA13, CTA2=CTA2)[name]
    h, pairs, blocks = dict(CTA13=cta13_model, CTA2=cta2_model)[name]()
    L, q = h.shape
    B = ps.sparse_site_z_bounds(h, L, q, pairs, blocks)
    assert ps.is_dyadic(h, blocks, 10) and B.max() < 2.0 ** 13
    m = ais.annealed_near_tie_margin(q, 0.0, 1.0, B)
    if name == "CTA13":
        return ais.AnnealedSampler(h, dense_J(L, q, pairs, blocks), case["seed"], case["n"], margin=m)
    return ais.AnnealedSparseSampler(h, pairs, blocks, case["seed"], case["n"], margin=m)


# ---- exact log Z ---------------------------------------------------------------------------------------------------

def test_exact_forms_equal_enumeration():
    for L, q, seed in ((5, 4, 1), (6, 3, 2), (2, 32, 3)):
        m = synthetic.chain_potts_model(L, q, seed, coupling_scale=1.0,
                                        alphabet=(synthetic.ALPHABET + "BJOUXZ12345")[:q])
        assert math.isclose(ais.log_z_chain(m["h"], m["J"]), ais.log_z_enumeration(m["h"], m["J"]), rel_tol=1e-13)
    for L, q, n, seed in ((6, 3, 2, 4), (7, 3, 3, 5), (4, 8, 1, 6)):
        m = synthetic.planted_potts_model(L, q, n, seed, alphabet=(synthetic.ALPHABET + "BJOUXZ12345")[:q])
        exact = ais.log_z_enumeration(m["h"], m["J"])
        assert math.isclose(ais.log_z_disjoint_pairs(m["h"], m["J"], m["contacts"]), exact, rel_tol=1e-13)
    h, J = small_model(4, 3, 1)
    assert math.isclose(ais.log_z_enumeration(h, np.zeros_like(J)), ais.log_z0(h), rel_tol=1e-13)
    with pytest.raises(ValueError, match="j != i \\+ 1"):
        ais.log_z_chain(h, J)
    with pytest.raises(ValueError, match="outside the listed pairs"):
        ais.log_z_disjoint_pairs(h, J, [[0, 2]])


def test_chain_model_is_dyadic_and_nearest_neighbour():
    m = synthetic.chain_potts_model(30, 21, 9)
    assert ps.is_dyadic(m["h"], m["J"], 10)
    iu, ju = np.triu_indices(30, 1)
    nz = np.abs(m["J"]).reshape(len(iu), -1).max(axis=1) > 0
    assert np.all(ju[nz] == iu[nz] + 1) and nz.sum() == 29
    b = synthetic.chain_potts_model(30, 21, 9)
    assert np.array_equal(m["J"], b["J"]) and np.array_equal(m["h"], b["h"])


# ---- the restatement -----------------------------------------------------------------------------------------------

def test_zero_couplings_give_zero_weights():
    h, J = small_model(4, 3, 7)
    s = ais.AnnealedSampler(h, np.zeros_like(J), 3, 500)
    fwd, rev = ais.restated_log_weights(s, 16, 4)
    assert not fwd.any() and not rev.any()
    log_mean, ess, se = model_ops.ais_summary(fwd)
    assert log_mean == 0.0 and ess == 500 and se == 0.0
    assert ais.log_z0(h) + log_mean == ais.log_z0(h)


def test_split_schedules_and_offsets_agree():
    h, J = small_model(4, 3, 1)
    b = ais.linear_schedule(64)
    a = ais.AnnealedSampler(h, J, 5, 64)
    a.anneal(b[:17])
    a.anneal(b[16:])
    one = ais.AnnealedSampler(h, J, 5, 64)
    one.anneal(b)
    part = ais.AnnealedSampler(h, J, 5, 24, chain_offset=40)
    part.anneal(b)
    assert np.array_equal(a.codes(), one.codes()) and np.array_equal(a.logw, one.logw)
    assert np.array_equal(part.codes(), one.codes()[40:]) and np.array_equal(part.logw, one.logw[40:])


def test_annealed_draw_at_beta_one_is_the_models():
    """v = h + 1 (Z - h) differs from Z by roundings only; with dyadic Z it is Z, so the annealed sweep at beta = 1
    is the plain chain's sweep code for code."""
    h, J = draw_model(12, 21, 3)
    a = ais.AnnealedSampler(h, J, 9, 300)
    b = ps.Sampler(h, J, 9, 300)
    a.anneal([1.0, 1.0, 1.0, 1.0])
    b.run(3, 1.0)
    assert np.array_equal(a.codes(), b.codes())


def test_margin_covers_the_plain_one():
    """The annealed margin is never below the plain draw's at beta = 1 with the same bounds when Z is rounded."""
    for q, B, zerr in ((2, 3.0, 1e-5), (21, 40.0, 1e-4), (32, 9.0, 0.0)):
        a = ais.annealed_near_tie_margin(q, zerr, 1.0, B)
        if zerr:
            assert a >= ps.near_tie_margin(q, zerr, 1.0, B)
        assert a > 0 and ais.annealed_near_tie_margin(q, 0.0, 0.0, B) <= a


@pytest.mark.parametrize("L,q", ENUM_MODELS)
def test_restated_estimates_within_their_standard_errors(L, q):
    h, J = small_model(L, q, 10 * L + q)
    exact = ais.log_z_enumeration(h, J)
    z0 = ais.log_z0(h)
    s = ais.AnnealedSampler(h, J, ENUM_SEED, ENUM_CHAINS)
    fwd, rev = ais.restated_log_weights(s, ENUM_K, ENUM_K)
    lf, _, sf = model_ops.ais_summary(fwd)
    lr, _, sr = model_ops.ais_summary(rev)
    assert within(z0 + lf, exact, sf), (z0 + lf, exact, sf)
    assert within(z0 - lr, exact, sr), (z0 - lr, exact, sr)
    # the reverse direction from exact samples of the model, drawn by enumeration
    p = ps.exact_distribution(h, J, 1.0, L, q)
    idx = np.random.default_rng(ENUM_SEED).choice(len(p), ENUM_CHAINS, p=p)
    e = ais.AnnealedSampler(h, J, ENUM_SEED, ENUM_CHAINS, init=np.array(np.unravel_index(idx, (q,) * L)).T)
    e.anneal(ais.linear_schedule(ENUM_K)[::-1])
    le, _, se = model_ops.ais_summary(e.logw)
    assert within(z0 - le, exact, se), (z0 - le, exact, se)


@pytest.mark.parametrize("L,q", DRAW_CASES)
def test_draw_comparison_power(L, q):
    h, J = draw_model(L, q, 1000 * L + q)
    ref = ais.AnnealedSampler(h, J, DRAW["seed"], DRAW["n"], margin=draw_margin(h, J))
    compared = 0
    for t, b in enumerate(sweep_schedules(DRAW["K"])):
        ref.anneal(b)
        compared += int(clean_after(ref, t).sum())
    share = compared / (DRAW["n"] * (DRAW["K"] + 1))
    print("L=%d q=%d: compared %.3f of the chain-sweeps, %.3f of the chains flagged, %d clean past t = 32"
          % (L, q, share, (ref.first_tie >= 0).mean(), clean_after(ref, ps.REFRESH).sum()))
    assert share >= DRAW_POWER[(L, q)]


@pytest.mark.parametrize("name", ["CTA13", "CTA2"])
def test_geometry_comparison_power(name):
    ref = geometry_restatement(name)
    case = dict(CTA13=CTA13, CTA2=CTA2)[name]
    compared = np.zeros(case["n"], dtype=np.int64)
    for t, b in enumerate(sweep_schedules(GEOMETRY_K, GEOMETRY_SWEEPS)):
        ref.anneal(b)
        compared += clean_after(ref, t)
    share = compared.sum() / (case["n"] * GEOMETRY_SWEEPS)
    print("%s: compared %.3f of the chain-sweeps, %d chains past sweep 32" % (name, share,
                                                                              (compared > ps.REFRESH).sum()))
    assert share >= GEOMETRY_POWER[name]
    assert (compared > ps.REFRESH).sum() >= 3
    per_cta = chains_per_cta(case["L"], case["q"])
    assert (compared[-(case["n"] % per_cta):] > 0).any()        # the partial last CTA is compared


# ---- the command line and the library's refusals -------------------------------------------------------------------

def test_cli_arguments():
    o = logz_cli.parse_args(["m.model"])
    assert o == dict(model="m.model", chains=logz_cli.DEFAULT_CHAINS, temperatures=logz_cli.DEFAULT_TEMPERATURES,
                     burn_in=logz_cli.DEFAULT_TEMPERATURES, seed=0, alignment=None, focus=None, output=None)
    o = logz_cli.parse_args(["m.model", "--chains", "5", "--temperatures", "8", "--burn-in", "0", "--seed",
                             "18446744073709551615", "--alignment", "a.a2m", "--focus", "seq0", "-o", "p.csv"])
    assert (o["chains"], o["temperatures"], o["burn_in"], o["seed"]) == (5, 8, 0, 2 ** 64 - 1)
    assert logz_cli.parse_args(["m.model", "--temperatures", "16"])["burn_in"] == 16
    for bad in ([],                                                        # no model
                ["m.model", "--chains", "0"],
                ["m.model", "--temperatures", "0"],
                ["m.model", "--temperatures", "100"],                      # not a power of two
                ["m.model", "--temperatures", str(1 << 31)],
                ["m.model", "--burn-in", "-1"],
                ["m.model", "--seed", "-1"],
                ["m.model", "--seed", str(1 << 64)],
                ["m.model", "-o", "p.csv"],                                # -o without --alignment
                ["m.model", "--focus", "seq0"],
                ["m.model", "--chains", "many"],
                ["m.model", "--sweeps", "3"]):
        with pytest.raises(logz_cli.CliError):
            logz_cli.parse_args(bad)
        err = io.StringIO()
        assert logz_cli.main(bad, stderr=err) == 2 and "evcplm-logz" in err.getvalue()


def test_cli_reports_a_missing_model_file(tmp_path):
    err = io.StringIO()
    assert logz_cli.main([str(tmp_path / "none.model")], stdout=io.StringIO(), stderr=err) == 1
    assert "No such file" in err.getvalue()


def test_log_partition_refuses_bad_arguments():
    m = synthetic.planted_potts_model(6, 3, 1, 1)
    for kw in (dict(n_chains=0), dict(temperatures=0), dict(temperatures=3), dict(burn_in=-1)):
        with pytest.raises(ValueError):
            model_ops.log_partition(m, **kw)


def test_log_probabilities_refuses_symbols_outside_the_states():
    m = synthetic.planted_potts_model(6, 20, 1, 1, alphabet="ACDEFGHIKLMNPQRSTVWY")   # no gap state
    with pytest.raises(ValueError, match="2 of 3 sequences have symbols outside the model's 20 states"):
        model_ops.log_probabilities(m, ["ACDEFG", "AC-EFG", "ACDEF-"], 0.0)
    with pytest.raises(ValueError, match="1 of 2 sequences"):
        model_ops.log_probabilities(m, np.array([[0, 1, 2, 3, 4, 5], [0, 1, 2, 3, 4, 20]]), 0.0)
    with pytest.raises(ValueError, match="1 of 1 sequences"):
        model_ops.log_probabilities(m, np.array([[0, 1, 2, 3, 4, -1]]), 0.0)
    with pytest.raises(ValueError, match="L = 6"):
        model_ops.log_probabilities(m, ["ACDEF"], 0.0)


def test_library_checks_anneal_arguments_without_a_device():
    from evcouplings_b200 import _lib
    lib = _lib.load()
    fake = ctypes.c_void_p(256)          # never dereferenced: every call below is refused first
    good = np.array([0.0, 0.5, 1.0], dtype=np.float32)
    vp = good.ctypes.data_as(ctypes.c_void_p)
    assert lib.evc_sampler_anneal(fake, vp, -1, fake, None, None) != 0
    assert b"K must be >= 0" in lib.evc_last_error()
    assert lib.evc_sampler_anneal(fake, None, 2, fake, None, None) != 0 and b"null pointer" in lib.evc_last_error()
    assert lib.evc_sampler_anneal(fake, vp, 2, None, None, None) != 0 and b"null pointer" in lib.evc_last_error()
    for bad in (np.nan, np.inf, -np.inf):
        b = good.copy()
        b[2] = bad
        assert lib.evc_sampler_anneal(fake, b.ctypes.data_as(ctypes.c_void_p), 2, fake, None, None) != 0
        assert b"betas[2] is not finite" in lib.evc_last_error()
    assert lib.evc_sampler_anneal(None, vp, 2, fake, None, None) != 0 and b"null handle" in lib.evc_last_error()
