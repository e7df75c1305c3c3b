"""Boltzmann-machine learning on the CPU: the exact regularised-likelihood optimum of small models, the float64
restatement of the update loop (oracle/boltzmann.py) approaching it, a planted model whose connected correlations
the refinement reproduces better than the pseudo-likelihood start, and the argument checks of the command line, the
Python class and the library (no device is touched)."""
import ctypes
import io

import numpy as np
import pytest

from evcouplings_b200 import bmdca_cli, model_ops
from oracle import boltzmann as bm
from test_potts_sampler_oracle import small_model

# The enumeration models: targets f = the exact marginals of small_model(L, q, 10 L + q) at beta = 1, header
# n_eff = 1 and lambda_h = lambda_J = ENUM_LAMBDA, so F is strictly convex and theta* unique.  The loop starts at
# theta = 0 and runs ENUM_UPDATES updates of ENUM_SWEEPS sweeps with ENUM_CHAINS chains and learning rate ENUM_ETA.
ENUM_MODELS = [(4, 3), (3, 5)]
ENUM_LAMBDA = 0.01
ENUM_CHAINS, ENUM_SWEEPS, ENUM_ETA, ENUM_UPDATES, ENUM_SEED = 4096, 5, 0.5, 200, 1

# The bound on max_k |theta_k - theta*_k| after the loop: bias + ENUM_Z * sqrt(ENUM_TAU * eta / (M (2 - eta h_max))).
# Near theta* one update is delta' = (I - eta H) delta - eta xi, H = Cov(phi) + 2 lambda' I the Hessian of F and xi
# = c/M - E[phi] the chains' error, of covariance tau Cov(phi) / M (tau >= 1 allows for the correlation of persistent
# chains S sweeps apart).  In an eigendirection of H with eigenvalue h >= sigma (the Cov(phi) eigenvalue) the
# stationary variance is eta^2 tau sigma / M / (1 - (1 - eta h)^2) = eta tau sigma / (M h (2 - eta h))
# <= tau eta / (M (2 - eta h_max)), and a coordinate is a unit combination of eigendirections, so the same bound holds
# per coordinate.  bias = the distance the same number of exact-gradient updates (M -> infinity) leaves, computed.
# ENUM_TAU = 2 for 5 sweeps of these 4- and 3-site models; ENUM_Z = 6 standard deviations covers the 66 and 90
# coordinates with room.  Fixed before any GPU run: the restatement reaches 0.010 and 0.015 against bounds of about
# 0.09 and 0.10 (set by the noise term, 0.0143 sd at these settings).
ENUM_TAU, ENUM_Z = 2.0, 6.0


def enum_model(L, q):
    h, J = small_model(L, q, 10 * L + q)
    f = bm.exact_marginals(np.concatenate([h.ravel(), J.ravel()]), L, q).astype(np.float32)
    npairs = L * (L - 1) // 2
    alphabet = "ACDEFGHIKLMNPQRSTVWY"[:q]
    return dict(L=L, q=q, n_valid=0, n_invalid=0, num_iter=0, theta=0.0, lambda_h=ENUM_LAMBDA,
                lambda_J=ENUM_LAMBDA, lambda_group=0.0, n_eff=1.0, alphabet=alphabet,
                weights=np.zeros(0, dtype=np.float32), target_seq=alphabet[0] * L,
                index_list=np.arange(1, L + 1, dtype=np.int32), fi=f[:L * q].reshape(L, q),
                h=np.zeros((L, q), dtype=np.float32), fij=f[L * q:].reshape(npairs, q, q),
                J=np.zeros((npairs, q, q), dtype=np.float32))


def enum_targets(m):
    return np.concatenate([m["fi"].ravel(), m["fij"].ravel()])


def enum_bound(L, q):
    """(theta*, the bound on max |theta - theta*| after the loop)."""
    m = enum_model(L, q)
    f = enum_targets(m)
    lam = ENUM_LAMBDA / m["n_eff"]
    theta, _ = bm.optimum(f, L, q, lam, lam)
    bias = np.abs(bm.exact_descent(f, L, q, lam, lam, ENUM_ETA, ENUM_UPDATES) - theta).max()
    h_max = bm.hessian_max_eigenvalue(theta, L, q, lam, lam)
    assert ENUM_ETA * h_max < 2.0
    return theta, bias + ENUM_Z * np.sqrt(ENUM_TAU * ENUM_ETA / (ENUM_CHAINS * (2.0 - ENUM_ETA * h_max)))


@pytest.mark.parametrize("L,q", ENUM_MODELS)
def test_optimum_matches_moments(L, q):
    m = enum_model(L, q)
    theta, gmax = bm.optimum(enum_targets(m), L, q, ENUM_LAMBDA, ENUM_LAMBDA)
    assert gmax <= 1e-10
    # the moment condition itself: E_theta*[phi] - f = -2 lambda' theta*
    d = bm.exact_marginals(theta, L, q) - enum_targets(m).astype(np.float64)
    assert np.abs(d + 2 * ENUM_LAMBDA * theta).max() <= 1e-10


@pytest.mark.parametrize("L,q", ENUM_MODELS)
def test_restated_loop_approaches_the_optimum(L, q):
    m = enum_model(L, q)
    theta, bound = enum_bound(L, q)
    lam2_h, lam2_J = model_ops.bm_regularisation(m)
    x = bm.learn(model_ops.model_x(m), enum_targets(m), L, q, lam2_h, lam2_J, ENUM_UPDATES, ENUM_CHAINS,
                 seed=ENUM_SEED, sweeps=ENUM_SWEEPS, eta=ENUM_ETA)
    err = np.abs(x - theta).max()
    assert err <= bound, (err, bound)
    assert np.abs(theta).max() > 5 * bound          # the bound says something: theta = 0 would fail it


def test_update_restatement_rounds_each_operation():
    rng = np.random.default_rng(4)
    n, Lq, M = 500, 60, 777
    x = rng.normal(0, 1, n).astype(np.float32)
    c = rng.integers(0, M + 1, n).astype(np.uint32)
    f = rng.uniform(0, 1, n).astype(np.float32)
    new, st = bm.update(x, c, M, f, Lq, 0.05, 0.02, 0.3)
    for k in range(n):                               # Python floats: IEEE double, one rounding per operation
        d = float(c[k]) / M - float(f[k])
        g = d + (0.02 if k < Lq else 0.3) * float(x[k])
        assert new[k] == np.float32(float(x[k]) - 0.05 * g)
    ad = np.abs(c / M - f.astype(np.float64))
    assert st[0] == ad[:Lq].max() and st[1] == ad[Lq:].max()


def test_code_counts_layout():
    codes = np.array([[0, 1, 2], [2, 1, 0], [0, 1, 2]], dtype=np.uint8)
    c = bm.code_counts(codes, 3, 3)
    assert len(c) == 9 + 3 * 9
    assert list(c[:9]) == [2, 0, 1, 0, 3, 0, 1, 0, 2]
    assert c[9 + 0 * 3 + 1] == 2 and c[9 + 2 * 3 + 1] == 1           # pair (0, 1)
    assert c[18 + 0 * 3 + 2] == 2 and c[18 + 2 * 3 + 0] == 1          # pair (0, 2)
    assert c[27 + 1 * 3 + 2] == 2 and c[27 + 1 * 3 + 0] == 1          # pair (1, 2)
    assert all(c[9 + 9 * p: 18 + 9 * p].sum() == 3 for p in range(3))


def test_regularisation_from_the_header():
    m = enum_model(3, 5)
    assert model_ops.bm_regularisation(dict(m, lambda_h=0.01, lambda_J=16.2, n_eff=8.0)) == (2 * 0.01 / 8.0,
                                                                                             2 * 16.2 / 8.0)
    assert model_ops.bm_regularisation(dict(m, lambda_h=0.0, lambda_J=0.0, n_eff=0.0)) == (0.0, 0.0)
    for bad, msg in ((dict(lambda_h=-1.0), "mean-field"), (dict(n_eff=0.0), "n_eff"),
                     (dict(n_eff=-2.0, lambda_h=0.0), "n_eff")):
        with pytest.raises(ValueError, match=msg):
            model_ops.bm_regularisation(dict(m, **bad))


def test_learner_refuses_before_device_work():
    m = enum_model(3, 5)
    for kw, msg in ((dict(learning_rate=0.0), "learning_rate"), (dict(learning_rate=float("nan")), "learning_rate"),
                    (dict(learning_rate=-0.1), "learning_rate"), (dict(learning_rate=float("inf")), "learning_rate"),
                    (dict(n_chains=0), "chain"), (dict(burn_in=-1), "burn_in")):
        with pytest.raises(ValueError, match=msg):
            model_ops.BoltzmannLearner(m, engine=object(), **kw)
    with pytest.raises(ValueError, match="mean-field"):
        model_ops.BoltzmannLearner(dict(m, lambda_h=-1.0), engine=object())
    with pytest.raises(ValueError, match="n_eff"):
        model_ops.BoltzmannLearner(dict(m, n_eff=0.0), engine=object())
    for kw in (dict(updates=-1), dict(updates=2, sweeps=-1)):
        with pytest.raises(ValueError, match=">= 0"):
            model_ops.boltzmann_refine(m, engine=object(), **kw)


def test_cli_arguments():
    o = bmdca_cli.parse_args(["m.model", "--updates", "10", "-o", "out.model"])
    assert o == dict(model="m.model", updates=10, chains=10000, sweeps=10, learning_rate=0.05, burn_in=0, seed=0,
                     output="out.model", ecs=None)
    o = bmdca_cli.parse_args(["m.model", "--updates", "0", "--chains", "3", "--sweeps", "0", "--learning-rate", "1.5",
                              "--burn-in", "7", "--seed", "18446744073709551615", "-o", "x", "-c", "e.txt"])
    assert o == dict(model="m.model", updates=0, chains=3, sweeps=0, learning_rate=1.5, burn_in=7,
                     seed=2 ** 64 - 1, output="x", ecs="e.txt")
    for bad in (["m.model", "-o", "x"],                                        # no --updates
                ["m.model", "--updates", "5"],                                 # no -o
                ["--updates", "5", "-o", "x"],                                 # no model
                ["m.model", "--updates", "-1", "-o", "x"],
                ["m.model", "--updates", "5", "--chains", "0", "-o", "x"],
                ["m.model", "--updates", "5", "--sweeps", "-1", "-o", "x"],
                ["m.model", "--updates", "5", "--burn-in", "-1", "-o", "x"],
                ["m.model", "--updates", "5", "--learning-rate", "0", "-o", "x"],
                ["m.model", "--updates", "5", "--learning-rate", "nan", "-o", "x"],
                ["m.model", "--updates", "5", "--learning-rate", "-1", "-o", "x"],
                ["m.model", "--updates", "5", "--seed", "-1", "-o", "x"],
                ["m.model", "--updates", "five", "-o", "x"],
                ["m.model", "--updates", "5", "-o", "x", "--beta", "2"]):
        with pytest.raises(bmdca_cli.CliError):
            bmdca_cli.parse_args(bad)
        err = io.StringIO()
        assert bmdca_cli.main(bad, stderr=err) == 2 and "evcplm-bmdca" in err.getvalue()


def test_cli_reports_a_missing_model_file(tmp_path):
    err = io.StringIO()
    rc = bmdca_cli.main([str(tmp_path / "none.model"), "--updates", "1", "-o", str(tmp_path / "o.model")],
                        stderr=err)
    assert rc == 1 and "No such file" in err.getvalue()


def test_cli_refuses_a_mean_field_model_before_device_work(tmp_path):
    from evcouplings_b200 import model_io
    m = enum_model(3, 5)
    path = str(tmp_path / "m.model")
    model_io.write_model_file(path, 3, 5, 0, 0, 0, 0.0, 0.0, 0.0, 0.0, 0.0, m["alphabet"], m["weights"],
                              m["target_seq"], m["index_list"], m["fi"], m["h"], m["fij"], m["J"])
    raw = bytearray(open(path, "rb").read())
    raw[24:28] = np.array([-1.0], dtype="<f4").tobytes()             # lambda_h < 0: the mean-field marker
    open(path, "wb").write(bytes(raw))
    err = io.StringIO()
    assert bmdca_cli.main([path, "--updates", "1", "-o", str(tmp_path / "o.model")], engine=object(),
                          stderr=err) == 1
    assert "mean-field" in err.getvalue()


def test_library_checks_arguments_without_a_device():
    from evcouplings_b200 import _lib
    lib = _lib.load()
    fake = ctypes.c_void_p(256)          # never dereferenced: every call below is refused first

    def err():
        return lib.evc_last_error().decode()

    for q in (1, 33):
        assert lib.evc_code_counts(fake, 10, 5, q, fake, None) != 0 and "q=%d" % q in err()
    assert lib.evc_code_counts(fake, 10, 0, 21, fake, None) != 0 and "L=0" in err()
    assert lib.evc_code_counts(fake, 10, 32769, 21, fake, None) != 0 and "L=32769" in err()
    for N in (0, 2 ** 31):
        assert lib.evc_code_counts(fake, N, 5, 21, fake, None) != 0 and "N must be" in err()
    assert lib.evc_code_counts(None, 10, 5, 21, fake, None) != 0 and "null pointer" in err()
    assert lib.evc_bm_update(fake, fake, 0, fake, 10, 5, 0.1, 0.0, 0.0, fake, None) != 0 and "M must" in err()
    assert lib.evc_bm_update(fake, fake, 5, fake, 10, 11, 0.1, 0.0, 0.0, fake, None) != 0 and "Lq" in err()
    assert lib.evc_bm_update(fake, fake, 5, fake, 10, 5, float("nan"), 0.0, 0.0, fake, None) != 0
    assert "finite" in err()
    assert lib.evc_bm_update(fake, fake, 5, fake, 10, 5, 0.1, 0.0, 0.0, None, None) != 0 and "null" in err()
    assert lib.evc_sampler_set_model(None, fake, None) != 0 and "null pointer" in err()
