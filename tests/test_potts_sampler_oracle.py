"""The Gibbs sampler's contract on the CPU: the counter-based uniforms, the float64 restatement
(oracle/potts_sampler.py) against exact enumeration, a planted model recovered by sampling and fitting, the
evcplm-sample command line and the library's argument checks (no device is touched)."""
import ctypes

import numpy as np
import pytest

from evcouplings_b200 import model_io, model_ops, sample_cli, synthetic
from oracle import plm_oracle, potts_sampler as ps

# (seed, c, t, i, L) -> u(c, t, i), from the definition in include/evcplm.h
PINNED_U = {
    (0, 0, 0, 0, 4): 0.3380524814128876,
    (1, 7, 3, 2, 4): 0.5776095688343048,
    (12345, 4095, 39, 63, 64): 0.7117485702037811,
    (2 ** 64 - 1, 0, -1, 0, 3): 0.40003541111946106,
}

# The planted model of the end-to-end recovery, here (oracle sampler + float64 fit) and on the GPU (evcplm-sample +
# evcplm-plmc).  RECOVERY_FRACTION is the share of planted pairs among the top n_contacts CN pairs that this CPU run
# reached (4 of 4), fixed before any GPU run.
PLANTED = dict(L=20, q=21, n_contacts=4, seed=3)
PLANTED_SAMPLES, PLANTED_SWEEPS, PLANTED_SAMPLE_SEED = 3000, 50, 1
RECOVERY_FRACTION = 1.0


def _mix_int(z):
    m = (1 << 64) - 1
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & m
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & m
    return z ^ (z >> 31)


def _u_int(seed, c, t, i, L):
    """u(c, t, i) with Python integers, independent of the numpy restatement."""
    m, phi = (1 << 64) - 1, 0x9E3779B97F4A7C15
    key = _mix_int(seed ^ _mix_int(((c + 1) * phi) & m))
    k = (t * L + i + 1) & m
    return ((_mix_int((key + k * phi) & m) >> 40) + 0.5) * 2.0 ** -24


def small_model(L, q, seed):
    """Fields U(-1, 1), couplings of magnitude U(0.5, 1) and random sign: the enumeration models."""
    rng = np.random.default_rng(seed)
    h = rng.uniform(-1.0, 1.0, (L, q))
    J = rng.uniform(0.5, 1.0, (L * (L - 1) // 2, q, q)) * rng.choice([-1.0, 1.0], (L * (L - 1) // 2, q, q))
    return h.astype(np.float32), J.astype(np.float32)


def distribution_bounds(p, n, tail=1e-6):
    """Bounds on the total-variation distance and Pearson's chi^2 of n independent draws from p, each exceeded with
    probability about `tail`: TV <= E[TV] + sqrt(ln(1/tail) / (2 n)) (E[TV] <= sum_k sqrt(p_k (1 - p_k) / (2 pi n)),
    the mean absolute deviation of a binomial count; the deviation term is McDiarmid's inequality, one draw moving TV
    by at most 1/n), and the chi^2 quantile 1 - tail with len(p) - 1 degrees of freedom."""
    from scipy.stats import chi2
    tv = np.sum(np.sqrt(p * (1 - p) / (2 * np.pi * n))) + np.sqrt(np.log(1 / tail) / (2 * n))
    return tv, chi2.ppf(1 - tail, len(p) - 1)


def check_against_enumeration(codes, h, J, beta):
    L, q = h.shape
    p = ps.exact_distribution(h, J, beta, L, q)
    n = len(codes)
    counts = np.bincount(ps.state_index(codes, q), minlength=len(p))
    tv = 0.5 * np.abs(counts / n - p).sum()
    x2 = np.sum((counts - n * p) ** 2 / (n * p))
    tv_max, x2_max = distribution_bounds(p, n)
    assert tv <= tv_max and x2 <= x2_max, (tv, tv_max, x2, x2_max)
    return tv, x2


def test_counter_pinned_values():
    for (seed, c, t, i, L), u in PINNED_U.items():
        assert _u_int(seed, c, t, i, L) == u
        assert ps.uniform(ps.chain_key(seed, np.array([c])), t, i, L)[0] == u
        # 25 significant bits: exact in float64, strictly inside (0, 1)
        assert 0.0 < u < 1.0 and (u * 2 ** 25) == int(u * 2 ** 25)


def test_uniform_start_covers_codes_evenly():
    from scipy.stats import chi2
    for q in (2, 5, 21, 32):
        s = ps.uniform_start(7, 20000, 3, q, chain_offset=5)
        for i in range(3):
            n = np.bincount(s[:, i], minlength=q)
            assert len(n) == q
            e = len(s) / q
            assert np.sum((n - e) ** 2 / e) <= chi2.ppf(1 - 1e-6, q - 1)
    # the same chains with another chain_offset split
    a = ps.uniform_start(7, 100, 4, 21)
    assert np.array_equal(a[40:], ps.uniform_start(7, 60, 4, 21, chain_offset=40))


@pytest.mark.parametrize("L,q", [(4, 3), (3, 5)])
@pytest.mark.parametrize("beta", [0.0, 0.5, 1.0])
def test_oracle_sampler_matches_enumeration(L, q, beta):
    h, J = small_model(L, q, 10 * L + q)
    s = ps.Sampler(h, J, seed=11, n_chains=40000)
    s.run(32, beta)
    check_against_enumeration(s.codes(), h, J, beta)


def test_oracle_split_runs_and_offsets_agree():
    h, J = small_model(4, 3, 1)
    a = ps.Sampler(h, J, 5, 64)
    a.run(13)
    a.run(27)
    b = ps.Sampler(h, J, 5, 64)
    b.run(40)
    c = ps.Sampler(h, J, 5, 32, chain_offset=32)
    c.run(40)
    assert np.array_equal(a.codes(), b.codes()) and np.array_equal(b.codes()[32:], c.codes())


def planted_recovery(cn, L, contacts):
    iu, ju = np.triu_indices(L, 1)
    top = np.argsort(-np.asarray(cn), kind="stable")[:len(contacts)]
    found = {(int(iu[k]), int(ju[k])) for k in top}
    return len(found & {tuple(int(v) for v in p) for p in contacts}) / len(contacts)


def test_planted_model_recovered_on_cpu():
    """oracle sampler -> float64 pseudo-likelihood fit -> CN scores: the planted pairs rank first."""
    m = synthetic.planted_potts_model(**PLANTED)
    L, q = m["L"], m["q"]
    s = ps.Sampler(m["h"], m["J"], PLANTED_SAMPLE_SEED, PLANTED_SAMPLES)
    s.run(PLANTED_SWEEPS)
    codes = s.codes()
    x, _ = plm_oracle.fit(codes, np.ones(len(codes)), q, 0.01, 1.0, max_iter=40)
    cn = plm_oracle.cn_scores(x[L * q:].reshape(-1, q, q), L)
    assert planted_recovery(cn, L, m["contacts"]) >= RECOVERY_FRACTION


def test_planted_model_is_deterministic_and_writable(tmp_path):
    a = synthetic.planted_potts_model(30, 21, 5, 9)
    b = synthetic.planted_potts_model(30, 21, 5, 9)
    assert all(np.array_equal(a[k], b[k]) if isinstance(a[k], np.ndarray) else a[k] == b[k] for k in a)
    pairs = a["contacts"]
    assert len(pairs) == 5 and np.all(pairs[:, 1] - pairs[:, 0] >= 2) and len(set(pairs.ravel())) == 10
    iu, ju = np.triu_indices(30, 1)
    strong = {(int(i), int(j)) for i, j, blk in zip(iu, ju, a["J"]) if np.abs(blk).max() > 0}
    assert strong == {tuple(int(v) for v in p) for p in pairs}
    path = str(tmp_path / "planted.model")
    model_io.write_model_file(path, a["L"], a["q"], a["n_valid"], a["n_invalid"], a["num_iter"], a["theta"],
                              a["lambda_h"], a["lambda_J"], a["lambda_group"], a["n_eff"], a["alphabet"],
                              a["weights"], a["target_seq"], a["index_list"], a["fi"], a["h"], a["fij"], a["J"])
    r = model_ops.read_model(path)
    assert r["alphabet"] == a["alphabet"] and r["target_seq"] == a["target_seq"]
    assert np.array_equal(r["h"], a["h"]) and np.array_equal(r["J"], a["J"])
    assert np.array_equal(model_ops.model_x(r), np.concatenate([a["h"].ravel(), a["J"].ravel()]))


def test_write_a2m_alphabet_keyword(tmp_path):
    codes = np.array([[0, 1, 2], [3, 2, 1]], dtype=np.uint8)
    synthetic.write_a2m(str(tmp_path / "a.a2m"), codes)
    assert (tmp_path / "a.a2m").read_text() == ">seq0/1-3\n-AC\n>seq1/1-3\nDCA\n"
    synthetic.write_a2m(str(tmp_path / "b.a2m"), codes, alphabet="ACGT")
    assert (tmp_path / "b.a2m").read_text() == ">seq0/1-3\nACG\n>seq1/1-3\nTGC\n"


def test_cli_arguments():
    o = sample_cli.parse_args(["m.model", "-n", "10", "--sweeps", "5", "-o", "out.a2m"])
    assert o == dict(model="m.model", n=10, sweeps=5, seed=0, beta=1.0, init="random", output="out.a2m")
    o = sample_cli.parse_args(["m.model", "-n", "3", "--sweeps", "0", "--seed", "18446744073709551615", "--beta",
                               "0.5", "--init", "target", "-o", "x"])
    assert o["seed"] == 2 ** 64 - 1 and o["beta"] == 0.5 and o["init"] == "target" and o["sweeps"] == 0
    for bad in (["m.model", "--sweeps", "5", "-o", "x"],                       # no -n
                ["m.model", "-n", "10", "-o", "x"],                            # no --sweeps
                ["m.model", "-n", "10", "--sweeps", "5"],                      # no -o
                ["-n", "10", "--sweeps", "5", "-o", "x"],                      # no model
                ["m.model", "-n", "0", "--sweeps", "5", "-o", "x"],
                ["m.model", "-n", "10", "--sweeps", "-1", "-o", "x"],
                ["m.model", "-n", "10", "--sweeps", "5", "--seed", "-1", "-o", "x"],
                ["m.model", "-n", "10", "--sweeps", "5", "--beta", "nan", "-o", "x"],
                ["m.model", "-n", "10", "--sweeps", "5", "--init", "target2", "-o", "x"],
                ["m.model", "-n", "ten", "--sweeps", "5", "-o", "x"],
                ["m.model", "-n", "10", "--sweeps", "5", "-o", "x", "--thin", "2"]):
        with pytest.raises(sample_cli.CliError):
            sample_cli.parse_args(bad)
        import io
        err = io.StringIO()
        assert sample_cli.main(bad, stderr=err) == 2 and "evcplm-sample" in err.getvalue()


def test_cli_reports_a_missing_model_file(tmp_path):
    import io
    err = io.StringIO()
    rc = sample_cli.main([str(tmp_path / "none.model"), "-n", "2", "--sweeps", "1", "-o", str(tmp_path / "o.a2m")],
                         stderr=err)
    assert rc == 1 and "No such file" in err.getvalue()


def test_library_checks_sampler_arguments_without_a_device():
    from evcouplings_b200 import _lib
    lib = _lib.load()
    fake_x = ctypes.c_void_p(256)        # never dereferenced: every call below is refused first
    s = ctypes.c_void_p()

    def create(L, q, n, init=None, x=fake_x, offset=0):
        p = None if init is None else init.ctypes.data_as(ctypes.c_void_p)
        rc = lib.evc_sampler_create(ctypes.byref(s), x, L, q, p, n, offset, 1, 0)
        return rc, lib.evc_last_error().decode()

    for q in (1, 33, 0, -5):
        rc, msg = create(10, q, 4)
        assert rc != 0 and "q=%d" % q in msg
    init = np.zeros((4, 10), dtype=np.uint8)
    init[2, 7] = 21
    rc, msg = create(10, 21, 4, init)
    assert rc != 0 and "init code 21 at chain 2, site 7 out of range" in msg
    rc, msg = create(10, 21, 0)
    assert rc != 0 and "n_chains" in msg
    rc, msg = create(10, 21, 4, offset=-1)
    assert rc != 0 and "chain_offset" in msg
    rc, msg = create(1, 21, 4)
    assert rc != 0 and "L >= 2" in msg
    for L, q in ((2768, 21), (1816, 32)):          # 4 L q + L > 227 KB
        rc, msg = create(L, q, 4)
        assert rc != 0 and "shared memory" in msg and "58 000" in msg
    rc, msg = create(10, 21, 4, x=None)
    assert rc != 0 and "null pointer" in msg
    assert lib.evc_sampler_run(None, 1, 1.0, None, None) != 0 and b"null handle" in lib.evc_last_error()
    assert lib.evc_sampler_codes(None, None, None) != 0
    lib.evc_sampler_destroy(None)
