"""Conditional sampling on the CPU: the float64 restatement (oracle/conditional_sampler.py) against the plain one and
against exact enumeration of the conditional distribution, the parsing of position specs, and every refusal of the
command line, of model_ops and of the library that comes before any device work."""
import ctypes
import io

import numpy as np
import pytest

from evcouplings_b200 import model_io, model_ops, sample_cli, synthetic
from oracle import conditional_sampler as cs, potts_sampler as ps
from test_potts_sampler_oracle import distribution_bounds, small_model


def check_conditional(codes, h, J, beta, free, context, allowed=None):
    """TV and chi^2 of the free sites' states in ``codes`` against the exact conditional, within the bounds of their
    sampling distributions (states of probability 0 must never be drawn)."""
    q = h.shape[1]
    p = cs.exact_conditional(h, J, beta, free, context, allowed)
    n = len(codes)
    counts = np.bincount(ps.state_index(codes[:, free], q), minlength=len(p))
    assert counts[p == 0].sum() == 0
    tv = 0.5 * np.abs(counts / n - p).sum()
    live = p > 0
    x2 = np.sum((counts[live] - n * p[live]) ** 2 / (n * p[live]))
    tv_max, x2_max = distribution_bounds(p[live], n)
    assert tv <= tv_max and x2 <= x2_max, (tv, tv_max, x2, x2_max)
    return tv, x2


def two_contexts(L, q, n, seed):
    """n chains: the first half start at one random context, the second half at another."""
    rng = np.random.default_rng(seed)
    ctx = rng.integers(0, q, (2, L))
    return np.repeat(ctx, [n // 2, n - n // 2], axis=0), ctx


def planted_model():
    return synthetic.planted_potts_model(12, 21, 2, 4)


def test_all_free_equals_the_plain_restatement():
    for L, q, beta in ((5, 3, 1.0), (7, 21, 0.5)):
        h, J = small_model(L, q, L + q)
        margin = ps.near_tie_margin(q, 1e-6, beta, ps.z_bound(h, J, L, q))
        n = 300
        a = ps.Sampler(h, J, 3, n, chain_offset=17, margin=margin)
        b = cs.ConditionalSampler.from_model(h, J, 3, n, np.arange(L), chain_offset=17, margin=margin)
        assert np.array_equal(b.hc, np.repeat(np.asarray(h, dtype=np.float64)[None], n, axis=0))
        for _ in range(5):
            assert a.run(7, beta) == b.run(7, beta)
            assert np.array_equal(a.codes(), b.codes())
        assert np.array_equal(a.first_tie, b.first_tie)


def test_fold_and_reduced_couplings_agree_with_their_sparse_forms():
    m = planted_model()
    L, q = m["L"], m["q"]
    free = np.array([0, 3, 4, 11])
    init, _ = two_contexts(L, q, 6, 1)
    pairs = np.array(np.triu_indices(L, 1)).T
    assert np.array_equal(cs.fold(m["h"], m["J"], free, init), cs.fold_sparse(m["h"], pairs, m["J"], free, init))
    assert np.array_equal(cs.reduced_couplings(m["J"], L, q, free),
                          cs.reduced_couplings_sparse(L, q, pairs, m["J"], free))
    # the fold is the field of the full model at the free sites: Z_i(a) with the free sites' couplings removed
    U = ps.full_couplings(m["J"], L, q)
    clamped = cs.clamped_sites(L, free)
    for c in range(len(init)):
        for k, i in enumerate(free):
            want = m["h"][i].astype(np.float64) + sum(U[i, :, j, init[c, j]] for j in clamped)
            assert np.array_equal(cs.fold(m["h"], m["J"], free, init)[c, k], want)


@pytest.mark.parametrize("allowed", [None, [0b111, 0b101, 0b011], [0b010, 0b111, 0b110]])
@pytest.mark.parametrize("beta", [0.5, 1.0])
def test_restatement_matches_the_exact_conditional(allowed, beta):
    """L = 6, q = 3, three free sites, two contexts; masks that remove a state and a single-state mask."""
    L, q = 6, 3
    h, J = small_model(L, q, 60 + q)
    free = np.array([1, 3, 4])
    n = 40000
    init, ctx = two_contexts(L, q, n, 5)
    s = cs.ConditionalSampler.from_model(h, J, 11, n, free, allowed=allowed, init=init)
    s.run(32, beta)
    codes = s.codes().astype(np.int64)
    clamped = cs.clamped_sites(L, free)
    assert np.array_equal(codes[:, clamped], init[:, clamped])
    check_conditional(codes[:n // 2], h, J, beta, free, ctx[0], allowed)
    check_conditional(codes[n // 2:], h, J, beta, free, ctx[1], allowed)


def test_masked_draw_keeps_to_allowed_states():
    s = cs.ConditionalSampler(np.zeros((2, 1, 4)), np.zeros((4, 4)), [0], 2, 1, allowed=[0b0110],
                              context=np.zeros((2, 2), dtype=np.int64))
    assert list(s.highest) == [2]
    s.run(1)
    assert set(s.codes()[:, 0]) <= {1, 2}


def test_position_specs():
    assert sample_cli.parse_positions("30-33,60") == [30, 31, 32, 33, 60]
    assert sample_cli.parse_positions("5") == [5]
    assert sample_cli.parse_positions(" 2-2 , 7") == [2, 7]
    for bad in ("", "3-", "-3", "a", "5-3", "1,,2", "1-2-3", "1.5"):
        with pytest.raises(sample_cli.CliError):
            sample_cli.parse_positions(bad)
    assert sample_cli.parse_allow(["33:AVILM", "2:C"]) == {33: "AVILM", 2: "C"}
    for bad in (["33"], ["33:"], [":AV"], ["x:AV"], ["3:A", "3:C"]):
        with pytest.raises(sample_cli.CliError):
            sample_cli.parse_allow(bad)


def test_cli_options_parse():
    o = sample_cli.parse_args(["m.model", "-n", "2", "--sweeps", "1", "--free", "3-5,9", "--allow", "4:AC",
                               "--allow", "9:W", "--init", "target", "-o", "x"])
    assert o["free"] == [3, 4, 5, 9] and o["allow"] == {4: "AC", 9: "W"} and o["init"] == "target"
    o = sample_cli.parse_args(["m.model", "-n", "10", "--sweeps", "5", "-o", "out.a2m"])
    assert "free" not in o and "allow" not in o


@pytest.fixture
def model_file(tmp_path):
    m = planted_model()
    path = str(tmp_path / "planted.model")
    model_io.write_model_file(path, m["L"], m["q"], m["n_valid"], m["n_invalid"], m["num_iter"], m["theta"],
                              m["lambda_h"], m["lambda_J"], m["lambda_group"], m["n_eff"], m["alphabet"],
                              m["weights"], m["target_seq"], m["index_list"], m["fi"], m["h"], m["fij"], m["J"])
    return path, m


def test_cli_refusals(tmp_path, model_file):
    path, m = model_file
    good = str(tmp_path / "init.fa")
    synthetic.write_a2m(good, np.zeros((3, m["L"]), dtype=np.uint8), alphabet=m["alphabet"])
    short = str(tmp_path / "short.fa")
    with open(short, "w") as f:
        f.write(">a\n" + "A" * (m["L"] - 1) + "\n>b\n" + "A" * m["L"] + "\n>c\n" + "A" * m["L"] + "\n")
    foreign = str(tmp_path / "foreign.fa")
    with open(foreign, "w") as f:
        f.write("".join(">s\n" + "B" * m["L"] + "\n" for _ in range(3)))
    base = [path, "-n", "3", "--sweeps", "1", "-o", str(tmp_path / "o.a2m")]
    for extra in (["--free", "3-"],                                   # malformed spec
                  ["--free", "1-3", "--allow", "2"],                  # malformed allow
                  ["--free", "0-3", "--init", "target"],              # position 0 is not in index_list (1..L)
                  ["--free", "1-3,99", "--init", "target"],
                  ["--free", "1-3", "--allow", "2:B", "--init", "target"],     # B is not in the alphabet
                  ["--free", "1-3", "--allow", "5:A", "--init", "target"],     # 5 is clamped
                  ["--allow", "99:A"],                                # every site free, 99 still unknown
                  ["--free", "1-3"],                                  # clamped sites with --init random
                  ["--free", "1-3", "--init", "target2"],             # neither a keyword nor a file
                  ["--free", "1-3", "--init", short],
                  ["--free", "1-3", "--init", foreign],
                  ["--free", "1-3", "--init", good, "-n", "4"]):      # 3 rows, -n 4
        err = io.StringIO()
        assert sample_cli.main(base + extra, stderr=err) == 2, (extra, err.getvalue())
        assert "evcplm-sample" in err.getvalue()
    assert not (tmp_path / "o.a2m").exists()
    assert sample_cli.read_init_file(good, m, 3).shape == (3, m["L"])


def test_python_refusals_come_before_any_device_work():
    m = planted_model()
    tgt = "target"
    for kw, what in ((dict(free=[0], init=tgt), "index_list"),
                     (dict(free=[1, 2, 400], init=tgt), "index_list"),
                     (dict(free=[1, 2], allowed={2: "AZ"}, init=tgt), "alphabet"),
                     (dict(free=[1, 2], allowed={3: "A"}, init=tgt), "clamped"),
                     (dict(free=[1, 2], allowed={2: ""}, init=tgt), "letter"),
                     (dict(allowed={99: "A"}), "index_list"),
                     (dict(free=[], init=tgt), "at least one"),
                     (dict(free=[1, 2]), "context")):
        for call in (lambda: model_ops.PottsSampler(m, 4, **kw),
                     lambda: model_ops.sample_codes(m, 4, 1, **kw),
                     lambda: model_ops.sample_sequences(m, 4, 1, num_gpus=2, backend="gloo", **kw)):
            with pytest.raises(ValueError, match=what):
                call()
    sites, masks = model_ops.conditional_sites(m, [12, 1, 1, 5], {5: "AC-"}, "target")
    assert sites.tolist() == [0, 4, 11] and sites.dtype == np.int32
    a = m["alphabet"]
    assert masks.tolist() == [(1 << 21) - 1, (1 << a.index("A")) | (1 << a.index("C")) | 1, (1 << 21) - 1]
    sites, masks = model_ops.conditional_sites(m, None, {3: "W"})
    assert sites.tolist() == list(range(12)) and masks[2] == 1 << a.index("W")


def test_library_checks_conditional_arguments_without_a_device():
    from evcouplings_b200 import _lib
    lib = _lib.load()
    fake_x = ctypes.c_void_p(256)        # never dereferenced: every call below is refused first
    s = ctypes.c_void_p()

    def create(L, q, free, allowed=None, init=None, n=4, x=fake_x):
        f = np.ascontiguousarray(free, dtype=np.int32)
        a = None if allowed is None else np.ascontiguousarray(allowed, dtype=np.uint32)
        rc = lib.evc_sampler_create_conditional(
            ctypes.byref(s), x, L, q, f.ctypes.data_as(ctypes.c_void_p), len(f),
            None if a is None else a.ctypes.data_as(ctypes.c_void_p),
            None if init is None else init.ctypes.data_as(ctypes.c_void_p), n, 0, 1, 0)
        return rc, lib.evc_last_error().decode()

    init = np.zeros((4, 10), dtype=np.uint8)
    for free, what in (([], "nf"), (list(range(11)), "nf"), ([3, 2], "ascending"), ([2, 2], "ascending"),
                       ([-1, 2], "ascending"), ([2, 10], "ascending")):
        rc, msg = create(10, 21, free, init=init)
        assert rc != 0 and what in msg, (free, msg)
    for mask in (0, 1 << 21, (1 << 22) - 1):
        rc, msg = create(10, 21, [1, 2], [1, mask], init=init)
        assert rc != 0 and "allowed[1]" in msg, msg
    rc, msg = create(10, 21, [1, 2])
    assert rc != 0 and "init is required" in msg
    bad = init.copy()
    bad[3, 9] = 21
    rc, msg = create(10, 21, [1, 2], init=bad)
    assert rc != 0 and "init code 21 at chain 3, site 9 out of range" in msg
    rc, msg = create(3200, 21, list(range(2768)), init=np.zeros((4, 3200), dtype=np.uint8))
    assert rc != 0 and "shared memory" in msg and "nf q" in msg
    rc, msg = create(10, 21, [1, 2], init=init, x=None)
    assert rc != 0 and "null pointer" in msg
    rc, msg = create(10, 21, [1, 2], init=init, n=0)
    assert rc != 0 and "n_chains" in msg
    rc, msg = create(10, 1, [1, 2], init=init)
    assert rc != 0 and "q=1" in msg
    assert lib.evc_sampler_conditional_fields(None, None, None) != 0
