"""Host-side logic (no GPU): ingest, log/PlmcResult contract, writers, L-BFGS control flow.
The numerical backend here is the TEST-ONLY oracle engine (tests/cpu_engine.py)."""
import os

import numpy as np
import pytest

from evcouplings_b200 import lbfgs, model_io, msa, synthetic, tools
from oracle import plm_oracle as po
from cpu_engine import OracleEngine, OracleProblem

import golden_npz


def test_ingest_matches_oracle_restatement(tmp_path):
    """product ingest (numpy-vectorised) == oracle's per-character restatement, incl. invalid rows,
    lower-case insert columns, '.' gaps, focus selection and index_list."""
    rng = np.random.default_rng(0)
    alpha = "-ACDEFGHIKLMNPQRSTVWY"
    rows = []
    width = 30
    focus = list("".join(rng.choice(list(alpha[1:]), width)))
    for c in (0, 1, 2, 27, 28, 29):
        focus[c] = focus[c].lower()
    focus[10] = "-"
    rows.append("".join(focus))
    for k in range(40):
        s = list("".join(rng.choice(list(alpha), width)))
        for c in (0, 1, 2, 27, 28, 29):
            s[c] = s[c].lower() if s[c] != "-" else "."
        if k == 5:
            s[7] = "X"
        if k == 9:
            s[1] = "x"          # invalid because of an insert column
        if k == 11:
            s[15] = "B"
        rows.append("".join(s))
    p = tmp_path / "a.a2m"
    with open(p, "w") as f:
        for k, s in enumerate(rows):
            f.write(">%s\n%s\n%s\n" % ("FOC/11-39" if k == 0 else "s%d/1-30" % k, s[:17], s[17:]))
    for ig in (False, True):
        ali = msa.load_alignment(str(p), focus="FOC", ignore_gaps=ig)
        ids, seqs = po.read_a2m(str(p))
        ref = po.prepare_alignment(ids, seqs, focus="FOC", ignore_gaps=ig)
        assert ali.n_total == 41 and ali.n_valid == 38 == ref["n_valid"]
        assert (ali.valid == ref["valid"]).all()
        assert np.array_equal(ali.codes, ref["codes"])
        assert ali.q == ref["q"] and ali.gap_code == ref["gap_code"]
        assert ali.target_seq == ref["target_seq"]
        assert np.array_equal(ali.index_list, ref["index_list"])
        assert ali.region_start == 11 and ali.num_total_sites == 29 == ref["num_total_sites"]
        assert ali.codes.shape[1] == 23
    # non-focus mode uses every column
    ali = msa.load_alignment(str(p), focus=None)
    assert ali.codes.shape[1] == 30 and ali.focus_index is None


def test_ingest_errors(tmp_path):
    p = tmp_path / "ragged.fa"
    p.write_text(">a\nACD\n>b\nAC\n")
    with pytest.raises(msa.AlignmentError):
        msa.load_alignment(str(p))
    p2 = tmp_path / "empty.fa"
    p2.write_text("")
    with pytest.raises(msa.AlignmentError):
        msa.load_alignment(str(p2))
    p3 = tmp_path / "ok.fa"
    p3.write_text(">a\nACD\n>b\nACE\n")
    with pytest.raises(msa.AlignmentError):
        msa.load_alignment(str(p3), focus="zzz")


def test_threshold_rule():
    for theta, L in [(0.8, 40), (0.8, 50), (0.8, 82), (0.7, 33), (0.9, 200), (0.2, 17), (1.0, 9)]:
        assert msa.identity_threshold_count(theta, L) == po.identity_threshold_count(theta, L)
        c = msa.identity_threshold_count(theta, L)
        assert c / float(L) >= theta and (c == 0 or (c - 1) / float(L) < theta)


def test_model_writer_bytes_equal_golden(golden_dir, tmp_path):
    """product writer reproduces, byte for byte, the tiny.model that the reference's CouplingsModel read."""
    m = po.read_model(os.path.join(golden_dir, "tiny.model"))
    out = tmp_path / "w.model"
    model_io.write_model_file(str(out), m["L"], m["q"], m["n_valid"], m["n_invalid"], m["num_iter"], m["theta"],
                              m["lambda_h"], m["lambda_J"], m["lambda_group"], m["n_eff"], m["alphabet"],
                              m["weights"], m["target_seq"], m["index_list"], m["fi"], m["h"], m["fij"], m["J"])
    assert out.read_bytes() == open(os.path.join(golden_dir, "tiny.model"), "rb").read()
    assert os.path.getsize(out) == model_io.model_file_size(m["L"], m["q"], m["n_valid"] + m["n_invalid"])
    with pytest.raises(ValueError):
        model_io.write_model_file(str(out), m["L"], m["q"], m["n_valid"], m["n_invalid"], 1, 0.2, -1.0, 1.0, 0.0,
                                  1.0, m["alphabet"], m["weights"], m["target_seq"], m["index_list"], m["fi"],
                                  m["h"], m["fij"], m["J"])


def test_ec_writer_equals_golden_text(golden_dir, tmp_path):
    m = po.read_model(os.path.join(golden_dir, "tiny.model"))
    fn = np.sqrt((m["J"].astype(np.float64) ** 2).sum(axis=(1, 2)))
    out = tmp_path / "ecs.txt"
    model_io.write_ec_file(str(out), fn, m["L"], m["index_list"], m["target_seq"])
    assert out.read_text() == open(os.path.join(golden_dir, "tiny_ECs.txt")).read()


def test_pabp_ec_text_from_golden_J(golden_dir, tmp_path):
    g = golden_npz.load("pabp_golden")
    fn = np.sqrt((g["J"].astype(np.float64) ** 2).sum(axis=(1, 2)))
    out = tmp_path / "ecs.txt"
    cn = model_io.write_ec_file(str(out), fn, 82, g["index_list"], str(g["target_seq"]))
    assert np.abs(cn - g["ec_cn"]).max() < 2e-6
    first = out.read_text().split("\n")[0].split(" ")
    assert first[:5] == ["123", "K", "124", "G", "0"] and abs(float(first[5]) - 0.796611) < 2e-6


def test_lbfgs_control_flow_converges_to_scipy_optimum():
    """product L-BFGS (More-Thuente) driven with a numpy space reaches the optimum found by scipy."""
    codes = po.synthetic_msa_codes(60, 7, 3)
    counts = po.hamming_counts(codes, 0.8)
    w = 1.0 / counts
    prob = OracleProblem(codes, w, 21, -1, 0.01, 0.4, m=6)
    res = prob.fit(np.zeros(prob.n), lbfgs.default_params(max_iterations=0, epsilon=1e-6))
    assert res.status == lbfgs.LBFGS_SUCCESS
    xs, _ = po.fit(codes, w, 21, 0.01, 0.4, max_iter=3000)
    assert np.abs(prob.x - xs).max() < 2e-5
    # iteration cap is honoured and reported like libLBFGS
    prob2 = OracleProblem(codes, w, 21, -1, 0.01, 0.4, m=6)
    res2 = prob2.fit(np.zeros(prob.n), lbfgs.default_params(max_iterations=5, epsilon=1e-7))
    assert res2.status == lbfgs.LBFGSERR_MAXIMUMITERATION and res2.iterations == 5
    # already-minimised start
    prob3 = OracleProblem(codes, w, 21, -1, 0.01, 0.4, m=6)
    res3 = prob3.fit(prob.x.copy(), lbfgs.default_params(max_iterations=0, epsilon=1e-3))
    assert res3.status == lbfgs.LBFGS_ALREADY_MINIMIZED


def test_line_search_on_1d_functions():
    import math
    p = lbfgs.default_params()
    # phi(t) = (t-2)^2 : from t=0, phi'(0) = -4
    st, step, f, n = lbfgs.line_search_morethuente(lambda t: ((t - 2) ** 2, 2 * (t - 2)), 4.0, -4.0, 1.0, p)
    assert st is None and f <= 4.0 + 1e-4 * step * -4.0
    st, step, f, n = lbfgs.line_search_morethuente(lambda t: (math.exp(t) - 5 * t, math.exp(t) - 5), 1.0, -4.0, 10.0, p)
    assert st is None and abs(math.exp(step) - 5) <= 0.9 * 4
    st, _, _, _ = lbfgs.line_search_morethuente(lambda t: (t, 1.0), 0.0, 1.0, 1.0, p)
    assert st == lbfgs.LBFGSERR_INCREASEGRADIENT


def test_run_plmc_contract_with_oracle_engine(tmp_path):
    """run_plmc host logic: files, log lines, PlmcResult fields (engine = test-only oracle)."""
    codes = synthetic.synthetic_msa_codes(120, 14, 9)
    a2m = tmp_path / "in" / "ali.a2m"
    os.makedirs(a2m.parent)
    synthetic.write_a2m(str(a2m), codes)
    for ig in (False, True):
        ecs = tmp_path / ("out%d" % ig) / "x_ECs.txt"
        model = tmp_path / ("out%d" % ig) / "x.model"
        res, run = tools.run_plmc(str(a2m), str(ecs), str(model), focus_seq="seq0/1-14", theta=0.8,
                                  ignore_gaps=ig, iterations=20, lambda_h=0.01, lambda_J=0.01 * 20 * 13,
                                  cpu=4, engine=OracleEngine(), return_run=True)
        assert res.couplings_file == str(ecs) and res.param_file == str(model)
        assert res.num_valid_seqs == 120 and res.num_total_seqs == 120
        assert res.num_valid_sites == 14 and res.num_total_sites == 14
        assert res.focus_seq_index == 1 and res.region_start == 1
        assert abs(res.effective_samples - run.n_eff) < 0.06
        assert res.optimization_status == "LBFGSERR_MAXIMUMITERATION"
        assert list(res.iteration_table.columns) == tools.ITER_FIELDS
        assert len(res.iteration_table) == 20
        assert all(isinstance(v, (int, float, str)) or v is None for k, v in res._asdict().items()
                   if k != "iteration_table")
        m = po.read_model(str(model))
        q = 20 if ig else 21
        assert (m["L"], m["q"], m["n_valid"], m["n_invalid"], m["num_iter"]) == (14, q, 120, 0, 20)
        assert abs(m["theta"] - 0.2) < 1e-7 and abs(m["lambda_J"] - 0.01 * 20 * 13) < 1e-5
        assert m["alphabet"] == ("ACDEFGHIKLMNPQRSTVWY" if ig else "-ACDEFGHIKLMNPQRSTVWY")
        assert np.array_equal(m["weights"].astype(np.int64), run.counts)
        assert np.allclose(m["h"].ravel(), run.x[:14 * q]) and np.allclose(m["J"].ravel(), run.x[14 * q:])
        fi_o, fij_o = po.frequencies(run.alignment.codes, run.weights, q, run.alignment.gap_code)
        assert np.abs(m["fi"] - fi_o).max() < 1e-6 and np.abs(m["fij"] - fij_o).max() < 1e-6
        lines = open(ecs).read().strip().split("\n")
        assert len(lines) == 14 * 13 // 2
        cn = po.cn_scores(m["J"], 14)
        assert abs(float(lines[3].split(" ")[5]) - cn[3]) < 1e-6
    with pytest.raises(tools.ResourceError):
        tools.run_plmc(str(tmp_path / "missing.a2m"), str(tmp_path / "e.txt"), engine=OracleEngine())
    with pytest.raises(tools.InvalidParameterError):
        tools.run_plmc(str(a2m), str(tmp_path / "e.txt"), lambda_g=0.5, engine=OracleEngine())


def test_default_engine_fails_loudly_without_gpu(tmp_path):
    """no CPU fallback: without a usable CUDA device the product path raises."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from evcouplings_b200 import _lib
    codes = synthetic.synthetic_msa_codes(20, 6, 1)
    a2m = tmp_path / "a.a2m"
    synthetic.write_a2m(str(a2m), codes)
    with pytest.raises(_lib.EngineUnavailableError):
        tools.run_plmc(str(a2m), str(tmp_path / "e.txt"), focus_seq="seq0")


def test_shard_bounds():
    from evcouplings_b200.engine import shard_bounds
    for n, w in [(10, 3), (7, 8), (100, 4), (1, 1), (50000, 8)]:
        cover = []
        for r in range(w):
            lo, hi = shard_bounds(n, w, r)
            assert 0 <= lo <= hi <= n
            cover += list(range(lo, hi))
        assert cover == list(range(n))


def test_ingest_property_random_alignments():
    """hypothesis: for random A2M-like alignments (mixed case, '.', '-', invalid characters, wrapped lines) the
    product ingest equals the oracle's per-character restatement of plmc's rules, in both gap modes."""
    import tempfile
    from hypothesis import given, settings, strategies as st, HealthCheck

    chars = "ACDEFGHIKLMNPQRSTVWY" + "acdefghiklmnpqrstvwy" + "--..XBZxb*"

    @settings(max_examples=60, deadline=None, suppress_health_check=list(HealthCheck))
    @given(st.integers(2, 9), st.integers(4, 40), st.integers(0, 2 ** 31 - 1), st.booleans(), st.booleans())
    def check(n_rows, width, seed, ignore_gaps, use_focus):
        rng = np.random.default_rng(seed)
        rows = ["".join(rng.choice(list(chars), width)) for _ in range(n_rows)]
        # the focus row needs >= 2 upper-case residues to define model sites
        f = list(rows[0])
        f[0], f[width // 2] = "A", "W"
        rows[0] = "".join(f)
        with tempfile.TemporaryDirectory() as d:
            p = os.path.join(d, "r.a2m")
            with open(p, "w") as fh:
                for k, s in enumerate(rows):
                    cut = int(rng.integers(1, width))
                    fh.write(">%s/%d-%d some text\n%s\n%s\n" % ("q%d" % k, 7 + k, 7 + k + width, s[:cut], s[cut:]))
            focus = "q0" if use_focus else None
            ids, seqs = po.read_a2m(p)
            try:
                ref = po.prepare_alignment(ids, seqs, focus=focus, ignore_gaps=ignore_gaps)
            except Exception:
                ref = None
            try:
                ali = msa.load_alignment(p, focus=focus, ignore_gaps=ignore_gaps)
            except msa.AlignmentError:
                ali = None
            if ref is None or ali is None:
                # both must reject (e.g. fewer than two model sites)
                assert ali is None and (ref is None or len(ref["focus_cols"]) < 2)
                return
            assert np.array_equal(ali.valid, ref["valid"])
            assert np.array_equal(ali.codes, ref["codes"])
            assert ali.q == ref["q"] and ali.gap_code == ref["gap_code"]
            assert np.array_equal(ali.index_list, ref["index_list"])
            assert ali.region_start == ref["region_start"] and ali.num_total_sites == ref["num_total_sites"]
            if use_focus:
                assert ali.target_seq == ref["target_seq"] and ali.focus_index == 0

    check()


def test_apc_and_frequency_normalisation_properties():
    rng = np.random.default_rng(1)
    for L, q in ((5, 21), (12, 20), (30, 5)):
        Jt = rng.normal(0, 0.3, (L * (L - 1) // 2, q, q))
        fn = np.sqrt((Jt ** 2).sum(axis=(1, 2)))
        assert np.abs(model_io.apc_cn_scores(fn, L) - po.cn_scores(Jt, L)).max() < 1e-12
        fi_c = rng.uniform(0, 5, (L, q))
        fij_c = rng.uniform(0, 5, (L * (L - 1) // 2, q, q))
        fi, fij = model_io.normalise_frequencies(fi_c, fij_c, 7.5, True)
        assert np.allclose(fi.sum(axis=1), 1) and np.allclose(fij.sum(axis=(1, 2)), 1)
        fi, fij = model_io.normalise_frequencies(fi_c, fij_c, 7.5, False)
        assert np.allclose(fi, fi_c / 7.5) and np.allclose(fij, fij_c / 7.5)
    # an all-gap column under ignore_gaps must not produce NaN
    fi, fij = model_io.normalise_frequencies(np.zeros((3, 20)), np.zeros((3, 20, 20)), 1.0, True)
    assert np.isfinite(fi).all() and np.isfinite(fij).all()
    assert (model_io.apc_cn_scores(np.zeros(3), 3) == 0).all()


def test_fx_limb_packing_is_exact_under_fp32_allreduce():
    """Design invariant behind the single [g, -loglk] collective (csrc/vecops.cu pack_fx_kernel / unpack_fx,
    restated here in numpy): -loglk is sent as three fixed-point limbs of 18 / 18 / <= 17 bits (resolution 2^-16); any
    fp32 summation order over up to 64 ranks reproduces the sum of the per-rank values to that resolution, identically
    on every rank."""
    rng = np.random.default_rng(0)
    BITS, SCALE = 18, 65536.0
    mask = (1 << BITS) - 1

    def pack(v):
        q = int(np.rint(np.clip(v * SCALE, -9.0e15, 9.0e15)))
        return np.array([q & mask, (q >> BITS) & mask, q >> (2 * BITS)], dtype=np.float32)      # arithmetic shift keeps the sign

    def unpack(l):
        q = int(l[0]) + (int(l[1]) << BITS) + int(l[2]) * (1 << (2 * BITS))
        return q / SCALE

    for world in (1, 2, 8, 64):
        for scale in (1.0, 1e3, 1e6, 6.5e8, 1.3e11 / world):
            vals = rng.uniform(-1.0, 1.0, world) * scale
            vals[0] = abs(vals[0])
            limbs = np.stack([pack(v) for v in vals])                 # (world, 3) float32
            exact = sum(int(np.rint(v * SCALE)) for v in vals) / SCALE
            for order in (np.arange(world), rng.permutation(world), np.arange(world)[::-1]):
                acc = np.zeros(3, dtype=np.float32)
                for r in order:                                        # a ring / tree all-reduce is some such order
                    acc = (acc + limbs[r]).astype(np.float32)
                assert unpack(acc) == exact, (world, scale)
            assert abs(exact - vals.sum()) <= world * 0.5 / SCALE + 1e-9 * abs(vals.sum())
