"""
Drop-in boundary tests (CPU): this project's run_plmc behind the reference's OWN couplings protocol
(evcouplings/couplings/protocol.py:363-429 ``standard`` -> ``infer_plmc`` :56-257, ``complex`` :480-594), its own
run_plmc driving the plmc-compatible executable (tools.py:126-307), and its own readers (CouplingsModel
model.py:317-400, read_raw_ec_file pairs.py:34-65, parse_plmc_log tools.py:20-108) on the files written here.

What the reference did is stored in tests/golden/reference_protocol.part*.npz (tests/golden/make_golden.py ran the
same inputs through the unmodified reference once): the arguments its protocol handed to run_plmc, the stage
outputs it derived, and what its readers read.  These tests make the same calls with the same arguments and
compare what this project writes and reads now against those stored values.  The numerical engine is the
test-only oracle engine (no GPU needed); the same host code runs over the CUDA engine in tests/test_gpu_parity.py.
"""
import io
import json
import os

import numpy as np
import pytest

import golden_npz


@pytest.fixture(scope="module")
def golden():
    return golden_npz.load("reference_protocol")


def _loads(a):
    return json.loads(str(a))


def _paths(v, tmp_path):
    if isinstance(v, str):
        return v.replace("{tmp}", str(tmp_path))
    if isinstance(v, list):
        return [_paths(x, tmp_path) for x in v]
    return v


def _call(golden, key, tmp_path):
    """the run_plmc call the reference's protocol made, with the paths moved under tmp_path"""
    call = _loads(golden[key])
    args = _paths(call["args"], tmp_path)
    kwargs = {k: _paths(v, tmp_path) for k, v in call["kwargs"].items()}
    for p in args[1:]:
        os.makedirs(os.path.dirname(p), exist_ok=True)
    return args, kwargs


def _read_ecs(path):
    t = np.loadtxt(path, dtype=str)
    return t[:, [0, 2]].astype(np.int32), t[:, 5].astype(np.float64)


def _assert_iteration_table(df, columns, values):
    assert list(df.columns) == columns and len(df) == len(values)
    keep = [k for k, c in enumerate(columns) if c != "time"]          # wall time differs from run to run
    assert np.allclose(df.to_numpy(dtype=np.float64)[:, keep], values[:, keep], rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("ignore_gaps", [True, False])
def test_reference_standard_protocol_over_our_run_plmc(golden, tmp_path, ignore_gaps):
    from evcouplings_b200 import synthetic, tools
    from cpu_engine import OracleEngine
    from oracle import plm_oracle as po
    N, L = 200, 40                      # BASELINE configs[0]
    codes = synthetic.synthetic_msa_codes(N, L, 1)
    synthetic.write_a2m(str(tmp_path / "cfg1.a2m"), codes)
    k = "std_%d_" % int(ignore_gaps)
    args, kwargs = _call(golden, k + "call", tmp_path)

    # the protocol handed run_plmc lambda_J already scaled by (q_eff - 1) * (L - 1)   (protocol.py:157-179)
    q_eff = 20 if ignore_gaps else 21
    assert abs(kwargs["lambda_J"] - 0.01 * (q_eff - 1) * (L - 1)) < 1e-12
    assert kwargs["focus_seq"] == "seq0/1-40" and kwargs["theta"] == 0.8 and kwargs["ignore_gaps"] == ignore_gaps
    res, run = tools.run_plmc(*args, engine=OracleEngine(), return_run=True, **kwargs)

    # stage outputs the protocol derived from the PlmcResult
    outcfg = _loads(golden[k + "outcfg"])
    assert outcfg["num_sites"] == res.num_valid_sites == L and outcfg["num_valid_sequences"] == res.num_valid_seqs == N
    assert abs(outcfg["effective_sequences"] - res.effective_samples) < 1e-9
    assert abs(outcfg["effective_sequences"] - run.n_eff) < 0.06 and outcfg["region_start"] == res.region_start == 1

    # the model file: what the reference's CouplingsModel read, and what is written now
    ref_model = _loads(golden[k + "model"])
    m = po.read_model(args[2])
    assert (m["L"], m["q"], m["n_valid"]) == (ref_model["L"], ref_model["num_symbols"], ref_model["N_valid"]) == (L, q_eff, N)
    assert "".join(m["alphabet"]) == ref_model["alphabet"] == ("ACDEFGHIKLMNPQRSTVWY" if ignore_gaps else "-ACDEFGHIKLMNPQRSTVWY")
    assert abs(m["theta"] - ref_model["theta"]) < 1e-7 and abs(m["n_eff"] - ref_model["N_eff"]) < 1e-3
    assert "".join(m["target_seq"]) == ref_model["target_seq"] == run.alignment.target_seq
    h = run.x[:L * q_eff].reshape(L, q_eff)
    J = run.x[L * q_eff:].reshape(-1, q_eff, q_eff)
    assert np.array_equal(m["h"], h) and np.array_equal(m["J"], J)
    assert np.allclose(h, golden[k + "h"], rtol=1e-5, atol=1e-6)
    sample = golden[k + "pair_index"]
    assert np.allclose(J[sample], golden[k + "J_upper"], rtol=1e-5, atol=1e-6)
    assert np.allclose(J[sample].transpose(0, 2, 1), golden[k + "J_lower"], rtol=1e-5, atol=1e-6)

    # the raw EC file as the reference's read_raw_ec_file read it
    ij, cn = _read_ecs(args[1])
    assert np.array_equal(ij, golden[k + "ec_ij"]) and len(cn) == L * (L - 1) // 2
    assert np.allclose(cn, golden[k + "ec_cn"], rtol=1e-4, atol=1e-6)
    assert np.abs(cn - po.cn_scores(J, L)).max() < 1e-6

    # the reference's log parser on the log written here
    it, fields = tools.parse_plmc_log(run.log)
    _assert_iteration_table(it, _loads(golden[k + "iter_columns"]), golden[k + "iter_values"])
    assert json.loads(json.dumps(list(fields), default=float)) == _loads(golden[k + "fields"])


def test_reference_parse_of_realistic_failure_modes(golden):
    """mandatory log lines: the reference raises KeyError without them (tools.py:97-99); ours too."""
    from evcouplings_b200 import tools
    assert str(golden["parse_failure"]) == "KeyError"
    with pytest.raises(KeyError):
        tools.parse_plmc_log("nothing useful")


def test_product_ingest_on_real_pabp_alignment(golden_dir, tmp_path):
    """product ingest of the real A2M shipped with the reference (PABP_YEAST: 151,496 valid + 545 invalid records)
    == the golden fixture, which the oracle's per-character restatement produced and plmc's own header / weights
    confirm.  A fixed sample of the file's records is stored (the focus record, every 200th record, every 20th
    invalid one); focus columns, validity and codes are per record, so the sample ingests to the same rows."""
    import lzma
    from evcouplings_b200 import msa
    s = golden_npz.load("pabp_a2m_sample")
    rows = s["rows"]
    path = tmp_path / "PABP_YEAST_sample.a2m"
    path.write_bytes(lzma.decompress(s["a2m_xz"].tobytes()))
    ali = msa.load_alignment(str(path), focus="PABP_YEAST", ignore_gaps=True)
    c = golden_npz.load("pabp_codes")
    valid = np.unpackbits(c["valid_packed"])[: int(c["n_total"])].astype(bool)
    assert (int(valid.sum()), int((~valid).sum())) == (151496, 545)
    vsel = valid[rows]
    assert vsel.sum() > 0 and (~vsel).sum() > 0
    rank = np.cumsum(valid) - 1                                   # row of a valid record in the golden codes
    assert np.array_equal(ali.valid, vsel) and np.array_equal(ali.codes, c["codes"][rank[rows[vsel]]])
    assert ali.target_seq == str(c["target_seq"]) and np.array_equal(ali.index_list, c["index_list"])
    assert (ali.n_valid, ali.n_total - ali.n_valid, ali.region_start, ali.num_total_sites) == \
        (int(vsel.sum()), int((~vsel).sum()), 115, 96)


def test_unmodified_reference_run_plmc_over_plmc_compatible_cli(golden, tmp_path):
    """Secondary plug point: the reference's OWN run_plmc (tools.py:126-307) drives the plmc-compatible executable
    with an argv it builds and scrapes stderr.  Stored: that argv and the PlmcResult the reference built from the
    log.  The same argv goes to the executable's entry point here (test-only oracle engine; bin/evcplm-plmc is the
    same entry point with the CUDA engine), and the log it writes must yield the same PlmcResult."""
    from evcouplings_b200 import plmc_cli, synthetic, tools
    from cpu_engine import OracleEngine
    from oracle import plm_oracle as po
    codes = synthetic.synthetic_msa_codes(150, 16, 3)
    synthetic.write_a2m(str(tmp_path / "in.a2m"), codes)
    argv = _paths(_loads(golden["cli_argv"]), tmp_path)
    ecs, model = argv[argv.index("-c") + 1], argv[argv.index("-o") + 1]
    os.makedirs(os.path.dirname(ecs), exist_ok=True)
    err = io.StringIO()
    assert plmc_cli.main(argv, engine=OracleEngine(), stderr=err) == 0
    it, fields = tools.parse_plmc_log(err.getvalue())
    res = tools.PlmcResult(ecs, model, it, *fields)
    ref = _loads(golden["cli_result"])
    for name, v in ref.items():
        if name in ("couplings_file", "param_file"):
            continue
        got = getattr(res, name)
        assert (abs(got - v) < 1e-9) if isinstance(v, float) else (got == v), (name, got, v)
    assert res.num_valid_seqs == 150 and res.num_total_seqs == 150 and res.num_valid_sites == 16
    assert res.focus_seq_index == 1 and res.region_start == 1
    assert res.optimization_status == "LBFGSERR_MAXIMUMITERATION" and len(res.iteration_table) == 12
    _assert_iteration_table(res.iteration_table, _loads(golden["cli_iter_columns"]), golden["cli_iter_values"])
    m = po.read_model(model)
    assert (m["L"], m["q"], m["num_iter"]) == (16, 20, 12) and abs(m["theta"] - 0.2) < 1e-6
    assert abs(m["lambda_J"] - 2.5) < 1e-6 and abs(res.effective_samples - m["n_eff"]) < 0.06
    assert len(open(ecs).read().strip().split("\n")) == 16 * 15 // 2


def test_plmc_cli_argument_handling():
    from evcouplings_b200 import plmc_cli
    ali, o = plmc_cli.parse_args(["-c", "e.txt", "-o", "m.model", "-f", "SEQ", "-g", "-m", "100", "-t", "0.2",
                                  "-lh", "0.01", "-le", "16.2", "-n", "4", "in.a2m"])
    assert ali == "in.a2m" and o["couplings_file"] == "e.txt" and o["param_file"] == "m.model"
    assert o["focus_seq"] == "SEQ" and o["ignore_gaps"] and o["iterations"] == 100
    assert abs(o["theta"] - 0.8) < 1e-12 and o["lambda_h"] == 0.01 and o["lambda_J"] == 16.2 and o["cpu"] == "4"
    import io
    for bad in (["-c"], ["in.a2m"], ["-c", "e", "a", "b"], ["-zz", "1", "-c", "e", "a"]):
        assert plmc_cli.main(bad, stderr=io.StringIO()) == 2
    err = io.StringIO()
    assert plmc_cli.main(["-c", "/tmp/e.txt", "/nonexistent/file.a2m"], stderr=err) == 1 and "ResourceError" in err.getvalue()


def test_reference_complex_protocol_over_our_run_plmc(golden, tmp_path):
    """BASELINE configs[4] flavour (EVcomplex concatenated two-chain alignment): the reference's ``complex``
    protocol (protocol.py:480-594; same infer_plmc -> run_plmc boundary, two segments, inter-chain EC table) over
    this run_plmc.  Stored: the run_plmc call it made, its stage outputs, and the inter-chain ECs it derived from
    the raw EC file written here.  Small shapes (2 x 12 sites); the engine itself is parity- and bench-tested at
    L=800 on the GPU."""
    from evcouplings_b200 import synthetic, tools
    from cpu_engine import OracleEngine
    from oracle import plm_oracle as po
    N, L1, L2 = 160, 12, 12
    L = L1 + L2
    codes = synthetic.synthetic_msa_codes(N, L, 8)
    synthetic.write_a2m(str(tmp_path / "complex.a2m"), codes, focus_name="A_B")   # "A_B/1-24" like complex/alignment.py:85-92
    args, kwargs = _call(golden, "cx_call", tmp_path)
    assert kwargs["focus_seq"] == "A_B/1-%d" % L and kwargs["ignore_gaps"]
    res = tools.run_plmc(*args, engine=OracleEngine(), **kwargs)
    outcfg = _loads(golden["cx_outcfg"])
    assert outcfg["num_sites"] == res.num_valid_sites == L and outcfg["num_valid_sequences"] == res.num_valid_seqs == N
    # inter-chain ECs: the protocol's table holds the cn of the L1 x L2 cross pairs of the raw EC file
    assert _loads(golden["cx_inter_segments"]) == [["A_1"], ["B_1"]]
    ij, cn = _read_ecs(args[1])
    cross = (ij[:, 0] <= L1) & (ij[:, 1] > L1)
    ref_cn = golden["cx_inter_cn"]
    assert cross.sum() == len(ref_cn) == L1 * L2
    assert np.allclose(np.sort(cn[cross]), np.sort(ref_cn), rtol=1e-4, atol=1e-6)
    assert {"i", "j", "segment_i", "segment_j", "cn", "probability"} <= set(_loads(golden["cx_ec_columns"]))
    m = po.read_model(args[2])
    ref_model = _loads(golden["cx_model"])
    assert (m["L"], m["q"]) == (ref_model["L"], ref_model["num_symbols"]) == (L, 20)
