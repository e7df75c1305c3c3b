"""
Drop-in boundary on the GPU (-m gpu): the reference's OWN couplings protocol and its OWN run_plmc over the CUDA
engine, replayed from what the unmodified reference did (tests/golden/reference_protocol.part*.npz, written by
tests/golden/make_golden.py over the oracle engine on the same inputs):

  1. primary plug point: evcouplings.couplings.protocol.run(protocol="standard") (protocol.py:363-429 ->
     infer_plmc :56-257) calls run_plmc with stored arguments; the same call goes to evcouplings_b200.run_plmc
     with the CudaEngine (default wgmma path), and what it writes is compared with what the reference's readers
     read from the oracle run and with the oracle engine driven by the same host logic;
  2. secondary plug point: the reference's run_plmc (tools.py:126-307) builds an argv for the plmc executable and
     parses its stderr; the stored argv goes to bin/evcplm-plmc, i.e. the real executable with the real engine,
     and the log it writes must yield the PlmcResult the reference built.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import golden_npz

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def golden():
    return golden_npz.load("reference_protocol")


@pytest.fixture(scope="module")
def engine():
    from evcouplings_b200.engine import CudaEngine
    return CudaEngine()


def _loads(a):
    return json.loads(str(a))


def _paths(v, tmp_path):
    if isinstance(v, str):
        return v.replace("{tmp}", str(tmp_path))
    if isinstance(v, list):
        return [_paths(x, tmp_path) for x in v]
    return v


@pytest.mark.parametrize("ignore_gaps", [True, False])
def test_reference_standard_protocol_over_cuda_engine(golden, engine, tmp_path, ignore_gaps):
    """BASELINE configs[0] (N=200, L=40) through the reference's stage driver, numerics on the GPU."""
    from evcouplings_b200 import synthetic, tools
    from cpu_engine import OracleEngine
    from oracle import plm_oracle as po
    N, L = 200, 40
    codes = synthetic.synthetic_msa_codes(N, L, 1)
    synthetic.write_a2m(str(tmp_path / "cfg1.a2m"), codes)
    k = "gpu_std_%d_" % int(ignore_gaps)
    call = _loads(golden[k + "call"])
    args = _paths(call["args"], tmp_path)
    kwargs = {a: _paths(v, tmp_path) for a, v in call["kwargs"].items()}
    for p in args[1:]:
        os.makedirs(os.path.dirname(p), exist_ok=True)
    q_eff = 20 if ignore_gaps else 21
    lam_J = 0.01 * (q_eff - 1) * (L - 1)
    assert abs(kwargs["lambda_J"] - lam_J) < 1e-12 and kwargs["iterations"] == 40     # protocol.py:157-179
    res, run = tools.run_plmc(*args, engine=engine, return_run=True, num_gpus=1, **kwargs)

    # stage outputs the protocol derived from the PlmcResult (neighbour counts are exact integers on the GPU)
    outcfg = _loads(golden[k + "outcfg"])
    assert outcfg["num_sites"] == res.num_valid_sites == L and outcfg["num_valid_sequences"] == res.num_valid_seqs == N
    assert outcfg["region_start"] == res.region_start == 1
    assert abs(outcfg["effective_sequences"] - res.effective_samples) < 1e-9
    assert abs(outcfg["effective_sequences"] - run.n_eff) < 0.06
    for p in args[1:]:
        assert os.path.getsize(p) > 0

    # the files the CUDA engine wrote: the reader sees exactly the parameters, with the reference's model header
    ref_model = _loads(golden[k + "model"])
    m = po.read_model(args[2])
    assert (m["L"], m["q"], m["n_valid"]) == (ref_model["L"], ref_model["num_symbols"], ref_model["N_valid"])
    assert "".join(m["alphabet"]) == ref_model["alphabet"] and "".join(m["target_seq"]) == ref_model["target_seq"]
    assert abs(m["theta"] - ref_model["theta"]) < 1e-7 and abs(m["n_eff"] - ref_model["N_eff"]) < 1e-3
    h = run.x[:L * q_eff].reshape(L, q_eff)
    J = run.x[L * q_eff:].reshape(-1, q_eff, q_eff)
    assert np.array_equal(m["h"], h) and np.array_equal(m["J"], J)
    t = np.loadtxt(args[1], dtype=str)
    ij, cn = t[:, [0, 2]].astype(np.int32), t[:, 5].astype(np.float64)
    assert np.array_equal(ij, golden[k + "ec_ij"]) and len(cn) == L * (L - 1) // 2
    assert np.abs(cn - po.cn_scores(J.astype(np.float64), L)).max() < 2e-6

    # the log: the reference's parser produced these fields and this table from the oracle run; the CUDA engine
    # runs the same L-BFGS, so the fields agree exactly and the objective trajectory to fp32 noise
    it, fields = tools.parse_plmc_log(run.log)
    assert json.loads(json.dumps(list(fields), default=float)) == _loads(golden[k + "fields"])
    assert fields[-1] == "LBFGSERR_MAXIMUMITERATION" and len(it) == 40
    cols = _loads(golden[k + "iter_columns"])
    assert list(it.columns) == cols
    f_ref = golden[k + "iter_values"][:, cols.index("fx")]
    f_gpu = it["fx"].astype(float).values
    assert np.abs(f_gpu - f_ref).max() <= 2e-5 * np.abs(f_ref).max()
    # EC scores: against what the reference read from the oracle run, and against the oracle engine now
    assert np.sqrt(np.mean((cn - golden[k + "ec_cn"]) ** 2)) < 2e-3
    r2, _ = tools.run_plmc(args[0], str(tmp_path / "c_ECs.txt"), str(tmp_path / "c.model"), focus_seq="seq0/1-40",
                           theta=0.8, ignore_gaps=ignore_gaps, iterations=40, lambda_h=0.01, lambda_J=lam_J,
                           engine=OracleEngine(), return_run=True)
    f2 = r2.iteration_table["fx"].astype(float).values
    assert np.abs(f_gpu - f2).max() <= 2e-5 * np.abs(f2).max()
    cn2 = np.loadtxt(str(tmp_path / "c_ECs.txt"), usecols=5)
    assert np.sqrt(np.mean((cn - cn2) ** 2)) < 2e-3


def test_unmodified_reference_run_plmc_over_real_executable(golden, tmp_path):
    """The argv the reference's run_plmc builds, run as a subprocess of bin/evcplm-plmc with the CUDA engine; the
    stderr it writes must parse into the PlmcResult the reference built, and the files it checks must exist."""
    from evcouplings_b200 import synthetic, tools
    from oracle import plm_oracle as po
    codes = synthetic.synthetic_msa_codes(300, 24, 3)
    synthetic.write_a2m(str(tmp_path / "in.a2m"), codes)
    argv = _paths(_loads(golden["gpu_cli_argv"]), tmp_path)
    ecs, model = argv[argv.index("-c") + 1], argv[argv.index("-o") + 1]
    os.makedirs(os.path.dirname(ecs), exist_ok=True)
    env = dict(os.environ, EVC_NUM_GPUS="1")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bin", "evcplm-plmc")] + argv, capture_output=True,
                       text=True, env=env, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    assert os.path.getsize(ecs) > 0 and os.path.getsize(model) > 0
    it, fields = tools.parse_plmc_log(p.stderr)
    res = tools.PlmcResult(ecs, model, it, *fields)
    for name, v in _loads(golden["gpu_cli_result"]).items():
        if name in ("couplings_file", "param_file"):
            continue
        got = getattr(res, name)
        assert (abs(got - v) < 1e-9) if isinstance(v, float) else (got == v), (name, got, v)
    assert res.num_valid_seqs == 300 and res.num_total_seqs == 300 and res.num_valid_sites == 24
    assert res.optimization_status == "LBFGSERR_MAXIMUMITERATION" and len(res.iteration_table) == 20
    m = po.read_model(model)
    assert (m["L"], m["q"], m["num_iter"]) == (24, 20, 20) and abs(m["lambda_J"] - 4.0) < 1e-6
    assert abs(res.effective_samples - m["n_eff"]) < 0.06
    fx = res.iteration_table["fx"].astype(float).values
    assert np.all(np.diff(fx) <= 1e-6 * np.abs(fx[:-1]))          # monotone descent
    cols = _loads(golden["gpu_cli_iter_columns"])
    f_ref = golden["gpu_cli_iter_values"][:, cols.index("fx")]
    assert np.abs(fx - f_ref).max() <= 2e-5 * np.abs(f_ref).max()
