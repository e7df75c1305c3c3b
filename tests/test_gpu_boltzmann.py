"""Boltzmann-machine learning on the device (evc_code_counts, evc_bm_update, evc_sampler_set_model,
model_ops.BoltzmannLearner, bin/evcplm-bmdca): exact counts and bit-exact updates against oracle/boltzmann.py, the
sampler after set_model against its float64 restatement draw for draw, bit-identical split refinements, the
enumeration models against their exact optimum, plmc's PABP model and the command line end to end."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

from evcouplings_b200 import model_io, model_ops, synthetic
from oracle import boltzmann as bm, potts_sampler as ps
from test_boltzmann_oracle import (ENUM_CHAINS, ENUM_ETA, ENUM_MODELS, ENUM_SEED, ENUM_SWEEPS, ENUM_UPDATES,
                                   enum_bound, enum_model)
from test_gpu_potts_sampler import dyadic_model, model_dict
from test_potts_sampler_oracle import PLANTED, PLANTED_SAMPLES, PLANTED_SAMPLE_SEED, PLANTED_SWEEPS

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def eng():
    from evcouplings_b200.engine import CudaEngine
    return CudaEngine()


def device_counts(eng, codes, L, q):
    import torch
    d = torch.from_numpy(np.ascontiguousarray(codes, dtype=np.uint8)).to(eng.device)
    out = torch.full((L * q + L * (L - 1) // 2 * q * q,), -1, dtype=torch.int32, device=eng.device)
    rc = eng.lib.evc_code_counts(eng.ptr(d), len(codes), L, q, eng.ptr(out), eng.stream())
    assert rc == 0, eng.lib.evc_last_error()
    return out.cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("q", [2, 20, 21, 32])
@pytest.mark.parametrize("L", [2, 3, 82, 200])
def test_code_counts_exact(eng, L, q):
    rng = np.random.default_rng(L * 100 + q)
    N = 1237                                # not a multiple of any stage or tile
    codes = rng.integers(0, q, (N, L)).astype(np.uint8)
    codes[: N // 3, 0] = q - 1              # a skewed site: many increments of one counter
    got = device_counts(eng, codes, L, q)
    assert np.array_equal(got, bm.code_counts(codes, L, q))
    assert np.array_equal(device_counts(eng, codes[:1], L, q), bm.code_counts(codes[:1], L, q))
    a, b = device_counts(eng, codes[:500], L, q), device_counts(eng, codes[500:], L, q)
    assert np.array_equal(a + b, got)


@pytest.mark.parametrize("eta,lam2_h,lam2_J", [(0.05, 0.0, 0.0), (0.7, 0.002, 0.03), (0.0, 0.5, 1e-3)])
def test_bm_update_bit_exact(eng, eta, lam2_h, lam2_J):
    import torch
    rng = np.random.default_rng(int(eta * 100) + 7)
    n, Lq, M = 200003, 4100, 16384
    x = rng.normal(0, 1, n).astype(np.float32)
    c = rng.integers(0, M + 1, n).astype(np.uint32)
    f = (rng.integers(0, M + 1, n) / M + rng.normal(0, 1e-3, n)).astype(np.float32)
    want, st = bm.update(x, c, M, f, Lq, eta, lam2_h, lam2_J)
    dx = torch.from_numpy(x.copy()).to(eng.device)
    dc = torch.from_numpy(c.view(np.int32)).to(eng.device)
    df = torch.from_numpy(f).to(eng.device)
    ds = torch.full((2,), -1.0, dtype=torch.float64, device=eng.device)
    assert eng.lib.evc_bm_update(eng.ptr(dx), eng.ptr(dc), M, eng.ptr(df), n, Lq, eta, lam2_h, lam2_J, eng.ptr(ds),
                                 eng.stream()) == 0
    assert np.array_equal(dx.cpu().numpy().view(np.uint32), want.view(np.uint32))
    assert np.array_equal(ds.cpu().numpy(), st)


def set_model(s, eng, h, J):
    import torch
    dx = torch.from_numpy(np.concatenate([np.ravel(h), np.ravel(J)]).astype(np.float32)).to(eng.device)
    assert eng.lib.evc_sampler_set_model(s.handle, eng.ptr(dx), eng.stream()) == 0
    torch.cuda.synchronize()


def test_set_model_same_parameters_at_a_refresh_changes_nothing(eng):
    h, J = dyadic_model(30, 21, 5)
    m = model_dict(h * 3.1, J * 7.3)
    with model_ops.PottsSampler(m, 2048, seed=4, engine=eng) as a, \
            model_ops.PottsSampler(m, 2048, seed=4, engine=eng) as b:
        a.run(32)
        set_model(a, eng, m["h"], m["J"])
        ca = a.run(20)
        b.run(32)
        cb = b.run(20)
        assert ca == cb and np.array_equal(a.codes(), b.codes())


@pytest.mark.parametrize("L,q", [(12, 21), (64, 2), (64, 32)])
def test_set_model_follows_the_restatement(eng, L, q):
    """New parameters loaded at sweep 13 (not a refresh index): every chain still follows the restatement draw for
    draw until its first near-tie draw, across the refresh at t = 32."""
    h1, J1 = dyadic_model(L, q, 7 * L + q)
    h2, J2 = dyadic_model(L, q, 11 * L + q)
    z_err = max(ps.z_error_bound(h, J, L, q, bits=10) for h, J in ((h1, J1), (h2, J2)))
    assert z_err == 0.0
    margin = ps.near_tie_margin(q, z_err, 1.0, max(ps.z_bound(h1, J1, L, q), ps.z_bound(h2, J2, L, q)))
    n, seed = 4096, 21
    ref = bm.Sampler(h1, J1, seed, n, margin=margin)
    diverged = np.zeros(n, dtype=bool)
    compared = 0
    with model_ops.PottsSampler(model_dict(h1, J1), n, seed=seed, engine=eng) as s:
        for t in range(40):
            if t == 13:
                set_model(s, eng, h2, J2)
                ref.set_params(h2, J2)
            s.run(1)
            ref.run(1)
            clean = (ref.first_tie < 0) | (ref.first_tie >= (t + 1) * L)
            same = np.all(s.codes() == ref.codes(), axis=1)
            assert same[clean].all(), (t, np.flatnonzero(clean & ~same)[:8])
            diverged |= ~same
            compared += int(clean.sum())
    assert not (diverged & (ref.first_tie < 0)).any()
    assert compared >= n * 40 // 8


def test_split_runs_across_set_model(eng):
    h, J = dyadic_model(30, 21, 5)
    m = model_dict(h * 3.1, J * 7.3)
    h2, J2 = m["h"] * 0.7, m["J"] * 1.3
    with model_ops.PottsSampler(m, 2048, seed=8, engine=eng) as a, \
            model_ops.PottsSampler(m, 2048, seed=8, engine=eng) as b:
        a.run(13)
        set_model(a, eng, h2, J2)
        ca = a.run(27)
        b.run(13)
        set_model(b, eng, h2, J2)
        assert b.run(0) == 0
        cb = b.run(10) + b.run(17)
        assert ca == cb and np.array_equal(a.codes(), b.codes())


def test_learner_split_updates_are_bit_identical(eng):
    m = synthetic.planted_potts_model(20, 21, 4, 3)
    m.update(lambda_h=0.01, lambda_J=1.0, n_eff=3000.0,
             fi=np.random.default_rng(0).dirichlet(np.ones(21), 20).astype(np.float32))
    kw = dict(n_chains=3000, seed=5, learning_rate=0.3, burn_in=7, engine=eng)
    with model_ops.BoltzmannLearner(m, **kw) as a, model_ops.BoltzmannLearner(m, **kw) as b:
        a.run(3, sweeps=4).run(0).run(5, sweeps=4)
        trace = []
        b.run(8, sweeps=4, progress=lambda k, st: trace.append(k))
        assert trace == list(range(8)) and a.updates == b.updates == 8
        ha, Ja = a.parameters()
        hb, Jb = b.parameters()
        assert np.array_equal(ha.view(np.uint32), hb.view(np.uint32)) and np.array_equal(Ja, Jb)
        assert np.array_equal(a.sampler.codes(), b.sampler.codes())
    again = model_ops.boltzmann_refine(m, 8, sweeps=4, **kw)
    assert np.array_equal(again["h"], ha) and np.array_equal(again["J"], Ja) and again["num_iter"] == 8
    assert again["fij"] is m["fij"] and again["lambda_J"] == 1.0
    assert not np.array_equal(ha, m["h"])


@pytest.mark.parametrize("L,q", ENUM_MODELS)
def test_learner_reaches_the_optimum_of_enumeration_models(eng, L, q):
    m = enum_model(L, q)
    theta, bound = enum_bound(L, q)
    out = model_ops.boltzmann_refine(m, ENUM_UPDATES, n_chains=ENUM_CHAINS, sweeps=ENUM_SWEEPS, seed=ENUM_SEED,
                                     learning_rate=ENUM_ETA, engine=eng)
    err = np.abs(model_ops.model_x(out).astype(np.float64) - theta).max()
    assert err <= bound, (err, bound)


def pabp_model(eng):
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import golden_npz
    g = golden_npz.load("pabp_golden")
    c = golden_npz.load("pabp_codes")
    valid = np.unpackbits(c["valid_packed"])[: int(c["n_total"])].astype(bool)
    counts = c["golden_counts_all"][valid]
    w = (1.0 / counts).astype(np.float64)
    L, q = 82, 20
    lh, lj = float(g["hdr_f"][1]), float(g["hdr_f"][2])
    problem = eng.plm_problem(c["codes"], w.astype(np.float32), q, q, lh, lj)
    fi_c, fij_c = problem.weighted_counts()
    fi, fij = model_io.normalise_frequencies(fi_c, fij_c, w.sum(), True)
    return dict(L=L, q=q, n_valid=len(w), n_invalid=0, num_iter=0, theta=float(g["hdr_f"][0]), lambda_h=lh,
                lambda_J=lj, lambda_group=0.0, n_eff=float(w.sum()), alphabet=str(g["alphabet"]),
                weights=w.astype(np.float32), target_seq=str(g["target_seq"]), index_list=g["index_list"],
                fi=fi.astype(np.float32), h=g["h"], fij=fij.astype(np.float32), J=g["J"])


# PABP: 10 000 chains, 10 sweeps per update after 100 burn-in sweeps, the default learning rate, 60 updates
PABP_UPDATES = 60


def test_pabp_refinement_improves_pair_statistics(eng):
    m = pabp_model(eng)
    trace = []
    with model_ops.BoltzmannLearner(m, 10000, seed=0, burn_in=100, engine=eng) as learner:
        learner.run(PABP_UPDATES, progress=lambda k, st: trace.append(st))
    first, last = trace[0], trace[-1]
    print("PABP update 0: %s; update %d: %s" % (first, PABP_UPDATES - 1, last))
    assert last["connected_pearson"] > first["connected_pearson"], (first, last)
    assert last["max_coupling_dev"] < first["max_coupling_dev"], (first, last)


def test_planted_model_through_the_command_line(tmp_path):
    """evcplm-sample -> evcplm-plmc -> evcplm-bmdca: the refined model and ECs are written, keep the input's header
    and statistics, and equal the library's refinement of the same model bit for bit."""
    m = synthetic.planted_potts_model(**PLANTED)
    path = str(tmp_path / "planted.model")
    model_io.write_model_file(path, m["L"], m["q"], m["n_valid"], m["n_invalid"], m["num_iter"], m["theta"],
                              m["lambda_h"], m["lambda_J"], m["lambda_group"], m["n_eff"], m["alphabet"],
                              m["weights"], m["target_seq"], m["index_list"], m["fi"], m["h"], m["fij"], m["J"])
    a2m, plm, ecs0 = str(tmp_path / "s.a2m"), str(tmp_path / "plm.model"), str(tmp_path / "plm_ECs.txt")
    out, ecs = str(tmp_path / "bm.model"), str(tmp_path / "bm_ECs.txt")
    subprocess.run([sys.executable, os.path.join(ROOT, "bin", "evcplm-sample"), path, "-n", str(PLANTED_SAMPLES),
                    "--sweeps", str(PLANTED_SWEEPS), "--seed", str(PLANTED_SAMPLE_SEED), "-o", a2m], check=True)
    subprocess.run([sys.executable, os.path.join(ROOT, "bin", "evcplm-plmc"), "-c", ecs0, "-o", plm, a2m],
                   check=True, stderr=subprocess.DEVNULL)
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bin", "evcplm-bmdca"), plm, "--updates", "12",
                        "--chains", "2048", "--learning-rate", "0.5", "--burn-in", "20", "--seed", "3", "-o", out,
                        "-c", ecs], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    rows = [r for r in p.stderr.splitlines() if r.strip() and r.split()[0].isdigit()]
    assert [int(r.split()[0]) for r in rows] == list(range(12))
    start, got = model_ops.read_model(plm), model_ops.read_model(out)
    assert got["num_iter"] == 12
    for k in ("L", "q", "n_valid", "n_invalid", "theta", "lambda_h", "lambda_J", "n_eff", "alphabet", "target_seq"):
        assert got[k] == start[k], k
    for k in ("weights", "index_list", "fi", "fij"):
        assert np.array_equal(got[k], start[k]), k
    want = model_ops.boltzmann_refine(start, 12, n_chains=2048, learning_rate=0.5, burn_in=20, seed=3)
    assert np.array_equal(got["h"], want["h"]) and np.array_equal(got["J"], want["J"])
    assert not np.array_equal(got["J"], start["J"])
    ec = np.loadtxt(ecs, usecols=(0, 2, 5))
    assert len(ec) == m["L"] * (m["L"] - 1) // 2
    fn = np.sqrt((got["J"].astype(np.float64) ** 2).sum(axis=(1, 2)))
    assert np.allclose(ec[:, 2], model_io.apc_cn_scores(fn, m["L"]), atol=2e-6)
