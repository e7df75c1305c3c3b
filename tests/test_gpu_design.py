"""Design on the device (evc_sampler_record_best / _best / _descend, PottsSampler.record_best / best / descend,
model_ops.design_codes, evcplm-design): every descent decision, settled flag and record against the teacher-forced fp32
replay (oracle/design_replay.py), recording against no recording, splits, single-site optimality in float64, planted
and enumerated optima, conditional constraints, ranks and the command line."""
import io
import os
import subprocess
import sys

import numpy as np
import pytest

from evcouplings_b200 import design_cli, model_ops, synthetic
from oracle import conditional_sampler as cs, design as dz, design_replay as dr, potts_sampler as ps
from test_gpu_conditional_sampler import dyadic_model, model_dict, write_model

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def eng():
    from evcouplings_b200.engine import CudaEngine
    return CudaEngine()


def random_model(L, q, seed):
    h, J = dyadic_model(L, q, seed)
    return model_dict(h * 3.1, J * 7.3)               # not dyadic: fp32 rounding everywhere


def check_replay(name, rep):
    print("%s: %d descent decisions, %d draws (%d checked), %d descent violations, %d settled mismatches, "
          "%d record mismatches" % (name, rep.decisions_checked, rep.draws, rep.checked, rep.n_descent_violations,
                                    rep.settled_mismatch, len(rep.record_mismatch)))
    assert rep.n_descent_violations == 0, rep.descent_violations[:4]
    assert rep.settled_mismatch == 0
    assert not rep.record_mismatch, rep.record_mismatch[:1]
    assert rep.decisions_checked > 0
    assert rep.clean()


def drive(s, rep, sample, record_sweeps, descent_sweeps, beta):
    """One sweep per call on the device handle ``s``, the replay following each; the record checked after every
    sweep and the descent after each of its sweeps."""
    s.record_best()
    rep.record_best()
    for _ in range(record_sweeps):
        if sample == "temper":
            s.temper(1)
            rep.temper(1, codes=s.codes()[None], rungs=s.rungs()[None], energies=s.energies()[None])
        else:
            s.run(1, beta)
            rep.run(1, beta, codes=s.codes()[None])
        rep.best(*s.best())
    for _ in range(descent_sweeps):
        settled, _ch = s.descend(1)
        rep.descend(1, codes=s.codes()[None], settled=settled)
    rep.best(*s.best())


def plain_replay_case(eng, name, m, n, seed, record_sweeps=20, descent_sweeps=24, beta=1.5):
    h, J = np.asarray(m["h"], dtype=np.float32), np.asarray(m["J"], dtype=np.float32)
    with model_ops.PottsSampler(m, n, seed=seed, engine=eng) as s:
        rep = dr.DesignReplay(h, J, seed=seed, n_chains=n, init=s.codes())
        drive(s, rep, "run", record_sweeps, descent_sweeps, beta)
        final = s.codes()
    with model_ops.PottsSampler(m, n, seed=seed, engine=eng) as whole:       # the same calls, whole
        whole.record_best()
        whole.run(record_sweeps, beta)
        whole.descend(descent_sweeps)
        assert np.array_equal(whole.codes(), final)
        for a, b in zip(whole.best(), (rep.best_energy, rep.best_codes, rep.best_sweep)):
            assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
    check_replay(name, rep)


# 1. the replay checks every descent decision, settled flag and record
def test_replay_pabp(eng):
    from test_gpu_boltzmann import pabp_model
    plain_replay_case(eng, "PABP", pabp_model(eng), 512, 11)


def test_replay_run_plmc_model(eng, tmp_path):
    """L = 200, q = 21: 13 chains per CTA, 252 chains, the last of 20 CTAs holding 5."""
    from evcouplings_b200 import tools
    L, N = 200, 1500
    codes = synthetic.synthetic_msa_codes(N, L, 21)
    a2m = str(tmp_path / "a.a2m")
    synthetic.write_a2m(a2m, codes)
    path = str(tmp_path / "a.model")
    tools.run_plmc(a2m, str(tmp_path / "a_ECs.txt"), path, focus_seq="seq0/1-200", theta=0.8, iterations=30,
                   lambda_h=0.01, lambda_J=0.01 * 20 * (L - 1), num_gpus=1, engine=eng)
    m = model_ops.read_model(path)
    assert not np.all(np.round(m["J"] * 1024) == m["J"] * 1024)
    plain_replay_case(eng, "run_plmc L=200", m, 252, 12, record_sweeps=13, descent_sweeps=27)


@pytest.mark.parametrize("q", [2, 32])
def test_replay_random_models(eng, q):
    plain_replay_case(eng, "random L=64 q=%d" % q, random_model(64, q, 40 + q), 301, q, beta=2.0)


def test_replay_conditional_handle_with_masks(eng):
    L, q, n = 48, 21, 130
    m = random_model(L, q, 7)
    free = list(range(5, 30)) + [40]
    allowed = {6: "ACDEF", 12: "W", 40: "KLMN"}
    ctx = np.random.default_rng(3).integers(0, q, (n, L)).astype(np.uint8)
    with model_ops.PottsSampler(m, n, seed=9, init=ctx, engine=eng, free=positions(m, free),
                                allowed={int(m["index_list"][k]): v for k, v in allowed.items()}) as s:
        sites, masks = s.free_sites, model_ops.conditional_sites(
            m, positions(m, free), {int(m["index_list"][k]): v for k, v in allowed.items()}, ctx)[1]
        hc = s.conditional_fields()
        Jr = cs.reduced_couplings(m["J"], L, q, sites).reshape(len(sites), q, len(sites), q)
        iu, ju = np.triu_indices(len(sites), 1)
        rep = dr.DesignReplay(hc[0], Jr[iu, :, ju, :].astype(np.float32), seed=9, n_chains=n, hc=hc, free=sites,
                              context=ctx, allowed=masks)
        drive(s, rep, "run", 13, 27, 1.5)
        out = s.codes()
    check_replay("conditional", rep)
    clamped = np.setdiff1d(np.arange(L), sites)
    assert np.array_equal(out[:, clamped], ctx[:, clamped])


def test_replay_ladder_handle(eng):
    m = random_model(40, 21, 5)
    h, J = np.asarray(m["h"], dtype=np.float32), np.asarray(m["J"], dtype=np.float32)
    ladder = model_ops.geometric_ladder(0.5, 2.0, 4)
    with model_ops.PottsSampler(m, 4 * 50, seed=3, engine=eng) as s:
        rep = dr.TemperedDesignReplay(h, J, seed=3, n_chains=200, init=s.codes(), ladder=ladder, swap_interval=2)
        s.set_ladder(ladder, 2)
        drive(s, rep, "temper", 21, 20, None)
    check_replay("ladder", rep)
    assert rep.n_swap_violations == 0


def positions(m, sites):
    return [int(m["index_list"][k]) for k in sites]


# 2. recording leaves the chain as it is; a record and a descent split over calls are one call
@pytest.mark.parametrize("conditional", [False, True])
def test_recording_changes_nothing_and_splits_are_one_call(eng, conditional):
    m = random_model(64, 21, 17)
    free = positions(m, range(64)) if conditional else None
    runs = {}
    for rec in (False, True):
        with model_ops.PottsSampler(m, 333, seed=2, engine=eng, free=free) as s:
            if rec:
                s.record_best()
            ch = [s.run(13, 1.3), s.run(27, 1.3), s.run(9, 1.3)]      # across the refresh at t = 32
            runs[rec] = (s.codes(), ch)
    assert np.array_equal(runs[False][0], runs[True][0]) and runs[False][1] == runs[True][1]
    outs = []
    for split in ((40,), (13, 27)):
        with model_ops.PottsSampler(m, 333, seed=2, engine=eng, free=free) as s:
            s.record_best()
            for k in split:
                s.run(k, 1.3)
            best = s.best()
            d = [s.descend(k) for k in split]
            outs.append((best, s.codes(), d[-1][0], sum(x[1] for x in d)))
    (b1, c1, s1, n1), (b2, c2, s2, n2) = outs
    assert all(np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8)) for a, b in zip(b1, b2))
    assert np.array_equal(c1, c2) and np.array_equal(s1, s2) and n1 == n2


# 3. outputs are single-site optima in float64 within the fp32 bound; descent from the target does not lose
def test_outputs_are_local_optima_and_descent_from_target_keeps_h(eng):
    m = random_model(30, 8, 23)
    h, J = np.asarray(m["h"], dtype=np.float64), np.asarray(m["J"], dtype=np.float64)
    bound = 2 * ps.z_error_bound(h, J, 30, 8)
    res = model_ops.design_codes(m, 200, 50, seed=1, beta_start=0.2, beta=3.0, engine=eng)
    assert res["settled"].all()
    assert (dz.single_site_gains(h, J, res["codes"]).max(axis=(1, 2)) <= bound).all()
    assert np.array_equal(res["energy"], model_ops.hamiltonians(m, res["codes"], eng)[:, 0])
    assert (res["found_at"] >= 0).all() and (res["found_at"] < 50).all()
    tgt = model_ops.hamiltonians(m, [m["target_seq"]], eng)[0, 0]
    res = model_ops.design_codes(m, 8, 0, init="target", engine=eng)
    assert (res["energy"] >= tgt - bound).all() and res["settled"].all()


# 4. a planted unique optimum is recovered by every chain; enumerated models reach the global maximum
def test_planted_unique_optimum(eng):
    L, q = 50, 21
    rng = np.random.default_rng(4)
    star = rng.integers(0, q, L)
    h = rng.normal(0, 0.1, (L, q)).astype(np.float32)
    h[np.arange(L), star] += 3.0
    J = rng.normal(0, 0.01, (L * (L - 1) // 2, q, q)).astype(np.float32)
    m = model_dict(h, J)
    res = model_ops.design_codes(m, 256, 10, seed=5, engine=eng)
    assert (res["codes"] == star[None, :]).all() and res["settled"].all()


@pytest.mark.parametrize("L, q", [(8, 3), (6, 4)])
def test_enumerated_global_maximum(eng, L, q):
    m = random_model(L, q, 100 + L)
    Hmax, _ = dz.global_max(m["h"], m["J"])
    res = model_ops.design_codes(m, 64, 100, seed=3, beta_start=0.2, beta=4.0, engine=eng)
    assert abs(res["energy"].max() - Hmax) <= 1e-5
    assert dz.is_local_max(m["h"], m["J"], res["codes"], tol=1e-5).all()


# 5. conditional outputs keep their context and use only allowed letters, even against the unrestricted argmax
def test_conditional_constraints(eng):
    L, q = 40, 21
    rng = np.random.default_rng(8)
    h = rng.normal(0, 0.1, (L, q)).astype(np.float32)
    h[12, 5] = 4.0                                    # the unrestricted argmax of site 12, forbidden below
    J = rng.normal(0, 0.02, (L * (L - 1) // 2, q, q)).astype(np.float32)
    m = model_dict(h, J)
    alphabet = m["alphabet"]
    free = positions(m, range(10, 20))
    allowed = {free[2]: alphabet[:5] + alphabet[6:9], free[4]: alphabet[3]}
    res = model_ops.design_codes(m, 100, 30, seed=2, init="target", free=free, allowed=allowed, engine=eng,
                                 ladder=[0.5, 1.0, 2.0])
    tgt = model_ops.encode_sequences(m, [m["target_seq"]])[0]
    clamped = np.r_[0:10, 20:L]
    assert (res["codes"][:, clamped] == tgt[clamped]).all()
    assert (res["codes"][:, 12] != 5).all() and np.isin(res["codes"][:, 12], [0, 1, 2, 3, 4, 6, 7, 8]).all()
    assert (res["codes"][:, 14] == 3).all() and res["settled"].all()
    assert "swap_statistics" in res


# 6. 2 and 3 gloo ranks sharing device 0: Python and --gpus give the bits of one process
@pytest.mark.parametrize("R", [2, 3])
def test_ranks_give_the_bits_of_one_process(eng, tmp_path, R):
    m = synthetic.planted_potts_model(40, 21, 4, 6)
    kw = dict(seed=4, init="target", free=list(range(10, 25)), descent_sweeps=64)
    for extra in (dict(beta_start=0.3, beta=2.0), dict(ladder=model_ops.geometric_ladder(0.5, 2.0, 4),
                                                       swap_interval=2)):
        one = model_ops.design_codes(m, 31, 9, engine=eng, **kw, **extra)
        got = model_ops.design_codes(m, 31, 9, num_gpus=R, backend="gloo", **kw, **extra)
        for k in ("codes", "energy", "settled", "found_at"):
            assert np.array_equal(np.asarray(got[k]).view(np.uint8), np.asarray(one[k]).view(np.uint8)), k
    path = write_model(str(tmp_path / "m.model"), m)
    for tag, extra in (("one", []), ("ranks", ["--gpus", str(R)])):
        err = io.StringIO()
        argv = [path, "-n", "31", "--sweeps", "9", "--seed", "4", "--anneal", "0.3", "--beta", "2", "-o",
                str(tmp_path / (tag + ".fasta"))] + extra
        assert design_cli.main(argv, stderr=err, backend="gloo") == 0, err.getvalue()
    with open(tmp_path / "one.fasta", "rb") as a, open(tmp_path / "ranks.fasta", "rb") as b:
        assert a.read() == b.read()


# 7. the command line redesigns a window of a planted model; the headers' H is hamiltonians()
def test_command_line_redesigns_a_window(tmp_path):
    m = synthetic.planted_potts_model(60, 21, 6, 2)
    path = write_model(str(tmp_path / "m.model"), m)
    out = str(tmp_path / "design.fasta")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bin", "evcplm-design"), path, "-n", "50", "--sweeps",
                        "40", "--free", "30-45", "--allow", "33:AVILM", "--init", "target", "--tempering", "4",
                        "--beta-min", "0.5", "--beta", "2", "-o", out], check=True, capture_output=True, text=True)
    assert "best H" in r.stderr and "round trips" in r.stderr, r.stderr
    with open(out) as f:
        lines = f.read().split("\n")
    heads, rows = lines[0::2][:50], lines[1::2][:50]
    tgt = m["target_seq"]
    for row in rows:
        assert len(row) == 60 and row[:29] == tgt[:29] and row[45:] == tgt[45:] and row[32] in "AVILM"
    H = model_ops.hamiltonians(m, rows)[:, 0]
    for k, head in enumerate(heads):
        assert head.startswith(">design_%d H=%.6f settled=" % (k, H[k])), head
