"""Replica exchange on the device (evc_sampler_set_ladder / evc_sampler_temper, PottsSampler.set_ladder / temper,
sample_codes(ladder=), evcplm-sample --tempering/--ladder): the per-chain beta bit for bit against evc_sampler_run, the
float64 restatement (oracle/tempering.py) chain for chain and swap for swap, the exact rung distributions, the
Curie-Weiss modes, bit-identity over splits, handles, reruns and ranks, the refusals and the command line."""
import ctypes
import io
import os
import sys

import numpy as np
import pytest

from evcouplings_b200 import _lib, model_ops, sample_cli, synthetic
from oracle import conditional_sampler as cs, potts_sampler as ps, tempering as tp
from test_gpu_conditional_sampler import dyadic_model, model_dict, positions, write_model, masks_to_letters
from test_potts_sampler_oracle import small_model
from test_tempering_oracle import CW, CW_PLAIN_SWEEPS, check_against, curie_weiss_ladder

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# the restatement test compares every ladder with no near-tie draw or swap decision; its share of the ladders,
# fixed on the CPU with the restatement alone (0.118: near ties end most ladders within 13 sweeps)
COMPARED_SHARE = 0.11


@pytest.fixture(scope="module")
def eng():
    from evcouplings_b200.engine import CudaEngine
    return CudaEngine()


# 1. the tempered sweep at each chain's beta is the plain sweep at that beta, bit for bit (no swap round reached)
@pytest.mark.parametrize("L,q", [(12, 2), (12, 32), (64, 21), (200, 21), (200, 2)])
@pytest.mark.parametrize("conditional", [False, True])
def test_per_chain_beta_is_the_plain_sweep_bit_for_bit(eng, L, q, conditional):
    h, J = dyadic_model(L, q, 3 * L + q)
    m = model_dict(h * 3.1, J * 7.3)                  # not dyadic: fp32 rounding everywhere
    ladder = np.float32([0.5, 0.75, 1.0])
    R, G, sweeps = len(ladder), 101, 40
    free = range(1, L + 1) if conditional else None
    with model_ops.PottsSampler(m, G * R, seed=5, chain_offset=3 * R, engine=eng, free=free) as t:
        t.set_ladder(ladder, swap_interval=sweeps + 1)
        a = t.temper(13) + t.temper(27)               # across the refresh at t = 32
        codes = t.codes()
        assert np.array_equal(t.rungs(), np.tile(np.arange(R), G))
    for k in range(R):
        with model_ops.PottsSampler(m, G * R, seed=5, chain_offset=3 * R, engine=eng, free=free) as p:
            p.run(sweeps, float(ladder[k]))
            assert np.array_equal(p.codes()[k::R], codes[k::R]), k
    assert a > 0


def restatement_case(L, q, R, G, seed, interval, sweeps):
    """The restatement run one sweep at a time: per sweep, the ladders with no near-tie draw or swap decision so far
    (ok), their codes, rungs and the energies of the last round."""
    h, J = dyadic_model(L, q, 900 + L, scale=0.1)
    h = h * np.float32(0.25)                          # multiples of 2^-12: Z stays exact, and near ties rare
    assert ps.z_error_bound(h, J, L, q, bits=12) == 0.0
    ladder = np.float32(np.linspace(0.5, 1.0, R))
    zb = ps.site_z_bounds(h, J, L, q)
    base = ps.Sampler(h, J, seed, G * R, chain_offset=R * 7, margin=ps.near_tie_margin(q, 0.0, 1.0, zb))
    T = tp.Tempered(base, ladder, interval, seed, ladder_offset=7,
                    swap_margin=tp.swap_margin(L, float(zb.max()), 1.0))
    steps = []
    for _ in range(sweeps):
        T.run(1)
        ok = (T.ladder_first_tie() < 0) & (T.first_swap_tie < 0)
        steps.append((ok, base.codes().reshape(G, R, L).copy(), T.rung.copy(), np.array(T.energy).reshape(G, R)))
    return h, J, ladder, T, steps


# 2. chain for chain and swap for swap against the float64 restatement on a dyadic model, each ladder until its first
# near tie: 13 chains per CTA at L = 200, q = 21 with a partial last CTA, sweeps across the refresh at t = 32, swap
# rounds every 3 sweeps
def test_against_restatement(eng):
    L, q, R, G, seed, interval, sweeps = 200, 21, 4, 15, 8, 3, 40        # 60 chains: 4 CTAs of 13 and one of 8
    h, J, ladder, T, steps = restatement_case(L, q, R, G, seed, interval, sweeps)
    share = np.mean([ok.mean() for ok, _, _, _ in steps])
    assert share >= COMPARED_SHARE, share
    m = model_dict(h, J)
    with model_ops.PottsSampler(m, G * R, seed=seed, chain_offset=R * 7, engine=eng) as s:
        s.set_ladder(ladder, interval)
        for t, (ok, codes, rung, energy) in enumerate(steps):
            s.temper(1)
            assert np.array_equal(s.codes().reshape(G, R, L)[ok], codes[ok]), t
            assert np.array_equal(s.rungs().reshape(G, R)[ok], rung[ok]), t
            e = s.energies().reshape(G, R)
            assert np.abs(e[ok] - energy[ok]).max(initial=0.0) <= 1e-9 * np.abs(energy).max(), t
        stats = s.swap_statistics()
    assert np.array_equal(stats["attempted"], T.attempted)
    print("restatement: %.3f of the ladder-sweeps compared" % share)


# 3. 131 072 chains as ladders: every rung meets the enumeration bounds, plain and conditional with masks
@pytest.mark.parametrize("L,q", [(4, 3), (3, 5)])
def test_rungs_match_enumeration(eng, L, q):
    h, J = small_model(L, q, 10 * L + q)
    ladder = np.float32([0.25, 0.5, 0.75, 1.0])
    R, G = len(ladder), 131072 // 4
    with model_ops.PottsSampler(model_dict(h, J), G * R, seed=4, engine=eng) as s:
        s.set_ladder(ladder, 1)
        s.temper(64)
        for k in range(R):
            check_against(ps.state_index(s.rung_codes(k), q), ps.exact_distribution(h, J, float(ladder[k]), L, q))
        st = s.swap_statistics()
    assert np.all(st["attempted"] == G * 32) and np.all(st["accepted"] > 0)


def test_conditional_rungs_match_enumeration(eng):
    L, q = 6, 3
    h, J = small_model(L, q, 63)
    m = model_dict(h, J)
    free = np.array([1, 3, 4])
    allowed = [0b111, 0b101, 0b011]
    ladder = np.float32([0.5, 1.0, 1.5])
    R, G = len(ladder), 131072 // 3
    ctx = np.random.default_rng(2).integers(0, q, L)
    init = np.repeat(ctx[None], G * R, axis=0)
    with model_ops.PottsSampler(m, G * R, seed=6, init=init, engine=eng, free=positions(free),
                                allowed=masks_to_letters(m, free, allowed)) as s:
        s.set_ladder(ladder, 2)
        s.temper(64)
        for k in range(R):
            codes = s.rung_codes(k).astype(np.int64)
            assert np.array_equal(codes[:, cs.clamped_sites(L, free)], init[:G, cs.clamped_sites(L, free)])
            check_against(ps.state_index(codes[:, free], q), cs.exact_conditional(h, J, float(ladder[k]), free, ctx,
                                                                                  allowed))


# 4. the Curie-Weiss Potts model with the CPU-fixed parameters (test_tempering_oracle.CW)
def test_curie_weiss_modes(eng):
    L, q, K = CW["L"], CW["q"], CW["K"]
    h, J = tp.curie_weiss_model(L, q, K)
    m = model_dict(h, J)
    n = 16384
    zero = np.zeros((n, L), dtype=np.uint8)
    with model_ops.PottsSampler(m, n, seed=1, init=zero, engine=eng) as s:
        s.run(CW_PLAIN_SWEEPS, 1.0)
        plain = (tp.mode_of(s.codes(), q) == 0).mean()
    assert plain >= 0.99, plain
    ladder = curie_weiss_ladder()
    R, G = len(ladder), 16384
    with model_ops.PottsSampler(m, G * R, seed=2, init=np.zeros((G * R, L), dtype=np.uint8), engine=eng) as s:
        s.set_ladder(ladder, 1)
        s.temper(2000)
        freq = np.bincount(tp.mode_of(s.rung_codes(R - 1), q), minlength=q) / G
        st = s.swap_statistics()
    p = tp.curie_weiss_mode_probabilities(L, q, K, float(ladder[-1]))
    assert np.abs(freq - p).max() <= tp.mode_bound(p, G), (freq, p)
    print("curie-weiss: plain %.4f in mode 0; ladder modes %s; acceptance %s; round trips per ladder %.2f" %
          (plain, freq, np.round(st["acceptance"], 3), st["round_trips"].mean()))


def tempered_state(m, n, seed, offset, ladder, interval, calls, eng, **kw):
    with model_ops.PottsSampler(m, n, seed=seed, chain_offset=offset, engine=eng, **kw) as s:
        s.set_ladder(ladder, interval)
        ch = sum(s.temper(k) for k in calls)
        st = s.swap_statistics()
        return s.codes(), s.rungs(), s.energies(), st, ch


# 5. bit-identity: splits at and between swap rounds, two handles over ladder offsets, reruns
@pytest.mark.parametrize("conditional", [False, True])
def test_bit_identity(eng, conditional):
    m = synthetic.planted_potts_model(40, 21, 4, 6)
    ladder = model_ops.geometric_ladder(0.4, 1.5, 5)
    R, G, interval = len(ladder), 60, 4
    kw = dict(free=list(range(5, 30)), allowed={8: "ACDE"}) if conditional else {}
    init = "target" if conditional else "random"
    one = tempered_state(m, G * R, 3, 0, ladder, interval, [45], eng, init=init, **kw)
    for calls in ([4, 8, 33], [3, 5, 1, 36], [45]):          # at rounds, between rounds, a rerun
        got = tempered_state(m, G * R, 3, 0, ladder, interval, calls, eng, init=init, **kw)
        assert all(np.array_equal(a, b) for a, b in zip(one[:3], got[:3])) and one[4] == got[4]
        assert all(np.array_equal(one[3][k], got[3][k]) for k in ("attempted", "accepted", "round_trips"))
    a = tempered_state(m, 23 * R, 3, 0, ladder, interval, [20, 25], eng, init=init, **kw)
    b = tempered_state(m, 37 * R, 3, 23 * R, ladder, interval, [45], eng, init=init, **kw)
    assert np.array_equal(np.concatenate([a[0], b[0]]), one[0])
    assert np.array_equal(np.concatenate([a[1], b[1]]), one[1])
    assert np.array_equal(np.concatenate([a[2], b[2]]), one[2])
    assert np.array_equal(a[3]["accepted"] + b[3]["accepted"], one[3]["accepted"])
    assert np.array_equal(np.concatenate([a[3]["round_trips"], b[3]["round_trips"]]), one[3]["round_trips"])


# 6. the refusals of a tempered handle
def test_refusals(eng):
    m = synthetic.planted_potts_model(12, 21, 2, 4)
    lad = np.float32([0.5, 1.0, 2.0])
    with model_ops.PottsSampler(m, 10, engine=eng) as s:
        with pytest.raises(_lib.EngineError, match="multiple of R"):
            s.set_ladder(lad)
    with model_ops.PottsSampler(m, 9, chain_offset=4, engine=eng) as s:
        with pytest.raises(_lib.EngineError, match="chain_offset"):
            s.set_ladder(lad)
    with model_ops.PottsSampler(m, 9, engine=eng) as s:
        for bad in ([1.0], [0.5, 0.5, 1.0], [1.0, 0.5, 2.0], [-0.5, 0.5, 1.0], [0.5, np.nan, 1.0]):
            with pytest.raises(_lib.EngineError, match="R >= 2|strictly ascending"):
                s.set_ladder(bad)
        with pytest.raises(_lib.EngineError, match="swap_interval"):
            s.set_ladder(lad, 0)
        with pytest.raises(ValueError, match="set_ladder"):
            s.temper(1)
        s.set_ladder(lad, 2)
        s.set_ladder(lad, 2)                                      # the same ladder again: nothing happens
        with pytest.raises(_lib.EngineError, match="different ladder"):
            s.set_ladder(lad, 3)
        with pytest.raises(_lib.EngineError, match="tempered"):
            s.anneal([0.0, 0.5])
        dx = __import__("torch").from_numpy(model_ops.model_x(m)).to(eng.device)
        with pytest.raises(_lib.EngineError, match="tempered"):
            _lib.check(eng.lib.evc_sampler_set_model(s.handle, eng.ptr(dx), eng.stream()), "evc_sampler_set_model")
        s.temper(3)
        s.run(2, 1.0)                                             # legal, advances t
        s.temper(3)
        # 3 ladders; rounds 0 (pair 0), 2 (pair 0) and 3 (pair 1): round 1 fell in run()'s sweeps
        assert np.array_equal(s.swap_statistics()["attempted"], [6, 3])
    ctx = np.zeros((6, 12), dtype=np.uint8)
    ctx[4, 0] = 1                                                 # chain 4 of ladder 1 has another context
    with model_ops.PottsSampler(m, 6, init=ctx, free=list(range(3, 13)), engine=eng) as s:
        with pytest.raises(ValueError, match="different contexts"):
            s.set_ladder(lad)
        with pytest.raises(_lib.EngineError, match="different contexts"):        # the library's own check
            _lib.check(eng.lib.evc_sampler_set_ladder(s.handle, lad.ctypes.data_as(ctypes.c_void_p), 3, 1),
                       "evc_sampler_set_ladder")
    ctx[4, 0] = 0
    with model_ops.PottsSampler(m, 6, init=ctx, free=list(range(3, 13)), engine=eng) as s:
        s.set_ladder(lad)


# 7. ladders over 2 and 3 gloo ranks: Python and --gpus give the bits of one process
@pytest.mark.parametrize("R", [2, 3])
def test_ranks_write_the_bits_of_one_process(eng, tmp_path, R):
    m = synthetic.planted_potts_model(40, 21, 4, 6)
    ladder = model_ops.geometric_ladder(0.5, 2.0, 4)
    one, st1 = model_ops.sample_codes(m, 31, 9, seed=4, init="target", engine=eng, ladder=ladder, swap_interval=2,
                                      free=list(range(10, 25)), return_statistics=True)
    got, st = model_ops.sample_codes(m, 31, 9, seed=4, init="target", num_gpus=R, backend="gloo", ladder=ladder,
                                     swap_interval=2, free=list(range(10, 25)), return_statistics=True)
    assert np.array_equal(got, one)
    assert all(np.array_equal(st[k], st1[k]) for k in ("attempted", "accepted", "round_trips"))
    path = write_model(str(tmp_path / "m.model"), m)
    errs = {}
    for tag, extra in (("one", []), ("ranks", ["--gpus", str(R)])):
        err = io.StringIO()
        argv = [path, "-n", "31", "--sweeps", "9", "--seed", "4", "--tempering", "4", "--beta-min", "0.5", "--beta",
                "2", "--swap-interval", "2", "-o", str(tmp_path / (tag + ".a2m"))] + extra
        assert sample_cli.main(argv, stderr=err, backend="gloo") == 0, err.getvalue()
        errs[tag] = err.getvalue()
    with open(tmp_path / "one.a2m", "rb") as a, open(tmp_path / "ranks.a2m", "rb") as b:
        assert a.read() == b.read()
    assert errs["one"] == errs["ranks"] and "round trips" in errs["one"]


# 8. the command line redesigns a window of a planted model with a ladder and reports the swaps
def test_command_line_redesigns_a_window(tmp_path):
    import subprocess
    m = synthetic.planted_potts_model(60, 21, 6, 2)
    path = write_model(str(tmp_path / "m.model"), m)
    out = str(tmp_path / "design.a2m")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bin", "evcplm-sample"), path, "-n", "200", "--sweeps",
                        "40", "--free", "30-45", "--allow", "33:AVILM", "--init", "target", "--beta", "2",
                        "--tempering", "6", "--beta-min", "0.5", "--swap-interval", "2", "-o", out],
                       check=True, capture_output=True, text=True)
    assert r.stderr.count(" pair ") == 5 and "round trips" in r.stderr, r.stderr
    with open(out) as f:
        rows = f.read().split("\n")[1::2]
    assert len(rows) == 200
    tgt = m["target_seq"]
    for row in rows:
        assert len(row) == 60 and row[:29] == tgt[:29] and row[45:] == tgt[45:] and row[32] in "AVILM"
    assert len({row[29:45] for row in rows}) > 1


# 9. every draw and every swap decision of real models against the teacher-forced fp32 replay
# (oracle/tempered_replay.TemperedReplay): one sweep per call so that the replay sees the codes, rungs and energies
# after every sweep; a second handle runs the sweeps whole and must give the same bits
def tempered_replay_case(eng, name, m, n, seed, ladder, interval, sweeps):
    import time
    from oracle import tempered_replay as sr
    h, J = np.asarray(m["h"], dtype=np.float32), np.asarray(m["J"], dtype=np.float32)
    t0 = time.time()
    with model_ops.PottsSampler(m, n, seed=seed, engine=eng) as s, \
            model_ops.PottsSampler(m, n, seed=seed, engine=eng) as whole:
        rep = sr.TemperedReplay(h, J, seed=seed, n_chains=n, init=s.codes(), ladder=ladder, swap_interval=interval)
        s.set_ladder(ladder, interval)
        whole.set_ladder(ladder, interval)
        for _ in range(sweeps):
            ch = s.temper(1)
            rep.temper(1, codes=s.codes()[None], rungs=s.rungs()[None], energies=s.energies()[None])
            assert ch == rep.call_changes[-1]
        assert whole.temper(sweeps) == sum(rep.call_changes)
        for a, b in ((whole.codes(), s.codes()), (whole.rungs(), s.rungs()),
                     (whole.energies().view(np.uint64), s.energies().view(np.uint64))):
            assert np.array_equal(a, b)
        assert np.array_equal(s.codes(), rep.s)
        st = s.swap_statistics()
    print("%s: %d draws over %d sweeps, checked %.6f outside the near-tie band, %d near ties, %d violations; "
          "%d swap decisions, %d near ties, %d violations, %d energy mismatches; accepted %s of %s; %.1f s" %
          (name, rep.draws, rep.t, rep.checked_share(), rep.ties, rep.n_violations, rep.decisions, rep.swap_ties,
           rep.n_swap_violations, len(rep.energy_mismatch), st["accepted"], st["attempted"], time.time() - t0))
    assert rep.n_violations == 0, rep.violations[:4]
    assert not rep.energy_mismatch, rep.energy_mismatch[:1]
    assert rep.n_swap_violations == 0, rep.swap_violations[:4]
    assert rep.checked_share() >= 0.99
    assert np.array_equal(st["attempted"], rep.attempted) and np.array_equal(st["accepted"], rep.accepted)
    assert np.array_equal(st["round_trips"], rep.trips)
    return rep


def test_replay_pabp(eng):
    """plmc's PABP model (L = 82, q = 20): 256 ladders of 4 from beta = 0.5 to 1, a swap round after every sweep,
    40 sweeps across the refresh at t = 32."""
    from test_gpu_boltzmann import pabp_model
    m = pabp_model(eng)
    tempered_replay_case(eng, "PABP", m, 1024, 11, model_ops.geometric_ladder(0.5, 1.0, 4), 1, 40)


def test_replay_run_plmc_model(eng, tmp_path):
    """A model fitted by run_plmc on a synthetic L = 200, q = 21 alignment: 63 ladders of 4 (252 chains, 13 per CTA,
    the last of 20 CTAs holding 5), swap rounds every 3 sweeps, 36 sweeps across the refresh at t = 32."""
    from evcouplings_b200 import tools
    L, N = 200, 1500
    codes = synthetic.synthetic_msa_codes(N, L, 21)
    a2m = str(tmp_path / "a.a2m")
    synthetic.write_a2m(a2m, codes)
    path = str(tmp_path / "a.model")
    tools.run_plmc(a2m, str(tmp_path / "a_ECs.txt"), path, focus_seq="seq0/1-200", theta=0.8, iterations=30,
                   lambda_h=0.01, lambda_J=0.01 * 20 * (L - 1), num_gpus=1, engine=eng)
    m = model_ops.read_model(path)
    assert not np.all(np.round(m["J"] * 1024) == m["J"] * 1024)       # not dyadic
    tempered_replay_case(eng, "run_plmc L=200", m, 252, 12, model_ops.geometric_ladder(0.5, 1.0, 4), 3, 36)
