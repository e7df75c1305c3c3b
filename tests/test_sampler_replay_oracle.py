"""The teacher-forced fp32 replay of the Gibbs sampler (oracle/sampler_replay.py) on the CPU: its generate mode
replays clean, on dyadic models it agrees with the float64 restatements (oracle/potts_sampler.py, oracle/ais.py) up to
their first near tie, and each of a list of plausible kernel mistakes, committed by generate mode, is caught by the
replay of the correct arithmetic within 256 chains x 40 sweeps.  The device side is tests/test_gpu_sampler_replay.py."""
import time

import numpy as np
import pytest

from oracle import ais, potts_sampler as ps, sampler_replay as sr
from test_sampler_geometry_oracle import dense_J, random_pairs


def random_model(L, q, seed, h_scale=0.5, j_scale=0.1, j_offset=0.0):
    """Non-dyadic float32 fields N(0, h_scale) and couplings N(0, j_scale) + j_offset / (L - 1)."""
    rng = np.random.default_rng(seed)
    h = (rng.normal(0, h_scale, (L, q)) * 1.0001).astype(np.float32)
    J = (rng.normal(0, j_scale, (L * (L - 1) // 2, q, q)) * 1.0001 + j_offset / (L - 1)).astype(np.float32)
    return h, J


def check_clean(r, what):
    assert r.n_violations == 0, (what, r.n_violations, r.violations[:4])
    assert not r.logw_mismatch, (what, r.logw_mismatch[:2])
    assert r.checked_share() >= 0.99, (what, r.checked_share())


@pytest.mark.parametrize("q", [2, 21, 32])
def test_generate_mode_replays_clean(q):
    """Split runs at two temperatures across the refresh at t = 32, a non-dyadic anneal in both directions, a
    set_model and the sweeps after it: zero violations, the same changes per call, and log w bit-identical."""
    L, C, seed = 24, 128, 40 + q
    h, J = random_model(L, q, q)
    h2, J2 = random_model(L, q, q + 1)
    g = sr.Replay(h, J, seed=seed, n_chains=C)
    start = g.s.copy()
    g.run(3, 1.0)
    g.run(9, 0.37)
    g.anneal(np.float32([0, 0.1, 0.37, 0.8, 1.0]))
    g.run(17, 1.0)                                       # t = 16 .. 32
    g.anneal(np.float32([1.0, 0.55, 0.0]))
    g.set_model(h2, J2)
    g.run(4, 1.0)
    g.anneal([0, 1])
    assert g.t == 40
    r = sr.replay_calls(sr.Replay(h, J, seed=seed, n_chains=C, init=start), g.calls)
    check_clean(r, q)
    assert r.call_changes == g.call_changes and np.array_equal(r.s, g.s)
    assert np.array_equal(r.logw.view(np.uint64), g.logw.view(np.uint64)) and (r.logw != 0).all()
    assert np.array_equal(r.Z.view(np.uint32), g.Z.view(np.uint32))
    print("q=%d: %d draws, checked %.6f, %d near ties" % (q, r.draws, r.checked_share(), r.ties))


def test_sparse_replay_equals_dense():
    """A model coupled on a few pairs, given as pairs and blocks, replays the trajectory generated from its dense J
    (zero outside the pairs) with the same fields Z bit for bit: the adds of zero rows leave fp32 values unchanged."""
    L, q, C = 40, 21, 64
    pairs = random_pairs(L, L, 9)
    rng = np.random.default_rng(4)
    h = (rng.normal(0, 0.5, (L, q)) * 1.0001).astype(np.float32)
    blocks = (rng.normal(0, 0.2, (len(pairs), q, q)) * 1.0001).astype(np.float32)
    J = dense_J(L, q, pairs, blocks).astype(np.float32)
    g = sr.Replay(h, J, seed=2, n_chains=C)
    start = g.s.copy()
    g.run(20, 1.0)
    g.anneal(np.float32([0, 0.3, 1.0]))
    g.run(11, 0.7)
    g.anneal([0, 1])
    r = sr.replay_calls(sr.Replay(h, seed=2, n_chains=C, init=start, pairs=pairs, blocks=blocks), g.calls)
    check_clean(r, "sparse")
    assert np.array_equal(r.Z.view(np.uint32), g.Z.view(np.uint32))
    assert np.array_equal(r.logw.view(np.uint64), g.logw.view(np.uint64))


@pytest.mark.parametrize("q", [2, 21, 32])
def test_generate_mode_equals_float64_restatement_on_dyadic_models(q):
    """On a dyadic model (Z exact in fp32) generate mode's codes equal oracle.potts_sampler.Sampler's, and its log
    weights oracle.ais.AnnealedSampler's bit for bit, for every chain before its first near tie there."""
    L, C, seed = 12, 512, 7
    rng = np.random.default_rng(q)
    h = (np.round(rng.normal(0, 0.5, (L, q)) * 1024) / 1024).astype(np.float32)
    J = (np.round(rng.normal(0, 0.1, (L * (L - 1) // 2, q, q)) * 1024) / 1024).astype(np.float32)
    assert ps.z_error_bound(h, J, L, q, bits=10) == 0.0
    B = ps.z_bound(h, J, L, q)
    g = sr.Replay(h, J, seed=seed, n_chains=C)
    ref = ps.Sampler(h, J, seed, C, margin=ps.near_tie_margin(q, 0.0, 1.0, B))
    compared = 0
    for t in range(40):                                  # across the refresh at t = 32
        g.run(1, 1.0)
        ref.run(1, 1.0)
        clean = (ref.first_tie < 0) | (ref.first_tie >= (t + 1) * L)
        assert np.array_equal(g.s[clean], ref.s[clean]), t
        compared += int(clean.sum())
    assert compared >= C * 40 // 2
    betas = ais.linear_schedule(16)
    a = sr.Replay(h, J, seed=seed + 1, n_chains=C)
    aref = ais.AnnealedSampler(h, J, seed + 1, C, margin=ais.annealed_near_tie_margin(q, 0.0, 1.0, B))
    for k in range(16):
        a.anneal(betas[k:k + 2])
        aref.anneal(betas[k:k + 2])
        clean = (aref.first_tie < 0) | (aref.first_tie >= (k + 1) * L)
        assert np.array_equal(a.s[clean], aref.s[clean]), k
        assert np.array_equal(a.logw[clean].view(np.uint64), aref.logw[clean].view(np.uint64)), k
    assert clean.mean() >= 0.5 and (a.logw != 0).all()


def mutation_model(mutation):
    """L = 24, q = 21, non-dyadic.  Fields shifted by 512, so that each fp32 rounding of Z is large, with one nearly
    free site (fields and couplings ~2^-40), whose H_J term needs the low bits of a double: the order of the H_J sum
    shows.  fma_logit moves one annealed logit in four by one ulp, and a draw can only show an ulp above the expf
    band (relative ~2e-6): its model has couplings that sum to about 16384 per site instead."""
    L, q = 24, 21
    if mutation == "fma_logit":
        return random_model(L, q, 1, j_offset=16384.0)
    h, J = random_model(L, q, 1)
    h += np.float32(512.0)
    h[3] *= np.float32(2.0 ** -49)
    iu, ju = np.triu_indices(L, 1)
    J[(iu == 3) | (ju == 3)] *= np.float32(2.0 ** -40)
    return h, J


def mutation_trajectory(r):
    """40 sweeps: plain runs at beta = 1 and 0.37 in calls of 5, a non-dyadic anneal up and down (beta - beta' is not
    exact in fp32 between betas a factor > 2 apart), and probe sweeps anneal([0, 1]) at t = 31 and 32, whose weight
    is H_J read off Z bit for bit on either side of the refresh at t = 32."""
    r.run(5, 1.0)
    r.run(5, 0.37)
    r.anneal(np.float32([0, 0.1, 0.37, 0.55, 0.8, 1.0]))
    r.anneal(np.float32([1.0, 0.8, 0.55, 0.37, 0.1, 0.0]))
    r.run(11, 1.0)
    r.anneal([0, 1])
    r.anneal([0, 1])
    r.run(7, 1.0)
    assert r.t == 40


def test_mutation_trajectory_replays_clean():
    for m in (None, "fma_logit"):
        h, J = mutation_model(m)
        g = sr.Replay(h, J, seed=5, n_chains=256)
        start = g.s.copy()
        mutation_trajectory(g)
        check_clean(sr.replay_calls(sr.Replay(h, J, seed=5, n_chains=256, init=start), g.calls), m)


@pytest.mark.parametrize("mutation", sr.MUTATIONS)
def test_mutation_is_caught(mutation):
    h, J = mutation_model(mutation)
    t0 = time.time()
    g = sr.Replay(h, J, seed=5, n_chains=256, mutation=mutation)
    start = g.s.copy()
    mutation_trajectory(g)
    r = sr.replay_calls(sr.Replay(h, J, seed=5, n_chains=256, init=start), g.calls)
    first_w = r.logw_mismatch[0][0] if r.logw_mismatch else None
    print("%s: caught: %d draw violations (first %s), log w differs from sweep %s on (%.1f s)"
          % (mutation, r.n_violations, r.violations[:1], first_w, time.time() - t0))
    assert not r.clean()
