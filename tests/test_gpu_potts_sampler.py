"""The device Gibbs sampler (evc_sampler_*, model_ops.PottsSampler, bin/evcplm-sample) against exact enumeration,
against its float64 restatement (oracle/potts_sampler.py) draw for draw, bit for bit against itself across call
splits, handles and chain counts, generatively on plmc's PABP model, and end to end on a planted model."""
import os
import subprocess
import sys

import numpy as np
import pytest

from evcouplings_b200 import model_io, model_ops, synthetic
from oracle import potts_sampler as ps
from test_potts_sampler_oracle import (PLANTED, PLANTED_SAMPLES, PLANTED_SWEEPS, PLANTED_SAMPLE_SEED,
                                       RECOVERY_FRACTION, check_against_enumeration, planted_recovery, small_model)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Pearson r of the sampled f_i against the stored f_i of plmc's PABP model: the float64 restatement reached 0.9921
# with these chains (2048 chains, seed 0, 100 sweeps from the uniform start); the bound leaves room for the draws the
# two decide differently and for their sampling noise.
PABP_PEARSON_MIN = 0.98


@pytest.fixture(scope="module")
def eng():
    from evcouplings_b200.engine import CudaEngine
    return CudaEngine()


def model_dict(h, J, alphabet=None):
    L, q = h.shape
    alphabet = alphabet or (synthetic.ALPHABET + "BJOUXZ12345")[:q]
    return dict(L=L, q=q, h=np.asarray(h, dtype=np.float32), J=np.asarray(J, dtype=np.float32), alphabet=alphabet,
                target_seq="".join(alphabet[(3 * i + 1) % q] for i in range(L)))


def dyadic_model(L, q, seed):
    """Fields N(0, 0.5) and couplings N(0, 0.05), rounded to multiples of 2^-10: every partial sum the device forms
    is then exact in fp32 (ps.z_error_bound), and only the softmax and the prefix sum can round."""
    rng = np.random.default_rng(seed)
    h = np.round(rng.normal(0, 0.5, (L, q)) * 1024) / 1024
    J = np.round(rng.normal(0, 0.05, (L * (L - 1) // 2, q, q)) * 1024) / 1024
    return h.astype(np.float32), J.astype(np.float32)


@pytest.mark.parametrize("L,q", [(4, 3), (3, 5)])
@pytest.mark.parametrize("beta", [0.0, 0.5, 1.0])
def test_exact_distribution(eng, L, q, beta):
    h, J = small_model(L, q, 10 * L + q)
    with model_ops.PottsSampler(model_dict(h, J), 131072, seed=11, engine=eng) as s:
        s.run(32, beta)
        codes = s.codes()
    check_against_enumeration(codes, h, J, beta)


@pytest.mark.parametrize("L,q,beta,alphabet", [(12, 2, 1.0, None), (12, 21, 1.0, None), (12, 32, 0.5, None),
                                                (64, 2, 1.0, None), (64, 21, 1.0, None), (64, 32, 1.0, None),
                                                (64, 20, 1.0, "ACDEFGHIKLMNPQRSTVWY")])
def test_against_restatement(eng, L, q, beta, alphabet):
    """Every chain's codes equal the restatement's after every sweep before the sweep of its first near-tie draw;
    the chains that leave the restatement are all flagged by it.  40 sweeps cross the refresh at t = 32."""
    h, J = dyadic_model(L, q, 1000 * L + q)
    z_err = ps.z_error_bound(h, J, L, q, bits=10)
    assert z_err == 0.0
    margin = ps.near_tie_margin(q, z_err, beta, ps.z_bound(h, J, L, q))
    n, sweeps, seed = 4096, 40, 77
    ref = ps.Sampler(h, J, seed, n, margin=margin)
    diverged = np.zeros(n, dtype=bool)
    compared = 0
    with model_ops.PottsSampler(model_dict(h, J, alphabet), n, seed=seed, engine=eng) as s:
        for t in range(sweeps):
            ch = s.run(1, beta)
            ref.run(1, beta)
            clean = (ref.first_tie < 0) | (ref.first_tie >= (t + 1) * L)
            same = np.all(s.codes() == ref.codes(), axis=1)
            assert same[clean].all(), (t, np.flatnonzero(clean & ~same)[:8])
            if clean.all():
                assert ch == ref.changes
            diverged |= ~same
            compared += int(clean.sum())
    flagged = ref.first_tie >= 0
    assert not (diverged & ~flagged).any()
    assert diverged.mean() <= flagged.mean()
    # the comparison has power: the restatement run on the CPU keeps 37 to 99 % of the chain-sweeps before the first
    # near-tie for these models
    assert compared >= n * sweeps // 8, (compared, flagged.mean())
    if alphabet is not None:
        seqs = model_ops.sample_sequences(model_dict(h, J, alphabet), 64, 3, seed=1, engine=eng)
        assert all(len(x) == L and set(x) <= set(alphabet) for x in seqs)


def test_reproducible_bit_for_bit(eng):
    h, J = dyadic_model(30, 21, 5)
    h = h * 3.1                       # not dyadic any more: fp32 rounding everywhere
    m = model_dict(h, J * 7.3)
    n = 4096
    with model_ops.PottsSampler(m, n, seed=9, engine=eng) as a, model_ops.PottsSampler(m, n, seed=9, engine=eng) as b:
        ca = a.run(13) + a.run(27)
        cb = b.run(40)
        assert ca == cb and np.array_equal(a.codes(), b.codes())
        whole = b.codes()
    parts = []
    for off in (0, 2048):
        with model_ops.PottsSampler(m, 2048, seed=9, chain_offset=off, engine=eng) as p:
            p.run(40)
            parts.append(p.codes())
    assert np.array_equal(np.concatenate(parts), whole)
    with model_ops.PottsSampler(m, 1000, seed=9, engine=eng) as few:
        few.run(40)
        assert np.array_equal(few.codes(), whole[:1000])
    with model_ops.PottsSampler(m, 7, seed=9, init="target", engine=eng) as t:
        tgt = model_ops.encode_sequences(m, [m["target_seq"]])[0]
        assert np.array_equal(t.codes(), np.repeat(tgt[None], 7, axis=0))
        assert t.run(0) == 0 and np.array_equal(t.codes(), np.repeat(tgt[None], 7, axis=0))
    init = np.random.default_rng(0).integers(0, 21, (5, 30)).astype(np.uint8)
    with model_ops.PottsSampler(m, 5, seed=9, init=init, engine=eng) as t:
        assert np.array_equal(t.codes(), init)


def test_pabp_generative_check(eng):
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import golden_npz
    g = golden_npz.load("pabp_golden")
    L, q = 82, 20
    m = dict(L=L, q=q, h=g["h"], J=g["J"], alphabet=str(g["alphabet"]), target_seq=str(g["target_seq"]))
    with model_ops.PottsSampler(m, 2048, seed=0, engine=eng) as s:
        s.run(100)
        codes = s.codes()
    fi = np.stack([np.bincount(codes[:, i], minlength=q) for i in range(L)]) / len(codes)
    r = np.corrcoef(fi.ravel(), g["fi"].ravel())[0, 1]
    assert r >= PABP_PEARSON_MIN, r


def test_planted_recovery_through_the_command_line(tmp_path):
    m = synthetic.planted_potts_model(**PLANTED)
    path = str(tmp_path / "planted.model")
    model_io.write_model_file(path, m["L"], m["q"], m["n_valid"], m["n_invalid"], m["num_iter"], m["theta"],
                              m["lambda_h"], m["lambda_J"], m["lambda_group"], m["n_eff"], m["alphabet"],
                              m["weights"], m["target_seq"], m["index_list"], m["fi"], m["h"], m["fij"], m["J"])
    a2m, ecs = str(tmp_path / "samples.a2m"), str(tmp_path / "planted_ECs.txt")
    subprocess.run([sys.executable, os.path.join(ROOT, "bin", "evcplm-sample"), path, "-n", str(PLANTED_SAMPLES),
                    "--sweeps", str(PLANTED_SWEEPS), "--seed", str(PLANTED_SAMPLE_SEED), "-o", a2m], check=True)
    with open(a2m) as f:
        lines = f.read().split("\n")
    assert len(lines) == 2 * PLANTED_SAMPLES + 1 and all(len(x) == m["L"] for x in lines[1::2])
    subprocess.run([sys.executable, os.path.join(ROOT, "bin", "evcplm-plmc"), "-c", ecs, a2m], check=True,
                   stderr=subprocess.DEVNULL)
    ec = np.loadtxt(ecs, usecols=(0, 2, 5))
    order = np.lexsort((ec[:, 1], ec[:, 0]))         # back to pair order i < j, row-major
    assert np.array_equal(ec[order, 0], np.triu_indices(m["L"], 1)[0] + 1)
    assert planted_recovery(ec[order, 2], m["L"], m["contacts"]) >= RECOVERY_FRACTION
