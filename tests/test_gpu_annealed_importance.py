"""Annealed importance sampling on the device (evc_sampler_anneal, model_ops.log_partition, bin/evcplm-logz): draw for
draw and weight for weight against the float64 restatement of oracle/ais.py, at the sampler's launch geometries, bit
for bit against itself over split schedules, chain offsets and reruns, and against exact log Z on the enumeration
models and at production size.  Every bound, chain count and comparison share is fixed on the CPU, in
tests/test_annealed_importance_oracle.py."""
import csv
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

from evcouplings_b200 import model_io, model_ops, synthetic
from oracle import ais, potts_sampler as ps
from test_annealed_importance_oracle import (CTA2, CTA13, DRAW, DRAW_CASES, DRAW_POWER, ENUM_DEVICE_CHAINS, ENUM_K,
                                             ENUM_MODELS, GEOMETRY_K, GEOMETRY_POWER, GEOMETRY_SWEEPS, N_SIGMA,
                                             PRODUCTION, PRODUCTION_MODELS, draw_margin, draw_model, exact_log_z,
                                             geometry_restatement, production_model, sweep_schedules, within)
from test_potts_sampler_oracle import small_model
from test_sampler_geometry_oracle import chains_per_cta, clean_after, cta2_model, cta13_model

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXTRA = (synthetic.ALPHABET + "BJOUXZ12345")

# PABP (plmc's model, tests/golden): oracle.ais.restated_log_weights (the procedure of model_ops.log_partition) with
# 512 chains, seed 0 and burn-in K gave these estimates and standard errors on the CPU (forward ESS 387 and 471,
# reverse 366 and 476; reverse - forward 0.012 and 0.022).  The device's estimates, with more chains and the same
# seed, must lie within N_SIGMA combined standard errors of them.
PABP_CPU = {256: dict(log_z=399.090436, stderr=0.0252, log_z_reverse=399.102340, stderr_reverse=0.0279),
            1024: dict(log_z=399.126158, stderr=0.0130, log_z_reverse=399.148554, stderr_reverse=0.0122)}
PABP_CHAINS = 16384


@pytest.fixture(scope="module")
def eng():
    from evcouplings_b200 import _lib
    from evcouplings_b200.engine import CudaEngine
    _lib.require_device()
    return CudaEngine()


def model_dict(h, J, alphabet=None):
    L, q = h.shape
    alphabet = alphabet or EXTRA[:q]
    return dict(L=L, q=q, h=np.asarray(h, dtype=np.float32), J=np.asarray(J, dtype=np.float32), alphabet=alphabet,
                target_seq="".join(alphabet[(3 * i + 1) % q] for i in range(L)))


def follow(dev, ref, schedules, n):
    """Runs both one schedule per call; after each, every chain clean so far has the restatement's codes and
    bit-identical log weight.  Returns (compared chain-sweeps per chain, diverged chains)."""
    compared = np.zeros(n, dtype=np.int64)
    diverged = np.zeros(n, dtype=bool)
    for t, b in enumerate(schedules):
        ch = dev.anneal(b)
        ref.anneal(b)
        clean = clean_after(ref, t)
        codes, logw = dev.codes(), dev.log_weights()
        same = np.all(codes == ref.codes(), axis=1)
        assert same[clean].all(), (t, np.flatnonzero(clean & ~same)[:8])
        bad = clean & (logw != ref.logw)
        assert not bad.any(), (t, np.flatnonzero(bad)[:8], logw[bad][:4], ref.logw[bad][:4])
        if clean.all():
            assert ch == ref.changes
        diverged |= ~same
        compared += clean
    assert not (diverged & (ref.first_tie < 0)).any()
    return compared, diverged


@pytest.mark.parametrize("L,q", DRAW_CASES)
def test_draw_for_draw(eng, L, q):
    h, J = draw_model(L, q, 1000 * L + q)
    n = DRAW["n"]
    ref = ais.AnnealedSampler(h, J, DRAW["seed"], n, margin=draw_margin(h, J))
    with model_ops.PottsSampler(model_dict(h, J), n, seed=DRAW["seed"], engine=eng) as dev:
        compared, _ = follow(dev, ref, sweep_schedules(DRAW["K"]), n)
    assert compared.sum() >= DRAW_POWER[(L, q)] * n * (DRAW["K"] + 1)


class _DeviceX(object):
    """A PottsSampler-like wrapper of evc_sampler_* on an x already on the device (sparse test models)."""

    def __init__(self, eng, x, L, q, n, seed):
        import torch
        from evcouplings_b200 import _lib
        self.eng, self.L, self.n, self._lib = eng, L, n, _lib
        torch.cuda.synchronize()
        self.handle = ctypes.c_void_p()
        _lib.check(eng.lib.evc_sampler_create(ctypes.byref(self.handle), eng.ptr(x), L, q, None, n, 0, seed,
                                              eng.device_index), "evc_sampler_create")
        self.logw = torch.zeros(n, dtype=torch.float64, device=eng.device)

    def anneal(self, b):
        b = np.ascontiguousarray(b, dtype=np.float32)
        ch = ctypes.c_int64()
        self._lib.check(self.eng.lib.evc_sampler_anneal(self.handle, b.ctypes.data_as(ctypes.c_void_p), b.size - 1,
                                                        self.eng.ptr(self.logw), ctypes.byref(ch), self.eng.stream()),
                        "evc_sampler_anneal")
        return int(ch.value)

    def codes(self):
        import torch
        out = torch.empty((self.n, self.L), dtype=torch.uint8, device=self.eng.device)
        assert self.eng.lib.evc_sampler_codes(self.handle, self.eng.ptr(out), self.eng.stream()) == 0
        return out.cpu().numpy()

    def log_weights(self):
        return self.logw.cpu().numpy()

    def close(self):
        if self.handle:
            self.eng.lib.evc_sampler_destroy(self.handle)
            self.handle = None


@pytest.mark.parametrize("name", ["CTA13", "CTA2"])
def test_geometry_draw_for_draw(eng, name):
    """13 chains per CTA with a partial last CTA (L = 200, q = 21) and 2 per CTA (L = 5000, q = 4), across the
    refresh at t = 32."""
    from test_gpu_consumer_geometry import device_x
    case = dict(CTA13=CTA13, CTA2=CTA2)[name]
    h, pairs, blocks = dict(CTA13=cta13_model, CTA2=cta2_model)[name]()
    L, q, n = case["L"], case["q"], case["n"]
    ref = geometry_restatement(name)
    dev = _DeviceX(eng, device_x(eng, h, pairs, blocks), L, q, n, case["seed"])
    try:
        compared, _ = follow(dev, ref, sweep_schedules(GEOMETRY_K, GEOMETRY_SWEEPS), n)
    finally:
        dev.close()
    assert compared.sum() >= GEOMETRY_POWER[name] * n * GEOMETRY_SWEEPS
    per_cta = chains_per_cta(L, q)
    assert (compared[-(n % per_cta):] > 0).any()            # the partial last CTA was compared
    assert (compared > ps.REFRESH).sum() >= 3


def test_bit_identity(eng):
    """A schedule split 16 + 48 against one call of 64, two handles over chain offsets against one, a rerun; then a
    plain run after the anneal still follows the restatement."""
    h, J = draw_model(30, 21, 5)
    m = model_dict(h * 3.1, J * 7.3)              # not dyadic: fp32 rounding everywhere
    b = ais.linear_schedule(64)
    n = 3000
    runs = []
    for split in (False, False, True):
        with model_ops.PottsSampler(m, n, seed=9, engine=eng) as s:
            s.anneal([0.0, 0.0])
            if split:
                s.anneal(b[:17])
                s.anneal(b[16:])
            else:
                s.anneal(b)
            runs.append((s.codes(), s.log_weights()))
    for codes, logw in runs[1:]:
        assert np.array_equal(codes, runs[0][0]) and np.array_equal(logw, runs[0][1])
    parts = []
    for off, cnt in ((0, 1234), (1234, n - 1234)):
        with model_ops.PottsSampler(m, cnt, seed=9, chain_offset=off, engine=eng) as p:
            p.anneal([0.0, 0.0])
            p.anneal(b)
            parts.append((p.codes(), p.log_weights()))
    assert np.array_equal(np.concatenate([c for c, _ in parts]), runs[0][0])
    assert np.array_equal(np.concatenate([w for _, w in parts]), runs[0][1])
    # a plain run after an anneal on the same handle (dyadic model: the restatement can follow it)
    h, J = draw_model(12, 21, 1000 * 12 + 21)
    ref = ais.AnnealedSampler(h, J, 4, 2048, margin=draw_margin(h, J))
    ref_plain = ps.near_tie_margin(21, 0.0, 1.0, ps.z_bound(h, J, 12, 21))
    with model_ops.PottsSampler(model_dict(h, J), 2048, seed=4, engine=eng) as s:
        for x in (s, ref):
            x.anneal([0.0, 0.0])
            x.anneal(ais.linear_schedule(16))
        assert np.array_equal(s.log_weights()[ref.first_tie < 0], ref.logw[ref.first_tie < 0])
        ref.margin = np.maximum(ref.margin, ref_plain)
        for t in range(17, 17 + 20):                 # sweeps 17..36 cross the refresh at t = 32
            ch = s.run(1)
            ref.run(1, 1.0)
            clean = clean_after(ref, t)
            assert np.all(s.codes() == ref.codes(), axis=1)[clean].all(), t
            if clean.all():
                assert ch == ref.changes
        assert clean.mean() > 0.5


def test_zero_couplings_give_zero_weights(eng):
    h, J = small_model(12, 21, 3)
    m = model_dict(h, np.zeros_like(J))
    r = model_ops.log_partition(m, 4096, 16, 8, seed=2, engine=eng)
    assert r["log_z"] == r["log_z0"] == r["log_z_reverse"] and r["ess"] == 4096 and r["stderr"] == 0.0
    with model_ops.PottsSampler(m, 1000, seed=1, engine=eng) as s:
        s.anneal(ais.linear_schedule(32))
        assert not s.log_weights().any()


@pytest.mark.parametrize("L,q", ENUM_MODELS)
def test_enumeration_models_exact(eng, L, q):
    h, J = small_model(L, q, 10 * L + q)
    exact = ais.log_z_enumeration(h, J)
    r = model_ops.log_partition(model_dict(h, J), ENUM_DEVICE_CHAINS, ENUM_K, ENUM_K, seed=3, engine=eng)
    print("L=%d q=%d: exact %.6f forward %.6f (se %.2e) reverse %.6f (se %.2e)"
          % (L, q, exact, r["log_z"], r["stderr"], r["log_z_reverse"], r["stderr_reverse"]))
    assert within(r["log_z"], exact, r["stderr"]) and within(r["log_z_reverse"], exact, r["stderr_reverse"])


@pytest.mark.parametrize("name", PRODUCTION_MODELS)
def test_production_size_exact(eng, name):
    m = production_model(name)
    exact = exact_log_z(m)
    r = model_ops.log_partition(m, engine=eng, **PRODUCTION)
    print("%s: exact %.6f forward %+.2e (se %.2e, ESS %.0f) reverse %+.2e (se %.2e, ESS %.0f)"
          % (name, exact, r["log_z"] - exact, r["stderr"], r["ess"], r["log_z_reverse"] - exact, r["stderr_reverse"],
             r["ess_reverse"]))
    assert within(r["log_z"], exact, r["stderr"]) and within(r["log_z_reverse"], exact, r["stderr_reverse"])


def test_pabp(eng):
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import golden_npz
    g = golden_npz.load("pabp_golden")
    m = dict(L=82, q=20, h=g["h"], J=g["J"], alphabet=str(g["alphabet"]), target_seq=str(g["target_seq"]))
    for K, cpu in sorted(PABP_CPU.items()):
        r = model_ops.log_partition(m, PABP_CHAINS, K, K, seed=0, engine=eng)
        print("PABP K=%d: forward %.6f (ESS %.0f, se %.2e) reverse %.6f (ESS %.0f, se %.2e) gap %.4f"
              % (K, r["log_z"], r["ess"], r["stderr"], r["log_z_reverse"], r["ess_reverse"], r["stderr_reverse"],
                 r["log_z_reverse"] - r["log_z"]))
        for key, se in (("log_z", "stderr"), ("log_z_reverse", "stderr_reverse")):
            assert abs(r[key] - cpu[key]) <= N_SIGMA * np.hypot(r[se], cpu[se]), (K, key, r[key], cpu[key])


def test_command_line(eng, tmp_path):
    m = synthetic.planted_potts_model(20, 20, 4, 3, alphabet="ACDEFGHIKLMNPQRSTVWY")     # no gap state
    path = str(tmp_path / "planted.model")
    model_io.write_model_file(path, m["L"], m["q"], m["n_valid"], m["n_invalid"], m["num_iter"], m["theta"],
                              m["lambda_h"], m["lambda_J"], m["lambda_group"], m["n_eff"], m["alphabet"],
                              m["weights"], m["target_seq"], m["index_list"], m["fi"], m["h"], m["fij"], m["J"])
    seqs = model_ops.sample_sequences(m, 300, 20, seed=1, engine=eng)
    gapped = {5, 77, 211}
    for k in gapped:
        seqs[k] = seqs[k][:3] + "-" + seqs[k][4:]
    a2m = str(tmp_path / "rows.a2m")
    with open(a2m, "w") as f:
        for k, s in enumerate(seqs):
            f.write(">row%d/1-%d\n%s\n" % (k, m["L"], s))
    out = str(tmp_path / "logp.csv")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bin", "evcplm-logz"), path, "--chains", "4096",
                        "--temperatures", "256", "--alignment", a2m, "--focus", "row0", "-o", out],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    print(p.stdout)
    fwd = [l for l in p.stdout.splitlines() if l.startswith("log Z forward")][0].split()
    log_z, se = float(fwd[3]), float(fwd[7])
    assert within(log_z, ais.log_z_disjoint_pairs(m["h"], m["J"], m["contacts"]), se)
    assert "skipped for symbols outside the model's states 3" in p.stdout
    with open(out) as f:
        rows = list(csv.reader(f))
    assert rows[0] == ["id", "log_p"] and len(rows) == 1 + 300 - len(gapped)
    keep = [k for k in range(300) if k not in gapped]
    assert [r[0] for r in rows[1:]] == ["row%d/1-%d" % (k, m["L"]) for k in keep]
    lib = model_ops.log_probabilities(m, [seqs[k] for k in keep], log_z, engine=eng)
    assert np.array_equal(np.array([float(r[1]) for r in rows[1:]]), lib)
