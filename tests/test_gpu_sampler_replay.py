"""Every Gibbs draw and every AIS weight of the device sampler (evc_sampler_run / _anneal / _set_model) on real and
non-dyadic models, against the teacher-forced fp32 replay of oracle/sampler_replay.py (-m gpu).

Each trajectory runs one sweep per call, so that the replay sees the codes after every sweep (and the log weights
after every annealed sweep); a second handle runs the same calls whole, and its codes and weights must be the same
bits.  For every case: no draw outside its near-tie band, log w bit-identical after every annealed sweep, each
call's changes_out equal to the replay's count, and at least 0.99 of the draws checked outside the band.  Probe
sweeps anneal([0, 1]) at t = 31 and t = 32 weigh H_J read off Z just before and just after the refresh at t = 32."""
import ctypes
import time

import numpy as np
import pytest

from oracle import ais, sampler_replay as sr
from test_gpu_boltzmann import pabp_model
from test_gpu_consumer_geometry import device_x, need_device
from test_sampler_geometry_oracle import (CTA2, FAR, FAR_SITES, chains_per_cta, cta2_model, far_model)

pytestmark = pytest.mark.gpu

CHECKED_MIN = 0.99


@pytest.fixture(scope="module")
def eng():
    from evcouplings_b200 import _lib
    from evcouplings_b200.engine import CudaEngine
    _lib.require_device()
    return CudaEngine()


class Device(object):
    """One evc_sampler handle on x (a device tensor), uniform start."""

    def __init__(self, eng, x, L, q, n, seed):
        import torch
        from evcouplings_b200 import _lib
        self.eng, self.L, self.q, self.n = eng, L, q, n
        torch.cuda.synchronize()
        self.handle = ctypes.c_void_p()
        _lib.check(eng.lib.evc_sampler_create(ctypes.byref(self.handle), eng.ptr(x), L, q, None, n, 0, seed,
                                              eng.device_index), "evc_sampler_create")
        self.logw = torch.zeros(n, dtype=torch.float64, device=eng.device)

    def run(self, sweeps, beta):
        from evcouplings_b200 import _lib
        ch = ctypes.c_int64()
        _lib.check(self.eng.lib.evc_sampler_run(self.handle, sweeps, float(beta), ctypes.byref(ch),
                                                self.eng.stream()), "evc_sampler_run")
        return int(ch.value)

    def anneal(self, betas):
        from evcouplings_b200 import _lib
        b = np.ascontiguousarray(betas, dtype=np.float32)
        ch = ctypes.c_int64()
        _lib.check(self.eng.lib.evc_sampler_anneal(self.handle, b.ctypes.data_as(ctypes.c_void_p), b.size - 1,
                                                   self.eng.ptr(self.logw), ctypes.byref(ch), self.eng.stream()),
                   "evc_sampler_anneal")
        return int(ch.value)

    def set_model(self, x):
        import torch
        from evcouplings_b200 import _lib
        _lib.check(self.eng.lib.evc_sampler_set_model(self.handle, self.eng.ptr(x), self.eng.stream()),
                   "evc_sampler_set_model")
        torch.cuda.synchronize()

    def codes(self):
        import torch
        out = torch.empty((self.n, self.L), dtype=torch.uint8, device=self.eng.device)
        assert self.eng.lib.evc_sampler_codes(self.handle, self.eng.ptr(out), self.eng.stream()) == 0
        return out.cpu().numpy()

    def weights(self):
        return self.logw.cpu().numpy()

    def close(self):
        if self.handle:
            self.eng.lib.evc_sampler_destroy(self.handle)
            self.handle = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


class Driven(object):
    """A device handle stepped one sweep per call with the replay following it."""

    def __init__(self, dev, rep):
        self.dev, self.rep = dev, rep
        self.device_s = 0.0

    def _timed(self, f, *a):
        t0 = time.time()
        out = f(*a)
        self.device_s += time.time() - t0
        return out

    def run(self, sweeps, beta):
        for _ in range(sweeps):
            ch = self._timed(self.dev.run, 1, beta)
            self.rep.run(1, beta, codes=self._timed(self.dev.codes)[None])
            assert ch == self.rep.call_changes[-1], (self.rep.t, ch, self.rep.call_changes[-1])

    def anneal(self, betas):
        betas = np.asarray(betas, dtype=np.float32)
        for k in range(len(betas) - 1):
            ch = self._timed(self.dev.anneal, betas[k:k + 2])
            codes, logw = self._timed(self.dev.codes), self._timed(self.dev.weights)
            self.rep.anneal(betas[k:k + 2], codes=codes[None], logw=logw[None])
            assert ch == self.rep.call_changes[-1], (self.rep.t, ch, self.rep.call_changes[-1])

    def reset_weights(self):
        self.dev.logw.zero_()
        self.rep.logw[:] = 0.0


def whole_calls(dev, calls):
    """The calls of a Driven trajectory, each as one device call: returns the total changes."""
    ch = 0
    for c in calls:
        if c[0] == "run":
            ch += dev.run(c[1], c[2])
        elif c[0] == "anneal":
            ch += dev.anneal(c[1])
        else:
            dev.logw.zero_()
    return ch


def drive(d, calls):
    for c in calls:
        if c[0] == "run":
            d.run(c[1], c[2])
        elif c[0] == "anneal":
            d.anneal(c[1])
        else:
            d.reset_weights()


def report(name, rep, t0, device_s):
    print("%s: %d draws over %d sweeps, checked %.6f outside the near-tie band, %d near ties, %d violations, "
          "%d sweeps with a log w mismatch; %.1f s in all, %.1f s on the device"
          % (name, rep.draws, rep.t, rep.checked_share(), rep.ties, rep.n_violations, len(rep.logw_mismatch),
             time.time() - t0, device_s))
    assert rep.n_violations == 0, (name, rep.violations[:8])
    assert not rep.logw_mismatch, (name, rep.logw_mismatch[:2])
    assert rep.checked_share() >= CHECKED_MIN, (name, rep.checked_share())


def x_of(h, J):
    return np.concatenate([np.ravel(h), np.ravel(J)]).astype(np.float32)


def check_case(eng, name, h, J, n, seed, calls, pairs=None, blocks=None, x=None):
    """Drives ``calls`` one sweep at a time on a handle with the replay following, then runs them whole on a second
    handle: the same codes, weights and change total."""
    import torch
    L, q = h.shape
    if x is None:
        x = torch.from_numpy(x_of(h, J)).to(eng.device)
    t0 = time.time()
    with Device(eng, x, L, q, n, seed) as dev, Device(eng, x, L, q, n, seed) as whole:
        start = dev.codes()
        rep = sr.Replay(h, None if pairs is not None else J, seed=seed, n_chains=n, init=start, pairs=pairs,
                        blocks=blocks)
        d = Driven(dev, rep)
        drive(d, calls)
        assert whole_calls(whole, calls) == sum(rep.call_changes)
        assert np.array_equal(whole.codes(), dev.codes())
        assert np.array_equal(whole.weights().view(np.uint64), dev.weights().view(np.uint64))
        assert np.array_equal(dev.codes(), rep.s)
        report(name, rep, t0, d.device_s)
    return rep


def probes():
    """Probe sweeps at t = 31 and t = 32 (the calls before them end at t = 30)."""
    return [("anneal", [0.0, 1.0]), ("anneal", [0.0, 1.0])]


# ---- plmc's PABP model ------------------------------------------------------------------------------------------

def test_pabp_plain_probes_and_ais(eng):
    """1024 chains: 31 sweeps at beta = 1 and 0.37, probes at t = 31 and 32, 7 more at 0.37; then the procedure of
    model_ops.log_partition with K = 32 and burn-in 8 (one sweep at beta = 0, the forward anneal, burn-in at beta =
    1, the reverse anneal), across the refreshes at t = 64 and 96."""
    m = pabp_model(eng)
    h, J = np.asarray(m["h"], dtype=np.float32), np.asarray(m["J"], dtype=np.float32)
    betas = ais.linear_schedule(32)
    calls = ([("run", 20, 1.0), ("run", 11, 0.37)] + probes() + [("run", 7, 0.37)] +
             [("reset",), ("anneal", [0.0, 0.0]), ("anneal", betas), ("reset",), ("run", 8, 1.0),
              ("anneal", betas[::-1])])
    rep = check_case(eng, "PABP", h, J, 1024, 11, calls)
    assert rep.t == 113 and (rep.logw != 0).all()


def test_pabp_boltzmann_updates(eng):
    """Two bmDCA updates of 10 sweeps each, driven through evc_sampler_run, evc_code_counts, evc_bm_update and
    evc_sampler_set_model with the replay following every sweep and both set_model calls; the final parameters equal
    BoltzmannLearner's for the same settings bit for bit."""
    import torch
    from evcouplings_b200 import _lib, model_ops
    m = pabp_model(eng)
    L, q, n, seed, eta, sweeps = 82, 20, 1024, 3, 0.05, 10
    lam2_h, lam2_J = model_ops.bm_regularisation(m)
    h, J = np.asarray(m["h"], dtype=np.float32), np.asarray(m["J"], dtype=np.float32)
    x = torch.from_numpy(x_of(h, J)).to(eng.device)
    f = torch.from_numpy(x_of(m["fi"], m["fij"])).to(eng.device)
    counts = torch.empty(x.numel(), dtype=torch.int32, device=eng.device)
    codes = torch.empty((n, L), dtype=torch.uint8, device=eng.device)
    stats = torch.zeros(2, dtype=torch.float64, device=eng.device)
    t0 = time.time()
    with Device(eng, x, L, q, n, seed) as dev:
        rep = sr.Replay(h, J, seed=seed, n_chains=n, init=dev.codes())
        d = Driven(dev, rep)
        for _ in range(2):
            d.run(sweeps, 1.0)
            assert eng.lib.evc_sampler_codes(dev.handle, eng.ptr(codes), eng.stream()) == 0
            _lib.check(eng.lib.evc_code_counts(eng.ptr(codes), n, L, q, eng.ptr(counts), eng.stream()),
                       "evc_code_counts")
            _lib.check(eng.lib.evc_bm_update(eng.ptr(x), eng.ptr(counts), n, eng.ptr(f), x.numel(), L * q, eta,
                                             lam2_h, lam2_J, eng.ptr(stats), eng.stream()), "evc_bm_update")
            dev.set_model(x)
            xh = x.cpu().numpy()
            rep.set_model(xh[:L * q].reshape(L, q), xh[L * q:].reshape(-1, q, q))
        d.run(2, 1.0)                                       # the sweep after set_model refreshes from the new model
        report("PABP bmDCA", rep, t0, d.device_s)
    with model_ops.BoltzmannLearner(m, n, seed=seed, learning_rate=eta, engine=eng) as learner:
        learner.run(2, sweeps)
        lh, lJ = learner.parameters()
    xh = x.cpu().numpy()
    assert np.array_equal(xh.view(np.uint32), x_of(lh, lJ).view(np.uint32))


# ---- a model fitted on the device ----------------------------------------------------------------------------------

def test_run_plmc_model(eng, tmp_path):
    """A model fitted by run_plmc on a synthetic L = 200, q = 21 alignment: 252 chains (13 per CTA, the last of 20
    CTAs holding 5), 36 sweeps with probes at t = 31 and 32."""
    from evcouplings_b200 import model_ops, synthetic, tools
    L, N = 200, 1500
    codes = synthetic.synthetic_msa_codes(N, L, 21)
    a2m = str(tmp_path / "a.a2m")
    synthetic.write_a2m(a2m, codes)
    path = str(tmp_path / "a.model")
    tools.run_plmc(a2m, str(tmp_path / "a_ECs.txt"), path, focus_seq="seq0/1-200", theta=0.8, iterations=30,
                   lambda_h=0.01, lambda_J=0.01 * 20 * (L - 1), num_gpus=1, engine=eng)
    m = model_ops.read_model(path)
    h, J = np.asarray(m["h"], dtype=np.float32), np.asarray(m["J"], dtype=np.float32)
    assert h.shape == (L, 21) and chains_per_cta(L, 21) == 13 and 252 % 13 == 5
    assert not np.all(np.round(J * 1024) == J * 1024)                  # not dyadic
    calls = [("run", 31, 1.0)] + probes() + [("run", 3, 1.0)]
    rep = check_case(eng, "run_plmc L=200", h, J, 252, 12, calls)
    assert rep.t == 36


# ---- random non-dyadic dense models at the lane edges --------------------------------------------------------------

@pytest.mark.parametrize("q", [2, 32])
def test_random_dense_models(eng, q):
    L, n = 64, 512
    rng = np.random.default_rng(q)
    h = (rng.normal(0, 0.5, (L, q)) * 1.0001).astype(np.float32)
    J = (rng.normal(0, 0.1, (L * (L - 1) // 2, q, q)) * 1.0001).astype(np.float32)
    calls = ([("run", 20, 1.0), ("run", 11, 0.37)] + probes() +
             [("anneal", np.float32([0.0, 0.1, 0.37, 0.8, 1.0])), ("run", 4, 1.0)])
    check_case(eng, "dense L=64 q=%d" % q, h, J, n, 13 + q, calls)


# ---- sparse non-dyadic models at the 2- and 1-chain-per-CTA geometries ---------------------------------------------

def nondyadic(model):
    h, pairs, blocks = model
    return (h * 1.0001).astype(np.float32), pairs, (blocks * 1.0001).astype(np.float32)


def test_sparse_two_chains_per_cta(eng):
    """L = 5000, q = 4, 81 chains (the last CTA holds one), 40 sweeps across the refresh with probes at t = 31, 32."""
    L, q, n = CTA2["L"], CTA2["q"], CTA2["n"]
    h, pairs, blocks = nondyadic(cta2_model())
    assert chains_per_cta(L, q) == 2 and n % 2 == 1
    lq = L * q
    need_device(eng, 4 * (2 * lq * lq + L * (L - 1) // 2 * q * q) + (1 << 30))
    calls = [("run", 31, 1.0)] + probes() + [("run", 7, 1.0)]
    x = device_x(eng, h, pairs, blocks)
    check_case(eng, "sparse L=5000 q=4", h, None, n, CTA2["seed"], calls, pairs=pairs, blocks=blocks, x=x)


def test_sparse_one_chain_per_cta_beyond_2_31(eng):
    """L = 2300, q = 21, 96 chains over 4 sweeps (a probe at t = 2): U has 2.33e9 entries and the rows of the last
    three coupled sites start beyond entry 2^31."""
    import torch
    L, q, n = FAR["L"], FAR["q"], FAR["n"]
    h, pairs, blocks = nondyadic(far_model())
    assert chains_per_cta(L, q) == 1 and all(i * q * L * q > 2 ** 31 for i in FAR_SITES[-3:])
    lq = L * q
    need_device(eng, 4 * (2 * lq * lq + L * (L - 1) // 2 * q * q + n * lq) + (2 << 30))
    calls = [("run", 2, 1.0), ("anneal", [0.0, 1.0]), ("run", 1, 1.0)]
    x = device_x(eng, h, pairs, blocks)
    rep = check_case(eng, "sparse L=2300 q=21", h, None, n, FAR["seed"], calls, pairs=pairs, blocks=blocks, x=x)
    del x
    torch.cuda.empty_cache()
    assert rep.t == 4
