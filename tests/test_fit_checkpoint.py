"""
Checkpoint / resume of the L-BFGS fit on the CPU: the Python driver's state machine with the oracle problem, the
checkpoint file (atomic write, fingerprint, checksums, disk space), run_plmc's iteration table across resumes, and
the multi-rank plumbing (gloo ranks through the launcher, a worker stopped by SIGTERM).
"""
import json
import os
import signal
import subprocess
import sys
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from cpu_engine import OracleEngine, OracleProblem, ShardedOracleEngine, ShardedOracleProblem  # noqa: E402
from evcouplings_b200 import checkpoint, lbfgs, synthetic, tools  # noqa: E402


class _CheckpointSpace(object):
    """What a checkpointed fit needs from the oracle problem beyond the vector-space protocol."""
    evaluations_total = 0
    stop_at = None              # request a stop once the progress callback has seen this iteration
    sleep_s = 0.0

    def evaluate(self, x):
        type(self).evaluations_total += 1
        if self.sleep_s:
            time.sleep(self.sleep_s)
        if isinstance(self, ShardedOracleProblem):
            return super().evaluate(x)
        # one thread: the oracle's OpenMP reduction order, and so its last bit, changes from call to call otherwise
        from oracle import c_oracle as co
        fx, g, nll = co.plm_eval(self.codes, self.w, x, self.q, self.lambda_h, self.lambda_J,
                                 precision=self.precision, nthreads=1)
        self.g[:] = g
        self.last_negloglk = nll
        self.evaluations += 1
        return fx

    def get_history_scalars(self):
        return list(self.ys), self.yy

    def set_history_scalars(self, ys, yy):
        self.ys[:] = ys
        self.yy = yy

    def data_digest(self):
        return checkpoint.data_digest(self.codes, self.w.astype(np.float32))

    def fit(self, x0, params, progress=None, checkpoint=None, checkpoint_interval=900.0):
        stop_at = type(self).stop_at

        def prog(k, *a):
            out = progress(k, *a) if progress is not None else False
            if stop_at is not None and k >= stop_at:
                globals()["checkpoint"].request_stop()
            return out
        if checkpoint is None:
            return super().fit(x0, params, prog)
        ck = checkpoint if isinstance(checkpoint, globals()["checkpoint"].CheckpointFile) else \
            globals()["checkpoint"].CheckpointFile(checkpoint, checkpoint_interval)
        self.x[:] = x0
        ckm = globals()["checkpoint"]
        return ckm.fit_python(self, params, prog, ck, ckm.fingerprint(self, params, ck.extra),
                              engine=getattr(self, "engine", None))


class CkOracleProblem(_CheckpointSpace, OracleProblem):
    pass


class CkOracleEngine(OracleEngine):
    def plm_problem(self, codes, weights, q, gap_code, lambda_h, lambda_J, m=6):
        return CkOracleProblem(codes, weights, q, gap_code, lambda_h, lambda_J, m, self.precision)


class CkShardedProblem(_CheckpointSpace, ShardedOracleProblem):
    pass


class CkShardedEngine(ShardedOracleEngine):
    def plm_problem(self, codes, weights, q, gap_code, lambda_h, lambda_J, m=6):
        return CkShardedProblem(self, codes, weights, q, gap_code, lambda_h, lambda_J, m, self.precision)


class SlowOracleProblem(CkOracleProblem):
    sleep_s = 0.05


class SlowOracleEngine(OracleEngine):
    """CkOracleEngine with a pause per evaluation, so that a test can signal a worker in the middle of its fit."""

    def plm_problem(self, codes, weights, q, gap_code, lambda_h, lambda_J, m=6):
        return SlowOracleProblem(codes, weights, q, gap_code, lambda_h, lambda_J, m, self.precision)


@pytest.fixture(autouse=True)
def _clean_stop():
    checkpoint._stop["requested"] = False
    CkOracleProblem.stop_at = None
    yield
    checkpoint._stop["requested"] = False
    CkOracleProblem.stop_at = None


def _problem(m=6):
    from oracle import c_oracle as co
    from oracle import plm_oracle as po
    codes = po.synthetic_msa_codes(160, 8, 3)
    w = (1.0 / co.hamming_counts(codes, po.identity_threshold_count(0.8, 8))).astype(np.float32)
    return CkOracleProblem(codes, w.astype(np.float64), 21, -1, 0.01, 0.3, m=m)


# ---- the Python driver ----------------------------------------------------------------------------------------------
def test_python_driver_cancel_and_resume_is_bit_identical(tmp_path):
    params = lbfgs.default_params(max_iterations=25, epsilon=1e-9)
    ref = _problem()
    r0 = ref.fit(np.zeros(ref.n), params)
    assert r0.status == lbfgs.LBFGSERR_MAXIMUMITERATION and r0.iterations == 25
    path = str(tmp_path / "fit.ckpt")
    CkOracleProblem.stop_at = 9
    a = _problem()
    r1 = a.fit(np.zeros(a.n), params, checkpoint=path, checkpoint_interval=-1)
    assert r1.status == lbfgs.LBFGSERR_CANCELED and r1.iterations == 9
    hdr = checkpoint.CheckpointFile(path).read_header()
    assert hdr["state"]["k"] == 9 and hdr["state"]["hist"] == 6 and len(hdr["vectors"]) == 2 + 2 * 6
    CkOracleProblem.stop_at = None
    checkpoint._stop["requested"] = False
    b = _problem()
    r2 = b.fit(np.full(b.n, 7.0), params, checkpoint=path, checkpoint_interval=-1)    # x0 is not used
    assert (r2.status, r2.iterations, r2.evaluations, r2.fx) == (r0.status, r0.iterations, r0.evaluations, r0.fx)
    assert np.array_equal(b.x, ref.x)
    # a cap of 10 continued to 25 equals 25 uninterrupted iterations
    path2 = str(tmp_path / "cap.ckpt")
    c = _problem()
    r3 = c.fit(np.zeros(c.n), lbfgs.default_params(max_iterations=10, epsilon=1e-9), checkpoint=path2)
    assert r3.status == lbfgs.LBFGSERR_MAXIMUMITERATION and r3.iterations == 10
    d = _problem()
    r4 = d.fit(np.zeros(d.n), params, checkpoint=path2)
    assert (r4.status, r4.iterations, r4.evaluations, r4.fx) == (r0.status, r0.iterations, r0.evaluations, r0.fx)
    assert np.array_equal(d.x, ref.x)


def test_checksum_model_is_order_independent():
    v = np.random.default_rng(0).normal(size=1001).astype(np.float32)
    words = v.view(np.uint32)
    whole = checkpoint.checksum_words(words)
    parts = (checkpoint.checksum_words(words[:300]) + checkpoint.checksum_words(words[300:], offset=300)) % (1 << 64)
    assert whole == parts
    flipped = words.copy()
    flipped[500] ^= 1
    assert checkpoint.checksum_words(flipped) != whole
    swapped = words.copy()
    swapped[[3, 4]] = swapped[[4, 3]]
    assert words[3] == words[4] or checkpoint.checksum_words(swapped) != whole


# ---- run_plmc ---------------------------------------------------------------------------------------------------------
def _alignment(tmp_path, seed=6, name="in.a2m", change_one=False):
    codes = synthetic.synthetic_msa_codes(200, 12, seed)
    if change_one:
        codes = codes.copy()
        codes[5, 3] = (codes[5, 3] + 1) % 20
    a2m = str(tmp_path / name)
    synthetic.write_a2m(a2m, codes)
    return a2m


def _kw(a2m, tmp_path, tag, **extra):
    kw = dict(alignment=a2m, couplings_file=str(tmp_path / (tag + "_ECs.txt")),
              param_file=str(tmp_path / (tag + ".model")), focus_seq="seq0/1-12", theta=0.8, ignore_gaps=True,
              iterations=25, lambda_h=0.01, lambda_J=2.0, epsilon=1e-9)
    kw.update(extra)
    return kw


def _table(res):
    t = res.iteration_table
    return t["iter"].astype(int).tolist(), t["fx"].tolist(), t["cond"].tolist()


def test_run_plmc_resume_continues_the_iteration_table(tmp_path, monkeypatch):
    a2m = _alignment(tmp_path)
    ref = tools.run_plmc(engine=CkOracleEngine(), **_kw(a2m, tmp_path, "ref"))
    ck = str(tmp_path / "run.ckpt")
    renames = []
    real_replace = os.replace

    def replace(src, dst):
        renames.append((src, dst, os.path.getsize(src)))
        return real_replace(src, dst)
    monkeypatch.setattr(os, "replace", replace)
    CkOracleProblem.stop_at = 9
    with pytest.raises(tools.FitInterrupted, match="iteration 9"):
        tools.run_plmc(engine=CkOracleEngine(), checkpoint=ck, **_kw(a2m, tmp_path, "a"))
    assert renames and all(s == ck + ".tmp" and d == ck for s, d, _ in renames)
    assert os.path.getsize(ck) == renames[-1][2] and not os.path.exists(ck + ".tmp")
    assert not checkpoint.stop_requested()          # the fit that honoured the request cleared it
    CkOracleProblem.stop_at = None
    res, run = tools.run_plmc(engine=CkOracleEngine(), checkpoint=ck, return_run=True, **_kw(a2m, tmp_path, "a"))
    assert _table(res) == _table(ref) and _table(res)[0] == list(range(1, 26))
    assert res.optimization_status == ref.optimization_status
    assert run.timings["checkpoint_resumes"] == 1
    assert open(str(tmp_path / "a_ECs.txt")).read() == open(str(tmp_path / "ref_ECs.txt")).read()
    assert os.path.exists(ck)                       # not converged: kept
    # a cap of 25 already reached: outputs from the stored state, no new iteration
    n0 = CkOracleProblem.evaluations_total
    before = open(ck, "rb").read()
    res2, run2 = tools.run_plmc(engine=CkOracleEngine(), checkpoint=ck, return_run=True, **_kw(a2m, tmp_path, "b"))
    assert CkOracleProblem.evaluations_total == n0 and _table(res2) == _table(ref)
    assert run2.timings["checkpoint_writes"] == 0 and open(ck, "rb").read() == before     # not written again
    assert open(str(tmp_path / "b.model"), "rb").read() == open(str(tmp_path / "ref.model"), "rb").read()


def test_run_plmc_deletes_the_checkpoint_after_convergence(tmp_path, monkeypatch):
    a2m = _alignment(tmp_path)
    monkeypatch.setenv("EVC_CHECKPOINT", "1")
    kw = _kw(a2m, tmp_path, "c", iterations="max", epsilon=1e-2)
    res = tools.run_plmc(engine=CkOracleEngine(), **kw)
    assert res.optimization_status == "LBFGS_SUCCESS"
    assert not os.path.exists(kw["param_file"] + ".ckpt")


def test_checkpoint_of_another_fit_is_refused_before_the_fit(tmp_path):
    a2m = _alignment(tmp_path)
    ck = str(tmp_path / "f.ckpt")
    tools.run_plmc(engine=CkOracleEngine(), checkpoint=ck, **_kw(a2m, tmp_path, "f", iterations=5))
    before = open(ck, "rb").read()
    other = _alignment(tmp_path, name="other.a2m", change_one=True)
    for kw, field in ((dict(lambda_J=3.0), "lambda_J"), (dict(alignment=other), "data_sha256"),
                      (dict(history=5), "m"), (dict(iterations=3), "requested cap")):
        n0 = CkOracleProblem.evaluations_total
        with pytest.raises(tools.InvalidParameterError, match=field):
            tools.run_plmc(engine=CkOracleEngine(), checkpoint=ck, **dict(_kw(a2m, tmp_path, "g", iterations=5), **kw))
        assert CkOracleProblem.evaluations_total == n0
        assert open(ck, "rb").read() == before


def test_corrupt_or_truncated_checkpoint_names_file_and_vector(tmp_path):
    a2m = _alignment(tmp_path)
    ck = str(tmp_path / "h.ckpt")
    tools.run_plmc(engine=CkOracleEngine(), checkpoint=ck, **_kw(a2m, tmp_path, "h", iterations=4))
    good = open(ck, "rb").read()
    hdr = checkpoint.CheckpointFile(ck).read_header()
    last = hdr["vectors"][-1]
    with open(ck, "wb") as f:
        f.write(good[:-100])
    with pytest.raises(checkpoint.CheckpointError, match=r"h\.ckpt is truncated in vector %s\[%d\]"
                       % (last["name"], last["slot"])):
        tools.run_plmc(engine=CkOracleEngine(), checkpoint=ck, **_kw(a2m, tmp_path, "h", iterations=6))
    bad = bytearray(good)
    bad[hdr["_data_offset"] + 8 * 3 + 1] ^= 0x10          # inside x (float64 vectors of the oracle problem)
    with open(ck, "wb") as f:
        f.write(bytes(bad))
    with pytest.raises(checkpoint.CheckpointError, match=r"h\.ckpt: vector x fails its checksum"):
        tools.run_plmc(engine=CkOracleEngine(), checkpoint=ck, **_kw(a2m, tmp_path, "h", iterations=6))
    bad = bytearray(good)
    bad[60] ^= 0x01                                       # inside the header
    with open(ck, "wb") as f:
        f.write(bytes(bad))
    with pytest.raises(checkpoint.CheckpointError, match="header"):
        tools.run_plmc(engine=CkOracleEngine(), checkpoint=ck, **_kw(a2m, tmp_path, "h", iterations=6))


def test_too_little_disk_raises_resource_error(tmp_path, monkeypatch):
    a2m = _alignment(tmp_path)

    class Vfs(object):
        f_bavail, f_frsize = 10, 4096
    monkeypatch.setattr(os, "statvfs", lambda p: Vfs())
    with pytest.raises(tools.ResourceError, match=r"needs \d+ bytes .* 40960 bytes are available"):
        tools.run_plmc(engine=CkOracleEngine(), checkpoint=str(tmp_path / "d.ckpt"), **_kw(a2m, tmp_path, "d"))
    assert not os.path.exists(str(tmp_path / "d.ckpt"))


def test_cli_checkpoint_options():
    from evcouplings_b200 import plmc_cli
    _, opts = plmc_cli.parse_args(["-c", "x_ECs.txt", "--checkpoint", "f.ckpt", "--checkpoint-interval", "60",
                                   "a.a2m"])
    assert opts["checkpoint"] == "f.ckpt" and opts["checkpoint_interval"] == 60.0
    with pytest.raises(plmc_cli.CliError):
        plmc_cli.parse_args(["-c", "x_ECs.txt", "--checkpoint-interval", "60", "a.a2m"])


# ---- several ranks ------------------------------------------------------------------------------------------------------
def _pythonpath():
    env_pp = os.environ.get("PYTHONPATH", "")
    return env_pp, os.path.join(ROOT, "tests") + os.pathsep + ROOT + os.pathsep + env_pp


def test_two_gloo_ranks_save_and_resume_on_one_or_two_ranks(tmp_path):
    from evcouplings_b200 import launcher
    a2m = _alignment(tmp_path)
    ref = tools.run_plmc(engine=CkOracleEngine(), **_kw(a2m, tmp_path, "ref"))
    ck = str(tmp_path / "m.ckpt")
    env_pp, pp = _pythonpath()
    os.environ["PYTHONPATH"] = pp
    try:
        run2 = lambda kw: launcher.run_plmc_multi_gpu(2, kw, backend="gloo", timeout=600,  # noqa: E731
                                                      engine_factory="test_fit_checkpoint:CkShardedEngine")
        r10 = run2(_kw(a2m, tmp_path, "m10", iterations=10, checkpoint=ck))
        assert len(r10.iteration_table) == 10 and os.path.exists(ck)
        hdr = checkpoint.CheckpointFile(ck).read_header()
        assert hdr["info"]["world"] == 2 and hdr["state"]["k"] == 10
        import shutil
        shutil.copy(ck, str(tmp_path / "m1.ckpt"))
        r25 = run2(_kw(a2m, tmp_path, "m25", checkpoint=ck))
    finally:
        os.environ["PYTHONPATH"] = env_pp
    r1 = tools.run_plmc(engine=CkOracleEngine(), checkpoint=str(tmp_path / "m1.ckpt"), **_kw(a2m, tmp_path, "s25"))
    f_ref = np.array(ref.iteration_table["fx"].astype(float))
    for res in (r25, r1):
        assert _table(res)[0] == list(range(1, 26))
        f = np.array(res.iteration_table["fx"].astype(float))
        assert np.abs(f - f_ref).max() <= 1e-9 * np.abs(f_ref).max()
    cn_ref = np.loadtxt(str(tmp_path / "ref_ECs.txt"), usecols=5)
    for tag in ("m25", "s25"):
        assert np.abs(np.loadtxt(str(tmp_path / (tag + "_ECs.txt")), usecols=5) - cn_ref).max() < 1e-6


def test_worker_stopped_by_sigterm_saves_and_the_resumed_fit_matches(tmp_path):
    a2m = _alignment(tmp_path)
    kw = _kw(a2m, tmp_path, "w", iterations=60)
    ref = tools.run_plmc(engine=CkOracleEngine(), **dict(kw, param_file=str(tmp_path / "ref.model"),
                                                         couplings_file=str(tmp_path / "ref_ECs.txt")))
    ck = str(tmp_path / "w.ckpt")
    spec = str(tmp_path / "spec.json")
    with open(spec, "w") as f:
        json.dump(dict(kwargs=dict(kw, checkpoint=ck, checkpoint_interval=0.0), backend="gloo",
                       engine_factory="test_fit_checkpoint:SlowOracleEngine", result=str(tmp_path / "r.pkl")), f)
    _, pp = _pythonpath()
    env = dict(os.environ, PYTHONPATH=pp, RANK="0", LOCAL_RANK="0", WORLD_SIZE="1", MASTER_ADDR="127.0.0.1",
               MASTER_PORT=str(30000 + os.getpid() % 2000))
    p = subprocess.Popen([sys.executable, "-m", "evcouplings_b200.worker", spec], env=env, cwd=ROOT,
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    try:
        t0 = time.time()
        while not os.path.exists(ck) and p.poll() is None and time.time() - t0 < 300:
            time.sleep(0.05)
        assert p.poll() is None, p.stdout.read().decode()[-2000:]
        p.send_signal(signal.SIGTERM)
        out = p.communicate(timeout=300)[0].decode()
    finally:
        if p.poll() is None:
            p.kill()
            p.wait()
    assert p.returncode != 0 and "FitInterrupted" in out, out[-2000:]
    k = checkpoint.CheckpointFile(ck).read_header()["state"]["k"]
    assert 1 <= k < 60
    res = tools.run_plmc(engine=CkOracleEngine(), checkpoint=ck, **kw)
    assert _table(res) == _table(ref)
    assert open(kw["couplings_file"]).read() == open(str(tmp_path / "ref_ECs.txt")).read()


def test_a_stop_request_stops_one_fit(tmp_path):
    params = lbfgs.default_params(max_iterations=6, epsilon=1e-9)
    checkpoint.request_stop()
    a = _problem()
    r1 = a.fit(np.zeros(a.n), params, checkpoint=str(tmp_path / "a.ckpt"))
    assert r1.status == lbfgs.LBFGSERR_CANCELED and r1.iterations == 1 and not checkpoint.stop_requested()
    b = _problem()
    r2 = b.fit(np.zeros(b.n), params, checkpoint=str(tmp_path / "b.ckpt"))
    assert r2.status == lbfgs.LBFGSERR_MAXIMUMITERATION and r2.iterations == 6


def test_an_interrupt_during_a_write_is_agreed_and_reraised(tmp_path, monkeypatch):
    ck = checkpoint.CheckpointFile(str(tmp_path / "i.ckpt"))

    def write(*a, **k):
        raise KeyboardInterrupt()
    monkeypatch.setattr(ck, "write", write)
    agreed = []
    real = checkpoint.agree_flags
    monkeypatch.setattr(checkpoint, "agree_flags", lambda e, f: agreed.append(list(f)) or real(e, f))
    gate = checkpoint.Gate(None, -1.0)
    state = dict(k=3, evaluations=4, hist=3, end=3, switched_at=-1)
    with pytest.raises(KeyboardInterrupt):
        checkpoint.write_state(ck, gate, state, [], {}, None)
    assert agreed == [[True]] and gate.last_key is None
