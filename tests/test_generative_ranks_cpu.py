"""
The multi-rank plumbing of the generative tools without a GPU: the chain partition and its refusals, --gpus of
evcplm-sample / evcplm-bmdca / evcplm-logz and their refusals (exit code 2 before any rank or device work), and the
launcher's job dispatch, chain-order gather and failure relay with a stand-in job on three gloo ranks.
"""
import io
import os
import sys
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

from evcouplings_b200 import bmdca_cli, launcher, logz_cli, model_ops, sample_cli, tools  # noqa: E402


# ----------------------------------------------------------------------------------------------------------------------
# the chain partition
# ----------------------------------------------------------------------------------------------------------------------
def ranges(M, R):
    return [model_ops.chain_range(M, R, r) for r in range(R)]


@pytest.mark.parametrize("M,R,want", [
    (2, 2, [(0, 1), (1, 2)]),
    (3, 3, [(0, 1), (1, 2), (2, 3)]),
    (3, 2, [(0, 2), (2, 3)]),
    (4, 3, [(0, 2), (2, 3), (3, 4)]),
    (1001, 3, [(0, 334), (334, 668), (668, 1001)]),
    (16384, 8, [(2048 * r, 2048 * (r + 1)) for r in range(8)]),
])
def test_chain_partition(M, R, want):
    got = ranges(M, R)
    assert got == want
    assert got[0][0] == 0 and got[-1][1] == M and all(a[1] == b[0] for a, b in zip(got, got[1:]))
    sizes = [hi - lo for lo, hi in got]
    assert min(sizes) >= 1 and max(sizes) - min(sizes) <= 1 and sizes[0] == max(sizes)


def test_chain_partition_refusals():
    for M, R in ((1, 2), (2, 3), (7, 8)):
        with pytest.raises(ValueError, match="at least one chain"):
            model_ops.chain_range(M, R, 0)
    with pytest.raises(ValueError, match="int32"):
        model_ops.chain_range(1 << 31, 2, 0)
    assert model_ops.chain_range((1 << 31) - 1, 2, 1) == (1 << 30, (1 << 31) - 1)


def test_num_gpus_refusals():
    assert model_ops.check_num_gpus(1, 1) == 1                 # one GPU: no device query, no partition
    with pytest.raises(ValueError, match="at least 1"):
        model_ops.check_num_gpus(0, 10)
    with pytest.raises(ValueError, match="at least one chain"):
        model_ops.check_num_gpus(3, 2, backend="gloo")
    with pytest.raises(ValueError, match="int32"):
        model_ops.check_num_gpus(2, 1 << 31, backend="gloo")
    assert model_ops.check_num_gpus(3, 3, backend="gloo") == 3  # gloo ranks may share a device


def test_num_gpus_above_the_visible_devices_is_refused(monkeypatch):
    import torch
    monkeypatch.setattr(torch.cuda, "device_count", lambda: 2)
    assert model_ops.check_num_gpus(2, 10) == 2
    with pytest.raises(ValueError, match="2 GPUs are visible"):
        model_ops.check_num_gpus(3, 10)


def test_the_python_api_refuses_before_any_device_work():
    model = dict(L=3, q=2, h=np.zeros((3, 2)), alphabet="AB")
    for call in (lambda: model_ops.sample_sequences(model, 1, 1, num_gpus=2, backend="gloo"),
                 lambda: model_ops.log_partition(model, 2, 4, num_gpus=3, backend="gloo"),
                 lambda: model_ops.boltzmann_refine(model, 1, n_chains=1, num_gpus=2, backend="gloo"),
                 lambda: model_ops.sample_sequences(model, 5, 1, num_gpus=0)):
        with pytest.raises(ValueError):
            call()


def test_sharded_refusals_come_before_device_work():
    class Group(object):            # an engine of a 3-rank group with no device: any device work would fail
        world, rank = 3, 0
    m = model_ops.read_model(os.path.join(ROOT, "tests", "golden", "tiny.model"))
    for call in (lambda: model_ops.BoltzmannLearner(m, 2, engine=Group()),
                 lambda: model_ops.log_partition(m, 2, 4, engine=Group()),
                 lambda: model_ops.sample_sequences(m, 2, 1, engine=Group()),
                 lambda: model_ops.BoltzmannLearner(m, 1 << 31, engine=Group())):
        with pytest.raises(ValueError, match="at least one chain|int32"):
            call()


# ----------------------------------------------------------------------------------------------------------------------
# --gpus of the three command lines
# ----------------------------------------------------------------------------------------------------------------------
CLIS = [
    (sample_cli, ["m.model", "-n", "4", "--sweeps", "1", "-o", "x.a2m"], "evcplm-sample"),
    (bmdca_cli, ["m.model", "--updates", "1", "--chains", "4", "-o", "x.model"], "evcplm-bmdca"),
    (logz_cli, ["m.model", "--chains", "4"], "evcplm-logz"),
]


@pytest.mark.parametrize("cli,argv,prog", CLIS, ids=[c[2] for c in CLIS])
def test_gpus_option(cli, argv, prog):
    assert "gpus" not in cli.parse_args(argv)                   # the options of a one-GPU run are unchanged
    assert cli.parse_args(argv + ["--gpus", "1"])["gpus"] == 1
    assert cli.parse_args(["--gpus", "3"] + argv)["gpus"] == 3
    for bad in (["--gpus", "0"], ["--gpus", "-2"], ["--gpus", "two"], ["--gpus"], ["-g", "2"]):
        with pytest.raises(cli.CliError, match=prog):
            cli.parse_args(argv + bad)


@pytest.mark.parametrize("cli,argv,prog", CLIS, ids=[c[2] for c in CLIS])
def test_gpus_refusals_exit_2_before_any_work(cli, argv, prog, monkeypatch, tmp_path):
    """The model file does not exist: a refusal that got as far as reading it would exit 1, not 2."""
    import torch
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(torch.cuda, "device_count", lambda: 2)
    started = []
    monkeypatch.setattr(launcher, "_start_ranks", lambda *a, **k: started.append(a))
    for extra, backend, why in ((["--gpus", "0"], "nccl", "at least 1"),
                                (["--gpus", "3"], "nccl", "2 GPUs are visible"),
                                (["--gpus", "5"], "gloo", "4 chains cannot be split over 5 ranks")):
        err = io.StringIO()
        assert cli.main(argv + extra, stderr=err, backend=backend) == 2, err.getvalue()
        assert err.getvalue().startswith(prog) and why in err.getvalue(), err.getvalue()
    assert not started and not os.listdir(str(tmp_path))
    err = io.StringIO()
    assert cli.main(argv + ["--gpus", "2"], stderr=err) == 1            # accepted; then the missing model file
    assert "FileNotFoundError" in err.getvalue() and not started


# ----------------------------------------------------------------------------------------------------------------------
# launcher and worker with a stand-in job
# ----------------------------------------------------------------------------------------------------------------------
class StandInEngine(object):
    """What the generative jobs use of an engine, on the CPU: rank, world, device and the gather of the process group."""

    def __init__(self):
        from evcouplings_b200.dist import Collective
        import torch
        self.coll = Collective()
        self.rank, self.world = self.coll.rank, self.coll.world
        self.device = torch.device("cpu")

    def all_gather(self, tensor):
        return self.coll.all_gather(tensor)


def per_chain(M):
    """a float64 value per chain with -0.0, +0.0, a NaN payload and subnormals among them, and uint8 rows"""
    v = np.linspace(-3.0, 3.0, M)
    v[::5] = -0.0
    v[1::7] = 0.0
    v[2::11] = 5e-324
    v[-1] = np.frombuffer(np.uint64(0x7ff8dead00000001).tobytes(), dtype=np.float64)[0]
    rows = (np.arange(M * 6) % 251).astype(np.uint8).reshape(M, 6)
    return v, rows


def stand_in_job(engine, n_chains, fail_rank=None):
    """Every rank gathers its block of per_chain(n_chains) in chain order; rank ``fail_rank`` fails instead, while the
    others wait long enough for the launcher to see that failure first and stop them."""
    if fail_rank is not None:
        if engine.rank == fail_rank:
            raise RuntimeError("stand-in failure on rank %d" % engine.rank)
        time.sleep(20)
    lo, hi = model_ops.chain_range(n_chains, engine.world, engine.rank)
    v, rows = per_chain(n_chains)
    return dict(world=engine.world, lo=lo, hi=hi, v=model_ops._gather_chains(engine, v[lo:hi].copy(), n_chains),
                rows=model_ops._gather_chains(engine, rows[lo:hi].copy(), n_chains))


@pytest.fixture
def tests_on_path():
    old = os.environ.get("PYTHONPATH", "")
    os.environ["PYTHONPATH"] = os.path.join(ROOT, "tests") + os.pathsep + ROOT + os.pathsep + old
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    try:
        yield
    finally:
        os.environ["PYTHONPATH"] = old
        sys.path.remove(os.path.join(ROOT, "tests"))


def run_stand_in(R, **kw):
    return launcher.run_job("test_generative_ranks_cpu:stand_in_job", R, kw, backend="gloo",
                            engine_factory="test_generative_ranks_cpu:StandInEngine", timeout=600)


@pytest.mark.parametrize("R,M", [(3, 1001), (3, 3), (2, 3)])
def test_launcher_runs_a_job_and_gathers_in_chain_order(tests_on_path, R, M):
    out = run_stand_in(R, n_chains=M)
    v, rows = per_chain(M)
    assert out["world"] == R and (out["lo"], out["hi"]) == model_ops.chain_range(M, R, 0)
    assert out["v"].dtype == np.float64 and out["v"].tobytes() == v.tobytes()       # -0.0 and the NaN payload kept
    assert out["rows"].dtype == np.uint8 and np.array_equal(out["rows"], rows)


def test_launcher_relays_a_failing_rank(tests_on_path):
    """rank 1 fails; the others are stopped, and its output comes back in the error"""
    t0 = time.time()
    with pytest.raises(tools.ExternalToolError) as e:
        run_stand_in(3, n_chains=10, fail_rank=1)
    assert "run failed (rank 1)" in str(e.value) and "stand-in failure on rank 1" in str(e.value)
    assert time.time() - t0 < 20


def test_launcher_refuses_an_unknown_job():
    with pytest.raises(ValueError, match="unknown job"):
        launcher.run_job("fit", 2, {})
    assert launcher.JOBS == ("run_plmc", "sample", "bmdca", "logz")
