"""
The Gibbs sampler, Boltzmann-machine refinement (bmDCA) and annealed importance sampling on several ranks give the
bits of one process (-m gpu; one device is enough, two for the NCCL test).

1. Library level, in one process: samplers over adjacent chain ranges each count their chains (evc_code_counts); the
   integer sum of the counts equals the counts of one sampler over all chains, and evc_bm_update on that sum gives the
   single-handle parameters bit for bit -- at L = 200, q = 21 with partly filled CTAs, at q = 2 and q = 32, and with
   shards of a single chain.
2. Two and three real ranks on device 0 over gloo, through the launcher and the worker: evcplm-bmdca, evcplm-logz and
   evcplm-sample with --gpus write and print exactly what they write and print without it.
3. Inside an initialised process group: BoltzmannLearner (burn-in, updates split over run() calls, M not divisible by
   the rank count), log_partition and sample_sequences return on every rank what one process returns.
4. Two GPUs over NCCL, with placement by LOCAL_RANK (skipped below two GPUs).
"""
import io
import os
import pickle
import socket
import subprocess
import sys

import numpy as np
import pytest

from evcouplings_b200 import _lib, bmdca_cli, logz_cli, model_io, model_ops, sample_cli, synthetic

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY = os.path.join(ROOT, "tests", "golden", "tiny.model")
RANK_TIMEOUT_S = 900


@pytest.fixture(scope="module")
def eng():
    from evcouplings_b200.engine import CudaEngine
    return CudaEngine(standalone=True)


def random_model(L, q, seed, scale=0.1):
    rng = np.random.default_rng(seed)
    alphabet = "".join(chr(c) for c in range(ord("A"), ord("A") + q)) if q <= 26 else \
        "".join(chr(c) for c in range(ord("A"), ord("A") + 26)) + "012345"[:q - 26]
    npairs = L * (L - 1) // 2
    fi = rng.dirichlet(np.ones(q), L).astype(np.float32)
    fij = rng.dirichlet(np.ones(q * q), npairs).astype(np.float32).reshape(npairs, q, q)
    return dict(L=L, q=q, alphabet=alphabet, h=rng.normal(0, 0.5, (L, q)).astype(np.float32),
                J=rng.normal(0, scale, (npairs, q, q)).astype(np.float32), fi=fi, fij=fij,
                target_seq="".join(alphabet[(3 * i + 1) % q] for i in range(L)))


def write_model(path, m):
    model_io.write_model_file(path, m["L"], m["q"], m["n_valid"], m["n_invalid"], m["num_iter"], m["theta"],
                              m["lambda_h"], m["lambda_J"], m["lambda_group"], m["n_eff"], m["alphabet"],
                              m["weights"], m["target_seq"], m["index_list"], m["fi"], m["h"], m["fij"], m["J"])
    return path


def l200_model():
    """a synthetic L = 200, q = 21 model with a regularised header: 20 planted contacts on random couplings"""
    m = synthetic.planted_potts_model(200, 21, 20, seed=4)
    rng = np.random.default_rng(4)
    m["J"] = (m["J"] + rng.normal(0, 0.02, m["J"].shape)).astype(np.float32)
    m.update(lambda_h=0.01, lambda_J=0.5, n_eff=300.0)
    return m


# ----------------------------------------------------------------------------------------------------------------------
# 1. library level
# ----------------------------------------------------------------------------------------------------------------------
def counts_of(eng, sampler):
    import torch
    L, q, n = sampler.L, sampler.q, sampler.n_chains
    codes = torch.empty((n, L), dtype=torch.uint8, device=eng.device)
    _lib.check(eng.lib.evc_sampler_codes(sampler.handle, eng.ptr(codes), eng.stream()), "evc_sampler_codes")
    out = torch.full((L * q + L * (L - 1) // 2 * q * q,), -1, dtype=torch.int32, device=eng.device)
    _lib.check(eng.lib.evc_code_counts(eng.ptr(codes), n, L, q, eng.ptr(out), eng.stream()), "evc_code_counts")
    return out


def bm_update(eng, x, counts, M, f, Lq):
    import torch
    x = x.clone()
    stats = torch.zeros(2, dtype=torch.float64, device=eng.device)
    _lib.check(eng.lib.evc_bm_update(eng.ptr(x), eng.ptr(counts), M, eng.ptr(f), x.numel(), Lq, 0.25, 0.003, 0.02,
                                     eng.ptr(stats), eng.stream()), "evc_bm_update")
    return x.cpu().numpy(), stats.cpu().numpy()


# (L, q, M, R, sweeps, edge)
LIBRARY_CASES = [
    (200, 21, 1001, 3, 3, "shards 334/334/333: 13 chains per CTA, the last CTA of every shard partly filled"),
    (200, 21, 1001, 2, 3, "shards 501/500"),
    (64, 2, 97, 3, 5, "q = 2"),
    (40, 32, 50, 2, 5, "q = 32"),
    (30, 21, 3, 3, 4, "shards of a single chain"),
    (30, 21, 5, 3, 4, "a single-chain shard next to two-chain ones"),
]


@pytest.mark.parametrize("L,q,M,R,sweeps,edge", LIBRARY_CASES, ids=["L%dq%dM%dR%d" % c[:4] for c in LIBRARY_CASES])
def test_shard_counts_sum_to_the_whole_and_update_the_same(eng, L, q, M, R, sweeps, edge):
    import torch
    m = random_model(L, q, seed=L + q + M)
    x = torch.from_numpy(model_ops.model_x(m)).to(eng.device)
    f = torch.from_numpy(np.concatenate([m["fi"].ravel(), m["fij"].ravel()])).to(eng.device)
    with model_ops.PottsSampler(m, M, seed=17, engine=eng) as whole:
        whole.run(sweeps)
        want = counts_of(eng, whole)
        want_codes = whole.codes()
    total = torch.zeros_like(want)
    codes = []
    for r in range(R):
        lo, hi = model_ops.chain_range(M, R, r)
        with model_ops.PottsSampler(m, hi - lo, seed=17, chain_offset=lo, engine=eng) as s:
            s.run(sweeps)
            part = counts_of(eng, s)
            codes.append(s.codes())
        assert int(part[:L * q].sum().item()) == (hi - lo) * L
        total += part
    assert np.array_equal(np.concatenate(codes), want_codes), edge
    assert torch.equal(total, want), edge
    x1, st1 = bm_update(eng, x, want, M, f, L * q)
    xR, stR = bm_update(eng, x, total, M, f, L * q)
    assert x1.tobytes() == xR.tobytes() and st1.tobytes() == stR.tobytes(), edge
    assert not np.array_equal(x1, x.cpu().numpy())


# ----------------------------------------------------------------------------------------------------------------------
# 2. real ranks through the launcher and the worker
# ----------------------------------------------------------------------------------------------------------------------
def run_cli(cli, argv, backend="gloo"):
    out, err = io.StringIO(), io.StringIO()
    kw = dict(stdout=out) if cli is logz_cli else {}
    rc = cli.main(argv, stderr=err, backend=backend, **kw)
    assert rc == 0, err.getvalue()
    return out.getvalue(), err.getvalue()


def same_files(a, b):
    with open(a, "rb") as fa, open(b, "rb") as fb:
        return fa.read() == fb.read()


@pytest.fixture(scope="module")
def l200_path(tmp_path_factory):
    return write_model(str(tmp_path_factory.mktemp("l200") / "l200.model"), l200_model())


BMDCA_CASES = [("tiny", 2, ["--updates", "6", "--chains", "301", "--sweeps", "3", "--burn-in", "5",
                             "--learning-rate", "0.2", "--seed", "11"]),
               ("tiny", 3, ["--updates", "6", "--chains", "301", "--sweeps", "3", "--burn-in", "5",
                            "--learning-rate", "0.2", "--seed", "11"]),
               ("l200", 3, ["--updates", "4", "--chains", "1001", "--sweeps", "2", "--burn-in", "3", "--seed", "2"])]


@pytest.mark.parametrize("which,R,args", BMDCA_CASES, ids=["%s-R%d" % c[:2] for c in BMDCA_CASES])
def test_bmdca_command_on_ranks_writes_the_same_bytes(tmp_path, l200_path, which, R, args):
    model = TINY if which == "tiny" else l200_path
    outs = {}
    for tag, extra in (("one", []), ("ranks", ["--gpus", str(R)])):
        out_m, out_e = str(tmp_path / (tag + ".model")), str(tmp_path / (tag + "_ECs.txt"))
        outs[tag] = run_cli(bmdca_cli, [model] + args + ["-o", out_m, "-c", out_e] + extra)
    assert outs["ranks"] == outs["one"]
    assert len(outs["one"][1].splitlines()) == 1 + int(args[1])         # header + one row per update
    assert same_files(str(tmp_path / "one.model"), str(tmp_path / "ranks.model"))
    assert same_files(str(tmp_path / "one_ECs.txt"), str(tmp_path / "ranks_ECs.txt"))


@pytest.mark.parametrize("R", [2, 3])
def test_logz_command_on_ranks_prints_the_same_lines(tmp_path, R):
    argv = [TINY, "--chains", "1000", "--temperatures", "64", "--burn-in", "16", "--seed", "5"]
    one = run_cli(logz_cli, argv)
    ranks = run_cli(logz_cli, argv + ["--gpus", str(R)])
    assert ranks == one and "log Z forward" in one[0] and "log Z reverse" in one[0]


@pytest.mark.parametrize("R", [2, 3])
def test_sample_command_on_ranks_writes_the_same_a2m(tmp_path, R):
    for tag, extra in (("one", []), ("ranks", ["--gpus", str(R)])):
        run_cli(sample_cli, [TINY, "-n", "1001", "--sweeps", "7", "--seed", "3", "-o", str(tmp_path / (tag + ".a2m"))]
                + extra)
    assert same_files(str(tmp_path / "one.a2m"), str(tmp_path / "ranks.a2m"))


def test_python_api_on_ranks_returns_the_same_values(eng):
    m = model_ops.read_model(TINY)
    rows1, rowsR = [], []
    want = model_ops.boltzmann_refine(m, 4, n_chains=200, sweeps=2, seed=1, learning_rate=0.3, burn_in=3,
                                      progress=lambda k, st: rows1.append((k, st)), engine=eng)
    got = model_ops.boltzmann_refine(m, 4, n_chains=200, sweeps=2, seed=1, learning_rate=0.3, burn_in=3,
                                     progress=lambda k, st: rowsR.append((k, st)), num_gpus=3, backend="gloo")
    assert got["h"].tobytes() == want["h"].tobytes() and got["J"].tobytes() == want["J"].tobytes()
    assert repr(rowsR) == repr(rows1) and [k for k, _ in rows1] == [0, 1, 2, 3]
    assert got["num_iter"] == 4
    assert model_ops.log_partition(m, 300, 16, 4, seed=2, num_gpus=2, backend="gloo") == \
        model_ops.log_partition(m, 300, 16, 4, seed=2, engine=eng)
    assert model_ops.sample_sequences(m, 50, 3, seed=8, init="target", num_gpus=2, backend="gloo") == \
        model_ops.sample_sequences(m, 50, 3, seed=8, init="target", engine=eng)


# ----------------------------------------------------------------------------------------------------------------------
# 3. inside an initialised process group
# ----------------------------------------------------------------------------------------------------------------------
RANK_SCRIPT = r'''
import os, pickle, sys
sys.path.insert(0, sys.argv[1])
import torch
import torch.distributed as dist
backend, model_path, out_path = sys.argv[2:5]
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
local = int(os.environ["LOCAL_RANK"]) if backend == "nccl" else 0
torch.cuda.set_device(local)
if backend == "nccl":
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
else:
    dist.init_process_group(backend, rank=rank, world_size=world)
from evcouplings_b200 import model_ops
from evcouplings_b200.engine import CudaEngine
eng = CudaEngine()
assert eng.world == world and eng.device_index == local
with open(model_path, "rb") as f:
    job = pickle.load(f)
m = job["model"]
out = dict(rank=rank, device=eng.device_index)
rows = []
with model_ops.BoltzmannLearner(m, job["chains"], seed=4, learning_rate=0.25, burn_in=5, engine=eng) as bl:
    out["range"] = (bl.lo, bl.hi)
    bl.run(3, 2, progress=lambda k, st: rows.append((k, st)))
    bl.run(5, 2, progress=lambda k, st: rows.append((k, st)))
    out["params"] = bl.parameters()
    out["fn"] = bl.fn_scores()
out["rows"] = rows
out["logz"] = model_ops.log_partition(m, job["chains"], 32, 8, seed=6, engine=eng)
out["sample"] = model_ops.sample_sequences(m, job["chains"], 4, seed=9, engine=eng)
torch.cuda.synchronize()
out["device_bytes_in_use"] = torch.cuda.mem_get_info()[1] - torch.cuda.mem_get_info()[0]
with open(out_path % rank, "wb") as f:
    pickle.dump(out, f)
dist.destroy_process_group()
'''


def _free_port():
    s = socket.socket(socket.AF_INET, socket.SOCK_STREAM)
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def run_group(tmp_path, R, backend, model, chains):
    script = str(tmp_path / "rank.py")
    with open(script, "w") as f:
        f.write(RANK_SCRIPT)
    job = str(tmp_path / "job.pkl")
    with open(job, "wb") as f:
        pickle.dump(dict(model=model, chains=chains), f)
    out = str(tmp_path / "rank%d.pkl")
    port = _free_port()
    procs = []
    for r in range(R):
        env = dict(os.environ, RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE=str(R), MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(port))
        procs.append(subprocess.Popen([sys.executable, script, ROOT, backend, job, out], env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    logs = []
    try:
        for p in procs:
            logs.append(p.communicate(timeout=RANK_TIMEOUT_S)[0])
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()
    assert [p.returncode for p in procs] == [0] * R, "\n".join(l[-3000:] for l in logs)
    res = []
    for r in range(R):
        with open(out % r, "rb") as f:
            res.append(pickle.load(f))
    return res


def one_process(eng, m, chains):
    rows = []
    with model_ops.BoltzmannLearner(m, chains, seed=4, learning_rate=0.25, burn_in=5, engine=eng) as bl:
        bl.run(8, 2, progress=lambda k, st: rows.append((k, st)))
        params, fn = bl.parameters(), bl.fn_scores()
    return dict(params=params, fn=fn, rows=rows,
                logz=model_ops.log_partition(m, chains, 32, 8, seed=6, engine=eng),
                sample=model_ops.sample_sequences(m, chains, 4, seed=9, engine=eng))


def check_group_equals_one(res, want, R, chains):
    for r, got in enumerate(res):
        assert got["range"] == model_ops.chain_range(chains, R, r)
        assert got["params"][0].tobytes() == want["params"][0].tobytes(), r
        assert got["params"][1].tobytes() == want["params"][1].tobytes(), r
        assert got["fn"].tobytes() == want["fn"].tobytes(), r
        assert repr(got["rows"]) == repr(want["rows"]), r     # repr: exact digits, and a NaN r equals a NaN r
        assert got["logz"] == want["logz"], r
        assert got["sample"] == want["sample"], r


@pytest.mark.parametrize("which,R,chains", [("tiny", 2, 301), ("tiny", 3, 301), ("l200", 3, 1001)])
def test_initialised_group_returns_one_process_values_on_every_rank(tmp_path, eng, which, R, chains):
    m = model_ops.read_model(TINY) if which == "tiny" else l200_model()
    res = run_group(tmp_path, R, "gloo", m, chains)
    want = one_process(eng, m, chains)
    check_group_equals_one(res, want, R, chains)
    print("\n%s, %d ranks on one device, M = %d: device memory in use after the run %.1f MB (all ranks)"
          % (which, R, chains, res[0]["device_bytes_in_use"] / 2 ** 20))


# ----------------------------------------------------------------------------------------------------------------------
# 4. two GPUs over NCCL
# ----------------------------------------------------------------------------------------------------------------------
def _two_gpus():
    import torch
    return torch.cuda.device_count() >= 2


@pytest.mark.skipif(not _two_gpus(), reason="needs two GPUs")
def test_two_gpus_over_nccl(tmp_path, eng):
    m = model_ops.read_model(TINY)
    res = run_group(tmp_path, 2, "nccl", m, 301)
    assert [r["device"] for r in res] == [0, 1]
    check_group_equals_one(res, one_process(eng, m, 301), 2, 301)
    args = [TINY, "--updates", "5", "--chains", "301", "--sweeps", "3", "--burn-in", "4", "--seed", "3"]
    outs = {}
    for tag, extra in (("one", []), ("two", ["--gpus", "2"])):
        outs[tag] = run_cli(bmdca_cli, args + ["-o", str(tmp_path / (tag + ".model")),
                                               "-c", str(tmp_path / (tag + "_ECs.txt"))] + extra, backend="nccl")
    assert outs["one"] == outs["two"]
    assert same_files(str(tmp_path / "one.model"), str(tmp_path / "two.model"))
    assert same_files(str(tmp_path / "one_ECs.txt"), str(tmp_path / "two_ECs.txt"))
    argv = [TINY, "--chains", "1000", "--temperatures", "64", "--burn-in", "16", "--seed", "5"]
    assert run_cli(logz_cli, argv + ["--gpus", "2"], backend="nccl") == run_cli(logz_cli, argv, backend="nccl")
