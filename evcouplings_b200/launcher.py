"""
Multi-GPU from a single-process call (SURVEY.md 8b "owns its CUDA streams/NCCL comm internally", VERDICT r1
missing #3).  The reference calls ``run_plmc`` from ONE blocking Python process and forwards ``cpu`` as plmc's
``-n`` (evcouplings/couplings/tools.py:257-259); to give that call all GPUs of the box this module starts one
rank per GPU (``python -m evcouplings_b200.worker``), each of which runs the same ``tools.run_plmc`` as a member
of a torch.distributed / NCCL group on 127.0.0.1: sequences sharded over ranks, ONE all-reduce of [g, -loglk]
per evaluation, rank 0 writes the files.  The parent waits, relays failures as ExternalToolError and rebuilds
the PlmcResult from rank 0's plmc-style log (same parser as the reference's, tools.py:20-108).

The same start / wait / failure relay / cleanup serves the generative tools (run_job: the Gibbs sampler, bmDCA and
annealed importance sampling of model_ops, ``num_gpus=N``): each rank runs its block of chains and rank 0's result,
which equals the single-process one bit for bit, comes back to the caller.
"""
import json
import os
import pickle
import socket
import subprocess
import sys
import tempfile
import time


# how long an interrupted launcher waits for ranks that save a checkpoint before it kills them
RANK_EXIT_TIMEOUT_S = 600


def _free_port():
    s = socket.socket(socket.AF_INET, socket.SOCK_STREAM)
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


# jobs a rank can run (evcouplings_b200.worker): "run_plmc" is tools.run_plmc; the generative tools are
# model_ops.run_job -- the Gibbs sampler, Boltzmann-machine refinement and annealed importance sampling
JOBS = ("run_plmc", "sample", "bmdca", "logz")
# the jobs of model_ops.run_job: those generative tools and sequence design (model_ops.design_codes)
GENERATIVE_JOBS = JOBS[1:] + ("design",)


def _start_ranks(job, ndev, kwargs, args=None, backend="nccl", engine_factory=None, timeout=None, label=None):
    """Start ``ndev`` ranks of ``job`` (``python -m evcouplings_b200.worker``), wait for all of them and return the
    result rank 0 stored, with the launch time.  ``kwargs`` go to the ranks as JSON, ``args`` (anything picklable,
    such as a model's arrays) as a pickle.  A failing rank, or the timeout, stops the others and raises
    ExternalToolError with the end of that rank's output.  ``job`` may also be "module:function", called as
    function(engine, **kwargs), for tests of this plumbing; so may ``engine_factory``."""
    from . import tools
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    workdir = tempfile.mkdtemp(prefix="evcplm_ranks_")
    spec_path = os.path.join(workdir, "spec.json")
    result_path = os.path.join(workdir, "rank0.pkl")
    spec = dict(job=job, kwargs=kwargs, backend=backend, engine_factory=engine_factory, result=result_path)
    if args is not None:
        spec["args"] = os.path.join(workdir, "args.pkl")
        with open(spec["args"], "wb") as f:
            pickle.dump(args, f, protocol=pickle.HIGHEST_PROTOCOL)
    with open(spec_path, "w") as f:
        json.dump(spec, f)
    port = _free_port()
    procs, logs = [], []
    for r in range(ndev):
        env = dict(os.environ)
        env.update(RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE=str(ndev), MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(port))
        env["PYTHONPATH"] = root + os.pathsep + env.get("PYTHONPATH", "")
        env.pop("EVC_NUM_GPUS", None)
        # like torchrun: one OpenMP / BLAS thread per rank unless the caller decided otherwise -- ndev ranks each
        # spinning a full-size host thread pool starve the threads that drive the GPUs
        for var in ("OMP_NUM_THREADS", "MKL_NUM_THREADS", "OPENBLAS_NUM_THREADS"):
            env.setdefault(var, "1")
        log = open(os.path.join(workdir, "rank%d.err" % r), "w+")
        logs.append(log)
        procs.append(subprocess.Popen([sys.executable, "-m", "evcouplings_b200.worker", spec_path],
                                      env=env, stdout=log, stderr=subprocess.STDOUT, cwd=root))
    t0 = time.time()
    failed = None
    interrupted = False
    try:
        while True:
            codes = [p.poll() for p in procs]
            bad = [r for r, c in enumerate(codes) if c not in (None, 0)]
            if bad:
                failed = bad[0]
                break
            if all(c == 0 for c in codes):
                break
            if timeout is not None and time.time() - t0 > timeout:
                failed = -1
                break
            time.sleep(0.05)
    except BaseException:
        # this call was interrupted (KeyboardInterrupt, SystemExit from a signal handler): the ranks get SIGTERM, which
        # a checkpointed fit turns into a saved state at its next iteration boundary; they are waited for below
        interrupted = True
        raise
    finally:
        for p in procs:                       # our own children, by PID
            if p.poll() is None and (failed is not None or interrupted):
                p.terminate()
        for p in procs:
            try:
                p.wait(timeout=RANK_EXIT_TIMEOUT_S if interrupted and kwargs.get("checkpoint") else 30)
            except subprocess.TimeoutExpired:
                p.kill()
                p.wait()
    if failed is not None:
        tail = ""
        if failed >= 0:
            logs[failed].seek(0)
            tail = logs[failed].read()[-2000:]
        for log in logs:
            log.close()
        raise tools.ExternalToolError("multi-GPU %s run failed (%s): %s"
                                      % (label or job, "timeout" if failed < 0 else "rank %d" % failed, tail))
    if os.environ.get("EVC_TRACE"):
        for r, log in enumerate(logs):
            log.seek(0)
            for ln in log.read().splitlines():
                if "evc-trace" in ln:
                    sys.stderr.write("[rank %d] %s\n" % (r, ln))
    for log in logs:
        log.close()
    with open(result_path, "rb") as f:
        rec = pickle.load(f)
    for name in os.listdir(workdir):
        os.unlink(os.path.join(workdir, name))
    os.rmdir(workdir)
    return rec, t0


def run_job(job, ndev, kwargs, backend="nccl", engine_factory=None, timeout=None):
    """Run the generative ``job`` ("sample", "bmdca", "logz" or "design": model_ops.run_job) with ``kwargs`` on ``ndev``
    ranks, one per GPU, and return rank 0's result, which every rank holds."""
    if job not in GENERATIVE_JOBS and ":" not in job:
        raise ValueError("unknown job %r; one of %s" % (job, ", ".join(GENERATIVE_JOBS)))
    rec, _t0 = _start_ranks(job, ndev, {}, args=kwargs, backend=backend, engine_factory=engine_factory,
                            timeout=timeout)
    return rec["value"]


def run_plmc_multi_gpu(ndev, kwargs, return_run=False, backend="nccl", engine_factory=None, timeout=None):
    """Run tools.run_plmc(**kwargs) on ``ndev`` ranks (one per GPU).  ``engine_factory`` ("module:attr") and
    ``backend`` exist for the CPU/gloo test of this plumbing; the product default is the CUDA engine over NCCL."""
    from . import tools
    rec, t0 = _start_ranks("run_plmc", ndev, kwargs, backend=backend, engine_factory=engine_factory,
                           timeout=timeout, label="plmc")
    run = tools.PlmcRun()
    from . import lbfgs as _lbfgs
    run.log, run.timings, run.n_eff = rec["log"], rec["timings"], rec["n_eff"]
    run.lbfgs = _lbfgs.LbfgsResult(*rec["lbfgs"]) if rec["lbfgs"] is not None else None
    run.timings["ranks"] = ndev
    run.timings["launcher_total_s"] = time.time() - t0
    iter_df, fields = tools.parse_plmc_log(run.log)
    k = kwargs
    tools._require_file("plmc returned no couplings", k["couplings_file"])
    if k.get("param_file") is not None:
        tools._require_file("plmc returned no parameter file", k["param_file"])
    result = tools.PlmcResult(k["couplings_file"], k.get("param_file"), iter_df, *fields)
    run.result = result
    if return_run:
        return result, run
    return result
