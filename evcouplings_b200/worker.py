"""One rank of a multi-GPU run started by evcouplings_b200.launcher (``python -m evcouplings_b200.worker SPEC``): the
spec's job ("run_plmc", the default, or a generative job of model_ops.run_job) with its engine in the process group;
rank 0 stores the result for the launcher."""
import importlib
import json
import os
import pickle
import sys


def main(argv=None):
    argv = sys.argv[1:] if argv is None else argv
    with open(argv[0]) as f:
        spec = json.load(f)
    from evcouplings_b200.tools import _trace
    _trace("worker start")
    import torch
    import torch.distributed as dist
    _trace("torch imported")
    if spec["kwargs"].get("checkpoint"):
        # stop at the next iteration boundary with the state saved, instead of dying inside a collective
        import signal
        from evcouplings_b200 import checkpoint
        signal.signal(signal.SIGTERM, checkpoint.request_stop)
        signal.signal(signal.SIGUSR1, checkpoint.request_stop)
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local_rank = int(os.environ.get("LOCAL_RANK", rank))
    backend = spec.get("backend") or "nccl"
    if backend == "nccl":
        torch.cuda.set_device(local_rank)
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local_rank))
    else:
        dist.init_process_group(backend, rank=rank, world_size=world)
    _trace("process group ready")
    from evcouplings_b200 import tools
    try:
        factory = spec.get("engine_factory")
        if factory:
            mod, attr = factory.split(":")
            engine = getattr(importlib.import_module(mod), attr)()
        else:
            from evcouplings_b200.engine import CudaEngine
            engine = CudaEngine()
        job = spec.get("job") or "run_plmc"
        if job == "run_plmc":
            result, run = tools.run_plmc(engine=engine, return_run=True, **spec["kwargs"])
            rec = dict(log=run.log, timings=run.timings, n_eff=run.n_eff,
                       lbfgs=tuple(run.lbfgs) if run.lbfgs is not None else None)
        else:
            kwargs = dict(spec["kwargs"])
            if spec.get("args"):
                with open(spec["args"], "rb") as f:
                    kwargs.update(pickle.load(f))
            if ":" in job:                  # "module:function", a stand-in job for tests of this plumbing
                mod, attr = job.split(":")
                rec = dict(value=getattr(importlib.import_module(mod), attr)(engine, **kwargs))
            else:
                from evcouplings_b200 import model_ops
                rec = dict(value=model_ops.run_job(job, engine, **kwargs))
        if rank == 0:
            with open(spec["result"], "wb") as f:
                pickle.dump(rec, f, protocol=pickle.HIGHEST_PROTOCOL)
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
