"""One rank of a multi-GPU run started by evcouplings_b200.launcher (``python -m evcouplings_b200.worker SPEC``)."""
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
        result, run = tools.run_plmc(engine=engine, return_run=True, **spec["kwargs"])
        if rank == 0:
            with open(spec["result"], "wb") as f:
                pickle.dump(dict(log=run.log, timings=run.timings, n_eff=run.n_eff,
                                 lbfgs=tuple(run.lbfgs) if run.lbfgs is not None else None), f)
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
