"""Cost of the generative tools on R ranks, one per GPU (NCCL), for R = 1, 2, 4, 8 as far as the GPUs of the machine
allow.  Per bmDCA update (model_ops.BoltzmannLearner over the ranks), each part timed with CUDA events on rank 0:
sampling (evc_sampler_run of the rank's chains), counts (evc_sampler_codes + evc_code_counts), the all-reduce of the
4n bytes of int32 counts, and the update (evc_bm_update + evc_sampler_set_model); median of --updates updates after
two warm-up updates.  Also the wall time of model_ops.log_partition over the same ranks.  The model is the config-2
synthetic alignment (N = 50 000, L = 200, q = 21) fitted by run_plmc (--fit-iterations caps the fit).  The card's
name, power limit and the device count are read in the same run.  Without a second GPU no speed-up is measured; the
one-rank parts then give the expectation (sampling + counts) / R + update + all-reduce.

    python scripts/generative_ranks_probe.py [--out RESULT.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def rank_job(engine, model, chains, sweeps, updates, temperatures, logz_chains):
    """One rank's timings (launcher job "generative_ranks_probe:rank_job"; also called in-process for R = 1)."""
    import torch
    from evcouplings_b200 import model_ops
    parts = dict(sampling=[], counts=[], allreduce=[], update=[])
    with model_ops.BoltzmannLearner(model, chains, seed=1, engine=engine) as bl:
        bl.run(2, sweeps)                                    # warm-up, including the first collectives
        lib, e = bl.eng.lib, bl.eng
        for _ in range(updates):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
            ev[0].record()
            bl._sweep(sweeps)
            ev[1].record()
            lib.evc_sampler_codes(bl.sampler.handle, e.ptr(bl.codes), e.stream())
            lib.evc_code_counts(e.ptr(bl.codes), bl.hi - bl.lo, bl.L, bl.q, e.ptr(bl.counts), e.stream())
            ev[2].record()
            if bl.world > 1:
                e.all_reduce(bl.counts)
            ev[3].record()
            lib.evc_bm_update(e.ptr(bl.x), e.ptr(bl.counts), bl.n_chains, e.ptr(bl.f), bl.x.numel(), bl.L * bl.q,
                              bl.eta, bl.lam2_h, bl.lam2_J, e.ptr(bl.stats), e.stream())
            lib.evc_sampler_set_model(bl.sampler.handle, e.ptr(bl.x), e.stream())
            ev[4].record()
            ev[4].synchronize()
            for k, (a, b) in zip(parts, ((0, 1), (1, 2), (2, 3), (3, 4))):
                parts[k].append(ev[a].elapsed_time(ev[b]))
        count_bytes = 4 * bl.counts.numel()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    model_ops.log_partition(model, logz_chains, temperatures, temperatures, seed=2, engine=engine)
    torch.cuda.synchronize()
    logz_s = time.perf_counter() - t0
    out = {k + "_ms": float(np.median(v)) for k, v in parts.items()}
    out.update(update_total_ms=sum(out[k + "_ms"] for k in parts), count_bytes=count_bytes, logz_s=logz_s)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", type=int, default=16384)
    ap.add_argument("--sweeps", type=int, default=10)
    ap.add_argument("--updates", type=int, default=5)
    ap.add_argument("--temperatures", type=int, default=128, help="log_partition's K, also its burn-in")
    ap.add_argument("--logz-chains", type=int, default=8192)
    ap.add_argument("--fit-iterations", type=int, default=100)
    ap.add_argument("--out", default=None, help="also write the full result as JSON to this file")
    a = ap.parse_args()
    import torch
    from sampler_probe import card, config2_model
    from evcouplings_b200 import launcher
    from evcouplings_b200.engine import CudaEngine
    eng = CudaEngine()
    ndev = torch.cuda.device_count()
    result = dict(card=card(), device_count=ndev, chains=a.chains, sweeps=a.sweeps, updates=a.updates,
                  temperatures=a.temperatures, logz_chains=a.logz_chains, ranks={})
    model, _fit_s = config2_model(eng, a.fit_iterations)
    kw = dict(model=model, chains=a.chains, sweeps=a.sweeps, updates=a.updates, temperatures=a.temperatures,
              logz_chains=a.logz_chains)
    os.environ["PYTHONPATH"] = os.path.join(ROOT, "scripts") + os.pathsep + os.environ.get("PYTHONPATH", "")
    for R in (1, 2, 4, 8):
        if R > ndev:
            result["ranks"][str(R)] = "not measured: %d GPU%s visible" % (ndev, "" if ndev == 1 else "s")
            print("R = %d: not measured (%d GPU%s visible)" % (R, ndev, "" if ndev == 1 else "s"), flush=True)
            continue
        r = rank_job(eng, **kw) if R == 1 else launcher.run_job("generative_ranks_probe:rank_job", R, kw)
        result["ranks"][str(R)] = r
        print("R = %d: bmDCA update %.2f ms (sampling %.2f, counts %.2f, all-reduce of %.0f MB %.2f, update %.2f); "
              "log_partition %.2f s" % (R, r["update_total_ms"], r["sampling_ms"], r["counts_ms"],
                                         r["count_bytes"] / 1e6, r["allreduce_ms"], r["update_ms"], r["logz_s"]),
              flush=True)
    one = result["ranks"]["1"]
    result["expected_update_ms"] = {
        str(R): "(%.2f + %.2f) / %d + %.2f + all-reduce (not measured)" % (one["sampling_ms"], one["counts_ms"], R,
                                                                          one["update_ms"])
        if not isinstance(result["ranks"][str(R)], dict) else result["ranks"][str(R)]["update_total_ms"]
        for R in (2, 4, 8)}
    result["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(dict(card=result["card"], device_count=ndev, expected_update_ms=result["expected_update_ms"])))


if __name__ == "__main__":
    main()
