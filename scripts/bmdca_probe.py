"""Cost of one Boltzmann-machine update (model_ops.BoltzmannLearner) on the device, split into its three parts:
sampling (evc_sampler_run, S sweeps), counts (evc_sampler_codes + evc_code_counts) and update (evc_bm_update +
evc_sampler_set_model), each timed with CUDA events around every update; median and range of --repeats repeats of
--updates updates.  Models: plmc's PABP model with the -g statistics of its alignment as targets, and the config-2
synthetic alignment (N = 50 000, L = 200, q = 21) fitted by run_plmc (--fit-iterations caps the fit), both at
--chains chains.  Also the PABP trace of the chains' connected-correlation Pearson r over --trace-updates updates.
The card's name and power limit are read in the same run.

    python scripts/bmdca_probe.py [--out RESULT.json]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from sampler_probe import card, config2_model  # noqa: E402


def pabp_model(eng):
    from test_gpu_boltzmann import pabp_model as build
    return build(eng)


def time_updates(eng, model, chains, sweeps, updates, repeats):
    import torch
    from evcouplings_b200 import model_ops
    parts = dict(sampling=[], counts=[], update=[])
    with model_ops.BoltzmannLearner(model, chains, seed=1, engine=eng) as bl:
        bl.run(2, sweeps)                        # warm-up
        for _ in range(repeats):
            acc = dict(sampling=0.0, counts=0.0, update=0.0)
            for _ in range(updates):
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
                ev[0].record()
                bl._sweep(sweeps)
                ev[1].record()
                bl._counts()
                ev[2].record()
                lib = bl.eng.lib
                lib.evc_bm_update(bl.eng.ptr(bl.x), bl.eng.ptr(bl.counts), bl.n_chains, bl.eng.ptr(bl.f),
                                  bl.x.numel(), bl.L * bl.q, bl.eta, bl.lam2_h, bl.lam2_J, bl.eng.ptr(bl.stats),
                                  bl.eng.stream())
                lib.evc_sampler_set_model(bl.sampler.handle, bl.eng.ptr(bl.x), bl.eng.stream())
                ev[3].record()
                ev[3].synchronize()
                acc["sampling"] += ev[0].elapsed_time(ev[1])
                acc["counts"] += ev[1].elapsed_time(ev[2])
                acc["update"] += ev[2].elapsed_time(ev[3])
            for k in acc:
                parts[k].append(acc[k] / updates)
    out = {}
    for k, v in parts.items():
        out[k + "_ms"] = dict(median=float(np.median(v)), min=float(min(v)), max=float(max(v)), repeats=v)
    total = sum(out[k + "_ms"]["median"] for k in parts)
    out["counts_and_update_share"] = (out["counts_ms"]["median"] + out["update_ms"]["median"]) / total
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", type=int, default=16384)
    ap.add_argument("--sweeps", type=int, default=10)
    ap.add_argument("--updates", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--trace-updates", type=int, default=100)
    ap.add_argument("--fit-iterations", type=int, default=100)
    ap.add_argument("--out", default=None, help="also write the full result as JSON to this file")
    a = ap.parse_args()
    from evcouplings_b200 import model_ops
    from evcouplings_b200.engine import CudaEngine
    eng = CudaEngine()
    result = dict(card=card(), chains=a.chains, sweeps=a.sweeps, updates=a.updates, models={})
    pabp = pabp_model(eng)
    c2, fit_s = config2_model(eng, a.fit_iterations)
    for name, model in (("pabp_L82_q20", pabp), ("config2_L200_q21", c2)):
        entry = dict(L=model["L"], q=model["q"], **time_updates(eng, model, a.chains, a.sweeps, a.updates, a.repeats))
        if name.startswith("config2"):
            entry["fit_seconds"], entry["fit_iterations_cap"] = fit_s, a.fit_iterations
        result["models"][name] = entry
        print("%s: sampling %.3f ms, counts %.3f ms, update %.3f ms per update (medians); counts + update %.2f %%"
              % (name, entry["sampling_ms"]["median"], entry["counts_ms"]["median"], entry["update_ms"]["median"],
                 100 * entry["counts_and_update_share"]), flush=True)
    trace = []
    with model_ops.BoltzmannLearner(pabp, a.chains, seed=0, burn_in=100, engine=eng) as bl:
        bl.run(a.trace_updates, a.sweeps, progress=lambda k, st: trace.append(dict(update=k, **st)))
    result["pabp_trace"] = trace
    for t in trace[::10] + [trace[-1]]:
        print("PABP update %3d: pearson %.4f, max|dfi| %.4g, max|dfij| %.4g" % (
            t["update"], t["connected_pearson"], t["max_field_dev"], t["max_coupling_dev"]), flush=True)
    result["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
