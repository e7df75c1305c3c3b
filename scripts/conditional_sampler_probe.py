"""Throughput of conditional sampling (evc_sampler_create_conditional) against the plain sampler (evc_sampler_run).

Models as in sampler_probe.py: plmc's PABP model (L = 82, q = 20, from tests/golden) and a model fitted with run_plmc
on the config-2 synthetic alignment (N = 50 000, L = 200, q = 21; --fit-iterations caps its fit).  At --chains chains
(default 16 384) and beta = 1 the variants are
    plain       evc_sampler_run on the whole model,
    all_free    a conditional handle with every site free (it moves the same bytes as plain),
    free_10, free_20, free_50   a window of that many sites centred in the model, every other site clamped at the
                target sequence.
Every handle runs a warm-up, then --repeats rounds in which each variant in turn times --sweeps sweeps with CUDA
events, so the variants alternate.  Reported per timing: chain-sweeps per second, the change rate (site changes per
chain-sweep) and the algorithmic bytes: 8 F q per change (the two coupling rows) plus F rows of 4 F q bytes per chain
at each refresh (F = L for plain), over the time.  create_s is the host time of the synchronising create call:
allocation, the coupling build and, for a conditional handle, the fold.  The card's name and power limit are read in
the same run.

    python scripts/conditional_sampler_probe.py [--out RESULT.json]
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
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from sampler_probe import REFRESH, card, config2_model, pabp_model  # noqa: E402


def variants(model):
    L = model["L"]
    index = list(model["index_list"])
    out = [("plain", None), ("all_free", index)]
    for F in (10, 20, 50):
        lo = (L - F) // 2
        out.append(("free_%d" % F, index[lo:lo + F]))
    return out


def run_model(eng, model, n_chains, sweeps, warmup, repeats):
    import torch
    from evcouplings_b200 import model_ops
    L, q = model["L"], model["q"]
    handles, rows = {}, {}
    try:
        for name, free in variants(model):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            s = model_ops.PottsSampler(model, n_chains, seed=1, init="target", engine=eng, free=free)
            torch.cuda.synchronize()
            F = L if free is None else len(free)
            handles[name] = (s, F)
            rows[name] = dict(free_sites=F, create_s=time.perf_counter() - t0, timings=[])
            s.run(warmup)
        t = warmup
        for _ in range(repeats):
            refreshes = sum(1 for k in range(t, t + sweeps) if k % REFRESH == 0)
            for name, (s, F) in handles.items():
                start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                start.record()
                changes = s.run(sweeps)
                stop.record()
                stop.synchronize()
                sec = start.elapsed_time(stop) / 1e3
                bytes_ = 8.0 * F * q * changes + refreshes * n_chains * 4.0 * F * F * q
                rows[name]["timings"].append(dict(
                    seconds=sec, chain_sweeps_per_s=n_chains * sweeps / sec,
                    changes_per_chain_sweep=changes / (n_chains * sweeps),
                    change_rate_per_free_site=changes / (n_chains * sweeps * F),
                    algorithmic_bytes=bytes_, algorithmic_GB_per_s=bytes_ / sec / 1e9))
            t += sweeps
    finally:
        for s, _ in handles.values():
            s.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", type=int, default=16384)
    ap.add_argument("--sweeps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--fit-iterations", type=int, default=100)
    ap.add_argument("--out", default=None, help="also write the full result as JSON to this file")
    a = ap.parse_args()
    from evcouplings_b200.engine import CudaEngine
    eng = CudaEngine()
    result = dict(card=card(), chains=a.chains, sweeps=a.sweeps, warmup=a.warmup, beta=1.0, models={})
    c2, fit_s = config2_model(eng, a.fit_iterations)
    pabp = pabp_model()
    pabp["index_list"] = np.arange(1, pabp["L"] + 1)
    for name, model in (("pabp_L82_q20", pabp), ("config2_L200_q21", c2)):
        rows = run_model(eng, model, a.chains, a.sweeps, a.warmup, a.repeats)
        result["models"][name] = dict(L=model["L"], q=model["q"], variants=rows)
        if name.startswith("config2"):
            result["models"][name].update(fit_seconds=fit_s, fit_iterations_cap=a.fit_iterations)
        for v, r in rows.items():
            rate = [x["chain_sweeps_per_s"] for x in r["timings"]]
            print("%s %s (F=%d): %.4g chain-sweeps/s (min %.4g, max %.4g), %.2f changes/chain-sweep, %.0f GB/s, "
                  "create %.3f s" % (name, v, r["free_sites"], np.median(rate), min(rate), max(rate),
                                     r["timings"][0]["changes_per_chain_sweep"],
                                     np.median([x["algorithmic_GB_per_s"] for x in r["timings"]]), r["create_s"]),
                  flush=True)
    result["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
