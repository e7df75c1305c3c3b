"""Annealed importance sampling on the device (evc_sampler_anneal, model_ops.log_partition): cost and quality.

Models: plmc's PABP model (L = 82, q = 20, from tests/golden) and a model fitted with run_plmc on the config-2
synthetic alignment (N = 50 000, L = 200, q = 21; --fit-iterations caps its fit), as in scripts/sampler_probe.py.
  * annealed against plain chain-sweeps per second at 16 384 chains, both at beta = 1 so that both change the same
    sites: a warm-up, then --sweeps sweeps timed with CUDA events, --repeats times, the two kinds alternating;
    median and range;
  * wall time of log_partition at the command line's defaults (M = 8192, K = 1024, burn-in K), --repeats times;
  * the forward and reverse estimates, their ESS and their gap for K = 256, 1024 and 4096 (--gap-chains chains).
The card's name and power limit are read in the same run.

    python scripts/ais_probe.py [--out RESULT.json]
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

from sampler_probe import card, config2_model, pabp_model  # noqa: E402


def timed(fn):
    import torch
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / 1e3


def sweep_rates(eng, model, n_chains, sweeps, warmup, repeats):
    """chain-sweeps/s of plain sweeps at beta = 1 and annealed sweeps at a constant beta = 1 (the same target, so the
    same change rate and coupling-row traffic) on one handle, alternating; and the site changes per chain-sweep of
    each."""
    from evcouplings_b200 import model_ops
    ones = np.ones(sweeps + 1, dtype=np.float32)
    plain, annealed, changes = [], [], [0, 0]
    with model_ops.PottsSampler(model, n_chains, seed=1, engine=eng) as s:
        s.run(warmup)
        s.anneal(ones[:warmup + 1])
        for _ in range(repeats):
            box = []
            plain.append(n_chains * sweeps / timed(lambda: box.append(s.run(sweeps))))
            annealed.append(n_chains * sweeps / timed(lambda: box.append(s.anneal(ones))))
            changes[0] += box[0]
            changes[1] += box[1]
    per = float(n_chains * sweeps * repeats)
    return plain, annealed, (changes[0] / per, changes[1] / per)


def summary(v):
    return dict(median=float(np.median(v)), min=float(min(v)), max=float(max(v)), all=[float(x) for x in v])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweeps", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--fit-iterations", type=int, default=100)
    ap.add_argument("--gap-chains", type=int, default=2048)
    ap.add_argument("--out", default=None, help="also write the full result as JSON to this file")
    a = ap.parse_args()
    from evcouplings_b200 import logz_cli, model_ops
    from evcouplings_b200.engine import CudaEngine
    eng = CudaEngine()
    result = dict(card=card(), models={})
    c2, fit_s = config2_model(eng, a.fit_iterations)
    for name, model in (("pabp_L82_q20", pabp_model()), ("config2_L200_q21", c2)):
        entry = dict(L=model["L"], q=model["q"])
        plain, annealed, changes = sweep_rates(eng, model, 16384, a.sweeps, a.warmup, a.repeats)
        entry["plain_chain_sweeps_per_s"], entry["annealed_chain_sweeps_per_s"] = summary(plain), summary(annealed)
        entry["changes_per_chain_sweep"] = dict(plain=changes[0], annealed=changes[1])
        print("%s 16384 chains at beta = 1: plain %.3g chain-sweeps/s (%.3g..%.3g), annealed %.3g (%.3g..%.3g): "
              "ratio %.3f; changes per chain-sweep %.2f and %.2f"
              % (name, np.median(plain), min(plain), max(plain), np.median(annealed), min(annealed), max(annealed),
                 np.median(annealed) / np.median(plain), changes[0], changes[1]), flush=True)
        walls = []
        for _ in range(a.repeats):
            t0 = time.time()
            r = model_ops.log_partition(model, logz_cli.DEFAULT_CHAINS, logz_cli.DEFAULT_TEMPERATURES, engine=eng)
            walls.append(time.time() - t0)
        entry["log_partition_defaults"] = dict(seconds=summary(walls), result=r)
        print("%s log_partition(M=%d, K=%d, burn-in K): %.2f s (%.2f..%.2f); forward %.5f reverse %.5f gap %.4f"
              % (name, logz_cli.DEFAULT_CHAINS, logz_cli.DEFAULT_TEMPERATURES, np.median(walls), min(walls),
                 max(walls), r["log_z"], r["log_z_reverse"], r["log_z_reverse"] - r["log_z"]), flush=True)
        entry["gap"] = {}
        for K in (256, 1024, 4096):
            r = model_ops.log_partition(model, a.gap_chains, K, engine=eng)
            entry["gap"][str(K)] = r
            print("%s K=%d (%d chains): forward %.5f (ESS %.0f, se %.2e) reverse %.5f (ESS %.0f, se %.2e) gap %.4f"
                  % (name, K, a.gap_chains, r["log_z"], r["ess"], r["stderr"], r["log_z_reverse"], r["ess_reverse"],
                     r["stderr_reverse"], r["log_z_reverse"] - r["log_z"]), flush=True)
        if name.startswith("config2"):
            entry["fit_seconds"], entry["fit_iterations_cap"] = fit_s, a.fit_iterations
        result["models"][name] = entry
    result["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
