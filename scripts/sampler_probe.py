"""Throughput of the Gibbs sampler (evc_sampler_run) on the device, with the float64 CPU restatement for scale.

Models: plmc's PABP model (L = 82, q = 20, from tests/golden) and a model fitted with run_plmc on the config-2
synthetic alignment (N = 50 000, L = 200, q = 21; --fit-iterations caps its fit).  For 16 384 and 65 536 chains: a
warm-up, then --sweeps timed sweeps with CUDA events, --repeats times.  Reported per repeat: chain-sweeps per second,
the measured change rate (site changes per chain-sweep) and the algorithmic bytes those imply: 8 L q per change (the
two coupling rows a change streams) plus the refresh, L rows of 4 L q bytes per chain every EVC_SAMPLER_REFRESH
sweeps, over the time.  The card's name and power limit are read in the same run.

    python scripts/sampler_probe.py [--out RESULT.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

REFRESH = 32


def card():
    import torch
    out = dict(name=torch.cuda.get_device_name(0))
    try:
        out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                            capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out["power_limit"] = "not read: %s" % e
    return out


def pabp_model():
    import golden_npz
    g = golden_npz.load("pabp_golden")
    return dict(L=82, q=20, h=g["h"], J=g["J"], alphabet=str(g["alphabet"]), target_seq=str(g["target_seq"]))


def config2_model(eng, iterations):
    from evcouplings_b200 import model_ops, synthetic, tools
    N, L, seed = synthetic.CONFIG_SEEDS[2]
    with tempfile.TemporaryDirectory() as td:
        a2m = os.path.join(td, "c2.a2m")
        synthetic.write_a2m(a2m, synthetic.synthetic_msa_codes(N, L, seed))
        t0 = time.time()
        tools.run_plmc(a2m, os.path.join(td, "c2_ECs.txt"), os.path.join(td, "c2.model"), focus_seq="seq0",
                       iterations=iterations, engine=eng)
        fit_s = time.time() - t0
        return model_ops.read_model(os.path.join(td, "c2.model")), fit_s


def time_sampler(eng, model, n_chains, sweeps, warmup, repeats):
    import torch
    from evcouplings_b200 import model_ops
    L, q = model["L"], model["q"]
    rows = []
    with model_ops.PottsSampler(model, n_chains, seed=1, engine=eng) as s:
        s.run(warmup)
        t = warmup                              # global index of the next sweep
        for _ in range(repeats):
            start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            changes = s.run(sweeps)             # synchronises the stream to return the count
            stop.record()
            stop.synchronize()
            sec = start.elapsed_time(stop) / 1e3
            refreshes = sum(1 for k in range(t, t + sweeps) if k % REFRESH == 0)
            t += sweeps
            bytes_ = 8.0 * L * q * changes + refreshes * n_chains * 4.0 * L * L * q
            rows.append(dict(seconds=sec, chain_sweeps_per_s=n_chains * sweeps / sec,
                             changes_per_chain_sweep=changes / (n_chains * sweeps),
                             change_rate_per_site=changes / (n_chains * sweeps * L),
                             algorithmic_bytes=bytes_, algorithmic_GB_per_s=bytes_ / sec / 1e9))
    return rows


def cpu_rate(model, chains=256, sweeps=2):
    from oracle import potts_sampler as ps
    s = ps.Sampler(model["h"], model["J"], 1, chains)
    t0 = time.time()
    s.run(sweeps)
    return chains * sweeps / (time.time() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweeps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--fit-iterations", type=int, default=100)
    ap.add_argument("--out", default=None, help="also write the full result as JSON to this file")
    a = ap.parse_args()
    from evcouplings_b200.engine import CudaEngine
    eng = CudaEngine()
    result = dict(card=card(), sweeps=a.sweeps, warmup=a.warmup, models={})
    c2, fit_s = config2_model(eng, a.fit_iterations)
    for name, model in (("pabp_L82_q20", pabp_model()), ("config2_L200_q21", c2)):
        entry = dict(L=model["L"], q=model["q"], cpu_restatement_chain_sweeps_per_s=cpu_rate(model), chains={})
        if name.startswith("config2"):
            entry["fit_seconds"], entry["fit_iterations_cap"] = fit_s, a.fit_iterations
        for n in (16384, 65536):
            entry["chains"][str(n)] = time_sampler(eng, model, n, a.sweeps, a.warmup, a.repeats)
            r = [x["chain_sweeps_per_s"] for x in entry["chains"][str(n)]]
            print("%s chains=%d: %.3g chain-sweeps/s (min %.3g, max %.3g), %.1f changes/chain-sweep, %.0f GB/s"
                  % (name, n, np.median(r), min(r), max(r), entry["chains"][str(n)][0]["changes_per_chain_sweep"],
                     np.median([x["algorithmic_GB_per_s"] for x in entry["chains"][str(n)]])), flush=True)
        result["models"][name] = entry
    result["card"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
