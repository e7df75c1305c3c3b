"""
Alphabet-size probe (one GPU, one call; a measurement, not a test): ms per objective + gradient evaluation on the
default tensor-core path at N = 50,000 sequences, L = 200 sites for q in {2, 6, 21, 22, 32} model states (gap as a
state, precision fp32).  The five problems are set up once and alternated, median of 3 rounds of 20 timed
evaluations each (CUDA events), after 5 warm-up evaluations.  The GEMMs grow as (L q)^2, so the ratio to q = 21 is
reported next to (q / 21)^2.

The card's name and power limit are read in the same run (read-only nvidia-smi query).

    python scripts/alphabet_probe.py OUTDIR
"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from evcouplings_b200.engine import CudaEngine  # noqa: E402

QS = (2, 6, 21, 22, 32)
N, L = 50000, 200


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip()


def codes_for(q, seed):
    """family-structured codes over q states: 1000 centres, per-sequence mutation probability U(0.1, 0.6)"""
    rng = np.random.default_rng(seed)
    centres = rng.integers(0, q, size=(1000, L))
    codes = centres[rng.integers(0, 1000, size=N)]
    mut = rng.random((N, L)) < rng.uniform(0.1, 0.6, size=N)[:, None]
    return np.ascontiguousarray(np.where(mut, rng.integers(0, q, size=(N, L)), codes).astype(np.uint8))


def time_evals(torch, p, steps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(steps):
        p.evaluate_async(p.x)
    ev[1].record()
    ev[1].synchronize()
    return ev[0].elapsed_time(ev[1]) / steps


def main():
    if len(sys.argv) != 2:
        sys.exit("usage: python scripts/alphabet_probe.py OUTDIR")
    outdir = sys.argv[1]
    os.makedirs(outdir, exist_ok=True)
    import torch
    res = {"card": card(), "N": N, "L": L}
    print(res["card"], flush=True)
    eng = CudaEngine()
    probs = {}
    for q in QS:
        rng = np.random.default_rng(q)
        w = rng.uniform(0.05, 1.0, N).astype(np.float32)
        x = rng.normal(0, 0.05, L * q + L * (L - 1) // 2 * q * q).astype(np.float32)
        p = eng.plm_problem(codes_for(q, q), w, q, -1, 0.01, 2.0, forward="tc", precision="fp32", seq_chunk=0)
        p.set_x(x)
        time_evals(torch, p, 5)
        probs[q] = p
    times = {q: [] for q in QS}
    for _ in range(3):
        for q in QS:
            times[q].append(time_evals(torch, probs[q], 20))
    med21 = float(np.median(times[21]))
    out = {}
    for q in QS:
        med = float(np.median(times[q]))
        out["q%d" % q] = dict(q=q, device_bytes=probs[q].device_bytes(), ms_per_eval_runs=times[q],
                              ms_per_eval_median=med, ratio_to_q21=med / med21, gemm_ratio_q_over_21_sq=(q / 21.0) ** 2)
        probs[q].close()
    res["evaluations"] = out
    res["card_after"] = card()
    path = os.path.join(outdir, "alphabet_probe.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))
    print("wrote", path)


if __name__ == "__main__":
    main()
