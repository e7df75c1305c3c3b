"""What working on distinct rows saves, and what the distinct pass costs (GPU).

    python scripts/unique_rows_probe.py [--rounds 3] [--iterations 100] [--evals 20]

PABP (tests/golden/pabp_codes: 151,496 valid rows, 70,300 distinct over 82 columns, q = 20 with the gap ignored):
    reweight_ms        the Hamming reweighting on the full rows, and on the distinct rows with multiplicities
                       (distinct: evc_msa_unique plus the weighted pass; unique_ms is the distinct pass alone)
    eval_ms            one objective + gradient evaluation at plmc's optimum, full rows vs distinct rows
    run_plmc_s         the whole run_plmc (alignment file to output files) at --iterations iterations, full rows vs
                       distinct rows (the full-row run uses an engine that reports every row as distinct)
Config 2 (synthetic, N = 50,000, L = 200, no repeats):
    unique_share       the distinct pass's seconds over run_plmc's total at --iterations iterations

Every figure is the median of --rounds rounds in which the compared variants alternate.  Card name and power limit
are read in the same process.  Prints one JSON line."""
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
from evcouplings_b200 import msa, synthetic, tools  # noqa: E402
from evcouplings_b200.engine import CudaEngine  # noqa: E402
import golden_npz  # noqa: E402


class FullRowsEngine(CudaEngine):
    """Reports every row as distinct: run_plmc takes the full-row path."""

    def unique_rows(self, codes):
        n = len(codes)
        return np.arange(n), np.arange(n), np.ones(n, dtype=np.int64)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iterations", type=int, default=100)
    ap.add_argument("--evals", type=int, default=20)
    a = ap.parse_args()
    eng, full_eng = CudaEngine(), FullRowsEngine()
    c = golden_npz.load("pabp_codes")
    g = golden_npz.load("pabp_golden")
    codes = np.ascontiguousarray(c["codes"])
    L, q = codes.shape[1], 20
    thr = msa.identity_threshold_count(0.8, L)
    res = dict(card=card(), pabp_rows=len(codes))

    def distinct_pass():
        return eng.unique_rows(codes)

    def reweight_distinct():
        first, inverse, mult = eng.unique_rows(codes)
        return eng.hamming_counts(codes[first], thr, mult=mult)[inverse]

    first, inverse, mult = distinct_pass()
    res["pabp_distinct_rows"] = len(first)
    ref = eng.hamming_counts(codes, thr)
    assert np.array_equal(reweight_distinct(), ref)                         # warm-up and check
    rw = {"full": [], "distinct": [], "unique": []}
    for _ in range(a.rounds):
        rw["full"].append(timed(lambda: eng.hamming_counts(codes, thr))[0])
        rw["distinct"].append(timed(reweight_distinct)[0])
        rw["unique"].append(timed(distinct_pass)[0])
    res["reweight_ms"] = {k: 1e3 * float(np.median(rw[k])) for k in ("full", "distinct")}
    res["unique_ms"] = 1e3 * float(np.median(rw["unique"]))

    # one evaluation at plmc's optimum
    w = 1.0 / ref.astype(np.float64)
    x = np.concatenate([g["h"].ravel(), g["J"].ravel()]).astype(np.float32)
    probs = {"full": eng.plm_problem(codes, w.astype(np.float32), q, q, 0.01, 16.2),
             "distinct": eng.plm_problem(codes[first], (mult * w[first]).astype(np.float32), q, q, 0.01, 16.2)}
    ev = {k: [] for k in probs}
    fx = {}
    for p in probs.values():
        p.set_x(x)
        p.evaluate(p.x)
    for _ in range(a.rounds):
        for k, p in probs.items():
            def run(p=p):
                for _ in range(a.evals):
                    p.evaluate_async(p.x)
            ev[k].append(timed(run)[0] / a.evals)
            fx[k] = p.evaluate(p.x)
    for p in probs.values():
        p.close()
    res["eval_ms"] = {k: 1e3 * float(np.median(v)) for k, v in ev.items()}
    res["eval_fx"] = fx

    # whole run_plmc
    with tempfile.TemporaryDirectory() as td:
        a2m = os.path.join(td, "pabp.a2m")
        synthetic.write_a2m(a2m, np.where(codes == q, 0, codes + 1).astype(np.uint8))
        kw = dict(alignment=a2m, theta=0.8, ignore_gaps=True, iterations=a.iterations, lambda_h=0.01, lambda_J=16.2)
        runs = {"full": [], "distinct": []}
        for r in range(a.rounds + 1):                                         # round 0 warms up
            for k, e in (("full", full_eng), ("distinct", eng)):
                t, (out, run) = timed(lambda: tools.run_plmc(couplings_file=os.path.join(td, k + "_ECs.txt"),
                                                             param_file=os.path.join(td, k + ".model"), engine=e,
                                                             return_run=True, **kw))
                if r:
                    runs[k].append(t)
                res.setdefault("run_plmc_unique_rows", {})[k] = run.timings["unique_rows"]
        res["run_plmc_s"] = {k: float(np.median(v)) for k, v in runs.items()}

        # config 2: no repeats, the distinct pass is pure overhead
        N2, L2, seed = synthetic.CONFIG_SEEDS[2]
        c2 = synthetic.synthetic_msa_codes(N2, L2, seed)
        a2m2 = os.path.join(td, "cfg2.a2m")
        synthetic.write_a2m(a2m2, c2)
        kw2 = dict(alignment=a2m2, focus_seq="seq0/1-%d" % L2, theta=0.8, iterations=a.iterations, lambda_h=0.01,
                   lambda_J=0.01 * (L2 - 1) * 20)
        shares, uniq, total = [], [], []
        for r in range(a.rounds + 1):
            out, run = tools.run_plmc(couplings_file=os.path.join(td, "c2_ECs.txt"), engine=eng, return_run=True,
                                      **kw2)
            if r:
                shares.append(run.timings["unique_s"] / run.timings["total_s"])
                uniq.append(run.timings["unique_s"])
                total.append(run.timings["total_s"])
        res["config2"] = dict(rows=N2, distinct_rows=run.timings["unique_rows"], unique_s=float(np.median(uniq)),
                              total_s=float(np.median(total)), unique_share=float(np.median(shares)))
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
