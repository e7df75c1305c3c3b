"""Throughput of design (evc_sampler_record_best, evc_sampler_descend) and the best H against annealing length.

Models as in sampler_probe.py: plmc's PABP model (L = 82, q = 20, from tests/golden) and a model fitted with run_plmc
on the config-2 synthetic alignment (N = 50 000, L = 200, q = 21; --fit-iterations caps its fit).  At --chains chains
(default 16 384):
    record off / on   evc_sampler_run at beta = 1 on two handles, one recording (RECORD instantiation): after a
                      warm-up, --repeats rounds in which each times --sweeps sweeps with CUDA events, alternating;
                      median and range of chain-sweeps per second,
    descent moving    the first --descent-sweeps descent sweeps from the sampled states (chains still changing),
    descent settled   --descent-sweeps more sweeps once every chain has settled (no site changes),
    anneal S          design_codes with beta_start = 0.1, beta = 1, S annealing sweeps: the best and the median H of
                      the designs and the wall time (host loop of one launch per sweep, descent and scoring included).
The card's name and power limit are read in the same run.

    python scripts/design_probe.py [--out RESULT.json]
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

from sampler_probe import card, config2_model, pabp_model  # noqa: E402
from tempering_probe import timed  # noqa: E402


def recording(eng, model, n, sweeps, warmup, repeats):
    from evcouplings_b200 import model_ops
    rows = {"off": [], "on": []}
    with model_ops.PottsSampler(model, n, seed=1, init="target", engine=eng) as off, \
            model_ops.PottsSampler(model, n, seed=1, init="target", engine=eng) as on:
        on.record_best()
        off.run(warmup)
        on.run(warmup)
        for _ in range(repeats):
            for name, s in (("off", off), ("on", on)):
                rows[name].append(n * sweeps / timed(lambda s=s: s.run(sweeps)))
        assert np.array_equal(off.codes(), on.codes())
    out = {k: dict(median=float(np.median(v)), min=float(min(v)), max=float(max(v))) for k, v in rows.items()}
    out["on_relative_to_off"] = out["on"]["median"] / out["off"]["median"]
    return out


def descent(eng, model, n, sweeps):
    from evcouplings_b200 import model_ops
    with model_ops.PottsSampler(model, n, seed=2, engine=eng) as s:
        s.run(10)
        s.descend(1)                                  # warm-up of the descent kernel
        res = {}
        out = {}
        res["moving"] = n * sweeps / timed(lambda: out.update(m=s.descend(sweeps)))
        moving_changes = out["m"][1]
        for _ in range(64):
            settled, ch = s.descend(sweeps)
            if settled.all() and ch == 0:
                break
        res["settled"] = n * sweeps / timed(lambda: out.update(s=s.descend(sweeps)))
    return dict(moving_chain_sweeps_per_s=res["moving"], moving_changes_per_chain_sweep=moving_changes / (n * sweeps),
                settled_chain_sweeps_per_s=res["settled"], settled_changes=out["s"][1])


def anneal_curve(eng, model, n, lengths):
    from evcouplings_b200 import model_ops
    rows = []
    for S in lengths:
        t0 = time.time()
        r = model_ops.design_codes(model, n, S, seed=3, beta_start=0.1, beta=1.0, engine=eng)
        rows.append(dict(sweeps=S, best_H=float(r["energy"].max()), median_H=float(np.median(r["energy"])),
                         settled=float(r["settled"].mean()), seconds=time.time() - t0))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", type=int, default=16384)
    ap.add_argument("--sweeps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--descent-sweeps", type=int, default=32, dest="descent_sweeps")
    ap.add_argument("--anneal", default="10,100,1000", help="annealing lengths (sweeps) of the best-H curve")
    ap.add_argument("--fit-iterations", type=int, default=100)
    ap.add_argument("--out", default=None, help="also write the full result as JSON to this file")
    a = ap.parse_args()
    from evcouplings_b200.engine import CudaEngine
    eng = CudaEngine()
    result = dict(card=card(), chains=a.chains, sweeps=a.sweeps, repeats=a.repeats, models={})
    c2, _fit_s = config2_model(eng, a.fit_iterations)
    pabp = pabp_model()
    pabp["index_list"] = np.arange(1, pabp["L"] + 1)
    for name, model in (("pabp_L82_q20", pabp), ("config2_L200_q21", c2)):
        r = dict(L=model["L"], q=model["q"])
        r["recording"] = recording(eng, model, a.chains, a.sweeps, a.warmup, a.repeats)
        print(name, "recording", json.dumps(r["recording"]), flush=True)
        r["descent"] = descent(eng, model, a.chains, a.descent_sweeps)
        print(name, "descent", json.dumps(r["descent"]), flush=True)
        r["anneal"] = anneal_curve(eng, model, a.chains, [int(x) for x in a.anneal.split(",")])
        print(name, "anneal", json.dumps(r["anneal"]), flush=True)
        result["models"][name] = r
    result["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
