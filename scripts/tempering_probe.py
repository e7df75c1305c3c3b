"""Throughput of replica exchange (evc_sampler_temper) against the plain sampler (evc_sampler_run), the swap kernel's
share of the time, the acceptance of a geometric ladder and the round trips on the Curie-Weiss Potts model.

Models as in sampler_probe.py: plmc's PABP model (L = 82, q = 20, from tests/golden) and a model fitted with run_plmc
on the config-2 synthetic alignment (N = 50 000, L = 200, q = 21; --fit-iterations caps its fit).  At --chains chains
(default 16 384) the variants are
    plain        evc_sampler_run at beta = 1,
    R8, R16      ladders of 8 or 16 rungs, geometric from beta = 0.5 to 1, a swap round after every sweep,
    R8_narrow    a ladder of 8 rungs from beta = 0.99 to 1, a swap round after every sweep: the change rate of plain,
                 so it isolates the cost of the tempering itself (a launch per swap interval, the energies, the swaps)
                 from that of the extra site changes a hotter rung makes,
    R8_narrow_k100  the same ladder with a swap round every 100 sweeps: one sweep launch per timed call, as plain.
Every handle runs a warm-up, then --repeats rounds in which each variant in turn times --sweeps sweeps with CUDA
events, so the variants alternate; reported are the median and range of chain-sweeps per second.  The swap kernel's
share is its device time over all kernels' in one more --sweeps call of each ladder, from torch.profiler.  The
acceptance per pair is over all the ladder's rounds.  Curie-Weiss (q = 3, L = 16, K = 1/2, the ladder of
tests/test_tempering_oracle.py): round trips per ladder per 1 000 sweeps after a 1 000-sweep warm-up.  The card's
name and power limit are read in the same run.

    python scripts/tempering_probe.py [--out RESULT.json]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from sampler_probe import card, config2_model, pabp_model  # noqa: E402


def timed(fn):
    import torch
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / 1e3


def swap_share(s, sweeps):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        s.temper(sweeps)
        import torch
        torch.cuda.synchronize()
    total = swap = 0.0
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if "kernel" in ev.key:
            total += t
            if "swap" in ev.key:
                swap += t
    return swap / total if total else float("nan")


def run_model(eng, model, n_chains, sweeps, warmup, repeats):
    from evcouplings_b200 import model_ops
    handles, rows = {}, {}
    try:
        for name, R, lo, k in (("plain", None, None, None), ("R8", 8, 0.5, 1), ("R16", 16, 0.5, 1),
                               ("R8_narrow", 8, 0.99, 1), ("R8_narrow_k100", 8, 0.99, 100)):
            s = model_ops.PottsSampler(model, n_chains, seed=1, init="target", engine=eng)
            handles[name] = s
            rows[name] = dict(timings=[], swap_interval=k)
            if R:
                s.set_ladder(model_ops.geometric_ladder(lo, 1.0, R), k)
                s.temper(warmup)
            else:
                s.run(warmup)
        for _ in range(repeats):
            for name, s in handles.items():
                out = {}
                sec = timed((lambda s=s: out.update(c=s.run(sweeps))) if name == "plain" else
                            (lambda s=s: out.update(c=s.temper(sweeps))))
                rows[name]["timings"].append(dict(seconds=sec, chain_sweeps_per_s=n_chains * sweeps / sec,
                                                  changes_per_chain_sweep=out["c"] / (n_chains * sweeps)))
        for name, s in handles.items():
            r = rows[name]
            rate = [x["chain_sweeps_per_s"] for x in r["timings"]]
            r.update(median=float(np.median(rate)), min=float(min(rate)), max=float(max(rate)),
                     changes_per_chain_sweep=float(np.median([x["changes_per_chain_sweep"] for x in r["timings"]])))
            if name != "plain":
                r["swap_kernel_share"] = swap_share(s, sweeps)
                st = s.swap_statistics()
                r["ladder"] = [float(b) for b in s.ladder]
                r["acceptance"] = [float(a) for a in st["acceptance"]]
                r["round_trips_per_ladder"] = float(st["round_trips"].mean())
                r["relative_to_plain"] = r["median"] / rows["plain"]["median"]
    finally:
        for s in handles.values():
            s.close()
    return rows


def curie_weiss(eng, ladders):
    from evcouplings_b200 import model_ops
    from oracle import tempering as tp
    L, q, K = 16, 3, 0.5
    h, J = tp.curie_weiss_model(L, q, K)
    m = dict(L=L, q=q, h=h, J=J, alphabet="ACD", target_seq="A" * L, index_list=np.arange(1, L + 1))
    ladder = model_ops.geometric_ladder(0.125, 1.0, 8)
    R = len(ladder)
    with model_ops.PottsSampler(m, ladders * R, seed=2, init="target", engine=eng) as s:
        s.set_ladder(ladder, 1)
        s.temper(1000)
        before = s.swap_statistics()["round_trips"].copy()
        sec = timed(lambda: s.temper(1000))
        st = s.swap_statistics()
    return dict(L=L, q=q, K=K, ladder=[float(b) for b in ladder], ladders=ladders,
                round_trips_per_ladder_per_1000_sweeps=float((st["round_trips"] - before).mean()),
                acceptance=[float(a) for a in st["acceptance"]], seconds_per_1000_sweeps=sec)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", type=int, default=16384)
    ap.add_argument("--sweeps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--fit-iterations", type=int, default=100)
    ap.add_argument("--cw-ladders", type=int, default=4096)
    ap.add_argument("--out", default=None, help="also write the full result as JSON to this file")
    a = ap.parse_args()
    from evcouplings_b200.engine import CudaEngine
    eng = CudaEngine()
    result = dict(card=card(), chains=a.chains, sweeps=a.sweeps, warmup=a.warmup, repeats=a.repeats, models={})
    c2, fit_s = config2_model(eng, a.fit_iterations)
    pabp = pabp_model()
    pabp["index_list"] = np.arange(1, pabp["L"] + 1)
    for name, model in (("pabp_L82_q20", pabp), ("config2_L200_q21", c2)):
        rows = run_model(eng, model, a.chains, a.sweeps, a.warmup, a.repeats)
        result["models"][name] = dict(L=model["L"], q=model["q"], variants=rows)
        for v, r in rows.items():
            extra = "" if v == "plain" else ", %.3f of plain, swap kernel %.4f of kernel time, acceptance %s" % (
                r["relative_to_plain"], r["swap_kernel_share"], " ".join("%.3f" % x for x in r["acceptance"]))
            print("%s %s: %.4g chain-sweeps/s (min %.4g, max %.4g), %.1f changes/chain-sweep%s" % (
                name, v, r["median"], r["min"], r["max"], r["changes_per_chain_sweep"], extra), flush=True)
    result["curie_weiss"] = curie_weiss(eng, a.cw_ladders)
    print("curie-weiss:", json.dumps(result["curie_weiss"]), flush=True)
    result["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
