"""
Host-history probe (one GPU, one call): what keeping L-BFGS correction pairs in pinned host memory costs, and a fit
whose history does not fit the GPU end to end.

  1. Pinned host <-> device copy bandwidth (1 GiB copies, CUDA events): the reference rate of the PCIe link; and the
     rate of the library's streaming dot kernel reading two pinned vectors through their mapped addresses.
  2. Config 2 (N=50,000, L=200, q=21): ms per evc_plm_fit iteration with k = 0, 3 and 6 of the m = 6 pairs on the
     host, alternated, median of 3 rounds of 20 iterations; the iteration tables must be identical.  For the
     two-loop recursion and the pair update: the history bytes crossing the link per iteration (from the ring
     schedule, history_link_bytes), and the rate that the extra time per iteration over k = 0 implies.
  3. L=2000, q=21, N=20,000 synthetic (it does not fit one 80 GB GPU with the whole history on the device): the
     planner's decision, device and host bytes, the pin time, a 10-iteration run_plmc, and seconds per iteration
     split into objective evaluations and the rest (two-loop recursion, pair update, line-search vector passes).
     Skipped, with the reason recorded, when the host lacks the memory.

The card's name and power limit are read in the same run (read-only nvidia-smi query).

    python scripts/host_history_probe.py OUTDIR
"""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from evcouplings_b200 import lbfgs, synthetic, tools  # noqa: E402
from evcouplings_b200.engine import (CudaEngine, fit_workspace_bytes, host_history_budget_bytes,  # noqa: E402
                                     num_params, plan_fit_memory)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip()


def copy_bandwidth(torch, res):
    nb = 1 << 30
    host = torch.empty(nb, dtype=torch.uint8, pin_memory=True)
    dev = torch.empty(nb, dtype=torch.uint8, device="cuda")
    out = {}
    for name, dst, src in (("h2d", dev, host), ("d2h", host, dev)):
        dst.copy_(src, non_blocking=True)
        times = []
        for _ in range(5):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            dst.copy_(src, non_blocking=True)
            ev[1].record()
            ev[1].synchronize()
            times.append(ev[0].elapsed_time(ev[1]) / 1e3)
        out[name + "_GBps"] = nb / float(np.median(times)) / 1e9
    del host, dev
    res["pinned_copy"] = out
    print(json.dumps(out), flush=True)


def zero_copy_read(eng, torch, res):
    """The library's streaming dot kernel (evc_vec_dot) over two pinned host vectors read through their mapped
    addresses, and over the same vectors in device memory: the rate one fixed-grid streaming kernel gets from
    zero-copy reads, to compare with the pinned-copy rate and with the fit's history rate."""
    import ctypes
    n = 64 << 20                                        # 256 MB per vector
    lib = eng.lib
    host = [torch.ones(n, dtype=torch.float32, pin_memory=True) for _ in range(2)]
    dev = [t.to(eng.device) for t in host]
    out = torch.zeros(1, dtype=torch.float64, device=eng.device)
    res_out = {}
    for name, (a, b) in (("zero_copy", host), ("device", dev)):
        args = (ctypes.c_void_p(a.data_ptr()), ctypes.c_void_p(b.data_ptr()), n, ctypes.c_void_p(out.data_ptr()),
                eng.stream())
        assert lib.evc_vec_dot(*args) == 0
        times = []
        for _ in range(5):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            assert lib.evc_vec_dot(*args) == 0
            ev[1].record()
            ev[1].synchronize()
            times.append(ev[0].elapsed_time(ev[1]) / 1e3)
        assert float(out.item()) == float(n)
        res_out[name + "_read_GBps"] = 2 * 4 * n / float(np.median(times)) / 1e9
    res_out["zero_copy_ratio_to_pinned_h2d"] = res_out["zero_copy_read_GBps"] / res["pinned_copy"]["h2d_GBps"]
    del host, dev
    res["dot_kernel"] = res_out
    print(json.dumps(res_out), flush=True)


def history_link_bytes(iterations, m, k, vec):
    """(read, written) history bytes crossing PCIe in an evc_plm_fit run of `iterations` iterations with k of its m
    ring slots (the last k) in host memory, from the ring schedule of fit.cu: after every accepted iteration but the
    last, the new pair is written into slot `end` (2 vectors), then the two-loop recursion over the `bound` newest
    pairs reads every s and every y of its window twice, and y of the oldest pair once more (its last first-loop
    step passes that vector as both operands; counted as crossing the link twice).  Assumes no restart of the
    history (fp32 products throughout) and no early stop."""
    host = set(range(m - k, m))
    read = written = 0
    hist = end = 0
    for _ in range(iterations - 1):
        if end in host:
            written += 2 * vec
        hist = min(m, hist + 1)
        end = (end + 1) % m
        window = [(end - 1 - i) % m for i in range(hist)]
        read += sum(4 * vec for j in window if j in host)
        if window[-1] in host:
            read += vec
    return read, written


def config2(eng, torch, res, monkeypatch_env):
    N, L, seed = synthetic.CONFIG_SEEDS[2]
    q, m, iters = 21, 6, 20
    codes = synthetic.synthetic_msa_codes(N, L, seed)
    w = np.random.default_rng(2).uniform(0.05, 1.0, N).astype(np.float32)
    ks = (0, 3, 6)
    probs = {}
    for k in ks:
        monkeypatch_env(k)
        p = eng.plm_problem(codes, w, q, -1, 0.01, 0.01 * (q - 1) * (L - 1), m=m, seq_chunk=0)
        p.fit(np.zeros(p.n, dtype=np.float32), lbfgs.default_params(max_iterations=2, epsilon=1e-9, m=m))  # allocate
        probs[k] = p
    n = probs[0].n
    times = {k: [] for k in ks}
    rows = {}
    for _ in range(3):
        for k in ks:
            tab = []
            p = probs[k]
            res_k = p.fit(np.zeros(n, dtype=np.float32), lbfgs.default_params(max_iterations=iters, epsilon=1e-9, m=m),
                          lambda *r: tab.append(r) and False)
            times[k].append(p.fit_seconds * 1e3 / max(1, res_k.iterations))
            rows.setdefault(k, tab)
            assert tab == rows[k]
    vec = (n + 4 + 63) // 64 * 64 * 4
    out = {"n": n, "iterations": iters, "vector_bytes": vec}
    base = float(np.median(times[0]))
    for k in ks:
        med = float(np.median(times[k]))
        read, written = history_link_bytes(iters, m, k, vec)
        hist_bytes = (read + written) / iters
        extra = (med - base) / 1e3
        out["k=%d" % k] = dict(ms_per_iteration_runs=times[k], ms_per_iteration_median=med,
                               device_bytes=probs[k].device_bytes(), host_bytes=probs[k].host_bytes()[0],
                               pin_s=probs[k].host_bytes()[1], history_bytes_over_pcie_per_iteration=hist_bytes,
                               history_read_bytes_per_iteration=read / iters,
                               history_written_bytes_per_iteration=written / iters,
                               extra_ms_per_iteration=med - base,
                               implied_GBps=(hist_bytes / extra / 1e9) if k and extra > 0 else None,
                               table_identical_to_k0=rows[k] == rows[0])
    for p in probs.values():
        p.close()
    h2d = res["pinned_copy"]["h2d_GBps"]
    for k in ks[1:]:
        r = out["k=%d" % k]
        r["ratio_to_pinned_h2d"] = r["implied_GBps"] / h2d if r["implied_GBps"] else None
    res["config2"] = out
    print(json.dumps(out, indent=1), flush=True)


def large(eng, torch, res, monkeypatch_env):
    N, L, q, m = 20000, 2000, 21, 6
    monkeypatch_env(None)
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info(eng.device)
    host_budget = host_history_budget_bytes(1)
    sm = eng.sm_count()
    n = num_params(L, q)
    info = dict(N=N, L=L, q=q, m=m, free_bytes=free, total_bytes=total, host_budget_bytes=host_budget)
    try:
        chunk, k = plan_fit_memory(N, L, q, -1, m, sm, free, host_budget)
    except Exception as e:          # recorded, not hidden: the probe reports why it could not run
        info["skipped"] = "%s: %s" % (type(e).__name__, e)
        res["large"] = info
        print(json.dumps(info), flush=True)
        return
    dev, host = fit_workspace_bytes(n, m, k)
    info.update(planned_seq_chunk=chunk, planned_host_pairs=k, fit_device_bytes=dev, fit_host_bytes=host)
    print(json.dumps(info), flush=True)
    codes = synthetic.synthetic_msa_codes(N, L, 21)
    lam_J = 0.01 * (q - 1) * (L - 1)
    with tempfile.TemporaryDirectory() as tmp:
        a2m = os.path.join(tmp, "large.a2m")
        synthetic.write_a2m(a2m, codes)
        t0 = time.time()
        r, run = tools.run_plmc(a2m, os.path.join(tmp, "o_ECs.txt"), None, focus_seq="seq0/1-%d" % L, theta=0.8,
                                iterations=10, lambda_h=0.01, lambda_J=lam_J, engine=eng, return_run=True)
        info["run_plmc_wall_s"] = time.time() - t0
    info["run_plmc_timings"] = run.timings
    info["run_plmc_iterations"] = int(run.lbfgs.iterations)
    info["run_plmc_evaluations"] = int(run.lbfgs.evaluations)
    info["run_plmc_status"] = r.optimization_status
    res["large"] = info
    print(json.dumps(info, default=str), flush=True)
    # time of one objective evaluation on the same plan, to split the iteration time
    w = np.asarray(run.weights, dtype=np.float32)
    p = eng.plm_problem(run.alignment.codes, w, q, run.alignment.gap_code, 0.01, lam_J, m=m, seq_chunk=chunk)
    try:
        p.evaluate(p.x)
        torch.cuda.synchronize()
        t0 = time.time()
        for _ in range(2):
            p.evaluate(p.x)
        t_eval = (time.time() - t0) / 2
    finally:
        p.close()
    its, evs = max(1, run.lbfgs.iterations), run.lbfgs.evaluations
    opt = run.timings["fit_fit_s"]
    info.update(s_per_evaluation=t_eval, s_per_iteration=opt / its,
                s_per_iteration_evaluations=t_eval * evs / its, s_per_iteration_rest=(opt - t_eval * evs) / its)
    res["large"] = info
    print(json.dumps(info, default=str), flush=True)


def main():
    if len(sys.argv) != 2:
        sys.exit("usage: python scripts/host_history_probe.py OUTDIR")
    outdir = sys.argv[1]
    os.makedirs(outdir, exist_ok=True)
    import torch
    res = {"card": card()}
    print(res["card"], flush=True)
    eng = CudaEngine()

    def set_pairs(k):
        if k is None:
            os.environ.pop("EVC_HOST_HISTORY", None)
        else:
            os.environ["EVC_HOST_HISTORY"] = str(k)

    path = os.path.join(outdir, "host_history_probe.json")
    try:
        copy_bandwidth(torch, res)
        zero_copy_read(eng, torch, res)
        config2(eng, torch, res, set_pairs)
        large(eng, torch, res, set_pairs)
    finally:
        set_pairs(None)
        res["card_after"] = card()
        with open(path, "w") as f:
            json.dump(res, f, indent=1, default=str)
    print("wrote", path)


if __name__ == "__main__":
    main()
