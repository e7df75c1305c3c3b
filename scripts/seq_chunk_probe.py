"""
Sequence-chunk probe (one GPU, one call): what streaming the sequences through chunk-sized buffers costs, and an
alignment larger than the GPU memory end to end.

  1. Config 2 (N=50,000, L=200, q=21): ms per objective + gradient evaluation unchunked and with 2, 4 and 8 forced
     chunks, the four variants alternated, median of 3 rounds of 20 timed evaluations each (CUDA events).
  2. N=2,000,000, L=200, q=21 (about 103 GB unchunked): the chunk the planner picks from the free memory; one chunked
     evaluation against the sum of the two halves of the alignment evaluated separately (no regulariser: -loglk to
     ~1e-12 relative, gradient to 1e-6 relative L2); then a 5-iteration run_plmc on the synthetic A2M of that size.

The card's name and power limit are read in the same run (read-only nvidia-smi query).

    python scripts/seq_chunk_probe.py OUTDIR
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

from evcouplings_b200 import synthetic, tools  # noqa: E402
from evcouplings_b200.engine import (CudaEngine, SEQ_CHUNK_ALIGN, plan_seq_chunk,  # noqa: E402
                                     seq_chunk_reserve_bytes, tc_bytes)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip()


def chunk_for(N, k):
    """Chunk size (multiple of 768) that cuts N sequences into k chunks."""
    c = -(-N // k)
    return -(-c // SEQ_CHUNK_ALIGN) * SEQ_CHUNK_ALIGN


def time_evals(torch, p, steps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(steps):
        p.evaluate_async(p.x)
    ev[1].record()
    ev[1].synchronize()
    return ev[0].elapsed_time(ev[1]) / steps


def config2_overhead(eng, torch, res):
    N, L, seed = synthetic.CONFIG_SEEDS[2]
    codes = synthetic.synthetic_msa_codes(N, L, seed)
    rng = np.random.default_rng(2)
    w = rng.uniform(0.05, 1.0, N).astype(np.float32)
    x = rng.normal(0, 0.05, L * 21 + L * (L - 1) // 2 * 441).astype(np.float32)
    variants = [("unchunked", 0)] + [("%d chunks" % k, chunk_for(N, k)) for k in (2, 4, 8)]
    probs = {}
    for name, c in variants:
        p = eng.plm_problem(codes, w, 21, -1, 0.01, 2.0, seq_chunk=c)
        p.set_x(x)
        time_evals(torch, p, 5)                       # warm-up
        probs[name] = p
    ref_fx = probs["unchunked"].fxbuf.cpu().numpy().copy()
    times = {name: [] for name, _ in variants}
    for _ in range(3):
        for name, _c in variants:
            times[name].append(time_evals(torch, probs[name], 20))
    out = {}
    for name, c in variants:
        p = probs[name]
        out[name] = dict(seq_chunk=c, n_chunks=p.n_chunks, device_bytes=p.device_bytes(),
                         ms_per_eval_runs=times[name], ms_per_eval_median=float(np.median(times[name])),
                         fx_equal_unchunked=bool(np.array_equal(p.fxbuf.cpu().numpy(), ref_fx)))
    for p in probs.values():
        p.close()
    res["config2"] = out
    print(json.dumps(out, indent=1), flush=True)


def evaluate_data(eng, torch, codes, w, x, q):
    """-loglk and gradient of the data term (lambda = 0), seq_chunk planned from the free memory."""
    p = eng.plm_problem(codes, w, q, -1, 0.0, 0.0)
    try:
        p.set_x(x)
        torch.cuda.synchronize()
        t0 = time.time()
        p.evaluate(p.x)
        dt = time.time() - t0
        return float(p.fxbuf[0].item()), p.g.cpu().numpy().astype(np.float64), p.n_chunks, p.seq_chunk, dt
    finally:
        p.close()


def large(eng, torch, res, outdir):
    N, L, q = 2000000, 200, 21
    torch.cuda.empty_cache()
    free, total = torch.cuda.mem_get_info(eng.device)
    sm = eng.sm_count()
    need_whole = tc_bytes(N, L, q, -1, 0, sm) + seq_chunk_reserve_bytes(L, q, 6)
    planned = plan_seq_chunk(N, L, q, -1, 6, sm, free)
    info = dict(N=N, L=L, q=q, free_bytes=free, total_bytes=total, whole_shard_need_bytes=need_whole,
                planned_seq_chunk=planned)
    print(json.dumps(info), flush=True)
    t0 = time.time()
    codes = synthetic.synthetic_msa_codes(N, L, 11)
    info["synthetic_s"] = time.time() - t0
    rng = np.random.default_rng(11)
    w = rng.uniform(0.05, 1.0, N).astype(np.float32)
    x = rng.normal(0, 0.05, L * q + L * (L - 1) // 2 * q * q).astype(np.float32)
    nll, g, nch, chunk, dt = evaluate_data(eng, torch, codes, w, x, q)
    info.update(full_n_chunks=nch, full_seq_chunk=chunk, full_first_eval_s=dt)
    h = N // 2
    nll_a, g_a, nch_a, _, _ = evaluate_data(eng, torch, np.ascontiguousarray(codes[:h]), w[:h], x, q)
    nll_b, g_b, nch_b, _, _ = evaluate_data(eng, torch, np.ascontiguousarray(codes[h:]), w[h:], x, q)
    gs = g_a + g_b
    info.update(half_n_chunks=[nch_a, nch_b], negloglk_full=nll, negloglk_halves=nll_a + nll_b,
                negloglk_rel_diff=abs(nll - (nll_a + nll_b)) / abs(nll),
                grad_rel_l2_diff=float(np.linalg.norm(g - gs) / np.linalg.norm(gs)))
    print(json.dumps(info), flush=True)
    del g, g_a, g_b, gs
    # 5-iteration run_plmc on the synthetic A2M of that size
    with tempfile.TemporaryDirectory() as tmp:
        a2m = os.path.join(tmp, "large.a2m")
        t0 = time.time()
        synthetic.write_a2m(a2m, codes)
        info["write_a2m_s"] = time.time() - t0
        del codes
        t0 = time.time()
        r, run = tools.run_plmc(a2m, os.path.join(tmp, "o_ECs.txt"), os.path.join(tmp, "o.model"),
                                focus_seq="seq0/1-%d" % L, theta=0.8, iterations=5, lambda_h=0.01,
                                lambda_J=0.01 * (q - 1) * (L - 1), return_run=True, num_gpus=1)
        info["run_plmc_wall_s"] = time.time() - t0
        info["run_plmc_timings"] = run.timings
        info["run_plmc_iterations"] = int(run.lbfgs.iterations)
        info["run_plmc_evaluations"] = int(run.lbfgs.evaluations)
        info["run_plmc_status"] = r.optimization_status
        info["s_per_iteration"] = run.timings["optimisation_s"] / max(1, run.lbfgs.iterations)
        info["s_per_evaluation"] = run.timings["optimisation_s"] / max(1, run.lbfgs.evaluations)
    res["large"] = info
    print(json.dumps(info, default=str), flush=True)


def main():
    if len(sys.argv) != 2:
        sys.exit("usage: python scripts/seq_chunk_probe.py OUTDIR")
    outdir = sys.argv[1]
    os.makedirs(outdir, exist_ok=True)
    import torch
    res = {"card": card()}
    print(res["card"], flush=True)
    eng = CudaEngine()
    path = os.path.join(outdir, "seq_chunk_probe.json")
    try:
        config2_overhead(eng, torch, res)
        large(eng, torch, res, outdir)
    finally:
        res["card_after"] = card()
        with open(path, "w") as f:
            json.dump(res, f, indent=1, default=str)
    print("wrote", path)


if __name__ == "__main__":
    main()
