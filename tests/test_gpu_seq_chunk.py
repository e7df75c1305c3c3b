"""
Sequence chunks of the tensor-core path (-m gpu): an evaluation that streams the shard through chunk-sized
buffers must give the objective and g_h bit for bit, and g_J and the pair counts up to the summation order of the
backward product, compared with the unchunked evaluation.  Also: the fused-forward fallback, the device byte
count after a fit, a planned fit under a pretend memory budget, a converged run_plmc with forced chunks, and the
batched hamiltonians.
"""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from evcouplings_b200 import lbfgs, model_ops, msa, synthetic, tools  # noqa: E402

pytestmark = pytest.mark.gpu

N, L = 6000, 60
# chunk size -> chunks of N = 6000: 3072 -> 2, 2304 -> 3 (last 1392), 768 -> 8 (last 624), 6144 -> 1
CHUNKS = ((3072, 2), (2304, 3), (768, 8), (6144, 1))
LAM_H, LAM_J = 0.01, 2.0


@pytest.fixture(scope="module")
def engine():
    from evcouplings_b200.engine import CudaEngine
    return CudaEngine()


def _inputs(q, gap, seed=41):
    codes = synthetic.synthetic_msa_codes(N, L, seed)
    if gap:
        codes = synthetic.to_ignore_gaps_codes(codes, q)
    rng = np.random.default_rng(seed)
    w = rng.uniform(0.05, 1.0, N).astype(np.float32)
    x = rng.normal(0, 0.1, L * q + L * (L - 1) // 2 * q * q).astype(np.float32)
    return codes, w, x


def _run(engine, codes, w, x, q, gap_code, prec, seq_chunk, forward="tc", counts=False):
    p = engine.plm_problem(codes, w, q, gap_code, LAM_H, LAM_J, forward=forward, backward="tc", precision=prec,
                           seq_chunk=seq_chunk)
    try:
        p.set_x(x)
        p.evaluate(p.x)
        out = dict(fx=p.fxbuf.cpu().numpy().copy(), g=p.g.cpu().numpy().copy(), n_chunks=p.n_chunks)
        if counts:
            out["fi"], out["fij"] = p.weighted_counts()
    finally:
        p.close()
    return out


@pytest.mark.parametrize("prec", ["fp32", "bf16"])
@pytest.mark.parametrize("q,gap", [(21, False), (20, True)])
def test_chunked_evaluation_matches_unchunked(engine, q, gap, prec):
    from oracle import c_oracle as co
    codes, w, x = _inputs(q, gap)
    gap_code = q if gap else -1
    counts = prec == "fp32"
    ref = _run(engine, codes, w, x, q, gap_code, prec, 0, counts=counts)
    assert ref["n_chunks"] == 1
    nh = L * q
    g64 = None
    if prec == "fp32":
        _fx64, g64, _nll64 = co.plm_eval(codes, w.astype(np.float64), x.astype(np.float64), q, LAM_H, LAM_J, "f64")
    for chunk, n_chunks in CHUNKS:
        got = _run(engine, codes, w, x, q, gap_code, prec, chunk, counts=counts)
        assert got["n_chunks"] == n_chunks
        # the forward does not depend on the chunking and the g_h / fx partials are summed in the same order
        assert np.array_equal(got["fx"], ref["fx"]), (chunk, got["fx"], ref["fx"])
        assert np.array_equal(got["g"][:nh], ref["g"][:nh]), chunk
        gJ, gJ1 = got["g"][nh:].astype(np.float64), ref["g"][nh:].astype(np.float64)
        assert np.linalg.norm(gJ - gJ1) <= 1e-6 * np.linalg.norm(gJ1), (chunk, np.linalg.norm(gJ - gJ1))
        if counts:
            assert np.array_equal(got["fi"], ref["fi"]), chunk
            assert np.abs(got["fij"] - ref["fij"]).max() <= 1e-6 * np.abs(ref["fij"]).max(), chunk
        if g64 is not None:
            g = got["g"].astype(np.float64)
            assert np.linalg.norm(g - g64) <= 5e-6 * np.linalg.norm(g64), chunk


def test_fused_forward_falls_back_under_chunks(engine):
    codes, w, x = _inputs(21, False)
    tc = _run(engine, codes, w, x, 21, -1, "fp32", 2304)
    fused = _run(engine, codes, w, x, 21, -1, "fp32", 2304, forward="tcfused")
    assert fused["n_chunks"] == 3
    assert np.array_equal(fused["fx"], tc["fx"]) and np.array_equal(fused["g"], tc["g"])


def test_set_seq_chunk_after_allocation(engine):
    import ctypes
    from evcouplings_b200 import _lib
    lib = engine.lib
    codes, w, _x = _inputs(21, False)
    h = ctypes.c_void_p()
    _lib.check(lib.evc_plm_create(ctypes.byref(h), codes.ctypes.data_as(ctypes.c_void_p), N, L, 21, -1,
                                  w.ctypes.data_as(ctypes.c_void_p), engine.device_index), "evc_plm_create")
    try:
        assert lib.evc_plm_set_seq_chunk(h, 6144) == 0          # >= N: whole shard
        assert lib.evc_plm_set_forward(h, 1) == 0
        assert lib.evc_plm_set_seq_chunk(h, 0) == 0             # same layout
        assert lib.evc_plm_set_seq_chunk(h, 768) != 0
        assert b"already exist" in lib.evc_last_error()
    finally:
        lib.evc_plm_destroy(h)


def test_device_bytes_and_planned_budget(engine):
    import torch
    from evcouplings_b200.engine import plan_seq_chunk, seq_chunk_reserve_bytes, tc_bytes
    q, m = 21, 6
    codes, w, _x = _inputs(q, False)
    sm = engine.sm_count()
    budget = tc_bytes(N, L, q, -1, 0, sm) + seq_chunk_reserve_bytes(L, q, m) - 1     # the whole shard misses by 1 B
    chunk = plan_seq_chunk(N, L, q, -1, m, sm, budget)
    assert chunk > 0 and chunk % 768 == 0
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated(engine.device)
    torch.cuda.reset_peak_memory_stats(engine.device)
    p = engine.plm_problem(codes, w, q, -1, LAM_H, LAM_J, m=m, seq_chunk=chunk)
    try:
        assert p.n_chunks > 1
        assert p.device_bytes() == tc_bytes(N, L, q, -1, chunk, sm)
        p.weighted_counts()
        params = lbfgs.default_params(max_iterations=3, epsilon=1e-5, m=m)
        p.fit(np.zeros(p.n, dtype=np.float32), params)
        fit_ws = int(engine.lib.evc_fit_workspace_bytes(p.n, m))
        assert p.device_bytes() == tc_bytes(N, L, q, -1, chunk, sm) + fit_ws
        torch.cuda.synchronize()
        peak_torch = torch.cuda.max_memory_allocated(engine.device) - base
        print("chunk %d: handle %d B, torch peak %d B, budget %d B" % (chunk, p.device_bytes(), peak_torch, budget))
        assert p.device_bytes() + peak_torch <= budget
    finally:
        p.close()


def test_run_plmc_with_forced_chunks_reaches_the_oracle_optimum(engine, tmp_path, monkeypatch):
    """Converged run_plmc with EVC_SEQ_CHUNK = 768 (1600 sequences: 3 chunks) vs the float64 oracle optimum,
    with the tolerance of the unchunked end-to-end test: EC (cn) rms <= 1e-4."""
    from oracle import c_oracle as co
    from oracle import plm_oracle as po
    n_seq, n_site = 1600, 16
    codes = synthetic.synthetic_msa_codes(n_seq, n_site, 7)
    a2m = tmp_path / "chunked.a2m"
    synthetic.write_a2m(str(a2m), codes)
    q = 21
    lam_J = 0.01 * (q - 1) * (n_site - 1)
    monkeypatch.setenv("EVC_SEQ_CHUNK", "768")
    res, run = tools.run_plmc(str(a2m), str(tmp_path / "o_ECs.txt"), str(tmp_path / "o.model"),
                              focus_seq="seq0/1-%d" % n_site, theta=0.8, ignore_gaps=False, iterations=3000,
                              lambda_h=0.01, lambda_J=lam_J, engine=engine, return_run=True, epsilon=1e-5)
    assert run.timings["seq_chunks"] == 3
    ali = run.alignment
    counts_o = co.hamming_counts(ali.codes, msa.identity_threshold_count(0.8, n_site))
    assert np.array_equal(run.counts, counts_o)
    w = 1.0 / counts_o
    xo, _info = po.fit(ali.codes, w, q, 0.01, lam_J, ali.gap_code, x0=tools.initial_point(
        po.frequencies(ali.codes, w, q, ali.gap_code)[0], w.sum(), n_site, q).astype(np.float64), max_iter=4000,
        objective_fn=lambda v: co.plm_eval(ali.codes, w, v, q, 0.01, lam_J, "f64"))
    cn = np.loadtxt(str(tmp_path / "o_ECs.txt"), usecols=5)
    cn_o = po.cn_scores(xo[n_site * q:].reshape(-1, q, q), n_site)
    rms = np.sqrt(np.mean((cn - cn_o) ** 2))
    print("status", res.optimization_status, "iters", run.lbfgs.iterations, "cn rms", rms)
    assert rms <= 1e-4


def test_hamiltonians_batches_are_bit_identical(engine):
    rng = np.random.default_rng(5)
    n_site, q = 30, 21
    npair = n_site * (n_site - 1) // 2
    model = dict(L=n_site, q=q, h=rng.normal(0, 0.5, (n_site, q)).astype(np.float32),
                 J=rng.normal(0, 0.1, (npair, q, q)).astype(np.float32))
    codes = synthetic.synthetic_msa_codes(5000, n_site, 5)
    codes[100, 3] = q                     # one ignored symbol, in the first batch only
    one = model_ops.hamiltonians(model, codes, engine, batch_size=len(codes))
    for bs in (2048, 1000, None):
        got = model_ops.hamiltonians(model, codes, engine, batch_size=bs)
        assert np.array_equal(got, one), bs
