"""
Correction pairs of the L-BFGS history in pinned host memory (-m gpu): a fit with k of its m pairs on the host
must take bit-identical iterations (every row of the iteration table and the final x) to the fit with the whole
history on the device; the handle's device and host byte counts must match the prediction; run_plmc with forced
host pairs must write byte-identical output files.  Also one evaluation at L = 2300, where (L q)^2 > 2^31, checked
block by block against float64.
"""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from evcouplings_b200 import lbfgs, synthetic, tools  # noqa: E402

pytestmark = pytest.mark.gpu

N, L, M = 6000, 60, 6
LAM_H, LAM_J = 0.01, 2.0


@pytest.fixture(scope="module")
def engine():
    from evcouplings_b200.engine import CudaEngine
    return CudaEngine()


def _inputs(q, gap, seed=43):
    codes = synthetic.synthetic_msa_codes(N, L, seed)
    if gap:
        codes = synthetic.to_ignore_gaps_codes(codes, q)
    w = np.random.default_rng(seed).uniform(0.05, 1.0, N).astype(np.float32)
    return codes, w


def _fit(engine, monkeypatch, codes, w, q, gap_code, prec, host_pairs, seq_chunk=0, iters=30, eps=1e-9):
    monkeypatch.setenv("EVC_HOST_HISTORY", str(host_pairs))
    p = engine.plm_problem(codes, w, q, gap_code, LAM_H, LAM_J, m=M, precision=prec, seq_chunk=seq_chunk)
    rows = []
    try:
        assert p.host_pairs == host_pairs
        params = lbfgs.default_params(max_iterations=iters, epsilon=eps, m=M)
        res = p.fit(np.zeros(p.n, dtype=np.float32), params,
                    lambda k, fx, xn, gn, st, nls: rows.append((k, fx, xn, gn, st, nls)) and False)
        out = dict(rows=rows, x=p.get_x(), res=tuple(res), n_chunks=p.n_chunks, switched=p.switched_at,
                   device_bytes=p.device_bytes(), host=p.host_bytes(), n=p.n)
    finally:
        p.close()
    return out


@pytest.mark.parametrize("prec", ["fp32", "auto"])
@pytest.mark.parametrize("q,gap", [(21, False), (20, True)])
def test_trajectory_is_bit_identical(engine, monkeypatch, q, gap, prec):
    codes, w = _inputs(q, gap)
    gap_code = q if gap else -1
    eps = 1e-9
    if prec == "auto":
        # "auto" runs bf16 products until |g| / max(1, |x|) <= 10 eps, then drops the history and restarts the ring
        # in fp32.  epsilon only enters the stopping tests, so a run with a tiny epsilon gives the bf16 trajectory;
        # 10 eps just above its smallest ratio in the first 10 iterations makes the switch certain by then.
        probe = _fit(engine, monkeypatch, codes, w, q, gap_code, prec, 0, iters=10)
        eps = min(gn / max(1.0, xn) for _k, _fx, xn, gn, _st, _n in probe["rows"]) / 10 * 1.001
    ref = _fit(engine, monkeypatch, codes, w, q, gap_code, prec, 0, eps=eps)
    assert len(ref["rows"]) >= 10
    assert ref["host"] == (0, 0.0)
    print(prec, q, "iterations", len(ref["rows"]), "switched at", ref["switched"])
    if prec == "auto":
        # switched within the first 10 iterations, then at least 3 iterations refill the ring (host slots included)
        assert 0 <= ref["switched"] <= 10 and len(ref["rows"]) >= ref["switched"] + 3, ref["switched"]
    for k in (M, 2):
        got = _fit(engine, monkeypatch, codes, w, q, gap_code, prec, k, eps=eps)
        assert got["rows"] == ref["rows"], k
        assert got["res"] == ref["res"] and got["switched"] == ref["switched"], k
        assert np.array_equal(got["x"], ref["x"]), k
        assert got["host"][0] > 0, k


def test_trajectory_with_sequence_chunks(engine, monkeypatch):
    codes, w = _inputs(21, False)
    ref = _fit(engine, monkeypatch, codes, w, 21, -1, "fp32", 0, seq_chunk=2304)
    got = _fit(engine, monkeypatch, codes, w, 21, -1, "fp32", 3, seq_chunk=2304)
    assert ref["n_chunks"] == got["n_chunks"] == 3
    assert got["rows"] == ref["rows"] and np.array_equal(got["x"], ref["x"])


def test_python_driver_refuses_host_pairs(engine, monkeypatch):
    from evcouplings_b200.engine import DeviceMemoryError
    codes, w = _inputs(21, False)
    monkeypatch.setenv("EVC_HOST_HISTORY", "2")
    p = engine.plm_problem(codes, w, 21, -1, LAM_H, LAM_J, m=M, seq_chunk=0)
    try:
        with pytest.raises(DeviceMemoryError, match="driver='device'"):
            p.fit(np.zeros(p.n, dtype=np.float32), lbfgs.default_params(max_iterations=2, m=M), driver="python")
    finally:
        p.close()


def test_device_and_host_bytes_match_the_prediction(engine, monkeypatch):
    from evcouplings_b200.engine import fit_workspace_bytes, tc_bytes
    codes, w = _inputs(21, False)
    sm = engine.sm_count()
    for k in (0, 1, M):
        got = _fit(engine, monkeypatch, codes, w, 21, -1, "fp32", k, iters=3)
        dev, host = fit_workspace_bytes(got["n"], M, k)
        assert got["device_bytes"] == tc_bytes(N, L, 21, -1, 0, sm) + dev, k
        assert got["host"][0] == host, k
        assert (got["host"][1] > 0) == (k > 0), k


def test_run_plmc_files_are_byte_identical(engine, tmp_path, monkeypatch):
    n_seq, n_site = 1600, 24
    codes = synthetic.synthetic_msa_codes(n_seq, n_site, 9)
    a2m = tmp_path / "hh.a2m"
    synthetic.write_a2m(str(a2m), codes)
    lam_J = 0.01 * 20 * (n_site - 1)
    out = {}
    for k in (None, "6"):
        if k is None:
            monkeypatch.delenv("EVC_HOST_HISTORY", raising=False)
        else:
            monkeypatch.setenv("EVC_HOST_HISTORY", k)
        tag = "dev" if k is None else "host"
        ecs, model = tmp_path / (tag + "_ECs.txt"), tmp_path / (tag + ".model")
        _res, run = tools.run_plmc(str(a2m), str(ecs), str(model), focus_seq="seq0/1-%d" % n_site, theta=0.8,
                                   iterations=40, lambda_h=0.01, lambda_J=lam_J, engine=engine, return_run=True,
                                   epsilon=1e-6)
        out[tag] = (ecs.read_bytes(), model.read_bytes(), run.timings)
    assert out["dev"][2]["host_history_pairs"] == 0 and out["host"][2]["host_history_pairs"] == 6
    assert out["host"][2]["fit_host_history_bytes"] > 0 and out["host"][2]["fit_host_history_pin_s"] > 0
    assert out["host"][0] == out["dev"][0]
    assert out["host"][1] == out["dev"][1]


def _mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def test_large_index_gradient_blocks(engine):
    """L = 2300, q = 21: (L q)^2 = 2.33e9 > 2^31 elements in the coupling operand and the backward planes.  J is
    nonzero only in the blocks of six test sites (against every other site), so the float64 conditionals of all
    sites are cheap; the fields and every J block of the test sites, including the last ones, are compared."""
    import torch
    from evcouplings_b200.engine import num_params
    Lb, q, Nb = 2300, 21, 768
    assert (Lb * q) ** 2 > 2 ** 31
    n = num_params(Lb, q)
    if _mem_available() < 20e9:
        pytest.skip("needs about 15 GB of host memory for the float64 check, %d bytes available" % _mem_available())
    rng = np.random.default_rng(11)
    codes = synthetic.synthetic_msa_codes(Nb, Lb, 17)
    w = rng.uniform(0.2, 1.0, Nb).astype(np.float32).astype(np.float64)
    T = [0, 1, Lb // 2, Lb - 3, Lb - 2, Lb - 1]
    lq = Lb * q
    x = np.zeros(n, dtype=np.float32)
    x[:lq] = rng.normal(0, 0.1, lq)
    Jt = x[lq:].reshape(-1, q, q)

    def pair_index(i, j):          # i < j, arrays
        return i * (2 * Lb - i - 1) // 2 + (j - i - 1)

    ks = np.arange(Lb)
    for t in T:                    # J_tk for every k (blocks shared by two test sites are drawn twice: fine)
        lo, hi = ks[ks < t], ks[ks > t]
        Jt[pair_index(lo, t)] = rng.normal(0, 0.05, (len(lo), q, q))
        Jt[pair_index(t, hi)] = rng.normal(0, 0.05, (len(hi), q, q))
    h = x[:lq].reshape(Lb, q).astype(np.float64)

    def full_row(t):               # F[k, a, b] = J_tk(a, b), a = state at t, b = state at k
        F = np.zeros((Lb, q, q))
        lo, hi = ks[ks < t], ks[ks > t]
        F[lo] = Jt[pair_index(lo, t)].transpose(0, 2, 1)
        F[hi] = Jt[pair_index(t, hi)]
        return F

    Fs = {t: full_row(t) for t in T}
    Z = np.broadcast_to(h, (Nb, Lb, q)).copy()
    for t in T:                    # sites outside T see the test sites only
        Z += Fs[t][:, codes[:, t], :].transpose(1, 0, 2)
    for t in T:                    # test sites see every site
        Z[:, t, :] = h[t] + Fs[t][ks[None, :], :, codes].sum(axis=1)
    Z -= Z.max(axis=2, keepdims=True)
    P = np.exp(Z)
    P /= P.sum(axis=2, keepdims=True)
    X = np.zeros((Nb, Lb, q))
    X[np.arange(Nb)[:, None], ks[None, :], codes] = 1.0
    R = w[:, None, None] * (P - X)
    del Z, P
    Xf, Rf = X.reshape(Nb, lq), R.reshape(Nb, lq)

    p = engine.plm_problem(codes, w.astype(np.float32), q, -1, LAM_H, LAM_J, m=M, seq_chunk=0)
    try:
        p.x.copy_(torch.from_numpy(x))
        p.evaluate(p.x)
        g = p.g.cpu().numpy()
    finally:
        p.close()
    gJt = g[lq:].reshape(-1, q, q)
    for t in T:
        A = (R[:, t, :].T @ Xf).reshape(q, Lb, q)          # sum_s R[s,t,a] [s_k = b]
        B = (X[:, t, :].T @ Rf).reshape(q, Lb, q)          # sum_s [s_t = a] R[s,k,b]
        want = (A + B).transpose(1, 0, 2) + 2 * LAM_J * Fs[t]
        want[t] = 0.0
        lo, hi = ks[ks < t], ks[ks > t]
        got = np.zeros((Lb, q, q))
        got[lo] = gJt[pair_index(lo, t)].transpose(0, 2, 1)
        got[hi] = gJt[pair_index(t, hi)]
        gh_want = R[:, t, :].sum(axis=0) + 2 * LAM_H * h[t]
        gh_got = g[t * q:(t + 1) * q].astype(np.float64)
        err = np.sqrt(np.sum((got - want) ** 2) + np.sum((gh_got - gh_want) ** 2))
        ref = np.sqrt(np.sum(want ** 2) + np.sum(gh_want ** 2))
        print("site %d: gradient rel L2 %.2e against float64" % (t, err / ref))
        assert err <= 5e-6 * ref, (t, err / ref)
