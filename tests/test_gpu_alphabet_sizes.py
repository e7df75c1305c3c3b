"""
Alphabets of any size on the GPU (-m gpu): 2 <= q <= 32 states with the gap as a state, 2 <= q <= 31 with the gap
ignored.  New q run the register-bounded softmax kernels (8 / 16 / 32 states), expand_tc_kernel with dynamic shared
memory (q > 21), finalize_pairs_tc_kernel with a tile sized from q (q > 21) and plm_energy_kernel<S> for every odd
stride S <= 33.

* Objective and gradient against the float64 model of the device's own bf16 arithmetic (po.objective(operands=...,
  bounds=...)) with the per-site / per-block error model of test_gpu_tc_edges.py, in both precision modes; L * q on
  and beside the 64 / 128 / 192 tile edges, N beside the 192- and 256-sequence tiles.  In the fp32 mode also against
  the exact float64 objective: whole-gradient relative L2 <= 2e-5, fx relative <= 2e-6.  The handle's device bytes
  equal evc_plm_tc_bytes_alphabet (the real allocations, q = 32 included).  Handles come from
  evc_plm_create_alphabet; evc_plm_create keeps taking q in {4, 5, 20, 21} only.
* Sequence chunks at q = 22 and 32: fx and g_h bit-identical to the unchunked evaluation, g_J within the model's
  tolerance of the summation order.
* Pair counts, Hamming counts with codes up to 31, run_plmc end to end (and bin/evcplm-plmc -a), model consumers,
  and the refusal of the gather kernels outside q in {4, 5, 20, 21}.
"""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

from evcouplings_b200 import _lib, model_io, model_ops, msa, tools  # noqa: E402
from oracle import c_oracle as co  # noqa: E402
from oracle import plm_oracle as po  # noqa: E402

import test_gpu_tc_edges as edges  # noqa: E402
from test_alphabet_sizes import (DNA_N, PROTEIN_X, TWO_LETTERS, alphabet_codes, alphabet_of,  # noqa: E402
                                 write_alphabet_a2m)


@pytest.fixture(scope="module")
def lib():
    l = _lib.load()
    _lib.require_device()
    return l


@pytest.fixture(scope="module")
def engine(lib):
    from evcouplings_b200.engine import CudaEngine
    return CudaEngine()


def make_inputs(N, L, q, gap, seed, xscale=0.1):
    """codes over q states (gap: plus the ignored gap, coded q), weights U(0.05, 1), x ~ N(0, xscale)"""
    if gap:
        c = alphabet_codes(N, L, q + 1, seed)                 # 0 = gap
        codes = np.where(c == 0, q, c - 1).astype(np.uint8)
    else:
        codes = alphabet_codes(N, L, q, seed)
    rng = np.random.default_rng(seed)
    w = rng.uniform(0.05, 1.0, N).astype(np.float32)
    x = rng.normal(0, xscale, L * q + L * (L - 1) // 2 * q * q).astype(np.float32)
    return np.ascontiguousarray(codes), w, x


# (q, gap ignored, L, N): L * q on or beside the tile edges, N beside the 192- and 256-sequence tiles
OBJECTIVE_CASES = [
    (2, False, 192, 257),     # Lq = 384 = 6 * 64 = 3 * 128 = 2 * 192
    (3, False, 128, 191),     # 384
    (3, True, 43, 257),       # 129: one beside 128
    (6, False, 64, 193),      # 384
    (6, True, 32, 255),       # 192
    (7, False, 55, 257),      # 385: one above 384
    (13, True, 15, 191),      # 195: beside 192
    (22, False, 17, 257),     # 374
    (22, True, 6, 300),       # 132
    (24, False, 16, 191),     # 384
    (25, True, 8, 257),       # 200
    (31, False, 7, 193),      # 217
    (31, True, 13, 193),      # 403
    (32, False, 12, 256),     # 384
    (32, False, 6, 257),      # 192
]


def tc_bytes(lib, N, L, q, gap_code, seq_chunk, sm):
    out = ctypes.c_int64()
    _lib.check(lib.evc_plm_tc_bytes_alphabet(N, L, q, gap_code, seq_chunk, sm, ctypes.byref(out)),
               "evc_plm_tc_bytes_alphabet")
    return int(out.value)


def gpu_eval(lib, codes, w, x, q, gap_code, precision, seq_chunk=0):
    """the evaluation of test_gpu_tc_edges on a handle of evc_plm_create_alphabet (tensor-core forward, lambda = 0)"""
    N, L = codes.shape
    h = ctypes.c_void_p()
    vp = ctypes.c_void_p
    _lib.check(lib.evc_plm_create_alphabet(ctypes.byref(h), codes.ctypes.data_as(vp), N, L, q, gap_code,
                                           w.ctypes.data_as(vp), 0), "evc_plm_create_alphabet")
    try:
        if seq_chunk:
            _lib.check(lib.evc_plm_set_seq_chunk(h, seq_chunk), "evc_plm_set_seq_chunk")
        _lib.check(lib.evc_plm_set_forward(h, 1), "evc_plm_set_forward")
        _lib.check(lib.evc_plm_set_precision(h, 1 if precision == "bf16" else 0), "evc_plm_set_precision")
        nbytes = int(lib.evc_plm_device_bytes(h))
        g = np.zeros_like(x)
        fx = np.zeros(2, dtype=np.float64)
        _lib.check(lib.evc_plm_eval_host(h, x.ctypes.data_as(vp), g.ctypes.data_as(vp), fx.ctypes.data_as(vp),
                                         0.0, 0.0), "evc_plm_eval_host")
    finally:
        lib.evc_plm_destroy(h)
    return dict(fx=fx[1], g=g, nll=fx[0], bytes=nbytes)


def _exact(codes, w, x, q, gap_code):
    fx, g, nll = po.objective(x.astype(np.float64), codes, w.astype(np.float64), q, 0.0, 0.0, gap_code)
    return fx, g


@pytest.mark.parametrize("q,gap,L,N", OBJECTIVE_CASES,
                         ids=lambda v: str(v) if not isinstance(v, bool) else ("ig" if v else "gs"))
def test_objective_vs_rounding_model(lib, q, gap, L, N):
    gap_code = q if gap else -1
    codes, w, x = make_inputs(N, L, q, gap, 1000 * q + L)
    sm = edges._sm_count(lib)
    geo = edges.geometry(N, L, q, gap, 0, sm)
    nbytes = tc_bytes(lib, N, L, q, gap_code, 0, sm)
    assert geo["bytes"] == nbytes, "geometry mirror out of date"
    print("\n[q=%d%s L=%d N=%d] %s" % (q, " gap ignored" if gap else "", L, N, edges._fmt_geometry(geo)))
    fx_e, g_e = _exact(codes, w, x, q, gap_code)
    key = ("alphabet", N, L, q, gap)
    for prec in ("fp32", "bf16"):
        got = gpu_eval(lib, codes, w, x, q, gap_code, prec)
        assert got["bytes"] == nbytes, (got["bytes"], nbytes)        # the real allocations
        m = edges.model(key, codes, w, x, q, gap_code, prec)
        edges.compare("  tc %s" % prec, got, m, L, q)
        if prec == "fp32":
            ge = np.linalg.norm(got["g"] - g_e) / np.linalg.norm(g_e)
            fe = abs(got["fx"] - fx_e) / abs(fx_e)
            print("  fp32 vs exact float64: grad rel L2 %.2e, fx rel %.1e" % (ge, fe))
            assert ge <= 2e-5 and fe <= 2e-6, (ge, fe)


@pytest.mark.parametrize("q,L", [(22, 12), (32, 10)])
def test_chunked_matches_unchunked(lib, q, L):
    N = 2001
    codes, w, x = make_inputs(N, L, q, False, 7 * q)
    whole = gpu_eval(lib, codes, w, x, q, -1, "fp32")
    for prec in ("fp32", "bf16"):
        ref = whole if prec == "fp32" else gpu_eval(lib, codes, w, x, q, -1, prec)
        got = gpu_eval(lib, codes, w, x, q, -1, prec, seq_chunk=768)
        nh = L * q
        assert got["fx"] == ref["fx"] and got["nll"] == ref["nll"], prec
        assert np.array_equal(got["g"][:nh], ref["g"][:nh]), prec
        m = edges.model(("chunk", N, L, q), codes, w, x, q, -1, prec)
        edges.compare("  3 chunks of 768, %s" % prec, got, m, L, q)
        d = np.abs(got["g"][nh:] - ref["g"][nh:]).reshape(-1, q * q)
        tol = 2 * edges.EPS_ACC * np.linalg.norm(m["g_abs"][nh:].reshape(-1, q * q), axis=1)
        assert (np.linalg.norm(d, axis=1) <= tol).all(), prec


@pytest.mark.parametrize("q,gap,N,L,chunk", [(3, False, 300, 50, 0), (13, True, 769, 20, 0), (22, False, 257, 14, 0),
                                             (32, False, 1537, 9, 768), (31, True, 300, 9, 0)])
def test_weighted_counts_vs_rounding_model(engine, q, gap, N, L, chunk):
    codes, _w, _x = make_inputs(N, L, q, gap, 17 + q)
    w = (1.0 / np.random.default_rng(17).integers(1, 50, N)).astype(np.float32)
    p = engine.plm_problem(codes, w, q, q if gap else -1, 0.0, 0.0, forward="tc", seq_chunk=chunk)
    try:
        fic, fijc = p.weighted_counts()
    finally:
        p.close()
    fi, fij = model_io.normalise_frequencies(fic, fijc, float(w.astype(np.float64).sum()), gap)
    fi_m, fij_m = po.frequencies(codes, w.astype(np.float64), q, q if gap else -1, weights="hi+lo")
    assert np.abs(fi - fi_m).max() <= 2.0 ** -21 * np.abs(fi_m).max()
    assert (np.abs(fij - fij_m) <= 2.0 ** -20 * fij_m).all()


@pytest.mark.parametrize("n_codes", [32, 31])
def test_hamming_counts_with_codes_up_to_31(engine, lib, n_codes):
    """q = 32 (codes 0..31), and q = 31 with the ignored gap coded 31"""
    rng = np.random.default_rng(5)
    centres = rng.integers(0, n_codes, size=(14, 70))
    codes = centres[rng.integers(0, 14, size=700)]
    mut = rng.random(codes.shape) < rng.uniform(0.0, 0.3, size=700)[:, None]      # identities around 0.8
    codes = np.where(mut, rng.integers(0, n_codes, size=codes.shape), codes).astype(np.uint8)
    if n_codes == 31:
        codes[rng.random(codes.shape) < 0.02] = 31                                    # the ignored gap
    assert codes.max() == 31
    for theta in (0.8, 0.5):
        thr = msa.identity_threshold_count(theta, codes.shape[1])
        ref = co.hamming_counts(codes, thr)
        assert ref.max() > 1
        assert np.array_equal(engine.hamming_counts(codes, thr), ref)
        got = np.zeros(codes.shape[0], dtype=np.int32)
        vp = ctypes.c_void_p
        _lib.check(lib.evc_hamming_counts(codes.ctypes.data_as(vp), codes.shape[0], codes.shape[1], thr, 0,
                                          got.ctypes.data_as(vp)), "evc_hamming_counts")
        assert np.array_equal(got, ref)


@pytest.mark.parametrize("alphabet,L", [(PROTEIN_X, 40), (DNA_N, 40), (TWO_LETTERS, 24)],
                         ids=lambda v: "q%d" % len(v) if isinstance(v, str) else "L%d" % v)
def test_run_plmc_converges_to_the_float64_optimum(engine, tmp_path, alphabet, L):
    """N = 200 sequences as config 1 of test_gpu_parity.py.  The fit ends when the float32 objective no longer
    resolves a line-search step (LBFGSERR_ROUNDING_ERROR), which is where the EC rms stands then depends on the
    shape.  On an H100: q = 22 at 3.6e-5 (L = 24) and passes at L = 40; q = 6 at 1.6e-4 (L = 24) and 5.9e-5 (L = 40);
    q = 2 at 4.5e-5 (L = 24) and 1.5e-4 (L = 40); the objective gap stayed below 1e-6 in all six."""
    q, N = len(alphabet), 200
    codes = alphabet_codes(N, L, q, 11 + q)
    a2m = tmp_path / "a.a2m"
    write_alphabet_a2m(str(a2m), codes, alphabet)
    lam_J = 0.01 * (q - 1) * (L - 1)
    res, run = tools.run_plmc(str(a2m), str(tmp_path / "o_ECs.txt"), str(tmp_path / "o.model"), alphabet=alphabet,
                              theta=0.8, iterations=3000, lambda_h=0.01, lambda_J=lam_J, engine=engine,
                              return_run=True, epsilon=1e-5)
    ali = run.alignment
    assert ali.q == q and np.array_equal(ali.codes, codes)
    w = 1.0 / co.hamming_counts(ali.codes, msa.identity_threshold_count(0.8, L))
    assert np.allclose(run.weights, w)
    xo, _info = po.fit(ali.codes, w, q, 0.01, lam_J, -1, x0=tools.initial_point(
        po.frequencies(ali.codes, w, q, -1)[0], w.sum(), L, q).astype(np.float64), max_iter=4000,
        objective_fn=lambda v: co.plm_eval(ali.codes, w, v, q, 0.01, lam_J, "f64"))
    m = model_ops.read_model(str(tmp_path / "o.model"))
    assert (m["q"], m["alphabet"], m["L"]) == (q, alphabet, L)
    x = np.concatenate([m["h"].ravel(), m["J"].ravel()]).astype(np.float64)
    cn = np.loadtxt(str(tmp_path / "o_ECs.txt"), usecols=5)
    cn_o = po.cn_scores(xo[L * q:].reshape(-1, q, q), L)
    f_gpu = po.objective(x, ali.codes, w, q, 0.01, lam_J, -1)[0]
    f_opt = po.objective(xo, ali.codes, w, q, 0.01, lam_J, -1)[0]
    rms = float(np.sqrt(np.mean((cn - cn_o) ** 2)))
    print("q=%d: %s after %d iterations, cn rms %.2e, rel objective gap %.2e"
          % (q, res.optimization_status, run.lbfgs.iterations, rms, (f_gpu - f_opt) / f_opt))
    assert rms <= 1e-4
    assert 0 <= (f_gpu - f_opt) / f_opt <= 1e-6


def test_cli_alphabets(tmp_path):
    """bin/evcplm-plmc -a with the three alphabets of the end-to-end test (a new process per run)"""
    for alphabet in (PROTEIN_X, DNA_N, TWO_LETTERS):
        q = len(alphabet)
        a2m = tmp_path / ("a%d.a2m" % q)
        write_alphabet_a2m(str(a2m), alphabet_codes(150, 12, q, q), alphabet)
        ecs, model = tmp_path / ("e%d_ECs.txt" % q), tmp_path / ("m%d.model" % q)
        p = subprocess.run([sys.executable, os.path.join(ROOT, "bin", "evcplm-plmc"), "-c", str(ecs), "-o", str(model),
                            "-a", alphabet, "-m", "50", "-le", "%g" % (0.01 * (q - 1) * 11), str(a2m)],
                           capture_output=True, text=True, timeout=600)
        assert p.returncode == 0, p.stderr[-2000:]
        assert "150 valid sequences out of 150" in p.stderr
        m = model_ops.read_model(str(model))
        assert (m["q"], m["alphabet"], m["L"]) == (q, alphabet, 12)
        assert len(open(ecs).read().strip().split("\n")) == 12 * 11 // 2


def _consumer_model(L, q, seed):
    rng = np.random.default_rng(seed)
    npair = L * (L - 1) // 2
    fi = rng.dirichlet(np.ones(q), size=L).astype(np.float32)
    fij = rng.dirichlet(np.ones(q * q), size=npair).reshape(npair, q, q).astype(np.float32)
    fi[0, : q // 2] = 0.0
    fij[:, 0, :] = 0.0
    return dict(L=L, q=q, h=rng.normal(0, 0.5, (L, q)).astype(np.float32),
                J=rng.normal(0, 0.2, (npair, q, q)).astype(np.float32), fi=fi, fij=fij, alphabet=alphabet_of(q))


@pytest.mark.parametrize("gaps", [False, True])
@pytest.mark.parametrize("q", [3, 22, 32])
@pytest.mark.parametrize("L", [2, 13, 25])
def test_hamiltonians_every_row(engine, L, q, gaps):
    """tolerances of test_gpu_model_ops_alphabets.py; L = 13 / 25 span two / three 12-site chunks at S = 33"""
    m = _consumer_model(L, q, 100 * L + q)
    rng = np.random.default_rng(L + q)
    if gaps and q == 32:
        codes = rng.integers(0, q + 1, size=(5, L)).astype(np.uint8)
        codes[0, 0] = q
        with pytest.raises(ValueError, match="no code left"):
            model_ops.hamiltonians(m, codes, engine)
        return
    J = po.full_couplings(m["J"].astype(np.float64), L, q)
    Jp = np.zeros((L, L, q + 1, q + 1))
    Jp[:, :, :q, :q] = J
    hp = np.zeros((L, q + 1))
    hp[:, :q] = m["h"]
    for N in (1, 511, 513):
        codes = rng.integers(0, q, size=(N, L)).astype(np.uint8)
        if gaps:
            codes[rng.random((N, L)) < 0.15] = q
            codes[0, :] = q
        H = model_ops.hamiltonians(m, codes, engine)
        i, j = np.triu_indices(L, 1)
        terms = Jp[i[None, :], j[None, :], codes[:, i], codes[:, j]]
        hj, hh = terms.sum(axis=1), hp[np.arange(L)[None, :], codes].sum(axis=1)
        scale = np.abs(terms).sum(axis=1) + np.abs(hp[np.arange(L)[None, :], codes]).sum(axis=1)
        tol = L * 2.0 ** -24 * scale + 1e-12
        for col, ref in ((0, hj + hh), (1, hj), (2, hh)):
            bad = np.nonzero(np.abs(H[:, col] - ref) > tol)[0]
            assert len(bad) == 0, (L, q, gaps, N, col, bad[:5])
        if gaps:
            assert H[0, 0] == 0.0 and H[0, 1] == 0.0 and H[0, 2] == 0.0


@pytest.mark.parametrize("q", [3, 22, 32])
@pytest.mark.parametrize("L", [2, 25])
def test_pair_scores_every_pair(engine, L, q):
    m = _consumer_model(L, q, 7 * L + q)
    fn_raw, fn_zs, mi = model_ops.pair_scores(m, engine)
    J = m["J"].astype(np.float64)
    raw = np.sqrt((J ** 2).sum(axis=(1, 2)))
    Jz = J - J.mean(axis=1, keepdims=True) - J.mean(axis=2, keepdims=True) + J.mean(axis=(1, 2), keepdims=True)
    zs = np.sqrt((Jz ** 2).sum(axis=(1, 2)))
    i, j = np.triu_indices(L, 1)
    F = m["fij"].astype(np.float64)
    P = m["fi"].astype(np.float64)[i][:, :, None] * m["fi"].astype(np.float64)[j][:, None, :]
    ok = (F > 0) & (P > 0)
    t = np.where(ok, F * np.log(np.where(ok, F, 1.0) / np.where(ok, P, 1.0)), 0.0)
    mi_ref = t.sum(axis=(1, 2))
    assert (np.abs(fn_raw - raw) <= 2.0 ** -23 * raw + 1e-30).all()
    assert (np.abs(fn_zs - zs) <= 2.0 ** -23 * zs + 1e-12 * raw).all()
    assert (np.abs(mi - mi_ref) <= 2.0 ** -23 * np.abs(mi_ref) + 1e-12 * np.abs(t).sum(axis=(1, 2))).all()


def test_plm_create_alphabet_argument_checks(lib):
    """evc_plm_create_alphabet checks the arguments evc_plm_create checks, with q = 33 as the out-of-range alphabet,
    and takes q = 7, which evc_plm_create refuses"""
    vp = ctypes.c_void_p
    codes = np.zeros((4, 6), dtype=np.uint8)
    w = np.ones(4, dtype=np.float32)
    h = ctypes.c_void_p()
    for q, gap in ((33, -1), (21, 5), (32, 32)):
        rc = lib.evc_plm_create_alphabet(ctypes.byref(h), codes.ctypes.data_as(vp), 4, 6, q, gap, w.ctypes.data_as(vp),
                                         0)
        assert rc != 0 and lib.evc_last_error()
    assert lib.evc_plm_create_alphabet(ctypes.byref(h), codes.ctypes.data_as(vp), 0, 6, 21, -1, w.ctypes.data_as(vp),
                                       0) != 0
    assert lib.evc_plm_create(ctypes.byref(h), codes.ctypes.data_as(vp), 4, 6, 7, -1, w.ctypes.data_as(vp), 0) != 0
    _lib.check(lib.evc_plm_create_alphabet(ctypes.byref(h), codes.ctypes.data_as(vp), 4, 6, 7, -1,
                                           w.ctypes.data_as(vp), 0), "evc_plm_create_alphabet")
    assert lib.evc_plm_num_params(h) == 6 * 7 + 15 * 49
    lib.evc_plm_destroy(h)


def test_gather_kernels_refuse_other_alphabets(engine, lib):
    q, N, L = 22, 100, 6
    codes, w, x = make_inputs(N, L, q, False, 3)
    for fwd, bwd in (("gather", "gather"), ("gather", "tc")):
        with pytest.raises(_lib.EngineError, match=r"evc_plm_set_forward\(h, 1\)"):
            engine.plm_problem(codes, w, q, -1, 0.0, 0.0, forward=fwd, backward=bwd, seq_chunk=0)
    # a raw C handle left at the C defaults (gather forward and backward)
    vp = ctypes.c_void_p
    h = ctypes.c_void_p()
    _lib.check(lib.evc_plm_create_alphabet(ctypes.byref(h), codes.ctypes.data_as(vp), N, L, q, -1,
                                           w.ctypes.data_as(vp), 0), "evc_plm_create_alphabet")
    try:
        g = np.zeros_like(x)
        fx = np.zeros(2)
        assert lib.evc_plm_eval_host(h, x.ctypes.data_as(vp), g.ctypes.data_as(vp), fx.ctypes.data_as(vp), 0.0,
                                     0.0) != 0
        assert b"evc_plm_set_forward(h, 1)" in lib.evc_last_error(), lib.evc_last_error()
        assert lib.evc_plm_set_backward(h, 0) != 0 and b"evc_plm_set_forward(h, 1)" in lib.evc_last_error()
        assert lib.evc_plm_set_forward(h, 0) != 0 and b"evc_plm_set_forward(h, 1)" in lib.evc_last_error()
        # the tensor-core path then evaluates this handle
        _lib.check(lib.evc_plm_set_forward(h, 1), "evc_plm_set_forward")
        _lib.check(lib.evc_plm_eval_host(h, x.ctypes.data_as(vp), g.ctypes.data_as(vp), fx.ctypes.data_as(vp), 0.0,
                                         0.0), "evc_plm_eval_host")
        assert np.isfinite(fx).all() and np.isfinite(g).all()
    finally:
        lib.evc_plm_destroy(h)
