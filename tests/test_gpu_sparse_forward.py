"""The 2:4-sparse tensor-core forward on the device (-m gpu): the one-hot operand byte for byte against the numpy
specification in test_sparse_onehot_format.py, the logits against the float64 rounding model at every 2:4 pattern,
switching between the sparse and the fused forward on one handle, and bit-identical results for both cluster sizes."""
import ctypes
import importlib.util
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from evcouplings_b200 import _lib  # noqa: E402


def _load(name):
    spec = importlib.util.spec_from_file_location("_sf_" + name, os.path.join(HERE, name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


fmt = _load("test_sparse_onehot_format")
edges = _load("test_gpu_tc_edges")


@pytest.fixture(scope="module")
def lib():
    l = _lib.load()
    _lib.require_device()
    return l


def _handle(lib, codes, q, gap_code, w=None, seq_chunk=0):
    N, L = codes.shape
    w = np.ones(N, dtype=np.float32) if w is None else w
    h = ctypes.c_void_p()
    vp = ctypes.c_void_p
    _lib.check(lib.evc_plm_create_alphabet(ctypes.byref(h), codes.ctypes.data_as(vp), N, L, q, gap_code,
                                           w.ctypes.data_as(vp), 0), "evc_plm_create_alphabet")
    if seq_chunk:
        _lib.check(lib.evc_plm_set_seq_chunk(h, seq_chunk), "evc_plm_set_seq_chunk")
    return h


def _copy(lib, h, xrows, kw):
    buf = np.zeros(xrows * kw * 2, dtype=np.uint8)
    _lib.check(lib.evc_plm_copy_onehot(h, buf.ctypes.data_as(ctypes.c_void_p), buf.size), "evc_plm_copy_onehot")
    return buf


def _eval(lib, h, x):
    g = np.zeros_like(x)
    fx = np.zeros(2, dtype=np.float64)
    vp = ctypes.c_void_p
    _lib.check(lib.evc_plm_eval_host(h, x.ctypes.data_as(vp), g.ctypes.data_as(vp), fx.ctypes.data_as(vp), 0.0, 0.0),
               "evc_plm_eval_host")
    return fx, g


FORMAT_CASES = [(q, gap, off) for q, gap in ((2, False), (3, False), (4, False), (5, False), (20, True), (21, False),
                                             (32, False)) for off in range(4)]


@pytest.mark.parametrize("q,gap,off", FORMAT_CASES)
def test_device_operand_matches_the_model(lib, q, gap, off):
    """q in {2, 3, 4, 5, 20 (ignored gap), 21, 32}, L so that the last site ends at offset `off` of a group of 4
    where q allows it; N = 300 leaves rows beyond N in the 384-row allocation."""
    L = next((L for L in range(7, 11) if (L * q) % 4 == off), None)
    if L is None:
        pytest.skip("q = %d never ends a site at offset %d of a group" % (q, off))
    N = 300
    codes = fmt._codes(N, L, q, gap, 11 * q + off)
    h = _handle(lib, codes, q, q if gap else -1)
    try:
        _lib.check(lib.evc_plm_set_forward(h, 1), "evc_plm_set_forward")
        xrows, kw = fmt._ru(N, 384), fmt._ru(L * q, 64)
        got = _copy(lib, h, xrows, kw)
    finally:
        lib.evc_plm_destroy(h)
    want = fmt.sparse_onehot(fmt.dense_onehot(codes, q, 0, N, xrows, kw))
    assert np.array_equal(got[:want.size], want)


def test_device_operand_of_the_last_chunk(lib):
    """Sequence chunks: after an evaluation the buffer holds the last chunk (n0 = 1536 > 0, 264 real rows of 768)."""
    N, L, q = 1800, 13, 21
    codes = fmt._codes(N, L, q, False, 5)
    h = _handle(lib, codes, q, -1, seq_chunk=768)
    try:
        _lib.check(lib.evc_plm_set_forward(h, 1), "evc_plm_set_forward")
        x = np.random.default_rng(0).normal(0, 0.1, L * q + L * (L - 1) // 2 * q * q).astype(np.float32)
        _eval(lib, h, x)
        got = _copy(lib, h, 768, fmt._ru(L * q, 64))
    finally:
        lib.evc_plm_destroy(h)
    want = fmt.sparse_onehot(fmt.dense_onehot(codes, q, 1536, N - 1536, 768, fmt._ru(L * q, 64)))
    assert np.array_equal(got[:want.size], want)


# every 2:4 pattern: q = 2 and 3 put a site boundary at each position of a group and give groups with 0, 1 and 2
# nonzeros (the ignored gap and an all-gap row give empty and one-nonzero groups); q = 6, 7 and 9 move the boundary
# through the group along K.  (q, ignored gap, L, N)
PATTERN_CASES = [(2, False, 40, 300), (3, False, 41, 300), (3, True, 33, 300), (6, False, 37, 257), (7, True, 29, 385),
                 (9, False, 23, 129)]


@pytest.mark.parametrize("q,gap,L,N", PATTERN_CASES)
def test_sparse_logits_vs_rounding_model(lib, q, gap, L, N):
    gap_code = q if gap else -1
    codes = fmt._codes(N, L, q, gap, 31 * q + L)
    if gap:
        codes[7] = q
    rng = np.random.default_rng(q + L)
    w = rng.uniform(0.05, 1.0, N).astype(np.float32)
    x = rng.normal(0, 0.1, L * q + L * (L - 1) // 2 * q * q).astype(np.float32)
    for prec in ("fp32", "bf16"):
        h = _handle(lib, codes, q, gap_code, w=w)
        try:
            _lib.check(lib.evc_plm_set_forward(h, 1), "evc_plm_set_forward")
            _lib.check(lib.evc_plm_set_precision(h, 1 if prec == "bf16" else 0), "evc_plm_set_precision")
            fx, g = _eval(lib, h, x)
        finally:
            lib.evc_plm_destroy(h)
        m = edges.model(("sparse", N, L, q, gap), codes, w, x, q, gap_code, prec)
        edges.compare("  tc %s q=%d L=%d N=%d" % (prec, q, L, N), dict(fx=fx[1], g=g, nll=fx[0]), m, L, q)


def test_forward_mode_switch_keeps_results(lib):
    """One handle: sparse (1) -> fused (2, dense operand) -> sparse (1); the sparse results repeat bit for bit."""
    N, L, q = 500, 30, 21
    codes, w, x = edges.make_inputs(N, L, q, False, 3)
    h = _handle(lib, codes, q, -1, w=w)
    try:
        out = []
        for mode in (1, 2, 1):
            _lib.check(lib.evc_plm_set_forward(h, mode), "evc_plm_set_forward")
            out.append(_eval(lib, h, x))
    finally:
        lib.evc_plm_destroy(h)
    assert np.array_equal(out[0][0], out[2][0]) and np.array_equal(out[0][1], out[2][1])
    assert abs(out[1][0][1] - out[0][0][1]) <= 2e-6 * abs(out[0][0][1])
    assert np.linalg.norm(out[1][1] - out[0][1]) <= 2e-5 * np.linalg.norm(out[0][1])


_CHILD = r'''
import json, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from evcouplings_b200.engine import CudaEngine
from evcouplings_b200 import synthetic
eng = CudaEngine()
res = {}
for N, L, q in ((300, 50, 21), (1000, 70, 4)):
    codes = synthetic.synthetic_msa_codes(N, L, 1)
    if q == 4:
        codes = (codes % 4).astype(np.uint8)
    rng = np.random.default_rng(N)
    w = rng.uniform(0.1, 1, N).astype(np.float32)
    x = rng.normal(0, 0.1, L * q + L * (L - 1) // 2 * q * q).astype(np.float32)
    for prec in ("fp32", "bf16"):
        p = eng.plm_problem(codes, w, q, -1, 0.01, 1.0, forward="tc", backward="tc", precision=prec, m=3)
        p.set_x(x)
        fx = p.evaluate(p.x)
        res["%d/%s" % (N, prec)] = [float(fx), p.g.cpu().numpy().astype(np.float64).tobytes().hex()]
        p.close()
print(json.dumps(res))
'''


def test_cluster_sizes_are_bit_identical(lib):
    """EVC_FWD_CLUSTER = 1 and 2 (read once per process, so each in its own process) give the same bits, with an odd
    number of 128-sequence tiles (N = 300: 3; N = 1000: 8)."""
    out = {}
    for cs in ("1", "2"):
        env = dict(os.environ, EVC_FWD_CLUSTER=cs)
        r = subprocess.run([sys.executable, "-c", _CHILD, ROOT], env=env, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        out[cs] = json.loads(r.stdout.strip().splitlines()[-1])
    assert out["1"] == out["2"]
