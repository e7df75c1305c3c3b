"""
Tensor-core objective at the tile, chunk and alphabet edges (-m gpu), against a float64 model of its own arithmetic.

The reference is ``po.objective(..., operands=...)``: the couplings and the backward product's residuals rounded to
bf16 exactly as expand_tc_kernel and the softmax kernels round them (hi + lo in precision mode 0 "fp32", hi only in
mode 1 "bf16"), the one-hot operand exact, every sum in float64.  What remains between the device and that model
is the device's own float32 arithmetic, so the tolerances can be tight in BOTH precision modes.

Error model, per site (g_h) and per coupling block (g_J), in L2 over the block B:
    || g_gpu - g_model ||_B  <=  EPS_ACC * || g_abs ||_B  +  || g_flip ||_B
* g_abs: per entry, the sum of |terms| of the model's products (oracle ``bounds``).  EPS_ACC = 2^-16 covers the
  float32 accumulation of the wgmma products (tensor-core adds that do not round to nearest, in K chains of at most
  32 blocks of 64 before an IEEE add), the float32 logits, expf / logf and the per-tile partial sums.
* g_flip: per entry, the sum over its terms of the largest change of the residual operand when the residual moves by
  NU * w (the oracle's ``bounds=NU``): a residual within float32 noise of a bf16 rounding boundary can round to the
  other neighbour on the device.  In hi-only mode that is one bf16 step of that term; in hi + lo mode about NU * w.
  NU = 2^-18 (about 30 float32 ulps of the weight).
Whole gradient: relative L2 <= 2e-5 in both modes (250x tighter than the 5e-3 that bounds the bf16 mode against
exact operands in test_gpu_parity.py).  fx and -loglk: relative 2e-6 (float32 logits, float64 sums of the
per-sequence terms).
The per-block relative L2 error was estimated at about 1e-5 in both modes from the shapes.  Measured over this
file on an H100 80GB HBM3 (400 W power limit): per-block relative L2 at most 2.8e-6 (fp32) and 5.5e-5 (bf16, at
L = 390, N = 200: small blocks where one residual rounded to the other neighbour is a large share), whole-vector 1.0e-6 / 7.3e-6, fx
1.0e-6 / 3e-8, error / tolerance at most 0.08 / 0.52.  The measured values are printed per case next to the error
of the C/OpenMP fp32 port against float64 (the yardstick of _check_eval in test_gpu_parity.py).

Every shape below names the tile edge it targets; the geometry table (Mp, Np, Kw, Ns, Kp, Xrows, ksplit) is printed
for each case and checked against the library's own byte count (evc_plm_tc_bytes), which is built from the same
geometry.
"""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))

from evcouplings_b200 import _lib, model_io, synthetic  # noqa: E402
from oracle import c_oracle as co  # noqa: E402
from oracle import plm_oracle as po  # noqa: E402

EPS_ACC = 2.0 ** -16
NU = 2.0 ** -18
FX_REL = 2e-6
VEC_REL = 2e-5
OPERANDS = {"fp32": "hi+lo", "bf16": "hi"}


@pytest.fixture(scope="module")
def lib():
    l = _lib.load()
    _lib.require_device()
    return l


def _ru(a, b):
    return -(-a // b) * b


def _sm_count(lib):
    sm = ctypes.c_int32()
    _lib.check(lib.evc_device_info(0, ctypes.byref(sm), None, None, None), "evc_device_info")
    return int(sm.value)


def _ksplit(tiles, num_kb, sm):
    """backward_ksplit of plm_tc.cu (EVC_KSPLIT honoured like the library does)"""
    e = int(os.environ.get("EVC_KSPLIT", "0") or 0)
    ks = 1
    if e > 0:
        ks = min(e, 8)
    else:
        best = 0.0
        for s in range(1, 5):
            if s > num_kb:
                break
            units = tiles * s
            eff = units / (sm * -(-units // sm))
            if eff >= 0.97:
                ks = s
                break
            if eff > best:
                best, ks = eff, s
    ks = max(1, min(ks, num_kb))
    return -(-num_kb // -(-num_kb // ks))


def geometry(N, L, q, gap, seq_chunk, sm):
    """The tensor-core geometry of plm_tc_geometry / plm_tcf_geometry / plm_tcff_geometry, and the byte count
    evc_plm_tc_bytes derives from it (checked against the library in run_case)."""
    lq = L * q
    c = _ru(seq_chunk, 768) if seq_chunk > 0 else 0
    C = N if (c == 0 or c >= N) else c
    n_chunks = -(-N // C)
    Mp, Np, Kw, Kp = _ru(lq, 128), _ru(lq, 192), _ru(lq, 64), _ru(C, 64)
    tiles = (Mp // 128) * (Np // 192)
    kp_last = _ru(min(C, N - (n_chunks - 1) * C), 64)
    g = dict(N=N, L=L, q=q, Lq=lq, C=C, n_chunks=n_chunks, Mp=Mp, Np=Np, Kw=Kw, Kp=Kp, Ns=_ru(C, 192),
             Xrows=_ru(C, 384), ksplit=_ksplit(tiles, Kp // 64, sm), ksplit_last=_ksplit(tiles, kp_last // 64, sm))
    g["planes"] = max(g["ksplit"], g["ksplit_last"])
    g["m_tiles"] = Mp // 128
    g["mgroup"] = {p: max(1, min(g["m_tiles"], int(24e6 / (128.0 * Kw * 2 * (2 if p == "fp32" else 1)))))
                   for p in ("fp32", "bf16")}
    g["fused"] = (q in (20, 21)) and lq <= 8192 and n_chunks == 1
    S = q if q % 2 else q + 1
    ntiles_s = -(-N // 256)
    g["bytes"] = (N * L + (_ru(L, 4) // 4) * _ru(N, 32) * 4 + 4 * N + Mp * Kp * 2 + 2 * Np * Kp * 2
                  + g["planes"] * Mp * Np * 4 + g["Xrows"] * Kw * 2 + 2 * Mp * Kw * 2 + Mp * g["Ns"] * 4
                  + L * ntiles_s * S * 4 + L * ntiles_s * 8)
    return g


def _fmt_geometry(g):
    return ("Lq=%d Mp=%d Np=%d Kw=%d Ns=%d Kp=%d Xrows=%d ksplit=%d/%d chunks=%d mgroup=%d/%d of %d"
            % (g["Lq"], g["Mp"], g["Np"], g["Kw"], g["Ns"], g["Kp"], g["Xrows"], g["ksplit"], g["ksplit_last"],
               g["n_chunks"], g["mgroup"]["fp32"], g["mgroup"]["bf16"], g["m_tiles"]))


def tc_bytes(lib, N, L, q, gap_code, seq_chunk, sm):
    out = ctypes.c_int64()
    _lib.check(lib.evc_plm_tc_bytes(N, L, q, gap_code, seq_chunk, sm, ctypes.byref(out)), "evc_plm_tc_bytes")
    return int(out.value)


# ------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------
def make_inputs(N, L, q, gap, seed, xscale=0.1, special=None):
    """Synthetic alignment in the code convention of q / gap (gap: ignored gap code q), uniform weights, normal x.
    special: "gaps" (sequence 7 % N all gaps, site 5 % L all gaps, every third weight and the last one zero),
    "zero_w" (all weights zero)."""
    codes = synthetic.synthetic_msa_codes(N, L, seed)
    if q in (4, 5):
        codes = (codes % 5).astype(np.uint8)             # q = 4 with gap: code 4 is the ignored gap
    elif gap:
        codes = synthetic.to_ignore_gaps_codes(codes, q)
    gap_sym = q if gap else 0
    rng = np.random.default_rng(seed)
    w = rng.uniform(0.05, 1.0, N).astype(np.float32)
    if special == "gaps":
        codes[7 % N, :] = gap_sym
        codes[:, 5 % L] = gap_sym
        w[::3] = 0.0
        w[-1] = 0.0
    elif special == "zero_w":
        w[:] = 0.0
    x = rng.normal(0, xscale, L * q + L * (L - 1) // 2 * q * q).astype(np.float32)
    return np.ascontiguousarray(codes), w, x


def gpu_eval(lib, codes, w, x, q, gap_code, forward, precision, seq_chunk=0):
    """One evaluation through the C ABI (lambda = 0: the data term only).  Returns fx, g, -loglk and the handle's
    device bytes before the evaluation (these tell the fused forward from its unfused fallback)."""
    N, L = codes.shape
    h = ctypes.c_void_p()
    vp = ctypes.c_void_p
    _lib.check(lib.evc_plm_create(ctypes.byref(h), codes.ctypes.data_as(vp), N, L, q, gap_code, w.ctypes.data_as(vp),
                                  0), "evc_plm_create")
    try:
        if seq_chunk:
            _lib.check(lib.evc_plm_set_seq_chunk(h, seq_chunk), "evc_plm_set_seq_chunk")
        _lib.check(lib.evc_plm_set_forward(h, 2 if forward == "tcfused" else 1), "evc_plm_set_forward")
        _lib.check(lib.evc_plm_set_precision(h, 1 if precision == "bf16" else 0), "evc_plm_set_precision")
        nbytes = int(lib.evc_plm_device_bytes(h))
        g = np.zeros_like(x)
        fx = np.zeros(2, dtype=np.float64)
        _lib.check(lib.evc_plm_eval_host(h, x.ctypes.data_as(vp), g.ctypes.data_as(vp), fx.ctypes.data_as(vp),
                                         0.0, 0.0), "evc_plm_eval_host")
    finally:
        lib.evc_plm_destroy(h)
    return dict(fx=fx[1], g=g, nll=fx[0], bytes=nbytes)


_MODEL_CACHE = {}


def model(key, codes, w, x, q, gap_code, precision):
    k = (key, precision)
    if k not in _MODEL_CACHE:
        if len(_MODEL_CACHE) > 8:
            _MODEL_CACHE.clear()
        fx, g, nll, b = po.objective(x.astype(np.float64), codes, w.astype(np.float64), q, 0.0, 0.0, gap_code,
                                     operands=OPERANDS[precision], bounds=NU)
        _MODEL_CACHE[k] = dict(fx=fx, g=g, nll=nll, **b)
    return _MODEL_CACHE[k]


def _blocks(v, L, q):
    nh = L * q
    return v[:nh].reshape(L, q), v[nh:].reshape(-1, q * q)


def compare(label, got, m, L, q, yard=None):
    """Asserts the error model of the module docstring per site and per coupling block; prints the measured
    errors.  Returns (max per-block relative L2 error, max error / tolerance)."""
    d = got["g"].astype(np.float64) - m["g"]
    worst_rel, worst_ratio = 0.0, 0.0
    for dv, mv, av, fv in zip(_blocks(d, L, q), _blocks(m["g"], L, q), _blocks(m["g_abs"], L, q),
                              _blocks(m["g_flip"], L, q)):
        err = np.linalg.norm(dv, axis=1)
        tol = EPS_ACC * np.linalg.norm(av, axis=1) + np.linalg.norm(fv, axis=1)
        ref = np.linalg.norm(mv, axis=1)
        nz = ref > 0
        if nz.any():
            worst_rel = max(worst_rel, float((err[nz] / ref[nz]).max()))
        pos = tol > 0
        if pos.any():
            worst_ratio = max(worst_ratio, float((err[pos] / tol[pos]).max()))
        bad = np.nonzero(err > tol)[0]
        assert len(bad) == 0, "%s: %d blocks over tolerance, first %d: err %.3e tol %.3e ref %.3e" % (
            label, len(bad), bad[0], err[bad[0]], tol[bad[0]], ref[bad[0]])
    fx_rel = abs(got["fx"] - m["fx"]) / max(abs(m["fx"]), 1e-300)
    nll_rel = abs(got["nll"] - m["nll"]) / max(abs(m["nll"]), 1e-300)
    gn = np.linalg.norm(m["g"])
    assert np.linalg.norm(d) <= VEC_REL * gn, (label, np.linalg.norm(d) / gn)
    assert abs(got["fx"] - m["fx"]) <= FX_REL * abs(m["fx"]), (label, got["fx"], m["fx"])
    assert abs(got["nll"] - m["nll"]) <= FX_REL * abs(m["nll"]), (label, got["nll"], m["nll"])
    print("%-58s block rel L2 max %.2e (err/tol %.2f), vector rel L2 %.2e, fx rel %.1e%s" % (
        label, worst_rel, worst_ratio, np.linalg.norm(d) / gn if gn > 0 else 0.0, max(fx_rel, nll_rel),
        "" if yard is None else ", C fp32 port vs float64 %.2e" % yard))
    return worst_rel, worst_ratio


def yardstick(codes, w, x, q):
    _f, g64, _n = co.plm_eval(codes, w.astype(np.float64), x.astype(np.float64), q, 0.0, 0.0, "f64")
    _f, g32, _n = co.plm_eval(codes, w, x, q, 0.0, 0.0, "f32")
    n = np.linalg.norm(g64)
    return float(np.linalg.norm(g32 - g64) / n) if n > 0 else 0.0


def run_case(lib, case, forwards=("tc", "tcfused"), precisions=("fp32", "bf16"), env_results=None):
    """Evaluate one input set on the device for every forward / precision and compare with the model.
    env_results: device results computed in a subprocess (keyed like the loop below) instead of in-process."""
    N, L, q, gap = case["N"], case["L"], case["q"], case["gap"]
    gap_code = q if gap else -1
    codes, w, x = make_inputs(N, L, q, gap, case.get("seed", 1), case.get("xscale", 0.1), case.get("special"))
    sm = _sm_count(lib)
    chunk = case.get("seq_chunk", 0)
    geo = geometry(N, L, q, gap, chunk, sm)
    if env_results is None:
        assert geo["bytes"] == tc_bytes(lib, N, L, q, gap_code, chunk, sm), "geometry mirror out of date"
    print("\n[%s] N=%d L=%d q=%d%s: %s" % (case["target"], N, L, q, " (gap ignored)" if gap else "",
                                          _fmt_geometry(geo)))
    yard = yardstick(codes, w, x, q)
    key = (N, L, q, gap, case.get("seed", 1), case.get("xscale", 0.1), case.get("special"))
    out = {}
    for prec in precisions:
        m = model(key, codes, w, x, q, gap_code, prec)
        for fwd in forwards:
            if env_results is not None:
                got = env_results["%s/%s" % (fwd, prec)]
            else:
                got = gpu_eval(lib, codes, w, x, q, gap_code, fwd, prec, chunk)
                # the unfused forward owns exactly the buffers evc_plm_tc_bytes counts; the fused one does not
                unfused = got["bytes"] == tc_bytes(lib, N, L, q, gap_code, chunk, sm)
                assert unfused == (fwd == "tc" or not geo["fused"]), (fwd, geo["fused"], got["bytes"])
            out[(fwd, prec)] = compare("  %s %s%s" % (fwd, prec, "" if fwd == "tc" or geo["fused"] else
                                                       " (falls back to tc)"), got, m, L, q, yard)
    return out


# ------------------------------------------------------------------------------------------------
# 1. L*q on and around every tile edge; the fused forward's 8-site tiles and its L*q <= 8192 limit
# ------------------------------------------------------------------------------------------------
SITE_CASES = [
    # q = 21: 2688 = 21 * 128 = 14 * 192 = 42 * 64 (no padding in M, N or K); L = 128 = 16 * 8 sites
    dict(N=300, L=128, q=21, gap=False, target="Lq=2688 on the 64/128/192 tiles, L%8=0"),
    dict(N=300, L=127, q=21, gap=False, target="one site below 2688, L%8=7"),
    dict(N=300, L=129, q=21, gap=False, target="one site above 2688, L%8=1"),
    # q = 20 (ignored gap): 1920 = 15 * 128 = 10 * 192 = 30 * 64; L = 96 = 12 * 8 sites
    dict(N=300, L=96, q=20, gap=True, target="Lq=1920 on the 64/128/192 tiles, L%8=0"),
    dict(N=300, L=95, q=20, gap=True, target="one site below 1920, L%8=7"),
    dict(N=300, L=97, q=20, gap=True, target="one site above 1920, L%8=1"),
    # nucleotide alphabets (the fused forward falls back to tc): 1920 = 5 * 384, 384 = 4 * 96
    dict(N=300, L=384, q=5, gap=False, target="Lq=1920 on the 64/128/192 tiles, q=5"),
    dict(N=300, L=96, q=4, gap=True, target="Lq=384 on the 64/128/192 tiles, q=4"),
    dict(N=300, L=97, q=4, gap=True, target="one site above 384, q=4"),
    # the fused forward's limit: 390 * 21 = 8190 <= 8192 (fused, one K chain of 128 blocks);
    # 391 * 21 = 8211 > 8192 (falls back; 129 K blocks: the forward's 32-block K chain promotion)
    dict(N=200, L=390, q=21, gap=False, target="Lq=8190: last fused shape, mgroup remainder"),
    dict(N=200, L=391, q=21, gap=False, target="Lq=8211: fused falls back, forward K chain"),
]


@pytest.mark.parametrize("case", SITE_CASES, ids=lambda c: "L%d_q%d" % (c["L"], c["q"]))
def test_site_edges_vs_rounding_model(lib, case):
    run_case(lib, case)


# ------------------------------------------------------------------------------------------------
# 2. sequence counts on and around the K block (64), forward tile (192), softmax tile (256), X rows (384) and
#    chunk (768) edges, and the backward's K chain (2048 = 32 blocks); alphabet sizes at a few of them
# ------------------------------------------------------------------------------------------------
SEQ_COUNTS = [1, 63, 64, 65, 191, 192, 193, 255, 256, 257, 383, 384, 767, 768, 769, 2048, 4096, 4097]


@pytest.mark.parametrize("N", SEQ_COUNTS)
def test_sequence_count_edges_vs_rounding_model(lib, N):
    run_case(lib, dict(N=N, L=24, q=21, gap=False, seed=N, target="N=%d" % N))


@pytest.mark.parametrize("q,gap", [(20, True), (5, False), (4, True)])
@pytest.mark.parametrize("N", [1, 256, 257, 769])
def test_sequence_count_edges_other_alphabets(lib, q, gap, N):
    run_case(lib, dict(N=N, L=25, q=q, gap=gap, seed=N + q, target="N=%d, q=%d" % (N, q)))


# ------------------------------------------------------------------------------------------------
# 3. inputs: a sequence of gaps only, a column of gaps only, zero weights, x = 0, peaked logits
# ------------------------------------------------------------------------------------------------
INPUT_CASES = [
    dict(N=500, L=40, q=21, gap=False, special="gaps", target="gap row + gap column + zero weights"),
    dict(N=500, L=40, q=20, gap=True, special="gaps", target="gap row + gap column + zero weights, ignored gap"),
    dict(N=300, L=30, q=4, gap=True, special="gaps", target="gap row + gap column + zero weights, q=4"),
    dict(N=257, L=24, q=21, gap=False, special="zero_w", target="all weights zero"),
    dict(N=400, L=24, q=21, gap=False, xscale=0.0, target="x = 0: uniform softmax"),
    dict(N=400, L=24, q=21, gap=False, xscale=1.0, target="xscale = 1: peaked softmax"),
    dict(N=400, L=24, q=20, gap=True, xscale=1.0, target="xscale = 1: peaked softmax, ignored gap"),
]


@pytest.mark.parametrize("case", INPUT_CASES, ids=lambda c: c["target"].split(":")[0].replace(" ", "_"))
def test_input_edges_vs_rounding_model(lib, case):
    run_case(lib, case)         # all weights zero: the model is exactly zero, and so the tolerance


# ------------------------------------------------------------------------------------------------
# 4. chunks: N = 2 * 768 + 1 with 768-sequence chunks (the last chunk holds one sequence); forced ksplit = 3 in a
#    subprocess (EVC_KSPLIT is read once per process), where the last chunk's single K block gives ksplit_last = 1
# ------------------------------------------------------------------------------------------------
CHUNK_CASE = dict(N=1537, L=24, q=21, gap=False, seq_chunk=768, seed=5, target="3 chunks of 768, last holds 1")

_SUB = """
import json, sys
import numpy as np
sys.path.insert(0, %r); sys.path.insert(0, %r)
import test_gpu_tc_edges as t
from evcouplings_b200 import _lib
lib = _lib.load()
cases = json.loads(sys.argv[2])
out = {}
for k, c in enumerate(cases):
    codes, w, x = t.make_inputs(c["N"], c["L"], c["q"], c["gap"], c.get("seed", 1), c.get("xscale", 0.1))
    for fwd in c["forwards"]:
        for prec in c["precisions"]:
            r = t.gpu_eval(lib, codes, w, x, c["q"], c["q"] if c["gap"] else -1, fwd, prec, c.get("seq_chunk", 0))
            for f in ("fx", "nll", "g"):
                out["%%d/%%s/%%s/%%s" %% (k, fwd, prec, f)] = r[f]
np.savez(sys.argv[1], **out)
""" % (ROOT, HERE)


def run_subprocess(tmp_path, env_extra, cases):
    path = str(tmp_path / ("sub_%s.npz" % "_".join("%s%s" % kv for kv in sorted(env_extra.items()))))
    env = {k: v for k, v in os.environ.items() if k not in ("EVC_KSPLIT", "EVC_MGROUP", "EVC_KCHUNK")}
    env.update(env_extra)
    p = subprocess.run([sys.executable, "-c", _SUB, path, json.dumps(cases)], capture_output=True, text=True,
                       env=env, timeout=900)
    assert p.returncode == 0, p.stderr[-3000:]
    d = np.load(path)
    res = []
    for k, c in enumerate(cases):
        res.append({"%s/%s" % (fwd, prec): {f: d["%d/%s/%s/%s" % (k, fwd, prec, f)] for f in ("fx", "nll", "g")}
                    for fwd in c["forwards"] for prec in c["precisions"]})
    return res


def test_last_chunk_holds_one_sequence(lib):
    sm = _sm_count(lib)
    geo = geometry(1537, 24, 21, False, 768, sm)
    assert geo["n_chunks"] == 3 and geo["Kp"] == 768
    run_case(lib, CHUNK_CASE)                  # the fused forward falls back under chunks (asserted in run_case)


def test_last_chunk_with_forced_ksplit(lib, tmp_path, monkeypatch):
    sm = _sm_count(lib)
    monkeypatch.setenv("EVC_KSPLIT", "3")
    geo = geometry(1537, 24, 21, False, 768, sm)
    assert (geo["ksplit"], geo["ksplit_last"], geo["planes"]) == (3, 1, 3)
    c = dict(CHUNK_CASE, forwards=["tc"], precisions=["fp32", "bf16"])
    res = run_subprocess(tmp_path, {"EVC_KSPLIT": "3"}, [c])[0]
    run_case(lib, dict(CHUNK_CASE, target="3 chunks, ksplit 3 / last 1"), forwards=("tc",), env_results=res)


def test_backward_k_chain_without_split(lib, tmp_path, monkeypatch):
    """EVC_KSPLIT=1: one slice holds the whole K extent, 32, 64 and 65 blocks of 64 sequences, i.e. one, two and
    two full wgmma chains (+ one block) promoted into the IEEE accumulator"""
    monkeypatch.setenv("EVC_KSPLIT", "1")
    cases = [dict(N=n, L=24, q=21, gap=False, seed=n, forwards=["tc"], precisions=["fp32", "bf16"],
                  target="N=%d, ksplit 1" % n) for n in (2048, 4096, 4097)]
    res = run_subprocess(tmp_path, {"EVC_KSPLIT": "1"}, cases)
    for c, r in zip(cases, res):
        run_case(lib, c, forwards=("tc",), env_results=r)


# ------------------------------------------------------------------------------------------------
# 5. tile order: the forward's M-tile grouping must not change a bit; the backward's K-chunk length stays within
#    the model tolerance
# ------------------------------------------------------------------------------------------------
MGROUP_CASE = dict(N=700, L=75, q=21, gap=False, seed=3, forwards=["tc"], precisions=["fp32", "bf16"],
                   target="L*q=1575: 13 M tiles")


def test_forward_tile_grouping_is_bit_identical(lib, tmp_path):
    geo = geometry(700, 75, 21, False, 0, _sm_count(lib))
    m = geo["m_tiles"]
    assert m == 13                              # not a multiple of 3 or 12: every grouping has a remainder group
    ref = run_subprocess(tmp_path, {}, [MGROUP_CASE])[0]
    for mg in (1, 3, m - 1):
        got = run_subprocess(tmp_path, {"EVC_MGROUP": str(mg)}, [MGROUP_CASE])[0]
        for k in ref:
            for f in ("fx", "nll", "g"):
                assert np.array_equal(got[k][f], ref[k][f]), (mg, k, f)
    run_case(lib, MGROUP_CASE, forwards=("tc",), env_results=ref)


@pytest.mark.parametrize("kchunk", [1, 5, 1000])
def test_backward_k_chunk_length_within_model_tolerance(lib, tmp_path, kchunk):
    """N = 4097: 65 K blocks in ksplit slices; EVC_KCHUNK = 1 promotes every block, 5 leaves a short last chain,
    1000 is longer than the K extent (one chain)"""
    c = dict(N=4097, L=24, q=21, gap=False, seed=4097, forwards=["tc"], precisions=["fp32", "bf16"],
             target="N=4097, EVC_KCHUNK=%d" % kchunk)
    res = run_subprocess(tmp_path, {"EVC_KCHUNK": str(kchunk)}, [c])[0]
    run_case(lib, c, forwards=("tc",), env_results=res)


# ------------------------------------------------------------------------------------------------
# 6. weighted counts (f_i, f_ij of the .model) in both precision modes: the pair counts take the weights as bf16
#    hi + lo in either mode (po.frequencies(weights="hi+lo")); positive sums, so a relative bound per entry
# ------------------------------------------------------------------------------------------------
COUNT_CASES = [(300, 128, 21, False, 0), (769, 96, 20, True, 0), (257, 384, 5, False, 0), (1537, 96, 4, True, 768)]


@pytest.fixture(scope="module")
def engine(lib):
    from evcouplings_b200.engine import CudaEngine
    return CudaEngine()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("N,L,q,gap,chunk", COUNT_CASES)
def test_weighted_counts_vs_rounding_model(engine, precision, N, L, q, gap, chunk):
    eng = engine
    codes, _w, _x = make_inputs(N, L, q, gap, 17)
    w = (1.0 / np.random.default_rng(17).integers(1, 50, N)).astype(np.float32)     # 1/k: more than 16 mantissa bits
    p = eng.plm_problem(codes, w, q, q if gap else -1, 0.0, 0.0, forward="tc", precision=precision, seq_chunk=chunk)
    try:
        fic, fijc = p.weighted_counts()
    finally:
        p.close()
    fi, fij = model_io.normalise_frequencies(fic, fijc, float(w.astype(np.float64).sum()), gap)
    fi_m, fij_m = po.frequencies(codes, w.astype(np.float64), q, q if gap else -1, weights="hi+lo")
    fi_x, fij_x = po.frequencies(codes, w.astype(np.float64), q, q if gap else -1)
    e_i = np.abs(fi - fi_m).max() / np.abs(fi_m).max()
    rel = np.abs(fij - fij_m) / np.maximum(fij_m, 1e-30)
    print("counts N=%d L=%d q=%d %s: f_i max rel %.2e; f_ij max rel %.2e vs the hi+lo model (vs exact weights %.2e)"
          % (N, L, q, precision, e_i, rel[fij_m > 0].max(), (np.abs(fij - fij_x) / np.maximum(fij_x, 1e-30))[fij_x > 0].max()))
    # float32 sums of positive terms, 2^-20 relative per entry (measured at most 3.7e-7 = 2^-21.4, 9.2e-8 for f_i);
    # zero stays exactly zero.  Exact weights would miss by up to 2^-17 (measured 2.4e-6 to 6.6e-6).
    assert e_i <= 2.0 ** -21
    assert (np.abs(fij - fij_m) <= 2.0 ** -20 * fij_m).all()
