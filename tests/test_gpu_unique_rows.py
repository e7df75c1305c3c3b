"""
Distinct rows on the H100 (-m gpu): evc_msa_unique against np.unique (exact, repeatable, stream-independent, and exact
under forced hash collisions), the multiplicity-weighted Hamming counts against plmc's own PABP counts and the
full-row pass under every pruning hook, the objective / gradient / pair counts of the distinct problem against the
full-row problem and the float64 oracle, and run_plmc end to end.
"""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from evcouplings_b200 import _lib, model_io, msa, synthetic, tools  # noqa: E402
from test_unique_rows import model_head, unique_rows_model  # noqa: E402

import golden_npz  # noqa: E402

vp = ctypes.c_void_p


@pytest.fixture(scope="module")
def lib():
    l = _lib.load()
    _lib.require_device()
    return l


@pytest.fixture(scope="module")
def engine(lib):
    from evcouplings_b200.engine import CudaEngine
    return CudaEngine()


@pytest.fixture(scope="module")
def pabp():
    c = golden_npz.load("pabp_codes")
    valid = np.unpackbits(c["valid_packed"])[: int(c["n_total"])].astype(bool)
    return dict(codes=np.ascontiguousarray(c["codes"]), counts=c["golden_counts_all"][valid])


def host_unique(lib, codes):
    codes = np.ascontiguousarray(codes, dtype=np.uint8)
    N, L = codes.shape
    first, inverse, mult = (np.zeros(N, dtype=np.int32) for _ in range(3))
    U = ctypes.c_int64()
    _lib.check(lib.evc_msa_unique_host(codes.ctypes.data_as(vp), N, L, 0, first.ctypes.data_as(vp),
                                       inverse.ctypes.data_as(vp), mult.ctypes.data_as(vp), ctypes.byref(U)),
               "evc_msa_unique_host")
    U = U.value
    return first[:U].astype(np.int64), inverse.astype(np.int64), mult[:U].astype(np.int64)


def hamming(lib, codes, thr, mult=None):
    codes = np.ascontiguousarray(codes, dtype=np.uint8)
    N, L = codes.shape
    out = np.zeros(N, dtype=np.int32)
    if mult is None:
        _lib.check(lib.evc_hamming_counts(codes.ctypes.data_as(vp), N, L, thr, 0, out.ctypes.data_as(vp)), "hamming")
    else:
        m = np.ascontiguousarray(mult, dtype=np.int32)
        _lib.check(lib.evc_hamming_counts_mult(codes.ctypes.data_as(vp), m.ctypes.data_as(vp), N, L, thr, 0,
                                               out.ctypes.data_as(vp)), "hamming_mult")
    return out


def _case(name):
    rng = np.random.default_rng(sum(map(ord, name)))
    if name == "all_equal":
        return np.tile(rng.integers(0, 21, 40).astype(np.uint8), (3000, 1))
    if name == "one_row":
        return rng.integers(0, 21, (1, 50)).astype(np.uint8)
    N, L, hi, rep = {"random": (5000, 82, 21, False), "repeats": (5000, 82, 21, True), "L1": (4000, 1, 32, False),
                     "L31": (3000, 31, 32, True), "L33": (3000, 33, 2, True), "L300": (2000, 300, 32, True)}[name]
    codes = rng.integers(0, hi, (N, L)).astype(np.uint8)
    if rep:
        codes[rng.integers(0, N, N // 2)] = codes[rng.integers(0, N, N // 2)]
    return codes


@pytest.mark.parametrize("name", ["random", "repeats", "all_equal", "one_row", "L1", "L31", "L33", "L300"])
def test_unique_matches_np_unique(lib, name):
    codes = _case(name)
    got = host_unique(lib, codes)
    ref = unique_rows_model(codes)
    for a, b in zip(got, ref):
        assert np.array_equal(a, b)
    if name == "random":
        assert np.array_equal(got[0], np.arange(len(codes)))         # no repeats: the identity
    again = host_unique(lib, codes)
    assert all(np.array_equal(a, b) for a, b in zip(got, again))


def test_unique_does_not_depend_on_the_stream(lib, engine):
    import torch
    codes = _case("repeats")
    ref = host_unique(lib, codes)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = engine.unique_rows(codes)
    torch.cuda.synchronize()
    assert all(np.array_equal(a, b) for a, b in zip(got, ref))


@pytest.mark.parametrize("bits", [1, 3, 8])
def test_hash_collisions_never_merge_distinct_rows(lib, monkeypatch, bits):
    """with the hash cut to a few bits nearly every row collides; rows that differ in one code must stay apart"""
    rng = np.random.default_rng(bits)
    base = rng.integers(0, 21, (1500, 60)).astype(np.uint8)
    near = base.copy()
    near[np.arange(1500), rng.integers(0, 60, 1500)] ^= 1            # one code changed per row
    codes = np.concatenate([base, near, base[::3]])
    ref = unique_rows_model(codes)
    monkeypatch.setenv("EVC_UNIQUE_HASH_BITS", str(bits))
    got = host_unique(lib, codes)
    assert all(np.array_equal(a, b) for a, b in zip(got, ref))


def test_pabp_distinct_rows(lib, pabp):
    got = host_unique(lib, pabp["codes"])
    assert len(got[0]) == 70300 and got[2].max() == 983
    ref = unique_rows_model(pabp["codes"])
    assert all(np.array_equal(a, b) for a, b in zip(got, ref))


def test_pabp_multiplicity_counts(lib, engine, pabp):
    """counts over the distinct rows, spread back to the rows, are plmc's own counts; two tile ranges summed too"""
    import torch
    codes = pabp["codes"]
    thr = msa.identity_threshold_count(0.8, 82)
    first, inverse, mult = host_unique(lib, codes)
    cu = codes[first]
    counts_u = hamming(lib, cu, thr, mult)
    assert np.array_equal(counts_u[inverse], pabp["counts"])
    assert np.array_equal(counts_u[inverse], hamming(lib, codes, thr))
    U = len(first)
    d_codes = torch.from_numpy(cu).cuda()
    d_mult = torch.from_numpy(mult.astype(np.int32)).cuda()
    d_planes = torch.empty(lib.evc_hamming_plane_words(U, 82), dtype=torch.int32, device="cuda")
    d_counts = torch.zeros(U, dtype=torch.int32, device="cuda")
    p = lambda t: vp(t.data_ptr())  # noqa: E731
    _lib.check(lib.evc_hamming_pack(p(d_codes), U, 82, p(d_planes), None), "pack")
    T = lib.evc_hamming_num_tiles(U)
    for lo, hi in ((0, T // 3), (T // 3, T)):
        _lib.check(lib.evc_hamming_count_tiles_mult(p(d_planes), p(d_mult), U, 82, thr, lo, hi, p(d_counts), None),
                   "count_tiles_mult")
    assert np.array_equal(d_counts.cpu().numpy(), counts_u)


def test_multiplicity_counts_under_the_pruning_hooks():
    """PABP (single-phase pass, early termination on / off) and a long synthetic alignment with repeats (filter +
    verify, a 100-entry candidate buffer that overflows, single phase): distinct counts == full-row counts.  The
    hooks are read once per process, so each setting runs in its own."""
    code = (
        "import sys, ctypes, numpy as np; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "from evcouplings_b200 import _lib, msa, synthetic\nimport golden_npz\n"
        "from test_gpu_unique_rows import host_unique, hamming\n"
        "lib = _lib.load()\n"
        "pabp = golden_npz.load('pabp_codes')['codes']\n"
        "syn = synthetic.synthetic_msa_codes(3000, 300, 6); rng = np.random.default_rng(1)\n"
        "syn[rng.integers(0, 3000, 1200)] = syn[rng.integers(0, 3000, 1200)]\n"
        "for codes in (pabp, syn):\n"
        "    thr = msa.identity_threshold_count(0.8, codes.shape[1])\n"
        "    first, inverse, mult = host_unique(lib, codes)\n"
        "    assert len(first) < len(codes)\n"
        "    assert np.array_equal(hamming(lib, codes[first], thr, mult)[inverse], hamming(lib, codes, thr))\n"
        "print('exact')\n" % (ROOT, os.path.join(ROOT, "tests")))
    for hook in (None, ("EVC_HAMMING_NO_PRUNE", "1"), ("EVC_HAMMING_CAND_CAP", "100"),
                 ("EVC_HAMMING_SINGLE_PHASE", "1")):
        env = dict(os.environ, PYTHONPATH=os.path.join(ROOT, "tests", "golden"))
        if hook:
            env[hook[0]] = hook[1]
        p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=600)
        assert p.returncode == 0 and "exact" in p.stdout, (hook, p.stderr[-2000:])


def test_objective_and_pair_counts_on_distinct_rows(engine, pabp):
    """A PABP subsample at plmc's optimum: the distinct problem with merged weights against the full rows, on the
    device and in the float64 oracle."""
    from oracle import plm_oracle as po
    g = golden_npz.load("pabp_golden")
    rng = np.random.default_rng(0)
    rows = np.sort(rng.choice(len(pabp["codes"]), 6000, replace=False))
    codes = pabp["codes"][rows]
    counts = pabp["counts"][rows]                # any positive counts do: the weights only need to be shared
    first, inverse, mult = unique_rows_model(codes)
    assert len(first) < 0.9 * len(codes)
    w = 1.0 / counts.astype(np.float64)
    w_u = (mult / counts[first].astype(np.float64)).astype(np.float32)
    x = np.concatenate([g["h"].ravel(), g["J"].ravel()]).astype(np.float32)
    L, q = 82, 20
    out = {}
    for tag, c, ww in (("full", codes, w.astype(np.float32)), ("dist", codes[first], w_u)):
        prob = engine.plm_problem(c, ww, q, q, 0.0, 0.0)
        prob.set_x(x)
        prob.evaluate(prob.x)
        fic, fijc = prob.weighted_counts()
        out[tag] = (prob.last_negloglk, prob.g.cpu().numpy().astype(np.float64), fic, fijc)
        prob.close()
    fx_o, g_o, nll_o, sc = po.objective(x.astype(np.float64), codes, w.astype(np.float32).astype(np.float64), q,
                                        0.0, 0.0, gap_code=q, operands="hi+lo", bounds=0.0)
    nll_f, g_f, fi_f, fij_f = out["full"]
    nll_d, g_d, fi_d, fij_d = out["dist"]
    assert abs(nll_d - nll_f) <= 1e-6 * abs(nll_f) and abs(nll_d - nll_o) <= 1e-6 * abs(nll_o)
    for ref in (g_f, g_o):
        assert np.linalg.norm(g_d - ref) <= 5e-6 * np.linalg.norm(ref)
    # g_h and f_i per site, against the site's sum of |terms|
    gh_scale = sc["g_abs"][:L * q].reshape(L, q).sum(axis=1)
    gh_err = np.abs(g_d[:L * q] - g_f[:L * q]).reshape(L, q).max(axis=1)
    assert np.all(gh_err <= 2.0 ** -20 * gh_scale), (gh_err / gh_scale).max()
    fi_scale = fi_f.sum(axis=1)
    assert np.all(np.abs(fi_d - fi_f).max(axis=1) <= 2.0 ** -20 * fi_scale)
    n_eff = float(w.sum())
    fi1, fij1 = model_io.normalise_frequencies(fi_d, fij_d, n_eff, True)
    fi2, fij2 = model_io.normalise_frequencies(fi_f, fij_f, n_eff, True)
    fi_o, fij_o = po.frequencies(codes, w.astype(np.float32).astype(np.float64), q, q)
    for ref_i, ref_ij in ((fi2, fij2), (fi_o, fij_o)):
        assert np.abs(fi1 - ref_i).max() < 2e-6 and np.abs(fij1 - ref_ij).max() < 2e-6


class FullRowsEngine(object):
    """CudaEngine that reports every row as distinct: run_plmc then takes the full-row path."""

    def __new__(cls):
        from evcouplings_b200.engine import CudaEngine

        class _E(CudaEngine):
            def unique_rows(self, codes):
                n = len(codes)
                return np.arange(n), np.arange(n), np.ones(n, dtype=np.int64)
        return _E()


def _kw(a2m, tmp_path, tag, L, **extra):
    kw = dict(alignment=a2m, couplings_file=str(tmp_path / (tag + "_ECs.txt")),
              param_file=str(tmp_path / (tag + ".model")), focus_seq="seq0/1-%d" % L, theta=0.8, ignore_gaps=True,
              iterations="max", lambda_h=0.01, lambda_J=2.0, epsilon=1e-6)
    kw.update(extra)
    return kw


@pytest.mark.parametrize("source", ["synthetic", "pabp"])
def test_run_plmc_with_repeats(engine, tmp_path, source, pabp):
    from cpu_engine import OracleEngine
    if source == "synthetic":
        codes = synthetic.synthetic_msa_codes(600, 20, 4)
        rng = np.random.default_rng(4)
        codes[rng.integers(1, 600, 250)] = codes[rng.integers(0, 600, 250)]
    else:
        rows = np.sort(np.random.default_rng(1).choice(len(pabp["codes"]), 1500, replace=False))
        codes = np.where(pabp["codes"][rows, :24] == 20, 0, pabp["codes"][rows, :24] + 1).astype(np.uint8)
        codes = np.concatenate([np.arange(1, 25, dtype=np.uint8)[None] % 20 + 1, codes])   # a gap-free focus
    L = codes.shape[1]
    a2m = str(tmp_path / "in.a2m")
    synthetic.write_a2m(a2m, codes)
    lam = dict(lambda_J=2.0 if source == "synthetic" else 30.0)     # the PABP columns: a better-conditioned optimum
    rd, run_d = tools.run_plmc(engine=engine, return_run=True, **_kw(a2m, tmp_path, "d", L, **lam))
    rf, run_f = tools.run_plmc(engine=FullRowsEngine(), return_run=True, **_kw(a2m, tmp_path, "f", L, **lam))
    ro, run_o = tools.run_plmc(engine=OracleEngine(), return_run=True,
                               **_kw(a2m, tmp_path, "o", L, epsilon=1e-8, **lam))
    assert run_d.timings["unique_rows"] < run_f.timings["unique_rows"] == run_d.alignment.n_valid
    assert np.array_equal(run_d.counts, run_f.counts) and np.array_equal(run_d.weights, run_f.weights)
    assert run_d.n_eff == run_f.n_eff and model_head(rd.param_file) == model_head(rf.param_file)
    cn_d, cn_f, cn_o = (np.loadtxt(r.couplings_file, usecols=5) for r in (rd, rf, ro))
    rms = lambda a: float(np.sqrt(np.mean((a - cn_o) ** 2)))  # noqa: E731
    assert rms(cn_d) < 1e-4, (rms(cn_d), rms(cn_f), rd.optimization_status, rf.optimization_status)


def test_run_plmc_without_repeats_is_byte_identical(engine, tmp_path):
    codes = synthetic.synthetic_msa_codes(500, 30, 8)
    assert len(unique_rows_model(codes)[0]) == 500
    a2m = str(tmp_path / "in.a2m")
    synthetic.write_a2m(a2m, codes)
    rd, run_d = tools.run_plmc(engine=engine, return_run=True, **_kw(a2m, tmp_path, "d", 30, iterations=30))
    rf = tools.run_plmc(engine=FullRowsEngine(), **_kw(a2m, tmp_path, "f", 30, iterations=30))
    assert run_d.timings["unique_rows"] == 500
    for suffix in ("_ECs.txt", ".model"):
        assert open(str(tmp_path / ("d" + suffix)), "rb").read() == open(str(tmp_path / ("f" + suffix)), "rb").read()
