"""
The objective's gradient and the weighted pair counts, bit for bit against an exact reference (-m gpu).

On the dyadic case of tests/test_exact_dyadic_model.py every softmax probability is 0 or 1/2^k and every weight and
coupling a short dyadic number, so every residual, product and partial sum on the device is exact in float32, in
both precision modes.  The result then depends on nothing the kernels choose: not the summation order, split-K,
chunks, tile shapes, clusters, M groups or ranks.  Every path must equal the reference exactly, at any N, so a slip
of one sequence, one stale padding row or one K block counted twice fails here at any size, and the failure names the
entry.  (A sequence of weight 0 adds nothing to any sum, so zero weights are kept off the last sequence and off the
sequences next to every 64-sequence edge, which include the tile, X row and chunk edges.)  A relative tolerance (test_gpu_tc_edges.py: whole vector 2e-5) sees such a slip only while its share of the
gradient is above the tolerance.  Measured once by hand on an H100 80GB HBM3 (700 W power limit), with
plm_softmax_kernel changed to drop the last sequence of an even N: this file failed at config 3 (N = 200 000, L = 300,
q = 21; 360 744 entries off, the first g_h(0, 1) by 2 u); on test_gpu_tc_edges.py's own inputs at that size the same
slip moved the gradient by 6.4e-4 relative L2, which its 2e-5 would also have caught.  With the uniform weights of the
dyadic case a one-sequence slip is 3.7 to 3.8 times that tolerance at N = 100 000 (test_exact_dyadic_model.py).

* reference: the backward restated in float64 with torch on the device (G = X^T R, chunked over N, then the two
  conditionals of each pair added), and the counts X^T diag(w) X.  Float64 sums of these values are exact.  It is
  cross-checked against the numpy bincount closed form of test_exact_dyadic_model.py on every site and on at least 64
  pair blocks, among them the first and last sites and the sites on the 64 / 128 / 192 tile edges of L q;
* compared bit for bit: g, and f_i / f_ij before normalisation (evc_plm_weighted_counts);
* fx and -loglk: float64 closed form (log |A_i| is not exact), relative 2e-6;
* a mismatch names its first entry (i, j, a, b), the two backward tiles (M of 128, N of 192) it is summed in and its
  size in units of the resolution u.

What the construction cannot see: a coupling block misplaced between two slots outside the A sets (the logits there
underflow to 0 either way).

The option matrix runs in subprocesses (the EVC_* hooks are read once per process): EVC_KSPLIT 1 / 2 / 3 / 8,
EVC_KCHUNK 1 / 5 / 1000, EVC_FWD_TILE 128, EVC_FWD_CLUSTER 1, EVC_MGROUP 1 / 3.  Each case prints its geometry
(test_gpu_tc_edges.geometry), the budget 2 sum(w) / u and its time.  The budget reached 2^21.6 (config 3) with every
path bit-exact, so the guard bits were enough.  The whole file took 244 s on an H100 80GB HBM3 (700 W power limit);
config 5 (N = 100 000, L = 800, the gather kernels included) 27 s of it, the option matrix 15 to 18 s per process.
"""
import ctypes
import math
import os
import subprocess
import sys
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from evcouplings_b200 import _lib  # noqa: E402
import test_exact_dyadic_model as dm  # noqa: E402
import test_gpu_alphabet_sizes as alph  # noqa: E402
import test_gpu_ranks_one_device as ranks  # noqa: E402
import test_gpu_sparse_forward as sparse  # noqa: E402
import test_gpu_tc_edges as edges  # noqa: E402

GATHER_Q = (4, 5, 20, 21)
FX_REL = 2e-6
vp = ctypes.c_void_p


@pytest.fixture(scope="module")
def engine():
    from evcouplings_b200.engine import CudaEngine
    return CudaEngine()


# ------------------------------------------------------------------------------------------------
# the exact reference
# ------------------------------------------------------------------------------------------------
def couplings_matrix(x, L, q, device):
    """W[(j, b), (i, a)] = J_ij(a, b) in float64 (po.objective's layout): logits = X W + h."""
    import torch
    iu, ju = np.triu_indices(L, 1)
    Jt = torch.from_numpy(x[L * q:]).to(device).double().view(-1, q, q)
    W = torch.zeros((L, q, L, q), dtype=torch.float64, device=device)
    iu_t, ju_t = torch.from_numpy(iu).to(device), torch.from_numpy(ju).to(device)
    W[ju_t, :, iu_t, :] = Jt.transpose(1, 2)
    W[iu_t, :, ju_t, :] = Jt
    return W.view(L * q, L * q)


def reference(case, device="cuda", chunk=None, nll=True):
    """Exact gradient (float64 tensor on ``device``, layout of x), weighted counts f_i (L, q) and f_ij (pairs, q, q),
    and the float64 -loglk of the dyadic case."""
    import torch
    codes, w, A, q = case["codes"], case["w"], case["A"], case["q"]
    N, L = codes.shape
    lq = L * q
    if chunk is None:
        chunk = max(64, min(8192, int(2 ** 28 // (lq * 8))))
    P = torch.from_numpy(dm.probabilities(A)).to(device)
    logA = torch.log(torch.from_numpy(A.sum(axis=1).astype(np.float64)).to(device))
    h = torch.from_numpy(case["x"][:lq]).to(device).double().view(L, q)
    G = torch.zeros((lq, lq), dtype=torch.float64, device=device)
    F = torch.zeros((lq, lq), dtype=torch.float64, device=device)
    W = couplings_matrix(case["x"], L, q, device) if nll else None
    Amask = torch.from_numpy(A).to(device)
    gh = torch.zeros((L, q), dtype=torch.float64, device=device)
    nll_sum = 0.0
    for s0 in range(0, N, chunk):
        c = torch.from_numpy(codes[s0:s0 + chunk].astype(np.int64)).to(device)
        n = c.shape[0]
        X = torch.zeros((n, L, q + 1), dtype=torch.float64, device=device)
        X.scatter_(2, c[:, :, None], 1.0)
        X = X[:, :, :q]                                      # an ignored gap (code q) has no column
        pres = X.sum(dim=2)
        ww = torch.from_numpy(w[s0:s0 + chunk].astype(np.float64)).to(device)
        R = ww[:, None, None] * pres[:, :, None] * (P[None] - X)
        gh += R.sum(dim=0)
        X2 = X.reshape(n, lq)
        G += X2.T @ R.reshape(n, lq)
        F += X2.T @ (ww[:, None] * X2)
        if nll:
            Z = (X2 @ W).view(n, L, q) + h[None]
            assert bool((Z[:, Amask] == 0).all()), "a logit on an A set is not 0"
            zobs = (Z * X).sum(dim=2)
            nll_sum += float((ww[:, None] * pres * (logA[None] - zobs)).sum())
        del X, R, X2
    del W
    iu, ju = (torch.from_numpy(v).to(device) for v in np.triu_indices(L, 1))
    G4 = G.view(L, q, L, q)                                  # [j, b, i, a]
    gJ = G4[ju, :, iu, :].transpose(1, 2) + G4[iu, :, ju, :]
    del G, G4
    F4 = F.view(L, q, L, q)
    fi = torch.einsum("iaia->ia", F4).clone()
    fij = F4[iu, :, ju, :].contiguous()
    del F, F4
    g = torch.cat([gh.reshape(-1), gJ.reshape(-1)])
    return dict(g=g, fi=fi, fij=fij, nll=nll_sum)


def sample_sites(L, q):
    """The first and last sites and the sites on which L q crosses a 64-, 128- or 192-wide tile edge."""
    s = {0, L - 1}
    for t in (64, 128, 192):
        for e in range(t, L * q, t):
            s.add(e // q)
            s.add(max(0, (e - 1) // q))
    return sorted(s)


def sample_pairs(L, q, seed, count=64):
    sites = sample_sites(L, q)
    rng = np.random.default_rng(seed)
    pairs = set()
    if L < 2:
        return []
    for i in sites:                                          # every sampled site meets its neighbours and the ends
        for j in (0, L - 1, i + 1, i - 1):
            if 0 <= j < L and j != i:
                pairs.add((min(i, j), max(i, j)))
    while len(pairs) < min(count, L * (L - 1) // 2):
        i, j = sorted(rng.choice(sites + list(rng.integers(0, L, 4)), 2, replace=False))
        if i != j:
            pairs.add((int(i), int(j)))
    return sorted(pairs)


def cross_check(case, ref, seed=0):
    """The device reference against the numpy bincount closed form: every site, >= 64 sampled pair blocks."""
    codes, w, A, q, L = case["codes"], case["w"], case["A"], case["q"], case["L"]
    g = ref["g"]
    gh = g[:L * q].view(L, q).cpu().numpy()
    fi = ref["fi"].cpu().numpy()
    for i in range(L):
        gb, fb = dm.exact_site_block(codes, w, A, q, i)
        assert np.array_equal(gh[i], gb) and np.array_equal(fi[i], fb), ("reference site", i)
    pairs = sample_pairs(L, q, seed)
    for i, j in pairs:
        p = dm.pair_index(L, i, j)
        gb, Fb = dm.exact_pair_block(codes, w, A, q, i, j)
        off = L * q + p * q * q
        assert np.array_equal(g[off:off + q * q].view(q, q).cpu().numpy(), gb), ("reference pair", i, j)
        assert np.array_equal(ref["fij"][p].cpu().numpy(), Fb), ("reference counts", i, j)
    return len(pairs)


# ------------------------------------------------------------------------------------------------
# comparison
# ------------------------------------------------------------------------------------------------
def locate(k, L, q):
    """Entry k of the parameter vector -> where the backward product sums it."""
    nh = L * q
    if k < nh:
        i, a = divmod(k, q)
        return "g_h(i=%d, a=%d) (softmax tile partial sums)" % (i, a)
    p, ab = divmod(k - nh, q * q)
    a, b = divmod(ab, q)
    iu, ju = np.triu_indices(L, 1)
    i, j = int(iu[p]), int(ju[p])
    r1, c1 = j * q + b, i * q + a                            # Gd[(j, b), (i, a)]: conditional i
    return ("g_J(i=%d, j=%d, a=%d, b=%d): Gd[%d, %d] in backward tile M %d / N %d + Gd[%d, %d] in tile M %d / N %d"
            % (i, j, a, b, r1, c1, r1 // 128, c1 // 192, c1, r1, c1 // 128, r1 // 192))


def assert_bits(label, got, want, case, what="g"):
    """got, want: tensors on the same device.  Bit-exact or a message naming the first mismatch."""
    import torch
    got = got.reshape(-1).double()
    want = want.reshape(-1)
    bad = torch.nonzero(got != want).flatten()
    if bad.numel() == 0:
        return
    k = int(bad[0])
    L, q = case["L"], case["q"]
    d = float(got[k] - want[k])
    if what == "g":
        where = locate(k, L, q)
    elif what == "fi":
        where = "f_i(i=%d, a=%d)" % divmod(k, q)
    else:
        p, ab = divmod(k, q * q)
        iu, ju = np.triu_indices(L, 1)
        where = "f_ij(i=%d, j=%d, a=%d, b=%d)" % ((iu[p], ju[p]) + divmod(ab, q))
    raise AssertionError("%s: %s not bit-exact: %d of %d entries differ; first %s: got %r want %r (%+.6g u)"
                         % (label, what, bad.numel(), got.numel(), where, float(got[k]), float(want[k]),
                            d / case["u"]))


def device_eval(engine, case, forward, backward, precision, seq_chunk=0, counts=True, codes=None, w=None):
    codes = case["codes"] if codes is None else codes
    w = case["w"] if w is None else w
    p = engine.plm_problem(codes, w, case["q"], case["gap_code"], 0.0, 0.0, m=1, forward=forward,
                           backward=backward, precision=precision, seq_chunk=seq_chunk)
    try:
        p.set_x(case["x"])
        p.evaluate(p.x)
        out = dict(g=p.g.clone(), nll=p.last_negloglk)
        if counts:
            fi, fij = p.weighted_counts()
            out["fi"], out["fij"] = fi, fij
    finally:
        p.close()
    return out


def check_result(label, got, ref, case):
    import torch
    dev = ref["g"].device
    assert_bits(label, got["g"].to(dev), ref["g"], case)
    if "fi" in got:
        assert_bits(label, torch.from_numpy(got["fi"]).to(dev), ref["fi"], case, "fi")
        assert_bits(label, torch.from_numpy(np.ascontiguousarray(got["fij"])).to(dev), ref["fij"], case, "fij")
    assert abs(got["nll"] - ref["nll"]) <= FX_REL * abs(ref["nll"]), (label, got["nll"], ref["nll"])


def paths(q, fused, chunked, gather=True):
    """(forward, backward, precision) of every path the library runs for this shape (the fused forward where it does
    not fall back to tc; the gather kernels where q allows them)."""
    out = [("tc", "tc", "fp32"), ("tc", "tc", "bf16")]
    if fused and not chunked:
        out += [("tcfused", "tc", "fp32"), ("tcfused", "tc", "bf16")]
    if gather and q in GATHER_Q and not chunked:
        out += [("gather", "gather", "fp32"), ("gather", "tc", "fp32"), ("gather", "tc", "bf16")]
    return out


def run_case(engine, spec, gather=True, tc_only=False, chunks=(0, 768), counts=True, label=None):
    """Builds the dyadic case of ``spec`` and checks every path / chunk size against the reference."""
    t0 = time.time()
    case = make_case(spec)
    N, L, q, gap = case["N"], case["L"], case["q"], case["gap"]
    sm = engine.sm_count()
    ref = reference(case)
    n_pairs = cross_check(case, ref, seed=N + L)
    t_ref = time.time() - t0
    done = []
    for chunk in chunks:
        if chunk and chunk >= N:
            continue
        geo = edges.geometry(N, L, q, gap, chunk, sm)
        print("\n[%s] N=%d L=%d q=%d%s chunk %d: %s; budget 2 sum(w) / u = %.3g (2^%.1f), reference cross-checked "
              "on %d sites and %d pair blocks"
              % (label or spec.get("target", ""), N, L, q, " (gap ignored)" if gap else "", chunk,
                 edges._fmt_geometry(geo), case["budget"], math.log2(case["budget"]), L, n_pairs))
        todo = paths(q, geo["fused"], chunk > 0, gather) if not tc_only else [("tc", "tc", "fp32"), ("tc", "tc", "bf16")]
        for fwd, bwd, prec in todo:
            t1 = time.time()
            got = device_eval(engine, case, fwd, bwd, prec, chunk, counts=counts)
            check_result("%s fwd %s bwd %s %s chunk %d" % (label or "", fwd, bwd, prec, chunk), got, ref, case)
            done.append("%s/%s/%s" % (fwd, bwd, prec))
            print("  forward %-8s backward %-6s %s: bit-exact (g%s), -loglk rel %.1e  %.2f s"
                  % (fwd, bwd, prec, ", f_i, f_ij" if counts else "",
                     abs(got["nll"] - ref["nll"]) / abs(ref["nll"]), time.time() - t1))
    print("  reference %.1f s, case %.1f s" % (t_ref, time.time() - t0))
    return case, ref


def make_case(spec):
    """spec: N, L, q, gap (+ dyadic_case keywords; by default |A| <= 8 and weights k / 4, k <= 3, 5 % zero, none of
    them on the last sequence or next to a 64-sequence edge)."""
    kw = {k: v for k, v in spec.items() if k not in ("N", "L", "q", "gap", "target")}
    kw.setdefault("seed", spec["N"] + 7 * spec["L"] + spec["q"])
    for k, v in (("amax", 8), ("wk", 3), ("we", 2), ("zero_w", 0.05)):
        kw.setdefault(k, v)
    return dm.dyadic_case(spec["N"], spec["L"], spec["q"], spec["gap"], **kw)


# ------------------------------------------------------------------------------------------------
# 1. the edge tables of the tolerance tests, bit for bit
# ------------------------------------------------------------------------------------------------
EDGE_SPECS = ([dict(N=c["N"], L=c["L"], q=c["q"], gap=c["gap"], target=c["target"]) for c in edges.SITE_CASES]
              + [dict(N=n, L=24, q=21, gap=False, target="N=%d" % n) for n in edges.SEQ_COUNTS]
              + [dict(N=n, L=25, q=q, gap=g, target="N=%d, q=%d" % (n, q)) for q, g in ((20, True), (5, False),
                                                                                        (4, True))
                 for n in (1, 256, 257, 769)]
              + [dict(N=N, L=L, q=q, gap=g, target="alphabet q=%d" % q) for q, g, L, N in alph.OBJECTIVE_CASES]
              + [dict(N=N, L=L, q=q, gap=g, target="2:4 pattern q=%d" % q) for q, g, L, N in sparse.PATTERN_CASES])


@pytest.mark.parametrize("spec", EDGE_SPECS, ids=["%02d-N%d-L%d-q%d%s" % (k, s["N"], s["L"], s["q"], "g" if s["gap"] else "")
                                                  for k, s in enumerate(EDGE_SPECS)])
def test_edge_tables_bit_exact(engine, spec):
    run_case(engine, spec)


# ------------------------------------------------------------------------------------------------
# 2. the shapes no tolerance can police at one-sequence resolution
# ------------------------------------------------------------------------------------------------
LARGE_SPECS = [
    # config 3: |A| <= 8, w = 1: 2 sum(w) / u = 3.2e6 < 2^22
    dict(N=200_000, L=300, q=21, gap=False, amax=8, wk=1, we=0, zero_w=0.0, target="config 3"),
    # config 5
    dict(N=100_000, L=800, q=21, gap=False, amax=8, wk=1, we=0, zero_w=0.0, target="config 5"),
    # 171 chunks of 768 + one chunk of one sequence
    dict(N=171 * 768 + 1, L=64, q=21, gap=False, amax=8, wk=1, we=0, zero_w=0.0,
         target="N = 171 * 768 + 1 > 2^17"),
    # L q = 8192: K is one accumulation chain, 256-row forward tiles
    dict(N=20_001, L=256, q=32, gap=False, amax=16, wk=3, we=2, target="q = 32, L q = 8192"),
]


@pytest.mark.parametrize("spec", LARGE_SPECS, ids=lambda s: s["target"].split(":")[0].replace(" ", "_"))
def test_large_shapes_bit_exact(engine, spec):
    """Every path at each shape: at configs 3 and 5 (q = 21) the gather kernels too, unchunked (they are not
    chunked); the fused forward where L q <= 8192 (config 3)."""
    import torch
    chunks = (0, 768)
    if spec["target"].startswith("N = 171"):
        chunks = (768,)
    run_case(engine, spec, chunks=chunks)
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------
# 3. the option matrix, one process per setting of the hooks
# ------------------------------------------------------------------------------------------------
OPTION_SPECS = [
    dict(N=4097, L=24, q=21, gap=False, target="65 K blocks"),
    dict(N=1537, L=24, q=21, gap=False, target="3 chunks of 768, the last holds 1"),
    dict(N=700, L=75, q=21, gap=False, target="13 M tiles"),
    dict(N=1025, L=256, q=32, gap=False, target="L q = 8192: 256-row forward tiles"),
    dict(N=300, L=391, q=21, gap=False, target="L q = 8211: 129 K blocks"),
    dict(N=2000, L=40, q=20, gap=True, target="ignored gap"),
    dict(N=3000, L=96, q=4, gap=True, target="q = 4, ignored gap"),
]
OPTIONS = [("EVC_KSPLIT", v) for v in ("1", "2", "3", "8")] + [("EVC_KCHUNK", v) for v in ("1", "5", "1000")] + \
          [("EVC_FWD_TILE", "128"), ("EVC_FWD_CLUSTER", "1")] + \
          [("EVC_MGROUP", v) for v in ("1", "3")]
HOOKS = ("EVC_KSPLIT", "EVC_KCHUNK", "EVC_FWD_TILE", "EVC_FWD_CLUSTER", "EVC_MGROUP", "EVC_MGROUP_MB")

_CHILD = r'''
import json, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[2])
import test_gpu_exact_dyadic as t
from evcouplings_b200.engine import CudaEngine
eng = CudaEngine()
for spec in t.OPTION_SPECS:
    t.run_case(eng, spec, tc_only=True, label=sys.argv[3] + " " + spec["target"])
print(json.dumps("ok"))
'''


@pytest.mark.parametrize("name,value", OPTIONS, ids=["%s=%s" % o for o in OPTIONS])
def test_option_matrix_bit_exact(name, value):
    t0 = time.time()
    env = {k: v for k, v in os.environ.items() if k not in HOOKS}
    env[name] = value
    tag = "%s=%s" % (name, value)
    r = subprocess.run([sys.executable, "-c", _CHILD, ROOT, HERE, tag], env=env, capture_output=True, text=True,
                       timeout=900)
    print(r.stdout[-6000:])
    assert r.returncode == 0, r.stderr[-4000:]
    print("%s: %d cases bit-exact on every path, %.1f s" % (tag, len(OPTION_SPECS), time.time() - t0))


# ------------------------------------------------------------------------------------------------
# 4. distinct rows, shards, the regulariser
# ------------------------------------------------------------------------------------------------
def test_distinct_rows_bit_identical_to_full_rows(engine):
    """12 000 rows drawn from 400 distinct ones: the problem on unique_rows with w mult is the full problem."""
    t0 = time.time()
    U, N, L, q = 400, 12_000, 60, 21
    base = dm.dyadic_case(U, L, q, seed=5, amax=4, wk=1, we=1, wmult=80)
    rng = np.random.default_rng(5)
    idx = rng.integers(0, U, N)
    full = dict(base, codes=np.ascontiguousarray(base["codes"][idx]), w=base["w"][idx], N=N)
    full["budget"] = 2 * float(full["w"].astype(np.float64).sum()) / base["u"]
    assert full["budget"] <= dm.BUDGET
    first, inverse, mult = engine.unique_rows(full["codes"])
    assert len(first) <= U and int(mult.max()) <= 80
    wu = (full["w"][first].astype(np.float64) * mult).astype(np.float32)
    assert np.array_equal(wu.astype(np.float64), full["w"][first].astype(np.float64) * mult)
    ref = reference(full)
    cross_check(full, ref)
    print("\n[distinct rows] N=%d -> %d distinct, largest multiplicity %d; budget %.3g"
          % (N, len(first), int(mult.max()), full["budget"]))
    for fwd, bwd, prec in paths(q, True, False):
        a = device_eval(engine, full, fwd, bwd, prec)
        b = device_eval(engine, full, fwd, bwd, prec, codes=np.ascontiguousarray(full["codes"][first]), w=wu)
        check_result("full rows %s/%s/%s" % (fwd, bwd, prec), a, ref, full)
        check_result("distinct rows %s/%s/%s" % (fwd, bwd, prec), b, ref, full)
        print("  forward %-8s backward %-6s %s: full and distinct rows bit-exact" % (fwd, bwd, prec))
    print("  %.1f s" % (time.time() - t0))


SHARD_SPECS = [dict(N=3001, L=40, q=21, gap=False), dict(N=1025, L=40, q=20, gap=True)]


@pytest.mark.parametrize("spec", SHARD_SPECS, ids=["q21", "q20gap"])
def test_shard_sums_bit_exact(engine, spec):
    t0 = time.time()
    lib = engine.lib
    case = make_case(spec)
    ref = reference(case)
    print("\n[shards] N=%d L=%d q=%d budget %.3g" % (case["N"], case["L"], case["q"], case["budget"]))
    for world in (2, 3, 8):
        for prec in ("fp32", "bf16"):
            for order in ranks.ORDERS:
                got = ranks.sharded_eval(lib, case["codes"], case["w"], case["x"], case["q"], case["gap_code"], world,
                                         0.0, 0.0, order, precision=prec)
                import torch
                assert_bits("world %d %s %s" % (world, prec, order), torch.from_numpy(got["g"]).to(ref["g"].device),
                            ref["g"], case)
                assert abs(got["nll"] - ref["nll"]) <= FX_REL * abs(ref["nll"])
            print("  world %d %s: summed shard gradients bit-exact in every order %s" % (world, prec, ranks.ORDERS))
    print("  %.1f s" % (time.time() - t0))


def test_regulariser_at_the_h_j_boundary(engine):
    """lambda_h != lambda_J, both dyadic, on a case where x[L q - 1] = h_{L-1}(q-1) and x[L q] = J_01(0, 0) are both
    nonzero: g = data gradient + 2 lambda x bit for bit, so a lambda_h / lambda_J mix-up at either side of the boundary
    changes an asserted entry; lambda |x|^2 (evc_plm_add_regulariser, and |h|^2, |J|^2 with lambda = (1, 0) / (0, 1))
    and g.g, g.x (evc_vec_dot) as exact integer sums.

    The fused |h|^2, |J|^2, g.g and g.d that reg_dots_kernel hands to evc_plm_fit are not reached here: the ABI entry
    point passes no output for them.  tests/test_gpu_lbfgs_replay.py checks them at every accepted iterate of real
    fits, as the reported norms and through the strong Wolfe conditions, within the bound of the reduction tree."""
    import torch
    lib = engine.lib
    lam_h, lam_J = 0.125, 0.09375
    N, L, q = 3001, 40, 21
    nh = L * q
    case = dm.dyadic_case(N, L, q, seed=9, amax=8, wk=3, we=2, lam=(lam_h, lam_J),
                          outside=((0, 0), (1, 0), (L - 1, q - 1)))
    if case["x"][nh] == 0:
        case["x"][nh] = 37.0 / 64                      # J_01(0, 0): both states outside their A sets
    x64 = case["x"].astype(np.float64)
    assert x64[nh - 1] == dm.H_OUT and x64[nh] != 0
    ref = reference(case)
    lam = np.where(np.arange(x64.size) < nh, lam_h, lam_J)
    want = ref["g"].cpu().numpy() + 2 * lam * x64
    # the boundary one element off in either direction changes an entry the comparison sees
    for off in (-1, 1):
        lam_off = np.where(np.arange(x64.size) < nh + off, lam_h, lam_J)
        assert (ref["g"].cpu().numpy() + 2 * lam_off * x64 != want).any(), off
    codes, w, x = case["codes"], case["w"], case["x"]
    h = vp()
    _lib.check(lib.evc_plm_create_alphabet(ctypes.byref(h), codes.ctypes.data_as(vp), N, L, q, -1,
                                           w.ctypes.data_as(vp), 0), "evc_plm_create_alphabet")
    try:
        _lib.check(lib.evc_plm_set_forward(h, 1), "evc_plm_set_forward")
        g = np.zeros_like(x)
        fx = np.zeros(2)
        _lib.check(lib.evc_plm_eval_host(h, x.ctypes.data_as(vp), g.ctypes.data_as(vp), fx.ctypes.data_as(vp),
                                         lam_h, lam_J), "evc_plm_eval_host")
        assert_bits("regularised", torch.from_numpy(g), torch.from_numpy(want), case)
        # the scalars: x / 2^-6 and g / u are integers; float64 sums of their products are exact below 2^53
        xi = [int(v) for v in np.round(x64 * 64).astype(np.int64)]
        gi = [int(v) for v in np.round(g.astype(np.float64) / case["u"]).astype(np.int64)]
        assert np.array_equal(np.array(gi, dtype=np.float64) * case["u"], g.astype(np.float64))
        hh = sum(v * v for v in xi[:nh])                      # |h|^2 * 2^12
        jj = sum(v * v for v in xi[nh:])                      # |J|^2 * 2^12
        gg = sum(v * v for v in gi)                           # g.g / u^2
        gx = sum(a * b for a, b in zip(gi, xi))               # g.x / (u 2^-6)
        assert max(hh, jj, gg, abs(gx)) < 2 ** 53
        assert xi[nh] ** 2 > 0                               # |h|^2 and |J|^2 change if x[L q] changes sides
        d_x = torch.from_numpy(x).cuda()
        d_g = torch.from_numpy(g).cuda()
        scal = {}
        for name, lh, lj in (("|h|^2", 1.0, 0.0), ("|J|^2", 0.0, 1.0), ("lambda |x|^2", lam_h, lam_J)):
            zero = torch.zeros_like(d_x)
            d_fx = torch.zeros(2, dtype=torch.float64, device="cuda")
            _lib.check(lib.evc_plm_add_regulariser(h, vp(d_x.data_ptr()), vp(zero.data_ptr()), vp(d_fx.data_ptr()),
                                                   lh, lj, None), "evc_plm_add_regulariser")
            scal[name] = float(d_fx[1].item())
        for name, a, b in (("g.g", d_g, d_g), ("g.x", d_g, d_x)):
            out = torch.zeros(1, dtype=torch.float64, device="cuda")
            _lib.check(lib.evc_vec_dot(vp(a.data_ptr()), vp(b.data_ptr()), a.numel(), vp(out.data_ptr()), None),
                       "evc_vec_dot")
            scal[name] = float(out.item())
    finally:
        lib.evc_plm_destroy(h)
    want_s = {"|h|^2": hh / 4096.0, "|J|^2": jj / 4096.0, "lambda |x|^2": lam_h * hh / 4096.0 + lam_J * jj / 4096.0,
              "g.g": gg * case["u"] ** 2, "g.x": gx * case["u"] / 64}
    for k, v in want_s.items():
        assert scal[k] == v, (k, scal[k], v)
    assert abs(fx[1] - (ref["nll"] + want_s["lambda |x|^2"])) <= FX_REL * abs(fx[1])
    print("\n[regulariser] lambda_h %g lambda_J %g: g bit-exact (x[L q - 1] = %r -> g %r, x[L q] = %r -> g %r); "
          "lambda |x|^2, |h|^2, |J|^2 (evc_plm_add_regulariser), g.g, g.x (evc_vec_dot) exact"
          % (lam_h, lam_J, float(x64[nh - 1]), float(g[nh - 1]), float(x64[nh]), float(g[nh])))
