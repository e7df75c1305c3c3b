"""
The data-parallel device path on ONE GPU (-m gpu; exactly one device is needed).

The arithmetic of a rank is a handle over a slice of the sequences, so R "ranks" are R handles on one device in one
process, and the test plays the collective with a float32 sum whose order it controls.  Four parts:

1. the -loglk limb transport (evc_plm_pack_fx / evc_plm_unpack_fx) against the Python-integer model of
   tests/test_fx_limb_model.py, bit for bit, for every order of the float32 sum, and NaN for what it cannot carry;
2. shard sums: evc_plm_eval_data per shard + limbs + evc_plm_add_regulariser against the float64 oracle of the whole
   alignment and against one handle over the whole alignment, at the shard / tile / chunk edges; and evc_plm_fit with
   an all-reduce callback (the regulariser's limb branch);
3. Hamming tile ranges (evc_hamming_count_tiles, _mult) summed over ranks against the exact CPU counts;
4. two real rank processes sharing device 0 over gloo, through the product's own launcher and worker: lock-step fits,
   the iteration table against one rank, checkpoints saved and resumed by two ranks.

Shards against one handle over the whole alignment differ by the summation order only.  Measured over the cases of
part 2 on an H100 80GB HBM3 (700 W power limit): g_h at most 1.4e-7 and g_J at most 3.5e-7 relative L2 (the bf16-tiles
mode included: its operands are rounded per sequence, before any sum), -loglk at most 1.0e-5 absolute on 64 ranks,
where the bound of one rounding to 2^-16 per rank is 4.9e-4; against float64 the gradient is within 2.7e-6 and fx
within 3.2e-7 in the fp32-equivalent mode.  The asserted bounds are about four times the measured values.

What this cannot check is NCCL itself, device placement by LOCAL_RANK and scaling: tests/test_gpu_multi.py, on two GPUs.
"""
import ctypes
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from evcouplings_b200 import _lib, msa, synthetic  # noqa: E402
from evcouplings_b200.dist import shard_bounds  # noqa: E402
from oracle import c_oracle as co  # noqa: E402
import test_fx_limb_model as fxm  # noqa: E402

vp = ctypes.c_void_p
RANK_TIMEOUT_S = 600


@pytest.fixture(scope="module")
def lib():
    l = _lib.load()
    _lib.require_device()
    return l


def p(t):
    return vp(t.data_ptr())


def float32_sum(bufs, order, seed=0):
    """The all-reduce the test plays: float32 sum of the ranks' device buffers as a running sum in rank order,
    reversed or permuted, or as a pairwise tree."""
    if order == "tree":
        return fxm.sum_tree([b.clone() for b in bufs], lambda a, b: a + b)
    acc = None
    for r in fxm.sum_orders(len(bufs), seed)[order]:
        acc = bufs[r].clone() if acc is None else acc + bufs[r]
    return acc


ORDERS = ("rank", "reversed", "tree", "permuted")


# ----------------------------------------------------------------------------------------------------------------------
# 1. the limb transport
# ----------------------------------------------------------------------------------------------------------------------
def pack(lib, values):
    """evc_plm_pack_fx of each value into its own 4 floats; returns the list of device buffers"""
    import torch
    d_fx = torch.tensor([float(v) for v in values], dtype=torch.float64, device="cuda")
    bufs = [torch.full((4,), 7.0, dtype=torch.float32, device="cuda") for _ in values]
    for r, b in enumerate(bufs):
        _lib.check(lib.evc_plm_pack_fx(p(d_fx[r:r + 1]), p(b), None), "evc_plm_pack_fx")
    return bufs


def unpack(lib, limbs):
    import torch
    out = torch.full((1,), -7.0, dtype=torch.float64, device="cuda")
    _lib.check(lib.evc_plm_unpack_fx(p(limbs), p(out), None), "evc_plm_unpack_fx")
    return float(out.item())


def test_single_values_pack_to_documented_limbs_and_decode_exactly(lib):
    values = fxm.edge_values() + fxm.seeded_values(50, 7)
    for v, b in zip(values, pack(lib, values)):
        limbs = b.cpu().numpy().astype(np.float64)
        l0, l1, l2, l3 = limbs
        assert all(x == int(x) for x in limbs), (v, limbs)
        assert 0 <= l0 < 2 ** 18 and 0 <= l1 < 2 ** 18 and abs(l2) < 2 ** 17 and l3 == 0, (v, limbs)
        assert (int(l0), int(l1), int(l2)) == fxm.split(fxm.Q(v)), (v, limbs)
        assert unpack(lib, b) == fxm.Q(v) / 65536, v


@pytest.mark.parametrize("R", [2, 3, 8, 64])
def test_limb_sums_over_ranks_are_exact_in_every_order(lib, R):
    import torch
    top = ((130966 << 36) | ((1 << 36) - 1)) / 65536          # the largest carried value with both low limbs at 2^18 - 1
    seeded = fxm.seeded_values(R, 100 + R)
    half = fxm.seeded_values(R // 2, 200 + R)
    cancel = half + [-v for v in half] + [0.0] * (R % 2)
    sets = {"seeded": seeded, "largest": [top] * R, "most negative": [-top] * R, "cancel": cancel,
            "half ulp ties": [2.0 ** -17 * (2 * r + 1) for r in range(R)]}
    for name, values in sets.items():
        want = fxm.transported(values)
        if name == "cancel":
            assert want == 0.0
        bufs = pack(lib, values)
        for order in ORDERS:
            assert unpack(lib, float32_sum(bufs, order, seed=R)) == want, (name, order)
    # limbs beyond what pack emits: every rank's low limbs at 2^18 - 1 and its top limb at +-(2^17 - 1); the sums
    # reach 2^24 - R and stay exact
    for sign in (1, -1):
        limbs = (fxm.MASK, fxm.MASK, sign * (2 ** 17 - 1))
        bufs = [torch.tensor(limbs + (0,), dtype=torch.float32, device="cuda") for _ in range(R)]
        for order in ORDERS:
            tot = float32_sum(bufs, order, seed=R)
            assert [int(v) for v in tot.tolist()] == [R * l for l in limbs] + [0]
            assert unpack(lib, tot) == fxm.decode([R * l for l in limbs])


def test_values_that_cannot_be_carried_decode_to_nan_on_every_rank(lib):
    """A rank's NaN, infinite or out-of-range -loglk must not arrive as a large finite number: a single rank reads
    its NaN directly, and a line search that sees a huge finite decrease on several ranks would accept the step."""
    bad = [float("nan"), float("inf"), float("-inf"), 2e11, -2e11]
    for v, b in zip(bad, pack(lib, bad)):
        assert np.isnan(b.cpu().numpy()[3]), v
        assert np.isnan(unpack(lib, b)), v
    good = fxm.seeded_values(7, 9)
    for v in bad:
        for where in (0, 3, 7):
            bufs = pack(lib, good[:where] + [v] + good[where:])
            for order in ORDERS:
                assert np.isnan(unpack(lib, float32_sum(bufs, order, seed=where))), (v, where, order)
    assert unpack(lib, float32_sum(pack(lib, good + [1.0]), "rank")) == fxm.transported(good + [1.0])


# ----------------------------------------------------------------------------------------------------------------------
# 2. shards sum to the whole
# ----------------------------------------------------------------------------------------------------------------------
def num_params(L, q):
    return L * q + L * (L - 1) // 2 * q * q


def make_case(N, L, q, gap, seed=1, xscale=0.1):
    """codes in the convention of (q, gap) (gap: the ignored gap code q), weights in [0.05, 1], normal x"""
    rng = np.random.default_rng(seed)
    if q in (20, 21):
        codes = synthetic.synthetic_msa_codes(N, L, seed)
        if gap:
            codes = synthetic.to_ignore_gaps_codes(codes, q)
    else:
        codes = rng.integers(0, q + (1 if gap else 0), size=(N, L)).astype(np.uint8)
    w = rng.uniform(0.05, 1.0, N).astype(np.float32)
    x = (rng.normal(0, xscale, num_params(L, q)) if xscale else np.zeros(num_params(L, q))).astype(np.float32)
    return np.ascontiguousarray(codes), w, x


def create_handle(lib, codes, w, q, gap_code, precision=None, seq_chunk=0):
    """what CudaPlmProblem does for its shard"""
    codes = np.ascontiguousarray(codes)
    w = np.ascontiguousarray(w)
    h = vp()
    _lib.check(lib.evc_plm_create_alphabet(ctypes.byref(h), codes.ctypes.data_as(vp), codes.shape[0], codes.shape[1],
                                           q, gap_code, w.ctypes.data_as(vp), 0), "evc_plm_create_alphabet")
    try:
        if seq_chunk:
            _lib.check(lib.evc_plm_set_seq_chunk(h, seq_chunk), "evc_plm_set_seq_chunk")
        _lib.check(lib.evc_plm_set_forward(h, 1), "evc_plm_set_forward")
        if precision == "bf16":
            _lib.check(lib.evc_plm_set_precision(h, 1), "evc_plm_set_precision")
    except Exception:
        lib.evc_plm_destroy(h)
        raise
    return h


def sharded_eval(lib, codes, w, x, q, gap_code, world, lam_h, lam_J, order, **handle_opts):
    """CudaPlmProblem.evaluate_async of every rank of a ``world``-rank run, in one process on one device: per rank
    shard_bounds -> handle on the slice -> evc_plm_eval_data into n + 4 floats -> evc_plm_pack_fx into the last 4;
    then the collective as a float32 sum in ``order``; then evc_plm_unpack_fx and evc_plm_add_regulariser.
    Returns -loglk, fx, g, the ranks' own -loglk (read before packing) and the ranks' limbs."""
    import torch
    N, L = codes.shape
    n = num_params(L, q)
    d_x = torch.from_numpy(x).cuda()
    bufs, nll_r = [], []
    h = None
    try:
        for r in range(world):
            lo, hi = shard_bounds(N, world, r)
            assert hi > lo
            if h is not None:
                lib.evc_plm_destroy(h)
                h = None
            h = create_handle(lib, codes[lo:hi], w[lo:hi], q, gap_code, **handle_opts)
            assert lib.evc_plm_num_params(h) == n
            buf = torch.zeros(n + 4, dtype=torch.float32, device="cuda")
            d_fx = torch.zeros(2, dtype=torch.float64, device="cuda")
            _lib.check(lib.evc_plm_eval_data(h, p(d_x), p(buf), p(d_fx), None), "evc_plm_eval_data")
            _lib.check(lib.evc_plm_pack_fx(p(d_fx), p(buf[n:]), None), "evc_plm_pack_fx")
            nll_r.append(float(d_fx[0].item()))
            bufs.append(buf)
        total = float32_sum(bufs, order)
        fx = torch.zeros(2, dtype=torch.float64, device="cuda")
        _lib.check(lib.evc_plm_unpack_fx(p(total[n:]), p(fx), None), "evc_plm_unpack_fx")
        _lib.check(lib.evc_plm_add_regulariser(h, p(d_x), p(total), p(fx), lam_h, lam_J, None),
                   "evc_plm_add_regulariser")
        nll, f = fx.tolist()
    finally:
        if h is not None:
            lib.evc_plm_destroy(h)
    limbs = [b[n:].cpu().numpy() for b in bufs]
    return dict(nll=nll, fx=f, g=total[:n].cpu().numpy().astype(np.float64), nll_r=nll_r, limbs=limbs)


def whole_eval(lib, codes, w, x, q, gap_code, lam_h, lam_J, **handle_opts):
    import torch
    n = x.size
    h = create_handle(lib, codes, w, q, gap_code, **handle_opts)
    try:
        d_x = torch.from_numpy(x).cuda()
        g = torch.zeros(n, dtype=torch.float32, device="cuda")
        fx = torch.zeros(2, dtype=torch.float64, device="cuda")
        _lib.check(lib.evc_plm_eval_data(h, p(d_x), p(g), p(fx), None), "evc_plm_eval_data")
        _lib.check(lib.evc_plm_add_regulariser(h, p(d_x), p(g), p(fx), lam_h, lam_J, None), "evc_plm_add_regulariser")
        nll, f = fx.tolist()
    finally:
        lib.evc_plm_destroy(h)
    return dict(nll=nll, fx=f, g=g.cpu().numpy().astype(np.float64))


def rel_l2(a, b):
    nb = np.linalg.norm(b)
    return float(np.linalg.norm(a - b) / nb) if nb > 0 else float(np.linalg.norm(a - b))


# (N, L, q, gap, world, options, edge)
SHARD_CASES = [
    (2, 2, 21, False, 2, {}, "one sequence per rank, smallest problem"),
    (3, 5, 21, False, 3, {}, "one sequence per rank"),
    (8, 7, 2, False, 8, {}, "one sequence per rank, q = 2"),
    (9, 7, 32, False, 8, {}, "shard sizes 2,1,1,...: the remainder branch of shard_bounds, q = 32"),
    (513, 33, 21, False, 2, {}, "shards 257 / 256: one past and exactly on the 256-sequence partial tile"),
    (1025, 40, 20, True, 2, {}, "256-row forward pairs, odd tile count per shard, ignored gap"),
    (1025, 40, 20, True, 3, {}, "256-row forward pairs, three shards, ignored gap"),
    (3001, 40, 21, False, 2, {}, "the shape of test_gpu_multi.py"),
    (3001, 40, 21, False, 8, {}, "the shape of test_gpu_multi.py on 8 ranks"),
    (3001, 40, 21, False, 2, dict(precision="bf16"), "bf16-tiles mode"),
    (4000, 26, 21, False, 2, dict(seq_chunk=768), "shards x chunks: 3 chunks per shard, the last one partial"),
    (600, 24, 21, False, 3, dict(special="zero_rank"), "rank 1 has only zero weights: exact zeros and limbs 0"),
    (600, 24, 20, True, 2, dict(special="gap_rank"), "rank 0 has only gaps: no conditional at all"),
    (600, 24, 5, False, 64, {}, "64 ranks, the documented maximum of the limb sums"),
    (3001, 40, 21, False, 2, dict(xscale=1.0), "large couplings, large -loglk"),
    (3001, 40, 21, False, 2, dict(wscale=64.0), "weights x 64: -loglk above 2^20, top limb in use"),
    (3001, 40, 21, False, 2, dict(xscale=0.0), "x = 0"),
]


@pytest.mark.parametrize("N,L,q,gap,world,opts,edge", SHARD_CASES,
                         ids=["%dx%dq%d%s-w%d%s" % (c[0], c[1], c[2], "g" if c[3] else "", c[4],
                                                   "".join("-%s%s" % kv for kv in sorted(c[5].items())))
                              for c in SHARD_CASES])
def test_shards_sum_to_the_whole(lib, N, L, q, gap, world, opts, edge):
    opts = dict(opts)
    special = opts.pop("special", None)
    codes, w, x = make_case(N, L, q, gap, seed=N + L + world, xscale=opts.pop("xscale", 0.1))
    wscale = opts.pop("wscale", None)
    if wscale:
        w *= np.float32(wscale)
    gap_code = q if gap else -1
    quiet = None
    if special == "zero_rank":
        quiet = 1
        lo, hi = shard_bounds(N, world, quiet)
        w[lo:hi] = 0.0
    elif special == "gap_rank":
        quiet = 0
        lo, hi = shard_bounds(N, world, quiet)
        codes[lo:hi] = q
    lam_h, lam_J = 0.01, 1.5
    bf16 = opts.get("precision") == "bf16"
    nh = L * q

    got = sharded_eval(lib, codes, w, x, q, gap_code, world, lam_h, lam_J, "rank", **opts)
    rev = sharded_eval(lib, codes, w, x, q, gap_code, world, lam_h, lam_J, "reversed", **opts)
    # the transport is exact and does not depend on the order of the sum
    want_nll = fxm.transported(got["nll_r"])
    assert got["nll_r"] == rev["nll_r"]
    assert got["nll"] == want_nll and rev["nll"] == want_nll, (got["nll"], rev["nll"], want_nll)
    for limbs, v in zip(got["limbs"], got["nll_r"]):
        assert tuple(int(l) for l in limbs) == fxm.split(fxm.Q(v)) + (0,)
    if wscale:
        assert all(l[2] > 0 for l in got["limbs"])
    if quiet is not None:
        assert got["nll_r"][quiet] == 0.0 and not got["limbs"][quiet].any()

    # the regulariser is added once, after the sum
    x64 = x.astype(np.float64)
    reg = lam_h * float(x64[:nh] @ x64[:nh]) + lam_J * float(x64[nh:] @ x64[nh:])
    assert abs((got["fx"] - got["nll"]) - reg) <= 1e-9 * abs(got["fx"]), (got["fx"] - got["nll"], reg)

    # against float64 on the whole alignment: the single-GPU tolerances; sharding may not loosen them
    fx64, g64, nll64 = co.plm_eval(codes, w.astype(np.float64), x64, q, lam_h, lam_J, "f64")
    ftol, gtol = (5e-3, 5e-3) if bf16 else (2e-6, 5e-6)
    e_fx, e_nll, e_g = abs(got["fx"] - fx64) / abs(fx64), abs(got["nll"] - nll64) / abs(nll64), rel_l2(got["g"], g64)
    assert e_fx <= ftol and e_nll <= ftol and e_g <= gtol, (e_fx, e_nll, e_g)

    # against one handle over the whole alignment: the summation order only
    one = whole_eval(lib, codes, w, x, q, gap_code, lam_h, lam_J, **opts)
    d_nll = abs(got["nll"] - one["nll"])
    nll_bound = world * 2.0 ** -17 + 1e-11 * abs(one["nll"])       # each rank rounds once to 2^-16; float64 sums
    e_h, e_J = rel_l2(got["g"][:nh], one["g"][:nh]), rel_l2(got["g"][nh:], one["g"][nh:])
    print("\n[%s] N=%d L=%d q=%d world=%d %s: vs float64 fx %.1e g %.1e; shards vs whole |d nll| %.2e (bound %.2e) "
          "g_h %.1e g_J %.1e" % (edge, N, L, q, world, opts, max(e_fx, e_nll), e_g, d_nll,
                                 nll_bound, e_h, e_J))
    assert d_nll <= nll_bound
    assert e_h <= 6e-7 and e_J <= 1.5e-6, (e_h, e_J)
    if world == 2:
        assert np.array_equal(got["g"], rev["g"])                         # a two-term float sum commutes


def test_fit_with_an_allreduce_callback_decodes_the_limbs(lib):
    """evc_plm_fit takes the regulariser's limb branch only when it is given an all-reduce callback.  The callback
    here doubles the n + 4 floats, i.e. plays a second rank holding the same shard: every -loglk the fit reports is then
    2 Q(-loglk of the shard) / 2^16 exactly, and the fit is the fit of one handle with the weights doubled."""
    import torch
    from evcouplings_b200.engine import _DevicePointer
    N, L, q = 600, 24, 21
    codes, w, _x = make_case(N, L, q, False, seed=5)
    n = num_params(L, q)
    fp = _lib.FitParams()
    lib.evc_fit_default_params(ctypes.byref(fp))
    fp.max_iterations, fp.lambda_h, fp.lambda_J, fp.epsilon = 10, 0.01, 2.0, 1e-9

    def fit(weights, allreduce):
        h = create_handle(lib, codes, weights, q, -1)
        rows = []
        cb = _lib.PROGRESS_CB(lambda u, k, f, xn, gn, st, nls, nll, hn, en: rows.append((f, nll)) or 0)
        ar = _lib.ALLREDUCE_CB(allreduce) if allreduce is not None else None
        res = _lib.FitResult()
        d_x = torch.zeros(n, dtype=torch.float32, device="cuda")
        try:
            _lib.check(lib.evc_plm_fit(h, p(d_x), ctypes.byref(fp), ctypes.cast(ar, vp) if ar is not None else None,
                                       None, ctypes.cast(cb, vp), None, ctypes.byref(res), None), "evc_plm_fit")
        finally:
            lib.evc_plm_destroy(h)
        return res, rows, d_x.cpu().numpy()

    calls = []

    def double(user, d_buf, count, stream):
        calls.append(count)
        torch.as_tensor(_DevicePointer(d_buf, count), device="cuda").mul_(2.0)
        return 0

    res2, rows2, x2 = fit(w, double)
    res1, rows1, x1 = fit((2.0 * w).astype(np.float32), None)
    assert res2.iterations == 10 and len(calls) == res2.evaluations and set(calls) == {n + 4}
    for _f, nll in rows2:
        units = nll * 65536
        assert units == int(units) and int(units) % 2 == 0, nll      # an even count of 2^-16 units: decoded limbs
    assert any(nll * 65536 != int(nll * 65536) for _f, nll in rows1)   # the raw double is not such a number
    f2, f1 = np.array([r[0] for r in rows2]), np.array([r[0] for r in rows1])
    assert len(f1) == len(f2) and np.abs(f2 - f1).max() <= 2e-5 * np.abs(f1).max()
    assert np.abs(x2 - x1).max() < 5e-3


# ----------------------------------------------------------------------------------------------------------------------
# 3. Hamming tile ranges
# ----------------------------------------------------------------------------------------------------------------------
def rows_with_repeats(codes, seed):
    """row 0, then 40 % of the rows, each 1-5 times, shuffled"""
    rng = np.random.default_rng(seed)
    pick = rng.choice(len(codes), int(0.4 * len(codes)), replace=False)
    rows = np.repeat(codes[pick], rng.integers(1, 6, len(pick)), axis=0)
    return np.ascontiguousarray(np.concatenate([codes[:1], rows[rng.permutation(len(rows))]]))


def hamming_codes(N, L, seed):
    """a synthetic alignment in which a third of the rows are copies of other rows with 4 % of the sites changed, so
    that neighbours exist at every length and threshold below"""
    codes = synthetic.synthetic_msa_codes(N, L, seed)
    rng = np.random.default_rng(seed)
    dst, src = rng.choice(N, N // 3, replace=False), rng.integers(0, N, N // 3)
    near = codes[src]
    flip = rng.random(near.shape) < 0.04
    near[flip] = rng.integers(0, 21, int(flip.sum()))
    codes[dst] = near
    return codes


class Tiles(object):
    """the packed planes of one alignment and evc_hamming_count_tiles(_mult) over a range into a given buffer"""

    def __init__(self, lib, codes, thr, mult=None):
        import torch
        self.lib, self.thr = lib, thr
        self.N, self.L = codes.shape
        d_codes = torch.from_numpy(np.ascontiguousarray(codes)).cuda()
        self.planes = torch.empty(lib.evc_hamming_plane_words(self.N, self.L), dtype=torch.int32, device="cuda")
        _lib.check(lib.evc_hamming_pack(p(d_codes), self.N, self.L, p(self.planes), None), "evc_hamming_pack")
        self.ntiles = int(lib.evc_hamming_num_tiles(self.N))
        self.mult = None if mult is None else torch.from_numpy(np.asarray(mult, dtype=np.int32)).cuda()

    def count_rc(self, lo, hi, counts):
        if self.mult is None:
            return self.lib.evc_hamming_count_tiles(p(self.planes), self.N, self.L, self.thr, lo, hi, p(counts), None)
        return self.lib.evc_hamming_count_tiles_mult(p(self.planes), p(self.mult), self.N, self.L, self.thr, lo, hi,
                                                     p(counts), None)

    def ranges_summed(self, ranges, prefill=0):
        """each range into its own buffer (the first one prefilled), summed like the int32 all-reduce"""
        import torch
        total = torch.zeros(self.N, dtype=torch.int64, device="cuda")
        for k, (lo, hi) in enumerate(ranges):
            counts = torch.full((self.N,), prefill if k == 0 else 0, dtype=torch.int32, device="cuda")
            _lib.check(self.count_rc(lo, hi, counts), "evc_hamming_count_tiles")
            if hi == lo:
                assert int(counts.abs().sum().item()) == (prefill * self.N if k == 0 else 0)
            total += counts
        return total.cpu().numpy() - prefill


def _partitions(ntiles, seed):
    for world in sorted({1, 2, 3, 8, ntiles, ntiles + 3}):
        yield "world %d" % world, [shard_bounds(ntiles, world, r) for r in range(world)]
    cuts = [0] + sorted(int(c) for c in np.random.default_rng(seed).integers(0, ntiles + 1, 4)) + [ntiles]
    yield "uneven", list(zip(cuts[:-1], cuts[1:]))


HAMMING_SHAPES = [(100, 40, 0.8), (128, 33, 0.8), (129, 33, 0.8), (257, 97, 0.7), (1000, 97, 0.7), (3000, 300, 0.8),
                  (777, 800, 0.9)]


@pytest.mark.parametrize("N,L,theta", HAMMING_SHAPES)
def test_tile_ranges_sum_to_the_exact_counts(lib, N, L, theta):
    codes = hamming_codes(N, L, N + L)
    thr = msa.identity_threshold_count(theta, L)
    exact = co.hamming_counts(codes, thr)
    assert exact.min() >= 1 and (exact > 1).sum() >= N // 4
    t = Tiles(lib, codes, thr)
    assert t.ntiles == (-(-N // 128)) * (-(-N // 128) + 1) // 2
    for name, ranges in _partitions(t.ntiles, N):
        assert np.array_equal(t.ranges_summed(ranges, prefill=7), exact), name        # += : the 7s are added to
    if N == 100:
        assert [shard_bounds(t.ntiles, 2, r) for r in range(2)] == [(0, 1), (1, 1)]    # rank 1: the empty range


@pytest.mark.parametrize("N,L,theta", HAMMING_SHAPES)
def test_tile_ranges_with_multiplicities(lib, N, L, theta):
    from test_gpu_unique_rows import host_unique
    rows = rows_with_repeats(hamming_codes(N, L, N + L), N)
    thr = msa.identity_threshold_count(theta, L)
    exact = co.hamming_counts(rows, thr)
    first, inverse, mult = host_unique(lib, rows)
    assert len(first) < len(rows)
    t = Tiles(lib, rows[first], thr, mult)
    for name, ranges in _partitions(t.ntiles, N):
        assert np.array_equal(t.ranges_summed(ranges)[inverse], exact), name


def test_tile_range_out_of_bounds_is_refused(lib):
    import torch
    codes = synthetic.synthetic_msa_codes(300, 40, 1)
    t = Tiles(lib, codes, 32)
    tm = Tiles(lib, codes, 32, np.ones(300))
    counts = torch.full((300,), 7, dtype=torch.int32, device="cuda")
    for tiles in (t, tm):
        for lo, hi in ((-1, 1), (0, t.ntiles + 1), (2, 1)):
            assert tiles.count_rc(lo, hi, counts) != 0
            assert b"tile range out of bounds" in lib.evc_last_error()
    torch.cuda.synchronize()
    assert bool((counts == 7).all())


# ----------------------------------------------------------------------------------------------------------------------
# 4. two real ranks on one device
# ----------------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket(socket.AF_INET, socket.SOCK_STREAM)
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def two_processes(script, *args):
    """Two rank processes with the environment the launcher gives them, both on the current device; each is waited
    for under a timeout and killed if it does not end."""
    port = _free_port()
    procs = []
    for r in range(2):
        env = dict(os.environ, RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1",
                   MASTER_PORT=str(port))
        env.pop("EVC_NUM_GPUS", None)
        procs.append(subprocess.Popen([sys.executable, script] + list(args), env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.STDOUT, text=True))
    outs = []
    try:
        for pr in procs:
            outs.append(pr.communicate(timeout=RANK_TIMEOUT_S)[0])
    finally:
        for pr in procs:
            if pr.poll() is None:
                pr.kill()
                pr.wait()
    assert [pr.returncode for pr in procs] == [0, 0], "\n".join(o[-2000:] for o in outs)


def gloo_two_ranks(**kw):
    """run_plmc on two ranks through the product's launcher and worker, with the default (CUDA) engine; the ranks
    share the current device and all-reduce its buffers over gloo"""
    from evcouplings_b200 import launcher
    return launcher.run_plmc_multi_gpu(2, kw, return_run=True, backend="gloo", timeout=RANK_TIMEOUT_S)


def test_two_ranks_one_device_lockstep(tmp_path):
    from test_gpu_multi import check_full_fit_lockstep
    codes = rows_with_repeats(synthetic.synthetic_msa_codes(1000, 40, 17), 17)      # ranks shard the distinct rows
    assert len(codes) >= 400
    run = check_full_fit_lockstep(tmp_path, codes[:400], "gloo", two_processes)
    assert run.timings["unique_rows"] < run.alignment.n_valid == 400


def test_launcher_two_ranks_one_device(tmp_path):
    from test_gpu_multi import check_two_ranks_equal_one
    check_two_ranks_equal_one(tmp_path, synthetic.synthetic_msa_codes(600, 40, 19), gloo_two_ranks)


def test_launcher_two_ranks_one_device_precision_schedule(tmp_path):
    """precision "auto": the bf16 phase, the switch to hi + lo products (which evaluates again through the callback)
    and the convergence test run on two ranks"""
    from test_gpu_multi import check_two_ranks_equal_one
    (r2, run2), (r1, run1) = check_two_ranks_equal_one(
        tmp_path, synthetic.synthetic_msa_codes(3001, 40, 1), gloo_two_ranks, precision="auto", iterations="max",
        epsilon=1e-3, lambda_J=2.0)
    s2, s1 = run2.timings["fit_switched_at"], run1.timings["fit_switched_at"]
    two = np.loadtxt(str(tmp_path / "two_ECs.txt"), usecols=5)
    one = np.loadtxt(str(tmp_path / "one_ECs.txt"), usecols=5)
    rms = float(np.sqrt(np.mean((two - one) ** 2)))
    print("\nprecision auto: left bf16 at iteration %d on two ranks (%d iterations, %s), %d on one (%d, %s); EC rms %.2e"
          % (s2, len(r2.iteration_table), r2.optimization_status, s1, len(r1.iteration_table),
             r1.optimization_status, rms))
    assert s2 >= 1 and s1 >= 1
    assert s2 == s1 or rms <= 1e-4


def test_two_ranks_one_device_save_and_resume(tmp_path):
    """the 2-int agreement all-reduce of the checkpoint gate and "rank 0 writes, every rank reads" on a device"""
    from test_gpu_fit_checkpoint import check_two_ranks_save_and_resume
    check_two_ranks_save_and_resume(tmp_path, lambda **kw: gloo_two_ranks(**kw)[0])
