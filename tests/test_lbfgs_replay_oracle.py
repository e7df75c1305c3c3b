"""
CPU checks of oracle/lbfgs_replay.py, the replay of the device L-BFGS step that tests/test_gpu_lbfgs_replay.py compares
the device with: its fp32 fma against libm and exact rationals, its two-loop against a plain float64 two-loop, its
summation bound against a model of the device's reduction tree, and every kernel mistake in MUTATIONS rejected by the
checks the GPU tests make.
"""
import ctypes
import ctypes.util
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle import lbfgs_replay as lr

F32 = np.float32


def _libm_fmaf():
    libm = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
    f = libm.fmaf
    f.restype = ctypes.c_float
    f.argtypes = [ctypes.c_float] * 3
    return f


def _round_f32(r):
    """Fraction -> nearest fp32, ties to even."""
    f = F32(float(r))
    best = None
    for c in (np.nextafter(f, F32(-np.inf)), f, np.nextafter(f, F32(np.inf))):
        dist = abs(Fraction(float(c)) - r)
        key = (dist, int(np.array(c, dtype=F32).view(np.uint32)) & 1)
        if best is None or key < best[0]:
            best = (key, c)
    return best[1]


def _midpoint_triples(rng, k=4000):
    """a b + c within one float64 ulp of an fp32 midpoint c +- h (h = half an ulp of c): a b = h (1 - 2^-2j),
    j = 15..23, just inside the midpoint, or h (1 + 2^-e) from a factorisation 2^e + 1 = A B, just outside it"""
    c = (rng.uniform(1, 2, k) * 2.0 ** rng.integers(-60, 60, k)).astype(F32)
    c *= np.where(rng.random(k) < 0.5, -1, 1).astype(F32)
    h = np.spacing(np.abs(c)).astype(np.float64) / 2
    j = rng.integers(15, 24, k)
    a = h * (1 + 2.0 ** -j)
    b = 1 - 2.0 ** -j
    fac = np.array([(641, 6700417, 32), (1774001, 38737, 36), (17, 15790321, 28)], dtype=np.float64)
    pick = fac[rng.integers(0, 3, k)]
    out = rng.random(k) < 0.5
    a = np.where(out, h * pick[:, 0] * 2.0 ** -pick[:, 2], a)
    b = np.where(out, pick[:, 1], b)
    b = np.where(rng.random(k) < 0.5, -b, b)                # towards either neighbour midpoint
    return a.astype(F32), b.astype(F32), c


def test_fmaf32_matches_libm_on_random_and_midpoint_triples():
    fmaf = _libm_fmaf()
    rng = np.random.default_rng(0)
    n = 100_000
    a = (rng.normal(size=n) * 2.0 ** rng.integers(-20, 20, n)).astype(F32)
    b = (rng.normal(size=n) * 2.0 ** rng.integers(-20, 20, n)).astype(F32)
    c = (rng.normal(size=n) * 2.0 ** rng.integers(-40, 40, n)).astype(F32)
    ma, mb, mc = _midpoint_triples(rng)
    a, b, c = np.concatenate([a, ma]), np.concatenate([b, mb]), np.concatenate([c, mc])
    got = lr.fmaf32(a, b, c)
    want = np.array([fmaf(float(x), float(y), float(z)) for x, y, z in zip(a, b, c)], dtype=F32)
    assert lr.same_bits(got, want), lr.first_mismatch(got, want)
    # the midpoint triples are where rounding the float64 sum straight to fp32 goes wrong
    naive = (ma.astype(np.float64) * mb + mc).astype(F32)
    assert np.count_nonzero(naive != lr.fmaf32(ma, mb, mc)) > len(ma) // 4


def test_fmaf32_matches_exact_rationals():
    rng = np.random.default_rng(1)
    a = rng.normal(size=1000).astype(F32)
    b = rng.normal(size=1000).astype(F32)
    c = rng.normal(size=1000).astype(F32)
    ma, mb, mc = _midpoint_triples(rng, 1000)
    a, b, c = np.concatenate([a, ma]), np.concatenate([b, mb]), np.concatenate([c, mc])
    got = lr.fmaf32(a, b, c)
    want = np.array([_round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z)))
                     for x, y, z in zip(a, b, c)], dtype=F32)
    assert lr.same_bits(got, want), lr.first_mismatch(got, want)


def _history(rng, n, m, pairs):
    """`pairs` pairs pushed into a ring of m: S, Y per slot, ys per slot, yy of the newest, end."""
    S, Y = [np.zeros(n, F32) for _ in range(m)], [np.zeros(n, F32) for _ in range(m)]
    ys = np.zeros(m)
    end, yy = 0, 0.0
    for _ in range(pairs):
        s = (0.1 * rng.normal(size=n)).astype(F32)
        y = (s * rng.uniform(0.5, 2.0, n) + 0.01 * rng.normal(size=n)).astype(F32)
        S[end], Y[end] = s, y
        ys[end] = lr.exact_sum(s.astype(np.float64) * y)
        yy = lr.exact_sum(y.astype(np.float64) * y)
        end = (end + 1) % m
    return S, Y, ys, yy, end


@pytest.mark.parametrize("m,pairs", [(1, 1), (1, 3), (5, 5), (5, 8), (32, 32), (32, 45)])
def test_direction_agrees_with_a_float64_two_loop(m, pairs):
    rng = np.random.default_rng(m * 100 + pairs)
    n = 3000
    S, Y, ys, yy, end = _history(rng, n, m, pairs)
    g = rng.normal(size=n).astype(F32)
    bound = min(m, pairs)
    (d,), opened = lr.direction(g, S, Y, ys, yy, m, bound, end, branches=False)
    assert opened == 0
    ref = lr.plain_two_loop(g, S, Y, m, bound, end)
    assert np.linalg.norm(d - ref) <= 4e-6 * math.sqrt(bound) * np.linalg.norm(ref)
    # the bracketing replay and the tree model agree on it
    cands, opened = lr.direction(g, S, Y, ys, yy, m, bound, end)
    (gen,), _ = lr.direction(g, S, Y, ys, yy, m, bound, end, generate=True)
    assert lr.match(gen, cands) >= 0 and opened <= 2


def _terms(rng, n, kind):
    if kind == "random":
        return rng.normal(size=n) * rng.normal(size=n)
    # adversarial cancellation: large terms that cancel pairwise and across the tree, and a tiny remainder
    big = rng.normal(size=n // 2) * 2.0 ** rng.integers(0, 40, n // 2)
    p = np.concatenate([big, -big * (1 + 2.0 ** -30), rng.normal(size=n - 2 * (n // 2)) * 1e-3])
    return p[rng.permutation(n)]


@pytest.mark.parametrize("n", [lr.GRID - 1, lr.GRID, lr.GRID + 1, 8_780_100])
@pytest.mark.parametrize("kind", ["random", "cancel"])
def test_tree_bound_contains_the_device_tree(n, kind):
    rng = np.random.default_rng(n % 1000 + (kind == "cancel"))
    p = _terms(rng, n, kind)
    ref, bound = lr.sum_bound(p)
    assert abs(ref - math.fsum(p.tolist())) <= 2 * lr.U64 * abs(ref) + 1e-300
    tree = lr.device_tree_sum(p)
    assert abs(tree - ref) <= bound, (tree, ref, bound)
    # the bound is not vacuous: a slip of one term is far outside it
    assert bound < np.sort(np.abs(p))[n // 2]


def test_every_mutation_is_rejected():
    rng = np.random.default_rng(7)
    n, m, L, q = 2000, 5, 8, 4
    nh = L * q
    S, Y, ys, yy, end = _history(rng, n, m, 7)              # wrapped: end = 2, the walk crosses slot 0
    g = rng.normal(size=n).astype(F32)
    x = rng.normal(size=n).astype(F32)
    g_data = rng.normal(size=n).astype(F32)
    xp = (x - 0.1 * rng.normal(size=n)).astype(F32)
    gp = rng.normal(size=n).astype(F32)
    lam_h, lam_J = F32(0.01), F32(1.7)

    def direction_ok(mutation):
        (d,), _ = lr.direction(g, S, Y, ys, yy, m, m, end, generate=True, mutation=mutation)
        cands, _ = lr.direction(g, S, Y, ys, yy, m, m, end)
        return lr.match(d, cands) >= 0

    def regulariser_ok(mutation):
        return lr.same_bits(lr.regulariser(x, g_data, nh, lam_h, lam_J, mutation),
                            lr.regulariser(x, g_data, nh, lam_h, lam_J))

    def pair_ok(mutation):
        s, y = lr.pair(x, xp, g, gp, mutation)
        s0, y0 = lr.pair(x, xp, g, gp)
        return lr.same_bits(s, s0) and lr.same_bits(y, y0)

    assert direction_ok(None) and regulariser_ok(None) and pair_ok(None)
    caught = {}
    for mut in lr.MUTATIONS:
        caught[mut] = not (direction_ok(mut) and regulariser_ok(mut) and pair_ok(mut))
    assert all(caught.values()), caught
