"""
Replay of the device L-BFGS step (vecops.cu, driven by fit.cu) in the device's own fp32 arithmetic.  Test
infrastructure, not product code.

Every n-vector the fit forms is an fp32 operation whose rounding is fully specified, so the replay rebuilds it bit
for bit; every scalar is a double sum along the kernels' fixed reduction tree, which the replay brackets instead:

  * fp32 fma is correctly rounded (fmaf32): the product a b of two fp32 values is exact in float64, s = p + c is
    formed with its exact error e (TwoSum), s is rounded to odd (one ulp towards e when e != 0 and s has an even last
    bit), and only then rounded to fp32.  Round-to-odd at 53 bits followed by a rounding to 24 bits is the correctly
    rounded result.
  * step           x_try = fmaf(float(t), d, x)
  * regulariser    g = fmaf(lam + lam, x, g_data), lam = lambda_h on the first L q entries and lambda_J on the rest
  * pair           s = x - xp, y = g - gp (one fp32 subtraction each); y.s and y.y summed in double
  * two-loop       over the `bound` pairs before ring slot `end` (newest first):
                       d = -g;  for j newest .. oldest:  alpha_j = (s_j . d) / ys_j;  d = fmaf(-float(alpha_j), y_j, d)
                       d = d * gamma  (one fp32 multiply after the oldest pair), gamma = float(ys_newest / yy)
                       for j oldest .. newest:  coef = alpha_j - (y_j . d) / ys_j;  d = fmaf(float(coef), s_j, d)
                   alpha, coef and ys_newest / yy are formed in double and rounded to fp32 only where they meet d.
  * double sums    a per-thread chain over the grid-stride loop (ceil(n / (1184 * 256)) terms), a 5-level xor
                   butterfly, 8 warps added in sequence, at most 2 partials per thread of final_sum and a 10-level tree:
                   a tree of depth k = chain + 25.  The replay takes the exact float64 products, sums them by a
                   compensated pairwise sum (TwoSum at every level) and allows the device gamma_k sum |p_i| around it,
                   a bound that follows from the tree (device_tree_sum is a numpy model of it, for the CPU tests).
  * ambiguity      a double that is later rounded to fp32 (alpha, coef) may have two fp32 roundings inside its
                   interval.  The replay then carries every rounding forward as a branch, and a device vector must
                   equal one branch bit for bit; the number of branches opened is reported.

Generate mode (direction(..., generate=True)) forms the scalars with the tree model instead of intervals and gives one
vector; ``mutation`` makes it commit one plausible kernel mistake (MUTATIONS), so the CPU tests can show that the
checkers the GPU tests use reject it.
"""
import math

import numpy as np

F32 = np.float32
F64 = np.float64
RED_BLOCKS, RED_THREADS = 1184, 256
GRID = RED_BLOCKS * RED_THREADS
U64 = 2.0 ** -53

MUTATIONS = ("gamma_oldest",          # gamma = ys_oldest / yy instead of the newest pair's
             "no_gamma",              # no gamma scaling after the first loop
             "first_loop_ascending",  # the first loop walks the pairs oldest -> newest
             "coef_double",           # alpha / coef applied in double, d = float(d + coef v)
             "reg_unfused",           # g = (2 lam x) + g_data as a rounded multiply and a rounded add
             "lambda_nh_plus",        # lambda_h reaches one entry past L q
             "lambda_nh_minus",       # lambda_J starts one entry before L q
             "y_reversed",            # y = gp - g
             "ring_wrap_off_by_one")  # after the walk wraps past slot 0, every slot is one too low


# ---- fp32 arithmetic ------------------------------------------------------------------------------------------------
def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def fmaf32(a, b, c):
    """Correctly rounded fp32 fma(a, b, c), elementwise (broadcasting)."""
    a = np.asarray(a, dtype=F32).astype(F64)
    b = np.asarray(b, dtype=F32).astype(F64)
    c = np.asarray(c, dtype=F32).astype(F64)
    p = a * b                                    # exact: 24 + 24 significant bits
    s, e = _two_sum(p, c)
    s = np.atleast_1d(s)
    e = np.broadcast_to(e, s.shape)
    bump = (e != 0) & ((s.view(np.int64) & 1) == 0)
    if bump.any():
        s = s.copy()
        s[bump] = np.nextafter(s[bump], np.where(e[bump] > 0, np.inf, -np.inf))
    out = s.astype(F32)
    return out if np.ndim(p) else out[0]


def step(x, d, t):
    """The trial point of the line search: fmaf(float(t), d, x)."""
    return fmaf32(F32(t), d, x)


def lambdas(n, nh, lambda_h, lambda_J, mutation=None):
    nh = nh + (1 if mutation == "lambda_nh_plus" else -1 if mutation == "lambda_nh_minus" else 0)
    lam = np.full(n, F32(lambda_J), dtype=F32)
    lam[:max(0, min(n, nh))] = F32(lambda_h)
    return lam


def regulariser(x, g_data, nh, lambda_h, lambda_J, mutation=None):
    """g_data + 2 lambda x as the regulariser kernel forms it."""
    lam = lambdas(len(x), nh, lambda_h, lambda_J, mutation)
    if mutation == "reg_unfused":
        return ((lam + lam) * x) + g_data
    return fmaf32(lam + lam, x, g_data)


def pair(x, xp, g, gp, mutation=None):
    """The correction pair (s, y) of pair_update_kernel."""
    return x - xp, (gp - g if mutation == "y_reversed" else g - gp)


# ---- double sums ----------------------------------------------------------------------------------------------------
def exact_sum(p):
    """sum(p) by a compensated pairwise sum: TwoSum at every level, the errors summed on the side."""
    s = np.asarray(p, dtype=F64)
    errs = []
    while s.size > 1:
        if s.size & 1:
            s = np.append(s, 0.0)
        s, e = _two_sum(s[0::2], s[1::2])
        errs.append(float(np.sum(e)))
    return float(s[0] if s.size else 0.0) + math.fsum(errs)


def tree_depth(n):
    return max(1, -(-int(n) // GRID)) + 5 + 8 + 2 + 10


def gamma_k(k):
    return k * U64 / (1.0 - k * U64)


def sum_bound(p, extra=0):
    """(reference, bound): the device's double sum of the terms p lies within reference +- bound.  `extra` adds
    roundings the terms themselves carry (a product that is not exact in double)."""
    p = np.asarray(p, dtype=F64)
    ref = exact_sum(p)
    return ref, gamma_k(tree_depth(p.size) + extra) * float(np.sum(np.abs(p))) + 2 * U64 * abs(ref)


def dot_bound(a, b):
    return sum_bound(np.asarray(a, dtype=F32).astype(F64) * np.asarray(b, dtype=F32).astype(F64))


def device_tree_sum(p):
    """numpy model of the device's double reduction: grid-stride chain, xor butterfly, 8 warps, final_sum's tree."""
    p = np.asarray(p, dtype=F64)
    chain = max(1, -(-p.size // GRID))
    a = np.zeros(chain * GRID)
    a[:p.size] = p
    a = a.reshape(chain, GRID)
    acc = np.zeros(GRID)
    for i in range(chain):
        acc = acc + a[i]
    v = acc.reshape(RED_BLOCKS * 8, 32)
    lane = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[:, lane ^ o]
    w = v[:, 0].reshape(RED_BLOCKS, 8)
    part = np.zeros(RED_BLOCKS)
    for k in range(8):
        part = part + w[:, k]
    s = np.zeros(1024)
    s = s + part[:1024]
    s[:RED_BLOCKS - 1024] = s[:RED_BLOCKS - 1024] + part[1024:]
    o = 512
    while o > 0:
        s[:o] = s[:o] + s[o:2 * o]
        o >>= 1
    return float(s[0])


def within(value, ref_bound, slack=0.0):
    ref, b = ref_bound
    return abs(float(value) - ref) <= b + slack


# ---- the two-loop recursion -----------------------------------------------------------------------------------------
def _outward(lo, hi):
    return float(np.nextafter(lo, -np.inf)), float(np.nextafter(hi, np.inf))


def f32_candidates(lo, hi):
    """Every fp32 rounding of a double in [lo, hi] (rounding is monotone: the ones between the ends' roundings)."""
    a, b = F32(lo), F32(hi)
    out = [a]
    while out[-1] < b and len(out) < 8:
        out.append(np.nextafter(out[-1], F32(np.inf)))
    return out


class TooManyBranches(RuntimeError):
    pass


def ring_order(m, bound, end, mutation=None):
    """Ring slots of the `bound` pairs before `end`, newest first."""
    order = []
    for i in range(bound):
        j = (end - 1 - i) % m
        if mutation == "ring_wrap_off_by_one" and end - 1 - i < 0:
            j = (j - 1) % m
        order.append(j)
    return order


def direction(g, S, Y, ys, yy, m, bound, end, alphas=None, generate=False, mutation=None, branches=True,
              max_branches=64, bad_alphas=None):
    """d = -H g as lbfgs_direction forms it.  S[j], Y[j]: ring slot j (fp32); ys[j] (double per slot) and yy (the
    newest pair's y.y) as the device holds them.  alphas: the device's double alpha per slot, when read back: the
    first loop then follows them without branching, and every alpha outside its interval is appended to
    `bad_alphas`.  Returns (list of candidate d, branches opened); generate mode, or branches=False (every double
    taken at its reference value), gives exactly one candidate."""
    bad_alphas = [] if bad_alphas is None else bad_alphas
    g = np.asarray(g, dtype=F32)
    d0 = -g
    if bound == 0:
        return [d0], 0
    order = ring_order(m, bound, end, mutation)
    first = order[::-1] if mutation == "first_loop_ascending" else order
    second = order[::-1]
    newest, oldest = order[0], order[-1]
    gamma = F32(1.0) if mutation == "no_gamma" else F32(ys[oldest if mutation == "gamma_oldest" else newest] / yy)
    point = generate or not branches

    def dot_iv(u, v):
        p = u.astype(F64) * v.astype(F64)
        if generate:
            t = device_tree_sum(p)
            return t, t
        ref, b = sum_bound(p)
        return (ref, ref) if not branches else (ref - b, ref + b)

    def div_iv(iv, den):
        lo, hi = sorted((iv[0] / den, iv[1] / den))
        return (lo, hi) if point else _outward(lo, hi)

    def sub_iv(a, b):
        lo, hi = a[0] - b[1], a[1] - b[0]
        return (lo, hi) if point else _outward(lo, hi)

    def update(d, c, v, sign):
        if mutation == "coef_double":
            return (d.astype(F64) + sign * c * v.astype(F64)).astype(F32)
        return fmaf32(F32(sign) * F32(c), v, d)

    def rounding(iv):
        if mutation == "coef_double":
            return [iv[0]]
        return f32_candidates(*iv) if branches and not generate else [F32(iv[0])]

    ops = [("alpha", j, i == bound - 1) for i, j in enumerate(first)] + [("coef", j, False) for j in second]
    results, opened = [], [0]

    def run(d, start, alpha):
        for idx in range(start, len(ops)):
            kind, j, last = ops[idx]
            if kind == "alpha":
                alpha[j] = div_iv(dot_iv(S[j], d), ys[j])
                if alphas is not None:
                    if not alpha[j][0] <= alphas[j] <= alpha[j][1]:
                        bad_alphas.append((j, float(alphas[j]), alpha[j]))
                    alpha[j] = (float(alphas[j]), float(alphas[j]))
                iv, v, sign = alpha[j], Y[j], -1.0
            else:
                iv = sub_iv(alpha[j], div_iv(dot_iv(Y[j], d), ys[j]))
                v, sign = S[j], 1.0
            cands = rounding(iv)
            if len(cands) > 1:
                opened[0] += 1
                if opened[0] > max_branches:
                    raise TooManyBranches("more than %d branches" % max_branches)
                for c in cands[1:]:
                    nd = update(d, c, v, sign)
                    run(nd * gamma if kind == "alpha" and last else nd, idx + 1, dict(alpha))
            d = update(d, cands[0], v, sign)
            if kind == "alpha" and last:
                d = d * gamma
        results.append(d)

    run(d0, 0, {})
    return results, opened[0]


def match(dev, candidates):
    """Index of the candidate equal to the device vector bit for bit, or -1."""
    dev = np.ascontiguousarray(dev, dtype=F32).view(np.uint32)
    for i, c in enumerate(candidates):
        if np.array_equal(dev, np.ascontiguousarray(c, dtype=F32).view(np.uint32)):
            return i
    return -1


def same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a, dtype=F32).view(np.uint32),
                          np.ascontiguousarray(b, dtype=F32).view(np.uint32))


def first_mismatch(a, b):
    a = np.ascontiguousarray(a, dtype=F32).view(np.uint32)
    b = np.ascontiguousarray(b, dtype=F32).view(np.uint32)
    bad = np.flatnonzero(a != b)
    return int(bad[0]) if bad.size else -1


def plain_two_loop(g, S, Y, m, bound, end):
    """float64 two-loop over the same ring (ys, yy and gamma recomputed in float64), the CPU tests' yardstick."""
    d = -np.asarray(g, dtype=F64)
    order = ring_order(m, bound, end)
    S64 = {j: np.asarray(S[j], dtype=F64) for j in order}
    Y64 = {j: np.asarray(Y[j], dtype=F64) for j in order}
    ys = {j: float(Y64[j] @ S64[j]) for j in order}
    alpha = {}
    for j in order:
        alpha[j] = float(S64[j] @ d) / ys[j]
        d = d - alpha[j] * Y64[j]
    if order:
        d = d * (ys[order[0]] / float(Y64[order[0]] @ Y64[order[0]]))
    for j in order[::-1]:
        d = d + (alpha[j] - float(Y64[j] @ d) / ys[j]) * S64[j]
    return d
