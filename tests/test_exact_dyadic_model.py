"""
The dyadic case: inputs on which the PLM objective's gradient and pair counts are exact in float32, so that every
device path can be compared with an exact reference bit for bit (tests/test_gpu_exact_dyadic.py).  This file checks
the construction on the CPU.

Per site i a set A_i of |A_i| in {1, 2, 4, 8, 16} states (|A_i| <= q):
* h_i(a) = 0 on A_i and H_OUT = -2048 elsewhere (exact in bf16; far enough below zero that float64 exp underflows to
  exactly 0 as well);
* J_ij(a, b) = k / 64 with |k| <= 255 (exact in bf16 hi, lo = 0), nonzero only when a is not in A_i and b is not in
  A_j, and L max|J| <= 1000: a logit outside A_i is at most -1048, so its exp is 0 in float32 and float64;
* every logit on A_i is exactly 0 whatever the sequence, so P_i(a) = 1 / |A_i| on A_i and 0 elsewhere, exactly;
* weights w_n = k_n 2^-e with small k_n (with distinct rows, w mult follows the same rule); a sequence with an
  ignored gap at site i has no conditional i and no one-hot column at i.
Then r(n, i, a) = w_n (P_i(a) - [s_ni = a]) is exact, and the data gradient has the closed form
    g_h(i, a)       = sum_n r(n, i, a)
    g_J(i,j)(a, b)  = P_i(a) C_j^(i)(b) + C_i^(j)(a) P_j(b) - 2 F_ij(a, b)
with F_ij the weighted pair count and C^(.) its marginals over the sequences that are not gaps at the other site.

Exactness budget: u = 2^-e / max|A| (and the resolution of the regulariser's 2 lambda x where it is used) divides
every residual, product and partial sum; the sum of |terms| of an entry is at most 2 sum(w) (+ max |2 lambda x|).
dyadic_case asserts that this bound over u is <= 2^22 (two guard bits below float32's 24, for the alignment of the
tensor core's accumulation inside a K group), and k_n (max|A| - 1) < 2^8 so that every residual has at most 8
significant bits (the bf16-tiles mode keeps only the hi term).  Then the sum does not depend on its order, on
split-K, chunks, tiles, clusters or ranks, and both precision modes must give the exact gradient.

What the construction cannot see: a coupling block misplaced between two slots outside the A sets changes logits
that underflow to 0 either way.  A block that lands on an A-state slot moves a logit off 0 and is caught.

fx is not exact (log |A_i|), and the loops oracle and the C port take log of an exact 0 (+inf) for an observed state
outside A_i, where the device forms z_s - max - log sum and stays finite.  fx and -loglk are therefore compared with
the log-sum-exp form of po.objective (relative 2e-6).  po.objective is not used as the exact gradient: it forms P as
exp(Z - lse), one float64 ulp away from 1/8 at |A| = 8.

The sensitivity table (N = 100 000, L = 20, q = 21, w = 1) prints how far one-sequence slips move the exact gradient:
dropping one sequence or counting one twice changes about 1 650 entries by up to 16 u, 7.4e-5 to 7.6e-5 relative L2;
dropping a 64-sequence K block 8.7e-4.  The whole-vector tolerance VEC_REL = 2e-5 of test_gpu_tc_edges.py would see
these on this data; it would not see a slip whose share of the gradient is below 2e-5, and it never says where.
"""
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import c_oracle as co  # noqa: E402
from oracle import plm_oracle as po  # noqa: E402

H_OUT = -2048.0
A_SIZES = (1, 2, 4, 8, 16)
BUDGET = 2 ** 22
VEC_REL = 2e-5          # whole-vector relative L2 tolerance of tests/test_gpu_tc_edges.py


def lsb(v):
    """The largest power of two that divides the nonzero dyadic float v (its last significant bit)."""
    m, e = math.frexp(abs(float(v)))
    k = int(m * 2 ** 53)
    return 2.0 ** (e - 53) * (k & -k)


def dyadic_case(N, L, q, gap=False, seed=0, amax=8, wk=1, we=0, zero_w=0.0, gap_prob=0.05, jdensity=0.5,
                lam=None, wmult=1, outside=()):
    """Codes, weights w = k 2^-we (k uniform in 1..wk, a share zero_w of them 0), parameters x of the dyadic case,
    the A sets and the resolution u.  A zero weight hides its sequence from every sum, so it never falls on the last
    sequence or on a sequence next to a 64-sequence edge (n % 64 in {0, 63}; every K block, tile, X row and chunk edge
    of the device is a multiple of 64).  gap: codes q are ignored gaps (a share gap_prob of them).  lam = (lambda_h,
    lambda_J): dyadic regulariser weights whose 2 lambda x terms enter the budget.  wmult: the largest multiplicity a
    weight will be multiplied by (distinct rows).  outside: (site, state) pairs kept out of the A sets.  Asserts the
    exactness budget of the module docstring."""
    rng = np.random.default_rng(seed)
    sizes = np.array([s for s in A_SIZES if s <= min(q, amax)])
    asize = rng.choice(sizes, L)
    A = np.zeros((L, q), dtype=bool)
    for i in range(L):
        banned = [a for s, a in outside if s == i]
        if banned:
            allowed = np.setdiff1d(np.arange(q), banned)
            while asize[i] > len(allowed):
                asize[i] //= 2
            A[i, rng.choice(allowed, asize[i], replace=False)] = True
        else:
            A[i, rng.choice(q, asize[i], replace=False)] = True
    codes = rng.integers(0, q, size=(N, L), dtype=np.uint8)
    if gap:
        codes[rng.random((N, L)) < gap_prob] = q
    k = rng.integers(1, wk + 1, N)
    if zero_w:
        zero = rng.random(N) < zero_w
        n = np.arange(N)
        zero &= (n % 64 != 0) & (n % 64 != 63) & (n != N - 1)
        k[zero] = 0
    w = (k * 2.0 ** -we).astype(np.float32)
    jmax = min(255, 64000 // L)                      # L max|J| <= 1000
    h = np.where(A, 0.0, H_OUT).astype(np.float32)
    iu, ju = np.triu_indices(L, 1)
    J = np.zeros((len(iu), q, q), dtype=np.float32)
    out = ~A
    step = max(1, (1 << 22) // (q * q))
    for p0 in range(0, len(iu), step):
        sl = slice(p0, p0 + step)
        mask = out[iu[sl]][:, :, None] & out[ju[sl]][:, None, :]
        mask &= rng.random(mask.shape, dtype=np.float32) < jdensity
        val = rng.integers(-jmax, jmax + 1, size=mask.shape, dtype=np.int16)
        J[sl] = np.where(mask, val, 0).astype(np.float32) / 64
    x = np.concatenate([h.ravel(), J.ravel()])
    amx = int(asize.max())
    u = 2.0 ** -we / amx
    extra = 0.0
    if lam is not None:
        lam_h, lam_J = lam
        for l, v in ((lam_h, -H_OUT), (lam_J, 1.0 / 64)):
            if l:
                u = min(u, lsb(2 * l) * lsb(v))
        extra = max(2 * lam_h * -H_OUT, 2 * lam_J * jmax / 64)
    budget = (2 * float(w.astype(np.float64).sum()) + extra) / u
    assert budget <= BUDGET, "exactness budget %.3g > 2^22" % budget
    assert wk * wmult * (amx - 1) < 2 ** 8, "residuals need more than 8 significant bits"
    return dict(codes=codes, w=w, x=x, A=A, asize=asize, u=u, budget=budget, q=q, gap=gap,
                gap_code=q if gap else -1, N=N, L=L)


def one_hot(codes, q):
    """(n, L q) float64 one-hot; codes >= q (ignored gaps) give zero rows."""
    n, L = codes.shape
    X = np.zeros((n, L * q))
    r, c = np.nonzero(codes < q)
    X[r, c * q + codes[r, c]] = 1.0
    return X


def probabilities(A):
    return A / A.sum(axis=1, keepdims=True)


def pair_counts(codes, w, q, chunk=8192):
    """F = X^T diag(w) X in float64, (L q) x (L q): exact sums of dyadic weights."""
    N, L = codes.shape
    F = np.zeros((L * q, L * q))
    w = np.asarray(w, dtype=np.float64)
    for s0 in range(0, N, chunk):
        X = one_hot(codes[s0:s0 + chunk], q)
        F += X.T @ (w[s0:s0 + chunk, None] * X)
    return F


def gradient_from_counts(F, A):
    """The closed form of the module docstring from the pair counts F."""
    L, q = A.shape
    P = probabilities(A)
    F4 = F.reshape(L, q, L, q)
    fi = np.einsum("iaia->ia", F4)
    gh = P * fi.sum(axis=1, keepdims=True) - fi
    iu, ju = np.triu_indices(L, 1)
    Fij = F4[iu, :, ju, :]                            # (pairs, a, b)
    gJ = P[iu][:, :, None] * Fij.sum(axis=1)[:, None, :] + Fij.sum(axis=2)[:, :, None] * P[ju][:, None, :] - 2 * Fij
    return np.concatenate([gh.ravel(), gJ.ravel()])


def exact_gradient(codes, w, A, q):
    """The exact data gradient of the dyadic case, float64, in the layout of x."""
    return gradient_from_counts(pair_counts(codes, w, q), A)


def exact_counts(codes, w, q):
    """Weighted counts before normalisation, as evc_plm_weighted_counts returns them: f_i (L, q), f_ij (pairs, q, q)."""
    L = codes.shape[1]
    F4 = pair_counts(codes, w, q).reshape(L, q, L, q)
    iu, ju = np.triu_indices(L, 1)
    return np.einsum("iaia->ia", F4), F4[iu, :, ju, :]


def pair_index(L, i, j):
    """Index of block (i < j) among the L (L - 1) / 2 tri blocks."""
    return i * L - i * (i + 1) // 2 + (j - i - 1)


def exact_site_block(codes, w, A, q, i):
    """g_h(i, .) and f_i(i, .) by bincount."""
    c = codes[:, i].astype(np.int64)
    m = c < q
    fi = np.bincount(c[m], weights=np.asarray(w, dtype=np.float64)[m], minlength=q)
    return probabilities(A)[i] * fi.sum() - fi, fi


def exact_pair_block(codes, w, A, q, i, j):
    """g_J(i, j) (q, q) and F_ij (q, q) for i < j by bincount: the sampled-block restatement for large shapes."""
    ci, cj = codes[:, i].astype(np.int64), codes[:, j].astype(np.int64)
    m = (ci < q) & (cj < q)
    F = np.bincount(ci[m] * q + cj[m], weights=np.asarray(w, dtype=np.float64)[m], minlength=q * q).reshape(q, q)
    P = probabilities(A)
    g = P[i][:, None] * F.sum(axis=0)[None, :] + F.sum(axis=1)[:, None] * P[j][None, :] - 2 * F
    return g, F


def negloglk(case):
    """-loglk in the log-sum-exp form (po.objective, float64; without a regulariser fx is the same number); finite
    where the observed state is not in A_i."""
    fx, _g, nll = po.objective(case["x"].astype(np.float64), case["codes"], case["w"].astype(np.float64), case["q"],
                               0.0, 0.0, case["gap_code"])
    return nll


# (N, L, q, gap, amax, wk, we)
CPU_CASES = [
    (40, 5, 2, False, 2, 3, 2),
    (60, 6, 4, True, 4, 5, 3),
    (60, 6, 4, False, 4, 7, 3),
    (50, 5, 5, False, 4, 3, 1),
    (60, 6, 20, True, 16, 3, 3),
    (50, 6, 21, False, 16, 7, 3),
    (45, 4, 21, False, 8, 1, 0),
    (40, 5, 32, False, 16, 3, 2),
]
C_PORT_Q = (4, 5, 20, 21)


@pytest.mark.parametrize("N,L,q,gap,amax,wk,we", CPU_CASES)
def test_closed_form_is_the_loops_oracle_and_the_c_fp32_port(N, L, q, gap, amax, wk, we):
    case = dyadic_case(N, L, q, gap, seed=N + L + q, amax=amax, wk=wk, we=we, zero_w=0.1)
    codes, w, x, A = case["codes"], case["w"], case["x"], case["A"]
    want = exact_gradient(codes, w, A, q)
    assert np.array_equal(want / case["u"], np.round(want / case["u"])), "not a multiple of u"
    with np.errstate(divide="ignore", invalid="ignore"):
        fx, g, nll = po.objective_loops(x.astype(np.float64), codes, w.astype(np.float64), q, 0.0, 0.0,
                                        case["gap_code"])
    assert np.array_equal(g, want), np.abs(g - want).max()
    # an observed state outside A_i: log 0 in the loops oracle (times a zero weight: NaN)
    outside = [(n, i) for n in range(N) for i in range(L) if codes[n, i] < q and not A[i, codes[n, i]]]
    assert np.isfinite(fx) != bool(outside)
    if q in C_PORT_Q:
        with np.errstate(divide="ignore", invalid="ignore"):
            _f, g32, _n = co.plm_eval(codes, w, x, q, 0.0, 0.0, "f32")
        assert np.array_equal(g32.astype(np.float64), want), np.abs(g32 - want).max()
    fi, fij = exact_counts(codes, w, q)
    iu, ju = np.triu_indices(L, 1)
    for p in range(len(iu)):
        gb, Fb = exact_pair_block(codes, w, A, q, iu[p], ju[p])
        assert np.array_equal(gb, want[L * q:].reshape(-1, q, q)[p]) and np.array_equal(Fb, fij[p])
    for i in range(L):
        gb, fb = exact_site_block(codes, w, A, q, i)
        assert np.array_equal(gb, want[:L * q].reshape(L, q)[i]) and np.array_equal(fb, fi[i])
    # the lse form's -loglk is finite; its gradient is within an ulp of the exact one, not equal to it
    nll_lse = negloglk(case)
    assert np.isfinite(nll_lse)
    print("\nN=%d L=%d q=%d%s |A| %s: budget 2 sum(w) / u = %.3g, exact (loops%s), -loglk %.6g"
          % (N, L, q, " (gap ignored)" if gap else "", sorted(set(case["asize"].tolist())), case["budget"],
             ", C fp32 port" if q in C_PORT_Q else "", nll_lse))


def test_logits_on_the_a_sets_are_zero():
    """The premise: whatever the sequence, the logits on A_i are 0 and the others at most -1048, so P is 1/|A_i|."""
    case = dyadic_case(300, 40, 21, seed=3, amax=16)
    L, q = 40, 21
    h, Jt = po.unpack(case["x"].astype(np.float64), L, q)
    W = po.full_couplings(Jt, L, q).transpose(1, 3, 0, 2).reshape(L * q, L * q)
    Z = (one_hot(case["codes"], q) @ W).reshape(-1, L, q) + h[None]
    A = case["A"]
    assert (Z[:, A] == 0).all()
    assert Z[:, ~A].max() <= H_OUT + 1000
    assert np.abs(Jt).max() * L <= 1000


def test_zero_weights_avoid_the_edges_and_outside_states_stay_out():
    case = dyadic_case(4097, 6, 21, seed=2, zero_w=0.5, outside=((0, 0), (1, 0), (5, 20)))
    n = np.flatnonzero(case["w"] == 0)
    assert len(n) > 1000 and not ((n % 64 == 0) | (n % 64 == 63) | (n == 4096)).any()
    A = case["A"]
    assert not A[0, 0] and not A[1, 0] and not A[5, 20]
    assert set(A.sum(axis=1).tolist()) <= set(A_SIZES)


def test_regulariser_budget_includes_two_lambda_x():
    case = dyadic_case(100, 10, 21, seed=1, lam=(0.125, 0.09375))
    assert case["u"] == lsb(2 * 0.09375) / 64
    with pytest.raises(AssertionError):
        dyadic_case(200000, 10, 21, seed=1, wk=4)          # 2 sum(w) / u > 2^22


# ------------------------------------------------------------------------------------------------
# the blind spot of a tolerance: one-sequence slips at N = 100k
# ------------------------------------------------------------------------------------------------
def test_one_sequence_slips_change_the_exact_gradient():
    N, L, q = 100_000, 20, 21
    case = dyadic_case(N, L, q, seed=11, amax=8, wk=1)
    codes, w, A = case["codes"], case["w"], case["A"]
    g0 = exact_gradient(codes, w, A, q)
    k = 1001                                       # a 64-sequence K block in the middle
    slips = {
        "drop the last sequence": (codes[:-1], w[:-1]),
        "drop one sequence in the middle": (np.delete(codes, N // 2, 0), np.delete(w, N // 2)),
        "drop one 64-sequence K block": (np.delete(codes, np.s_[64 * k:64 * k + 64], 0),
                                         np.delete(w, np.s_[64 * k:64 * k + 64])),
        "one stale row (a sequence counted twice)": (np.concatenate([codes, codes[N - 769:N - 768]]),
                                                     np.concatenate([w, w[N - 769:N - 768]])),
    }
    n0 = np.linalg.norm(g0)
    print("\nN=%d L=%d q=%d, w = 1, budget %.3g: relative L2 change of the exact gradient (VEC_REL = %.0e)"
          % (N, L, q, case["budget"], VEC_REL))
    for name, (c, ww) in slips.items():
        g = exact_gradient(c, ww, A, q)
        d = g - g0
        rel = np.linalg.norm(d) / n0
        print("  %-42s %.2e = %.1f VEC_REL  (%d entries change, largest by %d u)"
              % (name, rel, rel / VEC_REL, int((d != 0).sum()), int(np.abs(d).max() / case["u"])))
        assert (d != 0).any(), name
