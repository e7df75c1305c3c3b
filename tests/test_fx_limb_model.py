"""
Python-integer model of the -loglk limb transport (evc_plm_pack_fx / evc_plm_unpack_fx, include/evcplm.h), checked here
against fractions.Fraction and against float32 sums in numpy, so that the reference tests/test_gpu_ranks_one_device.py
compares the device with is itself tested where there is no GPU.

    Q(v)      = round-half-even(v * 2^16)                           the integer a rank transports
    split(q)  = (q mod 2^18, (q >> 18) mod 2^18, q >> 36)           three limbs, the top one signed (floor shift)
    decode(s) = (s0 + s1 * 2^18 + s2 * 2^36) / 2^16                 from the limb sums over the ranks
"""
from fractions import Fraction

import numpy as np

LIMB_BITS = 18
MASK = (1 << LIMB_BITS) - 1
SCALE = 1 << 16
Q_LIMIT = 9 * 10 ** 15              # |Q(v)| <= Q_LIMIT is carried; beyond it the device flags the 4th float with NaN
MAX_RANKS = 64


def Q(v):
    """round-half-even(v * 2^16) as a Python integer (v: a finite double; v * 2^16 is exact in binary)."""
    return round(Fraction(float(v)) * SCALE)


def in_contract(v):
    return np.isfinite(v) and abs(Fraction(float(v)) * SCALE) <= Q_LIMIT


def split(q):
    return q & MASK, (q >> LIMB_BITS) & MASK, q >> (2 * LIMB_BITS)


def join(limbs):
    return int(limbs[0]) + (int(limbs[1]) << LIMB_BITS) + int(limbs[2]) * (1 << (2 * LIMB_BITS))


def decode(limb_sums):
    """The double the device returns for these limb sums: the integer, rounded to nearest even if it needs more than
    53 bits, over 2^16 (Python's int / int is the correctly rounded quotient, and a division by 2^16 is exact)."""
    return join(limb_sums) / SCALE


def transported(values):
    """What every rank decodes when rank r contributes values[r]."""
    return sum(Q(v) for v in values) / SCALE


def sum_orders(R, seed):
    """Index sequences for a rank-order, a reversed and a permuted running sum; the pairwise tree is sum_tree."""
    return {"rank": list(range(R)), "reversed": list(range(R))[::-1],
            "permuted": [int(i) for i in np.random.default_rng(seed).permutation(R)]}


def sum_tree(items, add):
    items = list(items)
    while len(items) > 1:
        items = [add(items[i], items[i + 1]) if i + 1 < len(items) else items[i] for i in range(0, len(items), 2)]
    return items[0]


def edge_values():
    """Single values at the edges of the limb split (the ties, each limb at 0 and at 2^18 - 1, the sign)."""
    e = 2.0 ** -17
    vals = [0.0, e, -e, 3 * e, -3 * e, 2 * e, -2 * e, 1 - 2 * e, -1.0, 1.3e11, -1.3e11]
    for q in (MASK, MASK << LIMB_BITS, (MASK << LIMB_BITS) | MASK, 1 << LIMB_BITS, 1 << (2 * LIMB_BITS),
              (1 << (2 * LIMB_BITS)) - 1, -(1 << LIMB_BITS), -(1 << (2 * LIMB_BITS)), -((1 << (2 * LIMB_BITS)) + 1),
              Q_LIMIT, -Q_LIMIT, (130966 << (2 * LIMB_BITS)) | ((1 << (2 * LIMB_BITS)) - 1)):
        vals.append(q / SCALE)
    return vals


def seeded_values(count, seed):
    """log-uniform in [1e-3, 1e11], both signs"""
    rng = np.random.default_rng(seed)
    return [float(s * 10.0 ** p) for s, p in zip(rng.choice([-1.0, 1.0], count), rng.uniform(-3, 11, count))]


# ---- the model against Fraction and float32 -------------------------------------------------------------------------
def test_Q_rounds_half_to_even():
    e = Fraction(1, 1 << 17)
    assert [Q(float(k * e)) for k in (1, -1, 3, -3, 5, 2, -2)] == [0, 0, 2, -2, 2, 1, -1]
    assert Q(1 - 2.0 ** -16) == SCALE - 1 and Q(-1.0) == -SCALE
    for v in seeded_values(200, 1):
        exact = Fraction(v) * SCALE
        assert abs(Q(v) - exact) <= Fraction(1, 2)
        assert Q(-v) == -Q(v)


def test_split_ranges_and_join():
    assert split(-1) == (MASK, MASK, -1)             # what a logical shift of the top limb would break
    assert split(Q(-1.0)) == ((1 << 18) - SCALE, MASK, -1) and join(split(Q(-1.0))) == -SCALE
    for v in edge_values() + seeded_values(200, 2):
        assert in_contract(v)
        q = Q(v)
        l0, l1, l2 = split(q)
        assert 0 <= l0 <= MASK and 0 <= l1 <= MASK and abs(l2) < (1 << 17)
        assert join((l0, l1, l2)) == q
        assert all(float(np.float32(l)) == l for l in (l0, l1, l2))        # each limb is a float32 integer
        assert decode((l0, l1, l2)) == float(Fraction(q, SCALE))


def test_float32_sums_of_64_ranks_are_exact_in_any_order():
    rng = np.random.default_rng(3)
    worst = [(MASK, MASK, (1 << 17) - 1)] * MAX_RANKS
    mixed = [split(Q(v)) for v in seeded_values(MAX_RANKS, 4)]
    for limbs in (worst, [(a, b, -c) for a, b, c in worst], mixed):
        want = [sum(l[k] for l in limbs) for k in range(3)]
        assert max(abs(w) for w in want) <= (1 << 24) - MAX_RANKS
        arr = np.array(limbs, dtype=np.float32)
        for order in list(sum_orders(MAX_RANKS, 5).values()) + [list(rng.permutation(MAX_RANKS))]:
            acc = np.zeros(3, dtype=np.float32)
            for r in order:
                acc = acc + arr[r]
            assert [int(a) for a in acc] == want
        tree = sum_tree([arr[r] for r in range(MAX_RANKS)], lambda a, b: a + b)
        assert tree.dtype == np.float32 and [int(a) for a in tree] == want
        assert decode(want) == float(Fraction(join(want), SCALE))


def test_transported_value_is_the_sum_of_the_quantised_terms():
    for R in (2, 3, 8, 64):
        vals = seeded_values(R, 10 + R)
        sums = [sum(split(Q(v))[k] for v in vals) for k in range(3)]
        assert decode(sums) == transported(vals) == float(Fraction(sum(Q(v) for v in vals), SCALE))
        assert abs(Fraction(transported(vals)) - sum(Fraction(v) for v in vals)) <= Fraction(R, 1 << 17) + \
            abs(Fraction(transported(vals))) * Fraction(1, 1 << 52)
    vals = seeded_values(32, 20)
    assert transported(vals + [-v for v in vals]) == 0.0
    assert not in_contract(2e11) and not in_contract(float("nan")) and not in_contract(float("inf"))
