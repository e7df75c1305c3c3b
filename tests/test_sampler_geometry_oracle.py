"""The sparse restatement of the Gibbs chain (oracle/potts_sampler.py SparseSampler) against the dense one, its per-site
bounds, and the models and comparison power of the sampler's launch-geometry checks on the device
(tests/test_gpu_consumer_geometry.py): the share of chain-sweeps those checks compare is a property of the
restatement alone, so it is fixed here, on the CPU."""
import numpy as np
import pytest

from oracle import potts_sampler as ps


def dyadic(rng, scale, shape):
    """N(0, scale) rounded to multiples of 2^-10."""
    return np.round(rng.normal(0, scale, shape) * 1024) / 1024


def pair_index(i, j, L):
    """Position of pair i < j in the row-major list of pairs (arrays)."""
    i, j = np.asarray(i, dtype=np.int64), np.asarray(j, dtype=np.int64)
    return i * (2 * L - i - 1) // 2 + (j - i - 1)


def sparse_model(L, q, pairs, seed, j_scale=0.05):
    """Fields N(0, 0.5) and the listed coupling blocks N(0, j_scale), all multiples of 2^-10; pairs sorted, i < j."""
    rng = np.random.default_rng(seed)
    pairs = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    pairs = pairs[np.argsort(pair_index(pairs[:, 0], pairs[:, 1], L))]
    return dyadic(rng, 0.5, (L, q)), pairs, dyadic(rng, j_scale, (len(pairs), q, q))


def dense_J(L, q, pairs, blocks):
    J = np.zeros((L * (L - 1) // 2, q, q))
    J[pair_index(pairs[:, 0], pairs[:, 1], L)] = blocks
    return J


def random_pairs(L, n, seed):
    """The path (i, i + 1) plus n random distinct pairs."""
    rng = np.random.default_rng(seed)
    i = rng.integers(0, L, 4 * n)
    j = rng.integers(0, L, 4 * n)
    keep = i != j
    p = np.stack([np.minimum(i, j), np.maximum(i, j)], axis=1)[keep]
    p = np.unique(p, axis=0)[:n]
    path = np.stack([np.arange(L - 1), np.arange(1, L)], axis=1)
    return np.unique(np.concatenate([path, p]), axis=0)


def star_pairs(L, T):
    """Every pair of a site in T with every other site."""
    out = {(min(t, j), max(t, j)) for t in T for j in range(L) if j != t}
    return np.array(sorted(out), dtype=np.int64)


# ---- the sampler's launch geometries (row_bytes = round_up(4 L q + L, 16), min(16, 232448 / row_bytes) chains per CTA)

def chains_per_cta(L, q):
    row_bytes = -(-(4 * L * q + L) // 16) * 16
    return min(16, 232448 // row_bytes)


# 13 chains per CTA at L = 200, q = 21, the last of 20 CTAs holding 5; a dense model; 40 sweeps cross the refresh
CTA13 = dict(L=200, q=21, n=13 * 19 + 5, sweeps=40, seed=31, beta=1.0)
# 2 chains per CTA at L = 5000, q = 4, the last CTA holding one; the path of couplings plus 5000 random pairs
CTA2 = dict(L=5000, q=4, n=2 * 40 + 1, sweeps=40, seed=32, beta=1.0)
# one chain per CTA at L = 2300, q = 21: (L q)^2 = 2.33e9 > 2^31 entries of U.  J is nonzero only in the blocks of six
# test sites against every other site, the last three among them.
FAR = dict(L=2300, q=21, n=96, sweeps=4, seed=33, beta=1.0)
FAR_SITES = (0, 1, 1150, 2297, 2298, 2299)

# The least share of chain-sweeps each case compares draw for draw (clean so far).  The restatement alone reaches
# 0.337 (CTA13, 33 chains clean past the refresh), 0.326 (CTA2, 7 chains past the refresh) and 0.185 (FAR) with these
# models, chains and sweeps (test_comparison_power).
POWER = dict(CTA13=0.30, CTA2=0.30, FAR=0.15)


def cta13_model():
    L, q = CTA13["L"], CTA13["q"]
    iu, ju = np.triu_indices(L, 1)
    # weak couplings: a small B keeps the margin, and so the near-ties, near their floor (q - 1) 2^-24 + 2^-22
    return sparse_model(L, q, np.stack([iu, ju], axis=1), 200, j_scale=0.005)


def cta2_model():
    L, q = CTA2["L"], CTA2["q"]
    return sparse_model(L, q, random_pairs(L, L, 5), 201)


def far_model():
    L, q = FAR["L"], FAR["q"]
    return sparse_model(L, q, star_pairs(L, FAR_SITES), 202)


def margins(h, pairs, blocks, beta):
    """Per-site near-tie margins of a dyadic model (Z exact on the device: z_error = 0)."""
    L, q = h.shape
    B = ps.sparse_site_z_bounds(h, L, q, pairs, blocks)
    assert ps.is_dyadic(h, blocks, 10) and B.max() < 2.0 ** 13
    return ps.near_tie_margin(q, 0.0, beta, B)


def restatement(case, model):
    h, pairs, blocks = model
    L, q = h.shape
    m = margins(h, pairs, blocks, case["beta"])
    if case is CTA13:
        return ps.Sampler(h, dense_J(L, q, pairs, blocks), case["seed"], case["n"], margin=m)
    return ps.SparseSampler(h, pairs, blocks, case["seed"], case["n"], margin=m)


def clean_after(ref, t):
    """Chains with no near-tie draw up to the end of sweep t (0-based)."""
    return (ref.first_tie < 0) | (ref.first_tie >= (t + 1) * ref.L)


# ---- the sparse restatement against the dense one ------------------------------------------------------------------

@pytest.mark.parametrize("beta", [0.5, 1.0])
@pytest.mark.parametrize("q", [2, 21, 32])
@pytest.mark.parametrize("L", [12, 40])
def test_sparse_restatement_equals_dense(L, q, beta):
    """Code for code, with the same first_tie and change counts, over split runs and chain offsets; the couplings
    of a few sites are strong so that their per-site margins differ from the others'."""
    rng = np.random.default_rng(L * 100 + q)
    pairs = random_pairs(L, L, 3 * L + q)
    h, pairs, blocks = sparse_model(L, q, pairs, L + q)
    blocks[pairs[:, 0] == 1] *= 8                     # site 1 couples strongly
    J = dense_J(L, q, pairs, blocks)
    B = ps.sparse_site_z_bounds(h, L, q, pairs, blocks)
    assert np.array_equal(B, ps.site_z_bounds(h, J, L, q)) and B.max() == ps.z_bound(h, J, L, q)
    # margins scaled up from the device's so that about half of the chains meet a near-tie in 9 sweeps
    m = ps.near_tie_margin(q, 0.0, beta, B)
    scale = 0.04 / (L * (q - 1) * np.median(m))
    m = scale * m
    n, seed = 200, int(rng.integers(1 << 62))
    dense = ps.Sampler(h, J, seed, n, margin=m)
    ch_dense = dense.run(9, beta)
    sparse = ps.SparseSampler(h, pairs, blocks, seed, n, margin=m)
    ch_sparse = sparse.run(4, beta) + sparse.run(5, beta)
    assert np.array_equal(sparse.codes(), dense.codes())
    assert np.array_equal(sparse.first_tie, dense.first_tie) and ch_sparse == ch_dense
    assert (dense.first_tie >= 0).any() and (dense.first_tie < 0).any()
    tail = ps.SparseSampler(h, pairs, blocks, seed, n - 77, chain_offset=77, margin=m)
    tail.run(9, beta)
    assert np.array_equal(tail.codes(), dense.codes()[77:]) and np.array_equal(tail.first_tie, dense.first_tie[77:])
    # one global margin: the dense restatement's scalar form
    g = scale * ps.near_tie_margin(q, 0.0, beta, ps.z_bound(h, J, L, q))
    a, b = ps.Sampler(h, J, seed, n, margin=g), ps.SparseSampler(h, pairs, blocks, seed, n, margin=g)
    a.run(3, beta)
    b.run(3, beta)
    assert np.array_equal(a.first_tie, b.first_tie) and np.array_equal(a.codes(), b.codes())
    # a run from given codes
    init = rng.integers(0, q, (5, L))
    a, b = ps.Sampler(h, J, seed, 5, init=init), ps.SparseSampler(h, pairs, blocks, seed, 5, init=init)
    assert a.run(3, beta) == b.run(3, beta) and np.array_equal(a.codes(), b.codes())


@pytest.mark.parametrize("L,q", [(12, 2), (40, 21), (40, 32)])
def test_site_bounds_cover_every_field_seen(L, q):
    h, pairs, blocks = sparse_model(L, q, random_pairs(L, 2 * L, L), 7)
    blocks[pairs[:, 1] == L - 1] *= 16
    s = ps.SparseSampler(h, pairs, blocks, 3, 300)
    s.run(6)
    B = ps.sparse_site_z_bounds(h, L, q, pairs, blocks)
    assert (s.z_seen <= B).all() and (s.z_seen > 0).all()
    assert B.max() > 2 * np.median(B)                 # the bound differs between sites


def test_sparse_neighbours_refuses_bad_pairs():
    blk = np.zeros((1, 3, 3))
    for bad in ([[2, 1]], [[0, 5]], [[-1, 2]]):
        with pytest.raises(ValueError, match="0 <= i < j < L"):
            ps.sparse_neighbours(5, 3, bad, blk)
    with pytest.raises(ValueError, match="twice"):
        ps.sparse_neighbours(5, 3, [[0, 1], [0, 1]], np.zeros((2, 3, 3)))


# ---- the device cases: geometry and power --------------------------------------------------------------------------

def test_geometry_of_the_device_cases():
    assert chains_per_cta(CTA13["L"], CTA13["q"]) == 13 and CTA13["n"] % 13 == 5
    assert chains_per_cta(CTA2["L"], CTA2["q"]) == 2 and CTA2["n"] % 2 == 1
    assert chains_per_cta(FAR["L"], FAR["q"]) == 1 and (FAR["L"] * FAR["q"]) ** 2 > 2 ** 31
    # the rows of the last three sites start beyond entry 2^31 of U
    assert all(i * FAR["q"] * FAR["L"] * FAR["q"] > 2 ** 31 for i in FAR_SITES[-3:])
    assert CTA13["sweeps"] > ps.REFRESH and CTA2["sweeps"] > ps.REFRESH


@pytest.mark.parametrize("name", ["CTA13", "CTA2", "FAR"])
def test_comparison_power(name):
    """The share of chain-sweeps the device check compares, chains of the partial last CTA among them; past the
    refresh at t = 32 where the run crosses it; for FAR, changes of each of the last three sites in the compared
    prefix (their far rows of U were streamed)."""
    case = dict(CTA13=CTA13, CTA2=CTA2, FAR=FAR)[name]
    model = dict(CTA13=cta13_model, CTA2=cta2_model, FAR=far_model)[name]()
    ref = restatement(case, model)
    compared = np.zeros(case["n"], dtype=np.int64)          # compared sweeps per chain
    last = np.zeros(3, dtype=np.int64)
    for t in range(case["sweeps"]):
        before = ref.s[:, -3:].copy()
        ref.run(1, case["beta"])
        clean = clean_after(ref, t)
        compared += clean
        last += ((ref.s[:, -3:] != before) & clean[:, None]).sum(axis=0)
    frac = compared.sum() / (case["n"] * case["sweeps"])
    print("%s: compared %.3f of the chain-sweeps, %d chains past sweep 32, %.3f of the chains flagged, "
          "last-site changes %s" % (name, frac, (compared > ps.REFRESH).sum(), (ref.first_tie >= 0).mean(), last))
    assert frac >= POWER[name]
    per_cta = chains_per_cta(case["L"], case["q"])
    if per_cta > 1:                                         # the partial last CTA was compared
        assert (compared[-(case["n"] % per_cta):] > 0).all()
    if case["sweeps"] > ps.REFRESH:
        assert (compared > ps.REFRESH).sum() >= 3
    assert (last > 0).all()
