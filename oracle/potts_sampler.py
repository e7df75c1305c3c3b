"""
CPU restatement of the library's Gibbs sampler (evc_sampler_*, contract in include/evcplm.h), in numpy float64 and
vectorised over chains: the same target, the same systematic scan, the same draw rule and the same counter-based
uniforms, so a chain here follows the device chain draw for draw until a draw whose outcome the device's fp32
arithmetic could decide differently (a near-tie, see near_tie_margin).  Also the exact distribution of small models by
enumeration.  Test infrastructure, not product code.
"""
import numpy as np

PHI = np.uint64(0x9E3779B97F4A7C15)
REFRESH = 32                    # EVC_SAMPLER_REFRESH
EPS32 = 2.0 ** -24              # unit roundoff of fp32


def mix(z):
    """splitmix64's finaliser on uint64 arrays (wrapping arithmetic)."""
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def chain_key(seed, c):
    """key(c) = mix(seed ^ mix((c + 1) phi)), c the global chain index (array)."""
    c = np.asarray(c, dtype=np.uint64)
    with np.errstate(over="ignore"):
        return mix(np.uint64(seed) ^ mix((c + np.uint64(1)) * PHI))


def uniform(key, t, i, L):
    """u(c, t, i) = ((mix(key + k phi) >> 40) + 0.5) 2^-24, k = (t L + i + 1) mod 2^64 (float64, exact)."""
    k = np.uint64((int(t) * int(L) + int(i) + 1) % (1 << 64))
    with np.errstate(over="ignore"):
        d = mix(np.asarray(key, dtype=np.uint64) + k * PHI) >> np.uint64(40)
    return (d.astype(np.float64) + 0.5) * 2.0 ** -24


def full_couplings(J, L, q):
    """(L, q, L, q) float64: U[i, a, j, b] = J_ij(a, b) from the packed (L(L-1)/2, q, q) blocks, zero for i == j."""
    U = np.zeros((L, q, L, q))
    iu, ju = np.triu_indices(L, 1)
    Jt = np.asarray(J, dtype=np.float64).reshape(-1, q, q)
    U[iu, :, ju, :] = Jt
    U[ju, :, iu, :] = Jt.transpose(0, 2, 1)
    return U


def energies(h, J, codes):
    """H(s) = sum_i h_i(s_i) + sum_{i<j} J_ij(s_i, s_j) for every row of codes (float64)."""
    codes = np.asarray(codes, dtype=np.int64)
    L = codes.shape[1]
    h = np.asarray(h, dtype=np.float64)
    q = h.shape[1]
    Jt = np.asarray(J, dtype=np.float64).reshape(-1, q, q)
    iu, ju = np.triu_indices(L, 1)
    E = h[np.arange(L), codes].sum(axis=1)
    return E + Jt[np.arange(len(iu)), codes[:, iu], codes[:, ju]].sum(axis=1)


def exact_distribution(h, J, beta, L, q):
    """P(s) over all q^L states, index = sum_i s_i q^(L-1-i) (the row-major order of the codes)."""
    if q ** L > 4096:
        raise ValueError("enumeration is for q^L <= 4096")
    states = np.array(np.unravel_index(np.arange(q ** L), (q,) * L)).T
    logp = beta * energies(h, J, states)
    p = np.exp(logp - logp.max())
    return p / p.sum()


def state_index(codes, q):
    codes = np.asarray(codes, dtype=np.int64)
    return codes @ (q ** np.arange(codes.shape[1] - 1, -1, -1))


def uniform_start(seed, n_chains, L, q, chain_offset=0):
    """t = -1: s_i = floor(u q)."""
    key = chain_key(seed, np.arange(chain_offset, chain_offset + n_chains))
    return np.stack([np.floor(uniform(key, -1, i, L) * q) for i in range(L)], axis=1).astype(np.int64)


def near_tie_margin(q, z_error=0.0, beta=1.0, z_bound=0.0):
    """Half-width, on the normalised cumulative F_a = c_a / c_{q-1}, of the band in which the device's fp32 draw can
    end on another state than this float64 restatement.

    With eps = 2^-24 (fp32 unit roundoff):
      * Z_i(a) is off by at most z_error (see z_error_bound);
      * v = beta Z in fp32 adds eps |beta| z_bound, and v - m another 2 eps |beta| z_bound (|v - m| <= 2 |beta| z_bound),
        so the exponent of p_a is off by at most eta = 2 |beta| z_error + 3 eps |beta| z_bound (m is itself one of the
        v and carries at most the same error, hence the factor 2);
      * expf is within 2 ulp: relative 2^-22 at most;
      * the inclusive prefix sum of q positive terms: relative (q - 1) eps;
    so every c_a is within the relative error rho = (e^eta - 1) + 2^-22 + (q - 1) eps, and F_a within 2 rho.  The
    comparison u c_{q-1} < c_a is exact on the device (double).  The margin is twice that bound."""
    eta = 2.0 * abs(beta) * z_error + 3.0 * EPS32 * abs(beta) * z_bound
    rho = np.expm1(eta) + 2.0 ** -22 + (q - 1) * EPS32
    return 2.0 * (2.0 * rho)


def z_bound(h, J, L, q):
    """B = max_{i,a} |h_i(a)| + sum_{j != i} max_b |J_ij(a, b)|: no field value or partial sum of one exceeds it."""
    return float(site_z_bounds(h, J, L, q).max())


def site_z_bounds(h, J, L, q):
    """B_i = max_a |h_i(a)| + sum_{j != i} max_b |J_ij(a, b)| per site (float64, length L): the bound of z_bound for
    the values the draw at site i forms.  near_tie_margin's derivation holds per site with B_i in place of B."""
    U = np.abs(full_couplings(J, L, q))
    return (np.abs(np.asarray(h, dtype=np.float64)) + U.max(axis=3).sum(axis=2)).max(axis=1)


def is_dyadic(h, J, bits):
    """Every parameter is a multiple of 2^-bits."""
    v = np.concatenate([np.ravel(h), np.ravel(J)]).astype(np.float64) * 2.0 ** bits
    return bool(np.all(v == np.round(v)))


def z_error_bound(h, J, L, q, bits=None):
    """Largest error of the device's fp32 Z_i(a) over one refresh interval of REFRESH sweeps.

    The refresh sums L + 1 terms of magnitude sum <= B (z_bound) in fp32: error <= L eps B.  Each later change of a
    site adds one difference of two couplings: z + (U_b - U_a), two roundings, error <= eps (2 Jmax + B + 2 Jmax); an
    interval has at most REFRESH * L changes.  Total: eps (L B + REFRESH L (B + 4 Jmax)).

    When every parameter is a multiple of 2^-bits and B < 2^(24 - bits), every value the device forms (each U
    entry, each U_b - U_a, each partial sum) is a multiple of 2^-bits below 2^(24 - bits) in magnitude, so it has
    at most 24 significant bits and fp32 holds it exactly: the bound is 0 and Z is exact."""
    B = z_bound(h, J, L, q)
    if bits is not None and is_dyadic(h, J, bits) and B < 2.0 ** (23 - bits):
        return 0.0
    Jmax = float(np.abs(np.asarray(J, dtype=np.float64)).max(initial=0.0))
    return EPS32 * (L * B + REFRESH * L * (B + 4.0 * Jmax))


class Sampler(object):
    """The chain of evc_sampler_* for n_chains chains with global indices chain_offset + 0..n_chains-1.

    ``margin``: the near-tie half-width (near_tie_margin), one for every site or one per site; ``first_tie`` then
    holds, per chain, the global draw number t L + i of its first near-tie draw (-1: none yet).  ``changes`` counts
    site changes of the last run()."""

    def __init__(self, h, J, seed, n_chains, init=None, chain_offset=0, margin=0.0):
        self.h = np.asarray(h, dtype=np.float64)
        self.L, self.q = self.h.shape
        self.U = full_couplings(J, self.L, self.q)
        self._start(seed, n_chains, init, chain_offset, margin)

    def _start(self, seed, n_chains, init, chain_offset, margin):
        self.key = chain_key(seed, np.arange(chain_offset, chain_offset + n_chains))
        if init is None:
            self.s = uniform_start(seed, n_chains, self.L, self.q, chain_offset)
        else:
            self.s = np.array(init, dtype=np.int64).reshape(n_chains, self.L)
        self.t = 0
        self.margin = np.broadcast_to(np.asarray(margin, dtype=np.float64), (self.L,))
        self.first_tie = np.full(n_chains, -1, dtype=np.int64)
        self.changes = 0

    def _draw(self, i, Z, beta):
        """The draw at site i of every chain from Z (q, C) in float64; records near-ties.  Returns the new codes."""
        q, L = self.q, self.L
        v = beta * Z
        p = np.exp(v - v.max(axis=0))
        c = np.cumsum(p, axis=0)
        thr = uniform(self.key, self.t, i, L) * c[-1]
        hit = thr[None, :] < c
        b = np.where(hit.any(axis=0), hit.argmax(axis=0), q - 1)
        if self.margin[i] > 0:
            tie = (np.abs(thr[None, :] - c[:-1]) <= self.margin[i] * c[-1]).any(axis=0)
            new = tie & (self.first_tie < 0)
            self.first_tie[new] = self.t * L + i
        self.changes += int((b != self.s[:, i]).sum())
        return b

    def run(self, sweeps, beta=1.0):
        L, q = self.L, self.q
        C = self.s.shape[0]
        rows = np.arange(C)
        Uf = self.U.reshape(L * q, L * q)
        cols = [np.ascontiguousarray(Uf[:, i * q:(i + 1) * q]) for i in range(L)]
        X = np.zeros((C, L * q))                # one-hot of the states: Z_i = X U[:, (i, .)] + h_i
        X[rows[:, None], np.arange(L) * q + self.s] = 1.0
        self.changes = 0
        for _ in range(sweeps):
            for i in range(L):
                Z = (X @ cols[i]).T + self.h[i][:, None]      # (q, C)
                b = self._draw(i, Z, beta)
                X[rows, i * q + self.s[:, i]] = 0.0
                X[rows, i * q + b] = 1.0
                self.s[:, i] = b
            self.t += 1
        return self.changes

    def codes(self):
        return self.s.astype(np.uint8)


def sparse_neighbours(L, q, pairs, blocks):
    """Per site i: (j, M) with j the sites coupled to i (ascending) and M[k, b, a] = J_{i j_k}(a, b), from pair blocks
    J_ij(a, b) of pairs i < j (every pair not listed has J_ij = 0)."""
    pairs = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    blocks = np.asarray(blocks, dtype=np.float64).reshape(-1, q, q)
    if len(pairs) and not (np.all(pairs[:, 0] < pairs[:, 1]) and pairs.min() >= 0 and pairs.max() < L):
        raise ValueError("pairs must be 0 <= i < j < L")
    if len(np.unique(pairs[:, 0] * L + pairs[:, 1])) != len(pairs):
        raise ValueError("a pair is listed twice")
    site = np.concatenate([pairs[:, 0], pairs[:, 1]])
    other = np.concatenate([pairs[:, 1], pairs[:, 0]])
    # at i (the first site) M[b, a] = J(a, b); at j (the second) M[a, b'] with a the state of i: J(a, b') = J^T
    Ms = np.concatenate([blocks.transpose(0, 2, 1), blocks])
    order = np.lexsort((other, site))
    site, other, Ms = site[order], other[order], Ms[order]
    bounds = np.searchsorted(site, np.arange(L + 1))
    return [(other[bounds[i]:bounds[i + 1]], Ms[bounds[i]:bounds[i + 1]]) for i in range(L)]


def sparse_site_z_bounds(h, L, q, pairs, blocks):
    """site_z_bounds of a model whose couplings are the pair blocks of SparseSampler."""
    h = np.abs(np.asarray(h, dtype=np.float64).reshape(L, q))
    # M[k, b, a]: max over b is the max over the other site's state
    return np.array([(h[i] + np.abs(M).max(axis=1).sum(axis=0)).max() for i, (_, M) in
                     enumerate(sparse_neighbours(L, q, pairs, blocks))])


class SparseSampler(Sampler):
    """Sampler for a model whose couplings are nonzero only in the pair blocks ``blocks[k] = J_ij`` of ``pairs[k] =
    (i, j)``, i < j: the same counters, draw rule and near-tie bookkeeping, with Z_i(a) = h_i(a) + sum over the
    neighbours j of J_ij(a, s_j) formed in float64 from the neighbours only, so no (L q)^2 matrix is built.  The
    margin is best given per site (near_tie_margin with sparse_site_z_bounds).  ``z_seen[i]`` is the largest
    |Z_i(a)| the chains formed at site i over all run() calls."""

    def __init__(self, h, pairs, blocks, seed, n_chains, init=None, chain_offset=0, margin=0.0):
        self.h = np.asarray(h, dtype=np.float64)
        self.L, self.q = self.h.shape
        self.nbr = sparse_neighbours(self.L, self.q, pairs, blocks)
        self.z_seen = np.zeros(self.L)
        self._start(seed, n_chains, init, chain_offset, margin)

    def run(self, sweeps, beta=1.0):
        self.changes = 0
        for _ in range(sweeps):
            for i in range(self.L):
                j, M = self.nbr[i]
                Z = self.h[i][:, None] + M[np.arange(len(j)), self.s[:, j]].sum(axis=1).T     # (q, C)
                self.z_seen[i] = max(self.z_seen[i], float(np.abs(Z).max()))
                self.s[:, i] = self._draw(i, Z, beta)
            self.t += 1
        return self.changes
