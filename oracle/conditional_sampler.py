"""
CPU restatement of the library's conditional Gibbs sampler (evc_sampler_create_conditional, contract in
include/evcplm.h), in numpy float64 and vectorised over chains: the fold of each chain's context into the fields of the
free sites, the reduced couplings U_FF, the refresh-free float64 fields, the counters at the original site index and
the masked draw with its fallback, so a chain here follows the device chain draw for draw until a near tie
(potts_sampler.near_tie_margin over the free sites' fields).  Also the exact conditional distribution of the free
sites given a context, by enumeration.  Test infrastructure, not product code.
"""
import numpy as np

from oracle import potts_sampler as ps


def clamped_sites(L, free):
    free = set(int(k) for k in free)
    return np.array([j for j in range(L) if j not in free], dtype=np.int64)


def fold(h, J, free, init):
    """(C, nf, q) float64 hc[c, k, a] = h_{F_k}(a) + sum over clamped j ascending of J_{F_k j}(a, init[c, j])."""
    h = np.asarray(h, dtype=np.float64)
    L, q = h.shape
    free = np.asarray(free, dtype=np.int64)
    init = np.asarray(init, dtype=np.int64).reshape(-1, L)
    Uf = ps.full_couplings(J, L, q)[free]                       # (nf, q, L, q)
    hc = np.repeat(h[free][None], len(init), axis=0)
    for j in clamped_sites(L, free):
        hc += Uf[:, :, j, init[:, j]].transpose(2, 0, 1)
    return hc


def fold_sparse(h, pairs, blocks, free, init):
    """fold() of a model whose couplings are the pair blocks J_ij = blocks[k] of pairs[k] = (i, j), i < j (every other
    pair zero), without the (L q)^2 matrix."""
    h = np.asarray(h, dtype=np.float64)
    L, q = h.shape
    free = np.asarray(free, dtype=np.int64)
    slot = {int(k): n for n, k in enumerate(free)}
    init = np.asarray(init, dtype=np.int64).reshape(-1, L)
    hc = np.repeat(h[free][None], len(init), axis=0)
    for (i, j), B in zip(np.asarray(pairs).reshape(-1, 2), np.asarray(blocks, dtype=np.float64).reshape(-1, q, q)):
        i, j = int(i), int(j)
        if i in slot and j not in slot:
            hc[:, slot[i], :] += B[:, init[:, j]].T
        elif j in slot and i not in slot:
            hc[:, slot[j], :] += B[init[:, i], :]
    return hc


def reduced_couplings(J, L, q, free):
    """(nf q, nf q) float64 U_FF: U restricted to the free sites, zero diagonal blocks."""
    free = np.asarray(free, dtype=np.int64)
    U = ps.full_couplings(J, L, q)
    return U[free][:, :, free, :].reshape(len(free) * q, len(free) * q)


def reduced_couplings_sparse(L, q, pairs, blocks, free):
    """reduced_couplings() of the pair-block model of fold_sparse."""
    free = np.asarray(free, dtype=np.int64)
    slot = {int(k): n for n, k in enumerate(free)}
    U = np.zeros((len(free), q, len(free), q))
    for (i, j), B in zip(np.asarray(pairs).reshape(-1, 2), np.asarray(blocks, dtype=np.float64).reshape(-1, q, q)):
        if int(i) in slot and int(j) in slot:
            U[slot[int(i)], :, slot[int(j)], :] = B
            U[slot[int(j)], :, slot[int(i)], :] = B.T
    return U.reshape(len(free) * q, len(free) * q)


def reduced_z_bounds(hc, UFF, q):
    """B_k = max over chains and a of |hc| + sum_{k'} max_b |U_FF[(k, a), (k', b)]| per free site: the site_z_bounds
    of the reduced model, for near_tie_margin."""
    nf = hc.shape[1]
    U = np.abs(UFF).reshape(nf, q, nf, q)
    return (np.abs(hc).max(axis=0) + U.max(axis=3).sum(axis=2)).max(axis=1)


def full_masks(nf, q):
    return np.full(nf, (1 << q) - 1, dtype=np.int64)


class ConditionalSampler(object):
    """The chains of a conditional evc_sampler handle: the free sites ``free`` (ascending site indices of a model of
    L sites) with per-chain fields ``hc`` (C, nf, q), couplings ``UFF`` and allowed-state masks ``allowed`` (nf ints,
    None = every state); ``context`` (C, L) is each chain's start, whose clamped sites never change.  ``context`` None
    is the uniform start (only with nf = L).  ``margin``, ``first_tie`` and ``changes`` as in potts_sampler.Sampler,
    with the margin given per free site."""

    def __init__(self, hc, UFF, free, L, seed, allowed=None, context=None, chain_offset=0, margin=0.0):
        self.hc = np.asarray(hc, dtype=np.float64)
        C, nf, q = self.hc.shape
        self.L, self.q, self.free = int(L), q, np.asarray(free, dtype=np.int64)
        self.UFF = np.asarray(UFF, dtype=np.float64)
        self.allowed = full_masks(nf, q) if allowed is None else np.asarray(allowed, dtype=np.int64)
        self.ok = (self.allowed[:, None] >> np.arange(q)[None, :]) & 1 == 1        # (nf, q)
        self.highest = np.array([np.flatnonzero(r).max() for r in self.ok])
        self.key = ps.chain_key(seed, np.arange(chain_offset, chain_offset + C))
        if context is None:
            if nf != self.L:
                raise ValueError("the uniform start needs every site free")
            context = ps.uniform_start(seed, C, self.L, q, chain_offset)
        self.context = np.array(context, dtype=np.int64).reshape(C, self.L)
        self.s = self.context[:, self.free].copy()
        self.t = 0
        self.margin = np.broadcast_to(np.asarray(margin, dtype=np.float64), (nf,))
        self.first_tie = np.full(C, -1, dtype=np.int64)
        self.changes = 0

    @classmethod
    def from_model(cls, h, J, seed, n_chains, free, allowed=None, init=None, chain_offset=0, margin=0.0):
        h = np.asarray(h, dtype=np.float64)
        L, q = h.shape
        free = np.asarray(free, dtype=np.int64)
        if init is None:
            init = ps.uniform_start(seed, n_chains, L, q, chain_offset)
        init = np.asarray(init, dtype=np.int64).reshape(n_chains, L)
        return cls(fold(h, J, free, init), reduced_couplings(J, L, q, free), free, L, seed, allowed, init,
                   chain_offset, margin)

    def _draw(self, k, Z, beta):
        """The masked draw at free site k of every chain from Z (q, C); records near ties.  Returns the new codes."""
        q = self.q
        ok = self.ok[k][:, None]
        v = np.where(ok, beta * Z, -np.inf)
        p = np.where(ok, np.exp(v - v.max(axis=0)), 0.0)
        c = np.cumsum(p, axis=0)
        i = int(self.free[k])
        thr = ps.uniform(self.key, self.t, i, self.L) * c[-1]
        hit = thr[None, :] < c
        b = np.where(hit.any(axis=0), hit.argmax(axis=0), self.highest[k])
        if self.margin[k] > 0:
            tie = (np.abs(thr[None, :] - c[:-1]) <= self.margin[k] * c[-1]).any(axis=0)
            new = tie & (self.first_tie < 0)
            self.first_tie[new] = self.t * self.L + i
        self.changes += int((b != self.s[:, k]).sum())
        return b

    def run(self, sweeps, beta=1.0):
        q, nf = self.q, len(self.free)
        C = self.s.shape[0]
        rows = np.arange(C)
        cols = [np.ascontiguousarray(self.UFF[:, k * q:(k + 1) * q]) for k in range(nf)]
        X = np.zeros((C, nf * q))
        X[rows[:, None], np.arange(nf) * q + self.s] = 1.0
        self.changes = 0
        for _ in range(sweeps):
            for k in range(nf):
                Z = (X @ cols[k]).T + self.hc[:, k, :].T
                b = self._draw(k, Z, beta)
                X[rows, k * q + self.s[:, k]] = 0.0
                X[rows, k * q + b] = 1.0
                self.s[:, k] = b
            self.t += 1
        return self.changes

    def codes(self):
        out = self.context.copy()
        out[:, self.free] = self.s
        return out.astype(np.uint8)


def exact_conditional(h, J, beta, free, context, allowed=None):
    """P(s_F | context) over all q^nf states of the free sites (index = potts_sampler.state_index of the free codes),
    restricted to the allowed states, by enumeration in float64."""
    h = np.asarray(h, dtype=np.float64)
    L, q = h.shape
    free = np.asarray(free, dtype=np.int64)
    nf = len(free)
    if q ** nf > 10000:
        raise ValueError("enumeration is for q^nf <= 10000")
    states = np.array(np.unravel_index(np.arange(q ** nf), (q,) * nf)).T
    full = np.repeat(np.asarray(context, dtype=np.int64).reshape(1, L), len(states), axis=0)
    full[:, free] = states
    logp = beta * ps.energies(h, J, full)
    if allowed is not None:
        ok = np.all((np.asarray(allowed, dtype=np.int64)[None, :] >> states) & 1 == 1, axis=1)
        logp = np.where(ok, logp, -np.inf)
    p = np.exp(logp - logp.max())
    return p / p.sum()
