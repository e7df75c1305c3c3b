"""
CPU restatement of the library's replica exchange (evc_sampler_set_ladder / evc_sampler_temper, contract in
include/evcplm.h), in numpy float64: ladders of chains of potts_sampler.Sampler or conditional_sampler.ConditionalSampler
swept at the beta of the rung each holds, the energy formed before every swap round, the even-odd swap rounds with
their counter-based uniforms, label exchange and round trips.  A chain here follows the device chain draw for draw
until a near tie, of a draw (the base sampler's margin) or of a swap decision (swap_margin).  Also the exact rung
distributions of small models by enumeration and the Curie-Weiss Potts model, whose mode probabilities are exact.
Test infrastructure, not product code.
"""
import math

import numpy as np

from oracle import potts_sampler as ps

HEAD_NONE, HEAD_UP, HEAD_DOWN = 0, 1, 2


def swap_key(seed, g):
    """swap_key(g) = key(2^63 + g): the chain key of an index no chain has."""
    return ps.chain_key(seed, np.asarray(g, dtype=np.uint64) | np.uint64(1 << 63))


def swap_uniform(key, n, k, R):
    """u(g, n, k) = ((mix(swap_key(g) + (n R + k + 1) phi) >> 40) + 0.5) 2^-24."""
    return ps.uniform(key, n, k, R)


def swap_rounds(t0, sweeps, interval):
    """The (global sweep count after the round, round n) of the swap rounds that sweeps t0 .. t0 + sweeps - 1 reach."""
    return [(t + 1, (t + 1) // interval - 1) for t in range(t0, t0 + sweeps) if (t + 1) % interval == 0]


class Tempered(object):
    """The G = C / R ladders over the C chains of ``base`` (a potts_sampler.Sampler or a
    conditional_sampler.ConditionalSampler, whose chain c is the handle's chain c): ladder l is the chains l R ..
    l R + R - 1, global ladder index ``ladder_offset`` + l.

    ``swap_margin``: half-width on log u of a near-tie swap decision (the device forms H from fp32 fields and takes
    exp in double); ``first_swap_tie[l]`` then holds the first round of ladder l with such a decision (-1: none), and
    ``first_tie`` of each ladder the earliest near-tie draw of its chains (global draw number) or -1.
    ``mutation`` plants a mistake, for the tests of the checks: "energy_site_order" (H summed over sites in order,
    a single chain of additions), "delta_sign" (Delta of the wrong sign), "swap_states" (codes exchanged instead of
    labels) or "round_parity" (round n tries the pairs of parity n + 1)."""

    def __init__(self, base, ladder, swap_interval, seed, ladder_offset=0, swap_margin=0.0, mutation=None):
        self.base = base
        self.ladder = np.asarray(ladder, dtype=np.float32)
        self.R = R = self.ladder.size
        C = base.s.shape[0]
        if R < 2 or C % R:
            raise ValueError("need R >= 2 and whole ladders")
        self.G = G = C // R
        self.interval = int(swap_interval)
        self.holder = np.tile(np.arange(R), (G, 1))          # holder[l, k]: the chain of ladder l at rung k
        self.rung = self.holder.copy()                        # rung[l, x]: the rung chain x of ladder l holds
        self.heading = np.where(self.rung == 0, HEAD_UP, HEAD_NONE)
        self.trips = np.zeros(G, dtype=np.int64)
        self.attempted = np.zeros(R - 1, dtype=np.int64)
        self.accepted = np.zeros(R - 1, dtype=np.int64)
        self.energy = np.zeros(C)
        self.key = swap_key(seed, np.arange(ladder_offset, ladder_offset + G))
        self.swap_margin = float(swap_margin)
        self.first_swap_tie = np.full(G, -1, dtype=np.int64)
        self.decisions = []                                   # per round: (n, (G, pairs) accepted)
        self.mutation = mutation
        self.changes = 0

    def chain_betas(self):
        """(C,) float64: the beta each chain runs at, the fp32 ladder value of its rung."""
        return self.ladder[self.rung.ravel()].astype(np.float64)

    def energies(self):
        """(C,) float64 H of every chain: sum_i h_i(s_i) + 1/2 sum_i (Z_i(s_i) - h_i(s_i)), over the free sites with
        hc in place of h on a conditional base."""
        b = self.base
        C = b.s.shape[0]
        rows = np.arange(C)[:, None]
        if hasattr(b, "hc"):
            q, nf = b.q, len(b.free)
            hs = b.hc[rows, np.arange(nf)[None, :], b.s]                          # (C, nf)
            X = np.zeros((C, nf * q))
            X[rows, np.arange(nf) * q + b.s] = 1.0
            Js = (X @ b.UFF).reshape(C, nf, q)[rows, np.arange(nf)[None, :], b.s]
        else:
            L, q = b.L, b.q
            hs = b.h[np.arange(L)[None, :], b.s]
            X = np.zeros((C, L * q))
            X[rows, np.arange(L) * q + b.s] = 1.0
            Js = (X @ b.U.reshape(L * q, L * q)).reshape(C, L, q)[rows, np.arange(L)[None, :], b.s]
        if self.mutation == "energy_site_order":
            # one chain of fp32 additions in site order instead of the lanes' double sums
            acc = np.zeros(C, dtype=np.float32)
            for i in range(hs.shape[1]):
                acc = acc + (hs[:, i] + 0.5 * Js[:, i]).astype(np.float32)
            return acc.astype(np.float64)
        return hs.sum(axis=1) + 0.5 * Js.sum(axis=1)

    def run(self, sweeps):
        """``sweeps`` tempered sweeps with their swap rounds; returns the site changes."""
        b = self.base
        done, changes = 0, 0
        while done < sweeps:
            to_round = self.interval - b.t % self.interval
            k = min(sweeps - done, to_round)
            changes += b.run(k, beta=self.chain_betas())
            done += k
            if k == to_round:
                self._round(b.t // self.interval - 1)
        self.changes = changes
        return changes

    def _round(self, n):
        G, R = self.G, self.R
        E = self.energy = self.energies().reshape(G, R)
        lad = np.arange(G)
        first = (n + (1 if self.mutation == "round_parity" else 0)) % 2
        acc_round = np.zeros((G, R - 1), dtype=bool)
        for k in range(first, R - 1, 2):
            x, y = self.holder[:, k].copy(), self.holder[:, k + 1].copy()
            d = (float(self.ladder[k + 1]) - float(self.ladder[k])) * (E[lad, x] - E[lad, y])
            if self.mutation == "delta_sign":
                d = -d
            u = swap_uniform(self.key, n, k, R)
            accept = (d >= 0) | (u < np.exp(np.minimum(d, 0.0)))
            if self.swap_margin > 0:
                tie = np.abs(np.log(u) - d) <= self.swap_margin
                new = tie & (self.first_swap_tie < 0)
                self.first_swap_tie[new] = n
            self.attempted[k] += G
            self.accepted[k] += int(accept.sum())
            acc_round[:, k] = accept
            a = lad[accept]
            if self.mutation == "swap_states":
                cx, cy = a * R + x[accept], a * R + y[accept]
                s = self.base.s
                s[cx], s[cy] = s[cy].copy(), s[cx].copy()
                continue
            self.holder[a, k], self.holder[a, k + 1] = y[accept], x[accept]
            self.rung[a, x[accept]] = k + 1
            self.rung[a, y[accept]] = k
        self.decisions.append((n, acc_round))
        bottom, top = self.holder[:, 0], self.holder[:, R - 1]
        self.trips += self.heading[lad, bottom] == HEAD_DOWN
        self.heading[lad, bottom] = HEAD_UP
        up = self.heading[lad, top] == HEAD_UP
        self.heading[lad[up], top[up]] = HEAD_DOWN

    def rung_codes(self, k):
        """(G, L) codes of the chain at rung k of every ladder."""
        codes = self.base.codes().reshape(self.G, self.R, -1)
        return codes[np.arange(self.G), self.holder[:, k]]

    def ladder_first_tie(self):
        """(G,) the earliest near-tie draw (global draw number t L + i) of any chain of each ladder, -1 if none."""
        ft = self.base.first_tie.reshape(self.G, self.R)
        big = np.iinfo(np.int64).max
        m = np.where(ft < 0, big, ft).min(axis=1)
        return np.where(m == big, -1, m)


def swap_margin(L, z_bound, beta_max, bits=None):
    """Half-width on log u of the swap decisions the device could decide differently: H is a double sum of at most
    2 L terms of magnitude <= z_bound (exact fp32 fields on dyadic models; otherwise the caller adds the fields' own
    error), so |dH| <= 4 L eps64 L z_bound per chain; Delta carries twice that times beta_max, and exp in double is
    within a few ulps.  The margin is a hundred times that, plus 1e-12."""
    eps64 = 2.0 ** -53
    return 100.0 * (2.0 * beta_max * 4.0 * L * L * eps64 * z_bound) + 1e-12


# ---- Curie-Weiss Potts model: J_ij(a, b) = K delta_ab for every pair, h = 0 ----------------------------------------

def curie_weiss_model(L, q, K):
    """(h, J) float32 of the Curie-Weiss Potts model."""
    h = np.zeros((L, q), dtype=np.float32)
    J = np.repeat((K * np.eye(q, dtype=np.float64))[None], L * (L - 1) // 2, axis=0).astype(np.float32)
    return h, J


def compositions(L, q):
    """(M, q) every occupation vector n >= 0 with sum L."""
    if q == 1:
        return np.array([[L]])
    return np.array([[a] + list(rest) for a in range(L, -1, -1) for rest in compositions(L - a, q - 1)])


def occupation(codes, q):
    codes = np.asarray(codes, dtype=np.int64)
    return np.stack([(codes == a).sum(axis=1) for a in range(q)], axis=1)


def mode_of(codes, q):
    """The most occupied state of every row, ties to the smallest state."""
    return occupation(codes, q).argmax(axis=1)


def curie_weiss_mode_probabilities(L, q, K, beta):
    """P(mode = a) exactly, from P(n) ~ L! / prod n_a! exp(beta K / 2 (sum n_a^2 - L)) over the compositions, with
    mode_of's tie rule (so not exactly 1/q when ties are possible)."""
    n = compositions(L, q)
    logp = np.array([math.lgamma(L + 1) - sum(math.lgamma(v + 1) for v in row) for row in n])
    logp = logp + beta * K / 2.0 * ((n * n).sum(axis=1) - L)
    p = np.exp(logp - logp.max())
    p /= p.sum()
    mode = n.argmax(axis=1)
    return np.array([p[mode == a].sum() for a in range(q)])


def mode_bound(p, n, tail=1e-6):
    """Largest deviation |freq - p_a| of n independent mode draws allowed with probability about ``tail`` for each
    state: Hoeffding, sqrt(ln(2 q / tail) / (2 n))."""
    return math.sqrt(math.log(2 * len(p) / tail) / (2.0 * n))
