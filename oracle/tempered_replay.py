"""
Teacher-forced fp32 replay of the library's replica exchange (evc_sampler_set_ladder / evc_sampler_temper, contract
in include/evcplm.h), built on oracle/sampler_replay.py's Replay: the same fields, refresh, draws and draw check, with
each chain at the fp32 beta of its rung, and every energy and swap decision checked.  Test infrastructure, not
product code.
"""
import numpy as np

from oracle import potts_sampler as ps
from oracle.sampler_replay import F32, MUTATIONS, Replay, replay_calls


# energy_site_order: H summed by one thread in site order, in float.  (The same order in double changes no bit when
# the double sums are exact, as they are for fp32 terms of similar magnitude; the bit check catches it otherwise.)
TEMPER_MUTATIONS = ("energy_site_order",
                    "delta_sign",          # Delta of the wrong sign
                    "swap_states",         # an accepted swap exchanges the chains' codes, not their rung labels
                    "round_parity")        # round n tries the pairs of parity n + 1
SWAP_BAND = 8.0 * 2.0 ** -53               # relative band around exp(Delta): exp in double is within a few ulps


def lane_sum(d):
    """Sum over axis 1 of (C, n) float64 terms in the kernel's order: lane l adds terms l, l + 32, ... in turn, then
    the xor butterfly over offsets 16, 8, 4, 2, 1."""
    C, n = d.shape
    nb = -(-n // 32)
    pad = np.zeros((C, nb * 32))
    pad[:, :n] = d
    pad = pad.reshape(C, nb, 32)
    lanes = np.zeros((C, 32))
    for k in range(nb):
        lanes = lanes + pad[:, k, :]
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, idx ^ o]
    return lanes[:, 0]


class TemperedReplay(Replay):
    """The ladders of a tempered plain handle (evc_sampler_set_ladder on evc_sampler_create's handle), replayed in the
    device's fp32 arithmetic: every chain sweeps at the fp32 beta of the rung it holds (v = beta_c Z), and after the
    last sweep before each swap round H = sum h_i(s_i) + 1/2 sum (Z_i(s_i) - h_i(s_i)) is rebuilt from the replay's own
    Z in double, in the kernel's lane and butterfly order (lane_sum), so it is the device's H bit for bit.  Delta =
    (beta_{k+1} - beta_k)(H(x) - H(y)) is then the device's Delta bit for bit, and only exp(Delta) is not reproduced:
    a decision is checked unless u lies within SWAP_BAND of exp(Delta) (a near tie), where either outcome is accepted.

    ``temper(sweeps, codes, rungs, energies)`` takes the device's codes, rungs and energies after every sweep; the
    decisions are read off the rungs and followed.  Results besides Replay's: ``energy_mismatch`` (t, chains whose
    device energy differs in any bit), ``swap_violations`` ((t, ladder, pair, device accepted, replay accepted) or
    (t, "rungs") when the device's rungs are not the outcome of the round's pairs), ``n_swap_violations``,
    ``decisions``, ``swap_ties``, and the counts ``attempted``, ``accepted``, ``trips`` of the device's statistics.
    Without device data it generates the trajectory (``mutation`` from TEMPER_MUTATIONS plants a mistake, or one of
    MUTATIONS as in Replay)."""

    def __init__(self, h, J=None, seed=0, n_chains=1, init=None, chain_offset=0, ladder=(0.5, 1.0), swap_interval=1,
                 pairs=None, blocks=None, mutation=None):
        if mutation is not None and mutation not in TEMPER_MUTATIONS and mutation not in MUTATIONS:
            raise ValueError("unknown mutation %r" % (mutation,))
        tmut = mutation if mutation in TEMPER_MUTATIONS else None
        super().__init__(h, J, seed, n_chains, init, chain_offset, pairs, blocks, None if tmut else mutation)
        self.tmutation = tmut
        self.ladder = np.asarray(ladder, dtype=F32)
        self.R = R = self.ladder.size
        if n_chains % R or chain_offset % R:
            raise ValueError("whole ladders only")
        self.G = G = n_chains // R
        self.interval = int(swap_interval)
        self.holder = np.tile(np.arange(R), (G, 1))
        self.rung = self.holder.copy()
        self.heading = np.where(self.rung == 0, 1, 0)
        self.trips = np.zeros(G, dtype=np.int64)
        self.attempted = np.zeros(R - 1, dtype=np.int64)
        self.accepted = np.zeros(R - 1, dtype=np.int64)
        self.energy = np.zeros(n_chains)
        self.swap_key = ps.chain_key(seed, np.arange(chain_offset // R, chain_offset // R + G, dtype=np.uint64) |
                                     np.uint64(1 << 63))
        self.energy_mismatch, self.swap_violations = [], []
        self.n_swap_violations = self.decisions = self.swap_ties = 0

    def energies(self):
        L = self.L
        rows, sites = np.arange(self.C)[:, None], np.arange(L)[None, :]
        hs = self.model.h[sites, self.s].astype(np.float64)
        dj = self.Z[rows, sites, self.s].astype(np.float64) - hs
        if self.tmutation == "energy_site_order":
            eh, ej = np.zeros(self.C, dtype=F32), np.zeros(self.C, dtype=F32)
            for k in range(L):
                eh, ej = eh + hs[:, k].astype(F32), ej + dj[:, k].astype(F32)
            eh, ej = eh.astype(np.float64), ej.astype(np.float64)
        else:
            eh, ej = lane_sum(hs), lane_sum(dj)
        return eh + 0.5 * ej

    def temper(self, sweeps, codes=None, rungs=None, energies=None):
        """evc_sampler_temper: ``sweeps`` sweeps with their swap rounds; returns the site changes."""
        gen = codes is None
        rec = ([], [], []) if gen else None
        t_call = self.t
        changes = 0
        for k in range(int(sweeps)):
            beta = self.ladder[self.rung.ravel()][:, None]
            changes += self._sweep(beta, None, None if gen else codes[k], t_call)
            if self.t % self.interval == 0:
                self.energy = self.energies()
                if not gen:
                    bad = np.flatnonzero(np.asarray(energies[k], dtype=np.float64).view(np.uint64) !=
                                         self.energy.view(np.uint64))
                    if len(bad):
                        self.energy_mismatch.append((self.t, bad))
                self._round(self.t // self.interval - 1, None if gen else np.asarray(rungs[k]).reshape(self.G, self.R))
            if gen:
                rec[0].append(self.s.astype(np.uint8))
                rec[1].append(self.rung.ravel().astype(np.int32))
                rec[2].append(self.energy.copy())
        if gen:
            self.calls.append(("temper", (int(sweeps),), np.array(rec[0]).reshape(-1, self.C, self.L),
                               (np.array(rec[1]).reshape(-1, self.C), np.array(rec[2]).reshape(-1, self.C))))
        self.call_changes.append(changes)
        return changes

    def _round(self, n, dev_rung):
        G, R = self.G, self.R
        E = self.energy.reshape(G, R)
        lad = np.arange(G)
        first = (n + (1 if self.tmutation == "round_parity" else 0)) % 2
        for k in range(first if dev_rung is None else n % 2, R - 1, 2):
            x, y = self.holder[:, k].copy(), self.holder[:, k + 1].copy()
            d = (np.float64(self.ladder[k + 1]) - np.float64(self.ladder[k])) * (E[lad, x] - E[lad, y])
            if self.tmutation == "delta_sign":
                d = -d
            u = ps.uniform(self.swap_key, n, k, R)
            e = np.exp(np.minimum(d, 0.0))
            mine = (d >= 0) | (u < e)
            tie = (d < 0) & (np.abs(u - e) <= SWAP_BAND * e)
            self.decisions += G
            self.swap_ties += int(tie.sum())
            if dev_rung is None:
                acc = mine
            else:
                acc = dev_rung[lad, x] == k + 1
                bad = np.flatnonzero((acc != mine) & ~tie)
                self.n_swap_violations += len(bad)
                for l in bad[:max(0, self.MAX_REPORT - len(self.swap_violations))]:
                    self.swap_violations.append((self.t, int(l), k, bool(acc[l]), bool(mine[l])))
            self.attempted[k] += G
            self.accepted[k] += int(acc.sum())
            a = lad[acc]
            if self.tmutation == "swap_states":
                cx, cy = a * R + x[acc], a * R + y[acc]
                self.s[cx], self.s[cy] = self.s[cy].copy(), self.s[cx].copy()
                self._refresh()
                continue
            self.holder[a, k], self.holder[a, k + 1] = y[acc], x[acc]
            self.rung[a, x[acc]] = k + 1
            self.rung[a, y[acc]] = k
        if dev_rung is not None and not np.array_equal(dev_rung, self.rung):
            self.n_swap_violations += 1
            if len(self.swap_violations) < self.MAX_REPORT:
                self.swap_violations.append((self.t, "rungs"))
            self.rung = dev_rung.copy()
            self.holder = np.argsort(self.rung, axis=1)
        bottom, top = self.holder[:, 0], self.holder[:, R - 1]
        self.trips += self.heading[lad, bottom] == 2
        self.heading[lad, bottom] = 1
        up = self.heading[lad, top] == 1
        self.heading[lad[up], top[up]] = 2

    def clean(self):
        return super().clean() and not self.energy_mismatch and self.n_swap_violations == 0


def replay_tempered_calls(replay, calls):
    """replay_calls for a TemperedReplay: also ("temper", (sweeps,), codes, (rungs, energies))."""
    for call in calls:
        if call[0] == "temper":
            replay.temper(call[1][0], codes=call[2], rungs=call[3][0], energies=call[3][1])
        else:
            replay_calls(replay, [call])
    return replay
