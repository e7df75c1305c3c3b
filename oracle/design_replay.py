"""
Teacher-forced fp32 replay of the library's design calls (evc_sampler_record_best / _best / _descend, contract in
include/evcplm.h), built on oracle/sampler_replay.py's Replay and oracle/tempered_replay.py's TemperedReplay: the same
fields, refresh rule and change update, plus each chain's record and the zero-temperature descent.  Test
infrastructure, not product code.

Nothing here needs a near-tie band.  The replay rebuilds Z bit for bit, the descent's argmax and its equality tests
involve no expf, and the record's H is summed in lane_sum's order from that Z, so every descent decision, every
settled flag and every record (energy, codes, sweep) must match the device exactly.

Conditional handles (``hc`` given): the replay runs over the free sites, with the per-chain fields hc (the device's
conditional_fields(), which match the fold bit for bit) and the couplings between free sites (reduced_couplings).  Its
sampling sweeps are followed from the device's codes, with their draws unchecked (the counters are positional in the
full model); the record and the descent are checked as on a plain handle.
"""
import numpy as np

from oracle.sampler_replay import F32, MUTATIONS, Replay, replay_calls
from oracle.tempered_replay import TEMPER_MUTATIONS, TemperedReplay, lane_sum, replay_tempered_calls

DESIGN_MUTATIONS = ("tie_to_smallest",       # a tie goes to the smallest state even when the current state is tied
                    "keep_disallowed",       # a disallowed current state is kept
                    "record_ge",             # the record is updated on H >= best instead of H > best
                    "record_before_sweep",   # the record's H and codes are taken before the sweep, not after it
                    "descent_skip_refresh")  # the descent never refreshes Z


class _Design(object):
    """The record and the descent, mixed into Replay or TemperedReplay (see DesignReplay, TemperedDesignReplay)."""

    def _design_init(self, mutation, hc, free, context, allowed):
        self.dmutation = mutation
        self.hc = None if hc is None else np.ascontiguousarray(hc, dtype=F32)
        if self.hc is not None:
            self.free = np.asarray(free, dtype=np.int64)
            self.context = np.array(context, dtype=np.int64)
        q = self.q
        masks = np.full(self.L, (1 << q) - 1, dtype=np.int64) if allowed is None else np.asarray(allowed, np.int64)
        self.ok = (masks[:, None] >> np.arange(q)[None, :]) & 1 == 1              # (sites, q)
        self.recording = False
        self.record_mismatch, self.descent_violations = [], []
        self.n_descent_violations = self.settled_mismatch = self.decisions_checked = 0

    # ---- rows, fields and energy ----------------------------------------------------------------------------------

    def full_codes(self):
        """(C, L_model) codes: the chains' rows, clamped sites included."""
        if self.hc is None:
            return self.s.astype(np.uint8)
        out = self.context.copy()
        out[:, self.free] = self.s
        return out.astype(np.uint8)

    def _fields(self):
        return self.model.h[None] if self.hc is None else self.hc

    def _refresh(self):
        if self.hc is None:
            return super()._refresh()
        acc = self.hc + F32(0.0)
        for sites, js, Ms in self.model.ranks:
            acc[:, sites, :] = acc[:, sites, :] + Ms[np.arange(len(sites))[None, :], self.s[:, js], :]
        self.Z = acc

    def design_energy(self):
        """H of every chain from its Z in double, lane_sum's order: sum hc(s) + 0.5 sum (Z(s) - hc(s))."""
        rows, sites = np.arange(self.C)[:, None], np.arange(self.L)[None, :]
        f = np.broadcast_to(self._fields(), (self.C, self.L, self.q))
        hs = f[rows, sites, self.s].astype(np.float64)
        dj = self.Z[rows, sites, self.s].astype(np.float64) - hs
        return lane_sum(hs) + 0.5 * lane_sum(dj)

    # ---- the record -----------------------------------------------------------------------------------------------

    def record_best(self):
        """evc_sampler_record_best: -inf, the current codes and sweep -1 for every chain."""
        self.recording = True
        self.best_energy = np.full(self.C, -np.inf)
        self.best_codes = self.full_codes()
        self.best_sweep = np.full(self.C, -1, dtype=np.int64)
        self.calls.append(("record_best", (), None, None))

    def _update_record(self, H, codes, t):
        better = H >= self.best_energy if self.dmutation == "record_ge" else H > self.best_energy
        self.best_energy = np.where(better, H, self.best_energy)
        self.best_codes[better] = codes[better]
        self.best_sweep[better] = t

    def _sweep(self, *args, **kw):
        if self.hc is not None and args[2] is not None:          # the device's full rows -> the free sites
            args = args[:2] + (np.asarray(args[2])[:, self.free],) + args[3:]
        if not self.recording:
            return super()._sweep(*args, **kw)
        if self.dmutation == "record_before_sweep":
            if self._refresh_due(args[3]):
                self._refresh()
                self.refresh_next = False
            H, codes, t = self.design_energy(), self.full_codes(), self.t
            changes = super()._sweep(*args, **kw)
        else:
            changes = super()._sweep(*args, **kw)
            H, codes, t = self.design_energy(), self.full_codes(), self.t - 1
        self._update_record(H, codes, t)
        return changes

    def best(self, energy=None, codes=None, sweep=None):
        """evc_sampler_best: checks the device's record (when given) bit for bit; returns the replay's."""
        if energy is None:
            self.calls.append(("best", (), None, (self.best_energy.copy(), self.best_codes.copy(),
                                                  self.best_sweep.copy())))
        else:
            bad = np.flatnonzero((np.asarray(energy, dtype=np.float64).view(np.uint64) !=
                                  self.best_energy.view(np.uint64)) |
                                 (np.asarray(codes) != self.best_codes).any(axis=1) |
                                 (np.asarray(sweep) != self.best_sweep))
            if len(bad):
                self.record_mismatch.append((self.t, bad))
        return self.best_energy.copy(), self.best_codes.copy(), self.best_sweep.copy()

    # ---- the descent ----------------------------------------------------------------------------------------------

    def descend(self, sweeps, codes=None, settled=None):
        """evc_sampler_descend: ``sweeps`` zero-temperature sweeps; ``codes`` the device's full rows after every sweep,
        ``settled`` its flags after the call.  Returns (settled, changes)."""
        gen = codes is None
        rec = [] if gen else None
        t_call = self.t
        changes, last = 0, np.zeros(self.C, dtype=np.int64)
        for k in range(int(sweeps)):
            if self.dmutation != "descent_skip_refresh" and self._refresh_due(t_call):
                self._refresh()
            self.refresh_next = False
            dev = None if gen else np.asarray(codes[k], dtype=np.int64)
            if dev is not None and self.hc is not None:
                dev = dev[:, self.free]
            last[:] = 0
            for i in range(self.L):
                b = self._argmax(i)
                if dev is not None:
                    self.decisions_checked += self.C
                    bad = np.flatnonzero(dev[:, i] != b)
                    self.n_descent_violations += len(bad)
                    for c_ in bad[:max(0, self.MAX_REPORT - len(self.descent_violations))]:
                        self.descent_violations.append((int(c_), self.t, i, int(dev[c_, i]), int(b[c_])))
                    b = dev[:, i]
                a = self.s[:, i]
                ch = np.flatnonzero(b != a)
                if len(ch):
                    self._change(i, ch, a[ch], b[ch])
                    self.s[ch, i] = b[ch]
                    last[ch] += 1
                    changes += len(ch)
            self.t += 1
            if gen:
                rec.append(self.full_codes())
        mine = (last == 0) if int(sweeps) > 0 else np.zeros(self.C, dtype=bool)
        if gen:
            self.calls.append(("descend", (int(sweeps),), np.array(rec).reshape(-1, self.C, self.full_codes().shape[1]),
                               mine.astype(np.uint8)))
        elif settled is not None and int(sweeps) > 0:
            self.settled_mismatch += int((np.asarray(settled).astype(bool) != mine).sum())
        self.call_changes.append(changes)
        return mine, changes

    def _argmax(self, i):
        """The descent's state at site i for every chain, from the fp32 row Z_i."""
        ok = self.ok[i][None, :]
        v = np.where(ok, self.Z[:, i, :], F32(-np.inf))
        m = v.max(axis=1, keepdims=True)
        top = ok & (v == m)
        a = self.s[:, i]
        rows = np.arange(self.C)
        keep = top[rows, a] | ~top.any(axis=1)
        if self.dmutation == "tie_to_smallest":
            keep = ~top.any(axis=1)
        elif self.dmutation == "keep_disallowed":
            keep = keep | ~self.ok[i][a]
        return np.where(keep, a, top.argmax(axis=1))

    def clean(self):
        return (super().clean() and not self.record_mismatch and self.n_descent_violations == 0 and
                self.settled_mismatch == 0)


def _split(mutation, own):
    if mutation is not None and mutation not in DESIGN_MUTATIONS and mutation not in own:
        raise ValueError("unknown mutation %r" % (mutation,))
    return (mutation, None) if mutation in DESIGN_MUTATIONS else (None, mutation)


class DesignReplay(_Design, Replay):
    """Replay of a plain handle (h, J or pairs / blocks as in Replay) or, with ``hc`` (C, nf, q), of a conditional one:
    then ``free`` (nf ascending sites), ``context`` (C, L) the start rows, ``allowed`` (nf masks or None), and
    h / J / pairs / blocks the reduced model over the free sites (its h is not used).  Results besides Replay's:
    ``record_mismatch`` (t, chains whose device record differs in any bit), ``descent_violations`` (chain, t, site,
    device state, replay state) of the first MAX_REPORT, ``n_descent_violations``, ``settled_mismatch`` and
    ``decisions_checked``.  ``mutation``: one of DESIGN_MUTATIONS, or of MUTATIONS as in Replay."""

    def __init__(self, h, J=None, seed=0, n_chains=1, init=None, chain_offset=0, pairs=None, blocks=None,
                 mutation=None, hc=None, free=None, context=None, allowed=None):
        dmut, mut = _split(mutation, MUTATIONS)
        if hc is not None:
            init = np.asarray(context)[:, np.asarray(free)]
        super().__init__(h, J, seed, n_chains, init, chain_offset, pairs, blocks, mut)
        self._design_init(dmut, hc, free, context, allowed)

    def _check(self, dv, u, b, i):
        if self.hc is None:
            return super()._check(dv, u, b, i)
        self.draws += self.C                    # followed, not checked: see the module's docstring

    def _generate(self, dv, u):
        if self.hc is not None:
            raise ValueError("a conditional replay follows the device's sampling sweeps; it generates only descents")
        return super()._generate(dv, u)


class TemperedDesignReplay(_Design, TemperedReplay):
    """TemperedReplay (a plain handle's ladders) with the record and the descent; results as in DesignReplay."""

    def __init__(self, h, J=None, seed=0, n_chains=1, init=None, chain_offset=0, ladder=(0.5, 1.0), swap_interval=1,
                 pairs=None, blocks=None, mutation=None):
        dmut, mut = _split(mutation, MUTATIONS + TEMPER_MUTATIONS)
        super().__init__(h, J, seed, n_chains, init, chain_offset, ladder, swap_interval, pairs, blocks, mut)
        self._design_init(dmut, None, None, None, None)


def replay_design_calls(replay, calls):
    """replay_tempered_calls (or replay_calls) for a design replay: also ("record_best", (), None, None), ("descend",
    (sweeps,), codes, settled) and ("best", (), None, (energy, codes, sweep))."""
    for call in calls:
        kind = call[0]
        if kind == "record_best":
            replay.record_best()
        elif kind == "descend":
            replay.descend(call[1][0], codes=call[2], settled=call[3])
        elif kind == "best":
            replay.best(*call[3])
        elif kind == "temper":
            replay_tempered_calls(replay, [call])
        else:
            replay_calls(replay, [call])
    return replay
