"""
Teacher-forced replay of the library's Gibbs sampler (evc_sampler_run / _anneal / _set_model, contract in
include/evcplm.h) in the device's own fp32 arithmetic.  Test infrastructure, not product code.

The float64 restatements (oracle/potts_sampler.py, oracle/ais.py) follow a device chain only until its first draw the
device's rounding could decide differently.  This replay instead rebuilds, bit for bit, every value the kernel forms
before its softmax, and is driven by the device's trajectory: given the codes after every sweep it knows every site
change and its order (a sweep visits sites 0 .. L-1 once each), so it keeps each chain's field row Z exactly as the
device does and never loses a chain:

  * Z is a float32 array per chain.  A refresh (at global sweep t % REFRESH == 0, and on the sweep right after
    set_model) forms h, then adds the row of every site j in ascending j, one fp32 add at a time.  Between refreshes
    each change a -> b at site i adds (rb - ra), formed in fp32, to Z.  Couplings are kept per coupled pair only:
    the device's adds of the zero rows of uncoupled pairs leave fp32 values unchanged (x + 0 = x, and no Z value is
    ever -0: the refresh adds the zero of the site's own diagonal block, which this replay does as h + 0).
  * the logit is v = beta Z (plain) or h + beta (Z - h) (annealed), in fp32, each operation rounded on its own; m =
    max v and v - m in fp32, as on the device.  Only expf (within 2 ulp) and the fp32 prefix sum are not reproduced:
    p = exp(v - m) is taken in float64, and a draw is checked unless u lies within a margin of a boundary of the
    normalised cumulative F (see draw_margin).  At such a near tie the replay accepts the states that border it.
  * before an annealed sweep, H_J = 1/2 sum_i (Z_i(s_i) - h_i(s_i)) is summed in double with the kernel's lane stride
    of 32 and xor butterfly, and log w += (double(beta_k) - double(beta_{k-1})) (0.5 e): bit for bit the device's.

Generate mode (no device codes given) draws with the same arithmetic, exp rounded once to fp32 and the prefix sum in
fp32 along the kernel's shuffle scan, and records the trajectory; ``mutation`` makes generate mode commit one
plausible kernel mistake (MUTATIONS), so the CPU tests can show that the replay catches it.  One mistake no draw
check can see is u rounded to fp32: it moves u by at most 2^-25, and only when u >= 1/2, where every band is wider
(4 rho F_b >= 2^-21).
"""
import math

import numpy as np

from oracle import potts_sampler as ps

F32 = np.float32
REFRESH = ps.REFRESH
EPS32 = ps.EPS32
TINY32 = 2.0 ** -126            # smallest normal fp32: expf below it is subnormal or 0

MUTATIONS = ("skip_refresh",        # no refresh after the first sweep's
             "call_refresh",        # refresh at each call's first sweep instead of at global t % REFRESH == 0
             "refresh_descending",  # refresh adds the rows in descending j
             "refresh_h_last",      # refresh adds h after the rows
             "update_z_rb_ra",      # a change adds (z + rb) - ra
             "swap_rows",           # a change adds ra - rb
             "fma_logit",           # annealed logit contracted to fmaf(beta, z - h, h)
             "sequential_hj",       # H_J summed in site order by one thread
             "dbeta_f32")           # beta_k - beta_{k-1} formed in fp32


def draw_margin(q):
    """Half-width, relative to F_b, of the band around each boundary F_b = c_b / c_{q-1} in which the device's draw
    may differ from the exact-exp draw on the same fp32 v - m.  Each term expf(v - m) is within 2 ulp (relative
    2^-22) and the inclusive shuffle scan passes each term through at most ceil(log2 q) fp32 adds of positive values
    (relative ceil(log2 q) eps), so every c_b, c_{q-1} included, is within rho = 2^-22 + ceil(log2 q) eps (1 + q eps)
    of its exact value and F_b within 2 rho F_b / (1 - rho).  The margin is twice that: 4 rho F_b.  draw_abs adds the
    subnormal range of expf (each of q terms off by at most 2^-126 absolute; c_{q-1} >= 1 since m is one of the v)."""
    rho = 2.0 ** -22 + math.ceil(math.log2(q)) * EPS32 * (1.0 + q * EPS32)
    return 4.0 * rho


def draw_abs(q):
    return 2.0 * q * TINY32


class _Model(object):
    """h (L, q) float32 and, per site i, its coupled sites (ascending) with the blocks D_i[k, b, a] = J_{i j_k}(a, b),
    b the state of j_k, a that of i, in float32; ``ranks[r]`` groups the r-th neighbour of every site (for the
    refresh, which adds each site's neighbours in order)."""

    def __init__(self, h, pairs, blocks, descending=False):
        self.h = np.ascontiguousarray(h, dtype=F32)
        self.L, self.q = self.h.shape
        nbr = ps.sparse_neighbours(self.L, self.q, pairs, np.asarray(blocks, dtype=F32))
        self.nbr = [(j, np.ascontiguousarray(M, dtype=F32)) for j, M in nbr]
        # a change at site i moves Z_j(x) of each neighbour j by J_ji(x, b) - J_ji(x, a) = M_i[k, x, b] - M_i[k, x, a]
        self.upd = [(j, np.ascontiguousarray(M.transpose(0, 2, 1))) for j, M in self.nbr]
        deg = np.array([len(j) for j, _ in self.nbr])
        self.ranks = []
        for r in range(int(deg.max(initial=0))):
            sites = np.flatnonzero(deg > r)
            pick = [(len(self.nbr[i][0]) - 1 - r) if descending else r for i in sites]
            js = np.array([self.nbr[i][0][k] for i, k in zip(sites, pick)], dtype=np.int64)
            Ms = np.stack([self.nbr[i][1][k] for i, k in zip(sites, pick)])
            self.ranks.append((sites, js, Ms))


def dense_pairs(L):
    iu, ju = np.triu_indices(L, 1)
    return np.stack([iu, ju], axis=1)


class Replay(object):
    """The chains of one sampler handle: ``n_chains`` chains with global indices chain_offset + 0 .., from the codes
    ``init`` (the device's codes before the first call).  The model is given either dense (J: the packed
    (L (L - 1) / 2, q, q) blocks) or sparse (pairs (n, 2), i < j, and their blocks).

    Each call takes the device's codes after every sweep (``codes``: (sweeps, n_chains, L)) and, for anneal, its log
    weights after every sweep (``logw``: (K, n_chains)); without them it generates the sweeps itself and appends them
    to ``calls``.  Results, over all calls: ``violations`` (chain, t, site, device state, allowed states) of the
    first MAX_REPORT, ``n_violations``, ``draws``, ``checked`` (draws outside every near-tie band), ``ties``,
    ``logw`` (replayed), ``logw_mismatch`` (t, chains whose device log weight differs in any bit), ``call_changes``
    (site changes of each call)."""

    MAX_REPORT = 64

    def __init__(self, h, J=None, seed=0, n_chains=1, init=None, chain_offset=0, pairs=None, blocks=None,
                 mutation=None):
        if mutation is not None and mutation not in MUTATIONS:
            raise ValueError("unknown mutation %r" % (mutation,))
        self.mutation = mutation
        self._set(h, J, pairs, blocks)
        self.key = ps.chain_key(seed, np.arange(chain_offset, chain_offset + n_chains))
        if init is None:
            init = ps.uniform_start(seed, n_chains, self.L, self.q, chain_offset)
        self.s = np.array(init, dtype=np.int64).reshape(n_chains, self.L)
        self.C = n_chains
        self.Z = np.zeros((n_chains, self.L, self.q), dtype=F32)
        self.t = 0
        self.refresh_next = False
        self.logw = np.zeros(n_chains)
        self.margin, self.abs = draw_margin(self.q), draw_abs(self.q)
        self.violations, self.n_violations = [], 0
        self.draws = self.checked = self.ties = 0
        self.logw_mismatch = []
        self.call_changes = []
        self.calls = []

    def _set(self, h, J, pairs, blocks):
        h = np.asarray(h, dtype=F32)
        L, q = h.shape
        if J is not None:
            pairs, blocks = dense_pairs(L), np.asarray(J, dtype=F32).reshape(-1, q, q)
        self.model = _Model(h, pairs, blocks, descending=self.mutation == "refresh_descending")
        self.L, self.q = L, q

    # ---- the calls ------------------------------------------------------------------------------------------------

    def run(self, sweeps, beta=1.0, codes=None):
        """evc_sampler_run: ``sweeps`` sweeps at beta; returns the site changes."""
        gen = codes is None
        rec = [] if gen else None
        t_call = self.t
        changes = 0
        for k in range(int(sweeps)):
            changes += self._sweep(F32(beta), None, None if gen else codes[k], t_call)
            if gen:
                rec.append(self.s.astype(np.uint8))
        if gen:
            self.calls.append(("run", (int(sweeps), float(beta)), np.array(rec).reshape(-1, self.C, self.L), None))
        self.call_changes.append(changes)
        return changes

    def anneal(self, betas, codes=None, logw=None):
        """evc_sampler_anneal: len(betas) - 1 sweeps, sweep k at betas[k + 1] after log w += (betas[k + 1] -
        betas[k]) H_J; returns the site changes."""
        b = np.asarray(betas, dtype=F32)
        gen = codes is None
        rec, recw = ([], []) if gen else (None, None)
        t_call = self.t
        changes = 0
        for k in range(len(b) - 1):
            changes += self._sweep(b[k + 1], b[k], None if gen else codes[k], t_call,
                                   None if gen else logw[k])
            if gen:
                rec.append(self.s.astype(np.uint8))
                recw.append(self.logw.copy())
        if gen:
            self.calls.append(("anneal", (b.copy(),), np.array(rec).reshape(-1, self.C, self.L),
                               np.array(recw).reshape(-1, self.C)))
        self.call_changes.append(changes)
        return changes

    def set_model(self, h, J=None, pairs=None, blocks=None):
        """evc_sampler_set_model: the next sweep refreshes Z from the new parameters."""
        self._set(h, J, pairs, blocks)
        self.refresh_next = True
        self.calls.append(("set_model", (np.asarray(h, dtype=F32).copy(),
                                         None if J is None else np.asarray(J, dtype=F32).copy(), pairs, blocks),
                           None, None))

    # ---- one sweep ------------------------------------------------------------------------------------------------

    def _refresh_due(self, t_call):
        mut, t = self.mutation, self.t
        if self.refresh_next:
            return True
        if mut == "skip_refresh":
            return t == 0
        if mut == "call_refresh":
            return t == t_call
        return t % REFRESH == 0

    def _refresh(self):
        md = self.model
        if self.mutation == "refresh_h_last":
            acc = np.zeros((self.C, self.L, self.q), dtype=F32)
        else:
            acc = np.broadcast_to(md.h + F32(0.0), (self.C, self.L, self.q)).copy()
        for sites, js, Ms in md.ranks:
            acc[:, sites, :] = acc[:, sites, :] + Ms[np.arange(len(sites))[None, :], self.s[:, js], :]
        if self.mutation == "refresh_h_last":
            acc = acc + md.h
        self.Z = acc

    def _hj_terms(self):
        """e of every chain: the double sum of Z_i(s_i) - h_i(s_i) in the kernel's order."""
        L = self.L
        rows = np.arange(self.C)[:, None]
        sites = np.arange(L)[None, :]
        d = self.Z[rows, sites, self.s].astype(np.float64) - self.model.h[sites, self.s].astype(np.float64)
        if self.mutation == "sequential_hj":
            e = np.zeros(self.C)
            for k in range(L):
                e = e + d[:, k]
            return e
        nb = -(-L // 32)
        pad = np.zeros((self.C, nb * 32))
        pad[:, :L] = d
        pad = pad.reshape(self.C, nb, 32)
        lanes = np.zeros((self.C, 32))
        for k in range(nb):                           # lane l adds sites l, l + 32, ... in turn (then + 0 past L)
            lanes = lanes + pad[:, k, :]
        idx = np.arange(32)
        for o in (16, 8, 4, 2, 1):
            lanes = lanes + lanes[:, idx ^ o]
        return lanes[:, 0]

    def _sweep(self, beta, beta0, after, t_call, logw_dev=None):
        """One sweep at fp32 beta (annealed when beta0 is not None).  ``after``: the device's codes after it, or None
        to generate.  Returns the site changes."""
        md, L, q, C = self.model, self.L, self.q, self.C
        if self._refresh_due(t_call):
            self._refresh()
        self.refresh_next = False
        if beta0 is not None:
            e = self._hj_terms()
            if self.mutation == "dbeta_f32":
                db = np.float64(F32(beta - beta0))
            else:
                db = np.float64(beta) - np.float64(beta0)
            self.logw = self.logw + db * (0.5 * e)
            if logw_dev is not None:
                bad = np.flatnonzero(np.asarray(logw_dev, dtype=np.float64).view(np.uint64) !=
                                     self.logw.view(np.uint64))
                if len(bad):
                    self.logw_mismatch.append((self.t, bad))
        rows = np.arange(C)
        changes = 0
        for i in range(L):
            z = self.Z[:, i, :]
            if beta0 is not None:
                hi = md.h[i][None, :]
                if self.mutation == "fma_logit":
                    v = (np.float64(beta) * (z - hi).astype(np.float64) + hi.astype(np.float64)).astype(F32)
                else:
                    v = hi + beta * (z - hi)
            else:
                v = beta * z
            dv = v - v.max(axis=1, keepdims=True)
            u = ps.uniform(self.key, self.t, i, L)
            if after is None:
                b = self._generate(dv, u)
            else:
                b = np.asarray(after[:, i], dtype=np.int64)
            self._check(dv, u, b, i)
            a = self.s[:, i]
            ch = np.flatnonzero(b != a)
            if len(ch):
                self._change(i, ch, a[ch], b[ch])
                self.s[ch, i] = b[ch]
                changes += len(ch)
        self.t += 1
        return changes

    def _generate(self, dv, u):
        """The draw with exp rounded once to fp32 and the kernel's fp32 shuffle scan."""
        cum = np.exp(dv.astype(np.float64)).astype(F32)
        o = 1
        while o < self.q:
            y = np.zeros_like(cum)
            y[:, o:] = cum[:, :-o]
            cum = cum + y
            o <<= 1
        tot = cum[:, -1].astype(np.float64)
        hit = (u * tot)[:, None] < cum.astype(np.float64)
        return np.where(hit.any(axis=1), hit.argmax(axis=1), self.q - 1)

    def _check(self, dv, u, b, i):
        """Records the draw of every chain at site i: the device's state b must lie in the band of u."""
        q = self.q
        p = np.exp(dv.astype(np.float64))
        c = np.cumsum(p, axis=1)
        F = c / c[:, -1:]
        band = self.margin * F + self.abs
        rows = np.arange(self.C)
        lo = np.where(b > 0, F[rows, np.maximum(b - 1, 0)], 0.0)
        lo_band = np.where(b > 0, band[rows, np.maximum(b - 1, 0)], 0.0)
        hi = np.where(b < q - 1, F[rows, b], np.inf)
        hi_band = np.where(b < q - 1, band[rows, b], 0.0)
        ok = (u >= lo - lo_band) & (u < hi + hi_band)
        tie = (np.abs(u[:, None] - F[:, :-1]) <= band[:, :-1]).any(axis=1)
        self.draws += self.C
        self.ties += int(tie.sum())
        self.checked += int((~tie).sum())
        bad = np.flatnonzero(~ok)
        if len(bad):
            self.n_violations += len(bad)
            for c_ in bad[:max(0, self.MAX_REPORT - len(self.violations))]:
                lo_edges = np.concatenate([[0.0], F[c_, :-1]])
                hi_edges = np.concatenate([F[c_, :-1], [np.inf]])
                bl = np.concatenate([[0.0], band[c_, :-1]])
                bh = np.concatenate([band[c_, :-1], [0.0]])
                allowed = tuple(int(x) for x in np.flatnonzero((u[c_] >= lo_edges - bl) & (u[c_] < hi_edges + bh)))
                self.violations.append((int(c_), self.t, i, int(b[c_]), allowed))

    def _change(self, i, ch, a, b):
        """Z of the chains ch after site i changed a -> b: every neighbour's block adds rb - ra in fp32."""
        js, Mt = self.model.upd[i]
        if not len(js):
            return
        k = np.arange(len(js))[None, :]
        rb = Mt[k, b[:, None], :]                     # (len(ch), m, q): J_ji(., b)
        ra = Mt[k, a[:, None], :]
        sel = (ch[:, None], js[None, :])
        if self.mutation == "update_z_rb_ra":
            self.Z[sel] = (self.Z[sel] + rb) - ra
        elif self.mutation == "swap_rows":
            self.Z[sel] = self.Z[sel] + (ra - rb)
        else:
            self.Z[sel] = self.Z[sel] + (rb - ra)

    # ---- summaries -------------------------------------------------------------------------------------------------

    def checked_share(self):
        return self.checked / max(1, self.draws)

    def clean(self):
        """No draw outside its band and every log weight bit-identical."""
        return self.n_violations == 0 and not self.logw_mismatch


def replay_calls(replay, calls):
    """Drives ``replay`` with a recorded list of calls (Replay.calls of a generate-mode run, or the same shape from
    the device): ("run", (sweeps, beta), codes, None), ("anneal", (betas,), codes, logw), ("set_model", (h, J,
    pairs, blocks), None, None)."""
    for kind, args, codes, logw in calls:
        if kind == "run":
            replay.run(args[0], args[1], codes=codes)
        elif kind == "anneal":
            replay.anneal(args[0], codes=codes, logw=logw)
        else:
            replay.set_model(*args)
    return replay
