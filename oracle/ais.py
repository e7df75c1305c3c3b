"""
CPU restatement of annealed importance sampling on the library's Gibbs sampler (evc_sampler_anneal, contract in
include/evcplm.h; estimator in model_ops.log_partition), and exact log partition functions to hold it against.

The annealed sweep is the chain of oracle/potts_sampler.py with the draw taken from v_a = h_i(a) + beta (Z_i(a) -
h_i(a)), formed in numpy float32 with the device's roundings (numpy rounds every float32 operation on its own, as
__fsub_rn / __fmul_rn / __fadd_rn do), and the per-chain log weight gains (beta_k - beta_{k-1}) H_J(s) before each
sweep.  Test infrastructure, not product code.
"""
import numpy as np

from oracle import potts_sampler as ps


def linear_schedule(K):
    """beta_k = k / K, k = 0..K, float32 (dyadic, so exact, when K is a power of two)."""
    return (np.arange(K + 1, dtype=np.float64) / K).astype(np.float32)


def annealed_logits(h_i, Z, beta):
    """v (q, C) of the annealed draw at one site, float32 as on the device, returned as float64."""
    h32 = np.asarray(h_i, dtype=np.float32)[:, None]
    b32 = np.float32(beta)
    return (h32 + b32 * (Z.astype(np.float32) - h32)).astype(np.float64)


def annealed_near_tie_margin(q, z_error=0.0, beta=1.0, z_bound=0.0):
    """Half-width, on F_a = c_a / c_{q-1}, of the band in which the device's annealed draw can end on another state
    than this restatement (the counterpart of potts_sampler.near_tie_margin for v = h + beta (Z - h)).

    With eps = 2^-24, B = z_bound (|h_i(a)| + sum_j max_b |J_ij(a, b)| <= B, so |Z - h| <= B), delta = z_error and
    Bv = max(1, |beta|) (B + delta), which bounds |v| on both sides:
      * delta = 0: the device's Z is exact, so is this restatement's float64 Z, and both form v from the same float32
        values with the same roundings: every v is the same bits on both sides, and so is m = max v.  The device then
        rounds v - m (|v - m| <= 2 Bv: error 2 eps Bv); this side's exp and sums are float64.  eta = 2 eps Bv.
      * delta > 0: each side's v is off the exact h + beta (Z - h) by at most
            eta_v = |beta| delta + 2 eps |beta| (B + delta) + eps Bv
        (Z - h: delta plus one rounding; times beta: one rounding; plus h: one rounding of a value <= Bv), so v - m
        by 2 eta_v on each side, and the device's rounding of v - m adds 2 eps Bv: eta = 4 eta_v + 2 eps Bv.
    Then, as in near_tie_margin, every c_a is within the relative error rho = (e^eta - 1) + 2^-22 (expf) + (q - 1) eps
    (the fp32 prefix sum), F_a within 2 rho, and the margin is twice that bound."""
    eps, b = ps.EPS32, abs(float(beta))
    bv = max(1.0, b) * (np.asarray(z_bound, dtype=np.float64) + z_error)
    if z_error == 0.0:
        eta = 2.0 * eps * bv
    else:
        eta_v = b * z_error + 2.0 * eps * b * (np.asarray(z_bound, dtype=np.float64) + z_error) + eps * bv
        eta = 4.0 * eta_v + 2.0 * eps * bv
    rho = np.expm1(eta) + 2.0 ** -22 + (q - 1) * eps
    return 2.0 * (2.0 * rho)


def coupling_energy_error_bound(L, z_error):
    """Largest error of the device's H_J = 1/2 sum_i (Z_i(s_i) - h_i(s_i)) when each Z_i(a) is within z_error:
    L z_error / 2 (the differences and the sum are formed in double, whose roundings, below 2^-53 L B, are
    negligible next to it).  Over a monotone schedule from 0 to 1 the increments' factors beta_k - beta_{k-1} are
    >= 0 and sum to 1, so log w is off by at most the same L z_error / 2 (0 when Z is exact: dyadic models)."""
    return 0.5 * L * z_error


class _Annealed(object):
    """AIS on top of a restated chain (potts_sampler.Sampler or SparseSampler): ``logw`` (float64 per chain)
    accumulates like the device's d_logw, and run() still runs the plain chain."""

    _annealing = False

    def _init_weights(self):
        self.logw = np.zeros(self.s.shape[0])

    def _draw(self, i, Z, beta):
        if self._annealing:
            # v is the annealed logit; the base draw at beta = 1 computes 1.0 * v = v exactly
            return super(_Annealed, self)._draw(i, annealed_logits(self.h[i], Z, beta), 1.0)
        return super(_Annealed, self)._draw(i, Z, beta)

    def coupling_energy(self):
        """H_J(s) = sum_{i<j} J_ij(s_i, s_j) of every chain, float64 (exact for dyadic models)."""
        raise NotImplementedError

    def anneal(self, betas):
        """evc_sampler_anneal: K = len(betas) - 1 sweeps; returns the site changes."""
        betas = np.asarray(betas, dtype=np.float32)
        changes = 0
        for k in range(1, len(betas)):
            d = np.float64(betas[k]) - np.float64(betas[k - 1])
            self.logw = self.logw + d * self.coupling_energy()
            self._annealing = True
            try:
                changes += self.run(1, float(betas[k]))
            finally:
                self._annealing = False
        self.changes = changes
        return changes


class AnnealedSampler(_Annealed, ps.Sampler):
    """The dense restatement (potts_sampler.Sampler) with annealing."""

    def __init__(self, h, J, seed, n_chains, init=None, chain_offset=0, margin=0.0):
        ps.Sampler.__init__(self, h, J, seed, n_chains, init=init, chain_offset=chain_offset, margin=margin)
        self._init_weights()

    def coupling_energy(self):
        L = self.L
        iu, ju = np.triu_indices(L, 1)
        return self.U[iu[None, :], self.s[:, iu], ju[None, :], self.s[:, ju]].sum(axis=1)


class AnnealedSparseSampler(_Annealed, ps.SparseSampler):
    """The sparse restatement (potts_sampler.SparseSampler) with annealing."""

    def __init__(self, h, pairs, blocks, seed, n_chains, init=None, chain_offset=0, margin=0.0):
        ps.SparseSampler.__init__(self, h, pairs, blocks, seed, n_chains, init=init, chain_offset=chain_offset,
                                  margin=margin)
        self._init_weights()

    def coupling_energy(self):
        # every pair is listed at both of its sites: half of the sum over sites and neighbours
        e = np.zeros(self.s.shape[0])
        for i, (j, M) in enumerate(self.nbr):
            if len(j):
                e += M[np.arange(len(j))[None, :], self.s[:, j], self.s[:, i][:, None]].sum(axis=1)
        return 0.5 * e


def restated_log_weights(sampler, K, burn_in):
    """The procedure of model_ops.log_partition on a restated sampler fresh from its start: one sweep at beta = 0,
    the forward anneal 0 -> 1 over linear_schedule(K), burn_in plain sweeps at beta = 1, the reverse anneal 1 -> 0.
    Returns (forward log w, reverse log w)."""
    sampler.anneal([0.0, 0.0])
    sampler.anneal(linear_schedule(K))
    fwd = sampler.logw.copy()
    sampler.logw[:] = 0.0
    sampler.run(burn_in, 1.0)
    sampler.anneal(linear_schedule(K)[::-1])
    return fwd, sampler.logw.copy()


# ---- exact log Z -------------------------------------------------------------------------------------------------

def _logsumexp(x, axis=None):
    x = np.asarray(x, dtype=np.float64)
    m = np.max(x, axis=axis, keepdims=True)
    out = m + np.log(np.sum(np.exp(x - m), axis=axis, keepdims=True))
    return np.squeeze(out, axis=axis) if axis is not None else float(out.ravel()[0])


def log_z0(h):
    """log Z of the independent-site model: sum_i log sum_a exp h_i(a)."""
    return float(np.sum(_logsumexp(np.asarray(h, dtype=np.float64), axis=1)))


def log_z_enumeration(h, J):
    """log sum_s exp H(s) over all q^L states (q^L <= 4096)."""
    h = np.asarray(h, dtype=np.float64)
    L, q = h.shape
    if q ** L > 4096:
        raise ValueError("enumeration is for q^L <= 4096")
    states = np.array(np.unravel_index(np.arange(q ** L), (q,) * L)).T
    return _logsumexp(ps.energies(h, J, states))


def log_z_disjoint_pairs(h, J, pairs):
    """log Z of a model whose couplings are nonzero only on disjoint site pairs (synthetic.planted_potts_model's
    contacts): the sum over free sites of logsumexp h_i plus, per pair, log sum_ab exp(h_i(a) + h_j(b) + J_ij(a, b))."""
    h = np.asarray(h, dtype=np.float64)
    L, q = h.shape
    Jt = np.asarray(J, dtype=np.float64).reshape(-1, q, q)
    pairs = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    used = pairs.ravel()
    if len(set(used.tolist())) != len(used):
        raise ValueError("the pairs are not disjoint")
    iu, ju = np.triu_indices(L, 1)
    listed = np.zeros(len(iu), dtype=bool)
    out = 0.0
    for i, j in pairs:
        p = int(i * L - i * (i + 1) // 2 + (j - i - 1))
        listed[p] = True
        out += _logsumexp(h[i][:, None] + h[j][None, :] + Jt[p])
    if np.any(Jt[~listed] != 0):
        raise ValueError("a coupling outside the listed pairs is nonzero")
    free = np.setdiff1d(np.arange(L), used)
    return out + float(np.sum(_logsumexp(h[free], axis=1))) if len(free) else out


def log_z_chain(h, J):
    """log Z of a nearest-neighbour chain model (J_ij = 0 unless j = i + 1) by transfer matrices in float64, at any
    L: alpha_{i+1}(b) = h_{i+1}(b) + logsumexp_a(alpha_i(a) + J_{i,i+1}(a, b))."""
    h = np.asarray(h, dtype=np.float64)
    L, q = h.shape
    Jt = np.asarray(J, dtype=np.float64).reshape(-1, q, q)
    near = np.array([i * L - i * (i + 1) // 2 for i in range(L - 1)], dtype=np.int64)   # pair (i, i + 1)
    mask = np.ones(len(Jt), dtype=bool)
    mask[near] = False
    if np.any(Jt[mask] != 0):
        raise ValueError("a coupling J_ij with j != i + 1 is nonzero")
    alpha = h[0].copy()
    for i in range(L - 1):
        alpha = h[i + 1] + _logsumexp(alpha[:, None] + Jt[near[i]], axis=0)
    return _logsumexp(alpha)
