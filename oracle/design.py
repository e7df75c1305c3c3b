"""
Float64 restatement of the library's design (model_ops.design_codes): the record of each chain's best state while it
anneals (potts_sampler.Sampler, one sweep per inverse temperature), the zero-temperature descent with the device's tie
rules, single-site optimality and the global maximum by enumeration, for exhaustive checks on small models.  Test
infrastructure, not product code.
"""
import numpy as np

from oracle import potts_sampler as ps


def all_states(L, q):
    return np.array(np.unravel_index(np.arange(q ** L), (q,) * L)).T


def global_max(h, J, free=None, context=None, allowed=None):
    """(H*, states attaining it) over every state of the free sites (all sites when free is None) given ``context``,
    each free site restricted to its ``allowed`` mask, by enumeration in float64."""
    h = np.asarray(h, dtype=np.float64)
    L, q = h.shape
    free = np.arange(L) if free is None else np.asarray(free, dtype=np.int64)
    if q ** len(free) > 1 << 16:
        raise ValueError("enumeration is for q^nf <= 65536")
    states = all_states(len(free), q)
    if allowed is not None:
        ok = np.all((np.asarray(allowed, dtype=np.int64)[None, :] >> states) & 1 == 1, axis=1)
        states = states[ok]
    full = np.zeros((len(states), L), dtype=np.int64) if context is None else \
        np.repeat(np.asarray(context, dtype=np.int64).reshape(1, L), len(states), axis=0)
    full[:, free] = states
    E = ps.energies(h, J, full)
    return float(E.max()), full[E == E.max()]


def single_site_gains(h, J, codes, free=None, allowed=None):
    """(C, nf, q) float64 H(s with site F_k set to a) - H(s), -inf for a disallowed a."""
    h = np.asarray(h, dtype=np.float64)
    L, q = h.shape
    codes = np.asarray(codes, dtype=np.int64)
    C = len(codes)
    free = np.arange(L) if free is None else np.asarray(free, dtype=np.int64)
    U = ps.full_couplings(J, L, q)
    rows = np.arange(C)
    out = np.empty((C, len(free), q))
    for k, i in enumerate(free):
        z = h[i][None, :] + sum(U[i, :, j, codes[:, j]] for j in range(L) if j != i)    # (C, q)
        out[:, k, :] = z - z[rows, codes[:, i]][:, None]
        if allowed is not None:
            out[:, k, :] = np.where((int(allowed[k]) >> np.arange(q)) & 1 == 1, out[:, k, :], -np.inf)
    return out


def is_local_max(h, J, codes, free=None, allowed=None, tol=0.0):
    """(C,) bool: no allowed single-site change raises H by more than ``tol``."""
    return single_site_gains(h, J, codes, free, allowed).max(axis=(1, 2)) <= tol


def descend(h, J, codes, free=None, allowed=None, max_sweeps=1000):
    """The device's descent in float64: per free site in order, keep s_i if it is allowed and attains the max of
    Z_i over the allowed states, else take the smallest allowed state attaining it; repeated until a sweep changes
    nothing.  Returns (codes, settled)."""
    h = np.asarray(h, dtype=np.float64)
    L, q = h.shape
    s = np.array(codes, dtype=np.int64)
    C = len(s)
    free = np.arange(L) if free is None else np.asarray(free, dtype=np.int64)
    masks = np.full(len(free), (1 << q) - 1) if allowed is None else np.asarray(allowed, dtype=np.int64)
    U = ps.full_couplings(J, L, q)
    rows = np.arange(C)
    settled = np.zeros(C, dtype=bool)
    for _ in range(int(max_sweeps)):
        moved = np.zeros(C, dtype=bool)
        for k, i in enumerate(free):
            ok = (int(masks[k]) >> np.arange(q)) & 1 == 1
            z = h[i][None, :] + sum(U[i, :, j, s[:, j]] for j in range(L) if j != i)
            v = np.where(ok[None, :], z, -np.inf)
            top = v == v.max(axis=1, keepdims=True)
            b = np.where(top[rows, s[:, i]], s[:, i], top.argmax(axis=1))
            moved |= b != s[:, i]
            s[:, i] = b
        settled = ~moved
        if settled.all():
            break
    return s, settled


def anneal_record(h, J, seed, n_chains, schedule, init=None):
    """Chains of potts_sampler.Sampler, one sweep at each inverse temperature of ``schedule``, each keeping the best
    state (float64 H, strictly greater) reached after a sweep.  Returns (best H, best codes)."""
    s = ps.Sampler(h, J, seed, n_chains, init=init)
    best_E = np.full(n_chains, -np.inf)
    best = s.codes().astype(np.int64)
    for b in schedule:
        s.run(1, float(b))
        c = s.codes().astype(np.int64)
        E = ps.energies(h, J, c)
        up = E > best_E
        best_E[up], best[up] = E[up], c[up]
    return best_E, best
