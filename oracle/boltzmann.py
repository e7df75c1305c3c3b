"""
Float64 restatement of the library's Boltzmann-machine learning (evc_code_counts, evc_bm_update,
model_ops.BoltzmannLearner; contract in include/evcplm.h), driven by the Gibbs-chain restatement of
oracle/potts_sampler.py, and the exact regularised-likelihood optimum of models small enough to enumerate.  Test
infrastructure, not product code.
"""
import numpy as np

from . import potts_sampler as ps


def code_counts(codes, L, q):
    """uint32 counts of the rows of codes in x layout: [i q + a], then [pair i < j row-major][a][b]."""
    codes = np.asarray(codes, dtype=np.int64).reshape(-1, L)
    site = np.concatenate([np.bincount(codes[:, i], minlength=q) for i in range(L)])
    iu, ju = np.triu_indices(L, 1)
    pair = [np.bincount(codes[:, i] * q + codes[:, j], minlength=q * q) for i, j in zip(iu, ju)]
    return np.concatenate([site] + pair).astype(np.uint32)


def update(x, counts, M, f, Lq, eta, lam2_h, lam2_J):
    """One evc_bm_update: returns (new x as float32, [max |c/M - f| over fields, over couplings]).  numpy float64
    rounds every operation on its own, which is the device's order: d = c/M - f, g = d + lam2 theta,
    theta - eta g, then round to fp32."""
    th = np.asarray(x, dtype=np.float32).astype(np.float64)
    d = np.asarray(counts, dtype=np.float64) / float(M) - np.asarray(f, dtype=np.float32).astype(np.float64)
    lam2 = np.full(len(th), float(lam2_J))
    lam2[:Lq] = float(lam2_h)
    g = d + lam2 * th
    new = (th - float(eta) * g).astype(np.float32)
    ad = np.abs(d)
    return new, np.array([ad[:Lq].max(initial=0.0), ad[Lq:].max(initial=0.0)])


class Sampler(ps.Sampler):
    """potts_sampler.Sampler with set_params: the restated chain keeps no field state (run() recomputes every Z from
    the codes in float64), so loading new parameters is replacing h and U."""

    def set_params(self, h, J):
        self.h = np.asarray(h, dtype=np.float64).reshape(self.L, self.q)
        self.U = ps.full_couplings(J, self.L, self.q)


def split(x, L, q):
    return x[:L * q].reshape(L, q), x[L * q:].reshape(-1, q, q)


def learn(x0, f, L, q, lam2_h, lam2_J, updates, n_chains, seed=0, sweeps=10, eta=0.05, burn_in=0, progress=None):
    """The update loop of model_ops.BoltzmannLearner from x0 (float32): burn-in sweeps, then per update S sweeps,
    exact counts, evc_bm_update and set_params.  progress(k, codes, stats) is called after each update's counts."""
    x = np.asarray(x0, dtype=np.float32).copy()
    s = Sampler(*split(x, L, q), seed, n_chains)
    if burn_in:
        s.run(burn_in)
    for k in range(updates):
        s.run(sweeps)
        codes = s.codes()
        x, stats = update(x, code_counts(codes, L, q), n_chains, f, L * q, eta, lam2_h, lam2_J)
        if progress is not None:
            progress(k, codes, stats)
        s.set_params(*split(x, L, q))
    return x


# ---- the exact optimum of small models ----------------------------------------------------------------------------

def features(L, q):
    """(q^L, n) 0/1 matrix: the one- and two-site indicators of every state in x layout (state order of
    potts_sampler.exact_distribution)."""
    states = np.array(np.unravel_index(np.arange(q ** L), (q,) * L)).T
    n = L * q + L * (L - 1) // 2 * q * q
    phi = np.zeros((len(states), n))
    rows = np.arange(len(states))
    for i in range(L):
        phi[rows, i * q + states[:, i]] = 1.0
    iu, ju = np.triu_indices(L, 1)
    for p, (i, j) in enumerate(zip(iu, ju)):
        phi[rows, L * q + p * q * q + states[:, i] * q + states[:, j]] = 1.0
    return phi


def exact_marginals(x, L, q):
    """E[phi] under P(s) ~ exp(H(s)) of x (float64, x layout)."""
    phi = features(L, q)
    e = phi @ np.asarray(x, dtype=np.float64)
    p = np.exp(e - e.max())
    return phi.T @ (p / p.sum())


def objective(theta, f, phi, lam_h, lam_J, Lq):
    """F(theta) = -theta.f + log Z + lam_h |h|^2 + lam_J |J|^2 and its exact gradient (float64)."""
    e = phi @ theta
    m = e.max()
    p = np.exp(e - m)
    Z = p.sum()
    lam = np.full(len(theta), lam_J)
    lam[:Lq] = lam_h
    F = -theta @ f + m + np.log(Z) + np.sum(lam * theta * theta)
    g = -f + phi.T @ (p / Z) + 2.0 * lam * theta
    return F, g


def optimum(f, L, q, lam_h, lam_J, tol=1e-13):
    """theta* = argmin F by scipy L-BFGS in float64 over all q^L states (q^L <= 4096); lam_h, lam_J are the lambda'
    of the contract (already divided by n_eff).  Returns (theta*, max |gradient| at theta*)."""
    from scipy.optimize import minimize
    if q ** L > 4096:
        raise ValueError("enumeration is for q^L <= 4096")
    phi = features(L, q)
    f = np.asarray(f, dtype=np.float64)
    r = minimize(objective, np.zeros(len(f)), args=(f, phi, lam_h, lam_J, L * q), jac=True, method="L-BFGS-B",
                 options=dict(maxiter=20000, maxcor=30, ftol=0.0, gtol=tol))
    theta = r.x
    lam = np.full(len(theta), lam_J)
    lam[:L * q] = lam_h
    for _ in range(20):                 # Newton polish with the exact Hessian Cov_P(phi) + 2 diag(lam)
        g = objective(theta, f, phi, lam_h, lam_J, L * q)[1]
        if np.abs(g).max() <= tol:
            break
        e = phi @ theta
        p = np.exp(e - e.max())
        p /= p.sum()
        mu = phi.T @ p
        H = (phi * p[:, None]).T @ phi - np.outer(mu, mu) + 2.0 * np.diag(lam)
        theta = theta - np.linalg.solve(H, g)
    return theta, float(np.abs(objective(theta, f, phi, lam_h, lam_J, L * q)[1]).max())


def hessian_max_eigenvalue(theta, L, q, lam_h, lam_J):
    """Largest eigenvalue of the Hessian of F at theta."""
    phi = features(L, q)
    e = phi @ theta
    p = np.exp(e - e.max())
    p /= p.sum()
    mu = phi.T @ p
    lam = np.full(len(theta), lam_J)
    lam[:L * q] = lam_h
    return float(np.linalg.eigvalsh((phi * p[:, None]).T @ phi - np.outer(mu, mu) + 2.0 * np.diag(lam))[-1])


def exact_descent(f, L, q, lam_h, lam_J, eta, updates):
    """The update of the contract with exact marginals in place of chain counts (M -> infinity), from theta = 0."""
    phi = features(L, q)
    theta = np.zeros(len(f))
    for _ in range(updates):
        theta = theta - eta * objective(theta, np.asarray(f, dtype=np.float64), phi, lam_h, lam_J, L * q)[1]
    return theta


# ---- statistics ---------------------------------------------------------------------------------------------------

def connected(f, L, q):
    """C_ij(a, b) = f_ij(a, b) - f_i(a) f_j(b) for pairs i < j, flattened (f in x layout)."""
    f = np.asarray(f, dtype=np.float64)
    fi, fij = f[:L * q].reshape(L, q), f[L * q:].reshape(-1, q, q)
    iu, ju = np.triu_indices(L, 1)
    return (fij - fi[iu][:, :, None] * fi[ju][:, None, :]).ravel()


def connected_pearson(f_model, f_data, L, q):
    """Pearson r of the connected correlations of two statistics vectors in x layout."""
    return float(np.corrcoef(connected(f_model, L, q), connected(f_data, L, q))[0, 1])
