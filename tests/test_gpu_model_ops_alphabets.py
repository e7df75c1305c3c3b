"""
Model consumers at every alphabet size (-m gpu): statistical energies (model_ops.hamiltonians, evc_plm_energies:
plm_energy_kernel<21> for q = 20 / 21 and <5> for q = 4 / 5) and EC block scores (model_ops.pair_scores,
evc_ec_scores: raw and zero-sum Frobenius norms, mutual information), every row against float64 numpy.
Shapes: L = 2 (one pair), 23 / 24 / 25 around the 24-site shared-memory chunk EN_JC of the energy kernel, 49
(three chunks); N = 1 and 511 / 512 / 513 around the 512 sequences of one energy CTA.
"""
import numpy as np
import pytest

from oracle import plm_oracle as po

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine():
    from evcouplings_b200 import _lib
    from evcouplings_b200.engine import CudaEngine
    _lib.require_device()
    return CudaEngine()


def _model(L, q, seed):
    rng = np.random.default_rng(seed)
    npair = L * (L - 1) // 2
    fi = rng.dirichlet(np.ones(q), size=L).astype(np.float32)
    fij = rng.dirichlet(np.ones(q * q), size=npair).reshape(npair, q, q).astype(np.float32)
    fi[0, : q // 2] = 0.0                               # MI: some zero f_i and f_ij entries
    fij[:, 0, :] = 0.0
    fij[0, :, 1] = 0.0
    return dict(L=L, q=q, h=rng.normal(0, 0.5, (L, q)).astype(np.float32),
                J=rng.normal(0, 0.2, (npair, q, q)).astype(np.float32), fi=fi, fij=fij)


@pytest.mark.parametrize("gaps", [False, True])
@pytest.mark.parametrize("q", [4, 5, 20, 21])
@pytest.mark.parametrize("L", [2, 23, 24, 25, 49])
def test_hamiltonians_every_row(engine, L, q, gaps):
    from evcouplings_b200 import model_ops
    m = _model(L, q, 100 * L + q)
    J = po.full_couplings(m["J"].astype(np.float64), L, q)
    Jp = np.zeros((L, L, q + 1, q + 1))                 # gap symbol q: row / column of zeros
    Jp[:, :, :q, :q] = J
    hp = np.zeros((L, q + 1))
    hp[:, :q] = m["h"]
    rng = np.random.default_rng(L + q)
    for N in (1, 511, 512, 513):
        codes = rng.integers(0, q, size=(N, L)).astype(np.uint8)
        if gaps:
            codes[rng.random((N, L)) < 0.15] = q
            codes[0, :] = q                             # one sequence of gaps only
        H = model_ops.hamiltonians(m, codes, engine)
        i, j = np.triu_indices(L, 1)
        terms = Jp[i[None, :], j[None, :], codes[:, i], codes[:, j]]          # N x npair
        hj, hh = terms.sum(axis=1), hp[np.arange(L)[None, :], codes].sum(axis=1)
        scale = np.abs(terms).sum(axis=1) + np.abs(hp[np.arange(L)[None, :], codes]).sum(axis=1)
        # per-site float32 partial sums of at most L - 1 couplings, then float64: L * 2^-24 of the |terms|
        tol = L * 2.0 ** -24 * scale + 1e-12
        for col, ref in ((0, hj + hh), (1, hj), (2, hh)):
            bad = np.nonzero(np.abs(H[:, col] - ref) > tol)[0]
            assert len(bad) == 0, (L, q, gaps, N, col, bad[:5], H[bad[:5], col], ref[bad[:5]])
        if gaps:
            assert H[0, 0] == 0.0 and H[0, 1] == 0.0 and H[0, 2] == 0.0


@pytest.mark.parametrize("q", [4, 5, 20, 21])
@pytest.mark.parametrize("L", [2, 23, 24, 25, 49])
def test_pair_scores_every_pair(engine, L, q):
    from evcouplings_b200 import model_ops
    m = _model(L, q, 7 * L + q)
    fn_raw, fn_zs, mi = model_ops.pair_scores(m, engine)
    J = m["J"].astype(np.float64)
    raw = np.sqrt((J ** 2).sum(axis=(1, 2)))
    Jz = J - J.mean(axis=1, keepdims=True) - J.mean(axis=2, keepdims=True) + J.mean(axis=(1, 2), keepdims=True)
    zs = np.sqrt((Jz ** 2).sum(axis=(1, 2)))
    i, j = np.triu_indices(L, 1)
    F = m["fij"].astype(np.float64)
    P = m["fi"].astype(np.float64)[i][:, :, None] * m["fi"].astype(np.float64)[j][:, None, :]
    ok = (F > 0) & (P > 0)
    t = np.where(ok, F * np.log(np.where(ok, F, 1.0) / np.where(ok, P, 1.0)), 0.0)
    mi_ref = t.sum(axis=(1, 2))
    # float64 on the device, rounded once to float32
    assert (np.abs(fn_raw - raw) <= 2.0 ** -23 * raw + 1e-30).all()
    assert (np.abs(fn_zs - zs) <= 2.0 ** -23 * zs + 1e-12 * raw).all()
    assert (np.abs(mi - mi_ref) <= 2.0 ** -23 * np.abs(mi_ref) + 1e-12 * np.abs(t).sum(axis=(1, 2))).all()
    assert (ok.sum(axis=(1, 2)) < q * q).all()        # the zero entries were skipped, not all of them
