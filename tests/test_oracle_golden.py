"""
Pins the CPU oracle (oracle/) against the golden plmc run shipped with the
reference (notebooks/example/PABP_YEAST.*) and against outputs of the
reference's own in-tree Python twins; fixtures made by tests/golden/make_golden.py.
"""
import os

import numpy as np
import pytest

from oracle import c_oracle as co
from oracle import plm_oracle as po

import golden_npz


@pytest.fixture(scope="module")
def pabp(golden_dir):
    c = golden_npz.load("pabp_codes")
    g = golden_npz.load("pabp_golden")
    valid = np.unpackbits(c["valid_packed"])[: int(c["n_total"])].astype(bool)
    return dict(codes=c["codes"], valid=valid, counts_all=c["golden_counts_all"], g=g, c=c)


def test_pabp_validity_and_header(pabp):
    g = pabp["g"]
    L, q, nv, ni, it = g["hdr_i"]
    assert (L, q, nv, ni, it) == (82, 20, 151496, 545, 200)
    assert pabp["codes"].shape == (nv, L)
    assert pabp["valid"].sum() == nv and (~pabp["valid"]).sum() == ni
    # golden `weights` = integer neighbour counts, zero exactly on the invalid rows
    assert (pabp["counts_all"][~pabp["valid"]] == 0).all()
    assert (pabp["counts_all"][pabp["valid"]] >= 1).all()
    assert str(pabp["c"]["target_seq"]) == str(g["target_seq"])
    assert (pabp["c"]["index_list"] == g["index_list"]).all()
    assert int(pabp["c"]["region_start"]) == 115
    # theta stored in plmc convention (1 - 0.8)
    assert abs(float(g["hdr_f"][0]) - 0.2) < 1e-7


def test_pabp_hamming_counts_exact(pabp):
    """hot path (b): exact integer equality with the counts plmc stored."""
    codes = pabp["codes"]
    gold = pabp["counts_all"][pabp["valid"]]
    thr = po.identity_threshold_count(0.8, codes.shape[1])
    assert thr == 66
    for r0, r1 in [(0, 3000), (70000, 73000), (148496, 151496)]:
        got = co.hamming_counts(codes, thr, rows=(r0, r1))
        assert (got == gold[r0:r1]).all()
    n_eff = (1.0 / gold.astype(np.float64)).sum()
    assert abs(n_eff - float(pabp["g"]["hdr_f"][4])) < 0.01


def test_pabp_frequencies(pabp):
    """row a6: f_i and f_ij (ignore_gaps normalisation) <= 1e-6 of golden."""
    g = pabp["g"]
    codes = pabp["codes"]
    q = 20
    w = 1.0 / pabp["counts_all"][pabp["valid"]].astype(np.float64)
    fi = np.zeros((codes.shape[1], q))
    for a in range(q):
        fi[:, a] = ((codes == a) * w[:, None]).sum(axis=0)
    fi /= fi.sum(axis=1, keepdims=True)
    assert np.abs(fi - g["fi"]).max() < 1e-6
    for (i, j), blk in zip(g["fij_pairs"], g["fij_blocks"]):
        ci, cj = codes[:, i].astype(np.int64), codes[:, j].astype(np.int64)
        m = (ci < q) & (cj < q)
        F = np.bincount(ci[m] * q + cj[m], weights=w[m], minlength=q * q).reshape(q, q)
        F /= F.sum()
        assert np.abs(F - blk).max() < 1e-6


def test_pabp_frequencies_function_subset(pabp):
    """po.frequencies agrees with the direct statement above on a subsample."""
    codes = pabp["codes"][:1500, :12]
    w = np.random.default_rng(0).uniform(0.1, 1.0, size=len(codes))
    fi, fij = po.frequencies(codes, w, 20, gap_code=20)
    q = 20
    ci, cj = codes[:, 2].astype(np.int64), codes[:, 7].astype(np.int64)
    m = (ci < q) & (cj < q)
    F = np.bincount(ci[m] * q + cj[m], weights=w[m], minlength=q * q).reshape(q, q)
    F /= F.sum()
    iu, ju = np.triu_indices(12, 1)
    k = np.nonzero((iu == 2) & (ju == 7))[0][0]
    assert np.abs(fij[k] - F).max() < 1e-12


def test_pabp_ec_scores_from_golden_J(pabp):
    """row a10: cn = APC(Frobenius norm) in the file's gauge reproduces _ECs.txt."""
    g = pabp["g"]
    cn = po.cn_scores(g["J"], 82)
    assert np.sqrt(np.mean((cn - g["ec_cn"]) ** 2)) < 1e-6
    assert np.abs(cn - g["ec_cn"]).max() < 2e-6
    # the reference's CouplingsModel.cn_scores (zero-sum gauge first) is a DIFFERENT score
    assert np.sqrt(np.mean((g["ref_cn_zero_sum"] - g["ec_cn"]) ** 2)) > 1e-3
    iu, ju = np.triu_indices(82, 1)
    assert (g["index_list"][iu] == g["ec_i"]).all() and (g["index_list"][ju] == g["ec_j"]).all()
    ts = str(g["target_seq"])
    assert all(ts[i] == a for i, a in zip(iu[:200], g["ec_Ai"][:200]))


def test_pabp_reader_kats(pabp):
    g = pabp["g"]
    iu, ju = np.triu_indices(82, 1)
    ts = str(g["target_seq"])
    alph = str(g["alphabet"])
    i, j = 127 - 123, 172 - 123
    k = np.nonzero((iu == i) & (ju == j))[0][0]
    assert abs(g["J"][k][alph.index(ts[i]), alph.index(ts[j])] - float(g["kat_Jij_127_172"])) < 1e-7
    assert abs(g["h"][i, alph.index(ts[i])] - float(g["kat_hi_127"])) < 1e-7
    # notebook KATs (model_parameters_mutation_effects.ipynb): hi(127)=0.30619758, Jij(127,172)=-0.2060956
    assert abs(float(g["kat_hi_127"]) - 0.30619758) < 1e-6
    assert abs(float(g["kat_Jij_127_172"]) + 0.2060956209897995) < 1e-6


@pytest.mark.slow
def test_pabp_objective_scaling_at_golden_optimum(pabp):
    """row a7: at plmc's (unconverged, 200-iteration) optimum the data gradient
    balances 2*lambda_J*J: per-block median ratio in [0.9, 1.1].  Rules out a
    1/2 lambda coefficient (0.5) and an N_eff-normalised likelihood (~5e-5)."""
    g = pabp["g"]
    codes = pabp["codes"]
    w = 1.0 / pabp["counts_all"][pabp["valid"]].astype(np.float64)
    L, q = 82, 20
    x = np.concatenate([g["h"].ravel(), g["J"].ravel()]).astype(np.float64)
    fx, grad, nll = co.plm_eval(codes, w, x, q, 0.0, 0.0, precision="f64")
    gJ = grad[L * q:].reshape(-1, q, q)
    lamJ = float(g["hdr_f"][2])
    for k in g["fij_pair_index"]:
        J = g["J"][k].astype(np.float64)
        m = np.abs(J) > 0.02
        ratio = (-gJ[k][m]) / (2 * lamJ * J[m])
        assert 0.9 < np.median(ratio) < 1.1
    # h rows are centred by the L2 penalty (sum_a h_i(a) ~ 0)
    assert np.abs(g["h"].sum(axis=1)).max() < 1e-4


def test_intree_twins(golden_dir):
    """Oracle vs the reference's numba twins (alignment.py:1078-1233), gap-as-state."""
    d = np.load(os.path.join(golden_dir, "intree_twins.npz"))
    for name in ("cfg1", "tie", "odd"):
        codes = d[name + "_codes"]
        theta = float(d[name + "_theta"])
        counts = po.hamming_counts(codes, theta)
        assert (counts == d[name + "_counts"]).all()
        thr = po.identity_threshold_count(theta, codes.shape[1])
        assert (co.hamming_counts(codes, thr) == d[name + "_counts"]).all()
        w = 1.0 / counts
        fi, fij = po.frequencies(codes, w, 21)
        assert np.abs(fi - d[name + "_fi"]).max() < 1e-12
        assert np.abs(fij - d[name + "_fij_tri"]).max() < 1e-12
    # theta*L is an exact integer tie for cfg1 (0.8*40) and tie (0.8*50): >= keeps the pair
    assert po.identity_threshold_count(0.8, 40) == 32
    assert po.identity_threshold_count(0.8, 50) == 40
    assert po.identity_threshold_count(0.8, 82) == 66
    assert po.identity_threshold_count(0.7, 33) == 24


def test_objective_vectorised_vs_loops_and_c():
    rng = np.random.default_rng(3)
    for q, gap_code in ((21, -1), (20, 20)):
        N, L = 23, 6
        codes = rng.integers(0, 21, size=(N, L)).astype(np.uint8)
        if gap_code >= 0:
            codes = np.where(codes == 0, 20, codes - 1).astype(np.uint8)
        w = rng.uniform(0.2, 1.0, N)
        n = L * q + L * (L - 1) // 2 * q * q
        x = rng.normal(0, 0.3, n)
        f1, g1, n1 = po.objective(x, codes, w, q, 0.01, 1.3, gap_code)
        f2, g2, n2 = po.objective_loops(x, codes, w, q, 0.01, 1.3, gap_code)
        assert abs(f1 - f2) < 1e-9 * abs(f2)
        assert np.abs(g1 - g2).max() < 1e-10
        f3, g3, n3 = co.plm_eval(codes, w, x, q, 0.01, 1.3, precision="f64")
        assert abs(f3 - f2) < 1e-9 * abs(f2) and abs(n3 - n2) < 1e-9 * abs(n2)
        assert np.abs(g3 - g2).max() < 1e-10
        f4, g4, n4 = co.plm_eval(codes, w, x, q, 0.01, 1.3, precision="f32")
        assert abs(f4 - f2) < 1e-5 * abs(f2)
        assert np.abs(g4 - g2).max() < 1e-4
        # finite differences
        for k in rng.integers(0, n, 6):
            e = np.zeros(n)
            e[k] = 1e-5
            fp = po.objective(x + e, codes, w, q, 0.01, 1.3, gap_code)[0]
            fm = po.objective(x - e, codes, w, q, 0.01, 1.3, gap_code)[0]
            assert abs((fp - fm) / 2e-5 - g1[k]) < 1e-5 * max(1.0, abs(g1[k]))


def test_tiny_model_layout_vs_reference_reader(golden_dir, tmp_path):
    """row a9: bytes written by the oracle writer were read by the reference's
    CouplingsModel (model.py:317-389); our bulk reader sees the same numbers."""
    r = np.load(os.path.join(golden_dir, "tiny_ref_read.npz"))
    m = po.read_model(os.path.join(golden_dir, "tiny.model"))
    assert m["L"] == int(r["ref_L"]) and m["q"] == int(r["ref_q"])
    assert np.array_equal(m["J"].astype(np.float64), r["ref_J_tri"])
    assert np.array_equal(m["h"].astype(np.float64), r["ref_h"])
    assert np.array_equal(m["fi"].astype(np.float64), r["ref_fi"])
    assert np.array_equal(m["fij"].astype(np.float64), r["ref_fij_tri"])
    assert m["alphabet"] == str(r["ref_alphabet"]) and m["target_seq"] == str(r["ref_target"])
    assert (m["index_list"] == r["ref_index_list"]).all()
    # Frobenius norms agree with the reference's fn_scores (raw gauge: model.py:805-827)
    L = m["L"]
    F = po.fn_scores(m["J"], L)
    iu, ju = np.triu_indices(L, 1)
    # reference fn_scores are computed after the zero-sum shift, so only the text ECs are comparable:
    cn = po.cn_scores(m["J"], L)
    assert np.abs(cn - r["ecs_cn"]).max() < 1e-6
    assert (r["ecs_i"] == m["index_list"][iu]).all() and (r["ecs_j"] == m["index_list"][ju]).all()
    assert F.shape == (L, L)
    # size formula of the layout
    sz = 40 + m["q"] + 4 * (m["n_valid"] + m["n_invalid"]) + L + 4 * L + 8 * L * m["q"] \
        + 8 * (L * (L - 1) // 2) * m["q"] ** 2
    assert os.path.getsize(os.path.join(golden_dir, "tiny.model")) == sz


def test_fit_reaches_stationary_point():
    codes = po.synthetic_msa_codes(80, 8, 5)
    counts = po.hamming_counts(codes, 0.8)
    w = po.sequence_weights(counts)
    x, res = po.fit(codes, w, 21, 0.01, 0.5, max_iter=2000)
    fx, g, _ = po.objective(x, codes, w, 21, 0.01, 0.5)
    assert np.abs(g).max() < 1e-5
