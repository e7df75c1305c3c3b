"""
The operand-rounding model of the float64 oracle (CPU only): ``rn_bf16`` / ``bf16_operand`` and the ``operands=``
argument of ``po.objective`` (the arithmetic of the tensor-core path: bf16 couplings and residuals, exact one-hot,
sums in float64) and ``weights=`` of ``po.frequencies``.  The GPU tests of tests/test_gpu_tc_edges.py compare the
device with this model, so the model itself is pinned here against torch's bfloat16 conversion and against the
exact objective.
"""
import numpy as np
import pytest
import torch

from evcouplings_b200 import synthetic
from oracle import plm_oracle as po


def _torch_bf16(v):
    return torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32)).to(torch.bfloat16).float().numpy()


def _same_bits(a, b):
    a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    nan = np.isnan(a)
    return np.array_equal(nan, np.isnan(b)) and np.array_equal(a[~nan].view(np.uint32), b[~nan].view(np.uint32))


def test_rn_bf16_matches_torch_on_random_values():
    rng = np.random.default_rng(0)
    # random float32 bit patterns (every exponent, subnormals, infinities and NaNs included) ...
    bits = rng.integers(0, 2 ** 32, size=500_000, dtype=np.uint64).astype(np.uint32)
    a = bits.view(np.float32)
    # ... and values of the sizes the kernels round: couplings, residuals, weights
    b = (rng.normal(size=500_000) * 10.0 ** rng.uniform(-6, 2, size=500_000)).astype(np.float32)
    for v in (a, b):
        assert _same_bits(po.rn_bf16(v), _torch_bf16(v))


def test_rn_bf16_edges():
    f32 = np.float32
    one_ulp = np.finfo(f32).eps                  # 2^-23
    tiny = np.finfo(f32).smallest_subnormal
    vals = []
    for hi in (0x3F80, 0x3F81, 0x4000, 0x4001, 0x7F7F, 0x0001, 0x0000, 0x807F, 0xBF80, 0xBF81):
        for lo in (0x0000, 0x0001, 0x7FFF, 0x8000, 0x8001, 0xFFFF):    # exact ties at 0x8000
            vals.append(((hi << 16) | lo))
    edges = np.array(vals, dtype=np.uint32).view(np.float32)
    specials = np.array([0.0, -0.0, 1.0, -1.0, 1.0 + one_ulp, 1.0 - one_ulp / 2, 2.0 - one_ulp, 2.0 + 2 * one_ulp,
                         0.5 - one_ulp / 4, tiny, -tiny, 2 * tiny, np.finfo(f32).tiny, np.finfo(f32).tiny * (1 - 2 ** -10),
                         np.finfo(f32).max, -np.finfo(f32).max, 3.3895314e38, 3.3961776e38, np.inf, -np.inf, np.nan],
                        dtype=f32)
    powers = np.ldexp(np.float32(1.0), np.arange(-149, 128)).astype(f32)
    near = np.concatenate([np.nextafter(powers, f32(0)), powers, np.nextafter(powers, f32(np.inf))])
    for v in (edges, specials, near, -near):
        assert _same_bits(po.rn_bf16(v), _torch_bf16(v))
    # ties go to the even neighbour; +-0 keep their sign; the largest float32 values overflow to infinity
    assert po.rn_bf16(np.array([0x3F808000], np.uint32).view(f32))[0] == np.float32(1.0)
    assert po.rn_bf16(np.array([0x3F818000], np.uint32).view(f32))[0] == np.array([0x3F820000], np.uint32).view(f32)[0]
    assert np.signbit(po.rn_bf16(np.array([-0.0], f32)))[0]
    assert np.isinf(po.rn_bf16(np.array([np.finfo(f32).max], f32)))[0]


def test_bf16_operand_error_per_operand():
    rng = np.random.default_rng(1)
    v = (rng.normal(size=200_000) * 10.0 ** rng.uniform(-5, 1, size=200_000)).astype(np.float32).astype(np.float64)
    hl = po.bf16_operand(v, "hi+lo")
    hi = po.bf16_operand(v, "hi")
    # hi + lo keeps 16 mantissa bits: |error| <= 2^-17 |v| (within the 2^-16 the path is specified with)
    assert (np.abs(hl - v) <= 2.0 ** -17 * np.abs(v)).all()
    # hi alone: round to nearest with 8 significant bits, |error| <= 2^-8 |v|, and some operands need all of it
    rel = np.abs(hi - v) / np.abs(v)
    assert rel.max() <= 2.0 ** -8 and rel.max() > 0.9 * 2.0 ** -8
    assert 2.0 ** -11 < np.sqrt(np.mean(rel ** 2)) < 2.0 ** -8
    with pytest.raises(ValueError):
        po.bf16_operand(v, "lo")


def _case(N=60, L=7, q=21, seed=3, gap=False, xscale=0.3):
    codes = synthetic.synthetic_msa_codes(N, L, seed)
    if gap:
        codes = synthetic.to_ignore_gaps_codes(codes)
    rng = np.random.default_rng(seed)
    w = rng.uniform(0.05, 1.0, N).astype(np.float32).astype(np.float64)
    x = rng.normal(0, xscale, L * q + L * (L - 1) // 2 * q * q).astype(np.float32).astype(np.float64)
    return codes, w, x


@pytest.mark.parametrize("q,gap", [(21, False), (20, True)])
def test_objective_exact_operands_unchanged(q, gap):
    codes, w, x = _case(q=q, gap=gap)
    gc = q if gap else -1
    fx, g, nll = po.objective(x, codes, w, q, 0.01, 0.5, gc)
    fx0, g0, nll0 = po.objective(x, codes, w, q, 0.01, 0.5, gc, operands=None)
    assert fx == fx0 and nll == nll0 and np.array_equal(g, g0)
    fl, gl, nl = po.objective_loops(x, codes, w, q, 0.01, 0.5, gc)
    assert abs(fx - fl) <= 1e-12 * abs(fl) and abs(nll - nl) <= 1e-12 * abs(nl)
    assert np.abs(g - gl).max() <= 1e-12 * np.abs(gl).max()
    # the error-model scales leave the result alone
    fb, gb, nb, bnd = po.objective(x, codes, w, q, 0.01, 0.5, gc, operands="hi+lo", bounds=1e-6)
    fh, gh, nh = po.objective(x, codes, w, q, 0.01, 0.5, gc, operands="hi+lo")
    assert fb == fh and nb == nh and np.array_equal(gb, gh)


def test_objective_operand_modes_against_a_loop_statement():
    """operands="hi+lo" / "hi" against the pure-loop objective fed with the rounded couplings, plus the rounded
    residuals in the pair gradient written out by hand: the model rounds exactly these two operands"""
    N, L, q = 20, 5, 21
    codes, w, x = _case(N=N, L=L, q=q, seed=5)
    for mode in ("hi+lo", "hi"):
        fx, g, nll = po.objective(x, codes, w, q, 0.0, 0.0, operands=mode)
        h, Jt = po.unpack(x, L, q)
        Jr = po.full_couplings(po.bf16_operand(Jt, mode), L, q)
        gJf = np.zeros_like(Jr)
        gh = np.zeros((L, q))
        f = 0.0
        for s in range(N):
            for i in range(L):
                z = h[i] + sum(Jr[i, j, :, codes[s, j]] for j in range(L) if j != i)
                p = np.exp(z - z.max()) / np.exp(z - z.max()).sum()
                f -= w[s] * np.log(p[codes[s, i]])
                r = w[s] * p
                r[codes[s, i]] -= w[s]
                gh[i] += r
                rop = po.bf16_operand(r, mode)
                for j in range(L):
                    if j != i:
                        gJf[i, j, :, codes[s, j]] += rop
        iu, ju = np.triu_indices(L, 1)
        gJ = gJf[iu, ju] + gJf[ju, iu].transpose(0, 2, 1)
        assert abs(fx - f) <= 1e-12 * abs(f) and abs(nll - f) <= 1e-12 * abs(f)
        assert np.abs(g[:L * q] - gh.ravel()).max() <= 1e-12 * np.abs(gh).max()
        assert np.abs(g[L * q:] - gJ.ravel()).max() <= 1e-12 * np.abs(gJ).max()


@pytest.mark.parametrize("q,gap", [(21, False), (20, True), (5, False)])
def test_objective_operand_modes_against_exact(q, gap):
    codes, w, x = _case(N=150, L=9, q=q, gap=gap, seed=7)
    if q == 5:
        codes = (codes % 5).astype(np.uint8)
    gc = q if gap else -1
    fx, g, nll = po.objective(x, codes, w, q, 0.0, 0.0, gc)
    out = {}
    for mode in ("hi+lo", "hi"):
        fm, gm, nm, bnd = po.objective(x, codes, w, q, 0.0, 0.0, gc, operands=mode, bounds=0.0)
        out[mode] = (abs(fm - fx) / abs(fx), np.linalg.norm(gm - g) / np.linalg.norm(g))
        # the sum of |terms| bounds every entry; without noise no operand can round differently
        assert (bnd["g_abs"] >= np.abs(gm) * (1 - 1e-12)).all() and (bnd["g_flip"] == 0).all()
    # hi + lo: 16 mantissa bits, the objective moves by O(2^-17); hi alone: 8 bits, O(2^-9)
    assert out["hi+lo"][0] < 2.0 ** -17 and out["hi+lo"][1] < 2.0 ** -15
    assert 2.0 ** -16 < out["hi"][1] < 2.0 ** -7 and out["hi"][0] < 2.0 ** -9
    assert out["hi"][1] > 30 * out["hi+lo"][1]


def test_flip_allowance_marks_operands_near_a_rounding_boundary():
    codes, w, x = _case(N=80, L=6, seed=9)
    _f, _g, _n, b0 = po.objective(x, codes, w, 21, 0.0, 0.0, operands="hi", bounds=0.0)
    _f, _g, _n, b1 = po.objective(x, codes, w, 21, 0.0, 0.0, operands="hi", bounds=2.0 ** -12)
    _f, _g, _n, b2 = po.objective(x, codes, w, 21, 0.0, 0.0, operands="hi", bounds=2.0 ** -16)
    _f, _g, _n, b3 = po.objective(x, codes, w, 21, 0.0, 0.0, operands="hi+lo", bounds=2.0 ** -12)
    assert (b0["g_flip"] == 0).all() and b2["g_flip"].max() > 0
    # a larger noise marks more operands
    assert (b2["g_flip"] <= b1["g_flip"]).all() and b2["g_flip"].sum() < 0.5 * b1["g_flip"].sum()
    # hi + lo follows the residual (16 bits): any noise moves every operand it touches
    nz = b3["g_abs"][21 * 6:] > 0
    assert (b3["g_flip"][21 * 6:][nz] > 0).all()


@pytest.mark.parametrize("gap", [False, True])
def test_frequencies_weights_hi_lo(gap):
    codes = synthetic.synthetic_msa_codes(500, 12, 4)
    if gap:
        codes = synthetic.to_ignore_gaps_codes(codes)
    q = 20 if gap else 21
    gc = q if gap else -1
    w = (1.0 / np.random.default_rng(4).integers(1, 40, 500)).astype(np.float32).astype(np.float64)
    fi, fij = po.frequencies(codes, w, q, gc)
    fi0, fij0 = po.frequencies(codes, w, q, gc, weights=None)
    assert np.array_equal(fi, fi0) and np.array_equal(fij, fij0)
    fi2, fij2 = po.frequencies(codes, w, q, gc, weights="hi+lo")
    assert np.array_equal(fi2, fi)                      # f_i takes the weights as given
    # f_ij: sums of positive weights, each within 2^-17 of its float32 value (two normalisations under ignore_gaps)
    rel = 2.0 ** -17 * (2 if gap else 1)
    assert (np.abs(fij2 - fij) <= rel * fij + 1e-300).all()
    assert np.abs(fij2 - fij).max() > 0                 # 1/k weights need more than 16 mantissa bits
