"""
The stage references of oracle/tc_stages.py (no GPU): composed they reproduce the float64 rounding model of the
whole evaluation (po.objective(operands=...)) and of the counts (po.frequencies(weights="hi+lo")); the padded row
map is expand_row<true>; the buffers of generate mode pass every check; and every plausible kernel mistake of
MUTATIONS fails a check that names its stage and an element.
"""
import numpy as np
import pytest
import torch

from evcouplings_b200 import synthetic
from oracle import plm_oracle as po
from oracle import tc_stages as ts


def inputs(N=300, L=10, q=21, gap=False, seed=3):
    codes = synthetic.synthetic_msa_codes(N, L, seed)
    if gap:
        codes = synthetic.to_ignore_gaps_codes(codes, q)
    rng = np.random.default_rng(seed)
    w = rng.uniform(0.05, 1.0, N).astype(np.float32)
    x = rng.normal(0, 0.3, L * q + L * (L - 1) // 2 * q * q).astype(np.float32)
    return np.ascontiguousarray(codes), w, x


def test_rn_bf16_matches_the_bit_operation():
    v = np.random.default_rng(0).normal(0, 1, 100000).astype(np.float32) * np.float32(3.0) ** np.arange(-20, 20)[
        np.arange(100000) % 40].astype(np.float32)
    assert np.array_equal(ts.rn_bf16(torch.from_numpy(v)).float().numpy(), po.rn_bf16(v))


def test_padded_row_map_is_expand_row_padded():
    """expand_row<true>: (i / 8) * 176 + ((i % 8) / 4) * 88 + (i % 4) * 21 + a; every row of a 176-row tile is hit at
    most once, 84 per 88-row half, the last 4 of each half never"""
    L, q = 19, 21
    m = ts.padded_rows(L, q)
    for i in range(L):
        for a in range(q):
            assert int(m[i, a]) == (i // 8) * 176 + ((i % 8) // 4) * 88 + (i % 4) * 21 + a
    flat = m.reshape(-1)
    assert len(set(flat.tolist())) == L * q
    assert all(r % 88 < 84 for r in flat.tolist())


@pytest.mark.parametrize("q,gap,single", [(21, False, False), (21, False, True), (20, True, False), (4, True, True)])
def test_stage_references_compose_to_the_rounding_model(q, gap, single):
    """expand -> logits (float64 of the operand) -> softmax -> backward -> finalize in float64 is
    po.objective(operands=...) to float64 rounding; the counts' residual operand gives po.frequencies(weights=hi+lo)"""
    codes, w, x = inputs(N=257, L=9, q=q, gap=gap)
    gap_code = q if gap else -1
    N, L = codes.shape
    Lq = L * q
    c = torch.from_numpy(codes.astype(np.int64))
    xt = torch.from_numpy(x)
    v = ts.coupling_rows(xt, L, q, torch.arange(Lq))
    hi, lo = ts.split_hi_lo(v)
    Z, _A = ts.logits_ref(hi, None if single else lo, c, q)
    z = Z.T.reshape(N, L, q) + xt[:Lq].double().view(1, L, q)
    r, _rb, fx, _fxb = ts.softmax_ref(z, c, torch.from_numpy(w), q)
    R = r.reshape(N, Lq).T
    Rop = torch.from_numpy(po.bf16_operand(R.numpy(), "hi" if single else "hi+lo"))
    G = ts.one_hot(c, q).T @ Rop.T
    Gf = G.to(torch.float64).reshape(1, Lq, Lq)
    S4 = Gf[0].reshape(L, q, L, q)
    iu, ju = torch.triu_indices(L, L, 1)
    gJ = S4[ju, :, iu, :].transpose(1, 2) + S4[iu, :, ju, :]
    fx_m, g_m, nll_m = po.objective(x.astype(np.float64), codes, w.astype(np.float64), q, 0.0, 0.0, gap_code,
                                    operands="hi" if single else "hi+lo")
    g = np.concatenate([r.sum(dim=0).reshape(-1).numpy(), gJ.reshape(-1).numpy()])
    assert np.allclose(g, g_m, rtol=1e-12, atol=1e-12 * np.abs(g_m).max())
    assert abs(fx.sum().item() - nll_m) <= 1e-12 * abs(nll_m)
    # counts: f_ij from the exact counts residual through the same product
    chi, clo = ts.counts_residual(c, torch.from_numpy(w), q)
    F = ts.one_hot(c, q).T @ ts.bf16_value(chi, clo).T
    F4 = F.reshape(L, q, L, q)
    fij = 0.5 * (F4[ju, :, iu, :].transpose(1, 2) + F4[iu, :, ju, :])
    _fi, fij_m = po.frequencies(codes, w.astype(np.float64), q, gap_code, weights="hi+lo")
    if gap_code < 0:
        fij = fij / w.astype(np.float64).sum()
    else:
        fij = fij / fij.sum(dim=(1, 2), keepdim=True).clamp_min(1e-300)
    assert np.allclose(fij.numpy(), fij_m, rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("single", [False, True])
def test_generate_mode_passes_every_check(single):
    codes, w, x = inputs(N=300, L=10)
    buf = ts.generate(x, codes, w, 21, single=single)
    rep = ts.check_generated(buf, x, codes, w, 21)
    print("\n".join(rep.lines()))
    assert {"expand", "Xt", "logits", "softmax Rt", "softmax gh_part", "backward", "finalize_pairs",
            "finalize_fields", "counts Rt", "counts backward"} <= set(rep)
    for stage, (n, ratio) in rep.items():
        assert n > 0 and (ratio is None or ratio <= 1.0), stage


def test_counts_gh_part_replay_matches_a_plain_float32_reference():
    """the butterfly replay is a float32 sum of the tile's weights per state: equal to float64 within 10 u"""
    codes, w, _x = inputs(N=700, L=6, q=21)
    c = torch.from_numpy(codes.astype(np.int64))
    gh = ts.counts_gh_replay(c, torch.from_numpy(w), 21, 21, 3).double()
    X = ts.one_hot(c, 21).view(700, 6, 21) * torch.from_numpy(w).double().view(-1, 1, 1)
    ref = torch.nn.functional.pad(X, (0, 0, 0, 0, 0, 68)).view(3, 256, 6, 21).sum(dim=1).permute(1, 0, 2)
    assert ((gh - ref).abs() <= 10 * 2.0 ** -24 * ref.abs()).all()


# the stage each mistake is caught at: the first check of check_generated that sees it
EXPECTED_STAGE = {
    "expand_hi_rz": "expand hi",
    "rt_lo_dropped": "softmax Rt",
    "rt_hi_rz": "softmax Rt_hi",
    "onehot_wrong_state": "softmax Rt",
    "gd_block_transposed": "backward plane 0",
    "plane_order_reversed": "finalize_pairs",
    "gh_tile_off_by_one": "softmax gh_part",
    "fx_local_float": "softmax fx_part",
    "stale_rt_meets_xt": "Xt",
}


@pytest.mark.parametrize("mutation", ts.MUTATIONS)
def test_every_mutation_fails_at_its_stage(mutation):
    codes, w, x = inputs(N=300, L=10)
    buf = ts.generate(x, codes, w, 21, mutation=mutation)
    with pytest.raises(ts.StageMismatch) as e:
        ts.check_generated(buf, x, codes, w, 21)
    print(mutation, "->", e.value)
    assert e.value.stage == EXPECTED_STAGE[mutation], str(e.value)
    assert len(e.value.index) >= 1


def test_stale_residual_meeting_nonzero_xt_fails_the_backward_check():
    """the backward check on its own (Xt taken as the device wrote it) sees the stale column's contribution"""
    codes, w, x = inputs(N=300, L=10)
    buf = ts.generate(x, codes, w, 21, mutation="stale_rt_meets_xt")
    Lq = 210
    with pytest.raises(ts.StageMismatch) as e:
        ts.check_backward(ts.Report(), buf["Gd"], 10, 21, 300, ts.xt_columns(buf["Xt"], Lq),
                          ts.rt_columns(buf["Rt_hi"], buf["Rt_lo"], Lq), ksplit=3, num_kb=buf["Kp"] // 64)
    assert e.value.stage.startswith("backward")


def test_float_fx_local_fails_on_a_larger_alignment():
    """fx_local as a float: each warp's sum becomes a float32 number, but the double combine of the 4 warps leaves
    only about a quarter of the partials float32 numbers, and the error stays inside the bound.  The check on the
    partials' significant bits still fails it (N = 2048, L = 60: 480 partials)."""
    codes, w, x = inputs(N=2048, L=60, seed=4)
    good = ts.generate(x, codes, w, 21, ksplit=1)
    ts.check_generated(good, x, codes, w, 21)
    buf = ts.generate(x, codes, w, 21, ksplit=1, mutation="fx_local_float")
    f = buf["fx_part"]
    share = float((f.to(torch.float32).to(torch.float64) == f).double().mean())
    assert 0.05 < share < 0.6, share
    with pytest.raises(ts.StageMismatch) as e:
        ts.check_generated(buf, x, codes, w, 21)
    assert e.value.stage == "softmax fx_part" and "float32 numbers" in str(e.value)
