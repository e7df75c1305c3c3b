"""Conditional sampling on the device (evc_sampler_create_conditional, PottsSampler(free=, allowed=),
evcplm-sample --free/--allow): bit for bit the plain sampler when every site is free, the exact conditional
distribution by enumeration, the float64 restatement (oracle/conditional_sampler.py) draw for draw, its invariants,
a model beyond 2^31 floats that the plain sampler refuses, plmc's PABP model, several ranks and the command line."""
import ctypes
import io
import json
import os
import sys
import time

import numpy as np
import pytest

from evcouplings_b200 import _lib, model_io, model_ops, sample_cli, synthetic
from oracle import conditional_sampler as cs, potts_sampler as ps
from test_conditional_sampler_oracle import check_conditional, two_contexts
from test_potts_sampler_oracle import distribution_bounds, small_model

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# where the large-model test records its time and device memory, when set
RECORD = os.environ.get("EVC_CONDITIONAL_RECORD")


@pytest.fixture(scope="module")
def eng():
    from evcouplings_b200.engine import CudaEngine
    return CudaEngine()


def model_dict(h, J, alphabet=None):
    L, q = h.shape
    alphabet = alphabet or (synthetic.ALPHABET + "BJOUXZ12345")[:q]
    return dict(L=L, q=q, h=np.asarray(h, dtype=np.float32), J=np.asarray(J, dtype=np.float32), alphabet=alphabet,
                target_seq="".join(alphabet[(3 * i + 1) % q] for i in range(L)),
                index_list=np.arange(1, L + 1, dtype=np.int32))


def dyadic_model(L, q, seed, scale=1.0):
    """Fields N(0, 0.5) and couplings N(0, 0.05 scale), multiples of 2^-10: every fold, refresh and change the device
    forms is exact in fp32 (checked with potts_sampler.z_error_bound)."""
    rng = np.random.default_rng(seed)
    h = np.round(rng.normal(0, 0.5, (L, q)) * 1024) / 1024
    J = np.round(rng.normal(0, 0.05 * scale, (L * (L - 1) // 2, q, q)) * 1024) / 1024
    return h.astype(np.float32), J.astype(np.float32)


def positions(sites):
    return [int(k) + 1 for k in sites]          # model_dict's index_list is 1..L


def masks_to_letters(m, sites, masks):
    return {int(k) + 1: "".join(m["alphabet"][a] for a in range(m["q"]) if (int(mk) >> a) & 1)
            for k, mk in zip(sites, masks)}


# 1. with every site free and full masks the conditional handle is the plain one, bit for bit
@pytest.mark.parametrize("L,q,beta", [(12, 2, 1.0), (12, 21, 0.5), (12, 32, 1.0), (64, 21, 1.0), (64, 32, 0.5),
                                      (200, 21, 1.0), (200, 2, 0.5)])
@pytest.mark.parametrize("start", ["uniform", "given"])
def test_all_free_is_the_plain_sampler_bit_for_bit(eng, L, q, beta, start):
    h, J = dyadic_model(L, q, 7 * L + q)
    m = model_dict(h * 3.1, J * 7.3)                  # not dyadic: fp32 rounding everywhere
    n = 1000
    init = "random" if start == "uniform" else np.random.default_rng(L).integers(0, q, (n, L))
    with model_ops.PottsSampler(m, n, seed=5, init=init, chain_offset=3, engine=eng) as plain, \
            model_ops.PottsSampler(m, n, seed=5, init=init, chain_offset=3, engine=eng,
                                   free=range(1, L + 1)) as cond:
        assert cond.conditional and not plain.conditional
        assert np.array_equal(cond.codes(), plain.codes())
        assert np.array_equal(cond.conditional_fields(), np.repeat(m["h"][None], n, axis=0))
        a = plain.run(40, beta)
        b = cond.run(13, beta) + cond.run(27, beta)              # split across the refresh at t = 32
        assert a == b and np.array_equal(cond.codes(), plain.codes())


# 2. the exact conditional distribution, per-chain contexts, masks and single-state masks
@pytest.mark.parametrize("allowed", [None, [0b111, 0b101, 0b011], [0b010, 0b111, 0b110]])
def test_exact_conditionals(eng, allowed):
    L, q, beta = 6, 3, 1.0
    h, J = small_model(L, q, 60 + q)
    m = model_dict(h, J)
    free = np.array([1, 3, 4])
    n = 131072
    init, ctx = two_contexts(L, q, n, 5)
    letters = None if allowed is None else masks_to_letters(m, free, allowed)
    with model_ops.PottsSampler(m, n, seed=11, init=init, engine=eng, free=positions(free), allowed=letters) as s:
        s.run(32, beta)
        codes = s.codes().astype(np.int64)
    clamped = cs.clamped_sites(L, free)
    assert np.array_equal(codes[:, clamped], init[:, clamped])
    check_conditional(codes[:n // 2], h, J, beta, free, ctx[0], allowed)
    check_conditional(codes[n // 2:], h, J, beta, free, ctx[1], allowed)


# 3. draw for draw against the float64 restatement until each chain's first near tie
@pytest.mark.parametrize("nf", [1, 17, 39])
@pytest.mark.parametrize("beta", [1.0, 0.5])
def test_against_restatement(eng, nf, beta):
    L, q = 40, 21
    h, J = dyadic_model(L, q, 100 + nf)
    assert ps.z_error_bound(h, J, L, q, bits=10) == 0.0
    m = model_dict(h, J)
    rng = np.random.default_rng(nf)
    free = np.sort(rng.choice(L, nf, replace=False))
    masks = np.full(nf, (1 << q) - 1, dtype=np.int64)
    masks[::3] = rng.integers(1, 1 << q, len(masks[::3]))        # every third free site restricted
    if nf > 1:
        masks[1] = 1 << 7                                           # one single-state site
    n, sweeps, seed = 16 * 63 + 5, 40, 21                           # 16 chains per CTA, a last CTA of 5
    init = rng.integers(0, q, (n, L))
    hc = cs.fold(h, J, free, init)
    UFF = cs.reduced_couplings(J, L, q, free)
    margin = ps.near_tie_margin(q, 0.0, beta, cs.reduced_z_bounds(hc, UFF, q))
    ref = cs.ConditionalSampler(hc, UFF, free, L, seed, masks, init, margin=margin)
    compared = 0
    with model_ops.PottsSampler(m, n, seed=seed, init=init, engine=eng, free=positions(free),
                                allowed=masks_to_letters(m, free, masks)) as s:
        assert np.array_equal(s.conditional_fields(), hc.astype(np.float32))
        for t in range(sweeps):
            ch = s.run(1, beta)
            ref.run(1, beta)
            clean = (ref.first_tie < 0) | (ref.first_tie >= (t + 1) * L)
            same = np.all(s.codes() == ref.codes(), axis=1)
            assert same[clean].all(), (t, np.flatnonzero(clean & ~same)[:8])
            if clean.all():
                assert ch == ref.changes
            compared += int(clean.sum())
    # fixed on the CPU from the restatement alone: it keeps at least an eighth of the chain-sweeps before a near tie
    assert compared >= n * sweeps // 8, compared


# 4. invariants of a conditional handle
def test_invariants(eng):
    L, q = 30, 21
    h, J = dyadic_model(L, q, 3)
    m = model_dict(h * 3.1, J * 7.3)
    n = 2048
    rng = np.random.default_rng(4)
    init = rng.integers(0, q, (n, L)).astype(np.uint8)
    free = [3, 4, 5, 17, 29]
    sites = np.array(free) - 1
    allowed = {4: "ACD", 17: "W", 29: "KLMNPQ"}
    kw = dict(seed=9, engine=eng, free=free, allowed=allowed)
    with model_ops.PottsSampler(m, n, init=init, **kw) as a, model_ops.PottsSampler(m, n, init=init, **kw) as b:
        clamped = np.setdiff1d(np.arange(L), sites)
        for sweeps in (1, 12, 27):
            a.run(sweeps)
            c = a.codes()
            assert c.shape == (n, L) and np.array_equal(c[:, clamped], init[:, clamped])
            for p, letters in allowed.items():
                assert set(c[:, p - 1]) <= {m["alphabet"].index(x) for x in letters}
        b.run(40)
        assert np.array_equal(a.codes(), b.codes())
        whole = b.codes()
        with pytest.raises(ValueError, match="anneal"):
            a.anneal([0.0, 1.0])
        lib, dx = eng.lib, ctypes.c_void_p(256)
        assert lib.evc_sampler_set_model(a.handle, dx, None) == 1 and b"conditional" in lib.evc_last_error()
        betas = np.zeros(2, dtype=np.float32)
        assert lib.evc_sampler_anneal(a.handle, betas.ctypes.data_as(ctypes.c_void_p), 1, dx, None, None) == 1
        assert b"conditional" in lib.evc_last_error()
        assert np.array_equal(a.codes(), whole)                   # the refused calls changed nothing
    parts = []
    for off in (0, 1000):
        hi = 1000 if off == 0 else n
        with model_ops.PottsSampler(m, hi - off, init=init[off:hi], chain_offset=off, **kw) as p:
            p.run(40)
            parts.append(p.codes())
    assert np.array_equal(np.concatenate(parts), whole)
    with model_ops.PottsSampler(m, n, init=init, **kw) as again:
        again.run(40)
        assert np.array_equal(again.codes(), whole)
    with model_ops.PottsSampler(m, 8, seed=1, engine=eng) as plain:
        out = np.empty(1, dtype=np.float32)
        assert eng.lib.evc_sampler_conditional_fields(plain.handle, out.ctypes.data_as(ctypes.c_void_p), None) == 1


# 5. a model beyond 2^31 floats whose L q the plain sampler refuses
def test_large_model_beyond_int32_offsets(eng):
    import torch
    L, q = 3200, 21
    Lq, qq = L * q, q * q
    n_x = Lq + L * (L - 1) // 2 * qq
    assert n_x > 2 ** 31
    rng = np.random.default_rng(32)
    free = np.sort(np.concatenate([rng.choice(L - 8, 56, replace=False), np.arange(L - 8, L)]))
    pairs = set()
    for i in free:                                           # 4 partners per free site, free or clamped
        for j in rng.choice(L, 4, replace=False):
            if j != i:
                pairs.add((min(int(i), int(j)), max(int(i), int(j))))
    pairs.add((L - 2, L - 1))
    pairs = np.array(sorted(pairs))
    blocks = (np.round(rng.normal(0, 0.25, (len(pairs), q, q)) * 1024) / 1024).astype(np.float32)
    h = (np.round(rng.normal(0, 0.5, (L, q)) * 1024) / 1024).astype(np.float32)
    t0 = time.perf_counter()
    torch.cuda.reset_peak_memory_stats(eng.device)
    x = torch.zeros(n_x, dtype=torch.float32, device=eng.device)
    x[:Lq] = torch.from_numpy(h.ravel()).to(eng.device)
    offs = Lq + (pairs[:, 0] * L - pairs[:, 0] * (pairs[:, 0] + 1) // 2 + (pairs[:, 1] - pairs[:, 0] - 1)) * qq
    assert offs.max() > 2 ** 31
    idx = torch.from_numpy((offs[:, None] + np.arange(qq)[None, :]).ravel()).to(eng.device)
    x[idx] = torch.from_numpy(blocks.ravel()).to(eng.device)
    n = 256
    init = rng.integers(0, q, (n, L)).astype(np.uint8)
    lib = eng.lib
    handle = ctypes.c_void_p()
    vp = ctypes.c_void_p
    rc = lib.evc_sampler_create(ctypes.byref(handle), eng.ptr(x), L, q, init.ctypes.data_as(vp), n, 0, 1,
                                eng.device_index)
    assert rc == 1 and b"shared memory" in lib.evc_last_error()
    sites = np.ascontiguousarray(free, dtype=np.int32)
    masks = np.full(len(free), (1 << q) - 1, dtype=np.uint32)
    masks[-1] = 0b1011
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    _lib.check(lib.evc_sampler_create_conditional(ctypes.byref(handle), eng.ptr(x), L, q, sites.ctypes.data_as(vp),
                                                  len(sites), masks.ctypes.data_as(vp), init.ctypes.data_as(vp), n,
                                                  0, 7, eng.device_index), "evc_sampler_create_conditional")
    t_create = time.perf_counter() - t1
    try:
        hc_dev = torch.empty((n, len(free) * q), dtype=torch.float32, device=eng.device)
        _lib.check(lib.evc_sampler_conditional_fields(handle, eng.ptr(hc_dev), eng.stream()), "fields")
        hc = cs.fold_sparse(h, pairs, blocks, free, init)
        assert np.array_equal(hc_dev.cpu().numpy().reshape(n, len(free), q), hc.astype(np.float32))
        UFF = cs.reduced_couplings_sparse(L, q, pairs, blocks, free)
        margin = ps.near_tie_margin(q, 0.0, 1.0, cs.reduced_z_bounds(hc, UFF, q))
        ref = cs.ConditionalSampler(hc, UFF, free, L, 7, masks, init, margin=margin)
        codes = torch.empty((n, L), dtype=torch.uint8, device=eng.device)
        compared = 0
        t1 = time.perf_counter()
        for t in range(4):
            _lib.check(lib.evc_sampler_run(handle, 1, 1.0, None, eng.stream()), "evc_sampler_run")
            _lib.check(lib.evc_sampler_codes(handle, eng.ptr(codes), eng.stream()), "evc_sampler_codes")
            got = codes.cpu().numpy()
            ref.run(1)
            clean = (ref.first_tie < 0) | (ref.first_tie >= (t + 1) * L)
            same = np.all(got == ref.codes(), axis=1)
            assert same[clean].all(), (t, np.flatnonzero(clean & ~same)[:8])
            compared += int(clean.sum())
        assert compared >= n * 4 // 2, compared
        t_run = time.perf_counter() - t1
    finally:
        lib.evc_sampler_destroy(handle)
    peak = torch.cuda.max_memory_allocated(eng.device)
    free_b, total_b = torch.cuda.mem_get_info(eng.device)
    rec = dict(L=L, q=q, nf=len(free), n_chains=n, x_floats=n_x, create_s=round(t_create, 3),
               four_sweeps_with_copies_s=round(t_run, 3), test_s=round(time.perf_counter() - t0, 1),
               torch_peak_bytes=peak, device_used_bytes=total_b - free_b, device=torch.cuda.get_device_name(0))
    print("large conditional model:", json.dumps(rec))
    if RECORD:
        with open(RECORD, "w") as f:
            json.dump(rec, f)
    del x


# 6. plmc's PABP model, all but three sites clamped at the target, against enumeration of the 20^3 states
def test_pabp_three_free_sites(eng):
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import golden_npz
    g = golden_npz.load("pabp_golden")
    L, q = 82, 20
    m = dict(L=L, q=q, h=g["h"], J=g["J"], alphabet=str(g["alphabet"]), target_seq=str(g["target_seq"]),
             index_list=np.arange(1, L + 1, dtype=np.int32))
    free = np.array([40, 41, 45])
    M = 131072
    with model_ops.PottsSampler(m, M, seed=3, init="target", engine=eng, free=positions(free)) as s:
        s.run(64)
        codes = s.codes().astype(np.int64)
    tgt = model_ops.encode_sequences(m, [m["target_seq"]])[0].astype(np.int64)
    p = cs.exact_conditional(np.asarray(g["h"], dtype=np.float64), np.asarray(g["J"], dtype=np.float64), 1.0, free,
                             tgt)
    counts = np.bincount(ps.state_index(codes[:, free], q), minlength=len(p))
    tv = 0.5 * np.abs(counts / M - p).sum()
    tv_max, _ = distribution_bounds(p, M)
    assert np.array_equal(np.delete(codes, free, axis=1), np.repeat(np.delete(tgt, free)[None], M, axis=0))
    assert tv <= tv_max, (tv, tv_max)


# 7. several ranks return the bits of one process
def write_model(path, m):
    model_io.write_model_file(path, m["L"], m["q"], m["n_valid"], m["n_invalid"], m["num_iter"], m["theta"],
                              m["lambda_h"], m["lambda_J"], m["lambda_group"], m["n_eff"], m["alphabet"],
                              m["weights"], m["target_seq"], m["index_list"], m["fi"], m["h"], m["fij"], m["J"])
    return path


@pytest.mark.parametrize("R", [2, 3])
def test_ranks_write_the_bits_of_one_process(eng, tmp_path, R):
    m = synthetic.planted_potts_model(40, 21, 4, 6)
    free, allowed = list(range(10, 25)) + [40], {12: "ACDE", 40: "W"}
    one = model_ops.sample_sequences(m, 301, 9, seed=4, init="target", engine=eng, free=free, allowed=allowed)
    got = model_ops.sample_sequences(m, 301, 9, seed=4, init="target", free=free, allowed=allowed, num_gpus=R,
                                     backend="gloo")
    assert got == one
    path = write_model(str(tmp_path / "m.model"), m)
    start = str(tmp_path / "start.a2m")
    synthetic.write_a2m(start, np.random.default_rng(R).integers(0, 21, (301, 40)).astype(np.uint8),
                        alphabet=m["alphabet"])
    for tag, extra in (("one", []), ("ranks", ["--gpus", str(R)])):
        err = io.StringIO()
        argv = [path, "-n", "301", "--sweeps", "9", "--seed", "4", "--free", "10-24,40", "--allow", "12:ACDE",
                "--allow", "40:W", "--init", start, "-o", str(tmp_path / (tag + ".a2m"))] + extra
        assert sample_cli.main(argv, stderr=err, backend="gloo") == 0, err.getvalue()
    with open(tmp_path / "one.a2m", "rb") as a, open(tmp_path / "ranks.a2m", "rb") as b:
        assert a.read() == b.read()


# 8. the command line redesigns a window of a planted model
def test_command_line_redesigns_a_window(tmp_path):
    import subprocess
    m = synthetic.planted_potts_model(60, 21, 6, 2)
    path = write_model(str(tmp_path / "m.model"), m)
    out = str(tmp_path / "design.a2m")
    allow = {33: "AVILM", 35: "FWY"}
    subprocess.run([sys.executable, os.path.join(ROOT, "bin", "evcplm-sample"), path, "-n", "500", "--sweeps", "20",
                    "--free", "30-45", "--allow", "33:AVILM", "--allow", "35:FWY", "--init", "target", "--beta", "2",
                    "-o", out], check=True)
    with open(out) as f:
        rows = f.read().split("\n")[1::2]
    assert len(rows) == 500
    tgt = m["target_seq"]
    for r in rows:
        assert len(r) == 60 and r[:29] == tgt[:29] and r[45:] == tgt[45:]
        for p, letters in allow.items():
            assert r[p - 1] in letters
    assert len({r[29:45] for r in rows}) > 1
