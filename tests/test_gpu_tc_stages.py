"""
Every stage of a tensor-core evaluation, element by element, against float64 built from the device's own inputs to
that stage (-m gpu).  The references and bounds are oracle/tc_stages.py (derivations in its docstring); the buffers
come out of the handle through evc_plm_copy_stage, straight into torch tensors on the device.

Per case: one evc_plm_eval_data and (tensor-core forward) one evc_plm_weighted_counts, and then
* expand (Wt, or the fused forward's Wp) bit for bit against the expansion of x;
* Xt bit for bit against the one-hot of the codes;
* the logits Zt against float64 products of the device's Wt, within EPS_ACC * sum |terms|;
* the softmax's residuals Rt (hi + lo / hi), its g_h and -loglk partials, from the device's Zt (the fused forward:
  from float64 logits, with their error added to the bound);
* the backward product: the sum of the Gd planes (and, unchunked, each plane on its K slice) against float64
  products of the device's Xt and Rt over the real sequences;
* finalize_pairs and finalize_fields replayed bit for bit from the device's Gd and partials: g and -loglk of the
  evaluation must equal the replay;
* the counts: Rt = w as bf16 hi + lo, their g_h partials and f_i replayed bit for bit, f_ij from the device's Gd.
Inputs are not dyadic: x ~ N(0, 0.1), weights in U(0.05, 1), synthetic alignments with gaps.  Each case prints, per
stage, the elements checked and the largest error / bound, and the run time and device memory of the case.
"""
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

import test_gpu_tc_edges as te  # noqa: E402
from evcouplings_b200 import _lib, synthetic  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    l = _lib.load()
    _lib.require_device()
    return l


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def copy_stage(lib, h, name, shape, dtype):
    import torch
    out = torch.empty(shape, dtype=dtype, device="cuda")
    _lib.check(lib.evc_plm_copy_stage(h, _lib.STAGE[name], _ptr(out), out.numel() * out.element_size()),
               "evc_plm_copy_stage(%s)" % name)
    return out


class Handle:
    def __init__(self, lib, codes, w, q, gap_code, forward, precision, seq_chunk=0):
        self.lib = lib
        N, L = codes.shape
        self.h = ctypes.c_void_p()
        vp = ctypes.c_void_p
        _lib.check(lib.evc_plm_create_alphabet(ctypes.byref(self.h), codes.ctypes.data_as(vp), N, L, q, gap_code,
                                               w.ctypes.data_as(vp), 0), "evc_plm_create_alphabet")
        if seq_chunk:
            _lib.check(lib.evc_plm_set_seq_chunk(self.h, seq_chunk), "evc_plm_set_seq_chunk")
        _lib.check(lib.evc_plm_set_forward(self.h, forward), "evc_plm_set_forward")
        _lib.check(lib.evc_plm_set_precision(self.h, precision), "evc_plm_set_precision")

    def copy(self, name, shape, dtype):
        return copy_stage(self.lib, self.h, name, shape, dtype)

    def close(self):
        self.lib.evc_plm_destroy(self.h)


def run_case(lib, case):
    """One case: evaluation + counts on a fresh handle, every stage checked.  Returns the Reports.
    case["keep"] (a dict) receives the chunk's Zt and Rt columns; case["check"] = False only evaluates and keeps."""
    import torch
    from oracle import tc_stages as ts
    N, L, q, gap = case["N"], case["L"], case["q"], case["gap"]
    fwd, prec, chunk = case.get("forward", 1), case.get("precision", 0), case.get("seq_chunk", 0)
    single = prec == 1
    gap_code = q if gap else -1
    codes, w, x = te.make_inputs(N, L, q, gap, case.get("seed", 1))
    sm = te._sm_count(lib)
    geo = te.geometry(N, L, q, gap, chunk, sm)
    fused = fwd == 2 and geo["fused"]
    Lq, Mp, Np, Kw, Kp, Ns, C = geo["Lq"], geo["Mp"], geo["Np"], geo["Kw"], geo["Kp"], geo["Ns"], geo["C"]
    S = q if q % 2 else q + 1
    n0 = (geo["n_chunks"] - 1) * C                      # the chunk whose buffers the handle holds after a run
    nreal = N - n0
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    dc = torch.from_numpy(codes.astype(np.int64)).cuda()
    dw = torch.from_numpy(w).cuda()
    dx = torch.from_numpy(x).cuda()
    H = Handle(lib, codes, w, q, gap_code, fwd, prec, chunk)
    rep, crep = ts.Report(), ts.Report()
    try:
        dg = torch.zeros_like(dx)
        dfx = torch.zeros(2, dtype=torch.float64, device="cuda")
        _lib.check(lib.evc_plm_eval_data(H.h, _ptr(dx), _ptr(dg), _ptr(dfx), None), "evc_plm_eval_data")
        torch.cuda.synchronize()
        t_eval = time.time() - t0
        handle_bytes = int(lib.evc_plm_device_bytes(H.h))
        bf = torch.bfloat16
        if not case.get("check", True):
            case["keep"].update(zt=H.copy("Zt", (Mp, Ns), torch.float32)[:, :nreal].clone(),
                                rt_hi=H.copy("Rt_hi", (Np, Kp), bf)[:, :nreal].clone(),
                                rt_lo=None if single else H.copy("Rt_lo", (Np, Kp), bf)[:, :nreal].clone())
            return None
        # expand
        if fused:
            m_tiles = -(-N // 128)
            npf = -(-L // 8) * 176
            whi, wlo = H.copy("Wp_hi", (npf, Kw), bf), H.copy("Wp_lo", (npf, Kw), bf)
            ts.check_expand(rep, whi, wlo, dx, L, q, single, padded=True)
            prow = ts.padded_rows(L, q).reshape(-1).cuda()
            W = (whi[prow], None if single else wlo[prow])
            del whi, wlo
        else:
            whi, wlo = H.copy("Wt_hi", (Mp, Kw), bf), H.copy("Wt_lo", (Mp, Kw), bf)
            ts.check_expand(rep, whi, wlo, dx, L, q, single)
            W = (whi, None if single else wlo)
        # Xt
        xt = H.copy("Xt", (Mp, Kp), bf)
        ts.check_xt(rep, xt, dc[n0:], q, nreal)
        # logits and softmax on the column ranges of the case (default: every real sequence of the chunk)
        cols = case.get("cols") or [(0, nreal)]
        rt_hi = H.copy("Rt_hi", (Np, Kp), bf)
        rt_lo = None if single else H.copy("Rt_lo", (Np, Kp), bf)
        if fused:
            ntp = m_tiles * 4
            gh = H.copy("gh_part", (L, ntp, S), torch.float32)
            fxp = H.copy("fx_part", (L, ntp), torch.float64)
            ts.check_softmax(rep, None, dx[:Lq], dc, dw, q, N, 0, single, rt_hi, rt_lo, gh, fxp, cols, tile=32,
                             fused=W, full_columns=True)
        else:
            zt = H.copy("Zt", (Mp, Ns), torch.float32)
            ts.check_logits(rep, zt, W[0], W[1], dc[n0:], q, cols)
            ntl = -(-N // 256)
            gh = H.copy("gh_part", (L, ntl, S), torch.float32)
            fxp = H.copy("fx_part", (L, ntl), torch.float64)
            ts.check_softmax(rep, zt, dx[:Lq], dc[n0:], dw[n0:], q, N, n0, single, rt_hi, rt_lo, gh, fxp, cols,
                             full_columns=geo["n_chunks"] == 1)
            if case.get("keep") is not None:
                case["keep"].update(zt=zt[:, :nreal].clone(), rt_hi=rt_hi[:, :nreal].clone(),
                                    rt_lo=None if single else rt_lo[:, :nreal].clone())
            del zt
        del W
        ts.check_finalize_fields(rep, gh, fxp, q, dg[:Lq], dfx[0])
        # backward and finalize_pairs
        gd = H.copy("Gd", (geo["planes"], Mp, Np), torch.float32)
        if geo["n_chunks"] == 1:
            ts.check_backward(rep, gd, L, q, N, ts.xt_columns(xt, Lq), ts.rt_columns(rt_hi, rt_lo, Lq),
                              ksplit=geo["ksplit"], num_kb=Kp // 64)
        else:
            ref = case["unchunked"]
            ts.check_backward(rep, gd, L, q, N, ts.codes_columns(dc, q),
                              ts.rt_columns(ref["rt_hi"], ref["rt_lo"], Lq))
        ts.check_finalize_pairs(rep, gd, L, q, 1.0, dg[Lq:])
        del gd, rt_hi, rt_lo
        # the counts through the same backward product (the fused handle's counts run on the gather kernels)
        if not fused:
            fi = torch.zeros(Lq, dtype=torch.float32, device="cuda")
            fij = torch.zeros(dx.numel() - Lq, dtype=torch.float32, device="cuda")
            _lib.check(lib.evc_plm_weighted_counts(H.h, _ptr(fi), _ptr(fij), None), "evc_plm_weighted_counts")
            crh, crl = H.copy("Rt_hi", (Np, Kp), bf), H.copy("Rt_lo", (Np, Kp), bf)
            ts.check_counts_residual(crep, crh, crl, dc[n0:], dw[n0:], q, nreal, full_columns=geo["n_chunks"] == 1)
            cgh = H.copy("gh_part", (L, -(-N // 256), S), torch.float32)
            n_gh = ts._assert_equal_bits("counts gh_part", cgh, ts.counts_gh_replay(dc, dw, q, S, -(-N // 256)))
            crep.add("counts gh_part", n_gh)
            ts.check_finalize_fields(crep, cgh, None, q, fi, None)
            cgd = H.copy("Gd", (geo["planes"], Mp, Np), torch.float32)
            if geo["n_chunks"] == 1:
                xt = H.copy("Xt", (Mp, Kp), bf)
                ts.check_backward(crep, cgd, L, q, N, ts.xt_columns(xt, Lq), ts.rt_columns(crh, crl, Lq),
                                  ksplit=geo["ksplit"], num_kb=Kp // 64, label="counts backward")
            else:
                chi, clo = ts.counts_residual(dc, dw, q)
                ts.check_backward(crep, cgd, L, q, N, ts.codes_columns(dc, q), ts.rt_columns(chi, clo, Lq),
                                  label="counts backward")
            ts.check_finalize_pairs(crep, cgd, L, q, 0.5, fij)
    finally:
        H.close()
    torch.cuda.synchronize()
    print("\n[%s] N=%d L=%d q=%d%s forward %d precision %d chunk %d: %s" % (
        case["target"], N, L, q, " (gap ignored)" if gap else "", fwd, prec, chunk, te._fmt_geometry(geo)))
    print("\n".join(rep.lines() + crep.lines()))
    print("  evaluation %.2f s, whole case %.1f s; handle %.2f GB, checks peak %.2f GB of torch memory" % (
        t_eval, time.time() - t0, handle_bytes / 1e9, torch.cuda.max_memory_allocated() / 1e9))
    return rep, crep


# ------------------------------------------------------------------------------------------------
# production shapes
# ------------------------------------------------------------------------------------------------
CONFIG2 = dict(N=50000, L=200, q=21, gap=False, seed=2)


@pytest.mark.parametrize("forward,precision", [(1, 0), (1, 1), (2, 0)], ids=["sparse-fp32", "sparse-bf16", "fused-fp32"])
def test_config2_every_stage(lib, forward, precision):
    geo = te.geometry(50000, 200, 21, False, 0, te._sm_count(lib))
    assert geo["fused"] and geo["ksplit"] >= 1
    run_case(lib, dict(CONFIG2, forward=forward, precision=precision,
                       target="config 2, %s" % ("fused" if forward == 2 else "sparse")))


def test_config5_every_stage_on_first_middle_last_tiles(lib):
    """N = 100 000, L = 800: K is 263 blocks, so the 128-row forward tiles and the k_chunk promotion run.  Logits and
    residuals on the first, a middle and the last (partial) 256-sequence tiles; Xt, Gd, g and the counts in full."""
    N = 100000
    last = (N // 256) * 256
    geo = te.geometry(N, 800, 21, False, 0, te._sm_count(lib))
    assert geo["Kw"] // 64 == 263
    run_case(lib, dict(N=N, L=800, q=21, gap=False, seed=5, cols=[(0, 256), (195 * 256, 196 * 256), (last, N)],
                       target="config 5"))


# ------------------------------------------------------------------------------------------------
# chunks: the last chunk partial; its Zt / Rt bits equal the unchunked handle's, Gd against the float64 product of
# the unchunked handle's residuals
# ------------------------------------------------------------------------------------------------
def test_config2_chunked_last_chunk_partial(lib):
    chunk = 22 * 768                                    # 16896: 3 chunks, the last holds 16208 sequences
    geo = te.geometry(50000, 200, 21, False, chunk, te._sm_count(lib))
    assert geo["n_chunks"] == 3 and 50000 - 2 * geo["C"] < geo["C"]
    keep = {}
    run_case(lib, dict(CONFIG2, keep=keep, check=False, target="config 2 unchunked"))
    n0 = 2 * geo["C"]
    ref = dict(rt_hi=keep["rt_hi"], rt_lo=keep["rt_lo"])
    got = {}
    run_case(lib, dict(CONFIG2, seq_chunk=chunk, unchunked=ref, keep=got, target="config 2, 3 chunks"))
    for k in ("zt", "rt_hi", "rt_lo"):
        a, b = got[k], keep[k][:, n0:]
        assert a.shape == b.shape and bool((a.view(-1).view(dtype=_int(a)) == b.contiguous().view(-1).view(
            dtype=_int(b))).all()), k


def _int(t):
    import torch
    return {torch.bfloat16: torch.int16, torch.float32: torch.int32}[t.dtype]


# ------------------------------------------------------------------------------------------------
# alphabets, tile edges and sequence counts
# ------------------------------------------------------------------------------------------------
EDGE_CASES = [
    dict(N=3000, L=60, q=4, gap=True, target="q=4, gap ignored"),
    dict(N=3000, L=60, q=20, gap=True, target="q=20, gap ignored"),
    dict(N=3000, L=40, q=32, gap=False, target="q=32: WIDE expand and finalize"),
    dict(N=1000, L=256, q=32, gap=False, target="Lq=8192: 256-sequence forward tiles"),
    dict(N=1000, L=391, q=21, gap=False, target="Lq=8211: 128-sequence forward tiles"),
    dict(N=1000, L=390, q=21, gap=False, forward=2, target="Lq=8190: fused"),
] + [dict(N=n, L=30, q=21, gap=False, seed=n, target="N=%d" % n) for n in (1, 255, 257, 385)] + [
    dict(N=385, L=30, q=21, gap=False, precision=1, seed=7, target="N=385, bf16"),
    dict(N=257, L=30, q=21, gap=False, forward=2, seed=8, target="N=257, fused")]


@pytest.mark.parametrize("case", EDGE_CASES, ids=lambda c: c["target"].split(":")[0].replace(" ", "_"))
def test_edges_every_stage(lib, case):
    run_case(lib, case)


# ------------------------------------------------------------------------------------------------
# the tuning hooks (read once per process): a forced 3-way K split of the backward, and k_chunk = 1
# ------------------------------------------------------------------------------------------------
_SUB = """
import json, sys
sys.path.insert(0, %r); sys.path.insert(0, %r)
import test_gpu_tc_stages as t
from evcouplings_b200 import _lib
lib = _lib.load()
for c in json.loads(sys.argv[1]):
    t.run_case(lib, c)
""" % (ROOT, HERE)


@pytest.mark.parametrize("env", [{"EVC_KSPLIT": "3"}, {"EVC_KCHUNK": "1"}], ids=["ksplit3", "kchunk1"])
def test_hooks_every_stage(lib, env):
    cases = [dict(N=4097, L=40, q=21, gap=False, seed=11, target="N=4097 %s" % env),
             dict(N=4097, L=40, q=21, gap=False, seed=11, precision=1, target="N=4097 bf16 %s" % env)]
    e = {k: v for k, v in os.environ.items() if k not in ("EVC_KSPLIT", "EVC_KCHUNK", "EVC_MGROUP")}
    e.update(env)
    p = subprocess.run([sys.executable, "-c", _SUB, json.dumps(cases)], capture_output=True, text=True, env=e,
                       timeout=900)
    print(p.stdout)
    assert p.returncode == 0, p.stderr[-4000:]


# ------------------------------------------------------------------------------------------------
# 64-bit offsets: L = 2300, q = 21 puts Wt (48 384 x 48 320) and the Gd plane (48 384 x 48 384) past 2^31 elements;
# their rows on both sides of element 2^31 (and the first, last and padding rows) are checked
# ------------------------------------------------------------------------------------------------
def test_l2300_rows_across_the_2_31_element_offset(lib):
    import torch
    from oracle import tc_stages as ts
    N, L, q = 100, 2300, 21
    geo = te.geometry(N, L, q, False, 0, te._sm_count(lib))
    Lq, Mp, Np, Kw, Kp = geo["Lq"], geo["Mp"], geo["Np"], geo["Kw"], geo["Kp"]
    assert Mp * Kw > 2 ** 31 and Mp * Np > 2 ** 31 and geo["planes"] == 1
    codes = np.ascontiguousarray(synthetic.synthetic_msa_codes(N, L, 23))   # x is drawn on the device (1.2e9 values)
    w = np.random.default_rng(23).uniform(0.05, 1.0, N).astype(np.float32)
    gen = torch.Generator(device="cuda").manual_seed(23)
    n_params = Lq + L * (L - 1) // 2 * q * q
    t0 = time.time()
    dx = torch.randn(n_params, device="cuda", generator=gen, dtype=torch.float32) * 0.1
    dc = torch.from_numpy(codes.astype(np.int64)).cuda()
    dw = torch.from_numpy(w).cuda()
    H = Handle(lib, codes, w, q, -1, 1, 0)
    rep = ts.Report()
    try:
        dg = torch.zeros_like(dx)
        dfx = torch.zeros(2, dtype=torch.float64, device="cuda")
        _lib.check(lib.evc_plm_eval_data(H.h, _ptr(dx), _ptr(dg), _ptr(dfx), None), "evc_plm_eval_data")
        del dg
        handle_bytes = int(lib.evc_plm_device_bytes(H.h))

        def around(ld, rows_total):
            b = 2 ** 31 // ld                        # the row holding element 2^31
            r = sorted({0, Lq - 1, Lq, rows_total - 1} | set(range(b - 2, b + 3)))
            return torch.tensor([v for v in r if 0 <= v < rows_total], dtype=torch.int64)

        rows_w = around(Kw, Mp)
        for name in ("Wt_hi", "Wt_lo"):
            buf = H.copy(name, (Mp, Kw), torch.bfloat16)
            ts.check_expand(rep, buf if name == "Wt_hi" else None, buf if name == "Wt_lo" else None, dx, L, q,
                            False, rows=rows_w, block=16)
            del buf
        xt = H.copy("Xt", (Mp, Kp), torch.bfloat16)
        ts.check_xt(rep, xt, dc, q, N)
        rt_hi, rt_lo = H.copy("Rt_hi", (Np, Kp), torch.bfloat16), H.copy("Rt_lo", (Np, Kp), torch.bfloat16)
        gd = H.copy("Gd", (1, Mp, Np), torch.float32)
        rows_g = around(Np, Mp)
        ts.check_backward_rows(rep, gd, rows_g, L, q, N, ts.xt_columns(xt, Lq), ts.rt_columns(rt_hi, rt_lo, Lq))
        del gd
    finally:
        H.close()
    torch.cuda.synchronize()
    print("\n[L=2300] N=%d: %s; Wt rows %s, Gd rows %s" % (N, te._fmt_geometry(geo), rows_w.tolist(),
                                                          rows_g.tolist()))
    print("\n".join(rep.lines()))
    print("  whole case %.1f s; handle %.2f GB, checks peak %.2f GB of torch memory" % (
        time.time() - t0, handle_bytes / 1e9, torch.cuda.max_memory_allocated() / 1e9))


# ------------------------------------------------------------------------------------------------
# the failure contract of evc_plm_copy_stage
# ------------------------------------------------------------------------------------------------
def test_copy_stage_refuses_what_it_cannot_copy(lib):
    import torch
    codes, w, _x = te.make_inputs(300, 20, 21, False, 3)
    geo = te.geometry(300, 20, 21, False, 0, te._sm_count(lib))
    buf = torch.empty(geo["Mp"] * geo["Kw"], dtype=torch.bfloat16, device="cuda")
    nbytes = buf.numel() * 2
    for forward in (1, 2):
        H = Handle(lib, codes, w, 21, -1, forward, 0)
        try:
            assert lib.evc_plm_copy_stage(H.h, 12, _ptr(buf), nbytes) != 0
            assert b"unknown stage 12" in lib.evc_last_error()
            assert lib.evc_plm_copy_stage(H.h, -1, _ptr(buf), nbytes) != 0
            assert lib.evc_plm_copy_stage(H.h, _lib.STAGE["Wt_hi"], None, nbytes) != 0
            assert b"null pointer" in lib.evc_last_error()
            missing = "Wp_hi" if forward == 1 else "Wt_hi"
            assert lib.evc_plm_copy_stage(H.h, _lib.STAGE[missing], _ptr(buf), nbytes) != 0
            assert b"has not allocated " + missing.encode() in lib.evc_last_error()
            present = "Wt_hi" if forward == 1 else "Wp_hi"
            assert lib.evc_plm_copy_stage(H.h, _lib.STAGE[present], _ptr(buf), nbytes + 2) != 0
            assert b"bytes must be the allocation of " + present.encode() in lib.evc_last_error()
            if forward == 1:
                _lib.check(lib.evc_plm_copy_stage(H.h, _lib.STAGE["Wt_hi"], _ptr(buf), nbytes), "copy Wt_hi")
                host = np.empty(nbytes, dtype=np.uint8)
                _lib.check(lib.evc_plm_copy_stage(H.h, _lib.STAGE["Wt_hi"], host.ctypes.data_as(ctypes.c_void_p),
                                                  nbytes), "copy Wt_hi to host")
                assert np.array_equal(host, buf.view(torch.uint8).cpu().numpy())
        finally:
            H.close()
