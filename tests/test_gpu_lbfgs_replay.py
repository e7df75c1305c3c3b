"""
The device L-BFGS step against its fp32 replay (oracle/lbfgs_replay.py) on the H100.

ABI level: evc_lbfgs_update_pair, evc_lbfgs_direction, evc_vec_dot and evc_plm_add_regulariser on random data at
n = 1, 1000, 1184 * 256 (one element per thread of the reduction grid), one past it and 8 780 100 (L = 200, q = 21):
every vector bit for bit, every double within the bound of the reduction tree, the alphas read back from the scratch.

Fit level: evc_plm_fit_checkpointed with a checkpoint at every iteration boundary.  At each boundary k the test keeps
x_k, g_k, the newest pair and the state, and afterwards re-evaluates the data term at every x_k on the same handle in
the precision x_k was taken in.  Then, at every k: nll and g_k = fmaf(2 lambda, x_k, g_data(x_k)) bit for bit; fx - nll
and the norms within the tree bound; the pair bit for bit and ys / yy within the bound; x_{k+1} = fmaf(float(step),
d_k, x_k) for a branch of the replayed direction d_k; the strong Wolfe conditions in float64; and the step and
evaluation counts of the driver's rules.  A wrong gamma pair, a skipped or misordered ring slot, a wrongly mapped
host slot or a wrong regulariser boundary changes some x_{k+1} bit.
"""
import ctypes
import math
import time

import numpy as np
import pytest

from evcouplings_b200 import _lib, synthetic
from oracle import lbfgs_replay as lr

pytestmark = pytest.mark.gpu

F32 = np.float32
U = lr.U64


@pytest.fixture(scope="module")
def eng():
    from evcouplings_b200.engine import CudaEngine
    return CudaEngine()


def _dev(eng, a, dtype=None):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).to(eng.device)


def _host(t):
    return t.detach().cpu().numpy()


def _in(value, ref_bound, what):
    ref, b = ref_bound
    assert abs(float(value) - ref) <= b, "%s = %r, reference %r, bound %r" % (what, float(value), ref, b)


# ---- ABI level -------------------------------------------------------------------------------------------------------
def _slot_data(torch, gen, n, device):
    xp = torch.randn(n, generator=gen, device=device)
    x = xp + 0.1 * torch.randn(n, generator=gen, device=device)
    g = torch.randn(n, generator=gen, device=device)
    gp = g - (x - xp) * (0.5 + 1.5 * torch.rand(n, generator=gen, device=device))
    return x, xp, g, gp


@pytest.mark.parametrize("n", [1, 1000, lr.GRID, lr.GRID + 1, 8_780_100])
def test_abi_pair_direction_and_dot(eng, n):
    """Every (m, bound, end) with m in {1, 5, 32}, bound in {0, 1, m}, end in {0, m - 1, a random slot}; at
    n = 8 780 100 the m = 32 ring runs bound 0 and 1 only (a full replay of 32 pairs there takes minutes)."""
    import torch
    lib, e = eng.lib, eng
    gen = torch.Generator(device=e.device)
    gen.manual_seed(n)
    rng = np.random.default_rng(n)
    t0 = time.time()
    opened_total = 0
    for m in (1, 5, 32):
        S = torch.zeros((m, n), dtype=torch.float32, device=e.device)
        Y = torch.zeros_like(S)
        ys = torch.zeros(m, dtype=torch.float64, device=e.device)
        scratch = torch.zeros(m + 2, dtype=torch.float64, device=e.device)
        yy_slot = np.zeros(m)
        Sh, Yh = [None] * m, [None] * m
        for j in range(m):
            x, xp, g, gp = _slot_data(torch, gen, n, e.device)
            _lib.check(lib.evc_lbfgs_update_pair(e.ptr(S[j]), e.ptr(Y[j]), e.ptr(x), e.ptr(xp), e.ptr(g), e.ptr(gp),
                                                 e.ptr(ys[j:j + 1]), e.ptr(scratch[0:1]), n, e.stream()),
                       "evc_lbfgs_update_pair")
            s_ref, y_ref = lr.pair(_host(x), _host(xp), _host(g), _host(gp))
            Sh[j], Yh[j] = _host(S[j]), _host(Y[j])
            assert lr.same_bits(Sh[j], s_ref), (m, j, lr.first_mismatch(Sh[j], s_ref))
            assert lr.same_bits(Yh[j], y_ref), (m, j, lr.first_mismatch(Yh[j], y_ref))
            yy_slot[j] = float(scratch[0].item())
            _in(ys[j].item(), lr.dot_bound(y_ref, s_ref), "ys")
            _in(yy_slot[j], lr.dot_bound(y_ref, y_ref), "yy")
        ys_h = _host(ys)
        g = torch.randn(n, generator=gen, device=e.device)
        gh = _host(g)
        d = torch.empty(n, dtype=torch.float32, device=e.device)
        bounds = sorted({0, 1, m}) if not (m == 32 and n > 10 ** 6) else [0, 1]
        for bound in bounds:
            for end in sorted({0, m - 1, int(rng.integers(0, m))}):
                newest = (end - 1) % m
                scratch[0] = yy_slot[newest]
                _lib.check(lib.evc_lbfgs_direction(e.ptr(d), e.ptr(g), e.ptr(S), e.ptr(Y), e.ptr(ys), e.ptr(scratch),
                                                   n, m, bound, end, e.stream()), "evc_lbfgs_direction")
                dh, alphas = _host(d), _host(scratch)[2:]
                bad = []
                cands, opened = lr.direction(gh, Sh, Yh, ys_h, yy_slot[newest], m, bound, end, alphas=alphas,
                                             bad_alphas=bad)
                opened_total += opened
                assert not bad, (m, bound, end, bad)
                assert lr.match(dh, cands) >= 0, (m, bound, end, opened, lr.first_mismatch(dh, cands[0]))
    # evc_vec_dot on the last ring's vectors and on a cancelling pair
    out = torch.zeros(1, dtype=torch.float64, device=e.device)
    a, b = _host(S[0]), _host(Y[0])
    for u, v in ((a, b), (a, (-a).astype(F32)), (gh, gh)):
        tu, tv = _dev(e, u), _dev(e, v)
        _lib.check(lib.evc_vec_dot(e.ptr(tu), e.ptr(tv), n, e.ptr(out), e.stream()), "evc_vec_dot")
        _in(out.item(), lr.dot_bound(u, v), "dot")
    print("n=%d branches opened %d, %.1f s" % (n, opened_total, time.time() - t0))


@pytest.mark.parametrize("L,q", [(2, 2), (7, 21), (200, 21)])
def test_abi_regulariser(eng, L, q):
    """g += 2 lambda x bit for bit, with lambda_h != lambda_J and x nonzero on both sides of L q, and d_fx[1]."""
    import torch
    lib, e = eng.lib, eng
    codes = np.random.default_rng(L).integers(0, q, size=(16, L)).astype(np.uint8)
    p = e.plm_problem(codes, np.ones(16, dtype=np.float32), q, -1, 0.01, 1.0)
    try:
        n, nh = p.n, L * q
        rng = np.random.default_rng(L * 100 + q)
        x = (rng.normal(size=n) * 2.0 ** rng.integers(-8, 8, n)).astype(F32)
        g0 = rng.normal(size=n).astype(F32)
        for lam_h, lam_J in ((F32(0.01), F32(39.8)), (F32(3.3), F32(0.07))):
            g, tx = _dev(e, g0), _dev(e, x)
            fx = torch.tensor([12345.678, 0.0], dtype=torch.float64, device=e.device)
            _lib.check(lib.evc_plm_add_regulariser(p.handle, e.ptr(tx), e.ptr(g), e.ptr(fx), lam_h, lam_J,
                                                   e.stream()), "evc_plm_add_regulariser")
            want = lr.regulariser(x, g0, nh, lam_h, lam_J)
            assert lr.same_bits(_host(g), want), lr.first_mismatch(_host(g), want)
            lam = lr.lambdas(n, nh, lam_h, lam_J).astype(np.float64)
            ref, b = lr.sum_bound(lam * x.astype(np.float64) ** 2, extra=2)
            f0, f1 = _host(fx)
            assert f0 == 12345.678
            assert abs(f1 - (f0 + ref)) <= b + 2 * U * abs(f1), (f1, f0 + ref, b)
    finally:
        p.close()


# ---- fit level -------------------------------------------------------------------------------------------------------
class _Recorder(object):
    """Progress rows and, at every boundary, x, g, the newest pair and the state, copied off the device."""

    def __init__(self, eng, p, m):
        self.eng, self.p, self.m = eng, p, m
        self.rows, self.bounds, self.errors = {}, {}, []
        self.final = None

    def vector(self, which, slot=0):
        import torch
        from evcouplings_b200.engine import _DevicePointer
        ptr = ctypes.c_void_p()
        _lib.check(self.eng.lib.evc_plm_fit_vector(self.p.handle, which, slot, ctypes.byref(ptr)),
                   "evc_plm_fit_vector")
        torch.cuda.synchronize(self.eng.device)
        if which in (_lib.FIT_VEC_S, _lib.FIT_VEC_Y) and slot >= self.m - self.p.host_pairs:
            return np.ctypeslib.as_array((ctypes.c_float * self.p.n).from_address(ptr.value)).copy()
        return torch.as_tensor(_DevicePointer(ptr.value, self.p.n), device=self.eng.device).cpu().numpy().copy()

    def progress(self, user, k, fx, xnorm, gnorm, step, count, nll, hnorm, enorm):
        self.rows[k] = dict(fx=fx, xnorm=xnorm, gnorm=gnorm, step=step, count=count, nll=nll, hnorm=hnorm,
                            enorm=enorm)
        return 0

    def state(self, user, sp, stream):
        try:
            s = sp.contents
            if s.returning and s.k in self.bounds:
                # the fit returns from this boundary; after a failed line search its count includes that search
                self.final = dict(status=s.status, evaluations=s.evaluations)
                return 0
            b = dict(k=s.k, evaluations=s.evaluations, hist=s.hist, end=s.end, low=s.low,
                     switched_at=s.switched_at, ys=np.array([s.ys[j] for j in range(s.m)]), yy=s.yy,
                     returning=s.returning, status=s.status)
            b["x"] = self.vector(_lib.FIT_VEC_X)
            b["g"] = self.vector(_lib.FIT_VEC_G)
            if s.hist > 0:
                newest = (s.end - 1) % s.m
                b["s"] = self.vector(_lib.FIT_VEC_S, newest)
                b["y"] = self.vector(_lib.FIT_VEC_Y, newest)
            self.bounds[s.k] = b
            return 0
        except BaseException as exc:       # never across the C boundary
            self.errors.append(exc)
            return 1


def _eval_data(eng, p, x, low):
    import torch
    _lib.check(eng.lib.evc_plm_set_precision(p.handle, 1 if low else 0), "evc_plm_set_precision")
    g = torch.empty(p.n, dtype=torch.float32, device=eng.device)
    fx = torch.zeros(2, dtype=torch.float64, device=eng.device)
    tx = _dev(eng, x)
    _lib.check(eng.lib.evc_plm_eval_data(p.handle, eng.ptr(tx), eng.ptr(g), eng.ptr(fx), eng.stream()),
               "evc_plm_eval_data")
    return float(fx[0].item()), _host(g)


def _norm_ok(norm, terms, what):
    ref, b = lr.sum_bound(terms)
    assert abs(norm * norm - ref) <= b + 6 * U * ref, (what, norm * norm, ref, b)


def _replay_fit(eng, codes, w, q, lam_h, lam_J, m, iters, host_pairs=0, schedule=0, epsilon=1e-12):
    lib = eng.lib
    t_start = time.time()
    lam_h, lam_J = F32(lam_h), F32(lam_J)
    p = eng.plm_problem(codes, w, q, -1, float(lam_h), float(lam_J), m=m, seq_chunk=0)
    try:
        if host_pairs:
            _lib.check(lib.evc_plm_set_host_history(p.handle, host_pairs), "evc_plm_set_host_history")
            p.host_pairs = host_pairs
        n, nh = p.n, codes.shape[1] * q
        fp = _lib.FitParams()
        lib.evc_fit_default_params(ctypes.byref(fp))
        fp.max_iterations, fp.m, fp.epsilon = iters, m, epsilon
        fp.lambda_h, fp.lambda_J, fp.precision_schedule = lam_h, lam_J, schedule
        rec = _Recorder(eng, p, m)
        pr_cb, ck_cb = _lib.PROGRESS_CB(rec.progress), _lib.CHECKPOINT_CB(rec.state)
        x0 = np.zeros(n, dtype=F32)
        p.set_x(x0)
        res = _lib.FitResult()
        rc = lib.evc_plm_fit_checkpointed(p.handle, eng.ptr(p.x), ctypes.byref(fp), None, None,
                                          ctypes.cast(pr_cb, ctypes.c_void_p), None,
                                          ctypes.cast(ck_cb, ctypes.c_void_p), None, 0.0, None, ctypes.byref(res),
                                          eng.stream())
        if rec.errors:
            raise rec.errors[0]
        _lib.check(rc, "evc_plm_fit_checkpointed")
        t_fit = time.time()
        B, R = rec.bounds, rec.rows
        K = res.iterations
        assert sorted(B) == list(range(1, K + 1)) and sorted(R) == list(range(1, K + 1)), (sorted(B), K)
        lam = lr.lambdas(n, nh, lam_h, lam_J)
        lam64 = lam.astype(np.float64)

        # the iterates: x_0 and its gradient in the start precision, then every boundary's
        low0 = schedule == 1
        X, G, low = {0: x0}, {}, {0: low0}
        for k in range(1, K + 1):
            X[k], low[k] = B[k]["x"], bool(B[k]["low"])
        nll = {}
        for k in range(0, K + 1):
            nll[k], gd = _eval_data(eng, p, X[k], low[k])
            G[k] = lr.regulariser(X[k], gd, nh, lam_h, lam_J)
            if k:
                assert nll[k] == R[k]["nll"], (k, nll[k], R[k]["nll"])                           # check 1
                assert lr.same_bits(B[k]["g"], G[k]), (k, lr.first_mismatch(B[k]["g"], G[k]))
        # the precision switch: the first boundary taken in hi+lo after bf16 ones; g' at the iterate before it
        switch = next((k for k in range(1, K + 1) if low[k - 1] and not low[k]), None)
        if schedule:
            assert switch is not None and B[K]["switched_at"] in (switch - 1, switch), (switch, B[K]["switched_at"])
        Gp = dict(G)
        f = {k: R[k]["fx"] for k in range(1, K + 1)}
        f[0] = nll[0] + float(np.sum(lam64 * X[0].astype(np.float64) ** 2))
        fpre = dict(f)
        if switch is not None:
            nll_s, gd = _eval_data(eng, p, X[switch - 1], False)
            Gp[switch - 1] = lr.regulariser(X[switch - 1], gd, nh, lam_h, lam_J)
            fpre[switch - 1] = nll_s + lr.exact_sum(lam64 * X[switch - 1].astype(np.float64) ** 2)

        for k in range(1, K + 1):                                                                 # check 2
            x64, g64 = X[k].astype(np.float64), G[k].astype(np.float64)
            ref, b = lr.sum_bound(lam64 * x64 * x64, extra=2)
            assert abs((R[k]["fx"] - R[k]["nll"]) - ref) <= b + 2 * U * abs(R[k]["fx"]), k
            _norm_ok(R[k]["xnorm"], x64 * x64, "xnorm")
            _norm_ok(R[k]["gnorm"], g64 * g64, "gnorm")
            _norm_ok(R[k]["hnorm"], x64[:nh] ** 2, "hnorm")
            _norm_ok(R[k]["enorm"], x64[nh:] ** 2, "enorm")

        # a switch at boundary switch - 1 re-evaluates once; a switch after a failed bf16 line search also spent
        # that search's evaluations, which no callback reports
        lost_evals = switch is not None and B[K]["switched_at"] == switch
        ring_s, ring_y = {}, {}
        opened_total, evals = 0, 1
        for k in range(0, K):
            bk = B.get(k)
            hist, end = (bk["hist"], bk["end"]) if k else (0, 0)
            if hist:                                                                              # check 3
                newest = (end - 1) % m
                s_ref, y_ref = lr.pair(X[k], X[k - 1], G[k], Gp[k - 1])
                assert lr.same_bits(bk["s"], s_ref), (k, lr.first_mismatch(bk["s"], s_ref))
                assert lr.same_bits(bk["y"], y_ref), (k, lr.first_mismatch(bk["y"], y_ref))
                _in(bk["ys"][newest], lr.dot_bound(y_ref, s_ref), "ys at %d" % k)
                _in(bk["yy"], lr.dot_bound(y_ref, y_ref), "yy at %d" % k)
                ring_s[newest], ring_y[newest] = bk["s"], bk["y"]
            if switch is not None and k == switch - 1:
                hist = 0                       # history dropped: d = -g' at the re-evaluated iterate
            if switch is not None and k == switch:
                assert (bk["hist"], bk["end"]) == (1, 1), (bk["hist"], bk["end"])
            gk = Gp[k]
            if hist:
                cands, opened = lr.direction(gk, ring_s, ring_y, bk["ys"], bk["yy"], m, hist, end)
                opened_total += opened
            else:
                cands = [-gk]
            # check 4: x_{k+1} from x_k along a branch of d_k with the reported step
            st = R[k + 1]["step"]
            hit = [i for i, dk in enumerate(cands) if lr.same_bits(X[k + 1], lr.step(X[k], dk, st))]
            assert hit, (k, len(cands), lr.first_mismatch(X[k + 1], lr.step(X[k], cands[0], st)))
            dk = cands[hit[0]].astype(np.float64)
            # check 5: strong Wolfe in float64 with the device's fx and the replayed d_k
            dg0 = lr.exact_sum(gk.astype(np.float64) * dk)
            dg1 = lr.exact_sum(G[k + 1].astype(np.float64) * dk)
            assert dg0 < 0, k
            assert f[k + 1] <= fpre[k] + 1e-4 * st * dg0 + 1e-12 * abs(fpre[k]), (k, f[k + 1], fpre[k], st, dg0)
            assert abs(dg1) <= 0.9 * abs(dg0) * (1 + 1e-9), (k, dg1, dg0)
            # check 6: the step and evaluation rules
            count = R[k + 1]["count"]
            if count == 1:
                if hist:
                    assert st == 1.0, (k, st)
                else:
                    gg = lr.sum_bound(gk.astype(np.float64) ** 2)
                    assert abs(st * math.sqrt(gg[0]) - 1.0) <= gg[1] / gg[0] + 8 * U, (k, st)
            evals += count + (1 if switch is not None and k + 1 == switch else 0)
            if lost_evals and k + 1 >= switch:
                assert B[k + 1]["evaluations"] >= evals, (k + 1, B[k + 1]["evaluations"], evals)
                evals = B[k + 1]["evaluations"]
            else:
                assert B[k + 1]["evaluations"] == evals, (k + 1, B[k + 1]["evaluations"], evals)
        if rec.final is not None:
            assert rec.final["evaluations"] >= evals and rec.final["status"] == res.status, (rec.final, evals)
        print("n=%d m=%d host_pairs=%d iterations %d, switch %s, branches opened %d, fit %.1f s, check %.1f s"
              % (n, m, host_pairs, K, switch, opened_total, t_fit - t_start, time.time() - t_fit))
        return res, B, opened_total
    finally:
        p.close()


def _production(N=2000, L=200):
    codes = synthetic.synthetic_msa_codes(N, L, 3)
    w = np.random.default_rng(4).uniform(0.2, 1.0, N).astype(np.float32)
    return codes, w


@pytest.mark.parametrize("m,host_pairs", [(6, 0), (5, 3)])
def test_fit_production_shape(eng, m, host_pairs):
    """L = 200, q = 21, N = 2000 (n = 8 780 100), 10 iterations: the ring wraps; with 3 of 5 pairs in host memory."""
    codes, w = _production()
    res, B, opened = _replay_fit(eng, codes, w, 21, 0.01, 0.01 * 20 * 199, m, 10, host_pairs=host_pairs)
    assert res.status == -1004 and res.iterations == 10
    assert opened <= 4


@pytest.mark.parametrize("m,iters", [(32, 40), (1, 20)])
def test_fit_history_edges(eng, m, iters):
    """m = 32 (the whole SC_YS / SC_ALPHA layout, the ring wrapping after 32 pairs) and m = 1 on L = 40, weakly
    regularised so that the cap is reached before the line search stalls."""
    codes = synthetic.synthetic_msa_codes(3001, 40, 5)
    w = np.random.default_rng(6).uniform(0.2, 1.0, 3001).astype(np.float32)
    res, B, opened = _replay_fit(eng, codes, w, 21, 0.01, 0.5, m, iters)
    assert res.status == -1004 and res.iterations == iters, (res.status, res.iterations)
    assert opened <= 4


def test_fit_across_the_precision_switch(eng):
    """The bf16 -> hi+lo schedule (the data of test_gpu_fit_checkpoint's switch test): the history is dropped and
    the first direction after the switch is -g' at the re-evaluated iterate."""
    N, L = 3001, 40
    codes = synthetic.synthetic_msa_codes(N, L, 1)
    w = np.random.default_rng(2).uniform(0.2, 1.0, N).astype(np.float32)
    res, B, opened = _replay_fit(eng, codes, w, 21, 0.01, 2.0, 6, 0, schedule=1, epsilon=1e-3)
    assert 1 <= res.switched_at < res.iterations
    assert opened <= 4
