"""The kernels that consume a fitted model, at the launch geometries and 64-bit offsets their other tests never reach
(-m gpu), each against a plain float64 or integer reference:

* the Gibbs sampler (sample.cu) with 13, 2 and 1 chains per CTA, partial last CTAs, and U beyond 2^31 entries,
  draw for draw against the restatement of oracle/potts_sampler.py (models and power: test_sampler_geometry_oracle);
* evc_code_counts with several site CTAs, one code row per stage and more than 2^31 counters, and evc_bm_update on
  that many parameters, against oracle/boltzmann.py;
* the energy kernel at every row stride S = 3 ... 33 and its chunk widths 24, 20, 16 and 12, at L = 2300 (W beyond
  2^31 floats), and over batches of hamiltonians();
* evc_fn_scores and evc_ec_scores for every q in 2 ... 32 up to L = 800.

The large cases print their runtime and the device memory in use at their largest point (total minus free)."""
import ctypes
import time

import numpy as np
import pytest

from oracle import boltzmann as bm
from test_sampler_geometry_oracle import (CTA2, CTA13, FAR, FAR_SITES, POWER, chains_per_cta, clean_after, cta2_model,
                                          cta13_model, far_model, pair_index, restatement)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from evcouplings_b200 import _lib
    from evcouplings_b200.engine import CudaEngine
    _lib.require_device()
    return CudaEngine()


def _mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def device_free(eng):
    import torch
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info(eng.device)[0]


def device_used(eng):
    import torch
    torch.cuda.synchronize()
    free, total = torch.cuda.mem_get_info(eng.device)
    return total - free


def need_device(eng, nbytes):
    free = device_free(eng)
    if free < nbytes:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (nbytes / 1e9, free / 1e9))


def need_host(nbytes):
    if _mem_available() < nbytes:
        pytest.skip("needs %.1f GB of host memory, %.1f GB available" % (nbytes / 1e9, _mem_available() / 1e9))


def pairs_of(p, L):
    """(i, j) of pair indices p (row-major i < j)."""
    i0 = np.arange(L, dtype=np.int64)
    first = i0 * (2 * L - i0 - 1) // 2
    i = np.searchsorted(first, p, side="right") - 1
    return i, p - first[i] + i + 1


# ---- the sampler ---------------------------------------------------------------------------------------------------

def device_x(eng, h, pairs, blocks):
    """x = [h | J] on the device, J zero outside the listed pair blocks (no host copy of the whole J)."""
    import torch
    L, q = h.shape
    lq = L * q
    x = torch.zeros(lq + L * (L - 1) // 2 * q * q, dtype=torch.float32, device=eng.device)
    x[:lq] = torch.from_numpy(np.ascontiguousarray(h, dtype=np.float32).ravel()).to(eng.device)
    idx = torch.from_numpy(pair_index(pairs[:, 0], pairs[:, 1], L)).to(eng.device)
    x[lq:].view(-1, q * q)[idx] = torch.from_numpy(blocks.reshape(-1, q * q).astype(np.float32)).to(eng.device)
    return x


class DeviceChains(object):
    """evc_sampler_* on an x already on the device."""

    def __init__(self, eng, x, L, q, n, seed):
        import torch
        from evcouplings_b200 import _lib
        self.eng, self.L, self.n = eng, L, n
        torch.cuda.synchronize()
        self.handle = ctypes.c_void_p()
        _lib.check(eng.lib.evc_sampler_create(ctypes.byref(self.handle), eng.ptr(x), L, q, None, n, 0, seed,
                                              eng.device_index), "evc_sampler_create")

    def run(self, sweeps, beta):
        from evcouplings_b200 import _lib
        ch = ctypes.c_int64()
        _lib.check(self.eng.lib.evc_sampler_run(self.handle, sweeps, beta, ctypes.byref(ch), self.eng.stream()),
                   "evc_sampler_run")
        return int(ch.value)

    def codes(self):
        import torch
        out = torch.empty((self.n, self.L), dtype=torch.uint8, device=self.eng.device)
        assert self.eng.lib.evc_sampler_codes(self.handle, self.eng.ptr(out), self.eng.stream()) == 0
        return out.cpu().numpy()

    def close(self):
        if self.handle:
            self.eng.lib.evc_sampler_destroy(self.handle)
            self.handle = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


@pytest.mark.parametrize("name", ["CTA13", "CTA2", "FAR"])
def test_sampler_geometry_against_restatement(eng, name):
    """Every chain's codes equal the restatement's after every sweep before the sweep of its first near-tie draw, the
    chains that leave it are all flagged, and the share compared is the one fixed on the CPU.  FAR: one chain per
    CTA, U of (L q)^2 = 2.33e9 entries; the last three sites change within the compared prefix, so the refresh and
    those changes read rows of U beyond entry 2^31."""
    case = dict(CTA13=CTA13, CTA2=CTA2, FAR=FAR)[name]
    h, pairs, blocks = dict(CTA13=cta13_model, CTA2=cta2_model, FAR=far_model)[name]()
    L, q, n, sweeps, beta = case["L"], case["q"], case["n"], case["sweeps"], case["beta"]
    lq = L * q
    need_device(eng, 4 * (lq * lq + lq + L * (L - 1) // 2 * q * q + n * lq) + (1 << 30))
    ref = restatement(case, (h, pairs, blocks))
    base = device_used(eng)
    t0 = time.time()
    x = device_x(eng, h, pairs, blocks)
    diverged = np.zeros(n, dtype=bool)
    compared = np.zeros(n, dtype=np.int64)
    last = np.zeros(3, dtype=np.int64)
    device_s = 0.0
    with DeviceChains(eng, x, L, q, n, case["seed"]) as s:
        peak = device_used(eng) - base
        del x
        before = s.codes()
        for t in range(sweeps):
            t1 = time.time()
            ch = s.run(1, beta)
            got = s.codes()
            device_s += time.time() - t1
            ref.run(1, beta)
            clean = clean_after(ref, t)
            same = np.all(got == ref.codes(), axis=1)
            assert same[clean].all(), (name, t, np.flatnonzero(clean & ~same)[:8])
            if clean.all():
                assert ch == ref.changes
            diverged |= ~same
            compared += clean
            last += ((got[:, -3:] != before[:, -3:]) & clean[:, None]).sum(axis=0)
            before = got
    print("%s: L=%d q=%d, %d chains (%d per CTA), %d sweeps: %.1f s in all, %.1f s on the device; %.2f GB device "
          "memory for the sampler; compared %.3f of the chain-sweeps; last-site changes %s"
          % (name, L, q, n, chains_per_cta(L, q), sweeps, time.time() - t0, device_s, peak / 1e9,
             compared.sum() / (n * sweeps), last))
    flagged = ref.first_tie >= 0
    assert not (diverged & ~flagged).any()
    assert compared.sum() >= POWER[name] * n * sweeps
    per_cta = chains_per_cta(L, q)
    if per_cta > 1:                                                     # the partial last CTA was compared
        assert (compared[-(n % per_cta):] > 0).all()
    if name == "FAR":
        assert (last > 0).all() and FAR_SITES[-3:] == (L - 3, L - 2, L - 1)


# ---- counts and the update ----------------------------------------------------------------------------------------

def device_counts(eng, d_codes, N, L, q):
    import torch
    out = torch.full((L * q + L * (L - 1) // 2 * q * q,), -1, dtype=torch.int32, device=eng.device)
    assert eng.lib.evc_code_counts(eng.ptr(d_codes), N, L, q, eng.ptr(out), eng.stream()) == 0, \
        eng.lib.evc_last_error()
    return out


def site_counts(codes, L, q):
    return np.concatenate([np.bincount(codes[:, i], minlength=q) for i in range(L)]).astype(np.uint32)


def pair_counts(codes, q, p, L):
    """(len(p), q q) uint32 integer counts of the pairs with indices p."""
    i, j = pairs_of(np.asarray(p, dtype=np.int64), L)
    c = codes.astype(np.int64)
    idx = (np.arange(len(p), dtype=np.int64) * q * q)[None, :] + c[:, i] * q + c[:, j]
    return np.bincount(idx.ravel(), minlength=len(p) * q * q).astype(np.uint32).reshape(len(p), q * q)


def check_every_counter(eng, codes, L, q):
    import torch
    N = len(codes)
    d = torch.from_numpy(np.ascontiguousarray(codes)).to(eng.device)
    got = device_counts(eng, d, N, L, q)
    lq, npairs = L * q, L * (L - 1) // 2
    assert np.array_equal(got[:lq].cpu().numpy().view(np.uint32), site_counts(codes, L, q))
    step = max(1, (1 << 24) // max(N, q * q))
    pc = got[lq:].view(npairs, q * q)
    for p0 in range(0, npairs, step):
        p = np.arange(p0, min(npairs, p0 + step))
        want = pair_counts(codes, q, p, L)
        assert np.array_equal(pc[p0:p0 + len(p)].cpu().numpy().view(np.uint32), want), (L, q, N, p0)


@pytest.mark.parametrize("L,q,Ns", [(513, 32, (1, 1237)), (1025, 32, (1, 333)), (781, 21, (1, 1237)),
                                    (16385, 2, (1, 3)), (20000, 2, (5,))])
def test_code_counts_plan_edges(eng, L, q, Ns):
    """2 and 3 site CTAs at q = 32 (512 sites per CTA), 2 at q = 21 (780), one code row per stage from L = 16385
    on (the 32 KB stage holds one row and rows * L does not divide it)."""
    per_site_cta = min(L, 65536 // (4 * q))
    assert L > per_site_cta or L >= 16385
    assert (32768 // L <= 1) == (L >= 16385)
    rng = np.random.default_rng(L + q)
    for N in Ns:
        codes = rng.integers(0, q, (N, L)).astype(np.uint8)
        if N > 1:
            codes[: N // 3, -1] = q - 1                 # a skewed last site
        check_every_counter(eng, codes, L, q)


def test_counts_and_update_beyond_2_31(eng):
    """q = 3, L = 22000: n = 2.18e9 > 2^31 counters and parameters.  Counts: every site counter, the first and last
    pair blocks, the blocks whose counters straddle index 2^31 and 20000 random blocks.  evc_bm_update: slices at the
    start, around 2^31 and at the end bit for bit against oracle/boltzmann.py, and both maxima against torch float64
    over all n (the largest coupling deviation is planted beyond 2^31)."""
    import torch
    L, q, N = 22000, 3, 5
    lq, npairs = L * q, L * (L - 1) // 2
    n = lq + npairs * q * q
    assert n > 2 ** 31
    need_device(eng, 3 * 4 * n + (6 << 30))
    rng = np.random.default_rng(22)
    codes = rng.integers(0, q, (N, L)).astype(np.uint8)
    codes[:2, L - 1] = 0
    base = device_used(eng)
    t0 = time.time()
    got = device_counts(eng, torch.from_numpy(codes).to(eng.device), N, L, q)
    torch.cuda.synchronize()
    t_counts = time.time() - t0
    assert np.array_equal(got[:lq].cpu().numpy().view(np.uint32), site_counts(codes, L, q))
    p_mid = (2 ** 31 - lq) // (q * q)
    blocks = np.unique(np.concatenate([np.arange(4), np.arange(npairs - 4, npairs), np.arange(p_mid - 3, p_mid + 4),
                                       rng.integers(0, npairs, 20000)]))
    assert lq + p_mid * q * q <= 2 ** 31 < lq + (p_mid + 1) * q * q
    pc = got[lq:].view(npairs, q * q)
    want = pair_counts(codes, q, blocks, L)
    assert np.array_equal(pc[torch.from_numpy(blocks).to(eng.device)].cpu().numpy().view(np.uint32), want)

    # the update: x, f uniform; f = 1.5 at one coupling beyond 2^31 with a zero count there: |c/M - f| <= 1 elsewhere
    g = torch.Generator(device=eng.device)
    g.manual_seed(5)
    x = torch.rand(n, generator=g, device=eng.device).sub_(0.5)
    f = torch.rand(n, generator=g, device=eng.device).mul_(0.5)
    k_far = n - 1234567
    k_far += int(np.flatnonzero(got[k_far:k_far + 100].cpu().numpy() == 0)[0])
    assert k_far > 2 ** 31
    f[k_far] = 1.5
    slices = [(0, 2 * lq), (2 ** 31 - 40000, 2 ** 31 + 40000), (k_far - 1000, k_far + 1000), (n - 50000, n)]
    before = [(x[a:b].cpu().numpy(), got[a:b].cpu().numpy().view(np.uint32), f[a:b].cpu().numpy()) for a, b in slices]
    stats = torch.full((2,), -1.0, dtype=torch.float64, device=eng.device)
    eta, lam2_h, lam2_J = 0.3, 0.01, 0.002
    peak = device_used(eng) - base
    t1 = time.time()
    assert eng.lib.evc_bm_update(eng.ptr(x), eng.ptr(got), N, eng.ptr(f), n, lq, eta, lam2_h, lam2_J,
                                 eng.ptr(stats), eng.stream()) == 0
    torch.cuda.synchronize()
    t_update = time.time() - t1
    for (a, b), (xs, cs, fs) in zip(slices, before):
        want_x, want_st = bm.update(xs, cs, N, fs, max(0, min(b, lq) - a), eta, lam2_h, lam2_J)
        assert np.array_equal(x[a:b].cpu().numpy().view(np.uint32), want_x.view(np.uint32)), (a, b)
    dev = [0.0, 0.0]
    step = 1 << 27
    for a in range(0, n, step):
        b = min(n, a + step)
        d = (got[a:b].to(torch.float64) / N - f[a:b].to(torch.float64)).abs()
        if a < lq:
            dev[0] = max(dev[0], float(d[:lq - a].max()))
        if b > lq:
            dev[1] = max(dev[1], float(d[max(0, lq - a):].max()))
    assert dev[1] == 1.5
    assert stats.cpu().numpy().tolist() == dev
    print("counts and update at n = %d: counts %.2f s, update %.3f s, %.1f GB device memory" %
          (n, t_counts, t_update, peak / 1e9))


# ---- energies -------------------------------------------------------------------------------------------------------

def energy_jc(S):
    """Sites per streamed chunk of the energy kernel (model_ops.cu energy_jc)."""
    return min(24, 113 * 1024 // (2 * S * (S + 1) * 4) // 4 * 4)


def stride(q):
    return q if q % 2 else q + 1


def test_every_chunk_width_is_covered():
    widths = {energy_jc(stride(q)) for q in range(2, 33)}
    assert widths == {24, 20, 16, 12}
    assert [energy_jc(S) for S in (23, 25, 27, 29, 31, 33)] == [24, 20, 16, 16, 12, 12]


def energy_reference(h, J, codes):
    """(N, 3) float64 energies and the per-row scale sum |terms| (codes == q: ignored gap)."""
    N, L = codes.shape
    q = h.shape[1]
    hp = np.zeros((L, q + 1))
    hp[:, :q] = h
    Jp = np.zeros((len(J), q + 1, q + 1))
    Jp[:, :q, :q] = J
    iu, ju = np.triu_indices(L, 1)
    terms = Jp[np.arange(len(iu))[None, :], codes[:, iu], codes[:, ju]]
    ht = hp[np.arange(L)[None, :], codes]
    hj, hh = terms.sum(axis=1), ht.sum(axis=1)
    return np.stack([hj + hh, hj, hh], axis=1), np.abs(terms).sum(axis=1) + np.abs(ht).sum(axis=1)


def check_energies(H, ref, scale, L, what):
    tol = L * 2.0 ** -24 * scale + 1e-12                 # tolerance of test_gpu_model_ops_alphabets.py
    for col in range(3):
        bad = np.nonzero(np.abs(H[:, col] - ref[:, col]) > tol)[0]
        assert len(bad) == 0, (what, col, bad[:5], H[bad[:5], col], ref[bad[:5], col])


ENERGY_CASES = [(q, L, gaps) for q in range(2, 33)
                for L in sorted({energy_jc(stride(q)), energy_jc(stride(q)) + 1, 2 * energy_jc(stride(q)) + 1})
                for gaps in ((False, True) if q < 32 else (False,))]


@pytest.mark.parametrize("q,L,gaps", ENERGY_CASES)
def test_hamiltonians_every_stride(eng, q, L, gaps):
    """Every q (so every stride S = 3 ... 33) at L = W, W + 1 and 2 W + 1 for its chunk width W, N = 1, 511, 513."""
    from evcouplings_b200 import model_ops
    rng = np.random.default_rng(1000 * q + L + gaps)
    m = dict(L=L, q=q, h=rng.normal(0, 0.5, (L, q)).astype(np.float32),
             J=rng.normal(0, 0.2, (L * (L - 1) // 2, q, q)).astype(np.float32))
    for N in (1, 511, 513):
        codes = rng.integers(0, q, (N, L)).astype(np.uint8)
        if gaps:
            codes[rng.random((N, L)) < 0.15] = q
            codes[0, :] = q
        H = model_ops.hamiltonians(m, codes, eng)
        ref, scale = energy_reference(m["h"].astype(np.float64), m["J"].astype(np.float64), codes)
        check_energies(H, ref, scale, L, (q, L, gaps, N))
        if gaps:
            assert (H[0] == 0.0).all()


def test_hamiltonians_beyond_2_31_and_batching(eng):
    """L = 2300, q = 21 (the FAR model): the per-site offsets of W pass 2^31 floats from site 2160 on.  Every row
    against float64, and two batchings that split N unevenly bit-identical to one batch."""
    from evcouplings_b200 import model_ops
    h, pairs, blocks = far_model()
    L, q = h.shape
    npairs = L * (L - 1) // 2
    S, Lp = stride(q), -(-L // 4) * 4
    assert (L - 1) * Lp * (q + 1) * S > 2 ** 31
    need_host(12 * npairs * q * q + (4 << 30))
    need_device(eng, 2 * L * Lp * (q + 1) * S * 4 + 4 * npairs * q * q + (4 << 30))
    J = np.zeros((npairs, q, q), dtype=np.float32)
    J[pair_index(pairs[:, 0], pairs[:, 1], L)] = blocks
    m = dict(L=L, q=q, h=h.astype(np.float32), J=J)
    rng = np.random.default_rng(23)
    N = 700
    codes = rng.integers(0, q, (N, L)).astype(np.uint8)
    base = device_used(eng)
    t0 = time.time()
    H = model_ops.hamiltonians(m, codes, eng)
    t_one = time.time() - t0
    hp = h.astype(np.float64)
    terms = blocks[np.arange(len(pairs))[None, :], codes[:, pairs[:, 0]], codes[:, pairs[:, 1]]]
    ht = hp[np.arange(L)[None, :], codes]
    ref = np.stack([terms.sum(axis=1) + ht.sum(axis=1), terms.sum(axis=1), ht.sum(axis=1)], axis=1)
    check_energies(H, ref, np.abs(terms).sum(axis=1) + np.abs(ht).sum(axis=1), L, "L=2300")
    for bs in (256, 300):
        Hb = model_ops.hamiltonians(m, codes, eng, batch_size=bs)
        assert np.array_equal(Hb.view(np.uint64), H.view(np.uint64)), bs
    print("hamiltonians at L = 2300, q = 21, N = 700: %.1f s for one batch (device memory in use before: %.1f GB)"
          % (t_one, base / 1e9))


def test_hamiltonians_batching_small(eng):
    from evcouplings_b200 import model_ops
    rng = np.random.default_rng(3)
    L, q = 30, 21
    m = dict(L=L, q=q, h=rng.normal(0, 0.5, (L, q)).astype(np.float32),
             J=rng.normal(0, 0.2, (L * (L - 1) // 2, q, q)).astype(np.float32))
    codes = rng.integers(0, q + 1, (1237, L)).astype(np.uint8)
    H = model_ops.hamiltonians(m, codes, eng)
    for bs in (1, 100, 513, 2048):
        assert np.array_equal(model_ops.hamiltonians(m, codes, eng, batch_size=bs).view(np.uint64), H.view(np.uint64))


# ---- EC scores ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("L", [2, 33, 800])
@pytest.mark.parametrize("q", list(range(2, 33)))
def test_pair_scores_every_alphabet(eng, q, L):
    """evc_ec_scores (raw and zero-sum FN, MI) and evc_fn_scores per pair against torch float64, with the tolerances
    of test_pair_scores_every_pair.  At L = 800 the pair -> (i, j) walk of the MI reaches i = 798."""
    import torch
    from evcouplings_b200 import _lib
    dev = eng.device
    npair = L * (L - 1) // 2
    g = torch.Generator(device=dev)
    g.manual_seed(100 * q + L)
    J = torch.randn((npair, q, q), generator=g, device=dev) * 0.2
    fij = torch.rand((npair, q, q), generator=g, device=dev)
    fij[:, 0, :] = 0.0                                  # zero f_ij entries are skipped by the MI
    fij /= fij.sum(dim=(1, 2), keepdim=True)
    fi = torch.rand((L, q), generator=g, device=dev)
    fi[0, : q // 2] = 0.0
    fi /= fi.sum(dim=1, keepdim=True)
    out = torch.zeros((4, npair), dtype=torch.float32, device=dev)
    _lib.check(eng.lib.evc_ec_scores(eng.ptr(J), eng.ptr(fij), eng.ptr(fi), L, q, eng.ptr(out[0]), eng.ptr(out[1]),
                                     eng.ptr(out[2]), eng.stream()), "evc_ec_scores")
    _lib.check(eng.lib.evc_fn_scores(eng.ptr(J), L, q, eng.ptr(out[3]), eng.stream()), "evc_fn_scores")
    iu, ju = (torch.from_numpy(v).to(dev) for v in np.triu_indices(L, 1))
    fi64 = fi.double()
    step = max(1, (1 << 24) // (q * q))
    for a in range(0, npair, step):
        b = min(npair, a + step)
        Jd = J[a:b].double()
        raw = Jd.square().sum(dim=(1, 2)).sqrt()
        Jz = Jd - Jd.mean(dim=1, keepdim=True) - Jd.mean(dim=2, keepdim=True) + Jd.mean(dim=(1, 2), keepdim=True)
        zs = Jz.square().sum(dim=(1, 2)).sqrt()
        F = fij[a:b].double()
        P = fi64[iu[a:b]][:, :, None] * fi64[ju[a:b]][:, None, :]
        ok = (F > 0) & (P > 0)
        t = torch.where(ok, F * torch.log(torch.where(ok, F, 1.0) / torch.where(ok, P, 1.0)), 0.0)
        mi = t.sum(dim=(1, 2))
        o = out[:, a:b].double()
        assert bool(((o[0] - raw).abs() <= 2.0 ** -23 * raw + 1e-30).all()), (q, L, a)
        assert bool(((o[3] - raw).abs() <= 2.0 ** -23 * raw + 1e-30).all()), (q, L, a)
        assert bool(((o[1] - zs).abs() <= 2.0 ** -23 * zs + 1e-12 * raw).all()), (q, L, a)
        assert bool(((o[2] - mi).abs() <= 2.0 ** -23 * mi.abs() + 1e-12 * t.abs().sum(dim=(1, 2))).all()), (q, L, a)
        assert bool((ok.sum(dim=(1, 2)) < q * q).all())
