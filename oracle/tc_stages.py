"""
Stage-by-stage float64 references of one tensor-core evaluation (plm_tc.cu), taken from the device's own inputs to
each stage (teacher forcing), with a bound per element where the stage is not exactly reproducible.

The evaluation is six kernels with stored intermediates (evc_plm_eval_data, buffers of evc_plm_copy_stage):

    expand_tc -> Wt_hi / Wt_lo -> sparse logits GEMM -> Zt -> plm_softmax -> Rt_hi / Rt_lo, gh_part, fx_part
    -> backward GEMM (Xt x Rt) -> Gd planes -> finalize_pairs_tc (g_J) / finalize_fields (g_h, -loglk)

Every check below compares one stage's output with a reference built from the device's copy of that stage's inputs,
so a mistake fails at the stage and the element where it happens, at any N.  A failure raises StageMismatch, which
names the stage and the first offending element.  Arrays are torch tensors; the functions run on whatever device the
tensors live on (float64 products on the GPU at production size, on the CPU in the tests of the oracle itself).

Exact stages (compared bit for bit):
* expand.  v = J_ij(a,b) for i < j, J_ji(b,a) for i > j, +0 on the diagonal blocks; hi = rn_bf16(v),
  lo = rn_bf16(v - hi) (v - hi is exact in float32).  Rows [Lq, Mp) and columns [Lq, Kw) are zero; precision mode 1
  writes no lo (it stays zero) and the same hi.  The fused forward's Wp uses the padded row map of
  expand_row<true>: row (i,a) -> (i // 8) 176 + ((i % 8) // 4) 88 + (i % 4) 21 + a, every other row zero.
* Xt.  Xt[(j,b), n] = [s_nj = b] for the chunk's real sequences, zero columns for sequences >= N, zero rows >= Lq.
* counts residuals (evc_plm_weighted_counts).  Rt_hi = rn_bf16(w_n), Rt_lo = rn_bf16(w_n - Rt_hi) at (i, s_ni),
  zero at the other states and for gaps.  gh_part is replayed bit for bit: per warp the pair sums
  z(2t) + z(2t + 1), the xor butterfly of warp_sum (offsets 16, 8, 4, 2, 1), then 0 + warp 0 + ... + warp 3.
* finalize_fields.  g_h[i,a] = sum over p = 0..7 (in order, float32) of the float32 sums of gh_part[i, t, a] over
  t = p, p + 8, ...; -loglk = the tree of 256 strided float64 sums (acc[k] = sum of fx_part[e], e = k mod 256,
  then s[k] += s[k + o] for o = 128, 64, ..., 1).
* finalize_pairs.  g_J(i<j)[a][b] = fp32(scale (B + A)), B and A the float32 plane sums (plane 0 first) of
  Gd[(j,b),(i,a)] and Gd[(i,a),(j,b)]; scale 1 for the objective, 0.5 for the counts.

Bounded stages (u = 2^-24, the float32 unit roundoff):
* logits.  |Zt - Z64| <= EPS_ACC * A, Z64 = sum_(j,b) W[(i,a),(j,b)] [s_nj = b] in float64 with W = hi + lo of the
  device's Wt (hi only in mode 1), A = the same sum of |W|; codes >= q contribute no term, so A = 0 forces Zt = 0.
  Accumulation model: the tensor core adds each wgmma's products into the float32 accumulator without rounding to
  nearest (an error below 2 u of the running sum per add, not centred); at most k_chunk K blocks (32 blocks of 64)
  are chained before the chunk is promoted by an IEEE add.  A wgmma whose products are all zero adds an exact zero,
  so only the K steps that touch one of the sequence's L present sites err: about 2 L adds (hi and lo).  The running
  sum is at most A, so the worst case is about 4 L u A (2^-14 A at L = 200), but the errors of a random-sign sum grow
  with the running sum (about sqrt(L) |W|, not A = L |W|): EPS_ACC = 2^-16, the constant of the suite's per-block
  rounding model (test_gpu_tc_edges.py), is used per element; the largest error / bound measured on an H100 was 0.06
  for the logits and 0.15 for the backward (DESIGN.md 2), and a logit off by one coupling (|W| ~ 0.1) is far above it.
* softmax.  From the device's Zt: z = fp32(Zt + h) exactly as the kernel forms it; then in float64 the max m,
  d = z - m, P = exp(d) / sum exp(d), r = w P - w [a = s], and the -loglk term w (log sum exp(d) - d_s).
  expf and logf are within 2 ulp (4 u relative) and 1 ulp; fl(z - m) moves exp(d) by |d| u.  So every device
  exp(d_a) is within theta_a = (|d_a| + 4) u of exp(d_a), the float32 sum of the q terms within max theta + (q - 1) u,
  and w / sum, P w and the subtraction of w add u each:
      |r_dev - r| <= w P rel + u |r| + w 2^-120,   rel = (2 max|d| + q + 13) u
  (the last term covers expf's underflow to a denormal).  The stored residual is hi + lo in mode 0, within
  1/2 ulp_bf16(lo) <= 2^-16 |r_dev| of r_dev, and hi in mode 1, within 1/2 ulp_bf16(hi) <= 2^-8 |r_dev|.  Exact structure: |lo| <= 1/2 ulp_bf16(hi) (a non-nearest hi
  breaks it), and residual and weight are 0 for ignored gaps and for the sequences >= N of the pair (n0, n0 + 1).
  The -loglk term is float32 (z_s - m) - logf(sum) widened to double: within w ((|d_s| + |log sum|) 3 u + sum's
  error) of the float64 value.  gh_part[i, tile, a] sums the float32 residuals of the tile's sequences in a tree of
  depth 10 (pair, 5 butterfly levels, 4 warps): |gh_dev - gh64| <= sum |r_dev - r| + 10 u sum |r|.  fx_part sums exact
  float64 products w * float32 in double: the bound is the sum of the term bounds plus 2^-50 of the absolute sum.
  A double sum of such products carries about 48 significant bits, so a non-zero partial that is a float32 number
  is a chance of about 2^-24: more than max(2, 1 %) of them fails.  A float32 per-thread sum and warp sum (fx_local
  declared float) makes every warp's sum a float32 number, and about a quarter of the double sums of the 4 warps too;
  its error stays inside the bound, which is dominated by the terms' own float32 error.
  Fused forward (mode 2): its logits are never stored, so z is the float64 logit Z64 + h and the residual bound adds
  the logit error dz_a = EPS_ACC A_a + u |z_a|: |dr_a| <= 2 w P_a max dz, |d fx term| <= 2 w max dz.
* backward.  |sum of the Gd planes - G64| <= EPS_ACC * A, G64[(j,b),(i,a)] = sum_{n < N} Xt[(j,b),n] R[(i,a),n] in
  float64 with R = hi + lo of the device's Rt (hi in mode 1), over real sequences only (a stale Rt column beyond N
  that met a non-zero Xt column would show), A the same sum of |R|.  Unchunked, each plane s is also checked against
  its K slice of ceil(num_kb / ksplit) blocks.  The same accumulation model as the logits, with up to 2 N / 16 adds
  of which only the K steps holding a sequence with s_j = b count.

generate(...) builds every buffer as the kernels would, in float32 on the CPU, and commits one of MUTATIONS (a
plausible kernel mistake) on request, so that the CPU tests show that each check catches what it is meant to.
"""
import numpy as np
import torch

EPS_ACC = 2.0 ** -16
U = 2.0 ** -24
TF_BN, TF_SITES = 176, 8

MUTATIONS = (
    "expand_hi_rz",          # expand: hi rounded toward zero instead of to nearest
    "rt_lo_dropped",         # softmax: the lo residual not written (mode 0)
    "rt_hi_rz",              # softmax: the residual's hi rounded toward zero
    "onehot_wrong_state",    # softmax: w subtracted at state s + 1 instead of s
    "gd_block_transposed",   # backward: one site pair's Gd block written transposed
    "plane_order_reversed",  # finalize_pairs: the planes summed from the last one
    "gh_tile_off_by_one",    # softmax: the g_h partials written one tile further
    "fx_local_float",        # softmax: the per-thread -loglk sum and its warp sum in float32 (fx_local a float)
    "stale_rt_meets_xt",     # backward: a stale residual column beyond N meets a non-zero Xt column
)


class StageMismatch(AssertionError):
    """A stage's output differs from its reference beyond its bound; names the stage and the element."""

    def __init__(self, stage, index, msg):
        self.stage, self.index = stage, tuple(int(v) for v in index)
        super().__init__("%s: element %s: %s" % (stage, self.index, msg))


def _first(mask):
    return tuple(int(v) for v in torch.nonzero(mask)[0].tolist())


_INT = {torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64}


def _assert_equal_bits(stage, got, want):
    """bit equality (so -0 differs from +0, as it would in the device's next stage)"""
    want = want.to(got.dtype)
    bad = got.contiguous().view(_INT[got.dtype]) != want.contiguous().view(_INT[got.dtype])
    if bool(bad.any()):
        idx = _first(bad)
        raise StageMismatch(stage, idx, "device %r, replay %r (%d elements differ)" % (
            got[idx].item(), want[idx].item(), int(bad.sum())))
    return int(got.numel())


def _assert_within(stage, err, bound, offset=(0, 0)):
    """err <= bound elementwise; returns the largest err / bound (0 / 0 counts as 0)."""
    bad = err > bound
    if bool(bad.any()):
        idx = _first(bad)
        pos = tuple(i + o for i, o in zip(idx, offset)) + idx[len(offset):]
        raise StageMismatch(stage, pos, "error %.3e over bound %.3e (%d elements)" % (
            err[idx].item(), bound[idx].item(), int(bad.sum())))
    pos = bound > 0
    return float((err[pos] / bound[pos]).max().item()) if bool(pos.any()) else 0.0


class Report(dict):
    """stage -> [elements checked, largest error / bound (None for exact stages)]"""

    def add(self, stage, n, ratio=None):
        e = self.setdefault(stage, [0, None])
        e[0] += int(n)
        if ratio is not None:
            e[1] = max(e[1] or 0.0, float(ratio))

    def lines(self):
        return ["  %-16s %12d elements  %s" % (k, v[0], "exact" if v[1] is None else "max err/bound %.3f" % v[1])
                for k, v in self.items()]


# ------------------------------------------------------------------------------------------------
# layouts
# ------------------------------------------------------------------------------------------------
def pair_index(i, j, L):
    return i * (2 * L - i - 1) // 2 + (j - i - 1)


def padded_rows(L, q):
    """expand_row<true>: the fused forward's row of (i,a), for all i, a (shape (L, q))."""
    i = torch.arange(L).view(L, 1)
    a = torch.arange(q).view(1, q)
    return (i // TF_SITES) * TF_BN + ((i % TF_SITES) // 4) * 88 + (i % 4) * 21 + a


def coupling_rows(x, L, q, rows):
    """float32 v[r, (j,b)] of the expanded couplings for the rows r = (i,a) in `rows` (1-D int64), all L q columns."""
    Lq = L * q
    rows = rows.to(x.device)
    i, a = (rows // q).view(-1, 1), (rows % q).view(-1, 1)
    c = torch.arange(Lq, device=x.device).view(1, -1)
    j, b = c // q, c % q
    lo_i, hi_j = torch.minimum(i, j), torch.maximum(i, j)
    same = i == j
    p = torch.where(same, 0, pair_index(lo_i, hi_j, L))
    off = torch.where(i < j, a * q + b, b * q + a)
    v = x[Lq + p * q * q + off]
    return torch.where(same, torch.zeros((), dtype=x.dtype, device=x.device), v)


def rn_bf16(v):
    """round to nearest even bf16 (__float2bfloat16_rn) of float32 values"""
    return v.to(torch.float32).to(torch.bfloat16)


def split_hi_lo(v):
    hi = rn_bf16(v)
    return hi, rn_bf16(v.to(torch.float32) - hi.to(torch.float32))


def bf16_value(hi, lo=None):
    """float64 value of the bf16 operand hi (+ lo)"""
    v = hi.to(torch.float64)
    return v if lo is None else v + lo.to(torch.float64)


def one_hot(codes, q, dtype=torch.float64):
    """(n, L) codes -> (n, L q) one-hot; codes >= q give zero rows"""
    n, L = codes.shape
    X = torch.zeros(n, L, q + 1, dtype=dtype, device=codes.device)
    X.scatter_(2, torch.clamp(codes, max=q).unsqueeze(2).to(torch.int64), 1.0)
    return X[:, :, :q].reshape(n, L * q)


def _row_blocks(n, size):
    return [(s, min(n, s + size)) for s in range(0, n, size)]


# ------------------------------------------------------------------------------------------------
# exact stages
# ------------------------------------------------------------------------------------------------
def check_expand(rep, hi, lo, x, L, q, single, padded=False, rows=None, block=1024):
    """Wt (Wp with padded=True) against the expansion of x, bit for bit.  rows: the operand rows to check (default
    all); hi or lo None to skip it.  Returns the number of elements checked."""
    stage = "expand" + (" (Wp)" if padded else "")
    ref = hi if hi is not None else lo                   # either buffer may be left out (None)
    Lq, Kw = L * q, ref.shape[1]
    if padded:
        rmap = padded_rows(L, q).reshape(-1).to(ref.device)
    else:
        rmap = torch.arange(Lq, device=ref.device)
    src = torch.full((ref.shape[0],), -1, dtype=torch.int64, device=ref.device)
    src[rmap] = torch.arange(Lq, device=ref.device)
    rows = torch.arange(ref.shape[0], device=ref.device) if rows is None else rows.to(ref.device)
    n = 0
    for s, e in _row_blocks(len(rows), block):
        r = rows[s:e]
        sr = src[r]
        real = sr >= 0
        v = torch.zeros(len(r), Kw, dtype=torch.float32, device=ref.device)
        if bool(real.any()):
            v[real, :Lq] = coupling_rows(x, L, q, sr[real]).to(torch.float32)
        h_ref, l_ref = split_hi_lo(v)
        for name, got, want in (("hi", hi, h_ref), ("lo", lo, l_ref)):
            if got is None:
                continue
            if name == "lo" and single:
                want = torch.zeros_like(want)
            g = got[r]
            bad = g.view(torch.int16) != want.view(torch.int16)
            if bool(bad.any()):
                k, c = _first(bad)
                raise StageMismatch(stage + " " + name, (int(r[k]), c), "device %r, expected %r" % (
                    g[k, c].item(), want[k, c].item()))
            n += g.numel()
    rep.add(stage, n)
    return n


def check_xt(rep, xt, codes, q, nreal, cols=None):
    """Xt [Mp][Kp] of a chunk whose first nreal columns are the sequences codes[:nreal] (codes: (nreal, L))."""
    Lq = codes.shape[1] * q
    cols = [(0, xt.shape[1])] if cols is None else cols
    n = 0
    for c0, c1 in cols:
        for s, e in _row_blocks(c1 - c0, 8192):
            a, b = c0 + s, c0 + e
            want = torch.zeros(xt.shape[0], b - a, dtype=torch.bfloat16, device=xt.device)
            r1 = min(b, nreal)
            if r1 > a:
                want[:Lq, :r1 - a] = one_hot(codes[a:r1], q, torch.float32).T.to(torch.bfloat16)
            bad = xt[:, a:b].view(torch.int16) != want.view(torch.int16)
            if bool(bad.any()):
                r, c = _first(bad)
                raise StageMismatch("Xt", (r, a + c), "device %r, expected %r" % (
                    xt[r, a + c].item(), want[r, c].item()))
            n += want.numel()
    rep.add("Xt", n)
    return n


def finalize_fields_replay(gh_part, fx_part, q):
    """finalize_fields_kernel: gh_part (L, ntiles, S) float32, fx_part (L ntiles,) float64 or None"""
    L, nt, _ = gh_part.shape
    parts = []
    for p in range(8):
        tot = torch.zeros(L, q, dtype=torch.float32, device=gh_part.device)
        for t in range(p, nt, 8):
            tot = tot + gh_part[:, t, :q]
        parts.append(tot)
    gh = torch.zeros(L, q, dtype=torch.float32, device=gh_part.device)
    for p in range(8):
        gh = gh + parts[p]
    if fx_part is None:
        return gh, None
    f = fx_part.reshape(-1)
    m = -(-f.numel() // 256) * 256
    pad = torch.zeros(m, dtype=torch.float64, device=f.device)
    pad[:f.numel()] = f
    pad = pad.view(-1, 256)
    acc = torch.zeros(256, dtype=torch.float64, device=f.device)
    for k in range(pad.shape[0]):
        acc = acc + pad[k]
    o = 128
    while o > 0:
        acc = torch.cat([acc[:o] + acc[o:2 * o], acc[o:]])
        o //= 2
    return gh, acc[0]


def check_finalize_fields(rep, gh_part, fx_part, q, g_h, fx):
    gh, f = finalize_fields_replay(gh_part, fx_part, q)
    n = _assert_equal_bits("finalize_fields g_h", g_h.reshape(gh.shape), gh)
    if fx_part is not None:
        _assert_equal_bits("finalize_fields fx", fx.reshape(1), f.reshape(1))
        n += 1
    rep.add("finalize_fields", n)
    return n


def plane_sum(gd, L, q):
    """float32 sum of the planes of Gd (P, Mp, Np) in order, restricted to [Lq, Lq]"""
    Lq = L * q
    s = gd[0, :Lq, :Lq].clone()
    for p in range(1, gd.shape[0]):
        s = s + gd[p, :Lq, :Lq]
    return s


def finalize_pairs_replay(gd, L, q, scale):
    S4 = plane_sum(gd, L, q).reshape(L, q, L, q)                  # [j, b, i, a]
    iu, ju = torch.triu_indices(L, L, 1, device=gd.device)
    B = S4[ju, :, iu, :].transpose(1, 2)                          # Gd[(j,b),(i,a)] as [a][b]
    A = S4[iu, :, ju, :]                                          # Gd[(i,a),(j,b)]
    return (B + A) * torch.tensor(scale, dtype=torch.float32, device=gd.device)


def check_finalize_pairs(rep, gd, L, q, scale, gJ):
    want = finalize_pairs_replay(gd, L, q, scale)
    n = _assert_equal_bits("finalize_pairs", gJ.reshape(want.shape), want)
    rep.add("finalize_pairs", n)
    return n


def counts_residual(codes, w, q):
    """(hi, lo) of the counts' residual operand rows (i,a) x sequences: w_n at (i, s_ni); codes (n, L), w (n,) fp32"""
    hi, lo = split_hi_lo(w)
    X = one_hot(codes, q, torch.float32).T > 0                    # (Lq, n)
    zero = torch.zeros((), dtype=torch.bfloat16, device=X.device)  # +0 at the other states, as the kernel writes
    return torch.where(X, hi.view(1, -1), zero), torch.where(X, lo.view(1, -1), zero)


def counts_gh_replay(codes, w, q, S, ntiles, block=32):
    """gh_part (L, ntiles, S) float32 of plm_softmax_kernel<ONEHOT> for the 256-sequence tiles covering codes
    (n, L) with weights w (n,); sequences beyond n have weight 0.  Computed `block` tiles at a time."""
    n, L = codes.shape
    out = torch.zeros(L, ntiles, S, dtype=torch.float32, device=codes.device)
    for t0 in range(0, ntiles, block):
        t1 = min(ntiles, t0 + block)
        out[:, t0:t1] = _counts_gh_tiles(codes[t0 * 256:t1 * 256], w[t0 * 256:t1 * 256], q, S)
    return out


def _counts_gh_tiles(codes, w, q, S):
    n, L = codes.shape
    nt = -(-n // 256)
    c = torch.full((nt * 256, L), q, dtype=torch.int64, device=codes.device)
    c[:n] = codes
    ww = torch.zeros(nt * 256, dtype=torch.float32, device=codes.device)
    ww[:n] = w
    ww = ww.view(-1, 1) * (c < q)
    z = torch.zeros(nt * 256, L, q, dtype=torch.float32, device=codes.device)
    z.scatter_(2, torch.clamp(c, max=q - 1).unsqueeze(2), ww.unsqueeze(2))
    z = torch.where((c < q).unsqueeze(2), z, torch.zeros((), device=z.device))
    z = z.view(nt, 4, 32, 2, L, q)                                # tile, warp, lane, pair, site, state
    v = z[:, :, :, 0] + z[:, :, :, 1]                            # (nt, 4, 32, L, q)
    lane = torch.arange(32, device=z.device)
    for o in (16, 8, 4, 2, 1):
        v = v + v[:, :, lane ^ o]
    v = v[:, :, 0]                                                # lane 0: (nt, 4, L, q)
    tot = torch.zeros(nt, L, q, dtype=torch.float32, device=z.device)
    for wi in range(4):
        tot = tot + v[:, wi]
    out = torch.zeros(L, nt, S, dtype=torch.float32, device=z.device)
    out[:, :, :q] = tot.permute(1, 0, 2)
    return out


def check_counts_residual(rep, rt_hi, rt_lo, codes, w, q, nreal, full_columns=True):
    """the counts' Rt of a chunk: nreal real columns, exact zeros beyond (full_columns: up to Kp, unchunked)"""
    hi, lo = counts_residual(codes[:nreal], w[:nreal], q)
    Lq = hi.shape[0]
    c1 = rt_hi.shape[1] if full_columns else nreal
    n = 0
    for name, got, want in (("hi", rt_hi, hi), ("lo", rt_lo, lo)):
        full = torch.zeros(got.shape[0], c1, dtype=torch.bfloat16, device=got.device)
        full[:Lq, :nreal] = want
        n += _assert_equal_bits("counts Rt_" + name, got[:, :c1], full)
    rep.add("counts Rt", n)
    return n


# ------------------------------------------------------------------------------------------------
# bounded stages
# ------------------------------------------------------------------------------------------------
def logits_ref(W_hi, W_lo, codes, q):
    """Z64 and A (Lq x n) for the sequences codes (n, L); W_lo None in mode 1"""
    Lq = codes.shape[1] * q
    W = bf16_value(W_hi[:Lq, :Lq], None if W_lo is None else W_lo[:Lq, :Lq])
    Xt = one_hot(codes, q).T
    return W @ Xt, W.abs() @ Xt


def check_logits(rep, zt, W_hi, W_lo, codes, q, cols, eps=EPS_ACC, block=8192):
    """Zt [Mp][Ns] (chunk-local columns) on the column ranges cols, codes[c] the sequence of column c"""
    Lq = codes.shape[1] * q
    worst, n = 0.0, 0
    W = bf16_value(W_hi[:Lq, :Lq], None if W_lo is None else W_lo[:Lq, :Lq])
    Wa = W.abs()
    for c0, c1 in cols:
        for s, e in _row_blocks(c1 - c0, block):
            a, b = c0 + s, c0 + e
            Xt = one_hot(codes[a:b], q).T
            Z, A = W @ Xt, Wa @ Xt
            got = zt[:Lq, a:b].to(torch.float64)
            worst = max(worst, _assert_within("logits", (got - Z).abs(), eps * A, (0, a)))
            n += Z.numel()
    rep.add("logits", n, worst)
    return worst


def softmax_ref(z, s, w, q, dz=None):
    """z (n, L, q) logits with h (float32 as the kernel forms them, or float64 with dz (n, L, q) their error bound),
    s (n, L) codes, w (n,) float32 (0 beyond N).  Returns float64 r, r_bound, fx term and its bound, and the fp32
    weight actually used (0 for gaps)."""
    z = z.to(torch.float64)
    present = s < q
    we = torch.where(present, w.to(torch.float64).view(-1, 1), torch.zeros((), dtype=torch.float64, device=z.device))
    m = z.max(dim=2, keepdim=True).values
    d = z - m
    e = torch.exp(d)
    se = e.sum(dim=2, keepdim=True)
    P = e / se
    X = torch.zeros_like(z)
    X.scatter_(2, torch.clamp(s, max=q - 1).unsqueeze(2).to(torch.int64), 1.0)
    X = X * present.unsqueeze(2)
    W = we.unsqueeze(2)
    r = W * (P - X)
    dmax = d.abs().max(dim=2, keepdim=True).values
    rel = (2 * dmax + q + 13) * U
    rb = W * P * rel + U * r.abs() + W * 2.0 ** -120
    ls = torch.log(se)[..., 0]
    ds = (d * X).sum(dim=2)
    fx = we * (ls - ds)
    fxb = we * ((ds.abs() + ls.abs()) * 3 * U + rel[..., 0] + U * (ls - ds).abs())
    if dz is not None:
        dzm = dz.max(dim=2, keepdim=True).values * 1.01
        rb = rb + 2 * W * P * dzm
        fxb = fxb + 2 * we * dzm[..., 0]
    return r, rb, fx, fxb


def check_softmax(rep, zt_or_z, h, codes, w, q, N, n0, single, rt_hi, rt_lo, gh_part, fx_part, cols, tile=256,
                  fused=None, full_columns=False, block=8192):
    """plm_softmax_kernel (or the fused epilogue) on the chunk starting at global sequence n0.
    zt_or_z: the device's Zt [Mp][Ns] (chunk-local columns); fused: (W_hi, W_lo) of the fused forward, whose logits
    are recomputed in float64 from the codes (zt_or_z is then ignored).  codes / w: the chunk's sequences (n, L) /
    (n,) (w = 0 beyond N).  cols: column ranges, starting on `tile` boundaries of the global sequence index.
    gh_part (L, ntiles, S) and fx_part (L, ntiles) are checked on the tiles those ranges cover.
    full_columns: the Rt columns from N to Kp (never written, or written as zeros) must be zero as well."""
    L = codes.shape[1]
    Lq = L * q
    hq = h.reshape(L, q).to(torch.float32)
    worst_r, worst_gh, worst_fx, n_r, n_t = 0.0, 0.0, 0.0, 0, 0
    fx_part = fx_part.reshape(L, -1)
    n_fp32_fx, n_fx, first_fp32 = 0, 0, None
    for c0, c1 in cols:
        for s0, e0 in _row_blocks(c1 - c0, block):
            a, b = c0 + s0, c0 + e0
            nb = b - a
            sc = codes[a:b].to(torch.int64)
            wc = w[a:b].to(torch.float32)
            if fused is None:
                z = (zt_or_z[:Lq, a:b].T.reshape(nb, L, q) + hq.unsqueeze(0))         # float32, as the kernel
                r, rb, fx, fxb = softmax_ref(z, sc, wc, q)
            else:
                Z, A = logits_ref(fused[0], fused[1], codes[a:b], q)
                z = Z.T.reshape(nb, L, q) + hq.to(torch.float64).unsqueeze(0)
                dz = EPS_ACC * A.T.reshape(nb, L, q) + U * z.abs()
                r, rb, fx, fxb = softmax_ref(z, sc, wc, q, dz)
            # stored residuals
            hi = rt_hi[:Lq, a:b].T.reshape(nb, L, q)
            if single:
                dev = hi.to(torch.float64)
                bound = rb + 2.0 ** -8 * (r.abs() + rb)
            else:
                lo = rt_lo[:Lq, a:b].T.reshape(nb, L, q)
                dev = hi.to(torch.float64) + lo.to(torch.float64)
                bound = rb + 2.0 ** -16 * (r.abs() + rb)
                # |lo| <= 1/2 ulp_bf16(hi): hi is the nearest bf16 of the float32 residual
                hv = hi.to(torch.float32)
                _m, ex = torch.frexp(hv)
                half = torch.where(hv != 0, torch.ldexp(torch.ones_like(hv), ex - 9),
                                   torch.full_like(hv, 2.0 ** -126))
                bad = lo.to(torch.float32).abs() > half
                if bool(bad.any()):
                    k, i, st = _first(bad)
                    raise StageMismatch("softmax Rt_hi", (i * q + st, a + k), "hi %r is not the nearest bf16: lo %r" % (
                        hv[k, i, st].item(), lo[k, i, st].item()))
            zero = (r == 0) & (rb == 0)                    # gaps and sequences >= N: exactly zero
            bad = zero & (dev != 0)
            if bool(bad.any()):
                k, i, st = _first(bad)
                raise StageMismatch("softmax Rt", (i * q + st, a + k), "residual %r of a zero-weight entry" %
                                    dev[k, i, st].item())
            err = (dev - r).abs()
            bad = err > bound
            if bool(bad.any()):
                k, i, st = _first(bad)
                raise StageMismatch("softmax Rt", (i * q + st, a + k), "residual %r, float64 %r, bound %.3e" % (
                    dev[k, i, st].item(), r[k, i, st].item(), bound[k, i, st].item()))
            pos = bound > 0
            if bool(pos.any()):
                worst_r = max(worst_r, float((err[pos] / bound[pos]).max()))
            n_r += r.numel()
            # per-tile partials (the block starts on a tile boundary of the global index)
            g0 = (n0 + a) // tile
            nt = -(-nb // tile)
            pad = nt * tile - nb
            rr = torch.nn.functional.pad(r, (0, 0, 0, 0, 0, pad)).view(nt, tile, L, q)
            rbb = torch.nn.functional.pad(rb, (0, 0, 0, 0, 0, pad)).view(nt, tile, L, q)
            gh64 = rr.sum(dim=1).permute(1, 0, 2)                                     # (L, nt, q)
            ghb = (rbb.sum(dim=1) + 10 * U * (rr.abs() + rbb).sum(dim=1)).permute(1, 0, 2)
            ghd = gh_part[:, g0:g0 + nt, :].to(torch.float64)
            if ghd.shape[2] > q and bool((ghd[:, :, q:] != 0).any()):
                i, t, st = _first(ghd[:, :, q:] != 0)
                raise StageMismatch("softmax gh_part", (i, g0 + t, q + st), "padding state not zero")
            worst_gh = max(worst_gh, _assert_within("softmax gh_part", (ghd[:, :, :q] - gh64).abs(), ghb, (0, g0)))
            fxx = torch.nn.functional.pad(fx, (0, 0, 0, pad)).view(nt, tile, L)
            fxbb = torch.nn.functional.pad(fxb, (0, 0, 0, pad)).view(nt, tile, L)
            f64 = fxx.sum(dim=1).T                                                    # (L, nt)
            fb = fxbb.sum(dim=1).T + 2.0 ** -50 * fxx.abs().sum(dim=1).T
            fd = fx_part[:, g0:g0 + nt]
            worst_fx = max(worst_fx, _assert_within("softmax fx_part", (fd - f64).abs(), fb, (0, g0)))
            nzf = fd != 0
            n_fx += int(nzf.sum())
            is32 = nzf & (fd.to(torch.float32).to(torch.float64) == fd)
            n_fp32_fx += int(is32.sum())
            if first_fp32 is None and bool(is32.any()):
                i_, t_ = _first(is32)
                first_fp32 = (i_, g0 + t_)
            n_t += gh64.numel()
    if n_fp32_fx > max(2, n_fx // 100):
        raise StageMismatch("softmax fx_part", first_fp32, "%d of %d partials are float32 numbers: the -loglk terms were "
                            "not summed in float64" % (n_fp32_fx, n_fx))
    if full_columns:
        c_end = max(c1 for _c0, c1 in cols)
        for name, buf in (("hi", rt_hi), ("lo", rt_lo)):
            if buf is None:
                continue
            tail = buf[:, c_end:]
            if tail.numel() and bool((tail.to(torch.float32) != 0).any()):
                r_, c_ = _first(tail.to(torch.float32) != 0)
                raise StageMismatch("softmax Rt_" + name, (r_, c_end + c_), "column beyond N not zero")
            pad_rows = buf[Lq:, :c_end]
            if pad_rows.numel() and bool((pad_rows.to(torch.float32) != 0).any()):
                r_, c_ = _first(pad_rows.to(torch.float32) != 0)
                raise StageMismatch("softmax Rt_" + name, (Lq + r_, c_), "padding row not zero")
    rep.add("softmax Rt", n_r, worst_r)
    rep.add("softmax gh_part", n_t, worst_gh)
    rep.add("softmax fx_part", n_t // q if q else 0, worst_fx)
    return worst_r


def xt_columns(xt, Lq):
    """column provider of check_backward: the device's Xt"""
    return lambda a, b: xt[:Lq, a:b].to(torch.float64)


def codes_columns(codes, q):
    """column provider of check_backward: the one-hot of the codes (n, L) (the chunked runs: Xt holds one chunk)"""
    return lambda a, b: one_hot(codes[a:b], q).T


def rt_columns(rt_hi, rt_lo, Lq):
    """column provider of check_backward: the device's residual operand, hi + lo (rt_lo None: hi)"""
    return lambda a, b: bf16_value(rt_hi[:Lq, a:b], None if rt_lo is None else rt_lo[:Lq, a:b])


def check_backward(rep, gd, L, q, nreal, X, R, ksplit=None, num_kb=None, eps=EPS_ACC, block=8192, label="backward"):
    """Gd planes against the float64 product sum_{n < nreal} X[:, n] R[:, n]^T; X and R are column providers
    (xt_columns, codes_columns, rt_columns).  ksplit (with num_kb, the K blocks of the product): check every plane
    against its K slice of ceil(num_kb / ksplit) blocks too (unchunked runs)."""
    Lq = L * q

    def product(a, b):
        G = torch.zeros(Lq, Lq, dtype=torch.float64, device=gd.device)
        A = torch.zeros_like(G)
        for s, e in _row_blocks(max(0, b - a), block):
            Xb, Rb = X(a + s, a + e), R(a + s, a + e)
            G += Xb @ Rb.T
            A += Xb @ Rb.abs().T
        return G, A

    worst, n = 0.0, 0
    if ksplit is not None and ksplit > 1:
        per = -(-num_kb // ksplit)
        for p in range(ksplit):
            a, b = p * per * 64, min(num_kb, (p + 1) * per) * 64
            G, A = product(a, min(b, nreal))
            worst = max(worst, _assert_within("%s plane %d" % (label, p),
                                              (gd[p, :Lq, :Lq].to(torch.float64) - G).abs(), eps * A))
            n += G.numel()
    G, A = product(0, nreal)
    tot = gd[:, :Lq, :Lq].to(torch.float64).sum(dim=0)
    worst = max(worst, _assert_within(label, (tot - G).abs(), eps * A))
    n += G.numel()
    for p in range(gd.shape[0]):
        for blk, off in ((gd[p, Lq:, :], (p, Lq, 0)), (gd[p, :Lq, Lq:], (p, 0, Lq))):
            if blk.numel() and bool((blk != 0).any()):
                r, c = _first(blk != 0)
                raise StageMismatch(label, (p, off[1] + r, off[2] + c), "padding of Gd not zero")
    rep.add(label, n, worst)
    return worst


def check_backward_rows(rep, gd, rows, L, q, nreal, X, R, eps=EPS_ACC, label="backward rows"):
    """the rows `rows` (1-D int64) of the plane sum of Gd against float64, as check_backward (for Gd too large to
    hold a float64 copy of: the rows on both sides of an element offset)"""
    Lq = L * q
    rows = rows.to(gd.device)
    Xr = X(0, nreal)                                   # (Lq, nreal)
    real = rows < Lq
    G = torch.zeros(len(rows), Lq, dtype=torch.float64, device=gd.device)
    A = torch.zeros_like(G)
    if bool(real.any()):
        Xs, Rb = Xr[rows[real]], R(0, nreal)
        G[real], A[real] = Xs @ Rb.T, Xs @ Rb.abs().T
    got = gd[:, rows, :].to(torch.float64).sum(dim=0)
    worst = _assert_within(label, (got[:, :Lq] - G).abs(), eps * A)
    if got.shape[1] > Lq and bool((got[:, Lq:] != 0).any()):
        r, c = _first(got[:, Lq:] != 0)
        raise StageMismatch(label, (int(rows[r]), Lq + c), "padding column of Gd not zero")
    rep.add(label, G.numel(), worst)
    return worst


# ------------------------------------------------------------------------------------------------
# generate mode: every buffer as the kernels would write it (float32, CPU), with an optional mutation
# ------------------------------------------------------------------------------------------------
def _rz_bf16(v):
    return (v.to(torch.float32).view(torch.int32) & ~0xFFFF).view(torch.float32).to(torch.bfloat16)


def generate(x, codes, w, q, single=False, ksplit=3, mutation=None):
    """Buffers of one unchunked evaluation and of the counts, built in float32 / float64 on the CPU as the kernels
    would (logits and the backward product as float32 roundings of float64 sums, the softmax in float32 as
    plm_softmax_kernel).  x float32 (n_params,), codes (N, L) uint8, w (N,) float32.  Returns a dict of torch
    tensors in the layouts of evc_plm_copy_stage plus g, fx and the counts."""
    if mutation is not None and mutation not in MUTATIONS:
        raise ValueError("unknown mutation " + mutation)
    x = torch.as_tensor(x, dtype=torch.float32)
    c = torch.as_tensor(codes.astype(np.int64))
    N, L = c.shape
    Lq = L * q
    S = q if q % 2 else q + 1
    ru = lambda a, b: -(-a // b) * b                                           # noqa: E731
    Mp, Np, Kw, Kp = ru(Lq, 128), ru(Lq, 192), ru(Lq, 64), ru(N, 64)
    nt = -(-N // 256)
    wt = torch.as_tensor(w, dtype=torch.float32)
    out = dict(Mp=Mp, Np=Np, Kw=Kw, Kp=Kp, ntiles=nt, ksplit=ksplit, N=N, L=L, q=q, single=single)
    # expand
    v = torch.zeros(Mp, Kw, dtype=torch.float32)
    v[:Lq, :Lq] = coupling_rows(x, L, q, torch.arange(Lq))
    hi, lo = split_hi_lo(v)
    if mutation == "expand_hi_rz":
        hi = _rz_bf16(v)
        lo = rn_bf16(v - hi.to(torch.float32))
    if single:
        lo = torch.zeros_like(lo)
    out["Wt_hi"], out["Wt_lo"] = hi, lo
    # logits
    Z, _A = logits_ref(hi, None if single else lo, c, q)
    zt = torch.zeros(Mp, ru(N, 192), dtype=torch.float32)
    zt[:Lq, :N] = Z.to(torch.float32)
    out["Zt"] = zt
    # softmax, in float32 like plm_softmax_kernel
    h = x[:Lq].view(L, q)
    z = zt[:Lq, :N].T.reshape(N, L, q) + h
    mx = z.max(dim=2, keepdim=True).values
    e = torch.exp(z - mx)
    ssum = torch.zeros(N, L, 1, dtype=torch.float32)
    for a in range(q):
        ssum = ssum + e[:, :, a:a + 1]
    present = c < q
    wn = torch.where(present, wt.view(-1, 1), torch.zeros(()))
    inv = wn.unsqueeze(2) / ssum
    state = (c + 1) % q if mutation == "onehot_wrong_state" else c
    X = torch.zeros(N, L, q)
    X.scatter_(2, torch.clamp(state, max=q - 1).unsqueeze(2), 1.0)
    X = X * present.unsqueeze(2)
    r = e * inv - X * wn.unsqueeze(2)
    zs = (z * X).sum(dim=2) if mutation != "onehot_wrong_state" else (z * torch.nn.functional.one_hot(
        torch.clamp(c, max=q - 1), q) * present.unsqueeze(2)).sum(dim=2)
    term32 = (zs - mx[..., 0]) - torch.log(ssum[..., 0])                    # float32 as the kernel
    prod = wn.to(torch.float64) * term32.to(torch.float64)         # exact products, as the kernel forms them
    rt_hi = torch.zeros(Np, Kp, dtype=torch.bfloat16)
    rt_lo = torch.zeros(Np, Kp, dtype=torch.bfloat16)
    rf = r.reshape(N, Lq).T
    rh, rl = split_hi_lo(rf)
    if mutation == "rt_hi_rz":
        rh = _rz_bf16(rf)
        rl = rn_bf16(rf - rh.to(torch.float32))
    if mutation == "rt_lo_dropped":
        rl = torch.zeros_like(rl)
    rt_hi[:Lq, :N] = rh
    if not single:
        rt_lo[:Lq, :N] = rl
    if mutation == "stale_rt_meets_xt" and Kp > N:
        rt_hi[:Lq, N:] = rt_hi[:Lq, :1]
    out["Rt_hi"], out["Rt_lo"] = rt_hi, (None if single else rt_lo)
    # per-tile partials (float32 tree, float64 -loglk)
    pad = nt * 256 - N
    rp = torch.nn.functional.pad(r, (0, 0, 0, 0, 0, pad)).view(nt, 128, 2, L, q)
    gt = torch.zeros(nt, L, q, dtype=torch.float32)
    for k in range(128):
        gt = gt + (rp[:, k, 0] + rp[:, k, 1])
    gh_part = torch.zeros(L, nt, S, dtype=torch.float32)
    gh_part[:, :, :q] = gt.permute(1, 0, 2)
    if mutation == "gh_tile_off_by_one":
        gh_part = torch.roll(gh_part, 1, dims=1)
    fx_part = _fx_tiles(prod, nt, mutation == "fx_local_float")
    out["gh_part"], out["fx_part"] = gh_part, fx_part
    # backward
    xt = torch.zeros(Mp, Kp, dtype=torch.bfloat16)
    xt[:Lq, :N] = one_hot(c, q, torch.float32).T.to(torch.bfloat16)
    if mutation == "stale_rt_meets_xt" and Kp > N:
        xt[:Lq, N:] = xt[:Lq, :1]
    out["Xt"] = xt
    R = bf16_value(rt_hi, None if single else rt_lo)
    num_kb = Kp // 64
    per = -(-num_kb // ksplit)
    gd = torch.zeros(ksplit, Mp, Np, dtype=torch.float32)
    for p in range(ksplit):
        a, b = p * per * 64, min(num_kb, (p + 1) * per) * 64
        gd[p] = (xt[:, a:b].to(torch.float64) @ R[:, a:b].T).to(torch.float32)
    if mutation == "gd_block_transposed":
        i, j = 0, L - 1
        blk = gd[0, j * q:(j + 1) * q, i * q:(i + 1) * q].clone()
        gd[0, j * q:(j + 1) * q, i * q:(i + 1) * q] = blk.T
    out["Gd"] = gd
    gJ = finalize_pairs_replay(gd.flip(0) if mutation == "plane_order_reversed" else gd, L, q, 1.0)
    gh, fx = finalize_fields_replay(gh_part, fx_part, q)
    out["g"] = torch.cat([gh.reshape(-1), gJ.reshape(-1)])
    out["fx"] = fx
    # counts
    chi, clo = counts_residual(c, wt, q)
    crt_hi = torch.zeros(Np, Kp, dtype=torch.bfloat16)
    crt_lo = torch.zeros(Np, Kp, dtype=torch.bfloat16)
    crt_hi[:Lq, :N], crt_lo[:Lq, :N] = chi, clo
    cgh = counts_gh_replay(c, wt, q, S, nt)
    CR = bf16_value(crt_hi, crt_lo)
    cgd = torch.zeros(1, Mp, Np, dtype=torch.float32)
    cgd[0] = (xt.to(torch.float64) @ CR.T).to(torch.float32)
    fi, _ = finalize_fields_replay(cgh, None, q)
    out["counts"] = dict(Rt_hi=crt_hi, Rt_lo=crt_lo, gh_part=cgh, Gd=cgd, fi=fi.reshape(-1),
                         fij=finalize_pairs_replay(cgd, L, q, 0.5).reshape(-1))
    return out


def _fx_tiles(prod, nt, float_acc=False):
    """fx_part (L, nt) of plm_softmax_kernel from the products w * float32 term (N, L): per thread
    fx_local = (0 - p(2t)) - p(2t + 1), the xor butterfly of warp_sum, then (s0 + s1) + (s2 + s3) in double.
    float_acc: fx_local and its warp sum in float32 (each double result rounded on assignment)."""
    N, L = prod.shape
    p = torch.nn.functional.pad(prod, (0, 0, 0, nt * 256 - N)).view(nt, 4, 32, 2, L)
    if float_acc:
        v = (0.0 - p[:, :, :, 0]).to(torch.float32)
        v = (v.to(torch.float64) - p[:, :, :, 1]).to(torch.float32)
    else:
        v = (0.0 - p[:, :, :, 0]) - p[:, :, :, 1]
    lane = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[:, :, lane ^ o]
    sw = v[:, :, 0].to(torch.float64)                               # (nt, 4, L)
    return ((sw[:, 0] + sw[:, 1]) + (sw[:, 2] + sw[:, 3])).T.contiguous()


def check_generated(buf, x, codes, w, q):
    """Every check on the buffers of generate(); returns the Report"""
    rep = Report()
    x = torch.as_tensor(x, dtype=torch.float32)
    c = torch.as_tensor(codes.astype(np.int64))
    wt = torch.as_tensor(w, dtype=torch.float32)
    N, L = c.shape
    Lq = L * q
    single = buf["single"]
    check_expand(rep, buf["Wt_hi"], buf["Wt_lo"], x, L, q, single)
    check_xt(rep, buf["Xt"], c, q, N)
    check_logits(rep, buf["Zt"], buf["Wt_hi"], None if single else buf["Wt_lo"], c, q, [(0, N)])
    check_softmax(rep, buf["Zt"], x[:Lq], c, wt, q, N, 0, single, buf["Rt_hi"], buf["Rt_lo"], buf["gh_part"],
                  buf["fx_part"], [(0, N)], full_columns=True)
    check_backward(rep, buf["Gd"], L, q, N, xt_columns(buf["Xt"], Lq), rt_columns(buf["Rt_hi"], buf["Rt_lo"], Lq),
                   ksplit=buf["ksplit"], num_kb=buf["Kp"] // 64)
    check_finalize_pairs(rep, buf["Gd"], L, q, 1.0, buf["g"][Lq:])
    check_finalize_fields(rep, buf["gh_part"], buf["fx_part"], q, buf["g"][:Lq], buf["fx"])
    cb = buf["counts"]
    check_counts_residual(rep, cb["Rt_hi"], cb["Rt_lo"], c, wt, q, N)
    S = q if q % 2 else q + 1
    _assert_equal_bits("counts gh_part", cb["gh_part"], counts_gh_replay(c, wt, q, S, buf["ntiles"]))
    check_finalize_fields(rep, cb["gh_part"], None, q, cb["fi"], None)
    check_backward(rep, cb["Gd"], L, q, N, xt_columns(buf["Xt"], Lq), rt_columns(cb["Rt_hi"], cb["Rt_lo"], Lq),
                   label="counts backward")
    check_finalize_pairs(rep, cb["Gd"], L, q, 0.5, cb["fij"])
    return rep
