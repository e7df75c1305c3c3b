"""The one-hot operand of the tensor-core forward in its 2:4-sparse, fragment-ready form (no GPU needed).

This module is the specification of what build_xsp_kernel (evcouplings_b200/csrc/plm_tc.cu) writes and
tc_sparse_logits_kernel reads; tests/test_gpu_sparse_forward.py compares the device buffer with it byte for byte.

X[r, (j,b)] = [s_(n0+r),j = b] for the rows r < nreal of a chunk (rows beyond are zeros), K = (j,b) fastest, padded
with zero columns to Kw = round_up(L q, 64).  Every aligned group of 4 K columns holds at most 2 nonzeros (it touches
at most two sites, each with at most one nonzero), so X is the sparse A operand of wgmma.mma_async.sp.  Per group
the kept positions i0 < i1 are the nonzeros, padded with zero positions: none -> (0, 1); one at p -> (0, 1) if p <= 1,
else (0, p); two -> both.  Metadata nibble i0 | i1 << 2; kept values bf16 1.0 (0x3F80) or 0.

Layout: sequence tile T (128 rows) and K block kb (64 columns) own 10240 contiguous bytes at (T * (Kw/64) + kb) * 10240:
four fragments of 2560 bytes, [warpgroup cw = 0, 1][k32 step = 0, 1].  A fragment is 128 uint32x4 A words then 128
uint32 metadata words, one of each per thread t of the warpgroup.  Thread t covers rows r = 128 T + 64 cw + 16 (t/32)
+ (t%32)/4 and r + 8, and the 8 groups g = 16 kb + 8 step + (0..7) of the step:
    A word    {val(r, c), val(r+8, c), val(r, 4+c), val(r+8, 4+c)},  c = t % 4, val = v0 | v1 << 16
    metadata  sum_i nib(r, 4h+i) << 4i  |  nib(r+8, 4h+i) << (16 + 4i),  h = t % 2
"""
import numpy as np
import pytest

FRAG = 2560
KB_BYTES = 4 * FRAG
BF16_ONE = 0x3F80


def _ru(a, b):
    return -(-a // b) * b


def dense_onehot(codes, q, n0, nreal, xrows, kw):
    """X[r, k] as 0/1 for the rows r < xrows of the chunk starting at sequence n0 (codes >= q, the ignored gap, are
    all-zero sites)."""
    L = codes.shape[1]
    X = np.zeros((xrows, kw), dtype=np.uint8)
    rows = codes[n0:n0 + nreal].astype(np.int64)
    r, j = np.nonzero(rows < q)
    X[r, j * q + rows[r, j]] = 1
    assert L * q <= kw
    return X


def _group_tables():
    i0 = np.zeros(16, dtype=np.int64)
    i1 = np.ones(16, dtype=np.int64)
    for m in range(16):
        bits = [p for p in range(4) if m >> p & 1]
        if len(bits) == 2:
            i0[m], i1[m] = bits
        elif len(bits) == 1 and bits[0] > 1:
            i1[m] = bits[0]
    return i0, i1


def sparse_onehot(X):
    """The fragment-ready bytes of dense X (xrows x kw, xrows % 128 == 0, kw % 64 == 0)."""
    xrows, kw = X.shape
    G = X.reshape(xrows, kw // 4, 4).astype(np.int64)
    assert G.sum(axis=2).max(initial=0) <= 2, "a group of 4 holds more than 2 nonzeros"
    mask = G[..., 0] | G[..., 1] << 1 | G[..., 2] << 2 | G[..., 3] << 3
    t0, t1 = _group_tables()
    i0, i1 = t0[mask], t1[mask]
    nib = (i0 | i1 << 2).astype(np.uint32)
    val = (((mask >> i0) & 1) * BF16_ONE | (((mask >> i1) & 1) * BF16_ONE) << 16).astype(np.uint32)
    nT, nkb = xrows // 128, kw // 64
    T, kb, cw, st, t = np.meshgrid(np.arange(nT), np.arange(nkb), np.arange(2), np.arange(2), np.arange(128),
                                   indexing="ij")
    r0 = T * 128 + cw * 64 + 16 * (t >> 5) + ((t & 31) >> 2)
    r1 = r0 + 8
    g0 = kb * 16 + st * 8
    c, h = t & 3, t & 1
    A = np.stack([val[r0, g0 + c], val[r1, g0 + c], val[r0, g0 + 4 + c], val[r1, g0 + 4 + c]], axis=-1)
    E = np.zeros(r0.shape, dtype=np.uint32)
    for i in range(4):
        E |= nib[r0, g0 + 4 * h + i] << np.uint32(4 * i)
        E |= nib[r1, g0 + 4 * h + i] << np.uint32(16 + 4 * i)
    frag = np.concatenate([A.reshape(A.shape[:-2] + (512,)), E], axis=-1)      # [..., 128 * 4 + 128] uint32
    return np.ascontiguousarray(frag.astype("<u4")).view(np.uint8).reshape(-1)


def decompress(buf, xrows, kw):
    """Dense X from the fragment-ready bytes: the kept values placed at their metadata positions."""
    nT, nkb = xrows // 128, kw // 64
    words = buf[:nT * nkb * KB_BYTES].view("<u4").reshape(nT, nkb, 2, 2, 640)
    A = words[..., :512].reshape(nT, nkb, 2, 2, 128, 4)
    E = words[..., 512:]
    X = np.zeros((xrows, kw), dtype=np.uint8)
    T, kb, cw, st, t = np.meshgrid(np.arange(nT), np.arange(nkb), np.arange(2), np.arange(2), np.arange(128),
                                   indexing="ij")
    r0 = T * 128 + cw * 64 + 16 * (t >> 5) + ((t & 31) >> 2)
    g0 = kb * 16 + st * 8
    c, h = t & 3, t & 1
    # the value words each thread holds: (row offset, group offset, register)
    for roff, gsel, reg in ((0, 0, 0), (8, 0, 1), (0, 4, 2), (8, 4, 3)):
        g = g0 + gsel + c
        # metadata of (row, group) lives with the thread of the same row whose t % 2 selects the group's half
        half = (gsel + c) // 4
        tm = (t & ~3) | (half & 1) | (c & 2)           # same row; t % 2 = half (t % 4 = half or half + 2)
        e = E[T, kb, cw, st, tm] >> np.uint32((16 if roff else 0) + 4 * ((gsel + c) % 4))
        i0, i1 = e & 3, (e >> 2) & 3
        v = A[..., reg]
        rows = r0 + roff
        for idx, word in ((i0, v & 0xFFFF), (i1, v >> 16)):
            assert np.isin(word, (0, BF16_ONE)).all()
            X[rows, 4 * g + idx] |= (word == BF16_ONE).astype(np.uint8)
    return X


def _codes(N, L, q, gap, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, q + (1 if gap else 0), size=(N, L)).astype(np.uint8)


@pytest.mark.parametrize("gap", [False, True])
@pytest.mark.parametrize("q", range(2, 33))
def test_every_group_of_four_holds_at_most_two_nonzeros(q, gap):
    """For every alignment and every K padding: a group of 4 K columns touches at most two sites."""
    if gap and q == 32:
        pytest.skip("the ignored gap needs a code q <= 31")
    for L in range(2, 2 + 16):
        kw = _ru(L * q, 64)
        site = np.arange(kw) // q
        site[L * q:] = -1
        groups = site.reshape(-1, 4)
        for g in groups:
            real = set(int(s) for s in g if s >= 0)
            assert len(real) <= 2
        # and on data: every code pattern of two rows (all symbols, gaps included) stays within 2 per group
        codes = _codes(64, L, q, gap, q * 100 + L)
        X = dense_onehot(codes, q, 0, 64, 128, kw)
        assert X.reshape(128, -1, 4).sum(axis=2).max() <= 2


@pytest.mark.parametrize("q,gap", [(2, False), (3, False), (4, True), (5, False), (20, True), (21, False),
                                   (32, False)])
@pytest.mark.parametrize("L_off", range(4))
def test_decompression_gives_back_dense_x(q, gap, L_off):
    """The model's values and metadata decompress to dense X exactly, with the last site ending at each offset
    within a group of 4, rows beyond the chunk's real ones, and a chunk that starts at n0 > 0."""
    L = next((L for L in range(3, 7) if (L * q) % 4 == L_off), None)
    if L is None:
        pytest.skip("q = %d never ends a site at offset %d of a group" % (q, L_off))
    N = 300
    codes = _codes(N, L, q, gap, 7 * q + L_off)
    kw = _ru(L * q, 64)
    for n0, nreal, xrows in ((0, N, _ru(N, 384)), (200, 100, 384)):
        X = dense_onehot(codes, q, n0, nreal, xrows, kw)
        buf = sparse_onehot(X)
        assert buf.size == xrows // 128 * kw // 64 * KB_BYTES <= xrows * kw * 2
        assert np.array_equal(decompress(buf, xrows, kw), X)


def test_group_patterns_and_metadata_values():
    """Each 2:4 pattern's kept positions: 0, 1 or 2 nonzeros, a nonzero in each of the 4 positions."""
    i0, i1 = _group_tables()
    expect = {0b0000: (0, 1), 0b0001: (0, 1), 0b0010: (0, 1), 0b0100: (0, 2), 0b1000: (0, 3), 0b0011: (0, 1),
              0b0101: (0, 2), 0b1001: (0, 3), 0b0110: (1, 2), 0b1010: (1, 3), 0b1100: (2, 3)}
    for m, (a, b) in expect.items():
        assert (i0[m], i1[m]) == (a, b), m
        assert a < b
