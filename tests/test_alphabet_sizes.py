"""
Alphabets of any size the engine supports (no GPU): 2 <= q <= 32 model states with the gap as a state, 2 <= q <= 31
with ignore_gaps (the gap is coded q), i.e. every code below 32, the 5 bit-planes of the Hamming pass.

* run_plmc and bin/evcplm-plmc -a refuse an alphabet outside that range before ingest and before any engine exists;
* evc_plm_tc_bytes_alphabet / evc_plm_create_alphabet / evc_hamming_counts (host code of the built library) accept
  exactly that range, while evc_plm_tc_bytes / evc_plm_create keep taking q in {4, 5, 20, 21} only;
* with the test-only oracle engine, run_plmc at q = 22 and q = 6 writes a .model that reads back intact.

The helpers below (alphabets, synthetic alignments over any alphabet) are shared with test_gpu_alphabet_sizes.py.
"""
import ctypes
import io
import os

import numpy as np
import pytest

from evcouplings_b200 import _lib, model_ops, msa, plmc_cli, tools
from oracle import plm_oracle as po

# gap first; 32 distinct characters in all (digits are plain symbols of the alphabet)
SYMBOLS = "-ACDEFGHIKLMNPQRSTVWYXBZJOU123456789"
PROTEIN_X = "-ACDEFGHIKLMNPQRSTVWYX"          # q = 22: protein with X kept as a state
DNA_N = "-ACGTN"                              # q = 6: a sixth nucleotide state
TWO_LETTERS = "AB"                            # q = 2: 'A' is the alphabet's gap character, a state


def alphabet_of(n):
    """n distinct characters, gap first"""
    assert 1 <= n <= len(SYMBOLS)
    return SYMBOLS[:n]


def alphabet_codes(N, L, n_symbols, seed, gap_prob=0.05):
    """Family-structured (N, L) codes over n_symbols characters in the gap-as-state convention (0 = the alphabet's
    first character): ceil(N / 50) random centres, per-sequence mutation probability U(0.1, 0.6), per-site gaps;
    row 0 has no gap."""
    rng = np.random.default_rng(seed)
    K = max(1, -(-N // 50))
    centres = rng.integers(0, n_symbols, size=(K, L))
    codes = centres[rng.integers(0, K, size=N)]
    mut = rng.random((N, L)) < rng.uniform(0.1, 0.6, size=N)[:, None]
    codes = np.where(mut, rng.integers(0, n_symbols, size=(N, L)), codes)
    gaps = rng.random((N, L)) < gap_prob
    gaps[0, :] = False
    return np.where(gaps, 0, codes).astype(np.uint8)


def write_alphabet_a2m(path, codes, alphabet):
    """codes in the gap-as-state convention of ``alphabet`` -> A2M text"""
    chars = np.frombuffer(alphabet.encode("ascii"), dtype=np.uint8)[codes]
    with open(path, "w") as f:
        for n in range(codes.shape[0]):
            f.write(">seq%d/1-%d\n%s\n" % (n, codes.shape[1], bytes(chars[n]).decode("ascii")))


class _NoEngine(object):
    """An engine that must never be touched."""

    def __getattr__(self, name):
        raise AssertionError("the engine was used (%s) although the alphabet is invalid" % name)


# (alphabet, ignore_gaps): 1, 33 and 34 characters; 2 characters with the gap ignored (q = 1)
INVALID = [(alphabet_of(1), False), (alphabet_of(33), False), (alphabet_of(34), False), (alphabet_of(2), True),
           (alphabet_of(33), True), (alphabet_of(1), True)]


@pytest.mark.parametrize("alphabet,ignore_gaps", INVALID, ids=lambda v: str(len(v)) if isinstance(v, str) else
                         ("ignore_gaps" if v else "gap_state"))
def test_run_plmc_refuses_alphabet_before_any_work(tmp_path, monkeypatch, alphabet, ignore_gaps):
    a2m = tmp_path / "a.a2m"
    write_alphabet_a2m(str(a2m), alphabet_codes(20, 6, 2, 1), "AB")

    def no_ingest(*a, **k):
        raise AssertionError("the alignment was read although the alphabet is invalid")

    monkeypatch.setattr(msa, "load_alignment", no_ingest)
    monkeypatch.setattr(tools, "_default_engine", lambda: _NoEngine())
    for engine in (_NoEngine(), None):
        with pytest.raises(tools.InvalidParameterError, match=r"2 <= q <= 3[12]"):
            tools.run_plmc(str(a2m), str(tmp_path / "x_ECs.txt"), str(tmp_path / "x.model"), alphabet=alphabet,
                           ignore_gaps=ignore_gaps, engine=engine)
    assert not os.path.exists(tmp_path / "x_ECs.txt")


@pytest.mark.parametrize("alphabet,ignore_gaps", INVALID, ids=lambda v: str(len(v)) if isinstance(v, str) else
                         ("ignore_gaps" if v else "gap_state"))
def test_cli_refuses_alphabet(tmp_path, alphabet, ignore_gaps):
    a2m = tmp_path / "a.a2m"
    write_alphabet_a2m(str(a2m), alphabet_codes(20, 6, 2, 1), "AB")
    argv = ["-c", str(tmp_path / "x_ECs.txt"), "-a", alphabet] + (["-g"] if ignore_gaps else []) + [str(a2m)]
    err = io.StringIO()
    assert plmc_cli.main(argv, engine=_NoEngine(), stderr=err) == 2
    assert "-a:" in err.getvalue() and "below 32" in err.getvalue(), err.getvalue()


def test_alphabet_range():
    for n in range(2, 33):
        assert msa.alphabet_states(alphabet_of(n)) == n
    for n in range(3, 33):
        assert msa.alphabet_states(alphabet_of(n), ignore_gaps=True) == n - 1
    with pytest.raises(ValueError, match="repeated"):
        msa.alphabet_states("-AA")
    ids, raw = ["s0", "s1"], np.frombuffer(b"ACGTACGT", dtype=np.uint8).reshape(2, 4)
    with pytest.raises(msa.AlignmentError, match="2 <= q <= 32"):
        msa.encode_alignment(ids, raw, alphabet=alphabet_of(33))
    ali = msa.encode_alignment(ids, raw, alphabet="-ACGTN", ignore_gaps=True)
    assert (ali.q, ali.gap_code, ali.model_alphabet) == (5, 5, "ACGTN")


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def _tc_bytes(lib, N, L, q, gap_code, seq_chunk=0, sm=132):
    out = ctypes.c_int64(-1)
    rc = lib.evc_plm_tc_bytes_alphabet(N, L, q, gap_code, seq_chunk, sm, ctypes.byref(out))
    return rc, int(out.value)


def test_tc_bytes_accepts_exactly_the_supported_range(lib):
    for q in range(0, 36):
        for gap in (-1, q):
            rc, _ = _tc_bytes(lib, 1000, 50, q, gap)
            ok = 2 <= q <= (31 if gap >= 0 else 32)
            assert (rc == 0) == ok, (q, gap, lib.evc_last_error())
            if not ok:
                assert b"2 <= q <= 32" in lib.evc_last_error()
            # the existing entry point keeps its alphabets; where both apply they agree
            out = ctypes.c_int64(-1)
            rc_old = lib.evc_plm_tc_bytes(1000, 50, q, gap, 0, 132, ctypes.byref(out))
            assert (rc_old == 0) == (q in (4, 5, 20, 21)), (q, gap)
            if rc_old == 0:
                assert int(out.value) == _tc_bytes(lib, 1000, 50, q, gap)[1]


def test_alphabet_tc_bytes_rejects_bad_arguments():
    """engine.alphabet_tc_bytes (what the planners use): the arguments engine.tc_bytes checks, and a number of states
    outside 2..32 (q = 7 is an alphabet like any other here; engine.tc_bytes still refuses it)"""
    from evcouplings_b200.engine import alphabet_tc_bytes, plan_seq_chunk, tc_bytes
    SM = 132
    for args in ((0, 10, 21, -1, 0, SM), (100, 1, 21, -1, 0, SM), (100, 10, 33, -1, 0, SM), (100, 10, 32, 32, 0, SM),
                 (100, 10, 21, 5, 0, SM), (100, 10, 21, -1, -1, SM), (100, 10, 21, -1, 0, 0)):
        with pytest.raises(_lib.EngineError):
            alphabet_tc_bytes(*args)
    assert alphabet_tc_bytes(100, 10, 7, -1, 0, SM) > 0
    with pytest.raises(_lib.EngineError):
        tc_bytes(100, 10, 7, -1, 0, SM)
    assert alphabet_tc_bytes(50000, 200, 21, -1, 0, SM) == tc_bytes(50000, 200, 21, -1, 0, SM)
    # the planner takes any supported alphabet: q = 32, 300k x 150 needs chunks with 9 GB free
    c = plan_seq_chunk(300000, 150, 32, -1, 6, SM, 9e9)
    assert c > 0 and c % 768 == 0


@pytest.mark.parametrize("q,gap", [(3, False), (13, True), (22, False), (25, True), (31, True), (32, False)])
def test_tc_bytes_matches_the_geometry_mirror(lib, q, gap):
    """the byte count is built from the tensor-core geometry at every q (mirror of test_gpu_tc_edges.geometry, the
    device-side check compares it with the handle's real allocations)"""
    import test_gpu_tc_edges as edges
    for N, L, chunk in ((1000, 50, 0), (2001, 97, 768), (300, 7, 0)):
        g = edges.geometry(N, L, q, gap, chunk, 132)
        assert _tc_bytes(lib, N, L, q, q if gap else -1, chunk)[1] == g["bytes"], (N, L, q, gap)


def test_create_and_hamming_refuse_codes_beyond_the_range(lib):
    """host-side checks of the built library, before any device work"""
    vp = ctypes.c_void_p
    w = np.ones(4, dtype=np.float32)
    codes = np.zeros((4, 3), dtype=np.uint8)
    h = ctypes.c_void_p()
    for q, gap in ((1, -1), (33, -1), (32, 32), (0, -1)):
        rc = lib.evc_plm_create_alphabet(ctypes.byref(h), codes.ctypes.data_as(vp), 4, 3, q, gap, w.ctypes.data_as(vp),
                                         0)
        assert rc != 0 and b"unsupported number of states" in lib.evc_last_error(), lib.evc_last_error()
    for q in (7, 22, 32):           # evc_plm_create keeps its alphabets and names the entry point that takes these
        rc = lib.evc_plm_create(ctypes.byref(h), codes.ctypes.data_as(vp), 4, 3, q, -1, w.ctypes.data_as(vp), 0)
        assert rc != 0 and b"evc_plm_create_alphabet" in lib.evc_last_error(), lib.evc_last_error()
    counts = np.zeros(4, dtype=np.int32)
    codes[1, 2] = 32
    rc = lib.evc_hamming_counts(codes.ctypes.data_as(vp), 4, 3, 2, 0, counts.ctypes.data_as(vp))
    assert rc != 0 and b"codes must be < 32" in lib.evc_last_error(), lib.evc_last_error()


@pytest.mark.parametrize("alphabet", [PROTEIN_X, DNA_N])
def test_run_plmc_with_oracle_engine_writes_the_alphabet(tmp_path, alphabet):
    from cpu_engine import OracleEngine
    q, N, L = len(alphabet), 90, 9
    codes = alphabet_codes(N, L, q, 3)
    a2m = tmp_path / "a.a2m"
    write_alphabet_a2m(str(a2m), codes, alphabet)
    ecs, model = tmp_path / "x_ECs.txt", tmp_path / "x.model"
    res, run = tools.run_plmc(str(a2m), str(ecs), str(model), alphabet=alphabet, theta=0.8, iterations=8,
                              lambda_h=0.01, lambda_J=0.01 * (q - 1) * (L - 1), engine=OracleEngine(),
                              return_run=True)
    assert run.alignment.q == q and np.array_equal(run.alignment.codes, codes)
    m = model_ops.read_model(str(model))
    assert (m["L"], m["q"], m["n_valid"], m["alphabet"]) == (L, q, N, alphabet)
    assert m["h"].shape == (L, q) and m["J"].shape == (L * (L - 1) // 2, q, q)
    assert np.allclose(m["J"].ravel(), run.x[L * q:]) and np.allclose(m["h"].ravel(), run.x[:L * q])
    fi_o, fij_o = po.frequencies(run.alignment.codes, run.weights, q, -1)
    assert np.abs(m["fi"] - fi_o).max() < 1e-6 and np.abs(m["fij"] - fij_o).max() < 1e-6
    m2 = po.read_model(str(model))
    assert m2["alphabet"] == alphabet and m2["q"] == q
    assert len(open(ecs).read().strip().split("\n")) == L * (L - 1) // 2
    # the same alphabet without its gap state
    res, run = tools.run_plmc(str(a2m), str(ecs), str(model), alphabet=alphabet, ignore_gaps=True, theta=0.8,
                              iterations=4, engine=OracleEngine(), return_run=True)
    m = model_ops.read_model(str(model))
    assert (m["q"], m["alphabet"]) == (q - 1, alphabet[1:]) and run.alignment.gap_code == q - 1
