"""
Distinct rows on the CPU: run_plmc's host logic when some valid rows repeat over the focus columns.  A test-only
engine gives the oracle backend a numpy model of evc_msa_unique and of the multiplicity-weighted Hamming counts; the
model itself is checked here against np.unique and the full-row oracle counts.  Covers the bit-identical counts,
weights, N_eff and .model header, the untouched path without repeats, two gloo ranks sharding the distinct pair
tiles, and checkpoints (bit-identical resume, a changed row table refused).
"""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from evcouplings_b200 import checkpoint, synthetic, tools  # noqa: E402
from test_fit_checkpoint import CkOracleEngine, CkOracleProblem, CkShardedEngine  # noqa: E402


# ---- numpy models -------------------------------------------------------------------------------------------------
def unique_rows_model(codes):
    """(first, inverse, mult) as evc_msa_unique defines them, from np.unique with the distinct rows re-sorted by
    their first occurrence."""
    codes = np.ascontiguousarray(codes, dtype=np.uint8)
    _, idx, inv, cnt = np.unique(codes, axis=0, return_index=True, return_inverse=True, return_counts=True)
    order = np.argsort(idx)
    rank = np.empty(len(order), dtype=np.int64)
    rank[order] = np.arange(len(order))
    return idx[order].astype(np.int64), rank[np.asarray(inv).reshape(-1)], cnt[order].astype(np.int64)


def hamming_tiles_model(codes, thr, mult, lo=0, hi=None):
    """evc_hamming_count_tiles_mult over upper-triangular 128 x 128 tiles lo..hi: a neighbour pair credits mult[col]
    to its row and, off the diagonal tiles, mult[row] to its column."""
    from evcouplings_b200.dist import hamming_tile_coords
    codes = np.ascontiguousarray(codes, dtype=np.uint8)
    N = len(codes)
    T = (N + 127) // 128
    hi = T * (T + 1) // 2 if hi is None else hi
    mult = np.asarray(mult, dtype=np.int64)
    counts = np.zeros(N, dtype=np.int64)
    for k in range(lo, hi):
        R, C = hamming_tile_coords(k, T)
        r0, r1, c0, c1 = R * 128, min(N, R * 128 + 128), C * 128, min(N, C * 128 + 128)
        ident = (codes[r0:r1, None, :] == codes[None, c0:c1, :]).sum(axis=2) >= thr
        counts[r0:r1] += ident.astype(np.int64) @ mult[c0:c1]
        if R != C:
            counts[c0:c1] += mult[r0:r1] @ ident.astype(np.int64)
    return counts


class _Distinct(object):
    """unique_rows / hamming_counts(mult=) of CudaEngine, on the numpy models."""
    table_calls = 0

    def unique_rows(self, codes):
        type(self).table_calls += 1
        return unique_rows_model(codes)

    def hamming_counts(self, codes, min_identical, mult=None):
        if mult is None:
            return super().hamming_counts(codes, min_identical)
        from evcouplings_b200.dist import shard_bounds
        N = len(codes)
        T = (N + 127) // 128
        lo, hi = shard_bounds(T * (T + 1) // 2, getattr(self, "world", 1), getattr(self, "rank", 0))
        counts = hamming_tiles_model(codes, min_identical, mult, lo, hi)
        if getattr(self, "world", 1) > 1:
            import torch
            t = torch.from_numpy(counts)
            self.coll.all_reduce_sum(t)
            counts = t.numpy()
        return counts.astype(np.int32)


class Recording(object):
    """Keeps the arrays the PLM problem was created with."""
    problems = []

    def plm_problem(self, codes, weights, *a, **k):
        type(self).problems.append((codes, weights))
        return super().plm_problem(codes, weights, *a, **k)


class DistinctEngine(_Distinct, Recording, CkOracleEngine):
    pass


class FullEngine(Recording, CkOracleEngine):
    pass


class DistinctShardedEngine(_Distinct, CkShardedEngine):
    pass


# ---- alignments ---------------------------------------------------------------------------------------------------
def _repeats(N=240, L=12, seed=6):
    """synthetic rows with blocks of exact copies, scattered through the alignment (row 0 is the focus)"""
    rng = np.random.default_rng(seed)
    codes = synthetic.synthetic_msa_codes(N, L, seed)
    for src in (0, 3, 17, 40):
        dst = rng.choice(np.arange(1, N), size=int(rng.integers(3, 30)), replace=False)
        codes[dst] = codes[src]
    return codes


def _a2m(tmp_path, codes, name="in.a2m"):
    path = str(tmp_path / name)
    synthetic.write_a2m(path, codes)
    return path


def _kw(a2m, tmp_path, tag, L=12, **extra):
    kw = dict(alignment=a2m, couplings_file=str(tmp_path / (tag + "_ECs.txt")),
              param_file=str(tmp_path / (tag + ".model")), focus_seq="seq0/1-%d" % L, theta=0.8, ignore_gaps=True,
              iterations=25, lambda_h=0.01, lambda_J=2.0, epsilon=1e-9)
    kw.update(extra)
    return kw


def model_head(path):
    """The .model bytes before f_i but the iteration count: dimensions, theta, lambdas, N_eff, alphabet, weights,
    target and index list."""
    raw = open(path, "rb").read()
    L, q, n_valid, n_invalid = np.frombuffer(raw[:16], dtype="<i4")
    return raw[:16] + raw[20:40 + q + 4 * (n_valid + n_invalid) + 5 * L]


@pytest.fixture(autouse=True)
def _reset():
    Recording.problems = []
    checkpoint._stop["requested"] = False
    CkOracleProblem.stop_at = None
    yield
    checkpoint._stop["requested"] = False
    CkOracleProblem.stop_at = None


# ---- the models -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,L,hi", [(1, 5, 21), (300, 1, 4), (500, 31, 32), (700, 33, 2), (257, 300, 32)])
def test_models_agree_with_full_rows(N, L, hi):
    from oracle import c_oracle as co
    rng = np.random.default_rng(N + L)
    codes = rng.integers(0, hi, size=(N, L)).astype(np.uint8)
    if N > 10:
        codes[rng.integers(0, N, N // 3)] = codes[rng.integers(0, N, N // 3)]
    first, inverse, mult = unique_rows_model(codes)
    assert np.all(np.diff(first) > 0) and mult.sum() == N
    assert np.array_equal(codes[first][inverse], codes)
    assert np.array_equal(first[inverse[first]], first)          # a first row is its own representative
    thr = max(0, int(0.8 * L))
    full = co.hamming_counts(codes, thr)
    assert np.array_equal(hamming_tiles_model(codes[first], thr, mult)[inverse], full)


# ---- run_plmc -------------------------------------------------------------------------------------------------------
def test_run_plmc_on_distinct_rows_matches_the_full_rows(tmp_path):
    codes = _repeats()
    a2m = _a2m(tmp_path, codes)
    kw = dict(iterations="max", epsilon=1e-7)
    rd, run_d = tools.run_plmc(engine=DistinctEngine(), return_run=True, **_kw(a2m, tmp_path, "d", **kw))
    rf, run_f = tools.run_plmc(engine=FullEngine(), return_run=True, **_kw(a2m, tmp_path, "f", **kw))
    (codes_d, w_d), (codes_f, w_f) = Recording.problems
    first, inverse, mult = unique_rows_model(run_f.alignment.codes)
    assert run_d.timings["unique_rows"] == len(first) < len(codes) and run_f.timings["unique_rows"] == len(codes)
    assert "unique_s" in run_d.timings
    # the problem is the distinct rows with merged float32 weights c_u * scale / n_u
    assert np.array_equal(codes_d, codes_f[first])
    assert np.array_equal(w_d, (mult / run_f.counts[first].astype(np.float64)).astype(np.float32))
    # counts, weights, N_eff bit-identical; the .model header and weights too
    assert np.array_equal(run_d.counts, run_f.counts) and np.array_equal(run_d.weights, run_f.weights)
    assert run_d.n_eff == run_f.n_eff and rd.effective_samples == rf.effective_samples
    assert model_head(rd.param_file) == model_head(rf.param_file)
    # the fitted couplings: both runs reach the float64 optimum
    cn_d = np.loadtxt(rd.couplings_file, usecols=5)
    cn_f = np.loadtxt(rf.couplings_file, usecols=5)
    assert np.sqrt(np.mean((run_d.x - run_f.x).astype(np.float64) ** 2)) < 1e-4
    assert np.abs(cn_d - cn_f).max() < 1e-4


def test_without_repeats_the_problem_gets_the_original_arrays(tmp_path):
    codes = synthetic.synthetic_msa_codes(200, 30, 6)
    assert len(unique_rows_model(codes)[0]) == 200
    a2m = _a2m(tmp_path, codes)
    rd, run_d = tools.run_plmc(engine=DistinctEngine(), return_run=True, **_kw(a2m, tmp_path, "d", L=30))
    rf = tools.run_plmc(engine=FullEngine(), **_kw(a2m, tmp_path, "f", L=30))
    (codes_d, w_d), (codes_f, w_f) = Recording.problems
    assert codes_d is run_d.alignment.codes
    assert np.array_equal(codes_d, codes_f) and np.array_equal(w_d, w_f) and w_d.dtype == np.float32
    assert run_d.timings["unique_rows"] == 200
    for suffix in ("_ECs.txt", ".model"):
        assert open(str(tmp_path / ("d" + suffix)), "rb").read() == open(str(tmp_path / ("f" + suffix)), "rb").read()


def test_two_gloo_ranks_shard_the_distinct_pair_tiles(tmp_path):
    from evcouplings_b200 import launcher
    codes = _repeats(N=300, seed=9)
    a2m = _a2m(tmp_path, codes)
    r1, run1 = tools.run_plmc(engine=DistinctEngine(), return_run=True, **_kw(a2m, tmp_path, "one", iterations=12))
    env_pp = os.environ.get("PYTHONPATH", "")
    os.environ["PYTHONPATH"] = os.path.join(ROOT, "tests") + os.pathsep + ROOT + os.pathsep + env_pp
    try:
        r2, run2 = launcher.run_plmc_multi_gpu(2, _kw(a2m, tmp_path, "two", iterations=12), return_run=True,
                                               backend="gloo", timeout=600,
                                               engine_factory="test_unique_rows:DistinctShardedEngine")
    finally:
        os.environ["PYTHONPATH"] = env_pp
    assert run2.timings["ranks"] == 2
    assert run2.timings["unique_rows"] == run1.timings["unique_rows"] < 300
    assert r2.effective_samples == r1.effective_samples
    f1 = np.array(r1.iteration_table["fx"].astype(float))
    f2 = np.array(r2.iteration_table["fx"].astype(float))
    assert len(f2) == 12 and np.abs(f1 - f2).max() <= 1e-9 * np.abs(f1).max()
    assert model_head(r1.param_file) == model_head(r2.param_file)
    cn1 = np.loadtxt(r1.couplings_file, usecols=5)
    cn2 = np.loadtxt(r2.couplings_file, usecols=5)
    assert np.abs(cn1 - cn2).max() < 1e-6


def test_checkpointed_fit_on_distinct_rows_resumes_bit_identically(tmp_path):
    codes = _repeats()
    a2m = _a2m(tmp_path, codes)
    ref = tools.run_plmc(engine=DistinctEngine(), **_kw(a2m, tmp_path, "ref"))
    ck = str(tmp_path / "u.ckpt")
    CkOracleProblem.stop_at = 9
    with pytest.raises(tools.FitInterrupted, match="iteration 9"):
        tools.run_plmc(engine=DistinctEngine(), checkpoint=ck, **_kw(a2m, tmp_path, "a"))
    hdr = checkpoint.CheckpointFile(ck).read_header()
    assert hdr["info"]["unique_rows"] == len(unique_rows_model(codes)[0]) and hdr["info"]["valid_rows"] == 240
    CkOracleProblem.stop_at = None
    res = tools.run_plmc(engine=DistinctEngine(), checkpoint=ck, **_kw(a2m, tmp_path, "a"))
    t_ref, t_res = ref.iteration_table, res.iteration_table
    assert t_res["iter"].tolist() == t_ref["iter"].tolist() and t_res["fx"].tolist() == t_ref["fx"].tolist()
    for suffix in ("_ECs.txt", ".model"):
        assert open(str(tmp_path / ("a" + suffix)), "rb").read() == open(str(tmp_path / ("ref" + suffix)), "rb").read()


def test_checkpoint_of_another_row_table_is_refused(tmp_path):
    codes = _repeats()
    a2m = _a2m(tmp_path, codes)
    ck = str(tmp_path / "r.ckpt")
    tools.run_plmc(engine=FullEngine(), checkpoint=ck, **_kw(a2m, tmp_path, "full", iterations=5))
    before = open(ck, "rb").read()
    n0 = CkOracleProblem.evaluations_total
    with pytest.raises(tools.InvalidParameterError, match="distinct sequences"):
        tools.run_plmc(engine=DistinctEngine(), checkpoint=ck, **_kw(a2m, tmp_path, "dist", iterations=8))
    assert CkOracleProblem.evaluations_total == n0 and open(ck, "rb").read() == before
    # a file that does not record the table stands for a fit on every valid row
    hdr = checkpoint.CheckpointFile(ck).read_header()
    assert hdr["info"]["unique_rows"] == hdr["info"]["valid_rows"] == 240
