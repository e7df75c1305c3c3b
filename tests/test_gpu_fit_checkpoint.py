"""
Checkpoint / resume of the device L-BFGS fit (evc_plm_fit_checkpointed) on the H100: a fit cancelled through its
progress callback and resumed from the file gives the bits of the fit that never stopped -- with host-resident
correction pairs on either side, in sequence chunks, across the bf16 -> hi+lo switch and at the alphabet edges --
and evc_vec_checksum equals its numpy model.
"""
import os

import numpy as np
import pytest

from evcouplings_b200 import checkpoint, lbfgs, synthetic, tools

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from evcouplings_b200.engine import CudaEngine
    return CudaEngine()


def _data(N=3001, L=40, q=21, seed=1):
    if q == 21:
        codes = synthetic.synthetic_msa_codes(N, L, seed)
    else:
        codes = np.random.default_rng(seed).integers(0, q, size=(N, L)).astype(np.uint8)
    w = np.random.default_rng(seed + 1).uniform(0.2, 1.0, N).astype(np.float32)
    return codes, w, q


def _fit(eng, data, iters, ck=None, stop_at=None, epsilon=1e-9, **kw):
    codes, w, q = data
    p = eng.plm_problem(codes, w, q, -1, 0.01, 2.0, data_digest=True, **kw)
    rows = []

    def progress(k, fx, xnorm, gnorm, step, n_ls):
        rows.append((k, fx))
        return stop_at is not None and k >= stop_at
    try:
        res = p.fit(np.zeros(p.n, dtype=np.float32), lbfgs.default_params(max_iterations=iters, epsilon=epsilon),
                    progress, checkpoint=ck, checkpoint_interval=-1)
        return res, p.get_x(), rows, getattr(p, "switched_at", -1), _ec_scores(p.fn_scores(), data[0].shape[1])
    finally:
        p.close()


def _ec_scores(fn, L):
    """The APC-corrected EC scores of the _ECs.txt file (model_io.apc_cn_scores) from the raw Frobenius norms."""
    from evcouplings_b200 import model_io
    return np.asarray(model_io.apc_cn_scores(np.asarray(fn, dtype=np.float64), L))


def _resume_matches(eng, tmp_path, data, stop_at=9, iters=25, save_env=None, load_env=None, monkeypatch=None,
                    **kw):
    ref = _fit(eng, data, iters, **kw)
    ck = str(tmp_path / ("fit_%d.ckpt" % stop_at))
    assert not os.path.exists(ck)
    for k, v in (save_env or {}).items():
        monkeypatch.setenv(k, v)
    a = _fit(eng, data, iters, ck=ck, stop_at=stop_at, **kw)
    assert a[0].status == lbfgs.LBFGSERR_CANCELED and a[0].iterations == stop_at
    for k, v in (load_env or {}).items():
        monkeypatch.setenv(k, v)
    b = _fit(eng, data, iters, ck=ck, **kw)
    assert tuple(b[0]) == tuple(ref[0]), (b[0], ref[0])
    assert np.array_equal(b[1], ref[1])
    assert a[2] + b[2] == ref[2]
    assert b[3] == ref[3]
    return ref, b


def test_device_driver_cancel_and_resume_is_bit_identical(eng, tmp_path):
    _resume_matches(eng, tmp_path, _data())


@pytest.mark.parametrize("save,load", [("3", "0"), ("0", "3")])
def test_host_resident_pairs_do_not_change_the_bits(eng, tmp_path, monkeypatch, save, load):
    _resume_matches(eng, tmp_path, _data(), save_env={"EVC_HOST_HISTORY": save},
                    load_env={"EVC_HOST_HISTORY": load}, monkeypatch=monkeypatch)


def test_sequence_chunks(eng, tmp_path, monkeypatch):
    monkeypatch.setenv("EVC_SEQ_CHUNK", "768")
    ref, _ = _resume_matches(eng, tmp_path, _data())
    ck = str(tmp_path / "chunk.ckpt")
    _fit(eng, _data(), 25, ck=ck, stop_at=9)
    monkeypatch.setenv("EVC_SEQ_CHUNK", "0")           # resumed unchunked: same objective, other summation order
    c = _fit(eng, _data(), 25, ck=ck)
    assert c[0].iterations == 25
    assert abs(c[0].fx - ref[0].fx) <= 1e-6 * abs(ref[0].fx)
    assert np.sqrt(np.mean((c[4] - ref[4]) ** 2)) <= 1e-4           # EC rms (APC-corrected scores)


def test_precision_schedule_before_and_after_the_switch(eng, tmp_path):
    data = _data()
    ref = _fit(eng, data, 0, epsilon=1e-3, precision="auto")
    s, K = ref[3], ref[0].iterations
    assert s >= 2 and K > s + 1, (s, K)
    for stop in (s - 1, s, s + 1):
        _resume_matches(eng, tmp_path, data, stop_at=stop, iters=0, epsilon=1e-3, precision="auto")


@pytest.mark.parametrize("q", [2, 32])
def test_alphabet_edges(eng, tmp_path, q):
    _resume_matches(eng, tmp_path, _data(N=1000, L=12, q=q))


def test_checksum_kernel_matches_numpy_model(eng):
    import torch
    from evcouplings_b200 import _lib
    out = torch.zeros(1, dtype=torch.int64, device=eng.device)
    rng = np.random.default_rng(5)
    for n in (1, 255, 257, 1000003):
        v = rng.normal(size=n).astype(np.float32)
        want = checkpoint.checksum_words(v.view(np.uint32))
        for t in (torch.from_numpy(v).to(eng.device), torch.from_numpy(v).pin_memory()):
            _lib.check(eng.lib.evc_vec_checksum(eng.ptr(t), n, eng.ptr(out), eng.stream()), "evc_vec_checksum")
            assert int(out.item()) & ((1 << 64) - 1) == want, (n, t.device)


def test_run_plmc_cap_continued_equals_uninterrupted(eng, tmp_path):
    codes = synthetic.synthetic_msa_codes(3001, 40, 2)
    a2m = str(tmp_path / "in.a2m")
    synthetic.write_a2m(a2m, codes)

    def kw(tag, iters, **extra):
        return dict(alignment=a2m, couplings_file=str(tmp_path / (tag + "_ECs.txt")),
                    param_file=str(tmp_path / (tag + ".model")), focus_seq="seq0/1-40", theta=0.8, iterations=iters,
                    lambda_h=0.01, lambda_J=2.0, num_gpus=1, **extra)
    ref = tools.run_plmc(**kw("ref", 25))
    ck = str(tmp_path / "run.ckpt")
    r10 = tools.run_plmc(**kw("a", 10, checkpoint=ck))
    assert len(r10.iteration_table) == 10 and os.path.exists(ck)
    r25, run = tools.run_plmc(return_run=True, **kw("a", 25, checkpoint=ck))
    assert run.timings["checkpoint_resumes"] == 1
    for ext in (".model", "_ECs.txt"):
        assert open(str(tmp_path / ("a" + ext)), "rb").read() == open(str(tmp_path / ("ref" + ext)), "rb").read()
    assert r25.iteration_table["fx"].tolist() == ref.iteration_table["fx"].tolist()
    assert r25.iteration_table["cond"].tolist() == ref.iteration_table["cond"].tolist()


def check_two_ranks_save_and_resume(tmp_path, run2):
    """``run2(**kwargs)``: a run_plmc call on two ranks.  A run capped at 10 iterations with a checkpoint and continued
    to 25 on two ranks writes the files of the uninterrupted two-rank run; the 10-iteration file continued on one rank
    agrees within the summation order."""
    import shutil
    codes = synthetic.synthetic_msa_codes(3001, 40, 3)
    a2m = str(tmp_path / "in.a2m")
    synthetic.write_a2m(a2m, codes)

    def kw(tag, iters, ck):
        return dict(alignment=a2m, couplings_file=str(tmp_path / (tag + "_ECs.txt")),
                    param_file=str(tmp_path / (tag + ".model")), focus_seq="seq0/1-40", theta=0.8, iterations=iters,
                    lambda_h=0.01, lambda_J=2.0, checkpoint=ck)
    ref = run2(**kw("ref", 25, None))
    ck = str(tmp_path / "m.ckpt")
    run2(**kw("a", 10, ck))
    shutil.copy(ck, str(tmp_path / "one.ckpt"))
    run2(**kw("a", 25, ck))
    for ext in ("_ECs.txt", ".model"):
        assert open(str(tmp_path / ("a" + ext)), "rb").read() == open(str(tmp_path / ("ref" + ext)), "rb").read()
    assert len(ref.iteration_table) == 25
    tools.run_plmc(num_gpus=1, **kw("b", 25, str(tmp_path / "one.ckpt")))
    cn_ref = np.loadtxt(str(tmp_path / "ref_ECs.txt"), usecols=5)
    cn_one = np.loadtxt(str(tmp_path / "b_ECs.txt"), usecols=5)
    assert np.sqrt(np.mean((cn_one - cn_ref) ** 2)) <= 1e-3


def test_two_ranks_save_and_resume(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    check_two_ranks_save_and_resume(tmp_path, lambda **kw: tools.run_plmc(num_gpus=2, **kw))
