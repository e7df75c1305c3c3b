"""Run every kernel of libevcplm once at small sizes (meant to be run under compute-sanitizer):
    compute-sanitizer --tool memcheck  python scripts/sanitize_all_kernels.py
    compute-sanitizer --tool racecheck python scripts/sanitize_all_kernels.py
"""
import os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from evcouplings_b200 import synthetic, msa, model_ops, lbfgs
from evcouplings_b200.engine import CudaEngine

eng = CudaEngine()
# Hamming: single-phase (short L) and two-phase (L >= 161) paths, ragged N
for N, L in ((300, 40), (333, 200)):
    codes = synthetic.synthetic_msa_codes(N, L, 1)
    c = eng.hamming_counts(codes, msa.identity_threshold_count(0.8, L))
    assert c.min() >= 1
    # distinct rows (hash, sort, group compare, numbering) and the multiplicity-weighted tile / verify kernels
    codes[::3] = codes[0]
    thr = msa.identity_threshold_count(0.8, L)
    first, inverse, mult = eng.unique_rows(codes)
    assert (eng.hamming_counts(codes[first], thr, mult=mult)[inverse] == eng.hamming_counts(codes, thr)).all()
print("hamming ok")
N, L, q = 300, 24, 21
codes = synthetic.synthetic_msa_codes(N, L, 2)
w = np.random.default_rng(0).uniform(0.1, 1, N).astype(np.float32)
x = np.random.default_rng(1).normal(0, 0.1, L * q + L * (L - 1) // 2 * q * q).astype(np.float32)
ref = None
for fwd, bwd in (("gather", "gather"), ("gather", "tc"), ("tc", "tc"), ("tcfused", "tc")):
    p = eng.plm_problem(codes, w, q, -1, 0.01, 1.0, forward=fwd, backward=bwd, m=3, data_digest=True)
    p.set_x(x)
    fx = p.evaluate(p.x)
    g = p.g.cpu().numpy()
    if ref is None:
        ref = (fx, g)
        fi, fij = p.weighted_counts()
        p.fn_scores()
        res = p.fit(np.zeros_like(x), lbfgs.default_params(max_iterations=4))
        # checksum kernel (evc_vec_checksum) on the fit's vectors, through a checkpointed fit and its resume
        import tempfile
        with tempfile.TemporaryDirectory() as td:
            ck = os.path.join(td, "s.ckpt")
            p.fit(np.zeros_like(x), lbfgs.default_params(max_iterations=2), checkpoint=ck, checkpoint_interval=0)
            p.fit(np.zeros_like(x), lbfgs.default_params(max_iterations=4), checkpoint=ck, checkpoint_interval=0)
    else:
        assert abs(fx - ref[0]) < 1e-4 * abs(ref[0]) and np.abs(g - ref[1]).max() < 1e-2
    p.close()
    print("plm", fwd, bwd, "ok", fx)
# the one-hot operand rebuilt in the other format when one handle switches forward: sparse -> fused -> sparse
# (build_xsp_kernel, build_x_kernel, tc_sparse_logits_kernel; EVC_FWD_CLUSTER=1 runs the unclustered variant)
p = eng.plm_problem(codes, w, q, -1, 0.01, 1.0, forward="tc", backward="tc", m=3)
p.set_x(x)
for mode in (2, 1):
    assert eng.lib.evc_plm_set_forward(p.handle, mode) == 0
    p.evaluate(p.x)
p.close()
print("forward switch ok")
codes_g = synthetic.to_ignore_gaps_codes(codes)
p = eng.plm_problem(codes_g, w, 20, 20, 0.01, 1.0)
p.set_x(np.zeros(p.n, dtype=np.float32)); p.evaluate(p.x); p.close()
model = dict(L=L, q=q, alphabet=synthetic.ALPHABET, target_seq="A" * L, index_list=np.arange(1, L + 1),
             fi=np.full((L, q), 1.0 / q, dtype=np.float32), h=x[:L * q].reshape(L, q),
             J=x[L * q:].reshape(-1, q, q), fij=np.full((L * (L - 1) // 2, q, q), 1.0 / (q * q), dtype=np.float32))
model_ops.ec_table(model, eng)
model_ops.hamiltonians(model, codes, eng)
print("model ops ok")
# other alphabets: the register-bounded softmax (8 / 16 / 32 states), expand with dynamic shared memory and the
# q-sized finalize tile (q > 21), plm_energy_kernel at strides 7, 13 and 33
L2 = 9
for q2, gap2 in ((6, -1), (13, 13), (31, 31), (32, -1)):
    rng = np.random.default_rng(q2)
    c2 = rng.integers(0, q2 + (1 if gap2 >= 0 else 0), size=(N, L2)).astype(np.uint8)
    x2 = rng.normal(0, 0.1, L2 * q2 + L2 * (L2 - 1) // 2 * q2 * q2).astype(np.float32)
    for chunk in (0, 768):
        nn = N if chunk == 0 else 1000
        c3 = c2 if chunk == 0 else rng.integers(0, q2, size=(nn, L2)).astype(np.uint8)
        p = eng.plm_problem(c3, np.ones(nn, dtype=np.float32), q2, gap2 if chunk == 0 else -1, 0.01, 1.0, m=3,
                            seq_chunk=chunk)
        p.set_x(x2)
        p.evaluate(p.x)
        p.weighted_counts()
        p.close()
    m2 = dict(L=L2, q=q2, alphabet=msa.ALPHABET_PROTEIN[:1] + "ACDEFGHIKLMNPQRSTVWYXBZJOU123456"[:q2 - 1],
              h=x2[:L2 * q2].reshape(L2, q2), J=x2[L2 * q2:].reshape(-1, q2, q2))
    model_ops.hamiltonians(m2, c2, eng)
    print("q", q2, "gap", gap2, "ok")
# Gibbs sampler: couplings build, uniform start, sweeps across the refresh (t = 32) in two calls, target start
for q3, n3 in ((21, 37), (2, 5)):
    m3 = synthetic.planted_potts_model(12, q3, 2, 4, alphabet=(synthetic.ALPHABET + "BJOUXZ12345")[:q3])
    with model_ops.PottsSampler(m3, n3, seed=3, engine=eng) as s3:
        s3.run(20)
        s3.run(20, beta=0.5)
        assert s3.codes().max() < q3
    with model_ops.PottsSampler(m3, n3, init="target", engine=eng) as s3:
        s3.run(1)
# 13 chains per CTA (L = 200, q = 21), the second CTA holding 5
m3 = dict(L=200, q=21, alphabet=(synthetic.ALPHABET + "BJOUXZ12345")[:21], h=np.zeros((200, 21), dtype=np.float32),
          J=np.full((200 * 199 // 2, 21, 21), 0.01, dtype=np.float32), target_seq="A" * 200)
with model_ops.PottsSampler(m3, 18, seed=3, engine=eng) as s3:
    s3.run(2)
print("sampler ok")
# conditional sampler: the fold, the U_FF build and the masked sweep across the refresh (t = 32) in two calls, with a
# partial last CTA
m3 = synthetic.planted_potts_model(12, 21, 2, 4)
with model_ops.PottsSampler(m3, 37, seed=3, init="target", free=[2, 3, 4, 10], allowed={3: "ACD"}, engine=eng) as s3:
    s3.run(20)
    s3.run(20)
    assert s3.conditional_fields().shape == (37, 4, 21)
print("conditional sampler ok")
# replica exchange: the ladder start, tempered sweeps (plain and conditional) across the refresh (t = 32) split between
# swap rounds, the swap kernel with a partial last block of ladders, the ladder state copies
with model_ops.PottsSampler(m3, 13 * 4, seed=3, engine=eng) as s3:
    s3.set_ladder(model_ops.geometric_ladder(0.5, 1.0, 4), 3)
    s3.temper(20)
    s3.temper(20)
    assert s3.rung_codes(3).shape == (13, 12) and s3.swap_statistics()["attempted"].sum() == 13 * 20
with model_ops.PottsSampler(m3, 37 * 3, seed=3, init="target", free=[2, 3, 4, 10], allowed={3: "ACD"},
                            engine=eng) as s3:
    s3.set_ladder([0.5, 1.0, 2.0], 1)
    s3.temper(35)
    s3.energies()
print("tempering ok")
# design: the record start, recording sweeps (plain, conditional, tempered) across the refresh (t = 32), the record
# copies and the descent kernel (plain and conditional) with a partial last CTA
with model_ops.PottsSampler(m3, 37, seed=3, engine=eng) as s3:
    s3.record_best()
    s3.run(20)
    s3.run(20)
    s3.descend(30)
    assert s3.best()[2].min() >= 0
with model_ops.PottsSampler(m3, 37 * 3, seed=3, init="target", free=[2, 3, 4, 10], allowed={3: "ACD"},
                            engine=eng) as s3:
    s3.set_ladder([0.5, 1.0, 2.0], 1)
    s3.record_best()
    s3.temper(35)
    s3.descend(35)
    s3.best()
print("design ok")
# annealed sweeps: across the refresh (t = 32), a schedule split over two calls, a plain run after them, log_partition
m3 = synthetic.planted_potts_model(12, 21, 2, 4)
with model_ops.PottsSampler(m3, 37, seed=3, engine=eng) as s3:
    b3 = np.arange(41, dtype=np.float32) / 40
    s3.anneal(b3[:17])
    s3.anneal(b3[16:])
    s3.run(3)
    assert np.isfinite(s3.log_weights()).all()
model_ops.log_partition(m3, 19, 8, 4, engine=eng)
print("annealing ok")
# counts at their plan edges: two site CTAs (L = 513, q = 32), one code row per stage (L = 16385, q = 2)
for L5, q5 in ((513, 32), (16385, 2)):
    c5 = torch.from_numpy(np.random.default_rng(5).integers(0, q5, (3, L5)).astype(np.uint8)).to(eng.device)
    o5 = torch.empty(L5 * q5 + L5 * (L5 - 1) // 2 * q5 * q5, dtype=torch.int32, device=eng.device)
    assert eng.lib.evc_code_counts(eng.ptr(c5), 3, L5, q5, eng.ptr(o5), eng.stream()) == 0
    torch.cuda.synchronize()
    del o5
print("count plans ok")
# Boltzmann-machine learning: counts (sites and pairs, q = 2 and 32, a row count off every tile), the fused update,
# set_model between sweeps
for q4, L4 in ((2, 40), (32, 9)):
    m4 = synthetic.planted_potts_model(L4, q4, 2, 5, alphabet=(synthetic.ALPHABET + "BJOUXZ12345")[:q4])
    m4.update(lambda_h=0.01, lambda_J=1.0, n_eff=100.0)
    with model_ops.BoltzmannLearner(m4, 77, seed=2, learning_rate=0.5, burn_in=3, engine=eng) as b4:
        b4.run(2, sweeps=3)
        b4.run(1, sweeps=33, progress=lambda k, st: None)
print("boltzmann ok")
