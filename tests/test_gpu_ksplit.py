"""
Split-K backward (-m gpu): the tensor-core backward product cuts its K extent (the sequences) into slices that
write separate planes of Gd, summed by finalize_pairs_tc in a fixed order.  The slice count is forced through
EVC_KSPLIT (read once per process, hence one subprocess per value): the objective must be bit-identical (the
forward does not depend on it), the gradient and the weighted pair counts may differ only by the summation order.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# N = 6000 -> 94 K blocks of 64 sequences; L = 60, q = 21 -> 10 x 7 output tiles
_SCRIPT = """
import sys, numpy as np
sys.path.insert(0, %r)
from evcouplings_b200 import synthetic
from evcouplings_b200.engine import CudaEngine
N, L, q = 6000, 60, 21
codes = synthetic.synthetic_msa_codes(N, L, 31)
rng = np.random.default_rng(31)
w = rng.uniform(0.05, 1.0, N).astype(np.float32)
x = rng.normal(0, 0.1, L * q + L * (L - 1) // 2 * q * q).astype(np.float32)
out = {}
eng = CudaEngine()
for prec in ("fp32", "bf16"):
    p = eng.plm_problem(codes, w, q, -1, 0.01, 2.0, forward="tc", backward="tc", precision=prec)
    p.set_x(x)
    p.evaluate(p.x)
    out["fx_" + prec] = p.fxbuf.cpu().numpy()
    out["g_" + prec] = p.g.cpu().numpy()
    if prec == "fp32":
        out["fi"], out["fij"] = p.weighted_counts()
    p.close()
np.savez(sys.argv[1], **out)
""" % ROOT


def _run(tmp_path, ksplit):
    path = str(tmp_path / ("ks%d.npz" % ksplit))
    env = dict(os.environ, EVC_KSPLIT=str(ksplit))
    p = subprocess.run([sys.executable, "-c", _SCRIPT, path], capture_output=True, text=True, env=env, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    return np.load(path)


def test_ksplit_changes_only_the_backward_summation_order(tmp_path):
    ref = _run(tmp_path, 1)
    for ks in (2, 3, 8):
        got = _run(tmp_path, ks)
        for prec in ("fp32", "bf16"):
            assert np.array_equal(got["fx_" + prec], ref["fx_" + prec]), (ks, prec)
            g, g1 = got["g_" + prec].astype(np.float64), ref["g_" + prec].astype(np.float64)
            assert np.linalg.norm(g - g1) <= 1e-6 * np.linalg.norm(g1), (ks, prec)
        assert np.array_equal(got["fi"], ref["fi"])
        assert np.abs(got["fij"] - ref["fij"]).max() <= 1e-6 * np.abs(ref["fij"]).max(), ks
