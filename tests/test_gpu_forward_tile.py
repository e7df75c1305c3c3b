"""The 256-sequence tiles of the sparse forward (-m gpu): the default kernel and the 128-sequence one that
EVC_FWD_TILE=128 forces give bit-identical fx and gradients, at the alphabet, tile, cluster, chunk and K edges."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (name, N, L, q, ignored gap, sequence chunk, precisions)
CASES = [
    ("q2", 300, 40, 2, False, 0, ("fp32",)),
    ("q4", 300, 40, 4, False, 0, ("fp32",)),
    ("q21", 300, 30, 21, False, 0, ("fp32", "bf16")),
    ("q32", 300, 25, 32, False, 0, ("fp32",)),
    ("q20gap", 300, 30, 20, True, 0, ("fp32", "bf16")),
    # 128-sequence tiles 1, 2, 2, 3, 4 and 9: 256-sequence tiles 1, 1, 1, 2, 2 and 5 (odd: 1 and 5)
    ("N1", 1, 20, 21, False, 0, ("fp32",)),
    ("N129", 129, 20, 21, False, 0, ("fp32",)),
    ("N255", 255, 20, 21, False, 0, ("fp32",)),
    ("N257", 257, 20, 21, False, 0, ("fp32", "bf16")),
    ("N385", 385, 20, 21, False, 0, ("fp32",)),
    ("N1025", 1025, 20, 21, False, 0, ("fp32", "bf16")),
    # chunks of 768 sequences: n0 = 768 and 1536, the last with 264 real rows (3 tiles of 128)
    ("chunks", 1800, 13, 21, False, 768, ("fp32", "bf16")),
    # L q = 8192: 128 K blocks, one accumulation chain (256-row tiles); L q = 8211: 129 K blocks (128-row tiles)
    ("Lq8192", 300, 256, 32, False, 0, ("fp32",)),
    ("Lq8211", 300, 391, 21, False, 0, ("fp32",)),
]

_CHILD = r'''
import hashlib, json, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from evcouplings_b200.engine import CudaEngine
cases = json.loads(sys.argv[2])
eng = CudaEngine()
res = {}
for name, N, L, q, gap, chunk, precs in cases:
    rng = np.random.default_rng(N * 1000 + L * 10 + q)
    codes = rng.integers(0, q + (1 if gap else 0), size=(N, L)).astype(np.uint8)
    w = rng.uniform(0.1, 1, N).astype(np.float32)
    x = rng.normal(0, 0.1, L * q + L * (L - 1) // 2 * q * q).astype(np.float32)
    for prec in precs:
        p = eng.plm_problem(codes, w, q, q if gap else -1, 0.01, 1.0, forward="tc", backward="tc", precision=prec,
                            m=3, seq_chunk=chunk or None)
        p.set_x(x)
        fx = p.evaluate(p.x)
        g = p.g.cpu().numpy()
        res["%s/%s" % (name, prec)] = [float(fx).hex(), hashlib.sha256(g.tobytes()).hexdigest(),
                                       bool(np.isfinite(g).all())]
        p.close()
print(json.dumps(res))
'''


def _run(tile, cluster):
    env = dict(os.environ, EVC_FWD_CLUSTER=cluster)
    env.pop("EVC_FWD_TILE", None)
    if tile:
        env["EVC_FWD_TILE"] = tile
    r = subprocess.run([sys.executable, "-c", _CHILD, ROOT, json.dumps(CASES)], env=env, capture_output=True,
                       text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("cluster", ["1", "2"])
def test_256_row_tiles_are_bit_identical(cluster):
    """Per case and precision: fx and the SHA-256 of the gradient's bytes agree between the 256-row kernel (the
    default where K is one accumulation chain) and the 128-row kernel, for 1- and 2-CTA clusters."""
    new, old = _run(None, cluster), _run("128", cluster)
    assert set(new) == set(old)
    assert all(v[2] for v in new.values()), [k for k, v in new.items() if not v[2]]
    diff = [k for k in sorted(new) if new[k] != old[k]]
    assert not diff, diff
