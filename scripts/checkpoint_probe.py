"""Pause per checkpoint and state bytes of the device fit (evc_plm_fit_checkpointed through CudaPlmProblem.fit).

    python scripts/checkpoint_probe.py [--L 200] [--N 50000] [--m 6] [--host-pairs K] [--full-writes 4] [--dir DIR]

After an untimed warm-up fit (workspace allocation, pinning of host pairs, first launches), it times the same fit
of m + full_writes iterations without checkpoints, then with a checkpoint at every iteration boundary.  The history
fills during the first m iterations, so only the last full_writes states hold all m pairs: the figures below are
taken over those full-history writes only, each (2 + 2m) n 4 bytes plus the header.

    pause_s            seconds one full-history write keeps the fit waiting (the whole callback: checksums, device
                       to host copies through the pinned staging buffer, file write, fsync and rename)
    checksum_s         the evc_vec_checksum share of it
    d2h_s              the same vectors copied to host memory and discarded, no file (timed separately)
    file_GBps          bytes / pause_s
    pause_s_by_diff    cross-check: (checkpointed fit - plain fit) / number of writes, over all writes, whose mean
                       size is mean_bytes_all_writes

Prints one JSON line.  The file goes to --dir (default: a temporary directory) and is removed."""
import argparse
import ctypes
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from evcouplings_b200 import _lib, checkpoint, lbfgs, synthetic  # noqa: E402
from evcouplings_b200.engine import CudaEngine  # noqa: E402


class _Discard(object):
    def write(self, b):
        return len(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=50000)
    ap.add_argument("--L", type=int, default=200)
    ap.add_argument("--m", type=int, default=6)
    ap.add_argument("--full-writes", type=int, default=4)
    ap.add_argument("--host-pairs", type=int, default=None)
    ap.add_argument("--dir", default=None)
    a = ap.parse_args()
    if a.host_pairs is not None:
        os.environ["EVC_HOST_HISTORY"] = str(a.host_pairs)
    import torch
    eng = CudaEngine()
    codes = synthetic.synthetic_msa_codes(a.N, a.L, 1)
    w = np.ones(a.N, dtype=np.float32)
    p = eng.plm_problem(codes, w, 21, -1, 0.01, 2.0, m=a.m, data_digest=True)
    iters = a.m + a.full_writes
    params = lbfgs.default_params(max_iterations=iters, epsilon=1e-9, m=a.m)
    x0 = np.zeros(p.n, dtype=np.float32)
    p.fit(x0, params)                                   # warm-up, untimed
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res_plain = p.fit(x0, params)
    plain_s = time.perf_counter() - t0
    d = a.dir or tempfile.mkdtemp(prefix="evc_ckpt_probe_")
    path = os.path.join(d, "probe.ckpt")
    ck = checkpoint.CheckpointFile(path, 0.0)
    t0 = time.perf_counter()
    res = p.fit(x0, params, checkpoint=ck)
    ck_s = time.perf_counter() - t0
    assert res.iterations == res_plain.iterations == iters and res.fx == res_plain.fx
    full = [r for r in ck.write_log if r["hist"] == a.m]
    assert full, "no full-history write: raise --full-writes"

    # device-to-host share: the full-history vectors of the workspace through the same staging buffer, no file
    staging = checkpoint._Staging(p.n)
    first_host = a.m - p.host_pairs
    vecs = []
    for which, slot in [(_lib.FIT_VEC_X, -1), (_lib.FIT_VEC_G, -1)] + [
            (kind, j) for j in range(a.m) for kind in (_lib.FIT_VEC_S, _lib.FIT_VEC_Y)]:
        ptr = ctypes.c_void_p()
        _lib.check(p.lib.evc_plm_fit_vector(p.handle, which, max(slot, 0), ctypes.byref(ptr)), "evc_plm_fit_vector")
        vecs.append(checkpoint.DeviceVector(eng, ptr.value, p.n, host=slot >= first_host))
    for v in vecs[:1]:
        v.write(_Discard(), staging)                    # allocates the staging buffer
    t0 = time.perf_counter()
    for v in vecs:
        v.write(_Discard(), staging)
    d2h_s = time.perf_counter() - t0

    recorded = checkpoint.CheckpointFile(path).read_header()["info"]
    p.close()
    shutil.rmtree(d) if a.dir is None else os.unlink(path)
    mean = lambda key, rows: sum(r[key] for r in rows) / len(rows)        # noqa: E731
    pause = mean("seconds", full)
    out = dict(gpu=torch.cuda.get_device_name(0), N=a.N, L=a.L, q=21, n=p.n, m=a.m, host_pairs=p.host_pairs,
               iterations=iters, s_per_iteration_plain=round(plain_s / iters, 4),
               full_history_writes=len(full), full_history_bytes=int(mean("bytes", full)),
               pause_s=round(pause, 4), checksum_s=round(mean("checksum_s", full), 4), d2h_s=round(d2h_s, 4),
               file_GBps=round(mean("bytes", full) / pause / 1e9, 3),
               all_writes=len(ck.write_log), mean_bytes_all_writes=int(mean("bytes", ck.write_log)),
               pause_s_by_diff=round((ck_s - plain_s) / len(ck.write_log), 4), recorded=recorded)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
