"""
Vector-kernel probe (one GPU, one call; a measurement, not a test): this tree against its parent commit after the
L-BFGS vector kernels of evc_plm_fit became the only ones, so that evc_vec_dot, evc_lbfgs_* and
evc_plm_add_regulariser run them too.  Parent and branch run in subprocesses.  It reports, in this order, rewriting
OUTDIR/vector_kernels_probe.json after each,

    outputs      bench.py --dump-outputs: gradient and fx[0] bit for bit, the relative difference of fx[1]
    device fit   evc_plm_fit x (SHA-256) and iteration table, parent against branch: config 2 (N = 50,000, L = 200,
                 q = 21) for 40 iterations, 3 of 6 correction pairs in host memory (N = 3001, L = 40),
                 precision="auto" to convergence (N = 3001, L = 40)
    python fit   the Python L-BFGS driver (evc_vec_*, evc_lbfgs_*, evc_plm_add_regulariser) parent against branch,
                 and how close it comes to evc_plm_fit in each tree (N = 1200, L = 30, 25 iterations)
    timing       bench.py --no-subrecords ms_per_step in fp32 and bf16 modes, parent and branch alternated over 3
                 rounds: median and range

The parent tree must be exported and built beforehand (it cross-compiles; no GPU needed):
    mkdir -p _parent && git archive HEAD~1 | tar -x -C _parent && _parent/evcouplings_b200/csrc/build.sh
The card's name and power limit are read in the same run (read-only nvidia-smi query).

    python scripts/vector_kernels_probe.py OUTDIR [PARENT_TREE]
"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROUNDS = 3

# one fit through the engine of the tree given as argv[1]: case name, output .npy path for x
_CHILD = r'''
import hashlib, json, os, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from evcouplings_b200 import lbfgs, synthetic
from evcouplings_b200.engine import CudaEngine
case, xout = sys.argv[2], sys.argv[3]
N, L, q, iters, eps, kw, drivers = {
    "config2": (50000, 200, 21, 40, 1e-9, {}, ("device",)),
    "host_pairs": (3001, 40, 21, 25, 1e-9, {}, ("device",)),
    "auto": (3001, 40, 21, 0, 1e-3, {"precision": "auto"}, ("device",)),
    "drivers": (1200, 30, 21, 25, 1e-9, {}, ("device", "python")),
}[case]
codes = synthetic.synthetic_msa_codes(N, L, 1)
w = np.random.default_rng(2).uniform(0.2, 1.0, N).astype(np.float32)
eng = CudaEngine()
out = {}
for driver in drivers:
    p = eng.plm_problem(codes, w, q, -1, 0.01, 0.01 * (q - 1) * (L - 1), **kw)
    rows = []
    res = p.fit(np.zeros(p.n, dtype=np.float32), lbfgs.default_params(max_iterations=iters, epsilon=eps),
                lambda *r: rows.append([float(v) for v in r]) and False, driver=driver)
    x = p.get_x()
    np.save(xout + "_" + driver + ".npy", x)
    out[driver] = {"status": res.status, "iterations": res.iterations, "evaluations": res.evaluations,
                   "fx": res.fx, "x_sha256": hashlib.sha256(x.tobytes()).hexdigest(), "rows": rows,
                   "host_pairs": p.host_pairs}
    p.close()
print(json.dumps(out))
'''


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip()


def run(cmd, env=None, cwd=None):
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=cwd, timeout=1800)
    if r.returncode != 0:
        raise RuntimeError("%s failed:\n%s" % (" ".join(cmd), r.stderr[-4000:]))
    return r.stdout


def bench(tree, args, dump=None):
    cmd = [sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--no-subrecords"] + args + \
        (["--dump-outputs", dump] if dump else [])
    line = [l for l in run(cmd, cwd=tree).splitlines() if l.startswith("{")][-1]
    return json.loads(line)["ms_per_step"]


def child(tree, case, xout, env=None):
    return json.loads(run([sys.executable, "-c", _CHILD, tree, case, xout], env=env).strip().splitlines()[-1])


def stats(v):
    v = np.asarray(v, dtype=np.float64)
    return {"median": float(np.median(v)), "min": float(v.min()), "max": float(v.max())}


def save(outdir, res):
    with open(os.path.join(outdir, "vector_kernels_probe.json"), "w") as f:
        json.dump(res, f, indent=1)


def bits_equal(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def main():
    if len(sys.argv) not in (2, 3):
        sys.exit("usage: python scripts/vector_kernels_probe.py OUTDIR [PARENT_TREE]")
    outdir = os.path.abspath(sys.argv[1])
    parent = os.path.abspath(sys.argv[2]) if len(sys.argv) == 3 else os.path.join(ROOT, "_parent")
    os.makedirs(outdir, exist_ok=True)
    trees = (("parent", parent), ("branch", ROOT))
    res = {"card": card(), "rounds": ROUNDS}
    print(res["card"], flush=True)

    res["outputs"] = {}
    for prec in ("fp32", "bf16"):
        d = {}
        for tag, tree in trees:
            dd = os.path.join(outdir, "dump_%s_%s" % (tag, prec))
            bench(tree, ["--precision", prec, "--steps", "20"], dd)
            d[tag] = {k: np.load(os.path.join(dd, k + ".npy")) for k in ("fx", "gradient")}
        fp, fb = d["parent"]["fx"], d["branch"]["fx"]
        res["outputs"][prec] = {
            "gradient_bit_identical": bits_equal(d["parent"]["gradient"], d["branch"]["gradient"]),
            "fx0_bit_identical": bits_equal(fp[:1], fb[:1]),
            "fx1_rel_diff": float(abs(fb[1] - fp[1]) / abs(fp[1])),
            "fx": {"parent": fp.tolist(), "branch": fb.tolist()}}
        print("outputs", prec, json.dumps(res["outputs"][prec]), flush=True)
        save(outdir, res)

    res["device_fit"] = {}
    for case, env in (("config2", None), ("host_pairs", dict(os.environ, EVC_HOST_HISTORY="3")), ("auto", None)):
        r = {tag: child(tree, case, os.path.join(outdir, "x_%s_%s" % (case, tag)), env)["device"]
             for tag, tree in trees}
        rec = {"bit_identical": r["parent"]["x_sha256"] == r["branch"]["x_sha256"] and
               r["parent"]["rows"] == r["branch"]["rows"] and
               r["parent"]["evaluations"] == r["branch"]["evaluations"],
               "host_pairs": r["branch"]["host_pairs"], "iterations": r["branch"]["iterations"],
               "evaluations": r["branch"]["evaluations"], "status": r["branch"]["status"]}
        res["device_fit"][case] = rec
        print("device_fit", case, json.dumps(rec), flush=True)
        save(outdir, res)

    r = {tag: child(tree, "drivers", os.path.join(outdir, "x_drivers_%s" % tag)) for tag, tree in trees}

    def table(t):
        return np.array(t["rows"], dtype=np.float64)     # k, fx, xnorm, gnorm, step, line-search evaluations

    def x(tag, driver):
        return np.load(os.path.join(outdir, "x_drivers_%s_%s.npy" % (tag, driver))).astype(np.float64)

    rec = {}
    pp, pb = table(r["parent"]["python"]), table(r["branch"]["python"])
    rec["python_parent_vs_branch"] = {
        "fx_max_rel_diff": float(np.abs(pb[:, 1] - pp[:, 1]).max() / np.abs(pp[:, 1]).max()),
        "x_max_abs_diff": float(np.abs(x("branch", "python") - x("parent", "python")).max()),
        "line_search_equal": bool(np.array_equal(pp[:, 5], pb[:, 5]))}
    for tag in ("parent", "branch"):
        td, tp = table(r[tag]["device"]), table(r[tag]["python"])
        rec["device_vs_python_" + tag] = {
            "fx_max_rel_diff": float(np.abs(td[:, 1] - tp[:, 1]).max() / np.abs(tp[:, 1]).max()),
            "fx_equal": bool(np.array_equal(td[:, 1], tp[:, 1])),
            "line_search_equal": bool(np.array_equal(td[:, 5], tp[:, 5])),
            "x_max_abs_diff": float(np.abs(x(tag, "device") - x(tag, "python")).max()),
            "evaluations": [r[tag]["device"]["evaluations"], r[tag]["python"]["evaluations"]]}
    res["python_driver"] = rec
    print("python_driver", json.dumps(rec), flush=True)
    save(outdir, res)

    res["ms_per_step"] = {}
    for prec in ("fp32", "bf16"):
        runs = {"parent": [], "branch": []}
        for _ in range(ROUNDS):
            for tag, tree in trees:
                runs[tag].append(bench(tree, ["--precision", prec]))
        res["ms_per_step"][prec] = {k: dict(stats(v), runs=v) for k, v in runs.items()}
        print("ms_per_step", prec, json.dumps(res["ms_per_step"][prec]), flush=True)
        save(outdir, res)


if __name__ == "__main__":
    main()
