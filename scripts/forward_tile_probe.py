"""Forward-tile probe (one GPU, one call; a measurement, not a test): the sparse forward with 256-sequence CTA tiles
(this tree) against the parent commit's 128-sequence tiles, alternating parent and branch in subprocesses, 3 rounds,
median and range of ms per evaluation and of the forward stage (evc_plm_last_stage_ms), for
    config 2 (N = 50,000, L = 200, q = 21) in fp32 and bf16 modes          (bench.py --no-subrecords)
    N = 20,000, L = 500: 129 K blocks, the 128-row kernel on both sides   (bench.py --no-subrecords)
    q = 32 at N = 50,000, L = 200; config 2 in 2 sequence chunks          (engine, CUDA events)
plus EVC_FWD_TILE=128 on this tree at config 2 (the same build with the old tile), and fx and the gradient of parent
and branch on the same seeded inputs (bench.py --dump-outputs), which must be bit-identical.

The parent tree must be exported and built beforehand (it cross-compiles; no GPU needed):
    mkdir -p _parent && git archive HEAD~1 | tar -x -C _parent && _parent/evcouplings_b200/csrc/build.sh
The card's name, power limit and SM clocks are read in the same run (read-only nvidia-smi query).

    python scripts/forward_tile_probe.py OUTDIR [PARENT_TREE] [--shapes NAME,NAME] [--no-outputs]

--shapes runs a subset (names as in the JSON), --no-outputs skips the output comparison, so that the probe can be
split over several shorter runs; each run writes forward_tile_probe_<shapes>.json.
"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROUNDS = 3

# one timed problem through the engine of the tree given as argv[1]: q, N, L, sequence chunk, precision
_CHILD = r'''
import json, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
import torch
from evcouplings_b200.engine import CudaEngine
q, N, L, chunk, prec = int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5]), sys.argv[6]
rng = np.random.default_rng(q)
centres = rng.integers(0, q, size=(1000, L))
codes = centres[rng.integers(0, 1000, size=N)]
mut = rng.random((N, L)) < rng.uniform(0.1, 0.6, size=N)[:, None]
codes = np.ascontiguousarray(np.where(mut, rng.integers(0, q, size=(N, L)), codes).astype(np.uint8))
x = rng.normal(0, 0.02, L * q + L * (L - 1) // 2 * q * q).astype(np.float32)
eng = CudaEngine()
p = eng.plm_problem(codes, np.ones(N, dtype=np.float32), q, -1, 0.01, 0.01 * (q - 1) * (L - 1), forward="tc",
                    backward="tc", precision=prec, seq_chunk=chunk or None)
p.set_x(x)
for _ in range(5):
    p.evaluate_async(p.x)
torch.cuda.synchronize()
stage = np.zeros(5, dtype=np.float32)
ok = chunk == 0
if ok:
    eng.lib.evc_plm_set_profiling(p.handle, 1)
ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
steps, ssum = 20, np.zeros(5)
ev[0].record()
for _ in range(steps):
    p.evaluate_async(p.x)
    if ok:
        import ctypes
        eng.lib.evc_plm_last_stage_ms(p.handle, stage.ctypes.data_as(ctypes.c_void_p))
        ssum += stage
ev[1].record()
ev[1].synchronize()
print(json.dumps({"ms": ev[0].elapsed_time(ev[1]) / steps, "stage_ms": (ssum / steps).tolist() if ok else None}))
'''


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip()


def run(cmd, env=None, cwd=None):
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=cwd, timeout=1800)
    if r.returncode != 0:
        raise RuntimeError("%s failed:\n%s" % (" ".join(cmd), r.stderr[-4000:]))
    return r.stdout


def bench(tree, args, env=None, dump=None):
    cmd = [sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", "50", "--warmup", "5",
           "--no-subrecords"] + args + (["--dump-outputs", dump] if dump else [])
    line = [l for l in run(cmd, env=env, cwd=tree).splitlines() if l.startswith("{")][-1]
    rec = json.loads(line)
    st = rec.get("roofline", {}).get("stage_ms", {})
    return {"ms": rec["ms_per_step"], "stage_ms": list(st.values()), "stage_names": list(st.keys())}


def child(tree, q, N, L, chunk, prec, env=None):
    return json.loads(run([sys.executable, "-c", _CHILD, tree, str(q), str(N), str(L), str(chunk), prec],
                          env=env).strip().splitlines()[-1])


def stats(v):
    v = np.asarray(v, dtype=np.float64)
    return {"median": float(np.median(v)), "min": float(v.min()), "max": float(v.max())}


def main():
    argv = sys.argv[1:]
    only = None
    if "--shapes" in argv:
        i = argv.index("--shapes")
        only = argv[i + 1].split(",")
        del argv[i:i + 2]
    outputs = "--no-outputs" not in argv
    argv = [a for a in argv if a != "--no-outputs"]
    if len(argv) not in (1, 2):
        sys.exit("usage: python scripts/forward_tile_probe.py OUTDIR [PARENT_TREE] [--shapes NAME,NAME] [--no-outputs]")
    outdir = os.path.abspath(argv[0])
    parent = os.path.abspath(argv[1]) if len(argv) == 2 else os.path.join(ROOT, "_parent")
    os.makedirs(outdir, exist_ok=True)
    res = {"card": card(), "rounds": ROUNDS, "shapes": {}}
    print(res["card"], flush=True)
    env128 = dict(os.environ, EVC_FWD_TILE="128")
    shapes = {
        "config2_fp32": lambda t, e: bench(t, ["--precision", "fp32"], e),
        "config2_bf16": lambda t, e: bench(t, ["--precision", "bf16"], e),
        "L500_N20k_fp32": lambda t, e: bench(t, ["--sites", "500", "--seqs", "20000"], e),
        "q32_fp32": lambda t, e: child(t, 32, 50000, 200, 0, "fp32", e),
        "config2_2chunks_fp32": lambda t, e: child(t, 21, 50000, 200, 25344, "fp32", e),
    }
    if only is not None:
        unknown = set(only) - set(shapes)
        if unknown:
            sys.exit("unknown shapes: %s" % ", ".join(sorted(unknown)))
        shapes = {k: v for k, v in shapes.items() if k in only}
    for name, fn in shapes.items():
        runs = {"parent": [], "branch": [], "branch_tile128": []}
        for _ in range(ROUNDS):
            runs["parent"].append(fn(parent, None))
            runs["branch"].append(fn(ROOT, None))
            if name.startswith("config2_") and "chunks" not in name:
                runs["branch_tile128"].append(fn(ROOT, env128))
        rec = {}
        for k, v in runs.items():
            if not v:
                continue
            rec[k] = {"ms_per_eval": stats([r["ms"] for r in v]), "ms_rounds": [r["ms"] for r in v]}
            if v[0]["stage_ms"]:
                rec[k]["stage_ms_median"] = np.median(np.array([r["stage_ms"] for r in v]), axis=0).tolist()
                if "stage_names" in v[0]:
                    rec[k]["stage_names"] = v[0]["stage_names"]
                rec[k]["forward_ms"] = stats([r["stage_ms"][1] for r in v])
                rec[k]["forward_rounds"] = [r["stage_ms"][1] for r in v]
        rec["speedup_ms_per_eval"] = rec["parent"]["ms_per_eval"]["median"] / rec["branch"]["ms_per_eval"]["median"]
        if "forward_ms" in rec["branch"]:
            rec["speedup_forward"] = rec["parent"]["forward_ms"]["median"] / rec["branch"]["forward_ms"]["median"]
        res["shapes"][name] = rec
        print(name, json.dumps(rec), flush=True)
    # outputs on identical seeded inputs (config 2, both precisions): bit for bit
    res["outputs"] = {}
    for prec in ("fp32", "bf16") if outputs else ():
        d = {}
        for tag, tree in (("parent", parent), ("branch", ROOT)):
            dd = os.path.join(outdir, "dump_%s_%s" % (tag, prec))
            bench(tree, ["--precision", prec], None, dd)
            d[tag] = {k: np.load(os.path.join(dd, k + ".npy")) for k in ("fx", "gradient")}
        res["outputs"][prec] = {k: bool(np.array_equal(d["branch"][k], d["parent"][k])) for k in ("fx", "gradient")}
        print("outputs bit-identical", prec, res["outputs"][prec], flush=True)
    res["card_after"] = card()
    tag = "_".join(shapes) or "outputs"
    with open(os.path.join(outdir, "forward_tile_probe_%s.json" % tag), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
