"""
Generate the committed golden fixtures in tests/golden/.

Needs a checkout of the reference:  EVC_REFERENCE=<EVcouplings checkout> python tests/golden/make_golden.py

Sources of truth
  (1) the real plmc run shipped with the reference:
      notebooks/example/PABP_YEAST.{a2m,model_params}, PABP_YEAST_ECs.txt
      (presumed command: plmc -f PABP_YEAST -g -m 200 -t 0.2 -lh 0.01 -le 16.2)
  (2) the reference's own Python, imported unmodified via ref_harness:
      evcouplings/align/alignment.py:1192-1233 num_cluster_members,
      :1078-1153 frequencies / pair_frequencies,
      evcouplings/couplings/model.py:317-400 CouplingsModel reader (+ cn/fn scores :744-827),
      evcouplings/couplings/tools.py:20-108 parse_plmc_log.
Nothing from the reference's *source code* is copied; only its outputs on
seeded inputs are stored.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import golden_npz  # noqa: E402
import ref_harness  # noqa: E402
from oracle import plm_oracle as po  # noqa: E402

EX = os.path.join(ref_harness.REFERENCE_ROOT or "", "notebooks", "example")


def pabp():
    ids, seqs = po.read_a2m(os.path.join(EX, "PABP_YEAST.a2m"))
    prep = po.prepare_alignment(ids, seqs, focus="PABP_YEAST", alphabet=None, ignore_gaps=True)
    gm = po.read_model(os.path.join(EX, "PABP_YEAST.model_params"))
    counts_all = gm["weights"].astype(np.int32)           # golden stores integer neighbour counts
    golden_npz.save(
        "pabp_codes",
        codes=prep["codes"], valid_packed=np.packbits(prep["valid"]),
        n_total=prep["n_total"], golden_counts_all=counts_all,
        focus_cols=prep["focus_cols"], index_list=prep["index_list"],
        target_seq=np.array(prep["target_seq"]), region_start=prep["region_start"],
    )
    # EC text
    ec = np.loadtxt(os.path.join(EX, "PABP_YEAST_ECs.txt"), dtype=str)
    pairs = [(0, 1), (6, 8), (3, 60), (20, 21), (33, 70), (50, 81)]
    L = gm["L"]
    iu, ju = np.triu_indices(L, 1)
    pidx = np.array([np.nonzero((iu == i) & (ju == j))[0][0] for i, j in pairs])
    # reference reader KATs on the golden file
    ref_harness.install()
    from evcouplings.couplings.model import CouplingsModel
    cm = CouplingsModel(os.path.join(EX, "PABP_YEAST.model_params"))
    kat = dict(
        hi_127=float(cm.hi(127, cm.seq(127))),
        Jij_127_172=float(cm.Jij(127, 172, cm.seq(127), cm.seq(172))),
        ref_cn_zero_sum=cm.cn_scores[iu, ju].astype(np.float64),   # model.py:788-803 (zero-sum gauge first)
    )
    golden_npz.save(
        "pabp_golden",
        hdr_i=np.array([gm["L"], gm["q"], gm["n_valid"], gm["n_invalid"], gm["num_iter"]], dtype=np.int32),
        hdr_f=np.array([gm["theta"], gm["lambda_h"], gm["lambda_J"], gm["lambda_group"], gm["n_eff"]],
                       dtype=np.float32),
        alphabet=np.array(gm["alphabet"]), target_seq=np.array(gm["target_seq"]),
        index_list=gm["index_list"], fi=gm["fi"], h=gm["h"], J=gm["J"],
        fij_pairs=np.array(pairs, dtype=np.int32), fij_pair_index=pidx, fij_blocks=gm["fij"][pidx],
        ec_i=ec[:, 0].astype(np.int32), ec_Ai=ec[:, 1], ec_j=ec[:, 2].astype(np.int32), ec_Aj=ec[:, 3],
        ec_cn=ec[:, 5].astype(np.float64),
        kat_hi_127=kat["hi_127"], kat_Jij_127_172=kat["Jij_127_172"],
        ref_cn_zero_sum=kat["ref_cn_zero_sum"],
    )
    print("pabp fixtures written; valid=%d" % prep["n_valid"])


def in_tree_twins():
    """Reference numba kernels on the seeded config-1 alignment (N=200, L=40, q=21)."""
    ref_harness.install()
    from evcouplings.align import alignment as al
    out = {}
    for name, (N, L, seed, theta) in dict(cfg1=(200, 40, 1, 0.8), tie=(300, 50, 7, 0.8),
                                          odd=(257, 33, 11, 0.7)).items():
        codes = po.synthetic_msa_codes(N, L, seed)
        m = codes.astype(np.int64)
        counts = al.num_cluster_members(m, theta)
        w = 1.0 / counts
        fi = al.frequencies(m, w, 21)
        fij = al.pair_frequencies(m, w, 21, fi)
        iu, ju = np.triu_indices(L, 1)
        out[name + "_codes"] = codes
        out[name + "_theta"] = theta
        out[name + "_counts"] = counts.astype(np.int32)
        out[name + "_fi"] = fi
        out[name + "_fij_tri"] = fij[iu, ju]
    np.savez_compressed(os.path.join(HERE, "intree_twins.npz"), **out)
    print("in-tree twin fixtures written")


def tiny_model():
    """Tiny model written in plmc_v2 layout, read back by the reference's CouplingsModel."""
    ref_harness.install()
    from evcouplings.couplings.model import CouplingsModel
    N, L, q = 60, 12, 21
    codes = po.synthetic_msa_codes(N, L, 21)
    counts = po.hamming_counts(codes, 0.8)
    w = po.sequence_weights(counts)
    fi, fij = po.frequencies(codes, w, q)
    x, res = po.fit(codes, w, q, 0.01, 0.01 * (q - 1) * (L - 1), max_iter=400)
    h, Jt = po.unpack(x, L, q)
    alphabet = po.ALPHABET_PROTEIN
    target = "".join(alphabet[c] for c in codes[0])
    index_list = np.arange(5, 5 + L, dtype=np.int32)
    path = os.path.join(HERE, "tiny.model")
    po.write_model(path, L, q, N, 0, int(res.nit), 0.2, 0.01, 0.01 * (q - 1) * (L - 1), 0.0, w.sum(),
                   alphabet, counts.astype(np.float32), target, index_list, fi, h, fij, Jt)
    ecs_path = os.path.join(HERE, "tiny_ECs.txt")
    po.write_ecs(ecs_path, Jt.astype(np.float32), L, index_list, target)
    cm = CouplingsModel(path)
    iu, ju = np.triu_indices(L, 1)
    from evcouplings.couplings.pairs import read_raw_ec_file
    ecs = read_raw_ec_file(ecs_path, sort=False)
    np.savez_compressed(
        os.path.join(HERE, "tiny_ref_read.npz"),
        codes=codes, counts=counts, x=x.astype(np.float64),
        ref_J_tri=cm.J_ij[iu, ju], ref_h=cm.h_i, ref_fi=cm.f_i, ref_fij_tri=cm.f_ij[iu, ju],
        ref_L=cm.L, ref_q=cm.num_symbols, ref_N_eff=cm.N_eff, ref_theta=cm.theta,
        ref_lambda_J=cm.lambda_J, ref_alphabet=np.array("".join(cm.alphabet)),
        ref_target=np.array("".join(cm.target_seq)), ref_index_list=cm.index_list,
        ref_fn=cm.fn_scores[iu, ju], ref_cn_zero_sum=cm.cn_scores[iu, ju],
        ecs_i=ecs["i"].values, ecs_j=ecs["j"].values, ecs_cn=ecs["cn"].values,
        ecs_Ai=ecs["A_i"].values.astype(str), ecs_Aj=ecs["A_j"].values.astype(str),
    )
    print("tiny model fixtures written; iters=%d" % res.nit)


def model_consumers():
    """Reference CouplingsModel outputs (model.py) on the tiny model and on the golden PABP model:
    ecs table scores, hamiltonians, single-mutant matrix, delta_hamiltonian."""
    ref_harness.install()
    from evcouplings.couplings.model import CouplingsModel
    rng = np.random.default_rng(5)
    out = {}
    for name, path in (("tiny", os.path.join(HERE, "tiny.model")),
                       ("pabp", os.path.join(EX, "PABP_YEAST.model_params"))):
        cm = CouplingsModel(path)
        L, q = cm.L, cm.num_symbols
        iu, ju = np.triu_indices(L, 1)
        alphabet = "".join(cm.alphabet)
        tgt = "".join(cm.target_seq)
        seqs = [tgt] + ["".join(alphabet[k] for k in rng.integers(0, q, L)) for _ in range(40)]
        # a few sequences close to the target
        for _ in range(20):
            s = list(tgt)
            for p in rng.integers(0, L, 3):
                s[p] = alphabet[rng.integers(0, q)]
            seqs.append("".join(s))
        out[name + "_seqs"] = np.array(seqs)
        out[name + "_H"] = cm.hamiltonians(seqs)
        out[name + "_smm"] = cm.single_mut_mat_full
        out[name + "_fn"] = cm.fn_scores[iu, ju]
        out[name + "_cn"] = cm.cn_scores[iu, ju]
        if name == "tiny":
            out[name + "_mi_raw"] = cm.mi_scores_raw[iu, ju]
            out[name + "_mi_apc"] = cm.mi_scores_apc[iu, ju]
        variants = []
        for _ in range(12):
            ps = sorted(set(int(p) for p in rng.integers(0, L, 2)))
            variants.append([(int(cm.index_list[p]), tgt[p], alphabet[rng.integers(0, q)]) for p in ps])
        out[name + "_var_pos"] = np.array([[v[0][0], v[-1][0]] for v in variants])
        out[name + "_variants"] = np.array([";".join("%d,%s,%s" % s for s in v) for v in variants])
        out[name + "_dH"] = np.array([cm.delta_hamiltonian(v) for v in variants])
    np.savez_compressed(os.path.join(HERE, "model_consumers.npz"), **out)
    print("model consumer fixtures written; PABP H(target) = %.10f, smm(127,E) = %.10f" % (
        out["pabp_H"][0, 0], out["pabp_smm"][127 - 123, "ACDEFGHIKLMNPQRSTVWY".index("E"), 0]))


def _json(obj):
    def conv(v):
        if isinstance(v, (np.integer,)):
            return int(v)
        if isinstance(v, (np.floating,)):
            return float(v)
        if isinstance(v, np.ndarray):
            return v.tolist()
        if isinstance(v, (list, tuple)):
            return [conv(x) for x in v]
        if isinstance(v, dict):
            return {k: conv(x) for k, x in v.items()}
        return v
    return np.array(__import__("json").dumps(conv(obj)))


def _untmp(v, tmp):
    """paths under the scratch directory become "{tmp}/..." so that a test can substitute its own"""
    if isinstance(v, str):
        return v.replace(tmp, "{tmp}")
    if isinstance(v, (list, tuple)):
        return [_untmp(x, tmp) for x in v]
    return v


def _iter_table(df):
    return dict(columns=list(df.columns), values=df.to_numpy(dtype=np.float64))


def _protocol_kwargs(prefix, a2m, L, ignore_gaps, iterations=30, cpu=2):
    return dict(
        protocol="standard", prefix=prefix, alignment_file=a2m, focus_mode=True, focus_sequence="seq0/1-%d" % L,
        theta=0.8, alphabet=None, segments=[["A_1", "aa", "seq0", 1, L, list(range(1, L + 1))]],
        ignore_gaps=ignore_gaps, iterations=iterations, lambda_h=0.01, lambda_J=0.01, lambda_J_times_Lq=True,
        lambda_group=None, scale_clusters=None, cpu=cpu, plmc="plmc", reuse_ecs=False, min_sequence_distance=6,
        frequencies_file=None, scoring_model="skewnormal",
    )


def _standard_protocol(out, key, rng, iterations, cpu):
    """the reference's standard protocol on BASELINE configs[0] (N=200, L=40) over this project's run_plmc with the
    oracle engine, both gap modes; stored under key + "<ignore_gaps>_" """
    import tempfile
    from cpu_engine import OracleEngine
    from evcouplings_b200 import synthetic, tools
    import evcouplings.couplings.tools as ct
    import evcouplings.couplings.protocol as cpr
    import evcouplings.couplings.model as cm
    import evcouplings.couplings.pairs as cp
    for ig in (True, False):
        tmp = tempfile.mkdtemp(prefix="evc_golden_")
        N, L = 200, 40
        codes = synthetic.synthetic_msa_codes(N, L, 1)
        a2m = os.path.join(tmp, "cfg1.a2m")
        synthetic.write_a2m(a2m, codes)
        captured = {}

        def run_plmc(*args, **kwargs):
            res, run = tools.run_plmc(*args, engine=OracleEngine(), return_run=True, **kwargs)
            captured["run"], captured["kwargs"], captured["args"] = run, kwargs, args
            return res

        original = ct.run_plmc
        ct.run_plmc = run_plmc
        try:
            outcfg = cpr.run(**_protocol_kwargs(os.path.join(tmp, "out", "job"), a2m, L, ig, iterations, cpu))
        finally:
            ct.run_plmc = original
        run = captured["run"]
        model = cm.CouplingsModel(outcfg["model_file"])
        iu, ju = np.triu_indices(L, 1)
        sample = np.sort(rng.choice(iu.size, size=40, replace=False))
        ecs = cp.read_raw_ec_file(outcfg["raw_ec_file"], sort=False)
        it, fields = ct.parse_plmc_log(run.log)
        k = "%s%d_" % (key, int(ig))
        out[k + "call"] = _json(dict(args=_untmp(list(captured["args"]), tmp),
                                     kwargs={a: _untmp(v, tmp) for a, v in captured["kwargs"].items()}))
        out[k + "outcfg"] = _json({a: outcfg[a] for a in ("num_sites", "num_valid_sequences", "effective_sequences",
                                                          "region_start")})
        out[k + "model"] = _json(dict(L=model.L, num_symbols=model.num_symbols, N_valid=model.N_valid,
                                      alphabet="".join(model.alphabet), theta=model.theta, N_eff=model.N_eff,
                                      target_seq="".join(model.target_seq)))
        out[k + "h"] = np.asarray(model.h_i, dtype=np.float64)
        out[k + "pair_index"] = sample
        out[k + "J_upper"] = np.asarray(model.J_ij[iu[sample], ju[sample]], dtype=np.float64)
        out[k + "J_lower"] = np.asarray(model.J_ij[ju[sample], iu[sample]], dtype=np.float64)
        out[k + "ec_cn"] = ecs["cn"].values.astype(np.float64)
        out[k + "ec_ij"] = ecs[["i", "j"]].values.astype(np.int32)
        t = _iter_table(it)
        out[k + "iter_columns"] = _json(t["columns"])
        out[k + "iter_values"] = t["values"]
        out[k + "fields"] = _json(list(fields))


def _cli(out, key, N, L, iterations, lambda_J):
    """the reference's run_plmc (argv, subprocess, stderr parsing) over the plmc-compatible CLI (oracle engine);
    stored: the argv it built, the PlmcResult it parsed"""
    import json
    import stat
    import tempfile
    from evcouplings_b200 import synthetic
    import evcouplings.couplings.tools as ct
    tmp = tempfile.mkdtemp(prefix="evc_golden_")
    codes = synthetic.synthetic_msa_codes(N, L, 3)
    a2m = os.path.join(tmp, "in.a2m")
    synthetic.write_a2m(a2m, codes)
    argv_file = os.path.join(tmp, "argv.json")
    wrapper = os.path.join(tmp, "plmc_test_wrapper")
    with open(wrapper, "w") as f:
        f.write("#!%s\nimport sys, json\nsys.path.insert(0, %r); sys.path.insert(0, %r)\n"
                "json.dump(sys.argv[1:], open(%r, 'w'))\n"
                "from cpu_engine import OracleEngine\nfrom evcouplings_b200.plmc_cli import main\n"
                "sys.exit(main(engine=OracleEngine()))\n" % (sys.executable, ROOT, os.path.join(ROOT, "tests"), argv_file))
    os.chmod(wrapper, os.stat(wrapper).st_mode | stat.S_IEXEC)
    ecs, model = os.path.join(tmp, "o", "x_ECs.txt"), os.path.join(tmp, "o", "x.model")
    res = ct.run_plmc(a2m, ecs, model, focus_seq="seq0/1-%d" % L, alphabet=None, theta=0.8, scale=None,
                      ignore_gaps=True, iterations=iterations, lambda_h=0.01, lambda_J=lambda_J, lambda_g=None, cpu=2,
                      binary=wrapper)
    out[key + "argv"] = _json(_untmp(json.load(open(argv_file)), tmp))
    out[key + "result"] = _json({a: getattr(res, a) for a in res._fields if a not in ("iteration_table",)})
    t = _iter_table(res.iteration_table)
    out[key + "iter_columns"] = _json(t["columns"])
    out[key + "iter_values"] = t["values"]


def reference_protocol():
    """What the reference's own couplings protocol, run_plmc and readers did with this project's run_plmc
    (tests/test_reference_protocol.py, tests/test_gpu_reference_protocol.py): the arguments the protocol handed to
    run_plmc, the stage outputs it derived, the argv its run_plmc built for the plmc-compatible executable, and what
    its readers (CouplingsModel, read_raw_ec_file, parse_plmc_log) read from the files written here.  The engine is
    the test-only oracle engine, so the run is deterministic on the CPU.  Keys "std_" / "cli_": the CPU tests'
    inputs; "gpu_std_" / "gpu_cli_": the GPU tests' inputs (40 iterations, one rank; 300 x 24 CLI run)."""
    import tempfile
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from cpu_engine import OracleEngine
    from evcouplings_b200 import synthetic, tools
    ref_harness.install()
    import evcouplings.couplings.tools as ct
    import evcouplings.couplings.protocol as cpr
    import evcouplings.couplings.model as cm
    out = {}
    rng = np.random.default_rng(17)
    _standard_protocol(out, "std_", rng, iterations=30, cpu=2)

    # parse_plmc_log on a log without the mandatory lines
    try:
        ct.parse_plmc_log("nothing useful")
        out["parse_failure"] = np.array("none")
    except Exception as e:
        out["parse_failure"] = np.array(type(e).__name__)

    _cli(out, "cli_", 150, 16, iterations=12, lambda_J=2.5)

    # the complex protocol (two segments, inter-chain EC table)
    import pandas as pd
    tmp = tempfile.mkdtemp(prefix="evc_golden_")
    N, L1, L2 = 160, 12, 12
    L = L1 + L2
    codes = synthetic.synthetic_msa_codes(N, L, 8)
    a2m = os.path.join(tmp, "complex.a2m")
    synthetic.write_a2m(a2m, codes, focus_name="A_B")
    captured = {}

    def run_plmc_cx(*args, **kwargs):
        captured["args"], captured["kwargs"] = args, kwargs
        return tools.run_plmc(*args, engine=OracleEngine(), **kwargs)

    original = ct.run_plmc
    ct.run_plmc = run_plmc_cx
    try:
        kw = _protocol_kwargs(os.path.join(tmp, "cx", "job"), a2m, L, True)
        kw.update(protocol="complex", focus_sequence="A_B/1-%d" % L, use_all_ecs_for_scoring=False,
                  segments=[["A_1", "aa", "A", 1, L1, list(range(1, L1 + 1))],
                            ["B_1", "aa", "B", 1, L2, list(range(1, L2 + 1))]])
        outcfg = cpr.run(**kw)
    finally:
        ct.run_plmc = original
    inter = pd.read_csv(outcfg["inter_ec_file"])
    allecs = pd.read_csv(outcfg["ec_file"])
    model = cm.CouplingsModel(outcfg["model_file"])
    out["cx_call"] = _json(dict(args=_untmp(list(captured["args"]), tmp),
                                kwargs={a: _untmp(v, tmp) for a, v in captured["kwargs"].items()}))
    out["cx_outcfg"] = _json({a: outcfg[a] for a in ("num_sites", "num_valid_sequences")})
    out["cx_inter_segments"] = _json([sorted(set(inter["segment_i"])), sorted(set(inter["segment_j"]))])
    out["cx_inter_cn"] = inter["cn"].values.astype(np.float64)
    out["cx_ec_columns"] = _json(list(allecs.columns))
    out["cx_model"] = _json(dict(L=model.L, num_symbols=model.num_symbols))
    _standard_protocol(out, "gpu_std_", rng, iterations=40, cpu=1)
    _cli(out, "gpu_cli_", 300, 24, iterations=20, lambda_J=4.0)
    golden_npz.save("reference_protocol", **out)


def pabp_a2m_sample():
    """A fixed, seeded sample of the real PABP_YEAST.a2m shipped with the reference (the focus record, every 200th
    record after it and some invalid records), with the row numbers, for the product-ingest test."""
    import lzma
    c = golden_npz.load("pabp_codes")
    valid = np.unpackbits(c["valid_packed"])[: int(c["n_total"])].astype(bool)
    with open(os.path.join(EX, "PABP_YEAST.a2m")) as f:
        text = f.read()
    records = [">" + r for r in text.split(">")[1:]]
    assert len(records) == valid.size
    rows = set(range(0, len(records), 200)) | set(np.nonzero(~valid)[0][::20].tolist()) | {0}
    rows = np.array(sorted(rows), dtype=np.int64)
    sample = "".join(records[r] for r in rows)
    golden_npz.save("pabp_a2m_sample", rows=rows,
                    a2m_xz=np.frombuffer(lzma.compress(sample.encode()), dtype=np.uint8))


if __name__ == "__main__":
    pabp()
    in_tree_twins()
    tiny_model()
    model_consumers()
    reference_protocol()
    pabp_a2m_sample()
