"""
Command line of Boltzmann-machine learning: refine a fitted Potts model (a plmc_v2 ``.model``) until its Gibbs
samples reproduce the stored one- and two-site statistics, and write the refined model (and its ECs).

    evcplm-bmdca MODEL --updates T [--chains M] [--sweeps S] [--learning-rate ETA] [--burn-in B] [--seed K]
                 [--gpus G] -o OUT.model [-c OUT_ECs.txt]

One table row per update goes to stderr.  The same arguments give the same files (model_ops.BoltzmannLearner),
whatever --gpus (the chains are split over G GPUs, one process each, and their counts summed; default 1).  With
G > 1 the table is written when the ranks have finished.
"""
import argparse
import math
import sys

USAGE = __doc__


class CliError(Exception):
    pass


class _Parser(argparse.ArgumentParser):
    def error(self, message):
        raise CliError("evcplm-bmdca: " + message)


def parse_args(argv):
    """Returns the options as a dict: model, updates, chains, sweeps, learning_rate, burn_in, seed, output, ecs,
    and gpus if --gpus is given."""
    p = _Parser(prog="evcplm-bmdca", description=USAGE, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("model")
    p.add_argument("--updates", type=int, required=True)
    p.add_argument("--chains", type=int, default=10000)
    p.add_argument("--sweeps", type=int, default=10)
    p.add_argument("--learning-rate", type=float, default=0.05, dest="learning_rate")
    p.add_argument("--burn-in", type=int, default=0, dest="burn_in")
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("-o", "--output", required=True)
    p.add_argument("-c", "--ecs", default=None)
    p.add_argument("--gpus", type=int, default=argparse.SUPPRESS)
    a = p.parse_args(argv)
    if getattr(a, "gpus", 1) < 1:
        raise CliError("evcplm-bmdca: --gpus must be at least 1")
    if a.updates < 0:
        raise CliError("evcplm-bmdca: --updates must be >= 0")
    if a.chains < 1:
        raise CliError("evcplm-bmdca: --chains must be at least 1")
    for name, v in (("--sweeps", a.sweeps), ("--burn-in", a.burn_in)):
        if v < 0 or v >= 1 << 31:
            raise CliError("evcplm-bmdca: %s must be in [0, 2^31)" % name)
    if not math.isfinite(a.learning_rate) or a.learning_rate <= 0:
        raise CliError("evcplm-bmdca: --learning-rate must be finite and > 0")
    if not 0 <= a.seed < 1 << 64:
        raise CliError("evcplm-bmdca: --seed must be in [0, 2^64)")
    return vars(a)


def main(argv=None, engine=None, stderr=None, backend="nccl"):
    """``backend``: the torch.distributed backend of the ranks --gpus starts ("gloo" lets them share one device)."""
    from . import model_io, model_ops
    argv = sys.argv[1:] if argv is None else argv
    stderr = stderr or sys.stderr
    try:
        opts = parse_args(argv)
        gpus = model_ops.check_num_gpus(opts.get("gpus", 1), opts["chains"], backend)
    except (CliError, ValueError) as e:
        stderr.write("%s\n" % e if isinstance(e, CliError) else "evcplm-bmdca: --gpus: %s\n" % e)
        return 2
    try:
        model = model_ops.read_model(opts["model"])
        stderr.write("%7s %14s %14s %12s %10s\n" % ("update", "max|dfi|", "max|dfij|", "changes", "C pearson"))

        def row(k, st):
            stderr.write("%7d %14.6e %14.6e %12d %10.6f\n" % (k, st["max_field_dev"], st["max_coupling_dev"],
                                                              st["changes"], st["connected_pearson"]))
            stderr.flush()

        if gpus > 1:
            m = model_ops.boltzmann_refine(model, opts["updates"], opts["chains"], opts["sweeps"], opts["seed"],
                                           opts["learning_rate"], opts["burn_in"], progress=row,
                                           num_gpus=gpus, backend=backend)
            fn = model_ops.fn_scores(m, engine) if opts["ecs"] else None
        else:
            with model_ops.BoltzmannLearner(model, opts["chains"], seed=opts["seed"],
                                            learning_rate=opts["learning_rate"], burn_in=opts["burn_in"],
                                            engine=engine) as learner:
                learner.run(opts["updates"], opts["sweeps"], progress=row)
                m = learner.model()
                fn = learner.fn_scores() if opts["ecs"] else None
        model_io.write_model_file(opts["output"], m["L"], m["q"], m["n_valid"], m["n_invalid"], m["num_iter"],
                                  m["theta"], m["lambda_h"], m["lambda_J"], m["lambda_group"], m["n_eff"],
                                  m["alphabet"], m["weights"], m["target_seq"], m["index_list"], m["fi"], m["h"],
                                  m["fij"], m["J"])
        if opts["ecs"]:
            model_io.write_ec_file(opts["ecs"], fn, m["L"], m["index_list"], m["target_seq"])
    except Exception as e:
        stderr.write("evcplm-bmdca: %s: %s\n" % (type(e).__name__, e))
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
