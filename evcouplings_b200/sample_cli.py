"""
Command line of the Gibbs sampler: draw sequences from a fitted Potts model (a plmc_v2 ``.model`` file) and write
them as A2M in the model's alphabet.

    evcplm-sample MODEL -n N --sweeps S [--seed K] [--beta B] [--init random|target] [--gpus G] -o OUT.a2m

Sequence k is the state of chain k after S sweeps (model_ops.PottsSampler); the same arguments give the same file,
whatever --gpus (the chains are split over G GPUs, one process each; default 1).
"""
import argparse
import math
import sys

USAGE = __doc__


class CliError(Exception):
    pass


class _Parser(argparse.ArgumentParser):
    def error(self, message):
        raise CliError("evcplm-sample: " + message)


def parse_args(argv):
    """Returns the options as a dict: model, n, sweeps, seed, beta, init, output, and gpus if --gpus
    is given."""
    p = _Parser(prog="evcplm-sample", description=USAGE, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("model")
    p.add_argument("-n", type=int, required=True, dest="n")
    p.add_argument("--sweeps", type=int, required=True)
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--beta", type=float, default=1.0)
    p.add_argument("--init", choices=("random", "target"), default="random")
    p.add_argument("-o", "--output", required=True)
    p.add_argument("--gpus", type=int, default=argparse.SUPPRESS)
    a = p.parse_args(argv)
    if getattr(a, "gpus", 1) < 1:
        raise CliError("evcplm-sample: --gpus must be at least 1")
    if a.n < 1:
        raise CliError("evcplm-sample: -n must be at least 1")
    if a.sweeps < 0 or a.sweeps >= 1 << 31:
        raise CliError("evcplm-sample: --sweeps must be in [0, 2^31)")
    if not 0 <= a.seed < 1 << 64:
        raise CliError("evcplm-sample: --seed must be in [0, 2^64)")
    if not math.isfinite(a.beta):
        raise CliError("evcplm-sample: --beta must be finite")
    return vars(a)


def main(argv=None, engine=None, stderr=None, backend="nccl"):
    """``backend``: the torch.distributed backend of the ranks --gpus starts ("gloo" lets them share one device)."""
    from . import model_ops, synthetic
    argv = sys.argv[1:] if argv is None else argv
    stderr = stderr or sys.stderr
    try:
        opts = parse_args(argv)
        gpus = model_ops.check_num_gpus(opts.get("gpus", 1), opts["n"], backend)
    except (CliError, ValueError) as e:
        stderr.write("%s\n" % e if isinstance(e, CliError) else "evcplm-sample: --gpus: %s\n" % e)
        return 2
    try:
        model = model_ops.read_model(opts["model"])
        codes = model_ops.sample_codes(model, opts["n"], opts["sweeps"], opts["seed"], opts["beta"], opts["init"],
                                       engine=engine, num_gpus=gpus, backend=backend)
        synthetic.write_a2m(opts["output"], codes, alphabet=model["alphabet"])
    except Exception as e:
        stderr.write("evcplm-sample: %s: %s\n" % (type(e).__name__, e))
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
