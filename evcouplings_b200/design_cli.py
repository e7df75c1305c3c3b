"""
Command line of sequence design: sequences that score high under a fitted Potts model (a plmc_v2 ``.model`` file),
written as FASTA in the model's alphabet.

    evcplm-design MODEL -n N --sweeps S [--beta B] [--anneal B0 | --tempering R --beta-min B0 | --ladder b0,...]
                  [--swap-interval K] [--descent-sweeps D] [--seed K] [--init random|target|FILE]
                  [--free 30-45] [--allow 33:AVILM ...] [--gpus G] -o OUT.fasta

Each of N chains (or ladders) samples S sweeps while keeping the best state it reaches, and a zero-temperature descent
then moves that state to a single-site optimum: no change of one site raises H (model_ops.design_codes).  The chains
sample at --beta (default 1), or anneal from --anneal B0 up to --beta along a geometric schedule, or run replica
exchange (--tempering / --beta-min / --ladder / --swap-interval as in evcplm-sample).  The descent runs at most D
sweeps (--descent-sweeps, default 256).  --init, --free and --allow are those of evcplm-sample: with --free only the
listed positions change, each restricted to its --allow letters.

Row k is the design of chain (or ladder) k, with the header ``>design_<k> H=<energy> settled=<0|1> found_at=<t>``:
H from model_ops.hamiltonians, settled = 1 when the descent's last sweep changed nothing, and found_at the sweep at
which the sampling stage recorded the state the descent started from.  The rows are L letters of the model alphabet,
so --init FILE reads them back.  The same arguments give the same file, whatever --gpus.  A summary goes to standard
error: the best H, the number of distinct designs, the number not settled, and the swap statistics of a ladder.
"""
import argparse
import math
import os
import sys

import numpy as np

from .sample_cli import CliError, format_swap_statistics, parse_allow, parse_positions, read_init_file
from . import sample_cli

USAGE = __doc__
PROG = "evcplm-design"


class _Parser(argparse.ArgumentParser):
    def error(self, message):
        raise CliError("%s: %s" % (PROG, message))


def _own(e):
    """A CliError of sample_cli's shared parsers, under this command's name."""
    return CliError(str(e).replace("evcplm-sample:", PROG + ":", 1))


def parse_args(argv):
    """Returns the options as a dict: model, n, sweeps, seed, beta, init, output, descent_sweeps, and gpus, free,
    allow, anneal (beta_start) and ladder / swap_interval if given."""
    p = _Parser(prog=PROG, description=USAGE, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("model")
    p.add_argument("-n", type=int, required=True, dest="n")
    p.add_argument("--sweeps", type=int, required=True)
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--beta", type=float, default=1.0)
    p.add_argument("--init", default="random")
    p.add_argument("-o", "--output", required=True)
    p.add_argument("--descent-sweeps", type=int, default=256, dest="descent_sweeps")
    p.add_argument("--anneal", type=float, default=argparse.SUPPRESS)
    p.add_argument("--gpus", type=int, default=argparse.SUPPRESS)
    p.add_argument("--free", default=argparse.SUPPRESS)
    p.add_argument("--allow", action="append", default=argparse.SUPPRESS)
    p.add_argument("--tempering", type=int, default=argparse.SUPPRESS)
    p.add_argument("--beta-min", type=float, default=argparse.SUPPRESS, dest="beta_min")
    p.add_argument("--ladder", default=argparse.SUPPRESS)
    p.add_argument("--swap-interval", type=int, default=argparse.SUPPRESS, dest="swap_interval")
    a = p.parse_args(argv)
    if getattr(a, "gpus", 1) < 1:
        raise CliError("%s: --gpus must be at least 1" % PROG)
    if a.n < 1:
        raise CliError("%s: -n must be at least 1" % PROG)
    if a.sweeps < 0 or a.sweeps >= 1 << 31:
        raise CliError("%s: --sweeps must be in [0, 2^31)" % PROG)
    if a.descent_sweeps < 0 or a.descent_sweeps >= 1 << 31:
        raise CliError("%s: --descent-sweeps must be in [0, 2^31)" % PROG)
    if not 0 <= a.seed < 1 << 64:
        raise CliError("%s: --seed must be in [0, 2^64)" % PROG)
    if not math.isfinite(a.beta):
        raise CliError("%s: --beta must be finite" % PROG)
    if a.init not in ("random", "target") and not os.path.isfile(a.init):
        raise CliError("%s: --init must be random, target or an existing FASTA file, not %r" % (PROG, a.init))
    if hasattr(a, "anneal") and (hasattr(a, "tempering") or hasattr(a, "ladder")):
        raise CliError("%s: give either --anneal or --tempering/--beta-min/--ladder, not both" % PROG)
    try:
        if hasattr(a, "anneal"):
            from .model_ops import anneal_schedule
            anneal_schedule(a.anneal, a.beta, 2)
        if hasattr(a, "free"):
            a.free = parse_positions(a.free)
        if hasattr(a, "allow"):
            a.allow = parse_allow(a.allow)
        sample_cli._ladder_args(a)
    except CliError as e:
        raise _own(e)
    except ValueError as e:
        raise CliError("%s: --anneal: %s" % (PROG, e))
    return vars(a)


def write_designs(path, result, alphabet):
    """FASTA, one row per design in index order, headers >design_<k> H=<%.6f> settled=<0|1> found_at=<t>."""
    lut = np.frombuffer(alphabet.encode("ascii"), dtype=np.uint8)
    chars = lut[result["codes"]]
    with open(path, "w") as f:
        for k in range(len(chars)):
            f.write(">design_%d H=%.6f settled=%d found_at=%d\n%s\n" % (
                k, result["energy"][k], int(result["settled"][k]), int(result["found_at"][k]),
                bytes(chars[k]).decode("ascii")))


def format_summary(result):
    """The lines evcplm-design prints on standard error."""
    E, codes = result["energy"], result["codes"]
    distinct = len(np.unique(codes, axis=0))
    return ("%s: %d designs, best H = %.6f, %d distinct, %d not settled\n" %
            (PROG, len(E), float(E.max()), distinct, int((~result["settled"]).sum())))


def main(argv=None, engine=None, stderr=None, backend="nccl"):
    """``backend``: the torch.distributed backend of the ranks --gpus starts ("gloo" lets them share one device)."""
    from . import model_ops
    argv = sys.argv[1:] if argv is None else argv
    stderr = stderr or sys.stderr
    try:
        opts = parse_args(argv)
        gpus = model_ops.check_num_gpus(opts.get("gpus", 1), opts["n"], backend)
    except (CliError, ValueError) as e:
        stderr.write("%s\n" % e if isinstance(e, CliError) else "%s: --gpus: %s\n" % (PROG, e))
        return 2
    try:
        model = model_ops.read_model(opts["model"])
    except Exception as e:
        stderr.write("%s: %s: %s\n" % (PROG, type(e).__name__, e))
        return 1
    init, free, allow = opts["init"], opts.get("free"), opts.get("allow")
    try:
        if init not in ("random", "target"):
            init = read_init_file(init, model, opts["n"])
        if free is not None or allow is not None:
            model_ops.conditional_sites(model, free, allow, init)
    except CliError as e:
        stderr.write("%s\n" % _own(e))
        return 2
    except ValueError as e:
        stderr.write("%s: %s\n" % (PROG, e))
        return 2
    try:
        ladder = opts.get("ladder")
        result = model_ops.design_codes(model, opts["n"], opts["sweeps"], opts["seed"], opts["beta"],
                                        beta_start=opts.get("anneal"), init=init, free=free, allowed=allow,
                                        ladder=ladder, swap_interval=opts.get("swap_interval", 1),
                                        descent_sweeps=opts["descent_sweeps"], engine=engine, num_gpus=gpus,
                                        backend=backend)
        write_designs(opts["output"], result, model["alphabet"])
        stderr.write(format_summary(result))
        if ladder is not None:
            stderr.write(format_swap_statistics(ladder, result["swap_statistics"]))
    except Exception as e:
        stderr.write("%s: %s: %s\n" % (PROG, type(e).__name__, e))
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
