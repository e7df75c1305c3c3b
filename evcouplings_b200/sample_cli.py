"""
Command line of the Gibbs sampler: draw sequences from a fitted Potts model (a plmc_v2 ``.model`` file) and write
them as A2M in the model's alphabet.

    evcplm-sample MODEL -n N --sweeps S [--seed K] [--beta B] [--init random|target|FILE] [--gpus G]
                  [--free 30-45,60] [--allow 33:AVILM ...]
                  [--tempering R --beta-min B0 | --ladder b0,b1,...] [--swap-interval K] -o OUT.a2m

Sequence k is the state of chain k after S sweeps (model_ops.PottsSampler); the same arguments give the same file,
whatever --gpus (the chains are split over G GPUs, one process each; default 1).

--init FILE starts chain k at row k of a FASTA file (rows of exactly L letters of the model alphabet, as this command
writes them; -n must equal the number of rows).  --free samples only the listed positions (index_list numbering,
ranges inclusive) given the other sites of each chain's start, which stay as they are, so it needs --init target or
FILE when it leaves sites clamped.  --allow POS:LETTERS restricts a free position to those letters; it may be
repeated.  With --allow and no --free every position is free.

--tempering R --beta-min B0 runs replica exchange (parallel tempering): -n ladders of R chains each, at the geometric
ladder from B0 up to --beta (computed in double, rounded to fp32; refused unless strictly ascending).  --ladder gives
the inverse temperatures instead, ascending; its last one is the output's.  Adjacent rungs try to swap their
temperatures after every K sweeps (--swap-interval, default 1).  Sequence k is the chain at the top rung of ladder k;
the chains of a ladder all start from row k of --init.  The acceptance of each adjacent pair and the round trips
(rung 0 to the top and back) are printed on standard error: a pair accepting few swaps splits the ladder, and no round
trips mean the chains did not cross between the hot and cold ends.
"""
import argparse
import math
import os
import sys

import numpy as np

USAGE = __doc__


class CliError(Exception):
    pass


class _Parser(argparse.ArgumentParser):
    def error(self, message):
        raise CliError("evcplm-sample: " + message)


def parse_positions(spec):
    """"30-45,60" -> [30, ..., 45, 60]: comma-separated positions and inclusive ranges lo-hi, lo <= hi."""
    out = []
    for item in spec.split(","):
        lo, sep, hi = item.strip().partition("-")
        try:
            a, b = int(lo), int(hi) if sep else int(lo)
        except ValueError:
            raise CliError("evcplm-sample: --free: malformed position or range %r in %r" % (item, spec))
        if a > b or a < 0:
            raise CliError("evcplm-sample: --free: range %r must be lo-hi with 0 <= lo <= hi" % item)
        out.extend(range(a, b + 1))
    return out


def parse_allow(specs):
    """["33:AVILM", ...] -> {33: "AVILM", ...}; each position at most once, at least one letter."""
    out = {}
    for spec in specs:
        pos, sep, letters = spec.partition(":")
        try:
            p = int(pos)
        except ValueError:
            p = None
        if not sep or p is None or not letters:
            raise CliError("evcplm-sample: --allow: malformed %r (POSITION:LETTERS, e.g. 33:AVILM)" % spec)
        if p in out:
            raise CliError("evcplm-sample: --allow: position %d given twice" % p)
        out[p] = letters
    return out


def read_init_file(path, model, n):
    """(n, L) uint8 codes from a FASTA file of exactly n rows of L letters of the model alphabet."""
    L, alphabet = int(model["L"]), model["alphabet"]
    rows, cur = [], None
    with open(path) as f:
        for line in f:
            line = line.strip()
            if line.startswith(">"):
                if cur is not None:
                    rows.append("".join(cur))
                cur = []
            elif line:
                if cur is None:
                    raise CliError("evcplm-sample: --init %s: sequence data before the first '>' header" % path)
                cur.append(line)
    if cur is not None:
        rows.append("".join(cur))
    if len(rows) != n:
        raise CliError("evcplm-sample: --init %s has %d rows but -n is %d" % (path, len(rows), n))
    for k, r in enumerate(rows):
        if len(r) != L or set(r) - set(alphabet):
            raise CliError("evcplm-sample: --init %s: row %d must be %d letters of the model alphabet %r" %
                           (path, k, L, alphabet))
    lut = {ch: a for a, ch in enumerate(alphabet)}
    return np.array([[lut[ch] for ch in r] for r in rows], dtype=np.uint8).reshape(n, L)


def parse_ladder(spec):
    """"0.5,0.8,1" -> [0.5, 0.8, 1.0]."""
    try:
        return [float(v) for v in spec.split(",")]
    except ValueError:
        raise CliError("evcplm-sample: --ladder: malformed list of inverse temperatures %r" % spec)


def parse_args(argv):
    """Returns the options as a dict: model, n, sweeps, seed, beta, init, output, and gpus, free (a list of positions),
    allow (a dict position -> letters), ladder (float32 inverse temperatures, from --tempering/--beta-min or --ladder)
    and swap_interval if given."""
    p = _Parser(prog="evcplm-sample", description=USAGE, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("model")
    p.add_argument("-n", type=int, required=True, dest="n")
    p.add_argument("--sweeps", type=int, required=True)
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--beta", type=float, default=1.0)
    p.add_argument("--init", default="random")
    p.add_argument("-o", "--output", required=True)
    p.add_argument("--gpus", type=int, default=argparse.SUPPRESS)
    p.add_argument("--free", default=argparse.SUPPRESS)
    p.add_argument("--allow", action="append", default=argparse.SUPPRESS)
    p.add_argument("--tempering", type=int, default=argparse.SUPPRESS)
    p.add_argument("--beta-min", type=float, default=argparse.SUPPRESS, dest="beta_min")
    p.add_argument("--ladder", default=argparse.SUPPRESS)
    p.add_argument("--swap-interval", type=int, default=argparse.SUPPRESS, dest="swap_interval")
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
    if a.init not in ("random", "target") and not os.path.isfile(a.init):
        raise CliError("evcplm-sample: --init must be random, target or an existing FASTA file, not %r" % a.init)
    if hasattr(a, "free"):
        a.free = parse_positions(a.free)
    if hasattr(a, "allow"):
        a.allow = parse_allow(a.allow)
    _ladder_args(a)
    return vars(a)


def _ladder_args(a):
    from .model_ops import check_ladder, geometric_ladder
    if hasattr(a, "tempering") != hasattr(a, "beta_min"):
        raise CliError("evcplm-sample: --tempering R and --beta-min B0 go together")
    if hasattr(a, "tempering") and hasattr(a, "ladder"):
        raise CliError("evcplm-sample: give either --tempering/--beta-min or --ladder, not both")
    if hasattr(a, "swap_interval") and not (hasattr(a, "tempering") or hasattr(a, "ladder")):
        raise CliError("evcplm-sample: --swap-interval needs --tempering or --ladder")
    interval = getattr(a, "swap_interval", 1)
    try:
        if hasattr(a, "tempering"):
            a.ladder = geometric_ladder(a.beta_min, a.beta, a.tempering)
            del a.tempering, a.beta_min
        elif hasattr(a, "ladder"):
            a.ladder = check_ladder(parse_ladder(a.ladder))
        if hasattr(a, "ladder"):
            check_ladder(a.ladder, interval)
    except ValueError as e:
        raise CliError("evcplm-sample: %s" % e)
    if hasattr(a, "ladder"):
        a.swap_interval = interval


def format_swap_statistics(ladder, stats):
    """The lines evcplm-sample prints on standard error after a tempered run."""
    lines = ["evcplm-sample: replica exchange over %d ladders of %d rungs" % (len(stats["round_trips"]), len(ladder))]
    for k in range(len(ladder) - 1):
        lines.append("  pair %2d  beta %.6g <-> %.6g  accepted %d of %d (%.4f)" % (
            k, ladder[k], ladder[k + 1], stats["accepted"][k], stats["attempted"][k], stats["acceptance"][k]))
    trips = stats["round_trips"]
    lines.append("  round trips: %d in all, %.4f per ladder" % (int(trips.sum()), float(trips.mean())))
    return "\n".join(lines) + "\n"


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
    except Exception as e:
        stderr.write("evcplm-sample: %s: %s\n" % (type(e).__name__, e))
        return 1
    init, free, allow = opts["init"], opts.get("free"), opts.get("allow")
    try:
        if init not in ("random", "target"):
            init = read_init_file(init, model, opts["n"])
        if free is not None or allow is not None:
            model_ops.conditional_sites(model, free, allow, init)
    except (CliError, ValueError) as e:
        stderr.write("%s\n" % e if isinstance(e, CliError) else "evcplm-sample: %s\n" % e)
        return 2
    try:
        ladder = opts.get("ladder")
        if ladder is None:
            codes = model_ops.sample_codes(model, opts["n"], opts["sweeps"], opts["seed"], opts["beta"], init,
                                           engine=engine, num_gpus=gpus, backend=backend, free=free, allowed=allow)
        else:
            codes, stats = model_ops.sample_codes(model, opts["n"], opts["sweeps"], opts["seed"], opts["beta"], init,
                                                  engine=engine, num_gpus=gpus, backend=backend, free=free,
                                                  allowed=allow, ladder=ladder,
                                                  swap_interval=opts["swap_interval"], return_statistics=True)
        synthetic.write_a2m(opts["output"], codes, alphabet=model["alphabet"])
        if ladder is not None:
            stderr.write(format_swap_statistics(ladder, stats))
    except Exception as e:
        stderr.write("evcplm-sample: %s: %s\n" % (type(e).__name__, e))
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
