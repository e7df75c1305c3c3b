"""
Command line of annealed importance sampling: the log partition function log Z of a fitted Potts model (a plmc_v2
``.model``), and optionally the log-probability of every row of an alignment under it.

    evcplm-logz MODEL [--chains M] [--temperatures K] [--burn-in B] [--seed S] [--gpus G]
                [--alignment A2M [--focus ID]] [-o OUT.csv]

log Z is estimated in both directions (model_ops.log_partition): forward from the independent-site model, and reverse
from the model after B sweeps; their gap shows how far to trust either.  With --alignment the rows are read with the
focus and validity rules of evcplm-plmc; rows with a symbol outside the model's states (a gap under a model fitted
with ignored gaps) are counted and skipped; the mean log P per scored row is printed, and -o writes id,log_p per
scored row, with log P = H(s) - log Z (forward).  The same arguments give the same output, whatever --gpus (the
chains are split over G GPUs, one process each; default 1; the alignment's rows are scored on one GPU).
"""
import argparse
import sys

USAGE = __doc__
DEFAULT_CHAINS, DEFAULT_TEMPERATURES = 8192, 1024


class CliError(Exception):
    pass


class _Parser(argparse.ArgumentParser):
    def error(self, message):
        raise CliError("evcplm-logz: " + message)


def parse_args(argv):
    """Returns the options as a dict: model, chains, temperatures, burn_in, seed, alignment, focus, output, and gpus
    if --gpus is given."""
    p = _Parser(prog="evcplm-logz", description=USAGE, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("model")
    p.add_argument("--chains", type=int, default=DEFAULT_CHAINS)
    p.add_argument("--temperatures", type=int, default=DEFAULT_TEMPERATURES)
    p.add_argument("--burn-in", type=int, default=None, dest="burn_in")
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--alignment", default=None)
    p.add_argument("--focus", default=None)
    p.add_argument("-o", "--output", default=None)
    p.add_argument("--gpus", type=int, default=argparse.SUPPRESS)
    a = p.parse_args(argv)
    if a.chains < 1:
        raise CliError("evcplm-logz: --chains must be at least 1")
    if getattr(a, "gpus", 1) < 1:
        raise CliError("evcplm-logz: --gpus must be at least 1")
    K = a.temperatures
    if K < 1 or K >= 1 << 31 or K & (K - 1):
        raise CliError("evcplm-logz: --temperatures must be a power of two below 2^31")
    if a.burn_in is None:
        a.burn_in = K
    if a.burn_in < 0 or a.burn_in >= 1 << 31:
        raise CliError("evcplm-logz: --burn-in must be in [0, 2^31)")
    if not 0 <= a.seed < 1 << 64:
        raise CliError("evcplm-logz: --seed must be in [0, 2^64)")
    if a.alignment is None and (a.focus is not None or a.output is not None):
        raise CliError("evcplm-logz: --focus and -o need --alignment")
    return vars(a)


def score_alignment(model, path, focus, log_z, engine=None):
    """(ids, log P) of the alignment's scored rows, the number of rows skipped for symbols outside the model's states
    and the number of invalid rows (characters outside the alphabet).  The rows are read as evcplm-plmc reads them; a model without the gap among its states (fitted with
    ignored gaps) reads the gap as a non-state symbol."""
    import numpy as np
    from . import model_ops, msa
    alphabet = model["alphabet"]
    gapless = "-" not in alphabet
    ids, raw = msa.read_fasta_matrix(path)
    enc = msa.encode_alignment(ids, raw, focus=focus, alphabet=("-" + alphabet) if gapless else alphabet,
                               ignore_gaps=gapless)
    if len(enc.focus_cols) != model["L"]:
        raise ValueError("the alignment has %d focus columns, the model %d sites" % (len(enc.focus_cols), model["L"]))
    row_ids = [(n.split() or [n])[0] for n, ok in zip(ids, enc.valid) if ok]
    keep = (enc.codes < model["q"]).all(axis=1)
    codes = enc.codes[keep]
    logp = model_ops.log_probabilities(model, codes, log_z, engine) if len(codes) else np.zeros(0)
    return [r for r, k in zip(row_ids, keep) if k], logp, int((~keep).sum()), enc.n_total - enc.n_valid


def main(argv=None, engine=None, stdout=None, stderr=None, backend="nccl"):
    """``backend``: the torch.distributed backend of the ranks --gpus starts ("gloo" lets them share one device)."""
    from . import model_ops
    argv = sys.argv[1:] if argv is None else argv
    stdout = stdout or sys.stdout
    stderr = stderr or sys.stderr
    try:
        opts = parse_args(argv)
        gpus = model_ops.check_num_gpus(opts.get("gpus", 1), opts["chains"], backend)
    except (CliError, ValueError) as e:
        stderr.write("%s\n" % e if isinstance(e, CliError) else "evcplm-logz: --gpus: %s\n" % e)
        return 2
    try:
        model = model_ops.read_model(opts["model"])
        r = model_ops.log_partition(model, opts["chains"], opts["temperatures"], opts["burn_in"], opts["seed"],
                                    engine=engine, num_gpus=gpus, backend=backend)
        stdout.write("chains %d, temperatures %d, burn-in %d, seed %d\n"
                     % (r["n_chains"], r["temperatures"], r["burn_in"], r["seed"]))
        stdout.write("log Z0 (independent sites) %.10g\n" % r["log_z0"])
        stdout.write("log Z forward  %.17g  ESS %.1f  stderr %.3g\n" % (r["log_z"], r["ess"], r["stderr"]))
        stdout.write("log Z reverse  %.17g  ESS %.1f  stderr %.3g\n" % (r["log_z_reverse"], r["ess_reverse"],
                                                                          r["stderr_reverse"]))
        stdout.write("gap (reverse - forward) %.3g\n" % (r["log_z_reverse"] - r["log_z"]))
        if opts["alignment"]:
            ids, logp, skipped, invalid = score_alignment(model, opts["alignment"], opts["focus"], r["log_z"], engine)
            stdout.write("rows scored %d, skipped for symbols outside the model's states %d, invalid %d\n"
                         % (len(ids), skipped, invalid))
            if len(ids):
                stdout.write("mean log P per row %.10g\n" % float(logp.mean()))
            if opts["output"]:
                with open(opts["output"], "w") as f:
                    f.write("id,log_p\n")
                    for i, v in zip(ids, logp):
                        f.write("%s,%r\n" % (i, float(v)))
    except Exception as e:
        stderr.write("evcplm-logz: %s: %s\n" % (type(e).__name__, e))
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
