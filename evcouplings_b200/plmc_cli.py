"""
plmc-compatible command line (secondary plug point, SURVEY.md 8b): accepts the argv the reference builds in
evcouplings/couplings/tools.py:202-262

    plmc -c ECS_FILE [-o MODEL_FILE] [-f FOCUS] [-g] [-m MAXITER] [-a ALPHABET] [-t THETA_PLMC]
         [-s SCALE] [-lh LAMBDA_H] [-le LAMBDA_E] [-lg LAMBDA_G] [-n NCORES] ALIGNMENT

writes the same two files and prints the plmc-style log to STDERR (the reference parses stderr,
tools.py:266-286).  Point the pipeline's ``tools: plmc:`` config key at ``bin/evcplm-plmc`` and the unmodified
reference runs on the GPU.  ``-t`` is in plmc convention (1 - identity threshold); ``-n`` is accepted and ignored.
``--checkpoint FILE [--checkpoint-interval SECONDS]`` saves the fit's state to FILE and continues from it on a re-run
(tools.run_plmc ``checkpoint``).
"""
import sys


USAGE = __doc__


class CliError(Exception):
    pass


def parse_args(argv):
    """Returns the keyword arguments for evcouplings_b200.tools.run_plmc."""
    opts = dict(couplings_file=None, param_file=None, focus_seq=None, ignore_gaps=False, iterations=None,
                alphabet=None, theta=None, scale=None, lambda_h=None, lambda_J=None, lambda_g=None, cpu=None)
    checkpoint = {}
    alignment = None
    takes_value = {"-c": "couplings_file", "-o": "param_file", "-f": "focus_seq", "-m": "iterations",
                   "-a": "alphabet", "-t": "theta", "-s": "scale", "-lh": "lambda_h", "-le": "lambda_J",
                   "-lg": "lambda_g", "-n": "cpu",
                   "--couplings": "couplings_file", "--output": "param_file", "--focus": "focus_seq",
                   "--maxiter": "iterations", "--alphabet": "alphabet", "--theta": "theta", "--scale": "scale",
                   "--lambdah": "lambda_h", "--lambdae": "lambda_J", "--lambdag": "lambda_g", "--ncores": "cpu"}
    k = 0
    while k < len(argv):
        a = argv[k]
        if a in ("-g", "--gapignore"):
            opts["ignore_gaps"] = True
        elif a in ("-h", "--help"):
            raise CliError(USAGE)
        elif a in ("--checkpoint", "--checkpoint-interval"):
            if k + 1 >= len(argv):
                raise CliError("option %s needs a value" % a)
            checkpoint[a] = argv[k + 1]
            k += 1
        elif a in takes_value:
            if k + 1 >= len(argv):
                raise CliError("option %s needs a value" % a)
            opts[takes_value[a]] = argv[k + 1]
            k += 1
        elif a.startswith("-") and len(a) > 1 and not a[1:].replace(".", "").isdigit():
            raise CliError("unknown option %s" % a)
        else:
            if alignment is not None:
                raise CliError("more than one alignment file given (%s, %s)" % (alignment, a))
            alignment = a
        k += 1
    if alignment is None:
        raise CliError("no alignment file given")
    if opts["couplings_file"] is None:
        raise CliError("-c COUPLINGS_FILE is required")
    for key in ("scale", "lambda_h", "lambda_J", "lambda_g"):
        if opts[key] is not None:
            opts[key] = float(opts[key])
    if opts["theta"] is not None:
        opts["theta"] = 1.0 - float(opts["theta"])        # plmc convention -> identity threshold (tools.py:236-239)
    if opts["iterations"] is not None and opts["iterations"] != "max":
        opts["iterations"] = int(opts["iterations"])
    if "--checkpoint" in checkpoint:
        opts["checkpoint"] = checkpoint["--checkpoint"]
    if "--checkpoint-interval" in checkpoint:
        if "--checkpoint" not in checkpoint:
            raise CliError("--checkpoint-interval needs --checkpoint FILE")
        try:
            opts["checkpoint_interval"] = float(checkpoint["--checkpoint-interval"])
        except ValueError:
            raise CliError("--checkpoint-interval: not a number of seconds: %s" % checkpoint["--checkpoint-interval"])
    if opts["alphabet"] is not None:
        from .msa import alphabet_states
        try:
            alphabet_states(opts["alphabet"], opts["ignore_gaps"])
        except ValueError as e:
            raise CliError("-a: %s" % e)
    return alignment, opts


def main(argv=None, engine=None, stderr=None):
    from . import tools
    argv = sys.argv[1:] if argv is None else argv
    stderr = stderr or sys.stderr
    try:
        alignment, opts = parse_args(argv)
    except CliError as e:
        stderr.write(str(e) + "\n")
        return 2
    try:
        result, run = tools.run_plmc(alignment, engine=engine, return_run=True, **opts)
    except Exception as e:      # plmc reports failures on stderr with a non-zero exit code
        stderr.write("evcplm-plmc: %s: %s\n" % (type(e).__name__, e))
        return 1
    stderr.write(run.log)
    return 0


if __name__ == "__main__":
    sys.exit(main())
