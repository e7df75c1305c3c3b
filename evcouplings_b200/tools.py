"""
Drop-in replacement for ``evcouplings.couplings.tools`` (the reference's plmc
wrapper, evcouplings/couplings/tools.py:20-307): same ``run_plmc`` signature,
same ``PlmcResult`` fields, same output files -- but the inference runs on the
GPU through libevcplm instead of fork/exec of the plmc binary.

Plug-in point (evcouplings/couplings/protocol.py:14,203 calls ``ct.run_plmc``):

    import evcouplings.couplings.tools as ct
    import evcouplings_b200.tools as b200
    ct.run_plmc = b200.run_plmc

The function also produces a plmc-style stderr log (``PlmcRun.log``) whose lines
satisfy the regular expressions of the reference's ``parse_plmc_log``
(tools.py:50-61), so either parser can be used on it.
"""
import os
import re
import time
from collections import namedtuple

import numpy as np

from . import lbfgs as _lbfgs
from . import model_io, msa

try:  # raise the pipeline's own exception types when the reference package is importable
    from evcouplings.utils.system import ResourceError, ExternalToolError   # noqa: F401
    from evcouplings.utils.config import InvalidParameterError               # noqa: F401
except Exception:  # pragma: no cover - reference not installed
    class ResourceError(Exception):
        pass

    class ExternalToolError(Exception):
        pass

    class InvalidParameterError(Exception):
        pass


class FitInterrupted(ExternalToolError):
    """A checkpointed fit was asked to stop (SIGTERM / SIGUSR1 in a worker, checkpoint.request_stop); its state is
    in the checkpoint file and the same call continues from it."""

# same field names / order as evcouplings/couplings/tools.py:113-123
PlmcResult = namedtuple(
    "PlmcResult",
    [
        "couplings_file", "param_file",
        "iteration_table", "focus_seq_index",
        "num_valid_seqs", "num_total_seqs",
        "num_valid_sites", "num_total_sites",
        "region_start", "effective_samples",
        "optimization_status"
    ]
)

# plmc defaults when the pipeline passes None (recalled from plmc's usage text, not pinned)
DEFAULT_THETA = 0.8          # plmc -t 0.2
DEFAULT_SCALE = 1.0
DEFAULT_LAMBDA_H = 0.01
DEFAULT_LAMBDA_J = 100.0
DEFAULT_EPSILON = 1e-3
DEFAULT_HISTORY = 6

ITER_FIELDS = ["iter", "time", "cond", "fx", "-loglk", "||h||", "||e||"]


def parse_plmc_log(log):
    """Same contract as evcouplings/couplings/tools.py:20-108 (own implementation):
    returns (iteration DataFrame of strings, (focus_index, valid_seqs, total_seqs, valid_sites,
    total_sites, region_start, eff_samples, opt_status)).  KeyError if a mandatory line is missing."""
    import pandas as pd
    pats = {
        "focus": re.compile(r"Found focus (.+) as sequence (\d+)"),
        "seqs": re.compile(r"(\d+) valid sequences out of (\d+)"),
        "sites": re.compile(r"(\d+) sites out of (\d+)"),
        "region": re.compile(r"Region starts at (\d+)"),
        "samples": re.compile(r"Effective number of samples: (\d+\.\d+)"),
        "optimization": re.compile(r"Gradient optimization: (.+)"),
    }
    row = re.compile(r"(\d+)" + r"\s+(\d+\.\d+)" * 6)
    found, fields, rows = {}, None, []
    for line in log.split("\n"):
        for name, pat in pats.items():
            m = pat.search(line)
            if m:
                found[name] = m.groups()
        if line.startswith("iter"):
            fields = line.split()
        m = row.search(line)
        if m:
            rows.append(m.groups())
    iter_df = pd.DataFrame(rows, columns=fields) if fields is not None else None
    focus_index, valid_sites, total_sites, region_start = None, None, None, 1
    if "focus" in found and "sites" in found and "region" in found:
        focus_index = int(found["focus"][1])
        valid_sites, total_sites = int(found["sites"][0]), int(found["sites"][1])
        region_start = int(found["region"][0])
    valid_seqs, total_seqs = int(found["seqs"][0]), int(found["seqs"][1])
    eff = float(found["samples"][0])
    status = found["optimization"][0]
    return iter_df, (focus_index, valid_seqs, total_seqs, valid_sites, total_sites, region_start, eff, status)


def _require_file(msg, path):
    if path is None or not os.path.isfile(path) or os.path.getsize(path) == 0:
        raise ResourceError("{}: {}".format(msg, path))


def _make_dirs(path):
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)


def initial_point(fi, n_eff, L, q):
    """Independent-site start: h = log of pseudo-counted frequencies, centred per site; J = 0.
    (plmc's start as recalled; it only affects the path, the objective is strictly convex.)"""
    h = np.log((np.asarray(fi, dtype=np.float64) * n_eff + 1.0) / (n_eff + q))
    h -= h.mean(axis=1, keepdims=True)
    x0 = np.zeros(L * q + L * (L - 1) // 2 * q * q, dtype=np.float32)
    x0[:L * q] = h.ravel()
    return x0


class PlmcRun(object):
    """Everything run_plmc computed, for callers that want more than PlmcResult."""
    def __init__(self):
        self.log = ""
        self.result = None
        self.x = None
        self.weights = None
        self.counts = None
        self.n_eff = None
        self.alignment = None
        self.lbfgs = None
        self.cn = None
        self.timings = {}


def _trace(msg):
    """Wall-clock trace of the stages of run_plmc on stderr (EVC_TRACE=1; used to time rank start-up under the launcher)."""
    if os.environ.get("EVC_TRACE"):
        import sys
        sys.stderr.write("[evc-trace %.3f pid %d] %s\n" % (time.time(), os.getpid(), msg))
        sys.stderr.flush()


def distinct_rows(engine, codes):
    """(first, inverse, mult) of ``codes`` from engine.unique_rows when some rows repeat, None when every row is
    distinct (the full arrays then take the path they always took).  An engine without unique_rows, such as a
    test double of the host logic, works on the full rows."""
    unique = getattr(engine, "unique_rows", None)
    if unique is None:
        return None
    first, inverse, mult = unique(codes)
    return None if len(first) == len(codes) else (first, inverse, mult)


def _default_engine():
    from .engine import CudaEngine     # raises EngineUnavailableError without library / GPU
    return CudaEngine()


# single-GPU throughput used to decide whether spawning one rank per GPU pays (start-up of the ranks: ~15 s)
_CELLS_PER_SECOND_1GPU = 8.0e12
_MULTI_GPU_MIN_SECONDS = 20.0


def _resolve_num_gpus(num_gpus, cpu, n_valid, L, q, max_iter):
    """How many GPUs a single-process call should use.  The reference forwards ``cpu`` to plmc as ``-n``
    (evcouplings/couplings/tools.py:257-259, utils/pipeline.py:92,187); here it caps the number of GPUs.
    Explicit ``num_gpus`` / EVC_NUM_GPUS win; otherwise all visible GPUs are used when the estimated
    single-GPU time of the fit exceeds the cost of starting the ranks."""
    try:
        import torch
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            return 1                    # this process already IS one rank of a multi-GPU job
        visible = torch.cuda.device_count()
    except Exception:
        return 1
    if visible <= 1:
        return 1
    env = os.environ.get("EVC_NUM_GPUS")
    if num_gpus is None and env:
        num_gpus = int(env)
    if num_gpus is not None:
        return max(1, min(int(num_gpus), visible))
    cap = visible if cpu is None else max(1, min(int(cpu), visible))
    iters = max_iter if max_iter else 200
    est = float(n_valid) * L * L * q * iters / _CELLS_PER_SECOND_1GPU
    return cap if est >= _MULTI_GPU_MIN_SECONDS else 1


def run_plmc(alignment, couplings_file, param_file=None,
             focus_seq=None, alphabet=None, theta=None,
             scale=None, ignore_gaps=False, iterations=None,
             lambda_h=None, lambda_J=None, lambda_g=None,
             cpu=None, binary="plmc", engine=None, return_run=False,
             epsilon=DEFAULT_EPSILON, history=DEFAULT_HISTORY, store_inverse_weights=False,
             precision=None, num_gpus=None, checkpoint=None, checkpoint_interval=900.0):
    """
    Same parameters and return value as the reference's run_plmc
    (evcouplings/couplings/tools.py:126-194).  ``theta`` is the EVcouplings identity threshold
    (sequences with identity >= theta are clustered); ``lambda_J`` arrives already scaled by the
    protocol (protocol.py:179); ``binary`` is accepted and ignored.  ``cpu`` (plmc ``-n``, tools.py:257-259)
    caps the number of GPUs: a plain single-process call on a multi-GPU box starts one rank per GPU itself
    (evcouplings_b200.launcher) when the fit is long enough to pay for it; inside an initialised
    torch.distributed group (torchrun) the call is one rank of that group.

    Extra keyword arguments (not in the reference): ``engine`` (a CudaEngine; default: create one,
    which fails loudly without libevcplm.so + a CUDA device), ``return_run`` (also return the
    PlmcRun record), ``epsilon`` / ``history`` (L-BFGS stop criterion and memory), ``precision``
    ("fp32" default | "bf16" | "auto", see engine.PRECISIONS), ``num_gpus`` (explicit GPU count),
    ``checkpoint`` (a path, or True for ``<param_file or couplings_file>.ckpt``; EVC_CHECKPOINT=1 means True) and
    ``checkpoint_interval`` (seconds between saves).  With a checkpoint the fit's state is saved every interval, when
    the fit is stopped (FitInterrupted; a re-run continues from the file) and when it ends unconverged (an
    iteration cap: a re-run with a higher cap continues).  A file of another problem, or one already past the cap,
    raises InvalidParameterError before the fit; the file is deleted once the fit converges.  The iteration table
    holds every row 1..K across resumes.

    Trajectory note: plmc's L-BFGS start point, epsilon and history are recalled, not pinned (no plmc
    source); with an iteration cap the written parameters depend on the optimiser path, so agreement with
    a plmc run at the same cap is statistical (INTEGRATION.md), exact only at convergence.
    """
    run = PlmcRun()
    t_start = time.time()
    _trace("run_plmc start")
    _make_dirs(couplings_file)
    _require_file("Alignment file does not exist", alignment)
    if param_file is not None:
        _make_dirs(param_file)
    if lambda_g is not None and float(lambda_g) != 0.0:
        raise InvalidParameterError("lambda_group (group-L1 regularisation, plmc -lg) is not supported "
                                    "by the H100 engine; set it to null/0")
    if alphabet is not None:            # before ingest, reweighting or any device work
        try:
            msa.alphabet_states(alphabet, ignore_gaps)
        except ValueError as e:
            raise InvalidParameterError(str(e))
    theta =DEFAULT_THETA if theta is None else float(theta)
    scale = DEFAULT_SCALE if scale is None else float(scale)
    lambda_h = DEFAULT_LAMBDA_H if lambda_h is None else float(lambda_h)
    lambda_J = DEFAULT_LAMBDA_J if lambda_J is None else float(lambda_J)
    if iterations is None or str(iterations) == "max":
        max_iter = 0
    else:
        max_iter = int(iterations)
    if focus_seq is not None:
        focus_seq = focus_seq.split("/")[0]          # tools.py:219
    if checkpoint is None and os.environ.get("EVC_CHECKPOINT", "") not in ("", "0"):
        checkpoint = True
    if checkpoint is True:
        checkpoint = (param_file if param_file is not None else couplings_file) + ".ckpt"
    checkpoint_interval = float(checkpoint_interval)

    log = []
    try:
        ali = msa.load_alignment(alignment, focus=focus_seq, alphabet=alphabet, ignore_gaps=ignore_gaps)
    except msa.AlignmentError as e:
        raise ExternalToolError("Could not read alignment {}: {}".format(alignment, e))
    run.alignment = ali
    run.timings["ingest_s"] = time.time() - t_start
    _trace("ingest done")
    if ali.n_valid < 1:
        raise ExternalToolError("no valid sequences in alignment {}".format(alignment))
    L, q = ali.codes.shape[1], ali.q
    if focus_seq is not None:
        log.append("Found focus %s as sequence %d" % (focus_seq, ali.focus_index + 1))
    log.append("%d valid sequences out of %d " % (ali.n_valid, ali.n_total))
    if focus_seq is not None:
        log.append("%d sites out of %d" % (L, ali.num_total_sites))
        log.append("Region starts at %d" % ali.region_start)

    t0 = time.time()
    if engine is None:
        ndev = _resolve_num_gpus(num_gpus, cpu, ali.n_valid, L, q, max_iter)
        if ndev > 1:
            from . import launcher
            return launcher.run_plmc_multi_gpu(
                ndev, return_run=return_run,
                kwargs=dict(alignment=alignment, couplings_file=couplings_file, param_file=param_file,
                            focus_seq=focus_seq, alphabet=alphabet, theta=theta, scale=scale,
                            ignore_gaps=ignore_gaps, iterations=iterations, lambda_h=lambda_h, lambda_J=lambda_J,
                            lambda_g=lambda_g, epsilon=epsilon, history=history,
                            store_inverse_weights=store_inverse_weights, precision=precision,
                            checkpoint=checkpoint or None, checkpoint_interval=checkpoint_interval))
        engine = _default_engine()
    rank = getattr(engine, "rank", 0)
    run.timings["engine_init_s"] = time.time() - t0
    _trace("engine ready")

    # distinct rows: the reweighting, the pair counts and the fit run once per distinct row with its multiplicity
    t0 = time.time()
    table = distinct_rows(engine, ali.codes)
    run.timings["unique_rows"] = ali.n_valid if table is None else len(table[0])
    run.timings["unique_s"] = time.time() - t0

    # (b) sequence reweighting
    t0 = time.time()
    thr = msa.identity_threshold_count(theta, L)
    if table is None:
        counts = np.asarray(engine.hamming_counts(ali.codes, thr), dtype=np.int64)
    else:
        first, inverse, mult = table
        codes_u = ali.codes[first]
        counts_u = np.asarray(engine.hamming_counts(codes_u, thr, mult=mult), dtype=np.int64)
        counts = counts_u[inverse]
    if counts.min() < 1:
        raise ExternalToolError("sequence reweighting returned a zero neighbour count")
    weights = scale / counts.astype(np.float64)
    n_eff = float(weights.sum())
    if table is None:
        fit_codes, fit_weights = ali.codes, weights.astype(np.float32)
    else:
        # every copy of row u has the same codes and weight: one row of weight c_u * scale / n_u carries them all
        fit_codes, fit_weights = codes_u, (mult * scale / counts_u.astype(np.float64)).astype(np.float32)
    run.counts, run.weights, run.n_eff = counts, weights, n_eff
    run.timings["reweighting_s"] = time.time() - t0
    _trace("reweighting done")
    log.append("Effective number of samples: %.1f\t(%.0f%% identical neighborhood = %.3f samples)"
               % (n_eff, 100.0 * theta, scale))

    # (a) PLM inference
    t0 = time.time()
    extra = {} if precision is None else {"precision": precision}
    from .engine import DeviceMemoryError
    try:
        problem = engine.plm_problem(fit_codes, fit_weights, q, ali.gap_code, lambda_h, lambda_J, m=history, **extra)
    except DeviceMemoryError as e:
        raise ResourceError(str(e))
    run.timings["problem_setup_s"] = time.time() - t0
    run.timings["seq_chunks"] = getattr(problem, "n_chunks", 1)
    run.timings["host_history_pairs"] = getattr(problem, "host_pairs", 0)
    try:
        t0 = time.time()
        fi_counts, fij_counts = problem.weighted_counts()
        fi, fij = model_io.normalise_frequencies(fi_counts, fij_counts, n_eff, ignore_gaps)
        run.timings["frequencies_s"] = time.time() - t0
        _trace("frequencies done")
        x0 = initial_point(fi, n_eff, L, q)

        log.append("\t".join(ITER_FIELDS))
        t_opt = time.time()
        ck = None
        fit_kw = {}
        if checkpoint:
            from . import checkpoint as _ckpt
            ck = _ckpt.CheckpointFile(checkpoint, checkpoint_interval, extra=dict(
                alphabet=ali.model_alphabet, data_sha256=_ckpt.data_digest(ali.codes, weights.astype(np.float32))))
            ck.info.update(max_iterations=max_iter, world=int(getattr(engine, "world", 1)), valid_rows=ali.n_valid,
                           unique_rows=run.timings["unique_rows"])
            fit_kw = dict(checkpoint=ck, checkpoint_interval=checkpoint_interval)
        rows = ck.rows if ck is not None else log
        t_prior = []

        def progress(k, fx, xnorm, gnorm, step, n_ls):
            if not t_prior:             # the time column continues across resumes
                t_prior.append(float(ck.header["state"]["seconds"]) if ck is not None and ck.header else 0.0)
            hn, en = problem.norms()
            rows.append("%d\t%.1f\t%.6f\t%.4f\t%.4f\t%.4f\t%.4f" % (
                k, t_prior[0] + time.time() - t_opt, gnorm / max(1.0, xnorm), fx, problem.last_negloglk, hn, en))
            return ck is not None and _ckpt.stop_requested()

        params = _lbfgs.default_params(max_iterations=max_iter, epsilon=epsilon, m=history)
        try:
            res = problem.fit(x0, params, progress, **fit_kw)
        except DeviceMemoryError as e:          # the fit workspace could not be allocated (device or pinned host)
            raise ResourceError(str(e))
        run.lbfgs = res
        run.timings["optimisation_s"] = time.time() - t_opt
        _trace("optimisation done")
        for key, val in (getattr(problem, "fit_stats", None) or {}).items():
            run.timings["fit_" + key] = val
        if ck is not None:
            log.extend(ck.rows)
            for key, val in ck.stats.items():
                run.timings["checkpoint_" + key] = val
            if res.status == _lbfgs.LBFGSERR_CANCELED:
                raise FitInterrupted("the fit stopped at iteration %d; its state is in %s and the same call "
                                     "continues from it" % (res.iterations, ck.path))
            if rank == 0 and res.status in (_lbfgs.LBFGS_SUCCESS, _lbfgs.LBFGS_ALREADY_MINIMIZED):
                ck.remove()
        log.append("Gradient optimization: %s" % res.status)

        x = problem.get_x()
        fn = problem.fn_scores()
    finally:
        close = getattr(problem, "close", None)
        if close is not None:
            close()
    run.x = x
    h = x[:L * q].reshape(L, q)
    J = x[L * q:].reshape(L * (L - 1) // 2, q, q)

    t0 = time.time()
    write_error = None
    if rank == 0:
        try:
            run.cn = model_io.write_ec_file(couplings_file, fn, L, ali.index_list, ali.target_seq)
            if param_file is not None:
                w_all = np.zeros(ali.n_total, dtype=np.float32)
                # golden plmc run stores the integer neighbour counts (0 on invalid rows); newer plmc
                # versions may store 1/n -- nothing in the reference reads this field numerically
                w_all[ali.valid] = (weights if store_inverse_weights else counts).astype(np.float32)
                model_io.write_model_file(
                    param_file, L, q, ali.n_valid, ali.n_total - ali.n_valid, int(res.iterations),
                    1.0 - theta, lambda_h, lambda_J, 0.0, n_eff, ali.model_alphabet, w_all,
                    ali.target_seq, ali.index_list, fi, h, fij, J)
        except Exception as e:          # agreed across ranks below: nobody is left waiting in a collective
            write_error = e
    agree = getattr(engine, "agree_any", None)
    failed = agree(write_error is not None) if agree is not None else (write_error is not None)
    if failed:
        if write_error is not None:
            raise write_error
        raise ResourceError("rank 0 failed to write the plmc output files")
    run.timings["write_files_s"] = time.time() - t0
    run.log = "\n".join(log) + "\n"
    run.timings["total_s"] = time.time() - t_start

    iter_df, fields = parse_plmc_log(run.log)
    if rank == 0:
        _require_file("plmc returned no couplings", couplings_file)
        if param_file is not None:
            _require_file("plmc returned no parameter file", param_file)
    result = PlmcResult(couplings_file, param_file, iter_df, *fields)
    run.result = result
    if return_run:
        return result, run
    return result
