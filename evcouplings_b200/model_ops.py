"""
SURVEY.md 8(f) rows f1 / f2: GPU versions of what the reference's ``CouplingsModel`` does with a fitted
model (evcouplings/couplings/model.py) -- same numbers, same table layout, no per-pair Python loops:

* ``read_model``            bulk plmc_v2 reader (the reference issues L(L-1) np.fromfile calls, model.py:375-389)
* ``ec_table``              FN / CN (zero-sum gauge + APC) / MI scores  <- _calculate_ecs  model.py:777-827
* ``hamiltonians``          statistical energies of many sequences     <- _hamiltonians    model.py:25-60
* ``single_mutant_matrix``  all single substitutions of the target     <- _single_mutant_hamiltonians model.py:63-109
* ``delta_hamiltonians``    energies of variants relative to the target <- delta_hamiltonian model.py:672-712
* ``PottsSampler`` / ``sample_sequences``  Gibbs samples of P(s) ~ exp(beta H(s)) (evc_sampler_*, include/evcplm.h),
                            or of chosen free sites given the rest of each chain's start (``free``, ``allowed``)
* ``BoltzmannLearner`` / ``boltzmann_refine``  bmDCA refinement of a fitted model (evc_code_counts, evc_bm_update)
* ``log_partition`` / ``log_probabilities``  log Z by annealed importance sampling (evc_sampler_anneal) and log P(s)
* ``design_codes``          high-scoring sequences: each chain's best state while sampling, annealing or tempering, then
                            a zero-temperature descent to a single-site optimum (evc_sampler_record_best, _descend)
"""
import ctypes
import math

import numpy as np

from . import _lib


def read_model(path):
    """Bulk reader of the plmc_v2 layout (model.py:317-389); tri blocks stay packed (npairs, q, q)."""
    with open(path, "rb") as f:
        L, q, nv, ni, it = (int(v) for v in np.fromfile(f, "<i4", 5))
        theta, lh, lj, lg, neff = (float(v) for v in np.fromfile(f, "<f4", 5))
        alphabet = f.read(q).decode("ascii")
        weights = np.fromfile(f, "<f4", nv + ni)
        target = f.read(L).decode("ascii")
        index_list = np.fromfile(f, "<i4", L)
        fi = np.fromfile(f, "<f4", L * q).reshape(L, q)
        h = np.fromfile(f, "<f4", L * q).reshape(L, q)
        npair = L * (L - 1) // 2
        fij = np.fromfile(f, "<f4", npair * q * q).reshape(npair, q, q)
        J = np.fromfile(f, "<f4", npair * q * q).reshape(npair, q, q)
    if J.size != npair * q * q:
        raise ValueError("truncated model file: " + str(path))
    return dict(L=L, q=q, n_valid=nv, n_invalid=ni, num_iter=it, theta=theta, lambda_h=lh, lambda_J=lj,
                lambda_group=lg, n_eff=neff, alphabet=alphabet, weights=weights, target_seq=target,
                index_list=index_list, fi=fi, h=h, fij=fij, J=J)


def _engine(engine):
    if engine is not None:
        return engine
    from .engine import CudaEngine
    return CudaEngine()


def apc(matrix):
    """Average product correction exactly as model.py:744-775 (diagonal blanked)."""
    L = matrix.shape[0]
    col_means = np.mean(matrix, axis=0) * L / (L - 1)
    matrix_mean = np.mean(matrix) * L / (L - 1)
    out = matrix - np.outer(col_means, col_means) / matrix_mean
    out[np.diag_indices(L)] = 0
    return out


def pair_scores(model, engine=None):
    """Per-pair raw-gauge FN, zero-sum-gauge FN and MI (pair order i<j row-major) from the device."""
    import torch
    eng = _engine(engine)
    L, q = model["L"], model["q"]
    dev = eng.device
    J = torch.from_numpy(np.ascontiguousarray(model["J"], dtype=np.float32)).to(dev)
    fij = torch.from_numpy(np.ascontiguousarray(model["fij"], dtype=np.float32)).to(dev)
    fi = torch.from_numpy(np.ascontiguousarray(model["fi"], dtype=np.float32)).to(dev)
    npair = L * (L - 1) // 2
    out = torch.zeros((3, npair), dtype=torch.float32, device=dev)
    _lib.check(eng.lib.evc_ec_scores(eng.ptr(J), eng.ptr(fij), eng.ptr(fi), L, q, eng.ptr(out[0]), eng.ptr(out[1]),
                                     eng.ptr(out[2]), eng.stream()), "evc_ec_scores")
    eng.kernel_launches += 1
    o = out.cpu().numpy().astype(np.float64)
    return o[0], o[1], o[2]


def ec_table(model, engine=None):
    """DataFrame with the columns of CouplingsModel.ecs (model.py:806-827), sorted by cn descending."""
    import pandas as pd
    L = model["L"]
    fn_raw, fn_zs, mi = pair_scores(model, engine)
    iu, ju = np.triu_indices(L, 1)

    def full(v):
        m = np.zeros((L, L))
        m[iu, ju] = v
        return m + m.T

    cn = apc(full(fn_zs))[iu, ju]
    mi_apc = apc(full(mi))[iu, ju]
    idx = np.asarray(model["index_list"])
    tgt = model["target_seq"]
    df = pd.DataFrame({
        "i": idx[iu], "A_i": [tgt[k] for k in iu], "j": idx[ju], "A_j": [tgt[k] for k in ju],
        "seqdist": np.abs(idx[iu] - idx[ju]), "mi_raw": mi, "mi_apc": mi_apc, "fn": fn_zs, "cn": cn,
    })
    return df.sort_values(by="cn", ascending=False)


def encode_sequences(model, sequences):
    """list of strings -> (N, L) uint8 codes in the model alphabet; characters outside it become q (ignored)."""
    q = model["q"]
    lut = np.full(256, q, dtype=np.uint8)
    for k, ch in enumerate(model["alphabet"]):
        lut[ord(ch)] = k
    arr = np.frombuffer("".join(sequences).encode("ascii"), dtype=np.uint8).reshape(len(sequences), model["L"])
    return lut[arr]


# sequences per batch of hamiltonians() are a multiple of this (the gather kernels' 2048-sequence tile)
HAMILTONIAN_BATCH_ALIGN = 2048
_HAMILTONIAN_MARGIN_BYTES = 512 << 20


def hamiltonian_batch_size(L, q, free_bytes):
    """Sequences per evc_plm_energies call that fit ``free_bytes``: the handle's gather-path buffers are two
    expanded coupling tensors (L-dependent) plus, per sequence, the L * S float residual row that holds the
    per-site partials, the codes, the packed MSA, the bucket lists and the output row."""
    S = q if q % 2 else q + 1
    QB, Lp = q + 1, -(-L // 4) * 4
    fixed = 2 * L * Lp * QB * S * 4 + 4 * (L * q + L * (L - 1) // 2 * q * q) + _HAMILTONIAN_MARGIN_BYTES
    per_seq = L * (4 * S + 8) + 64
    n = (int(free_bytes) - fixed) // per_seq
    return max(HAMILTONIAN_BATCH_ALIGN, n // HAMILTONIAN_BATCH_ALIGN * HAMILTONIAN_BATCH_ALIGN)


def model_x(model):
    """The parameter vector x = [h | J] of the library (plmc layout), float32."""
    return np.concatenate([np.asarray(model["h"], dtype=np.float32).ravel(),
                           np.asarray(model["J"], dtype=np.float32).ravel()])


def hamiltonians(model, sequences, engine=None, batch_size=None):
    """(N, 3) float64: total, couplings and fields part of the statistical energy of every sequence
    (strings, or an (N, L) integer matrix already mapped to the model alphabet).  The sequences are processed in
    batches sized from the free device memory (``batch_size`` overrides); every sequence's energy is computed on
    its own, so the result does not depend on the batching."""
    import torch
    eng = _engine(engine)
    if len(sequences) and isinstance(sequences[0], str):
        codes = encode_sequences(model, sequences)
    else:
        arr = np.ascontiguousarray(sequences)
        if arr.size and (arr.min() < 0 or arr.max() > model["q"]):
            raise ValueError("mapped sequence symbols must be in [0, %d] (%d = gap)" % (model["q"], model["q"]))
        codes = arr.astype(np.uint8)
    N, L = codes.shape
    q = model["q"]
    gap_code = q if int(codes.max(initial=0)) >= q else -1      # one layout for every batch
    if gap_code >= 0 and q >= 32:
        raise ValueError("a %d-state model has no code left for symbols outside its alphabet (codes must be < 32); "
                         "map every symbol to a model state" % q)
    dx = torch.from_numpy(model_x(model)).to(eng.device)
    if batch_size is None:
        torch.cuda.empty_cache()
        free, _total = torch.cuda.mem_get_info(eng.device)
        batch_size = hamiltonian_batch_size(L, q, free)
    batch_size = max(1, int(batch_size))
    res = np.empty((N, 3), dtype=np.float64)
    for b0 in range(0, N, batch_size):
        b1 = min(N, b0 + batch_size)
        batch = np.ascontiguousarray(codes[b0:b1])
        w = np.ones(b1 - b0, dtype=np.float32)
        handle = ctypes.c_void_p()
        _lib.check(eng.lib.evc_plm_create_alphabet(ctypes.byref(handle), batch.ctypes.data_as(ctypes.c_void_p), b1 - b0,
                                                   L, q, gap_code, w.ctypes.data_as(ctypes.c_void_p), eng.device_index),
                   "evc_plm_create_alphabet")
        try:
            out = torch.zeros((b1 - b0, 3), dtype=torch.float64, device=eng.device)
            _lib.check(eng.lib.evc_plm_energies(handle, eng.ptr(dx), eng.ptr(out), eng.stream()), "evc_plm_energies")
            eng.kernel_launches += 3
            res[b0:b1] = out.cpu().numpy()
        finally:
            eng.lib.evc_plm_destroy(handle)
        del out
    return res


def single_mutant_matrix(model, engine=None):
    """(L, q, 3) energy differences of every single substitution of the target sequence
    (model.py:63-109), obtained as energies of the L*q single mutants minus the target's."""
    L, q = model["L"], model["q"]
    tgt = encode_sequences(model, [model["target_seq"]])[0]
    muts = np.repeat(tgt[None, :], L * q + 1, axis=0)
    for i in range(L):
        muts[1 + i * q: 1 + (i + 1) * q, i] = np.arange(q)
    H = hamiltonians(model, muts, engine)
    return (H[1:] - H[0]).reshape(L, q, 3)


def delta_hamiltonians(model, variants, engine=None):
    """variants: list of substitution lists [(pos, from, to), ...] in index_list numbering (model.py:672-712).
    Returns (len(variants), 3)."""
    pos_of = {int(p): k for k, p in enumerate(model["index_list"])}
    amap = {ch: k for k, ch in enumerate(model["alphabet"])}
    tgt = encode_sequences(model, [model["target_seq"]])[0]
    seqs = np.repeat(tgt[None, :], len(variants) + 1, axis=0)
    for v, subs in enumerate(variants):
        for (p, a_from, a_to) in subs:
            k = pos_of[int(p)]
            if a_from != model["target_seq"][k]:
                raise ValueError("Inconsistency with target sequence: pos={} target={} subs={}".format(
                    p, model["target_seq"][k], a_from))
            seqs[v + 1, k] = amap[a_to]
    H = hamiltonians(model, seqs, engine)
    return H[1:] - H[0]


def conditional_sites(model, free=None, allowed=None, init="random"):
    """(sites, masks) of a conditional sampler: the free sites as ascending site indices (int32) and one allowed-state
    mask per free site (uint32, bit a = state a of the model alphabet).

    ``free``: positions in the model's ``index_list`` numbering (the numbering of delta_hamiltonians), any order,
    None for every site.  ``allowed``: dict position -> string of letters of the model alphabet, each position free;
    the other free sites allow every state.  Refuses unknown positions, letters outside the alphabet, ``allowed`` on a
    clamped site and init="random" with clamped sites (each chain's start is its context), with ValueError and before
    any device work."""
    L, q, alphabet = int(model["L"]), int(model["q"]), model["alphabet"]
    pos_of = {int(p): k for k, p in enumerate(model["index_list"])}
    if free is None:
        sites = list(range(L))
    else:
        free = [int(p) for p in free]
        unknown = sorted(set(p for p in free if p not in pos_of))
        if unknown:
            raise ValueError("free positions not in the model's index_list: %s" % unknown[:10])
        sites = sorted(set(pos_of[p] for p in free))
        if not sites:
            raise ValueError("free must name at least one position")
    masks = np.full(len(sites), (1 << q) - 1, dtype=np.uint64)
    slot = {k: n for n, k in enumerate(sites)}
    for p, letters in (allowed or {}).items():
        if int(p) not in pos_of:
            raise ValueError("allowed position %d is not in the model's index_list" % int(p))
        k = pos_of[int(p)]
        if k not in slot:
            raise ValueError("allowed position %d is clamped: only free positions can be restricted" % int(p))
        bad = sorted(set(letters) - set(alphabet))
        if bad or not letters:
            raise ValueError("allowed letters %r at position %d: need at least one letter, all in the model alphabet "
                             "%r" % (letters, int(p), alphabet))
        masks[slot[k]] = sum(1 << alphabet.index(ch) for ch in set(letters))
    if isinstance(init, str) and init == "random" and len(sites) < L:
        raise ValueError('init="random" with clamped sites: each chain needs a context, so give init="target" or a '
                         "matrix of codes")
    return np.array(sites, dtype=np.int32), masks.astype(np.uint32)


def check_ladder_contexts(start, free_sites, R):
    """Refuses (ValueError) ladders of R consecutive chains whose clamped codes differ: a swap exchanges the states
    of two chains, which is only valid between chains sampling the same conditional model."""
    start = np.asarray(start)
    clamped = np.setdiff1d(np.arange(start.shape[1]), np.asarray(free_sites))
    x = start[:, clamped].reshape(start.shape[0] // R, R, len(clamped))
    bad = np.flatnonzero((x != x[:, :1]).any(axis=(1, 2)))
    if len(bad):
        raise ValueError("the chains of ladder %d (chains %d..%d) have different contexts: every chain of a ladder "
                         "must share its clamped sites" % (bad[0], bad[0] * R, bad[0] * R + R - 1))


class PottsSampler(object):
    """Gibbs chains of P(s) ~ exp(beta H(s)) on the device (evc_sampler_*; the chain is specified in
    include/evcplm.h).  Chain k of this object is the global chain ``chain_offset + k``: its trajectory depends only on
    the model, its start, ``seed``, that index, the sweeps run and beta, so handles over disjoint index ranges (on one
    device or several) together give the chains one handle over the whole range gives.

    ``init``: "random" (uniform start drawn from the chain's counter), "target" (every chain starts at the model's
    target sequence) or an (n_chains, L) integer matrix of codes < q.

    ``free`` / ``allowed`` (conditional_sites) make a conditional sampler (evc_sampler_create_conditional), even when
    every site is free: the chains redraw only the free sites, each from its allowed letters, given the other sites,
    which keep each chain's start.  A free site may start outside its allowed letters; it holds an allowed one after
    the first sweep.  A conditional sampler cannot anneal."""

    def __init__(self, model, n_chains, seed=0, init="random", chain_offset=0, engine=None, free=None, allowed=None):
        import torch
        self.conditional = free is not None or allowed is not None
        if self.conditional:
            self.free_sites, masks = conditional_sites(model, free, allowed, init)
        self.eng = _engine(engine)
        self.L, self.q = int(model["L"]), int(model["q"])
        self.n_chains = int(n_chains)
        self.alphabet = model["alphabet"]
        self.chain_offset = int(chain_offset)
        self.ladder = None              # set_ladder(): the rungs' betas (float32), swap interval and swap counts
        self.recording = False          # record_best() has run
        if isinstance(init, str):
            if init == "random":
                start = None
            elif init == "target":
                start = np.repeat(encode_sequences(model, [model["target_seq"]]), max(self.n_chains, 0), axis=0)
            else:
                raise ValueError('init must be "random", "target" or a matrix of codes, not %r' % init)
        else:
            start = np.asarray(init)
            if start.shape != (self.n_chains, self.L):
                raise ValueError("init codes must have shape (%d, %d), not %s" % (self.n_chains, self.L, start.shape))
            if start.size and (start.min() < 0 or start.max() >= self.q):
                raise ValueError("init codes must be in [0, %d]" % (self.q - 1))
        if start is not None:
            start = np.ascontiguousarray(start, dtype=np.uint8)
        # a conditional sampler's clamped codes, which the chains of one ladder must share (set_ladder)
        self._context = start if self.conditional and len(self.free_sites) < self.L else None
        self.t = 0                      # the handle's global sweep index
        dx = torch.from_numpy(model_x(model)).to(self.eng.device)
        torch.cuda.synchronize(self.eng.device)
        self._logw = None               # anneal(): device log weights, allocated at the first call
        self.handle = ctypes.c_void_p()
        if self.conditional:
            _lib.check(self.eng.lib.evc_sampler_create_conditional(
                ctypes.byref(self.handle), self.eng.ptr(dx), self.L, self.q,
                self.free_sites.ctypes.data_as(ctypes.c_void_p), len(self.free_sites),
                masks.ctypes.data_as(ctypes.c_void_p), None if start is None else start.ctypes.data_as(ctypes.c_void_p),
                self.n_chains, int(chain_offset), int(seed) % (1 << 64), self.eng.device_index),
                "evc_sampler_create_conditional")
            self.eng.kernel_launches += 3
            return
        _lib.check(self.eng.lib.evc_sampler_create(
            ctypes.byref(self.handle), self.eng.ptr(dx), self.L, self.q,
            None if start is None else start.ctypes.data_as(ctypes.c_void_p), self.n_chains, int(chain_offset),
            int(seed) % (1 << 64), self.eng.device_index), "evc_sampler_create")
        self.eng.kernel_launches += 2

    def run(self, sweeps, beta=1.0):
        """Runs ``sweeps`` sweeps of every chain at inverse temperature ``beta``; returns the number of site changes."""
        changes = ctypes.c_int64()
        _lib.check(self.eng.lib.evc_sampler_run(self.handle, int(sweeps), float(beta), ctypes.byref(changes),
                                                self.eng.stream()), "evc_sampler_run")
        self.eng.kernel_launches += 1
        self.t += int(sweeps)
        return int(changes.value)

    def anneal(self, betas):
        """Runs len(betas) - 1 annealed sweeps along the schedule ``betas`` (evc_sampler_anneal: couplings scaled by
        beta, fields not), accumulating each chain's log importance weight into a device buffer this object owns
        (zero at creation, see log_weights); returns the number of site changes."""
        import torch
        if self.conditional:
            raise ValueError("a conditional sampler cannot anneal: AIS runs over every site of the model")
        if self.recording:
            raise ValueError("a recording sampler (record_best) cannot anneal")
        b = np.ascontiguousarray(betas, dtype=np.float32)
        if b.ndim != 1 or b.size < 1:
            raise ValueError("betas must be a non-empty 1-d schedule")
        if self._logw is None:
            self._logw = torch.zeros(self.n_chains, dtype=torch.float64, device=self.eng.device)
        changes = ctypes.c_int64()
        _lib.check(self.eng.lib.evc_sampler_anneal(self.handle, b.ctypes.data_as(ctypes.c_void_p), b.size - 1,
                                                   self.eng.ptr(self._logw), ctypes.byref(changes), self.eng.stream()),
                   "evc_sampler_anneal")
        self.eng.kernel_launches += 1
        self.t += b.size - 1
        return int(changes.value)

    def log_weights(self):
        """(n_chains,) float64 numpy array of the log weights accumulated by anneal() since creation or the last
        reset_log_weights()."""
        if self._logw is None:
            return np.zeros(self.n_chains)
        return self._logw.cpu().numpy()

    def reset_log_weights(self):
        """Sets every log weight back to 0."""
        if self._logw is not None:
            self._logw.zero_()

    def set_ladder(self, betas, swap_interval=1):
        """Makes the chains replica-exchange ladders (evc_sampler_set_ladder): ``betas`` are R >= 2 inverse
        temperatures, strictly ascending from betas[0] >= 0 once rounded to float32; ladder l is the chains l R ..
        l R + R - 1 (global ladder chain_offset / R + l), chain l R + k starting at rung k.  After every
        ``swap_interval`` sweeps of temper() the adjacent rungs (k, k + 1), k of the round's parity, try to exchange
        their betas.  n_chains and chain_offset must be multiples of R.  Once set, anneal() is refused."""
        import torch
        b = np.ascontiguousarray(betas, dtype=np.float32)
        if b.ndim != 1:
            raise ValueError("betas must be a 1-d ladder")
        if self._context is not None and b.size >= 2 and self.n_chains % b.size == 0:
            check_ladder_contexts(self._context, self.free_sites, b.size)
        _lib.check(self.eng.lib.evc_sampler_set_ladder(self.handle, b.ctypes.data_as(ctypes.c_void_p), b.size,
                                                       int(swap_interval)), "evc_sampler_set_ladder")
        if self.ladder is None:
            self.ladder = b
            self.swap_interval = int(swap_interval)
            self._swaps = torch.zeros(2 * (b.size - 1), dtype=torch.int64, device=self.eng.device)
            self.eng.kernel_launches += 1

    def temper(self, sweeps):
        """Runs ``sweeps`` sweeps of every chain at the beta of the rung it holds, with the swap rounds they reach
        (evc_sampler_temper); returns the number of site changes."""
        if self.ladder is None:
            raise ValueError("temper() needs a ladder: call set_ladder() first")
        changes = ctypes.c_int64()
        _lib.check(self.eng.lib.evc_sampler_temper(self.handle, int(sweeps), self.eng.ptr(self._swaps),
                                                   ctypes.byref(changes), self.eng.stream()), "evc_sampler_temper")
        # one sweep launch per segment (each ends at a swap round or at the call's end), one swap launch per round
        t, k, K = self.t, int(sweeps), self.swap_interval
        rounds = (t + k) // K - t // K
        self.eng.kernel_launches += 2 * rounds + (1 if k > 0 and (t + k) % K else 0)
        self.t += k
        return int(changes.value)

    def _ladder_state(self):
        import torch
        R = self.ladder.size
        rung = torch.empty(self.n_chains, dtype=torch.int32, device=self.eng.device)
        energy = torch.empty(self.n_chains, dtype=torch.float64, device=self.eng.device)
        trips = torch.empty(self.n_chains // R, dtype=torch.int64, device=self.eng.device)
        _lib.check(self.eng.lib.evc_sampler_ladder_state(self.handle, self.eng.ptr(rung), self.eng.ptr(energy),
                                                         self.eng.ptr(trips), self.eng.stream()),
                   "evc_sampler_ladder_state")
        return rung.cpu().numpy(), energy.cpu().numpy(), trips.cpu().numpy()

    def rungs(self):
        """(n_chains,) int32: the rung each chain holds."""
        return self._ladder_state()[0]

    def energies(self):
        """(n_chains,) float64: each chain's energy H at the last swap round (0 before the first)."""
        return self._ladder_state()[1]

    def rung_codes(self, k):
        """(G, L) uint8: the codes of the chain holding rung ``k`` of each of the G ladders, in ladder order."""
        if self.ladder is None:
            raise ValueError("rung_codes() needs a ladder: call set_ladder() first")
        R = self.ladder.size
        if not 0 <= int(k) < R:
            raise ValueError("rung %r is not in [0, %d)" % (k, R))
        rung = self.rungs().reshape(-1, R)
        at = np.argmax(rung == int(k), axis=1)
        return self.codes().reshape(-1, R, self.L)[np.arange(len(rung)), at]

    def swap_statistics(self):
        """dict of int64 numpy arrays over the pairs (k, k + 1): ``attempted`` and ``accepted`` swaps since set_ladder,
        ``acceptance`` = accepted / attempted (nan before an attempt), and ``round_trips`` per ladder."""
        if self.ladder is None:
            raise ValueError("swap_statistics() needs a ladder: call set_ladder() first")
        R = self.ladder.size
        counts = self._swaps.cpu().numpy()
        trips = self._ladder_state()[2]
        return _swap_summary(counts[:R - 1], counts[R - 1:], trips)

    def record_best(self):
        """Starts (or restarts) each chain's record (evc_sampler_record_best): every later sweep of run() and temper()
        keeps, per chain, the highest energy H its state reached after a sweep (on a conditional sampler the energy of
        the free sites given the context), those codes and that sweep.  A recording sampler cannot anneal."""
        _lib.check(self.eng.lib.evc_sampler_record_best(self.handle, self.eng.stream()), "evc_sampler_record_best")
        self.eng.kernel_launches += 1
        self.recording = True

    def best(self):
        """(energy, codes, sweep) of the record (evc_sampler_best): (n_chains,) float64, (n_chains, L) uint8 full rows
        and (n_chains,) int64 global sweep indices; -inf, the codes at record_best() and -1 for a chain no sweep has
        recorded yet."""
        import torch
        if not self.recording:
            raise ValueError("best() needs a record: call record_best() first")
        energy = torch.empty(self.n_chains, dtype=torch.float64, device=self.eng.device)
        codes = torch.empty((self.n_chains, self.L), dtype=torch.uint8, device=self.eng.device)
        sweep = torch.empty(self.n_chains, dtype=torch.int64, device=self.eng.device)
        _lib.check(self.eng.lib.evc_sampler_best(self.handle, self.eng.ptr(energy), self.eng.ptr(codes),
                                                 self.eng.ptr(sweep), self.eng.stream()), "evc_sampler_best")
        return energy.cpu().numpy(), codes.cpu().numpy(), sweep.cpu().numpy()

    def descend(self, sweeps):
        """Runs ``sweeps`` zero-temperature sweeps of every chain (evc_sampler_descend: each site to its best allowed
        state given the others, ties to the current state, then to the smallest); returns (settled, changes):
        settled (n_chains,) bool, true for a chain whose last sweep changed nothing (all false when sweeps = 0)."""
        import torch
        if int(sweeps) < 0:
            raise ValueError("sweeps must be >= 0, not %r" % sweeps)
        settled = torch.zeros(self.n_chains, dtype=torch.uint8, device=self.eng.device)
        changes = ctypes.c_int64()
        _lib.check(self.eng.lib.evc_sampler_descend(self.handle, int(sweeps), self.eng.ptr(settled),
                                                    ctypes.byref(changes), self.eng.stream()), "evc_sampler_descend")
        self.eng.kernel_launches += 1 if int(sweeps) else 0
        self.t += int(sweeps)
        return settled.cpu().numpy().astype(bool), int(changes.value)

    def codes(self):
        """(n_chains, L) uint8 numpy array of the chains' current codes."""
        import torch
        out = torch.empty((self.n_chains, self.L), dtype=torch.uint8, device=self.eng.device)
        _lib.check(self.eng.lib.evc_sampler_codes(self.handle, self.eng.ptr(out), self.eng.stream()),
                   "evc_sampler_codes")
        return out.cpu().numpy()

    def conditional_fields(self):
        """(n_chains, nf, q) float32 numpy array of a conditional sampler's folded fields hc: h of the free sites plus
        the couplings to each chain's clamped sites (evc_sampler_conditional_fields)."""
        import torch
        out = torch.empty((self.n_chains, len(self.free_sites), self.q), dtype=torch.float32, device=self.eng.device)
        _lib.check(self.eng.lib.evc_sampler_conditional_fields(self.handle, self.eng.ptr(out), self.eng.stream()),
                   "evc_sampler_conditional_fields")
        return out.cpu().numpy()

    def close(self):
        if getattr(self, "handle", None):
            self.eng.lib.evc_sampler_destroy(self.handle)
            self.handle = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# Several ranks (one process per GPU, torch.distributed): M global chains are split in contiguous blocks, rank r
# holding chains [lo, hi) of dist.shard_bounds as a PottsSampler with chain_offset = lo.  A chain's trajectory does
# not depend on which handle runs it, so the ranks together run exactly the chains of one process.
MAX_SHARDED_CHAINS = (1 << 31) - 1          # the summed pair counts are int32


def chain_range(n_chains, world, rank):
    """(lo, hi) of the global chains rank ``rank`` of ``world`` runs.  Refuses fewer chains than ranks (a rank
    without chains) and more than MAX_SHARDED_CHAINS (the int32 sum of the pair counts), before any device work."""
    M, R = int(n_chains), int(world)
    if M < R:
        raise ValueError("%d chains cannot be split over %d ranks: every rank needs at least one chain" % (M, R))
    if M > MAX_SHARDED_CHAINS:
        raise ValueError("%d chains: split over ranks the pair counts are summed in int32, so at most 2^31 - 1 "
                         "chains" % M)
    from .dist import shard_bounds
    return shard_bounds(M, R, int(rank))


def _ranks(eng):
    return int(getattr(eng, "world", 1)), int(getattr(eng, "rank", 0))


def _gather_chains(eng, local, n_chains):
    """This rank's rows of a per-chain numpy array, gathered from every rank in global chain order: an all-gather of
    blocks padded to the largest shard (rank 0's), then trimmed; the bits of every row travel unchanged."""
    import torch
    world, _rank = _ranks(eng)
    if world == 1:
        return local
    width = chain_range(n_chains, world, 0)[1]
    buf = torch.zeros((width,) + local.shape[1:], dtype=torch.from_numpy(local[:0]).dtype, device=eng.device)
    buf[:len(local)] = torch.from_numpy(np.ascontiguousarray(local)).to(eng.device)
    blocks = eng.all_gather(buf)
    out = []
    for r, b in enumerate(blocks):
        lo, hi = chain_range(n_chains, world, r)
        out.append(b[:hi - lo].cpu().numpy())
    return np.concatenate(out)


def check_num_gpus(num_gpus, n_chains, backend="nccl"):
    """Refuses a rank count the generative tools cannot run, before any rank starts: fewer than one, more GPUs than
    are visible (over NCCL every rank needs its own device; gloo ranks may share one) and fewer chains than ranks."""
    R = int(num_gpus)
    if R < 1:
        raise ValueError("num_gpus must be at least 1, not %r" % num_gpus)
    if R > 1 and backend == "nccl":
        import torch
        visible = torch.cuda.device_count()
        if R > visible:
            raise ValueError("num_gpus = %d but %d GPU%s visible" % (R, visible, " is" if visible == 1 else "s are"))
    if R > 1:
        chain_range(n_chains, R, 0)
    return R


def _on_ranks(job, num_gpus, backend, kwargs):
    from . import launcher
    return launcher.run_job(job, num_gpus, kwargs, backend=backend)


def check_ladder(betas, swap_interval=1):
    """The ladder as float32: R >= 2 finite betas, strictly ascending from betas[0] >= 0 once rounded to float32, and
    swap_interval >= 1; ValueError otherwise (the checks of evc_sampler_set_ladder, before any device work)."""
    b = np.asarray(betas, dtype=np.float64)
    if b.ndim != 1 or b.size < 2:
        raise ValueError("a ladder needs at least 2 inverse temperatures")
    if not np.all(np.isfinite(b)):
        raise ValueError("the ladder's inverse temperatures must be finite")
    b = b.astype(np.float32)
    if b[0] < 0 or np.any(np.diff(b) <= 0):
        raise ValueError("the ladder must be strictly ascending from beta_0 >= 0 once rounded to float32: %s" %
                         ", ".join("%.9g" % v for v in b))
    if int(swap_interval) < 1:
        raise ValueError("swap_interval must be at least 1, not %r" % swap_interval)
    return b


def geometric_ladder(beta_min, beta_max, R):
    """R inverse temperatures beta_min (beta_max / beta_min)^(k / (R - 1)), computed in double and rounded to float32,
    the ends exact; refused (ValueError) unless 0 < beta_min < beta_max and the rounded ladder strictly ascends."""
    R = int(R)
    if R < 2:
        raise ValueError("a ladder needs at least 2 rungs, not %d" % R)
    lo, hi = float(beta_min), float(beta_max)
    if not (np.isfinite(lo) and np.isfinite(hi) and 0 < lo < hi):
        raise ValueError("a geometric ladder needs 0 < beta_min < beta_max (got %r, %r)" % (beta_min, beta_max))
    b = lo * (hi / lo) ** (np.arange(R, dtype=np.float64) / (R - 1))
    b[0], b[-1] = lo, hi
    return check_ladder(b)


def _swap_summary(attempted, accepted, trips):
    attempted = np.asarray(attempted, dtype=np.int64)
    accepted = np.asarray(accepted, dtype=np.int64)
    with np.errstate(invalid="ignore", divide="ignore"):
        rate = accepted / attempted
    return dict(attempted=attempted, accepted=accepted, acceptance=rate,
                round_trips=np.asarray(trips, dtype=np.int64))


def sample_codes(model, n, sweeps, seed=0, beta=1.0, init="random", engine=None, num_gpus=1, backend="nccl",
                 free=None, allowed=None, ladder=None, swap_interval=1, return_statistics=False):
    """(n, L) uint8 codes: the states of chains 0..n-1 after ``sweeps`` sweeps (PottsSampler).  With an engine whose
    collective has several ranks, each rank runs its block of chains and every rank returns all n rows in chain order;
    ``num_gpus`` > 1 starts that many ranks (evcouplings_b200.launcher) and returns their result.  ``free`` and
    ``allowed`` sample only the free sites given the rest of each chain's start (PottsSampler, conditional_sites);
    they are checked before any rank starts.

    ``ladder`` (R inverse temperatures, check_ladder) runs n replica-exchange ladders instead (PottsSampler.set_ladder,
    temper): ladder l is the chains l R .. l R + R - 1, all starting from row l of an ``init`` matrix (one row per
    ladder), and row l of the result is the chain at the top rung, beta = ladder[-1] (``beta`` is not used).  Ranks
    run whole ladders.  ``return_statistics`` also returns swap_statistics() of all n ladders (the swap counts summed
    as int64 over the ranks, the round trips in ladder order): (codes, statistics)."""
    if free is not None or allowed is not None:
        conditional_sites(model, free, allowed, init)
    if ladder is not None:
        ladder = check_ladder(ladder, swap_interval)
    elif return_statistics:
        raise ValueError("return_statistics needs a ladder")
    if check_num_gpus(num_gpus, n, backend) > 1:
        return _on_ranks("sample", num_gpus, backend, dict(model=model, n=n, sweeps=sweeps, seed=seed, beta=beta,
                                                           init=init, free=free, allowed=allowed, ladder=ladder,
                                                           swap_interval=swap_interval,
                                                           return_statistics=return_statistics))
    eng = _engine(engine)
    world, rank = _ranks(eng)
    lo, hi = (0, int(n)) if world == 1 else chain_range(n, world, rank)
    if not isinstance(init, str):
        init = np.asarray(init)
        if init.shape != (int(n), int(model["L"])):
            raise ValueError("init codes must have shape (%d, %d), not %s" % (int(n), model["L"], init.shape))
        init = init[lo:hi]
    if ladder is None:
        with PottsSampler(model, hi - lo, seed=seed, init=init, chain_offset=lo, engine=eng, free=free,
                          allowed=allowed) as sampler:
            sampler.run(sweeps, beta)
            codes = sampler.codes()
        return _gather_chains(eng, codes, n)
    R = ladder.size
    if not isinstance(init, str):
        init = np.repeat(init, R, axis=0)
    with PottsSampler(model, (hi - lo) * R, seed=seed, init=init, chain_offset=lo * R, engine=eng, free=free,
                      allowed=allowed) as sampler:
        sampler.set_ladder(ladder, swap_interval)
        sampler.temper(sweeps)
        codes = _gather_chains(eng, sampler.rung_codes(R - 1), n)
        swaps = sampler._swaps.clone()
        trips = _gather_chains(eng, sampler._ladder_state()[2], n)
    if not return_statistics:
        return codes
    if world > 1:
        eng.all_reduce(swaps)
    swaps = swaps.cpu().numpy()
    return codes, _swap_summary(swaps[:R - 1], swaps[R - 1:], trips)


def sample_sequences(model, n, sweeps, seed=0, beta=1.0, init="random", engine=None, num_gpus=1, backend="nccl",
                     free=None, allowed=None, ladder=None, swap_interval=1):
    """``n`` sequences (strings in the model alphabet): the states of chains 0..n-1 after ``sweeps`` sweeps, or with
    ``ladder`` the top rung of n ladders.  ``num_gpus`` and sharding over an engine's ranks as in sample_codes, whose
    result does not depend on either; ``free``, ``allowed``, ``ladder`` and ``swap_interval`` as there."""
    codes = sample_codes(model, n, sweeps, seed, beta, init, engine, num_gpus, backend, free, allowed, ladder,
                         swap_interval)
    lut = np.frombuffer(model["alphabet"].encode("ascii"), dtype=np.uint8)
    return [bytes(row).decode("ascii") for row in lut[codes]]


DESCENT_BLOCK = 32      # descent sweeps per evc_sampler_descend call of design_codes: EVC_SAMPLER_REFRESH


def anneal_schedule(beta_start, beta, sweeps):
    """The inverse temperatures of ``sweeps`` annealing sweeps, geometric from beta_start to beta as geometric_ladder
    computes a ladder (in double, rounded to float32, the ends exact); refused unless 0 < beta_start < beta, finite."""
    lo, hi, S = float(beta_start), float(beta), int(sweeps)
    if not (np.isfinite(lo) and np.isfinite(hi) and 0 < lo < hi):
        raise ValueError("annealing needs 0 < beta_start < beta (got %r, %r)" % (beta_start, beta))
    if S < 2:
        return np.full(max(S, 0), hi, dtype=np.float32)
    b = lo * (hi / lo) ** (np.arange(S, dtype=np.float64) / (S - 1))
    b[0], b[-1] = lo, hi
    return b.astype(np.float32)


def design_codes(model, n, sweeps, seed=0, beta=1.0, beta_start=None, init="random", free=None, allowed=None,
                 ladder=None, swap_interval=1, descent_sweeps=256, engine=None, num_gpus=1, backend="nccl"):
    """Designs n sequences that score high under the model: each chain (or ladder) records its best state while it
    samples, and a zero-temperature descent then takes that state to a single-site optimum.

      1. A record is started (PottsSampler.record_best) and the chains run one of three schedules: ``beta_start``
         given, simulated annealing, one run(1, beta_k) per sweep along anneal_schedule(beta_start, beta, sweeps);
         ``ladder`` given, replica exchange (set_ladder, temper(sweeps)), each ladder's candidate being its chain with
         the highest record (ties to the lowest chain); otherwise run(sweeps, beta).
      2. A new sampler (conditional with the same ``free`` / ``allowed`` when given) starts from the candidates and
         descends in blocks of DESCENT_BLOCK sweeps until every chain's last sweep changed nothing or
         ``descent_sweeps`` sweeps have run.
      3. The results are scored with hamiltonians().

    Returns a dict: ``codes`` (n, L) uint8, ``energy`` (n,) float64 H of each row (hamiltonians), ``settled`` (n,)
    bool (the descent's last sweep left the row unchanged: a single-site optimum of the fp32 fields), ``found_at`` (n,)
    int64 (the global sweep at which step 1 recorded the candidate, -1 if none), and with ``ladder`` also
    ``swap_statistics`` (as sample_codes).  Chains, ladders, ``init``, ``free`` and ``allowed`` as in sample_codes;
    ranks shard them as there and the result does not depend on ``num_gpus`` or on the number of ranks."""
    if free is not None or allowed is not None:
        conditional_sites(model, free, allowed, init)
    if ladder is not None and beta_start is not None:
        raise ValueError("give either beta_start (annealing) or ladder (replica exchange), not both")
    if ladder is not None:
        ladder = check_ladder(ladder, swap_interval)
    if int(sweeps) < 0 or int(sweeps) >= 1 << 31:
        raise ValueError("sweeps must be in [0, 2^31), not %r" % sweeps)
    if int(descent_sweeps) < 0:
        raise ValueError("descent_sweeps must be >= 0, not %r" % descent_sweeps)
    if not math.isfinite(float(beta)):
        raise ValueError("beta must be finite, not %r" % beta)
    schedule = None if beta_start is None else anneal_schedule(beta_start, beta, sweeps)
    if check_num_gpus(num_gpus, n, backend) > 1:
        return _on_ranks("design", num_gpus, backend, dict(
            model=model, n=n, sweeps=sweeps, seed=seed, beta=beta, beta_start=beta_start, init=init, free=free,
            allowed=allowed, ladder=ladder, swap_interval=swap_interval, descent_sweeps=descent_sweeps))
    eng = _engine(engine)
    world, rank = _ranks(eng)
    lo, hi = (0, int(n)) if world == 1 else chain_range(n, world, rank)
    L = int(model["L"])
    if not isinstance(init, str):
        init = np.asarray(init)
        if init.shape != (int(n), L):
            raise ValueError("init codes must have shape (%d, %d), not %s" % (int(n), L, init.shape))
        init = init[lo:hi]
    out = {}
    if ladder is None:
        with PottsSampler(model, hi - lo, seed=seed, init=init, chain_offset=lo, engine=eng, free=free,
                          allowed=allowed) as s:
            s.record_best()
            if schedule is None:
                s.run(sweeps, beta)
            else:
                for b in schedule:
                    s.run(1, b)
            _energy, start, found = s.best()
    else:
        R = ladder.size
        if not isinstance(init, str):
            init = np.repeat(init, R, axis=0)
        with PottsSampler(model, (hi - lo) * R, seed=seed, init=init, chain_offset=lo * R, engine=eng, free=free,
                          allowed=allowed) as s:
            s.set_ladder(ladder, swap_interval)
            s.record_best()
            s.temper(sweeps)
            energy, codes, sweep = s.best()
            pick = np.arange(hi - lo) * R + np.argmax(energy.reshape(-1, R), axis=1)   # first of the maxima
            start, found = codes[pick], sweep[pick]
            swaps = s._swaps.clone()
            trips = _gather_chains(eng, s._ladder_state()[2], n)
        if world > 1:
            eng.all_reduce(swaps)
        swaps = swaps.cpu().numpy()
        out["swap_statistics"] = _swap_summary(swaps[:R - 1], swaps[R - 1:], trips)
    settled = np.zeros(hi - lo, dtype=bool)
    with PottsSampler(model, hi - lo, seed=seed, init=start, chain_offset=lo, engine=eng, free=free,
                      allowed=allowed) as d:
        done = 0
        while done < int(descent_sweeps):
            k = min(DESCENT_BLOCK, int(descent_sweeps) - done)
            settled, _changes = d.descend(k)
            done += k
            moving = not settled.all()
            if world > 1:
                moving = eng.agree_any(moving)      # every rank runs the same blocks, as one process would
            if not moving:
                break
        codes = d.codes()
    out["codes"] = _gather_chains(eng, codes, n)
    out["energy"] = _gather_chains(eng, np.ascontiguousarray(hamiltonians(model, codes, eng)[:, 0]), n)
    out["settled"] = _gather_chains(eng, settled.astype(np.uint8), n).astype(bool)
    out["found_at"] = _gather_chains(eng, found, n)
    return out


def ais_summary(log_w):
    """(log mean w, ESS, standard error) of importance weights given as logs, in float64: ESS = (sum w)^2 / sum w^2
    and the delta-method standard error of log mean w, sqrt(1 / ESS - 1 / M)."""
    lw = np.asarray(log_w, dtype=np.float64)
    M = lw.size
    m = lw.max()
    w = np.exp(lw - m)
    s1, s2 = w.sum(), (w * w).sum()
    ess = s1 * s1 / s2
    return float(m + np.log(s1) - np.log(M)), float(ess), float(math.sqrt(max(0.0, 1.0 / ess - 1.0 / M)))


def log_partition(model, n_chains=8192, temperatures=1024, burn_in=None, seed=0, engine=None, num_gpus=1,
                  backend="nccl"):
    """log Z of a plmc_v2 model by annealed importance sampling on the device (evc_sampler_anneal).

    ``n_chains`` chains start uniformly, take one exact sample of the independent-site model p_0 (a sweep at beta = 0),
    and anneal along beta_k = k / K, K = ``temperatures`` (a power of two, so every beta is dyadic), to the model:
    log Z = log Z_0 + logsumexp(log w) - log M.  The same chains then run ``burn_in`` sweeps at beta = 1 (default K)
    and anneal back to 0, which gives log Z_reverse = log Z_0 - (logsumexp(log w_rev) - log M): with equilibrated
    starts a stochastic upper estimate against the forward lower one, so their gap shows how far to trust either.
    Returns a dict: log_z, log_z_reverse, log_z0, ess, ess_reverse, stderr, stderr_reverse (the delta-method standard
    errors of ais_summary) and the arguments n_chains, temperatures, burn_in, seed.

    With an engine whose collective has several ranks, each rank anneals its block of chains (forward, burn-in,
    reverse), the per-chain log weights are gathered in chain order and every rank returns the dict of one process,
    bit for bit.  ``num_gpus`` > 1 starts that many ranks (evcouplings_b200.launcher) and returns their result."""
    M, K = int(n_chains), int(temperatures)
    B = K if burn_in is None else int(burn_in)
    if M < 1:
        raise ValueError("need at least one chain, not %r" % n_chains)
    if K < 1 or K >= 1 << 31 or K & (K - 1):
        raise ValueError("temperatures must be a power of two in [1, 2^30], not %r" % temperatures)
    if B < 0 or B >= 1 << 31:
        raise ValueError("burn_in must be in [0, 2^31), not %r" % burn_in)
    if check_num_gpus(num_gpus, M, backend) > 1:
        return _on_ranks("logz", num_gpus, backend, dict(model=model, n_chains=M, temperatures=K, burn_in=B,
                                                         seed=seed))
    eng = _engine(engine)
    world, rank = _ranks(eng)
    lo, hi = (0, M) if world == 1 else chain_range(M, world, rank)
    h = np.asarray(model["h"], dtype=np.float64)
    m = h.max(axis=1, keepdims=True)
    log_z0 = float(np.sum(m[:, 0] + np.log(np.exp(h - m).sum(axis=1))))
    betas = (np.arange(K + 1, dtype=np.float64) / K).astype(np.float32)
    with PottsSampler(model, hi - lo, seed=seed, chain_offset=lo, engine=eng) as s:
        s.anneal([0.0, 0.0])
        s.anneal(betas)
        lw_fwd = s.log_weights()
        s.reset_log_weights()
        s.run(B, 1.0)
        s.anneal(betas[::-1])
        lw_rev = s.log_weights()
    fwd = ais_summary(_gather_chains(eng, lw_fwd, M))
    rev = ais_summary(_gather_chains(eng, lw_rev, M))
    return dict(log_z=log_z0 + fwd[0], log_z_reverse=log_z0 - rev[0], log_z0=log_z0, ess=fwd[1], ess_reverse=rev[1],
                stderr=fwd[2], stderr_reverse=rev[2], n_chains=M, temperatures=K, burn_in=B, seed=int(seed))


def log_probabilities(model, sequences, log_z, engine=None):
    """(N,) float64 log P(s) = H(s) - log Z of every sequence (strings, or an (N, L) integer matrix of codes), with
    H from hamiltonians().  Refuses sequences with a symbol outside the model's q states (for example a gap under a
    model fitted with ignored gaps, whose states do not include it): P is not defined there."""
    if len(sequences) and isinstance(sequences[0], str):
        if any(len(x) != model["L"] for x in sequences):
            raise ValueError("every sequence must have the model's L = %d sites" % model["L"])
        codes = encode_sequences(model, sequences)
    else:
        codes = np.asarray(sequences)
        if codes.ndim != 2 or codes.shape[1] != model["L"]:
            raise ValueError("codes must have shape (N, %d), not %s" % (model["L"], codes.shape))
    bad = int(np.count_nonzero(((codes < 0) | (codes >= model["q"])).any(axis=1))) if codes.size else 0
    if bad:
        raise ValueError("%d of %d sequences have symbols outside the model's %d states; log P is not defined for "
                         "them" % (bad, len(codes), model["q"]))
    if not len(codes):
        return np.zeros(0)
    return hamiltonians(model, codes.astype(np.uint8), engine)[:, 0] - float(log_z)


def bm_regularisation(model):
    """(lam2_h, lam2_J) = (2 lambda_h / n_eff, 2 lambda_J / n_eff) of the Boltzmann-machine objective (include/evcplm.h)
    from the .model header, in double; both 0 when n_eff <= 0 and both lambda are 0.  Refuses a mean-field header
    and n_eff <= 0 with a non-zero lambda."""
    lh, lj, neff = float(model["lambda_h"]), float(model["lambda_J"]), float(model["n_eff"])
    if lh < 0:
        raise ValueError("lambda_h < 0 marks a mean-field model; Boltzmann-machine learning refines a "
                         "pseudo-likelihood model")
    if not (math.isfinite(lh) and math.isfinite(lj) and math.isfinite(neff)) or lj < 0:
        raise ValueError("the model header needs finite lambda_h, lambda_J >= 0 and n_eff")
    if neff <= 0:
        if lh != 0 or lj != 0:
            raise ValueError("n_eff = %g <= 0 with a non-zero lambda: the regularisation lambda / n_eff is undefined"
                             % neff)
        return 0.0, 0.0
    return 2.0 * lh / neff, 2.0 * lj / neff


class BoltzmannLearner(object):
    """Boltzmann-machine learning (bmDCA) of a plmc_v2 model on the device: ``n_chains`` persistent Gibbs chains
    (PottsSampler) estimate the model's one- and two-site marginals, and each update moves h and J by
    -learning_rate times the gradient of the regularised full-likelihood objective, so that those marginals approach
    the model's stored f_i, f_ij (include/evcplm.h has the objective and the update).  ``burn_in`` sweeps run once,
    before the first update.  The result depends only on the model, seed, n_chains, sweeps, burn_in, learning_rate
    and the number of updates run, not on how the updates are split over run() calls.

    With an engine whose collective has several ranks, rank r runs chains [lo, hi) (chain_range) and counts them;
    the int32 counts are summed over the ranks, which is exact, and every rank then takes the update with the global
    M.  Every rank so holds, after every update, the parameters one process computes, bit for bit."""

    def __init__(self, model, n_chains=10000, seed=0, learning_rate=0.05, burn_in=0, engine=None):
        import torch
        self.lam2_h, self.lam2_J = bm_regularisation(model)
        eta = float(learning_rate)
        if not math.isfinite(eta) or eta <= 0:
            raise ValueError("learning_rate must be finite and > 0, not %r" % learning_rate)
        if int(n_chains) < 1:
            raise ValueError("need at least one chain, not %r" % n_chains)
        if int(burn_in) < 0:
            raise ValueError("burn_in must be >= 0, not %r" % burn_in)
        self.source = model
        self.L, self.q = int(model["L"]), int(model["q"])
        self.n_chains, self.eta, self.burn_in = int(n_chains), eta, int(burn_in)
        self.updates = 0
        self.eng = _engine(engine)
        self.world, self.rank = _ranks(self.eng)
        self.lo, self.hi = (0, self.n_chains) if self.world == 1 else chain_range(self.n_chains, self.world,
                                                                                 self.rank)
        dev = self.eng.device
        Lq = self.L * self.q
        self.x = torch.from_numpy(model_x(model)).to(dev)
        self.f = torch.from_numpy(np.concatenate([np.asarray(model["fi"], dtype=np.float32).ravel(),
                                                  np.asarray(model["fij"], dtype=np.float32).ravel()])).to(dev)
        if self.f.numel() != self.x.numel() or self.x.numel() < Lq:
            raise ValueError("f_i, f_ij and h, J of the model have different sizes")
        self.counts = torch.empty(self.x.numel(), dtype=torch.int32, device=dev)
        self.codes = torch.empty((self.hi - self.lo, self.L), dtype=torch.uint8, device=dev)
        self.stats = torch.zeros(2, dtype=torch.float64, device=dev)
        self.sampler = PottsSampler(model, self.hi - self.lo, seed=seed, chain_offset=self.lo, engine=self.eng)

    def _counts(self):
        _lib.check(self.eng.lib.evc_sampler_codes(self.sampler.handle, self.eng.ptr(self.codes), self.eng.stream()),
                   "evc_sampler_codes")
        _lib.check(self.eng.lib.evc_code_counts(self.eng.ptr(self.codes), self.hi - self.lo, self.L, self.q,
                                                self.eng.ptr(self.counts), self.eng.stream()), "evc_code_counts")
        self.eng.kernel_launches += 1
        if self.world > 1:
            self.eng.all_reduce(self.counts)        # integers: exact, in any order

    def _changes(self, changes):
        """The site changes of every rank's chains, summed in int64."""
        if self.world == 1:
            return changes
        import torch
        t = torch.tensor([changes], dtype=torch.int64, device=self.eng.device)
        self.eng.all_reduce(t)
        return int(t.item())

    def _connected_pearson(self):
        """Pearson r of C_ij(a, b) = f_ij - f_i f_j of the chains (from the current counts) against the targets,
        in float64 on the device (reporting only)."""
        import torch
        Lq, q = self.L * self.q, self.q
        iu, ju = np.triu_indices(self.L, 1)
        iu, ju = torch.from_numpy(iu).to(self.x.device), torch.from_numpy(ju).to(self.x.device)

        def connected(v):
            fi, fij = v[:Lq].view(self.L, q), v[Lq:].view(-1, q, q)
            return (fij - fi[iu][:, :, None] * fi[ju][:, None, :]).ravel()

        a = connected(self.counts.to(torch.float64) / self.n_chains)
        b = connected(self.f.to(torch.float64))
        return float(torch.corrcoef(torch.stack([a, b]))[0, 1])

    def run(self, updates, sweeps=10, progress=None):
        """Runs ``updates`` updates of ``sweeps`` sweeps each.  ``progress(update, stats)`` (optional) is called after
        each update with update = its global index (0-based) and stats = dict(max_field_dev, max_coupling_dev,
        changes, connected_pearson): max |c/M - f| over the fields and over the couplings, the site changes of its
        sweeps and the Pearson r of the chains' connected correlations against the targets, all measured on the
        chains before the update's step."""
        if int(updates) < 0 or int(sweeps) < 0:
            raise ValueError("updates and sweeps must be >= 0")
        if self.updates == 0 and self.burn_in and int(updates) > 0:
            self.sampler.run(self.burn_in)
        for _ in range(int(updates)):
            changes = self.sampler.run(int(sweeps)) if progress is not None else self._sweep(int(sweeps))
            self._counts()
            if progress is not None:
                changes = self._changes(changes)
            pearson = self._connected_pearson() if progress is not None else None
            _lib.check(self.eng.lib.evc_bm_update(self.eng.ptr(self.x), self.eng.ptr(self.counts), self.n_chains,
                                                  self.eng.ptr(self.f), self.x.numel(), self.L * self.q, self.eta,
                                                  self.lam2_h, self.lam2_J, self.eng.ptr(self.stats),
                                                  self.eng.stream()), "evc_bm_update")
            _lib.check(self.eng.lib.evc_sampler_set_model(self.sampler.handle, self.eng.ptr(self.x),
                                                          self.eng.stream()), "evc_sampler_set_model")
            self.eng.kernel_launches += 3
            if progress is not None:
                st = self.stats.cpu().numpy()
                progress(self.updates, dict(max_field_dev=float(st[0]), max_coupling_dev=float(st[1]),
                                            changes=changes, connected_pearson=pearson))
            self.updates += 1
        return self

    def _sweep(self, sweeps):
        """Sweeps without waiting for the change count (evc_sampler_run with no host output)."""
        _lib.check(self.eng.lib.evc_sampler_run(self.sampler.handle, sweeps, 1.0, None, self.eng.stream()),
                   "evc_sampler_run")
        self.eng.kernel_launches += 1
        return None

    def parameters(self):
        """(h (L, q), J (npairs, q, q)) float32 numpy arrays of the current model."""
        x = self.x.cpu().numpy()
        Lq = self.L * self.q
        return x[:Lq].reshape(self.L, self.q), x[Lq:].reshape(-1, self.q, self.q)

    def fn_scores(self):
        """Raw-gauge Frobenius norms of the current J blocks (evc_fn_scores, pair order i < j), as run_plmc writes
        them into _ECs.txt."""
        import torch
        L, q = self.L, self.q
        out = torch.zeros(L * (L - 1) // 2, dtype=torch.float32, device=self.x.device)
        _lib.check(self.eng.lib.evc_fn_scores(self.eng.ptr(self.x[L * q:]), L, q, self.eng.ptr(out),
                                              self.eng.stream()), "evc_fn_scores")
        self.eng.kernel_launches += 1
        return out.cpu().numpy()

    def model(self):
        """A read_model-shaped dict: the input's header, weights, f_i and f_ij, the refined h and J, and num_iter =
        the number of updates run."""
        out = dict(self.source)
        out["h"], out["J"] = self.parameters()
        out["num_iter"] = self.updates
        return out

    def close(self):
        if getattr(self, "sampler", None) is not None:
            self.sampler.close()
            self.sampler = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def boltzmann_refine(model, updates, n_chains=10000, sweeps=10, seed=0, learning_rate=0.05, burn_in=0,
                     progress=None, engine=None, num_gpus=1, backend="nccl"):
    """The model refined by ``updates`` Boltzmann-machine updates (BoltzmannLearner), as a read_model-shaped dict.
    ``num_gpus`` > 1 runs the chains on that many ranks (evcouplings_b200.launcher) for the same result; ``progress``
    is then called with rank 0's rows, in order, once the ranks have finished."""
    if int(updates) < 0 or int(sweeps) < 0:
        raise ValueError("updates and sweeps must be >= 0")
    if check_num_gpus(num_gpus, n_chains, backend) > 1:
        out = _on_ranks("bmdca", num_gpus, backend, dict(
            model=model, updates=updates, n_chains=n_chains, sweeps=sweeps, seed=seed, learning_rate=learning_rate,
            burn_in=burn_in, progress=progress is not None))
        if progress is not None:
            for k, stats in out["rows"]:
                progress(k, stats)
        return out["model"]
    with BoltzmannLearner(model, n_chains, seed=seed, learning_rate=learning_rate, burn_in=burn_in,
                          engine=engine) as learner:
        learner.run(updates, sweeps, progress)
        return learner.model()


def fn_scores(model, engine=None):
    """Raw-gauge Frobenius norms of a model's J blocks (evc_fn_scores, pair order i < j), as run_plmc writes them
    into _ECs.txt; the numbers BoltzmannLearner.fn_scores gives for the same parameters."""
    import torch
    eng = _engine(engine)
    L, q = int(model["L"]), int(model["q"])
    J = torch.from_numpy(np.ascontiguousarray(model["J"], dtype=np.float32).ravel()).to(eng.device)
    out = torch.zeros(L * (L - 1) // 2, dtype=torch.float32, device=eng.device)
    _lib.check(eng.lib.evc_fn_scores(eng.ptr(J), L, q, eng.ptr(out), eng.stream()), "evc_fn_scores")
    eng.kernel_launches += 1
    return out.cpu().numpy()


def run_job(job, engine, **kwargs):
    """One rank's part of a ``job`` ("sample", "bmdca", "logz" or "design") started by evcouplings_b200.launcher: the same
    call as one process, sharded over the ranks of ``engine``; returns what the caller of the launcher receives."""
    if job == "sample":
        return sample_codes(engine=engine, **kwargs)
    if job == "logz":
        return log_partition(engine=engine, **kwargs)
    if job == "design":
        return design_codes(engine=engine, **kwargs)
    if job == "bmdca":
        rows = []
        collect = (lambda k, stats: rows.append((k, stats))) if kwargs.pop("progress") else None
        return dict(model=boltzmann_refine(progress=collect, engine=engine, **kwargs), rows=rows)
    raise ValueError("unknown job %r" % job)
