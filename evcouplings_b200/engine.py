"""
CUDA engine: device memory / streams / collectives (torch) around the C ABI of
libevcplm.so.  This is the only execution path of the package -- there is no
CPU implementation behind it; construction raises EngineUnavailableError when
the library or a CUDA device is missing.

Multi-GPU (one process per GPU, torch.distributed / NCCL): sequences are
sharded in contiguous blocks over ranks, parameters are replicated, and every
objective evaluation does ONE all-reduce of the gradient (+ one 8-byte
all-reduce of -loglk); the regulariser and the whole L-BFGS update then run
identically (bit-for-bit, deterministic reductions) on every rank.  The Hamming
pass shards the upper-triangular pair tiles and all-reduces the int32 counters.
"""
import ctypes
import os
import time

import numpy as np

from . import _lib
from . import lbfgs as _lbfgs


# backward implementation of the data term: "gather" (shared-memory bucket kernel) or "tc" (wgmma GEMM)
DEFAULT_BACKWARD = "tc"
DEFAULT_FORWARD = "tc"
# arithmetic of the tensor-core products: "fp32" (bf16 hi+lo pairs, fp32-equivalent; default), "bf16" (one bf16
# product, BASELINE configs[4] "bf16 tiles / fp32 parameters"), "auto" (fit only: bf16 until close to convergence,
# then fp32 to the end)
DEFAULT_PRECISION = "fp32"
PRECISIONS = ("fp32", "bf16", "auto")

# Sequence chunks of the tensor-core path (evc_plm_set_seq_chunk): chunk sizes are multiples of 768 sequences.
SEQ_CHUNK_ALIGN = 768
# Kept free beyond what the planner counts: torch's allocator rounding, the small scratch buffers of the library
# and of the host code, the tensor maps' and events' driver memory.
SEQ_CHUNK_MARGIN_BYTES = 512 << 20
# Host memory left to the system and to the other processes beyond the pinned correction pairs
# (evc_plm_set_host_history), subtracted from MemAvailable before it is shared by the ranks of the node.
HOST_HISTORY_MARGIN_BYTES = 4 << 30
# Host bytes per parameter that a fit through this package keeps while the pairs are pinned, counted against the
# same budget: run_plmc's float64 pair counts (8) and frequencies (8), the float32 start point (4) and result (4).
HOST_FIT_BYTES_PER_PARAM = 24


class DeviceMemoryError(RuntimeError):
    """The problem does not fit the device memory even with the smallest sequence chunk."""


class HostMemoryError(DeviceMemoryError):
    """The correction pairs that would make the problem fit the device do not fit the host memory budget."""


def num_params(L, q):
    return L * q + L * (L - 1) // 2 * q * q


def tc_bytes(N, L, q, gap_code, seq_chunk, sm_count):
    """Device bytes of a handle on the default tensor-core path (evc_plm_tc_bytes; host only, no device)."""
    lib = _lib.load()
    out = ctypes.c_int64()
    _lib.check(lib.evc_plm_tc_bytes(int(N), int(L), int(q), int(gap_code), int(seq_chunk), int(sm_count),
                                    ctypes.byref(out)), "evc_plm_tc_bytes")
    return int(out.value)


def alphabet_tc_bytes(N, L, q, gap_code, seq_chunk, sm_count):
    """tc_bytes for any supported alphabet, 2 <= q <= 32 (q <= 31 with the ignored gap): the handles of this package
    (evc_plm_create_alphabet; evc_plm_tc_bytes_alphabet, host only).  Equal to tc_bytes where both apply."""
    lib = _lib.load()
    out = ctypes.c_int64()
    _lib.check(lib.evc_plm_tc_bytes_alphabet(int(N), int(L), int(q), int(gap_code), int(seq_chunk), int(sm_count),
                                             ctypes.byref(out)), "evc_plm_tc_bytes_alphabet")
    return int(out.value)


def seq_chunk_reserve_bytes(L, q, m):
    """Device bytes a fit holds at its peak besides the handle: the evc_plm_fit workspace ((5 + 2m) vectors of n
    floats plus scalars), the problem's x and g_packed, the weighted-counts buffer, and a fixed margin."""
    n = num_params(L, q)
    fit = int(_lib.load().evc_fit_workspace_bytes(n, int(m)))
    own = 4 * n + 4 * (n + 4) + 4 * n + 2 * 8 + 8          # x, g_packed, weighted counts, fxbuf, dotbuf
    return fit + own + SEQ_CHUNK_MARGIN_BYTES


def plan_seq_chunk(N, L, q, gap_code, m, sm_count, free_bytes):
    """Sequences per chunk for a shard of N sequences given ``free_bytes`` of device memory: 0 (the whole shard,
    unchunked) when everything fits, else the largest multiple of SEQ_CHUNK_ALIGN that fits.  Raises
    DeviceMemoryError, naming the required and the available bytes, when even one chunk of SEQ_CHUNK_ALIGN
    sequences does not fit."""
    return _plan_chunk(N, L, q, gap_code, sm_count, free_bytes, seq_chunk_reserve_bytes(L, q, m))


def fit_workspace_bytes(n, m, host_pairs):
    """(device, pinned host) bytes of the evc_plm_fit workspace with ``host_pairs`` of its m correction pairs in
    host memory (evc_fit_workspace_split_bytes; host only)."""
    dev, host = ctypes.c_int64(), ctypes.c_int64()
    _lib.check(_lib.load().evc_fit_workspace_split_bytes(int(n), int(m), int(host_pairs), ctypes.byref(dev),
                                                         ctypes.byref(host)), "evc_fit_workspace_split_bytes")
    return int(dev.value), int(host.value)


def host_history_budget_bytes(ranks_on_node=1, meminfo="/proc/meminfo"):
    """Pinned host bytes one rank may use for its correction pairs: MemAvailable minus HOST_HISTORY_MARGIN_BYTES,
    shared equally by the ranks on this node (each rank pins its own history)."""
    avail = 0
    with open(meminfo) as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                avail = int(line.split()[1]) * 1024
                break
    return max(0, avail - HOST_HISTORY_MARGIN_BYTES) // max(1, int(ranks_on_node))


def plan_fit_memory(N, L, q, gap_code, m, sm_count, free_bytes, host_free_bytes, host_pairs=None):
    """(seq_chunk, host_pairs) for a fit of a shard of N sequences given ``free_bytes`` of device memory and
    ``host_free_bytes`` of host memory this rank may pin.  When plan_seq_chunk finds a plan, that plan with every
    correction pair on the device.  Otherwise the fewest pairs k (1 <= k <= m) whose move to pinned host memory lets
    one SEQ_CHUNK_ALIGN chunk fit, and the sequence chunk planned again with that smaller device reserve.
    With k > 0 the host needs the pinned pairs plus HOST_FIT_BYTES_PER_PARAM bytes per parameter for the fit's own
    host arrays.  ``host_pairs`` forces k (EVC_HOST_HISTORY).  Raises DeviceMemoryError naming the device and host
    bytes required and available when no k fits (HostMemoryError when the device would fit but the host memory does
    not)."""
    n = num_params(L, q)
    base = seq_chunk_reserve_bytes(L, q, m) - fit_workspace_bytes(n, m, 0)[0]
    if host_pairs is None:
        try:
            return plan_seq_chunk(N, L, q, gap_code, m, sm_count, free_bytes), 0
        except DeviceMemoryError:
            pass
        candidates = range(1, int(m) + 1)
    else:
        if not 0 <= int(host_pairs) <= int(m):
            raise ValueError("host_pairs must be in 0..m (m = %d)" % m)
        candidates = (int(host_pairs),)
    smallest = alphabet_tc_bytes(N, L, q, gap_code, SEQ_CHUNK_ALIGN, sm_count)
    for k in candidates:
        dev, host = fit_workspace_bytes(n, m, k)
        host_need = host + (HOST_FIT_BYTES_PER_PARAM * n if k else 0)
        need = smallest + base + dev
        if need > free_bytes and k != candidates[-1]:
            continue
        if need > free_bytes or host_need > host_free_bytes:
            cls = DeviceMemoryError if need > free_bytes else HostMemoryError
            raise cls(
                "the PLM fit (N=%d sequences, L=%d, q=%d, history m=%d) needs %d bytes of device memory with the "
                "smallest sequence chunk (%d sequences) and %d of the %d correction pairs in host memory; %d bytes "
                "are available.  Those pairs need %d bytes of pinned host memory, %d bytes of host memory with the "
                "fit's own host arrays; %d bytes are available"
                % (N, L, q, m, need, SEQ_CHUNK_ALIGN, k, m, free_bytes, host, host_need, host_free_bytes))
        return _plan_chunk(N, L, q, gap_code, sm_count, free_bytes, base + dev), k
    raise AssertionError("unreachable")


def _plan_chunk(N, L, q, gap_code, sm_count, free_bytes, reserve):
    if alphabet_tc_bytes(N, L, q, gap_code, 0, sm_count) + reserve <= free_bytes:
        return 0
    need = alphabet_tc_bytes(N, L, q, gap_code, SEQ_CHUNK_ALIGN, sm_count) + reserve
    k_max = (int(N) - 1) // SEQ_CHUNK_ALIGN          # chunks strictly smaller than the shard
    if k_max < 1 or need > free_bytes:
        raise DeviceMemoryError(
            "the PLM problem (N=%d sequences, L=%d, q=%d) needs %d bytes of device memory even with the smallest "
            "sequence chunk (%d sequences); %d bytes are available" % (N, L, q, need, SEQ_CHUNK_ALIGN, free_bytes))
    lo, hi = 1, k_max                                # the byte count is monotone in the chunk size
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if alphabet_tc_bytes(N, L, q, gap_code, mid * SEQ_CHUNK_ALIGN, sm_count) + reserve <= free_bytes:
            lo = mid
        else:
            hi = mid - 1
    return lo * SEQ_CHUNK_ALIGN


def seq_chunk_count(N, seq_chunk):
    """Chunks an evaluation of N sequences runs in (1 when unchunked)."""
    if not seq_chunk:
        return 1
    c = -(-int(seq_chunk) // SEQ_CHUNK_ALIGN) * SEQ_CHUNK_ALIGN
    return 1 if c >= N else -(-int(N) // c)


def _torch():
    import torch
    return torch


from .dist import Collective, shard_bounds   # noqa: E402,F401


class CudaEngine(object):
    def __init__(self, device=None, group=None, standalone=False):
        """``standalone=True``: ignore an initialised torch.distributed group (this process works alone on its
        GPU, e.g. rank 0 checking a sharded result against a single-GPU evaluation)."""
        self.lib = _lib.load()
        _lib.require_device()
        torch = _torch()
        if not torch.cuda.is_available():
            raise _lib.EngineUnavailableError("torch sees no CUDA device; the PLM engine has no CPU fallback")
        self.coll = Collective(group, standalone=standalone)
        self.rank, self.world = self.coll.rank, self.coll.world
        if device is None:
            device = torch.cuda.current_device()
        self.device_index = int(device)
        self.device = torch.device("cuda", self.device_index)
        torch.cuda.set_device(self.device)
        self.kernel_launches = 0

    # -- helpers ---------------------------------------------------------------------------
    def stream(self):
        return ctypes.c_void_p(_torch().cuda.current_stream(self.device).cuda_stream)

    def all_reduce(self, tensor):
        self.coll.all_reduce_sum(tensor)

    def all_gather(self, tensor):
        return self.coll.all_gather(tensor)

    def agree_any(self, flag):
        """True on every rank if ``flag`` is true on any rank (doubles as the barrier after rank 0 wrote files)."""
        if self.world == 1:
            return bool(flag)
        t = _torch().tensor([1 if flag else 0], dtype=_torch().int32, device=self.device)
        self.coll.all_reduce_max(t)
        return bool(int(t.item()))

    @staticmethod
    def ptr(t):
        return ctypes.c_void_p(t.data_ptr())

    # -- (b) Hamming reweighting -----------------------------------------------------------
    def hamming_counts(self, codes, min_identical, mult=None):
        """codes: (N, L) uint8 numpy (replicated on every rank).  Returns int32 numpy counts.  ``mult``: int
        multiplicities of the rows when they are distinct rows (unique_rows); a neighbour then counts its
        multiplicity instead of 1, which gives each distinct row the count of every one of its copies."""
        torch = _torch()
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        N, L = codes.shape
        if int(codes.max(initial=0)) >= 32:
            raise ValueError("sequence codes must be < 32")
        d_mult = None
        if mult is not None:
            mult = np.ascontiguousarray(mult, dtype=np.int64)
            if mult.shape != (N,) or (N and int(mult.min()) < 1) or int(mult.sum()) >= 2 ** 31:
                raise ValueError("mult must hold one multiplicity >= 1 per row, summing to less than 2^31")
            d_mult = torch.from_numpy(mult.astype(np.int32)).to(self.device)
        d_codes = torch.from_numpy(codes).to(self.device)
        d_counts = self.hamming_counts_device(d_codes, N, L, min_identical, d_mult)
        return d_counts.cpu().numpy()

    def hamming_counts_device(self, d_codes, N, L, min_identical, d_mult=None):
        torch = _torch()
        lib = self.lib
        words = lib.evc_hamming_plane_words(N, L)
        d_planes = torch.empty(words, dtype=torch.int32, device=self.device)
        d_counts = torch.zeros(N, dtype=torch.int32, device=self.device)
        _lib.check(lib.evc_hamming_pack(self.ptr(d_codes), N, L, self.ptr(d_planes), self.stream()),
                   "evc_hamming_pack")
        ntiles = lib.evc_hamming_num_tiles(N)
        lo, hi = shard_bounds(ntiles, self.world, self.rank)
        if d_mult is None:
            _lib.check(lib.evc_hamming_count_tiles(self.ptr(d_planes), N, L, int(min_identical), lo, hi,
                                                   self.ptr(d_counts), self.stream()), "evc_hamming_count_tiles")
        else:
            _lib.check(lib.evc_hamming_count_tiles_mult(self.ptr(d_planes), self.ptr(d_mult), N, L,
                                                        int(min_identical), lo, hi, self.ptr(d_counts),
                                                        self.stream()), "evc_hamming_count_tiles_mult")
        self.kernel_launches += 2
        self.all_reduce(d_counts)
        return d_counts

    def unique_rows(self, codes):
        """Distinct rows of codes: (N, L) uint8 numpy (evc_msa_unique).  Returns (first, inverse, mult): int64
        numpy arrays with first[U] the first row of each distinct row in ascending order, inverse[N] each row's
        distinct index and mult[U] the multiplicities.  Deterministic, so every rank derives the same table from its
        replicated codes without a collective."""
        torch = _torch()
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        N, L = codes.shape
        d_codes = torch.from_numpy(codes).to(self.device)
        d_out = torch.empty((3, N), dtype=torch.int32, device=self.device)
        U = ctypes.c_int64()
        _lib.check(self.lib.evc_msa_unique(self.ptr(d_codes), N, L, self.ptr(d_out[0]), self.ptr(d_out[1]),
                                           self.ptr(d_out[2]), ctypes.byref(U), self.stream()), "evc_msa_unique")
        self.kernel_launches += 7
        U = int(U.value)
        out = d_out.cpu().numpy().astype(np.int64)
        return out[0, :U].copy(), out[1].copy(), out[2, :U].copy()

    # -- (a) PLM ---------------------------------------------------------------------------
    def plm_problem(self, codes, weights, q, gap_code, lambda_h, lambda_J, m=6, backward=None, forward=None,
                    precision=None, seq_chunk=None, data_digest=False):
        return CudaPlmProblem(self, codes, weights, q, gap_code, lambda_h, lambda_J, m, backward, forward, precision,
                              seq_chunk, data_digest)

    def sm_count(self):
        sm = ctypes.c_int32()
        _lib.check(self.lib.evc_device_info(self.device_index, ctypes.byref(sm), None, None, None), "evc_device_info")
        return int(sm.value)


class _DevicePointer(object):
    """Zero-copy torch view of library-owned device memory (CUDA array interface)."""

    def __init__(self, ptr, count):
        self.__cuda_array_interface__ = {"shape": (int(count),), "typestr": "<f4", "data": (int(ptr), False),
                                         "version": 2}


class CudaPlmProblem(object):
    """PLM objective on this rank's sequence shard + the L-BFGS vector space
    (see lbfgs.py for the protocol).  All n-vectors are torch CUDA tensors."""

    def __init__(self, engine, codes, weights, q, gap_code, lambda_h, lambda_J, m=6, backward=None,
                 forward=None, precision=None, seq_chunk=None, data_digest=False):
        """``seq_chunk``: sequences per chunk of the tensor-core path (evc_plm_set_seq_chunk; 0 = whole shard).
        None = EVC_SEQ_CHUNK if set, else planned from the free device memory and this rank's share of the host
        memory (plan_fit_memory): the shard is streamed through chunk-sized buffers only when it does not fit
        whole, and correction pairs of the fit move to pinned host memory (``host_pairs``) only when even one
        chunk does not fit with all of them on the device.  EVC_HOST_HISTORY=k forces k host pairs, a knob for tests
        and sweeps: the host budget is checked only when the planner runs (seq_chunk None and no EVC_SEQ_CHUNK);
        with an explicit chunk, k is used as given.  The gather forward is never chunked.  The Python L-BFGS driver
        keeps its whole history on the device, so ``fit(driver="python")`` refuses a problem with host pairs.
        ``data_digest``: True hashes the codes and weights now (checkpoint.data_digest), for the fingerprint of a
        checkpointed fit that is not given one (run_plmc gives one); a string is taken as that digest."""
        torch = _torch()
        if precision is None:
            precision = os.environ.get("EVC_PRECISION", DEFAULT_PRECISION)
        if precision not in PRECISIONS:
            raise ValueError("precision must be one of %s" % (PRECISIONS,))
        self.precision = precision
        if forward is None:
            forward = os.environ.get("EVC_FORWARD", DEFAULT_FORWARD)
        if forward not in ("gather", "tc", "tcfused"):
            raise ValueError("forward must be 'gather', 'tc' or 'tcfused'")
        if forward in ("tc", "tcfused"):
            backward = "tc"
        self.forward = forward
        if backward is None:
            backward = os.environ.get("EVC_BACKWARD", DEFAULT_BACKWARD)
        if backward not in ("gather", "tc"):
            raise ValueError("backward must be 'gather' or 'tc'")
        self.backward = backward
        self.engine = engine
        self.lib = engine.lib
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        weights = np.ascontiguousarray(weights, dtype=np.float32)
        N, L = codes.shape
        if weights.shape != (N,):
            raise ValueError("weights must have one entry per sequence")
        n_states = int(q) + (1 if int(gap_code) >= 0 else 0)
        if N and int(codes.max()) >= n_states:
            raise ValueError("sequence codes must be < %d (q%s)" % (n_states, " + ignored gap" if gap_code >= 0 else ""))
        self.N_total, self.L, self.q, self.gap_code = N, L, int(q), int(gap_code)
        self.lambda_h, self.lambda_J = float(lambda_h), float(lambda_J)
        lo, hi = shard_bounds(N, engine.world, engine.rank)
        if hi <= lo:
            raise ValueError("fewer sequences than ranks")
        self.shard = (lo, hi)
        env_pairs = os.environ.get("EVC_HOST_HISTORY")
        host_pairs = int(env_pairs) if env_pairs else None
        if forward == "gather":
            if seq_chunk:
                raise ValueError("sequence chunks need the tensor-core forward ('tc' or 'tcfused')")
            seq_chunk = 0
        elif seq_chunk is None:
            env = os.environ.get("EVC_SEQ_CHUNK")
            if env:
                seq_chunk = int(env)
            else:
                # the Hamming pass's cached blocks go back to the device before the free memory is read
                torch.cuda.empty_cache()
                free, _total = torch.cuda.mem_get_info(engine.device)
                ranks = int(os.environ.get("LOCAL_WORLD_SIZE", engine.world))
                seq_chunk, host_pairs = plan_fit_memory(hi - lo, L, self.q, self.gap_code, m, engine.sm_count(),
                                                        free, host_history_budget_bytes(ranks), host_pairs)
        self.host_pairs = int(host_pairs or 0)
        if not 0 <= self.host_pairs <= m:
            raise ValueError("EVC_HOST_HISTORY must be in 0..m (m = %d)" % m)
        seq_chunk = int(seq_chunk)
        if seq_chunk < 0:
            raise ValueError("seq_chunk must be >= 0 (0: whole shard)")
        self.n_chunks = seq_chunk_count(hi - lo, seq_chunk)
        self.seq_chunk = 0 if self.n_chunks == 1 else -(-seq_chunk // SEQ_CHUNK_ALIGN) * SEQ_CHUNK_ALIGN
        if data_digest is True:
            from .checkpoint import data_digest as _digest
            data_digest = _digest(codes, weights)
        self._data_digest = data_digest or None
        c_shard = np.ascontiguousarray(codes[lo:hi])
        w_shard = np.ascontiguousarray(weights[lo:hi])
        self.handle = ctypes.c_void_p()
        _lib.check(self.lib.evc_plm_create_alphabet(ctypes.byref(self.handle), c_shard.ctypes.data_as(ctypes.c_void_p),
                                                    hi - lo, L, self.q, self.gap_code,
                                                    w_shard.ctypes.data_as(ctypes.c_void_p), engine.device_index),
                   "evc_plm_create_alphabet")
        if self.seq_chunk:
            _lib.check(self.lib.evc_plm_set_seq_chunk(self.handle, self.seq_chunk), "evc_plm_set_seq_chunk")
        if self.host_pairs:
            _lib.check(self.lib.evc_plm_set_host_history(self.handle, self.host_pairs), "evc_plm_set_host_history")
        # the gather modes are the handle's default; selecting them explicitly refuses an alphabet they do not serve
        _lib.check(self.lib.evc_plm_set_backward(self.handle, 1 if backward == "tc" else 0), "evc_plm_set_backward")
        _lib.check(self.lib.evc_plm_set_forward(self.handle, {"gather": 0, "tc": 1, "tcfused": 2}[forward]),
                   "evc_plm_set_forward")
        if precision == "bf16":
            _lib.check(self.lib.evc_plm_set_precision(self.handle, 1), "evc_plm_set_precision")
        self.n = int(self.lib.evc_plm_num_params(self.handle))
        dev = engine.device
        self.m = m
        f32 = dict(dtype=torch.float32, device=dev)
        self.x = torch.zeros(self.n, **f32)
        # gradient + 4 trailing floats: -loglk rides behind g as exact fixed-point limbs => ONE all-reduce
        self.g_packed = torch.zeros(self.n + 4, **f32)
        self.g = self.g_packed[:self.n]
        self._python_space = False          # vectors of the Python L-BFGS driver are allocated on demand
        self.fxbuf = torch.zeros(2, dtype=torch.float64, device=dev)
        self.dotbuf = torch.zeros(1, dtype=torch.float64, device=dev)
        self.last_negloglk = float("nan")
        self.evaluations = 0
        # own kernels per evaluate(): expand, fwd, bwd, finalize pairs + fields, add_reg x2
        self.launches_per_eval = {"tc": 8, "tcfused": 7, "gather": 7}[forward]
        if self.n_chunks > 1:           # expand, 5 per chunk (one-hot X, Xt, logits, softmax, backward), 2 + 2
            self.launches_per_eval = 5 + 5 * self.n_chunks

    def device_bytes(self):
        """Device bytes the handle holds (evc_plm_device_bytes; with the fit workspace once a fit ran)."""
        return int(self.lib.evc_plm_device_bytes(self.handle))

    def host_bytes(self):
        """(pinned host bytes, seconds their allocation took) of the host-resident correction pairs
        (evc_plm_host_bytes; (0, 0.0) before the first fit or with every pair on the device)."""
        b, s = ctypes.c_int64(), ctypes.c_double()
        _lib.check(self.lib.evc_plm_host_bytes(self.handle, ctypes.byref(b), ctypes.byref(s)), "evc_plm_host_bytes")
        return int(b.value), float(s.value)

    def close(self):
        if self.handle:
            self.lib.evc_plm_destroy(self.handle)
            self.handle = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- objective ----------------------------------------------------------------------------
    def evaluate_async(self, x):
        """Launch data term + all-reduce + regulariser on the current stream; results in self.g / self.fxbuf."""
        e, p = self.engine, self.engine.ptr
        _lib.check(self.lib.evc_plm_eval_data(self.handle, p(x), p(self.g), p(self.fxbuf), e.stream()),
                   "evc_plm_eval_data")
        if e.world > 1:
            limbs = self.g_packed[self.n:]
            _lib.check(self.lib.evc_plm_pack_fx(p(self.fxbuf), p(limbs), e.stream()), "evc_plm_pack_fx")
            timed = getattr(self, "time_collective", False)
            if timed:
                torch = _torch()
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                ev[0].record()
            e.all_reduce(self.g_packed)                     # ONE collective: [g, -loglk]
            if timed:
                ev[1].record()
                self.collective_events.append(ev)
            _lib.check(self.lib.evc_plm_unpack_fx(p(limbs), p(self.fxbuf), e.stream()), "evc_plm_unpack_fx")
            e.kernel_launches += 2
        _lib.check(self.lib.evc_plm_add_regulariser(self.handle, p(x), p(self.g), p(self.fxbuf),
                                                    self.lambda_h, self.lambda_J, e.stream()),
                   "evc_plm_add_regulariser")
        self.evaluations += 1
        e.kernel_launches += self.launches_per_eval

    def evaluate(self, x):
        self.evaluate_async(x)
        nll, fx = self.fxbuf.tolist()
        self.last_negloglk = nll
        return fx

    def evaluate_host(self, x_host, g_host):
        """Public host-buffer entry: x_host / g_host are CPU float32 torch tensors (pinned for speed).
        H2D of x, evaluation (incl. the all-reduce), D2H of the gradient and of fx, then synchronise."""
        self.x.copy_(x_host, non_blocking=True)
        self.evaluate_async(self.x)
        g_host.copy_(self.g, non_blocking=True)
        nll, fx = self.fxbuf.tolist()          # D2H of the result scalars; synchronises the stream
        self.last_negloglk = nll
        return fx

    # -- vector space protocol (Python L-BFGS driver, kept for comparison / tests) -------------------
    def _ensure_python_space(self):
        if self._python_space:
            return
        torch = _torch()
        f32 = dict(dtype=torch.float32, device=self.engine.device)
        m = self.m
        self.xp = torch.zeros(self.n, **f32)
        self.gp = torch.zeros(self.n, **f32)
        self.d = torch.zeros(self.n, **f32)
        self.S = torch.zeros((m, self.n), **f32)
        self.Y = torch.zeros((m, self.n), **f32)
        self.ys = torch.zeros(m, dtype=torch.float64, device=self.engine.device)
        self.scratch = torch.zeros(m + 2, dtype=torch.float64, device=self.engine.device)
        self._python_space = True

    def get_history_scalars(self):
        ys = self.ys.tolist()
        return ys, float(self.scratch[0].item())

    def set_history_scalars(self, ys, yy):
        torch = _torch()
        self.ys.copy_(torch.tensor([float(v) for v in ys], dtype=torch.float64))
        self.scratch[0] = float(yy)

    def data_digest(self):
        """SHA-256 of all ranks' sequence codes and float32 weights (the checkpoint fingerprint), when the problem
        was created with ``data_digest``."""
        if self._data_digest is None:
            raise ValueError("a checkpointed fit needs the data digest of its fingerprint: create the problem with "
                             "data_digest=True, or pass checkpoint.CheckpointFile(path, extra={'data_sha256': ...})")
        return self._data_digest

    def dot(self, a, b):
        e = self.engine
        _lib.check(self.lib.evc_vec_dot(e.ptr(a), e.ptr(b), self.n, e.ptr(self.dotbuf), e.stream()), "evc_vec_dot")
        e.kernel_launches += 2
        return float(self.dotbuf.item())

    def copy(self, dst, src):
        e = self.engine
        _lib.check(self.lib.evc_vec_copy(e.ptr(dst), e.ptr(src), self.n, e.stream()), "evc_vec_copy")

    def axpby(self, y, x, a, b):
        e = self.engine
        _lib.check(self.lib.evc_vec_axpby(e.ptr(y), e.ptr(x), float(a), float(b), self.n, e.stream()),
                   "evc_vec_axpby")
        e.kernel_launches += 1

    def update_pair(self, slot, xp, gp):
        e, p = self.engine, self.engine.ptr
        _lib.check(self.lib.evc_lbfgs_update_pair(p(self.S[slot]), p(self.Y[slot]), p(self.x), p(xp), p(self.g),
                                                  p(gp), p(self.ys[slot:slot + 1]), p(self.scratch[0:1]),
                                                  self.n, e.stream()), "evc_lbfgs_update_pair")
        e.kernel_launches += 3

    def direction(self, d, bound, end):
        e, p = self.engine, self.engine.ptr
        _lib.check(self.lib.evc_lbfgs_direction(p(d), p(self.g), p(self.S), p(self.Y), p(self.ys), p(self.scratch),
                                                self.n, self.m, int(bound), int(end), e.stream()),
                   "evc_lbfgs_direction")
        e.kernel_launches += 1 + 4 * int(bound)

    # -- a6 / a10 ---------------------------------------------------------------------------------
    def weighted_counts(self):
        """Returns (fi_counts (L,q), fij_counts (npairs,q,q)) float64 numpy, summed over all ranks."""
        torch = _torch()
        e = self.engine
        L, q = self.L, self.q
        buf = torch.zeros(self.n, dtype=torch.float32, device=e.device)
        _lib.check(self.lib.evc_plm_weighted_counts(self.handle, e.ptr(buf), e.ptr(buf[L * q:]), e.stream()),
                   "evc_plm_weighted_counts")
        e.kernel_launches += 5
        e.all_reduce(buf)
        host = buf.cpu().numpy().astype(np.float64)
        return host[:L * q].reshape(L, q), host[L * q:].reshape(L * (L - 1) // 2, q, q)

    def fn_scores(self, x=None):
        torch = _torch()
        e = self.engine
        x = self.x if x is None else x
        L, q = self.L, self.q
        out = torch.zeros(L * (L - 1) // 2, dtype=torch.float32, device=e.device)
        _lib.check(self.lib.evc_fn_scores(e.ptr(x[L * q:]), L, q, e.ptr(out), e.stream()), "evc_fn_scores")
        e.kernel_launches += 1
        return out.cpu().numpy()

    def set_x(self, x_host):
        torch = _torch()
        self.x.copy_(torch.from_numpy(np.ascontiguousarray(x_host, dtype=np.float32)))

    def get_x(self):
        return self.x.cpu().numpy()

    def norms(self):
        """(|h|, |J|) of the current parameters (for the iteration table)."""
        import math
        cached = getattr(self, "_cached_norms", None)
        if cached is not None:                  # evc_plm_fit reports them with every iteration
            return cached
        e = self.engine
        nh = self.L * self.q
        out = []
        for lo, n in ((0, nh), (nh, self.n - nh)):
            v = self.x[lo:lo + n]
            _lib.check(self.lib.evc_vec_dot(e.ptr(v), e.ptr(v), n, e.ptr(self.dotbuf), e.stream()), "evc_vec_dot")
            e.kernel_launches += 2
            out.append(math.sqrt(float(self.dotbuf.item())))
        return out[0], out[1]

    def fit(self, x0, params, progress=None, driver="device", checkpoint=None, checkpoint_interval=900.0):
        """Minimise from x0.  driver "device": the whole L-BFGS loop runs inside libevcplm (evc_plm_fit);
        "python": the same algorithm with host-side control (lbfgs.py), kept for comparison.
        ``progress(k, fx, xnorm, gnorm, step, n_ls)``; returns lbfgs.LbfgsResult.  The Python driver allocates its
        whole history on the device: it raises DeviceMemoryError for a problem planned with host pairs.

        ``checkpoint``: a path or a checkpoint.CheckpointFile.  The fit's state is saved there every
        ``checkpoint_interval`` seconds (0: every iteration), when it is cancelled (progress, or
        checkpoint.request_stop) and when it returns; when the file already holds a state of this problem (same
        fingerprint, checkpoint.FINGERPRINT_KEYS) the fit continues from it and x0 is not used.  With several
        ranks, rank 0 writes and every rank reads the same file."""
        ck = None
        if checkpoint is not None:
            from .checkpoint import CheckpointFile
            ck = checkpoint if isinstance(checkpoint, CheckpointFile) else CheckpointFile(checkpoint,
                                                                                          checkpoint_interval)
        if driver == "python" and self.host_pairs:
            raise DeviceMemoryError(
                "this problem keeps %d of its %d correction pairs in host memory because the whole history does not "
                "fit the device; the Python L-BFGS driver keeps its history on the device: use driver='device'"
                % (self.host_pairs, self.m))
        self.set_x(x0)
        if driver == "python":
            self._ensure_python_space()
            self._cached_norms = None
            if ck is not None:
                from . import checkpoint as _ckpt
                return _ckpt.fit_python(self, params, progress, ck, _ckpt.fingerprint(self, params, ck.extra),
                                        engine=self.engine)
            return _lbfgs.minimize(self, params, progress)
        return self._fit_device(params, progress, ck)

    def _fit_device(self, params, progress, ck=None):
        e, lib = self.engine, self.lib
        torch = _torch()
        fp = _lib.FitParams()
        lib.evc_fit_default_params(ctypes.byref(fp))
        fp.max_iterations, fp.m, fp.epsilon = int(params.max_iterations), int(params.m), float(params.epsilon)
        fp.lambda_h, fp.lambda_J = self.lambda_h, self.lambda_J
        fp.max_linesearch = int(params.max_linesearch)
        fp.min_step, fp.max_step = float(params.min_step), float(params.max_step)
        fp.ftol, fp.gtol, fp.xtol = float(params.ftol), float(params.gtol), float(params.xtol)
        fp.precision_schedule = 1 if self.precision == "auto" else 0
        errors = []
        views = {}

        stats = {"allreduce_calls": 0, "allreduce_callback_s": 0.0}

        def allreduce(user, d_buf, count, stream):
            try:
                t_cb = time.perf_counter()
                key = (d_buf, count)
                if key not in views:
                    views[key] = torch.as_tensor(_DevicePointer(d_buf, count), device=e.device)
                e.all_reduce(views[key])
                stats["allreduce_calls"] += 1
                stats["allreduce_callback_s"] += time.perf_counter() - t_cb      # host time only (the collective is async)
                return 0
            except BaseException as exc:          # never let an exception cross the C boundary
                errors.append(exc)
                return 1

        def on_iteration(user, k, fx, xnorm, gnorm, step, n_ls, nll, hnorm, enorm):
            try:
                self.last_negloglk = nll
                self._cached_norms = (hnorm, enorm)
                if progress is not None and progress(k, fx, xnorm, gnorm, step, n_ls):
                    return 1
                return 0
            except BaseException as exc:
                errors.append(exc)
                return 1

        ar_cb = _lib.ALLREDUCE_CB(allreduce) if e.world > 1 else None
        res = _lib.FitResult()
        if ck is None:
            pr_cb = _lib.PROGRESS_CB(on_iteration)
            rc = lib.evc_plm_fit(self.handle, e.ptr(self.x), ctypes.byref(fp),
                                 ctypes.cast(ar_cb, ctypes.c_void_p) if ar_cb is not None else None, None,
                                 ctypes.cast(pr_cb, ctypes.c_void_p), None, ctypes.byref(res), e.stream())
        else:
            rc = self._fit_device_checkpointed(params, fp, ar_cb, on_iteration, res, errors, ck)
        self._cached_norms = None
        if errors:
            raise errors[0]
        if rc != 0:
            msg = (lib.evc_last_error() or b"").decode()
            if "workspace allocation failed" in msg:      # device or pinned host memory for the L-BFGS vectors
                raise DeviceMemoryError("evc_plm_fit failed: %s (%d of the %d correction pairs in host memory)"
                                        % (msg, self.host_pairs, self.m))
        _lib.check(rc, "evc_plm_fit")
        self.last_negloglk = res.negloglk
        self.evaluations += res.evaluations
        e.kernel_launches += res.evaluations * (self.launches_per_eval + 2)
        self.fit_seconds = res.seconds
        self.switched_at = res.switched_at
        host_b, pin_s = self.host_bytes()
        self.fit_stats = dict(stats, fit_s=res.seconds, evaluations=res.evaluations, iterations=res.iterations,
                              switched_at=res.switched_at, host_history_bytes=host_b, host_history_pin_s=pin_s)
        return _lbfgs.LbfgsResult(_lib.LBFGS_STATUS.get(res.status, "LBFGSERR_UNKNOWNERROR"), res.iterations,
                                  res.fx, res.evaluations)

    def _fit_device_checkpointed(self, params, fp, ar_cb, on_iteration, res, errors, ck):
        """evc_plm_fit_checkpointed with the file ``ck``: resume from it when it holds this problem's state, save
        into it at the boundaries the checkpoint.Gate agrees on.  The library is asked for every boundary
        (interval 0) so that all ranks reach the same callbacks; the gate decides which of them write."""
        from . import checkpoint as _ckpt
        e, lib = self.engine, self.lib
        fprint = _ckpt.fingerprint(self, params, ck.extra)
        header = ck.check(fprint, params.max_iterations)
        ck.check_space(self.n, params.m)
        ck.info.update(max_iterations=int(params.max_iterations), world=int(e.world), seq_chunk=int(self.seq_chunk),
                       host_pairs=int(self.host_pairs), device=_torch().cuda.get_device_name(e.device))
        staging = _ckpt._Staging(self.n)
        first_host = int(params.m) - int(self.host_pairs)

        def vector(name, slot):
            which = {"x": _lib.FIT_VEC_X, "g": _lib.FIT_VEC_G, "s": _lib.FIT_VEC_S, "y": _lib.FIT_VEC_Y}[name]
            ptr = ctypes.c_void_p()
            _lib.check(lib.evc_plm_fit_vector(self.handle, which, max(slot, 0), ctypes.byref(ptr)),
                       "evc_plm_fit_vector")
            return _ckpt.DeviceVector(e, ptr.value, self.n, host=slot >= first_host)

        resume = None
        if header is not None:
            _lib.check(lib.evc_plm_fit_prepare(self.handle, int(params.m)), "evc_plm_fit_prepare")
            ck.load_vectors(vector, staging)
            st = header["state"]
            resume = _lib.FitState()
            for name, _t in _lib.FitState._fields_:
                if name == "ys":
                    for j, v in enumerate(st["ys"]):
                        resume.ys[j] = v
                elif name == "version":
                    resume.version = _lib.FIT_STATE_VERSION
                elif name in st:
                    setattr(resume, name, st[name])
            resume.returning = resume.status = 0
        gate = _ckpt.Gate(e, ck.interval, header)

        def on_boundary(user, k, fx, xnorm, gnorm, step, n_ls, nll, hnorm, enorm):
            local = on_iteration(user, k, fx, xnorm, gnorm, step, n_ls, nll, hnorm, enorm)
            try:
                return 1 if gate.boundary(bool(local)) else 0
            except BaseException as exc:
                errors.append(exc)
                return 1

        def on_state(user, state_ptr, stream):
            try:
                s = state_ptr.contents
                reason = _lib.LBFGS_STATUS.get(s.status, "LBFGSERR_UNKNOWNERROR") if s.returning else None
                if not _ckpt.wants(reason, gate):
                    return 0
                st = {name: getattr(s, name) for name, _t in _lib.FitState._fields_ if name != "ys"}
                st["ys"] = [float(s.ys[j]) for j in range(s.m)]
                st["reason"] = reason
                names = _ckpt.state_vector_names(st)
                _ckpt.write_state(ck, gate, st, [(nm, sl, vector(nm, sl)) for nm, sl in names], fprint, staging)
                return 0
            except BaseException as exc:
                errors.append(exc)
                return 1

        pr_cb = _lib.PROGRESS_CB(on_boundary)
        ck_cb = _lib.CHECKPOINT_CB(on_state)
        return lib.evc_plm_fit_checkpointed(
            self.handle, e.ptr(self.x), ctypes.byref(fp), ctypes.cast(ar_cb, ctypes.c_void_p) if ar_cb is not None
            else None, None, ctypes.cast(pr_cb, ctypes.c_void_p), None, ctypes.cast(ck_cb, ctypes.c_void_p), None,
            0.0, ctypes.byref(resume) if resume is not None else None, ctypes.byref(res), e.stream())
