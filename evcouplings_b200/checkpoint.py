"""
Checkpoint files of the L-BFGS fit: the fit's state at an iteration boundary, so that an interrupted fit, or one
stopped at its iteration cap, continues with the same bits as a fit that never stopped.

File layout (little-endian):

    b"EVCPLMCK" | uint32 format version | uint32 header bytes | 32-byte SHA-256 of the header | header (JSON) |
    the vectors, raw, in the order the header lists them

The header holds the state scalars (evc_fit_state_t: k, evaluations, hist, end, ys, yy, fx, ...), the problem
fingerprint, a checksum per vector (evc_vec_checksum: a position-mixed sum of the 32-bit words modulo 2^64), the
iteration-table rows written so far, and what was recorded but not fingerprinted (iteration cap, ranks, sequence
chunk, host pairs, device).  The vectors are x and g of the accepted iterate, then S and Y of the ``hist`` stored
correction pairs, oldest first, each under its ring slot: (2 + 2 hist) n words in all.

A write goes to ``<path>.tmp``, is fsynced and renamed over ``<path>``: a kill during a write leaves the previous
checkpoint intact.  Device vectors stream through one bounded pinned staging buffer; host-resident correction pairs
(mapped pinned memory) are written from where they live.  No n-sized host buffer is allocated.
"""
import hashlib
import json
import os
import struct
import time

import numpy as np

from .tools import InvalidParameterError, ResourceError

MAGIC = b"EVCPLMCK"
FORMAT_VERSION = 1
STAGING_BYTES = 32 << 20            # pinned staging buffer of the device vectors
HEADER_RESERVE_BYTES = 1 << 20      # counted for the header in the disk-space check
_PRE = struct.Struct("<8sII32s")
_M64 = (1 << 64) - 1
_K0, _K1, _K2 = np.uint64(0x9E3779B97F4A7C15), np.uint64(0xBF58476D1CE4E5B9), np.uint64(0x94D049BB133111EB)
_CHUNK_WORDS = 1 << 22

# fingerprint keys, in the order a mismatch is reported
FINGERPRINT_KEYS = ("L", "q", "gap_code", "alphabet", "n", "data_sha256", "lambda_h", "lambda_J", "m", "epsilon",
                    "max_linesearch", "min_step", "max_step", "ftol", "gtol", "xtol", "precision")

_stop = {"requested": False}


class CheckpointError(ResourceError):
    """A checkpoint file is truncated or corrupt."""


def request_stop(*_args):
    """Ask a checkpointed fit to save its state and stop at the next iteration boundary (signal handlers).  One
    request stops one fit: the fit that honours it clears it, so a later fit in the same process runs normally."""
    _stop["requested"] = True


def stop_requested():
    return _stop["requested"]


def clear_stop():
    _stop["requested"] = False


def state_key(state):
    """What identifies a state among those of one fit (a resumed state, or the interval and the return at one
    boundary, are the same state)."""
    return tuple(int(state[k]) for k in ("k", "evaluations", "hist", "end", "switched_at"))


def checksum_words(words, offset=0):
    """numpy model of evc_vec_checksum over uint32 words whose first index is ``offset``."""
    words = np.asarray(words, dtype=np.uint32).ravel()
    total = 0
    with np.errstate(over="ignore"):
        for lo in range(0, len(words), _CHUNK_WORDS):
            w = words[lo:lo + _CHUNK_WORDS].astype(np.uint64)
            z = (np.arange(offset + lo + 1, offset + lo + 1 + len(w), dtype=np.uint64) * _K0) ^ w
            z = (z ^ (z >> np.uint64(30))) * _K1
            z = (z ^ (z >> np.uint64(27))) * _K2
            z ^= z >> np.uint64(31)
            total = (total + int(z.sum(dtype=np.uint64))) & _M64
    return total


def data_digest(codes, weights):
    """SHA-256 of the valid sequence codes (uint8, N x L) and their float32 weights, in order."""
    h = hashlib.sha256()
    h.update(np.ascontiguousarray(codes, dtype=np.uint8).tobytes())
    h.update(np.ascontiguousarray(weights, dtype=np.float32).tobytes())
    return h.hexdigest()


def fingerprint(problem, params, extra=None):
    """What must match to resume: the problem (L, q, gap code, n, data digest, lambdas, precision), the L-BFGS
    parameters except the iteration cap, and ``extra`` (run_plmc adds the alphabet and the data digest it already
    computed)."""
    extra = dict(extra or {})
    digest = extra.pop("data_sha256", None) or problem.data_digest()
    fp = dict(L=int(problem.L), q=int(problem.q), gap_code=int(problem.gap_code), alphabet=None, n=int(problem.n),
              data_sha256=digest, lambda_h=float(problem.lambda_h),
              lambda_J=float(problem.lambda_J), m=int(params.m), epsilon=float(params.epsilon),
              max_linesearch=int(params.max_linesearch), min_step=float(params.min_step),
              max_step=float(params.max_step), ftol=float(params.ftol), gtol=float(params.gtol),
              xtol=float(params.xtol), precision=str(getattr(problem, "precision", None)))
    fp.update(extra)
    return fp


# ---- vectors ----------------------------------------------------------------------------------------------------
class HostVector(object):
    """A contiguous host array (numpy), e.g. the vectors of the oracle problem or mapped pinned host memory."""

    def __init__(self, arr):
        self.arr = arr
        self.nbytes = arr.nbytes
        self.dtype = str(arr.dtype)

    def checksum(self):
        return checksum_words(self.arr.view(np.uint32))

    def write(self, f, staging):
        mv = memoryview(self.arr).cast("B")
        for lo in range(0, self.nbytes, STAGING_BYTES):
            f.write(mv[lo:lo + STAGING_BYTES])

    def read(self, f, staging):
        mv = memoryview(self.arr).cast("B")
        got = 0
        while got < self.nbytes:
            r = f.readinto(mv[got:got + STAGING_BYTES])
            if not r:
                return False
            got += r
        return True


class DeviceVector(object):
    """n float32 on the device at ``ptr`` (or the device address of mapped pinned host memory: ``host=True``)."""

    def __init__(self, engine, ptr, n, host=False):
        self.engine, self.ptr, self.n, self.host = engine, int(ptr), int(n), host
        self.nbytes = 4 * self.n
        self.dtype = "float32"

    def _host_view(self):
        import ctypes
        return np.ctypeslib.as_array((ctypes.c_float * self.n).from_address(self.ptr))

    def _tensor(self):
        import torch
        from .engine import _DevicePointer
        return torch.as_tensor(_DevicePointer(self.ptr, self.n), device=self.engine.device)

    def checksum(self):
        import torch
        from . import _lib
        e = self.engine
        out = torch.zeros(1, dtype=torch.int64, device=e.device)
        _lib.check(e.lib.evc_vec_checksum(self.ptr, self.n, e.ptr(out), e.stream()), "evc_vec_checksum")
        return int(out.item()) & _M64

    def write(self, f, staging):
        if self.host:
            torch_sync(self.engine)
            return HostVector(self._host_view()).write(f, staging)
        src = self._tensor()
        buf = staging.get(self.engine)
        step = buf.numel()
        for lo in range(0, self.n, step):
            c = min(step, self.n - lo)
            buf[:c].copy_(src[lo:lo + c])          # synchronous D2H into pinned memory
            f.write(memoryview(buf[:c].numpy()).cast("B"))

    def read(self, f, staging):
        if self.host:
            torch_sync(self.engine)
            return HostVector(self._host_view()).read(f, staging)
        dst = self._tensor()
        buf = staging.get(self.engine)
        step = buf.numel()
        for lo in range(0, self.n, step):
            c = min(step, self.n - lo)
            mv = memoryview(buf[:c].numpy()).cast("B")
            got = 0
            while got < 4 * c:
                r = f.readinto(mv[got:])
                if not r:
                    return False
                got += r
            dst[lo:lo + c].copy_(buf[:c])
        return True


def torch_sync(engine):
    import torch
    torch.cuda.current_stream(engine.device).synchronize()


class _Staging(object):
    """The pinned staging buffer, allocated on first use and kept for the fit."""

    def __init__(self, n):
        self.n = max(1, min(int(n), STAGING_BYTES // 4))
        self.buf = None

    def get(self, engine):
        if self.buf is None:
            import torch
            self.buf = torch.empty(self.n, dtype=torch.float32, pin_memory=True)
        return self.buf


def state_vector_names(state):
    """(name, ring slot) of the vectors a state stores, in file order."""
    m, hist, end = int(state["m"]), int(state["hist"]), int(state["end"])
    out = [("x", -1), ("g", -1)]
    for i in range(hist):
        slot = (end - hist + i) % m
        out += [("s", slot), ("y", slot)]
    return out


# ---- the file -----------------------------------------------------------------------------------------------------
class CheckpointFile(object):
    """One checkpoint path.  ``rows`` are the iteration-table rows stored with each state (run_plmc keeps them
    current); ``extra`` joins the fingerprint; ``info`` is recorded, and of it only ``unique_rows`` (the distinct
    sequences run_plmc fits, with ``valid_rows`` standing in for a file that does not record it) must match."""

    def __init__(self, path, interval=900.0, extra=None):
        self.path = os.path.abspath(str(path))
        self.tmp = self.path + ".tmp"
        self.interval = float(interval)
        self.extra = dict(extra or {})
        self.info = {}
        self.rows = []
        self.header = None
        self.stats = dict(resumes=0, writes=0, seconds=0.0, bytes=0)
        self.write_log = []     # per write: bytes, stored pairs, seconds in all, seconds of the checksums

    def exists(self):
        return os.path.isfile(self.path)

    def read_header(self):
        try:
            with open(self.path, "rb") as f:
                pre = f.read(_PRE.size)
                if len(pre) != _PRE.size:
                    raise CheckpointError("checkpoint %s is truncated in its header" % self.path)
                magic, version, hlen, digest = _PRE.unpack(pre)
                if magic != MAGIC:
                    raise CheckpointError("%s is not a fit checkpoint (bad magic)" % self.path)
                if version != FORMAT_VERSION:
                    raise CheckpointError("checkpoint %s has format version %d; this version reads %d"
                                          % (self.path, version, FORMAT_VERSION))
                raw = f.read(hlen)
        except OSError as e:
            raise CheckpointError("cannot read checkpoint %s: %s" % (self.path, e))
        if len(raw) != hlen:
            raise CheckpointError("checkpoint %s is truncated in its header" % self.path)
        if hashlib.sha256(raw).digest() != digest:
            raise CheckpointError("checkpoint %s: the header fails its checksum" % self.path)
        header = json.loads(raw.decode())
        header["_data_offset"] = _PRE.size + hlen
        return header

    def check(self, fp, max_iterations):
        """The stored header if this path holds a checkpoint of the same problem, None if there is none.  Raises
        InvalidParameterError naming the first field that differs, or when the state is past ``max_iterations``;
        the file is never touched."""
        if not self.exists():
            return None
        header = self.read_header()
        stored = header["fingerprint"]
        for key in FINGERPRINT_KEYS:
            if stored.get(key) != fp.get(key):
                raise InvalidParameterError(
                    "checkpoint %s belongs to another fit: %s is %r there and %r here (the file is left in place; "
                    "remove it or choose another checkpoint path to start a new fit)"
                    % (self.path, key, stored.get(key), fp.get(key)))
        if "unique_rows" in self.info:
            # the fit runs on the distinct rows: another row table sums the objective in another order, so its
            # iterates would not continue bit for bit.  A file without the field was fitted on every valid row.
            info = header.get("info", {})
            have = info.get("unique_rows", self.info.get("valid_rows"))
            if have != self.info["unique_rows"]:
                raise InvalidParameterError(
                    "checkpoint %s was fitted on %r distinct sequences, this fit has %r (the file is left in place; "
                    "remove it or choose another checkpoint path to start a new fit)"
                    % (self.path, have, self.info["unique_rows"]))
        k = int(header["state"]["k"])
        if max_iterations and k > int(max_iterations):
            raise InvalidParameterError(
                "checkpoint %s holds %d iterations, more than the requested cap of %d iterations"
                % (self.path, k, int(max_iterations)))
        self.header = header
        self.rows[:] = header.get("rows", [])
        return header

    def check_space(self, n, m, itemsize=4):
        """Raise ResourceError unless the file system holds a full-history checkpoint in the temp file next to
        the existing one (which stays until the rename)."""
        need = (2 + 2 * int(m)) * int(n) * int(itemsize) + HEADER_RESERVE_BYTES
        d = os.path.dirname(self.path)
        os.makedirs(d, exist_ok=True)
        st = os.statvfs(d)
        avail = st.f_bavail * st.f_frsize
        if need > avail:
            have = os.path.getsize(self.path) if self.exists() else 0
            raise ResourceError(
                "checkpoint %s needs %d bytes of disk for its temporary file (the existing checkpoint holds %d "
                "more until it is replaced); %d bytes are available" % (self.path, need, have, avail))
        return need

    def write(self, state, vectors, fp, staging):
        """Write ``state`` (dict) and ``vectors`` (list of (name, slot, HostVector | DeviceVector)) atomically."""
        t0 = time.perf_counter()
        entries = [dict(name=name, slot=slot, dtype=v.dtype, nbytes=v.nbytes, checksum=v.checksum())
                   for name, slot, v in vectors]
        t_sum = time.perf_counter() - t0
        header = dict(format=FORMAT_VERSION, state=state, fingerprint=fp, vectors=entries, rows=list(self.rows),
                      info=dict(self.info, resumes=self.stats["resumes"]), written=time.time())
        raw = json.dumps(header, sort_keys=True).encode()
        with open(self.tmp, "wb") as f:
            f.write(_PRE.pack(MAGIC, FORMAT_VERSION, len(raw), hashlib.sha256(raw).digest()))
            f.write(raw)
            for _name, _slot, v in vectors:
                v.write(f, staging)
            f.flush()
            os.fsync(f.fileno())
            size = f.tell()
        os.replace(self.tmp, self.path)
        try:
            dfd = os.open(os.path.dirname(self.path), os.O_RDONLY)
            try:
                os.fsync(dfd)
            finally:
                os.close(dfd)
        except OSError:
            pass
        dt = time.perf_counter() - t0
        self.stats["writes"] += 1
        self.stats["bytes"] = size
        self.stats["seconds"] += dt
        self.write_log.append(dict(bytes=size, hist=int(state["hist"]), seconds=dt, checksum_s=t_sum))

    def load_vectors(self, sink, staging):
        """Read the vectors of the checked header into ``sink(name, slot)`` -> HostVector | DeviceVector and verify
        each checksum; CheckpointError names the file and the vector on a short or corrupt file."""
        header = self.header
        with open(self.path, "rb") as f:
            f.seek(header["_data_offset"])
            for e in header["vectors"]:
                label = e["name"] if e["slot"] < 0 else "%s[%d]" % (e["name"], e["slot"])
                v = sink(e["name"], e["slot"])
                if v.nbytes != e["nbytes"] or v.dtype != e["dtype"]:
                    raise CheckpointError("checkpoint %s: vector %s holds %d bytes of %s, the fit needs %d of %s"
                                          % (self.path, label, e["nbytes"], e["dtype"], v.nbytes, v.dtype))
                if not v.read(f, staging):
                    raise CheckpointError("checkpoint %s is truncated in vector %s" % (self.path, label))
                if v.checksum() != e["checksum"]:
                    raise CheckpointError("checkpoint %s: vector %s fails its checksum" % (self.path, label))
        self.stats["resumes"] += 1

    def remove(self):
        for p in (self.path, self.tmp):
            if os.path.exists(p):
                os.unlink(p)


# ---- driving a fit -------------------------------------------------------------------------------------------------
def agree_flags(engine, flags):
    """Element-wise OR of small integer flags over all ranks: one all-reduce of len(flags) ints."""
    if engine is None or getattr(engine, "world", 1) <= 1:
        return [bool(f) for f in flags]
    import torch
    dev = getattr(engine, "device", None)
    t = torch.tensor([1 if f else 0 for f in flags], dtype=torch.int32,
                     device=dev if dev is not None and getattr(dev, "type", "cpu") == "cuda" else "cpu")
    engine.coll.all_reduce_max(t)
    return [bool(v) for v in t.tolist()]


class Gate(object):
    """Per-boundary decisions of a checkpointed fit, the same on every rank: cancel (a stop request or an exception
    in the progress callback on any rank) and whether the interval-driven state is written (rank 0's clock)."""

    def __init__(self, engine, interval, header=None):
        self.engine = engine
        self.interval = interval
        self.rank = getattr(engine, "rank", 0) if engine is not None else 0
        self.t_last = time.perf_counter()
        self.write_now = False
        # the state on disk: a resumed fit that returns at once (stored k == cap) does not write it again
        self.last_key = state_key(header["state"]) if header is not None else None

    def boundary(self, local_cancel):
        due = self.rank == 0 and self.interval >= 0 and time.perf_counter() - self.t_last >= self.interval
        cancel, self.write_now = agree_flags(self.engine, [local_cancel or stop_requested(), due])
        if cancel:
            clear_stop()        # this fit honours the request
        return cancel

    def written(self):
        self.t_last = time.perf_counter()
        self.write_now = False


def wants(reason, gate):
    """Whether a state handed over at a boundary is written: at the agreed interval, and when the fit returns
    without having converged (a converged fit leaves nothing to continue)."""
    if reason is None:
        return gate.write_now
    return reason != "LBFGS_SUCCESS"


def write_state(ck, gate, state, vectors, fp, staging):
    """Rank 0 writes; every rank learns whether that worked (one all-reduce), so no rank is left in a collective.
    A state equal to the one just written (the interval and the return at the same boundary) is not written again."""
    key = state_key(state)
    if key == gate.last_key:
        gate.written()
        return
    err = None
    if gate.rank == 0:
        try:
            ck.write(state, vectors, fp, staging)
        except BaseException as e:  # agreed below, KeyboardInterrupt / SystemExit included, then re-raised
            err = e
    failed = agree_flags(gate.engine, [err is not None])[0]
    gate.written()
    if not failed:
        gate.last_key = key
    if failed:
        raise err if err is not None else ResourceError("rank 0 failed to write checkpoint %s" % ck.path)


def fit_python(space, params, progress, ck, fp, engine=None):
    """lbfgs.minimize with checkpoints in ``ck``: resumes from the file when it holds a state of this problem.
    ``space`` provides x, g, S, Y (host arrays or device tensors) and get/set_history_scalars."""
    from . import lbfgs as _lbfgs
    header = ck.check(fp, params.max_iterations)
    itemsize = space.x.element_size() if hasattr(space.x, "element_size") else space.x.itemsize
    ck.check_space(space.n, params.m, itemsize)
    staging = _Staging(space.n)

    def vec(a):
        if hasattr(a, "data_ptr"):
            return DeviceVector(engine, a.data_ptr(), a.numel())
        return HostVector(a)

    def sink(name, slot):
        return vec({"x": space.x, "g": space.g}[name] if slot < 0 else (space.S if name == "s" else space.Y)[slot])

    resume = None
    if header is not None:
        ck.load_vectors(sink, staging)
        resume = dict(header["state"])
    gate = Gate(engine, ck.interval, header)
    errors = []

    def on_progress(*a):
        try:
            local = bool(progress(*a)) if progress is not None else False
        except BaseException as exc:          # e.g. SystemExit from a signal handler: save, then re-raise
            errors.append(exc)
            local = True
        return gate.boundary(local)

    def on_state(state):
        if not wants(state["reason"], gate):
            return
        names = state_vector_names(state)
        write_state(ck, gate, state, [(nm, sl, sink(nm, sl)) for nm, sl in names], fp, staging)

    res = _lbfgs.minimize(space, params, on_progress, checkpoint=on_state, checkpoint_interval=0.0, resume=resume)
    if errors:
        raise errors[0]
    return res
