"""
Alignment ingest for the PLM engine: A2M/FASTA text -> uint8 code matrix.

Mirrors what plmc does before inference (SURVEY.md 8a row a4, behaviour pinned
by the golden run in the reference's notebooks/example/):

* rows are upper-cased, '.' is a gap;
* a row is invalid if ANY character of the row (insert columns included) is
  outside alphabet + {'-', '.'} (case-insensitive);
* focus mode: model sites = columns where the focus sequence has an upper-case
  non-gap character; ``index_list`` numbers them by residue offset from the
  ``/start-end`` of the focus header ("Region starts at");
* with ignore_gaps (plmc -g) the gap (alphabet[0]) is not a model state: residues
  are coded 0..q-1 in alphabet[1:] order and the gap is coded q.

The reference side of this boundary is evcouplings/couplings/tools.py:213-233
(focus name passed with ``/range`` stripped, alphabet with gap first).
"""
import os
from collections import namedtuple

import numpy as np

ALPHABET_PROTEIN = "-ACDEFGHIKLMNPQRSTVWY"   # evcouplings/align/alignment.py:21-26

EncodedAlignment = namedtuple("EncodedAlignment", [
    "codes",            # (n_valid, L) uint8, C-contiguous
    "valid",            # (n_total,) bool
    "q",                # number of model states
    "gap_code",         # -1 (gap is a state) or q (ignore_gaps)
    "model_alphabet",   # str of length q
    "focus_index",      # int or None
    "focus_cols",       # (L,) int64 column indices into the raw alignment
    "index_list",       # (L,) int32
    "target_seq",       # str of length L
    "region_start",     # int
    "n_total", "n_valid", "num_total_sites",
])


class AlignmentError(ValueError):
    pass


# Codes of the model states (and of the ignored gap) must fit the 5 bit-planes of the Hamming pass: codes < 32.
MAX_STATES = 32


def alphabet_states(alphabet, ignore_gaps=False):
    """Number of model states q of ``alphabet`` (gap first), or a ValueError naming the limit: 2 <= q <= 32 with the
    gap as a state (2 to 32 characters), 2 <= q <= 31 with ignore_gaps, whose gap is coded q (3 to 32 characters)."""
    n = len(alphabet)
    if len(set(alphabet)) != n:
        raise ValueError("alphabet has repeated characters")
    q = n - 1 if ignore_gaps else n
    top = MAX_STATES - 1 if ignore_gaps else MAX_STATES
    if not 2 <= q <= top:
        raise ValueError(
            "alphabet %r gives q=%d model states%s; the engine supports 2 <= q <= %d (%d to %d characters%s): every "
            "code must be below %d, the 5 bit-planes of the sequence reweighting"
            % (alphabet, q, " (gap ignored)" if ignore_gaps else "", top, 3 if ignore_gaps else 2, MAX_STATES,
               ", the gap coded q" if ignore_gaps else "", MAX_STATES))
    return q


def read_fasta_matrix(path):
    """Read FASTA/A2M into (ids, uint8 matrix n_total x width of raw characters) with the compiled reader of
    libevcplm (csrc/a2m_reader.cu: mmap + memchr, SURVEY 8f row f4).  Sequences may be wrapped over several lines."""
    import ctypes
    from . import _lib
    lib = _lib.load()
    n_rows, width, ids_bytes = ctypes.c_int64(0), ctypes.c_int64(0), ctypes.c_int64(0)
    bpath = os.fsencode(path)
    rc = lib.evc_a2m_scan(bpath, ctypes.byref(n_rows), ctypes.byref(width), ctypes.byref(ids_bytes))
    if rc == 2:
        raise AlignmentError(lib.evc_last_error().decode())
    _lib.check(rc, "evc_a2m_scan")
    raw = np.empty((n_rows.value, width.value), dtype=np.uint8)
    idbuf = ctypes.create_string_buffer(max(1, ids_bytes.value))
    rc = lib.evc_a2m_read(bpath, n_rows.value, width.value, raw.ctypes.data_as(ctypes.c_void_p), idbuf, ids_bytes.value)
    if rc == 2:
        raise AlignmentError(lib.evc_last_error().decode())
    _lib.check(rc, "evc_a2m_read")
    ids = idbuf.raw[:ids_bytes.value].decode("ascii", "replace").split("\0")[:n_rows.value]
    return ids, raw


def read_fasta_matrix_py(path):
    """Pure-Python twin of read_fasta_matrix (kept as the cross-check of the compiled reader in the tests)."""
    ids, chunks, cur = [], [], None
    with open(path, "rb") as f:
        for line in f:
            if line.startswith(b">"):
                if cur is not None:
                    chunks.append(b"".join(cur))
                ids.append(line[1:].strip().decode("ascii", "replace"))
                cur = []
            elif cur is not None:
                cur.append(line.strip())
    if cur is not None:
        chunks.append(b"".join(cur))
    if not chunks:
        raise AlignmentError("alignment %s contains no sequences" % path)
    width = len(chunks[0])
    if width == 0:
        raise AlignmentError("alignment %s has zero-length sequences" % path)
    for k, c in enumerate(chunks):
        if len(c) != width:
            raise AlignmentError("ragged alignment: row %d has length %d, expected %d" % (k, len(c), width))
    mat = np.frombuffer(b"".join(chunks), dtype=np.uint8).reshape(len(chunks), width)
    return ids, mat


def _find_focus(ids, focus):
    key = focus.split("/")[0]
    for k, name in enumerate(ids):
        tok = name.split()[0] if name.split() else name
        if tok == focus or tok.split("/")[0] == key:
            return k, tok
    raise AlignmentError("focus sequence %r not found in alignment" % focus)


def encode_alignment(ids, raw, focus=None, alphabet=None, ignore_gaps=False):
    """raw: (n_total, width) uint8 characters.  Returns EncodedAlignment."""
    if alphabet is None:
        alphabet = ALPHABET_PROTEIN
    try:
        alphabet_states(alphabet, ignore_gaps)
    except ValueError as e:
        raise AlignmentError(str(e))
    gap = alphabet[0]
    n_total, width = raw.shape

    upper = np.arange(256, dtype=np.uint8)
    upper[ord("a"):ord("z") + 1] -= 32

    focus_index, region_start = None, 1
    if focus is not None:
        focus_index, tok = _find_focus(ids, focus)
        if "/" in tok:
            try:
                region_start = int(tok.split("/")[-1].split("-")[0])
            except ValueError:
                region_start = 1
        frow = raw[focus_index]
        is_gap = (frow == ord(gap)) | (frow == ord(".")) | (frow == ord("-"))
        is_upper = (upper[frow] == frow)
        residue_offset = np.cumsum(~is_gap) - 1
        keep = (~is_gap) & is_upper
        cols = np.nonzero(keep)[0]
        index_list = (region_start + residue_offset[cols]).astype(np.int32)
        num_total_sites = int((~is_gap).sum())
    else:
        cols = np.arange(width)
        index_list = np.arange(1, width + 1, dtype=np.int32)
        num_total_sites = width
    if len(cols) < 2:
        raise AlignmentError("fewer than 2 model sites selected")

    # one table: raw character (either case) -> model code, 255 = character outside alphabet + {'-', '.'}
    lut = np.full(256, 255, dtype=np.uint8)
    if ignore_gaps:
        q = len(alphabet) - 1
        for k, ch in enumerate(alphabet[1:]):
            lut[ord(ch)] = k
        gap_code = q
        model_alphabet = alphabet[1:]
        gcode = q
    else:
        q = len(alphabet)
        for k, ch in enumerate(alphabet):
            lut[ord(ch)] = k
        gap_code = -1
        model_alphabet = alphabet
        gcode = 0
    lut[ord(gap)] = gcode
    lut[ord("-")] = gcode
    lut[ord(".")] = gcode
    for c in range(ord("a"), ord("z") + 1):      # case-insensitive (rows are upper-cased by plmc)
        lut[c] = lut[c - 32]
    codes, valid = _encode_rows(raw, lut, cols)
    if focus_index is not None:
        target = bytes(upper[raw[focus_index, cols]]).decode("ascii")
    else:
        target = bytes(upper[raw[0, cols]]).decode("ascii").replace(".", "-")
    return EncodedAlignment(
        codes=codes, valid=valid, q=q, gap_code=gap_code, model_alphabet=model_alphabet,
        focus_index=focus_index, focus_cols=cols.astype(np.int64), index_list=index_list,
        target_seq=target, region_start=region_start, n_total=n_total,
        n_valid=int(valid.sum()), num_total_sites=num_total_sites,
    )


def _encode_rows(raw, lut, cols):
    """codes of the selected columns of the valid rows + the validity mask, by the compiled encoder
    (evc_msa_encode: threaded, two passes over the character matrix)."""
    import ctypes
    from . import _lib
    lib = _lib.load()
    raw = np.ascontiguousarray(raw, dtype=np.uint8)
    n_total, width = raw.shape
    cols64 = np.ascontiguousarray(cols, dtype=np.int64)
    valid8 = np.empty(n_total, dtype=np.uint8)
    codes = np.empty((n_total, len(cols64)), dtype=np.uint8)
    n_valid = ctypes.c_int64(0)
    vp = ctypes.c_void_p
    _lib.check(lib.evc_msa_encode(raw.ctypes.data_as(vp), n_total, width, lut.ctypes.data_as(vp),
                                  cols64.ctypes.data_as(vp), len(cols64), valid8.ctypes.data_as(vp),
                                  codes.ctypes.data_as(vp), ctypes.byref(n_valid)), "evc_msa_encode")
    return codes[:n_valid.value], valid8.astype(bool)


def load_alignment(path, focus=None, alphabet=None, ignore_gaps=False):
    ids, raw = read_fasta_matrix(path)
    return encode_alignment(ids, raw, focus=focus, alphabet=alphabet, ignore_gaps=ignore_gaps)


def identity_threshold_count(theta, L):
    """Integer form of the in-tree rule ``pair_id / L >= theta``
    (evcouplings/align/alignment.py:1229): the smallest count c with
    c / float(L) >= theta, evaluated in the same float64 arithmetic."""
    c = int(theta * L)
    while c > 0 and (c - 1) / float(L) >= theta:
        c -= 1
    while c / float(L) < theta:
        c += 1
    return c
