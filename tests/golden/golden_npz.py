"""
Golden fixtures are kept below 1 MB per file: a fixture `<name>` is stored as `<name>.part<k>.npz`, and an array too
large for one file is cut along its first axis into keys `<key>__<i>` spread over several parts.  load() reassembles
the arrays; save() writes them.

Why split rather than sample: two fixtures are larger than 1 MB compressed and are needed whole.  `pabp_codes` is the
full PABP_YEAST alignment (151,496 x 82), because plmc's stored neighbour counts, which the Hamming kernel must match
bit for bit, depend on every pair of sequences.  `pabp_golden` holds plmc's full couplings J (3321 x 20 x 20),
because the gradient-balance, objective-scaling and EC checks evaluate the objective and its gradient at plmc's own
optimum, which needs every coupling.  Fixtures that a sample serves (the PABP A2M text for the ingest test) are
sampled instead.
"""
import glob
import io
import os
import re

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PART_BYTES = 900_000


def _parts(name):
    paths = glob.glob(os.path.join(HERE, name + ".part*.npz"))
    return sorted(paths, key=lambda p: int(re.search(r"\.part(\d+)\.npz$", p).group(1)))


def load(name):
    """{key: array} of fixture `name`, pieces of split arrays concatenated in order."""
    paths = _parts(name)
    if not paths:
        raise FileNotFoundError("golden fixture %r not found in %s" % (name, HERE))
    out, pieces = {}, {}
    for p in paths:
        with np.load(p) as d:
            for k in d.files:
                base, sep, i = k.rpartition("__")
                if sep and i.isdigit():
                    pieces.setdefault(base, {})[int(i)] = d[k]
                else:
                    out[k] = d[k]
    for k, v in pieces.items():
        out[k] = np.concatenate([v[i] for i in sorted(v)])
    return out


def _compressed_size(arrays):
    b = io.BytesIO()
    np.savez_compressed(b, **arrays)
    return b.tell()


def save(name, **arrays):
    """Writes fixture `name`: small arrays together in part 0, every array that does not fit split over parts."""
    for p in _parts(name):
        os.remove(p)
    small = {k: np.asarray(v) for k, v in arrays.items() if _compressed_size({k: v}) < PART_BYTES // 8}
    parts = [small]
    for k, v in arrays.items():
        if k in small:
            continue
        n = 1
        while max(_compressed_size({"x": c}) for c in np.array_split(np.asarray(v), n)) >= PART_BYTES:
            n += 1
        for i, c in enumerate(np.array_split(np.asarray(v), n)):
            parts.append({"%s__%d" % (k, i): c})
    for i, p in enumerate(parts):
        np.savez_compressed(os.path.join(HERE, "%s.part%d.npz" % (name, i)), **p)
