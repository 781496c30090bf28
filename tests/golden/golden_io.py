"""Golden records are .npz files; a record whose compressed size would exceed MAX_BYTES is stored as `name.npz` plus
`name.part1.npz`, `name.part2.npz`, ... (disjoint key sets).  tests/conftest.py merges them on load."""
import io
import os

import numpy as np

MAX_BYTES = 1000 * 1000


def _compressed_size(arrays):
    buf = io.BytesIO()
    np.savez_compressed(buf, **arrays)
    return buf.tell()


def savez_split(path, arrays, max_bytes=MAX_BYTES):
    """np.savez_compressed(path, **arrays), split by keys (in order) into parts of at most max_bytes each."""
    stem = path[:-4] if path.endswith(".npz") else path
    parts, cur = [], {}
    for k in arrays:
        trial = dict(cur, **{k: arrays[k]})
        if cur and _compressed_size(trial) > max_bytes:
            parts.append(cur)
            cur = {k: arrays[k]}
        else:
            cur = trial
    parts.append(cur)
    d = os.path.dirname(stem) or "."
    base = os.path.basename(stem)
    for q in os.listdir(d):
        if q.startswith(base + ".part") and q.endswith(".npz"):
            os.remove(os.path.join(d, q))
    for i, part in enumerate(parts):
        np.savez_compressed(stem + (".npz" if i == 0 else ".part%d.npz" % i), **part)
