"""Golden vectors stored in parts: no committed file exceeds 1 MB.

`save(path, arrays)` writes `path` and, where the compressed arrays do not fit one file, `<stem>.part<i>.npz`
files beside it; an array too large for a part by itself is cut along its first axis into chunks stored as
`<name>@<j>`.  `load(path)` returns the merged arrays as a dict, chunks concatenated in order."""
from __future__ import annotations

import glob
import io
import os

import numpy as np

PART_BYTES = 900 * 1024


def _compressed_size(a: np.ndarray) -> int:
    buf = io.BytesIO()
    np.savez_compressed(buf, a=a)
    return buf.tell()


def _pieces(name, a):
    """(key, array, compressed bytes) pieces of one array, each small enough for a part."""
    size = _compressed_size(a)
    if size <= PART_BYTES or a.ndim == 0 or a.shape[0] < 2:
        return [(name, a, size)]
    n = min(a.shape[0], -(-size // (PART_BYTES * 9 // 10)))
    out = []
    for j, c in enumerate(np.array_split(a, n, axis=0)):
        out.append((f"{name}@{j}", c, _compressed_size(c)))
    return out


def save(path: str, arrays: dict) -> list:
    """Write `arrays` to `path` (+ parts); returns the files written."""
    stem = path[:-4] if path.endswith(".npz") else path
    for old in glob.glob(f"{stem}.part*.npz"):
        os.remove(old)
    parts, cur, cur_bytes = [], {}, 0
    for name, a in arrays.items():
        for key, piece, size in _pieces(name, np.asarray(a)):
            if cur and cur_bytes + size > PART_BYTES:
                parts.append(cur)
                cur, cur_bytes = {}, 0
            cur[key] = piece
            cur_bytes += size
    parts.append(cur)
    files = []
    for i, part in enumerate(parts):
        f = f"{stem}.npz" if i == 0 else f"{stem}.part{i}.npz"
        np.savez_compressed(f, **part)
        files.append(f)
    return files


def load(path: str) -> dict:
    stem = path[:-4] if path.endswith(".npz") else path
    files = [f"{stem}.npz"] + sorted(glob.glob(f"{stem}.part*.npz"), key=lambda f: int(f[len(stem) + 5:-4]))
    merged, chunks = {}, {}
    for f in files:
        with np.load(f) as d:
            for k in d.files:
                if "@" in k:
                    name, j = k.rsplit("@", 1)
                    chunks.setdefault(name, {})[int(j)] = d[k]
                else:
                    merged[k] = d[k]
    for name, cs in chunks.items():
        merged[name] = np.concatenate([cs[j] for j in sorted(cs)], axis=0)
    return merged
