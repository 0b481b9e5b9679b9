"""Golden fixtures as .npz files of at most 1 MB each: a fixture `<stem>.npz` that would be larger continues in
`<stem>.part2.npz`, `<stem>.part3.npz`, ...  save() splits, load() merges every part back into one dict."""
from __future__ import annotations

import glob
import io
import os

import numpy as np

LIMIT = 1_000_000


def _size(arrays: dict) -> int:
    buf = io.BytesIO()
    np.savez_compressed(buf, **arrays)
    return buf.tell()


def save(path: str, arrays: dict) -> list:
    """Write `arrays` (name -> ndarray) to `path` and as many parts as needed to keep each file under LIMIT bytes."""
    stem = path[:-4]
    for old in glob.glob(stem + ".part*.npz"):
        os.remove(old)
    parts, cur = [], {}
    for k in sorted(arrays):
        trial = dict(cur, **{k: arrays[k]})
        if cur and _size(trial) > LIMIT:
            parts.append(cur)
            cur = {k: arrays[k]}
        else:
            cur = trial
    parts.append(cur)
    paths = [path] + [f"{stem}.part{i}.npz" for i in range(2, len(parts) + 1)]
    for p, a in zip(paths, parts):
        if _size(a) > LIMIT:
            raise ValueError(f"{p}: a single array exceeds {LIMIT} bytes; store a sample of it")
        np.savez_compressed(p, **a)
    return paths


def load(path: str) -> dict:
    """name -> ndarray over `path` and its parts."""
    stem = path[:-4]
    out = {}
    for p in [path] + sorted(glob.glob(stem + ".part*.npz")):
        with np.load(p) as d:
            out.update({k: d[k] for k in d.files})
    return out
