"""Golden fixtures under tests/golden/.  A fixture is one ``<name>.npz`` or, when it would exceed the repository's
1 MB limit on a single file, numbered parts ``<name>.<i>.npz`` that together hold its arrays.  ``load`` returns
the arrays of either form as one mapping with the ``.files`` list of an ``np.load`` result."""

from __future__ import annotations

import glob
import os

import numpy as np

DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
PART_BYTES = 900_000      # uncompressed bytes per part: the compressed part stays below 1 MB
MAX_FILE_BYTES = 1_000_000


class Golden(dict):
    @property
    def files(self) -> list:
        return list(self.keys())


def load(name: str) -> Golden:
    paths = sorted(glob.glob(os.path.join(DIR, f"{name}.[0-9]*.npz"))) or [os.path.join(DIR, f"{name}.npz")]
    g = Golden()
    for p in paths:
        with np.load(p) as z:
            g.update({k: z[k] for k in z.files})
    return g


def save(name: str, arrays: dict, out_dir: str = DIR) -> None:
    """np.savez_compressed of ``arrays`` as ``<name>.npz``, or as parts of at most PART_BYTES (uncompressed).
    Every file written must stay below MAX_FILE_BYTES: store a sample of an array that does not fit."""
    for p in glob.glob(os.path.join(out_dir, f"{name}.[0-9]*.npz")) + glob.glob(os.path.join(out_dir, f"{name}.npz")):
        os.remove(p)
    if sum(np.asarray(a).nbytes for a in arrays.values()) <= PART_BYTES:
        _write(os.path.join(out_dir, f"{name}.npz"), arrays)
        return
    parts, cur, size = [], {}, 0
    for k, a in arrays.items():
        n = np.asarray(a).nbytes
        if cur and size + n > PART_BYTES:
            parts.append(cur)
            cur, size = {}, 0
        cur[k] = a
        size += n
    parts.append(cur)
    for i, part in enumerate(parts):
        _write(os.path.join(out_dir, f"{name}.{i}.npz"), part)


def _write(path: str, arrays: dict) -> None:
    np.savez_compressed(path, **arrays)
    size = os.path.getsize(path)
    if size >= MAX_FILE_BYTES:
        os.remove(path)
        raise ValueError(f"{path}: {size} bytes, above the {MAX_FILE_BYTES}-byte limit for a fixture file")
