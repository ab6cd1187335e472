"""Golden fixtures as compressed .npz files of at most ~1 MB each.

A fixture `name` is either `name.npz` or the parts `name.0.npz`, `name.1.npz`, ... (arrays grouped in write order);
`load_golden` returns one mapping of array name -> array either way.
"""
from __future__ import annotations

import glob
import os
import re

import numpy as np

PART_BYTES = 900_000  # raw bytes of the arrays grouped into one part (float data barely compresses)


def save_golden(directory: str, name: str, **arrays) -> None:
    for stale in glob.glob(os.path.join(directory, f"{name}.npz")) + glob.glob(os.path.join(directory, f"{name}.*.npz")):
        os.remove(stale)
    parts, cur, size = [], {}, 0
    for key, value in arrays.items():
        a = np.asarray(value)
        if cur and size + a.nbytes > PART_BYTES:
            parts.append(cur)
            cur, size = {}, 0
        cur[key] = a
        size += a.nbytes
    parts.append(cur)
    if len(parts) == 1:
        np.savez_compressed(os.path.join(directory, f"{name}.npz"), **parts[0])
        return
    for i, part in enumerate(parts):
        np.savez_compressed(os.path.join(directory, f"{name}.{i}.npz"), **part)


def load_golden(directory: str, name: str) -> dict:
    single = os.path.join(directory, f"{name}.npz")
    if os.path.exists(single):
        paths = [single]
    else:
        pat = re.compile(re.escape(name) + r"\.(\d+)\.npz$")
        found = [(int(m.group(1)), p) for p in glob.glob(os.path.join(directory, f"{name}.*.npz"))
                 if (m := pat.search(os.path.basename(p)))]
        paths = [p for _, p in sorted(found)]
    if not paths:
        raise FileNotFoundError(f"golden fixture {name!r} not found in {directory}")
    out = {}
    for p in paths:
        with np.load(p) as z:
            out.update({k: z[k] for k in z.files})
    return out
