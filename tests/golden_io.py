"""Loading of golden fixtures that are stored in several files (each file is kept under 1 MB)."""
from pathlib import Path

import numpy as np


def load_golden(golden_dir: Path, stem: str) -> dict:
    """The arrays of golden_dir/<stem>.npz and of its pieces <stem>_part<N>.npz, as one dict."""
    out = {}
    for p in [golden_dir / f"{stem}.npz", *sorted(golden_dir.glob(f"{stem}_part*.npz"))]:
        with np.load(p) as z:
            for k in z.files:
                assert k not in out, f"{k} stored twice"
                out[k] = z[k]
    return out


def save_golden(golden_dir: Path, stem: str, arrays: dict, max_bytes: int = 900_000) -> None:
    """Writes `arrays` as golden_dir/<stem>.npz plus as many <stem>_part<N>.npz as needed to keep every file's
    uncompressed payload under max_bytes (arrays are never cut; stale parts are removed first)."""
    for p in golden_dir.glob(f"{stem}_part*.npz"):
        p.unlink()
    files, cur, size = [], {}, 0
    for k in sorted(arrays, key=lambda k: -np.asarray(arrays[k]).nbytes):
        n = np.asarray(arrays[k]).nbytes
        assert n <= max_bytes, f"{k}: {n} bytes do not fit one file"
        if cur and size + n > max_bytes:
            files.append(cur)
            cur, size = {}, 0
        cur[k] = arrays[k]
        size += n
    files.append(cur)
    for i, group in enumerate(files):
        name = f"{stem}.npz" if i == 0 else f"{stem}_part{i}.npz"
        np.savez_compressed(golden_dir / name, **group)
