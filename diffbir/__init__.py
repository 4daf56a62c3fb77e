"""`diffbir` — import-path alias of the H100-native engine (package `diffbir_b200`).

Reference-side callers (`run_gradio.py`, notebooks, third-party scripts) import
`diffbir.pipeline`, `diffbir.model`, `diffbir.sampler`, `diffbir.inference`, `diffbir.utils.common`;
with this directory on sys.path ahead of the reference checkout those imports resolve to the
sm_90a engine without edits. Every public name of the reference's packages exists here:
names on the accelerated path are the `diffbir_b200` classes themselves, names outside it
(SURVEY.md 8f) are placeholders that raise NotImplementedError when constructed, so a caller fails
at the point of use with a message naming the supported alternative, never silently on a slow path.
"""
from diffbir_b200 import lib as _lib  # noqa: F401  (fails loudly if the CUDA library is missing at first use)

__all__ = ["pipeline", "model", "sampler", "inference", "utils"]
