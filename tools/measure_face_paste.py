"""Times the unaligned-face paste-back on the host (cv2 / numpy) against the engine (csrc/face_paste.cu), per face,
on synthetic scenes (synth.synthetic_paste_scene: overlapping and edge-cut faces) at 1024^2 and 2048^2 with 1, 4 and
35 faces, one sample. Prints the card and its power limit first, then per scene the median and range of the
alternating host / engine windows, and checks the bytes are equal in every scene.

    python tools/measure_face_paste.py
"""
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
ROUNDS = 3
WINDOW_S = 0.5


def window_ms(fn):
    """Mean ms per call over a window of at least WINDOW_S seconds (each call ends with its photo on the host)."""
    t, n = time.perf_counter(), 0
    while True:
        fn()
        n += 1
        if time.perf_counter() - t >= WINDOW_S:
            return (time.perf_counter() - t) / n * 1e3


def main():
    from diffbir_b200 import lib
    from diffbir_b200.utils.synth import synthetic_paste_scene
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip())
    lib.load()
    for side in (1024, 2048):
        for n in (1, 4, 35):
            helper, bgs, faces, masks = synthetic_paste_scene(side, n, samples=1, seed=side + n)
            dmasks = torch.from_numpy(masks).cuda()

            def host():
                helper.restored_faces = list(faces[0])
                return helper.paste_faces_to_input_image(bgs[0], list(masks))

            def engine():
                return helper.paste_faces_device(bgs, faces, dmasks)[0]

            same = np.array_equal(host(), engine())
            assert helper.paste_path == "engine", "the scene must take the engine path"
            hs, es = [], []
            for _ in range(ROUNDS):
                hs.append(window_ms(host))
                es.append(window_ms(engine))
            print(f"{side}^2, {n:2d} faces: host {np.median(hs) / n:8.2f} ms/face (range {min(hs) / n:.2f}-"
                  f"{max(hs) / n:.2f}); engine {np.median(es) / n:6.3f} ms/face (range {min(es) / n:.3f}-"
                  f"{max(es) / n:.3f}), {np.median(es):.2f} ms per photo; bytes equal: {same}")
            assert same


if __name__ == "__main__":
    main()
