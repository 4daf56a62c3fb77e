"""Times the unaligned-face loop's networks on the GPU against the same networks as PyTorch fp32 modules (cuDNN,
torch's default TF32 setting), on synthetic weights. Prints the card and its power limit first.

    python tools/measure_faces.py

Engine and baseline windows alternate (5 rounds of at least 0.5 s each); the median and the spread over the rounds
are printed. The engine's peak added device memory is read before the baseline runs. The host paste is timed on a
2048^2 photo with the detector's class bias raised until it finds faces.
"""
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
ROUNDS = 5
WINDOW_S = 0.5


def window_ms(fn):
    """Mean ms per call over a window of at least WINDOW_S seconds (ends in a device synchronise)."""
    torch.cuda.synchronize()
    t, n = time.perf_counter(), 0
    while True:
        fn()
        n += 1
        if n % 4 == 0:
            torch.cuda.synchronize()
            if time.perf_counter() - t >= WINDOW_S:
                return (time.perf_counter() - t) / n * 1e3


def compare(label, engine, baseline):
    e, b = [], []
    for _ in range(ROUNDS):
        e.append(window_ms(engine))
        b.append(window_ms(baseline))
    print(f"{label}: engine {np.median(e):.2f} ms (min {min(e):.2f}, max {max(e):.2f}); "
          f"torch fp32 {np.median(b):.2f} ms (min {min(b):.2f}, max {max(b):.2f})")


def main():
    from diffbir_b200.engine.parsenet import MAX_BATCH, ParseNetEngine
    from diffbir_b200.engine.retinaface import RetinaFaceEngine
    from diffbir_b200.utils.face import FaceRestoreHelper
    from diffbir_b200.utils.synth import synthetic_face_nets, synthetic_lq
    from oracle import face as of
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip())
    det, parse = synthetic_face_nets(231)
    imgs = {side: synthetic_lq(side, side, seed=side)[0] for side in (1024, 2048)}
    faces = [synthetic_lq(512, 512, seed=s)[0] for s in range(8)]
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    deng, peng = RetinaFaceEngine(det), ParseNetEngine(parse)
    first = {}
    for side, img in imgs.items():
        t = time.perf_counter()
        deng.heads(img)
        torch.cuda.synchronize()
        first[side] = (time.perf_counter() - t) * 1e3
    for n in (1, 4, 8):
        peng.masks(faces[:n])
    torch.cuda.synchronize()
    peak = (torch.cuda.max_memory_allocated() - m0) / 2 ** 30
    print(f"engines' peak added device memory (weights + workspaces, detector up to 2048^2, parser {MAX_BATCH} faces "
          f"per forward): {peak:.2f} GiB")
    dsd, psd = ({k: v.cuda() for k, v in sd.items()} for sd in (det, parse))
    for side, img in imgs.items():
        x = (torch.from_numpy(img).cuda().float() - torch.tensor(of.DETECTOR_MEAN, device="cuda")).permute(2, 0, 1)
        x = x[None].contiguous()
        with torch.no_grad():
            compare(f"detector {side}x{side} (first engine call {first[side]:.1f} ms)", lambda: deng.heads(img),
                    lambda: of.retinaface_forward(dsd, x))
    for n in (1, 4):
        xs = torch.stack([torch.from_numpy(np.ascontiguousarray(f[:, :, ::-1].transpose(2, 0, 1))) for f in faces[:n]])
        xs = ((xs.cuda().float() / 255 - 0.5) / 0.5).contiguous()
        with torch.no_grad():
            compare(f"parser {n} face(s)", lambda: peng.masks(faces[:n]), lambda: of.parsenet_forward(psd, xs))
    img = imgs[2048]
    for bias in (-1.4, -1.0, -0.6, -0.2, 0.2):
        d2, _ = synthetic_face_nets(231, class_bias=bias)
        h = FaceRestoreHelper("cuda", detector=RetinaFaceEngine(d2).candidates, parser=peng.masks)
        h.read_image(img)
        n = h.get_face_landmarks_5(resize=640, eye_dist_threshold=5)
        if n:
            break
    if not n:
        print("host paste at 2048x2048: no face detected, not measured")
        return
    h.align_warp_face()
    h.get_inverse_affine()
    for f in h.cropped_faces:
        h.add_restored_face(f)
    masks = h.parse_faces(h.restored_faces)
    h.paste_faces_to_input_image(img, masks)
    t = time.perf_counter()
    for _ in range(3):
        h.paste_faces_to_input_image(img, masks)
    ms = (time.perf_counter() - t) / 3 * 1e3
    print(f"host paste at 2048x2048: {ms / n:.1f} ms per face ({n} faces, class bias {bias})")


if __name__ == "__main__":
    main()
