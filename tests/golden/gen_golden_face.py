"""Fixture for the unaligned-face loop's host helper, produced by the REFERENCE module diffbir/utils/face.py
(FaceRestoreHelper, unmodified) on the CPU in fp32:

    python tests/golden/gen_golden_face.py          # needs /root/reference; writes face_small.npz (no network)

facexlib is replaced, in this process only, by a stand-in backed by oracle/face.py: init_detection_model returns the
fp32 RetinaFace-ResNet50 with facexlib's detect_faces post-processing (torchvision.ops.nms), init_parsing_model the
fp32 ParseNet, and img2tensor / imwrite restate facexlib.utils.misc. Weights are synthetic_face_nets(seed,
class_bias=...). The generator walks the seed and the class-head bias until, in both scenes, two to six faces survive,
at least one detection is dropped by the eye-distance filter, every kept face's score is at least 0.02 from 0.8 and no
two scores above 0.8 are equal (so the order, and with it the NMS, has no ties). A margin on every prior's score is
not asked for: with thousands of priors near the threshold no seed meets it, and the reference and the oracle-backed
helper compute the very same scores, so no decision can differ.

Two scenes follow UnAlignedBFRInferenceLoop: an LQ image bicubic up-scaled x4 to 384 x 512 (read_image brings it to a
min side of 512) and to 544 x 640 (detection scales it by 640 / 544). For n_samples = 2, sample k's restored faces and
background are derived from the crops and the scene (`restored_faces`, `restored_background`), and the pasted image of
each sample is stored. The fixture also stores the seeds, the input checksum, the stand-in's detections, the kept
boxes and landmarks, the affine matrices, checksums and strided samples of the crops, and the parse masks.
"""
import hashlib
import sys
import types
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(HERE))

SCENES = (("small", 96, 128, 11), ("mid", 136, 160, 12))     # name, LQ h, w, LQ seed; x4 up-scale
N_SAMPLES = 2
STRIDE = 7


def scene_image(h: int, w: int, seed: int) -> np.ndarray:
    """The loop's `upscaled_bg`: the synthetic LQ image bicubic up-scaled x4 (PIL), uint8 RGB."""
    from PIL import Image
    from diffbir_b200.utils.synth import synthetic_lq
    lq = Image.fromarray(synthetic_lq(h, w, seed=seed)[0])
    return np.array(lq.resize((4 * w, 4 * h), Image.BICUBIC))


def restored_faces(crop: np.ndarray, k: int) -> np.ndarray:
    """Sample k's "restored" face of a crop (any deterministic image will do: the paste is what is pinned)."""
    return np.ascontiguousarray(np.roll(255 - crop, 7 * k, axis=1))


def restored_background(up: np.ndarray, k: int) -> np.ndarray:
    return np.ascontiguousarray(np.roll(up, 5 * (k + 1), axis=0)[:, ::-1])


def sha(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _img2tensor(imgs, bgr2rgb=True, float32=True):
    """facexlib.utils.misc.img2tensor."""
    import cv2

    def one(img):
        if img.shape[2] == 3 and bgr2rgb:
            if img.dtype == "float64":
                img = img.astype("float32")
            img = cv2.cvtColor(img, cv2.COLOR_BGR2RGB)
        img = torch.from_numpy(img.transpose(2, 0, 1))
        return img.float() if float32 else img
    return [one(i) for i in imgs] if isinstance(imgs, list) else one(imgs)


def install_facexlib(det_sd, parse_sd, log):
    """sys.modules['facexlib...'] stand-ins backed by oracle/face.py; `log` collects detections and parse masks."""
    import torchvision
    from oracle import face as of
    lut = np.array(of.MASK_COLORMAP, dtype=np.uint8)

    class Detector:
        def detect_faces(self, img, conf_threshold=0.8, nms_threshold=0.4, use_origin_size=True):
            out = of.detect_faces(det_sd, img, conf_threshold, nms_threshold, nms=torchvision.ops.nms)
            log["detections"].append(out)
            return out

    class Parser:
        def __call__(self, x):
            with torch.no_grad():
                logits = of.parsenet_forward(parse_sd, x.contiguous())
            log["parse"].append(lut[logits.argmax(dim=1).squeeze().numpy()])
            return logits, None

    mods = {n: types.ModuleType(n) for n in ("facexlib", "facexlib.detection", "facexlib.parsing", "facexlib.utils",
                                             "facexlib.utils.misc")}
    mods["facexlib.detection"].init_detection_model = lambda name, half=False, device=None: Detector()
    mods["facexlib.parsing"].init_parsing_model = lambda model_name="parsenet", device=None: Parser()
    mods["facexlib.utils.misc"].img2tensor = _img2tensor
    mods["facexlib.utils.misc"].imwrite = lambda *a, **k: None
    for n in [m for m in sys.modules if m == "facexlib" or m.startswith("facexlib.")]:
        del sys.modules[n]
    sys.modules.update(mods)


def detection_image(up: np.ndarray) -> np.ndarray:
    """What get_face_landmarks_5(resize=640) hands the detector: read_image's min side 512, then the 640 scaling."""
    import cv2
    img = up
    if min(img.shape[:2]) < 512:
        f = 512.0 / min(img.shape[:2])
        img = cv2.resize(img, (0, 0), fx=f, fy=f, interpolation=cv2.INTER_LINEAR)
    s = max(1, 640 / min(img.shape[:2]))
    return cv2.resize(img, (int(img.shape[1] * s), int(img.shape[0] * s)), interpolation=cv2.INTER_LINEAR), s


def calibrate():
    """(seed, class_bias) meeting the fixture's conditions in both scenes, from one forward per seed and scene."""
    from diffbir_b200.utils.face import select_faces
    from diffbir_b200.utils.synth import synthetic_face_nets
    from oracle import face as of
    for seed in range(231, 251):
        det, _ = synthetic_face_nets(seed, class_bias=0.0)
        cands = []
        for _, h, w, s in SCENES:
            img, scale = detection_image(scene_image(h, w, s))
            b, sc, lm = of.detect_candidates(det, img)
            cands.append((b, torch.log(sc) - torch.log1p(-sc), lm, scale))
        for bias in np.arange(-2.0, 1.0, 0.05):
            ok = True
            for b, logit, lm, scale in cands:
                sc = torch.sigmoid(logit + float(bias))
                top = sc[sc > 0.8]
                if len(top.unique()) != len(top):
                    ok = False
                    break
                rows = select_faces(b, sc, lm) / scale
                kept = [r for r in rows if np.linalg.norm([r[6] - r[8], r[7] - r[9]]) >= 5]
                if not 2 <= len(kept) <= 6 or len(kept) == len(rows) or min(abs(r[4] - 0.8) for r in kept) < 0.03:
                    ok = False
                    break
            if ok:
                return seed, round(float(bias), 2)
    raise SystemExit("no seed / class bias met the fixture's conditions")


def main():
    from _ref_import import use_reference
    sys.path.insert(0, str(ROOT / "tests"))
    from golden_io import save_golden
    use_reference()
    from diffbir_b200.utils.synth import synthetic_face_nets
    seed, bias = calibrate()
    det, parse = synthetic_face_nets(seed, class_bias=bias)
    log = {"detections": [], "parse": []}
    install_facexlib(det, parse, log)
    from diffbir.utils.face import FaceRestoreHelper           # the reference module, unmodified
    helper = FaceRestoreHelper(upscale_factor=1, face_size=512, use_parse=True, det_model="retinaface_resnet50",
                               device="cpu")
    arrays = {"seed": np.array(seed), "class_bias": np.array(bias)}
    for name, h, w, s in SCENES:
        up = scene_image(h, w, s)
        log["detections"].clear()
        log["parse"].clear()
        helper.clean_all()
        helper.read_image(up)
        helper.get_face_landmarks_5(resize=640, eye_dist_threshold=5)
        helper.align_warp_face()
        helper.get_inverse_affine()
        (dets,) = log["detections"]
        n = len(helper.cropped_faces)
        assert 2 <= n < len(dets) and min(abs(f[4] - 0.8) for f in helper.det_faces) >= 0.02, (name, n, len(dets))
        pasted = []
        for k in range(N_SAMPLES):
            for crop in helper.cropped_faces:
                helper.add_restored_face(restored_faces(crop, k))
            pasted.append(helper.paste_faces_to_input_image(upsample_img=restored_background(up, k)))
            helper.restored_faces.clear()
        p = name + "_"
        arrays.update({
            p + "input_sha": np.array(sha(up)), p + "input_img_shape": np.array(helper.input_img.shape),
            p + "detections": dets, p + "det_faces": np.stack(helper.det_faces),
            p + "landmarks": np.stack(helper.all_landmarks_5), p + "affine": np.stack(helper.affine_matrices),
            p + "crop_sha": np.array([sha(c) for c in helper.cropped_faces]),
            p + "crop_strided": np.stack([c[::STRIDE, ::STRIDE] for c in helper.cropped_faces]),
            p + "parse_bits": np.packbits(np.stack(log["parse"]) > 0, axis=-1),
            p + "pasted_sha": np.array([sha(x) for x in pasted]),
            p + "pasted_strided": np.stack([x[::STRIDE, ::STRIDE] for x in pasted])})
        print(f"{name}: input {up.shape} -> {helper.input_img.shape}, {len(dets)} detections, {n} faces kept")
    save_golden(HERE, "face_small", arrays)
    print(f"seed {seed}, class bias {bias}")


if __name__ == "__main__":
    main()
