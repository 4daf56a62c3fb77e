"""-m gpu: the paste-back's engine path (csrc/face_paste.cu) byte for byte against cv2: each kernel over its region of
interest, the whole paste on the face_small fixture scenes and on a 2048^2 35-face scene, and `--task unaligned_face`
writing the same PNG bytes on both paths."""
import hashlib
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from diffbir_b200.utils import face as fc  # noqa: E402

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
DEV = "cuda"


def _lib():
    from diffbir_b200 import lib
    lib.load()
    return lib


def _host_soft(square, edge):
    soft = cv2.erode(square, np.ones((2 * edge, 2 * edge), np.uint8))
    return cv2.GaussianBlur(soft, (2 * edge + 1, 2 * edge + 1), 0)


@pytest.mark.parametrize("side,n,seed", [(1024, 6, 0), (640, 5, 3), (2048, 4, 7)])
def test_square_and_soft_kernels_match_cv2(side, n, seed):
    """Rotated, scaled and edge-cut squares: the warp + 2x2 erode, the fp64 sum and the soft mask over the ROI equal
    cv2 on the full frame, and the frame outside the ROI is 0 in cv2's images."""
    from diffbir_b200.utils.synth import synthetic_paste_scene
    L = _lib()
    helper = synthetic_paste_scene(side, n, seed=seed)[0]
    h, w = helper.input_img.shape[:2]
    for inv in helper.inverse_affine_matrices:
        ref = cv2.erode(cv2.warpAffine(np.ones((512, 512), np.float32), inv, (w, h)), np.ones((2, 2), np.uint8))
        roi = fc.paste_roi(inv, 512, h, w)
        x0, y0, rw, rh = roi
        sq = torch.empty(rh, rw, device=DEV)
        total = torch.zeros(1, dtype=torch.float64, device=DEV)
        L.paste_square(fc.warp_map(inv), 512, h, w, roi, sq, total)
        got = np.zeros_like(ref)
        got[y0:y0 + rh, x0:x0 + rw] = sq.cpu().numpy()
        assert np.array_equal(got, ref)
        edge = int(np.sum(ref) ** 0.5) // 20
        assert fc.paste_edge(total.item(), lambda: got) == edge
        if edge in (1, 2):          # 3- and 5-tap blurs: photos with such faces take the cv2 path
            continue
        taps = torch.from_numpy(cv2.getGaussianKernel(2 * edge + 1, 0, cv2.CV_32F).ravel()).to(DEV)
        soft = torch.empty_like(sq)
        L.paste_soft(sq, h, w, roi, edge, taps, torch.empty_like(sq), soft)
        got = np.zeros_like(ref)
        got[y0:y0 + rh, x0:x0 + rw] = soft.cpu().numpy()
        assert np.array_equal(got, _host_soft(ref, edge))


def test_soft_kernel_edge_zero_and_border_columns():
    """edge 0 (the empty erode kernel, a 1-tap blur) and a square whose blur reaches the columns of cv2's 4-wide loop
    (w = 8 k + 4) and the frame's last column."""
    L = _lib()
    h, w = 200, 132
    for inv, edge in ((np.array([[0.02, 0.0, 40.0], [0.0, 0.02, 30.0]]), 0),
                      (np.array([[0.3, 0.05, 90.0], [-0.05, 0.3, 20.0]]), None)):
        ref = cv2.erode(cv2.warpAffine(np.ones((512, 512), np.float32), inv, (w, h)), np.ones((2, 2), np.uint8))
        e = int(np.sum(ref) ** 0.5) // 20
        assert edge is None or e == edge
        roi = fc.paste_roi(inv, 512, h, w)
        x0, y0, rw, rh = roi
        sq = torch.from_numpy(np.ascontiguousarray(ref[y0:y0 + rh, x0:x0 + rw])).to(DEV)
        taps = torch.from_numpy(cv2.getGaussianKernel(2 * e + 1, 0, cv2.CV_32F).ravel()).to(DEV)
        soft = torch.empty_like(sq)
        L.paste_soft(sq, h, w, roi, e, taps, torch.empty_like(sq), soft)
        got = np.zeros_like(ref)
        got[y0:y0 + rh, x0:x0 + rw] = soft.cpu().numpy()
        want = cv2.GaussianBlur(cv2.erode(ref, np.ones((2 * e, 2 * e), np.uint8)), (2 * e + 1,) * 2, 0)
        assert np.array_equal(got, want), e
        if edge is None:
            assert x0 + rw > w // 8 * 8


def test_parse_blur_matches_cv2():
    L = _lib()
    from diffbir_b200.utils.synth import synthetic_paste_scene
    masks = synthetic_paste_scene(512, 3, samples=2, seed=4)[3]
    masks[0, :40] = 255                                   # mask content at the border: reflect-101
    taps = torch.from_numpy(cv2.getGaussianKernel(101, 11, cv2.CV_64F).ravel()).to(DEV)
    m = torch.from_numpy(masks).to(DEV)
    out = torch.empty(m.shape, dtype=torch.float64, device=DEV)
    L.paste_parse_blur(m, taps, torch.empty_like(out), out)
    for got, mk in zip(out.cpu().numpy(), masks):
        pm = cv2.GaussianBlur(cv2.GaussianBlur(mk.astype(np.float64), (101, 101), 11), (101, 101), 11)
        pm[:10, :] = 0
        pm[-10:, :] = 0
        pm[:, :10] = 0
        pm[:, -10:] = 0
        assert np.array_equal(got, cv2.resize(pm / 255., (512, 512)))


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def test_paste_reproduces_the_fixture():
    """The face_small scenes of test_face.py through paste_faces_device: the pasted_sha of both samples."""
    from oracle import face as of
    from diffbir_b200.utils import synth
    sys.path.insert(0, str(ROOT / "tests" / "golden"))
    import gen_golden_face as gen
    from tests.golden_io import load_golden
    fx = load_golden(ROOT / "tests" / "golden", "face_small")
    det, parse = synth.synthetic_face_nets(int(fx["seed"]), class_bias=float(fx["class_bias"]))
    paths = []
    for name, hh, ww, seed in gen.SCENES:
        up = gen.scene_image(hh, ww, seed)
        h = fc.FaceRestoreHelper(DEV, detector=lambda im: of.detect_candidates(det, im),
                                 parser=lambda faces: torch.from_numpy(np.stack([of.parse_face(parse, f)
                                                                                 for f in faces])).to(DEV))
        h.read_image(up)
        h.get_face_landmarks_5(resize=640, eye_dist_threshold=5)
        h.align_warp_face()
        h.get_inverse_affine()
        per_sample = [[gen.restored_faces(c, k) for c in h.cropped_faces] for k in range(gen.N_SAMPLES)]
        masks = h.parse_faces([f for faces in per_sample for f in faces])
        assert isinstance(masks, torch.Tensor)
        outs = h.paste_faces_device([gen.restored_background(up, k) for k in range(gen.N_SAMPLES)], per_sample, masks)
        assert [_sha(o) for o in outs] == [str(s) for s in fx[name + "_pasted_sha"]], name
        paths.append(h.paste_path)
    assert "engine" in paths


def test_paste_2048_35_faces_two_samples_equals_host():
    """Overlapping and edge-cut faces on a 2048^2 photo, n_samples 2: the engine's bytes are the cv2 path's."""
    from diffbir_b200.utils.synth import synthetic_paste_scene
    helper, bgs, faces, masks = synthetic_paste_scene(2048, 35, samples=2, seed=1)
    got = helper.paste_faces_device(bgs, faces, torch.from_numpy(masks).to(DEV))
    assert helper.paste_path == "engine"
    for k in range(2):
        helper.restored_faces = list(faces[k])
        want = helper.paste_faces_to_input_image(bgs[k], list(masks[k * 35:(k + 1) * 35]))
        assert helper.paste_path == "host"
        assert np.array_equal(got[k], want), k


def test_cli_writes_the_host_paths_bytes(tmp_path, monkeypatch):
    """`--task unaligned_face --synthetic` on the engine paste and, with the parser's masks brought to numpy, on the
    cv2 paste: the same PNG bytes."""
    import inference as cli
    from PIL import Image
    from diffbir_b200.inference.unaligned_bfr_loop import UnAlignedBFRInferenceLoop
    from diffbir_b200.utils.synth import synthetic_lq
    (tmp_path / "in").mkdir()
    Image.fromarray(synthetic_lq(128, 160, seed=5)[0]).save(tmp_path / "in" / "img.png")
    args = ["--task", "unaligned_face", "--version", "v2.1", "--upscale", "4", "--sampler", "spaced", "--steps", "2",
            "--pos_prompt", "", "--neg_prompt", "low quality", "--input", str(tmp_path / "in"), "--synthetic",
            "--n_samples", "2", "--precision", "bf16" if _lib().operand_dtype() == torch.bfloat16 else "fp16"]
    cli.main(args + ["--output", str(tmp_path / "engine")])
    original = UnAlignedBFRInferenceLoop.face_networks

    def host_networks(self):
        det, parse = original(self)
        return det, lambda faces: list(parse(faces).cpu().numpy())

    monkeypatch.setattr(UnAlignedBFRInferenceLoop, "face_networks", host_networks)
    cli.main(args + ["--output", str(tmp_path / "host")])
    names = sorted(p.name for p in (tmp_path / "engine").iterdir() if p.suffix == ".png")
    assert names == ["img_0.png", "img_1.png"]
    for n in names:
        assert (tmp_path / "engine" / n).read_bytes() == (tmp_path / "host" / n).read_bytes(), n


def test_compose_of_overlapping_faces_matches_cv2():
    """The kernels chained by hand on two overlapping faces, the second cut by the frame's edge: begin, square, soft,
    parse blur, compose in face order, end -- the host paste's bytes."""
    L = _lib()
    from diffbir_b200.utils.synth import synthetic_lq
    h, w = 512, 640                     # read_image keeps a min side of 512
    helper = fc.FaceRestoreHelper(DEV, detector=lambda im: None, parser=lambda faces: None)
    helper.read_image(synthetic_lq(h, w, seed=2)[0])
    helper.inverse_affine_matrices = [np.array([[0.6, -0.1, 150.0], [0.1, 0.6, 80.0]]),
                                      np.array([[0.5, 0.2, 420.0], [-0.2, 0.5, 250.0]])]
    faces = [synthetic_lq(512, 512, seed=s)[0] for s in (3, 4)]
    masks = np.zeros((2, 512, 512), np.uint8)
    cv2.circle(masks[0], (256, 256), 200, 255, -1)
    cv2.ellipse(masks[1], (250, 270), (180, 230), 20, 0, 360, 255, -1)
    bg = synthetic_lq(h, w, seed=5)[0]
    frame = torch.empty(1, h, w, 3, dtype=torch.float64, device=DEV)
    L.paste_begin(torch.from_numpy(bg).to(DEV), frame)
    taps = torch.from_numpy(cv2.getGaussianKernel(101, 11, cv2.CV_64F).ravel()).to(DEV)
    m = torch.from_numpy(masks).to(DEV)
    pms = torch.empty(m.shape, dtype=torch.float64, device=DEV)
    L.paste_parse_blur(m, taps, torch.empty_like(pms), pms)
    for i, inv in enumerate(helper.inverse_affine_matrices):
        roi = fc.paste_roi(inv, 512, h, w)
        sq = torch.empty(roi[3], roi[2], device=DEV)
        total = torch.zeros(1, dtype=torch.float64, device=DEV)
        L.paste_square(fc.warp_map(inv), 512, h, w, roi, sq, total)
        edge = fc.paste_edge(total.item(), lambda: None)
        soft = torch.empty_like(sq)
        L.paste_soft(sq, h, w, roi, edge, torch.from_numpy(cv2.getGaussianKernel(2 * edge + 1, 0, cv2.CV_32F).ravel())
                     .to(DEV), torch.empty_like(sq), soft)
        L.paste_compose(torch.from_numpy(faces[i]).to(DEV)[None], pms[i:i + 1], sq, soft, fc.warp_map(inv), h, w, roi,
                        frame)
    out = torch.empty(1, h, w, 3, dtype=torch.uint8, device=DEV)
    L.paste_end(frame, out)
    helper.restored_faces = faces
    assert np.array_equal(out[0].cpu().numpy(), helper.paste_faces_to_input_image(bg, list(masks)))
