"""CPU: the unaligned-face loop's surface -- facexlib key layouts and strict loaders, the detector post-processing,
the host face helper on the fp32 oracle networks, and UnAlignedBFRInferenceLoop with stub pipelines."""
import csv
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
from PIL import Image

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import inference as cli  # noqa: E402
from diffbir_b200 import arch  # noqa: E402
from diffbir_b200.inference.pretrained_models import resolve  # noqa: E402
from diffbir_b200.utils import synth  # noqa: E402
from diffbir_b200.utils.face import FaceRestoreHelper, nms, select_faces  # noqa: E402

cv2 = pytest.importorskip("cv2")


def test_shape_tables_follow_facexlib():
    r = arch.retinaface_shapes()
    assert r["body.conv1.weight"] == (64, 3, 7, 7) and r["body.layer2.0.conv2.weight"] == (128, 128, 3, 3)
    assert r["body.layer4.0.downsample.0.weight"] == (2048, 1024, 1, 1) and "body.layer4.1.downsample.0.weight" not in r
    assert r["fpn.output3.0.weight"] == (256, 2048, 1, 1) and r["fpn.merge1.1.running_var"] == (256,)
    assert r["ssh2.conv7x7_3.0.weight"] == (64, 64, 3, 3) and r["ssh1.conv3X3.0.weight"] == (128, 256, 3, 3)
    assert (r["ClassHead.2.conv1x1.weight"], r["BboxHead.0.conv1x1.bias"], r["LandmarkHead.1.conv1x1.weight"]) == \
        ((4, 256, 1, 1), (8,), (20, 256, 1, 1))
    assert sum(int(np.prod(s)) for s in r.values()) == 27351584          # resnet50 body + FPN + SSH + heads
    p = arch.parsenet_shapes()
    assert p["encoder.0.conv2d.bias"] == (64,) and p["encoder.3.shortcut_func.conv2d.weight"] == (256, 256, 3, 3)
    assert "body.0.shortcut_func.conv2d.weight" not in p and p["body.9.conv2.norm.norm.weight"] == (256,)
    assert p["decoder.3.conv1.conv2d.weight"] == (64, 128, 3, 3) and "decoder.3.conv1.conv2d.bias" not in p
    assert p["out_mask_conv.conv2d.weight"] == (19, 64, 3, 3) and p["out_img_conv.conv2d.bias"] == (3,)


def test_strict_loaders_strip_prefix_and_name_bad_keys():
    sd = synth.make_state_dict(arch.parsenet_shapes(), 1)
    ck = {"module." + k: v for k, v in sd.items()}
    ck["module.encoder.1.conv1.norm.norm.num_batches_tracked"] = torch.tensor(7)
    out = arch.parsenet_state_dict(ck)
    assert set(out) == set(sd)
    bad = dict(sd)
    del bad["body.3.conv1.conv2d.weight"]
    bad["body.3.extra"] = torch.zeros(1)
    bad["encoder.0.conv2d.bias"] = torch.zeros(3)
    with pytest.raises(ValueError, match=r"body\.3\.conv1\.conv2d\.weight.*body\.3\.extra.*encoder\.0\.conv2d\.bias"):
        arch.parsenet_state_dict(bad)
    det = synth.make_state_dict(arch.retinaface_shapes(), 2)
    assert set(arch.retinaface_state_dict({"state_dict": det})) == set(det)


def test_bn_fold_matches_eval_batchnorm():
    g = torch.Generator().manual_seed(0)
    w = torch.randn(8, 4, 3, 3, generator=g)
    sd = {"bn.weight": torch.rand(8, generator=g) + 0.5, "bn.bias": torch.randn(8, generator=g),
          "bn.running_mean": torch.randn(8, generator=g), "bn.running_var": torch.rand(8, generator=g) + 0.5}
    x = torch.randn(2, 4, 9, 9, generator=g, dtype=torch.float64)
    wf, bf = arch.fold_bn(w, sd, "bn")
    ref = torch.nn.functional.batch_norm(torch.nn.functional.conv2d(x, w.double()), sd["bn.running_mean"].double(),
                                         sd["bn.running_var"].double(), sd["bn.weight"].double(), sd["bn.bias"].double(),
                                         False, 0.0, 1e-5)
    assert torch.allclose(torch.nn.functional.conv2d(x, wf.double(), bf.double()), ref, atol=1e-5)


def test_registry_keys_resolve_locally(tmp_path):
    for key, name in (("retinaface_resnet50", "detection_Resnet50_Final.pth"), ("parsenet", "parsing_parsenet.pth")):
        with pytest.raises(FileNotFoundError, match=name):
            resolve(key, str(tmp_path))
        (tmp_path / name).write_bytes(b"x")
        assert resolve(key, str(tmp_path)).endswith(name)


def _lq():
    return Image.fromarray(synth.synthetic_lq(128, 160, seed=5)[0])


@pytest.fixture(scope="module")
def oracle_nets():
    from oracle import face as of
    det, parse = synth.synthetic_face_nets(231)
    return of, det, parse


def test_nms_matches_torchvision(oracle_nets):
    tv = pytest.importorskip("torchvision")
    of, det, _ = oracle_nets
    img = cv2.resize(np.array(_lq().resize((640, 512), Image.BICUBIC)), (800, 640), interpolation=cv2.INTER_LINEAR)
    boxes, scores, _ = of.detect_candidates(det, img)
    top = torch.argsort(scores, descending=True)[:600]           # the densest part: overlapping strong priors
    for thr in (0.4, 0.2, 0.7):
        assert torch.equal(nms(boxes[top], scores[top], thr), tv.ops.nms(boxes[top], scores[top], thr))
        assert torch.equal(of.nms_reference(boxes[top], scores[top], thr), tv.ops.nms(boxes[top], scores[top], thr))


def test_helper_on_oracle_nets_detects_aligns_and_pastes(oracle_nets):
    """The calibrated synthetic detector finds 1-4 faces in the loop's test input; each crop is the LMEDS similarity
    warp of its landmarks; pasting touches nothing outside the warped face squares."""
    of, det, parse = oracle_nets
    h = FaceRestoreHelper("cpu", detector=lambda im: of.detect_candidates(det, im),
                          parser=lambda faces: [of.parse_face(parse, f) for f in faces])
    up = np.array(_lq().resize((640, 512), Image.BICUBIC))
    h.read_image(up)
    assert h.input_img.shape == (512, 640, 3)
    n = h.get_face_landmarks_5(resize=640, eye_dist_threshold=5)
    h.align_warp_face()
    assert 1 <= n <= 4 and len(h.cropped_faces) == n and all(f.shape == (512, 512, 3) for f in h.cropped_faces)
    ref = of.detect_faces(det, cv2.resize(h.input_img, (800, 640), interpolation=cv2.INTER_LINEAR)) / 1.25
    ref = np.stack([r for r in ref if np.linalg.norm([r[6] - r[8], r[7] - r[9]]) >= 5])
    assert np.array_equal(np.stack(h.det_faces), ref[:, :5])
    h.get_inverse_affine()
    bg = np.full((512, 640, 3), 77, np.uint8)
    for f in h.cropped_faces:
        h.add_restored_face(f)
    out = h.paste_faces_to_input_image(bg)
    assert out.shape == (512, 640, 3) and out.dtype == np.uint8
    union = np.zeros(out.shape[:2], np.float32)
    for inv in h.inverse_affine_matrices:
        union = np.maximum(union, cv2.warpAffine(np.ones((512, 512), np.float32), inv, (640, 512)))
    assert np.array_equal(out[union == 0], cv2.resize(bg, (640, 512), interpolation=cv2.INTER_LANCZOS4)[union == 0])


def test_helper_reproduces_the_reference_fixture():
    """face_small.npz comes from the reference's own FaceRestoreHelper with facexlib backed by the fp32 oracle nets
    (tests/golden/gen_golden_face.py). The product helper on the same nets reproduces it bit for bit: detections, kept
    faces, affine matrices, crops, parse masks and the pasted image of both samples, in a scene that read_image up-sizes
    and in one that only the detection up-sizes."""
    import hashlib
    from oracle import face as of
    sys.path.insert(0, str(ROOT / "tests" / "golden"))
    import gen_golden_face as gen
    from tests.golden_io import load_golden
    fx = load_golden(ROOT / "tests" / "golden", "face_small")
    det, parse = synth.synthetic_face_nets(int(fx["seed"]), class_bias=float(fx["class_bias"]))

    def sha(a):
        return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()

    for name, hh, ww, seed in gen.SCENES:
        p = name + "_"
        up = gen.scene_image(hh, ww, seed)
        assert sha(up) == str(fx[p + "input_sha"])
        h = FaceRestoreHelper("cpu", detector=lambda im: of.detect_candidates(det, im),
                              parser=lambda faces: [of.parse_face(parse, f) for f in faces])
        h.read_image(up)
        assert h.input_img.shape == tuple(fx[p + "input_img_shape"])
        img, _ = gen.detection_image(up)
        assert np.array_equal(h.detect_faces(img), fx[p + "detections"])
        h.get_face_landmarks_5(resize=640, eye_dist_threshold=5)
        h.align_warp_face()
        assert np.array_equal(np.stack(h.det_faces), fx[p + "det_faces"])
        assert np.array_equal(np.stack(h.all_landmarks_5), fx[p + "landmarks"])
        assert np.array_equal(np.stack(h.affine_matrices), fx[p + "affine"])
        assert [sha(c) for c in h.cropped_faces] == list(fx[p + "crop_sha"])
        h.get_inverse_affine()
        per_sample = [[gen.restored_faces(c, k) for c in h.cropped_faces] for k in range(gen.N_SAMPLES)]
        masks = h.parse_faces([f for faces in per_sample for f in faces])
        assert np.array_equal(np.packbits(np.stack(masks) > 0, axis=-1), fx[p + "parse_bits"])
        n = len(h.cropped_faces)
        for k, faces in enumerate(per_sample):
            for f in faces:
                h.add_restored_face(f)
            out = h.paste_faces_to_input_image(gen.restored_background(up, k), masks[k * n:(k + 1) * n])
            assert sha(out) == str(fx[p + "pasted_sha"][k]), (name, k)
            h.restored_faces.clear()


def test_select_faces_threshold_order_and_nms():
    boxes = torch.tensor([[0, 0, 10, 10], [1, 1, 11, 11], [50, 50, 60, 60], [0, 0, 5, 5]], dtype=torch.float32)
    scores = torch.tensor([0.85, 0.95, 0.9, 0.5])
    lm = torch.arange(40, dtype=torch.float32).view(4, 10)
    rows = select_faces(boxes, scores, lm)
    assert rows.dtype == np.float32 and rows.shape == (2, 15)
    assert rows[:, 4].tolist() == pytest.approx([0.95, 0.9]) and rows[0, 5] == 10 and rows[1, 5] == 20
    # equal scores: facexlib's argsort()[::-1] visits the later index first, so NMS keeps that box
    tied = select_faces(boxes[:2], torch.tensor([0.9, 0.9]), lm[:2])
    assert tied.shape == (1, 15) and tied[0, 5] == 10


# ---- the loop with stub pipelines -----------------------------------------------------------------------------
class StubPipeline:
    def __init__(self, name, calls):
        self.name, self.calls = name, calls

    def run(self, *a):
        lq = a[0]
        self.calls.append((self.name, lq.shape))
        return np.stack([np.full(lq.shape[1:], 20 * len(self.calls) + i, dtype=np.uint8) for i in range(lq.shape[0])])


def make_loop(tmp_path, faces, *extra):
    from diffbir_b200.inference.unaligned_bfr_loop import UnAlignedBFRInferenceLoop
    args = cli.parse_args(["--input", str(tmp_path / "in"), "--output", str(tmp_path / "out"), "--task",
                           "unaligned_face", "--pos_prompt", "p", "--neg_prompt", "n", *extra])
    lp = UnAlignedBFRInferenceLoop.__new__(UnAlignedBFRInferenceLoop)     # skip model loading (needs the GPU library)
    lp.args, lp.loop_ctx, lp.pipeline, lp.calls = args, {}, None, []
    lp.bg_requires_upscale = args.version == "v2.1"
    lp.pipeline_dict = {"background": StubPipeline("bg", lp.calls), "face": StubPipeline("face", lp.calls)}

    def detector(img):            # `faces` fixed detections in the detection image's pixels
        boxes = torch.tensor([f[:4] for f in faces], dtype=torch.float32).view(-1, 4)
        lms = torch.tensor([f[4:] for f in faces], dtype=torch.float32).view(-1, 10)
        return boxes, torch.full((len(faces),), 0.9), lms

    lp.face_networks = lambda: (detector, lambda fs: [np.full((512, 512), 255, np.uint8) for _ in fs])
    return lp


def _face(cx, cy, s):
    t = (np.array([[193, 240], [319, 240], [257, 314], [201, 371], [313, 371]]) - 256) * s / 512
    return [cx - s / 2, cy - s / 2, cx + s / 2, cy + s / 2] + list((t + [cx, cy]).reshape(-1))


@pytest.mark.parametrize("version", ["v2.1", "v2"])
def test_loop_yields_faces_then_background_and_saves(tmp_path, version):
    (tmp_path / "in").mkdir()
    Image.fromarray(np.zeros((160, 200, 3), np.uint8)).save(tmp_path / "in" / "pic.png")
    faces = [_face(200, 300, 200), _face(600, 300, 160)]          # in the 640 x 800 detection image
    lp = make_loop(tmp_path, faces, "--version", version, "--n_samples", "2", "--upscale", "2")
    lp.run()
    kinds = [c[0] for c in lp.calls]
    assert kinds == ["face"] * 4 + ["bg"] * 2                  # faces first; n_samples 2 at batch size 1
    assert lp.calls[0][1] == (1, 512, 512, 3)
    assert lp.calls[4][1] == ((1, 320, 400, 3) if version == "v2.1" else (1, 160, 200, 3))   # v2.1 up-scales first
    out = tmp_path / "out"
    assert sorted(p.name for p in (out / "restored_faces").iterdir()) == \
        ["pic_face_0_0.png", "pic_face_0_1.png", "pic_face_1_0.png", "pic_face_1_1.png"]
    assert sorted(p.name for p in (out / "cropped_faces").iterdir()) == ["pic_face_0_1.png", "pic_face_1_1.png"]
    assert sorted(p.name for p in (out / "restored_backgrounds").iterdir()) == ["pic_0.png", "pic_1.png"]
    assert sorted(p.name for p in out.iterdir() if p.is_file()) == ["pic_0.png", "pic_1.png", "prompt.csv"]
    rows = list(csv.reader(open(out / "prompt.csv")))
    assert rows == [["file_name", "pos_prompt", "neg_prompt"], ["pic_face_0", "p", "n"], ["pic_face_1", "p", "n"],
                    ["pic", "p", "n"]]
    # the pasted photo has the detection image's size (read_image brought 320 x 400 to a min side of 512)
    assert np.array(Image.open(out / "pic_1.png")).shape == (512, 640, 3)
    # sample k of the photo receives sample k of every face (the transposition): stub value 20 x call number
    helper_faces = [[int(f[0, 0, 0]) for f in faces] for faces in map(list, zip(*lp.face_samples))]
    assert helper_faces == [[20, 60], [40, 80]]


def test_loop_without_faces_writes_no_png(tmp_path):
    (tmp_path / "in").mkdir()
    Image.fromarray(np.zeros((40, 50, 3), np.uint8)).save(tmp_path / "in" / "empty.png")
    lp = make_loop(tmp_path, [])
    lp.run()
    out = tmp_path / "out"
    assert [c[0] for c in lp.calls] == ["bg"]
    assert not list(out.rglob("*.png"))
    assert list(csv.reader(open(out / "prompt.csv")))[1:] == [["empty", "p", "n"]]


def test_v1_is_refused_before_the_models(tmp_path, monkeypatch):
    from diffbir_b200.inference.unaligned_bfr_loop import UnAlignedBFRInferenceLoop
    args = cli.parse_args(["--input", "x", "--output", "y", "--task", "unaligned_face", "--version", "v1"])
    monkeypatch.setattr(UnAlignedBFRInferenceLoop, "load_cldm", lambda self: pytest.fail("load_cldm before cleaner"))
    with pytest.raises(ValueError, match="doesn't support unaligned BFR"):
        UnAlignedBFRInferenceLoop(args)


def test_cli_dispatches_unaligned_face(monkeypatch):
    import diffbir_b200.inference as inf
    seen = []

    class Recorder:
        def __init__(self, args):
            seen.append(args.task)

        def run(self):
            seen.append("run")

    monkeypatch.setattr(inf, "UnAlignedBFRInferenceLoop", Recorder)
    monkeypatch.setattr(cli.torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(cli, "set_seed", lambda s: None)
    cli.main(["--input", "x", "--output", "y", "--task", "unaligned_face"])
    assert seen == ["unaligned_face", "run"]
    import diffbir.inference as di
    with pytest.raises(NotImplementedError, match="--task unaligned_face"):
        di.UnAlignedBFRInferenceLoop()
