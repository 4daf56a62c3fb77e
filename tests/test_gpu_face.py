"""-m gpu: the unaligned-face loop's kernels against fp64 references, RetinaFaceEngine / ParseNetEngine against the fp32
oracle (TF32 off), the paste with engine masks, and `--task unaligned_face` end to end on synthetic weights."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from tests.gpu_util import no_tf32, rel_rms, to_dev  # noqa: E402

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
DEV = "cuda"


def _lib():
    from diffbir_b200 import lib
    lib.load()
    return lib


def _op(t):
    return t.to(DEV, _lib().operand_dtype())


# ---- kernels --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c,ksize,stride,reflect,up2,h,w", [(3, 7, 2, False, False, 37, 50), (64, 3, 2, False, False, 33, 20),
                                                            (64, 3, 1, True, False, 17, 23), (128, 3, 2, True, False, 32, 32),
                                                            (128, 3, 1, True, True, 9, 14), (64, 1, 2, False, False, 41, 63),
                                                            (3, 3, 1, True, False, 16, 16)])
def test_patch_gather(c, ksize, stride, reflect, up2, h, w):
    L = _lib()
    g = torch.Generator().manual_seed(c + ksize + h)
    x = torch.randn(2, h, w, c, generator=g)
    x16 = _op(x)
    ho, wo = L.patch_gather_shape(h, w, ksize, stride, up2)
    kp = (ksize * ksize * c + 63) // 64 * 64
    out = torch.full((2 * ho * wo, kp), 7.0, device=DEV, dtype=L.operand_dtype())
    L.patch_gather(x16, c, 2, h, w, c, ksize, stride, kp, out, reflect=reflect, up2=up2)
    src = x16.double().cpu().permute(0, 3, 1, 2)
    if up2:
        src = F.interpolate(src, scale_factor=2, mode="nearest")
    p = ksize // 2
    src = F.pad(src, (p, p, p, p), mode="reflect" if reflect else "constant")
    ref = F.unfold(src, ksize, stride=stride)                                   # [n, c*k*k, L], c-major
    ref = ref.view(2, c, ksize * ksize, -1).permute(0, 3, 2, 1).reshape(2 * ho * wo, ksize * ksize * c)
    got = out.double().cpu()
    assert torch.equal(got[:, :ksize * ksize * c], ref) and not got[:, ksize * ksize * c:].any()


def test_maxpool_fpn_add_relu_cast_and_input():
    L = _lib()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(1, 325, 500, 64, generator=g)
    x16 = _op(x)
    out = torch.empty(163 * 250, 64, device=DEV, dtype=L.operand_dtype())
    L.maxpool3s2(x16, 1, 325, 500, 64, out)
    ref = F.max_pool2d(x16.double().cpu().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1).reshape(-1, 64)
    assert torch.equal(out.double().cpu(), ref)
    for (h, w), (hb, wb) in (((82, 125), (41, 63)), ((41, 63), (21, 32)), ((64, 64), (32, 32)), ((13, 7), (13, 7))):
        a = torch.randn(h * w, 256, generator=g).to(DEV)
        b = _op(torch.randn(hb * wb, 256, generator=g))
        o = torch.empty(h * w, 256, device=DEV, dtype=L.operand_dtype())
        L.fpn_add_up(a, b, 1, h, w, hb, wb, 256, o)
        up = F.interpolate(b.float().cpu().view(1, hb, wb, 256).permute(0, 3, 1, 2), size=(h, w), mode="nearest")
        refo = (a.cpu() + up.permute(0, 2, 3, 1).reshape(-1, 256)).to(L.operand_dtype())
        assert torch.equal(o.cpu(), refo), (h, w, hb, wb)
    z = torch.randn(1000, 64, generator=g).to(DEV)
    y16 = torch.empty(1000, 64, device=DEV, dtype=L.operand_dtype())
    y = torch.empty_like(z)
    L.relu_cast(z, z.numel(), y16, y=y)
    assert torch.equal(y, z.clamp(min=0)) and torch.equal(y16, z.clamp(min=0).to(L.operand_dtype()))
    img = torch.randint(0, 256, (2, 5, 7, 3), dtype=torch.uint8, generator=g)
    o = torch.empty(70, 3, device=DEV, dtype=L.operand_dtype())
    L.face_input(img.to(DEV), 2, 5, 7, o, shift=(104.0, 117.0, 123.0))
    assert torch.equal(o.double().cpu(), (img.double() - torch.tensor([104.0, 117.0, 123.0])).view(-1, 3))
    L.face_input(img.to(DEV), 2, 5, 7, o, scale=1 / 255, shift=(0.5, 0.5, 0.5), div=0.5, reverse=True)
    ref = ((img.flip(-1).double() / 255 - 0.5) / 0.5).view(-1, 3)
    assert (o.double().cpu() - ref).abs().max() < 1e-2


@pytest.mark.parametrize("h,w", [(640, 640), (650, 1000), (97, 131)])
def test_retinaface_decode_and_parse_mask(h, w):
    L = _lib()
    from oracle import face as of
    g = torch.Generator().manual_seed(h)
    rows = sum(((h + s - 1) // s) * ((w + s - 1) // s) for s in (8, 16, 32))
    head = torch.randn(rows, 32, generator=g)
    out = torch.empty(2 * rows, 15, device=DEV)
    L.retinaface_decode(head.to(DEV), h, w, out)
    loc, conf, lm = head[:, 4:12].reshape(-1, 4), head[:, :4].reshape(-1, 2), head[:, 12:].reshape(-1, 10)
    boxes, scores, lms = of.decode(loc.double(), conf.double(), lm.double(), h, w)
    ref = torch.cat([boxes, scores[:, None], lms], 1)
    assert (out.double().cpu() - ref).abs().max() < 1e-3 * max(h, w)
    logits = torch.randn(5000, 32, generator=g)
    logits[:100, 3] = logits[:100, 14] = 9.0                                    # ties: the first maximum wins
    m = torch.empty(5000, dtype=torch.uint8, device=DEV)
    L.parse_mask(logits.to(DEV), 32, 5000, 19, m)
    lut = torch.tensor(of.MASK_COLORMAP, dtype=torch.uint8)
    assert torch.equal(m.cpu(), lut[logits[:, :19].argmax(1)])


# ---- engines --------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def nets():
    return _nets_cache()


def _image(h, w, seed):
    from diffbir_b200.utils.synth import synthetic_lq
    return synthetic_lq(h, w, seed=seed)[0]


@pytest.mark.parametrize("h,w", [(640, 640), (768, 1024), (650, 1000)])
def test_retinaface_engine_matches_oracle(h, w):
    no_tf32()
    from oracle import face as of
    from diffbir_b200.utils.face import select_faces
    from diffbir_b200.utils.synth import synthetic_face_nets
    det, _ = synthetic_face_nets(231, class_bias=-1.0)        # a few faces on these test images
    eng = _detector_for_test(det)
    bf16 = _lib().operand_dtype() == torch.bfloat16
    img = _image(h, w, h + w)
    head = eng.heads(img).cpu()
    sd = to_dev(det)
    x = (torch.from_numpy(img).to(DEV).float() - torch.tensor(of.DETECTOR_MEAN, device=DEV)).permute(2, 0, 1)[None]
    with torch.no_grad():
        loc, conf, lm = of.retinaface_forward(sd, x.contiguous())
    got = torch.cat([head[:, :4].reshape(-1, 2), head[:, 4:12].reshape(-1, 4), head[:, 12:].reshape(-1, 10)], 1)
    ref = torch.cat([conf[0], loc[0], lm[0]], 1).cpu()
    err = rel_rms(got, ref)
    print(f"RetinaFace {h}x{w}: head rel-RMS {err:.2e}")
    assert err <= (5e-2 if bf16 else 1e-2)
    rb, rs, rl = of.decode(loc[0], conf[0], lm[0], h, w)
    gb, gs, gl = eng.candidates(img)
    clear = (rs - 0.8).abs() >= 0.02
    assert torch.equal((gs > 0.8)[clear], (rs > 0.8)[clear])
    a, b = select_faces(gb, gs, gl), select_faces(rb, rs, rl)
    bar = 2.0 if bf16 else 0.5

    def nearest(row, rows):                     # landmark error to the closest face of the other list (any order)
        return np.abs(rows[:, 5:] - row[5:]).max(axis=1).min() if len(rows) else np.inf

    # the kept faces are the same wherever the scores are clear of the threshold: every oracle face scoring >= 0.82 is
    # kept by the engine and every engine face scoring >= 0.82 is kept by the oracle, landmarks within the bar
    clear_b = [r for r in b if r[4] >= 0.82]
    clear_a = [r for r in a if r[4] >= 0.82]
    assert clear_b, "the test image must yield a face"
    err = max([nearest(r, a) for r in clear_b] + [nearest(r, b) for r in clear_a])
    print(f"  {len(a)} / {len(b)} faces (engine / oracle), {len(clear_b)} clear; landmark max error {err:.3f} px")
    assert err <= bar


def test_parsenet_engine_matches_oracle_and_batches_exactly(nets):
    no_tf32()
    from oracle import face as of
    _, parse, _, eng = nets
    faces = [_image(512, 512, s) for s in range(6)]
    batch = eng.masks(faces)                                   # two forwards: 4 + 2 faces
    singles = [eng.masks([f])[0] for f in faces]
    assert all(np.array_equal(a, b) for a, b in zip(batch, singles))
    sd = to_dev(parse)
    agree = np.mean([np.mean(m == of.parse_face(sd, f)) for m, f in zip(batch, faces)])
    print(f"ParseNet mask agreement with the oracle: {agree:.5f}")
    if _lib().operand_dtype() == torch.float16:
        assert agree >= 0.995


def test_paste_with_engine_masks_matches_oracle_masks(nets):
    from oracle import face as of
    from diffbir_b200.utils.face import FaceRestoreHelper
    det, parse, deng, peng = nets
    sd = to_dev(parse)
    from PIL import Image
    img = np.array(Image.fromarray(_image(128, 160, 5)).resize((640, 512), Image.BICUBIC))   # the CLI test's photo
    bg = _image(512, 640, 9)
    out = {}
    for name, parser in (("engine", peng.masks), ("oracle", lambda fs: [of.parse_face(sd, f) for f in fs])):
        h = FaceRestoreHelper(DEV, detector=deng.candidates, parser=parser)
        h.read_image(img)
        h.get_face_landmarks_5(resize=640, eye_dist_threshold=5)
        h.align_warp_face()
        h.get_inverse_affine()
        for f in h.cropped_faces:
            h.add_restored_face(255 - f)
        assert h.restored_faces
        out[name] = h.paste_faces_to_input_image(bg).astype(np.float64)
    mse = ((out["engine"] - out["oracle"]) ** 2).mean()
    psnr = float("inf") if mse == 0 else 10 * np.log10(255.0 ** 2 / mse)
    print(f"paste with engine vs oracle masks: {psnr:.1f} dB")
    assert psnr >= 50.0


# ---- command line ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("version", ["v2.1", "v2"])
def test_cli_unaligned_face_end_to_end(tmp_path, version):
    import inference as cli
    from PIL import Image
    from diffbir_b200.utils.face import FaceRestoreHelper
    (tmp_path / "in").mkdir()
    lq = _image(128, 160, 5)                                   # x4 = 512 x 640: read_image keeps the size
    Image.fromarray(lq).save(tmp_path / "in" / "img.png")
    cli.main(["--task", "unaligned_face", "--version", version, "--upscale", "4", "--sampler", "spaced", "--steps", "2",
              "--pos_prompt", "", "--neg_prompt", "low quality", "--input", str(tmp_path / "in"), "--output",
              str(tmp_path / "out"), "--synthetic", "--precision",
              "bf16" if _lib().operand_dtype() == torch.bfloat16 else "fp16"])
    out = tmp_path / "out"
    faces = sorted(p.name for p in (out / "restored_faces").iterdir())
    assert 1 <= len(faces) <= 4, faces
    assert faces == [f"img_face_{i}_0.png" for i in range(len(faces))]
    assert sorted(p.name for p in (out / "cropped_faces").iterdir()) == faces
    assert all(np.array(Image.open(out / "restored_faces" / f)).shape == (512, 512, 3) for f in faces)
    bg = np.array(Image.open(out / "restored_backgrounds" / "img_0.png"))
    res = np.array(Image.open(out / "img_0.png"))
    assert bg.shape == res.shape == (512, 640, 3)
    assert len(list(open(out / "prompt.csv"))) == 1 + len(faces) + 1
    # outside the union of the warped face squares the mask is 0 and a same-size Lanczos resize is a copy
    _, _, deng, peng = _nets_cache()
    h = FaceRestoreHelper(DEV, detector=deng.candidates, parser=peng.masks)
    h.read_image(np.array(Image.fromarray(lq).resize((640, 512), Image.BICUBIC)))
    assert h.get_face_landmarks_5(resize=640, eye_dist_threshold=5) == len(faces)
    h.align_warp_face()
    h.get_inverse_affine()
    union = np.zeros((512, 640), np.float32)
    for inv in h.inverse_affine_matrices:
        union = np.maximum(union, cv2.warpAffine(np.ones((512, 512), np.float32), inv, (640, 512)))
    assert (union == 0).mean() > 0.2 and np.array_equal(res[union == 0], bg[union == 0])


_CACHE = {}


def _detector_for_test(det):
    if "det_test" not in _CACHE:
        from diffbir_b200.engine.retinaface import RetinaFaceEngine
        _CACHE["det_test"] = RetinaFaceEngine(det, device=DEV)
    return _CACHE["det_test"]


def _nets_cache():
    if "v" not in _CACHE:
        from diffbir_b200.engine.parsenet import ParseNetEngine
        from diffbir_b200.engine.retinaface import RetinaFaceEngine
        from diffbir_b200.utils.synth import synthetic_face_nets
        det, parse = synthetic_face_nets(231)
        _CACHE["v"] = (det, parse, RetinaFaceEngine(det, device=DEV), ParseNetEngine(parse, device=DEV))
    return _CACHE["v"]
