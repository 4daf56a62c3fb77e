"""CPU: the paste-back's engine path without a GPU -- the region-of-interest and `edge` rules, the numpy / tensor
dispatch, and a plain-numpy statement of every cv2 recipe csrc/face_paste.cu restates (fixed-point warpAffine, erode,
GaussianBlur tap order), checked against this host's cv2 on small random images."""
import sys
from fractions import Fraction
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from diffbir_b200.utils import face as fc  # noqa: E402

cv2 = pytest.importorskip("cv2")


# ---- the recipes, restated ----------------------------------------------------------------------------------------
def _px(img, y, x):
    h, w = img.shape[:2]
    ok = (y >= 0) & (y < h) & (x >= 0) & (x < w)
    v = img[np.clip(y, 0, h - 1), np.clip(x, 0, w - 1)]
    return np.where(ok[..., None] if img.ndim == 3 else ok, v, 0)


def warp(src, m, w, h):
    """cv2.warpAffine(src, m, (w, h)), bilinear, BORDER_CONSTANT 0: 1/32-pixel source positions from the inverted
    map, weights (32-fy)(32-fx)/1024 etc.; u8 in integers of 1/32768 rounded by >> 15, floats summed in tap order."""
    mi = fc.warp_map(m)
    xs, ys = np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64)
    adx, ady = np.rint(mi[0] * xs * 1024).astype(np.int64), np.rint(mi[3] * xs * 1024).astype(np.int64)
    x0, y0 = np.rint((mi[1] * ys + mi[2]) * 1024).astype(np.int64), np.rint((mi[4] * ys + mi[5]) * 1024).astype(np.int64)
    X = (x0[:, None] + 16 + adx[None]) >> 5
    Y = (y0[:, None] + 16 + ady[None]) >> 5
    ix, fx, iy, fy = X >> 5, X & 31, Y >> 5, Y & 31
    taps = [_px(src, iy, ix), _px(src, iy, ix + 1), _px(src, iy + 1, ix), _px(src, iy + 1, ix + 1)]
    wts = [(32 - fy) * (32 - fx), (32 - fy) * fx, fy * (32 - fx), fy * fx]
    if src.ndim == 3:
        wts = [t[..., None] for t in wts]
    if src.dtype == np.uint8:
        s = sum(t.astype(np.int64) * (wt * 32) for t, wt in zip(taps, wts))
        return ((s + (1 << 14)) >> 15).astype(np.uint8)
    wts = [(wt.astype(np.float32) / np.float32(1024)).astype(src.dtype) for wt in wts]
    s = taps[0] * wts[0]
    for t, wt in zip(taps[1:], wts[1:]):
        s = s + t * wt
    return s.astype(src.dtype)


def erode(img, k):
    """cv2.erode with a k x k ones kernel (k = 0: the empty kernel, 3 x 3): the minimum over [c - a, c + k - 1 - a],
    a = k // 2, of the taps inside the image."""
    lo, hi = (-(k // 2), k - 1 - k // 2) if k else (-1, 1)
    h, w = img.shape
    p = np.pad(img, ((-lo, hi), (-lo, hi)), constant_values=np.inf)
    out = np.full_like(img, np.inf)
    for dy in range(hi - lo + 1):
        for dx in range(hi - lo + 1):
            out = np.minimum(out, p[dy:dy + h, dx:dx + w])
    return out


def _fma32(a, b, c):      # a * b is exact in 64 significant bits; one more rounding to 24 bits
    return (a.astype(np.longdouble) * b + c).astype(np.float32)


_fma64 = np.frompyfunc(lambda a, b, c: float(Fraction(a) * Fraction(b) + Fraction(c)), 3, 1)


def blur(img, taps):
    """cv2.GaussianBlur with the 1-D kernel `taps`, BORDER_REFLECT_101. Rows: s = k0 x0, s = fma(k_j, x_j, s).
    Columns: s = k_r x_c, s += k_{r+i} (x_{c-i} + x_{c+i}): fused for f32 columns under 8 * (w // 8), unfused for the
    f32 columns behind them (w a multiple of 4) and for f64."""
    f32 = img.dtype == np.float32
    h, w = img.shape
    n = len(taps)
    r = n // 2
    taps = taps.astype(img.dtype)

    def refl(i, m):
        i = np.abs(i)
        return np.where(i >= m, 2 * (m - 1) - i, i)

    def fma(a, b, c):
        return _fma32(np.full_like(c, a), b, c) if f32 else _fma64(np.full_like(c, a), b, c).astype(np.float64)

    cols = refl(np.arange(w)[:, None] + np.arange(n)[None] - r, w)
    s = img[:, cols[:, 0]] * taps[0]
    for j in range(1, n):
        s = fma(taps[j], img[:, cols[:, j]], s)
    rows = np.arange(h)
    o = s * taps[r]
    fused = (np.arange(w) < w // 8 * 8) if f32 else np.zeros(w, bool)
    for i in range(1, r + 1):
        ab = s[refl(rows - i, h)] + s[refl(rows + i, h)]
        o = np.where(fused[None], fma(taps[r + i], ab, o), o + taps[r + i] * ab)
    return o


def _map(rng, scale=1.0, shift=20.0):
    a, t = rng.uniform(0.3, 1.6) * scale, rng.uniform(-np.pi, np.pi)
    return np.array([[a * np.cos(t), -a * np.sin(t), rng.uniform(-shift, shift)],
                     [a * np.sin(t), a * np.cos(t), rng.uniform(-shift, shift)]])


@pytest.mark.parametrize("seed", range(6))
def test_warp_affine_recipe_matches_cv2(seed):
    rng = np.random.default_rng(seed)
    m = _map(rng)
    if seed == 5:       # translations on 1/32 boundaries: the rounding of X0 + 16 decides the tap
        m = np.array([[1.0, 0.0, 3 + 1 / 64], [0.0, 1.0, -2 - 3 / 64]])
    for src in (rng.integers(0, 256, (37, 41, 3)).astype(np.uint8), rng.random((37, 41)).astype(np.float32),
                np.ones((37, 41), np.float32), rng.random((37, 41))):
        assert np.array_equal(cv2.warpAffine(src, m, (60, 52)), warp(src, m, 60, 52)), src.dtype
    pm = rng.random((64, 64))
    assert np.array_equal(cv2.warpAffine(pm, m, (70, 66), flags=3), warp(pm, m, 70, 66))     # INTER_AREA: bilinear


@pytest.mark.parametrize("k", [0, 2, 3, 6, 10])
def test_erode_recipe_matches_cv2(k):
    rng = np.random.default_rng(k)
    img = rng.random((30, 44)).astype(np.float32)
    img[:4] = 1.0
    img[:, -3:] = 1.0                   # the image border never lowers the minimum
    assert np.array_equal(cv2.erode(img, np.ones((k, k), np.uint8)), erode(img, k))


@pytest.mark.parametrize("n,w", [(7, 60), (9, 44), (15, 64), (41, 84)])
def test_gaussian_blur_f32_recipe_matches_cv2(n, w):
    rng = np.random.default_rng(n)
    img = ((rng.random((n + 12, w)) < 0.7) * rng.random((n + 12, w))).astype(np.float32)
    taps = cv2.getGaussianKernel(n, 0, cv2.CV_32F).ravel()
    assert np.array_equal(cv2.GaussianBlur(img, (n, n), 0), blur(img, taps))


def test_gaussian_blur_f64_recipe_matches_cv2():
    rng = np.random.default_rng(1)
    img = rng.integers(0, 2, (112, 128)).astype(np.float64) * 255
    taps = cv2.getGaussianKernel(101, 11, cv2.CV_64F).ravel()
    assert np.array_equal(cv2.GaussianBlur(img, (101, 101), 11), blur(img, taps))


# ---- region of interest, edge and dispatch ------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(4))
def test_roi_holds_everything_a_face_changes(seed):
    """Outside paste_roi the warped square, its soft mask and the warped parse mask are exactly 0, including for a
    face cut by the frame's edge."""
    rng = np.random.default_rng(seed)
    h, w, fs = 120, 160, 64
    inv = _map(rng, 1.0, 0.0)
    inv[:, 2] = [rng.uniform(-30, w), rng.uniform(-30, h)]
    roi = fc.paste_roi(inv, fs, h, w)
    square = cv2.erode(cv2.warpAffine(np.ones((fs, fs), np.float32), inv, (w, h)), np.ones((2, 2), np.uint8))
    edge = int(np.sum(square) ** 0.5) // 20
    soft = cv2.GaussianBlur(cv2.erode(square, np.ones((2 * edge, 2 * edge), np.uint8)), (2 * edge + 1,) * 2, 0)
    pm = cv2.warpAffine(np.ones((fs, fs)), inv, (w, h), flags=3)
    inside = np.zeros((h, w), bool)
    if roi is not None:
        x0, y0, rw, rh = roi
        inside[y0:y0 + rh, x0:x0 + rw] = True
    for a in (square, soft, pm):
        assert not a[~inside].any()


def test_edge_uses_numpy_near_a_step():
    calls = []

    def frame():
        calls.append(1)
        return np.full((20, 20), 0.999, np.float32)          # numpy's sum: under 400

    assert fc.paste_edge(123456.7, frame) == int(123456.7 ** 0.5) // 20 and not calls
    assert fc.paste_edge(400.0, frame) == 0 and calls        # at (20 k)^2 numpy's own sum decides
    assert fc.paste_edge(1600.0 * 1.00001, lambda: np.ones((40, 40), np.float32)) == 2


def _helper(parser_out):
    h = fc.FaceRestoreHelper("cpu", detector=lambda im: None, parser=lambda faces: parser_out)
    h.read_image(np.zeros((512, 640, 3), np.uint8))
    h.inverse_affine_matrices = [cv2.invertAffineTransform(np.array([[0.5, 0.0, 40.0], [0.0, 0.5, 30.0]]))]
    return h


def test_numpy_takes_cv2_and_tensors_take_the_engine(monkeypatch):
    h = _helper([np.full((512, 512), 255, np.uint8)])
    h.add_restored_face(np.full((512, 512, 3), 200, np.uint8))
    bg = np.full((512, 640, 3), 10, np.uint8)
    out = h.paste_faces_to_input_image(bg)
    assert h.paste_path == "host" and out.shape == bg.shape and out[100, 100, 0] == 200
    seen = []
    monkeypatch.setattr(fc.FaceRestoreHelper, "paste_faces_device",
                        lambda self, imgs, faces, masks: seen.append((len(imgs), len(faces[0]), type(masks))) or [bg])
    h2 = _helper(torch.full((1, 512, 512), 255, dtype=torch.uint8))
    h2.add_restored_face(np.full((512, 512, 3), 200, np.uint8))
    assert isinstance(h2.parse_faces(h2.restored_faces), torch.Tensor)
    h2.paste_faces_to_input_image(bg)
    assert seen == [(1, 1, torch.Tensor)]


def test_unrestated_geometry_takes_the_cv2_recipe():
    """A frame width that is not a multiple of 4 has cv2 tap orders the kernels do not restate: the engine entry
    point pastes it with the cv2 recipe (no device is touched) and says so."""
    h = _helper(None)
    h.input_img = np.zeros((512, 642, 3), np.uint8)
    face = np.full((512, 512, 3), 200, np.uint8)
    bg = np.full((512, 642, 3), 10, np.uint8)
    masks = torch.full((1, 512, 512), 255, dtype=torch.uint8)
    out = h.paste_faces_device([bg], [[face]], masks)[0]
    assert h.paste_path == "host"
    h.add_restored_face(face)
    assert np.array_equal(out, h.paste_faces_to_input_image(bg, [masks[0].numpy()]))
