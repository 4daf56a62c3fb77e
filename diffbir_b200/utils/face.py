"""Face detection, alignment and paste-back of the unaligned-face loop.

Restates the part of the reference's FaceRestoreHelper (diffbir/utils/face.py) that UnAlignedBFRInferenceLoop
reaches: upscale_factor 1, 512 faces on the 5-point FFHQ template, the retinaface_resnet50 detector with its
(resize=640, eye_dist_threshold=5) landmarks, the square soft mask and the ParseNet mask. Geometry and blending
use cv2 exactly as the reference does, so the same detections and restored faces give the same bytes.

The two networks are callables, so tests can plug in the fp32 oracle:
- detector(img uint8 HWC) -> (boxes [P, 4], scores [P], landmarks [P, 10]) of every prior, fp32 tensors;
- parser(faces: list of uint8 512x512x3 RGB) -> list of uint8 512x512 masks in {0, 255}.
The inference loop passes the sm_90a engines (RetinaFaceEngine.candidates, ParseNetEngine.masks). The score threshold
runs in torch on the device the candidates live on; the ordering and the NMS run on the CPU copy of the candidates
above the threshold (a handful per photo), as facexlib does.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence

import numpy as np
import torch

FACE_TEMPLATE_512 = np.array([[192.98138, 239.94708], [318.90277, 240.1936], [256.63416, 314.01935],
                              [201.26117, 371.41043], [313.08905, 371.15118]])
BORDER_GRAY = (135, 133, 132)
CONF_THRESHOLD = 0.8
NMS_THRESHOLD = 0.4


def _cv2():
    import cv2
    return cv2


def nms(boxes: torch.Tensor, scores: torch.Tensor, iou_threshold: float) -> torch.Tensor:
    """Greedy NMS with torchvision.ops.nms semantics: boxes (x1, y1, x2, y2) fp32, visited in descending score order,
    a box is dropped when its IoU (no +1) with a kept box exceeds the threshold. Returns kept indices, best first."""
    order = torch.argsort(scores, descending=True, stable=True)
    b = boxes[order].float()
    area = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    alive = torch.ones(len(order), dtype=torch.bool, device=boxes.device)
    keep = []
    for i in range(len(order)):
        if not bool(alive[i]):
            continue
        keep.append(i)
        r = b[i + 1:]
        w = (torch.minimum(b[i, 2], r[:, 2]) - torch.maximum(b[i, 0], r[:, 0])).clamp(min=0)
        h = (torch.minimum(b[i, 3], r[:, 3]) - torch.maximum(b[i, 1], r[:, 1])).clamp(min=0)
        inter = w * h
        alive[i + 1:] &= ~(inter / (area[i] + area[i + 1:] - inter) > iou_threshold)
    return order[torch.tensor(keep, dtype=torch.int64, device=boxes.device)]


def select_faces(boxes: torch.Tensor, scores: torch.Tensor, landmarks: torch.Tensor,
                 conf_threshold: float = CONF_THRESHOLD, nms_threshold: float = NMS_THRESHOLD) -> np.ndarray:
    """detect_faces' post-processing: score > threshold, descending score, NMS -> float32 rows
    [x1, y1, x2, y2, score, l1x, l1y, ..., l5x, l5y]. Equal scores are ordered as facexlib's `argsort()[::-1]`
    orders them (reverse index order), so a tie keeps the same box as the reference."""
    idx = torch.nonzero(scores > conf_threshold).flatten()
    boxes, scores, landmarks = boxes[idx].cpu(), scores[idx].cpu(), landmarks[idx].cpu()
    order = torch.argsort(scores, stable=True).flip(0)
    boxes, scores, landmarks = boxes[order], scores[order], landmarks[order]
    keep = nms(boxes, scores, nms_threshold)
    rows = torch.cat([boxes[keep], scores[keep, None], landmarks[keep]], 1)
    return rows.float().cpu().numpy()


class FaceRestoreHelper:
    def __init__(self, device="cuda", upscale_factor: int = 1, face_size: int = 512, use_parse: bool = True,
                 det_model: str = "retinaface_resnet50", detector: Optional[Callable] = None,
                 parser: Optional[Callable] = None) -> None:
        if detector is None or parser is None:
            raise ValueError("FaceRestoreHelper needs the detector and parser callables (e.g. the engines'"
                             " RetinaFaceEngine.candidates and ParseNetEngine.masks)")
        if int(upscale_factor) != 1 or not use_parse or det_model != "retinaface_resnet50":
            raise NotImplementedError("FaceRestoreHelper: only upscale_factor=1, use_parse=True and the "
                                      "retinaface_resnet50 detector are built (the unaligned-face loop's settings)")
        self.device = device
        self.upscale_factor = 1
        self.face_size = (face_size, face_size)
        self.face_template = FACE_TEMPLATE_512 * (face_size / 512.0)
        self.detector, self.parser = detector, parser
        self.clean_all()

    def clean_all(self) -> None:
        self.all_landmarks_5: List[np.ndarray] = []
        self.det_faces: List[np.ndarray] = []
        self.affine_matrices: List[np.ndarray] = []
        self.inverse_affine_matrices: List[np.ndarray] = []
        self.cropped_faces: List[np.ndarray] = []
        self.restored_faces: List[np.ndarray] = []

    def read_image(self, img: np.ndarray) -> None:
        """img: uint8 HWC, used with its channels as given. Brought to a min side of 512 (bilinear) if smaller."""
        assert img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3, "read_image takes uint8 HWC 3-channel"
        self.input_img = img
        short = min(img.shape[:2])
        if short < 512:
            f = 512.0 / short
            self.input_img = _cv2().resize(img, (0, 0), fx=f, fy=f, interpolation=_cv2().INTER_LINEAR)

    def detect_faces(self, img: np.ndarray) -> np.ndarray:
        boxes, scores, landmarks = self.detector(img)
        return select_faces(boxes, scores, landmarks)

    def get_face_landmarks_5(self, resize: Optional[int] = 640, eye_dist_threshold: Optional[float] = 5) -> int:
        """Detect on the image scaled up so its min side is at least `resize`, map back, and keep the faces whose
        "eye distance" norm([b6 - b8, b7 - b9]) reaches the threshold. That pairs the left eye's x with its y and the
        right eye's x with its y, as the reference does; it is kept so the same faces are dropped."""
        cv2 = _cv2()
        scale = 1
        img = self.input_img
        if resize is not None:
            h, w = img.shape[:2]
            scale = max(1, resize / min(h, w))
            img = cv2.resize(img, (int(w * scale), int(h * scale)),
                             interpolation=cv2.INTER_AREA if scale < 1 else cv2.INTER_LINEAR)
        dets = self.detect_faces(img)
        if dets.shape[0] == 0:
            return 0
        dets = dets / scale
        for d in dets:
            if eye_dist_threshold is not None and np.linalg.norm([d[6] - d[8], d[7] - d[9]]) < eye_dist_threshold:
                continue
            self.all_landmarks_5.append(np.array([[d[i], d[i + 1]] for i in range(5, 15, 2)]))
            self.det_faces.append(d[0:5])
        return len(self.all_landmarks_5)

    def align_warp_face(self) -> None:
        """Similarity transform (LMEDS) of each landmark set onto the template, then the 512 crop on a gray border."""
        cv2 = _cv2()
        for lm in self.all_landmarks_5:
            m = cv2.estimateAffinePartial2D(lm, self.face_template, method=cv2.LMEDS)[0]
            self.affine_matrices.append(m)
            self.cropped_faces.append(cv2.warpAffine(self.input_img, m, self.face_size, borderMode=cv2.BORDER_CONSTANT,
                                                     borderValue=BORDER_GRAY))

    def get_inverse_affine(self) -> None:
        cv2 = _cv2()
        for m in self.affine_matrices:
            self.inverse_affine_matrices.append(cv2.invertAffineTransform(m) * self.upscale_factor)

    def add_restored_face(self, face: np.ndarray) -> None:
        self.restored_faces.append(face)

    def parse_faces(self, faces: Sequence[np.ndarray]) -> List[np.ndarray]:
        """Parse masks (uint8 {0, 255}) of restored faces, all in one call of the parser."""
        cv2 = _cv2()
        return list(self.parser([cv2.resize(f, (512, 512), interpolation=cv2.INTER_LINEAR) for f in faces])) \
            if len(faces) else []

    def paste_faces_to_input_image(self, upsample_img: np.ndarray,
                                   parse_masks: Optional[Sequence[np.ndarray]] = None) -> np.ndarray:
        """Blend every restored face into `upsample_img` (resized to the detection image with Lanczos) through
        min(parse mask, soft square mask); `parse_masks` may hold the restored faces' masks already parsed."""
        cv2 = _cv2()
        h, w = self.input_img.shape[:2]
        out = cv2.resize(upsample_img, (w, h), interpolation=cv2.INTER_LANCZOS4)
        assert len(self.restored_faces) == len(self.inverse_affine_matrices), \
            "length of restored_faces and affine_matrices are different."
        if parse_masks is None:
            parse_masks = self.parse_faces(self.restored_faces)
        for face, inv, parsed in zip(self.restored_faces, self.inverse_affine_matrices, parse_masks):
            inv_restored = cv2.warpAffine(face, inv, (w, h))
            square = cv2.warpAffine(np.ones(self.face_size, dtype=np.float32), inv, (w, h))
            square = cv2.erode(square, np.ones((2, 2), np.uint8))           # drop the black border of the warp
            pasted = square[:, :, None] * inv_restored
            edge = int(np.sum(square) ** 0.5) // 20
            soft = cv2.erode(square, np.ones((2 * edge, 2 * edge), np.uint8))
            soft = cv2.GaussianBlur(soft, (2 * edge + 1, 2 * edge + 1), 0)[:, :, None]
            pm = parsed.astype(np.float64)
            pm = cv2.GaussianBlur(pm, (101, 101), 11)
            pm = cv2.GaussianBlur(pm, (101, 101), 11)
            pm[:10, :] = 0
            pm[-10:, :] = 0
            pm[:, :10] = 0
            pm[:, -10:] = 0
            pm = cv2.resize(pm / 255., self.face_size)
            pm = cv2.warpAffine(pm, inv, (w, h), flags=3)[:, :, None]
            take = (pm < soft).astype("int")
            mask = pm * take + soft * (1 - take)
            out = mask * pasted + (1 - mask) * out
        return out.astype(np.uint8)
