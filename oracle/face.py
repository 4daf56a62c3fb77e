"""Plain-torch fp32 RetinaFace-ResNet50, ParseNet and facexlib's `detect_faces` post-processing, on state dicts in
facexlib's key layout (diffbir_b200.arch.retinaface_shapes / parsenet_shapes). Eval-mode BatchNorm (eps 1e-5).

These are the references the face engines are tested against and the networks behind the facexlib stand-in of
tests/golden/gen_golden_face.py."""
from itertools import product
from math import ceil

import numpy as np
import torch
import torch.nn.functional as F

from diffbir_b200.arch import RETINAFACE_CFG

DETECTOR_MEAN = (104.0, 117.0, 123.0)
# ParseNet(in_size=512, out_size=512) as facexlib builds it: (key prefix, cin, cout, scale) of every ResidualBlock
PARSENET_BLOCKS = ([("encoder.1.", 64, 128, "down"), ("encoder.2.", 128, 256, "down"), ("encoder.3.", 256, 256, "down"),
                    ("encoder.4.", 256, 256, "down")] + [(f"body.{i}.", 256, 256, "none") for i in range(10)] +
                   [("decoder.0.", 256, 256, "up"), ("decoder.1.", 256, 256, "up"), ("decoder.2.", 256, 128, "up"),
                    ("decoder.3.", 128, 64, "up")])
MASK_COLORMAP = [0, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 0, 255, 0, 0, 0]


def _bn(sd, p, x):
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"],
                        False, 0.0, 1e-5)


def _conv_bn(sd, p, x, stride=1, relu=True):
    w = sd[p + ".0.weight"]
    x = _bn(sd, p + ".1", F.conv2d(x, w, None, stride, w.shape[-1] // 2))
    return F.relu(x) if relu else x


def resnet50_body(sd, x, layers=(3, 4, 6, 3)):
    """torchvision resnet50 (v1.5) up to layer4 -> the outputs of layer2, layer3, layer4."""
    x = F.relu(_bn(sd, "body.bn1", F.conv2d(x, sd["body.conv1.weight"], None, 2, 3)))
    x = F.max_pool2d(x, 3, 2, 1)
    outs = []
    for li, blocks in enumerate(layers):
        for b in range(blocks):
            p = f"body.layer{li + 1}.{b}."
            stride = 2 if (b == 0 and li > 0) else 1
            y = F.relu(_bn(sd, p + "bn1", F.conv2d(x, sd[p + "conv1.weight"])))
            y = F.relu(_bn(sd, p + "bn2", F.conv2d(y, sd[p + "conv2.weight"], None, stride, 1)))
            y = _bn(sd, p + "bn3", F.conv2d(y, sd[p + "conv3.weight"]))
            idn = _bn(sd, p + "downsample.1", F.conv2d(x, sd[p + "downsample.0.weight"], None, stride)) if b == 0 else x
            x = F.relu(y + idn)
        if li > 0:
            outs.append(x)
    return outs


def _ssh(sd, p, x):
    c3 = _conv_bn(sd, p + "conv3X3", x, relu=False)
    c5_1 = _conv_bn(sd, p + "conv5X5_1", x)
    c5 = _conv_bn(sd, p + "conv5X5_2", c5_1, relu=False)
    c7_2 = _conv_bn(sd, p + "conv7X7_2", c5_1)
    c7 = _conv_bn(sd, p + "conv7x7_3", c7_2, relu=False)
    return F.relu(torch.cat([c3, c5, c7], 1))


def retinaface_forward(sd, x):
    """x fp32 NCHW (mean already subtracted) -> (loc [B, P, 4], class logits [B, P, 2], landmarks [B, P, 10]),
    priors in (level, row, column, anchor) order. The class logits are returned before the softmax."""
    c2, c3, c4 = resnet50_body(sd, x)
    o1 = _conv_bn(sd, "fpn.output1", c2)
    o2 = _conv_bn(sd, "fpn.output2", c3)
    o3 = _conv_bn(sd, "fpn.output3", c4)
    o2 = _conv_bn(sd, "fpn.merge2", o2 + F.interpolate(o3, size=o2.shape[2:], mode="nearest"))
    o1 = _conv_bn(sd, "fpn.merge1", o1 + F.interpolate(o2, size=o1.shape[2:], mode="nearest"))
    feats = [_ssh(sd, f"ssh{i + 1}.", f) for i, f in enumerate((o1, o2, o3))]

    def head(name, k):
        outs = []
        for i, f in enumerate(feats):
            y = F.conv2d(f, sd[f"{name}.{i}.conv1x1.weight"], sd[f"{name}.{i}.conv1x1.bias"])
            outs.append(y.permute(0, 2, 3, 1).reshape(y.shape[0], -1, k))
        return torch.cat(outs, 1)
    return head("BboxHead", 4), head("ClassHead", 2), head("LandmarkHead", 10)


def priors(h, w, cfg=None):
    """facexlib PriorBox(cfg, image_size=(h, w)).forward(): Python doubles, then a float32 tensor [P, 4]."""
    cfg = RETINAFACE_CFG if cfg is None else cfg
    anchors = []
    for step, sizes in zip(cfg["steps"], cfg["min_sizes"]):
        for i, j in product(range(ceil(h / step)), range(ceil(w / step))):
            for ms in sizes:
                anchors += [(j + 0.5) * step / w, (i + 0.5) * step / h, ms / w, ms / h]
    return torch.tensor(anchors, dtype=torch.float32).view(-1, 4)


def decode(loc, conf_logits, landm, h, w, cfg=None):
    """facexlib decode / decode_landm and the softmax score, scaled to input pixels -> (boxes [P, 4], scores [P],
    landmarks [P, 10]), fp32."""
    cfg = RETINAFACE_CFG if cfg is None else cfg
    pr = priors(h, w, cfg).to(loc.device)
    v0, v1 = cfg["variance"]
    boxes = torch.cat((pr[:, :2] + loc[:, :2] * v0 * pr[:, 2:], pr[:, 2:] * torch.exp(loc[:, 2:] * v1)), 1)
    boxes[:, :2] -= boxes[:, 2:] / 2
    boxes[:, 2:] += boxes[:, :2]
    lm = torch.cat([pr[:, :2] + landm[:, 2 * k:2 * k + 2] * v0 * pr[:, 2:] for k in range(5)], 1)
    scale = torch.tensor([w, h, w, h], dtype=torch.float32, device=loc.device)
    return boxes * scale, F.softmax(conf_logits, dim=-1)[:, 1], lm * scale.repeat(3)[:10]


def detect_candidates(sd, img):
    """The detector half of facexlib's detect_faces(img, use_origin_size=True) up to the score threshold:
    img uint8 HWC (channels used as given) -> device-independent fp32 (boxes, scores, landmarks) of every prior."""
    dev = next(iter(sd.values())).device
    x = torch.from_numpy(np.ascontiguousarray(img)).to(dev).float() - torch.tensor(DETECTOR_MEAN, device=dev)
    x = x.permute(2, 0, 1)[None].contiguous()
    with torch.no_grad():
        loc, conf, landm = retinaface_forward(sd, x)
    return decode(loc[0], conf[0], landm[0], img.shape[0], img.shape[1])


def nms_reference(boxes, scores, iou_threshold):
    """Greedy NMS with torchvision.ops.nms semantics (IoU without +1, keep in descending score order)."""
    order = torch.argsort(scores, descending=True)
    boxes = boxes.double()
    area = (boxes[:, 2] - boxes[:, 0]) * (boxes[:, 3] - boxes[:, 1])
    keep, removed = [], torch.zeros(len(order), dtype=torch.bool)
    for a in range(len(order)):
        i = order[a]
        if removed[a]:
            continue
        keep.append(int(i))
        j = order[a + 1:]
        xx1 = torch.maximum(boxes[i, 0], boxes[j, 0])
        yy1 = torch.maximum(boxes[i, 1], boxes[j, 1])
        xx2 = torch.minimum(boxes[i, 2], boxes[j, 2])
        yy2 = torch.minimum(boxes[i, 3], boxes[j, 3])
        inter = (xx2 - xx1).clamp(min=0) * (yy2 - yy1).clamp(min=0)
        removed[a + 1:] |= inter / (area[i] + area[j] - inter) > iou_threshold
    return torch.tensor(keep, dtype=torch.int64)


def detect_faces(sd, img, conf_threshold=0.8, nms_threshold=0.4, nms=nms_reference):
    """facexlib RetinaFace.detect_faces(img, conf_threshold, nms_threshold, use_origin_size=True) -> float32 numpy
    rows [x1, y1, x2, y2, score, l1x, l1y, ..., l5x, l5y]. `nms(boxes, scores, iou)` may be torchvision.ops.nms."""
    boxes, scores, landms = (t.cpu().numpy() for t in detect_candidates(sd, img))
    inds = np.where(scores > conf_threshold)[0]
    boxes, landms, scores = boxes[inds], landms[inds], scores[inds]
    order = scores.argsort()[::-1]
    boxes, landms, scores = boxes[order], landms[order], scores[order]
    dets = np.hstack((boxes, scores[:, None])).astype(np.float32, copy=False)
    keep = nms(torch.from_numpy(dets[:, :4]), torch.from_numpy(dets[:, 4]), nms_threshold).numpy()
    return np.concatenate((dets[keep], landms[keep]), axis=1)


def _conv_layer(sd, p, x, scale="none", norm=False, act=False):
    """ParseNet ConvLayer: optional nearest-2x, ReflectionPad2d(1), 3x3 conv (stride 2 for `down`), BN, LeakyReLU(0.2)."""
    if scale == "up":
        x = F.interpolate(x, scale_factor=2, mode="nearest")
    x = F.conv2d(F.pad(x, (1, 1, 1, 1), mode="reflect"), sd[p + "conv2d.weight"], sd.get(p + "conv2d.bias"),
                 2 if scale == "down" else 1)
    if norm:
        x = _bn(sd, p + "norm.norm", x)
    return F.leaky_relu(x, 0.2) if act else x


def parsenet_forward(sd, x):
    """ParseNet(in_size=512, out_size=512, parsing_ch=19) -> out_mask logits (out_img_conv is never needed)."""
    x = _conv_layer(sd, "encoder.0.", x)
    feat = None
    for p, ci, co, scale in PARSENET_BLOCKS:
        if p.startswith("body.") and feat is None:
            feat = x
        if p.startswith("decoder.") and feat is not None:
            x, feat = feat + x, None
        idn = x if (scale == "none" and ci == co) else _conv_layer(sd, p + "shortcut_func.", x, scale)
        r = _conv_layer(sd, p + "conv1.", x, "up" if scale == "up" else "none", norm=True, act=True)
        x = idn + _conv_layer(sd, p + "conv2.", r, "down" if scale == "down" else "none", norm=True)
    return _conv_layer(sd, "out_mask_conv.", x)


def parse_face(sd, face_rgb):
    """The parse step of FaceRestoreHelper.paste_faces_to_input_image for a 512x512 RGB uint8 face: img2tensor
    (bgr2rgb=True swaps it to BGR), (x - 0.5) / 0.5, ParseNet, argmax -> uint8 mask in {0, 255}."""
    dev = next(iter(sd.values())).device
    x = face_rgb[:, :, ::-1].astype("float32") / 255.
    x = torch.from_numpy(np.ascontiguousarray(x.transpose(2, 0, 1))).to(dev)
    x = ((x - 0.5) / 0.5)[None]
    with torch.no_grad():
        out = parsenet_forward(sd, x).argmax(dim=1).squeeze().cpu().numpy()
    lut = np.array(MASK_COLORMAP, dtype=np.uint8)
    return lut[out]
