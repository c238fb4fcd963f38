"""Shared by the face-loss tests: the drop-in module built offline (weight loader replaced by an empty state dict) and filled
like tools/make_golden_face_loss.py fills the reference, and an fp64 restatement of the face loss in torch ops over the same
parameters, written from the loss's definition (crop with zero fill, antialiased bilinear Resize(256), CenterCrop(254),
faces[:6], the ResNet-50 taps, the weighted L1 sums)."""
import importlib.util
import os

import torch
import torch.nn.functional as F

from conftest import GOLDEN, ROOT

_spec = importlib.util.spec_from_file_location("make_golden_face_loss", os.path.join(ROOT, "tools", "make_golden_face_loss.py"))
golden_tool = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(golden_tool)


def load_golden():
    return torch.load(os.path.join(GOLDEN, "face_loss.pt"), weights_only=False)


def build_face_loss():
    """losses.face_loss.FaceLoss() with the weight loader replaced (no weight file)."""
    import losses.face_loss as fl
    saved = fl.load_weights
    fl.load_weights = lambda path: {}
    try:
        return fl.FaceLoss()
    finally:
        fl.load_weights = saved


def seeded_face_loss(case):
    from oracle.seeded import fill_seeded
    m = build_face_loss()
    checks = fill_seeded(m, case["seed"])
    golden_tool.adjust(m, case["seed"])
    return m.eval(), checks


def case_inputs(case):
    return golden_tool.images(case["seed"], case["size"], case["batch"])


def _crop(img, x0, y0, x1, y1):
    _, h, w = img.shape
    out = img.new_zeros((img.shape[0], y1 - y0, x1 - x0))
    ya, yb, xa, xb = max(y0, 0), min(y1, h), max(x0, 0), min(x1, w)
    if yb > ya and xb > xa:
        out[:, ya - y0:yb - y0, xa - x0:xb - x0] = img[:, ya:yb, xa:xb]
    return out


def prepare(img, rec, boxes):
    """Stacked crops [gt..., gen...][:6] (None without boxes)."""
    crops = [[], []]
    for i, r, bb in zip(img, rec, boxes):
        for x0, y0, x1, y1 in (tuple(int(v) for v in b[:4]) for b in bb):
            for side, src in enumerate((i, r)):
                c = _crop(src, x0, y0, x1, y1)
                h, w = c.shape[1:]
                size = (256, int(256 * w / h)) if h <= w else (int(256 * h / w), 256)
                if size != (h, w):
                    c = F.interpolate(c[None], size=size, mode="bilinear", align_corners=False, antialias=True)[0]
                t, l = int(round((c.shape[1] - 254) / 2.0)), int(round((c.shape[2] - 254) / 2.0))
                crops[side].append(c[:, t:t + 254, l:l + 254])
    if not crops[0]:
        return None
    return torch.stack(crops[0] + crops[1])[:6]


def _bn(x, bn, dtype):
    return F.batch_norm(x, bn.running_mean.to(dtype), bn.running_var.to(dtype), bn.weight.to(dtype), bn.bias.to(dtype),
                        False, 0.0, bn.eps)


def features(m, x, dtype=torch.float64):
    """The five taps of the ResNet-50 of module m on crops x."""
    def conv(h, c):
        return F.conv2d(h, c.weight.to(dtype), None, c.stride, c.padding)
    x = x.to(dtype)
    f0 = conv(x, m.conv1)
    h = F.max_pool2d(F.relu(_bn(f0, m.bn1, dtype)), 3, 2, 0, ceil_mode=True)
    out = [f0]
    for layer in (m.layer1, m.layer2, m.layer3, m.layer4):
        for blk in layer:
            r = h if blk.downsample is None else _bn(conv(h, blk.downsample[0]), blk.downsample[1], dtype)
            y = F.relu(_bn(conv(h, blk.conv1), blk.bn1, dtype))
            y = F.relu(_bn(conv(y, blk.conv2), blk.bn2, dtype))
            h = F.relu(_bn(conv(y, blk.conv3), blk.bn3, dtype) + r)
        out.append(h)
    return out


def restated_loss(m, img, rec, boxes, signs=None, dtype=torch.float64):
    """(crops, features, level terms, loss) of the face loss in `dtype`. signs: optional per-level sign patterns [P, C, H, W]
    of (a - b); the loss then takes sum signs * (a - b) in place of |a - b| (same value where the signs agree, and the
    gradient seeded with those signs)."""
    x = prepare(img.to(dtype), rec.to(dtype), boxes)
    if x is None:
        return None
    feats = features(m, x, dtype)
    terms = []
    for l, (a, f) in enumerate(zip(m.alphas, feats)):
        p, q = f.chunk(2)
        d = (p - q) if signs is None else signs[l].to(dtype) * (p - q)
        terms.append(a * (d.abs() if signs is None else d).sum(dim=0).mean())
    return x, feats, terms, sum(terms)
