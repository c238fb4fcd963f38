"""Shared by the object-loss tests: the golden fixture, the drop-in module with a fixture case's LPIPS parameters, and the
per-box loop of the fixture tool restated in plain torch ops (crop as zero-padding / slicing, LPIPS from lpips_common)."""
import importlib.util
import os

import torch
import torch.nn.functional as F

from conftest import GOLDEN, ROOT
from lpips_common import golden_tool, reference_lpips, seeded_lpips

_spec = importlib.util.spec_from_file_location("make_golden_object_loss", os.path.join(ROOT, "tools", "make_golden_object_loss.py"))
object_tool = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(object_tool)


def load_golden():
    return torch.load(os.path.join(GOLDEN, "object_loss.pt"), weights_only=False)


def case_module(case):
    """(ObjectLoss over the case's seeded LPIPS, that LPIPS)."""
    from losses.object_loss import ObjectLoss
    m, _ = seeded_lpips(dict(seed=case["seed"], bias5_3=0.0))
    return ObjectLoss(m), m


def case_images(case):
    return golden_tool.images(case["seed"], case["size"], case["batch"])


def crop(x, top, left, h, w):
    """torchvision's crop of [C, H, W] x: zeros where the box leaves the image (negative padding crops)."""
    H, W = x.shape[-2:]
    return F.pad(x, (-left, left + w - W, -top, top + h - H))


def restated_loop(m, images, recs, kept, dtype=torch.float64):
    """(loss, per-box p) of the per-box loop over kept boxes [[x0, y0, x1, y1], ...] per image, in `dtype`."""
    total, ps = 0, []
    for img, rec, bboxes in zip(images, recs, kept):
        s = 0
        for x0, y0, x1, y1 in bboxes:
            p = reference_lpips(m, crop(img, y0, x0, y1 - y0, x1 - x0)[None], crop(rec, y0, x0, y1 - y0, x1 - x0)[None],
                                dtype=dtype).mean()
            ps.append(p)
            s = s + p
        total = total + s / (len(bboxes) + 1)
    return total, torch.stack(ps)
