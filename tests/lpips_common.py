"""Shared by the LPIPS tests: the drop-in module built offline (the weight sources replaced by a torch.nn VGG16 `features`
stand-in and an empty checkpoint) and filled like tools/make_golden_lpips.py fills the reference, and an fp64 LPIPS in
torch ops over the same parameters."""
import importlib.util
import os
from types import SimpleNamespace

import torch
import torch.nn as nn
import torch.nn.functional as F

from conftest import ROOT

_spec = importlib.util.spec_from_file_location("make_golden_lpips", os.path.join(ROOT, "tools", "make_golden_lpips.py"))
golden_tool = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(golden_tool)

VGG16_CFG = [64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512, "M"]


def vgg_features():
    layers, c = [], 3
    for v in VGG16_CFG:
        if v == "M":
            layers.append(nn.MaxPool2d(kernel_size=2, stride=2))
        else:
            layers += [nn.Conv2d(c, v, kernel_size=3, padding=1), nn.ReLU(inplace=True)]
            c = v
    return nn.Sequential(*layers)


def build_lpips():
    """losses.lpips.LPIPS() with the weight sources replaced (no torchvision, no network)."""
    import losses.lpips as lp
    saved = lp.vgg16, lp.get_ckpt_path, lp.load_checkpoint
    lp.vgg16 = lambda pretrained=True: SimpleNamespace(features=vgg_features())
    lp.get_ckpt_path = lambda name, root=None: "unused"
    lp.load_checkpoint = lambda path: {}
    try:
        return lp.LPIPS().eval()
    finally:
        lp.vgg16, lp.get_ckpt_path, lp.load_checkpoint = saved


def seeded_lpips(case):
    """The module with the fixture case's parameters: fill_seeded, then the tool's LPIPS adjustment."""
    from oracle.seeded import fill_seeded
    m = build_lpips()
    checks = fill_seeded(m, case["seed"])
    golden_tool.adjust(m, case["bias5_3"])
    return m, checks


def convs_of(m):
    return [(c.weight, c.bias) for s in (m.vgg.slice1, m.vgg.slice2, m.vgg.slice3, m.vgg.slice4, m.vgg.slice5)
            for c in s if isinstance(c, nn.Conv2d)]


def reference_lpips(m, real, fake, dtype=torch.float64):
    """LPIPS.forward of the reference in plain torch ops (dtype: the computation's precision)."""
    convs = [(w.to(dtype), b.to(dtype)) for w, b in convs_of(m)]
    lins = [lin.model[1].weight.to(dtype) for lin in m.lins]
    shift, scale = m.scaling_layer.shift.to(dtype), m.scaling_layer.scale.to(dtype)

    def feats(x):
        h = (x.to(dtype) - shift) / scale
        out, ci = [], 0
        for blk, n in enumerate((2, 2, 3, 3, 3)):
            if blk:
                h = F.max_pool2d(h, 2, 2)
            for _ in range(n):
                h = F.relu(F.conv2d(h, convs[ci][0], convs[ci][1], padding=1))
                ci += 1
            out.append(h)
        return out

    fr, ff = feats(real), feats(fake)
    total = 0
    for l in range(5):
        nr = fr[l] / (torch.sqrt((fr[l] ** 2).sum(1, keepdim=True)) + 1e-10)
        nf = ff[l] / (torch.sqrt((ff[l] ** 2).sum(1, keepdim=True)) + 1e-10)
        total = total + F.conv2d((nr - nf) ** 2, lins[l]).mean([2, 3], keepdim=True)
    return total
