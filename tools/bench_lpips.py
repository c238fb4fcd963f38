"""LPIPS at the VQ-IMG training shape: the drop-in losses.lpips against stock PyTorch modules with the same weights.

    python tools/bench_lpips.py [--batch 32] [--size 256] [--steps 10] [--warmup 3] [--profile]

Both arms time loss_img.py's sequence per step: the forward on (images, reconstructions), the data gradient by
autograd.grad(retain_graph=True), then backward(). The stock arm is nn.Conv2d / nn.ReLU / nn.MaxPool2d with the head in
torch ops (cuDNN, PyTorch's default TF32 convolutions; no torchvision needed). Parameters are seeded, not pretrained:
timing does not depend on their values. TFLOP/s are against the convolution FLOP count of the reference (both VGG passes
in the forward, one data-gradient pass over the fake half per backward). --profile adds our per-entry breakdown (CUDA
events around every C-ABI call) of one step."""
import argparse
import os
import subprocess
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "make-a-scene_b200"), os.path.join(ROOT, "tests")]

CHANNELS = [(3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256), (256, 512), (512, 512), (512, 512),
            (512, 512), (512, 512), (512, 512)]
LEVEL = [0, 0, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4]


def conv_flop(images, size):
    """2 * Cin * Cout * 9 per output pixel, per VGG pass over `images` images."""
    return sum(2.0 * ci * co * 9 * images * (size >> LEVEL[k]) ** 2 for k, (ci, co) in enumerate(CHANNELS))


class Stock(nn.Module):
    def __init__(self, m):
        super().__init__()
        layers = []
        for s in (m.vgg.slice1, m.vgg.slice2, m.vgg.slice3, m.vgg.slice4, m.vgg.slice5):
            layers.append(nn.Sequential(*[nn.ReLU() if isinstance(l, nn.ReLU) else l for l in s]))
        self.slices = nn.ModuleList(layers)
        self.lins = [lin.model[1].weight for lin in m.lins]
        self.shift, self.scale = m.scaling_layer.shift, m.scaling_layer.scale

    def forward(self, real, fake):
        def feats(x):
            h, out = (x - self.shift) / self.scale, []
            for s in self.slices:
                h = s(h)
                out.append(h)
            return out
        total = 0
        for fr, ff, w in zip(feats(real), feats(fake), self.lins):
            nr = fr / (torch.sqrt((fr ** 2).sum(1, keepdim=True)) + 1e-10)
            nf = ff / (torch.sqrt((ff ** 2).sum(1, keepdim=True)) + 1e-10)
            total = total + F.conv2d((nr - nf) ** 2, w).mean([2, 3], keepdim=True)
        return total


def step(model, real, rec):
    p = model(real, rec)
    loss = p.mean()
    torch.autograd.grad(loss, rec, retain_graph=True)
    loss.backward()
    rec.grad = None


def timed(model, real, rec, steps, warmup):
    for _ in range(warmup):
        step(model, real, rec)
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(4)] for _ in range(steps)]
    for e in ev:
        e[0].record()
        p = model(real, rec)
        loss = p.mean()
        e[1].record()
        torch.autograd.grad(loss, rec, retain_graph=True)
        e[2].record()
        loss.backward()
        e[3].record()
        rec.grad = None
    torch.cuda.synchronize()
    return [sum(e[i].elapsed_time(e[i + 1]) for e in ev) / steps for i in range(3)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lpips needs a CUDA device")
    from lpips_common import seeded_lpips
    from mas_b200 import _lib
    dev = torch.device("cuda:0")
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True).stdout.strip()
    except OSError:
        pl = "unknown"
    print("GPU: %s | power limit, max SM clock: %s" % (torch.cuda.get_device_name(0), pl))
    m, _ = seeded_lpips({"seed": 21, "bias5_3": 0.0})
    m.to(dev)
    stock = Stock(m).to(dev)
    g = torch.Generator().manual_seed(0)
    real = (torch.rand(a.batch, 3, a.size, a.size, generator=g) * 2 - 1).to(dev)
    rec = (torch.rand(a.batch, 3, a.size, a.size, generator=g) * 2 - 1).to(dev).requires_grad_(True)
    fwd_flop = conv_flop(2 * a.batch, a.size)
    bwd_flop = conv_flop(a.batch, a.size)   # data gradient of the fake half (conv1_1's data gradient counted like a forward)
    print("batch %d, %dx%d: forward %.2f TFLOP, one data-gradient pass %.2f TFLOP" % (a.batch, a.size, a.size, fwd_flop / 1e12,
                                                                                     bwd_flop / 1e12))
    res = {}
    for name, model in (("stock", stock), ("ours", m), ("stock", stock), ("ours", m)):
        res.setdefault(name, []).append(timed(model, real, rec, a.steps, a.warmup))
    for name, runs in res.items():
        for f, g1, g2 in runs:
            print("%-5s forward %8.2f ms (%6.1f TFLOP/s) | autograd.grad %8.2f ms (%6.1f TFLOP/s) | backward %7.2f ms | "
                  "step %8.2f ms" % (name, f, fwd_flop / f / 1e9, g1, bwd_flop / g1 / 1e9, g2, f + g1 + g2))
    if a.profile:
        _lib.profile_start()
        step(m, real, rec)
        rep = _lib.profile_report()
        total = sum(t for _, t in rep.values())
        print("per-entry breakdown of one step of ours (%.2f ms in C-ABI calls):" % total)
        for k, (c, t) in sorted(rep.items(), key=lambda kv: -kv[1][1]):
            print("  %-60s %3d calls %8.3f ms %5.1f%%" % (k, c, t, 100 * t / total))


if __name__ == "__main__":
    main()
