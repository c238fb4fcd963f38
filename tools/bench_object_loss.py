"""The object-aware loss: losses.object_loss.ObjectLoss (one masked LPIPS pass per size class) against the per-box loop.

    python tools/bench_object_loss.py [--batch 8 32] [--size 256] [--steps 5] [--warmup 2] [--seed 0]

Boxes: per image a seeded count of 4 to 12 boxes, each side log-uniform in [16, 256] and its corner uniform so that the box
lies inside the image. Three arms, each timed for forward + backward (the data gradient of the reconstructions):
  - ObjectLoss;
  - the per-box loop of the reference's commented-out code over our losses.lpips.LPIPS (one LPIPS call per box);
  - the same loop over stock torch modules (nn.Conv2d / nn.ReLU / nn.MaxPool2d, cuDNN, PyTorch's default TF32 convolutions).
Reported per arm: ms per step, boxes per second, kernel launches of libmas_b200 per step (ours only) and peak memory.
Parameters are seeded, not pretrained: timing does not depend on their values."""
import argparse
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "make-a-scene_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]


def boxes_for(batch, size, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(batch):
        n = int(torch.randint(4, 13, (1,), generator=g))
        bb = []
        for _ in range(n):
            h, w = (int(round(math.exp(math.log(16) + float(torch.rand(1, generator=g)) * math.log(size / 16)))) for _ in range(2))
            y0 = int(torch.randint(0, size - h + 1, (1,), generator=g))
            x0 = int(torch.randint(0, size - w + 1, (1,), generator=g))
            bb.append([x0, y0, x0 + w, y0 + h])
        out.append(bb)
    return out


def loop_loss(model, images, recs, boxes):
    """loss_img.py's commented-out object loss with `self.object_loss` = model (crops inside the image: plain slicing)."""
    total = images.new_tensor(0)
    for img, rec, bboxes in zip(images, recs, boxes):
        s = img.new_tensor(0)
        for x0, y0, x1, y1 in bboxes:
            s = s + model(img[None, :, y0:y1, x0:x1].contiguous(), rec[None, :, y0:y1, x0:x1].contiguous()).mean()
        total = total + s / (len(bboxes) + 1)
    return total


def timed(fn, rec, steps, warmup):
    from mas_b200 import _lib
    for _ in range(warmup):
        fn().backward()
        rec.grad = None
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    l0 = _lib.launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn().backward()
        rec.grad = None
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, (_lib.launch_count() - l0) / steps, (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="+", default=[8, 32])
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_object_loss needs a CUDA device")
    from bench_lpips import Stock
    from lpips_common import seeded_lpips
    from losses.object_loss import ObjectLoss
    from mas_b200 import ops
    dev = torch.device("cuda:0")
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True).stdout.strip()
    except OSError:
        pl = "unknown"
    print("GPU: %s | power limit, max SM clock, SM clock: %s" % (torch.cuda.get_device_name(0), pl))
    m, _ = seeded_lpips({"seed": 21, "bias5_3": 0.0})
    m.to(dev)
    obj, stock = ObjectLoss(m), Stock(m).to(dev)
    for batch in a.batch:
        g = torch.Generator().manual_seed(a.seed + batch)
        img = (torch.rand(batch, 3, a.size, a.size, generator=g) * 2 - 1).to(dev)
        rec = (torch.rand(batch, 3, a.size, a.size, generator=g) * 2 - 1).to(dev).requires_grad_(True)
        boxes = boxes_for(batch, a.size, a.seed + batch)
        plan = ops.ObjectPlan(img.shape, rec.shape, boxes)
        print("batch %d, %dx%d: %d boxes in %d size classes" % (batch, a.size, a.size, plan.K, len(plan.classes)))
        arms = (("ObjectLoss", lambda: obj(img, rec, boxes)), ("loop, our LPIPS", lambda: loop_loss(m, img, rec, boxes)),
                ("loop, stock", lambda: loop_loss(stock, img, rec, boxes)))
        for name, fn in arms:
            ms, launches, peak = timed(fn, rec, a.steps, a.warmup)
            print("  %-16s %9.2f ms  %9.1f boxes/s  %7.0f launches  peak +%8.1f MiB"
                  % (name, ms, plan.K / ms * 1e3, launches, peak) if name != "loop, stock" else
                  "  %-16s %9.2f ms  %9.1f boxes/s  %7s launches  peak +%8.1f MiB" % (name, ms, plan.K / ms * 1e3, "-", peak))


if __name__ == "__main__":
    main()
