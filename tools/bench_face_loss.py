"""VGGFace2 face loss at the VQ-IMG generator-step shape: the drop-in losses.face_loss against stock PyTorch modules with the
same weights.

    python tools/bench_face_loss.py [--faces 1 3] [--size 512] [--steps 20] [--warmup 5]

Per face count n (boxes in a batch of 2 images at --size), both arms time the forward, the backward (one backward() into the
reconstructions, as loss_img.py traverses the face loss) and the whole step, with CUDA events after warm-up. The stock arm is
the module's own nn.Conv2d / nn.BatchNorm2d / nn.MaxPool2d layers (cuDNN, PyTorch's default TF32 convolutions) with the crops
by F.interpolate(antialias=True); no torchvision is needed. Parameters are seeded, not pretrained: timing does not depend on
their values. TFLOP/s are against FWD_GFLOP_6, the forward FLOP count at six crops (the run counts the stock forward with
FlopCounterMode and stops if the two differ by more than 0.1 GFLOP), scaled to the crops that run. Our per-entry breakdown
comes from CUDA events around every C-ABI call of one step; the step time not spent inside those calls is reported as host
time, with the share of it that builds the crop table (ops.FacePlan) and the folded parameters (ops.face_params)."""
import argparse
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "make-a-scene_b200"), os.path.join(ROOT, "tests")]

FWD_GFLOP_6 = 60.1     # ResNet-50 forward over six 254x254 crops (FlopCounterMode, convolutions)


def stock_loss(m, img, rec, boxes):
    from face_common import prepare
    x = prepare(img, rec, boxes)
    h = m.conv1(x)
    feats = [h]
    h = m.maxpool(torch.relu(m.bn1(h)))
    for layer in (m.layer1, m.layer2, m.layer3, m.layer4):
        for b in layer:
            r = h if b.downsample is None else b.downsample(h)
            y = torch.relu(b.bn1(b.conv1(h)))
            y = torch.relu(b.bn2(b.conv2(y)))
            h = torch.relu(b.bn3(b.conv3(y)) + r)
        feats.append(h)
    return sum(a * (p - q).abs().sum(0).mean() for a, (p, q) in zip(m.alphas, (f.chunk(2) for f in feats)))


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def boxes_for(n, size):
    per = [[], []]
    for k in range(n):
        x0, y0 = 20 + 37 * k, 30 + 29 * k
        per[k % 2].append([x0, y0, x0 + 180 + 10 * k, y0 + 220 - 8 * k])
    return per


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--faces", type=int, nargs="+", default=[1, 3])
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_face_loss needs a CUDA device")
    from face_common import golden_tool, seeded_face_loss
    from mas_b200 import _lib as L
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("device:", torch.cuda.get_device_name(0), "|", q)
    m, _ = seeded_face_loss({"seed": 41})
    m = m.to(dev)
    img, rec = golden_tool.images(41, a.size, 2)
    img, rec = img.to(dev), rec.to(dev)

    from torch.utils.flop_counter import FlopCounterMode
    with torch.no_grad(), FlopCounterMode(display=False) as fc:
        stock_loss(m, img, rec, boxes_for(3, a.size))
    counted = fc.get_total_flops() / 1e9
    print("stock forward FLOP at six crops: %.2f GFLOP (FWD_GFLOP_6 = %.1f)" % (counted, FWD_GFLOP_6))
    if abs(counted - FWD_GFLOP_6) > 0.1:
        raise SystemExit("FWD_GFLOP_6 no longer matches the counted forward (%.2f GFLOP)" % counted)

    for n in a.faces:
        boxes = boxes_for(n, a.size)
        crops = min(6, 2 * n)
        gflop = FWD_GFLOP_6 * crops / 6
        for arm, fn in (("stock", lambda r, b=boxes: stock_loss(m, img, r, b)), ("ours", lambda r, b=boxes: m(img, r, b))):
            r = rec.clone().requires_grad_(True)
            fwd = timed(lambda: fn(r), a.steps, a.warmup)

            def step():
                r.grad = None
                fn(r).backward()
            st = timed(step, a.steps, a.warmup)
            st_ours = st
            print("n=%d (%d crops) %-5s forward %.3f ms (%.0f TFLOP/s)  backward %.3f ms  step %.3f ms"
                  % (n, crops, arm, fwd, gflop / fwd, st - fwd, st))
        r = rec.clone().requires_grad_(True)
        m(img, r, boxes).backward()
        torch.cuda.synchronize()
        L.profile_start()
        r.grad = None
        m(img, r, boxes).backward()
        rep = L.profile_report()
        tot = sum(t for _, t in rep.values())
        from mas_b200 import ops
        t0 = time.perf_counter()
        for _ in range(a.steps):
            ops.FacePlan(img.shape, r.shape, boxes)
            ops.face_params(m)
        prep = (time.perf_counter() - t0) * 1e3 / a.steps
        print("n=%d host time of the step outside the calls: %.3f ms, of it crop table + folded parameters %.3f ms"
              % (n, st_ours - tot, prep))
        print("n=%d per-entry breakdown of one step (CUDA events around each call), %.3f ms in calls:" % (n, tot))
        for name, (c, t) in sorted(rep.items(), key=lambda kv: -kv[1][1]):
            print("  %-48s %4d calls %8.3f ms %5.1f%%" % (name, c, t, 100 * t / tot))


if __name__ == "__main__":
    main()
