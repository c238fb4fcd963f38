"""Times the PatchGAN discriminator work of one VQ-IMG training step (the reference's train.py:84-98 with
losses/loss_img.py) on losses.discriminator (the sm_90a kernels) and on the stock torch.nn modules (cuDNN, PyTorch's
default TF32 settings), alternating the two paths over --rounds rounds on the same GPU:

  fwd3   D(real), D(fake) with D trainable, D(rec) with D frozen           3 forwards
  d_bwd  hinge loss backward: weight gradients of every layer, data gradients of all but the first      (discriminator step)
  g_bwd  autograd.grad(-mean D(rec), rec, retain_graph=True), then backward(): two data-gradient passes (generator step)

TFLOP/s are against the algorithmic FLOPs of each pass (2 * MACs of the convolutions; a weight gradient or a data
gradient costs what the layer's forward costs).  A per-layer breakdown of the new path follows, from CUDA events around
every C-ABI call.  Prints one JSON line at the end.

    python tools/bench_discriminator.py [--batch 32] [--size 256] [--iters 5] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "make-a-scene_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import torch  # noqa: E402
from torch import nn  # noqa: E402


def layer_flops(batch, size):
    """Forward FLOPs of model.0, .2, .5, .8, .11 (2 * N * Hout * Wout * Cout * Cin * 16)."""
    out, h, cin = [], size, 3
    for cout, s in ((64, 2), (128, 2), (256, 2), (512, 1), (1, 1)):
        h = (h - 2) // s + 1
        out.append(2.0 * batch * h * h * cout * cin * 16)
        cin = cout
    return out


def stock(ours):
    """The reference's module graph (stock nn.Conv2d / BatchNorm2d / LeakyReLU) with the same weights."""
    layers = []
    for m in ours.model:
        if isinstance(m, nn.Conv2d):
            layers.append(nn.Conv2d(m.in_channels, m.out_channels, 4, m.stride, 1, bias=m.bias is not None))
        elif isinstance(m, nn.BatchNorm2d):
            layers.append(nn.BatchNorm2d(m.num_features))
        else:
            layers.append(nn.LeakyReLU(0.2, m.inplace))
    ref = nn.Module()
    ref.model = nn.Sequential(*layers)
    ref.load_state_dict(ours.state_dict())
    ref.forward = lambda x: ref.model(x)
    return ref


def step(D, real, fake, ev):
    """One step's discriminator work; ev: four CUDA events bracketing fwd3 / d_bwd / g_bwd (recorded in order)."""
    for p in D.parameters():
        p.requires_grad_(True)
        p.grad = None
    rec = fake.clone().requires_grad_(True)
    ev[0].record()
    lr, lf = D(real), D(fake)
    for p in D.parameters():
        p.requires_grad_(False)
    lg = D(rec)
    ev[1].record()
    loss_d = 0.5 * (torch.relu(1.0 - lr).mean() + torch.relu(1.0 + lf).mean())
    loss_d.backward()
    ev[2].record()
    g_loss = -torch.mean(lg)
    torch.autograd.grad(g_loss, rec, retain_graph=True)
    g_loss.backward()
    ev[3].record()


def time_path(D, real, fake, iters):
    tot = [0.0, 0.0, 0.0]
    for _ in range(iters):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        step(D, real, fake, ev)
        torch.cuda.synchronize()
        for k in range(3):
            tot[k] += ev[k].elapsed_time(ev[k + 1])
    return [t / iters for t in tot]


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the card name from torch is still reported
        return "%s (nvidia-smi unavailable: %s)" % (torch.cuda.get_device_name(0), e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_discriminator: needs a CUDA device")
    from mas_b200 import _lib
    from losses import discriminator as Dm
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    ours = Dm.Discriminator()
    ours.apply(Dm.weights_init)
    ref = stock(ours)
    ours.to(dev).train()
    ref.to(dev).train()
    g = torch.Generator().manual_seed(1)
    real = torch.rand(a.batch, 3, a.size, a.size, generator=g).to(dev)
    fake = torch.rand(a.batch, 3, a.size, a.size, generator=g).to(dev)

    F = layer_flops(a.batch, a.size)
    sF = sum(F)
    pass_flops = [3 * sF, 2 * sF + 2 * (sF - F[0]), 2 * sF]
    names = ["fwd3", "d_bwd", "g_bwd"]
    print("GPU:", gpu_info())
    print("batch %d, %dx%d; GFLOP per pass: %s" % (a.batch, a.size, a.size,
                                                   ", ".join("%s %.0f" % (n, f / 1e9) for n, f in zip(names, pass_flops))))
    for D in (ours, ref):       # warm-up: module loads, cuDNN algorithm choice, weight packing
        time_path(D, real, fake, 2)
    res = {"ours": [], "cudnn": []}
    for r in range(a.rounds):
        for tag, D in (("ours", ours), ("cudnn", ref)):
            ms = time_path(D, real, fake, a.iters)
            res[tag].append(ms)
            print("round %d %-6s " % (r, tag) + "  ".join("%s %8.2f ms (%6.1f TFLOP/s)" % (n, t, f / t / 1e9)
                                                          for n, t, f in zip(names, ms, pass_flops))
                  + "  total %8.2f ms" % sum(ms))

    _lib.profile_start()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    step(ours, real, fake, ev)
    prof = _lib.profile_report()
    print("\nper C-ABI entry and shape (new path, one step): calls, ms")
    for k, (c, t) in sorted(prof.items(), key=lambda kv: -kv[1][1]):
        print("  %-48s %4d %9.3f" % (k, c, t))
    out = {"gpu": gpu_info(), "batch": a.batch, "size": a.size, "pass_gflop": dict(zip(names, [f / 1e9 for f in pass_flops])),
           "ms": {tag: [dict(zip(names, ms)) for ms in v] for tag, v in res.items()}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
