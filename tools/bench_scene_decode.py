"""Decoding VQ-SEG logits into compact scene maps and scoring them, at the model's own layout (the decoder's padded
channels-last view [B, 159, H, W] with channel pitch 160):

  decode:     scene.decode (mas_scene_decode) against the torch expression of the same rule on the same view (slice, argmax,
              threshold and stack; tests/test_scene_decode_cpu.py's decode_torch), checked equal;
  confusion:  scene.confusion (mas_scene_confusion) against torch.bincount over target * K + prediction per plane, checked equal;
  model:      VQBASE.decode_scene against decode_code alone, on the seg_config model (bench.py's SEG_CFG).

    python tools/bench_scene_decode.py [--batch 32] [--res 256] [--iters 20] [--rounds 5]

CUDA events over --iters calls per arm, the arms alternated over --rounds rounds; medians (min / max) of the rounds.  GB/s
are over algorithmic bytes: B*H*W*(160*4 + 4) for the decode (every float of the padded view read once, 4 bytes written),
2*B*4*H*W for the confusion, against the H100 SXM data-sheet 3.35 TB/s.  Prints the card and its power limit first."""
import argparse
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "make-a-scene_b200"), os.path.join(ROOT, "tests")]

PEAK = 3.35e12


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable (%s)" % e


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def compare(arms, iters, rounds):
    for fn in arms.values():          # warm-up: module loads, allocator, cached weight images
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            times[k].append(timed(fn, iters))
    return {k: (statistics.median(v), min(v), max(v)) for k, v in times.items()}


def report(title, res, nbytes=None):
    print(title)
    for k, (med, lo, hi) in res.items():
        bw = "" if nbytes is None else "  %7.1f GB/s (%4.1f %% of 3.35 TB/s)" % (nbytes / med / 1e6, 100 * nbytes / med / 1e-3 / PEAK)
        print("  %-28s %9.3f ms  (%.3f .. %.3f)%s" % (k, med, lo, hi, bw))


def torch_confusion(pred, target):
    out = []
    for p, k in enumerate((134, 21, 6, 2)):
        t, y = target[:, p].long(), pred[:, p].long()
        if p == 3:
            t, y = t.clamp(max=1), y.clamp(max=1)
        out.append(torch.bincount((t * k + y).flatten(), minlength=k * k))
    return torch.cat(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    from bench import SEG_CFG
    from mas_b200 import scene
    from models import VQBASE
    from test_scene_decode_cpu import decode_torch
    dev = torch.device("cuda:0")
    b, r = a.batch, a.res
    print("card:", card())
    print("batch %d, %d x %d, padded channels-last logits (pitch 160)" % (b, r, r))

    g = torch.Generator(device=dev).manual_seed(0)
    base = torch.randn((b, r, r, 160), device=dev, generator=g) * 2 - 2
    logits = base.permute(0, 3, 1, 2)[:, :159]
    got, want = scene.decode(logits), decode_torch(logits)
    assert torch.equal(got, want), "decode differs from the torch expression"
    res = compare({"scene.decode (kernel)": lambda: scene.decode(logits), "torch expression": lambda: decode_torch(logits)},
                  a.iters, a.rounds)
    report("decode", res, b * r * r * (160 * 4 + 4))

    target = scene.decode(torch.roll(logits, 1, 3))
    pred = got
    conf = scene.confusion(pred, target)
    flat = torch.cat([conf[k].flatten() for k in scene.GROUPS])
    assert torch.equal(flat, torch_confusion(pred, target)), "confusion differs from torch.bincount"
    res = compare({"scene.confusion (kernel)": lambda: scene.confusion(pred, target),
                   "torch.bincount": lambda: torch_confusion(pred, target)}, a.iters, a.rounds)
    report("confusion", res, 2 * b * 4 * r * r)
    del base, logits, got, want, target, pred

    torch.manual_seed(0)
    m = VQBASE(SEG_CFG, 1024, 256, 2000, 12500)
    with torch.no_grad():
        m.quantize.embedding.weight.normal_()
    m = m.to(dev).eval()
    f = 2 ** (len(SEG_CFG["channels"]) - 2)
    tok = torch.randint(0, 1024, (b, r // f, r // f), device=dev, generator=g)
    iters = max(1, a.iters // 4)
    with torch.no_grad():
        res = compare({"decode_code": lambda: m.decode_code(tok), "decode_scene": lambda: m.decode_scene(tok)}, iters, a.rounds)
    report("model (seg_config decoder, tokens %d x %d)" % (r // f, r // f), res)
    d = res["decode_scene"][0] - res["decode_code"][0]
    print("  decode_scene - decode_code: %.3f ms (%.1f %% of decode_code)" % (d, 100 * d / res["decode_code"][0]))


if __name__ == "__main__":
    main()
