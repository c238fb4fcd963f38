"""Weight gradient vs forward convolution, per ResnetBlock 3x3 layer of the VQ-IMG model (bench.IMG_CFG) at batch 32, 256x256:
times wgrad_t16 (+ its split-K reduction, as the model launches it) and shift_gemm_t16 on the same shape with CUDA events and
prints TFLOP/s of both and their ratio. Both do 2 * N * H * W * Cin * Cout * 9 FLOPs. The layer shapes come from a batch-1
forward of the model with hooks on its ResnetBlocks, so they follow the configuration.
Usage: python tools/bench_wgrad.py [--batch B] [--iters I] [--json FILE]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "make-a-scene_b200")]
import torch  # noqa: E402

import bench  # noqa: E402
from mas_b200 import _lib as L, ops  # noqa: E402
from models.modules import ResnetBlock  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = "nvidia-smi unavailable (%s)" % e
    return name, q


def resnet_conv_shapes(dev):
    """(Cin, Cout, H, W) -> number of 3x3 stride-1 convolutions of that shape in the model's ResnetBlocks."""
    m = bench.build_model().to(dev)
    seen = []

    def hook(mod, inp):
        _, cin, h, w = inp[0].shape
        cout = mod.conv1.weight.shape[0]
        seen.append((cin, cout, h, w))
        seen.append((cout, cout, h, w))

    hs = [mod.register_forward_pre_hook(hook) for mod in m.modules() if isinstance(mod, ResnetBlock)]
    with torch.no_grad():
        m(torch.rand(1, 3, bench.RES, bench.RES, device=dev))
    for h in hs:
        h.remove()
    del m
    torch.cuda.empty_cache()
    counts = {}
    for s in seen:
        counts[s] = counts.get(s, 0) + 1
    return counts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=bench.BATCH)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--json", default=None, help="also write the rows to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_wgrad.py needs a GPU")
    if not (ops.f16_operands() and ops.conv_tma_on()):
        raise SystemExit("the fp16-shadow kernels are switched off (MAS_CONV_TMA / operand format): nothing to time")
    dev = torch.device("cuda:0")
    name, q = card()
    print("card: %s | power.limit, clocks.max.sm: %s" % (name, q))
    B = args.batch
    rows = []
    print("%5s %5s %4s %4s %3s | %9s %9s | %8s %8s | %6s" % ("Cin", "Cout", "H", "W", "n", "wgrad ms", "fprop ms", "wgrad TF", "fprop TF", "ratio"))
    for (cin, cout, h, w), n in sorted(resnet_conv_shapes(dev).items(), key=lambda kv: (-kv[0][2], kv[0][0], kv[0][1])):
        g = torch.Generator(device=dev).manual_seed(7)
        x = torch.randn(B, cin, h, w, device=dev, generator=g).contiguous(memory_format=torch.channels_last)
        x16 = ops.to_half(x)
        del x
        wt = torch.randn(cout, cin, 3, 3, device=dev, generator=g) * 0.03
        b = torch.zeros(cout, device=dev)
        y = torch.empty(B, cout, h, w, device=dev).contiguous(memory_format=torch.channels_last)
        wpk = ops._packed_conv_weight(wt, wt, cout, cin, False, dev, False, True)
        ffn = lambda: L.call("mas_conv3x3_fprop_tc16h", x16, L.t4(x16), wpk, b, None, y, L.t4(y), None, None)  # noqa: E731
        t_f = bench.time_kernel(ffn, iters=args.iters, warm=3)
        del y
        dy = torch.randn(B, cout, h, w, device=dev, generator=g).contiguous(memory_format=torch.channels_last) * 1e-6
        am = ops.amax(dy)
        dy16 = ops.to_half(dy, am)
        del dy
        gfn = lambda: ops.conv3x3_wgrad_raw(x16, dy16, cout, cin, L.CONV_S1, dy_amax=am)  # noqa: E731
        t_w = bench.time_kernel(gfn, iters=args.iters, warm=3)
        del x16, dy16
        flop = 2.0 * B * h * w * cin * cout * 9
        r = dict(cin=cin, cout=cout, h=h, w=w, layers=n, batch=B, wgrad_ms=t_w * 1e3, fprop_ms=t_f * 1e3,
                 wgrad_tflops=flop / t_w / 1e12, fprop_tflops=flop / t_f / 1e12, ratio=t_f / t_w)
        rows.append(r)
        print("%5d %5d %4d %4d %3d | %9.3f %9.3f | %8.1f %8.1f | %6.3f" % (cin, cout, h, w, n, r["wgrad_ms"], r["fprop_ms"],
                                                                       r["wgrad_tflops"], r["fprop_tflops"], r["ratio"]), flush=True)
    tw = sum(r["wgrad_ms"] * r["layers"] for r in rows)
    tf = sum(r["fprop_ms"] * r["layers"] for r in rows)
    print("all ResnetBlock 3x3 layers, one pass each: wgrad %.2f ms, fprop %.2f ms (ratio %.3f)" % (tw, tf, tf / tw))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": name, "power_limit_clocks": q, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
