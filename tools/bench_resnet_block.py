"""Forward convolutions of the VQ-IMG model's ResnetBlocks (bench.IMG_CFG at 256x256, batch 32) on the TMA-fed fp16 kernel
(shift_gemm_t16, csrc/conv_tma.cu), timed with CUDA events: conv1's form (bias + GroupNorm-statistics epilogue) and conv2's
form (bias + residual + statistics), each as ops.conv3x3_h_raw launches it. The residual form's extra time over the bias
form is what staging the residual costs; TFLOP/s count 2 * N * H * W * Cin * Cout * 9 per launch, GB/s the fp16 input, the
fp32 output and (conv2) the fp32 residual. Each time is the median of --repeats windows of --iters launches, the two forms
alternating window by window; the min-max range over the windows is printed beside it as the spread.
Usage: python tools/bench_resnet_block.py [--batch B] [--iters I] [--repeats R] [--json FILE]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "make-a-scene_b200"), os.path.join(ROOT, "tools")]
import torch  # noqa: E402

from bench_wgrad import card  # noqa: E402
from mas_b200 import ops  # noqa: E402

# (cin, cout, h): the distinct 3x3 convolutions of the model's ResnetBlocks at 256^2 (conv1 of a block changing the width
# reads cin channels, conv2 always cout)
SHAPES = [(128, 128, 256), (128, 128, 128), (128, 256, 64), (256, 256, 64), (256, 512, 32), (512, 512, 32), (512, 512, 16)]


def _ms(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--json")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_resnet_block.py needs a CUDA device"
    dev = torch.device("cuda:0")
    ops.set_operand_format("f16")
    rows = []
    print(card())
    for cin, cout, h in SHAPES:
        n = args.batch
        g = torch.Generator(device=dev).manual_seed(cin + cout + h)
        x16 = ops.to_half(torch.randn(n, cin, h, h, device=dev, generator=g).contiguous(memory_format=torch.channels_last))
        wt = torch.randn(cout, cin, 3, 3, device=dev, generator=g) * 0.03
        b = torch.randn(cout, device=dev, generator=g) * 0.1
        res = torch.randn(n, cout, h, h, device=dev, generator=g).contiguous(memory_format=torch.channels_last)
        flop = 2.0 * n * h * h * cin * cout * 9
        act = n * h * h * cout * 4
        row = {"cin": cin, "cout": cout, "hw": h, "batch": n}
        forms = (("bias", None), ("residual", res))
        for _, r in forms:    # warm-up: module load, weight packing
            for _ in range(3):
                ops.conv3x3_h_raw(x16, wt, b, r, want_stats=True)
        torch.cuda.synchronize()
        times = {name: [] for name, _ in forms}
        for _ in range(args.repeats):
            for name, r in forms:
                times[name].append(_ms(lambda: ops.conv3x3_h_raw(x16, wt, b, r, want_stats=True), args.iters))
        for name, r in forms:
            ts = sorted(times[name])
            ms = ts[len(ts) // 2]
            nbytes = n * h * h * cin * 2 + act * (2 if r is not None else 1)
            row[name + "_ms"], row[name + "_ms_min"], row[name + "_ms_max"] = ms, ts[0], ts[-1]
            row[name + "_tflops"] = flop / ms * 1e-9
            row[name + "_gbs"] = nbytes / ms * 1e-6
        rows.append(row)
        print("%4d -> %4d @ %3d^2 x %d: bias+stats %7.3f ms [%.3f-%.3f] (%4.0f TFLOP/s)   residual+stats %7.3f ms [%.3f-%.3f] "
              "(%4.0f TFLOP/s, %4.0f GB/s)"
              % (cin, cout, h, n, row["bias_ms"], row["bias_ms_min"], row["bias_ms_max"], row["bias_tflops"], row["residual_ms"],
                 row["residual_ms_min"], row["residual_ms_max"], row["residual_tflops"], row["residual_gbs"]), flush=True)
        del x16, res
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card(), "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
