"""FP8 against fp16 Linear kernels, for the four Linear layers of a TransformerLayer (1024 wide: qkv 3072x1024, out_proj
1024x1024, lin1 4096x1024, lin2 1024x4096) at M = 8 x 640 and 16 x 1408 rows (bench_transformer's batch and sequence, and the
VQ configs' sequence):
  * forward y = x.W^T: rows_gemm_f8<e4m3.e4m3> vs rows_gemm_t16;
  * data gradient dx = dy.W: rows_gemm_f8<e4m3.e5m2> vs rows_gemm_t16 on the transposed image;
  * weight gradient dW = dy^T.x: rows_gemm_f8 (+ split-K reduction) vs rows_wgrad_t16 (+ reduction; it also sums the bias
    gradient, which the FP8 route takes from the dy cast pass);
  * the cast passes: x -> e4m3 in both layouts, dy -> e5m2 in both layouts with the bias column sums, against mas_to_half.
Each entry is timed with CUDA events over --iters calls, FP8 and fp16 alternated over --rounds rounds (median). TFLOP/s count
2 M N K; GB/s count the fp32 read and the bytes written. The card, its power limit and the SM clocks sampled during the run are
printed beside the numbers. One JSON line per (shape, M).
Usage: python tools/bench_linear_fp8.py [--iters I] [--rounds R]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "make-a-scene_b200")]
import torch  # noqa: E402

import bench  # noqa: E402
from mas_b200 import ops  # noqa: E402

SHAPES = {"qkv": (3072, 1024), "out_proj": (1024, 1024), "lin1": (4096, 1024), "lin2": (1024, 4096)}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = "nvidia-smi unavailable (%s)" % e
    return name, q


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    os.environ["MAS_LINEAR_F16"] = "1"
    dev = torch.device("cuda:0")
    name, limits = card()
    sampler = bench.ClockSampler(0)
    sampler.start()
    rows = []
    for M in (8 * 640, 16 * 1408):
        for layer, (N, K) in SHAPES.items():
            g = torch.Generator().manual_seed(M + N + K)
            x = torch.randn(M, K, generator=g).to(dev)
            dy = (torch.randn(M, N, generator=g) * 1e-3).to(dev)
            W = (torch.randn(N, K, generator=g) * 0.03).to(dev).requires_grad_(True)
            x16, amx = ops.rows_to_half(x)
            dy16, amd = ops.rows_to_half(dy)
            w8, w8t, amw = ops.fp8_weight(W)
            x8, x8t, _, _ = ops.to_fp8(x, ops.FP8_E4M3, cols=True, am=amx)
            dy8, dy8t, _, _ = ops.to_fp8(dy, ops.FP8_E5M2, cols=True, colsum=True, am=amd)
            cases = {
                "forward": (lambda: ops.gemm_rows_f8(x8, amx, ops.FP8_E4M3, w8, amw),
                            lambda: ops.gemm_rows_f16(x16, amx, W), 2.0 * M * N * K),
                "data_grad": (lambda: ops.gemm_rows_f8(dy8, amd, ops.FP8_E5M2, w8t, amw),
                              lambda: ops.gemm_rows_f16(dy16, amd, W, True), 2.0 * M * N * K),
                "weight_grad": (lambda: ops.wgrad_rows_f8(x8t, amx, dy8t, amd, M),
                                lambda: ops.wgrad_rows_f16(x16, amx, dy16, amd, True), 2.0 * M * N * K),
                "cast_x": (lambda: ops.to_fp8(x, ops.FP8_E4M3, cols=True, am=amx),
                           lambda: ops.rows_to_half(x, amx), 4.0 * M * K + 2 * M * K),
                "cast_dy": (lambda: ops.to_fp8(dy, ops.FP8_E5M2, cols=True, colsum=True, am=amd),
                            lambda: ops.rows_to_half(dy, amd), 4.0 * M * N + 2 * M * N),
            }
            out = {"layer": layer, "M": M, "N": N, "K": K}
            for case, (f8, f16, work) in cases.items():
                t8, t16 = [], []
                for _ in range(args.rounds):
                    t8.append(timed(f8, args.iters))
                    t16.append(timed(f16, args.iters))
                t8, t16 = sorted(t8)[len(t8) // 2], sorted(t16)[len(t16) // 2]
                if case.startswith("cast"):
                    # 4 bytes read and 2 written per element either way: fp8 in two layouts, fp16 in one
                    out[case] = {"fp8_ms": t8, "fp8_GBps": work / t8 / 1e6, "fp16_ms": t16, "fp16_GBps": work / t16 / 1e6}
                else:
                    out[case] = {"fp8_ms": t8, "fp8_TFLOPs": work / t8 / 1e9, "fp16_ms": t16, "fp16_TFLOPs": work / t16 / 1e9,
                                 "speedup": t16 / t8}
            rows.append(out)
            del x, dy, W, x16, dy16, x8, x8t, dy8, dy8t, w8, w8t
            torch.cuda.empty_cache()
    clocks = sampler.stop()
    for r in rows:
        r.update(gpu=name, limits=limits, clocks=clocks)
        print(json.dumps(r))


if __name__ == "__main__":
    main()
