"""Upsample / Downsample convolutions of the VQ-IMG model (bench.IMG_CFG) at batch 32, 256x256: times the forward, data
gradient and weight gradient of every such layer through ops.Conv3x3Fn exactly as the model launches them (shadow
conversions, weight packing, space-to-depth, sum-pool, unpack helpers included), once per route: MAS_CONV_PHASE=0 (the
register-staged kernels over the nearest-x2 / space-to-depth maps) and MAS_CONV_PHASE=1 (phase-decomposed, TMA-fed fp16:
shift_gemm_t16 for the forward and data gradient, wgrad_t16 + conv_wgrad_fold16 / conv_wgrad_reduce for the weight gradient).
The dy passed to the backward has no fp16 shadow here, so both backward passes include its amax and fp16 conversion.
TFLOP/s are against the REFERENCE FLOP count of the layer, 2 * N * Hout * Wout * C * C * 9 per pass (what nn.Conv2d does
on the upsampled / padded map), not against what either route executes. Layer shapes come from a batch-1 forward of the
model with hooks on its Upsample / Downsample modules.
Usage: python tools/bench_resample.py [--batch B] [--iters I] [--routes 0,1] [--json FILE]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "make-a-scene_b200"), os.path.join(ROOT, "tools")]
import torch  # noqa: E402

import bench  # noqa: E402
from bench_wgrad import card  # noqa: E402
from mas_b200 import _lib as L, ops  # noqa: E402
from models.modules import Downsample, Upsample  # noqa: E402


def resample_shapes(dev):
    """(kind, C, H_in, W_in) of every Upsample / Downsample in model order."""
    m = bench.build_model().to(dev)
    seen = []

    def hook(kind):
        return lambda mod, inp: seen.append((kind, inp[0].shape[1], inp[0].shape[2], inp[0].shape[3]))

    hs = [mod.register_forward_pre_hook(hook("up" if isinstance(mod, Upsample) else "down"))
          for mod in m.modules() if isinstance(mod, (Upsample, Downsample))]
    with torch.no_grad():
        m(torch.rand(1, 3, bench.RES, bench.RES, device=dev))
    for h in hs:
        h.remove()
    del m
    torch.cuda.empty_cache()
    return seen


class _Ctx:
    """Stand-in for the autograd context, so that one pass of Conv3x3Fn can be timed on its own."""

    def __init__(self, needs):
        self.needs_input_grad = needs

    def save_for_backward(self, *t):
        self.saved_tensors = t


def time_layer(kind, c, h, w, B, iters, dev):
    mode = L.CONV_UP if kind == "up" else L.CONV_S2
    g = torch.Generator(device=dev).manual_seed(11)
    x = torch.randn(B, c, h, w, device=dev, generator=g).contiguous(memory_format=torch.channels_last)
    wt = torch.randn(c, c, 3, 3, device=dev, generator=g) * 0.03
    b = torch.randn(c, device=dev, generator=g) * 0.1
    ho, wo = (2 * h, 2 * w) if kind == "up" else (h // 2, w // 2)
    dy = torch.randn(B, c, ho, wo, device=dev, generator=g).contiguous(memory_format=torch.channels_last) * 1e-4
    grads = (True, True, True, False, False, False)

    def fwd():
        ctx = _Ctx(grads)
        return ctx, ops.Conv3x3Fn.forward(ctx, x, wt, b, None, mode, False)

    ctx, _ = fwd()
    out = {"fwd": bench.time_kernel(fwd, iters=iters, warm=3)}
    for name, needs in (("dgrad", (True, False, False, False, False, False)), ("wgrad", (False, True, True, False, False, False))):
        ctx.needs_input_grad = needs
        out[name] = bench.time_kernel(lambda: ops.Conv3x3Fn.backward(ctx, dy), iters=iters, warm=3)
    return out, 2.0 * B * ho * wo * c * c * 9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=bench.BATCH)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--routes", default="0,1", help="values of MAS_CONV_PHASE to time, in this order")
    ap.add_argument("--json", default=None, help="also write the rows to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_resample.py needs a GPU")
    dev = torch.device("cuda:0")
    name, q = card()
    print("card: %s | power.limit, clocks.max.sm: %s" % (name, q))
    print("TFLOP/s below are against the reference FLOP count 2*N*Hout*Wout*C*C*9 per pass")
    B = args.batch
    routes = [r.strip() for r in args.routes.split(",") if r.strip()]
    rows = []
    print("%4s %4s %4s %5s | %5s | %9s %9s %9s | %7s %7s %7s" % ("kind", "C", "Hin", "route", "B", "fwd ms", "dgrad ms",
                                                               "wgrad ms", "fwd TF", "dgr TF", "wgr TF"))
    for kind, c, h, w in resample_shapes(dev):
        for r in routes:
            os.environ["MAS_CONV_PHASE"] = r
            t, flop = time_layer(kind, c, h, w, B, args.iters, dev)
            row = dict(kind=kind, c=c, h_in=h, w_in=w, route=r, batch=B, ref_flop_per_pass=flop,
                       **{k + "_ms": v * 1e3 for k, v in t.items()}, **{k + "_tflops": flop / v / 1e12 for k, v in t.items()})
            rows.append(row)
            print("%4s %4d %4d %5s | %5d | %9.3f %9.3f %9.3f | %7.1f %7.1f %7.1f" % (
                kind, c, h, r, B, row["fwd_ms"], row["dgrad_ms"], row["wgrad_ms"], row["fwd_tflops"], row["dgrad_tflops"],
                row["wgrad_tflops"]), flush=True)
            torch.cuda.empty_cache()
    for r in routes:
        tot = sum(row["fwd_ms"] + row["dgrad_ms"] + row["wgrad_ms"] for row in rows if row["route"] == r)
        print("route MAS_CONV_PHASE=%s: all Upsample / Downsample passes %.2f ms" % (r, tot))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": name, "power_limit_clocks": q, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
